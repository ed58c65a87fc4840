"""Streamed clip inference without a GPU: the frame / clip stage split of compiler.split_stages, a sliding-window run of
the two stages on the CPU plan emulator (tests/plan_emulator.py), and ClipStream.push through the product's own host
path on the stand-in device (tests/fake_cuda.py --arithmetic, with a numpy stand-in for dh_clip_window_f32 defined here).
"""
import collections
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from deephar_b200 import action, compiler, reception, spnet
from deephar_b200.config import ModelConfig, pa16j2d, pa17j3d
from deephar_b200.graph import Graph
from oracle import synth
from plan_emulator import PlanEmulator  # noqa: E402

PENN_KW = dict(num_actions=[15], num_pyramids=2, action_pyramids=[1, 2], num_levels=4, pose_replica=True,
               num_pose_features=160, num_visual_features=160)


def _c4():
    return spnet.build(ModelConfig((16, 256, 256, 3), pa16j2d, num_actions=[15], num_pyramids=6, action_pyramids=[5, 6],
                                   num_levels=4, pose_replica=True, num_pose_features=160, num_visual_features=160))


def _c5():
    return spnet.build(ModelConfig((16, 256, 256, 3), pa17j3d, num_actions=[60], num_pyramids=2, action_pyramids=[1, 2],
                                   num_levels=4, num_pose_features=192, num_visual_features=192))


def _spnet_t(T, res=128):
    return spnet.build(ModelConfig((T, res, res, 3), pa16j2d, **PENN_KW))


def _merge(pose_dim, res=64, T=None):
    if pose_dim == 2:
        pe = reception.build((res, res, 3), 16, dim=2, num_blocks=2, num_context_per_joint=2, ksize=(5, 5),
                             concat_pose_confidence=False)
        return action.build_merge_model(pe, 15, (res, res, 3), T or 16, 16, 2, pose_dim=2)
    pe = reception.build((res, res, 3), 20, dim=3, num_blocks=2, depth_maps=8, ksize=(5, 5))
    return action.build_merge_model(pe, 60, (res, res, 3), T or 20, 20, 2, pose_dim=3, depth_maps=8,
                                    num_context_per_joint=0, pose_net_version='v2', output_poses=True)


def _canon(v):
    if isinstance(v, dict):
        return tuple(sorted((k, _canon(x)) for k, x in v.items()))
    if isinstance(v, (list, tuple)):
        return tuple(_canon(x) for x in v)
    if hasattr(v, 'id') and hasattr(v, 'shape'):       # a tensor (concat copies name their source)
        return ('T', v.id)
    return v


def _tid(t):
    """tensor identity across compilations: the soft-argmax scratch outputs are made afresh by each one"""
    return t.id if t.node is None or any(o is t for o in t.node.outs) else ('scratch', t.node.id, t.out_index)


def _op_key(k):
    return (k.kind, tuple(_tid(t) for t in k.ins), tuple(_tid(t) for t in k.outs), _canon(k.attrs))


def _check_split(model, outputs=None):
    g = model.graph
    full = model.plan if outputs is None else compiler.compile_graph(g, outputs)
    st = compiler.split_stages(g, outputs)
    # the same kernel ops, no more, no fewer
    assert collections.Counter(_op_key(k) for k in st.frame.kops + st.clip.kops) == \
        collections.Counter(_op_key(k) for k in full.kops)
    assert all(t.kind == 'frame' for k in st.frame.kops for t in k.ins + k.outs)
    assert all(t.kind == 'clip' for k in st.clip.kops for t in k.outs)
    # boundary tensors are exactly the operands of the to_clip views of the selected outputs' network
    to_clip = set()
    stack, seen = list(g.outputs if outputs is None else outputs), set()
    while stack:
        t = stack.pop()
        if t.node is None or t.node.id in seen:
            continue
        seen.add(t.node.id)
        if t.node.op == 'to_clip':
            to_clip.add(t.node.inputs[0].id)
        stack.extend(t.node.inputs)
    assert to_clip and set(t.id for t in st.boundary) == to_clip
    assert set(t.id for t in st.clip.inputs) == to_clip
    sel = g.outputs if outputs is None else outputs
    assert [t for t in st.frame.outputs if t.kind == 'frame' and t in sel] == [t for t in sel if t.kind == 'frame']
    assert st.clip.outputs == [t for t in sel if t.kind == 'clip']
    for stage in (st.frame, st.clip):
        assert compiler.verify_plan(stage, stage) > 0
    return st


@pytest.mark.parametrize('build', [_c4, _c5, lambda: _merge(2), lambda: _merge(3), lambda: _spnet_t(8)],
                         ids=['c4', 'c5', 'merge_2d', 'merge_3d', 'spnet_t8'])
def test_stage_split_holds_the_full_plans_ops(build):
    m = build()
    before = [_op_key(k) for k in m.plan.kops], dict(m.plan.stats)
    st = _check_split(m)
    assert len(st.frame.kops) + len(st.clip.kops) == len(m.plan.kops)
    assert ([_op_key(k) for k in m.plan.kops], m.plan.stats) == before          # splitting leaves the model's plan alone
    assert ([_op_key(k) for k in compiler.compile_graph(m.graph).kops]) == before[0]


def test_split_of_the_action_view_skips_the_pose_outputs():
    m = _spnet_t(8)
    cfg = m.cfg
    pm, am = spnet.split_model(m, cfg)
    sel = [m.graph.outputs[i] for i in am.indices]
    st = _check_split(m, sel)
    assert not [t for t in st.frame.outputs if t in m.graph.outputs]      # only the boundary leaves the frame stage
    full = compiler.split_stages(m.graph)
    assert len(st.frame.kops) < len(full.frame.kops) and len(st.clip.kops) == len(full.clip.kops)


def test_clip_to_frame_edge_is_rejected():
    g = Graph('bad')
    g.frames_per_clip = 4
    x = g.input((1, 16, 2))
    from deephar_b200.layers import frames_to_clip
    c = frames_to_clip(x)
    y = g.op('scale', [c], c.shape, {'value': 2.0}, kind='frame')     # a clip-kind tensor feeding a frame-kind op
    g.outputs = [y]
    with pytest.raises(ValueError, match='scale op .* reads a clip-kind tensor'):
        compiler.split_stages(g)


# ---- the two stages + the window step on the plan emulator ---------------------------------------------------------------
class _Stage(object):
    """What PlanEmulator reads from a model, for one stage plan."""

    def __init__(self, model, plan):
        self.plan, self.graph, self._w = plan, model.graph, model.get_weights()

    def get_weights(self):
        return self._w


def _emulate(emu, n_frames, feeds, outputs):
    emu.n_frames = n_frames
    emu.slots = [np.full(emu._items(kind) * fl, np.nan) for (kind, fl) in emu.plan.phys]
    for t, v in feeds.items():
        emu.put(t, v)
    for k in emu.plan.kops:
        emu._step(k)
    return [emu.get(t) for t in outputs]


def test_stages_with_a_window_step_equal_the_full_plan_on_every_ready_window():
    m = _spnet_t(4).init_synthetic_weights(5)
    T, S = m.graph.frames_per_clip, 2
    st = compiler.split_stages(m.graph)
    fe, ce = PlanEmulator(_Stage(m, st.frame)), PlanEmulator(_Stage(m, st.clip))
    full = PlanEmulator(m)
    t_in = m.graph.inputs[0]
    frame_out = [t for t in m.graph.outputs if t.kind == 'frame']
    clip_out = [t for t in m.graph.outputs if t.kind == 'clip']
    n_push = 2 * T + 5
    video = synth.synth_frames(S * n_push, 128, 128, seed=9).astype(np.float64).reshape(n_push, S, 128, 128, 3)
    rings = {t.id: np.zeros((S, T) + t.shape) for t in st.boundary}
    count, pos, history = np.zeros(S, int), 0, [[] for _ in range(S)]
    resets = {3: [1], T + 2: [0], T + 4: [0, 1]}
    checked = 0
    for i in range(n_push):
        for s in resets.get(i, []):
            count[s], history[s] = 0, []
        outs = _emulate(fe, S, {t_in: video[i]}, frame_out + st.boundary)
        new = dict(zip([t.id for t in st.boundary], outs[len(frame_out):]))
        feeds = {}
        for t in st.boundary:                       # numpy restatement of dh_clip_window_f32
            r = rings[t.id]
            r[:, pos] = new[t.id]
            win = np.concatenate([r[:, (pos + 1 + j) % T][:, None] for j in range(T)], axis=1)
            feeds[t] = win.reshape((S * T,) + t.shape)
        pos = (pos + 1) % T
        clip = _emulate(ce, S * T, feeds, clip_out)
        count += 1
        for s in range(S):
            history[s].append(video[i, s])
            if count[s] < T:
                continue
            want = full.run(np.stack(history[s][-T:])[None])
            for o, t in zip(clip, clip_out):
                r = want[m.graph.outputs.index(t)][0]
                assert np.abs(o[s].reshape(r.shape) - r).max() <= 1e-10 * max(1.0, np.abs(r).max())
            for o, t in zip(outs[:len(frame_out)], frame_out):
                r = want[m.graph.outputs.index(t)][0, T - 1]
                assert np.abs(o[s].reshape(r.shape) - r).max() <= 1e-10 * max(1.0, np.abs(r).max())
            checked += 1
    assert checked == 9                             # the ready (stream, push) pairs of this reset schedule


# ---- ClipStream on the stand-in device -----------------------------------------------------------------------------------
def _clip_window(ctx, table, n, S, T, counter, stream):
    """numpy stand-in for dh_clip_window_f32 (include/deephar_b200.h), for tests/fake_cuda.py --arithmetic"""
    from deephar_b200._ffi import dh_clip_window
    import fake_cuda
    if fake_cuda.CAPTURING:          # the stand-in graph also runs what it records; on the device a captured launch
        return                       # runs on replay only, and this one advances the ring position
    cnt = np.ctypeslib.as_array(C.cast(counter, C.POINTER(C.c_int32)), shape=(2,))
    pos = int(cnt[0])
    entries = C.cast(table, C.POINTER(dh_clip_window))
    for i in range(n):
        e = entries[i]
        src, dst = fake_cuda._struct_view(e.src), fake_cuda._struct_view(e.dst)
        ring = fake_cuda._f32(e.ring, src.size * T).reshape((S, T) + src.shape[1:])
        ring[:, pos] = src
        dst.reshape((S, T) + src.shape[1:])[...] = ring[:, [(pos + 1 + j) % T for j in range(T)]]
    cnt[0] = (pos + 1) % T


def _host_path_check():
    """run under the stand-in device: ClipStream.push == Model.predict on each ready window (S = 3, staggered resets),
    CUDA-graph replay included, and the action view of split_model"""
    import torch
    from deephar_b200.stream import ClipStream
    m = _spnet_t(4).init_synthetic_weights(1234)
    T, S = 4, 3
    pm, am = spnet.split_model(m, m.cfg)
    streams = [ClipStream(m, S), ClipStream(am, S)]
    n_push = 2 * T + 1
    video = synth.synth_frames(S * n_push, 128, 128, seed=21).astype(np.float32).reshape(n_push, S, 128, 128, 3)
    hist = [[] for _ in range(S)]
    resets = {2: [1], T + 1: [2]}
    n_checked = 0
    for i in range(n_push):
        for s in resets.get(i, []):
            hist[s] = []
            for cs in streams:
                cs.reset([s])
        outs = [cs.push(torch.from_numpy(video[i])) for cs in streams]
        for s in range(S):
            hist[s].append(video[i, s])
        for cs, out in zip(streams, outs):
            assert out.ready.tolist() == [len(h) >= T for h in hist]
            for s in range(S):
                if not out.ready[s]:
                    assert all(np.isnan(o[s].numpy()).all() for o in out.clip_outputs)
                    continue
                want = m.predict(np.stack(hist[s][-T:])[None])
                sel = [want[m.graph.outputs.index(t)][0] for t in cs.clip_output_tensors]
                for o, r in zip(out.clip_outputs, sel):
                    assert np.abs(o[s].numpy() - r).max() <= 1e-5 and o[s].numpy().argmax() == r.argmax()
                fr = [want[m.graph.outputs.index(t)][0, T - 1] for t in cs.frame_output_tensors]
                for o, r in zip(out.frame_outputs, fr):
                    assert np.abs(o[s].numpy() - r).max() <= 1e-5
                n_checked += 1
    assert streams[0]._graph is not None and len(streams[1].frame_output_tensors) == 0
    assert len(streams[0].frame_output_tensors) == m.graph.num_pose_outputs
    print('host path ok: %d windows' % n_checked)


@pytest.mark.timeout(900)
def test_clip_stream_equals_predict_through_the_host_path():
    out = subprocess.run([sys.executable, os.path.abspath(__file__)], capture_output=True, text=True, timeout=880, cwd=ROOT)
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-3000:]
    assert 'host path ok' in out.stdout


def test_single_frame_model_is_rejected():
    from deephar_b200.stream import ClipStream
    m = reception.build((64, 64, 3), 16, dim=2, num_blocks=1)
    with pytest.raises(ValueError, match='single frames'):
        ClipStream(m, 2)


if __name__ == '__main__':
    sys.path.insert(0, os.path.join(ROOT, 'tests'))
    import fake_cuda
    fake_cuda.ARITHMETIC['dh_clip_window_f32'] = _clip_window
    fake_cuda.install(arithmetic=True)
    _host_path_check()
