"""Streamed clip inference on the GPU (deephar_b200/stream.py): the window kernel dh_clip_window_f32 against numpy
(bit-exact: it is a copy), and ClipStream.push against Model.predict on each ready window, with CUDA-graph replay,
launch counts and the CUDA-core fallback counter."""
import ctypes as C

import numpy as np
import pytest

from deephar_b200 import _ffi, action, compiler, reception, spnet
from deephar_b200.config import ModelConfig, pa16j2d, pa17j3d
from deephar_b200.stream import ClipStream
from oracle import synth

pytestmark = pytest.mark.gpu

PENN_KW = dict(num_actions=[15], num_pyramids=2, action_pyramids=[1, 2], num_levels=4, pose_replica=True,
               num_pose_features=160, num_visual_features=160)
NTU_KW = dict(num_actions=[60], num_pyramids=2, action_pyramids=[1, 2], num_levels=4, num_pose_features=192,
              num_visual_features=192)


# ---- the window kernel ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('T', [8, 16])
@pytest.mark.parametrize('S', [1, 3, 5])
@pytest.mark.parametrize('graph', [False, True], ids=['launches', 'graph'])
def test_window_kernel_is_an_exact_sliding_window(cuda, S, T, graph):
    torch = cuda
    ctx = _ffi.Context(torch.cuda.current_device())
    lib = _ffi.lib()
    rng = np.random.default_rng(S * 100 + T)
    # (h, w, c, src ld, src channel offset, dst ld, dst channel offset): dense, concat-resident, odd sizes
    geoms = [(1, 16, 2, 2, 0, 2, 0), (1, 16, 1, 7, 3, 1, 0), (1, 16, 160, 200, 24, 170, 5), (2, 3, 5, 9, 4, 6, 1)]
    keep, entries, srcs, dsts, rings = [], [], [], [], []
    for (h, w, c, lds, offs, ldd, offd) in geoms:
        src = torch.full((S, h, w, lds), float('nan'), device='cuda')
        dst = torch.full((S * T, h, w, ldd), float('nan'), device='cuda')
        ring = torch.zeros(S * T * h * w * c, device='cuda')
        srcs.append((src, offs, c))
        dsts.append((dst, offd, c))
        rings.append(ring)
        entries.append(_ffi.dh_clip_window(_ffi.dh_view(src.data_ptr() + 4 * offs, S, h, w, c, lds),
                                           _ffi.dh_view(dst.data_ptr() + 4 * offd, S * T, h, w, c, ldd), ring.data_ptr()))
    table = (_ffi.dh_clip_window * len(entries))(*entries)
    table_dev = torch.from_numpy(np.frombuffer(bytearray(table), np.uint8).copy()).cuda()
    counter = torch.zeros(2, dtype=torch.int32, device='cuda')
    keep += [table_dev, counter]

    def launch():
        rc = lib.dh_clip_window_f32(ctx.handle, C.c_void_p(table_dev.data_ptr()), len(entries), S, T,
                                    C.c_void_p(counter.data_ptr()), torch.cuda.current_stream().cuda_stream)
        _ffi.check(rc, 'dh_clip_window_f32')

    g = None
    if graph:
        g = torch.cuda.CUDAGraph()
        torch.cuda.synchronize()
        with torch.cuda.graph(g):
            launch()
    history = [[np.zeros((S, h, w, c), np.float32)] * T for (h, w, c, *_) in geoms]
    for step in range(2 * T + 3):
        for i, (src, offs, c) in enumerate(srcs):
            frame = rng.standard_normal((S,) + tuple(src.shape[1:3]) + (c,)).astype(np.float32)
            src[..., offs:offs + c] = torch.from_numpy(frame).cuda()
            history[i] = history[i][1:] + [frame]
        if g is not None:
            g.replay()
        else:
            launch()
        torch.cuda.synchronize()
        assert int(counter[0]) == (step + 1) % T and int(counter[1]) == 0
        for i, (dst, offd, c) in enumerate(dsts):
            got = dst[..., offd:offd + c].cpu().numpy().reshape((S, T) + history[i][0].shape[1:])
            want = np.stack(history[i], axis=1)
            assert np.array_equal(got, want), (step, i)
            # channels outside the view are untouched
            rest = np.delete(dst.cpu().numpy(), np.s_[offd:offd + c], axis=-1)
            assert np.isnan(rest).all()


# ---- ClipStream == predict ---------------------------------------------------------------------------------------------------
def _penn_t8():
    return spnet.build(ModelConfig((8, 128, 128, 3), pa16j2d, **PENN_KW))


def _ntu_t16():
    return spnet.build(ModelConfig((16, 128, 128, 3), pa17j3d, **NTU_KW))


def _merge_2d():
    pe = reception.build((128, 128, 3), 16, dim=2, num_blocks=2, num_context_per_joint=2, ksize=(5, 5),
                         concat_pose_confidence=False)
    return action.build_merge_model(pe, 15, (128, 128, 3), 16, 16, 2, pose_dim=2)


def _c4():
    return spnet.build(ModelConfig((16, 256, 256, 3), pa16j2d, num_actions=[15], num_pyramids=6, action_pyramids=[5, 6],
                                   num_levels=4, pose_replica=True, num_pose_features=160, num_visual_features=160))


def _stream_vs_predict(torch, m, S, n_push, resets, res, view=None):
    """Pushes n_push frames per stream through ClipStream(view or m) -- once with CUDA-graph replay, once with plain
    launches -- and checks every ready window against m.predict of that clip."""
    T = m.graph.frames_per_clip
    video = synth.synth_frames(S * n_push, res, res, seed=17).reshape(n_push, S, res, res, 3)
    target = view or m
    m.use_cuda_graph = True
    cs = ClipStream(target, S)
    plain = ClipStream(target, S)
    hist = [[] for _ in range(S)]
    checked = 0
    for i in range(n_push):
        for s in resets.get(i, []):
            hist[s] = []
            cs.reset([s])
            plain.reset([s])
        x = torch.from_numpy(video[i]).cuda()
        out = cs.push(x)
        got_c = [o.cpu().numpy() for o in out.clip_outputs]
        got_f = [o.cpu().numpy() for o in out.frame_outputs]
        m.use_cuda_graph = False
        ref = plain.push(x)
        m.use_cuda_graph = True
        for a, b in zip(got_c + got_f, [o.cpu().numpy() for o in ref.clip_outputs + ref.frame_outputs]):
            assert np.array_equal(a, b, equal_nan=True), 'graph replay differs from plain launches'
        for s in range(S):
            hist[s].append(video[i, s])
        assert out.ready.tolist() == [len(h) >= T for h in hist]
        for s in range(S):
            if not out.ready[s]:
                assert all(np.isnan(o[s]).all() for o in got_c)
                continue
            want = m.predict(np.stack(hist[s][-T:])[None])
            want = want if isinstance(want, list) else [want]
            for o, t in zip(got_c, cs.clip_output_tensors):
                r = want[m.graph.outputs.index(t)][0]
                assert np.abs(o[s] - r).max() <= 1e-5, (i, s, t, float(np.abs(o[s] - r).max()))
                assert o[s].argmax() == r.argmax()
            for o, t in zip(got_f, cs.frame_output_tensors):
                r = want[m.graph.outputs.index(t)][0, T - 1]
                assert np.abs(o[s] - r).max() <= 1e-5, (i, s, t, float(np.abs(o[s] - r).max()))
            checked += 1
    assert cs._graph is not None and plain._graph is None
    return cs, checked


@pytest.mark.parametrize('build,res', [(_penn_t8, 128), (_ntu_t16, 128), (_merge_2d, 128)],
                         ids=['penn_like_t8', 'ntu_like_t16_3d', 'merge_2d'])
def test_clip_stream_equals_predict(cuda, build, res):
    m = build().init_synthetic_weights(1234)
    T = m.graph.frames_per_clip
    S = 3
    cs, checked = _stream_vs_predict(cuda, m, S, T + 4, {1: [1], T: [2]}, res)
    assert checked == 5 + 4 + 1              # ready windows of this reset schedule, streams 0, 1, 2


def test_clip_stream_of_the_action_view(cuda):
    m = _penn_t8().init_synthetic_weights(1234)
    pm, am = spnet.split_model(m, m.cfg)
    cs, checked = _stream_vs_predict(cuda, m, 3, 10, {4: [0]}, 128, view=am)
    assert not cs.frame_output_tensors and len(cs.clip_output_tensors) == len(am.outputs) and checked > 0


def test_clip_stream_c4_full_size(cuda):
    m = _c4().init_synthetic_weights(1234)
    _, checked = _stream_vs_predict(cuda, m, 3, 18, {1: [1]}, 256)
    assert checked == 3 + 2 + 3


def test_launches_per_push_and_no_new_fallback(cuda):
    torch = cuda
    m = _penn_t8().init_synthetic_weights(1234)
    T, S = m.graph.frames_per_clip, 3
    m.use_cuda_graph = False
    lib = _ffi.lib()
    clip = synth.synth_frames(T, 128, 128, seed=3)[None]
    m.predict(clip)
    m._ctx.launch_count(reset=True)
    lib.dh_fallback_count(m._ctx.handle, 1)
    m.predict(clip)
    forward_launches = m._ctx.launch_count(reset=True)
    forward_fallbacks = int(lib.dh_fallback_count(m._ctx.handle, 1))
    cs = ClipStream(m, S)
    x = torch.from_numpy(synth.synth_frames(S, 128, 128, seed=4)).cuda()
    cs.push(x)
    torch.cuda.synchronize()
    m._ctx.launch_count(reset=True)
    lib.dh_fallback_count(m._ctx.handle, 1)
    cs.push(x)
    assert m._ctx.launch_count(reset=True) == forward_launches + 1
    assert int(lib.dh_fallback_count(m._ctx.handle, 1)) <= forward_fallbacks
    st = cs.stages
    assert cs.launches_per_push() == len(st.frame.kops) + len(st.clip.kops) + 1 == len(m.plan.kops) + 1


def test_single_frame_model_is_rejected(cuda):
    m = reception.build((64, 64, 3), 16, dim=2, num_blocks=1).init_synthetic_weights(1)
    with pytest.raises(ValueError):
        ClipStream(m, 2)
    assert compiler.split_stages(_penn_t8().graph).boundary
