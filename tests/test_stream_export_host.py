"""ClipStream.export without a GPU: on the stand-in device (tests/fake_cuda.py) reduced SPNet at T = 2 and T = 4, both
merge models and an SPNet action view are streamed at S = 1 and 3 and exported.  Reading each file back gives both
stages' bound launch lists -- entry point, every scalar, every struct field, every pointer as the same (arena, byte
offset) -- the stream's boundary table and the outputs push returns; the library's own parser, dh_stream_inspect
(host-only), reports S, T, the launch and slot counts, the arena bytes and the output shapes.  A file edited in one field
so that a launch reaches into the other stage, a boundary disagrees with S, T or itself, a ring has the wrong size, the
window's buffers overlap or a clip output has the wrong item count is refused with a message naming the record, as are
truncated files, a wrong magic or version, and a file of one kind given to the other kind's parser."""
import ctypes as C
import json
import os
import struct
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from deephar_b200 import _ffi, export  # noqa: E402

MODELS = ['spnet_t2', 'spnet_t4', 'merge2d', 'merge3d', 'action_view']
CASES = ['%s-s%d' % (m, s) for m in MODELS for s in (1, 3)]


# ---- in the subprocess: the stand-in device, the streams, their export --------------------------------------------------
def _target(name):
    """name -> (model or view to stream, the Model underneath)"""
    sys.path.insert(0, os.path.join(ROOT, 'tests', 'golden'))
    from deephar_b200 import action, reception, spnet
    from deephar_b200.config import ModelConfig, pa16j2d
    from ref_cases import MERGE3D_CASE, MERGE_CASE
    if name.startswith('spnet') or name == 'action_view':
        T = 4 if name == 'spnet_t4' else 2
        cfg = ModelConfig((T, 128, 128, 3), pa16j2d, num_actions=[15], num_pyramids=2, action_pyramids=[1, 2],
                          num_levels=4, pose_replica=True, num_pose_features=160, num_visual_features=160)
        m = spnet.build(cfg).init_synthetic_weights(1234)
        return (spnet.split_model(m, cfg)[1] if name == 'action_view' else m), m
    mc = MERGE3D_CASE if name == 'merge3d' else MERGE_CASE
    pe = reception.build(mc['input_shape'], **mc['reception'])
    kw = dict(pose_dim=3, depth_maps=mc['depth_maps'], output_poses=True) if name == 'merge3d' else dict(pose_dim=2)
    m = action.build_merge_model(pe, mc['num_actions'], mc['input_shape'], mc['num_frames'], mc['num_joints'],
                                 mc['num_blocks'], **kw)
    return m, m.init_synthetic_weights(mc['seed'])


class _Arenas(object):
    """device address -> (arena, byte offset) over the stream's own buffers, in the file's arena order"""

    def __init__(self, cs):
        m = cs.model
        packed = m._dev_packed if m._packed_info else None
        bufs = [(m._dev, 4), (packed, 2), (cs._frame.workspace, 4), (cs._clip.workspace, 4)] + \
            [(s, 4) for s in cs._frame.slots + cs._clip.slots + cs._rings]
        self.ranges = [(t.data_ptr(), t.numel() * e) if t is not None else (0, 0) for t, e in bufs]

    def __call__(self, p):
        if not p:
            return None
        hits = [(i, p - base) for i, (base, n) in enumerate(self.ranges) if n and base <= p < base + n]
        assert len(hits) == 1, hex(p)
        return hits[0]


def _as_file(v, arenas):
    """a ctypes value of b.calls in export.read_stream()'s form"""
    if isinstance(v, C.Structure):
        out = {}
        for name, ty in v._fields_:
            f = getattr(v, name)
            if ty is C.c_void_p:
                out[name] = arenas(f)
            elif isinstance(f, C.Array):
                out[name] = [_as_file(e, arenas) for e in f]
            else:
                out[name] = _as_file(f, arenas)
        return out
    return v


def _pointees(v):
    if v is None:
        return []
    if isinstance(v, C.Array):
        return list(v)
    if isinstance(v, C._Pointer):
        return [v.contents] if v else []
    return [v._obj]


def _jsonable(x):
    return json.loads(json.dumps(x, default=list))


def _same_launches(got, calls, arenas, what):
    lib = _ffi.lib()
    assert len(got) == len(calls), what
    for n, (launch, call) in enumerate(zip(got, calls)):
        assert getattr(lib, launch['entry']) is call[1], (what, n, launch['entry'], call[0])
        sig = export.signature(launch['entry'])
        assert ''.join(t for t, _ in launch['args']) == sig and len(call) == 3 + len(sig), (what, n)
        for k, ((tag, v_file), v) in enumerate(zip(launch['args'], call[3:])):
            if tag == 'i':
                want = int(v)
            elif tag == 'f':
                want = float(np.float32(v.value))
            elif tag == 'p':
                want = arenas(v)
            else:
                want = [_as_file(s, arenas) for s in _pointees(v)]
            assert _jsonable(v_file) == _jsonable(want), (what, n, call[0], k, v_file, want)


def _export(case, out_dir):
    import torch

    from deephar_b200.stream import ClipStream
    name, S = case.rsplit('-s', 1)
    S = int(S)
    target, m = _target(name)
    cs = ClipStream(target, S)
    T = cs.frames_per_clip
    t_in = m.graph.inputs[0]
    out = cs.push(torch.zeros((S,) + tuple(t_in.shape), device='cuda'))       # a stream with state: one push, a reset
    cs.reset([0])
    state = (list(m._bound), cs._count.copy(), cs._counter.cpu().numpy().copy(), [r.cpu().numpy().copy() for r in cs._rings])
    path = os.path.join(out_dir, case + '.dhs')
    cs.export(path)
    assert list(m._bound) == state[0] and np.array_equal(cs._count, state[1])
    assert np.array_equal(cs._counter.cpu().numpy(), state[2])
    assert all(np.array_equal(r.cpu().numpy(), r0) for r, r0 in zip(cs._rings, state[3]))
    rec = export.read_stream(path)
    arenas = _Arenas(cs)
    st = cs.stages
    assert len(cs._frame.calls) == len(st.frame.kops) and len(cs._clip.calls) == len(st.clip.kops)
    _same_launches(rec['frame_launches'], cs._frame.calls, arenas, 'frame stage')
    _same_launches(rec['clip_launches'], cs._clip.calls, arenas, 'clip stage')
    table = np.frombuffer(cs._table.cpu().numpy().tobytes(), np.uint8)
    entries = [_ffi.dh_clip_window.from_buffer_copy(table[i * C.sizeof(_ffi.dh_clip_window):].tobytes()
                                                    [:C.sizeof(_ffi.dh_clip_window)]) for i in range(len(cs._rings))]
    assert len(rec['boundary']) == len(entries) == len(st.boundary) >= 1
    for b, e in zip(rec['boundary'], entries):
        assert _jsonable({k: b[k] for k in ('src', 'dst', 'ring')}) == \
            _jsonable({'src': _as_file(e.src, arenas), 'dst': _as_file(e.dst, arenas), 'ring': arenas(e.ring)})
    assert rec['weights'] == m._dev.numpy().tobytes()
    if m._packed_info:
        assert rec['packed'] == m._dev_packed.numpy().tobytes() and rec['use_tensor_cores'] == 1
    assert rec['frame_slot_bytes'] == [s.numel() * 4 for s in cs._frame.slots]
    assert rec['clip_slot_bytes'] == [s.numel() * 4 for s in cs._clip.slots]
    assert rec['ring_bytes'] == [r.numel() * 4 for r in cs._rings] == \
        [4 * S * T * int(np.prod(t.shape)) for t in st.boundary]
    assert rec['frame_workspace_bytes'] == cs._frame.workspace.numel() * 4
    assert rec['clip_workspace_bytes'] == cs._clip.workspace.numel() * 4
    assert (rec['n_streams'], rec['frames_per_clip'], tuple(rec['input_shape'])) == (S, T, (S,) + tuple(t_in.shape))
    names = [(t.node.attrs.get('name') if t.node is not None else None) or 'output_%d' % m.graph.outputs.index(t)
             for t in cs.frame_output_tensors + cs.clip_output_tensors]
    pushed = [list(o.shape) for o in out.frame_outputs + out.clip_outputs]
    recorded = rec['frame_outputs'] + rec['clip_outputs']
    assert [list(o['shape']) for o in recorded] == pushed and [o['name'] for o in recorded] == names
    # export refuses what push refuses
    keep, m._dev = m._dev, m._dev.clone()
    for fn in (lambda: cs.export(path + '.stale'), lambda: cs.push(torch.zeros((S,) + tuple(t_in.shape), device='cuda'))):
        try:
            fn()
            raise AssertionError('a stream over replaced weights was accepted')
        except RuntimeError as e:
            assert 'replaced' in str(e)
    m._dev = keep
    assert not os.path.exists(path + '.stale')
    model_path = os.path.join(out_dir, case + '.dhm') if case == 'merge3d-s1' else None
    if model_path:
        m.export(model_path, T)
    return {'path': path, 'model_path': model_path, 'S': S, 'T': T, 'frame_launches': len(st.frame.kops),
            'clip_launches': len(st.clip.kops), 'frame_slots': rec['frame_slot_bytes'],
            'clip_slots': rec['clip_slot_bytes'], 'rings': rec['ring_bytes'], 'shapes': pushed, 'names': names,
            'n_frame_outputs': len(out.frame_outputs), 'weights': len(rec['weights']), 'packed': len(rec['packed']),
            'workspaces': [rec['frame_workspace_bytes'], rec['clip_workspace_bytes']],
            'input_shape': list(rec['input_shape']),
            'frame_slot0': rec['frame_slot0'], 'clip_slot0': rec['clip_slot0'], 'ring0': rec['ring0'],
            'boundary': [dict(b, src=list(b['src'].items()), dst=list(b['dst'].items())) for b in rec['boundary']],
            'clip_outputs': [o['file_offset'] for o in rec['clip_outputs']],
            # record starts: every boundary entry and output, the first two and the last launch of each stage
            'records': sorted([o['file_offset'] for o in recorded] + [b['file_offset'] for b in rec['boundary']] +
                              [l['file_offset'] for ls in (rec['frame_launches'], rec['clip_launches'])
                               for l in ls[:2] + ls[-1:]]),
            'first_launch': [(l['file_offset'] + 12 + len(l['label'].encode()), l['args'][0][0])
                             for l in (rec['frame_launches'][0], rec['clip_launches'][0])]}


# ---- in the test: the library's parser on its own CDLL (the stand-in keeps only a few host entry points) ---------------------
@pytest.fixture(scope='module')
def exported(tmp_path_factory):
    d = str(tmp_path_factory.mktemp('stream_export'))
    out = subprocess.run([sys.executable, os.path.abspath(__file__), d] + CASES, capture_output=True, text=True,
                         timeout=1200, cwd=ROOT)
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-3000:]
    return json.loads(out.stdout.strip().splitlines()[-1])


def _lib():
    lib = C.CDLL(_ffi.LIB_PATH)
    for name in ('dh_stream_inspect', 'dh_model_inspect', 'dh_last_error'):
        getattr(lib, name).restype, getattr(lib, name).argtypes = _ffi.SIGNATURES[name]
    return lib


def _inspect(path, max_outputs=64):
    lib = _lib()
    info = _ffi.dh_stream_info()
    outs = (_ffi.dh_model_output_info * max_outputs)()
    rc = lib.dh_stream_inspect(path.encode(), C.byref(info), outs, max_outputs)
    return rc, lib.dh_last_error().decode(), info, list(outs)


@pytest.mark.timeout(1200)
@pytest.mark.parametrize('case', CASES)
def test_inspect_reports_the_bound_stream(exported, case):
    r = exported[case]
    rc, err, info, outs = _inspect(r['path'])
    assert rc == 0, err
    assert info.version == export.STREAM_VERSION
    assert (info.n_streams, info.frames_per_clip) == (r['S'], r['T'])
    assert (info.n_frame_launches, info.n_clip_launches) == (r['frame_launches'], r['clip_launches'])
    assert (info.n_frame_slots, info.n_clip_slots) == (len(r['frame_slots']), len(r['clip_slots']))
    assert info.activation_bytes == sum(r['frame_slots']) + sum(r['clip_slots'])
    assert info.ring_bytes == sum(r['rings']) and info.n_boundary == len(r['rings'])
    assert [info.frame_workspace_bytes, info.clip_workspace_bytes] == r['workspaces']
    assert (info.weight_bytes, info.packed_bytes) == (r['weights'], r['packed'])
    assert list(info.input_shape[:info.input_rank]) == r['input_shape']
    assert info.n_frame_outputs == r['n_frame_outputs'] and info.n_frame_outputs + info.n_clip_outputs == len(r['shapes'])
    assert info.device_bytes >= info.weight_bytes + info.packed_bytes + info.activation_bytes + info.ring_bytes
    for o, shp, nm in zip(outs, r['shapes'], r['names']):
        assert list(o.shape[:o.rank]) == shp and all(d == 0 for d in o.shape[o.rank:])
        assert o.name.decode() == nm[:63]


def _refused(data, tmp_path, what, kind='stream'):
    p = str(tmp_path / 'bad.dhs')
    with open(p, 'wb') as f:
        f.write(bytes(data))
    rc, err, _, _ = _inspect(p)
    assert rc < 0, 'a file with %s was accepted' % what
    assert err.startswith('deephar_b200 %s file' % kind), err
    return err


def _read(r):
    return bytearray(open(r['path'], 'rb').read())


def _view_at(b, which):
    """file offset of the view `which` ('src' or 'dst') of a boundary record, and its fields"""
    return b['file_offset'] + (0 if which == 'src' else 32), dict(b[which])


def test_a_launch_into_the_other_stage_is_refused(exported, tmp_path):
    r = exported['spnet_t2-s3']
    data = _read(r)
    for stage, (at, tag), arenas in (('frame', r['first_launch'][0], (r['clip_slot0'], r['ring0'])),
                                     ('clip', r['first_launch'][1], (r['frame_slot0'], r['ring0']))):
        assert tag in 'vp' and data[at] == ord(tag)
        ptr_at = at + 1 + (4 if tag == 'v' else 0)          # after the tag (and a view argument's count)
        assert struct.unpack_from('<i', data, ptr_at)[0] >= 0
        for arena in arenas:
            bad = bytearray(data)
            struct.pack_into('<iq', bad, ptr_at, arena, 0)
            err = _refused(bad, tmp_path, 'a %s launch pointing into arena %d' % (stage, arena))
            assert '%s launch 0' % stage in err and 'outside the %s stage' % stage in err, err


def test_boundaries_that_disagree_with_S_T_or_themselves_are_refused(exported, tmp_path):
    r = exported['spnet_t2-s3']
    S, T = r['S'], r['T']
    b = r['boundary'][0]
    data = _read(r)
    src_at, src = _view_at(b, 'src')
    dst_at, dst = _view_at(b, 'dst')
    assert struct.unpack_from('<i', data, src_at + 12)[0] == src['n'] == S
    assert struct.unpack_from('<i', data, dst_at + 12)[0] == dst['n'] == S * T
    for at, v, why in ((src_at + 12, S - 1, 'src has n = %d, expected S = %d' % (S - 1, S)),
                       (dst_at + 12, S * T - 1, 'dst has n = %d, expected S*T = %d' % (S * T - 1, S * T))):
        bad = bytearray(data)
        struct.pack_into('<i', bad, at, v)
        err = _refused(bad, tmp_path, 'a boundary of the wrong item count')
        assert 'boundary 0' in err and why in err, err
    for field, k in (('h', 16), ('w', 20), ('c', 24)):
        if dst[field] > 1:
            bad = bytearray(data)
            struct.pack_into('<i', bad, dst_at + k, dst[field] - 1)
            err = _refused(bad, tmp_path, 'src and dst of different %s' % field)
            assert 'boundary 0' in err and 'differ' in err, err
    # the ring sizes precede the boundary table
    B = len(r['rings'])
    size_at = r['boundary'][0]['file_offset'] - 8 * B
    assert struct.unpack_from('<q', data, size_at)[0] == r['rings'][0]
    bad = bytearray(data)
    struct.pack_into('<q', bad, size_at, r['rings'][0] + 4)
    err = _refused(bad, tmp_path, 'a ring one float too large')
    assert 'boundary 0' in err and 'S*T*h*w*c floats' in err, err


def test_overlapping_window_buffers_are_refused(exported, tmp_path):
    """one boundary's dst (or ring) moved onto another's: the window kernel would write the same memory twice"""
    r = next(r for k, r in sorted(exported.items()) if len(r['rings']) >= 2)
    data = _read(r)
    bs = r['boundary']
    # a ring shared by two boundaries of the same ring size
    pair = next(((i, j) for i in range(len(bs)) for j in range(len(bs)) if i != j and r['rings'][i] == r['rings'][j]),
                None)
    if pair is not None:
        i, j = pair
        bad = bytearray(data)
        struct.pack_into('<iq', bad, bs[j]['file_offset'] + 64, *bs[i]['ring'])
        err = _refused(bad, tmp_path, 'a shared ring')
        assert 'overlap' in err and 'ring' in err, err
    # a dst moved onto another dst of its clip slot (or the first float of it)
    for i in range(len(bs)):
        for j in range(len(bs)):
            di, dj = dict(bs[i]['dst']), dict(bs[j]['dst'])
            if i == j or di['p'][0] != dj['p'][0] or di['ld'] != dj['ld']:
                continue
            bad = bytearray(data)
            struct.pack_into('<iq', bad, bs[j]['file_offset'] + 32, *di['p'])
            err = _refused(bad, tmp_path, 'two dst views on the same channels')
            assert 'overlap' in err or 'overrun' in err, err
            if 'overlap' in err:
                assert 'dst' in err
                return
    assert pair is not None, 'no boundary pair to overlap'


def test_a_clip_output_of_the_wrong_item_count_is_refused(exported, tmp_path):
    r = exported['merge2d-s3']
    data = _read(r)
    at = r['clip_outputs'][0]
    assert struct.unpack_from('<i', data, at + 12)[0] == r['S']
    bad = bytearray(data)
    struct.pack_into('<i', bad, at + 12, r['S'] - 1)
    err = _refused(bad, tmp_path, 'a clip output with n = S - 1')
    assert 'clip outputs' in err and 'clip output 0 has n = %d, expected S = %d' % (r['S'] - 1, r['S']) in err, err


def test_truncated_files_are_refused(exported, tmp_path):
    r = exported['spnet_t2-s3']
    data = _read(r)
    cuts = sorted(set([0, 5, 9, 13, 29, len(data) - 1] + r['records'] + [c + 4 for c in r['records']]
                      + list(np.random.default_rng(0).integers(0, len(data), 6))))
    for cut in cuts:
        err = _refused(data[:int(cut)], tmp_path, 'its last %d bytes cut' % (len(data) - cut))
        assert 'truncated' in err or 'magic' in err, (cut, err)
    err = _refused(data + b'\0', tmp_path, 'a trailing byte')
    assert 'after the last launch' in err


def test_wrong_magic_version_and_kind_are_refused(exported, tmp_path):
    r = exported['merge3d-s1']
    data = _read(r)
    bad = bytearray(data)
    bad[2] ^= 1
    assert 'magic' in _refused(bad, tmp_path, 'a bad magic')
    bad = bytearray(data)
    struct.pack_into('<I', bad, 9, export.STREAM_VERSION + 1)
    assert 'version %d' % (export.STREAM_VERSION + 1) in _refused(bad, tmp_path, 'a later version')
    # a model file is not a stream file, and the reverse
    rc, err, _, _ = _inspect(r['model_path'])
    assert rc < 0 and err.startswith('deephar_b200 stream file') and 'magic' in err, err
    lib = _lib()
    info = _ffi.dh_model_info()
    assert lib.dh_model_inspect(r['path'].encode(), C.byref(info), None, 0, None, 0) < 0
    err = lib.dh_last_error().decode()
    assert err.startswith('deephar_b200 model file') and 'magic' in err, err


if __name__ == '__main__':
    sys.path.insert(0, os.path.join(ROOT, 'tests'))
    import fake_cuda
    fake_cuda.install()
    print(json.dumps({case: _export(case, sys.argv[1]) for case in sys.argv[2:]}))
