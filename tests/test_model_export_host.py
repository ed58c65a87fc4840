"""Model.export without a GPU: on the stand-in device (tests/fake_cuda.py) reduced ReceptionNet 2-D / 3-D, SPNet T = 2,
both merge models, a split_model view and random graphs of the compiler fuzzer are bound and exported.  Reading the file
back gives the bound launch list -- entry point, every scalar, every struct field, every pointer as the same (arena,
byte offset) -- and the library's own parser, dh_model_inspect (host-only), reports the plan's launch count, slot sizes
and output shapes.  Truncated files, a flipped pointer, a wrong version, an out-of-range argument and a bad signature
are refused with a message before any device work."""
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

MODELS = ['reception2d', 'reception3d', 'spnet_penn_t2', 'spnet_action_view', 'merge2d', 'merge3d'] + \
    ['fuzz%d' % s for s in range(10)]


# ---- in the subprocess: the stand-in device, the models, their export --------------------------------------------------
def _model(name):
    """name -> (model or output view, the Model underneath, items exported)"""
    sys.path.insert(0, os.path.join(ROOT, 'tests', 'golden'))
    from deephar_b200 import action, reception, spnet
    from deephar_b200.config import ModelConfig, pa16j2d
    from ref_cases import MERGE3D_CASE
    from test_launch_check_host import _models
    if name == 'reception3d':
        m = reception.build((128, 128, 3), num_joints=16, dim=3, num_blocks=2, depth_maps=8, ksize=(5, 5))
        m.init_synthetic_weights(1234)
        return m, m, 3
    if name == 'merge3d':
        mc = MERGE3D_CASE
        pe = reception.build(mc['input_shape'], **mc['reception'])
        m = action.build_merge_model(pe, mc['num_actions'], mc['input_shape'], mc['num_frames'], mc['num_joints'],
                                     mc['num_blocks'], pose_dim=3, depth_maps=mc['depth_maps'], output_poses=True)
        m.init_synthetic_weights(mc['seed'])
        return m, m, 2
    if name == 'spnet_action_view':
        cfg = ModelConfig((2, 128, 128, 3), pa16j2d, num_actions=[15], num_pyramids=2, action_pyramids=[1, 2],
                          num_levels=4, pose_replica=True, num_pose_features=160, num_visual_features=160)
        m = spnet.build(cfg).init_synthetic_weights(1234)
        return spnet.split_model(m, cfg)[1], m, 2
    m, x = _models(name)
    items = 2 if m.graph.frames_per_clip > 1 else 3
    return m, m, items


class _Arenas(object):
    """device address -> (arena, byte offset), from the bound buffers themselves"""

    def __init__(self, m, b):
        packed = getattr(m, '_dev_packed', None) if m._packed_info else None
        self.ranges = [(m._dev.data_ptr(), m._dev.numel() * 4),
                       (packed.data_ptr(), packed.numel() * 2) if packed is not None else (0, 0),
                       (b.workspace.data_ptr(), b.workspace.numel() * 4)] + \
            [(s.data_ptr(), s.numel() * 4) for s in b.slots]

    def __call__(self, p):
        if not p:
            return None
        hits = [(i, p - base) for i, (base, n) in enumerate(self.ranges) if base <= p < base + n]
        assert len(hits) == 1, hex(p)
        return hits[0]


def _as_file(v, arenas):
    """a ctypes value of b.calls in export.read()'s form"""
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
    if isinstance(v, list):
        return [list(e) if isinstance(e, tuple) else e for e in v]
    return v


def _pointees(v):
    if v is None:
        return []
    if isinstance(v, C.Array):
        return list(v)
    if isinstance(v, C._Pointer):
        return [v.contents] if v else []
    return [v._obj]


def _input_view(m, b, n_frames):
    t = m.graph.inputs[0]
    s = m.plan.storage[t.id]
    assert s.c_off == 0 and s.ld == t.shape[2]
    return (b.slots[s.buf.phys].data_ptr(), n_frames) + tuple(t.shape) + (s.ld,)


def _jsonable(x):
    return json.loads(json.dumps(x, default=list))


def _export(name, out_dir):
    import fake_cuda
    fake_cuda.install()
    view, m, items = _model(name)
    n_frames = items * m.graph.frames_per_clip
    path = os.path.join(out_dir, name + '.dhm')
    view.export(path, n_frames)
    bound_after_export = list(m._bound)
    b = m._bind(n_frames)
    rec = export.read(path)
    arenas = _Arenas(m, b)
    lib = _ffi.lib()
    assert len(rec['launches']) == len(b.calls) == len(m.plan.kops)
    for n, (launch, call) in enumerate(zip(rec['launches'], b.calls)):
        assert getattr(lib, launch['entry']) is call[1], (n, launch['entry'], call[0])
        sig = export.signature(launch['entry'])
        assert ''.join(t for t, _ in launch['args']) == sig and len(call) == 3 + len(sig), n
        for k, ((tag, got), v) in enumerate(zip(launch['args'], call[3:])):
            if tag == 'i':
                want = int(v)
            elif tag == 'f':
                want = float(np.float32(v.value))
            elif tag == 'p':
                want = arenas(v)
            else:
                want = [_as_file(s, arenas) for s in _pointees(v)]
            assert _jsonable(got) == _jsonable(want), (name, n, call[0], k, got, want)
    assert rec['weights'] == m._dev.numpy().tobytes()
    if m._packed_info:
        assert rec['packed'] == m._dev_packed.numpy().tobytes() and rec['use_tensor_cores'] == 1
    assert rec['slot_bytes'] == [s.numel() * 4 for s in b.slots]
    assert rec['workspace_bytes'] == b.workspace.numel() * 4
    idx = getattr(view, 'indices', range(len(m.graph.outputs)))
    shapes = []
    for i in idx:
        t = m.graph.outputs[i]
        shapes.append(list(m._keras_shape(t, m._items(t.kind, n_frames) if t.kind == 'clip' else n_frames)))
    assert [list(o['shape']) for o in rec['outputs']] == shapes
    assert rec['input'] == _as_file(_ffi.dh_view(*_input_view(m, b, n_frames)), arenas)
    return {'path': path, 'launches': len(b.calls), 'slot_bytes': rec['slot_bytes'], 'shapes': shapes,
            'names': [o['name'] for o in rec['outputs']], 'workspace': rec['workspace_bytes'],
            'weights': len(rec['weights']), 'packed': len(rec['packed']), 'frames': n_frames,
            'bound_after_export': bound_after_export,
            'launch_offsets': [(l['entry'], l['file_offset'], len(l['label'].encode()), l['args'][0][1] and len(l['args'][0][1]))
                               for l in rec['launches']]}


# ---- in the test: the library's parser on its own CDLL (the stand-in keeps only a few host entry points) ---------------------
@pytest.fixture(scope='module')
def exported(tmp_path_factory):
    d = str(tmp_path_factory.mktemp('export'))
    out = subprocess.run([sys.executable, os.path.abspath(__file__), d] + MODELS, capture_output=True, text=True,
                         timeout=1200, cwd=ROOT)
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-3000:]
    return json.loads(out.stdout.strip().splitlines()[-1])


def _lib():
    lib = C.CDLL(_ffi.LIB_PATH)
    for name in ('dh_model_inspect', 'dh_last_error'):
        getattr(lib, name).restype, getattr(lib, name).argtypes = _ffi.SIGNATURES[name]
    return lib


def _inspect(path, max_slots=256, max_outputs=64):
    lib = _lib()
    info = _ffi.dh_model_info()
    slots = (C.c_int64 * max_slots)()
    outs = (_ffi.dh_model_output_info * max_outputs)()
    rc = lib.dh_model_inspect(path.encode(), C.byref(info), slots, max_slots, outs, max_outputs)
    return rc, lib.dh_last_error().decode(), info, list(slots), list(outs)


@pytest.mark.timeout(1200)
@pytest.mark.parametrize('name', MODELS)
def test_inspect_reports_the_bound_plan(exported, name):
    r = exported[name]
    rc, err, info, slots, outs = _inspect(r['path'])
    assert rc == 0, err
    assert info.version == export.VERSION and info.n_launches == r['launches']
    assert info.n_slots == len(r['slot_bytes']) and slots[:info.n_slots] == r['slot_bytes']
    assert info.activation_bytes == sum(r['slot_bytes']) and info.workspace_bytes == r['workspace']
    assert info.weight_bytes == r['weights'] and info.packed_bytes == r['packed']
    assert info.n_outputs == len(r['shapes'])
    for o, shp, nm in zip(outs, r['shapes'], r['names']):
        assert list(o.shape[:o.rank]) == shp and all(d == 0 for d in o.shape[o.rank:])
        assert o.name.decode() == nm[:63]
    lead = list(info.input_shape[:info.input_rank])
    assert int(np.prod(lead[:-3])) == info.frame_items == r['frames']
    assert info.clip_items * info.frames_per_clip == r['frames']


def test_the_fuzz_exports_reach_every_head_and_fused_kind(exported):
    entries = set(e for r in exported.values() for e, _, _, _ in r['launch_offsets'])
    assert {'dh_conv2d_f32', 'dh_sepconv2d_f32', 'dh_softargmax2d_f32', 'dh_kron_pool_f32', 'dh_add_n_f32',
            'dh_softargmax3d_ex_f32', 'dh_mask_mul_f32', 'dh_global_maxmin_softmax_f32'} <= entries, sorted(entries)


def _refused(data, tmp_path, what):
    p = str(tmp_path / 'bad.dhm')
    with open(p, 'wb') as f:
        f.write(bytes(data))
    rc, err, _, _, _ = _inspect(p)
    assert rc < 0, 'a file with %s was accepted' % what
    assert err.startswith('deephar_b200 model file'), err
    return err


def _launch(r, entry):
    """(file offset of the first argument, first-argument view count) of the first launch of `entry`"""
    for e, at, nlabel, nviews in r['launch_offsets']:
        if e == entry:
            return at + 12 + nlabel, nviews
    raise AssertionError(entry)


def test_truncated_files_are_refused(exported, tmp_path):
    r = exported['reception2d']
    data = open(r['path'], 'rb').read()
    cuts = sorted(set([0, 4, 8, 11, 20, 40, 60, len(data) - 1, len(data) - 7]
                      + list(np.random.default_rng(0).integers(0, len(data), 40))))
    for cut in cuts:
        err = _refused(data[:int(cut)], tmp_path, 'its last %d bytes cut' % (len(data) - cut))
        assert 'truncated' in err or 'magic' in err, (cut, err)
    err = _refused(data + b'\0', tmp_path, 'a trailing byte')
    assert 'after the last launch' in err


def test_wrong_magic_and_version_are_refused(exported, tmp_path):
    data = bytearray(open(exported['reception2d']['path'], 'rb').read())
    bad = bytearray(data)
    bad[0] ^= 1
    assert 'magic' in _refused(bad, tmp_path, 'a bad magic')
    bad = bytearray(data)
    struct.pack_into('<I', bad, 8, export.VERSION + 1)
    assert 'version %d' % (export.VERSION + 1) in _refused(bad, tmp_path, 'a later version')


def test_flipped_pointers_are_refused(exported, tmp_path):
    """the first launch's input view (tag, count, then arena and byte offset): moved past its arena's end, into an arena
    the file does not have, onto an unaligned address"""
    r = exported['reception2d']
    data = bytearray(open(r['path'], 'rb').read())
    at, _ = _launch(r, 'dh_conv2d_f32')
    assert data[at] == ord('v')
    arena, off = struct.unpack_from('<iq', data, at + 5)
    assert arena >= export.ARENA_SLOT0
    size = r['slot_bytes'][arena - export.ARENA_SLOT0]
    for new_arena, new_off, why in ((arena, size - 4, 'overrun arena'), (arena, off + (1 << 40), 'overrun arena'),
                                    (arena + 500, off, 'points into arena'), (arena, off + 2, 'not 4-byte aligned')):
        bad = bytearray(data)
        struct.pack_into('<iq', bad, at + 5, new_arena, new_off)
        err = _refused(bad, tmp_path, 'a flipped pointer')
        assert 'launch 0 (conv' in err and why in err, err


def test_out_of_range_arguments_are_refused(exported, tmp_path):
    r = next(r for r in exported.values() if any(e == 'dh_add_n_f32' for e, _, _, _ in r['launch_offsets']))
    data = bytearray(open(r['path'], 'rb').read())
    at, nviews = _launch(r, 'dh_add_n_f32')                      # (views, n_in, scale, shift, relu, out)
    n_in_at = at + 1 + 4 + 32 * nviews
    assert data[n_in_at] == ord('i') and struct.unpack_from('<q', data, n_in_at + 1)[0] == nviews
    for v, why in ((9, 'n_in'), (nviews + 1 if nviews < 4 else 1, 'views for n_in')):
        bad = bytearray(data)
        struct.pack_into('<q', bad, n_in_at + 1, v)
        assert why in _refused(bad, tmp_path, 'n_in = %d' % v)
    bad = bytearray(data)
    bad[n_in_at] = ord('f')
    assert "expects 'i'" in _refused(bad, tmp_path, 'a wrong argument tag')
    r = exported['reception2d']
    data = bytearray(open(r['path'], 'rb').read())
    at, _ = _launch(r, 'dh_conv2d_f32')                         # desc after x (view), w (ptr), packed
    data_at = at + 1 + 4 + 32 + 13
    assert data[data_at] == ord('w')
    count = struct.unpack_from('<i', data, data_at + 1)[0]
    desc_at = data_at + 5 + count * 32
    assert data[desc_at] == ord('d')
    for field, v, why in ((0, 0, 'kh'), (2, 0, 'sh'), (7, 3, 'n_res')):
        bad = bytearray(data)
        struct.pack_into('<i', bad, desc_at + 5 + 4 * field, v)
        assert why in _refused(bad, tmp_path, 'desc field %d = %d' % (field, v))



def test_view_extents_that_wrap_64_bits_are_refused(exported, tmp_path):
    """n * h * w = 2^32 + 1 rows of leading dimension 2^30: 2^62 + 1 floats, whose byte count wraps to 4 in 64 bits.
    Every view of a dh_add_n_f32 launch (its inputs and its output, which the kernel only checks for equal shapes) made
    so must be refused by its extent, not let through to the kernel."""
    r = next(r for r in exported.values() if any(e == 'dh_add_n_f32' for e, _, _, _ in r['launch_offsets']))
    data = bytearray(open(r['path'], 'rb').read())
    at, nviews = _launch(r, 'dh_add_n_f32')                      # (views, n_in, scale, shift, relu, out)
    out_at = at + 1 + 4 + 32 * nviews + 9 + 13 + 13 + 9
    assert data[out_at] == ord('v') and struct.unpack_from('<i', data, out_at + 1)[0] == 1
    fields = [at + 5 + 32 * j + 12 for j in range(nviews)] + [out_at + 5 + 12]
    assert 641 * 6700417 == 2 ** 32 + 1
    for which in (fields[-1:], fields):
        bad = bytearray(data)
        for f in which:
            struct.pack_into('<5i', bad, f, 641, 6700417, 1, 1, 2 ** 30)
        err = _refused(bad, tmp_path, 'a view whose byte extent wraps')
        assert 'overrun arena' in err and 'launch' in err, err
    bad = bytearray(data)                                       # the same view one row short of the wrap: also refused
    struct.pack_into('<5i', bad, fields[-1], 641, 6700417, 1, 1, 2 ** 20)
    assert 'overrun arena' in _refused(bad, tmp_path, 'a view larger than its arena')


def test_export_leaves_the_models_bound_batch_sizes_alone(exported):
    assert all(r['bound_after_export'] == [] for r in exported.values())


if __name__ == '__main__':
    sys.path.insert(0, os.path.join(ROOT, 'tests'))
    res = {}
    for nm in sys.argv[2:]:
        res[nm] = _export(nm, sys.argv[1])
    print(json.dumps(res))
