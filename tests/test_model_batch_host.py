"""Model files at any batch up to the exported one, without a GPU.  Version 2 of the model format records each
activation slot's kind (frame or clip items); on the stand-in device (tests/fake_cuda.py) ReceptionNet 2-D / 3-D, SPNet
with T = 2, both merge models and random graphs of the compiler fuzzer are exported, and the kind table must be the
plan's `plan.phys`.  The rule dh_model_set_batch applies -- every view into an activation slot, and dh_mask_mul_f32's
rows over one, scale by n / N -- is restated here and must turn the launch list exported at N into the one exported at
n, record for record.  The library's own parser (dh_model_inspect, host-only) reads version 2, still reads version 1,
and refuses a view whose item count disagrees with its slot's kind, naming the launch."""
import ctypes as C
import json
import os
import struct
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from deephar_b200 import _ffi, export  # noqa: E402

MODELS = ['reception2d', 'reception3d', 'spnet_penn_t2', 'merge2d', 'merge3d'] + ['fuzz%d' % s for s in range(10)]
VIEW_BYTES = 32             # a view in the file: ptr (i32 arena + i64 offset) + five i32
DESC_BYTES = 8 * 4 + 4 * 12 + 3 * VIEW_BYTES + 2 * 4


# ---- in the subprocess: the stand-in device, each model exported at N and at a smaller n ----------------------------------
def _export(name, out_dir):
    import fake_cuda
    fake_cuda.install()
    from test_model_export_host import _model
    view, m, N = _model(name)
    T = m.graph.frames_per_clip
    r = {'N': N, 'T': T, 'phys': [kind for kind, _ in m.plan.phys], 'paths': {}}
    for n in sorted({1, N - 1, N} - {0}):
        path = os.path.join(out_dir, '%s_%d.dhm' % (name, n))
        view.export(path, n * T)
        r['paths'][n] = path
    return r


@pytest.fixture(scope='module')
def exported(tmp_path_factory):
    d = str(tmp_path_factory.mktemp('batch'))
    out = subprocess.run([sys.executable, os.path.abspath(__file__), d] + MODELS, capture_output=True, text=True,
                         timeout=1200, cwd=ROOT)
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-3000:]
    res = json.loads(out.stdout.strip().splitlines()[-1])
    for r in res.values():
        r['paths'] = {int(n): p for n, p in r['paths'].items()}
    return res


def _lib():
    lib = C.CDLL(_ffi.LIB_PATH)
    for name in ('dh_model_inspect', 'dh_last_error'):
        getattr(lib, name).restype, getattr(lib, name).argtypes = _ffi.SIGNATURES[name]
    return lib


def _inspect(path):
    lib = _lib()
    info = _ffi.dh_model_info()
    rc = lib.dh_model_inspect(path.encode(), C.byref(info), None, 0, None, 0)
    return rc, lib.dh_last_error().decode(), info


def _inspect_bytes(data, tmp_path):
    p = str(tmp_path / 'edited.dhm')
    with open(p, 'wb') as f:
        f.write(bytes(data))
    return _inspect(p)


def _kind_table_offset(rec):
    """file offset of the kind table: magic, version, five i32, the input shape, both blobs, the slot sizes"""
    return 8 + 4 + 20 + 4 + 8 * len(rec['input_shape']) + 8 + len(rec['weights']) + 8 + len(rec['packed']) + \
        4 + 8 * len(rec['slot_bytes'])


def _views(launch):
    """(file offset, view) of every view a launch record holds: its view arguments, then its descriptor's"""
    at = launch['file_offset'] + 12 + len(launch['label'].encode())
    out = []
    for tag, v in launch['args']:
        at += 1
        if tag == 'i':
            at += 8
        elif tag == 'f':
            at += 4
        elif tag == 'p':
            at += 12
        elif tag == 'v':
            out += [(at + 4 + VIEW_BYTES * j, x) for j, x in enumerate(v)]
            at += 4 + VIEW_BYTES * len(v)
        elif tag == 'd':
            for d in v:
                base = at + 4 + 8 * 4 + 4 * 12
                out += [(base + VIEW_BYTES * j, x) for j, x in enumerate(d['res'])]
                out.append((base + 2 * VIEW_BYTES + 8, d['pool_out']))
            at += 4 + DESC_BYTES * len(v)
        else:
            at += 4 + 32 * len(v)
    return out


def _in_slot(p):
    return p is not None and p[0] >= export.ARENA_SLOT0


def _rebatch(rec, N, n):
    """dh_model_set_batch's rule, restated: slot views and dh_mask_mul_f32's rows over a slot scale by n / N"""
    def view(v):
        if _in_slot(v['p']):
            assert v['n'] % N == 0
            v = dict(v, n=v['n'] // N * n)
        return v
    out = []
    for L in rec['launches']:
        args = []
        for tag, v in L['args']:
            if tag == 'v':
                v = [view(x) for x in v]
            elif tag == 'd':
                v = [dict(d, res=[view(x) for x in d['res']], pool_out=view(d['pool_out'])) for d in v]
            args.append((tag, v))
        if L['entry'] == 'dh_mask_mul_f32' and _in_slot(L['args'][0][1]):
            args[2] = ('i', args[2][1] // N * n)
        out.append((L['entry'], L['label'], args))
    return out, view(rec['input']), [(view(o['view']), (n,) + tuple(o['shape'][1:]), o['name']) for o in rec['outputs']]


def _as_json(x):
    return json.loads(json.dumps(x, default=list))


@pytest.mark.timeout(1200)
@pytest.mark.parametrize('name', MODELS)
def test_kind_table_is_the_plans_slot_kinds(exported, name):
    r = exported[name]
    rec = export.read(r['paths'][r['N']])
    assert rec['version'] == export.VERSION == 2
    assert rec['slot_kinds'] == r['phys']
    if name.startswith(('spnet', 'merge')):
        assert {'frame', 'clip'} <= set(rec['slot_kinds'])
    rc, err, info = _inspect(r['paths'][r['N']])
    assert rc == 0, err
    assert info.version == 2 and info.n_slots == len(r['phys']) and info.clip_items == r['N']


@pytest.mark.timeout(1200)
@pytest.mark.parametrize('name', MODELS)
def test_rebatch_rule_gives_the_launch_list_exported_at_n(exported, name):
    """the launch list exported at N, rewritten for n, is the one exported at n: same entry points, scalars, struct
    fields and (arena, byte offset) pointers -- a slot view's byte offset is a channel offset, whatever the batch"""
    r = exported[name]
    N = r['N']
    full = export.read(r['paths'][N])
    for n, path in r['paths'].items():
        small = export.read(path)
        launches, inp, outs = _rebatch(full, N, n)
        want = [(L['entry'], L['label'], L['args']) for L in small['launches']]
        assert _as_json(launches) == _as_json(want), (name, n)
        assert _as_json(inp) == _as_json(small['input'])
        assert _as_json(outs) == _as_json([(o['view'], o['shape'], o['name']) for o in small['outputs']])
        assert small['slot_kinds'] == full['slot_kinds']
        assert small['workspace_bytes'] <= full['workspace_bytes']


def test_clip_views_of_frame_slots_are_clip_counts(exported):
    """where frames_to_clip reads a frame slot as clips, the view holds N clips of T frames: the scale is still n / N"""
    seen = 0
    for name in ('spnet_penn_t2', 'merge2d', 'merge3d'):
        r = exported[name]
        rec = export.read(r['paths'][r['N']])
        for L in rec['launches']:
            for _, v in _views(L):
                if _in_slot(v['p']) and rec['slot_kinds'][v['p'][0] - export.ARENA_SLOT0] == 'frame' and \
                        v['n'] == r['N'] and r['T'] > 1:
                    assert v['h'] == r['T'], (name, L['label'], v)
                    seen += 1
    assert seen


def test_version_1_files_are_still_read(exported, tmp_path):
    for name in ('reception2d', 'merge3d'):
        r = exported[name]
        data = bytearray(open(r['paths'][r['N']], 'rb').read())
        rec = export.read(r['paths'][r['N']])
        at = _kind_table_offset(rec)
        assert list(data[at:at + len(r['phys'])]) == [export.SLOT_KINDS.index(k) for k in r['phys']]
        v1 = data[:at] + data[at + len(r['phys']):]
        struct.pack_into('<I', v1, 8, 1)
        rc, err, info = _inspect_bytes(v1, tmp_path)
        assert rc == 0, err
        assert info.version == 1 and info.n_launches == len(rec['launches'])
        # the same bytes as version 2 lack their kind table: refused, not misread
        struct.pack_into('<I', v1, 8, 2)
        rc, err, _ = _inspect_bytes(v1, tmp_path)
        assert rc < 0 and err.startswith('deephar_b200 model file'), err


def _first_view(rec, kind):
    for i, L in enumerate(rec['launches']):
        for at, v in _views(L):
            if _in_slot(v['p']) and rec['slot_kinds'][v['p'][0] - export.ARENA_SLOT0] == kind:
                return i, L, at, v
    raise AssertionError(kind)


def test_a_view_whose_items_disagree_with_its_slot_is_refused(exported, tmp_path):
    for name, kind in (('reception2d', 'frame'), ('merge2d', 'frame'), ('spnet_penn_t2', 'clip')):
        r = exported[name]
        data = bytearray(open(r['paths'][r['N']], 'rb').read())
        rec = export.read(r['paths'][r['N']])
        i, L, at, v = _first_view(rec, kind)
        assert struct.unpack_from('<i', data, at + 12)[0] == v['n']
        bad = bytearray(data)
        struct.pack_into('<i', bad, at + 12, v['n'] - 1)          # fewer items: within the arena, so only this refuses
        rc, err, _ = _inspect_bytes(bad, tmp_path)
        assert rc < 0, (name, kind)
        assert 'launch %d (%s)' % (i, L['label']) in err and 'in %s slot' % kind in err, err
        # the same edit in a version-1 file (no kind table) is a smaller batch the loader has no reason to refuse
        k = _kind_table_offset(rec)
        v1 = bad[:k] + bad[k + len(r['phys']):]
        struct.pack_into('<I', v1, 8, 1)
        rc, err, _ = _inspect_bytes(v1, tmp_path)
        assert rc == 0, err


def test_bad_kind_bytes_and_batches_are_refused(exported, tmp_path):
    r = exported['merge2d']
    data = bytearray(open(r['paths'][r['N']], 'rb').read())
    rec = export.read(r['paths'][r['N']])
    at = _kind_table_offset(rec)
    bad = bytearray(data)
    bad[at + 1] = 2
    rc, err, _ = _inspect_bytes(bad, tmp_path)
    assert rc < 0 and 'slot 1: kind 2' in err, err
    # a clip slot relabelled as a frame slot: its views hold N items, a clip count a frame slot may hold, so the label
    # that refuses is the other way round -- a frame slot with N * T frames relabelled clip
    frame = next(s for s, k in enumerate(r['phys']) if k == 'frame')
    bad = bytearray(data)
    bad[at + frame] = 1
    rc, err, _ = _inspect_bytes(bad, tmp_path)
    assert rc < 0 and 'in clip slot %d' % frame in err, err
    bad = bytearray(data)                                         # clip_items no longer frame_items / T
    struct.pack_into('<i', bad, 8 + 4 + 12, r['N'] - 1)
    rc, err, _ = _inspect_bytes(bad, tmp_path)
    assert rc < 0 and 'frame_items' in err, err
    r = next(exported[n] for n in MODELS if any(L['entry'] == 'dh_mask_mul_f32'
                                                 for L in export.read(exported[n]['paths'][exported[n]['N']])['launches']))
    rec = export.read(r['paths'][r['N']])
    data = bytearray(open(r['paths'][r['N']], 'rb').read())
    L = next(L for L in rec['launches'] if L['entry'] == 'dh_mask_mul_f32')
    rows_at = L['file_offset'] + 12 + len(L['label'].encode()) + 13 + 13 + 1
    assert struct.unpack_from('<q', data, rows_at)[0] == L['args'][2][1]
    bad = bytearray(data)
    struct.pack_into('<q', bad, rows_at, L['args'][2][1] - 1)
    rc, err, _ = _inspect_bytes(bad, tmp_path)
    assert rc < 0 and 'not a multiple of the batch' in err, err


if __name__ == '__main__':
    sys.path.insert(0, os.path.join(ROOT, 'tests'))
    res = {}
    for nm in sys.argv[2:]:
        res[nm] = _export(nm, sys.argv[1])
    print(json.dumps(res))
