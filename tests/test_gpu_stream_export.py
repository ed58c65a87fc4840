"""ClipStream.export on the GPU: the exported stream, loaded and pushed through the C ABI (dh_stream_load /
dh_stream_push), computes what ClipStream.push computes, bit for bit, push after push with resets -- penn-like T = 8,
NTU-like T = 16 3-D, the 2-D merge model, an SPNet action view and full-size C4 -- and its ready flags are
ClipStream.ready.  A push captured into a CUDA graph and replayed with resets in between keeps its readiness on the
device.  dh_stream_ready_f32 is checked on its own against its contract; a push is one launch more than
ClipStream.push, with no new CUDA-core fallback; streams and a model in one context stay independent; bad resets and output
indices are refused; dh_stream_free returns every byte; examples/run_stream.c writes the same bytes as ClipStream.

    pytest -m gpu tests/test_gpu_stream_export.py -s        (-s: the C vs Python push times of C4 at S = 8)
"""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

from deephar_b200 import _ffi
from deephar_b200.stream import ClipStream
from oracle import synth

from test_gpu_model_export import CModel, _cudart
from test_gpu_stream import _c4, _merge_2d, _ntu_t16, _penn_t8

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _inspect(path):
    info = _ffi.dh_stream_info()
    _ffi.check(_ffi.lib().dh_stream_inspect(path.encode(), C.byref(info), None, 0), 'dh_stream_inspect')
    return info


class CStream(object):
    """a loaded stream file, driven through the C ABI only"""

    def __init__(self, ctx, path):
        self.lib, self.rt = _ffi.lib(), _cudart()
        self.info = _inspect(path)
        self.n_outputs = self.info.n_frame_outputs + self.info.n_clip_outputs
        self.h = C.c_void_p()
        _ffi.check(self.lib.dh_stream_load(ctx.handle, path.encode(), C.byref(self.h)), 'dh_stream_load')

    def set_input(self, x):
        """x: float32 CUDA tensor (S, H, W, 3), copied on the legacy default stream (ordered with torch's)"""
        v = _ffi.dh_view()
        _ffi.check(self.lib.dh_stream_input(self.h, C.byref(v)), 'dh_stream_input')
        assert x.is_contiguous() and x.numel() == v.n * v.h * v.w * v.c and v.ld == v.c
        assert self.rt.cudaMemcpy(v.p, C.c_void_p(x.data_ptr()), x.numel() * 4, 3) == 0

    def push(self, stream):
        _ffi.check(self.lib.dh_stream_push(self.h, stream), 'dh_stream_push')

    def reset(self, ids, stream):
        """ids: None (all streams) or a list; returns the library's return code"""
        if ids is None:
            return self.lib.dh_stream_reset(self.h, None, 0, stream)
        arr = (C.c_int32 * len(ids))(*ids)
        return self.lib.dh_stream_reset(self.h, arr, len(ids), stream)

    def outputs(self):
        """frame outputs, then clip outputs, as host arrays of their (S, ...) shapes"""
        res = []
        for k in range(self.n_outputs):
            v, info = _ffi.dh_view(), _ffi.dh_model_output_info()
            _ffi.check(self.lib.dh_stream_output(self.h, k, C.byref(v), C.byref(info)), 'dh_stream_output')
            rows = v.n * v.h * v.w
            host = np.empty((rows, v.c), np.float32)
            assert self.rt.cudaMemcpy2D(host.ctypes.data, v.c * 4, v.p, v.ld * 4, v.c * 4, rows, 2) == 0
            res.append(host.reshape(tuple(info.shape[:info.rank])))
        return res

    def ready(self):
        p = C.c_void_p()
        _ffi.check(self.lib.dh_stream_ready(self.h, C.byref(p)), 'dh_stream_ready')
        host = np.empty(self.info.n_streams, np.int32)
        assert self.rt.cudaMemcpy(host.ctypes.data, p, host.nbytes, 2) == 0
        return host

    def free(self):
        if self.h:
            _ffi.check(self.lib.dh_stream_free(self.h), 'dh_stream_free')
            self.h = C.c_void_p()


def _same(got, want, what):
    assert len(got) == len(want), what
    for i, (a, b) in enumerate(zip(got, want)):
        assert a.shape == b.shape, (what, i, a.shape, b.shape)
        assert np.array_equal(a, b, equal_nan=True), '%s: output %d differs from ClipStream.push' % (what, i)
        assert np.array_equal(np.isnan(a), np.isnan(b)), (what, i)


def _python(out):
    return [o.cpu().numpy() for o in out.frame_outputs + out.clip_outputs]


def _video(S, n_push, res, seed=17):
    return synth.synth_frames(S * n_push, res, res, seed=seed).reshape(n_push, S, res, res, 3)


def _c_equals_python(torch, tmp_path, m, S, n_push, resets, res, target=None, predict_at=None):
    """ClipStream(target or m) and its export, pushed the same frames with the same resets ('all' = every stream):
    on every push the C outputs equal the Python ones bit for bit and the ready flags equal ClipStream.ready.
    predict_at = (push, stream): that window's clip outputs also against m.predict at 1e-5."""
    T = m.graph.frames_per_clip
    video = _video(S, n_push, res)
    m.use_cuda_graph = True
    cs = ClipStream(target or m, S)
    path = str(tmp_path / 'stream.dhs')
    cs.export(path)
    ctx = _ffi.Context(torch.cuda.current_device())
    c = CStream(ctx, path)
    s = torch.cuda.current_stream().cuda_stream
    seen = set()
    try:
        for i in range(n_push):
            if i in resets:
                ids = None if resets[i] == 'all' else resets[i]
                cs.reset(ids)
                assert c.reset(ids, s) == 0
            x = torch.from_numpy(video[i]).cuda()
            out = cs.push(x)
            c.set_input(x)
            c.push(s)
            torch.cuda.synchronize()
            got = c.outputs()
            _same(got, _python(out), 'push %d' % i)
            assert c.ready().tolist() == out.ready.astype(np.int32).tolist(), i
            seen.add(tuple(out.ready.tolist()))
            if predict_at is not None and predict_at[0] == i:
                k = predict_at[1]
                assert out.ready[k]
                want = m.predict(video[i - T + 1:i + 1, k][None])
                want = want if isinstance(want, list) else [want]
                n_f = c.info.n_frame_outputs
                for o, t in zip(got[n_f:], cs.clip_output_tensors):
                    r = want[m.graph.outputs.index(t)][0]
                    assert np.abs(o[k] - r).max() <= 1e-5, (i, k, t, float(np.abs(o[k] - r).max()))
        assert cs._graph is not None
        assert len(seen) > 2, seen                  # the schedule moved streams in and out of readiness
    finally:
        c.free()


@pytest.mark.parametrize('build', [_penn_t8, _ntu_t16, _merge_2d], ids=['penn_like_t8', 'ntu_like_t16_3d', 'merge_2d'])
def test_c_push_equals_clip_stream(cuda, tmp_path, build):
    m = build().init_synthetic_weights(1234)
    T = m.graph.frames_per_clip
    _c_equals_python(cuda, tmp_path, m, 3, T + 4, {1: [1], T: [2], T + 2: 'all'}, 128)


def test_c_push_equals_clip_stream_of_the_action_view(cuda, tmp_path):
    from deephar_b200 import spnet
    m = _penn_t8().init_synthetic_weights(1234)
    am = spnet.split_model(m, m.cfg)[1]
    T = m.graph.frames_per_clip
    _c_equals_python(cuda, tmp_path, m, 3, T + 4, {1: [1], T: [2], T + 2: 'all'}, 128, target=am)


def test_c_push_equals_clip_stream_c4_full_size(cuda, tmp_path):
    m = _c4().init_synthetic_weights(1234)
    _c_equals_python(cuda, tmp_path, m, 3, 18, {1: [1], 16: [2]}, 256, predict_at=(17, 0))


def test_graph_replay_keeps_readiness_on_the_device(cuda, tmp_path):
    """one dh_stream_push captured after a plain push and replayed 2T + 3 times, with dh_stream_reset between replays
    (outside the graph): outputs and flags equal a second loaded stream driven by plain pushes"""
    torch = cuda
    m = _penn_t8().init_synthetic_weights(1234)
    T, S = m.graph.frames_per_clip, 3
    path = str(tmp_path / 'penn.dhs')
    ClipStream(m, S).export(path)
    video = _video(S, 2 * T + 4, 128, seed=23)
    resets = {3: [1], T + 1: [0, 2], T + 5: None, 2 * T + 1: [2]}
    ctx = _ffi.Context(torch.cuda.current_device())
    a, b = CStream(ctx, path), CStream(ctx, path)
    s = torch.cuda.current_stream().cuda_stream
    g = None
    seen = set()
    try:
        for i in range(2 * T + 4):
            if i in resets:
                assert a.reset(resets[i], s) == 0 and b.reset(resets[i], s) == 0
            x = torch.from_numpy(video[i]).cuda()
            a.set_input(x)
            b.set_input(x)
            if i == 0:
                a.push(s)
                torch.cuda.synchronize()
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    a.push(torch.cuda.current_stream().cuda_stream)
            else:
                g.replay()
            b.push(s)
            torch.cuda.synchronize()
            _same(a.outputs(), b.outputs(), 'replay %d' % i)
            ready = a.ready()
            assert ready.tolist() == b.ready().tolist(), i
            seen.add(tuple(ready.tolist()))
        assert len(seen) >= 3, seen
        del g
    finally:
        a.free()
        b.free()


@pytest.mark.parametrize('S', [1, 3, 257])
@pytest.mark.parametrize('T', [2, 16])
def test_ready_kernel_contract(cuda, S, T):
    torch = cuda
    lib = _ffi.lib()
    ctx = _ffi.Context(torch.cuda.current_device())
    rng = np.random.default_rng(S * 100 + T)
    start = rng.choice([0, T - 1, T], S).astype(np.int32)
    start[:min(S, 3)] = [0, T - 1, T][:min(S, 3)]
    G = 64                                               # guard floats before and after every buffer
    # (item shape of the buffer, channel offset of the view, channels of the view)
    geoms = [((5,), 0, 5), ((4, 4, 7), 0, 7), ((3, 2, 11), 2, 6)]
    bufs, views = [], []
    for shape, off, c in geoms:
        host = rng.standard_normal(2 * G + S * int(np.prod(shape))).astype(np.float32)
        dev = torch.from_numpy(host).cuda()
        bufs.append((host, dev, shape, off, c))
        h, w = (1, 1) if len(shape) == 1 else shape[:2]
        views.append(_ffi.dh_view(dev.data_ptr() + 4 * (G + off), S, h, w, c, shape[-1]))
    table = (_ffi.dh_view * len(views))(*views)
    table_dev = torch.from_numpy(np.frombuffer(bytearray(table), np.uint8).copy()).cuda()
    counts = torch.from_numpy(start.copy()).cuda()
    ready = torch.full((S,), -7, dtype=torch.int32, device='cuda')
    count = start.copy()
    expect = [host.copy() for host, *_ in bufs]         # NaN rows of a call stay NaN: ready rows are never written
    for call in range(2):                                # the second call: counts saturate or keep counting
        rc = lib.dh_stream_ready_f32(ctx.handle, C.c_void_p(counts.data_ptr()), S, T, C.c_void_p(table_dev.data_ptr()),
                                     len(views), C.c_void_p(ready.data_ptr()), torch.cuda.current_stream().cuda_stream)
        _ffi.check(rc, 'dh_stream_ready_f32')
        torch.cuda.synchronize()
        count = np.minimum(count + 1, T)
        assert counts.cpu().numpy().tolist() == count.tolist(), call
        assert ready.cpu().numpy().tolist() == (count >= T).astype(np.int32).tolist(), call
        for want, (host, dev, shape, off, c) in zip(expect, bufs):
            body = want[G:G + S * int(np.prod(shape))].reshape((S, -1, shape[-1]))
            body[count < T, :, off:off + c] = np.float32('nan')
            got = dev.cpu().numpy()
            nanbits = got.view(np.uint32)[G:-G].reshape(body.shape)[count < T][..., off:off + c]
            assert (nanbits == 0x7FC00000).all(), (call, shape)
            assert np.array_equal(got.view(np.uint32)[np.isfinite(want)], want.view(np.uint32)[np.isfinite(want)])
            assert np.array_equal(np.isnan(got), np.isnan(want)), (call, shape)


def test_launches_per_push_and_no_new_fallback(cuda, tmp_path):
    torch = cuda
    lib = _ffi.lib()
    m = _penn_t8().init_synthetic_weights(1234)
    S = 3
    m.use_cuda_graph = False
    cs = ClipStream(m, S)
    x = torch.from_numpy(_video(S, 1, 128)[0]).cuda()
    cs.push(x)
    torch.cuda.synchronize()
    m._ctx.launch_count(reset=True)
    lib.dh_fallback_count(m._ctx.handle, 1)
    cs.push(x)
    py_launches = m._ctx.launch_count(reset=True)
    py_fallbacks = int(lib.dh_fallback_count(m._ctx.handle, 1))
    # launches_per_push() counts one launch per separable conv on the tensor-core build; one the CUDA-core kernels
    # take runs as two (depthwise, then pointwise)
    simt_sep = sum(1 for b in (cs._frame, cs._clip) for k, info in b.conv_plans if k.kind == 'sepconv' and info.path == 0)
    assert py_launches == cs.launches_per_push() + simt_sep
    path = str(tmp_path / 'penn.dhs')
    cs.export(path)
    ctx = _ffi.Context(torch.cuda.current_device())
    c = CStream(ctx, path)
    s = torch.cuda.current_stream().cuda_stream
    try:
        c.set_input(x)
        c.push(s)
        torch.cuda.synchronize()
        ctx.launch_count(reset=True)
        lib.dh_fallback_count(ctx.handle, 1)
        c.push(s)
        assert ctx.launch_count(reset=True) == py_launches + 1 == cs.launches_per_push() + 1 + simt_sep
        assert int(lib.dh_fallback_count(ctx.handle, 1)) <= py_fallbacks
    finally:
        c.free()


def test_streams_and_a_model_in_one_context_stay_independent(cuda, tmp_path):
    torch = cuda
    ma = _penn_t8().init_synthetic_weights(1234)
    mb = _merge_2d().init_synthetic_weights(77)
    Ta, Sa, Sb = ma.graph.frames_per_clip, 3, 2
    ma.use_cuda_graph = mb.use_cuda_graph = False
    pa, pb, pm = str(tmp_path / 'a.dhs'), str(tmp_path / 'b.dhs'), str(tmp_path / 'm.dhm')
    csa, csb = ClipStream(ma, Sa), ClipStream(mb, Sb)
    csa.export(pa)
    csb.export(pb)
    ma.export(pm, Ta)
    n = Ta + 2
    va, vb = _video(Sa, n + 1, 128, seed=1), _video(Sb, n, 128, seed=2)
    clip = torch.from_numpy(_video(1, Ta, 128, seed=3).reshape(1, Ta, 128, 128, 3)).cuda()
    want_m = [o.cpu().numpy() for o in ma.forward_device(clip)]
    ctx = _ffi.Context(torch.cuda.current_device())
    a, b, cm = CStream(ctx, pa), CStream(ctx, pb), CModel(ctx, pm)
    s = torch.cuda.current_stream().cuda_stream
    try:
        cm.set_input(clip.cpu().numpy())
        for i in range(n):
            xa, xb = torch.from_numpy(va[i]).cuda(), torch.from_numpy(vb[i]).cuda()
            a.set_input(xa)
            a.push(s)
            cm.forward(s)
            b.set_input(xb)
            b.push(s)
            want_a, want_b = _python(csa.push(xa)), _python(csb.push(xb))
            torch.cuda.synchronize()
            _same(a.outputs(), want_a, 'stream a, push %d' % i)
            _same(b.outputs(), want_b, 'stream b, push %d' % i)
            _same(cm.outputs(), want_m, 'model, push %d' % i)
            assert a.ready().tolist() == csa.ready.astype(np.int32).tolist()
            assert b.ready().tolist() == csb.ready.astype(np.int32).tolist()
        # a reset with an id out of range changes nothing: the next push equals a push without it
        assert a.reset([0, Sa], s) < 0 and a.reset([-1], s) < 0
        assert 'outside' in _ffi.lib().dh_last_error().decode()
        x = torch.from_numpy(va[n]).cuda()
        a.set_input(x)
        a.push(s)
        want = _python(csa.push(x))
        torch.cuda.synchronize()
        _same(a.outputs(), want, 'after a refused reset')
        assert a.ready().tolist() == [1] * Sa
        v = _ffi.dh_view()
        for k in (-1, a.n_outputs):
            assert _ffi.lib().dh_stream_output(a.h, k, C.byref(v), None) < 0
    finally:
        a.free()
        b.free()
        cm.free()


def test_free_returns_all_device_memory(cuda, tmp_path):
    torch = cuda
    m = _penn_t8().init_synthetic_weights(1234)
    path = str(tmp_path / 'penn.dhs')
    ClipStream(m, 3).export(path)
    x = torch.from_numpy(_video(3, 1, 128)[0]).cuda()
    rt = _cudart()
    ctx = _ffi.Context(torch.cuda.current_device())
    free0, free1, total = C.c_size_t(), C.c_size_t(), C.c_size_t()
    for cycle in range(2):          # the first cycle also loads what the runtime loads lazily
        torch.cuda.synchronize()
        assert rt.cudaMemGetInfo(C.byref(free0), C.byref(total)) == 0
        c = CStream(ctx, path)
        c.set_input(x)
        c.push(torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        assert rt.cudaMemGetInfo(C.byref(free1), C.byref(total)) == 0
        assert free0.value - free1.value >= c.info.device_bytes
        c.free()
    assert rt.cudaMemGetInfo(C.byref(free1), C.byref(total)) == 0
    assert free1.value == free0.value, (free0.value, free1.value)


def test_c_example_writes_the_same_bytes(cuda, tmp_path):
    """examples/run_stream.c built with the documented line and run as its own process, plain and graph-replayed"""
    torch = cuda
    cc = shutil.which('gcc') or shutil.which('cc')
    assert cc, 'no C compiler'
    cuda_home = os.environ.get('CUDA_HOME', '/usr/local/cuda')
    libdir = os.path.dirname(_ffi.LIB_PATH)
    exe = str(tmp_path / 'run_stream')
    subprocess.check_call([cc, '-std=c99', '-O2', '-Wall', '-Werror', '-I', os.path.join(ROOT, 'include'),
                           '-I', os.path.join(cuda_home, 'include'), os.path.join(ROOT, 'examples', 'run_stream.c'),
                           '-o', exe, '-L', libdir, '-ldeephar_b200', '-L', os.path.join(cuda_home, 'lib64'), '-lcudart',
                           '-Wl,-rpath,' + libdir + ':' + os.path.join(cuda_home, 'lib64')])
    m = _penn_t8().init_synthetic_weights(1234)
    T, S = m.graph.frames_per_clip, 3
    n_push = T + 4
    resets = {1: [1], T: [2], T + 2: None}
    video = _video(S, n_push, 128, seed=31)
    cs = ClipStream(m, S)
    path, frames, rfile, prefix = [str(tmp_path / f) for f in ('penn.dhs', 'frames.f32', 'resets.txt', 'out')]
    cs.export(path)
    video.tofile(frames)
    with open(rfile, 'w') as f:
        for i, ids in sorted(resets.items()):
            f.write('%d %s\n' % (i, ' '.join(str(k) for k in (ids or []))))
    want, ready = [], []
    for i in range(n_push):
        if i in resets:
            cs.reset(resets[i])
        out = cs.push(torch.from_numpy(video[i]).cuda())
        want.append(_python(out))
        ready.append(out.ready.astype(np.int32))
    env = {k: v for k, v in os.environ.items() if not k.startswith('PYTHON')}
    out = subprocess.run([exe, path, frames, prefix, rfile], capture_output=True, text=True, timeout=600, env=env)
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-2000:]
    for tag in ('', 'graph.'):
        for k in range(len(want[0])):
            got = np.fromfile('%s.%s%d.f32' % (prefix, tag, k), np.float32).reshape((n_push,) + want[0][k].shape)
            _same([got[i] for i in range(n_push)], [w[k] for w in want], 'run_stream %s output %d' % (tag or 'plain', k))
        got = np.fromfile('%s.%sready.i32' % (prefix, tag), np.int32).reshape(n_push, S)
        assert got.tolist() == np.stack(ready).tolist(), tag


def test_c_push_time_against_clip_stream(cuda, tmp_path):
    """C4 at S = 8: graph replays of dh_stream_push against ClipStream.push (itself a graph replay plus the host's
    readiness bookkeeping), interleaved, best of three"""
    torch = cuda
    m = _c4().init_synthetic_weights(1234)
    m.use_cuda_graph = True
    S = 8
    cs = ClipStream(m, S)
    x = torch.from_numpy(_video(S, 1, 256, seed=5)[0]).cuda()
    cs.push(x)
    cs.push(x)                                       # second push: captured into the stream's graph
    path = str(tmp_path / 'c4.dhs')
    cs.export(path)
    ctx = _ffi.Context(torch.cuda.current_device())
    c = CStream(ctx, path)
    try:
        c.set_input(x)
        c.push(torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            c.push(torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()

        def timed(fn, reps=20):
            for _ in range(3):
                fn()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(reps):
                fn()
            e1.record()
            e1.synchronize()
            return e0.elapsed_time(e1) / reps
        t_py, t_c = [], []
        for _ in range(3):
            t_py.append(timed(lambda: cs.push(x)))
            t_c.append(timed(g.replay))
        print('\nC4 x %d streams (%s): ClipStream.push %.3f ms, dh_stream_push (graph replay) %.3f ms, ratio %.3f'
              % (S, torch.cuda.get_device_name(), min(t_py), min(t_c), min(t_c) / min(t_py)))
        # the numbers are the report; the bound only catches a C path that adds work (the GPU may be shared)
        assert min(t_c) <= 1.5 * min(t_py), (t_py, t_c)
        del g
    finally:
        c.free()
