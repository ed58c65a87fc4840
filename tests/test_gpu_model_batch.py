"""Model files run at fewer items than they were exported at (dh_model_set_batch), on the GPU.

Each case is exported at N items (frames, or clips of a clip model) and loaded once; at every n the C forward must
equal forward_device on the same first n items bit for bit -- both issue the same entry points with the same arguments
apart from pointers -- and leave items n .. N-1 of every output as the NaN sentinel written before it.  Cases: C2 at
full size exported at 40 frames (also at a batch whose persistent tensor-core kernels end on a different partial round
of tiles), C3 at 5 frames, C4 and C5 at 3 and 2 clips, both merge models at 3 clips, C2 with use_tensor_cores = False
and random graphs of the compiler fuzzer.  Also: a CUDA graph captured per batch replays equal to plain launches and keeps its
batch after the next dh_model_set_batch; setting the batch back to N gives the original bytes; refused batches change
nothing and launch nothing; a version-1 file runs at N only; examples/run_model.c with a batch argument writes the
forward_device bytes.

    pytest -m gpu tests/test_gpu_model_batch.py
"""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

from deephar_b200 import _ffi, export

from test_gpu_launch_contracts import _build, _input
from test_gpu_model_export import CModel, _case, _expected, _same

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SENTINEL = 0xFFFFFFFF           # every byte 0xFF: a NaN no kernel writes
PERSISTENT_PATHS = (1, 2, 4)    # dh_conv_plan_info.path of the persistent tensor-core kernels


class BModel(CModel):
    def set_batch(self, n):
        return self.lib.dh_model_set_batch(self.h, n)

    def batch(self):
        return self.lib.dh_model_batch(self.h)

    def input_view(self):
        v = _ffi.dh_view()
        _ffi.check(self.lib.dh_model_input(self.h, C.byref(v)), 'dh_model_input')
        return v

    def views(self):
        return [self._output(k)[0] for k in range(self.n_outputs)]


def _fill(rt, views, stream):
    for v in views:
        assert rt.cudaMemset2DAsync(v.p, v.ld * 4, 0xFF, v.c * 4, v.n * v.h * v.w, stream) == 0


def _untouched(rt, views, N, n, what):
    """items n .. N-1 of the N-item output views still hold the sentinel"""
    for k, v in enumerate(views):
        rows = v.n * v.h * v.w
        host = np.empty((rows, v.c), np.uint32)
        assert rt.cudaMemcpy2D(host.ctypes.data, v.c * 4, v.p, v.ld * 4, v.c * 4, rows, 2) == 0
        first = v.n // N * n * v.h * v.w
        assert (host[first:] == SENTINEL).all(), '%s: output %d was written past item %d' % (what, k, n)


def _tail_batch(m, N, avoid):
    """A batch at which some persistent tensor-core convolution runs more than one round of tiles per CTA and ends
    on a partial round of another size than at N: read from the library's plans as forward_device binds them."""
    def tails(n):
        b = m._bind_plan(m.plan, n)
        out = {id(k): (info.n_mtiles, info.grid_x) for k, info in b.conv_plans if info.path in PERSISTENT_PATHS}
        del b
        return out
    at_n = tails(N)
    for n in range(N - 2, 2, -1):
        if n in avoid:
            continue
        for key, (tiles, grid) in tails(n).items():
            if tiles > grid and tiles % grid and tiles % grid != at_n[key][0] % at_n[key][1]:
                return n
    raise AssertionError('no batch below %d changes a persistent kernel\'s last round' % N)


def _run_batches(torch, tmp_path, name, m, exp, x, idx, ns):
    """export at N = len(x) items, then at each n in ns: C forward vs forward_device, untouched items, graph replay"""
    N = x.shape[0]
    T = m.graph.frames_per_clip
    path = str(tmp_path / (name + '.dhm'))
    exp.export(path, N * T)
    want_full = _expected(m, x, idx)
    ctx = _ffi.Context(torch.cuda.current_device())
    cm = BModel(ctx, path)
    stream = torch.cuda.current_stream()
    s = stream.cuda_stream
    graphs = {}
    try:
        assert cm.batch() == N
        cm.set_input(x.cpu().numpy())
        cm.forward(s)
        torch.cuda.synchronize()
        first = cm.outputs()
        _same(first, want_full, '%s at N = %d' % (name, N))
        full_views = cm.views()
        for n in ns:
            what = '%s at n = %d of %d' % (name, n, N)
            assert cm.set_batch(n) == 0, cm.lib.dh_last_error()
            assert cm.batch() == n
            assert cm.input_view().n == n * T
            for v, full in zip(cm.views(), full_views):
                assert (v.p, v.h, v.w, v.c, v.ld) == (full.p, full.h, full.w, full.c, full.ld)
                assert v.n == full.n // N * n
            xs = x[:n].contiguous()
            want = _expected(m, xs, idx)
            _fill(cm.rt, full_views, s)
            cm.set_input(xs.cpu().numpy())
            cm.forward(s)
            torch.cuda.synchronize()
            got = cm.outputs()
            for o in got:
                assert o.shape[0] == n
            _same(got, want, what + ', plain launches')
            _untouched(cm.rt, full_views, N, n, what)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                cm.forward(torch.cuda.current_stream().cuda_stream)
            _fill(cm.rt, full_views, s)
            g.replay()
            torch.cuda.synchronize()
            _same(cm.outputs(), want, what + ', CUDA-graph replay')
            _untouched(cm.rt, full_views, N, n, what + ', CUDA-graph replay')
            graphs[n] = (g, want)
        # a graph keeps the batch it was captured at, whatever the model's batch now is
        n1 = ns[0]
        g, want = graphs[n1]
        assert cm.set_batch(N) == 0
        cm.set_input(x.cpu().numpy())
        _fill(cm.rt, full_views, s)
        g.replay()
        torch.cuda.synchronize()
        _untouched(cm.rt, full_views, N, n1, '%s: graph of n = %d replayed at batch %d' % (name, n1, N))
        assert cm.set_batch(n1) == 0
        _same(cm.outputs(), want, '%s: graph of n = %d replayed at batch %d' % (name, n1, N))
        # back at N: the original bytes
        assert cm.set_batch(N) == 0 and cm.batch() == N
        cm.forward(s)
        torch.cuda.synchronize()
        _same(cm.outputs(), first, '%s back at N' % name)
    finally:
        graphs.clear()
        cm.free()
    m._bound = {}
    torch.cuda.empty_cache()
    return path


CASES = [('C2', 40), ('C3', 5), ('C4', 3), ('C5', 2), ('merge2d', 3), ('merge3d', 3)]


@pytest.mark.parametrize('which,N', CASES)
def test_batches_equal_forward_device(cuda, tmp_path, which, N):
    m = _build(which).init_synthetic_weights(1234)
    x = _input(cuda, m, N, seed=11)
    ns = sorted({1, 2, N - 1, N} - {0})
    if which == 'C2':
        ns.append(_tail_batch(m, N, ns))
    _run_batches(cuda, tmp_path, which, m, m, x, None, ns)


def test_batches_equal_forward_device_on_cuda_cores(cuda, tmp_path):
    m = _build('C2').init_synthetic_weights(1234)
    m.use_tensor_cores = False
    x = _input(cuda, m, 5, seed=12)
    path = _run_batches(cuda, tmp_path, 'C2_cuda_cores', m, m, x, None, [1, 2, 4, 5])
    assert export.read(path)['use_tensor_cores'] == 0


@pytest.mark.parametrize('seed', range(8))
def test_fuzz_batches_equal_forward_device(cuda, tmp_path, seed):
    m, exp, x, idx = _case(cuda, 'fuzz%d' % seed)
    _run_batches(cuda, tmp_path, 'fuzz%d' % seed, m, exp, x, idx, [1, 2, 3])


def test_refused_batches_change_nothing(cuda, tmp_path):
    m, exp, x, idx = _case(cuda, 'merge2d-3')
    path = str(tmp_path / 'm.dhm')
    exp.export(path, 3 * m.graph.frames_per_clip)
    ctx = _ffi.Context(cuda.cuda.current_device())
    cm = BModel(ctx, path)
    try:
        assert cm.set_batch(2) == 0
        views = [(v.p, v.n) for v in cm.views()]
        cuda.cuda.synchronize()
        for n in (0, 4, -1, -(1 << 31)):
            launches = ctx.launch_count()
            assert cm.set_batch(n) < 0
            err = cm.lib.dh_last_error().decode()
            assert 'dh_model_set_batch' in err and 'outside [1, 3]' in err, err
            assert cm.batch() == 2 and ctx.launch_count() == launches
            assert [(v.p, v.n) for v in cm.views()] == views and cm.input_view().n == 2 * m.graph.frames_per_clip
        # an accepted call is host-only too
        launches = ctx.launch_count()
        assert cm.set_batch(1) == 0 and ctx.launch_count() == launches
    finally:
        cm.free()


def test_version_1_files_run_at_their_batch_only(cuda, tmp_path):
    m, exp, x, idx = _case(cuda, 'C2-4')
    want = _expected(m, x, idx)
    path = str(tmp_path / 'v2.dhm')
    exp.export(path, 4)
    rec = export.read(path)
    data = bytearray(open(path, 'rb').read())
    at = 8 + 4 + 20 + 4 + 8 * len(rec['input_shape']) + 8 + len(rec['weights']) + 8 + len(rec['packed']) + \
        4 + 8 * len(rec['slot_bytes'])
    v1 = data[:at] + data[at + len(rec['slot_bytes']):]
    v1[8:12] = (1).to_bytes(4, 'little')
    p1 = str(tmp_path / 'v1.dhm')
    with open(p1, 'wb') as f:
        f.write(bytes(v1))
    ctx = _ffi.Context(cuda.cuda.current_device())
    cm = BModel(ctx, p1)
    try:
        assert cm.batch() == 4
        for n in (1, 3):
            assert cm.set_batch(n) < 0
            err = cm.lib.dh_last_error().decode()
            assert 'version 1' in err and 'export the model again' in err, err
            assert cm.batch() == 4
        assert cm.set_batch(4) == 0
        cm.set_input(x.cpu().numpy())
        cm.forward(cuda.cuda.current_stream().cuda_stream)
        cuda.cuda.synchronize()
        _same(cm.outputs(), want, 'version-1 file')
    finally:
        cm.free()


def test_c_example_with_a_batch_writes_the_same_bytes(cuda, tmp_path):
    cc = shutil.which('gcc') or shutil.which('cc')
    assert cc, 'no C compiler'
    cuda_home = os.environ.get('CUDA_HOME', '/usr/local/cuda')
    libdir = os.path.dirname(_ffi.LIB_PATH)
    exe = str(tmp_path / 'run_model')
    subprocess.check_call([cc, '-std=c99', '-O2', '-Wall', '-Werror', '-I', os.path.join(ROOT, 'include'),
                           '-I', os.path.join(cuda_home, 'include'), os.path.join(ROOT, 'examples', 'run_model.c'),
                           '-o', exe, '-L', libdir, '-ldeephar_b200', '-L', os.path.join(cuda_home, 'lib64'), '-lcudart',
                           '-Wl,-rpath,' + libdir + ':' + os.path.join(cuda_home, 'lib64')])
    env = {k: v for k, v in os.environ.items() if not k.startswith('PYTHON')}
    for name, n in (('C4-3', 2), ('merge3d-3', 1), ('fuzz2', 2)):
        m, exp, x, idx = _case(cuda, name)
        N = x.shape[0]
        path, xin, prefix = str(tmp_path / (name + '.dhm')), str(tmp_path / (name + '.in.f32')), str(tmp_path / name)
        exp.export(path, N * m.graph.frames_per_clip)
        xs = x[:n].contiguous()
        want = _expected(m, xs, idx)
        xs.cpu().numpy().tofile(xin)
        out = subprocess.run([exe, path, xin, prefix, str(n)], capture_output=True, text=True, timeout=600, env=env)
        assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-2000:]
        assert 'batch %d of %d' % (n, N) in out.stdout
        for tag in ('', 'graph.'):
            got = [np.fromfile('%s.%s%d.f32' % (prefix, tag, k), np.float32).reshape(w.shape) for k, w in enumerate(want)]
            _same(got, want, '%s: run_model %s at n = %d' % (name, tag or 'plain', n))
        bad = subprocess.run([exe, path, xin, prefix, str(N + 1)], capture_output=True, text=True, timeout=600, env=env)
        assert bad.returncode == 2 and 'BATCH' in bad.stderr
        m._bound = {}
