"""Model.export on the GPU: the exported file, loaded and run through the C ABI (dh_model_load / dh_model_forward),
computes what forward_device computes, bit for bit -- on the BASELINE configs at the batch sizes bench.py runs (C2 at
256 frames, C4 at 16 clips x 16 frames), C3, C5, both merge models, a keras_compat model, an SPNet action view and random
graphs of the compiler fuzzer; as plain launches and as a CUDA-graph replay; at precision 1 and on the CUDA-core path.
examples/run_model.c, a plain C program with no Python in its process, writes the same bytes.  Two models in one
context stay independent, and dh_model_free returns every byte dh_model_load took.

    pytest -m gpu tests/test_gpu_model_export.py -s        (-s: the C vs Python forward times of C2)
"""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

from deephar_b200 import _ffi, spnet
from deephar_b200.config import ModelConfig, pa16j2d
from deephar_b200.model import Model

from test_compiler_fuzz import _random_graph
from test_gpu_launch_contracts import _build, _input

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _cudart():
    _ffi.lib()                                       # libcudart.so.12 is loaded with the library: bind that one
    rt = C.CDLL('libcudart.so.12')
    rt.cudaMemcpy.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int]
    rt.cudaMemcpy2D.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t, C.c_int]
    rt.cudaMemset2DAsync.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_size_t, C.c_size_t, C.c_void_p]
    rt.cudaMemGetInfo.argtypes = [C.POINTER(C.c_size_t), C.POINTER(C.c_size_t)]
    return rt


def _inspect(path):
    info = _ffi.dh_model_info()
    _ffi.check(_ffi.lib().dh_model_inspect(path.encode(), C.byref(info), None, 0, None, 0), 'dh_model_inspect')
    return info


class CModel(object):
    """a loaded model file, driven through the C ABI only"""

    def __init__(self, ctx, path):
        self.lib, self.rt = _ffi.lib(), _cudart()
        self.n_outputs = _inspect(path).n_outputs
        self.h = C.c_void_p()
        _ffi.check(self.lib.dh_model_load(ctx.handle, path.encode(), C.byref(self.h)), 'dh_model_load')

    def set_input(self, x):
        v = _ffi.dh_view()
        _ffi.check(self.lib.dh_model_input(self.h, C.byref(v)), 'dh_model_input')
        x = np.ascontiguousarray(x, np.float32)
        assert x.size == v.n * v.h * v.w * v.c and v.ld == v.c
        assert self.rt.cudaMemcpy(v.p, x.ctypes.data, x.nbytes, 1) == 0

    def forward(self, stream):
        _ffi.check(self.lib.dh_model_forward(self.h, stream), 'dh_model_forward')

    def _output(self, k):
        v, info = _ffi.dh_view(), _ffi.dh_model_output_info()
        _ffi.check(self.lib.dh_model_output(self.h, k, C.byref(v), C.byref(info)), 'dh_model_output')
        return v, info

    def outputs(self):
        res = []
        for k in range(self.n_outputs):
            v, info = self._output(k)
            rows = v.n * v.h * v.w
            host = np.empty((rows, v.c), np.float32)
            assert self.rt.cudaMemcpy2D(host.ctypes.data, v.c * 4, v.p, v.ld * 4, v.c * 4, rows, 2) == 0
            res.append(host.reshape(tuple(info.shape[:info.rank])))
        return res

    def clear_outputs(self, stream):
        for k in range(self.n_outputs):
            v, _ = self._output(k)
            assert self.rt.cudaMemset2DAsync(v.p, v.ld * 4, 0, v.c * 4, v.n * v.h * v.w, stream) == 0

    def free(self):
        if self.h:
            _ffi.check(self.lib.dh_model_free(self.h), 'dh_model_free')
            self.h = C.c_void_p()


def _case(torch, name):
    """name -> (model, exported object (the model or a view of it), device input, indices of the outputs exported)"""
    if name == 'keras_compat':
        from test_keras_compat import _models
        m = _models()[0]
        x = torch.from_numpy(np.random.default_rng(0).uniform(-1, 1, (3, 32, 32, 3)).astype(np.float32)).cuda()
        return m.init_synthetic_weights(7), m, x, None
    if name == 'spnet_action_view':
        cfg = ModelConfig((2, 128, 128, 3), pa16j2d, num_actions=[15], num_pyramids=2, action_pyramids=[1, 2],
                          num_levels=4, pose_replica=True, num_pose_features=160, num_visual_features=160)
        m = spnet.build(cfg).init_synthetic_weights(1234)
        view = spnet.split_model(m, cfg)[1]
        return m, view, _input(torch, m, 2, seed=5), view.indices
    if name.startswith('fuzz'):
        seed = int(name[4:])
        g, side = _random_graph(seed)
        m = Model(g, name=g.name).init_synthetic_weights(seed)
        x = np.random.default_rng(1000 + seed).uniform(-1, 1, (3, side, side, 3)).astype(np.float32)
        return m, m, torch.from_numpy(x).cuda(), None
    which, items = name.split('-')
    m = _build(which).init_synthetic_weights(1234)
    return m, m, _input(torch, m, int(items), seed=3), None


def _expected(m, x, idx):
    outs = [o.cpu().numpy() for o in m.forward_device(x)]
    return outs if idx is None else [outs[i] for i in idx]


def _same(got, want, what):
    assert len(got) == len(want), what
    for i, (a, b) in enumerate(zip(got, want)):
        assert a.shape == b.shape, (what, i, a.shape, b.shape)
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), '%s: output %d differs from forward_device' % (what, i)


def _run_file(torch, path, x, want, what, graph=True):
    """load the file in a fresh context, one plain forward and (graph=True) one captured replay; both must give `want`"""
    ctx = _ffi.Context(torch.cuda.current_device())
    cm = CModel(ctx, path)
    try:
        cm.set_input(x.cpu().numpy())
        stream = torch.cuda.current_stream()
        cm.forward(stream.cuda_stream)
        torch.cuda.synchronize()
        _same(cm.outputs(), want, what + ', plain launches')
        if graph:
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                cm.forward(torch.cuda.current_stream().cuda_stream)
            cm.clear_outputs(stream.cuda_stream)
            g.replay()
            torch.cuda.synchronize()
            _same(cm.outputs(), want, what + ', CUDA-graph replay')
            del g
    finally:
        cm.free()


CASES = ['C2-256', 'C3-32', 'C4-16', 'C5-2', 'merge2d-1', 'merge3d-1', 'keras_compat', 'spnet_action_view'] + \
    ['fuzz%d' % s for s in range(8)]


@pytest.mark.parametrize('name', CASES)
def test_c_forward_equals_forward_device(cuda, tmp_path, name):
    m, exp, x, idx = _case(cuda, name)
    want = _expected(m, x, idx)
    n_frames = int(np.prod(x.shape[:-3]))
    path = str(tmp_path / (name + '.dhm'))
    exp.export(path, n_frames)
    info = _inspect(path)
    assert info.n_launches == len(m.plan.kops) and info.n_outputs == len(want)
    _run_file(cuda, path, x, want, name)
    m._bound = {}
    cuda.cuda.empty_cache()


@pytest.mark.parametrize('setting', ['precision1', 'cuda_cores'])
def test_c_forward_equals_forward_device_off_the_defaults(cuda, tmp_path, setting):
    for name in ('C2-8', 'merge2d-1', 'fuzz3') if setting == 'precision1' else ('C2-8', 'C4-1', 'merge2d-1', 'keras_compat',
                                                                                 'fuzz3'):
        m, exp, x, idx = _case(cuda, name)
        if setting == 'precision1':
            m.precision = 1
        else:
            m.use_tensor_cores = False
        want = _expected(m, x, idx)
        path = str(tmp_path / (name + '.dhm'))
        exp.export(path, int(np.prod(x.shape[:-3])))
        info = _inspect(path)
        assert info.precision == m.precision and info.use_tensor_cores == (setting != 'cuda_cores')
        _run_file(cuda, path, x, want, '%s %s' % (name, setting))


def test_two_models_in_one_context_stay_independent(cuda, tmp_path):
    ma, _, xa, _ = _case(cuda, 'C2-4')
    mb, _, xb, _ = _case(cuda, 'fuzz5')
    wa, wb = _expected(ma, xa, None), _expected(mb, xb, None)
    xa2 = xa.flip(0).contiguous()
    wa2 = _expected(ma, xa2, None)
    pa, pb = str(tmp_path / 'a.dhm'), str(tmp_path / 'b.dhm')
    ma.export(pa, 4)
    mb.export(pb, 3)
    ctx = _ffi.Context(cuda.cuda.current_device())
    a, b = CModel(ctx, pa), CModel(ctx, pb)
    s = cuda.cuda.current_stream().cuda_stream
    try:
        a.set_input(xa.cpu().numpy())
        b.set_input(xb.cpu().numpy())
        a.forward(s)
        b.forward(s)
        cuda.cuda.synchronize()
        _same(a.outputs(), wa, 'model a after model b ran')
        _same(b.outputs(), wb, 'model b')
        a.set_input(xa2.cpu().numpy())
        a.forward(s)
        cuda.cuda.synchronize()
        _same(a.outputs(), wa2, 'model a, second input')
        _same(b.outputs(), wb, 'model b after model a ran again')
    finally:
        a.free()
        b.free()


def test_free_returns_all_device_memory(cuda, tmp_path):
    m, _, x, _ = _case(cuda, 'C2-8')
    want = _expected(m, x, None)                     # loads every kernel the file uses
    path = str(tmp_path / 'c2.dhm')
    m.export(path, 8)
    rt = _cudart()
    ctx = _ffi.Context(cuda.cuda.current_device())
    free0, free1, total = C.c_size_t(), C.c_size_t(), C.c_size_t()
    for cycle in range(2):          # the first cycle also loads what the runtime loads lazily (its memset kernels)
        cuda.cuda.synchronize()
        assert rt.cudaMemGetInfo(C.byref(free0), C.byref(total)) == 0
        cm = CModel(ctx, path)
        cm.set_input(x.cpu().numpy())
        cm.forward(cuda.cuda.current_stream().cuda_stream)
        cuda.cuda.synchronize()
        _same(cm.outputs(), want, 'C2-8')
        assert rt.cudaMemGetInfo(C.byref(free1), C.byref(total)) == 0
        assert free0.value - free1.value >= _inspect(path).device_bytes
        cm.free()
    assert rt.cudaMemGetInfo(C.byref(free1), C.byref(total)) == 0
    assert free1.value == free0.value, (free0.value, free1.value)


def test_c_example_writes_the_same_bytes(cuda, tmp_path):
    """examples/run_model.c built with the documented line and run as its own process"""
    cc = shutil.which('gcc') or shutil.which('cc')
    assert cc, 'no C compiler'
    cuda_home = os.environ.get('CUDA_HOME', '/usr/local/cuda')
    libdir = os.path.dirname(_ffi.LIB_PATH)
    exe = str(tmp_path / 'run_model')
    subprocess.check_call([cc, '-std=c99', '-O2', '-Wall', '-Werror', '-I', os.path.join(ROOT, 'include'),
                           '-I', os.path.join(cuda_home, 'include'), os.path.join(ROOT, 'examples', 'run_model.c'),
                           '-o', exe, '-L', libdir, '-ldeephar_b200', '-L', os.path.join(cuda_home, 'lib64'), '-lcudart',
                           '-Wl,-rpath,' + libdir + ':' + os.path.join(cuda_home, 'lib64')])
    for name in ('C4-2', 'merge3d-1'):
        m, exp, x, idx = _case(cuda, name)
        want = _expected(m, x, idx)
        path, xin, prefix = str(tmp_path / (name + '.dhm')), str(tmp_path / (name + '.in.f32')), str(tmp_path / name)
        exp.export(path, int(np.prod(x.shape[:-3])))
        x.cpu().numpy().tofile(xin)
        env = {k: v for k, v in os.environ.items() if not k.startswith('PYTHON')}
        out = subprocess.run([exe, path, xin, prefix], capture_output=True, text=True, timeout=600, env=env)
        assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-2000:]
        for tag in ('', 'graph.'):
            got = [np.fromfile('%s.%s%d.f32' % (prefix, tag, k), np.float32).reshape(w.shape) for k, w in enumerate(want)]
            _same(got, want, '%s: run_model %s' % (name, tag or 'plain'))
        m._bound = {}


def test_c_forward_time_matches_forward_device(cuda, tmp_path):
    """C2 at 256 frames, both as CUDA-graph replays of the same launch list: the C ABI adds no device work"""
    m, _, x, _ = _case(cuda, 'C2-256')
    want = _expected(m, x, None)
    m.forward_device(x)                              # second call: captured into the model's graph
    path = str(tmp_path / 'c2.dhm')
    m.export(path, 256)
    ctx = _ffi.Context(cuda.cuda.current_device())
    cm = CModel(ctx, path)
    try:
        cm.set_input(x.cpu().numpy())
        s = cuda.cuda.current_stream()
        cm.forward(s.cuda_stream)
        g = cuda.cuda.CUDAGraph()
        with cuda.cuda.graph(g):
            cm.forward(cuda.cuda.current_stream().cuda_stream)
        cuda.cuda.synchronize()

        def timed(fn, reps=20):
            for _ in range(3):
                fn()
            e0, e1 = cuda.cuda.Event(enable_timing=True), cuda.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(reps):
                fn()
            e1.record()
            e1.synchronize()
            return e0.elapsed_time(e1) / reps
        t_py, t_c = [], []
        for _ in range(3):                            # interleaved, best of three
            t_py.append(timed(lambda: m.forward_device(x)))
            t_c.append(timed(g.replay))
        g.replay()
        cuda.cuda.synchronize()
        _same(cm.outputs(), want, 'C2-256 timed replay')
        print('\nC2 x 256 frames: forward_device %.3f ms, dh_model_forward (graph replay) %.3f ms, ratio %.3f'
              % (min(t_py), min(t_c), min(t_c) / min(t_py)))
        # the number is the report; the bound only catches a C path that adds work (the GPU may be shared)
        assert min(t_c) <= 1.5 * min(t_py), (t_py, t_c)
        del g
    finally:
        cm.free()
