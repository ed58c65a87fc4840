"""A stand-in CUDA device for HOST-LOGIC tests -- TEST INFRASTRUCTURE (never imported by the product).

    python tests/fake_cuda.py bench.py --gpus 1 --steps 1 ...          (or under torch.distributed.run)

`install()` makes the host side of deephar_b200 and bench.py runnable on a machine without a GPU so that their control
flow can be exercised: `torch.cuda` reports one device whose "device memory" is host memory (`device='cuda'` allocations,
`.cuda()`, `.pin_memory()` become host tensors), streams / events / graphs are inert objects (an event pair reports wall
time), `init_process_group('nccl')` becomes gloo, and the C library keeps its pure host entry points (`dh_tc_k_pad`,
`dh_version`, ...) while EVERY DEVICE ENTRY POINT IS A NO-OP RETURNING 0.  No arithmetic is done: outputs are whatever the
buffers held.  What this covers is everything around the kernels -- batching, shard arithmetic, buffer binding, descriptor
construction (ctypes argument types are still checked by the stubs' signatures), copy pipelining, the collective plumbing
and the JSON line of bench.py -- at any world size.  Numbers printed under it mean nothing and are labelled as such.

`install(arithmetic=True)` goes one step further for the entry points of the model forward (convolutions, pooling,
upsampling, adds, soft-argmax heads, kronecker product, action-head ops): the stubs decode their raw arguments -- `dh_view`
pointers with channel offsets and leading dimensions, `dh_conv_desc` with its scale / shift / residual / pooled-output
fields, weight pointers into the model's flat arena -- exactly as the CUDA side does, and compute the entry point's
float64 contract (tests/kernel_contracts.py, shared with the plan emulator), rounding to the fp32 buffers.  `Model.predict`
then produces real numbers on the CPU through the product's OWN `_bind` / `_Bound.issue` / copy pipeline, which
tests/test_host_path.py compares with the oracle.  Still test infrastructure: the product never imports this file and has
no CPU path.
"""
import contextlib
import ctypes as C
import os
import runpy
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import kernel_contracts as K  # noqa: E402

HOST_ENTRY_POINTS = ('dh_tc_k_pad', 'dh_tc_cout_pad', 'dh_version', 'dh_last_error')
CAPTURING = []          # the stand-in CUDA graph being captured, if any


def _is_cuda(dev):
    return dev is not None and str(dev).startswith('cuda')


# ---- optional arithmetic behind the forward-path entry points (see the module docstring) -----------------------------------
def _f32(ptr, count):
    import numpy as np
    return np.ctypeslib.as_array(C.cast(ptr, C.POINTER(C.c_float)), shape=(int(count),))


def _view(vp):
    """dh_view* -> writable float32 numpy view (n, h, w, c) with the view's leading dimension"""
    import numpy as np
    v = vp.contents
    n, h, w, c, ld = int(v.n), int(v.h), int(v.w), int(v.c), int(v.ld)
    flat = _f32(v.p, (n * h * w - 1) * ld + c)
    return np.lib.stride_tricks.as_strided(flat, shape=(n, h, w, c), strides=(h * w * ld * 4, w * ld * 4, ld * 4, 4))


def _struct_view(v):
    return _view(C.pointer(v))


def _dense(ptr, *shape):
    import numpy as np
    return _f32(ptr, int(np.prod(shape))).reshape(shape)


def _dense64(ptr, *shape):
    import numpy as np
    return np.ctypeslib.as_array(C.cast(ptr, C.POINTER(C.c_double)), shape=(int(np.prod(shape)),)).reshape(shape)


def _in(vp):
    """dh_view* -> its contents in float64 (None for a NULL pointer or a NULL-p view)"""
    return _view(vp).astype('float64') if vp and vp.contents.p else None


def _put(ptr, y):
    """y into the dense fp32 buffer at ptr"""
    _dense(ptr, *y.shape)[...] = y


def _conv(ctx, x, *rest):
    """dh_conv2d_f32 (one weight pointer: HWIO) and dh_sepconv2d_f32 (two: depthwise, pointwise)"""
    *wp, packed, d, out, stream = rest
    d = d.contents
    a, o = _in(x), _view(out)
    cin, cout, kh, kw = a.shape[-1], o.shape[-1], int(d.kh), int(d.kw)
    if len(wp) == 2:
        w = (_dense(wp[0], kh, kw, cin, 1).astype('float64'), _dense(wp[1], 1, 1, cin, cout).astype('float64'))
    else:
        w = _dense(wp[0], kh, kw, cin, cout).astype('float64')
    pre = (_f32(d.pre_scale, cin), _f32(d.pre_shift, cin)) if d.pre_scale else None
    post = (_f32(d.post_scale, cout), _f32(d.post_shift, cout)) if d.post_scale else None
    res = [_in(C.pointer(d.res[i])) for i in range(int(d.n_res))]
    ys = K.conv(a, w, (int(d.sh), int(d.sw)), 'same' if d.pad_same else 'valid', pre, d.pre_relu, post, d.post_relu,
                res, int(d.res_up2x), bool(d.pool_out.p))
    assert ys[0].shape == o.shape, (ys[0].shape, o.shape)
    o[...] = ys[0]
    if d.pool_out.p:
        _struct_view(d.pool_out)[...] = ys[1]


def _maxpool(ctx, x, kh, kw, sh, sw, pad_same, out, stream):
    _view(out)[...] = K.maxpool(_in(x), (kh, kw), (sh, sw), 'same' if pad_same else 'valid')


def _upsample_add(ctx, a, b, out, stream):
    _view(out)[...] = K.upsample2x_add(_in(b), _in(a))


def _add_n(ctx, ins, n_in, scale, shift, relu, out, stream):
    c = out.contents.c
    _view(out)[...] = K.add_n([_in(C.pointer(ins[i])) for i in range(n_in)], _f32(scale, c) if scale else None,
                              _f32(shift, c) if scale else None, relu)


def _head(outs, out_pose, out_vis, prob_out=None):
    """a soft-argmax head's pose and confidence into their dense buffers, its probabilities into prob_out if not NULL"""
    _put(out_pose, outs[0])
    _put(out_vis, outs[1])
    if prob_out and prob_out.contents.p:
        _view(prob_out)[...] = outs[2]


def _softargmax2d(ctx, h, d, alpha, conf_on_prob, out_pose, out_conf, prob_out, stream):
    _head(K.softargmax2d(_in(h), alpha, conf_on_prob, _in(d)), out_pose, out_conf, prob_out)


def _softargmax2d_ctx(ctx, h, nj, n_ctx, alpha_mix, out_pose, out_vis, stream):
    _head(K.softargmax2d_ctx(_in(h), nj, n_ctx, alpha_mix), out_pose, out_vis)


def _softargmax3d_ex(ctx, h, nj, depth, vis_scale, out_pose, out_vis, prob_out, stream):
    _head(K.softargmax3d(_in(h), nj, depth, vis_scale), out_pose, out_vis, prob_out)


def _softargmax3d(ctx, h, nj, depth, out_pose, out_vis, stream):
    _softargmax3d_ex(ctx, h, nj, depth, 1.0, out_pose, out_vis, None, stream)


def _kron(ctx, p, z, out, stream):
    _put(out, K.kron_pool(_in(p), _in(z)))


def _zeropad(ctx, x, top, left, out, stream):
    _view(out)[...] = K.zeropad(_in(x), top, left, (out.contents.h, out.contents.w))


def _maxmin_pool(ctx, x, out, stream):
    _view(out)[...] = K.maxmin_pool(_in(x))


def _global_maxmin_softmax(ctx, x, out, stream):
    _put(out, K.global_maxmin_softmax(_in(x)))


def _mask_mul(ctx, p, c, rows, dim, out, stream):
    _put(out, K.mask_mul(_dense(p, rows, dim).astype('float64'), _dense(c, rows, 1).astype('float64')))


def _pose_eval(ctx, pred, ldp, afmat, per_sample, inverse, y_true, head, refp, n, nj, out_pose, hits, valid, dsum, stream):
    """csrc/postprocess.cu: (inverse) affine of the poses, per-joint hit / valid counters and distance sums accumulated;
    float64 throughout, the threshold too"""
    import numpy as np
    P = _dense64(pred, n, nj, ldp)
    A = _dense64(afmat, n if per_sample else 1, 3, 3)
    M = A
    if inverse:                                     # a singular map gives NaN poses
        M = np.stack([np.linalg.inv(a) if np.linalg.matrix_rank(a) == 3 else np.full((3, 3), np.nan) for a in A])
    M = np.broadcast_to(M, (n, 3, 3))
    t = np.einsum('nij,nkj->nki', M[:, :2, :2], P[:, :, :2]) + M[:, None, :2, 2]
    _dense64(out_pose, n, nj, 2)[...] = t
    if y_true:
        g = _dense64(y_true, n, nj, 2)
        ok = (g[..., 0] > -1e6) & (g[..., 1] > -1e6)
        d = np.sqrt(((g - t) ** 2).sum(axis=-1))
        np.ctypeslib.as_array(C.cast(valid, C.POINTER(C.c_int32)), shape=(nj,))[...] += ok.sum(axis=0).astype(np.int32)
        np.ctypeslib.as_array(C.cast(dsum, C.POINTER(C.c_double)), shape=(nj,))[...] += np.where(ok, d, 0.0).sum(axis=0)
        if head:
            d = d / _dense64(head, n, 1)
        hit = ok & (d <= float(refp))
        np.ctypeslib.as_array(C.cast(hits, C.POINTER(C.c_int32)), shape=(nj,))[...] += hit.sum(axis=0).astype(np.int32)


def _crop_resize_norm(ctx, table, n, max_ch, bounds, coefs, rh, rw, power, tmp, tmp_stride, out, stream):
    """csrc/preprocess.cu: per frame crop window (outside the image = 0) -> Pillow's bilinear resize -> flip ->
    normalize_channels; the resampling tables the host sent are not read here: the oracle derives its own"""
    import numpy as np
    from deephar_b200._ffi import dh_frame_src
    from oracle import preprocess as OP
    frames = C.cast(table, C.POINTER(dh_frame_src))
    o = _dense(out, n, rh, rw, 3)
    pw = 1 if not power else tuple(float(v) for v in _f32(power, 3))
    for i in range(n):
        f = frames[i]
        img = np.ctypeslib.as_array(C.cast(f.data, C.POINTER(C.c_uint8)), shape=(int(f.h), int(f.stride)))[:, :int(f.w) * 3]
        img = img.reshape(int(f.h), int(f.w), 3)
        box = (int(f.x0), int(f.y0), int(f.x0) + int(f.cw), int(f.y0) + int(f.ch))
        o[i] = OP.eval_frame(img, box, (rw, rh), hflip=bool(f.hflip), channel_power=pw)


def _allgather(ctx, send, recv, count, stream):
    """csrc/comm.cu dh_allgather_f32 (ncclAllGather): recv[r * count ...] = rank r's send -- over gloo here"""
    import torch
    import torch.distributed as dist
    world = dist.get_world_size()
    src = torch.from_numpy(_f32(send, count).copy())
    dst = torch.empty(world * count, dtype=torch.float32)
    dist.all_gather_into_tensor(dst, src)
    _f32(recv, world * count)[...] = dst.numpy()


ARITHMETIC = {
    'dh_allgather_f32': _allgather, 'dh_pose_eval_f64': _pose_eval, 'dh_crop_resize_norm_u8': _crop_resize_norm,
    'dh_conv2d_f32': _conv, 'dh_sepconv2d_f32': _conv, 'dh_maxpool2d_f32': _maxpool,
    'dh_upsample2x_add_f32': _upsample_add, 'dh_add_n_f32': _add_n, 'dh_softargmax2d_f32': _softargmax2d,
    'dh_softargmax2d_ctx_f32': _softargmax2d_ctx, 'dh_softargmax3d_f32': _softargmax3d,
    'dh_softargmax3d_ex_f32': _softargmax3d_ex, 'dh_kron_pool_f32': _kron, 'dh_zeropad2d_f32': _zeropad,
    'dh_maxmin_pool2d_f32': _maxmin_pool, 'dh_global_maxmin_softmax_f32': _global_maxmin_softmax, 'dh_mask_mul_f32': _mask_mul,
}


def install(arithmetic=False):
    import torch
    import torch.distributed as dist

    from deephar_b200 import _ffi

    # ---- tensors: device memory is host memory -------------------------------------------------------------------------
    def strip_device(fn):
        def wrapper(*args, **kwargs):
            if _is_cuda(kwargs.get('device')):
                kwargs['device'] = 'cpu'
            return fn(*args, **kwargs)
        return wrapper
    for name in ('empty', 'zeros', 'ones', 'full', 'tensor', 'randn', 'rand', 'arange', 'as_tensor'):
        setattr(torch, name, strip_device(getattr(torch, name)))
    real_generator = torch.Generator
    torch.Generator = lambda device=None: real_generator()
    torch.Tensor.cuda = lambda self, *a, **k: self
    torch.Tensor.pin_memory = lambda self, *a, **k: self
    torch.Tensor.record_stream = lambda self, stream: None
    torch.Tensor.is_cuda = property(lambda self: True)
    real_to = torch.Tensor.to

    def to(self, *args, **kwargs):
        args = tuple('cpu' if _is_cuda(a) and not isinstance(a, torch.dtype) else a for a in args)
        if _is_cuda(kwargs.get('device')):
            kwargs['device'] = 'cpu'
        return real_to(self, *args, **kwargs)
    torch.Tensor.to = to

    # ---- torch.cuda: one inert device ----------------------------------------------------------------------------------
    class Event(object):
        def __init__(self, enable_timing=False, **kw):
            self.t = None

        def record(self, stream=None):
            self.t = time.perf_counter()

        def elapsed_time(self, other):
            return max(1e-3, (other.t - self.t) * 1000.0)

        def synchronize(self):
            pass

        def query(self):
            return True

    class Stream(object):
        cuda_stream = 0

        def __init__(self, *a, **k):
            pass

        def synchronize(self):
            pass

        def wait_event(self, event):
            pass

        def wait_stream(self, stream):
            pass

        def record_event(self, event=None):
            event = event or Event()
            event.record()
            return event

    class CUDAGraph(object):
        """records the library calls issued while it is being captured and issues them again on replay()"""

        def __init__(self):
            self.ops = []

        def replay(self):
            for fn, args in self.ops:
                fn(*args)

    @contextlib.contextmanager
    def capture(g, *a, **k):
        CAPTURING.append(g)
        try:
            yield
        finally:
            CAPTURING.pop()

    cuda = torch.cuda
    the_stream = Stream()
    cuda.is_available = lambda: True
    cuda.device_count = lambda: int(os.environ.get('FAKE_CUDA_DEVICES', '8'))
    cuda.current_device = lambda: 0
    cuda.set_device = lambda d: None
    cuda.synchronize = lambda *a, **k: None
    cuda.empty_cache = lambda: None
    cuda.current_stream = lambda *a, **k: the_stream
    cuda.Stream = Stream
    cuda.Event = Event
    cuda.CUDAGraph = CUDAGraph
    cuda.stream = lambda s: contextlib.nullcontext()
    cuda.graph = capture
    cuda.device = lambda d: contextlib.nullcontext()

    # ---- torch.distributed: NCCL -> gloo -------------------------------------------------------------------------------
    real_init = dist.init_process_group

    def init_process_group(backend=None, *args, **kwargs):
        kwargs.pop('device_id', None)
        return real_init('gloo', *args, **kwargs)
    dist.init_process_group = init_process_group
    dist.get_backend = lambda group=None: 'gloo'

    # ---- the C library: host entry points are real, device entry points are no-ops -----------------------------------
    real = _ffi.lib()

    class FakeLib(object):
        calls = {}

        def __getattr__(self, name):
            if name in HOST_ENTRY_POINTS:
                return getattr(real, name)
            if name not in _ffi.SIGNATURES:
                raise AttributeError(name)
            restype, argtypes = _ffi.SIGNATURES[name]
            proto = C.CFUNCTYPE(restype, *argtypes)             # converts / type-checks the arguments as the real call does

            def body(*args):
                FakeLib.calls[name] = FakeLib.calls.get(name, 0) + 1
                if CAPTURING:
                    CAPTURING[-1].ops.append((body, args))
                return 0
            if name == 'dh_ctx_create':
                def body(out, device):                          # noqa: F811
                    C.cast(out, C.POINTER(C.c_void_p))[0] = 0xB200
                    return 0
            if arithmetic and name in ARITHMETIC:
                op = ARITHMETIC[name]

                def body(*args, _op=op, _name=name):            # noqa: F811
                    FakeLib.calls[_name] = FakeLib.calls.get(_name, 0) + 1
                    if CAPTURING:
                        CAPTURING[-1].ops.append((body, args))
                    _op(*args)
                    return 0
            fn = proto(body)
            setattr(self, name, fn)
            return fn
    fake = FakeLib()
    _ffi._lib = fake
    _ffi.lib = lambda: fake
    return fake


def main():
    """python tests/fake_cuda.py [--arithmetic] <script.py | -m module> [args ...]"""
    argv = sys.argv[1:]
    arithmetic = bool(argv) and argv[0] == '--arithmetic'
    if arithmetic:
        argv = argv[1:]
    install(arithmetic=arithmetic)
    if argv[0] == '-m':
        sys.argv = argv[1:]
        runpy.run_module(argv[1], run_name='__main__', alter_sys=True)
    else:
        sys.argv = argv
        runpy.run_path(argv[0], run_name='__main__')


if __name__ == '__main__':
    main()
