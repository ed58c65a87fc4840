"""Helpers for the -m gpu parity tests: call the C ABI on torch device buffers."""
import ctypes as C

import numpy as np

from deephar_b200 import _ffi


class Dev(object):
    def __init__(self, torch):
        self.torch = torch
        self.ctx = _ffi.Context(torch.cuda.current_device())
        self.lib = _ffi.lib()
        self.keep = []
        self.ws = torch.empty(64 << 20, dtype=torch.float32, device='cuda')
        self.ctx.set_workspace(self.ws.data_ptr(), self.ws.numel() * 4)

    def put(self, a):
        t = self.torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).cuda()
        self.keep.append(t)
        return t

    def empty(self, *shape):
        t = self.torch.full(shape, float('nan'), dtype=self.torch.float32, device='cuda')
        self.keep.append(t)
        return t

    def view(self, t, c0=None, c1=None):
        """dh_view of an NHWC tensor, optionally a channel slice [c0:c1)."""
        n, h, w, c = t.shape
        if c0 is None:
            return _ffi.dh_view(t.data_ptr(), n, h, w, c, c)
        return _ffi.dh_view(t.data_ptr() + 4 * c0, n, h, w, c1 - c0, c)

    def stream(self):
        return self.torch.cuda.current_stream().cuda_stream

    def call(self, name, *args):
        rc = getattr(self.lib, name)(self.ctx.handle, *args, self.stream())
        _ffi.check(rc, name)
        self.torch.cuda.synchronize()


def packed_weights(dev, w_k_by_cout):
    """(K, Cout) weights as the bf16 hi / lo K-major operand of the tensor-core kernels (tc.pack_matrix), on the device."""
    from deephar_b200 import tc
    hi, lo, cp, kp = tc.pack_matrix(np.asarray(w_k_by_cout, np.float32))
    th = dev.torch.from_numpy(hi.view(np.int16).copy()).cuda()
    tl = dev.torch.from_numpy(lo.view(np.int16).copy()).cuda()
    dev.keep += [th, tl]
    return _ffi.dh_packed_w(th.data_ptr(), tl.data_ptr(), cp, kp)


def conv_desc(dev, size, strides=(1, 1), padding='same', pre_relu=False, post_relu=False,
              pre=None, post=None, res=(), precision=3):
    d = _ffi.dh_conv_desc()
    d.kh, d.kw = size
    d.sh, d.sw = strides
    d.pad_same = 1 if padding == 'same' else 0
    d.pre_relu = int(pre_relu)
    d.post_relu = int(post_relu)
    if pre is not None:
        d.pre_scale, d.pre_shift = dev.put(pre[0]).data_ptr(), dev.put(pre[1]).data_ptr()
    if post is not None:
        d.post_scale, d.post_shift = dev.put(post[0]).data_ptr(), dev.put(post[1]).data_ptr()
    d.n_res = len(res)
    for i, r in enumerate(res):
        d.res[i] = r
    d.precision = precision
    return d


def close(got, ref, tol=2e-5):
    """max |got - ref| within tol relative to the output scale (2e-5: fp32 CUDA-core path vs the fp64 oracle)"""
    scale = max(1.0, float(np.abs(ref).max()))
    err = float(np.abs(got.astype(np.float64) - ref).max())
    assert err <= tol * scale, 'max err %g (scale %g)' % (err, scale)


def num_sms(dev):
    return dev.torch.cuda.get_device_properties(dev.torch.cuda.current_device()).multi_processor_count


def loop_batch(dev, items_per_frame):
    """A batch size at which the grid-stride kernels of elementwise.cu (grid capped at num_sms * 16 CTAs of 256
    threads) give every thread at least two iterations over items_per_frame work items per frame."""
    return 2 * num_sms(dev) * 16 * 256 // items_per_frame + 1


SENT = 7.25     # fills the channels of a wider buffer outside a view


def sliced(dev, x, c0, ld):
    """x on the device as the channel slice [c0, c0 + C) of a buffer of ld channels whose other channels hold SENT"""
    big = np.full(x.shape[:3] + (ld,), SENT)
    big[..., c0:c0 + x.shape[3]] = x
    return dev.view(dev.put(big), c0, c0 + x.shape[3])


class Out(object):
    """An output view: a dense NaN-filled buffer, or the channel slice [c0, c0 + C) of a buffer of ld channels filled
    with SENT.  get() checks that nothing outside the slice was written and returns the view's contents."""
    def __init__(self, dev, shape, c0=None, ld=None):
        self.c0, self.c = c0, shape[3]
        if c0 is None:
            self.t = dev.empty(*shape)
            self.view = dev.view(self.t)
        else:
            self.t = dev.empty(*shape[:3], ld)
            self.t.fill_(SENT)
            self.view = dev.view(self.t, c0, c0 + self.c)

    def get(self):
        a = self.t.cpu().numpy()
        if self.c0 is None:
            return a
        assert np.all(a[..., :self.c0] == SENT) and np.all(a[..., self.c0 + self.c:] == SENT), 'wrote outside the view'
        return a[..., self.c0:self.c0 + self.c]


def layout_io(dev, x, out_shape, layout):
    """(input view, Out) of a memory-bound kernel: 'slice' puts the input at channels [4, 4 + C) of a buffer and the
    output at [8, 8 + C), both 16-byte aligned for a C that is a multiple of 4; any other layout is dense"""
    if layout == 'slice':
        return sliced(dev, x, 4, x.shape[3] + 8), Out(dev, out_shape, 8, out_shape[3] + 12)
    return dev.view(dev.put(x)), Out(dev, out_shape)


NULLV = C.cast(None, C.POINTER(_ffi.dh_view))
NULLP = C.cast(None, C.POINTER(_ffi.dh_packed_w))


# ---- per-element error bounds of the convolutions against the fp64 oracle ------------------------------------------------
# |got - ref| <= bound, with
#   S = sum_k |a_k w_k|, Q = sqrt(sum_k (a_k w_k)^2)      (a: the MMA's A operand -- prologue(x), or the depthwise
#                                                           output of a separable layer; times |BN scale|)
# precision 3 (bf16x3, paths 1, 2, 4):  a = hi + lo + r with |r| <= 2^-17 |a| (hi, lo round to nearest even:
#   |a - hi| <= 2^-8 |a|, and the rounding of a - hi to lo leaves at most 2^-9 of its own 2^-8), the same for w, and the
#   dropped lo * lo is <= 2^-16 |a w|: each product is off by at most 2^-15 |a_k w_k|.  Those are independent
#   round-to-nearest errors of either sign, so their sum has a standard deviation of at most 2^-15 Q / sqrt(3) (uniform
#   within the bound), and Z standard deviations bound it: Z3 = Z / sqrt(3).
#   fp32 accumulation: one rounding of at most 2^-23 of the running sum (<= S) per accumulating wgmma k-step, 3 K / 16
#   of them (K / 16 at precision 1), independent as above: NU = Z3 * 2^-23 * sqrt(k-steps).
# fp32 FFMA (the CUDA-core paths 0 and 3): exact products, one rounding of at most 2^-24 of the running sum per term:
#   Z3 * 2^-24 * sqrt(K) * S.  One dropped term |a_k w_k| ~ S / K is far above that for every K the networks use.
# The separable depthwise is KS^2 fp32 FMAs per value, a worst case of KS^2 * 2^-24 relative to |dw| * |x|, which S
#   carries through |pw| (plus one rounding of the BN-prologue FMA); a dense layer's prologue FMA is 2^-23 S.
# epilogue: BN FMA, +res0, +res1, each rounded once in fp32: EPS = 4 * 2^-24, of |ref| + |res0| + |res1|.
Z = 6.0
Z3 = Z / np.sqrt(3.0)
EPS = 4 * 2.0 ** -24


def bf16(a):
    """fp64 -> fp32 -> bf16 (round to nearest even), as fp64."""
    u = np.ascontiguousarray(a, np.float32).view(np.uint32).astype(np.uint64)
    r = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16) << 16
    return r.astype(np.uint32).view(np.float32).astype(np.float64)


def near_tie(a, delta):
    """operands whose bf16 rounding can flip within +-delta (the fp32 error of the value computed on the GPU)"""
    return bf16(a - delta) != bf16(a + delta)


def f32(a):
    return np.asarray(a, np.float32).astype(np.float64)


def tc_dense_bound(q, s, k):
    """Conv2D at precision 3 on the wgmma paths, K = kh * kw * Cin, before the epilogue"""
    return Z3 * 2.0 ** -15 * q + (Z3 * 2.0 ** -23 * np.sqrt(3 * k / 16) + 2.0 ** -23) * s


def tc_sep_bound(q, s, cin, ks):
    """SeparableConv2D at precision 3 on the wgmma paths (Q, S over the depthwise output), before the epilogue"""
    return Z3 * 2.0 ** -15 * q + (Z3 * 2.0 ** -23 * np.sqrt(3 * cin / 16) + (ks * ks + 1) * 2.0 ** -24) * s


def ffma_dense_bound(s, k):
    """Conv2D on the fp32 CUDA-core paths, before the epilogue"""
    return (Z3 * 2.0 ** -24 * np.sqrt(k) + 2.0 ** -23) * s


def ffma_sep_bound(s, cin, ks):
    """SeparableConv2D on the fp32 CUDA-core path (depthwise, then the pointwise over Cin), before the epilogue"""
    return (Z3 * 2.0 ** -24 * np.sqrt(cin) + (ks * ks + 1) * 2.0 ** -24) * s


def epilogue_bound(bound, post_scale, ref, res):
    """the bound of a conv's MMA result carried through the BN epilogue (post_scale or None) and the residual adds"""
    if post_scale is not None:
        bound = bound * np.abs(post_scale)
    return bound + EPS * (np.abs(ref) + sum(np.abs(r) for r in res))
