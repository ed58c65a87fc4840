"""wgmma path parity (conv_tc.cu, conv_sep.cu, conv_patch.cu): the tensor-core kernels vs the fp64 oracle, at the layer
shapes of the models and at ragged / tail shapes.  Each test asserts through
dh_last_conv_path() that the tensor-core kernel really served the call."""
import ctypes as C
import zlib

import numpy as np
import pytest

from deephar_b200 import _ffi, tc
from oracle import ops_np

from gpu_util import Dev, conv_desc

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def dev(cuda):
    return Dev(cuda)


def _packed(dev, w_k_by_cout):
    hi, lo, cp, kp = tc.pack_matrix(np.asarray(w_k_by_cout, np.float32))
    th = dev.torch.from_numpy(hi.view(np.int16).copy()).cuda()
    tl = dev.torch.from_numpy(lo.view(np.int16).copy()).cuda()
    dev.keep += [th, tl]
    return _ffi.dh_packed_w(th.data_ptr(), tl.data_ptr(), cp, kp)


def _err(got, ref):
    return float(np.abs(got.astype(np.float64) - ref).max()) / max(1.0, float(np.abs(ref).max()))


TOL3 = 3e-5      # bf16x3 split: operand error ~2^-16, fp32 accumulate
TOL1 = 3e-2      # plain bf16 (precision = 1)

CONV_CASES = [
    # N, H, W, Cin, Cout, size, strides, fused(pre_relu+post_bn+res)
    (2, 12, 12, 32, 64, (1, 1), (1, 1), False),
    (1, 13, 11, 8, 20, (3, 3), (1, 1), True),
    (1, 9, 9, 16, 24, (5, 1), (1, 1), False),
    (1, 9, 9, 16, 24, (1, 5), (1, 1), True),
    (2, 32, 32, 576, 48, (1, 1), (1, 1), True),      # RegMap
    (2, 32, 32, 48, 576, (1, 1), (1, 1), True),      # fReMap (+2 residuals)
    (3, 16, 16, 576, 288, (1, 1), (1, 1), True),     # rBlock reduce (three N CTAs)
    (2, 32, 32, 384, 576, (1, 1), (1, 1), True),     # stem shortcut (six N CTAs)
    (1, 64, 64, 192, 192, (3, 3), (2, 2), True),     # stem 3x3 stride 2
    (1, 32, 32, 32, 64, (3, 3), (1, 1), False),      # K-block straddles taps (Cin = 32)
    (1, 7, 5, 12, 272, (1, 1), (1, 1), False),       # M tail, ragged Cout (3-D RegMap width)
    (1, 16, 16, 64, 17, (1, 1), (1, 1), False),      # Cout = 17 (SPNet heat-maps): scalar epilogue
    # --- shapes of the TMA-staged patch kernel (conv_patch.cu) ---
    (2, 128, 128, 32, 64, (3, 3), (1, 1), False),    # stem conv3: one image row per tile, 130-pixel patch rows
    (1, 128, 128, 32, 32, (3, 3), (1, 1), False),    # stem conv2
    (1, 64, 64, 64, 96, (3, 3), (1, 1), False),      # stem 3x3 at 64x64: two channel blocks x 9 taps
    (1, 64, 64, 64, 64, (5, 1), (1, 1), False),      # stem 5x1
    (1, 64, 64, 64, 64, (1, 5), (1, 1), False),      # stem 1x5
    (1, 64, 64, 160, 64, (1, 1), (1, 1), False),     # stem 1x1 on the concat (Cin = 5 blocks)
    (3, 16, 16, 288, 576, (1, 1), (1, 1), True),     # rBlock expand (six N CTAs)
    (2, 32, 32, 144, 288, (3, 3), (1, 1), True),     # SPNet residual unit 3x3 with BN prologue (masked halo)
    (2, 128, 128, 48, 96, (3, 3), (1, 1), True),     # SPNet entry 3x3, Cin = 48 (half-empty channel block)
    (5, 8, 8, 480, 16, (1, 1), (1, 1), True),        # SPNet heat-map conv at 8x8: odd frame count, 64-pixel virtual rows
    (3, 8, 8, 64, 64, (3, 3), (1, 1), True),         # two frames per tile, tail tile, BN prologue mask
    (7, 4, 4, 96, 32, (3, 3), (1, 1), True),         # 4x4 maps are not taken by the patch kernel (falls to conv_tc)
    # --- ragged channel counts: conv_tc.cu's scalar-gather producer (no CUDA-core fallback) ---
    (1, 64, 64, 3, 64, (7, 7), (2, 2), False),       # SPNet first conv: 7x7 stride 2 on RGB
    (2, 32, 32, 17, 288, (1, 1), (1, 1), True),      # heat-map re-injection, 17 joints
    (1, 16, 16, 34, 384, (1, 1), (1, 1), True),      # heat-maps + depth maps
    (2, 8, 10, 15, 160, (3, 3), (1, 1), True),       # action head on (frames, joints) maps
    (1, 5, 7, 2, 8, (3, 1), (1, 1), False),          # PoseAR first conv: 2 input channels
]


def _patch_eligible(case):
    n, h, w, cin, cout, size, strides, fused = case
    if strides != (1, 1) or cin % 8:
        return False
    if size == (1, 1):
        vw = 128
        while vw > 1 and (h * w) % vw:
            vw //= 2
        if vw < 8:
            return False
        pc, pr, fn = vw, 128 // vw, 1
    else:
        if w not in (128, 64, 32, 16, 8):
            return False
        tr = 128 // w
        if (h % tr if tr <= h else tr % h) != 0:
            return False
        pc, pr, fn = w + size[1] - 1, min(tr, h) + size[0] - 1, max(1, tr // h)
    cp = (cout + 15) // 16 * 16
    gy = (cp + 95) // 96
    bn = ((cp + gy - 1) // gy + 15) // 16 * 16
    stride = (128 * pc * pr * fn + 1023) // 1024 * 1024
    fixed = 3 * 2 * 8192 + 4 * bn * 64 + 512
    return fixed + 2 * stride <= 227 * 1024


@pytest.mark.parametrize('case', CONV_CASES)
@pytest.mark.parametrize('precision', [3, 1])
@pytest.mark.parametrize('kernel', ['patch', 'reg'])
def test_conv_tc(dev, case, precision, kernel):
    """kernel = 'patch': conv_patch.cu (TMA-staged input patch, path 4) where it applies; 'reg': conv_tc.cu's
    register im2col producer (path 1)."""
    n, h, w, cin, cout, size, strides, fused = case
    if kernel == 'reg' and n * h * w * cin > (1 << 21) and precision == 1:
        pytest.skip('large case: the register-producer kernel is covered at precision 3')
    expect = 4 if (kernel == 'patch' and _patch_eligible(case)) else 1
    rng = np.random.default_rng(zlib.crc32(repr(case).encode()))
    x = rng.standard_normal((n, h, w, cin))
    wt = rng.standard_normal(size + (cin, cout)) / np.sqrt(size[0] * size[1] * cin)
    pre = post = None
    res = []
    xin = x
    if fused:
        pre = (rng.uniform(0.5, 1.5, cin), rng.standard_normal(cin) * 0.3)
        post = (rng.uniform(0.5, 1.5, cout), rng.standard_normal(cout) * 0.3)
        xin = np.maximum(x * pre[0] + pre[1], 0)
    ref = ops_np.conv2d(xin, wt, strides, 'same')
    if fused:
        ref = ref * post[0] + post[1]
        r0, r1 = rng.standard_normal(ref.shape), rng.standard_normal(ref.shape)
        ref = ref + r0 + r1
        res = [dev.view(dev.put(r0)), dev.view(dev.put(r1))]
    out = dev.empty(*ref.shape)
    d = conv_desc(dev, size, strides, 'same', pre_relu=fused, pre=pre, post=post, res=res, precision=precision)
    pk = _packed(dev, wt.reshape(-1, cout))
    xv, ov = dev.view(dev.put(x)), dev.view(out)
    # the wide / small-Cin 1x1 shapes would be served by the CUDA-core pointwise kernel (test_gpu_ops.py):
    # switch it off so that this test keeps exercising the tensor-core kernel on them
    _ffi.check(dev.lib.dh_set_option(dev.ctx.handle, b'pw_smallk', 0))
    _ffi.check(dev.lib.dh_set_option(dev.ctx.handle, b'dense_patch', 1 if kernel == 'patch' else 0))
    try:
        dev.call('dh_conv2d_f32', C.byref(xv), dev.put(wt).data_ptr(), C.byref(pk), C.byref(d), C.byref(ov))
    finally:
        _ffi.check(dev.lib.dh_set_option(dev.ctx.handle, b'pw_smallk', 1))
        _ffi.check(dev.lib.dh_set_option(dev.ctx.handle, b'dense_patch', 1))
    assert dev.lib.dh_last_conv_path(dev.ctx.handle) == expect, 'unexpected kernel path'
    e = _err(out.cpu().numpy(), ref)
    assert e <= (TOL3 if precision == 3 else TOL1), e


SEP_CASES = [
    # N, H, W, Cin, Cout, k, mode
    (2, 16, 16, 32, 48, 5, 'act_bn_res'),
    (1, 8, 8, 24, 24, 3, 'plain'),                  # half-empty tile (M = 64)
    (3, 4, 4, 64, 64, 5, 'bn_act'),                 # 4x4 maps: 8 frames per tile, tail tile
    (2, 32, 32, 576, 576, 5, 'act_bn_res'),         # the hot layer (reception l1 / SepConv)
    (2, 16, 16, 288, 288, 5, 'act_bn_res'),
    (3, 8, 8, 288, 288, 5, 'act_bn_res'),
    (2, 16, 16, 288, 576, 5, 'act_bn_res'),
    (1, 32, 32, 384, 576, 3, 'act_bn_res'),         # stem sepconv1
    (2, 32, 32, 288, 288, 5, 'bn_act'),             # SPNet level 0
    (2, 16, 16, 384, 384, 5, 'bn_act'),
    (2, 8, 8, 480, 480, 5, 'bn_act'),
    (8, 4, 4, 576, 576, 5, 'bn_act'),
    (2, 16, 16, 64, 96, 3, 'plain'),                # TMA-staged kernel without ReLU prologue
    (5, 8, 8, 96, 80, 5, 'act_bn_res'),             # 8x8 maps: two frames per tile, odd frame count
]


def _tma_eligible(case):
    n, h, w, cin, cout, k, mode = case
    return w in (32, 16, 8) and cin % 32 == 0          # (BN-prologue layers included: the halo is masked after the affine)


@pytest.mark.parametrize('case', SEP_CASES)
@pytest.mark.parametrize('precision', [3, 1])
@pytest.mark.parametrize('kernel', ['tma', 'reg'])
def test_sepconv_tc(dev, case, precision, kernel):
    """kernel = 'tma': conv_sep.cu (TMA-staged patch, path 2) where it applies; 'reg': conv_tc.cu's
    register-sliding producer (path 1)."""
    _ffi.check(dev.lib.dh_set_option(dev.ctx.handle, b'sep_tma', 1 if kernel == 'tma' else 0))
    try:
        _run_sepconv(dev, case, precision, 2 if (kernel == 'tma' and _tma_eligible(case)) else 1)
    finally:
        _ffi.check(dev.lib.dh_set_option(dev.ctx.handle, b'sep_tma', 1))


def _run_sepconv(dev, case, precision, expect_path):
    n, h, w, cin, cout, k, mode = case
    rng = np.random.default_rng(zlib.crc32(repr(case).encode()))
    x = rng.standard_normal((n, h, w, cin))
    dw = rng.standard_normal((k, k, cin, 1)) / k
    pw = rng.standard_normal((1, 1, cin, cout)) / np.sqrt(cin)
    pre = post = None
    res = []
    xin = x
    if mode == 'act_bn_res':
        xin = np.maximum(x, 0)
        post = (rng.uniform(0.5, 1.5, cout), rng.standard_normal(cout) * 0.3)
    elif mode == 'bn_act':
        pre = (rng.uniform(0.5, 1.5, cin), rng.standard_normal(cin) * 0.3)
        xin = np.maximum(x * pre[0] + pre[1], 0)
    ref = ops_np.separable_conv2d(xin, dw, pw, (1, 1), 'same')
    if mode == 'act_bn_res':
        ref = ref * post[0] + post[1]
        r0 = rng.standard_normal(ref.shape)
        ref = ref + r0
        res = [dev.view(dev.put(r0))]
    out = dev.empty(*ref.shape)
    d = conv_desc(dev, (k, k), (1, 1), 'same', pre_relu=(mode != 'plain'), pre=pre, post=post, res=res,
                  precision=precision)
    pk = _packed(dev, pw.reshape(cin, cout))
    xv, ov = dev.view(dev.put(x)), dev.view(out)
    dev.call('dh_sepconv2d_f32', C.byref(xv), dev.put(dw).data_ptr(), dev.put(pw).data_ptr(), C.byref(pk),
             C.byref(d), C.byref(ov))
    assert dev.lib.dh_last_conv_path(dev.ctx.handle) == expect_path, 'unexpected kernel path'
    e = _err(out.cpu().numpy(), ref)
    assert e <= (TOL3 if precision == 3 else TOL1), e


def test_tc_channel_views(dev):
    """concat / slice views through the tensor-core kernel (ld != c, channel offsets)."""
    rng = np.random.default_rng(3)
    big = rng.standard_normal((2, 16, 16, 96))
    wt = rng.standard_normal((1, 1, 64, 32)) / 8.0
    ref = ops_np.conv2d(big[..., 16:80], wt)
    cat = dev.empty(2, 16, 16, 40)
    cat.fill_(7.0)
    d = conv_desc(dev, (1, 1))
    pk = _packed(dev, wt.reshape(64, 32))
    xv, ov = dev.view(dev.put(big), 16, 80), dev.view(cat, 4, 36)
    dev.call('dh_conv2d_f32', C.byref(xv), dev.put(wt).data_ptr(), C.byref(pk), C.byref(d), C.byref(ov))
    assert dev.lib.dh_last_conv_path(dev.ctx.handle) == 4          # the patch kernel takes channel-sliced views
    got = cat.cpu().numpy()
    assert _err(got[..., 4:36], ref) <= TOL3
    assert np.all(got[..., :4] == 7.0) and np.all(got[..., 36:] == 7.0)
    # a slice at a channel offset that is not 16-byte aligned (17-joint heat-maps inside a concat): the
    # tensor-core kernel's scalar gather takes it, still no CUDA-core fallback
    big = rng.standard_normal((2, 16, 16, 51))
    wt = rng.standard_normal((1, 1, 34, 48)) / 6.0
    ref = ops_np.conv2d(big[..., 17:51], wt)
    out = dev.empty(2, 16, 16, 48)
    pk = _packed(dev, wt.reshape(34, 48))
    xv, ov = dev.view(dev.put(big), 17, 51), dev.view(out)
    dev.lib.dh_fallback_count(dev.ctx.handle, 1)
    dev.call('dh_conv2d_f32', C.byref(xv), dev.put(wt).data_ptr(), C.byref(pk), C.byref(d), C.byref(ov))
    assert dev.lib.dh_last_conv_path(dev.ctx.handle) == 1 and dev.lib.dh_fallback_count(dev.ctx.handle, 0) == 0
    assert _err(out.cpu().numpy(), ref) <= TOL3


@pytest.mark.parametrize('share', [1, 0])
def test_sepconv_cluster_share_matches(dev, share):
    """Layers split over an even number of N parts run as 2-CTA clusters sharing the depthwise A tile over DSMEM (share_a = 1);
    the result must match the oracle exactly like the independent-CTA path (share_a = 0)."""
    _ffi.check(dev.lib.dh_set_option(dev.ctx.handle, b'share_a', share))
    try:
        for case in [(3, 32, 32, 576, 576, 5, 'act_bn_res'), (2, 16, 16, 288, 576, 5, 'act_bn_res'),
                     (1, 32, 32, 384, 576, 3, 'act_bn_res'), (5, 8, 8, 128, 576, 5, 'bn_act')]:
            _ffi.check(dev.lib.dh_set_option(dev.ctx.handle, b'sep_tma', 0))      # exercise conv_tc.cu's SHARE path
            _run_sepconv(dev, case, 3, 1)
    finally:
        _ffi.check(dev.lib.dh_set_option(dev.ctx.handle, b'share_a', 1))
        _ffi.check(dev.lib.dh_set_option(dev.ctx.handle, b'sep_tma', 1))


@pytest.mark.parametrize('case', [(2, 32, 32, 576, 576, 5, 2), (3, 32, 32, 64, 96, 3, 1), (1, 64, 32, 32, 32, 3, 2),
                                  (5, 16, 16, 288, 288, 5, 2), (3, 16, 16, 64, 96, 3, 1), (1, 12, 16, 32, 64, 5, 2)])
def test_sepconv_upsampled_residual(dev, case):
    """keras `add([a, UpSampling2D(b)])` (reception.py:122-127) folded into the epilogue of the conv that produces a:
    the LAST residual is a half-resolution tensor (dh_conv_desc.res_up2x); n_res = 2: identity shortcut + upsampled."""
    n, h, w, cin, cout, k, n_res = case
    rng = np.random.default_rng(zlib.crc32(repr(case).encode()))
    x = rng.standard_normal((n, h, w, cin))
    dw = rng.standard_normal((k, k, cin, 1)) / k
    pw = rng.standard_normal((1, 1, cin, cout)) / np.sqrt(cin)
    post = (rng.uniform(0.5, 1.5, cout), rng.standard_normal(cout) * 0.3)
    r_full = rng.standard_normal((n, h, w, cout))
    r_half = rng.standard_normal((n, h // 2, w // 2, cout))
    ref = ops_np.separable_conv2d(np.maximum(x, 0), dw, pw, (1, 1), 'same') * post[0] + post[1]
    ref = ref + np.repeat(np.repeat(r_half, 2, axis=1), 2, axis=2)
    res = [dev.view(dev.put(r_half))]
    if n_res == 2:
        ref = ref + r_full
        res = [dev.view(dev.put(r_full))] + res
    out = dev.empty(*ref.shape)
    d = conv_desc(dev, (k, k), (1, 1), 'same', pre_relu=True, post=post, res=res, precision=3)
    d.res_up2x = 1 << (n_res - 1)
    pk = _packed(dev, pw.reshape(cin, cout))
    xv, ov = dev.view(dev.put(x)), dev.view(out)
    dev.call('dh_sepconv2d_f32', C.byref(xv), dev.put(dw).data_ptr(), dev.put(pw).data_ptr(), C.byref(pk),
             C.byref(d), C.byref(ov))
    # 2 = conv_sep.cu; 1 = conv_tc.cu's separable path (heights conv_sep does not tile) -- same epilogue
    assert dev.lib.dh_last_conv_path(dev.ctx.handle) == (2 if h % 8 == 0 else 1)
    assert _err(out.cpu().numpy(), ref) <= TOL3
    # a residual flagged as upsampled must have half the output's size
    d.res[n_res - 1] = dev.view(dev.put(r_full))
    rc = dev.lib.dh_sepconv2d_f32(dev.ctx.handle, C.byref(xv), dev.put(dw).data_ptr(), dev.put(pw).data_ptr(), C.byref(pk),
                                  C.byref(d), C.byref(ov), dev.stream())
    assert rc < 0 and b'shape mismatch' in dev.lib.dh_last_error()
