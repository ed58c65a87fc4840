"""wgmma path parity (conv_tc.cu, conv_sep.cu, conv_patch.cu): the tensor-core kernels vs the fp64 oracle, at the layer
shapes of the models and at ragged / tail shapes.  Each test asserts through
dh_last_conv_path() that the tensor-core kernel really served the call."""
import ctypes as C
import zlib

import numpy as np
import pytest

from deephar_b200 import _ffi
from oracle import ops_np

from gpu_util import NULLP, Dev, conv_desc, packed_weights

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def dev(cuda):
    return Dev(cuda)


def _err(got, ref):
    return float(np.abs(got.astype(np.float64) - ref).max()) / max(1.0, float(np.abs(ref).max()))


TOL3 = 3e-5      # bf16x3 split: operand error ~2^-16, fp32 accumulate
TOL1 = 3e-2      # plain bf16 (precision = 1)

CONV_CASES = [
    # N, H, W, Cin, Cout, size, strides, fused(pre_relu+post_bn+res),
    # path with dense_patch on (4 conv_patch.cu, 1 conv_tc.cu)
    (2, 12, 12, 32, 64, (1, 1), (1, 1), False, 4),
    (1, 13, 11, 8, 20, (3, 3), (1, 1), True, 1),
    (1, 9, 9, 16, 24, (5, 1), (1, 1), False, 1),
    (1, 9, 9, 16, 24, (1, 5), (1, 1), True, 1),
    (2, 32, 32, 576, 48, (1, 1), (1, 1), True, 4),      # RegMap
    (2, 32, 32, 48, 576, (1, 1), (1, 1), True, 4),      # fReMap (+2 residuals)
    (3, 16, 16, 576, 288, (1, 1), (1, 1), True, 4),     # rBlock reduce (three N CTAs)
    (2, 32, 32, 384, 576, (1, 1), (1, 1), True, 4),     # stem shortcut (six N CTAs)
    (1, 64, 64, 192, 192, (3, 3), (2, 2), True, 1),     # stem 3x3 stride 2
    (1, 32, 32, 32, 64, (3, 3), (1, 1), False, 4),      # K-block straddles taps (Cin = 32)
    (1, 7, 5, 12, 272, (1, 1), (1, 1), False, 1),       # M tail, ragged Cout (3-D RegMap width)
    (1, 16, 16, 64, 17, (1, 1), (1, 1), False, 4),      # Cout = 17 (SPNet heat-maps): scalar epilogue
    # --- shapes of the TMA-staged patch kernel (conv_patch.cu) ---
    (2, 128, 128, 32, 64, (3, 3), (1, 1), False, 4),    # stem conv3: one image row per tile, 130-pixel patch rows
    (1, 128, 128, 32, 32, (3, 3), (1, 1), False, 4),    # stem conv2
    (1, 64, 64, 64, 96, (3, 3), (1, 1), False, 4),      # stem 3x3 at 64x64: two channel blocks x 9 taps
    (1, 64, 64, 64, 64, (5, 1), (1, 1), False, 4),      # stem 5x1
    (1, 64, 64, 64, 64, (1, 5), (1, 1), False, 4),      # stem 1x5
    (1, 64, 64, 160, 64, (1, 1), (1, 1), False, 4),     # stem 1x1 on the concat (Cin = 5 blocks)
    (3, 16, 16, 288, 576, (1, 1), (1, 1), True, 4),     # rBlock expand (six N CTAs)
    (2, 32, 32, 144, 288, (3, 3), (1, 1), True, 4),     # SPNet residual unit 3x3 with BN prologue (masked halo)
    (2, 128, 128, 48, 96, (3, 3), (1, 1), True, 4),     # SPNet entry 3x3, Cin = 48 (half-empty channel block)
    (5, 8, 8, 480, 16, (1, 1), (1, 1), True, 4),        # SPNet heat-map conv at 8x8: odd frame count, 64-pixel virtual rows
    (3, 8, 8, 64, 64, (3, 3), (1, 1), True, 4),         # two frames per tile, tail tile, BN prologue mask
    (7, 4, 4, 96, 32, (3, 3), (1, 1), True, 1),         # 4x4 maps are not taken by the patch kernel (falls to conv_tc)
    # --- ragged channel counts: conv_tc.cu's scalar-gather producer (no CUDA-core fallback) ---
    (1, 64, 64, 3, 64, (7, 7), (2, 2), False, 1),       # SPNet first conv: 7x7 stride 2 on RGB
    (2, 32, 32, 17, 288, (1, 1), (1, 1), True, 1),      # heat-map re-injection, 17 joints
    (1, 16, 16, 34, 384, (1, 1), (1, 1), True, 1),      # heat-maps + depth maps
    (2, 8, 10, 15, 160, (3, 3), (1, 1), True, 1),       # action head on (frames, joints) maps
    (1, 5, 7, 2, 8, (3, 1), (1, 1), False, 1),          # PoseAR first conv: 2 input channels
]


@pytest.mark.parametrize('case', CONV_CASES)
@pytest.mark.parametrize('precision', [3, 1])
@pytest.mark.parametrize('kernel', ['patch', 'reg'])
def test_conv_tc(dev, case, precision, kernel):
    """kernel = 'patch': conv_patch.cu (TMA-staged input patch, path 4) where it applies; 'reg': conv_tc.cu's
    register im2col producer (path 1)."""
    case, patch_path = case[:-1], case[-1]
    n, h, w, cin, cout, size, strides, fused = case
    if kernel == 'reg' and n * h * w * cin > (1 << 21) and precision == 1:
        pytest.skip('large case: the register-producer kernel is covered at precision 3')
    expect = patch_path if kernel == 'patch' else 1
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
    pk = packed_weights(dev, wt.reshape(-1, cout))
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
    # N, H, W, Cin, Cout, k, mode, path with sep_tma on (2 conv_sep.cu, 1 conv_tc.cu)
    (2, 16, 16, 32, 48, 5, 'act_bn_res', 2),
    (1, 8, 8, 24, 24, 3, 'plain', 1),                  # half-empty tile (M = 64)
    (3, 4, 4, 64, 64, 5, 'bn_act', 1),                 # 4x4 maps: 8 frames per tile, tail tile
    (2, 32, 32, 576, 576, 5, 'act_bn_res', 2),         # the hot layer (reception l1 / SepConv)
    (2, 16, 16, 288, 288, 5, 'act_bn_res', 2),
    (3, 8, 8, 288, 288, 5, 'act_bn_res', 2),
    (2, 16, 16, 288, 576, 5, 'act_bn_res', 2),
    (1, 32, 32, 384, 576, 3, 'act_bn_res', 2),         # stem sepconv1
    (2, 32, 32, 288, 288, 5, 'bn_act', 2),             # SPNet level 0
    (2, 16, 16, 384, 384, 5, 'bn_act', 2),
    (2, 8, 8, 480, 480, 5, 'bn_act', 2),
    (8, 4, 4, 576, 576, 5, 'bn_act', 1),
    (2, 16, 16, 64, 96, 3, 'plain', 2),                # TMA-staged kernel without ReLU prologue
    (5, 8, 8, 96, 80, 5, 'act_bn_res', 2),             # 8x8 maps: two frames per tile, odd frame count
    (3, 4, 8, 64, 96, 5, 'act_bn_res', 1),             # 4x8 maps: four frames per tile, 48 KB patches: conv_sep.cu's
                                                       # rings do not fit shared memory at bn_cta = 96 (falls to conv_tc)
]


@pytest.mark.parametrize('case', SEP_CASES)
@pytest.mark.parametrize('precision', [3, 1])
@pytest.mark.parametrize('kernel', ['tma', 'reg'])
def test_sepconv_tc(dev, case, precision, kernel):
    """kernel = 'tma': conv_sep.cu (TMA-staged patch, path 2) where it applies; 'reg': conv_tc.cu's
    register-sliding producer (path 1)."""
    _ffi.check(dev.lib.dh_set_option(dev.ctx.handle, b'sep_tma', 1 if kernel == 'tma' else 0))
    try:
        _run_sepconv(dev, case[:-1], precision, case[-1] if kernel == 'tma' else 1)
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
    pk = packed_weights(dev, pw.reshape(cin, cout))
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
    pk = packed_weights(dev, wt.reshape(64, 32))
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
    pk = packed_weights(dev, wt.reshape(34, 48))
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


# N, H, W, Cin, Cout, k, n_res; path: 2 = conv_sep.cu, 1 = conv_tc.cu's separable path (heights conv_sep does not
# tile) -- same epilogue; 0 = the two-kernel CUDA-core path (no packed weights), whose pointwise GEMM reads the residual
@pytest.mark.parametrize('case', [((2, 32, 32, 576, 576, 5, 2), 2), ((3, 32, 32, 64, 96, 3, 1), 2),
                                  ((1, 64, 32, 32, 32, 3, 2), 2), ((5, 16, 16, 288, 288, 5, 2), 2),
                                  ((3, 16, 16, 64, 96, 3, 1), 2), ((1, 12, 16, 32, 64, 5, 2), 1),
                                  ((2, 32, 32, 64, 96, 5, 2), 0)])
def test_sepconv_upsampled_residual(dev, case):
    """keras `add([a, UpSampling2D(b)])` (reception.py:122-127) folded into the epilogue of the conv that produces a:
    the LAST residual is a half-resolution tensor (dh_conv_desc.res_up2x); n_res = 2: identity shortcut + upsampled."""
    case, path = case
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
    pk = C.byref(packed_weights(dev, pw.reshape(cin, cout))) if path else NULLP
    xv, ov = dev.view(dev.put(x)), dev.view(out)
    dev.call('dh_sepconv2d_f32', C.byref(xv), dev.put(dw).data_ptr(), dev.put(pw).data_ptr(), pk,
             C.byref(d), C.byref(ov))
    assert dev.lib.dh_last_conv_path(dev.ctx.handle) == path
    assert _err(out.cpu().numpy(), ref) <= TOL3
    # a residual flagged as upsampled must have half the output's size
    d.res[n_res - 1] = dev.view(dev.put(r_full))
    rc = dev.lib.dh_sepconv2d_f32(dev.ctx.handle, C.byref(xv), dev.put(dw).data_ptr(), dev.put(pw).data_ptr(), pk,
                                  C.byref(d), C.byref(ov), dev.stream())
    assert rc < 0 and b'shape mismatch' in dev.lib.dh_last_error()
