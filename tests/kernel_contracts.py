"""The forward kernel contracts of include/deephar_b200.h in float64 -- TEST INFRASTRUCTURE (never imported by the product).
One function per entry point takes the operands as arrays and the entry point's own scalar arguments and returns what the
kernel writes, with the oracle's primitives (`oracle/ops_np.py`).  The stand-in device (tests/fake_cuda.py) calls them
from ctypes arguments, the plan emulator (tests/plan_emulator.py) from plan ops, and so the GPU tests' launch checker."""
import numpy as np

from oracle import ops_np as O


def prologue(x, pre=None, pre_relu=False):
    """a convolution's input after its fused pre = (pre_scale, pre_shift) and ReLU: the MMA's operand"""
    if pre is not None:
        x = x * pre[0] + pre[1]
    if pre_relu:
        x = np.maximum(x, 0.0)
    return x


def conv(x, w, strides, padding, pre=None, pre_relu=False, post=None, post_relu=False, res=(), res_up2x=0,
         pool_out=False):
    """dh_conv2d_f32 (w: HWIO kernel) and dh_sepconv2d_f32 (w: (depthwise, pointwise)) in dh_conv_desc's order ->
    [y], or [y, MaxPooling2D((2, 2))(y)] with pool_out; bit i of res_up2x upsamples res[i] 2x"""
    x = prologue(x, pre, pre_relu)
    if isinstance(w, tuple):
        y = O.separable_conv2d(x, w[0], w[1], strides, padding)
    else:
        y = O.conv2d(x, w, strides, padding)
    if post is not None:
        y = y * post[0] + post[1]
    if post_relu:
        y = np.maximum(y, 0.0)
    for i, r in enumerate(res):
        if (res_up2x >> i) & 1:
            r = O.upsample2d(r)
        y = y + r
    return [y, O.maxpool2d(y, (2, 2))] if pool_out else [y]


def maxpool(x, pool, strides, padding):
    """dh_maxpool2d_f32"""
    return O.maxpool2d(x, pool, strides, padding)


def upsample2x_add(b, a=None):
    """dh_upsample2x_add_f32: UpSampling2D((2, 2))(b), plus a unless it is None"""
    y = O.upsample2d(b)
    return y if a is None else y + a


def add_n(ins, scale=None, shift=None, relu=False):
    """dh_add_n_f32: the sum of ins, then * scale + shift unless scale is None, then ReLU"""
    y = sum(ins)
    if scale is not None:
        y = y * scale + shift
    if relu:
        y = np.maximum(y, 0.0)
    return y


def softargmax2d(h, alpha, conf_on_prob, d=None):
    """dh_softargmax2d_f32 -> pose (N, C, 2, or 3 with d's depth expectation), confidence (N, C, 1) of p (of h if not
    conf_on_prob), the probabilities p (N, H, W, C)"""
    p = O.channel_softmax_2d(h, alpha)
    pose = O.softargmax2d(p)
    if d is not None:
        pose = np.concatenate([pose, np.sum(O.sigmoid(d) * p, axis=(1, 2))[..., None]], axis=-1)     # spnet.py:201-205
    return pose, O.keypoint_confidence(p if conf_on_prob else h), p


def softargmax2d_ctx(h, nj, n_ctx, alpha_mix):
    """dh_softargmax2d_ctx_f32 -> pose (N, nj, 2), visibility (N, nj, 1)"""
    hs, hc = h[..., :nj], h[..., nj:]
    ys, yc = O.softargmax2d(O.channel_softmax_2d(hs)), O.softargmax2d(O.channel_softmax_2d(hc))
    pc = O.keypoint_confidence(hc)                                          # on RAW maps (blocks.py:328-343)
    grp = lambda v: v.reshape(v.shape[0], nj, n_ctx, -1).sum(axis=2)       # noqa: E731   blocks.py:227-233
    with np.errstate(divide='ignore', invalid='ignore'):
        pose = alpha_mix * ys + (1 - alpha_mix) * grp(yc * pc) / grp(pc)
    return pose, O.keypoint_confidence(hs)


def softargmax3d(h, nj, depth_maps, vis_scale=1.0):
    """dh_softargmax3d_f32 (vis_scale 1) and dh_softargmax3d_ex_f32 (h's channel d * nj + j: depth d of joint j) ->
    pose (N, nj, 3), visibility (N, nj, 1), the probabilities channel_softmax_2d(hxy) (N, H, W, nj)"""
    n, hh, ww, _ = h.shape
    h5 = h.reshape(n, hh, ww, depth_maps, nj)
    hxy, hz = h5.mean(axis=3), h5.mean(axis=(1, 2))
    p = O.channel_softmax_2d(hxy)
    pose = np.concatenate([O.softargmax2d(p), O.lin_interpolation_1d(O.channel_softmax_1d(hz))], axis=-1)
    return pose, O.sigmoid(vis_scale * (hxy.max(axis=(1, 2)) + hz.max(axis=1)))[..., None], p


def kron_pool(p, z):
    """dh_kron_pool_f32 -> (N, nj, F)"""
    return np.einsum('nhwj,nhwf->njf', p, z)


def zeropad(x, top, left, out_hw):
    """dh_zeropad2d_f32: x at row top, column left of zero maps of out_hw = (height, width)"""
    (oh, ow), (_, h, w, _) = out_hw, x.shape
    return O.zeropad2d(x, ((top, oh - top - h), (left, ow - left - w)))


def maxmin_pool(x):
    """dh_maxmin_pool2d_f32"""
    return O.max_min_pooling(x, (2, 2), 'same')


def global_maxmin_softmax(x):
    """dh_global_maxmin_softmax_f32 -> (N, C)"""
    return O.softmax(O.global_max_min_pooling(x))


def mask_mul(p, c):
    """dh_mask_mul_f32: each row of p times its row of c"""
    return p * c
