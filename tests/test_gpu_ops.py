"""Per-kernel parity: every C-ABI op vs the fp64 oracle on seeded inputs, including the edge
cases the domain has (TF SAME asymmetric padding, stride 2, ragged channel counts, channel-sliced
views, -inf pool padding, one-hot / uniform heat-maps)."""
import ctypes as C
import zlib

import numpy as np
import pytest

from deephar_b200 import _ffi  # noqa: E402
from oracle import ops_np
from oracle import reception as oracle_reception

from gpu_util import NULLP, NULLV, Dev, close, conv_desc, layout_io, loop_batch, sam2d_ref

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def dev(cuda):
    return Dev(cuda)


CONV_CASES = [
    # (N,H,W,Cin,Cout, size, strides, padding)
    (2, 16, 16, 3, 32, (3, 3), (2, 2), 'same'),
    (1, 13, 11, 8, 20, (3, 3), (1, 1), 'same'),
    (2, 12, 12, 32, 64, (1, 1), (1, 1), 'same'),
    (1, 9, 9, 16, 24, (5, 1), (1, 1), 'same'),
    (1, 9, 9, 16, 24, (1, 5), (1, 1), 'same'),
    (1, 16, 16, 6, 10, (7, 7), (2, 2), 'same'),
    (1, 10, 10, 5, 7, (3, 3), (1, 1), 'valid'),
    (3, 8, 17, 2, 40, (3, 5), (1, 1), 'same'),
    (1, 32, 32, 64, 96, (3, 3), (2, 2), 'same'),
]


@pytest.mark.parametrize('case', CONV_CASES)
@pytest.mark.parametrize('fused', [False, True])
def test_conv2d(dev, case, fused):
    n, h, w, cin, cout, size, strides, padding = case
    rng = np.random.default_rng(zlib.crc32(repr(case).encode()))
    x = rng.standard_normal((n, h, w, cin))
    wt = rng.standard_normal(size + (cin, cout)) / np.sqrt(size[0] * size[1] * cin)
    xin = x
    pre = post = None
    res = []
    if fused:
        pre = (rng.uniform(0.5, 1.5, cin), rng.standard_normal(cin) * 0.3)
        post = (rng.uniform(0.5, 1.5, cout), rng.standard_normal(cout) * 0.3)
        xin = np.maximum(x * pre[0] + pre[1], 0)
    ref = ops_np.conv2d(xin, wt, strides, padding)
    if fused:
        ref = np.maximum(ref * post[0] + post[1], 0)
        r0, r1 = rng.standard_normal(ref.shape), rng.standard_normal(ref.shape)
        ref = ref + r0 + r1
        res = [dev.view(dev.put(r0)), dev.view(dev.put(r1))]
    xd, wd = dev.put(x), dev.put(wt)
    out = dev.empty(*ref.shape)
    d = conv_desc(dev, size, strides, padding, pre_relu=fused, post_relu=fused, pre=pre, post=post, res=res)
    xv, ov = dev.view(xd), dev.view(out)
    dev.call('dh_conv2d_f32', C.byref(xv), wd.data_ptr(), NULLP, C.byref(d), C.byref(ov))
    close(out.cpu().numpy(), ref)


def test_conv2d_channel_views(dev):
    """input = channel slice of a wider buffer, output = slice of a concat buffer."""
    rng = np.random.default_rng(5)
    big = rng.standard_normal((2, 8, 8, 24))
    wt = rng.standard_normal((3, 3, 10, 12)) * 0.1
    ref = ops_np.conv2d(big[..., 6:16], wt)
    bd, wd = dev.put(big), dev.put(wt)
    cat = dev.empty(2, 8, 8, 30)
    cat.fill_(7.0)
    d = conv_desc(dev, (3, 3))
    xv, ov = dev.view(bd, 6, 16), dev.view(cat, 5, 17)
    dev.call('dh_conv2d_f32', C.byref(xv), wd.data_ptr(), NULLP, C.byref(d), C.byref(ov))
    got = cat.cpu().numpy()
    close(got[..., 5:17], ref)
    assert np.all(got[..., :5] == 7.0) and np.all(got[..., 17:] == 7.0)


PW_CASES = [
    # N, H, W, Cin, Cout, n_res, prologue -- wide 1x1 convs with a small reduction (conv_pw_smallk_kernel)
    (2, 32, 32, 48, 576, 2, True),       # fReMap + block-end add (reception.py:156-164, :194-196)
    (1, 7, 5, 12, 272, 0, False),        # M tail (35 pixels), Cout not a multiple of 128
    (3, 9, 9, 64, 128, 1, True),         # largest Cin, one residual
    (1, 16, 16, 4, 576, 2, False),       # smallest Cin
]


@pytest.mark.parametrize('case', PW_CASES)
def test_conv2d_pointwise_smallk(dev, case):
    n, h, w, cin, cout, nres, prologue = case
    rng = np.random.default_rng(zlib.crc32(repr(case).encode()))
    x = rng.standard_normal((n, h, w, cin))
    wt = rng.standard_normal((1, 1, cin, cout)) / np.sqrt(cin)
    post = (rng.uniform(0.5, 1.5, cout), rng.standard_normal(cout) * 0.3)
    pre = None
    xin = x
    if prologue:
        pre = (rng.uniform(0.5, 1.5, cin), rng.standard_normal(cin) * 0.3)
        xin = np.maximum(x * pre[0] + pre[1], 0)
    ref = ops_np.conv2d(xin, wt) * post[0] + post[1]
    # residuals are channel slices of wider buffers (ld != C), output is a slice of a concat buffer
    rbig = [rng.standard_normal((n, h, w, cout + 8)) for _ in range(nres)]
    for r in rbig:
        ref = ref + r[..., 4:4 + cout]
    res = [dev.view(dev.put(r), 4, 4 + cout) for r in rbig]
    cat = dev.empty(n, h, w, cout + 12)
    cat.fill_(3.0)
    d = conv_desc(dev, (1, 1), pre_relu=prologue, pre=pre, post=post, res=res)
    xv, ov = dev.view(dev.put(x)), dev.view(cat, 8, 8 + cout)
    dev.call('dh_conv2d_f32', C.byref(xv), dev.put(wt).data_ptr(), NULLP, C.byref(d), C.byref(ov))
    assert dev.lib.dh_last_conv_path(dev.ctx.handle) == 3, 'pointwise small-K kernel was not taken'
    got = cat.cpu().numpy()
    close(got[..., 8:8 + cout], ref)
    assert np.all(got[..., :8] == 3.0) and np.all(got[..., 8 + cout:] == 3.0)


@pytest.mark.parametrize('case', [(3, 32, 32, 48, 576, 2), (2, 6, 32, 16, 128, 0)])
def test_conv2d_pointwise_pooled_second_output(dev, case):
    """dh_conv_desc.pool_out: the hourglass max-pools the tensor the block-end add produces (reception.py:108-110,
    194-196) -- the wide pointwise kernel writes MaxPooling2D((2,2)) of its result as a second output."""
    n, h, w, cin, cout, nres = case
    rng = np.random.default_rng(zlib.crc32(repr(case).encode()))
    x = rng.standard_normal((n, h, w, cin))
    wt = rng.standard_normal((1, 1, cin, cout)) / np.sqrt(cin)
    post = (rng.uniform(0.5, 1.5, cout), rng.standard_normal(cout) * 0.3)
    ref = ops_np.conv2d(np.maximum(x, 0), wt) * post[0] + post[1]
    rs = [rng.standard_normal(ref.shape) for _ in range(nres)]
    for r in rs:
        ref = ref + r
    pooled = ref.reshape(n, h // 2, 2, w // 2, 2, cout).max(axis=(2, 4))
    out, pout = dev.empty(*ref.shape), dev.empty(*pooled.shape)
    d = conv_desc(dev, (1, 1), pre_relu=True, post=post, res=[dev.view(dev.put(r)) for r in rs])
    d.pool_out = dev.view(pout)
    xv, ov = dev.view(dev.put(x)), dev.view(out)
    dev.call('dh_conv2d_f32', C.byref(xv), dev.put(wt).data_ptr(), NULLP, C.byref(d), C.byref(ov))
    assert dev.lib.dh_last_conv_path(dev.ctx.handle) == 3
    close(out.cpu().numpy(), ref)
    got = pout.cpu().numpy()
    close(got, pooled)
    assert np.array_equal(got, out.cpu().numpy().reshape(n, h // 2, 2, w // 2, 2, cout).max(axis=(2, 4)))   # exact max
    # wrong pooled shape, and a layer no pooling kernel takes: loud errors
    d.pool_out = dev.view(dev.empty(n, h // 2, w // 2, cout + 4))
    rc = dev.lib.dh_conv2d_f32(dev.ctx.handle, C.byref(xv), dev.put(wt).data_ptr(), NULLP, C.byref(d), C.byref(ov), dev.stream())
    assert rc < 0 and b'pool_out must be' in dev.lib.dh_last_error()
    x16 = dev.put(rng.standard_normal((n, 16, 16, cin)))
    o16, p16 = dev.empty(n, 16, 16, cout), dev.empty(n, 8, 8, cout)
    d2 = conv_desc(dev, (1, 1), pre_relu=True, post=post)
    d2.pool_out = dev.view(p16)
    xv16, ov16 = dev.view(x16), dev.view(o16)
    args16 = (C.byref(xv16), dev.put(wt).data_ptr(), NULLP, C.byref(d2), C.byref(ov16))
    # ... and the 3x3x3 stem conv, whose direct small-K kernel writes no pooled output; the plan refuses both too
    xs, ws = dev.put(rng.standard_normal((n, 16, 16, 3))), dev.put(rng.standard_normal((3, 3, 3, 32)) / np.sqrt(27))
    os_, ps = dev.empty(n, 16, 16, 32), dev.empty(n, 8, 8, 32)
    d3 = conv_desc(dev, (3, 3))
    xvs, ovs = dev.view(xs), dev.view(os_)
    args_stem = (C.byref(xvs), ws.data_ptr(), NULLP, C.byref(d3), C.byref(ovs))
    info = _ffi.dh_conv_plan_info()
    assert dev.lib.dh_conv2d_plan(dev.ctx.handle, *args_stem, C.byref(info)) == 0 and info.path == 0   # small-K kernel
    d3.pool_out = dev.view(ps)
    for args in (args16, args_stem):
        rc = dev.lib.dh_conv2d_f32(dev.ctx.handle, *args, dev.stream())
        assert rc < 0 and b'wide pointwise kernel only' in dev.lib.dh_last_error()
        rc = dev.lib.dh_conv2d_plan(dev.ctx.handle, *args, C.byref(info))
        assert rc < 0 and b'wide pointwise kernel only' in dev.lib.dh_last_error()
    dev.torch.cuda.synchronize()
    assert np.isnan(ps.cpu().numpy()).all() and np.isnan(os_.cpu().numpy()).all()        # nothing launched


SEP_CASES = [
    (2, 16, 16, 32, 48, (5, 5), (1, 1)),
    (1, 8, 8, 24, 24, (3, 3), (1, 1)),
    (1, 9, 7, 17, 33, (5, 5), (1, 1)),
    (1, 16, 16, 16, 32, (3, 3), (2, 2)),
    (2, 4, 4, 64, 64, (5, 5), (1, 1)),
]


@pytest.mark.parametrize('case', SEP_CASES)
@pytest.mark.parametrize('mode', ['plain', 'act_bn_res', 'bn_act'])
def test_sepconv2d(dev, case, mode):
    n, h, w, cin, cout, size, strides = case
    rng = np.random.default_rng(zlib.crc32(repr(case).encode()))
    x = rng.standard_normal((n, h, w, cin))
    dw = rng.standard_normal(size + (cin, 1)) / np.sqrt(size[0] * size[1])
    pw = rng.standard_normal((1, 1, cin, cout)) / np.sqrt(cin)
    pre = post = None
    res = []
    xin = x
    if mode == 'act_bn_res':          # reception.py:43-59 _sepconv_residual
        xin = np.maximum(x, 0)
        post = (rng.uniform(0.5, 1.5, cout), rng.standard_normal(cout) * 0.3)
    elif mode == 'bn_act':            # models/common.py:50-55 residual_unit (BN -> ReLU -> sepconv)
        pre = (rng.uniform(0.5, 1.5, cin), rng.standard_normal(cin) * 0.3)
        xin = np.maximum(x * pre[0] + pre[1], 0)
    ref = ops_np.separable_conv2d(xin, dw, pw, strides, 'same')
    if mode == 'act_bn_res':
        ref = ref * post[0] + post[1]
        r0 = rng.standard_normal(ref.shape)
        ref = ref + r0
        res = [dev.view(dev.put(r0))]
    xd = dev.put(x)
    out = dev.empty(*ref.shape)
    d = conv_desc(dev, size, strides, 'same', pre_relu=(mode != 'plain'), pre=pre, post=post, res=res)
    xv, ov = dev.view(xd), dev.view(out)
    dev.call('dh_sepconv2d_f32', C.byref(xv), dev.put(dw).data_ptr(), dev.put(pw).data_ptr(), NULLP,
             C.byref(d), C.byref(ov))
    close(out.cpu().numpy(), ref)


POOLS = [((3, 3), (2, 2), 'same'), ((2, 2), (2, 2), 'valid'), ((2, 2), (2, 2), 'same'), ((2, 2), (1, 2), 'same')]


# layouts: 'scalar' C = 13 (pool_kernel<0, 1>); 'float4' C = 16 (pool_kernel<0, 4>); 'slice' input and output are
# 16-byte aligned channel slices of wider buffers (float4 too); 'large' enough work for two grid-stride iterations
@pytest.mark.parametrize('case', [pl + (layout,) for layout in ('scalar', 'float4', 'slice', 'large') for pl in POOLS])
def test_maxpool(dev, case):
    pool, strides, padding, layout = case
    rng = np.random.default_rng(7)
    shape = {'scalar': (2, 9, 11, 13), 'float4': (2, 9, 11, 16), 'slice': (2, 9, 11, 16), 'large': (1, 18, 22, 64)}[layout]
    if layout == 'large':
        _, ho, wo, _ = ops_np.maxpool2d(np.zeros((1, 18, 22, 1)), pool, strides, padding).shape
        shape = (loop_batch(dev, ho * wo * 64 // 4),) + shape[1:]
    x = rng.standard_normal(shape) - 3.0          # negative values: -inf padding matters
    ref = ops_np.maxpool2d(x, pool, strides, padding).astype(np.float32)
    xv, out = layout_io(dev, x, ref.shape, layout)
    dev.call('dh_maxpool2d_f32', C.byref(xv), pool[0], pool[1], strides[0], strides[1],
             1 if padding == 'same' else 0, C.byref(out.view))
    assert np.array_equal(out.get(), ref)


def test_upsample_add_and_add_n(dev):
    rng = np.random.default_rng(8)
    a = rng.standard_normal((2, 8, 6, 10))
    b = rng.standard_normal((2, 4, 3, 10))
    out = dev.empty(2, 8, 6, 10)
    av, bv, ov = dev.view(dev.put(a)), dev.view(dev.put(b)), dev.view(out)
    dev.call('dh_upsample2x_add_f32', C.byref(av), C.byref(bv), C.byref(ov))
    close(out.cpu().numpy(), a + ops_np.upsample2d(b), 1e-6)
    dev.call('dh_upsample2x_add_f32', NULLV, C.byref(bv), C.byref(ov))
    close(out.cpu().numpy(), ops_np.upsample2d(b), 1e-7)
    from deephar_b200 import _ffi
    c = rng.standard_normal(a.shape)
    arr = (_ffi.dh_view * 3)(dev.view(dev.put(a)), dev.view(dev.put(c)), dev.view(dev.put(a)))
    sc, sh = rng.uniform(0.5, 1.5, 10), rng.standard_normal(10)
    dev.call('dh_add_n_f32', arr, 3, dev.put(sc).data_ptr(), dev.put(sh).data_ptr(), 1, C.byref(ov))
    close(out.cpu().numpy(), np.maximum((2 * a + c) * sc + sh, 0), 1e-6)


SAM_SHAPES = [(3, 32, 32, 16), (2, 16, 16, 17), (5, 8, 8, 16), (4, 4, 4, 17), (2, 32, 32, 48), (1, 6, 9, 5)]


@pytest.mark.parametrize('shape', SAM_SHAPES)
@pytest.mark.parametrize('conf_on_prob', [0, 1])
def test_softargmax2d(dev, shape, conf_on_prob):
    rng = np.random.default_rng(sum(shape))
    h = rng.standard_normal(shape) * 3.0
    n, hh, ww, c = shape
    for i in range(n):                      # planted peaks (SURVEY 8d micro-bench recipe)
        for j in range(c):
            h[i, rng.integers(hh), rng.integers(ww), j] += 12.0
    alpha = 1.0 if conf_on_prob == 0 else 0.8
    xy, conf, p = sam2d_ref(h, alpha, conf_on_prob)
    pose, cf, prob = dev.empty(n, c, 2), dev.empty(n, c, 1), dev.empty(*shape)
    hv, pv = dev.view(dev.put(h)), dev.view(prob)
    dev.call('dh_softargmax2d_f32', C.byref(hv), NULLV, C.c_float(alpha), conf_on_prob,
             pose.data_ptr(), cf.data_ptr(), C.byref(pv))
    close(pose.cpu().numpy(), xy, 2e-6)
    close(cf.cpu().numpy(), conf, 5e-6)
    close(prob.cpu().numpy(), p, 2e-6)
    # argmax pixel of every map must be identical to the oracle's (north_star: bit-exact indices)
    got_arg = prob.cpu().numpy().reshape(n, -1, c).argmax(axis=1)
    assert np.array_equal(got_arg, p.reshape(n, -1, c).argmax(axis=1))


def test_softargmax2d_depth(dev):
    rng = np.random.default_rng(11)
    shape = (3, 16, 16, 17)
    h, d = rng.standard_normal(shape) * 3, rng.standard_normal(shape) * 2
    xyz, conf, _ = sam2d_ref(h, 1.0, 1, d)
    pose, cf = dev.empty(3, 17, 3), dev.empty(3, 17, 1)
    hv, dv = dev.view(dev.put(h)), dev.view(dev.put(d))
    dev.call('dh_softargmax2d_f32', C.byref(hv), C.byref(dv), C.c_float(1.0), 1, pose.data_ptr(),
             cf.data_ptr(), NULLV)
    close(pose.cpu().numpy(), xyz, 2e-6)
    close(cf.cpu().numpy(), conf, 5e-6)


def test_softargmax2d_known_answers(dev):
    """one-hot -> grid coordinate, uniform -> (0.5, 0.5), confidence 1 and 4/R^2 (SURVEY 8c)."""
    R, C_ = 16, 4
    h = np.full((2, R, R, C_), -80.0)
    peaks = [(0, 0), (15, 15), (3, 9), (8, 1)]
    for c, (r, q) in enumerate(peaks):
        h[0, r, q, c] = 80.0
    h[1] = 0.0
    pose, cf = dev.empty(2, C_, 2), dev.empty(2, C_, 1)
    hv = dev.view(dev.put(h))
    dev.call('dh_softargmax2d_f32', C.byref(hv), NULLV, C.c_float(1.0), 1, pose.data_ptr(), cf.data_ptr(), NULLV)
    p, c_ = pose.cpu().numpy(), cf.cpu().numpy()
    for c, (r, q) in enumerate(peaks):
        assert np.allclose(p[0, c], [q / (R - 1), r / (R - 1)], atol=1e-6)
    assert np.allclose(c_[0], 1.0, atol=1e-6)
    assert np.allclose(p[1], 0.5, atol=1e-6)
    assert np.allclose(c_[1], 4.0 / R ** 2, rtol=1e-5)


@pytest.mark.parametrize('shape,nj,nctx', [((3, 32, 32, 48), 16, 2), ((2, 16, 16, 20), 5, 3)])
def test_softargmax2d_context(dev, shape, nj, nctx):
    rng = np.random.default_rng(12)
    h = rng.standard_normal(shape) * 3.0 + 1.0
    pose, vis, _ = oracle_reception.pose_regression_2d_context(ops_np, h, nj, nctx, 0.8)
    po, vo = dev.empty(shape[0], nj, 2), dev.empty(shape[0], nj, 1)
    hv = dev.view(dev.put(h))
    dev.call('dh_softargmax2d_ctx_f32', C.byref(hv), nj, nctx, C.c_float(0.8), po.data_ptr(), vo.data_ptr())
    close(po.cpu().numpy(), pose, 3e-6)
    close(vo.cpu().numpy(), vis, 3e-6)


@pytest.mark.parametrize('shape,nj,D', [((2, 32, 32, 272), 17, 16), ((3, 8, 8, 30), 5, 6), ((5, 8, 8, 160), 20, 8),
                                        ((3, 16, 16, 272), 17, 16)])
@pytest.mark.parametrize('stream', [1, 0])
def test_softargmax3d(dev, shape, nj, D, stream):
    """stream = 1: the cluster-split streaming kernel (softargmax.cu) where it applies (dense volumes whose
    pixel count splits into 4 x 16-pixel chunks, C % 4 == 0); 0: the staged one-CTA-per-frame kernel."""
    rng = np.random.default_rng(13)
    h = rng.standard_normal(shape) * 3.0
    h[0, 3, 5, 2 * nj + 1] += 40.0                       # a planted peak: joint 1 at depth slice 2, pixel (3, 5)
    pose, vis, _ = oracle_reception.pose_regression_3d(ops_np, h, nj, D)
    po, vo = dev.empty(shape[0], nj, 3), dev.empty(shape[0], nj, 1)
    hv = dev.view(dev.put(h))
    _ffi.check(dev.lib.dh_set_option(dev.ctx.handle, b'sam3d_stream', stream))
    try:
        dev.call('dh_softargmax3d_f32', C.byref(hv), nj, D, po.data_ptr(), vo.data_ptr())
    finally:
        _ffi.check(dev.lib.dh_set_option(dev.ctx.handle, b'sam3d_stream', 1))
    close(po.cpu().numpy(), pose, 3e-6)
    close(vo.cpu().numpy(), vis, 3e-6)


def test_softargmax3d_ex_merge_variant(dev):
    """action.py:291-295: visible = sigmoid(2 * (max hxy + max hz)) and hs = channel_softmax_2d(hxy)."""
    rng = np.random.default_rng(15)
    nj, D = 20, 8
    h = rng.standard_normal((3, 16, 16, nj * D)) * 2.0
    pose, _, hxy = oracle_reception.pose_regression_3d(ops_np, h, nj, D)
    h5 = h.reshape(3, 16, 16, D, nj)
    vis = 1.0 / (1.0 + np.exp(-2.0 * (h5.mean(3).max((1, 2)) + h5.mean((1, 2)).max(1))))[..., None]
    prob = ops_np.channel_softmax_2d(hxy)
    po, vo, pr = dev.empty(3, nj, 3), dev.empty(3, nj, 1), dev.empty(3, 16, 16, nj)
    hv, pv = dev.view(dev.put(h)), dev.view(pr)
    dev.call('dh_softargmax3d_ex_f32', C.byref(hv), nj, D, C.c_float(2.0), po.data_ptr(), vo.data_ptr(), C.byref(pv))
    close(po.cpu().numpy(), pose, 3e-6)
    close(vo.cpu().numpy(), vis, 3e-6)
    close(pr.cpu().numpy(), prob, 3e-6)


@pytest.mark.parametrize('head,shape,stream', [('2d', (2, 32, 32, 48), 1), ('2d', (3, 32, 32, 16), 1),
                                               ('3d', (3, 16, 16, 160), 1), ('3d', (3, 16, 16, 160), 0)])
def test_softargmax_no_prob(dev, head, shape, stream):
    """The heads without a probability output, on shapes the streaming kernels take: the plain 2-D head (alpha 1,
    confidence on the raw maps, no depth) and the merge model's 3-D head (vis_scale 2; stream = 0 runs the staged
    kernel)."""
    rng = np.random.default_rng(16)
    n = shape[0]
    h = rng.standard_normal(shape) * 3.0
    if head == '2d':
        xy, conf, _ = sam2d_ref(h, 1.0, 0)
        pose, cf = dev.empty(n, shape[3], 2), dev.empty(n, shape[3], 1)
        hv = dev.view(dev.put(h))
        dev.call('dh_softargmax2d_f32', C.byref(hv), NULLV, C.c_float(1.0), 0, pose.data_ptr(), cf.data_ptr(), NULLV)
        close(pose.cpu().numpy(), xy, 2e-6)
        close(cf.cpu().numpy(), conf, 5e-6)
        return
    nj, D = 20, 8
    pose, _, _ = oracle_reception.pose_regression_3d(ops_np, h, nj, D)
    h5 = h.reshape(shape[:3] + (D, nj))
    vis = 1.0 / (1.0 + np.exp(-2.0 * (h5.mean(3).max((1, 2)) + h5.mean((1, 2)).max(1))))[..., None]
    po, vo = dev.empty(n, nj, 3), dev.empty(n, nj, 1)
    hv = dev.view(dev.put(h))
    _ffi.check(dev.lib.dh_set_option(dev.ctx.handle, b'sam3d_stream', stream))
    try:
        dev.call('dh_softargmax3d_ex_f32', C.byref(hv), nj, D, C.c_float(2.0), po.data_ptr(), vo.data_ptr(), NULLV)
    finally:
        _ffi.check(dev.lib.dh_set_option(dev.ctx.handle, b'sam3d_stream', 1))
    close(po.cpu().numpy(), pose, 3e-6)
    close(vo.cpu().numpy(), vis, 3e-6)


def test_kron_maxmin_softmax_mask(dev):
    rng = np.random.default_rng(14)
    p = ops_np.channel_softmax_2d(rng.standard_normal((6, 8, 8, 17)) * 2)
    z = rng.standard_normal((6, 8, 8, 150))
    ref = np.einsum('nhwj,nhwf->njf', p, z)
    out = dev.empty(6, 17, 150)
    pv, zv = dev.view(dev.put(p)), dev.view(dev.put(z))
    dev.call('dh_kron_pool_f32', C.byref(pv), C.byref(zv), out.data_ptr())
    close(out.cpu().numpy(), ref, 1e-5)

    x = rng.standard_normal((3, 5, 9, 15))
    mm = dev.empty(3, 3, 5, 15)
    xv, mv = dev.view(dev.put(x)), dev.view(mm)
    dev.call('dh_maxmin_pool2d_f32', C.byref(xv), C.byref(mv))
    close(mm.cpu().numpy(), ops_np.max_min_pooling(x), 1e-6)
    sm = dev.empty(3, 15)
    dev.call('dh_global_maxmin_softmax_f32', C.byref(xv), sm.data_ptr())
    close(sm.cpu().numpy(), ops_np.softmax(ops_np.global_max_min_pooling(x)), 1e-6)

    pp, cc = rng.standard_normal((4, 16, 17, 3)), rng.uniform(size=(4, 16, 17, 1))
    mo = dev.empty(4, 16, 17, 3)
    dev.call('dh_mask_mul_f32', dev.put(pp).data_ptr(), dev.put(cc).data_ptr(), 4 * 16 * 17, 3, mo.data_ptr())
    close(mo.cpu().numpy(), pp * cc, 1e-6)


def test_argument_errors(dev):
    """shape mismatches are reported as errors, not executed."""
    from deephar_b200 import _ffi
    x = dev.put(np.zeros((1, 8, 8, 4)))
    out = dev.empty(1, 8, 8, 5)
    w = dev.put(np.zeros((3, 3, 4, 6)))
    d = conv_desc(dev, (3, 3))
    xv, ov = dev.view(x), dev.view(out)          # out has 5 channels, weights say 6 -> fine for conv (uses out.c)
    ov.h = 7
    rc = dev.lib.dh_conv2d_f32(dev.ctx.handle, C.byref(xv), w.data_ptr(), NULLP, C.byref(d), C.byref(ov), dev.stream())
    assert rc < 0 and b'expected' in dev.lib.dh_last_error()
