"""The soft-argmax heads and the memory-bound kernels on the paths the network runs, against the fp64 oracle: the
streaming 2-D head with several frames per CTA, maps too narrow for it, the staged heads on channel views, the 3-D
heads on non-square and wide volumes, kronecker pooling at its limits, and the pooling / upsample / add / pad kernels
on their float4 paths, on channel slices and with grid-stride loops.  Where the kernel's float32 arithmetic can be
reproduced the comparison is exact.  One test per group asserts which kernel each case reaches."""
import ctypes as C
import json
import os
import tempfile
import zlib

import numpy as np
import pytest

from deephar_b200 import _ffi
from oracle import ops_np
from oracle import reception as oracle_reception

from gpu_util import NULLV, Dev, Out, close, layout_io, loop_batch, num_sms, sam2d_ref, sliced

pytestmark = pytest.mark.gpu
F32 = np.float32


@pytest.fixture(scope='module')
def dev(cuda):
    return Dev(cuda)


def launched(dev, fn):
    """The names of the CUDA kernels fn() launches, from a torch.profiler trace.  fn launches at least the fill of an
    output buffer; a trace that holds no kernel at all (the profiler occasionally returns one) is taken again."""
    from torch.profiler import ProfilerActivity, profile
    for _ in range(3):
        dev.torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            fn()
            dev.torch.cuda.synchronize()
        with tempfile.TemporaryDirectory() as d:
            path = os.path.join(d, 'trace.json')
            prof.export_chrome_trace(path)
            with open(path) as f:
                names = sorted({e['name'] for e in json.load(f)['traceEvents'] if e.get('cat') == 'kernel'})
        if names:
            return names
    return names


def _rng(*case):
    return np.random.default_rng(zlib.crc32(repr(case).encode()))


def planted(shape, *seed):
    """N(0, 3) heat-maps with a +12 peak at a random pixel of every map (as test_gpu_ops.test_softargmax2d)"""
    rng = _rng(shape, *seed)
    n, hh, ww, c = shape
    h = rng.standard_normal(shape) * 3.0
    h[np.arange(n)[:, None], rng.integers(hh, size=(n, c)), rng.integers(ww, size=(n, c)), np.arange(c)] += 12.0
    return h


# ------------------------------------------------------------------------------------------------------------------
# 2-D heads
# ------------------------------------------------------------------------------------------------------------------
def run_sam2d(dev, hv, n, c, ctx=None):
    """plain head (alpha 1, confidence on the raw maps), or the context head with ctx = (nj, n_ctx) and alpha_mix 0.8
    -> (pose, confidence)"""
    if ctx:
        nj, nctx = ctx
        pose, conf = dev.empty(n, nj, 2), dev.empty(n, nj, 1)
        dev.call('dh_softargmax2d_ctx_f32', C.byref(hv), nj, nctx, C.c_float(0.8), pose.data_ptr(), conf.data_ptr())
    else:
        pose, conf = dev.empty(n, c, 2), dev.empty(n, c, 1)
        dev.call('dh_softargmax2d_f32', C.byref(hv), NULLV, C.c_float(1.0), 0, pose.data_ptr(), conf.data_ptr(), NULLV)
    return pose.cpu().numpy(), conf.cpu().numpy()


def check_sam2d(got, h, ctx):
    """against the fp64 oracle, at test_gpu_ops' tolerances for the plain and the context head"""
    if ctx:
        pose, conf, _ = oracle_reception.pose_regression_2d_context(ops_np, h, ctx[0], ctx[1], 0.8)
        close(got[0], pose, 3e-6)
        close(got[1], conf, 3e-6)
    else:
        pose, conf, _ = sam2d_ref(h, 1.0, 0)
        close(got[0], pose, 2e-6)
        close(got[1], conf, 5e-6)


def stream_frames(dev):
    """frames at which the persistent streaming kernel (grid = num_sms) runs 3 frames on CTAs 0-4 and 2 on the rest"""
    return 2 * num_sms(dev) + 5


# (H, W, C), context: the ReceptionNet head maps the streaming kernel serves
STREAM_CASES = [((32, 32, 48), None), ((32, 32, 16), None), ((32, 32, 48), (16, 2))]


@pytest.mark.parametrize('hwc,ctx', STREAM_CASES)
def test_sam2d_stream_several_frames_per_cta(dev, hwc, ctx):
    """The streaming kernel's TMA ring runs across frame boundaries; the same maps as channels [0, C) of a buffer with
    ld = C + 4 go to the staged kernel, whose confidence -- (top-left + top-right) + (bottom-left + bottom-right) in
    float32, then the max -- must be the streaming kernel's bit for bit."""
    n = stream_frames(dev)
    h = planted((n,) + hwc)
    streamed = run_sam2d(dev, dev.view(dev.put(h)), n, hwc[2], ctx)
    staged = run_sam2d(dev, sliced(dev, h, 0, hwc[2] + 4), n, hwc[2], ctx)
    check_sam2d(streamed, h, ctx)
    check_sam2d(staged, h, ctx)
    assert np.array_equal(streamed[1], staged[1])


# (N, H, W, C), context, kernel.  W < 4 leaves fewer streaming consumer threads (W * C/4) than channels, and the
# combine and output steps need one per channel: the staged kernel serves those maps.  (16, 4, 256) is the boundary
# W * C/4 == C and streams.
NARROW_CASES = [((2, 64, 2, 128), None, 'softargmax2d_kernel'), ((2, 44, 3, 128), None, 'softargmax2d_kernel'),
                ((2, 16, 2, 512), None, 'softargmax2d_kernel'), ((2, 64, 2, 128), (32, 3), 'softargmax2d_kernel'),
                ((2, 16, 4, 256), None, 'sam_stream_kernel')]


@pytest.mark.parametrize('shape,ctx', [c[:2] for c in NARROW_CASES])
def test_sam2d_narrow_maps(dev, shape, ctx):
    h = planted(shape, ctx)
    check_sam2d(run_sam2d(dev, dev.view(dev.put(h)), shape[0], shape[3], ctx), h, ctx)


# heat-map channel offset (in a buffer of C + 8 channels: a multiple of 4 stages with float4 loads, any other offset
# with scalar ones), depth-map offset, probability-export offset (None: not given), conf_on_prob, alpha
VIEW_CASES = [(4, 4, 8, 0, 1.0), (1, 3, 5, 1, 0.8), (4, None, 2, 1, 1.25), (3, 2, None, 0, 0.7)]
VIEW_SHAPE = (3, 16, 12, 20)


def run_sam2d_views(dev, h, d, case):
    hoff, doff, poff, conf_on_prob, alpha = case
    n, _, _, c = h.shape
    ld = c + 8
    pose, conf = dev.empty(n, c, 2 if d is None else 3), dev.empty(n, c, 1)
    prob = Out(dev, h.shape, poff, ld) if poff is not None else None
    hv = sliced(dev, h, hoff, ld)
    dv = C.byref(sliced(dev, d, doff, ld)) if d is not None else NULLV
    dev.call('dh_softargmax2d_f32', C.byref(hv), dv, C.c_float(alpha), conf_on_prob, pose.data_ptr(),
             conf.data_ptr(), C.byref(prob.view) if prob else NULLV)
    return pose.cpu().numpy(), conf.cpu().numpy(), prob.get() if prob else None


@pytest.mark.parametrize('case', VIEW_CASES)
def test_sam2d_staged_views(dev, case):
    """The staged 2-D head on heat-maps and depth maps that are channel slices, exporting the probabilities into a
    slice of a wider buffer whose other channels must survive."""
    h = planted(VIEW_SHAPE, case)
    d = _rng(case).standard_normal(VIEW_SHAPE) * 2.0 if case[1] is not None else None
    xy, conf, p = sam2d_ref(h, case[4], case[3], d)
    got_pose, got_conf, got_prob = run_sam2d_views(dev, h, d, case)
    close(got_pose, xy, 2e-6)
    close(got_conf, conf, 5e-6)
    if got_prob is not None:
        close(got_prob, p, 2e-6)


HEAD2D_PATHS = ([(('stream',) + c, 'sam_stream_kernel') for c in STREAM_CASES] +
                [(('stream_wide_ld',) + c, 'softargmax2d_kernel') for c in STREAM_CASES] +
                [(('narrow', s, ctx), k) for s, ctx, k in NARROW_CASES] +
                [(('views', c), 'softargmax2d_kernel') for c in VIEW_CASES])


@pytest.mark.parametrize('case,kernel', HEAD2D_PATHS)
def test_head2d_paths(dev, case, kernel):
    """Each 2-D head case above reaches the kernel its test is about."""
    what = case[0]
    if what in ('stream', 'stream_wide_ld'):
        hwc, ctx = case[1:]
        n = stream_frames(dev)
        h = planted((n,) + hwc)
        hv = dev.view(dev.put(h)) if what == 'stream' else sliced(dev, h, 0, hwc[2] + 4)
        names = launched(dev, lambda: run_sam2d(dev, hv, n, hwc[2], ctx))
    elif what == 'narrow':
        shape, ctx = case[1:]
        hv = dev.view(dev.put(planted(shape, ctx)))
        names = launched(dev, lambda: run_sam2d(dev, hv, shape[0], shape[3], ctx))
    else:
        h = planted(VIEW_SHAPE, case[1])
        d = h * 0.5 if case[1][1] is not None else None
        names = launched(dev, lambda: run_sam2d_views(dev, h, d, case[1]))
    heads = [s for s in names if 'softargmax' in s or 'sam_stream' in s]
    assert len(heads) == 1 and kernel in heads[0], names


# ------------------------------------------------------------------------------------------------------------------
# 3-D heads
# ------------------------------------------------------------------------------------------------------------------
def volume(shape, nj, *seed):
    """N(0, 3) volumes, channel d * nj + j, with a +40 peak at a random pixel and depth of every joint"""
    rng = _rng(shape, nj, *seed)
    n, hh, ww, c = shape
    h = rng.standard_normal(shape) * 3.0
    ch = rng.integers(c // nj, size=(n, nj)) * nj + np.arange(nj)
    h[np.arange(n)[:, None], rng.integers(hh, size=(n, nj)), rng.integers(ww, size=(n, nj)), ch] += 40.0
    return h


def run_sam3d(dev, hv, n, nj, D, stream, vis_scale=None, prob=None):
    """sam3d_stream = stream (0: the staged kernel even where the streaming plan applies), restored to 1 afterwards;
    vis_scale None calls dh_softargmax3d_f32, else dh_softargmax3d_ex_f32 -> (pose, visibility)"""
    po, vo = dev.empty(n, nj, 3), dev.empty(n, nj, 1)
    _ffi.check(dev.lib.dh_set_option(dev.ctx.handle, b'sam3d_stream', stream))
    try:
        if vis_scale is None:
            dev.call('dh_softargmax3d_f32', C.byref(hv), nj, D, po.data_ptr(), vo.data_ptr())
        else:
            dev.call('dh_softargmax3d_ex_f32', C.byref(hv), nj, D, C.c_float(vis_scale), po.data_ptr(), vo.data_ptr(),
                     C.byref(prob.view) if prob else NULLV)
    finally:
        _ffi.check(dev.lib.dh_set_option(dev.ctx.handle, b'sam3d_stream', 1))
    return po.cpu().numpy(), vo.cpu().numpy()


# (N, H, W, C), nj, D, sam3d_stream, kernel.  (6, 32): P = 192, so each CTA of the 4-CTA cluster takes 48 pixels in
# 3 chunks and the quarters of ranks 1 and 3 start mid-row.  nj = 17, D = 32: C = 544 > 512, so each staged thread
# accumulates two depth-marginal channels (and the streaming plan, C <= 480, refuses it).
SAM3D_CASES = [((5, 6, 32, 272), 17, 16, 1, 'sam3d_stream_kernel'), ((5, 6, 32, 272), 17, 16, 0, 'softargmax3d_kernel'),
               ((2, 8, 6, 544), 17, 32, 1, 'softargmax3d_kernel')]


@pytest.mark.parametrize('shape,nj,D,stream', [c[:4] for c in SAM3D_CASES])
def test_sam3d(dev, shape, nj, D, stream):
    h = volume(shape, nj)
    pose, vis, _ = oracle_reception.pose_regression_3d(ops_np, h, nj, D)
    got = run_sam3d(dev, dev.view(dev.put(h)), shape[0], nj, D, stream)
    close(got[0], pose, 3e-6)
    close(got[1], vis, 3e-6)


PROB3D_SHAPE, PROB3D_NJ, PROB3D_D = (3, 16, 16, 160), 20, 8


def test_sam3d_prob_export_into_slice(dev):
    """The merge model's head (vis_scale 2, action.py:291-295) exporting channel_softmax_2d(hxy) into channels
    [3, 3 + nj) of a wider buffer."""
    n, hh, ww, c = PROB3D_SHAPE
    h = volume(PROB3D_SHAPE, PROB3D_NJ)
    pose, _, hxy = oracle_reception.pose_regression_3d(ops_np, h, PROB3D_NJ, PROB3D_D)
    h5 = h.reshape(n, hh, ww, PROB3D_D, PROB3D_NJ)
    vis = 1.0 / (1.0 + np.exp(-2.0 * (h5.mean(3).max((1, 2)) + h5.mean((1, 2)).max(1))))[..., None]
    prob = Out(dev, (n, hh, ww, PROB3D_NJ), 3, PROB3D_NJ + 8)
    got = run_sam3d(dev, dev.view(dev.put(h)), n, PROB3D_NJ, PROB3D_D, 1, 2.0, prob)
    close(got[0], pose, 3e-6)
    close(got[1], vis, 3e-6)
    close(prob.get(), ops_np.channel_softmax_2d(hxy), 3e-6)


def test_head3d_paths(dev):
    """Each 3-D head case above reaches the kernel its test is about; the probability export stays staged."""
    for shape, nj, D, stream, kernel in SAM3D_CASES:
        hv = dev.view(dev.put(volume(shape, nj)))
        names = launched(dev, lambda: run_sam3d(dev, hv, shape[0], nj, D, stream))
        assert [s for s in names if 'softargmax3d' in s or 'sam3d' in s] == [s for s in names if kernel in s], names
        assert any(kernel in s for s in names), names
    n, hh, ww, _ = PROB3D_SHAPE
    hv = dev.view(dev.put(volume(PROB3D_SHAPE, PROB3D_NJ)))
    prob = Out(dev, (n, hh, ww, PROB3D_NJ), 3, PROB3D_NJ + 8)
    names = launched(dev, lambda: run_sam3d(dev, hv, n, PROB3D_NJ, PROB3D_D, 1, 2.0, prob))
    assert any('softargmax3d_kernel' in s for s in names) and not any('sam3d_stream' in s for s in names), names


@pytest.mark.parametrize('views', [False, True])
def test_kron_pool_limits(dev, views):
    """nj = 32 (KR_MAXJ), F = 300 (not a multiple of the 128-feature CTA), P = 150 (not a multiple of the 64-pixel
    chunk); views: both operands are channel slices."""
    rng = _rng('kron', views)
    n, hh, ww, nj, f = 3, 10, 15, 32, 300
    p = ops_np.channel_softmax_2d(rng.standard_normal((n, hh, ww, nj)) * 2)
    z = rng.standard_normal((n, hh, ww, f))
    ref = np.einsum('nhwj,nhwf->njf', p, z)
    pv = sliced(dev, p, 2, nj + 5) if views else dev.view(dev.put(p))
    zv = sliced(dev, z, 5, f + 7) if views else dev.view(dev.put(z))
    out = dev.empty(n, nj, f)
    dev.call('dh_kron_pool_f32', C.byref(pv), C.byref(zv), out.data_ptr())
    close(out.cpu().numpy(), ref, 1e-5)


# ------------------------------------------------------------------------------------------------------------------
# memory-bound kernels (elementwise.cu).  Layouts: 'float4' dense with C % 4 == 0; 'slice' input and output channel
# slices, 16-byte aligned (gpu_util.layout_io); 'large' dense with more than two grid-strides of work.
# ------------------------------------------------------------------------------------------------------------------
LAYOUTS = ['float4', 'slice', 'large']


def frames(dev, layout, items_per_frame):
    return loop_batch(dev, items_per_frame) if layout == 'large' else 2


def run_maxmin(dev, x, layout):
    """MaxMinPooling2D((2, 2), same): max + min of every window, in float32"""
    out_shape = (x.shape[0], -(-x.shape[1] // 2), -(-x.shape[2] // 2), x.shape[3])
    xv, out = layout_io(dev, x, out_shape, layout)
    dev.call('dh_maxmin_pool2d_f32', C.byref(xv), C.byref(out.view))
    return out.get()


@pytest.mark.parametrize('layout', LAYOUTS)
def test_maxmin_pool(dev, layout):
    hwc = (9, 11, 16) if layout != 'large' else (18, 22, 64)
    n = frames(dev, layout, -(-hwc[0] // 2) * -(-hwc[1] // 2) * hwc[2] // 4)
    x = _rng('maxmin', layout).standard_normal((n,) + hwc).astype(F32)
    ref = ops_np.maxpool2d(x, (2, 2), None, 'same') + -ops_np.maxpool2d(-x, (2, 2), None, 'same')
    assert ref.dtype == F32
    assert np.array_equal(run_maxmin(dev, x, layout), ref)


def run_upsample_add(dev, a, b, layout):
    """a + UpSampling2D(b), or UpSampling2D(b) when a is None; in the 'slice' layout a is a slice at offset 12"""
    n, hb, wb, c = b.shape
    bv, out = layout_io(dev, b, (n, 2 * hb, 2 * wb, c), layout)
    av = NULLV
    if a is not None:
        av = C.byref(sliced(dev, a, 12, c + 16) if layout == 'slice' else dev.view(dev.put(a)))
    dev.call('dh_upsample2x_add_f32', av, C.byref(bv), C.byref(out.view))
    return out.get()


@pytest.mark.parametrize('layout', LAYOUTS)
@pytest.mark.parametrize('with_a', [True, False])
def test_upsample2x_add(dev, layout, with_a):
    hwc = (4, 5, 16) if layout != 'large' else (16, 16, 64)
    n = frames(dev, layout, 4 * hwc[0] * hwc[1] * hwc[2] // 4)
    rng = _rng('upsample', layout, with_a)
    b = rng.standard_normal((n,) + hwc).astype(F32)
    ref = ops_np.upsample2d(b)
    a = None
    if with_a:
        a = rng.standard_normal(ref.shape).astype(F32)
        ref = a + ref
    assert np.array_equal(run_upsample_add(dev, a, b, layout), ref)


def run_add_n(dev, xs, affine, layout):
    """sum of xs [* scale + shift, ReLU]; in the 'slice' layout input i is the slice at offset 4 * i"""
    c = xs[0].shape[3]
    out = Out(dev, xs[0].shape, 8, c + 12) if layout == 'slice' else Out(dev, xs[0].shape)
    views = (_ffi.dh_view * len(xs))(*[sliced(dev, x, 4 * i, c + 16) if layout == 'slice' else dev.view(dev.put(x))
                                       for i, x in enumerate(xs)])
    sc = sh = None
    if affine:
        sc, sh = dev.put(affine[0]).data_ptr(), dev.put(affine[1]).data_ptr()
    dev.call('dh_add_n_f32', views, len(xs), sc, sh, 1 if affine else 0, C.byref(out.view))
    return out.get()


ADD_CASES = ([(n_in, affine, layout) for layout in ('float4', 'slice') for n_in in (1, 2, 3, 4) for affine in (False, True)] +
             [(4, False, 'large'), (3, True, 'large')])


@pytest.mark.parametrize('n_in,affine,layout', ADD_CASES)
def test_add_n(dev, n_in, affine, layout):
    """Without the affine the kernel's float32 sum ((0 + in0) + in1) + ... is reproduced exactly; with scale, shift
    and ReLU it is compared with the fp64 oracle."""
    rng = _rng('add_n', n_in, affine, layout)
    hwc = (7, 9, 24) if layout != 'large' else (32, 32, 64)
    n = frames(dev, layout, hwc[0] * hwc[1] * hwc[2] // 4)
    xs = [rng.standard_normal((n,) + hwc).astype(F32) for _ in range(n_in)]
    aff = (rng.uniform(0.5, 1.5, hwc[2]), rng.standard_normal(hwc[2])) if affine else None
    got = run_add_n(dev, xs, aff, layout)
    if affine:
        close(got, np.maximum(sum(x.astype(np.float64) for x in xs) * aff[0] + aff[1], 0), 1e-6)
    else:
        ref = np.zeros(xs[0].shape, F32)
        for x in xs:
            ref = ref + x
        assert np.array_equal(got, ref)


# name, input (H, W, C), top, left, output (H, W), views.  'spnet': the pose and visual features of the NTU action
# branch, 17 joints padded to 20 (spnet.py:124-132; 16 frames need no padding), at a batch large enough for two
# grid-strides; 'asym': frames and joints padded unevenly; 'views': the input a channel slice, the output a slice
# of a concat buffer.
PAD_CASES = [('spnet', (16, 17, 192), 0, 1, (16, 20), False), ('asym', (7, 13, 24), 2, 1, (10, 17), False),
             ('views', (7, 13, 24), 1, 3, (9, 18), True)]


@pytest.mark.parametrize('name,hwc,top,left,out_hw,views', PAD_CASES)
def test_zeropad(dev, name, hwc, top, left, out_hw, views):
    n = loop_batch(dev, out_hw[0] * out_hw[1] * hwc[2]) if name == 'spnet' else 3
    x = _rng('pad', name).standard_normal((n,) + hwc).astype(F32)
    ref = ops_np.zeropad2d(x, ((top, out_hw[0] - hwc[0] - top), (left, out_hw[1] - hwc[1] - left)))
    xv = sliced(dev, x, 5, hwc[2] + 16) if views else dev.view(dev.put(x))
    out = Out(dev, ref.shape, 8, hwc[2] + 24) if views else Out(dev, ref.shape)
    dev.call('dh_zeropad2d_f32', C.byref(xv), top, left, C.byref(out.view))
    assert np.array_equal(out.get(), ref)


def test_global_maxmin_softmax_many_channels(dev):
    """C = 600 over the 128 threads of the CTA: each thread owns several channels."""
    x = _rng('gmm').standard_normal((3, 5, 9, 600))
    sm = dev.empty(3, 600)
    dev.call('dh_global_maxmin_softmax_f32', C.byref(dev.view(dev.put(x))), sm.data_ptr())
    close(sm.cpu().numpy(), ops_np.softmax(ops_np.global_max_min_pooling(x)), 1e-6)


def test_mask_mul_large(dev):
    rows, dim = loop_batch(dev, 3), 3
    rng = _rng('mask')
    p, c = rng.standard_normal((rows, dim)).astype(F32), rng.uniform(size=(rows, 1)).astype(F32)
    out = dev.torch.full((rows, dim), float('nan'), device='cuda')
    dev.call('dh_mask_mul_f32', dev.put(p).data_ptr(), dev.put(c).data_ptr(), rows, dim, out.data_ptr())
    assert np.array_equal(out.cpu().numpy(), p * c)


def _pool(dev, layout, c):
    x = _rng('pool', layout, c).standard_normal((2, 9, 11, c))
    xv, out = layout_io(dev, x, (2, 5, 6, c), layout)
    dev.call('dh_maxpool2d_f32', C.byref(xv), 2, 2, 2, 2, 1, C.byref(out.view))


ELT_PATHS = [('maxpool C=13', lambda dev: _pool(dev, 'dense', 13), 'pool_kernel<0, 1>'),
             ('maxpool float4', lambda dev: _pool(dev, 'dense', 16), 'pool_kernel<0, 4>'),
             ('maxpool slice', lambda dev: _pool(dev, 'slice', 16), 'pool_kernel<0, 4>'),
             ('maxmin float4', lambda dev: run_maxmin(dev, np.ones((2, 9, 11, 16), F32), 'float4'), 'pool_kernel<1, 4>'),
             ('maxmin slice', lambda dev: run_maxmin(dev, np.ones((2, 9, 11, 16), F32), 'slice'), 'pool_kernel<1, 4>')]
for _lay in ('float4', 'slice'):
    for _a in (True, False):
        ELT_PATHS.append(('upsample %s a=%d' % (_lay, _a),
                          lambda dev, lay=_lay, a=_a: run_upsample_add(dev, np.ones((2, 8, 10, 16), F32) if a else None,
                                                                       np.ones((2, 4, 5, 16), F32), lay),
                          'upsample2x_add_kernel<4>'))
    for _n in (1, 4):
        for _aff in (False, True):
            ELT_PATHS.append(('add_n %s n=%d affine=%d' % (_lay, _n, _aff),
                              lambda dev, lay=_lay, n=_n, aff=_aff: run_add_n(
                                  dev, [np.ones((2, 7, 9, 24), F32)] * n, (np.ones(24), np.zeros(24)) if aff else None, lay),
                              'add_n_kernel<4>'))


@pytest.mark.parametrize('name,fn,kernel', ELT_PATHS, ids=[p[0] for p in ELT_PATHS])
def test_elementwise_paths(dev, name, fn, kernel):
    """The float4 and slice layouts above reach the 4-wide instantiations; C = 13 the scalar one."""
    names = launched(dev, lambda: fn(dev))
    assert any(kernel in s for s in names), names
