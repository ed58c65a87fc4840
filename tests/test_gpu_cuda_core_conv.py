"""The CUDA-core convolution kernels (conv_simt.cu) at their edges and schedules, against the fp64 oracle per element.

  direct stem      conv_smallk_kernel: the 3x3x3 first conv (path 0, not a fallback), Cout 32 and 64
  wide pointwise   conv_pw_smallk_kernel: 1x1, Cin <= 64, Cout >= 128 (path 3), with and without the pooled output
  implicit GEMM    conv_simt_kernel: every other Conv2D without packed weights (path 0, fallback)
  separable        depthwise_simt_kernel into the workspace, then the implicit GEMM (path 0, fallback)

Every case asks dh_conv2d_plan / dh_sepconv2d_plan first and asserts the path, the fallback flag and the workspace the
launch needs; schedule cases read their claim ("every CTA makes two grid-stride passes", "three tiles on the busiest
CTA") from the plan's bm / n_mtiles / grid_x.  Outputs start NaN (or SENT around a channel view) and are held per
element to gpu_util's fp32 FFMA bound plus the epilogue's roundings.  A failure names the frame, pixel, channel, M-tile
and CTA.  Each output of these kernels is computed in an order that does not depend on the tile, the CTA or the
grid-stride pass, so every schedule case also checks that a batch of n frames equals n one-frame calls bit for bit.
In a forward, Model.launches_per_forward counts both kernels of each separable conv on this path.

    pytest -m gpu tests/test_gpu_cuda_core_conv.py
"""
import ctypes as C
import zlib

import numpy as np
import pytest

from deephar_b200 import _ffi
from deephar_b200.compiler import PW_SMALLK_SMEM_MAX, pw_smallk_smem
from oracle import ops_np

from gpu_util import NULLP, UNDERFLOW, Dev, Out, conv_desc, epilogue_bound, f32, ffma_dense_bound, ffma_sep_bound, \
    num_sms, sliced

pytestmark = pytest.mark.gpu

WORST = {}      # kernel -> largest error / bound of the cases that ran


@pytest.fixture(scope='module')
def dev(cuda):
    return Dev(cuda)


def _affine(rng, c, shift):
    return f32(rng.uniform(0.5, 1.5, c)), f32(rng.standard_normal(c) * shift)


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


class Conv(object):
    """One Conv2D (sep = False) or SeparableConv2D call on fp32 data, its device launch and its fp64 reference.
    pre / post: None, 'bn', 'relu' or 'bn_relu'; n_res residuals, the last one half-resolution if up; *_lay: None for a
    dense tensor, or (c0, ld) for the channel slice [c0, c0 + C) of a buffer of ld channels."""

    def __init__(self, name, sep, n, h, w, cin, cout, ks=(3, 3), strides=(1, 1), padding='same', pre=None, post=None,
                 n_res=0, up=False, x_lay=None, out_lay=None, res_lay=None, pool=False, shift=0.3):
        rng = np.random.default_rng(zlib.crc32(name.encode()))
        self.sep, self.ks, self.strides, self.padding = sep, ks, strides, padding
        self.cin, self.cout, self.up, self.pool = cin, cout, up, pool
        self.x_lay, self.out_lay, self.res_lay = x_lay, out_lay, res_lay
        self.x = f32(rng.standard_normal((n, h, w, cin)))
        if sep:
            self.dw = f32(rng.standard_normal(ks + (cin, 1)) / ks[0])
            self.w = f32(rng.standard_normal((1, 1, cin, cout)) / np.sqrt(cin))
        else:
            self.w = f32(rng.standard_normal(ks + (cin, cout)) / np.sqrt(ks[0] * ks[1] * cin))
        self.pre = _affine(rng, cin, shift) if pre in ('bn', 'bn_relu') else None
        self.pre_relu = pre in ('relu', 'bn_relu')
        self.post = _affine(rng, cout, 0.3) if post in ('bn', 'bn_relu') else None
        self.post_relu = post in ('relu', 'bn_relu')
        self.ho, self.wo = ops_np._out_and_pad(h, w, ks[0], ks[1], strides[0], strides[1], padding)[:2]
        self.res = []
        for i in range(n_res):
            half = up and i == n_res - 1
            self.res.append(f32(rng.standard_normal((n, self.ho // (2 if half else 1), self.wo // (2 if half else 1), cout))))

    @property
    def n(self):
        return self.x.shape[0]

    @property
    def m(self):
        return self.n * self.ho * self.wo

    def _place(self, dev, a, lay):
        return dev.view(dev.put(a)) if lay is None else sliced(dev, a, lay[0], lay[1])

    def args(self, dev, frames):
        """(x view, weights, desc, Out, pooled Out or None) of the call on `frames`; the buffers stay in dev.keep"""
        xv = self._place(dev, self.x[frames], self.x_lay)
        res = [self._place(dev, r[frames], self.res_lay) for r in self.res]
        d = conv_desc(dev, self.ks, self.strides, self.padding, self.pre_relu, self.post_relu, self.pre, self.post, res)
        if self.up:
            d.res_up2x = 1 << (len(res) - 1)
        nf = len(frames)
        out = Out(dev, (nf, self.ho, self.wo, self.cout), *(self.out_lay or ()))
        pool = None
        if self.pool:
            pool = Out(dev, (nf, self.ho // 2, self.wo // 2, self.cout))
            d.pool_out = pool.view
        w = (dev.put(self.dw).data_ptr(), dev.put(self.w).data_ptr()) if self.sep else (dev.put(self.w).data_ptr(),)
        return xv, w, d, out, pool

    def plan(self, dev, frames=None):
        frames = list(range(self.n)) if frames is None else frames
        keep = len(dev.keep)
        xv, w, d, out, _ = self.args(dev, frames)
        info = _ffi.dh_conv_plan_info()
        fn = dev.lib.dh_sepconv2d_plan if self.sep else dev.lib.dh_conv2d_plan
        rc = fn(dev.ctx.handle, C.byref(xv), *w, NULLP, C.byref(d), C.byref(out.view), C.byref(info))
        del dev.keep[keep:]
        _ffi.check(rc, 'plan')
        return info

    def launch(self, dev, frames=None):
        """-> (output, pooled output or None) of one call on `frames` (all)"""
        frames = list(range(self.n)) if frames is None else frames
        keep = len(dev.keep)
        xv, w, d, out, pool = self.args(dev, frames)
        dev.call('dh_sepconv2d_f32' if self.sep else 'dh_conv2d_f32', C.byref(xv), *w, NULLP, C.byref(d),
                 C.byref(out.view))
        got = (out.get(), pool.get() if pool else None)
        del dev.keep[keep:]
        return got

    def reference(self):
        """(fp64 result, per-element bound)"""
        a = self.x
        if self.pre is not None:
            a = a * self.pre[0] + self.pre[1]
        if self.pre_relu:
            a = np.maximum(a, 0)
        if self.sep:
            ref = ops_np.separable_conv2d(a, self.dw, self.w, self.strides, self.padding)
            s = ops_np.separable_conv2d(np.abs(a), np.abs(self.dw), np.abs(self.w), self.strides, self.padding)
            bound = ffma_sep_bound(s, self.cin, self.ks[0])
        else:
            ref = ops_np.conv2d(a, self.w, self.strides, self.padding)
            s = ops_np.conv2d(np.abs(a), np.abs(self.w), self.strides, self.padding)
            bound = ffma_dense_bound(s, self.ks[0] * self.ks[1] * self.cin)
        if self.post is not None:
            ref = ref * self.post[0] + self.post[1]
        if self.post_relu:
            ref = np.maximum(ref, 0)
        res = [np.repeat(np.repeat(r, 2, 1), 2, 2) if r.shape[1] != self.ho else r for r in self.res]
        ref = ref + sum(res)
        return ref, epilogue_bound(bound, None if self.post is None else self.post[0], ref, res) + UNDERFLOW


def _within(kernel, got, ref, bound, info, what):
    err = np.abs(got.astype(np.float64) - ref)
    bad = ~(err <= bound)
    if bad.any():
        n, y, x, c = np.argwhere(bad)[0]
        ho, wo = ref.shape[1:3]
        m = (n * ho + y) * wo + x
        tile = m // max(1, info.bm)
        raise AssertionError('%s: %d of %d elements off; first at frame %d pixel (%d, %d) channel %d, M-tile %d of CTA '
                             '(%d, %d): got %r, want %r, bound %.3g' % (
                                 what, int(bad.sum()), bad.size, n, y, x, c, tile, tile % max(1, info.grid_x),
                                 c // max(1, info.bn_cta), float(got[n, y, x, c]), float(ref[n, y, x, c]),
                                 float(bound[n, y, x, c])))
    r = float((err / bound).max())
    WORST[kernel] = max(WORST.get(kernel, 0.0), r)
    return r


def _expect(info, path, fallback, workspace=0):
    assert (info.path, info.fallback, info.workspace_bytes) == (path, fallback, workspace), \
        'plan: path %d, fallback %d, workspace %d' % (info.path, info.fallback, info.workspace_bytes)


def run(dev, kernel, case, path, fallback, per_frame=False):
    """plan, launch and check one case; per_frame: also n one-frame calls, each bit for bit the batch's frame"""
    info = case.plan(dev)
    _expect(info, path, fallback, 4 * case.m * case.cin if case.sep and path == 0 else 0)
    got, pooled = case.launch(dev)
    assert dev.lib.dh_last_conv_path(dev.ctx.handle) == path
    ref, bound = case.reference()
    _within(kernel, got, ref, bound, info, kernel)
    if pooled is not None:
        n, ho, wo, c = got.shape
        want = got.reshape(n, ho // 2, 2, wo // 2, 2, c).max(axis=(2, 4))
        assert np.array_equal(_bits(pooled), _bits(want)), 'pooled output is not the 2x2 max of the first output'
    if per_frame:
        for i in range(case.n):
            one, one_pooled = case.launch(dev, [i])
            assert np.array_equal(_bits(one[0]), _bits(got[i])), 'frame %d alone differs from the batch' % i
            if pooled is not None:
                assert np.array_equal(_bits(one_pooled[0]), _bits(pooled[i])), 'pooled frame %d alone differs' % i
    return info


# ---- direct stem: conv_smallk_kernel<Cout / 8, 3, 3, 3> -----------------------------------------------------------------
STEM = [
    # name, Cout, H, W, stride, padding, post, x layout, out layout
    ('c32 s2 same odd', 32, 33, 31, 2, 'same', 'bn_relu', None, None),
    ('c64 s2 same odd', 64, 31, 33, 2, 'same', 'bn', None, None),
    ('c32 s1 same odd', 32, 17, 19, 1, 'same', 'relu', None, None),
    ('c64 s1 valid', 64, 20, 18, 1, 'valid', None, None, None),
    ('c32 s2 valid', 32, 21, 20, 2, 'valid', None, None, None),
    ('c32 x in 4 channels', 32, 16, 15, 1, 'same', 'bn_relu', (0, 4), None),
    ('c64 x at channel 5 of 8', 64, 15, 16, 2, 'same', 'bn_relu', (5, 8), None),
    ('c32 out at channel 8 of 48', 32, 16, 16, 1, 'same', 'bn', None, (8, 48)),
    ('c64 out at channel 4 of 72', 64, 13, 16, 2, 'same', 'bn_relu', (1, 4), (4, 72)),
]


@pytest.mark.parametrize('case', STEM, ids=[c[0] for c in STEM])
def test_stem(dev, case):
    name, cout, h, w, s, padding, post, xl, ol = case
    c = Conv(name, False, 2, h, w, 3, cout, (3, 3), (s, s), padding, post=post, x_lay=xl, out_lay=ol)
    info = run(dev, 'stem', c, 0, 0)
    assert info.bm == 256 // (cout // 8) and info.bn_cta == cout


@pytest.mark.parametrize('cout', [32, 64])
def test_stem_grid_stride(dev, cout):
    """enough pixels that every CTA of the capped grid makes at least two passes, with a tail pass"""
    frames = 19 if cout == 32 else 10
    c = Conv('stem sched %d' % cout, False, frames, 127, 129, 3, cout, (3, 3), (1, 1), 'same', post='bn_relu')
    info = c.plan(dev)
    assert info.n_mtiles >= 2 * info.grid_x and info.grid_x == 16 * num_sms(dev) and c.m % info.bm != 0, \
        (info.n_mtiles, info.grid_x, c.m)
    run(dev, 'stem', c, 0, 0, per_frame=True)


STEM_OFF = [
    # what breaks the direct kernel's conditions -> the generic implicit GEMM must take the call
    ('out not 16-byte aligned', dict(cout=32, out_lay=(2, 40))),
    ('ldo % 4 != 0', dict(cout=32, out_lay=(0, 33))),
    ('Cout 48', dict(cout=48)),
    ('BN prologue', dict(cout=32, pre='bn')),
    ('residual', dict(cout=64, n_res=1)),
]


@pytest.mark.parametrize('case', STEM_OFF, ids=[c[0] for c in STEM_OFF])
def test_stem_ineligible_goes_to_the_implicit_gemm(dev, case):
    name, kw = case
    kw = dict(kw)
    cout = kw.pop('cout')
    c = Conv('stem off ' + name, False, 2, 17, 16, 3, cout, (3, 3), (2, 2), 'same', post='bn_relu', **kw)
    run(dev, 'gemm', c, 0, 1)


# ---- wide pointwise: conv_pw_smallk_kernel ----------------------------------------------------------------------------------
# the widest Cout (a multiple of 4) whose [Cin][Cout] weights, BN vectors, prologue vectors and 64 x Cin input tile fit
# the kernel's 200 KB of shared memory at Cin 64 (conv_simt.cu, pw_smallk_smem; restated as compiler.pw_smallk_smem)
PW_COUT_MAX64 = max(c for c in range(128, 1024, 4) if pw_smallk_smem(64, c) <= PW_SMALLK_SMEM_MAX)

PW = [
    # name, Cin, Cout, prologue, post, n_res, x layout, residual layout
    ('4->128 no prologue', 4, 128, None, None, 0, None, None),
    ('8->132 bn prologue', 8, 132, 'bn', 'bn', 1, (4, 16), (4, 140)),
    ('60->272 relu prologue', 60, 272, 'relu', 'bn_relu', 2, (4, 68), (8, 284)),
    ('64->576 bn relu prologue', 64, 576, 'bn_relu', 'relu', 2, None, (4, 584)),
    ('48->576 fremap', 48, 576, 'bn_relu', 'bn', 2, (0, 52), (576, 1152)),
    ('64->max fitting Cout', 64, PW_COUT_MAX64, 'bn', None, 1, None, None),
]


@pytest.mark.parametrize('case', PW, ids=[c[0] for c in PW])
def test_wide_pointwise(dev, case):
    name, cin, cout, pre, post, n_res, xl, rl = case
    c = Conv(name, False, 3, 7, 9, cin, cout, (1, 1), pre=pre, post=post, n_res=n_res, x_lay=xl, res_lay=rl,
             out_lay=(4, cout + 8) if n_res == 2 else None)
    info = run(dev, 'pw', c, 3, 0)
    assert (info.bm, info.grid_y, info.bn_cta) == (64, 1, cout)


def test_wide_pointwise_schedule(dev):
    """>= 3 tiles on the busiest CTA, CTAs with unequal tile counts and an M tail in the last tile"""
    c = Conv('pw sched', False, 88, 15, 13, 48, 576, (1, 1), pre='bn_relu', post='bn', n_res=2, res_lay=(4, 584))
    info = c.plan(dev)
    assert info.grid_x == num_sms(dev) and info.n_mtiles > 2 * info.grid_x and info.n_mtiles % info.grid_x != 0 \
        and c.m % 64 != 0, (info.n_mtiles, info.grid_x, c.m)
    run(dev, 'pw', c, 3, 0, per_frame=True)


@pytest.mark.parametrize('frames,h', [(34, 16), (3, 2)])
def test_wide_pointwise_pooled(dev, frames, h):
    """the pooled second output: several tiles per CTA over many frames, and the minimal Ho = 2"""
    c = Conv('pw pool %d %d' % (frames, h), False, frames, h, 32, 48, 576, (1, 1), pre='bn_relu', post='bn', n_res=2,
             res_lay=(4, 584), pool=True)
    info = c.plan(dev)
    if frames > 3:
        assert info.n_mtiles > 2 * info.grid_x and info.n_mtiles % info.grid_x != 0, (info.n_mtiles, info.grid_x)
    run(dev, 'pw', c, 3, 0, per_frame=True)


PW_OFF = [
    ('Cin 68', dict(cin=68)),
    ('Cin 6', dict(cin=6)),
    ('x at channel 1', dict(x_lay=(1, 52))),
    ('Cout 124', dict(cout=124)),
    ('Cout past 200 KB', dict(cin=64, cout=PW_COUT_MAX64 + 4)),
]


@pytest.mark.parametrize('case', PW_OFF, ids=[c[0] for c in PW_OFF])
def test_wide_pointwise_ineligible(dev, case):
    name, kw = case
    kw = dict(dict(cin=48, cout=576), **kw)
    if name == 'Cout past 200 KB':
        assert pw_smallk_smem(64, kw['cout']) > PW_SMALLK_SMEM_MAX
    c = Conv('pw off ' + name, False, 2, 8, 8, kw.pop('cin'), kw.pop('cout'), (1, 1), pre='bn_relu', post='bn',
             n_res=1, **kw)
    run(dev, 'gemm', c, 0, 1)
    # ... and asking it for a pooled output is an error, not a silent second kernel
    c.pool = True
    with pytest.raises(_ffi.DeepharB200Error, match='pool_out'):
        c.plan(dev)


# ---- implicit GEMM: conv_simt_kernel -----------------------------------------------------------------------------------------
GEMM = [
    # name, N, H, W, Cin, Cout, ks, stride, padding, kwargs
    ('K % 16 = 1', 2, 9, 11, 9, 24, (3, 3), 1, 'same', dict(pre='bn_relu', post='bn')),
    ('K % 16 = 15', 2, 10, 9, 7, 40, (3, 3), 1, 'same', dict(pre='relu', post='bn_relu')),
    ('Cout % 64 = 1', 2, 12, 12, 16, 65, (3, 3), 1, 'same', dict(post='bn', n_res=1, res_lay=(3, 70))),
    ('Cout % 64 = 63', 2, 12, 12, 16, 127, (1, 1), 1, 'same', dict(pre='bn', n_res=2)),
    ('Cout 63', 1, 9, 13, 20, 63, (3, 3), 2, 'valid', dict(post='relu')),
    ('M and N blocks', 3, 20, 22, 24, 130, (3, 3), 1, 'same', dict(pre='bn_relu', post='bn', n_res=1)),
    ('1x5', 2, 11, 14, 16, 32, (1, 5), 1, 'same', dict(pre='bn', post='bn')),
    ('5x1', 2, 14, 11, 16, 32, (5, 1), 1, 'same', dict(pre='relu')),
    ('7x7 stride 2', 2, 37, 35, 3, 64, (7, 7), 2, 'same', dict(post='bn_relu')),
    ('bn prologue no relu, views', 2, 12, 10, 20, 36, (3, 3), 1, 'same',
     dict(pre='bn', post='bn', n_res=2, x_lay=(2, 23), res_lay=(1, 40), out_lay=(3, 41))),
    ('concat slice out', 2, 8, 8, 32, 48, (3, 3), 2, 'same', dict(pre='bn_relu', out_lay=(17, 80))),
    ('upsampled residual W 32', 2, 16, 32, 24, 40, (3, 3), 1, 'same', dict(pre='relu', post='bn', n_res=2, up=True)),
    ('upsampled residual W 16', 3, 8, 16, 20, 36, (1, 1), 1, 'same', dict(post='bn_relu', n_res=1, up=True,
                                                                           res_lay=(2, 40))),
]


@pytest.mark.parametrize('case', GEMM, ids=[c[0] for c in GEMM])
def test_implicit_gemm(dev, case):
    name, n, h, w, cin, cout, ks, s, padding, kw = case
    c = Conv(name, False, n, h, w, cin, cout, ks, (s, s), padding, **kw)
    info = run(dev, 'gemm', c, 0, 1, per_frame=True)
    k = ks[0] * ks[1] * cin
    assert (info.bm, info.bn_cta, info.n_kblocks, info.grid_x, info.grid_y) == \
        (128, 64, -(-k // 16), info.n_mtiles, -(-cout // 64))
    if name.startswith('K %'):
        assert k % 16 == int(name.split()[-1])
    if name == 'M and N blocks':
        assert info.n_mtiles >= 3 and info.grid_y == 3


# ---- two-kernel separable: depthwise_simt_kernel + the implicit GEMM --------------------------------------------------------
SEP = [
    # name, N, H, W, Cin, Cout, k, stride, kwargs
    ('k3', 2, 12, 12, 32, 48, 3, 1, dict(pre='relu', post='bn', n_res=1)),
    ('k5', 2, 10, 11, 24, 40, 5, 1, dict(pre='bn_relu', post='bn_relu')),
    ('k7', 2, 9, 9, 16, 20, 7, 1, dict(post='bn')),
    ('k5 stride 2', 2, 15, 14, 24, 32, 5, 2, dict(pre='relu', post='bn')),
    ('k3 stride 2 views', 2, 16, 16, 20, 36, 3, 2,
     dict(pre='bn_relu', post='bn', n_res=2, x_lay=(3, 27), res_lay=(1, 38), out_lay=(5, 44))),
    ('large positive BN shift', 2, 9, 10, 16, 24, 5, 1, dict(pre='bn_relu', shift=5.0)),
    ('upsampled residual', 2, 16, 32, 32, 48, 5, 1, dict(pre='relu', post='bn', n_res=2, up=True)),
]


@pytest.mark.parametrize('case', SEP, ids=[c[0] for c in SEP])
def test_separable(dev, case):
    name, n, h, w, cin, cout, k, s, kw = case
    c = Conv(name, True, n, h, w, cin, cout, (k, k), (s, s), 'same', **kw)
    info = run(dev, 'sep', c, 0, 1, per_frame=True)
    assert (info.bm, info.bn_cta, info.n_kblocks) == (128, 64, -(-cin // 16))


def test_separable_depthwise_grid_stride(dev):
    """M * Cin above the depthwise grid (16 CTAs of 256 threads per SM): its grid-stride loop runs again"""
    c = Conv('sep stride loop', True, 9, 32, 32, 64, 96, (5, 5), pre='bn_relu', post='bn', n_res=1)
    assert c.m * c.cin > num_sms(dev) * 16 * 256
    run(dev, 'sep', c, 0, 1, per_frame=True)


def test_separable_workspace_edge(dev):
    """exactly workspace_bytes runs; one float less is refused, writes nothing and counts nothing"""
    c = Conv('sep workspace', True, 3, 16, 16, 40, 56, (5, 5), pre='bn_relu', post='bn', n_res=1)
    info = c.plan(dev)
    need = info.workspace_bytes
    assert need == 4 * c.m * c.cin
    lib, h = dev.lib, dev.ctx.handle
    ref, bound = c.reference()
    try:
        for nbytes in (need, need - 4):
            ws = dev.torch.empty(nbytes // 4, dtype=dev.torch.float32, device='cuda')
            dev.ctx.set_workspace(ws.data_ptr(), nbytes)
            # a call on path 3 first, so that a refused call which still set dh_last_conv_path would show
            Conv('path 3 first', False, 1, 4, 4, 8, 128, (1, 1)).launch(dev)
            before = (lib.dh_launch_count(h, 0), lib.dh_fallback_count(h, 0), lib.dh_last_conv_path(h))
            assert before[2] == 3
            keep = len(dev.keep)
            xv, w, d, out, _ = c.args(dev, list(range(c.n)))
            rc = lib.dh_sepconv2d_f32(h, C.byref(xv), *w, NULLP, C.byref(d), C.byref(out.view), dev.stream())
            dev.torch.cuda.synchronize()
            got = out.get()
            del dev.keep[keep:]
            after = (lib.dh_launch_count(h, 0), lib.dh_fallback_count(h, 0), lib.dh_last_conv_path(h))
            if nbytes == need:
                assert rc == 0 and after == (before[0] + 2, before[1] + 1, 0)
                _within('sep', got, ref, bound, info, 'exact workspace')
            else:
                assert rc < 0 and b'workspace too small' in lib.dh_last_error()
                assert np.isnan(got).all(), 'a refused call wrote its output'
                assert after == before, 'a refused call moved the counters: %s -> %s' % (before, after)
            del ws
    finally:
        dev.ctx.set_workspace(dev.ws.data_ptr(), dev.ws.numel() * 4)


# ---- the two-kernel separable path in a forward -----------------------------------------------------------------------------
@pytest.mark.parametrize('which', ['C5', 'C2_cuda_cores'])
def test_launches_per_forward_counts_both_separable_kernels(cuda, which):
    """Model.launches_per_forward equals what one forward launches (dh_launch_count), with a separable conv on the
    CUDA-core path counted as two: C5's separable convs on its 2-frame action maps, which no tensor-core kernel takes,
    and every separable conv of C2 with use_tensor_cores = False"""
    from deephar_b200 import reception, spnet
    from deephar_b200.config import ModelConfig, pa17j3d
    from oracle import synth
    if which == 'C5':
        m = spnet.build(ModelConfig((2, 256, 256, 3), pa17j3d, num_actions=[60], num_pyramids=2, action_pyramids=[1, 2],
                                    num_levels=4, num_pose_features=192, num_visual_features=192))
        x = synth.synth_frames(2, seed=3)[None]
    else:
        m = reception.build((256, 256, 3), num_joints=16, dim=2, num_context_per_joint=2, num_blocks=8, ksize=(5, 5),
                            concat_pose_confidence=False)
        m.use_tensor_cores = False
        x = synth.synth_frames(2, seed=3)
    m.init_synthetic_weights(1234)
    m.use_cuda_graph = False
    m.predict(x)
    m._ctx.launch_count(reset=True)
    m.predict(x)
    assert m._ctx.launch_count(reset=True) == m.launches_per_forward(2) > len(m._bind(2).calls)
    m._bound = {}


# ---- the compiler's pool fusion against the library's ---------------------------------------------------------------------
POOL_GRID = [(cin, cout, before, after) for cin, top in ((64, PW_COUT_MAX64), (48, 960)) for cout in (top, top + 4)
             for before, after in ((0, 0), (3, 0), (4, 0), (4, 1))]


@pytest.mark.parametrize('cin,cout,before,after', POOL_GRID)
def test_pool_fusion_matches_the_library(dev, cin, cout, before, after):
    """the compiler fuses MaxPooling2D into the wide 1x1 conv exactly where dh_conv2d_plan takes pool_out for the same
    views (the conv's input at channel `before` of a before + cin + after channel concat), and the model binds"""
    from deephar_b200.model import Model
    from test_compiler_fuzz import _pool_fused, pool_edge_graph
    assert pw_smallk_smem(48, 960) <= PW_SMALLK_SMEM_MAX < pw_smallk_smem(48, 964)
    g = pool_edge_graph(cin, cout, before, after)
    m = Model(g, name=g.name).init_synthetic_weights(3)
    c = Conv('pool grid', False, 2, 32, 32, cin, cout, (1, 1), pre='relu', pool=True,
             x_lay=(before, before + cin + after) if before or after else None)
    try:
        accepted = c.plan(dev).path == 3
    except _ffi.DeepharB200Error as e:
        assert 'pool_out' in str(e)
        accepted = False
    assert _pool_fused(m) == accepted
    b = m._bind(2)
    assert len(b.conv_plans) == sum(1 for k in m.plan.kops if k.kind == 'conv')
    m._bound = {}


def test_report(dev):
    """worst error / bound per kernel over the cases above (printed with -s)"""
    if not WORST:
        pytest.skip('no case ran')
    print('\nworst error / bound: ' + ', '.join('%s %.3f' % kv for kv in sorted(WORST.items())))
    print('peak device memory allocated: %.2f GB' % (dev.torch.cuda.max_memory_allocated() / 1e9))
    assert all(r <= 1.0 for r in WORST.values())
