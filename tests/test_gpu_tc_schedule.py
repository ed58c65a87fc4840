"""The persistent tensor-core convolutions (conv_sep.cu, conv_patch.cu, conv_tc.cu) on grids where each CTA runs many
tiles.  CTA (x, y) runs the M-tiles x, x + gx, ... of N part y, and in the patch-staged kernels its two consumer
warpgroups take alternate tiles (ping-pong).  test_gpu_tc.py pins the arithmetic at shapes where a CTA almost never
runs a second tile; here every case is built so that CTAs run several, and it says which part of the schedule it
reaches: the second consumer warpgroup and its hand-off, rings wrapping across tiles (nkb = 1 included), CTAs with
different tile counts, a partial tail tile owned by warpgroup 1, the per-tile BN-prologue masks.

  1. Each case states its kernel and what it covers, and asserts both against the library's own plan of the launch
     (dh_conv2d_plan / dh_sepconv2d_plan) before the kernel runs, so a change of the launch rule fails here instead of
     quietly turning a case back into a single-tile test.  The tile rows (128, or 64 on conv_sep.cu's 64 x 144 tiles)
     come from that plan.
  2. Multi-tile cases of every kernel instantiation against the fp64 oracle, with a per-element error bound:
     conv_sep.cu's 128 x 96 tiles on solo CTAs and 2-CTA pairs, its 64 x 144 tiles with the shared-memory and the
     register epilogue, conv_patch.cu and conv_tc.cu.  Also conv_sep.cu's two geometries against each other, and its
     shared-memory epilogue on channel views.
  3. Every tensor-core layer of the compiled C2 (batch 32), C4 and C5 plans at its production size: the multi-tile run
     must equal runs whose own plans give every CTA a single tile, bit for bit."""
import ctypes as C
import zlib

import numpy as np
import pytest

from deephar_b200 import _ffi, reception, spnet, tc
from deephar_b200.config import ModelConfig, pa16j2d, pa17j3d
from oracle import ops_np

from gpu_util import (EPS, SENT, Z3, Dev, bf16, conv_desc, f32, near_tie, packed_weights, tc_dense_bound,
                      tc_sep_bound)
from test_gpu_tc import TOL1, TOL3, _err

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def dev(cuda):
    return Dev(cuda)


# ----------------------------------------------------------------------------------------------------------------------
# 1. the launch rule
# ----------------------------------------------------------------------------------------------------------------------
# The case shapes below are sized for an H100 SXM's 132 SMs (collection must not touch the device); each case checks
# its claims against the library's plan on the real device before it runs.
SIZING_SMS = 132


def plan_info(dev, fn, args):
    """The library's plan of the launch fn(ctx, *args, stream) under the options set now: dh_conv2d_plan /
    dh_sepconv2d_plan on the same arguments."""
    query = dev.lib.dh_conv2d_plan if fn == 'dh_conv2d_f32' else dev.lib.dh_sepconv2d_plan
    info = _ffi.dh_conv_plan_info()
    _ffi.check(query(dev.ctx.handle, *args, C.byref(info)), fn)
    return info


def tile_schedule(info, m):
    """The tile loop of a persistent kernel on the grid of `info` (a plan of m output pixels): CTA x runs the M-tiles
    x, x + gx, ...; the patch-staged kernels (paths 2, 4) hand a CTA's tiles to their two consumer warpgroups in turn."""
    gx, n_mtiles, bm = info.grid_x, info.n_mtiles, info.bm
    assert n_mtiles == -(-m // bm), 'the plan has %d M-tiles of %d rows for %d pixels' % (n_mtiles, bm, m)
    tiles_mine = [(n_mtiles - x + gx - 1) // gx for x in range(gx)]
    tail = n_mtiles - 1
    return dict(path=info.path, m=m, bm=bm, epi_tma=bool(info.epi_tma), n_mtiles=n_mtiles, gy=info.grid_y,
                bn_cta=info.bn_cta, gx=gx, cluster=bool(info.cluster), nkb=info.n_kblocks, stages=info.stages,
                tiles_mine=tiles_mine, max_tiles=max(tiles_mine), mixed=len(set(tiles_mine)) > 1,
                partial_tail=m % bm != 0, tail_wg=(tail // gx) % 2 if info.path in (2, 4) else 0)


def planned_schedule(dev, fn, args, m, path, claims):
    """The schedule of the launch about to run, checked to be on kernel `path` (1 conv_tc.cu, 2 conv_sep.cu,
    4 conv_patch.cu) and to cover `claims`."""
    info = plan_info(dev, fn, args)
    assert info.path == path, 'the library plans path %d for a case written for path %d' % (info.path, path)
    sch = tile_schedule(info, m)
    check_claims(sch, claims)
    return sch


def check_claims(sch, claims):
    """claims: max_tiles (>=); mixed, nkb, stages, cluster, partial_tail, tail_wg, bm, epi_tma, gy, bn_cta, gx (==)
    -- what the case is meant to reach."""
    for key, want in claims.items():
        got = sch[key]
        ok = got >= want if key == 'max_tiles' else got == want
        assert ok, 'schedule no longer covers %s: %r (wanted %r); %r' % (key, got, want, sch)


# ----------------------------------------------------------------------------------------------------------------------
# 2. multi-tile cases against the fp64 oracle
# ----------------------------------------------------------------------------------------------------------------------
# Error bound per output element: gpu_util's tc_dense_bound / tc_sep_bound at precision 3, carried through the
# epilogue (EPS * (|res0| + |res1| + |ref|)).
# precision 1: the reference is built on the bf16 (round-to-nearest-even) operands, so only the accumulation term
#   remains -- except for an operand a_k that sits so close to a bf16 rounding boundary that its fp32 value on the GPU
#   and its fp64 value here may round to different bf16s (flagged below, near_tie): the reference keeps such an a_k
#   unrounded, and either rounding is within one bf16 half-ulp of it, 2^-8 |a_k w_k|, plus that fp32 error.
def hi_weights(w2d):
    """the bf16 hi half of the packed weights, as (K, Cout) fp64: the B operand at precision 1"""
    hi, _, _, _ = tc.pack_matrix(np.asarray(w2d, np.float32))
    k, cout = w2d.shape
    return (hi.astype(np.uint32) << 16).view(np.float32)[:cout, :k].T.astype(np.float64)


def report_tile(sch, viol):
    """viol[m, c] > 0 where the bound is broken: name the worst tile by its place in the schedule"""
    bm = sch['bm']
    v = viol.reshape(-1, viol.shape[-1])
    row = np.max(v, axis=1)
    t = int(np.argmax(row)) // bm
    y = int(np.argmax(np.max(v[t * bm:(t + 1) * bm], axis=0))) // sch['bn_cta']
    x, ti = t % sch['gx'], t // sch['gx']
    return ('worst tile %d: CTA x = %d, N-part y = %d, ti = %d, warpgroup %d (excess %.3g); %d of %d tiles break the bound'
            % (t, x, y, ti, ti % 2 if sch['path'] in (2, 4) else 0,
               float(row.max()), len({int(i) // bm for i in np.nonzero(row > 0)[0]}), sch['n_mtiles']))


def check(sch, got, ref, bound):
    err = np.abs(got.astype(np.float64) - ref)
    viol = np.where(np.isfinite(err), err - bound, np.inf)
    assert np.all(viol <= 0), report_tile(sch, viol)


def set_opts(dev, **kw):
    for k, v in kw.items():
        _ffi.check(dev.lib.dh_set_option(dev.ctx.handle, k.encode(), int(v)))


DEFAULT_OPTS = dict(share_a=1, sep_tma=1, dense_patch=1, pw_smallk=1)


def run_dense(dev, path, case, claims, opts=()):
    """case: n, h, w, cin, cout, size, strides, fused (pre BN + ReLU, post BN, two residuals), precision"""
    n, h, w, cin, cout, size, strides, fused, precision = case
    rng = np.random.default_rng(zlib.crc32(repr(case).encode()))
    x = f32(rng.standard_normal((n, h, w, cin)))
    wt = f32(rng.standard_normal(size + (cin, cout)) / np.sqrt(size[0] * size[1] * cin))
    pre = post = None
    a, da = x, 0.0
    if fused:
        pre = (f32(rng.uniform(0.5, 1.5, cin)), f32(rng.standard_normal(cin) * 0.3))
        post = (f32(rng.uniform(0.5, 1.5, cout)), f32(rng.standard_normal(cout) * 0.3))
        a = np.maximum(x * pre[0] + pre[1], 0)
        da = 2.0 ** -23 * (np.abs(x * pre[0]) + np.abs(pre[1]))          # the fp32 FMA of the prologue
    k = size[0] * size[1] * cin
    conv = lambda u, v: ops_np.conv2d(u, v, strides, 'same')
    s = conv(np.abs(a), np.abs(wt))
    if precision == 3:
        ref = conv(a, wt)
        q = np.sqrt(conv(a * a, wt * wt))
        bound = tc_dense_bound(q, s, k)
    else:
        wb = hi_weights(wt.reshape(k, cout)).reshape(wt.shape)
        tie = near_tie(a, da) if fused else np.zeros(a.shape, bool)
        ref = conv(np.where(tie, a, bf16(a)), wb)
        bound = Z3 * 2.0 ** -23 * np.sqrt(k / 16) * s + conv((2.0 ** -8 * np.abs(a) + da) * tie, np.abs(wt))
    return _finish_and_run(dev, path, claims, 'dh_conv2d_f32', x, (dev.put(wt).data_ptr(),), wt.reshape(k, cout), size,
                           strides, pre, post, 2 if fused else 0, ref, bound, rng, precision,
                           dict(DEFAULT_OPTS, **dict(opts)))


def _finish_and_run(dev, path, claims, fn, x, wargs, w2d, size, strides, pre, post, n_res, ref, bound, rng, precision,
                    opts, up2x=False, out_view=None):
    res, rviews = [], []
    if post is not None:
        ref = ref * post[0] + post[1]
        bound = bound * np.abs(post[0])
    if n_res:
        r0 = f32(rng.standard_normal(ref.shape))
        rs = [r0]
        if n_res == 2:
            n, ho, wo, c = ref.shape
            r1 = f32(rng.standard_normal((n, ho // 2, wo // 2, c) if up2x else ref.shape))
            rs.append(r1)
        for i, r in enumerate(rs):
            rr = np.repeat(np.repeat(r, 2, axis=1), 2, axis=2) if (up2x and i == 1) else r
            res.append(np.abs(rr))
            ref = ref + rr
            rviews.append(dev.view(dev.put(r)))
    bound = bound + EPS * (np.abs(ref) + sum(res) if res else np.abs(ref))
    d = conv_desc(dev, size, strides, 'same', pre_relu=pre is not None or fn == 'dh_sepconv2d_f32', pre=pre, post=post,
                  res=rviews, precision=precision)
    if up2x:
        d.res_up2x = 2
    pk = packed_weights(dev, w2d)
    if out_view is None:
        out = dev.empty(*ref.shape)
        ov = dev.view(out)
    else:
        out, ov = out_view
    args = (C.byref(dev.view(dev.put(x))),) + tuple(wargs) + (C.byref(pk), C.byref(d), C.byref(ov))
    set_opts(dev, **opts)
    try:
        sch = planned_schedule(dev, fn, args, ref.shape[0] * ref.shape[1] * ref.shape[2], path, claims)
        dev.call(fn, *args)
    finally:
        set_opts(dev, **DEFAULT_OPTS)
    assert dev.lib.dh_last_conv_path(dev.ctx.handle) == path, 'unexpected kernel path'
    got = out.cpu().numpy()
    if out_view is None:
        check(sch, got, ref, bound)
    return got, ref, bound


def run_sep(dev, path, case, claims, opts=()):
    """case: n, h, w, cin, cout, k, mode ('act_bn_res' | 'bn_act' | 'up2x': act_bn + identity and upsampled residual |
    'bn_res2': bn_act + two full-resolution residuals), precision"""
    n, h, w, cin, cout, ks, mode, precision = case
    rng = np.random.default_rng(zlib.crc32(repr(case).encode()))
    x = f32(rng.standard_normal((n, h, w, cin)))
    dw = f32(rng.standard_normal((ks, ks, cin, 1)) / ks)
    pw = f32(rng.standard_normal((1, 1, cin, cout)) / np.sqrt(cin))
    pre = post = None
    if mode in ('bn_act', 'bn_res2'):
        pre = (f32(rng.uniform(0.5, 1.5, cin)), f32(rng.standard_normal(cin) * 0.3))
        a = np.maximum(x * pre[0] + pre[1], 0)
    else:
        post = (f32(rng.uniform(0.5, 1.5, cout)), f32(rng.standard_normal(cout) * 0.3))
        a = np.maximum(x, 0)
    dep = ops_np.depthwise_conv2d(a, dw)
    dabs = ops_np.depthwise_conv2d(np.abs(a), np.abs(dw))          # the fp32 depthwise errs by <= KS^2 2^-24 of this
    s = ops_np.conv2d(dabs, np.abs(pw))
    if precision == 3:
        ref = ops_np.conv2d(dep, pw)
        q = np.sqrt(ops_np.conv2d(dep * dep, pw * pw))
        bound = tc_sep_bound(q, s, cin, ks)
    else:
        pb = hi_weights(pw.reshape(cin, cout)).reshape(pw.shape)
        delta = (ks * ks + 1) * 2.0 ** -24 * dabs
        tie = near_tie(dep, delta)
        ref = ops_np.conv2d(np.where(tie, dep, bf16(dep)), pb)
        bound = Z3 * 2.0 ** -23 * np.sqrt(cin / 16) * s + ops_np.conv2d((2.0 ** -8 * np.abs(dep) + delta) * tie, np.abs(pw))
    n_res = {'act_bn_res': 1, 'bn_act': 0, 'up2x': 2, 'bn_res2': 2}[mode]
    return _finish_and_run(dev, path, claims, 'dh_sepconv2d_f32', x, (dev.put(dw).data_ptr(), dev.put(pw).data_ptr()),
                           pw.reshape(cin, cout), (ks, ks), (1, 1), pre, post, n_res, ref, bound, rng, precision,
                           dict(DEFAULT_OPTS, **dict(opts)), up2x=(mode == 'up2x'))


def frames_for(tiles, h, w, odd=False, bm=128):
    """frames of h x w pixels that make at least `tiles` M-tiles of bm rows (an odd count if asked)"""
    n = -(-tiles * bm // (h * w))
    return n + 1 if odd and n % 2 == 0 else n


# --- conv_sep.cu (path 2): every instantiation KS x TW x BNPRO x LO x SHARE ----------------------------------------------
def _sep_grid():
    out = []
    for i, (ks, tw, bnpro, prec, share) in enumerate(
            (ks, tw, b, p, s) for ks in (3, 5) for tw in (32, 16, 8) for b in (False, True) for p in (3, 1)
            for s in (True, False)):
        cout = (576, 384)[i % 2] if share else (288, 96)[i % 2]          # gy 6 / 4 (even) vs 3 / 1 (odd)
        cin = 32 if i % 3 == 0 else 64                                     # nkb = 1 on every third
        gx = SIZING_SMS // {576: 6, 384: 4, 288: 3, 96: 1}[cout]          # N parts of 96 columns or fewer
        want = 5 if i % 4 == 0 else 3
        # (want - 1) full rounds plus part of one: CTAs with `want` and `want - 1` tiles
        n = frames_for((want - 1) * gx + gx // 2 + 1, tw, tw, odd=(tw == 8))
        claims = dict(bm=128, max_tiles=want, mixed=True, cluster=share, nkb=cin // 32)
        if tw == 8:
            claims['partial_tail'] = True                 # two frames per tile, odd frame count: half-empty tail tile
        out.append(((n, tw, tw, cin, cout, ks, 'bn_act' if bnpro else 'act_bn_res', prec), claims))
    return out


SEP_GRID = _sep_grid()


@pytest.mark.parametrize('case,claims', SEP_GRID, ids=['ks%d-tw%d-%s-p%d-%s' % (c[5], c[2], c[6], c[7], 'share' if cl['cluster'] else 'solo')
                                                       for c, cl in SEP_GRID])
def test_sep_multitile(dev, case, claims):
    run_sep(dev, 2, case, claims)


SEP_SPECIAL = [
    # 5x5, W = 8, odd frame count: the half-empty tail tile is warpgroup 1's (ti = 5 on 132 SMs)
    ((1323, 8, 8, 64, 96, 5, 'bn_act', 3), dict(max_tiles=6, mixed=True, partial_tail=True, tail_wg=1, nkb=2), ()),
    # W = 8, 3x3, three N parts, odd frame count: half-empty tail tile on warpgroup 1 (ti = 3)
    ((279, 8, 8, 96, 288, 3, 'act_bn_res', 3), dict(max_tiles=4, mixed=True, partial_tail=True, tail_wg=1, nkb=3), ()),
    # the hot layer's shape class with share_a = 0 on an even gy: independent CTAs
    ((12, 32, 32, 64, 576, 5, 'act_bn_res', 3), dict(max_tiles=5, mixed=True, cluster=False), (('share_a', 0),)),
    ((12, 32, 32, 64, 576, 5, 'act_bn_res', 1), dict(max_tiles=5, mixed=True, cluster=True), ()),
    # two residuals, the second upsampled 2x (res1_src maps rows across frames on the later tiles)
    ((45, 16, 16, 64, 288, 5, 'up2x', 3), dict(max_tiles=3, mixed=True), ()),
    ((23, 16, 16, 32, 576, 5, 'up2x', 3), dict(max_tiles=3, mixed=True, cluster=True, nkb=1), ()),
]


@pytest.mark.parametrize('case,claims,opts', SEP_SPECIAL)
def test_sep_schedule_edges(dev, case, claims, opts):
    run_sep(dev, 2, case, claims, opts)


# --- conv_sep.cu's 2-CTA pairs at nkb = 4 and 5 ----------------------------------------------------------------------
# K-block g of a pair's common tile sequence is produced by rank g % 2, so with an odd nkb the rank that produces a
# tile's K-block kb alternates from tile to tile, while A stage s is always produced by rank s % 2.  A stage's empty
# barrier counts the consumers of both CTAs only on the CTA that produces it; the other CTA waits only for its own
# consumers before re-arming the stage.  SEP_GRID runs the pairs at nkb = 1 and 2; here every instantiation runs at
# nkb = 4 and 5, one case in three with a half-empty last N part (Cout 528).
def _pair_grid():
    out = []
    for i, (ks, tw, bnpro, prec) in enumerate(
            (ks, tw, b, p) for ks in (3, 5) for tw in (32, 16, 8) for b in (False, True) for p in (3, 1)):
        cin = 32 * (4, 5)[i % 2]                           # nkb = 4, 5
        cout = 528 if i % 3 == 2 else 576                  # six N parts; at 528 the last one is half empty
        gx = SIZING_SMS // 6
        want = 4 if i % 4 == 0 else 3                      # tiles of the busiest CTA
        # (want - 1) full rounds plus part of one: CTAs with `want` and `want - 1` tiles
        n = frames_for((want - 1) * gx + gx // 2 + 1, tw, tw, odd=(tw == 8))
        claims = dict(bm=128, max_tiles=want, mixed=True, cluster=True, gy=6, gx=gx, nkb=cin // 32)
        if tw == 8:
            claims['partial_tail'] = True                  # two frames per tile, odd frame count: half-empty tail tile
        out.append(((n, tw, tw, cin, cout, ks, 'bn_act' if bnpro else 'act_bn_res', prec), claims))
    return out


SEP_PAIRS = _pair_grid()


@pytest.mark.parametrize('case,claims', SEP_PAIRS, ids=['ks%d-tw%d-%s-p%d-nkb%d-n%d' % (
    c[5], c[2], c[6], c[7], c[3] // 32, c[4]) for c, _ in SEP_PAIRS])
def test_sep_pair_multitile(dev, case, claims):
    run_sep(dev, 2, case, claims)


# --- conv_sep.cu's 64 x 144 tiles ------------------------------------------------------------------------------------
# The library tiles a separable layer 64 pixels x 144 output channels, two N parts per cluster pair, when its Cout
# splits into an even number of full 144-column N parts (272-288 or 544-576 columns) and Cin >= 288 (DESIGN §4.1).
# The epilogue is staged in shared memory (residuals loaded by TMA during the mainloop, the tile stored by TMA) when
# every view it touches is TMA-encodable and the layer has no second full-resolution residual; otherwise it runs from
# the registers.  These cases also hold test_gpu_tc.py's per-layer tolerance.
def _tile64_case(shape, want, odd, epi_tma):
    """shape (h, w, cin, cout, ks, mode, precision) on 64-row tiles, with `want` tiles on the busiest CTA and
    want - 1 on others; odd: an odd frame count of 4 x 8 maps (two frames per tile), so the tail tile is half empty"""
    h, w, cin, cout, ks, mode, prec = shape
    gy = 2 if cout < 300 else 4                            # one or two pairs per pixel tile
    gx = SIZING_SMS // gy
    n = frames_for((want - 1) * gx + gx // 2 + 1, h, w, odd=odd, bm=64)
    return ((n, h, w, cin, cout, ks, mode, prec),
            dict(bm=64, epi_tma=epi_tma, cluster=True, gy=gy, bn_cta=144, gx=gx, max_tiles=want, mixed=True,
                 partial_tail=odd))


def _tile64_grid():
    """every instantiation of the 64-row kernel (KS x TW x BN prologue x precision): gy 2 and 4, full and ragged last
    N parts (Cout 280, 560), odd and even nkb (so the rank that produces a tile's K-block alternates from tile to
    tile), no residual or one, on the shared-memory epilogue; then the register epilogue: a BN prologue with two
    full-resolution residuals, the shape of C4's 384 -> 288 layer at 32 x 32"""
    out = []
    for i, (ks, (h, w), bnpro, prec) in enumerate(
            (ks, hw, b, p) for ks in (3, 5) for hw in ((32, 32), (16, 16), (8, 8), (4, 8)) for b in (False, True)
            for p in (3, 1)):
        cout = (288, 576, 280, 560)[i % 4]
        cin = (288, 352, 320)[i % 3]                       # nkb 9, 11, 10
        mode = 'bn_act' if bnpro else 'act_bn_res'
        out.append(_tile64_case((h, w, cin, cout, ks, mode, prec), 4 if i % 4 == 0 else 3, h * w < 64, True))
    for shape, want, odd in [((32, 32, 384, 288, 5, 'bn_res2', 3), 3, False),
                             ((16, 16, 288, 560, 3, 'bn_res2', 1), 4, False),
                             ((8, 8, 352, 576, 5, 'bn_res2', 3), 3, False),
                             ((4, 8, 320, 280, 3, 'bn_res2', 1), 3, True)]:
        out.append(_tile64_case(shape, want, odd, False))
    return out


SEP_TILE64 = _tile64_grid()


@pytest.mark.parametrize('case,claims', SEP_TILE64, ids=['ks%d-%dx%d-%s-p%d-c%d-nkb%d' % (
    c[5], c[1], c[2], c[6], c[7], c[4], c[3] // 32) for c, _ in SEP_TILE64])
def test_sep_tile64_multitile(dev, case, claims):
    got, ref, _ = run_sep(dev, 2, case, claims)
    assert _err(got, ref) <= (TOL3 if case[7] == 3 else TOL1)


# the shared-memory epilogue: the up2x residual at W = 32 and 16 (the library takes an upsampled residual only at
# Wo = 16 or a multiple of 32), ragged last N parts, half-empty tail tiles on 4 x 8 maps, no residual at all (nothing
# to load), and CTAs that run enough tiles that the buffer's barriers wrap many times
SEP_EPI_SMEM = [_tile64_case(shape, want, odd, True) for shape, want, odd in [
    ((32, 32, 288, 288, 5, 'up2x', 3), 3, False),
    ((16, 16, 288, 576, 3, 'up2x', 3), 3, False),
    ((16, 16, 320, 560, 5, 'up2x', 1), 3, False),
    ((8, 8, 320, 560, 5, 'act_bn_res', 1), 3, False),
    ((4, 8, 288, 280, 5, 'bn_act', 3), 3, True),
    ((4, 8, 352, 576, 3, 'act_bn_res', 3), 4, True),
    ((16, 16, 288, 288, 5, 'act_bn_res', 3), 12, False),
    ((8, 8, 288, 288, 3, 'bn_act', 1), 10, False),
]]


@pytest.mark.parametrize('case,claims', SEP_EPI_SMEM, ids=['ks%d-%dx%d-%s-p%d-c%d-t%d' % (
    c[5], c[1], c[2], c[6], c[7], c[4], cl['max_tiles']) for c, cl in SEP_EPI_SMEM])
def test_sep_epi_smem_multitile(dev, case, claims):
    got, ref, _ = run_sep(dev, 2, case, claims)
    assert _err(got, ref) <= (TOL3 if case[7] == 3 else TOL1)


# the separable layers of the C2 model (ReLU prologue, BN epilogue): H, W, Cin, Cout, k, residuals (the second one
# upsampled)
C2_SEP_LAYERS = [(32, 32, 576, 576, 5, 0), (32, 32, 576, 576, 5, 2), (32, 32, 384, 576, 3, 1),
                 (16, 16, 288, 288, 5, 1), (16, 16, 288, 288, 5, 2), (8, 8, 288, 288, 5, 1), (16, 16, 288, 576, 5, 1)]


@pytest.mark.parametrize('layer', C2_SEP_LAYERS, ids=['%dx%d-%d-%d-k%d-r%d' % l for l in C2_SEP_LAYERS])
@pytest.mark.parametrize('precision', [3, 1])
def test_sep_tile64_equals_tile128(dev, layer, precision):
    """The two geometries compute each output element with the same operations in the same order (depthwise taps in
    (ky, kx) order, K-blocks and k-steps ascending, the same epilogue), so the 64 x 144 result equals the 128 x 96 one
    (share_a = 0 plans the latter) bit for bit."""
    h, w, cin, cout, k, n_res = layer
    n = 12 if h < 32 else 4
    rng = np.random.default_rng(zlib.crc32(repr((layer, precision)).encode()))
    x = dev.put(rng.standard_normal((n, h, w, cin)))
    dw = dev.put(rng.standard_normal((k, k, cin, 1)) / k)
    pw = rng.standard_normal((1, 1, cin, cout)) / np.sqrt(cin)
    post = (rng.uniform(0.5, 1.5, cout), rng.standard_normal(cout) * 0.3)
    res = [dev.view(dev.put(rng.standard_normal((n, h, w, cout))))] if n_res else []
    if n_res == 2:
        res.append(dev.view(dev.put(rng.standard_normal((n, h // 2, w // 2, cout)))))
    d = conv_desc(dev, (k, k), pre_relu=True, post=post, res=res, precision=precision)
    if n_res == 2:
        d.res_up2x = 2
    pk = packed_weights(dev, pw.reshape(cin, cout))
    pwd = dev.put(pw)
    outs = []
    for share in (1, 0):
        out = dev.empty(n, h, w, cout)
        args = (C.byref(dev.view(x)), dw.data_ptr(), pwd.data_ptr(), C.byref(pk), C.byref(d), C.byref(dev.view(out)))
        set_opts(dev, share_a=share)
        try:
            info = plan_info(dev, 'dh_sepconv2d_f32', args)
            dev.call('dh_sepconv2d_f32', *args)
        finally:
            set_opts(dev, **DEFAULT_OPTS)
        assert info.path == 2 and info.bm == (64 if share else 128), (share, info.path, info.bm)
        assert dev.lib.dh_last_conv_path(dev.ctx.handle) == 2
        outs.append(out.cpu().numpy())
    assert not np.isnan(outs[0]).any()
    assert np.array_equal(outs[0], outs[1]), 'max |64 x 144 - 128 x 96| = %g' % float(np.abs(outs[0] - outs[1]).max())


def _wide(dev, a, c0, ctot):
    """a (n, h, w, c) placed at channels [c0, c0 + c) of a ctot-channel buffer filled with SENT -> (buffer, view)"""
    n, h, w, c = a.shape
    buf = np.full((n, h, w, ctot), SENT, np.float32)
    buf[..., c0:c0 + c] = a
    t = dev.put(buf)
    return t, dev.view(t, c0, c0 + c)


# (out channel offset, out buffer channels), (res0 offset, buffer channels), (res1 offset, buffer channels) or None,
# expected epi_tma.  Cout 288; offsets and pitches in floats: the driver needs multiples of 4.
SLICES = [
    ((32, 352), (4, 296), None, 1),
    ((0, 576), (288, 576), (8, 304), 1),
    ((0, 288), (2, 296), None, 0),             # residual base 8 bytes past a 16-byte boundary
    ((0, 290), (0, 288), None, 0),             # output row pitch 1160 bytes
    ((4, 296), (0, 288), (2, 290), 0),         # up2x residual base and pitch
]


@pytest.mark.parametrize('outs,r0s,r1s,epi', SLICES, ids=['out%d-%d_r%d-%d_%s_epi%d' % (
    o + r + (('u%d-%d' % u) if u else 'nou',) + (e,)) for o, r, u, e in SLICES])
def test_sep_epi_smem_views(dev, outs, r0s, r1s, epi):
    """Residual and output views of the shared-memory epilogue that are channel slices of wider buffers: the result
    equals the one on whole buffers bit for bit, and the channels outside the output slice are untouched.  A view the
    driver cannot encode plans the register epilogue, which computes the same bits.  (The buffer planner never gives a
    layer's output the storage of one of its inputs, so the output never aliases a residual.)"""
    n, h, w, cin, cout, ks = 8, 16, 16, 288, 288, 5
    rng = np.random.default_rng(zlib.crc32(repr((outs, r0s, r1s)).encode()))
    x = dev.put(rng.standard_normal((n, h, w, cin)))
    dw_np = rng.standard_normal((ks, ks, cin, 1)) / ks
    pw_np = rng.standard_normal((1, 1, cin, cout)) / np.sqrt(cin)
    post = (rng.uniform(0.5, 1.5, cout), rng.standard_normal(cout) * 0.3)
    r0 = rng.standard_normal((n, h, w, cout)).astype(np.float32)
    r1 = rng.standard_normal((n, h // 2, w // 2, cout)).astype(np.float32) if r1s else None
    dw, pwd = dev.put(dw_np), dev.put(pw_np)
    pk = packed_weights(dev, pw_np.reshape(cin, cout))

    def run(out_at, r0_at, r1_at):
        res = [_wide(dev, r0, *r0_at)[1]]
        if r1 is not None:
            res.append(_wide(dev, r1, *r1_at)[1])
        d = conv_desc(dev, (ks, ks), pre_relu=True, post=post, res=res, precision=3)
        if r1 is not None:
            d.res_up2x = 2
        ot, ov = _wide(dev, np.full((n, h, w, cout), np.nan, np.float32), *out_at)
        args = (C.byref(dev.view(x)), dw.data_ptr(), pwd.data_ptr(), C.byref(pk), C.byref(d), C.byref(ov))
        info = plan_info(dev, 'dh_sepconv2d_f32', args)
        dev.call('dh_sepconv2d_f32', *args)
        assert dev.lib.dh_last_conv_path(dev.ctx.handle) == 2
        o = ot.cpu().numpy()
        c0 = out_at[0]
        outside = np.concatenate([o[..., :c0], o[..., c0 + cout:]], axis=-1)
        assert np.all(outside == SENT), 'the output view wrote outside its channels'
        return info, o[..., c0:c0 + cout]

    info_w, whole = run((0, cout), (0, cout), (0, cout))
    assert info_w.bm == 64 and info_w.epi_tma == 1
    info, got = run(outs, r0s, r1s)
    assert info.bm == 64 and info.epi_tma == epi, 'planned epi_tma %d' % info.epi_tma
    a = ops_np.depthwise_conv2d(np.maximum(x.cpu().numpy().astype(np.float64), 0), dw_np)
    ref = ops_np.conv2d(a, pw_np) * post[0] + post[1] + r0
    if r1 is not None:
        ref = ref + np.repeat(np.repeat(r1, 2, axis=1), 2, axis=2)
    assert _err(whole, ref) <= TOL3
    assert np.array_equal(got, whole), 'max |sliced - whole| = %g' % float(np.nanmax(np.abs(got - whole)))


# --- conv_patch.cu (path 4) ------------------------------------------------------------------------------------------
NOSMALLK = (('pw_smallk', 0),)
PATCH_CASES = [
    # n, h, w, cin, cout, size, strides, fused, precision
    # 1x1 on virtual rows: nkb = 1 (every K-block a new patch: the ntaps = 1 walk advances two patches per step)
    ((67, 32, 32, 32, 64, (1, 1), (1, 1), False, 3), dict(max_tiles=5, mixed=True, nkb=1)),
    ((67, 32, 32, 32, 64, (1, 1), (1, 1), True, 1), dict(max_tiles=5, mixed=True, nkb=1)),
    # 1x1, 24-pixel frames (8-pixel virtual rows), partial tail tile; nkb = 2 with a half-empty second block
    ((2821, 4, 6, 48, 96, (1, 1), (1, 1), True, 3), dict(max_tiles=4, mixed=True, nkb=2, partial_tail=True)),
    # 1x1 RegMap-like, nkb = 18
    ((34, 32, 32, 576, 48, (1, 1), (1, 1), True, 3), dict(max_tiles=3, mixed=True, nkb=18)),
    # 3x3 at W = 128 (one image row per tile), 5x1 at W = 64, 1x5 at W = 32, with and without the BN-prologue mask
    ((14, 40, 128, 32, 64, (3, 3), (1, 1), False, 3), dict(max_tiles=5, mixed=True, nkb=9)),
    ((14, 40, 128, 32, 64, (3, 3), (1, 1), True, 1), dict(max_tiles=5, mixed=True, nkb=9)),
    ((9, 64, 64, 64, 64, (5, 1), (1, 1), True, 3), dict(max_tiles=3, mixed=True, nkb=10)),
    ((35, 32, 32, 64, 64, (1, 5), (1, 1), True, 3), dict(max_tiles=3, mixed=True, nkb=10)),
    # W = 8: two frames per tile (fn = 2), odd frame count, BN-prologue mask, partial tail tile on warpgroup 1
    ((567, 8, 8, 64, 96, (3, 3), (1, 1), True, 3), dict(max_tiles=3, mixed=True, partial_tail=True, tail_wg=0)),
    ((799, 8, 8, 64, 96, (3, 3), (1, 1), True, 3), dict(max_tiles=4, mixed=True, partial_tail=True, tail_wg=1)),
    # Cin = 48 (half-empty channel block), two N parts
    ((5, 64, 64, 48, 192, (3, 3), (1, 1), True, 3), dict(max_tiles=3, mixed=True, nkb=18)),
]


@pytest.mark.parametrize('case,claims', PATCH_CASES)
def test_patch_multitile(dev, case, claims):
    run_dense(dev, 4, case, claims, NOSMALLK)


def test_patch_channel_views_multitile(dev):
    """input and output are channel slices of wider tensors (ld != C, channel offsets); the columns outside the output
    slice hold sentinels that must survive every tile"""
    n, h, w, cin, cout = 35, 32, 32, 64, 64
    rng = np.random.default_rng(11)
    big = f32(rng.standard_normal((n, h, w, 96)))
    x = big[..., 16:80]
    wt = f32(rng.standard_normal((3, 3, cin, cout)) / 24.0)
    ref = ops_np.conv2d(x, wt)
    s = ops_np.conv2d(np.abs(x), np.abs(wt))
    q = np.sqrt(ops_np.conv2d(x * x, wt * wt))
    bound = tc_dense_bound(q, s, 9 * cin) + EPS * np.abs(ref)
    cat = dev.empty(n, h, w, 88)
    cat.fill_(7.0)
    d = conv_desc(dev, (3, 3))
    pk = packed_weights(dev, wt.reshape(-1, cout))
    xv, ov = dev.view(dev.put(big), 16, 80), dev.view(cat, 8, 72)
    args = (C.byref(xv), dev.put(wt).data_ptr(), C.byref(pk), C.byref(d), C.byref(ov))
    sch = planned_schedule(dev, 'dh_conv2d_f32', args, n * h * w, 4, dict(max_tiles=3, mixed=True, nkb=18))
    dev.call('dh_conv2d_f32', *args)
    assert dev.lib.dh_last_conv_path(dev.ctx.handle) == 4
    got = cat.cpu().numpy()
    check(sch, got[..., 8:72], ref, bound)
    assert np.all(got[..., :8] == 7.0) and np.all(got[..., 72:] == 7.0)


# --- conv_tc.cu (path 1) ---------------------------------------------------------------------------------------------
REG = (('dense_patch', 0), ('pw_smallk', 0))
TC_CASES = [
    # vectorised gather, 3x3, K = 576: 4 stages
    ((67, 32, 32, 64, 96, (3, 3), (1, 1), True, 3), dict(max_tiles=5, mixed=True, nkb=9, stages=4)),
    ((67, 32, 32, 64, 96, (3, 3), (1, 1), True, 1), dict(max_tiles=5, mixed=True, nkb=9, stages=4)),
    # K <= 64: one K-block per tile and a one-stage ring
    ((67, 32, 32, 32, 64, (1, 1), (1, 1), True, 3), dict(max_tiles=5, mixed=True, nkb=1, stages=1)),
    ((67, 32, 32, 32, 64, (1, 1), (1, 1), False, 1), dict(max_tiles=5, mixed=True, nkb=1, stages=1)),
    # scalar gather: Cin 17 (three N parts), Cin 3 (7x7 stride 2), Cin 15 on 8x10 maps (partial tail)
    ((23, 32, 32, 17, 288, (1, 1), (1, 1), True, 3), dict(max_tiles=5, mixed=True, nkb=1, stages=1)),
    ((67, 64, 64, 3, 64, (7, 7), (2, 2), False, 3), dict(max_tiles=5, mixed=True, nkb=3, stages=3)),
    ((213, 8, 10, 15, 160, (3, 3), (1, 1), True, 3), dict(max_tiles=3, mixed=True, nkb=3, partial_tail=True)),
    # the stem 3x3 stride 2
    ((9, 128, 128, 64, 96, (3, 3), (2, 2), False, 3), dict(max_tiles=3, mixed=True, nkb=9, stages=4)),
]


@pytest.mark.parametrize('case,claims', TC_CASES)
def test_tc_dense_multitile(dev, case, claims):
    run_dense(dev, 1, case, claims, REG)


TC_SEP_CASES = [
    # conv_tc.cu's separable register producer (sep_tma = 0): 4x4 maps (8 frames per tile) and 12x16 maps (a height
    # conv_sep.cu does not tile), with and without the 2-CTA A sharing
    ((4232, 4, 4, 64, 64, 5, 'bn_act', 3), dict(max_tiles=5, mixed=True, nkb=1, stages=1, cluster=False), ()),
    ((360, 4, 4, 128, 576, 5, 'act_bn_res', 3), dict(max_tiles=3, mixed=True, nkb=2, cluster=True), ()),
    ((360, 4, 4, 128, 576, 5, 'act_bn_res', 3), dict(max_tiles=3, mixed=True, nkb=2, cluster=False), (('share_a', 0),)),
    ((45, 12, 16, 128, 384, 3, 'act_bn_res', 3), dict(max_tiles=3, mixed=True, cluster=True, partial_tail=True), ()),
    ((45, 12, 16, 128, 384, 3, 'bn_act', 1), dict(max_tiles=3, mixed=True, cluster=True, partial_tail=True), ()),
    ((31, 12, 16, 256, 576, 5, 'up2x', 3), dict(max_tiles=3, mixed=True, nkb=4, stages=4, cluster=True), ()),
]


@pytest.mark.parametrize('case,claims,opts', TC_SEP_CASES)
def test_tc_sep_multitile(dev, case, claims, opts):
    run_sep(dev, 1, case, claims, (('sep_tma', 0),) + tuple(opts))


# ----------------------------------------------------------------------------------------------------------------------
# 3. production layers: the multi-tile run equals single-tile runs bit for bit
# ----------------------------------------------------------------------------------------------------------------------
# A row's arithmetic does not depend on the CTA, tile slot or warpgroup that computes it: the K-block order within a
# tile is fixed, so is each thread's depthwise tap order, and the epilogue is BN FMA, ReLU, +res0, +res1.  So a layer
# run at its production size (CTAs with up to ~31 tiles) must equal the same layer run on groups of frames small
# enough that no CTA runs a second tile -- the single-tile runs are what the oracle tests above and test_gpu_tc.py pin.
C2_KW = dict(num_joints=16, dim=2, num_context_per_joint=2, num_blocks=8, ksize=(5, 5), concat_pose_confidence=False)


def _production_layers():
    frames = 16
    models = {
        'C2': reception.build((256, 256, 3), **C2_KW),
        'C4': spnet.build(ModelConfig((frames, 256, 256, 3), pa16j2d, num_actions=[15], num_pyramids=6,
                                      action_pyramids=[5, 6], num_levels=4, pose_replica=True, num_pose_features=160,
                                      num_visual_features=160)),
        'C5': spnet.build(ModelConfig((frames, 256, 256, 3), pa17j3d, num_actions=[60], num_pyramids=2,
                                      action_pyramids=[1, 2], num_levels=4, num_pose_features=192,
                                      num_visual_features=192)),
    }
    seen = {}
    for name, m in models.items():
        for k in m.plan.kops:
            if k.kind not in ('conv', 'sepconv') or k.attrs.get('pool_out'):
                continue
            a = k.attrs
            h, w, cin = k.ins[0].shape
            key = (k.kind, h, w, cin, k.outs[0].shape[2], tuple(a['size']), tuple(a['strides']), a['padding'],
                   bool(a['pre_relu']), a['pre_bn'] is not None, a['post_bn'] is not None, bool(a['post_relu']),
                   a['n_res'], a['res_up2x'])
            # batch 32 frames (C2; C4 / C5 frame stages: two 16-frame clips); clip-kind layers: 16 clips
            seen.setdefault(key, (name, 32 if k.outs[0].kind == 'frame' else 16))
    return sorted(seen.items(), key=lambda kv: (kv[1][0], kv[0]))


PROD = _production_layers()


def _layer_run(dev, key, fr0, fr1, data, share_a=1):
    kind, h, w, cin, cout, size, strides, padding, pre_relu, pre_bn, post_bn, post_relu, n_res, up2x = key
    torch = dev.torch
    x, wd, wp, pk, pre, post, res = data
    ho, wo = -(-h // strides[0]), -(-w // strides[1])
    d = _ffi.dh_conv_desc()
    d.kh, d.kw = size
    d.sh, d.sw = strides
    d.pad_same = 1 if padding == 'same' else 0
    d.pre_relu, d.post_relu = int(pre_relu), int(post_relu)
    if pre is not None:
        d.pre_scale, d.pre_shift = pre[0].data_ptr(), pre[1].data_ptr()
    if post is not None:
        d.post_scale, d.post_shift = post[0].data_ptr(), post[1].data_ptr()
    d.n_res = n_res
    d.res_up2x = up2x
    for i, r in enumerate(res):
        d.res[i] = dev.view(r[fr0:fr1])
    d.precision = 3
    out = torch.full((fr1 - fr0, ho, wo, cout), float('nan'), dtype=torch.float32, device='cuda')
    xv, ov = dev.view(x[fr0:fr1]), dev.view(out)
    fn = 'dh_conv2d_f32' if kind == 'conv' else 'dh_sepconv2d_f32'
    wargs = (wd.data_ptr(),) if kind == 'conv' else (wd.data_ptr(), wp.data_ptr())
    args = (C.byref(xv),) + wargs + (C.byref(pk), C.byref(d), C.byref(ov))
    set_opts(dev, share_a=share_a)
    try:
        info = plan_info(dev, fn, args)
        dev.call(fn, *args)
    finally:
        set_opts(dev, **DEFAULT_OPTS)
    return out, dev.lib.dh_last_conv_path(dev.ctx.handle), info


@pytest.mark.parametrize('key,where', PROD, ids=['%s-%s-%dx%d-%d-%d-k%dx%d-s%d-%s%s%s-r%d%s' % (
    w[0], k[0], k[1], k[2], k[3], k[4], k[5][0], k[5][1], k[6][0], 'p' if k[9] else '', 'a' if k[8] else '',
    'b' if k[10] else '', k[12], '-up' if k[13] else '') for k, w in PROD])
def test_production_layer_row_invariance(dev, key, where):
    """The layer at its production size equals the same layer run on groups of frames whose own plans give every CTA
    a single tile.  A separable layer on an even gy must also give the same bits with share_a = 0: that turns the
    2-CTA pairs off, and with them the 64 x 144 tiles, so on the layers that take those it also checks that the
    64 x 144 and 128 x 96 geometries agree at production shapes."""
    kind, h, w, cin, cout, size, strides, padding, pre_relu, pre_bn, post_bn, post_relu, n_res, up2x = key
    n = where[1]
    torch = dev.torch
    g = torch.Generator(device='cuda')
    g.manual_seed(zlib.crc32(repr(key).encode()))
    rnd = lambda *shape: torch.randn(*shape, generator=g, device='cuda', dtype=torch.float32)
    ho, wo = -(-h // strides[0]), -(-w // strides[1])
    x = rnd(n, h, w, cin)
    if kind == 'conv':
        wt = rnd(size[0], size[1], cin, cout) / float(np.sqrt(size[0] * size[1] * cin))
        wd, wp = wt, None
        w2d = wt.reshape(-1, cout)
    else:
        wd = rnd(size[0], size[1], cin, 1) / float(size[0])
        wp = rnd(1, 1, cin, cout) / float(np.sqrt(cin))
        w2d = wp.reshape(cin, cout)
    pk = packed_weights(dev, w2d.cpu().numpy())
    pre = (rnd(cin).abs() + 0.5, rnd(cin) * 0.3) if pre_bn else None
    post = (rnd(cout).abs() + 0.5, rnd(cout) * 0.3) if post_bn else None
    res = [rnd(n, ho // 2, wo // 2, cout) if (up2x >> i) & 1 else rnd(n, ho, wo, cout) for i in range(n_res)]
    data = (x, wd, wp, pk, pre, post, res)
    full, path, info = _layer_run(dev, key, 0, n, data)
    assert info.path == path
    if path not in (1, 2, 4):
        pytest.skip('path %d: not a tensor-core kernel' % path)
    sch = tile_schedule(info, n * ho * wo)
    per = ho * wo
    grp = max(1, min(n, sch['gx'] * sch['bm'] // per))          # frames per group: at most gx tiles
    parts = []
    for f in range(0, n, grp):
        out, p, gi = _layer_run(dev, key, f, min(n, f + grp), data)
        assert p == path, 'the single-tile runs took another kernel'
        gsch = tile_schedule(gi, (min(n, f + grp) - f) * per)
        assert gsch['max_tiles'] == 1, 'groups of %d frames make CTAs run a second tile: %r' % (grp, gsch)
        parts.append(out)
    single = torch.cat(parts)
    a, b = full.cpu().numpy(), single.cpu().numpy()
    assert not np.isnan(a).any()
    if not np.array_equal(a, b):
        check(sch, a, b.astype(np.float64), np.zeros(a.shape))
    if path in (1, 2) and kind == 'sepconv' and sch['gy'] % 2 == 0:
        solo, p2, _ = _layer_run(dev, key, 0, n, data, share_a=0)
        assert p2 == path
        s = solo.cpu().numpy()
        if not np.array_equal(a, s):
            check(sch, s, a.astype(np.float64), np.zeros(a.shape))
