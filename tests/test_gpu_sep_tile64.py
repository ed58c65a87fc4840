"""conv_sep.cu's 64 x 144 tiles: 64 output pixels x 144 output channels per CTA, two N parts per cluster pair, which
the library plans for separable layers whose Cout splits into an even number of full 144-column N parts (272-288 or
544-576 columns) and Cin >= 288 (DESIGN §4.1).

  1. Every instantiation of the 64-row kernel (KS 3 / 5 x TW 32 / 16 / 8 x BN prologue x precision 1 / 3) against the
     fp64 oracle, with test_gpu_tc_schedule.py's per-element bound and test_gpu_tc.py's per-layer tolerance.  The
     cases cycle through 0, 1 and 2 residuals (the second one upsampled 2x), one and two pairs per pixel tile (gy = 2
     and 4), ragged last N parts (Cout 280 and 560), odd and even K-block counts (so the rank that produces a tile's
     K-block alternates from tile to tile), CTAs with different tile counts and enough tiles per CTA that every ring
     wraps.  The 4 x 8 maps (two frames per 64-row tile) run an odd frame count, so the tail tile is half empty.
     Each case asserts the library's plan of the launch (tile rows, cluster, N parts, tiles) before it runs.
  2. The two geometries compute each output element with the same operations in the same order (depthwise taps in
     (ky, kx) order, K-blocks and k-steps ascending, the same epilogue), so on the layers of the C2 model the 64 x 144
     result equals the 128 x 96 one (share_a = 0 plans the latter) bit for bit."""
import ctypes as C
import zlib

import numpy as np
import pytest

import test_gpu_tc_schedule as sched
from deephar_b200 import _ffi
from gpu_util import Dev, conv_desc, packed_weights

pytestmark = pytest.mark.gpu

BM64 = 64
TOL3, TOL1 = 3e-5, 3e-2          # test_gpu_tc.py: max |err| / max(1, max |ref|) at precision 3 / 1


@pytest.fixture(scope='module')
def dev(cuda):
    return Dev(cuda)


def _frames(tiles, h, w, odd=False):
    """frames of h x w pixels that make at least `tiles` 64-row M-tiles (an odd count if asked)"""
    n = -(-tiles * BM64 // (h * w))
    return n + 1 if odd and n % 2 == 0 else n


def _cases():
    out = []
    for i, (ks, hw, bnpro, prec) in enumerate(
            (ks, hw, b, p) for ks in (3, 5) for hw in ((32, 32), (16, 16), (8, 8), (4, 8)) for b in (False, True)
            for p in (3, 1)):
        h, w = hw
        cout = (288, 576, 280, 560)[i % 4]                  # gy 2 / 4, full or ragged last N part
        gy = 2 if cout < 300 else 4
        cin = (288, 352, 320)[i % 3]                        # nkb 9, 11 (odd), 10
        mode = 'bn_act' if bnpro else ('act_bn_res', 'up2x')[(i // 2) % 2]     # 0, 1, 2 residuals
        gx = sched.SIZING_SMS // gy
        want = 4 if i % 4 == 0 else 3                       # tiles of the busiest CTA
        # (want - 1) full rounds plus part of one: CTAs with `want` and `want - 1` tiles
        n = _frames((want - 1) * gx + gx // 2 + 1, h, w, odd=(h * w < BM64))
        out.append(((n, h, w, cin, cout, ks, mode, prec), dict(gy=gy, want=want, partial_tail=h * w < BM64)))
    return out


CASES = _cases()


@pytest.mark.parametrize('case,want', CASES, ids=['ks%d-%dx%d-%s-p%d-c%d-nkb%d' % (
    c[5], c[1], c[2], c[6], c[7], c[4], c[3] // 32) for c, _ in CASES])
def test_sep_tile64_multitile(dev, monkeypatch, case, want):
    planned = sched.planned_schedule

    def planned_checked(dev_, fn, args, m, path, claims_):
        info = sched.plan_info(dev_, fn, args)
        assert info.path == 2 and info.bm == BM64, 'planned path %d, %d-row tiles' % (info.path, info.bm)
        assert info.cluster == 1 and info.grid_y == want['gy'] and info.bn_cta == 144, (
            'planned cluster %d, %d N parts of %d' % (info.cluster, info.grid_y, info.bn_cta))
        assert info.n_mtiles == -(-m // BM64) and info.grid_x == min(info.n_mtiles, sched.SIZING_SMS // want['gy'])
        tiles = [(info.n_mtiles - x + info.grid_x - 1) // info.grid_x for x in range(info.grid_x)]
        assert max(tiles) >= want['want'] and len(set(tiles)) > 1, 'tiles per CTA %r' % sorted(set(tiles))
        assert (m % BM64 != 0) == want['partial_tail'], 'half-empty tail tile: m = %d' % m
        return planned(dev_, fn, args, m, path, claims_)

    monkeypatch.setattr(sched, 'planned_schedule', planned_checked)
    got, ref, _ = sched.run_sep(dev, 2, case, {})
    err = float(np.abs(got.astype(np.float64) - ref).max()) / max(1.0, float(np.abs(ref).max()))
    assert err <= (TOL3 if case[7] == 3 else TOL1), err


# the separable layers of the C2 model (ReLU prologue, BN epilogue): H, W, Cin, Cout, k, residuals (the second one
# upsampled)
C2_LAYERS = [(32, 32, 576, 576, 5, 0), (32, 32, 576, 576, 5, 2), (32, 32, 384, 576, 3, 1), (16, 16, 288, 288, 5, 1),
             (16, 16, 288, 288, 5, 2), (8, 8, 288, 288, 5, 1), (16, 16, 288, 576, 5, 1)]


@pytest.mark.parametrize('layer', C2_LAYERS, ids=['%dx%d-%d-%d-k%d-r%d' % l for l in C2_LAYERS])
@pytest.mark.parametrize('precision', [3, 1])
def test_sep_tile64_equals_tile128(dev, layer, precision):
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
        sched.set_opts(dev, share_a=share)
        try:
            info = sched.plan_info(dev, 'dh_sepconv2d_f32', args)
            dev.call('dh_sepconv2d_f32', *args)
        finally:
            sched.set_opts(dev, **sched.DEFAULT_OPTS)
        assert info.path == 2 and info.bm == (BM64 if share else 128), (share, info.path, info.bm)
        assert dev.lib.dh_last_conv_path(dev.ctx.handle) == 2
        outs.append(out.cpu().numpy())
    assert not np.isnan(outs[0]).any()
    assert np.array_equal(outs[0], outs[1]), 'max |64 x 144 - 128 x 96| = %g' % float(np.abs(outs[0] - outs[1]).max())
