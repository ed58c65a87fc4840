"""conv_sep.cu's shared-memory epilogue on the 64 x 144 tiles: the residuals of a tile are loaded by TMA into one
fp32 buffer during the mainloop, the consumer warpgroup adds them to its accumulators there, and the tile leaves by
TMA store (DESIGN §4).  The library plans it when the driver can encode every view the epilogue touches (16-byte
aligned base, row pitch a multiple of 16 bytes) and the layer has no second full-resolution residual; every other
64-row layer keeps the register epilogue.

  1. Multi-tile cases against the fp64 oracle with test_gpu_tc_schedule.py's per-element bound: the up2x residual at
     W = 32 and 16 (the library takes an upsampled residual only at Wo = 16 or a multiple of 32), ragged last N parts
     (Cout 280 and 560), half-empty tail tiles on 4 x 8 maps, no residual at all (nothing to load), and CTAs that run
     enough tiles that the buffer's barriers wrap many times.  Each case asserts the library's plan (64-row tiles,
     shared-memory epilogue, tiles per CTA) before it runs.
  2. Residual and output views that are channel slices of wider buffers: the result equals the one on whole buffers
     bit for bit, and the channels outside the output slice are untouched.  A view the driver cannot encode plans the
     register epilogue, which computes the same bits.

The buffer planner (compiler._layout) never gives a layer's output the storage of one of its inputs (a buffer is
free for reuse only after the last op that reads it), so the output never aliases a residual."""
import ctypes as C
import zlib

import numpy as np
import pytest

import test_gpu_tc_schedule as sched
from gpu_util import SENT, Dev, conv_desc, packed_weights
from oracle import ops_np

pytestmark = pytest.mark.gpu

BM64 = 64
TOL3, TOL1 = 3e-5, 3e-2          # test_gpu_tc.py: max |err| / max(1, max |ref|) at precision 3 / 1


@pytest.fixture(scope='module')
def dev(cuda):
    return Dev(cuda)


def _frames(tiles, h, w, odd=False):
    n = -(-tiles * BM64 // (h * w))
    return n + 1 if odd and n % 2 == 0 else n


# (h, w, cin, cout, ks, mode, precision), tiles of the busiest CTA, odd frame count (4 x 8 maps: half-empty tail tile)
_SHAPES = [
    ((32, 32, 288, 288, 5, 'up2x', 3), 3, False),
    ((16, 16, 288, 576, 3, 'up2x', 3), 3, False),
    ((16, 16, 320, 560, 5, 'up2x', 1), 3, False),
    ((8, 8, 320, 560, 5, 'act_bn_res', 1), 3, False),
    ((4, 8, 288, 280, 5, 'bn_act', 3), 3, True),
    ((4, 8, 352, 576, 3, 'act_bn_res', 3), 4, True),
    ((16, 16, 288, 288, 5, 'act_bn_res', 3), 12, False),
    ((8, 8, 288, 288, 3, 'bn_act', 1), 10, False),
]


def _cases():
    out = []
    for (h, w, cin, cout, ks, mode, prec), want, odd in _SHAPES:
        gy = 2 if cout < 300 else 4
        gx = sched.SIZING_SMS // gy
        n = _frames((want - 1) * gx + gx // 2 + 1, h, w, odd=odd)
        out.append(((n, h, w, cin, cout, ks, mode, prec), dict(gy=gy, want=want, partial_tail=odd)))
    return out


CASES = _cases()


@pytest.mark.parametrize('case,want', CASES, ids=['ks%d-%dx%d-%s-p%d-c%d-t%d' % (
    c[5], c[1], c[2], c[6], c[7], c[4], w['want']) for c, w in CASES])
def test_sep_epi_smem_multitile(dev, monkeypatch, case, want):
    planned = sched.planned_schedule

    def planned_checked(dev_, fn, args, m, path, claims_):
        info = sched.plan_info(dev_, fn, args)
        assert info.path == 2 and info.bm == BM64 and info.epi_tma == 1, (
            'planned path %d, %d-row tiles, epi_tma %d' % (info.path, info.bm, info.epi_tma))
        assert info.cluster == 1 and info.grid_y == want['gy'] and info.bn_cta == 144
        tiles = [(info.n_mtiles - x + info.grid_x - 1) // info.grid_x for x in range(info.grid_x)]
        assert max(tiles) >= want['want'], 'tiles per CTA %r' % sorted(set(tiles))
        assert (m % BM64 != 0) == want['partial_tail'], 'half-empty tail tile: m = %d' % m
        return planned(dev_, fn, args, m, path, claims_)

    monkeypatch.setattr(sched, 'planned_schedule', planned_checked)
    got, ref, _ = sched.run_sep(dev, 2, case, {})
    err = float(np.abs(got.astype(np.float64) - ref).max()) / max(1.0, float(np.abs(ref).max()))
    assert err <= (TOL3 if case[7] == 3 else TOL1), err


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
        info = sched.plan_info(dev, 'dh_sepconv2d_f32', args)
        dev.call('dh_sepconv2d_f32', *args)
        assert dev.lib.dh_last_conv_path(dev.ctx.handle) == 2
        o = ot.cpu().numpy()
        c0 = out_at[0]
        outside = np.concatenate([o[..., :c0], o[..., c0 + cout:]], axis=-1)
        assert np.all(outside == SENT), 'the output view wrote outside its channels'
        return info, o[..., c0:c0 + cout]

    info_w, whole = run((0, cout), (0, cout), (0, cout))
    assert info_w.bm == BM64 and info_w.epi_tma == 1
    info, got = run(outs, r0s, r1s)
    assert info.bm == BM64 and info.epi_tma == epi, 'planned epi_tma %d' % info.epi_tma
    a = ops_np.depthwise_conv2d(np.maximum(x.cpu().numpy().astype(np.float64), 0), dw_np)
    ref = ops_np.conv2d(a, pw_np) * post[0] + post[1] + r0
    if r1 is not None:
        ref = ref + np.repeat(np.repeat(r1, 2, axis=1), 2, axis=2)
    err = float(np.abs(whole.astype(np.float64) - ref).max()) / max(1.0, float(np.abs(ref).max()))
    assert err <= TOL3, err
    assert np.array_equal(got, whole), 'max |sliced - whole| = %g' % float(np.nanmax(np.abs(got - whole)))
