"""conv_sep.cu's 2-CTA clusters (layers split over an even number of N parts) on grids where each CTA runs several
tiles, with 4 or 5 K-blocks per tile.  K-block g of a pair's common tile sequence is produced by rank g % 2, so with an
odd nkb the rank that produces a tile's K-block kb alternates from tile to tile, while A stage s is always produced by
rank s % 2.  A stage's empty barrier counts the consumers of both CTAs only on the CTA that produces it; the other CTA
waits only for its own consumers before re-arming the stage.  test_gpu_tc_schedule.py covers the pairs at nkb = 1
and 2; here every instantiation (KS 3 / 5 x TW 32 / 16 / 8 x BN prologue x precision 1 / 3) runs at nkb = 4 and 5,
on CTAs with different tile counts (at W = 8 with a half-empty tail tile), one case in three with a half-empty last
N part (Cout 528), against the fp64 oracle and the error bound of test_gpu_tc_schedule.py.  Each case asserts the
plan's cluster and grid before it runs."""
import pytest

import test_gpu_tc_schedule as sched
from gpu_util import Dev

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def dev(cuda):
    return Dev(cuda)


def _cases():
    out = []
    for i, (ks, tw, bnpro, prec) in enumerate(
            (ks, tw, b, p) for ks in (3, 5) for tw in (32, 16, 8) for b in (False, True) for p in (3, 1)):
        cin = 32 * (4, 5)[i % 2]                           # nkb = 4, 5
        cout = 528 if i % 3 == 2 else 576                  # six N parts; at 528 the last one is half empty
        gx = sched.SIZING_SMS // 6                         # checked against the plan below
        want = 4 if i % 4 == 0 else 3                      # tiles of the busiest CTA
        # (want - 1) full rounds plus part of one: CTAs with `want` and `want - 1` tiles
        n = sched.frames_for((want - 1) * gx + gx // 2 + 1, tw, tw, odd=(tw == 8))
        claims = dict(max_tiles=want, mixed=True, cluster=True, nkb=cin // 32)
        if tw == 8:
            claims['partial_tail'] = True                  # two frames per tile, odd frame count: half-empty tail tile
        out.append(((n, tw, tw, cin, cout, ks, 'bn_act' if bnpro else 'act_bn_res', prec), claims))
    return out


CASES = _cases()


@pytest.mark.parametrize('case,claims', CASES, ids=['ks%d-tw%d-%s-p%d-nkb%d-n%d' % (
    c[5], c[2], c[6], c[7], c[3] // 32, c[4]) for c, _ in CASES])
def test_sep_pair_multitile(dev, monkeypatch, case, claims):
    planned = sched.planned_schedule

    def planned_checked(dev_, fn, args, m, path, claims_):
        info = sched.plan_info(dev_, fn, args)
        assert info.cluster == 1 and info.grid_y == 6, 'planned cluster %d, %d N parts' % (info.cluster, info.grid_y)
        assert info.grid_x == min(info.n_mtiles, sched.SIZING_SMS // 6), 'grid_x %d' % info.grid_x
        return planned(dev_, fn, args, m, path, claims_)

    monkeypatch.setattr(sched, 'planned_schedule', planned_checked)
    sched.run_sep(dev, 2, case, claims)
