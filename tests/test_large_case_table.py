"""The case table of tests/test_gpu_large_tensors.py, checked without a GPU: every case's offsets recomputed from its
shapes and views, its crossing claims, where its probe frames land, and its device memory."""
import numpy as np
import pytest

from oracle import ops_np

import large_cases as L


@pytest.mark.parametrize('case', L.CASES, ids=lambda c: c.name)
def test_offsets_from_shapes(case):
    """each view's last element, found from numpy's row-major index of its last (frame, row, column, channel) in the
    buffer, less the view's channel offset; and the buffer ends ld - c0 - c elements after it"""
    for name, t in case.tensors().items():
        last = np.ravel_multi_index((t.n - 1, t.h - 1, t.w - 1, t.c0 + t.c - 1), (t.n, t.h, t.w, t.ld)) - t.c0
        assert t.last_elem == last, name
        assert t.buffer_elems - 1 - (t.c0 + t.last_elem) == t.ld - t.c0 - t.c, name
        assert np.prod((t.n, t.h, t.w, t.ld), dtype=np.int64) == t.buffer_elems
    x, out = case.tensors()['x'], case.tensors()['out']
    assert (x.n, x.h, x.w, x.c) == (case.n, case.h, case.w, case.cin)
    ho = ops_np._out_and_pad(case.h, case.w, case.ks[0], case.ks[1], case.strides[0], case.strides[1], 'same')[:2]
    assert (out.h, out.w, out.c) == tuple(ho) + (case.cout,)


@pytest.mark.parametrize('case', L.CASES, ids=lambda c: c.name)
def test_claims_hold(case):
    """each claimed side is crossed; every view past 2^31 bytes says so (no crossing goes unclaimed); every case
    claims at least one crossing"""
    assert case.cross, 'a case must claim a crossing'
    for name, t in case.tensors().items():
        sides = case.cross.get(name, ())
        for side in ('bytes', 'elements'):
            assert t.crosses(side) == (side in sides), (name, side, t.last_byte)


@pytest.mark.parametrize('case', L.CASES, ids=lambda c: c.name)
def test_probes_land_mid_row_and_mid_tile(case):
    """byte 2^31 of each crossing view lies in an interior probe frame, neither at a row's first or last pixel nor at a
    tile's first or last row (the tiles of the launch's kernel, over the output pixels that read or write it); element
    2^31 lies in a probe frame; first and last frames are probes"""
    probes = case.probes()
    assert probes[0] == 0 and probes[-1] == case.n - 1
    assert len(probes) >= 3
    for name, sides in case.cross.items():
        t = case.tensors()[name]
        if 'bytes' in sides:
            f, y, x, m, ch = t.locate(L.BYTE_EDGE // 4)
            assert f in probes and 0 < f < case.n - 1, (name, f)
            assert 0 < x < t.w - 1, '%s: byte 2^31 at column %d of %d' % (name, x, t.w)
            slot = case.output_pixel(name, f, y, x) % case.tile_rows     # in the tiles of the launch's kernel
            assert 0 < slot < case.tile_rows - 1, '%s: byte 2^31 feeds row %d of a %d-row tile' % (
                name, slot, case.tile_rows)
            assert 4 * (f * t.frame_elems) < L.BYTE_EDGE <= 4 * ((f + 1) * t.frame_elems)
        if 'elements' in sides:
            f = t.locate(L.ELEM_EDGE)[0]
            assert f in probes and f < case.n
            assert f * t.frame_elems <= L.ELEM_EDGE < (f + 1) * t.frame_elems


@pytest.mark.parametrize('case', L.EDGE_CASES, ids=lambda c: c.name)
def test_edge_cases_straddle_the_product(case):
    """below: N * H * W * ldx < 2^31 and one more frame reaches it; past: the product is 2^31 or more and the last
    input element read lies past element 2^31"""
    frame = case.h * case.w * case.x_lay[1]
    if case.edge == 'below':
        assert case.guard_product() < L.ELEM_EDGE <= case.guard_product() + frame
    else:
        assert case.guard_product() - frame < L.ELEM_EDGE <= case.guard_product()
        assert case.tensors()['x'].last_elem >= L.ELEM_EDGE


def test_edge_cases_pair_up():
    names = [c.name for c in L.EDGE_CASES]
    assert len(names) == 2 * len(L.EDGE_CLASSES)
    for below, past in zip(L.EDGE_CASES[::2], L.EDGE_CASES[1::2]):
        assert (below.edge, past.edge) == ('below', 'past') and past.n == below.n + 1


@pytest.mark.parametrize('case', L.CASES, ids=lambda c: c.name)
def test_memory(case):
    """a case's buffers fit the file's device-memory budget, and its small probe run fits easily"""
    assert case.device_bytes() <= L.MAX_DEVICE_BYTES
    assert case.resized(len(case.probes())).device_bytes() < 64 << 20


def test_names_unique():
    names = [c.name for c in L.CASES]
    assert len(names) == len(set(names))
