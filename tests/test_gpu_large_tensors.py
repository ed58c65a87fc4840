"""The convolution kernels on tensors past 2^31 bytes and 2^31 elements (the cases are in tests/large_cases.py).

Every kernel here treats frames independently, which gives a cheap oracle at any size: a large launch, checked on a few
probe frames against a small one.  Each case

  1. asserts its own claim first: the table's views cross 2^31 bytes / elements where it says (test_large_case_table.py
     recomputes that arithmetic without a GPU), and dh_conv2d_plan / dh_sepconv2d_plan report the path, fallback flag
     and workspace (and, on conv_sep.cu, the tile rows and epilogue) the case was written for;
  2. allocates the whole batch, NaN everywhere except the probe frames (first, the frames holding byte 2^31 and element
     2^31 of each crossing view, last), which hold seeded data; output views start NaN inside SENT channels, with a SENT
     guard band after every output buffer;
  3. runs the large launch, then the same launch on just the probe frames as a small batch, and checks that the probe
     outputs equal the small run's bit for bit (a row's bits do not depend on the CTA, tile slot or batch:
     test_gpu_tc_schedule.py, test_gpu_cuda_core_conv.py), hold no NaN (a read from a wrong frame would bring one), that
     nothing outside the output views was written, and that the small run is within gpu_util's per-element bound of
     the fp64 oracle.

The edge cases put one layer of each class tc_layer_ok judges one frame below and one frame past 2^31 elements of its
input; past the edge the layer stays on its tensor-core kernel.  Separable layers 64 and 128 pixels wide, which
conv_tc.cu's producer cannot tile, are checked to run on the CUDA-core path.  Buffers are freed after each case; a case
that does not fit the free device memory is skipped with the numbers.

    pytest -m gpu tests/test_gpu_large_tensors.py -s      (-s: peak memory and wall time at the end)
"""
import ctypes as C
import time
import zlib

import numpy as np
import pytest

from deephar_b200 import _ffi
from oracle import ops_np

from gpu_util import NULLP, SENT, UNDERFLOW, Dev, conv_desc, epilogue_bound, f32, ffma_dense_bound, ffma_sep_bound, \
    packed_weights, tc_dense_bound, tc_sep_bound
import large_cases as L

pytestmark = pytest.mark.gpu

T0 = time.time()
PATH_NAMES = {0: 'CUDA-core', 1: 'conv_tc.cu', 2: 'conv_sep.cu', 3: 'wide pointwise', 4: 'conv_patch.cu'}
PAST_EDGE = {}      # edge case name -> (path, fallback) the library took


@pytest.fixture(scope='module')
def dev(cuda):
    cuda.cuda.reset_peak_memory_stats()
    return Dev(cuda)


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _affine(rng, c):
    return f32(rng.uniform(0.5, 1.5, c)), f32(rng.standard_normal(c) * 0.3)


class Weights(object):
    """a case's weights and BN affines, on the host and the device"""

    def __init__(self, dev, case):
        rng = np.random.default_rng(zlib.crc32(case.name.encode()))
        kh, kw = case.ks
        if case.sep:
            self.dw = f32(rng.standard_normal((kh, kw, case.cin, 1)) / kh)
            self.w = f32(rng.standard_normal((1, 1, case.cin, case.cout)) / np.sqrt(case.cin))
            self.ptrs = (dev.put(self.dw).data_ptr(), dev.put(self.w).data_ptr())
            k = case.cin
        else:
            self.w = f32(rng.standard_normal((kh, kw, case.cin, case.cout)) / np.sqrt(kh * kw * case.cin))
            self.ptrs = (dev.put(self.w).data_ptr(),)
            k = kh * kw * case.cin
        self.pre = _affine(rng, case.cin) if case.pre else None
        self.post = _affine(rng, case.cout) if case.post else None
        self.packed = packed_weights(dev, self.w.reshape(k, case.cout)) if case.packed else None


def probe_data(case, probes):
    """{name: (len(probes), h, w, c) seeded data} of every input view, one frame per probe"""
    out = {}
    for name, t in case.tensors().items():
        if name == 'x' or name.startswith('res'):
            out[name] = np.stack([f32(np.random.default_rng(zlib.crc32(('%s/%s/%d' % (case.name, name, f)).encode()))
                                      .standard_normal((t.h, t.w, t.c))) for f in probes])
    return out


class Buffers(object):
    """The device buffers of one launch of `case`: inputs NaN except frames `at` (which get `data`), outputs NaN inside
    their views and SENT outside them and in a guard band past the end; the workspace when the path needs one."""

    def __init__(self, dev, case, at, data):
        torch = dev.torch
        self.dev, self.ts, self.bufs, self.views = dev, case.tensors(), {}, {}
        for name, t in self.ts.items():
            if name == 'ws':
                continue
            out = name in ('out', 'pool')
            b = torch.full((t.buffer_elems + L.GUARD,), SENT if out else float('nan'), dtype=torch.float32,
                           device='cuda')
            self.bufs[name] = b
            if out:
                self.body(name)[..., t.c0:t.c0 + t.c].fill_(float('nan'))
            self.views[name] = _ffi.dh_view(b.data_ptr() + 4 * t.c0, t.n, t.h, t.w, t.c, t.ld)
        for name, a in data.items():
            t = self.ts[name]
            for i, f in enumerate(at):
                self.body(name)[f, :, :, t.c0:t.c0 + t.c] = torch.from_numpy(a[i]).cuda()
        self.ws = None
        if 'ws' in self.ts:
            self.ws = torch.empty(case.workspace // 4, dtype=torch.float32, device='cuda')
            dev.ctx.set_workspace(self.ws.data_ptr(), case.workspace)

    def body(self, name):
        t = self.ts[name]
        return self.bufs[name][:t.buffer_elems].view(t.n, t.h, t.w, t.ld)

    def get(self, name, frames):
        t = self.ts[name]
        idx = self.dev.torch.tensor(frames, device='cuda')
        return self.body(name).index_select(0, idx)[..., t.c0:t.c0 + t.c].cpu().numpy()

    def check_untouched(self):
        """nothing outside the output views was written: SENT channels and guard bands"""
        for name in ('out', 'pool'):
            if name not in self.bufs:
                continue
            t, b = self.ts[name], self.bufs[name]
            assert bool((b[t.buffer_elems:] == SENT).all()), '%s: the guard band after the buffer was written' % name
            body = self.body(name)
            if t.c0:
                assert bool((body[..., :t.c0] == SENT).all()), '%s: wrote below the view' % name
            if t.c0 + t.c < t.ld:
                assert bool((body[..., t.c0 + t.c:] == SENT).all()), '%s: wrote above the view' % name

    def release(self):
        if self.ws is not None:
            self.dev.ctx.set_workspace(self.dev.ws.data_ptr(), self.dev.ws.numel() * 4)
        self.bufs = self.views = self.ws = None


def launch(dev, case, wts, bufs, expect=None):
    """plan the case on `bufs`, check the plan with expect(info) before anything runs, then run it; -> the plan's
    dh_conv_plan_info"""
    res = [bufs.views['res%d' % i] for i in range(case.n_res)]
    d = conv_desc(dev, case.ks, case.strides, 'same', pre=wts.pre, post=wts.post, res=res)
    if case.up:
        d.res_up2x = 1 << (case.n_res - 1)
    if 'pool' in bufs.views:
        d.pool_out = bufs.views['pool']
    pk = C.byref(wts.packed) if wts.packed is not None else NULLP
    args = (C.byref(bufs.views['x']),) + wts.ptrs + (pk, C.byref(d), C.byref(bufs.views['out']))
    fn = 'dh_sepconv2d_f32' if case.sep else 'dh_conv2d_f32'
    query = dev.lib.dh_sepconv2d_plan if case.sep else dev.lib.dh_conv2d_plan
    for k, v in case.opts.items():
        _ffi.check(dev.lib.dh_set_option(dev.ctx.handle, k.encode(), int(v)))
    try:
        info = _ffi.dh_conv_plan_info()
        _ffi.check(query(dev.ctx.handle, *args, C.byref(info)), fn)
        if expect is not None:
            expect(info)
        fb0 = dev.lib.dh_fallback_count(dev.ctx.handle, 0)
        dev.call(fn, *args)
        assert dev.lib.dh_last_conv_path(dev.ctx.handle) == info.path
        assert dev.lib.dh_fallback_count(dev.ctx.handle, 0) - fb0 == info.fallback
    finally:
        for k in case.opts:
            _ffi.check(dev.lib.dh_set_option(dev.ctx.handle, k.encode(), 1))
    return info


def expect_plan(case, info):
    got = (info.path, info.fallback, info.workspace_bytes)
    want = (case.path, case.fallback, case.workspace)
    assert got == want, '%s: the library plans path %d, fallback %d, workspace %d; the case was written for %r' % (
        case.name, info.path, info.fallback, info.workspace_bytes, want)
    assert info.bm == case.tile_rows, 'tile rows %d, not %d' % (info.bm, case.tile_rows)
    if case.epi_tma is not None:
        assert info.epi_tma == case.epi_tma, 'epi_tma %d, not %d' % (info.epi_tma, case.epi_tma)


def reference(case, wts, data):
    """(fp64 output, per-element bound) of the probe frames"""
    a = data['x'].astype(np.float64)
    if wts.pre is not None:
        a = a * wts.pre[0] + wts.pre[1]
    tc = case.path in (1, 2, 4)
    if case.sep:
        dep = ops_np.depthwise_conv2d(a, wts.dw)
        ref = ops_np.conv2d(dep, wts.w)
        s = ops_np.conv2d(ops_np.depthwise_conv2d(np.abs(a), np.abs(wts.dw)), np.abs(wts.w))
        bound = (tc_sep_bound(np.sqrt(ops_np.conv2d(dep * dep, wts.w * wts.w)), s, case.cin, case.ks[0]) if tc
                 else ffma_sep_bound(s, case.cin, case.ks[0]))
    else:
        conv = lambda u, v: ops_np.conv2d(u, v, case.strides, 'same')
        k = case.ks[0] * case.ks[1] * case.cin
        ref = conv(a, wts.w)
        s = conv(np.abs(a), np.abs(wts.w))
        bound = tc_dense_bound(np.sqrt(conv(a * a, wts.w * wts.w)), s, k) if tc else ffma_dense_bound(s, k)
    if wts.post is not None:
        ref = ref * wts.post[0] + wts.post[1]
    res = []
    for i in range(case.n_res):
        r = data['res%d' % i].astype(np.float64)
        if r.shape[1] != case.ho:
            r = np.repeat(np.repeat(r, 2, 1), 2, 2)
        res.append(r)
        ref = ref + r
    return ref, epilogue_bound(bound, None if wts.post is None else wts.post[0], ref, [np.abs(r) for r in res]) \
        + UNDERFLOW


def check_claims(case):
    for name, sides in case.cross.items():
        t = case.tensors()[name]
        for side in sides:
            assert t.crosses(side), '%s of %s no longer crosses 2^31 %s' % (name, case.name, side)
    if case.edge == 'below':
        assert case.guard_product() < L.ELEM_EDGE
    if case.edge == 'past':
        assert case.guard_product() >= L.ELEM_EDGE and case.tensors()['x'].last_elem >= L.ELEM_EDGE


@pytest.mark.parametrize('case', L.CASES, ids=lambda c: c.name)
def test_large_conv(dev, case):
    check_claims(case)
    run_case(dev, case)


# conv_tc.cu's separable producer tiles a 128-pixel tile with 4-row strips, so it takes W <= 32; wider separable layers
# with packed weights go to the two-kernel CUDA-core path (they used to be planned on conv_tc.cu, which produced only
# 32 columns of 4 rows per tile)
WIDE_SEP = [L.ConvCase('separable w%d, packed' % w, True, 3, 8, w, 64, 64, (ks, ks), path=0, fallback=1)
            for w, ks in ((64, 3), (128, 5))]


@pytest.mark.parametrize('case', WIDE_SEP, ids=lambda c: c.name)
def test_wide_separable_leaves_conv_tc(dev, case):
    run_case(dev, case)


def run_case(dev, case):
    torch = dev.torch
    free = torch.cuda.mem_get_info()[0]
    need = case.device_bytes() + (1 << 30)
    if free < need:
        pytest.skip('%.1f GB of device memory free, the case needs %.1f GB' % (free / 1e9, need / 1e9))
    probes = case.probes()
    small = case.resized(len(probes))
    keep = len(dev.keep)            # the case's weights and descriptors go too when it ends
    try:
        wts = Weights(dev, case)
        data = probe_data(case, probes)
        big = Buffers(dev, case, probes, data)
        try:
            info = launch(dev, case, wts, big, expect=lambda i: expect_plan(case, i))
            if case.edge == 'past':
                PAST_EDGE[case.name] = (info.path, info.fallback)
            big.check_untouched()
            got = big.get('out', probes)
            pooled = big.get('pool', probes) if 'pool' in big.bufs else None
        finally:
            big.release()
            del big
            torch.cuda.empty_cache()
        sb = Buffers(dev, small, list(range(len(probes))), data)
        try:
            sinfo = launch(dev, small, wts, sb)
            assert sinfo.path == info.path, 'the probe frames alone run on path %d, not %d' % (sinfo.path, info.path)
            sb.check_untouched()
            want = sb.get('out', list(range(len(probes))))
            want_pool = sb.get('pool', list(range(len(probes)))) if pooled is not None else None
        finally:
            sb.release()
    finally:
        del dev.keep[keep:]
    assert not np.isnan(got).any(), 'NaN in probe frame %d' % probes[int(np.argwhere(np.isnan(got))[0][0])]
    for i, f in enumerate(probes):
        assert np.array_equal(_bits(got[i]), _bits(want[i])), 'frame %d of %d differs from the same frame run alone' % (
            f, case.n)
    ref, bound = reference(case, wts, data)
    err = np.abs(want.astype(np.float64) - ref)
    bad = ~(err <= bound)
    assert not bad.any(), '%d elements past the bound; first at %r: got %r, want %r' % (
        int(bad.sum()), tuple(np.argwhere(bad)[0]), float(want[bad][0]), float(ref[bad][0]))
    if pooled is not None:
        n, ho, wo, c = want.shape
        assert np.array_equal(_bits(want_pool), _bits(want.reshape(n, ho // 2, 2, wo // 2, 2, c).max(axis=(2, 4))))
        assert np.array_equal(_bits(pooled), _bits(want_pool)), 'pooled probe frames differ from the small run'


def test_report(dev):
    """peak device memory and wall time of the file so far, and the path each past-the-edge layer took"""
    torch = dev.torch
    for name, (path, fb) in sorted(PAST_EDGE.items()):
        print('%-45s path %d (%s), fallback %d' % (name, path, PATH_NAMES[path], fb))
    print('peak device memory %.2f GB, wall time %.0f s on %s' % (torch.cuda.max_memory_allocated() / 1e9,
                                                                  time.time() - T0, torch.cuda.get_device_name()))
