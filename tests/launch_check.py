"""Every launch of a bound plan checked against its contract on the device -- TEST INFRASTRUCTURE (never imported by
the product).

`LaunchChecker(model).run(x)` binds the model's plan with `Model._bind_plan`, as the product does, but with every
activation slot and the workspace carved out of ONE allocation, each slot between guard bands of at least 64 KB.  The
whole arena starts as a NaN payload no arithmetic produces (ARENA_FILL); then the input goes in and the launches run one
at a time, each followed by two checks.

Write set.  The launch's output regions come from the plan (items x pixels x [c_off, c_off + C) at ld of every output
tensor: a conv's pooled second output, a head's dense outputs and probability export; a concat copy's channel range),
not from the ctypes arguments, so a binding mistake shows too.  Before the launch those regions hold a second payload
(POISON) in the arena and in a device snapshot of it.  After it, no output element may still hold POISON, and once the
outputs are copied into the snapshot the arena must equal it bit for bit: nothing outside the output regions, guards
included, may change -- except the workspace range a two-kernel separable convolution reports it needs
(dh_conv_plan_info.workspace_bytes), its scratch.  A launch's input and output regions must be element-disjoint.  At the end the weight arenas
(`Model._dev`, `Model._dev_packed`) must be bitwise what they were.

Values.  The launch's inputs as the device holds them (frames {0, n/2 + 1, n - 1} of a frame-kind launch, every clip of
a clip-kind one) go through `PlanEmulator.evaluate` in float64, with the fp32 folded BatchNorm vectors the device has,
and the device's outputs must be within the launch's bound:
  conv / sepconv        gpu_util's per-element bounds: bf16x3 on paths 1, 2, 4, fp32 FFMA on paths 0, 3, plus the
                        absolute terms of results and split operands below the normal range; the pooled
                        second output bitwise the 2x2 max of the device's own first output
  one fp32 op or none   (maxpool, upsample, zeropad, copy, maxminpool, scale, mask_mul, upsample_add, two-input add)
                        bitwise the fp32 rounding of the fp64 result
  n-ary add / affine    (n + 1) 2^-24 sum |terms|
  heads, kron, softmax  the tolerances of tests/test_gpu_head_paths.py and tests/test_gpu_ops.py for the same kernels
                        (the softmax's plus 8 L 2^-24 of p for logits of size L);
                        the 2-D context pose scaled by the condition number of its context division, joints above 100
                        left out as tests/test_gpu_reception.py does
A failure names the launch (index, kind, layer, conv path), the item, pixel and channel of the first bad element and how
many elements are bad.  `worst` keeps the largest error / bound ratio per (kind, path).
"""
import numpy as np

from deephar_b200 import _ffi
from deephar_b200.model import _weight_key
from deephar_b200.weights import fold_batchnorm
from oracle import ops_np as O

import gpu_util as G
import kernel_contracts as K
from plan_emulator import PlanEmulator

GUARD = 16384                   # floats (64 KB) of guard band before and after every slot
ARENA_FILL = 0x7F8DEAD1         # signalling NaNs: arithmetic on a NaN returns a quiet one, so neither payload is
POISON = 0x7FA5A5A5             # ever the result of a computation
COND_MAX = 100.0

EXACT = ('maxpool', 'upsample', 'zeropad', 'copy', 'maxminpool', 'scale', 'mask_mul', 'upsample_add')
HEAD_TOL = {            # kind: tolerance of each output, relative to max(1, max |ref|) of that output
    'pose_regression_2d_context': (3e-6, 3e-6),
    'pose_regression_2d': (2e-6, 5e-6),
    'sam2d': (2e-6, 5e-6, 2e-6),
    'pose_regression_3d': (3e-6, 3e-6),
    'pose_regression_3d_ex': (3e-6, 3e-6, 3e-6),
    'kron': (1e-5,),
    'global_maxmin_softmax': (1e-6,),
}


class LaunchError(AssertionError):
    pass


class _DeviceArithmetic(PlanEmulator):
    """PlanEmulator.evaluate on the fp32 folded BatchNorm vectors the device holds (weights.fold_batchnorm)."""

    def __init__(self, model):
        PlanEmulator.__init__(self, model)
        self._folds = {}

    def fold(self, bn):
        if bn['name'] not in self._folds:
            w, hw = bn['weights'], self.model.get_weights()
            sc, sh = fold_batchnorm(hw[w['gamma']] if 'gamma' in w else None, hw[w['beta']], hw[w['mean']], hw[w['var']])
            self._folds[bn['name']] = (np.float64(sc), np.float64(sh))
        return self._folds[bn['name']]


class _Region(object):
    """items x pixels x [c0, c1) at ld of physical slot `phys`"""

    def __init__(self, phys, items, hw, ld, c0, c1):
        self.phys, self.items, self.hw, self.ld, self.c0, self.c1 = phys, items, hw, ld, c0, c1

    def of(self, flat):
        return flat[:self.items * self.hw * self.ld].view(self.items, self.hw, self.ld)[:, :, self.c0:self.c1]

    def extent(self):
        return self.c0, (self.items * self.hw - 1) * self.ld + self.c1


def conv_paths(b):
    return {id(k): int(info.path) for k, info in b.conv_plans}


class LaunchChecker(object):
    def __init__(self, model, values=True):
        self.m = model
        self.values = values
        self.worst = {}             # (kind, path or None) -> largest error / bound
        self.checked = set()        # (kind, path or None) of every launch whose values were checked
        self.launches = 0

    # ---- the guarded binding ---------------------------------------------------------------------------------------
    def _bind(self, n):
        import torch
        m, plan = self.m, self.m.plan
        m._ensure_device_weights()
        probe = m._bind_plan(plan, n)            # the workspace the launches need, and the paths of a plain binding
        ws = probe.workspace.numel()
        self.plain_paths = [int(info.path) for _, info in probe.conv_plans]
        del probe
        torch.cuda.empty_cache()
        sizes = [m._items(kind, n) * fl for (kind, fl) in plan.phys] + [ws]
        offs, off = [], GUARD
        for s in sizes:
            offs.append(off)
            off += -(-s // GUARD) * GUARD + GUARD
        self.arena = torch.empty(off, dtype=torch.float32, device='cuda')
        self.arena.view(torch.int32).fill_(ARENA_FILL)
        self.offs, self.sizes = offs, sizes
        handed = []
        real_empty = torch.empty

        def carve(*shape, **kw):
            numel = int(np.prod(shape[0] if len(shape) == 1 and isinstance(shape[0], (tuple, list)) else shape))
            i = len(handed)
            assert i < len(sizes) and numel == sizes[i], 'unexpected allocation %r in _bind_plan' % (shape,)
            handed.append(i)
            return self.arena[offs[i]:offs[i] + numel]
        torch.empty = carve
        try:
            b = m._bind_plan(plan, n)
        finally:
            torch.empty = real_empty
        assert len(handed) == len(sizes), 'the binding allocated %d buffers, the plan has %d' % (len(handed), len(sizes))
        assert [int(info.path) for _, info in b.conv_plans] == self.plain_paths, 'the guarded binding changed a conv path'
        self.conv_choices = [(k, int(info.path), int(info.fallback)) for k, info in b.conv_plans]
        return b

    def region(self, t, n, c_off=0, channels=None):
        s = self.m.plan.storage[t.id]
        c0 = s.c_off + c_off
        return _Region(s.buf.phys, self.m._items(t.kind, n), t.shape[0] * t.shape[1], s.ld, c0,
                       c0 + (t.shape[2] if channels is None else channels))

    def out_regions(self, k, n):
        if k.kind == 'copy':
            return [(k.outs[0], self.region(k.outs[0], n, k.attrs['c_off'], k.attrs['channels']))]
        return [(t, self.region(t, n)) for t in k.outs]

    def slot(self, flat, phys):
        return flat[self.offs[phys]:self.offs[phys] + self.sizes[phys]]

    # ---- reporting ---------------------------------------------------------------------------------------------------
    def label(self, i, k, path):
        layer = _weight_key(k) if k.kind in ('conv', 'sepconv') else \
            (k.attrs.get('name') if isinstance(k.attrs, dict) and k.attrs.get('name') else repr(k.outs[0]))
        return 'launch %d (%s, layer %s%s)' % (i, k.kind, layer, '' if path is None else ', path %d' % path)

    def where(self, flat_index):
        """arena index -> 'slot s item i pixel p channel c' (with the ld of a launch tensor in that slot) or 'guard'"""
        for phys, (o, sz) in enumerate(zip(self.offs, self.sizes)):
            if o <= flat_index < o + sz:
                r = flat_index - o
                what = 'workspace' if phys == len(self.m.plan.phys) else 'slot %d' % phys
                reg = self._ctx_regions.get(phys)
                if reg is None:
                    return '%s, float %d' % (what, r)
                per = reg.hw * reg.ld
                return '%s item %d pixel %d channel %d' % (what, r // per, (r % per) // reg.ld, r % reg.ld)
        before = [o for o in self.offs if o > flat_index]
        return 'guard band (float %d of the arena, %d before the next slot)' % (
            flat_index, (before[0] - flat_index) if before else -1)

    # ---- one launch ----------------------------------------------------------------------------------------------------
    def _fill(self, regs, value):
        import torch
        for _, r in regs:
            for flat in (self.arena, self.snap):
                r.of(self.slot(flat, r.phys).view(torch.int32)).fill_(value)

    def _disjoint(self, k, n, regs, what):
        import torch
        for t in k.ins:
            ri = self.region(t, n)
            for _, ro in regs:
                if ro.phys != ri.phys:
                    continue
                (a0, a1), (b0, b1) = ri.extent(), ro.extent()
                if a1 <= b0 or b1 <= a0:
                    continue
                mark = torch.zeros(self.sizes[ri.phys], dtype=torch.bool, device=self.arena.device)
                ro.of(mark).fill_(True)
                hit = int(ri.of(mark).sum())
                if hit:
                    raise LaunchError('%s: input %r and output %r share %d elements' % (what, t, ro, hit))

    def _check_writes(self, regs, scratch, what):
        """scratch: floats at the start of the workspace the launch may use (the two-kernel separable convolution keeps
        its depthwise output there); they need not be written, and the rest of the workspace must stay as it was"""
        import torch
        iv = self.arena.view(torch.int32)
        for t, r in regs:
            got = r.of(self.slot(iv, r.phys))
            bad = got == POISON
            nbad = int(bad.sum())
            if nbad:
                i, p, c = [int(v) for v in torch.nonzero(bad)[0]]
                raise LaunchError('%s: output %r left %d elements unwritten; first at item %d pixel %d channel %d' % (
                    what, t, nbad, i, p, r.c0 + c))
            r.of(self.slot(self.snap, r.phys)).copy_(r.of(self.slot(self.arena, r.phys)))
        ws = self.offs[-1]
        self.snap[ws:ws + scratch].copy_(self.arena[ws:ws + scratch])
        sv = self.snap.view(torch.int32)
        chunk = 1 << 28
        for s in range(0, iv.numel(), chunk):
            d = iv[s:s + chunk] != sv[s:s + chunk]
            if bool(d.any()):
                idx = torch.nonzero(d)
                nbad = int(d.sum()) + sum(int((iv[e:e + chunk] != sv[e:e + chunk]).sum())
                                          for e in range(s + chunk, iv.numel(), chunk))
                raise LaunchError('%s: wrote %d elements outside its outputs; first at %s' % (
                    what, nbad, self.where(s + int(idx[0]))))

    def run(self, x):
        """x: (N,H,W,3) frames or (B,T,H,W,3) clips (a torch tensor on the device, or numpy) -> the model's outputs as
        host numpy arrays in Keras shapes.  Raises LaunchError at the first launch that breaks its contract."""
        import torch
        m = self.m
        x = torch.as_tensor(np.asarray(x, np.float32) if isinstance(x, np.ndarray) else x).cuda()
        n = int(np.prod(x.shape[:-3]))
        b = self._bind(n)
        try:
            return self._run(b, x, n)
        finally:
            b.graph = None
            self.arena = self.snap = None
            del b
            torch.cuda.empty_cache()

    def _run(self, b, x, n):
        import torch
        m = self.m
        w0 = m._dev.clone()
        p0 = m._dev_packed.clone() if getattr(m, '_dev_packed', None) is not None and m._uses_tc() else None
        t_in = m.graph.inputs[0]
        self.region(t_in, n).of(self.slot(self.arena, self.m.plan.storage[t_in.id].buf.phys)).copy_(
            x.reshape(n, -1, t_in.shape[2]))
        self.snap = self.arena.clone()
        m._ctx.set_workspace(b.workspace.data_ptr(), b.workspace.numel() * 4)
        stream = torch.cuda.current_stream().cuda_stream
        paths = conv_paths(b)
        scratch = {id(k): -(-int(info.workspace_bytes) // 4) for k, info in b.conv_plans}
        emu = _DeviceArithmetic(m)
        assert len(b.calls) == len(m.plan.kops)
        for i, (k, call) in enumerate(zip(m.plan.kops, b.calls)):
            assert call[0] == k.kind
            path = paths.get(id(k))
            what = self.label(i, k, path)
            regs = self.out_regions(k, n)
            self._ctx_regions = {r.phys: r for _, r in regs}
            self._disjoint(k, n, regs, what)
            self._fill(regs, POISON)
            rc = call[1](*call[2:], stream)
            if rc != 0:
                raise LaunchError('%s: the library refused it (rc %d): %s' % (what, rc, _ffi.lib().dh_last_error().decode()))
            torch.cuda.synchronize()
            self._check_writes(regs, scratch.get(id(k), 0), what)
            if self.values:
                self._check_values(emu, k, n, path, what)
            self.launches += 1
        if not torch.equal(m._dev.view(torch.int32), w0.view(torch.int32)):
            raise LaunchError('the fp32 weight arena changed during the forward')
        if p0 is not None and not torch.equal(m._dev_packed, p0):
            raise LaunchError('the packed bf16 weight arena changed during the forward')
        outs = []
        for t in m.graph.outputs:
            o = m._output_tensor(b, t, n).cpu().numpy().copy()
            outs.append(o.reshape(m._keras_shape(t, m._items(t.kind, n) if t.kind == 'clip' else n)))
        return outs

    # ---- values ------------------------------------------------------------------------------------------------------
    def _read(self, t, n, items, c_off=0, channels=None):
        import torch
        r = self.region(t, n, c_off, channels)
        a = r.of(self.slot(self.arena, r.phys))
        if items is not None:
            a = a.index_select(0, torch.as_tensor(items, device=a.device))
        a = a.cpu().numpy().astype(np.float64)
        return a.reshape((a.shape[0],) + tuple(t.shape[:2]) + (a.shape[-1],))

    def _check_values(self, emu, k, n, path, what):
        kind = k.outs[0].kind
        items = None
        if kind == 'frame':
            items = sorted(set(i for i in (0, n // 2 + 1, n - 1) if i < n))
        pick = lambda t: items if t.kind == kind else None           # noqa: E731
        ins = [self._read(t, n, pick(t)) for t in k.ins]
        if k.kind == 'copy':
            got = [self._read(k.outs[0], n, pick(k.outs[0]), k.attrs['c_off'], k.attrs['channels'])]
        else:
            got = [self._read(t, n, pick(t)) for t in k.outs]
        refs = emu.evaluate(k, ins)
        key = (k.kind, path)
        self.checked.add(key)
        if k.kind in ('conv', 'sepconv'):
            bound = self.conv_bound(emu, k, ins, refs[0], path)
            self._within(what, k.outs[0], got[0], refs[0], bound, key)
            if k.attrs.get('pool_out'):
                dev = np.float32(got[0])
                nn, hh, ww, cc = dev.shape
                pooled = dev.reshape(nn, hh // 2, 2, ww // 2, 2, cc).max(axis=(2, 4))
                self._exact(what + ' pooled output', k.outs[1], np.float32(got[1]), pooled, ('pool_out', path))
        elif k.kind in EXACT or (k.kind == 'add' and len(k.ins) == 2):
            self._exact(what, k.outs[0], np.float32(got[0]), np.float32(refs[0]), key)
        elif k.kind in ('add', 'affine'):
            terms = sum(np.abs(a) for a in ins)
            nops = len(k.ins)
            if k.kind == 'affine' and k.attrs['bn']:
                sc, sh = emu.fold(k.attrs['bn'])
                terms = terms * np.abs(sc) + np.abs(sh)
                nops += 1
            self._within(what, k.outs[0], got[0], refs[0], (nops + 1) * 2.0 ** -24 * terms, key)
        elif k.kind in HEAD_TOL:
            for j, (t, g, r, tol) in enumerate(zip(k.outs, got, refs, HEAD_TOL[k.kind])):
                r = r.reshape(g.shape)
                lim = np.full(r.shape, tol * max(1.0, float(np.abs(r).max())))
                if k.kind == 'pose_regression_2d_context' and j == 0:
                    cond = self.context_cond(k, ins[0]).reshape(g.shape[:-1] + (1,))
                    lim = np.where(cond > COND_MAX, np.inf, np.maximum(lim, 0.2 * lim * cond))
                if k.kind == 'global_maxmin_softmax':
                    lim = lim + self.softmax_logit_bound(ins[0], r)
                self._within('%s output %d' % (what, j), t, g, r, lim, key)
        else:
            raise LaunchError('%s: no value check for this kind' % what)

    @staticmethod
    def context_cond(k, h):
        """(items, nj) condition number of the context head's sum(pc * yc) / sum(pc) (oracle/reception.py)"""
        nj, nc = k.attrs['num_joints'], k.attrs['num_context']
        pc = O.keypoint_confidence(h[..., nj:]).reshape(h.shape[0], nj, nc)
        return np.abs(pc).sum(-1) / np.maximum(np.abs(pc.sum(-1)), 1e-300)

    @staticmethod
    def softmax_logit_bound(x, p):
        """global_maxmin_softmax (elementwise.cu): the logits s_c = max_c + min_c and s_c - max_j s_j are rounded to fp32,
        each off by up to 2^-24 of values up to L = max_c(|max_c| + |min_c|) and 2 L; each probability's exponent is
        then off by up to 4 L 2^-24, and its normalisation by as much again: 8 L 2^-24 of p.  x: (items, H, W, C)"""
        L = (np.abs(x.max(axis=(1, 2))) + np.abs(x.min(axis=(1, 2)))).max(axis=-1)
        return 8 * 2.0 ** -24 * L.reshape((-1,) + (1,) * (p.ndim - 1)) * np.abs(p)

    def conv_bound(self, emu, k, ins, ref, path):
        a = k.attrs
        x = K.prologue(ins[0], emu.fold(a['pre_bn']) if a['pre_bn'] else None, a['pre_relu'])
        st, pad = tuple(a['strides']), a['padding']
        hw = emu.hw
        if k.kind == 'conv':
            w = hw[a['kernel']]
            s = O.conv2d(np.abs(x), np.abs(w), st, pad)
            kk = w.shape[0] * w.shape[1] * w.shape[2]
            if path in (1, 2, 4):
                bound = G.tc_dense_bound(np.sqrt(O.conv2d(x * x, w * w, st, pad)), s, kk)
            else:
                bound = G.ffma_dense_bound(s, kk)
        else:
            dw, pw = hw[a['depthwise']], hw[a['pointwise']]
            dep = O.depthwise_conv2d(x, dw, st, pad)
            s = O.conv2d(O.depthwise_conv2d(np.abs(x), np.abs(dw), st, pad), np.abs(pw), (1, 1), 'valid')
            cin, ks = dw.shape[2], max(dw.shape[0], dw.shape[1])
            if path in (1, 2, 4):
                bound = G.tc_sep_bound(np.sqrt(O.conv2d(dep * dep, pw * pw, (1, 1), 'valid')), s, cin, ks)
            else:
                bound = G.ffma_sep_bound(s, cin, ks)
        # underflow (gpu_util): 2^-150 per fp32 rounding -- one per term on the CUDA cores, fewer on the tensor cores; a
        # separable layer's depthwise roundings reach the result through |pw| -- and on the bf16x3 paths 2^-134 per
        # split A operand, through |w|
        if k.kind == 'conv':
            wsum = np.abs(w).sum(axis=(0, 1, 2))
            floor = G.UNDERFLOW * kk
        else:
            wsum = np.abs(pw).reshape(cin, -1).sum(axis=0)
            floor = G.UNDERFLOW * ((ks * ks + 1) * wsum + cin)
        if path in (1, 2, 4):
            floor = floor + G.SPLIT_FLOOR * wsum
        bound = bound + floor
        res = []
        for i in range(a['n_res']):
            r = ins[1 + i]
            res.append(O.upsample2d(r) if (a.get('res_up2x', 0) >> i) & 1 else r)
        post = emu.fold(a['post_bn'])[0] if a['post_bn'] else None
        return G.epilogue_bound(bound, post, ref, res) + 4 * G.UNDERFLOW

    def _first_bad(self, what, t, bad, detail):
        idx = np.argwhere(bad)[0]
        item, pix, ch = int(idx[0]), int(np.ravel_multi_index(tuple(idx[1:-1]), bad.shape[1:-1])), int(idx[-1])
        raise LaunchError('%s: %d of %d elements of %r out of bound; first at (sampled) item %d pixel %d channel %d: %s'
                          % (what, int(bad.sum()), bad.size, t, item, pix, ch, detail(tuple(idx))))

    def _within(self, what, t, got, ref, bound, key):
        ref = np.asarray(ref, np.float64).reshape(got.shape)
        bound = np.broadcast_to(bound, got.shape)
        err = np.abs(got - ref)
        bad = ~(err <= bound)
        if bad.any():
            self._first_bad(what, t, bad, lambda i: 'got %r, want %r, bound %.3g' % (got[i], ref[i], bound[i]))
        fin = np.isfinite(bound) & (bound > 0)
        ratio = float((err[fin] / bound[fin]).max()) if fin.any() else 0.0
        self.worst[key] = max(self.worst.get(key, 0.0), ratio)

    def _exact(self, what, t, got, ref, key):
        ref = np.asarray(ref, np.float32).reshape(got.shape)
        bad = ~(got == ref)
        if bad.any():
            self._first_bad(what, t, bad, lambda i: 'got %r, want %r exactly' % (got[i], ref[i]))
        self.checked.add(key)
        self.worst.setdefault(key, 0.0)
