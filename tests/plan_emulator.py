"""CPU emulation of a compiled plan -- TEST INFRASTRUCTURE (never imported by the product).

`deephar_b200.compiler.compile_graph` turns a layer graph into a sequence of kernel ops over a planned set of buffers:
BatchNormalization / ReLU folded into conv prologues and epilogues, residual adds (one of them through a 2x upsampling) and
a pooled second output fused into conv kernels, concatenations turned into channel-offset views or copies, soft-max heads
fused into one op, buffers aliased by liveness.  On the GPU that plan is executed by `Model._bind` / `_Bound.issue` through the C
ABI.  Here the SAME plan is executed on the CPU, op by op, on numpy float64 buffers laid out exactly as the plan says
(physical slot, per-item stride, channel offset, leading dimension), each op by the float64 contract
(tests/kernel_contracts.py) of the include/deephar_b200.h entry point the product launches for it.  Slots start NaN-filled,
so a read of memory no launch has written, or a buffer recycled while still live, poisons the outputs.

What this checks without a GPU: the compiler's fusion decisions, operand order, attribute plumbing, which BatchNormalization
folds into which conv, concat / slice / clip views and the liveness-based slot reuse -- for any model, including the
ones recorded from Keras-style code.  What it does not check: the CUDA kernels (the `-m gpu` tests do).
"""
import numpy as np

from oracle import ops_np as O

import kernel_contracts as K


def _bn_fold(hw, bn):
    """(scale, shift) of an inference BatchNormalization in float64 (the product folds the same way and rounds the result
    to fp32 for the device, `weights.fold_batchnorm`; tests/test_plan_emulator.py compares the two)."""
    w = bn['weights']
    scale = 1.0 / np.sqrt(hw[w['var']] + O.EPS_BN)
    if 'gamma' in w:
        scale = scale * hw[w['gamma']]
    return scale, hw[w['beta']] - hw[w['mean']] * scale


# plan ops that are their contract applied to the op's inputs, with no attributes
_ON_THE_INPUTS = {'upsample': K.upsample2x_add, 'kron': K.kron_pool, 'mask_mul': K.mask_mul, 'maxminpool': K.maxmin_pool,
                  'global_maxmin_softmax': K.global_maxmin_softmax}


class PlanEmulator(object):
    def __init__(self, model):
        self.model, self.plan, self.graph = model, model.plan, model.graph
        self.hw = {k: np.asarray(v, np.float64) for k, v in model.get_weights().items()}
        self.launches = 0

    # ---- storage: the plan's own layout -----------------------------------------------------------------------------
    def _items(self, kind):
        return self.n_frames if kind == 'frame' else self.n_frames // self.graph.frames_per_clip

    def _region(self, t):
        s = self.plan.storage[t.id]
        items = self._items(t.kind)
        hw = t.shape[0] * t.shape[1]
        flat = self.slots[s.buf.phys]
        assert items * hw * s.ld <= flat.size, 'tensor %r does not fit its slot' % (t,)
        return flat[:items * hw * s.ld].reshape(items, hw, s.ld), s.c_off

    def get(self, t):
        reg, off = self._region(t)
        a = reg[:, :, off:off + t.shape[2]]
        return a.reshape((a.shape[0],) + tuple(t.shape)).copy()

    def put(self, t, value, c_off=0, channels=None):
        reg, off = self._region(t)
        c = t.shape[2] if channels is None else channels
        value = np.asarray(value, np.float64)
        assert value.size == reg.shape[0] * reg.shape[1] * c, (t, value.shape)
        reg[:, :, off + c_off:off + c_off + c] = value.reshape(reg.shape[0], reg.shape[1], c)

    # ---- ops (include/deephar_b200.h) ---------------------------------------------------------------------------------
    def fold(self, bn):
        """(scale, shift) of a BatchNormalization the plan folds into a launch"""
        return _bn_fold(self.hw, bn)

    def evaluate(self, k, ins):
        """launch k on its inputs `ins` (float64, one (items, H, W, C) array per k.ins) -> one array per output of k, in
        the order of k.outs; a concat copy's is its channel range [attrs c_off, + channels) of k.outs[0]"""
        kd, a = k.kind, k.attrs
        if kd in _ON_THE_INPUTS:
            return [_ON_THE_INPUTS[kd](*ins)]
        if kd in ('conv', 'sepconv'):
            w = self.hw[a['kernel']] if kd == 'conv' else (self.hw[a['depthwise']], self.hw[a['pointwise']])
            pre, post = [self.fold(a[bn]) if a[bn] else None for bn in ('pre_bn', 'post_bn')]
            return K.conv(ins[0], w, tuple(a['strides']), a['padding'], pre, a['pre_relu'], post, a['post_relu'],
                          ins[1:1 + a['n_res']], a.get('res_up2x', 0), a.get('pool_out'))
        if kd == 'maxpool':
            return [K.maxpool(ins[0], tuple(a['pool']), tuple(a['strides']), a['padding'])]
        if kd == 'upsample_add':
            return [K.upsample2x_add(ins[1], ins[0])]
        if kd in ('add', 'affine', 'copy'):
            sc, sh = self.fold(a['bn']) if kd == 'affine' and a['bn'] else (None, None)
            return [K.add_n(ins, sc, sh, kd == 'affine' and a['relu'])]
        if kd == 'scale':
            return [ins[0] * float(a['value'])]
        if kd == 'pose_regression_2d_context':
            return K.softargmax2d_ctx(ins[0], a['num_joints'], a['num_context'], a['alpha'])
        if kd == 'pose_regression_2d':
            return K.softargmax2d(ins[0], 1, 0)[:len(k.outs)]
        if kd in ('pose_regression_3d', 'pose_regression_3d_ex'):
            return K.softargmax3d(ins[0], a['num_joints'], a['depth_maps'], a.get('vis_scale', 1.0))[:len(k.outs)]
        if kd == 'sam2d':
            return K.softargmax2d(ins[0], a['alpha'], 1, ins[1] if a['depth'] else None)[:len(k.outs)]
        if kd == 'zeropad':
            (top, _), (left, _) = a['pads']
            return [K.zeropad(ins[0], top, left, k.outs[0].shape[:2])]
        raise NotImplementedError('plan emulator: kernel op %s' % kd)

    def _step(self, k):
        outs = self.evaluate(k, [self.get(t) for t in k.ins])
        if k.kind == 'copy':
            self.put(k.outs[0], outs[0], c_off=k.attrs['c_off'], channels=k.attrs['channels'])
        else:
            for t, v in zip(k.outs, outs):
                self.put(t, v)
        self.launches += 1

    def run(self, x):
        """x: (N,H,W,3) frames or (B,T,H,W,3) clips -> the model's outputs in Keras shapes (float64)."""
        x = np.asarray(x, np.float64)
        self.n_frames = int(np.prod(x.shape[:-3]))
        self.slots = [np.full(self._items(kind) * fl, np.nan) for (kind, fl) in self.plan.phys]
        t_in = self.graph.inputs[0]
        self.put(t_in, x.reshape((self.n_frames,) + tuple(t_in.shape)))
        for k in self.plan.kops:
            self._step(k)
        outs = []
        for t in self.graph.outputs:
            items = self._items(t.kind) if t.kind == 'clip' else self.n_frames
            outs.append(self.get(t).reshape(self.model._keras_shape(t, items)))
        return outs
