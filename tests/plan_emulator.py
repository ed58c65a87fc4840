"""CPU emulation of a compiled plan -- TEST INFRASTRUCTURE (never imported by the product).

`deephar_b200.compiler.compile_graph` turns a layer graph into a sequence of kernel ops over a planned set of buffers:
BatchNormalization / ReLU folded into conv prologues and epilogues, residual adds (one of them through a 2x upsampling) and
a pooled second output fused into conv kernels, concatenations turned into channel-offset views or copies, soft-max heads
fused into one op, buffers aliased by liveness.  On the GPU that plan is executed by `Model._bind` / `_issue` through the C
ABI.  Here the SAME plan is executed on the CPU, op by op, on numpy float64 buffers laid out exactly as the plan says
(physical slot, per-item stride, channel offset, leading dimension), each op following the contract written in
include/deephar_b200.h with the oracle's primitives (`oracle/ops_np.py`) doing the arithmetic.  Slots start NaN-filled, so
a read of memory no launch has written, or a buffer recycled while still live, poisons the outputs.

What this checks without a GPU: the compiler's fusion decisions, operand order, attribute plumbing, which BatchNormalization
folds into which conv, concat / slice / clip views and the liveness-based slot reuse -- for any model, including the
ones recorded from Keras-style code.  What it does not check: the CUDA kernels (the `-m gpu` tests do).
"""
import numpy as np

from oracle import ops_np as O


def _bn_fold(hw, bn):
    """(scale, shift) of an inference BatchNormalization in float64 (the product folds the same way and rounds the result
    to fp32 for the device, `weights.fold_batchnorm`; tests/test_plan_emulator.py compares the two)."""
    w = bn['weights']
    scale = 1.0 / np.sqrt(hw[w['var']] + O.EPS_BN)
    if 'gamma' in w:
        scale = scale * hw[w['gamma']]
    return scale, hw[w['beta']] - hw[w['mean']] * scale


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

    def prologue(self, k, x):
        """a conv / sepconv launch's input after its fused BatchNormalization and ReLU (the MMA's operand)"""
        a = k.attrs
        if a['pre_bn']:
            sc, sh = self.fold(a['pre_bn'])
            x = x * sc + sh
        if a['pre_relu']:
            x = np.maximum(x, 0.0)
        return x

    def _conv(self, k, ins):
        a = k.attrs
        x = self.prologue(k, ins[0])
        if k.kind == 'sepconv':
            y = O.separable_conv2d(x, self.hw[a['depthwise']], self.hw[a['pointwise']], tuple(a['strides']), a['padding'])
        else:
            y = O.conv2d(x, self.hw[a['kernel']], tuple(a['strides']), a['padding'])
        if a['post_bn']:
            sc, sh = self.fold(a['post_bn'])
            y = y * sc + sh
        if a['post_relu']:
            y = np.maximum(y, 0.0)
        for i in range(a['n_res']):
            r = ins[1 + i]
            if (a.get('res_up2x', 0) >> i) & 1:
                r = O.upsample2d(r)
            y = y + r
        return [y, O.maxpool2d(y, (2, 2))] if a.get('pool_out') else [y]

    def _sam2d(self, k, ins):
        a = k.attrs
        p = O.channel_softmax_2d(ins[0], a['alpha'])
        pose = O.softargmax2d(p)
        if a['depth']:
            z = np.sum(O.sigmoid(ins[1]) * p, axis=(1, 2))[..., None]          # spnet.py:201-205
            pose = np.concatenate([pose, z], axis=-1)
        return [pose, O.keypoint_confidence(p)] + ([p] if a['prob'] else [])

    def _pose3d(self, k, h, vis_scale=1.0, prob=False):
        a = k.attrs
        n, hh, ww, ch = h.shape
        h5 = h.reshape(n, hh, ww, a['depth_maps'], a['num_joints'])
        hxy, hz = h5.mean(axis=3), h5.mean(axis=(1, 2))
        pose = np.concatenate([O.softargmax2d(O.channel_softmax_2d(hxy)), O.lin_interpolation_1d(O.channel_softmax_1d(hz))],
                              axis=-1)
        vis = O.sigmoid(vis_scale * (hxy.max(axis=(1, 2)) + hz.max(axis=1)))[..., None]
        return [pose, vis] + ([O.channel_softmax_2d(hxy)] if prob else [])

    def evaluate(self, k, ins):
        """launch k on its inputs `ins` (float64, one (items, H, W, C) array per k.ins) -> one array per output of k, in
        the order of k.outs; a concat copy's is its channel range [attrs c_off, + channels) of k.outs[0]"""
        kd, a = k.kind, k.attrs
        if kd in ('conv', 'sepconv'):
            return self._conv(k, ins)
        if kd == 'maxpool':
            return [O.maxpool2d(ins[0], tuple(a['pool']), tuple(a['strides']), a['padding'])]
        if kd == 'upsample_add':
            return [ins[0] + O.upsample2d(ins[1])]
        if kd == 'upsample':
            return [O.upsample2d(ins[0])]
        if kd in ('add', 'affine', 'copy'):
            y = sum(ins)
            if kd == 'affine':
                if a['bn']:
                    sc, sh = self.fold(a['bn'])
                    y = y * sc + sh
                if a['relu']:
                    y = np.maximum(y, 0.0)
            return [y]
        if kd == 'scale':
            return [ins[0] * float(a['value'])]
        if kd == 'pose_regression_2d_context':
            h = ins[0]
            nj, nc = a['num_joints'], a['num_context']
            hs, hc = h[..., :nj], h[..., nj:]
            ys, yc = O.softargmax2d(O.channel_softmax_2d(hs)), O.softargmax2d(O.channel_softmax_2d(hc))
            pc = O.keypoint_confidence(hc)                                   # on RAW maps (blocks.py:328-343)
            grp = lambda v: v.reshape(v.shape[0], nj, nc, -1).sum(axis=2)     # noqa: E731   blocks.py:227-233
            return [a['alpha'] * ys + (1 - a['alpha']) * grp(yc * pc) / grp(pc), O.keypoint_confidence(hs)]
        if kd == 'pose_regression_2d':
            return [O.softargmax2d(O.channel_softmax_2d(ins[0])), O.keypoint_confidence(ins[0])]
        if kd == 'pose_regression_3d':
            return self._pose3d(k, ins[0])
        if kd == 'pose_regression_3d_ex':
            return self._pose3d(k, ins[0], vis_scale=a['vis_scale'], prob=True)
        if kd == 'sam2d':
            return self._sam2d(k, ins)
        if kd == 'kron':
            return [np.einsum('nhwj,nhwf->njf', ins[0], ins[1])]
        if kd == 'mask_mul':
            return [ins[0] * ins[1]]
        if kd == 'zeropad':
            return [O.zeropad2d(ins[0], a['pads'])]
        if kd == 'maxminpool':
            return [O.max_min_pooling(ins[0], (2, 2), 'same')]
        if kd == 'global_maxmin_softmax':
            return [O.softmax(O.global_max_min_pooling(ins[0]))]
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
