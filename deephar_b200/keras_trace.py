"""Backend-op tracing for Keras-style model code (the other half of keras_compat.py).

The reference's builders do part of their arithmetic in `Lambda` bodies and `keras.backend` calls: the channel soft-max
(deephar/activations.py:3-16), the soft-argmax as a frozen SeparableConv2D with a grid kernel (layers.py:160-200), the
joint confidence (layers.py:107-119), max+min pooling (layers.py:411-442), the heat-map x feature "kronecker" product
(layers.py:478-508), the confidence mask and the depth expectation of SPNet (spnet.py:110-111, 201-204) and the 3-D
head of ReceptionNet (reception.py:193-222).  None of that is a layer the kernels know.  This module

  1. gives those bodies something to run on: the `keras.backend` functions they call (`K.exp`, `K.sum`, `K.tile`, ...)
     and tensor arithmetic record *backend-op nodes* (`k_*`, kind 'raw') whose shapes follow Keras' rules -- a frame
     tensor of a clip model is 5-D (None, T, H, W, C) there, which is what makes the reference take its
     TimeDistributed branches;
  2. rewrites, when the model is built, every group of backend-op nodes that IS one of the reference's parameter-free
     constructions into the single fused layer op deephar_b200's kernels implement (`rewrite`), checking what it
     absorbs (axes, pool sizes, the frozen grid values against deephar/utils/math.py:6-19); a backend op left over
     that an output depends on is an error naming the node -- nothing is approximated.

The result is the same layer graph deephar_b200's own builders record, so the reference's unmodified
`reception.build()` / `spnet.build()` produce the compiled H100 model (tests/reference_dropin, tests/test_keras_compat.py).
"""
import numpy as np

from . import layers as L
from .graph import Graph, Tensor, conv_out_hw

EPSILON = 1e-7          # keras.backend.epsilon()


# ---------------------------------------------------------------------------------------------------------------------
# Keras' view of a graph tensor
# ---------------------------------------------------------------------------------------------------------------------
_DENSE = ('softargmax2d', 'keypoint_confidence', 'depth_expect', 'kron', 'global_maxmin', 'softmax',
          'pose_regression_2d', 'pose_regression_2d_context', 'pose_regression_3d', 'pose_regression_3d_ex')
_PASS = ('concat', 'slice', 'add', 'multiply', 'relu', 'sigmoid', 'bn', 'scale')


def is_raw(t):
    return t.kind == 'raw'


def _is_dense(t):
    """Layer ops that produce per-joint / per-class vectors store them as (1, n, c) or (1, 1, c); Keras sees (n, c) / (c,)."""
    nd = t.node
    while nd is not None and nd.op in _PASS:
        nd = nd.inputs[0].node
    return nd is not None and (nd.op in _DENSE or nd.op.startswith('head_'))


def kshape(t):
    """Per-sample shape as Keras has it (no batch axis): frames of a clip model carry their time axis."""
    if is_raw(t):
        return t.shape
    s = t.shape
    if _is_dense(t):
        if s[0] == 1:
            s = s[1:]
            if s[0] == 1:
                s = s[1:]
    if t.kind == 'frame' and t.g.frames_per_clip > 1:
        s = (t.g.frames_per_clip,) + s
    return tuple(s)


def int_shape(x):
    return (None,) + kshape(x)


def ndim(x):
    return len(kshape(x)) + 1


def epsilon():
    return EPSILON


def image_data_format():
    return 'channels_last'


def set_image_data_format(fmt):
    assert fmt == 'channels_last'


def unify(ts):
    """Tensors that descend from different Inputs end up in one graph the first time an op combines them."""
    g = ts[0].g
    for t in ts[1:]:
        if t.g is not g:
            if t.g.frames_per_clip != g.frames_per_clip:
                raise ValueError('inputs of one model with different clip lengths')
            g.absorb(t.g)
    return g


def _raw(op, inputs, shape, **attrs):
    return inputs[0].g.op('k_' + op, list(inputs), [tuple(int(d) for d in shape)], attrs, kind='raw')


def _axes(x, axis):
    """Keras axis argument(s) (batch axis counted, negatives allowed) -> sorted per-sample indices."""
    r = ndim(x)
    ax = (axis,) if isinstance(axis, int) else tuple(axis)
    out = []
    for a in ax:
        a = a + r if a < 0 else a
        if not 1 <= a < r:
            raise NotImplementedError('backend op over the batch axis / an axis out of range (%r of rank %d)' % (axis, r))
        out.append(a - 1)
    return tuple(sorted(out))


# ---------------------------------------------------------------------------------------------------------------------
# keras.backend functions
# ---------------------------------------------------------------------------------------------------------------------
def expand_dims(x, axis=-1):
    r = ndim(x) + 1
    a = axis + r if axis < 0 else axis
    if not 1 <= a < r:
        raise NotImplementedError('expand_dims on the batch axis')
    ks = list(kshape(x))
    ks.insert(a - 1, 1)
    return _raw('expand_dims', [x], ks, axis=a - 1)


def squeeze(x, axis):
    (a,) = _axes(x, axis)
    ks = list(kshape(x))
    if ks[a] != 1:
        raise ValueError('squeeze of an axis of size %d' % ks[a])
    del ks[a]
    return _raw('squeeze', [x], ks, axis=a)


def tile(x, n):
    n = tuple(int(v) for v in n)
    ks = kshape(x)
    if len(n) != len(ks) + 1 or n[0] != 1:
        raise NotImplementedError('tile%r of a rank-%d tensor' % (n, len(ks) + 1))
    return _raw('tile', [x], [d * m for d, m in zip(ks, n[1:])], reps=n[1:])


def _reduce(op, x, axis, keepdims):
    if axis is None:
        raise NotImplementedError('K.%s over all axes' % op)
    ax = _axes(x, axis)
    ks = kshape(x)
    out = [1 if i in ax else d for i, d in enumerate(ks)] if keepdims else [d for i, d in enumerate(ks) if i not in ax]
    return _raw(op, [x], out, axes=ax, keepdims=bool(keepdims))


def sum(x, axis=None, keepdims=False):      # noqa: A001  (keras.backend.sum)
    return _reduce('sum', x, axis, keepdims)


def mean(x, axis=None, keepdims=False):
    return _reduce('mean', x, axis, keepdims)


def max(x, axis=None, keepdims=False):      # noqa: A001
    return _reduce('max', x, axis, keepdims)


def exp(x):
    return _raw('exp', [x], kshape(x))


def clip(x, min_value, max_value):
    return _raw('clip', [x], kshape(x), lo=min_value, hi=max_value)


def stop_gradient(x):
    return _raw('stop_gradient', [x], kshape(x))


def reshape(x, shape):
    shape = tuple(shape)
    if shape[0] not in (-1, None):
        raise NotImplementedError('reshape that fixes the batch axis')
    new = tuple(int(d) for d in shape[1:])
    if int(np.prod(new)) != int(np.prod(kshape(x))):
        raise ValueError('reshape %s -> %s changes the number of elements' % (kshape(x), new))
    return _raw('reshape', [x], new)


def arith(op, a, b):
    """a (op) b for tensors / Python scalars, with numpy broadcasting over the per-sample axes."""
    if isinstance(b, Tensor) and not isinstance(a, Tensor):
        a, b = b, a
        if op != 'mul':
            raise NotImplementedError('scalar %s tensor' % op)
    if not isinstance(b, Tensor):
        if op != 'mul':
            raise NotImplementedError('tensor %s scalar' % op)
        return _raw('scale', [a], kshape(a), s=float(b))
    unify([a, b])
    return _raw(op, [a, b], np.broadcast_shapes(kshape(a), kshape(b)))


def neg(x):
    return _raw('neg', [x], kshape(x))


def getitem(x, idx):
    """x[:, ..., a:b]: a slice of the channel axis is a layer op (a view); nothing else can be indexed."""
    idx = idx if isinstance(idx, tuple) else (idx,)
    full = slice(None, None, None)
    if len(idx) != ndim(x) or any(i != full for i in idx[:-1]) or not isinstance(idx[-1], slice) \
            or idx[-1].step not in (None, 1):
        raise NotImplementedError('Lambda: of all indexing only channel slices x[..., a:b] can be recorded')
    if is_raw(x):
        raise NotImplementedError('Lambda: channel slice of a backend-op result')
    a, b, _ = idx[-1].indices(x.channels)
    return L.channel_slice(x, a, b)


# ---------------------------------------------------------------------------------------------------------------------
# parameter-free Keras layers that only occur inside the reference's Lambda bodies / 3-D head
# ---------------------------------------------------------------------------------------------------------------------
def average_pooling_2d(x, pool, strides, padding):
    ks = kshape(x)
    ho, wo = conv_out_hw(ks[-3], ks[-2], pool, strides, padding)
    return _raw('avgpool', [x], ks[:-3] + (ho, wo, ks[-1]), pool=tuple(pool), strides=tuple(strides), padding=padding)


def global_max_pooling_2d(x):
    ks = kshape(x)
    return _raw('gmax2d', [x], ks[:-3] + (ks[-1],))


def global_max_pooling_1d(x):
    ks = kshape(x)
    return _raw('gmax1d', [x], ks[:-2] + (ks[-1],))


def activation(x, fn, name=None):
    """Activation('sigmoid' | 'softmax') of a backend-op result."""
    return _raw('act', [x], kshape(x), fn=fn, name=name)


def merge(op, ts, name=None):
    """concatenate / add with a backend-op operand."""
    ks = [kshape(t) for t in ts]
    if op == 'multiply':
        shape = np.broadcast_shapes(*ks)
    elif op == 'concat':
        if any(k[:-1] != ks[0][:-1] for k in ks):
            raise ValueError('concatenate of shapes %s' % ks)
        shape = ks[0][:-1] + (int(np.sum([k[-1] for k in ks])),)
    else:
        if any(k != ks[0] for k in ks):
            raise ValueError('%s of shapes %s' % (op, ks))
        shape = ks[0]
    return _raw(op, list(ts), shape, name=name)


def as_map(x, per_frame):
    """A backend-op result handed to a spatial layer (Conv2D, MaxPooling2D, ...): its last three axes are the image.
    per_frame: the layer is wrapped in TimeDistributed, so the leading time axis stays folded in the batch."""
    ks = kshape(x)
    g = x.g
    if per_frame:
        if len(ks) != 4 or ks[0] != g.frames_per_clip:
            raise NotImplementedError('TimeDistributed layer on a backend-op result of shape %s' % (ks,))
        return g.op('k_as_map', [x], [ks[1:]], {}, kind='frame')
    if len(ks) != 3:
        raise NotImplementedError('spatial layer on a backend-op result of shape %s' % (ks,))
    return g.op('k_as_map', [x], [ks], {}, kind='clip' if g.frames_per_clip > 1 else 'frame')


def freeze_separable(node, weights):
    """`layer.set_weights(w); layer.trainable = False` on a SeparableConv2D (layers.py:184-194): its kernels become
    constants of the graph -- checked against the grid when the soft-argmax is rewritten -- and leave the weight list."""
    g = node.outs[0].g
    names = (node.attrs['depthwise'], node.attrs['pointwise'])
    g.weight_specs = [(n, s) for n, s in g.weight_specs if n not in names]
    g._weight_names.difference_update(names)
    node.op = 'k_const_sepconv'
    node.attrs['const'] = [np.array(w, dtype=np.float64) for w in weights]


# ---------------------------------------------------------------------------------------------------------------------
# rewrite: backend-op groups -> fused layer ops
# ---------------------------------------------------------------------------------------------------------------------
class _NoMatch(Exception):
    pass


def _is_product(nd):
    return not (nd.op.startswith('k_') or nd.op.startswith('head_'))


def needs_rewrite(g):
    return any(not _is_product(nd) for nd in g.nodes)


class _Rewriter(object):
    def __init__(self, g):
        self.g = g
        new = Graph(g.name)
        new.frames_per_clip = g.frames_per_clip
        new.weight_specs = list(g.weight_specs)
        new._weight_names = set(g._weight_names)
        new._counters = g._counters
        self.new = new
        self.tmap = {}                  # tensor id of g -> tensor of `new`
        self.clips = {}                 # tensor id of `new` (frame) -> its to_clip view
        self.p3d = {}                   # heat-map tensor id of g -> outputs of its pose_regression_3d
        self.used_jprob = set()
        self.cons = {}
        for nd in g.nodes:
            for t in nd.inputs:
                self.cons.setdefault(t.id, []).append(nd)

    # ---- matching helpers ------------------------------------------------------------------------------------------
    def node(self, t, op, **attrs):
        nd = t.node
        if nd is None or nd.op != op:
            raise _NoMatch()
        for k, v in attrs.items():
            if nd.attrs.get(k) != v:
                raise _NoMatch()
        return nd

    def got(self, t):
        """The rewritten tensor of `t`, which must already exist (its producer was copied or fused)."""
        t = self.through(t)
        if t.id not in self.tmap:
            raise _NoMatch()
        return self.tmap[t.id]

    def through(self, t):
        while t.node is not None and t.node.op == 'k_stop_gradient':
            t = t.node.inputs[0]
        return t

    def hw_axes(self, t):
        """per-sample indices of the (rows, cols) axes of a map-shaped tensor."""
        n = len(kshape(t))
        return (n - 3, n - 2)

    def to_clip(self, t_new):
        if t_new.kind != 'frame':
            return t_new
        if t_new.id not in self.clips:
            self.clips[t_new.id] = L.frames_to_clip(t_new)
        return self.clips[t_new.id]

    # ---- driver ----------------------------------------------------------------------------------------------------
    def run(self, outputs):
        for nd in self.g.nodes:
            if all(o.id in self.tmap for o in nd.outs):
                continue                                    # resolved ahead by the pattern of another root
            if nd.op == 'input':
                self.tmap[nd.outs[0].id] = self.new.input(nd.outs[0].shape, nd.outs[0].kind)
                continue
            if _is_product(nd):
                if all(t.id in self.tmap for t in nd.inputs):
                    self.copy(nd)
                continue
            for pat in self.PATTERNS:
                try:
                    res = pat(self, nd)
                except _NoMatch:
                    continue
                if res is not None:
                    self.tmap[nd.outs[0].id] = res
                    break
        outs = []
        for t in outputs:
            t = self.through(t)
            if t.id not in self.tmap:
                raise NotImplementedError(
                    'model output %r depends on backend arithmetic (Lambda / keras.backend ops) that is not one of the '
                    "reference's parameter-free constructions: %s" % (t, self.blame(t)))
            outs.append(self.tmap[t.id])
        return self.new, outs

    def blame(self, t):
        seen, stack, bad = set(), [t], []
        while stack:
            u = stack.pop()
            if u.id in seen or u.id in self.tmap:
                continue
            seen.add(u.id)
            if u.node is not None:
                bad.append(u.node)
                stack.extend(u.node.inputs)
        bad.sort(key=lambda n: n.id)
        return ', '.join('%s%s' % (n.op, kshape(n.outs[0])) for n in bad[:8])

    def copy(self, nd):
        attrs = {k: (dict(v) if isinstance(v, dict) else v) for k, v in nd.attrs.items()}
        outs = self.new.op(nd.op, [self.tmap[t.id] for t in nd.inputs], [o.shape for o in nd.outs], attrs,
                           kind=nd.outs[0].kind)
        outs = outs if isinstance(outs, tuple) else (outs,)
        for o_src, o_new in zip(nd.outs, outs):
            self.tmap[o_src.id] = o_new

    # ---- patterns (each takes the LAST node of a construction) -----------------------------------------------------
    def p_identity(self, nd):
        if nd.op != 'k_stop_gradient':
            raise _NoMatch()
        return self.got(nd.inputs[0])

    def _softmax_parts(self, nd):
        """activations.py:9-14: e = exp(a*x - max_hw(a*x)); e / clip(sum_hw(e), eps, inf)  ->  (x, a)."""
        if nd.op != 'k_div':
            raise _NoMatch()
        e, s = nd.inputs
        c = self.node(s, 'k_clip')
        if c.attrs['hi'] is not None or abs(c.attrs['lo'] - EPSILON) > 1e-12:
            raise _NoMatch()
        sm = self.node(c.inputs[0], 'k_sum', keepdims=True)
        ex = self.node(e, 'k_exp')
        if sm.inputs[0] is not e:
            raise _NoMatch()
        sub = self.node(ex.inputs[0], 'k_sub')
        y, m = sub.inputs
        mx = self.node(m, 'k_max', keepdims=True)
        if mx.inputs[0] is not y:
            raise _NoMatch()
        alpha, x = 1.0, y
        if y.node is not None and y.node.op == 'k_scale':
            alpha, x = y.node.attrs['s'], y.node.inputs[0]
        if sm.attrs['axes'] != self.hw_axes(x) or mx.attrs['axes'] != self.hw_axes(x):
            raise _NoMatch()
        return x, alpha

    def p_softmax2d(self, nd):
        x, alpha = self._softmax_parts(nd)
        if is_raw(x):
            # softmax of the depth-averaged volume (action.py:294-295): third output of the extended 3-D head
            h, depth, nj, _ = self._volume_xy(x)
            if alpha != 1.0:
                raise _NoMatch()
            return self._pose3d(h, depth, nj)[2]
        return L.channel_softmax_2d(self.got(x), alpha=alpha, name=nd.attrs.get('name'))

    def _lin_interp(self, t, dim):
        """layers.py:160-200: frozen SeparableConv2D((rows, cols), valid) with depthwise = the grid of utils/math.py:6-19
        along `dim`, pointwise = identity, then squeeze, squeeze, expand_dims -> (.., C, 1).  Returns the input map."""
        e = self.node(t, 'k_expand_dims')
        if e.attrs['axis'] != len(kshape(t)) - 1:
            raise _NoMatch()
        s2 = self.node(e.inputs[0], 'k_squeeze')
        s1 = self.node(s2.inputs[0], 'k_squeeze')
        cv = self.node(s1.inputs[0], 'k_const_sepconv')
        x = cv.inputs[0]
        rows, cols, ch = x.shape
        if tuple(cv.attrs['size']) != (rows, cols) or cv.attrs['padding'] != 'valid' or tuple(cv.attrs['strides']) != (1, 1) \
                or cv.outs[0].shape != (1, 1, ch):
            raise _NoMatch()
        dw, pw = cv.attrs['const']
        lin_c = np.linspace(0.0, 1.0, cols)
        lin_r = np.linspace(0.0, 1.0, rows)
        grid = np.tile(lin_c[None, :], (rows, 1)) if dim == 0 else np.tile(lin_r[:, None], (1, cols))
        if dw.shape != (rows, cols, ch, 1) or np.abs(dw[:, :, :, 0] - grid[:, :, None]).max() > 1e-6 \
                or pw.shape != (1, 1, ch, ch) or np.abs(pw[0, 0] - np.eye(ch)).max() > 0:
            raise NotImplementedError('frozen SeparableConv2D %r is not the soft-argmax grid of the reference '
                                      '(deephar/layers.py:184-194)' % cv.attrs.get('name'))
        return x

    def p_softargmax2d(self, nd):
        if nd.op != 'k_concat' or len(nd.inputs) != 2:
            raise _NoMatch()
        xa = self._lin_interp(nd.inputs[0], 0)
        xb = self._lin_interp(nd.inputs[1], 1)
        if self.got(xa) is not self.got(xb):
            raise _NoMatch()
        return L.softargmax2d(self.got(xa), name=nd.attrs.get('name'))

    def _four_avg_max(self, t):
        """max_hw(4 * AveragePooling2D((2,2), strides 1, valid)(x)) -> x"""
        gm = self.node(t, 'k_gmax2d')
        sc = self.node(gm.inputs[0], 'k_scale')
        av = self.node(sc.inputs[0], 'k_avgpool', pool=(2, 2), strides=(1, 1), padding='valid')
        if abs(sc.attrs['s'] - 4.0) > 0:
            raise _NoMatch()
        return av.inputs[0]

    def p_keypoint_confidence(self, nd):
        """layers.py:111-115 on probability maps."""
        if nd.op != 'k_expand_dims' or nd.attrs['axis'] != len(kshape(nd.outs[0])) - 1:
            raise _NoMatch()
        x = self._four_avg_max(nd.inputs[0])
        xn = self.got(x)
        if xn.node.op != 'softmax2d':
            raise _NoMatch()
        return L.keypoint_confidence(xn, name=nd.attrs.get('name'))

    def _neg_of(self, t, x):
        m = t.node
        if m is not None and m.op == 'k_as_map':
            t = m.inputs[0]
        n = self.node(t, 'k_neg')
        if n.inputs[0] is not x:
            raise _NoMatch()

    def p_max_min_pooling(self, nd):
        """layers.py:420-423: MaxPooling2D(x) - MaxPooling2D(-x)."""
        if nd.op != 'k_sub':
            raise _NoMatch()
        a = self.node(nd.inputs[0], 'maxpool')
        b = self.node(nd.inputs[1], 'maxpool')
        if any(a.attrs[k] != b.attrs[k] for k in ('pool', 'strides', 'padding')):
            raise _NoMatch()
        x = a.inputs[0]
        self._neg_of(b.inputs[0], x)
        if a.attrs['pool'] != (2, 2) or a.attrs['strides'] != (2, 2) or a.attrs['padding'] != 'same':
            raise NotImplementedError('max_min_pooling other than (2, 2) / same')
        return L.max_min_pooling(self.got(x), (2, 2))

    def p_global_max_min_pooling(self, nd):
        """layers.py:437-440: GlobalMaxPooling2D(x) - GlobalMaxPooling2D(-x)."""
        if nd.op != 'k_sub':
            raise _NoMatch()
        a = self.node(nd.inputs[0], 'k_gmax2d')
        b = self.node(nd.inputs[1], 'k_gmax2d')
        x = a.inputs[0]
        self._neg_of(b.inputs[0], x)
        return L.global_max_min_pooling(self.got(x))

    def p_activation(self, nd):
        if nd.op != 'k_act' or nd.attrs['fn'] != 'softmax':
            raise _NoMatch()
        return L.softmax_lastaxis(self.got(nd.inputs[0]), name=nd.attrs.get('name'))

    def p_kron(self, nd):
        """layers.py:482-506: sum_hw(tile(hm[..., None], nf) * tile(x[..., None, :], nj))."""
        if nd.op != 'k_sum' or nd.attrs['keepdims']:
            raise _NoMatch()
        mul = self.node(nd.inputs[0], 'k_mul')
        ta = self.node(mul.inputs[0], 'k_tile')
        tb = self.node(mul.inputs[1], 'k_tile')
        ea = self.node(ta.inputs[0], 'k_expand_dims')
        eb = self.node(tb.inputs[0], 'k_expand_dims')
        hm, x = ea.inputs[0], eb.inputs[0]
        nj, nf = hm.channels, x.channels
        r = len(kshape(hm))
        if ea.attrs['axis'] != r or eb.attrs['axis'] != r - 1 or ta.attrs['reps'] != (1,) * r + (nf,) \
                or tb.attrs['reps'] != (1,) * (r - 1) + (nj, 1):
            raise _NoMatch()
        if nd.attrs['axes'] != self.hw_axes(hm):
            # 5-D operands (no time axis): the reference's axis=(2, 3) then sums cols and joints (SURVEY App. C)
            raise NotImplementedError('kronecker_prod is only defined for clip tensors in the reference '
                                      '(layers.py:478-508)')
        return L.kronecker_prod(self.got(hm), self.got(x), name=nd.attrs.get('name'))

    def p_mask_multiply(self, nd):
        """spnet.py:110-111: p * tile(c, dim) on (T, joints, dim) pose tensors -> the (frames x joints) image."""
        if nd.op != 'k_mul':
            raise _NoMatch()
        p, m = nd.inputs
        tl = self.node(m, 'k_tile')
        c = tl.inputs[0]
        kp, kc = kshape(p), kshape(c)
        if len(kp) != 3 or kc != kp[:-1] + (1,) or tl.attrs['reps'] != (1, 1, kp[-1]):
            raise _NoMatch()
        return L.mask_multiply(self.to_clip(self.got(p)), self.to_clip(self.got(c)))

    def p_as_map(self, nd):
        if nd.op != 'k_as_map':
            raise _NoMatch()
        x = self.got(nd.inputs[0])
        if nd.outs[0].kind == 'clip' and x.kind == 'frame' and kshape(nd.inputs[0]) == nd.outs[0].shape:
            return self.to_clip(x)
        if x.kind == nd.outs[0].kind and x.shape == nd.outs[0].shape:
            return x
        raise _NoMatch()

    def p_depth_expectation(self, nd):
        """spnet.py:201-204: expand_dims(sum_hw(sigmoid(d) * h))."""
        if nd.op != 'k_expand_dims' or nd.attrs['axis'] != len(kshape(nd.outs[0])) - 1:
            raise _NoMatch()
        sm = self.node(nd.inputs[0], 'k_sum', keepdims=False)
        mul = sm.inputs[0].node
        if mul is None or mul.op not in ('multiply', 'k_multiply') or len(mul.inputs) != 2:
            raise _NoMatch()
        d, h = mul.inputs
        sg = self.node(d, 'sigmoid')
        if sm.attrs['axes'] != self.hw_axes(h):
            raise _NoMatch()
        return L.depth_expectation(self.got(sg.inputs[0]), self.got(h))

    def p_merge(self, nd):
        if nd.op == 'k_concat':
            return L.concatenate([self.got(t) for t in nd.inputs], name=nd.attrs.get('name'))
        if nd.op == 'k_add':
            return L.add([self.got(t) for t in nd.inputs])
        raise _NoMatch()

    # -- ReceptionNet heads (reception.py:167-222; the head models themselves are keras_compat._Head objects) --------
    def _sliced(self, t):
        nd = t.node
        if nd is not None and nd.op == 'slice':
            return nd.inputs[0], nd.attrs['c0'], nd.attrs['c1']
        return t, 0, t.channels

    def _visibility_of(self, h, c0, c1, outs):
        """The joint-probability head on the maps h[..., c0:c1] -- or on s * those maps (`sjProb(4 * hs)`, action.py:200:
        max of a 2x2 mean is positively homogeneous, so that is s * the fused op's second output) -- gets `outs[1]`."""
        def maps_of(j):
            t, s = j.inputs[0], 1.0
            if t.node is not None and t.node.op == 'k_scale' and t.node.attrs['s'] > 0:
                t, s = t.node.inputs[0], t.node.attrs['s']
            return self._sliced(t), s

        vis = [j for j in self.g.nodes if j.op == 'head_jprob' and j.id not in self.used_jprob
               and maps_of(j)[0][0] is h and maps_of(j)[0][1:] == (c0, c1)]
        if len(vis) != 1:
            raise NotImplementedError('soft-argmax head without its joint-probability model on the same maps')
        self.used_jprob.add(vis[0].id)
        scale = maps_of(vis[0])[1]
        v = outs[1]
        if scale != 1.0:
            v = self.new.op('scale', [v], v.shape, {'value': float(scale)})
        self.tmap[vis[0].outs[0].id] = v

    def p_head_context(self, nd):
        """agg([sam2d(h[..., :nj]), sam2d(h[..., nj:]), jprob(h[..., nj:])]) + jprob(h[..., :nj])."""
        if nd.op != 'head_agg':
            raise _NoMatch()
        ys, yc, pc = nd.inputs
        if not (ys.node.op == 'head_sam2d' and yc.node.op == 'head_sam2d' and pc.node.op == 'head_jprob'):
            raise NotImplementedError('context aggregation of tensors that are not soft-argmax / probability heads')
        h, a0, a1 = self._sliced(ys.node.inputs[0])
        h2, b0, b1 = self._sliced(yc.node.inputs[0])
        h3, c0, c1 = self._sliced(pc.node.inputs[0])
        nj, nc = nd.attrs['num_joints'], nd.attrs['num_context']
        if not (h is h2 is h3 and (a0, a1) == (0, nj) and (b0, b1) == (c0, c1) == (nj, h.channels)
                and h.channels == nj * (nc + 1)):
            raise NotImplementedError('context aggregation over an unexpected split of the heat-maps')
        self.used_jprob.add(pc.node.id)
        outs = self.new.op('pose_regression_2d_context', [self.got(h)], [(1, nj, 2), (1, nj, 1)],
                           {'num_joints': nj, 'num_context': nc, 'alpha': nd.attrs['alpha']})
        self._visibility_of(h, 0, nj, outs)
        return outs[0]

    def p_head_plain(self, nd):
        """sam2d(h) + jprob(h)."""
        if nd.op != 'head_sam2d':
            raise _NoMatch()
        users = self.cons.get(nd.outs[0].id, [])
        if any(u.op in ('head_agg', 'k_concat') for u in users):
            raise _NoMatch()                                # operand of the context / 3-D construction
        t = nd.inputs[0]
        if is_raw(t):
            raise _NoMatch()
        c = t.channels
        outs = self.new.op('pose_regression_2d', [self.got(t)], [(1, c, 2), (1, c, 1)], {})
        self._visibility_of(*(self._sliced(t) + (outs,)))
        return outs[0]

    def _volume_xy(self, hxy):
        """reception.py:196-204: h (H, W, D*nj) -> reshape (H, W, D, nj) (depth-major channels); hxy = mean over D."""
        mxy = self.node(hxy, 'k_mean', keepdims=False)
        rs = self.node(mxy.inputs[0], 'k_reshape')
        ex = self.node(rs.inputs[0], 'k_expand_dims')
        h = ex.inputs[0]
        if is_raw(h):
            raise _NoMatch()
        rows, cols, ch = h.shape
        vol = kshape(rs.outs[0])
        n = len(vol)
        if vol[-4:-2] != (rows, cols) or vol[-2] * vol[-1] != ch or mxy.attrs['axes'] != (n - 2,):
            raise _NoMatch()
        return h, vol[-2], vol[-1], rs

    def _volume(self, hxy, hz):
        """... and hz = mean over (H, W) of the same volume (reception.py:205)."""
        h, depth, nj, rs = self._volume_xy(hxy)
        mz = self.node(hz, 'k_mean', keepdims=False)
        n = len(kshape(rs.outs[0]))
        if mz.inputs[0] is not rs.outs[0] or mz.attrs['axes'] != (n - 4, n - 3):
            raise _NoMatch()
        return h, depth, nj

    def _visibility_3d(self, nd):
        """sigmoid(s * expand_dims(GlobalMaxPooling2D(hxy) + GlobalMaxPooling1D(hz)))  ->  (h, D, nj, s);
        s = 1 in reception.py:217-220, 2 in action.py:291-292."""
        if nd.op != 'k_act' or nd.attrs['fn'] != 'sigmoid':
            raise _NoMatch()
        t, scale = nd.inputs[0], 1.0
        if t.node is not None and t.node.op == 'k_scale':
            t, scale = t.node.inputs[0], t.node.attrs['s']
        ex = self.node(t, 'k_expand_dims')
        ad = self.node(ex.inputs[0], 'k_add')
        if len(ad.inputs) != 2:
            raise _NoMatch()
        g2 = self.node(ad.inputs[0], 'k_gmax2d')
        g1 = self.node(ad.inputs[1], 'k_gmax1d')
        return self._volume(g2.inputs[0], g1.inputs[0]) + (scale,)

    def _pose3d(self, h, depth, nj):
        """The fused 3-D head of the heat-map volume h: (pose, visibility) -- or, when the model also takes the
        soft-max of the depth-averaged maps or scales the visibility logit (the CVPR'18 clip model), the extended op
        (pose, visibility, probability maps)."""
        if h.id in self.p3d:
            return self.p3d[h.id]
        scale, wants_prob = 1.0, False
        for nd in self.g.nodes:
            try:
                hv, _, _, sv = self._visibility_3d(nd)
                if hv is h:
                    scale = sv
            except _NoMatch:
                pass
            try:
                x, _ = self._softmax_parts(nd)
                wants_prob = wants_prob or (is_raw(x) and self._volume_xy(x)[0] is h)
            except _NoMatch:
                pass
        if scale == 1.0 and not wants_prob:
            outs = self.new.op('pose_regression_3d', [self.got(h)], [(1, nj, 3), (1, nj, 1)],
                               {'num_joints': nj, 'depth_maps': depth})
        else:
            rows, cols, _ = h.shape
            outs = self.new.op('pose_regression_3d_ex', [self.got(h)], [(1, nj, 3), (1, nj, 1), (rows, cols, nj)],
                               {'num_joints': nj, 'depth_maps': depth, 'vis_scale': float(scale)})
        self.p3d[h.id] = outs
        return outs

    def p_head_3d_pose(self, nd):
        """concatenate([sSAM(hxy), zSAM(hz)])."""
        if nd.op != 'k_concat' or len(nd.inputs) != 2:
            raise _NoMatch()
        sxy = self.node(nd.inputs[0], 'head_sam2d')
        sz = self.node(nd.inputs[1], 'head_sam1d')
        h, depth, nj = self._volume(sxy.inputs[0], sz.inputs[0])
        return self._pose3d(h, depth, nj)[0]

    def p_head_3d_visibility(self, nd):
        h, depth, nj, _ = self._visibility_3d(nd)
        return self._pose3d(h, depth, nj)[1]

    PATTERNS = (p_identity, p_softmax2d, p_softargmax2d, p_keypoint_confidence, p_max_min_pooling,
                p_global_max_min_pooling, p_activation, p_kron, p_mask_multiply, p_as_map, p_depth_expectation,
                p_head_context, p_head_plain, p_head_3d_pose, p_head_3d_visibility, p_merge)


def rewrite(g, outputs):
    """(graph recorded by keras_compat, its output tensors) -> (layer graph of fused ops only, outputs)."""
    if not needs_rewrite(g):
        return g, outputs
    new, outs = _Rewriter(g).run(outputs)
    for attr in ('act_cnt',):
        if hasattr(g, attr):
            setattr(new, attr, getattr(g, attr))
    return new, outs
