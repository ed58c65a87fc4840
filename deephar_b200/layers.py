"""Host-side mirror of deephar/layers.py (+ the few keras.layers the models call
directly): same helper names, argument order and defaults, but operating on symbolic
`graph.Tensor`s.  Nothing is computed here; compiler.py fuses the recorded layers into
sm_90a kernels.  TimeDistributed wrapping (layers.py:66-104) is implicit: 'frame'
tensors already carry the folded B*T axis.

All convolutions are bias-free (layers.py:69,78).  BatchNormalization in the layers.py
combos has scale=False (layers.py:209,236,...), models/common.py uses the Keras default
scale=True -- the `scale` argument here selects which weights exist.
"""
from .graph import Tensor, conv_out_hw


def int_shape(x):
    """K.int_shape: (None,) + per-item shape."""
    return (None,) + tuple(x.shape)


def appstr(s, a):
    """deephar/utils/parser.py:254-259."""
    try:
        return s + a
    except Exception:
        return None


def _pair(v):
    return (v, v) if isinstance(v, int) else tuple(v)


# ---------------------------------------------------------------------------
# keras.layers primitives
# ---------------------------------------------------------------------------
def Activation(x, kind, name=None):
    assert kind in ('relu', 'sigmoid', 'softmax'), kind
    return x.g.op(kind, [x], x.shape, {'name': name})


def relu(x, leakyrelu=False, name=None):
    """layers.py:51-55."""
    assert not leakyrelu, 'LeakyReLU is never enabled on the forward hot path'
    return Activation(x, 'relu', name=name)


def BatchNormalization(x, scale=True, name=None):
    g = x.g
    name = name or g.auto_name('batch_normalization')
    q = g.qualify(name)
    c = x.channels
    w = {}
    if scale:
        w['gamma'] = g.add_weight(q, 'gamma', (c,))
    w['beta'] = g.add_weight(q, 'beta', (c,))
    w['mean'] = g.add_weight(q, 'moving_mean', (c,))
    w['var'] = g.add_weight(q, 'moving_variance', (c,))
    return g.op('bn', [x], x.shape, {'name': q, 'weights': w})


def conv2d(x, filters, kernel_size, strides=(1, 1), padding='same', name=None):
    """layers.py:66-71."""
    g = x.g
    kernel_size, strides = _pair(kernel_size), _pair(strides)
    name = name or g.auto_name('conv2d')
    q = g.qualify(name)
    h, w, cin = x.shape
    kname = g.add_weight(q, 'kernel', (kernel_size[0], kernel_size[1], cin, filters))
    ho, wo = conv_out_hw(h, w, kernel_size, strides, padding)
    return g.op('conv', [x], (ho, wo, filters),
                {'name': q, 'kernel': kname, 'size': kernel_size, 'strides': strides,
                 'padding': padding})


def sepconv2d(x, filters, kernel_size, strides=(1, 1), padding='same', name=None):
    """layers.py:74-80."""
    g = x.g
    kernel_size, strides = _pair(kernel_size), _pair(strides)
    name = name or g.auto_name('separable_conv2d')
    q = g.qualify(name)
    h, w, cin = x.shape
    dw = g.add_weight(q, 'depthwise_kernel', (kernel_size[0], kernel_size[1], cin, 1))
    pw = g.add_weight(q, 'pointwise_kernel', (1, 1, cin, filters))
    ho, wo = conv_out_hw(h, w, kernel_size, strides, padding)
    return g.op('sepconv', [x], (ho, wo, filters),
                {'name': q, 'depthwise': dw, 'pointwise': pw, 'size': kernel_size,
                 'strides': strides, 'padding': padding})


def MaxPooling2D(x, pool_size=(2, 2), strides=None, padding='valid', name=None):
    """keras default: strides = pool_size, padding 'valid'."""
    pool_size = _pair(pool_size)
    strides = pool_size if strides is None else _pair(strides)
    h, w, c = x.shape
    ho, wo = conv_out_hw(h, w, pool_size, strides, padding)
    return x.g.op('maxpool', [x], (ho, wo, c),
                  {'pool': pool_size, 'strides': strides, 'padding': padding})


def maxpooling2d(x, kernel_size=(2, 2), strides=(2, 2), padding='same', name=None):
    """layers.py:92-97 (note the different defaults: strides (2,2), padding 'same')."""
    return MaxPooling2D(x, kernel_size, strides, padding, name)


def UpSampling2D(x, size=(2, 2), name=None):
    size = _pair(size)
    assert size == (2, 2), 'only nearest x2 is used by the reference models'
    h, w, c = x.shape
    return x.g.op('upsample', [x], (2 * h, 2 * w, c), {})


def upsampling2d(x, kernel_size=(2, 2), name=None):
    """layers.py:100-104."""
    return UpSampling2D(x, kernel_size, name)


def ZeroPadding2D(x, padding):
    (pt, pb), (pl, pr) = padding
    h, w, c = x.shape
    return x.g.op('zeropad', [x], (h + pt + pb, w + pl + pr, c), {'pads': ((pt, pb), (pl, pr))})


def add(ts, name=None):
    assert len(ts) >= 2
    for t in ts[1:]:
        assert t.shape == ts[0].shape and t.kind == ts[0].kind, (ts[0], t)
    return ts[0].g.op('add', list(ts), ts[0].shape, {})


def concatenate(ts, name=None):
    """channel (last-axis) concatenation."""
    base = ts[0].shape[:-1]
    for t in ts:
        assert t.shape[:-1] == base and t.kind == ts[0].kind, (ts[0], t)
    c = sum(t.shape[-1] for t in ts)
    return ts[0].g.op('concat', list(ts), base + (c,), {'name': name})


def multiply(ts, name=None):
    assert len(ts) == 2
    return ts[0].g.op('multiply', list(ts), ts[0].shape, {})


def channel_slice(x, c0, c1):
    """Lambda(lambda x: x[..., c0:c1]) (reception.py:171-172)."""
    assert 0 <= c0 < c1 <= x.channels
    return x.g.op('slice', [x], x.shape[:-1] + (c1 - c0,), {'c0': c0, 'c1': c1})


# ---------------------------------------------------------------------------
# layers.py combos (layers.py:202-325)
# ---------------------------------------------------------------------------
conv = conv2d


def conv_bn(x, filters, size, strides=(1, 1), padding='same', name=None):
    x = conv(x, filters, size, strides, padding, appstr(name, '_conv'))
    return BatchNormalization(x, scale=False, name=name)


def conv_act(x, filters, size, strides=(1, 1), padding='same', name=None):
    x = conv(x, filters, size, strides, padding, appstr(name, '_conv'))
    return relu(x, name=name)


def conv_bn_act(x, filters, size, strides=(1, 1), padding='same', name=None):
    x = conv(x, filters, size, strides, padding, appstr(name, '_conv'))
    x = BatchNormalization(x, scale=False, name=appstr(name, '_bn'))
    return relu(x, name=name)


def bn_act_conv(x, filters, size, strides=(1, 1), padding='same', name=None):
    x = BatchNormalization(x, scale=False, name=appstr(name, '_bn'))
    x = relu(x, name=appstr(name, '_act'))
    return conv(x, filters, size, strides, padding, name)


def act_conv_bn(x, filters, size, strides=(1, 1), padding='same', name=None):
    x = relu(x, name=appstr(name, '_act'))
    x = conv(x, filters, size, strides, padding, appstr(name, '_conv'))
    return BatchNormalization(x, scale=False, name=name)


def separable_conv_bn_act(x, filters, size, strides=(1, 1), padding='same', name=None):
    x = sepconv2d(x, filters, size, strides, padding, appstr(name, '_conv'))
    x = BatchNormalization(x, scale=False, name=appstr(name, '_bn'))
    return relu(x, name=name)


def separable_act_conv_bn(x, filters, size, strides=(1, 1), padding='same', name=None):
    x = relu(x, name=appstr(name, '_act'))
    x = sepconv2d(x, filters, size, strides, padding, appstr(name, '_conv'))
    return BatchNormalization(x, scale=False, name=name)


def separable_conv_bn(x, filters, size, strides=(1, 1), padding='same', name=None):
    x = sepconv2d(x, filters, size, strides, padding, appstr(name, '_conv'))
    return BatchNormalization(x, scale=False, name=name)


def act_conv(x, filters, size, strides=(1, 1), padding='same', name=None):
    x = relu(x, name=appstr(name, '_act'))
    return conv(x, filters, size, strides, padding, name)


# ---------------------------------------------------------------------------
# soft-argmax family (layers.py:107-200, activations.py)
# ---------------------------------------------------------------------------
def channel_softmax_2d(x, alpha=1, name=None):
    """Activation(activations.channel_softmax_2d(alpha)) (activations.py:3-16)."""
    return x.g.op('softmax2d', [x], x.shape, {'alpha': float(alpha), 'name': name})


def act_channel_softmax(x, name=None):
    """layers.py:361-363."""
    return channel_softmax_2d(x, 1, name)


def softargmax2d(x, limits=(0, 0, 1, 1), name=None):
    """layers.py:122-129.  `limits` is accepted and ignored, exactly like the reference
    (lin_interpolation_2d never uses vmin/vmax, layers.py:160-200; SURVEY App. C.1)."""
    h, w, c = x.shape
    return x.g.op('softargmax2d', [x], (1, c, 2), {'name': name})


def keypoint_confidence(x, name=None):
    """layers.py:107-119: 4*AveragePooling2D((2,2),strides 1) -> GlobalMaxPooling2D."""
    h, w, c = x.shape
    return x.g.op('keypoint_confidence', [x], (1, c, 1), {'name': name})


def max_min_pooling(x, strides=(2, 2), padding='same', name=None):
    """layers.py:411-425 (the `strides` argument is the pool size there)."""
    assert _pair(strides) == (2, 2) and padding == 'same'
    h, w, c = x.shape
    ho, wo = conv_out_hw(h, w, (2, 2), (2, 2), 'same')
    return x.g.op('maxminpool', [x], (ho, wo, c), {})


def global_max_min_pooling(x, name=None):
    """layers.py:428-442 -> (C,) logits."""
    return x.g.op('global_maxmin', [x], (1, 1, x.channels), {})


def kronecker_prod(h, f, name='Kronecker_prod'):
    """layers.py:478-508 for clip tensors: (..,H,W,nj) x (..,H,W,F) -> per frame (nj, F)."""
    assert h.shape[:2] == f.shape[:2]
    return h.g.op('kron', [h, f], (1, h.channels, f.channels), {'name': name})


# ---------------------------------------------------------------------------
# SPNet-only helpers (spnet.py:178-235, 98-111)
# ---------------------------------------------------------------------------
def depth_expectation(d_logits, h, name=None):
    """spnet.py:201-205: d = sigmoid(d_logits); z = sum_{h,w}(d * h); expand_dims -> (nj, 1).
    Four parameter-free reference layers (Activation, multiply, two Lambdas) as one graph op."""
    assert d_logits.shape == h.shape
    return h.g.op('depth_expect', [d_logits, h], (1, h.channels, 1), {'name': name})


def frames_to_clip(x):
    """(B*T frames, 1, nj, C) -> (B clips, T, nj, C).  The reference's tensors are (B,T,nj,C) once
    TimeDistributed unfolds; with clip-major frame order this is a free reinterpretation."""
    t = x.g.frames_per_clip
    assert x.kind == 'frame' and x.shape[0] == 1
    return x.g.op('to_clip', [x], (t, x.shape[1], x.shape[2]), {}, kind='clip')


def mask_multiply(p, c):
    """spnet.py:110-111: mask = tile(c, dim); x = p * mask."""
    assert p.shape[:2] == c.shape[:2] and c.shape[2] == 1
    return p.g.op('mask_mul', [p, c], p.shape, {})


def softmax_lastaxis(x, name=None):
    """Activation('softmax') on (B, n_act) logits (spnet.py:66-68)."""
    return x.g.op('softmax', [x], x.shape, {'name': name})
