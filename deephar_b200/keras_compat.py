"""Keras-signature front end: write (or keep) model code in the `keras.layers` functional style the reference's
builders use -- `Conv2D(filters, size, use_bias=False, name=...)(x)`, `BatchNormalization(name=...)(x)`,
`add([a, b])`, `Model(inputs=inp, outputs=outs)` -- and get a compiled H100 model instead of a TensorFlow graph.

    from deephar_b200.keras_compat import Input, Conv2D, BatchNormalization, Activation, add, Model
    inp = Input(shape=(256, 256, 3))
    x = Conv2D(64, (7, 7), strides=(2, 2), padding='same', use_bias=False, name='conv1')(inp)
    x = Activation('relu')(BatchNormalization(name='bn1')(x))
    model = Model(inputs=inp, outputs=[x])          # -> deephar_b200.model.Model: predict / load_weights / ...

Every layer object records a node of the symbolic graph (graph.py) when it is called; nothing is computed here.
Layer classes, argument names and DEFAULTS are those of Keras 2.1.4 (the version the reference pins: Conv2D padding
'valid', use_bias True, BatchNormalization scale/center True, MaxPooling2D strides = pool_size ...), so code written for
the reference means the same thing.  What the forward path of the reference models never uses is rejected at build
time, not silently approximated: biases (all reference convs are `use_bias=False`, deephar/layers.py:69,78),
activations fused into a conv via `activation=`, dilation, depth_multiplier != 1, `data_format='channels_first'`.
The reference's own helper layer on top of Keras (deephar/layers.py, deephar/activations.py) is mirrored function-style
in deephar_b200.layers and re-exported here (`channel_softmax_2d`, `softargmax2d`, `kronecker_prod`, ...).
`TimeDistributed(layer, name=...)` is the identity on the folded B*T frame axis and passes its name to the wrapped
layer, which is how Keras names the weights of a wrapped layer in a checkpoint.
"""
from . import keras_trace as backend          # `from deephar_b200.keras_compat import backend as K`
from . import layers as L
from .graph import Graph, Tensor
from .layers import (act_channel_softmax, channel_slice, channel_softmax_2d, depth_expectation,  # noqa: F401
                     global_max_min_pooling, keypoint_confidence, kronecker_prod, max_min_pooling, softargmax2d)
from .model import Model as _Model


# Keras numbers auto-named layers (conv2d_7, batch_normalization_12) with ONE counter per class for the whole
# session, across sub-models: every graph started here shares this table until clear_session().
_SESSION_COUNTERS = {}


def clear_session():
    """keras.backend.clear_session(): restart the auto-name counters (call between two independent models)."""
    _SESSION_COUNTERS.clear()


def Input(shape=None, batch_shape=None, name=None, graph=None, frames_per_clip=None):
    """keras.layers.Input.  shape (H, W, C) -> per-frame tensor; shape (T, H, W, C) -> a clip input whose frames are
    folded into the batch axis (what TimeDistributed does in the reference, deephar/models/spnet.py:283-296).  A new
    symbolic graph starts at every Input unless `graph` is given."""
    if shape is None and batch_shape is not None:
        shape = tuple(batch_shape)[1:]
    if shape is None:
        raise ValueError('Input: shape is required')
    shape = tuple(int(s) for s in shape)
    if graph is not None:
        g = graph
    else:
        g = Graph(name or 'model')
        g._counters = _SESSION_COUNTERS
    if len(shape) == 4:
        g.frames_per_clip = int(shape[0])
        shape = shape[1:]
    elif frames_per_clip:
        g.frames_per_clip = int(frames_per_clip)
    if len(shape) != 3:
        raise ValueError('Input: expected (H, W, C) or (T, H, W, C), got %r' % (shape,))
    return g.input(shape)


class Layer(object):
    """A Keras layer object: constructed with its hyper-parameters, applied by calling it on a tensor."""

    def __init__(self, name=None, **kwargs):
        unknown = set(kwargs) - {'trainable', 'input_shape', 'dtype'}
        if unknown:
            raise TypeError('%s: unsupported argument(s) %s' % (type(self).__name__, sorted(unknown)))
        self.name = name
        self._built = False

    def __call__(self, x):
        if self._built and self._has_weights:
            raise NotImplementedError('%s %r: calling a weighted layer twice (weight sharing) is not used by the '
                                      'reference models' % (type(self).__name__, self.name))
        self._built = True
        if self._spatial and isinstance(x, Tensor):
            x = _as_image(x)
        return self.call(x)

    _has_weights = False
    _spatial = False            # works on the (rows, cols, channels) axes of its input


_TD_DEPTH = [0]                 # > 0 while a TimeDistributed wrapper applies its layer


def _as_image(x):
    """What a spatial layer sees.  Backend-op results and per-joint tensors are 4-D (None, T, joints, c) for Keras: a
    plain Conv2D / MaxPooling2D treats (T, joints) as the image (spnet.py:113-132) -- here a clip-axis tensor."""
    if backend.is_raw(x):
        return backend.as_map(x, per_frame=_TD_DEPTH[0] > 0)
    if _TD_DEPTH[0] == 0 and x.kind == 'frame' and x.g.frames_per_clip > 1 and x.shape[0] == 1 and backend._is_dense(x):
        return L.frames_to_clip(x)
    return x


def _no(cond, what):
    if cond:
        raise NotImplementedError(what + ' is not on the forward path of the reference models')


class Conv2D(Layer):
    _has_weights = True
    _spatial = True

    def __init__(self, filters, kernel_size, strides=(1, 1), padding='valid', data_format=None, dilation_rate=(1, 1),
                 activation=None, use_bias=True, name=None, **kwargs):
        Layer.__init__(self, name, **{k: v for k, v in kwargs.items() if not k.endswith(('_initializer', '_regularizer',
                                                                                           '_constraint'))})
        _no(use_bias, 'Conv2D(use_bias=True)')
        _no(activation not in (None, 'linear'), 'Conv2D(activation=...)')
        _no(L._pair(dilation_rate) != (1, 1), 'dilated convolution')
        _no(data_format not in (None, 'channels_last'), 'channels_first')
        self.filters, self.kernel_size, self.strides, self.padding = int(filters), kernel_size, strides, padding

    def call(self, x):
        return L.conv2d(x, self.filters, self.kernel_size, self.strides, self.padding, name=self.name)


class SeparableConv2D(Layer):
    _has_weights = True
    _spatial = True

    def __init__(self, filters, kernel_size, strides=(1, 1), padding='valid', data_format=None, depth_multiplier=1,
                 activation=None, use_bias=True, name=None, **kwargs):
        Layer.__init__(self, name, **{k: v for k, v in kwargs.items() if not k.endswith(('_initializer', '_regularizer',
                                                                                           '_constraint'))})
        _no(use_bias, 'SeparableConv2D(use_bias=True)')
        _no(activation not in (None, 'linear'), 'SeparableConv2D(activation=...)')
        _no(depth_multiplier != 1, 'depth_multiplier != 1')
        _no(data_format not in (None, 'channels_last'), 'channels_first')
        self.filters, self.kernel_size, self.strides, self.padding = int(filters), kernel_size, strides, padding

    def call(self, x):
        out = L.sepconv2d(x, self.filters, self.kernel_size, self.strides, self.padding, name=self.name)
        self._node = out.node
        return out

    # The reference freezes a SeparableConv2D into a constant operator (the soft-argmax grid, layers.py:184-194):
    # get_weights() -> edit -> set_weights(); trainable = False.  The kernels then are constants of the graph.
    def get_weights(self):
        import numpy as np
        g = self._node.outs[0].g
        shapes = dict(g.weight_specs)
        return [np.zeros(shapes[self._node.attrs[k]], np.float32) for k in ('depthwise', 'pointwise')]

    def set_weights(self, weights):
        self._assigned = weights
        if not self._trainable:
            backend.freeze_separable(self._node, weights)

    @property
    def trainable(self):
        return self._trainable

    @trainable.setter
    def trainable(self, value):
        self._trainable = bool(value)
        if not value and self._assigned is not None and self._node.op == 'sepconv':
            backend.freeze_separable(self._node, self._assigned)

    _trainable, _assigned = True, None


class BatchNormalization(Layer):
    _has_weights = True
    _spatial = True

    def __init__(self, axis=-1, momentum=0.99, epsilon=1e-3, center=True, scale=True, name=None, **kwargs):
        Layer.__init__(self, name, **{k: v for k, v in kwargs.items() if not k.endswith(('_initializer', '_regularizer',
                                                                                           '_constraint'))})
        _no(axis not in (-1, 3), 'BatchNormalization over an axis other than channels')
        _no(not center, 'BatchNormalization(center=False)')
        if abs(float(epsilon) - 1e-3) > 1e-12:
            raise NotImplementedError('BatchNormalization: epsilon is fixed at the Keras default 1e-3 (got %r)' % epsilon)
        self.scale = bool(scale)

    def call(self, x):
        return L.BatchNormalization(x, scale=self.scale, name=self.name)


class Activation(Layer):
    """Activation('relu' | 'sigmoid' | 'softmax'), or Activation(function): the function is run on the symbolic tensor
    (`Activation(channel_softmax_2d(alpha=...))`, deephar/activations.py:3-16) and must come out as a known op."""

    def __init__(self, activation, name=None, **kwargs):
        Layer.__init__(self, name, **kwargs)
        if not callable(activation) and activation not in ('relu', 'sigmoid', 'softmax'):
            raise NotImplementedError('Activation(%r): the reference models use relu / sigmoid / softmax and the '
                                      'helpers channel_softmax_2d(...)' % (activation,))
        self.activation = activation

    def call(self, x):
        if callable(self.activation):
            out = self.activation(x)
            if not isinstance(out, Tensor):
                raise NotImplementedError('Activation(function): the function did not return a tensor')
            if backend.is_raw(out):
                out.node.attrs['name'] = self.name
            return out
        if backend.is_raw(x):
            if self.activation != 'relu':
                return backend.activation(x, self.activation, name=self.name)
            x = _as_image(x)                    # relu of e.g. a max+min pooling: a map again
        if self.activation == 'softmax' and x.kind != 'frame':
            return L.softmax_lastaxis(x, name=self.name)
        return L.Activation(x, self.activation, name=self.name)


class MaxPooling2D(Layer):
    _spatial = True

    def __init__(self, pool_size=(2, 2), strides=None, padding='valid', data_format=None, name=None, **kwargs):
        Layer.__init__(self, name, **kwargs)
        self.pool_size, self.strides, self.padding = pool_size, strides, padding

    def call(self, x):
        return L.MaxPooling2D(x, self.pool_size, self.strides, self.padding, name=self.name)


class UpSampling2D(Layer):
    _spatial = True

    def __init__(self, size=(2, 2), data_format=None, name=None, **kwargs):
        Layer.__init__(self, name, **kwargs)
        self.size = size

    def call(self, x):
        return L.UpSampling2D(x, self.size, name=self.name)


class ZeroPadding2D(Layer):
    _spatial = True

    def __init__(self, padding=(1, 1), data_format=None, name=None, **kwargs):
        Layer.__init__(self, name, **kwargs)
        if isinstance(padding, int):
            padding = ((padding, padding), (padding, padding))
        elif isinstance(padding[0], int):
            padding = ((padding[0], padding[0]), (padding[1], padding[1]))
        self.padding = tuple(tuple(p) for p in padding)

    def call(self, x):
        return L.ZeroPadding2D(x, self.padding)


class AveragePooling2D(Layer):
    """Only inside the joint-confidence construction (layers.py:111-115): recorded as a backend op."""

    def __init__(self, pool_size=(2, 2), strides=None, padding='valid', data_format=None, name=None, **kwargs):
        Layer.__init__(self, name, **kwargs)
        self.pool_size = L._pair(pool_size)
        self.strides = self.pool_size if strides is None else L._pair(strides)
        self.padding = padding

    def call(self, x):
        return backend.average_pooling_2d(x, self.pool_size, self.strides, self.padding)


class GlobalMaxPooling2D(Layer):
    def __init__(self, data_format=None, name=None, **kwargs):
        Layer.__init__(self, name, **kwargs)

    def call(self, x):
        return backend.global_max_pooling_2d(x)


class GlobalMaxPooling1D(Layer):
    def __init__(self, name=None, **kwargs):
        Layer.__init__(self, name, **kwargs)

    def call(self, x):
        return backend.global_max_pooling_1d(x)


class Lambda(Layer):
    """keras.layers.Lambda.  The body runs on the symbolic tensor(s): a slice of the channel axis
    (`Lambda(lambda x: x[:,:,:,:num_joints])`, reception.py:171-172) is a view; arithmetic and `keras.backend` calls
    (`K.tile`, `K.sum`, `4 * AveragePooling2D(...)(x)`, ...) record backend-op nodes (keras_trace.py) which must add up
    to one of the reference's parameter-free constructions when the model is built -- any other body is rejected then,
    naming the ops.  Indexing other than a channel slice is rejected here."""

    def __init__(self, function, name=None, **kwargs):
        Layer.__init__(self, name, **{k: v for k, v in kwargs.items() if k not in ('output_shape', 'arguments', 'mask')})
        self.function = function

    def call(self, x):
        try:
            out = self.function(list(x) if isinstance(x, (list, tuple)) else x)
        except NotImplementedError:
            raise
        except (TypeError, AttributeError, IndexError) as e:            # Python / numpy arithmetic on a symbolic tensor
            raise NotImplementedError('Lambda: the body cannot be recorded (%s: %s)' % (type(e).__name__, e))
        if not isinstance(out, Tensor):
            raise NotImplementedError('Lambda: the body did not return a tensor')
        if backend.is_raw(out) and self.name is not None:
            out.node.attrs['name'] = self.name
        return out


class TimeDistributed(Layer):
    """keras.layers.TimeDistributed: frames already sit on the batch axis, so the wrapper only hands its name down
    (a wrapped nested Model keeps its own name: its weights live under that scope)."""

    def __init__(self, layer, name=None, **kwargs):
        Layer.__init__(self, name, **kwargs)
        self.layer = layer
        if name is not None and isinstance(layer, Layer):
            layer.name = name

    def call(self, x):
        _TD_DEPTH[0] += 1
        try:
            return self.layer(x)
        finally:
            _TD_DEPTH[0] -= 1


class _Merge(Layer):
    fn = None
    raw = None

    def call(self, ts):
        ts = list(ts)
        backend.unify(ts)
        if any(backend.is_raw(t) for t in ts):
            if self.raw is None:
                raise NotImplementedError('%s of a backend-op result' % type(self).__name__)
            return backend.merge(self.raw, ts, name=self.name)
        return type(self).fn(ts, name=self.name)


class Add(_Merge):
    fn = staticmethod(L.add)
    raw = 'add'


class Concatenate(_Merge):
    fn = staticmethod(L.concatenate)
    raw = 'concat'

    def __init__(self, axis=-1, name=None, **kwargs):
        _Merge.__init__(self, name, **kwargs)
        _no(axis != -1, 'concatenation over an axis other than channels')


class Multiply(_Merge):
    fn = staticmethod(L.multiply)
    raw = 'multiply'


def add(inputs, name=None):
    return Add(name=name)(inputs)


def concatenate(inputs, axis=-1, name=None):
    return Concatenate(axis=axis, name=name)(inputs)


def multiply(inputs, name=None):
    return Multiply(name=name)(inputs)


# ---------------------------------------------------------------------------------------------------------------------
# The reference's parameter-free head models (deephar/models/blocks.py:217-343).  In Keras they are small sub-models of
# Lambda / pooling / frozen Dense and SeparableConv2D layers; here each is ONE recordable object, and the combination the
# builders make of them (reception.py:167-190) is rewritten into the single fused graph op the kernels implement.
# ---------------------------------------------------------------------------------------------------------------------
class _Head(object):
    def __init__(self, kind, name=None, **attrs):
        self.kind, self.name, self.attrs = kind, name, attrs
        self.trainable = False

    def __call__(self, x):
        xs = list(x) if isinstance(x, (list, tuple)) else [x]
        backend.unify(xs)
        if self.name is not None:
            xs[0].g.layers.setdefault(self.name, self)
        ks = backend.kshape(xs[0])
        if self.kind == 'sam2d':
            shape = ks[:-3] + (ks[-1], 2)
        elif self.kind == 'jprob':
            shape = ks[:-3] + (ks[-1], 1)
        elif self.kind == 'sam1d':
            shape = ks[:-2] + (ks[-1], 1)
        else:
            shape = ks[:-2] + (self.attrs['num_joints'], 2)
        return xs[0].g.op('head_' + self.kind, xs, [shape], dict(self.attrs, name=self.name), kind='raw')


def build_softargmax_2d(input_shape, rho=0., name=None):
    """blocks.py:306-325: channel softmax + the two linear interpolations = soft-argmax of every map -> (C, 2)."""
    _no(rho > 0, 'kl_divergence_regularizer (rho > 0)')
    return _Head('sam2d', name)


def build_joints_probability(input_shape, name=None, verbose=0):
    """blocks.py:328-343: 4 * AveragePooling2D((2,2), strides 1) -> GlobalMaxPooling2D on the raw maps -> (C, 1)."""
    return _Head('jprob', name)


def build_context_aggregation(num_joints, num_context, alpha, num_frames=1, name=None):
    """blocks.py:217-285: pose = alpha * ys + (1 - alpha) * sum(pc * yc) / sum(pc) over each joint's context maps."""
    return _Head('agg', name, num_joints=int(num_joints), num_context=int(num_context), alpha=float(alpha))


def build_softargmax_1d(input_shape, name=None):
    """blocks.py:288-303 (zSAM of the 3-D head).  Built by reception.build for every model, only CALLED for dim = 3."""
    return _Head('sam1d', name)


def _weight_names(attrs, known):
    """(path in attrs, weight name) for every attribute value that names a weight of the recorded graph."""
    for key, val in attrs.items():
        if isinstance(val, str) and val in known:
            yield (key, None), val
        elif isinstance(val, dict):
            for k2, v2 in val.items():
                if isinstance(v2, str) and v2 in known:
                    yield (key, k2), v2


class Model(object):
    """keras.models.Model(inputs, outputs, name).

    * used as a MODEL (`predict`, `load_weights`, `weight_specs`, `output_shape`, ...): the recorded graph is compiled
      for H100 on first use (layers that reach no output are dropped, as Keras drops them) and every attribute of
      deephar_b200.model.Model is available on this object.  `model.input` / `model.outputs` are the symbolic tensors, so
      `Model(full.input, full.outputs[:n])` (deephar/models/spnet.py:443-446) makes a model of a subset of the outputs;
    * used as a LAYER -- `Stem = Model(inp, x, name='Stem'); y = Stem(frames)`, the way the reference wraps its blocks
      (deephar/models/reception.py:96-98, 128-131) -- its layers are re-recorded into the caller's graph under the
      scope `name`, which is how Keras names the weights of a nested model in a checkpoint ("Stem/conv2d_1/kernel");
      layers that already carry the scope of an inner sub-model keep it (one scope per weight: Keras layer names are
      unique per session).  A nested model is applied once per graph (no weight sharing inside one model); applying it
      again in ANOTHER model -- `TimeDistributed(model_pe.get_layer('Stem'))(clips)`, action.py:117-125 -- records the
      same layers, with the same weight names, there.  Models with several Inputs can be nested (`model_pose([y, p])`,
      action.py:354) but not compiled on their own.
    """

    _OWN = ('_impl', '_applied_to', '_graph', '_inputs', '_outputs', '_single', '_name', 'trainable', '_fetched_from')

    def __init__(self, inputs=None, outputs=None, name=None):
        self._inputs = list(inputs) if isinstance(inputs, (list, tuple)) else [inputs]
        self._outputs = list(outputs) if isinstance(outputs, (list, tuple)) else [outputs]
        self._single = not isinstance(outputs, (list, tuple))
        g = backend.unify(self._inputs + self._outputs)
        if any(t not in g.inputs for t in self._inputs):
            raise ValueError('Model: `inputs` must be Input tensors')
        if len(set(id(t) for t in self._inputs)) != len(g.inputs):
            raise ValueError('Model: the outputs depend on an Input that is not listed in `inputs`')
        self._graph = g
        self._name = name or g.auto_name('model')
        self._impl = None
        self._applied_to = []
        self.trainable = True

    name = property(lambda self: self._name)
    input = property(lambda self: self._inputs[0] if len(self._inputs) == 1 else list(self._inputs))
    inputs = property(lambda self: list(self._inputs))
    output = property(lambda self: self._outputs[0] if len(self._outputs) == 1 else list(self._outputs))
    outputs = property(lambda self: list(self._outputs))

    def get_layer(self, name=None, index=None):
        """The nested sub-model / parameter-free head model applied in this model under `name`."""
        if name is None or name not in self._graph.layers:
            raise ValueError('No such layer: %s' % (name,))
        layer = self._graph.layers[name]
        if isinstance(layer, Model):
            layer._fetched_from = self          # Keras shares the layer objects: weights already loaded here go along
        return layer

    def summary(self, *args, **kwargs):
        if not self._applied_to and len(self._inputs) == 1:
            self._compiled().summary(*args, **kwargs)

    # ---- as a model ---------------------------------------------------------------------------------------------
    def _compiled(self):
        if self._impl is None:
            if self._applied_to:
                raise NotImplementedError('Model %r was applied as a layer of another model; compile that one' % self._name)
            if len(self._inputs) != 1:
                raise NotImplementedError('Model %r: a model with several Inputs can only be used inside another model'
                                          % self._name)
            # a model of SOME outputs of a model that is already compiled (spnet.split_model after build + load_weights,
            # eval_penn_multitask.py:66-81) is a view of that network: same weights, same buffers
            for outs_full, impl in getattr(self._graph, 'compiled', []):
                where = [next((i for i, o in enumerate(outs_full) if o is t), None) for t in self._outputs]
                if None not in where:
                    self._impl = impl.output_subset(where, name=self._name)
                    return self._impl
            g, outs = backend.rewrite(self._graph, self._outputs)
            g.outputs = outs
            g.name = self._name
            self._impl = _Model(g, name=self._name)
            # Keras models share their layer OBJECTS, so weights already loaded into one model are the weights of every
            # model made of the same layers: sub-models fetched with get_layer() from `src` (action.py:117-125), and new
            # outputs built on the tensors of a model that is already loaded (eval_h36m.py:48-59 concatenates pose and
            # visibility per block AFTER load_weights).  Carried over once, when this model is compiled.
            mine = set(n for n, _ in self._impl.weight_specs)
            donors = [src._impl for src in getattr(self._graph, 'shares_with', []) if src._impl is not None]
            donors += [impl for _, impl in getattr(self._graph, 'compiled', [])]
            shared = {}
            for impl in donors:
                held = getattr(impl, '_host_weights', None)
                if held:
                    shared.update({n: w for n, w in held.items() if n in mine and n not in shared})
            if shared:
                self._impl._backbone_weights = shared
                optional = set(self._impl.optional_weights)
                if all(n in shared or n in optional for n in mine):      # nothing new to load: the model is ready
                    self._impl.set_weights(shared)
            if not hasattr(self._graph, 'compiled'):
                self._graph.compiled = []
            self._graph.compiled.append((list(self._outputs), self._impl))
        return self._impl

    def __getattr__(self, attr):
        # only reached for names this wrapper does not define: everything else is the compiled model's
        if attr.startswith('__') or attr in Model._OWN:
            raise AttributeError(attr)
        return getattr(self._compiled(), attr)

    # ---- as a layer ---------------------------------------------------------------------------------------------
    def __call__(self, x):
        xs = list(x) if isinstance(x, (list, tuple)) else [x]
        if self._impl is not None:
            raise NotImplementedError('Model %r was already compiled as a model of its own' % self._name)
        if len(xs) != len(self._inputs):
            raise ValueError('Model %r expects %d input(s), got %d' % (self._name, len(self._inputs), len(xs)))
        sub, tgt = self._graph, backend.unify(xs)
        if tgt is sub:
            raise ValueError('Model %r applied to a tensor of its own graph' % self._name)
        if any(g is tgt for g in self._applied_to):
            raise NotImplementedError('Model %r: a nested model is applied once per model (no weight sharing on the '
                                      "reference's forward path)" % self._name)
        per_frame = _TD_DEPTH[0] > 0
        if any(nd.outs[0].kind == 'raw' for nd in sub.nodes) and per_frame and tgt.frames_per_clip != sub.frames_per_clip:
            raise NotImplementedError('Model %r holds backend arithmetic and is applied under TimeDistributed' % self._name)
        new = {}
        for x, src_in in zip(xs, self._inputs):
            x = _as_image(x)            # per-joint tensors (None, T, joints, c): (T, joints) is the image of the sub-model
            if tuple(x.shape) != tuple(src_in.shape):
                raise ValueError('Model %r expects input shape %s, got %s' % (self._name, src_in.shape, x.shape))
            new[src_in.id] = x
        kind = new[self._inputs[0].id].kind
        self._applied_to.append(tgt)
        tgt.layers.setdefault(self._name, self)
        if getattr(self, '_fetched_from', None) is not None:
            if not hasattr(tgt, 'shares_with'):
                tgt.shares_with = []
            if all(m is not self._fetched_from for m in tgt.shares_with):
                tgt.shares_with.append(self._fetched_from)

        prefix = tgt.qualify(self._name)
        scoped = lambda n, parts: n if n.count('/') >= parts else prefix + '/' + n      # noqa: E731
        known = {}
        for wname, shape in sub.weight_specs:                        # creation order is kept
            layer, leaf = wname.rsplit('/', 1)
            known[wname] = tgt.add_weight(scoped(layer, 1), leaf, shape)
        for nd in sub.nodes:
            if nd.op == 'input':
                continue
            attrs = {}
            for k, v in nd.attrs.items():
                attrs[k] = dict(v) if isinstance(v, dict) else v
            touched = list(_weight_names(nd.attrs, known))
            if touched and isinstance(attrs.get('name'), str):
                attrs['name'] = scoped(attrs['name'], 1)
            for (k1, k2), w in touched:
                if k2 is None:
                    attrs[k1] = known[w]
                else:
                    attrs[k1][k2] = known[w]
            outs = tgt.op(nd.op, [new[t.id] for t in nd.inputs], [o.shape for o in nd.outs], attrs,
                          kind=kind if nd.outs[0].kind == 'frame' else nd.outs[0].kind)
            outs = outs if isinstance(outs, tuple) else (outs,)
            for o_src, o_new in zip(nd.outs, outs):
                new[o_src.id] = o_new
        res = [new[t.id] for t in self._outputs]
        return res[0] if self._single else res
