"""Symbolic layer graph recorded by the model builders (deephar_b200/reception.py,
spnet.py).  It plays the role of the Keras functional graph in the reference: the
builders call Keras-like layer helpers (deephar_b200/layers.py) on `Tensor`s; nothing is
computed here.  compiler.py turns the graph into fused sm_90a kernel launches.

Tensor shapes are per-item NHWC without the batch axis: (H, W, C).  `kind` says which
batch axis the tensor lives on: 'frame' (N = B*T frames; TimeDistributed in the reference
folds T into the batch, layers.py:66-104) or 'clip' (B clips; the action head treats
(T, joints) as an image, spnet.py:109-146).
"""


def _trace():
    from . import keras_trace
    return keras_trace


class Tensor(object):
    __slots__ = ('g', 'id', 'shape', 'kind', 'node', 'out_index')

    def __init__(self, g, shape, kind, node, out_index=0):
        self.g = g
        self.id = len(g.tensors)
        self.shape = tuple(int(s) for s in shape)
        self.kind = kind
        self.node = node
        self.out_index = out_index
        g.tensors.append(self)

    @property
    def channels(self):
        return self.shape[-1]

    def __repr__(self):
        return 'T%d%s<%s>' % (self.id, self.shape, self.node.op if self.node else 'input')

    # Arithmetic and indexing exist for the bodies of `Lambda` layers in Keras-style model code: each records a
    # backend-op node (keras_trace.py) that the front end rewrites into a fused layer op, or rejects, at build time.
    def __mul__(self, o):
        return _trace().arith('mul', self, o)

    def __rmul__(self, o):
        return _trace().arith('mul', self, o)

    def __sub__(self, o):
        return _trace().arith('sub', self, o)

    def __truediv__(self, o):
        return _trace().arith('div', self, o)

    def __neg__(self):
        return _trace().neg(self)

    def __getitem__(self, idx):
        return _trace().getitem(self, idx)

    __hash__ = object.__hash__


class Node(object):
    __slots__ = ('id', 'op', 'inputs', 'outs', 'attrs')

    def __init__(self, g, op, inputs, attrs):
        self.id = len(g.nodes)
        self.op = op
        self.inputs = list(inputs)
        self.outs = []
        self.attrs = attrs
        g.nodes.append(self)

    @property
    def out(self):
        return self.outs[0]

    def __repr__(self):
        return 'N%d:%s' % (self.id, self.op)


class Graph(object):
    def __init__(self, name='model'):
        self.name = name
        self.nodes = []
        self.tensors = []
        self.inputs = []
        self.outputs = []
        self.output_names = []
        self.weight_specs = []      # ordered [(name, shape)] in layer-creation order
        self._weight_names = set()
        self._counters = {}
        self._scope = []
        self.frames_per_clip = 1    # T (TimeDistributed fold); 1 for single-frame models
        self.layers = {}            # name -> sub-model / head model applied in this graph (keras `get_layer`)

    # --- naming (Keras auto names: one global counter per class prefix) --------
    def auto_name(self, prefix):
        n = self._counters.get(prefix, 0) + 1
        self._counters[prefix] = n
        return '%s_%d' % (prefix, n)

    def scope(self, name):
        g = self

        class _Scope(object):
            def __enter__(self_):
                g._scope.append(name)

            def __exit__(self_, *a):
                g._scope.pop()

        return _Scope()

    def qualify(self, layer):
        return '/'.join(self._scope + [layer])

    def add_weight(self, layer_qualified, leaf, shape):
        name = layer_qualified + '/' + leaf
        if name in self._weight_names:
            raise ValueError('duplicate weight name %s' % name)
        self._weight_names.add(name)
        self.weight_specs.append((name, tuple(int(s) for s in shape)))
        return name

    # --- graph construction --------------------------------------------------
    def input(self, shape, kind='frame'):
        node = Node(self, 'input', [], {})
        t = Tensor(self, shape, kind, node)
        node.outs.append(t)
        self.inputs.append(t)
        return t

    def op(self, op, inputs, out_shapes, attrs=None, kind=None):
        node = Node(self, op, inputs, attrs or {})
        kind = kind or inputs[0].kind
        if out_shapes and not isinstance(out_shapes[0], (tuple, list)):
            out_shapes = [out_shapes]
        for i, s in enumerate(out_shapes):
            node.outs.append(Tensor(self, s, kind, node, i))
        return node.outs[0] if len(node.outs) == 1 else tuple(node.outs)

    def absorb(self, other):
        """Move every node, tensor, input and weight of `other` into this graph (Keras Inputs are independent; a model
        with several of them becomes one graph the first time an op combines their tensors).  `other` is left empty."""
        if other is self:
            return
        for nd in other.nodes:
            nd.id = len(self.nodes)
            self.nodes.append(nd)
        for t in other.tensors:
            t.id = len(self.tensors)
            t.g = self
            self.tensors.append(t)
        self.inputs.extend(other.inputs)
        for name, shape in other.weight_specs:
            if name in self._weight_names:
                raise ValueError('duplicate weight name %s' % name)
            self._weight_names.add(name)
            self.weight_specs.append((name, shape))
        for k, v in getattr(other, 'layers', {}).items():
            self.layers.setdefault(k, v)
        other.nodes, other.tensors, other.inputs, other.weight_specs = [], [], [], []
        other._weight_names = set()
        other.merged_into = self

    def signatures(self, tensors=None):
        """One digest per tensor (default: the outputs) of the expression that computes it: op, attributes (weight and
        layer names included), operand digests, shapes.  Two graphs whose outputs have equal digests are the same
        function of the same weights, whatever order their nodes were recorded in."""
        import hashlib
        memo = {}

        def canon(v):
            if isinstance(v, dict):
                return tuple(sorted((k, canon(x)) for k, x in v.items()))
            if isinstance(v, (list, tuple)):
                return tuple(canon(x) for x in v)
            return v

        def sig(t):
            if t.id not in memo:
                nd = t.node
                attrs = nd.attrs
                if nd.op in ('conv', 'sepconv') and tuple(attrs['size']) == (1, 1) and tuple(attrs['strides']) == (1, 1):
                    attrs = dict(attrs, padding='same')         # a 1x1 / stride-1 window needs no padding either way
                body = repr((nd.op, canon(attrs), [sig(i) for i in nd.inputs], t.out_index, t.shape, t.kind))
                memo[t.id] = hashlib.sha1(body.encode()).hexdigest()
            return memo[t.id]

        import sys
        limit = sys.getrecursionlimit()
        sys.setrecursionlimit(max(limit, 20000))
        try:
            return [sig(t) for t in (self.outputs if tensors is None else tensors)]
        finally:
            sys.setrecursionlimit(limit)

    def num_params(self):
        n = 0
        for _, s in self.weight_specs:
            k = 1
            for d in s:
                k *= d
            n += k
        return n


def same_pad(in_size, k, s):
    """TF 'SAME': out = ceil(in/s); extra pad on bottom/right (SURVEY.md App. A)."""
    out = -(-in_size // s)
    total = max((out - 1) * s + k - in_size, 0)
    return out, total // 2, total - total // 2


def conv_out_hw(h, w, size, strides, padding):
    if padding == 'same':
        return same_pad(h, size[0], strides[0])[0], same_pad(w, size[1], strides[1])[0]
    if padding == 'valid':
        return (h - size[0]) // strides[0] + 1, (w - size[1]) // strides[1] + 1
    raise ValueError('padding must be "same" or "valid", got %r' % (padding,))
