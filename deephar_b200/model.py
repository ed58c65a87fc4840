"""keras.Model-like object over a compiled deephar_b200 graph.

Protocol kept for the reference's evaluators (exp/common/mpii_tools.py:63-90,
h36m_tools.py:12-50, penn_tools.py:13-60): `.predict(x, batch_size, verbose)` returning a
list of numpy arrays (a single array if the model has one output), `.outputs`,
`.input_shape`, `.get_input_shape_at(0)`, `.name`, `.load_weights`, `.set_weights`.

PyTorch is used only as the device-memory / stream container; every FLOP runs in
libdeephar_b200.so.  There is no CPU path: constructing the engine without a CUDA device
raises.
"""
import ctypes as C

import numpy as np

from . import _ffi
from .compiler import compile_graph
from .weights import fold_batchnorm, load_calibration, synthetic_weights


def _align(n, a=4):
    return (n + a - 1) // a * a


def _weight_key(k):
    """the weight a conv / sepconv op's packed tensor-core operand is made from: its kernel, or its pointwise kernel"""
    return k.attrs['kernel'] if k.kind == 'conv' else k.attrs['pointwise']


def _conv_macs(k):
    """multiply-adds of a conv / sepconv op per item"""
    ho, wo, cout = k.outs[0].shape
    cin = k.ins[0].shape[2]
    kh, kw = k.attrs['size']
    return ho * wo * (kh * kw * cin * cout if k.kind == 'conv' else kh * kw * cin + cin * cout)


def _item_dims(t):
    """a tensor's per-item (H, W, C) as the Keras shapes here trim it: (C,) when H = W = 1, (W, C) when H = 1"""
    h, w, c = t.shape
    if h == 1 and w == 1:
        return (c,)
    if h == 1:
        return (w, c)
    return (h, w, c)


def _graphed(use_graph, graph, uses, issue):
    """issue(stream) on torch's current stream, under the CUDA-graph policy of a forward and of a push: plain launches
    on the first use (which also warm every kernel up), captured into a CUDA graph on the second, replayed after that;
    plain launches every time without use_graph.  Returns the (graph, uses) to keep for the next call: with use_graph,
    a graph that is not None was replayed."""
    import torch
    if not use_graph:
        issue(torch.cuda.current_stream().cuda_stream)
        return graph, uses
    if graph is None:
        uses += 1
        if uses < 2:
            issue(torch.cuda.current_stream().cuda_stream)
            return None, uses
        graph = torch.cuda.CUDAGraph()
        torch.cuda.synchronize()
        with torch.cuda.graph(graph):
            issue(torch.cuda.current_stream().cuda_stream)
    graph.replay()
    return graph, uses


class _Bound(object):
    """A plan bound to a batch size: its activation slots and workspace, the ctypes argument list of every launch
    (`calls`: (kind, function, ctx, args ...) tuples), and the model settings it was bound with."""

    def __init__(self, model, plan, n_items, packed):
        # no reference to the model: a model's bindings are released with it, not by the cycle collector
        self.plan, self.n_items, self.ctx = plan, n_items, model._ctx
        self.items = {kind: model._items(kind, n_items) for kind in ('frame', 'clip')}
        self.precision, self.use_tensor_cores = model.precision, model.use_tensor_cores
        self.packed = packed        # the convolutions get the packed bf16 operands (else NULL: CUDA-core kernels only)
        self.calls = []
        self.keep = []
        self.slots = []
        self.conv_plans = []        # (conv / sepconv op, its dh_conv_plan_info): the library's kernel choice at bind
        self.graph, self.uses = None, 0

    def current(self, model):
        """made with the model's current precision and use_tensor_cores"""
        return (self.precision, self.use_tensor_cores) == (model.precision, model.use_tensor_cores)

    def view(self, t):
        """the dh_view of plan tensor t"""
        s = self.plan.storage[t.id]
        return _ffi.dh_view(self.slots[s.buf.phys].data_ptr() + 4 * s.c_off, self.items[t.kind], t.shape[0],
                            t.shape[1], t.shape[2], s.ld)

    def tensor(self, t):
        """plan tensor t as a device tensor (items, H * W, C): a view into its slot"""
        s = self.plan.storage[t.id]
        base = self.slots[s.buf.phys].view(self.items[t.kind], s.buf.hw, s.ld)
        return base[:, :, s.c_off:s.c_off + t.shape[2]]

    def issue(self, stream_ptr, events=None):
        """Every launch, in order, on stream stream_ptr.  events: a list that receives a pair of timing CUDA events
        recorded around each launch."""
        self.ctx.set_workspace(self.workspace.data_ptr(), self.workspace.numel() * 4)
        for call in self.calls:
            if events is not None:
                import torch
                events.append((torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)))
                events[-1][0].record()
            rc = call[1](*call[2:], stream_ptr)
            if events is not None:
                events[-1][1].record()
            if rc != 0:
                _ffi.check(rc, call[0])


class Model(object):
    def __init__(self, graph, calib_key=None, name=None):
        self.graph = graph
        self.name = name or graph.name
        self.plan = compile_graph(graph)
        self.calib_key = calib_key
        self.weight_specs = list(graph.weight_specs)
        # Weights of layers the builders create but whose outputs never reach a model output (e.g. the
        # re-injection convs after the LAST prediction block, spnet.py:249-262).  keras.Model drops such
        # layers, so the reference's checkpoints do not contain them: they are optional when loading.
        live = set()
        stack = [t.node for t in graph.outputs]
        seen = set()
        while stack:
            nd = stack.pop()
            if nd is None or nd.id in seen:
                continue
            seen.add(nd.id)
            if 'name' in nd.attrs:
                live.add(nd.attrs['name'])
            stack.extend(t.node for t in nd.inputs)
        self.optional_weights = [n for n, _ in self.weight_specs if n.rsplit('/', 1)[0] not in live]
        self._host_weights = None
        self._dev = None            # device-side weight arena (torch tensor) + pointer table
        self._packed_info = None    # weight -> its packed tensor-core operands (built on first need), in _dev_packed
        self._dev_packed = None
        self._ptr = {}
        self._ctx = None
        self._bound = {}
        self.precision = 3          # tensor-core split precision (bf16 x3 ~ fp32); 1 = plain bf16
        self.use_tensor_cores = True
        # One forward is 150-350 kernel launches issued through ctypes (~4 us each on the host): at small batches
        # (C1: one frame; the 64-frames-per-GPU strong-scaling point) the GPU would wait for the host.  The launch
        # sequence of a bound batch size is therefore captured ONCE into a CUDA graph and replayed.
        self.use_cuda_graph = True
        self.max_bound = 2          # bound batch sizes kept alive (LRU): each holds a full activation arena

    # ---- keras.Model protocol ------------------------------------------------------
    @property
    def outputs(self):
        return list(self.graph.outputs)

    @property
    def input_shape(self):
        t = self.graph.inputs[0]
        if self.graph.frames_per_clip > 1:
            return (None, self.graph.frames_per_clip) + t.shape
        return (None,) + t.shape

    def get_input_shape_at(self, i):
        assert i == 0
        return self.input_shape

    @property
    def output_shape(self):
        return [self._keras_shape(t, None) for t in self.graph.outputs]

    def count_params(self):
        return self.graph.num_params()

    def summary(self, line_length=None, positions=None, print_fn=None):
        """keras.Model.summary (exp/ntu/predict_bboxes.py:45): what this model is on the H100 -- layer scopes with their
        parameter counts, then the compiled plan."""
        out = print_fn or print
        out('Model %r on deephar_b200: input %s, %d outputs' % (self.name, self.input_shape, len(self.graph.outputs)))
        scopes = {}
        for name, shape in self.weight_specs:
            scope = name.split('/')[0]
            scopes[scope] = scopes.get(scope, 0) + int(np.prod(shape))
        for scope, n in scopes.items():
            out('  %-40s %12d' % (scope, n))
        kinds = {}
        for k in self.plan.kops:
            kinds[k.kind] = kinds.get(k.kind, 0) + 1
        out('Total params: %d in %d weights' % (self.count_params(), len(self.weight_specs)))
        out('Plan: %d kernel launches per forward (%s); %.2f GFLOP per frame; %d activation buffers in %d slots'
            % (len(self.plan.kops), ', '.join('%d %s' % (n, kd) for kd, n in sorted(kinds.items(), key=lambda kv: -kv[1])),
               self.conv_flops_per_frame() / 1e9, self.plan.stats['buffers'], self.plan.stats['phys_slots']))

    def compile(self, *args, **kwargs):
        raise NotImplementedError('deephar_b200 builds the forward (inference) path; training stays with the reference')

    fit = fit_generator = compile

    def conv_flops_per_frame(self):
        """2 x MAC of every Conv2D / SeparableConv2D per input frame (SURVEY.md 8d); clip-level
        (action head) convs are divided by the frames per clip."""
        total = 0.0
        for k in self.plan.kops:
            if k.kind not in ('conv', 'sepconv'):
                continue
            mac = _conv_macs(k)
            if k.outs[0].kind == 'clip':
                mac /= float(self.graph.frames_per_clip)
            total += 2.0 * mac
        return total

    # ---- weights -----------------------------------------------------------------
    def set_weights(self, table):
        """table: {name: array} in the Keras layouts listed by `weight_specs`."""
        host = {}
        optional = set(self.optional_weights)
        for name, shape in self.weight_specs:
            if name not in table:
                if name in optional:                    # dead layer: absent from reference checkpoints
                    host[name] = np.zeros(shape, dtype=np.float32)
                    continue
                raise KeyError('missing weight %s %s' % (name, shape))
            a = np.asarray(table[name], dtype=np.float32)
            if tuple(a.shape) != tuple(shape):
                raise ValueError('weight %s has shape %s, expected %s' % (name, a.shape, shape))
            host[name] = a
        self._host_weights = host
        self._dev = None
        self._bound = {}

    def get_weights(self):
        return dict(self._host_weights)

    def init_synthetic_weights(self, seed=1234):
        calib = load_calibration(self.calib_key) if self.calib_key else {}
        table = synthetic_weights(self.weight_specs, seed, calib)
        table.update(getattr(self, '_backbone_weights', {}))     # layers shared with another model
        self.set_weights(table)
        return self

    def load_weights(self, path, by_name=False):
        """keras.Model.load_weights: a Keras HDF5 weight file (`save_weights` / `save` output, read by
        the pure-Python reader in hdf5.py / keras_h5.py -- the call every reference evaluator makes:
        eval_mpii_singleperson.py:54, eval_h36m.py:53, eval_penn_multitask.py:76) or an .npz written by
        `save_weights` here.  by_name=False requires every (non-optional) weight of the model to be in
        the file; by_name=True loads the layers whose names match and keeps the rest."""
        path = str(path)
        if path.endswith(('.h5', '.hdf5', '.keras')):
            from . import keras_h5
            table, unused = keras_h5.load(path, self.weight_specs, self.optional_weights, by_name=by_name)
            self.unused_file_weights = unused
        else:
            with np.load(path) as z:
                table = {k: z[k] for k in z.files}
            known = set(n for n, _ in self.weight_specs)
            self.unused_file_weights = [k for k in table if k not in known]
            table = {k: v for k, v in table.items() if k in known}
        if by_name:                 # layers the file does not name keep what they hold: weights set earlier, or the
            merged = dict(getattr(self, '_backbone_weights', None) or {})      # ones shared with a model loaded before
            merged.update(self._host_weights or {})
            merged.update(table)
            table = merged
        self.set_weights(table)

    def save_weights(self, path):
        """Keras-layout HDF5 for '*.h5' (loadable by keras.Model.load_weights of the reference), else .npz."""
        path = str(path)
        if path.endswith(('.h5', '.hdf5', '.keras')):
            from . import keras_h5
            keras_h5.save(path, self.weight_specs, self._host_weights)
        else:
            np.savez(path, **self._host_weights)

    # ---- engine --------------------------------------------------------------------
    def _torch(self):
        import torch
        if not torch.cuda.is_available():
            raise _ffi.DeepharB200Error('deephar_b200 needs a CUDA device (B200, sm_100a); '
                                        'there is no CPU fallback')
        return torch

    def _ensure_device_weights(self):
        if self._dev is not None:
            return
        torch = self._torch()
        if self._host_weights is None:
            raise RuntimeError('weights not set: call load_weights / set_weights / init_synthetic_weights')
        if self._ctx is None:
            self._ctx = _ffi.Context(torch.cuda.current_device())
        hw = self._host_weights
        chunks, offsets, off = [], {}, 0

        def put(key, arr):
            nonlocal off
            arr = np.ascontiguousarray(arr, dtype=np.float32).ravel()
            offsets[key] = off
            chunks.append(arr)
            pad = _align(arr.size) - arr.size
            if pad:
                chunks.append(np.zeros(pad, np.float32))
            off += _align(arr.size)

        for name, _ in self.weight_specs:
            put(name, hw[name])
        for k in self.plan.kops:
            for key in ('pre_bn', 'post_bn', 'bn'):
                bn = k.attrs.get(key) if isinstance(k.attrs, dict) else None
                if bn and ('fold:' + bn['name']) not in offsets:
                    w = bn['weights']
                    scale, shift = fold_batchnorm(hw[w['gamma']] if 'gamma' in w else None,
                                                  hw[w['beta']], hw[w['mean']], hw[w['var']])
                    put('fold:' + bn['name'], scale)
                    put('shift:' + bn['name'], shift)
        scales = [k for k in self.plan.kops if k.kind == 'scale']     # per-channel constant vectors
        if scales:
            cmax = max(4, max(k.ins[0].shape[2] for k in scales))
            for val in sorted(set([0.0] + [float(k.attrs['value']) for k in scales])):
                put('const:%r' % val, np.full(cmax, val, np.float32))
        flat = np.concatenate(chunks) if chunks else np.zeros(4, np.float32)
        self._dev = torch.from_numpy(flat).cuda()
        base = self._dev.data_ptr()
        self._ptr = {k: base + 4 * o for k, o in offsets.items()}
        self._packed_info, self._dev_packed = None, None

    def _ensure_packed(self):
        """bf16 hi/lo operand copies of the conv weights for the wgmma path (tc.py / conv_tc.cu); False if the model
        has no convolution"""
        if self._packed_info is None:
            from . import tc
            torch = self._torch()
            self._packed_info = {}
            parts, poff = [], 0
            for k in self.plan.kops:
                if k.kind not in ('conv', 'sepconv'):
                    continue
                key = _weight_key(k)
                if key in self._packed_info:
                    continue
                w = self._host_weights[key]
                hi, lo, cp, kp = tc.pack_conv_kernel(w)
                rec = {'cout_pad': cp, 'k_pad': kp}
                for nm, arr in (('hi', hi), ('lo', lo)):
                    rec[nm] = poff
                    parts.append(arr.ravel())
                    pad = (-arr.size) % 128
                    if pad:
                        parts.append(np.zeros(pad, np.uint16))
                    poff += arr.size + pad
                self._packed_info[key] = rec
            if parts:
                arena = np.concatenate(parts).view(np.int16)
                self._dev_packed = torch.from_numpy(arena).cuda()
                pbase = self._dev_packed.data_ptr()
                for rec in self._packed_info.values():
                    rec['hi'] = pbase + 2 * rec['hi']
                    rec['lo'] = pbase + 2 * rec['lo']
        return bool(self._packed_info)

    def _keras_shape(self, t, n):
        lead = (n,)
        if t.kind == 'frame' and self.graph.frames_per_clip > 1 and n is not None:
            lead = (n // self.graph.frames_per_clip, self.graph.frames_per_clip)
        elif t.kind == 'frame' and self.graph.frames_per_clip > 1:
            lead = (None, self.graph.frames_per_clip)
        return lead + _item_dims(t)

    def _items(self, kind, n_frames):
        return n_frames if kind == 'frame' else n_frames // self.graph.frames_per_clip

    def _bind(self, n_frames):
        """the binding forwards at n_frames frames use; one made under other settings is replaced"""
        b = self._bound.pop(n_frames, None)
        if b is None or not b.current(self):
            b = None                    # released before its replacement is made
            self._torch()
            while len(self._bound) >= max(1, self.max_bound):     # evict the least recently used arena
                old = self._bound.pop(next(iter(self._bound)))
                old.graph = None
                del old
            b = self._bind_plan(self.plan, n_frames)
        self._bound[n_frames] = b               # most recently used last
        return b

    def _bind_plan(self, plan, n_frames):
        """`plan` (the model's own, or a stage of compiler.split_stages) bound to n_frames frames: its activation
        slots, workspace and the ctypes argument list of every launch, on this model's device weights and settings."""
        torch = self._torch()
        self._ensure_device_weights()
        lib = _ffi.lib()
        b = _Bound(self, plan, n_frames, self.use_tensor_cores and self._ensure_packed())
        for (kind, fl) in plan.phys:
            b.slots.append(torch.empty(self._items(kind, n_frames) * fl, dtype=torch.float32, device='cuda'))
        ctxh = self._ctx.handle
        P = self._ptr

        def view(t):
            v = b.view(t)
            b.keep.append(v)        # the launches hold pointers to it
            return v

        def dense_ptr(t):
            s = plan.storage[t.id]
            assert s.c_off == 0 and s.ld == t.shape[2], 'dense output expected'
            return b.slots[s.buf.phys].data_ptr()

        def conv_desc(k):
            a = k.attrs
            d = _ffi.dh_conv_desc()
            d.kh, d.kw = a['size']
            d.sh, d.sw = a['strides']
            d.pad_same = 1 if a['padding'] == 'same' else 0
            d.pre_relu = 1 if a['pre_relu'] else 0
            d.post_relu = 1 if a['post_relu'] else 0
            if a['pre_bn']:
                d.pre_scale = P['fold:' + a['pre_bn']['name']]
                d.pre_shift = P['shift:' + a['pre_bn']['name']]
            if a['post_bn']:
                d.post_scale = P['fold:' + a['post_bn']['name']]
                d.post_shift = P['shift:' + a['post_bn']['name']]
            d.n_res = a['n_res']
            d.res_up2x = a.get('res_up2x', 0)
            if a.get('pool_out'):
                d.pool_out = view(k.outs[1])
            for i in range(a['n_res']):
                d.res[i] = view(k.ins[1 + i])
            d.precision = b.precision
            b.keep.append(d)
            return d

        nullv = C.cast(None, C.POINTER(_ffi.dh_view))
        nullp = C.cast(None, C.POINTER(_ffi.dh_packed_w))
        for k in plan.kops:
            kd = k.kind
            if kd in ('conv', 'sepconv'):
                wargs = (P[k.attrs['kernel']],) if kd == 'conv' else (P[k.attrs['depthwise']], P[k.attrs['pointwise']])
                cargs = (ctxh, C.byref(view(k.ins[0]))) + wargs + (self._packed(k, b) or nullp, C.byref(conv_desc(k)),
                                                                  C.byref(view(k.outs[0])))
                info = _ffi.dh_conv_plan_info()
                rc = (lib.dh_conv2d_plan if kd == 'conv' else lib.dh_sepconv2d_plan)(*cargs, C.byref(info))
                if rc != 0:
                    raise _ffi.DeepharB200Error('%s layer %s: no kernel takes it (rc=%d): %s' % (
                        kd, _weight_key(k), rc, lib.dh_last_error().decode()))
                b.conv_plans.append((k, info))
                args = (lib.dh_conv2d_f32 if kd == 'conv' else lib.dh_sepconv2d_f32,) + cargs
            elif kd == 'maxpool':
                a = k.attrs
                args = (lib.dh_maxpool2d_f32, ctxh, C.byref(view(k.ins[0])), a['pool'][0], a['pool'][1],
                        a['strides'][0], a['strides'][1], 1 if a['padding'] == 'same' else 0,
                        C.byref(view(k.outs[0])))
            elif kd == 'upsample_add':
                args = (lib.dh_upsample2x_add_f32, ctxh, C.byref(view(k.ins[0])), C.byref(view(k.ins[1])),
                        C.byref(view(k.outs[0])))
            elif kd == 'upsample':
                args = (lib.dh_upsample2x_add_f32, ctxh, nullv, C.byref(view(k.ins[0])),
                        C.byref(view(k.outs[0])))
            elif kd in ('add', 'affine', 'copy'):
                arr = (_ffi.dh_view * len(k.ins))(*[view(t) for t in k.ins])
                b.keep.append(arr)
                scale = shift = None
                relu = 0
                if kd == 'affine':
                    if k.attrs['bn']:
                        scale = P['fold:' + k.attrs['bn']['name']]
                        shift = P['shift:' + k.attrs['bn']['name']]
                    relu = 1 if k.attrs['relu'] else 0
                ov = view(k.outs[0])
                if kd == 'copy':
                    ov.p = ov.p + 4 * k.attrs['c_off']
                    ov.c = k.attrs['channels']
                args = (lib.dh_add_n_f32, ctxh, arr, len(k.ins), scale, shift, relu, C.byref(ov))
            elif kd == 'pose_regression_2d_context':
                a = k.attrs
                args = (lib.dh_softargmax2d_ctx_f32, ctxh, C.byref(view(k.ins[0])), a['num_joints'],
                        a['num_context'], C.c_float(a['alpha']), dense_ptr(k.outs[0]), dense_ptr(k.outs[1]))
            elif kd == 'pose_regression_2d':
                args = (lib.dh_softargmax2d_f32, ctxh, C.byref(view(k.ins[0])), nullv, C.c_float(1.0), 0,
                        dense_ptr(k.outs[0]), dense_ptr(k.outs[1]), nullv)
            elif kd == 'pose_regression_3d':
                a = k.attrs
                args = (lib.dh_softargmax3d_f32, ctxh, C.byref(view(k.ins[0])), a['num_joints'],
                        a['depth_maps'], dense_ptr(k.outs[0]), dense_ptr(k.outs[1]))
            elif kd == 'pose_regression_3d_ex':
                a = k.attrs
                args = (lib.dh_softargmax3d_ex_f32, ctxh, C.byref(view(k.ins[0])), a['num_joints'], a['depth_maps'],
                        C.c_float(a['vis_scale']), dense_ptr(k.outs[0]), dense_ptr(k.outs[1]), C.byref(view(k.outs[2])))
            elif kd == 'scale':
                key = 'const:%r' % float(k.attrs['value'])
                arr = (_ffi.dh_view * 1)(view(k.ins[0]))
                b.keep.append(arr)
                args = (lib.dh_add_n_f32, ctxh, arr, 1, P[key], P['const:0.0'], 0, C.byref(view(k.outs[0])))
            elif kd == 'sam2d':
                a = k.attrs
                dv = C.byref(view(k.ins[1])) if a['depth'] else nullv
                pv = C.byref(view(k.outs[2])) if a['prob'] else nullv
                args = (lib.dh_softargmax2d_f32, ctxh, C.byref(view(k.ins[0])), dv, C.c_float(a['alpha']), 1,
                        dense_ptr(k.outs[0]), dense_ptr(k.outs[1]), pv)
            elif kd == 'kron':
                args = (lib.dh_kron_pool_f32, ctxh, C.byref(view(k.ins[0])), C.byref(view(k.ins[1])),
                        dense_ptr(k.outs[0]))
            elif kd == 'mask_mul':
                t = k.ins[0]
                rows = self._items(t.kind, n_frames) * t.shape[0] * t.shape[1]
                args = (lib.dh_mask_mul_f32, ctxh, dense_ptr(k.ins[0]), dense_ptr(k.ins[1]), rows, t.shape[2],
                        dense_ptr(k.outs[0]))
            elif kd == 'zeropad':
                (pt, pb), (pl, pr) = k.attrs['pads']
                args = (lib.dh_zeropad2d_f32, ctxh, C.byref(view(k.ins[0])), pt, pl, C.byref(view(k.outs[0])))
            elif kd == 'maxminpool':
                args = (lib.dh_maxmin_pool2d_f32, ctxh, C.byref(view(k.ins[0])), C.byref(view(k.outs[0])))
            elif kd == 'global_maxmin_softmax':
                args = (lib.dh_global_maxmin_softmax_f32, ctxh, C.byref(view(k.ins[0])), dense_ptr(k.outs[0]))
            else:
                raise NotImplementedError('kernel op %s' % kd)
            b.calls.append((kd,) + args)
        ws_bytes = max([16] + [info.workspace_bytes for _, info in b.conv_plans])
        b.workspace = torch.empty(-(-ws_bytes // 4), dtype=torch.float32, device='cuda')
        # kernels one issue launches: a separable conv on the CUDA-core kernels (path 0) runs as two, depthwise into
        # the workspace, then pointwise
        b.kernels = len(b.calls) + sum(1 for k, info in b.conv_plans if k.kind == 'sepconv' and info.path == 0)
        return b

    def _packed(self, k, b):
        if not b.packed:
            return None
        rec = self._packed_info[_weight_key(k)]
        pw = _ffi.dh_packed_w(rec['hi'], rec['lo'], rec['cout_pad'], rec['k_pad'])
        b.keep.append(pw)
        return C.pointer(pw)

    def _run(self, b):
        """One forward over the bound buffers on torch's current stream (the CUDA-graph policy of _graphed)."""
        self.launch_total = getattr(self, 'launch_total', 0) + b.kernels     # kernels put on the stream
        b.graph, b.uses = _graphed(self.use_cuda_graph, b.graph, b.uses, b.issue)
        if self.use_cuda_graph and b.graph is not None:
            self._graph_replays = getattr(self, '_graph_replays', 0) + 1

    def export(self, path, n_frames, outputs=None):
        """Write the forward at n_frames frames (n_frames // T clips of a clip model) to one file that the C ABI loads
        and runs with no Python in the process (dh_model_load / dh_model_forward, include/deephar_b200.h): the launch
        list this model binds, its weights and its buffer sizes.  outputs: indices of the outputs to record (all).
        n_frames is the largest batch the file runs: dh_model_set_batch runs it at fewer frames (clips).
        The batch sizes the model keeps bound for forward_device are left as they were: an unbound n_frames is bound
        for this call only."""
        from . import export
        if n_frames < 1 or n_frames % self.graph.frames_per_clip:
            raise ValueError('n_frames must be a positive multiple of the %d frames per clip' % self.graph.frames_per_clip)
        export.write(self, str(path), int(n_frames), outputs)

    def _output_tensor(self, b, t, n_frames, plan=None):
        """b.tensor(t), for callers that also name the binding's frames and plan (tests/launch_check.py)"""
        assert n_frames == b.n_items and (plan or self.plan) is b.plan
        return b.tensor(t)

    def forward_device(self, x_dev):
        """x_dev: float32 CUDA tensor (N,H,W,3) (or (B,T,H,W,3)); returns device tensors (views into
        the plan's buffers, valid until the next call)."""
        n_frames = int(np.prod(x_dev.shape[:-3]))
        b = self._bind(n_frames)
        t_in = self.graph.inputs[0]
        s = self.plan.storage[t_in.id]
        b.slots[s.buf.phys].copy_(x_dev.reshape(-1), non_blocking=True)
        self._run(b)
        return [b.tensor(t).reshape(self._keras_shape(t, self._items(t.kind, n_frames))) for t in self.graph.outputs]

    def _host_input(self, x):
        """What keras.Model.predict accepts for a single-input model: the array itself or a list holding it
        (`inputs = [fval]`, exp/common/mpii_tools.py:80-86); returned as contiguous float32 of the model's input shape."""
        if isinstance(x, (list, tuple)):
            if len(x) != 1:
                raise ValueError('model %r has one input, predict() got a list of %d arrays' % (self.name, len(x)))
            x = x[0]
        x = np.ascontiguousarray(x, dtype=np.float32)
        T = self.graph.frames_per_clip
        lead = 2 if T > 1 else 1
        exp = tuple(self.graph.inputs[0].shape)
        if tuple(x.shape[lead:]) != exp or (T > 1 and x.shape[1] != T):
            raise ValueError('input shape %s does not match model input %s' % (x.shape, self.input_shape))
        return x

    def predict(self, x, batch_size=32, verbose=0):
        """keras.Model.predict: host numpy in, list of host numpy out.  `batch_size` counts items
        of the leading axis (frames, or clips for clip models), as in Keras."""
        x = self._host_input(x)
        if batch_size is None:      # keras: None means the default of 32
            batch_size = 32
        if int(batch_size) != batch_size or batch_size < 1:
            raise ValueError('batch_size must be a positive integer, got %r' % (batch_size,))
        batch_size = int(batch_size)
        torch = self._torch()
        T = self.graph.frames_per_clip
        n = x.shape[0]
        if n == 0:                  # keras returns empty arrays of the right trailing shape
            outs = [np.zeros((0,) + tuple(d for d in self._keras_shape(t, 0)[1:]), np.float32) for t in self.graph.outputs]
            return outs[0] if len(outs) == 1 else outs
        xt = torch.from_numpy(x)
        pinned = xt.is_pinned()
        item = int(np.prod(x.shape[1:]))
        if not pinned:
            if getattr(self, '_stage', None) is None or self._stage.numel() < batch_size * item:
                self._stage = torch.empty(batch_size * item, dtype=torch.float32).pin_memory()
        # per-output pinned result buffers for the whole call (one D2H copy per output per batch), kept for the next call
        # with the same item count: page-locking 2 x (number of outputs) buffers costs more than a small forward, and the
        # evaluators call predict once per clip (exp/common/penn_tools.py:124).  The caller gets copies.
        held = getattr(self, '_pinned_results', None)
        if held is not None and held[0] == n:
            res = held[1]
        else:
            res = []
            for t in self.graph.outputs:
                shp = self._keras_shape(t, n if t.kind == 'clip' or T == 1 else n * T)
                res.append(torch.empty(shp, dtype=torch.float32).pin_memory())
            self._pinned_results = (n, res)
        # The host->device copy of batch k+1 runs on a side stream while batch k computes
        # (two device staging buffers; events order copy -> compute -> buffer reuse).
        main = torch.cuda.current_stream()
        if getattr(self, '_copy_stream', None) is None:
            self._copy_stream = torch.cuda.Stream()
        copy_stream = self._copy_stream
        spans = [(i, min(i + batch_size, n)) for i in range(0, n, batch_size)]
        dev = [None, None]
        ready = [torch.cuda.Event(), torch.cuda.Event()]
        consumed = [torch.cuda.Event(), torch.cuda.Event()]

        def issue_copy(k):
            i, j = spans[k]
            slot = k & 1
            if pinned:
                src = xt[i:j]
            else:
                copy_stream.synchronize()                     # pinned staging buffer reuse
                src = self._stage[:(j - i) * item].view((j - i,) + tuple(x.shape[1:]))
                src.copy_(xt[i:j])
            with torch.cuda.stream(copy_stream):
                if k >= 2:
                    copy_stream.wait_event(consumed[slot])    # compute of batch k-2 has read the buffer
                if dev[slot] is None or dev[slot].shape != src.shape:
                    dev[slot] = torch.empty(src.shape, dtype=torch.float32, device='cuda')
                dev[slot].copy_(src, non_blocking=True)
                ready[slot].record(copy_stream)

        issue_copy(0)
        for k, (i, j) in enumerate(spans):
            slot = k & 1
            if k + 1 < len(spans):
                issue_copy(k + 1)
            main.wait_event(ready[slot])
            outs = self.forward_device(dev[slot])
            consumed[slot].record(main)
            for r, o in zip(res, outs):
                r[i:j].copy_(o, non_blocking=True)
        torch.cuda.current_stream().synchronize()
        outs = [r.numpy().copy() for r in res]
        return outs[0] if len(outs) == 1 else outs

    def output_subset(self, indices, name=None):
        """A keras-`Model(full.input, full.outputs[a:b])`-like view (spnet.split_model): shares the
        compiled network, weights and device buffers with this model and returns only the
        selected outputs."""
        return _OutputSubset(self, list(indices), name)

    def _mode(self):
        """(precision, packed operands passed) of the most recently used binding; before one, of the current settings"""
        b = next(reversed(self._bound.values()), None)
        if b is None:
            return self.precision, bool(self.use_tensor_cores and self._packed_info)
        return b.precision, b.packed

    def math_mode(self):
        """Arithmetic the convolutions run in (bench.py `dtype`)."""
        precision, packed = self._mode()
        if packed:
            return 'bf16x%d split (fp32 accumulate, wgmma)' % precision if precision != 1 else 'bf16'
        return 'f32'

    def _uses_tc(self):
        return self._mode()[1]

    def profile(self, x_dev):
        """One forward with CUDA events around every kernel op (launch stream = torch's current
        stream).  Returns {label: {'label','ms','launches','flops'}} aggregated per op shape."""
        torch = self._torch()
        n_frames = int(np.prod(x_dev.shape[:-3]))
        b = self._bind(n_frames)
        s = self.plan.storage[self.graph.inputs[0].id]
        b.slots[s.buf.phys].copy_(x_dev.reshape(-1))
        evs = []
        b.issue(torch.cuda.current_stream().cuda_stream, evs)
        torch.cuda.synchronize()
        out = {}
        for k, (e0, e1) in zip(self.plan.kops, evs):
            label = '%s %s->%s' % (k.kind, 'x'.join(map(str, k.ins[0].shape)), 'x'.join(map(str, k.outs[0].shape)))
            flops = 0.0
            if k.kind in ('conv', 'sepconv'):
                label += ' k%dx%d' % tuple(k.attrs['size'])
                flops = 2.0 * _conv_macs(k) * self._items(k.outs[0].kind, n_frames)
            r = out.setdefault(label, {'label': label, 'ms': 0.0, 'launches': 0, 'flops': flops})
            r['ms'] += e0.elapsed_time(e1)
            r['launches'] += 1
        return out

    def launches_per_forward(self, n_frames):
        """kernels one forward at n_frames frames launches"""
        return self._bind(n_frames).kernels


class _OutputSubset(object):
    """Result of spnet.split_model: same network, subset of the outputs (spnet.py:443-446)."""

    def __init__(self, full, indices, name):
        self.full = full
        self.indices = indices
        self.name = name or full.name

    @property
    def outputs(self):
        return [self.full.outputs[i] for i in self.indices]

    @property
    def input_shape(self):
        return self.full.input_shape

    def get_input_shape_at(self, i):
        return self.full.get_input_shape_at(i)

    @property
    def output_shape(self):
        shp = self.full.output_shape
        return [shp[i] for i in self.indices]

    def predict(self, x, batch_size=32, verbose=0):
        outs = self.full.predict(x, batch_size=batch_size, verbose=verbose)
        if not isinstance(outs, list):
            outs = [outs]
        sel = [outs[i] for i in self.indices]
        return sel[0] if len(sel) == 1 else sel

    def load_weights(self, path, by_name=False):
        return self.full.load_weights(path, by_name=by_name)

    def export(self, path, n_frames):
        """Model.export of the selected outputs"""
        return self.full.export(path, n_frames, outputs=self.indices)

    def summary(self, *args, **kwargs):
        return self.full.summary(*args, **kwargs)
