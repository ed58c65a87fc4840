"""Model.export / ClipStream.export: a bound plan written to one file that the C ABI runs with no Python in the process.

The file records what `Model._bind_plan` produced for one batch size -- every launch of `b.calls` with its arguments --
and the memory those arguments point into, so `dh_model_load` / `dh_model_forward` (csrc/model_rt.cu) replay the same
launch list: kernel selection, fusion and buffer planning stay in the Python compiler.  The format is documented in
include/deephar_b200.h ("whole model"); this module writes it and reads it back (`read`, for tests and tools).

Every device pointer is stored as (arena, byte offset).  Arenas: 0 = the fp32 weight arena (folded BatchNormalization
vectors and constants included), 1 = the bf16 hi / lo tensor-core operands, 2 = the convolution workspace, 3 + s =
activation slot s of the plan.  Each slot's kind (frame or clip items, `plan.phys`) is recorded too, so the C runtime
can run the file at any batch up to the exported one (dh_model_set_batch).

A ClipStream writes its two stages to one stream file (`write_stream`, read back by `read_stream`): the same launch
records, with the arenas of both stages, the rings and the boundary table of its window launch
(dh_stream_load / dh_stream_push).
"""
import ctypes as C
import struct

import numpy as np

from . import _ffi

MAGIC = b'DHMODEL\0'
VERSION = 2
SLOT_KINDS = ('frame', 'clip')      # the kind table of a model file: slot s holds frame (0) or clip (1) items
STREAM_MAGIC = b'DHSTREAM\0'
STREAM_VERSION = 1
STREAM_ARENA_SLOT0 = 4      # stream files: 2 / 3 = the frame / clip workspace, then frame slots, clip slots, rings
MAX_RANK = 6
ARENA_WEIGHTS, ARENA_PACKED, ARENA_WORKSPACE, ARENA_SLOT0 = 0, 1, 2, 3

# entry-point ids of the file: the forward's launches, in this order (csrc/model_rt.cu keeps the same table)
ENTRY_POINTS = ('dh_conv2d_f32', 'dh_sepconv2d_f32', 'dh_maxpool2d_f32', 'dh_upsample2x_add_f32', 'dh_add_n_f32',
                'dh_softargmax2d_f32', 'dh_softargmax2d_ctx_f32', 'dh_softargmax3d_f32', 'dh_softargmax3d_ex_f32',
                'dh_kron_pool_f32', 'dh_zeropad2d_f32', 'dh_maxmin_pool2d_f32', 'dh_global_maxmin_softmax_f32',
                'dh_mask_mul_f32')


def arg_tag(argtype):
    """one-letter tag of an argument type of the binding: i integer, f float, p device pointer, v dh_view pointer
    (a view, an array of views or NULL), d dh_conv_desc pointer, w dh_packed_w pointer (or NULL)"""
    if argtype is _ffi._VP:
        return 'v'
    if argtype is _ffi._DP:
        return 'd'
    if argtype is _ffi._PP:
        return 'w'
    if argtype is C.c_void_p:
        return 'p'
    if argtype is C.c_float:
        return 'f'
    if argtype in (C.c_int, C.c_int32, C.c_int64):
        return 'i'
    raise TypeError('no file encoding for argument type %r' % (argtype,))


def signature(name):
    """the tags of an entry point's arguments between the context and the stream"""
    return ''.join(arg_tag(t) for t in _ffi.SIGNATURES[name][1][1:-1])


class _Writer(object):
    def __init__(self, arenas):
        self.out = bytearray()
        self.arenas = arenas            # [(base address, bytes)] by arena id

    def raw(self, fmt, *v):
        self.out += struct.pack('<' + fmt, *v)

    def ptr(self, p):
        if not p:
            return self.raw('iq', -1, 0)
        for i, (base, n) in enumerate(self.arenas):
            if n and base <= p < base + n:
                return self.raw('iq', i, p - base)
        raise ValueError('pointer 0x%x lies in none of the model arenas' % p)

    def field(self, ty, v):
        if ty is C.c_void_p:
            self.ptr(v)
        elif ty is C.c_int32:
            self.raw('i', v)
        elif isinstance(ty, type) and issubclass(ty, C.Structure):
            self.struct(v)
        elif isinstance(ty, type) and issubclass(ty, C.Array):
            for e in v:
                self.field(ty._type_, e)
        else:
            raise TypeError('no file encoding for field type %r' % (ty,))

    def struct(self, s):
        for name, ty in s._fields_:
            self.field(ty, getattr(s, name))

    def view(self, v):
        self.struct(v)

    def shape(self, shp):
        self.raw('i', len(shp))
        self.raw('%dq' % len(shp), *[int(d) for d in shp])

    def arg(self, tag, v):
        self.raw('B', ord(tag))
        if tag == 'i':
            self.raw('q', int(v))
        elif tag == 'f':
            self.raw('f', v.value if isinstance(v, C.c_float) else float(v))
        elif tag == 'p':
            self.ptr(v.value if isinstance(v, C.c_void_p) else v)
        elif tag in 'vdw':
            objs = _pointees(v)
            self.raw('i', len(objs))
            for o in objs:
                self.struct(o)
        else:
            raise AssertionError(tag)


def _pointees(v):
    """the structs a pointer argument of b.calls points at: byref(s), pointer(s), an array of structs, or NULL"""
    if v is None:
        return []
    if isinstance(v, C.Array):
        return list(v)
    if isinstance(v, C._Pointer):
        return [v.contents] if v else []
    if isinstance(v, C.Structure):
        return [v]
    obj = getattr(v, '_obj', None)          # C.byref(s)
    if isinstance(obj, C.Structure):
        return [obj]
    raise TypeError('unexpected pointer argument %r' % (v,))


def _host_bytes(t):
    return t.detach().cpu().contiguous().view(-1).numpy().view(np.uint8).tobytes()


def _arenas(model, bindings, rings=()):
    """the file's arena table [(base address, bytes)]: weights, packed operands (if the bindings pass them), each
    binding's workspace, each binding's slots, the rings"""
    packed = model._dev_packed if bindings[0].packed else None
    tensors = [(model._dev, 4), (packed, 2)] + [(b.workspace, 4) for b in bindings] + \
        [(s, 4) for b in bindings for s in b.slots] + [(r, 4) for r in rings]
    return [(t.data_ptr(), t.numel() * e) if t is not None else (0, 0) for t, e in tensors]


def _write_blobs(w, model, packed):
    for blob in (_host_bytes(model._dev), _host_bytes(model._dev_packed) if packed else b''):
        w.raw('q', len(blob))
        w.out += blob


def _write_output(w, view, shape, name):
    w.view(view)
    w.shape(shape)
    name = name.encode()
    w.raw('i', len(name))
    w.out += name


def _output_name(t, i):
    return (t.node.attrs.get('name') if t.node is not None else None) or 'output_%d' % i


def _write_launches(w, plan, b):
    """i32 count, then every launch of b.calls: entry point, label and its arguments between ctx and stream"""
    lib = _ffi.lib()
    ids = {id(getattr(lib, name)): i for i, name in enumerate(ENTRY_POINTS)}
    sigs = [signature(name) for name in ENTRY_POINTS]
    labels = _labels(plan, b)
    w.raw('i', len(b.calls))
    for n, call in enumerate(b.calls):
        ep = ids.get(id(call[1]))
        if ep is None:
            raise ValueError('launch %d (%s) calls an entry point the file format does not record' % (n, call[0]))
        args = call[3:]                     # (kind, function, ctx, args ...); the stream is added at issue time
        sig = sigs[ep]
        if len(args) != len(sig):
            raise ValueError('launch %d (%s): %d arguments, %s takes %d' % (n, call[0], len(args), ENTRY_POINTS[ep],
                                                                           len(sig)))
        label = labels[n].encode()
        w.raw('iii', ep, len(args), len(label))
        w.out += label
        for tag, v in zip(sig, args):
            w.arg(tag, v)


def write(model, path, n_frames, outputs=None):
    """Bind `model` at n_frames frames (as forward_device does) and write the launch list to `path`.
    outputs: indices of the model outputs to record (all by default).  A batch size the model has bound already with
    its current settings is written from that binding; otherwise the binding is made for this call only and its buffers
    are released when it returns, so exporting neither evicts nor adds a bound batch size of the model."""
    b = model._bound.get(n_frames)
    if b is None or not b.current(model):
        b = model._bind_plan(model.plan, n_frames)
    arenas = _arenas(model, [b])
    w = _Writer(arenas)
    g, plan = model.graph, model.plan
    in_shape = (n_frames // g.frames_per_clip, g.frames_per_clip) + g.inputs[0].shape if g.frames_per_clip > 1 \
        else (n_frames,) + g.inputs[0].shape
    w.out += MAGIC
    w.raw('I', VERSION)
    w.raw('iiiii', int(b.precision), int(b.packed), model._items('frame', n_frames),
          model._items('clip', n_frames), g.frames_per_clip)
    w.shape(in_shape)
    _write_blobs(w, model, b.packed)
    w.raw('i', len(b.slots))
    w.raw('%dq' % len(b.slots), *[n for _, n in arenas[ARENA_SLOT0:]])
    w.raw('%dB' % len(b.slots), *[SLOT_KINDS.index(kind) for kind, _ in plan.phys])
    w.raw('q', arenas[ARENA_WORKSPACE][1])
    w.view(b.view(g.inputs[0]))
    idx = list(range(len(g.outputs))) if outputs is None else [int(i) for i in outputs]
    w.raw('i', len(idx))
    for i in idx:
        t = g.outputs[i]
        shp = model._keras_shape(t, model._items(t.kind, n_frames))
        if len(shp) > MAX_RANK:
            raise ValueError('output %d has rank %d > %d' % (i, len(shp), MAX_RANK))
        _write_output(w, b.view(t), shp, _output_name(t, i))
    _write_launches(w, plan, b)
    with open(path, 'wb') as f:
        f.write(bytes(w.out))


def write_stream(stream, path):
    """Write what ClipStream `stream` has bound -- its frame stage at S frames, its clip stage at S * T, the boundary
    table of its window launch, its outputs -- to `path` (the stream format of include/deephar_b200.h).  The stream's
    run-time state (rings, ring position, counts) is not recorded: a loaded stream starts with no stream ready."""
    from .model import _item_dims
    m, S, T, st = stream.model, stream.n_streams, stream.frames_per_clip, stream.stages
    if m._dev is not stream._weights:
        raise RuntimeError('the model\'s weights were replaced after this ClipStream was built: build a new one')
    bf, bc = stream._frame, stream._clip
    w = _Writer(_arenas(m, [bf, bc], stream._rings))
    t_in = m.graph.inputs[0]
    w.out += STREAM_MAGIC
    w.raw('I', STREAM_VERSION)
    w.raw('iiii', int(bf.precision), int(bf.packed), S, T)
    w.shape((S,) + tuple(t_in.shape))
    _write_blobs(w, m, bf.packed)

    def sizes(arrays):
        w.raw('i', len(arrays))
        w.raw('%dq' % len(arrays), *[a.numel() * 4 for a in arrays])
    sizes(bf.slots)
    w.raw('q', bf.workspace.numel() * 4)
    sizes(bc.slots)
    w.raw('q', bc.workspace.numel() * 4)
    sizes(stream._rings)
    for t, ring in zip(st.boundary, stream._rings):
        w.view(bf.view(t))
        w.view(bc.view(t))
        w.ptr(ring.data_ptr())
    w.view(bf.view(t_in))
    for b, outs in ((bf, stream.frame_output_tensors), (bc, stream.clip_output_tensors)):
        w.raw('i', len(outs))
        for t in outs:
            shp = (S,) + _item_dims(t)
            if len(shp) > MAX_RANK:
                raise ValueError('output %r has rank %d > %d' % (t, len(shp), MAX_RANK))
            _write_output(w, b.view(t), shp, _output_name(t, m.graph.outputs.index(t)))
    _write_launches(w, st.frame, bf)
    _write_launches(w, st.clip, bc)
    with open(path, 'wb') as f:
        f.write(bytes(w.out))


def _labels(plan, b):
    """launch n -> 'kind' or 'kind layer' (the weight the layer's conv reads), for error messages of the C side"""
    from .model import _weight_key
    names = iter(_weight_key(k) for k, _ in b.conv_plans)
    return ['%s %s' % (c[0], next(names)) if c[0] in ('conv', 'sepconv') else c[0] for c in b.calls]


# ---- reading (tests and tools; the C side has its own validating parser) --------------------------------------------------
class _Reader(object):
    def __init__(self, data):
        self.data, self.pos = data, 0

    def raw(self, fmt):
        fmt = '<' + fmt
        n = struct.calcsize(fmt)
        if self.pos + n > len(self.data):
            raise ValueError('truncated model file')
        v = struct.unpack_from(fmt, self.data, self.pos)
        self.pos += n
        return v

    def one(self, fmt):
        return self.raw(fmt)[0]

    def bytes(self, n):
        if n < 0 or self.pos + n > len(self.data):
            raise ValueError('truncated model file')
        v = self.data[self.pos:self.pos + n]
        self.pos += n
        return v

    def ptr(self):
        a, off = self.raw('iq')
        return None if a < 0 else (a, off)

    def field(self, ty):
        if ty is C.c_void_p:
            return self.ptr()
        if ty is C.c_int32:
            return self.one('i')
        if issubclass(ty, C.Structure):
            return self.struct(ty)
        if issubclass(ty, C.Array):
            return [self.field(ty._type_) for _ in range(ty._length_)]
        raise TypeError(ty)

    def struct(self, ty):
        return {name: self.field(t) for name, t in ty._fields_}

    def shape(self):
        r = self.one('i')
        return self.raw('%dq' % r)


_STRUCT = {'v': _ffi.dh_view, 'd': _ffi.dh_conv_desc, 'w': _ffi.dh_packed_w}


def read(path):
    """The file as plain Python values: pointers are (arena, byte offset) or None, structs are dicts of their fields;
    each launch and output also gives the file offset its record starts at.  'slot_kinds' is 'frame' or 'clip' per
    activation slot (None in a version-1 file)."""
    with open(path, 'rb') as f:
        r = _Reader(f.read())
    if r.bytes(8) != MAGIC:
        raise ValueError('not a deephar_b200 model file')
    m = {'version': r.one('I')}
    m['precision'], m['use_tensor_cores'], m['frame_items'], m['clip_items'], m['frames_per_clip'] = r.raw('iiiii')
    m['input_shape'] = r.shape()
    m['weights'] = r.bytes(r.one('q'))
    m['packed'] = r.bytes(r.one('q'))
    m['slot_bytes'] = list(r.raw('%dq' % r.one('i')))
    # version 1 has no kind table: its file runs at the exported batch only
    m['slot_kinds'] = [SLOT_KINDS[k] for k in r.raw('%dB' % len(m['slot_bytes']))] if m['version'] >= 2 else None
    m['workspace_bytes'] = r.one('q')
    m['input'] = r.struct(_ffi.dh_view)
    m['outputs'] = _read_outputs(r)
    m['launches'] = _read_launches(r)
    _read_end(r)
    return m


def _read_outputs(r):
    outs = []
    for _ in range(r.one('i')):
        at = r.pos
        v = r.struct(_ffi.dh_view)
        shp = r.shape()
        outs.append({'view': v, 'shape': shp, 'name': r.bytes(r.one('i')).decode(), 'file_offset': at})
    return outs


def _read_launches(r):
    launches = []
    for _ in range(r.one('i')):
        at = r.pos
        ep, nargs, nlabel = r.raw('iii')
        launch = {'entry': ENTRY_POINTS[ep], 'label': r.bytes(nlabel).decode(), 'args': [], 'file_offset': at}
        for _ in range(nargs):
            tag = chr(r.one('B'))
            if tag == 'i':
                v = r.one('q')
            elif tag == 'f':
                v = r.one('f')
            elif tag == 'p':
                v = r.ptr()
            else:
                v = [r.struct(_STRUCT[tag]) for _ in range(r.one('i'))]
            launch['args'].append((tag, v))
        launches.append(launch)
    return launches


def _read_end(r):
    if r.pos != len(r.data):
        raise ValueError('%d bytes after the last launch' % (len(r.data) - r.pos))


def read_stream(path):
    """A stream file (ClipStream.export) as plain Python values, in read()'s form.  Arena ids: 0 weights, 1 packed,
    2 / 3 the frame / clip workspace, then the frame slots, the clip slots and the rings; 'frame_slot0', 'clip_slot0'
    and 'ring0' give the first id of each group.  Each boundary entry also gives the file offset it starts at."""
    with open(path, 'rb') as f:
        r = _Reader(f.read())
    if r.bytes(len(STREAM_MAGIC)) != STREAM_MAGIC:
        raise ValueError('not a deephar_b200 stream file')
    m = {'version': r.one('I')}
    m['precision'], m['use_tensor_cores'], m['n_streams'], m['frames_per_clip'] = r.raw('iiii')
    m['input_shape'] = r.shape()
    m['weights'] = r.bytes(r.one('q'))
    m['packed'] = r.bytes(r.one('q'))
    m['frame_slot_bytes'] = list(r.raw('%dq' % r.one('i')))
    m['frame_workspace_bytes'] = r.one('q')
    m['clip_slot_bytes'] = list(r.raw('%dq' % r.one('i')))
    m['clip_workspace_bytes'] = r.one('q')
    m['ring_bytes'] = list(r.raw('%dq' % r.one('i')))
    m['frame_slot0'] = STREAM_ARENA_SLOT0
    m['clip_slot0'] = STREAM_ARENA_SLOT0 + len(m['frame_slot_bytes'])
    m['ring0'] = m['clip_slot0'] + len(m['clip_slot_bytes'])
    m['boundary'] = []
    for _ in m['ring_bytes']:
        at = r.pos
        m['boundary'].append({'src': r.struct(_ffi.dh_view), 'dst': r.struct(_ffi.dh_view), 'ring': r.ptr(),
                              'file_offset': at})
    m['input'] = r.struct(_ffi.dh_view)
    m['frame_outputs'] = _read_outputs(r)
    m['clip_outputs'] = _read_outputs(r)
    m['frame_launches'] = _read_launches(r)
    m['clip_launches'] = _read_launches(r)
    _read_end(r)
    return m
