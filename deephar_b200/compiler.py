r"""Graph -> fused kernel plan.

The reference executes one TF op per Keras layer (conv, BN, ReLU, add, pool, upsample,
concat, ... -- roughly 10 launches and 10 HBM round trips per residual unit).  Here every
convolution absorbs the layers around it:

  [BatchNormalization] -> [ReLU] -> conv/sepconv -> [BatchNormalization] -> [ReLU] -> [add]
   \__ prologue in the A-tile producer __/          \________ epilogue _______________/

(the prologue is legal because the reference is pre-activated: layers.py:258-301,
models/common.py:25-67; padding is applied after it, as Keras pads the activated tensor),
`concatenate` and channel slices become views (`ld` / channel offset of dh_view), and
UpSampling2D followed by add becomes one kernel.  Buffers are planned with liveness so a
whole forward fits comfortably in HBM and micro-batches stay L2-resident.
"""
from collections import defaultdict

CONV_OPS = ('conv', 'sepconv')
# graph ops that map 1:1 onto a C-ABI call in model.py::_bind
KERNEL_OPS = ('maxpool', 'zeropad', 'maxminpool', 'scale', 'pose_regression_2d_context', 'pose_regression_2d',
              'pose_regression_3d', 'pose_regression_3d_ex', 'kron', 'mask_mul')
DENSE_OUT_OPS = ('scale', 'pose_regression_2d_context', 'pose_regression_2d', 'pose_regression_3d', 'pose_regression_3d_ex',
                 'sam2d', 'kron', 'global_maxmin_softmax', 'mask_mul')


class KOp(object):
    """One kernel launch (or a short fixed sequence) of the C ABI."""
    __slots__ = ('kind', 'ins', 'outs', 'attrs', 'pos')

    def __init__(self, kind, ins, outs, attrs, pos):
        self.kind = kind
        self.ins = ins
        self.outs = outs
        self.attrs = attrs
        self.pos = pos

    def __repr__(self):
        return 'K[%s %s -> %s]' % (self.kind, self.ins, self.outs)


class Storage(object):
    __slots__ = ('buf', 'c_off', 'ld')

    def __init__(self, buf, c_off, ld):
        self.buf = buf
        self.c_off = c_off
        self.ld = ld


class Buffer(object):
    __slots__ = ('id', 'kind', 'hw', 'ld', 'first', 'last', 'phys', 'is_output', 'is_input')

    def __init__(self, id, kind, hw, ld):
        self.id = id
        self.kind = kind
        self.hw = hw
        self.ld = ld
        self.first = None
        self.last = -1
        self.phys = None
        self.is_output = False
        self.is_input = False

    @property
    def floats_per_item(self):
        return self.hw * self.ld


class Plan(object):
    def __init__(self):
        self.kops = []
        self.storage = {}      # tensor id -> Storage
        self.buffers = []
        self.phys = []         # physical slots: (kind, floats_per_item)
        self.bn_folds = []     # bn node attrs whose (scale, shift) must be uploaded
        self.stats = {}


def _live_nodes(g):
    """Nodes that reach a model output.  The builders follow the reference and also create layers that feed
    nothing (e.g. the re-injection convs after the LAST prediction block, spnet.py:249-262); keras.Model prunes
    them, and so does the plan: no launches, no buffers (their weights stay in weight_specs as optional)."""
    live, stack = set(), [t.node for t in g.outputs]
    while stack:
        nd = stack.pop()
        if nd is None or nd.id in live:
            continue
        live.add(nd.id)
        stack.extend(t.node for t in nd.inputs)
    return live


def _consumers(nodes):
    cons = defaultdict(list)
    for n in nodes:
        for i, t in enumerate(n.inputs):
            cons[t.id].append(n)
    return cons


class _LiveGraph(object):
    """View of a Graph restricted to the live nodes (same attributes compile_graph reads)."""

    def __init__(self, g):
        live = _live_nodes(g)
        self.nodes = [n for n in g.nodes if n.id in live or n.op == 'input']
        self.tensors, self.inputs, self.outputs = g.tensors, g.inputs, g.outputs
        self.dead = len(g.nodes) - len(self.nodes)


def _up_fusable(ch):
    """Can this conv chain take one more residual that is upsampled 2x in its epilogue?  Mirrors the C side:
    TMA-staged separable kernel (conv_sep.cu), output width 16 or 32, at most one residual so far, and no
    residual already flagged."""
    n = ch['conv']
    if n.op != 'sepconv' or len(ch['res']) > 1 or ch.get('res_up2x'):
        return False
    h, w, cin = n.inputs[0].shape
    a = n.attrs
    return (a['size'] in ((3, 3), (5, 5)) and a['strides'] == (1, 1) and a['padding'] == 'same' and w in (16, 32) and h % 4 == 0
            and cin % 32 == 0)


def pw_smallk_smem(cin, cout):
    """Dynamic shared memory of the wide pointwise kernel (conv_simt.cu, pw_smallk_smem at its 64-pixel tile): the
    [Cin][Cout] weights, the BN scale and shift per output channel, the prologue scale and shift per input channel and
    the 64 x Cin input tile, in floats.  The library takes a layer only where this is at most 200 KB."""
    return 4 * (cin * cout + 2 * cout + 2 * cin + 64 * cin)


PW_SMALLK_SMEM_MAX = 200 * 1024


def _pool_fusable(ch, pool):
    """MaxPooling2D((2,2)) of a conv chain's result as the conv's SECOND output (dh_conv_desc.pool_out).  Mirrors the C
    side (conv_simt.cu, dh_pw_smallk_supported): the wide pointwise CUDA-core kernel -- 1x1 stride 1, Cin <= 64 and
    a multiple of 4, Cout >= 128 and a multiple of 4, weights and tile within its shared memory, 32-pixel-wide maps of
    even height, no upsampled residual.  Its views must also be 16-byte aligned: _layout checks that once storage is
    placed (_pool_views_ok) and splits the pool off again where they are not."""
    n = ch['conv']
    a, pa = n.attrs, pool.attrs
    if n.op != 'conv' or ch.get('res_up2x') or 'pool' in ch:
        return False
    h, w, cin = n.inputs[0].shape
    cout = n.out.shape[2]
    return (a['size'] == (1, 1) and a['strides'] == (1, 1) and w == 32 and h % 2 == 0 and cin <= 64 and cin % 4 == 0
            and cout >= 128 and cout % 4 == 0 and pw_smallk_smem(cin, cout) <= PW_SMALLK_SMEM_MAX
            and pa['pool'] == (2, 2) and pa['strides'] == (2, 2))


def _pool_views_ok(storage, k):
    """the wide pointwise kernel reads and writes float4s: every operand view of a pool-fused conv (input, residuals,
    output, pooled output) must start 16 bytes into its buffer's rows and have a row length of whole float4s"""
    return all(storage[t.id].c_off % 4 == 0 and storage[t.id].ld % 4 == 0 for t in k.ins + k.outs)


class _OutputsOf(object):
    """A graph whose outputs are a subset of another's (the network behind a split_model view)."""

    def __init__(self, g, outputs):
        self.nodes, self.tensors, self.inputs = g.nodes, g.tensors, g.inputs
        self.outputs = list(outputs)


def _stats(plan, **head):
    head.update({
        'kernel_ops': len(plan.kops),
        'buffers': len(plan.buffers),
        'phys_slots': len(plan.phys),
        'floats_per_item_frame': sum(f for (kd, f) in plan.phys if kd == 'frame'),
        'floats_per_item_clip': sum(f for (kd, f) in plan.phys if kd == 'clip'),
    })
    return head


def compile_graph(g_full, outputs=None):
    """Plan of the graph's outputs, or of the subset `outputs` of them (whatever only other outputs need is pruned)."""
    src = g_full if outputs is None else _OutputsOf(g_full, outputs)
    g, kops = _schedule(src)
    plan = _layout(kops, g.inputs, g.outputs)
    plan.stats = _stats(plan, graph_nodes=len(g_full.nodes), dead_nodes=g.dead)
    return plan


class Stages(object):
    """A clip model's plan cut where frames become clips (stream.py).
      frame: the ops whose outputs are frame-kind, bound at one frame per stream; it writes the frame-kind model
             outputs and the `boundary` tensors (the operands of `to_clip`).
      clip:  every clip-kind op, bound at one clip per stream; its inputs are the boundary tensors of T frames per
             clip, read through the same `to_clip` alias the full plan uses.
    Each plan has `inputs` / `outputs` (tensor lists) next to its storage, so verify_plan(stage, stage) checks it."""

    def __init__(self, frame, clip, boundary):
        self.frame, self.clip, self.boundary = frame, clip, boundary


def split_stages(g_full, outputs=None):
    """The plan of compile_graph(g_full, outputs) as two Stages.  Together the stages hold the full plan's kernel ops
    (same kinds, operands and attributes); each has its own storage and liveness plan (_layout).  Raises ValueError if
    a clip-kind tensor feeds a frame-kind op, or a clip-kind op reads a frame-kind tensor other than through to_clip:
    such a graph has no per-frame part that can run once per frame."""
    src = g_full if outputs is None else _OutputsOf(g_full, outputs)
    g, kops = _schedule(src)
    frame_ops, clip_ops, boundary = [], [], []
    for k in kops:
        kinds_in = set(t.kind for t in k.ins)
        kinds_out = set(t.kind for t in k.outs)
        if k.kind == 'to_clip':
            if k.ins[0] not in boundary:
                boundary.append(k.ins[0])
            clip_ops.append(k)
        elif kinds_out == {'frame'}:
            if 'clip' in kinds_in:
                raise ValueError('%s op writing %r reads a clip-kind tensor (%r): a clip result feeds the per-frame '
                                 'network, which cannot then run once per frame'
                                 % (k.kind, k.outs[0], [t for t in k.ins if t.kind == 'clip'][0]))
            frame_ops.append(k)
        else:
            if kinds_in != {'clip'} or kinds_out != {'clip'}:
                raise ValueError('%s op writing %r mixes frame- and clip-kind tensors other than through frames_to_clip'
                                 % (k.kind, k.outs[0]))
            clip_ops.append(k)

    def own(ops):           # _layout records concat placement in the op attributes: each stage gets its own ops
        return [KOp(k.kind, k.ins, k.outs, dict(k.attrs), k.pos) for k in ops]

    frame_out = [t for t in g.outputs if t.kind == 'frame']
    frame_out += [t for t in boundary if t not in frame_out]
    clip_out = [t for t in g.outputs if t.kind == 'clip']
    stages = []
    for ops, ins, outs in ((frame_ops, g.inputs, frame_out), (clip_ops, boundary, clip_out)):
        p = _layout(own(ops), ins, outs)
        p.stats = _stats(p)
        p.inputs, p.outputs = list(ins), outs
        stages.append(p)
    return Stages(stages[0], stages[1], boundary)


def _schedule(g_full):
    """Phases 1-3: fusion decisions and the kernel ops in schedule order, views (slice / concat / to_clip) still
    included as pseudo-ops.  -> (live graph, ops)."""
    g = _LiveGraph(g_full)
    cons = _consumers(g.nodes)
    out_ids = set(t.id for t in g.outputs)

    def sole_consumer(t, op):
        if t.id in out_ids:
            return None
        c = cons[t.id]
        if len(c) == 1 and c[0].op == op:
            return c[0]
        return None

    # ---- phase 1: producer-side (epilogue) fusion for conv chains ----------------
    chains = {}            # conv node id -> dict
    fused_into = {}        # node id (bn/relu/add) -> conv node id that absorbed it as epilogue
    add_claim = {}         # add node id -> conv node id
    for n in g.nodes:
        if n.op not in CONV_OPS:
            continue
        ch = {'conv': n, 'post_bn': None, 'post_relu': False, 'add': None, 'end': n.out, 'pos': n.id}
        cur = n.out
        b = sole_consumer(cur, 'bn')
        if b is not None:
            ch['post_bn'] = b
            cur = b.out
        r = sole_consumer(cur, 'relu')
        if r is not None:
            ch['post_relu'] = r
            cur = r.out
        ch['end_pre_add'] = cur
        chains[n.id] = ch
    for cid, ch in chains.items():
        for key in ('post_bn', 'post_relu'):
            nd = ch[key]
            if nd:
                fused_into[nd.id] = cid
                ch['pos'] = max(ch['pos'], nd.id)
        ch['end'] = ch['end_pre_add']
        ch['res'] = []
    # adds (keras `add([...])`): absorbed into the epilogue of the latest conv chain whose current
    # end tensor feeds it -- also chained adds (residual add followed by a lateral add), as long as
    # the epilogue carries at most two residual operands.
    chain_end = {ch['end'].id: cid for cid, ch in chains.items()}
    up_claimed = set()     # upsample nodes absorbed by a conv epilogue
    for n in g.nodes:
        if n.op != 'add':
            continue
        if len(n.inputs) == 2 and any(t.node.op == 'upsample' and len(cons[t.id]) == 1 and t.id not in out_ids
                                      for t in n.inputs):
            # keras `add([a, UpSampling2D(b)])` (reception.py:122-127).  If `a` is the end of a fused separable conv on
            # maps whose width is a multiple of 32, the half-resolution `b` becomes the conv's LAST residual operand,
            # upsampled on the fly by the epilogue (dh_conv_desc.res_up2x) -- otherwise it is a kernel of its own.
            up = [t for t in n.inputs if t.node.op == 'upsample' and len(cons[t.id]) == 1 and t.id not in out_ids][-1]
            other = n.inputs[0] if n.inputs[1] is up else n.inputs[1]
            cid = chain_end.get(other.id)
            if cid is not None and other.id not in out_ids and len(cons[other.id]) == 1 and _up_fusable(chains[cid]):
                ch = chains[cid]
                ch['res'].append(up.node.inputs[0])
                ch['res_up2x'] = 1 << (len(ch['res']) - 1)
                up_claimed.add(up.node.id)
                add_claim[n.id] = cid
                fused_into[n.id] = cid
                del chain_end[other.id]
                chain_end[n.out.id] = cid
                ch['pos'] = max(ch['pos'], n.id)
                ch['end'] = n.out
            continue        # else: UpSampling2D + add is one kernel of its own (upsample_add)
        best = None
        for t in n.inputs:
            cid = chain_end.get(t.id)
            if cid is None or t.id in out_ids or len(cons[t.id]) != 1:
                continue
            # the upsampled residual must stay the LAST operand of the epilogue (dh_conv_desc.res_up2x)
            if len(chains[cid]['res']) + len(n.inputs) - 1 > 2 or chains[cid].get('res_up2x'):
                continue
            if best is None or chains[cid]['pos'] > chains[best]['pos']:
                best = cid
        if best is not None:
            ch = chains[best]
            endt = ch['end']
            ch['res'] += [t for t in n.inputs if t is not endt]
            add_claim[n.id] = best
            fused_into[n.id] = best
            del chain_end[endt.id]
            chain_end[n.out.id] = best
            ch['pos'] = max(ch['pos'], n.id)
            ch['end'] = n.out

    # ---- phase 2: consumer-side (prologue) fusion ---------------------------------
    absorbed_edges = set()   # (producer node id, consumer node id) edges that need no materialisation
    for cid, ch in chains.items():
        n = ch['conv']
        t = n.inputs[0]
        pre_relu, pre_bn = False, None
        if t.node.op == 'relu' and t.node.id not in fused_into:
            pre_relu = True
            absorbed_edges.add((t.node.id, n.id))
            rnode = t.node
            t = rnode.inputs[0]
            if t.node.op == 'bn' and t.node.id not in fused_into:
                pre_bn = t.node
                absorbed_edges.add((t.node.id, rnode.id))   # provisional: valid if relu not materialised
                t = t.node.inputs[0]
        elif t.node.op == 'bn' and t.node.id not in fused_into:
            pre_bn = t.node
            absorbed_edges.add((t.node.id, n.id))
            t = t.node.inputs[0]
        ch['pre_relu'], ch['pre_bn'], ch['src'] = pre_relu, pre_bn, t

    # which bn / relu nodes still need their own kernel?
    def needs_materialise(nd):
        if nd.id in fused_into:
            return False
        if nd.out.id in out_ids:
            return True
        for c in cons[nd.out.id]:
            if (nd.id, c.id) in absorbed_edges:
                # edge bn->relu only counts if that relu itself is not materialised
                if c.op == 'relu' and nd.op == 'bn' and needs_materialise(c):
                    return True
                continue
            return True
        return False

    # MaxPooling2D((2,2)) of a chain's final tensor (the hourglass pools the block-end add, reception.py:108-110): a
    # second output of the conv kernel when that kernel is the wide pointwise one
    pool_claimed = set()
    end_chain = {ch['end'].id: cid for cid, ch in chains.items()}
    for n in g.nodes:
        if n.op == 'maxpool':
            cid = end_chain.get(n.inputs[0].id)
            if cid is not None and _pool_fusable(chains[cid], n):
                chains[cid]['pool'] = n
                pool_claimed.add(n.id)

    # ---- phase 3: emit kernel ops in schedule order --------------------------------
    emitted = []           # (pos, seq, KOp)
    seq = [0]

    def emit(kind, ins, outs, attrs, pos):
        k = KOp(kind, list(ins), list(outs), attrs, pos)
        emitted.append((pos, seq[0], k))
        seq[0] += 1
        return k

    up_fused = set()
    sam_skip = set()
    for n in g.nodes:           # pre-scan: (x,y)+z concats that the fused soft-argmax kernel writes directly
        if n.op == 'depth_expect':
            cat = sole_consumer(n.out, 'concat')
            if cat is not None:
                sam_skip.add(cat.id)
    for n in g.nodes:
        op = n.op
        if op == 'input':
            continue
        if op in CONV_OPS:
            ch = chains[n.id]
            res = ch['res']
            attrs = dict(n.attrs)
            attrs.update({'pre_relu': ch['pre_relu'], 'pre_bn': ch['pre_bn'].attrs if ch['pre_bn'] else None,
                          'post_bn': ch['post_bn'].attrs if ch['post_bn'] else None,
                          'post_relu': bool(ch['post_relu']), 'n_res': len(res), 'res_up2x': ch.get('res_up2x', 0),
                          'pool_out': 'pool' in ch})
            if 'pool' in ch:
                attrs['pool_attrs'] = dict(ch['pool'].attrs)        # for _layout, should it split the pool off again
            emit(op, [ch['src']] + res, [ch['end']] + ([ch['pool'].out] if 'pool' in ch else []), attrs, ch['pos'])
            continue
        if op in ('bn', 'relu'):
            if needs_materialise(n):
                src = n.inputs[0]
                attrs = {'bn': n.attrs if op == 'bn' else None, 'relu': op == 'relu'}
                # bn -> relu pair where only the relu is materialised: fold the bn in
                if op == 'relu' and src.node.op == 'bn' and src.node.id not in fused_into \
                        and not needs_materialise(src.node):
                    attrs['bn'] = src.node.attrs
                    src = src.node.inputs[0]
                emit('affine', [src], [n.out], attrs, n.id)
            continue
        if op == 'add':
            if n.id in add_claim:
                continue
            ups = [t for t in n.inputs if t.node.op == 'upsample' and t.id not in out_ids
                   and len(cons[t.id]) == 1]
            if len(n.inputs) == 2 and len(ups) >= 1:
                u = ups[-1]
                other = n.inputs[0] if n.inputs[1] is u else n.inputs[1]
                up_fused.add(u.node.id)
                emit('upsample_add', [other, u.node.inputs[0]], [n.out], {}, n.id)
            else:
                emit('add', n.inputs, [n.out], {}, n.id)
            continue
        if op == 'upsample':
            # decided when its consumer add is visited; emit lazily below if not fused
            if n.id in up_claimed:
                continue
            emit('upsample?', [n.inputs[0]], [n.out], {'node': n.id}, n.id)
            continue
        if op in ('slice', 'concat', 'to_clip'):
            if op == 'concat' and n.id in sam_skip:
                continue
            emit(op, n.inputs, [n.out], dict(n.attrs), n.id)
            continue
        if op == 'softmax2d':
            # channel_softmax_2d -> {softargmax2d, keypoint_confidence, depth expectation, kronecker
            # product} (spnet.py:178-235): ONE kernel; the probability map is only written if the
            # kronecker product needs it.
            users = cons[n.out.id]
            sa = [u for u in users if u.op == 'softargmax2d']
            kc = [u for u in users if u.op == 'keypoint_confidence']
            de = [u for u in users if u.op == 'depth_expect']
            kr = [u for u in users if u.op == 'kron']
            if len(sa) > 1 or len(kc) > 1 or len(de) > 1 or len(sa) + len(kc) + len(de) + len(kr) != len(users) \
                    or n.out.id in out_ids or (de and not sa) or len(sa) != len(kc):
                raise NotImplementedError('unsupported use of channel_softmax_2d output')
            if not sa:
                # probabilities only (merge model: softmax(hs) -> kronecker_prod, action.py:202,359):
                # the kernel still needs somewhere to put (x, y) and the confidence -> scratch tensors
                from .graph import Tensor
                c_ = n.out.shape[2]
                scratch = [Tensor(g_full, (1, c_, 2), n.out.kind, n, 1), Tensor(g_full, (1, c_, 1), n.out.kind, n, 2)]
                emit('sam2d', [n.inputs[0]], scratch + [n.out], {'alpha': n.attrs['alpha'], 'depth': False,
                                                                 'prob': True}, n.id)
                continue
            pose_t, pos, ins = sa[0].out, max(sa[0].id, kc[0].id), [n.inputs[0]]
            sam_skip.update([sa[0].id, kc[0].id])
            if de:
                cat = sole_consumer(sa[0].out, 'concat')
                if cat is None or sole_consumer(de[0].out, 'concat') is not cat or len(cat.inputs) != 2 \
                        or cat.inputs[0] is not sa[0].out:
                    raise NotImplementedError('depth expectation must be concatenated right after (x, y)')
                pose_t, pos = cat.out, max(pos, cat.id)
                ins.append(de[0].inputs[0])
                sam_skip.update([de[0].id, cat.id])
            outs = [pose_t, kc[0].out] + ([n.out] if kr else [])
            emit('sam2d', ins, outs, {'alpha': n.attrs['alpha'], 'depth': bool(de), 'prob': bool(kr)}, pos)
            continue
        if op in ('softargmax2d', 'keypoint_confidence', 'depth_expect'):
            if n.id not in sam_skip and not any(c_.op == 'softmax2d' for c_ in [n.inputs[-1].node]):
                raise NotImplementedError('%s is only supported on channel_softmax_2d outputs' % op)
            continue
        if op == 'global_maxmin':
            sm = sole_consumer(n.out, 'softmax')
            if sm is None:
                raise NotImplementedError('global_max_min_pooling must feed Activation(softmax)')
            emit('global_maxmin_softmax', [n.inputs[0]], [sm.out], {}, sm.id)
            continue
        if op == 'softmax':
            if n.inputs[0].node.op != 'global_maxmin':
                raise NotImplementedError('Activation(softmax) is only supported right after global_max_min_pooling')
            continue
        if op == 'maxpool' and n.id in pool_claimed:
            continue
        # everything else maps 1:1 onto a kernel op
        if op not in KERNEL_OPS:
            raise NotImplementedError('no kernel for layer op %r (node %d)' % (op, n.id))
        emit(op, n.inputs, n.outs, dict(n.attrs), n.id)

    emitted.sort(key=lambda e: (e[0], e[1]))
    kops = []
    for _, _, k in emitted:
        if k.kind == 'upsample?':
            if k.attrs['node'] in up_fused:
                continue
            k.kind = 'upsample'
        kops.append(k)
    return g, kops


def _layout(kops, inputs, outputs):
    """Phases 4-5 over scheduled ops (_schedule) that read `inputs` and must leave `outputs` intact: views become
    storage aliases, concat inputs that are not placed become copies, and buffers get physical slots by liveness.
    Sets attrs['copies'] on the concat ops it is given.  -> Plan (without stats)."""
    plan = Plan()
    out_ids = set(t.id for t in outputs)

    # ---- phase 4: storage ----------------------------------------------------------
    def new_buffer(kind, hw, ld):
        b = Buffer(len(plan.buffers), kind, hw, ld)
        plan.buffers.append(b)
        return b

    def hw_of(t):
        return t.shape[0] * t.shape[1]

    written_by = {}
    for k in kops:
        for t in k.outs:
            written_by[t.id] = k

    # concat placement: claim inputs that are plain kernel outputs
    placed = {}     # tensor id -> (concat out tensor, offset)
    for k in kops:
        if k.kind != 'concat':
            continue
        off = 0
        copies = []
        for t in k.ins:
            w = written_by.get(t.id)
            ok = (w is not None and w.kind not in ('slice', 'concat', 'to_clip') and w.kind not in DENSE_OUT_OPS
                  and t.id not in placed and t.id not in out_ids)
            if ok:
                placed[t.id] = (k.outs[0], off)
            else:
                copies.append((t, off))
            off += t.channels
        k.attrs['copies'] = copies

    def storage_of(t):
        s = plan.storage.get(t.id)
        if s is not None:
            return s
        if t.id in placed:
            parent, off = placed[t.id]
            ps = storage_of(parent)
            s = Storage(ps.buf, ps.c_off + off, ps.ld)
        else:
            w = written_by.get(t.id)
            if w is not None and w.kind == 'slice':
                ps = storage_of(w.ins[0])
                s = Storage(ps.buf, ps.c_off + w.attrs['c0'], ps.ld)
            elif w is not None and w.kind == 'to_clip':
                ps = storage_of(w.ins[0])        # (B*T, 1, nj, C) frames == (B, T, nj, C) clips
                s = Storage(ps.buf, ps.c_off, ps.ld)
            else:
                b = new_buffer(t.kind, hw_of(t), t.channels)
                s = Storage(b, 0, t.channels)
                if w is None:
                    if t.id not in input_ids:
                        raise RuntimeError('tensor %r is read by the plan but no kernel writes it (layer op %r has '
                                           'no fused or stand-alone kernel)' % (t, t.node.op if t.node else None))
                    b.is_input = True
        plan.storage[t.id] = s
        return s

    input_ids = set(t.id for t in inputs)
    for t in inputs:
        storage_of(t)
    final_kops = []
    for k in kops:
        for t in k.ins:
            storage_of(t)
        for t in k.outs:
            storage_of(t)
        if k.kind in ('slice', 'to_clip'):
            continue
        if k.kind == 'concat':
            for (t, off) in k.attrs['copies']:
                final_kops.append(KOp('copy', [t], [k.outs[0]], {'c_off': off, 'channels': t.channels}, k.pos))
            continue
        if k.attrs.get('pool_out') and not _pool_views_ok(plan.storage, k):
            # a view the wide pointwise kernel cannot take (e.g. the input at channel 3 of a concat): conv + maxpool
            attrs = dict(k.attrs, pool_out=False)
            final_kops.append(KOp(k.kind, k.ins, k.outs[:1], attrs, k.pos))
            final_kops.append(KOp('maxpool', k.outs[:1], k.outs[1:], attrs.pop('pool_attrs'), k.pos))
            continue
        final_kops.append(k)
    plan.kops = final_kops

    # ---- phase 5: liveness + physical slots -----------------------------------------
    for i, k in enumerate(plan.kops):
        for t in k.outs:
            b = plan.storage[t.id].buf
            if b.first is None:
                b.first = i
            b.last = max(b.last, i)
        for t in k.ins:
            b = plan.storage[t.id].buf
            b.last = max(b.last, i)
    for t in outputs:
        plan.storage[t.id].buf.is_output = True
    for b in plan.buffers:
        if b.is_input:
            b.first = -1
        if b.first is None:
            b.first = 0
    free = defaultdict(list)
    events = sorted(plan.buffers, key=lambda b: b.first)
    active = []
    for b in events:
        # release finished buffers
        still = []
        for a in active:
            if a.last < b.first and not a.is_output and not a.is_input:
                free[(a.kind, a.floats_per_item)].append(a.phys)
            else:
                still.append(a)
        active = still
        key = (b.kind, b.floats_per_item)
        if b.is_output or b.is_input or not free[key]:
            b.phys = len(plan.phys)
            plan.phys.append(key)
        else:
            b.phys = free[key].pop()
        active.append(b)
    return plan


def verify_plan(plan, g):
    """Independent replay of a plan's buffer assignment (the planner above is liveness + greedy slot reuse; this is
    the check that it is memory-safe, used by the tests on every BASELINE model): walking the launches in order,
      * every channel range a launch reads was written before, by launches of the SAME logical buffer, and no other
        buffer has taken over the physical slot in between;
      * no launch writes a slot it is reading through another buffer, or a channel range of its own input;
      * every model output is intact after the last launch;
      * a conv with a pooled second output is one the wide pointwise kernel takes: its shared memory within the limit
        and every view 16-byte aligned.
    Returns the number of (launch, operand) pairs checked; raises AssertionError naming the launch otherwise."""
    owner, written, checked = {}, {}, 0

    def covered(spans, lo, hi):
        pos = lo
        for a, b in sorted(spans):
            if a > pos:
                break
            pos = max(pos, b)
        return pos >= hi

    def span(t):
        s = plan.storage[t.id]
        return s.buf, s.c_off, s.c_off + t.channels

    for t in g.inputs:
        b, lo, hi = span(t)
        owner[b.phys] = b.id
        written[b.id] = [(lo, hi)]
    for i, k in enumerate(plan.kops):
        if k.attrs.get('pool_out'):
            assert pw_smallk_smem(k.ins[0].channels, k.outs[0].channels) <= PW_SMALLK_SMEM_MAX, \
                'launch %d (%s) fuses a pool but its weights do not fit the wide pointwise kernel' % (i, k.kind)
            assert _pool_views_ok(plan.storage, k), \
                'launch %d (%s) fuses a pool but not all of its views are 16-byte aligned' % (i, k.kind)
        reads = [span(t) for t in k.ins]
        for t, (b, lo, hi) in zip(k.ins, reads):
            assert owner.get(b.phys) == b.id, \
                'launch %d (%s) reads %r but its slot %d holds buffer %r' % (i, k.kind, t, b.phys, owner.get(b.phys))
            assert covered(written[b.id], lo, hi), \
                'launch %d (%s) reads channels [%d, %d) of %r that no earlier launch wrote' % (i, k.kind, lo, hi, t)
            checked += 1
        for t in k.outs:
            b, lo, hi = span(t)
            if k.kind == 'copy':        # a concat input copied into place: only its own channel range is written
                lo, hi = lo + k.attrs['c_off'], lo + k.attrs['c_off'] + k.attrs['channels']
            for u, (bu, ulo, uhi) in zip(k.ins, reads):
                if bu.phys != b.phys:
                    continue
                assert bu is b, 'launch %d (%s) writes %r into the slot of its own operand %r' % (i, k.kind, t, u)
                assert hi <= ulo or uhi <= lo, \
                    'launch %d (%s) overwrites channels of its own operand %r' % (i, k.kind, u)
            if owner.get(b.phys) != b.id:
                owner[b.phys] = b.id
                written[b.id] = []
            written[b.id].append((lo, hi))
            checked += 1
    for t in g.outputs:
        b, lo, hi = span(t)
        assert owner.get(b.phys) == b.id and covered(written[b.id], lo, hi), 'model output %r is not intact' % (t,)
    return checked
