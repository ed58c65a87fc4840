"""Compiler fuzzing without a GPU: random layer graphs (Conv2D / SeparableConv2D with strides and 'same' / 'valid' padding,
BatchNormalization with and without gamma, ReLU, n-ary add, max-pooling, 2x upsampling, concatenation, channel slices,
zero padding, fused soft-argmax heads with depth expectation and kronecker product; several outputs, shared sub-expressions, tensors that are both an output and an operand) are compiled, the
plan is replayed for memory safety (`compiler.verify_plan`) and EXECUTED on the CPU by tests/plan_emulator.py, and the
result must equal a plain node-by-node evaluation of the un-fused graph.  Whatever fusion, view or buffer-reuse decision
the compiler takes on a topology the reference models never produce, it may not change the function."""
import numpy as np
import pytest

from deephar_b200 import layers as L
from deephar_b200.compiler import verify_plan
from deephar_b200.graph import Graph
from deephar_b200.model import Model
from oracle import ops_np as O
from plan_emulator import PlanEmulator


def _interpret(g, weights, x):
    """The layer graph as Keras would run it: one op per node, nothing fused, every tensor its own array."""
    hw = {k: np.asarray(v, np.float64) for k, v in weights.items()}
    val = {g.inputs[0].id: np.asarray(x, np.float64)}

    def ev(t):
        if t.id in val:
            return val[t.id]
        nd, a = t.node, t.node.attrs
        ins = [ev(i) for i in nd.inputs]
        if nd.op == 'conv':
            y = O.conv2d(ins[0], hw[a['kernel']], tuple(a['strides']), a['padding'])
        elif nd.op == 'sepconv':
            y = O.separable_conv2d(ins[0], hw[a['depthwise']], hw[a['pointwise']], tuple(a['strides']), a['padding'])
        elif nd.op == 'bn':
            w = a['weights']
            y = O.batchnorm(ins[0], hw[w['gamma']] if 'gamma' in w else None, hw[w['beta']], hw[w['mean']], hw[w['var']])
        elif nd.op == 'relu':
            y = O.relu(ins[0])
        elif nd.op == 'add':
            y = sum(ins)
        elif nd.op == 'maxpool':
            y = O.maxpool2d(ins[0], tuple(a['pool']), tuple(a['strides']), a['padding'])
        elif nd.op == 'upsample':
            y = O.upsample2d(ins[0])
        elif nd.op == 'concat':
            y = np.concatenate(ins, axis=-1)
        elif nd.op == 'slice':
            y = ins[0][..., a['c0']:a['c1']]
        elif nd.op == 'zeropad':
            y = O.zeropad2d(ins[0], a['pads'])
        elif nd.op == 'softmax2d':
            y = O.channel_softmax_2d(ins[0], a['alpha'])
        elif nd.op == 'softargmax2d':
            y = O.softargmax2d(ins[0])
        elif nd.op == 'keypoint_confidence':
            y = O.keypoint_confidence(ins[0])
        elif nd.op == 'depth_expect':
            y = np.sum(O.sigmoid(ins[0]) * ins[1], axis=(1, 2))[..., None]
        elif nd.op == 'kron':
            y = np.einsum('nhwj,nhwf->njf', ins[0], ins[1])
        else:
            raise NotImplementedError(nd.op)
        val[t.id] = y
        return y
    return [ev(t) for t in g.outputs]


def _random_graph(seed):
    rng = np.random.default_rng(seed)
    g = Graph('fuzz%d' % seed)
    side = int(rng.choice([16, 32]))
    pool = [L.conv2d(g.input((side, side, 3)), int(rng.choice([8, 16])), (3, 3), strides=(1, 1))]
    heads = []
    pick = lambda: pool[int(rng.integers(max(0, len(pool) - 6), len(pool)))]           # noqa: E731  (recent tensors)
    for _ in range(int(rng.integers(10, 26))):
        op = rng.choice(['conv', 'conv', 'sepconv', 'sepconv', 'bn', 'relu', 'relu', 'add', 'add', 'pool', 'up', 'concat',
                         'slice', 'pad', 'hourglass', 'blockend', 'head'])
        x = pick()
        h, w, c = x.shape
        if op == 'hourglass':
            # the shape the compiler fuses into ONE separable-conv launch: add([sepconv(..), UpSampling2D(low)]) on 16- / 32-
            # pixel-wide maps with a multiple of 32 channels (reception.py:122-127) -- plus near misses of that shape
            wide = [t for t in pool if t.shape[1] in (16, 32) and t.shape[0] % 2 == 0]
            if not wide:
                continue
            x = wide[int(rng.integers(len(wide)))]
            h, w, c = x.shape
            ch = int(rng.choice([32, 64, 48]))
            if c != ch:
                x = L.conv2d(L.relu(x), ch, (1, 1))
                pool.append(x)
            low = L.sepconv2d(L.relu(L.MaxPooling2D(x, (2, 2))), ch, (3, 3))
            a = L.BatchNormalization(L.sepconv2d(L.relu(x), ch, (int(rng.choice([3, 5])),) * 2), scale=False)
            y = L.add([a, L.UpSampling2D(low)] if rng.random() < 0.7 else [L.UpSampling2D(low), a, x])
        elif op == 'head':
            # prediction heads as the compiler fuses them into one launch (spnet.py:178-235): heat-maps -> channel soft-max
            # -> soft-argmax + joint confidence [+ depth expectation concatenated as z] [+ kronecker product with features]
            if min(h, w) < 4:
                continue
            nj = int(rng.choice([5, 8, 16]))
            hm = L.conv2d(L.relu(x), nj, (1, 1))
            prob = L.channel_softmax_2d(hm, alpha=float(rng.choice([1.0, 2.0])))
            pose, conf = L.softargmax2d(prob), L.keypoint_confidence(prob)
            if rng.random() < 0.4:
                pose = L.concatenate([pose, L.depth_expectation(L.conv2d(L.relu(x), nj, (1, 1)), prob)])
            heads.extend([pose, conf])
            if rng.random() < 0.5:
                heads.append(L.kronecker_prod(prob, x))
            y = L.conv2d(L.relu(L.concatenate([hm, x])), c, (1, 1))                    # re-injection of the heat-maps
        elif op == 'blockend':
            # ... and the block-end: add([x, wide 1x1 conv of a narrow map]) whose 2x2 max-pool becomes the conv kernel's
            # second output on 32-pixel-wide maps (reception.py:108-110, 285-312)
            if w != 32 or h % 2:
                continue
            cout = int(rng.choice([128, 160]))
            trunk = L.conv2d(L.relu(x), cout, (1, 1)) if c != cout else x
            narrow = L.conv2d(L.relu(trunk), int(rng.choice([48, 64, 24])), (1, 1), padding='valid')
            y = L.add([trunk, L.BatchNormalization(L.conv2d(L.relu(narrow), cout, (1, 1)), scale=False)])
            pool.append(y)
            y = L.MaxPooling2D(y, (2, 2))
        elif op in ('conv', 'sepconv'):
            k = int(rng.choice([1, 3, 5])) if op == 'conv' else int(rng.choice([3, 5]))
            s = 2 if (h >= 8 and h % 2 == 0 and rng.random() < 0.25) else 1
            padding = 'valid' if (k <= min(h, w) and k > 1 and h - k + 1 >= 4 and rng.random() < 0.15) else 'same'
            f = int(rng.choice([8, 12, 16, 24, 32]))
            y = (L.conv2d if op == 'conv' else L.sepconv2d)(x, f, (k, k), strides=(s, s), padding=padding)
        elif op == 'bn':
            y = L.BatchNormalization(x, scale=bool(rng.random() < 0.5))
        elif op == 'relu':
            y = L.relu(x)
        elif op == 'add':
            same = [t for t in pool if t.shape == x.shape and t is not x]
            if not same:
                continue
            others = [same[int(i)] for i in rng.choice(len(same), size=min(len(same), int(rng.integers(1, 4))), replace=False)]
            y = L.add([x] + others)
        elif op == 'pool':
            if h < 4 or w < 4:
                continue
            kind = int(rng.integers(3))
            y = (L.MaxPooling2D(x, (2, 2)) if kind == 0 and h % 2 == 0 else
                 L.maxpooling2d(x) if kind == 1 else L.MaxPooling2D(x, (3, 3), strides=(2, 2), padding='same'))
        elif op == 'up':
            if h > 16:
                continue
            y = L.UpSampling2D(x)
        elif op == 'concat':
            same = [t for t in pool if t.shape[:2] == x.shape[:2] and t is not x]
            if not same:
                continue
            y = L.concatenate([x, same[int(rng.integers(len(same)))]])
        elif op == 'slice':
            if c < 4:
                continue
            c0 = int(rng.integers(0, c - 2))
            y = L.channel_slice(x, c0, int(rng.integers(c0 + 1, c + 1)))
        else:
            y = L.ZeroPadding2D(x, ((int(rng.integers(0, 2)), int(rng.integers(0, 3))), (int(rng.integers(0, 3)), 0)))
        pool.append(y)
    n_out = int(rng.integers(1, 4))
    outs = [pool[-1]] + [pool[int(i)] for i in rng.choice(len(pool) - 1, size=min(n_out - 1, len(pool) - 1), replace=False)]
    g.outputs = outs + heads
    return g, side


def test_the_fuzzer_reaches_the_special_fusions():
    fused_up = fused_pool = heads = heads_z = heads_kron = 0
    for seed in range(60):
        g, _ = _random_graph(seed)
        kops = Model(g, name=g.name).plan.kops
        fused_up += sum(1 for k in kops if k.kind == 'sepconv' and k.attrs.get('res_up2x'))
        fused_pool += sum(1 for k in kops if k.kind == 'conv' and k.attrs.get('pool_out'))
        heads += sum(1 for k in kops if k.kind == 'sam2d')
        heads_z += sum(1 for k in kops if k.kind == 'sam2d' and k.attrs['depth'])
        heads_kron += sum(1 for k in kops if k.kind == 'sam2d' and k.attrs['prob'])
    assert fused_up >= 5 and fused_pool >= 5 and heads >= 20 and heads_z >= 5 and heads_kron >= 5, \
        (fused_up, fused_pool, heads, heads_z, heads_kron)


def test_upsampled_residual_is_the_last():
    """dh_conv_desc.res_up2x may only flag a conv's last residual (include/deephar_b200.h); the library refuses any
    other launch.  Seed 24 once fused a further add behind the upsampled residual of an hourglass sepconv."""
    for seed in range(60):
        g, _ = _random_graph(seed)
        for k in Model(g, name=g.name).plan.kops:
            if k.kind in ('conv', 'sepconv') and k.attrs.get('res_up2x'):
                assert k.attrs['res_up2x'] == 1 << (k.attrs['n_res'] - 1), (seed, k)


@pytest.mark.parametrize('seed', range(60))
def test_random_graph_compiles_to_the_same_function(seed):
    g, side = _random_graph(seed)
    m = Model(g, name=g.name).init_synthetic_weights(seed)
    assert verify_plan(m.plan, m.graph) > 0
    x = np.random.default_rng(1000 + seed).uniform(-1, 1, (2, side, side, 3))
    want = _interpret(m.graph, m.get_weights(), x)
    got = PlanEmulator(m).run(x)
    assert len(got) == len(want)
    for i, (o, r) in enumerate(zip(got, want)):
        r = r.reshape(o.shape)
        assert np.isfinite(o).all(), (seed, i)
        assert np.abs(o - r).max() <= 1e-9 * max(1.0, np.abs(r).max()), (seed, i, float(np.abs(o - r).max()))


def pool_edge_graph(cin, cout, before=0, after=0):
    """MaxPooling2D((2,2)) of a wide 1x1 conv (cin -> cout) on 32 x 32 maps: the shape the compiler fuses into the wide
    pointwise kernel as its pooled second output.  The conv reads a map b of cin channels that sits at channel `before`
    of concatenate([conv(x, before), b, conv(x, after)]) when before or after is set (a view with ld = before + cin +
    after), so the shared-memory limit and the view alignment of the fusion can each be put at their edges."""
    g = Graph('pool_edge_%d_%d_%d_%d' % (cin, cout, before, after))
    x = g.input((32, 32, 3))
    b = L.conv2d(x, cin, (1, 1), name='b')
    y = L.conv2d(L.relu(b), cout, (1, 1), name='wide')
    g.outputs = [L.MaxPooling2D(y, (2, 2))]
    if before or after:
        parts = ([L.conv2d(x, before, (1, 1), name='before')] if before else []) + [b] + \
                ([L.conv2d(x, after, (1, 1), name='after')] if after else [])
        g.outputs.append(L.concatenate(parts))
    return g


def _pool_fused(m):
    wide = [k for k in m.plan.kops if k.kind == 'conv' and k.attrs['kernel'].startswith('wide/')]
    assert len(wide) == 1
    return bool(wide[0].attrs.get('pool_out'))


# (cin, cout, before, after, fused): 708 and 960 are the widest Cout (multiple of 4) whose weights and 64-pixel tile fit
# the wide pointwise kernel's 200 KB at Cin 64 and 48 (compiler.pw_smallk_smem: 64 -> 712 needs 204 864 B); a view at
# channel 3 of 51 or with ld = 53 is not 16-byte aligned
POOL_EDGES = [(64, 708, 0, 0, True), (64, 712, 0, 0, False), (48, 960, 0, 0, True), (48, 964, 0, 0, False),
              (48, 128, 3, 0, False), (48, 128, 4, 0, True), (48, 128, 4, 1, False)]


@pytest.mark.parametrize('cin,cout,before,after,fused', POOL_EDGES)
def test_pool_fusion_only_where_the_wide_pointwise_kernel_takes_it(cin, cout, before, after, fused):
    """the compiler fuses the pool only where dh_pw_smallk_supported takes the conv; elsewhere it is a conv and a
    maxpool launch, and the plan still computes the graph"""
    from deephar_b200.compiler import pw_smallk_smem
    assert (pw_smallk_smem(cin, cout) <= 200 * 1024) == bool(fused or before % 4 or (before + cin + after) % 4)
    g = pool_edge_graph(cin, cout, before, after)
    m = Model(g, name=g.name).init_synthetic_weights(7)
    assert _pool_fused(m) == fused
    kinds = [k.kind for k in m.plan.kops]
    assert kinds.count('maxpool') == (0 if fused else 1)
    assert verify_plan(m.plan, m.graph) > 0
    x = np.random.default_rng(cout).uniform(-1, 1, (2, 32, 32, 3))
    want = _interpret(m.graph, m.get_weights(), x)
    got = PlanEmulator(m).run(x)
    for i, (o, r) in enumerate(zip(got, want)):
        assert np.abs(o - r.reshape(o.shape)).max() <= 1e-9 * max(1.0, np.abs(r).max()), i


def test_verify_plan_refuses_a_pool_on_a_view_the_kernel_cannot_take():
    g = pool_edge_graph(48, 128, 3, 0)
    m = Model(g, name=g.name)
    k = next(k for k in m.plan.kops if k.kind == 'conv' and k.attrs['kernel'].startswith('wide/'))
    i = m.plan.kops.index(k)
    pool = m.plan.kops[i + 1]
    assert pool.kind == 'maxpool' and pool.ins == k.outs
    # undo the split: the conv writes the pooled map itself, from its input at channel 3 of 51
    m.plan.kops[i:i + 2] = [type(k)(k.kind, k.ins, k.outs + pool.outs, dict(k.attrs, pool_out=True), k.pos)]
    with pytest.raises(AssertionError, match='16-byte aligned'):
        verify_plan(m.plan, m.graph)
