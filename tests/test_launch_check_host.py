"""tests/launch_check.py checked without a GPU: on the stand-in device (tests/fake_cuda.py --arithmetic) it must pass
the correct stand-in kernels on reduced models and fuzz graphs, and catch -- naming the launch -- each of a set of
wrong stand-ins: a write outside the output view, a skipped item, a write into a slot's guard band, an unwritten head
output, an unwritten pooled output, one dropped product term of a convolution.  Its conv error bounds are checked on
numpy emulations of the kernels' arithmetic: they hold, and they break when one K-term is dropped."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import gpu_util as G  # noqa: E402


# ---- the models ----------------------------------------------------------------------------------------------------------
def _models(name):
    """name -> (model with weights, input)"""
    sys.path.insert(0, os.path.join(ROOT, 'tests', 'golden'))
    from deephar_b200 import action, reception, spnet
    from deephar_b200.config import ModelConfig, pa16j2d
    from deephar_b200.model import Model
    from oracle import synth
    from ref_cases import MERGE_CASE
    from test_compiler_fuzz import _random_graph
    if name == 'reception2d':
        m = reception.build((128, 128, 3), num_joints=16, dim=2, num_context_per_joint=2, num_blocks=2, ksize=(5, 5),
                            concat_pose_confidence=False)
        return m.init_synthetic_weights(1234), synth.synth_frames(3, 128, 128, seed=5)
    if name == 'spnet_penn_t2':
        m = spnet.build(ModelConfig((2, 128, 128, 3), pa16j2d, num_actions=[15], num_pyramids=2, action_pyramids=[1, 2],
                                    num_levels=4, pose_replica=True, num_pose_features=160, num_visual_features=160))
        return m.init_synthetic_weights(1234), synth.synth_frames(4, 128, 128, seed=6).reshape(2, 2, 128, 128, 3)
    if name == 'merge2d':
        mc = MERGE_CASE
        pe = reception.build(mc['input_shape'], **mc['reception'])
        m = action.build_merge_model(pe, mc['num_actions'], mc['input_shape'], mc['num_frames'], mc['num_joints'],
                                     mc['num_blocks'], pose_dim=2)
        x = synth.synth_frames(mc['num_frames'], 64, 64, seed=7).reshape((1, mc['num_frames'], 64, 64, 3))
        return m.init_synthetic_weights(mc['seed']), x
    seed = int(name[len('fuzz'):])
    g, side = _random_graph(seed)
    m = Model(g, name=g.name).init_synthetic_weights(seed)
    return m, np.random.default_rng(1000 + seed).uniform(-1, 1, (3, side, side, 3))


def _first_fuzz_with_pool_out():
    from deephar_b200.model import Model
    from test_compiler_fuzz import _random_graph
    for seed in range(60):
        g, _ = _random_graph(seed)
        if any(k.kind == 'conv' and k.attrs.get('pool_out') for k in Model(g, name=g.name).plan.kops):
            return 'fuzz%d' % seed


# ---- wrong stand-ins ---------------------------------------------------------------------------------------------------------
def _first(m, pred):
    return next(i for i, k in enumerate(m.plan.kops) if pred(k))


def _dense(m, t):
    s = m.plan.storage[t.id]
    return s.c_off == 0 and s.ld == t.shape[2]


def _mutate(name, m):
    """installs the wrong stand-in `name` into fake_cuda.ARITHMETIC; returns the index of the launch that must be named"""
    import fake_cuda as F
    A = F.ARITHMETIC
    conv, pool = A['dh_conv2d_f32'], A['dh_maxpool2d_f32']
    if name == 'conv_writes_past_its_channels':
        def op(ctx, x, w, packed, d, out, stream):
            conv(ctx, x, w, packed, d, out, stream)
            v = out.contents
            if v.ld > v.c:                      # channel c of the view: the next slice of the concat buffer
                F._f32(v.p, (v.n * v.h * v.w - 1) * v.ld + v.c + 1)[v.c::v.ld] = 1.0
        A['dh_conv2d_f32'] = op
        return _first(m, lambda k: k.kind == 'conv' and m.plan.storage[k.outs[0].id].ld > k.outs[0].shape[2])
    if name == 'maxpool_skips_last_item':
        def op(ctx, x, kh, kw, sh, sw, pad, out, stream):
            o = F._view(out)
            keep = o[-1].copy()
            pool(ctx, x, kh, kw, sh, sw, pad, out, stream)
            o[-1] = keep
        A['dh_maxpool2d_f32'] = op
        return _first(m, lambda k: k.kind == 'maxpool')
    if name == 'write_past_the_slot':
        def op(ctx, x, kh, kw, sh, sw, pad, out, stream):
            pool(ctx, x, kh, kw, sh, sw, pad, out, stream)
            v = out.contents
            if v.ld == v.c:                     # a dense output: the float after its last element is past the slot
                end = v.n * v.h * v.w * v.ld
                F._f32(v.p, end + 1)[end] = 0.5
        A['dh_maxpool2d_f32'] = op
        return _first(m, lambda k: k.kind == 'maxpool' and _dense(m, k.outs[0]))
    if name == 'head_leaves_last_confidence':
        base = A['dh_softargmax2d_ctx_f32']

        def op(ctx, h, nj, n_ctx, alpha, out_pose, out_vis, stream):
            vis = F._f32(out_vis, h.contents.n * nj)
            keep = vis[-1:].copy()              # bit for bit: a float() round trip would quieten a signalling NaN
            base(ctx, h, nj, n_ctx, alpha, out_pose, out_vis, stream)
            vis[-1:] = keep
        A['dh_softargmax2d_ctx_f32'] = op
        return _first(m, lambda k: k.kind == 'pose_regression_2d_context')
    if name == 'pool_out_never_written':
        def op(ctx, x, w, packed, d, out, stream):
            dd = d.contents
            keep = dd.pool_out.p
            dd.pool_out.p = None
            try:
                conv(ctx, x, w, packed, d, out, stream)
            finally:
                dd.pool_out.p = keep
        A['dh_conv2d_f32'] = op
        return _first(m, lambda k: k.kind == 'conv' and k.attrs.get('pool_out'))
    if name == 'conv_drops_one_term':
        def op(ctx, x, w, packed, d, out, stream):
            dd = d.contents
            cin, cout = x.contents.c, out.contents.c
            wt = F._f32(w, dd.kh * dd.kw * cin * cout)
            at = ((dd.kh // 2) * dd.kw + dd.kw // 2) * cin * cout      # centre tap, input channel 0, output channel 0
            keep = float(wt[at])
            wt[at] = 0.0
            try:
                conv(ctx, x, w, packed, d, out, stream)
            finally:
                wt[at] = keep
        A['dh_conv2d_f32'] = op
        return _first(m, lambda k: k.kind == 'conv')
    raise KeyError(name)


MUTATIONS = {       # mutation: the model it runs on
    'conv_writes_past_its_channels': 'reception2d',
    'maxpool_skips_last_item': 'reception2d',
    'write_past_the_slot': 'reception2d',
    'head_leaves_last_confidence': 'reception2d',
    'pool_out_never_written': None,          # the first fuzz graph with a pooled second output
    'conv_drops_one_term': 'reception2d',
}


def _run(scenario):
    """in the subprocess: the stand-in device, then the checker on `scenario` -> one JSON line"""
    import fake_cuda
    from launch_check import LaunchChecker, LaunchError
    if scenario in MUTATIONS:
        model = MUTATIONS[scenario] or _first_fuzz_with_pool_out()
        fake_cuda.install(arithmetic=True)
        m, x = _models(model)
        expect = _mutate(scenario, m)
        try:
            LaunchChecker(m).run(x)
            err = None
        except LaunchError as e:
            err = str(e)
        print(json.dumps({'model': model, 'expect': expect, 'error': err}))
        return
    fake_cuda.install(arithmetic=True)
    names = scenario.split(',')
    res = {}
    for name in names:
        m, x = _models(name)
        ch = LaunchChecker(m)
        outs = ch.run(x)
        want = m.predict(np.asarray(x, np.float32))
        want = want if isinstance(want, list) else [want]
        same = len(outs) == len(want) and all(np.array_equal(o, w.reshape(o.shape)) for o, w in zip(outs, want))
        res[name] = dict(launches=ch.launches, kops=len(m.plan.kops), same_as_predict=same,
                         checked=sorted('%s/%s' % kp for kp in ch.checked))
    print(json.dumps(res))


def _subprocess(scenario):
    out = subprocess.run([sys.executable, os.path.abspath(__file__), scenario], capture_output=True, text=True,
                         timeout=1700, cwd=ROOT)
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-3000:]
    return json.loads(out.stdout.strip().splitlines()[-1])


@pytest.mark.timeout(1800)
@pytest.mark.parametrize('models', ['reception2d,merge2d', 'spnet_penn_t2', ','.join('fuzz%d' % s for s in range(10))])
def test_checker_passes_the_stand_in(models):
    res = _subprocess(models)
    for name, r in res.items():
        assert r['launches'] == r['kops'], (name, r)
        assert r['same_as_predict'], (name, r)      # the product's own forward on the same stand-in kernels


@pytest.mark.timeout(1800)
@pytest.mark.parametrize('mutation', sorted(MUTATIONS))
def test_checker_catches_and_names_the_launch(mutation):
    r = _subprocess(mutation)
    assert r['error'] is not None, 'the checker passed a wrong %s' % mutation
    assert r['error'].startswith('launch %d (' % r['expect']), (r['expect'], r['error'])
    if mutation == 'write_past_the_slot':
        assert 'guard band' in r['error'], r['error']
    if mutation == 'conv_drops_one_term':
        assert 'out of bound' in r['error'] and 'channel 0:' in r['error'], r['error']
    if mutation in ('maxpool_skips_last_item', 'head_leaves_last_confidence', 'pool_out_never_written'):
        assert 'unwritten' in r['error'], r['error']


# ---- the conv bounds on emulated kernel arithmetic -------------------------------------------------------------------------
def _layer(seed=3, m=256, k=576, n=48):
    rng = np.random.default_rng(seed)
    a = G.f32(np.maximum(rng.standard_normal((m, k)), 0))          # a ReLU'd activation
    w = G.f32(rng.standard_normal((k, n)) / np.sqrt(k))
    return a, w


def _bf16x3_terms(a, w):
    """(M, K, N) products of the three bf16 pairs the split-precision MMA accumulates: hi*hi + hi*lo + lo*hi"""
    ah, wh = G.bf16(a), G.bf16(w)
    al, wl = G.bf16(a - ah), G.bf16(w - wh)
    return ah[:, :, None] * wh[None] + ah[:, :, None] * wl[None] + al[:, :, None] * wh[None]


def _accumulate(terms, step):
    """fp32 accumulation of the K axis, rounded once per k-step of `step` terms"""
    acc = np.zeros((terms.shape[0], terms.shape[2]), np.float32)
    for k0 in range(0, terms.shape[1], step):
        acc = np.float32(acc + terms[:, k0:k0 + step].sum(axis=1))
    return acc.astype(np.float64)


def _drop(terms, k0=7, n0=5):
    t = terms.copy()
    t[:, k0, n0] = 0.0
    return t


@pytest.mark.parametrize('arith', ['bf16x3', 'ffma'])
def test_conv_bound_holds_and_catches_one_dropped_term(arith):
    a, w = _layer()
    ref = a @ w
    s = np.abs(a) @ np.abs(w)
    k = a.shape[1]
    if arith == 'bf16x3':
        terms = _bf16x3_terms(a, w)
        step = 16
        bound = G.tc_dense_bound(np.sqrt((a * a) @ (w * w)), s, k)
    else:
        terms = a[:, :, None] * w[None]
        step = 1
        bound = G.ffma_dense_bound(s, k)
    got = _accumulate(terms, step)
    assert np.all(np.abs(got - ref) <= bound)
    assert np.abs(got - ref).max() > 0                         # the emulation does round
    bad = np.abs(_accumulate(_drop(terms), step) - ref) > bound
    assert not bad[:, np.arange(w.shape[1]) != 5].any()
    nz = a[:, 7] != 0                                          # rows whose dropped term is not zero
    assert nz.sum() > 50 and bad[nz, 5].mean() > 0.9, bad[nz, 5].mean()


def test_ffma_bound_holds_where_the_products_underflow():
    """outputs below 2^-126 (an action-head conv on near-zero pose maps) are subnormal: fp32 rounds them to multiples
    of 2^-149, an absolute error the relative bound alone misses and the 2^-150 per rounding of gpu_util covers"""
    a, w = _layer()
    a = G.f32(a * 2.0 ** -140)
    ref = a @ w
    s = np.abs(a) @ np.abs(w)
    k = a.shape[1]
    got = _accumulate(a[:, :, None] * w[None], 1)
    assert np.abs(ref).max() < 2.0 ** -126 and np.abs(got - ref).max() > 0
    relative = G.ffma_dense_bound(s, k)
    assert (np.abs(got - ref) > relative).mean() > 0.5
    assert np.all(np.abs(got - ref) <= relative + G.UNDERFLOW * k)


def test_bf16x3_bound_holds_where_the_operands_are_subnormal():
    """A operands near 1e-39 (below 2^-117) split into bf16 parts of subnormal spacing 2^-133: the relative split term
    misses it, the 2^-134 * sum |w| of gpu_util covers it"""
    a, w = _layer()
    a = G.f32(a * 2.0 ** -130)
    ref = a @ w
    s = np.abs(a) @ np.abs(w)
    k = a.shape[1]
    got = _accumulate(_bf16x3_terms(a, w), 16)
    relative = G.tc_dense_bound(np.sqrt((a * a) @ (w * w)), s, k) + G.UNDERFLOW * k
    assert (np.abs(got - ref) > relative).mean() > 0.5
    assert np.all(np.abs(got - ref) <= relative + G.SPLIT_FLOOR * np.abs(w).sum(axis=0))


def _maxmin_softmax_f32(x):
    """elementwise.cu's global_maxmin_softmax_kernel in fp32: s_c = max + min over the map, softmax over c"""
    x = np.float32(x)
    s = np.float32(x.max(axis=(1, 2)) + x.min(axis=(1, 2)))
    e = np.exp(np.float32(s - s.max(axis=-1, keepdims=True)))
    return (e / np.float32(e.sum(axis=-1, keepdims=True, dtype=np.float32))).astype(np.float64)


def test_softmax_bound_scales_with_the_logits():
    """logits in the hundreds: rounding s_c and s_c - max costs ~2^-24 * |s| of each exponent, more than the flat 1e-6;
    the 8 L 2^-24 p of the launch checker covers it"""
    from launch_check import HEAD_TOL, LaunchChecker
    x = G.f32(np.random.default_rng(5).uniform(-1, 1, (64, 4, 4, 15)) * 2 + 150)     # close logits near 300
    s = x.max(axis=(1, 2)) + x.min(axis=(1, 2))
    e = np.exp(s - s.max(axis=-1, keepdims=True))
    ref = e / e.sum(axis=-1, keepdims=True)
    err = np.abs(_maxmin_softmax_f32(x) - ref)
    flat = HEAD_TOL['global_maxmin_softmax'][0]
    assert (err > flat).any()
    assert np.all(err <= flat + LaunchChecker.softmax_logit_bound(x, ref))


if __name__ == '__main__':
    sys.path.insert(0, os.path.join(ROOT, 'tests'))
    _run(sys.argv[1])
