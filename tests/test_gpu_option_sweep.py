"""The builder options off the BASELINE configs (tests/golden/ref_option_sweep.npz: no / one context map, alpha, heat-map
and feature export, depth_maps, 3x3 kernels, 3 pyramid levels, growth, predict_rootz, pa20j3d, two action sets, sam_alpha,
image_div, 3 pyramids) on the GPU.  Their layers -- separable convolutions on 4x4 and 2x2 maps, 3x3 BN-prologue layers on
288-480 channels, action-head convolutions on 2-3 channels, 20-joint heads down to 2x2 maps -- run nowhere else on the GPU.

  * parity: Model.predict against the reference builders' stored outputs, per element within 1e-3 of max(1, |ref|), under
    the policy of test_reference_golden.py::test_product_matches_reference_graph (context poses bounded by the condition
    number of the context division, exported heat-maps by their arg-max pixel);
  * launch contracts (tests/launch_check.py) on the stored input, and on a batch that gives every persistent kernel
    several tiles or frames per CTA (2 * SMs + 5 frames), where the outputs must also equal a plain forward and a
    CUDA-graph replay bit for bit;
  * the convolutions the library leaves to the generic CUDA-core kernel, per case.

    pytest -m gpu tests/test_gpu_option_sweep.py -s
"""
import os
import sys

import numpy as np
import pytest

from deephar_b200 import _ffi
from deephar_b200.model import _weight_key
from oracle import ops_np
from oracle import reception as oracle_reception

from test_gpu_launch_contracts import _check, _input, _report

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden'))
from ref_cases import option_sweep_cases  # noqa: E402

pytestmark = pytest.mark.gpu

SWEEP = option_sweep_cases()

# the convolutions each case leaves to the generic CUDA-core kernel at its stored input (measured on an H100 SXM): the
# separable convs on 2x2 maps and the action-head separable convs on 4 or 8 x 10 maps, which no tensor-core kernel takes
FALLBACKS = {          # case: layers, in binding order
    0: ['rBlock1/sepconv_l3_1_conv', 'rBlock1/sepconv_l3_2_conv', 'rBlock1/sepconv_l3_3_conv'],
    1: ['rBlock1/sepconv_l3_1_conv', 'rBlock1/sepconv_l3_2_conv', 'rBlock1/sepconv_l3_3_conv',
        'rBlock2/sepconv_l3_1_conv', 'rBlock2/sepconv_l3_2_conv', 'rBlock2/sepconv_l3_3_conv'],
    2: ['rBlock1/sepconv_l3_1_conv', 'rBlock1/sepconv_l3_2_conv', 'rBlock1/sepconv_l3_3_conv',
        'rBlock2/sepconv_l3_1_conv', 'rBlock2/sepconv_l3_2_conv', 'rBlock2/sepconv_l3_3_conv'],
    3: ['rBlock1/sepconv_l3_1_conv', 'rBlock1/sepconv_l3_2_conv', 'rBlock1/sepconv_l3_3_conv',
        'rBlock2/sepconv_l3_1_conv', 'rBlock2/sepconv_l3_2_conv', 'rBlock2/sepconv_l3_3_conv'],
    4: [],
    5: ['dp1_du3_r0_conv1', 'dp1_pb3_r1_conv1', 'dp1_pb3_conv1'],
    6: ['dp1_du3_r0_conv1', 'dp1_pb3_r1_conv1', 'dp1_pb3_conv1'],
    7: ['dp1_du2_action_r0_conv1', 'dp1_du3_r0_conv1', 'dp1_du3_action_r0_conv1', 'dp1_pb3_r1_conv1',
        'dp1_pb3_conv1', 'up2_uu2_action_r0_conv1', 'up2_uu1_action_r0_conv1', 'up2_uu0_action_r0_conv1'],
    8: ['up2_uu1_action_r0_conv1', 'up2_uu0_action_r0_conv1'],
    9: ['dp1_du3_r0_conv1', 'dp1_pb3_r1_conv1', 'dp1_pb3_conv1', 'dp3_du3_r0_conv1', 'dp3_pb3_r1_conv1',
        'dp3_pb3_conv1'],
}

# SPNet pose outputs (soft-argmax depth, visibility) that amplify the rounding of the launches before them ~10^4-fold:
# every launch is within its own bound (the launch-contract tests below), yet even the fp32 CUDA-core kernels alone miss
# 1e-3 on one of them.  Worst element at the stored input on an H100 SXM, fp32 CUDA-core kernels only
# (use_tensor_cores = False) / bf16x3 tensor cores: case 7 output 3: 3.5e-4 / 6.4e-3, output 4: 3.4e-3 / 1.5e-2; case 8
# output 2: 1.1e-4 / 1.4e-3, output 3: 5.3e-5 / 1.9e-3; case 9 output 4: 4.1e-4 / 4.7e-3.  These outputs are held to
# twice the tensor-core error, every other output of the case to 1e-3.
ILL_CONDITIONED = {(7, 3): 1.3e-2, (7, 4): 3e-2, (8, 2): 3e-3, (8, 3): 4e-3, (9, 4): 1e-2}


CASES = pytest.mark.parametrize('i', range(len(SWEEP)), ids=['%d-%s' % (i, c.spec['builder']) for i, c in enumerate(SWEEP)])


# what the cases below checked: (kind, conv path or None) -> worst error / bound, and the cases that ran
CHECKED = {}
RAN = set()


def _frames(x):
    return int(np.prod(x.shape[:-3]))


def _context_cond(c, m, x):
    """per block, (N, joints) condition number of the context division (None without context maps)"""
    if c.spec['builder'] != 'reception' or not c.kw.get('num_context_per_joint'):
        return None
    dbg = {}
    kw = {k: v for k, v in c.kw.items() if k != 'export_vfeat_block'}        # only adds an output
    oracle_reception.forward(ops_np, m.get_weights(), x.astype(np.float64), c.spec['num_joints'], debug=dbg, **kw)
    return [np.asarray(k, np.float64) for k in dbg['ctx_cond']]


@CASES
def test_matches_reference_builders(cuda, i):
    c = SWEEP[i]
    m = c.build()
    x = np.asarray(c.x, np.float32)
    outs = m.predict(x)
    outs = list(outs) if isinstance(outs, (list, tuple)) else [outs]
    assert len(outs) == len(c.refs), (c.tag, len(outs), len(c.refs))
    cond = _context_cond(c, m, x)
    # ReceptionNet: per block the pose (pose and visibility without concat_pose_confidence) and the exported heat-maps,
    # then the exported features
    rec = c.spec['builder'] == 'reception'
    per_block = (1 + (not c.kw.get('concat_pose_confidence', True)) + bool(c.kw.get('export_heatmaps'))) if rec else 0
    heads = per_block * c.kw.get('num_blocks', 0)
    skipped = total = ties = maps = 0
    for k, (o, (shape, idx, r)) in enumerate(zip(outs, c.refs)):
        assert o.shape == shape, (c.tag, k, o.shape, shape)
        got = o.reshape(-1)[idx].astype(np.float64)
        err = np.abs(got - r) / np.maximum(np.abs(r), 1.0)
        lim = ILL_CONDITIONED.get((i, k), 1e-3)
        if k < heads and c.kw.get('export_heatmaps') and k % per_block == per_block - 1:
            # exported heat-maps: the arg-max pixel of every joint map is the reference's, unless the reference's two best
            # pixels tie within the value tolerance
            assert idx.size == np.prod(shape), 'the heat-map sample must hold the whole output'
            n_, h_, w_, c_ = shape
            fo, fr = got.reshape(n_, h_ * w_, c_), r.reshape(n_, h_ * w_, c_)
            top2 = np.sort(fr, axis=1)[:, -2:, :]
            tie = (top2[:, 1] - top2[:, 0]) <= 2e-3 * np.maximum(1.0, np.abs(top2[:, 1]))
            same = fo.argmax(axis=1) == fr.argmax(axis=1)
            assert np.all(same | tie), '%s output %d: arg-max pixel differs on %d maps' % (c.tag, k, int((~(same | tie)).sum()))
            ties += int(tie.sum())
            maps += tie.size
            err = np.abs(got - r) / max(1.0, float(np.abs(r).max()))
        if cond is not None and k < heads and k % per_block == 0:
            kc = cond[k // per_block]
            bad = kc > 100.0
            skipped += int(bad.sum())
            total += bad.size
            nj = np.unravel_index(idx, shape)[:2]             # (item, joint) of every sampled pose element
            err = np.where(bad[nj], 0.0, err)
            lim = np.maximum(1e-3, 0.2 * 1e-3 * kc[nj])
        assert np.all(err <= lim), '%s output %d: max err %g' % (c.tag, k, float(err.max()))
    if total:
        assert skipped <= max(1, total // 50), (skipped, total)
    if maps:
        assert ties <= max(1, maps // 20), '%d of %d heat-maps have an unresolvable top-2 tie' % (ties, maps)
    RAN.add('parity%d' % i)


@CASES
def test_launch_contracts_stored_input(cuda, i):
    c = SWEEP[i]
    _check(cuda, 'stored%d' % i, c.build(), cuda.from_numpy(np.asarray(c.x, np.float32)).cuda(), against_plain=False,
           checked=CHECKED, ran=RAN)


@CASES
def test_launch_contracts_several_tiles_per_cta(cuda, i):
    """2 * SMs + 5 frames (SPNet: that many frames rounded up to whole clips): each persistent kernel's CTAs run several
    tiles or frames, the last ones a ragged tail; the outputs also equal a plain forward and a CUDA-graph replay"""
    m = SWEEP[i].build()
    frames = 2 * cuda.cuda.get_device_properties(0).multi_processor_count + 5
    items = -(-frames // m.graph.frames_per_clip)
    _check(cuda, 'large%d' % i, m, _input(cuda, m, items, seed=5), against_plain=True, checked=CHECKED, ran=RAN)


@CASES
def test_cuda_core_fallbacks(cuda, i):
    """the convolutions bound to the generic CUDA-core kernel are the ones pinned above, and the ones the library counts"""
    c = SWEEP[i]
    m = c.build()
    x = np.asarray(c.x, np.float32)
    m.use_cuda_graph = False
    m.predict(x)
    lib = _ffi.lib()
    lib.dh_fallback_count(m._ctx.handle, 1)
    m.predict(x)
    counted = int(lib.dh_fallback_count(m._ctx.handle, 1))
    flagged = [k for k, info in m._bind(_frames(x)).conv_plans if info.fallback]
    names = [_weight_key(k).rsplit('/', 1)[0] for k in flagged]
    assert names == FALLBACKS[i], '%s: the CUDA-core kernel takes\n%s\nnot\n%s' % (c.tag, '\n'.join(
        '%s %s %r -> %r' % (k.kind, n, k.ins[0].shape, k.outs[0].shape) for k, n in zip(flagged, names)), FALLBACKS[i])
    assert counted == len(flagged), (counted, names)
    RAN.add('fallbacks%d' % i)


def test_coverage(cuda):
    """every case above ran, and every launch kind of the sweep's plans had its values checked"""
    want = set('%s%d' % (t, i) for t in ('parity', 'stored', 'large', 'fallbacks') for i in range(len(SWEEP)))
    if not want <= RAN:
        pytest.skip('needs every case of this module (%d of %d ran)' % (len(RAN & want), len(want)))
    kinds = set(k.kind for c in SWEEP for k in c.build().plan.kops)
    missing = sorted(kinds - set(k for k, _ in CHECKED))
    assert not missing, 'launch kinds no case checked: %s' % missing
    assert max(CHECKED.values()) <= 1.0
    print(_report(CHECKED))
    print('peak device memory allocated: %.2f GB' % (cuda.cuda.max_memory_allocated() / 1e9))
