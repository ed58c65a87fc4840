"""Every launch of the compiled networks on the GPU against its contract (tests/launch_check.py): what it writes -- all
of its outputs and nothing else, guard bands and weights included -- and what it computes, on the inputs the device
actually holds, against the fp64 reference within each launch's bound.  At the batch sizes the product runs (256 frames
of C2 / C3, 16 clips x 16 frames of C4 / C5, as bench.py), at small batches, on both merge models and on random graphs
of the compiler fuzzer; at production size the launch-by-launch outputs must equal a plain forward's bit for bit.

    pytest -m gpu tests/test_gpu_launch_contracts.py -k C4
"""
import numpy as np
import pytest

from deephar_b200 import action, reception, spnet
from deephar_b200.config import ModelConfig, pa16j2d, pa17j3d
from deephar_b200.model import Model
from oracle import synth

from launch_check import LaunchChecker
from test_compiler_fuzz import _random_graph

pytestmark = pytest.mark.gpu

C2_KW = dict(num_joints=16, dim=2, num_context_per_joint=2, num_blocks=8, ksize=(5, 5), concat_pose_confidence=False)
C3_KW = dict(num_joints=17, dim=3, num_blocks=8, ksize=(5, 5), concat_pose_confidence=False)
FUZZ_SEEDS = range(40)

# what the cases below checked: (kind, conv path or None) -> worst error / bound, and the cases that ran
CHECKED = {}
RAN = set()


def _record(name, ch, checked=CHECKED, ran=RAN):
    ran.add(name)
    for key, r in ch.worst.items():
        checked[key] = max(checked.get(key, 0.0), r)
    for key in ch.checked:
        checked.setdefault(key, 0.0)


def _report(checked):
    lines = ['%-28s %-6s %.3f' % (k, '' if p is None else 'path %d' % p, r)
             for (k, p), r in sorted(checked.items(), key=lambda kv: (kv[0][0], -1 if kv[0][1] is None else kv[0][1]))]
    return 'worst error / bound per launch kind:\n' + '\n'.join(lines)


def _build(which, frames=16):
    if which == 'C2':
        return reception.build((256, 256, 3), **C2_KW)
    if which == 'C3':
        return reception.build((256, 256, 3), **C3_KW)
    if which == 'C4':
        return spnet.build(ModelConfig((frames, 256, 256, 3), pa16j2d, num_actions=[15], num_pyramids=6,
                                       action_pyramids=[5, 6], num_levels=4, pose_replica=True, num_pose_features=160,
                                       num_visual_features=160))
    if which == 'C5':
        return spnet.build(ModelConfig((frames, 256, 256, 3), pa17j3d, num_actions=[60], num_pyramids=2,
                                       action_pyramids=[1, 2], num_levels=4, num_pose_features=192, num_visual_features=192))
    import sys
    import os
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden'))
    from ref_cases import MERGE3D_CASE, MERGE_CASE
    mc = MERGE_CASE if which == 'merge2d' else MERGE3D_CASE
    pe = reception.build(mc['input_shape'], **mc['reception'])
    if which == 'merge2d':
        return action.build_merge_model(pe, mc['num_actions'], mc['input_shape'], mc['num_frames'], mc['num_joints'],
                                        mc['num_blocks'], pose_dim=2)
    return action.build_merge_model(pe, mc['num_actions'], mc['input_shape'], mc['num_frames'], mc['num_joints'],
                                    mc['num_blocks'], pose_dim=3, depth_maps=mc['depth_maps'], output_poses=True)


def _input(torch, m, items, seed):
    """device input: `items` frames, or `items` clips of a clip model; smooth synthetic frames"""
    T = m.graph.frames_per_clip
    h, w, _ = m.graph.inputs[0].shape
    n = items * T
    x = torch.from_numpy(np.ascontiguousarray(synth.synth_frames(n, h, w, seed=seed), np.float32)).cuda()
    return x.reshape((items, T, h, w, 3) if T > 1 else (n, h, w, 3))


def _check(torch, name, m, x, against_plain, checked=CHECKED, ran=RAN):
    """`checked` / `ran`: the tables of the module whose coverage test reports this case"""
    m.init_synthetic_weights(1234)
    ch = LaunchChecker(m)
    outs = ch.run(x)
    assert ch.launches == len(m.plan.kops)
    _record(name, ch, checked, ran)
    if not m.use_tensor_cores:
        _record_cuda_cores(name, ch)
    if against_plain:
        m.use_cuda_graph = True
        for run in ('plain launches', 'CUDA-graph replay'):
            got = [o.cpu().numpy() for o in m.forward_device(x)]
            for i, (a, b) in enumerate(zip(outs, got)):
                assert np.array_equal(a.reshape(b.shape), b, equal_nan=False), \
                    '%s: output %d of the %s differs from the launch-by-launch run' % (name, i, run)
        assert m._graph_replays >= 1
    m._bound = {}
    torch.cuda.empty_cache()


@pytest.mark.parametrize('which,items', [('C2', 256), ('C3', 256), ('C4', 16), ('C5', 16)])
def test_production_batch(cuda, which, items):
    """256 frames of C2 / C3, 16 clips x 16 frames of C4 / C5 (bench.py's forward calls); the outputs equal a plain
    forward_device run, first launch and graph replay, bit for bit"""
    m = _build(which)
    _check(cuda, '%s-%d' % (which, items), m, _input(cuda, m, items, seed=3), against_plain=True)


@pytest.mark.parametrize('which,items', [('C2', 3), ('C4', 1), ('C5', 1), ('merge2d', 1), ('merge3d', 1)])
def test_small_batch(cuda, which, items):
    m = _build(which)
    _check(cuda, '%s-%d' % (which, items), m, _input(cuda, m, items, seed=4), against_plain=False)


@pytest.mark.parametrize('frames', [3, 261])
@pytest.mark.parametrize('seed', FUZZ_SEEDS)
def test_fuzz_graph(cuda, seed, frames):
    """random graphs of tests/test_compiler_fuzz.py; a plan the library refuses to bind fails here"""
    g, side = _random_graph(seed)
    m = Model(g, name=g.name)
    x = np.random.default_rng(1000 + seed).uniform(-1, 1, (frames, side, side, 3)).astype(np.float32)
    _check(cuda, 'fuzz%d-%d' % (seed, frames), m, cuda.from_numpy(x).cuda(), against_plain=False)


# ---- the same networks with use_tensor_cores = False: every convolution on the CUDA-core kernels (paths 0 and 3) ----
CC_CHECKED = {}
CC_RAN = set()
CC_SEEN = set()         # what the CUDA-core convolutions of these cases ran (_record_cuda_cores)


def _record_cuda_cores(name, ch):
    CC_RAN.add(name)
    for k, path, fallback in ch.conv_choices:
        assert path in (0, 3), '%s: %s layer %s went to path %d without tensor cores' % (name, k.kind, k.attrs.get(
            'kernel', k.attrs.get('pointwise')), path)
        if path == 0 and k.attrs.get('res_up2x'):
            CC_SEEN.add('implicit GEMM with an upsampled residual')
        if path == 0 and k.kind == 'sepconv':
            CC_SEEN.add('two-kernel separable with its workspace')
        if path == 0 and k.kind == 'conv' and not fallback:
            CC_SEEN.add('direct stem')
        if path == 3 and k.attrs.get('pool_out'):
            CC_SEEN.add('pool_out on path 3')


def _cuda_cores(m):
    m.use_tensor_cores = False
    return m


@pytest.mark.parametrize('which,items', [('C2', 3), ('C4', 1), ('C5', 1), ('merge2d', 1), ('merge3d', 1)])
def test_small_batch_cuda_cores(cuda, which, items):
    m = _cuda_cores(_build(which))
    _check(cuda, 'cc-%s-%d' % (which, items), m, _input(cuda, m, items, seed=4), against_plain=False,
           checked=CC_CHECKED, ran=CC_RAN)


@pytest.mark.parametrize('seed', FUZZ_SEEDS)
def test_fuzz_graph_cuda_cores(cuda, seed):
    g, side = _random_graph(seed)
    m = _cuda_cores(Model(g, name=g.name))
    x = np.random.default_rng(1000 + seed).uniform(-1, 1, (3, side, side, 3)).astype(np.float32)
    _check(cuda, 'cc-fuzz%d-3' % seed, m, cuda.from_numpy(x).cuda(), against_plain=False, checked=CC_CHECKED, ran=CC_RAN)


def test_c2_cuda_cores_grid_stride(cuda):
    """C2 at 2 x SMs + 5 frames on the CUDA-core kernels: the persistent grids run several tiles per CTA and the
    grid-stride loops several passes; the launch-by-launch outputs equal a plain forward and a graph replay bit for bit"""
    sms = cuda.cuda.get_device_properties(cuda.cuda.current_device()).multi_processor_count
    items = 2 * sms + 5
    m = _cuda_cores(_build('C2'))
    _check(cuda, 'cc-C2-%d' % items, m, _input(cuda, m, items, seed=5), against_plain=True, checked=CC_CHECKED,
           ran=CC_RAN)


def test_coverage_cuda_cores(cuda):
    """every CUDA-core convolution kind the networks use had its values checked by the cases above"""
    want = set('cc-%s-%d' % c for c in (('C2', 3), ('C4', 1), ('C5', 1), ('merge2d', 1), ('merge3d', 1)))
    want |= set('cc-fuzz%d-3' % s for s in FUZZ_SEEDS)
    if not want <= CC_RAN or not any(r.startswith('cc-C2-') and r != 'cc-C2-3' for r in CC_RAN):
        pytest.skip('needs every case of this module (%d of %d ran)' % (len(CC_RAN & want), len(want) + 1))
    assert CC_SEEN == {'implicit GEMM with an upsampled residual', 'two-kernel separable with its workspace',
                       'direct stem', 'pool_out on path 3'}, CC_SEEN
    assert set(p for k, p in CC_CHECKED if k in ('conv', 'sepconv')) == {0, 3}
    assert ('pool_out', 3) in CC_CHECKED
    print(_report(CC_CHECKED))
    print('peak device memory allocated: %.2f GB' % (cuda.cuda.max_memory_allocated() / 1e9))


# kinds Model._bind_plan issues, and why a kind no case above reaches is left out
BIND_KINDS = ('conv', 'sepconv', 'maxpool', 'upsample_add', 'upsample', 'add', 'affine', 'copy',
              'pose_regression_2d_context', 'pose_regression_2d', 'pose_regression_3d', 'pose_regression_3d_ex', 'scale',
              'sam2d', 'kron', 'mask_mul', 'zeropad', 'maxminpool', 'global_maxmin_softmax')
NOT_REACHED = {
    'pose_regression_2d': 'only models recorded from Keras code (keras_trace.py) emit it; tests/test_gpu_head_paths.py '
                          'checks dh_softargmax2d_f32 on raw-map confidences',
}


def test_coverage(cuda):
    """every kind of launch and every convolution path 0-4 had its values checked by at least one case above"""
    want = set(['%s-%d' % c for c in (('C2', 256), ('C3', 256), ('C4', 16), ('C5', 16), ('C2', 3), ('C4', 1), ('C5', 1),
                                       ('merge2d', 1), ('merge3d', 1))])
    want |= set('fuzz%d-%d' % (s, f) for s in FUZZ_SEEDS for f in (3, 261))
    if not want <= RAN:
        pytest.skip('needs every case of this module (%d of %d ran)' % (len(RAN & want), len(want)))
    kinds = set(k for k, _ in CHECKED)
    missing = [k for k in BIND_KINDS if k not in kinds and k not in NOT_REACHED]
    assert not missing, 'launch kinds no case checked: %s' % missing
    assert not [k for k in NOT_REACHED if k in kinds], 'a kind listed as not reached was reached: update NOT_REACHED'
    paths = set(p for k, p in CHECKED if k in ('conv', 'sepconv'))
    assert paths >= {0, 1, 2, 3, 4}, 'convolution paths checked: %s' % sorted(paths)
    assert ('pool_out', 3) in CHECKED
    print(_report(CHECKED))
    print('peak device memory allocated: %.2f GB' % (cuda.cuda.max_memory_allocated() / 1e9))
