"""Host-side logic (no GPU): the product's layer graph must expose exactly the weight list
(names, Keras layouts, creation order) that the oracle's independent restatement consumes;
synthetic weight generators agree; fusion plan sanity; FLOP counts of SURVEY.md 8(d)."""
import os

import numpy as np
import pytest

from deephar_b200 import reception
from deephar_b200.weights import load_calibration, split_bf16, synthetic_weight
from oracle import ops_torch
from oracle import reception as oracle_reception
from oracle import synth


def _oracle_used(res, **kw):
    tab = synth.SyntheticTable(1234)
    x = synth.synth_frames(1, res, res)
    _, used = oracle_reception.forward(ops_torch, tab, x, return_weights_used=True, **kw)
    return used


def test_weight_specs_match_oracle_2d():
    kw = dict(num_joints=16, dim=2, num_context_per_joint=2, num_blocks=3, ksize=(5, 5))
    m = reception.build((64, 64, 3), **kw)
    assert m.weight_specs == _oracle_used(64, **kw)


def test_weight_specs_match_oracle_3d():
    kw = dict(num_joints=17, dim=3, num_blocks=2, ksize=(3, 3))
    m = reception.build((64, 64, 3), **kw)
    assert m.weight_specs == _oracle_used(64, **kw)


def test_synthetic_generators_agree():
    calib = load_calibration('reception_j16_d2_c2_k5')
    assert len(calib) > 50
    m = reception.build((64, 64, 3), 16, 2, num_blocks=1, ksize=(5, 5))
    for name, shape in m.weight_specs[:40] + m.weight_specs[-10:]:
        a = synthetic_weight(1234, name, shape, calib)
        b = synth.synth_weight(1234, name, shape, calib)
        assert np.array_equal(a, b), name


def test_param_count_and_plan():
    m = reception.build((256, 256, 3), 16, 2, num_context_per_joint=2, num_blocks=8, ksize=(5, 5),
                        concat_pose_confidence=False)
    assert m.count_params() == 14746560          # SURVEY.md 6: 14.75 M
    assert len(m.outputs) == 16
    assert m.input_shape == (None, 256, 256, 3)
    st = m.plan.stats
    assert st['kernel_ops'] < st['graph_nodes'] / 2.5     # BN/ReLU/add/concat fused away
    kinds = [k.kind for k in m.plan.kops]
    assert 'affine' not in kinds and 'add' not in kinds and 'copy' not in kinds
    assert kinds.count('pose_regression_2d_context') == 8
    flops = m.conv_flops_per_frame()
    assert abs(flops - 19.67e9) / 19.67e9 < 0.005            # SURVEY.md 8(d)
    # hourglass glue fused into the neighbouring conv kernels (reception.py:108-110, 122-127):
    # 2 x 8 `add([a, UpSampling2D(b)])` as the last (half-resolution) residual of the sepconv producing a,
    # 7 MaxPooling2D of the block-end add as the second output of the fReMap kernel that computes it
    up = [k for k in m.plan.kops if k.attrs.get('res_up2x')]
    assert len(up) == 16 and all(k.kind == 'sepconv' and k.ins[-1].shape[0] * 2 == k.outs[0].shape[0] for k in up)
    assert sorted(set(k.outs[0].shape[1] for k in up)) == [16, 32]
    pooled = [k for k in m.plan.kops if k.attrs.get('pool_out')]
    assert len(pooled) == 7 and all(k.kind == 'conv' and k.attrs['size'] == (1, 1) and len(k.outs) == 2 and
                                    k.outs[1].shape == (16, 16, 576) for k in pooled)
    assert 'upsample_add' not in kinds and kinds.count('maxpool') == 11 and len(kinds) == 127


def test_fusions_are_refused_where_the_kernels_cannot_take_them():
    from deephar_b200 import layers as L
    from deephar_b200.graph import Graph
    from deephar_b200.model import Model
    # pooled second output needs the wide pointwise kernel (Cin <= 64): a 272-channel fReMap (3-D model) keeps its max-pool
    m3 = reception.build((256, 256, 3), 17, 3, num_blocks=2, ksize=(5, 5))
    k3 = [k.kind for k in m3.plan.kops]
    assert not any(k.attrs.get('pool_out') for k in m3.plan.kops) and k3.count('maxpool') >= 4
    # upsampled residual: 8-pixel-wide maps and stride-2 / dense producers stay separate `upsample_add` kernels
    g = Graph('t')
    x = g.input((8, 8, 32))
    a = L.BatchNormalization(L.sepconv2d(L.relu(x), 32, (3, 3), name='s'), name='b')
    low = L.conv2d(L.maxpooling2d(x), 32, (1, 1), name='c')
    g.outputs = [L.add([a, L.UpSampling2D(low)])]
    kk = [k.kind for k in Model(g).plan.kops]
    assert 'upsample_add' in kk


def test_flops_3d():
    m = reception.build((256, 256, 3), 17, 3, num_blocks=8, ksize=(5, 5), concat_pose_confidence=False)
    assert abs(m.conv_flops_per_frame() - 23.63e9) / 23.63e9 < 0.005
    assert m.count_params() == 16683712 or abs(m.count_params() - 16.68e6) < 0.01e6


def test_output_order_and_shapes():
    m = reception.build((64, 64, 3), 16, 2, num_blocks=2, ksize=(3, 3))
    assert m.output_shape == [(None, 16, 3), (None, 16, 3)]
    m = reception.build((64, 64, 3), 17, 3, num_blocks=2, concat_pose_confidence=False)
    assert m.output_shape == [(None, 17, 3), (None, 17, 1)] * 2


def test_argument_errors_match_reference():
    import pytest
    with pytest.raises(ValueError):
        reception.build((64, 64, 3), 16, 4)
    with pytest.raises(AssertionError):
        reception.build((64, 64, 3), 17, 3, num_context_per_joint=2)


def test_split_bf16_reconstructs():
    rng = np.random.default_rng(0)
    w = rng.standard_normal(4096).astype(np.float32)
    hi, lo = split_bf16(w)
    rec = (hi.astype(np.uint32) << 16).view(np.float32) + (lo.astype(np.uint32) << 16).view(np.float32)
    assert np.abs(rec - w).max() <= np.abs(w).max() * 2.0 ** -16


def _baseline_models():
    from deephar_b200 import action, reception, spnet
    from deephar_b200.config import ModelConfig, pa16j2d, pa17j3d
    yield 'c1', reception.build((256, 256, 3), 16, dim=2, num_blocks=8, num_context_per_joint=2, ksize=(5, 5),
                                concat_pose_confidence=False)
    yield 'c1_heatmaps', reception.build((256, 256, 3), 16, dim=2, num_blocks=8, num_context_per_joint=2, ksize=(5, 5),
                                         export_heatmaps=True)
    yield 'c3', reception.build((256, 256, 3), 17, dim=3, num_blocks=8, ksize=(5, 5), concat_pose_confidence=False)
    yield 'c4', spnet.build(ModelConfig((16, 256, 256, 3), pa16j2d, num_actions=[15], num_pyramids=6,
                                        action_pyramids=[5, 6], num_levels=4, pose_replica=True,
                                        num_pose_features=160, num_visual_features=160))
    yield 'c5', spnet.build(ModelConfig((16, 256, 256, 3), pa17j3d, num_actions=[60], num_pyramids=2,
                                        action_pyramids=[1, 2], num_levels=4, pose_replica=False,
                                        num_pose_features=192, num_visual_features=192))
    pe = reception.build((256, 256, 3), 16, dim=2, num_blocks=4, num_context_per_joint=2, ksize=(5, 5))
    yield 'merge2d', action.build_merge_model(pe, 15, (256, 256, 3), 16, 16, 4, pose_dim=2)
    pe = reception.build((256, 256, 3), 20, dim=3, num_blocks=4, depth_maps=8, ksize=(5, 5))
    yield 'merge3d', action.build_merge_model(pe, 60, (256, 256, 3), 16, 20, 4, pose_dim=3, depth_maps=8,
                                              output_poses=True)


def test_buffer_plans_of_every_baseline_model_are_memory_safe():
    """compiler.verify_plan replays the launches over the physical slots: every read sees what its producer wrote, no
    launch writes over an operand, outputs survive.  (The planner reuses a slot as soon as its buffer is dead; the
    headline model runs in 35 slots instead of 140 buffers.)"""
    from deephar_b200.compiler import verify_plan
    seen = {}
    for name, m in _baseline_models():
        n = verify_plan(m.plan, m.graph)
        assert n > 2 * len(m.plan.kops)
        seen[name] = (len(m.plan.kops), m.plan.stats['phys_slots'], m.plan.stats['buffers'])
    assert seen['c1'][0] == 127 and seen['c3'][0] == 134 and seen['c4'][0] == 345 and seen['c5'][0] == 237
    assert all(slots < bufs for _, slots, bufs in seen.values())


def test_verify_plan_catches_a_clobbered_buffer():
    from deephar_b200 import reception
    from deephar_b200.compiler import verify_plan
    m = reception.build((64, 64, 3), 16, dim=2, num_blocks=2, num_context_per_joint=2, ksize=(5, 5))
    plan = m.plan
    verify_plan(plan, m.graph)
    # put a long-lived buffer (a block's identity branch) on the slot of a buffer that is written while it is live
    bufs = sorted((b for b in plan.buffers if not b.is_input and not b.is_output), key=lambda b: b.first - b.last)
    victim = bufs[0]
    other = next(b for b in plan.buffers if victim.first < b.first < victim.last and b.phys != victim.phys
                 and not b.is_input and not b.is_output)
    keep = other.phys
    other.phys = victim.phys
    try:
        with pytest.raises(AssertionError, match='launch'):
            verify_plan(plan, m.graph)
    finally:
        other.phys = keep
    # a launch that no longer has its operand written
    k = next(k for k in plan.kops if k.kind in ('conv', 'sepconv') and len(k.ins) > 1)
    dropped = plan.kops.index(next(p for p in plan.kops if k.ins[1] in p.outs))
    removed = plan.kops.pop(dropped)
    try:
        with pytest.raises(AssertionError):
            verify_plan(plan, m.graph)
    finally:
        plan.kops.insert(dropped, removed)
    verify_plan(plan, m.graph)


def test_roofline_accounting_matches_the_flop_counter_and_the_committed_profile():
    """tools/roofline_by_layer.py: the per-launch algorithmic flops add up to Model.conv_flops_per_frame, the labels are
    the ones of the committed per-op profile, and every launch moves at least its output once."""
    import importlib.util
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    spec = importlib.util.spec_from_file_location('roofline_by_layer', os.path.join(root, 'tools', 'roofline_by_layer.py'))
    rl = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(rl)
    m = reception.build((256, 256, 3), 16, dim=2, num_blocks=8, num_context_per_joint=2, ksize=(5, 5),
                        concat_pose_confidence=False)
    work = [rl.work_of(k, 256, 1) for k in m.plan.kops]
    assert abs(sum(f for _, f in work) / 256 - m.conv_flops_per_frame()) / m.conv_flops_per_frame() < 1e-9
    assert all(b >= 4.0 * 256 * np.prod(k.outs[0].shape) for (b, _), k in zip(work, m.plan.kops))
    prof = open(os.path.join(root, 'profiles', 'h100_prof_reception2d.txt')).read()
    assert all(rl.label_of(k) in prof for k in m.plan.kops)


def test_summary_and_training_entry_points():
    """keras.Model.summary (exp/ntu/predict_bboxes.py:45) describes the compiled model; compile / fit are refused."""
    m = reception.build((64, 64, 3), 16, dim=2, num_blocks=2, num_context_per_joint=2, ksize=(5, 5))
    lines = []
    m.summary(print_fn=lines.append)
    text = '\n'.join(lines)
    assert 'Stem' in text and 'rBlock2' in text and 'Total params: %d' % m.count_params() in text
    assert '%d kernel launches' % len(m.plan.kops) in text
    for call in (m.compile, m.fit, m.fit_generator):
        with pytest.raises(NotImplementedError):
            call()
