"""SURVEY.md 8 f3: evaluator post-processing.  CPU: the oracle vs the outputs of the reference's own numpy code
(tests/golden/ref_postprocess.npz, written by make_postprocess_golden.py).  GPU: dh_pose_eval_f64 vs both."""
import os

import numpy as np
import pytest

from oracle import postprocess as oracle_pp

Z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'ref_postprocess.npz'))


def test_oracle_matches_reference_postprocessing():
    y = oracle_pp.transform_pose_sequence(Z['A'], Z['y_pred_crop'], inverse=True)
    assert np.abs(y - Z['y_pred']).max() <= 1e-9 * np.abs(Z['y_pred']).max()
    f = oracle_pp.transform_pose_sequence(Z['A'][0], Z['y_pred_crop'], inverse=False)
    assert np.abs(f - Z['fwd']).max() <= 1e-12
    assert oracle_pp.pckh(Z['y_true'], Z['y_pred'], Z['head'], 0.5) == pytest.approx(float(Z['pckh05']), abs=1e-12)
    assert oracle_pp.pckh(Z['y_true'], Z['y_pred'], Z['head'], 0.2) == pytest.approx(float(Z['pckh02']), abs=1e-12)
    assert oracle_pp.mean_distance_error(Z['y_true'], Z['y_pred']) == pytest.approx(float(Z['mde']), rel=1e-12)


def test_oracle_per_joint_pckh_matches_the_table_the_reference_prints():
    """tests/golden/ref_pckh_per_joint.npz: the ' %.2f | ' cells of deephar/measures.py::pckh_per_joint's printout"""
    G = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'ref_pckh_per_joint.npz'))
    for refp in (0.5, 0.2):
        got = 100.0 * oracle_pp.pckh_per_joint(Z['y_true'], Z['y_pred'], Z['head'], refp)
        assert got.shape == (16,) and np.abs(got - G['percent_%s' % refp]).max() <= 0.005 + 1e-9


@pytest.mark.gpu
def test_gpu_per_joint_pckh(cuda):
    from deephar_b200 import postprocess as pp
    G = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'ref_pckh_per_joint.npz'))
    for refp in (0.5, 0.2):
        got = 100.0 * pp.pckh_per_joint(Z['y_true'], Z['y_pred_crop'], Z['head'], refp, A=Z['A'])
        # the same counts as the reference: only the printout's 2-decimal rounding separates the two
        assert got.shape == (16,) and np.abs(got - G['percent_%s' % refp]).max() <= 0.005 + 1e-9
        assert np.array_equal(got, 100.0 * oracle_pp.pckh_per_joint(Z['y_true'], Z['y_pred'], Z['head'], refp))


@pytest.mark.gpu
def test_gpu_postprocessing_matches_reference(cuda):
    from deephar_b200 import postprocess as pp
    y = pp.transform_pose_sequence(Z['A'], Z['y_pred_crop'], inverse=True)
    assert y.dtype == np.float64                                    # float64 in, float64 out, as the reference
    assert np.abs(y - Z['y_pred']).max() <= 1e-9 * np.abs(Z['y_pred']).max()      # the oracle's bound above
    f = pp.transform_pose_sequence(Z['A'][0], Z['y_pred_crop'], inverse=False)
    assert np.abs(f - Z['fwd']).max() <= 1e-12
    # the score from crop-space predictions in ONE kernel (inverse map + threshold), as the evaluator does in two steps
    assert pp.pckh(Z['y_true'], Z['y_pred_crop'], Z['head'], 0.5, A=Z['A']) == float(Z['pckh05'])
    assert pp.pckh(Z['y_true'], Z['y_pred'], Z['head'], 0.2) == float(Z['pckh02'])
    assert pp.mean_distance_error(Z['y_true'], Z['y_pred']) == pytest.approx(float(Z['mde']), rel=1e-12)


@pytest.mark.gpu
def test_eval_singleperson_pckh_end_to_end(cuda):
    """exp/common/mpii_tools.py:63-129 on a tiny model: the device path must give the score the host path gives."""
    from deephar_b200 import postprocess as pp
    from deephar_b200 import reception
    from oracle import synth
    m = reception.build((64, 64, 3), num_joints=16, dim=2, num_context_per_joint=2, num_blocks=2, ksize=(3, 3),
                        concat_pose_confidence=False).init_synthetic_weights(5)
    n = 6
    x = synth.synth_frames(n, 64, 64, seed=9)
    rng = np.random.default_rng(1)
    A = np.tile(np.array([[1 / 200.0, 0, 0.1], [0, 1 / 200.0, 0.2], [0, 0, 1]]), (n, 1, 1))
    pval = rng.uniform(0.2, 0.8, (n, 16, 2))
    head = rng.uniform(30, 50, (n, 1))
    scores = pp.eval_singleperson_pckh(m, x, pval, A, head, batch_size=4, refp=0.5, pred_per_block=2)
    outs = m.predict(x, batch_size=4)
    y_true = oracle_pp.transform_pose_sequence(A, pval, inverse=True)
    for b in range(2):
        y_pred = oracle_pp.transform_pose_sequence(A, outs[2 * b], inverse=True)
        assert scores[b] == oracle_pp.pckh(y_true, y_pred, head, 0.5)


def test_multiclip_action_scores_match_the_reference_evaluator():
    """tests/golden/ref_action_eval.npz: scores printed by the reference's own eval_multiclip_dataset
    (exp/common/penn_tools.py:85-150) on seeded probabilities (make_action_eval_golden.py)."""
    from deephar_b200 import postprocess as pp
    G = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'ref_action_eval.npz'))
    want = G['scores']
    assert want.shape == (4,) and want[-1] > want[0]
    got_o = oracle_pp.multiclip_action_scores(G['probs'], G['video_of_item'], G['truth'])
    got_p = pp.multiclip_action_scores(G['probs'], G['video_of_item'], G['truth'])
    assert np.array_equal(got_o, want) and np.array_equal(got_p, want)
    # list-of-blocks input, one-hot labels, items in another order (a product does not care), bad shapes
    perm = np.random.default_rng(0).permutation(len(G['video_of_item']))
    onehot = np.eye(15)[G['truth']]
    got2 = pp.multiclip_action_scores([p[perm] for p in G['probs']], G['video_of_item'][perm], onehot)
    assert np.array_equal(got2, want)
    with pytest.raises(ValueError):
        pp.multiclip_action_scores(G['probs'][0], G['video_of_item'], G['truth'])
    with pytest.raises(ValueError):
        pp.multiclip_action_scores(G['probs'], G['video_of_item'][:-1], G['truth'])
    single = pp.singleclip_action_scores(list(G['probs']), G['truth'][G['video_of_item']])
    assert len(single) == 4 and all(0.0 <= v <= 1.0 for v in single) and single[-1] > single[0]


def test_human36m_mpjpe_matches_the_reference_evaluator():
    """tests/golden/ref_h36m_eval.npz: errors returned by the reference's own eval_human36m_sc_error
    (exp/common/h36m_tools.py:12-136, deephar/utils/camera.py) on seeded predictions and cameras with distortion."""
    from deephar_b200 import postprocess as pp
    G = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'ref_h36m_eval.npz'))
    want = G['scores']
    assert want.shape == (3,) and want[0] > want[2] > 1.0
    args = (list(G['preds']), G['afmat'], G['rootz'], G['scam'], G['pose_w'])
    got_o = oracle_pp.human36m_mpjpe(*args, resol_z=float(G['resol_z']))
    got_p = pp.human36m_mpjpe(*args, resol_z=float(G['resol_z']))
    assert np.allclose(got_o, want, rtol=1e-12, atol=1e-9)          # same dtype-preserving in-place steps as the reference
    # the product computes in float64 throughout; the reference rounds its float32 predictions after every step
    assert np.allclose(got_p, want, rtol=1e-6)
    assert np.allclose(got_p, oracle_pp.human36m_mpjpe([q.astype(np.float64) for q in args[0]], *args[1:],
                                                       resol_z=float(G['resol_z'])), rtol=1e-12)
    # cameras without distortion coefficients, a joint re-mapping, and a length mismatch
    ident = list(range(17))
    assert np.allclose(pp.human36m_mpjpe(*args, resol_z=float(G['resol_z']), map_to_pa17j=ident), got_p, rtol=1e-12)
    nod = pp.human36m_mpjpe(args[0], args[1], args[2], G['scam'][:, :18], args[4])
    assert all(abs(a - b) < 5.0 for a, b in zip(nod, want)) and not np.allclose(nod, want, rtol=1e-5)
    with pytest.raises(ValueError):
        pp.human36m_mpjpe([G['preds'][0][:-1]], args[1], args[2], args[3], args[4])


def test_bbox_from_poses_matches_the_reference_helper():
    """tests/golden/ref_bbox_from_poses.npz: boxes returned by the reference's own exp/common/generic.py::get_bbox_from_poses
    (make_bbox_golden.py) for frame batches, a clip and 3-D rows; two scales."""
    from deephar_b200 import postprocess as pp
    G = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'ref_bbox_from_poses.npz'))
    cases = sorted(set(n.split('/')[0] for n in G.files))
    assert len(cases) == 6
    for k in cases:
        got = pp.bbox_from_poses(G[k + '/poses'], G[k + '/afmat'], scale=float(G[k + '/scale']))
        assert np.abs(got - G[k + '/bbox']).max() <= 1e-9 * np.abs(G[k + '/bbox']).max(), k
    poses = G['frames_1.5/poses'].copy()
    poses[2, :, -2] = 0.0                                          # a frame with no joint above the threshold
    with pytest.raises(ValueError):
        pp.bbox_from_poses(poses, G['frames_1.5/afmat'])
    with pytest.raises(ValueError):
        pp.bbox_from_poses(poses[0], G['frames_1.5/afmat'])
