"""Evaluator-side post-processing on the GPU (SURVEY.md 8 f3) -- the step AFTER the forward path in the
reference's evaluators: poses back to image coordinates with the inverse crop affine, then PCKh / mean distance
(exp/common/mpii_tools.py:93-129, deephar/utils/transform.py:136-209, deephar/measures.py:5-93).  Same function
names and argument meaning as the reference; arrays may be numpy (copied to the device) or CUDA tensors, results
come back as numpy / python floats.  One kernel (dh_pose_eval_f64), in float64 like the reference's numpy code, so
the counts are the reference's exactly; no CPU path for the pose arithmetic.
The action evaluators' arithmetic after the forward (penn_tools.py:13-36, 85-150: a product of a few KB of
probabilities per video and an arg-max) is host code here as it is there: `multiclip_action_scores`.
"""
import ctypes as C

import numpy as np

from . import _ffi

# measures.py:63-65: pelvis and thorax are ignored, "according to the file 'annolist2matrix.m'"
PCKH_USED_JOINTS = [2, 3, 4, 5, 6, 7, 10, 11, 12, 13, 14, 15, 8, 9]

_ctx = {}


def _context(torch):
    dev = torch.cuda.current_device()
    if dev not in _ctx:
        _ctx[dev] = _ffi.Context(dev)
    return _ctx[dev]


def _dev(torch, a):
    """`a` as a contiguous float64 CUDA tensor, the reference's precision: numpy arrays (annotations, affine maps, head
    sizes) are converted on the host, CUDA tensors (the model's float32 outputs) on the device."""
    if not torch.is_tensor(a):
        a = torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64))
    return a.to(device='cuda', dtype=torch.float64).contiguous()


def _run(poses, A, inverse, y_true=None, head_size=None, refp=0.5):
    import torch
    if not torch.cuda.is_available():
        raise _ffi.DeepharB200Error('deephar_b200.postprocess needs a CUDA device; there is no CPU fallback')
    if not torch.is_tensor(poses):
        poses = np.asarray(poses)
    assert poses.ndim == 3 and poses.shape[2] >= 2, 'transform_pose_sequence: expected 3D tensor, got %s' % (tuple(poses.shape),)
    if torch.is_tensor(poses) and poses.is_cuda and poses.dtype == torch.float64 and poses.is_contiguous():
        p = poses                                   # (x, y[, z][, v]) rows read in place through pred_ld
    else:
        p = _dev(torch, poses[:, :, :2])            # only (x, y) is converted: N x nj x 2 values
    a = _dev(torch, A)
    per_sample = a.dim() == 3
    if per_sample:
        assert len(a) == len(p), 'A is %s and poses is %s' % (tuple(a.shape), tuple(p.shape))
    n, nj = int(p.shape[0]), int(p.shape[1])
    out = torch.empty(n, nj, 2, device='cuda', dtype=torch.float64)
    hits = torch.zeros(nj, device='cuda', dtype=torch.int32)
    valid = torch.zeros(nj, device='cuda', dtype=torch.int32)
    dsum = torch.zeros(nj, device='cuda', dtype=torch.float64)
    yt = _dev(torch, y_true)[:, :, :2].contiguous() if y_true is not None else None
    hs = _dev(torch, head_size).reshape(-1) if head_size is not None else None
    if yt is not None:
        assert yt.shape[:2] == p.shape[:2]
    if hs is not None:
        assert len(hs) == n
    ctx = _context(torch)
    rc = _ffi.lib().dh_pose_eval_f64(ctx.handle, p.data_ptr(), int(p.shape[2]), a.data_ptr(), 1 if per_sample else 0,
                                     1 if inverse else 0, yt.data_ptr() if yt is not None else None,
                                     hs.data_ptr() if hs is not None else None, C.c_double(refp), n, nj, out.data_ptr(),
                                     hits.data_ptr(), valid.data_ptr(), dsum.data_ptr(),
                                     torch.cuda.current_stream().cuda_stream)
    _ffi.check(rc, 'dh_pose_eval_f64')
    return out, hits, valid, dsum


def transform_pose_sequence(A, poses, inverse=True):
    """deephar/utils/transform.py:174-209: [num_samples, num_points, 2] poses through A (one [3,3] map or one per
    sample), inverted first if `inverse`.  float64, as the reference returns."""
    out, _, _, _ = _run(poses, A, inverse)
    return out.cpu().numpy()


def pckh(y_true, y_pred, head_size, refp=0.5, A=None):
    """deephar/measures.py:49-76.  With `A` the predictions are first mapped by inv(A) (what the evaluator does
    on the host before calling pckh, mpii_tools.py:118-119) -- one kernel for both."""
    import torch
    eye = np.eye(3)
    _, hits, valid, _ = _run(y_pred, A if A is not None else eye, A is not None, y_true, head_size, refp)
    used = torch.tensor(PCKH_USED_JOINTS, device='cuda')
    return float(hits[used].sum().item()) / float(valid[used].sum().item())


def pckh_per_joint(y_true, y_pred, head_size, refp=0.5, A=None):
    """deephar/measures.py:108-146 (the table the MPII evaluator prints for its last block, mpii_tools.py:124-127) as an
    array: per joint, the share of annotated samples whose prediction lies within refp x head size; NaN for a joint no
    sample annotates.  Same kernel launch as `pckh` (its per-joint counters), `A` as there."""
    eye = np.eye(3)
    _, hits, valid, _ = _run(y_pred, A if A is not None else eye, A is not None, y_true, head_size, refp)
    hits, valid = hits.cpu().numpy().astype(np.float64), valid.cpu().numpy().astype(np.float64)
    with np.errstate(invalid='ignore', divide='ignore'):
        return hits / valid


def mean_distance_error(y_true, y_pred):
    """deephar/measures.py:18-47 for 2-D poses."""
    _, _, valid, dsum = _run(y_pred, np.eye(3), False, y_true, None, 0.0)
    return float(dsum.sum().item()) / float(valid.sum().item())


def eval_singleperson_pckh(model, fval, pval, afmat_val, headsize_val, batch_size=8, refp=0.5, pred_per_block=1):
    """exp/common/mpii_tools.py:63-129 for single-frame models: predict, map every block's pose back with
    inv(afmat) and score it -- poses stay on the device between the soft-argmax head and the score."""
    import torch
    fval = np.ascontiguousarray(fval, dtype=np.float32)
    num_blocks = int(len(model.outputs) / pred_per_block)
    y_true = transform_pose_sequence(np.array(afmat_val, dtype=np.float64), np.asarray(pval)[:, :, :2], inverse=True)
    hits = [None] * num_blocks
    valid = [None] * num_blocks
    for i in range(0, len(fval), batch_size):
        outs = model.forward_device(torch.from_numpy(fval[i:i + batch_size]).cuda())
        for b in range(num_blocks):
            _, h, v, _ = _run(outs[pred_per_block * b][:, :, :2], afmat_val[i:i + batch_size], True,
                              y_true[i:i + batch_size], headsize_val[i:i + batch_size], refp)
            hits[b] = h if hits[b] is None else hits[b] + h
            valid[b] = v if valid[b] is None else valid[b] + v
    used = torch.tensor(PCKH_USED_JOINTS, device='cuda')
    return [float(hits[b][used].sum().item()) / float(valid[b][used].sum().item()) for b in range(num_blocks)]


def multiclip_action_scores(probs, video_of_item, truth, n_videos=None):
    """exp/common/penn_tools.py:85-150 / ntu_tools.py after the predictions: every video is scored by the product, over
    its clips x {no flip, h-flip}, of each prediction block's action probabilities; arg-max against the label; accuracy
    in percent per block.  probs: (num_blocks, N_items, n_act) or a list of per-block (N_items, n_act) arrays (what
    `model.predict` returns for a batch of all clips); video_of_item (N_items,); truth (n_videos,) class indices or
    (n_videos, n_act) one-hot.  A few KB of arithmetic: done on the host in float64 like the reference (the forward
    that produces `probs` is where the time goes -- run it batched, not clip by clip as the reference does)."""
    probs = np.stack([np.asarray(p) for p in probs]) if isinstance(probs, (list, tuple)) else np.asarray(probs)
    if probs.ndim != 3:
        raise ValueError('multiclip_action_scores: probs must be (num_blocks, N_items, n_act), got %s' % (probs.shape,))
    video_of_item = np.asarray(video_of_item, np.int64).reshape(-1)
    truth = np.asarray(truth)
    if truth.ndim == 2:
        truth = truth.argmax(axis=-1)
    nb, n_items, n_act = probs.shape
    if len(video_of_item) != n_items:
        raise ValueError('multiclip_action_scores: %d items but %d video indices' % (n_items, len(video_of_item)))
    n_videos = int(n_videos if n_videos is not None else len(truth))
    a_pred = np.ones((nb, n_videos, n_act), np.float64)
    for b in range(nb):
        np.multiply.at(a_pred[b], video_of_item, probs[b].astype(np.float64))     # unbuffered: items in order
    correct = a_pred.argmax(axis=-1) == truth[None, :]
    return 100.0 * correct.sum(axis=-1) / n_videos


def singleclip_action_scores(preds, action_true):
    """exp/common/penn_tools.py:13-36 after the predict: fraction of clips whose arg-max class is the label's, per block."""
    action_true = np.asarray(action_true)
    label = action_true.argmax(axis=-1) if action_true.ndim == 2 else action_true
    return [float(np.mean(np.asarray(p).argmax(axis=-1) == label)) for p in preds]


def human36m_mpjpe(preds, afmat, rootz, scam, pose_w, resol_z=2000., map_to_pa17j=None):
    """exp/common/h36m_tools.py:12-99 after the predict (the H36M evaluator's score): per prediction block, (x, y) of
    the normalised predictions back to image pixels with the inverse crop affine, z = resol_z * (z - 0.5) + rootz,
    camera inverse projection (deephar/utils/camera.py:52-71, distortion coefficients included) with each sample's
    serialised camera [R(9) t(3) f(2) c(2) p(2) k(3)], predicted and true poses root-centred, mean per-joint distance
    in mm.  preds: list of (N, nj, >= 3) arrays (what `model.predict` returns); -> list of errors, one per block.
    Vectorised over samples on the host in float64: N x 17 x 3 numbers (the reference loops per sample)."""
    afmat = np.asarray(afmat, np.float64)
    scam = np.asarray(scam, np.float64)
    rootz = np.asarray(rootz, np.float64).reshape(-1, 1)
    y_true = np.array(pose_w, np.float64)
    if map_to_pa17j is not None:
        y_true = y_true[:, map_to_pa17j, :]
    y_true = y_true - y_true[:, 0:1, :]
    n = len(y_true)
    R = scam[:, 0:9].reshape(n, 3, 3)
    t, f, c, p = scam[:, None, 9:12], scam[:, None, 12:14], scam[:, None, 14:16], scam[:, None, 16:18]
    k = scam[:, 18:21] if scam.shape[1] > 18 else None
    Rinv = np.linalg.inv(R)
    Ainv = np.linalg.inv(afmat)
    valid = np.all(y_true > -1e6, axis=-1)
    out = []
    for pred in preds:
        y = np.array(pred, np.float64)[:, :, 0:3]
        if y.shape[0] != n:
            raise ValueError('human36m_mpjpe: %d predictions for %d samples' % (y.shape[0], n))
        xy = np.einsum('nij,nkj->nki', Ainv[:, :2, :2], y[:, :, 0:2]) + Ainv[:, None, :2, 2]
        z = resol_z * (y[:, :, 2] - 0.5) + rootz
        if map_to_pa17j is not None:
            xy, z = xy[:, map_to_pa17j], z[:, map_to_pa17j]
        x = (xy - c) / f
        if k is not None:
            r2 = x[..., 0] ** 2 + x[..., 1] ** 2
            radial = 1. + r2 * k[:, None, 0] + r2 ** 2 * k[:, None, 1] + r2 ** 3 * k[:, None, 2]
            tan = np.sum(x * p, axis=-1)
            x = (x - r2[..., None] * p) / (radial + tan)[..., None]
        cam = np.concatenate([x * z[..., None], z[..., None]], axis=-1)
        w = np.einsum('nij,nkj->nki', Rinv, cam) + t
        w = w - w[:, 0:1, :]
        dist = np.sqrt(np.sum((y_true - w) ** 2, axis=-1))
        out.append(float((dist * valid).sum() / valid.sum()))
    return out


def bbox_from_poses(poses, afmat, scale=1.5, min_confidence=0.25):
    """exp/common/generic.py:7-28 (`get_bbox_from_poses`, the step after `model.predict` in exp/*/predict_bboxes.py):
    the person's bounding box in IMAGE coordinates from one frame batch (N, nj, >= 3) or one clip (1, T, nj, >= 3) of
    predicted poses.  Per frame: the joints whose confidence column -- the second to last one, as the reference slices it
    (`poses[..., -2:-1]`: the last coordinate for (x, y, v) and (x, y, z, v) rows alike) -- exceeds `min_confidence`,
    the square box of `scale` x their extent around their centre (deephar/utils/bbox.py:53-76); then the union over the
    frames, its two corners through the inverse crop affine (transform.py:136-171), re-ordered.  A frame without a joint
    above the threshold raises ValueError as the reference does.  A few dozen floats: host arithmetic in float64."""
    poses = np.asarray(poses, np.float64)
    if poses.ndim == 4:
        poses = poses[0]
    elif poses.ndim != 3:
        raise ValueError('Invalid poses shape {}'.format(poses.shape))
    xy, keep = poses[:, :, 0:2], poses[:, :, -2] > min_confidence
    if not keep.any(axis=1).all():
        raise ValueError('get_valid_bbox: all points are invalid!')
    lo = np.where(keep[..., None], xy, np.inf).min(axis=1)
    hi = np.where(keep[..., None], xy, -np.inf).max(axis=1)
    centre = (lo + hi) / 2.0
    half = np.max(scale * (hi - lo) / 2.0, axis=1, keepdims=True)          # square=True: the larger half-extent
    corners = np.array([(centre - half).min(axis=0), (centre + half).max(axis=0)])       # union over the frames
    A = np.linalg.inv(np.asarray(afmat, np.float64))
    img = corners @ A[0:2, 0:2].T + A[0:2, 2]
    return np.concatenate([img.min(axis=0), img.max(axis=0)])

