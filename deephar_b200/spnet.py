"""H100-native drop-in for deephar/models/spnet.py (SPNet v1, TPAMI'20 multitask pose + action).

`build(cfg)` keeps the reference signature (spnet.py:355) and output ordering: pose outputs
(B,T,nj,dim+1) named dp1_pb1.. in pyramid order, then the action outputs (B,n_act)
(spnet.py:398-408, SURVEY.md App. F); `split_model` / `get_num_predictions` follow
spnet.py:413-448.  Every layer carries the reference's name, so `load_weights(by_name=True)` of a released
checkpoint finds its weights; tests/test_reference_golden.py pins the weight list (names and shapes) and the
outputs against the reference's own builder.  The topology is expressed here in this package's own terms:
one pyramid walker for both directions, one soft-argmax head used for the prediction and its action-side
replica, one pad-and-pool helper for the two feature streams of the action head.
"""
import math

from .common import add_tensorlist, concat_tensorlist, downscaling, residual, upscaling
from .config import ModelConfig
from .graph import Graph
from .layers import (BatchNormalization, UpSampling2D, ZeroPadding2D, add, appstr,
                     channel_softmax_2d, concatenate, conv2d, depth_expectation, frames_to_clip,
                     global_max_min_pooling, keypoint_confidence, kronecker_prod, mask_multiply,
                     max_min_pooling, maxpooling2d, relu, sepconv2d, softargmax2d, softmax_lastaxis)


# ------------------------------------------------------------------------------------------------------
# heads
# ------------------------------------------------------------------------------------------------------
def prediction_branch(x, cfg, pred_activate=True, replica=None, forward_maps=True, name=None):
    """spnet.py:24-48: features -> nj heat-maps (`pred_maps`, optionally a second set for the action side)
    -> back to features.  Returns (re-injected features, pred_maps, replica maps or the falsy input)."""
    nj, width = cfg.num_joints, x.channels
    feats = relu(x, name=appstr(name, '_act1'))
    pred_maps = conv2d(feats, nj, (1, 1), name=appstr(name, '_conv1'))
    if replica:
        replica = conv2d(feats, nj, (1, 1), name=appstr(name, '_conv1_replica'))
    back = pred_maps
    if forward_maps:
        back = concatenate([conv2d(feats, nj, (1, 1), name=appstr(name, '_fw_maps')), pred_maps])
    if pred_activate:
        back = relu(back, name=appstr(name, '_act2'))
    return conv2d(back, width, (1, 1), name=appstr(name, '_conv2')), pred_maps, replica


def _soft_argmax_head(cfg, maps, depth_maps, prefix, suffix=''):
    """spnet.py:190-205 (and :216-229 for the action-side copy): probability maps, (x, y) expectation, joint
    confidence and -- for 3-D layouts -- the depth expectation appended as z.  One fused kernel downstream."""
    box = (cfg.xmin, cfg.ymin, 1 - cfg.xmin, 1 - cfg.ymin)
    prob = channel_softmax_2d(maps, alpha=cfg.sam_alpha, name=appstr(prefix, '_probmaps' + suffix))
    pose = softargmax2d(prob, limits=box, name=appstr(prefix, '_xy' + suffix))
    conf = keypoint_confidence(prob, name=appstr(prefix, '_vis' + suffix))
    if depth_maps is not None:
        pose = concatenate([pose, depth_expectation(depth_maps, prob)], name=appstr(prefix, '_xyz' + suffix))
    return prob, pose, conf


def action_prediction_early_fusion(xa, p, c, af, cfg, name=None):
    """spnet.py:51-148.  p (T,nj,dim), c (T,nj,1), af (T,nj,F) are clip tensors; xa is the action feature map of
    the previous prediction block (or None).  Returns ([action probabilities per action set], new xa)."""
    pose_w, vis_w = cfg.num_pose_features, cfg.num_visual_features
    tag = name[0:7] if name is not None else None

    # the (frames x joints) map is padded to a multiple of (2 * time_stride, 4) and pooled (spnet.py:98-107,124-132)
    frames, joints = p.shape[0], p.shape[1]
    t_stride = 2 if frames >= 16 else 1
    fill = lambda unit, n: int(unit * math.ceil(n / unit) - n)
    pad_t, pad_j = fill(2 * t_stride, frames), fill(4, joints)
    pads = ((pad_t // 2, (pad_t + 1) // 2), (pad_j // 2, (pad_j + 1) // 2))

    def pad_and_pool(t):
        if pad_t + pad_j > 0:
            t = ZeroPadding2D(t, pads)
        return maxpooling2d(t, (2, 2), strides=(t_stride, 2))

    # pose stream: confidence-masked coordinates through three temporal kernels, then a bottleneck residual
    masked = mask_multiply(p, c)
    taps = [conv2d(masked, pose_w // div, ks, name=appstr(name, '_p_conv0' + tag_))
            for div, ks, tag_ in ((16, (3, 1), 'a'), (8, (3, 3), 'b'), (4, (3, 5), 'c'))]
    pose_feat = residual(concatenate(taps), (3, 3), out_size=pose_w, convtype='normal', features_div=2,
                         name=appstr(name, '_r1'))
    streams = [pad_and_pool(pose_feat),
               pad_and_pool(conv2d(af, vis_w, (1, 1), name=appstr(name, '_v_conv0')))]      # appearance stream
    if xa is not None:
        streams.append(xa)
    fused = residual(concat_tensorlist(streams), (3, 3), out_size=max(pose_w, vis_w), convtype='normal',
                     features_div=4, name=appstr(name, '_r2'))

    # classification head (spnet.py:64-96): one heat-map set per action set, each pooled to probabilities
    head = appstr(name, '_pred')
    width = fused.channels
    mid = conv2d(relu(BatchNormalization(fused, name=appstr(head, '_bn1')), name=appstr(head, '_act1')),
                 width, (3, 3), name=appstr(head, '_conv1'))
    pooled = relu(BatchNormalization(max_min_pooling(mid, (2, 2)), name=appstr(head, '_bn2')), name=appstr(head, '_act2'))
    maps = [conv2d(pooled, n_act, (3, 3), name=appstr(head, '_conv2h%d' % i)) for i, n_act in enumerate(cfg.num_actions)]
    probs = [softmax_lastaxis(global_max_min_pooling(m), name=appstr(appstr(tag, '_a'), '%d' % i))
             for i, m in enumerate(maps)]
    back = conv2d(relu(UpSampling2D(concat_tensorlist(maps), (2, 2)), name=appstr(head, '_act3')),
                  width, (3, 3), name=appstr(head, '_conv3'))
    return probs, add([fused, mid, back])


def prediction_block(xp, xa, zp, outlist, cfg, do_action, name=None):
    """spnet.py:151-248 (the dbg_decoupled_* debug outputs are not built).  Appends this block's pose output
    (and action outputs) to `outlist`; returns the features handed to the next block."""
    g = xp.g
    width = xp.channels
    replica = cfg.pose_replica and do_action
    three_d = cfg.dim == 3

    trunk = residual(xp, cfg.kernel_size, name=appstr(name, '_r1'))
    conv = sepconv2d(relu(BatchNormalization(trunk, name=appstr(name, '_bn1')), name=appstr(name, '_act1')),
                     width, cfg.kernel_size, name=appstr(name, '_conv1'))
    normed = BatchNormalization(conv, name=appstr(name, '_bn2'))
    reinject = [trunk, conv]

    back, maps, maps_rep = prediction_branch(normed, cfg, pred_activate=True, replica=replica,
                                             name=appstr(name, '_heatmaps'))
    reinject.append(back)
    depth = depth_rep = None
    if three_d:
        back, depth, depth_rep = prediction_branch(normed, cfg, pred_activate=False, replica=replica,
                                                   forward_maps=False, name=appstr(name, '_depthmaps'))
    prob, pose, conf = _soft_argmax_head(cfg, maps, depth, name)
    if three_d:
        reinject.append(back)

    if do_action:
        # the reference numbers the action blocks with a module-level counter (spnet.py:210-214)
        g.act_cnt = getattr(g, 'act_cnt', 0) + 1
        act = 'act%d' % g.act_cnt
        a_prob, a_pose, a_conf = _soft_argmax_head(cfg, maps_rep if replica else maps,
                                                   (depth_rep if replica else depth) if three_d else None, act, '2')
        appearance = kronecker_prod(a_prob, zp, name=appstr(act, '_kron'))
        probs, xa = action_prediction_early_fusion(xa, frames_to_clip(a_pose), frames_to_clip(a_conf),
                                                   frames_to_clip(appearance), cfg, name=appstr(act, '_action'))
        outlist[1] += probs
    outlist[0].append(concatenate([pose, conf], name=name))
    return add_tensorlist(reinject), xa


# ------------------------------------------------------------------------------------------------------
# pyramids
# ------------------------------------------------------------------------------------------------------
def _walk_pyramid(levels, step, tag, lp, la, lzp, outlist, cfg, do_action, name):
    """One sweep over the resolution levels (spnet.py:251-314).  `step` rescales the pose features between
    levels (+growth channels going down, -growth going up); lp / la are the lateral pose / action
    connections left by the previous sweep and refreshed by this one, lzp the appearance features per level."""
    assert len(lp) == len(la), 'Pose and action must have the same number of levels!'
    start = levels[0] - 1 if tag == 'du' else levels[0] + 1
    xp, xa = lp[start], la[start]
    if lzp[0] is None:
        lzp[0] = xp
    for i in levels:
        grow = cfg.growth if tag == 'du' else -cfg.growth
        xp = step(xp, cfg, out_size=xp.channels + grow, name=appstr(name, '_%s%d' % (tag, i)))
        if lzp[i] is None:
            lzp[i] = xp
        if lp[i] is not None:
            xp = add([xp, lp[i]])
        if xa is not None and do_action:
            xa = residual(xa, (3, 3), name=appstr(name, '_%s%d_action_r0' % (tag, i)))
            if la[i] is not None:
                xa = add([xa, la[i]])
        xp, xa = prediction_block(xp, xa, lzp[i], outlist, cfg, do_action, name=appstr(name, '_pb%d' % i))
        lp[i], la[i] = xp, xa


def downscaling_pyramid(lp, la, lzp, outlist, cfg, do_action, name=None):
    """spnet.py:251-281: levels 1 .. L-1, halving the resolution."""
    _walk_pyramid(list(range(1, len(lp))), downscaling, 'du', lp, la, lzp, outlist, cfg, do_action, name)


def upscaling_pyramid(lp, la, lzp, outlist, cfg, do_action, name=None):
    """spnet.py:284-314: levels L-2 .. 0, doubling the resolution."""
    _walk_pyramid(list(range(len(lp) - 1))[::-1], upscaling, 'uu', lp, la, lzp, outlist, cfg, do_action, name)


def entry_flow(x, cfg):
    """spnet.py:317-352: 7x7/2 conv, then bottleneck residual pairs separated by poolings until the map is
    1/image_div of the input."""
    assert (cfg.image_div & (cfg.image_div - 1) == 0) and cfg.image_div >= 4, \
        'Invalid image_div ({}).'.format(cfg.image_div)
    assert cfg.downsampling_type in ['maxpooling', 'conv'], \
        'Invalid downsampling_type ({}).'.format(cfg.downsampling_type)
    if cfg.downsampling_type != 'maxpooling':
        raise NotImplementedError("downsampling_type='conv' is not used by the reference scripts")

    x = conv2d(x, 64, (7, 7), strides=(2, 2), name='conv1')
    x = residual(x, (3, 3), out_size=cfg.growth, convtype='normal', name='res0')
    x = maxpooling2d(x, (3, 3), strides=(2, 2))
    width, index, scale = 2 * cfg.growth, 1, 4
    while True:
        for _ in range(2):
            x = residual(x, (3, 3), out_size=width, convtype='normal', name='res%d' % index)
            index += 1
        if scale >= cfg.image_div:
            return x
        x = maxpooling2d(x, (2, 2), strides=(2, 2))
        width += cfg.growth
        scale *= 2


def build(cfg, stop_grad_stem=False):
    """Sequential Pyramid Networks for 3D human pose estimation and action recognition
    (spnet.py:355-410).  `stop_grad_stem` only matters for training and is ignored."""
    from .model import Model

    assert type(cfg) == ModelConfig, 'type(cfg) ({}) is not ModelConfig'.format(type(cfg))
    input_shape = tuple(cfg.input_shape)
    assert len(input_shape) in [3, 4], 'Invalid input_shape ({})'.format(input_shape)
    if cfg.dbg_decoupled_pose or cfg.dbg_decoupled_h:
        raise NotImplementedError('dbg_decoupled_* debug outputs are not built (SURVEY App. C.7)')
    clips = len(input_shape) == 4

    g = Graph('SPNet')
    if clips:
        g.frames_per_clip = int(input_shape[0])
    frame_shape = input_shape[-3:]
    inp = g.input(frame_shape)
    cfg.xmin, cfg.ymin = 1 / (2 * frame_shape[1]), 1 / (2 * frame_shape[0])      # half a pixel (spnet.py:379-380)

    outlist = [[] for _ in range(len(cfg.num_actions) + 1)]          # [[poses], [actions of set 1], ...]
    lp, la, lzp = ([None] * cfg.num_levels for _ in range(3))
    lp[0] = entry_flow(inp, cfg)
    for pyr in range(1, cfg.num_pyramids + 1):
        do_action = pyr in cfg.action_pyramids
        if do_action and not clips:
            raise ValueError('action recognition needs clip input (T,H,W,3): kronecker_prod is only '
                             'defined for clip tensors in the reference (layers.py:478-508)')
        sweep, tag = (downscaling_pyramid, 'dp') if pyr % 2 == 1 else (upscaling_pyramid, 'up')
        sweep(lp, la, lzp, outlist, cfg, do_action, name='%s%d' % (tag, pyr))

    g.outputs = [t for group in outlist for t in group]
    g.num_pose_outputs = len(outlist[0])
    key = 'spnet_j%d_d%d_p%d_a%s_r%d_f%d' % (cfg.num_joints, cfg.dim, cfg.num_pyramids,
                                              '-'.join(str(a) for a in cfg.action_pyramids),
                                              int(bool(cfg.pose_replica)), cfg.num_pose_features)
    m = Model(g, calib_key=key, name='SPNet')
    m.cfg = cfg
    return m


def get_num_predictions(num_pyramids, num_levels):
    """spnet.py:413-414."""
    return num_pyramids * (num_levels - 1)


def split_model(full_model, cfg, interlaced=False, model_names=[None, None]):
    """spnet.py:417-448: [pose model, action model] sharing the same compiled network."""
    n_pose = get_num_predictions(cfg.num_pyramids, cfg.num_levels)
    n_act = get_num_predictions(len(cfg.action_pyramids), cfg.num_levels)
    assert len(full_model.outputs) == n_pose + len(cfg.num_actions) * n_act, \
        'The given model and config are not compatible!'
    assert n_act > 0, 'You are trying to split a "pose only" model.'
    if interlaced:
        raise NotImplementedError('interlaced=True is only used by the training scripts')
    return [full_model.output_subset(range(0, n_pose), name=model_names[0]),
            full_model.output_subset(range(n_pose, len(full_model.outputs)), name=model_names[1])]
