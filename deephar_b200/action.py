"""H100-native drop-in for deephar/models/action.py::build_merge_model -- the CVPR'18 clip model
(ReceptionNet pose estimation re-wired under TimeDistributed + PoseAR + GuidedVisAR action nets): the 2-D
pose variant used by exp/pennaction/eval_penn_ar_pe_merge.py:42-62 and the 3-D one (action.py:208-297,
`pose_dim=3`, volumetric heat-maps with `depth_maps` slices).

Signature, output order ([pose, visibility,] p1..p4, v1..v4, m: action.py:340-396) and weight
names (backbone keeps the ReceptionNet layer names; PoseAR/, GuidedVisAR/ sub-models) follow the
reference.
"""
from . import reception as R
from .graph import Graph
from .layers import (MaxPooling2D, UpSampling2D, act_conv, act_conv_bn, add, channel_slice,
                     channel_softmax_2d, concatenate, conv_bn, conv_bn_act, frames_to_clip,
                     global_max_min_pooling, kronecker_prod, mask_multiply, max_min_pooling,
                     sepconv2d, softmax_lastaxis)


def action_top(x, name=None):
    """action.py:14-17."""
    x = global_max_min_pooling(x)
    return softmax_lastaxis(x, name=name)


def build_act_pred_block(x, num_out, name=None, last=False, include_top=True):
    """One action prediction stage (action.py:20-42): bottleneck residual (1x1 to half the width, 3x3 back), a 3x3
    conv whose (max + min)-pooled output carries the `num_out` action maps; unless `last`, the maps are upsampled,
    widened again and summed with both earlier tensors for the next stage."""
    width = x.channels
    trunk = add([x, act_conv_bn(act_conv_bn(x, width // 2, (1, 1)), width, (3, 3))])
    wide = act_conv_bn(trunk, width, (3, 3))
    pooled = max_min_pooling(wide, (2, 2))
    maps = act_conv(pooled, num_out, (3, 3))
    y = action_top(maps) if include_top else maps
    if last:
        return pooled, y
    back = act_conv_bn(UpSampling2D(maps, (2, 2)), width, (3, 3))
    return add([trunk, wide, back]), y


def _four_stages(x, num_actions, include_top):
    """y1..y4 of both action nets (action.py:74-81, 101-108): three chained stages and a last one without re-injection."""
    ys = []
    for i in range(1, 5):
        x, y = build_act_pred_block(x, num_actions, name='y%d' % i, include_top=include_top, last=(i == 4))
        ys.append(y)
    return ys


# widths of the pose net's two multi-branch layers (action.py:55-72): (3x1, 3x3, 3x5 branch), (3x3 / 1x1 -> 3x3 branch, 1x1)
_POSE_NET_WIDTHS = {'v1': ((8, 16, 24), (56, 32)), 'v2': ((12, 24, 36), (112, 64))}


def build_pose_model(y, p, num_actions, name='PoseAR', include_top=True, network_version='v1'):
    """action.py:45-90 applied to clip tensors y (T,nj,dim), p (T,nj,1): confidence-masked coordinates as a (T, nj)
    image -> three kernel shapes side by side -> two 3x3 branches -> (max + min) pooling -> four stages."""
    if network_version not in _POSE_NET_WIDTHS:
        raise Exception('Unkown network version "{}"'.format(network_version))
    first, (wide, squeeze) = _POSE_NET_WIDTHS[network_version]
    with y.g.scope(name):
        x = mask_multiply(y, p)
        x = concatenate([conv_bn_act(x, w, (3, kw)) for w, kw in zip(first, (1, 3, 5))])
        direct = conv_bn(x, wide, (3, 3))
        x = concatenate([direct, conv_bn(conv_bn(x, squeeze, (1, 1)), wide, (3, 3))])
        return _four_stages(max_min_pooling(x, (2, 2)), num_actions, include_top)


def build_visual_model(f, num_actions, name='GuidedVisAR', include_top=True):
    """action.py:93-109 applied to the clip tensor f (T,nj,F)."""
    with f.g.scope(name):
        return _four_stages(MaxPooling2D(conv_bn(f, 256, (1, 1)), (2, 2)), num_actions, include_top)


def _get_2d_pose_estimation_from_model(inp, num_joints, num_blocks, num_context_per_joint, ksize):
    """action.py:112-203: the ReceptionNet layers re-wired so that only the last block regresses
    the pose.  Layers are created in reception.build's order so the weight names are identical."""
    h, xb1 = _backbone_to_heatmaps(inp, (num_context_per_joint + 1) * num_joints, num_blocks, ksize)
    # ys/yc/pc/Agg (alpha 0.8) = the same parameter-free head as reception.py:167-182
    y, vis, _ = R.pose_regression_2d_context(h, num_joints, num_context_per_joint, 0.8)
    # p = sjProb(4 * hs)  (action.py:200): 4 x the raw 2x2-window maximum
    p = y.g.op('scale', [vis], vis.shape, {'value': 4.0})
    hs = channel_slice(h, 0, num_joints)
    hs = channel_softmax_2d(hs, name='td_ChannelSoftmax')                 # action.py:202-203
    return y, p, hs, xb1


def _backbone_to_heatmaps(inp, num_heatmaps, num_blocks, ksize):
    """The layer re-wiring shared by action.py:112-152 and :208-248: every block but the last feeds its
    heat-maps back (fReMap), only the last block's heat-maps are regressed."""
    x1 = R._stem(inp)
    xb1 = R.build_reception_block(x1, name='rBlock1', ksize=ksize)
    nfilt = xb1.channels
    x = xb1
    for i in range(1, num_blocks):
        t1 = x if i == 1 else R.build_reception_block(x, name='rBlock%d' % i, ksize=ksize)
        t2 = R.build_sconv_block(t1, name='SepConv%d' % i, ksize=ksize)
        t3 = R.build_fremap_block(R.build_regmap_block(t2, num_heatmaps, name='RegMap%d' % i), nfilt,
                                  name='fReMap%d' % i)
        x = add([t1, t2, t3])
    x = R.build_reception_block(x, name='rBlock%d' % num_blocks, ksize=ksize)
    x = R.build_sconv_block(x, name='SepConv%d' % num_blocks, ksize=ksize)
    return R.build_regmap_block(x, num_heatmaps, name='RegMap%d' % num_blocks), xb1


def _get_3d_pose_estimation_from_model(inp, num_joints, num_blocks, depth_maps, ksize):
    """action.py:208-297: volumetric head on the last block.  One kernel (dh_softargmax3d_ex_f32) reads the
    (D * nj)-channel volume once and produces pose = (x, y) from mean_d, z from mean_hw, visible =
    sigmoid(2 * (max hxy + max hz)) (action.py:291-292 -- twice the logit of reception.py:217-220) and
    hs = channel_softmax_2d(hxy) for the kronecker product (action.py:294-295)."""
    h, xb1 = _backbone_to_heatmaps(inp, depth_maps * num_joints, num_blocks, ksize)
    hh, ww, _ = h.shape
    pose, visible, hs = h.g.op('pose_regression_3d_ex', [h],
                               [(1, num_joints, 3), (1, num_joints, 1), (hh, ww, num_joints)],
                               {'num_joints': num_joints, 'depth_maps': depth_maps, 'vis_scale': 2.0})
    return pose, visible, hs, xb1


def build_merge_model(model_pe,
                      num_actions,
                      input_shape,
                      num_frames,
                      num_joints,
                      num_blocks,
                      pose_dim=2,
                      depth_maps=8,
                      num_context_per_joint=2,
                      pose_net_version='v1',
                      output_poses=False,
                      weighted_merge=True,
                      ar_pose_weights=None,
                      ar_visual_weights=None,
                      full_trainable=False):
    """action.py:319-400."""
    from .model import Model

    if pose_dim not in (2, 3):
        raise ValueError('"pose_dim" must be 2 or 3 and not (%r)' % (pose_dim,))
    if ar_pose_weights is not None or ar_visual_weights is not None:
        raise NotImplementedError('load the merged weight file with Model.load_weights instead')
    ksize = getattr(model_pe, 'build_args', {}).get('ksize', (3, 3))

    g = Graph('MergeModel')
    g.frames_per_clip = int(num_frames)
    inp = g.input(tuple(input_shape))
    outputs = []

    if pose_dim == 2:
        y, p, hs, xb1 = _get_2d_pose_estimation_from_model(inp, num_joints, num_blocks,
                                                           num_context_per_joint, ksize)
    else:
        y, p, hs, xb1 = _get_3d_pose_estimation_from_model(inp, num_joints, num_blocks, depth_maps, ksize)
    n_backbone = len(g.weight_specs)
    if g.weight_specs != model_pe.weight_specs[:n_backbone] or n_backbone != len(model_pe.weight_specs):
        raise ValueError('model_pe does not match (num_joints, num_blocks, num_context_per_joint / depth_maps)')

    if output_poses:
        outputs.append(y)
        outputs.append(p)

    yc, pc = frames_to_clip(y), frames_to_clip(p)
    out_pose = build_pose_model(yc, pc, num_actions, include_top=False, name='PoseAR',
                                network_version=pose_net_version)

    f = kronecker_prod(hs, xb1)
    out_vis = build_visual_model(frames_to_clip(f), num_actions, include_top=False, name='GuidedVisAR')

    for i in range(len(out_pose)):
        outputs.append(action_top(out_pose[i], name='p%d' % (i + 1)))
    for i in range(len(out_vis)):
        outputs.append(action_top(out_vis[i], name='v%d' % (i + 1)))

    pm = out_pose[-1]
    vm = out_vis[-1]

    def _heatmap_weighting(t):
        """action.py:377-390: SeparableConv2D(C, (1,1)) initialised to identity (its weights are part of
        the model's weight list, so a trained file may hold anything)."""
        return sepconv2d(t, t.channels, (1, 1))

    if weighted_merge:
        pm = _heatmap_weighting(pm)
        vm = _heatmap_weighting(vm)

    m = add([pm, vm])
    outputs.append(action_top(m, name='m'))

    g.outputs = outputs
    model = Model(g, calib_key='merge%s_j%d_b%d_k%d' % ('' if pose_dim == 2 else '3d', num_joints, num_blocks, ksize[0]),
                  name='MergeModel')
    if getattr(model_pe, '_host_weights', None):
        model._backbone_weights = dict(model_pe._host_weights)      # shared layers (Keras shares them)
    return model
