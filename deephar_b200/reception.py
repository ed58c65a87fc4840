"""H100-native drop-in for deephar/models/reception.py (CVPR'18 ReceptionNet).

`build(...)` keeps the reference signature (reception.py:225-234) and returns a
`deephar_b200.model.Model` whose `.predict` / `.outputs` / `.input_shape` /
`.load_weights` follow the keras.Model protocol the reference evaluators use
(exp/common/mpii_tools.py:63-90, h36m_tools.py:12-50).  The layer graph recorded here is
the reference's, layer for layer; model.py compiles it into fused sm_90a kernels.
"""
from .graph import Graph
from .layers import (MaxPooling2D, UpSampling2D, act_conv, act_conv_bn, add, concatenate,
                     conv_bn, conv_bn_act, separable_act_conv_bn)


def _sepconv_residual(x, out_size, name, kernel_size=(3, 3)):
    """reception.py:43-59: pre-activated separable residual unit.  The shortcut is the input itself when the
    width is kept, else a 1x1 projection; a narrowing unit first reduces the width with another 1x1."""
    width = x.channels
    ident = x if width == out_size else act_conv_bn(x, out_size, (1, 1), name=name + '_shortcut')
    if out_size < width:
        x = act_conv_bn(x, out_size, (1, 1), name=name + '_reduce')
    return add([ident, separable_act_conv_bn(x, out_size, kernel_size, name=name)])


def _chain(x, steps):
    """Apply [(layer helper, filters, kernel size[, strides])...] in sequence (layers are created in list order,
    which is what numbers keras' auto-named conv2d_N / batch_normalization_N layers)."""
    for step in steps:
        fn, filters, size = step[:3]
        x = fn(x, filters, size, strides=step[3]) if len(step) > 3 else fn(x, filters, size)
    return x


def _stem(inp, old_model=False):
    """reception.py:61-98 (Inception-v4 style stem, 256x256x3 -> 32x32x576): three 3x3 convs, then three
    two-branch stages whose branches are concatenated, then a widening separable residual."""
    assert not old_model, 'old_model=True is not used by any shipped script and is not supported'
    with inp.g.scope('Stem'):
        x = _chain(inp, [(conv_bn_act, 32, (3, 3), (2, 2)), (conv_bn_act, 32, (3, 3)), (conv_bn_act, 64, (3, 3))])
        x = concatenate([conv_bn_act(x, 96, (3, 3), strides=(2, 2)),
                         MaxPooling2D(x, (3, 3), strides=(2, 2), padding='same')])
        x = concatenate([_chain(x, [(conv_bn_act, 64, (1, 1)), (conv_bn, 96, (3, 3))]),
                         _chain(x, [(conv_bn_act, 64, (1, 1)), (conv_bn_act, 64, (5, 1)), (conv_bn_act, 64, (1, 5)),
                                    (conv_bn, 96, (3, 3))])])
        x = concatenate([act_conv_bn(x, 192, (3, 3), strides=(2, 2)), MaxPooling2D(x, (2, 2), strides=(2, 2))])
        return _sepconv_residual(x, 3 * 192, name='sepconv1')


def build_reception_block(inp, name, ksize=(3, 3)):
    """reception.py:101-131: three-level hourglass.  Level 1 keeps the input width, levels 2 and 3 run at half
    the width on 2x / 4x pooled maps; each level's result is upsampled and added to the level above."""
    full, half = inp.channels, int(inp.channels / 2)

    def unit(t, width, tag):
        return _sepconv_residual(t, width, name='sepconv_' + tag, kernel_size=ksize)

    with inp.g.scope(name):
        top = unit(inp, full, 'l1')
        mid_in = unit(act_conv_bn(MaxPooling2D(inp, (2, 2)), half, (1, 1)), half, 'l2_1')
        mid = unit(mid_in, half, 'l2_2')
        low = MaxPooling2D(mid_in, (2, 2))
        for tag in ('l3_1', 'l3_2', 'l3_3'):
            low = unit(low, half, tag)
        mid = unit(add([mid, UpSampling2D(low, (2, 2))]), full, 'l2_3')
        return add([top, UpSampling2D(mid, (2, 2))])


def build_sconv_block(inp, name=None, ksize=(3, 3)):
    """reception.py:134-142."""
    with inp.g.scope(name):
        return separable_act_conv_bn(inp, inp.channels, ksize)


def build_regmap_block(inp, num_maps, name=None):
    """reception.py:145-153."""
    with inp.g.scope(name):
        return act_conv(inp, num_maps, (1, 1))


def build_fremap_block(inp, num_filters, name=None):
    """reception.py:156-164."""
    with inp.g.scope(name):
        return act_conv_bn(inp, num_filters, (1, 1))


def pose_regression_2d_context(h, num_joints, num_context_per_joint, alpha):
    """reception.py:167-182 with sSAM/cSAM (blocks.py:306-325), sjProb/cjProb on the RAW maps
    (blocks.py:328-343) and Agg (blocks.py:217-285) -- one parameter-free graph op, one kernel."""
    pose, visible = h.g.op('pose_regression_2d_context', [h],
                           [(1, num_joints, 2), (1, num_joints, 1)],
                           {'num_joints': num_joints, 'num_context': num_context_per_joint,
                            'alpha': float(alpha)})
    from .layers import channel_slice
    hs = channel_slice(h, 0, num_joints)
    return pose, visible, hs


def pose_regression_2d(h):
    """reception.py:185-190 (unreachable from build(): num_context_per_joint defaults to 2)."""
    c = h.channels
    pose, visible = h.g.op('pose_regression_2d', [h], [(1, c, 2), (1, c, 1)], {})
    return pose, visible, h


def pose_regression_3d(h, num_joints, depth_maps):
    """reception.py:193-222 (zSAM: blocks.py:288-303)."""
    assert h.channels == depth_maps * num_joints
    pose, visible = h.g.op('pose_regression_3d', [h], [(1, num_joints, 3), (1, num_joints, 1)],
                           {'num_joints': num_joints, 'depth_maps': depth_maps})
    return pose, visible, None


def build(input_shape, num_joints, dim,
          num_context_per_joint=None,
          alpha=0.8,
          num_blocks=4,
          depth_maps=16,
          ksize=(3, 3),
          export_heatmaps=False,
          export_vfeat_block=None,
          old_model=False,
          concat_pose_confidence=True):
    """reception.py:225-319."""
    from .model import Model

    if dim == 2:
        if num_context_per_joint is None:
            num_context_per_joint = 2
        num_heatmaps = (num_context_per_joint + 1) * num_joints
    elif dim == 3:
        assert num_context_per_joint is None, \
            'For 3D pose estimation, contextual heat maps are not allowed.'
        num_heatmaps = depth_maps * num_joints
    else:
        raise ValueError('"dim" must be 2 or 3 and not (%d)' % dim)
    if export_heatmaps and dim == 3:
        raise NotImplementedError('export_heatmaps with dim=3 (hxy marginal) is not exported')

    g = Graph('ReceptionNet')
    x = _stem(g.input(tuple(input_shape)), old_model=old_model)
    width = x.channels
    outputs, vfeat = [], None
    for block in range(1, num_blocks + 1):
        trunk = build_reception_block(x, name='rBlock%d' % block, ksize=ksize)
        if export_vfeat_block == block:
            vfeat = trunk
        feat = build_sconv_block(trunk, name='SepConv%d' % block, ksize=ksize)
        h = build_regmap_block(feat, num_heatmaps, name='RegMap%d' % block)

        # parameter-free regression head on the heat-maps (one kernel)
        if dim == 3:
            pose, visible, hm = pose_regression_3d(h, num_joints, depth_maps)
        elif num_context_per_joint is not None:
            pose, visible, hm = pose_regression_2d_context(h, num_joints, num_context_per_joint, alpha)
        else:
            pose, visible, hm = pose_regression_2d(h)
        outputs += [concatenate([pose, visible])] if concat_pose_confidence else [pose, visible]
        if export_heatmaps:
            outputs.append(hm)

        if block < num_blocks:      # re-inject the heat-maps into the feature stream of the next block
            x = add([trunk, feat, build_fremap_block(h, width, name='fReMap%d' % block)])
    if vfeat is not None:
        outputs.append(vfeat)

    g.outputs = outputs
    calib_key = 'reception_j%d_d%d_c%s_k%d' % (num_joints, dim, num_context_per_joint, ksize[0])
    m = Model(g, calib_key=calib_key)
    m.build_args = dict(num_joints=num_joints, dim=dim, num_context_per_joint=num_context_per_joint,
                        num_blocks=num_blocks, ksize=tuple(ksize))
    return m
