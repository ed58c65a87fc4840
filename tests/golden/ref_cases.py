"""Case table shared by make_reference_golden.py (which runs the REFERENCE builders on keras_shim) and
tests/test_reference_golden.py (which checks the oracle and the product against the fixtures it wrote)."""

RECEPTION_CASES = {
    # case: (input shape, reception.build kwargs, weight seed, input seed[, frames])
    'reception2d_ctx': ((64, 64, 3), dict(num_joints=16, dim=2, num_blocks=2, ksize=(5, 5), num_context_per_joint=2,
                                          concat_pose_confidence=False), 1234, 1),
    'reception2d_heatmaps': ((64, 64, 3), dict(num_joints=16, dim=2, num_blocks=2, ksize=(3, 3), export_heatmaps=True), 7, 22),
    'reception3d': ((64, 64, 3), dict(num_joints=17, dim=3, num_blocks=2, ksize=(5, 5), concat_pose_confidence=False), 1234, 23),
    # the BASELINE.json configs[1] model at full size (eval_penn_ar_pe_merge.py:51-53 / eval_mpii_singleperson.py:47), 1 frame
    'reception2d_c1_fullsize': ((256, 256, 3), dict(num_joints=16, dim=2, num_blocks=8, ksize=(5, 5), num_context_per_joint=2,
                                                    concat_pose_confidence=False), 1234, 31, 1),
}

# full-size BASELINE configs, inputs regenerated from their seed (the fixture stores seed + checksum, not the frames)
RECEPTION_CASES.update({
    # configs[2]: exp/h36m/eval_h36m.py:42-48 -- 3-D pose, 17 joints, 8 blocks, 256x256
    'reception3d_c3_fullsize': ((256, 256, 3), dict(num_joints=17, dim=3, num_blocks=8, ksize=(5, 5),
                                                    concat_pose_confidence=False), 1234, 41, 1),
    # configs[0]/[1] with every block's heat-maps exported: arg-max pixels of all 8 heads
    'reception2d_c1_heatmaps': ((256, 256, 3), dict(num_joints=16, dim=2, num_blocks=8, ksize=(5, 5), num_context_per_joint=2,
                                                    concat_pose_confidence=False, export_heatmaps=True), 1234, 43, 1),
})
LARGE_INPUT_CASES = ('reception3d_c3_fullsize', 'reception2d_c1_heatmaps', 'spnet_penn_c4_t16', 'spnet_ntu_c5_t16')

SPNET_CASES = {
    # case: (cfg input shape, pose layout name, ModelConfig kwargs, weight seed, batch)
    'spnet_penn_like': ((2, 128, 128, 3), 'pa16j2d',
                        dict(num_actions=[15], num_pyramids=2, action_pyramids=[1, 2], num_levels=4, pose_replica=True,
                             num_pose_features=160, num_visual_features=160), 1234, 1),
    'spnet_ntu_like': ((2, 128, 128, 3), 'pa17j3d',
                       dict(num_actions=[60], num_pyramids=2, action_pyramids=[1, 2], num_levels=4, num_pose_features=192,
                            num_visual_features=192), 1234, 1),
    'spnet_pose_only': ((128, 128, 3), 'pa16j2d', dict(num_pyramids=2, action_pyramids=[], num_levels=4), 5, 2),
    # the BASELINE.json configs[3] architecture (exp/pennaction/eval_penn_multitask.py:37-40) at full resolution; the clip
    # is cut to 2 frames (the clip length only sets the temporal extent of the action head's input)
    'spnet_penn_c4_t2': ((2, 256, 256, 3), 'pa16j2d',
                         dict(num_actions=[15], num_pyramids=6, action_pyramids=[5, 6], num_levels=4, pose_replica=True,
                              num_pose_features=160, num_visual_features=160), 1234, 1),
}

# full clips: x = default_rng(seed_x).uniform(-1, 1, (batch,) + shape) (own generator per case)
SPNET_FULL_CASES = {
    # case: (cfg input shape, pose layout, ModelConfig kwargs, weight seed, batch, input seed)
    # configs[3] (exp/pennaction/eval_penn_multitask.py:37-40 with 8 -> 16 frames): time_stride = 2 in the action head
    'spnet_penn_c4_t16': ((16, 256, 256, 3), 'pa16j2d',
                          dict(num_actions=[15], num_pyramids=6, action_pyramids=[5, 6], num_levels=4, pose_replica=True,
                               num_pose_features=160, num_visual_features=160), 1234, 1, 101),
    # configs[4] (exp/ntu/eval_ntu_multitask.py:35-38 with 8 -> 16 frames), 3-D poses, 60 actions
    'spnet_ntu_c5_t16': ((16, 256, 256, 3), 'pa17j3d',
                         dict(num_actions=[60], num_pyramids=2, action_pyramids=[1, 2], num_levels=4, num_pose_features=192,
                              num_visual_features=192), 1234, 1, 102),
}

# CVPR'18 merge model (exp/pennaction/eval_penn_ar_pe_merge.py:42-62), small geometry
def positive_last_regmap(table, num_blocks):
    """Weight hook of the merge-model cases: |kernel| for the LAST RegMap conv.  Its input is ReLU(x) >= 0, so the
    heat-maps and with them the raw joint confidences are >= 0 and the context aggregation's division by
    sum(pc) (blocks.py:264-267) is perfectly conditioned for every joint -- the action outputs, which consume ALL
    joints' poses, can then be held to the 1e-3 bar instead of being bounded by the worst joint's cancellation."""
    import numpy as np
    out = dict(table)
    for name in table:
        if name.startswith('RegMap%d/' % num_blocks) and name.endswith('/kernel'):
            out[name] = np.abs(table[name])
    return out


MERGE_CASE = dict(input_shape=(64, 64, 3), num_frames=4, num_actions=15, num_joints=16, num_blocks=4, seed=3,
                  reception=dict(num_joints=16, dim=2, num_blocks=4, num_context_per_joint=2, ksize=(5, 5)))

# the 3-D variant of the merge model (action.py:208-297 via build_merge_model(pose_dim=3)); 20 joints (pa20j3d):
# the PoseAR net pools and re-upsamples the joint axis, which only closes for joint counts divisible by 4
MERGE3D_CASE = dict(input_shape=(64, 64, 3), num_frames=4, num_actions=15, num_joints=20, num_blocks=2, depth_maps=8, seed=9,
                    reception=dict(num_joints=20, dim=3, num_blocks=2, depth_maps=8, ksize=(5, 5)))


class SweepCase(object):
    """One configuration of ref_option_sweep.npz (written by make_option_sweep_golden.py).

    tag      the generator's label of the configuration
    spec     its builder arguments as stored: builder ('reception' / 'spnet'), shape, num_joints or layout, kw
    x        the float64 input: the draw of default_rng(2020) that belongs to this case, in case order
    kw       the builder's keyword arguments (kernel sizes as tuples)
    refs     per output of the reference builders: (shape, flat indices of the stored sample, sampled values)
    build()  the product's model for the same arguments, with init_synthetic_weights(1234)
    """

    def __init__(self, tag, spec, x, refs):
        self.tag, self.spec, self.x, self.refs = tag, spec, x, refs
        self.kw = {k: (tuple(v) if k in ('ksize', 'kernel_size') else v) for k, v in spec['kw'].items()}

    def build(self):
        from deephar_b200 import config, reception, spnet
        s, kw = self.spec, self.kw
        if s['builder'] == 'reception':
            m = reception.build(tuple(s['shape']), s['num_joints'], **kw)
        else:
            m = spnet.build(config.ModelConfig(tuple(s['shape']), getattr(config, s['layout']), **kw))
        return m.init_synthetic_weights(1234)


def option_sweep_cases():
    """The 10 stored option-sweep cases, in file order.  Every input is drawn, so any one case's input is the one the
    fixture was made with."""
    import json
    import os
    import numpy as np
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'ref_option_sweep.npz'))
    rng = np.random.default_rng(2020)
    cases = []
    for i in range(sum(1 for k in g.files if k.endswith('/case'))):
        spec = json.loads(str(g['%d/case' % i]))
        x = rng.uniform(-1, 1, tuple(spec['x_shape']))
        refs = [(tuple(int(d) for d in g['%d/shape%02d' % (i, k)]), g['%d/idx%02d' % (i, k)], g['%d/out%02d' % (i, k)])
                for k in range(sum(1 for f in g.files if f.startswith('%d/out' % i)))]
        cases.append(SweepCase(spec['tag'], spec, x, refs))
    return cases
