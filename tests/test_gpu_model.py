"""Engine-level behaviour on the GPU: CUDA-graph replay == plain launches, no silent CUDA-core fallbacks at the
BASELINE configs, keras predict edge cases, Keras HDF5 weights through the device path."""
import numpy as np
import pytest

from deephar_b200 import _ffi, reception, spnet
from deephar_b200.config import ModelConfig, pa16j2d, pa17j3d
from oracle import synth

pytestmark = pytest.mark.gpu

C2_KW = dict(num_joints=16, dim=2, num_context_per_joint=2, num_blocks=8, ksize=(5, 5), concat_pose_confidence=False)
C3_KW = dict(num_joints=17, dim=3, num_blocks=8, ksize=(5, 5), concat_pose_confidence=False)


def _spnet(which, frames=2):
    if which == 'C4':
        return spnet.build(ModelConfig((frames, 256, 256, 3), pa16j2d, num_actions=[15], num_pyramids=6, action_pyramids=[5, 6],
                                       num_levels=4, pose_replica=True, num_pose_features=160, num_visual_features=160))
    return spnet.build(ModelConfig((frames, 256, 256, 3), pa17j3d, num_actions=[60], num_pyramids=2, action_pyramids=[1, 2],
                                   num_levels=4, num_pose_features=192, num_visual_features=192))


def test_cuda_graph_replay_equals_plain_launches(cuda):
    m = reception.build((128, 128, 3), **dict(C2_KW, num_blocks=2)).init_synthetic_weights(1234)
    x = synth.synth_frames(3, 128, 128, seed=5)
    m.use_cuda_graph = False
    ref = m.predict(x, batch_size=3)
    m.use_cuda_graph = True
    m._bound = {}
    first = m.predict(x, batch_size=3)            # plain launches (first use of the bound batch size)
    second = m.predict(x, batch_size=3)           # captures the graph, replays it
    third = m.predict(x[::-1].copy(), batch_size=3)[0][::-1]     # replay on other data
    b = m._bind(3)
    assert getattr(b, 'graph', None) is not None and m._graph_replays >= 2
    for a, r, s in zip(first, ref, second):
        assert np.array_equal(a, r) and np.array_equal(s, r)
    assert np.array_equal(third, ref[0])


# fallbacks: the convolutions each BASELINE config leaves to the CUDA-core fallback (2-frame clips for C4 / C5)
@pytest.mark.parametrize('which,fallbacks', [('C2', 0), ('C3', 0), ('C4', 5), ('C5', 5)])
def test_no_unexpected_cuda_core_fallback(cuda, which, fallbacks):
    """Every convolution of the BASELINE models must be served by a tensor-core / specialised kernel.  The only
    layers left to the two-kernel CUDA-core path are SPNet's separable convs on the action maps (maps that do not tile
    into 128-pixel tiles): they must be exactly the ones the library counts (dh_fallback_count) and flags when the
    plan is bound, and carry < 0.5 % of the model's convolution FLOPs.  C2 / C3 (ReceptionNet) have none."""
    if which in ('C2', 'C3'):
        m = reception.build((256, 256, 3), **(C2_KW if which == 'C2' else C3_KW)).init_synthetic_weights(1234)
        x = synth.synth_frames(2, seed=3)
    else:
        m = _spnet(which).init_synthetic_weights(1234)
        x = np.stack([synth.synth_frames(2, seed=3)])
    m.use_cuda_graph = False
    m.predict(x)
    lib = _ffi.lib()
    lib.dh_fallback_count(m._ctx.handle, 1)
    m.predict(x)
    got = int(lib.dh_fallback_count(m._ctx.handle, 1))
    convs = [k for k in m.plan.kops if k.kind in ('conv', 'sepconv')]
    flagged = [k for k, info in m._bind(2).conv_plans if info.fallback]

    def flops(k):
        ho, wo, cout = k.outs[0].shape
        cin = k.ins[0].shape[2]
        kh, kw = k.attrs['size']
        f = ho * wo * (kh * kw * cin * cout if k.kind == 'conv' else kh * kw * cin + cin * cout)
        return f / (m.graph.frames_per_clip if k.outs[0].kind == 'clip' else 1.0)
    share = sum(flops(k) for k in flagged) / sum(flops(k) for k in convs)
    assert got == fallbacks, '%d convolutions fell back to the CUDA-core kernel, %d expected' % (got, fallbacks)
    assert len(flagged) == fallbacks, flagged
    assert all(k.kind == 'sepconv' and k.outs[0].kind == 'clip' for k in flagged), flagged
    assert share < 0.005, share


def test_predict_edge_cases(cuda):
    m = reception.build((64, 64, 3), **dict(C2_KW, num_blocks=1)).init_synthetic_weights(7)
    outs = m.predict(np.zeros((0, 64, 64, 3), np.float32))
    assert [o.shape for o in outs] == [(0, 16, 2), (0, 16, 1)]
    x = synth.synth_frames(5, 64, 64, seed=2)
    a = m.predict(x, batch_size=2)               # ragged tail batch (2 + 2 + 1): three bound sizes, LRU of two
    b = m.predict(x, batch_size=5)
    for u, v in zip(a, b):
        assert np.abs(u - v).max() <= 1e-6
    assert len(m._bound) <= m.max_bound
    with pytest.raises(ValueError):
        m.predict(np.zeros((1, 32, 32, 3), np.float32))
    # results are the caller's: a later call with the same batch size (the pinned result buffers are kept) must not
    # write into arrays handed out earlier; a one-element input list is the array (keras)
    y = synth.synth_frames(5, 64, 64, seed=3)
    first = [o.copy() for o in b]
    c = m.predict([y], batch_size=5)
    assert all(np.array_equal(u, v) for u, v in zip(b, first)) and np.abs(c[0] - b[0]).max() > 1e-4
    d = m.predict(x, batch_size=None)
    assert all(np.abs(u - v).max() <= 1e-6 for u, v in zip(d, first))


def test_keras_h5_weights_drive_the_device_path(cuda, tmp_path):
    """save_weights('.h5') -> fresh model -> load_weights('.h5') -> identical predictions (SURVEY.md 8 f1)."""
    kw = dict(C2_KW, num_blocks=1)
    m = reception.build((64, 64, 3), **kw).init_synthetic_weights(11)
    p = str(tmp_path / 'weights_PE_tiny.h5')
    m.save_weights(p)
    m2 = reception.build((64, 64, 3), **kw)
    m2.load_weights(p)
    x = synth.synth_frames(2, 64, 64, seed=4)
    for a, b in zip(m.predict(x), m2.predict(x)):
        assert np.array_equal(a, b)
