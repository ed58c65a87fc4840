"""Run the kernel plan of a model several times on the same input (plain launches, one sync at the end of each
forward) and report, per forward, the first kernel op whose output differs BITWISE from the first forward's --
every kernel here is deterministic by construction, so any difference is a race.

    python tools/determinism_check.py reception2d|reception2d_k3|reception3d|spnet_penn|spnet_ntu RES N REPS [graph]
"""
import os
import sys
import zlib

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from deephar_b200 import _ffi, reception, spnet  # noqa: E402
from deephar_b200.config import ModelConfig, pa16j2d, pa17j3d  # noqa: E402


def build(name, res, frames=2):
    """-> (model, whether it takes clips)"""
    if name == 'reception2d':
        return reception.build((res, res, 3), num_joints=16, dim=2, num_context_per_joint=2, num_blocks=2, ksize=(5, 5),
                               concat_pose_confidence=False), False
    if name == 'reception2d_k3':
        return reception.build((res, res, 3), num_joints=16, dim=2, num_blocks=2, ksize=(3, 3), export_heatmaps=True), False
    if name == 'reception3d':
        return reception.build((res, res, 3), num_joints=17, dim=3, num_blocks=2, ksize=(5, 5), concat_pose_confidence=False), False
    if name == 'spnet_penn':
        return spnet.build(ModelConfig((frames, res, res, 3), pa16j2d, num_actions=[15], num_pyramids=2, action_pyramids=[1, 2],
                                       num_levels=4, pose_replica=True, num_pose_features=160, num_visual_features=160)), True
    return spnet.build(ModelConfig((frames, res, res, 3), pa17j3d, num_actions=[60], num_pyramids=2, action_pyramids=[1, 2],
                                   num_levels=4, num_pose_features=192, num_visual_features=192)), True


def main():
    name, res, n, reps = sys.argv[1], int(sys.argv[2]), int(sys.argv[3]), int(sys.argv[4])
    m, clip = build(name, res)
    m.init_synthetic_weights(1234)
    m.use_cuda_graph = False
    T = m.graph.frames_per_clip
    rng = np.random.default_rng(5)
    x = rng.uniform(-1, 1, ((n, T, res, res, 3) if clip else (n, res, res, 3))).astype(np.float32)
    n_frames = n * T if clip else n
    b = m._bind(n_frames)
    plan = m.plan
    s_in = plan.storage[m.graph.inputs[0].id]
    stream = torch.cuda.current_stream().cuda_stream
    m._ctx.set_workspace(b.workspace.data_ptr(), b.workspace.numel() * 4)
    xd = torch.from_numpy(x).reshape(-1).cuda()

    def out_tensor(t):
        s = plan.storage[t.id]
        items = m._items(t.kind, n_frames)
        base = b.slots[s.buf.phys].view(items, t.shape[0], t.shape[1], s.ld)
        return base[..., s.c_off:s.c_off + t.shape[2]]

    first = None
    bad_runs = 0
    for rep in range(reps):
        b.slots[s_in.buf.phys].copy_(xd)
        snaps = []
        for k, call in zip(plan.kops, b.calls):
            rc = call[1](*call[2:], stream)
            _ffi.check(rc, call[0])
            # snapshot the op's outputs on the device (stream-ordered clone: no host sync between kernels)
            snaps.append([out_tensor(t).clone() for t in k.outs])
        torch.cuda.synchronize()
        sig = [[zlib.crc32(t.cpu().numpy().tobytes()) for t in ts] for ts in snaps]
        if first is None:
            first, first_snaps = sig, snaps
            continue
        for i, (a, c) in enumerate(zip(first, sig)):
            if a != c:
                k = plan.kops[i]
                d = (snaps[i][0] != first_snaps[i][0])
                idx = d.nonzero()
                label = '%s %s->%s %s' % (k.kind, 'x'.join(map(str, k.ins[0].shape)), 'x'.join(map(str, k.outs[0].shape)),
                                          k.attrs.get('size', '') if isinstance(k.attrs, dict) else '')
                mx = (snaps[i][0] - first_snaps[i][0]).abs().max().item()
                print('rep %d: FIRST DIFFERENCE at op %d  %s : %d elements differ (max |d| %.3e); first at %s'
                      % (rep, i, label, int(d.sum().item()), mx, idx[0].tolist() if len(idx) else None))
                bad_runs += 1
                break
    print('%s res %d n %d: %d of %d repeated forwards differ from the first' % (name, res, n, bad_runs, reps - 1))


if __name__ == '__main__':
    main()
