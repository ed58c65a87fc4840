"""Streamed clip inference (deephar_b200/stream.py) vs whole-clip forwards, on one GPU.

For C4 (PennAction SPNet) and C5 (NTU SPNet), 256 x 256 frames, T = 16, synthetic weights and frames, and S streams:
  push       ClipStream.push of one new frame per stream: ms per push (CUDA events around warmed CUDA-graph replays) and
             windows/s (S decisions per push)
  clips      Model.forward_device on the same S windows as S clips of T frames: ms per call, windows/s
Prints the card's name and power limit next to the numbers, one JSON line per (config, S) and a summary table.

    python tools/stream_bench.py [--configs C4 C5] [--streams 1 8 32] [--steps 20] [--warmup 3] [--out results.json]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

FRAMES = 16


def build(name):
    from deephar_b200 import spnet
    from deephar_b200.config import ModelConfig, pa16j2d, pa17j3d
    if name == 'C4':
        cfg = ModelConfig((FRAMES, 256, 256, 3), pa16j2d, num_actions=[15], num_pyramids=6, action_pyramids=[5, 6],
                          num_levels=4, pose_replica=True, num_pose_features=160, num_visual_features=160)
    else:
        cfg = ModelConfig((FRAMES, 256, 256, 3), pa17j3d, num_actions=[60], num_pyramids=2, action_pyramids=[1, 2],
                          num_levels=4, num_pose_features=192, num_visual_features=192)
    return spnet.build(cfg).init_synthetic_weights(1234)


def card(torch):
    """name and power limit of the device, read in the same run as the measurement"""
    info = {'name': torch.cuda.get_device_name(0), 'power_limit_w': None}
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader,nounits', '-i', '0'],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        if out:
            info['power_limit_w'] = float(out.split(',')[-1])
    except (OSError, ValueError, subprocess.SubprocessError):
        pass
    return info


def timed(torch, fn, steps):
    """ms per call of fn over `steps` back-to-back calls, from CUDA events"""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / steps


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--configs', nargs='+', default=['C4', 'C5'], choices=['C4', 'C5'])
    ap.add_argument('--streams', nargs='+', type=int, default=[1, 8, 32])
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--out', default=None, help='also write the result lines to this JSON file')
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit('stream_bench: no CUDA device (the numbers are GPU timings; there is nothing to measure here)')
    from deephar_b200.stream import ClipStream
    from oracle import synth
    dev = card(torch)
    print('device: %s, power limit %s W' % (dev['name'], dev['power_limit_w']))
    rows = []
    for name in args.configs:
        m = build(name)
        m.max_bound = 1
        for S in args.streams:
            frames = torch.from_numpy(synth.synth_frames(S, 256, 256, seed=S)).cuda()
            cs = ClipStream(m, S)
            for _ in range(max(args.warmup, 2) + FRAMES):       # graph captured on the 2nd push; ring filled
                out = cs.push(frames)
            assert out.ready.all()
            push_ms = timed(torch, lambda: cs.push(frames), args.steps)
            del cs, out
            clips = torch.from_numpy(np.stack([synth.synth_frames(FRAMES, 256, 256, seed=100 + s) for s in range(S)])).cuda()
            for _ in range(max(args.warmup, 2)):
                m.forward_device(clips)
            clip_ms = timed(torch, lambda: m.forward_device(clips), args.steps)
            del clips
            m._bound = {}
            torch.cuda.empty_cache()
            r = {'config': name, 'streams': S, 'frames_per_clip': FRAMES, 'push_ms': round(push_ms, 4),
                 'push_windows_per_s': round(S * 1000.0 / push_ms, 1), 'clip_forward_ms': round(clip_ms, 4),
                 'clip_forward_windows_per_s': round(S * 1000.0 / clip_ms, 1),
                 'speedup': round(clip_ms / push_ms, 2), 'device': dev['name'], 'power_limit_w': dev['power_limit_w'],
                 'steps': args.steps}
            rows.append(r)
            print(json.dumps(r), flush=True)
    print('\n%-4s %4s | %10s %12s | %12s %12s | %7s' % ('cfg', 'S', 'push ms', 'windows/s', 'clip fwd ms', 'windows/s',
                                                        'speedup'))
    for r in rows:
        print('%-4s %4d | %10.3f %12.1f | %12.3f %12.1f | %6.2fx' % (
            r['config'], r['streams'], r['push_ms'], r['push_windows_per_s'], r['clip_forward_ms'],
            r['clip_forward_windows_per_s'], r['speedup']))
    if args.out:
        with open(args.out, 'w') as f:
            json.dump({'device': dev, 'results': rows}, f, indent=1)


if __name__ == '__main__':
    main()
