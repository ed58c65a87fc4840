"""A model file run at fewer items than it was exported at (dh_model_set_batch) vs the padded forward, on one GPU.

C2 (8-block ReceptionNet, 256 x 256) exported at 256 frames and C4 (PennAction SPNet, 256 x 256, T = 16) exported at
16 clips, synthetic weights and frames, loaded once through the C ABI.  For each n, dh_model_set_batch(n), one forward
captured into a CUDA graph, warmed, then timed with CUDA events over back-to-back replays (best of --rounds):
  ms         per dh_model_forward at n items
  padded_ms  per dh_model_forward at N items, what padding n items to the exported batch costs
Prints the card's name and power limit next to the numbers, one JSON line per (config, n) and a summary table.

    python tools/model_batch_bench.py [--configs C2 C4] [--batches 1 8 32] [--steps 20] [--warmup 3] [--out f.json]
"""
import argparse
import ctypes as C
import json
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, 'tools')):
    if p not in sys.path:
        sys.path.insert(0, p)

from stream_bench import card, timed  # noqa: E402

EXPORTED = {'C2': 256, 'C4': 16}          # N: frames of C2, clips of C4 (bench.py's batch sizes)


def build(name):
    from deephar_b200 import reception
    if name == 'C2':
        return reception.build((256, 256, 3), num_joints=16, dim=2, num_context_per_joint=2, num_blocks=8, ksize=(5, 5),
                               concat_pose_confidence=False).init_synthetic_weights(1234)
    from stream_bench import build as build_spnet
    return build_spnet('C4')


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--configs', nargs='+', default=['C2', 'C4'], choices=sorted(EXPORTED))
    ap.add_argument('--batches', nargs='+', type=int, default=[1, 8, 32])
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--out', default=None, help='also write the result lines to this JSON file')
    args = ap.parse_args()
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        sys.exit('model_batch_bench: no CUDA device (the numbers are GPU timings; there is nothing to measure here)')
    from deephar_b200 import _ffi
    from oracle import synth
    lib = _ffi.lib()
    rt = C.CDLL('libcudart.so.12')
    rt.cudaMemcpy.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int]
    dev = card(torch)
    print('device: %s, power limit %s W' % (dev['name'], dev['power_limit_w']))
    rows = []
    tmp = tempfile.mkdtemp(prefix='model_batch_bench_')
    for name in args.configs:
        N = EXPORTED[name]
        m = build(name)
        T = m.graph.frames_per_clip
        path = os.path.join(tmp, name + '.dhm')
        m.export(path, N * T)
        del m
        torch.cuda.empty_cache()
        ctx = _ffi.Context(torch.cuda.current_device())
        h = C.c_void_p()
        _ffi.check(lib.dh_model_load(ctx.handle, path.encode(), C.byref(h)), 'dh_model_load')
        os.remove(path)
        v = _ffi.dh_view()
        _ffi.check(lib.dh_model_input(h, C.byref(v)), 'dh_model_input')
        x = np.ascontiguousarray(synth.synth_frames(N * T, v.h, v.w, seed=7), np.float32)
        assert rt.cudaMemcpy(v.p, x.ctypes.data, x.nbytes, 1) == 0
        stream = torch.cuda.Stream()

        def ms_at(n):
            _ffi.check(lib.dh_model_set_batch(h, n), 'dh_model_set_batch')
            with torch.cuda.stream(stream):
                _ffi.check(lib.dh_model_forward(h, stream.cuda_stream), 'dh_model_forward')    # warms every kernel
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g, stream=stream):
                    _ffi.check(lib.dh_model_forward(h, stream.cuda_stream), 'dh_model_forward')
                for _ in range(args.warmup):
                    g.replay()
                best = min(timed(torch, g.replay, args.steps) for _ in range(args.rounds))
            torch.cuda.synchronize()
            del g
            return best
        padded = ms_at(N)
        for n in sorted(set(b for b in args.batches if 1 <= b <= N) | {N}):
            ms = padded if n == N else ms_at(n)
            r = {'config': name, 'exported': N, 'frames_per_clip': T, 'n': n, 'ms': round(ms, 4),
                 'padded_ms': round(padded, 4), 'padded_over_n': round(padded / ms, 2),
                 'items_per_s': round(n * 1000.0 / ms, 1), 'device': dev['name'], 'power_limit_w': dev['power_limit_w'],
                 'steps': args.steps, 'rounds': args.rounds}
            rows.append(r)
            print(json.dumps(r), flush=True)
        _ffi.check(lib.dh_model_free(h), 'dh_model_free')
        del ctx
        torch.cuda.empty_cache()
    os.rmdir(tmp)
    print('\n%-4s %4s %4s | %9s %10s %9s | %10s' % ('cfg', 'N', 'n', 'ms', 'padded ms', 'padded/n', 'items/s'))
    for r in rows:
        print('%-4s %4d %4d | %9.3f %10.3f %8.2fx | %10.1f' % (r['config'], r['exported'], r['n'], r['ms'],
                                                              r['padded_ms'], r['padded_over_n'], r['items_per_s']))
    if args.out:
        with open(args.out, 'w') as f:
            json.dump({'device': dev, 'results': rows}, f, indent=1)


if __name__ == '__main__':
    main()
