"""Frame preparation on the device (FramePipeline.from_device, dh_prepare_frames_u8) against FramePipeline.__call__, and
what it adds to a live-video push, on one GPU.

  frames   VGA (640 x 480) uint8 images -> 256 x 256 frames at batch 32 and 256, one window per image:
             call     FramePipeline.__call__ on host numpy images (host planning, packed upload, two launches)
             device   FramePipeline.from_device on the same images already in device memory (boxes from numpy)
           ms per batch, wall clock around the public call ended by a device synchronise, best of --rounds; the two
           outputs are checked bit-identical in the same run.
  push     C4 (PennAction SPNet, T = 16) at S = 8 through the C ABI (dh_stream_*): one CUDA graph of box upload +
           dh_prepare_frames_u8 + dh_stream_push against one graph of dh_stream_push alone, ms per replay from CUDA events.
Prints the card's name and power limit next to the numbers and one JSON line per measurement.

    python tools/prepare_bench.py [--batches 32 256] [--streams 8] [--steps 20] [--rounds 3] [--out results.json]
"""
import argparse
import ctypes as C
import json
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

from stream_bench import build, card  # noqa: E402

H, W, RES = 480, 640, (256, 256)


def windows(rng, n):
    pos = np.stack([320 + rng.uniform(-60, 60, n), 240 + rng.uniform(-40, 40, n)], axis=1)
    return pos, np.stack([rng.uniform(200, 460, n), rng.uniform(200, 470, n)], axis=1), rng.integers(0, 2, n)


def wall(torch, fn, steps, rounds):
    best = float('inf')
    for _ in range(rounds):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(steps):
            fn()
        torch.cuda.synchronize()
        best = min(best, (time.perf_counter() - t0) * 1000.0 / steps)
    return best


def replay_ms(torch, g, steps, rounds):
    best = float('inf')
    for _ in range(rounds):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            g.replay()
        e1.record()
        e1.synchronize()
        best = min(best, e0.elapsed_time(e1) / steps)
    return best


def frames_bench(torch, n, steps, rounds, dev):
    from deephar_b200 import preprocess
    rng = np.random.default_rng(n)
    imgs = [rng.integers(0, 256, (H, W, 3), dtype=np.uint8) for _ in range(n)]
    on_dev = [torch.from_numpy(im).cuda() for im in imgs]
    pos, win, hflip = windows(rng, n)
    pipe = preprocess.FramePipeline(RES)
    a = pipe(imgs, pos, win, hflip=hflip)[0]
    b = pipe.from_device(on_dev, pos, win, hflip=hflip)[0]
    assert torch.equal(a, b), 'from_device differs from __call__'
    call_ms = wall(torch, lambda: pipe(imgs, pos, win, hflip=hflip), steps, rounds)
    dev_ms = wall(torch, lambda: pipe.from_device(on_dev, pos, win, hflip=hflip), steps, rounds)
    return {'bench': 'frames', 'batch': n, 'image': '%dx%d' % (W, H), 'out': '%dx%d' % RES, 'call_ms': round(call_ms, 3),
            'from_device_ms': round(dev_ms, 3), 'speedup': round(call_ms / dev_ms, 2), 'device': dev['name'],
            'power_limit_w': dev['power_limit_w'], 'steps': steps, 'rounds': rounds}


def push_bench(torch, S, steps, rounds, dev):
    from deephar_b200 import _ffi
    from deephar_b200.stream import ClipStream
    lib = _ffi.lib()
    m = build('C4')
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, 'c4.dhs')
        ClipStream(m, S).export(path)
        ctx = _ffi.Context(torch.cuda.current_device())
        st = C.c_void_p()
        _ffi.check(lib.dh_stream_load(ctx.handle, path.encode(), C.byref(st)), 'dh_stream_load')
    try:
        inp = _ffi.dh_view()
        _ffi.check(lib.dh_stream_input(st, C.byref(inp)), 'dh_stream_input')
        rng = np.random.default_rng(S)
        imgs = torch.from_numpy(rng.integers(0, 256, (S, H, W, 3), dtype=np.uint8)).cuda()
        pos, win, hflip = windows(rng, S)
        rec = (_ffi.dh_frame_box * S)()
        for s in range(S):
            rec[s].data, rec[s].h, rec[s].w, rec[s].stride = imgs[s].data_ptr(), H, W, W * 3
            rec[s].hflip = int(hflip[s])
            rec[s].objpos[:], rec[s].winsize[:] = list(pos[s]), list(win[s])
        host = torch.from_numpy(np.frombuffer(rec, np.uint8).copy()).pin_memory()
        boxes = torch.empty_like(host, device='cuda')
        mc = (480, 480)
        ws_bytes = lib.dh_prepare_frames_workspace(S, mc[0], mc[1], inp.h, inp.w)
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device='cuda')
        afmat = torch.empty((S, 3, 3), dtype=torch.float64, device='cuda')
        status = torch.empty(S, dtype=torch.int32, device='cuda')

        def push():
            _ffi.check(lib.dh_stream_push(st, torch.cuda.current_stream().cuda_stream), 'dh_stream_push')

        def prepare_push():
            boxes.copy_(host, non_blocking=True)
            _ffi.check(lib.dh_prepare_frames_u8(ctx.handle, boxes.data_ptr(), S, mc[0], mc[1], inp.h, inp.w, None,
                                                ws.data_ptr(), ws_bytes, inp.p, afmat.data_ptr(), status.data_ptr(),
                                                torch.cuda.current_stream().cuda_stream), 'dh_prepare_frames_u8')
            push()
        side = torch.cuda.Stream()
        graphs = {}
        for name, fn in (('push', push), ('prepare_push', prepare_push)):
            with torch.cuda.stream(side):
                for _ in range(3):
                    fn()
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                fn()
            graphs[name] = g
        for g in graphs.values():
            for _ in range(3):
                g.replay()
        assert not status.any(), status
        t = {k: replay_ms(torch, g, steps, rounds) for k, g in graphs.items()}
    finally:
        torch.cuda.synchronize()
        lib.dh_stream_free(st)
    return {'bench': 'push', 'config': 'C4', 'streams': S, 'image': '%dx%d' % (W, H), 'push_ms': round(t['push'], 4),
            'prepare_push_ms': round(t['prepare_push'], 4), 'added_ms': round(t['prepare_push'] - t['push'], 4),
            'device': dev['name'], 'power_limit_w': dev['power_limit_w'], 'steps': steps, 'rounds': rounds}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--batches', nargs='+', type=int, default=[32, 256])
    ap.add_argument('--streams', nargs='+', type=int, default=[8])
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--out', default=None, help='also write the result lines to this JSON file')
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit('prepare_bench: no CUDA device (the numbers are GPU timings; there is nothing to measure here)')
    dev = card(torch)
    print('device: %s, power limit %s W' % (dev['name'], dev['power_limit_w']))
    rows = [frames_bench(torch, n, args.steps, args.rounds, dev) for n in args.batches]
    for r in rows:
        print(json.dumps(r), flush=True)
    for S in args.streams:
        rows.append(push_bench(torch, S, args.steps, args.rounds, dev))
        print(json.dumps(rows[-1]), flush=True)
    if args.out:
        with open(args.out, 'w') as f:
            json.dump({'device': dev, 'results': rows}, f, indent=1)


if __name__ == '__main__':
    main()
