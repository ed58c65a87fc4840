"""JPEG files -> network input frames: `ImageDecoder` (Pillow on every host core) + `FramePipeline` against
`FramePipeline.from_jpeg` (GPU decode), wall clock around each public call ended by a device synchronise, outputs
checked bit-identical in the same run.  Seeded synthetic 4:2:0 quality-90 files (smooth natural-like content and a
noise worst case) at VGA and 1080p, batches of 32 and 256; also CUDA-event times of the three decode stages,
compressed bytes per image, host core count, card name and power limit.

    python tools/jpeg_bench.py [--batches 32 256] [--reps 5] [--out jpeg_bench.json]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

SIZES = {'vga': (480, 640), '1080p': (1080, 1920)}


def synth(h, w, seed, content):
    rng = np.random.default_rng(seed)
    if content == 'noise':
        return rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    y, x = np.mgrid[0:h, 0:w].astype(np.float32)
    ph = rng.uniform(0, 6.3, 6)
    a = np.stack([128 + 60 * np.sin(x / (23 + 9 * k) + ph[k]) * np.cos(y / (31 + 7 * k) + ph[k + 3])
                  + 30 * np.sin((x + y) / (11 + 3 * k)) for k in range(3)], -1)
    return np.clip(a + rng.normal(0, 4, a.shape), 0, 255).astype(np.uint8)


def card():
    try:
        out = subprocess.check_output(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                                      text=True).strip().splitlines()[0]
        name, limit = [s.strip() for s in out.split(',')]
        return name, limit
    except Exception as e:                  # noqa: BLE001 -- reported, not fatal
        return 'unknown (%s)' % e, 'unknown'


def timed(fn, torch, reps):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts)), ts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batches', type=int, nargs='+', default=[32, 256])
    ap.add_argument('--sizes', nargs='+', default=['vga', '1080p'])
    ap.add_argument('--contents', nargs='+', default=['smooth', 'noise'])
    ap.add_argument('--distinct', type=int, default=16, help='distinct files per configuration (cycled)')
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('jpeg_bench: needs a CUDA device')
    from PIL import Image
    from deephar_b200 import jpeg, preprocess
    name, limit = card()
    cores = os.cpu_count()
    rows = []
    decoder = preprocess.ImageDecoder(workers=cores, arena_mb=2048)
    pipe = preprocess.FramePipeline((256, 256))
    with tempfile.TemporaryDirectory() as tmp:
        for size in args.sizes:
            h, w = SIZES[size]
            for content in args.contents:
                files = []
                for s in range(args.distinct):
                    p = os.path.join(tmp, '%s_%s_%d.jpg' % (size, content, s))
                    Image.fromarray(synth(h, w, s, content)).save(p, quality=90, subsampling=2)
                    files.append(p)
                nbytes = float(np.mean([os.path.getsize(p) for p in files]))
                for batch in args.batches:
                    paths = [files[k % len(files)] for k in range(batch)]
                    objpos = np.tile([[w / 2.0, h / 2.0]], (batch, 1))
                    win = 0.8 * min(h, w)
                    res = {}
                    t_cpu, _ = timed(lambda: res.__setitem__('cpu', pipe(decoder(paths), objpos, win)), torch, args.reps)
                    t_gpu, _ = timed(lambda: res.__setitem__('gpu', pipe.from_jpeg(paths, objpos, win)), torch, args.reps)
                    same = (torch.equal(res['cpu'][0], res['gpu'][0]) and np.array_equal(res['cpu'][1], res['gpu'][1]))
                    dec = pipe._jpeg
                    dec.time_stages = True
                    dec(paths)
                    stage_ms = dict(dec.stage_ms)
                    dec.time_stages = False
                    row = dict(size=size, content=content, batch=batch, bytes_per_image=round(nbytes),
                               cpu_decode_pipeline_s=t_cpu, gpu_from_jpeg_s=t_gpu,
                               cpu_frames_per_s=batch / t_cpu, gpu_frames_per_s=batch / t_gpu,
                               speedup=t_cpu / t_gpu, stage_ms=stage_ms, host_decoded=len(dec.host_decoded),
                               bit_identical=bool(same))
                    rows.append(row)
                    print(json.dumps(row), flush=True)
    decoder.close()
    out = dict(card=name, power_limit=limit, host_cores=cores, reps=args.reps, rows=rows)
    print(json.dumps(dict(card=name, power_limit=limit, host_cores=cores)))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            json.dump(out, f, indent=1)
    if not all(r['bit_identical'] for r in rows):
        raise SystemExit('jpeg_bench: outputs differ')


if __name__ == '__main__':
    main()
