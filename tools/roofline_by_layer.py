"""Per-layer roofline accounting of one forward: joins a measured per-op profile (tools/profile_model.py output,
CUDA events around every launch, committed under profiles/) with the ALGORITHMIC work of each launch derived from the
compiled plan on the CPU -- bytes every operand is read / written exactly once (fp32 activations, residuals, pooled
second outputs, weights once per launch) and 2 x MAC flops -- and prints, per layer shape, the time the binding roofline
would allow and the fraction of it that was achieved.  No GPU needed: the timings are the committed measurements.

    python tools/roofline_by_layer.py reception2d profiles/h100_prof_reception2d.txt

Peaks: the H100 SXM data sheet (HBM3 3350 GB/s, dense bf16 989 TFLOP/s at 700 W), or PEAK_HBM_GBS / PEAK_BF16_TFLOPS.
The tensor floor is quoted twice: for the algorithmic flops, and x3 for what the bf16x3 (fp32-accurate) split executes.
"""
import os
import re
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

HBM_GBS = float(os.environ.get('PEAK_HBM_GBS', 3350.0))
BF16_TFLOPS = float(os.environ.get('PEAK_BF16_TFLOPS', 989.0))


def build(name):
    import bench
    model, clip_model, _ = bench.build_workload(name)
    return model, clip_model


def label_of(k):
    """The label Model.profile() gives a launch (deephar_b200/model.py)."""
    label = '%s %s->%s' % (k.kind, 'x'.join(map(str, k.ins[0].shape)), 'x'.join(map(str, k.outs[0].shape)))
    if k.kind in ('conv', 'sepconv'):
        label += ' k%dx%d' % tuple(k.attrs['size'])
    return label


def work_of(k, n_frames, frames_per_clip):
    """(algorithmic bytes, flops) of one launch at n_frames."""
    def items(t):
        return n_frames if t.kind == 'frame' else n_frames // frames_per_clip

    def numel(t):
        return items(t) * t.shape[0] * t.shape[1] * t.shape[2]

    nbytes = 4.0 * (sum(numel(t) for t in k.ins) + sum(numel(t) for t in k.outs))
    flops = 0.0
    if k.kind in ('conv', 'sepconv'):
        ho, wo, cout = k.outs[0].shape
        cin = k.ins[0].shape[2]
        kh, kw = k.attrs['size']
        mac = kh * kw * cin * cout if k.kind == 'conv' else kh * kw * cin + cin * cout
        nbytes += 4.0 * mac                                          # the weights, once per launch
        flops = 2.0 * mac * ho * wo * items(k.outs[0])
    return nbytes, flops


def main():
    name, path = sys.argv[1], sys.argv[2]
    head = open(path).readline()
    n_frames = int(re.search(r'N=(\d+)', head).group(1))
    measured = {}
    for line in open(path).read().splitlines()[1:]:
        m = re.match(r'^(.*?)\s+([\d.]+) ms\s+([\d.]+)%\s+x(\d+)', line)
        if m:
            measured[m.group(1).strip()] = (float(m.group(2)), int(m.group(4)))
    model, _ = build(name)
    T = model.graph.frames_per_clip
    rows = {}
    for k in model.plan.kops:
        r = rows.setdefault(label_of(k), {'bytes': 0.0, 'flops': 0.0, 'n': 0})
        b, f = work_of(k, n_frames, T)
        r['bytes'] += b
        r['flops'] += f
        r['n'] += 1
    missing = [l for l in rows if l not in measured]
    if missing or any(measured[l][1] != rows[l]['n'] for l in rows):
        raise SystemExit('profile %s does not match the plan of %s (labels %s)' % (path, name, missing[:3]))

    print('%s  N=%d frames  one forward = %d launches; measured (CUDA events) vs the roofline floor of the algorithmic work'
          % (name, n_frames, len(model.plan.kops)))
    print('peaks: HBM %.1f GB/s, bf16 dense %.1f TFLOP/s sustained; floor = max(bytes / HBM, 3 x flops / bf16) per launch '
          '(x3: the bf16x3 split the fp32-accurate convs execute)' % (HBM_GBS, BF16_TFLOPS))
    print('frac alg = max(hbm us, tc us) / measured: the ALGORITHMIC roofline fraction (bench.py\'s roofline.frac); '
          'frac x3 = max(hbm us, tc x3 us) / measured')
    print('%-52s %4s %9s %8s %8s %9s %9s %9s %8s %7s %s' % ('layer', 'x', 'meas ms', 'GB', 'GFLOP', 'hbm us', 'tc us', 'tc x3 us',
                                                           'frac alg', 'frac x3', 'bound'))
    tot = {'ms': 0.0, 'floor': 0.0, 'alg': 0.0, 'hbm': 0.0, 'tc3': 0.0, 'bytes': 0.0, 'flops': 0.0}
    for label, r in sorted(rows.items(), key=lambda kv: -measured[kv[0]][0]):
        ms = measured[label][0]
        hbm_us = r['bytes'] / (HBM_GBS * 1e9) * 1e6
        tc_us = r['flops'] / (BF16_TFLOPS * 1e12) * 1e6
        floor_us = max(hbm_us, 3 * tc_us)
        print('%-52s %4d %9.3f %8.3f %8.1f %9.1f %9.1f %9.1f %8.2f %7.2f %s'
              % (label, r['n'], ms, r['bytes'] / 1e9, r['flops'] / 1e9, hbm_us, tc_us, 3 * tc_us,
                 max(hbm_us, tc_us) / (ms * 1e3), floor_us / (ms * 1e3), 'hbm' if hbm_us >= 3 * tc_us else 'tensor'))
        tot['ms'] += ms
        tot['floor'] += floor_us
        tot['alg'] += max(hbm_us, tc_us)
        tot['hbm'] += hbm_us
        tot['tc3'] += 3 * tc_us
        tot['bytes'] += r['bytes']
        tot['flops'] += r['flops']
    print('%-52s %4d %9.3f %8.3f %8.1f %9.1f %9.1f %9.1f %8.2f %7.2f' % (
        'TOTAL', len(model.plan.kops), tot['ms'], tot['bytes'] / 1e9, tot['flops'] / 1e9, tot['hbm'], tot['tc3'] / 3, tot['tc3'],
        tot['alg'] / (tot['ms'] * 1e3), tot['floor'] / (tot['ms'] * 1e3)))
    print('per frame: measured %.1f us; sum of per-launch floors %.1f us algorithmic, %.1f us with the x3 split; %.1f MB of '
          'operand traffic and %.2f GFLOP per frame as launched (i.e. with the fusions of this plan)'
          % (tot['ms'] * 1e3 / n_frames, tot['alg'] / n_frames, tot['floor'] / n_frames, tot['bytes'] / n_frames / 1e6,
             tot['flops'] / n_frames / 1e9))


if __name__ == '__main__':
    main()
