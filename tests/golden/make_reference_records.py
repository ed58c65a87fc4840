"""Regenerates tests/golden/reference_records.json.gz: what the reference's own builder code records on the product's
recording keras (tests/reference_dropin/run_reference_backbone.py, one run per case), stored so that
tests/test_keras_compat.py compares the product's builders with it without the reference tree.

    DEEPHAR_REFERENCE=<reference checkout> python tests/golden/make_reference_records.py
"""
import gzip
import json
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
RUNNER = os.path.join(os.path.dirname(HERE), 'reference_dropin', 'run_reference_backbone.py')
OUT = os.path.join(HERE, 'reference_records.json.gz')

# case name -> run_reference_backbone.py arguments
CASES = {
    'backbone3': ['3'],
    'spnet': ['spnet'],
    'full2d_0': ['full2d', '0'],
    'full2d_1': ['full2d', '1'],
    'full3d': ['full3d'],
    'spnet_full_penn': ['spnet_full', 'penn'],
    'spnet_full_ntu': ['spnet_full', 'ntu'],
    'merge_2_v1': ['merge', '2', 'v1'],
    'merge_3_v1': ['merge', '3', 'v1'],
    'merge_2_v2': ['merge', '2', 'v2'],
    'sweep': ['sweep'],
}


def main():
    records = {}
    for name, args in CASES.items():
        out = subprocess.run([sys.executable, RUNNER] + args, capture_output=True, text=True, timeout=1800, check=True)
        records[name] = [json.loads(l) for l in out.stdout.splitlines() if l.startswith('{')]
        print(name, len(records[name]))
    with gzip.GzipFile(OUT, 'wb', mtime=0) as f:
        f.write(json.dumps(records, sort_keys=True).encode())


if __name__ == '__main__':
    main()
