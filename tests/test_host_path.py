"""The `-m gpu` model tests, executed on the CPU through the product's OWN host path.

tests/fake_cuda.py --arithmetic replaces the device by host memory and puts numpy arithmetic (the oracle's primitives)
behind the C entry points of the model forward, decoding the raw `dh_view` / `dh_conv_desc` / weight-pointer arguments as
the CUDA side does.  Everything above the kernels is the product's: `Model._bind` (buffer slots, channel offsets, leading
dimensions, folded BatchNormalization vectors, residual / pooled-output descriptors), `_Bound.issue`, the CUDA-graph branch
(captured calls are re-issued on replay), the copy-pipelined `predict`, `load_weights`, `split_model` views, the
keras_compat front end.  The unchanged GPU tests then hold at their GPU tolerances: ReceptionNet 2-D / 3-D vs the oracle,
SPNet and merge-model parity, CUDA-graph replay == plain launches, predict edge cases, Keras-HDF5-driven forward, and the
reference-builder goldens (C1 / C3 at full size, C4 at full resolution with 2 frames, the merge models).  Deselected: tests that read kernel-internal counters
(`dh_fallback_count`), the 64-forward batch-independence test (CPU time), and the direct C-ABI op tests (test_gpu_ops /
test_gpu_tc: they test the kernels themselves, which only a GPU can).  The input-pipeline and evaluator entry points have
stand-ins too (the oracle's Pillow-exact resampler and PCKh arithmetic behind `dh_crop_resize_norm_u8` / `dh_pose_eval_f64`),
so their GPU tests and `__graft_entry__.smoke()` -- the first thing the driver runs on the GPU box -- go through
FramePipeline's planning / packing and postprocess' argument marshalling as well."""
import os
import re
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.timeout(900)
def test_gpu_model_tests_hold_on_the_cpu_through_the_products_host_path():
    files = ['tests/test_reference_golden.py', 'tests/test_gpu_reception.py', 'tests/test_gpu_spnet.py',
             'tests/test_merge_model.py', 'tests/test_keras_compat.py', 'tests/test_gpu_model.py',
             'tests/test_postprocess.py', 'tests/test_preprocess.py']
    cmd = [sys.executable, os.path.join(ROOT, 'tests', 'fake_cuda.py'), '--arithmetic', '-m', 'pytest'] + files + [
        '-m', 'gpu', '-q', '-p', 'no:cacheprovider',
        '--deselect', 'tests/test_gpu_model.py::test_no_unexpected_cuda_core_fallback',
        '--deselect', 'tests/test_gpu_reception.py::test_c2_batch32_equals_32_single_frame_calls',
        # the two 16-frame full-size SPNet goldens: CPU time (their plans are executed by test_compiled_plan_matches_...)
        '--deselect', 'tests/test_reference_golden.py::test_product_matches_reference_graph[spnet_penn_c4_t16]',
        '--deselect', 'tests/test_reference_golden.py::test_product_matches_reference_graph[spnet_ntu_c5_t16]']
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=880, cwd=ROOT)
    tail = out.stdout[-3000:]
    assert out.returncode == 0, tail + out.stderr[-2000:]
    m = re.search(r'(\d+) passed', tail)
    assert m and int(m.group(1)) >= 30 and 'failed' not in tail and 'skipped' not in tail.split('\n')[-2], tail


@pytest.mark.timeout(300)
def test_smoke_entry_point_through_the_host_path():
    out = subprocess.run([sys.executable, os.path.join(ROOT, 'tests', 'fake_cuda.py'), '--arithmetic',
                          os.path.join(ROOT, '__graft_entry__.py'), 'smoke'], capture_output=True, text=True, timeout=280, cwd=ROOT)
    assert out.returncode == 0, out.stdout[-1500:] + out.stderr[-1500:]
    assert 'smoke ok: input pipeline bit-exact' in out.stdout


@pytest.mark.timeout(300)
@pytest.mark.parametrize('world,n_clips', [(2, 5), (4, 3)])
def test_sharded_forward_and_exchange_through_the_c_abi(world, n_clips):
    """SURVEY 8e on the stand-in device: every rank runs the product's forward on its contiguous shard (ragged shards; with
    4 ranks and 3 clips one rank holds nothing) and the outputs are exchanged with dist.Comm -- dh_comm_unique_id /
    dh_comm_init / dh_allgather_f32 through the ctypes binding, gloo standing in for NCCL -- into the whole batch's
    result, in clip order, equal to the oracle's forward of the unsharded batch."""
    import json
    import socket
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    port = s.getsockname()[1]
    s.close()
    env = {k: v for k, v in os.environ.items() if k not in ('RANK', 'WORLD_SIZE', 'LOCAL_RANK')}
    out = subprocess.run([sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node', str(world),
                          '--master-addr', '127.0.0.1', '--master-port', str(port), os.path.join(ROOT, 'tests', 'fake_cuda.py'),
                          '--arithmetic', os.path.join(ROOT, 'tests', 'run_sharded_forward.py'), str(n_clips)],
                         capture_output=True, text=True, timeout=280, cwd=ROOT, env=env)
    assert out.returncode == 0, out.stderr[-3000:]
    got = json.loads([l for l in out.stdout.splitlines() if l.startswith('{')][-1])
    assert got['world'] == world and got['shape'] == [n_clips, 6, 15] and got['pose_shape'] == [n_clips, 4 * 16 * 3]
    assert got['max_err'] <= 1e-3 and got['pose_max_err'] <= 1e-3 and got['argmax_equal']

