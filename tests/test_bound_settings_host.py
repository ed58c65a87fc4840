"""What a bound plan records, checked without a GPU on the stand-in device (tests/fake_cuda.py).  A forward runs the
`precision` and `use_tensor_cores` the model has when it is called, also at a batch size bound under other settings:
the launches, math_mode() and an export all agree with what runs.  Assigning a setting its current value keeps the
bindings and their CUDA graphs; a ClipStream keeps the settings it was built with.  launches_per_forward and
launches_per_push count what the library's plans launch: a separable conv on the CUDA-core path (0) is two kernels."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _conv_records(launches):
    """(dh_conv_desc, dh_packed_w list) of every conv / sepconv launch of a file read back by export.read"""
    out = []
    for launch in launches:
        args = dict((tag, v) for tag, v in launch['args'] if tag in 'dw')
        if 'd' in args:
            out.append((args['d'][0], args['w']))
    return out


def _bound_precisions(b):
    return set(call[-2]._obj.precision for call in b.calls if call[0] in ('conv', 'sepconv'))


def _scenario(name, tmp):
    import torch

    from deephar_b200 import export, reception
    from deephar_b200.stream import ClipStream
    from test_stream_export_host import _target
    m = reception.build((64, 64, 3), 16, dim=2, num_blocks=1).init_synthetic_weights(1)
    x = torch.zeros(2, 64, 64, 3, device='cuda')
    path = os.path.join(tmp, name + '.dhm')
    if name == 'precision':
        m.forward_device(x)
        m.precision = 1
        m.forward_device(x)
        assert _bound_precisions(m._bind(2)) == {1} and m.math_mode() == 'bf16'
        m.export(path, 2)
        rec = export.read(path)
        convs = _conv_records(rec['launches'])
        assert rec['precision'] == 1 and convs and all(d['precision'] == 1 for d, _ in convs)
        assert rec['use_tensor_cores'] == 1 and all(len(w) == 1 for _, w in convs)
    elif name == 'cuda_cores':
        m.forward_device(x)
        m.use_tensor_cores = False
        m.forward_device(x)
        assert m.math_mode() == 'f32' and not m._uses_tc()
        m.export(path, 2)
        rec = export.read(path)
        convs = _conv_records(rec['launches'])
        assert convs and all(w == [] for _, w in convs)
        assert rec['use_tensor_cores'] == 0 and rec['packed'] == b''
        m.use_tensor_cores = True                   # and back: the packed operands are passed again
        m.forward_device(x)
        assert all(call[5] for call in m._bind(2).calls if call[0] == 'conv') and m._uses_tc()
    elif name == 'same_value':
        m.max_bound = 2
        for n in (2, 3):
            for _ in range(3):                      # plain launches, capture, replay
                m.forward_device(torch.zeros(n, 64, 64, 3, device='cuda'))
        bound = dict(m._bound)
        graphs = [b.graph for b in bound.values()]
        assert all(g is not None for g in graphs)
        m.precision, m.use_tensor_cores = 3, True
        m.forward_device(x)
        assert m._bound.keys() == bound.keys() and all(m._bound[n] is b for n, b in bound.items())
        assert [b.graph for b in bound.values()] == graphs
    elif name == 'stream':
        _, sm = _target('spnet_t2')
        cs = ClipStream(sm, 3)
        sm.precision, sm.use_tensor_cores = 1, False
        cs.push(torch.zeros((3,) + tuple(sm.graph.inputs[0].shape), device='cuda'))
        cs.export(path)
        rec = export.read_stream(path)
        assert rec['precision'] == 3 and rec['use_tensor_cores'] == 1 and rec['packed']
        for launches in (rec['frame_launches'], rec['clip_launches']):
            assert all(d['precision'] == 3 for d, _ in _conv_records(launches))
        assert _bound_precisions(cs._frame) == _bound_precisions(cs._clip) == {3}
    elif name == 'launch_counts':
        def simt_sep(b):
            return sum(1 for k, info in b.conv_plans if k.kind == 'sepconv' and info.path == 0)
        b = m._bind(2)
        assert simt_sep(b) > 0                      # the stand-in's plans report path 0 for every conv
        assert m.launches_per_forward(2) == len(b.calls) + simt_sep(b)
        _, sm = _target('spnet_t2')
        cs = ClipStream(sm, 3)
        assert cs.launches_per_push() == len(cs._frame.calls) + len(cs._clip.calls) + 1 + \
            simt_sep(cs._frame) + simt_sep(cs._clip)
        sm.launch_total = 0
        sm.forward_device(torch.zeros((2,) + tuple(sm.input_shape[1:]), device='cuda'))
        assert sm.launch_total == sm.launches_per_forward(4)
    else:
        raise AssertionError(name)


@pytest.mark.parametrize('name', ['precision', 'cuda_cores', 'same_value', 'stream', 'launch_counts'])
def test_bound_settings(name, tmp_path):
    out = subprocess.run([sys.executable, os.path.abspath(__file__), name, str(tmp_path)], capture_output=True,
                         text=True, timeout=600, cwd=ROOT)
    assert out.returncode == 0 and out.stdout.strip().endswith('ok'), out.stdout[-2000:] + out.stderr[-3000:]


if __name__ == '__main__':
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, 'tests'))
    import fake_cuda
    fake_cuda.install()
    _scenario(sys.argv[1], sys.argv[2])
    print('ok')
