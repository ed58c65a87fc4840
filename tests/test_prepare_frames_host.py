"""FramePipeline.from_device and the two entry points behind it, without a GPU: the frame preparation runs on the
stand-in device (tests/fake_cuda.py with arithmetic, and the contracts and stand-ins of tests/prepare_contracts.py), so
what is checked here is the product's host side -- the dh_frame_box records it packs (image pointers, row strides, objpos / winsize / hflip
broadcast from numpy or from device tensors), the workspace it sizes, the default max_crop and the status / NaN of
flagged frames.  The struct mirror and the workspace size are checked against the real library."""
import ctypes as C
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _images(rng, shapes):
    return [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for h, w in shapes]


def _scenario(name):
    import torch

    from deephar_b200 import _ffi, postprocess, preprocess
    rng = np.random.default_rng(7)
    pipe = preprocess.FramePipeline((24, 20))                                   # (w, h)
    shapes = [(40, 50), (33, 17), (60, 64), (5, 7), (40, 50)]
    imgs = _images(rng, shapes)
    objpos = np.array([[25.3, 20.1], [8.0, 16.5], [70.2, -3.9], [3.5, 2.5], [0.4, 0.6]])
    winsize = np.array([[30.7, 41.2], [17.0, 33.0], [44.0, 20.5], [1.2, 1.0], [130.0, 121.0]])
    hflip = np.array([0, 1, 0, 1, 2])                                           # 2: no flip, as in __call__
    want, want_a = pipe(imgs, objpos, winsize, hflip=hflip, channel_power=(1.0, 1.5, 0.7))
    want = want.numpy()
    dev = [torch.from_numpy(im).cuda() for im in imgs]
    if name == 'host_boxes':
        frames, afmat, status = pipe.from_device(dev, objpos, winsize, hflip=hflip, channel_power=(1.0, 1.5, 0.7))
        assert pipe.launches == 2 + 3                                           # __call__'s two, from_device's three
    elif name == 'device_boxes':
        frames, afmat, status = pipe.from_device(dev, torch.from_numpy(objpos).cuda(), torch.from_numpy(winsize).cuda(),
                                                 hflip=torch.from_numpy(hflip).cuda(), channel_power=(1.0, 1.5, 0.7),
                                                 max_crop=(130, 121))
    elif name == 'padded_rows':                                                  # images viewed out of wider rows
        wide = [torch.from_numpy(np.ascontiguousarray(np.pad(im, ((0, 0), (0, 9), (0, 0))))).cuda() for im in imgs]
        dev = [w[:, :im.shape[1]] for w, im in zip(wide, imgs)]
        assert dev[0].stride(0) == 3 * (imgs[0].shape[1] + 9)
        frames, afmat, status = pipe.from_device(dev, objpos, winsize, hflip=hflip, channel_power=(1.0, 1.5, 0.7))
    elif name == 'scalar_window':
        want, want_a = pipe(imgs, objpos, 31.5, hflip=1)
        frames, afmat, status = pipe.from_device(dev, objpos, 31.5, hflip=1)
        want = want.numpy()
    elif name == 'flagged':
        bad_pos = objpos.copy()
        bad_win = winsize.copy()
        bad_pos[1], bad_win[1] = [8.5, 16.5], [0.5, 40.0]                       # 8.25 .. 8.75: cw = 0, empty
        bad_pos[2] = [np.nan, 3.0]                                              # not finite
        bad_win[3] = [np.inf, 1.0]
        bad_pos[0] = [3e9, 5.0]                                                 # an edge outside int32
        frames, afmat, status = pipe.from_device(dev, bad_pos, bad_win, hflip=hflip, channel_power=(1.0, 1.5, 0.7),
                                                 max_crop=(128, 120))           # frame 4 is 129 x 120: too large
        E, L, B = _ffi.FRAME_EMPTY, _ffi.FRAME_TOO_LARGE, _ffi.FRAME_BAD_BOX
        assert status.numpy().tolist() == [B, E, B, B, L], status
        assert np.isnan(frames.numpy()).all() and np.isnan(afmat.numpy()).all()
        # the same call with one good frame among them: only it has numbers, and they are __call__'s
        bad_pos[2] = objpos[2]
        frames, afmat, status = pipe.from_device(dev, bad_pos, bad_win, hflip=hflip, channel_power=(1.0, 1.5, 0.7),
                                                 max_crop=(128, 120))
        assert status.numpy().tolist() == [B, E, 0, B, L], status
        assert np.array_equal(frames.numpy()[2], want[2]) and np.array_equal(afmat.numpy()[2], want_a[2])
        assert np.isnan(np.delete(frames.numpy(), 2, axis=0)).all()
        # a window exactly max_crop wide and high is accepted
        box = preprocess.crop_box(objpos[4], winsize[4])
        assert (box[2] - box[0], box[3] - box[1]) == (129, 120)
        frames, afmat, status = pipe.from_device(dev, objpos, winsize, hflip=hflip, channel_power=(1.0, 1.5, 0.7),
                                                 max_crop=(129, 120))
        assert status.numpy().tolist() == [0] * 5
        assert np.array_equal(frames.numpy(), want)
        # FramePipeline raises where the device flags
        with pytest.raises(ValueError, match='empty crop window'):
            pipe(imgs, bad_pos, bad_win)
        return
    elif name == 'pose_to_image':
        n, nj = 5, 4
        poses = rng.uniform(-0.2, 1.2, (n, nj, 3)).astype(np.float32)
        buf = torch.full((n, nj, 5), -7.0)
        buf[:, :, 1:4] = torch.from_numpy(poses)                               # a channel window: ld 5, c 3
        v = _ffi.dh_view(buf.data_ptr() + 4, n, 1, nj, 3, 5)
        A = want_a.copy()
        A[3] = [[1, 2, 0], [2, 4, 0], [0, 0, 1]]                                # singular
        a = torch.from_numpy(A).cuda()
        out = torch.empty(n, nj, 2, dtype=torch.float64)
        ctx = _ffi.Context(0)
        _ffi.check(_ffi.lib().dh_pose_to_image_f32(ctx.handle, C.byref(v), a.data_ptr(), 1, out.data_ptr(), None), 'p2i')
        ref = postprocess.transform_pose_sequence(np.delete(A, 3, axis=0), np.delete(poses, 3, axis=0).astype(np.float64))
        got = out.numpy()
        assert np.array_equal(np.delete(got, 3, axis=0), ref) and np.isnan(got[3]).all()
        _ffi.check(_ffi.lib().dh_pose_to_image_f32(ctx.handle, C.byref(v), a.data_ptr(), 0, out.data_ptr(), None), 'p2i')
        assert np.array_equal(out.numpy(), postprocess.transform_pose_sequence(A[0], poses.astype(np.float64)))
        return
    else:
        raise AssertionError(name)
    assert status.numpy().tolist() == [0] * len(imgs), status
    assert frames.shape == want.shape and np.array_equal(frames.numpy(), want)
    assert afmat.dtype == torch.float64 and np.array_equal(afmat.numpy(), want_a)
    for i in range(len(imgs)):
        box = preprocess.crop_box(objpos[i], winsize[i] if name != 'scalar_window' else 31.5)
        assert np.array_equal(afmat.numpy()[i], preprocess.affine_map(box, (24, 20), (hflip if name != 'scalar_window'
                                                                                     else [1] * 5)[i] == 1))


@pytest.mark.parametrize('name', ['host_boxes', 'device_boxes', 'padded_rows', 'scalar_window', 'flagged',
                                  'pose_to_image'])
def test_from_device_on_the_stand_in_device(name):
    out = subprocess.run([sys.executable, os.path.abspath(__file__), name], capture_output=True, text=True, timeout=600,
                         cwd=ROOT)
    assert out.returncode == 0 and out.stdout.strip().endswith('ok'), out.stdout[-2000:] + out.stderr[-3000:]


def test_frame_box_struct_matches_the_header():
    from deephar_b200 import _ffi
    gcc = shutil.which('gcc')
    if gcc is None:
        pytest.skip('no gcc')
    with tempfile.TemporaryDirectory() as d:
        src = os.path.join(d, 's.c')
        open(src, 'w').write('#include <stdio.h>\n#include <stddef.h>\n#include "deephar_b200.h"\nint main(void) { '
                             'printf("%zu %zu %zu %zu\\n", sizeof(dh_frame_box), offsetof(dh_frame_box, hflip), '
                             'offsetof(dh_frame_box, objpos), offsetof(dh_frame_box, winsize)); return 0; }\n')
        exe = os.path.join(d, 's')
        subprocess.check_call([gcc, '-std=c99', '-I', os.path.join(ROOT, 'include'), src, '-o', exe])
        got = [int(v) for v in subprocess.check_output([exe]).split()]
    B = _ffi.dh_frame_box
    assert got == [C.sizeof(B), B.hflip.offset, B.objpos.offset, B.winsize.offset]


def _layout(n, mw, mh, oh, ow):
    """the header's workspace layout, restated"""
    def taps(i, o):
        return int(np.ceil(max(i / o, 1.0))) * 2 + 1

    def up(v, a):
        return -(-v // a) * a
    kx, ky = taps(mw, ow), taps(mh, oh)
    B = up(64 * n, 256)
    K = up(B + 8 * n * (ow + oh), 256)
    X = up(K + 4 * n * (ow * kx + oh * ky), 256)
    return X + n * up(mh * ow * 3, 16)


@pytest.mark.parametrize('sizes', [(1, 1, 1, 1, 1), (3, 1100, 700, 256, 256), (65535, 9, 9, 8, 8), (7, 4000, 1920, 8, 8),
                                   (2600, 1100, 1100, 256, 256), (0, 5, 5, 4, 4)])
def test_workspace_size_is_the_documented_layout(sizes):
    from deephar_b200 import _ffi
    assert _ffi.lib().dh_prepare_frames_workspace(*sizes) == _layout(*sizes)


@pytest.mark.parametrize('sizes', [(-1, 5, 5, 4, 4), (65536, 5, 5, 4, 4), (1, 0, 5, 4, 4), (1, 5, 5, 0, 4),
                                   (1, 1 << 18 | 1, 5, 4, 4), (65535, 262144, 262144, 262144, 262144)])
def test_workspace_refuses_sizes(sizes):
    from deephar_b200 import _ffi
    assert _ffi.lib().dh_prepare_frames_workspace(*sizes) < 0
    assert b'dh_prepare_frames' in _ffi.lib().dh_last_error()


if __name__ == '__main__':
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, 'tests'))
    import prepare_contracts
    prepare_contracts.install()
    _scenario(sys.argv[1])
    print('ok')
