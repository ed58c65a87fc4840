"""Frames prepared on the device (dh_prepare_frames_u8, through FramePipeline.from_device and directly) and poses mapped
back to image pixels (dh_pose_to_image_f32).

The tables the geometry kernel writes, read back from the workspace at the offsets the header documents, equal
preprocess.resample_tables bit for bit for every crop size 1 ... 1100 -> 256 and -> 64, and 1920 / 4000 -> 8.  The frames
equal FramePipeline.__call__ (itself pinned to the oracle and Pillow) on test_gpu_pre_post's seeded sweep and named
edges, at a scratch past 2^31 bytes and at 65 535 frames; on jpeg.decode's images they equal from_jpeg.  afmat equals
preprocess.affine_map as values.  Each status case flags its frame and writes NaN there, and leaves its neighbours bit
for bit as a run without it.  The pose mapping equals dh_pose_eval_f64 on the widened poses bit for bit.
examples/run_camera.c, plain and graph-replayed, writes what from_device -> ClipStream.push -> transform_pose_sequence
computes in Python.
"""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

from deephar_b200 import _ffi, postprocess, preprocess
from test_gpu_pre_post import EDGES, SWEEP_RES, _decoded, _image, _jpeg, _window

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _dev(cuda, imgs):
    return [cuda.from_numpy(np.ascontiguousarray(im)).cuda() for im in imgs]


def _pairs(wins):
    return [(w, w) if np.isscalar(w) else w for w in wins]


def _prepare(cuda, imgs, objpos, winsize, hflip, res, max_crop, ws_extra=0):
    """dh_prepare_frames_u8 called directly -> (frames, afmat, status, workspace bytes on the host, rc)"""
    torch = cuda
    n = len(imgs)
    rw, rh = res
    lib = _ffi.lib()
    ctx = _ffi.Context(torch.cuda.current_device())
    rec = (_ffi.dh_frame_box * n)()
    for i, im in enumerate(imgs):
        rec[i].data, rec[i].h, rec[i].w, rec[i].stride = im.data_ptr(), im.shape[0], im.shape[1], im.stride(0)
        rec[i].hflip = int(hflip[i] == 1)
        rec[i].objpos[:] = [float(v) for v in objpos[i]]
        rec[i].winsize[:] = [float(v) for v in winsize[i]]
    boxes = torch.from_numpy(np.frombuffer(rec, np.uint8).copy()).cuda()
    need = lib.dh_prepare_frames_workspace(n, max_crop[0], max_crop[1], rh, rw)
    assert need > 0
    ws = torch.empty(need + max(ws_extra, 0), dtype=torch.uint8, device='cuda')
    out = torch.full((n, rh, rw, 3), 7.0, device='cuda')
    afmat = torch.zeros((n, 3, 3), dtype=torch.float64, device='cuda')
    status = torch.full((n,), -1, dtype=torch.int32, device='cuda')
    rc = lib.dh_prepare_frames_u8(ctx.handle, boxes.data_ptr(), n, max_crop[0], max_crop[1], rh, rw, None, ws.data_ptr(),
                                  need + ws_extra, out.data_ptr(), afmat.data_ptr(), status.data_ptr(),
                                  torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return out, afmat, status, ws, rc, ctx


# ---- tables --------------------------------------------------------------------------------------------------------------

def _tables(ws, n, res, max_crop):
    """frame i's (x bounds, x coefs, y bounds, y coefs) at the header's documented offsets"""
    rw, rh = res

    def taps(i, o):
        return int(np.ceil(max(i / o, 1.0))) * 2 + 1

    def up(v, a):
        return -(-v // a) * a
    kx, ky = taps(max_crop[0], rw), taps(max_crop[1], rh)
    raw = ws.cpu().numpy()
    frames = (_ffi.dh_frame_src * n).from_buffer_copy(raw[:C.sizeof(_ffi.dh_frame_src) * n].tobytes())
    B = up(64 * n, 256)
    K = up(B + 8 * n * (rw + rh), 256)
    bounds = raw[B:B + 8 * n * (rw + rh)].view(np.int32)
    coefs = raw[K:K + 4 * n * (rw * kx + rh * ky)].view(np.int32)
    out = []
    for i in range(n):
        f = frames[i]
        b0, c0 = i * 2 * (rw + rh), i * (rw * kx + rh * ky)
        assert (f.kx_off, f.ky_off, f.kx_coef_off, f.ky_coef_off) == (b0, b0 + 2 * rw, c0, c0 + rw * kx)
        out.append((bounds[b0:b0 + 2 * rw].reshape(rw, 2), coefs[c0:c0 + rw * f.ksx].reshape(rw, f.ksx),
                    bounds[b0 + 2 * rw:b0 + 2 * rw + 2 * rh].reshape(rh, 2),
                    coefs[c0 + rw * kx:c0 + rw * kx + rh * f.ksy].reshape(rh, f.ksy)))
    return out


@pytest.mark.parametrize('res,sizes', [((256, 64), list(range(1, 1101))), ((8, 8), [1920, 4000])],
                         ids=['1_to_1100', 'full_hd_and_4k_to_8'])
def test_tables_equal_resample_tables(cuda, res, sizes):
    """crop k x k for every k: the x tables are k -> res[0], the y tables k -> res[1]"""
    n, m = len(sizes), max(sizes)
    imgs = _dev(cuda, [np.zeros((4, 4, 3), np.uint8)] * n)
    pos = [(k / 2, k / 2) for k in sizes]                       # box [0, 0, k, k]
    wins = [(float(k), float(k)) for k in sizes]
    _, _, status, ws, rc, _ = _prepare(cuda, imgs, pos, wins, [0] * n, res, (m, m))
    assert rc == 0 and not status.any()
    for k, (bx, cx, by, cy) in zip(sizes, _tables(ws, n, res, (m, m))):
        for (b, c), out in (((bx, cx), res[0]), ((by, cy), res[1])):
            wb, wc = preprocess.resample_tables(k, out)
            assert np.array_equal(b, wb) and np.array_equal(c, wc), (k, out)


# ---- frames --------------------------------------------------------------------------------------------------------------

@pytest.fixture(scope='module')
def sweep():
    """test_gpu_pre_post's seeded sweep, drawn again from its seed"""
    rng = np.random.default_rng(20261018)
    batches = []
    for res in SWEEP_RES:
        imgs, pos, wins = [], [], []
        for _ in range(36):
            h, w = (int(v) for v in np.exp(rng.uniform(0, np.log(700), 2)).round().clip(1, 700))
            imgs.append(_image(rng, h, w))
            p, win = _window(rng, h, w)
            pos.append(p)
            wins.append(win)
        batches.append((res, imgs, pos, wins, rng.integers(0, 2, len(imgs))))
    return batches


def _same_as_call(cuda, res, imgs, pos, wins, hflip, power=1, device_boxes=False):
    pipe = preprocess.FramePipeline(res)
    want, a_want = pipe(imgs, pos, wins, hflip=hflip, channel_power=power)
    dev = _dev(cuda, imgs)
    if device_boxes:
        boxes = [preprocess.crop_box(p, w) for p, w in zip(pos, wins)]
        mc = (max(int(b[2] - b[0]) for b in boxes), max(int(b[3] - b[1]) for b in boxes))
        t = lambda a: cuda.from_numpy(np.asarray(a, np.float64)).cuda()          # noqa: E731
        got, afmat, status = pipe.from_device(dev, t(pos), t(wins), hflip=cuda.from_numpy(np.asarray(hflip)).cuda(),
                                              channel_power=power, max_crop=mc)
    else:
        got, afmat, status = pipe.from_device(dev, pos, wins, hflip=hflip, channel_power=power)
    cuda.cuda.synchronize()
    assert not status.any(), status
    assert cuda.equal(got, want)
    a = afmat.cpu().numpy()
    assert np.array_equal(a, a_want)
    for i in range(len(imgs)):
        assert np.array_equal(a[i], preprocess.affine_map(preprocess.crop_box(pos[i], wins[i]), res, hflip[i] == 1))
    return got


def test_sweep_equals_call(cuda, sweep):
    for k, (res, imgs, pos, wins, hflip) in enumerate(sweep):
        power = (1.0, 1.5, 0.7) if k == 2 else 1
        _same_as_call(cuda, res, imgs, pos, _pairs(wins), hflip, power, device_boxes=k % 2 == 1)


@pytest.mark.parametrize('name', sorted(EDGES))
def test_named_edge_equals_call(cuda, name):
    res, imgs, pos, wins, hflip = EDGES[name]
    _same_as_call(cuda, res, imgs, pos, wins, np.asarray(hflip))


def test_scratch_past_2_gib(cuda):
    """test_gpu_pre_post's 32 windows 64 wide x 100 000 tall: the horizontal pass's scratch is 2.46 GB"""
    rng = np.random.default_rng(64)
    n, res = 32, (256, 256)
    imgs = [_image(rng, int(h), int(w)) for h, w in rng.integers(20, 60, (n, 2))]
    pos = [(im.shape[1] / 2, im.shape[0] / 2 + off) for im, off in zip(imgs, np.linspace(49000, -49900, n))]
    wins = [(64.0, 100000.0)] * n
    assert _ffi.lib().dh_prepare_frames_workspace(n, 64, 100000, 256, 256) > 2 ** 31
    _same_as_call(cuda, res, imgs, pos, wins, np.arange(n) % 2)


def test_65535_frames_and_one_more_refused(cuda):
    torch = cuda
    rng = np.random.default_rng(65535)
    n = 65535
    stack = rng.integers(0, 256, (n + 1, 4, 4, 3), dtype=np.uint8)
    pos = np.tile([[2.0, 2.0]], (n + 1, 1)) + rng.integers(-2, 3, (n + 1, 2))
    hflip = (np.arange(n + 1) % 3 == 0).astype(np.int64)
    pipe = preprocess.FramePipeline((8, 8))
    want, a_want = pipe(list(stack[:n]), pos[:n], 4.0, hflip=hflip[:n])
    dev = torch.from_numpy(stack).cuda()
    imgs = [dev[i] for i in range(n + 1)]
    got, afmat, status = pipe.from_device(imgs[:n], pos[:n], 4.0, hflip=hflip[:n])
    torch.cuda.synchronize()
    assert torch.equal(got, want) and not status.any()
    assert np.array_equal(afmat.cpu().numpy(), a_want)
    ctx = pipe._context()
    before = ctx.launch_count()
    with pytest.raises(_ffi.DeepharB200Error, match='65535'):
        pipe.from_device(imgs, pos, 4.0, hflip=hflip)
    assert ctx.launch_count() == before


def test_jpeg_decode_images_equal_from_jpeg(cuda):
    from deephar_b200 import jpeg
    res, imgs, pos, wins, hflip = EDGES['tallest_not_first']
    rng = np.random.default_rng(5)
    imgs = imgs + [_image(rng, 480, 640), _image(rng, 100, 37)]
    pos = pos + [(320.0, 240.0), (10.0, 90.0)]
    wins = wins + [(500.0, 470.0), (30.0, 31.0)]
    hflip = list(hflip) + [1, 0]
    src = [_jpeg(im) for im in imgs]
    pipe = preprocess.FramePipeline(res)
    want, a_want = pipe.from_jpeg(src, pos, wins, hflip=hflip)
    decoded = jpeg.decode(src)
    got, afmat, status = pipe.from_device(decoded, pos, wins, hflip=hflip)
    cuda.cuda.synchronize()
    assert cuda.equal(got, want) and not status.any()
    assert np.array_equal(afmat.cpu().numpy(), a_want)
    assert cuda.equal(got, pipe(_decoded(src), pos, wins, hflip=hflip)[0])


# ---- flagged frames and refused calls ------------------------------------------------------------------------------------

def test_flagged_frames_leave_their_neighbours_alone(cuda):
    rng = np.random.default_rng(11)
    res, n = (48, 40), 9
    imgs = [_image(rng, 60 + 7 * i, 80 - 3 * i) for i in range(n)]
    pos = [(30.0 + i, 25.0 + 2 * i) for i in range(n)]
    wins = [(40.0 + 3 * i, 35.0 + 2 * i) for i in range(n)]
    hflip = [i % 2 for i in range(n)]
    mc = (64, 51)
    dev = _dev(cuda, imgs)
    base, a_base, s_base, _, rc, _ = _prepare(cuda, dev, pos, wins, hflip, res, mc)
    assert rc == 0 and not s_base.any()
    assert cuda.equal(base, preprocess.FramePipeline(res)(imgs, pos, wins, hflip=hflip)[0])
    E, L, B = _ffi.FRAME_EMPTY, _ffi.FRAME_TOO_LARGE, _ffi.FRAME_BAD_BOX
    # box [8, 25, 8 + cw, ...]: cw = 64 is max_crop_w, 65 one more
    cases = {
        'empty_w': (1, (8.5, 26.0), (0.5, 30.0), E), 'empty_h': (2, (30.0, 26.5), (30.0, 0.9), E),
        'negative': (3, (30.0, 26.0), (-4.0, 30.0), E),
        'at_max': (4, (40.0, 45.0), (64.0, 51.0), 0), 'wider_than_max': (4, (40.5, 45.0), (65.0, 51.0), L),
        'taller_than_max': (5, (40.0, 45.5), (64.0, 53.0), L),
        'nan_pos': (6, (np.nan, 3.0), (30.0, 30.0), B), 'inf_win': (7, (30.0, 3.0), (30.0, np.inf), B),
        'outside_int32': (8, (2.2e9, 3.0), (30.0, 30.0), B), 'edge_outside_int32': (0, (-2147483000.0, 3.0), (2000.0, 30.0), B),
    }
    for name, (i, p, w, bit) in cases.items():
        pos2, wins2 = list(pos), list(wins)
        pos2[i], wins2[i] = p, w
        out, afmat, status, _, rc, _ = _prepare(cuda, dev, pos2, wins2, hflip, res, mc)
        assert rc == 0
        st = status.cpu().numpy()
        assert st[i] == bit and not np.delete(st, i).any(), (name, st)
        keep = [k for k in range(n) if k != i]
        assert cuda.equal(out[keep], base[keep]), name
        assert np.array_equal(afmat.cpu().numpy()[keep], a_base.cpu().numpy()[keep]), name
        if bit:
            assert bool(out[i].isnan().all()) and bool(afmat[i].isnan().all()), name
        else:
            want = preprocess.FramePipeline(res)([imgs[i]], [p], [w], hflip=[hflip[i]])[0]
            assert cuda.equal(out[i:i + 1], want), name


def test_short_workspace_is_refused_before_any_launch(cuda):
    rng = np.random.default_rng(3)
    imgs = _dev(cuda, [_image(rng, 30, 40)] * 3)
    pos, wins = [(20.0, 15.0)] * 3, [(30.0, 20.0)] * 3
    for extra, ok in ((-1, False), (0, True)):
        out, _, status, _, rc, ctx = _prepare(cuda, imgs, pos, wins, [0] * 3, (16, 16), (30, 20), ws_extra=extra)
        launches = ctx.launch_count()
        if ok:
            assert rc == 0 and launches == 3 and not status.any()
        else:
            assert rc < 0 and launches == 0 and b'workspace' in _ffi.lib().dh_last_error()
            assert bool((out == 7.0).all()) and bool((status == -1).all())


# ---- pose mapping --------------------------------------------------------------------------------------------------------

def _p2i(cuda, buf, c0, c, nj, A, per_sample):
    """dh_pose_to_image_f32 on channels c0 .. c0 + c of buf (n, nj, ld)"""
    n, ld = buf.shape[0], buf.shape[2]
    v = _ffi.dh_view(buf.data_ptr() + 4 * c0, n, 1, nj, c, ld)
    out = cuda.full((n, nj, 2), 5.0, dtype=cuda.float64, device='cuda')
    ctx = _ffi.Context(cuda.cuda.current_device())
    _ffi.check(_ffi.lib().dh_pose_to_image_f32(ctx.handle, C.byref(v), A.data_ptr(), per_sample, out.data_ptr(),
                                               cuda.cuda.current_stream().cuda_stream), 'dh_pose_to_image_f32')
    return out


@pytest.mark.parametrize('per_sample', [0, 1])
@pytest.mark.parametrize('window', [(0, 2, 2), (1, 3, 6)], ids=['dense', 'channel_window'])
def test_pose_mapping_equals_pose_eval(cuda, per_sample, window):
    torch = cuda
    rng = np.random.default_rng(per_sample * 10 + window[0])
    n, nj = 3001, 17
    c0, c, ld = window
    buf = torch.from_numpy(rng.uniform(-0.3, 1.3, (n, nj, ld)).astype(np.float32)).cuda()
    A = rng.normal(0, 1, (n if per_sample else 1, 3, 3)) * [1e-3, 1e-3, 0.5]
    A[:, 2] = [0, 0, 1]
    A[:, 0, 0] += 1 / 640
    A[:, 1, 1] += 1 / 480
    if per_sample:
        A[5] = [[1, 2, 0], [2, 4, 0], [0, 0, 1]]                    # singular: NaN poses
    Ad = torch.from_numpy(A).cuda()
    got = _p2i(cuda, buf, c0, c, nj, Ad, per_sample)
    wide = buf[:, :, c0:c0 + 2].to(torch.float64).contiguous()      # exact widening
    want, _, _, _ = postprocess._run(wide, Ad if per_sample else Ad[0], True)
    torch.cuda.synchronize()
    g, w = got.cpu().numpy(), want.cpu().numpy()
    assert np.array_equal(g, w, equal_nan=True)
    if per_sample:
        assert np.isnan(g[5]).all() and not np.isnan(np.delete(g, 5, axis=0)).any()


# ---- end to end: examples/run_camera.c -----------------------------------------------------------------------------------

def test_run_camera_equals_python(cuda, tmp_path):
    """C4-like penn frames (VGA, 256 x 256 crops, S = 3, T = 16 + 3 pushes, resets), a window per frame that drifts and
    one frame whose window is larger than max_crop: the C program's plain and graph-replayed outputs, image-space poses,
    ready flags and status equal from_device -> ClipStream.push -> transform_pose_sequence"""
    torch = cuda
    from deephar_b200.stream import ClipStream
    from oracle import synth
    from test_gpu_stream import _c4
    cc = shutil.which('gcc') or shutil.which('cc')
    assert cc, 'no C compiler'
    cuda_home = os.environ.get('CUDA_HOME', '/usr/local/cuda')
    libdir = os.path.dirname(_ffi.LIB_PATH)
    exe = str(tmp_path / 'run_camera')
    subprocess.check_call([cc, '-std=c99', '-O2', '-Wall', '-Werror', '-I', os.path.join(ROOT, 'include'),
                           '-I', os.path.join(cuda_home, 'include'), os.path.join(ROOT, 'examples', 'run_camera.c'),
                           '-o', exe, '-L', libdir, '-ldeephar_b200', '-L', os.path.join(cuda_home, 'lib64'), '-lcudart',
                           '-Wl,-rpath,' + libdir + ':' + os.path.join(cuda_home, 'lib64')])
    m = _c4().init_synthetic_weights(1234)
    T, S, H, W = m.graph.frames_per_clip, 3, 480, 640
    n_push = T + 3
    resets = {1: [1], T: [2], T + 2: None}
    rng = np.random.default_rng(41)
    video = ((synth.synth_frames(n_push * S, H // 4, W // 4, seed=23) + 1) * 127.5).clip(0, 255).astype(np.uint8)
    video = np.repeat(np.repeat(video, 4, axis=1), 4, axis=2).reshape(n_push, S, H, W, 3)
    boxes = np.zeros((n_push, S, 5))
    boxes[..., 0] = 320 + rng.uniform(-40, 40, (n_push, S))
    boxes[..., 1] = 240 + rng.uniform(-30, 30, (n_push, S))
    boxes[..., 2] = rng.uniform(200, 420, (n_push, S))
    boxes[..., 3] = rng.uniform(200, 470, (n_push, S))
    boxes[..., 4] = rng.integers(0, 2, (n_push, S))
    boxes[4, 1, 2] = 700.0                                              # wider than max_crop: flagged, NaN
    max_crop = (480, 480)
    cs = ClipStream(m, S)
    path, frames, bfile, rfile, prefix = [str(tmp_path / f) for f in ('c4.dhs', 'f.u8', 'b.f64', 'r.txt', 'out')]
    cs.export(path)
    video.tofile(frames)
    boxes.tofile(bfile)
    with open(rfile, 'w') as f:
        for i, ids in sorted(resets.items()):
            f.write('%d %s\n' % (i, ' '.join(str(k) for k in (ids or []))))
    pipe = preprocess.FramePipeline((256, 256))
    want, poses, ready, status = [], [], [], []
    for i in range(n_push):
        if i in resets:
            cs.reset(resets[i])
        imgs = _dev(cuda, list(video[i]))
        x, afmat, st = pipe.from_device(imgs, boxes[i, :, :2], boxes[i, :, 2:4], hflip=boxes[i, :, 4].astype(np.int64),
                                        max_crop=max_crop)
        out = cs.push(x)
        want.append([o.cpu().numpy() for o in out.frame_outputs + out.clip_outputs])
        p = out.frame_outputs[0].reshape(S, -1, out.frame_outputs[0].shape[-1])
        poses.append(postprocess.transform_pose_sequence(afmat, p, inverse=True))
        ready.append(out.ready.astype(np.int32))
        status.append(st.cpu().numpy())
    assert status[4][1] == _ffi.FRAME_TOO_LARGE
    env = {k: v for k, v in os.environ.items() if not k.startswith('PYTHON')}
    run = subprocess.run([exe, path, frames, str(H), str(W), bfile, str(max_crop[0]), str(max_crop[1]), prefix, rfile],
                         capture_output=True, text=True, timeout=900, env=env)
    assert run.returncode == 0, run.stdout[-2000:] + run.stderr[-2000:]
    for tag in ('', 'graph.'):
        for k in range(len(want[0])):
            got = np.fromfile('%s.%s%d.f32' % (prefix, tag, k), np.float32).reshape((n_push,) + want[0][k].shape)
            for i in range(n_push):
                assert np.array_equal(got[i], want[i][k], equal_nan=True), (tag, k, i)
        got = np.fromfile('%s.%spose.f64' % (prefix, tag), np.float64).reshape((n_push,) + poses[0].shape)
        for i in range(n_push):
            assert np.array_equal(got[i], poses[i], equal_nan=True), (tag, 'pose', i)
        assert np.fromfile('%s.%sready.i32' % (prefix, tag), np.int32).reshape(n_push, S).tolist() == \
            np.stack(ready).tolist(), tag
        assert np.fromfile('%s.%sstatus.i32' % (prefix, tag), np.int32).reshape(n_push, S).tolist() == \
            np.stack(status).tolist(), tag
