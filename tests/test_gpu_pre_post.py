"""The two kernels on either side of the forward, at their edges.

dh_crop_resize_norm_u8 (csrc/preprocess.cu, through FramePipeline and FramePipeline.from_jpeg) bit for bit against
oracle.preprocess.eval_frame, which tests/test_preprocess.py pins against Pillow: a seeded sweep of image sizes, windows,
centres, output resolutions and flips; named edges (a window outside the image, a window equal to the image, a 1-pixel
crop, 1920 x 1080 -> 8 x 8, the tallest crop in the middle of a batch, 64+ resampling tables in one batch); a batch whose
`tmp` scratch passes 2^31 bytes; the 65 535-frame grid limit; channel_power within the accuracy CUDA states for powf.

dh_pose_eval_f64 (csrc/postprocess.cu, through deephar_b200.postprocess) against a plain float64 restatement of the
reference's deephar/utils/transform.py:136-209 and deephar/measures.py:5-146 written out below: np.linalg.inv, np.dot,
sqrt(sum(x ** 2)) / head_size <= refp with the double refp.  Hit and valid counts must be the reference's exactly,
including samples planted within 1e-6 ... 1e-10 (relative) of the threshold and the float32(0.2) sample that a float32
threshold counts as a hit.  Behaviour the reference does not have is pinned: a singular affine map (np.linalg.inv
raises) gives NaN poses that count as valid and never as hits.
"""
import io

import numpy as np
import pytest

from deephar_b200 import preprocess
from oracle import preprocess as opre

pytestmark = pytest.mark.gpu

EPS = np.finfo(np.float64).eps


# ---- crop / resize / normalise ---------------------------------------------------------------------------------------

def _image(rng, h, w):
    return rng.integers(0, 256, (h, w, 3), dtype=np.uint8)


def _want(img, objpos, win, res, hflip, power=1):
    return opre.eval_frame(img, preprocess.crop_box(objpos, win), res, hflip=bool(hflip), channel_power=power)


def _jpeg(img):
    from PIL import Image
    buf = io.BytesIO()
    Image.fromarray(img).save(buf, format='JPEG', quality=92)
    return buf.getvalue()


def _decoded(sources):
    """Pillow's decode of JPEG bytes, as the reference's loaders open their frames"""
    from PIL import Image
    return [np.asarray(Image.open(io.BytesIO(s)).convert('RGB')) for s in sources]


def _same_from_jpeg(cuda, res, imgs, objpos, wins, hflip=0, power=1):
    """from_jpeg(JPEG bytes) == __call__(Pillow's decode of the same bytes), bit for bit; -> the frames"""
    src = [_jpeg(im) for im in imgs]
    pipe = preprocess.FramePipeline(res)
    want, a_want = pipe(_decoded(src), objpos, wins, hflip=hflip, channel_power=power)
    got, a_got = pipe.from_jpeg(src, objpos, wins, hflip=hflip, channel_power=power)
    cuda.cuda.synchronize()
    assert np.array_equal(a_got, a_want)
    assert cuda.equal(got, want)
    return got


def _window(rng, h, w):
    """(objpos, winsize) of one sweep frame: a window of 1 px .. 3x the image, square (scalar) or (w, h); its centre
    inside the image, on one of its corners, or far enough out that the window misses the image."""
    while True:
        if rng.random() < 0.4:
            side = float(np.exp(rng.uniform(0.0, np.log(3 * max(h, w)))))
            win, ww, wh = side, side, side
        else:
            ww, wh = (float(np.exp(rng.uniform(0.0, np.log(3 * s)))) for s in (w, h))
            win = (ww, wh)
        kind = rng.integers(3)
        if kind == 0:
            pos = (rng.uniform(0, w), rng.uniform(0, h))
        elif kind == 1:
            pos = (float(w * rng.integers(2)), float(h * rng.integers(2)))
        else:
            sx, sy = rng.choice([-1, 1], 2)
            pos = (w / 2 + sx * (w / 2 + ww / 2 + rng.uniform(1, 50)), h / 2 + sy * (h / 2 + wh / 2 + rng.uniform(1, 50)))
        box = preprocess.crop_box(pos, win)
        if box[2] > box[0] and box[3] > box[1]:
            return pos, win


SWEEP_RES = [(1, 37), (23, 1), (7, 5), (17, 64), (256, 8), (64, 64), (1, 1)]


@pytest.fixture(scope='module')
def sweep():
    """7 batches of 36 frames (252 in all), one output resolution (w, h) each"""
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


def test_sweep_matches_oracle(cuda, sweep):
    n = 0
    for res, imgs, pos, wins, hflip in sweep:
        pipe = preprocess.FramePipeline(res)
        # FramePipeline takes one winsize form per batch: (w, h) pairs, a square side broadcast to both
        pairs = [(w, w) if np.isscalar(w) else w for w in wins]
        out, afmat = pipe(imgs, pos, pairs, hflip=hflip)
        out = out.cpu().numpy()
        for i, im in enumerate(imgs):
            assert np.array_equal(out[i], _want(im, pos[i], wins[i], res, hflip[i])), (res, i, im.shape, pos[i], wins[i])
            assert np.array_equal(afmat[i], preprocess.affine_map(preprocess.crop_box(pos[i], wins[i]), res, hflip[i] == 1))
        n += len(imgs)
    assert n >= 200


def test_sweep_square_windows_as_scalars(cuda, sweep):
    """the (N,) scalar-side form of winsize, on the sweep frames whose windows are square"""
    for res, imgs, pos, wins, hflip in sweep[:3]:
        k = [i for i, w in enumerate(wins) if np.isscalar(w)]
        assert len(k) >= 5
        out, _ = preprocess.FramePipeline(res)([imgs[i] for i in k], [pos[i] for i in k], [wins[i] for i in k],
                                                 hflip=hflip[k])
        out = out.cpu().numpy()
        for j, i in enumerate(k):
            assert np.array_equal(out[j], _want(imgs[i], pos[i], wins[i], res, hflip[i])), (res, i)


def test_sweep_from_jpeg(cuda, sweep):
    res, imgs, pos, wins, hflip = sweep[3]
    _same_from_jpeg(cuda, res, imgs[:12], pos[:12], [(w, w) if np.isscalar(w) else w for w in wins[:12]], hflip[:12])


def _edge_cases():
    rng = np.random.default_rng(7)
    img = _image(rng, 48, 64)
    tall = [_image(rng, h, w) for h, w in [(30, 40), (50, 20), (600, 90), (25, 300), (80, 80)]]
    keys = [_image(rng, 20 + 3 * i, 30 + 5 * i) for i in range(40)]
    return {
        # name: (resolution (w, h), images, objpos, winsize, hflip)
        'outside': ((32, 24), [img, img], [(-500.0, 20.0), (100.0, 400.0)], [(60.0, 40.0), (90.0, 200.0)], [0, 1]),
        'identity': ((64, 48), [img, img], [(32.0, 24.0)] * 2, [(64.0, 48.0)] * 2, [0, 1]),
        'one_pixel': ((256, 256), [img, img], [(10.5, 7.5), (63.5, 47.5)], [(1.0, 1.0)] * 2, [0, 1]),
        'full_hd_to_8': ((8, 8), [_image(rng, 1080, 1920)], [(960.0, 540.0)], [(1920.0, 1080.0)], [1]),
        'tallest_not_first': ((40, 56), tall, [(20.0, 15.0), (10.0, 25.0), (45.0, 300.0), (150.0, 12.0), (40.0, 40.0)],
                              [(40.0, 30.0), (20.0, 50.0), (90.0, 600.0), (300.0, 25.0), (70.0, 90.0)], [0, 1, 0, 1, 0]),
        'many_tables': ((48, 40), keys, [(15.0 + 2.5 * i, 10.0 + 1.5 * i) for i in range(40)],
                        [(30.0 + 5 * i, 20.0 + 3 * i) for i in range(40)], [i % 2 for i in range(40)]),
    }


EDGES = _edge_cases()


@pytest.mark.parametrize('name', sorted(EDGES))
def test_named_edge(cuda, name):
    res, imgs, pos, wins, hflip = EDGES[name]
    pipe = preprocess.FramePipeline(res)
    frames, bounds, coefs, boxes, afmat, max_ch = pipe.plan([im.shape[:2] for im in imgs], pos, wins, hflip)
    out = pipe(imgs, pos, wins, hflip=hflip)[0].cpu().numpy()
    for i, im in enumerate(imgs):
        assert np.array_equal(out[i], _want(im, pos[i], wins[i], res, hflip[i])), (name, i)
    if name == 'outside':
        assert np.all(out == -1.0)
    elif name == 'identity':
        norm = opre.normalize_channels(imgs[0])
        assert np.array_equal(out[0], norm) and np.array_equal(out[1], norm[:, ::-1])
    elif name == 'one_pixel':
        for i, (x, y) in enumerate([(10, 7), (63, 47)]):
            assert np.array_equal(out[i], np.broadcast_to(opre.normalize_channels(imgs[i][y:y + 1, x:x + 1]), out[i].shape))
    elif name == 'tallest_not_first':
        assert max_ch == 600 and int(np.argmax(boxes[:, 3] - boxes[:, 1])) == 2
    elif name == 'many_tables':
        keys = {(f.kx_off, f.ksx) for f in frames} | {(f.ky_off, f.ksy) for f in frames}
        assert len(keys) >= 64
    _same_from_jpeg(cuda, res, imgs, pos, wins, hflip)


def test_tmp_offsets_past_2_gib(cuda):
    """32 windows 64 wide x 100 000 tall on small images, 256 x 256 out: the horizontal pass's scratch is
    32 * 100 000 * 256 * 3 bytes (2.46 GB), so the last four frames lie wholly past 2^31 in it.  The image sits at a
    different height of each window (the last frame's near the bottom, the deepest bytes of the scratch)."""
    rng = np.random.default_rng(64)
    n, res = 32, (256, 256)
    assert n * 100000 * res[0] * 3 > 2 ** 31
    imgs = [_image(rng, int(h), int(w)) for h, w in rng.integers(20, 60, (n, 2))]
    pos = [(im.shape[1] / 2, im.shape[0] / 2 + off) for im, off in zip(imgs, np.linspace(49000, -49900, n))]
    wins = [(64.0, 100000.0)] * n
    hflip = np.arange(n) % 2
    pipe = preprocess.FramePipeline(res)
    out = pipe(imgs, pos, wins, hflip=hflip)[0]
    for i in (0, n // 2, n - 1):
        want = _want(imgs[i], pos[i], wins[i], res, hflip[i])
        assert np.any(want > -1.0), i                        # the image shows in the output
        assert np.array_equal(out[i].cpu().numpy(), want), i
    del out
    got = _same_from_jpeg(cuda, res, imgs, pos, wins, hflip)
    assert got.shape[0] == n


def test_grid_limit(cuda):
    """65 535 frames (the most one launch's grid.z holds) are right at both ends; 65 536 raise the library's error and
    leave `out` untouched"""
    from deephar_b200 import _ffi
    rng = np.random.default_rng(65535)
    n = 65535
    stack = rng.integers(0, 256, (n + 1, 4, 4, 3), dtype=np.uint8)
    imgs = list(stack)
    pos = np.tile([[2.0, 2.0]], (n + 1, 1)) + rng.integers(-2, 3, (n + 1, 2))
    hflip = np.arange(n + 1) % 3 == 0
    pipe = preprocess.FramePipeline((8, 8))
    out = pipe(imgs[:n], pos[:n], 4.0, hflip=hflip[:n])[0]
    check = [0, 1, 2, n // 2, n - 3, n - 2, n - 1]
    for i in check:
        assert np.array_equal(out[i].cpu().numpy(), _want(imgs[i], pos[i], 4.0, (8, 8), hflip[i])), i
    sentinel = torch_full_like(cuda, out, 7.0, n + 1)
    with pytest.raises(_ffi.DeepharB200Error, match='65535'):
        pipe(imgs, pos, 4.0, hflip=hflip, out=sentinel)
    cuda.cuda.synchronize()
    assert bool((sentinel == 7.0).all())
    src = [_jpeg(im) for im in imgs[:n]]
    got = pipe.from_jpeg(src, pos[:n], 4.0, hflip=hflip[:n])[0]
    dec = _decoded([src[i] for i in check])
    for j, i in enumerate(check):
        assert np.array_equal(got[i].cpu().numpy(), _want(dec[j], pos[i], 4.0, (8, 8), hflip[i])), i


def torch_full_like(torch, ref, value, n):
    return torch.full((n,) + tuple(ref.shape[1:]), value, dtype=ref.dtype, device=ref.device)


# CUDA C++ Programming Guide, "Mathematical Functions" appendix, single-precision table: powf(x, y) has a maximum error
# of 4 ulp (full range, without -use_fast_math, which this library is not built with).  numpy's float32 power is held
# to 1 ulp of the float64 power rounded to float32 below, so the kernel's x ** p lies within 4 + 1 ulp of numpy's.
POWF_ULP = 4
NUMPY_POW_ULP = 1


def _steps(t, k):
    """t moved k float32 ulps (k < 0: down)"""
    t = t.copy()
    for _ in range(abs(k)):
        t = np.nextafter(t, np.float32(np.inf if k > 0 else -np.inf))
    return t


def test_channel_power_within_powf_accuracy(cuda):
    """every uint8 level, through an identity crop so the resampler passes the pixels through unchanged"""
    levels = np.arange(256, dtype=np.uint8)
    img = np.stack([np.roll(levels, 85 * c) for c in range(3)], axis=-1).reshape(16, 16, 3)
    imgs, pos, wins = [img, img[::-1].copy()], [(8.0, 8.0)] * 2, [(16.0, 16.0)] * 2
    for power in [(0.45, 1.7, 2.2), (3.1, 0.9, 1.0), (0.1, 1.0, 5.0)]:
        out = preprocess.FramePipeline((16, 16))(imgs, pos, wins, hflip=[0, 1], channel_power=power)[0].cpu().numpy()
        for i, im in enumerate(imgs):
            src = im[:, ::-1] if i else im
            x = src.astype(np.float32) / np.float32(255.0)
            p = np.asarray(power, np.float32)
            t = np.power(x, p)
            exact = np.power(x.astype(np.float64), p.astype(np.float64)).astype(np.float32)
            assert np.all(np.abs(t.view(np.int32) - exact.view(np.int32)) <= NUMPY_POW_ULP)
            t = np.where(p == 1, x, t)                                      # the reference skips ** 1
            lo = (_steps(t, -(POWF_ULP + NUMPY_POW_ULP)) - np.float32(0.5)) * np.float32(2.0)
            hi = (_steps(t, POWF_ULP + NUMPY_POW_ULP) - np.float32(0.5)) * np.float32(2.0)
            assert np.all((lo <= out[i]) & (out[i] <= hi)), (power, i)
            exact_ch = p == 1
            assert np.array_equal(out[i][..., exact_ch], ((t - np.float32(0.5)) * np.float32(2.0))[..., exact_ch])
    _same_from_jpeg(cuda, (16, 16), [img], [(8.0, 8.0)], [(16.0, 16.0)], power=(0.45, 1.7, 2.2))


# ---- pose evaluation -------------------------------------------------------------------------------------------------

USED = [2, 3, 4, 5, 6, 7, 10, 11, 12, 13, 14, 15, 8, 9]                       # measures.py:65


def ref_transform(A, poses, inverse=True):
    """transform.py:136-209 (transform_pose_sequence / transform_2d_points), float64"""
    A = np.array(A, np.float64)
    poses = np.asarray(poses, np.float64)
    if inverse:
        if A.ndim == 3:
            for i in range(len(A)):
                A[i] = np.linalg.inv(A[i])
        else:
            A = np.linalg.inv(A)
    y = np.empty(poses.shape[:2] + (2,))
    for j in range(len(poses)):
        M = A[j] if A.ndim == 3 else A
        h = np.ones((3, poses.shape[1]))
        h[0:2, :] = poses[j, :, 0:2].T
        y[j] = np.dot(M, h)[0:2].T
    return y, A


def ref_measures(y_true, y_pred, head_size, refp):
    """measures.py:5-16 (_norm, _valid_joints) and the per-sample lines of pckh / pckh_per_joint / mean_distance_error:
    -> (hit, valid, dist) per (sample, joint); dist not divided by the head size"""
    y_true = np.asarray(y_true, np.float64)
    valid = np.all(y_true > -1e6, axis=-1)
    dist = np.sqrt(np.sum(np.power(y_true - y_pred, 2), axis=-1))
    norm = dist / np.asarray(head_size, np.float64).reshape(-1, 1) if head_size is not None else dist
    return (norm <= refp) & valid, valid, dist


def _affines(rng, n, general=False):
    """MPII-style crop maps: scale 1/(200 s) (never a float32), translation to the crop corner; `general` adds a
    rotation and an anisotropic scale (factor 1.3)"""
    s = 1.0 / (200.0 * rng.uniform(0.8, 4.0, n))
    A = np.zeros((n, 3, 3))
    A[:, 0, 0] = A[:, 1, 1] = s
    if general:
        th = rng.uniform(-0.5, 0.5, n)
        A[:, 0, 0], A[:, 0, 1] = s * np.cos(th), -s * np.sin(th) * 1.3
        A[:, 1, 0], A[:, 1, 1] = s * np.sin(th), s * np.cos(th) * 1.3
    A[:, 0, 2] = -s * rng.uniform(0, 1500, n)
    A[:, 1, 2] = -s * rng.uniform(0, 1000, n)
    A[:, 2, 2] = 1.0
    return A


def _pose_bound(M, pred):
    """|GPU - reference| allowed per coordinate: 32 fp64 ulps of the terms summed.  The two 3x3 inverses (cofactors
    on the GPU, LU in LAPACK) differ by up to ~14 such ulps on the maps of `_affines`."""
    M = np.broadcast_to(M, (len(pred), 3, 3))
    h = np.concatenate([np.abs(pred[:, :, :2]), np.ones(pred.shape[:2] + (1,))], axis=-1)
    return 32 * EPS * np.einsum('nij,nkj->nki', np.abs(M[:, :2, :]), h)


def _device(cuda, a, width):
    """(N, nj, 2) float64 -> a contiguous (N, nj, width) float64 CUDA tensor (extra columns: z / visibility)"""
    full = np.concatenate([a, np.full(a.shape[:2] + (width - 2,), 0.25)], axis=-1) if width > 2 else a
    return cuda.from_numpy(np.ascontiguousarray(full)).cuda()


def _check_eval(cuda, pred, A, inverse, y_true, head, refp, width=2):
    """one kernel launch against the restatement: counts exact, poses and distance sums within their bounds"""
    from deephar_b200 import postprocess as pp
    want_pose, M = ref_transform(A, pred, inverse)
    hit, valid, dist = ref_measures(y_true, want_pose, head, refp)
    out, hits, valid_g, dsum = pp._run(_device(cuda, pred, width), A, inverse, y_true, head, refp)
    assert out.dtype == cuda.float64
    out, hits, valid_g, dsum = (t.cpu().numpy() for t in (out, hits, valid_g, dsum))
    assert np.array_equal(valid_g, valid.sum(axis=0))
    assert np.array_equal(hits, hit.sum(axis=0)), (hits - hit.sum(axis=0)).nonzero()
    assert np.all(np.abs(out - want_pose) <= _pose_bound(M, pred))
    # the atomics add in any order: |error| <= (n - 1) eps sum(d) (recursive summation) + the poses' own error
    d = np.where(valid, dist, 0.0)
    pose_err = np.sqrt(2.0) * _pose_bound(M, pred).max(axis=-1)
    bound = (len(pred) * EPS * d.sum(axis=0)) + np.where(valid, pose_err, 0.0).sum(axis=0)
    assert np.all(np.abs(dsum - d.sum(axis=0)) <= bound)
    return out, hits, dsum


@pytest.mark.parametrize('nj,n,width', [(16, 100000, 2), (17, 3001, 3), (20, 257, 4)])
@pytest.mark.parametrize('per_sample', [0, 1])
@pytest.mark.parametrize('inverse', [0, 1])
def test_pose_eval_matches_float64_reference(cuda, nj, n, width, per_sample, inverse):
    rng = np.random.default_rng(nj * 1000 + n + 7 * per_sample + 3 * inverse)
    A = _affines(rng, n if per_sample else 1, general=bool(n % 2))
    A = A if per_sample else A[0]
    if not inverse:
        A = np.linalg.inv(A)                                           # the crop -> image map, applied as given
    pred = rng.uniform(0.0, 1.0, (n, nj, 2))
    truth, _ = ref_transform(A, pred, inverse)
    head = rng.uniform(20.0, 60.0, (n, 1))
    y_true = truth + rng.normal(0.0, 0.3, truth.shape) * head[:, :, None]
    y_true[rng.random((n, nj)) < 0.05, 0] = -1e9                      # unannotated joints
    for refp in (0.5, 0.2):
        _check_eval(cuda, pred, A, inverse, y_true, head, refp, width)


def _near_ties(rng, n, nj, refp, A, sign):
    """poses whose reference distance / head size is refp * (1 + m), m = sign * {1e-6, 1e-8, 1e-10} (joint j gets the
    sign sign * (-1) ** j, so all of one joint's ties sit on one side of the threshold and one flip changes its count);
    head sizes and maps are not float32-representable."""
    pred = rng.uniform(0.05, 0.95, (n, nj, 2))
    truth, _ = ref_transform(A, pred, True)
    head = rng.uniform(20.0, 60.0, (n, 1))
    assert np.all(head != head.astype(np.float32))
    m = np.array([1e-6, 1e-8, 1e-10])[np.arange(n * nj).reshape(n, nj) % 3]
    m = m * sign * (-1.0) ** np.arange(nj)
    ang = rng.uniform(0, 2 * np.pi, (n, nj))
    r = refp * head * (1.0 + m)
    y_true = truth + np.stack([r * np.cos(ang), r * np.sin(ang)], axis=-1)
    return pred, y_true, head, m


@pytest.mark.parametrize('refp', [0.5, 0.2])
@pytest.mark.parametrize('per_sample', [0, 1])
def test_near_tie_counts_are_exact(cuda, refp, per_sample):
    rng = np.random.default_rng(int(refp * 10) + 2 * per_sample)
    n, nj = 600, 16
    for sign in (1.0, -1.0):
        A = _affines(rng, n if per_sample else 1)
        A = A if per_sample else A[0]
        pred, y_true, head, m = _near_ties(rng, n, nj, refp, A, sign)
        want_pose, _ = ref_transform(A, pred, True)
        hit, _, dist = ref_measures(y_true, want_pose, head, refp)
        assert np.array_equal(hit, m < 0)                              # the planted side, as the reference sees it
        _, hits, _ = _check_eval(cuda, pred, A, 1, y_true, head, refp)
        assert np.array_equal(hits, (m < 0).sum(axis=0))


def test_float32_threshold_sample(cuda):
    """d = float32(0.2) = 0.20000000298...: a miss against the double 0.2 the reference compares with"""
    from deephar_b200 import postprocess as pp
    pred = np.array([[[np.float32(0.2), 0.0]]])
    y_true = np.zeros((1, 1, 2))
    for inverse in (0, 1):
        _, hits, valid, _ = (t.cpu().numpy() for t in pp._run(pred, np.eye(3), inverse, y_true, np.ones(1), 0.2))
        assert valid.tolist() == [1] and hits.tolist() == [0]
    _, hits, _, _ = pp._run(pred, np.eye(3), 0, y_true, np.ones(1), float(np.float32(0.2)))
    assert hits.cpu().tolist() == [1]


def test_exact_ties_invalid_annotations_and_nan_predictions(cuda):
    """one launch per sample: d == refp is a hit (<=); an annotation is valid only when both coordinates are > -1e6
    (strictly); a NaN prediction counts as valid, is never a hit and makes the distance sum NaN, as in the reference"""
    from deephar_b200 import postprocess as pp
    lo = np.nextafter(-1e6, 0.0)                                       # valid; float32 would round it to -1e6
    cases = [  # (pred x, pred y), (true x, true y), head, (hit, valid) in the reference
        ((0.5, 0.0), (0.0, 0.0), 1.0, (1, 1)), ((3.0, 4.0), (0.0, 0.0), 10.0, (1, 1)),
        ((3.0, 4.0), (0.0, 0.0), 9.999999999999998, (0, 1)), ((1.0, 1.0), (-1e6, 0.0), 1.0, (0, 0)),
        ((1.0, 1.0), (0.0, -1e6), 1.0, (0, 0)), ((1.0, 1.0), (-1e6, -1e6), 1.0, (0, 0)),
        ((1.0, 1.0), (-2e6, 5.0), 1.0, (0, 0)), ((lo + 0.25, 0.0), (lo, 0.0), 1.0, (1, 1)),
        ((np.nan, 0.0), (0.0, 0.0), 1.0, (0, 1)), ((0.0, np.nan), (0.0, 0.0), 1.0, (0, 1))]
    for k, (p, t, h, (want_hit, want_valid)) in enumerate(cases):
        pred, y_true, head = np.array([[p]]), np.array([[t]]), np.array([[h]])
        hit, valid, dist = ref_measures(y_true, pred, head, 0.5)
        assert (int(hit.sum()), int(valid.sum())) == (want_hit, want_valid), k
        out, hits, valid_g, dsum = (a.cpu().numpy() for a in pp._run(pred, np.eye(3), 0, y_true, head, 0.5))
        # (M [x, y, 1])[0:2] with a NaN coordinate: both rows meet it (0 * NaN is NaN)
        assert np.array_equal(out, np.where(np.isnan(pred).any(), np.nan, pred), equal_nan=True), k
        assert (hits.tolist(), valid_g.tolist()) == ([want_hit], [want_valid]), k
        want_sum = (dist * valid).sum() if want_valid else 0.0          # measures.py:42: dist * valid
        assert np.array_equal(dsum, [want_sum], equal_nan=True), k


def test_singular_map_gives_nan_poses(cuda):
    """np.linalg.inv raises on an exactly singular map; the kernel writes NaN poses for that sample instead: valid where
    annotated, never a hit, NaN in the joint's distance sum.  The other samples are unaffected."""
    from deephar_b200 import postprocess as pp
    rng = np.random.default_rng(3)
    A = _affines(rng, 4)
    A[2] = [[1.0, 2.0, 0.0], [2.0, 4.0, 0.0], [0.0, 0.0, 1.0]]
    with pytest.raises(np.linalg.LinAlgError):
        np.linalg.inv(A[2])
    pred = rng.uniform(0, 1, (4, 16, 2))
    keep = [0, 1, 3]
    truth, _ = ref_transform(A[keep], pred[keep], True)
    y_true = np.zeros((4, 16, 2))
    y_true[keep] = truth + rng.normal(0, 3.0, truth.shape)
    y_true[2, 5] = -1e9
    head = rng.uniform(20, 60, (4, 1))
    out, hits, valid, dsum = (t.cpu().numpy() for t in pp._run(pred, A, 1, y_true, head, 0.5))
    assert np.all(np.isnan(out[2])) and not np.any(np.isnan(out[keep]))
    hit, v, _ = ref_measures(y_true[keep], truth, head[keep], 0.5)
    assert np.array_equal(hits, hit.sum(axis=0))
    assert np.array_equal(valid, v.sum(axis=0) + (np.arange(16) != 5))
    assert np.all(np.isnan(np.delete(dsum, 5))) and not np.isnan(dsum[5])


def test_public_scores_equal_the_reference(cuda):
    """pckh / pckh_per_joint (counts -> identical doubles), mean_distance_error (exact when every distance is an integer;
    otherwise within the summation bound), transform_pose_sequence (float64, within the pose bound)"""
    from deephar_b200 import postprocess as pp
    rng = np.random.default_rng(11)
    n = 5000
    A = _affines(rng, n)
    pred = rng.uniform(0, 1, (n, 16, 2)).astype(np.float32)             # what the model returns
    y_pred, M = ref_transform(A, pred, True)
    y_true = y_pred + rng.normal(0, 8.0, y_pred.shape)
    y_true[rng.random((n, 16)) < 0.1] = -1e9
    head = rng.uniform(20, 60, (n, 1))
    for refp in (0.5, 0.2):
        hit, valid, dist = ref_measures(y_true, y_pred, head, refp)
        want = (hit[:, USED].sum() / valid[:, USED].sum())
        assert pp.pckh(y_true, pred, head, refp, A=A) == want
        assert pp.pckh(y_true, y_pred, head, refp) == want
        with np.errstate(invalid='ignore'):
            assert np.array_equal(pp.pckh_per_joint(y_true, pred, head, refp, A=A), hit.sum(axis=0) / valid.sum(axis=0))
    got = pp.transform_pose_sequence(A, pred, inverse=True)
    assert got.dtype == np.float64 and np.all(np.abs(got - y_pred) <= _pose_bound(M, pred.astype(np.float64)))
    # mean_distance_error: measures.py:18-47
    _, valid, dist = ref_measures(y_true, y_pred, head, 0.5)
    want = (dist * valid).sum() / valid.sum()
    assert abs(pp.mean_distance_error(y_true, y_pred) - want) <= 2 * valid.sum() * EPS * want
    legs = rng.choice([(3, 4), (5, 12), (8, 15), (0, 7)], (n, 16))
    y_int = np.round(y_pred) + legs
    _, valid, dist = ref_measures(y_int, np.round(y_pred), head, 0.5)
    assert np.all(dist == np.round(dist))
    assert pp.mean_distance_error(y_int, np.round(y_pred)) == (dist * valid).sum() / valid.sum()


def test_eval_singleperson_pckh_equals_the_reference(cuda):
    """exp/common/mpii_tools.py:93-129: the model's float32 predictions, widened on the device, score exactly what the
    reference's transform_pose_sequence + pckh score on the same predictions"""
    from deephar_b200 import postprocess as pp
    from deephar_b200 import reception
    from oracle import synth
    m = reception.build((64, 64, 3), num_joints=16, dim=2, num_context_per_joint=2, num_blocks=2, ksize=(3, 3),
                        concat_pose_confidence=False).init_synthetic_weights(5)
    n = 12
    x = synth.synth_frames(n, 64, 64, seed=9)
    rng = np.random.default_rng(1)
    A = _affines(rng, n)
    pval = rng.uniform(0.2, 0.8, (n, 16, 2))
    head = rng.uniform(3, 8, (n, 1))
    scores = pp.eval_singleperson_pckh(m, x, pval, A, head, batch_size=4, refp=0.5, pred_per_block=2)
    outs = [np.concatenate(o) for o in zip(*[m.predict(x[i:i + 4], batch_size=4) for i in range(0, n, 4)])]
    y_true, _ = ref_transform(A, pval, True)
    for b in range(2):
        y_pred, _ = ref_transform(A, outs[2 * b][:, :, :2], True)
        hit, valid, _ = ref_measures(y_true[:, USED], y_pred[:, USED], head, 0.5)
        assert scores[b] == hit.sum() / valid.sum()
