"""Evaluation-time input pipeline on the GPU (SURVEY.md 8 f4) -- the step in front of the forward path.

Mirrors what deephar/data/mpii.py:91-122 does per sample with the fixed (evaluation) data configuration,

    imgt = T(Image.open(...)); imgt.rotate_crop(0, objpos, winsize); imgt.resize(crop_resolution)
    [imgt.horizontal_flip()]; imgt.normalize_affinemap(); frame = normalize_channels(imgt.asarray(), chpower)

(deephar/utils/transform.py:46-134, 212-231) for a whole batch of decoded uint8 images in two kernel launches
(csrc/preprocess.cu, C ABI `dh_crop_resize_norm_u8`), writing the (N, H, W, 3) fp32 NHWC tensor the network reads and
returning the per-sample affine maps `afmat` the evaluator needs to carry predictions back to image coordinates.
`Image.resize(BILINEAR)` is Pillow's fixed-point two-pass resampler; its weight tables are computed here on the host
in double precision exactly as Pillow computes them, the pixel arithmetic runs on the device: uint8 results are
bit-identical to Pillow's, the float32 frames bit-identical to the reference's (tests/test_preprocess.py).

Only angle == 0 is supported (the evaluation configuration; rotation is training-time augmentation, SURVEY.md 8:
out of scope).  No CPU path: without the CUDA library the call raises.
"""
import ctypes as C
import functools

import numpy as np

PRECISION_BITS = 32 - 8 - 2


@functools.lru_cache(maxsize=4096)
def resample_tables(in_size, out_size):
    """Bilinear (triangle) resampling tables of one axis: bounds int32 (out, 2) = (first source index, tap count),
    coefs int32 (out, ksize) 22-bit fixed point.  Vectorised over the output index; the normalising sum is taken tap
    by tap in source order so that every double rounds as in Pillow."""
    in_size, out_size = int(in_size), int(out_size)
    if in_size < 1 or out_size < 1:
        raise ValueError('resample_tables: sizes must be positive, got %d -> %d' % (in_size, out_size))
    scale = in_size / out_size
    fscale = max(scale, 1.0)
    support = 1.0 * fscale
    ksize = int(np.ceil(support)) * 2 + 1
    centers = (np.arange(out_size, dtype=np.float64) + 0.5) * scale
    first = np.maximum(np.trunc(centers - support + 0.5).astype(np.int64), 0)
    last = np.minimum(np.trunc(centers + support + 0.5).astype(np.int64), in_size)
    count = last - first
    taps = np.arange(ksize, dtype=np.int64)[None, :]
    v = np.abs((taps + first[:, None] - centers[:, None] + 0.5) * (1.0 / fscale))
    w = np.where((v < 1.0) & (taps < count[:, None]), 1.0 - v, 0.0)
    total = np.zeros(out_size, np.float64)
    for t in range(ksize):
        total = total + w[:, t]
    w = np.where(total[:, None] != 0.0, w / np.where(total == 0.0, 1.0, total)[:, None], w)
    coefs = np.trunc(0.5 + w * float(1 << PRECISION_BITS)).astype(np.int32)
    bounds = np.stack([first, count], axis=1).astype(np.int32)
    bounds.setflags(write=False)
    coefs.setflags(write=False)
    return bounds, coefs


def crop_box(objpos, winsize):
    """transform.py:112-114 with angle 0: the integer (truncated) box [x0, y0, x1, y1] around `objpos`."""
    cx, cy = float(objpos[0]), float(objpos[1])
    ww, wh = (float(winsize), float(winsize)) if np.isscalar(winsize) else (float(winsize[0]), float(winsize[1]))
    return np.array([cx - ww / 2, cy - wh / 2, cx + ww / 2, cy + wh / 2], dtype=int)


def affine_map(box, crop_resolution, hflip):
    """The 3x3 `afmat` of the sample after crop -> resize -> [flip] -> normalize_affinemap (transform.py:5-44, 57-71,
    116-121): image pixel coordinates -> [0, 1]^2 of the network input."""
    def apply(t, a):
        return np.dot(t, a)

    def translate(x, y):
        t = np.eye(3)
        t[0, 2], t[1, 2] = x, y
        return t

    def scale(sx, sy):
        t = np.eye(3)
        t[0, 0], t[1, 1] = sx, sy
        return t

    cw, ch = int(box[2] - box[0]), int(box[3] - box[1])
    rw, rh = crop_resolution
    a = np.eye(3)
    a = apply(translate(-box[0], -box[1]), a)
    a = apply(scale(rw / cw, rh / ch), a)
    if hflip:
        a = apply(scale(-1, 1), a)
        a = apply(translate(rw, 0), a)
    return apply(scale(1 / rw, 1 / rh), a)


def mpii_windows(objpos, scale, dconf=None):
    """deephar/data/mpii.py:99-105: the crop window of an MPII single-person sample from its annotation --
    `scale` enlarged by 1.25, the centre moved 12 * scale down (+ scale * (transx, transy)), a square window of
    200 * dconf['scale'] * scale pixels.  objpos (N, 2), scale (N,); dconf = `dataconf.get_fixed_config()`.
    -> (objpos (N, 2), winsize (N,)) as FramePipeline takes them."""
    dconf = dconf or {'scale': 1, 'transx': 0, 'transy': 0}
    scale = 1.25 * np.asarray(scale, np.float64).reshape(-1)
    pos = np.array(objpos, dtype=np.float64).reshape(-1, 2)
    pos[:, 1] += 12 * scale
    pos += scale[:, None] * np.array([dconf['transx'], dconf['transy']], np.float64)
    return pos, 200 * dconf['scale'] * scale


def clip_frame_index(sequence_size, subsample, num_frames):
    """deephar/data/datasets.py:6-38 with random_clip=False: the frame indices of the evaluation clip of a video --
    `num_frames` frames `subsample` apart, centred; the step shrinks for short videos and videos shorter than the clip
    repeat frames (the index grid is stretched by 1.5 until it fits)."""
    if not (isinstance(subsample, (int, np.integer)) and subsample > 0):
        raise ValueError('clip_frame_index: subsample must be a positive integer')
    stretch, size = 1.0, float(sequence_size)
    while stretch * sequence_size < num_frames:
        stretch *= 1.5
    size = sequence_size * stretch
    subsample = min(int(subsample), int(size / num_frames))
    span = subsample * (num_frames - 1) + 1
    start = int((size - span) / 2)
    frames = list(range(start, start + span, subsample))
    return [int(f / stretch) for f in frames] if stretch > 1 else frames


def clip_window(image_size, dconf=None, bbox=None):
    """deephar/data/pennaction.py:118-134 (the same lines in data/ntu.py): the ONE crop window shared by all frames of an
    evaluation clip -- centre and size of `bbox` [x0, y0, x1, y1] (ground-truth or predicted), or, without one, a square
    of dconf['scale'] * max(w, h) around the image centre; windows thinner than 32 pixels become 32 x 32; the centre
    moves by scale * (transx, transy).  -> (objpos (2,), winsize (2,)) as FramePipeline takes them (repeat per frame)."""
    dconf = dconf or {'scale': 1, 'transx': 0, 'transy': 0}
    w, h = image_size
    if bbox is None:
        side = dconf['scale'] * max(w, h)
        objpos, winsize = np.array([w / 2, h / 2], np.float64), (side, side)
    else:
        bbox = np.asarray(bbox, np.float64)
        objpos = np.array([(bbox[0] + bbox[2]) / 2, (bbox[1] + bbox[3]) / 2])
        winsize = (bbox[2] - bbox[0], bbox[3] - bbox[1])
    if min(winsize) < 32:
        winsize = (32, 32)
    objpos = objpos + dconf['scale'] * np.array([dconf['transx'], dconf['transy']], np.float64)
    return objpos, np.array(winsize, np.float64)


def _decode_one(path):
    from PIL import Image
    with Image.open(path) as im:
        return np.asarray(im if im.mode == 'RGB' else im.convert('RGB'))


_ARENA = None       # shared anonymous mapping the decoder's workers write into (set in the parent before they are forked)


def _probe(path):
    from PIL import Image
    with Image.open(path) as im:        # header only
        return im.size[1], im.size[0]


def _decode_into(job):
    path, offset, nbytes = job
    a = _decode_one(path)
    if a.size != nbytes:
        raise ValueError('%s: decoded %d bytes, its header announced %d' % (path, a.size, nbytes))
    np.frombuffer(_ARENA, dtype=np.uint8, count=nbytes, offset=offset)[:] = a.reshape(-1)
    return a.shape


class ImageDecoder(object):
    """`Image.open(path)` of the reference's loaders (data/mpii.py:83, data/pennaction.py:152, data/ntu.py:221,
    data/human36m.py:110) for a whole batch: decoded RGB uint8 (H, W, 3) arrays in the order of the paths, ready for
    FramePipeline.  Decoding stays on the host and stays Pillow's (the frames must be the reference's, bit for bit), but
    one core decodes ~300-400 VGA JPEGs per second and the forward consumes thousands: the batch is spread over a pool of
    worker PROCESSES (Pillow holds the GIL while it decodes, threads do not scale), forked on first use and kept -- as
    torch's DataLoader forks its workers: they only ever run Pillow and never touch the parent's CUDA state.  The pixels
    come back through one shared anonymous mapping (`arena_mb`), not through pickles.  Grey-scale / palette files are
    converted to RGB (the models take 3 channels).

        decode = ImageDecoder(workers=16)
        frames, afmat = pipe(decode(paths), objpos, winsize)
    """

    def __init__(self, workers=None, arena_mb=256):
        import os
        self.workers = max(1, int(workers or min(32, os.cpu_count() or 1)))
        self.arena_bytes = int(arena_mb) << 20
        self._pool = None

    def _start(self):
        global _ARENA
        import mmap
        import multiprocessing
        self._arena = _ARENA = mmap.mmap(-1, self.arena_bytes)         # MAP_SHARED | MAP_ANONYMOUS: inherited by the fork
        self._pool = multiprocessing.get_context('fork').Pool(self.workers)
        _ARENA = None

    def __call__(self, paths):
        paths = [str(p) for p in paths]
        if self.workers == 1 or len(paths) < 2:
            return [_decode_one(p) for p in paths]
        if self._pool is None:
            self._start()
        chunk = max(1, len(paths) // (4 * self.workers))
        sizes = self._pool.map(_probe, paths, chunksize=chunk)
        out, i = [None] * len(paths), 0
        while i < len(paths):
            jobs, used = [], 0
            while i + len(jobs) < len(paths):                           # as many images as fit the arena
                h, w = sizes[i + len(jobs)]
                if used + h * w * 3 > self.arena_bytes:
                    break
                jobs.append((paths[i + len(jobs)], used, h * w * 3))
                used += h * w * 3
            if not jobs:                                                # one image larger than the arena
                out[i] = _decode_one(paths[i])
                i += 1
                continue
            shapes = self._pool.map(_decode_into, jobs, chunksize=max(1, len(jobs) // (4 * self.workers)))
            for k, ((_, off, n), shp) in enumerate(zip(jobs, shapes)):
                out[i + k] = np.frombuffer(self._arena, dtype=np.uint8, count=n, offset=off).reshape(shp).copy()
            i += len(jobs)
        return out

    def close(self):
        if self._pool is not None:
            self._pool.terminate()
            self._pool.join()
            self._pool = None
            self._arena.close()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:       # interpreter shutdown
            pass


def decode_images(paths, workers=1):
    """One-shot form of ImageDecoder (in-process by default; a pool started for one call costs more than it saves)."""
    with ImageDecoder(workers) as dec:
        return dec(paths)


class FramePipeline(object):
    """Batched evaluation input pipeline bound to one device.

        pipe = FramePipeline(crop_resolution=(256, 256))
        frames, afmat = pipe(images, objpos, winsize, hflip=0, channel_power=1)

    images: sequence of uint8 (H, W, 3) numpy arrays (decoded RGB, sizes may differ); objpos (N, 2); winsize scalar,
    (N,) or (N, 2).  frames: torch fp32 (N, res_h, res_w, 3) on the device; afmat: float64 (N, 3, 3).
    """

    def __init__(self, crop_resolution=(256, 256), device='cuda:0'):
        import torch
        from . import _ffi
        self._torch, self._ffi = torch, _ffi
        self.crop_resolution = (int(crop_resolution[0]), int(crop_resolution[1]))     # (w, h) as PIL
        self.device = torch.device(device)
        self._ctx = None
        self._host = self._dev = self._uploaded = None
        self.launches = 0
        self.h2d_bytes = 0

    def _context(self):
        if self._ctx is None:
            if not self._torch.cuda.is_available():
                raise self._ffi.DeepharB200Error('deephar_b200.preprocess needs a CUDA device; there is no CPU fallback')
            self._ctx = self._ffi.Context(self.device.index or 0)      # raises when the CUDA library is missing
        return self._ctx

    def _staging(self, nbytes):
        """Grow-only pinned host / device staging pair; reused only after the previous call's kernels consumed it."""
        torch = self._torch
        if self._host is None or self._host.numel() < nbytes:
            cap = int(nbytes * 1.25) + 4096
            self._host = torch.empty(cap, dtype=torch.uint8).pin_memory()
            self._dev = torch.empty(cap, dtype=torch.uint8, device=self.device)
            self._uploaded = torch.cuda.Event()
        else:
            self._uploaded.synchronize()
        return self._host[:nbytes], self._dev

    def plan(self, shapes, objpos, winsize, hflip=0):
        """Host-side geometry of one batch: -> (frame table, bounds, coefs, boxes, afmat, max crop height).  Source
        offsets in the table are relative to the start of the packed image buffer."""
        n = len(shapes)
        objpos = np.asarray(objpos, np.float64).reshape(n, 2)
        winsize = np.asarray(winsize, np.float64)
        winsize = np.broadcast_to(winsize.reshape(-1, 1) if winsize.ndim <= 1 else winsize, (n, 2))
        hflip = np.broadcast_to(np.asarray(hflip, np.int64), (n,))
        rw, rh = self.crop_resolution
        tables, b_parts, c_parts = {}, [], []
        b_len = c_len = 0
        frames = (self._ffi.dh_frame_src * max(n, 1))()
        boxes = np.zeros((n, 4), np.int64)
        afmat = np.zeros((n, 3, 3), np.float64)
        offset = max_ch = 0
        for i, (h, w) in enumerate(shapes):
            box = crop_box(objpos[i], winsize[i])
            cw, ch = int(box[2] - box[0]), int(box[3] - box[1])
            if cw < 1 or ch < 1:
                raise ValueError('sample %d: empty crop window %s' % (i, box.tolist()))
            slots = []
            for key in ((cw, rw), (ch, rh)):
                if key not in tables:
                    bounds, coefs = resample_tables(*key)
                    tables[key] = (b_len, c_len, coefs.shape[1])
                    b_parts.append(bounds.reshape(-1))
                    c_parts.append(coefs.reshape(-1))
                    b_len += bounds.size
                    c_len += coefs.size
                slots.append(tables[key])
            f = frames[i]
            f.data = offset
            f.h, f.w, f.stride = int(h), int(w), int(w) * 3
            f.x0, f.y0, f.cw, f.ch, f.hflip = int(box[0]), int(box[1]), cw, ch, int(hflip[i] == 1)
            f.kx_off, f.kx_coef_off, f.ksx = slots[0]
            f.ky_off, f.ky_coef_off, f.ksy = slots[1]
            boxes[i] = box
            afmat[i] = affine_map(box, self.crop_resolution, hflip[i] == 1)
            offset += int(h) * int(w) * 3
            max_ch = max(max_ch, ch)
        bounds = np.concatenate(b_parts) if b_parts else np.zeros(0, np.int32)
        coefs = np.concatenate(c_parts) if c_parts else np.zeros(0, np.int32)
        return frames, bounds, coefs, boxes, afmat, max_ch

    def __call__(self, images, objpos, winsize, hflip=0, channel_power=1, angle=0, out=None):
        torch = self._torch
        if np.any(np.asarray(angle) != 0):
            raise NotImplementedError('FramePipeline: only angle == 0 (the evaluation configuration) is supported')
        images = [np.ascontiguousarray(im) for im in images]
        for im in images:
            if im.dtype != np.uint8 or im.ndim != 3 or im.shape[2] != 3:
                raise ValueError('FramePipeline: images must be uint8 (H, W, 3), got %s %s' % (im.dtype, im.shape))
        n = len(images)
        rw, rh = self.crop_resolution
        frames, bounds, coefs, boxes, afmat, max_ch = self.plan([im.shape[:2] for im in images], objpos, winsize, hflip)
        ctx = self._context()
        if out is None:
            out = torch.empty((n, rh, rw, 3), dtype=torch.float32, device=self.device)
        elif tuple(out.shape) != (n, rh, rw, 3) or out.dtype != torch.float32 or not out.is_contiguous():
            raise ValueError('FramePipeline: out must be a contiguous fp32 (%d, %d, %d, 3) tensor' % (n, rh, rw))
        if n == 0:
            return out, afmat
        # one packed upload: [images | frame table | bounds | coefs], pinned -> device
        table = np.frombuffer(frames, dtype=np.uint8, count=C.sizeof(self._ffi.dh_frame_src) * n)
        px_bytes = sum(im.size for im in images)
        pad = (-px_bytes) % 16
        sizes = [px_bytes + pad, table.size + (-table.size) % 16, bounds.nbytes + (-bounds.nbytes) % 16, coefs.nbytes]
        host, dev = self._staging(sum(sizes))
        hv = host.numpy()
        pos = 0
        for im in images:
            hv[pos:pos + im.size] = im.reshape(-1)
            pos += im.size
        o_tab, o_b, o_c = sizes[0], sizes[0] + sizes[1], sizes[0] + sizes[1] + sizes[2]
        base = dev.data_ptr()
        for i in range(n):                                           # offsets -> device addresses
            frames[i].data = base + frames[i].data
        hv[o_tab:o_tab + table.size] = np.frombuffer(frames, dtype=np.uint8, count=table.size)
        hv[o_b:o_b + bounds.nbytes] = bounds.view(np.uint8)
        hv[o_c:o_c + coefs.nbytes] = coefs.view(np.uint8)
        stream = torch.cuda.current_stream(self.device)
        with torch.cuda.device(self.device):
            dev[:host.numel()].copy_(host, non_blocking=True)
            tmp_stride = max_ch * rw * 3
            tmp_stride += (-tmp_stride) % 16
            tmp = torch.empty(n * tmp_stride, dtype=torch.uint8, device=self.device)
            power = None
            if not (np.isscalar(channel_power) and channel_power == 1):
                power = (C.c_float * 3)(*np.broadcast_to(np.asarray(channel_power, np.float32), (3,)))
            rc = self._ffi.lib().dh_crop_resize_norm_u8(ctx.handle, base + o_tab, n, max_ch, base + o_b, base + o_c, rh, rw, power,
                                                        tmp.data_ptr(), tmp_stride, out.data_ptr(), stream.cuda_stream)
            self._ffi.check(rc, 'dh_crop_resize_norm_u8')
            self._uploaded.record(stream)       # staging pair is free again once the kernels have consumed it
            tmp.record_stream(stream)
        self.launches += 2
        self.h2d_bytes = int(sum(sizes))
        return out, afmat

    def from_device(self, images, objpos, winsize, hflip=0, channel_power=1, out=None, max_crop=None):
        """Frames from images already on the device, with the geometry computed there too (dh_prepare_frames_u8): no
        pixel crosses PCIe and no per-frame Python runs.  images: CUDA uint8 (H, W, 3) tensors (rows may be padded),
        e.g. jpeg.decode's; objpos (N, 2), winsize scalar, (N,) or (N, 2), hflip scalar or (N,), as __call__ takes them,
        as numpy arrays or as CUDA tensors.  max_crop = (w, h) bounds the crop windows and sizes the scratch; it is
        required when a box is a CUDA tensor (reading the boxes back would synchronise), and defaults to the largest
        window of host boxes.  -> (frames, afmat, status), all on the device: frames fp32 (N, res_h, res_w, 3) equal to
        __call__'s, afmat float64 (N, 3, 3) equal to affine_map's, status int32 (N,) with the _ffi.FRAME_* bits of a
        frame whose window is empty, larger than max_crop or not finite -- that frame and its afmat are NaN."""
        torch, ffi = self._torch, self._ffi
        n = len(images)
        rw, rh = self.crop_resolution
        for im in images:
            if (not torch.is_tensor(im) or not im.is_cuda or im.dtype != torch.uint8 or im.dim() != 3 or im.shape[2] != 3
                    or im.stride(2) != 1 or im.stride(1) != 3):
                raise ValueError('FramePipeline.from_device: images must be CUDA uint8 (H, W, 3) tensors with packed pixels')
        on_device = [torch.is_tensor(a) for a in (objpos, winsize, hflip)]
        if any(on_device) and max_crop is None:
            raise ValueError('FramePipeline.from_device: max_crop is required when the boxes are on the device')
        if not on_device[0]:
            objpos = np.asarray(objpos, np.float64).reshape(n, 2)
        if not on_device[1]:
            winsize = np.asarray(winsize, np.float64)
            winsize = np.broadcast_to(winsize.reshape(-1, 1) if winsize.ndim <= 1 else winsize, (n, 2))
        if max_crop is None:
            max_crop = (1, 1)
            with np.errstate(invalid='ignore', over='ignore'):
                edges = np.concatenate([objpos - winsize / 2, objpos + winsize / 2], axis=1)
            ok = np.all((edges > -2147483649.0) & (edges < 2147483648.0), axis=1)       # NaN: False
            if ok.any():
                box = np.trunc(edges[ok])
                max_crop = (max(1, int((box[:, 2] - box[:, 0]).max())), max(1, int((box[:, 3] - box[:, 1]).max())))
        mw, mh = int(max_crop[0]), int(max_crop[1])
        if out is None:
            out = torch.empty((n, rh, rw, 3), dtype=torch.float32, device=self.device)
        elif tuple(out.shape) != (n, rh, rw, 3) or out.dtype != torch.float32 or not out.is_contiguous():
            raise ValueError('FramePipeline: out must be a contiguous fp32 (%d, %d, %d, 3) tensor' % (n, rh, rw))
        afmat = torch.empty((n, 3, 3), dtype=torch.float64, device=self.device)
        status = torch.empty(n, dtype=torch.int32, device=self.device)
        if n == 0:
            return out, afmat, status
        ctx = self._context()
        lib = ffi.lib()
        ws_bytes = lib.dh_prepare_frames_workspace(n, mw, mh, rh, rw)
        if ws_bytes < 0:
            ffi.check(-1, 'dh_prepare_frames_workspace')
        # the box records: image fields from the tensors, then objpos / winsize / hflip from wherever they are
        rec = (ffi.dh_frame_box * n)()
        for i, im in enumerate(images):
            rec[i].data, rec[i].h, rec[i].w, rec[i].stride = im.data_ptr(), im.shape[0], im.shape[1], im.stride(0)
        host = np.frombuffer(rec, np.uint8).reshape(n, C.sizeof(ffi.dh_frame_box))
        geo = host[:, ffi.dh_frame_box.objpos.offset:].view(np.float64)               # (n, 4): objpos, winsize
        if not on_device[0]:
            geo[:, 0:2] = objpos
        if not on_device[1]:
            geo[:, 2:4] = winsize
        if not on_device[2]:
            host[:, ffi.dh_frame_box.hflip.offset:ffi.dh_frame_box.hflip.offset + 4].view(np.int32)[:, 0] = \
                np.broadcast_to(np.asarray(hflip) == 1, (n,))
        stream = torch.cuda.current_stream(self.device)
        with torch.cuda.device(self.device):
            boxes = torch.from_numpy(host).pin_memory().to(self.device, non_blocking=True)
            if any(on_device):
                dgeo = boxes[:, ffi.dh_frame_box.objpos.offset:].view(torch.float64)
                if on_device[0]:
                    dgeo[:, 0:2] = objpos.reshape(n, 2).to(self.device, torch.float64)
                if on_device[1]:
                    wsz = winsize.to(self.device, torch.float64)
                    dgeo[:, 2:4] = (wsz.reshape(-1, 1) if wsz.dim() <= 1 else wsz).expand(n, 2)
                if on_device[2]:
                    o = ffi.dh_frame_box.hflip.offset
                    boxes[:, o:o + 4].view(torch.int32)[:, 0] = (hflip.to(self.device) == 1).to(torch.int32).expand(n)
            ws = torch.empty(ws_bytes, dtype=torch.uint8, device=self.device)
            power = None
            if not (np.isscalar(channel_power) and channel_power == 1):
                power = (C.c_float * 3)(*np.broadcast_to(np.asarray(channel_power, np.float32), (3,)))
            rc = lib.dh_prepare_frames_u8(ctx.handle, boxes.data_ptr(), n, mw, mh, rh, rw, power, ws.data_ptr(), ws_bytes,
                                          out.data_ptr(), afmat.data_ptr(), status.data_ptr(), stream.cuda_stream)
            ffi.check(rc, 'dh_prepare_frames_u8')
            ws.record_stream(stream)
            boxes.record_stream(stream)
            for im in images:
                im.record_stream(stream)
        self.launches += 3
        self.h2d_bytes = host.nbytes
        return out, afmat, status

    def from_jpeg(self, sources, objpos, winsize, hflip=0, channel_power=1, out=None):
        """The same result as `self(decode_images(sources), objpos, winsize, hflip, channel_power)`, with the JPEG
        decode on the GPU (deephar_b200/jpeg.py): the frame table points into the decoded images on the device
        instead of into uploaded pixels, so only the compressed bytes cross PCIe.  sources: paths or bytes, any
        format Pillow reads (what the GPU decoder does not take, Pillow decodes)."""
        from . import jpeg
        torch = self._torch
        ctx = self._context()
        if getattr(self, '_jpeg', None) is None:
            self._jpeg = jpeg.JpegDecoder(self.device, ctx=ctx)
        dec = self._jpeg
        items, total = dec.plan(sources)
        n = len(items)
        rw, rh = self.crop_resolution
        frames, bounds, coefs, boxes, afmat, max_ch = self.plan([it.shape[:2] for it in items], objpos, winsize, hflip)
        if out is None:
            out = torch.empty((n, rh, rw, 3), dtype=torch.float32, device=self.device)
        elif tuple(out.shape) != (n, rh, rw, 3) or out.dtype != torch.float32 or not out.is_contiguous():
            raise ValueError('FramePipeline: out must be a contiguous fp32 (%d, %d, %d, 3) tensor' % (n, rh, rw))
        if n == 0:
            return out, afmat
        arena = torch.empty(total, dtype=torch.uint8, device=self.device)
        for i, it in enumerate(items):
            frames[i].data = arena.data_ptr() + it.out
        table = np.frombuffer(frames, dtype=np.uint8, count=C.sizeof(self._ffi.dh_frame_src) * n)
        state, (d_tab, d_b, d_c) = dec.launch(items, arena, extra=(table, bounds, coefs))   # one upload
        dec.finish(state)
        stream = torch.cuda.current_stream(self.device)
        with torch.cuda.device(self.device):
            tmp_stride = max_ch * rw * 3
            tmp_stride += (-tmp_stride) % 16
            tmp = torch.empty(n * tmp_stride, dtype=torch.uint8, device=self.device)
            power = None
            if not (np.isscalar(channel_power) and channel_power == 1):
                power = (C.c_float * 3)(*np.broadcast_to(np.asarray(channel_power, np.float32), (3,)))
            rc = self._ffi.lib().dh_crop_resize_norm_u8(ctx.handle, d_tab, n, max_ch, d_b, d_c, rh, rw, power,
                                                        tmp.data_ptr(), tmp_stride, out.data_ptr(), stream.cuda_stream)
            self._ffi.check(rc, 'dh_crop_resize_norm_u8')
            tmp.record_stream(stream)
            arena.record_stream(stream)
        self.launches += 2
        self.h2d_bytes = dec.h2d_bytes
        return out, afmat
