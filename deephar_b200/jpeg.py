"""Baseline JPEG decoding on the GPU, bit-identical to Pillow, in front of the input pipeline.

    frames = jpeg.decode(paths)                       # device uint8 (H, W, 3) tensors
    frames, afmat = FramePipeline(...).from_jpeg(paths, objpos, winsize)

`decode(sources)[i]` equals `np.asarray(Image.open(sources[i]).convert('RGB'))` for every input `ImageDecoder`
accepts.  The marker parser below decides per file: 8-bit sequential Huffman-coded files with one interleaved scan,
grey or JFIF YCbCr with luma sampling 1x1, 2x1 or 2x2 and chroma 1x1 (4:4:4, 4:2:2, 4:2:0), restart markers or
not, are decoded by csrc/jpeg.cu; everything else (progressive, arithmetic-coded, 12-bit, lossless, CMYK / YCCK,
Adobe RGB, 4:4:0, 4:1:1, PNG, truncated files, ...) is decoded by Pillow on the host exactly as
`preprocess.ImageDecoder` does.  Files the kernels flag (a bad Huffman code, an interval that runs out of data, an
IDCT outside the range where libjpeg-turbo's C and SIMD IDCTs agree -- oracle/jpeg.py) are re-decoded by Pillow after
one status read-back, so the caller gets Pillow's pixels, or Pillow's exception.  The tables, per-image geometry and
the entropy-coded bytes of a batch go up in one pinned upload.
"""
import ctypes as C
import functools
import io
import os
import re

import numpy as np

from . import preprocess

ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20,
                   13, 6, 7, 14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52,
                   45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63], np.int64)     # zigzag index -> natural index
SAMPLINGS = {(1, 1), (2, 1), (2, 2)}
STAGES = ('entropy', 'idct', 'color')
_MARKER = re.compile(rb'\xff[^\x00]')       # in entropy-coded data: a marker (0xFF 0x00 is a stuffed 0xFF)


class Frame(object):
    """A file the GPU decoder takes: geometry, tables (natural-order quantisation, (bits, vals) Huffman) and the
    entropy-coded segments as byte ranges of `data[scan:scan_end]`."""

    def __init__(self, **kw):
        self.__dict__.update(kw)


class Host(object):
    """A file Pillow decodes, and why."""

    def __init__(self, reason):
        self.reason = reason


def huffman_table(bits, vals):
    """Canonical code assignment of one DHT table (ITU T.81 Annex C) -> dict(lut (512,) uint16: next 9 bits ->
    (length << 8) | symbol or 0, maxcode (18,) int32 and valoff (18,) int32 per length, vals (256,) uint8,
    codes [(length, code, symbol)]).  ValueError for a table libjpeg refuses.  Read-only and shared: files from one
    encoder repeat the same tables, which are built once."""
    return _huffman_table(bytes(bytearray(bits)), bytes(bytearray(vals)))


@functools.lru_cache(maxsize=1024)
def _huffman_table(bits, vals):
    bits, vals = list(bits), list(vals)
    if len(bits) != 16 or sum(bits) > 256 or len(vals) < sum(bits):
        raise ValueError('bad Huffman table')
    lut = np.zeros(512, np.uint16)
    maxcode = np.full(18, -1, np.int32)
    valoff = np.zeros(18, np.int32)
    codes, code, k = [], 0, 0
    for length in range(1, 17):
        n = bits[length - 1]
        if n:
            maxcode[length], valoff[length] = code + n - 1, k - code
        for j in range(n):
            codes.append((length, code + j, vals[k + j]))
            if length <= 9:
                lut[(code + j) << (9 - length):(code + j + 1) << (9 - length)] = (length << 8) | vals[k + j]
        code, k = code + n, k + n
        if code >= (1 << length):
            raise ValueError('bad Huffman table: codes overflow length %d' % length)
        code <<= 1
    out = np.zeros(256, np.uint8)
    out[:len(vals[:256])] = vals[:256]
    for a in (lut, maxcode, valoff, out):
        a.setflags(write=False)
    return dict(lut=lut, maxcode=maxcode, valoff=valoff, vals=out, codes=tuple(codes))


def parse(data):
    """Markers of one file -> Frame (the GPU decodes it) or Host (Pillow does).  Never raises for bad input: Pillow
    decides what a broken file does."""
    try:
        return _parse(bytes(data) if not isinstance(data, bytes) else data)
    except (IndexError, ValueError) as e:
        return Host('unreadable markers: %s' % e)


def _parse(data):
    n = len(data)
    if n < 4 or data[0] != 0xFF or data[1] != 0xD8:
        return Host('not a JPEG')
    p, qt, dc, ac, dri, jfif, adobe, sof = 2, {}, {}, {}, 0, False, None, None
    while True:
        if p + 4 > n or data[p] != 0xFF:
            return Host('truncated or malformed header')
        while p < n and data[p] == 0xFF:
            p += 1
        m = data[p]
        ln = (data[p + 1] << 8) | data[p + 2]
        if ln < 2 or p + 1 + ln > n:
            return Host('truncated header')
        seg, p = data[p + 3:p + 1 + ln], p + 1 + ln
        if m == 0xDB:
            q = 0
            while q < len(seg):
                pq, tq = seg[q] >> 4, seg[q] & 15
                size = 128 if pq else 64
                if pq > 1 or tq > 3 or q + 1 + size > len(seg):
                    return Host('bad DQT')
                v = np.frombuffer(seg[q + 1:q + 1 + size], '>u2' if pq else 'u1').astype(np.uint16)
                qt[tq] = np.zeros(64, np.uint16)
                qt[tq][ZIGZAG] = v
                q += 1 + size
        elif m == 0xC4:
            q = 0
            while q < len(seg):
                tc, th = seg[q] >> 4, seg[q] & 15
                bits = list(seg[q + 1:q + 17])
                cnt = sum(bits)
                if tc > 1 or th > 3 or len(bits) != 16 or cnt > 256 or q + 17 + cnt > len(seg):
                    return Host('bad DHT')
                (ac if tc else dc)[th] = (bytes(bits), bytes(seg[q + 17:q + 17 + cnt]))
                q += 17 + cnt
        elif m in (0xC0, 0xC1):
            if sof is not None or len(seg) < 6:
                return Host('bad SOF')
            nf = seg[5]
            if len(seg) < 6 + 3 * nf:
                return Host('bad SOF')
            sof = dict(prec=seg[0], h=(seg[1] << 8) | seg[2], w=(seg[3] << 8) | seg[4],
                       comps=[(seg[6 + 3 * i], seg[7 + 3 * i] >> 4, seg[7 + 3 * i] & 15, seg[8 + 3 * i])
                              for i in range(nf)])
        elif m == 0xDD:
            if len(seg) < 2:
                return Host('bad DRI')
            dri = (seg[0] << 8) | seg[1]
        elif m == 0xE0:
            jfif = jfif or (len(seg) >= 14 and seg[:5] == b'JFIF\x00')
        elif m == 0xEE:
            if len(seg) >= 12 and seg[:5] == b'Adobe':
                adobe = seg[11]
        elif 0xE1 <= m <= 0xEF or m == 0xFE:
            pass
        elif m == 0xDA:
            return _scan(data, p, seg, sof, qt, dc, ac, dri, jfif, adobe)
        else:
            return Host('marker 0x%02X (not baseline / extended sequential Huffman)' % m)


def _scan(data, p, sos, sof, qt, dc, ac, dri, jfif, adobe):
    if sof is None:
        return Host('no SOF0 / SOF1 before the scan')
    comps, h, w = sof['comps'], sof['h'], sof['w']
    if sof['prec'] != 8:
        return Host('%d-bit samples' % sof['prec'])
    if h < 1 or w < 1:
        return Host('empty image or height in a DNL marker')
    if len(comps) not in (1, 3) or len({c[0] for c in comps}) != len(comps):
        return Host('%d components' % len(comps))
    if any(not (1 <= c[1] <= 4 and 1 <= c[2] <= 4) for c in comps):
        return Host('bad sampling factors')
    if len(comps) == 3:
        if (comps[0][1], comps[0][2]) not in SAMPLINGS or any((c[1], c[2]) != (1, 1) for c in comps[1:]):
            return Host('sampling %s' % [(c[1], c[2]) for c in comps])
        ids = tuple(c[0] for c in comps)
        if not jfif and (adobe == 0 or (adobe is None and ids == (82, 71, 66))):
            return Host('RGB colour space')
    ns = sos[0]
    if ns != len(comps) or len(sos) < 4 + 2 * ns:
        return Host('scan does not hold every component')
    scan = [(sos[1 + 2 * i], sos[2 + 2 * i] >> 4, sos[2 + 2 * i] & 15) for i in range(ns)]
    if [s[0] for s in scan] != [c[0] for c in comps]:
        return Host('scan component order')
    if (sos[1 + 2 * ns], sos[2 + 2 * ns], sos[3 + 2 * ns]) != (0, 63, 0):
        return Host('not a sequential scan')
    for c, (_, td, ta) in zip(comps, scan):
        if c[3] not in qt or td not in dc or ta not in ac:
            return Host('undefined table')
        if any(v > 15 for v in dc[td][1]):
            return Host('DC symbol above 15')
    tables = {}
    try:
        for _, td, ta in scan:
            tables[('dc', td)] = huffman_table(*dc[td])
            tables[('ac', ta)] = huffman_table(*ac[ta])
    except ValueError as e:
        return Host(str(e))
    if len(comps) == 1:
        hs = vs = 1
        mcus_x, mcus_y = -(-w // 8), -(-h // 8)
    else:
        hs, vs = comps[0][1], comps[0][2]
        mcus_x, mcus_y = -(-w // (8 * hs)), -(-h // (8 * vs))
    # entropy-coded data: up to the first marker that is not RSTn; 0xFF 0x00 is a stuffed 0xFF
    total = mcus_x * mcus_y
    nseg = -(-total // dri) if dri else 1
    rst, end = [], None
    for mo in _MARKER.finditer(data, p):
        code = data[mo.start() + 1]
        if code == 0xFF:
            return Host('fill bytes inside the scan')
        if 0xD0 <= code <= 0xD7:
            if code != 0xD0 + len(rst) % 8 or len(rst) >= nseg - 1:
                return Host('restart markers out of sequence')
            rst.append(mo.start() - p)
            continue
        if code != 0xD9:
            return Host('marker 0x%02X after the scan (more than one scan)' % code)
        end = mo.start() - p
        break
    if end is None:
        return Host('scan not terminated (truncated file)')
    if len(rst) != nseg - 1:
        return Host('restart markers out of sequence')
    rst = np.array(rst, np.int64)
    begins = np.concatenate([[0], rst + 2]).astype(np.int64)
    ends = np.concatenate([rst, [end]]).astype(np.int64)
    per = dri if dri else total
    mcu0 = np.arange(nseg, dtype=np.int64) * per
    return Frame(h=h, w=w, ncomp=len(comps), hs=hs, vs=vs, mcus_x=mcus_x, mcus_y=mcus_y,
                 qt=[qt[c[3]] for c in comps], dc=[tables[('dc', s_[1])] for s_ in scan],
                 ac=[tables[('ac', s_[2])] for s_ in scan], dc_key=[dc[s_[1]] for s_ in scan],
                 ac_key=[ac[s_[2]] for s_ in scan], dri=dri, scan=p, scan_end=p + end,
                 segments=np.stack([begins, ends, mcu0, np.minimum(per, total - mcu0)], axis=1))


def _align(n, a=16):
    return n + (-n) % a


class Item(object):
    """One source of a batch: its bytes, its path (None for in-memory bytes), the parse, the output shape and the
    byte offset of its RGB image in the output arena."""

    def __init__(self, src):
        if isinstance(src, (bytes, bytearray, memoryview)):
            self.path, self.data = None, bytes(src)
        else:
            self.path = os.fspath(src)
            with open(self.path, 'rb') as f:
                self.data = f.read()
        self.frame = parse(self.data)
        self.gpu = isinstance(self.frame, Frame)
        if self.gpu:
            self.shape = (self.frame.h, self.frame.w, 3)
        else:
            self.shape = preprocess._probe(self._pillow_src()) + (3,)      # header only; Pillow's errors propagate
        self.out = 0

    def _pillow_src(self):
        return self.path if self.path is not None else io.BytesIO(self.data)

    def pillow(self):
        a = preprocess._decode_one(self._pillow_src())
        if a.shape != self.shape:
            raise ValueError('%s: decoded %s, its header announced %s' % (self.path or '<bytes>', a.shape, self.shape))
        return a


def pack(frames, ffi):
    """Host tables of a batch of Frames -> (images, segments, huff, qtab, data chunks, workspace sizes) with every
    offset relative to its own array; Huffman and quantisation tables shared between files are uploaded once."""
    n = len(frames)
    images = (ffi.dh_jpeg_image * max(n, 1))()
    huff_idx, q_idx, huffs, qts, segs, chunks = {}, {}, [], [], [], []
    data_pos = coef_pos = plane_pos = 0
    max_blocks = 0

    def table(key, t):
        if key not in huff_idx:
            huff_idx[key] = len(huffs)
            huffs.append(t)
        return huff_idx[key]

    for i, f in enumerate(frames):
        im = images[i]
        im.data, im.h, im.w, im.ncomp, im.hs, im.vs = data_pos, f.h, f.w, f.ncomp, f.hs, f.vs
        im.mcus_x, im.mcus_y = f.mcus_x, f.mcus_y
        nb = 0
        for c in range(f.ncomp):
            hs, vs = (f.hs, f.vs) if c == 0 else (1, 1)
            bw, bh = f.mcus_x * hs, f.mcus_y * vs
            im.bw[c], im.bh[c] = bw, bh
            im.coef[c], im.plane[c] = coef_pos, plane_pos
            coef_pos += bw * bh * 64
            plane_pos += _align(bw * bh * 64)
            nb += bw * bh
            key = f.qt[c].tobytes()
            if key not in q_idx:
                q_idx[key] = len(qts)
                qts.append(f.qt[c])
            im.qt[c] = q_idx[key]
            im.dc[c] = table(('dc',) + f.dc_key[c], f.dc[c])
            im.ac[c] = table(('ac',) + f.ac_key[c], f.ac[c])
        im.nblocks = nb
        max_blocks = max(max_blocks, nb)
        sg = f.segments.copy()
        sg[:, :2] += data_pos
        segs.append(np.concatenate([sg[:, :2], np.stack([np.full(len(sg), i), sg[:, 2], sg[:, 3],
                                                          np.zeros(len(sg), np.int64)], 1)], 1))
        chunks.append((data_pos, f.scan, f.scan_end))
        data_pos += _align(f.scan_end - f.scan)
    seg = np.concatenate(segs) if segs else np.zeros((0, 6), np.int64)
    # dh_jpeg_segment = int64 begin, end; int32 image, mcu0, mcus, pad
    seg_bytes = np.zeros(len(seg), dtype=[('b', '<i8'), ('e', '<i8'), ('i', '<i4'), ('m', '<i4'), ('c', '<i4'),
                                          ('p', '<i4')])
    for k, name in enumerate(['b', 'e', 'i', 'm', 'c', 'p']):
        seg_bytes[name] = seg[:, k]
    huff = (ffi.dh_jpeg_huff * max(len(huffs), 1))()
    for k, t in enumerate(huffs):
        C.memmove(huff[k].lut, t['lut'].ctypes.data, 1024)
        C.memmove(huff[k].maxcode, t['maxcode'].ctypes.data, 72)
        C.memmove(huff[k].valoff, t['valoff'].ctypes.data, 72)
        C.memmove(huff[k].vals, t['vals'].ctypes.data, 256)
    qtab = np.concatenate(qts) if qts else np.zeros(64, np.uint16)
    return dict(images=images, segments=seg_bytes, huff=huff, n_huff=len(huffs), qtab=qtab, chunks=chunks,
                data_bytes=data_pos, coef_elems=coef_pos, plane_bytes=plane_pos, max_blocks=max_blocks)


class JpegDecoder(object):
    """Batched decoder bound to one device: grow-only pinned staging and device workspace, reused across calls.

        dec = JpegDecoder()
        images = dec(paths)            # list of device uint8 (H, W, 3) tensors

    `time_stages = True` puts CUDA events around the three kernels; `stage_ms` then holds their times of the last
    call (the stages run back to back either way)."""

    def __init__(self, device='cuda:0', ctx=None):
        import torch
        from . import _ffi
        self._torch, self._ffi = torch, _ffi
        self.device = torch.device(device)
        self._ctx = ctx
        self._host = self._dev = self._uploaded = None
        self._work = None
        self._status = None
        self.time_stages = False
        self.stage_ms = None
        self.h2d_bytes = 0
        self.launches = 0
        self.host_decoded = []          # indices of the last call's images that Pillow decoded

    def _context(self):
        if self._ctx is None:
            if not self._torch.cuda.is_available():
                raise self._ffi.DeepharB200Error('deephar_b200.jpeg needs a CUDA device; there is no CPU fallback')
            self._ctx = self._ffi.Context(self.device.index or 0)
        return self._ctx

    def _staging(self, nbytes):
        torch = self._torch
        if self._host is None or self._host.numel() < nbytes:
            cap = int(nbytes * 1.25) + 4096
            self._host = torch.empty(cap, dtype=torch.uint8).pin_memory()
            self._dev = torch.empty(cap, dtype=torch.uint8, device=self.device)
            self._uploaded = torch.cuda.Event()
        else:
            self._uploaded.synchronize()
        return self._host[:nbytes], self._dev

    def _workspace(self, nbytes):
        torch = self._torch
        if self._work is None or self._work.numel() < nbytes:
            self._work = torch.empty(int(nbytes * 1.25) + 4096, dtype=torch.uint8, device=self.device)
        return self._work

    def plan(self, sources):
        """Read and parse every source; the output offsets are those of one packed arena of all images."""
        items = [Item(s) for s in sources]
        pos = 0
        for it in items:
            it.out = pos
            pos += _align(int(np.prod(it.shape)))
        return items, pos

    def launch(self, items, arena, extra=()):
        """Upload the batch (and the `extra` byte arrays after it, in the same copy) and queue the decode of the GPU
        items into `arena` (device uint8).  -> (state for finish(), device addresses of the extra arrays)."""
        torch, ffi = self._torch, self._ffi
        ctx = self._context()
        gpu = [k for k, it in enumerate(items) if it.gpu]
        pk = pack([items[k].frame for k in gpu], ffi)
        for j, k in enumerate(gpu):
            pk['images'][j].out = items[k].out
        n = len(gpu)
        parts = [np.frombuffer(pk['images'], np.uint8, count=C.sizeof(ffi.dh_jpeg_image) * n),
                 pk['segments'].view(np.uint8).reshape(-1),
                 np.frombuffer(pk['huff'], np.uint8, count=C.sizeof(ffi.dh_jpeg_huff) * pk['n_huff']),
                 pk['qtab'].view(np.uint8)] + [np.asarray(e).view(np.uint8).reshape(-1) for e in extra]
        offs, pos = [], 0
        for a in parts:
            offs.append(pos)
            pos += _align(a.size)
        o_data = pos
        total = o_data + pk['data_bytes']
        host, dev = self._staging(total)
        hv = host.numpy()
        for a, o in zip(parts, offs):
            hv[o:o + a.size] = a
        for (dpos, b, e), k in zip(pk['chunks'], gpu):
            hv[o_data + dpos:o_data + dpos + (e - b)] = np.frombuffer(items[k].data, np.uint8, count=e - b, offset=b)
        coef_bytes = _align(pk['coef_elems'] * 2)
        work = self._workspace(coef_bytes + pk['plane_bytes'] + _align(4 * max(n, 1)))
        base, wb = dev.data_ptr(), work.data_ptr()
        b = ffi.dh_jpeg_batch(images=base + offs[0], segments=base + offs[1], huff=base + offs[2],
                              qtab=base + offs[3], data=base + o_data, coef=wb, planes=wb + coef_bytes,
                              out=arena.data_ptr(), status=wb + coef_bytes + pk['plane_bytes'],
                              coef_elems=pk['coef_elems'], n_images=n, n_segments=len(pk['segments']),
                              max_blocks=pk['max_blocks'],
                              max_h=max([items[k].shape[0] for k in gpu], default=0),
                              max_w=max([items[k].shape[1] for k in gpu], default=0))
        stream = torch.cuda.current_stream(self.device)
        if self._status is None or self._status.numel() < max(n, 1):
            self._status = torch.empty(max(n, 1) + 256, dtype=torch.int32).pin_memory()
        done = torch.cuda.Event()
        events = None
        with torch.cuda.device(self.device):
            dev[:total].copy_(host, non_blocking=True)
            self._uploaded.record(stream)
            if n:
                if self.time_stages:
                    events = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
                    events[0].record(stream)
                    for s in range(3):
                        self._ffi.check(ffi.lib().dh_jpeg_decode(ctx.handle, C.byref(b), 1 << s, stream.cuda_stream),
                                        'dh_jpeg_decode')
                        events[s + 1].record(stream)
                else:
                    self._ffi.check(ffi.lib().dh_jpeg_decode(ctx.handle, C.byref(b), 7, stream.cuda_stream),
                                    'dh_jpeg_decode')
                status = work[coef_bytes + pk['plane_bytes']:coef_bytes + pk['plane_bytes'] + 4 * n].view(torch.int32)
                self._status[:n].copy_(status, non_blocking=True)
                self.launches += 3
            done.record(stream)
        self.h2d_bytes = int(total)
        state = dict(items=items, gpu=gpu, done=done, events=events, arena=arena)
        return state, [base + o for o in offs[4:]]

    def finish(self, state):
        """Pillow decodes the items the GPU did not take (while the kernels run), one status read-back names the
        items the kernels flagged, and Pillow's pixels (or its exception) replace those."""
        torch = self._torch
        items, gpu, arena = state['items'], state['gpu'], state['arena']
        host = {}
        for k, it in enumerate(items):
            if not it.gpu:
                try:
                    host[k] = it.pillow()
                except Exception as e:          # raised below in source order
                    host[k] = e
        state['done'].synchronize()
        if state['events'] is not None:
            ev = state['events']
            self.stage_ms = {name: ev[s].elapsed_time(ev[s + 1]) for s, name in enumerate(STAGES)}
        status = self._status[:len(gpu)].numpy()
        for j, k in enumerate(gpu):
            if status[j]:
                host[k] = None
        self.host_decoded = sorted(host)
        with torch.cuda.device(self.device):
            for k in self.host_decoded:
                a = host[k]
                if isinstance(a, Exception):
                    raise a
                if a is None:
                    a = items[k].pillow()
                n = a.size
                arena[items[k].out:items[k].out + n].copy_(torch.from_numpy(np.array(a).reshape(-1)))
        return status

    def __call__(self, sources):
        torch = self._torch
        items, total = self.plan(sources)
        arena = torch.empty(max(total, 1), dtype=torch.uint8, device=self.device)
        if items:
            self.finish(self.launch(items, arena)[0])
        return [arena[it.out:it.out + int(np.prod(it.shape))].view(*it.shape) for it in items]


_DECODERS = {}


def decode(sources, device='cuda:0'):
    """Decode JPEG files / bytes (any other format Pillow reads too) -> list of device uint8 (H, W, 3) tensors, each
    equal to np.asarray(Image.open(source).convert('RGB'))."""
    import torch
    dev = torch.device(device)
    if dev not in _DECODERS:
        _DECODERS[dev] = JpegDecoder(dev)
    return _DECODERS[dev](sources)
