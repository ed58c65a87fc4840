"""Integer model of baseline JPEG decoding as libjpeg-turbo performs it in its default configuration (the decoder
behind Pillow's `Image.open(...).convert('RGB')`): Huffman decoding, dequantisation, the accurate integer IDCT
(`JDCT_ISLOW`) with its post-IDCT range-limit table, "fancy" triangle upsampling of 4:2:2 / 4:2:0 chroma and the
integer YCbCr -> RGB tables (SCALEBITS 16); `Deferred` marks the files whose IDCT leaves the range in which
libjpeg-turbo's C and SIMD IDCTs agree (see AGREE).  Pure Python / numpy and written for clarity, not speed: images up to
about 64 x 64.  It covers the files the GPU decoder (deephar_b200/jpeg.py, csrc/jpeg.cu) takes -- 8-bit sequential
Huffman, one interleaved scan, grey or YCbCr with luma sampling 1x1 / 2x1 / 2x2 and chroma 1x1, optional restart
markers -- and raises ValueError for anything else.  tests/test_jpeg.py pins it against Pillow bit for bit.
"""
import struct

import numpy as np

ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20,
                   13, 6, 7, 14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52,
                   45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63], np.int64)     # zigzag index -> natural index


def parse(data):
    """Markers up to the single scan -> dict(h, w, comps [(id, hs, vs, tq)], qt {tq: natural-order (64,)},
    dc / ac {th: (bits, vals)}, scan [(ci, td, ta)], dri, data (entropy-coded bytes up to the marker after the scan))."""
    data = bytes(data)
    if data[:2] != b'\xff\xd8':
        raise ValueError('not a JPEG')
    p, hdr = 2, dict(qt={}, dc={}, ac={}, dri=0)
    while True:
        while data[p] == 0xFF and data[p + 1] == 0xFF:
            p += 1
        if data[p] != 0xFF:
            raise ValueError('marker expected at %d' % p)
        m = data[p + 1]
        ln = struct.unpack('>H', data[p + 2:p + 4])[0]
        seg = data[p + 4:p + 2 + ln]
        p += 2 + ln
        if m == 0xDB:
            q = 0
            while q < len(seg):
                pq, tq = seg[q] >> 4, seg[q] & 15
                n = 128 if pq else 64
                v = np.frombuffer(seg[q + 1:q + 1 + n], '>u2' if pq else 'u1').astype(np.int64)
                hdr['qt'][tq] = np.zeros(64, np.int64)
                hdr['qt'][tq][ZIGZAG] = v
                q += 1 + n
        elif m == 0xC4:
            q = 0
            while q < len(seg):
                tc, th = seg[q] >> 4, seg[q] & 15
                bits = list(seg[q + 1:q + 17])
                vals = list(seg[q + 17:q + 17 + sum(bits)])
                (hdr['ac'] if tc else hdr['dc'])[th] = (bits, vals)
                q += 17 + sum(bits)
        elif m in (0xC0, 0xC1):
            if seg[0] != 8:
                raise ValueError('precision %d' % seg[0])
            hdr['h'], hdr['w'] = struct.unpack('>HH', seg[1:5])
            hdr['comps'] = [(seg[6 + 3 * i], seg[7 + 3 * i] >> 4, seg[7 + 3 * i] & 15, seg[8 + 3 * i])
                            for i in range(seg[5])]
        elif m == 0xDD:
            hdr['dri'] = struct.unpack('>H', seg[:2])[0]
        elif m == 0xDA:
            hdr['scan'] = [(seg[1 + 2 * i], seg[2 + 2 * i] >> 4, seg[2 + 2 * i] & 15) for i in range(seg[0])]
            end = p
            while not (data[end] == 0xFF and data[end + 1] not in (0x00, 0xFF) and not 0xD0 <= data[end + 1] <= 0xD7):
                end += 1
            hdr['data'] = data[p:end]
            return hdr
        elif 0xC2 <= m <= 0xCF and m not in (0xC4, 0xC8, 0xCC):
            raise ValueError('SOF%d not modelled' % (m - 0xC0))


class _Bits(object):
    """Entropy-coded bytes -> bits: 0xFF00 unstuffed; a restart marker ends the interval's bits."""

    def __init__(self, data):
        self.d, self.p, self.acc, self.n = data, 0, 0, 0

    def bit(self):
        if self.n == 0:
            if self.p >= len(self.d):
                raise ValueError('out of data')
            b = self.d[self.p]
            if b == 0xFF:
                if self.d[self.p + 1] != 0:
                    raise ValueError('marker inside an interval')
                self.p += 1
            self.p += 1
            self.acc, self.n = b, 8
        self.n -= 1
        return (self.acc >> self.n) & 1

    def bits(self, k):
        v = 0
        for _ in range(k):
            v = (v << 1) | self.bit()
        return v

    def restart(self, k):
        self.n = 0
        if self.d[self.p] != 0xFF or self.d[self.p + 1] != 0xD0 + (k & 7):
            raise ValueError('restart marker RST%d expected' % (k & 7))
        self.p += 2


def huffman_codes(bits, vals):
    """Canonical code assignment (ITU T.81 C.2): -> {(length, code): symbol}."""
    out, code, k = {}, 0, 0
    for length in range(1, 17):
        for _ in range(bits[length - 1]):
            out[(length, code)] = vals[k]
            code += 1
            k += 1
        if code >= (1 << length):
            raise ValueError('bad Huffman table')
        code <<= 1
    return out


def _decode_symbol(bs, codes):
    code = 0
    for length in range(1, 17):
        code = (code << 1) | bs.bit()
        if (length, code) in codes:
            return codes[(length, code)]
    raise ValueError('bad Huffman code')


def _extend(v, s):
    return v - (1 << s) + 1 if s and v < (1 << (s - 1)) else v


def coefficients(hdr):
    """Entropy decoding -> per component int64 (bh, bw, 64) blocks in natural order (quantised)."""
    h, w, comps = hdr['h'], hdr['w'], hdr['comps']
    if len(comps) == 1:
        hs = vs = 1
        comps = [(comps[0][0], 1, 1, comps[0][3])]
        mx, my = -(-w // 8), -(-h // 8)
    else:
        hs, vs = comps[0][1], comps[0][2]
        mx, my = -(-w // (8 * hs)), -(-h // (8 * vs))
    blocks = [np.zeros((my * c[2], mx * c[1], 64), np.int64) for c in comps]
    tabs = {}
    for ci, td, ta in hdr['scan']:
        tabs[ci] = (huffman_codes(*hdr['dc'][td]), huffman_codes(*hdr['ac'][ta]))
    bs = _Bits(hdr['data'])
    pred = [0] * len(comps)
    dri = hdr['dri']
    for m in range(mx * my):
        if dri and m and m % dri == 0:
            bs.restart(m // dri - 1)
            pred = [0] * len(comps)
        y, x = divmod(m, mx)
        for c, (cid, ch, cv, _) in enumerate(comps):
            dct, act = tabs[cid]
            for v in range(cv):
                for u in range(ch):
                    blk = blocks[c][y * cv + v, x * ch + u]
                    s = _decode_symbol(bs, dct)
                    pred[c] += _extend(bs.bits(s), s)
                    blk[0] = pred[c]
                    k = 1
                    while k < 64:
                        rs = _decode_symbol(bs, act)
                        r, s = rs >> 4, rs & 15
                        if s:
                            k += r
                            if k > 63:
                                raise ValueError('coefficient index past 63')
                            blk[ZIGZAG[k]] = _extend(bs.bits(s), s)
                            k += 1
                        elif r == 15:
                            k += 16
                        else:
                            break
    return blocks, (hs, vs)


FIX = dict(f0298=2446, f0390=3196, f0541=4433, f0765=6270, f0899=7373, f1175=9633, f1501=12299, f1847=15137,
           f1961=16069, f2053=16819, f2562=20995, f3072=25172)
CONST_BITS, PASS1_BITS = 13, 2


def _descale(x, n):
    return (x + (1 << (n - 1))) >> n


def _idct_1d(d0, d1, d2, d3, d4, d5, d6, d7):
    """One pass of the ISLOW butterfly (int64 arrays) -> the 8 outputs before descaling."""
    f = FIX
    z1 = (d2 + d6) * f['f0541']
    tmp2 = z1 + d6 * -f['f1847']
    tmp3 = z1 + d2 * f['f0765']
    tmp0 = (d0 + d4) << CONST_BITS
    tmp1 = (d0 - d4) << CONST_BITS
    t10, t13, t11, t12 = tmp0 + tmp3, tmp0 - tmp3, tmp1 + tmp2, tmp1 - tmp2
    o0, o1, o2, o3 = d7, d5, d3, d1
    z1, z2, z3, z4 = o0 + o3, o1 + o2, o0 + o2, o1 + o3
    z5 = (z3 + z4) * f['f1175']
    o0, o1, o2, o3 = o0 * f['f0298'], o1 * f['f2053'], o2 * f['f3072'], o3 * f['f1501']
    z1, z2 = z1 * -f['f0899'], z2 * -f['f2562']
    z3, z4 = z3 * -f['f1961'] + z5, z4 * -f['f0390'] + z5
    o0, o1, o2, o3 = o0 + z1 + z3, o1 + z2 + z4, o2 + z2 + z3, o3 + z1 + z4
    return [t10 + o3, t11 + o2, t12 + o1, t13 + o0, t13 - o0, t12 - o1, t11 - o2, t10 - o3]


def range_limit(x):
    """The C IDCT's post-IDCT range-limit table indexed by (x & 1023): x in [-128, 127] -> x + 128, larger values
    saturate at 255 and smaller at 0 as far as x in [-512, 511], beyond that the index wraps."""
    m = np.asarray(x) & 1023
    return np.where(m < 128, m + 128, np.where(m < 512, 255, np.where(m < 896, 0, m - 896))).astype(np.uint8)


# libjpeg-turbo runs this IDCT either as C (int arithmetic, the wrapping table above) or as SIMD code (dequantised
# values and the pass-1 workspace held in 16 bits, sums of two in 16 bits, saturating packs instead of the table).
# The two agree bit for bit while every dequantised coefficient and every workspace value stays within +-AGREE and
# every output x within [-512, 511]; Pillow's wheels run the SIMD code, so a block outside that range has no single
# right answer here and the decode defers it (the whole image) to Pillow.  Encoded 8-bit images stay far inside:
# |dequantised| ~ 1100, |workspace| ~ 4300, |x| ~ 180 at most over noise / checkerboards at qualities 5..100.
AGREE = 8191


class Deferred(ValueError):
    """A block left the range where libjpeg-turbo's C and SIMD IDCTs agree: Pillow decodes the image."""


def idct_islow(coef, qt):
    """(..., 64) quantised coefficients (natural order) x (64,) table -> ((..., 8, 8) uint8 samples, (...) bool:
    the block stays in the range where every libjpeg-turbo IDCT gives these samples)."""
    d = (np.asarray(coef, np.int64) * np.asarray(qt, np.int64)).reshape(coef.shape[:-1] + (8, 8))
    cols = _idct_1d(*[d[..., k, :] for k in range(8)])                       # pass 1: columns
    ws = np.stack([_descale(c, CONST_BITS - PASS1_BITS) for c in cols], axis=-2)
    rows = _idct_1d(*[ws[..., :, k] for k in range(8)])                      # pass 2: rows
    out = np.stack([_descale(r, CONST_BITS + PASS1_BITS + 3) for r in rows], axis=-1)
    ok = ((np.abs(d) <= AGREE).all(axis=(-2, -1)) & (np.abs(ws) <= AGREE).all(axis=(-2, -1))
          & ((out >= -512) & (out <= 511)).all(axis=(-2, -1)))
    return range_limit(out), ok


def _planes(blocks, qts):
    out = []
    for b, q in zip(blocks, qts):
        s, ok = idct_islow(b, q)                                              # (bh, bw, 8, 8)
        if not ok.all():
            raise Deferred('IDCT outside the range where the C and SIMD IDCTs agree')
        out.append(s.transpose(0, 2, 1, 3).reshape(b.shape[0] * 8, b.shape[1] * 8).astype(np.int64))
    return out


def upsample(plane, cw, ch, hs, vs, w, h):
    """Chroma plane (padded) -> full resolution (h, w), libjpeg's fancy triangle filters (h2v1: 3/4 + 1/4 with
    biases 1 / 2; h2v2: 9/16, 3/16, 3/16, 1/16 with biases 8 / 7; edges replicated, context rows at the image top
    and bottom replicated) -- box replication when the chroma plane is at most 2 samples wide."""
    if hs == 1 and vs == 1:
        return plane[:h, :w]
    ix = np.arange(w) // 2
    if cw <= 2:
        iy = np.arange(h) // vs
        return plane[iy][:, ix]
    left, right = np.maximum(ix - 1, 0), np.minimum(ix + 1, cw - 1)
    even = (np.arange(w) % 2) == 0
    if vs == 1:
        c = plane[:h]
        return np.where(even, (3 * c[:, ix] + c[:, left] + 1) >> 2, (3 * c[:, ix] + c[:, right] + 2) >> 2)
    iy = np.arange(h) // 2
    far = np.where(np.arange(h) % 2 == 0, np.maximum(iy - 1, 0), np.minimum(iy + 1, ch - 1))
    cs = 3 * plane[iy] + plane[far]                                           # column sums (h, padded width)
    return np.where(even, (3 * cs[:, ix] + cs[:, left] + 8) >> 4, (3 * cs[:, ix] + cs[:, right] + 7) >> 4)


def ycc_to_rgb(y, cb, cr):
    """jdcolor.c's integer tables, SCALEBITS 16, results clamped to 0..255."""
    one_half = 1 << 15
    cb, cr = cb - 128, cr - 128
    r = y + ((91881 * cr + one_half) >> 16)
    g = y + ((-22554 * cb + one_half - 46802 * cr) >> 16)
    b = y + ((116130 * cb + one_half) >> 16)
    return np.clip(np.stack([r, g, b], axis=-1), 0, 255).astype(np.uint8)


def decode(data):
    """JPEG bytes -> uint8 (H, W, 3), equal to np.asarray(Image.open(...).convert('RGB')) for the covered files."""
    hdr = parse(data)
    comps = hdr['comps']
    if len(comps) not in (1, 3) or len(hdr['scan']) != len(comps):
        raise ValueError('component layout not modelled')
    blocks, (hs, vs) = coefficients(hdr)
    planes = _planes(blocks, [hdr['qt'][c[3]] for c in (comps if len(comps) == 3 else comps[:1])])
    h, w = hdr['h'], hdr['w']
    if len(comps) == 1:
        return np.repeat(planes[0][:h, :w, None], 3, axis=2).astype(np.uint8)
    cw, ch = -(-w // hs), -(-h // vs)
    cb = upsample(planes[1], cw, ch, hs, vs, w, h)
    cr = upsample(planes[2], cw, ch, hs, vs, w, h)
    return ycc_to_rgb(planes[0][:h, :w], cb, cr)
