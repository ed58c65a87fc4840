"""JPEG test inputs shared by tests/test_jpeg.py (CPU) and tests/test_gpu_jpeg.py: seeded images encoded by Pillow
in every layout the decoder routes, and `with_coefficients`, which re-encodes a Pillow file's scan with chosen
quantised coefficients (same tables) -- the way to drive the IDCT far outside 0..255."""
import io

import numpy as np

from oracle import jpeg as oj


def encode(a, **kw):
    from PIL import Image
    b = io.BytesIO()
    Image.fromarray(a).save(b, 'JPEG', **kw)
    return b.getvalue()


def smooth(h, w, seed=0, c=3):
    """Natural-like content: low-frequency waves plus mild noise."""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w]
    a = np.stack([128 + 90 * np.sin(x / (5.0 + 7 * k) + k) * np.cos(y / (7.0 + 5 * k) - k) for k in range(c)], -1)
    a = np.clip(a + rng.normal(0, 6, a.shape), 0, 255).astype(np.uint8)
    return a[..., 0] if c == 1 else a


def noise(h, w, seed=0, c=3):
    a = np.random.default_rng(seed).integers(0, 256, (h, w, c), dtype=np.uint8)
    return a[..., 0] if c == 1 else a


def pillow_rgb(data):
    from PIL import Image
    with Image.open(io.BytesIO(data)) as im:
        return np.asarray(im.convert('RGB'))


SIZES = [(1, 1), (7, 9), (16, 16), (17, 33), (40, 56)]
QUALITIES = [5, 50, 90, 100]
LAYOUTS = {'444': dict(subsampling=0), '422': dict(subsampling=1), '420': dict(subsampling=2), 'grey': {},
           'optimize': dict(subsampling=2, optimize=True), 'rst_blocks': dict(subsampling=2, restart_marker_blocks=2),
           'rst_rows': dict(subsampling=1, restart_marker_rows=1)}


def layout_file(layout, h, w, quality, seed=0):
    """One file of the matrix: smooth content for the first seeds, noise for odd ones."""
    c = 1 if layout == 'grey' else 3
    a = smooth(h, w, seed, c) if seed % 2 == 0 else noise(h, w, seed, c)
    return encode(a, quality=quality, **LAYOUTS[layout])


class _BitWriter(object):
    def __init__(self):
        self.out, self.acc, self.n = bytearray(), 0, 0

    def put(self, v, k):
        for i in range(k - 1, -1, -1):
            self.acc = (self.acc << 1) | ((v >> i) & 1)
            self.n += 1
            if self.n == 8:
                self.out.append(self.acc)
                if self.acc == 0xFF:
                    self.out.append(0)
                self.acc = self.n = 0

    def flush(self):
        if self.n:
            self.put((1 << (8 - self.n)) - 1, 8 - self.n)
        return bytes(self.out)


def _category(v):
    return 0 if v == 0 else int(abs(v)).bit_length()


def with_coefficients(template, blocks):
    """Replace the scan of `template` (a Pillow grey JPEG without restart markers, any size) with `blocks`
    (nblocks, 64) quantised coefficients in natural order, raster block order; same quantisation and Huffman tables
    (Pillow's standard tables carry every DC category up to 11 and every AC (run, size) up to size 10)."""
    hdr = oj.parse(template)
    assert len(hdr['comps']) == 1 and not hdr['dri']
    _, td, ta = hdr['scan'][0]
    dc = {s: c for c, s in oj.huffman_codes(*hdr['dc'][td]).items()}
    ac = {s: c for c, s in oj.huffman_codes(*hdr['ac'][ta]).items()}
    bw = _BitWriter()
    pred = 0
    for blk in np.asarray(blocks, np.int64):
        zz = blk[oj.ZIGZAG]
        diff = int(zz[0]) - pred
        pred = int(zz[0])
        s = _category(diff)
        bw.put(dc[s][1], dc[s][0])
        bw.put(diff if diff >= 0 else diff + (1 << s) - 1, s)
        run = 0
        for k in range(1, 64):
            v = int(zz[k])
            if v == 0:
                run += 1
                continue
            while run > 15:
                bw.put(ac[0xF0][1], ac[0xF0][0])
                run -= 16
            s = _category(v)
            sym = (run << 4) | s
            bw.put(ac[sym][1], ac[sym][0])
            bw.put(v if v >= 0 else v + (1 << s) - 1, s)
            run = 0
        if run:
            bw.put(ac[0][1], ac[0][0])
    start = template.index(hdr['data'])
    return template[:start] + bw.flush() + b'\xff\xd9'
