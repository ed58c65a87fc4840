"""Baseline JPEG decoding (deephar_b200/jpeg.py, csrc/jpeg.cu) on the CPU: the marker parser routes each kind of file,
its Huffman tables are canonical, the integer model oracle/jpeg.py equals Pillow bit for bit on every layout the GPU
takes, and the C descriptors have their ctypes mirrors' sizes."""
import io
import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

from deephar_b200 import _ffi, jpeg
from oracle import jpeg as oj
import jpeg_cases as jc

Image = pytest.importorskip('PIL.Image')
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _host_files():
    a = jc.smooth(24, 40, 1)
    b = io.BytesIO()
    Image.fromarray(a).save(b, 'PNG')
    cmyk = io.BytesIO()
    Image.fromarray(a).convert('CMYK').save(cmyk, 'JPEG', quality=90)
    base = jc.encode(a, quality=90, subsampling=2)
    return {'progressive': jc.encode(a, quality=90, progressive=True), 'png': b.getvalue(), 'cmyk': cmyk.getvalue(),
            'truncated': base[:len(base) // 2], 'no_eoi': base[:-2], 'garbage': b'not an image at all',
            'two_scans': base[:-2] + base[base.index(b'\xff\xda'):]}


@pytest.mark.parametrize('layout', sorted(jc.LAYOUTS))
def test_parser_takes_baseline_layouts(layout):
    f = jpeg.parse(jc.layout_file(layout, 17, 33, 90))
    assert isinstance(f, jpeg.Frame), getattr(f, 'reason', None)
    assert (f.h, f.w) == (17, 33)
    assert f.ncomp == (1 if layout == 'grey' else 3)
    want = {'444': (1, 1), '422': (2, 1), 'rst_rows': (2, 1)}.get(layout, (1, 1) if layout == 'grey' else (2, 2))
    assert (f.hs, f.vs) == want
    total = f.mcus_x * f.mcus_y
    assert f.segments[:, 3].sum() == total and f.segments[0, 2] == 0
    if layout.startswith('rst'):
        assert f.dri > 0 and len(f.segments) == -(-total // f.dri) > 1
    else:
        assert len(f.segments) == 1


def test_parser_takes_custom_qtables():
    f = jpeg.parse(jc.encode(jc.noise(16, 16), qtables=[[255] * 64, [200] * 64], subsampling=0))
    assert isinstance(f, jpeg.Frame)
    assert int(f.qt[0][0]) == 255 and int(f.qt[1][5]) == 200


@pytest.mark.parametrize('kind', sorted(_host_files()))
def test_parser_routes_the_rest_to_pillow(kind):
    f = jpeg.parse(_host_files()[kind])
    assert isinstance(f, jpeg.Host) and f.reason


@pytest.mark.parametrize('layout', ['420', 'optimize', 'grey'])
def test_huffman_tables_are_canonical(layout):
    hdr = oj.parse(jc.layout_file(layout, 40, 56, 50, seed=1))
    for bits, vals in list(hdr['dc'].values()) + list(hdr['ac'].values()):
        t = jpeg.huffman_table(bits, vals)
        codes = {(l, c): s for l, c, s in t['codes']}
        assert codes == oj.huffman_codes(bits, vals)
        lengths = [l for l, _, _ in t['codes']]
        assert lengths == sorted(lengths)                                   # canonical: by length, then value
        for (l, c), s in codes.items():
            assert c < (1 << l) - (1 if l == max(lengths) else 0) or l < max(lengths)
            if l <= 9:
                lo, hi = c << (9 - l), (c + 1) << (9 - l)
                assert np.all(t['lut'][lo:hi] == ((l << 8) | s))
            else:
                assert t['lut'][c >> (l - 9)] == 0                          # long codes take the search
                assert c <= t['maxcode'][l] and t['vals'][c + t['valoff'][l]] == s
        assert np.count_nonzero(t['lut']) == sum(1 << (9 - l) for l in lengths if l <= 9)


def test_huffman_table_refuses_overfull_lengths():
    with pytest.raises(ValueError):
        jpeg.huffman_table([2] + [0] * 15, [0, 1])                          # two 1-bit codes: the all-ones code


@pytest.mark.parametrize('layout', sorted(jc.LAYOUTS))
@pytest.mark.parametrize('quality', jc.QUALITIES)
def test_oracle_matches_pillow(layout, quality):
    for seed, (h, w) in enumerate(jc.SIZES):
        data = jc.layout_file(layout, h, w, quality, seed)
        assert np.array_equal(oj.decode(data), jc.pillow_rgb(data)), (layout, quality, h, w)


@pytest.mark.parametrize('sub', [0, 1, 2])
def test_oracle_matches_pillow_narrow_chroma(sub):
    """Planes at most 2 samples wide are replicated, not triangle-filtered."""
    for h, w in [(2, 2), (3, 3), (4, 4), (5, 6), (9, 5), (6, 7)]:
        data = jc.encode(jc.noise(h, w, h * w), quality=75, subsampling=sub)
        assert np.array_equal(oj.decode(data), jc.pillow_rgb(data)), (sub, h, w)


def overshoot_files():
    """(name, bytes, in_range): Pillow files with large quantisation tables, and re-encoded scans whose coefficients
    drive the IDCT past the range the C and SIMD IDCTs agree on."""
    rng = np.random.default_rng(7)
    out = []
    for q, sub in [(255, 0), (200, 2), (128, 1)]:
        out.append(('qtables_%d_%d' % (q, sub), jc.encode(jc.noise(40, 56, q), qtables=[[q] * 64, [q] * 64],
                                                         subsampling=sub), True))
    for q, amp in [(64, 5), (255, 5), (255, 40), (16, 1000)]:
        tmpl = jc.encode(jc.noise(16, 24, c=1, seed=q), qtables=[[q] * 64])
        blocks = rng.integers(-amp, amp + 1, (6, 64))
        out.append(('crafted_%d_%d' % (q, amp), jc.with_coefficients(tmpl, blocks), False))
    tmpl = jc.encode(jc.noise(16, 16, c=1), qtables=[[20] * 64])            # large but agreed
    blocks = np.zeros((4, 64), np.int64)
    blocks[:, 0] = [-70, 70, -40, 40]                                       # |x| up to ~230: clamped samples
    blocks[:, 1] = [20, -20, 5, -5]
    out.append(('crafted_in_range', jc.with_coefficients(tmpl, blocks), True))
    return out


def test_oracle_idct_overshoot():
    for name, data, in_range in overshoot_files():
        want = jc.pillow_rgb(data)
        if in_range:
            assert np.array_equal(oj.decode(data), want), name
        else:
            with pytest.raises(oj.Deferred):
                oj.decode(data)


def test_range_limit_table():
    x = np.arange(-1100, 1100)
    t = oj.range_limit(x)
    inside = (x >= -512) & (x <= 511)
    assert np.array_equal(t[inside], np.clip(x[inside] + 128, 0, 255))    # a clamp where C and SIMD agree
    assert t[x == 512][0] == 0 and t[x == -513][0] == 255                   # the C table wraps beyond


def test_pack_offsets():
    datas = [jc.layout_file(l, 17, 33, 90, s) for s, l in enumerate(['420', 'grey', 'rst_blocks', '422'])]
    frames = [jpeg.parse(d) for d in datas]
    pk = jpeg.pack(frames, _ffi)
    assert pk['n_huff'] <= 4 * 2 and len(pk['qtab']) % 64 == 0
    for i, f in enumerate(frames):
        im = pk['images'][i]
        segs = pk['segments'][pk['segments']['i'] == i]
        assert segs['c'].sum() == f.mcus_x * f.mcus_y
        assert segs['b'][0] == im.data and np.all(segs['e'] <= im.data + f.scan_end - f.scan)
        assert im.nblocks == sum(im.bw[c] * im.bh[c] for c in range(f.ncomp))
    assert pk['coef_elems'] == sum(pk['images'][i].nblocks for i in range(4)) * 64


def test_structs_match_ctypes():
    gcc = shutil.which('gcc')
    if gcc is None:
        pytest.skip('no gcc')
    names = ['dh_jpeg_image', 'dh_jpeg_segment', 'dh_jpeg_huff', 'dh_jpeg_batch']
    with tempfile.TemporaryDirectory() as d:
        src = os.path.join(d, 's.c')
        with open(src, 'w') as f:
            f.write('#include <stdio.h>\n#include "deephar_b200.h"\nint main(void) {\n%s return 0; }\n'
                    % ''.join('printf("%%zu\\n", sizeof(%s));\n' % n for n in names))
        exe = os.path.join(d, 's')
        subprocess.check_call([gcc, '-std=c99', '-Wall', '-Werror', '-I', os.path.join(ROOT, 'include'), src, '-o', exe])
        sizes = [int(v) for v in subprocess.check_output([exe]).split()]
    import ctypes
    assert sizes == [ctypes.sizeof(getattr(_ffi, n)) for n in names]
