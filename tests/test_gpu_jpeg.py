"""GPU JPEG decoding (csrc/jpeg.cu through deephar_b200/jpeg.py) against Pillow, bit for bit: the layout x size x
quality matrix, VGA and 1080p frames, IDCT-overshoot tables, FramePipeline.from_jpeg against FramePipeline on
Pillow-decoded frames, a mixed batch with files only Pillow decodes and broken files, and a batch of 256 VGA files."""
import io

import numpy as np
import pytest

from deephar_b200 import jpeg, preprocess

import jpeg_cases as jc
from test_jpeg import overshoot_files

pytestmark = pytest.mark.gpu
Image = pytest.importorskip('PIL.Image')


def _check(dec, datas, gpu_expected=True):
    got = dec(datas)
    for k, (g, d) in enumerate(zip(got, datas)):
        want = jc.pillow_rgb(d)
        assert g.dtype.is_floating_point is False and tuple(g.shape) == want.shape, k
        assert np.array_equal(g.cpu().numpy(), want), k
    if gpu_expected:
        assert dec.host_decoded == [], dec.host_decoded          # the kernels decoded every file themselves
    return got


def test_decode_matrix(cuda):
    dec = jpeg.JpegDecoder()
    datas = [jc.layout_file(l, h, w, q, s) for l in sorted(jc.LAYOUTS) for q in jc.QUALITIES
             for s, (h, w) in enumerate(jc.SIZES)]
    datas += [jc.encode(jc.noise(h, w, h * w), quality=75, subsampling=sub)
              for sub in (0, 1, 2) for h, w in [(2, 2), (3, 3), (5, 6), (9, 5), (6, 7)]]
    _check(dec, datas)


def test_decode_vga_and_1080p(cuda):
    dec = jpeg.JpegDecoder()
    datas = []
    for h, w in [(480, 640), (1080, 1920)]:
        datas += [jc.encode(jc.smooth(h, w, 1), quality=90, subsampling=2),
                  jc.encode(jc.noise(h, w, 2), quality=90, subsampling=2),
                  jc.encode(jc.smooth(h, w, 3), quality=95, subsampling=0),
                  jc.encode(jc.smooth(h, w, 4), quality=80, subsampling=1, restart_marker_rows=2),
                  jc.encode(jc.smooth(h, w, 5, c=1), quality=90)]
    _check(dec, datas)


def test_decode_from_paths(cuda, tmp_path):
    paths = []
    for k, (h, w) in enumerate([(33, 47), (64, 48)]):
        p = tmp_path / ('f%d.jpg' % k)
        p.write_bytes(jc.layout_file('420', h, w, 85, k))
        paths.append(p)
    got = jpeg.decode(paths)
    for g, p in zip(got, paths):
        assert np.array_equal(g.cpu().numpy(), preprocess.decode_images([p])[0])


def test_idct_overshoot(cuda):
    dec = jpeg.JpegDecoder()
    files = overshoot_files()
    got = dec([d for _, d, _ in files])
    for (name, d, _), g in zip(files, got):
        assert np.array_equal(g.cpu().numpy(), jc.pillow_rgb(d)), name
    deferred = [k for k, (_, _, ok) in enumerate(files) if not ok]
    assert dec.host_decoded == deferred                          # the kernels flag exactly the out-of-range files


def _mixed(tmp_path, broken):
    """PNG, progressive and CMYK files among baseline ones; `broken` adds a file with corrupted entropy-coded bytes
    and a truncated one (Pillow raises for both)."""
    a = jc.smooth(48, 64, 9)
    png = tmp_path / 'a.png'
    Image.fromarray(a).save(png)
    cmyk = tmp_path / 'c.jpg'
    Image.fromarray(a).convert('CMYK').save(cmyk, quality=90)
    prog = tmp_path / 'p.jpg'
    prog.write_bytes(jc.encode(a, quality=90, progressive=True))
    good = jc.encode(jc.smooth(40, 72, 3), quality=90, subsampling=2)
    corrupt = bytearray(good)
    s = good.index(b'\xff\xda') + 14
    for k in range(s + 40, s + 60, 3):                           # flip bits inside the entropy-coded data
        corrupt[k] = (corrupt[k] ^ 0x5A) if (corrupt[k] ^ 0x5A) != 0xFF else corrupt[k]
    cpath = tmp_path / 'corrupt.jpg'
    cpath.write_bytes(bytes(corrupt))
    gpath = tmp_path / 'good.jpg'
    gpath.write_bytes(good)
    paths = [gpath, png, prog, cmyk, gpath]
    if broken:
        tpath = tmp_path / 'trunc.jpg'
        tpath.write_bytes(good[:len(good) // 2])
        paths[4:4] = [cpath, tpath]
    return paths


def test_mixed_batch(cuda, tmp_path):
    paths = _mixed(tmp_path, False)
    got = jpeg.decode(paths)
    want = preprocess.decode_images(paths)
    for g, w in zip(got, want):
        assert np.array_equal(g.cpu().numpy(), w)
    paths = _mixed(tmp_path, True)
    with pytest.raises(Exception) as ours:
        jpeg.decode(paths)
    with pytest.raises(Exception) as pillow:
        preprocess.decode_images(paths)
    assert type(ours.value) is type(pillow.value) and str(ours.value) == str(pillow.value)
    for k in (4, 5):                                             # each broken file on its own
        with pytest.raises(Exception) as ours:
            jpeg.decode([paths[0], paths[k]])
        with pytest.raises(Exception) as pillow:
            preprocess.decode_images([paths[0], paths[k]])
        assert type(ours.value) is type(pillow.value) and str(ours.value) == str(pillow.value)


@pytest.mark.parametrize('hflip,power', [(0, 1), ([0, 1, 1, 0, 1], (1.0, 1.5, 0.7))])
def test_from_jpeg_matches_pipeline(cuda, tmp_path, hflip, power):
    paths = _mixed(tmp_path, False)
    rng = np.random.default_rng(2)
    objpos = rng.uniform(10, 40, (len(paths), 2))
    winsize = rng.uniform(20, 70, len(paths))
    pipe = preprocess.FramePipeline((64, 48))
    want, want_af = pipe(preprocess.decode_images(paths), objpos, winsize, hflip=hflip, channel_power=power)
    got, got_af = pipe.from_jpeg(paths, objpos, winsize, hflip=hflip, channel_power=power)
    assert np.array_equal(got.cpu().numpy(), want.cpu().numpy())
    assert np.array_equal(got_af, want_af)


def test_batch_256_vga(cuda):
    datas = [jc.encode(jc.smooth(480, 640, s) if s % 4 else jc.noise(480, 640, s), quality=90, subsampling=2)
             for s in range(8)]
    datas = [datas[k % 8] for k in range(256)]
    dec = jpeg.JpegDecoder()
    got = dec(datas)
    assert dec.host_decoded == []
    wants = [jc.pillow_rgb(d) for d in datas[:8]]
    for k, g in enumerate(got):
        assert np.array_equal(g.cpu().numpy(), wants[k % 8]), k
    pipe = preprocess.FramePipeline((256, 256))
    objpos = np.tile([[320.0, 240.0]], (256, 1))
    want, _ = pipe(wants * 32, objpos, 300.0)
    got, _ = pipe.from_jpeg(datas, objpos, 300.0)
    assert np.array_equal(got.cpu().numpy(), want.cpu().numpy())
