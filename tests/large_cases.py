"""The convolution cases of tests/test_gpu_large_tensors.py: shapes, channel views and probe items of launches whose
tensors pass 2^31 bytes or 2^31 elements, and the arithmetic of those claims.  Pure Python, so that
tests/test_large_case_table.py checks the table without a GPU.

Offsets are counted from a view's base pointer, the way the kernels index it: element (pixel p, channel c) of a view of
leading dimension ld is element p * ld + c.  A tensor "crosses bytes" when the last byte of its last element lies at or
past byte 2^31, and "crosses elements" when its last element's index is 2^31 or more.

The probe items of a case are its first frame, the frame of each crossing tensor that holds byte 2^31 (element 2^29),
the frame that holds element 2^31 where a tensor reaches it, and the last frame.  Every other frame holds NaN."""

BYTE_EDGE = 1 << 31                 # bytes
ELEM_EDGE = 1 << 31                 # elements


class Tensor(object):
    """A (n, h, w, c) view at channels [c0, c0 + c) of a buffer of ld channels per pixel."""

    def __init__(self, name, n, h, w, c, c0=0, ld=None):
        self.name, self.n, self.h, self.w, self.c, self.c0 = name, n, h, w, c, c0
        self.ld = c if ld is None else ld
        assert 0 <= c0 and c0 + c <= self.ld, (name, c0, c, self.ld)

    @property
    def frame_elems(self):
        return self.h * self.w * self.ld

    @property
    def buffer_elems(self):
        return self.n * self.frame_elems

    @property
    def last_elem(self):
        """the largest element offset from the view's base that the view holds"""
        return (self.n * self.h * self.w - 1) * self.ld + self.c - 1

    @property
    def last_byte(self):
        return 4 * self.last_elem + 3

    def crosses(self, side):
        return self.last_byte >= BYTE_EDGE if side == 'bytes' else self.last_elem >= ELEM_EDGE

    def locate(self, elem):
        """(frame, row, column, pixel index in the batch, channel) of element `elem` from the view's base"""
        f, r = divmod(elem, self.frame_elems)
        p, ch = divmod(r, self.ld)
        y, x = divmod(p, self.w)
        return f, y, x, f * self.h * self.w + p, ch


class ConvCase(object):
    """One Conv2D (sep False) or SeparableConv2D launch at batch n.

    path / fallback: what dh_conv2d_plan / dh_sepconv2d_plan must report; packed: pass the bf16 operands (else NULL,
    the CUDA-core kernels only); opts: dh_set_option values for the launch; cross: {tensor name: sides} the case
    claims ('bytes', 'elements'); edge: None, or 'below' / 'past' the 2^31-element pixel * ld product of the input
    that tc_layer_ok used to refuse.  x_lay, out_lay, res_lay, pool_lay: None (dense) or (c0, ld)."""

    def __init__(self, name, sep, n, h, w, cin, cout, ks, strides=(1, 1), path=1, fallback=0, packed=True, pre=True,
                 post=True, n_res=0, up=False, x_lay=None, out_lay=None, res_lay=(), pool_lay=None, opts=(), cross=None,
                 edge=None, epi_tma=None, bm=None):
        self.name, self.sep, self.n, self.h, self.w, self.cin, self.cout = name, sep, n, h, w, cin, cout
        self.ks, self.strides, self.path, self.fallback, self.packed = ks, strides, path, fallback, packed
        self.pre, self.post, self.n_res, self.up = pre, post, n_res, up
        self.x_lay, self.out_lay, self.res_lay, self.pool_lay = x_lay, out_lay, tuple(res_lay), pool_lay
        self.opts, self.cross, self.edge, self.epi_tma, self.bm = dict(opts), dict(cross or {}), edge, epi_tma, bm
        self.ho = -(-h // strides[0])                 # SAME padding
        self.wo = -(-w // strides[1])

    @property
    def m(self):
        return self.n * self.ho * self.wo

    @property
    def workspace(self):
        """bytes of workspace the launch needs: the two-kernel CUDA-core separable path keeps its depthwise output"""
        return 4 * self.m * self.cin if self.sep and self.path == 0 else 0

    def resized(self, n):
        """the same case at batch n"""
        c = ConvCase.__new__(ConvCase)
        c.__dict__.update(self.__dict__)
        c.n = n
        return c

    def tensors(self):
        """name -> Tensor of every view the launch reads or writes"""
        def t(name, h, w, c, lay):
            return Tensor(name, self.n, h, w, c, *(lay or (0, None)))
        ts = {'x': t('x', self.h, self.w, self.cin, self.x_lay),
              'out': t('out', self.ho, self.wo, self.cout, self.out_lay)}
        for i in range(self.n_res):
            half = self.up and i == self.n_res - 1
            lay = self.res_lay[i] if i < len(self.res_lay) else None
            ts['res%d' % i] = t('res%d' % i, self.ho // (2 if half else 1), self.wo // (2 if half else 1), self.cout,
                                lay)
        if self.pool_lay is not None:
            ts['pool'] = t('pool', self.ho // 2, self.wo // 2, self.cout, self.pool_lay or None)
        if self.workspace:
            ts['ws'] = t('ws', self.ho, self.wo, self.cin, None)
        return ts

    @property
    def tile_rows(self):
        """output pixels per tile of the launch's kernel (dh_conv_plan_info's bm): conv_sep.cu's 64 or 128, 128 on the
        other tensor-core kernels, the implicit GEMM and the two-kernel separable path, 64 on the wide pointwise kernel,
        256 / (Cout / 8) on the direct stem"""
        if self.bm is not None:
            return self.bm
        if self.path == 3:
            return 64
        if self.path == 0 and not self.packed and not self.sep and self.cin == 3 and self.ks == (3, 3):
            return 256 // (self.cout // 8)
        return 128

    def output_pixel(self, name, f, y, x):
        """index in the batch of the output pixel that reads (input) or writes (output, residual, pooled, workspace)
        pixel (y, x) of frame f of view `name`: the first of the 2 x 2 it feeds for a half-resolution view"""
        t = self.tensors()[name]
        if name == 'x':
            y, x = y // self.strides[0], x // self.strides[1]
        elif t.h != self.ho:
            y, x = 2 * y, 2 * x
        return (f * self.ho + y) * self.wo + x

    def guard_product(self):
        """N * H * W * ldx of the input: the product tc_layer_ok compared with 2^31 before it was relaxed"""
        x = self.tensors()['x']
        return x.n * x.h * x.w * x.ld

    def probes(self):
        """sorted probe frames: first, the frames of byte 2^31 and element 2^31 of each crossing tensor, last"""
        fr = {0, self.n - 1}
        for name, sides in self.cross.items():
            t = self.tensors()[name]
            if 'bytes' in sides:
                fr.add(t.locate(BYTE_EDGE // 4)[0])
            if 'elements' in sides:
                fr.add(t.locate(ELEM_EDGE)[0])
        return sorted(fr)

    def device_bytes(self):
        """bytes of the buffers the large launch allocates (plus a guard band each)"""
        return sum(4 * (t.buffer_elems + GUARD) for t in self.tensors().values())


GUARD = 1024        # SENT floats after the end of every output buffer


def _sep(name, n, h, w, cin, cout, **kw):
    return ConvCase(name, True, n, h, w, cin, cout, kw.pop('ks', (3, 3)), **kw)


def _dense(name, n, h, w, cin, cout, ks, **kw):
    return ConvCase(name, False, n, h, w, cin, cout, ks, **kw)


# Each kernel at the 2^31-byte crossing.  Batches are the smallest that put byte 2^31 of the crossing views inside
# an interior frame, and the views' leading dimensions are picked so that the crossing falls mid-row and mid-tile.
BYTE_CASES = [
    # conv_tc.cu, 16-byte gather: a stride-2 3x3 (conv_patch.cu takes stride 1 only)
    _dense('tc gather 3x3 s2', 2732, 64, 64, 32, 64, (3, 3), strides=(2, 2), x_lay=(8, 52), cross={'x': ('bytes',)}),
    # conv_tc.cu, scalar gather: Cin 3, 7x7 stride 2 (SPNet's first conv) on a 16-byte aligned view of 12 channels
    _dense('tc scalar 7x7 s2 cin3', 2733, 128, 128, 3, 16, (7, 7), strides=(2, 2), x_lay=(4, 12),
           cross={'x': ('bytes',)}),
    # conv_tc.cu, separable register producer: Cin 48 is not a whole number of conv_sep.cu's 32-channel K-blocks
    _sep('tc sep 3x3 cin48', 5244, 32, 32, 48, 64, x_lay=(16, 100), cross={'x': ('bytes',)}),
    _sep('tc sep 5x5 w32 (sep_tma off)', 1749, 32, 32, 96, 96, ks=(5, 5), x_lay=(4, 300), opts=dict(sep_tma=0),
         cross={'x': ('bytes',)}),
    # conv_sep.cu 128 x 96 tiles
    _sep('sep_tma 128x96', 3277, 32, 32, 64, 96, path=2, bm=128, x_lay=(32, 164), out_lay=(4, 100),
         cross={'x': ('bytes',)}),
    # conv_sep.cu 64 x 144 tiles, shared-memory epilogue: residual and upsampled residual by TMA, output by TMA store
    _sep('sep_tma 64x144 smem epilogue', 1823, 32, 32, 288, 288, path=2, bm=64, epi_tma=1, n_res=2, up=True,
         out_lay=(4, 292), res_lay=((0, 292), (8, 1176)),
         cross={'x': ('bytes',), 'out': ('bytes',), 'res0': ('bytes',), 'res1': ('bytes',)}),
    # conv_sep.cu 64 x 144 tiles, register epilogue (the output view is not 16-byte aligned)
    _sep('sep_tma 64x144 register epilogue', 1823, 32, 32, 288, 288, path=2, bm=64, epi_tma=0, n_res=2, up=True,
         out_lay=(2, 292), res_lay=((0, 292), (8, 1176)),
         cross={'x': ('bytes',), 'out': ('bytes',), 'res0': ('bytes',), 'res1': ('bytes',)}),
    # conv_patch.cu: 1x1 (flat pixel rows) and 3x3
    _dense('patch 1x1', 3277, 32, 32, 128, 64, (1, 1), path=4, x_lay=(16, 164), cross={'x': ('bytes',)}),
    _dense('patch 3x3', 5461, 32, 32, 64, 64, (3, 3), path=4, x_lay=(8, 100), n_res=1, res_lay=((4, 100),),
           cross={'x': ('bytes',), 'res0': ('bytes',)}),
    # conv_simt.cu: the wide pointwise kernel with its pooled output
    _dense('wide pointwise pooled', 4097, 32, 32, 16, 128, (1, 1), path=3, packed=False, pre=False,
           out_lay=(0, 132), pool_lay=(4, 524), cross={'out': ('bytes',), 'pool': ('bytes',)}),
    # conv_simt.cu: the direct 3x3x3 stem
    _dense('direct stem', 1025, 128, 128, 3, 32, (3, 3), path=0, packed=False, pre=False, out_lay=(0, 36),
           cross={'out': ('bytes',)}),
    # conv_simt.cu: the implicit GEMM, and the two-kernel separable path with its workspace past 2^31 bytes
    _dense('implicit gemm 3x3', 2732, 64, 64, 32, 32, (3, 3), path=0, fallback=1, packed=False, x_lay=(8, 52),
           cross={'x': ('bytes',)}),
    _sep('simt separable', 7283, 32, 32, 72, 32, path=0, fallback=1, packed=False, x_lay=(0, 76),
         cross={'x': ('bytes',), 'ws': ('bytes',)}),
]

# One layer of each class tc_layer_ok judges, one frame below and one frame past the 2^31-element pixel * ld product
# of its input.  The views are wide (ldx >> Cin), so the input passes 2^31 elements (8 GiB) at a small amount of work.
EDGE_CLASSES = [
    # name, separable, h, w, cin, cout, ks, strides, x_lay, path, bm
    ('tc gather 3x3 s2', False, 32, 32, 32, 64, (3, 3), (2, 2), (4, 4108), 1, None),
    ('tc scalar 7x7 s2 cin3', False, 64, 64, 3, 16, (7, 7), (2, 2), (4, 1028), 1, None),
    ('tc sep 3x3 cin48', True, 32, 32, 48, 64, (3, 3), (1, 1), (8, 4108), 1, None),
    ('sep_tma 128x96', True, 32, 32, 64, 96, (3, 3), (1, 1), (8, 4108), 2, 128),
]


def edge_cases():
    out = []
    for name, sep, h, w, cin, cout, ks, strides, x_lay, path, bm in EDGE_CLASSES:
        frame = h * w * x_lay[1]
        below = (ELEM_EDGE - 1) // frame                 # the largest batch whose guard product is below 2^31
        for edge, n in (('below', below), ('past', below + 1)):
            cross = {'x': ('bytes', 'elements')} if edge == 'past' else {'x': ('bytes',)}
            out.append(ConvCase('%s, %s 2^31 elements' % (name, edge), sep, n, h, w, cin, cout, ks, strides, path=path,
                                x_lay=x_lay, cross=cross, edge=edge, bm=bm))
    return out


EDGE_CASES = edge_cases()
CASES = BYTE_CASES + EDGE_CASES
MAX_DEVICE_BYTES = 20 * 10 ** 9
