"""Helpers for the -m gpu parity tests: call the C ABI on torch device buffers."""
import ctypes as C

import numpy as np

from deephar_b200 import _ffi


class Dev(object):
    def __init__(self, torch):
        self.torch = torch
        self.ctx = _ffi.Context(torch.cuda.current_device())
        self.lib = _ffi.lib()
        self.keep = []
        self.ws = torch.empty(64 << 20, dtype=torch.float32, device='cuda')
        self.ctx.set_workspace(self.ws.data_ptr(), self.ws.numel() * 4)

    def put(self, a):
        t = self.torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).cuda()
        self.keep.append(t)
        return t

    def empty(self, *shape):
        t = self.torch.full(shape, float('nan'), dtype=self.torch.float32, device='cuda')
        self.keep.append(t)
        return t

    def view(self, t, c0=None, c1=None):
        """dh_view of an NHWC tensor, optionally a channel slice [c0:c1)."""
        n, h, w, c = t.shape
        if c0 is None:
            return _ffi.dh_view(t.data_ptr(), n, h, w, c, c)
        return _ffi.dh_view(t.data_ptr() + 4 * c0, n, h, w, c1 - c0, c)

    def stream(self):
        return self.torch.cuda.current_stream().cuda_stream

    def call(self, name, *args):
        rc = getattr(self.lib, name)(self.ctx.handle, *args, self.stream())
        _ffi.check(rc, name)
        self.torch.cuda.synchronize()


def packed_weights(dev, w_k_by_cout):
    """(K, Cout) weights as the bf16 hi / lo K-major operand of the tensor-core kernels (tc.pack_matrix), on the device."""
    from deephar_b200 import tc
    hi, lo, cp, kp = tc.pack_matrix(np.asarray(w_k_by_cout, np.float32))
    th = dev.torch.from_numpy(hi.view(np.int16).copy()).cuda()
    tl = dev.torch.from_numpy(lo.view(np.int16).copy()).cuda()
    dev.keep += [th, tl]
    return _ffi.dh_packed_w(th.data_ptr(), tl.data_ptr(), cp, kp)


def conv_desc(dev, size, strides=(1, 1), padding='same', pre_relu=False, post_relu=False,
              pre=None, post=None, res=(), precision=3):
    d = _ffi.dh_conv_desc()
    d.kh, d.kw = size
    d.sh, d.sw = strides
    d.pad_same = 1 if padding == 'same' else 0
    d.pre_relu = int(pre_relu)
    d.post_relu = int(post_relu)
    if pre is not None:
        d.pre_scale, d.pre_shift = dev.put(pre[0]).data_ptr(), dev.put(pre[1]).data_ptr()
    if post is not None:
        d.post_scale, d.post_shift = dev.put(post[0]).data_ptr(), dev.put(post[1]).data_ptr()
    d.n_res = len(res)
    for i, r in enumerate(res):
        d.res[i] = r
    d.precision = precision
    return d


NULLV = C.cast(None, C.POINTER(_ffi.dh_view))
NULLP = C.cast(None, C.POINTER(_ffi.dh_packed_w))
