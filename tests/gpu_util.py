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


def close(got, ref, tol=2e-5):
    """max |got - ref| within tol relative to the output scale (2e-5: fp32 CUDA-core path vs the fp64 oracle)"""
    scale = max(1.0, float(np.abs(ref).max()))
    err = float(np.abs(got.astype(np.float64) - ref).max())
    assert err <= tol * scale, 'max err %g (scale %g)' % (err, scale)


def sam2d_ref(h, alpha, conf_on_prob, d=None):
    """fp64 plain 2-D head: (pose (N,C,2), or (N,C,3) with the depth expectation of d), confidence, probabilities"""
    from oracle import ops_np
    p = ops_np.channel_softmax_2d(h, alpha)
    xy = ops_np.softargmax2d(p)
    conf = ops_np.keypoint_confidence(p if conf_on_prob else h)
    if d is not None:
        z = (ops_np.sigmoid(d) * p).sum(axis=(1, 2))[..., None]
        xy = np.concatenate([xy, z], axis=-1)
    return xy, conf, p


def num_sms(dev):
    return dev.torch.cuda.get_device_properties(dev.torch.cuda.current_device()).multi_processor_count


def loop_batch(dev, items_per_frame):
    """A batch size at which the grid-stride kernels of elementwise.cu (grid capped at num_sms * 16 CTAs of 256
    threads) give every thread at least two iterations over items_per_frame work items per frame."""
    return 2 * num_sms(dev) * 16 * 256 // items_per_frame + 1


SENT = 7.25     # fills the channels of a wider buffer outside a view


def sliced(dev, x, c0, ld):
    """x on the device as the channel slice [c0, c0 + C) of a buffer of ld channels whose other channels hold SENT"""
    big = np.full(x.shape[:3] + (ld,), SENT)
    big[..., c0:c0 + x.shape[3]] = x
    return dev.view(dev.put(big), c0, c0 + x.shape[3])


class Out(object):
    """An output view: a dense NaN-filled buffer, or the channel slice [c0, c0 + C) of a buffer of ld channels filled
    with SENT.  get() checks that nothing outside the slice was written and returns the view's contents."""
    def __init__(self, dev, shape, c0=None, ld=None):
        self.c0, self.c = c0, shape[3]
        if c0 is None:
            self.t = dev.empty(*shape)
            self.view = dev.view(self.t)
        else:
            self.t = dev.empty(*shape[:3], ld)
            self.t.fill_(SENT)
            self.view = dev.view(self.t, c0, c0 + self.c)

    def get(self):
        a = self.t.cpu().numpy()
        if self.c0 is None:
            return a
        assert np.all(a[..., :self.c0] == SENT) and np.all(a[..., self.c0 + self.c:] == SENT), 'wrote outside the view'
        return a[..., self.c0:self.c0 + self.c]


def layout_io(dev, x, out_shape, layout):
    """(input view, Out) of a memory-bound kernel: 'slice' puts the input at channels [4, 4 + C) of a buffer and the
    output at [8, 8 + C), both 16-byte aligned for a C that is a multiple of 4; any other layout is dense"""
    if layout == 'slice':
        return sliced(dev, x, 4, x.shape[3] + 8), Out(dev, out_shape, 8, out_shape[3] + 12)
    return dev.view(dev.put(x)), Out(dev, out_shape)


NULLV = C.cast(None, C.POINTER(_ffi.dh_view))
NULLP = C.cast(None, C.POINTER(_ffi.dh_packed_w))
