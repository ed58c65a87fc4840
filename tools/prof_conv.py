"""Launch one fused conv layer a few times (CUDA-event timing).  usage:
   python tools/prof_conv.py sep|conv N H W Cin Cout k [precision] [reps]"""
import ctypes as C
import sys
import os

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tests'))
from deephar_b200 import _ffi, tc  # noqa: E402
from gpu_util import Dev, conv_desc  # noqa: E402

kind = sys.argv[1]
n, h, w, cin, cout, k = [int(a) for a in sys.argv[2:8]]
precision = int(sys.argv[8]) if len(sys.argv) > 8 else 3
reps = int(sys.argv[9]) if len(sys.argv) > 9 else 5
dev = Dev(torch)
if os.environ.get('DH_DBG'):        # only in `make ABLATE=1` builds
    _ffi.check(dev.lib.dh_set_option(dev.ctx.handle, b'dbg', int(os.environ['DH_DBG'])), 'dbg (needs make ABLATE=1)')
if os.environ.get('DH_PATCH'):
    dev.lib.dh_set_option(dev.ctx.handle, b'dense_patch', int(os.environ['DH_PATCH']))
if os.environ.get('DH_PWSMALLK'):
    dev.lib.dh_set_option(dev.ctx.handle, b'pw_smallk', int(os.environ['DH_PWSMALLK']))
if os.environ.get('DH_SHARE'):
    dev.lib.dh_set_option(dev.ctx.handle, b'share_a', int(os.environ['DH_SHARE']))
rng = np.random.default_rng(0)
x = dev.put(rng.standard_normal((n, h, w, cin)))
r0 = dev.put(rng.standard_normal((n, h, w, cout)))
r1 = dev.put(rng.standard_normal((n, h, w, cout)))
out = dev.empty(n, h, w, cout)
post = (rng.uniform(0.5, 1.5, cout), rng.standard_normal(cout))
d = conv_desc(dev, (k, k), pre_relu=True, post=post, res=[] if os.environ.get('DH_NORES') else ([dev.view(r0), dev.view(r1)] if os.environ.get('DH_RES2') else [dev.view(r0)]),
              precision=precision)
xv, ov = dev.view(x), dev.view(out)
if kind == 'sep':
    dw = dev.put(rng.standard_normal((k, k, cin, 1)) / k)
    pw = rng.standard_normal((1, 1, cin, cout)) / np.sqrt(cin)
    hi, lo, cp, kp = tc.pack_matrix(pw.reshape(cin, cout).astype(np.float32))
    pwd = dev.put(pw)
else:
    wt = rng.standard_normal((k, k, cin, cout)) / np.sqrt(k * k * cin)
    hi, lo, cp, kp = tc.pack_matrix(wt.reshape(-1, cout).astype(np.float32))
    wd = dev.put(wt)
th = torch.from_numpy(hi.view(np.int16).copy()).cuda()
tl = torch.from_numpy(lo.view(np.int16).copy()).cuda()
pk = _ffi.dh_packed_w(th.data_ptr(), tl.data_ptr(), cp, kp)


def launch():
    if kind == 'sep':
        rc = dev.lib.dh_sepconv2d_f32(dev.ctx.handle, C.byref(xv), dw.data_ptr(), pwd.data_ptr(), C.byref(pk),
                                      C.byref(d), C.byref(ov), dev.stream())
    else:
        rc = dev.lib.dh_conv2d_f32(dev.ctx.handle, C.byref(xv), wd.data_ptr(), C.byref(pk), C.byref(d),
                                   C.byref(ov), dev.stream())
    _ffi.check(rc, 'launch')


for _ in range(3):
    launch()
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(reps):
    launch()
e1.record()
torch.cuda.synchronize()
ms = e0.elapsed_time(e1) / reps
mac = n * h * w * (cin * cout + (k * k * cin if kind == 'sep' else (k * k - 1) * cin * cout))
if os.environ.get('DH_SAVE'):
    np.save(os.environ['DH_SAVE'], out.cpu().numpy())
info = _ffi.dh_conv_plan_info()
if kind == 'sep':
    rc = dev.lib.dh_sepconv2d_plan(dev.ctx.handle, C.byref(xv), dw.data_ptr(), pwd.data_ptr(), C.byref(pk), C.byref(d),
                                   C.byref(ov), C.byref(info))
else:
    rc = dev.lib.dh_conv2d_plan(dev.ctx.handle, C.byref(xv), wd.data_ptr(), C.byref(pk), C.byref(d), C.byref(ov),
                                C.byref(info))
_ffi.check(rc, 'plan')
print('%s n%d %dx%dx%d->%d k%d prec%d: %.1f us/launch  %.1f TFLOP/s (algorithmic)  path=%d  tile %dx%d  grid %dx%d  '
      'cluster %d  epi_tma %d' % (kind, n, h, w, cin, cout, k, precision, ms * 1000, 2 * mac / ms / 1e9,
                      dev.lib.dh_last_conv_path(dev.ctx.handle), info.bm, info.bn_cta, info.grid_x, info.grid_y,
                      info.cluster, info.epi_tma))
