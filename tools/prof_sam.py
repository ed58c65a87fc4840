"""Launch a soft-argmax head kernel (CUDA-event timing).
   python tools/prof_sam.py N reps [2d|3d]     2d: N frames of (32,32,48) context maps (dh_softargmax2d_ctx_f32)
                                               3d: N frames of (32,32,16*17) volumes (dh_softargmax3d_f32)"""
import ctypes as C
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from deephar_b200 import _ffi  # noqa: E402

n = int(sys.argv[1]) if len(sys.argv) > 1 else 1024
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 10
mode = sys.argv[3] if len(sys.argv) > 3 else '2d'
ctx = _ffi.Context(0)
lib = _ffi.lib()
st = torch.cuda.current_stream().cuda_stream
if mode == '2d':
    h = torch.randn(n, 32, 32, 48, device='cuda') * 3.0
    pose = torch.empty(n, 16, 2, device='cuda')
    vis = torch.empty(n, 16, 1, device='cuda')
    hv = _ffi.dh_view(h.data_ptr(), n, 32, 32, 48, 48)
    per_frame = 32 * 32 * 48 * 4 + 16 * 3 * 4

    def launch():
        _ffi.check(lib.dh_softargmax2d_ctx_f32(ctx.handle, C.byref(hv), 16, 2, C.c_float(0.8), pose.data_ptr(), vis.data_ptr(), st))
else:
    nj, d = 17, 16
    h = torch.randn(n, 32, 32, nj * d, device='cuda') * 3.0
    pose = torch.empty(n, nj, 3, device='cuda')
    vis = torch.empty(n, nj, 1, device='cuda')
    hv = _ffi.dh_view(h.data_ptr(), n, 32, 32, nj * d, nj * d)
    per_frame = 32 * 32 * nj * d * 4 + nj * 4 * 4

    def launch():
        _ffi.check(lib.dh_softargmax3d_f32(ctx.handle, C.byref(hv), nj, d, pose.data_ptr(), vis.data_ptr(), st))
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
print('softargmax %s n=%d: %.1f us/launch, %.0f GB/s' % (mode, n, ms * 1e3, n * per_frame / ms / 1e6))
