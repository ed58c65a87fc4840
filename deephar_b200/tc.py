"""Host-side weight packing for the wgmma path (deephar_b200/csrc/conv_tc.cu).

Keras kernels stay the source of truth (HWIO fp32); at load time each Conv2D /
pointwise kernel is additionally laid out as the K-major B operand the wgmma reads:
bf16 [Cout_pad][K_pad] with K = (ky, kx, ci) flattened, split into hi + lo halves so
that three bf16 MMAs reproduce the fp32 product to ~2^-16 (see conv_tc.cu).
"""
import numpy as np

from . import _ffi
from .weights import split_bf16


def pack_matrix(w_k_by_cout):
    """w: (K, Cout) fp32 -> (hi, lo) uint16 [Cout_pad][K_pad] (zero padded)."""
    lib = _ffi.lib()
    k, cout = w_k_by_cout.shape
    kp, cp = lib.dh_tc_k_pad(k), lib.dh_tc_cout_pad(cout)
    full = np.zeros((cp, kp), dtype=np.float32)
    full[:cout, :k] = np.ascontiguousarray(w_k_by_cout.T)
    hi, lo = split_bf16(full)
    return hi.reshape(cp, kp), lo.reshape(cp, kp), cp, kp


def pack_conv_kernel(w_hwio):
    kh, kw, cin, cout = w_hwio.shape
    return pack_matrix(np.asarray(w_hwio, np.float32).reshape(kh * kw * cin, cout))
