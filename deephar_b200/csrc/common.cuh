// Shared helpers for the deephar_b200 kernels (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include "../../include/deephar_b200.h"

struct dh_ctx {
    int device;
    int num_sms;
    int64_t launches;
    void* workspace;
    int64_t workspace_bytes;
    int last_conv_path;   // 0 = CUDA-core kernels, 1 = wgmma kernel (test / bench introspection)
    int share_a;          // 1 = cluster pairs share the separable A tile (default), 0 = independent CTAs
    int sep_tma;          // 1 = TMA-staged separable kernel (conv_sep.cu) where it applies (default)
    int pw_smallk;        // 1 = CUDA-core kernel for wide 1x1 convs with Cin <= 64 (conv_simt.cu) (default)
    int sam3d_stream;     // 1 = cluster-split streaming kernel for the volumetric head (softargmax_stream.cu) (default)
    int dense_patch;      // 1 = TMA-staged patch kernel for stride-1 Conv2D (conv_patch.cu) where it applies (default)
    void* comm;           // ncclComm_t of the output all-gather (comm.cu), NULL until dh_comm_init
    int comm_rank, comm_world;
    int64_t fallbacks;    // convolutions served by the CUDA-core implicit-GEMM fallback (conv_simt.cu) since creation / reset
    int dbg;              // ablation bits for tools/ (0 in production; results are WRONG when set)
};

void dh_set_error(const char* fmt, ...);

#define DH_CHECK_ARG(cond, ...)            \
    do {                                   \
        if (!(cond)) {                     \
            dh_set_error(__VA_ARGS__);     \
            return -1;                     \
        }                                  \
    } while (0)

// After a launch: count it and surface launch-configuration errors.
#define DH_LAUNCH_EPILOGUE(ctx, nlaunch)                     \
    do {                                                     \
        (ctx)->launches += (nlaunch);                        \
        cudaError_t e__ = cudaGetLastError();                \
        if (e__ != cudaSuccess) {                            \
            dh_set_error("CUDA launch failed: %s (%s:%d)",   \
                         cudaGetErrorString(e__), __FILE__, __LINE__); \
            return (int)e__;                                 \
        }                                                    \
        return 0;                                            \
    } while (0)

// TF 'SAME' padding: out = ceil(in/s), extra pad goes bottom/right (SURVEY App. A).
static inline void dh_same_pad(int in, int k, int s, int* out, int* before) {
    int o = (in + s - 1) / s;
    int total = (o - 1) * s + k - in;
    if (total < 0) total = 0;
    *out = o;
    *before = total / 2;
}

static inline int dh_out_size(int in, int k, int s, int pad_same, int* before) {
    int o;
    if (pad_same) {
        dh_same_pad(in, k, s, &o, before);
    } else {
        o = (in - k) / s + 1;
        *before = 0;
    }
    return o;
}

static inline bool dh_aligned16(const void* p) { return (((uintptr_t)p) & 15u) == 0; }

// float2 arithmetic.  sm_90 has no packed fp32 instructions: two scalar round-to-nearest operations, the same
// results per component as a packed FFMA2 / FADD2 / FMUL2.
__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c) {
    return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}
__device__ __forceinline__ float2 fadd2(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ float2 fmul2(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
