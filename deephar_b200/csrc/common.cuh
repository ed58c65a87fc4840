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
    int last_conv_path;   // DhConvPath (conv_params.cuh): the kernel that served the last convolution
    int share_a;          // 1 = cluster pairs share the separable A tile (default), 0 = independent CTAs
    int sep_tma;          // 1 = TMA-staged separable kernel (conv_sep.cu) where it applies (default)
    int pw_smallk;        // 1 = CUDA-core kernel for wide 1x1 convs with Cin <= 64 (conv_simt.cu) (default)
    int sam3d_stream;     // 1 = cluster-split streaming kernel for the volumetric head (softargmax.cu) (default)
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

// ---- PTX wrappers shared by the TMA-fed kernels (the wgmma convolutions, the streaming soft-argmax heads) ----
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("{\n .reg .b64 st;\n mbarrier.arrive.shared::cta.b64 st, [%0];\n}" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("{\n .reg .b64 st;\n mbarrier.arrive.expect_tx.shared::cta.b64 st, [%0], %1;\n}" ::"r"(bar), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    uint32_t ok;
    do {
        asm volatile(
            "{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n selp.u32 %0, 1, 0, p;\n}"
            : "=r"(ok)
            : "r"(bar), "r"(parity)
            : "memory");
    } while (!ok);
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
// 1-D bulk copy global -> shared memory, completion counted on the mbarrier as transaction bytes
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
                 "l"(src), "r"(bytes), "r"(bar)
                 : "memory");
}
// ---- clusters: rank, shared-memory address in a peer CTA, full-cluster barrier ----
__device__ __forceinline__ uint32_t cluster_ctarank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
__device__ __forceinline__ uint32_t mapa_peer(uint32_t local_addr, uint32_t peer) {
    uint32_t r;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(local_addr), "r"(peer));
    return r;
}
__device__ __forceinline__ void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}

// opt-in dynamic shared memory, set once per kernel (and again only if a launch needs more): keeps the launch
// path free of attribute calls -- forwards are captured into CUDA graphs (deephar_b200/model.py)
template <auto Kernel>
static inline cudaError_t ensure_smem(size_t smem) {
    static size_t cur = 0;
    if (smem <= cur) return cudaSuccess;
    cudaError_t e = cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e == cudaSuccess) cur = smem;
    return e;
}

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
