// Streaming soft-argmax for large dense heat-maps (the 32x32x48 ReceptionNet maps: 196 608 B per
// frame per block) -- the kernel behind the "softargmax HBM GB/s" figure.
//
// replaces the same reference layers as softargmax.cu (channel_softmax_2d + the two grid
// SeparableConv2D + joint probability on the raw maps + context aggregation:
// activations.py:3-16, layers.py:160-200, blocks.py:217-343, reception.py:167-182).
//
// HBM-bound design (H100 SXM: 3.35 TB/s over 132 SMs, ~13 B/clk/SM): persistent CTAs (one per SM) loop over frames; a
// producer thread streams each frame through a ring of shared-memory stages with 1-D TMA bulk
// copies (cp.async.bulk + mbarrier complete_tx: ~150 KB in flight per SM, no registers held);
// 12 consumer warps own (column, channel-quad) pairs and keep ONLINE softmax statistics in
// registers (running max, sum, sum*y; sum*x follows from the fixed column), plus the running
// max of the 2x2 window sums of the raw map.  Nothing but 16 x 3 floats per frame is written.
#include <float.h>
#include "common.cuh"

namespace sstream {

constexpr int STAGES = 6;
constexpr int ROWS_PER_CHUNK = 4;

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("{\n .reg .b64 st;\n mbarrier.arrive.shared::cta.b64 st, [%0];\n}" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
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
__device__ __forceinline__ float ex2_approx(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
                 "l"(src), "r"(bytes), "r"(bar)
                 : "memory");
}

struct Params {
    const float* h;
    int N, H, W, C;
    int nj, n_ctx;          // n_ctx > 0: context aggregation; else plain (pose (N,C,2), conf (N,C,1))
    float alpha_mix;
    float* out_pose;
    float* out_conf;
    int chunks_per_frame;
    int chunk_floats;       // ROWS_PER_CHUNK * W * C
};

// consumer threads: NCONS = W * C/4, thread -> (column c = t / Q, channel quad q = t % Q)
__global__ void __launch_bounds__(512, 1) sam_stream_kernel(Params p) {
    extern __shared__ __align__(128) uint8_t smem_raw[];
    const int Q = p.C >> 2;
    const int NCONS = p.W * Q;
    const int tid = threadIdx.x;
    float* ring = reinterpret_cast<float*>(smem_raw);
    float* s_red = ring + (size_t)STAGES * p.chunk_floats;           // [4][W][C] : m, s, sy, wmax
    float* s_res = s_red + 4 * p.W * p.C;                            // [3][C]    : x, y, conf
    float* s_gy = s_res + 3 * p.C;                                   // [H] : linspace(0,1,H) as float32
    uint64_t* bars = reinterpret_cast<uint64_t*>(s_gy + p.H + ((3 * p.C + p.H) & 1));
    const uint32_t bar_full = smem_u32(bars), bar_empty = smem_u32(bars + STAGES);
    const int ncons_warps = (NCONS + 31) >> 5;

    {
        const double ystep = p.H > 1 ? 1.0 / (double)(p.H - 1) : 0.0;   // np.linspace(0,1,H) -> float32
        for (int i = tid; i < p.H; i += blockDim.x) s_gy[i] = (p.H > 1 && i == p.H - 1) ? 1.0f : (float)(i * ystep);
    }
    if (tid == 0) {
        for (int s = 0; s < STAGES; ++s) {
            mbar_init(bar_full + 8 * s, 1);
            mbar_init(bar_empty + 8 * s, ncons_warps);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    const int frames_mine = (p.N - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;
    const int total_chunks = frames_mine * p.chunks_per_frame;
    const uint32_t chunk_bytes = (uint32_t)p.chunk_floats * 4u;

    if (tid >= NCONS) {
        // ===================== producer (one thread of the last warp) =====================
        if (tid == (ncons_warps << 5)) {
            for (int i = 0; i < total_chunks; ++i) {
                const int s = i % STAGES;
                const uint32_t it = (uint32_t)(i / STAGES);
                mbar_wait(bar_empty + 8 * s, (it & 1) ^ 1);
                const int f = blockIdx.x + (i / p.chunks_per_frame) * gridDim.x;
                const int ck = i % p.chunks_per_frame;
                const float* src = p.h + ((size_t)f * p.chunks_per_frame + ck) * p.chunk_floats;
                mbar_expect_tx(bar_full + 8 * s, chunk_bytes);
                bulk_g2s(smem_u32(ring + (size_t)s * p.chunk_floats), src, chunk_bytes, bar_full + 8 * s);
            }
        }
        return;
    }

    // ===================== consumers =====================
    // e = ex2((v - m) * log2e): the difference is formed first (exact for nearby values), then one
    // packed multiply and one MUFU.EX2 per element; sums use packed f32x2 adds / FMAs.
    const int c = tid / Q, q = tid - c * Q;
    const int lane = tid & 31;
    const bool has_right = c + 1 < p.W;
    constexpr float LOG2E = 1.4426950408889634f;
    int chunk_idx = 0;
    for (int fi = 0; fi < frames_mine; ++fi) {
        const int f = blockIdx.x + fi * gridDim.x;
        float m2[4] = {-FLT_MAX, -FLT_MAX, -FLT_MAX, -FLT_MAX};
        float2 s01 = make_float2(0.f, 0.f), s23 = make_float2(0.f, 0.f);
        float2 sy01 = make_float2(0.f, 0.f), sy23 = make_float2(0.f, 0.f);
        float wm[4] = {-FLT_MAX, -FLT_MAX, -FLT_MAX, -FLT_MAX};
        float2 pp01 = make_float2(0.f, 0.f), pp23 = make_float2(0.f, 0.f);   // previous row: own + right
        for (int ck = 0; ck < p.chunks_per_frame; ++ck, ++chunk_idx) {
            const int st = chunk_idx % STAGES;
            const uint32_t it = (uint32_t)(chunk_idx / STAGES);
            mbar_wait(bar_full + 8 * st, it & 1);
            const float* base = ring + (size_t)st * p.chunk_floats + (size_t)c * p.C + q * 4;
            float4 v[ROWS_PER_CHUNK], vr[ROWS_PER_CHUNK];
#pragma unroll
            for (int r = 0; r < ROWS_PER_CHUNK; ++r) {
                v[r] = *reinterpret_cast<const float4*>(base + (size_t)r * p.W * p.C);
                vr[r] = has_right ? *reinterpret_cast<const float4*>(base + (size_t)r * p.W * p.C + p.C)
                                  : make_float4(0.f, 0.f, 0.f, 0.f);
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(bar_empty + 8 * st);      // this warp is done with the stage
            // chunk maxima -> at most one rescale per chunk
            float cm[4] = {v[0].x, v[0].y, v[0].z, v[0].w};
#pragma unroll
            for (int r = 1; r < ROWS_PER_CHUNK; ++r) {
                cm[0] = fmaxf(cm[0], v[r].x); cm[1] = fmaxf(cm[1], v[r].y);
                cm[2] = fmaxf(cm[2], v[r].z); cm[3] = fmaxf(cm[3], v[r].w);
            }
            float sc[4] = {1.f, 1.f, 1.f, 1.f};
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                if (cm[e] > m2[e]) {
                    sc[e] = ex2_approx((m2[e] - cm[e]) * LOG2E);
                    m2[e] = cm[e];
                }
            }
            s01.x *= sc[0]; s01.y *= sc[1]; s23.x *= sc[2]; s23.y *= sc[3];
            sy01.x *= sc[0]; sy01.y *= sc[1]; sy23.x *= sc[2]; sy23.y *= sc[3];
            const float2 nm01 = make_float2(-m2[0], -m2[1]), nm23 = make_float2(-m2[2], -m2[3]);
            const float2 l2 = make_float2(LOG2E, LOG2E);
#pragma unroll
            for (int r = 0; r < ROWS_PER_CHUNK; ++r) {
                const int row = ck * ROWS_PER_CHUNK + r;
                const float gy = s_gy[row];
                const float2 a01 = fmul2(fadd2(make_float2(v[r].x, v[r].y), nm01), l2);
                const float2 a23 = fmul2(fadd2(make_float2(v[r].z, v[r].w), nm23), l2);
                const float2 e01 = make_float2(ex2_approx(a01.x), ex2_approx(a01.y));
                const float2 e23 = make_float2(ex2_approx(a23.x), ex2_approx(a23.y));
                s01 = fadd2(s01, e01);
                s23 = fadd2(s23, e23);
                const float2 g2 = make_float2(gy, gy);
                sy01 = ffma2(e01, g2, sy01);
                sy23 = ffma2(e23, g2, sy23);
                // 2x2 window with top-left corner (row-1, c), raw values: (own + right) of both rows
                const float2 cp01 = fadd2(make_float2(v[r].x, v[r].y), make_float2(vr[r].x, vr[r].y));
                const float2 cp23 = fadd2(make_float2(v[r].z, v[r].w), make_float2(vr[r].z, vr[r].w));
                if (has_right && row > 0) {
                    const float2 w01 = fadd2(pp01, cp01), w23 = fadd2(pp23, cp23);
                    wm[0] = fmaxf(wm[0], w01.x); wm[1] = fmaxf(wm[1], w01.y);
                    wm[2] = fmaxf(wm[2], w23.x); wm[3] = fmaxf(wm[3], w23.y);
                }
                pp01 = cp01;
                pp23 = cp23;
            }
        }
        const float m[4] = {m2[0], m2[1], m2[2], m2[3]};
        const float s[4] = {s01.x, s01.y, s23.x, s23.y};
        const float sy[4] = {sy01.x, sy01.y, sy23.x, sy23.y};
        // ---- combine the W columns of every channel ----
        const int WC = p.W * p.C;
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const int idx = c * p.C + q * 4 + e;
            s_red[0 * WC + idx] = m[e];
            s_red[1 * WC + idx] = s[e];
            s_red[2 * WC + idx] = sy[e];
            s_red[3 * WC + idx] = wm[e];
        }
        asm volatile("bar.sync 1, %0;" ::"r"(ncons_warps << 5) : "memory");
        if (tid < p.C) {
            float M = -FLT_MAX, Wm = -FLT_MAX;
            for (int cc = 0; cc < p.W; ++cc) {
                M = fmaxf(M, s_red[0 * WC + cc * p.C + tid]);
                Wm = fmaxf(Wm, s_red[3 * WC + cc * p.C + tid]);
            }
            float S = 0.f, SX = 0.f, SY = 0.f;
            const double xstep = p.W > 1 ? 1.0 / (double)(p.W - 1) : 0.0;
            for (int cc = 0; cc < p.W; ++cc) {
                const float sc = __expf(s_red[0 * WC + cc * p.C + tid] - M);
                const float sv = s_red[1 * WC + cc * p.C + tid] * sc;
                const float gxc = (p.W > 1 && cc == p.W - 1) ? 1.0f : (float)(cc * xstep);
                S += sv;
                SX = fmaf(sv, gxc, SX);
                SY = fmaf(s_red[2 * WC + cc * p.C + tid], sc, SY);
            }
            const float den = fmaxf(S, 1e-7f);
            s_res[0 * p.C + tid] = SX / den;
            s_res[1 * p.C + tid] = SY / den;
            s_res[2 * p.C + tid] = Wm;
        }
        asm volatile("bar.sync 1, %0;" ::"r"(ncons_warps << 5) : "memory");
        if (p.n_ctx > 0) {
            if (tid < p.nj) {
                float pcs = 0.f, px = 0.f, py = 0.f;
                for (int i = 0; i < p.n_ctx; ++i) {
                    const int cc = p.nj + tid * p.n_ctx + i;
                    const float pc = s_res[2 * p.C + cc];
                    pcs += pc;
                    px = fmaf(s_res[0 * p.C + cc], pc, px);
                    py = fmaf(s_res[1 * p.C + cc], pc, py);
                }
                const float a = p.alpha_mix;
                p.out_pose[((size_t)f * p.nj + tid) * 2 + 0] = a * s_res[0 * p.C + tid] + (1.f - a) * (px / pcs);
                p.out_pose[((size_t)f * p.nj + tid) * 2 + 1] = a * s_res[1 * p.C + tid] + (1.f - a) * (py / pcs);
                p.out_conf[(size_t)f * p.nj + tid] = s_res[2 * p.C + tid];
            }
        } else if (tid < p.C) {
            p.out_pose[((size_t)f * p.C + tid) * 2 + 0] = s_res[0 * p.C + tid];
            p.out_pose[((size_t)f * p.C + tid) * 2 + 1] = s_res[1 * p.C + tid];
            p.out_conf[(size_t)f * p.C + tid] = s_res[2 * p.C + tid];
        }
        // s_red / s_res are rewritten only after the next frame's first bar.sync pair -> safe
    }
}

}  // namespace sstream

bool dh_sam_stream_supported(const dh_view* h, int conf_on_prob, float alpha, bool has_d, bool has_prob) {
    if (conf_on_prob != 0 || alpha != 1.0f || has_d || has_prob) return false;
    if (h->ld != h->c || (h->c & 3)) return false;
    if ((reinterpret_cast<uintptr_t>(h->p) & 15) != 0) return false;
    if (h->h % sstream::ROWS_PER_CHUNK != 0 || h->h < 2 || h->w < 2) return false;
    const int ncons = h->w * (h->c >> 2);
    if (ncons > 480 || ncons < 64 || (ncons & 31)) return false;
    const size_t chunk_bytes = (size_t)sstream::ROWS_PER_CHUNK * h->w * h->c * 4;
    if (chunk_bytes % 16 != 0) return false;
    const size_t smem = sstream::STAGES * chunk_bytes + (size_t)(4 * h->w * h->c + 3 * h->c + h->h + 2) * 4 + 2 * sstream::STAGES * 8 + 128;
    if (smem > 227 * 1024) return false;
    if ((size_t)h->h * h->w * h->c * 4 < 64 * 1024) return false;    // small maps: the staged kernel is fine
    return true;
}

int dh_sam_stream_launch(dh_ctx* ctx, const dh_view* h, int nj, int n_ctx, float alpha_mix, float* out_pose,
                         float* out_conf, void* stream) {
    using namespace sstream;
    Params p;
    p.h = h->p; p.N = h->n; p.H = h->h; p.W = h->w; p.C = h->c;
    p.nj = nj; p.n_ctx = n_ctx; p.alpha_mix = alpha_mix;
    p.out_pose = out_pose; p.out_conf = out_conf;
    p.chunks_per_frame = h->h / ROWS_PER_CHUNK;
    p.chunk_floats = ROWS_PER_CHUNK * h->w * h->c;
    const int ncons = h->w * (h->c >> 2);
    const int threads = ((ncons + 31) / 32) * 32 + 32;
    const size_t smem = (size_t)STAGES * p.chunk_floats * 4 + (size_t)(4 * h->w * h->c + 3 * h->c + h->h + 2) * 4 +
                        2 * STAGES * 8 + 128;
    cudaError_t e = cudaFuncSetAttribute(sam_stream_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) {
        dh_set_error("dh_sam_stream_launch: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
        return (int)e;
    }
    int grid = h->n < ctx->num_sms ? h->n : ctx->num_sms;
    sam_stream_kernel<<<grid, threads, smem, (cudaStream_t)stream>>>(p);
    DH_LAUNCH_EPILOGUE(ctx, 1);
}

// =====================================================================================================
// Volumetric (3-D) head, streaming version: reception.py:193-222 pose_regression_3d (+ the merge model's
// vis_scale = 2, action.py:291-292).  h (N,H,W,D*nj), channel = d*nj + j, 1 114 112 B per frame at C3.
//
// A frame is split over a CLUSTER of 4 CTAs (pixel quarters): with one CTA per frame the b32 step of C3 would
// keep 32 of 132 SMs busy.  Each CTA streams its 256 pixels through a 4-stage ring of 16-pixel chunks (1-D TMA
// bulk copies, ~70 KB in flight per CTA, two CTAs per SM) and accumulates on the fly
//   hxy[p][j] = mean_d h[p][d*nj+j]   (complete for its own pixels -> kept in shared memory, 17 KB)
//   hz[c]    += h[p][c]               (partial sums over its pixels)
// then reduces hxy to per-joint online-softmax statistics (max, sum e, sum e*x, sum e*y).  After a cluster
// barrier rank 0 reads the other CTAs' partials over distributed shared memory, merges them, runs the 1-D
// soft-argmax over depth and writes (x, y, z) and the visibility: 17 x 4 floats per frame, nothing else.
// =====================================================================================================
namespace sam3ds {
using sstream::bulk_g2s;
using sstream::mbar_arrive;
using sstream::mbar_expect_tx;
using sstream::mbar_init;
using sstream::mbar_wait;
using sstream::smem_u32;

constexpr int PXC = 16;        // pixels per chunk
constexpr int STAGES = 4;
constexpr int CL = 4;          // CTAs per frame (cluster size)
constexpr int PARTS = 16;      // pixel partitions of the per-joint reduction

struct Params {
    const float* h;
    int N, H, W, nj, D;
    float vis_scale;
    float* out_pose;           // (N, nj, 3)
    float* out_vis;            // (N, nj, 1)
    int ncons;                 // consumer threads (multiple of 32): >= max(PXC * nj, C)
};

__device__ __forceinline__ uint32_t cluster_rank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
__device__ __forceinline__ void cluster_sync() {
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ float ld_peer(const float* local, uint32_t rank) {
    uint32_t a;
    float v;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(a) : "r"(smem_u32(local)), "r"(rank));
    asm volatile("ld.shared::cluster.f32 %0, [%1];" : "=f"(v) : "r"(a) : "memory");
    return v;
}
__device__ __forceinline__ float gridv(int i, int n) {      // np.linspace(0, 1, n)[i] as float32 (utils/math.py:6-19)
    const double step = n > 1 ? 1.0 / (double)(n - 1) : 0.0;
    return (n > 1 && i == n - 1) ? 1.0f : (float)(i * step);
}

__global__ void __launch_bounds__(512) sam3d_stream_kernel(Params p) {
    extern __shared__ __align__(128) uint8_t smem_raw[];
    const int nj = p.nj, D = p.D, C = nj * D, P = p.H * p.W;
    const int PL = P / CL;                         // pixels of this CTA
    const int nchunks = PL / PXC;
    const int tid = threadIdx.x;
    const uint32_t rank = cluster_rank();
    const int n = blockIdx.y;
    float* ring = reinterpret_cast<float*>(smem_raw);                 // [STAGES][PXC][C]
    float* s_hxy = ring + (size_t)STAGES * PXC * C;                   // [PL][nj]
    float* s_hz = s_hxy + (size_t)PL * nj;                            // [C]   partial sums over this CTA's pixels
    float* s_st = s_hz + C;                                           // [4][nj]: m, s, sx, sy of this CTA's pixels
    float* s_part = s_st + 4 * nj;                                    // [PARTS][4][nj]
    float* s_tot = s_part + PARTS * 4 * nj;                           // [C]   rank 0: hz over the whole frame
    uint64_t* bars = reinterpret_cast<uint64_t*>(s_tot + C + ((PL * nj + 2 * C + 4 * nj + PARTS * 4 * nj) & 1));
    const uint32_t bar_full = smem_u32(bars), bar_empty = smem_u32(bars + STAGES);
    const int ncons = p.ncons;
    const uint32_t chunk_bytes = (uint32_t)(PXC * C) * 4u;

    if (tid == 0) {
        for (int s = 0; s < STAGES; ++s) {
            mbar_init(bar_full + 8 * s, 1);
            mbar_init(bar_empty + 8 * s, ncons >> 5);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (tid >= ncons) {
        // ===================== producer (one thread of the last warp) =====================
        if (tid == ncons) {
            const float* src = p.h + ((size_t)n * P + (size_t)rank * PL) * C;
            for (int i = 0; i < nchunks; ++i) {
                const int s = i % STAGES;
                const uint32_t it = (uint32_t)(i / STAGES);
                mbar_wait(bar_empty + 8 * s, (it & 1) ^ 1);
                mbar_expect_tx(bar_full + 8 * s, chunk_bytes);
                bulk_g2s(smem_u32(ring + (size_t)s * PXC * C), src + (size_t)i * PXC * C, chunk_bytes, bar_full + 8 * s);
            }
        }
    } else {
        // ===================== consumers =====================
        const int pa = tid / nj, ja = tid - pa * nj;       // role A: (chunk pixel, joint) -> mean over depth
        const bool role_a = tid < PXC * nj, role_b = tid < C;
        const float inv_d = 1.0f / (float)D;
        float hz_acc = 0.f;
        for (int i = 0; i < nchunks; ++i) {
            const int s = i % STAGES;
            mbar_wait(bar_full + 8 * s, (uint32_t)(i / STAGES) & 1);
            const float* ck = ring + (size_t)s * PXC * C;
            if (role_a) {
                float a = 0.f;
                for (int d = 0; d < D; ++d) a += ck[pa * C + d * nj + ja];
                s_hxy[(i * PXC + pa) * nj + ja] = a * inv_d;
            }
            if (role_b) {
                float a = 0.f;
#pragma unroll
                for (int q = 0; q < PXC; ++q) a += ck[q * C + tid];
                hz_acc += a;
            }
            __syncwarp();
            if ((tid & 31) == 0) mbar_arrive(bar_empty + 8 * s);
        }
        if (role_b) s_hz[tid] = hz_acc;
        asm volatile("bar.sync 1, %0;" ::"r"(ncons) : "memory");
        // per-joint statistics of this CTA's pixels: PARTS partitions, then one combine
        if (tid < PARTS * nj) {
            const int j = tid % nj, part = tid / nj;
            float m = -FLT_MAX;
            for (int px = part; px < PL; px += PARTS) m = fmaxf(m, s_hxy[px * nj + j]);
            float sum = 0.f, sx = 0.f, sy = 0.f;
            for (int px = part; px < PL; px += PARTS) {
                const int gp = (int)rank * PL + px;
                const int row = gp / p.W, col = gp - row * p.W;
                const float e = expf(s_hxy[px * nj + j] - m);
                sum += e;
                sx = fmaf(e, gridv(col, p.W), sx);
                sy = fmaf(e, gridv(row, p.H), sy);
            }
            s_part[(part * 4 + 0) * nj + j] = m;
            s_part[(part * 4 + 1) * nj + j] = sum;
            s_part[(part * 4 + 2) * nj + j] = sx;
            s_part[(part * 4 + 3) * nj + j] = sy;
        }
        asm volatile("bar.sync 1, %0;" ::"r"(ncons) : "memory");
        if (tid < nj) {
            float M = -FLT_MAX;
            for (int q = 0; q < PARTS; ++q) M = fmaxf(M, s_part[(q * 4 + 0) * nj + tid]);
            float S = 0.f, SX = 0.f, SY = 0.f;
            for (int q = 0; q < PARTS; ++q) {
                const float sc = expf(s_part[(q * 4 + 0) * nj + tid] - M);
                S = fmaf(s_part[(q * 4 + 1) * nj + tid], sc, S);
                SX = fmaf(s_part[(q * 4 + 2) * nj + tid], sc, SX);
                SY = fmaf(s_part[(q * 4 + 3) * nj + tid], sc, SY);
            }
            s_st[0 * nj + tid] = M;
            s_st[1 * nj + tid] = S;
            s_st[2 * nj + tid] = SX;
            s_st[3 * nj + tid] = SY;
        }
    }
    cluster_sync();                       // every CTA's s_st / s_hz is complete and visible cluster-wide
    if (rank == 0) {
        if (tid < C) {
            float a = 0.f;
            for (uint32_t r = 0; r < CL; ++r) a += ld_peer(s_hz + tid, r);
            s_tot[tid] = a / (float)P;                                  // hz = mean over all pixels
        }
        __syncthreads();
        if (tid < nj) {
            float M = -FLT_MAX;
            for (uint32_t r = 0; r < CL; ++r) M = fmaxf(M, ld_peer(s_st + 0 * nj + tid, r));
            float S = 0.f, SX = 0.f, SY = 0.f;
            for (uint32_t r = 0; r < CL; ++r) {
                const float sc = expf(ld_peer(s_st + 0 * nj + tid, r) - M);
                S = fmaf(ld_peer(s_st + 1 * nj + tid, r), sc, S);
                SX = fmaf(ld_peer(s_st + 2 * nj + tid, r), sc, SX);
                SY = fmaf(ld_peer(s_st + 3 * nj + tid, r), sc, SY);
            }
            const float den = fmaxf(S, 1e-7f);                          // activations.py:12 clip of the denominator
            // zSAM: blocks.py:288-303 -- softmax over depth, grid (k + 0.5) / D (layers.py:141-146)
            float zm = -FLT_MAX;
            for (int d = 0; d < D; ++d) zm = fmaxf(zm, s_tot[d * nj + tid]);
            const double start = 1.0 / (2.0 * D), step = D > 1 ? ((1.0 - start) - start) / (double)(D - 1) : 0.0;
            float zs = 0.f, ze = 0.f;
            for (int d = 0; d < D; ++d) {
                const float e = expf(s_tot[d * nj + tid] - zm);
                const float g = (D > 1 && d == D - 1) ? (float)(1.0 - start) : (float)(d * step + start);
                zs += e;
                ze = fmaf(e, g, ze);
            }
            float* o = p.out_pose + ((size_t)n * nj + tid) * 3;
            o[0] = SX / den;
            o[1] = SY / den;
            o[2] = ze / zs;
            p.out_vis[(size_t)n * nj + tid] = 1.f / (1.f + expf(-p.vis_scale * (M + zm)));   // max_p hxy == M
        }
    }
    cluster_sync();                       // peers keep their shared memory alive until rank 0 has read it
}

}  // namespace sam3ds

bool dh_sam3d_stream_supported(const dh_view* h, int nj, int depth_maps) {
    using namespace sam3ds;
    const int C = nj * depth_maps, P = h->h * h->w;
    if (h->ld != h->c || (C & 3) || (reinterpret_cast<uintptr_t>(h->p) & 15)) return false;
    if (P % (CL * PXC) != 0 || h->h < 2 || h->w < 2) return false;
    if (PXC * nj > 480 || C > 480 || PARTS * nj > 480) return false;
    return true;
}

int dh_sam3d_stream_launch(dh_ctx* ctx, const dh_view* h, int nj, int depth_maps, float vis_scale, float* out_pose,
                           float* out_vis, void* stream) {
    using namespace sam3ds;
    Params p;
    p.h = h->p; p.N = h->n; p.H = h->h; p.W = h->w; p.nj = nj; p.D = depth_maps; p.vis_scale = vis_scale;
    p.out_pose = out_pose; p.out_vis = out_vis;
    const int C = nj * depth_maps, PL = h->h * h->w / CL;
    int need = PXC * nj > C ? PXC * nj : C;
    if (PARTS * nj > need) need = PARTS * nj;
    p.ncons = (need + 31) / 32 * 32;
    const int threads = p.ncons + 32;
    const size_t smem = ((size_t)STAGES * PXC * C + (size_t)PL * nj + 2 * C + 4 * nj + PARTS * 4 * nj + 2) * 4 + 2 * STAGES * 8 + 128;
    static size_t cur = 0;
    if (smem > cur) {
        cudaError_t e = cudaFuncSetAttribute(sam3d_stream_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) {
            dh_set_error("dh_sam3d_stream_launch: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
            return (int)e;
        }
        cur = smem;
    }
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(CL, h->n);
    cfg.blockDim = dim3(threads);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = (cudaStream_t)stream;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeClusterDimension;
    at[0].val.clusterDim.x = CL; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
    cfg.attrs = at;
    cfg.numAttrs = 1;
    cudaError_t e = cudaLaunchKernelEx(&cfg, sam3d_stream_kernel, p);
    if (e != cudaSuccess) {
        dh_set_error("dh_sam3d_stream_launch: %s", cudaGetErrorString(e));
        return (int)e;
    }
    DH_LAUNCH_EPILOGUE(ctx, 1);
}
