// Soft-argmax heads: spatial softmax + coordinate expectation + joint confidence in one
// pass over the heat-maps; the probability maps are never written back to HBM.
//
// replaces (reference, per prediction block): channel_softmax_2d (activations.py:3-16),
// the two fixed-weight SeparableConv2D(R x R, valid) "grid" convolutions + squeezes +
// concat of lin_interpolation_2d / softargmax2d (layers.py:122-129,160-200, grid from
// utils/math.py:6-19), AveragePooling2D*4 + GlobalMaxPooling2D of keypoint_confidence /
// build_joints_probability (layers.py:107-119, blocks.py:328-343), the context
// aggregation model (blocks.py:217-285), the depth expectation (spnet.py:201-205) and the
// volumetric marginal regression (reception.py:193-222).
//
// Two kinds of kernel per head:
//   staged     (softargmax2d_kernel, softargmax3d_kernel): any H, W, C; one CTA per frame, frame staged in
//              shared memory;
//   streaming  (sam_stream_kernel, sam3d_stream_kernel): large dense maps streamed through a TMA ring, the
//              kernels behind the "softargmax HBM GB/s" figure.
// launch_sam2d / launch_sam3d take the streaming kernel where its plan accepts the input, else the staged one.
#include <float.h>
#include "common.cuh"

namespace {

constexpr float K_EPSILON = 1e-7f;  // keras.backend.epsilon(), activations.py:12

struct SamParams {
    const float* h; int ldh;
    const float* d; int ldd;
    int N, H, W, C;
    float alpha;
    int conf_on_prob;
    float* out_pose; int pose_dim;
    float* out_conf;
    float* prob; int ldp;
    int nj, n_ctx; float alpha_mix;  // context aggregation when n_ctx > 0
};

__device__ __forceinline__ float sigmoidf_(float x) { return 1.f / (1.f + expf(-x)); }

// np.linspace(0, 1, n)[i] cast to float32 (utils/math.py:8-19): i * (1/(n-1)) in double, last = 1.
__device__ __forceinline__ float linspace01(int i, int n) {
    const double step = n > 1 ? 1.0 / (double)(n - 1) : 0.0;
    return (n > 1 && i == n - 1) ? 1.0f : (float)(i * step);
}

// zSAM (blocks.py:288-303): softmax over the D depth bins of one joint's depth marginal hz[d * nj], grid
// (k + 0.5) / D (layers.py:141-146).  Returns (expected depth, max of the marginal).
__device__ __forceinline__ float2 zsam(const float* hz, int nj, int D) {
    float zm = -FLT_MAX;
    for (int d = 0; d < D; ++d) zm = fmaxf(zm, hz[d * nj]);
    const double start = 1.0 / (2.0 * D), step = D > 1 ? ((1.0 - start) - start) / (double)(D - 1) : 0.0;
    float zs = 0.f, ze = 0.f;
    for (int d = 0; d < D; ++d) {
        const float e = expf(hz[d * nj] - zm);
        const float g = (D > 1 && d == D - 1) ? (float)(1.0 - start) : (float)(d * step + start);
        zs += e;
        ze = fmaf(e, g, ze);
    }
    return make_float2(ze / zs, zm);
}

// Output of a 2-D head for frame n from the per-channel statistics in shared memory, s_res[0 * C + c] = E[x],
// [1 * C + c] = E[y], [2 * C + c] = conf: the context aggregation (blocks.py:217-285; channels [0, nj)
// specialised, then nj groups of n_ctx context maps) when n_ctx > 0, else x, y of every channel at the start of
// its pose_dim-float pose row, and its confidence.
__device__ __forceinline__ void sam2d_out(const float* s_res, int C, int nj, int n_ctx, float alpha_mix, int n,
                                          float* out_pose, int pose_dim, float* out_conf) {
    const int tid = threadIdx.x;
    if (n_ctx > 0) {
        if (tid < nj) {
            float pcs = 0.f, px = 0.f, py = 0.f;
            for (int i = 0; i < n_ctx; ++i) {
                const int cc = nj + tid * n_ctx + i;
                const float pc = s_res[2 * C + cc];
                pcs += pc;
                px = fmaf(s_res[0 * C + cc], pc, px);
                py = fmaf(s_res[1 * C + cc], pc, py);
            }
            const float a = alpha_mix;
            out_pose[((size_t)n * nj + tid) * 2 + 0] = a * s_res[0 * C + tid] + (1.f - a) * (px / pcs);
            out_pose[((size_t)n * nj + tid) * 2 + 1] = a * s_res[1 * C + tid] + (1.f - a) * (py / pcs);
            out_conf[(size_t)n * nj + tid] = s_res[2 * C + tid];
        }
    } else if (tid < C) {
        float* o = out_pose + ((size_t)n * C + tid) * pose_dim;
        o[0] = s_res[0 * C + tid];
        o[1] = s_res[1 * C + tid];
        out_conf[(size_t)n * C + tid] = s_res[2 * C + tid];
    }
}

// Per-channel soft-argmax statistics of an smem-resident frame s_h[P][C].
// On return (after the trailing __syncthreads) s_res holds, per channel c:
//   s_res[0*C+c] = E[x], [1*C+c] = E[y], [2*C+c] = conf, [3*C+c] = z, [4*C+c] = clipped denominator
// and s_h holds exp(alpha*h - max).  d (global, may be NULL) is the depth map of this frame.
__device__ void sam_stats(float* s_h, const float* s_gx, const float* s_gy, float* s_red, float* s_res,
                          int H, int W, int C, float alpha, int conf_on_prob, const float* d, int ldd) {
    const int tid = threadIdx.x, T = blockDim.x;
    const int P = H * W;
    const int parts = T / C;
    const bool active = tid < parts * C;
    const int c = tid % C, part = tid / C;

    float m = -FLT_MAX, wv = -FLT_MAX;
    if (active) {
        for (int pix = part; pix < P; pix += parts) {
            float v = s_h[pix * C + c];
            m = fmaxf(m, alpha * v);
            if (!conf_on_prob) {
                int row = pix / W, col = pix - row * W;
                if (row + 1 < H && col + 1 < W)
                    wv = fmaxf(wv, (v + s_h[(pix + 1) * C + c]) + (s_h[(pix + W) * C + c] + s_h[(pix + W + 1) * C + c]));
            }
        }
        s_red[tid] = m;
    }
    __syncthreads();
    if (active) {
        m = -FLT_MAX;
        for (int q = 0; q < parts; ++q) m = fmaxf(m, s_red[q * C + c]);
    }
    __syncthreads();

    float s = 0.f, sx = 0.f, sy = 0.f, z = 0.f;
    if (active) {
        for (int pix = part; pix < P; pix += parts) {
            int row = pix / W, col = pix - row * W;
            float e = expf(alpha * s_h[pix * C + c] - m);
            s_h[pix * C + c] = e;
            s += e;
            sx = fmaf(e, s_gx[col], sx);
            sy = fmaf(e, s_gy[row], sy);
            if (d) z = fmaf(e, sigmoidf_(__ldg(d + (size_t)pix * ldd + c)), z);
        }
    }
    __syncthreads();
    if (active && conf_on_prob) {
        for (int pix = part; pix < P; pix += parts) {
            int row = pix / W, col = pix - row * W;
            if (row + 1 < H && col + 1 < W)
                wv = fmaxf(wv, (s_h[pix * C + c] + s_h[(pix + 1) * C + c]) +
                                   (s_h[(pix + W) * C + c] + s_h[(pix + W + 1) * C + c]));
        }
    }
    if (active) {
        s_red[0 * T + tid] = s;
        s_red[1 * T + tid] = sx;
        s_red[2 * T + tid] = sy;
        s_red[3 * T + tid] = z;
        s_red[4 * T + tid] = wv;
    }
    __syncthreads();
    if (tid < C) {
        float S = 0.f, SX = 0.f, SY = 0.f, Z = 0.f, Wm = -FLT_MAX;
        for (int q = 0; q < parts; ++q) {
            int i = q * C + tid;
            S += s_red[0 * T + i];
            SX += s_red[1 * T + i];
            SY += s_red[2 * T + i];
            Z += s_red[3 * T + i];
            Wm = fmaxf(Wm, s_red[4 * T + i]);
        }
        float den = fmaxf(S, K_EPSILON);
        s_res[0 * C + tid] = SX / den;
        s_res[1 * C + tid] = SY / den;
        s_res[2 * C + tid] = conf_on_prob ? Wm / den : Wm;
        s_res[3 * C + tid] = Z / den;
        s_res[4 * C + tid] = den;
    }
    __syncthreads();
}

__global__ void __launch_bounds__(512) softargmax2d_kernel(SamParams p) {
    extern __shared__ __align__(16) float smem[];
    const int tid = threadIdx.x, T = blockDim.x;
    const int P = p.H * p.W, C = p.C;
    const int PC4 = (P * C + 3) & ~3;
    float* s_h = smem;
    float* s_gx = s_h + PC4;
    float* s_gy = s_gx + p.W;
    float* s_red = s_gy + p.H;
    float* s_res = s_red + 5 * T;
    const int n = blockIdx.x;

    for (int i = tid; i < p.W; i += T) s_gx[i] = linspace01(i, p.W);
    for (int i = tid; i < p.H; i += T) s_gy[i] = linspace01(i, p.H);
    const float* hb = p.h + (size_t)n * P * p.ldh;
    if ((C & 3) == 0 && (p.ldh & 3) == 0 && ((uintptr_t)p.h & 15) == 0) {
        const int C4 = C >> 2;
        for (int i = tid; i < P * C4; i += T) {
            int pix = i / C4, q = i - pix * C4;
            float4 v = __ldg(reinterpret_cast<const float4*>(hb + (size_t)pix * p.ldh) + q);
            reinterpret_cast<float4*>(s_h)[i] = v;
        }
    } else {
        for (int i = tid; i < P * C; i += T) {
            int pix = i / C, c = i - pix * C;
            s_h[i] = __ldg(hb + (size_t)pix * p.ldh + c);
        }
    }
    __syncthreads();

    const float* db = p.d ? p.d + (size_t)n * P * p.ldd : nullptr;
    sam_stats(s_h, s_gx, s_gy, s_red, s_res, p.H, p.W, C, p.alpha, p.conf_on_prob, db, p.ldd);

    sam2d_out(s_res, C, p.nj, p.n_ctx, p.alpha_mix, n, p.out_pose, p.pose_dim, p.out_conf);
    if (p.n_ctx > 0) return;
    if (p.pose_dim == 3 && tid < C) p.out_pose[((size_t)n * C + tid) * 3 + 2] = s_res[3 * C + tid];
    if (p.prob) {
        float* pb = p.prob + (size_t)n * P * p.ldp;
        for (int i = tid; i < P * C; i += T) {
            int pix = i / C, c = i - pix * C;
            pb[(size_t)pix * p.ldp + c] = s_h[i] / s_res[4 * C + c];
        }
    }
}

// ---------------------------------------------------------------------------
// Volumetric (reception 3-D) head: reception.py:193-222.
// h (N,H,W,D*nj) with channel = d*nj + j is streamed ONCE through shared memory in
// chunks of SAM3D_PCH pixels; both marginals (mean over d -> hxy, mean over hw -> hz) are
// accumulated on the fly, then the 2-D / 1-D soft-argmax run on the smem-resident
// marginals.
// ---------------------------------------------------------------------------
constexpr int SAM3D_PCH = 32;

struct Sam3dParams {
    const float* h; int ldh;
    int N, H, W, nj, D;
    float* out_pose; float* out_vis;
    float vis_scale;            // visible = sigmoid(vis_scale * (max hxy + max hz)): 1 reception.py:217-220, 2 action.py:291-292
    float* prob; int ldp;       // optional: channel_softmax_2d(hxy) (N,H,W,nj) for the kronecker product (action.py:294-295)
};

__global__ void __launch_bounds__(512) softargmax3d_kernel(Sam3dParams p) {
    extern __shared__ __align__(16) float smem[];
    const int tid = threadIdx.x, T = blockDim.x;
    const int P = p.H * p.W, nj = p.nj, D = p.D, C = nj * D;
    const int PJ4 = (P * nj + 3) & ~3;
    float* s_hxy = smem;                      // [P][nj]
    float* s_chunk = s_hxy + PJ4;             // [SAM3D_PCH][C]
    float* s_hz = s_chunk + SAM3D_PCH * C;    // [C]
    float* s_gx = s_hz + ((C + 3) & ~3);
    float* s_gy = s_gx + p.W;
    float* s_red = s_gy + p.H;
    float* s_res = s_red + 5 * T;
    const int n = blockIdx.x;

    for (int i = tid; i < p.W; i += T) s_gx[i] = linspace01(i, p.W);
    for (int i = tid; i < p.H; i += T) s_gy[i] = linspace01(i, p.H);
    const float* hb = p.h + (size_t)n * P * p.ldh;
    const bool vec = (C & 3) == 0 && (p.ldh & 3) == 0 && ((uintptr_t)p.h & 15) == 0;
    const int nch_slots = (C + T - 1) / T;  // channels per thread for the hz accumulation (<= 2)
    float hz_acc[2] = {0.f, 0.f};

    for (int p0 = 0; p0 < P; p0 += SAM3D_PCH) {
        const int np = min(SAM3D_PCH, P - p0);
        if (vec) {
            const int C4 = C >> 2;
            for (int i = tid; i < np * C4; i += T) {
                int pl = i / C4, q = i - pl * C4;
                reinterpret_cast<float4*>(s_chunk)[i] =
                    __ldg(reinterpret_cast<const float4*>(hb + (size_t)(p0 + pl) * p.ldh) + q);
            }
        } else {
            for (int i = tid; i < np * C; i += T) {
                int pl = i / C, c = i - pl * C;
                s_chunk[i] = __ldg(hb + (size_t)(p0 + pl) * p.ldh + c);
            }
        }
        __syncthreads();
        for (int sl = 0; sl < nch_slots; ++sl) {
            int ch = tid + sl * T;
            if (ch < C) {
                float a = 0.f;
                for (int pl = 0; pl < np; ++pl) a += s_chunk[pl * C + ch];
                hz_acc[sl] += a;
            }
        }
        for (int i = tid; i < np * nj; i += T) {
            int pl = i / nj, j = i - pl * nj;
            float a = 0.f;
            for (int dd = 0; dd < D; ++dd) a += s_chunk[pl * C + dd * nj + j];
            s_hxy[(p0 + pl) * nj + j] = a / (float)D;
        }
        __syncthreads();
    }
    for (int sl = 0; sl < nch_slots; ++sl) {
        int ch = tid + sl * T;
        if (ch < C) s_hz[ch] = hz_acc[sl] / (float)P;
    }
    __syncthreads();

    // vxy = max over pixels of hxy, before sam_stats overwrites s_hxy with exponentials:
    // sam_stats' "raw" confidence slot is not used here, so compute the max directly.
    float vmax = -FLT_MAX;
    {
        const int parts = T / nj;
        if (tid < parts * nj) {
            int c = tid % nj, part = tid / nj;
            for (int pix = part; pix < P; pix += parts) vmax = fmaxf(vmax, s_hxy[pix * nj + c]);
            s_red[tid] = vmax;
        }
        __syncthreads();
        if (tid < nj) {
            vmax = -FLT_MAX;
            for (int q = 0; q < parts; ++q) vmax = fmaxf(vmax, s_red[q * nj + tid]);
        }
        __syncthreads();
    }
    sam_stats(s_hxy, s_gx, s_gy, s_red, s_res, p.H, p.W, nj, 1.0f, 1, nullptr, 0);

    if (tid < nj) {
        const float2 z = zsam(s_hz + tid, nj, D);
        float* o = p.out_pose + ((size_t)n * nj + tid) * 3;
        o[0] = s_res[0 * nj + tid];
        o[1] = s_res[1 * nj + tid];
        o[2] = z.x;
        p.out_vis[(size_t)n * nj + tid] = sigmoidf_(p.vis_scale * (vmax + z.y));
    }
    if (p.prob) {
        float* pb = p.prob + (size_t)n * P * p.ldp;
        for (int i = tid; i < P * nj; i += T) {
            int pix = i / nj, c = i - pix * nj;
            pb[(size_t)pix * p.ldp + c] = s_hxy[i] / s_res[4 * nj + c];
        }
    }
}

// =====================================================================================================
// Streaming 2-D head for large dense heat-maps (the 32x32x48 ReceptionNet maps: 196 608 B per frame per block).
//
// HBM-bound design (H100 SXM: 3.35 TB/s over 132 SMs, ~13 B/clk/SM): persistent CTAs (one per SM) loop over frames; a
// producer thread streams each frame through a ring of shared-memory stages with 1-D TMA bulk
// copies (cp.async.bulk + mbarrier complete_tx: ~150 KB in flight per SM, no registers held);
// 12 consumer warps own (column, channel-quad) pairs and keep ONLINE softmax statistics in
// registers (running max, sum, sum*y; sum*x follows from the fixed column), plus the running
// max of the 2x2 window sums of the raw map.  Nothing but 16 x 3 floats per frame is written.
// =====================================================================================================
constexpr int ST2_STAGES = 6;
constexpr int ST2_ROWS_PER_CHUNK = 4;

__device__ __forceinline__ float ex2_approx(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

struct SamStreamParams {
    const float* h;
    int N, H, W, C;
    int nj, n_ctx;          // n_ctx > 0: context aggregation; else plain (pose (N,C,2), conf (N,C,1))
    float alpha_mix;
    float* out_pose;
    float* out_conf;
    int chunks_per_frame;
    int chunk_floats;       // ST2_ROWS_PER_CHUNK * W * C
};

// consumer threads: NCONS = W * C/4, thread -> (column c = t / Q, channel quad q = t % Q)
__global__ void __launch_bounds__(512, 1) sam_stream_kernel(SamStreamParams p) {
    extern __shared__ __align__(128) uint8_t smem_raw[];
    const int Q = p.C >> 2;
    const int NCONS = p.W * Q;
    const int tid = threadIdx.x;
    float* ring = reinterpret_cast<float*>(smem_raw);
    float* s_red = ring + (size_t)ST2_STAGES * p.chunk_floats;       // [4][W][C] : m, s, sy, wmax
    float* s_res = s_red + 4 * p.W * p.C;                            // [3][C]    : x, y, conf
    float* s_gy = s_res + 3 * p.C;                                   // [H] : linspace(0,1,H) as float32
    uint64_t* bars = reinterpret_cast<uint64_t*>(s_gy + p.H + ((3 * p.C + p.H) & 1));
    const uint32_t bar_full = smem_u32(bars), bar_empty = smem_u32(bars + ST2_STAGES);
    const int ncons_warps = (NCONS + 31) >> 5;

    for (int i = tid; i < p.H; i += blockDim.x) s_gy[i] = linspace01(i, p.H);
    if (tid == 0) {
        for (int s = 0; s < ST2_STAGES; ++s) {
            mbar_init(bar_full + 8 * s, 1);
            mbar_init(bar_empty + 8 * s, ncons_warps);
        }
        fence_barrier_init();
    }
    __syncthreads();

    const int frames_mine = (p.N - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;
    const int total_chunks = frames_mine * p.chunks_per_frame;
    const uint32_t chunk_bytes = (uint32_t)p.chunk_floats * 4u;

    if (tid >= NCONS) {
        // ===================== producer (one thread of the last warp) =====================
        if (tid == (ncons_warps << 5)) {
            for (int i = 0; i < total_chunks; ++i) {
                const int s = i % ST2_STAGES;
                const uint32_t it = (uint32_t)(i / ST2_STAGES);
                mbar_wait(bar_empty + 8 * s, (it & 1) ^ 1);
                const int f = blockIdx.x + (i / p.chunks_per_frame) * gridDim.x;
                const int ck = i % p.chunks_per_frame;
                const float* src = p.h + ((size_t)f * p.chunks_per_frame + ck) * p.chunk_floats;
                mbar_arrive_expect_tx(bar_full + 8 * s, chunk_bytes);
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
            const int st = chunk_idx % ST2_STAGES;
            const uint32_t it = (uint32_t)(chunk_idx / ST2_STAGES);
            mbar_wait(bar_full + 8 * st, it & 1);
            const float* base = ring + (size_t)st * p.chunk_floats + (size_t)c * p.C + q * 4;
            float4 v[ST2_ROWS_PER_CHUNK], vr[ST2_ROWS_PER_CHUNK];
#pragma unroll
            for (int r = 0; r < ST2_ROWS_PER_CHUNK; ++r) {
                v[r] = *reinterpret_cast<const float4*>(base + (size_t)r * p.W * p.C);
                vr[r] = has_right ? *reinterpret_cast<const float4*>(base + (size_t)r * p.W * p.C + p.C)
                                  : make_float4(0.f, 0.f, 0.f, 0.f);
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(bar_empty + 8 * st);      // this warp is done with the stage
            // chunk maxima -> at most one rescale per chunk
            float cm[4] = {v[0].x, v[0].y, v[0].z, v[0].w};
#pragma unroll
            for (int r = 1; r < ST2_ROWS_PER_CHUNK; ++r) {
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
            for (int r = 0; r < ST2_ROWS_PER_CHUNK; ++r) {
                const int row = ck * ST2_ROWS_PER_CHUNK + r;
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
            for (int cc = 0; cc < p.W; ++cc) {
                const float sc = __expf(s_red[0 * WC + cc * p.C + tid] - M);
                const float sv = s_red[1 * WC + cc * p.C + tid] * sc;
                S += sv;
                SX = fmaf(sv, linspace01(cc, p.W), SX);
                SY = fmaf(s_red[2 * WC + cc * p.C + tid], sc, SY);
            }
            const float den = fmaxf(S, K_EPSILON);
            s_res[0 * p.C + tid] = SX / den;
            s_res[1 * p.C + tid] = SY / den;
            s_res[2 * p.C + tid] = Wm;
        }
        asm volatile("bar.sync 1, %0;" ::"r"(ncons_warps << 5) : "memory");
        sam2d_out(s_res, p.C, p.nj, p.n_ctx, p.alpha_mix, f, p.out_pose, 2, p.out_conf);
        // s_red / s_res are rewritten only after the next frame's first bar.sync pair -> safe
    }
}

// =====================================================================================================
// Streaming volumetric (3-D) head: reception.py:193-222 pose_regression_3d (+ the merge model's
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
constexpr int ST3_PXC = 16;        // pixels per chunk
constexpr int ST3_STAGES = 4;
constexpr int ST3_CL = 4;          // CTAs per frame (cluster size)
constexpr int ST3_PARTS = 16;      // pixel partitions of the per-joint reduction

struct Sam3dStreamParams {
    const float* h;
    int N, H, W, nj, D;
    float vis_scale;
    float* out_pose;           // (N, nj, 3)
    float* out_vis;            // (N, nj, 1)
    int ncons;                 // consumer threads (multiple of 32): >= max(ST3_PXC * nj, C)
};

__device__ __forceinline__ float ld_peer(const float* local, uint32_t rank) {
    float v;
    asm volatile("ld.shared::cluster.f32 %0, [%1];" : "=f"(v) : "r"(mapa_peer(smem_u32(local), rank)) : "memory");
    return v;
}

__global__ void __launch_bounds__(512) sam3d_stream_kernel(Sam3dStreamParams p) {
    extern __shared__ __align__(128) uint8_t smem_raw[];
    const int nj = p.nj, D = p.D, C = nj * D, P = p.H * p.W;
    const int PL = P / ST3_CL;                     // pixels of this CTA
    const int nchunks = PL / ST3_PXC;
    const int tid = threadIdx.x;
    const uint32_t rank = cluster_ctarank();
    const int n = blockIdx.y;
    float* ring = reinterpret_cast<float*>(smem_raw);                 // [ST3_STAGES][ST3_PXC][C]
    float* s_hxy = ring + (size_t)ST3_STAGES * ST3_PXC * C;           // [PL][nj]
    float* s_hz = s_hxy + (size_t)PL * nj;                            // [C]   partial sums over this CTA's pixels
    float* s_st = s_hz + C;                                           // [4][nj]: m, s, sx, sy of this CTA's pixels
    float* s_part = s_st + 4 * nj;                                    // [ST3_PARTS][4][nj]
    float* s_tot = s_part + ST3_PARTS * 4 * nj;                       // [C]   rank 0: hz over the whole frame
    uint64_t* bars = reinterpret_cast<uint64_t*>(s_tot + C + ((PL * nj + 2 * C + 4 * nj + ST3_PARTS * 4 * nj) & 1));
    const uint32_t bar_full = smem_u32(bars), bar_empty = smem_u32(bars + ST3_STAGES);
    const int ncons = p.ncons;
    const uint32_t chunk_bytes = (uint32_t)(ST3_PXC * C) * 4u;

    if (tid == 0) {
        for (int s = 0; s < ST3_STAGES; ++s) {
            mbar_init(bar_full + 8 * s, 1);
            mbar_init(bar_empty + 8 * s, ncons >> 5);
        }
        fence_barrier_init();
    }
    __syncthreads();

    if (tid >= ncons) {
        // ===================== producer (one thread of the last warp) =====================
        if (tid == ncons) {
            const float* src = p.h + ((size_t)n * P + (size_t)rank * PL) * C;
            for (int i = 0; i < nchunks; ++i) {
                const int s = i % ST3_STAGES;
                const uint32_t it = (uint32_t)(i / ST3_STAGES);
                mbar_wait(bar_empty + 8 * s, (it & 1) ^ 1);
                mbar_arrive_expect_tx(bar_full + 8 * s, chunk_bytes);
                bulk_g2s(smem_u32(ring + (size_t)s * ST3_PXC * C), src + (size_t)i * ST3_PXC * C, chunk_bytes,
                         bar_full + 8 * s);
            }
        }
    } else {
        // ===================== consumers =====================
        const int pa = tid / nj, ja = tid - pa * nj;       // role A: (chunk pixel, joint) -> mean over depth
        const bool role_a = tid < ST3_PXC * nj, role_b = tid < C;
        const float inv_d = 1.0f / (float)D;
        float hz_acc = 0.f;
        for (int i = 0; i < nchunks; ++i) {
            const int s = i % ST3_STAGES;
            mbar_wait(bar_full + 8 * s, (uint32_t)(i / ST3_STAGES) & 1);
            const float* ck = ring + (size_t)s * ST3_PXC * C;
            if (role_a) {
                float a = 0.f;
                for (int d = 0; d < D; ++d) a += ck[pa * C + d * nj + ja];
                s_hxy[(i * ST3_PXC + pa) * nj + ja] = a * inv_d;
            }
            if (role_b) {
                float a = 0.f;
#pragma unroll
                for (int q = 0; q < ST3_PXC; ++q) a += ck[q * C + tid];
                hz_acc += a;
            }
            __syncwarp();
            if ((tid & 31) == 0) mbar_arrive(bar_empty + 8 * s);
        }
        if (role_b) s_hz[tid] = hz_acc;
        asm volatile("bar.sync 1, %0;" ::"r"(ncons) : "memory");
        // per-joint statistics of this CTA's pixels: ST3_PARTS partitions, then one combine
        if (tid < ST3_PARTS * nj) {
            const int j = tid % nj, part = tid / nj;
            float m = -FLT_MAX;
            for (int px = part; px < PL; px += ST3_PARTS) m = fmaxf(m, s_hxy[px * nj + j]);
            float sum = 0.f, sx = 0.f, sy = 0.f;
            for (int px = part; px < PL; px += ST3_PARTS) {
                const int gp = (int)rank * PL + px;
                const int row = gp / p.W, col = gp - row * p.W;
                const float e = expf(s_hxy[px * nj + j] - m);
                sum += e;
                sx = fmaf(e, linspace01(col, p.W), sx);
                sy = fmaf(e, linspace01(row, p.H), sy);
            }
            s_part[(part * 4 + 0) * nj + j] = m;
            s_part[(part * 4 + 1) * nj + j] = sum;
            s_part[(part * 4 + 2) * nj + j] = sx;
            s_part[(part * 4 + 3) * nj + j] = sy;
        }
        asm volatile("bar.sync 1, %0;" ::"r"(ncons) : "memory");
        if (tid < nj) {
            float M = -FLT_MAX;
            for (int q = 0; q < ST3_PARTS; ++q) M = fmaxf(M, s_part[(q * 4 + 0) * nj + tid]);
            float S = 0.f, SX = 0.f, SY = 0.f;
            for (int q = 0; q < ST3_PARTS; ++q) {
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
    cluster_sync_all();                   // every CTA's s_st / s_hz is complete and visible cluster-wide
    if (rank == 0) {
        if (tid < C) {
            float a = 0.f;
            for (uint32_t r = 0; r < ST3_CL; ++r) a += ld_peer(s_hz + tid, r);
            s_tot[tid] = a / (float)P;                                  // hz = mean over all pixels
        }
        __syncthreads();
        if (tid < nj) {
            float M = -FLT_MAX;
            for (uint32_t r = 0; r < ST3_CL; ++r) M = fmaxf(M, ld_peer(s_st + 0 * nj + tid, r));
            float S = 0.f, SX = 0.f, SY = 0.f;
            for (uint32_t r = 0; r < ST3_CL; ++r) {
                const float sc = expf(ld_peer(s_st + 0 * nj + tid, r) - M);
                S = fmaf(ld_peer(s_st + 1 * nj + tid, r), sc, S);
                SX = fmaf(ld_peer(s_st + 2 * nj + tid, r), sc, SX);
                SY = fmaf(ld_peer(s_st + 3 * nj + tid, r), sc, SY);
            }
            const float den = fmaxf(S, K_EPSILON);
            const float2 z = zsam(s_tot + tid, nj, D);
            float* o = p.out_pose + ((size_t)n * nj + tid) * 3;
            o[0] = SX / den;
            o[1] = SY / den;
            o[2] = z.x;
            p.out_vis[(size_t)n * nj + tid] = sigmoidf_(p.vis_scale * (M + z.y));   // max_p hxy == M
        }
    }
    cluster_sync_all();                   // peers keep their shared memory alive until rank 0 has read it
}

// layers.py:478-508: out[n,j,f] = sum_p P[n,p,j] * Z[n,p,f].  grid (N, ceil(F/128)), 128 threads;
// P is staged in shared memory in chunks of 64 pixels, each thread owns one feature f.
constexpr int KR_MAXJ = 32, KR_PCH = 64;
__global__ void __launch_bounds__(128) kron_kernel(const float* pm, int ldpm, const float* z, int ldz,
                                                   int P, int nj, int F, float* out) {
    __shared__ float s_p[KR_PCH * KR_MAXJ];
    const int n = blockIdx.x;
    const int f = blockIdx.y * 128 + threadIdx.x;
    float acc[KR_MAXJ];
#pragma unroll
    for (int j = 0; j < KR_MAXJ; ++j) acc[j] = 0.f;
    const float* pb = pm + (size_t)n * P * ldpm;
    const float* zb = z + (size_t)n * P * ldz;
    for (int p0 = 0; p0 < P; p0 += KR_PCH) {
        int np = min(KR_PCH, P - p0);
        __syncthreads();
        for (int i = threadIdx.x; i < np * nj; i += 128) {
            int pl = i / nj, j = i - pl * nj;
            s_p[pl * KR_MAXJ + j] = __ldg(pb + (size_t)(p0 + pl) * ldpm + j);
        }
        __syncthreads();
        if (f < F) {
            for (int pl = 0; pl < np; ++pl) {
                float zv = __ldg(zb + (size_t)(p0 + pl) * ldz + f);
#pragma unroll
                for (int j = 0; j < KR_MAXJ; ++j)
                    if (j < nj) acc[j] = fmaf(s_p[pl * KR_MAXJ + j], zv, acc[j]);
            }
        }
    }
    if (f < F) {
#pragma unroll
        for (int j = 0; j < KR_MAXJ; ++j)
            if (j < nj) out[((size_t)n * nj + j) * F + f] = acc[j];
    }
}

// ---------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------

// What a streaming kernel's plan decided for one input, and all its launch needs.
template <class Params>
struct StreamPlan {
    Params k;                  // kernel parameters
    dim3 grid;
    int threads;
    size_t smem;               // dynamic shared memory per CTA
    int cluster;               // CTAs per cluster along x (1: no cluster)
};

// The streaming 2-D kernel takes the plain head (alpha 1, confidence on the raw maps, no depth, no probability
// export) on dense, 16-byte aligned maps of at least 64 KB per frame whose H splits into chunks and whose W * C/4
// consumer threads fill whole warps of one CTA and number at least C (so W >= 4).  Returns false if it does not
// take the input.
bool plan_sam_stream(const dh_ctx* ctx, const SamParams& p, StreamPlan<SamStreamParams>* pl) {
    if (p.conf_on_prob != 0 || p.alpha != 1.0f || p.d || p.prob) return false;
    if (p.ldh != p.C || (p.C & 3)) return false;
    if ((reinterpret_cast<uintptr_t>(p.h) & 15) != 0) return false;
    if (p.H % ST2_ROWS_PER_CHUNK != 0 || p.H < 2 || p.W < 2) return false;
    const int ncons = p.W * (p.C >> 2);
    if (ncons > 480 || ncons < 64 || (ncons & 31)) return false;
    if (ncons < p.C) return false;    // the combine and output steps give each channel one consumer thread
    const size_t chunk_bytes = (size_t)ST2_ROWS_PER_CHUNK * p.W * p.C * 4;
    if (chunk_bytes % 16 != 0) return false;
    const size_t smem = ST2_STAGES * chunk_bytes + (size_t)(4 * p.W * p.C + 3 * p.C + p.H + 2) * 4 + 2 * ST2_STAGES * 8 + 128;
    if (smem > 227 * 1024) return false;
    if ((size_t)p.H * p.W * p.C * 4 < 64 * 1024) return false;    // small maps: the staged kernel is fine
    SamStreamParams& k = pl->k;
    k.h = p.h; k.N = p.N; k.H = p.H; k.W = p.W; k.C = p.C;
    k.nj = p.nj; k.n_ctx = p.n_ctx; k.alpha_mix = p.alpha_mix;
    k.out_pose = p.out_pose; k.out_conf = p.out_conf;
    k.chunks_per_frame = p.H / ST2_ROWS_PER_CHUNK;
    k.chunk_floats = ST2_ROWS_PER_CHUNK * p.W * p.C;
    pl->grid = dim3(p.N < ctx->num_sms ? p.N : ctx->num_sms);
    pl->threads = ((ncons + 31) / 32) * 32 + 32;
    pl->smem = smem;
    pl->cluster = 1;
    return true;
}

// The streaming 3-D kernel takes dense, 16-byte aligned volumes whose pixels split into ST3_CL quarters of
// ST3_PXC-pixel chunks and whose consumer roles fit one CTA.  Returns false if it does not take the input.
bool plan_sam3d_stream(const Sam3dParams& p, StreamPlan<Sam3dStreamParams>* pl) {
    const int nj = p.nj, C = nj * p.D, P = p.H * p.W;
    if (p.ldh != C || (C & 3) || (reinterpret_cast<uintptr_t>(p.h) & 15)) return false;
    if (P % (ST3_CL * ST3_PXC) != 0 || p.H < 2 || p.W < 2) return false;
    if (ST3_PXC * nj > 480 || C > 480 || ST3_PARTS * nj > 480) return false;
    Sam3dStreamParams& k = pl->k;
    k.h = p.h; k.N = p.N; k.H = p.H; k.W = p.W; k.nj = nj; k.D = p.D; k.vis_scale = p.vis_scale;
    k.out_pose = p.out_pose; k.out_vis = p.out_vis;
    int need = ST3_PXC * nj > C ? ST3_PXC * nj : C;
    if (ST3_PARTS * nj > need) need = ST3_PARTS * nj;
    k.ncons = (need + 31) / 32 * 32;
    const int PL = P / ST3_CL;
    pl->grid = dim3(ST3_CL, p.N);
    pl->threads = k.ncons + 32;
    pl->smem = ((size_t)ST3_STAGES * ST3_PXC * C + (size_t)PL * nj + 2 * C + 4 * nj + ST3_PARTS * 4 * nj + 2) * 4 +
               2 * ST3_STAGES * 8 + 128;
    pl->cluster = ST3_CL;
    return true;
}

template <auto Kernel, class Params>
int launch_stream(dh_ctx* ctx, const StreamPlan<Params>& pl, void* stream, const char* who) {
    cudaError_t e = ensure_smem<Kernel>(pl.smem);
    if (e == cudaSuccess) {
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = pl.grid;
        cfg.blockDim = dim3(pl.threads);
        cfg.dynamicSmemBytes = pl.smem;
        cfg.stream = (cudaStream_t)stream;
        cudaLaunchAttribute at[1];
        if (pl.cluster > 1) {
            at[0].id = cudaLaunchAttributeClusterDimension;
            at[0].val.clusterDim.x = pl.cluster; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
            cfg.attrs = at;
            cfg.numAttrs = 1;
        }
        e = cudaLaunchKernelEx(&cfg, Kernel, pl.k);
    }
    if (e != cudaSuccess) {
        dh_set_error("%s: launch setup failed: %s", who, cudaGetErrorString(e));
        return (int)e;
    }
    DH_LAUNCH_EPILOGUE(ctx, 1);
}

// 2-D heads: the streaming kernel where its plan takes the input, else the staged one
int launch_sam2d(dh_ctx* ctx, const SamParams& p, void* stream, const char* who) {
    StreamPlan<SamStreamParams> pl;
    if (plan_sam_stream(ctx, p, &pl)) return launch_stream<sam_stream_kernel>(ctx, pl, stream, who);
    const int P = p.H * p.W;
    DH_CHECK_ARG(p.C >= 1 && p.C <= 512, "%s: C=%d not in 1..512", who, p.C);
    // the confidence is a max over 2x2 windows (AveragePooling2D((2,2), valid) in the reference raises on smaller maps)
    DH_CHECK_ARG(p.H >= 2 && p.W >= 2, "%s: maps must be at least 2x2 (got %dx%d)", who, p.H, p.W);
    int T = (P * p.C <= 4096) ? 256 : 512;
    if (T < p.C) T = 512;
    size_t smem = (size_t)(((P * p.C + 3) & ~3) + p.W + p.H + 5 * T + 5 * p.C) * sizeof(float);
    DH_CHECK_ARG(smem <= 227 * 1024, "%s: frame of %d x %d x %d floats does not fit shared memory", who, p.H, p.W, p.C);
    cudaError_t e = ensure_smem<softargmax2d_kernel>(smem);
    if (e != cudaSuccess) { dh_set_error("%s: cudaFuncSetAttribute: %s", who, cudaGetErrorString(e)); return (int)e; }
    softargmax2d_kernel<<<p.N, T, smem, (cudaStream_t)stream>>>(p);
    DH_LAUNCH_EPILOGUE(ctx, 1);
}

int launch_sam3d(dh_ctx* ctx, const dh_view* h, int nj, int depth_maps, float vis_scale, float* out_pose,
                 float* out_vis, const dh_view* prob_out, void* stream, const char* who) {
    DH_CHECK_ARG(ctx && h && h->p && out_pose && out_vis, "%s: NULL argument", who);
    DH_CHECK_ARG(nj >= 1 && depth_maps >= 1 && h->c == nj * depth_maps,
                 "%s: C=%d is not depth_maps*nj = %d*%d", who, h->c, depth_maps, nj);
    DH_CHECK_ARG(h->h >= 2 && h->w >= 2, "%s: maps must be at least 2x2 (got %dx%d)", who, h->h, h->w);
    Sam3dParams p;
    p.h = h->p; p.ldh = h->ld; p.N = h->n; p.H = h->h; p.W = h->w; p.nj = nj; p.D = depth_maps;
    p.out_pose = out_pose; p.out_vis = out_vis;
    p.vis_scale = vis_scale;
    p.prob = nullptr; p.ldp = 0;
    // large dense volumes: the cluster-split streaming kernel; the probability export of the merge model and odd
    // shapes stay on the staged kernel
    StreamPlan<Sam3dStreamParams> pl;
    if (!(prob_out && prob_out->p) && ctx->sam3d_stream && plan_sam3d_stream(p, &pl))
        return launch_stream<sam3d_stream_kernel>(ctx, pl, stream, who);
    const int T = 512, C = h->c, P = h->h * h->w;
    DH_CHECK_ARG(C <= 2 * T && nj <= T, "%s: too many channels", who);
    if (prob_out && prob_out->p) {
        DH_CHECK_ARG(prob_out->n == h->n && prob_out->h == h->h && prob_out->w == h->w && prob_out->c == nj,
                     "%s: prob_out must be (N,H,W,nj)", who);
        p.prob = prob_out->p; p.ldp = prob_out->ld;
    }
    size_t smem = (size_t)(((P * nj + 3) & ~3) + SAM3D_PCH * C + ((C + 3) & ~3) + h->w + h->h + 5 * T + 5 * nj) * sizeof(float);
    DH_CHECK_ARG(smem <= 227 * 1024, "%s: marginal maps do not fit shared memory", who);
    cudaError_t e = ensure_smem<softargmax3d_kernel>(smem);
    if (e != cudaSuccess) { dh_set_error("%s: cudaFuncSetAttribute: %s", who, cudaGetErrorString(e)); return (int)e; }
    softargmax3d_kernel<<<p.N, T, smem, (cudaStream_t)stream>>>(p);
    DH_LAUNCH_EPILOGUE(ctx, 1);
}

}  // namespace

extern "C" int dh_softargmax2d_f32(dh_ctx* ctx, const dh_view* h, const dh_view* d, float alpha,
                                   int conf_on_prob, float* out_pose, float* out_conf,
                                   const dh_view* prob_out, void* stream) {
    DH_CHECK_ARG(ctx && h && h->p && out_pose && out_conf, "dh_softargmax2d_f32: NULL argument");
    SamParams p;
    p.h = h->p; p.ldh = h->ld; p.N = h->n; p.H = h->h; p.W = h->w; p.C = h->c;
    p.d = nullptr; p.ldd = 0;
    if (d && d->p) {
        DH_CHECK_ARG(d->n == h->n && d->h == h->h && d->w == h->w && d->c == h->c,
                     "dh_softargmax2d_f32: depth map shape mismatch");
        p.d = d->p; p.ldd = d->ld;
    }
    p.alpha = alpha; p.conf_on_prob = conf_on_prob;
    p.out_pose = out_pose; p.pose_dim = p.d ? 3 : 2; p.out_conf = out_conf;
    p.prob = nullptr; p.ldp = 0;
    if (prob_out && prob_out->p) {
        DH_CHECK_ARG(prob_out->n == h->n && prob_out->h == h->h && prob_out->w == h->w && prob_out->c == h->c,
                     "dh_softargmax2d_f32: prob_out shape mismatch");
        p.prob = prob_out->p; p.ldp = prob_out->ld;
    }
    p.nj = 0; p.n_ctx = 0; p.alpha_mix = 0.f;
    return launch_sam2d(ctx, p, stream, "dh_softargmax2d_f32");
}

extern "C" int dh_softargmax2d_ctx_f32(dh_ctx* ctx, const dh_view* h, int nj, int n_ctx,
                                       float alpha_mix, float* out_pose, float* out_vis, void* stream) {
    DH_CHECK_ARG(ctx && h && h->p && out_pose && out_vis, "dh_softargmax2d_ctx_f32: NULL argument");
    DH_CHECK_ARG(nj >= 1 && n_ctx >= 1 && h->c == nj * (1 + n_ctx),
                 "dh_softargmax2d_ctx_f32: C=%d is not nj*(1+n_ctx) = %d*(1+%d)", h->c, nj, n_ctx);
    SamParams p;
    p.h = h->p; p.ldh = h->ld; p.N = h->n; p.H = h->h; p.W = h->w; p.C = h->c;
    p.d = nullptr; p.ldd = 0; p.alpha = 1.0f; p.conf_on_prob = 0;
    p.out_pose = out_pose; p.pose_dim = 2; p.out_conf = out_vis; p.prob = nullptr; p.ldp = 0;
    p.nj = nj; p.n_ctx = n_ctx; p.alpha_mix = alpha_mix;
    return launch_sam2d(ctx, p, stream, "dh_softargmax2d_ctx_f32");
}

extern "C" int dh_softargmax3d_f32(dh_ctx* ctx, const dh_view* h, int nj, int depth_maps,
                                   float* out_pose, float* out_vis, void* stream) {
    return launch_sam3d(ctx, h, nj, depth_maps, 1.0f, out_pose, out_vis, nullptr, stream, "dh_softargmax3d_f32");
}

extern "C" int dh_softargmax3d_ex_f32(dh_ctx* ctx, const dh_view* h, int nj, int depth_maps, float vis_scale,
                                      float* out_pose, float* out_vis, const dh_view* prob_out, void* stream) {
    return launch_sam3d(ctx, h, nj, depth_maps, vis_scale, out_pose, out_vis, prob_out, stream, "dh_softargmax3d_ex_f32");
}

extern "C" int dh_kron_pool_f32(dh_ctx* ctx, const dh_view* pm, const dh_view* z, float* out, void* stream) {
    DH_CHECK_ARG(ctx && pm && z && pm->p && z->p && out, "dh_kron_pool_f32: NULL argument");
    DH_CHECK_ARG(pm->n == z->n && pm->h == z->h && pm->w == z->w, "dh_kron_pool_f32: P and Z spatial shapes differ");
    DH_CHECK_ARG(pm->c <= KR_MAXJ, "dh_kron_pool_f32: more than %d joints", KR_MAXJ);
    dim3 grid(pm->n, (z->c + 127) / 128);
    kron_kernel<<<grid, 128, 0, (cudaStream_t)stream>>>(pm->p, pm->ld, z->p, z->ld, pm->h * pm->w, pm->c, z->c, out);
    DH_LAUNCH_EPILOGUE(ctx, 1);
}
