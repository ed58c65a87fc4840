// CUDA-core (fp32 FFMA) convolution kernels: the general implicit-GEMM Conv2D used
// for shapes the tensor-core path does not take (Cin = 3 stem conv, the tiny action
// head convs, ragged channel counts), and the stand-alone depthwise stage.
//
// replaces: keras Conv2D / SeparableConv2D lowered by TF-1.6 to cuDNN
// (deephar/layers.py:66-80), with the BatchNormalization / ReLU / add layers
// around them fused in (layers.py:202-325, models/common.py:25-67).
#include "common.cuh"
#include "conv_params.cuh"

// ---------------------------------------------------------------------------
// Implicit GEMM:  out[m, co] = sum_k A[m, k] * W[k, co],  m = (n, oy, ox),
// k = (ky, kx, ci)  -- exactly the HWIO weight layout flattened to [K][Cout].
// Tile 128 x 64 x 16, 256 threads, 8x4 accumulators per thread.
// ---------------------------------------------------------------------------
namespace {

constexpr int BM = 128, BN = 64, BK = 16, NT = 256;
constexpr int A_ROWS_PER_PASS = NT / BK;       // 16
constexpr int A_PASSES = BM / A_ROWS_PER_PASS; // 8

__global__ void __launch_bounds__(NT) conv_simt_kernel(ConvParams p) {
    __shared__ __align__(16) float As[BK][BM + 4];
    __shared__ __align__(16) float Bs[BK][BN];

    const int tid = threadIdx.x;
    const int m0 = blockIdx.x * BM;
    const int n0 = blockIdx.y * BN;
    const int HoWo = p.Ho * p.Wo;

    // A-load assignment: fixed k-lane, 8 pixel rows.
    const int a_kk = tid % BK;
    const int a_r0 = tid / BK;
    int a_base[A_PASSES], a_iy[A_PASSES], a_ix[A_PASSES];
#pragma unroll
    for (int i = 0; i < A_PASSES; ++i) {
        int m = m0 + a_r0 + i * A_ROWS_PER_PASS;
        if (m < p.M) {
            int n = m / HoWo;
            int r = m - n * HoWo;
            int oy = r / p.Wo;
            int ox = r - oy * p.Wo;
            a_base[i] = n * p.H * p.W;
            a_iy[i] = oy * p.sh - p.pt;
            a_ix[i] = ox * p.sw - p.pl;
        } else {
            a_base[i] = 0;
            a_iy[i] = -(1 << 28);
            a_ix[i] = 0;
        }
    }
    // B-load assignment: one float4 per thread.
    const int b_row = tid / (BN / 4);
    const int b_col = (tid % (BN / 4)) * 4;
    const bool b_vec = (p.Cout % 4) == 0;

    const int tx = tid % 16;  // cout group (4 wide)
    const int ty = tid / 16;  // pixel group (8 tall)
    float acc[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

    for (int k0 = 0; k0 < p.K; k0 += BK) {
        // ---- A tile (gather + fused pre-ops) ----
        {
            int k = k0 + a_kk;
            bool kval = k < p.K;
            int tap = kval ? k / p.Cin : 0;
            int ci = k - tap * p.Cin;
            int ky = tap / p.kw;
            int kx = tap - ky * p.kw;
            float ps = 1.f, pb = 0.f;
            if (kval && p.pre_scale) {
                ps = __ldg(p.pre_scale + ci);
                pb = __ldg(p.pre_shift + ci);
            }
#pragma unroll
            for (int i = 0; i < A_PASSES; ++i) {
                int iy = a_iy[i] + ky, ix = a_ix[i] + kx;
                float v = 0.f;
                if (kval && iy >= 0 && iy < p.H && ix >= 0 && ix < p.W) {
                    v = __ldg(p.x + (size_t)(a_base[i] + iy * p.W + ix) * p.ldx + ci);
                    v = fmaf(v, ps, pb);
                    if (p.pre_relu) v = fmaxf(v, 0.f);
                }
                As[a_kk][a_r0 + i * A_ROWS_PER_PASS] = v;
            }
        }
        // ---- B tile ----
        {
            int k = k0 + b_row;
            int co = n0 + b_col;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (k < p.K) {
                const float* wp = p.w + (size_t)k * p.Cout + co;
                if (b_vec && co + 3 < p.Cout) {
                    v = __ldg(reinterpret_cast<const float4*>(wp));
                } else {
                    if (co + 0 < p.Cout) v.x = __ldg(wp + 0);
                    if (co + 1 < p.Cout) v.y = __ldg(wp + 1);
                    if (co + 2 < p.Cout) v.z = __ldg(wp + 2);
                    if (co + 3 < p.Cout) v.w = __ldg(wp + 3);
                }
            }
            *reinterpret_cast<float4*>(&Bs[b_row][b_col]) = v;
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < BK; ++kk) {
            float4 a0 = *reinterpret_cast<const float4*>(&As[kk][ty * 8]);
            float4 a1 = *reinterpret_cast<const float4*>(&As[kk][ty * 8 + 4]);
            float4 b = *reinterpret_cast<const float4*>(&Bs[kk][tx * 4]);
            float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
            float bb[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], bb[j], acc[i][j]);
        }
        __syncthreads();
    }

    // ---- epilogue: BN affine, ReLU, residual adds, store ----
    const int co0 = n0 + tx * 4;
    float sc[4], sf[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        int co = co0 + j;
        sc[j] = (p.post_scale && co < p.Cout) ? __ldg(p.post_scale + co) : 1.f;
        sf[j] = (p.post_shift && co < p.Cout) ? __ldg(p.post_shift + co) : 0.f;
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        int m = m0 + ty * 8 + i;
        if (m >= p.M) continue;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            int co = co0 + j;
            if (co >= p.Cout) continue;
            float v = fmaf(acc[i][j], sc[j], sf[j]);
            if (p.post_relu) v = fmaxf(v, 0.f);
            if (p.res0) v += __ldg(p.res0 + (size_t)m * p.ldr0 + co);
            if (p.res1) v += __ldg(p.res1 + (size_t)m * p.ldr1 + co);
            p.out[(size_t)m * p.ldo + co] = v;
        }
    }
}

// ---------------------------------------------------------------------------
// Stand-alone depthwise stage (only used when the fused tensor-core separable
// kernel does not apply).  One thread per (output pixel, channel).
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256) depthwise_simt_kernel(ConvParams p, float* __restrict__ tmp) {
    const int64_t total = (int64_t)p.M * p.Cin;
    for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total;
         idx += (int64_t)gridDim.x * blockDim.x) {
        int c = (int)(idx % p.Cin);
        int m = (int)(idx / p.Cin);
        int n = m / (p.Ho * p.Wo);
        int r = m - n * p.Ho * p.Wo;
        int oy = r / p.Wo, ox = r - oy * p.Wo;
        float ps = 1.f, pb = 0.f;
        if (p.pre_scale) {
            ps = __ldg(p.pre_scale + c);
            pb = __ldg(p.pre_shift + c);
        }
        float acc = 0.f;
        for (int ky = 0; ky < p.kh; ++ky) {
            int iy = oy * p.sh - p.pt + ky;
            if (iy < 0 || iy >= p.H) continue;
            for (int kx = 0; kx < p.kw; ++kx) {
                int ix = ox * p.sw - p.pl + kx;
                if (ix < 0 || ix >= p.W) continue;
                float v = __ldg(p.x + ((size_t)(n * p.H + iy) * p.W + ix) * p.ldx + c);
                v = fmaf(v, ps, pb);
                if (p.pre_relu) v = fmaxf(v, 0.f);
                acc = fmaf(v, __ldg(p.w_dw + (ky * p.kw + kx) * p.Cin + c), acc);
            }
        }
        tmp[idx] = acc;
    }
}

}  // namespace

int dh_fill_conv_params(ConvParams* p, const dh_view* x, const dh_conv_desc* d, const dh_view* out,
                        int cout, const char* who) {
    DH_CHECK_ARG(x && d && out && x->p && out->p, "%s: NULL argument", who);
    DH_CHECK_ARG(d->kh >= 1 && d->kw >= 1 && d->sh >= 1 && d->sw >= 1, "%s: bad kernel/stride", who);
    DH_CHECK_ARG(d->n_res >= 0 && d->n_res <= 2, "%s: n_res must be 0..2", who);
    DH_CHECK_ARG((d->pre_scale == nullptr) == (d->pre_shift == nullptr), "%s: pre_scale/pre_shift must come together", who);
    int pt, pl;
    int ho = dh_out_size(x->h, d->kh, d->sh, d->pad_same, &pt);
    int wo = dh_out_size(x->w, d->kw, d->sw, d->pad_same, &pl);
    DH_CHECK_ARG(ho >= 1 && wo >= 1, "%s: empty output (%dx%d input, %dx%d kernel)", who, x->h, x->w, d->kh, d->kw);
    DH_CHECK_ARG(out->n == x->n && out->h == ho && out->w == wo && out->c == cout,
                 "%s: output view is (%d,%d,%d,%d), expected (%d,%d,%d,%d)", who, out->n, out->h, out->w,
                 out->c, x->n, ho, wo, cout);
    DH_CHECK_ARG(x->ld >= x->c && out->ld >= out->c, "%s: ld smaller than c", who);
    DH_CHECK_ARG((d->res_up2x & ~3) == 0 && (d->res_up2x == 0 || d->res_up2x == (1 << (d->n_res - 1))),
                 "%s: res_up2x may only flag the LAST residual", who);
    for (int i = 0; i < d->n_res; ++i) {
        const int up = (d->res_up2x >> i) & 1;
        DH_CHECK_ARG(d->res[i].p && d->res[i].n == out->n && d->res[i].h * (up ? 2 : 1) == ho &&
                         d->res[i].w * (up ? 2 : 1) == wo && d->res[i].c == cout,
                     "%s: residual %d shape mismatch", who, i);
    }
    p->x = x->p; p->N = x->n; p->H = x->h; p->W = x->w; p->Cin = x->c; p->ldx = x->ld;
    p->w = nullptr; p->w_dw = nullptr;
    p->out = out->p; p->Ho = ho; p->Wo = wo; p->Cout = cout; p->ldo = out->ld;
    p->kh = d->kh; p->kw = d->kw; p->sh = d->sh; p->sw = d->sw; p->pt = pt; p->pl = pl;
    p->pre_scale = d->pre_scale; p->pre_shift = d->pre_shift;
    p->post_scale = d->post_scale; p->post_shift = d->post_shift;
    p->pre_relu = d->pre_relu; p->post_relu = d->post_relu;
    p->res0 = d->n_res > 0 ? d->res[0].p : nullptr; p->ldr0 = d->n_res > 0 ? d->res[0].ld : 0;
    p->res1 = d->n_res > 1 ? d->res[1].p : nullptr; p->ldr1 = d->n_res > 1 ? d->res[1].ld : 0;
    p->up1 = 0;
    if (d->res_up2x) {                  // the upsampled residual always travels in slot 1
        if (d->n_res == 1) { p->res1 = p->res0; p->ldr1 = p->ldr0; p->res0 = nullptr; p->ldr0 = 0; }
        p->up1 = 1;
        DH_CHECK_ARG(((wo % 32) == 0 || wo == 16) && (ho % 2) == 0, "%s: an upsampled residual needs Wo == 16 or Wo %% 32 == 0 (got %dx%d)", who, ho, wo);
    }
    p->pool = nullptr; p->ldp = 0;
    if (d->pool_out.p) {
        const dh_view& q = d->pool_out;
        DH_CHECK_ARG((ho % 2) == 0 && (wo % 2) == 0 && q.n == out->n && q.h == ho / 2 && q.w == wo / 2 && q.c == cout && q.ld >= q.c,
                     "%s: pool_out must be (%d,%d,%d,%d)", who, out->n, ho / 2, wo / 2, cout);
        p->pool = q.p; p->ldp = q.ld;
    }
    int64_t m = (int64_t)x->n * ho * wo;
    DH_CHECK_ARG(m < (1ll << 31) && (int64_t)x->n * x->h * x->w < (1ll << 31), "%s: too many pixels for int32 indexing", who);
    p->M = (int)m;
    p->K = d->kh * d->kw * x->c;
    return 0;
}

// ---------------------------------------------------------------------------------------------
// Direct convolution for a tiny reduction (the 3x3x3 first conv of the stem, K = 27,
// models/reception.py:61-66).  An implicit-GEMM tile would waste half its K and N; here 4 threads
// share one output pixel (8 output channels each): the K inputs of the pixel sit in registers, the
// [K][Cout] weights and the BN affine in shared memory (broadcast float4 reads), and the 4 threads of
// a pixel write 128 contiguous bytes -> a warp stores 1 KB rows.  No prologue, no residuals.
// ---------------------------------------------------------------------------------------------
constexpr int SK_MAX = 32;        // max K
constexpr int SK_NT = 256;        // threads per block = 64 pixels x 4 channel groups (Cout = 32) ...

template <int CG, int KH, int KW, int CIN>   // CG = Cout / 8 channel groups per pixel (4 | 8); compile-time taps
__global__ void __launch_bounds__(SK_NT) conv_smallk_kernel(const ConvParams p) {
    __shared__ __align__(16) float w_s[SK_MAX * 8 * CG];
    __shared__ __align__(16) float sc_s[8 * CG], sh_s[8 * CG];
    const int K = p.K, Cout = 8 * CG;
    for (int i = threadIdx.x; i < K * Cout; i += SK_NT) w_s[i] = __ldg(p.w + i);
    for (int i = threadIdx.x; i < Cout; i += SK_NT) {
        sc_s[i] = p.post_scale ? __ldg(p.post_scale + i) : 1.f;
        sh_s[i] = p.post_shift ? __ldg(p.post_shift + i) : 0.f;
    }
    __syncthreads();
    const int cg = threadIdx.x % CG;
    constexpr int PPB = SK_NT / CG;                       // pixels per block iteration
    for (int m = blockIdx.x * PPB + threadIdx.x / CG; m < p.M; m += gridDim.x * PPB) {
        const int ox = m % p.Wo, t = m / p.Wo, oy = t % p.Ho, n = t / p.Ho;
        const int iy0 = oy * p.sh - p.pt, ix0 = ox * p.sw - p.pl;
        const float* xb = p.x + (size_t)n * p.H * p.W * p.ldx;
        float in[KH * KW * CIN];
#pragma unroll
        for (int ky = 0; ky < KH; ++ky) {
            const int iy = iy0 + ky;
#pragma unroll
            for (int kx = 0; kx < KW; ++kx) {
                const int ix = ix0 + kx;
                const bool ok = iy >= 0 && iy < p.H && ix >= 0 && ix < p.W;
                const float* px = xb + ((size_t)iy * p.W + ix) * p.ldx;
#pragma unroll
                for (int ci = 0; ci < CIN; ++ci) in[(ky * KW + kx) * CIN + ci] = ok ? __ldg(px + ci) : 0.f;
            }
        }
        float acc[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] = 0.f;
#pragma unroll
        for (int kk = 0; kk < KH * KW * CIN; ++kk) {
            {
                const float4 w0 = *reinterpret_cast<const float4*>(w_s + kk * Cout + cg * 8);
                const float4 w1 = *reinterpret_cast<const float4*>(w_s + kk * Cout + cg * 8 + 4);
                acc[0] = fmaf(in[kk], w0.x, acc[0]); acc[1] = fmaf(in[kk], w0.y, acc[1]);
                acc[2] = fmaf(in[kk], w0.z, acc[2]); acc[3] = fmaf(in[kk], w0.w, acc[3]);
                acc[4] = fmaf(in[kk], w1.x, acc[4]); acc[5] = fmaf(in[kk], w1.y, acc[5]);
                acc[6] = fmaf(in[kk], w1.z, acc[6]); acc[7] = fmaf(in[kk], w1.w, acc[7]);
            }
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            acc[j] = fmaf(acc[j], sc_s[cg * 8 + j], sh_s[cg * 8 + j]);
            if (p.post_relu) acc[j] = fmaxf(acc[j], 0.f);
        }
        float* op = p.out + (size_t)m * p.ldo + cg * 8;
        *reinterpret_cast<float4*>(op) = make_float4(acc[0], acc[1], acc[2], acc[3]);
        *reinterpret_cast<float4*>(op + 4) = make_float4(acc[4], acc[5], acc[6], acc[7]);
    }
}

static bool smallk_ok(const ConvParams& p) {
    return p.kh == 3 && p.kw == 3 && p.Cin == 3 && p.K == 27 && (p.Cout == 32 || p.Cout == 64) && !p.pre_scale && !p.pre_relu && !p.res0 && !p.res1 &&
           (p.ldo & 3) == 0 && (reinterpret_cast<uintptr_t>(p.out) & 15) == 0;
}

// ---------------------------------------------------------------------------------------------
// Pointwise (1x1, stride 1) convolution with a SMALL reduction (Cin <= 64) and a wide output: the
// fReMap layers (48 -> 576 heat-map re-injection, models/reception.py:156-164 + the block-end add of
// :194-196).  Such a layer is all epilogue -- 48 MACs per output but three 302 MB streams (two
// residuals in, one out per 128 frames) -- so it runs on CUDA cores in exact fp32 with every thread
// taking part in the memory traffic: per 64-pixel tile the [Cin][Cout] weights, the BN vectors and the
// (prologue-applied) input tile sit in shared memory; warp = PW_PX pixels, lane = 4 consecutive output
// channels (x ceil(Cout/128) passes); the residual float4 loads of a pass are issued BEFORE its
// k-loop (64 KB in flight per SM), packed FFMA2 accumulate, 512-byte coalesced rows out.
// ---------------------------------------------------------------------------------------------
// POOL: the tile is two image rows of 32 pixels and a warp takes a 2x2 pixel block of them (instead of 4 pixels of
// one row), so the MaxPooling2D((2,2)) of the result is a max over the thread's own four pixels: second output.
template <int PW_PX, int PW_NT, bool PRE1, bool POOL>   // pixels per warp, threads per CTA, prefetch the 2nd residual before the k-loop
__global__ void __launch_bounds__(PW_NT, 1) conv_pw_smallk_kernel(const ConvParams p) {
    constexpr int PW_TILE = (PW_NT / 32) * PW_PX;
    static_assert(!POOL || (PW_PX == 4 && PW_TILE == 64), "POOL: 16 warps x (2x2 pixels) = two rows of 32");
    extern __shared__ __align__(16) float pw_smem[];
    const int K = p.Cin, Cout = p.Cout, CQ = Cout >> 2, K4 = K >> 2;
    float* w_s = pw_smem;                       // [K][Cout]
    float* sc_s = w_s + K * Cout;               // [Cout]
    float* sh_s = sc_s + Cout;                  // [Cout]
    float* ps_s = sh_s + Cout;                  // [K] prologue scale
    float* pb_s = ps_s + K;                     // [K] prologue shift
    float* h_s = pb_s + K;                      // [PW_TILE][K]
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    for (int i = tid; i < K * CQ; i += PW_NT)
        reinterpret_cast<float4*>(w_s)[i] = __ldg(reinterpret_cast<const float4*>(p.w) + i);
    for (int i = tid; i < Cout; i += PW_NT) {
        sc_s[i] = p.post_scale ? __ldg(p.post_scale + i) : 1.f;
        sh_s[i] = p.post_shift ? __ldg(p.post_shift + i) : 0.f;
    }
    for (int i = tid; i < K; i += PW_NT) {
        ps_s[i] = p.pre_scale ? __ldg(p.pre_scale + i) : 1.f;
        pb_s[i] = p.pre_shift ? __ldg(p.pre_shift + i) : 0.f;
    }
    const float lowb = p.pre_relu ? 0.f : -3.402823466e38f;
    const int ntiles = (p.M + PW_TILE - 1) / PW_TILE;
    for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const int m0 = tile * PW_TILE;
        __syncthreads();                         // previous tile's readers are done (and the tables are written)
        for (int i = tid; i < PW_TILE * K4; i += PW_NT) {
            const int row = i / K4, c4 = i - row * K4;
            const int m = m0 + row;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (m < p.M) {
                v = __ldg(reinterpret_cast<const float4*>(p.x + (size_t)m * p.ldx + c4 * 4));
                const float4 a = *reinterpret_cast<const float4*>(ps_s + c4 * 4);
                const float4 b = *reinterpret_cast<const float4*>(pb_s + c4 * 4);
                v.x = fmaxf(fmaf(v.x, a.x, b.x), lowb); v.y = fmaxf(fmaf(v.y, a.y, b.y), lowb);
                v.z = fmaxf(fmaf(v.z, a.z, b.z), lowb); v.w = fmaxf(fmaf(v.w, a.w, b.w), lowb);
            }
            reinterpret_cast<float4*>(h_s)[i] = v;
        }
        __syncthreads();
        // local index of this warp's pixel q inside the tile
        auto lidx = [&](int q) { return POOL ? ((q >> 1) * 32 + warp * 2 + (q & 1)) : (warp * PW_PX + q); };
        for (int cq = lane; cq < CQ; cq += 32) {
            const int co = cq * 4;
            float4 r0[PW_PX], r1[PW_PX];
#pragma unroll
            for (int q = 0; q < PW_PX; ++q) {
                r0[q] = make_float4(0.f, 0.f, 0.f, 0.f);
                r1[q] = make_float4(0.f, 0.f, 0.f, 0.f);
                const int m = m0 + lidx(q);
                if (m < p.M) {
                    if (p.res0) r0[q] = __ldg(reinterpret_cast<const float4*>(p.res0 + (size_t)m * p.ldr0 + co));
                    if (PRE1 && p.res1) r1[q] = __ldg(reinterpret_cast<const float4*>(p.res1 + (size_t)m * p.ldr1 + co));
                }
            }
            float2 a01[PW_PX], a23[PW_PX];
#pragma unroll
            for (int q = 0; q < PW_PX; ++q) { a01[q] = make_float2(0.f, 0.f); a23[q] = make_float2(0.f, 0.f); }
            for (int k = 0; k < K; k += 4) {
                const float4 w0 = *reinterpret_cast<const float4*>(w_s + (k + 0) * Cout + co);
                const float4 w1 = *reinterpret_cast<const float4*>(w_s + (k + 1) * Cout + co);
                const float4 w2 = *reinterpret_cast<const float4*>(w_s + (k + 2) * Cout + co);
                const float4 w3 = *reinterpret_cast<const float4*>(w_s + (k + 3) * Cout + co);
#pragma unroll
                for (int q = 0; q < PW_PX; ++q) {
                    const float4 h = *reinterpret_cast<const float4*>(h_s + lidx(q) * K + k);     // broadcast
                    a01[q] = ffma2(make_float2(h.x, h.x), make_float2(w0.x, w0.y), a01[q]);
                    a23[q] = ffma2(make_float2(h.x, h.x), make_float2(w0.z, w0.w), a23[q]);
                    a01[q] = ffma2(make_float2(h.y, h.y), make_float2(w1.x, w1.y), a01[q]);
                    a23[q] = ffma2(make_float2(h.y, h.y), make_float2(w1.z, w1.w), a23[q]);
                    a01[q] = ffma2(make_float2(h.z, h.z), make_float2(w2.x, w2.y), a01[q]);
                    a23[q] = ffma2(make_float2(h.z, h.z), make_float2(w2.z, w2.w), a23[q]);
                    a01[q] = ffma2(make_float2(h.w, h.w), make_float2(w3.x, w3.y), a01[q]);
                    a23[q] = ffma2(make_float2(h.w, h.w), make_float2(w3.z, w3.w), a23[q]);
                }
            }
            const float4 sc = *reinterpret_cast<const float4*>(sc_s + co);
            const float4 sh = *reinterpret_cast<const float4*>(sh_s + co);
            if (!PRE1 && p.res1) {
#pragma unroll
                for (int q = 0; q < PW_PX; ++q)
                    if (m0 + lidx(q) < p.M) r1[q] = __ldg(reinterpret_cast<const float4*>(p.res1 + (size_t)(m0 + lidx(q)) * p.ldr1 + co));
            }
            float4 pm = make_float4(-3.402823466e38f, -3.402823466e38f, -3.402823466e38f, -3.402823466e38f);
#pragma unroll
            for (int q = 0; q < PW_PX; ++q) {
                if (m0 + lidx(q) < p.M) {
                    float4 t;
                    t.x = fmaf(a01[q].x, sc.x, sh.x); t.y = fmaf(a01[q].y, sc.y, sh.y);
                    t.z = fmaf(a23[q].x, sc.z, sh.z); t.w = fmaf(a23[q].y, sc.w, sh.w);
                    if (p.post_relu) {
                        t.x = fmaxf(t.x, 0.f); t.y = fmaxf(t.y, 0.f); t.z = fmaxf(t.z, 0.f); t.w = fmaxf(t.w, 0.f);
                    }
                    t.x += r0[q].x + r1[q].x; t.y += r0[q].y + r1[q].y;
                    t.z += r0[q].z + r1[q].z; t.w += r0[q].w + r1[q].w;
                    *reinterpret_cast<float4*>(p.out + (size_t)(m0 + lidx(q)) * p.ldo + co) = t;
                    if (POOL) { pm.x = fmaxf(pm.x, t.x); pm.y = fmaxf(pm.y, t.y); pm.z = fmaxf(pm.z, t.z); pm.w = fmaxf(pm.w, t.w); }
                }
            }
            // tile = row pair `tile` of the batch (M % 64 == 0): pooled pixel tile * 16 + warp
            if (POOL) *reinterpret_cast<float4*>(p.pool + ((size_t)tile * 16 + warp) * p.ldp + co) = pm;
        }
    }
}

static size_t pw_smallk_smem(const ConvParams& p, int tile) {
    return sizeof(float) * ((size_t)p.Cin * p.Cout + 2 * (size_t)p.Cout + 2 * (size_t)p.Cin + (size_t)tile * p.Cin);
}

bool dh_pw_smallk_supported(const ConvParams& p) {
    auto a16 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
    if (!(p.kh == 1 && p.kw == 1 && p.sh == 1 && p.sw == 1)) return false;
    if (p.Cin > 64 || (p.Cin & 3) || (p.Cout & 3) || p.Cout < 128) return false;       // wide outputs only
    if ((p.ldx & 3) || (p.ldo & 3) || !a16(p.x) || !a16(p.out) || !a16(p.w)) return false;
    if (p.res0 && ((p.ldr0 & 3) || !a16(p.res0))) return false;
    if (p.res1 && ((p.ldr1 & 3) || !a16(p.res1))) return false;
    if (p.pool && !(p.Wo == 32 && (p.Ho & 1) == 0 && (p.ldp & 3) == 0 && a16(p.pool))) return false;
    return pw_smallk_smem(p, 64) <= 200 * 1024;
}

template <int PX, int NT, bool PRE1, bool POOL>
static int pw_launch(const ConvParams& p, int num_sms, cudaStream_t s) {
    constexpr int tile = (NT / 32) * PX;
    const size_t smem = pw_smallk_smem(p, tile);
    cudaError_t e = cudaFuncSetAttribute(conv_pw_smallk_kernel<PX, NT, PRE1, POOL>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) {
        dh_set_error("dh_launch_pw_smallk: %s", cudaGetErrorString(e));
        return (int)e;
    }
    int blocks = (p.M + tile - 1) / tile;
    if (blocks > num_sms) blocks = num_sms;
    conv_pw_smallk_kernel<PX, NT, PRE1, POOL><<<blocks, NT, smem, s>>>(p);
    return 0;
}

// Measured on the fReMap shape (128 frames, 48 -> 576, two residuals): 4 px x 512 threads 280 us,
// 8 px x 256 threads 298 us, 8 px x 384 threads 300 us, 4 px x 768 threads 295 us -- the kernel is bound by the
// fp32 FMA pipe (7.2 GFLOP at ~26 TFLOP/s), not by occupancy.
int dh_launch_pw_smallk(const ConvParams& p, int num_sms, cudaStream_t s) {
    if (p.pool) return pw_launch<4, 512, true, true>(p, num_sms, s);
    return pw_launch<4, 512, true, false>(p, num_sms, s);
}

// true if dh_launch_conv_simt serves `p` with the direct small-K kernel (not the generic implicit-GEMM fallback)
bool dh_conv_smallk_ok(const ConvParams& p) { return smallk_ok(p); }

void dh_launch_conv_simt(const ConvParams& p, cudaStream_t s) {
    if (smallk_ok(p)) {
        const int cgn = p.Cout / 8;
        const int ppb = SK_NT / cgn;
        int blocks = (p.M + ppb - 1) / ppb;
        if (blocks > 132 * 16) blocks = 132 * 16;     // 16 blocks per SM of an H100
        if (cgn == 4) conv_smallk_kernel<4, 3, 3, 3><<<blocks, SK_NT, 0, s>>>(p);
        else conv_smallk_kernel<8, 3, 3, 3><<<blocks, SK_NT, 0, s>>>(p);
        return;
    }
    dim3 grid((p.M + BM - 1) / BM, (p.Cout + BN - 1) / BN);
    conv_simt_kernel<<<grid, NT, 0, s>>>(p);
}

void dh_launch_depthwise_simt(const ConvParams& p, float* tmp, int num_sms, cudaStream_t s) {
    int64_t total = (int64_t)p.M * p.Cin;
    int64_t blocks = (total + 255) / 256;
    int64_t cap = (int64_t)num_sms * 16;
    if (blocks > cap) blocks = cap;
    depthwise_simt_kernel<<<(int)blocks, 256, 0, s>>>(p, tmp);
}
