// wgmma tensor-core convolutions for sm_90a: Conv2D (1x1 and dense kxk) and the fused
// SeparableConv2D (depthwise kxk + pointwise 1x1 in ONE kernel; the depthwise result never
// leaves the SM), with BatchNorm / ReLU prologue, BatchNorm / ReLU / residual-add epilogue.
//
// replaces: keras SeparableConv2D / Conv2D lowered by TF-1.6 to cuDNN (deephar/layers.py:66-80)
// and the BN / Activation / add layers around them (layers.py:202-325, models/common.py:25-67,
// models/reception.py:43-59).
//
// Shape of the computation (per CTA):  D[128 px, BN couts] = A[128 px, K] * W[K, BN]
//   A  : produced by 8 CUDA-core warps straight into the 128B-swizzled K-major wgmma layout in
//        shared memory.  dense / 1x1: im2col gather (+prologue).  separable: the depthwise kxk
//        (register-tiled: each thread owns 2 channels x 4x4 output pixels, 25 taps in registers).
//   W  : weights, pre-packed on the host as bf16 [Cout_pad][K_pad] K-major, loaded by TMA
//        (cp.async.bulk.tensor, 128B swizzle) into the same wgmma layout.
//   D  : fp32 accumulators in the registers of the consumer warpgroup (wgmma.mma_async m64nNk16, bf16).
//   precision = 3: both operands are split x = hi + lo (bf16 each) and three MMAs
//        (hi*hi + lo*hi + hi*lo) accumulate in fp32 -> ~2^-16 relative operand error, which keeps
//        the <=1e-3 parity bar through 8 stacked blocks; precision = 1 issues hi*hi only.
//   epilogue: accumulator registers -> BN affine, ReLU, residual adds -> global stores.
//
// Pipeline: `stages` x {A_hi, A_lo, W_hi, W_lo} ring; mbarriers full[s] (256 producer arrivals
// + TMA transaction bytes) / empty[s] (consumer warpgroup, after its wgmmas completed).
#include "tc_common.cuh"

namespace tc {
using R = tc::Roles<1>;
constexpr int WARP_EPI0 = R::WARP_EPI0, WARP_TMA = R::WARP_TMA, NTHREADS = R::NTHREADS,
              REGS_PROD = R::REGS_PROD, REGS_EPI = R::REGS_EPI, REGS_CTRL = R::REGS_CTRL;

// ---------------------------------------------------------------------------
// A-tile producers
// ---------------------------------------------------------------------------
// dense / 1x1: item = (pixel row, 4 consecutive k); 16 items per row, 8 rows per thread.
// The per-row pixel coordinates do not depend on the K-block: they are decoded once per CTA
// (DenseRows) so the K loop is 8 independent 16-byte loads issued back to back.
struct DenseRows {
    int base[8];   // (n*H)*W  -- pixel index of the frame origin, -1 = row outside M
    int yx[8];     // (oy*sh - pt) << 16 | ((ox*sw - pl) & 0xffff)
};

__device__ __forceinline__ void dense_rows_init(const ConvParams& c, int m0, int tid, DenseRows& R) {
    const int HoWo = c.Ho * c.Wo;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int m = m0 + (tid >> 4) + i * 16;
        if (m < c.M) {
            int n = m / HoWo;
            int rem = m - n * HoWo;
            int oy = rem / c.Wo;
            int ox = rem - oy * c.Wo;
            R.base[i] = n * c.H * c.W;
            R.yx[i] = ((oy * c.sh - c.pt) << 16) | ((ox * c.sw - c.pl) & 0xffff);
        } else {
            R.base[i] = -1;
            R.yx[i] = 0;
        }
    }
}

// Loads of K-block kb (8 x 16 B per thread) -- issued one K-block AHEAD of the shared-memory
// stage they will be written to, so the global/L2 latency overlaps the previous block's work.
struct DenseRegs {
    float4 v[8];
    unsigned ok;       // bit 4 i + e: component e of row i is inside the image (and k < K)
    float4 ps, pb;
};

__device__ __forceinline__ void dense_load(const TcParams& P, const DenseRows& R, int kb, int tid, DenseRegs& D) {
    const ConvParams& c = P.c;
    const int j = tid & 15;
    const int k = kb * BK + j * 4;          // k = tap*Cin + ci, groups of 4 never straddle a tap (Cin % 4 == 0)
    const bool kval = k < c.K;
    int ci = 0, ky = 0, kx = 0;
    if (kval) {
        int tap = k / c.Cin;
        ci = k - tap * c.Cin;
        ky = tap / c.kw;
        kx = tap - ky * c.kw;
    }
    D.ps = make_float4(1.f, 1.f, 1.f, 1.f);
    D.pb = make_float4(0.f, 0.f, 0.f, 0.f);
    if (kval && c.pre_scale) {
        D.ps = __ldg(reinterpret_cast<const float4*>(c.pre_scale + ci));
        D.pb = __ldg(reinterpret_cast<const float4*>(c.pre_shift + ci));
    }
    D.ok = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int iy = (R.yx[i] >> 16) + ky, ix = (int)(short)(R.yx[i] & 0xffff) + kx;
        const bool ok = kval && R.base[i] >= 0 && iy >= 0 && iy < c.H && ix >= 0 && ix < c.W;
        D.v[i] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (ok) {
            D.ok |= 0xfu << (4 * i);
            D.v[i] = __ldg(reinterpret_cast<const float4*>(c.x + (size_t)(R.base[i] + iy * c.W + ix) * c.ldx + ci));
        }
    }
}

// Same item, for layers the 16-byte gather cannot take: Cin not a multiple of 4 (SPNet's 7x7x3 first conv,
// models/spnet.py:317-325; the heat-map re-injection convs on nj / 2 nj channels, spnet.py:236-247), or a
// channel-sliced input view at an unaligned offset.  The 4 k's of an item then belong to different taps /
// pixels: each is decoded and loaded on its own (L1 serves the overlap between neighbouring pixels).
__device__ __forceinline__ void dense_load_scalar(const TcParams& P, const DenseRows& R, int kb, int tid, DenseRegs& D) {
    const ConvParams& c = P.c;
    const int k0 = kb * BK + (tid & 15) * 4;
    // per k: tap offsets (ky, kx) and the element offset of (ky, kx, ci) relative to the row's window origin
    int ky[4], kx[4], off[4];
    bool kv[4];
    float ps[4] = {1.f, 1.f, 1.f, 1.f}, pb[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int e = 0; e < 4; ++e) {
        const int k = k0 + e;
        kv[e] = k < c.K;
        const int tap = kv[e] ? k / c.Cin : 0;
        const int ci = kv[e] ? k - tap * c.Cin : 0;
        ky[e] = tap / c.kw;
        kx[e] = tap - ky[e] * c.kw;
        off[e] = (ky[e] * c.W + kx[e]) * c.ldx + ci;
        if (kv[e] && c.pre_scale) {
            ps[e] = __ldg(c.pre_scale + ci);
            pb[e] = __ldg(c.pre_shift + ci);
        }
    }
    D.ps = make_float4(ps[0], ps[1], ps[2], ps[3]);
    D.pb = make_float4(pb[0], pb[1], pb[2], pb[3]);
    D.ok = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        // window origin of this output pixel (may lie outside the image: only dereferenced where valid)
        const int iy0 = R.yx[i] >> 16, ix0 = (int)(short)(R.yx[i] & 0xffff);
        const bool rok = R.base[i] >= 0;
        const float* p0 = c.x + ((long long)R.base[i] + (long long)iy0 * c.W + ix0) * (long long)c.ldx;
        float v[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const bool ok = rok && kv[e] && (unsigned)(iy0 + ky[e]) < (unsigned)c.H && (unsigned)(ix0 + kx[e]) < (unsigned)c.W;
            v[e] = 0.f;
            if (ok) {
                D.ok |= 1u << (4 * i + e);
                v[e] = __ldg(p0 + off[e]);
            }
        }
        D.v[i] = make_float4(v[0], v[1], v[2], v[3]);
    }
}

__device__ __forceinline__ void dense_load_any(const TcParams& P, const DenseRows& R, int kb, int tid, DenseRegs& D);

__device__ __forceinline__ void dense_store(const TcParams& P, const DenseRegs& D, uint8_t* a_hi, uint8_t* a_lo,
                                            int tid, bool want_lo) {
    const ConvParams& c = P.c;
    const int j = tid & 15;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        float4 t = D.v[i];
        const unsigned m = (D.ok >> (4 * i)) & 0xfu;       // padding / K tail stay zero AFTER the prologue
        if (m) {
            t.x = fmaf(t.x, D.ps.x, D.pb.x); t.y = fmaf(t.y, D.ps.y, D.pb.y);
            t.z = fmaf(t.z, D.ps.z, D.pb.z); t.w = fmaf(t.w, D.ps.w, D.pb.w);
            if (c.pre_relu) {
                t.x = fmaxf(t.x, 0.f); t.y = fmaxf(t.y, 0.f); t.z = fmaxf(t.z, 0.f); t.w = fmaxf(t.w, 0.f);
            }
            if (m != 0xfu) {
                if (!(m & 1u)) t.x = 0.f;
                if (!(m & 2u)) t.y = 0.f;
                if (!(m & 4u)) t.z = 0.f;
                if (!(m & 8u)) t.w = 0.f;
            }
        }
        uint32_t h0, l0, h1, l1;
        split2(t.x, t.y, h0, l0);
        split2(t.z, t.w, h1, l1);
        const uint32_t off = swz((tid >> 4) + i * 16, j * 4);
        *reinterpret_cast<uint2*>(a_hi + off) = make_uint2(h0, h1);
        if (want_lo) *reinterpret_cast<uint2*>(a_lo + off) = make_uint2(l0, l1);
    }
}

// separable: thread = (2 channels, 4 columns, 4-row strip).  32 channel pairs x (128/16) pixel
// blocks = 256 threads per 64-channel K-block; the KSxKS taps of the thread's 2 channels live in
// registers; input rows slide through a 3-row rotating register buffer that is loaded two rows
// ahead of the FMAs (16-24 loads in flight per thread; every input value is loaded once per
// thread).  Stride 1, TF SAME padding (symmetric for odd KS).
template <int KS>
__device__ __forceinline__ void produce_sep(const TcParams& P, int kb, uint8_t* a_hi, uint8_t* a_lo, int m0,
                                            int tid, bool want_lo) {
    const ConvParams& c = P.c;
    constexpr int PAD = KS / 2;
    constexpr int NR = 4 + KS - 1;        // input rows (and columns) per thread
    const int cg = tid & 31;              // channel pair inside the K-block
    const int blk = tid >> 5;             // pixel block: 4 rows x 4 cols
    const int ch = kb * BK + cg * 2;
    const int W = c.W, H = c.H;
    const int cols4 = W >> 2;             // column groups per row
    const int strip = blk / cols4;        // 4-row strip inside the tile
    const int x0 = (blk - strip * cols4) * 4;
    const int mrow = m0 / W + strip * 4;  // global row index (n*H + y) of the strip's first row
    const int n = mrow / H;
    const int y0 = mrow - n * H;
    const bool cval = ch < c.Cin;
    const bool tile_valid = (m0 + strip * 4 * W) < c.M;   // whole strips are valid or not (M % (4W) == 0)

    float2 acc[4][4];          // (2 channels) x 4 rows x 4 cols -- updated with packed FFMA2
#pragma unroll
    for (int o = 0; o < 4; ++o)
#pragma unroll
        for (int q = 0; q < 4; ++q) acc[o][q] = make_float2(0.f, 0.f);

    if (cval && tile_valid) {
        const float* xb = c.x + (size_t)n * H * W * c.ldx + ch;
        unsigned colmask = 0;
#pragma unroll
        for (int q = 0; q < NR; ++q) {
            const int ix = x0 - PAD + q;
            if (ix >= 0 && ix < W) colmask |= 1u << q;
        }
        float2 buf[3][NR];
        auto load_row = [&](int r, float2* dst) {
            const int iy = y0 - PAD + r;
            const bool rowok = iy >= 0 && iy < H;
            const float* rp = xb + (size_t)(iy * W + x0 - PAD) * c.ldx;
#pragma unroll
            for (int q = 0; q < NR; ++q) {
                dst[q] = make_float2(0.f, 0.f);
                if (rowok && ((colmask >> q) & 1u)) dst[q] = __ldg(reinterpret_cast<const float2*>(rp + (size_t)q * c.ldx));
            }
        };
        load_row(0, buf[0]);
        load_row(1, buf[1]);
        float2 wt[KS][KS];
#pragma unroll
        for (int a = 0; a < KS; ++a)
#pragma unroll
            for (int b = 0; b < KS; ++b)
                wt[a][b] = __ldg(reinterpret_cast<const float2*>(c.w_dw + (size_t)(a * KS + b) * c.Cin + ch));
        float2 ps = make_float2(1.f, 1.f), pb = make_float2(0.f, 0.f);
        if (c.pre_scale) {
            ps = __ldg(reinterpret_cast<const float2*>(c.pre_scale + ch));
            pb = __ldg(reinterpret_cast<const float2*>(c.pre_shift + ch));
        }
#pragma unroll
        for (int r = 0; r < NR; ++r) {
            if (r + 2 < NR) load_row(r + 2, buf[(r + 2) % 3]);
            const int iy = y0 - PAD + r;
            const bool rowok = iy >= 0 && iy < H;
            float2 in[NR];
#pragma unroll
            for (int q = 0; q < NR; ++q) {
                float2 v = buf[r % 3][q];
                if (rowok && ((colmask >> q) & 1u)) {      // zero padding is applied AFTER BN/ReLU
                    v = ffma2(v, ps, pb);
                    if (c.pre_relu) { v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); }
                }
                in[q] = v;
            }
#pragma unroll
            for (int o = 0; o < 4; ++o) {
                const int ky = r - o;          // compile-time after unrolling
                if (ky >= 0 && ky < KS) {
#pragma unroll
                    for (int q = 0; q < 4; ++q)
#pragma unroll
                        for (int kx = 0; kx < KS; ++kx) acc[o][q] = ffma2(wt[ky][kx], in[q + kx], acc[o][q]);
                }
            }
        }
    }
    // write the 16 pixels x 2 channels into the swizzled A tile
#pragma unroll
    for (int o = 0; o < 4; ++o)
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const int row = (strip * 4 + o) * W + x0 + q;   // row inside the 128-pixel tile
            uint32_t hi, lo;
            split2(acc[o][q].x, acc[o][q].y, hi, lo);
            const uint32_t off = swz(row, cg * 2);
            *reinterpret_cast<uint32_t*>(a_hi + off) = hi;
            if (want_lo) *reinterpret_cast<uint32_t*>(a_lo + off) = lo;
        }
}

__device__ __forceinline__ void dense_load_any(const TcParams& P, const DenseRows& R, int kb, int tid, DenseRegs& D) {
    if (P.ks < 0) dense_load_scalar(P, R, kb, tid, D);     // ks = -1: scalar gather (set by the launcher)
    else dense_load(P, R, kb, tid, D);
}

// ---------------------------------------------------------------------------
// the kernel
// ---------------------------------------------------------------------------
// Persistent, warp-specialised kernel.  Every CTA (one per SM) loops over 128-pixel tiles
//   warps 0-7   A producers (CUDA cores)          warps 8-11  consumer warpgroup (wgmma, then the epilogue)
//   warp 12     TMA weight tiles (one thread)
// connected by the mbarrier ring of smem stages full[s]/empty[s] (K-blocks, counted across tiles): the
// producers of tile i+1 run ahead while the consumer drains tile i.  Registers are rebalanced with setmaxnreg.
//
// SHARE: two CTAs (N parts 2i, 2i + 1) of one 128-pixel tile form a cluster (1,2,1) and split the A
// production: with 2 stages, CTA r owns stage r (global K-block counter g with g % 2 == r); it
// pushes each finished tile to the peer with a DSMEM bulk copy that completes on the peer's
// full[r] barrier, and each consumer releases a stage on both CTAs' empty barriers.
template <int MODE, bool SHARE>   // MODE: 0 dense/1x1, 3 separable 3x3, 5 separable 5x5
__global__ void __launch_bounds__(NTHREADS, 1)
conv_tc_kernel(const __grid_constant__ TcParams P, const __grid_constant__ CUtensorMap map_hi,
               const __grid_constant__ CUtensorMap map_lo) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    // 1024-byte alignment as an OFFSET (not a uintptr_t round-trip) so that accesses stay in the shared state space
    if (smem_u32(smem_raw) & 1023u) __trap();      // swizzled wgmma / TMA tiles need the 1024-byte alignment declared above
    uint8_t* smem = smem_raw;
    const int tid = threadIdx.x;
    const int warp = tid >> 5, lane = tid & 31;
    const bool want_lo = P.precision == 3;
    const int b_tile_bytes = P.bn_cta * 128;
    const int stage_bytes = 2 * A_TILE_BYTES + 2 * b_tile_bytes;
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + (size_t)P.stages * stage_bytes);
    // bars: full[MAX_STAGES] | empty[MAX_STAGES]
    const uint32_t bar_full0 = smem_u32(bars), bar_empty0 = smem_u32(bars + MAX_STAGES);
    const int n0 = blockIdx.y * P.bn_cta;
    const int nkb = P.n_kblocks;

    if (warp == WARP_TMA && lane == 0) {
        tma_prefetch_desc(&map_hi);
        if (want_lo) tma_prefetch_desc(&map_lo);
        for (int s = 0; s < P.stages; ++s) {
            if (SHARE) {
                // own stage: TMA-thread arrive + elected producer arrive; peer stage: TMA-thread arrive
                // (the A tile arrives as transaction bytes of the peer's bulk copy)
                mbar_init(bar_full0 + 8 * s, (uint32_t)s == cluster_ctarank() ? 2u : 1u);
                mbar_init(bar_empty0 + 8 * s, 2 * R::EPQ);          // the consumers of both CTAs
            } else {
                mbar_init(bar_full0 + 8 * s, NPROD + 1);
                mbar_init(bar_empty0 + 8 * s, R::EPQ);
            }
        }
        fence_barrier_init();
    }
    if (SHARE) cluster_sync_all(); else __syncthreads();
    const uint32_t my_rank = SHARE ? cluster_ctarank() : 0u;

    if (warp < WARP_EPI0) {
        // ======================= A producers =======================
        reg_prod<REGS_PROD, R::LAUNCH_REGS>();
        DenseRows rows;
        DenseRegs cur, nxt;
        int ti = 0;
        if (MODE == 0 && !SHARE) {
            // dense, one CTA per tile column: flat loop over (tile, K-block) items with the global loads
            // running ONE ITEM AHEAD of the shared-memory stores -- also across tile boundaries, so that a
            // short-K layer (stem 3x3 convs: 5 K-blocks, fReMap: 1) does not expose the load latency at
            // the start of every tile.  The pixel decode (rows) belongs to the load side only.
            int t_l = blockIdx.x, kb_l = 0;
            if (t_l < P.n_mtiles) {
                dense_rows_init(P.c, t_l * BM, tid, rows);
                dense_load_any(P, rows, 0, tid, cur);
                if (++kb_l == nkb) { kb_l = 0; t_l += gridDim.x; }
            }
            int s = 0;
            uint32_t it = 0;
            for (int t = blockIdx.x; t < P.n_mtiles; t += gridDim.x) {
                for (int kb = 0; kb < nkb; ++kb) {
                    const bool more = t_l < P.n_mtiles;
                    if (more) {
                        if (kb_l == 0) dense_rows_init(P.c, t_l * BM, tid, rows);
                        dense_load_any(P, rows, kb_l, tid, nxt);
                        if (++kb_l == nkb) { kb_l = 0; t_l += gridDim.x; }
                    }
                    mbar_wait(bar_empty0 + 8 * s, (it & 1) ^ 1);
                    uint8_t* a_hi = smem + (size_t)s * stage_bytes;
                    dense_store(P, cur, a_hi, a_hi + A_TILE_BYTES, tid, want_lo);
                    if (more) cur = nxt;
                    fence_proxy_async();
                    mbar_arrive(bar_full0 + 8 * s);
                    if (++s == P.stages) { s = 0; ++it; }
                }
            }
        } else
        for (int t = blockIdx.x; t < P.n_mtiles; t += gridDim.x, ++ti) {
            const int m0 = t * BM;
            const int g0 = ti * nkb;
            const int kb_first = SHARE ? (int)((my_rank ^ (uint32_t)g0) & 1u) : 0;   // (g0 + kb) % 2 == my_rank
            if (MODE == 0) {
                dense_rows_init(P.c, m0, tid, rows);
                dense_load_any(P, rows, 0, tid, cur);
            }
            for (int kb = kb_first; kb < nkb; kb += SHARE ? 2 : 1) {
                const int g = g0 + kb;
                const int s = g % P.stages;
                const uint32_t it = (uint32_t)(g / P.stages);
                if (MODE == 0 && kb + 1 < nkb) dense_load_any(P, rows, kb + 1, tid, nxt);   // prefetch next K-block
                mbar_wait(bar_empty0 + 8 * s, (it & 1) ^ 1);
                uint8_t* a_hi = smem + (size_t)s * stage_bytes;
                uint8_t* a_lo = a_hi + A_TILE_BYTES;
                if (MODE == 0) {
                    dense_store(P, cur, a_hi, a_lo, tid, want_lo);
                    cur = nxt;
                } else if (MODE == 3) produce_sep<3>(P, kb, a_hi, a_lo, m0, tid, want_lo);
                else produce_sep<5>(P, kb, a_hi, a_lo, m0, tid, want_lo);
                fence_proxy_async();           // generic-proxy smem writes -> visible to the tensor core / bulk copy
                if (SHARE) {
                    asm volatile("bar.sync 1, %0;" ::"r"(NPROD) : "memory");      // all 256 producers wrote their part
                    if (tid == 0) {
                        mbar_arrive(bar_full0 + 8 * s);                            // local copy ready
                        const uint32_t peer = my_rank ^ 1u;
                        const uint32_t peer_full = mapa_peer(bar_full0 + 8 * s, peer);
                        bulk_s2peer(mapa_peer(smem_u32(a_hi), peer), smem_u32(a_hi), A_TILE_BYTES, peer_full);
                        if (want_lo) bulk_s2peer(mapa_peer(smem_u32(a_lo), peer), smem_u32(a_lo), A_TILE_BYTES, peer_full);
                    }
                } else {
                    mbar_arrive(bar_full0 + 8 * s);
                }
            }
        }
    } else if (warp < WARP_TMA) {
        // ======================= consumer: wgmma + epilogue =======================
        reg_inc<REGS_EPI>();
        const int wt = tid - 32 * WARP_EPI0;
        float acc[R::MH][ACC_N];
        const uint64_t dbase = make_desc(smem_u32(smem));
        const uint32_t st16 = (uint32_t)stage_bytes >> 4, alo16 = A_TILE_BYTES >> 4, b16 = (2 * A_TILE_BYTES) >> 4,
                       blo16 = (uint32_t)b_tile_bytes >> 4, half16 = (64 * 128) >> 4;
        int s = 0;
        uint32_t it = 0;                                   // use count of stage s
        for (int t = blockIdx.x; t < P.n_mtiles; t += gridDim.x) {
            for (int kb = 0; kb < nkb; ++kb) {
                mbar_wait(bar_full0 + 8 * s, it & 1);
                const uint64_t da = dbase + (uint64_t)((uint32_t)s * st16);
                wg_kblock<R::MH, BK / 16>(P.bn_cta, acc, da, half16, alo16, da + b16, blo16, want_lo, kb == 0);
                wg_release<SHARE>(bar_empty0 + 8 * s, 0, wt, my_rank ^ 1u);
                if (++s == P.stages) { s = 0; ++it; }
            }
            wg_epilogue<R::MH>(P, acc, t * BM, n0, wt);
        }
    } else {
        reg_dec<REGS_CTRL>();
        if (warp == WARP_TMA) {
            // ======================= weight tiles via TMA =======================
            if (lane == 0) {
                const uint32_t tx = (uint32_t)(want_lo ? 2 : 1) * (uint32_t)b_tile_bytes;
                const uint32_t tx_a = (uint32_t)(want_lo ? 2 : 1) * (uint32_t)A_TILE_BYTES;
                int g = 0;
                for (int t = blockIdx.x; t < P.n_mtiles; t += gridDim.x) {
                    for (int kb = 0; kb < nkb; ++kb, ++g) {
                        const int s = g % P.stages;
                        const uint32_t it = (uint32_t)(g / P.stages);
                        mbar_wait(bar_empty0 + 8 * s, (it & 1) ^ 1);
                        const uint32_t full = bar_full0 + 8 * s;
                        // SHARE: K-blocks produced by the peer deliver their A tile as transaction bytes
                        mbar_arrive_expect_tx(full, tx + ((SHARE && (uint32_t)s != my_rank) ? tx_a : 0u));
                        const uint32_t b_hi = smem_u32(smem + (size_t)s * stage_bytes + 2 * A_TILE_BYTES);
                        const uint32_t b_lo = b_hi + (uint32_t)b_tile_bytes;
                        tma_load_2d(b_hi, &map_hi, kb * BK, n0, full);
                        if (want_lo) tma_load_2d(b_lo, &map_lo, kb * BK, n0, full);
                    }
                }
            }
        }
    }
    if (SHARE) cluster_sync_all(); else __syncthreads();     // a peer's remote arrivals / copies target this CTA
}

}  // namespace tc

extern "C" int dh_tc_cout_pad(int cout) {
    int bn, gy;
    tc::tile_n(cout, &bn, &gy);
    return bn * gy;
}

extern "C" int dh_tc_k_pad(int k) { return (k + tc::BK - 1) / tc::BK * tc::BK; }

bool dh_tc_supported(const ConvParams& p, const dh_packed_w* packed, bool separable) {
    if (!packed || !packed->hi) return false;
    if (p.M < 1) return false;
    const bool x16 = (reinterpret_cast<uintptr_t>(p.x) & 15) == 0;
    if (separable && !x16) return false;
    const int K = separable ? p.Cin : p.kh * p.kw * p.Cin;
    if (packed->k != dh_tc_k_pad(K) || packed->cout_pad != dh_tc_cout_pad(p.Cout)) return false;
    if (separable && p.pre_scale && ((reinterpret_cast<uintptr_t>(p.pre_scale) & 15) || (reinterpret_cast<uintptr_t>(p.pre_shift) & 15)))
        return false;
    if ((int64_t)p.N * p.H * p.W * p.ldx >= (1ll << 31)) return false;    // int32 pixel*ld products in the producers
    if (separable) {
        if (!(p.kh == p.kw && (p.kh == 3 || p.kh == 5))) return false;
        if (p.sh != 1 || p.sw != 1) return false;
        if (p.Ho != p.H || p.Wo != p.W) return false;                 // SAME, stride 1
        if (p.W < 4 || (tc::BM % p.W) != 0 || (p.W & 3) || (p.H & 3)) return false;
        if ((p.Cin & 1) || (p.ldx & 1)) return false;
        if ((reinterpret_cast<uintptr_t>(p.w_dw) & 7) != 0) return false;
        if (p.M % (4 * p.W) != 0) return false;
        return true;
    }
    // dense: any Cin / alignment (the producer falls back to a scalar gather: dh_tc_scalar_gather)
    return true;
}

static bool dh_tc_scalar_gather(const ConvParams& p) {
    return (p.Cin & 3) || (p.ldx & 3) || (reinterpret_cast<uintptr_t>(p.x) & 15) ||
           (p.pre_scale && ((reinterpret_cast<uintptr_t>(p.pre_scale) & 15) || (reinterpret_cast<uintptr_t>(p.pre_shift) & 15)));
}

int dh_launch_conv_tc(dh_ctx* ctx, const ConvParams& p, const dh_packed_w* packed, bool separable, int precision,
                      cudaStream_t s) {
    using namespace tc;
    TcParams P;
    P.c = p;
    const int K = separable ? p.Cin : p.kh * p.kw * p.Cin;
    P.c.K = K;
    P.k_pad = packed->k;
    P.n_kblocks = packed->k / BK;
    int gy;
    tile_n(p.Cout, &P.bn_cta, &gy);
    P.precision = (precision == 1) ? 1 : 3;
    P.ks = separable ? p.kh : (dh_tc_scalar_gather(p) ? -1 : 0);
    P.dbg = 0;
    P.n_mtiles = (p.M + BM - 1) / BM;
    const int stage_bytes = 2 * A_TILE_BYTES + 2 * P.bn_cta * 128;
    const int budget = 227 * 1024 - 256 /*barriers*/;
    int stages = budget / stage_bytes;
    if (stages > MAX_STAGES) stages = MAX_STAGES;
    if (stages > P.n_kblocks) stages = P.n_kblocks;
    // A-tile sharing between pairs of N-part CTAs (clusters 1x2x1) of a separable layer split over an even number
    // of N parts: CTA r of the pair produces the K-blocks of stage r, so the ring is two stages deep
    const bool share = separable && gy % 2 == 0 && P.n_kblocks >= 2 && stages >= 2 && ctx->share_a;
    if (share) stages = 2;
    if (stages < 1) {
        dh_set_error("dh_launch_conv_tc: tile does not fit shared memory");
        return -1;
    }
    P.stages = stages;
    const size_t smem = (size_t)stages * stage_bytes + 256;

    CUtensorMap map_hi, map_lo;
    if (!make_map(&map_hi, packed->hi, packed->k, packed->cout_pad, P.bn_cta) ||
        !make_map(&map_lo, packed->lo ? packed->lo : packed->hi, packed->k, packed->cout_pad, P.bn_cta)) {
        dh_set_error("dh_launch_conv_tc: cuTensorMapEncodeTiled failed");
        return -1;
    }
    // persistent: one CTA per SM; CTA (x, y) handles M-tiles x, x + gridDim.x, ... of N part y
    int gx = ctx->num_sms / gy;
    if (gx < 1) gx = 1;
    if (gx > P.n_mtiles) gx = P.n_mtiles;
    dim3 grid(gx, gy);
    cudaError_t e;
#define DH_TC_LAUNCH(MODE)                                                                                   \
    do {                                                                                                     \
        if (share) {                                                                                         \
            e = ensure_smem<conv_tc_kernel<MODE, true>>(smem); \
            if (e == cudaSuccess) {                                                                          \
                cudaLaunchConfig_t cfg = {};                                                                 \
                cfg.gridDim = grid; cfg.blockDim = dim3(NTHREADS); cfg.dynamicSmemBytes = smem; cfg.stream = s; \
                cudaLaunchAttribute at[1];                                                                   \
                at[0].id = cudaLaunchAttributeClusterDimension;                                              \
                at[0].val.clusterDim.x = 1; at[0].val.clusterDim.y = 2; at[0].val.clusterDim.z = 1;          \
                cfg.attrs = at; cfg.numAttrs = 1;                                                            \
                e = cudaLaunchKernelEx(&cfg, conv_tc_kernel<MODE, true>, P, map_hi, map_lo);                 \
            }                                                                                                \
        } else {                                                                                             \
            e = ensure_smem<conv_tc_kernel<MODE, false>>(smem); \
            if (e == cudaSuccess) conv_tc_kernel<MODE, false><<<grid, NTHREADS, smem, s>>>(P, map_hi, map_lo); \
        }                                                                                                    \
    } while (0)
    if (!separable) DH_TC_LAUNCH(0);
    else if (p.kh == 3) DH_TC_LAUNCH(3);
    else DH_TC_LAUNCH(5);
#undef DH_TC_LAUNCH
    if (e != cudaSuccess) {
        dh_set_error("dh_launch_conv_tc: launch setup failed: %s", cudaGetErrorString(e));
        return (int)e;
    }
    return 0;
}
