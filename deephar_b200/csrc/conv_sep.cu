// Fused SeparableConv2D, TMA-staged variant (the hot kernel of the ReceptionNet / SPNet stacks).
//
// replaces: Activation('relu') -> SeparableConv2D(kxk, same) -> BatchNormalization -> add
// (deephar/layers.py:288-301, models/reception.py:43-59) -- depthwise + pointwise + BN + residual
// in ONE kernel; the depthwise result never leaves the SM.
//
// Per 128-pixel tile and 32-channel K-block:
//   patch : the zero-padded input window (tile rows + halo) x 32 channels, fp32, loaded by ONE 4-D TMA
//           (cp.async.bulk.tensor.4d over the NHWC tensor; out-of-bounds coordinates are zero filled,
//           which IS the TF 'SAME' padding since the prologue here is ReLU-only) into shared memory;
//   A     : depthwise kxk on CUDA cores from the patch: each thread owns 2 channels x a 4x4 pixel
//           block, taps in registers, packed FFMA2, shared-memory loads with immediate offsets and no
//           bounds logic; result split into bf16 hi/lo and stored in the 64B-swizzled K-major wgmma layout;
//   W     : bf16 hi/lo pointwise weight tiles by 2-D TMA (64B swizzle);
//   D     : fp32 in the registers of two consumer warpgroups (rows 0-63 / 64-127), wgmma m64nNk16, three
//           MMAs per k-step (bf16x3, see conv_tc.cu); epilogue shared with conv_tc.cu (tc_common.cuh).
// Roles: warps 0-3 = the producer warpgroup, warps 4-11 consumers, warp 12 weight TMA, warp 14 patch TMA.
// Layers split over an even number of N parts run as 2-CTA clusters: CTA r produces the K-blocks of stage r
// and pushes the finished A tile to its peer over DSMEM (same protocol as conv_tc.cu).
#include "tc_common.cuh"

namespace tcs {
using namespace tc;
using R = tc::Roles<2, 1>;
constexpr int WARP_EPI0 = R::WARP_EPI0, WARP_TMA = R::WARP_TMA, WARP_PATCH = R::WARP_PATCH, NTHREADS = R::NTHREADS,
              REGS_PROD = R::REGS_PROD, REGS_EPI = R::REGS_EPI, REGS_CTRL = R::REGS_CTRL;

constexpr int A_BYTES = BM * 64;           // 8 KB per (hi | lo)
constexpr int NWG = 128;                   // threads per producer warpgroup
constexpr int NPW = 1;                     // producer warpgroups (see tc_common.cuh Roles: one, with 192 registers)
constexpr int NA = 3;                      // A-tile ring depth (the weight ring stays 2 deep)

struct SepParams {
    TcParams t;
    int patch_stride;       // bytes between the two patch buffers (>= patch_bytes, 1024-aligned)
    int patch_bytes;
    int ry, fn;             // tile rows per frame, frames per tile
    int dbg;                // ablation bits (tools/ only): 1 no depthwise math, 2 no patch TMA, 8 no DSMEM push, 16 no weight TMA, 64 no MMA issue (32: epilogue without global traffic, tc_common.cuh)
};

template <int KS, int TW, bool SHARE, bool BNPRO>
__global__ void __launch_bounds__(NTHREADS, 1)
sep_tma_kernel(const __grid_constant__ SepParams SP, const __grid_constant__ CUtensorMap map_hi,
               const __grid_constant__ CUtensorMap map_lo, const __grid_constant__ CUtensorMap map_x) {
    constexpr int PAD = KS / 2;
    constexpr int PC = TW + 2 * PAD;          // patch columns
    constexpr int NR = 4 + KS - 1;            // input rows / cols per 4x4 block
#ifdef DH_ABLATE
    const int DBG = SP.dbg;          // timing-ablation bits (tools/ builds only; results are wrong when set)
#else
    constexpr int DBG = 0;
#endif
    const TcParams& P = SP.t;
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    // 1024-byte alignment as an OFFSET (not a uintptr_t round-trip) so that accesses stay in the shared state space
    if (smem_u32(smem_raw) & 1023u) __trap();      // swizzled wgmma / TMA tiles need the 1024-byte alignment declared above
    uint8_t* smem = smem_raw;
    const int tid = threadIdx.x;
    const int warp = tid >> 5, lane = tid & 31;
    const bool want_lo = P.precision == 3;
    const int b_bytes = P.bn_cta * 64;                       // per (hi | lo)
    // smem: A ring [NA][hi | lo] | weight ring [2][hi | lo] | patches [2] | barriers
    uint8_t* b_ring = smem + NA * 2 * A_BYTES;
    uint8_t* patch0 = b_ring + 2 * 2 * b_bytes;
    uint64_t* bars = reinterpret_cast<uint64_t*>(patch0 + 2 * SP.patch_stride);
    // bars: fullA[NA] | emptyA[NA][2] | fullB[2] | emptyB[2] | pfull[2] | pempty[2]
    // K-block g uses A stage g % NA (use g / NA) and weight stage g & 1 (use g >> 1).  In the cluster variant
    // K-block g is produced by CTA g & 1, so consecutive own productions land in different A stages and the
    // store of one does not have to wait for the MMAs of the previous one.
    // emptyA[s][u & 1] is signalled when use u of stage s has been consumed by the consumers (of both CTAs).  Two
    // barriers per stage, alternating by use, so that every waiter sees consecutive phases of its barrier.
    constexpr int NB_A = NA + 2 * NA;
    const uint32_t bar_full0 = smem_u32(bars), bar_empty0 = smem_u32(bars + NA), bar_fullb0 = smem_u32(bars + NB_A),
                   bar_emptyb0 = smem_u32(bars + NB_A + 2), bar_pfull0 = smem_u32(bars + NB_A + 4),
                   bar_pempty0 = smem_u32(bars + NB_A + 6);
    const int n0 = blockIdx.y * P.bn_cta;
    const int nkb = P.n_kblocks;
    const uint32_t my_rank = SHARE ? cluster_ctarank() : 0u;

    if (warp == WARP_TMA && lane == 0) {
        tma_prefetch_desc(&map_hi);
        if (want_lo) tma_prefetch_desc(&map_lo);
        tma_prefetch_desc(&map_x);
        for (int s = 0; s < NA; ++s) {
            // fullA: SHARE: one arrival per use -- the elected producer thread (own K-block) or the TMA thread's
            // arrive.expect_tx for the A bytes the peer pushes; else every producer thread of the warpgroup
            mbar_init(bar_full0 + 8 * s, SHARE ? 1u : (uint32_t)NWG);
            mbar_init(bar_empty0 + 16 * s, (SHARE ? 2u : 1u) * R::EPQ);            // consumer warpgroups (of both CTAs)
            mbar_init(bar_empty0 + 16 * s + 8, (SHARE ? 2u : 1u) * R::EPQ);
        }
        for (int s = 0; s < 2; ++s) {
            mbar_init(bar_fullb0 + 8 * s, 1);
            mbar_init(bar_emptyb0 + 8 * s, R::EPQ);
            mbar_init(bar_pfull0 + 8 * s, 1);
            mbar_init(bar_pempty0 + 8 * s, NWG);
        }
        fence_barrier_init();
    }
    if (SHARE) cluster_sync_all(); else __syncthreads();

    const int tiles_mine = ((int)P.n_mtiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;
    const int total_g = tiles_mine * nkb;       // K-blocks this CTA's consumers read
    // own K-blocks (the ones this CTA produces): SHARE: g = 2j + rank ; else g = j
    const int n_own = SHARE ? (total_g - (int)my_rank + 1) / 2 : total_g;

    if (warp < WARP_EPI0) {
        // ======================= depthwise producers (two warpgroups) =======================
        reg_prod<REGS_PROD, R::LAUNCH_REGS>();
        const ConvParams& c = P.c;
        const int w = warp >> 2;                       // producer warpgroup: own K-blocks j = w, w + NPW, ...; patch buffer j & 1
        const int tw = tid & (NWG - 1);
        const int cp = tw & 15;                        // channel pair inside the 32-channel K-block
        const int blk = tw >> 4;                       // 4x4 pixel block inside the 128-pixel tile
        constexpr int XB = TW / 4;
        const int strip = blk / XB, xb = blk - strip * XB;
        const int fn = (strip * 4) / SP.ry, ry = (strip * 4) - fn * SP.ry;
        const int prr = SP.ry + 2 * PAD;               // patch rows per frame
        const float* pbase0 = reinterpret_cast<const float*>(patch0) +
                             ((size_t)((fn * prr + ry) * PC + xb * 4)) * SBK + cp * 2;
        const int row0 = strip * 4 * TW + xb * 4;      // tile-local pixel of output (o = 0, q = 0)
        const float lowb = c.pre_relu ? 0.f : -3.402823466e38f;
        // BNPRO: BatchNormalization before the ReLU (models/common.py:25-67 residual units).  The TMA zero fill is
        // the padding of the RAW tensor; keras pads the ACTIVATED one, so out-of-image taps are forced back to zero
        // after the affine: per-thread column mask (fixed) x per-tile row mask.
        unsigned colmask = 0;
        if (BNPRO) {
#pragma unroll
            for (int q = 0; q < NR; ++q) {
                const int ix = xb * 4 + q - PAD;
                if (ix >= 0 && ix < TW) colmask |= 1u << q;
            }
        }
        // depthwise taps of the thread's two channels: loaded for the NEXT own K-block right after the math of the
        // current one (the registers are dead then), so the global-load latency hides behind the bf16 split / stage
        // hand-over instead of stalling the first FMA of every K-block
        float2 wt[KS][KS];
        auto load_taps = [&](int jn) {
            const int gn = SHARE ? 2 * jn + (int)my_rank : jn;
            const int kbn = gn % nkb;
            const float* wp = c.w_dw + kbn * SBK + cp * 2;
#pragma unroll
            for (int a = 0; a < KS; ++a)
#pragma unroll
                for (int b = 0; b < KS; ++b)
                    wt[a][b] = __ldg(reinterpret_cast<const float2*>(wp + (size_t)(a * KS + b) * c.Cin));
        };
        if (w < n_own) load_taps(w);
        for (int j = w; j < n_own; j += NPW) {
            const int pb_i = j & 1;                      // patch buffer of own K-block j (filled by the patch-TMA warp in j order)
            const uint32_t pfull = bar_pfull0 + 8 * pb_i, pempty = bar_pempty0 + 8 * pb_i;
            const float* pbase = pbase0 + (size_t)pb_i * (SP.patch_stride / 4);
            const int g = SHARE ? 2 * j + (int)my_rank : j;
            const int ti = g / nkb, kb = g - ti * nkb;
            const int ch = kb * SBK + cp * 2;
            // (the KS x KS tap pairs of this K-block's two channels were loaded one iteration ago: `wt`)
            float2 acc[4][4];
#pragma unroll
            for (int o = 0; o < 4; ++o)
#pragma unroll
                for (int q = 0; q < 4; ++q) acc[o][q] = make_float2(0.f, 0.f);
            float2 ps = make_float2(1.f, 1.f), pb = make_float2(0.f, 0.f);
            unsigned rowmask = 0;
            if (BNPRO) {
                ps = __ldg(reinterpret_cast<const float2*>(c.pre_scale + ch));
                pb = __ldg(reinterpret_cast<const float2*>(c.pre_shift + ch));
                const int t = blockIdx.x + ti * gridDim.x;
                const int y0 = SP.fn > 1 ? 0 : ((t * BM) / TW) % c.H;
#pragma unroll
                for (int r = 0; r < NR; ++r) {
                    const int iy = y0 + ry + r - PAD;
                    if (iy >= 0 && iy < c.H) rowmask |= 1u << r;
                }
            }

            if (!(DBG & 2)) mbar_wait_relaxed(pfull, (uint32_t)((j >> 1) & 1), (DBG & 2048) ? 32u : 0u);
            // input rows are loaded one row ahead of their FMAs (two register rows, compile-time ping-pong); within
            // a row the FMAs go tap-column by tap-column over all (output row, output column) accumulators, so
            // consecutive FFMA2 never touch the same accumulator
            auto load_row = [&](int r, float2* in) {
#pragma unroll
                for (int q = 0; q < NR; ++q) {
                    float2 v = *reinterpret_cast<const float2*>(pbase + (r * PC + q) * SBK);
                    if (BNPRO) v = ffma2(v, ps, pb);
                    v = make_float2(fmaxf(v.x, lowb), fmaxf(v.y, lowb));
                    if (BNPRO && !(((rowmask >> r) & 1u) && ((colmask >> q) & 1u))) v = make_float2(0.f, 0.f);
                    in[q] = v;
                }
            };
            if (!(DBG & 1)) {
                float2 inb[2][NR];
                load_row(0, inb[0]);
#pragma unroll
                for (int r = 0; r < NR; ++r) {
                    if (r + 1 < NR) load_row(r + 1, inb[(r + 1) & 1]);
                    const float2* in = inb[r & 1];
#pragma unroll
                    for (int kx = 0; kx < KS; ++kx)
#pragma unroll
                        for (int o = 0; o < 4; ++o) {
                            const int ky = r - o;          // compile-time after unrolling
                            if (ky >= 0 && ky < KS) {
#pragma unroll
                                for (int q = 0; q < 4; ++q) acc[o][q] = ffma2(wt[ky][kx], in[q + kx], acc[o][q]);
                            }
                        }
                }
            }
            if (j + NPW < n_own) load_taps(j + NPW);
            if (!(DBG & 2)) mbar_arrive(pempty);    // patch buffer may be refilled

            const int s = g % NA;
            const uint32_t it = (uint32_t)(g / NA);
            wait_stage_free(bar_empty0, s, it, (DBG & 2048) ? 32u : 0u);
            uint8_t* a_hi = smem + (size_t)s * (2 * A_BYTES);
            uint8_t* a_lo = a_hi + A_BYTES;
#pragma unroll
            for (int o = 0; o < 4; ++o)
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    uint32_t hi, lo;
                    split2(acc[o][q].x, acc[o][q].y, hi, lo);
                    const uint32_t off = swz64(row0 + o * TW + q, cp * 2);
                    *reinterpret_cast<uint32_t*>(a_hi + off) = hi;
                    if (want_lo) *reinterpret_cast<uint32_t*>(a_lo + off) = lo;
                }
            fence_proxy_async();
            if (SHARE) {
                asm volatile("bar.sync %0, %1;" ::"r"(1 + w), "r"(NWG) : "memory");
                if (tw == 0) {
                    mbar_arrive(bar_full0 + 8 * s);
                    const uint32_t peer = my_rank ^ 1u;
                    const uint32_t peer_full = mapa_peer(bar_full0 + 8 * s, peer);
                    if (!(DBG & 8)) {
                        bulk_s2peer(mapa_peer(smem_u32(a_hi), peer), smem_u32(a_hi), A_BYTES, peer_full);
                        if (want_lo) bulk_s2peer(mapa_peer(smem_u32(a_lo), peer), smem_u32(a_lo), A_BYTES, peer_full);
                    }
                }
            } else {
                mbar_arrive(bar_full0 + 8 * s);
            }
        }
    } else if (warp < WARP_TMA) {
        // ======================= consumers: wgmma + epilogue (warpgroup wg: rows 64 wg .. + 63) =======================
        reg_inc<REGS_EPI>();
        const int wg = (warp - WARP_EPI0) >> 2, wt = tid - 32 * WARP_EPI0 - 128 * wg;
        float acc[R::MH][ACC_N];
        const uint64_t dbase = make_desc64(smem_u32(smem) + (uint32_t)(wg * 64 * 64));
        const uint64_t dbase_b = make_desc64(smem_u32(b_ring));
        const uint32_t sta16 = (2 * A_BYTES) >> 4, stb16 = (uint32_t)(2 * b_bytes) >> 4, alo16 = A_BYTES >> 4,
                       blo16 = (uint32_t)b_bytes >> 4;
        int g = 0;
        for (int ti = 0; ti < tiles_mine; ++ti) {
            for (int kb = 0; kb < nkb; ++kb, ++g) {
                const int s = g % NA, sb = g & 1;
                const uint32_t it = (uint32_t)(g / NA);
                if (!(DBG & 128)) mbar_wait(bar_full0 + 8 * s, it & 1);
                mbar_wait(bar_fullb0 + 8 * sb, (uint32_t)(g >> 1) & 1);
                if (!(DBG & 64))
                    wg_kblock<R::MH, SBK / 16>(P.bn_cta, acc, dbase + (uint64_t)((uint32_t)s * sta16), 0u, alo16,
                                               dbase_b + (uint64_t)((uint32_t)sb * stb16), blo16, want_lo, kb == 0);
                wg_release<SHARE>(bar_empty0 + 16 * s + 8 * (it & 1), wg, wt, my_rank ^ 1u);
                if (wt == 0) mbar_arrive(bar_emptyb0 + 8 * sb);
            }
            wg_epilogue<R::MH>(P, acc, ((int)blockIdx.x + ti * (int)gridDim.x) * BM + 64 * wg, n0, wt);
        }
    } else {
        reg_dec<REGS_CTRL>();
        if (warp == WARP_TMA) {
            // ======================= weight tiles via TMA =======================
            if (lane == 0) {
                const uint32_t tx = (DBG & 16) ? 0u : (uint32_t)(want_lo ? 2 : 1) * (uint32_t)b_bytes;
                const uint32_t tx_a = (DBG & 8) ? 0u : (uint32_t)(want_lo ? 2 : 1) * (uint32_t)A_BYTES;
                for (int g = 0; g < total_g; ++g) {
                    const int ti = g / nkb, kb = g - ti * nkb;
                    const int sb = g & 1;
                    const uint32_t itb = (uint32_t)(g >> 1);
                    if (itb >= 1) mbar_wait_relaxed(bar_emptyb0 + 8 * sb, (itb - 1) & 1, (DBG & 2048) ? 64u : 0u);
                    const uint32_t full = bar_fullb0 + 8 * sb;
                    mbar_arrive_expect_tx(full, tx);
                    const uint32_t b_hi = smem_u32(b_ring + (size_t)sb * (2 * b_bytes));
                    const uint32_t b_lo = b_hi + (uint32_t)b_bytes;
                    if (!(DBG & 16)) {
                        tma_load_2d(b_hi, &map_hi, kb * SBK, n0, full);
                        if (want_lo) tma_load_2d(b_lo, &map_lo, kb * SBK, n0, full);
                    }
                    if (SHARE && (uint32_t)(g & 1) != my_rank) {
                        // the peer produces this K-block: arm our fullA for the bytes it will push (the previous
                        // use of the stage has been consumed by both CTAs, so the barrier is in the right phase)
                        const int sa = g % NA;
                        wait_stage_free(bar_empty0, sa, (uint32_t)(g / NA));
                        mbar_arrive_expect_tx(bar_full0 + 8 * sa, tx_a);
                    }
                }
            }
        } else if (warp == WARP_PATCH) {
            // ======================= input patches via 4-D TMA =======================
            if (lane == 0 && !(DBG & 2)) {
                const ConvParams& c = P.c;
                auto coords = [&](int j, int& kb, int& nf, int& y0) {
                    const int g = SHARE ? 2 * j + (int)my_rank : j;
                    const int ti = g / nkb;
                    kb = g - ti * nkb;
                    const int t = blockIdx.x + ti * gridDim.x;
                    const int grow = (t * BM) / TW;                 // global row index (n*H + y) of the tile's first row
                    nf = grow / c.H;
                    y0 = grow - nf * c.H;
                };
                for (int j = 0; j < n_own; ++j) {
                    int kb, nf, y0;
                    coords(j, kb, nf, y0);
                    const int w = j & 1;
                    const int pfd = (DBG & 1024) ? 2 : (DBG & 4096) ? 4 : (DBG & 8192) ? 9 : 0;   // L2 prefetch distance (K-blocks)
                    if (pfd && j + pfd < n_own) {
                        int kb2, nf2, y2;
                        coords(j + pfd, kb2, nf2, y2);
                        tma_prefetch_4d(&map_x, kb2 * SBK, -PAD, y2 - PAD, nf2);
                    }
                    mbar_wait_relaxed(bar_pempty0 + 8 * w, (uint32_t)(((j >> 1) & 1) ^ 1), (DBG & 2048) ? 64u : 0u);
                    const uint32_t pf = bar_pfull0 + 8 * w;
                    mbar_arrive_expect_tx(pf, (uint32_t)SP.patch_bytes);
                    tma_load_4d(smem_u32(patch0 + (size_t)w * SP.patch_stride), &map_x, kb * SBK, -PAD, y0 - PAD, nf, pf);
                }
            }
        }
    }
    if (SHARE) cluster_sync_all(); else __syncthreads();     // a peer's remote arrivals / copies target this CTA
}

// NHWC fp32 activations as a 4-D tensor (C, W, H, N); box = (32 ch, W + 2*PAD, rows + 2*PAD, frames)
static bool make_map_x(CUtensorMap* map, const ConvParams& p, int pc, int prr, int fn) {
    EncodeTiledFn enc = get_encode();
    if (!enc) return false;
    cuuint64_t dims[4] = {(cuuint64_t)p.Cin, (cuuint64_t)p.W, (cuuint64_t)p.H, (cuuint64_t)p.N};
    cuuint64_t strides[3] = {(cuuint64_t)p.ldx * 4, (cuuint64_t)p.W * p.ldx * 4, (cuuint64_t)p.H * p.W * p.ldx * 4};
    cuuint32_t box[4] = {(cuuint32_t)SBK, (cuuint32_t)pc, (cuuint32_t)prr, (cuuint32_t)fn};
    cuuint32_t estr[4] = {1, 1, 1, 1};
    return enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, const_cast<float*>(p.x), dims, strides, box, estr,
               CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

}  // namespace tcs

// Shapes the TMA-staged kernel takes (everything else stays on conv_tc.cu's register-sliding producer).
bool dh_sep_tma_supported(const dh_ctx* ctx, const ConvParams& p, const dh_packed_w* packed) {
    if (!ctx->sep_tma) return false;
    if (!packed || !packed->hi || !packed->lo) return false;
    if (!(p.kh == p.kw && (p.kh == 3 || p.kh == 5)) || p.sh != 1 || p.sw != 1) return false;
    if (p.Ho != p.H || p.Wo != p.W) return false;
    if (p.pre_scale && ((reinterpret_cast<uintptr_t>(p.pre_scale) & 7) || (reinterpret_cast<uintptr_t>(p.pre_shift) & 7))) return false;
    if (!(p.W == 32 || p.W == 16 || p.W == 8)) return false;
    const int tr = tc::BM / p.W;
    if (tr <= p.H ? (p.H % tr) != 0 : (tr % p.H) != 0) return false;
    if ((p.Cin % tcs::SBK) != 0 || (p.ldx & 3)) return false;
    if ((reinterpret_cast<uintptr_t>(p.x) & 15) || (reinterpret_cast<uintptr_t>(p.w_dw) & 7)) return false;
    if (packed->cout_pad != dh_tc_cout_pad(p.Cout) || packed->k < p.Cin) return false;
    return true;
}

int dh_launch_sep_tma(dh_ctx* ctx, const ConvParams& p, const dh_packed_w* packed, int precision, cudaStream_t s) {
    using namespace tc;
    using namespace tcs;
    SepParams SP;
    TcParams& P = SP.t;
    P.c = p;
    P.c.K = p.Cin;
    P.k_pad = packed->k;
    P.n_kblocks = p.Cin / SBK;
    int gy;
    tile_n(p.Cout, &P.bn_cta, &gy);
    P.precision = (precision == 1) ? 1 : 3;
    P.ks = p.kh;
    P.n_mtiles = (p.M + BM - 1) / BM;
    P.stages = 2;
    const int pad = p.kh / 2;
    const int tr = BM / p.W;
    SP.ry = tr <= p.H ? tr : p.H;
    SP.fn = tr <= p.H ? 1 : tr / p.H;
    const int pc = p.W + 2 * pad, prr = SP.ry + 2 * pad;
    SP.patch_bytes = SBK * 4 * pc * prr * SP.fn;
    SP.patch_stride = (SP.patch_bytes + 1023) / 1024 * 1024;
#ifdef DH_ABLATE
    SP.dbg = ctx->dbg;
    P.dbg = ctx->dbg;
#else
    SP.dbg = 0;
    P.dbg = 0;
#endif
    const size_t smem = (size_t)NA * 2 * A_BYTES + (size_t)2 * 2 * P.bn_cta * 64 + 2 * (size_t)SP.patch_stride + 512;
    if (smem > 227 * 1024) {
        dh_set_error("dh_launch_sep_tma: tile does not fit shared memory");
        return -1;
    }
    CUtensorMap map_hi, map_lo, map_x;
    if (!make_map_b64(&map_hi, packed->hi, packed->k, packed->cout_pad, P.bn_cta) ||
        !make_map_b64(&map_lo, packed->lo, packed->k, packed->cout_pad, P.bn_cta) ||
        !make_map_x(&map_x, p, pc, prr, SP.fn)) {
        dh_set_error("dh_launch_sep_tma: cuTensorMapEncodeTiled failed");
        return -1;
    }
    int gx = ctx->num_sms / gy;
    if (gx < 1) gx = 1;
    if (gx > P.n_mtiles) gx = P.n_mtiles;
    dim3 grid(gx, gy);
    const bool share = gy % 2 == 0 && ctx->share_a;
    cudaError_t e = cudaSuccess;
#define DH_SEP_LAUNCH_(KS_, TW_, BN_)                                                                                \
    do {                                                                                                         \
        if (share) {                                                                                             \
            e = ensure_smem<sep_tma_kernel<KS_, TW_, true, BN_>>(smem); \
            if (e == cudaSuccess) {                                                                              \
                cudaLaunchConfig_t cfg = {};                                                                     \
                cfg.gridDim = grid; cfg.blockDim = dim3(NTHREADS); cfg.dynamicSmemBytes = smem; cfg.stream = s;  \
                cudaLaunchAttribute at[1];                                                                       \
                at[0].id = cudaLaunchAttributeClusterDimension;                                                  \
                at[0].val.clusterDim.x = 1; at[0].val.clusterDim.y = 2; at[0].val.clusterDim.z = 1;              \
                cfg.attrs = at; cfg.numAttrs = 1;                                                                \
                e = cudaLaunchKernelEx(&cfg, sep_tma_kernel<KS_, TW_, true, BN_>, SP, map_hi, map_lo, map_x);         \
            }                                                                                                    \
        } else {                                                                                                 \
            e = ensure_smem<sep_tma_kernel<KS_, TW_, false, BN_>>(smem); \
            if (e == cudaSuccess) sep_tma_kernel<KS_, TW_, false, BN_><<<grid, NTHREADS, smem, s>>>(SP, map_hi, map_lo, map_x); \
        }                                                                                                        \
    } while (0)
#define DH_SEP_LAUNCH(KS_, TW_) do { if (p.pre_scale) DH_SEP_LAUNCH_(KS_, TW_, true); else DH_SEP_LAUNCH_(KS_, TW_, false); } while (0)
    if (p.kh == 5) {
        if (p.W == 32) DH_SEP_LAUNCH(5, 32); else if (p.W == 16) DH_SEP_LAUNCH(5, 16); else DH_SEP_LAUNCH(5, 8);
    } else {
        if (p.W == 32) DH_SEP_LAUNCH(3, 32); else if (p.W == 16) DH_SEP_LAUNCH(3, 16); else DH_SEP_LAUNCH(3, 8);
    }
#undef DH_SEP_LAUNCH
#undef DH_SEP_LAUNCH_
    if (e != cudaSuccess) {
        dh_set_error("dh_launch_sep_tma: launch setup failed: %s", cudaGetErrorString(e));
        return (int)e;
    }
    return 0;
}
