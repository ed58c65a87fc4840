// Fused SeparableConv2D, TMA-staged variant (the hot kernel of the ReceptionNet / SPNet stacks).
//
// replaces: Activation('relu') -> SeparableConv2D(kxk, same) -> BatchNormalization -> add
// (deephar/layers.py:288-301, models/reception.py:43-59) -- depthwise + pointwise + BN + residual
// in ONE kernel; the depthwise result never leaves the SM.
//
// Per pixel tile (128 x 96: 128 pixels, up to 96 output channels; or 64 x 144) and 32-channel K-block:
//   patch : the zero-padded input window (tile rows + halo) x 32 channels, fp32, loaded by ONE 4-D TMA
//           (cp.async.bulk.tensor.4d over the NHWC tensor; out-of-bounds coordinates are zero filled,
//           which IS the TF 'SAME' padding since the prologue here is ReLU-only) into shared memory;
//   A     : depthwise kxk on CUDA cores from the patch: each thread owns 2 channels x a 4x4 (64-row tiles: 2x4)
//           pixel block, taps in registers, packed FFMA2, shared-memory loads with immediate offsets and no
//           bounds logic; result split into bf16 hi/lo and stored in the 64B-swizzled K-major wgmma layout;
//   W     : bf16 hi/lo pointwise weight tiles by 2-D TMA (64B swizzle);
//   D     : fp32 in the registers of two consumer warpgroups that take alternate tiles (ping-pong: one runs its
//           epilogue while the other issues the next tile's wgmmas), wgmma m64nNk16, three MMAs per k-step
//           (bf16x3, see conv_tc.cu); epilogue shared with conv_tc.cu (tc_common.cuh).
//           64-row tiles stage the epilogue in shared memory instead (tc_common.cuh EpiSmem): residuals by TMA
//           during the mainloop, output by TMA store.
// Roles: warps 0-3 = the producer warpgroup, warps 4-11 consumers, warp 12 weight TMA, warp 13 residual TMA (64-row
// tiles), warp 14 patch TMA.
// Layers split over an even number of N parts run as 2-CTA clusters: CTA r produces the K-blocks of stage r
// and pushes the finished A tile to its peer over DSMEM (same protocol as conv_tc.cu).
#include "tc_common.cuh"

namespace tcs {
using namespace tc;
using R = tc::Roles<2, 1>;
constexpr int WARP_EPI0 = R::WARP_EPI0, WARP_TMA = R::WARP_TMA, WARP_PATCH = R::WARP_PATCH, NTHREADS = R::NTHREADS,
              REGS_PROD = R::REGS_PROD, REGS_EPI = R::REGS_EPI, REGS_CTRL = R::REGS_CTRL;

constexpr int NWG = 128;                   // threads per producer warpgroup
constexpr int NPW = 1;                     // producer warpgroups (see tc_common.cuh Roles: one, with 192 registers)
// Ring depths.  The consumers keep one K-block's wgmmas in flight and release its stages one K-block late, so every
// ring holds one K-block more than it would with a drained pipe.  At 5x5 the patch box of a 128-row tile is 30-36 KB
// (36 KB at W = 32: 4 x 16 KB (A) + 3 x 12 KB (weights at bn_cta = 96) + 3 x 36 KB (patches) = 208 KB of the 227 KB a
// block may use), except on 4 x 8 maps: a tile holds four frames and the patch is 48 KB, so the rings fit only up to
// bn_cta = 32.  A 64 x 144 tile needs 4 x 8 KB + 3 x 18 KB + 3 x 18-27 KB = 140-167 KB at the same depths,
// plus the shared-memory epilogue's buffer: 36 KB, and 9 KB more for an upsampled second residual (at most 214 KB).
// dh_plan_sep_tma leaves the layers that do not fit to conv_tc.cu.
constexpr int NA = 4;                      // A-tile ring (even: a CTA of a pair produces into stages r, r + 2)
constexpr int NB = 3;                      // weight ring
constexpr int NP = 3;                      // patch ring (own K-blocks)
#ifdef DH_ABLATE
constexpr int DBG_TILE64 = 1 << 14, DBG_TILE128 = 1 << 15;   // plan bits (tools/ builds): force a tile geometry
constexpr int DBG_EPI_REG = 1 << 16;                          // plan bit: 64-row tiles keep the register epilogue
#endif

// TBM: rows per tile, BM (tiles of 128 x bn_cta <= 96) or BM64 (64 x 144)
template <int TBM, int KS, int TW, bool SHARE, bool BNPRO, bool LO>   // LO: precision 3 (bf16x3), else 1
__global__ void __launch_bounds__(NTHREADS, 1)
sep_tma_kernel(const __grid_constant__ SepParams SP, const __grid_constant__ CUtensorMap map_hi,
               const __grid_constant__ CUtensorMap map_lo, const __grid_constant__ CUtensorMap map_x,
               const __grid_constant__ CUtensorMap map_out, const __grid_constant__ CUtensorMap map_r0,
               const __grid_constant__ CUtensorMap map_r1) {
    constexpr int PAD = KS / 2;
    constexpr int PC = TW + 2 * PAD;          // patch columns
    constexpr int OR = TBM / 32;              // output rows of a thread's pixel block (x 4 columns): 128 threads
    constexpr int NR = OR + KS - 1;           // input rows per pixel block
    constexpr int NC = 4 + KS - 1;            // input columns per pixel block
    constexpr int A_BYTES = TBM * 64;         // A tile of one K-block, per (hi | lo)
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
    constexpr bool want_lo = LO;
    const int b_bytes = P.bn_cta * 64;                       // per (hi | lo)
    // smem: A ring [NA][hi | lo] | weight ring [NB][hi | lo] | patches [NP] | epilogue buffer, up2x rows (64-row tiles:
    // SP.epi_smem bytes) | barriers (512 B) | BN scale / shift
    uint8_t* b_ring = smem + NA * 2 * A_BYTES;
    uint8_t* patch0 = b_ring + NB * 2 * b_bytes;
    uint8_t* epi_buf = patch0 + NP * SP.patch_stride;
    uint64_t* bars = reinterpret_cast<uint64_t*>(epi_buf + SP.epi_smem);
    float* post = reinterpret_cast<float*>(bars + 64);
    // bars: fullA[NA] | emptyA[NA][2] | fullB[NB] | emptyB[NB] | pfull[NP] | pempty[NP] | epi_full[2] | epi_empty
    // K-block g uses A stage g % NA (use g / NA) and weight stage g % NB (use g / NB); own K-block j uses patch
    // buffer j % NP.  In the cluster variant K-block g is produced by CTA g & 1, so consecutive own productions
    // land in different A stages and the store of one does not have to wait for the MMAs of the previous one.
    // emptyA[s][u & 1] is signalled when use u of stage s has been consumed by the consumer warpgroup that owns the
    // K-block's tile: in both CTAs on the CTA that produces the stage (its producer overwrites both copies), only in
    // this one on the other (its weight-TMA thread waits there only to re-arm fullA, so it does not wait for the
    // peer's consumers, and neither do the weight loads queued behind it).  Two barriers per stage, alternating by
    // use, so that every waiter sees consecutive phases of its barrier.
    constexpr int NB_A = NA + 2 * NA;
    const uint32_t bar_full0 = smem_u32(bars), bar_empty0 = smem_u32(bars + NA), bar_fullb0 = smem_u32(bars + NB_A),
                   bar_emptyb0 = smem_u32(bars + NB_A + NB), bar_pfull0 = smem_u32(bars + NB_A + 2 * NB),
                   bar_pempty0 = smem_u32(bars + NB_A + 2 * NB + NP), bar_epi_full0 = smem_u32(bars + NB_A + 2 * NB + 2 * NP),
                   bar_epi_empty = bar_epi_full0 + 16;
    const bool epi = TBM == BM64 && SP.epi_smem > 0;
    const int n0 = blockIdx.y * P.bn_cta;
    const int nkb = P.n_kblocks;
    const uint32_t my_rank = SHARE ? cluster_ctarank() : 0u;

    if (warp == WARP_TMA && lane == 0) {
        tma_prefetch_desc(&map_hi);
        if (want_lo) tma_prefetch_desc(&map_lo);
        tma_prefetch_desc(&map_x);
        if (epi) {
            tma_prefetch_desc(&map_out);
            mbar_init(bar_epi_full0, 1);
            mbar_init(bar_epi_full0 + 8, 1);
            mbar_init(bar_epi_empty, 1);
        }
        for (int s = 0; s < NA; ++s) {
            // fullA: SHARE: one arrival per use -- the elected producer thread (own K-block) or the TMA thread's
            // arrive.expect_tx for the A bytes the peer pushes; else every producer thread of the warpgroup
            mbar_init(bar_full0 + 8 * s, SHARE ? 1u : (uint32_t)NWG);
            const uint32_t releases = SHARE && (uint32_t)(s & 1) == my_rank ? 2u : 1u;
            mbar_init(bar_empty0 + 16 * s, releases);
            mbar_init(bar_empty0 + 16 * s + 8, releases);
        }
        for (int s = 0; s < NB; ++s) {
            mbar_init(bar_fullb0 + 8 * s, 1);
            mbar_init(bar_emptyb0 + 8 * s, 1);
        }
        for (int s = 0; s < NP; ++s) {
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
        const int w = warp >> 2;                       // producer warpgroup: own K-blocks j = w, w + NPW, ...; patch buffer j % NP
        const int tw = tid & (NWG - 1);
        const int cp = tw & 15;                        // channel pair inside the 32-channel K-block
        const int blk = tw >> 4;                       // OR x 4 pixel block inside the tile (8 blocks)
        constexpr int XB = TW / 4;
        const int strip = blk / XB, xb = blk - strip * XB;
        const int fn = (strip * OR) / SP.ry, ry = (strip * OR) - fn * SP.ry;
        const int prr = SP.ry + 2 * PAD;               // patch rows per frame
        const float* pbase0 = reinterpret_cast<const float*>(patch0) +
                             ((size_t)((fn * prr + ry) * PC + xb * 4)) * SBK + cp * 2;
        const int row0 = strip * OR * TW + xb * 4;     // tile-local pixel of output (o = 0, q = 0)
        const float lowb = c.pre_relu ? 0.f : -3.402823466e38f;
        // BNPRO: BatchNormalization before the ReLU (models/common.py:25-67 residual units).  The TMA zero fill is
        // the padding of the RAW tensor; keras pads the ACTIVATED one, so out-of-image taps are forced back to zero
        // after the affine: per-thread column mask (fixed) x per-tile row mask.
        unsigned colmask = 0;
        if (BNPRO) {
#pragma unroll
            for (int q = 0; q < NC; ++q) {
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
            const int pb_i = j % NP;                     // patch buffer of own K-block j (filled by the patch-TMA warp in j order)
            const uint32_t pfull = bar_pfull0 + 8 * pb_i, pempty = bar_pempty0 + 8 * pb_i;
            const float* pbase = pbase0 + (size_t)pb_i * (SP.patch_stride / 4);
            const int g = SHARE ? 2 * j + (int)my_rank : j;
            const int ti = g / nkb, kb = g - ti * nkb;
            const int ch = kb * SBK + cp * 2;
            // (the KS x KS tap pairs of this K-block's two channels were loaded one iteration ago: `wt`)
            float2 acc[OR][4];
#pragma unroll
            for (int o = 0; o < OR; ++o)
#pragma unroll
                for (int q = 0; q < 4; ++q) acc[o][q] = make_float2(0.f, 0.f);
            float2 ps = make_float2(1.f, 1.f), pb = make_float2(0.f, 0.f);
            unsigned rowmask = 0;
            if (BNPRO) {
                ps = __ldg(reinterpret_cast<const float2*>(c.pre_scale + ch));
                pb = __ldg(reinterpret_cast<const float2*>(c.pre_shift + ch));
                const int t = blockIdx.x + ti * gridDim.x;
                const int y0 = SP.fn > 1 ? 0 : ((t * TBM) / TW) % c.H;
#pragma unroll
                for (int r = 0; r < NR; ++r) {
                    const int iy = y0 + ry + r - PAD;
                    if (iy >= 0 && iy < c.H) rowmask |= 1u << r;
                }
            }

            if (!(DBG & 2)) mbar_wait_relaxed(pfull, (uint32_t)((j / NP) & 1), (DBG & 2048) ? 32u : 0u);
            // input rows are loaded one row ahead of their FMAs (two register rows, compile-time ping-pong); within
            // a row the FMAs go tap-column by tap-column over all (output row, output column) accumulators, so
            // consecutive FFMA2 never touch the same accumulator.  Each output's taps are summed in (ky, kx) order
            // whatever OR is, so both tile geometries compute the same depthwise values bit for bit.
            auto load_row = [&](int r, float2* in) {
#pragma unroll
                for (int q = 0; q < NC; ++q) {
                    float2 v = *reinterpret_cast<const float2*>(pbase + (r * PC + q) * SBK);
                    if (BNPRO) v = ffma2(v, ps, pb);
                    v = make_float2(fmaxf(v.x, lowb), fmaxf(v.y, lowb));
                    if (BNPRO && !(((rowmask >> r) & 1u) && ((colmask >> q) & 1u))) v = make_float2(0.f, 0.f);
                    in[q] = v;
                }
            };
            if (!(DBG & 1)) {
                float2 inb[2][NC];
                load_row(0, inb[0]);
#pragma unroll
                for (int r = 0; r < NR; ++r) {
                    if (r + 1 < NR) load_row(r + 1, inb[(r + 1) & 1]);
                    const float2* in = inb[r & 1];
#pragma unroll
                    for (int kx = 0; kx < KS; ++kx)
#pragma unroll
                        for (int o = 0; o < OR; ++o) {
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
            for (int o = 0; o < OR; ++o)
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
        // ============ consumers: wgmma + epilogue (ping-pong: warpgroup wg owns tiles ti = wg, wg + 2, ...) ============
        reg_inc<REGS_EPI>();
        stage_post<R::NEPI, bn_max(TBM)>(P, n0, post, tid - 32 * WARP_EPI0);
        const int wg = (warp - WARP_EPI0) >> 2, wt = tid - 32 * WARP_EPI0 - 128 * wg;
        const EpiSmem es{epi ? reinterpret_cast<float*>(epi_buf) : nullptr,
                         P.c.res1 ? reinterpret_cast<const float*>(epi_buf + EPI_BUF_BYTES) : nullptr, bar_epi_full0,
                         bar_epi_empty, &map_out};
        pp_consumer<SHARE, LO, NA, NB, TBM>(P, wg, wt, n0, tiles_mine, make_desc64(smem_u32(smem)), make_desc64(smem_u32(b_ring)),
                                       bar_full0, bar_empty0, bar_fullb0, bar_emptyb0, my_rank, post, DBG,
                                       es);
    } else {
        reg_dec<REGS_CTRL>();
        if (warp == WARP_TMA) {
            // ======================= weight tiles via TMA =======================
            if (lane == 0) {
                const uint32_t tx = (DBG & 16) ? 0u : (uint32_t)(want_lo ? 2 : 1) * (uint32_t)b_bytes;
                const uint32_t tx_a = (DBG & 8) ? 0u : (uint32_t)(want_lo ? 2 : 1) * (uint32_t)A_BYTES;
                for (int g = 0; g < total_g; ++g) {
                    const int ti = g / nkb, kb = g - ti * nkb;
                    const int sb = g % NB;
                    const uint32_t itb = (uint32_t)(g / NB);
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
                        // the peer produces this K-block: arm our fullA for the bytes it will push (our consumers
                        // have passed the previous use of the stage, so the barrier is in the right phase)
                        const int sa = g % NA;
                        wait_stage_free(bar_empty0, sa, (uint32_t)(g / NA));
                        mbar_arrive_expect_tx(bar_full0 + 8 * sa, tx_a);
                    }
                }
            }
        } else if (warp == WARP_TMA + 1) {
            // ============ residuals of the shared-memory epilogue via TMA (64-row tiles) ============
            // tile ti's boxes go into the buffer as soon as tile ti - 1's output has left it (normally early in tile
            // ti's mainloop); the up2x residual's source pixels of a 64-row tile are the 16 from m0 / 4 on
            if (lane == 0 && epi) {
                const ConvParams& c = P.c;
                const uint32_t tx = (DBG & 32) ? 0u
                                               : (c.res0 ? (uint32_t)EPI_BUF_BYTES : 0u) + (c.res1 ? (uint32_t)EPI_R1_BYTES : 0u);
                for (int ti = 0; ti < tiles_mine; ++ti) {
                    if (ti >= 1) mbar_wait_relaxed(bar_epi_empty, (uint32_t)((ti - 1) & 1), 0u);
                    const int m0 = ((int)blockIdx.x + ti * (int)gridDim.x) * TBM;
                    const uint32_t full = bar_epi_full0 + 8 * (ti & 1);
                    mbar_arrive_expect_tx(full, tx);
                    if (tx) {
                        if (c.res0) tma_load_2d(smem_u32(epi_buf), &map_r0, n0, m0, full);
                        if (c.res1) tma_load_2d(smem_u32(epi_buf + EPI_BUF_BYTES), &map_r1, n0, m0 / 4, full);
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
                    const int grow = (t * TBM) / TW;                // global row index (n*H + y) of the tile's first row
                    nf = grow / c.H;
                    y0 = grow - nf * c.H;
                };
                for (int j = 0; j < n_own; ++j) {
                    int kb, nf, y0;
                    coords(j, kb, nf, y0);
                    const int w = j % NP;
                    const int pfd = (DBG & 1024) ? 2 : (DBG & 4096) ? 4 : (DBG & 8192) ? 9 : 0;   // L2 prefetch distance (K-blocks)
                    if (pfd && j + pfd < n_own) {
                        int kb2, nf2, y2;
                        coords(j + pfd, kb2, nf2, y2);
                        tma_prefetch_4d(&map_x, kb2 * SBK, -PAD, y2 - PAD, nf2);
                    }
                    mbar_wait_relaxed(bar_pempty0 + 8 * w, (uint32_t)(((j / NP) & 1) ^ 1), (DBG & 2048) ? 64u : 0u);
                    const uint32_t pf = bar_pfull0 + 8 * w;
                    mbar_arrive_expect_tx(pf, (uint32_t)SP.patch_bytes);
                    tma_load_4d(smem_u32(patch0 + (size_t)w * SP.patch_stride), &map_x, kb * SBK, -PAD, y0 - PAD, nf, pf);
                }
            }
        }
    }
    if (SHARE) cluster_sync_all(); else __syncthreads();     // a peer's remote arrivals / copies target this CTA
}

}  // namespace tcs

// The TMA-staged kernel takes the separable layers of sep_layer_ok whose 128-row tiles are whole image rows (W = 32,
// 16, 8) and whose rings fit shared memory; everything else stays on conv_tc.cu's register-sliding producer.
//
// Tile geometry (DESIGN §4.1, measurements in §9): 64 x 144 where Cout splits into an even number of full 144-column
// N parts (Cout 272-288 or 544-576: one or two cluster pairs per pixel tile, so each depthwise K-block is computed
// once or twice per pixel instead of three times) and Cin >= 288, the layer class of the models, measured faster on
// every shape of it.  Everything else keeps 128 x 96.  The 64-row tile needs the pairs (share_a).
//
// Epilogue: a 64-row tile stages it in shared memory (residuals by TMA load, output by TMA store) when the driver can
// encode every view it touches (tma_view_ok: a concat slice may start at any channel) and the layer has no second
// full-resolution residual (no room for a second 36 KB box); else it keeps the register epilogue.
bool dh_plan_sep_tma(const dh_ctx* ctx, const ConvParams& p, const dh_packed_w* packed, int precision, tc::SepPlan* pl) {
    using namespace tc;
    using namespace tcs;
    if (!ctx->sep_tma || !packed->lo || !sep_layer_ok(p, packed)) return false;
    if (!(p.W == 32 || p.W == 16 || p.W == 8)) return false;
    const int tr = BM / p.W;
    if (tr <= p.H ? (p.H % tr) != 0 : (tr % p.H) != 0) return false;
    if ((p.Cin % SBK) != 0 || (p.ldx & 3)) return false;
    if ((int64_t)p.H * p.W * p.ldx * 4 >= (1ll << 40)) return false;              // TMA frame stride
    int bn64, gy64;
    tile_n(p.Cout, &bn64, &gy64, MAX_BN_CTA64);
    const bool fits64 = ctx->share_a && bn64 == MAX_BN_CTA64 && gy64 % 2 == 0;
    bool t64 = fits64 && p.Cin >= 288;
#ifdef DH_ABLATE
    if (ctx->dbg & DBG_TILE64) t64 = fits64;          // A/B timing of the two geometries in one build
    if (ctx->dbg & DBG_TILE128) t64 = false;
#endif
    SepParams& SP = pl->k;
    TcParams& P = SP.t;
    P.c = p;
    P.c.K = p.Cin;
    P.k_pad = packed->k;
    P.n_kblocks = p.Cin / SBK;
    P.precision = (precision == 1) ? 1 : 3;
    P.ks = p.kh;
    P.stages = 2;
    const int pad = p.kh / 2;
#ifdef DH_ABLATE
    SP.dbg = ctx->dbg;
    P.dbg = ctx->dbg;
#else
    SP.dbg = 0;
    P.dbg = 0;
#endif
    // the plan of one geometry; false when its rings do not fit shared memory
    auto geometry = [&](int bm) {
        int gy;
        tile_n(p.Cout, &P.bn_cta, &gy, bn_max(bm));
        const int trb = bm / p.W;                  // tile rows (BM64 / W also divides H: see the check above)
        SP.bm = bm;
        P.n_mtiles = (p.M + bm - 1) / bm;
        SP.ry = trb <= p.H ? trb : p.H;
        SP.fn = trb <= p.H ? 1 : trb / p.H;
        SP.patch_bytes = SBK * 4 * (p.W + 2 * pad) * (SP.ry + 2 * pad) * SP.fn;
        SP.patch_stride = (SP.patch_bytes + 1023) / 1024 * 1024;
        pl->smem = (size_t)NA * 2 * (bm * 64) + (size_t)NB * 2 * P.bn_cta * 64 + NP * (size_t)SP.patch_stride + 512 +
                   post_smem(bm);
        pl->gy = gy;
        return pl->smem <= SMEM_LIMIT;
    };
    SP.epi_smem = 0;
    if (!(t64 && geometry(BM64)) && !geometry(BM)) return false;
    bool epi = SP.bm == BM64 && tma_view_ok(p.out, p.ldo) && (!p.res0 || tma_view_ok(p.res0, p.ldr0)) &&
               (!p.res1 || (p.up1 && tma_view_ok(p.res1, p.ldr1)));
#ifdef DH_ABLATE
    if (ctx->dbg & DBG_EPI_REG) epi = false;
#endif
    const int epi_smem = EPI_BUF_BYTES + (p.res1 ? EPI_R1_BYTES : 0);
    if (epi && pl->smem + epi_smem <= SMEM_LIMIT) {
        SP.epi_smem = epi_smem;
        pl->smem += epi_smem;
    }
    pl->w = packed;
    pl->cluster = pl->gy % 2 == 0 && ctx->share_a;
    return true;
}

int dh_launch_sep_tma(const dh_ctx* ctx, const tc::SepPlan& pl, cudaStream_t s) {
    using namespace tc;
    using namespace tcs;
    const TcParams& P = pl.k.t;
    const ConvParams& c = P.c;
    const dh_packed_w* w = pl.w;
    const int pad = P.ks / 2;
    CUtensorMap map_hi, map_lo, map_x, map_out{}, map_r0{}, map_r1{};
    const bool epi = pl.k.epi_smem > 0;
    if (!make_map_w(&map_hi, w->hi, w->k, w->cout_pad, SBK, P.bn_cta) ||
        !make_map_w(&map_lo, w->lo, w->k, w->cout_pad, SBK, P.bn_cta) ||
        !make_map_x(&map_x, c.x, c.ldx, c.Cin, c.W, c.H, c.N, c.W + 2 * pad, pl.k.ry + 2 * pad, pl.k.fn) ||
        (epi && !make_map_rows(&map_out, c.out, c.Cout, c.M, c.ldo, MAX_BN_CTA64, BM64)) ||
        (epi && c.res0 && !make_map_rows(&map_r0, c.res0, c.Cout, c.M, c.ldr0, MAX_BN_CTA64, BM64)) ||
        (epi && c.res1 && !make_map_rows(&map_r1, c.res1, c.Cout, c.M / 4, c.ldr1, MAX_BN_CTA64, BM64 / 4))) {
        dh_set_error("dh_launch_sep_tma: cuTensorMapEncodeTiled failed");
        return -1;
    }
    return pick<5, 3>(P.ks, [&](auto ks) {
        return pick<32, 16, 8>(c.W, [&](auto tw) {
            return pick<true, false>(c.pre_scale != nullptr, [&](auto bnpro) {
                return pick<true, false>(P.precision == 3, [&](auto lo) {
                    if (pl.k.bm == BM64)          // 64-row tiles run as cluster pairs only
                        return launch_persistent<sep_tma_kernel<BM64, ks(), tw(), true, bnpro(), lo()>>(
                            "dh_launch_sep_tma", ctx, pl, P.n_mtiles, NTHREADS, s, map_hi, map_lo, map_x, map_out, map_r0, map_r1);
                    return pick<true, false>(pl.cluster, [&](auto share) {
                        return launch_persistent<sep_tma_kernel<BM, ks(), tw(), share(), bnpro(), lo()>>(
                            "dh_launch_sep_tma", ctx, pl, P.n_mtiles, NTHREADS, s, map_hi, map_lo, map_x, map_out, map_r0, map_r1);
                    });
                });
            });
        });
    });
}
