// Conv2D (1x1 and dense kxk, stride 1) on wgmma with a TMA-staged input patch.
//
// replaces: keras Conv2D(use_bias=False) (deephar/layers.py:66-71) with the BN / ReLU / add layers around it
// (layers.py:202-325): the stem convolutions (models/reception.py:61-98), the 1x1 convs of the hourglass
// (reception.py:101-131), RegMap (reception.py:145-153), and the 1x1 / 3x3 convs of the SPNet entry flow and
// residual units (models/spnet.py:317-352, models/common.py:25-67).
//
// Why a second dense kernel: conv_tc.cu gathers the im2col A tile global -> registers -> shared memory with
// one K-block of look-ahead; short-K layers (stem 3x3 convs: K = 288) and skinny ones (RegMap: N = 48) leave
// the SM with ~32 KB of loads in flight and run at 8-40 % of HBM.  Here the input travels the way the
// separable kernel's does (conv_sep.cu):
//   patch : per 128-pixel tile and 32-channel block, the zero-padded fp32 input window (tile rows + halo)
//           by ONE 4-D TMA into a ring of NP patch buffers (NP = whatever fits, up to 8: 64-200 KB in flight);
//   A     : per tap (ky, kx) the two producer warpgroups (alternating K-blocks) read the shifted window
//           from the patch (conflict-free LDS.128), apply the BN/ReLU prologue (padding positions masked to
//           zero AFTER the affine, as keras pads the activated tensor), split into bf16 hi/lo and store the
//           64B-swizzled K-major wgmma tile; global memory is read once per element, not once per tap;
//   W     : bf16 hi/lo weight tiles by 2-D TMA at K offset tap * Cin + 32 * cb;
//   D     : fp32 in the registers of two consumer warpgroups that take alternate tiles (ping-pong, as in
//           conv_sep.cu), three wgmma per k-step (bf16x3); epilogue shared with conv_tc.cu.
// 1x1 convolutions have no spatial structure: the pixel axis is viewed as rows of VW = 2^k <= 128 pixels
// ("virtual geometry") so any N*H*W works, including channel-sliced concat views.
// Roles: warps 0-3 / 4-7 producers, 8-15 consumers (wgmma + epilogue), 16 weight TMA, 18 patch TMA.
#include "tc_common.cuh"

namespace tcd {
using namespace tc;
using R = tc::Roles<2>;
constexpr int WARP_EPI0 = R::WARP_EPI0, WARP_TMA = R::WARP_TMA, WARP_PATCH = R::WARP_PATCH, NTHREADS = R::NTHREADS,
              REGS_PROD = R::REGS_PROD, REGS_EPI = R::REGS_EPI, REGS_CTRL = R::REGS_CTRL;

constexpr int NWG = 128;                   // threads per producer warpgroup
// A and weight ring depths.  The consumers keep one K-block's wgmmas in flight and release its stages one K-block
// late, so each ring is one K-block deeper than a drained pipe would need: the producers and the weight TMA still
// run two K-blocks ahead of the MMAs.
constexpr int NA = 4;                      // A-tile ring
constexpr int NB = 3;                      // weight ring
constexpr int MAX_NP = 8;                  // patch ring depth

template <bool LO>   // precision 3 (bf16x3), else 1
__global__ void __launch_bounds__(NTHREADS, 1)
patch_dense_kernel(const __grid_constant__ PatchParams PP, const __grid_constant__ CUtensorMap map_hi,
                   const __grid_constant__ CUtensorMap map_lo, const __grid_constant__ CUtensorMap map_x) {
    const TcParams& P = PP.t;
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    if (smem_u32(smem_raw) & 1023u) __trap();      // swizzled wgmma / TMA tiles need the 1024-byte alignment declared above
    uint8_t* smem = smem_raw;
    const int tid = threadIdx.x;
    const int warp = tid >> 5, lane = tid & 31;
    constexpr bool want_lo = LO;
    const int b_bytes = P.bn_cta * 64;                       // per (hi | lo)
    // smem: A ring [NA][hi | lo] | weight ring [NB][hi | lo] | patches [np] | barriers (512 B) | BN scale / shift
    uint8_t* b_ring = smem + NA * 2 * A_BYTES;
    uint8_t* patch0 = b_ring + NB * 2 * b_bytes;
    uint64_t* bars = reinterpret_cast<uint64_t*>(patch0 + (size_t)PP.np * PP.patch_stride);
    float* post = reinterpret_cast<float*>(bars + 64);
    // bars: fullA[NA] | emptyA[NA][2] | fullB[NB] | emptyB[NB] | pfull[MAX_NP] | pempty[MAX_NP]
    constexpr int NB_A = NA + 2 * NA;
    constexpr int NB_P = NB_A + 2 * NB;
    const uint32_t bar_full0 = smem_u32(bars), bar_empty0 = smem_u32(bars + NA), bar_fullb0 = smem_u32(bars + NB_A),
                   bar_emptyb0 = smem_u32(bars + NB_A + NB), bar_pfull0 = smem_u32(bars + NB_P),
                   bar_pempty0 = smem_u32(bars + NB_P + MAX_NP);
    const int n0 = blockIdx.y * P.bn_cta;
    const int nkb = P.n_kblocks;                              // = ncb * ntaps
    const int ntaps = PP.ntaps, ncb = PP.ncb, np = PP.np;

    if (warp == WARP_TMA && lane == 0) {
        tma_prefetch_desc(&map_hi);
        if (want_lo) tma_prefetch_desc(&map_lo);
        tma_prefetch_desc(&map_x);
        for (int s = 0; s < NA; ++s) {
            mbar_init(bar_full0 + 8 * s, (uint32_t)NWG);
            mbar_init(bar_empty0 + 16 * s, 1u);       // the consumer warpgroup that owns the K-block's tile
            mbar_init(bar_empty0 + 16 * s + 8, 1u);
        }
        for (int s = 0; s < NB; ++s) {
            mbar_init(bar_fullb0 + 8 * s, 1);
            mbar_init(bar_emptyb0 + 8 * s, 1);
        }
        for (int s = 0; s < MAX_NP; ++s) {
            mbar_init(bar_pfull0 + 8 * s, 1);
            // a patch is read by both producer warpgroups (alternating taps) unless it has a single tap
            mbar_init(bar_pempty0 + 8 * s, ntaps == 1 ? (uint32_t)NWG : (uint32_t)(2 * NWG));
        }
        fence_barrier_init();
    }
    __syncthreads();

    const int tiles_mine = ((int)P.n_mtiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;
    const int total_g = tiles_mine * nkb;       // K-blocks this CTA consumes: g = ((ti * ncb) + cb) * ntaps + tap
    const int n_patches = tiles_mine * ncb;
    const int rows_per_tile = BM / PP.tw;

    if (warp < WARP_EPI0) {
        // ======================= A producers (two warpgroups, alternating K-blocks) =======================
        reg_prod<REGS_PROD, R::LAUNCH_REGS>();
        const ConvParams& c = P.c;
        const int w = warp >> 2;
        const int tw = tid & (NWG - 1);
        const int ch4 = tw & 7;                          // 16-byte chunk (4 channels) of the 32-channel block
        const int prow = tw >> 3;                        // pixels prow + 16 i, i = 0..7
        uint32_t poff[8];
        int yy[8], xx[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int m = prow + 16 * i;
            const int ty = m / PP.tw, tx = m - ty * PP.tw;
            const int f = ty / PP.ry, r = ty - f * PP.ry;
            poff[i] = (uint32_t)(((f * PP.pr + r * PP.sh) * PP.pc + tx * PP.sw) * (SBK * 4) + ch4 * 16);
            yy[i] = r * PP.sh - PP.pt;
            xx[i] = tx * PP.sw - PP.pl;
        }
        const uint32_t patch_s = smem_u32(patch0);
        const bool relu = c.pre_relu != 0, has_bn = c.pre_scale != nullptr;
        uint32_t aoff[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) aoff[i] = swz64(prow + 16 * i, ch4 * 4);
        // K-block g = (patch p, tap): all indices are carried incrementally (g advances by 2 per iteration): this loop
        // is instruction-issue bound, and run-time integer divisions would be a third of it
        int tap = w % ntaps, p = w / ntaps;                   // ntaps >= 1, w in {0, 1}
        int cb = p % ncb, ti = p / ncb;
        int slot = p % np;
        uint32_t pphase = (uint32_t)(p / np) & 1u;
        int ky = tap / PP.kw, kx = tap - ky * PP.kw;
        int s = w % NA;
        uint32_t it = 0;
        int cb_loaded = -1, ti_masked = -1;
        float4 ps = make_float4(1.f, 1.f, 1.f, 1.f), pb = make_float4(0.f, 0.f, 0.f, 0.f);
        int y0 = 0;
        for (int g = w; g < total_g; g += 2) {
            // BN prologue vectors of this thread's 4 channels (channels past Cin: TMA zero fill must stay zero)
            if (has_bn && cb != cb_loaded) {
                cb_loaded = cb;
                const int ci = cb * SBK + ch4 * 4;
                if (ci < c.Cin) {
                    ps = __ldg(reinterpret_cast<const float4*>(c.pre_scale + ci));
                    pb = __ldg(reinterpret_cast<const float4*>(c.pre_shift + ci));
                } else {
                    ps = make_float4(0.f, 0.f, 0.f, 0.f);
                    pb = make_float4(0.f, 0.f, 0.f, 0.f);
                }
            }
            unsigned okmask = 0xffu;
            if (PP.mask) {
                if (ti != ti_masked) {
                    ti_masked = ti;
                    const int t = blockIdx.x + ti * gridDim.x;
                    y0 = PP.fn > 1 ? 0 : (t * rows_per_tile) % PP.rows_per_frame;
                }
                okmask = 0;
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    const int iy = y0 * PP.sh + yy[i] + ky, ix = xx[i] + kx;
                    if ((unsigned)iy < (unsigned)PP.vh && (unsigned)ix < (unsigned)PP.vw) okmask |= 1u << i;
                }
            }
            mbar_wait(bar_pfull0 + 8 * slot, pphase);
            const uint32_t base = patch_s + (uint32_t)slot * (uint32_t)PP.patch_stride +
                                  (uint32_t)((ky * PP.pc + kx) * (SBK * 4));
            float4 v[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) v[i] = lds128(base + poff[i]);

            wait_stage_free(bar_empty0, s, it);
            const uint32_t a_hi = smem_u32(smem) + (uint32_t)s * (2 * A_BYTES);
            const uint32_t a_lo = a_hi + A_BYTES;
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                float4 t4 = v[i];
                if (has_bn) {
                    t4.x = fmaf(t4.x, ps.x, pb.x); t4.y = fmaf(t4.y, ps.y, pb.y);
                    t4.z = fmaf(t4.z, ps.z, pb.z); t4.w = fmaf(t4.w, ps.w, pb.w);
                }
                if (relu) {
                    t4.x = fmaxf(t4.x, 0.f); t4.y = fmaxf(t4.y, 0.f); t4.z = fmaxf(t4.z, 0.f); t4.w = fmaxf(t4.w, 0.f);
                }
                if (!((okmask >> i) & 1u)) t4 = make_float4(0.f, 0.f, 0.f, 0.f);
                uint32_t h0, l0, h1, l1;
                split2(t4.x, t4.y, h0, l0);
                split2(t4.z, t4.w, h1, l1);
                asm volatile("st.shared.v2.b32 [%0], {%1, %2};" ::"r"(a_hi + aoff[i]), "r"(h0), "r"(h1) : "memory");
                if (want_lo) asm volatile("st.shared.v2.b32 [%0], {%1, %2};" ::"r"(a_lo + aoff[i]), "r"(l0), "r"(l1) : "memory");
            }
            const bool last_of_patch = tap + 2 >= ntaps;       // my last tap of this patch has been consumed
            if (last_of_patch) mbar_arrive(bar_pempty0 + 8 * slot);
            fence_proxy_async();
            mbar_arrive(bar_full0 + 8 * s);
            // advance (g += 2)
            s += 2;
            if (s >= NA) { s -= NA; ++it; }
            tap += 2;
            kx += 2;
            while (tap >= ntaps) {                              // next patch (at most twice: ntaps = 1)
                tap -= ntaps;
                ++p;
                if (++cb == ncb) { cb = 0; ++ti; }
                if (++slot == np) { slot = 0; pphase ^= 1u; }
                ky = 0; kx = tap;                               // tap in {0, 1} here
                if (kx >= PP.kw) { kx -= PP.kw; ky = 1; }       // kw = 1 (kh x 1 kernels): tap 1 = (ky 1, kx 0)
            }
            while (kx >= PP.kw) { kx -= PP.kw; ++ky; }
        }
    } else if (warp < WARP_TMA) {
        // ============ consumers: wgmma + epilogue (ping-pong: warpgroup wg owns tiles ti = wg, wg + 2, ...) ============
        reg_inc<REGS_EPI>();
        stage_post<R::NEPI>(P, n0, post, tid - 32 * WARP_EPI0);
        const int wg = (warp - WARP_EPI0) >> 2, wt = tid - 32 * WARP_EPI0 - 128 * wg;
        pp_consumer<false, LO, NA, NB>(P, wg, wt, n0, tiles_mine, make_desc64(smem_u32(smem)), make_desc64(smem_u32(b_ring)),
                                       bar_full0, bar_empty0, bar_fullb0, bar_emptyb0, 0u, post, 0);
    } else {
        reg_dec<REGS_CTRL>();
        if (warp == WARP_TMA) {
            // ======================= weight tiles via TMA =======================
            if (lane == 0) {
                const uint32_t tx = (uint32_t)(want_lo ? 2 : 1) * (uint32_t)b_bytes;
                for (int g = 0; g < total_g; ++g) {
                    const int p = g / ntaps, tap = g - p * ntaps;
                    const int cb = p % ncb;
                    const int kc = tap * P.c.Cin + cb * SBK;          // K offset of this block in the packed weights
                    const int sb = g % NB;
                    const uint32_t itb = (uint32_t)(g / NB);
                    if (itb >= 1) mbar_wait_relaxed(bar_emptyb0 + 8 * sb, (itb - 1) & 1, 0u);
                    const uint32_t full = bar_fullb0 + 8 * sb;
                    mbar_arrive_expect_tx(full, tx);
                    const uint32_t b_hi = smem_u32(b_ring + (size_t)sb * (2 * b_bytes));
                    const uint32_t b_lo = b_hi + (uint32_t)b_bytes;
                    tma_load_2d(b_hi, &map_hi, kc, n0, full);
                    if (want_lo) tma_load_2d(b_lo, &map_lo, kc, n0, full);
                }
            }
        } else if (warp == WARP_PATCH) {
            // ======================= input patches via 4-D TMA =======================
            if (lane == 0) {
                for (int p = 0; p < n_patches; ++p) {
                    const int ti = p / ncb, cb = p - ti * ncb;
                    const int t = blockIdx.x + ti * gridDim.x;
                    const int grow = t * rows_per_tile;               // global output row index of the tile's first row
                    const int nf = grow / PP.rows_per_frame;
                    const int y0 = grow - nf * PP.rows_per_frame;
                    const int slot = p % np;
                    const uint32_t u = (uint32_t)(p / np);
                    mbar_wait_relaxed(bar_pempty0 + 8 * slot, (u & 1u) ^ 1u, 0u);
                    const uint32_t pf = bar_pfull0 + 8 * slot;
                    mbar_arrive_expect_tx(pf, (uint32_t)PP.patch_bytes);
                    tma_load_4d(smem_u32(patch0 + (size_t)slot * PP.patch_stride), &map_x, cb * SBK, -PP.pl,
                                y0 * PP.sh - PP.pt, nf, pf);
                }
            }
        }
    }
}

// geometry of the patch for a conv (real for kxk, virtual rows of 2^k pixels for 1x1)
static bool plan_geom(const ConvParams& p, PatchParams* g) {
    if (p.sh != 1 || p.sw != 1) return false;
    if (p.kh == 1 && p.kw == 1) {
        // flat pixel axis viewed as rows of vw pixels (vw | H*W so that frames never straddle a partial row); the
        // whole batch is one virtual frame of vh rows
        const int64_t hw = (int64_t)p.H * p.W;
        int vw = 128;
        while (vw > 1 && (hw % vw) != 0) vw >>= 1;
        if (vw < 8) return false;
        g->tw = vw; g->ry = tc::BM / vw; g->fn = 1; g->pc = vw; g->pr = g->ry;
        g->vw = vw; g->vh = (int)(((int64_t)p.N * hw) / vw);
        g->rows_per_frame = g->vh; g->pt = g->pl = 0; g->kw = 1; g->ntaps = 1;
        return true;
    }
    if (p.Ho != p.H || p.Wo != p.W) return false;                       // SAME, stride 1
    if (!(p.W == 128 || p.W == 64 || p.W == 32 || p.W == 16 || p.W == 8)) return false;
    const int tr = tc::BM / p.W;
    if (tr <= p.H ? (p.H % tr) != 0 : (tr % p.H) != 0) return false;
    g->tw = p.W;
    g->ry = tr <= p.H ? tr : p.H;
    g->fn = tr <= p.H ? 1 : tr / p.H;
    g->pc = p.W + p.kw - 1;
    g->pr = g->ry + p.kh - 1;
    g->rows_per_frame = p.H; g->vh = p.H; g->vw = p.W;
    g->pt = p.pt; g->pl = p.pl; g->kw = p.kw; g->ntaps = p.kh * p.kw;
    return true;
}

}  // namespace tcd

bool dh_plan_patch(const dh_ctx* ctx, const ConvParams& p, const dh_packed_w* packed, int precision, tc::PatchPlan* pl) {
    using namespace tc;
    using namespace tcd;
    if (!ctx->dense_patch || !packed->lo) return false;
    if (p.M < 1) return false;
    if ((p.Cin & 7) || (p.ldx & 3) || (reinterpret_cast<uintptr_t>(p.x) & 15) || !bn_pro_aligned(p)) return false;
    if (!packed_fits(packed, p.kh * p.kw * p.Cin, p.Cout)) return false;
    PatchParams& PP = pl->k;
    if (!plan_geom(p, &PP)) return false;
    if (PP.pc > 256 || PP.pr > 256 || PP.fn > 256) return false;                  // TMA box dimensions
    if ((int64_t)PP.vh * PP.vw * p.ldx * 4 >= (1ll << 40)) return false;          // TMA frame stride
    TcParams& P = PP.t;
    P.c = p;
    P.c.K = p.kh * p.kw * p.Cin;
    P.k_pad = packed->k;
    PP.ncb = (p.Cin + SBK - 1) / SBK;
    P.n_kblocks = PP.ncb * PP.ntaps;
    int gy;
    tile_n(p.Cout, &P.bn_cta, &gy);
    P.precision = (precision == 1) ? 1 : 3;
    P.ks = 0;
    P.n_mtiles = (p.M + BM - 1) / BM;
    P.stages = 2;
    P.dbg = 0;
    PP.sh = 1; PP.sw = 1;
    PP.mask = (p.pre_scale != nullptr && PP.ntaps > 1) ? 1 : 0;
    PP.patch_bytes = SBK * 4 * PP.pc * PP.pr * PP.fn;
    PP.patch_stride = (PP.patch_bytes + 1023) / 1024 * 1024;
    // A and weight rings, barriers, BN scale / shift; patches in what is left, at least two
    const size_t fixed = (size_t)NA * 2 * A_BYTES + (size_t)NB * 2 * P.bn_cta * 64 + 512 + POST_SMEM;
    const int np = (int)((SMEM_LIMIT - fixed) / (size_t)PP.patch_stride);
    if (np < 2) return false;
    PP.np = np > MAX_NP ? MAX_NP : np;
    pl->w = packed;
    pl->gy = gy;
    pl->smem = fixed + (size_t)PP.np * PP.patch_stride;
    pl->cluster = false;
    return true;
}

int dh_launch_patch(const dh_ctx* ctx, const tc::PatchPlan& pl, cudaStream_t s) {
    using namespace tc;
    using namespace tcd;
    const PatchParams& PP = pl.k;
    const ConvParams& c = PP.t.c;
    const dh_packed_w* w = pl.w;
    const int vn = PP.ntaps == 1 ? 1 : c.N;            // a 1x1 conv's virtual geometry is one frame (plan_geom)
    CUtensorMap map_hi, map_lo, map_x;
    if (!make_map_w(&map_hi, w->hi, w->k, w->cout_pad, SBK, PP.t.bn_cta) ||
        !make_map_w(&map_lo, w->lo, w->k, w->cout_pad, SBK, PP.t.bn_cta) ||
        !make_map_x(&map_x, c.x, c.ldx, c.Cin, PP.vw, PP.vh, vn, PP.pc, PP.pr, PP.fn)) {
        dh_set_error("dh_launch_patch: cuTensorMapEncodeTiled failed");
        return -1;
    }
    return pick<true, false>(PP.t.precision == 3, [&](auto lo) {
        return launch_persistent<patch_dense_kernel<lo()>>("dh_launch_patch", ctx, pl, PP.t.n_mtiles, NTHREADS, s,
                                                           map_hi, map_lo, map_x);
    });
}
