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
//   D     : fp32 in the registers of two consumer warpgroups (rows 0-63 / 64-127), three wgmma per k-step
//           (bf16x3); epilogue shared with conv_tc.cu.
// 1x1 convolutions have no spatial structure: the pixel axis is viewed as rows of VW = 2^k <= 128 pixels
// ("virtual geometry") so any N*H*W works, including channel-sliced concat views.
// Roles: warps 0-3 / 4-7 producers, 8-15 consumers (wgmma + epilogue), 16 weight TMA, 18 patch TMA.
#include "tc_common.cuh"

namespace tcd {
using namespace tc;
using R = tc::Roles<2>;
constexpr int WARP_EPI0 = R::WARP_EPI0, WARP_TMA = R::WARP_TMA, WARP_PATCH = R::WARP_PATCH, NTHREADS = R::NTHREADS,
              REGS_PROD = R::REGS_PROD, REGS_EPI = R::REGS_EPI, REGS_CTRL = R::REGS_CTRL;

constexpr int A_BYTES = BM * 64;           // 8 KB per (hi | lo): 128 rows x 32 bf16
constexpr int NWG = 128;                   // threads per producer warpgroup
constexpr int NA = 3;                      // A-tile ring depth
constexpr int MAX_NP = 8;                  // patch ring depth

struct PatchParams {
    TcParams t;
    int np, patch_stride, patch_bytes;
    int ntaps, ncb;          // kh * kw ; ceil(Cin / 32)
    int tw;                  // tile width (output pixels per tile row)
    int ry, fn;              // output rows per frame per tile, frames per tile
    int pc, pr;              // patch columns, patch rows per frame
    int rows_per_frame;      // output rows per frame (tile -> frame / row decode)
    int kw;                  // taps per kernel row
    int pt, pl, sh, sw;      // padding before, strides
    int vh, vw;              // input height / width (for the prologue mask)
    int mask;                // 1 = BN prologue on a padded conv: out-of-image taps must be forced to zero
};

__global__ void __launch_bounds__(NTHREADS, 1)
patch_dense_kernel(const __grid_constant__ PatchParams PP, const __grid_constant__ CUtensorMap map_hi,
                   const __grid_constant__ CUtensorMap map_lo, const __grid_constant__ CUtensorMap map_x) {
    const TcParams& P = PP.t;
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    if (smem_u32(smem_raw) & 1023u) __trap();      // swizzled wgmma / TMA tiles need the 1024-byte alignment declared above
    uint8_t* smem = smem_raw;
    const int tid = threadIdx.x;
    const int warp = tid >> 5, lane = tid & 31;
    const bool want_lo = P.precision == 3;
    const int b_bytes = P.bn_cta * 64;                       // per (hi | lo)
    // smem: A ring [NA][hi | lo] | weight ring [2][hi | lo] | patches [np] | barriers
    uint8_t* b_ring = smem + NA * 2 * A_BYTES;
    uint8_t* patch0 = b_ring + 2 * 2 * b_bytes;
    uint64_t* bars = reinterpret_cast<uint64_t*>(patch0 + (size_t)PP.np * PP.patch_stride);
    // bars: fullA[NA] | emptyA[NA][2] | fullB[2] | emptyB[2] | pfull[MAX_NP] | pempty[MAX_NP]
    constexpr int NB_A = NA + 2 * NA;
    constexpr int NB_P = NB_A + 4;
    const uint32_t bar_full0 = smem_u32(bars), bar_empty0 = smem_u32(bars + NA), bar_fullb0 = smem_u32(bars + NB_A),
                   bar_emptyb0 = smem_u32(bars + NB_A + 2), bar_pfull0 = smem_u32(bars + NB_P),
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
            mbar_init(bar_empty0 + 16 * s, (uint32_t)R::EPQ);       // one arrival per consumer warpgroup
            mbar_init(bar_empty0 + 16 * s + 8, (uint32_t)R::EPQ);
        }
        for (int s = 0; s < 2; ++s) {
            mbar_init(bar_fullb0 + 8 * s, 1);
            mbar_init(bar_emptyb0 + 8 * s, R::EPQ);
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
            if (s >= 1) { s -= 1; it += 1; } else { s += 2; }
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
                mbar_wait(bar_full0 + 8 * s, it & 1);
                mbar_wait(bar_fullb0 + 8 * sb, (uint32_t)(g >> 1) & 1);
                wg_kblock<R::MH, SBK / 16>(P.bn_cta, acc, dbase + (uint64_t)((uint32_t)s * sta16), 0u, alo16,
                                           dbase_b + (uint64_t)((uint32_t)sb * stb16), blo16, want_lo, kb == 0);
                wg_release<false>(bar_empty0 + 16 * s + 8 * (it & 1), wg, wt, 0u);
                if (wt == 0) mbar_arrive(bar_emptyb0 + 8 * sb);
            }
            wg_epilogue<R::MH>(P, acc, ((int)blockIdx.x + ti * (int)gridDim.x) * BM + 64 * wg, n0, wt);
        }
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
                    const int sb = g & 1;
                    const uint32_t itb = (uint32_t)(g >> 1);
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
struct Geom {
    int tw, ry, fn, pc, pr, rows_per_frame, vh, vw, vn, pt, pl, kw, ntaps;
    int64_t w_stride, h_stride, n_stride;     // bytes
};

static bool plan_geom(const ConvParams& p, Geom* g) {
    if (p.sh != 1 || p.sw != 1) return false;
    if (p.kh == 1 && p.kw == 1) {
        // flat pixel axis viewed as rows of vw pixels (vw | H*W so that frames never straddle a partial row)
        const int64_t hw = (int64_t)p.H * p.W;
        int vw = 128;
        while (vw > 1 && (hw % vw) != 0) vw >>= 1;
        if (vw < 8) return false;
        g->tw = vw; g->ry = tc::BM / vw; g->fn = 1; g->pc = vw; g->pr = g->ry;
        g->vw = vw; g->vh = (int)(((int64_t)p.N * hw) / vw); g->vn = 1;
        g->rows_per_frame = g->vh; g->pt = g->pl = 0; g->kw = 1; g->ntaps = 1;
        g->w_stride = (int64_t)p.ldx * 4; g->h_stride = (int64_t)vw * p.ldx * 4;
        g->n_stride = (int64_t)g->vh * g->h_stride;
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
    g->rows_per_frame = p.H; g->vh = p.H; g->vw = p.W; g->vn = p.N;
    g->pt = p.pt; g->pl = p.pl; g->kw = p.kw; g->ntaps = p.kh * p.kw;
    g->w_stride = (int64_t)p.ldx * 4; g->h_stride = (int64_t)p.W * p.ldx * 4; g->n_stride = (int64_t)p.H * g->h_stride;
    return true;
}

static size_t fixed_smem(int bn_cta) {
    return (size_t)NA * 2 * A_BYTES + (size_t)2 * 2 * bn_cta * 64 + 512;
}

}  // namespace tcd

bool dh_patch_supported(const dh_ctx* ctx, const ConvParams& p, const dh_packed_w* packed) {
    using namespace tcd;
    if (!ctx->dense_patch) return false;
    if (!packed || !packed->hi || !packed->lo) return false;
    if (p.M < 1) return false;
    if ((p.Cin & 7) || (p.ldx & 3) || (reinterpret_cast<uintptr_t>(p.x) & 15)) return false;
    if (p.pre_scale && ((reinterpret_cast<uintptr_t>(p.pre_scale) & 15) || (reinterpret_cast<uintptr_t>(p.pre_shift) & 15)))
        return false;
    const int K = p.kh * p.kw * p.Cin;
    if (packed->k != dh_tc_k_pad(K) || packed->cout_pad != dh_tc_cout_pad(p.Cout)) return false;
    Geom g;
    if (!plan_geom(p, &g)) return false;
    if (g.pc > 256 || g.pr > 256 || g.fn > 256) return false;
    int bn_cta, gy;
    tc::tile_n(p.Cout, &bn_cta, &gy);
    const size_t patch = (size_t)tc::SBK * 4 * g.pc * g.pr * g.fn;
    const size_t stride = (patch + 1023) / 1024 * 1024;
    if (fixed_smem(bn_cta) + 2 * stride > 227 * 1024) return false;
    if ((g.w_stride & 15) || g.n_stride >= (1ll << 40)) return false;
    return true;
}

int dh_launch_patch(dh_ctx* ctx, const ConvParams& p, const dh_packed_w* packed, int precision, cudaStream_t s) {
    using namespace tc;
    using namespace tcd;
    PatchParams PP;
    TcParams& P = PP.t;
    Geom g;
    if (!plan_geom(p, &g)) {
        dh_set_error("dh_launch_patch: unsupported geometry");
        return -1;
    }
    P.c = p;
    P.c.K = p.kh * p.kw * p.Cin;
    P.k_pad = packed->k;
    PP.ntaps = g.ntaps;
    PP.ncb = (p.Cin + SBK - 1) / SBK;
    P.n_kblocks = PP.ncb * PP.ntaps;
    int gy;
    tile_n(p.Cout, &P.bn_cta, &gy);
    P.precision = (precision == 1) ? 1 : 3;
    P.ks = 0;
    P.n_mtiles = (p.M + BM - 1) / BM;
    P.stages = 2;
    P.dbg = 0;
    PP.tw = g.tw; PP.ry = g.ry; PP.fn = g.fn; PP.pc = g.pc; PP.pr = g.pr; PP.rows_per_frame = g.rows_per_frame;
    PP.kw = g.kw; PP.pt = g.pt; PP.pl = g.pl; PP.sh = 1; PP.sw = 1; PP.vh = g.vh; PP.vw = g.vw;
    PP.mask = (p.pre_scale != nullptr && g.ntaps > 1) ? 1 : 0;
    PP.patch_bytes = SBK * 4 * g.pc * g.pr * g.fn;
    PP.patch_stride = (PP.patch_bytes + 1023) / 1024 * 1024;
    const size_t fixed = fixed_smem(P.bn_cta);
    int np = (int)((227 * 1024 - fixed) / (size_t)PP.patch_stride);
    if (np > MAX_NP) np = MAX_NP;
    if (np < 2) {
        dh_set_error("dh_launch_patch: patch does not fit shared memory");
        return -1;
    }
    PP.np = np;
    const size_t smem = fixed + (size_t)np * PP.patch_stride;

    CUtensorMap map_hi, map_lo, map_x;
    EncodeTiledFn enc = get_encode();
    bool ok = enc && make_map_b64(&map_hi, packed->hi, packed->k, packed->cout_pad, P.bn_cta) &&
              make_map_b64(&map_lo, packed->lo, packed->k, packed->cout_pad, P.bn_cta);
    if (ok) {
        cuuint64_t dims[4] = {(cuuint64_t)p.Cin, (cuuint64_t)g.vw, (cuuint64_t)g.vh, (cuuint64_t)g.vn};
        cuuint64_t strides[3] = {(cuuint64_t)g.w_stride, (cuuint64_t)g.h_stride, (cuuint64_t)g.n_stride};
        cuuint32_t box[4] = {(cuuint32_t)SBK, (cuuint32_t)g.pc, (cuuint32_t)g.pr, (cuuint32_t)g.fn};
        cuuint32_t estr[4] = {1, 1, 1, 1};
        ok = enc(&map_x, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, const_cast<float*>(p.x), dims, strides, box, estr,
                 CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                 CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
    }
    if (!ok) {
        dh_set_error("dh_launch_patch: cuTensorMapEncodeTiled failed");
        return -1;
    }
    int gx = ctx->num_sms / gy;
    if (gx < 1) gx = 1;
    if (gx > P.n_mtiles) gx = P.n_mtiles;
    cudaError_t e = ensure_smem<patch_dense_kernel>(smem);
    if (e == cudaSuccess) {
        patch_dense_kernel<<<dim3(gx, gy), NTHREADS, smem, s>>>(PP, map_hi, map_lo, map_x);
    } else {
        dh_set_error("dh_launch_patch: launch setup failed: %s", cudaGetErrorString(e));
        return (int)e;
    }
    return 0;
}
