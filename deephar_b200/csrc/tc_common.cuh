// Shared pieces of the wgmma convolution kernels (conv_tc.cu, conv_sep.cu, conv_patch.cu): constants, launch
// parameters, PTX wrappers (mbarrier, TMA, wgmma, cluster/DSMEM, setmaxnreg), shared-memory matrix descriptors,
// the bf16 hi/lo split, the consumer warpgroups (wgmma issue + fused epilogue) and the host-side tensor-map /
// N-tiling helpers.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include "common.cuh"
#include "conv_params.cuh"

namespace tc {


constexpr int BM = 128;
constexpr int BK = 64;                 // bf16 per K-block = one 128-byte swizzle row
constexpr int NPROD = 256;             // A producers: warps 0..7 (two warpgroups)
// Columns (output channels) per CTA.  The fp32 accumulators of a 128 x MAX_BN_CTA tile live in the registers of
// the consumer warpgroups (Hopper has no tensor memory): 96 per thread with one consumer warpgroup (conv_tc.cu),
// 48 with two.  Wider layers are split over gridDim.y.
constexpr int MAX_BN_CTA = 96;
constexpr int ACC_N = MAX_BN_CTA / 2;  // fp32 accumulator registers per thread per m64 slice
// Warp roles: producers (NPW warpgroups) | consumers (Q warpgroups: wgmma issue, then the fused epilogue from
// the accumulator registers) | one control warpgroup (weight TMA, patch TMA, two spare warps).  With Q = 1 the
// consumer warpgroup owns both 64-row halves of the 128-pixel tile; with Q = 2 warpgroup h owns rows 64 h .. + 63.
// Register budget (setmaxnreg; ptxas allocates each role's code against its own value):
//   Q = 1: 512 threads launch with 128 registers: 256 * 168 + 128 * 144 + 128 * 32 = 65536
//   Q = 2, NPW = 1 (conv_sep.cu): 512 threads launch with 128: ONE producer warpgroup with 192 registers (the 5x5
//          depthwise keeps 25 tap pairs + 16 accumulator pairs + an input row in registers: ~115, and it spills
//          below that), 128 * 192 + 256 * 144 + 128 * 32 = 65536.
//   Q = 2, NPW = 2 (conv_patch.cu): 640 threads launch with 96 (65536 / 640 rounded down to the allocation unit).  setmaxnreg only
//          redistributes the CTA's OWN allocation, 640 * 96 = 61440 registers (asking for more blocks forever):
//          producers drop to 80 (the TMA-staged producers fit), control to 32, the consumers grow to 144:
//          256 * 80 + 256 * 144 + 128 * 32 = 61440.
template <int Q, int NPW = 2>
struct Roles {
    static constexpr int EPQ = Q;                           // consumer warpgroups
    static constexpr int MH = 2 / Q;                        // 64-row halves per consumer warpgroup
    static constexpr int NEPI = 128 * Q;
    static constexpr int WARP_EPI0 = 4 * NPW;               // first consumer warp
    static constexpr int WARP_TMA = WARP_EPI0 + 4 * Q, WARP_PATCH = WARP_TMA + 2;
    static constexpr int NTHREADS = 32 * (WARP_TMA + 4);
    static constexpr int REGS_PROD = Q == 1 ? 168 : (NPW == 1 ? 192 : 80), REGS_EPI = 144, REGS_CTRL = 32;
    static constexpr int LAUNCH_REGS = NTHREADS <= 512 ? 128 : 96;      // what ptxas reports for __launch_bounds__(NTHREADS, 1)
    static_assert(128 * NPW * REGS_PROD + NEPI * REGS_EPI + 128 * REGS_CTRL <= NTHREADS * LAUNCH_REGS,
                  "setmaxnreg budget exceeds the CTA's register allocation: the last setmaxnreg.inc would never return");
};
constexpr int A_TILE_BYTES = BM * 128; // 16 KB per (hi | lo)
constexpr int MAX_STAGES = 4;

struct TcParams {
    ConvParams c;
    int n_kblocks;
    int bn_cta;             // output channels per CTA = wgmma N (multiple of 16, <= MAX_BN_CTA)
    int stages;
    int precision;          // 1 | 3
    int ks;                 // separable: depthwise kernel size (3 | 5); 0 = dense
    int k_pad;
    int n_mtiles;           // ceil(M / 128); CTA (x, y) loops over tiles x, x + gridDim.x, ...
    int dbg;                // `make ABLATE=1` builds only: 32 = epilogue touches no global memory
};

// ---------------------------------------------------------------------------
// PTX wrappers
// ---------------------------------------------------------------------------
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
// same, for waits that are expected to be long (not on the MMA-issue critical path): sleep between polls so
// that the spinning warp does not take issue slots from the warps doing the work
__device__ __forceinline__ void mbar_wait_relaxed(uint32_t bar, uint32_t parity, uint32_t ns) {
    uint32_t ok;
    for (;;) {
        asm volatile(
            "{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n selp.u32 %0, 1, 0, p;\n}"
            : "=r"(ok)
            : "r"(bar), "r"(parity)
            : "memory");
        if (ok) break;
        if (ns) __nanosleep(ns);
    }
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, int c0, int c1, uint32_t bar) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
        ::"r"(dst), "l"(map), "r"(c0), "r"(c1), "r"(bar)
        : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory");
}
// ---- 2-CTA cluster helpers (A-tile sharing between the two N-part CTAs of one pixel tile) ----
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
// local shared memory -> peer CTA's shared memory, completion counted on the PEER's mbarrier
__device__ __forceinline__ void bulk_s2peer(uint32_t dst_cluster, uint32_t src_cta, uint32_t bytes, uint32_t bar_cluster) {
    asm volatile("cp.async.bulk.shared::cluster.shared::cta.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(dst_cluster), "r"(src_cta), "r"(bytes), "r"(bar_cluster)
                 : "memory");
}
template <int R> __device__ __forceinline__ void reg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R> __device__ __forceinline__ void reg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
// producers: grow (Q = 1) or shrink (Q = 2) from the launch register count to the role's budget
template <int R, int LAUNCH> __device__ __forceinline__ void reg_prod() {
    if constexpr (R > LAUNCH) reg_inc<R>();
    else if constexpr (R < LAUNCH) reg_dec<R>();
}
// local mbarrier arrive on the same offset in the peer CTA of a cluster pair
__device__ __forceinline__ void mbar_arrive_cluster(uint32_t bar_cluster) {
    asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(bar_cluster) : "memory");
}

// ---- wgmma: D[64 x N] (+)= A[64 x 16, smem desc] * B[N x 16, smem desc]^T, bf16 x bf16 -> fp32 registers ----
// Accumulator fragment of thread t of the warpgroup: d[4 j + 2 h + e] = D[16 (t / 32) + (t % 32) / 4 + 8 h][8 j + 2 (t % 4) + e]
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator accesses across wgmma_fence / wgmma_wait
__device__ __forceinline__ void acc_fence(float& r) { asm volatile("" : "+f"(r)::"memory"); }
template <int N> __device__ __forceinline__ void wgmma_bf16(float* d, uint64_t a, uint64_t b, uint32_t acc);
template <> __device__ __forceinline__ void wgmma_bf16<16>(float* d, uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile(
        "{\n .reg .pred p;\n setp.ne.b32 p, %10, 0;\n"
        " wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, 0, 0;\n}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "l"(a), "l"(b), "r"(acc));
}
template <> __device__ __forceinline__ void wgmma_bf16<32>(float* d, uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile(
        "{\n .reg .pred p;\n setp.ne.b32 p, %18, 0;\n"
        " wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(a), "l"(b), "r"(acc));
}
template <> __device__ __forceinline__ void wgmma_bf16<48>(float* d, uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile(
        "{\n .reg .pred p;\n setp.ne.b32 p, %26, 0;\n"
        " wgmma.mma_async.sync.aligned.m64n48k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23}, %24, %25, p, 1, 1, 0, 0;\n}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23])
        : "l"(a), "l"(b), "r"(acc));
}
template <> __device__ __forceinline__ void wgmma_bf16<64>(float* d, uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile(
        "{\n .reg .pred p;\n setp.ne.b32 p, %34, 0;\n"
        " wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(a), "l"(b), "r"(acc));
}
template <> __device__ __forceinline__ void wgmma_bf16<80>(float* d, uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile(
        "{\n .reg .pred p;\n setp.ne.b32 p, %42, 0;\n"
        " wgmma.mma_async.sync.aligned.m64n80k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39}, %40, %41, p, 1, 1, 0, 0;\n}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39])
        : "l"(a), "l"(b), "r"(acc));
}
template <> __device__ __forceinline__ void wgmma_bf16<96>(float* d, uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile(
        "{\n .reg .pred p;\n setp.ne.b32 p, %50, 0;\n"
        " wgmma.mma_async.sync.aligned.m64n96k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47}, %48, %49, p, 1, 1, 0, 0;\n}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47])
        : "l"(a), "l"(b), "r"(acc));
}

// K-major, 128-byte swizzle wgmma shared-memory descriptor: start>>4 [0,14) | LBO>>4 [16,30) (unused for
// swizzled K-major, 1) | SBO>>4 [32,46) = 1024 B (8 rows x 128 B per swizzle atom) | layout SWIZZLE_128B = 1 [62,64).
__device__ __forceinline__ uint64_t make_desc(uint32_t smem_addr) {
    return (uint64_t)((smem_addr >> 4) & 0x3FFF) | (1ull << 16) | ((uint64_t)(1024 >> 4) << 32) | (1ull << 62);
}


// fp32 -> (hi, lo) bf16 split, round-to-nearest-even: x ~= hi + lo to ~16 mantissa bits.
__device__ __forceinline__ void split2(float a, float b, uint32_t& hi, uint32_t& lo) {
    __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
    float ra = a - __low2float(h), rb = b - __high2float(h);
    __nv_bfloat162 l = __floats2bfloat162_rn(ra, rb);
    hi = *reinterpret_cast<uint32_t*>(&h);
    lo = *reinterpret_cast<uint32_t*>(&l);
}

// byte offset of element (row, k) inside a [rows][64 bf16] 128B-swizzled K-major tile
__device__ __forceinline__ uint32_t swz(int row, int k) {
    return (uint32_t)(row * 128 + ((((k >> 3) ^ (row & 7)) << 4) | ((k & 7) << 1)));
}


// ---- pieces shared by the patch-staged kernels (conv_sep.cu, conv_patch.cu): 32-channel K-blocks, 64B swizzle ----
constexpr int SBK = 32;                    // channels (bf16 K elements) per K-block = one 64-byte swizzle row
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* map, int c0, int c1, int c2, int c3,
                                            uint32_t bar) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5}], [%6];"
        ::"r"(dst), "l"(map), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(bar)
        : "memory");
}

__device__ __forceinline__ void tma_prefetch_4d(const CUtensorMap* map, int c0, int c1, int c2, int c3) {
    asm volatile("cp.async.bulk.prefetch.tensor.4d.L2.global [%0, {%1, %2, %3, %4}];"
                 ::"l"(map), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}

// K-major, 64-byte swizzle wgmma descriptor: SBO = 512 B (8 rows x 64 B), layout SWIZZLE_64B = 2.
__device__ __forceinline__ uint64_t make_desc64(uint32_t smem_addr) {
    return (uint64_t)((smem_addr >> 4) & 0x3FFF) | (1ull << 16) | ((uint64_t)(512 >> 4) << 32) | (2ull << 62);
}
// byte offset of element (row, k) inside a [rows][32 bf16] 64B-swizzled K-major tile (Swizzle<2,4,3>)
__device__ __forceinline__ uint32_t swz64(int row, int k) {
    return (uint32_t)(row * 64 + ((((k >> 3) ^ ((row >> 1) & 3)) << 4) | ((k & 7) << 1)));
}

__device__ __forceinline__ float4 lds128(uint32_t a) {
    float4 v;
    asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(a) : "memory");
    return v;
}

// use `it` (0,1,2,...) of stage s may start once use it-1 has been consumed
__device__ __forceinline__ void wait_stage_free(uint32_t bar_empty0, int s, uint32_t it, uint32_t ns = 0) {
    if (it >= 1) mbar_wait_relaxed(bar_empty0 + 16 * s + 8 * ((it - 1) & 1), ((it - 1) >> 1) & 1, ns);
}


// ---------------------------------------------------------------------------
// consumer warpgroups: wgmma issue + fused epilogue
// ---------------------------------------------------------------------------
// One K-block: NK16 k-steps of 16, MH 64-row slices of A (slice stride a_half16 in descriptor units of 16 B),
// hi*hi (+ lo*hi + hi*lo at precision 3) accumulated in fp32 registers.  Returns when the wgmmas have completed,
// so the caller may release the shared-memory stage.
template <int N, int MH, int NK16>
__device__ __forceinline__ void wg_kblock_n(float (&acc)[MH][ACC_N], uint64_t da, uint32_t a_half16, uint32_t alo16,
                                            uint64_t db, uint32_t blo16, bool want_lo, bool first) {
#pragma unroll
    for (int h = 0; h < MH; ++h)
#pragma unroll
        for (int i = 0; i < N / 2; ++i) acc_fence(acc[h][i]);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < NK16; ++k) {
        const uint32_t acc0 = (first && k == 0) ? 0u : 1u;
#pragma unroll
        for (int h = 0; h < MH; ++h) {
            const uint64_t a = da + (uint64_t)(h * a_half16 + 2 * k);
            wgmma_bf16<N>(acc[h], a, db + 2 * k, acc0);
            if (want_lo) {
                wgmma_bf16<N>(acc[h], a + alo16, db + 2 * k, 1u);
                wgmma_bf16<N>(acc[h], a, db + blo16 + 2 * k, 1u);
            }
        }
    }
    wgmma_commit();
    wgmma_wait<0>();
#pragma unroll
    for (int h = 0; h < MH; ++h)
#pragma unroll
        for (int i = 0; i < N / 2; ++i) acc_fence(acc[h][i]);
}

// wgmma N is an immediate: one instantiation per tile width bn_cta (16 .. MAX_BN_CTA, step 16)
template <int MH, int NK16>
__device__ __forceinline__ void wg_kblock(int bn, float (&acc)[MH][ACC_N], uint64_t da, uint32_t a_half16, uint32_t alo16,
                                          uint64_t db, uint32_t blo16, bool want_lo, bool first) {
    switch (bn) {
    case 16: wg_kblock_n<16, MH, NK16>(acc, da, a_half16, alo16, db, blo16, want_lo, first); break;
    case 32: wg_kblock_n<32, MH, NK16>(acc, da, a_half16, alo16, db, blo16, want_lo, first); break;
    case 48: wg_kblock_n<48, MH, NK16>(acc, da, a_half16, alo16, db, blo16, want_lo, first); break;
    case 64: wg_kblock_n<64, MH, NK16>(acc, da, a_half16, alo16, db, blo16, want_lo, first); break;
    case 80: wg_kblock_n<80, MH, NK16>(acc, da, a_half16, alo16, db, blo16, want_lo, first); break;
    default: wg_kblock_n<96, MH, NK16>(acc, da, a_half16, alo16, db, blo16, want_lo, first); break;
    }
}

// The consumer warpgroup `wg` has finished reading a stage: one arrival per warpgroup, plus one on the same barrier
// of the peer CTA when the pair shares its A tiles (the peer overwrites its copy, and pushes into ours, only after
// both CTAs have consumed the stage).
template <bool SHARE>
__device__ __forceinline__ void wg_release(uint32_t bar, int wg, int wt, uint32_t peer) {
    asm volatile("bar.sync %0, 128;" ::"r"(4 + wg) : "memory");
    if (wt == 0) {
        mbar_arrive(bar);
        if (SHARE) mbar_arrive_cluster(mapa_peer(bar, peer));
    }
}

// row of the second residual for output pixel m: the pixel itself, or (fused keras UpSampling2D, reception.py:122-127)
// its source pixel in the half-resolution tensor
__device__ __forceinline__ size_t res1_src(const ConvParams& c, int m) {
    if (!c.up1) return (size_t)m;
    const int hw = c.Ho * c.Wo;
    const int n = m / hw, rem = m - n * hw;
    const int y = rem / c.Wo, x = rem - y * c.Wo;
    return ((size_t)n * (c.Ho >> 1) + (y >> 1)) * (size_t)(c.Wo >> 1) + (size_t)(x >> 1);
}

__device__ __forceinline__ float2 ldg2(const float* p) { return __ldg(reinterpret_cast<const float2*>(p)); }

// Fused epilogue straight from the accumulator fragment: BN affine, ReLU, residual adds, store.  The warpgroup's
// rows are m0 + 64 h + (fragment row), its columns n0 + (fragment column); each quad of lanes writes 32 contiguous
// bytes of a row (float2 per lane wherever the pointers and leading dimensions allow, else scalars).
template <int MH>
__device__ __forceinline__ void wg_epilogue(const TcParams& P, const float (&acc)[MH][ACC_N], int m0, int n0, int wt) {
    const ConvParams& c = P.c;
#ifdef DH_ABLATE
    if (P.dbg & 32) return;
#endif
    const int rq = 16 * (wt >> 5) + ((wt & 31) >> 2);
    const int cq = 2 * (wt & 3);
    const bool v2 = !((c.ldo | c.Cout) & 1) && !(reinterpret_cast<uintptr_t>(c.out) & 7) &&
                    (!c.res0 || (!(c.ldr0 & 1) && !(reinterpret_cast<uintptr_t>(c.res0) & 7))) &&
                    (!c.res1 || (!(c.ldr1 & 1) && !(reinterpret_cast<uintptr_t>(c.res1) & 7))) &&
                    (!c.post_scale || (!(reinterpret_cast<uintptr_t>(c.post_scale) & 7) &&
                                       !(reinterpret_cast<uintptr_t>(c.post_shift) & 7)));
    const bool relu = c.post_relu != 0, has_post = c.post_scale != nullptr;
#pragma unroll
    for (int h = 0; h < MH; ++h)
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
            const int m = m0 + 64 * h + rq + 8 * hr;
            if (m >= c.M) continue;
            float* orow = c.out + (size_t)m * c.ldo;
            const float* r0row = c.res0 ? c.res0 + (size_t)m * c.ldr0 : nullptr;
            const float* r1row = c.res1 ? c.res1 + res1_src(c, m) * c.ldr1 : nullptr;
#pragma unroll
            for (int j = 0; j < ACC_N / 4; ++j) {
                if (8 * j >= P.bn_cta) break;
                const int co = n0 + 8 * j + cq;
                float2 v = make_float2(acc[h][4 * j + 2 * hr], acc[h][4 * j + 2 * hr + 1]);
                if (v2) {
                    if (co < c.Cout) {
                        if (has_post) v = ffma2(v, ldg2(c.post_scale + co), ldg2(c.post_shift + co));
                        if (relu) v = make_float2(fmaxf(v.x, 0.f), fmaxf(v.y, 0.f));
                        if (r0row) v = fadd2(v, ldg2(r0row + co));
                        if (r1row) v = fadd2(v, ldg2(r1row + co));
                        *reinterpret_cast<float2*>(orow + co) = v;
                    }
                } else {
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int cc = co + e;
                        if (cc < c.Cout) {
                            float t = e ? v.y : v.x;
                            if (has_post) t = fmaf(t, __ldg(c.post_scale + cc), __ldg(c.post_shift + cc));
                            if (relu) t = fmaxf(t, 0.f);
                            if (r0row) t += __ldg(r0row + cc);
                            if (r1row) t += __ldg(r1row + cc);
                            orow[cc] = t;
                        }
                    }
                }
            }
        }
}

// ---------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static inline EncodeTiledFn get_encode() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            fn = (EncodeTiledFn)p;
    }
    return fn;
}

static inline bool make_map(CUtensorMap* map, const void* base, int k_pad, int rows, int box_rows) {
    EncodeTiledFn enc = get_encode();
    if (!enc) return false;
    cuuint64_t dims[2] = {(cuuint64_t)k_pad, (cuuint64_t)rows};
    cuuint64_t strides[1] = {(cuuint64_t)k_pad * 2};
    cuuint32_t box[2] = {(cuuint32_t)BK, (cuuint32_t)box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS;
}

static inline bool make_map_b64(CUtensorMap* map, const void* base, int k_pad, int rows, int box_rows) {
    EncodeTiledFn enc = get_encode();
    if (!enc) return false;
    cuuint64_t dims[2] = {(cuuint64_t)k_pad, (cuuint64_t)rows};
    cuuint64_t strides[1] = {(cuuint64_t)k_pad * 2};
    cuuint32_t box[2] = {(cuuint32_t)SBK, (cuuint32_t)box_rows};
    cuuint32_t estr[2] = {1, 1};
    return enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
               CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
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


// N tiling rule shared with the host-side weight packer (dh_tc_cout_pad): Cout padded to 16 and split over gy CTAs
// of bn_cta <= MAX_BN_CTA columns (a multiple of 16: the wgmma N of the tile).
static inline void tile_n(int cout, int* bn_cta, int* gy) {
    const int cp = (cout + 15) / 16 * 16;
    const int g = (cp + MAX_BN_CTA - 1) / MAX_BN_CTA;
    *bn_cta = ((cp + g - 1) / g + 15) / 16 * 16;
    *gy = g;
}

}  // namespace tc
