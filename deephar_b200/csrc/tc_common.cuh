// Shared pieces of the wgmma convolution kernels (conv_tc.cu, conv_sep.cu, conv_patch.cu): constants, launch
// parameters, PTX wrappers (TMA, wgmma, DSMEM, setmaxnreg; the mbarrier and cluster basics are in common.cuh),
// shared-memory matrix descriptors, the bf16 hi/lo split, the consumer warpgroups (wgmma issue + fused epilogue)
// and the host side: tensor maps, N tiling, the eligibility rules the kernels share, their plans and the persistent launch.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <type_traits>
#include "common.cuh"
#include "conv_params.cuh"

namespace tc {


constexpr int BM = 128;
constexpr int BK = 64;                 // bf16 per K-block = one 128-byte swizzle row
constexpr int NPROD = 256;             // A producers: warps 0..7 (two warpgroups)
// Columns (output channels) per CTA.  The fp32 accumulators of a 128 x MAX_BN_CTA tile live in the registers of
// the consumer warpgroup that owns the tile (Hopper has no tensor memory): 96 per thread.  Wider layers are split
// over gridDim.y.
constexpr int MAX_BN_CTA = 96;
constexpr int ACC_N = MAX_BN_CTA / 2;  // fp32 accumulator registers per thread per m64 slice
constexpr int MH = BM / 64;            // m64 slices (wgmma M = 64) of a tile, all in one consumer warpgroup
// conv_sep.cu also runs 64-row tiles (one m64 slice) of up to 144 columns: 72 accumulator registers per thread.  The
// consumer code below takes the tile shape from its accumulator array, float[tile rows / 64][columns / 2].
constexpr int BM64 = 64;
constexpr int MAX_BN_CTA64 = 144;
constexpr int bn_max(int bm) { return bm == BM64 ? MAX_BN_CTA64 : MAX_BN_CTA; }
// Warp roles: producers (NPW warpgroups) | consumers (Q warpgroups: wgmma issue, then the fused epilogue from
// the accumulator registers) | one control warpgroup (weight TMA, patch TMA, two spare warps).  A consumer
// warpgroup always owns whole tiles; with Q = 2 the two take alternate tiles of the CTA (ping-pong), so
// that one runs its epilogue while the other issues the next tile's wgmmas.
// Register budget (setmaxnreg; ptxas allocates each role's code against its own value):
//   Q = 1: 512 threads launch with 128 registers: 256 * 168 + 128 * 144 + 128 * 32 = 65536
//   Q = 2, NPW = 1 (conv_sep.cu): 512 threads launch with 128: ONE producer warpgroup with 192 registers (the 5x5
//          depthwise keeps 25 tap pairs + 16 accumulator pairs + an input row in registers: ~115, and it spills
//          below that), 128 * 192 + 256 * 144 + 128 * 32 = 65536.
//   Q = 2, NPW = 2 (conv_patch.cu): 640 threads launch with 96 (65536 / 640 rounded down to the allocation unit).  setmaxnreg only
//          redistributes the CTA's OWN allocation, 640 * 96 = 61440 registers (asking for more blocks forever):
//          producers drop to 88 (the TMA-staged producers fit), control to 32, the consumers grow to 136 (96
//          accumulators + the epilogue's batch; 144 elsewhere): 256 * 88 + 256 * 136 + 128 * 32 = 61440.
template <int Q, int NPW = 2>
struct Roles {
    static constexpr int EPQ = Q;                           // consumer warpgroups
    static constexpr int NEPI = 128 * Q;
    static constexpr int WARP_EPI0 = 4 * NPW;               // first consumer warp
    static constexpr int WARP_TMA = WARP_EPI0 + 4 * Q, WARP_PATCH = WARP_TMA + 2;
    static constexpr int NTHREADS = 32 * (WARP_TMA + 4);
    static constexpr int REGS_PROD = Q == 1 ? 168 : (NPW == 1 ? 192 : 88);
    static constexpr int REGS_EPI = Q == 2 && NPW == 2 ? 136 : 144, REGS_CTRL = 32;
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

// conv_sep.cu
struct SepParams {
    TcParams t;
    int patch_stride;       // bytes between consecutive patch buffers (>= patch_bytes, 1024-aligned)
    int patch_bytes;
    int ry, fn;             // tile rows per frame, frames per tile
    int bm;                 // rows per M-tile: BM (128 x 96 tiles) or BM64 (64 x 144 tiles)
    int epi_smem;           // bytes of the shared-memory epilogue's buffers (EpiSmem; 64-row tiles), 0 = register epilogue
    int dbg;                // ablation bits (tools/ only): 1 no depthwise math, 2 no patch TMA, 8 no DSMEM push, 16 no weight TMA, 64 no MMA issue (32: epilogue without global traffic, TcParams::dbg); plan only: 16384 / 32768 force the 64 x 144 / 128 x 96 tile, 65536 the register epilogue
};

// conv_patch.cu
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

// ---------------------------------------------------------------------------
// PTX wrappers (the mbarrier, bulk-copy and cluster basics are in common.cuh)
// ---------------------------------------------------------------------------
// mbar_wait, for waits that are expected to be long (not on the MMA-issue critical path): sleep between polls so
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
// shared memory -> global box (bulk async-group completion: bulk_commit, then bulk_wait_read before the source is reused)
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* map, uint32_t src, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
                 ::"l"(map), "r"(src), "r"(c0), "r"(c1)
                 : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
// ---- 2-CTA cluster helpers (A-tile sharing between the two N-part CTAs of one pixel tile) ----
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

template <> __device__ __forceinline__ void wgmma_bf16<144>(float* d, uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile(
        "{\n .reg .pred p;\n setp.ne.b32 p, %74, 0;\n"
        " wgmma.mma_async.sync.aligned.m64n144k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71}, %72, %73, p, 1, 1, 0, 0;\n}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71])
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
constexpr int A_BYTES = BM * 64;           // A tile of one K-block: 8 KB per (hi | lo)
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
template <int N, int MHT, int ACCN>
__device__ __forceinline__ void acc_fence_all(float (&acc)[MHT][ACCN]) {
#pragma unroll
    for (int h = 0; h < MHT; ++h)
#pragma unroll
        for (int i = 0; i < N / 2; ++i) acc_fence(acc[h][i]);
}

// One K-block as ONE wgmma commit group: NK16 k-steps of 16 (ascending), the MH 64-row slices of A (slice stride
// a_half16 in descriptor units of 16 B); per k-step and slice hi*hi, then at precision 3 (LO) lo*hi and hi*lo,
// accumulated in fp32 registers.  No branch between the wgmmas, so ptxas issues them back to back.
template <int N, int NK16, bool LO, int MHT, int ACCN>
__device__ __forceinline__ void wg_issue_kblock(float (&acc)[MHT][ACCN], uint64_t da, uint32_t a_half16, uint32_t alo16,
                                                uint64_t db, uint32_t blo16, bool first) {
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < NK16; ++k) {
        const uint32_t acc0 = (first && k == 0) ? 0u : 1u;
#pragma unroll
        for (int h = 0; h < MHT; ++h) {
            const uint64_t a = da + (uint64_t)(h * a_half16 + 2 * k);
            wgmma_bf16<N>(acc[h], a, db + 2 * k, acc0);
            if (LO) {
                wgmma_bf16<N>(acc[h], a + alo16, db + 2 * k, 1u);
                wgmma_bf16<N>(acc[h], a, db + blo16 + 2 * k, 1u);
            }
        }
    }
    wgmma_commit();
}

// The K-blocks of one tile.  stage(kb, da, db) waits until K-block kb's operands are in shared memory and returns
// their A / B descriptors; release(kb) hands K-block kb's stages back to the producers.  One commit group stays in
// flight: K-block kb is issued before the stages of kb - 1 are released, so the tensor pipe does not drain between
// K-blocks; the tile's last K-block is drained before returning (the epilogue reads the accumulators).  Consecutive
// K-blocks must therefore sit in different stages of every ring (all rings are >= 2 deep when nkb >= 2).
// mma = false skips the wgmmas and keeps the synchronisation (timing ablation).
template <int N, int NK16, bool LO, int MHT, int ACCN, class Stage, class Release>
__device__ __forceinline__ void wg_tile_n(float (&acc)[MHT][ACCN], int nkb, uint32_t a_half16, uint32_t alo16,
                                          uint32_t blo16, bool mma, Stage& stage, Release& release) {
    for (int kb = 0; kb < nkb; ++kb) {
        uint64_t da, db;
        stage(kb, da, db);
        if (mma) {
            acc_fence_all<N>(acc);
            wg_issue_kblock<N, NK16, LO>(acc, da, a_half16, alo16, db, blo16, kb == 0);
        }
        wgmma_wait<1>();                // K-block kb - 1 has completed; kb may still run
        acc_fence_all<N>(acc);
        if (kb > 0) release(kb - 1);
    }
    wgmma_wait<0>();
    acc_fence_all<N>(acc);
    release(nkb - 1);
}

// wgmma N is an immediate: one instantiation per tile width bn_cta (16 .. MAX_BN_CTA, step 16), chosen once per tile.
// 64-row tiles are planned at bn_cta = MAX_BN_CTA64 only.
template <int NK16, bool LO, int MHT, int ACCN, class Stage, class Release>
__device__ __forceinline__ void wg_tile(int bn, float (&acc)[MHT][ACCN], int nkb, uint32_t a_half16, uint32_t alo16,
                                        uint32_t blo16, bool mma, Stage&& stage, Release&& release) {
    if constexpr (ACCN == MAX_BN_CTA64 / 2) {
        wg_tile_n<MAX_BN_CTA64, NK16, LO>(acc, nkb, a_half16, alo16, blo16, mma, stage, release);
    } else {
        switch (bn) {
        case 16: wg_tile_n<16, NK16, LO>(acc, nkb, a_half16, alo16, blo16, mma, stage, release); break;
        case 32: wg_tile_n<32, NK16, LO>(acc, nkb, a_half16, alo16, blo16, mma, stage, release); break;
        case 48: wg_tile_n<48, NK16, LO>(acc, nkb, a_half16, alo16, blo16, mma, stage, release); break;
        case 64: wg_tile_n<64, NK16, LO>(acc, nkb, a_half16, alo16, blo16, mma, stage, release); break;
        case 80: wg_tile_n<80, NK16, LO>(acc, nkb, a_half16, alo16, blo16, mma, stage, release); break;
        default: wg_tile_n<96, NK16, LO>(acc, nkb, a_half16, alo16, blo16, mma, stage, release); break;
        }
    }
}

// Ping-pong order of two consumer warpgroups (warpgroup wg owns the CTA's tiles ti = wg, wg + 2, ...).  The rings'
// full barriers are waited on by phase parity, which tells use u of a stage from use u - 1 but not from use u - 2:
// a warpgroup may start waiting for a tile's K-blocks only once every K-block of the tiles before it has arrived.
// So a warpgroup that has passed the full barriers of its tile's last K-block signals the other (pp_pass), and a
// warpgroup waits for that signal before its next tile (pp_wait).  Named barriers 6 and 7 ("tile of warpgroup 0 / 1
// has arrived"), 128 arriving + 128 waiting threads; every pp_pass has exactly one matching pp_wait.
__device__ __forceinline__ void pp_pass(int wg) { asm volatile("bar.arrive %0, 256;" ::"r"(6 + wg) : "memory"); }
__device__ __forceinline__ void pp_wait(int wg) { asm volatile("bar.sync %0, 256;" ::"r"(7 - wg) : "memory"); }

// The consumer warpgroup `wg` has finished reading a stage: one arrival per warpgroup, plus (remote) one on the same
// barrier of the peer CTA when that CTA writes the stage's A tile (it overwrites its copy, and pushes into ours, only
// after both CTAs have consumed the stage).
__device__ __forceinline__ void wg_release(uint32_t bar, int wg, int wt, bool remote, uint32_t peer) {
    asm volatile("bar.sync %0, 128;" ::"r"(4 + wg) : "memory");
    if (wt == 0) {
        mbar_arrive(bar);
        if (remote) mbar_arrive_cluster(mapa_peer(bar, peer));
    }
}

__device__ __forceinline__ float2 ldg2(const float* p) { return __ldg(reinterpret_cast<const float2*>(p)); }

// The BN scale / shift of the CTA's output columns n0 .. n0 + bn_cta - 1, staged in shared memory once per CTA for
// the epilogue (post[j] = scale, post[BNMAX + j] = shift of column n0 + j, BNMAX = bn_max(tile rows)): the epilogue
// then batches only its residual loads, which keeps it free of spills next to the 96 (72) accumulator registers.  Run
// by the NEPI consumer threads (ct = 0 .. NEPI - 1) before their first tile; named barrier 2 orders the stores before
// every read.
constexpr int post_smem(int bm) { return 2 * bn_max(bm) * 4; }
constexpr int POST_SMEM = post_smem(BM);
template <int NEPI, int BNMAX = MAX_BN_CTA>
__device__ __forceinline__ void stage_post(const TcParams& P, int n0, float* post, int ct) {
    const ConvParams& c = P.c;
    if (c.post_scale) {
        for (int j = ct; j < P.bn_cta; j += NEPI) {
            const int co = n0 + j;
            post[j] = co < c.Cout ? __ldg(c.post_scale + co) : 0.f;
            post[BNMAX + j] = co < c.Cout ? __ldg(c.post_shift + co) : 0.f;
        }
    }
    asm volatile("bar.sync 2, %0;" ::"n"(NEPI) : "memory");
}

// L2 prefetch of the residual rows a tile's epilogue will read (columns n0 .. n0 + bn_cta - 1, one row per thread of
// the consumer warpgroup; threads past the tile's TBM rows issue none), issued when the warpgroup starts the tile: its
// mainloop then covers the HBM latency, and the epilogue's few loads in flight (JC below) wait on L2 instead.  No
// registers stay live.
__device__ __forceinline__ void prefetch_l2(const float* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }
template <int TBM = BM>
__device__ __forceinline__ void wg_prefetch_res(const TcParams& P, int m0, int n0, int wt) {
    const ConvParams& c = P.c;
#ifdef DH_ABLATE
    if (P.dbg & 32) return;
#endif
    const int m = m0 + wt;
    if (wt >= TBM || m >= c.M) return;
    const int last = min(P.bn_cta, c.Cout - n0) - 1;        // 128-byte lines: every 32nd column, and the last one
    if (c.res0) {
        const float* r = c.res0 + (size_t)m * c.ldr0 + n0;
        for (int k = 0; k < last; k += 32) prefetch_l2(r + k);
        prefetch_l2(r + last);
    }
    if (c.res1) {
        const float* r = c.res1 + res1_src(c, m) * c.ldr1 + n0;
        for (int k = 0; k < last; k += 32) prefetch_l2(r + k);
        prefetch_l2(r + last);
    }
}

// Fused epilogue of one tile (MHT x 64 rows, up to 2 ACCN columns) straight from the accumulator fragment: BN affine,
// ReLU, residual adds, store.  Rows m0 + 64 h + (fragment row), columns n0 + (fragment column); each quad of lanes
// writes 32 contiguous bytes of a row (float2 per lane wherever the pointers and leading dimensions allow, else
// scalars).  `post`: stage_post, with BNMAX = 2 ACCN.
template <int MHT, int ACCN>
__device__ __forceinline__ void wg_epilogue(const TcParams& P, const float (&acc)[MHT][ACCN], int m0, int n0, int wt,
                                            const float* post) {
    const ConvParams& c = P.c;
#ifdef DH_ABLATE
    if (P.dbg & 32) return;
#endif
    const int rq = 16 * (wt >> 5) + ((wt & 31) >> 2);
    const int c0 = n0 + 2 * (wt & 3);               // the thread's first column; its others are c0 + 8 j (+ 1)
    const bool v2 = !((c.ldo | c.Cout) & 1) && !(reinterpret_cast<uintptr_t>(c.out) & 7) &&
                    (!c.res0 || (!(c.ldr0 & 1) && !(reinterpret_cast<uintptr_t>(c.res0) & 7))) &&
                    (!c.res1 || (!(c.ldr1 & 1) && !(reinterpret_cast<uintptr_t>(c.res1) & 7)));
    const bool relu = c.post_relu != 0, has_post = c.post_scale != nullptr;
    // columns c0 + 8 j + e exist for 8 j + e < ncol (past bn_cta: the next CTA's; past Cout: none).  All column
    // offsets are compile-time constants from per-row base pointers, so no per-column index stays live.
    const int ncol = min(P.bn_cta - 2 * (wt & 3), c.Cout - c0);
    const float* sc = post + (c0 - n0);
    const float* sh = sc + 2 * ACCN;
    // float2 path: the residual loads of JC column groups are issued together before their arithmetic and stores, so
    // that the global-load latency is paid once per JC groups rather than once per group (the stores in between would
    // otherwise keep the compiler from hoisting the next group's loads).  Next to the 96 accumulator registers a batch
    // of 3 groups (12 registers for two residuals) is what fits without spills.
    constexpr int JC = 3;
    static_assert((ACCN / 4) % JC == 0, "column groups per batch");
#pragma unroll
    for (int h = 0; h < MHT; ++h)
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
            const int m = m0 + 64 * h + rq + 8 * hr;
            if (m >= c.M) continue;
            float* orow = c.out + (size_t)m * c.ldo + c0;
            const float* r0row = c.res0 ? c.res0 + (size_t)m * c.ldr0 + c0 : nullptr;
            const float* r1row = c.res1 ? c.res1 + res1_src(c, m) * c.ldr1 + c0 : nullptr;
            if (v2) {
#pragma unroll
                for (int j0 = 0; j0 < ACCN / 4; j0 += JC) {
                    if (8 * j0 >= P.bn_cta) break;
                    float2 ra[JC], rb[JC];
#pragma unroll
                    for (int jj = 0; jj < JC; ++jj) {
                        if (8 * (j0 + jj) < ncol) {
                            if (r0row) ra[jj] = ldg2(r0row + 8 * (j0 + jj));
                            if (r1row) rb[jj] = ldg2(r1row + 8 * (j0 + jj));
                        }
                    }
#pragma unroll
                    for (int jj = 0; jj < JC; ++jj) {
                        const int j = j0 + jj;
                        if (8 * j < ncol) {
                            float2 v = make_float2(acc[h][4 * j + 2 * hr], acc[h][4 * j + 2 * hr + 1]);
                            if (has_post)
                                v = ffma2(v, *reinterpret_cast<const float2*>(sc + 8 * j),
                                          *reinterpret_cast<const float2*>(sh + 8 * j));
                            if (relu) v = make_float2(fmaxf(v.x, 0.f), fmaxf(v.y, 0.f));
                            if (r0row) v = fadd2(v, ra[jj]);
                            if (r1row) v = fadd2(v, rb[jj]);
                            *reinterpret_cast<float2*>(orow + 8 * j) = v;
                        }
                    }
                }
                continue;
            }
#pragma unroll
            for (int j = 0; j < ACCN / 4; ++j) {
                if (8 * j >= P.bn_cta) break;
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int k = 8 * j + e;
                    if (k < ncol) {
                        float t = acc[h][4 * j + 2 * hr + e];
                        if (has_post) t = fmaf(t, sc[k], sh[k]);
                        if (relu) t = fmaxf(t, 0.f);
                        if (r0row) t += __ldg(r0row + k);
                        if (r1row) t += __ldg(r1row + k);
                        orow[k] = t;
                    }
                }
            }
        }
}

// Shared-memory epilogue of conv_sep.cu's 64 x 144 tiles.  One fp32 buffer [64][144] (the TMA box layout) serves both
// consumer warpgroups: a control warp loads tile ti's first residual into it by TMA (and the up2x residual's 16
// half-resolution rows into r1) once tile ti - 1's output has left it (`empty`, one arrival per tile), completing on
// full0 + 8 (ti & 1) -- one barrier per warpgroup, so that each waiter sees consecutive phases.
struct EpiSmem {
    float* buf;                       // residual 0 on arrival, the output tile on departure; nullptr: register epilogue
    const float* r1;                  // [16][144] rows of the upsampled second residual, or nullptr
    uint32_t full0, empty;
    const CUtensorMap* map_out;
};
constexpr int EPI_BUF_BYTES = BM64 * MAX_BN_CTA64 * 4, EPI_R1_BYTES = BM64 / 4 * MAX_BN_CTA64 * 4;

// The epilogue of tile ti (rows m0 .., columns n0 ..) through the buffer: each thread adds the residuals of its
// accumulator fragment from shared memory with the operations, in the order, of wg_epilogue (so the results are the
// same bit for bit), writes the result in place, and one thread stores the tile by TMA.  The box clips the rows past
// M and the columns past Cout.  The warpgroup goes on to its next tile as soon as the store has read the buffer.
template <int ACCN>
__device__ __forceinline__ void wg_epilogue_smem(const TcParams& P, const float (&acc)[1][ACCN], int ti, int m0, int n0,
                                                 int wg, int wt, const float* post, const EpiSmem& es) {
    static_assert(2 * ACCN == MAX_BN_CTA64, "the buffer holds one 64 x 144 tile");
    const ConvParams& c = P.c;
    mbar_wait(es.full0 + 8 * wg, (uint32_t)(ti >> 1) & 1);
#ifdef DH_ABLATE
    const bool skip = P.dbg & 32;
#else
    constexpr bool skip = false;
#endif
    if (!skip) {
        const int rq = 16 * (wt >> 5) + ((wt & 31) >> 2);
        const int cq = 2 * (wt & 3);
        const bool relu = c.post_relu != 0, has_post = c.post_scale != nullptr, r0 = c.res0 != nullptr;
        const float* sc = post + cq;
        const float* sh = sc + 2 * ACCN;
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
            const int r = rq + 8 * hr;
            float* row = es.buf + r * MAX_BN_CTA64 + cq;
            const float* r1row = es.r1 ? es.r1 + (res1_src(c, m0 + r) - (size_t)(m0 / 4)) * MAX_BN_CTA64 + cq : nullptr;
#pragma unroll
            for (int j = 0; j < ACCN / 4; ++j) {
                float2 v = make_float2(acc[0][4 * j + 2 * hr], acc[0][4 * j + 2 * hr + 1]);
                if (has_post)
                    v = ffma2(v, *reinterpret_cast<const float2*>(sc + 8 * j), *reinterpret_cast<const float2*>(sh + 8 * j));
                if (relu) v = make_float2(fmaxf(v.x, 0.f), fmaxf(v.y, 0.f));
                if (r0) v = fadd2(v, *reinterpret_cast<const float2*>(row + 8 * j));
                if (r1row) v = fadd2(v, *reinterpret_cast<const float2*>(r1row + 8 * j));
                *reinterpret_cast<float2*>(row + 8 * j) = v;
            }
        }
        fence_proxy_async();                  // the generic-proxy writes above, before the TMA store reads them
    }
    asm volatile("bar.sync %0, 128;" ::"r"(4 + wg) : "memory");
    if (wt == 0) {
        if (!skip) {
            tma_store_2d(es.map_out, smem_u32(es.buf), n0, m0);
            bulk_commit();
            bulk_wait_read();
        }
        mbar_arrive(es.empty);
    }
}

// The consumer role of the patch-staged kernels (conv_sep.cu, conv_patch.cu): warpgroup wg (thread wt of it) runs the
// CTA's tiles ti = wg, wg + 2, ... of tiles_mine in ping-pong order (pp_pass / pp_wait).  K-block g of the CTA reads
// A stage g % NA (full0 / empty0: one full and two empty barriers per stage, the empty one chosen by use parity) and
// weight stage g % NB (fullb0 / emptyb0); dbase / dbase_b are the descriptors of the two rings' first stages.  SHARE:
// stage s is produced by the pair's CTA of rank s & 1, and the stages the peer produces are released on the peer too
// (NA is even).  TBM: rows per tile (BM, or BM64 with bn_cta = MAX_BN_CTA64).  es: the shared-memory epilogue of
// 64-row tiles (wg_epilogue_smem), unless es.buf is null.  dbg (`make ABLATE=1` builds): 64 = no
// wgmmas, 128 = no A waits.
template <bool SHARE, bool LO, int NA, int NB, int TBM = BM>
__device__ __forceinline__ void pp_consumer(const TcParams& P, int wg, int wt, int n0, int tiles_mine, uint64_t dbase,
                                            uint64_t dbase_b, uint32_t bar_full0, uint32_t bar_empty0,
                                            uint32_t bar_fullb0, uint32_t bar_emptyb0, uint32_t rank, const float* post,
                                            int dbg, EpiSmem es = {}) {
    static_assert(NA % 2 == 0 || !SHARE, "each A stage has one producing CTA of the pair");
    const int nkb = P.n_kblocks;
    const int b_bytes = P.bn_cta * 64;                       // per (hi | lo)
    constexpr int a_bytes = TBM * 64;                        // A tile of one K-block, per (hi | lo)
    float acc[TBM / 64][bn_max(TBM) / 2];
    const uint32_t sta16 = (2 * a_bytes) >> 4, stb16 = (uint32_t)(2 * b_bytes) >> 4, alo16 = a_bytes >> 4,
                   blo16 = (uint32_t)b_bytes >> 4, half16 = (64 * 64) >> 4;
    for (int ti = wg; ti < tiles_mine; ti += 2) {
        const int g0 = ti * nkb, m0 = ((int)blockIdx.x + ti * (int)gridDim.x) * TBM;
        if (ti > 0) pp_wait(wg);
        if (!es.buf) wg_prefetch_res<TBM>(P, m0, n0, wt);
        wg_tile<SBK / 16, LO>(
            P.bn_cta, acc, nkb, half16, alo16, blo16, !(dbg & 64),
            [&](int kb, uint64_t& da, uint64_t& db) {
                const int g = g0 + kb, s = g % NA, sb = g % NB;
                if (!(dbg & 128)) mbar_wait(bar_full0 + 8 * s, (uint32_t)(g / NA) & 1);
                mbar_wait(bar_fullb0 + 8 * sb, (uint32_t)(g / NB) & 1);
                if (kb == nkb - 1 && ti + 1 < tiles_mine) pp_pass(wg);
                da = dbase + (uint64_t)((uint32_t)s * sta16);
                db = dbase_b + (uint64_t)((uint32_t)sb * stb16);
            },
            [&](int kb) {
                const int g = g0 + kb, s = g % NA;
                const uint32_t producer = (uint32_t)(s & 1);
                wg_release(bar_empty0 + 16 * s + 8 * ((g / NA) & 1), wg, wt, SHARE && producer != rank, producer);
                if (wt == 0) mbar_arrive(bar_emptyb0 + 8 * (g % NB));
            });
        if constexpr (TBM == BM64) {
            if (es.buf) {
                wg_epilogue_smem(P, acc, ti, m0, n0, wg, wt, post, es);
                continue;
            }
        }
        wg_epilogue(P, acc, m0, n0, wt, post);
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

// weight tensor map: packed bf16 [rows][k_pad] (K-major), box = kblk x box_rows.  A box row of kblk bf16 is one
// swizzle row: kblk = BK (conv_tc.cu) -> 128B swizzle, kblk = SBK (patch-staged kernels) -> 64B swizzle.
static inline bool make_map_w(CUtensorMap* map, const void* base, int k_pad, int rows, int kblk, int box_rows) {
    EncodeTiledFn enc = get_encode();
    if (!enc) return false;
    cuuint64_t dims[2] = {(cuuint64_t)k_pad, (cuuint64_t)rows};
    cuuint64_t strides[1] = {(cuuint64_t)k_pad * 2};
    cuuint32_t box[2] = {(cuuint32_t)kblk, (cuuint32_t)box_rows};
    cuuint32_t estr[2] = {1, 1};
    return enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
               CU_TENSOR_MAP_INTERLEAVE_NONE, kblk == BK ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B,
               CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// fp32 activations, pixel stride ldx floats, as a 4-D tensor (C, W, H, N) for the patch TMA of the patch-staged
// kernels; box = (SBK channels, pc columns, pr rows, fn frames).  Out-of-bounds coordinates are zero filled.
static inline bool make_map_x(CUtensorMap* map, const float* x, int ldx, int c, int w, int h, int n, int pc, int pr,
                              int fn) {
    EncodeTiledFn enc = get_encode();
    if (!enc) return false;
    cuuint64_t dims[4] = {(cuuint64_t)c, (cuuint64_t)w, (cuuint64_t)h, (cuuint64_t)n};
    cuuint64_t strides[3] = {(cuuint64_t)ldx * 4, (cuuint64_t)w * ldx * 4, (cuuint64_t)h * w * ldx * 4};
    cuuint32_t box[4] = {(cuuint32_t)SBK, (cuuint32_t)pc, (cuuint32_t)pr, (cuuint32_t)fn};
    cuuint32_t estr[4] = {1, 1, 1, 1};
    return enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, const_cast<float*>(x), dims, strides, box, estr,
               CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// fp32 matrix view (rows of `cols` floats, ld floats apart) as a 2-D tensor (cols, rows); box = box_cols x box_rows.
// Out-of-bounds elements are zero filled on load and skipped on store.  The driver takes only views whose base is
// 16-byte aligned and whose row pitch is a multiple of 16 bytes (tma_view_ok).
static inline bool make_map_rows(CUtensorMap* map, const float* p, int cols, int rows, int ld, int box_cols, int box_rows) {
    EncodeTiledFn enc = get_encode();
    if (!enc) return false;
    cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
    cuuint64_t strides[1] = {(cuuint64_t)ld * 4};
    cuuint32_t box[2] = {(cuuint32_t)box_cols, (cuuint32_t)box_rows};
    cuuint32_t estr[2] = {1, 1};
    return enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(p), dims, strides, box, estr,
               CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}
static inline bool tma_view_ok(const float* p, int ld) { return !(reinterpret_cast<uintptr_t>(p) & 15) && !(ld & 3); }

// N tiling rule shared with the host-side weight packer (dh_tc_cout_pad): Cout padded to 16 and split over gy CTAs
// of bn_cta <= max_bn columns (a multiple of 16: the wgmma N of the tile).  The packing is the one of max_bn =
// MAX_BN_CTA; the 64-row tiles of conv_sep.cu read it in N parts of MAX_BN_CTA64 rows, rows past cout_pad zero filled.
static inline void tile_n(int cout, int* bn_cta, int* gy, int max_bn = MAX_BN_CTA) {
    const int cp = (cout + 15) / 16 * 16;
    const int g = (cp + max_bn - 1) / max_bn;
    *bn_cta = ((cp + g - 1) / g + 15) / 16 * 16;
    *gy = g;
}

constexpr size_t SMEM_LIMIT = 227 * 1024;     // dynamic shared memory a block may opt into on sm_90

// the packed weights are this layer's: K (kh * kw * Cin, or Cin for a pointwise stage) and Cout, padded by the packer
static inline bool packed_fits(const dh_packed_w* w, int K, int cout) {
    return w->k == dh_tc_k_pad(K) && w->cout_pad == dh_tc_cout_pad(cout);
}

// the BN-prologue vectors can be read 16 bytes at a time
static inline bool bn_pro_aligned(const ConvParams& p) {
    return !p.pre_scale || !((reinterpret_cast<uintptr_t>(p.pre_scale) | reinterpret_cast<uintptr_t>(p.pre_shift)) & 15);
}

// What conv_tc.cu needs of any layer.  Its producers and the epilogues index pixels in int32 (up to a tile past the
// last one) and form every product with ld in 64 bits -- pixel * ld, and the scalar gather's per-tap offset
// (ky * W + kx) * ldx -- so a view may span any number of elements; DenseRows packs a window origin's row and column
// into 16 bits each.
static inline bool tc_layer_ok(const ConvParams& p, const dh_packed_w* w, int K) {
    return p.M >= 1 && packed_fits(w, K, p.Cout) && (int64_t)p.N * p.H * p.W <= (1ll << 31) - 2 * BM &&
           (int64_t)p.M <= (1ll << 31) - 2 * BM && p.H < (1 << 15) && p.W < (1 << 15);
}

// separable layers both separable kernels (conv_tc.cu, conv_sep.cu) take: 3x3 or 5x5 depthwise, stride 1, SAME, and
// pixel blocks of 2 channels x 4 x 4 pixels that tile the 128-pixel tile without straddling a frame: the tile is whole
// 4-row strips (produce_sep), so W <= 32; at W = 64 or 128 the eight blocks would cover 4 rows of 32 columns instead
static inline bool sep_layer_ok(const ConvParams& p, const dh_packed_w* w) {
    if (!tc_layer_ok(p, w, p.Cin) || (reinterpret_cast<uintptr_t>(p.x) & 15) || !bn_pro_aligned(p)) return false;
    if (!(p.kh == p.kw && (p.kh == 3 || p.kh == 5))) return false;
    if (p.sh != 1 || p.sw != 1) return false;
    if (p.Ho != p.H || p.Wo != p.W) return false;                 // SAME, stride 1
    if (p.W < 4 || (BM % (4 * p.W)) != 0 || (p.W & 3) || (p.H & 3)) return false;
    if ((p.Cin & 1) || (p.ldx & 1)) return false;
    if ((reinterpret_cast<uintptr_t>(p.w_dw) & 7) != 0) return false;
    return p.M % (4 * p.W) == 0;
}

// What a kernel's plan function (dh_plan_*) decided for one layer, and all its launch function (dh_launch_*) needs.
// A plan is made only for a layer its kernel takes, shared-memory fit included, so the launch fails only on driver
// or runtime errors.
template <class Params>
struct Plan {
    Params k;                  // kernel parameters
    const dh_packed_w* w;      // packed weights (their tensor maps are encoded at launch)
    int gy;                    // N parts (gridDim.y)
    size_t smem;               // dynamic shared memory per CTA
    bool cluster;              // pairs of N parts run as (1, 2, 1) clusters sharing their A tiles
};
using TcPlan = Plan<TcParams>;
using SepPlan = Plan<SepParams>;
using PatchPlan = Plan<PatchParams>;

// f(std::integral_constant) of the first listed value equal to v, else of the last: turns a plan's run-time selectors
// into the template arguments of a kernel instantiation
template <auto V, auto... Vs, class T, class F>
static inline auto pick(T v, F&& f) {
    if constexpr (sizeof...(Vs) == 0) return f(std::integral_constant<decltype(V), V>{});
    else return v == V ? f(std::integral_constant<decltype(V), V>{}) : pick<Vs...>(v, f);
}

// Persistent grid: one CTA per SM, at most one per M-tile; CTA (x, y) runs M-tiles x, x + gridDim.x, ... of N part y.
static inline int persistent_gx(const dh_ctx* ctx, int gy, int n_mtiles) {
    int gx = ctx->num_sms / gy;
    if (gx < 1) gx = 1;
    if (gx > n_mtiles) gx = n_mtiles;
    return gx;
}

// Persistent launch on the grid of persistent_gx.  Returns 0, or the CUDA error with the message set.
template <auto Kernel, class Params, class... Maps>
static inline int launch_persistent(const char* who, const dh_ctx* ctx, const Plan<Params>& pl, int n_mtiles,
                                    int nthreads, cudaStream_t s, const Maps&... maps) {
    cudaError_t e = ensure_smem<Kernel>(pl.smem);
    if (e == cudaSuccess) {
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3(persistent_gx(ctx, pl.gy, n_mtiles), pl.gy);
        cfg.blockDim = dim3(nthreads);
        cfg.dynamicSmemBytes = pl.smem;
        cfg.stream = s;
        cudaLaunchAttribute at[1];
        if (pl.cluster) {
            at[0].id = cudaLaunchAttributeClusterDimension;
            at[0].val.clusterDim.x = 1; at[0].val.clusterDim.y = 2; at[0].val.clusterDim.z = 1;
            cfg.attrs = at;
            cfg.numAttrs = 1;
        }
        e = cudaLaunchKernelEx(&cfg, Kernel, pl.k, maps...);
    }
    if (e != cudaSuccess) {
        dh_set_error("%s: launch setup failed: %s", who, cudaGetErrorString(e));
        return (int)e;
    }
    return 0;
}

}  // namespace tc

// Plan and launch of each tensor-core convolution kernel.  The plan functions expect packed weights with a hi half.
bool dh_plan_patch(const dh_ctx* ctx, const ConvParams& p, const dh_packed_w* packed, int precision, tc::PatchPlan* pl);
int dh_launch_patch(const dh_ctx* ctx, const tc::PatchPlan& pl, cudaStream_t s);
bool dh_plan_sep_tma(const dh_ctx* ctx, const ConvParams& p, const dh_packed_w* packed, int precision, tc::SepPlan* pl);
int dh_launch_sep_tma(const dh_ctx* ctx, const tc::SepPlan& pl, cudaStream_t s);
bool dh_plan_conv_tc(const dh_ctx* ctx, const ConvParams& p, const dh_packed_w* packed, bool separable, int precision,
                     tc::TcPlan* pl);
int dh_launch_conv_tc(const dh_ctx* ctx, const tc::TcPlan& pl, cudaStream_t s);
