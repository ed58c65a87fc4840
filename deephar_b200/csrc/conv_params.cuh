#pragma once
#include "common.cuh"

struct ConvParams {
    const float* x;
    int N, H, W, Cin, ldx;
    const float* w;      // dense conv: HWIO flattened [K][Cout]; separable: pointwise [Cin][Cout]
    const float* w_dw;   // separable only: (kh,kw,Cin) depthwise taps
    float* out;
    int Ho, Wo, Cout, ldo;
    int kh, kw, sh, sw, pt, pl;
    const float *pre_scale, *pre_shift, *post_scale, *post_shift;
    int pre_relu, post_relu;
    const float* res0; int ldr0;
    const float* res1; int ldr1;
    int up1;   // res1 is (N, Ho/2, Wo/2, Cout), added through a nearest 2x upsampling
    float* pool; int ldp;   // optional second output: 2x2 max-pool of the result (wide pointwise kernel only)
    int M;  // N*Ho*Wo
    int K;  // kh*kw*Cin (dense) ; Cin (pointwise stage)
};

// row of the second residual for output pixel m: the pixel itself, or (fused keras UpSampling2D, reception.py:122-127)
// its source pixel in the half-resolution tensor
__device__ __forceinline__ size_t res1_src(const ConvParams& c, int m) {
    if (!c.up1) return (size_t)m;
    const int hw = c.Ho * c.Wo;
    const int n = m / hw, rem = m - n * hw;
    const int y = rem / c.Wo, x = rem - y * c.Wo;
    return ((size_t)n * (c.Ho >> 1) + (y >> 1)) * (size_t)(c.Wo >> 1) + (size_t)(x >> 1);
}

// Grid of a CUDA-core convolution kernel (dh_conv_plan_info reports it): output pixels per CTA pass (bm), M-tiles of bm
// pixels, CTAs along M and along Cout, output channels per CTA, K-blocks per tile.  The persistent kernels (direct
// small-K, wide pointwise) loop CTA x over M-tiles x, x + grid_x, ...
struct SimtSchedule {
    int bm, n_mtiles, grid_x, grid_y, bn_cta, n_kblocks;
};

int dh_fill_conv_params(ConvParams* p, const dh_view* x, const dh_conv_desc* d, const dh_view* out,
                        int cout, const char* who);
// the direct small-K kernel where dh_conv_smallk_ok(p), else the generic implicit GEMM
void dh_launch_conv_simt(const ConvParams& p, int num_sms, cudaStream_t s);
SimtSchedule dh_conv_simt_schedule(const ConvParams& p, int num_sms);
bool dh_conv_smallk_ok(const ConvParams& p);
// wide pointwise conv with a small reduction (conv_simt.cu), exact fp32
bool dh_pw_smallk_supported(const ConvParams& p);
int dh_launch_pw_smallk(const ConvParams& p, int num_sms, cudaStream_t s);
SimtSchedule dh_pw_smallk_schedule(const ConvParams& p, int num_sms);
void dh_launch_depthwise_simt(const ConvParams& p, float* tmp, int num_sms, cudaStream_t s);

// which kernel served the last convolution (dh_last_conv_path; tests and tools read the numbers)
enum DhConvPath {
    DH_PATH_SIMT = 0,          // CUDA-core kernels (conv_simt.cu): the implicit-GEMM fallback, the direct small-K conv
    DH_PATH_TC = 1,            // wgmma, register producers (conv_tc.cu)
    DH_PATH_SEP_TMA = 2,       // wgmma, TMA-staged separable (conv_sep.cu)
    DH_PATH_PW_SMALLK = 3,     // CUDA-core wide pointwise kernel (conv_simt.cu)
    DH_PATH_PATCH = 4,         // wgmma, TMA-staged dense (conv_patch.cu)
};
