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
    int up1;   // res1 is (N, Ho/2, Wo/2, Cout), added through a nearest 2x upsampling (tensor-core epilogues only)
    float* pool; int ldp;   // optional second output: 2x2 max-pool of the result (wide pointwise kernel only)
    int M;  // N*Ho*Wo
    int K;  // kh*kw*Cin (dense) ; Cin (pointwise stage)
};

int dh_fill_conv_params(ConvParams* p, const dh_view* x, const dh_conv_desc* d, const dh_view* out,
                        int cout, const char* who);
void dh_launch_conv_simt(const ConvParams& p, cudaStream_t s);
bool dh_conv_smallk_ok(const ConvParams& p);
// wide pointwise conv with a small reduction (conv_simt.cu), exact fp32
bool dh_pw_smallk_supported(const ConvParams& p);
int dh_launch_pw_smallk(const ConvParams& p, int num_sms, cudaStream_t s);
void dh_launch_depthwise_simt(const ConvParams& p, float* tmp, int num_sms, cudaStream_t s);

// which kernel served the last convolution (dh_last_conv_path; tests and tools read the numbers)
enum DhConvPath {
    DH_PATH_SIMT = 0,          // CUDA-core kernels (conv_simt.cu): the implicit-GEMM fallback, the direct small-K conv
    DH_PATH_TC = 1,            // wgmma, register producers (conv_tc.cu)
    DH_PATH_SEP_TMA = 2,       // wgmma, TMA-staged separable (conv_sep.cu)
    DH_PATH_PW_SMALLK = 3,     // CUDA-core wide pointwise kernel (conv_simt.cu)
    DH_PATH_PATCH = 4,         // wgmma, TMA-staged dense (conv_patch.cu)
};
