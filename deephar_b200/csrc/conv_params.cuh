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

// TMA-staged fused separable kernel (conv_sep.cu)
bool dh_sep_tma_supported(const dh_ctx* ctx, const ConvParams& p, const dh_packed_w* packed);
int dh_launch_sep_tma(dh_ctx* ctx, const ConvParams& p, const dh_packed_w* packed, int precision, cudaStream_t s);

// TMA-staged patch kernel for stride-1 Conv2D (conv_patch.cu)
bool dh_patch_supported(const dh_ctx* ctx, const ConvParams& p, const dh_packed_w* packed);
int dh_launch_patch(dh_ctx* ctx, const ConvParams& p, const dh_packed_w* packed, int precision, cudaStream_t s);

// tensor-core path (conv_tc.cu). Returns true if it took the op.
bool dh_tc_supported(const ConvParams& p, const dh_packed_w* packed, bool separable);
int dh_launch_conv_tc(dh_ctx* ctx, const ConvParams& p, const dh_packed_w* packed, bool separable,
                      int precision, cudaStream_t s);
