// extern "C" entry points for the convolutions: argument checking + dispatch between
// the wgmma tensor-core kernels (conv_tc.cu, conv_sep.cu, conv_patch.cu) and the CUDA-core kernels (conv_simt.cu).
#include "tc_common.cuh"

extern "C" int dh_conv2d_f32(dh_ctx* ctx, const dh_view* x, const float* w_hwio,
                             const dh_packed_w* packed, const dh_conv_desc* d, const dh_view* out,
                             void* stream) {
    DH_CHECK_ARG(ctx && w_hwio, "dh_conv2d_f32: NULL ctx or weights");
    ConvParams p;
    int rc = dh_fill_conv_params(&p, x, d, out, out ? out->c : 0, "dh_conv2d_f32");
    if (rc) return rc;
    p.w = w_hwio;
    cudaStream_t s = (cudaStream_t)stream;
    if (!p.up1 && dh_conv_smallk_ok(p)) {          // the 3x3x3 first conv of the stem: direct small-K kernel (conv_simt.cu)
        ctx->last_conv_path = DH_PATH_SIMT;
        dh_launch_conv_simt(p, s);
        DH_LAUNCH_EPILOGUE(ctx, 1);
    }
    if (ctx->pw_smallk && !p.up1 && dh_pw_smallk_supported(p)) {
        rc = dh_launch_pw_smallk(p, ctx->num_sms, s);
        if (rc) return rc;
        ctx->last_conv_path = DH_PATH_PW_SMALLK;
        DH_LAUNCH_EPILOGUE(ctx, 1);
    }
    DH_CHECK_ARG(!p.pool, "dh_conv2d_f32: pool_out is written by the wide pointwise kernel only (1x1, stride 1, Cin <= 64, "
                          "Cout >= 128, Wo == 32, even Ho); this layer is not one");
    if (packed && packed->hi) {
        tc::PatchPlan pp;
        if (dh_plan_patch(ctx, p, packed, d->precision, &pp)) {
            rc = dh_launch_patch(ctx, pp, s);
            if (rc) return rc;
            ctx->last_conv_path = DH_PATH_PATCH;
            DH_LAUNCH_EPILOGUE(ctx, 1);
        }
        tc::TcPlan tp;
        if (dh_plan_conv_tc(ctx, p, packed, false, d->precision, &tp)) {
            rc = dh_launch_conv_tc(ctx, tp, s);
            if (rc) return rc;
            ctx->last_conv_path = DH_PATH_TC;
            DH_LAUNCH_EPILOGUE(ctx, 1);
        }
    }
    DH_CHECK_ARG(!p.up1, "dh_conv2d_f32: an upsampled residual needs a tensor-core kernel; none takes this shape");
    ctx->last_conv_path = DH_PATH_SIMT;
    if (!dh_conv_smallk_ok(p)) ctx->fallbacks += 1;      // the direct K <= 32 kernel is a specialised path, not a fallback
    dh_launch_conv_simt(p, s);
    DH_LAUNCH_EPILOGUE(ctx, 1);
}

extern "C" int dh_sepconv2d_f32(dh_ctx* ctx, const dh_view* x, const float* w_dw, const float* w_pw,
                                const dh_packed_w* packed_pw, const dh_conv_desc* d,
                                const dh_view* out, void* stream) {
    DH_CHECK_ARG(ctx && w_dw && w_pw, "dh_sepconv2d_f32: NULL ctx or weights");
    ConvParams p;
    int rc = dh_fill_conv_params(&p, x, d, out, out ? out->c : 0, "dh_sepconv2d_f32");
    if (rc) return rc;
    p.w = w_pw;
    p.w_dw = w_dw;
    DH_CHECK_ARG(!p.pool, "dh_sepconv2d_f32: pool_out is not supported by the separable kernels");
    cudaStream_t s = (cudaStream_t)stream;
    if (packed_pw && packed_pw->hi) {
        tc::SepPlan sp;
        if (dh_plan_sep_tma(ctx, p, packed_pw, d->precision, &sp)) {
            rc = dh_launch_sep_tma(ctx, sp, s);
            if (rc) return rc;
            ctx->last_conv_path = DH_PATH_SEP_TMA;
            DH_LAUNCH_EPILOGUE(ctx, 1);
        }
        tc::TcPlan tp;
        if (dh_plan_conv_tc(ctx, p, packed_pw, true, d->precision, &tp)) {
            rc = dh_launch_conv_tc(ctx, tp, s);
            if (rc) return rc;
            ctx->last_conv_path = DH_PATH_TC;
            DH_LAUNCH_EPILOGUE(ctx, 1);
        }
    }
    DH_CHECK_ARG(!p.up1, "dh_sepconv2d_f32: an upsampled residual needs a tensor-core kernel; none takes this shape");
    ctx->last_conv_path = DH_PATH_SIMT;
    ctx->fallbacks += 1;
    // Two-kernel CUDA-core path: depthwise (with the fused pre-ops) into the caller's
    // workspace, then the pointwise 1x1 as an implicit GEMM with the fused post-ops.
    int64_t need = (int64_t)p.M * p.Cin * (int64_t)sizeof(float);
    DH_CHECK_ARG(ctx->workspace && ctx->workspace_bytes >= need,
                 "dh_sepconv2d_f32: workspace too small (%lld needed, %lld set via dh_set_workspace)",
                 (long long)need, (long long)ctx->workspace_bytes);
    float* tmp = (float*)ctx->workspace;
    dh_launch_depthwise_simt(p, tmp, ctx->num_sms, s);
    ConvParams q = p;
    q.x = tmp; q.N = p.N; q.H = p.Ho; q.W = p.Wo; q.ldx = p.Cin;
    q.kh = q.kw = 1; q.sh = q.sw = 1; q.pt = q.pl = 0;
    q.pre_scale = q.pre_shift = nullptr; q.pre_relu = 0;
    q.K = p.Cin;
    dh_launch_conv_simt(q, s);
    DH_LAUNCH_EPILOGUE(ctx, 2);
}
