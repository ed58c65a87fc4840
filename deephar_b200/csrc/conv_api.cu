// extern "C" entry points for the convolutions: argument checking, the choice between the wgmma tensor-core kernels
// (conv_tc.cu, conv_sep.cu, conv_patch.cu) and the CUDA-core kernels (conv_simt.cu), and its launch.
#include "tc_common.cuh"

namespace {

// The kernel that runs one convolution, and all its launch needs.
struct Choice {
    DhConvPath path;
    bool fallback;             // the generic CUDA-core kernel: counted by dh_fallback_count
    int64_t workspace_bytes;   // caller's workspace the launch needs
    tc::PatchPlan patch;       // the plan of the chosen tensor-core kernel
    tc::SepPlan sep;
    tc::TcPlan tcp;
};

// The one place that decides which kernel runs a convolution.  Conv2D: direct small-K, wide pointwise, conv_patch.cu,
// conv_tc.cu, the generic CUDA-core kernel; SeparableConv2D: conv_sep.cu, conv_tc.cu, the two-kernel CUDA-core path.
// No side effects.  Returns 0, or < 0 with the error set for a call no kernel may take.
int choose_conv(const dh_ctx* ctx, const ConvParams& p, const dh_packed_w* packed, bool separable, int precision,
                Choice* c) {
    const bool packed_hi = packed && packed->hi;
    c->fallback = false;
    c->workspace_bytes = 0;
    if (separable) {
        DH_CHECK_ARG(!p.pool, "dh_sepconv2d_f32: pool_out is not supported by the separable kernels");
        if (packed_hi && dh_plan_sep_tma(ctx, p, packed, precision, &c->sep)) { c->path = DH_PATH_SEP_TMA; return 0; }
    } else {
        // the 3x3x3 first conv of the stem: direct small-K kernel (conv_simt.cu), a specialised path, not a fallback.
        // It writes no pooled output, so a call with pool_out goes on to the check below.
        if (!p.up1 && !p.pool && dh_conv_smallk_ok(p)) { c->path = DH_PATH_SIMT; return 0; }
        if (ctx->pw_smallk && !p.up1 && dh_pw_smallk_supported(p)) { c->path = DH_PATH_PW_SMALLK; return 0; }
        DH_CHECK_ARG(!p.pool, "dh_conv2d_f32: pool_out is written by the wide pointwise kernel only (1x1, stride 1, "
                              "Cin <= 64, Cout >= 128, Wo == 32, even Ho); this layer is not one");
        if (packed_hi && dh_plan_patch(ctx, p, packed, precision, &c->patch)) { c->path = DH_PATH_PATCH; return 0; }
    }
    if (packed_hi && dh_plan_conv_tc(ctx, p, packed, separable, precision, &c->tcp)) { c->path = DH_PATH_TC; return 0; }
    c->path = DH_PATH_SIMT;
    c->fallback = true;
    // the two-kernel separable path keeps the depthwise output in the workspace
    if (separable) c->workspace_bytes = (int64_t)p.M * p.Cin * (int64_t)sizeof(float);
    return 0;
}

// Argument checks and parameters of a Conv2D (w_dw == nullptr) or SeparableConv2D call, and its choice.
int plan_conv(const dh_ctx* ctx, const dh_view* x, const float* w_dw, const float* w, const dh_packed_w* packed,
              const dh_conv_desc* d, const dh_view* out, bool separable, ConvParams* p, Choice* c) {
    const char* who = separable ? "dh_sepconv2d_f32" : "dh_conv2d_f32";
    DH_CHECK_ARG(ctx && w && (w_dw || !separable), "%s: NULL ctx or weights", who);
    int rc = dh_fill_conv_params(p, x, d, out, out ? out->c : 0, who);
    if (rc) return rc;
    p->w = w;
    p->w_dw = w_dw;
    return choose_conv(ctx, *p, packed, separable, d->precision, c);
}

// The pointwise stage of the two-kernel CUDA-core separable path: a 1x1 implicit GEMM over the depthwise output `tmp`
// (M x Cin, dense), with the fused post-ops (and residuals) of the layer.
ConvParams pointwise_stage(const ConvParams& p, float* tmp) {
    ConvParams q = p;
    q.x = tmp; q.H = p.Ho; q.W = p.Wo; q.ldx = p.Cin;
    q.kh = q.kw = 1; q.sh = q.sw = 1; q.pt = q.pl = 0;
    q.pre_scale = q.pre_shift = nullptr; q.pre_relu = 0;
    q.K = p.Cin;
    return q;
}

int launch_choice(dh_ctx* ctx, const ConvParams& p, const Choice& c, bool separable, cudaStream_t s) {
    // a refused call launches nothing and leaves the counters and dh_last_conv_path as they were
    DH_CHECK_ARG(c.workspace_bytes == 0 || (ctx->workspace && ctx->workspace_bytes >= c.workspace_bytes),
                 "dh_sepconv2d_f32: workspace too small (%lld needed, %lld set via dh_set_workspace)",
                 (long long)c.workspace_bytes, (long long)ctx->workspace_bytes);
    int rc = 0;
    switch (c.path) {
    case DH_PATH_TC: rc = dh_launch_conv_tc(ctx, c.tcp, s); break;
    case DH_PATH_SEP_TMA: rc = dh_launch_sep_tma(ctx, c.sep, s); break;
    case DH_PATH_PATCH: rc = dh_launch_patch(ctx, c.patch, s); break;
    case DH_PATH_PW_SMALLK: rc = dh_launch_pw_smallk(p, ctx->num_sms, s); break;
    case DH_PATH_SIMT: break;
    }
    if (rc) return rc;
    ctx->last_conv_path = c.path;
    ctx->fallbacks += c.fallback;
    if (c.path != DH_PATH_SIMT) DH_LAUNCH_EPILOGUE(ctx, 1);
    if (!separable) {
        dh_launch_conv_simt(p, ctx->num_sms, s);
        DH_LAUNCH_EPILOGUE(ctx, 1);
    }
    // Two-kernel CUDA-core path: depthwise (with the fused pre-ops) into the caller's
    // workspace, then the pointwise 1x1 as an implicit GEMM with the fused post-ops.
    float* tmp = (float*)ctx->workspace;
    dh_launch_depthwise_simt(p, tmp, ctx->num_sms, s);
    dh_launch_conv_simt(pointwise_stage(p, tmp), ctx->num_sms, s);
    DH_LAUNCH_EPILOGUE(ctx, 2);
}

template <class Params>
void tc_info(const dh_ctx* ctx, const tc::Plan<Params>& pl, const tc::TcParams& P, dh_conv_plan_info* info) {
    info->n_mtiles = P.n_mtiles;
    info->grid_x = tc::persistent_gx(ctx, pl.gy, P.n_mtiles);
    info->grid_y = pl.gy;
    info->bn_cta = P.bn_cta;
    info->n_kblocks = P.n_kblocks;
    info->cluster = pl.cluster;
    info->bm = tc::BM;
}

// the CUDA-core kernels' grids (paths 0 and 3): for the two-kernel separable path, its pointwise GEMM's
void simt_info(const SimtSchedule& g, dh_conv_plan_info* info) {
    info->bm = g.bm;
    info->n_mtiles = g.n_mtiles;
    info->grid_x = g.grid_x;
    info->grid_y = g.grid_y;
    info->bn_cta = g.bn_cta;
    info->n_kblocks = g.n_kblocks;
}

int plan_info(const dh_ctx* ctx, const ConvParams& p, bool separable, const Choice& c, dh_conv_plan_info* info) {
    DH_CHECK_ARG(info, "dh_conv_plan_info: NULL info");
    *info = dh_conv_plan_info{};
    info->path = c.path;
    info->fallback = c.fallback;
    info->workspace_bytes = c.workspace_bytes;
    if (c.path == DH_PATH_TC) {
        tc_info(ctx, c.tcp, c.tcp.k, info);
        info->stages = c.tcp.k.stages;
    }
    if (c.path == DH_PATH_SEP_TMA) {
        tc_info(ctx, c.sep, c.sep.k.t, info);
        info->bm = c.sep.k.bm;
        info->epi_tma = c.sep.k.epi_smem > 0;
    }
    if (c.path == DH_PATH_PATCH) tc_info(ctx, c.patch, c.patch.k.t, info);
    if (c.path == DH_PATH_PW_SMALLK) simt_info(dh_pw_smallk_schedule(p, ctx->num_sms), info);
    if (c.path == DH_PATH_SIMT)
        simt_info(dh_conv_simt_schedule(separable ? pointwise_stage(p, nullptr) : p, ctx->num_sms), info);
    return 0;
}

}  // namespace

extern "C" int dh_conv2d_f32(dh_ctx* ctx, const dh_view* x, const float* w_hwio,
                             const dh_packed_w* packed, const dh_conv_desc* d, const dh_view* out,
                             void* stream) {
    ConvParams p;
    Choice c;
    int rc = plan_conv(ctx, x, nullptr, w_hwio, packed, d, out, false, &p, &c);
    return rc ? rc : launch_choice(ctx, p, c, false, (cudaStream_t)stream);
}

extern "C" int dh_sepconv2d_f32(dh_ctx* ctx, const dh_view* x, const float* w_dw, const float* w_pw,
                                const dh_packed_w* packed_pw, const dh_conv_desc* d,
                                const dh_view* out, void* stream) {
    ConvParams p;
    Choice c;
    int rc = plan_conv(ctx, x, w_dw, w_pw, packed_pw, d, out, true, &p, &c);
    return rc ? rc : launch_choice(ctx, p, c, true, (cudaStream_t)stream);
}

extern "C" int dh_conv2d_plan(dh_ctx* ctx, const dh_view* x, const float* w_hwio, const dh_packed_w* packed,
                              const dh_conv_desc* d, const dh_view* out, dh_conv_plan_info* info) {
    ConvParams p;
    Choice c;
    int rc = plan_conv(ctx, x, nullptr, w_hwio, packed, d, out, false, &p, &c);
    return rc ? rc : plan_info(ctx, p, false, c, info);
}

extern "C" int dh_sepconv2d_plan(dh_ctx* ctx, const dh_view* x, const float* w_dw, const float* w_pw,
                                 const dh_packed_w* packed_pw, const dh_conv_desc* d, const dh_view* out,
                                 dh_conv_plan_info* info) {
    ConvParams p;
    Choice c;
    int rc = plan_conv(ctx, x, w_dw, w_pw, packed_pw, d, out, true, &p, &c);
    return rc ? rc : plan_info(ctx, p, true, c, info);
}
