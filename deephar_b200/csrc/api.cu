// Context, error reporting and version of the C ABI (include/deephar_b200.h).
#include <stdarg.h>
#include <string.h>
#include "common.cuh"

static thread_local char g_last_error[512] = "";

void dh_set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_last_error, sizeof(g_last_error), fmt, ap);
    va_end(ap);
}

extern "C" const char* dh_last_error(void) { return g_last_error; }

extern "C" int dh_version(void) { return 100; }

extern "C" int dh_ctx_create(dh_ctx** out, int device) {
    DH_CHECK_ARG(out != nullptr, "dh_ctx_create: out is NULL");
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count == 0) {
        dh_set_error("dh_ctx_create: no CUDA device (%s) -- this library has no CPU fallback",
                     cudaGetErrorString(e));
        return e == cudaSuccess ? (int)cudaErrorNoDevice : (int)e;
    }
    DH_CHECK_ARG(device >= 0 && device < count, "dh_ctx_create: device %d out of range", device);
    cudaDeviceProp prop;
    e = cudaGetDeviceProperties(&prop, device);
    if (e != cudaSuccess) {
        dh_set_error("cudaGetDeviceProperties: %s", cudaGetErrorString(e));
        return (int)e;
    }
    if (prop.major != 9 || prop.minor != 0) {
        dh_set_error("dh_ctx_create: device %d is sm_%d%d; this build targets sm_90a (H100) only",
                     device, prop.major, prop.minor);
        return -2;
    }
    dh_ctx* c = new dh_ctx();
    c->device = device;
    c->num_sms = prop.multiProcessorCount;
    c->launches = 0;
    c->workspace = nullptr;
    c->workspace_bytes = 0;
    c->last_conv_path = 0;
    c->share_a = 1;
    c->sep_tma = 1;
    c->dbg = 0;
    c->pw_smallk = 1;
    c->dense_patch = 1;
    c->sam3d_stream = 1;
    c->fallbacks = 0;
    c->comm = nullptr;
    c->comm_rank = -1;
    c->comm_world = 0;
    *out = c;
    return 0;
}

extern "C" int dh_comm_destroy(dh_ctx* ctx);

extern "C" int dh_ctx_destroy(dh_ctx* ctx) {
    if (ctx && ctx->comm) dh_comm_destroy(ctx);
    delete ctx;
    return 0;
}

extern "C" int64_t dh_launch_count(dh_ctx* ctx, int reset) {
    if (!ctx) return -1;
    int64_t v = ctx->launches;
    if (reset) ctx->launches = 0;
    return v;
}

extern "C" int dh_set_option(dh_ctx* ctx, const char* name, int value) {
    DH_CHECK_ARG(ctx && name, "dh_set_option: NULL argument");
    if (!strcmp(name, "share_a")) { ctx->share_a = value; return 0; }
    if (!strcmp(name, "sep_tma")) { ctx->sep_tma = value; return 0; }
#ifdef DH_ABLATE
    if (!strcmp(name, "dbg")) { ctx->dbg = value; return 0; }      // tools/ builds only (make ABLATE=1)
#endif
    if (!strcmp(name, "pw_smallk")) { ctx->pw_smallk = value; return 0; }
    if (!strcmp(name, "dense_patch")) { ctx->dense_patch = value; return 0; }
    if (!strcmp(name, "sam3d_stream")) { ctx->sam3d_stream = value; return 0; }
    dh_set_error("dh_set_option: unknown option %s", name);
    return -1;
}

extern "C" int dh_last_conv_path(dh_ctx* ctx) { return ctx ? ctx->last_conv_path : -1; }

extern "C" int64_t dh_fallback_count(dh_ctx* ctx, int reset) {
    if (!ctx) return -1;
    int64_t v = ctx->fallbacks;
    if (reset) ctx->fallbacks = 0;
    return v;
}

extern "C" int dh_set_workspace(dh_ctx* ctx, void* ptr, int64_t bytes) {
    DH_CHECK_ARG(ctx != nullptr, "dh_set_workspace: ctx is NULL");
    ctx->workspace = ptr;
    ctx->workspace_bytes = bytes;
    return 0;
}
