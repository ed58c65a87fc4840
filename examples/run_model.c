/* Run a model exported by deephar_b200's Model.export from C, with no Python in the process.
 *
 *   run_model MODEL.dhm INPUT.f32 OUT_PREFIX [BATCH]
 *
 * INPUT.f32 holds the raw fp32 input of the exported shape (frames or clips x frames, H, W, 3; NHWC), or with BATCH of
 * its first BATCH items (frames, or clips of a clip model; 1 <= BATCH <= the exported batch, dh_model_set_batch).  The
 * program runs one forward, writes each output k raw (fp32, its Keras shape, C order) to OUT_PREFIX.k.f32, then
 * captures the forward into a CUDA graph, clears the outputs, replays the graph and writes them again to
 * OUT_PREFIX.graph.k.f32.
 *
 * Build (from the repository root, after `make -C deephar_b200/csrc`):
 *   gcc -std=c99 -O2 -Iinclude -I/usr/local/cuda/include examples/run_model.c -o run_model \
 *       -Ldeephar_b200 -ldeephar_b200 -L/usr/local/cuda/lib64 -lcudart -Wl,-rpath,$PWD/deephar_b200
 * (or the same line with nvcc in place of gcc, without -std=c99). */
#include <stdio.h>
#include <stdlib.h>

#include <cuda_runtime_api.h>

#include "deephar_b200.h"

static int fail_dh(const char* what, int rc) {
    fprintf(stderr, "%s failed (rc=%d): %s\n", what, rc, dh_last_error());
    return 1;
}

static int fail_cuda(const char* what, cudaError_t e) {
    fprintf(stderr, "%s failed: %s\n", what, cudaGetErrorString(e));
    return 1;
}

#define DH(call)                                  \
    do {                                          \
        int rc_ = (call);                         \
        if (rc_) return fail_dh(#call, rc_);      \
    } while (0)
#define CU(call)                                  \
    do {                                          \
        cudaError_t e_ = (call);                  \
        if (e_ != cudaSuccess) return fail_cuda(#call, e_); \
    } while (0)

/* the view's elements, row by row (a view may be a channel window of a wider buffer: ld >= c) */
static int write_output(const dh_model* m, int k, const char* prefix, const char* tag) {
    dh_view v;
    dh_model_output_info info;
    DH(dh_model_output(m, k, &v, &info));
    size_t rows = (size_t)v.n * v.h * v.w, bytes = rows * v.c * sizeof(float);
    float* host = (float*)malloc(bytes);
    if (!host) return 1;
    CU(cudaMemcpy2D(host, v.c * sizeof(float), v.p, v.ld * sizeof(float), v.c * sizeof(float), rows,
                    cudaMemcpyDeviceToHost));
    char path[4096];
    snprintf(path, sizeof(path), "%s.%s%d.f32", prefix, tag, k);
    FILE* f = fopen(path, "wb");
    int bad = !f || fwrite(host, 1, bytes, f) != bytes;
    if (f) fclose(f);
    free(host);
    if (bad) {
        fprintf(stderr, "cannot write %s\n", path);
        return 1;
    }
    return 0;
}

int main(int argc, char** argv) {
    if (argc != 4 && argc != 5) {
        fprintf(stderr, "usage: %s MODEL.dhm INPUT.f32 OUT_PREFIX [BATCH]\n", argv[0]);
        return 2;
    }
    dh_model_info info;
    DH(dh_model_inspect(argv[1], &info, NULL, 0, NULL, 0));
    printf("%s: %lld launches, %d outputs, %.1f MB of device memory\n", argv[1], (long long)info.n_launches,
           info.n_outputs, info.device_bytes / 1e6);

    dh_ctx* ctx;
    dh_model* m;
    DH(dh_ctx_create(&ctx, 0));
    DH(dh_model_load(ctx, argv[1], &m));
    if (argc == 5) {
        char* end;
        long n = strtol(argv[4], &end, 10);
        if (!*argv[4] || *end || n < 1 || n > info.clip_items) {
            fprintf(stderr, "BATCH: an integer in [1, %d] expected, got %s\n", info.clip_items, argv[4]);
            return 2;
        }
        DH(dh_model_set_batch(m, (int)n));
        printf("batch %d of %d\n", dh_model_batch(m), info.clip_items);
    }

    /* the input: read it whole, copy it into the model's input view */
    dh_view in;
    DH(dh_model_input(m, &in));
    size_t in_bytes = (size_t)in.n * in.h * in.w * in.c * sizeof(float);
    float* x = (float*)malloc(in_bytes);
    FILE* f = fopen(argv[2], "rb");
    if (!x || !f || fread(x, 1, in_bytes, f) != in_bytes || fgetc(f) != EOF) {
        fprintf(stderr, "%s: expected %zu bytes of fp32 input\n", argv[2], in_bytes);
        return 1;
    }
    fclose(f);
    CU(cudaMemcpy(in.p, x, in_bytes, cudaMemcpyHostToDevice));
    free(x);

    cudaStream_t stream;
    CU(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
    DH(dh_model_forward(m, stream));
    CU(cudaStreamSynchronize(stream));
    for (int k = 0; k < info.n_outputs; ++k)
        if (write_output(m, k, argv[3], "")) return 1;

    /* the same forward as a CUDA graph: capture, clear the outputs, replay */
    cudaGraph_t graph;
    cudaGraphExec_t exec;
    CU(cudaStreamBeginCapture(stream, cudaStreamCaptureModeThreadLocal));
    DH(dh_model_forward(m, stream));
    CU(cudaStreamEndCapture(stream, &graph));
    CU(cudaGraphInstantiate(&exec, graph, 0));
    for (int k = 0; k < info.n_outputs; ++k) {
        dh_view v;
        DH(dh_model_output(m, k, &v, NULL));
        CU(cudaMemset2DAsync(v.p, v.ld * sizeof(float), 0, v.c * sizeof(float), (size_t)v.n * v.h * v.w, stream));
    }
    CU(cudaGraphLaunch(exec, stream));
    CU(cudaStreamSynchronize(stream));
    for (int k = 0; k < info.n_outputs; ++k)
        if (write_output(m, k, argv[3], "graph.")) return 1;

    CU(cudaGraphExecDestroy(exec));
    CU(cudaGraphDestroy(graph));
    CU(cudaStreamDestroy(stream));
    DH(dh_model_free(m));
    DH(dh_ctx_destroy(ctx));
    printf("ok\n");
    return 0;
}
