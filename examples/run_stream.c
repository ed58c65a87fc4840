/* Run live video through a clip stream exported by deephar_b200's ClipStream.export from C, with no Python in the process.
 *
 *   run_stream STREAM.dhs FRAMES.f32 OUT_PREFIX [RESETS.txt]
 *
 * FRAMES.f32 holds n_push batches of one raw fp32 frame per stream: (n_push, S, H, W, 3), NHWC.  RESETS.txt (optional)
 * has one line per reset, "PUSH ID ...": before push PUSH (0-based), streams ID ... start a new video; a line with PUSH
 * alone restarts every stream.  The program pushes each batch and appends, per push, output k (frame outputs first,
 * then clip outputs; fp32, C order) to OUT_PREFIX.k.f32 and the S int32 ready flags to OUT_PREFIX.ready.i32.  It then
 * loads the file again and runs the same frames with the first push plain and every later push a replay of one push
 * captured into a CUDA graph, writing OUT_PREFIX.graph.k.f32 and OUT_PREFIX.graph.ready.i32.
 *
 * Build (from the repository root, after `make -C deephar_b200/csrc`):
 *   gcc -std=c99 -O2 -Iinclude -I/usr/local/cuda/include examples/run_stream.c -o run_stream \
 *       -Ldeephar_b200 -ldeephar_b200 -L/usr/local/cuda/lib64 -lcudart -Wl,-rpath,$PWD/deephar_b200 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

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

/* one reset: before push `push`, streams ids[0..n) (n = 0: all) */
typedef struct {
    int push, n;
    int32_t ids[64];
} reset_t;

static int read_resets(const char* path, reset_t* resets, int max, int* count) {
    FILE* f = fopen(path, "r");
    char line[1024];
    *count = 0;
    if (!f) {
        fprintf(stderr, "cannot open %s\n", path);
        return 1;
    }
    while (fgets(line, sizeof(line), f)) {
        char* p = line;
        char* end;
        long v = strtol(p, &end, 10);
        if (end == p) continue;                     /* blank line */
        if (*count == max) {
            fprintf(stderr, "%s: more than %d resets\n", path, max);
            fclose(f);
            return 1;
        }
        reset_t* r = &resets[(*count)++];
        r->push = (int)v;
        r->n = 0;
        for (p = end; r->n < 64; p = end) {
            v = strtol(p, &end, 10);
            if (end == p) break;
            r->ids[r->n++] = (int32_t)v;
        }
    }
    fclose(f);
    return 0;
}

/* append the view's elements, row by row (a view may be a channel window of a wider buffer: ld >= c) */
static int append(const char* prefix, const char* tag, const char* name, const void* dev, size_t rows, size_t row_bytes,
                  size_t pitch, int first) {
    char path[4096];
    void* host = malloc(rows * row_bytes);
    if (!host) return 1;
    CU(cudaMemcpy2D(host, row_bytes, dev, pitch, row_bytes, rows, cudaMemcpyDeviceToHost));
    snprintf(path, sizeof(path), "%s.%s%s", prefix, tag, name);
    FILE* f = fopen(path, first ? "wb" : "ab");
    int bad = !f || fwrite(host, 1, rows * row_bytes, f) != rows * row_bytes;
    if (f) fclose(f);
    free(host);
    if (bad) {
        fprintf(stderr, "cannot write %s\n", path);
        return 1;
    }
    return 0;
}

static int write_push(const dh_stream* st, const dh_stream_info* info, const char* prefix, const char* tag, int first) {
    char name[64];
    int n_out = info->n_frame_outputs + info->n_clip_outputs;
    for (int k = 0; k < n_out; ++k) {
        dh_view v;
        DH(dh_stream_output(st, k, &v, NULL));
        snprintf(name, sizeof(name), "%d.f32", k);
        if (append(prefix, tag, name, v.p, (size_t)v.n * v.h * v.w, v.c * sizeof(float), v.ld * sizeof(float), first))
            return 1;
    }
    const int32_t* ready;
    DH(dh_stream_ready(st, &ready));
    return append(prefix, tag, "ready.i32", ready, 1, info->n_streams * sizeof(int32_t),
                  info->n_streams * sizeof(int32_t), first);
}

/* one run over every frame batch: graph = 0 plain pushes, 1 push 0 plain and later pushes replayed from a graph */
static int run(dh_ctx* ctx, const char* path, const dh_stream_info* info, const float* frames, int n_push,
               const reset_t* resets, int n_resets, const char* prefix, int graph) {
    dh_stream* st;
    dh_view in;
    cudaStream_t stream;
    cudaGraph_t g = NULL;
    cudaGraphExec_t exec = NULL;
    DH(dh_stream_load(ctx, path, &st));
    DH(dh_stream_input(st, &in));
    CU(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
    size_t frame_bytes = (size_t)in.n * in.h * in.w * in.c * sizeof(float);
    for (int i = 0; i < n_push; ++i) {
        for (int r = 0; r < n_resets; ++r)
            if (resets[r].push == i) DH(dh_stream_reset(st, resets[r].n ? resets[r].ids : NULL, resets[r].n, stream));
        CU(cudaMemcpyAsync(in.p, (const char*)frames + i * frame_bytes, frame_bytes, cudaMemcpyHostToDevice, stream));
        if (graph && i == 1) {               /* capture one push; it runs when the graph is launched */
            CU(cudaStreamBeginCapture(stream, cudaStreamCaptureModeThreadLocal));
            DH(dh_stream_push(st, stream));
            CU(cudaStreamEndCapture(stream, &g));
            CU(cudaGraphInstantiate(&exec, g, 0));
        }
        if (exec)
            CU(cudaGraphLaunch(exec, stream));
        else
            DH(dh_stream_push(st, stream));
        CU(cudaStreamSynchronize(stream));
        if (write_push(st, info, prefix, graph ? "graph." : "", i == 0)) return 1;
    }
    if (exec) {
        CU(cudaGraphExecDestroy(exec));
        CU(cudaGraphDestroy(g));
    }
    CU(cudaStreamDestroy(stream));
    DH(dh_stream_free(st));
    return 0;
}

int main(int argc, char** argv) {
    if (argc != 4 && argc != 5) {
        fprintf(stderr, "usage: %s STREAM.dhs FRAMES.f32 OUT_PREFIX [RESETS.txt]\n", argv[0]);
        return 2;
    }
    dh_stream_info info;
    DH(dh_stream_inspect(argv[1], &info, NULL, 0));
    printf("%s: %d streams, T = %d, %lld + 2 + %lld launches per push, %.1f MB of device memory\n", argv[1],
           info.n_streams, info.frames_per_clip, (long long)info.n_frame_launches, (long long)info.n_clip_launches,
           info.device_bytes / 1e6);

    static reset_t resets[256];
    int n_resets = 0;
    if (argc == 5 && read_resets(argv[4], resets, 256, &n_resets)) return 1;

    /* the frames: read them whole */
    size_t frame_bytes = sizeof(float);
    for (int i = 0; i < info.input_rank; ++i) frame_bytes *= (size_t)info.input_shape[i];
    FILE* f = fopen(argv[2], "rb");
    if (!f) {
        fprintf(stderr, "cannot open %s\n", argv[2]);
        return 1;
    }
    fseek(f, 0, SEEK_END);
    long size = ftell(f);
    fseek(f, 0, SEEK_SET);
    if (size <= 0 || size % frame_bytes) {
        fprintf(stderr, "%s: %ld bytes is not a whole number of %zu-byte frame batches\n", argv[2], size, frame_bytes);
        return 1;
    }
    int n_push = (int)(size / frame_bytes);
    float* frames = (float*)malloc(size);
    if (!frames || fread(frames, 1, size, f) != (size_t)size) {
        fprintf(stderr, "%s: read error\n", argv[2]);
        return 1;
    }
    fclose(f);

    dh_ctx* ctx;
    DH(dh_ctx_create(&ctx, 0));
    for (int graph = 0; graph < 2; ++graph)
        if (run(ctx, argv[1], &info, frames, n_push, resets, n_resets, argv[3], graph)) return 1;
    free(frames);
    DH(dh_ctx_destroy(ctx));
    printf("ok: %d pushes\n", n_push);
    return 0;
}
