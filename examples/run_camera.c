/* Run live video from camera-sized frames through a clip stream exported by deephar_b200's ClipStream.export, from C
 * with no Python in the process: each push crops and resizes the new frames on the device (dh_prepare_frames_u8),
 * advances the streams (dh_stream_push) and maps the pushed frames' poses back to image pixels (dh_pose_to_image_f32).
 *
 *   run_camera STREAM.dhs FRAMES.u8 H W BOXES.f64 MAX_CROP_W MAX_CROP_H OUT_PREFIX [RESETS.txt]
 *
 * FRAMES.u8 holds n_push batches of one raw RGB frame per stream: uint8 (n_push, S, H, W, 3).  BOXES.f64 holds one box
 * per frame: double (n_push, S, 5) = (centre x, centre y, window width, window height, hflip), in image pixels.
 * MAX_CROP_W / MAX_CROP_H bound the windows (a larger one is flagged and its frame is NaN).  RESETS.txt as for
 * run_stream: lines "PUSH ID ...", before push PUSH streams ID ... start a new video (PUSH alone: every stream).
 * Per push the program appends to
 *   OUT_PREFIX.k.f32          output k of the stream (frame outputs first, then clip outputs; fp32, C order)
 *   OUT_PREFIX.pose.f64       frame output 0 -- the pose of the frame just pushed -- in image pixels, (S, points, 2)
 *   OUT_PREFIX.ready.i32      the S ready flags
 *   OUT_PREFIX.status.i32     the S frame status words of dh_prepare_frames_u8
 * It runs the video once with plain calls, then again from a fresh load with prepare + push captured into one CUDA
 * graph (the box upload from a pinned buffer included) and replayed for every push, writing OUT_PREFIX.graph.*.
 * Copying the frames to the device stands in for a decoder that writes them there.
 *
 * Build (from the repository root, after `make -C deephar_b200/csrc`):
 *   gcc -std=c99 -O2 -Iinclude -I/usr/local/cuda/include examples/run_camera.c -o run_camera \
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
        if (end == p) continue;
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

static void* read_all(const char* path, size_t unit, size_t* count) {
    FILE* f = fopen(path, "rb");
    if (!f) {
        fprintf(stderr, "cannot open %s\n", path);
        return NULL;
    }
    fseek(f, 0, SEEK_END);
    long size = ftell(f);
    fseek(f, 0, SEEK_SET);
    void* p = size > 0 && size % unit == 0 ? malloc(size) : NULL;
    if (!p || fread(p, 1, size, f) != (size_t)size) {
        fprintf(stderr, "%s: %ld bytes is not a whole number of %zu-byte pushes\n", path, size, unit);
        free(p);
        fclose(f);
        return NULL;
    }
    fclose(f);
    *count = size / unit;
    return p;
}

/* append rows of row_bytes, pitch bytes apart, from device memory */
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

typedef struct {
    const char* path;
    const uint8_t* frames;        /* host (n_push, S, H, W, 3) */
    const double* boxes;          /* host (n_push, S, 5) */
    int n_push, S, H, W, max_crop_w, max_crop_h;
    const reset_t* resets;
    int n_resets;
    const char* prefix;
} job_t;

static int run(dh_ctx* ctx, const job_t* job, int graph) {
    const int S = job->S;
    const size_t frame_bytes = (size_t)job->H * job->W * 3;
    const char* tag = graph ? "graph." : "";
    dh_stream* st;
    dh_stream_info info;
    dh_view in, pose;
    cudaStream_t stream;
    cudaGraph_t g = NULL;
    cudaGraphExec_t exec = NULL;
    DH(dh_stream_inspect(job->path, &info, NULL, 0));
    if (info.n_frame_outputs < 1) {
        fprintf(stderr, "%s: the stream has no frame output to map\n", job->path);
        return 1;
    }
    DH(dh_stream_load(ctx, job->path, &st));
    DH(dh_stream_input(st, &in));
    DH(dh_stream_output(st, 0, &pose, NULL));
    const int64_t points = (int64_t)pose.h * pose.w;
    const int64_t ws_bytes = dh_prepare_frames_workspace(S, job->max_crop_w, job->max_crop_h, in.h, in.w);
    if (ws_bytes < 0) return fail_dh("dh_prepare_frames_workspace", -1);
    CU(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
    /* device: the images, the box records, the workspace, afmat, status, the image-space poses; host: pinned records */
    uint8_t *images, *ws;
    dh_frame_box *boxes_dev, *boxes_host;
    double *afmat, *pose_img;
    int32_t* status;
    CU(cudaMalloc((void**)&images, S * frame_bytes));
    CU(cudaMalloc((void**)&boxes_dev, S * sizeof(dh_frame_box)));
    CU(cudaMalloc((void**)&ws, ws_bytes));
    CU(cudaMalloc((void**)&afmat, S * 9 * sizeof(double)));
    CU(cudaMalloc((void**)&status, S * sizeof(int32_t)));
    CU(cudaMalloc((void**)&pose_img, S * points * 2 * sizeof(double)));
    CU(cudaMallocHost((void**)&boxes_host, S * sizeof(dh_frame_box)));
    for (int i = 0; i < job->n_push; ++i) {
        for (int r = 0; r < job->n_resets; ++r)
            if (job->resets[r].push == i)
                DH(dh_stream_reset(st, job->resets[r].n ? job->resets[r].ids : NULL, job->resets[r].n, stream));
        CU(cudaMemcpyAsync(images, job->frames + i * S * frame_bytes, S * frame_bytes, cudaMemcpyHostToDevice, stream));
        /* the only host work of a push: this push's boxes into the pinned records (the previous push has finished) */
        for (int s = 0; s < S; ++s) {
            const double* b = job->boxes + ((size_t)i * S + s) * 5;
            dh_frame_box* r = &boxes_host[s];
            r->data = images + s * frame_bytes;
            r->h = job->H;
            r->w = job->W;
            r->stride = job->W * 3;
            r->hflip = b[4] == 1.0;
            r->objpos[0] = b[0];
            r->objpos[1] = b[1];
            r->winsize[0] = b[2];
            r->winsize[1] = b[3];
        }
        if (graph && !exec) {             /* capture upload + prepare + push once; every push replays it */
            CU(cudaStreamBeginCapture(stream, cudaStreamCaptureModeThreadLocal));
        }
        if (!exec) {
            CU(cudaMemcpyAsync(boxes_dev, boxes_host, S * sizeof(dh_frame_box), cudaMemcpyHostToDevice, stream));
            DH(dh_prepare_frames_u8(ctx, boxes_dev, S, job->max_crop_w, job->max_crop_h, in.h, in.w, NULL, ws, ws_bytes,
                                    in.p, afmat, status, stream));
            DH(dh_stream_push(st, stream));
        }
        if (graph && !exec) {
            CU(cudaStreamEndCapture(stream, &g));
            CU(cudaGraphInstantiate(&exec, g, 0));
        }
        if (exec) CU(cudaGraphLaunch(exec, stream));
        DH(dh_pose_to_image_f32(ctx, &pose, afmat, 1, pose_img, stream));
        CU(cudaStreamSynchronize(stream));
        int n_out = info.n_frame_outputs + info.n_clip_outputs;
        char name[64];
        for (int k = 0; k < n_out; ++k) {
            dh_view v;
            DH(dh_stream_output(st, k, &v, NULL));
            snprintf(name, sizeof(name), "%d.f32", k);
            if (append(job->prefix, tag, name, v.p, (size_t)v.n * v.h * v.w, v.c * sizeof(float), v.ld * sizeof(float),
                       i == 0))
                return 1;
        }
        const int32_t* ready;
        DH(dh_stream_ready(st, &ready));
        if (append(job->prefix, tag, "pose.f64", pose_img, 1, S * points * 2 * sizeof(double), S * points * 2 * sizeof(double),
                   i == 0) ||
            append(job->prefix, tag, "ready.i32", ready, 1, S * sizeof(int32_t), S * sizeof(int32_t), i == 0) ||
            append(job->prefix, tag, "status.i32", status, 1, S * sizeof(int32_t), S * sizeof(int32_t), i == 0))
            return 1;
    }
    if (exec) {
        CU(cudaGraphExecDestroy(exec));
        CU(cudaGraphDestroy(g));
    }
    CU(cudaFreeHost(boxes_host));
    CU(cudaFree(pose_img));
    CU(cudaFree(status));
    CU(cudaFree(afmat));
    CU(cudaFree(ws));
    CU(cudaFree(boxes_dev));
    CU(cudaFree(images));
    CU(cudaStreamDestroy(stream));
    DH(dh_stream_free(st));
    return 0;
}

int main(int argc, char** argv) {
    if (argc != 9 && argc != 10) {
        fprintf(stderr, "usage: %s STREAM.dhs FRAMES.u8 H W BOXES.f64 MAX_CROP_W MAX_CROP_H OUT_PREFIX [RESETS.txt]\n",
                argv[0]);
        return 2;
    }
    dh_stream_info info;
    DH(dh_stream_inspect(argv[1], &info, NULL, 0));
    job_t job;
    job.path = argv[1];
    job.S = info.n_streams;
    job.H = atoi(argv[3]);
    job.W = atoi(argv[4]);
    job.max_crop_w = atoi(argv[6]);
    job.max_crop_h = atoi(argv[7]);
    job.prefix = argv[8];
    if (job.H < 1 || job.W < 1) {
        fprintf(stderr, "bad frame size %s x %s\n", argv[3], argv[4]);
        return 2;
    }
    static reset_t resets[256];
    job.resets = resets;
    job.n_resets = 0;
    if (argc == 10 && read_resets(argv[9], resets, 256, &job.n_resets)) return 1;
    size_t n_frames, n_boxes;
    uint8_t* frames = (uint8_t*)read_all(argv[2], (size_t)job.S * job.H * job.W * 3, &n_frames);
    double* boxes = (double*)read_all(argv[5], (size_t)job.S * 5 * sizeof(double), &n_boxes);
    if (!frames || !boxes) return 1;
    if (n_frames != n_boxes) {
        fprintf(stderr, "%zu frame batches but %zu box batches\n", n_frames, n_boxes);
        return 1;
    }
    job.frames = frames;
    job.boxes = boxes;
    job.n_push = (int)n_frames;
    printf("%s: %d streams, T = %d, %d x %d frames -> %lld x %lld, %d pushes\n", argv[1], job.S, info.frames_per_clip,
           job.W, job.H, (long long)info.input_shape[2], (long long)info.input_shape[1], job.n_push);
    dh_ctx* ctx;
    DH(dh_ctx_create(&ctx, 0));
    for (int graph = 0; graph < 2; ++graph)
        if (run(ctx, &job, graph)) return 1;
    free(frames);
    free(boxes);
    DH(dh_ctx_destroy(ctx));
    printf("ok: %d pushes\n", job.n_push);
    return 0;
}
