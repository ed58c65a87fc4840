// Sliding-window assembly for streamed clip inference (deephar_b200/stream.py): after the per-frame stage has run on
// one new frame per stream, every tensor that crosses from frames to clips (`frames_to_clip`, layers.py) is appended
// to a ring of the last T frames of its stream, and the clip stage's (S, T, ...) input is rewritten from that ring in
// time order.  The ring position is a device-side counter advanced by the launch itself, so the whole per-frame step
// replays as one CUDA graph with no host writes in between.  dh_stream_ready_f32 keeps the per-stream readiness of the C
// runtime's streams (dh_stream_push, model_rt.cu) on the device as well.
#include "common.cuh"

namespace {

// One launch for all tensors: every block takes its grid-stride share of (stream, window slot, element) of each tensor.
__global__ void __launch_bounds__(256) clip_window_kernel(const dh_clip_window* __restrict__ table, int n_tensors, int S,
                                                          int T, int* counter) {
    __shared__ int s_pos;
    if (threadIdx.x == 0) {
        s_pos = *reinterpret_cast<volatile int*>(counter);
        // ticket: the last block to read the position advances it (every other block has read it by then)
        __threadfence();
        if (atomicAdd(counter + 1, 1) == (int)gridDim.x - 1) {
            counter[1] = 0;
            counter[0] = (s_pos + 1) % T;
        }
    }
    __syncthreads();
    const int pos = s_pos;
    for (int i = 0; i < n_tensors; ++i) {
        const dh_clip_window e = table[i];
        const int hw = e.src.h * e.src.w, c = e.src.c;
        const int64_t per_frame = (int64_t)hw * c;
        const int64_t total = (int64_t)S * T * per_frame;
        for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total;
             idx += (int64_t)gridDim.x * blockDim.x) {
            const int64_t el = idx % per_frame;
            const int64_t st = idx / per_frame;      // s * T + j: window slot j of stream s
            const int j = (int)(st % T);
            const int s = (int)(st / T);
            const int64_t pix = el / c;
            const int ch = (int)(el % c);
            float v;
            if (j == T - 1) {                        // the new frame: into the window and into ring slot `pos`
                v = __ldg(e.src.p + ((int64_t)s * hw + pix) * e.src.ld + ch);
                e.ring[((int64_t)s * T + pos) * per_frame + el] = v;
            } else {                                 // older frames, oldest first; ring slot `pos` is not read here
                v = e.ring[((int64_t)s * T + (pos + 1 + j) % T) * per_frame + el];
            }
            e.dst.p[(st * hw + pix) * e.dst.ld + ch] = v;
        }
    }
}

// Readiness after a push.  Each stream's count is read and advanced by the one CTA that owns the stream (CTAs stride
// over streams), so no block can read a count another block has already advanced in this launch.
__global__ void __launch_bounds__(256) stream_ready_kernel(int32_t* __restrict__ count, int S, int T,
                                                           const dh_view* __restrict__ outs, int n_outs,
                                                           int32_t* __restrict__ ready) {
    __shared__ int s_ready;
    for (int s = blockIdx.x; s < S; s += gridDim.x) {
        if (threadIdx.x == 0) {
            const int c = min(count[s] + 1, T);       // saturates: never overflows however long a video runs
            count[s] = c;
            ready[s] = c >= T;
            s_ready = c >= T;
        }
        __syncthreads();
        const bool is_ready = s_ready;
        __syncthreads();                              // s_ready is rewritten for the next stream
        if (is_ready) continue;
        const float nan = __int_as_float(0x7FC00000);  // the bits torch's index_fill_(nan) writes
        for (int i = 0; i < n_outs; ++i) {
            const dh_view v = outs[i];
            const int64_t hw = (int64_t)v.h * v.w, per_item = hw * v.c;
            for (int64_t e = threadIdx.x; e < per_item; e += blockDim.x)
                v.p[((int64_t)s * hw + e / v.c) * v.ld + e % v.c] = nan;
        }
    }
}

}  // namespace

extern "C" int dh_stream_ready_f32(dh_ctx* ctx, int32_t* count_dev, int S, int T, const dh_view* outs_dev, int n_outs,
                                   int32_t* ready_dev, void* stream) {
    DH_CHECK_ARG(ctx && count_dev && ready_dev, "dh_stream_ready_f32: NULL argument");
    DH_CHECK_ARG(n_outs >= 0 && (outs_dev || n_outs == 0), "dh_stream_ready_f32: %d views at %p", n_outs,
                 (const void*)outs_dev);
    DH_CHECK_ARG(S >= 1 && T >= 1, "dh_stream_ready_f32: S and T must be positive (got %d, %d)", S, T);
    stream_ready_kernel<<<min(S, ctx->num_sms * 8), 256, 0, (cudaStream_t)stream>>>(count_dev, S, T, outs_dev, n_outs,
                                                                                     ready_dev);
    DH_LAUNCH_EPILOGUE(ctx, 1);
}

extern "C" int dh_clip_window_f32(dh_ctx* ctx, const dh_clip_window* table_dev, int n_tensors, int S, int T,
                                  int32_t* counter_dev, void* stream) {
    DH_CHECK_ARG(ctx && table_dev && counter_dev, "dh_clip_window_f32: NULL argument");
    DH_CHECK_ARG(n_tensors >= 1, "dh_clip_window_f32: n_tensors must be positive, got %d",
                 n_tensors);
    DH_CHECK_ARG(S >= 1 && T >= 1, "dh_clip_window_f32: S and T must be positive (got %d, %d)", S, T);
    // the sizes live in the device table: a fixed grid (8 CTAs per SM) covers every tensor with grid-stride loops
    clip_window_kernel<<<ctx->num_sms * 8, 256, 0, (cudaStream_t)stream>>>(table_dev, n_tensors, S, T, counter_dev);
    DH_LAUNCH_EPILOGUE(ctx, 1);
}
