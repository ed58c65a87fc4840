// Sliding-window assembly for streamed clip inference (deephar_b200/stream.py): after the per-frame stage has run on
// one new frame per stream, every tensor that crosses from frames to clips (`frames_to_clip`, layers.py) is appended
// to a ring of the last T frames of its stream, and the clip stage's (S, T, ...) input is rewritten from that ring in
// time order.  The ring position is a device-side counter advanced by the launch itself, so the whole per-frame step
// replays as one CUDA graph with no host writes in between.
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

}  // namespace

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
