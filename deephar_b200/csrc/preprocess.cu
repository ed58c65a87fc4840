// Evaluation-time input pipeline on the GPU (SURVEY.md 8 f4): the step BEFORE the forward path.
//   deephar/utils/transform.py:60-134   T.rotate_crop(angle 0) -> crop(integer box, zeros outside) ->
//                                       T.resize(crop_resolution, Image.BILINEAR) [-> horizontal_flip] -> asarray
//   deephar/utils/transform.py:212-231  normalize_channels: x / 255 [** chpower], (x - 0.5) * 2      (float32)
//   driven by deephar/data/mpii.py:91-122 (fixed evaluation config).
// `Image.resize(BILINEAR)` is Pillow's two-pass fixed-point resampler (libImaging/Resample.c): per output index a
// window of source pixels weighted by a triangle filter widened by the down-scaling factor, weights as 22-bit fixed
// point, horizontal pass -> uint8 -> vertical pass -> uint8.  The weight tables are computed on the host
// (deephar_b200/preprocess.py, double precision exactly as Pillow does) or, for dh_prepare_frames_u8, on the device
// by frame_geometry_kernel below; the kernels do the pixel work, bit-exact.
// Batched: one launch pair per batch of decoded uint8 frames of arbitrary sizes, output written straight into the
// (N, H, W, 3) fp32 NHWC input tensor of the network.
#include "common.cuh"

namespace {

constexpr int PREC = 22;

__device__ __forceinline__ int clip8(int v) { return v < 0 ? 0 : (v > 255 ? 255 : v); }

// horizontal pass: tmp[n][r][xx][c], r over the crop rows
__global__ void resize_h_kernel(const dh_frame_src* __restrict__ frames, const int32_t* __restrict__ bounds,
                                const int32_t* __restrict__ coefs, int out_w, uint8_t* __restrict__ tmp,
                                int64_t tmp_stride) {
    const dh_frame_src f = frames[blockIdx.z];
    const int xx = blockIdx.x * blockDim.x + threadIdx.x;
    const int r = blockIdx.y * blockDim.y + threadIdx.y;
    if (xx >= out_w || r >= f.ch) return;
    const int first = bounds[f.kx_off + 2 * xx], n = bounds[f.kx_off + 2 * xx + 1];
    const int32_t* k = coefs + (int64_t)f.kx_coef_off + (int64_t)xx * f.ksx;
    int a0 = 1 << (PREC - 1), a1 = a0, a2 = a0;
    const int sy = f.y0 + r;
    if (sy >= 0 && sy < f.h) {
        const uint8_t* row = f.data + (int64_t)sy * f.stride;
        for (int t = 0; t < n; ++t) {
            const int sx = f.x0 + first + t;
            if (sx >= 0 && sx < f.w) {                      // Image.crop fills the outside with zeros
                const int kk = k[t];
                a0 += row[sx * 3 + 0] * kk;
                a1 += row[sx * 3 + 1] * kk;
                a2 += row[sx * 3 + 2] * kk;
            }
        }
    }
    uint8_t* o = tmp + blockIdx.z * tmp_stride + ((int64_t)r * out_w + xx) * 3;
    o[0] = (uint8_t)clip8(a0 >> PREC);
    o[1] = (uint8_t)clip8(a1 >> PREC);
    o[2] = (uint8_t)clip8(a2 >> PREC);
}

// vertical pass + flip + normalize_channels -> out[n][yy][xo][c] fp32
__global__ void resize_v_norm_kernel(const dh_frame_src* __restrict__ frames, const int32_t* __restrict__ bounds,
                                     const int32_t* __restrict__ coefs, int out_h, int out_w,
                                     const uint8_t* __restrict__ tmp, int64_t tmp_stride, float p0, float p1, float p2,
                                     float* __restrict__ out) {
    const dh_frame_src f = frames[blockIdx.z];
    const int xx = blockIdx.x * blockDim.x + threadIdx.x;
    const int yy = blockIdx.y * blockDim.y + threadIdx.y;
    if (xx >= out_w || yy >= out_h) return;
    if (f.ch == 0) {                                         // a frame dh_prepare_frames_u8 flagged: NaN, nothing read
        float* o = out + (((int64_t)blockIdx.z * out_h + yy) * out_w + xx) * 3;
        o[0] = o[1] = o[2] = __int_as_float(0x7FC00000);
        return;
    }
    const int first = bounds[f.ky_off + 2 * yy], n = bounds[f.ky_off + 2 * yy + 1];
    const int32_t* k = coefs + (int64_t)f.ky_coef_off + (int64_t)yy * f.ksy;
    const uint8_t* col = tmp + blockIdx.z * tmp_stride + (int64_t)xx * 3;
    int a0 = 1 << (PREC - 1), a1 = a0, a2 = a0;
    for (int t = 0; t < n; ++t) {
        const uint8_t* px = col + (int64_t)(first + t) * out_w * 3;
        const int kk = k[t];
        a0 += px[0] * kk;
        a1 += px[1] * kk;
        a2 += px[2] * kk;
    }
    const int xo = f.hflip ? out_w - 1 - xx : xx;            // Image.transpose(FLIP_LEFT_RIGHT)
    float v[3] = {(float)clip8(a0 >> PREC), (float)clip8(a1 >> PREC), (float)clip8(a2 >> PREC)};
    const float pw[3] = {p0, p1, p2};
    float* o = out + (((int64_t)blockIdx.z * out_h + yy) * out_w + xo) * 3;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        float t = __fdiv_rn(v[c], 255.f);                    // frame /= 255.   (float32, correctly rounded)
        if (pw[c] != 1.f) t = powf(t, pw[c]);
        o[c] = __fmul_rn(__fsub_rn(t, 0.5f), 2.f);           // frame -= .5 ; frame *= 2.
    }
}

// ---- per-frame geometry on the device (dh_prepare_frames_u8) ----
// What FramePipeline.plan computes on the host, one frame per blockIdx.y: the box (preprocess.crop_box), both axes'
// tables (preprocess.resample_tables) and the afmat (preprocess.affine_map).  Every double operation is spelled as its
// correctly rounded intrinsic, in the order the numpy code performs it, so no multiply-add is contracted and the
// tables equal the host's bit for bit.

// resample_tables' ksize: taps per output index of an in -> out axis (plain division and ceil: exact on host and device)
__host__ __device__ inline int resample_taps(int in_size, int out_size) {
    const double scale = (double)in_size / (double)out_size;
    return (int)ceil(scale > 1.0 ? scale : 1.0) * 2 + 1;
}

// trunc(v) fits int32 (false for NaN)
__device__ __forceinline__ bool fits_i32(double v) { return v > -2147483649.0 && v < 2147483648.0; }

struct FrameGeom {
    int32_t status;                   // DH_FRAME_* bits, 0 = usable
    int32_t x0, y0, cw, ch;
};

__device__ FrameGeom frame_geom(const dh_frame_box& b, int max_crop_w, int max_crop_h) {
    FrameGeom g = {0, 0, 0, 0, 0};
    const bool image_ok = b.h >= 0 && b.w >= 0 && (int64_t)b.stride >= 3 * (int64_t)b.w && (b.data || !b.h || !b.w);
    const double hw = __ddiv_rn(b.winsize[0], 2.0), hh = __ddiv_rn(b.winsize[1], 2.0);
    const double e[4] = {__dsub_rn(b.objpos[0], hw), __dsub_rn(b.objpos[1], hh), __dadd_rn(b.objpos[0], hw),
                         __dadd_rn(b.objpos[1], hh)};
    bool ok = image_ok && isfinite(b.objpos[0]) && isfinite(b.objpos[1]) && isfinite(b.winsize[0]) && isfinite(b.winsize[1]);
    for (int k = 0; k < 4; ++k) ok = ok && fits_i32(e[k]);
    if (!ok) {                                               // checked before any cast: casting such a value is undefined
        g.status = DH_FRAME_BAD_BOX;
        return g;
    }
    const int32_t x0 = (int32_t)e[0], y0 = (int32_t)e[1], x1 = (int32_t)e[2], y1 = (int32_t)e[3];   // toward zero
    const int64_t cw = (int64_t)x1 - x0, ch = (int64_t)y1 - y0;
    if (cw < 1 || ch < 1) g.status = DH_FRAME_EMPTY;
    else if (cw > max_crop_w || ch > max_crop_h) g.status = DH_FRAME_TOO_LARGE;
    else g = FrameGeom{0, x0, y0, (int32_t)cw, (int32_t)ch};
    return g;
}

// tap t's triangle weight before normalisation, as resample_tables computes it
__device__ __forceinline__ double tap_weight(int t, int64_t first, int count, double center, double inv_fscale) {
    const double v = fabs(__dmul_rn(__dadd_rn(__dsub_rn((double)(t + first), center), 0.5), inv_fscale));
    return (v < 1.0 && t < count) ? __dsub_rn(1.0, v) : 0.0;
}

// output index o of an in -> out axis: (first, count) into bd, ks 22-bit fixed-point weights into cf
__device__ void resample_row(int in_size, int out_size, int o, int ks, int32_t* bd, int32_t* cf) {
    const double scale = __ddiv_rn((double)in_size, (double)out_size);
    const double fscale = scale > 1.0 ? scale : 1.0, support = fscale;
    const double center = __dmul_rn(__dadd_rn((double)o, 0.5), scale);
    int64_t first = (int64_t)trunc(__dadd_rn(__dsub_rn(center, support), 0.5));
    int64_t last = (int64_t)trunc(__dadd_rn(__dadd_rn(center, support), 0.5));
    first = first < 0 ? 0 : first;
    last = last > in_size ? in_size : last;
    const int count = (int)(last - first);
    const double inv_fscale = __ddiv_rn(1.0, fscale);
    double total = 0.0;
    for (int t = 0; t < ks; ++t) total = __dadd_rn(total, tap_weight(t, first, count, center, inv_fscale));
    for (int t = 0; t < ks; ++t) {
        double w = tap_weight(t, first, count, center, inv_fscale);
        if (total != 0.0) w = __ddiv_rn(w, total);
        cf[t] = (int32_t)trunc(__dadd_rn(0.5, __dmul_rn(w, (double)(1 << PREC))));
    }
    bd[0] = (int32_t)first;
    bd[1] = count;
}

// grid (ceil((out_w + out_h) / blockDim.x), n): thread t < out_w computes x index t, the next out_h threads the y
// indices; thread 0 also writes the frame's dh_frame_src, afmat and status
__global__ void frame_geometry_kernel(const dh_frame_box* __restrict__ boxes, int max_crop_w, int max_crop_h, int out_h,
                                      int out_w, int kx, int bounds_per, int coefs_per, dh_frame_src* __restrict__ frames,
                                      int32_t* __restrict__ bounds, int32_t* __restrict__ coefs,
                                      double* __restrict__ afmat, int32_t* __restrict__ status) {
    const int i = blockIdx.y;
    const dh_frame_box b = boxes[i];
    const FrameGeom g = frame_geom(b, max_crop_w, max_crop_h);
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    const int b_off = i * bounds_per, c_off = i * coefs_per;       // < 2^31: dh_prepare_frames_u8 checks the totals
    if (t == 0) {
        dh_frame_src f;
        f.data = g.status ? nullptr : b.data;
        f.h = g.status ? 0 : b.h;
        f.w = g.status ? 0 : b.w;
        f.stride = g.status ? 0 : b.stride;
        f.x0 = g.x0; f.y0 = g.y0; f.cw = g.cw; f.ch = g.ch;     // flagged: cw = ch = 0, the resize passes write NaN
        f.hflip = b.hflip == 1;
        f.kx_off = b_off; f.ky_off = b_off + 2 * out_w;
        f.kx_coef_off = c_off; f.ky_coef_off = c_off + out_w * kx;
        f.ksx = g.status ? 0 : resample_taps(g.cw, out_w);
        f.ksy = g.status ? 0 : resample_taps(g.ch, out_h);
        frames[i] = f;
        double* a = afmat + (int64_t)i * 9;
        if (g.status) {
            for (int k = 0; k < 9; ++k) a[k] = __longlong_as_double(0x7FF8000000000000LL);
        } else {                                             // affine_map: translate, scale, [flip], normalise
            const double sx = __ddiv_rn((double)out_w, (double)g.cw), sy = __ddiv_rn((double)out_h, (double)g.ch);
            double a00 = sx, a02 = __dmul_rn(sx, -(double)g.x0);
            const double a12 = __dmul_rn(sy, -(double)g.y0);
            if (f.hflip) {
                a00 = -sx;
                a02 = __dadd_rn(-a02, (double)out_w);
            }
            const double irw = __ddiv_rn(1.0, (double)out_w), irh = __ddiv_rn(1.0, (double)out_h);
            a[0] = __dmul_rn(a00, irw); a[1] = 0.0; a[2] = __dmul_rn(a02, irw);
            a[3] = 0.0; a[4] = __dmul_rn(sy, irh); a[5] = __dmul_rn(a12, irh);
            a[6] = 0.0; a[7] = 0.0; a[8] = 1.0;
        }
        status[i] = g.status;
    }
    if (g.status || t >= out_w + out_h) return;
    if (t < out_w) {
        const int ks = resample_taps(g.cw, out_w);
        resample_row(g.cw, out_w, t, ks, bounds + b_off + 2 * t, coefs + c_off + (int64_t)t * ks);
    } else {
        const int o = t - out_w, ks = resample_taps(g.ch, out_h);
        resample_row(g.ch, out_h, o, ks, bounds + b_off + 2 * out_w + 2 * o,
                     coefs + c_off + (int64_t)out_w * kx + (int64_t)o * ks);
    }
}

void launch_resize(const dh_frame_src* frames, int n, int max_crop_h, const int32_t* bounds, const int32_t* coefs,
                   int out_h, int out_w, const float* chpower3, uint8_t* tmp, int64_t tmp_stride, float* out,
                   cudaStream_t s) {
    const float p0 = chpower3 ? chpower3[0] : 1.f, p1 = chpower3 ? chpower3[1] : 1.f, p2 = chpower3 ? chpower3[2] : 1.f;
    dim3 block(32, 8);
    dim3 gh((out_w + 31) / 32, (max_crop_h + 7) / 8, n);
    resize_h_kernel<<<gh, block, 0, s>>>(frames, bounds, coefs, out_w, tmp, tmp_stride);
    dim3 gv((out_w + 31) / 32, (out_h + 7) / 8, n);
    resize_v_norm_kernel<<<gv, block, 0, s>>>(frames, bounds, coefs, out_h, out_w, tmp, tmp_stride, p0, p1, p2, out);
}

// the workspace of dh_prepare_frames_u8 (byte offsets; layout documented in the header)
struct PrepLayout {
    int kx, ky;                       // taps of the widest crop on each axis: the pitch of a frame's tables
    int64_t bounds_per, coefs_per;    // int32 per frame
    int64_t bounds, coefs, tmp, tmp_stride, total;
};

constexpr int kMaxPrepSize = 1 << 18;

int prep_layout(int n, int max_crop_w, int max_crop_h, int out_h, int out_w, PrepLayout* L) {
    DH_CHECK_ARG(n >= 0 && n <= 65535, "dh_prepare_frames: n = %d outside [0, 65535]", n);
    DH_CHECK_ARG(max_crop_w >= 1 && max_crop_h >= 1 && out_h >= 1 && out_w >= 1 && max_crop_w <= kMaxPrepSize &&
                     max_crop_h <= kMaxPrepSize && out_h <= kMaxPrepSize && out_w <= kMaxPrepSize,
                 "dh_prepare_frames: max_crop_w / max_crop_h / out_h / out_w must lie in [1, %d]", kMaxPrepSize);
    auto up = [](int64_t v, int64_t a) { return (v + a - 1) / a * a; };
    L->kx = resample_taps(max_crop_w, out_w);
    L->ky = resample_taps(max_crop_h, out_h);
    L->bounds_per = 2 * ((int64_t)out_w + out_h);
    L->coefs_per = (int64_t)out_w * L->kx + (int64_t)out_h * L->ky;
    DH_CHECK_ARG(n * L->bounds_per <= INT32_MAX && n * L->coefs_per <= INT32_MAX,
                 "dh_prepare_frames: the tables of %d frames exceed 2^31 int32 entries", n);
    L->tmp_stride = up((int64_t)max_crop_h * out_w * 3, 16);
    L->bounds = up((int64_t)n * sizeof(dh_frame_src), 256);
    L->coefs = up(L->bounds + n * L->bounds_per * 4, 256);
    L->tmp = up(L->coefs + n * L->coefs_per * 4, 256);
    L->total = L->tmp + n * L->tmp_stride;
    return 0;
}

}  // namespace

extern "C" int dh_crop_resize_norm_u8(dh_ctx* ctx, const dh_frame_src* frames_dev, int n, int max_crop_h,
                                      const int32_t* bounds_dev, const int32_t* coefs_dev, int out_h, int out_w,
                                      const float* chpower3, uint8_t* tmp_dev, int64_t tmp_stride, float* out_dev,
                                      void* stream) {
    DH_CHECK_ARG(ctx && frames_dev && bounds_dev && coefs_dev && tmp_dev && out_dev, "dh_crop_resize_norm_u8: NULL argument");
    DH_CHECK_ARG(n >= 0 && max_crop_h >= 1 && out_h >= 1 && out_w >= 1, "dh_crop_resize_norm_u8: bad sizes");
    DH_CHECK_ARG(tmp_stride >= (int64_t)max_crop_h * out_w * 3, "dh_crop_resize_norm_u8: tmp_stride too small");
    DH_CHECK_ARG(n <= 65535, "dh_crop_resize_norm_u8: at most 65535 frames per call");
    if (n == 0) return 0;
    launch_resize(frames_dev, n, max_crop_h, bounds_dev, coefs_dev, out_h, out_w, chpower3, tmp_dev, tmp_stride, out_dev,
                  (cudaStream_t)stream);
    DH_LAUNCH_EPILOGUE(ctx, 2);
}

extern "C" int64_t dh_prepare_frames_workspace(int n, int max_crop_w, int max_crop_h, int out_h, int out_w) {
    PrepLayout L;
    if (prep_layout(n, max_crop_w, max_crop_h, out_h, out_w, &L)) return -1;
    return L.total;
}

extern "C" int dh_prepare_frames_u8(dh_ctx* ctx, const dh_frame_box* boxes_dev, int n, int max_crop_w, int max_crop_h,
                                    int out_h, int out_w, const float* chpower3, void* ws, int64_t ws_bytes, float* out_dev,
                                    double* afmat_dev, int32_t* status_dev, void* stream) {
    DH_CHECK_ARG(ctx && boxes_dev && ws && out_dev && afmat_dev && status_dev, "dh_prepare_frames_u8: NULL argument");
    PrepLayout L;
    if (prep_layout(n, max_crop_w, max_crop_h, out_h, out_w, &L)) return -1;
    DH_CHECK_ARG(ws_bytes >= L.total, "dh_prepare_frames_u8: workspace of %lld bytes, %lld needed", (long long)ws_bytes,
                 (long long)L.total);
    DH_CHECK_ARG(((uintptr_t)ws & 255) == 0, "dh_prepare_frames_u8: workspace not 256-byte aligned");
    if (n == 0) return 0;
    uint8_t* w = (uint8_t*)ws;
    dh_frame_src* frames = (dh_frame_src*)w;
    int32_t* bounds = (int32_t*)(w + L.bounds);
    int32_t* coefs = (int32_t*)(w + L.coefs);
    cudaStream_t s = (cudaStream_t)stream;
    dim3 gg((out_w + out_h + 127) / 128, n);
    frame_geometry_kernel<<<gg, 128, 0, s>>>(boxes_dev, max_crop_w, max_crop_h, out_h, out_w, L.kx, (int)L.bounds_per,
                                             (int)L.coefs_per, frames, bounds, coefs, afmat_dev, status_dev);
    launch_resize(frames, n, max_crop_h, bounds, coefs, out_h, out_w, chpower3, w + L.tmp, L.tmp_stride, out_dev, s);
    DH_LAUNCH_EPILOGUE(ctx, 3);
}
