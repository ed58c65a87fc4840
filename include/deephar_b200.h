/* deephar_b200 -- C ABI of the H100-native deephar forward hot path.
 *
 * The reference (dluvizon/deephar) has no FFI / plugin interface: its seam is
 * Python (keras layers + keras.Model.predict).  This header is the boundary a
 * ctypes binding uses (deephar_b200/_ffi.py; INTEGRATION.md shows the stub a
 * maintainer of the reference would add).  Every entry point names the
 * reference code it replaces (paths relative to the reference tree).
 *
 * Conventions
 *   - plain C: pointers + sizes, no C++ / torch types.
 *   - all tensors are fp32 NHWC device memory owned by the CALLER; a `dh_view`
 *     is a (possibly channel-sliced) window: element (n,y,x,c) lives at
 *     p[((n*h + y)*w + x)*ld + c], so `ld` is the channel count of the
 *     underlying buffer (ld == c for a dense tensor) and a channel offset is
 *     folded into `p`.  This is how `concatenate` / Lambda-slices cost nothing.
 *   - every launch goes on the `stream` argument (a cudaStream_t passed as
 *     void*); no hidden synchronisation, no global mutable state besides the
 *     per-thread last-error string.
 *   - return value: 0 = ok; <0 = argument error (text via dh_last_error());
 *     >0 = cudaError_t.
 */
#ifndef DEEPHAR_B200_H
#define DEEPHAR_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct dh_view {
    float*  p;
    int32_t n, h, w, c;
    int32_t ld;
} dh_view;

/* Fused pre-/post-ops of a convolution.  Order of evaluation:
 *   a   = x                                   (input tap, 0 outside the image)
 *   a   = a * pre_scale[ci] + pre_shift[ci]   if pre_scale      (BatchNormalization before the conv)
 *   a   = max(a, 0)                           if pre_relu       (Activation('relu') before the conv)
 *   (zero padding is applied AFTER these, as keras pads the activated tensor)
 *   y   = conv(a)
 *   y   = y * post_scale[co] + post_shift[co] if post_scale     (BatchNormalization after the conv)
 *   y   = max(y, 0)                           if post_relu
 *   y  += res[0] (+ res[1])                   keras `add([...])`; the LAST residual may be a half-resolution tensor
 *                                             added through UpSampling2D((2,2)) (`res_up2x`; reception.py:122-127)
 * replaces: layers.py:202-325 (conv_bn, conv_bn_act, act_conv_bn, act_conv,
 * separable_act_conv_bn, ...), models/common.py:25-67 residual_unit,
 * models/reception.py:43-59 _sepconv_residual. */
typedef struct dh_conv_desc {
    int32_t kh, kw, sh, sw;
    int32_t pad_same;            /* 1 = TF 'SAME' (extra pad bottom/right), 0 = 'VALID' */
    int32_t pre_relu;
    int32_t post_relu;
    int32_t n_res;               /* 0..2 */
    const float* pre_scale;      /* [Cin] or NULL */
    const float* pre_shift;      /* [Cin] or NULL */
    const float* post_scale;     /* [Cout] or NULL */
    const float* post_shift;     /* [Cout] or NULL */
    dh_view res[2];
    int32_t precision;           /* tensor-core path: 1 = bf16 x1, 3 = bf16 x3 split (~fp32); 0 = library default */
    int32_t res_up2x;            /* bit i: res[i] is (N, Ho/2, Wo/2, Cout) and is nearest-upsampled 2x before the add
                                    (only the last residual; Wo == 16 or Wo % 32 == 0; every kernel but the direct
                                    stem and the wide pointwise one, which leave such a call to the others) */
    dh_view pool_out;            /* p != NULL: ALSO write MaxPooling2D((2,2)) of y, (N, Ho/2, Wo/2, Cout) -- the hourglass
                                    pools the tensor the block-end add produces (reception.py:108-110); taken by the wide
                                    pointwise kernel only (1x1, Cin <= 64, Wo == 32), an error elsewhere */
} dh_conv_desc;

/* Packed weights for the tensor-core path (built once at load time). */
typedef struct dh_packed_w {
    const void* hi;              /* bf16 [Cout_pad][K]  K-major, K = kh*kw*Cin */
    const void* lo;              /* bf16 residual (w - hi), same layout */
    int32_t cout_pad, k;
} dh_packed_w;

typedef struct dh_ctx dh_ctx;

/* --- context ------------------------------------------------------------- */
int         dh_ctx_create(dh_ctx** out, int device);
int         dh_ctx_destroy(dh_ctx* ctx);
const char* dh_last_error(void);
int         dh_version(void);
/* number of kernel launches issued through this context since creation / reset */
int64_t     dh_launch_count(dh_ctx* ctx, int reset);
/* scratch for two-kernel ops (owned by the caller): set before use */
int         dh_set_workspace(dh_ctx* ctx, void* ptr, int64_t bytes);
/* tuning switches: "share_a" (default 1) = 2-CTA clusters share the separable A tile over DSMEM;
 * "sep_tma" (default 1) = use the TMA-staged separable kernel where it applies;
 * "pw_smallk" (default 1) = CUDA-core kernel for wide 1x1 convs with Cin <= 64;
 * "dense_patch" (default 1) = TMA-staged patch kernel (conv_patch.cu) for stride-1 Conv2D where it applies;
 * "sam3d_stream" (default 1) = cluster-split streaming kernel for the volumetric soft-argmax;
 * (the round-1 "dbg" timing-ablation switch only exists in tools/ builds: make ABLATE=1) */
int         dh_set_option(dh_ctx* ctx, const char* name, int value);

/* --- convolutions -------------------------------------------------------- */
/* Tensor-core weight packing geometry: dh_packed_w.hi/lo are bf16 [dh_tc_cout_pad(Cout)][dh_tc_k_pad(K)]
 * (zero padded), K = kh*kw*Cin ordered (ky,kx,ci) for Conv2D, K = Cin for the pointwise stage. */
int dh_tc_cout_pad(int cout);
int dh_tc_k_pad(int k);
/* which kernel family served the last dh_conv2d_f32 / dh_sepconv2d_f32 on this context:
 * 0 = CUDA-core (fp32 FFMA), 1 = wgmma kernel (conv_tc.cu), 2 = TMA-staged wgmma separable kernel (conv_sep.cu),
 * 3 = CUDA-core wide pointwise kernel for 1x1 convs with Cin <= 64 and Cout >= 128 (exact fp32),
 * 4 = TMA-staged patch wgmma kernel for stride-1 Conv2D (conv_patch.cu). */
int dh_last_conv_path(dh_ctx* ctx);
/* convolutions that no tensor-core / specialised kernel took and that ran on the generic CUDA-core
 * implicit-GEMM kernel (path 0) since creation / reset: the silent-fallback counter. */
int64_t dh_fallback_count(dh_ctx* ctx, int reset);

/* keras Conv2D(use_bias=False) (layers.py:66-71) with fused pre/post ops.
 * w: HWIO (kh,kw,Cin,Cout) fp32 -- the keras kernel layout, unchanged.
 * packed may be NULL (CUDA-core path only). */
int dh_conv2d_f32(dh_ctx* ctx, const dh_view* x, const float* w_hwio, const dh_packed_w* packed,
                  const dh_conv_desc* d, const dh_view* out, void* stream);

/* keras SeparableConv2D(use_bias=False) (layers.py:74-80): depthwise kxk
 * (w_dw: (kh,kw,Cin,1)) then 1x1 pointwise (w_pw: (1,1,Cin,Cout)), nothing in between. */
int dh_sepconv2d_f32(dh_ctx* ctx, const dh_view* x, const float* w_dw, const float* w_pw,
                     const dh_packed_w* packed_pw, const dh_conv_desc* d, const dh_view* out,
                     void* stream);

/* What dh_conv2d_f32 / dh_sepconv2d_f32 would run for the same arguments and the context's current options.
 * The CUDA-core paths report their grids in the same fields:
 *   path 3 (wide pointwise):   bm = 64, grid_x = min(n_mtiles, SMs), grid_y = 1, bn_cta = Cout, n_kblocks = 1;
 *   path 0, direct 3x3x3 stem (fallback = 0): bm = pixels per CTA pass (64 at Cout 32, 32 at Cout 64),
 *                              grid_x = min(n_mtiles, 16 x SMs), grid_y = 1, bn_cta = Cout, n_kblocks = 1;
 *   path 0, implicit GEMM (fallback = 1; of a separable layer: its pointwise stage): bm = 128, one CTA per tile,
 *                              grid_x = n_mtiles, grid_y = ceil(Cout / 64), bn_cta = 64, n_kblocks = ceil(K / 16). */
typedef struct dh_conv_plan_info {
    int32_t path;                /* as dh_last_conv_path */
    int32_t fallback;            /* 1 = the launch adds one to dh_fallback_count */
    int64_t workspace_bytes;     /* dh_set_workspace bytes the launch needs */
    int32_t n_mtiles;            /* M-tiles of bm rows */
    int32_t grid_x, grid_y;      /* persistent grid: CTA (x, y) runs M-tiles x, x + grid_x, ... of N part y */
    int32_t bn_cta;              /* output channels per CTA */
    int32_t n_kblocks;           /* K-blocks per M-tile */
    int32_t stages;              /* ring depth of the register-producer kernel (path 1); 0 on the other paths */
    int32_t cluster;             /* 1 = pairs of N parts run as (1, 2, 1) clusters sharing their A tiles */
    int32_t bm;                  /* rows (output pixels) per M-tile: 128, or 64 on path 2's 64 x 144 tiles (and above) */
    int32_t epi_tma;             /* 1 = path 2's 64-row tiles stage the epilogue in shared memory (residuals loaded and
                                    the output stored by TMA); 0 = the epilogue works from registers */
} dh_conv_plan_info;
/* Host-only: launch nothing, touch neither the device nor the workspace, and leave dh_last_conv_path,
 * dh_fallback_count and dh_launch_count as they are.  Return < 0 with the launch's error text for a call the
 * launch would refuse. */
int dh_conv2d_plan(dh_ctx* ctx, const dh_view* x, const float* w_hwio, const dh_packed_w* packed,
                   const dh_conv_desc* d, const dh_view* out, dh_conv_plan_info* info);
int dh_sepconv2d_plan(dh_ctx* ctx, const dh_view* x, const float* w_dw, const float* w_pw,
                      const dh_packed_w* packed_pw, const dh_conv_desc* d, const dh_view* out,
                      dh_conv_plan_info* info);

/* --- pooling / resampling / elementwise ---------------------------------- */
/* keras MaxPooling2D (reception.py:74,86,108,115; layers.py:92-97); 'same' pads with -inf. */
int dh_maxpool2d_f32(dh_ctx* ctx, const dh_view* x, int kh, int kw, int sh, int sw, int pad_same,
                     const dh_view* out, void* stream);
/* out = a + UpSampling2D((2,2))(b)  (reception.py:122-127); a may be NULL-p (plain upsample). */
int dh_upsample2x_add_f32(dh_ctx* ctx, const dh_view* a, const dh_view* b, const dh_view* out,
                          void* stream);
/* out = sum of n_in (1..4) views, optional per-channel affine + relu on the sum
 * (keras add([...]) followed by BatchNormalization / Activation). */
int dh_add_n_f32(dh_ctx* ctx, const dh_view* in, int n_in, const float* scale, const float* shift,
                 int relu, const dh_view* out, void* stream);

/* --- soft-argmax heads ---------------------------------------------------- */
/* One pass over h (N,H,W,C): per (frame, channel)
 *   p = channel_softmax_2d(alpha)(h)                    activations.py:3-16
 *   xy = softargmax2d(p)  grid linspace(0,1) inclusive  layers.py:122-129,160-200; utils/math.py:6-19
 *   conf = max over 2x2 windows (stride 1, valid) of the window SUM of
 *          p   if conf_on_prob = 1   (keypoint_confidence, layers.py:107-119)
 *          h   if conf_on_prob = 0   (build_joints_probability on raw maps, blocks.py:328-343)
 *   z = sum_hw sigmoid(d) * p  if d != NULL             spnet.py:201-205
 * out_pose: (N, C, 2 or 3) dense; out_conf: (N, C, 1) dense; prob_out (optional,
 * may be NULL-p) receives p for the kronecker product.                        */
int dh_softargmax2d_f32(dh_ctx* ctx, const dh_view* h, const dh_view* d, float alpha,
                        int conf_on_prob, float* out_pose, float* out_conf,
                        const dh_view* prob_out, void* stream);

/* reception.py:167-182 pose_regression_2d_context: h = [hs (nj) | hc (nj*n_ctx)];
 * pose = a*sSAM(hs) + (1-a)*sum_ctx(pc*cSAM(hc))/sum_ctx(pc) (blocks.py:217-285),
 * visible = sjProb(hs) (raw maps).  out_pose (N,nj,2), out_vis (N,nj,1). */
int dh_softargmax2d_ctx_f32(dh_ctx* ctx, const dh_view* h, int nj, int n_ctx, float alpha_mix,
                            float* out_pose, float* out_vis, void* stream);

/* reception.py:193-222 pose_regression_3d: h (N,H,W,D*nj), channel = d*nj + j.
 * out_pose (N,nj,3), out_vis (N,nj,1) = sigmoid(max hxy + max hz). */
int dh_softargmax3d_f32(dh_ctx* ctx, const dh_view* h, int nj, int depth_maps,
                        float* out_pose, float* out_vis, void* stream);

/* deephar/models/action.py:208-297 _get_3d_pose_estimation_from_model (CVPR'18 merge model, 3-D pose): same head as
 * dh_softargmax3d_f32 with visible = sigmoid(vis_scale * (max hxy + max hz)) (vis_scale = 2, action.py:291-292)
 * and, if prob_out != NULL-p, prob_out (N,H,W,nj) = channel_softmax_2d(hxy) for the kronecker product (:294-295). */
int dh_softargmax3d_ex_f32(dh_ctx* ctx, const dh_view* h, int nj, int depth_maps, float vis_scale,
                           float* out_pose, float* out_vis, const dh_view* prob_out, void* stream);

/* layers.py:478-508 kronecker_prod for clips: out[n,j,f] = sum_hw P[n,h,w,j] * Z[n,h,w,f]. */
int dh_kron_pool_f32(dh_ctx* ctx, const dh_view* p, const dh_view* z, float* out, void* stream);

/* --- small action-head ops (spnet.py:51-148) ------------------------------ */
/* keras ZeroPadding2D(((top,bottom),(left,right))) (spnet.py:124-125,131-132): out is the padded view */
int dh_zeropad2d_f32(dh_ctx* ctx, const dh_view* x, int top, int left, const dh_view* out, void* stream);
/* layers.py:411-425 max_min_pooling 2x2 stride 2 'same' */
int dh_maxmin_pool2d_f32(dh_ctx* ctx, const dh_view* x, const dh_view* out, void* stream);
/* layers.py:428-442 + Activation('softmax'): out (B, C) */
int dh_global_maxmin_softmax_f32(dh_ctx* ctx, const dh_view* x, float* out, void* stream);
/* out[b,t,j,:] = p[b,t,j,:] * c[b,t,j,0]   (spnet.py:110-111) */
int dh_mask_mul_f32(dh_ctx* ctx, const float* p, const float* c, int64_t rows, int dim, float* out,
                    void* stream);

/* --- streamed clip inference (deephar_b200/stream.py) ------------------------------------
 * A clip model's per-frame network runs on one new frame per stream; each tensor that crosses from frames to clips
 * (frames_to_clip, layers.py) keeps the last T frames of every stream in a ring, and the clip network reads them as a
 * (S clips, T frames) input.  One entry per crossing tensor: */
typedef struct dh_clip_window {
    dh_view src;                  /* (S, h, w, c): the new frame's tensor, one item per stream (any ld / channel offset) */
    dh_view dst;                  /* (S*T, h, w, c): the clip input, stream-major, frames in time order (any ld) */
    float*  ring;                 /* S*T*h*w*c floats, dense: ring[s][slot] holds one earlier frame of stream s */
} dh_clip_window;
/* One launch for all n_tensors entries of table_dev (device memory): with pos = counter_dev[0],
 *   ring[s][pos] = src[s];  dst[s*T + j] = ring[s][(pos + 1 + j) % T] for j < T-1;  dst[s*T + T-1] = src[s]
 * i.e. the window ends at the new frame, oldest first.  The launch then advances counter_dev[0] to (pos + 1) % T
 * itself (counter_dev[1] is its scratch ticket; zero both before the first launch), so repeated launches need no
 * host writes and can be replayed from a CUDA graph.  All streams advance together; src, dst and ring must not
 * overlap. */
int dh_clip_window_f32(dh_ctx* ctx, const dh_clip_window* table_dev, int n_tensors, int S, int T, int32_t* counter_dev,
                       void* stream);
/* Readiness on the device, so a captured push replays with the counts of the moment it runs (dh_stream_push).
 * After a push: for each stream s, c = min(count[s] + 1, T); count[s] = c; ready[s] = (c >= T).
 * For each of the n_outs views (n = S items, any h/w/c, any ld >= c, channel windows allowed) the elements of
 * item s are set to NaN (0x7FC00000, the bits torch's index_fill_(nan) writes) when !ready[s]; nothing else is written.
 * outs_dev is a device table (may be NULL when n_outs = 0); count_dev and ready_dev hold S int32 each.  Zero count_dev[s]
 * to restart stream s; the count saturates at T. */
int dh_stream_ready_f32(dh_ctx* ctx, int32_t* count_dev, int S, int T, const dh_view* outs_dev, int n_outs,
                        int32_t* ready_dev, void* stream);

/* --- evaluation-time input pipeline (SURVEY.md 8 f4) -----------------------------------
 * deephar/utils/transform.py:60-134 (T.rotate_crop with angle 0 -> crop -> resize(BILINEAR) [-> horizontal_flip]) and
 * :212-231 normalize_channels, as deephar/data/mpii.py:91-122 drives them for evaluation.  One frame: */
typedef struct dh_frame_src {
    const uint8_t* data;          /* decoded RGB image, uint8 HWC, device memory */
    int32_t h, w, stride;         /* size and bytes per row */
    int32_t x0, y0, cw, ch;       /* crop box origin (may lie outside the image: zeros, as PIL) and size */
    int32_t hflip;                /* 1 = Image.transpose(FLIP_LEFT_RIGHT) after the resize */
    int32_t kx_off, ky_off;       /* offsets (in int32) of this frame's (first, count) pairs in `bounds` */
    int32_t kx_coef_off, ky_coef_off;   /* offsets (in int32) of its weight rows in `coefs` */
    int32_t ksx, ksy;             /* taps per output index (row pitch of the weight tables) */
} dh_frame_src;
/* Pillow's two-pass fixed-point bilinear resampler, bit-exact: the weight tables (22-bit fixed point, computed in
 * double exactly like libImaging/Resample.c) come in `bounds` / `coefs`.  Two sources compute them: the Python host
 * (deephar_b200/preprocess.py resample_tables), and dh_prepare_frames_u8 below, which writes the frame table and the
 * tables on the device and then runs this entry's two kernels.
 * tmp: uint8 scratch of n * tmp_stride bytes (tmp_stride >= max_crop_h * out_w * 3); out: (n, out_h, out_w, 3) fp32
 * = ((u8 / 255) ** chpower - 0.5) * 2, i.e. the NHWC input tensor of the network.  chpower3 may be NULL (= 1).
 * A frame with ch = 0 reads nothing and writes NaN in all its elements. */
int dh_crop_resize_norm_u8(dh_ctx* ctx, const dh_frame_src* frames_dev, int n, int max_crop_h,
                           const int32_t* bounds_dev, const int32_t* coefs_dev, int out_h, int out_w,
                           const float* chpower3, uint8_t* tmp_dev, int64_t tmp_stride, float* out_dev, void* stream);

/* Frames from images already in device memory, with the per-frame geometry on the device too: the caller supplies the
 * images and one box record per frame, nothing else.  For each frame, as FramePipeline (deephar_b200/preprocess.py):
 *   box    = [trunc(cx - ww/2), trunc(cy - wh/2), trunc(cx + ww/2), trunc(cy + wh/2)]   (crop_box), cw x ch pixels
 *   tables = resample_tables(cw, out_w) and resample_tables(ch, out_h), bit for bit (same double operations, same order)
 *   afmat  = affine_map(box, (out_w, out_h), hflip == 1): image pixels -> [0, 1]^2 of the frame, float64 row-major 3x3
 * and then the pixels of dh_crop_resize_norm_u8.  A frame whose box cannot be used gets status bits and NaN in all its
 * output elements and its afmat; the other frames are computed as without it. */
typedef struct dh_frame_box {
    const uint8_t* data;          /* decoded RGB image, uint8 HWC, device memory */
    int32_t h, w, stride;         /* size and bytes per row (stride >= 3 w) */
    int32_t hflip;                /* 1 = flip after the resize; any other value: no flip */
    double  objpos[2];            /* crop centre (x, y) in image pixels */
    double  winsize[2];           /* crop width, height */
} dh_frame_box;
#define DH_FRAME_EMPTY      1     /* cw < 1 or ch < 1 (FramePipeline raises) */
#define DH_FRAME_TOO_LARGE  2     /* cw > max_crop_w or ch > max_crop_h */
#define DH_FRAME_BAD_BOX    4     /* objpos / winsize not finite, a box edge outside int32, or an image with h < 0,
                                     w < 0, stride < 3 w or a NULL data pointer */
/* Bytes of workspace dh_prepare_frames_u8 needs for these sizes (< 0 with the reason for sizes it refuses).  With
 * kx = 2 ceil(max(max_crop_w / out_w, 1)) + 1 and ky = 2 ceil(max(max_crop_h / out_h, 1)) + 1 (the taps of the widest
 * crop), frame i's entries live at (byte offsets from ws; up(v, a) rounds v up to a multiple of a):
 *   frames  0                                       dh_frame_src[n]
 *   bounds  B = up(64 n, 256)                       int32 (first, count) pairs: frame i at B + 4 i (2 out_w + 2 out_h),
 *                                                   its out_w x-axis pairs, then its out_h y-axis pairs
 *   coefs   K = up(B + 8 n (out_w + out_h), 256)    int32 weights: frame i at K + 4 i (out_w kx + out_h ky), x rows
 *                                                   of ksx = 2 ceil(max(cw / out_w, 1)) + 1 taps, then at + 4 out_w kx
 *                                                   the y rows of ksy taps (ksx, ksy: the frame's dh_frame_src)
 *   tmp     X = up(K + 4 n (out_w kx + out_h ky), 256)   uint8 scratch of the horizontal pass, n x up(max_crop_h out_w 3, 16)
 * Tables of flagged frames are not written.  Refused: n outside [0, 65535], a size outside [1, 262144], or more than
 * 2^31 - 1 int32 of bounds or of coefs. */
int64_t dh_prepare_frames_workspace(int n, int max_crop_w, int max_crop_h, int out_h, int out_w);
/* Three launches on `stream` (geometry, then the two passes of dh_crop_resize_norm_u8), no host synchronisation: the
 * call can be captured into a CUDA graph.  boxes_dev: n records in device memory; ws: ws_bytes >= the size above,
 * 256-byte aligned; out_dev: (n, out_h, out_w, 3) fp32; afmat_dev: (n, 3, 3) double; status_dev: n int32, 0 or an OR
 * of DH_FRAME_*.  chpower3 (host, may be NULL) as in dh_crop_resize_norm_u8.  A refused call (bad sizes, NULL
 * pointers, a short workspace) returns < 0 and launches nothing. */
int dh_prepare_frames_u8(dh_ctx* ctx, const dh_frame_box* boxes_dev, int n, int max_crop_w, int max_crop_h, int out_h,
                         int out_w, const float* chpower3, void* ws, int64_t ws_bytes, float* out_dev, double* afmat_dev,
                         int32_t* status_dev, void* stream);

/* --- baseline JPEG decoding in front of the input pipeline ------------------------------
 * Pillow's Image.open(...).convert('RGB') of a baseline JPEG as its libjpeg-turbo computes it (Huffman decoding, ISLOW
 * integer IDCT, fancy upsampling, integer YCbCr -> RGB), bit for bit.  The host (deephar_b200/jpeg.py) parses the
 * markers, keeps the files the decoder takes (8-bit sequential Huffman, one interleaved scan, grey or YCbCr with
 * luma sampling 1x1 / 2x1 / 2x2 and chroma 1x1) and uploads, in one copy, the tables below and the entropy-coded
 * bytes.  Offsets are relative to the pointers of dh_jpeg_batch. */
typedef struct dh_jpeg_image {
    int64_t data;                 /* bytes: the image's entropy-coded data in `data` */
    int64_t coef[3];              /* int16 elements: each component's coefficient blocks in `coef` (64 per block) */
    int64_t plane[3];             /* bytes: each component's sample plane (bh*8 rows of bw*8) in `planes` */
    int64_t out;                  /* bytes: the packed RGB (h, w, 3) image in `out` */
    int32_t h, w;
    int32_t ncomp;                /* 1 (grey, replicated to RGB) or 3 (YCbCr) */
    int32_t hs, vs;               /* luma sampling factors, 1 or 2; chroma is 1 x 1 */
    int32_t mcus_x, mcus_y;
    int32_t bw[3], bh[3];         /* blocks per row / column of each component, padded to whole MCUs */
    int32_t qt[3], dc[3], ac[3];  /* each component's quantisation table (index into qtab) and Huffman tables */
    int32_t nblocks;              /* blocks of all components */
    int32_t pad;
} dh_jpeg_image;
typedef struct dh_jpeg_segment {  /* one restart interval, or the whole scan without restart markers */
    int64_t begin, end;           /* bytes in `data`, markers excluded (0xFF00 still stuffed) */
    int32_t image, mcu0, mcus, pad;
} dh_jpeg_segment;
typedef struct dh_jpeg_huff {     /* canonical decoding tables of one DHT table */
    uint16_t lut[512];            /* next 9 bits -> (length << 8) | symbol, 0 = code longer than 9 bits */
    int32_t maxcode[18];          /* largest code of each length 10..16 (-1: none) */
    int32_t valoff[18];           /* symbol index - code for the codes of each length */
    uint8_t vals[256];
} dh_jpeg_huff;
typedef struct dh_jpeg_batch {
    const dh_jpeg_image* images;  /* device memory, n_images entries */
    const dh_jpeg_segment* segments;
    const dh_jpeg_huff* huff;
    const uint16_t* qtab;         /* 64 entries per table, natural order */
    const uint8_t* data;
    int16_t* coef;                /* workspace: coef_elems int16 coefficients */
    uint8_t* planes;              /* workspace: component planes */
    uint8_t* out;                 /* RGB images */
    int32_t* status;              /* per image, 0 = decoded; otherwise an OR of DH_JPEG_* -- decode it on the host */
    int64_t coef_elems;
    int32_t n_images, n_segments;
    int32_t max_blocks;           /* largest nblocks of one image */
    int32_t max_h, max_w;
    int32_t pad;
} dh_jpeg_batch;
#define DH_JPEG_BAD_CODE   1      /* a Huffman code that no table holds */
#define DH_JPEG_NO_DATA    2      /* an interval ran out of entropy-coded data */
#define DH_JPEG_BAD_INDEX  4      /* a run of zeros past coefficient 63, or a DC value outside 16 bits */
#define DH_JPEG_RANGE      8      /* an IDCT left the range in which libjpeg-turbo's C and SIMD IDCTs agree */
/* stages: bit 0 = entropy decoding (zeroes coef and status first; one thread per segment), bit 1 = dequantisation +
 * IDCT (one thread per block), bit 2 = upsampling + colour conversion (one thread per pixel); 7 = the whole decode. */
int dh_jpeg_decode(dh_ctx* ctx, const dh_jpeg_batch* batch, int stages, void* stream);

/* --- evaluator-side post-processing (SURVEY.md 8 f3) ------------------------------
 * deephar/utils/transform.py:136-209 transform_pose_sequence(A, poses, inverse) + deephar/measures.py:5-93
 * (pckh, mean_distance_error) as the evaluators use them after predict (exp/common/mpii_tools.py:93-129):
 *   out_pose[n,j,:] = (M_n [x, y, 1]^T)[0:2],  M_n = inverse ? inv(A_n) : A_n   (fp64 inverse, like np.linalg.inv)
 * and, if y_true != NULL, per joint j over the samples whose annotation is valid (both coords > -1e6):
 *   valid[j] += 1;  dist_sum[j] += |y_true - out_pose|;  hits[j] += (dist / head_size[n] <= refp)
 * (head_size may be NULL: plain distance threshold).  Every array and refp is double, as the reference's numpy
 * arithmetic, and the distance is rounded as measures.py rounds it, so hits equal the reference's count for count.
 * pred: (N, nj, pred_ld >= 2) device doubles; afmat: (N,3,3) if per_sample_mat else (1,3,3); out_pose: (N, nj, 2);
 * hits / valid: int32 (nj), dist_sum: double (nj), accumulated (zero them first).  PCKh = sum(hits[used]) /
 * sum(valid[used]).  A singular afmat with inverse = 1 gives NaN poses (valid, never a hit, NaN in dist_sum). */
int dh_pose_eval_f64(dh_ctx* ctx, const double* pred, int pred_ld, const double* afmat, int per_sample_mat,
                     int inverse, const double* y_true, const double* head_size, double refp, int N, int nj,
                     double* out_pose, int* hits, int* valid, double* dist_sum, void* stream);
/* The transform of dh_pose_eval_f64 with inverse = 1 on float32 poses, read through the view dh_model_output /
 * dh_stream_output report: n items of h * w points, coordinates (x, y) = channels 0, 1 of c >= 2 (ld >= c).  Each
 * coordinate is widened exactly to double, so out equals dh_pose_eval_f64 on the widened poses bit for bit.
 * afmat: (n, 3, 3) if per_sample_mat else (1, 3, 3), e.g. dh_prepare_frames_u8's; out: (n, h * w, 2) double. */
int dh_pose_to_image_f32(dh_ctx* ctx, const dh_view* poses, const double* afmat, int per_sample_mat, double* out,
                         void* stream);

/* --- multi-GPU exchange step (SURVEY.md 8e) ---------------------------------
 * One process per GPU; the clip batch is sharded, weights replicated, and the ONLY communication of the forward
 * path is an all-gather of the per-rank outputs (action probabilities, optionally poses).  The reference has
 * no multi-GPU path (single process: exp/ntu/eval_ntu_multitask.py:35-54); these calls are what a data-parallel
 * evaluator runs after Model.predict() on its shard.  NCCL is bound at run time (dlopen), no link dependency.
 * Return values > 1000 are ncclResult_t + 1000. */
/* rank 0: 128-byte ncclUniqueId to hand to every rank (any out-of-band channel: torch.distributed store, MPI, file) */
int dh_comm_unique_id(void* out128);
/* collective over all `world` ranks (each with its own ctx / device) */
int dh_comm_init(dh_ctx* ctx, int rank, int world, const void* unique_id128);
int dh_comm_destroy(dh_ctx* ctx);
/* recv[r*count .. (r+1)*count) = rank r's send[0 .. count); fp32 device buffers; asynchronous on `stream` */
int dh_allgather_f32(dh_ctx* ctx, const float* send, float* recv, int64_t count, void* stream);
/* rank / world of the context's communicator (-1 / 0 if none) and the NCCL version in use (0 if not loadable) */
int dh_comm_info(dh_ctx* ctx, int* rank, int* world, int* nccl_version);

/* --- whole model (Model.export, deephar_b200/export.py) -------------------------------------------------------------
 * A compiled network bound to one batch size, written by the Python `Model.export(path, n_frames)` (also on split_model
 * / output_subset views), is run here with no Python in the process: the file holds the launch list the Python host
 * binds -- every launch of the entry points above with its arguments -- so kernel choice, fusion and buffer planning are
 * the Python compiler's, and the C side replays them.  A loaded model runs at the batch it was exported at, N items of
 * the input's first axis (frames, or clips of a clip model); dh_model_set_batch runs it at any n <= N with the same
 * launches, weights and memory.
 *
 * File format, version 2, little-endian, no padding between fields:
 *   char    magic[8]            "DHMODEL\0"
 *   u32     version             2 (version 1: the same without the kind table; it runs at its exported batch only)
 *   i32     precision           of the tensor-core convolutions (dh_conv_desc.precision)
 *   i32     use_tensor_cores    1 = packed bf16 hi / lo operands are recorded
 *   i32     frame_items, clip_items, frames_per_clip     items of each tensor kind, T
 *   shape   input               the Keras input shape, batch axes included
 *   i64 W,  u8[W]               arena 0: fp32 weights (folded BatchNormalization and constant vectors included)
 *   i64 Q,  u8[Q]               arena 1: bf16 hi / lo tensor-core operands
 *   i32 S,  i64[S]              arenas 3 .. 3+S-1: byte sizes of the activation slots
 *   u8[S]                       the slots' kinds: 0 = frame items (N*T per batch), 1 = clip items (N)
 *   i64                         arena 2: byte size of the convolution workspace
 *   view                        the input (dense; the caller writes it before dh_model_forward)
 *   i32 O,  O x { view, shape, i32 len, char[len] name }          the outputs, with their Keras shapes
 *   i32 L,  L x { i32 entry, i32 nargs, i32 len, char[len] label, nargs x { u8 tag, payload } }
 * where shape = i32 rank (1..DH_MODEL_MAX_RANK) + i64[rank]; ptr = i32 arena (-1 = NULL) + i64 byte offset in it;
 * view = the fields of dh_view in order (ptr p, i32 n, h, w, c, ld).  entry: 0 dh_conv2d_f32, 1 dh_sepconv2d_f32,
 * 2 dh_maxpool2d_f32, 3 dh_upsample2x_add_f32, 4 dh_add_n_f32, 5 dh_softargmax2d_f32, 6 dh_softargmax2d_ctx_f32,
 * 7 dh_softargmax3d_f32, 8 dh_softargmax3d_ex_f32, 9 dh_kron_pool_f32, 10 dh_zeropad2d_f32, 11 dh_maxmin_pool2d_f32,
 * 12 dh_global_maxmin_softmax_f32, 13 dh_mask_mul_f32; its arguments are those between `ctx` and `stream`, each:
 *   'i' i64 integer   'f' f32   'p' ptr   'v' i32 count + count views (0 = NULL pointer; dh_add_n_f32: n_in views)
 *   'd' i32 count (1) + dh_conv_desc field by field   'w' i32 count (0 = NULL, 1) + dh_packed_w (ptr hi, ptr lo, i32 x2)
 * The file ends after the last launch.  Loading checks everything before a kernel can see it: the signature of every
 * launch, integer ranges, every pointer's offset and extent against its arena, and each convolution through
 * dh_conv2d_plan / dh_sepconv2d_plan.  A malformed file returns < 0 with the reason (and the launch) in dh_last_error.
 * In version 2 it also checks what running at another batch relies on: every view into an activation slot has the
 * exported item count of its slot's kind (N clips, N*T frames, or N clips of T frames where a clip tensor reads a frame
 * slot), dh_mask_mul_f32's rows over a slot are a multiple of N, and every output's shape[0] is N. */
#define DH_MODEL_VERSION   2
#define DH_MODEL_MAX_RANK  6
typedef struct dh_model dh_model;
typedef struct dh_model_output_info {
    char    name[64];             /* the output layer's name, NUL-terminated (truncated) */
    int32_t rank;
    int32_t pad;
    int64_t shape[DH_MODEL_MAX_RANK];   /* Keras shape: (items, ...) or (clips, T, ...); unused entries 0 */
} dh_model_output_info;
typedef struct dh_model_info {
    int32_t version, precision, use_tensor_cores;
    int32_t frame_items, clip_items, frames_per_clip;
    int32_t input_rank, n_outputs;
    int64_t input_shape[DH_MODEL_MAX_RANK];
    int64_t n_launches;           /* launches of one dh_model_forward */
    int64_t n_slots;
    int64_t weight_bytes, packed_bytes, workspace_bytes, activation_bytes;   /* activation: sum of the slots */
    int64_t device_bytes;         /* what dh_model_load allocates (one allocation; arenas 512-byte aligned) */
} dh_model_info;
/* Host-only (no device, no context): parse and check a file.  slot_bytes (max_slots entries) and outputs (max_outputs)
 * may be NULL; the first min(count, max) entries are filled. */
int dh_model_inspect(const char* path, dh_model_info* info, int64_t* slot_bytes, int max_slots,
                     dh_model_output_info* outputs, int max_outputs);
/* Read and check a file, allocate its arenas on ctx's device (activations zeroed), upload the weights and plan every
 * convolution.  The model keeps ctx: destroy the model first. */
int dh_model_load(dh_ctx* ctx, const char* path, dh_model** out);
/* Run the model at n items of the input's first axis (frames, or clips of a clip model), 1 <= n <= N, the exported batch
 * that dh_model_load starts at.  Host-only (no device work, no launch): every launch's item counts are rewritten for n
 * and every convolution is planned again, within the file's workspace; dh_model_input / dh_model_output then report
 * views of n items (shape[0] = n) and dh_model_forward issues the same launches at n items, at no extra cost per
 * forward.  Items n .. N-1 of the outputs are left as they were, and the device memory stays the N-item allocation.
 * A CUDA graph captured from dh_model_forward keeps the batch it was captured at: capture one graph per batch size.
 * Atomic: a refused call (n out of range, a convolution no kernel takes at n, a version-1 file with n != N) returns < 0
 * with the reason in dh_last_error and leaves the previous batch in force. */
int dh_model_set_batch(dh_model* m, int n);
/* the batch forwards run at (< 0 if m is NULL) */
int dh_model_batch(const dh_model* m);
/* the dense input view: write the current batch's frames (or clips x T frames) there before a forward */
int dh_model_input(const dh_model* m, dh_view* view);
/* Set ctx's workspace to the model's and issue every launch on `stream`, in order.  No host synchronisation, so the
 * call may be captured into a CUDA graph; models in one ctx are independent, but forwards of one model are not
 * reentrant (they share its activations). */
int dh_model_forward(dh_model* m, void* stream);
/* output k at the current batch: its view into the activations (valid until dh_model_free or the next
 * dh_model_set_batch; possibly a channel window, ld >= c) and its shape */
int dh_model_output(const dh_model* m, int k, dh_view* view, dh_model_output_info* info);
/* free every device and host allocation of the model (synchronises the device before freeing) */
int dh_model_free(dh_model* m);

/* --- live video (ClipStream.export, deephar_b200/export.py) ---------------------------------------------------------
 * What a ClipStream (deephar_b200/stream.py) binds, written by the Python `ClipStream.export(path)`: S streams advancing
 * one frame per dh_stream_push through a clip model's frame stage (bound at S frames), the window kernel
 * (dh_clip_window_f32) and its clip stage (bound at S*T frames), then dh_stream_ready_f32.  Ring position, per-stream
 * counts and ready flags live on the device, so a push can be captured into a CUDA graph and replayed.  The stream's
 * run-time state is not recorded: a loaded stream starts with empty rings and every stream not ready.
 *
 * File format, version 1, little-endian, no padding; shape, ptr, view and the launch records as in the model format:
 *   char    magic[9]            "DHSTREAM\0"
 *   u32     version             1
 *   i32     precision, use_tensor_cores, S, T
 *   shape   input               (S, H, W, 3)
 *   i64 W,  u8[W]               arena 0: fp32 weights
 *   i64 Q,  u8[Q]               arena 1: bf16 hi / lo tensor-core operands
 *   i32 F,  i64[F]              arenas 4 .. 4+F-1: byte sizes of the frame stage's activation slots
 *   i64                         arena 2: byte size of the frame stage's workspace
 *   i32 C,  i64[C]              arenas 4+F .. 4+F+C-1: the clip stage's slots
 *   i64                         arena 3: byte size of the clip stage's workspace
 *   i32 B,  i64[B]              arenas 4+F+C .. 4+F+C+B-1: the rings (S*T*h*w*c floats each)
 *   B x { view src, view dst, ptr ring }     the boundary table (dh_clip_window): src in a frame slot (n = S), dst in
 *                                            a clip slot (n = S*T), ring = offset 0 of a ring arena
 *   view                        the input (dense, a frame slot)
 *   i32 OF, OF x { view, shape, i32 len, char[len] name }     frame outputs, shape (S, ...)
 *   i32 OC, OC x { view, shape, i32 len, char[len] name }     clip outputs, shape (S, ...)
 *   i32 LF, LF x launch          the frame stage: its pointers lie in arenas 0, 1 and the frame slots
 *   i32 LC, LC x launch          the clip stage: arenas 0, 1 and the clip slots
 * Loading makes every check of the model format on both launch lists, and refuses a launch that points into the other
 * stage's slots or a ring, boundaries whose views disagree with S, T or each other, a ring of the wrong size,
 * overlapping src / dst / ring, and outputs with n != S. */
#define DH_STREAM_VERSION  1
typedef struct dh_stream dh_stream;
typedef struct dh_stream_info {
    int32_t version, precision, use_tensor_cores;
    int32_t n_streams, frames_per_clip;             /* S, T */
    int32_t input_rank;
    int64_t input_shape[DH_MODEL_MAX_RANK];         /* (S, H, W, 3) */
    int32_t n_frame_outputs, n_clip_outputs;        /* dh_stream_output k: frame outputs first, then clip outputs */
    int32_t n_boundary;                             /* tensors crossing from the frame to the clip stage */
    int32_t pad;
    int64_t n_frame_launches, n_clip_launches;
    int64_t n_frame_slots, n_clip_slots;
    int64_t weight_bytes, packed_bytes;
    int64_t frame_workspace_bytes, clip_workspace_bytes;
    int64_t activation_bytes;                       /* the slots of both stages */
    int64_t ring_bytes;                             /* all rings */
    int64_t device_bytes;                           /* what dh_stream_load allocates (one allocation) */
} dh_stream_info;
/* Host-only (no device, no context): parse and check a file.  outputs (max_outputs entries) may be NULL. */
int dh_stream_inspect(const char* path, dh_stream_info* info, dh_model_output_info* outputs, int max_outputs);
/* Read and check a file, allocate everything in one device allocation (activations, rings and counters zeroed), upload
 * the weights and plan every convolution.  The stream keeps ctx: free the stream first. */
int dh_stream_load(dh_ctx* ctx, const char* path, dh_stream** out);
/* the dense (S, H, W, 3) input view: one new frame per stream, written before each push */
int dh_stream_input(const dh_stream* st, dh_view* view);
/* One frame per stream: frame stage, window, clip stage, readiness -- the launches of a ClipStream.push plus one, all
 * on `stream`, no host synchronisation: a push may be captured into a CUDA graph and replayed. */
int dh_stream_push(dh_stream* st, void* stream);
/* Restart streams ids[0..n) (ids NULL = all): their counts are zeroed on `stream`, ordered with the pushes.  Every id is
 * checked against [0, S) before anything is enqueued. */
int dh_stream_reset(dh_stream* st, const int32_t* ids, int n, void* stream);
/* output k (k < n_frame_outputs: frame output k, else clip output k - n_frame_outputs): its view and (S, ...) shape.
 * Clip-output items of streams that are not ready are NaN. */
int dh_stream_output(const dh_stream* st, int k, dh_view* view, dh_model_output_info* info);
/* the S int32 ready flags (device memory) each push writes: 1 = the stream has had >= T frames since its reset */
int dh_stream_ready(const dh_stream* st, const int32_t** ready_dev);
/* free every device and host allocation of the stream (synchronises the device before freeing) */
int dh_stream_free(dh_stream* st);

#ifdef __cplusplus
}
#endif
#endif /* DEEPHAR_B200_H */
