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
                                    (only the last residual; tensor-core kernels, Wo == 16 or Wo % 32 == 0) */
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
 * double on the host exactly like libImaging/Resample.c: deephar_b200/preprocess.py) come in `bounds` / `coefs`;
 * tmp: uint8 scratch of n * tmp_stride bytes (tmp_stride >= max_crop_h * out_w * 3); out: (n, out_h, out_w, 3) fp32
 * = ((u8 / 255) ** chpower - 0.5) * 2, i.e. the NHWC input tensor of the network.  chpower3 may be NULL (= 1). */
int dh_crop_resize_norm_u8(dh_ctx* ctx, const dh_frame_src* frames_dev, int n, int max_crop_h,
                           const int32_t* bounds_dev, const int32_t* coefs_dev, int out_h, int out_w,
                           const float* chpower3, uint8_t* tmp_dev, int64_t tmp_stride, float* out_dev, void* stream);

/* --- evaluator-side post-processing (SURVEY.md 8 f3) ------------------------------
 * deephar/utils/transform.py:136-209 transform_pose_sequence(A, poses, inverse) + deephar/measures.py:5-93
 * (pckh, mean_distance_error) as the evaluators use them after predict (exp/common/mpii_tools.py:93-129):
 *   out_pose[n,j,:] = (M_n [x, y, 1]^T)[0:2],  M_n = inverse ? inv(A_n) : A_n   (fp64 inverse, like np.linalg.inv)
 * and, if y_true != NULL, per joint j over the samples whose annotation is valid (both coords > -1e6):
 *   valid[j] += 1;  dist_sum[j] += |y_true - out_pose|;  hits[j] += (dist / head_size[n] <= refp)
 * (head_size may be NULL: plain distance threshold).  pred: (N, nj, pred_ld >= 2) device floats;
 * afmat: (N,3,3) if per_sample_mat else (1,3,3); hits / valid: int32 (nj), dist_sum: double (nj), accumulated
 * (zero them first).  PCKh = sum(hits[used]) / sum(valid[used]). */
int dh_pose_eval_f32(dh_ctx* ctx, const float* pred, int pred_ld, const float* afmat, int per_sample_mat,
                     int inverse, const float* y_true, const float* head_size, float refp, int N, int nj,
                     float* out_pose, int* hits, int* valid, double* dist_sum, void* stream);

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

#ifdef __cplusplus
}
#endif
#endif /* DEEPHAR_B200_H */
