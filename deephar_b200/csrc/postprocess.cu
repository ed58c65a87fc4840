// Evaluator-side post-processing on the GPU (SURVEY.md 8 f3): what the reference's evaluators do in numpy
// after model.predict -- map the predicted poses back to the original image with the inverse of the crop's
// affine matrix and score them against the annotations:
//   transform_pose_sequence(A, poses, inverse=True)          deephar/utils/transform.py:136-209
//   pckh / pckh_per_joint / mean_distance_error              deephar/measures.py:5-93
//   (driver: exp/common/mpii_tools.py:93-129, h36m_tools.py:58-99)
// One kernel, one thread per (sample, joint), all in fp64 as the reference's numpy code: 3x3 inverse (np.linalg.inv),
// transformed pose written back, per-joint hit / valid counters and distance sums accumulated with atomics -- the
// poses never leave the device between the soft-argmax head and the score.  Every input is a double, the threshold
// too: a float32 `refp`, annotation or head size moves samples within ~1e-7 relative of the threshold across it
// (d = float32(0.2) is a miss in the reference and would be a hit against (double)0.2f).  The distance is rounded as
// measures.py rounds it (x*x + y*y, sqrt, / head_size: no fused multiply-add), so a pose equal to the reference's
// gives the reference's hit bit for bit.
// A singular A with inverse = 1 (np.linalg.inv raises there) gives NaN poses: such a joint still counts as valid
// when its annotation is, adds NaN to dist_sum and is never a hit.
#include "common.cuh"

namespace {

struct PoseEvalParams {
    const double* pred; int ldp;     // (N, nj, >=2) predicted poses, crop-normalised coordinates
    const double* afmat;             // (N, 3, 3) or (1, 3, 3) row-major affine maps (image -> crop)
    int per_sample_mat;
    const double* y_true;            // (N, nj, 2) annotations in image coordinates, or NULL (transform only)
    const double* head_size;         // (N,) or NULL (distance not normalised)
    double refp;
    int N, nj;
    double* out_pose;                // (N, nj, 2)
    int* hits; int* valid;           // (nj,) accumulated
    double* dist_sum;                // (nj,) accumulated (valid joints only)
};

__device__ __forceinline__ bool inv3x3(const double* a, double* o) {
    const double a00 = a[0], a01 = a[1], a02 = a[2], a10 = a[3], a11 = a[4], a12 = a[5], a20 = a[6], a21 = a[7], a22 = a[8];
    const double c00 = a11 * a22 - a12 * a21, c01 = a12 * a20 - a10 * a22, c02 = a10 * a21 - a11 * a20;
    const double det = a00 * c00 + a01 * c01 + a02 * c02;
    if (det == 0.0) return false;
    const double r = 1.0 / det;
    o[0] = c00 * r; o[1] = (a02 * a21 - a01 * a22) * r; o[2] = (a01 * a12 - a02 * a11) * r;
    o[3] = c01 * r; o[4] = (a00 * a22 - a02 * a20) * r; o[5] = (a02 * a10 - a00 * a12) * r;
    o[6] = c02 * r; o[7] = (a01 * a20 - a00 * a21) * r; o[8] = (a00 * a11 - a01 * a10) * r;
    return true;
}

// transform_pose_sequence of one point: (M [x, y, 1]^T)[0:2], M = inverse ? inv(A) : A (NaN when A is singular).  The
// one copy of this arithmetic: dh_pose_eval_f64 and dh_pose_to_image_f32 give the same bits for the same doubles.
__device__ __forceinline__ void transform_point(const double* A, int inverse, double x, double y, double* tx, double* ty) {
    double M[9];
    if (inverse) {
        if (!inv3x3(A, M)) { for (int k = 0; k < 9; ++k) M[k] = nan(""); }
    } else {
        for (int k = 0; k < 9; ++k) M[k] = A[k];
    }
    // transform_2d_points: y = (A [x, y, 1]^T)[0:2]  (no homogeneous division: the maps are affine)
    *tx = M[0] * x + M[1] * y + M[2];
    *ty = M[3] * x + M[4] * y + M[5];
}

__global__ void pose_eval_kernel(PoseEvalParams p, int inverse) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= p.N * p.nj) return;
    const int n = i / p.nj, j = i - n * p.nj;
    const double* A = p.afmat + (p.per_sample_mat ? (size_t)n * 9 : 0);
    double tx, ty;
    transform_point(A, inverse, p.pred[(size_t)i * p.ldp + 0], p.pred[(size_t)i * p.ldp + 1], &tx, &ty);
    p.out_pose[(size_t)i * 2 + 0] = tx;
    p.out_pose[(size_t)i * 2 + 1] = ty;
    if (p.y_true) {
        const double gx = p.y_true[(size_t)i * 2 + 0], gy = p.y_true[(size_t)i * 2 + 1];
        const bool ok = gx > -1e6 && gy > -1e6;                 // measures.py:9-16 _valid_joints
        if (ok) {
            const double dx = gx - tx, dy = gy - ty;
            double d = sqrt(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)));   // measures.py:5-6 _norm
            atomicAdd(p.valid + j, 1);
            atomicAdd(p.dist_sum + j, d);
            if (p.head_size) d /= p.head_size[n];
            if (d <= p.refp) atomicAdd(p.hits + j, 1);
        }
    }
}

// one thread per point of a float32 pose view: items v.n of v.h * v.w points, (x, y) in channels 0, 1
__global__ void pose_to_image_kernel(dh_view v, const double* __restrict__ afmat, int per_sample_mat,
                                     double* __restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t points = (int64_t)v.h * v.w;
    if (i >= v.n * points) return;
    const int64_t n = i / points;
    const float* q = v.p + i * v.ld;
    double tx, ty;
    transform_point(afmat + (per_sample_mat ? n * 9 : 0), 1, (double)q[0], (double)q[1], &tx, &ty);
    out[i * 2 + 0] = tx;
    out[i * 2 + 1] = ty;
}

}  // namespace

extern "C" int dh_pose_eval_f64(dh_ctx* ctx, const double* pred, int pred_ld, const double* afmat, int per_sample_mat,
                                int inverse, const double* y_true, const double* head_size, double refp, int N, int nj,
                                double* out_pose, int* hits, int* valid, double* dist_sum, void* stream) {
    DH_CHECK_ARG(ctx && pred && afmat && out_pose, "dh_pose_eval_f64: NULL argument");
    DH_CHECK_ARG(N >= 0 && nj >= 1 && pred_ld >= 2, "dh_pose_eval_f64: bad sizes");
    DH_CHECK_ARG(!y_true || (hits && valid && dist_sum), "dh_pose_eval_f64: y_true needs the hits / valid / dist_sum accumulators");
    if (N == 0) return 0;
    PoseEvalParams p;
    p.pred = pred; p.ldp = pred_ld; p.afmat = afmat; p.per_sample_mat = per_sample_mat; p.y_true = y_true;
    p.head_size = head_size; p.refp = refp; p.N = N; p.nj = nj; p.out_pose = out_pose; p.hits = hits; p.valid = valid;
    p.dist_sum = dist_sum;
    const int total = N * nj;
    pose_eval_kernel<<<(total + 255) / 256, 256, 0, (cudaStream_t)stream>>>(p, inverse);
    DH_LAUNCH_EPILOGUE(ctx, 1);
}

extern "C" int dh_pose_to_image_f32(dh_ctx* ctx, const dh_view* poses, const double* afmat, int per_sample_mat, double* out,
                                    void* stream) {
    DH_CHECK_ARG(ctx && poses && afmat && out, "dh_pose_to_image_f32: NULL argument");
    const dh_view v = *poses;
    DH_CHECK_ARG(v.n >= 0 && v.h >= 1 && v.w >= 1 && v.c >= 2 && v.ld >= v.c, "dh_pose_to_image_f32: bad pose view");
    DH_CHECK_ARG(v.p || v.n == 0, "dh_pose_to_image_f32: NULL pose view");
    const int64_t total = (int64_t)v.n * v.h * v.w;
    DH_CHECK_ARG(total <= ((int64_t)1 << 40), "dh_pose_to_image_f32: too many points");
    if (total == 0) return 0;
    pose_to_image_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(v, afmat, per_sample_mat, out);
    DH_LAUNCH_EPILOGUE(ctx, 1);
}
