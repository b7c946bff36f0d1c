// Per-Gaussian 3D geometry shared by every kernel that builds a Gaussian's covariance from its parameters: K1 / K8
// (project.cu) and the 3DGS-MCMC position noise (mcmc.cu).  One copy of the quaternion -> rotation formula and of
// cov3D = (R S)(R S)^T, so the covariance the noise is shaped by is the one the rasterizer projects.
#pragma once
#include "common.cuh"

namespace b200gs {

namespace {

// ---- arithmetic with the evaluation order written out ---------------------------------------------------------------------
// The same inline function compiled into two kernels is NOT guaranteed to round the same way: where a product has several uses (x*x,
// b*b, ...) nvcc's fmul+fadd -> fma contraction depends on the surrounding code (observed: the SH colours of the single-view
// K1 and of the multi-view K1 of the sharded renderer differed in the last bit for ~1 % of the splats -> a sharded image 1 ulp off
// the single-GPU image).  Everything the FORWARD projection computes therefore goes through these helpers: __fmul_rn / __fadd_rn /
// __fmaf_rn (and the double versions) are never contracted, split or reassociated, so every kernel that inlines the functions below
// produces the same bits (tests/test_gpu_sharded_kernels.py).
__device__ __forceinline__ float xm(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float xa(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float xf(float a, float b, float c) { return __fmaf_rn(a, b, c); }
__device__ __forceinline__ double xm(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double xa(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double xf(double a, double b, double c) { return __fma_rn(a, b, c); }

// Geometry shared by forward and backward.  R = double in the forward: the conic is the inverse of a 2x2 matrix whose
// condition number reaches 1e4 for elongated splats, so fp32 intermediates put ~1e-4 of noise on pixels (measured: two
// fp32 evaluation orders of the same formulas differ by 1.1e-4 on a 256x256 render).  Evaluating the ~150 flops per
// Gaussian in fp64 (inputs and outputs stay fp32) removes that noise at a small cost per Gaussian.
template <typename R>
struct Proj {
    R tx, ty, tz;        // camera-space mean
    R cxp, cyp;          // clamped tx', ty' used in J
    bool clx, cly;       // clamp active
    R fx, fy;            // focal used by J
    R Rm[9];             // rotation from quaternion (row major)
    R s[3];              // scales * modifier
    R S3[6];             // cov3D upper triangle xx xy xz yy yz zz
    R T[6];              // T = J * Rw, rows 0,1 (2x3)
    R a, b, c, det;      // blurred cov2D and determinant
    R a0, c0, det0;      // un-blurred diag and determinant (gsplat compensation)
};

template <typename R>
__device__ __forceinline__ void quat_to_rot(const R* q, R* Rm) {
    const R r = q[0], x = q[1], y = q[2], z = q[3];
    const R two = R(2), one = R(1);
    Rm[0] = xf(-two, xf(z, z, xm(y, y)), one); Rm[1] = xm(two, xf(-r, z, xm(x, y))); Rm[2] = xm(two, xf(r, y, xm(x, z)));
    Rm[3] = xm(two, xf(r, z, xm(x, y))); Rm[4] = xf(-two, xf(z, z, xm(x, x)), one); Rm[5] = xm(two, xf(-r, x, xm(y, z)));
    Rm[6] = xm(two, xf(-r, y, xm(x, z))); Rm[7] = xm(two, xf(r, x, xm(y, z))); Rm[8] = xf(-two, xf(y, y, xm(x, x)), one);
}

// The camera-independent half of the geometry: rotation, scaled axes, cov3D = (R S)(R S)^T.  The multi-view kernels of the sharded
// renderer evaluate it ONCE per Gaussian (scale_modifier of views[0]) and only project_view per camera.
template <typename R>
__device__ __forceinline__ void gaussian_cov3d(const R* sc, const R* q, float scale_modifier, Proj<R>& g) {
    quat_to_rot<R>(q, g.Rm);
#pragma unroll
    for (int k = 0; k < 3; ++k) g.s[k] = xm(sc[k], R(scale_modifier));
    R M[9];
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int k = 0; k < 3; ++k) M[i * 3 + k] = xm(g.Rm[i * 3 + k], g.s[k]);
    g.S3[0] = xf(M[2], M[2], xf(M[1], M[1], xm(M[0], M[0])));
    g.S3[1] = xf(M[2], M[5], xf(M[1], M[4], xm(M[0], M[3])));
    g.S3[2] = xf(M[2], M[8], xf(M[1], M[7], xm(M[0], M[6])));
    g.S3[3] = xf(M[5], M[5], xf(M[4], M[4], xm(M[3], M[3])));
    g.S3[4] = xf(M[5], M[8], xf(M[4], M[7], xm(M[3], M[6])));
    g.S3[5] = xf(M[8], M[8], xf(M[7], M[7], xm(M[6], M[6])));
}

// Scales and unit quaternion of Gaussian i.  RAW: the model's raw parameters, activated here (exp of the log-scales,
// F.normalize of the quaternion); *inv_qnorm receives 1 / max(|q|, 1e-12) for the backward of the normalisation.
template <bool RAW, typename R>
__device__ __forceinline__ void load_scale_quat(const float* __restrict__ scales, const float* __restrict__ quats, int64_t i, R* sc, R* q,
                                                R* inv_qnorm) {
    const float s0 = __ldg(scales + 3 * i), s1 = __ldg(scales + 3 * i + 1), s2 = __ldg(scales + 3 * i + 2);
    const float4 q4 = __ldg(reinterpret_cast<const float4*>(quats) + i);
    if (RAW) {
        sc[0] = exp(R(s0)); sc[1] = exp(R(s1)); sc[2] = exp(R(s2));
        const R w = q4.x, x = q4.y, y = q4.z, z = q4.w;
        const R inv = R(1) / fmax(sqrt(xf(z, z, xf(y, y, xf(x, x, xm(w, w))))), R(1e-12));  // F.normalize eps
        q[0] = xm(w, inv); q[1] = xm(x, inv); q[2] = xm(y, inv); q[3] = xm(z, inv);
        *inv_qnorm = inv;
    } else {
        sc[0] = s0; sc[1] = s1; sc[2] = s2;
        q[0] = q4.x; q[1] = q4.y; q[2] = q4.z; q[3] = q4.w;
        *inv_qnorm = R(1);
    }
}

}  // namespace

}  // namespace b200gs
