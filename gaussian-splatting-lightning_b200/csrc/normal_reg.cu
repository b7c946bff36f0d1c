// K39-K42: the depth-normal consistency term of NormalRegModuleMixin.get_normal_reg_metrics (internal/metrics/normal_reg.py:27-38)
// and gsplat's utils.depth_to_normal, on a depth map d [H,W], an alpha map [H,W] and the rendered normal map [3,H,W]:
//     n_d[y,x] = alpha[y,x] normalize(cross(p[y+1,x] - p[y-1,x], p[y,x+1] - p[y,x-1])),   0 on the one-pixel border
//     p[y,x]   = o + d[y,x] R ((x - cx + 0.5) / fx, (y - cy + 0.5) / fy, 1)                 (R, o: the camera-to-world rotation, origin)
//     loss     = weight mean(1 - normal . n_d),     d loss / d normal = -weight / (H W) n_d
// normalize divides by max(|v|, 1e-12) as F.normalize does.  The origin cancels in the differences, so the kernels never form
// o + d R c: they take the camera-space differences d' c' - d c, rotate them and cross them.  In exact arithmetic that is the
// reference; in fp32 it keeps the bits the reference loses to cancellation when |o| is large against the depth.
//   * normal_from_depth computes n_d for one pixel; K39, K41 and K42 all call it, so the forward, the backward and the drop-in give
//     the same bits.  Its arithmetic is written with explicit round-to-nearest intrinsics, so the compiler has no contraction left to
//     choose, and the division and the square root are correctly rounded (the library builds with --use_fast_math).
//   * The rotation comes from a 4x4 matrix read on the device through its strides: K39 and K41 take the world-to-camera matrix and
//     invert its 3x3 block in double once per CTA (for an affine [R t; 0 1], the 3x3 block of the inverse is R^-1); K42 takes the
//     camera-to-world matrix and reads its block.  Nothing is copied to the host, and any caller's camera tensor works.
//   * K39 partials: one CTA per 16x16 tile with the depth tile and a one-pixel halo in shared memory; the tile's sum of
//     1 - normal . n_d goes through cta_sum_row.  normal is read through its strides (a channel slice of the permuted render).
//   * K40 reduce (one CTA of 1024): in double, thread t sums partials t, t + 1024, ... in order, an xor-butterfly warp reduction,
//     thread 0 adds the 32 warp sums in warp order.  It writes the loss and the backward's coefficient weight / (H W) to the workspace
//     head.  No float atomics: two calls are bit-identical.
//   * K41 bwd: one thread per pixel, n_d recomputed from the depth (four reads that the caches serve) rather than stored.
//   * K42 depth_to_normal: one thread per pixel, the [H,W,3] map.
#include "common.cuh"

namespace b200gs {

namespace {

constexpr int T = 16;                      // tile edge: one CTA per 16x16 pixels in every kernel here
constexpr int THREADS = T * T;
constexpr int HALO = T + 2;
constexpr int RED_THREADS = 1024;
constexpr int HEAD = 4;                    // workspace head: [backward coefficient, unused x 3], then one partial per tile

struct NCam {
    float r[9];                            // camera-to-world rotation, row-major
    float fx, fy, cx, cy;
};

struct Mat {
    const float* m;                        // 4x4 matrix (or its top-left 3x3) at m[i * s0 + j * s1]
    int64_t s0, s1;
    const float* k;                        // intrinsics 3x3 at k[i * k0 + j * k1]
    int64_t k0, k1;
};

// the camera of the CTA, computed by one thread: invert = 1 takes the inverse of the 3x3 block (in double, by the adjugate)
__device__ void load_camera(const Mat& a, int invert, NCam& c) {
    double m[9];
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) m[3 * i + j] = double(__ldg(a.m + i * a.s0 + j * a.s1));
    if (invert) {
        const double c00 = m[4] * m[8] - m[5] * m[7], c01 = m[5] * m[6] - m[3] * m[8], c02 = m[3] * m[7] - m[4] * m[6];
        const double inv_det = 1.0 / (m[0] * c00 + m[1] * c01 + m[2] * c02);
        const double r[9] = {c00, m[2] * m[7] - m[1] * m[8], m[1] * m[5] - m[2] * m[4],
                             c01, m[0] * m[8] - m[2] * m[6], m[2] * m[3] - m[0] * m[5],
                             c02, m[1] * m[6] - m[0] * m[7], m[0] * m[4] - m[1] * m[3]};
#pragma unroll
        for (int i = 0; i < 9; ++i) c.r[i] = float(r[i] * inv_det);
    } else {
#pragma unroll
        for (int i = 0; i < 9; ++i) c.r[i] = float(m[i]);
    }
    c.fx = __ldg(a.k);
    c.fy = __ldg(a.k + a.k0 + a.k1);
    c.cx = __ldg(a.k + 2 * a.k1);
    c.cy = __ldg(a.k + a.k0 + 2 * a.k1);
}

// (x - cx + 0.5) / f as torch evaluates it: (x - cx) + 0.5, correctly rounded division
__device__ __forceinline__ float ray(int x, float c, float f) { return __fdiv_rn(__fadd_rn(__fsub_rn(float(x), c), 0.5f), f); }

// R v, each row an explicit fma chain
__device__ __forceinline__ float3 rotate(const NCam& c, float3 v) {
    return make_float3(__fmaf_rn(c.r[2], v.z, __fmaf_rn(c.r[1], v.y, __fmul_rn(c.r[0], v.x))),
                       __fmaf_rn(c.r[5], v.z, __fmaf_rn(c.r[4], v.y, __fmul_rn(c.r[3], v.x))),
                       __fmaf_rn(c.r[8], v.z, __fmaf_rn(c.r[7], v.y, __fmul_rn(c.r[6], v.x))));
}

// n_d of pixel (x, y) from the depths above (dt), below (db), left (dl) and right (dr) of it and its alpha; 0 on the border
__device__ __forceinline__ float3 normal_from_depth(int x, int y, int height, int width, float dt, float db, float dl, float dr, float alpha,
                                                    const NCam& c) {
    if (x < 1 || y < 1 || x >= width - 1 || y >= height - 1) return make_float3(0.f, 0.f, 0.f);
    const float u = ray(x, c.cx, c.fx), ul = ray(x - 1, c.cx, c.fx), ur = ray(x + 1, c.cx, c.fx);
    const float v = ray(y, c.cy, c.fy), vt = ray(y - 1, c.cy, c.fy), vb = ray(y + 1, c.cy, c.fy);
    // camera-space p[y+1,x] - p[y-1,x] and p[y,x+1] - p[y,x-1]: the origin cancels
    const float3 a = make_float3(__fsub_rn(__fmul_rn(u, db), __fmul_rn(u, dt)), __fsub_rn(__fmul_rn(vb, db), __fmul_rn(vt, dt)),
                                 __fsub_rn(db, dt));
    const float3 b = make_float3(__fsub_rn(__fmul_rn(ur, dr), __fmul_rn(ul, dl)), __fsub_rn(__fmul_rn(v, dr), __fmul_rn(v, dl)),
                                 __fsub_rn(dr, dl));
    const float3 A = rotate(c, a), B = rotate(c, b);
    const float3 n = make_float3(__fmaf_rn(A.y, B.z, -__fmul_rn(A.z, B.y)), __fmaf_rn(A.z, B.x, -__fmul_rn(A.x, B.z)),
                                 __fmaf_rn(A.x, B.y, -__fmul_rn(A.y, B.x)));
    const float len = fmaxf(__fsqrt_rn(__fmaf_rn(n.z, n.z, __fmaf_rn(n.y, n.y, __fmul_rn(n.x, n.x)))), 1e-12f);
    return make_float3(__fmul_rn(__fdiv_rn(n.x, len), alpha), __fmul_rn(__fdiv_rn(n.y, len), alpha), __fmul_rn(__fdiv_rn(n.z, len), alpha));
}

__global__ void __launch_bounds__(THREADS) normal_reg_partials_kernel(int height, int width, const float* __restrict__ depth,
                                                                      const float* __restrict__ alpha, const float* __restrict__ normal,
                                                                      int64_t sc, int64_t sy, int64_t sx, Mat mat, float* __restrict__ partials) {
    __shared__ float s_d[HALO][HALO + 1];
    __shared__ NCam s_cam;
    __shared__ float s_red[THREADS / 32][1];
    const int tid = threadIdx.x, tx = tid % T, ty = tid / T;
    const int x0 = blockIdx.x * T, y0 = blockIdx.y * T;
    if (tid == 0) load_camera(mat, 1, s_cam);
    for (int i = tid; i < HALO * HALO; i += THREADS) {
        const int gy = y0 + i / HALO - 1, gx = x0 + i % HALO - 1;
        s_d[i / HALO][i % HALO] = (gx >= 0 && gy >= 0 && gx < width && gy < height) ? __ldg(depth + int64_t(gy) * width + gx) : 0.f;
    }
    __syncthreads();
    const int x = x0 + tx, y = y0 + ty;
    float v[1] = {0.f};
    if (x < width && y < height) {
        const float3 nd = normal_from_depth(x, y, height, width, s_d[ty][tx + 1], s_d[ty + 2][tx + 1], s_d[ty + 1][tx], s_d[ty + 1][tx + 2],
                                            __ldg(alpha + int64_t(y) * width + x), s_cam);
        const float* p = normal + int64_t(y) * sy + int64_t(x) * sx;
        const float dot = __fmaf_rn(__ldg(p + 2 * sc), nd.z, __fmaf_rn(__ldg(p + sc), nd.y, __fmul_rn(__ldg(p), nd.x)));
        v[0] = 1.f - dot;
    }
    cta_sum_row(v, s_red, tid, [&] { return partials + int64_t(blockIdx.y) * gridDim.x + blockIdx.x; });
}

__global__ void __launch_bounds__(RED_THREADS) normal_reg_reduce_kernel(int64_t n_tiles, double n_pixels, float weight,
                                                                        const float* __restrict__ partials, float* __restrict__ head,
                                                                        float* __restrict__ loss) {
    __shared__ double s[RED_THREADS / 32];
    const int t = threadIdx.x;
    double v = 0.0;
    for (int64_t b = t; b < n_tiles; b += RED_THREADS) v += double(partials[b]);
    v = warp_reduce<Sum>(v);
    if ((t & 31) == 0) s[t >> 5] = v;
    __syncthreads();
    if (t != 0) return;
    for (int w = 1; w < RED_THREADS / 32; ++w) v += s[w];
    loss[0] = float(double(weight) * (v / n_pixels));
    head[0] = float(double(weight) / n_pixels);
}

__device__ __forceinline__ float3 pixel_normal(int x, int y, int height, int width, const float* __restrict__ depth, float a, const NCam& c) {
    if (x < 1 || y < 1 || x >= width - 1 || y >= height - 1) return make_float3(0.f, 0.f, 0.f);
    const float* d = depth + int64_t(y) * width + x;
    return normal_from_depth(x, y, height, width, __ldg(d - width), __ldg(d + width), __ldg(d - 1), __ldg(d + 1), a, c);
}

__global__ void __launch_bounds__(THREADS) normal_reg_bwd_kernel(int height, int width, const float* __restrict__ depth,
                                                                 const float* __restrict__ alpha, Mat mat, const float* __restrict__ head,
                                                                 const float* __restrict__ v_loss, float* __restrict__ v_normal) {
    __shared__ NCam s_cam;
    if (threadIdx.x == 0) load_camera(mat, 1, s_cam);
    __syncthreads();
    const int x = blockIdx.x * T + threadIdx.x % T, y = blockIdx.y * T + threadIdx.x / T;
    if (x >= width || y >= height) return;
    const int64_t i = int64_t(y) * width + x, plane = int64_t(height) * width;
    const float3 nd = pixel_normal(x, y, height, width, depth, __ldg(alpha + i), s_cam);
    const float g = -__fmul_rn(__ldg(v_loss), __ldg(head));
    v_normal[i] = __fmul_rn(g, nd.x);
    v_normal[plane + i] = __fmul_rn(g, nd.y);
    v_normal[2 * plane + i] = __fmul_rn(g, nd.z);
}

__global__ void __launch_bounds__(THREADS) depth_to_normal_kernel(int height, int width, const float* __restrict__ depth, Mat mat,
                                                                  float* __restrict__ out) {
    __shared__ NCam s_cam;
    if (threadIdx.x == 0) load_camera(mat, 0, s_cam);
    __syncthreads();
    const int x = blockIdx.x * T + threadIdx.x % T, y = blockIdx.y * T + threadIdx.x / T;
    if (x >= width || y >= height) return;
    const float3 n = pixel_normal(x, y, height, width, depth, 1.f, s_cam);
    float* o = out + 3 * (int64_t(y) * width + x);
    o[0] = n.x;
    o[1] = n.y;
    o[2] = n.z;
}

dim3 tiles(int height, int width) { return dim3(unsigned(div_up(width, T)), unsigned(div_up(height, T))); }

Mat make_mat(const float* m, int64_t s0, int64_t s1, const float* k, int64_t k0, int64_t k1) { return Mat{m, s0, s1, k, k0, k1}; }

// the grid is tiles(height, width): its y dimension, ceil(H/T), is at most 65535
bool size_ok(int32_t height, int32_t width) {
    return height >= 1 && width >= 1 && height <= 65535 * T && int64_t(height) * width <= INT32_MAX;
}

size_t normal_reg_workspace_bytes(int height, int width) {
    const dim3 g = tiles(height, width);
    return size_t(HEAD + int64_t(g.x) * g.y) * sizeof(float);
}

// depth, alpha [H,W] contiguous; normal [3,H,W] read at normal[c sc + y sy + x sx]; v_normal [3,H,W] and the depth_to_normal output
// [H,W,3] contiguous; the 4x4 camera matrix (w2c for the loss, c2w for depth_to_normal) at m[i ms0 + j ms1] and K [3,3] at
// K[i ks0 + j ks1].  Shared by the three entry points; returns the error code, or 0 when the arguments are valid
int check_normal_maps(const char* fn, int32_t height, int32_t width, const float* depth, const float* cam, int64_t ms0, int64_t ms1,
                      const float* K, int64_t ks0, int64_t ks1) {
    if (height < 1 || width < 1) return fail(fn, "image size must be >= 1");
    if (!size_ok(height, width)) return fail(fn, "image too large");
    if (ms0 < 0 || ms1 < 0 || ks0 < 0 || ks1 < 0) return fail(fn, "negative matrix stride");
    if (!(depth && cam && K)) return fail(fn, "NULL pointer");
    return 0;
}

// the backward reads the coefficient its forward wrote to the workspace
int check_normal_reg_workspace(const char* fn, int32_t height, int32_t width, const float* alpha, const void* workspace,
                               size_t workspace_bytes) {
    if (!(alpha && workspace)) return fail(fn, "NULL pointer");
    if (workspace_bytes < normal_reg_workspace_bytes(height, width)) return workspace_too_small(fn);
    return 0;
}

}  // namespace

}  // namespace b200gs

using namespace b200gs;

extern "C" {

size_t b200gs_normal_reg_workspace_bytes(int32_t height, int32_t width) {
    return size_ok(height, width) ? normal_reg_workspace_bytes(height, width) : 0;
}

int b200gs_normal_reg_fwd(int32_t height, int32_t width, const float* normal, int64_t sc, int64_t sy, int64_t sx, const float* depth,
                          const float* alpha, const float* w2c, int64_t ms0, int64_t ms1, const float* K, int64_t ks0, int64_t ks1,
                          float weight, void* workspace, size_t workspace_bytes, float* loss, void* stream) {
    if (int rc = check_normal_maps(__func__, height, width, depth, w2c, ms0, ms1, K, ks0, ks1)) return rc;
    if (int rc = check_normal_reg_workspace(__func__, height, width, alpha, workspace, workspace_bytes)) return rc;
    B200GS_CHECK_ARG(normal && loss, "NULL pointer");
    B200GS_CHECK_ARG(sc >= 0 && sy >= 0 && sx >= 0, "negative normal stride");
    const cudaStream_t st = (cudaStream_t)stream;
    float* ws = static_cast<float*>(workspace);
    const dim3 g = tiles(height, width);
    const Mat mat = make_mat(w2c, ms0, ms1, K, ks0, ks1);
    normal_reg_partials_kernel<<<g, THREADS, 0, st>>>(height, width, depth, alpha, normal, sc, sy, sx, mat, ws + HEAD);
    B200GS_LAUNCH_CHECK();
    normal_reg_reduce_kernel<<<1, RED_THREADS, 0, st>>>(int64_t(g.x) * g.y, double(height) * double(width), weight, ws + HEAD, ws, loss);
    B200GS_LAUNCH_CHECK();
    return B200GS_OK;
}

int b200gs_normal_reg_bwd(int32_t height, int32_t width, const float* depth, const float* alpha, const float* w2c, int64_t ms0, int64_t ms1,
                          const float* K, int64_t ks0, int64_t ks1, const void* workspace, size_t workspace_bytes, const float* v_loss,
                          float* v_normal, void* stream) {
    if (int rc = check_normal_maps(__func__, height, width, depth, w2c, ms0, ms1, K, ks0, ks1)) return rc;
    if (int rc = check_normal_reg_workspace(__func__, height, width, alpha, workspace, workspace_bytes)) return rc;
    B200GS_CHECK_ARG(v_loss && v_normal, "NULL pointer");
    normal_reg_bwd_kernel<<<tiles(height, width), THREADS, 0, (cudaStream_t)stream>>>(
        height, width, depth, alpha, make_mat(w2c, ms0, ms1, K, ks0, ks1), static_cast<const float*>(workspace), v_loss, v_normal);
    B200GS_LAUNCH_CHECK();
    return B200GS_OK;
}

int b200gs_depth_to_normal(int32_t height, int32_t width, const float* depth, const float* c2w, int64_t ms0, int64_t ms1, const float* K,
                           int64_t ks0, int64_t ks1, float* normals, void* stream) {
    if (int rc = check_normal_maps(__func__, height, width, depth, c2w, ms0, ms1, K, ks0, ks1)) return rc;
    B200GS_CHECK_ARG(normals, "NULL pointer");
    depth_to_normal_kernel<<<tiles(height, width), THREADS, 0, (cudaStream_t)stream>>>(height, width, depth,
                                                                                       make_mat(c2w, ms0, ms1, K, ks0, ks1), normals);
    B200GS_LAUNCH_CHECK();
    return B200GS_OK;
}

}  // extern "C"
