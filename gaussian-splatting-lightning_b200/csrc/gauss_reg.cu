// K36-K38: the per-Gaussian regularisers of MCMCMetricsModuleMixin.reg_loss (internal/metrics/mcmc_metrics.py:39-59) and
// ScaleRegularizationMetricsModuleMixin.get_scale_regularization_metrics (internal/metrics/scale_regularization_metrics.py:51-115),
// on opacities o [N,1] and scales s [N,3] (raw: the logits and log-scales, activated here as sigmoid / exp):
//     o_reg           = w_o mean|o|
//     s_reg           = w_s mean|s|
//     scale_reg       = lambda   sum(s [s > max_scale]) / (n_s + 1)            n_s = #{s > max_scale}, elementwise
//     scale_ratio_reg = lambda_r sum(r [r > max_ratio]) / (n_r + 1)            r = max / (mid + 1e-8) of the sorted scales
// and the statistics [n_s, n_r, max of the largest scale, max r, mean r].
//   * K36 partials: grid-stride over the Gaussians; per CTA the sums of |o|, |s|, s [over], n_s, r [over], n_r, r and the maxima
//     of the largest scale and of r.  The grid depends only on N.
//   * K37 reduce (one CTA of 1024): in double, thread t sums partial rows t, t + 1024, ... in that order, each warp combines its
//     lanes by the xor butterfly of warp_reduce, and thread 0 adds the 32 warp results in warp order: a fixed order, so the result
//     is the same on every call.  It writes the terms, the statistics and the backward's coefficients (w_o / N, w_s / 3N,
//     lambda / (n_s + 1), lambda_r / (n_r + 1)) to the workspace head.
//   * K38 bwd: one thread per Gaussian; dense v_opacities and v_scales, exact zeros wherever no term applies.
// A term whose weight is 0 is off: no arithmetic, exact zeros in the gradient.  No float atomics: two calls are bit-identical.
// The library builds with --use_fast_math, so the activations call libdevice's expf and __fdiv_rn (expf and '/' would become
// __expf and an approximate division), and so does the ratio.  Signs and the zero test read the float's bits, which the
// flush-to-zero mode does not touch.
#include "common.cuh"

namespace b200gs {

namespace {

constexpr int THREADS = 256;
constexpr int PER_THREAD = 4;
constexpr int SPAN = THREADS * PER_THREAD;       // Gaussians per CTA before the grid saturates
constexpr int MAX_BLOCKS = 2048;                  // beyond MAX_BLOCKS * SPAN the CTAs stride over the rows
constexpr int RED_THREADS = 1024;
constexpr int NSUM = 7;                           // sum |o|, |s|, s [over], n_s, r [over], n_r, r
constexpr int PART = NSUM + 2;                    // + max of the largest scale, max r
constexpr int HEAD = 8;                           // backward coefficients
enum Sums { S_O, S_S, S_OVER, N_OVER, S_RATIO, N_RATIO, S_R };

struct RArgs {
    int64_t n;
    int raw, opacity, scale, over, ratio, sorted;   // sorted: the ratio or the statistics are needed
    float w_o, w_s, max_scale, max_ratio, lam, lam_r;
};

// libdevice's accurate expf, the function torch's fp32 exp and sigmoid kernels call (--use_fast_math maps expf to __expf)
extern "C" __device__ float __nv_expf(float);

__device__ __forceinline__ float exp_ref(float x) { return __nv_expf(x); }

// torch's fp32 sigmoid on the GPU, 1 / (1 + exp(-x)) with a correctly rounded division: exactly 0 once exp(-x) overflows,
// from x = -88.72283935546875 down
__device__ __forceinline__ float sigmoid_ref(float x) { return __fdiv_rn(1.f, __fadd_rn(1.f, __nv_expf(-x))); }

// sign(x) from the bits: torch.abs' subgradient, 0 at +-0; a subnormal keeps its sign (flush-to-zero would compare it as 0)
__device__ __forceinline__ float sign_bits(float x) {
    const unsigned b = __float_as_uint(x);
    return (b & 0x7fffffffu) == 0u ? 0.f : ((b >> 31) ? -1.f : 1.f);
}

__device__ __forceinline__ float abs_bits(float x) { return __uint_as_float(__float_as_uint(x) & 0x7fffffffu); }

struct Sorted {
    float v[3];
    int i[3];
};

// ascending sort of three values with their column indices, tied values routed as torch.sort routes them on the GPU.  For rows
// of <= 32 elements torch runs an unstable in-register bitonic network, whose routing of ties depends on the pattern of the row;
// it was measured on an H100 for every ordering of three values (13 with ties) and is tabulated here.  The table is indexed by
// the row's dense ranks r0 * 9 + r1 * 3 + r2 (r = the number of distinct smaller values) and holds the column of each sorted slot
// in 2-bit fields, 6 bits per entry, 10 entries per word.  (torch.sort on the CPU is stable, which routes some ties the other way.)
constexpr unsigned long long TIE_W0 = 0x240600918600846ull, TIE_W1 = 0x240000480006849ull, TIE_W2 = 0x180ull;

__device__ __forceinline__ int dense_rank(float x, float y, float z) {
    const bool ly = y < x, lz = z < x;
    return int(ly) + int(lz) - int(ly && lz && y == z);
}

__device__ __forceinline__ Sorted sort3(float a, float b, float c) {
    const int i = dense_rank(a, b, c) * 9 + dense_rank(b, a, c) * 3 + dense_rank(c, a, b);
    const unsigned long long w = i < 10 ? TIE_W0 : (i < 20 ? TIE_W1 : TIE_W2);
    const unsigned code = unsigned(w >> (6 * (i % 10))) & 63u;
    Sorted s;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const int col = (code >> (2 * k)) & 3;
        s.i[k] = col;
        s.v[k] = col == 0 ? a : (col == 1 ? b : c);
    }
    return s;
}

__device__ __forceinline__ void load(const RArgs& g, const float* __restrict__ opac, const float* __restrict__ scales, int64_t i,
                                     float& o, float (&s)[3]) {
    if (g.opacity) {
        o = __ldg(opac + i);
        if (g.raw) o = sigmoid_ref(o);
    }
    if (g.scale || g.over || g.sorted) {
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            s[k] = __ldg(scales + 3 * i + k);
            if (g.raw) s[k] = exp_ref(s[k]);
        }
    }
}

__global__ void __launch_bounds__(THREADS) reg_partials_kernel(RArgs g, const float* __restrict__ opac, const float* __restrict__ scales,
                                                               float* __restrict__ partials) {
    __shared__ float s_red[THREADS / 32][NSUM];
    __shared__ float s_max[THREADS / 32][2];
    float acc[NSUM] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    float mx_s = -INFINITY, mx_r = -INFINITY;
    for (int64_t i = int64_t(blockIdx.x) * THREADS + threadIdx.x; i < g.n; i += int64_t(gridDim.x) * THREADS) {
        float o = 0.f, s[3] = {0.f, 0.f, 0.f};
        load(g, opac, scales, i, o, s);
        if (g.opacity) acc[S_O] += abs_bits(o);
        if (g.scale) acc[S_S] += (abs_bits(s[0]) + abs_bits(s[1])) + abs_bits(s[2]);
        if (g.over) {
#pragma unroll
            for (int k = 0; k < 3; ++k)
                if (s[k] > g.max_scale) { acc[S_OVER] += s[k]; acc[N_OVER] += 1.f; }
        }
        if (g.sorted) {
            const Sorted q = sort3(s[0], s[1], s[2]);
            const float r = __fdiv_rn(q.v[2], __fadd_rn(q.v[1], 1e-8f));
            mx_s = fmaxf(mx_s, q.v[2]);
            mx_r = fmaxf(mx_r, r);
            acc[S_R] += r;
            if (g.ratio && r > g.max_ratio) { acc[S_RATIO] += r; acc[N_RATIO] += 1.f; }
        }
    }
    mx_s = warp_reduce<Max>(mx_s);
    mx_r = warp_reduce<Max>(mx_r);
    if ((threadIdx.x & 31) == 0) { s_max[threadIdx.x >> 5][0] = mx_s; s_max[threadIdx.x >> 5][1] = mx_r; }
    float* row = partials + int64_t(blockIdx.x) * PART;
    cta_sum_row(acc, s_red, threadIdx.x, [&] { return row; });        // synchronises the CTA, so s_max is complete
    if (threadIdx.x == NSUM) {
        for (int w = 1; w < THREADS / 32; ++w) { mx_s = fmaxf(mx_s, s_max[w][0]); mx_r = fmaxf(mx_r, s_max[w][1]); }
        row[NSUM] = mx_s;
        row[NSUM + 1] = mx_r;
    }
}

__global__ void __launch_bounds__(RED_THREADS) reg_reduce_kernel(RArgs g, int n_blocks, const float* __restrict__ partials,
                                                                 float* __restrict__ head, float* __restrict__ terms,
                                                                 float* __restrict__ stats) {
    __shared__ double s[RED_THREADS / 32][NSUM];
    __shared__ float s_m[RED_THREADS / 32][2];
    const int t = threadIdx.x, warp = t >> 5;
    double v[NSUM] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    float mx[2] = {-INFINITY, -INFINITY};
    for (int b = t; b < n_blocks; b += RED_THREADS) {
        const float* p = partials + int64_t(b) * PART;
#pragma unroll
        for (int k = 0; k < NSUM; ++k) v[k] += double(p[k]);
        mx[0] = fmaxf(mx[0], p[NSUM]);
        mx[1] = fmaxf(mx[1], p[NSUM + 1]);
    }
#pragma unroll
    for (int k = 0; k < NSUM; ++k) v[k] = warp_reduce<Sum>(v[k]);
    mx[0] = warp_reduce<Max>(mx[0]);
    mx[1] = warp_reduce<Max>(mx[1]);
    if ((t & 31) == 0) {
#pragma unroll
        for (int k = 0; k < NSUM; ++k) s[warp][k] = v[k];
        s_m[warp][0] = mx[0];
        s_m[warp][1] = mx[1];
    }
    __syncthreads();
    if (t != 0) return;
    for (int w = 1; w < RED_THREADS / 32; ++w) {
        for (int k = 0; k < NSUM; ++k) v[k] += s[w][k];
        mx[0] = fmaxf(mx[0], s_m[w][0]);
        mx[1] = fmaxf(mx[1], s_m[w][1]);
    }
    const double n = double(g.n);
    terms[0] = g.opacity ? float(double(g.w_o) * (v[S_O] / n)) : 0.f;
    terms[1] = g.scale ? float(double(g.w_s) * (v[S_S] / (3.0 * n))) : 0.f;
    terms[2] = g.over ? float(v[S_OVER] / (v[N_OVER] + 1.0) * double(g.lam)) : 0.f;
    terms[3] = g.ratio ? float(v[S_RATIO] / (v[N_RATIO] + 1.0) * double(g.lam_r)) : 0.f;
    head[0] = g.opacity ? float(double(g.w_o) / n) : 0.f;
    head[1] = g.scale ? float(double(g.w_s) / (3.0 * n)) : 0.f;
    head[2] = g.over ? float(double(g.lam) / (v[N_OVER] + 1.0)) : 0.f;
    head[3] = g.ratio ? float(double(g.lam_r) / (v[N_RATIO] + 1.0)) : 0.f;
    if (stats) {
        stats[0] = float(v[N_OVER]);
        stats[1] = float(v[N_RATIO]);
        stats[2] = mx[0];
        stats[3] = mx[1];
        stats[4] = float(v[S_R] / n);
    }
}

__global__ void __launch_bounds__(THREADS) reg_bwd_kernel(RArgs g, const float* __restrict__ opac, const float* __restrict__ scales,
                                                          const float* __restrict__ head, const float* __restrict__ v_terms,
                                                          float* __restrict__ v_opac, float* __restrict__ v_scales) {
    const int64_t i = int64_t(blockIdx.x) * THREADS + threadIdx.x;
    if (i >= g.n) return;
    float o = 0.f, s[3] = {0.f, 0.f, 0.f};
    load(g, opac, scales, i, o, s);
    if (v_opac) {
        float v = 0.f;
        if (g.opacity) {
            v = __ldg(v_terms) * __ldg(head) * sign_bits(o);
            if (g.raw) v = (v * (1.f - o)) * o;                          // torch's sigmoid backward, from the fp32 output
        }
        v_opac[i] = v;
    }
    if (!v_scales) return;
    float v[3] = {0.f, 0.f, 0.f};
    if (g.scale) {
        const float c = __ldg(v_terms + 1) * __ldg(head + 1);
#pragma unroll
        for (int k = 0; k < 3; ++k) v[k] = c * sign_bits(s[k]);
    }
    if (g.over) {
        const float c = __ldg(v_terms + 2) * __ldg(head + 2);
#pragma unroll
        for (int k = 0; k < 3; ++k)
            if (s[k] > g.max_scale) v[k] += c;
    }
    if (g.ratio) {
        const Sorted q = sort3(s[0], s[1], s[2]);
        const float d = __fadd_rn(q.v[1], 1e-8f);
        const float r = __fdiv_rn(q.v[2], d);
        if (r > g.max_ratio) {
            // torch's division backward: d r / d max = 1 / d, d r / d mid = -(max / d) / d
            const float c = __ldg(v_terms + 3) * __ldg(head + 3);
            const float gmax = __fdiv_rn(c, d), gmid = -c * __fdiv_rn(r, d);
#pragma unroll
            for (int k = 0; k < 3; ++k) {       // scatter back to the columns without dynamic register indexing
                if (q.i[2] == k) v[k] += gmax;
                if (q.i[1] == k) v[k] += gmid;
            }
        }
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) v_scales[3 * i + k] = g.raw ? v[k] * s[k] : v[k];   // torch's exp backward: grad * result
}

RArgs make_args(int64_t n, bool has_opac, bool has_scales, bool stats, int flags, float w_o, float w_s, float max_scale, float max_ratio,
                float lam, float lam_r) {
    RArgs g;
    g.n = n;
    g.raw = (flags & B200GS_GREG_RAW) != 0;
    // a term with weight 0 is off: it adds exact zeros, so it costs nothing
    g.opacity = has_opac && (flags & B200GS_GREG_OPACITY) && w_o != 0.f;
    g.scale = has_scales && (flags & B200GS_GREG_SCALE) && w_s != 0.f;
    g.over = has_scales && (flags & B200GS_GREG_OVER_SCALE) && lam != 0.f;
    g.ratio = has_scales && (flags & B200GS_GREG_OVER_RATIO) && lam_r != 0.f;
    g.sorted = g.ratio || (has_scales && stats);
    g.w_o = w_o; g.w_s = w_s; g.max_scale = max_scale; g.max_ratio = max_ratio; g.lam = lam; g.lam_r = lam_r;
    return g;
}

int reg_blocks(int64_t n) { return int(div_up64(n, SPAN) < MAX_BLOCKS ? div_up64(n, SPAN) : MAX_BLOCKS); }

bool gaussian_reg_size_ok(int64_t n) { return n >= 1 && n <= INT32_MAX; }

size_t gaussian_reg_workspace_bytes(int64_t n) { return size_t(HEAD + int64_t(reg_blocks(n)) * PART) * sizeof(float); }

// opacities [n,1] and scales [n,3] contiguous, either NULL when no term reads it; flags of b200gs.h.  The backward reads the
// coefficients its forward wrote to the workspace.  Shared by the forward and the backward; returns the error code, or 0 when the
// arguments are valid
int check_gaussian_reg(const char* fn, int64_t n, const float* opacities, const float* scales, int32_t flags, bool stats,
                       const void* workspace, size_t workspace_bytes) {
    constexpr int32_t all = B200GS_GREG_RAW | B200GS_GREG_OPACITY | B200GS_GREG_SCALE | B200GS_GREG_OVER_SCALE | B200GS_GREG_OVER_RATIO;
    if (n < 1) return fail(fn, "n must be >= 1");
    if (!gaussian_reg_size_ok(n)) return fail(fn, "n too large (> 2^31 - 1)");
    if (flags & ~all) return fail(fn, "unknown flags");
    if ((flags & B200GS_GREG_OPACITY) && !opacities) return fail(fn, "NULL pointer: opacities");
    if (((flags & (B200GS_GREG_SCALE | B200GS_GREG_OVER_SCALE | B200GS_GREG_OVER_RATIO)) || stats) && !scales)
        return fail(fn, "NULL pointer: scales");
    if (!workspace) return fail(fn, "NULL pointer: workspace");
    if (workspace_bytes < gaussian_reg_workspace_bytes(n)) return workspace_too_small(fn);
    return 0;
}

}  // namespace

}  // namespace b200gs

using namespace b200gs;

extern "C" {

size_t b200gs_gaussian_reg_workspace_bytes(int64_t n) { return gaussian_reg_size_ok(n) ? gaussian_reg_workspace_bytes(n) : 0; }

int b200gs_gaussian_reg_fwd(int64_t n, const float* opac, const float* scales, int32_t flags, float w_o, float w_s, float max_scale,
                            float max_ratio, float lam, float lam_r, void* workspace, size_t workspace_bytes, float* terms, float* stats,
                            void* stream) {
    if (int rc = check_gaussian_reg(__func__, n, opac, scales, flags, stats != nullptr, workspace, workspace_bytes)) return rc;
    B200GS_CHECK_ARG(terms, "NULL pointer: terms");
    const cudaStream_t st = (cudaStream_t)stream;
    float* ws = static_cast<float*>(workspace);
    const RArgs g = make_args(n, opac != nullptr, scales != nullptr, stats != nullptr, flags, w_o, w_s, max_scale, max_ratio, lam, lam_r);
    const int blocks = reg_blocks(n);
    reg_partials_kernel<<<blocks, THREADS, 0, st>>>(g, opac, scales, ws + HEAD);
    B200GS_LAUNCH_CHECK();
    reg_reduce_kernel<<<1, RED_THREADS, 0, st>>>(g, blocks, ws + HEAD, ws, terms, stats);
    B200GS_LAUNCH_CHECK();
    return B200GS_OK;
}

int b200gs_gaussian_reg_bwd(int64_t n, const float* opac, const float* scales, int32_t flags, float w_o, float w_s, float max_scale,
                            float max_ratio, float lam, float lam_r, const void* workspace, size_t workspace_bytes, const float* v_terms,
                            float* v_opac, float* v_scales, void* stream) {
    if (int rc = check_gaussian_reg(__func__, n, opac, scales, flags, false, workspace, workspace_bytes)) return rc;
    B200GS_CHECK_ARG(v_terms, "NULL pointer: v_terms");
    B200GS_CHECK_ARG(!opac || v_opac, "NULL pointer: v_opacities");
    B200GS_CHECK_ARG(!scales || v_scales, "NULL pointer: v_scales");
    // the backward needs the sort only for the ratio term
    const RArgs g = make_args(n, opac != nullptr, scales != nullptr, false, flags, w_o, w_s, max_scale, max_ratio, lam, lam_r);
    reg_bwd_kernel<<<int(div_up64(n, THREADS)), THREADS, 0, (cudaStream_t)stream>>>(g, opac, scales, static_cast<const float*>(workspace),
                                                                                    v_terms, opac ? v_opac : nullptr,
                                                                                    scales ? v_scales : nullptr);
    B200GS_LAUNCH_CHECK();
    return B200GS_OK;
}

}  // extern "C"
