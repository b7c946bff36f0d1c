// The appearance-feature similarity regulariser of internal/metrics/appearance_feature_similarity_regularization_metrics.py
// (SimilarityRegularizationMixin.get_similarity_metric, :63-102) and its backward, without the [S,K,K,D] broadcast:
//     loss = lambda mean_{s, i<j} r_sij w_sj,   w_sj = exp(-decay d_sj),
//     Cosine r = -n_i . n_j with n = f / max(|f|, 1e-12) (F.normalize),   Euclidean r = |f_i - f_j|,
// f_i the feature row idx[s,i], w indexed by the column j as weighted_similarities_reg[:, triu_mask] indexes it.
// K43 stages one sample's K rows in shared memory per warp; lane j owns row j and sums r_ij w_j over i < j.  K44 adds the per-sample
// sums in double in a fixed order.  The backward K45 writes one gradient row per (sample, neighbour) entry and the record
// {idx, entry}; the records are sorted by idx with the library's onesweep passes (stable, so each Gaussian's entries stay in entry
// order), one pass marks where each Gaussian's run starts and ends, and K46 sums each run into the dense [N,D] gradient.  No float atomics: repeats are bit-identical.
// The library builds with --use_fast_math, so exp, sqrt and division are the correctly rounded / libdevice forms torch uses.
#include <float.h>

#include "common.cuh"

extern "C" __device__ float __nv_expf(float);

namespace b200gs {

namespace {

constexpr float NORMALIZE_EPS = 1e-12f;   // F.normalize's default eps
constexpr int MAX_WARPS = 8;
constexpr int SMEM_BUDGET = 48 * 1024;
constexpr int COEF_STRIDE = 33;           // the Euclidean backward's per-lane coefficient rows

// row stride of the staged features: odd, so the 32 lanes reading one column of 32 rows hit 32 banks
__host__ __device__ inline int row_stride(int d) { return d | 1; }

inline int warp_floats(int k, int d, bool bwd) { return k * row_stride(d) + (bwd ? 32 * COEF_STRIDE : 0); }
inline int warps_per_cta(int k, int d, bool bwd) { return max(1, min(MAX_WARPS, SMEM_BUDGET / (4 * warp_floats(k, d, bwd)))); }

__device__ __forceinline__ float pair_weight(float decay, float dist) { return __nv_expf(__fmul_rn(-decay, dist)); }

// idx[e] clamped to [0, n): the contract asks for indices in range (knn_points only writes such), and a stray one then reads a
// real row instead of memory outside the features
__device__ __forceinline__ int64_t row_of(const int64_t* __restrict__ idx, int64_t e, int64_t n) { return min(max(idx[e], (int64_t)0), n - 1); }

// the sample's K rows -> f[i * DP + c]; Cosine: normalised in place, lane i < k returns its row's clamped norm
__device__ __forceinline__ float stage_rows(float* f, int64_t n, const float* __restrict__ features, const int64_t* __restrict__ idx, int64_t smp,
                                            int k, int d, bool cosine, unsigned lane) {
    const int dp = row_stride(d);
    for (int e = lane; e < k * d; e += 32) {
        const int i = e / d, c = e - i * d;
        f[i * dp + c] = features[row_of(idx, smp * k + i, n) * d + c];
    }
    __syncwarp();
    float den = 1.f;
    if (cosine && (int)lane < k) {
        float ss = 0.f;
        for (int c = 0; c < d; ++c) ss = __fmaf_rn(f[lane * dp + c], f[lane * dp + c], ss);
        den = fmaxf(__fsqrt_rn(ss), NORMALIZE_EPS);
        for (int c = 0; c < d; ++c) f[lane * dp + c] = __fdiv_rn(f[lane * dp + c], den);
    }
    __syncwarp();
    return den;
}

__device__ __forceinline__ float row_dist(const float* a, const float* b, int d) {
    float ss = 0.f;
    for (int c = 0; c < d; ++c) {
        const float t = __fsub_rn(a[c], b[c]);
        ss = __fmaf_rn(t, t, ss);
    }
    return __fsqrt_rn(ss);
}

// K43: partial[s] = sum_{i<j} r_ij w_j of sample s; weights[s,j] = w_j when weights is not NULL
__global__ void __launch_bounds__(MAX_WARPS * 32) similarity_fwd_kernel(int64_t n, int d, const float* __restrict__ features, int64_t s, int k,
                                                                       const int64_t* __restrict__ idx, const float* __restrict__ dists,
                                                                       int cosine, float decay, float* __restrict__ partial,
                                                                       float* __restrict__ weights) {
    extern __shared__ float smem[];
    const unsigned lane = threadIdx.x & 31u, w = threadIdx.x >> 5;
    const int64_t smp = int64_t(blockIdx.x) * (blockDim.x >> 5) + w;
    if (smp >= s) return;                          // whole warps only: nothing below synchronises the CTA
    const int dp = row_stride(d);
    float* f = smem + (size_t)w * k * dp;
    stage_rows(f, n, features, idx, smp, k, d, cosine != 0, lane);
    float part = 0.f;
    if ((int)lane < k) {
        const float wj = pair_weight(decay, dists[smp * k + lane]);
        if (weights) weights[smp * k + lane] = wj;
        const float* fj = f + lane * dp;
        float acc = 0.f;
        for (int i = 0; i < (int)lane; ++i) {
            const float* fi = f + i * dp;
            if (cosine) {
                float dot = 0.f;
                for (int c = 0; c < d; ++c) dot = __fmaf_rn(fi[c], fj[c], dot);
                acc = __fsub_rn(acc, dot);
            } else {
                acc = __fadd_rn(acc, row_dist(fi, fj, d));
            }
        }
        part = __fmul_rn(acc, wj);
    }
    part = warp_sum(part);
    if (lane == 0) partial[smp] = part;
}

// K44: one CTA adds the S partials in double in a fixed order (thread t sums t, t + 1024, ...; then the warp butterfly and the
// 32 warp sums in warp order): out[1] = the mean over S K (K - 1) / 2 pairs, out[0] = lambda out[1] in float, as the reference
constexpr int REDUCE_THREADS = 1024;

__global__ void __launch_bounds__(REDUCE_THREADS) similarity_reduce_kernel(int64_t s, int k, const float* __restrict__ partial, float lambda,
                                                                           float* __restrict__ out) {
    __shared__ double s_w[REDUCE_THREADS / 32];
    double t = 0.0;
    for (int64_t i = threadIdx.x; i < s; i += REDUCE_THREADS) t += (double)partial[i];
    t = warp_reduce<Sum>(t);
    if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = t;
    __syncthreads();
    if (threadIdx.x == 0) {
        double tot = 0.0;
        for (int i = 0; i < REDUCE_THREADS / 32; ++i) tot += s_w[i];
        const float mean = (float)(tot / ((double)s * (double)(k * (k - 1) / 2)));
        out[1] = mean;
        out[0] = __fmul_rn(mean, lambda);
    }
}

// K45: gent[e, :] = d loss / d f of entry e = s K + i, and rec[e] = {idx[e], e}
__global__ void __launch_bounds__(MAX_WARPS * 32) similarity_bwd_entry_kernel(int64_t n, int d, const float* __restrict__ features, int64_t s, int k,
                                                                             const int64_t* __restrict__ idx, const float* __restrict__ dists,
                                                                             int cosine, float decay, float lambda,
                                                                             const float* __restrict__ v_loss, float* __restrict__ gent,
                                                                             uint2* __restrict__ rec) {
    extern __shared__ float smem[];
    const unsigned lane = threadIdx.x & 31u, w = threadIdx.x >> 5;
    const int64_t smp = int64_t(blockIdx.x) * (blockDim.x >> 5) + w;
    if (smp >= s) return;
    const int dp = row_stride(d);
    float* f = smem + (size_t)w * (k * dp + 32 * COEF_STRIDE);
    float* coef = f + k * dp + lane * COEF_STRIDE;
    const float den = stage_rows(f, n, features, idx, smp, k, d, cosine != 0, lane);
    if ((int)lane >= k) return;
    // d loss / d (r_ij w_j) of every pair: (v lambda) / (S K (K - 1) / 2), as autograd forms it through "* lambda" and the mean
    const float cpair = __fdiv_rn(__fmul_rn(v_loss[0], lambda), (float)((double)s * (double)(k * (k - 1) / 2)));
    const int i = (int)lane;
    const int64_t e = smp * k + i;
    const float wi = pair_weight(decay, dists[e]);
    const float* fi = f + i * dp;
    float* g = gent + e * d;
    rec[e] = make_uint2((uint32_t)row_of(idx, e, n), (uint32_t)e);
    if (cosine) {
        // d loss / d n_i = -c (sum_{j>i} w_j n_j + w_i sum_{a<i} n_a); then F.normalize's backward: (g - n (g . n)) / |f| where
        // |f| >= eps, g / eps below it (clamp_min passes no gradient to the norm there)
        for (int j = 0; j < k; ++j) coef[j] = j > i ? pair_weight(decay, dists[smp * k + j]) : (j < i ? wi : 0.f);
        float gn_dot_n = 0.f;
        for (int c = 0; c < d; ++c) {
            float acc = 0.f;
            for (int j = 0; j < k; ++j) acc = __fmaf_rn(coef[j], f[j * dp + c], acc);
            const float gn = -__fmul_rn(cpair, acc);
            g[c] = gn;
            gn_dot_n = __fmaf_rn(gn, fi[c], gn_dot_n);
        }
        const bool clamped = !(den > NORMALIZE_EPS);
        for (int c = 0; c < d; ++c) g[c] = clamped ? __fdiv_rn(g[c], NORMALIZE_EPS) : __fdiv_rn(__fsub_rn(g[c], __fmul_rn(fi[c], gn_dot_n)), den);
    } else {
        // d r_ij / d f_i = (f_i - f_j) / r_ij, 0 where r_ij = 0 (torch's norm backward); the pair's weight is w_max(i,j)
        for (int j = 0; j < k; ++j) {
            float cj = 0.f;
            if (j != i) {
                const float r = row_dist(fi, f + j * dp, d);
                const float wj = j > i ? pair_weight(decay, dists[smp * k + j]) : wi;
                cj = r > 0.f ? __fdiv_rn(__fmul_rn(cpair, wj), r) : 0.f;
            }
            coef[j] = cj;
        }
        for (int c = 0; c < d; ++c) {
            float acc = 0.f;
            for (int j = 0; j < k; ++j) acc = __fmaf_rn(coef[j], __fsub_rn(fi[c], f[j * dp + c]), acc);
            g[c] = acc;
        }
    }
}

// the first and one-past-last position of every Gaussian's run of sorted records (run_lo = run_hi = 0, from the memset, for a
// Gaussian no sample reached)
__global__ void __launch_bounds__(256) similarity_runs_kernel(int64_t e_count, const uint2* __restrict__ rec, int* __restrict__ run_lo,
                                                              int* __restrict__ run_hi) {
    const int64_t e = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (e >= e_count) return;
    const uint32_t key = rec[e].x;
    if (e == 0 || rec[e - 1].x != key) run_lo[key] = (int)e;
    if (e == e_count - 1 || rec[e + 1].x != key) run_hi[key] = (int)e + 1;
}

// K46: v_features[g, :] = the sum of Gaussian g's entry rows in entry order (0 where no sample reached it); one thread per float4
// (or per float when D % 4 != 0) of the dense gradient, so the writes of all N rows are coalesced
template <int V>
__global__ void __launch_bounds__(256) similarity_bwd_gather_kernel(int64_t n, int d, const int* __restrict__ run_lo, const int* __restrict__ run_hi,
                                                                    const uint2* __restrict__ rec, const float* __restrict__ gent,
                                                                    float* __restrict__ v_features) {
    const int dv = d / V;
    const int64_t t = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (t >= n * dv) return;
    const int64_t g = t / dv;
    const int c = (int)(t - g * dv) * V;
    float acc[V];
#pragma unroll
    for (int v = 0; v < V; ++v) acc[v] = 0.f;
    for (int e = run_lo[g], end = run_hi[g]; e < end; ++e) {
        const float* row = gent + (int64_t)rec[e].y * d + c;
#pragma unroll
        for (int v = 0; v < V; ++v) acc[v] = __fadd_rn(acc[v], row[v]);
    }
    if (V == 4) {
        *reinterpret_cast<float4*>(v_features + g * d + c) = make_float4(acc[0], acc[V > 1 ? 1 : 0], acc[V > 2 ? 2 : 0], acc[V > 3 ? 3 : 0]);
    } else {
#pragma unroll
        for (int v = 0; v < V; ++v) v_features[g * d + c + v] = acc[v];
    }
}

// forward: the S partials.  backward: the entry rows, the records, the sort scratch and the run table (the last two zeroed there).
struct SimLayout {
    size_t gent, rec_a, rec_b, zero, sort_scratch, run_lo, run_hi, zero_bytes, total;
};

size_t sim_fwd_bytes(int64_t s) { return align_up((size_t)s * 4, 256); }

SimLayout sim_bwd_layout(int64_t n, int64_t s, int k, int d) {
    SimLayout L{};
    size_t off = 0;
    auto take = [&off](size_t bytes) { size_t o = off; off = align_up(off + bytes, 256); return o; };
    const int64_t e = s * k;
    L.gent = take((size_t)e * d * 4);
    L.rec_a = take((size_t)e * 8);
    L.rec_b = take((size_t)e * 8);
    L.zero = off;
    L.sort_scratch = take(record_sort_scratch_bytes(e));
    L.run_lo = take((size_t)n * 4);
    L.run_hi = take((size_t)n * 4);
    L.zero_bytes = off - L.zero;
    L.total = off;
    return L;
}

// features [N,D] contiguous, idx [S,K] int64, dists [S,K]; kind 0 Cosine, 1 Euclidean
size_t similarity_reg_workspace_bytes(int64_t n, int64_t s, int k, int d, bool backward) {
    return backward ? sim_bwd_layout(n, s, k, d).total : sim_fwd_bytes(s);
}

// shared by the similarity entry points; returns the error code, or 0 when the arguments are valid
int check_similarity(const char* fn, int64_t n, int32_t d, const float* features, int64_t s, int32_t k, const int64_t* idx, const float* dists,
                     int32_t kind, const void* workspace, size_t workspace_bytes, bool backward) {
    if (kind != 0 && kind != 1) return fail(fn, "kind must be 0 (Cosine) or 1 (Euclidean)");
    if (d < 1 || d > 256) return fail(fn, "feature dimension must be 1..256");
    if (k < 2 || k > 32) return fail(fn, "K must be 2..32");
    if (s < 1 || n < 1) return fail(fn, "S and N must be >= 1");
    if (n >= (int64_t(1) << 30) || s * k >= (int64_t(1) << 30)) return fail(fn, "N and S K must be < 2^30");
    if (!(features && idx && dists && workspace)) return fail(fn, "NULL pointer");
    if (workspace_bytes < similarity_reg_workspace_bytes(n, s, k, d, backward)) return workspace_too_small(fn);
    return 0;
}

}  // namespace

}  // namespace b200gs

using namespace b200gs;

extern "C" {

size_t b200gs_similarity_reg_workspace_bytes(int64_t n, int64_t s, int32_t k, int32_t d, int32_t backward) {
    const bool ok = n >= 1 && n < (int64_t(1) << 30) && s >= 1 && k >= 2 && k <= 32 && s * k < (int64_t(1) << 30) && d >= 1 && d <= 256;
    return ok ? similarity_reg_workspace_bytes(n, s, k, d, backward != 0) : 0;
}

int b200gs_similarity_reg_fwd(int64_t n, int32_t d, const float* features, int64_t s, int32_t k, const int64_t* idx, const float* dists,
                              int32_t kind, float decay, float lambda, void* workspace, size_t workspace_bytes, float* out, float* weights,
                              void* stream) {
    if (int rc = check_similarity(__func__, n, d, features, s, k, idx, dists, kind, workspace, workspace_bytes, false)) return rc;
    B200GS_CHECK_ARG(out, "NULL pointer");
    const cudaStream_t st = (cudaStream_t)stream;
    float* ws = static_cast<float*>(workspace);
    const int wpc = warps_per_cta(k, d, false);
    similarity_fwd_kernel<<<(unsigned)div_up64(s, wpc), wpc * 32, (size_t)wpc * warp_floats(k, d, false) * 4, st>>>(
        n, d, features, s, k, idx, dists, kind == 0, decay, ws, weights);
    B200GS_LAUNCH_CHECK();
    similarity_reduce_kernel<<<1, REDUCE_THREADS, 0, st>>>(s, k, ws, lambda, out);
    B200GS_LAUNCH_CHECK();
    return B200GS_OK;
}

int b200gs_similarity_reg_bwd(int64_t n, int32_t d, const float* features, int64_t s, int32_t k, const int64_t* idx, const float* dists,
                              int32_t kind, float decay, float lambda, void* workspace, size_t workspace_bytes, const float* v_loss,
                              float* v_features, void* stream) {
    if (int rc = check_similarity(__func__, n, d, features, s, k, idx, dists, kind, workspace, workspace_bytes, true)) return rc;
    B200GS_CHECK_ARG(v_loss && v_features, "NULL pointer");
    const cudaStream_t st = (cudaStream_t)stream;
    const SimLayout L = sim_bwd_layout(n, s, k, d);
    char* w = (char*)workspace;
    const int64_t e = s * k;
    B200GS_CUDA(cudaMemsetAsync(w + L.zero, 0, L.zero_bytes, st));
    const int wpc = warps_per_cta(k, d, true);
    similarity_bwd_entry_kernel<<<(unsigned)div_up64(s, wpc), wpc * 32, (size_t)wpc * warp_floats(k, d, true) * 4, st>>>(
        n, d, features, s, k, idx, dists, kind == 0, decay, lambda, v_loss, (float*)(w + L.gent), (uint2*)(w + L.rec_a));
    B200GS_LAUNCH_CHECK();
    const uint2* sorted = nullptr;
    if (int rc = launch_record_sort(e, record_key_bits(n - 1), (uint2*)(w + L.rec_a), (uint2*)(w + L.rec_b), w + L.sort_scratch, st, &sorted))
        return rc;
    int* run_lo = (int*)(w + L.run_lo);
    int* run_hi = (int*)(w + L.run_hi);
    similarity_runs_kernel<<<(unsigned)div_up64(e, 256), 256, 0, st>>>(e, sorted, run_lo, run_hi);
    B200GS_LAUNCH_CHECK();
    const float* gent = (const float*)(w + L.gent);
    if (d % 4 == 0 && (reinterpret_cast<uintptr_t>(v_features) & 15) == 0)
        similarity_bwd_gather_kernel<4><<<(unsigned)div_up64(n * (d / 4), 256), 256, 0, st>>>(n, d, run_lo, run_hi, sorted, gent, v_features);
    else
        similarity_bwd_gather_kernel<1><<<(unsigned)div_up64(n * d, 256), 256, 0, st>>>(n, d, run_lo, run_hi, sorted, gent, v_features);
    B200GS_LAUNCH_CHECK();
    return B200GS_OK;
}

}  // extern "C"
