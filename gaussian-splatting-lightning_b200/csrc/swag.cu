// SWAG in-the-wild appearance (internal/renderers/swag_renderer.py: SWAGRenderer.forward :32-66 with internal/models/swag_model.py):
// the per-Gaussian input rows of the appearance-conditioned network F_theta and their gradients, one thread per Gaussian.
//   x0[i] = [ rgb_i | enc_i | 0 .. ]   padded to row_stride floats (a multiple of 8: 40 for the defaults)
//     rgb_i = clamp_min(SH_deg(shs_i; dir_i) + 0.5, 0),  dir_i = (means_i - campos) / max(|means_i - campos|, 1e-12)   (eval_gaussian_
//             model_sh; the reference does not detach the means, so the backward returns their gradient through the direction)
//     enc_i = HashGrid((means_i - bbox_min) / bbox_size)   (the means detached; bbox_min | bbox_size: 6 floats on the device)
// The MLP itself, the colour sigmoid and the Gumbel-sigmoid opacity run on the appearance kernels K20/K21 (appearance.cu, epilogue 2).
//
// The hash grid restates tiny-cuda-nn's GridEncoding (HashGrid, linear interpolation) for 3-D inputs.  Per level l, on the host in
// fp32: scale_l = exp2f(l log2f(s)) base - 1, res_l = ceil(scale_l) + 1, size_l = min(next_multiple(res_l^3, 8), 2^log2_hashmap_size)
// vertices; the levels follow each other, a vertex is F contiguous floats (F = 4: one aligned 16-byte row).  A coordinate x maps to
// pos = fmaf(scale_l, x, 0.5f), cell = (uint32)(int)floor(pos), frac = pos - floor(pos) per axis; corner k = 0..7 has bit d on axis d
// and weight prod_d (bit d ? frac_d : 1 - frac_d), multiplied in axis order; enc[l F + f] = sum over k in order of fmaf(weight, v, .).
// The vertex of a corner is tcnn's grid_index in uint32 arithmetic: index = sum_d c_d stride_d with stride_0 = 1, stride_{d+1} =
// stride_d res_l while stride_d <= size_l; once the final stride exceeds size_l, index = c_0 ^ c_1 2654435761 ^ c_2 805459861 (the
// coherent prime hash); then index % size_l.  Coordinates outside [0, 1] are allowed (Gaussians leave the initial bounding box): a
// negative cell wraps through uint32 exactly as in tcnn.
//
//   * K49 swag_inputs_fwd_kernel: the SH colour (sh.cuh basis and loaders, the coefficients read in place: [N,K,3] or dc | rest),
//     the clamp bits, the normalised centre and 8 corners per level as 128-bit (F = 4) or 64-bit (F = 2) loads.  The rows are staged
//     per warp in shared memory and written as one coalesced span.  Without colour it encodes given points (hash_grid_encode).
//   * K50 swag_inputs_bwd_kernel: splits v_x0.  The colour columns go through the clamp bits (clamp_min passes the gradient where
//     x >= 0) to the SH coefficients and, through the view direction, to the means.  The encoding columns are scattered into the
//     table with sm_90's vector float atomics (red.global.add.v4.f32 / .v2.f32): one instruction per corner.  The order of those
//     additions is not fixed, so the table gradient is not bit-reproducible (as uv_grid_scatter_kernel's).
//
// HBM-bound.  Per Gaussian at degree 3 with the default grid (8 levels, F = 4, row_stride 40), algorithmic bytes:
//     forward  12 + 192 (means, coefficients) in, 160 + 1 (row, clamp bits) out, plus 64 corner rows of 16 B gathered (levels 0-2
//              are 1.2 MB and stay in L2; the hashed levels are 8 MB each);
//     backward 12 + 192 + 1 + 160 in, 192 + 12 out, plus 64 vector atomics of 16 B.
#include <algorithm>
#include <cmath>

#include "common.cuh"
#include "sh.cuh"

namespace b200gs {

namespace {

constexpr int HG_MAX_LEVELS = 16;
constexpr int SWAG_THREADS = 128;
constexpr int SWAG_MAX_ROW = 72;          // 3 colour columns + 16 levels x 4 features, rounded up to 8

struct HashLevels {
    int n, F;
    int64_t total;                                            // vertices of all levels
    float scale[HG_MAX_LEVELS];
    uint32_t res[HG_MAX_LEVELS], size[HG_MAX_LEVELS];
    int64_t offset[HG_MAX_LEVELS];                            // in vertices
};

bool hash_grid_ok(const B200gsHashGrid& g) {
    return g.n_levels >= 1 && g.n_levels <= HG_MAX_LEVELS && (g.n_features_per_level == 2 || g.n_features_per_level == 4) &&
           g.log2_hashmap_size >= 1 && g.log2_hashmap_size <= 24 && g.base_resolution >= 1 && g.per_level_scale >= 1.f &&
           std::isfinite(g.per_level_scale);
}

// The level table of a supported grid, or false when a scale is not finite or too large for the int cell conversion
// (scale_l >= 2^30).  Sizes in int64: res_l^3 overflows 32 bits long before the hash cap applies.
bool hash_levels(const B200gsHashGrid& g, HashLevels& L) {
    L = HashLevels{};
    if (!hash_grid_ok(g)) return false;
    L.n = g.n_levels;
    L.F = g.n_features_per_level;
    const float lg = std::log2(g.per_level_scale);
    const int64_t cap = int64_t(1) << g.log2_hashmap_size;
    int64_t total = 0;
    for (int l = 0; l < g.n_levels; ++l) {
        const float scale = std::exp2(float(l) * lg) * float(g.base_resolution) - 1.f;
        if (!std::isfinite(scale) || scale >= 1073741824.f) return false;
        const int64_t res = int64_t(std::ceil(scale)) + 1;
        const double dense = double(res) * double(res) * double(res);
        const int64_t size = dense >= double(cap) ? cap : std::min<int64_t>(cap, (res * res * res + 7) / 8 * 8);
        L.scale[l] = scale;
        L.res[l] = uint32_t(res);
        L.size[l] = uint32_t(size);
        L.offset[l] = total;
        total += size;
    }
    L.total = total;
    return true;
}

// tiny-cuda-nn's grid_index for a 3-D hash grid, in its uint32 arithmetic
__device__ __forceinline__ uint32_t grid_index(uint32_t cx, uint32_t cy, uint32_t cz, uint32_t res, uint32_t size) {
    uint32_t stride = 1, index = 0;
    const uint32_t c[3] = {cx, cy, cz};
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        if (stride > size) break;
        index += c[d] * stride;
        stride *= res;
    }
    if (size < stride) index = cx ^ (cy * 2654435761u) ^ (cz * 805459861u);
    return index % size;
}

struct Cell {
    uint32_t c[3];
    float f[3];
};

__device__ __forceinline__ Cell cell_of(float scale, float x, float y, float z) {
    Cell k;
    const float p[3] = {x, y, z};
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        const float pos = fmaf(scale, p[d], 0.5f);
        const float fl = floorf(pos);
        k.c[d] = uint32_t(int(fl));
        k.f[d] = pos - fl;
    }
    return k;
}

__device__ __forceinline__ float corner_weight(const Cell& k, int corner) {
    float w = 1.f;
#pragma unroll
    for (int d = 0; d < 3; ++d) w *= ((corner >> d) & 1) ? k.f[d] : 1.f - k.f[d];
    return w;
}

__device__ __forceinline__ uint32_t corner_vertex(const Cell& k, int corner, uint32_t res, uint32_t size) {
    return grid_index(k.c[0] + (corner & 1), k.c[1] + ((corner >> 1) & 1), k.c[2] + ((corner >> 2) & 1), res, size);
}

template <int F>
__device__ __forceinline__ void load_vertex(const float* __restrict__ p, float (&v)[4]) {
    if (F == 4) {
        const float4 t = __ldg(reinterpret_cast<const float4*>(p));
        v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
    } else {
        const float2 t = __ldg(reinterpret_cast<const float2*>(p));
        v[0] = t.x; v[1] = t.y; v[2] = v[3] = 0.f;
    }
}

template <int F>
__device__ __forceinline__ void add_vertex(float* p, const float (&g)[4]) {
    if (F == 4)
        atomicAdd(reinterpret_cast<float4*>(p), make_float4(g[0], g[1], g[2], g[3]));
    else
        atomicAdd(reinterpret_cast<float2*>(p), make_float2(g[0], g[1]));
}

struct SwagArgs {
    HashLevels L;
    int deg, sh_stride, row_stride;
    int64_t n;
    const float* means; const float* campos; const float* shs; const float* shs_rest; const float* bbox; const float* table;
    float* x0; uint8_t* clamped;                                               // forward
    const uint8_t* clamped_in; const float* v_x0; float* v_shs; float* v_shs_rest; float* v_means; float* v_table;   // backward
};

// The grid coordinate of Gaussian i: (means - bbox_min) / bbox_size as torch divides (IEEE, not the fast-math reciprocal), or the
// point itself without a box
__device__ __forceinline__ void grid_point(const SwagArgs& a, float px, float py, float pz, float& x, float& y, float& z) {
    if (a.bbox) {
        x = __fdiv_rn(px - __ldg(a.bbox), __ldg(a.bbox + 3));
        y = __fdiv_rn(py - __ldg(a.bbox + 1), __ldg(a.bbox + 4));
        z = __fdiv_rn(pz - __ldg(a.bbox + 2), __ldg(a.bbox + 5));
    } else {
        x = px; y = py; z = pz;
    }
}

template <bool COLOUR, bool SPLIT, int MC, int F>
__global__ void __launch_bounds__(SWAG_THREADS) swag_inputs_fwd_kernel(const SwagArgs a) {
    __shared__ float s_rows[SWAG_THREADS / 32][32 * (SWAG_MAX_ROW + 1)];
    const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    const unsigned lane = threadIdx.x & 31u;
    const int rw = a.row_stride;
    float* s_warp = s_rows[threadIdx.x >> 5];
    float* row = s_warp + lane * (rw | 1);
    if (i < a.n) {
        const float px = __ldg(a.means + 3 * i), py = __ldg(a.means + 3 * i + 1), pz = __ldg(a.means + 3 * i + 2);
        int c0 = 0;
        if (COLOUR) {
            float dx = px - __ldg(a.campos), dy = py - __ldg(a.campos + 1), dz = pz - __ldg(a.campos + 2);
            normalize_dir(dx, dy, dz);
            const int ncoef = (a.deg + 1) * (a.deg + 1);
            float bs[MC], sh[MC * 3];
            sh_basis<MC>(a.deg, dx, dy, dz, bs);
            load_sh_any<SPLIT, MC>(a.shs, a.shs_rest, i, a.sh_stride, ncoef, sh);
            float c[3] = {0.f, 0.f, 0.f};
#pragma unroll
            for (int k = 0; k < MC; ++k)
                if (k < ncoef) { c[0] += bs[k] * sh[3 * k]; c[1] += bs[k] * sh[3 * k + 1]; c[2] += bs[k] * sh[3 * k + 2]; }
            uint8_t cl = 0;
#pragma unroll
            for (int j = 0; j < 3; ++j) {
                const float v = c[j] + 0.5f;
                if (!(v >= 0.f)) cl |= uint8_t(1u << j);
                row[j] = v < 0.f ? 0.f : v;          // NaN stays NaN, as in torch.clamp_min
            }
            a.clamped[i] = cl;
            c0 = 3;
        }
        float x, y, z;
        grid_point(a, px, py, pz, x, y, z);
        for (int l = 0; l < a.L.n; ++l) {
            const Cell k = cell_of(a.L.scale[l], x, y, z);
            const float* lvl = a.table + a.L.offset[l] * F;
            float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
            for (int corner = 0; corner < 8; ++corner) {
                const float w = corner_weight(k, corner);
                float v[4];
                load_vertex<F>(lvl + int64_t(corner_vertex(k, corner, a.L.res[l], a.L.size[l])) * F, v);
#pragma unroll
                for (int f = 0; f < F; ++f) acc[f] = fmaf(w, v[f], acc[f]);
            }
#pragma unroll
            for (int f = 0; f < F; ++f) row[c0 + l * F + f] = acc[f];
        }
        for (int c = c0 + a.L.n * F; c < rw; ++c) row[c] = 0.f;
    }
    flush_sh_rows(s_warp, rw, i, a.n, lane, a.x0, false);
}

template <bool COLOUR, bool SPLIT, int MC, int F>
__global__ void __launch_bounds__(SWAG_THREADS) swag_inputs_bwd_kernel(const SwagArgs a) {
    const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= a.n) return;
    const float* g_row = a.v_x0 + i * int64_t(a.row_stride);
    const float px = __ldg(a.means + 3 * i), py = __ldg(a.means + 3 * i + 1), pz = __ldg(a.means + 3 * i + 2);
    int c0 = 0;
    if (COLOUR) {
        const uint8_t cl = __ldg(a.clamped_in + i);
        float g[3];
#pragma unroll
        for (int j = 0; j < 3; ++j) g[j] = ((cl >> j) & 1) ? 0.f : __ldg(g_row + j);
        float dx = px - __ldg(a.campos), dy = py - __ldg(a.campos + 1), dz = pz - __ldg(a.campos + 2);
        const float inv_len = normalize_dir(dx, dy, dz);
        const int ncoef = (a.deg + 1) * (a.deg + 1);
        float bs[MC], sh[MC * 3], w[MC];
        sh_basis<MC>(a.deg, dx, dy, dz, bs);
        load_sh_any<SPLIT, MC>(a.shs, a.shs_rest, i, a.sh_stride, ncoef, sh);
#pragma unroll
        for (int k = 0; k < MC; ++k) w[k] = k < ncoef ? sh[3 * k] * g[0] + sh[3 * k + 1] * g[1] + sh[3 * k + 2] * g[2] : 0.f;
        const float3 gm = view_dir_grad<MC>(a.deg, dx, dy, dz, inv_len, w);
        a.v_means[3 * i] = gm.x; a.v_means[3 * i + 1] = gm.y; a.v_means[3 * i + 2] = gm.z;
        // coefficient rows in the forward's layout, every column written (zeros at or beyond the degree)
        float* dst = SPLIT ? a.v_shs_rest + i * int64_t(a.sh_stride - 1) * 3 : a.v_shs + i * int64_t(a.sh_stride) * 3;
        if (SPLIT) { a.v_shs[3 * i] = bs[0] * g[0]; a.v_shs[3 * i + 1] = bs[0] * g[1]; a.v_shs[3 * i + 2] = bs[0] * g[2]; }
        const int k0 = SPLIT ? 1 : 0;
#pragma unroll
        for (int k = k0; k < MC; ++k) {
            if (k < a.sh_stride) {
                const float b = k < ncoef ? bs[k] : 0.f;
#pragma unroll
                for (int j = 0; j < 3; ++j) dst[(k - k0) * 3 + j] = b * g[j];
            }
        }
        for (int q = (MC - k0) * 3; q < (a.sh_stride - k0) * 3; ++q) dst[q] = 0.f;
        c0 = 3;
    }
    float x, y, z;
    grid_point(a, px, py, pz, x, y, z);
    for (int l = 0; l < a.L.n; ++l) {
        float ge[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int f = 0; f < F; ++f) ge[f] = __ldg(g_row + c0 + l * F + f);
        if (ge[0] == 0.f && ge[1] == 0.f && ge[2] == 0.f && ge[3] == 0.f) continue;     // adds nothing
        const Cell k = cell_of(a.L.scale[l], x, y, z);
        float* lvl = a.v_table + a.L.offset[l] * F;
#pragma unroll
        for (int corner = 0; corner < 8; ++corner) {
            const float w = corner_weight(k, corner);
            float gw[4];
#pragma unroll
            for (int f = 0; f < 4; ++f) gw[f] = w * ge[f];
            add_vertex<F>(lvl + int64_t(corner_vertex(k, corner, a.L.res[l], a.L.size[l])) * F, gw);
        }
    }
}

// The grid and the row layout, shared by both directions; colour: whether the colour columns are on (shs given)
int check_swag_inputs(const char* fn, const B200gsHashGrid* grid, HashLevels& L, int32_t degree, int64_t n, const float* means,
                      bool colour, const float* campos, const float* shs, const float* shs_rest, int32_t sh_stride, int32_t sh_split,
                      int32_t row_stride, const float* table_or_grad) {
    if (grid == nullptr) return fail(fn, "grid is NULL");
    if (!hash_levels(*grid, L))
        return fail(fn, "unsupported grid: n_levels 1..16, n_features_per_level 2 or 4, log2_hashmap_size 1..24, base_resolution >= 1, "
                        "per_level_scale >= 1 and every level's scale below 2^30");
    if (n < 0 || n > INT32_MAX) return fail(fn, "n out of range");
    const int c0 = colour ? 3 : 0;
    if (row_stride < c0 + L.n * L.F || row_stride > SWAG_MAX_ROW) return fail(fn, "row_stride must hold the row and be at most 72");
    if (colour) {
        if (degree < 0 || degree > 4) return fail(fn, "degree must be 0..4");
        if (sh_split != 0 && sh_split != 1) return fail(fn, "sh_split must be 0 or 1");
        if (sh_stride < (degree + 1) * (degree + 1)) return fail(fn, "sh_stride < (degree+1)^2");
    }
    if (n > 0) {
        if (!means || !table_or_grad) return fail(fn, "NULL pointer");
        if (colour && (!campos || !shs || (sh_split && sh_stride > 1 && !shs_rest))) return fail(fn, "NULL pointer");
        if ((reinterpret_cast<uintptr_t>(table_or_grad) & (L.F * 4 - 1)) != 0) return fail(fn, "the table must be aligned to one vertex");
    }
    return B200GS_OK;
}

int launch_swag(bool fwd, bool colour, bool split, int degree, const SwagArgs& a, cudaStream_t s) {
    using KP = void (*)(const SwagArgs);
    static const KP fwd_k[2][2][2][2] = {
        {{{swag_inputs_fwd_kernel<false, false, 16, 2>, swag_inputs_fwd_kernel<false, false, 16, 4>},
          {swag_inputs_fwd_kernel<false, false, 16, 2>, swag_inputs_fwd_kernel<false, false, 16, 4>}},
         {{swag_inputs_fwd_kernel<false, false, 16, 2>, swag_inputs_fwd_kernel<false, false, 16, 4>},
          {swag_inputs_fwd_kernel<false, false, 16, 2>, swag_inputs_fwd_kernel<false, false, 16, 4>}}},
        {{{swag_inputs_fwd_kernel<true, false, 16, 2>, swag_inputs_fwd_kernel<true, false, 16, 4>},
          {swag_inputs_fwd_kernel<true, false, 25, 2>, swag_inputs_fwd_kernel<true, false, 25, 4>}},
         {{swag_inputs_fwd_kernel<true, true, 16, 2>, swag_inputs_fwd_kernel<true, true, 16, 4>},
          {swag_inputs_fwd_kernel<true, true, 25, 2>, swag_inputs_fwd_kernel<true, true, 25, 4>}}}};
    static const KP bwd_k[2][2][2][2] = {
        {{{swag_inputs_bwd_kernel<false, false, 16, 2>, swag_inputs_bwd_kernel<false, false, 16, 4>},
          {swag_inputs_bwd_kernel<false, false, 16, 2>, swag_inputs_bwd_kernel<false, false, 16, 4>}},
         {{swag_inputs_bwd_kernel<false, false, 16, 2>, swag_inputs_bwd_kernel<false, false, 16, 4>},
          {swag_inputs_bwd_kernel<false, false, 16, 2>, swag_inputs_bwd_kernel<false, false, 16, 4>}}},
        {{{swag_inputs_bwd_kernel<true, false, 16, 2>, swag_inputs_bwd_kernel<true, false, 16, 4>},
          {swag_inputs_bwd_kernel<true, false, 25, 2>, swag_inputs_bwd_kernel<true, false, 25, 4>}},
         {{swag_inputs_bwd_kernel<true, true, 16, 2>, swag_inputs_bwd_kernel<true, true, 16, 4>},
          {swag_inputs_bwd_kernel<true, true, 25, 2>, swag_inputs_bwd_kernel<true, true, 25, 4>}}}};
    const KP k = (fwd ? fwd_k : bwd_k)[colour][colour && split][colour && degree > 3][a.L.F == 4];
    k<<<(unsigned)div_up64(a.n, SWAG_THREADS), SWAG_THREADS, 0, s>>>(a);
    B200GS_LAUNCH_CHECK();
    return B200GS_OK;
}

SwagArgs swag_args(const HashLevels& L, int32_t degree, int64_t n, const float* means, const float* campos, const float* shs,
                   const float* shs_rest, int32_t sh_stride, const float* bbox, int32_t row_stride) {
    SwagArgs a{};
    a.L = L;
    a.deg = degree; a.sh_stride = sh_stride; a.row_stride = row_stride; a.n = n;
    a.means = means; a.campos = campos; a.shs = shs; a.shs_rest = shs_rest; a.bbox = bbox;
    return a;
}

}  // namespace

}  // namespace b200gs

using namespace b200gs;

extern "C" {

int64_t b200gs_hash_grid_params(const B200gsHashGrid* grid) {
    HashLevels L;
    if (grid == nullptr || !hash_levels(*grid, L)) return 0;
    return L.total * L.F;
}

int b200gs_swag_inputs_fwd(const B200gsHashGrid* grid, int32_t degree, int64_t n, const float* means, const float* campos,
                           const float* shs, const float* shs_rest, int32_t sh_stride, int32_t sh_split, const float* bbox,
                           const float* table, int32_t row_stride, float* x0, uint8_t* clamped, void* stream) {
    HashLevels L;
    const bool colour = shs != nullptr;
    if (int rc = check_swag_inputs(__func__, grid, L, degree, n, means, colour, campos, shs, shs_rest, sh_stride, sh_split, row_stride, table))
        return rc;
    B200GS_CHECK_ARG(n == 0 || (x0 && (!colour || clamped)), "NULL pointer");
    if (n == 0) return B200GS_OK;
    SwagArgs a = swag_args(L, degree, n, means, campos, shs, shs_rest, sh_stride, bbox, row_stride);
    a.table = table; a.x0 = x0; a.clamped = clamped;
    return launch_swag(true, colour, sh_split != 0, degree, a, (cudaStream_t)stream);
}

int b200gs_swag_inputs_bwd(const B200gsHashGrid* grid, int32_t degree, int64_t n, const float* means, const float* campos,
                           const float* shs, const float* shs_rest, int32_t sh_stride, int32_t sh_split, const float* bbox,
                           const uint8_t* clamped, const float* v_x0, int32_t row_stride, float* v_shs, float* v_shs_rest,
                           float* v_means, float* v_table, void* stream) {
    HashLevels L;
    const bool colour = shs != nullptr;
    if (int rc = check_swag_inputs(__func__, grid, L, degree, n, means, colour, campos, shs, shs_rest, sh_stride, sh_split, row_stride,
                                   v_table))
        return rc;
    B200GS_CHECK_ARG(v_table, "NULL v_table");
    B200GS_CHECK_ARG(n == 0 || v_x0, "NULL v_x0");
    B200GS_CHECK_ARG(n == 0 || !colour || (clamped && v_shs && v_means && (!sh_split || sh_stride == 1 || v_shs_rest)), "NULL pointer");
    B200GS_CUDA(cudaMemsetAsync(v_table, 0, size_t(L.total) * L.F * sizeof(float), (cudaStream_t)stream));
    if (n == 0) return B200GS_OK;
    SwagArgs a = swag_args(L, degree, n, means, campos, shs, shs_rest, sh_stride, bbox, row_stride);
    a.clamped_in = clamped;
    a.v_x0 = v_x0; a.v_shs = v_shs; a.v_shs_rest = v_shs_rest; a.v_means = v_means; a.v_table = v_table;
    return launch_swag(false, colour, sh_split != 0, degree, a, (cudaStream_t)stream);
}

}  // extern "C"
