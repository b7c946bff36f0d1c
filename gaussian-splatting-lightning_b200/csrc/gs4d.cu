// 4DGS deformation (internal/model_components/gs4d_hexplane.py HexPlaneField + gs4d_deformation.py Deformation.forward_dynamic, as
// internal/renderers/vanilla_gs4d_renderer.py runs it every frame): per Gaussian a HexPlane lookup of (normalised mean, t), the
// trunk MLP and the enabled heads, added to the raw parameters.
//     p   = (means - aabb[0]) * (2 / (aabb[1] - aabb[0])) - 1          aabb[0] = xyz_max, aabb[1] = xyz_min; not clamped
//     f_l = prod over the planes (a,b) in (0,1),(0,2),(0,3),(1,2),(1,3),(2,3) of bilinear(plane_l^(a,b); (p,t)_a, (p,t)_b)
//           (grid_sample, align_corners=True, padding_mode='border'; the product starts from 1 and runs in plane order)
//     h   = Linear_{D'-1} relu .. relu Linear_0 [f_0 | .. | f_{L-1}]     D' = max(defor_depth, 1)
//     dx, ds, dr, dshs = Linear_2 relu Linear_1 relu h                  (each head enabled by its flag)
//     means' = means + dx,  log_scales' = log_scales + ds,  quats' = quats + dr or normalize(quats * dr),  shs' = shs + dshs
// The opacity head, timenet and the sin / cos encodings of the reference are never read there and are not computed.
//   * K52 gs4d_repack_kernel: once per model, each plane [C, res_b, res_a] (channel-first, as torch stores it) into the channel-last
//     [res_b, res_a, C], the planes level-major then in plane order, so one bilinear corner is one contiguous C-float row.
//   * K51 gs4d_deform_kernel: persistent CTAs of 8 warps walk tiles of 128 consecutive Gaussians.  Per tile:
//       gather: each warp builds its 16 rows of [f_0 | .. ] in shared memory, one channel per lane (C = 16: two rows per pass), so
//         each of a row's 24 L corner reads is one coalesced 64- or 128-byte load;
//       MLP: one layer at a time.  The CTA stages the layer's weights in shared memory (fp32, rows padded to stride K + 4 so the
//         fragment loads do not conflict), then every warp runs it on its 16 rows with the 3xTF32 warp GEMM of warp_mma.cuh.  At
//         net_width 128 one hidden layer is 64 KB, so the network does not fit at once; staging per layer keeps one CTA of 8 warps
//         per SM at either width, and the weights (at most 410 KB per tile of 128 Gaussians) come from L2;
//       epilogue: after each head's output layer, the warp adds the head to its rows' raw parameters and writes them.
//     Disabled heads copy their parameter through (dshs off: the SH outputs are not written at all).
#include <algorithm>
#include <cmath>

#include "common.cuh"
#include "warp_mma.cuh"

namespace b200gs {

namespace {

constexpr int GS4D_WARPS = 8;
constexpr int GS4D_ROWS = 16 * GS4D_WARPS;    // one tile
constexpr int GS4D_MAX_CTAS = 132;            // one persistent CTA per SM of an H100 SXM
constexpr int GS4D_SMEM_LIMIT = 227 * 1024;
constexpr int GS4D_MAX_LEVELS = 4;
constexpr int GS4D_PLANES = 6;
constexpr int GS4D_LAYERS = 10;               // trunk 0, trunk 1, then (hidden, output) of dx, ds, dr, dshs

constexpr int GS4D_THREADS = 32 * GS4D_WARPS;

// plane k = (a, b) of itertools.combinations(range(4), 2): (0,1), (0,2), (0,3), (1,2), (1,3), (2,3); a indexes the width
__host__ __device__ constexpr int plane_a(int k) { return k < 3 ? 0 : (k < 5 ? 1 : 2); }
__host__ __device__ constexpr int plane_b(int k) { return k < 3 ? k + 1 : (k == 3 ? 2 : 3); }
// outputs of head h: dx, ds, dr, dshs
__host__ __device__ constexpr int head_out(int h) { return h == 3 ? 48 : (h == 2 ? 4 : 3); }

struct Gs4dShape {
    int L, C, W, D, flags;
    int res[GS4D_MAX_LEVELS][4];          // per level: x, y, z, t
    __host__ __device__ int k0() const { return C * L; }
    __host__ __device__ int sa() const { return (k0() > W ? k0() : W) + 4; }
    __host__ __device__ int sb() const { return W + 4; }
    __host__ __device__ int trunk() const { return D < 1 ? 1 : D; }
};

struct Gs4dLayout {                       // offsets in floats into dynamic shared memory
    int A, B, Wt, bias, total;
};

__host__ __device__ inline Gs4dLayout gs4d_layout(const Gs4dShape& s) {
    Gs4dLayout a{};
    int o = 0;
    a.A = o; o += GS4D_ROWS * s.sa();
    a.B = o; o += GS4D_ROWS * s.sb();
    a.Wt = o; o += s.W * s.sa();          // the widest layer: W rows of max(K0, W) inputs
    a.bias = o; o += s.W;
    a.total = o;
    return a;
}

struct Gs4dParams {
    Gs4dShape s;
    int64_t n;
    int64_t off[GS4D_MAX_LEVELS][GS4D_PLANES];      // plane offsets (floats) into the repacked planes
    const float* planes; const float* aabb; const float* time;
    const float* means; const float* scales; const float* quats; const float* dc; const float* rest;
    const float* W[GS4D_LAYERS]; const float* b[GS4D_LAYERS];
    float* means_out; float* scales_out; float* quats_out; float* dc_out; float* rest_out;
};

// this warp's 16 rows of [f_0 | .. | f_{L-1}] (zeros past n), row stride sa
__device__ void gather(const Gs4dParams& p, float* X, int sa, int64_t row0, int lane) {
    const Gs4dShape& s = p.s;
    const int C = s.C, per = 32 / C, sub = lane / C, c = lane - sub * C;
    const float t = __ldg(p.time);
    float lo[3], scale[3];
#pragma unroll
    for (int d = 0; d < 3; ++d) {         // IEEE operations, as torch: no contraction, no approximate division
        lo[d] = __ldg(p.aabb + d);
        scale[d] = __fdiv_rn(2.f, __fsub_rn(__ldg(p.aabb + 3 + d), lo[d]));
    }
    for (int i = sub; i < 16; i += per) {
        const int64_t row = row0 + i;
        float* x = X + i * sa;
        if (row >= p.n) {
            for (int k = c; k < s.k0(); k += C) x[k] = 0.f;
            continue;
        }
        float q[4];
#pragma unroll
        for (int d = 0; d < 3; ++d) q[d] = __fsub_rn(__fmul_rn(__fsub_rn(__ldg(p.means + row * 3 + d), lo[d]), scale[d]), 1.f);
        q[3] = t;
        for (int l = 0; l < s.L; ++l) {
            int i0[4], i1[4];
            float f[4];
#pragma unroll
            for (int d = 0; d < 4; ++d) {        // grid_sample's source index (align_corners), clipped to the border
                const int r = s.res[l][d];
                float ix = __fmul_rn(__fmul_rn(__fadd_rn(q[d], 1.f), 0.5f), float(r - 1));
                ix = fminf(fmaxf(ix, 0.f), float(r - 1));
                const float fl = floorf(ix);
                i0[d] = int(fl);
                i1[d] = min(i0[d] + 1, r - 1);    // its weight is 0 when clipped to the last node
                f[d] = ix - fl;
            }
            float v[GS4D_PLANES];
#pragma unroll
            for (int k = 0; k < GS4D_PLANES; ++k) {
                const int a = plane_a(k), b = plane_b(k), ra = s.res[l][a];
                const float* P = p.planes + p.off[l][k] + c;
                const float v00 = __ldg(P + (i0[b] * ra + i0[a]) * C), v01 = __ldg(P + (i0[b] * ra + i1[a]) * C);
                const float v10 = __ldg(P + (i1[b] * ra + i0[a]) * C), v11 = __ldg(P + (i1[b] * ra + i1[a]) * C);
                const float fa = f[a], fb = f[b], ea = 1.f - fa, eb = 1.f - fb;
                v[k] = v00 * (ea * eb) + v01 * (fa * eb) + v10 * (ea * fb) + v11 * (fa * fb);
            }
            float prod = 1.f;
#pragma unroll
            for (int k = 0; k < GS4D_PLANES; ++k) prod *= v[k];
            x[l * C + c] = prod;
        }
    }
    __syncwarp();
}

// layer li's weights [rows, K] (rows padded with zeros to a multiple of 8) and bias into shared memory, by the whole CTA
__device__ void stage_layer(const Gs4dParams& p, const Gs4dLayout& lay, float* sm, int li, int K, int rows) {
    const int pad = (rows + 7) / 8 * 8, k4 = K / 4, S = K + 4;
    const float4* W = reinterpret_cast<const float4*>(p.W[li]);
    for (int i = threadIdx.x; i < pad * k4; i += blockDim.x) {
        const int r = i / k4, c4 = i - r * k4;
        const float4 v = r < rows ? __ldg(W + r * k4 + c4) : make_float4(0.f, 0.f, 0.f, 0.f);
        *reinterpret_cast<float4*>(sm + lay.Wt + r * S + 4 * c4) = v;
    }
    for (int i = threadIdx.x; i < pad; i += blockDim.x) sm[lay.bias + i] = i < rows ? __ldg(p.b[li] + i) : 0.f;
}

// this warp's 16 rows: Y = relu(X Wt^T + b), N = W outputs
__device__ void hidden_layer(const Gs4dLayout& lay, const float* sm, const float* X, int sx, int K, float* Y, int sy, int N, int lane) {
    const int g = lane >> 2, t = lane & 3;
    for (int n0 = 0; n0 < N; n0 += 64) {
        float acc[8][4];
        zero_acc(acc);
        warp_gemm<false>(X, sx, K, sm + lay.Wt, K + 4, n0, min(8, (N - n0) / 8), acc, lane);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int c = n0 + 8 * j + 2 * t;
            if (c < N) {
                const float b0 = sm[lay.bias + c], b1 = sm[lay.bias + c + 1];
                Y[g * sy + c] = fmaxf(acc[j][0] + b0, 0.f);
                Y[g * sy + c + 1] = fmaxf(acc[j][1] + b1, 0.f);
                Y[(g + 8) * sy + c] = fmaxf(acc[j][2] + b0, 0.f);
                Y[(g + 8) * sy + c + 1] = fmaxf(acc[j][3] + b1, 0.f);
            }
        }
    }
    __syncwarp();
}

// this warp's 16 rows of a head's output layer (N <= 48 outputs), written over the first N columns of its input X once read
__device__ void output_layer(const Gs4dLayout& lay, const float* sm, float* X, int sx, int K, int N, int lane) {
    const int g = lane >> 2, t = lane & 3, nt = (N + 7) / 8;
    float acc[6][4];
    zero_acc(acc);
    warp_gemm<false>(X, sx, K, sm + lay.Wt, K + 4, 0, nt, acc, lane);
    __syncwarp();
#pragma unroll
    for (int j = 0; j < 6; ++j) {
        const int c = 8 * j + 2 * t;
        if (j < nt) {
            const float b0 = sm[lay.bias + c], b1 = sm[lay.bias + c + 1];
            X[g * sx + c] = acc[j][0] + b0;
            X[g * sx + c + 1] = acc[j][1] + b1;
            X[(g + 8) * sx + c] = acc[j][2] + b0;
            X[(g + 8) * sx + c + 1] = acc[j][3] + b1;
        }
    }
    __syncwarp();
}

// head h's outputs Z (row stride sz) added to this warp's rows
__device__ void epilogue(const Gs4dParams& p, int h, const float* Z, int sz, int64_t row0, int lane) {
    if (h == 3) {                             // shs' = shs + dshs.reshape(16, 3): dc [n,1,3] and rest [n,15,3]
        for (int i = 0; i < 16; ++i) {
            const int64_t row = row0 + i;
            if (row >= p.n) break;
            for (int k = lane; k < 48; k += 32) {
                if (k < 3) p.dc_out[row * 3 + k] = __ldg(p.dc + row * 3 + k) + Z[i * sz + k];
                else p.rest_out[row * 45 + k - 3] = __ldg(p.rest + row * 45 + k - 3) + Z[i * sz + k];
            }
        }
        return;
    }
    const int64_t row = row0 + lane;
    if (lane >= 16 || row >= p.n) return;
    const float* z = Z + lane * sz;
    if (h == 0) {
        for (int d = 0; d < 3; ++d) p.means_out[row * 3 + d] = __ldg(p.means + row * 3 + d) + z[d];
    } else if (h == 1) {
        for (int d = 0; d < 3; ++d) p.scales_out[row * 3 + d] = __ldg(p.scales + row * 3 + d) + z[d];
    } else if (p.s.flags & B200GS_GS4D_APPLY_ROTATION) {     // batch_quaternion_multiply(q, dr), then divided by its norm
        const float4 a = *reinterpret_cast<const float4*>(p.quats + row * 4);
        const float w = a.x * z[0] - a.y * z[1] - a.z * z[2] - a.w * z[3];
        const float x = a.x * z[1] + a.y * z[0] + a.z * z[3] - a.w * z[2];
        const float y = a.x * z[2] - a.y * z[3] + a.z * z[0] + a.w * z[1];
        const float zz = a.x * z[3] + a.y * z[2] - a.z * z[1] + a.w * z[0];
        const float nrm = __fsqrt_rn(w * w + x * x + y * y + zz * zz);
        *reinterpret_cast<float4*>(p.quats_out + row * 4) =
            make_float4(__fdiv_rn(w, nrm), __fdiv_rn(x, nrm), __fdiv_rn(y, nrm), __fdiv_rn(zz, nrm));
    } else {
        const float4 a = *reinterpret_cast<const float4*>(p.quats + row * 4);
        *reinterpret_cast<float4*>(p.quats_out + row * 4) = make_float4(a.x + z[0], a.y + z[1], a.z + z[2], a.w + z[3]);
    }
}

// the parameters of disabled heads, copied through
__device__ void copy_through(const Gs4dParams& p, int64_t row0, int lane) {
    const int64_t row = row0 + lane;
    if (lane >= 16 || row >= p.n) return;
    const int f = p.s.flags;
    if (!(f & B200GS_GS4D_DX))
        for (int d = 0; d < 3; ++d) p.means_out[row * 3 + d] = __ldg(p.means + row * 3 + d);
    if (!(f & B200GS_GS4D_DS))
        for (int d = 0; d < 3; ++d) p.scales_out[row * 3 + d] = __ldg(p.scales + row * 3 + d);
    if (!(f & B200GS_GS4D_DR))
        *reinterpret_cast<float4*>(p.quats_out + row * 4) = __ldg(reinterpret_cast<const float4*>(p.quats) + row);
}

__global__ void __launch_bounds__(GS4D_THREADS, 1) gs4d_deform_kernel(const Gs4dParams p, const Gs4dLayout lay) {
    extern __shared__ __align__(16) float sm[];
    const Gs4dShape& s = p.s;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, sa = s.sa(), sb = s.sb();
    float* A = sm + lay.A + warp * 16 * sa;
    float* B = sm + lay.B + warp * 16 * sb;
    const int64_t tiles = (p.n + GS4D_ROWS - 1) / GS4D_ROWS;
    for (int64_t tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
        const int64_t row0 = tile * GS4D_ROWS + warp * 16;
        gather(p, A, sa, row0, lane);
        copy_through(p, row0, lane);
        // trunk: A -> B (-> A); every trunk output is read through a ReLU (the next trunk layer's or each head's first)
        float* T = A;
        int st = sa;
        for (int l = 0; l < s.trunk(); ++l) {
            __syncthreads();                  // every warp is done with the previous layer's weights
            stage_layer(p, lay, sm, l, l == 0 ? s.k0() : s.W, s.W);
            __syncthreads();
            float* Y = T == A ? B : A;
            const int sy = T == A ? sb : sa;
            hidden_layer(lay, sm, T, st, l == 0 ? s.k0() : s.W, Y, sy, s.W, lane);
            T = Y;
            st = sy;
        }
        float* S = T == A ? B : A;
        const int ss = T == A ? sb : sa;
        for (int h = 0; h < 4; ++h) {
            if (!(s.flags & (1 << h))) continue;
            __syncthreads();
            stage_layer(p, lay, sm, 2 + 2 * h, s.W, s.W);
            __syncthreads();
            hidden_layer(lay, sm, T, st, s.W, S, ss, s.W, lane);
            __syncthreads();
            stage_layer(p, lay, sm, 3 + 2 * h, s.W, head_out(h));
            __syncthreads();
            output_layer(lay, sm, S, ss, s.W, head_out(h), lane);
            epilogue(p, h, S, ss, row0, lane);
        }
    }
}

struct RepackParams {
    const float* src[GS4D_MAX_LEVELS * GS4D_PLANES];
    int64_t off[GS4D_MAX_LEVELS * GS4D_PLANES + 1];
    int ra[GS4D_MAX_LEVELS * GS4D_PLANES];
    int count, C;
    float* dst;
};

__global__ void gs4d_repack_kernel(const RepackParams p) {
    const int64_t total = p.off[p.count];
    for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += int64_t(gridDim.x) * blockDim.x) {
        int k = 0;
        while (i >= p.off[k + 1]) ++k;
        const int64_t local = i - p.off[k], cell = local / p.C, plane = (p.off[k + 1] - p.off[k]) / p.C;
        const int c = int(local - cell * p.C);
        p.dst[i] = __ldg(p.src[k] + c * plane + cell);
    }
}

bool gs4d_shape(const B200gsGs4d* g, Gs4dShape* s, int64_t off[GS4D_MAX_LEVELS][GS4D_PLANES], int64_t* total) {
    if (g == nullptr) return false;
    if (g->n_levels < 1 || g->n_levels > GS4D_MAX_LEVELS || (g->channels != 16 && g->channels != 32) ||
        (g->net_width != 64 && g->net_width != 128) || g->defor_depth < 0 || g->defor_depth > 2 || (g->flags & ~B200GS_GS4D_FLAGS) != 0)
        return false;
    *s = Gs4dShape{g->n_levels, g->channels, g->net_width, g->defor_depth, g->flags, {}};
    int64_t o = 0;
    for (int l = 0; l < g->n_levels; ++l) {
        for (int d = 0; d < 4; ++d) {
            const int r = g->resolution[l][d];
            if (r < 1 || r > B200GS_GS4D_MAX_RES) return false;
            s->res[l][d] = r;
        }
        for (int k = 0; k < GS4D_PLANES; ++k) {
            const int64_t floats = int64_t(s->res[l][plane_a(k)]) * s->res[l][plane_b(k)] * g->channels;
            if (floats > INT32_MAX) return false;     // K51 indexes within a plane in int
            if (off) off[l][k] = o;
            o += floats;
        }
    }
    if (size_t(gs4d_layout(*s).total) * 4 > GS4D_SMEM_LIMIT) return false;
    if (total) *total = o;
    return true;
}

}  // namespace

}  // namespace b200gs

using namespace b200gs;

extern "C" {

int64_t b200gs_gs4d_plane_floats(const B200gsGs4d* grid) {
    Gs4dShape s;
    int64_t total = 0;
    return gs4d_shape(grid, &s, nullptr, &total) ? total : 0;
}

int b200gs_gs4d_repack_planes(const B200gsGs4d* grid, const float* const* host_planes, float* planes, void* stream) {
    Gs4dShape s;
    int64_t off[GS4D_MAX_LEVELS][GS4D_PLANES], total = 0;
    if (!gs4d_shape(grid, &s, off, &total)) return fail(__func__, "grid outside the supported set (see b200gs_gs4d_plane_floats)");
    B200GS_CHECK_ARG(host_planes && planes, "NULL planes");
    RepackParams p{};
    p.count = s.L * GS4D_PLANES;
    p.C = s.C;
    p.dst = planes;
    for (int l = 0; l < s.L; ++l)
        for (int k = 0; k < GS4D_PLANES; ++k) {
            const int i = l * GS4D_PLANES + k;
            B200GS_CHECK_ARG(host_planes[i], "NULL plane");
            p.src[i] = host_planes[i];
            p.off[i] = off[l][k];
            p.ra[i] = s.res[l][plane_a(k)];
        }
    p.off[p.count] = total;
    const int grid_blocks = int(std::min<int64_t>(div_up64(total, 256), 132 * 16));
    gs4d_repack_kernel<<<grid_blocks, 256, 0, (cudaStream_t)stream>>>(p);
    B200GS_LAUNCH_CHECK();
    return B200GS_OK;
}

int b200gs_gs4d_deform_fwd(const B200gsGs4d* grid, int64_t n, const float* planes, const float* aabb, const float* time, const float* means,
                           const float* log_scales, const float* quats, const float* shs_dc, const float* shs_rest, float* means_out,
                           float* log_scales_out, float* quats_out, float* shs_dc_out, float* shs_rest_out, void* stream) {
    Gs4dParams p{};
    if (!gs4d_shape(grid, &p.s, p.off, nullptr)) return fail(__func__, "grid or network outside the supported set (see b200gs_gs4d_plane_floats)");
    B200GS_CHECK_ARG(n >= 0 && n <= INT32_MAX, "n out of range");
    const int layers[GS4D_LAYERS] = {1, p.s.D == 2, 1, 1, 1, 1, 1, 1, 1, 1};
    for (int i = 0; i < GS4D_LAYERS; ++i) {
        const bool used = layers[i] && (i < 2 || (p.s.flags & (1 << ((i - 2) / 2))));
        if (!used) continue;
        B200GS_CHECK_ARG(grid->weights[i] && grid->biases[i], "NULL weight or bias of a layer in use");
        B200GS_CHECK_ARG((reinterpret_cast<uintptr_t>(grid->weights[i]) & 15u) == 0, "weights must be 16-byte aligned");
        p.W[i] = grid->weights[i];
        p.b[i] = grid->biases[i];
    }
    if (n == 0) return B200GS_OK;
    B200GS_CHECK_ARG(planes && aabb && time && means && log_scales && quats, "NULL planes, aabb, time or Gaussian parameters");
    B200GS_CHECK_ARG(means_out && log_scales_out && quats_out, "NULL output");
    B200GS_CHECK_ARG(((reinterpret_cast<uintptr_t>(quats) | reinterpret_cast<uintptr_t>(quats_out)) & 15u) == 0,
                     "quats and quats_out must be 16-byte aligned");
    if (p.s.flags & B200GS_GS4D_DSHS) B200GS_CHECK_ARG(shs_dc && shs_rest && shs_dc_out && shs_rest_out, "NULL SH input or output with dshs on");
    p.n = n;
    p.planes = planes; p.aabb = aabb; p.time = time;
    p.means = means; p.scales = log_scales; p.quats = quats; p.dc = shs_dc; p.rest = shs_rest;
    p.means_out = means_out; p.scales_out = log_scales_out; p.quats_out = quats_out; p.dc_out = shs_dc_out; p.rest_out = shs_rest_out;
    const Gs4dLayout lay = gs4d_layout(p.s);
    const int smem = lay.total * 4;
    const int ctas = int(std::min<int64_t>(GS4D_MAX_CTAS, div_up64(n, GS4D_ROWS)));
    B200GS_CUDA(cudaFuncSetAttribute(gs4d_deform_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    gs4d_deform_kernel<<<ctas, GS4D_THREADS, smem, (cudaStream_t)stream>>>(p, lay);
    B200GS_LAUNCH_CHECK();
    return B200GS_OK;
}

}  // extern "C"
