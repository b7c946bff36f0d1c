// Appearance-embedding colour pass (internal/renderers/gsplat_appearance_embedding_renderer.py: Model.forward :77-93 and
// _get_rgbs_and_opacities :239-295): per visible Gaussian an MLP on its appearance features (and, optionally, the positional
// encoding of its view direction), a sigmoid, and the colour / opacity epilogue, in one kernel each way.
//     x0 = [ f | PE(d) | 0.. ]            f = features row (normalised when `normalize`), d = view direction, padded to K0p (mult. of 8)
//     h_l = relu(W_l h_{l-1} + b_l)       l = 0 .. L-2   (b_0 already holds the per-image embedding's product, see b200gs.h)
//     s   = sigmoid(W_{L-1} h_{L-2} + b_{L-1})           (3 or 4 outputs)
//     rgb = clamp(base + 0.5 + (2 s_{0..2} - 1), 0, 1);  offset = s_3;  opacity = min(raw + offset, 1)
//   * K20 appearance_mlp_fwd_kernel / K21 appearance_mlp_bwd_kernel: persistent CTAs.  A CTA walks chunks of blockDim.x consecutive
//     rows, interleaved over the grid; the rows whose mask byte is set are appended to a ring of row indices in shared memory (warp
//     ballots, no host read), the others get their zeros at once.  Whenever the ring holds a full tile (16 rows per warp) the CTA
//     runs it: each warp owns 16 rows, keeps their activations in its slice of shared memory and issues every GEMM as
//     mma.sync.m16n8k8 TF32 with FP32 accumulation.  Both operands are split in registers into a TF32 high part and the TF32
//     rounding of the remainder, and the three significant products are added small terms first (3xTF32: products carry ~21
//     mantissa bits instead of TF32's 10).  The weights sit in shared memory once, as FP32, padded to row strides = 4 (mod 8)
//     floats so neither operand's fragment loads conflict.
//   * K21 recomputes the activations, then per layer from the output down: the weight gradient dpre_l^T h_{l-1} as a CTA-wide GEMM
//     over the tile's rows (each 16 x 32 block of it by one warp, added to this CTA's partial block by that thread alone, so
//     the order of every sum is fixed), the bias gradient as column sums, and each warp's dh_{l-1} = dpre_l W_l, masked by
//     the ReLU, in place over h_{l-1}.  The last step writes v_features (through the normalisation Jacobian when on).
//   * K22 appearance_reduce_kernel adds the CTAs' partial blocks in block order.
// Epilogue 2 is SWAG's (swag_renderer.py:47-56; the rows come from K49, swag.cu): no output activation on o_3, and
//     colour = sigmoid(o_{0..2}),  z = (1 / temperature) ((log(|o_3| + eps) + log(u + eps)) - log(1 - u + eps)),
//     opacity = clamp_min(base_opacity - sigmoid(z), 0)
// with u read through a device pointer.  Only W_0's first w0_cols columns are read, the rest of its first F are zero: SWAG's rows are
// 35 real columns padded to 40, and the caller's W_0 has the image embedding in columns 35..58.
#include <algorithm>
#include <cmath>

#include "common.cuh"
#include "warp_mma.cuh"

namespace b200gs {

namespace {

constexpr int APP_MAX_LAYERS = 4;
constexpr int APP_MAX_CTAS = 132;           // one persistent CTA per SM of an H100 SXM; also the number of partial blocks
constexpr int APP_QUEUE = 512;              // ring of compacted row indices: >= tile rows + one chunk (128 + 256)
constexpr int APP_SMEM_LIMIT = 227 * 1024;  // opt-in dynamic shared memory of sm_90

struct AppShape {
    int F, n_freq, H, L, O;          // feature width, PE frequencies (< 0: no view direction), neurons, layers (output included), outputs
    __host__ __device__ int pe() const { return n_freq < 0 ? 0 : 3 * (2 * n_freq + 1); }
    __host__ __device__ int k0p() const { return (F + pe() + 7) / 8 * 8; }
    __host__ __device__ int in(int l) const { return l == 0 ? k0p() : H; }
    __host__ __device__ int out(int l) const { return l == L - 1 ? O : H; }            // rows of W_l
    __host__ __device__ int out_pad(int l) const { return l == L - 1 ? 8 : H; }        // as kept in shared memory
    // v_params / partial block: W_0 [H, k0p] | W_1 .. | W_{L-1} [O, H] | b_0 .. | b_{L-1}, dense
    __host__ __device__ int w_off(int l) const { int o = 0; for (int i = 0; i < l; ++i) o += out(i) * in(i); return o; }
    __host__ __device__ int b_off(int l) const { int o = w_off(L); for (int i = 0; i < l; ++i) o += out(i); return o; }
    __host__ __device__ int params() const { return b_off(L); }
};

struct AppLayout {                  // offsets in floats into dynamic shared memory
    int W[APP_MAX_LAYERS], b[APP_MAX_LAYERS], X0, Hb[APP_MAX_LAYERS - 1], DZ, norm, rows, queue, wcnt, total;
};

__host__ __device__ inline AppLayout app_layout(const AppShape& s, int warps, bool bwd) {
    AppLayout a{};
    const int R = 16 * warps;
    int o = 0;
    for (int l = 0; l < s.L; ++l) { a.W[l] = o; o += s.out_pad(l) * (s.in(l) + 4); }
    for (int l = 0; l < s.L; ++l) { a.b[l] = o; o += s.out_pad(l); }
    a.X0 = o; o += R * (s.k0p() + 4);
    const int nh = bwd ? s.L - 1 : (s.L - 1 < 2 ? s.L - 1 : 2);      // the forward ping-pongs between two
    for (int i = 0; i < nh; ++i) { a.Hb[i] = o; o += R * (s.H + 4); }
    a.DZ = o; o += bwd ? R * 12 : 0;
    a.norm = o; o += R;
    a.rows = o; o += R;
    a.queue = o; o += APP_QUEUE;
    a.wcnt = o; o += 8;
    a.total = o;
    return a;
}

// the most warps (8, 4, 2, 1) whose tile fits shared memory; 0: the network does not fit
inline int app_warps(const AppShape& s, bool bwd) {
    for (int w = 8; w >= 1; w >>= 1)
        if (size_t(app_layout(s, w, bwd).total) * 4 <= APP_SMEM_LIMIT) return w;
    return 0;
}

struct AppParams {
    AppShape s;
    int64_t n;
    int normalize, normalize_dirs, epilogue;
    const float* features; const uint8_t* mask; const float* base_rgb; const float* dirs; const float* cam; const float* raw_opacity;
    const float* W[APP_MAX_LAYERS]; const float* b[APP_MAX_LAYERS];
    int w0_stride, w0_pe_col, w0_cols;
    const float* u; float inv_temp, eps;                                                    // epilogue 2
    float* out; float* opacity_offsets; float* opacities;                                   // forward
    const float* v_out; const float* v_opacities; const float* v_opacity_offsets;           // backward
    float* v_base_rgb; float* v_features; float* v_raw_opacity; float* partials;
};

struct Tile {            // what every device function of a tile needs
    const AppParams& p;
    const AppLayout& lay;
    float* sm;
    int warp, lane, R;
    __device__ float* X0() const { return sm + lay.X0; }
    __device__ float* Hb(int i) const { return sm + lay.Hb[i]; }
    __device__ int* rows() const { return reinterpret_cast<int*>(sm + lay.rows); }
};

// sin and cos in fp64 (the build's fast-math fp32 versions lose bits the first layer amplifies): Cody-Waite reduction by pi/2 and
// the Taylor polynomials on [-pi/4, pi/4] (remainders < 1e-15); view directions are unit vectors, |x| <= 1
__device__ __forceinline__ void sincos_f64(double x, double* sn, double* cs) {
    const double q = rint(x * 0.63661977236758134);
    double r = fma(-q, 1.5707963267948966, x);
    r = fma(-q, 6.123233995736766e-17, r);
    const double r2 = r * r;
    double ps = -1. / 1307674368000.;
    ps = fma(ps, r2, 1. / 6227020800.); ps = fma(ps, r2, -1. / 39916800.); ps = fma(ps, r2, 1. / 362880.);
    ps = fma(ps, r2, -1. / 5040.); ps = fma(ps, r2, 1. / 120.); ps = fma(ps, r2, -1. / 6.);
    ps = fma(ps * r2, r, r);
    double pc = -1. / 87178291200.;
    pc = fma(pc, r2, 1. / 479001600.); pc = fma(pc, r2, -1. / 3628800.); pc = fma(pc, r2, 1. / 40320.);
    pc = fma(pc, r2, -1. / 720.); pc = fma(pc, r2, 1. / 24.); pc = fma(pc, r2, -0.5);
    pc = fma(pc, r2, 1.);
    const int k = int(q) & 3;
    const double s0 = (k & 1) ? pc : ps, c0 = (k & 1) ? ps : pc;
    *sn = (k & 2) ? -s0 : s0;
    *cs = ((k + 1) & 2) ? -c0 : c0;
}

__device__ __forceinline__ float sigmoidf(float z) { return 1.f / (1.f + expf(-z)); }

// weights and biases into shared memory, once per CTA: W_0 keeps its feature and view-direction columns (the embedding's are folded
// into b_0 by the caller), the output layer is padded to 8 rows of zeros
__device__ void load_weights(const AppParams& p, const AppLayout& lay, float* sm) {
    const AppShape& s = p.s;
    for (int l = 0; l < s.L; ++l) {
        const int in = s.in(l), S = in + 4, rows = s.out_pad(l), real = s.out(l);
        for (int i = threadIdx.x; i < rows * S; i += blockDim.x) {
            const int r = i / S, c = i - r * S;
            float v = 0.f;
            if (r < real && c < in) {
                if (l == 0) {
                    if (c < s.F) v = c < p.w0_cols ? __ldg(p.W[0] + int64_t(r) * p.w0_stride + c) : 0.f;
                    else if (c < s.F + s.pe()) v = __ldg(p.W[0] + int64_t(r) * p.w0_stride + p.w0_pe_col + (c - s.F));
                } else {
                    v = __ldg(p.W[l] + r * in + c);
                }
            }
            sm[lay.W[l] + i] = v;
        }
        for (int i = threadIdx.x; i < rows; i += blockDim.x) sm[lay.b[l] + i] = i < real ? __ldg(p.b[l] + i) : 0.f;
    }
}

// this warp's 16 rows of x0 (zeros for the rows of a short tile), and 1 / max(|f|, 1e-12) of each when normalising
__device__ void load_inputs(const Tile& T) {
    const AppParams& p = T.p;
    const AppShape& s = p.s;
    const int S = s.k0p() + 4, F = s.F, pe = s.pe();
    float* X = T.X0() + T.warp * 16 * S;
    const int* rows = T.rows() + T.warp * 16;
    for (int i = 0; i < 16; ++i) {
        const int row = rows[i];
        float ss = 0.f;
        for (int c = T.lane; c < F; c += 32) {
            const float v = row >= 0 ? __ldg(p.features + int64_t(row) * F + c) : 0.f;
            X[i * S + c] = v;
            ss = fmaf(v, v, ss);
        }
        for (int c = F + pe + T.lane; c < s.k0p(); c += 32) X[i * S + c] = 0.f;
        if (p.normalize) {
            const float inv = 1.f / fmaxf(sqrtf(warp_sum(ss)), 1e-12f);
            for (int c = T.lane; c < F; c += 32) X[i * S + c] *= inv;
            if (T.lane == 0) T.sm[T.lay.norm + T.warp * 16 + i] = inv;
        }
    }
    if (pe > 0 && T.lane < 16) {          // one row per lane: (d, sin 2^k d, cos 2^k d ..), the base angle in fp64, then angle doubling
        const int row = rows[T.lane];
        float* x = X + T.lane * S + F;
        double d[3] = {0., 0., 0.};
        if (row >= 0) {
#pragma unroll
            for (int c = 0; c < 3; ++c) d[c] = double(__ldg(p.dirs + int64_t(row) * 3 + c) - (p.cam ? __ldg(p.cam + c) : 0.f));
            if (p.normalize_dirs) {       // F.normalize in fp32, as the reference
                const float fx = float(d[0]), fy = float(d[1]), fz = float(d[2]);
                const float nrm = fmaxf(sqrtf(fx * fx + fy * fy + fz * fz), 1e-12f);
                d[0] = double(fx / nrm); d[1] = double(fy / nrm); d[2] = double(fz / nrm);
            }
        }
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            x[c] = float(d[c]);
            double sn, cs;
            sincos_f64(d[c], &sn, &cs);
            for (int k = 0; k < s.n_freq; ++k) {
                x[3 + 6 * k + c] = float(sn);
                x[6 + 6 * k + c] = float(cs);
                const double s2 = 2. * sn * cs;
                cs = 1. - 2. * sn * sn;
                sn = s2;
            }
        }
    }
    __syncwarp();
}

// the hidden layers on this warp's rows; returns the buffer index of h_{L-2}.  PINGPONG: two buffers (forward), else one per layer
template <bool PINGPONG>
__device__ int hidden_layers(const Tile& T) {
    const AppShape& s = T.p.s;
    const int g = T.lane >> 2, t = T.lane & 3, SH = s.H + 4;
    int prev = -1;
    for (int l = 0; l < s.L - 1; ++l) {
        const int cur = PINGPONG ? (l & 1) : l;
        const int sa = l == 0 ? s.k0p() + 4 : SH;
        const float* A = (l == 0 ? T.X0() : T.Hb(prev)) + T.warp * 16 * sa;
        float* Y = T.Hb(cur) + T.warp * 16 * SH;
        for (int n0 = 0; n0 < s.H; n0 += 64) {
            float acc[8][4];
            zero_acc(acc);
            warp_gemm<false>(A, sa, s.in(l), T.sm + T.lay.W[l], s.in(l) + 4, n0, min(8, (s.H - n0) / 8), acc, T.lane);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int c = n0 + 8 * j + 2 * t;
                if (c < s.H) {
                    const float b0 = T.sm[T.lay.b[l] + c], b1 = T.sm[T.lay.b[l] + c + 1];
                    Y[g * SH + c] = fmaxf(acc[j][0] + b0, 0.f);
                    Y[g * SH + c + 1] = fmaxf(acc[j][1] + b1, 0.f);
                    Y[(g + 8) * SH + c] = fmaxf(acc[j][2] + b0, 0.f);
                    Y[(g + 8) * SH + c + 1] = fmaxf(acc[j][3] + b1, 0.f);
                }
            }
        }
        __syncwarp();
        prev = cur;
    }
    return prev;
}

// output pre-activations of this warp's rows: z[0..1] = channels 2t, 2t+1 of row g, z[2..3] of row g + 8
__device__ __forceinline__ void output_layer(const Tile& T, int hbuf, float (&z)[4]) {
    const AppShape& s = T.p.s;
    const int t = T.lane & 3, l = s.L - 1, SH = s.H + 4;
    float acc[1][4];
    zero_acc(acc);
    warp_gemm<false>(T.Hb(hbuf) + T.warp * 16 * SH, SH, s.H, T.sm + T.lay.W[l], SH, 0, 1, acc, T.lane);
    const float b0 = T.sm[T.lay.b[l] + 2 * t], b1 = T.sm[T.lay.b[l] + 2 * t + 1];
    z[0] = acc[0][0] + b0; z[1] = acc[0][1] + b1;
    z[2] = acc[0][2] + b0; z[3] = acc[0][3] + b1;
}

// epilogue 2: sigmoid(z) of the Gumbel-sigmoid opacity term for output o_3 = o
__device__ __forceinline__ float swag_sigmoid_z(const AppParams& p, float o) {
    const float u = __ldg(p.u);
    return sigmoidf(p.inv_temp * ((logf(fabsf(o) + p.eps) + logf(u + p.eps)) - logf(1.f - u + p.eps)));
}

// Append the visible rows of chunk [base, base + blockDim.x) to the ring; returns how many.  `vis` tells the caller whether this
// thread's row exists and is masked out (it then writes that row's zeros).
__device__ __forceinline__ int scan_chunk(const AppParams& p, const AppLayout& lay, float* sm, int64_t base, int tail, bool& in_range, bool& vis) {
    const int64_t row = base + threadIdx.x;
    in_range = row < p.n;
    vis = in_range && (p.mask == nullptr || p.mask[row] != 0);
    const unsigned ballot = __ballot_sync(0xffffffffu, vis);
    int* wcnt = reinterpret_cast<int*>(sm + lay.wcnt);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0) wcnt[warp] = __popc(ballot);
    __syncthreads();
    int before = 0, total = 0;
    for (int w = 0; w < int(blockDim.x >> 5); ++w) {
        const int c = wcnt[w];
        before += w < warp ? c : 0;
        total += c;
    }
    if (vis) reinterpret_cast<int*>(sm + lay.queue)[(tail + before + __popc(ballot & ((1u << lane) - 1u))) & (APP_QUEUE - 1)] = int(row);
    __syncthreads();
    return total;
}

__device__ __forceinline__ void tile_rows(const Tile& T, int head, int count) {
    const int r = threadIdx.x;
    if (r < T.R) T.rows()[r] = r < count ? reinterpret_cast<const int*>(T.sm + T.lay.queue)[(head + r) & (APP_QUEUE - 1)] : -1;
    __syncthreads();
}

__device__ void fwd_tile(const Tile& T, int head, int count) {
    const AppParams& p = T.p;
    const AppShape& s = p.s;
    tile_rows(T, head, count);
    load_inputs(T);
    const int hb = hidden_layers<true>(T);
    float zo[4];
    output_layer(T, hb, zo);
    const int g = T.lane >> 2, t = T.lane & 3;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int row = T.rows()[T.warp * 16 + g + 8 * h];
        if (row < 0) continue;
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            const int c = 2 * t + e;
            const float v = sigmoidf(zo[2 * h + e]);
            if (c >= s.O) continue;
            if (p.epilogue == 2) {
                if (c < 3) {
                    p.out[int64_t(row) * 3 + c] = v;
                } else {
                    const float o = __ldg(p.raw_opacity + row) - swag_sigmoid_z(p, zo[2 * h + e]);
                    p.opacities[row] = o < 0.f ? 0.f : o;           // NaN stays NaN, as in torch.clamp_min
                }
            } else if (!p.epilogue) {
                p.out[int64_t(row) * s.O + c] = v;
            } else if (c < 3) {
                const float base = __ldg(p.base_rgb + int64_t(row) * 3 + c) + 0.5f;
                p.out[int64_t(row) * 3 + c] = fminf(fmaxf(base + (v * 2.f - 1.f), 0.f), 1.f);
            } else {
                p.opacity_offsets[row] = v;
                p.opacities[row] = fminf(v + __ldg(p.raw_opacity + row), 1.f);
            }
        }
    }
    __syncthreads();      // the ring slots and the row list are free again
}

__global__ void __launch_bounds__(256, 1) appearance_mlp_fwd_kernel(const AppParams p, const AppLayout lay) {
    extern __shared__ __align__(16) float sm[];
    const Tile T{p, lay, sm, int(threadIdx.x >> 5), int(threadIdx.x & 31), int(blockDim.x >> 5) * 16};
    load_weights(p, lay, sm);
    __syncthreads();
    int head = 0, tail = 0;
    for (int64_t base = int64_t(blockIdx.x) * blockDim.x; base < p.n; base += int64_t(gridDim.x) * blockDim.x) {
        bool in_range, vis;
        tail += scan_chunk(p, lay, sm, base, tail, in_range, vis);
        if (in_range && !vis) {           // a row outside the mask: zeros, and its own opacity
            const int64_t row = base + threadIdx.x;
            const int width = p.epilogue ? 3 : p.s.O;
            for (int c = 0; c < width; ++c) p.out[row * width + c] = 0.f;
            if (p.epilogue && p.s.O == 4) {
                p.opacity_offsets[row] = 0.f;
                p.opacities[row] = fminf(__ldg(p.raw_opacity + row), 1.f);
            }
        }
        while (tail - head >= T.R) {
            fwd_tile(T, head, T.R);
            head += T.R;
        }
    }
    if (tail > head) fwd_tile(T, head, tail - head);
}

// One warp: a 16 x (8 nt) block of dW_l = D^T P summed over the tile's R rows, added to this CTA's partial block.  D [R, M] holds
// dpre_l (row stride sd), P [R, in_l] the layer's input (stride sp).
__device__ void dw_block(const float* D, int sd, int m_pad, int m_real, const float* P, int sp, int R, int m0, int n0, int nt, float* dst, int ld,
                         int lane) {
    const int g = lane >> 2, t = lane & 3;
    const bool upper = m0 + g + 8 < m_pad;
    float acc[4][4];
    zero_acc(acc);
    for (int r0 = 0; r0 < R; r0 += 8) {
        uint32_t ah[4], al[4];
        split_tf32(D[(r0 + t) * sd + m0 + g], ah[0], al[0]);
        split_tf32(upper ? D[(r0 + t) * sd + m0 + g + 8] : 0.f, ah[1], al[1]);
        split_tf32(D[(r0 + t + 4) * sd + m0 + g], ah[2], al[2]);
        split_tf32(upper ? D[(r0 + t + 4) * sd + m0 + g + 8] : 0.f, ah[3], al[3]);
#pragma unroll
        for (int j = 0; j < 4; ++j)
            if (j < nt) mma_3xtf32(acc[j], ah, al, P[(r0 + t) * sp + n0 + 8 * j + g], P[(r0 + t + 4) * sp + n0 + 8 * j + g]);
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        if (j >= nt) continue;
        const int c = n0 + 8 * j + 2 * t;
        if (m0 + g < m_real) {
            atomicAdd(dst + (m0 + g) * ld + c, acc[j][0]);
            atomicAdd(dst + (m0 + g) * ld + c + 1, acc[j][1]);
        }
        if (m0 + g + 8 < m_real) {
            atomicAdd(dst + (m0 + g + 8) * ld + c, acc[j][2]);
            atomicAdd(dst + (m0 + g + 8) * ld + c + 1, acc[j][3]);
        }
    }
}

// dW_l and db_l of the tile, by the whole CTA.  Every element of the partial block is only ever touched by one thread.
__device__ void weight_grads(const Tile& T, int l, const float* D, int sd, const float* P, int sp, float* partial) {
    const AppShape& s = T.p.s;
    const int m_pad = s.out_pad(l), m_real = s.out(l), in = s.in(l);
    const int mt = (m_pad + 15) / 16, nc = (in / 8 + 3) / 4, warps = T.R / 16;
    for (int u = T.warp; u < mt * nc; u += warps) {
        const int m0 = (u / nc) * 16, n0 = (u % nc) * 32;
        dw_block(D, sd, m_pad, m_real, P, sp, T.R, m0, n0, min(4, (in - n0) / 8), partial + s.w_off(l), in, T.lane);
    }
    for (int j = threadIdx.x; j < m_real; j += blockDim.x) {
        float sum = 0.f;
        for (int r = 0; r < T.R; ++r) sum += D[r * sd + j];
        atomicAdd(partial + s.b_off(l) + j, sum);
    }
}

__device__ void bwd_tile(const Tile& T, int head, int count, float* partial) {
    const AppParams& p = T.p;
    const AppShape& s = p.s;
    const int g = T.lane >> 2, t = T.lane & 3, SH = s.H + 4, S0 = s.k0p() + 4;
    tile_rows(T, head, count);
    load_inputs(T);
    const int hb = hidden_layers<false>(T);
    float zo[4];
    output_layer(T, hb, zo);
    // the epilogue's gradient: dz of this thread's two channels of rows g and g + 8
    float* DZ = T.sm + T.lay.DZ;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int r = T.warp * 16 + g + 8 * h, row = T.rows()[r];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            const int c = 2 * t + e;
            const float v = sigmoidf(zo[2 * h + e]);
            float ds = 0.f, dz_raw = 0.f;
            if (row >= 0 && c < s.O && p.epilogue == 2) {
                if (c < 3) {
                    ds = __ldg(p.v_out + int64_t(row) * 3 + c);
                } else {        // o_3 has no activation: its gradient goes to DZ as it is
                    const float o = zo[2 * h + e], sz = swag_sigmoid_z(p, o);
                    const float gb = (__ldg(p.raw_opacity + row) - sz >= 0.f && p.v_opacities) ? __ldg(p.v_opacities + row) : 0.f;
                    p.v_raw_opacity[row] = gb;
                    const float ga = -gb * (sz * (1.f - sz)) * p.inv_temp / (fabsf(o) + p.eps);
                    dz_raw = o > 0.f ? ga : (o < 0.f ? -ga : 0.f);
                }
            } else if (row >= 0 && c < s.O) {
                if (!p.epilogue) {
                    ds = __ldg(p.v_out + int64_t(row) * s.O + c);
                } else if (c < 3) {
                    const float pre = (__ldg(p.base_rgb + int64_t(row) * 3 + c) + 0.5f) + (v * 2.f - 1.f);
                    const float gr = (pre >= 0.f && pre <= 1.f) ? __ldg(p.v_out + int64_t(row) * 3 + c) : 0.f;
                    p.v_base_rgb[int64_t(row) * 3 + c] = gr;
                    ds = 2.f * gr;
                } else {
                    const float raw = __ldg(p.raw_opacity + row);
                    const float go = (v + raw <= 1.f && p.v_opacities) ? __ldg(p.v_opacities + row) : 0.f;
                    p.v_raw_opacity[row] = go;
                    ds = go + (p.v_opacity_offsets ? __ldg(p.v_opacity_offsets + row) : 0.f);
                }
            }
            DZ[r * 12 + c] = (p.epilogue == 2 && c == 3) ? dz_raw : ds * v * (1.f - v);
        }
    }
    __syncthreads();
    for (int l = s.L - 1; l >= 0; --l) {
        const float* D = l == s.L - 1 ? DZ : T.Hb(l);
        const int sd = l == s.L - 1 ? 12 : SH;
        weight_grads(T, l, D, sd, l == 0 ? T.X0() : T.Hb(l - 1), l == 0 ? S0 : SH, partial);
        __syncthreads();        // every warp has read h_{l-1}; its owner may now overwrite it with dpre_{l-1}
        const float* Dw = D + T.warp * 16 * sd;
        const float* W = T.sm + T.lay.W[l];
        if (l > 0) {
            float* Y = T.Hb(l - 1) + T.warp * 16 * SH;
            for (int n0 = 0; n0 < s.H; n0 += 64) {
                float acc[8][4];
                zero_acc(acc);
                warp_gemm<true>(Dw, sd, s.out_pad(l), W, SH, n0, min(8, (s.H - n0) / 8), acc, T.lane);
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const int c = n0 + 8 * j + 2 * t;
                    if (c < s.H) {
                        Y[g * SH + c] = Y[g * SH + c] > 0.f ? acc[j][0] : 0.f;
                        Y[g * SH + c + 1] = Y[g * SH + c + 1] > 0.f ? acc[j][1] : 0.f;
                        Y[(g + 8) * SH + c] = Y[(g + 8) * SH + c] > 0.f ? acc[j][2] : 0.f;
                        Y[(g + 8) * SH + c + 1] = Y[(g + 8) * SH + c + 1] > 0.f ? acc[j][3] : 0.f;
                    }
                }
            }
        } else if (p.v_features) {
            // v_features = dpre_0 W_0[:, :F]; with `normalize`, y = f / |f|:  v_f = (dy - y (y . dy)) / |f|.  dy is staged in
            // v_features itself: each thread re-reads only what it wrote
            const float* X = T.X0() + T.warp * 16 * S0;
            const int row0 = T.rows()[T.warp * 16 + g], row1 = T.rows()[T.warp * 16 + g + 8];
            float dot0 = 0.f, dot1 = 0.f;
            for (int n0 = 0; n0 < s.F; n0 += 64) {
                float acc[8][4];
                zero_acc(acc);
                warp_gemm<true>(Dw, sd, s.out_pad(0), W, S0, n0, min(8, (s.F - n0) / 8), acc, T.lane);
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const int c = n0 + 8 * j + 2 * t;
                    if (c < s.F) {
                        dot0 += acc[j][0] * X[g * S0 + c] + acc[j][1] * X[g * S0 + c + 1];
                        dot1 += acc[j][2] * X[(g + 8) * S0 + c] + acc[j][3] * X[(g + 8) * S0 + c + 1];
                        if (row0 >= 0) *reinterpret_cast<float2*>(p.v_features + int64_t(row0) * s.F + c) = make_float2(acc[j][0], acc[j][1]);
                        if (row1 >= 0) *reinterpret_cast<float2*>(p.v_features + int64_t(row1) * s.F + c) = make_float2(acc[j][2], acc[j][3]);
                    }
                }
            }
            if (p.normalize) {
                dot0 += __shfl_xor_sync(0xffffffffu, dot0, 1); dot0 += __shfl_xor_sync(0xffffffffu, dot0, 2);
                dot1 += __shfl_xor_sync(0xffffffffu, dot1, 1); dot1 += __shfl_xor_sync(0xffffffffu, dot1, 2);
                const float inv0 = T.sm[T.lay.norm + T.warp * 16 + g], inv1 = T.sm[T.lay.norm + T.warp * 16 + g + 8];
                for (int c = 2 * t; c < s.F; c += 8) {
                    if (row0 >= 0) {
                        float2* q = reinterpret_cast<float2*>(p.v_features + int64_t(row0) * s.F + c);
                        const float2 dy = *q;
                        *q = make_float2((dy.x - X[g * S0 + c] * dot0) * inv0, (dy.y - X[g * S0 + c + 1] * dot0) * inv0);
                    }
                    if (row1 >= 0) {
                        float2* q = reinterpret_cast<float2*>(p.v_features + int64_t(row1) * s.F + c);
                        const float2 dy = *q;
                        *q = make_float2((dy.x - X[(g + 8) * S0 + c] * dot1) * inv1, (dy.y - X[(g + 8) * S0 + c + 1] * dot1) * inv1);
                    }
                }
            }
        }
        __syncthreads();        // dpre_{l-1} of every row is in place (and, after l = 0, the tile's buffers are free)
    }
}

__global__ void __launch_bounds__(256, 1) appearance_mlp_bwd_kernel(const AppParams p, const AppLayout lay) {
    extern __shared__ __align__(16) float sm[];
    const Tile T{p, lay, sm, int(threadIdx.x >> 5), int(threadIdx.x & 31), int(blockDim.x >> 5) * 16};
    float* partial = p.partials + int64_t(blockIdx.x) * p.s.params();
    for (int i = threadIdx.x; i < p.s.params(); i += blockDim.x) partial[i] = 0.f;
    load_weights(p, lay, sm);
    __syncthreads();
    int head = 0, tail = 0;
    for (int64_t base = int64_t(blockIdx.x) * blockDim.x; base < p.n; base += int64_t(gridDim.x) * blockDim.x) {
        bool in_range, vis;
        tail += scan_chunk(p, lay, sm, base, tail, in_range, vis);
        if (in_range && !vis) {           // a row outside the mask: zero gradients, and the opacity clamp's on its raw opacity
            const int64_t row = base + threadIdx.x;
            if (p.epilogue) p.v_base_rgb[row * 3] = p.v_base_rgb[row * 3 + 1] = p.v_base_rgb[row * 3 + 2] = 0.f;
            if (p.v_raw_opacity) p.v_raw_opacity[row] = (p.v_opacities && __ldg(p.raw_opacity + row) <= 1.f) ? __ldg(p.v_opacities + row) : 0.f;
            if (p.v_features) {
                float4* q = reinterpret_cast<float4*>(p.v_features + row * p.s.F);
                for (int c = 0; c < p.s.F / 4; ++c) q[c] = make_float4(0.f, 0.f, 0.f, 0.f);
            }
        }
        while (tail - head >= T.R) {
            bwd_tile(T, head, T.R, partial);
            head += T.R;
        }
    }
    if (tail > head) bwd_tile(T, head, tail - head, partial);
}

__global__ void appearance_reduce_kernel(const float* __restrict__ partials, int blocks, int params, float* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= params) return;
    float sum = 0.f;
    for (int b = 0; b < blocks; ++b) sum += partials[int64_t(b) * params + i];
    out[i] = sum;
}

bool appearance_mlp_fits(int feat_dim, int n_freq, int n_neurons, int n_layers, int n_out) {
    return app_warps(AppShape{feat_dim, n_freq, n_neurons, n_layers, n_out}, true) > 0;
}

size_t appearance_mlp_workspace_bytes(int feat_dim, int n_freq, int n_neurons, int n_layers, int n_out) {
    return size_t(APP_MAX_CTAS) * size_t(AppShape{feat_dim, n_freq, n_neurons, n_layers, n_out}.params()) * sizeof(float);
}

AppParams app_params(const B200gsAppearanceMlp& m, int64_t n, const float* features, const uint8_t* mask, const float* base_rgb,
                     const float* dirs, const float* cam, const float* raw_opacity) {
    AppParams p{};
    p.s = AppShape{m.feat_dim, m.n_freq, m.n_neurons, m.n_layers, m.n_out};
    p.n = n;
    p.normalize = m.normalize; p.normalize_dirs = m.normalize_dirs; p.epilogue = m.epilogue ? 1 : 0;
    p.features = features; p.mask = mask; p.base_rgb = base_rgb; p.dirs = dirs; p.cam = cam; p.raw_opacity = raw_opacity;
    for (int l = 0; l < m.n_layers; ++l) { p.W[l] = m.weights[l]; p.b[l] = m.biases[l]; }
    p.w0_stride = m.w0_stride; p.w0_pe_col = m.w0_pe_col; p.w0_cols = m.feat_dim;
    return p;
}

// SWAG's epilogue (2) and the real width of its padded rows
struct SwagEpilogue {
    int in_dim;
    const float* u;
    float inv_temp, eps;
};

void set_swag(AppParams& p, const SwagEpilogue* e) {
    if (e == nullptr) return;
    p.epilogue = 2;
    p.w0_cols = e->in_dim; p.u = e->u; p.inv_temp = e->inv_temp; p.eps = e->eps;
}

template <typename K>
int app_launch(K kernel, const AppParams& p, bool bwd, int* grid_out, cudaStream_t s) {
    const int warps = app_warps(p.s, bwd);
    const AppLayout lay = app_layout(p.s, warps, bwd);
    const int threads = 32 * warps, smem = lay.total * 4;
    const int grid = int(std::min<int64_t>(APP_MAX_CTAS, div_up64(p.n, threads)));
    B200GS_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    kernel<<<grid, threads, smem, s>>>(p, lay);
    B200GS_LAUNCH_CHECK();
    *grid_out = grid;
    return B200GS_OK;
}

// The launch path of both networks: the visibility MLP is an appearance MLP with n_freq -1, n_out 1, no normalisation and no
// epilogue.  The shape of m has been validated.
int launch_appearance_mlp_fwd(const B200gsAppearanceMlp& m, int64_t n, const float* features, const uint8_t* mask, const float* base_rgb,
                              const float* dirs, const float* cam, const float* raw_opacity, float* out, float* opacity_offsets,
                              float* opacities, cudaStream_t s, const SwagEpilogue* swag = nullptr) {
    AppParams p = app_params(m, n, features, mask, base_rgb, dirs, cam, raw_opacity);
    set_swag(p, swag);
    p.out = out; p.opacity_offsets = opacity_offsets; p.opacities = opacities;
    int grid;
    return n > 0 ? app_launch(appearance_mlp_fwd_kernel, p, false, &grid, s) : B200GS_OK;
}

int launch_appearance_mlp_bwd(const B200gsAppearanceMlp& m, int64_t n, const float* features, const uint8_t* mask, const float* base_rgb,
                              const float* dirs, const float* cam, const float* raw_opacity, const float* v_out, const float* v_opacities,
                              const float* v_opacity_offsets, float* v_base_rgb, float* v_features, float* v_raw_opacity, float* workspace,
                              float* v_params, cudaStream_t s, const SwagEpilogue* swag = nullptr) {
    AppParams p = app_params(m, n, features, mask, base_rgb, dirs, cam, raw_opacity);
    set_swag(p, swag);
    p.v_out = v_out; p.v_opacities = v_opacities; p.v_opacity_offsets = v_opacity_offsets;
    p.v_base_rgb = v_base_rgb; p.v_features = v_features; p.v_raw_opacity = v_raw_opacity; p.partials = workspace;
    int grid = 0;
    if (n > 0)
        if (int rc = app_launch(appearance_mlp_bwd_kernel, p, true, &grid, s)) return rc;
    const int params = p.s.params();
    appearance_reduce_kernel<<<div_up(params, 256), 256, 0, s>>>(workspace, grid, params, v_params);
    B200GS_LAUNCH_CHECK();
    return B200GS_OK;
}

bool appearance_shape_ok(int32_t feat_dim, int32_t n_freq, int32_t n_neurons, int32_t n_layers, int32_t n_out) {
    return feat_dim >= 8 && feat_dim % 8 == 0 && feat_dim <= 1024 && n_freq <= 16 && (n_neurons == 64 || n_neurons == 128) && n_layers >= 2 &&
           n_layers <= B200GS_APPEARANCE_MAX_LAYERS && (n_out == 3 || n_out == 4) &&
           appearance_mlp_fits(feat_dim, n_freq, n_neurons, n_layers, n_out);
}

int check_appearance(const char* fn, const B200gsAppearanceMlp* m, int64_t n, const float* features, const float* base_rgb,
                     const float* dirs, const float* raw_opacity) {
    if (m == nullptr) return fail(fn, "mlp is NULL");
    if (m->feat_dim < 8 || m->feat_dim % 8 != 0) return fail(fn, "feat_dim must be a positive multiple of 8");
    if (m->n_neurons != 64 && m->n_neurons != 128) return fail(fn, "n_neurons must be 64 or 128");
    if (m->n_layers < 2 || m->n_layers > B200GS_APPEARANCE_MAX_LAYERS) return fail(fn, "n_layers must be 2..4");
    if (m->n_out != 3 && m->n_out != 4) return fail(fn, "n_out must be 3 or 4");
    if (!appearance_shape_ok(m->feat_dim, m->n_freq, m->n_neurons, m->n_layers, m->n_out)) return fail(fn, "network does not fit shared memory");
    const int pe = m->n_freq < 0 ? 0 : 3 * (2 * m->n_freq + 1);
    if (m->w0_stride < m->feat_dim + pe || m->w0_pe_col < m->feat_dim || m->w0_pe_col + pe > m->w0_stride) return fail(fn, "bad w0_stride / w0_pe_col");
    if (n < 0 || n > INT32_MAX) return fail(fn, "n out of range");
    for (int l = 0; l < m->n_layers; ++l)
        if (!m->weights[l] || !m->biases[l]) return fail(fn, "NULL weight or bias pointer");
    if (n > 0) {
        if (!features) return fail(fn, "NULL features");
        if (m->n_freq >= 0 && !dirs) return fail(fn, "NULL dirs with a view direction");
        if (m->epilogue && !base_rgb) return fail(fn, "NULL base_rgb");
        if (m->epilogue && m->n_out == 4 && !raw_opacity) return fail(fn, "NULL raw_opacity");
    }
    return B200GS_OK;
}

bool visibility_shape_ok(int32_t feat_dim, int32_t n_neurons, int32_t n_layers) {
    return feat_dim >= 8 && feat_dim % 8 == 0 && feat_dim <= 32 && (n_neurons == 64 || n_neurons == 128) && n_layers >= 2 &&
           n_layers <= B200GS_APPEARANCE_MAX_LAYERS && appearance_mlp_fits(feat_dim, -1, n_neurons, n_layers, 1);
}

int check_visibility(const char* fn, const B200gsAppearanceMlp* m, int64_t n, const float* enc) {
    if (m == nullptr) return fail(fn, "mlp is NULL");
    if (m->n_freq != -1 || m->n_out != 1 || m->normalize || m->normalize_dirs || m->epilogue)
        return fail(fn, "a visibility network has n_freq -1, n_out 1 and no normalisation or epilogue");
    if (!visibility_shape_ok(m->feat_dim, m->n_neurons, m->n_layers))
        return fail(fn, "feat_dim must be 8, 16, 24 or 32, n_neurons 64 or 128, n_layers 2..4");
    if (m->w0_stride < m->feat_dim || m->w0_pe_col < m->feat_dim || m->w0_pe_col > m->w0_stride) return fail(fn, "bad w0_stride / w0_pe_col");
    if (n < 0 || n > INT32_MAX) return fail(fn, "n out of range");
    for (int l = 0; l < m->n_layers; ++l)
        if (!m->weights[l] || !m->biases[l]) return fail(fn, "NULL weight or bias pointer");
    if (n > 0 && !enc) return fail(fn, "NULL enc");
    return B200GS_OK;
}

bool swag_shape_ok(int32_t feat_dim, int32_t n_neurons, int32_t n_layers) {
    return feat_dim >= 8 && feat_dim % 8 == 0 && feat_dim <= 1024 && (n_neurons == 64 || n_neurons == 128) && n_layers >= 2 &&
           n_layers <= B200GS_APPEARANCE_MAX_LAYERS && appearance_mlp_fits(feat_dim, -1, n_neurons, n_layers, 4);
}

int check_swag(const char* fn, const B200gsAppearanceMlp* m, int32_t in_dim, int64_t n, const float* x0, const float* base_opacity,
               const float* u, float temperature, float eps) {
    if (m == nullptr) return fail(fn, "mlp is NULL");
    if (m->n_freq != -1 || m->n_out != 4 || m->normalize || m->normalize_dirs || m->epilogue != 2)
        return fail(fn, "a SWAG network has n_freq -1, n_out 4, no normalisation and epilogue 2");
    if (!swag_shape_ok(m->feat_dim, m->n_neurons, m->n_layers))
        return fail(fn, "feat_dim must be a positive multiple of 8 that fits shared memory, n_neurons 64 or 128, n_layers 2..4");
    if (in_dim > m->feat_dim || in_dim <= m->feat_dim - 8) return fail(fn, "in_dim must satisfy feat_dim - 8 < in_dim <= feat_dim");
    if (m->w0_stride < in_dim) return fail(fn, "w0_stride < in_dim");
    if (!(temperature > 0.f) || !std::isfinite(temperature) || !(eps >= 0.f) || !std::isfinite(eps))
        return fail(fn, "temperature must be positive and eps non-negative, both finite");
    if (n < 0 || n > INT32_MAX) return fail(fn, "n out of range");
    for (int l = 0; l < m->n_layers; ++l)
        if (!m->weights[l] || !m->biases[l]) return fail(fn, "NULL weight or bias pointer");
    if (n > 0 && !(x0 && base_opacity && u)) return fail(fn, "NULL x0, base_opacity or u");
    return B200GS_OK;
}

}  // namespace

}  // namespace b200gs

using namespace b200gs;

extern "C" {

size_t b200gs_appearance_mlp_workspace_bytes(int32_t feat_dim, int32_t n_freq, int32_t n_neurons, int32_t n_layers, int32_t n_out) {
    if (!appearance_shape_ok(feat_dim, n_freq, n_neurons, n_layers, n_out)) return 0;
    return appearance_mlp_workspace_bytes(feat_dim, n_freq, n_neurons, n_layers, n_out);
}

int b200gs_appearance_mlp_fwd(const B200gsAppearanceMlp* mlp, int64_t n, const float* features, const uint8_t* mask, const float* base_rgb,
                              const float* dirs, const float* cam, const float* raw_opacity, float* out, float* opacity_offsets,
                              float* opacities, void* stream) {
    if (int rc = check_appearance(__func__, mlp, n, features, base_rgb, dirs, raw_opacity)) return rc;
    B200GS_CHECK_ARG(n == 0 || out, "NULL out");
    B200GS_CHECK_ARG(n == 0 || !(mlp->epilogue && mlp->n_out == 4) || (opacity_offsets && opacities), "NULL opacity output");
    return launch_appearance_mlp_fwd(*mlp, n, features, mask, base_rgb, dirs, cam, raw_opacity, out, opacity_offsets, opacities,
                                     (cudaStream_t)stream);
}

int b200gs_appearance_mlp_bwd(const B200gsAppearanceMlp* mlp, int64_t n, const float* features, const uint8_t* mask, const float* base_rgb,
                              const float* dirs, const float* cam, const float* raw_opacity, const float* v_out, const float* v_opacities,
                              const float* v_opacity_offsets, float* v_base_rgb, float* v_features, float* v_raw_opacity, void* workspace,
                              size_t workspace_bytes, float* v_params, void* stream) {
    if (int rc = check_appearance(__func__, mlp, n, features, base_rgb, dirs, raw_opacity)) return rc;
    B200GS_CHECK_ARG(v_params, "NULL v_params");
    B200GS_CHECK_ARG(n == 0 || (v_out && workspace), "NULL v_out or workspace");
    B200GS_CHECK_ARG(n == 0 || !mlp->epilogue || v_base_rgb, "NULL v_base_rgb");
    B200GS_CHECK_ARG(n == 0 || !(mlp->epilogue && mlp->n_out == 4) || v_raw_opacity, "NULL v_raw_opacity");
    B200GS_CHECK_ARG((reinterpret_cast<uintptr_t>(v_features) & 15u) == 0, "v_features must be 16-byte aligned");
    if (n > 0 && workspace_bytes < appearance_mlp_workspace_bytes(mlp->feat_dim, mlp->n_freq, mlp->n_neurons, mlp->n_layers, mlp->n_out))
        return workspace_too_small(__func__);
    return launch_appearance_mlp_bwd(*mlp, n, features, mask, base_rgb, dirs, cam, raw_opacity, v_out, v_opacities, v_opacity_offsets,
                                     v_base_rgb, v_features, v_raw_opacity, static_cast<float*>(workspace), v_params, (cudaStream_t)stream);
}

size_t b200gs_visibility_mlp_workspace_bytes(int32_t feat_dim, int32_t n_neurons, int32_t n_layers) {
    if (!visibility_shape_ok(feat_dim, n_neurons, n_layers)) return 0;
    return appearance_mlp_workspace_bytes(feat_dim, -1, n_neurons, n_layers, 1);
}

int b200gs_visibility_mlp_fwd(const B200gsAppearanceMlp* mlp, int64_t n, const float* enc, float* out, void* stream) {
    if (int rc = check_visibility(__func__, mlp, n, enc)) return rc;
    B200GS_CHECK_ARG(n == 0 || out, "NULL out");
    return launch_appearance_mlp_fwd(*mlp, n, enc, nullptr, nullptr, nullptr, nullptr, nullptr, out, nullptr, nullptr, (cudaStream_t)stream);
}

int b200gs_visibility_mlp_bwd(const B200gsAppearanceMlp* mlp, int64_t n, const float* enc, const float* v_out, float* v_enc,
                              void* workspace, size_t workspace_bytes, float* v_params, void* stream) {
    if (int rc = check_visibility(__func__, mlp, n, enc)) return rc;
    B200GS_CHECK_ARG(v_params, "NULL v_params");
    B200GS_CHECK_ARG(n == 0 || (v_out && workspace), "NULL v_out or workspace");
    B200GS_CHECK_ARG((reinterpret_cast<uintptr_t>(v_enc) & 15u) == 0, "v_enc must be 16-byte aligned");
    if (n > 0 && workspace_bytes < appearance_mlp_workspace_bytes(mlp->feat_dim, -1, mlp->n_neurons, mlp->n_layers, 1))
        return workspace_too_small(__func__);
    return launch_appearance_mlp_bwd(*mlp, n, enc, nullptr, nullptr, nullptr, nullptr, nullptr, v_out, nullptr, nullptr, nullptr, v_enc,
                                     nullptr, static_cast<float*>(workspace), v_params, (cudaStream_t)stream);
}

size_t b200gs_swag_mlp_workspace_bytes(int32_t feat_dim, int32_t n_neurons, int32_t n_layers) {
    if (!swag_shape_ok(feat_dim, n_neurons, n_layers)) return 0;
    return appearance_mlp_workspace_bytes(feat_dim, -1, n_neurons, n_layers, 4);
}

int b200gs_swag_mlp_fwd(const B200gsAppearanceMlp* mlp, int32_t in_dim, int64_t n, const float* x0, const float* base_opacity, const float* u,
                        float temperature, float eps, float* colour, float* opacity, void* stream) {
    if (int rc = check_swag(__func__, mlp, in_dim, n, x0, base_opacity, u, temperature, eps)) return rc;
    B200GS_CHECK_ARG(n == 0 || (colour && opacity), "NULL colour or opacity");
    const SwagEpilogue e{in_dim, u, float(1.0 / double(temperature)), eps};
    return launch_appearance_mlp_fwd(*mlp, n, x0, nullptr, nullptr, nullptr, nullptr, base_opacity, colour, nullptr, opacity,
                                     (cudaStream_t)stream, &e);
}

int b200gs_swag_mlp_bwd(const B200gsAppearanceMlp* mlp, int32_t in_dim, int64_t n, const float* x0, const float* base_opacity, const float* u,
                        float temperature, float eps, const float* v_colour, const float* v_opacity, float* v_x0, float* v_base_opacity,
                        void* workspace, size_t workspace_bytes, float* v_params, void* stream) {
    if (int rc = check_swag(__func__, mlp, in_dim, n, x0, base_opacity, u, temperature, eps)) return rc;
    B200GS_CHECK_ARG(v_params, "NULL v_params");
    B200GS_CHECK_ARG(n == 0 || (v_colour && v_base_opacity && workspace), "NULL v_colour, v_base_opacity or workspace");
    B200GS_CHECK_ARG((reinterpret_cast<uintptr_t>(v_x0) & 15u) == 0, "v_x0 must be 16-byte aligned");
    if (n > 0 && workspace_bytes < appearance_mlp_workspace_bytes(mlp->feat_dim, -1, mlp->n_neurons, mlp->n_layers, 4))
        return workspace_too_small(__func__);
    const SwagEpilogue e{in_dim, u, float(1.0 / double(temperature)), eps};
    return launch_appearance_mlp_bwd(*mlp, n, x0, nullptr, nullptr, nullptr, nullptr, base_opacity, v_colour, v_opacity, nullptr, nullptr,
                                     v_x0, v_base_opacity, static_cast<float*>(workspace), v_params, (cudaStream_t)stream, &e);
}

}  // extern "C"
