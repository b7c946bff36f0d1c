// K1 / K8: per-Gaussian EWA projection + SH colour, forward and backward, both constant sets.
//
// One thread per Gaussian.  Forward restates the arithmetic of
//   internal/utils/gaussian_projection.py:6-138   (gsplat mode; live-pinned by tests/golden)
//   internal/utils/sh_utils.py:57-112             (SH polynomials)
// and, for vanilla mode, the published preprocessCUDA of diff-gaussian-rasterization@59f5f77 (SURVEY §8c).
// Backward is hand-derived (DESIGN.md §K8) and checked against torch autograd through the oracle.
//
// HBM-bound: per visible Gaussian 268 B fwd / 552 B bwd at SH degree 3.  SH coefficients are streamed with
// 128-bit read-only loads (ld.global.nc), outputs written with 64/128-bit stores where the layout allows.
#include "common.cuh"
#include "geometry.cuh"
#include "onesweep.cuh"
#include "sh.cuh"

#include <type_traits>

namespace b200gs {

namespace {

// The evaluation-order helpers xm / xa / xf, Proj, quat_to_rot, gaussian_cov3d and load_scale_quat are in geometry.cuh.

// unit view direction camera -> Gaussian and 1 / distance
__device__ __forceinline__ void view_dir(const float* p, const float* campos, float& dx, float& dy, float& dz, float& inv_len) {
    dx = xa(p[0], -campos[0]); dy = xa(p[1], -campos[1]); dz = xa(p[2], -campos[2]);
    inv_len = rsqrtf(xf(dz, dz, xf(dy, dy, xm(dx, dx))));
    dx = xm(dx, inv_len); dy = xm(dy, inv_len); dz = xm(dz, inv_len);
}

// The per-camera half: camera-space mean, Jacobian, cov2D (+ blur), determinants.  g.S3 (and Rm, s for the backward) are inputs.
template <bool GSPLAT, typename R>
__device__ __forceinline__ void project_view(const B200gsView& v, const float* p, Proj<R>& g) {
    const float* V = v.viewmatrix;
    const R p0 = p[0], p1 = p[1], p2 = p[2];
    g.tx = xa(xf(p2, R(V[8]), xf(p1, R(V[4]), xm(p0, R(V[0])))), R(V[12]));
    g.ty = xa(xf(p2, R(V[9]), xf(p1, R(V[5]), xm(p0, R(V[1])))), R(V[13]));
    g.tz = xa(xf(p2, R(V[10]), xf(p1, R(V[6]), xm(p0, R(V[2])))), R(V[14]));

    R tanx, tany;
    if (GSPLAT) {
        g.fx = v.fx; g.fy = v.fy;
        tanx = xm(R(0.5), R(v.width)) / R(v.fx);
        tany = xm(R(0.5), R(v.height)) / R(v.fy);
    } else {
        tanx = v.tanfovx; tany = v.tanfovy;
        g.fx = R(v.width) / xm(R(2), tanx);
        g.fy = R(v.height) / xm(R(2), tany);
    }
    const R limx = xm(R(1.3), tanx), limy = xm(R(1.3), tany);
    const R txtz = g.tx / g.tz, tytz = g.ty / g.tz;
    g.clx = (txtz < -limx) || (txtz > limx);
    g.cly = (tytz < -limy) || (tytz > limy);
    g.cxp = xm(fmin(limx, fmax(-limx, txtz)), g.tz);
    g.cyp = xm(fmin(limy, fmax(-limy, tytz)), g.tz);
    const R itz = R(1) / g.tz;
    const R j00 = xm(g.fx, itz), j02 = xm(xm(-xm(g.fx, g.cxp), itz), itz);
    const R j11 = xm(g.fy, itz), j12 = xm(xm(-xm(g.fy, g.cyp), itz), itz);
    // T = J * Rw ; Rw[j][i] = V[i*4+j]
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        g.T[i] = xf(j02, R(V[i * 4 + 2]), xm(j00, R(V[i * 4 + 0])));
        g.T[3 + i] = xf(j12, R(V[i * 4 + 2]), xm(j11, R(V[i * 4 + 1])));
    }
    // cov2D = T S3 T^T
    const R* S = g.S3;
    const R* T = g.T;
    const R u0 = xf(S[2], T[2], xf(S[1], T[1], xm(S[0], T[0])));
    const R u1 = xf(S[4], T[2], xf(S[3], T[1], xm(S[1], T[0])));
    const R u2 = xf(S[5], T[2], xf(S[4], T[1], xm(S[2], T[0])));
    const R w0 = xf(S[2], T[5], xf(S[1], T[4], xm(S[0], T[3])));
    const R w1 = xf(S[4], T[5], xf(S[3], T[4], xm(S[1], T[3])));
    const R w2 = xf(S[5], T[5], xf(S[4], T[4], xm(S[2], T[3])));
    g.a0 = xf(T[2], u2, xf(T[1], u1, xm(T[0], u0)));
    g.b = xf(T[5], u2, xf(T[4], u1, xm(T[3], u0)));
    g.c0 = xf(T[5], w2, xf(T[4], w1, xm(T[3], w0)));
    const R bb = xm(g.b, g.b);
    g.det0 = xf(g.a0, g.c0, -bb);
    g.a = xa(g.a0, R(v.eps2d));
    g.c = xa(g.c0, R(v.eps2d));
    g.det = xf(g.a, g.c, -bb);
    if (std::is_same<R, float>::value) {
        // The fp32 geometry (K8's) takes the determinants from forms without cancellation: a0 c0 - b^2 cancels completely
        // for a needle (cov2D of rank ~1), and K8 would differentiate a compensation and a conic other than the ones K1
        // rendered in fp64.  Cauchy-Binet: det0 = sum of the squared 2x2 minors of N = T M (cov2D = N N^T, M = Rm diag(s)),
        // and det = det0 + e (a0 + c0 + e) with e = eps2d.  Not used in fp64 (K1), whose bits stay those of the form above.
        R N[6];
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            N[k] = (T[0] * g.Rm[k] + T[1] * g.Rm[3 + k] + T[2] * g.Rm[6 + k]) * g.s[k];
            N[3 + k] = (T[3] * g.Rm[k] + T[4] * g.Rm[3 + k] + T[5] * g.Rm[6 + k]) * g.s[k];
        }
        const R m01 = N[0] * N[4] - N[1] * N[3], m02 = N[0] * N[5] - N[2] * N[3], m12 = N[1] * N[5] - N[2] * N[4];
        const R e = R(v.eps2d);
        g.det0 = m01 * m01 + m02 * m02 + m12 * m12;
        g.det = g.det0 + e * (g.a0 + g.c0 + e);
    }
}

// Optional fused-activation ("raw parameter") operands: the model's exp / normalize / sigmoid activations and the
// dc|rest concatenation (vanilla_gaussian.py:345-358, gaussian.py:250-254) folded into K1 / K8.
struct RawIO {
    const float* opac_in;    // [n] opacity logits
    const float* shs_rest;   // [n, sh_stride-1, 3]; the `shs` argument then points at shs_dc [n,1,3]
    float* opac_out;         // [n] opacity handed to the blend kernels (sigmoid, x compensation when anti_aliased; multi-view K1)
    float* v_opac_logit;     // [n]
    float* v_shs_rest;       // [n, sh_stride-1, 3]; `v_shs` then receives the dc gradient [n,1,3]
    int anti_aliased;
    // K8: cotangents come as [.,12] gradient rows (b200gs.h row layout), row row_offsets[i] for Gaussian i (NULL: row i), and
    // with accumulate != 0 the gradients are ADDED to the outputs (the sharded renderer's per-camera launches)
    const float* v_rows;
    const int32_t* row_offsets;
    int accumulate;
    float* v_mean2d;         // K8 (optional): [n, v_mean2d_cols] <- (dL/dmean2D.x, .y[, 0]) of every Gaussian, zeros for culled ones:
    int v_mean2d_cols;       // the `viewspace_points.grad` of the renderer contract, written here instead of by a fill + strided copy
};

template <bool GSPLAT>
__device__ __forceinline__ float near_of(const B200gsView& v) {
    return v.near_plane > 0.f ? v.near_plane : (GSPLAT ? 0.01f : 0.2f);
}

// K1's per-Gaussian prologue: mean p and camera-independent geometry g (gaussian_cov3d, with v's scale_modifier) of Gaussian i.
// A lane past the end (live == false) leaves p as it is and gets the geometry of a unit Gaussian.
template <bool RAW>
__device__ __forceinline__ void load_gaussian(const B200gsView& v, const float* __restrict__ means, const float* __restrict__ scales,
                                              const float* __restrict__ quats, int64_t i, bool live, float* p, Proj<double>& g) {
    double sc[3] = {1.0, 1.0, 1.0}, q[4] = {1.0, 0.0, 0.0, 0.0}, inv_qn;
    if (live) {
        p[0] = __ldg(means + 3 * i); p[1] = __ldg(means + 3 * i + 1); p[2] = __ldg(means + 3 * i + 2);
        load_scale_quat<RAW, double>(scales, quats, i, sc, q, &inv_qn);
    }
    gaussian_cov3d<double>(sc, q, v.scale_modifier, g);
}

// Destination of one view's projection outputs (element index `o` of every array).
struct ProjOut {
    float2* xy; float* depth; int32_t* radii; float* conic; float* comp; int32_t* tiles;
};

// What one (view, Gaussian) projection produces (all zero when the Gaussian is culled)
struct ProjVals {
    float px, py, depth, cA, cB, cC, comp, opac;
    int32_t radius, ntiles;
};

// Projection of Gaussian i (mean p, gaussian_cov3d already in g) into view v -> pv; returns the visibility.  cov3d_out (optional)
// receives cov3D at element o.
template <bool GSPLAT, bool RAW>
__device__ __forceinline__ bool project_one_view(const B200gsView& v, const RawIO& raw, int64_t i, int64_t o, const float* p, Proj<double>& g,
                                                 float* cov3d_out, ProjVals& pv) {
    typedef double R;
    project_view<GSPLAT, R>(v, p, g);

    const float near = near_of<GSPLAT>(v);
    bool vis = GSPLAT ? (float(g.tz) >= near) : (float(g.tz) > near);
    if (!GSPLAT) vis = vis && (g.det != R(0));

    R pxd, pyd;
    if (GSPLAT) {
        const R iz = R(1) / xa(g.tz, R(1e-6));
        const R zn = xm(g.tz, iz);
        pxd = xf(zn, R(v.cx), xm(xm(g.tx, iz), R(v.fx)));
        pyd = xf(zn, R(v.cy), xm(xm(g.ty, iz), R(v.fy)));
    } else {
        const float* P = v.projmatrix;
        const R p0 = p[0], p1 = p[1], p2 = p[2];
        const R hx = xa(xf(p2, R(P[8]), xf(p1, R(P[4]), xm(p0, R(P[0])))), R(P[12]));
        const R hy = xa(xf(p2, R(P[9]), xf(p1, R(P[5]), xm(p0, R(P[1])))), R(P[13]));
        const R hw = xa(xf(p2, R(P[11]), xf(p1, R(P[7]), xm(p0, R(P[3])))), R(P[15]));
        const R iw = R(1) / xa(hw, R(0.0000001));
        pxd = xm(xf(xf(hx, iw, R(1)), R(v.width), R(-1)), R(0.5));
        pyd = xm(xf(xf(hy, iw, R(1)), R(v.height), R(-1)), R(0.5));
    }
    const float px = float(pxd), py = float(pyd);
    const R inv_det = R(1) / g.det;
    const R mid = xm(R(0.5), xa(g.a, g.c));
    const R sq = sqrt(fmax(R(0.1), xf(mid, mid, -g.det)));
    const R lam = fmax(xa(mid, sq), xa(mid, -sq));
    const float radius = float(ceil(xm(R(3), sqrt(lam))));
    const int grid_x = div_up(v.width, TILE), grid_y = div_up(v.height, TILE);
    int x0, y0, x1, y1;
    tile_rect<GSPLAT>(px, py, radius, grid_x, grid_y, x0, y0, x1, y1);
    const int ntiles = (x1 - x0) * (y1 - y0);
    vis = vis && (ntiles > 0) && (radius > 0.f);  // NaN radius compares false

    pv.px = pv.py = pv.depth = pv.cA = pv.cB = pv.cC = pv.comp = pv.opac = 0.f;
    pv.radius = pv.ntiles = 0;
    if (vis) {
        pv.px = px; pv.py = py;
        pv.depth = float(g.tz);
        pv.radius = (int32_t)radius;
        pv.cA = float(xm(g.c, inv_det));
        pv.cB = float(xm(-g.b, inv_det));
        pv.cC = float(xm(g.a, inv_det));
        pv.ntiles = ntiles;
        pv.comp = GSPLAT ? float(sqrt(fmax(xm(g.det0, inv_det), R(0)))) : 1.0f;
        if (RAW) {
            const float op = __frcp_rn(xa(1.0f, __expf(-__ldg(raw.opac_in + i))));
            pv.opac = (GSPLAT && raw.anti_aliased) ? xm(op, pv.comp) : op;
        }
    }
    if (cov3d_out) {
#pragma unroll
        for (int k = 0; k < 6; ++k) cov3d_out[6 * o + k] = vis ? float(g.S3[k]) : 0.f;
    }
    return vis;
}

// separate-array outputs of one projection at element o
template <bool RAW>
__device__ __forceinline__ void store_soa(const ProjOut& out, float* opac_out, int64_t o, const ProjVals& pv) {
    out.xy[o] = make_float2(pv.px, pv.py);
    out.depth[o] = pv.depth;
    out.radii[o] = pv.radius;
    out.conic[3 * o + 0] = pv.cA; out.conic[3 * o + 1] = pv.cB; out.conic[3 * o + 2] = pv.cC;
    if (out.tiles) out.tiles[o] = pv.ntiles;
    if (out.comp) out.comp[o] = pv.radius > 0 ? pv.comp : 0.f;
    if (RAW) opac_out[o] = pv.opac;
}

// max(SH colour + 0.5, 0) of a visible Gaussian seen from v.campos; bit c of *cl set where channel c was clamped
template <int MC>
__device__ __forceinline__ void sh_color_one(const B200gsView& v, const float* p, const float* sh, float& r, float& gc, float& bc, uint8_t& cl) {
    const int deg = v.sh_degree;
    const int ncoef = (deg + 1) * (deg + 1);
    float dx, dy, dz, inv_len;
    view_dir(p, v.campos, dx, dy, dz, inv_len);
    float bs[MC];
    sh_basis<MC>(deg, dx, dy, dz, bs);
    r = xm(bs[0], sh[0]); gc = xm(bs[0], sh[1]); bc = xm(bs[0], sh[2]);
#pragma unroll
    for (int k = 1; k < MC; ++k) {
        if (k < ncoef) {
            r = xf(bs[k], sh[3 * k + 0], r);
            gc = xf(bs[k], sh[3 * k + 1], gc);
            bc = xf(bs[k], sh[3 * k + 2], bc);
        }
    }
    r = xa(r, 0.5f); gc = xa(gc, 0.5f); bc = xa(bc, 0.5f);
    cl = 0;
    if (r < 0.f) { r = 0.f; cl |= 1; }
    if (gc < 0.f) { gc = 0.f; cl |= 2; }
    if (bc < 0.f) { bc = 0.f; cl |= 4; }
}

// RAW: fused activations, and instead of the separate arrays ONE [n,12] row per Gaussian in rows_out (xy 0..1, depth 2, conic 3..5,
// compensation 6, blend opacity 7, rgb 8..10, radius bits 11) — three 128-bit stores; the binning and the blend kernels read the rows
// in place (one 48-byte record per splat instead of four separate sectors).  radii_out / clamped_out (what K8 needs) are still written.
template <bool GSPLAT, bool RAW, int MC>
__global__ void __launch_bounds__(256, 3) project_fwd_kernel(const __grid_constant__ B200gsView v, const RawIO raw, int64_t n,
                                                          const float* __restrict__ means, const float* __restrict__ scales,
                                                          const float* __restrict__ quats, const float* __restrict__ shs,
                                                          float2* __restrict__ xy_out, float* __restrict__ depth_out,
                                                          int32_t* __restrict__ radii_out, float* __restrict__ conic_out,
                                                          float* __restrict__ comp_out, int32_t* __restrict__ tiles_out,
                                                          float* __restrict__ cov3d_out, float* __restrict__ rgb_out,
                                                          uint8_t* __restrict__ clamped_out, float* __restrict__ rows_out) {
    const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float p[3];
    Proj<double> g;
    load_gaussian<RAW>(v, means, scales, quats, i, true, p, g);
    const ProjOut out{xy_out, depth_out, radii_out, conic_out, comp_out, tiles_out};
    ProjVals pv;
    const bool vis = project_one_view<GSPLAT, RAW>(v, raw, i, i, p, g, cov3d_out, pv);
    if (!RAW) store_soa<false>(out, nullptr, i, pv);
    float r = 0.f, gc = 0.f, bc = 0.f;
    uint8_t cl = 0;
    if (shs != nullptr) {
        if (vis) {
            const int deg = v.sh_degree;
            float sh[MC * 3];
            load_sh_any<RAW, MC>(shs, raw.shs_rest, i, v.sh_stride, (deg + 1) * (deg + 1), sh);
            sh_color_one<MC>(v, p, sh, r, gc, bc, cl);
        }
        if (!RAW) { rgb_out[3 * i + 0] = r; rgb_out[3 * i + 1] = gc; rgb_out[3 * i + 2] = bc; }
        clamped_out[i] = cl;
    }
    if (RAW) {
        float4* row = reinterpret_cast<float4*>(rows_out + i * B200GS_ROW_FLOATS);
        radii_out[i] = pv.radius;
        if (tiles_out) tiles_out[i] = pv.ntiles;
        row[0] = make_float4(pv.px, pv.py, pv.depth, pv.cA);             // zeros when culled (the mean2D columns are handed out)
        if (vis) row[1] = make_float4(pv.cB, pv.cC, pv.comp, pv.opac);
        row[2] = make_float4(r, gc, bc, __int_as_float(pv.radius));      // radius 0 = culled: all the kernels look at of such a row
    }
}

// The sharded renderer projects ONE shard into the W cameras of a step: one launch, the parameters (and the SH block, if any view
// sees the Gaussian) are read once per Gaussian instead of once per camera.  gsplat constants, raw parameters.  View j's outputs
// live at elements [j*n, (j+1)*n) of camera-major arrays.
struct ViewPack {
    B200gsView v[B200GS_MAX_VIEWS];
};

// SH colour of Gaussian i in each of the nviews cameras: the SH block is read once, if any camera sees the Gaussian (bit j of
// vismask), and store(j, r, g, b, clamped) receives camera j's colour (zeros for a camera that does not see it).
template <int MC, typename Store>
__device__ __forceinline__ void color_views(const ViewPack& vp, int nviews, const float* __restrict__ shs_dc, const float* __restrict__ shs_rest,
                                            int64_t i, const float* p, unsigned vismask, Store store) {
    float sh[MC * 3];
    if (vismask) {
        const int deg = vp.v[0].sh_degree;
        load_sh_any<true, MC>(shs_dc, shs_rest, i, vp.v[0].sh_stride, (deg + 1) * (deg + 1), sh);
    }
#pragma unroll 1
    for (int j = 0; j < nviews; ++j) {
        uint8_t cl = 0;
        float r = 0.f, gc = 0.f, bc = 0.f;
        if ((vismask >> j) & 1u) sh_color_one<MC>(vp.v[j], p, sh, r, gc, bc, cl);
        store(j, r, gc, bc, cl);
    }
}

template <int MC>
__global__ void __launch_bounds__(256) project_fwd_multi_kernel(const __grid_constant__ ViewPack vp, int nviews, const RawIO raw, int64_t n,
                                                                const float* __restrict__ means, const float* __restrict__ scales,
                                                                const float* __restrict__ quats, const float* __restrict__ shs_dc,
                                                                float2* __restrict__ xy_out, float* __restrict__ depth_out,
                                                                int32_t* __restrict__ radii_out, float* __restrict__ conic_out,
                                                                float* __restrict__ rgb_out, uint8_t* __restrict__ clamped_out) {
    const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float p[3];
    Proj<double> g3;
    load_gaussian<true>(vp.v[0], means, scales, quats, i, true, p, g3);      // once per Gaussian; project_one_view per camera
    const ProjOut out{xy_out, depth_out, radii_out, conic_out, nullptr, nullptr};
    unsigned vismask = 0;
#pragma unroll 1
    for (int j = 0; j < nviews; ++j) {
        ProjVals pv;
        if (project_one_view<true, true>(vp.v[j], raw, i, int64_t(j) * n + i, p, g3, nullptr, pv)) vismask |= 1u << j;
        store_soa<true>(out, raw.opac_out, int64_t(j) * n + i, pv);
    }
    color_views<MC>(vp, nviews, shs_dc, raw.shs_rest, i, p, vismask, [&](int j, float r, float gc, float bc, uint8_t cl) {
        const int64_t o = int64_t(j) * n + i;
        rgb_out[3 * o + 0] = r; rgb_out[3 * o + 1] = gc; rgb_out[3 * o + 2] = bc;
        clamped_out[o] = cl;
    });
}

// K1 of a shard for all W cameras FUSED with the exchange's packing: the visible splats of camera j leave this kernel as [.,12]
// rows stored straight into block `dst.p[j]` (capacity `cap` rows) of the rank that owns camera j — a peer GPU's receive buffer
// mapped over NVLink, or a local send buffer — in Gaussian-index order (what keeps the sharded image bit-identical to the
// single-GPU one).  No intermediate arrays, no separate scan / pack / pad kernels: blocks take tickets, every warp compacts its
// visible lanes per camera into a shared-memory row tile (ballot), warp j runs camera j's chained scan over the blocks
// (decoupled look-back, one value per block and camera), and the block copies its rows out as contiguous runs.  Rows beyond
// `cap` are dropped and show up in d_count[j] (total visible of camera j; the caller compares with cap and redoes the step with
// the exact exchange).  What the backward needs stays local: radii, clamped, row_index (block-relative row j*cap + k, or -1
// when dropped) at [j*n + i], and the mean2D (the per-camera viewspace points the renderer hands out).
struct PackDst {
    float* p[B200GS_MAX_VIEWS];
};
constexpr int PACK_THREADS = 256;
constexpr int PACK_WARPS = PACK_THREADS / 32;

template <int MC>
__global__ void __launch_bounds__(PACK_THREADS, (MC <= 16 ? 3 : 2)) project_pack_multi_kernel(const __grid_constant__ ViewPack vp, int nviews, const RawIO raw, int64_t n,
                                                                        const float* __restrict__ means, const float* __restrict__ scales,
                                                                        const float* __restrict__ quats, const float* __restrict__ shs_dc,
                                                                        float2* __restrict__ xy_out, int32_t* __restrict__ radii_out,
                                                                        uint8_t* __restrict__ clamped_out, int32_t* __restrict__ row_index_out,
                                                                        const PackDst dst, int64_t cap, uint32_t* __restrict__ ticket,
                                                                        uint32_t* __restrict__ scan_state /*[nviews][gridDim.x]*/,
                                                                        int64_t* __restrict__ d_count) {
    extern __shared__ float4 s_rows[];                           // [nviews][PACK_THREADS slots][3]: slot = warp * 32 + rank among the warp's visible lanes
    __shared__ int s_cnt[B200GS_MAX_VIEWS][PACK_WARPS];          // visible lanes per (camera, warp)
    __shared__ uint32_t s_pre[B200GS_MAX_VIEWS][PACK_WARPS];     // global row (within the block of `cap`) of the warp's first row
    __shared__ int s_tile;
    const int tid = threadIdx.x;
    const unsigned lane = tid & 31u, w = tid >> 5;
    if (tid == 0) s_tile = (int)atomicAdd(ticket, 1u);
    __syncthreads();
    const int t = s_tile;
    const int64_t i = int64_t(t) * PACK_THREADS + tid;
    const bool live = i < n;
    float p[3] = {0.f, 0.f, 0.f};
    Proj<double> g3;
    load_gaussian<true>(vp.v[0], means, scales, quats, i, live, p, g3);      // once per Gaussian; project_one_view per camera
    unsigned vismask = 0;
    unsigned long long kpos = 0;            // 8 bits per camera: this lane's rank among the warp's visible lanes
#pragma unroll 1
    for (int j = 0; j < nviews; ++j) {
        ProjVals pv;
        bool vis = false;
        if (live) vis = project_one_view<true, true>(vp.v[j], raw, i, 0, p, g3, nullptr, pv);
        const unsigned b = __ballot_sync(0xffffffffu, vis);
        const int k = __popc(b & ((1u << lane) - 1u));
        if (lane == 0) s_cnt[j][w] = __popc(b);
        if (live) {
            const int64_t o = int64_t(j) * n + i;
            xy_out[o] = make_float2(pv.px, pv.py);
            radii_out[o] = pv.radius;
        }
        if (vis) {
            vismask |= 1u << j;
            kpos |= (unsigned long long)k << (8 * j);
            float4* row = s_rows + (size_t(j) * PACK_THREADS + w * 32 + k) * 3;
            row[0] = make_float4(pv.px, pv.py, pv.depth, pv.cA);
            row[1] = make_float4(pv.cB, pv.cC, pv.comp, pv.opac);
            row[2].w = __int_as_float(pv.radius);
        }
    }
    color_views<MC>(vp, nviews, shs_dc, raw.shs_rest, i, p, vismask, [&](int j, float r, float gc, float bc, uint8_t cl) {
        if ((vismask >> j) & 1u) {
            float* row2 = reinterpret_cast<float*>(s_rows + (size_t(j) * PACK_THREADS + w * 32 + (int)((kpos >> (8 * j)) & 255ull)) * 3 + 2);
            row2[0] = r; row2[1] = gc; row2[2] = bc;
        }
        if (live) clamped_out[int64_t(j) * n + i] = cl;
    });
    __syncthreads();
    // warp j: camera j's block total -> chained scan over the blocks -> first row of every warp's run
    if ((int)w < nviews) {
        const int j = (int)w;
        const int c = (lane < PACK_WARPS) ? s_cnt[j][lane] : 0;
        int inc = c;
#pragma unroll
        for (int o = 1; o < PACK_WARPS; o <<= 1) {
            const int v = __shfl_up_sync(0xffffffffu, inc, o);
            if ((int)lane >= o) inc += v;
        }
        const int total = __shfl_sync(0xffffffffu, inc, PACK_WARPS - 1);
        const uint32_t base = sweep::chained_exclusive(scan_state + size_t(j) * gridDim.x, t, (uint32_t)total);
        if (lane < PACK_WARPS) s_pre[j][lane] = base + (uint32_t)(inc - c);
        if (lane == 0 && t == (int)gridDim.x - 1) d_count[j] = (int64_t)base + total;
    }
    __syncthreads();
#pragma unroll 1
    for (int j = 0; j < nviews; ++j) {
        if (live) {
            int32_t ri = -1;
            if ((vismask >> j) & 1u) {
                const int64_t pos = (int64_t)s_pre[j][w] + (int64_t)((kpos >> (8 * j)) & 255ull);
                ri = pos < cap ? (int32_t)(int64_t(j) * cap + pos) : -1;
            }
            row_index_out[int64_t(j) * n + i] = ri;
        }
        // copy-out: 8 warps x 32 slots x 3 float4 per camera; consecutive threads -> consecutive 16-byte pieces of a warp's run
        float4* out = reinterpret_cast<float4*>(dst.p[j]);
        const float4* src = s_rows + size_t(j) * PACK_THREADS * 3;
#pragma unroll
        for (int it = 0; it < 3; ++it) {
            const int item = it * PACK_THREADS + tid;       // = (warp segment * 32 + r) * 3 + part
            const int seg = item / 96, r = (item - seg * 96) / 3, part = item - seg * 96 - r * 3;
            if (r < s_cnt[j][seg]) {
                const int64_t pos = (int64_t)s_pre[j][seg] + r;
                if (pos < cap) out[pos * 3 + part] = src[(seg * 32 + r) * 3 + part];
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------------------------
// backward
// ------------------------------------------------------------------------------------------------------------------
constexpr int BWD_THREADS = 128;

// Cotangents of one view's projection outputs for one Gaussian
struct ProjCot {
    float vA, vB, vC;      // dL/dconic
    float2 vxy;            // dL/dmean2D (vanilla: NDC-scaled units)
    float vdepth;          // dL/ddepth (gsplat)
    float vcomp;           // dL/dcompensation (gsplat), incl. the part that reaches it through the blend opacity
};

// Adds view v's contribution to dL/dmean (dm), dL/dM-chain outputs: dL/dscale (activated scale, before the exp chain) and dL/dq
// (unit quaternion, before the normalisation chain).  g: gaussian_cov3d<float>(sc, q) and project_view<GSPLAT, float>(v, p) of the
// Gaussian with mean p, scales sc and unit quaternion q.
template <bool GSPLAT>
__device__ __forceinline__ void geometry_backward(const B200gsView& v, const float* p, const float* q, const Proj<float>& g, const ProjCot& c,
                                                  float* dm, float* dscale, float4& dq) {
    const float* V = v.viewmatrix;
    float dtx = 0.f, dty = 0.f, dtz = 0.f;  // dL/dt (camera)
    // ---- conic (+ compensation) -> blurred cov2D (a, b, c) ----------------------------------------------------
    const float inv_det = 1.0f / g.det;
    const float A = g.c * inv_det, B = -g.b * inv_det, C = g.a * inv_det;
    // X = -Q G Q, Q = [[A,B],[B,C]], G = [[vA, vB/2],[vB/2, vC]]
    const float hB = 0.5f * c.vB;
    const float m00 = A * c.vA + B * hB, m01 = A * hB + B * c.vC;
    const float m10 = B * c.vA + C * hB, m11 = B * hB + C * c.vC;
    float da = -(m00 * A + m01 * B);
    float db = -2.0f * (m00 * B + m01 * C);
    float dc = -(m10 * B + m11 * C);
    if (GSPLAT) {
        const float vc = c.vcomp;
        if (g.det0 > 0.f && vc != 0.f) {
            // d comp / d(a, b, c) of comp = sqrt(det0 / det) is 0.5 comp (c0 / det0 - c / det, -2 b (1 / det0 - 1 / det), a0 / det0 - a / det).
            // For a splat much larger than eps2d both quotients of each difference agree to ~eps2d / lambda, and fp32 subtraction
            // left none of their digits (measured: 1e-2 relative errors on the scale gradients of large off-screen splats).  With
            // det = det0 + e (a0 + c0 + e) and b^2 = a0 c0 - det0 the differences are e (c0^2 + c0 e + b^2) / (det0 det),
            // e (a0 + c0 + e) / (det0 det) and e (a0^2 + a0 e + b^2) / (det0 det): sums of positive terms, no cancellation.
            const float comp = sqrtf(g.det0 * inv_det);
            const float e = v.eps2d, bb = g.b * g.b;
            const float k = vc * 0.5f * comp * e * inv_det / g.det0;
            da += k * (g.c0 * (g.c0 + e) + bb);
            dc += k * (g.a0 * (g.a0 + e) + bb);
            db += -2.0f * g.b * k * (g.a0 + g.c0 + e);
        }
    }
    // symmetric gradient wrt the 2x2 cov: [[da, db/2],[db/2, dc]]
    const float g00 = da, g01 = 0.5f * db, g11 = dc;
    const float* T = g.T;
    // dL/dSigma3 = T^T Gc T  (symmetric 3x3)
    float dS[9];
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int cidx = 0; cidx < 3; ++cidx)
            dS[r * 3 + cidx] = T[r] * (g00 * T[cidx] + g01 * T[3 + cidx]) + T[3 + r] * (g01 * T[cidx] + g11 * T[3 + cidx]);
    // dL/dT = 2 Gc T Sigma3 (2x3)
    const float* S = g.S3;
    const float Sf[9] = {S[0], S[1], S[2], S[1], S[3], S[4], S[2], S[4], S[5]};
    float TS0[3], TS1[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        TS0[k] = T[0] * Sf[k] + T[1] * Sf[3 + k] + T[2] * Sf[6 + k];
        TS1[k] = T[3] * Sf[k] + T[4] * Sf[3 + k] + T[5] * Sf[6 + k];
    }
    float dT0[3], dT1[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        dT0[k] = 2.0f * (g00 * TS0[k] + g01 * TS1[k]);
        dT1[k] = 2.0f * (g01 * TS0[k] + g11 * TS1[k]);
    }
    // T = J Rw -> dL/dJ = dL/dT Rw^T ; Rw[j][i] = V[i*4+j]
    const float dJ00 = dT0[0] * V[0] + dT0[1] * V[4] + dT0[2] * V[8];
    const float dJ02 = dT0[0] * V[2] + dT0[1] * V[6] + dT0[2] * V[10];
    const float dJ11 = dT1[0] * V[1] + dT1[1] * V[5] + dT1[2] * V[9];
    const float dJ12 = dT1[0] * V[2] + dT1[1] * V[6] + dT1[2] * V[10];
    const float itz = 1.0f / g.tz, itz2 = itz * itz, itz3 = itz2 * itz;
    const float dcx = -g.fx * itz2 * dJ02;  // dL/d(tx')
    const float dcy = -g.fy * itz2 * dJ12;
    dtz += -g.fx * itz2 * dJ00 - g.fy * itz2 * dJ11 + 2.0f * g.fx * g.cxp * itz3 * dJ02 + 2.0f * g.fy * g.cyp * itz3 * dJ12;
    if (!g.clx) dtx += dcx; else if (GSPLAT) dtz += dcx * g.cxp * itz;  // dgr drops the clamped branch's z-dependence
    if (!g.cly) dty += dcy; else if (GSPLAT) dtz += dcy * g.cyp * itz;

    // ---- mean2D / depth --------------------------------------------------------------------------------------
    if (GSPLAT) {
        const float iz = 1.0f / (g.tz + 1e-6f);
        dtx += v.fx * iz * c.vxy.x;
        dty += v.fy * iz * c.vxy.y;
        dtz += (-v.fx * g.tx * iz * iz + v.cx * 1e-6f * iz * iz) * c.vxy.x + (-v.fy * g.ty * iz * iz + v.cy * 1e-6f * iz * iz) * c.vxy.y;
        dtz += c.vdepth;
    } else {
        // v_xy is dL/d(ndc) (pixel gradient x 0.5 W/H), straight through the 4x4 full projection
        const float* P = v.projmatrix;
        const float hw = p[0] * P[3] + p[1] * P[7] + p[2] * P[11] + P[15];
        const float mw = 1.0f / (hw + 0.0000001f);
        const float mul1 = (p[0] * P[0] + p[1] * P[4] + p[2] * P[8] + P[12]) * mw * mw;
        const float mul2 = (p[0] * P[1] + p[1] * P[5] + p[2] * P[9] + P[13]) * mw * mw;
        dm[0] += (P[0] * mw - P[3] * mul1) * c.vxy.x + (P[1] * mw - P[3] * mul2) * c.vxy.y;
        dm[1] += (P[4] * mw - P[7] * mul1) * c.vxy.x + (P[5] * mw - P[7] * mul2) * c.vxy.y;
        dm[2] += (P[8] * mw - P[11] * mul1) * c.vxy.x + (P[9] * mw - P[11] * mul2) * c.vxy.y;
    }
    // t = p * V[:3,:3] + V[3,:3]  ->  dL/dp_i = sum_j V[i][j] dt_j
    dm[0] += V[0] * dtx + V[1] * dty + V[2] * dtz;
    dm[1] += V[4] * dtx + V[5] * dty + V[6] * dtz;
    dm[2] += V[8] * dtx + V[9] * dty + V[10] * dtz;

    // ---- Sigma3 = M M^T, M = R diag(s) ------------------------------------------------------------------------
    float M[9], dM[9];
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int k = 0; k < 3; ++k) M[r * 3 + k] = g.Rm[r * 3 + k] * g.s[k];
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int k = 0; k < 3; ++k)
            dM[r * 3 + k] = 2.0f * (dS[r * 3 + 0] * M[0 + k] + dS[r * 3 + 1] * M[3 + k] + dS[r * 3 + 2] * M[6 + k]);
    float dR[9];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        dscale[k] += v.scale_modifier * (g.Rm[k] * dM[k] + g.Rm[3 + k] * dM[3 + k] + g.Rm[6 + k] * dM[6 + k]);
#pragma unroll
        for (int r = 0; r < 3; ++r) dR[r * 3 + k] = dM[r * 3 + k] * g.s[k];
    }
    const float r = q[0], x = q[1], y = q[2], z = q[3];
    dq.x += 2.f * (-z * dR[1] + y * dR[2] + z * dR[3] - x * dR[5] - y * dR[6] + x * dR[7]);
    dq.y += 2.f * (y * dR[1] + z * dR[2] + y * dR[3] - 2.f * x * dR[4] - r * dR[5] + z * dR[6] + r * dR[7] - 2.f * x * dR[8]);
    dq.z += 2.f * (-2.f * y * dR[0] + x * dR[1] + r * dR[2] + x * dR[3] + z * dR[5] - r * dR[6] + z * dR[7] - 2.f * y * dR[8]);
    dq.w += 2.f * (-2.f * z * dR[0] - r * dR[1] + x * dR[2] + r * dR[3] - 2.f * z * dR[4] + y * dR[5] + x * dR[6] + y * dR[7]);
}

// Opacity logit x: o = sigmoid(x) and 1 - o, taken as o1 = sigmoid(-x) (1.0f - o cancels at large logits: a 1e-2 relative error of
// the logit gradient at logit 12)
__device__ __forceinline__ void logit_sigmoid(float x, float& o, float& o1) {
    o = 1.0f / (1.0f + expf(-x));
    o1 = 1.0f / (1.0f + expf(x));
}

// The blend opacity is sigmoid(logit), times the compensation when anti-aliased: splits its cotangent vo, adding the compensation's
// share to c.vcomp and returning the sigmoid's (dL/dlogit is that times o o1).
template <bool GSPLAT>
__device__ __forceinline__ float sigmoid_cotangent(float vo, float o, int anti_aliased, const Proj<float>& g, ProjCot& c) {
    if (!(GSPLAT && anti_aliased)) return vo;
    c.vcomp += vo * o;
    return vo * sqrtf(fmaxf(g.det0 / g.det, 0.f));
}

// Through the fused activations of the raw parameters: scale = exp(log scale) (d exp(x) = exp(x)) and unit quaternion
// q = raw / |raw| (inv_qn = 1 / |raw|).
__device__ __forceinline__ void raw_param_backward(const float* sc, const float* q, float inv_qn, float* dscale, float4& dq) {
#pragma unroll
    for (int k = 0; k < 3; ++k) dscale[k] *= sc[k];
    const float dot = dq.x * q[0] + dq.y * q[1] + dq.z * q[2] + dq.w * q[3];
    dq.x = (dq.x - q[0] * dot) * inv_qn; dq.y = (dq.y - q[1] * dot) * inv_qn;
    dq.z = (dq.z - q[2] * dot) * inv_qn; dq.w = (dq.w - q[3] * dot) * inv_qn;
}

template <bool GSPLAT, bool RAW, int MC>
__global__ void __launch_bounds__(BWD_THREADS, (MC <= 16 ? (GSPLAT ? 7 : 6) : 3)) project_bwd_kernel(const __grid_constant__ B200gsView v, const RawIO raw, int64_t n,
                                                          const float* __restrict__ means, const float* __restrict__ scales,
                                                          const float* __restrict__ quats, const float* __restrict__ shs,
                                                          const int32_t* __restrict__ radii, const uint8_t* __restrict__ clamped,
                                                          const float2* __restrict__ v_xy, const float* __restrict__ v_depth,
                                                          const float* __restrict__ v_conic, const float* __restrict__ v_comp,
                                                          const float* __restrict__ v_rgb, float* __restrict__ v_means,
                                                          float* __restrict__ v_scales, float4* __restrict__ v_quats,
                                                          float* __restrict__ v_shs) {
    __shared__ float s_rows[BWD_THREADS / 32][32 * (MC * 3 + 1)];
    const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    const unsigned lane = threadIdx.x & 31u;
    const int warp = threadIdx.x >> 5;
    const bool in_range = i < n;
    const bool ACC = RAW && (raw.accumulate != 0);
    // RAW: the cotangents come as gradient rows.  A negative row index = the entry did not fit its fixed-size block (the caller
    // redoes such a step): treated as culled
    const int64_t ri = (RAW && in_range) ? (raw.row_offsets ? int64_t(raw.row_offsets[i]) : i) : 0;   // NULL offsets: row i
    const bool vis = in_range && (radii[i] > 0) && !(RAW && ri < 0);
    const int stride3 = v.sh_stride * 3;
    float p[3] = {0.f, 0.f, 0.f};
    if (vis) { p[0] = __ldg(means + 3 * i); p[1] = __ldg(means + 3 * i + 1); p[2] = __ldg(means + 3 * i + 2); }
    const float* vrow = (RAW && vis) ? raw.v_rows + ri * B200GS_ROW_FLOATS : nullptr;

    float dm[3] = {0.f, 0.f, 0.f};  // dL/dmean (world)

    // ---- SH colour -------------------------------------------------------------------------------------------
    if (v_shs != nullptr) {
        const int deg = v.sh_degree;
        const int ncoef = (deg + 1) * (deg + 1);
        float gr = 0.f, gg = 0.f, gb = 0.f, dx = 0.f, dy = 0.f, dz = 1.f, inv_len = 0.f;
        float bs[MC];
#pragma unroll
        for (int k = 0; k < MC; ++k) bs[k] = 0.f;
        if (vis) {
            const uint8_t cl = clamped[i];
            const float* crgb = RAW ? vrow + B200GS_ROW_RGB : v_rgb + 3 * i;
            gr = (cl & 1) ? 0.f : __ldg(crgb + 0);
            gg = (cl & 2) ? 0.f : __ldg(crgb + 1);
            gb = (cl & 4) ? 0.f : __ldg(crgb + 2);
            view_dir(p, v.campos, dx, dy, dz, inv_len);
            sh_basis<MC>(deg, dx, dy, dz, bs);
        }
        if (vis && !GSPLAT && deg > 0) {
            // view direction -> mean (dgr back-propagates it; gsplat renderers detach the direction)
            // w_k = <sh_k, v_rgb> first (the 48 coefficients are consumed as they arrive: 16 live values instead of 48), then the basis
            // derivatives
            const float* c0 = RAW ? raw.shs_rest + i * int64_t(v.sh_stride - 1) * 3 - 3 : shs + i * int64_t(v.sh_stride) * 3;   // coefficient k at c0 + 3 k (k >= 1)
            float w[MC];
#pragma unroll
            for (int k = 1; k < MC; ++k) w[k] = (k < ncoef) ? __ldg(c0 + 3 * k) * gr + __ldg(c0 + 3 * k + 1) * gg + __ldg(c0 + 3 * k + 2) * gb : 0.f;
            const float3 d = view_dir_grad<MC>(deg, dx, dy, dz, inv_len, w);
            dm[0] += d.x; dm[1] += d.y; dm[2] += d.z;
        }
        // SH-gradient row of this Gaussian (coefficient k, channel c: basis_k * v_rgb_c; zeros when culled).  RAW: the dc coefficient
        // goes to v_shs, the rest to the row of v_shs_rest.
        const int rw = RAW ? stride3 - 3 : stride3;          // floats per output row
        float* dst = RAW ? raw.v_shs_rest : v_shs;
        if (RAW && in_range) {
            float o0 = bs[0] * gr, o1 = bs[0] * gg, o2 = bs[0] * gb;
            if (ACC) { o0 += v_shs[3 * i]; o1 += v_shs[3 * i + 1]; o2 += v_shs[3 * i + 2]; }
            v_shs[3 * i] = o0; v_shs[3 * i + 1] = o1; v_shs[3 * i + 2] = o2;
        }
        if (rw <= MC * 3) {
            // straight into the warp's staging rows (48 values would otherwise sit in registers until the store: 96 registers,
            // 5 blocks per SM), then out coalesced
            float* row = s_rows[warp] + lane * (rw | 1);
#pragma unroll
            for (int k = RAW ? 1 : 0; k < MC; ++k) {
                const int c = RAW ? 3 * k - 3 : 3 * k;
                if (c < rw) {
                    const float bk = (k < ncoef) ? bs[k] : 0.f;
                    row[c] = bk * gr; row[c + 1] = bk * gg; row[c + 2] = bk * gb;
                }
            }
            flush_sh_rows(s_rows[warp], rw, i, n, lane, dst, ACC);
        } else if (in_range) {   // wider coefficient storage than the kernel evaluates: plain per-thread rows (ACC: add the evaluated ones)
            float* row = dst + i * int64_t(rw);
#pragma unroll
            for (int k = RAW ? 1 : 0; k < MC; ++k) {
                const int c = RAW ? 3 * k - 3 : 3 * k;
                const float bk = (k < ncoef) ? bs[k] : 0.f;
                if (!ACC) {
                    row[c] = bk * gr; row[c + 1] = bk * gg; row[c + 2] = bk * gb;
                } else if (k < ncoef) {
                    row[c] += bk * gr; row[c + 1] += bk * gg; row[c + 2] += bk * gb;
                }
            }
            if (!ACC)
                for (int c = MC * 3 - (RAW ? 3 : 0); c < rw; ++c) row[c] = 0.f;
        }
    }
    if (!in_range) return;
    if (RAW && raw.v_mean2d != nullptr) {
        float* m2 = raw.v_mean2d + i * raw.v_mean2d_cols;
        m2[0] = vis ? __ldg(vrow) : 0.f;
        m2[1] = vis ? __ldg(vrow + 1) : 0.f;
        if (raw.v_mean2d_cols > 2) m2[2] = 0.f;
    }
    if (!vis) {
        if (!ACC) {
            v_means[3 * i] = 0.f; v_means[3 * i + 1] = 0.f; v_means[3 * i + 2] = 0.f;
            v_scales[3 * i] = 0.f; v_scales[3 * i + 1] = 0.f; v_scales[3 * i + 2] = 0.f;
            v_quats[i] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (RAW) raw.v_opac_logit[i] = 0.f;
        }
        return;
    }
    float sc[3], q[4], inv_qn;
    load_scale_quat<RAW, float>(scales, quats, i, sc, q, &inv_qn);
    Proj<float> g;
    gaussian_cov3d<float>(sc, q, v.scale_modifier, g);
    project_view<GSPLAT, float>(v, p, g);

    ProjCot c;
    const float* ccon = RAW ? vrow + B200GS_ROW_CONIC : v_conic + 3 * i;
    c.vA = __ldg(ccon); c.vB = __ldg(ccon + 1); c.vC = __ldg(ccon + 2);
    c.vxy = RAW ? make_float2(__ldg(vrow), __ldg(vrow + 1)) : v_xy[i];
    c.vdepth = 0.f;
    if (GSPLAT) c.vdepth = RAW ? __ldg(vrow + B200GS_ROW_DEPTH) : (v_depth ? __ldg(v_depth + i) : 0.f);
    c.vcomp = (GSPLAT && v_comp != nullptr) ? __ldg(v_comp + i) : 0.f;
    if (RAW) {
        float o, o1;
        logit_sigmoid(__ldg(raw.opac_in + i), o, o1);
        const float v_sig = sigmoid_cotangent<GSPLAT>(__ldg(vrow + B200GS_ROW_OPACITY), o, raw.anti_aliased, g, c);
        // explicit fma: whether nvcc contracts the product into the add depends on the surrounding code (see xm / xa / xf)
        raw.v_opac_logit[i] = fmaf(v_sig * o, o1, ACC ? raw.v_opac_logit[i] : 0.f);
    }
    float dscale[3] = {0.f, 0.f, 0.f};
    float4 dq = make_float4(0.f, 0.f, 0.f, 0.f);
    geometry_backward<GSPLAT>(v, p, q, g, c, dm, dscale, dq);
    if (RAW) raw_param_backward(sc, q, inv_qn, dscale, dq);

    if (ACC) { dm[0] += v_means[3 * i]; dm[1] += v_means[3 * i + 1]; dm[2] += v_means[3 * i + 2]; }
    v_means[3 * i] = dm[0]; v_means[3 * i + 1] = dm[1]; v_means[3 * i + 2] = dm[2];
#pragma unroll
    for (int k = 0; k < 3; ++k) v_scales[3 * i + k] = dscale[k] + (ACC ? v_scales[3 * i + k] : 0.f);
    if (ACC) {
        const float4 old = v_quats[i];
        dq.x += old.x; dq.y += old.y; dq.z += old.z; dq.w += old.w;
    }
    v_quats[i] = dq;
}

// Backward of project_fwd_multi_kernel: every thread walks the W cameras of the step, accumulates the parameter gradients of
// its Gaussian in registers and writes them ONCE (the per-camera launches read-modify-wrote 236 B per Gaussian and camera).
// Cotangents are [.,12] gradient rows (b200gs.h row layout); view j's rows start at v_rows[j] (possibly a peer GPU's buffer
// mapped over NVLink), entry (j, i) uses row row_index[j*n + i] of it.
struct RowSources {
    const float* rows[B200GS_MAX_VIEWS];
};

template <int MC>
__global__ void __launch_bounds__(BWD_THREADS) project_bwd_multi_kernel(const __grid_constant__ ViewPack vp, int nviews, const RawIO raw,
                                                                       const __grid_constant__ RowSources src, int64_t n,
                                                                       const float* __restrict__ means, const float* __restrict__ scales,
                                                                       const float* __restrict__ quats, const int32_t* __restrict__ radii,
                                                                       const uint8_t* __restrict__ clamped, const int32_t* __restrict__ row_index,
                                                                       float* __restrict__ v_means, float* __restrict__ v_scales,
                                                                       float4* __restrict__ v_quats, float* __restrict__ v_shs_dc) {
    __shared__ float s_rows[BWD_THREADS / 32][32 * (MC * 3 + 1)];
    const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    const unsigned lane = threadIdx.x & 31u;
    const int warp = threadIdx.x >> 5;
    const bool in_range = i < n;
    const int stride3 = vp.v[0].sh_stride * 3;
    const int deg = vp.v[0].sh_degree;
    const int ncoef = (deg + 1) * (deg + 1);
    // SH-gradient accumulators over the cameras: the dc coefficient in registers, the rest in this lane's row of the staging buffer
    // (48 accumulator registers kept the kernel at 183 registers = 8 warps per SM)
    const int rw = stride3 - 3;                      // <= MC * 3: the launcher picks MC by the storage width
    float* my_row = s_rows[warp] + lane * (rw | 1);
    float dc_acc[3] = {0.f, 0.f, 0.f};
    for (int c = 0; c < rw; ++c) my_row[c] = 0.f;
    float dm[3] = {0.f, 0.f, 0.f}, dscale[3] = {0.f, 0.f, 0.f}, dlogit = 0.f;
    float4 dq = make_float4(0.f, 0.f, 0.f, 0.f);
    float p[3] = {0.f, 0.f, 0.f}, sc[3] = {1.f, 1.f, 1.f}, q[4] = {1.f, 0.f, 0.f, 0.f}, inv_qn = 1.f, o = 0.f, o1 = 0.f;
    bool loaded = false;
    Proj<float> g;
#pragma unroll 1
    for (int j = 0; j < nviews; ++j) {
        const int64_t e = int64_t(j) * n + i;
        if (!in_range || radii[e] <= 0) continue;
        const int ri = row_index[e];
        if (ri < 0) continue;     // did not fit its fixed-size block: the caller redoes such a step
        const float* vrow = src.rows[j] + int64_t(ri) * B200GS_ROW_FLOATS;
        const float4 w0 = *reinterpret_cast<const float4*>(vrow), w1 = *reinterpret_cast<const float4*>(vrow + 4),
                     w2 = *reinterpret_cast<const float4*>(vrow + 8);
        if (!loaded) {
            p[0] = __ldg(means + 3 * i); p[1] = __ldg(means + 3 * i + 1); p[2] = __ldg(means + 3 * i + 2);
            load_scale_quat<true, float>(scales, quats, i, sc, q, &inv_qn);
            logit_sigmoid(__ldg(raw.opac_in + i), o, o1);
            gaussian_cov3d<float>(sc, q, vp.v[0].scale_modifier, g);      // once per Gaussian; project_view per camera
            loaded = true;
        }
        const B200gsView& v = vp.v[j];
        // SH colour
        {
            const uint8_t cl = clamped[e];
            const float gr = (cl & 1) ? 0.f : w2.x, gg = (cl & 2) ? 0.f : w2.y, gb = (cl & 4) ? 0.f : w2.z;
            float dx, dy, dz, inv_len;
            view_dir(p, v.campos, dx, dy, dz, inv_len);
            float bs[MC];
            sh_basis<MC>(deg, dx, dy, dz, bs);
            dc_acc[0] = fmaf(bs[0], gr, dc_acc[0]); dc_acc[1] = fmaf(bs[0], gg, dc_acc[1]); dc_acc[2] = fmaf(bs[0], gb, dc_acc[2]);
#pragma unroll
            for (int k = 1; k < MC; ++k) {
                if (k < ncoef && 3 * k < rw + 3) {
                    float* a = my_row + 3 * k - 3;
                    a[0] = fmaf(bs[k], gr, a[0]); a[1] = fmaf(bs[k], gg, a[1]); a[2] = fmaf(bs[k], gb, a[2]);
                }
            }
        }
        project_view<true, float>(v, p, g);
        ProjCot c;
        c.vxy = make_float2(w0.x, w0.y);
        c.vdepth = w0.z;
        c.vA = w0.w; c.vB = w1.x; c.vC = w1.y;
        c.vcomp = 0.f;
        dlogit += sigmoid_cotangent<true>(w1.w, o, raw.anti_aliased, g, c) * o * o1;
        geometry_backward<true>(v, p, q, g, c, dm, dscale, dq);
    }
    if (in_range) { v_shs_dc[3 * i] = dc_acc[0]; v_shs_dc[3 * i + 1] = dc_acc[1]; v_shs_dc[3 * i + 2] = dc_acc[2]; }
    flush_sh_rows(s_rows[warp], rw, i, n, lane, raw.v_shs_rest, false);
    if (!in_range) return;
    raw_param_backward(sc, q, inv_qn, dscale, dq);
    v_means[3 * i] = dm[0]; v_means[3 * i + 1] = dm[1]; v_means[3 * i + 2] = dm[2];
    v_scales[3 * i] = dscale[0]; v_scales[3 * i + 1] = dscale[1]; v_scales[3 * i + 2] = dscale[2];
    v_quats[i] = dq;
    raw.v_opac_logit[i] = dlogit;
}

// ------------------------------------------------------------------------------------------------------------------
// standalone SH (gsplat.sh.spherical_harmonics)
// ------------------------------------------------------------------------------------------------------------------
// SPLIT = false: coeffs [n, stride, 3].  SPLIT = true (gsplat's spherical_harmonics_decomposed): coeffs = dc [n, 1, 3] and
// rest [n, stride - 1, 3] read in place through K1's RAW loader; a row with mask[i] == 0 (mask nullable) reads no coefficient and
// gets rgb = 0 and zero gradients.  The evaluation is the same code in both, so unmasked rows are bit-identical.
template <bool SPLIT>
__device__ __forceinline__ bool sh_row_masked(const uint8_t* __restrict__ mask, int64_t i) {
    return SPLIT && mask != nullptr && __ldg(mask + i) == 0;
}

template <bool SPLIT, int MC>
__global__ void __launch_bounds__(256) sh_fwd_kernel(int deg, int stride, int64_t n, const float* __restrict__ dirs,
                                                     const float* __restrict__ coeffs, const float* __restrict__ rest,
                                                     const uint8_t* __restrict__ mask, float* __restrict__ rgb) {
    const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (sh_row_masked<SPLIT>(mask, i)) {
        rgb[3 * i] = 0.f; rgb[3 * i + 1] = 0.f; rgb[3 * i + 2] = 0.f;
        return;
    }
    const int ncoef = (deg + 1) * (deg + 1);
    float dx = __ldg(dirs + 3 * i), dy = __ldg(dirs + 3 * i + 1), dz = __ldg(dirs + 3 * i + 2);
    const float inv_len = normalize_dir(dx, dy, dz);
    float sh[MC * 3];
    load_sh_any<SPLIT, MC>(coeffs, rest, i, stride, ncoef, sh);
    float bs[MC];
    sh_basis<MC>(deg, dx, dy, dz, bs);
    float r = 0.f, g = 0.f, b = 0.f;
#pragma unroll
    for (int k = 0; k < MC; ++k)
        if (k < ncoef) { r += bs[k] * sh[3 * k]; g += bs[k] * sh[3 * k + 1]; b += bs[k] * sh[3 * k + 2]; }
    rgb[3 * i] = r; rgb[3 * i + 1] = g; rgb[3 * i + 2] = b;
}

// SPLIT: v_coeffs = v_dc [n, 1, 3], v_rest [n, stride - 1, 3]; both fully written (zeros on masked rows)
template <bool SPLIT, int MC>
__global__ void __launch_bounds__(256) sh_bwd_kernel(int deg, int stride, int64_t n, const float* __restrict__ dirs,
                                                     const float* __restrict__ coeffs, const float* __restrict__ rest,
                                                     const uint8_t* __restrict__ mask, const float* __restrict__ v_rgb,
                                                     float* __restrict__ v_coeffs, float* __restrict__ v_rest, float* __restrict__ v_dirs) {
    const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int stride3 = stride * 3;
    // gradient row of coefficient k: [n, stride, 3], or dc (k = 0) | rest (k >= 1)
    const auto v_row = [&](int k) { return SPLIT ? (k == 0 ? v_coeffs + 3 * i : v_rest + (i * int64_t(stride - 1) + (k - 1)) * 3)
                                                 : v_coeffs + i * int64_t(stride3) + 3 * k; };
    if (sh_row_masked<SPLIT>(mask, i)) {
        for (int k = 0; k < stride; ++k) {
            float* o = v_row(k);
            o[0] = 0.f; o[1] = 0.f; o[2] = 0.f;
        }
        if (v_dirs != nullptr) { v_dirs[3 * i] = 0.f; v_dirs[3 * i + 1] = 0.f; v_dirs[3 * i + 2] = 0.f; }
        return;
    }
    const int ncoef = (deg + 1) * (deg + 1);
    float dx = __ldg(dirs + 3 * i), dy = __ldg(dirs + 3 * i + 1), dz = __ldg(dirs + 3 * i + 2);
    const float inv_len = normalize_dir(dx, dy, dz);
    const float gr = __ldg(v_rgb + 3 * i), gg = __ldg(v_rgb + 3 * i + 1), gb = __ldg(v_rgb + 3 * i + 2);
    float bs[MC];
    sh_basis<MC>(deg, dx, dy, dz, bs);
    for (int k = 0; k < stride; ++k) {
        const float bk = (k < ncoef) ? bs[k] : 0.f;
        float* o = v_row(k);
        o[0] = bk * gr; o[1] = bk * gg; o[2] = bk * gb;
    }
    if (v_dirs != nullptr) {
        float ddx = 0.f, ddy = 0.f, ddz = 0.f;
        if (deg > 0) {
            float sh[MC * 3];
            load_sh_any<SPLIT, MC>(coeffs, rest, i, stride, ncoef, sh);
            float w[MC];
#pragma unroll
            for (int k = 1; k < MC; ++k) w[k] = (k < ncoef) ? sh[3 * k] * gr + sh[3 * k + 1] * gg + sh[3 * k + 2] * gb : 0.f;
            const float3 d = view_dir_grad<MC>(deg, dx, dy, dz, inv_len, w);
            ddx = d.x; ddy = d.y; ddz = d.z;
        }
        v_dirs[3 * i] = ddx; v_dirs[3 * i + 1] = ddy; v_dirs[3 * i + 2] = ddz;
    }
}

}  // namespace

// Single-view K1 / K8 launch: the kernel comes from a table indexed by the view's mode (constant set) and by whether it needs 25 SH
// coefficients (MC = 25 iff SH is given and sh_degree > 3)
template <bool RAW>
static int project_fwd_launch(const B200gsView& v, const RawIO& raw, int64_t n, const float* means, const float* scales, const float* quats,
                              const float* shs, float* xy, float* depth, int32_t* radii, float* conic, float* comp, int32_t* tiles,
                              float* cov3d, float* rgb, uint8_t* clamped, float* rows, cudaStream_t s) {
    static constexpr decltype(&project_fwd_kernel<false, RAW, 16>) kernels[2][2] = {
        {project_fwd_kernel<false, RAW, 16>, project_fwd_kernel<false, RAW, 25>}, {project_fwd_kernel<true, RAW, 16>, project_fwd_kernel<true, RAW, 25>}};
    if (n == 0) return B200GS_OK;
    kernels[v.mode == B200GS_MODE_GSPLAT][shs != nullptr && v.sh_degree > 3]<<<(unsigned)div_up64(n, 256), 256, 0, s>>>(
        v, raw, n, means, scales, quats, shs, (float2*)xy, depth, radii, conic, comp, tiles, cov3d, rgb, clamped, rows);
    B200GS_LAUNCH_CHECK();
    return B200GS_OK;
}

template <bool RAW>
static int project_bwd_launch(const B200gsView& v, const RawIO& raw, int64_t n, const float* means, const float* scales, const float* quats,
                              const float* shs, const int32_t* radii, const uint8_t* clamped, const float* v_xy, const float* v_depth,
                              const float* v_conic, const float* v_comp, const float* v_rgb, float* v_means, float* v_scales, float* v_quats,
                              float* v_shs, cudaStream_t s) {
    static constexpr decltype(&project_bwd_kernel<false, RAW, 16>) kernels[2][2] = {
        {project_bwd_kernel<false, RAW, 16>, project_bwd_kernel<false, RAW, 25>}, {project_bwd_kernel<true, RAW, 16>, project_bwd_kernel<true, RAW, 25>}};
    if (n == 0) return B200GS_OK;
    kernels[v.mode == B200GS_MODE_GSPLAT][v_shs != nullptr && v.sh_degree > 3]<<<(unsigned)div_up64(n, BWD_THREADS), BWD_THREADS, 0, s>>>(
        v, raw, n, means, scales, quats, shs, radii, clamped, (const float2*)v_xy, v_depth, v_conic, v_comp, v_rgb, v_means, v_scales,
        (float4*)v_quats, v_shs);
    B200GS_LAUNCH_CHECK();
    return B200GS_OK;
}

// split = true: coeffs / v_coeffs are dc [n,1,3], rest / v_rest [n,stride-1,3] read and written in place, mask[n] (nullable) zeroes
// rows, as in sh_fwd_kernel; otherwise rest, mask and v_rest are ignored
static int launch_sh_fwd(int degree, int stride, int64_t n, const float* dirs, const float* coeffs, float* rgb, cudaStream_t s,
                         bool split = false, const float* rest = nullptr, const uint8_t* mask = nullptr) {
    static constexpr decltype(&sh_fwd_kernel<false, 16>) kernels[2][2] = {
        {sh_fwd_kernel<false, 16>, sh_fwd_kernel<false, 25>}, {sh_fwd_kernel<true, 16>, sh_fwd_kernel<true, 25>}};
    if (n == 0) return B200GS_OK;
    kernels[split][degree > 3]<<<(unsigned)div_up64(n, 256), 256, 0, s>>>(degree, stride, n, dirs, coeffs, rest, mask, rgb);
    B200GS_LAUNCH_CHECK();
    return B200GS_OK;
}

static int launch_sh_bwd(int degree, int stride, int64_t n, const float* dirs, const float* coeffs, const float* v_rgb, float* v_coeffs,
                         float* v_dirs, cudaStream_t s, bool split = false, const float* rest = nullptr, const uint8_t* mask = nullptr,
                         float* v_rest = nullptr) {
    static constexpr decltype(&sh_bwd_kernel<false, 16>) kernels[2][2] = {
        {sh_bwd_kernel<false, 16>, sh_bwd_kernel<false, 25>}, {sh_bwd_kernel<true, 16>, sh_bwd_kernel<true, 25>}};
    if (n == 0) return B200GS_OK;
    kernels[split][degree > 3]<<<(unsigned)div_up64(n, 256), 256, 0, s>>>(degree, stride, n, dirs, coeffs, rest, mask, v_rgb, v_coeffs,
                                                                          v_rest, v_dirs);
    B200GS_LAUNCH_CHECK();
    return B200GS_OK;
}

static int check_view(const B200gsView* v, bool needs_sh) {
    if (v == nullptr) { set_error("view is NULL"); return B200GS_EINVAL; }
    if (v->width <= 0 || v->height <= 0) { set_error("bad image size %dx%d", v->width, v->height); return B200GS_EINVAL; }
    if (v->mode != B200GS_MODE_VANILLA && v->mode != B200GS_MODE_GSPLAT) { set_error("bad mode %d", v->mode); return B200GS_EINVAL; }
    if (needs_sh) {
        if (v->sh_degree < 0 || v->sh_degree > 4) { set_error("sh_degree %d unsupported (0..4)", v->sh_degree); return B200GS_EINVAL; }
        if (v->sh_stride < (v->sh_degree + 1) * (v->sh_degree + 1)) {
            set_error("sh_stride %d < (sh_degree+1)^2", v->sh_stride);
            return B200GS_EINVAL;
        }
    }
    return B200GS_OK;
}

static int check_views(const B200gsView* views, int32_t n_views) {
    if (views == nullptr) { set_error("views is NULL"); return B200GS_EINVAL; }
    if (n_views < 1 || n_views > B200GS_MAX_VIEWS) { set_error("n_views %d out of range (1..%d)", n_views, B200GS_MAX_VIEWS); return B200GS_EINVAL; }
    for (int j = 0; j < n_views; ++j) {
        int rc = check_view(views + j, true);
        if (rc) return rc;
        if (views[j].mode != B200GS_MODE_GSPLAT) { set_error("multi-view projection supports gsplat constants only"); return B200GS_EINVAL; }
        if (views[j].sh_degree != views[0].sh_degree || views[j].sh_stride != views[0].sh_stride) {
            set_error("all views of a multi-view launch must share sh_degree / sh_stride");
            return B200GS_EINVAL;
        }
    }
    return B200GS_OK;
}

static size_t project_pack_workspace_bytes(int n_views, int64_t n) {
    return 256 + (size_t)n_views * (size_t)div_up64(n > 0 ? n : 1, PACK_THREADS) * sizeof(uint32_t);
}

}  // namespace b200gs

using namespace b200gs;

extern "C" {

int b200gs_project_fwd(const B200gsView* view, int64_t n, const float* means, const float* scales, const float* quats,
                       const float* shs, float* xy, float* depth, int32_t* radii, float* conic, float* comp,
                       int32_t* tiles, float* cov3d, float* rgb, uint8_t* clamped, void* stream) {
    int rc = check_view(view, shs != nullptr);
    if (rc) return rc;
    B200GS_CHECK_ARG(n >= 0, "n < 0");
    if (n > 0) {
        B200GS_CHECK_ARG(means && scales && quats, "means/scales/quats must not be NULL");
        B200GS_CHECK_ARG(xy && depth && radii && conic && tiles, "xy/depth/radii/conic/tiles must not be NULL");
        B200GS_CHECK_ARG(shs == nullptr || (rgb && clamped), "rgb/clamped required when shs is given");
    }
    return project_fwd_launch<false>(*view, RawIO{}, n, means, scales, quats, shs, xy, depth, radii, conic, comp, tiles, cov3d, rgb, clamped,
                                     nullptr, (cudaStream_t)stream);
}

int b200gs_project_bwd(const B200gsView* view, int64_t n, const float* means, const float* scales, const float* quats,
                       const float* shs, const int32_t* radii, const uint8_t* clamped, const float* v_xy,
                       const float* v_depth, const float* v_conic, const float* v_comp, const float* v_rgb,
                       float* v_means, float* v_scales, float* v_quats, float* v_shs, void* stream) {
    int rc = check_view(view, shs != nullptr);
    if (rc) return rc;
    B200GS_CHECK_ARG(n >= 0, "n < 0");
    if (n > 0) {
        B200GS_CHECK_ARG(means && scales && quats && radii, "means/scales/quats/radii must not be NULL");
        B200GS_CHECK_ARG(v_xy && v_conic, "v_xy/v_conic must not be NULL");
        B200GS_CHECK_ARG(v_means && v_scales && v_quats, "v_means/v_scales/v_quats must not be NULL");
        B200GS_CHECK_ARG((shs == nullptr) == (v_shs == nullptr), "shs and v_shs must be given together");
        B200GS_CHECK_ARG(shs == nullptr || (clamped && v_rgb), "clamped/v_rgb required when shs is given");
    }
    return project_bwd_launch<false>(*view, RawIO{}, n, means, scales, quats, shs, radii, clamped, v_xy, v_depth, v_conic, v_comp, v_rgb,
                                     v_means, v_scales, v_quats, v_shs, (cudaStream_t)stream);
}

int b200gs_project_fwd_rows(const B200gsView* view, int64_t n, const float* means, const float* log_scales, const float* raw_quats,
                            const float* opacity_logits, const float* shs_dc, const float* shs_rest, int32_t anti_aliased, float* rows,
                            int32_t* radii, uint8_t* clamped, int32_t* tiles, void* stream) {
    int rc = check_view(view, true);
    if (rc) return rc;
    B200GS_CHECK_ARG(n >= 0, "n < 0");
    if (n > 0) {
        B200GS_CHECK_ARG(means && log_scales && raw_quats && opacity_logits && shs_dc, "NULL input pointer");
        B200GS_CHECK_ARG(view->sh_stride == 1 || shs_rest, "shs_rest required when sh_stride > 1");
        B200GS_CHECK_ARG(rows && radii && clamped, "NULL output pointer");
        B200GS_CHECK_ARG((reinterpret_cast<uintptr_t>(rows) & 15u) == 0, "rows must be 16-byte aligned");
    }
    RawIO raw{};
    raw.opac_in = opacity_logits; raw.shs_rest = shs_rest; raw.anti_aliased = anti_aliased;
    return project_fwd_launch<true>(*view, raw, n, means, log_scales, raw_quats, shs_dc, nullptr, nullptr, radii, nullptr, nullptr, tiles,
                                    nullptr, nullptr, clamped, rows, (cudaStream_t)stream);
}

int b200gs_project_bwd_rows(const B200gsView* view, int64_t n, const float* means, const float* log_scales, const float* raw_quats,
                            const float* opacity_logits, const float* shs_dc, const float* shs_rest, int32_t anti_aliased,
                            const int32_t* radii, const uint8_t* clamped, const int32_t* row_offsets, const float* v_rows,
                            int32_t accumulate, float* v_means, float* v_log_scales, float* v_raw_quats, float* v_opacity_logits,
                            float* v_shs_dc, float* v_shs_rest, float* v_mean2d, int32_t v_mean2d_cols, void* stream) {
    int rc = check_view(view, true);
    if (rc) return rc;
    B200GS_CHECK_ARG(n >= 0, "n < 0");
    B200GS_CHECK_ARG(v_mean2d == nullptr || v_mean2d_cols == 2 || v_mean2d_cols == 3, "v_mean2d_cols must be 2 or 3");
    if (n > 0) {
        B200GS_CHECK_ARG(means && log_scales && raw_quats && opacity_logits && shs_dc && radii && clamped, "NULL input pointer");
        B200GS_CHECK_ARG(view->sh_stride == 1 || (shs_rest && v_shs_rest), "shs_rest / v_shs_rest required when sh_stride > 1");
        B200GS_CHECK_ARG(v_means && v_log_scales && v_raw_quats && v_opacity_logits && v_shs_dc, "NULL output pointer");
    }
    static const float dummy = 0.f;   // v_rows may be NULL when no Gaussian of the shard is visible: never dereferenced then
    RawIO raw{};
    raw.opac_in = opacity_logits; raw.shs_rest = shs_rest; raw.anti_aliased = anti_aliased;
    raw.v_opac_logit = v_opacity_logits; raw.v_shs_rest = v_shs_rest;
    raw.v_rows = v_rows ? v_rows : &dummy; raw.row_offsets = row_offsets; raw.accumulate = accumulate;
    raw.v_mean2d = v_mean2d; raw.v_mean2d_cols = v_mean2d_cols;
    return project_bwd_launch<true>(*view, raw, n, means, log_scales, raw_quats, shs_dc, radii, clamped, nullptr, nullptr, nullptr, nullptr,
                                    nullptr, v_means, v_log_scales, v_raw_quats, v_shs_dc, (cudaStream_t)stream);
}

int b200gs_project_fwd_raw_multi(const B200gsView* views, int32_t n_views, int64_t n, const float* means, const float* scales,
                                 const float* quats, const float* opac_logits, const float* shs_dc, const float* shs_rest,
                                 int32_t anti_aliased, float* xy, float* depth, int32_t* radii, float* conic, float* rgb, uint8_t* clamped,
                                 float* opac_out, void* stream) {
    int rc = check_views(views, n_views);
    if (rc) return rc;
    B200GS_CHECK_ARG(n >= 0, "n < 0");
    if (n > 0) {
        B200GS_CHECK_ARG(means && scales && quats && opac_logits && shs_dc, "NULL input pointer");
        B200GS_CHECK_ARG(views[0].sh_stride == 1 || shs_rest, "shs_rest required when sh_stride > 1");
        B200GS_CHECK_ARG(xy && depth && radii && conic && rgb && clamped && opac_out, "NULL output pointer");
    }
    if (n == 0 || n_views == 0) return B200GS_OK;
    ViewPack vp;
    for (int j = 0; j < n_views; ++j) vp.v[j] = views[j];
    for (int j = n_views; j < B200GS_MAX_VIEWS; ++j) vp.v[j] = views[0];
    RawIO raw{};
    raw.opac_in = opac_logits; raw.shs_rest = shs_rest; raw.opac_out = opac_out; raw.anti_aliased = anti_aliased;
    const auto kernel = views[0].sh_degree > 3 ? project_fwd_multi_kernel<25> : project_fwd_multi_kernel<16>;
    kernel<<<(unsigned)div_up64(n, 256), 256, 0, (cudaStream_t)stream>>>(vp, n_views, raw, n, means, scales, quats, shs_dc, (float2*)xy, depth,
                                                                         radii, conic, rgb, clamped);
    B200GS_LAUNCH_CHECK();
    return B200GS_OK;
}

size_t b200gs_project_pack_workspace_bytes(int32_t n_views, int64_t n) { return project_pack_workspace_bytes(n_views, n); }

int b200gs_project_pack_multi(const B200gsView* views, int32_t n_views, int64_t n, const float* means, const float* scales, const float* quats,
                              const float* opac_logits, const float* shs_dc, const float* shs_rest, int32_t anti_aliased, float* xy,
                              int32_t* radii, uint8_t* clamped, int32_t* row_index, void* const* dst_rows, int64_t cap, void* workspace,
                              size_t workspace_bytes, int64_t* d_count, void* stream) {
    B200GS_CHECK_ARG(views && n_views >= 1 && n_views <= B200GS_MAX_VIEWS, "n_views must be 1..B200GS_MAX_VIEWS");
    B200GS_CHECK_ARG(n >= 0 && n < (int64_t(1) << 30) && cap > 0 && cap < (int64_t(1) << 30), "bad size");
    B200GS_CHECK_ARG(int64_t(n_views - 1) * cap + cap <= INT32_MAX, "n_views * block_rows exceeds the int32 range of row_index");
    for (int j = 0; j < n_views; ++j) {
        int rc = check_view(views + j, true);
        if (rc) return rc;
        B200GS_CHECK_ARG(views[j].mode == B200GS_MODE_GSPLAT, "multi-view launches use the gsplat constant set");
        B200GS_CHECK_ARG(dst_rows && dst_rows[j] && (reinterpret_cast<uintptr_t>(dst_rows[j]) & 15u) == 0, "dst_rows: NULL or misaligned");
    }
    if (n > 0) {
        B200GS_CHECK_ARG(means && scales && quats && opac_logits && shs_dc, "NULL input pointer");
        B200GS_CHECK_ARG(views[0].sh_stride == 1 || shs_rest, "shs_rest required when sh_stride > 1");
        B200GS_CHECK_ARG(xy && radii && clamped && row_index && workspace, "NULL output pointer");
    }
    B200GS_CHECK_ARG(d_count, "NULL d_count");
    const cudaStream_t s = (cudaStream_t)stream;
    if (n_views == 0) return B200GS_OK;
    if (n == 0) {
        B200GS_CUDA(cudaMemsetAsync(d_count, 0, sizeof(int64_t) * (size_t)n_views, s));
        return B200GS_OK;
    }
    const size_t need = project_pack_workspace_bytes(n_views, n);
    if (workspace_bytes < need) {
        set_error("project_pack_multi: workspace too small (%zu < %zu bytes)", workspace_bytes, need);
        return B200GS_EINVAL;
    }
    ViewPack vp;
    PackDst dst;
    for (int j = 0; j < B200GS_MAX_VIEWS; ++j) {
        vp.v[j] = views[j < n_views ? j : 0];
        dst.p[j] = j < n_views ? (float*)dst_rows[j] : nullptr;
    }
    RawIO raw{};
    raw.opac_in = opac_logits; raw.shs_rest = shs_rest; raw.anti_aliased = anti_aliased;
    B200GS_CUDA(cudaMemsetAsync(workspace, 0, need, s));
    uint32_t* ticket = (uint32_t*)workspace;
    uint32_t* state = ticket + 64;
    const unsigned blocks = (unsigned)div_up64(n, PACK_THREADS);
    const size_t smem = (size_t)n_views * PACK_THREADS * 3 * sizeof(float4);
    // The first launch of each instantiation also raises its dynamic shared-memory limit (8 cameras: 96 KB)
    const auto launch = [&](auto mc) {
        const auto kernel = project_pack_multi_kernel<decltype(mc)::value>;
        static const cudaError_t attr_rc = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                                B200GS_MAX_VIEWS * PACK_THREADS * 3 * (int)sizeof(float4));
        if (attr_rc == cudaSuccess)
            kernel<<<blocks, PACK_THREADS, smem, s>>>(vp, n_views, raw, n, means, scales, quats, shs_dc, (float2*)xy, radii, clamped, row_index, dst,
                                                      cap, ticket, state, d_count);
        return attr_rc;
    };
    const cudaError_t attr_rc = views[0].sh_degree > 3 ? launch(std::integral_constant<int, 25>{}) : launch(std::integral_constant<int, 16>{});
    if (attr_rc != cudaSuccess) {
        set_error("project_pack_multi: cudaFuncSetAttribute failed: %s", cudaGetErrorString(attr_rc));
        return B200GS_ECUDA;
    }
    B200GS_LAUNCH_CHECK();
    return B200GS_OK;
}

int b200gs_project_bwd_rows_multi(const B200gsView* views, int32_t n_views, int64_t n, const float* means, const float* scales,
                                  const float* quats, const float* opac_logits, const float* shs_dc, const float* shs_rest,
                                  int32_t anti_aliased, const int32_t* radii, const uint8_t* clamped, const int32_t* row_index,
                                  const float* const* v_rows, float* v_means, float* v_scales, float* v_quats, float* v_opac_logit,
                                  float* v_shs_dc, float* v_shs_rest, void* stream) {
    int rc = check_views(views, n_views);
    if (rc) return rc;
    B200GS_CHECK_ARG(n >= 0, "n < 0");
    if (n > 0) {
        B200GS_CHECK_ARG(means && scales && quats && opac_logits && shs_dc && radii && clamped && row_index && v_rows, "NULL input pointer");
        B200GS_CHECK_ARG(views[0].sh_stride == 1 || (shs_rest && v_shs_rest), "shs_rest / v_shs_rest required when sh_stride > 1");
        B200GS_CHECK_ARG(v_means && v_scales && v_quats && v_opac_logit && v_shs_dc, "NULL output pointer");
    }
    if (n == 0 || n_views == 0) return B200GS_OK;
    ViewPack vp;
    RowSources src;
    static const float dummy[B200GS_ROW_FLOATS] = {0.f};
    for (int j = 0; j < B200GS_MAX_VIEWS; ++j) {
        vp.v[j] = views[j < n_views ? j : 0];
        src.rows[j] = (j < n_views && v_rows[j]) ? v_rows[j] : dummy;   // NULL only when no row of that view is ever read
    }
    RawIO raw{};
    raw.opac_in = opac_logits; raw.shs_rest = shs_rest; raw.anti_aliased = anti_aliased;
    raw.v_opac_logit = v_opac_logit; raw.v_shs_rest = v_shs_rest;
    // the SH-gradient rows accumulate in the kernel's staging buffer: coefficient storage wider than 16 takes the 25-coefficient instantiation
    if (views[0].sh_stride > 25) {
        set_error("project_bwd_multi: sh_stride %d exceeds 25 coefficients", views[0].sh_stride);
        return B200GS_EINVAL;
    }
    const auto kernel = views[0].sh_degree > 3 || views[0].sh_stride > 16 ? project_bwd_multi_kernel<25> : project_bwd_multi_kernel<16>;
    kernel<<<(unsigned)div_up64(n, BWD_THREADS), BWD_THREADS, 0, (cudaStream_t)stream>>>(vp, n_views, raw, src, n, means, scales, quats, radii,
                                                                                         clamped, row_index, v_means, v_scales,
                                                                                         (float4*)v_quats, v_shs_dc);
    B200GS_LAUNCH_CHECK();
    return B200GS_OK;
}

int b200gs_sh_fwd(int32_t degree, int32_t sh_stride, int64_t n, const float* dirs, const float* coeffs, float* rgb, void* stream) {
    B200GS_CHECK_ARG(degree >= 0 && degree <= 4, "degree must be 0..4");
    B200GS_CHECK_ARG(sh_stride >= (degree + 1) * (degree + 1), "sh_stride < (degree+1)^2");
    B200GS_CHECK_ARG(n >= 0, "n < 0");
    B200GS_CHECK_ARG(n == 0 || (dirs && coeffs && rgb), "NULL pointer");
    return launch_sh_fwd(degree, sh_stride, n, dirs, coeffs, rgb, (cudaStream_t)stream);
}

int b200gs_sh_bwd(int32_t degree, int32_t sh_stride, int64_t n, const float* dirs, const float* coeffs, const float* v_rgb,
                  float* v_coeffs, float* v_dirs, void* stream) {
    B200GS_CHECK_ARG(degree >= 0 && degree <= 4, "degree must be 0..4");
    B200GS_CHECK_ARG(sh_stride >= (degree + 1) * (degree + 1), "sh_stride < (degree+1)^2");
    B200GS_CHECK_ARG(n >= 0, "n < 0");
    B200GS_CHECK_ARG(n == 0 || (dirs && coeffs && v_rgb && v_coeffs), "NULL pointer");
    return launch_sh_bwd(degree, sh_stride, n, dirs, coeffs, v_rgb, v_coeffs, v_dirs, (cudaStream_t)stream);
}

int b200gs_sh_split_fwd(int32_t degree, int32_t k_rest, int64_t n, const float* dirs, const float* dc, const float* rest, const uint8_t* mask,
                        float* rgb, void* stream) {
    B200GS_CHECK_ARG(degree >= 0 && degree <= 4, "degree must be 0..4");
    B200GS_CHECK_ARG(k_rest >= 0 && k_rest + 1 >= (degree + 1) * (degree + 1), "1 + k_rest < (degree+1)^2");
    B200GS_CHECK_ARG(n >= 0, "n < 0");
    B200GS_CHECK_ARG(n == 0 || (dirs && dc && rgb && (k_rest == 0 || rest)), "NULL pointer");
    return launch_sh_fwd(degree, k_rest + 1, n, dirs, dc, rgb, (cudaStream_t)stream, true, rest, mask);
}

int b200gs_sh_split_bwd(int32_t degree, int32_t k_rest, int64_t n, const float* dirs, const float* dc, const float* rest, const uint8_t* mask,
                        const float* v_rgb, float* v_dc, float* v_rest, float* v_dirs, void* stream) {
    B200GS_CHECK_ARG(degree >= 0 && degree <= 4, "degree must be 0..4");
    B200GS_CHECK_ARG(k_rest >= 0 && k_rest + 1 >= (degree + 1) * (degree + 1), "1 + k_rest < (degree+1)^2");
    B200GS_CHECK_ARG(n >= 0, "n < 0");
    B200GS_CHECK_ARG(n == 0 || (dirs && dc && v_rgb && v_dc && (k_rest == 0 || (rest && v_rest))), "NULL pointer");
    return launch_sh_bwd(degree, k_rest + 1, n, dirs, dc, v_rgb, v_dc, v_dirs, (cudaStream_t)stream, true, rest, mask, v_rest);
}

}  // extern "C"
