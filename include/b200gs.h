/*
 * b200gs — C ABI of the sm_90a (H100) differentiable 3D-Gaussian rasterizer (libb200gs.so).
 *
 * This is the drop-in boundary for the hot path of yzslab/gaussian-splatting-lightning.  The reference has no
 * native code of its own: its renderers call two pip extensions through Python, and these entry points are what a
 * binding for those call sites needs (citations relative to the reference repository):
 *
 *   diff_gaussian_rasterization.GaussianRasterizer(...)(means3D, means2D, shs, colors_precomp, opacities, scales,
 *       rotations, cov3D_precomp) -> (color, radii)            internal/renderers/vanilla_renderer.py:62-77,111-120
 *   gsplat.v0_interfaces.project_gaussians(...) -> 7-tuple     internal/renderers/gsplat_renderer.py:64-79
 *   gsplat.sh.spherical_harmonics(deg, dirs, coeffs)           internal/renderers/gsplat_renderer.py:105
 *   gsplat.rasterize.rasterize_gaussians(...) -> [H,W,D](,alpha)  internal/renderers/gsplat_renderer.py:86-99
 *   gsplat.cuda._wrapper / gsplat.sh_decomposed / gsplat.cuda.isect_tiles_tile_based_culling / rasterize_to_pixels
 *                                                              internal/renderers/gsplat_v1_renderer.py:8-20
 *
 * Conventions
 *   - every pointer is a DEVICE pointer unless named host_*; all floating point is fp32, contiguous.
 *   - the library never allocates or frees device memory: the caller (PyTorch's caching allocator) owns every
 *     buffer including the workspace -> no hidden cudaMalloc, no hidden synchronisation (except where stated).
 *   - all work is enqueued on the cudaStream_t passed as `stream` (a CUstream handle; pass
 *     torch.cuda.current_stream().cuda_stream).
 *   - return 0 on success, a negative B200GS_E* code on failure; b200gs_last_error() gives a thread-local message.
 *     Nothing throws across the ABI; nothing calls exit().  Re-entrant: no global mutable state.
 *   - "mode": B200GS_MODE_VANILLA = diff-gaussian-rasterization semantics (near 0.2, mean2D via the NDC projection
 *     matrix, pixel sample at integer coords, alpha clamp 0.99 straight-through, stop T<1e-4, rect max uses +15);
 *     B200GS_MODE_GSPLAT = the semantics of internal/utils/gaussian_projection.py + gsplat's rasterizer (near 0.01,
 *     K t/(z+1e-6), blur compensation, pixel centres +0.5, alpha clamp 0.999 as a true clamp, stop T<=1e-4,
 *     rect max = int((p+r)/16)+1).
 */
#ifndef B200GS_H
#define B200GS_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define B200GS_API __attribute__((visibility("default")))
#else
#define B200GS_API
#endif

#define B200GS_MODE_VANILLA 0
#define B200GS_MODE_GSPLAT 1

#define B200GS_OK 0
#define B200GS_EINVAL (-1)    /* bad argument (null pointer, bad size, unsupported degree/channels) */
#define B200GS_ECUDA (-2)     /* a CUDA call or launch failed; message holds cudaGetErrorString */
#define B200GS_ENOSPACE (-3)  /* workspace or pair capacity too small */

#define B200GS_TILE 16

/* One view.  Matrices are stored exactly as the reference's Camera stores them (cameras.py:147-189):
 * viewmatrix = world_to_camera, "transposed" (row-major [4][4], translation in the last ROW; p_cam = p * M[:3,:3] + M[3,:3]);
 * projmatrix = full_projection = world_to_camera @ projection (same layout; vanilla mode only). */
typedef struct B200gsView {
    int32_t width;
    int32_t height;
    int32_t mode;           /* B200GS_MODE_* */
    int32_t sh_degree;      /* active degree 0..4 */
    int32_t sh_stride;      /* coefficients stored per Gaussian (K of shs[N,K,3]); >= (sh_degree+1)^2 */
    int32_t reserved0;
    float fx, fy, cx, cy;   /* gsplat mode intrinsics (gsplat_renderer.py:70-73) */
    float tanfovx, tanfovy; /* vanilla mode (vanilla_renderer.py:59-60) */
    float scale_modifier;
    float eps2d;            /* 2D low-pass added to the cov2D diagonal: 0.3 */
    float near_plane;       /* <=0 selects the mode default (0.2 vanilla / 0.01 gsplat) */
    float reserved1;
    float viewmatrix[16];
    float projmatrix[16];
    float campos[3];
    float reserved2;
} B200gsView;

B200GS_API const char* b200gs_last_error(void);
B200GS_API int b200gs_version(void);
/* number of CUDA kernels this library has launched in this process (monotonic; every launch site increments it) */
B200GS_API int64_t b200gs_launch_count(void);

/* ---- K1: per-Gaussian projection (+ optional fused SH colour) ------------------------------------------------
 * replaces dgr preprocessCUDA / gsplat project_gaussians (+ spherical_harmonics when shs != NULL).
 * in : means[n,3] scales[n,3] quats[n,4] (wxyz, used as given); shs[n,sh_stride,3] or NULL.
 * out: xy[n,2] depth[n] radii[n] conic[n,3] tiles[n]; comp[n] (gsplat, nullable); cov3d[n,6] upper triangle (nullable);
 *      rgb[n,3] = max(SH+0.5,0) and clamped[n] (bit c set when channel c was clamped) when shs != NULL.
 *      Culled Gaussians get zeros everywhere (radii 0, tiles 0).
 * SH view direction: normalize(mean - campos).  */
B200GS_API int b200gs_project_fwd(const B200gsView* view, int64_t n, const float* means, const float* scales, const float* quats,
                       const float* shs, float* xy, float* depth, int32_t* radii, float* conic, float* comp,
                       int32_t* tiles, float* cov3d, float* rgb, uint8_t* clamped, void* stream);

/* ---- K8: backward of K1 ------------------------------------------------------------------------------------------
 * in : the K1 inputs, radii (visibility), clamped (when shs), and cotangents v_xy[n,2] (vanilla: dgr's NDC-scaled
 *      dL/dmean2D, i.e. pixel gradient x (0.5W, 0.5H); gsplat: pixel units), v_depth[n] (nullable), v_conic[n,3] (true
 *      partials of power = -(A dx^2 + C dy^2)/2 - B dx dy), v_comp[n] (nullable), v_rgb[n,3] (nullable unless shs).
 * out: v_means[n,3] v_scales[n,3] v_quats[n,4] and v_shs[n,sh_stride,3] (when shs) — fully written (zeros for culled).
 * vanilla mode back-propagates the SH view direction into v_means; gsplat mode does not (renderers detach it). */
B200GS_API int b200gs_project_bwd(const B200gsView* view, int64_t n, const float* means, const float* scales, const float* quats,
                       const float* shs, const int32_t* radii, const uint8_t* clamped, const float* v_xy,
                       const float* v_depth, const float* v_conic, const float* v_comp, const float* v_rgb,
                       float* v_means, float* v_scales, float* v_quats, float* v_shs, void* stream);

/* ---- per-Gaussian passes next to the renderer in a training step (SURVEY §8f rank 4) ---------------------------------------
 * b200gs_selective_adam: visibility-masked Adam step of one [rows, width] parameter tensor (gsplat.optimizers.SelectiveAdam /
 *     diff-accel SparseGaussianAdam, internal/optimizers.py:26-90): for the rows with visible[row] != 0
 *     m = b1 m + (1-b1) g;  v = b2 v + (1-b2) g^2;  p -= lr m / (sqrt(v) + eps)   (no bias correction, like those kernels);
 *     rows that did not take part in the view keep parameter and moments untouched.
 * b200gs_densify_stats: VanillaDensityControllerImpl.update_states (vanilla_density_controller.py:101-123) in one pass: on the
 *     visible rows (visible[n] bytes, or radii > 0 when NULL) max_radii2d = max(max_radii2d, radii), grad_accum += |grad[:, :2] *
 *     (scale_x, scale_y)|, denom += 1.  grad has grad_stride floats per row (2 for gsplat xys, 3 for dgr's screenspace points). */
B200GS_API int b200gs_selective_adam(int64_t rows, int32_t width, float* param, const float* grad, float* exp_avg, float* exp_avg_sq,
                                     const uint8_t* visible, float lr, float beta1, float beta2, float eps, void* stream);
B200GS_API int b200gs_densify_stats(int64_t n, const int32_t* radii, const uint8_t* visible, const float* grad, int32_t grad_stride,
                                    float scale_x, float scale_y, float* max_radii2d, float* grad_accum, float* denom, void* stream);

/* ---- 3DGS-MCMC (internal/density_controllers/mcmc_density_controller.py) -------------------------------------------------
 * b200gs_mcmc_relocation: gsplat's compute_relocation (mcmc_density_controller.py:13,121-128), Eq. (9) of 3DGS-MCMC, one sampled
 *     Gaussian per thread.  With N = clamp(counts[i], 1, n_max):
 *         new_opacities[i] = o' = 1 - (1 - o)^(1/N)
 *         new_scales[i]    = scales[i] * o / D,   D = sum_{j=1..N} (-1)^(j-1) C(N,j) o'^j / sqrt(j)
 *     (the hockey-stick form of the paper's double sum), evaluated in fp64.  binoms is the controller's [n_max, n_max] table
 *     (mcmc_density_controller.py:53-60): it bounds N, and no entry of it is read (fp32 rounds every C(n,k) > 2^24, which
 *     moves D by up to 9e-5 relative), so unlike gsplat's kernel a count above n_max never reads outside it.
 * b200gs_mcmc_position_noise: MCMCDensityControllerImpl._add_xyz_noise (mcmc_density_controller.py:93-120) in one in-place pass
 *     over the raw parameters: means[i] += scale * w * Sigma z, Sigma = R(q) diag(s)^2 R(q)^T with s = exp(log_scales[i]) and
 *     q = raw_quats[i] / max(|raw_quats[i]|, 1e-12) (K8's fp32 geometry), o = sigmoid(opacity_logits[i]),
 *     w = 1 / (1 + exp(-100 ((1 - o) - 0.995))), and z three standard normals of Philox4x32-10 keyed by seed, subsequence
 *     offset + i.  scale = noise_lr * xyz_lr.  raw_quats must be 16-byte aligned (read as float4).
 * Algorithmic bytes: relocation 20 B in + 16 B out per sampled Gaussian; position noise 44 B in + 12 B out per Gaussian. */
B200GS_API int b200gs_mcmc_relocation(int64_t n, const float* opacities, const float* scales, const int32_t* counts, const float* binoms,
                                      int32_t n_max, float* new_opacities, float* new_scales, void* stream);
B200GS_API int b200gs_mcmc_position_noise(int64_t n, float* means, const float* log_scales, const float* raw_quats,
                                          const float* opacity_logits, float scale, uint64_t seed, uint64_t offset, void* stream);

/* ---- Bilateral-grid colour correction (internal/output_processors/bilagrid.py, internal/utils/lib_bilagrid.py) ------------------
 * b200gs_bilagrid_slice_fwd: lib_bilagrid's slice(...)["rgb"] as BilagridProcessorModule.forward calls it (bilagrid.py:115-124).
 *     grids float[n_grids,12,L,gh,gw] contiguous, xy float[batch,height,width,2] contiguous, grid_idx int64[n_idx] with n_idx == 1
 *     (one grid for every row) or n_idx == batch.  rgb and out are addressed as base[b sb + y sy + x sx + c sc] (element strides,
 *     so the processor's permuted CHW render needs no copy).  Per pixel, with G = grids[grid_idx[b]]:
 *         gray = 0.299 r + 0.587 g + 0.114 b,  ix = ((2 (x - 0.5) + 1) / 2) (gw - 1),  iy likewise with gh,
 *         iz = ((2 gray - 1 + 1) / 2) (L - 1),  each clipped to [0, size - 1];
 *         A[c] = trilinear interpolation of G[c] at (iz, iy, ix) (corners outside the grid contribute nothing),
 *         out_i = sum_j A[4i + j] rgb_j + A[4i + 3].
 *     A grid index outside [0, n_grids) reads no grid and sets that row's output to NaN.
 * b200gs_bilagrid_slice_bwd: v_out (same strides) -> v_rgb (same strides, NULL: not computed) and v_grids (accumulated into, NULL:
 *     not computed).  v_rgb includes the path through the guidance gray; a clipped coordinate passes no gradient, a coordinate
 *     exactly on 0 or size - 1 included (grid_sample's border rule).  xy gets no gradient.
 * b200gs_bilagrid_tv_fwd: lib_bilagrid's total_variation_loss (bilagrid.py:100-104) on grids float[n,channels,L,gh,gw]:
 *         tv = (1/n) sum_{axis in L,gh,gw} sum (x[.., i+1, ..] - x[.., i, ..])^2 / max(numel per grid of the difference, 1)
 *     as b200gs_bilagrid_tv_blocks(...) per-CTA partial sums, which the caller adds in a fixed order.
 * b200gs_bilagrid_tv_bwd: v_grids = v_tv[0] * d tv / d grids (v_tv a device scalar), written densely.
 * Algorithmic bytes: slice forward 8 (xy) + 12 (rgb) + 12 (out) per pixel + the grid; backward 8 + 12 + 12 (v_out) + 12 (v_rgb) per
 *     pixel + the grid and its gradient; tv forward 4 per grid element, backward 8. */
B200GS_API int b200gs_bilagrid_slice_fwd(int32_t n_grids, int32_t grid_l, int32_t grid_h, int32_t grid_w, const float* grids,
                                         int32_t batch, int32_t height, int32_t width, const float* xy, const float* rgb, int64_t sb,
                                         int64_t sy, int64_t sx, int64_t sc, const int64_t* grid_idx, int32_t n_idx, float* out,
                                         void* stream);
B200GS_API int b200gs_bilagrid_slice_bwd(int32_t n_grids, int32_t grid_l, int32_t grid_h, int32_t grid_w, const float* grids,
                                         int32_t batch, int32_t height, int32_t width, const float* xy, const float* rgb, int64_t sb,
                                         int64_t sy, int64_t sx, int64_t sc, const int64_t* grid_idx, int32_t n_idx,
                                         const float* v_out, float* v_rgb, float* v_grids, void* stream);
B200GS_API int64_t b200gs_bilagrid_tv_blocks(int32_t n, int32_t channels, int32_t grid_l, int32_t grid_h, int32_t grid_w);
B200GS_API int b200gs_bilagrid_tv_fwd(int32_t n, int32_t channels, int32_t grid_l, int32_t grid_h, int32_t grid_w, const float* grids,
                                      float* partials, void* stream);
B200GS_API int b200gs_bilagrid_tv_bwd(int32_t n, int32_t channels, int32_t grid_l, int32_t grid_h, int32_t grid_w, const float* grids,
                                      const float* v_tv, float* v_grids, void* stream);

/* ---- Appearance-embedding colour pass (internal/renderers/gsplat_appearance_embedding_renderer.py) ---------------------------------
 * The MLP of Model.forward (:77-93) and the colour / opacity epilogue of _get_rgbs_and_opacities (:239-295), on the tensor cores
 * (mma.sync TF32, each product as three TF32 products of split operands: FP32-level accuracy, FP32 accumulation).
 * B200gsAppearanceMlp (a HOST struct of sizes, flags and DEVICE pointers) describes the network:
 *     feat_dim F (a multiple of 8); n_freq: frequencies of PositionalEncoding(3, n_freq) of the view direction, < 0: no view direction;
 *     n_neurons 64 | 128; n_layers 2..4 linear layers, the output layer included; n_out 3 | 4.
 *     weights[l] / biases[l], l < n_layers: torch Linear layout [out, in].  weights[0] has w0_stride floats per row; the kernels read
 *     its columns [0, F) (features) and [w0_pe_col, w0_pe_col + 3 (2 n_freq + 1)) (view direction).  The per-image embedding is the
 *     same for every row, so the caller folds its columns into biases[0] = b_0 + W_0[:, F:F+E] e.
 *     normalize: rows of `features` are divided by max(|row|, 1e-12) first.  normalize_dirs: so is the view direction.
 *     epilogue: 0 = out[n, n_out] holds the sigmoid outputs; 1 = the renderer's colours, see below.
 * Rows: mask uint8[n] (NULL: every row); a row with mask[i] == 0 is not evaluated.  The view direction of row i is
 *     dirs[i] - cam (cam float[3] on the device, NULL: zero), both NULL when n_freq < 0.
 * b200gs_appearance_mlp_fwd, epilogue == 1, with s = the sigmoid outputs of a masked row:
 *         out[i] = clamp((base_rgb[i] + 0.5) + (2 s[0..2] - 1), 0, 1)                                    out float[n,3]
 *         n_out == 4: opacity_offsets[i] = s[3], opacities[i] = min(s[3] + raw_opacity[i], 1)
 *     and out[i] = 0, opacity_offsets[i] = 0, opacities[i] = min(raw_opacity[i], 1) for the other rows: every output is fully written.
 * b200gs_appearance_mlp_bwd: recomputes the activations.  v_out as out; v_opacities / v_opacity_offsets float[n], nullable.
 *     Writes v_base_rgb[n,3] and v_raw_opacity[n] (epilogue == 1; the latter when n_out == 4), v_features[n,F] (NULL: not computed;
 *     through the normalisation when on), each fully written with zeros in the unmasked rows, and v_params, one dense vector
 *         W_0 [n_neurons, K0p] | W_1 | .. | W_last [n_out, n_neurons] | b_0 | .. | b_last,   K0p = F + 3 (2 n_freq + 1) rounded up to 8,
 *     W_0's columns being the features, then the view direction, then zeros.  Every persistent CTA sums its rows into its own block
 *     of `workspace` (b200gs_appearance_mlp_workspace_bytes, 16-byte aligned) and a second kernel adds the blocks in a fixed order: two
 *     calls on the same inputs give bit-identical v_params.  No gradient reaches dirs or cam (the reference detaches them).
 * b200gs_appearance_mlp_workspace_bytes: 0 when the shape is not supported (sizes outside the sets above, or a first layer so wide
 *     that the weights and one 16-row tile of activations exceed 227 KB of shared memory).  A CTA runs 8 warps of 16 rows when
 *     they fit beside the weights (every 64-neuron network), else 4, 2 or 1.
 * Launches: forward 1, backward 2 (0 and 1 when n == 0), whatever the mask holds.
 * Algorithmic bytes per masked row, F = 64: forward 256 (features) + 12 + 12 (+ 12 dirs, + 4 + 8 opacity); backward 256 + 12 + 12
 *     in, 256 + 12 out.  FLOPs per masked row: 2 MACs x (K0p n_neurons + (n_layers - 2) n_neurons^2 + 8 n_neurons) forward; the
 *     backward recomputes that and adds twice as much again (gradients to the inputs and to the weights). */
#define B200GS_APPEARANCE_MAX_LAYERS 4
typedef struct B200gsAppearanceMlp {
    int32_t feat_dim, n_freq, n_neurons, n_layers, n_out;
    int32_t normalize, normalize_dirs, epilogue;
    int32_t w0_stride, w0_pe_col;
    const float* weights[B200GS_APPEARANCE_MAX_LAYERS];
    const float* biases[B200GS_APPEARANCE_MAX_LAYERS];
} B200gsAppearanceMlp;
B200GS_API size_t b200gs_appearance_mlp_workspace_bytes(int32_t feat_dim, int32_t n_freq, int32_t n_neurons, int32_t n_layers, int32_t n_out);
B200GS_API int b200gs_appearance_mlp_fwd(const B200gsAppearanceMlp* mlp, int64_t n, const float* features, const uint8_t* mask,
                                         const float* base_rgb, const float* dirs, const float* cam, const float* raw_opacity, float* out,
                                         float* opacity_offsets, float* opacities, void* stream);
B200GS_API int b200gs_appearance_mlp_bwd(const B200gsAppearanceMlp* mlp, int64_t n, const float* features, const uint8_t* mask,
                                         const float* base_rgb, const float* dirs, const float* cam, const float* raw_opacity,
                                         const float* v_out, const float* v_opacities, const float* v_opacity_offsets, float* v_base_rgb,
                                         float* v_features, float* v_raw_opacity, void* workspace, size_t workspace_bytes, float* v_params,
                                         void* stream);

/* ---- Learned exposure correction (internal/output_processors/exposure.py, ExposureProcessorModule.forward :112-143) ------------
 * b200gs_exposure_fwd: one view's colour transform.  render and out are float[3,H,W] addressed as base[c sc + y sy + x sx] (element
 *     strides, so the permuted [H,W,3] render of the v1 and appearance renderers needs no copy); channels must be 3.
 *     exposure_params float[n_appearances, n_params] contiguous, n_params 4 (no bias) or 7 (with_bias); the row is the int64 read
 *     from appearance_id on the device, or host_appearance_id when appearance_id is NULL.  shade float[shade_size, shade_size]
 *     contiguous (the reference's shade_correction[0]), NULL with shade_size 0 when shade correction is off.  With
 *     a = sigmoid(exposure_params[id]):
 *         M = sigmoid(shade) / max(max(sigmoid(shade)), 1e-4),
 *         m(y, x) = F.interpolate(M, (H, W), mode="bilinear", align_corners=True)   (1 without shade correction),
 *         x_c = (a_c max_gray_scale) (render_c m) [+ 2 a_{3+c} - 1],   out_c = (clamp(x_c, 0, 1) + 1e-5) ^ (a_last max_gamma).
 *     An id outside [0, n_appearances) reads no parameter row and makes out NaN.
 * b200gs_exposure_bwd: v_out (same strides) -> v_render (same strides; the clamp passes the gradient as identity, as the reference's
 *     straight-through clamp), v_params float[n_appearances, n_params] (written whole: rows other than id are zero) and, with shade
 *     correction, v_shade float[shade_size, shade_size] (written whole; no gradient through the detached max).  Parameter sums are
 *     per-CTA partials added in a fixed order and v_shade is gathered per cell in a fixed order: two calls on the same inputs give
 *     bit-identical gradients.  An out-of-range id makes v_render NaN and v_params, v_shade zero.
 * b200gs_exposure_workspace_bytes: device scratch of the forward (backward == 0) or the backward (backward != 0) at this image and
 *     shade size; 0 for sizes the kernels do not take (H or W < 1, H > 524280, H W > 2^31 - 1, shade_size outside 0..4096).
 * Launches: forward 2 (prologue, pixels), backward 3 (prologue, pixels, reduction).  No host synchronisation.
 * Algorithmic bytes: forward 12 in + 12 out per pixel; backward 24 in + 12 out per pixel, plus, with shade correction, v_m 4 out and
 *     4 in per pixel. */
B200GS_API size_t b200gs_exposure_workspace_bytes(int32_t height, int32_t width, int32_t shade_size, int32_t backward);
B200GS_API int b200gs_exposure_fwd(int32_t channels, int32_t height, int32_t width, const float* render, int64_t sc, int64_t sy, int64_t sx,
                                   int32_t n_appearances, int32_t n_params, const float* exposure_params, const int64_t* appearance_id,
                                   int64_t host_appearance_id, int32_t shade_size, const float* shade, float max_gray_scale,
                                   float max_gamma, void* workspace, size_t workspace_bytes, float* out, void* stream);
B200GS_API int b200gs_exposure_bwd(int32_t channels, int32_t height, int32_t width, const float* render, int64_t sc, int64_t sy, int64_t sx,
                                   int32_t n_appearances, int32_t n_params, const float* exposure_params, const int64_t* appearance_id,
                                   int64_t host_appearance_id, int32_t shade_size, const float* shade, float max_gray_scale,
                                   float max_gamma, void* workspace, size_t workspace_bytes, const float* v_out, float* v_render,
                                   float* v_params, float* v_shade, void* stream);

/* b200gs_knn_mean_dist2: simple_knn's distCUDA2 (vanilla_gaussian.py:122-125, the scale initialiser): mean_dist2[i] = mean of the squared
 *     distances from points[i] (float[n,3]) to its 3 nearest neighbours (exact).  Synchronises the stream once (the hash grid is sized
 *     on the host from the bounding box); init-time only. */
B200GS_API size_t b200gs_knn_workspace_bytes(int64_t n);
B200GS_API int b200gs_knn_mean_dist2(int64_t n, const float* points, float* mean_dist2, void* workspace, size_t workspace_bytes, void* stream);

/* ---- standalone SH (gsplat.sh.spherical_harmonics; gsplat_renderer.py:105) -------------------------------------------
 * dirs[n,3] need not be unit (normalised inside, as gsplat does).  out rgb[n,3] = SH (no +0.5, no clamp).
 * bwd: v_coeffs[n,sh_stride,3] fully written; v_dirs[n,3] nullable. */
B200GS_API int b200gs_sh_fwd(int32_t degree, int32_t sh_stride, int64_t n, const float* dirs, const float* coeffs, float* rgb, void* stream);
B200GS_API int b200gs_sh_bwd(int32_t degree, int32_t sh_stride, int64_t n, const float* dirs, const float* coeffs, const float* v_rgb,
                  float* v_coeffs, float* v_dirs, void* stream);

/* ---- split, masked SH (spherical_harmonics_decomposed of yzslab's gsplat fork) ------------------------------------------
 * Call sites: gsplat_v1_renderer.py:124 (separate_sh), gsplat_appearance_embedding_renderer.py:193,208, glossy_renderer.py:21,
 * gsplat_distributed_renderer.py:419.  The coefficients are dc[n,1,3] | rest[n,k_rest,3] read in place (no concatenation);
 * sh_stride = 1 + k_rest >= (degree+1)^2, rest may be NULL when k_rest = 0.  mask[n] (uint8, nullable): a row with mask[i] == 0
 * reads no coefficient and gets rgb = 0 and zero v_dc / v_rest / v_dirs.  The same kernels as b200gs_sh_fwd / _bwd with another
 * coefficient loader: unmasked rows are bit-identical to those on the concatenated tensor.
 * bwd: v_dc[n,1,3] and v_rest[n,k_rest,3] fully written; v_dirs[n,3] nullable.
 * Algorithmic bytes per unmasked row at degree 3: fwd 12 + 192 in, 12 out; bwd 24 + 192 in (v_dirs), 192 out (+12). */
B200GS_API int b200gs_sh_split_fwd(int32_t degree, int32_t k_rest, int64_t n, const float* dirs, const float* dc, const float* rest,
                                   const uint8_t* mask, float* rgb, void* stream);
B200GS_API int b200gs_sh_split_bwd(int32_t degree, int32_t k_rest, int64_t n, const float* dirs, const float* dc, const float* rest,
                                   const uint8_t* mask, const float* v_rgb, float* v_dc, float* v_rest, float* v_dirs, void* stream);

/* ---- K2-K5: tile binning ------------------------------------------------------------------------------------------
 * replaces dgr InclusiveSum + duplicateWithKeys + SortPairs + identifyTileRanges / gsplat isect_tiles + isect_offset_encode.
 * Result order is exactly that of a stable sort of (tile_id << 32 | float_bits(depth)) keys emitted Gaussian-major:
 * implemented as a stable depth sort of the visible Gaussians, a stable partition of (coarse cell, Gaussian) pairs (a
 * cell = 8x8 tiles) and an order-preserving multi-split of every cell's list into its 64 tiles that writes each id
 * once.  Both sorts are hand-written onesweep-style radix passes (decoupled look-back); no library sort is involved.
 *
 * Counters: d_counts = device int64[4], host_counts = host int64[4] (pinned or pageable; nullable):
 *     [0] number of (tile, Gaussian) pairs of the 3-sigma bounding rects — the reference's pair count, an upper bound
 *         of [2] and equal to it without culling                                              (written by phase A)
 *     [1] number of (coarse cell, Gaussian) pairs                                              (written by phase A)
 *     [2] number of pairs actually listed in sorted_ids / tile_ranges                          (written by phase B)
 *     [3] number of visible Gaussians (non-empty tile rect)                                    (written by phase A)
 *   Each phase ends by delivering d_counts to host_counts (when != NULL) in stream order — pinned/mapped host memory is
 *   written by a tiny kernel with system-scope stores (a D2H copy would queue on a copy engine behind the application's
 *   bulk transfers), pageable memory by cudaMemcpyAsync — and, when sync_host != 0, SYNCHRONISES the stream.
 *   Sync-free use: size max_coarse from the previous view's counts[1] and max_pairs from its counts[0] (the bound is known
 *   after phase A already), pass sync_host = 0, record an event after phase A and check
 *   counts[1] <= max_coarse && counts[0] <= max_pairs once the rest of the forward has been enqueued.
 * cull_conic[n,3] / cull_opacity[n] (both NULL, or both given): exact tile culling.  A (tile, Gaussian) pair is dropped
 *     when no pixel sample of the tile can reach alpha >= 1/255 for that Gaussian (minimum of the conic's quadratic
 *     over the tile box > ln(255*opacity)); the blend loop would have skipped it at every pixel, so images and
 *     gradients do not change while the pair list shrinks ~2x.  With NULL the pair list is exactly the reference's
 *     (every tile of the 3-sigma bounding rect).
 * b200gs_bin_count_workspace_bytes / b200gs_bin_sort_workspace_bytes: bytes of scratch for phase A (n Gaussians) and
 *     phase B (up to max_coarse coarse pairs).  Two buffers because counts[1] is only known after phase A.
 * b200gs_bin_count: phase A.  Compaction of the visible Gaussians, depth keys, stable depth sort; counts[0], [1], [3].  Everything
 *     phase B needs to know about a Gaussian (xy, radius, cull_conic, cull_opacity) is packed into workspace_a, which
 *     must stay untouched until phase B has been enqueued.
 * b200gs_bin_sort: phase B (reads workspace_a only; cull = whether phase A was given the cull arrays).  Writes sorted_ids (Gaussian ids, front to back inside each tile; capacity max_pairs),
 *     tile_ranges[n_tiles,2] (int32 [start,end), clamped to max_pairs) and counts[2].  Coarse pairs beyond max_coarse
 *     and ids beyond max_pairs are DROPPED (never written out of bounds): the caller compares the counters with the
 *     capacities and redoes the phase with larger buffers if either overflowed.  max_pairs = counts[0] and
 *     max_coarse = counts[1] can never overflow. */
B200GS_API size_t b200gs_bin_count_workspace_bytes(int64_t n);
B200GS_API size_t b200gs_bin_sort_workspace_bytes(int64_t n, int64_t max_coarse, int32_t width, int32_t height);
B200GS_API int b200gs_bin_count(int32_t mode, int32_t width, int32_t height, int64_t n, const float* xy, const float* depth,
                     const int32_t* radii, const float* cull_conic, const float* cull_opacity, void* workspace_a, size_t workspace_a_bytes,
                     int64_t* d_counts, int64_t* host_counts, int32_t sync_host, void* stream);
B200GS_API int b200gs_bin_sort(int32_t mode, int32_t width, int32_t height, int64_t n, int32_t cull, int64_t max_coarse, int64_t max_pairs,
                    int64_t* d_counts, const void* workspace_a, void* workspace_b, size_t workspace_b_bytes, int32_t* sorted_ids,
                    int32_t* tile_ranges, int64_t* host_counts, int32_t sync_host, void* stream);

/* ---- gsplat intersection keys and tile offsets of one camera (C = 1) ---------------------------------------------------
 * The gsplat-v1 contract isect_tiles -> isect_offset_encode -> rasterize_to_pixels (gsplat_v1_renderer.py:446,458,500-520,588).
 * b200gs_isect_keys: gsplat's isect_ids of a binning, one per listed pair and in list order:
 *     keys[i] = (int64(tile) << 32) | float_bits(depth[sorted_ids[i]])      (camera bits 0)
 *     tile_ranges[n_tiles,2] / sorted_ids are b200gs_bin_sort's outputs with n_pairs = counts[2]; no range may end past n_pairs.
 *     The binning order is a stable sort of these keys, so they are non-decreasing and, without culling, equal to gsplat's
 *     sorted keys element for element.  A separate pass: the binning never builds them.
 *     Algorithmic bytes: 4 B id + 4 B depth gather (L2) in, 8 B key out per pair; 8 B range per tile.
 * b200gs_isect_offsets: gsplat's isect_offset_encode for C = 1: offsets[t] = index of the first of the n_pairs sorted keys whose
 *     tile (key >> 32) is >= t, for t < n_tiles (an empty tile gets the next non-empty start, tiles past the last key n_pairs;
 *     all 0 when n_pairs = 0).  Computed from the keys alone, by a binary search per tile: O(n_tiles log n_pairs) reads.
 *     n_pairs < 2^31. */
B200GS_API int b200gs_isect_keys(int32_t n_tiles, const int32_t* tile_ranges, const int32_t* sorted_ids, int64_t n_pairs, const float* depth,
                                 int64_t* keys, void* stream);
B200GS_API int b200gs_isect_offsets(int64_t n_pairs, const int64_t* keys, int32_t n_tiles, int32_t* offsets, void* stream);

/* b200gs_publish_i64: deliver n device int64 counters to host memory in stream order, the way the binning phases do
 *     (kernel with system-scope stores for pinned/mapped memory, cudaMemcpyAsync for pageable): for callers that run their
 *     own sync-free capacity protocol (the sharded renderer's row exchange). */
B200GS_API int b200gs_publish_i64(const int64_t* d_values, int64_t* host_values, int32_t n, void* stream);

/* ---- K6: blend forward ---------------------------------------------------------------------------------------------
 * replaces dgr renderCUDA fwd / gsplat rasterize_to_pixels fwd.  channels in {1,2,3,4}.
 * in : xy[n,2] conic[n,3] opacity[n] colors[n,channels]; bg[channels] or NULL.
 * out: image, addressed as image[pixel*pix_stride + channel*ch_stride] (vanilla [C,H,W]: pix_stride 1, ch_stride H*W;
 *      gsplat [H,W,C]: pix_stride C, ch_stride 1); final_T[H*W]; n_contrib[H*W] (1-based position in the tile's list of
 *      the last contributing splat); alpha[H*W] = 1 - final_T (nullable). */
B200GS_API int b200gs_blend_fwd(int32_t mode, int32_t width, int32_t height, int32_t channels, const int32_t* tile_ranges,
                     const int32_t* sorted_ids, const float* xy, const float* conic, const float* opacity,
                     const float* colors, const float* bg, float* image, int64_t pix_stride, int64_t ch_stride,
                     float* final_T, int32_t* n_contrib, float* alpha, void* stream);
/* b200gs_blend_fwd_hits: the same, and hit_any[g] = 1 for every splat g that contributed to at least one pixel (caller zero-fills
 *     hit_any[n]): gsplat's `means2d.has_hit_any_pixels` (optimizers.py:39 SelectiveAdam; gsplat_v1_renderer.py:287 acc_vis). */
B200GS_API int b200gs_blend_fwd_hits(int32_t mode, int32_t width, int32_t height, int32_t channels, const int32_t* tile_ranges,
                     const int32_t* sorted_ids, const float* xy, const float* conic, const float* opacity,
                     const float* colors, const float* bg, float* image, int64_t pix_stride, int64_t ch_stride,
                     float* final_T, int32_t* n_contrib, float* alpha, uint8_t* hit_any, void* stream);

/* ---- K7: blend backward --------------------------------------------------------------------------------------------
 * replaces dgr renderCUDA bwd / gsplat rasterize_to_pixels bwd.
 * in : forward inputs + final_T, n_contrib + v_image (same addressing as image) + v_alpha[H*W] (nullable).
 * out (ACCUMULATED with atomics — caller zero-fills): v_xy[n,2] (pixel units x (xy_scale_x, xy_scale_y)),
 *      v_conic[n,3], v_opacity[n], v_colors[n,channels]; v_xy_abs[n,2] (nullable; sum of |pixel grad|, gsplat absgrad). */
B200GS_API int b200gs_blend_bwd(int32_t mode, int32_t width, int32_t height, int32_t channels, const int32_t* tile_ranges,
                     const int32_t* sorted_ids, const float* xy, const float* conic, const float* opacity,
                     const float* colors, const float* bg, const float* final_T, const int32_t* n_contrib,
                     const float* v_image, int64_t pix_stride, int64_t ch_stride, const float* v_alpha,
                     float xy_scale_x, float xy_scale_y, float* v_xy, float* v_conic, float* v_opacity,
                     float* v_colors, float* v_xy_abs, void* stream);

/* ---- wide feature maps: K6 / K7 for any channel count (gsplat mode) ------------------------------------------------------
 * gsplat rasterize_gaussians with colors [n, D], D >= 1 — the reference's feature renderers composite 32-channel features
 * (internal/segany_splatting.py, seganygs_renderer.py, feature_3dgs_renderer.py).  Processed in chunks of 32 channels over the same
 * tile lists; per channel the arithmetic is K6's, so the composite of every channel is bit-identical to K6 on the same lists.
 * The background is added as one FMA, fmaf(final_T, bg[c], composite); K6 rounds final_T * bg[c] separately for some channels,
 * so with a background a channel may differ from K6's by that one rounding.
 * in : xy[n,2] conic[n,3] opacity[n] features[n,channels] (contiguous); bg[channels] or NULL.
 * fwd out: image[H,W,channels], final_T[H*W], n_contrib[H*W], alpha[H*W] = 1 - final_T (nullable).
 * bwd in : final_T, n_contrib, v_image[H,W,channels], v_alpha[H*W] (nullable).
 * bwd out (ACCUMULATED with atomics — caller zero-fills): v_features[n,channels]; v_xy[n,2] (pixel units), v_conic[n,3],
 *      v_opacity[n] — all three given, or all NULL for the features-only kernel (no geometry work at all); v_xy_abs[n,2]
 *      (nullable, needs v_xy): gsplat absgrad, exact for channels <= 32, the sum of each 32-channel chunk's value beyond. */
B200GS_API int b200gs_blend_feat_fwd(int32_t width, int32_t height, int32_t channels, const int32_t* tile_ranges, const int32_t* sorted_ids,
                                     const float* xy, const float* conic, const float* opacity, const float* features, const float* bg,
                                     float* image, float* final_T, int32_t* n_contrib, float* alpha, void* stream);
B200GS_API int b200gs_blend_feat_bwd(int32_t width, int32_t height, int32_t channels, const int32_t* tile_ranges, const int32_t* sorted_ids,
                                     const float* xy, const float* conic, const float* opacity, const float* features, const float* bg,
                                     const float* final_T, const int32_t* n_contrib, const float* v_image, const float* v_alpha,
                                     float* v_features, float* v_xy, float* v_conic, float* v_opacity, float* v_xy_abs, void* stream);

/* ---- fused L1 + SSIM training loss on the rendered image (validated by tests/test_gpu_loss.py) ----------------------------------
 * replaces  loss = (1-lambda) * l1_loss(image, gt) + lambda * (1 - ssim(image, gt))   (internal/metrics/vanilla_metrics.py:57-74,
 * internal/utils/ssim.py:17-63: 11-tap Gaussian window sigma 1.5, zero padding, C1 = 0.01^2, C2 = 0.03^2).  image/target [C,H,W].
 * b200gs_loss_fwd: partials[b200gs_loss_blocks(...)][2] <- per-CTA sums of |image-target| and of the SSIM map (the caller sums them
 *     and divides by C*H*W); dmaps[3][C][H][W] <- partial derivatives of the SSIM map, kept for the backward.
 * b200gs_loss_bwd: v_image[C,H,W] <- (*v_loss or 1) * dloss/dimage. */
B200GS_API int64_t b200gs_loss_blocks(int32_t channels, int32_t width, int32_t height);
B200GS_API int b200gs_loss_fwd(int32_t channels, int32_t width, int32_t height, const float* image, const float* target, float* dmaps,
                               float* partials, void* stream);
B200GS_API int b200gs_loss_bwd(int32_t channels, int32_t width, int32_t height, const float* image, const float* target, const float* dmaps,
                               float lambda_dssim, const float* v_loss, float* v_image, void* stream);

/* ---- [n,12] splat rows: the exchange format of the Gaussian-sharded multi-GPU renderer ------------------------------
 * replaces the packing / splitting around the reference's all-to-all of projected splats
 * (internal/renderers/gsplat_distributed_renderer.py:127-217): one fp32 row per VISIBLE Gaussian,
 *   col 0-1 xy | 2 depth | 3-5 conic | 6 compensation | 7 opacity | 8-10 rgb | 11 radius (int32 bit pattern).
 * b200gs_pack_rows: compacts the visible (radii > 0) entries of K1's outputs into rows, in index order; row_index[n] (int32)
 *     = the row of entry i, kept for the backward; *d_count <- number of rows.
 * b200gs_bin_count_rows (then b200gs_bin_sort) / blend_fwd_rows / blend_bwd_rows: K2-K7 reading the rows IN PLACE (strided
 *     access, no split copies); blend_bwd_rows accumulates into a zero-filled [n,12] gradient row buffer that goes
 *     straight back through the all-to-all.  3 colour channels; cull != 0 enables exact tile culling.
 *     blend_fwd_rows / blend_bwd_rows read rows (and blend_bwd_rows accumulates into v_rows) with 16-byte accesses: both buffers
 *     must be 16-byte aligned (an allocation base is), or the call fails with B200GS_EINVAL. */
#define B200GS_MAX_VIEWS 8      /* cameras per multi-view launch / destination ranks per peer-mode pack (one NVSwitch box) */
#define B200GS_ROW_FLOATS 12
#define B200GS_ROW_XY 0
#define B200GS_ROW_DEPTH 2
#define B200GS_ROW_CONIC 3
#define B200GS_ROW_COMP 6
#define B200GS_ROW_OPACITY 7
#define B200GS_ROW_RGB 8
#define B200GS_ROW_RADIUS 11
/* Fused activations ("raw parameters"): the K1 / K8 entry points below read the RAW parameter tensors of VanillaGaussianModel
 *     (internal/models/vanilla_gaussian.py:66,345-358; internal/models/gaussian.py:250-254) instead of its getters: scales =
 *     exp(log_scales), quats = normalize(raw_quats), opacity = sigmoid(opacity_logits) (all evaluated inside the kernel, the geometry
 *     part in fp64), SH = shs_dc[n,1,3] | shs_rest[n,sh_stride-1,3] read in place (no torch.cat).  The blend opacity is that opacity
 *     x compensation in gsplat mode when anti_aliased != 0 (gsplat_renderer.py:81-83); gradients are w.r.t. the RAW tensors.
 * b200gs_project_fwd_rows: K1 (fused activations, either constant set) writing ONE [n,12] row per Gaussian instead of the separate
 *     arrays — the single-GPU renderers' fast path: K2-K7 read the rows in place (b200gs_bin_count_rows, b200gs_blend_fwd_rows,
 *     b200gs_blend_bwd_rows), K8 reads the gradient rows (b200gs_project_bwd_rows with row_offsets = NULL).  Rows of culled
 *     Gaussians have radius 0, zeros in columns 0..3 and 8..10 (columns 4..7 unspecified).  radii[n], clamped[n] (what K8 needs) are written too; tiles may be NULL. */
B200GS_API int b200gs_project_fwd_rows(const B200gsView* view, int64_t n, const float* means, const float* log_scales,
                                       const float* raw_quats, const float* opacity_logits, const float* shs_dc, const float* shs_rest,
                                       int32_t anti_aliased, float* rows, int32_t* radii, uint8_t* clamped, int32_t* tiles, void* stream);
/* b200gs_project_bwd_rows: K8 (fused activations) taking its cotangents straight from compacted [V,12] gradient rows
 *     (v_rows[row_offsets[i]] for visible i; row_offsets = NULL: v_rows[i]) and, when accumulate != 0, ADDING to the gradient buffers — the sharded
 *     renderer calls it once per camera of the step without unpack copies or separate sum kernels.
 *     v_mean2d (optional, may be NULL): [n, v_mean2d_cols] (2 or 3 columns) <- dL/dmean2D of every Gaussian (columns 0..1 of its gradient row; zeros
 *     for culled Gaussians and in column 2): the `.grad` of the renderer contract's `viewspace_points` (vanilla_renderer.py:55-56,
 *     vanilla_density_controller.py:101-123), written here instead of by a fill + strided copy after the kernel. */
B200GS_API int b200gs_project_bwd_rows(const B200gsView* view, int64_t n, const float* means, const float* log_scales,
                                       const float* raw_quats, const float* opacity_logits, const float* shs_dc, const float* shs_rest,
                                       int32_t anti_aliased, const int32_t* radii, const uint8_t* clamped, const int32_t* row_offsets,
                                       const float* v_rows, int32_t accumulate, float* v_means, float* v_log_scales, float* v_raw_quats,
                                       float* v_opacity_logits, float* v_shs_dc, float* v_shs_rest, float* v_mean2d, int32_t v_mean2d_cols,
                                       void* stream);
/* b200gs_project_fwd_raw_multi / b200gs_project_bwd_rows_multi: K1 / K8 of one shard for ALL n_views (<= B200GS_MAX_VIEWS) cameras of a
 *     step in one launch each (gsplat constants, raw parameters; sh_degree / sh_stride / scale_modifier of views[0] apply to all).
 *     fwd: camera-major outputs, view j at elements [j*n, (j+1)*n); parameters and SH blocks are read once per Gaussian.
 *     bwd: every thread accumulates its Gaussian's gradients over the cameras in registers and writes them once; cotangents are
 *     [.,12] gradient rows, entry (j, i) reads row row_index[j*n+i] of v_rows[j] — a HOST array of n_views device pointers, each
 *     of which may address a peer GPU's buffer (the camera owner's gradient rows are pulled over NVLink, no return all-to-all). */
B200GS_API int b200gs_project_fwd_raw_multi(const B200gsView* views, int32_t n_views, int64_t n, const float* means, const float* log_scales,
                                            const float* raw_quats, const float* opacity_logits, const float* shs_dc, const float* shs_rest,
                                            int32_t anti_aliased, float* xy, float* depth, int32_t* radii, float* conic, float* rgb,
                                            uint8_t* clamped, float* opacity_out, void* stream);
/* b200gs_project_pack_multi: K1 of one shard for all n_views cameras FUSED with the packing of the exchange.  The visible splats of
 *     camera j leave the kernel as [.,12] rows, in Gaussian-index order, stored straight into dst_rows[j] (a HOST array of n_views device
 *     pointers: block of block_rows rows in the receive buffer of the rank that owns camera j — peer memory over NVLink — or in a local
 *     send buffer); rows past block_rows are dropped.  d_count[j] = visible splats of camera j (compare with block_rows).  Kept locally
 *     for K8 and the renderer contract, camera-major ([j*n + i]): xy (mean2D), radii, clamped, row_index (j*block_rows + k, -1 = dropped).
 *     Replaces b200gs_project_fwd_raw_multi + b200gs_pack_rows (gsplat_distributed_renderer.py:127-217: project, then all-to-all). */
B200GS_API size_t b200gs_project_pack_workspace_bytes(int32_t n_views, int64_t n);
B200GS_API int b200gs_project_pack_multi(const B200gsView* views, int32_t n_views, int64_t n, const float* means, const float* log_scales,
                                         const float* raw_quats, const float* opacity_logits, const float* shs_dc, const float* shs_rest,
                                         int32_t anti_aliased, float* xy, int32_t* radii, uint8_t* clamped, int32_t* row_index,
                                         void* const* dst_rows, int64_t block_rows, void* workspace, size_t workspace_bytes,
                                         int64_t* d_count, void* stream);
B200GS_API int b200gs_project_bwd_rows_multi(const B200gsView* views, int32_t n_views, int64_t n, const float* means, const float* log_scales,
                                             const float* raw_quats, const float* opacity_logits, const float* shs_dc, const float* shs_rest,
                                             int32_t anti_aliased, const int32_t* radii, const uint8_t* clamped, const int32_t* row_index,
                                             const float* const* v_rows, float* v_means, float* v_log_scales, float* v_raw_quats,
                                             float* v_opacity_logits, float* v_shs_dc, float* v_shs_rest, void* stream);
/* b200gs_ipc_alloc / _handle / _open / _close / _free: device buffers that peer processes of the same box can map (cudaMalloc +
 *     CUDA IPC): the exchange buffers of the sharded renderer.  handle = 64 bytes to pass to the peers by any host channel. */
B200GS_API int b200gs_ipc_alloc(size_t bytes, void** dev_ptr, unsigned char* handle64);
B200GS_API int b200gs_ipc_open(const unsigned char* handle64, void** dev_ptr);
B200GS_API int b200gs_ipc_close(void* dev_ptr);
B200GS_API int b200gs_ipc_free(void* dev_ptr);
B200GS_API size_t b200gs_pack_rows_workspace_bytes(int64_t n);
B200GS_API int b200gs_pack_rows(int64_t n, const float* xy, const float* depth, const float* conic, const float* comp, const float* opacity,
                                const float* rgb, const int32_t* radii, void* workspace, size_t workspace_bytes, int32_t* row_index,
                                float* rows, int64_t* d_count, void* stream);
/* b200gs_bin_count_rows reads every row with three 16-byte loads: rows must be 16-byte aligned (an allocation base is), or the call
 *     fails with B200GS_EINVAL.  It always packs the conic and opacity columns for phase B, so its cull argument has no effect: the cull
 *     argument of b200gs_bin_sort decides whether the tiles are culled.
 * block_counts / block_rows (optional; NULL / 0 = every row counts): the rows arrive in blocks of block_rows rows of which only the first
 *     block_counts[b] are valid (the fixed-capacity exchange of the sharded renderer) — the rest reads as culled, so the receive buffer
 *     needs no padding pass. */
B200GS_API int b200gs_bin_count_rows(int32_t mode, int32_t width, int32_t height, int64_t n, const float* rows, int32_t cull,
                                     void* workspace_a, size_t workspace_a_bytes, int64_t* d_counts, int64_t* host_counts,
                                     int32_t sync_host, void* stream, const int64_t* block_counts, int64_t block_rows);
B200GS_API int b200gs_blend_fwd_rows(int32_t mode, int32_t width, int32_t height, const int32_t* tile_ranges, const int32_t* sorted_ids,
                                     const float* rows, const float* bg, float* image, int64_t pix_stride, int64_t ch_stride,
                                     float* final_T, int32_t* n_contrib, float* alpha, void* stream);
/* grad_scale_x / _y: factor on the mean2D columns of the gradient rows (vanilla renderers: 0.5 W, 0.5 H — the vanilla rasterizer's
 *     NDC-unit convention; gsplat renderers: 1, 1).  v_rows must be zero-filled: the kernel accumulates with 128-bit reductions. */
B200GS_API int b200gs_blend_bwd_rows(int32_t mode, int32_t width, int32_t height, const int32_t* tile_ranges, const int32_t* sorted_ids,
                                     const float* rows, const float* bg, const float* final_T, const int32_t* n_contrib,
                                     const float* v_image, int64_t pix_stride, int64_t ch_stride, const float* v_alpha,
                                     float grad_scale_x, float grad_scale_y, float* v_rows, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200GS_H */
