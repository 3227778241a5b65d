/*
 * gs_b200.h — C ABI of the B200-native differentiable Gaussian-splat rasterizer.
 *
 * Drop-in boundary: this library replaces L1+L0 of the reference
 * (graphdeco-inria/reduced-3dgs, submodules/diff-gaussian-rasterization):
 *
 *   gsb_forward        <-  CudaRasterizer::Rasterizer::forward          (cuda_rasterizer/rasterizer.h:33-58,
 *                                                                        rasterizer_impl.cu:359-504) and
 *                          CudaRasterizer::Rasterizer::inferenceForward (rasterizer.h:88-115,
 *                                                                        rasterizer_impl.cu:206-355; set sh_packed)
 *   gsb_backward       <-  CudaRasterizer::Rasterizer::backward         (rasterizer.h:60-86, rasterizer_impl.cu:508-630)
 *   gsb_mark_visible   <-  CudaRasterizer::Rasterizer::markVisible      (rasterizer.h:26-31, rasterizer_impl.cu:149-161)
 *   gsb_alloc_fn       <-  std::function<char*(size_t)> resize callbacks (rasterize_points.cu:33-41 resizeFunctional)
 *
 * The torch-facing functions the reference binds in ext.cpp:17-20 (rasterize_gaussians,
 * rasterize_gaussians_backward, rasterize_gaussians_variableSH_bands, mark_visible; signatures in
 * rasterize_points.h:18-93) are re-hosted in Python on top of these entry points
 * (reduced-3dgs_b200/diff_gaussian_rasterization/_C.py) — see INTEGRATION.md.
 *
 * Conventions: plain pointers and sizes only, no torch / C++ types.  All pointers are DEVICE pointers
 * unless marked [host].  fp32 contiguous tensors with the reference's contracts (SURVEY.md §8(b)):
 * opacities are RAW logits, scales exp-activated, rotations normalised (r,x,y,z), SH is [P,M,3]
 * coefficient-major, matrices are the transposed (row-vector convention) 4x4 the reference passes.
 * A NULL pointer means "absent" exactly where the reference accepts an empty tensor.
 * Every function returns 0 on success; on failure a negative GSB_E* code, with gsb_last_error()
 * giving the message (the reference throws std::runtime_error / AT_ERROR instead).
 * The stream argument is a cudaStream_t passed as void* (0 = legacy default stream).
 */
#ifndef GS_B200_H_INCLUDED
#define GS_B200_H_INCLUDED

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define GSB_API __attribute__((visibility("default")))
#else
#define GSB_API
#endif

#define GSB_OK 0
#define GSB_EINVAL (-1)   /* bad argument (e.g. missing tensor, P < 0)                       */
#define GSB_ECUDA (-2)    /* a CUDA runtime call or kernel failed; see gsb_last_error()      */
#define GSB_ENOMEM (-3)   /* an allocation callback returned NULL                            */
#define GSB_ERANGE (-4)   /* number of (Gaussian,tile) instances does not fit 31 bits        */

#define GSB_NUM_CODEBOOKS 20
#define GSB_CODEBOOK_SIZE 256

/* Scratch allocator: must return a device pointer to at least `nbytes` bytes, 256-byte aligned, that stays
 * valid until the paired backward has run (it is the "geomBuffer / binningBuffer / imgBuffer" the reference
 * returns to Python).  Replaces resizeFunctional, rasterize_points.cu:33-41. */
typedef char* (*gsb_alloc_fn)(void* user, size_t nbytes);

/* Codebook-quantised attributes (reduced-3dgs PLY layout, scene/gaussian_model.py:239-311, 371-387).
 * Fused de-quantisation == centers[ids] of gaussian_model.py:371-387 followed by exp (scaling),
 * normalize (rotation) of gaussian_model.py:141-146; opacity stays a logit (sigmoid is in-kernel anyway). */
typedef struct GsbQuant {
	const uint8_t* ids_dc;       /* [P,3]     codebook 0                                               */
	const uint8_t* ids_rest;     /* [P,15,3]  codebook 1+k for coefficient k (shared by R,G,B)          */
	const uint8_t* ids_opacity;  /* [P]       codebook 16 (centres are logits)                          */
	const uint8_t* ids_scaling;  /* [P,3]     codebook 17 (centres are log-scales)                      */
	const uint8_t* ids_rot;      /* [P,4]     col 0 -> codebook 18 (real), cols 1-3 -> codebook 19      */
	const float* centers;        /* [20,256]  fp32 centres (order: README.md:132-150)                   */
} GsbQuant;

typedef struct GsbScene {
	int32_t P;                   /* number of Gaussians                                                 */
	int32_t M;                   /* SH coefficients per Gaussian in the dense tensor (sh.size(1)); 0 = none */
	const float* means3D;        /* [P,3]                                                               */
	const float* opacities;      /* [P]   raw logits (NULL when quant != NULL)                          */
	const float* scales;         /* [P,3] or NULL                                                       */
	const float* rotations;      /* [P,4] or NULL                                                       */
	const float* cov3D_precomp;  /* [P,6] or NULL (exactly one of scales+rotations / cov3D_precomp)     */
	const float* shs;            /* dense [P,M,3], or packed per-degree groups when sh_packed, or NULL  */
	const float* colors_precomp; /* [P,3] or NULL (exactly one of shs / colors_precomp / quant)         */
	const int32_t* degrees;      /* [P]   active SH degree 0..3 per Gaussian (dense layout)             */
	float scale_modifier;
	int32_t sh_packed;           /* != 0: variable-SH inference layout, forward.cu:19-36 getSHOffset    */
	int32_t band_count[4];       /* [host] perBandPrimitiveCount (Gaussians are ordered by degree)      */
	const uint8_t* prune_mask;   /* [P] or NULL; 1 = pruned: behaves as culled (radii 0, no instances, zero grads) */
	const GsbQuant* quant;       /* [host struct] or NULL; when set, opacities/scales/rotations/shs are ignored */
} GsbScene;

typedef struct GsbCamera {
	int32_t width, height;
	float tan_fovx, tan_fovy;
	const float* viewmatrix;     /* [16] world_view_transform  (transposed)                              */
	const float* projmatrix;     /* [16] full_proj_transform   (transposed)                              */
	const float* campos;         /* [3]                                                                  */
	const float* background;     /* [3]                                                                  */
	int32_t prefiltered;         /* reference flag: a culled Gaussian is then an error (auxiliary.h:150-155) */
} GsbCamera;

/* Optional debug exports of forward intermediates in the REFERENCE's layouts (GeometryState,
 * rasterizer_impl.h:21-42), used by the parity tests; every pointer may be NULL. */
typedef struct GsbDebug {
	float* depths;          /* [P]     */
	float* means2D;         /* [P,2]   */
	float* cov3D;           /* [P,6]   */
	float* conic_opacity;   /* [P,4]   */
	float* rgb;             /* [P,3]   */
	uint32_t* tiles_touched;/* [P]     */
	uint8_t* clamped;       /* [P,3]   */
} GsbDebug;

typedef struct GsbGrads {
	float* dL_dmeans2D;     /* [P,3]  (z = 0)                         rasterize_points.cu:260 */
	float* dL_dcolors;      /* [P,3]                                                     :261 */
	float* dL_dopacity;     /* [P,1]  w.r.t. the raw logit                               :263 */
	float* dL_dmeans3D;     /* [P,3]                                                     :259 */
	float* dL_dcov3D;       /* [P,6]                                                     :264 */
	float* dL_dsh;          /* [P,M,3] (NULL when M == 0)                                :265 */
	float* dL_dscales;      /* [P,3]                                                     :266 */
	float* dL_drotations;   /* [P,4]                                                     :267 */
	float* dL_dconic;       /* [P,4] optional export (reference keeps it internal, :262); may be NULL */
	int32_t accumulate;     /* 0: outputs are overwritten (no caller memset needed). 1: per-view gradients are ADDED
	                           to the buffers (view-batch accumulation for the sharded multi-GPU path, SURVEY §8(e)) */
	float* dL_dmeans2D_view;/* [P,3] optional, accumulate mode only: THIS view's screen-space gradient, overwritten — the
	                           densification statistic is a per-view norm (scene/gaussian_model.py:693-695); may be NULL */
} GsbGrads;

/* Sizes of the three scratch blobs, for callers that pre-allocate.  gsb_image_bytes is the upper bound over all scenes of
 * that image size; gsb_image_bytes_for is what gsb_forward requests for a scene of P Gaussians (quantised != 0: codebook ids). */
GSB_API size_t gsb_geom_bytes(int32_t P);
GSB_API size_t gsb_image_bytes(int32_t width, int32_t height);
GSB_API size_t gsb_image_bytes_for(int32_t P, int32_t width, int32_t height, int32_t quantised);
GSB_API size_t gsb_binning_bytes(int64_t num_rendered);

/* Forward.  Writes out_color [3,H,W] and radii [P]; *num_rendered [host] receives R.
 * The stream is never drained: the instance count (which sizes the binning blob, rasterizer_impl.cu:445-450) is copied to the
 * host in the background while scatter / sort are already queued against the capacity recent frames needed, and the host
 * waits for that copy's EVENT only.  binning_alloc may therefore be called with a size above gsb_binning_bytes(R), and a
 * second time when R outgrew the speculation (the last blob handed out is the one to keep). */
GSB_API int gsb_forward(const GsbScene* scene, const GsbCamera* cam,
                gsb_alloc_fn geom_alloc, void* geom_user,
                gsb_alloc_fn binning_alloc, void* binning_user,
                gsb_alloc_fn image_alloc, void* image_user,
                float* out_color, int32_t* radii, int64_t* num_rendered,
                const GsbDebug* debug, void* stream);

/* Forward that also gathers the per-Gaussian visibility statistics of the SH-culling pass
 * (forward.cu:560-564 `calculate_mean_transmittance`, driven by reduced_3dgs.cu:96-152):
 *   touched_pixels[i]    = number of pixels Gaussian i contributed to              (int32 [P], zeroed here)
 *   transmittance_sum[i] = sum over those pixels of the transmittance T in front   (float [P], zeroed here)
 * Everything else as gsb_forward. */
GSB_API int gsb_forward_statistics(const GsbScene* scene, const GsbCamera* cam,
                gsb_alloc_fn geom_alloc, void* geom_user,
                gsb_alloc_fn binning_alloc, void* binning_user,
                gsb_alloc_fn image_alloc, void* image_user,
                float* out_color, int32_t* radii, int64_t* num_rendered,
                int32_t* touched_pixels, float* transmittance_sum, void* stream);

/* Backward from the blobs of the paired forward.  Fully asynchronous on `stream`. */
GSB_API int gsb_backward(const GsbScene* scene, const GsbCamera* cam, int64_t num_rendered, const int32_t* radii,
                 const char* geom_blob, const char* binning_blob, const char* image_blob,
                 const float* dL_dout_color /* [3,H,W] */, const GsbGrads* grads,
                 float lambda_sh_sparsity, void* stream);

/* present[i] = view-space z of means3D[i] > 0.2 (auxiliary.h:139-159). */
GSB_API int gsb_mark_visible(int32_t P, const float* means3D, const float* viewmatrix, const float* projmatrix,
                     uint8_t* present, void* stream);

/* Decode pieces of the private blobs (test / tooling helpers; layouts are private and may change). */
GSB_API int gsb_export_binning(const char* geom_blob, int32_t P, const char* binning_blob, int64_t num_rendered,
                       const char* image_blob, int32_t width, int32_t height,
                       uint64_t* keys_sorted /* tile << 32 | depth bits */, uint32_t* point_list, void* stream);
GSB_API int gsb_export_image(const char* image_blob, int32_t width, int32_t height, float* final_T, uint32_t* n_contrib,
                     uint32_t* ranges /* [tiles,2] */, void* stream);

/* Test helper: the fused de-quantisation on its own -> activated scales [P,3], normalised rotations [P,4]. */
GSB_API int gsb_debug_dequant(const GsbQuant* quant, int32_t P, float* scales, float* rotations, void* stream);

/* ---- reduced-3dgs tools on either side of the rasterizer (reference reduced_3dgs.h:19-67, bound in ext.cpp:21-25) ----
 *
 * One camera's update of the SH-culling colour statistics (the body of the camera loop of
 * Reduced3DGS::calculateColourVariance, reduced_3dgs.cu:150-201, with calculateColourCUDA of reduced_3dgs/sh_culling.cu fused in):
 * t = transmittance_sum / max(touched_pixels, 1); weight_sum += t; weight_sq_sum += t^2;
 * distance_accum[P,3] += t * ||colour(deg 3) - colour(deg d)||; mean[P,3] / variance[P,3] updated for visible Gaussians (radii > 0).
 * shs is the dense [P,M,3] tensor with M >= 16 (the reference hard-codes a 4-slot colour table, i.e. max_sh_degree = 3). */
GSB_API int gsb_sh_statistics_update(int32_t P, int32_t M, const int32_t* degrees, const float* means3D, const float* campos /* [3] */,
                const float* shs, const int32_t* radii, const int32_t* touched_pixels, const float* transmittance_sum,
                float* weight_sum /* [P] */, float* weight_sq_sum /* [P] */, float* distance_accum /* [P,3] */,
                float* mean /* [P,3] */, float* variance /* [P,3] */, void* stream);

/* pixel_sizes[i] = min over cameras of the world-space length of one pixel at Gaussian centre i, 10000 if no camera sees it
 * (Reduced3DGS::calculatePixelSize, reduced_3dgs.cu:246-268 + transformCentersNDCCUDA, redundancy_score.cu:45-101).
 * w2ndc / w2ndc_inverse: [n_cameras,4,4] exactly as the reference passes them; heights / widths: int32 [n_cameras] on the device. */
GSB_API int gsb_min_projected_pixel_size(int32_t P, const float* means3D, int32_t n_cameras, const float* w2ndc, const float* w2ndc_inverse,
                const int32_t* image_heights, const int32_t* image_widths, float* pixel_sizes /* [P] */, void* stream);

/* redundancy_values[i] = number of the knn neighbours whose (scale + sphere_radius[i]) ellipsoid contains centre i,
 * intersection_mask[i,k] = that test per neighbour (Reduced3DGS::intersectionTest, reduced_3dgs.cu:205-243 +
 * sphereEllipsoidIntersectionCUDA / buildRotationMatrixCUDA, redundancy_score.cu:119-205). */
GSB_API int gsb_sphere_ellipsoid_intersection(int32_t P, const float* means3D, const float* scales, const float* rotations,
                const int32_t* neighbours /* [P,knn] */, const float* sphere_radius /* [P] */, int32_t knn,
                int32_t* redundancy_values /* [P] */, uint8_t* intersection_mask /* [P,knn] */, void* stream);

/* minimum_redundancy_values[n] = min(P, min over (i,k) with intersection_mask[i,k] and neighbours[i,k] == n of redundancy_values[i])
 * (Reduced3DGS::assignFinalRedundancyValue, reduced_3dgs.cu:270-287 + findMinimumRedundancyValueCUDA, redundancy_score.cu:6-27). */
GSB_API int gsb_min_redundancy_value(int32_t P, const int32_t* redundancy_values, const int32_t* neighbours, const uint8_t* intersection_mask,
                int32_t knn, int32_t* minimum_redundancy_values /* [P] */, void* stream);

/* 1-D k-means of the codebook quantisation (Reduced3DGS::kmeans, reduced_3dgs.cu:289-338 + reduced_3dgs/kmeans.cu):
 * Lloyd iterations from centers_in until sum|old - new| < tol or max_iterations, then ids[i] = index of the nearest centre
 * (smallest sqrt((c - v)^2), first index on ties).  ids: int32 [n_values]; centers_out: float [n_centers] (n_centers <= 1024;
 * the reference supports exactly 256).  workspace: gsb_kmeans_workspace_bytes(n_values, n_centers) bytes of device memory.
 * Synchronises the stream every 16 iterations (the reference: every iteration). */
GSB_API size_t gsb_kmeans_workspace_bytes(int64_t n_values, int32_t n_centers);
GSB_API int gsb_kmeans(const float* values, int64_t n_values, const float* centers_in, int32_t n_centers, float tol, int32_t max_iterations,
                int32_t* ids, float* centers_out, char* workspace, void* stream);

/* Exact k nearest neighbours of points [P,3] (fp32) — the reference's second extension simple_knn._C (submodules/simple-knn:
 * distCUDA2, distIndex2, distIndexQ).  Squared distances d = (p - q).(p - q) evaluated as the reference evaluates them; the query
 * itself (by index, not by value: an exact duplicate counts at distance 0) is never its own neighbour.
 *   n_queries < 0: every point is a query and row i belongs to point i (query_ids unused); else row t belongs to query_ids[t], and a
 *                  query id outside [0, P) gives a row of (FLT_MAX, -1).
 *   n_candidates < 0: every point is a candidate (candidate_ids unused); else only the points listed in the first min(n_candidates,
 *                  P) entries of candidate_ids (the reference's fillIndex2Pos quirk); ids outside [0, P) are ignored.
 *   dists [rows*K] / indices [rows*K] (each may be NULL): row r holds its K nearest as (distance, index) ascending, ties by the
 *                  smaller index; missing neighbours are (FLT_MAX, -1).
 *   mean3 [rows] (may be NULL; needs K == 3): ((d0 + d1) + d2) / 3, the reference's distCUDA2.
 * 0 <= K <= GSB_KNN_MAX_K, P < 2^30, n_queries < 2^30.  workspace: gsb_knn_workspace_bytes(P, n_queries) bytes of device memory.  Fully asynchronous on `stream`
 * (no host synchronisation).  The result is a function of the points alone: identical bytes from run to run. */
#define GSB_KNN_MAX_K 64
GSB_API size_t gsb_knn_workspace_bytes(int32_t P, int32_t n_queries);
GSB_API int gsb_knn(const float* points, int32_t P, int32_t K, const int32_t* query_ids, int32_t n_queries, const int32_t* candidate_ids,
                int32_t n_candidates, float* mean3, float* dists, int32_t* indices, char* workspace, void* stream);

/* Loss side of the training step: (1 - lambda) * L1 + lambda * (1 - SSIM) of image vs gt, both [C,H,W] fp32
 * (reference utils/loss_utils.py:17-65 l1_loss / ssim with the 11x11 sigma-1.5 window and zero padding, combined as in
 * train.py:110-115).  Forward writes maps [3,C,H,W] (d ssim / d mu_x, E[x^2], E[xy]) and per-CTA partial sums
 * [gsb_l1_ssim_blocks(C,H,W)][2] = (sum of the SSIM map, sum |x - y|); the caller adds them up:
 *   ssim = sum(partial[:,0]) / (C H W),  l1 = sum(partial[:,1]) / (C H W).
 * Backward: dL/dimage = coef_l1 * (*upstream_l1) * d l1/dimage + coef_ssim * (*upstream_ssim) * d ssim/dimage; the upstreams are
 * DEVICE scalars (NULL = 1), so autograd's incoming gradients are consumed without a host synchronisation.  For the combined
 * loss (1 - lambda) l1 + lambda (1 - ssim): coef_l1 = 1 - lambda, coef_ssim = -lambda, both upstreams = dL/dloss. */
GSB_API int64_t gsb_l1_ssim_blocks(int32_t channels, int32_t height, int32_t width);
GSB_API int gsb_l1_ssim_forward(const float* image, const float* gt, int32_t channels, int32_t height, int32_t width,
                float* maps, float* partial_sums, void* stream);
GSB_API int gsb_l1_ssim_backward(const float* image, const float* gt, int32_t channels, int32_t height, int32_t width,
                const float* maps, float coef_l1, const float* upstream_l1, float coef_ssim, const float* upstream_ssim,
                float* dL_dimage, void* stream);

/* Number of kernels this library has launched since load (bench.py reports it as gpu_launches). */
GSB_API uint64_t gsb_launch_count(void);

/* Per-kernel device timing: when enabled, every kernel launch is bracketed by CUDA events on its stream;
 * gsb_profile_read() waits for them, returns per-kernel totals since the previous read and resets.
 * names[i] points to a static string. Returns the number of entries written. */
GSB_API void gsb_profile_enable(int on);
GSB_API int gsb_profile_read(int max_entries, const char** names, double* total_ms, uint64_t* launches);

GSB_API const char* gsb_last_error(void);
GSB_API const char* gsb_version(void);

#ifdef __cplusplus
}
#endif
#endif /* GS_B200_H_INCLUDED */
