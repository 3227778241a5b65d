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
	const float* filter_3D;      /* [P] or NULL: Mip-Splatting's 3D smoothing filter f >= 0 (DESIGN.md §5o).  Each activated scale
	                                becomes sqrt(s^2 + f^2) (then times scale_modifier) and the opacity sigmoid(logit) * c3,
	                                c3 = sqrt(prod s_k^2 / prod (s_k^2 + f^2)); a row with f == 0 is the unfiltered arithmetic exactly.
	                                The filter is a constant (no gradient).  With a filter the backward reads the opacity logits
	                                (opacities, or quant->ids_opacity).  Not with cov3D_precomp, nor with the statistics forward. */
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

/* ---- the rasterizer: one forward and one backward call, each taking a request ----
 *
 * gsb_forward renders one camera; gsb_backward runs the backward of one forward from the blobs that forward left.  Every option
 * is a field of the request and is absent when NULL or 0, so a zero-initialised request with the leading fields set is the
 * reference's plain forward / backward.  Fully asynchronous on `stream` unless a field says otherwise.
 *
 * Request checks.  Each call checks its request in one order and stops at the first refusal, before any CUDA call: nothing is
 * launched or written.  gsb_last_error() then starts with "forward: " or "backward: ".  The code is GSB_EINVAL except where marked.
 *   Forward:  1. scene NULL or P < 0;  2. features: F outside 1..GSB_FEATURES_MAX, a NULL out, and with P > 0 a NULL
 *             features->features;  3. one map output without the other;  4. statistics: one output without the other, then
 *             statistics together with the maps, antialiasing or raw, then with a scene filter_3D; with deterministic then a NULL
 *             workspace with P > 0, and GSB_ERANGE for width * height >= 2^28;  5. raw parameters: the raw checks (at GsbRawParams);  6. the camera: NULL, a bad
 *             image size, a NULL camera tensor;  7. with P > 0 the scene's tensors (means3D; the codebooks, or opacities and,
 *             without raw parameters, exactly one of shs / colors_precomp and of scales + rotations / cov3D_precomp, then a
 *             filter_3D with cov3D_precomp);
 *             8. out_color, num_rendered, and radii with P > 0.
 *   Backward: 1. scene NULL or P < 0;  2. features: deterministic set, then F outside 1..GSB_FEATURES_MAX, and with P > 0 NULL
 *             features, dL_dout or dL_dfeatures;  3. absgrad: features given, then grads->accumulate set;  4. num_rendered < 0;
 *             5. deterministic: GSB_ERANGE for num_rendered >= 2^30, then det_workspace NULL with P > 0 and num_rendered > 0;
 *             6. a camera output without camera_workspace;  7. raw_grads without raw, then with raw the raw checks;  8. the camera
 *             and the scene as in forward steps 6 and 7;  9. grads NULL;  10. with P > 0 a NULL blob, dL_dout_color or radii, then
 *             a NULL gradient output. */

/* Raw parameters (`pipe.fused_activations`, DESIGN.md §5h): the leaf tensors of the reference's GaussianModel as they are, with
 * get_scaling = exp(_scaling), get_rotation = F.normalize(_rotation) and get_features = cat(_features_dc, _features_rest) applied
 * inside the kernels (exp and the norm in torch's CUDA roundings), so no elementwise pass and no [P,16,3] copy runs in between.
 * All tensors fp32, contiguous, device memory.  With raw parameters the scene keeps P, means3D, opacities, degrees, prune_mask,
 * colors_precomp and scale_modifier; its scales, rotations, shs, cov3D_precomp and quant must be NULL, sh_packed 0, and M is
 * ignored.  Colour, radii, R, the maps, the blobs and every GsbDebug export are bit-identical to the activated call on
 * exp(scaling), F.normalize(rotation) and cat(features_dc, features_rest); so are the backward's per-Gaussian outputs other than
 * the four raw gradients.
 * The raw checks (forward step 5, backward step 7): C not in {0, 3, 8, 15}, a scene field above that must be NULL, and with P > 0
 * NULL scaling / rotation / degrees, or SH pointers that do not match colors_precomp and C; in the backward then grads or raw_grads
 * NULL, a grads field that must be NULL (see GsbRawGrads), and SH gradients that do not match colors_precomp or C. */
typedef struct GsbRawParams {
	const float* features_dc;    /* [P,1,3]  SH coefficient 0; NULL when the scene has colors_precomp                    */
	const float* features_rest;  /* [P,C,3]  SH coefficients 1..C; NULL when C == 0 or with colors_precomp               */
	int32_t C;                   /* rest coefficients per Gaussian: 0, 3, 8 or 15 (max SH degree 0..3)                   */
	const float* scaling;        /* [P,3]    log-scales (_scaling)                                                       */
	const float* rotation;       /* [P,4]    unnormalised quaternions (r,x,y,z) (_rotation)                              */
} GsbRawParams;

/* Gradients w.r.t. the four raw tensors, overwritten (or added to, with GsbGrads.accumulate).  dL_dfeatures_dc / _rest are the
 * SH gradient split at coefficient 1 (zeros outside each Gaussian's active bands; the sparsity sign term on the rest), and may be
 * NULL (then not written; they must be NULL with colors_precomp).  dL_dscaling = dL/ds * s (ExpBackward0's single multiply);
 * dL_drotation is autograd's chain through F.normalize in torch's CUDA roundings (tools/probe_torch_activations.py).
 * With raw_grads, grads->dL_dsh, dL_dscales and dL_drotations must be NULL (raw_grads replaces them); grads->dL_dcov3D and
 * dL_dcolors may be NULL (not written). */
typedef struct GsbRawGrads {
	float* dL_dfeatures_dc;      /* [P,1,3] or NULL */
	float* dL_dfeatures_rest;    /* [P,C,3] or NULL (NULL when C == 0) */
	float* dL_dscaling;          /* [P,3]           */
	float* dL_drotation;         /* [P,4]           */
} GsbRawGrads;

/* Per-Gaussian feature channels (DESIGN.md §5l): features [P,F] fp32, composited exactly like a colour channel with background 0,
 *   out[f](x,y) = sum_i features[i,f] * alpha_i * T_i
 * over the (pixel, Gaussian) pairs of the colour image, with its alpha, T, 1/255 skip and T < 1e-4 stop and the colour kernel's
 * arithmetic: channel f equals the colour channel of a colors_precomp render with bg = 0 and colour features[:,f], bit for bit.
 * The pass reads the forward's own blobs (dense, quantised, raw, anti-aliased, maps, variable-SH inference) and runs no preprocess,
 * binning or sort of its own; the forward's other outputs and its blobs are not modified. */
#define GSB_FEATURES_MAX 256
typedef struct GsbFeatures {
	int32_t F;                   /* channels, 1..GSB_FEATURES_MAX                              */
	const float* features;       /* [P,F]                                                      */
	float* out;                  /* [F,H,W] forward output (unused by the backward)            */
	const float* dL_dout;        /* [F,H,W] backward input (unused by the forward)             */
	float* dL_dfeatures;         /* [P,F]   backward output (unused by the forward)            */
} GsbFeatures;

/* Forward.  Writes out_color [3,H,W] and radii [P]; *num_rendered [host] receives R.
 * The stream is never drained: the instance count (which sizes the binning blob, rasterizer_impl.cu:445-450) is copied to the
 * host in the background while scatter / sort are already queued against the capacity recent frames needed, and the host
 * waits for that copy's EVENT only.  binning_alloc may therefore be called with a size above gsb_binning_bytes(R), and a
 * second time when R outgrew the speculation (the last blob handed out is the one to keep). */
typedef struct GsbForwardRequest {
	const GsbScene* scene;
	const GsbCamera* cam;
	gsb_alloc_fn geom_alloc; void* geom_user;
	gsb_alloc_fn binning_alloc; void* binning_user;
	gsb_alloc_fn image_alloc; void* image_user;
	float* out_color;            /* [3,H,W]                                                                                   */
	int32_t* radii;              /* [P]                                                                                       */
	int64_t* num_rendered;       /* [host] R                                                                                  */
	const GsbDebug* debug;       /* or NULL                                                                                   */
	/* Maps: the inverse-depth and alpha maps, rendered in the same pass as the colour image; both or neither.
	 *   out_invdepth [1,H,W] fp32: invdepth(x,y) = sum_i (1/depth_i) * alpha_i * T_i over exactly the (pixel, Gaussian) pairs that
	 *                composite the colour, with the same alpha and T.  depth_i is the preprocess view-space z (GsbDebug.depths),
	 *                1/depth_i is an IEEE division; no background term, no normalisation by alpha.
	 *   out_alpha    [1,H,W] fp32: 1 - final_T.
	 * P == 0 gives zero maps; a scene with no (Gaussian, tile) instance gives invdepth 0 and alpha 0.  Colour, radii, R and the blobs
	 * are bit-identical to the same request without maps, and the maps are the same bytes on every run. */
	float* out_invdepth;
	float* out_alpha;
	/* Anti-aliasing (the `antialiasing` option of upstream 3DGS: the Mip-Splatting 2D filter), != 0 to enable.  The 0.3 px^2
	 * dilation of cov2D stays; each visible Gaussian's opacity is scaled by s = sqrt(max(2.5e-5, det0 / det1)), det0 = a c - b^2 of
	 * the UNDILATED screen covariance and det1 = (a + 0.3)(c + 0.3) - b^2 of the dilated one, so that its integral no longer grows by
	 * (sigma^2 + 0.3) / sigma^2 when it is smaller than a pixel.  The scaled opacity o^ = sigmoid(logit) * s is what the record, the
	 * 1/255 cull threshold, every pair's alpha and GsbDebug.conic_opacity[:,3] hold.  Radii, tiles, depths, means2D, conic, cov3D,
	 * rgb, clamped, R and the binning are bit-identical to the same request without anti-aliasing; n_contrib, final_T, the colour
	 * and the maps may differ.  The blobs do not record the flag (checking it would need a host synchronisation): the backward of
	 * these blobs must get the same flag, and a mismatched pair gives wrong gradients without an error. */
	int32_t antialiasing;
	const GsbRawParams* raw;     /* or NULL: raw parameters (GsbRawParams)                                                    */
	/* Statistics: the per-Gaussian visibility statistics of the SH-culling pass (forward.cu:560-564 `calculate_mean_transmittance`,
	 * driven by reduced_3dgs.cu:96-152); both or neither.
	 *   touched_pixels[i]    = number of pixels Gaussian i contributed to              (int32 [P], zeroed here)
	 *   transmittance_sum[i] = sum over those pixels of the transmittance T in front   (float [P], zeroed here)
	 * Not together with the maps, antialiasing or raw: the SH-culling statistics keep the reference's definition. */
	int32_t* touched_pixels;
	float* transmittance_sum;
	/* Deterministic statistics (DESIGN.md §5j), deterministic != 0: the same outputs, and the same bytes on every run.  Each per-warp
	 * sum of transmittances is rounded to a multiple of 2^-36 and added as a 64-bit integer, so the order of the additions does not
	 * matter; each total is then rounded to float once (relative error below 1e-7 against the exact sum of the per-warp sums).
	 * workspace: gsb_statistics_workspace_bytes(P) bytes (8 bytes per Gaussian); one workspace serves every camera.  Width * height
	 * must stay below 2^28 (a Gaussian's total, at most width * height, must fit 64 bits at 2^36 per unit).  Without statistics the
	 * flag and the workspace are read by nothing: the colour, maps and feature passes are the same bytes on every run already. */
	int32_t deterministic;
	char* workspace;
	/* Feature channels (GsbFeatures) or NULL: after the render, features->out [F,H,W] receives the feature image of this forward's
	 * blobs (every element; zeros for P == 0 or no instance).  Same bytes on every run. */
	const GsbFeatures* features;
	void* stream;
} GsbForwardRequest;
GSB_API int gsb_forward(const GsbForwardRequest* req);
GSB_API size_t gsb_statistics_workspace_bytes(int32_t P);

/* Backward from the blobs of the paired forward. */
typedef struct GsbBackwardRequest {
	const GsbScene* scene;
	const GsbCamera* cam;
	int64_t num_rendered;        /* R of the paired forward                                                                   */
	const int32_t* radii;        /* [P] of the paired forward                                                                 */
	const char* geom_blob;
	const char* binning_blob;
	const char* image_blob;
	const float* dL_dout_color;  /* [3,H,W]                                                                                   */
	const GsbGrads* grads;
	/* The gradients of the two maps, [1,H,W] fp32 each, each of which may be NULL (= zero).  The maps depend only on the blobs, so
	 * these pair with any forward.  They add to dL_dopacity, dL_dmeans2D, the conic-driven dL_dmeans3D / dL_dscales / dL_drotations /
	 * dL_dcov3D; invdepth also adds its direct term -dL/dinvdepth_i / z_i^2 * (view[2], view[6], view[10]) to dL_dmeans3D.
	 * dL_dcolors and dL_dsh are unchanged. */
	const float* dL_dinvdepth;
	const float* dL_dalpha;
	float lambda_sh_sparsity;
	/* The gradient w.r.t. the camera: dL_dviewmatrix [16], dL_dprojmatrix [16], dL_dcampos [3] (fp32, the transposed layouts of
	 * GsbCamera; each may be NULL).  The camera gradient is the chain rule through the same expressions whose derivatives the
	 * backward already uses for dL_dmeans3D (the 1.3 tan_fov clamp masks of t, the 0.3 dilation of cov2D, the 1e-7 epsilons of the
	 * conic and of 1/w): it is not a finite-difference derivative of the forward.  Per visible Gaussian (t = m . view, T = W J,
	 * ndc = hom.xy * m_w):
	 *   dL/dview[4r+c] = dL/dt_c m_r (r = 0..3, m_3 = 1) + the direct terms through T (r = 0..2);
	 *   dL/dproj[4r+j] for j = 0, 1, 3 through ndc;  dL/dcampos = - the SH view-direction term of dL_dmeans3D.
	 * view[3,7,11,15] and proj[2,6,10,14] are not read by the preprocess: their gradients are exactly 0.  Culled and pruned
	 * Gaussians contribute nothing; P == 0, or no instance, gives zeros.  The camera outputs are always overwritten, also when
	 * grads->accumulate is set (each view has its own camera).  The reduction has a fixed order (per-CTA partial rows in the
	 * workspace, summed in double by one CTA): the same bytes on every run, no host synchronisation.  Per-Gaussian outputs:
	 * dL_dmeans2D (and dL_dmeans2D_view), dL_dcolors, dL_dopacity and dL_dconic are bit-identical to the same request without camera
	 * outputs; the others come from a separately compiled kernel whose multiply-adds may be fused differently and agree to fp32
	 * rounding.
	 * camera_workspace: gsb_camera_grad_workspace_bytes(P) bytes of device memory, required when any camera output is requested. */
	float* dL_dviewmatrix;
	float* dL_dprojmatrix;
	float* dL_dcampos;
	char* camera_workspace;
	/* Anti-aliasing: the forward's flag (see GsbForwardRequest.antialiasing).  dL_dopacity stays the gradient w.r.t. the raw logit;
	 * dL/do^ also reaches cov2D through s, and from there dL_dcov3D, dL_dscales, dL_drotations, dL_dmeans3D and the camera. */
	int32_t antialiasing;
	const GsbRawParams* raw;     /* or NULL: the forward's raw parameters (GsbRawParams)                                      */
	const GsbRawGrads* raw_grads;/* with raw: their gradients (GsbRawGrads)                                                   */
	/* Deterministic backward (DESIGN.md §5i), deterministic != 0: the same gradients as the default backward, summed in a fixed
	 * order, so the same inputs give the same bytes on every run, on any stream and device.  The render backward stores one partial
	 * per (Gaussian, tile) instance instead of adding into the per-Gaussian accumulator with float atomics; a gather adds each
	 * Gaussian's partials in row-major tile order.  No host synchronisation.  A num_rendered > 0 other than the blobs' instance
	 * count makes every accumulated gradient NaN (and no slot beyond num_rendered is written); num_rendered = 0 means nothing was
	 * rendered.  Every mode above has a deterministic form; the feature channels do not.
	 * det_workspace: gsb_deterministic_workspace_bytes(P, num_rendered, absgrad) bytes, absgrad != 0 with dL_dmeans2D_abs (slot
	 * offsets, scan scratch and 40 bytes per instance; with absgrad 8 more per instance). */
	int32_t deterministic;
	char* det_workspace;
	/* Feature channels (GsbFeatures) or NULL: dL_dout [F,H,W] is the gradient of the forward's feature image.  The backward of the
	 * colour image (and maps, camera, raw parameters as above) runs, then the feature image's share is added: dL_dfeatures [P,F]
	 * (overwritten; zero rows for culled and pruned Gaussians) and, through alpha, the same per-Gaussian gradients the colour image
	 * reaches (dL_dopacity, dL_dmeans2D, dL_dmeans3D, dL_dscales / dL_drotations / dL_dcov3D, raw_grads, the camera); dL_dcolors and
	 * the SH gradients are the colour image's alone.  The feature backward sums with float atomics: not with deterministic. */
	const GsbFeatures* features;
	/* Absolute screen-space gradient (AbsGS's homodirectional gradient, gsplat's `absgrad`; DESIGN.md §5m) or NULL: per Gaussian i
	 *   dL_dmeans2D_abs[i] = (0.5 W o_i sum_p |G dL/dalpha (a dx + b dy)|, 0.5 H o_i sum_p |G dL/dalpha (b dx + c dy)|, 0)
	 * over exactly the (pixel, Gaussian) pairs whose signed terms sum to dL_dmeans2D (same skips, same stop), with (a, b, c) the
	 * conic, o_i the (anti-aliased) opacity and (dx, dy) = mean2D - pixel: the sum of the absolute values of the per-pixel terms that
	 * dL_dmeans2D adds with their signs, so a Gaussian over detail whose pixels pull it in opposite directions keeps a large value.
	 * [P,3] fp32, overwritten; zero rows for culled and pruned Gaussians.  Every other output is bit-identical to the same request
	 * without it (deterministic) or agrees within the run-to-run spread of the float atomics (default); with deterministic it is the
	 * same bytes on every run too.  Not with grads->accumulate (there is no view-batch form) nor with features. */
	float* dL_dmeans2D_abs;
	void* stream;
} GsbBackwardRequest;
GSB_API int gsb_backward(const GsbBackwardRequest* req);
GSB_API size_t gsb_camera_grad_workspace_bytes(int32_t P);
GSB_API size_t gsb_deterministic_workspace_bytes(int32_t P, int64_t num_rendered, int32_t absgrad);

/* present[i] = view-space z of means3D[i] > 0.2 (auxiliary.h:139-159). */
GSB_API int gsb_mark_visible(int32_t P, const float* means3D, const float* viewmatrix, const float* projmatrix,
                     uint8_t* present, void* stream);

/* Decode pieces of the private blobs (test / tooling helpers; layouts are private and may change). */
GSB_API int gsb_export_binning(const char* geom_blob, int32_t P, const char* binning_blob, int64_t num_rendered,
                       const char* image_blob, int32_t width, int32_t height,
                       uint64_t* keys_sorted /* tile << 32 | depth bits */, uint32_t* point_list, void* stream);
GSB_API int gsb_export_image(const char* image_blob, int32_t width, int32_t height, float* final_T, uint32_t* n_contrib,
                     uint32_t* ranges /* [tiles,2] */, void* stream);

/* Contribution statistics of one view (DESIGN.md §5p), from the blobs of a finished gsb_forward (any mode: dense, quantised, raw,
 * pruned, anti-aliased, filter_3D, maps, features, variable-SH inference) with its P, R = *num_rendered and image size.  A pair
 * (pixel p, Gaussian i) contributes when the colour forward composited it (list position below n_contrib(p), alpha tests passed);
 * alpha and the transmittance T in front are the forward's bits, and the pair's weight is w = alpha * T (one rounding).  m(p) =
 * pixel_weights [H,W] fp32 clamped to [0, 1] on read (NaN reads as 0), or 1 when pixel_weights is NULL.  Outputs, overwritten:
 *   weight_sum [P] fp32   sum_p m(p) w                     weight_max [P] fp32   max_p w (0 where i contributes nowhere)
 *   pixels     [P] int32  number of contributing pairs (= the statistics forward's touched_pixels)
 *   top_id   [H,W] int32  the id of the pixel's pair with the largest w; on an exact tie the earlier one in the list; -1 where none
 * Culled, pruned and off-screen Gaussians get zeros; P == 0 or R == 0 gives zeros and -1.  Every output is the same bytes on every
 * run: each (warp, Gaussian) sum is rounded to a multiple of 2^-36 and added as a 64-bit integer (so W * H < 2^28), the maximum is
 * an integer maximum on the bits of a non-negative float, the count an integer add.  The blobs are read, not written.
 * workspace: gsb_contributions_workspace_bytes(P) bytes (8 per Gaussian), 8-byte aligned.
 * Errors, before any CUDA call (gsb_last_error() starts with "contributions: "): GSB_EINVAL for P < 0 or num_rendered < 0, width
 * or height < 1; GSB_ERANGE for width * height >= 2^28; GSB_EINVAL for a NULL output (top_id, and with P > 0 the three per-Gaussian
 * ones), a NULL blob with P > 0 or num_rendered > 0, a NULL or misaligned workspace with P > 0. */
GSB_API size_t gsb_contributions_workspace_bytes(int32_t P);
GSB_API int gsb_contributions(const char* geom_blob, int32_t P, const char* binning_blob, int64_t num_rendered, const char* image_blob,
                              int32_t width, int32_t height, const float* pixel_weights /* [H,W] or NULL */, float* weight_sum,
                              float* weight_max, int32_t* pixels, int32_t* top_id, void* workspace, void* stream);

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

/* Mip-Splatting's 3D smoothing filter (Yu et al., CVPR 2024, compute_3D_filter; DESIGN.md §5o) of every centre, for GsbScene.filter_3D.
 * Per centre x and camera c, with (x_v, y_v, z) = x in c's view space (xform_row of the transposed world_view_transform, the
 * preprocess's depth): c sees x if z > 0.2 and u = fl(fl(x_v / max(z, 0.001)) fx) + W/2 lies in [fl32(-0.15 W), fl32(1.15 W)], and
 * the same for v with y_v, fy and H.  dist = the smallest z of the cameras that see x; a centre no camera sees takes the largest
 * dist of the seen centres; f = fl(fl(dist / F) * fl32(sqrt(0.2))) with F the largest fx over ALL cameras (Mip-Splatting's choice,
 * kept).  No seen centre (or no camera): every f is 0.  viewmatrices [n,16] fp32 (world_view_transform, transposed), focals [n,2]
 * fp32 (fx = W / (2 tan(FoVx / 2)), fy likewise), sizes [n,2] int32 (W, H); any number of cameras.  Two launches, asynchronous on
 * `stream`, no host read; the same bytes on every run.  workspace: gsb_filter_3d_workspace_bytes() bytes of device memory.
 * Errors (GSB_EINVAL, nothing launched): P < 0 or P >= 2^30, n_cameras < 0, and with P > 0 a NULL means3D / filter / workspace or,
 * with n_cameras > 0, a NULL camera array. */
GSB_API size_t gsb_filter_3d_workspace_bytes(void);
GSB_API int gsb_filter_3d(int32_t P, const float* means3D, int32_t n_cameras, const float* viewmatrices, const float* focals,
                const int32_t* sizes, float* filter /* [P] */, void* workspace, void* stream);

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
 * the reference supports exactly 256).  workspace: gsb_kmeans_workspace_bytes(n_values, n_centers, deterministic) bytes of device
 * memory, 16-byte aligned with deterministic.  Synchronises the stream every 16 iterations (the reference: every iteration).
 * deterministic != 0 (DESIGN.md §5j): the same sort, assignment and tie rule, update, stopping rule and host poll; only the centre
 * sums change.  Each cluster's values are added in an order that is a function of the input alone (fixed-size chunks and blocks of
 * the sorted values, aligned pairwise trees; not of the grid, SM count, stream or workspace address), so the same input gives the
 * same centres and ids on every run and every H100.
 * Errors (nothing launched; gsb_last_error() starts with "kmeans: "): GSB_EINVAL for n_values < 0, n_centers <= 0 or
 * max_iterations < 0, then NULL centers_in / centers_out or, with n_values > 0, NULL values / ids / workspace, then with
 * deterministic a workspace that is not 16-byte aligned; GSB_ERANGE for n_values >= 2^30; GSB_EINVAL for n_centers > 1024. */
GSB_API size_t gsb_kmeans_workspace_bytes(int64_t n_values, int32_t n_centers, int32_t deterministic);
GSB_API int gsb_kmeans(const float* values, int64_t n_values, const float* centers_in, int32_t n_centers, float tol, int32_t max_iterations,
                int32_t deterministic, int32_t* ids, float* centers_out, char* workspace, void* stream);

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

/* ---- optimizer step (gs_b200.optim.GaussianAdam) ----
 *
 * One Adam step over a table of fp32 tensors, with the arithmetic of torch.optim.Adam's default (foreach) CUDA path, so that
 * param / exp_avg / exp_avg_sq are bit-identical to it (DESIGN.md §5f).  Per entry (scalars are the fp32 casts of the values
 * torch computes in double on the host: one_minus_beta1 = 1 - beta1, one_minus_beta2 = 1 - beta2,
 * bc2_sqrt = (1 - beta2^step)^0.5, step_size = -(lr / (1 - beta1^step))):
 *   m = lerp(m, g, one_minus_beta1);  v = v * beta2;  v = v + one_minus_beta2 * (g * g);
 *   p = p + step_size * (m / (sqrt(v) / bc2_sqrt + eps)).
 * Sparse modes.  With visibility [P] (u8, nonzero = update) and / or degrees [P] (int32, clamped to 0..3) every tensor is a
 * [P, row_width] matrix (numel == P * row_width) and element (i, c) is updated only if visibility[i] and, for an entry with
 * sh_offset = k >= 0 (an [P, C, 3] SH tensor whose column c / 3 is SH coefficient k + c / 3), only if k + c / 3 < (degrees[i] + 1)^2.
 * Skipped elements are neither read nor written.  Both NULL = dense: every element is updated and P is not read.
 * Any contiguous fp32 storage works (128-bit accesses where param, grad and both moments share their 16-byte alignment).
 * All tensors of one call take one kernel launch; none when no element exists.  No host synchronisation; deterministic.
 * Errors (GSB_EINVAL, nothing launched): tensors NULL with n > 0, n outside 0..GSB_ADAM_MAX_TENSORS, P < 0, numel < 0, a NULL
 * pointer of a non-empty entry, sh_offset < -1, sh_offset >= 0 with row_width not a positive multiple of 3, and in a sparse
 * mode row_width <= 0 or numel != P * row_width. */
#define GSB_ADAM_MAX_TENSORS 16
typedef struct GsbAdamTensor {
	float* param;
	const float* grad;
	float* exp_avg;
	float* exp_avg_sq;
	int64_t numel;
	int32_t row_width;        /* elements per row (numel / P); used in the sparse modes                                    */
	int32_t sh_offset;        /* -1: not banded; k >= 0: SH coefficient of column 0 (the reference's f_rest: 1, f_dc: 0)    */
	float one_minus_beta1, beta2, one_minus_beta2, eps, bc2_sqrt, step_size;
} GsbAdamTensor;
GSB_API int gsb_adam_step(const GsbAdamTensor* tensors, int32_t n, int32_t P, const uint8_t* visibility /* NULL = all */,
                const int32_t* degrees /* NULL = all bands */, void* stream);

/* ---- densification (gs_b200.densify) ----
 *
 * The reference's GaussianModel.add_densification_stats / densify_and_prune / prune / prune_points (gaussian_model.py:553-695)
 * as three calls, with the reference's arithmetic and row order (DESIGN.md §5g).  Every pointer is device memory; nothing
 * synchronises with the host; the work runs on `stream`.  All thresholds are the fp32 casts of the Python doubles the reference
 * forms (torch compares an fp32 tensor with a Python number in fp32).
 *
 * gsb_densify_stats: per iteration, for i < P (viewspace_grad is [P, grad_row_stride], its first two columns are read):
 *   xyz_gradient_accum[i] += sqrt(g0*g0 + g1*g1);  denom[i] += visibility[i] != 0;
 *   with radii (may be NULL): if visibility[i], max_radii2D[i] = max(max_radii2D[i], (float)radii[i]).
 * AbsGS (DESIGN.md §5m), for models that also keep xyz_gradient_accum_abs [P] (the norms of gsb_backward's dL_dmeans2D_abs):
 * viewspace_grad_abs and xyz_gradient_accum_abs are both set or both NULL.  When set, the same launch also adds
 *   xyz_gradient_accum_abs[i] += sqrt(a0*a0 + a1*a1) of row i of viewspace_grad_abs ([P, abs_row_stride], first two columns read);
 * denom is counted once.  abs_row_stride is read only with them.
 * Errors (GSB_EINVAL), in this order: P < 0; grad_row_stride < 2; one of viewspace_grad_abs / xyz_gradient_accum_abs without the
 * other (at any P); with them, abs_row_stride < 2; radii without max_radii2D.  Then P == 0 returns GSB_OK without a launch, and
 * with P > 0 a NULL viewspace_grad / visibility / xyz_gradient_accum / denom is refused. */
GSB_API int gsb_densify_stats(int32_t P, const float* viewspace_grad, int32_t grad_row_stride, const float* viewspace_grad_abs,
                int32_t abs_row_stride, const uint8_t* visibility, const int32_t* radii, float* xyz_gradient_accum,
                float* xyz_gradient_accum_abs, float* denom, float* max_radii2D, void* stream);

/* gsb_densify_plan: decides every row of the output and counts them into counts[GSB_DENSIFY_COUNTS] (device int64), which the
 * caller reads back once to size the outputs.  Modes:
 *   GSB_DENSIFY_CLONE_SPLIT  densify_and_prune: grads = accum / denom (NaN -> 0); clone if grads >= max_grad and
 *                            max(exp(scaling)) <= clone_max_scale; split if grads >= max_grad and max(exp(scaling)) > clone_max_scale;
 *                            then prune() over the result with max_radii2D = 0 (the reference has reset it by then).
 *                            With xyz_gradient_accum_abs (AbsGS, DESIGN.md §5m) the split test takes the absolute gradient: split
 *                            if accum_abs / denom >= max_grad_abs (NaN -> 0) and max(exp(scaling)) > clone_max_scale; the clone
 *                            test is as above, so clones are never split.  max_grad_abs is read only with xyz_gradient_accum_abs.
 *   GSB_DENSIFY_PRUNE        prune(): drop sigmoid(opacity) < min_opacity, or with screen_test, max_radii2D > max_screen_size or
 *                            max(exp(scaling)) > big_scale.
 *   GSB_DENSIFY_PRUNE_MASK   prune_points(mask): drop the rows where prune_mask (u8 [P]) is nonzero.
 * Output order: [kept originals][kept clones][kept first children][kept second children].  A split child has the parent's
 * scaling times split_scale_factor (the fp32 reciprocal of 0.8 * N that torch multiplies by) before the log, and is pruned on
 * its own reduced scaling.  The workspace (gsb_densify_workspace_bytes(P) bytes) keeps the plan for gsb_densify_emit and holds
 * exp(scaling) of the split parents, [n_split, 3] fp32 at byte offset gsb_densify_split_std_offset(P), for the caller's draw.
 * Errors (GSB_EINVAL): P < 0 or P >= 2^30, an unknown mode, xyz_gradient_accum_abs with a mode other than
 * GSB_DENSIFY_CLONE_SPLIT, NULL workspace / counts, NULL inputs the mode reads (P > 0). */
#define GSB_DENSIFY_CLONE_SPLIT 0
#define GSB_DENSIFY_PRUNE 1
#define GSB_DENSIFY_PRUNE_MASK 2
#define GSB_DENSIFY_COUNTS 8      /* kept originals, clones, kept clones, split parents, kept children per copy, P', pruned, 0 */
GSB_API size_t gsb_densify_workspace_bytes(int32_t P);
GSB_API size_t gsb_densify_split_std_offset(int32_t P);
GSB_API int gsb_densify_plan(int32_t P, int32_t mode, const float* xyz_gradient_accum, const float* xyz_gradient_accum_abs,
                const float* denom, const float* scaling, const float* opacity, const float* max_radii2D, const uint8_t* prune_mask,
                float max_grad, float max_grad_abs, float clone_max_scale, float min_opacity, int32_t screen_test, float max_screen_size,
                float big_scale, float split_scale_factor, void* workspace, int64_t* counts, void* stream);

/* gsb_densify_emit: writes every output row of every table entry in one launch, from the plan in `workspace` and the counts
 * read back.  Per entry: the [P, row_width] source rows of 4-byte elements (param, and optionally both moments and the grad)
 * go to [P', row_width] destinations.  Kept rows and clones are copies; new rows (clones and children) get zero moments and
 * grads.  Split children copy the parent except for kind GSB_DENSIFY_XYZ (rotation(parent) @ samples[j] + xyz, with
 * samples [2 * n_split, 3] and j = the parent's split rank, + n_split for the second child) and GSB_DENSIFY_SCALING
 * (log(exp(scaling) * split_scale_factor)); XYZ needs rotation [P, 4].  A moment pair or the grad pair is
 * either both NULL (absent) or both set.
 * Errors (GSB_EINVAL, nothing launched): tensors NULL with n > 0, n outside 0..GSB_DENSIFY_MAX_TENSORS, P outside 0..2^30,
 * negative counts, NULL workspace, row_width <= 0, an unknown kind or an XYZ / SCALING entry whose row_width is not 3, a
 * pointer not 4-byte aligned, and when the output has rows (n_kept + n_clones_kept + n_children_kept > 0), a NULL src / dst,
 * a half-given pair or, with children, NULL rotation / samples.  A call without output rows writes nothing. */
#define GSB_DENSIFY_MAX_TENSORS 16
#define GSB_DENSIFY_COPY 0
#define GSB_DENSIFY_XYZ 1
#define GSB_DENSIFY_SCALING 2
typedef struct GsbDensifyTensor {
	const void* src;              /* [P, row_width] 4-byte elements (fp32 params and statistics, int32 degrees)  */
	void* dst;                    /* [P', row_width]                                                             */
	const float* exp_avg_src;     /* moments: NULL pairs = none                                                  */
	float* exp_avg_dst;
	const float* exp_avg_sq_src;
	float* exp_avg_sq_dst;
	const float* grad_src;        /* grad: NULL pair = none                                                      */
	float* grad_dst;
	int32_t row_width;
	int32_t kind;                 /* GSB_DENSIFY_COPY / _XYZ / _SCALING                                          */
} GsbDensifyTensor;
GSB_API int gsb_densify_emit(const GsbDensifyTensor* tensors, int32_t n, int32_t P, const void* workspace, int64_t n_kept,
                int64_t n_clones_kept, int64_t n_split, int64_t n_children_kept, const float* rotation, const float* samples,
                float split_scale_factor, void* stream);

/* ---- resolution-aware redundancy pruning (gs_b200.densify.calculate_redundancy_metric / mercy_points, DESIGN.md §5k) ----
 *
 * gsb_redundancy_score: the reference's Scene.calculate_redundancy_metric (scene/__init__.py:142-174) in one call, fully
 * asynchronous on `stream`:
 *   pixel_sizes[i]   = gsb_min_projected_pixel_size of centre i (the reference's cube_size);
 *   radius[i]        = ((pixel_sizes[i] * pixel_scale) * sqrt(3)) / 2 in fp32;
 *   the K nearest neighbours of each centre (gsb_knn, indices only);
 *   red[i]           = 1 + the number of neighbours n (index >= 0) whose ellipsoid, scales grown by radius[i] and rotated by
 *                      Gaussian i's own rotation (the reference's quirk), contains centre i;
 *   min_redundancy[j] = min(P, red[j], min over the i that hit j of red[i]).
 * scales / rotations are the activated values (exp(scaling), normalised quaternions).  Missing neighbours (P <= K) are neither
 * tested nor counted.  The result is deterministic (integer minima).  workspace: gsb_redundancy_workspace_bytes(P, K) bytes.
 * Errors (GSB_EINVAL, nothing launched): P < 0 or P >= 2^30, K outside 1..GSB_KNN_MAX_K, n_cameras < 0 or > 1024, and with
 * P > 0 a NULL pointer (the camera arrays only when n_cameras > 0). */
GSB_API size_t gsb_redundancy_workspace_bytes(int32_t P, int32_t K);
GSB_API int gsb_redundancy_score(int32_t P, const float* means3D, const float* scales, const float* rotations, int32_t n_cameras,
                const float* w2ndc, const float* w2ndc_inverse, const int32_t* image_heights, const int32_t* image_widths,
                float pixel_scale, int32_t K, int32_t* min_redundancy /* [P] */, float* pixel_sizes /* [P] */, void* workspace,
                void* stream);

/* gsb_mercy_plan: the statistics and the prune mask of the reference's GaussianModel.mercy_points (gaussian_model.py:524-551),
 * asynchronous on `stream`.  counts: int32 [P] (the redundancy score); opacity_logits: fp32 [P] (sigmoid is applied here).
 *   thresholds[0] = mean + lambda_mercy * std of the counts (mean and unbiased variance formed in fp64 from exact integer sums,
 *                   each rounded to fp32, then fp32 ops; exact while sum(c^2) < 2^63);
 *   a row is redundant if (float)count > fp32(max(thresholds[0], mercy_minimum)) (Python's max: a NaN threshold stays NaN);
 *   mask[i] (u8) per type:
 *     GSB_MERCY_REDUNDANCY_OPACITY          redundant and opacity < the lower median of the redundant rows' opacities
 *     GSB_MERCY_REDUNDANCY_RANDOM           redundant and draws[j] < 0.5, j = the row's rank among the redundant rows
 *     GSB_MERCY_OPACITY                     opacity < torch.quantile(opacity, quantile_q)
 *     GSB_MERCY_REDUNDANCY_OPACITY_OPACITY  the first type, or opacity < min(torch.quantile(opacity, quantile_q), 0.05)
 *     GSB_MERCY_REDUNDANCY                  redundant (the reference's branch for any other type string)
 *   thresholds[1] = the opacity threshold of the two quantile types (NaN if an opacity is NaN), else 0;
 *   counts_out[0] = redundant rows, counts_out[1] = masked rows (int64, device).
 * The median is NaN (nothing pruned by it) with no redundant row or a NaN among them.  The quantile has no size limit.
 * The random type is two calls: without draws it writes thresholds and counts_out[0] only; the caller draws counts_out[0]
 * uniforms and calls again with them (n_draws = their number).  workspace: gsb_mercy_workspace_bytes(P) bytes.
 * Errors (GSB_EINVAL, nothing launched): P < 0 or P >= 2^30, an unknown type, NULL workspace / thresholds / counts_out,
 * draws for another type or with n_draws < 0, and with P > 0 NULL counts / mask, or NULL opacity_logits for a type that reads
 * them. */
#define GSB_MERCY_REDUNDANCY_OPACITY 0
#define GSB_MERCY_REDUNDANCY_RANDOM 1
#define GSB_MERCY_OPACITY 2
#define GSB_MERCY_REDUNDANCY_OPACITY_OPACITY 3
#define GSB_MERCY_REDUNDANCY 4
GSB_API size_t gsb_mercy_workspace_bytes(int32_t P);
GSB_API int gsb_mercy_plan(int32_t P, const int32_t* counts, const float* opacity_logits, int32_t type, float lambda_mercy,
                double mercy_minimum, float quantile_q, const float* draws, int64_t n_draws, void* workspace, uint8_t* mask,
                float* thresholds /* [2] */, int64_t* counts_out /* [2] */, void* stream);

/* ---- 3DGS-MCMC densification (gs_b200.mcmc, DESIGN.md §5n) ----
 *
 * Kheradmand et al., "3D Gaussian Splatting as Markov Chain Monte Carlo" (2024): position noise after every optimizer step, and
 * every densification interval the dead Gaussians moved onto live ones and the model grown towards a budget.  Notation:
 * o = sigmoid(opacity_logit) (torch's fp32 sigmoid), s = exp(scaling), q = F.normalize(rotation) (both in torch's fp32 roundings),
 * R(q) = build_rotation(q).  Every call is asynchronous on `stream`; none reads back to the host.
 *
 * gsb_mcmc_noise: for each row i < P, with the gate g = 1 / (1 + exp(-100 ((1 - o) - 0.995))),
 *   xyz[i] += R diag(s)^2 R^T v,   v = draws[i] * g * noise_lr * xyz_lr   (draws [P, 3]: standard-normal samples),
 * evaluated in double from the fp32 inputs (the gate from the fp32 o) and rounded once into xyz.  A row whose gate is 0 when torch
 * evaluates it in fp32 (exp overflows: o above about 0.892) is not written, so it keeps its bytes.  One launch, none for P == 0.
 * Errors (GSB_EINVAL, nothing launched): P < 0 or P >= 2^30, a non-finite noise_lr / xyz_lr, and with P > 0 a NULL pointer. */
GSB_API int gsb_mcmc_noise(int32_t P, float* xyz /* [P,3] */, const float* scaling /* [P,3] */, const float* rotation /* [P,4] */,
                const float* opacity_logits /* [P] */, const float* draws /* [P,3] */, float noise_lr, float xyz_lr, void* stream);

/* gsb_mcmc_plan: samples source rows by opacity and computes their relocated values, in two calls.
 *   Without draws (n = 0): marks the dead rows (GSB_MCMC_RELOCATE: dead_mask[i] != 0, or with dead_mask NULL o <= min_opacity;
 *   GSB_MCMC_ADD: none), weighs the candidate rows (the live rows; with ADD every row) W_i = floor(o_i 2^32) (0 for the others and
 *   for a NaN o), takes the exact inclusive prefix of W in row order and writes counts[GSB_MCMC_COUNTS] (int64, device) = {dead
 *   rows, total weight, 0, 0}.  The caller reads counts back to size the draws.
 *   With draws (int64 [n], uniform on [0, 2^62): torch.randint(0, 2**62, (n,))): draw j selects the first row whose prefix exceeds
 *   floor(d_j * total / 2^62) (a 128-bit product; a draw is taken modulo 2^62), so rows of weight 0 are never selected; a draw
 *   needs total > 0.  With RELOCATE only the first min(n, dead rows) draws are used.  A source row drawn c times gets N = min(c + 1,
 *   50) and (paper eq. 9, in double)
 *     o' = 1 - (1 - o)^(1/N),  D = sum_{i=1..N} sum_{k=0..i-1} C(i-1, k) (-1)^k o'^(k+1) / sqrt(k+1),  s' = s o / D,
 *   then o' is clamped to [0.005, 1 - 2^-23].  N = 1 gives o' = o and s' = s.  The workspace begins (byte offset 0) with a float4
 *   [P] table that holds (o', s'0, s'1, s'2) at every sampled source row before the logit / log gsb_mcmc_emit applies.  Counts per
 *   row are exact (integer atomics) and duplicate sources are resolved here, so the same inputs give the same bytes.
 *   workspace: gsb_mcmc_workspace_bytes(P) bytes; both calls and gsb_mcmc_emit take the same one.
 * Errors (GSB_EINVAL, nothing launched): P < 0 or P >= 2^30, an unknown mode, dead_mask with GSB_MCMC_ADD, NULL workspace, draws
 * with n outside 1..P or no draws with n != 0, NULL counts without draws, with P > 0 NULL opacity_logits, and with draws NULL
 * scaling. */
#define GSB_MCMC_RELOCATE 0
#define GSB_MCMC_ADD 1
#define GSB_MCMC_COUNTS 4         /* dead rows, total weight, 0, 0 */
GSB_API size_t gsb_mcmc_workspace_bytes(int32_t P);
GSB_API int gsb_mcmc_plan(int32_t P, int32_t mode, const float* opacity_logits, const float* scaling, const uint8_t* dead_mask,
                float min_opacity, int64_t n, const int64_t* draws, void* workspace, int64_t* counts, void* stream);

/* gsb_mcmc_emit: writes the rows of the plan's n draws over a GsbDensifyTensor table, in one launch.  A GSB_DENSIFY_SCALING entry
 * (row_width 3) stores log(s'), a GSB_MCMC_OPACITY entry (row_width 1) stores log(o' / (1 - o')) (fp32, torch's roundings), a
 * GSB_DENSIFY_COPY entry copies the source row.
 *   GSB_MCMC_RELOCATE, in place (dst == src, each moment pair's dst == src): dead row j (the j-th in row order) takes draw j's
 *     source row; every sampled source takes its relocated opacity / scaling and its moments are zeroed in every entry that has
 *     them.  The dead rows keep their moments.  Other rows are not written.
 *   GSB_MCMC_ADD, into [P + n, row_width] destinations: row i < P is row i of the source tensor (a sampled row with its relocated
 *     opacity / scaling and zero moments); row P + j is draw j's source row (relocated opacity / scaling) with zero moments.  A
 *     GSB_MCMC_FRESH entry (statistics; no moments) copies rows < P and zeroes the new ones.
 * Errors (GSB_EINVAL, nothing launched): tensors NULL with n_tensors > 0, n_tensors outside 0..GSB_DENSIFY_MAX_TENSORS, P < 0 or
 * P >= 2^30, an unknown mode, n outside 0..P, NULL workspace, row_width <= 0, a kind other than COPY / SCALING / MCMC_OPACITY /
 * MCMC_FRESH, a scaling entry without row_width 3 or an opacity entry without 1, an MCMC_FRESH entry with RELOCATE or with moments,
 * a grad pointer, a half-given moment pair, with P > 0 a NULL src / dst, with RELOCATE dst != src or a moment dst != its src, a
 * pointer not 4-byte aligned. */
#define GSB_MCMC_OPACITY 3
#define GSB_MCMC_FRESH 4
GSB_API int gsb_mcmc_emit(const GsbDensifyTensor* tensors, int32_t n_tensors, int32_t P, int32_t mode, int64_t n, const void* workspace,
                void* stream);

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
