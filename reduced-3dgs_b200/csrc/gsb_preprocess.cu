// gsb_preprocess.cu — fused per-Gaussian forward preprocess (sm_90a).
//
// Replaces reference forward.cu:354-456 preprocessCUDA, forward.cu:246-350 variableSHPreprocessCUDA and
// rasterizer_impl.cu:62-74 checkFrustum.  The reduced-3dgs extras are fused here so no PyTorch elementwise
// pass runs: per-Gaussian variable-degree SH (dense or packed layout), the prune mask, and the Gaussian's inputs in any of the three
// formats (activated, codebook ids with the 20 x 256 table staged in shared memory once per persistent block, raw parameters),
// read, activated and filtered by gsb_common.cuh GaussianReader exactly as the backward reads them.
// One 48-byte render record per visible Gaussian is written (see gsb_common.cuh GeomState).
#include "gsb_common.cuh"

namespace gsb {

struct PreArgs {
	SceneArgs s;
	int gx, gy;
	int packed; int cum[4]; long long group_base[4];   // packed SH: first vec3 index of each degree group
	const uint8_t* prune;
	GeomState g; int32_t* radii; uint32_t* tile_count;
	int hist_priv, chunk, T; uint32_t* cta_count;      // privatised tile counting (gsb_common.cuh BinPlan)
	int sh_vec4;                                       // dense fp32 SH rows can be read as 12 float4 (M == 16, 16-byte aligned)
	int rest_aligned;                                  // QUANT: ids_rest is 16-byte aligned (warp-cooperative staging allowed)
	GsbDebug dbg; int prefiltered;
};

// forward.cu:105-159 computeColorFromSH with the accumulation order of the reference build
// (oracle/gs_oracle.cpp color_from_sh).  sh(k, c) returns coefficient k, channel c.
template <class SH>
__device__ __forceinline__ void sh_to_rgb(int deg, float x, float y, float z, SH sh, float* res)
{
#pragma unroll
	for (int c = 0; c < 3; c++) res[c] = __fmul_rn(kSH_C0, sh(0, c));
	if (deg > 0)
	{
		const float c1y = __fmul_rn(y, kSH_C1), c1z = __fmul_rn(z, kSH_C1), c1x = __fmul_rn(x, kSH_C1);
#pragma unroll
		for (int c = 0; c < 3; c++)
		{
			float t = __fmaf_rn(-c1y, sh(1, c), res[c]);
			t = __fmaf_rn(c1z, sh(2, c), t);
			res[c] = __fmaf_rn(-c1x, sh(3, c), t);
		}
		if (deg > 1)
		{
			const float xx = __fmul_rn(x, x), yy = __fmul_rn(y, y), zz = __fmul_rn(z, z);
			const float xy = __fmul_rn(x, y), yz = __fmul_rn(y, z), xz = __fmul_rn(x, z);
			const float zz2 = __fadd_rn(zz, zz);
			const float w4 = __fmul_rn(xy, kSH_C2[0]), w5 = __fmul_rn(yz, kSH_C2[1]);
			const float w6 = __fmul_rn(__fsub_rn(__fsub_rn(zz2, xx), yy), kSH_C2[2]);
			const float w7 = __fmul_rn(xz, kSH_C2[3]), w8 = __fmul_rn(__fsub_rn(xx, yy), kSH_C2[4]);
#pragma unroll
			for (int c = 0; c < 3; c++)
			{
				float t = __fmaf_rn(w4, sh(4, c), res[c]);
				t = __fmaf_rn(w5, sh(5, c), t);
				t = __fmaf_rn(w6, sh(6, c), t);
				t = __fmaf_rn(w7, sh(7, c), t);
				res[c] = __fmaf_rn(w8, sh(8, c), t);
			}
			if (deg > 2)
			{
				const float q = __fsub_rn(__fmaf_rn(zz, 4.0f, -xx), yy);
				const float w9 = __fmul_rn(__fmul_rn(y, kSH_C3[0]), __fmaf_rn(xx, 3.0f, -yy));
				const float w10 = __fmul_rn(__fmul_rn(xy, kSH_C3[1]), z);
				const float w11 = __fmul_rn(__fmul_rn(y, kSH_C3[2]), q);
				const float w12 = __fmul_rn(__fmul_rn(z, kSH_C3[3]), __fmaf_rn(yy, -3.0f, __fmaf_rn(xx, -3.0f, zz2)));
				const float w13 = __fmul_rn(__fmul_rn(x, kSH_C3[4]), q);
				const float w14 = __fmul_rn(__fmul_rn(z, kSH_C3[5]), __fsub_rn(xx, yy));
				const float w15 = __fmul_rn(__fmul_rn(x, kSH_C3[6]), __fmaf_rn(yy, -3.0f, xx));
#pragma unroll
				for (int c = 0; c < 3; c++)
				{
					float t = __fmaf_rn(w9, sh(9, c), res[c]);
					t = __fmaf_rn(w10, sh(10, c), t);
					t = __fmaf_rn(w11, sh(11, c), t);
					t = __fmaf_rn(w12, sh(12, c), t);
					t = __fmaf_rn(w13, sh(13, c), t);
					t = __fmaf_rn(w14, sh(14, c), t);
					res[c] = __fmaf_rn(w15, sh(15, c), t);
				}
			}
		}
	}
}


// Load-path notes (the kernel is bound by L1 wavefronts, not by HBM).  A warp-wide 1- or 4-byte load
// whose lanes are 45 B (codebook ids) or 192 B (fp32 SH row) apart touches one 128-byte line per lane and costs up to 32
// L1 wavefronts; 45 such loads per Gaussian for the ids, 48 for a degree-3 SH row.  Hence:
//   * fp32 SH rows (M == 16) are read with 128-bit loads straight from the row (12 instead of 48 load instructions);
//   * the u8 ids of the SH rest coefficients are copied by the whole warp with 16-byte unit-stride loads (1440 contiguous bytes
//     per 32 Gaussians) into a per-warp shared-memory buffer and picked up from there;
//   * the four rotation ids are one 32-bit load.
#define IDS_REST_ROW 45
static_assert(32 * IDS_REST_ROW == GSB_IDS_STAGE_BYTES_PER_WARP, "staging buffer size");

// AA (anti-aliasing, DESIGN.md §5e): the opacity is scaled by aa_opacity_factor() of the undilated and dilated cov2D, everywhere
// the forward uses it (record r1.z, the cull threshold pth, the debug export).  Nothing else in the record, radii, rects or depths
// changes, so binning is the same as without it.
// IN (gsb_common.cuh InputMode): GaussianReader activates the inputs; IN_RAW reads SH coefficient k from _features_dc (k == 0) or
// _features_rest (k >= 1): the same values as the activated tensors, bit for bit.
// F3D (Mip-Splatting's 3D filter, DESIGN.md §5o): the reader filters the scales before the covariance, and the sigmoid is
// multiplied by its c3 before the AA factor, so everything downstream sees the filtered scale and opacity.
template <int IN, bool AA, bool F3D>
__global__ void __launch_bounds__(1024, 1) preprocess_kernel(const PreArgs a)
{
	constexpr bool QUANT = IN == IN_QUANT, RAW = IN == IN_RAW;
	extern __shared__ __align__(16) float s_cb[];   // QUANT: [20][256] centres; scaling row holds exp(centre)
	if (QUANT) stage_codebooks(a.s.q.centers, s_cb);
	uint32_t* s_hist = reinterpret_cast<uint32_t*>(s_cb + (QUANT ? GSB_NUM_CODEBOOKS * GSB_CODEBOOK_SIZE : 0));
	// QUANT: per-warp staging buffer of the rest-coefficient ids behind the histogram (16-byte aligned: T * 4 rounded up)
	uint8_t* s_rest = reinterpret_cast<uint8_t*>(s_hist + ((a.hist_priv ? a.T : 0) + 3) / 4 * 4) + (threadIdx.x >> 5) * (32 * IDS_REST_ROW);
	if (a.hist_priv)
	{
		for (int t = threadIdx.x; t < a.T; t += blockDim.x) s_hist[t] = 0;
		__syncthreads();
	}
	const int lane = threadIdx.x & 31;
	unsigned block_vis = 0;
	// privatised counting: CTA c owns the contiguous Gaussians [c*chunk, (c+1)*chunk) (the scatter kernel uses the same map)
	const long long first = a.hist_priv ? (long long)blockIdx.x * a.chunk : (long long)blockIdx.x * blockDim.x;
	const long long last = a.hist_priv ? min((long long)a.s.P, first + a.chunk) : (long long)a.s.P;
	const long long stride = a.hist_priv ? (long long)blockDim.x : (long long)gridDim.x * blockDim.x;
	for (long long base = first; base < last; base += stride)
	{
		const long long idx = base + threadIdx.x;
		bool visible = false;
		uint32_t tiles = 0; int radius_i = 0;
		uint2 rect = make_uint2(0, 0);
		float tz = 0.f, conx = 0.f, cony = 0.f, conz = 0.f, opacity = 0.f, pix_x = 0.f, pix_y = 0.f;
		float cov3D[6];
		GaussianReader<IN, F3D> in;
		uint32_t idc0 = 0, idc1 = 0, idc2 = 0;
		// ---- geometry: cull, project, covariance, radius, tile rectangle --------------------------------
		// A culled Gaussian costs ~16 wasted bytes of inputs requested up front (GaussianReader::load) instead of a stalled warp.
		if (idx < last)
		{
			const bool pruned = a.prune && a.prune[idx];
			in.load(a.s, idx, !a.s.colors_precomp && (QUANT || !a.packed));
			in.load_opacity(a.s, idx);
			if (QUANT && !a.s.colors_precomp) { const uint8_t* idc = a.s.q.ids_dc + 3 * idx; idc0 = idc[0]; idc1 = idc[1]; idc2 = idc[2]; }
			do {
				if (pruned) break;                                                        // pruned == culled
				tz = xform_row(a.s.view, 2, in.mx, in.my, in.mz);                     // auxiliary.h:139-159
				if (tz <= 0.2f)
				{
					if (a.prefiltered) atomicExch(&a.g.counters[3], 1u);
					break;
				}
				const float hx = xform_row(a.s.proj, 0, in.mx, in.my, in.mz);
				const float hy = xform_row(a.s.proj, 1, in.mx, in.my, in.mz);
				const float hw = xform_row(a.s.proj, 3, in.mx, in.my, in.mz);
				const float p_w = __frcp_rn(__fadd_rn(hw, 0.0000001f));
				const float projx = __fmul_rn(hx, p_w), projy = __fmul_rn(hy, p_w);
				const GaussianActive act = in.activate(a.s, s_cb, idx);
				for (int k = 0; k < 6; k++) cov3D[k] = act.cov3D[k];
				opacity = act.sigmoid;
				if (F3D) opacity = __fmul_rn(opacity, act.c3);
				const float tx = xform_row(a.s.view, 0, in.mx, in.my, in.mz), ty = xform_row(a.s.view, 1, in.mx, in.my, in.mz);
				const float3 cov_u = compute_cov2D_undilated(tx, ty, tz, a.s.focal_x, a.s.focal_y, a.s.tan_fovx, a.s.tan_fovy, cov3D, a.s.view);
				const float3 cov = dilate_cov2D(cov_u);
				const float det = __fmaf_rn(cov.x, cov.z, -__fmul_rn(cov.y, cov.y));   // forward.cu:419
				if (det == 0.0f) break;
				if (AA) opacity = __fmul_rn(opacity, aa_opacity_factor(cov_u, det));
				const float det_inv = __frcp_rn(det);
				conx = __fmul_rn(cov.z, det_inv); cony = __fmul_rn(-cov.y, det_inv); conz = __fmul_rn(cov.x, det_inv);
				const float mid = __fmul_rn(0.5f, __fadd_rn(cov.x, cov.z));
				const float sq = __fsqrt_rn(fmaxf(0.1f, __fmaf_rn(mid, mid, -det)));
				const float lambda1 = __fadd_rn(mid, sq), lambda2 = __fsub_rn(mid, sq);
				const float my_radius = ceilf(__fmul_rn(3.0f, __fsqrt_rn(fmaxf(lambda1, lambda2))));
				pix_x = ndc2pix(projx, a.s.W); pix_y = ndc2pix(projy, a.s.H);
				uint2 rmin, rmax;
				get_rect(pix_x, pix_y, (int)my_radius, a.gx, a.gy, rmin, rmax);
				if ((rmax.x - rmin.x) * (rmax.y - rmin.y) == 0) break;
				radius_i = (int)my_radius;
				tiles = (rmax.y - rmin.y) * (rmax.x - rmin.x);
				rect = TileRect::pack(rmin, rmax);
				visible = true;
			} while (false);
		}
		// ---- colour -----------------------------------------------------------------------------------
		const bool want_sh = visible && !a.s.colors_precomp;
		int deg = 0;
		if (want_sh)
		{
			if (!QUANT && a.packed)
			{
				// forward.cu:19-36 getSHOffset: degree follows from the position in the degree-sorted list
				if (idx >= a.cum[0]) deg = 1;
				if (idx >= a.cum[1]) deg = 2;
				if (idx >= a.cum[2]) deg = 3;
			}
			else deg = in.deg;
		}
		bool staged = false;
		if (QUANT)
		{
			// the warp's 32 rows of rest-coefficient ids are 1440 contiguous bytes: copy them with unit-stride 16-byte loads
			// (full warps only — the array's last, partial warp reads its bytes directly; rest_aligned: the base pointer is 16-byte aligned)
			const long long wbase = idx - lane;
			if (__any_sync(0xffffffffu, want_sh && deg > 0) && a.rest_aligned && wbase + 32 <= (long long)a.s.P)
			{
				const uint4* src = reinterpret_cast<const uint4*>(a.s.q.ids_rest + wbase * IDS_REST_ROW);
				uint4* dst = reinterpret_cast<uint4*>(s_rest);
				__syncwarp();
#pragma unroll
				for (int c = lane; c < 32 * IDS_REST_ROW / 16; c += 32) dst[c] = __ldcs(src + c);
				__syncwarp();
				staged = true;
			}
		}
		if (visible)
		{
			float rgb[3]; unsigned clamp_bits = 0;
			if (a.s.colors_precomp)
			{
#pragma unroll
				for (int c = 0; c < 3; c++) rgb[c] = a.s.colors_precomp[3 * idx + c];
			}
			else
			{
				const float dx0 = __fsub_rn(in.mx, a.s.campos[0]), dy0 = __fsub_rn(in.my, a.s.campos[1]), dz0 = __fsub_rn(in.mz, a.s.campos[2]);
				float l2 = __fmul_rn(dy0, dy0);
				l2 = __fmaf_rn(dx0, dx0, l2); l2 = __fmaf_rn(dz0, dz0, l2);
				const float len = __fsqrt_rn(l2);
				const float dx = __fdiv_rn(dx0, len), dy = __fdiv_rn(dy0, len), dz = __fdiv_rn(dz0, len);
				float res[3];
				if (QUANT)
				{
					const float dc[3] = { s_cb[idc0], s_cb[idc1], s_cb[idc2] };
					// two call sites: one pointer select for both would turn the staged shared-memory loads into generic loads
					if (staged)
					{
						const uint8_t* irest = s_rest + lane * IDS_REST_ROW;
						sh_to_rgb(deg, dx, dy, dz, [&](int k, int c) { return quant_sh(s_cb, dc[c], irest, k, c); }, res);
					}
					else
					{
						const uint8_t* irest = a.s.q.ids_rest + IDS_REST_ROW * idx;
						sh_to_rgb(deg, dx, dy, dz, [&](int k, int c) { return quant_sh(s_cb, dc[c], irest, k, c); }, res);
					}
				}
				else if (RAW)
				{
					// get_features = cat(_features_dc, _features_rest), gaussian_model.py:153-156, without the copy
					const float* dc = a.s.sh_dc + 3 * idx;
					const float* rest = a.s.sh_rest + 3 * (long long)a.s.n_rest * idx;
					sh_to_rgb(deg, dx, dy, dz, [&](int k, int c) { return k == 0 ? dc[c] : rest[3 * (k - 1) + c]; }, res);
				}
				else if (a.packed)
				{
					const long long gfirst = deg == 0 ? 0 : a.cum[deg - 1];
					const float* sh = a.s.shs + 3 * (a.group_base[deg] + (idx - gfirst) * (long long)((deg + 1) * (deg + 1)));
					sh_to_rgb(deg, dx, dy, dz, [&](int k, int c) { return sh[3 * k + c]; }, res);
				}
				else if (a.sh_vec4)
				{
					// M == 16, 16-byte aligned tensor: the row is 12 float4; every coefficient below is a compile-time slot of one of
					// them, repeated loads of the same float4 are merged by the compiler (read-only path), and only the float4 of the
					// Gaussian's active bands are ever requested
					const float4* row = reinterpret_cast<const float4*>(a.s.shs) + 12 * idx;
					sh_to_rgb(deg, dx, dy, dz, [&](int k, int c) {
						const float4 q = __ldg(row + ((3 * k + c) >> 2));
						const int e = (3 * k + c) & 3;
						return e == 0 ? q.x : (e == 1 ? q.y : (e == 2 ? q.z : q.w)); }, res);
				}
				else
				{
					const float* sh = a.s.shs + 3 * idx * a.s.M;
					sh_to_rgb(deg, dx, dy, dz, [&](int k, int c) { return sh[3 * k + c]; }, res);
				}
#pragma unroll
				for (int c = 0; c < 3; c++)
				{
					const float v = __fadd_rn(res[c], 0.5f);
					clamp_bits |= (v < 0.0f) ? (1u << c) : 0u;
					rgb[c] = fmaxf(v, 0.0f);
				}
			}
			// ---- stores -------------------------------------------------------------------------
			const float pth = -__logf(255.0f * opacity) - 1e-3f;
			float4* rec = a.g.rec + 3 * idx;
			rec[0] = make_float4(conx, cony, conz, pth);
			rec[1] = make_float4(pix_x, pix_y, opacity, rgb[0]);
			rec[2] = make_float4(rgb[1], rgb[2], tz, __uint_as_float((uint32_t)idx));   // .w: the Gaussian's own id (the backward's flush needs it after the staging buffer is recycled)
			a.g.clamped[idx] = (uint8_t)clamp_bits;
			a.g.dbits[idx] = __float_as_uint(tz);
			if (a.dbg.depths) a.dbg.depths[idx] = tz;
			if (a.dbg.means2D) { a.dbg.means2D[2 * idx] = pix_x; a.dbg.means2D[2 * idx + 1] = pix_y; }
			if (a.dbg.cov3D) { for (int k = 0; k < 6; k++) a.dbg.cov3D[6 * idx + k] = cov3D[k]; }
			if (a.dbg.conic_opacity) reinterpret_cast<float4*>(a.dbg.conic_opacity)[idx] = make_float4(conx, cony, conz, opacity);
			if (a.dbg.rgb) { for (int c = 0; c < 3; c++) a.dbg.rgb[3 * idx + c] = rgb[c]; }
			if (a.dbg.clamped) { for (int c = 0; c < 3; c++) a.dbg.clamped[3 * idx + c] = (clamp_bits >> c) & 1u; }
		}
		if (idx < last)
		{
			a.radii[idx] = radius_i;
			a.g.rect[idx] = rect;
			if (a.dbg.tiles_touched) a.dbg.tiles_touched[idx] = tiles;
		}
		const uint32_t my_tiles = tiles; const uint2 my_rect = rect;
		// per-tile instance counts (what the reference derives from sorted keys in identifyTileRanges): one RED per
		// (Gaussian, tile); Gaussians covering more than 32 tiles are spread over the warp
		{
			const TileRect tr(my_rect);
			const uint32_t w = tr.width();
			const bool big = my_tiles > 32;
			if (my_tiles && !big)
				for (uint32_t y = tr.miny; y < tr.maxy; y++)
					for (uint32_t x = tr.minx; x < tr.maxx; x++)
					{
						if (a.hist_priv) atomicAdd(&s_hist[y * a.gx + x], 1u); else atomicAdd(&a.tile_count[y * a.gx + x], 1u);
					}
			unsigned bigmask = __ballot_sync(0xffffffffu, big);
			while (bigmask)
			{
				const int src = __ffs(bigmask) - 1; bigmask &= bigmask - 1;
				const uint32_t bt = __shfl_sync(0xffffffffu, my_tiles, src), bw = __shfl_sync(0xffffffffu, w, src);
				const uint32_t bminx = __shfl_sync(0xffffffffu, tr.minx, src), bminy = __shfl_sync(0xffffffffu, tr.miny, src);
				for (uint32_t k = threadIdx.x & 31; k < bt; k += 32)
				{
					const uint32_t t = (bminy + k / bw) * a.gx + bminx + k % bw;
					if (a.hist_priv) atomicAdd(&s_hist[t], 1u); else atomicAdd(&a.tile_count[t], 1u);
				}
			}
		}
		block_vis += __popc(__ballot_sync(0xffffffffu, visible)) * ((threadIdx.x & 31) == 0);
	}
	// number of visible Gaussians (SH-sparsity multiplier, rasterizer_impl.cu:549-571) without a later reduction pass
	if ((threadIdx.x & 31) == 0 && block_vis) atomicAdd(&a.g.counters[1], block_vis);
	if (a.hist_priv)
	{
		__syncthreads();
		uint32_t* dst = a.cta_count + (size_t)blockIdx.x * a.T;
		for (int t = threadIdx.x; t < a.T; t += blockDim.x) dst[t] = s_hist[t];
	}
}

__global__ void mark_visible_kernel(int P, const float* __restrict__ means3D, const float* __restrict__ view, uint8_t* __restrict__ present)
{
	const int idx = blockIdx.x * blockDim.x + threadIdx.x;
	if (idx >= P) return;
	present[idx] = xform_row(view, 2, means3D[3 * idx], means3D[3 * idx + 1], means3D[3 * idx + 2]) > 0.2f;
}

// Debug/test export of the fused de-quantisation: activated scales [P,3] and normalised rotations [P,4] as GaussianReader<IN_QUANT>
// decodes them for the preprocess kernels (compared bit-for-bit with torch.exp / F.normalize in the tests).
__global__ void debug_dequant_kernel(SceneArgs a, float* __restrict__ scales, float* __restrict__ rots)
{
	__shared__ float s_cb[GSB_NUM_CODEBOOKS * GSB_CODEBOOK_SIZE];
	stage_codebooks(a.q.centers, s_cb);
	const int idx = blockIdx.x * blockDim.x + threadIdx.x;
	if (idx >= a.P) return;
	GaussianReader<IN_QUANT, false> in;
	in.load_shape(a, idx);
	const GaussianActive g = in.activate(a, s_cb, idx);
	for (int k = 0; k < 3; k++) scales[3 * (size_t)idx + k] = g.s[k];
	reinterpret_cast<float4*>(rots)[idx] = make_float4(g.r, g.x, g.y, g.z);
}

int launch_debug_dequant(const GsbQuant* q, int P, float* scales, float* rots, cudaStream_t stream)
{
	if (P <= 0) return GSB_OK;
	if ((reinterpret_cast<uintptr_t>(q->ids_rot) & 3) != 0) { set_error("gsb_debug_dequant: ids_rot must be 4-byte aligned"); return GSB_EINVAL; }
	SceneArgs a{};
	a.P = P; a.quant = 1; a.q = *q;
	debug_dequant_kernel<<<(P + 255) / 256, 256, 0, stream>>>(a, scales, rots);
	GSB_CUDA_OK(cudaGetLastError());
	return GSB_OK;
}

int launch_preprocess(const GsbForwardRequest& req, const GeomState& g, const ImageState& img, const BinPlan& plan)
{
	const GsbScene* s = req.scene; const GsbCamera* cam = req.cam;
	PreArgs a{};
	a.s = scene_args(s, cam, req.raw);
	const dim3 tiles = tile_grid(cam->width, cam->height);
	a.gx = tiles.x; a.gy = tiles.y;
	a.packed = s->sh_packed;
	if (s->sh_packed)
	{
		long long cum = 0, base = 0;
		for (int d = 0; d < 4; d++)
		{
			a.group_base[d] = base;
			base += (long long)s->band_count[d] * (d + 1) * (d + 1);
			cum += s->band_count[d];
			a.cum[d] = (int)cum;
		}
	}
	a.prune = s->prune_mask;
	a.g = g; a.radii = req.radii; a.tile_count = img.tile_count;
	a.hist_priv = plan.priv; a.chunk = plan.chunk; a.T = a.gx * a.gy; a.cta_count = img.cta_count;
	if (req.debug) a.dbg = *req.debug;
	a.prefiltered = cam->prefiltered;
	const bool quant = a.s.quant;
	a.sh_vec4 = !quant && !a.packed && a.s.shs && a.s.M == 16 && (reinterpret_cast<uintptr_t>(a.s.shs) & 15) == 0;
	a.rest_aligned = quant && (reinterpret_cast<uintptr_t>(a.s.q.ids_rest) & 15) == 0 && (reinterpret_cast<uintptr_t>(a.s.q.ids_rot) & 3) == 0;
	if (quant && (reinterpret_cast<uintptr_t>(a.s.q.ids_rot) & 3) != 0) { set_error("quantised scene: ids_rot must be 4-byte aligned"); return GSB_EINVAL; }
	const int blocks_needed = (s->P + 255) / 256;
	const int threads = plan.priv ? plan.threads : 256;
	const size_t hist_words = plan.priv ? (plan.hist_bytes / 4 + 3) / 4 * 4 : 0;
	const size_t smem = (quant ? GSB_NUM_CODEBOOKS * GSB_CODEBOOK_SIZE * sizeof(float) : 0) + hist_words * 4 +
		(quant ? size_t(threads / 32) * 32 * IDS_REST_ROW : 0);
	int grid = plan.priv ? plan.ctas : blocks_needed;
	if (!plan.priv && quant && grid > GSB_NUM_SMS * 8) grid = GSB_NUM_SMS * 8;                         // persistent: amortise the table load
	const InputMode in = quant ? IN_QUANT : (req.raw ? IN_RAW : IN_ACTIVATED);
	return dispatch([&](auto in, auto aa, auto f3d) -> int {
		auto kernel = preprocess_kernel<in, aa, f3d>;
		if (int e = ensure_dyn_smem((const void*)kernel, 220 * 1024)) return e;
		ProfScope prof(K_PREPROCESS, stream_of(req));
		kernel<<<grid, threads, smem, stream_of(req)>>>(a);
		GSB_LAUNCHED();
		GSB_CUDA_OK(cudaGetLastError());
		return GSB_OK;
	}, in, req.antialiasing != 0, s->filter_3D != nullptr);
}

int launch_mark_visible(int P, const float* means3D, const float* view, uint8_t* present, cudaStream_t stream)
{
	if (P <= 0) return GSB_OK;
	ProfScope prof(K_MARK_VISIBLE, stream);
	mark_visible_kernel<<<(P + 255) / 256, 256, 0, stream>>>(P, means3D, view, present);
	GSB_LAUNCHED();
	GSB_CUDA_OK(cudaGetLastError());
	return GSB_OK;
}

} // namespace gsb
