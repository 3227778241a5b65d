// gsb_features.cu — per-Gaussian feature channels composited over the colour pass (sm_90a), forward and backward.
//
// features [P, F] (fp32, 1 <= F <= GSB_FEATURES_MAX) are composited exactly like a colour channel with background 0:
//     out_f(p) = sum_i f_i * alpha_i(p) * T_i(p)
// over the (pixel, Gaussian) pairs of the colour forward.  Everything that decides those pairs is already in the blobs of any forward:
// the tile ranges and the depth-sorted point_list, the 48-byte records (conic, pth, mean, opacity with the anti-aliasing factor applied),
// n_contrib and tile_max_contrib.  A feature pass therefore runs no preprocess, scan, scatter or sort; it only composites.
//
// Layout of work: one CTA per (16x16 tile, chunk of CH channels); 8 warps of 8x4 pixels (WarpPixels) as in render_forward_kernel.  A
// batch of 256 list entries is staged into shared memory (the record's r0 / r1 and the CH-channel slice of each Gaussian's feature
// row), and the exact warp-rectangle cull (rect_may_contribute) picks the entries a warp visits.
//
// Which pairs contribute: a pair (p, i) with list position pos (0-based) contributes iff pos < n_contrib(p) and it passes the alpha
// tests (power <= 0, power >= pth, alpha >= 1/255).  This is the colour forward's rule restated with its result n_contrib: every
// candidate pair in front of the last contributor contributed, since a candidate that would drop T below 1e-4 ends the pixel.  The
// render backward uses the same rule.  The pair is evaluated by the colour kernels' own eval_pair (gsb_common.cuh) and accumulated with
// the same rounding intrinsics in the same order, so a feature channel equals the colour channel of a colors_precomp = features, bg = 0
// render bit for bit.
//
// Backward (back to front from final_T, the colour backward's T recursion T <- T / (1 - alpha) with MUFU.RCP): per contributing pair
//     dL/df_c  += alpha T g_c                          (g = dL/dout at the pixel)
//     dL/dalpha = T sum_c (f_c - ar_c) g_c             (ar_c: the channel's "colour behind" recurrence; no background term)
// The channels' dL/dalpha goes into the same per-Gaussian accumulator record the render backward fills (gsb_render.cu: dop, sx, sy,
// cxx, cxy, cyy, with the constant factors applied by the consumer), so the preprocess backward carries it to means2D/3D, opacity,
// scales / rotations / cov3D, the raw parameters, quant.grads and the camera unchanged.  Per (warp, Gaussian) the CH feature sums and
// the six accumulator terms are reduced over the warp's 32 pixels with a transposing butterfly (each step halves the values a lane
// carries) and added with one atomic per value.
#include <cstdlib>
#include "gsb_common.cuh"

namespace gsb {

#define FEAT_BATCH 256
#define FEAT_ACC_TERMS 6             // dop, sx, sy, cxx, cxy, cyy: slots 3..8 of the accumulator record

// Chunk width (channels per CTA), measured with tools/bench_features.py (DESIGN.md §5l): 8 up to F = 8, where a 16-wide chunk
// would carry idle channels, and 16 beyond, where fewer chunks re-walk the tile lists fewer times.  GSB_FEATURES_CH=8|16 forces
// one width for both kernels (a measurement knob, read once).
static int features_ch(int F)
{
	static const int forced = [] { const char* e = getenv("GSB_FEATURES_CH"); const int x = e ? atoi(e) : 0; return x == 8 || x == 16 ? x : 0; }();
	return forced ? forced : (F <= 8 ? 8 : 16);
}

// Stages list entries [first, first + n) of a tile (stage_records: r0 / r1 of the record and the Gaussian id), then the CH-channel
// slice [c0, c0 + CH) of each one's feature row (0 past F).
template <int CH>
__device__ __forceinline__ void stage_batch(const uint32_t* __restrict__ point_list, const float4* __restrict__ rec,
	const float* __restrict__ features, int F, int c0, int n, bool backwards, uint32_t base, uint32_t first, float4* s_rec, float* s_f,
	uint32_t* s_id)
{
	const int tid = threadIdx.x;
	stage_records(point_list, rec, n, backwards, base, first, s_rec, s_id);
	// consecutive threads read consecutive channels of one row
	for (int i = tid; i < n * CH; i += blockDim.x)
	{
		const int j = i / CH, c = c0 + (i % CH);
		s_f[i] = c < F ? __ldg(features + (size_t)s_id[j] * F + c) : 0.0f;
	}
	__syncthreads();
}

template <int CH>
__global__ void __launch_bounds__(256) features_forward_kernel(const uint2* __restrict__ ranges, const uint32_t* __restrict__ point_list,
	int W, int H, const float4* __restrict__ rec, const uint32_t* __restrict__ n_contrib, const uint32_t* __restrict__ tile_max,
	const float* __restrict__ features, int F, float* __restrict__ out)
{
	__shared__ __align__(16) float4 s_rec[FEAT_BATCH * 2];
	__shared__ __align__(16) float s_f[FEAT_BATCH * CH];
	__shared__ uint32_t s_id[FEAT_BATCH];
	const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
	const int tile = blockIdx.y * gridDim.x + blockIdx.x, c0 = blockIdx.z * CH;
	const WarpPixels wp(W, H, warp, lane);
	const size_t pid = wp.pid, N = (size_t)W * H;
	const uint32_t hi = tile_max[tile], start = ranges[tile].x;
	const uint32_t last = wp.inside ? n_contrib[pid] : 0u;
	const uint32_t wmax = warp_max(last);

	float T = 1.0f;
	float acc[CH];
#pragma unroll
	for (int k = 0; k < CH; k++) acc[k] = 0.0f;
	for (uint32_t b = 0; b < hi; b += FEAT_BATCH)
	{
		const int n = min((uint32_t)FEAT_BATCH, hi - b);
		stage_batch<CH>(point_list, rec, features, F, c0, n, false, start, b, s_rec, s_f, s_id);
		for (int cb = 0; cb < n && b + cb < wmax; cb += 32)
		{
			const int j = cb + lane;
			bool keep = false;
			if (j < n && b + j < wmax)
			{
				const float4 r0 = s_rec[2 * j], r1 = s_rec[2 * j + 1];
				keep = rect_may_contribute(r0, r1, wp);
			}
			unsigned mask = __ballot_sync(0xffffffffu, keep);
			while (mask)
			{
				const int e = cb + __ffs(mask) - 1; mask &= mask - 1;
				const float4 r0 = s_rec[2 * e], r1 = s_rec[2 * e + 1];
				const PairAlpha pa = eval_pair(r0, r1, wp);
				const float alpha = pa.alpha;
				if (pair_passes(b + e < last, pa, r0.w))
				{
					const float4* f4 = reinterpret_cast<const float4*>(s_f + e * CH);
#pragma unroll
					for (int q = 0; q < CH / 4; q++)
					{
						const float4 f = f4[q];
						acc[4 * q] = __fmaf_rn(T, __fmul_rn(f.x, alpha), acc[4 * q]);
						acc[4 * q + 1] = __fmaf_rn(T, __fmul_rn(f.y, alpha), acc[4 * q + 1]);
						acc[4 * q + 2] = __fmaf_rn(T, __fmul_rn(f.z, alpha), acc[4 * q + 2]);
						acc[4 * q + 3] = __fmaf_rn(T, __fmul_rn(f.w, alpha), acc[4 * q + 3]);
					}
					T = __fmul_rn(T, __fsub_rn(1.0f, alpha));
				}
			}
		}
		__syncthreads();                                       // the next batch overwrites the staging buffers
	}
	if (wp.inside)
	{
#pragma unroll
		for (int k = 0; k < CH; k++)
			if (c0 + k < F) out[(size_t)(c0 + k) * N + pid] = __fmaf_rn(0.0f, T, acc[k]);      // the colour output with bg = 0
	}
}

// Sum of v[0..NV) over the warp, transposed: each step exchanges half of the values a lane still carries with the partner lane, so
// NV = 16 takes 8+4+2+1+1 shuffles instead of 16 x 5.  -> the lane's value and its index (lanes that share an index hold the same sum).
template <int S, int NV>
__device__ __forceinline__ void transpose_step(float (&v)[NV], int lane, int& idx)
{
	constexpr int o = 16 >> S, half = NV >> (S + 1);
	if constexpr (half >= 1)
	{
		const bool up = (lane & o) != 0;
		if (up) idx += half;
#pragma unroll
		for (int i = 0; i < half; i++)
		{
			const float send = up ? v[i] : v[i + half];
			const float keep = up ? v[i + half] : v[i];
			v[i] = keep + __shfl_xor_sync(0xffffffffu, send, o);
		}
	}
	else v[0] += __shfl_xor_sync(0xffffffffu, v[0], o);
}
template <int NV>
__device__ __forceinline__ float warp_transpose_sum(float (&v)[NV], int lane, int& idx)
{
	idx = 0;
	transpose_step<0>(v, lane, idx); transpose_step<1>(v, lane, idx); transpose_step<2>(v, lane, idx);
	transpose_step<3>(v, lane, idx); transpose_step<4>(v, lane, idx);
	return v[0];
}

template <int CH>
__global__ void __launch_bounds__(256) features_backward_kernel(const uint2* __restrict__ ranges, const uint32_t* __restrict__ point_list,
	int W, int H, const float4* __restrict__ rec, const float* __restrict__ final_Ts, const uint32_t* __restrict__ n_contrib,
	const uint32_t* __restrict__ tile_max, const float* __restrict__ features, int F, const float* __restrict__ dL_dout,
	float* __restrict__ dL_dfeatures, float* __restrict__ acc)
{
	constexpr int NV = (CH + FEAT_ACC_TERMS <= 16) ? 16 : 32;
	__shared__ __align__(16) float4 s_rec[FEAT_BATCH * 2];
	__shared__ __align__(16) float s_f[FEAT_BATCH * CH];
	__shared__ uint32_t s_id[FEAT_BATCH];
	const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
	const int tile = blockIdx.y * gridDim.x + blockIdx.x, c0 = blockIdx.z * CH;
	const uint32_t hi = tile_max[tile];
	if (hi == 0) return;
	const WarpPixels wp(W, H, warp, lane);
	const size_t pid = wp.pid, N = (size_t)W * H;
	const uint32_t start = ranges[tile].x;
	const uint32_t last = wp.inside ? n_contrib[pid] : 0u;
	const uint32_t wmax = warp_max(last);

	float T = wp.inside ? final_Ts[pid] : 0.0f;
	float g[CH], ar[CH], lf[CH], last_alpha = 0.0f;
#pragma unroll
	for (int k = 0; k < CH; k++)
	{
		g[k] = (wp.inside && c0 + k < F) ? dL_dout[(size_t)(c0 + k) * N + pid] : 0.0f;
		ar[k] = 0.0f; lf[k] = 0.0f;
	}
	// entry j of batch b sits at list position hi - 1 - (b + j): the batches run from the back of the list to the front
	for (uint32_t b = 0; b < hi; b += FEAT_BATCH)
	{
		const int n = min((uint32_t)FEAT_BATCH, hi - b);
		stage_batch<CH>(point_list, rec, features, F, c0, n, true, start, hi - 1 - b, s_rec, s_f, s_id);
		for (int cb = 0; cb < n; cb += 32)
		{
			const int j = cb + lane;
			bool keep = false;
			if (j < n && hi - 1 - (b + j) < wmax)
			{
				const float4 r0 = s_rec[2 * j], r1 = s_rec[2 * j + 1];
				keep = rect_may_contribute(r0, r1, wp);
			}
			unsigned mask = __ballot_sync(0xffffffffu, keep);
			while (mask)
			{
				const int e = cb + __ffs(mask) - 1; mask &= mask - 1;
				const uint32_t pos = hi - 1 - (b + e);
				const float4 r0 = s_rec[2 * e], r1 = s_rec[2 * e + 1];
				const PairAlpha pa = eval_pair(r0, r1, wp);
				const float alpha = pa.alpha, dx = pa.dx, dy = pa.dy;
				const bool active = pair_passes(pos < last, pa, r0.w);
				if (!__any_sync(0xffffffffu, active)) continue;
				float v[NV];
#pragma unroll
				for (int k = 0; k < NV; k++) v[k] = 0.0f;
				if (active)
				{
					// render_backward_kernel's recursion: T before this Gaussian, and the "colour behind" of each channel
					T = T * rcp_approx(1.0f - alpha);
					const float u = alpha * T, oml = 1.0f - last_alpha;
					const float* f = s_f + e * CH;
					float dLda = 0.0f;
#pragma unroll
					for (int k = 0; k < CH; k++)
					{
						const float fk = f[k];
						ar[k] = last_alpha * lf[k] + oml * ar[k]; lf[k] = fk;
						dLda += (fk - ar[k]) * g[k];
						v[k] = u * g[k];
					}
					last_alpha = alpha;
					const float w = pa.G * (dLda * T);                     // G * dL/dalpha
					const float o = r1.z, wx = w * dx, wy = w * dy;
					v[CH] = w;
					v[CH + 1] = -o * (r0.x * wx + r0.y * wy);
					v[CH + 2] = -o * (r0.z * wy + r0.y * wx);
					v[CH + 3] = o * (wx * dx);
					v[CH + 4] = o * (wx * dy);
					v[CH + 5] = o * (wy * dy);
				}
				int idx;
				const float s = warp_transpose_sum<NV>(v, lane, idx);
				const bool writer = NV == 32 || (lane & 1) == 0;
				const uint32_t gid = s_id[e];
				if (writer && idx < CH)
				{
					if (c0 + idx < F) atomicAdd(dL_dfeatures + (size_t)gid * F + c0 + idx, s);
				}
				else if (writer && idx < CH + FEAT_ACC_TERMS) atomicAdd(acc + 12 * (size_t)gid + 3 + (idx - CH), s);
			}
		}
		__syncthreads();
	}
}

// Calls f with the chunk width as a std::integral_constant (as dispatch() hands over flags) and the grid: tiles x chunks of it.
template <class Fn> static int dispatch_ch(int W, int H, int F, Fn&& f)
{
	const int ch = features_ch(F);
	dim3 grid = tile_grid(W, H);
	grid.z = (F + ch - 1) / ch;
	return ch == 8 ? f(std::integral_constant<int, 8>{}, grid) : f(std::integral_constant<int, 16>{}, grid);
}

int launch_features_forward(const ImageState& img, const BinningState& b, const GeomState& g, int W, int H, const GsbFeatures& f,
	cudaStream_t stream)
{
	ProfScope prof(K_FEATURES_FWD, stream);
	return dispatch_ch(W, H, f.F, [&](auto ch, dim3 grid) -> int {
		features_forward_kernel<ch><<<grid, 256, 0, stream>>>(img.ranges, b.point_list, W, H, g.rec, img.n_contrib,
			img.tile_max_contrib, f.features, f.F, f.out);
		GSB_LAUNCHED();
		GSB_CUDA_OK(cudaGetLastError());
		return GSB_OK;
	});
}

int launch_features_backward(const ImageState& img, const BinningState& b, const GeomState& g, int P, int W, int H, const GsbFeatures& f,
	float* acc, cudaStream_t stream)
{
	ProfScope prof(K_FEATURES_BWD, stream);
	GSB_CUDA_OK(cudaMemsetAsync(f.dL_dfeatures, 0, size_t(P) * f.F * sizeof(float), stream));
	return dispatch_ch(W, H, f.F, [&](auto ch, dim3 grid) -> int {
		features_backward_kernel<ch><<<grid, 256, 0, stream>>>(img.ranges, b.point_list, W, H, g.rec, img.final_T,
			img.n_contrib, img.tile_max_contrib, f.features, f.F, f.dL_dout, f.dL_dfeatures, acc);
		GSB_LAUNCHED();
		GSB_CUDA_OK(cudaGetLastError());
		return GSB_OK;
	});
}

} // namespace gsb
