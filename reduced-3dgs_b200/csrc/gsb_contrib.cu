// gsb_contrib.cu — per-Gaussian contribution statistics of a finished forward (sm_90a): blending-weight sums, maxima, pixel counts and
// each pixel's dominant Gaussian (DESIGN.md §5p).
//
// A pair (p, i) contributes when the colour forward composited it: its list position is below n_contrib(p) and it passes the alpha
// tests (the feature pass's and the render backward's rule, gsb_features.cu).  T is rebuilt front to back with the forward's own
// arithmetic (eval_pair, T <- T * (1 - alpha) with the same roundings), so every pair's alpha and T have the forward's bits, and the
// pair's weight is w = alpha * T (one rounding).  Per Gaussian i, over the pixels p of one view, with m = the optional per-pixel map
// clamped to [0, 1] (NaN reads as 0; 1 without a map):
//     weight_sum[i] = sum_p m(p) w      weight_max[i] = max_p w      pixels[i] = number of contributing pairs
// and per pixel top_id[p] = the id of the pair with the largest w (the earlier one in the list on a tie; -1 where none contributes).
//
// Layout of work: the feature forward's.  One CTA per 16x16 tile, 8 warps of 8x4 pixels (WarpPixels); batches of 256 list entries
// (r0 / r1 of the record and the id) are staged into shared memory and culled per warp with rect_may_contribute; the walk stops at the
// tile's tile_max_contrib.  For each staged Gaussian that some lane's pair passes, the warp reduces once over its survivors and issues
// at most three atomics: the ballot's popcount (integer add), the shuffle sum of m * w (rounded to a multiple of 2^-36 and added as a
// 64-bit integer, the scheme of the deterministic statistics forward, §5j) and the shuffle max of w (atomicMax on the bits of a
// non-negative float).  Integer additions and maxima do not depend on their order, and top_id is sequential per pixel, so every
// output is the same bytes on every run.
#include "gsb_common.cuh"

namespace gsb {

#define CONTRIB_BATCH 256
#define CONTRIB_FIXED_SCALE 68719476736.0f      // 2^36: one unit of the fixed-point sums (stats_fixed_to_float_kernel divides by it)

__global__ void __launch_bounds__(256) contributions_kernel(const uint2* __restrict__ ranges, const uint32_t* __restrict__ point_list,
	int W, int H, const float4* __restrict__ rec, const uint32_t* __restrict__ n_contrib, const uint32_t* __restrict__ tile_max,
	const float* __restrict__ pixel_weights, unsigned long long* __restrict__ sum_fixed, uint32_t* __restrict__ max_bits,
	int32_t* __restrict__ pixels, int32_t* __restrict__ top_id)
{
	__shared__ __align__(16) float4 s_rec[CONTRIB_BATCH * 2];
	__shared__ uint32_t s_id[CONTRIB_BATCH];
	const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
	const int tile = blockIdx.y * gridDim.x + blockIdx.x;
	const WarpPixels wp(W, H, warp, lane);
	const uint32_t hi = tile_max[tile], start = ranges[tile].x;
	const uint32_t last = wp.inside ? n_contrib[wp.pid] : 0u;
	const uint32_t wmax = warp_max(last);
	// fmaxf(NaN, 0) = 0: a NaN weight reads as 0, +-inf as 1 / 0
	const float m = !wp.inside ? 0.0f : pixel_weights ? fminf(fmaxf(pixel_weights[wp.pid], 0.0f), 1.0f) : 1.0f;

	float T = 1.0f, best = 0.0f;
	int32_t best_id = -1;
	for (uint32_t b = 0; b < hi; b += CONTRIB_BATCH)
	{
		const int n = min((uint32_t)CONTRIB_BATCH, hi - b);
		stage_records(point_list, rec, n, false, start, b, s_rec, s_id);
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
				const bool pass = pair_passes(b + e < last, pa, r0.w);
				const unsigned cm = __ballot_sync(0xffffffffu, pass);
				if (!cm) continue;
				const uint32_t gid = s_id[e];
				const float w = pass ? __fmul_rn(pa.alpha, T) : 0.0f;
				if (w > best) { best = w; best_id = (int32_t)gid; }          // strictly greater: the earlier pair keeps a tie
				float s = __fmul_rn(m, w), mx = w;
#pragma unroll
				for (int o = 16; o > 0; o >>= 1)
				{
					s += __shfl_xor_sync(0xffffffffu, s, o);
					mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
				}
				if (lane == 0)
				{
					atomicAdd(&pixels[gid], (int)__popc(cm));
					atomicAdd(&sum_fixed[gid], __float2ull_rn(s * CONTRIB_FIXED_SCALE));
					atomicMax(&max_bits[gid], __float_as_uint(mx));
				}
				if (pass) T = __fmul_rn(T, __fsub_rn(1.0f, pa.alpha));
			}
		}
		__syncthreads();                                       // the next batch overwrites the staging buffers
	}
	if (wp.inside) top_id[wp.pid] = best_id;
}

int launch_contributions(const GeomState& g, const BinningState& b, const ImageState& img, int P, long long R, int W, int H,
	const float* pixel_weights, float* weight_sum, float* weight_max, int32_t* pixels, int32_t* top_id, unsigned long long* sum_fixed,
	cudaStream_t stream)
{
	const size_t N = size_t(W) * H;
	{
		ProfScope prof(K_CONTRIB, stream);
		GSB_CUDA_OK(cudaMemsetAsync(top_id, 0xff, N * sizeof(int32_t), stream));          // -1 where nothing contributes
		if (P == 0) return GSB_OK;
		GSB_CUDA_OK(cudaMemsetAsync(weight_max, 0, size_t(P) * sizeof(float), stream));
		GSB_CUDA_OK(cudaMemsetAsync(pixels, 0, size_t(P) * sizeof(int32_t), stream));
		if (R == 0)
		{
			GSB_CUDA_OK(cudaMemsetAsync(weight_sum, 0, size_t(P) * sizeof(float), stream));
			return GSB_OK;
		}
		GSB_CUDA_OK(cudaMemsetAsync(sum_fixed, 0, size_t(P) * sizeof(unsigned long long), stream));
		contributions_kernel<<<tile_grid(W, H), 256, 0, stream>>>(img.ranges, b.point_list, W, H, g.rec, img.n_contrib,
			img.tile_max_contrib, pixel_weights, sum_fixed, reinterpret_cast<uint32_t*>(weight_max), pixels, top_id);
		GSB_LAUNCHED();
		GSB_CUDA_OK(cudaGetLastError());
	}
	return launch_stats_fixed_to_float(P, sum_fixed, weight_sum, stream);
}

} // namespace gsb
