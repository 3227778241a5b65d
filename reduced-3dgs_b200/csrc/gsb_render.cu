// gsb_render.cu — per-tile alpha compositing, forward and backward (sm_90a).
//
// Replaces reference forward.cu:462-582 renderCUDA and backward.cu:438-595 renderCUDA.
//
// Layout of work: one CTA per 16x16 tile, 8 warps, each warp owns an 8x4 pixel sub-rectangle.  The tile's
// depth-sorted instance list is staged through shared memory in batches of 256 records of 48 bytes (three
// 128-bit gathers per instance).  For every 32 staged Gaussians each lane tests ONE Gaussian against the warp's
// 8x4 rectangle (closed-form bound on the Gaussian's maximum over the rectangle) and a ballot turns the
// results into a work mask, so the per-pixel loop only visits Gaussians that can reach alpha >= 1/255 somewhere
// in the warp.  Skipped (pixel, Gaussian) pairs are exactly pairs the reference `continue`s on, so n_contrib,
// final_T and colours are unchanged.  The per-pixel arithmetic is the reference's, operation for operation.  The warp's pixel block,
// the cull and the pair evaluation live in gsb_common.cuh (WarpPixels, rect_may_contribute, eval_pair): the feature kernels
// (gsb_features.cu) run the same code.
//
// Backward: instead of 9 global atomicAdds per contributing (pixel, Gaussian) pair (backward.cu:561-592) the 9
// per-Gaussian sums over a warp's 32 pixels are computed as a small matrix product on the tensor cores (3xTF32
// mma.sync, see below) and added to the per-Gaussian accumulator with three vector reductions per (warp, Gaussian).
// The tile's list is staged through a ring of shared-memory buffers filled by TMA bulk copies (mbarrier-tracked); the survivors
// of each staged batch are compacted into a per-warp work queue before the per-pixel loop.
#include <cstddef>
#include <cstdlib>
#include "gsb_common.cuh"

namespace gsb {

// Shared-memory staging record: 48 bytes per instance, r0 | r1 | (g, b, -, -); read with one address + immediate offsets.
#define SREC_BYTES 48
__device__ __forceinline__ float4 lds128(uint32_t addr)
{
	float4 v;
	asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr));
	return v;
}
__device__ __forceinline__ float2 lds64(uint32_t addr)
{
	float2 v;
	asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(addr));
	return v;
}

// ------------------------------------------------------------------------------------------------
// STATS = true additionally accumulates, per Gaussian, the number of pixels it contributed to and the sum of the
// transmittance T in front of it at those pixels (forward.cu:560-564, `calculate_mean_transmittance`): one pair of
// atomics per (warp, Gaussian) after a ballot / shuffle reduction instead of two per (pixel, Gaussian).
// Instruction budget (the kernel is issue-bound).  "This pixel is finished" is the SIGN
// BIT of T: a finished pixel has T < 0, so its test_T = T * (1 - alpha) <= 0 < 1e-4 takes the reference's stop branch again and
// changes nothing — no separate flag to carry, turn into a predicate and back on every iteration.  T is carried as its bit pattern
// (carried as a float, nvcc 12.9 folds the sign-setting arm of the update away — reproduced in isolation — and finished pixels
// resume).  The two constants of expf's range reduction come from the constant bank (exp_loop).  The per-pair arithmetic is
// untouched: colours, final_T and n_contrib stay bit-identical.
// What bounds this kernel: the FP32 pipe.  ~28 FADD/FMUL/FFMA-class warp instructions per (warp, entry) plus the cull
// arithmetic, and the per-pair arithmetic is the reference's (bit-identical results), so the kernel sits at the fp32 roofline of
// that arithmetic.
// Staging: the batch is gathered with three 128-bit loads per thread and stored to shared memory.  The alternative is the TMA path
// of the backward (one cp.async.bulk per 48-byte record, completion on an mbarrier): 256 small copies per batch serialise in the
// copy engine, while the load/store path issues them from 256 threads at once and this kernel has no other use for the time a
// ring would hide.
// MAPS = true also composites the inverse-depth map D = sum (1/depth) * alpha * T over the same pairs, with the colour channels'
// operation sequence, and writes D and the alpha map 1 - final_T.  1/depth (IEEE division) is computed once per staged instance and
// replaces the depth in the shared-memory copy of the record (r2.z), which the forward reads nowhere else.
#define STATS_FIXED_SCALE 68719476736.0f        // 2^36: one unit of the fixed-point transmittance sums is 2^-36
// FIXED = true (with STATS) is the deterministic statistics forward (DESIGN.md §5j): `transmittance` then points to 64-bit
// integers, and each (warp, Gaussian) sum ts is rounded to a multiple of 2^-36 and added with an integer atomic, whose total
// does not depend on the order of the additions.  stats_fixed_to_float_kernel turns the totals into floats.
template <bool STATS, bool MAPS, bool FIXED = false>
__global__ void __launch_bounds__(256, 6) render_forward_kernel(const uint2* __restrict__ ranges,
	const uint32_t* __restrict__ point_list,
	int W, int H, const float4* __restrict__ rec, const float* __restrict__ bg,
	float* __restrict__ final_T, uint32_t* __restrict__ n_contrib, float* __restrict__ out_color, uint32_t* __restrict__ tile_max,
	int32_t* __restrict__ touched_pixels, float* __restrict__ transmittance, float* __restrict__ out_invdepth, float* __restrict__ out_alpha)
{
	__shared__ __align__(16) float4 s_rec[256 * 3];
	__shared__ uint32_t s_id[STATS ? 256 : 1];
	__shared__ uint32_t s_max;
	const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
	const int tile = blockIdx.y * gridDim.x + blockIdx.x;
	const WarpPixels wp(W, H, warp, lane);
	const uint2 range = ranges[tile];
	uint32_t sbase = (uint32_t)__cvta_generic_to_shared(s_rec);
	asm volatile("" : "+r"(sbase));                       // keep the shared-window address in a register (otherwise re-derived from SR_CgaCtaId every iteration)
	if (tid == 0) s_max = 0;

	uint32_t Tb = wp.inside ? 0x3f800000u : 0xbf800000u;      // bits of T; sign set = finished
	float C0 = 0.0f, C1 = 0.0f, C2 = 0.0f, D = 0.0f;
	uint32_t last = 0;
	for (uint32_t b = range.x; b < range.y; b += 256)
	{
		if (__syncthreads_count((int)Tb < 0) == 256) break;
		const int n = min(256u, range.y - b);
		if (tid < n)
		{
			const uint32_t id = point_list[b + tid];
			const float4 r0 = rec[3 * (size_t)id], r1 = rec[3 * (size_t)id + 1], r2 = rec[3 * (size_t)id + 2];
			s_rec[3 * tid] = r0; s_rec[3 * tid + 1] = r1;
			s_rec[3 * tid + 2] = MAPS ? make_float4(r2.x, r2.y, __fdiv_rn(1.0f, r2.z), r2.w) : r2;
			if (STATS) s_id[tid] = id;
		}
		__syncthreads();
		bool warp_done = __all_sync(0xffffffffu, (int)Tb < 0);
		for (int c0 = 0; c0 < n && !warp_done; c0 += 32)
		{
			const int j = c0 + lane;
			bool keep = false;
			if (j < n)
			{
				const float4 r0 = lds128(sbase + j * SREC_BYTES), r1 = lds128(sbase + j * SREC_BYTES + 16);
				keep = rect_may_contribute(r0, r1, wp);
			}
			unsigned mask = __ballot_sync(0xffffffffu, keep);
			const uint32_t cbase = sbase + c0 * SREC_BYTES;
			uint32_t nbase = (b - range.x) + c0 + 1;                // 1-based list position of the chunk's first entry
			asm volatile("" : "+r"(nbase));                         // (kept in a vector register: `last = nbase + bit` is then one predicated add)
			// Branch-free per-pixel body: in a surviving warp some lane nearly always takes every path of the reference's
			// if/continue chain, so predicating costs nothing and removes the divergence bookkeeping.  The arithmetic and
			// the order of the tests are the reference's (forward.cu:535-569); a masked lane changes no state.
			while (mask)
			{
				const int bit = __ffs(mask) - 1; mask &= mask - 1;
				const uint32_t addr = cbase + bit * SREC_BYTES;
				const float4 r0 = lds128(addr), r1 = lds128(addr + 16);
				float2 gb; float invd = 0.0f;
				if (MAPS) { const float4 r2 = lds128(addr + 32); gb = make_float2(r2.x, r2.y); invd = r2.z; }
				else gb = lds64(addr + 32);
				const float T = __uint_as_float(Tb);
				const PairAlpha pa = eval_pair(r0, r1, wp);
				const float alpha = pa.alpha;
				const bool cand = pair_passes(true, pa, r0.w);
				const float test_T = __fmul_rn(T, __fsub_rn(1.0f, alpha));
				const bool stop = cand && (test_T < 0.0001f);           // also true for every finished pixel (T < 0)
				const bool v = cand && !(test_T < 0.0001f);
				if (STATS)
				{
					const unsigned cm = __ballot_sync(0xffffffffu, v);
					if (cm)
					{
						float ts = v ? T : 0.0f;
#pragma unroll
						for (int o = 16; o > 0; o >>= 1) ts += __shfl_xor_sync(0xffffffffu, ts, o);
						if (lane == 0)
						{
							const uint32_t gid = s_id[c0 + bit];
							atomicAdd(&touched_pixels[gid], (int)__popc(cm));
							if (FIXED) atomicAdd(reinterpret_cast<unsigned long long*>(transmittance) + gid, __float2ull_rn(ts * STATS_FIXED_SCALE));
							else atomicAdd(&transmittance[gid], ts);
						}
					}
				}
				if (v)
				{
					C0 = __fmaf_rn(T, __fmul_rn(r1.w, alpha), C0);
					C1 = __fmaf_rn(T, __fmul_rn(gb.x, alpha), C1);
					C2 = __fmaf_rn(T, __fmul_rn(gb.y, alpha), C2);
					if (MAPS) D = __fmaf_rn(T, __fmul_rn(invd, alpha), D);
					Tb = __float_as_uint(test_T);
					last = nbase + bit;
				}
				if (stop) Tb |= 0x80000000u;
			}
			warp_done = __all_sync(0xffffffffu, (int)Tb < 0);
		}
	}
	const float T = __uint_as_float(Tb & 0x7fffffffu);
	if (wp.inside)
	{
		const size_t pid = wp.pid, N = (size_t)W * H;
		final_T[pid] = T;
		n_contrib[pid] = last;
		out_color[pid] = __fmaf_rn(bg[0], T, C0);
		out_color[N + pid] = __fmaf_rn(bg[1], T, C1);
		out_color[2 * N + pid] = __fmaf_rn(bg[2], T, C2);
		if (MAPS) { out_invdepth[pid] = D; out_alpha[pid] = __fsub_rn(1.0f, T); }
	}
	// where the backward pass has to start for this tile
	const uint32_t m = warp_max(wp.inside ? last : 0u);
	__syncthreads();
	if (lane == 0 && m) atomicMax(&s_max, m);
	__syncthreads();
	if (tid == 0) tile_max[tile] = s_max;
}

// ------------------------------------------------------------------------------------------------
// Backward.  For one Gaussian and the 32 pixels of a warp the reference accumulates 9 sums (backward.cu:561-592).  With
//     u_p = alpha_p * T_p                 (dL/dcolour weight)        w_p = G_p * dL/dalpha_p
// and d = (X - px, Y - py) (X, Y = Gaussian centre, px, py = pixel, all tile-local) they are
//     dL/dcolour_c = sum_p u_p * dLdpix_c(p)            dL/dopacity = sum_p w_p =: M0
//     sum_p w_p dx   = X M0 - Mx        sum_p w_p dx^2  = X^2 M0 - 2X Mx + Mxx      (Mx = sum_p w_p px, ... the moments of w)
// i.e. [Gaussians x pixels] . [pixels x 9 per-pixel constants]: a tiny matrix product.  The kernel therefore stashes
// (w, u) for up to 16 surviving Gaussians per warp and lets the tensor cores do the pixel sums with 3xTF32-split
// m16n8k8 MMAs (fp32-level accuracy: operands are split hi/lo, the per-pixel weights 1, px, py, px^2, px*py, py^2 are exact in
// TF32), instead of a 14-shuffle butterfly + 9 products per (warp, Gaussian).  tcgen05 is not applicable to a per-warp
// 16x32x8 product (it needs 64/128-row tiles from shared-memory descriptors and TMEM); this is the warp-level MMA path.
#define BWD_BATCH 64
#define STASH_LD 36            // row stride of the (w, u) stash: conflict-free A-fragment loads
#define ACC_STRIDE 9           // per staged Gaussian: [dcol0 dcol1 dcol2 M0 Mx My Mxx Mxy Myy]

__device__ __forceinline__ void mma_tf32(float (&d)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1)
{
	asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
		: "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]) : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void split_tf32(float v, uint32_t& hi, uint32_t& lo)
{
	hi = __float_as_uint(v) & 0xffffe000u;                    // the MMA reads the top 19 bits: truncation is a valid TF32
	lo = __float_as_uint(v - __uint_as_float(hi));
}

// acc record written for the preprocess backward (12 floats per Gaussian, 48 B): [dcol.r dcol.g dcol.b dop | sx sy cxx cxy | cyy dinvd - -]
// sx = sum dL_dG*dG_ddelx, sy = sum dL_dG*dG_ddely, cxx = sum gdx*dx*dL_dG, cxy = sum gdx*dy*dL_dG, cyy = sum gdy*dy*dL_dG;
// the constant factors (0.5*W, 0.5*H, -0.5) of backward.cu:583-589 are applied once per Gaussian by the consumer.
// dinvd = sum alpha*T*dL/dinvdepth (written by the MAPS variant only; the memset leaves it 0 otherwise).
__device__ __forceinline__ void cp_async16(uint32_t smem_addr, const void* gptr)
{
	asm volatile("cp.async.ca.shared.global [%0], [%1], 16;" ::"r"(smem_addr), "l"(gptr) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }

#define BWD_STAGES 4
// Everything one warp owns privately sits in ONE block: a single base address in a register, every member an immediate offset
// (with separate per-member arrays ptxas re-derived five base addresses inside the hot loop once registers ran out).
// NCH: channels of the u product's B operand, 3 (colour) or 4 (colour + dL/dinvdepth, MAPS).
template <int NCH> struct BwdWarp {
	float w[16 * STASH_LD];                // stash of up to 16 surviving Gaussians: w = G * dL/dalpha per pixel lane
	float u[16 * STASH_LD];                //                                         u = alpha * T per pixel lane
	float dlp[NCH * 32];                   // dL/dpixel (and dL/dinvdepth) of the warp's 32 pixels, channel-major: B operand of the u product
	uint32_t rowid[16];                    // Gaussian id of each stashed row (rows outlive their staging buffer; the flush re-reads the record)
	uint8_t queue[BWD_BATCH + 16];         // work queue: batch indices of the entries that survived the warp's cull (+ slack: the loop reads one ahead)
};
#define BW_OFF_U (16 * STASH_LD * 4)
#define BW_OFF_ROWID(NCH) (2 * 16 * STASH_LD * 4 + (NCH) * 32 * 4)
#define BW_OFF_QUEUE(NCH) (BW_OFF_ROWID(NCH) + 16 * 4)
template <int NCH> struct BwdSmem {
	float4 rec[BWD_STAGES][BWD_BATCH * 3]; // ring of staged batches of the tile's list: one 48-byte TMA bulk copy per instance (the record carries its Gaussian id in r2.w)
	uint64_t full[BWD_STAGES];             // mbarrier: the stage's copies have landed (64 arrivals + transaction bytes)
	uint64_t empty[BWD_STAGES];            // mbarrier: all 8 warps are done reading the stage
	float wgt[8 * 32];                     // (1, qx, qy, qx^2, qx*qy, qy^2, 0, 0) of the 32 warp-local pixels: B operand of the moment product
	BwdWarp<NCH> wp[8];
};
static_assert(offsetof(BwdWarp<3>, u) == BW_OFF_U && offsetof(BwdWarp<3>, rowid) == BW_OFF_ROWID(3) && offsetof(BwdWarp<3>, queue) == BW_OFF_QUEUE(3), "BwdWarp layout");
static_assert(offsetof(BwdWarp<4>, u) == BW_OFF_U && offsetof(BwdWarp<4>, rowid) == BW_OFF_ROWID(4) && offsetof(BwdWarp<4>, queue) == BW_OFF_QUEUE(4), "BwdWarp layout");
static_assert(sizeof(BwdWarp<3>) % 16 == 0 && sizeof(BwdWarp<4>) % 16 == 0, "BwdWarp alignment");

__device__ __forceinline__ void red_add_v2(float* addr, float a, float b)
{
	asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(addr), "f"(a), "f"(b) : "memory");
}


// MAPS = true adds the gradients of the inverse-depth and alpha maps (render_forward_kernel<*, true>):
//  - alpha = 1 - T_final enters every pair exactly like the background term: bg.dL/dpixel becomes bg.dL/dpixel - dL/dalpha_map;
//  - invdepth is a fourth colour channel (colour 1/depth, no background): it is one more term of the pair loop's k, its
//    dL/dinvdepth fills the B column of the u product that is zero padding otherwise, and sum_p u_p * dL/dinvdepth(p) lands in
//    slot 9 of the accumulator, next to cyy (one vector reduction instead of the scalar one).
// 1/depth is the MUFU reciprocal here (the forward's IEEE value to 1 ulp; the result is a tolerance-compared gradient).
//
// DET = true is the deterministic variant (DESIGN.md §5i).  The pair arithmetic and the MMA pixel sums are the same; only the
// summation across warps and tiles changes.  A staged batch is processed in lockstep: every warp flushes its stash at the end of
// the batch and writes each row's 9 (10 with MAPS) values to its own shared-memory row of the batch entry (ebuf, zero for entries
// it culled); after a CTA barrier the threads add the 8 warps' rows in warp order 0..7 and STORE the sum to the instance's slot
// of `parts` (gsb_common.cuh TileRect; no atomics).  det_gather_kernel then adds each Gaussian's slots in slot order.  The stash
// rows keep their batch entry index instead of the Gaussian id: the records are still staged.
//
// ABS = true also accumulates the absolute screen-space gradient (AbsGS; DESIGN.md §5m), per Gaussian
//     ax = o * sum_p |w_p (a dx_p + b dy_p)|,   ay = o * sum_p |w_p (b dx_p + c dy_p)|
// over exactly the pairs the backward visits ((a, b, c) the conic, o the record's opacity), into accumulator slots 10 and 11.  The
// per-pair factor is linear in the pixel, so nothing is stashed for it: at flush time lane l rebuilds it for stashed row l / 2,
// component l % 2, from the row's record and the 32 stashed w (zero for the pairs the reference skips), and adds the 32 products
// in pixel order.  The pair loop is the same instruction stream as without ABS, and no shared memory is added.
#define DET_NS(MAPS) ((MAPS) ? 10 : 9)       // floats per slot: the accumulator's [dcol0 dcol1 dcol2 dop sx sy cxx cxy cyy (dinvd)]
template <bool MAPS, bool DET = false, bool ABS = false>
__global__ void __launch_bounds__(256, DET ? (ABS ? 2 : 3) : 4) render_backward_kernel(const uint2* __restrict__ ranges,
	const uint32_t* __restrict__ point_list,
	int W, int H, const float4* __restrict__ rec, const float* __restrict__ bg,
	const float* __restrict__ final_Ts, const uint32_t* __restrict__ n_contrib, const uint32_t* __restrict__ tile_max,
	const float* __restrict__ dL_dpixels, float* __restrict__ acc, const float* __restrict__ dL_dinvdepth, const float* __restrict__ dL_dalpha,
	float* __restrict__ parts = nullptr, const uint32_t* __restrict__ slot_offset = nullptr, const uint2* __restrict__ rect = nullptr,
	unsigned long long num_slots = 0)
{
	constexpr int NCH = MAPS ? 4 : 3;
	constexpr int NS = ABS ? DET_NS_ABS : DET_NS(MAPS);
	extern __shared__ __align__(16) unsigned char s_dyn_raw[];
	BwdSmem<NCH>& S = *reinterpret_cast<BwdSmem<NCH>*>(s_dyn_raw);
	float* const ebuf = reinterpret_cast<float*>(s_dyn_raw + sizeof(BwdSmem<NCH>));     // DET: [8 warps][BWD_BATCH entries][NS]
	const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
	const int tile = blockIdx.y * gridDim.x + blockIdx.x;
	const uint32_t hi = tile_max[tile];
	if (hi == 0) return;
	// The block of WarpPixels(W, H, warp, lane), formed from the tile-local pixel: in this form the 64-register variants fit without spilling.
	WarpPixels wp;
	const int lx = (warp & 1) * 8 + (lane & 7), ly = (warp >> 1) * 4 + (lane >> 3);
	const int tx0 = blockIdx.x * GSB_TILE_X, ty0 = blockIdx.y * GSB_TILE_Y;
	wp.px = tx0 + lx; wp.py = ty0 + ly;
	wp.inside = wp.px < W && wp.py < H;
	wp.pxf = (float)wp.px; wp.pyf = (float)wp.py;
	wp.rx0 = (float)(tx0 + (warp & 1) * 8); wp.rx1 = wp.rx0 + 7.0f; wp.ry0 = (float)(ty0 + (warp >> 1) * 4); wp.ry1 = wp.ry0 + 3.0f;
	const uint2 range = ranges[tile];
	const size_t pid = wp.pid = (size_t)W * wp.py + wp.px, N = (size_t)W * H;
	uint32_t sbase0 = (uint32_t)__cvta_generic_to_shared(&S.rec[0][0]);
	asm volatile("" : "+r"(sbase0));
	BwdWarp<NCH>& Wp = S.wp[warp];
	uint32_t wbase = (uint32_t)__cvta_generic_to_shared(&Wp);           // the warp's private block (see BwdWarp)
	asm volatile("" : "+r"(wbase));
	const unsigned lt_mask = (1u << lane) - 1u;

	const float T_final = wp.inside ? final_Ts[pid] : 0.0f;
	float T = T_final;
	const uint32_t last_contributor = wp.inside ? n_contrib[pid] : 0u;
	float dLp0 = 0.f, dLp1 = 0.f, dLp2 = 0.f;
	if (wp.inside) { dLp0 = dL_dpixels[pid]; dLp1 = dL_dpixels[N + pid]; dLp2 = dL_dpixels[2 * N + pid]; }
	float bg_dot_dpixel = bg[0] * dLp0 + bg[1] * dLp1 + bg[2] * dLp2;
	float dLd = 0.f;                                                             // MAPS: dL/dinvdepth
	if (MAPS && wp.inside)
	{
		if (dL_dinvdepth) dLd = dL_dinvdepth[pid];
		if (dL_dalpha) bg_dot_dpixel -= dL_dalpha[pid];
	}
	const float nbg = -T_final * bg_dot_dpixel;                                  // backward.cu:569-572 without its per-pair factor 1 / (1 - alpha)
	float ard = 0.f, dl = 0.f, la = 0.f;                                         // the colour recurrence, folded with dL/dpixel (see the pair loop)
	const uint32_t wmax = warp_max(last_contributor);

	// B fragments (m16n8k8: b0 = B[k = t][n = g], b1 = B[k = t + 4][n = g]; k = pixel lane of the k-step, n = output column) are
	// rebuilt inside flush_rows (a few shuffles per 16 Gaussians) instead of living in 24 registers: occupancy matters more.
	const int fg = lane >> 2, ft = lane & 3;
	float* sw = Wp.w;
	float* su = Wp.u;
	uint32_t nrows = 0;                                                           // warp-uniform: stashed Gaussians
	int buf = 0;

	// Pixel coordinates inside the moment product are WARP-local and centred (qx = lane%8 - 3.5, qy = lane/8 - 1.5: exact in
	// TF32, identical for every warp), and X, Y below are relative to the same centre: the shift back from moments to
	// sum w*dx^2 etc. then cancels as little as possible.
	if (tid < 32)
	{
		const float qx = (float)(tid & 7) - 3.5f, qy = (float)(tid >> 3) - 1.5f;
		S.wgt[0 * 32 + tid] = 1.0f; S.wgt[1 * 32 + tid] = qx; S.wgt[2 * 32 + tid] = qy;
		S.wgt[3 * 32 + tid] = qx * qx; S.wgt[4 * 32 + tid] = qx * qy; S.wgt[5 * 32 + tid] = qy * qy;
		S.wgt[6 * 32 + tid] = 0.0f; S.wgt[7 * 32 + tid] = 0.0f;
	}
	Wp.dlp[lane] = dLp0; Wp.dlp[32 + lane] = dLp1; Wp.dlp[64 + lane] = dLp2;
	if (MAPS) Wp.dlp[96 + lane] = dLd;
	const float cxw = wp.rx0 + 3.5f, cyw = wp.ry0 + 1.5f;                          // centre of the warp's 8x4 pixel block
	if (DET) for (int i = tid; i < 8 * BWD_BATCH * NS; i += 256) ebuf[i] = 0.0f;
	__syncthreads();

	// Pixel sums of the stashed rows on the tensor cores; lane (g, t = 0) then owns rows g and g + 8: it converts the moments
	// to the reference's sums and issues ONE set of global reductions per (warp, Gaussian) — no shared-memory accumulators,
	// no CTA-wide flush phase, no barrier besides the one that hands over the staging buffers.
	auto flush_rows = [&]() {
		if (nrows == 0) return;
		for (uint32_t r = nrows; r < 16; r++) { sw[r * STASH_LD + lane] = 0.f; su[r * STASH_LD + lane] = 0.f; }
		__syncwarp();
		if (!DET && ft == 0)                                                         // the epilogue re-reads the rows' records: pull them into L1 behind the MMAs
		{
			if (fg < nrows) asm volatile("prefetch.global.L1 [%0];" ::"l"(rec + 3 * (size_t)Wp.rowid[fg]));
			if (fg + 8 < nrows) asm volatile("prefetch.global.L1 [%0];" ::"l"(rec + 3 * (size_t)Wp.rowid[fg + 8]));
		}
		// ABS: lane l sums row l / 2, component l % 2 (rows 0..3 in the 8 lanes of a 128-bit shared-memory phase: no bank conflict),
		// ahead of the MMAs so that only its result is live across them.
		// a dx + b dy with dx = X' - qx, dy = Y' - qy (X', Y' relative to the warp centre, qx, qy the pixel's constants) is
		// K - a qx - b qy, K = a X' + b Y'; (a, b) -> (b, c) for the y component.
		float absv = 0.f;
		if (ABS)
		{
			const uint32_t ar = lane >> 1;
			if (ar < nrows)
			{
				const uint32_t gid = Wp.rowid[ar];
				float4 r0, r1;
				if (DET)
				{
					const uint32_t ra = sbase0 + (uint32_t)(buf * BWD_BATCH * 3) * 16u + gid * SREC_BYTES;
					r0 = lds128(ra); r1 = lds128(ra + 16);
				}
				else { r0 = __ldg(rec + 3 * (size_t)gid); r1 = __ldg(rec + 3 * (size_t)gid + 1); }
				const float ka = (lane & 1) ? r0.y : r0.x, kb = (lane & 1) ? r0.z : r0.y;
				const float K = ka * (r1.x - cxw) + kb * (r1.y - cyw);
				const uint32_t wrow = wbase + ar * (STASH_LD * 4);
				float s = 0.f;
#pragma unroll
				for (int j = 0; j < 8; j++)
				{
					const float4 w4 = lds128(wrow + 16 * j);
					const float wq[4] = { w4.x, w4.y, w4.z, w4.w };
#pragma unroll
					for (int i = 0; i < 4; i++)
					{
						const int p = 4 * j + i;
						const float v = fmaf(-ka, (float)(p & 7) - 3.5f, fmaf(-kb, (float)(p >> 3) - 1.5f, K));
						s = fmaf(fabsf(wq[i]), fabsf(v), s);
					}
				}
				absv = r1.z * s;
			}
		}
		float dw[4] = { 0.f, 0.f, 0.f, 0.f }, du[4] = { 0.f, 0.f, 0.f, 0.f };
		const float* dl = Wp.dlp + (fg < NCH ? fg : 0) * 32;
#pragma unroll
		for (int kk = 0; kk < 4; kk++)
		{
			const int c0 = 8 * kk + ft, c1 = c0 + 4;
			// B fragments: b0 = B[k = c0][n = fg], b1 = B[k = c1][n = fg]
			const uint32_t bw0 = __float_as_uint(S.wgt[fg * 32 + c0]), bw1 = __float_as_uint(S.wgt[fg * 32 + c1]);
			uint32_t buh0, buh1, bul0, bul1;
			split_tf32(fg < NCH ? dl[c0] : 0.0f, buh0, bul0);
			split_tf32(fg < NCH ? dl[c1] : 0.0f, buh1, bul1);
			uint32_t h0, h1, h2, h3, l0, l1, l2, l3;
			split_tf32(sw[fg * STASH_LD + c0], h0, l0); split_tf32(sw[(fg + 8) * STASH_LD + c0], h1, l1);
			split_tf32(sw[fg * STASH_LD + c1], h2, l2); split_tf32(sw[(fg + 8) * STASH_LD + c1], h3, l3);
			mma_tf32(dw, h0, h1, h2, h3, bw0, bw1);
			mma_tf32(dw, l0, l1, l2, l3, bw0, bw1);
			split_tf32(su[fg * STASH_LD + c0], h0, l0); split_tf32(su[(fg + 8) * STASH_LD + c0], h1, l1);
			split_tf32(su[fg * STASH_LD + c1], h2, l2); split_tf32(su[(fg + 8) * STASH_LD + c1], h3, l3);
			mma_tf32(du, h0, h1, h2, h3, buh0, buh1);
			mma_tf32(du, l0, l1, l2, l3, buh0, buh1);
			mma_tf32(du, h0, h1, h2, h3, bul0, bul1);
		}
		// D fragment: d[0] = D[g][2t], d[1] = D[g][2t+1], d[2] = D[g+8][2t], d[3] = D[g+8][2t+1]; columns of the w product:
		// (M0 Mx | My Mxx | Mxy Myy) in lanes t = 0 | 1 | 2, of the u product (c0 c1 | c2 -) in lanes t = 0 | 1 ((c0 c1 | c2 dinvd) with MAPS).
		const int q1 = (lane & ~3) | 1, q2 = (lane & ~3) | 2;
#pragma unroll
		for (int h = 0; h < 2; h++)
		{
			const float My = __shfl_sync(0xffffffffu, dw[2 * h], q1), Mxx = __shfl_sync(0xffffffffu, dw[2 * h + 1], q1);
			const float Mxy = __shfl_sync(0xffffffffu, dw[2 * h], q2), Myy = __shfl_sync(0xffffffffu, dw[2 * h + 1], q2);
			const float c2 = __shfl_sync(0xffffffffu, du[2 * h], q1);
			float dinvd = 0.f;
			if (MAPS) dinvd = __shfl_sync(0xffffffffu, du[2 * h + 1], q1);
			const uint32_t row = fg + 8 * h;
			float ax = 0.f, ay = 0.f;
			if (ABS) { ax = __shfl_sync(0xffffffffu, absv, 2 * row); ay = __shfl_sync(0xffffffffu, absv, 2 * row + 1); }
			if (ft == 0 && row < nrows)
			{
				const uint32_t gid = Wp.rowid[row];
				float4 r0, r1;
				if (DET)
				{
					// gid is the row's batch entry: its record is still in the current stage
					const uint32_t ra = sbase0 + (uint32_t)(buf * BWD_BATCH * 3) * 16u + gid * SREC_BYTES;
					r0 = lds128(ra); r1 = lds128(ra + 16);
				}
				else { r0 = __ldg(rec + 3 * (size_t)gid); r1 = __ldg(rec + 3 * (size_t)gid + 1); }      // L2-resident: staged moments ago
				const float X = r1.x - cxw, Y = r1.y - cyw, o = r1.z;
				const float M0 = dw[2 * h], Mx = dw[2 * h + 1];
				const float Sx = X * M0 - Mx, Sy = Y * M0 - My;
				const float Sxx = X * X * M0 - 2.0f * X * Mx + Mxx;
				const float Sxy = X * Y * M0 - X * My - Y * Mx + Mxy;
				const float Syy = Y * Y * M0 - 2.0f * Y * My + Myy;
				if (DET)
				{
					float* e = ebuf + (warp * BWD_BATCH + gid) * NS;
					e[0] = du[2 * h]; e[1] = du[2 * h + 1]; e[2] = c2; e[3] = M0;
					e[4] = -o * (r0.x * Sx + r0.y * Sy); e[5] = -o * (r0.z * Sy + r0.y * Sx); e[6] = o * Sxx; e[7] = o * Sxy;
					e[8] = o * Syy;
					if (MAPS) e[9] = dinvd;
					if (ABS) { e[10] = ax; e[11] = ay; }
					continue;
				}
				float* a = acc + 12 * (size_t)gid;
				red_add_v4(a, du[2 * h], du[2 * h + 1], c2, M0);
				red_add_v4(a + 4, -o * (r0.x * Sx + r0.y * Sy), -o * (r0.z * Sy + r0.y * Sx), o * Sxx, o * Sxy);
				if (ABS) red_add_v4(a + 8, o * Syy, dinvd, ax, ay);             // dinvd = 0 without the maps: slot 9 stays zero
				else if (MAPS) red_add_v2(a + 8, o * Syy, dinvd);
				else atomicAdd(a + 8, o * Syy);
			}
		}
		__syncwarp();
		nrows = 0;
	};

	// ---- staging ring: warps do NOT run in lockstep.  A batch of 96 list entries is gathered by 96 threads, one 48-byte TMA
	// bulk copy (cp.async.bulk, completion by mbarrier transaction bytes) per entry, BWD_STAGES - 1 batches ahead of the
	// slowest warp; a warp that finishes a batch early moves on to the next stage instead of waiting at a CTA barrier.
	auto list_id = [&](uint32_t bi) -> uint32_t {                                  // entry `tid` of batch bi (counted from the back of the list)
		const uint32_t k = bi * BWD_BATCH + tid;
		return (tid < BWD_BATCH && k < hi) ? point_list[range.x + (hi - 1 - k)] : 0xffffffffu;
	};
	auto issue = [&](uint32_t bi, uint32_t id) {                                   // threads tid < BWD_BATCH
		const int st = bi % BWD_STAGES;
		if (id != 0xffffffffu)
		{
			mbar_arrive_expect_tx(&S.full[st], 48u);
			tma_bulk_g2s(&S.rec[st][3 * tid], rec + 3 * (size_t)id, 48u, &S.full[st]);
		}
		else mbar_arrive(&S.full[st]);
	};
	const uint32_t nb = (hi + BWD_BATCH - 1) / BWD_BATCH;
	if (tid == 0)
	{
		for (int k = 0; k < BWD_STAGES; k++) { mbar_init(&S.full[k], BWD_BATCH); mbar_init(&S.empty[k], 8); }
		mbar_fence_init();
	}
	__syncthreads();
	uint32_t id_next = 0xffffffffu;
	if (tid < BWD_BATCH)
	{
		for (uint32_t k = 0; k < BWD_STAGES - 1 && k < nb; k++) issue(k, list_id(k));
		id_next = list_id(BWD_STAGES - 1);
	}
	for (uint32_t bi = 0; bi < nb; bi++)
	{
		const uint32_t b = bi * BWD_BATCH;
		const int n = min((uint32_t)BWD_BATCH, hi - b);
		buf = bi % BWD_STAGES;
		if (tid < BWD_BATCH && bi + BWD_STAGES - 1 < nb)
		{
			// the stage that batch bi + STAGES - 1 goes into was last read for batch bi - 1
			if (bi >= 1) mbar_wait(&S.empty[(bi - 1) % BWD_STAGES], ((bi - 1) / BWD_STAGES) & 1u);
			issue(bi + BWD_STAGES - 1, id_next);
			id_next = list_id(bi + BWD_STAGES);
		}
		mbar_wait(&S.full[buf], (bi / BWD_STAGES) & 1u);
		const uint32_t sbase = sbase0 + (uint32_t)(buf * BWD_BATCH * 3) * 16u;
		// ---- cull the batch into the warp's work queue (see render_forward_kernel) ----
		uint32_t qn = 0;
		for (int c0 = 0; c0 < n; c0 += 32)
		{
			const int j = c0 + lane;
			bool keep = false;
			if (j < n && (hi - 1 - b - j) < wmax)
			{
				const float4 r0 = lds128(sbase + j * SREC_BYTES), r1 = lds128(sbase + j * SREC_BYTES + 16);
				keep = rect_may_contribute(r0, r1, wp);
			}
			const unsigned mask = __ballot_sync(0xffffffffu, keep);
			if (keep) Wp.queue[qn + __popc(mask & lt_mask)] = (uint8_t)j;
			qn += __popc(mask);
		}
		__syncwarp();
		// pos < last_contributor with pos = (hi - 1 - b) - jj, the list position of batch entry jj (entries run backwards): jj > first
		const int first = (int)(hi - 1 - b) - (int)last_contributor;
		uint32_t jj = 0, jnext;
		if (qn) asm volatile("ld.shared.u8 %0, [%1+%2];" : "=r"(jj) : "r"(wbase), "n"(BW_OFF_QUEUE(NCH)));
		for (uint32_t qa = wbase, qe = wbase + qn; qa != qe; qa++, jj = jnext)
		{
			asm volatile("ld.shared.u8 %0, [%1+%2];" : "=r"(jnext) : "r"(qa), "n"(BW_OFF_QUEUE(NCH) + 1));   // next entry's index: off the critical path
			const uint32_t addr = sbase + jj * SREC_BYTES;
			const float4 r0 = lds128(addr), r1 = lds128(addr + 16);
			// eval_pair's exp_loop and not a bare MUFU.EX2 (6 instructions less): T below is rebuilt as final_T / prod (1 - alpha), which
			// only returns the forward's T when alpha is the forward's alpha bit for bit.  With a G that is off by 3e-7 the error grows
			// along the pixel's list (x alpha / (1 - alpha) per entry) and reaches 3e-5 of the gradients' scale at 1080p, 100x the
			// run-to-run gap.
			const PairAlpha pa = eval_pair(r0, r1, wp);
			const float G = pa.G, alpha = pa.alpha;
			// the forward's skips (pos < last_contributor replaces the `contributor` countdown)
			const bool active = pair_passes((int)jj > first, pa, r0.w);
			if (!__any_sync(0xffffffffu, active)) continue;
			float wv = 0.f, uv = 0.f;
			const float4 r2 = lds128(addr + 32);                               // (G, B, depth, Gaussian id)
			if (active)
			{
				// backward.cu:541 T = T / (1 - alpha), 1 - alpha in [0.01, 1]
				const float inv = rcp_approx(1.0f - alpha);
				T = T * inv;
				uv = alpha * T;
				// backward.cu:547-556 carries accum_rec_c = last_alpha * last_colour_c + (1 - last_alpha) * accum_rec_c per channel and
				// forms dL/dalpha = sum_c (colour_c - accum_rec_c) * dL/dpixel_c.  dL/dpixel is constant along the pixel's list and the
				// recurrence is linear, so its dot product is carried instead: k = colour . dL/dpixel (with MAPS: + 1/depth * dL/dinvdepth),
				// ard = sum_c accum_rec_c * dL/dpixel_c, and ard' = ard + last_alpha * (k_last - ard) is one FMA on dl = k_last - ard, the
				// difference the entry before has formed anyway (a single rounding: rounding alpha * dl first costs accuracy on
				// 1000-entry lists).  Two instructions and three registers of state for any number of channels.
				float k = r1.w * dLp0;
				k = fmaf(r2.x, dLp1, k);
				k = fmaf(r2.y, dLp2, k);
				if (MAPS) k = fmaf(rcp_approx(r2.z), dLd, k);
				ard = fmaf(la, dl, ard);
				const float d = k - ard;
				dl = d; la = alpha;
				wv = G * fmaf(inv, nbg, d * T);
			}
			{
				const uint32_t sa = wbase + (nrows * STASH_LD + lane) * 4;
				asm volatile("st.shared.f32 [%0], %1;" ::"r"(sa), "f"(wv) : "memory");
				asm volatile("st.shared.f32 [%0+%2], %1;" ::"r"(sa), "f"(uv), "n"(BW_OFF_U) : "memory");
				if (lane == 0) asm volatile("st.shared.f32 [%0+%2], %1;" ::"r"(wbase + nrows * 4), "f"(DET ? __uint_as_float(jj) : r2.w), "n"(BW_OFF_ROWID(NCH)) : "memory");
			}
			nrows++;
			if (nrows == 16) flush_rows();
		}
		if (DET)
		{
			flush_rows();
			__syncthreads();
			// 4 threads per batch entry j, components k0, k0 + 4, k0 + 8: the 8 warps' rows added in warp order, then zeroed
			const int j = tid >> 2;
			if (j < n)
			{
				const uint32_t gid = __float_as_uint(S.rec[buf][3 * j + 2].w);
				const TileRect tr(rect[gid]);
				const unsigned long long slot = tr.slot(slot_offset[gid], blockIdx.x, blockIdx.y);
				for (int k = tid & 3; k < NS; k += 4)
				{
					float s = ebuf[j * NS + k];
					ebuf[j * NS + k] = 0.0f;
#pragma unroll
					for (int w = 1; w < 8; w++)
					{
						s += ebuf[(w * BWD_BATCH + j) * NS + k];
						ebuf[(w * BWD_BATCH + j) * NS + k] = 0.0f;
					}
					if (slot < num_slots) parts[slot * NS + k] = s;       // out of range only for blobs that do not match R (det_gather flags it)
				}
			}
			__syncthreads();
		}
		__syncwarp();
		if (lane == 0) mbar_arrive(&S.empty[buf]);           // this warp no longer reads the stage (stashed rows carry their own data)
	}
	flush_rows();                                            // only the tile's tail is a partial block
}

// ------------------------------------------------------------------------------------------------
// The fixed-point totals of render_forward_kernel<true, false, true> as floats: one rounding each (the scaling is exact).
__global__ void __launch_bounds__(256) stats_fixed_to_float_kernel(int P, const unsigned long long* __restrict__ fixed, float* __restrict__ out)
{
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i < P) out[i] = __fmul_rn(__ull2float_rn(fixed[i]), 1.0f / STATS_FIXED_SCALE);
}

int launch_stats_fixed_to_float(int P, const unsigned long long* fixed, float* out, cudaStream_t stream)
{
	if (P <= 0) return GSB_OK;
	ProfScope prof(K_TOOLS, stream);
	stats_fixed_to_float_kernel<<<(P + 255) / 256, 256, 0, stream>>>(P, fixed, out);
	GSB_LAUNCHED();
	GSB_CUDA_OK(cudaGetLastError());
	return GSB_OK;
}

int launch_render_forward(const GsbForwardRequest& req, const ImageState& img, const BinningState& b, const GeomState& g)
{
	const int W = req.cam->width, H = req.cam->height;
	const dim3 grid = tile_grid(W, H);
	const bool stats = statistics(req), fixed = stats_fixed(req);
	const bool maps = !stats && req.out_invdepth && req.out_alpha;
	float* const transmittance = fixed ? reinterpret_cast<float*>(transmittance_fixed(req)) : req.transmittance_sum;
	const cudaStream_t stream = stream_of(req);
	ProfScope prof(K_RENDER_FWD, stream);
	return dispatch([&](auto stats, auto maps, auto fixed) -> int {
		// four variants exist: <F,F>, <F,T>, <T,F> and <T,F,T> (statistics go without maps; fixed point only with statistics)
		if constexpr (!(stats && maps) && (stats || !fixed))
			render_forward_kernel<stats, maps, fixed><<<grid, 256, 0, stream>>>(img.ranges, b.point_list, W, H, g.rec,
				req.cam->background, img.final_T, img.n_contrib, req.out_color, img.tile_max_contrib, stats ? req.touched_pixels : nullptr,
				stats ? transmittance : nullptr, maps ? req.out_invdepth : nullptr, maps ? req.out_alpha : nullptr);
		GSB_LAUNCHED();
		GSB_CUDA_OK(cudaGetLastError());
		return GSB_OK;
	}, stats, maps, fixed);
}

int launch_render_backward(const GsbBackwardRequest& req, const ImageState& img, const BinningState& b, const GeomState& g, float* acc,
	float* parts, const uint32_t* slot_offset)
{
	const int W = req.cam->width, H = req.cam->height;
	const dim3 grid = tile_grid(W, H);
	const cudaStream_t stream = stream_of(req);
	return dispatch([&](auto maps, auto det, auto abs) -> int {
		constexpr int ns = abs ? DET_NS_ABS : DET_NS(maps);
		const size_t smem = sizeof(BwdSmem<maps ? 4 : 3>) + (det ? size_t(8) * BWD_BATCH * ns * sizeof(float) : 0);
		auto kernel = render_backward_kernel<maps, det, abs>;
		if (int e = ensure_dyn_smem((const void*)kernel, (int)smem)) return e;
		if (det)
		{
			// instances behind a tile's last contributor (and tiles with none) are never visited: their slots must read as zero
			ProfScope prof(K_DET_CLEAR, stream);
			GSB_CUDA_OK(cudaMemsetAsync(parts, 0, size_t(req.num_rendered) * ns * sizeof(float), stream));
		}
		ProfScope prof(K_RENDER_BWD, stream);
		// the per-Gaussian accumulator the kernel reduces into (12 floats per Gaussian, inside the geometry blob)
		if (!det) GSB_CUDA_OK(cudaMemsetAsync(acc, 0, size_t(req.scene->P) * 48, stream));
		kernel<<<grid, 256, smem, stream>>>(img.ranges, b.point_list, W, H, g.rec, req.cam->background,
			img.final_T, img.n_contrib, img.tile_max_contrib, req.dL_dout_color, det ? nullptr : acc, req.dL_dinvdepth, req.dL_dalpha,
			parts, slot_offset, det ? g.rect : nullptr, det ? (unsigned long long)req.num_rendered : 0ull);
		GSB_LAUNCHED();
		GSB_CUDA_OK(cudaGetLastError());
		return GSB_OK;
	}, req.dL_dinvdepth || req.dL_dalpha, req.deterministic != 0, req.dL_dmeans2D_abs != nullptr);
}

// dL_dmeans2D_abs [P,3] = (0.5 W slot 10, 0.5 H slot 11, 0): the constant factors of backward.cu:583-589, applied as the preprocess
// backward applies them to slots 4 and 5; culled and pruned Gaussians (radii 0) get zero rows.
__global__ void __launch_bounds__(256) absgrad_finish_kernel(int P, const int32_t* __restrict__ radii, const float* __restrict__ acc,
	float half_w, float half_h, float* __restrict__ out)
{
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= P) return;
	const bool vis = radii[i] > 0;
	const float2 s = reinterpret_cast<const float2*>(acc)[6 * (size_t)i + 5];
	out[3 * (size_t)i] = vis ? s.x * half_w : 0.0f;
	out[3 * (size_t)i + 1] = vis ? s.y * half_h : 0.0f;
	out[3 * (size_t)i + 2] = 0.0f;
}

int launch_absgrad_finish(const GsbBackwardRequest& req, const float* acc)
{
	const int P = req.scene->P;
	if (P <= 0) return GSB_OK;
	const cudaStream_t stream = stream_of(req);
	ProfScope prof(K_ABSGRAD_FINISH, stream);
	absgrad_finish_kernel<<<(P + 255) / 256, 256, 0, stream>>>(P, req.radii, acc, 0.5f * req.cam->width, 0.5f * req.cam->height,
		req.dL_dmeans2D_abs);
	GSB_LAUNCHED();
	GSB_CUDA_OK(cudaGetLastError());
	return GSB_OK;
}

} // namespace gsb
