// gsb_densify.cu — densification statistics, clone / split / prune of the model and its optimizer state (gs_b200.densify;
// DESIGN.md §5g).
//
// The reference (gaussian_model.py:553-695) boolean-indexes and concatenates all six params and their twelve moments four
// times per densify_and_prune and synchronises the host about ten times.  Here:
//   densify_stats_kernel  the per-iteration statistics (train.py:134-135) in one pass;
//   densify_plan_kernel   per row: the clone / split / survive flags and their ranks, by one ordered scan (the decoupled
//                         look-back of the onesweep sort, five channels); the last tile writes the counts the host reads back;
//   densify_emit_kernel   every output row of every tensor in one launch: each source element goes to its kept row, its clone
//                         and its two children.
// Arithmetic: every op the reference runs through torch is spelled out with the rounding tools/probe_torch_densify.py observed
// on an H100: exp == exp_ref, sigmoid == 1 / (1 + exp(-x)) with IEEE division, the norm unfused, division by the Python scalar
// 0.8 * N a multiplication by its fp32 reciprocal, comparisons against the fp32 casts of the thresholds, log == CUDA logf
// (what torch.log calls).  torch.bmm's contraction order for the children's offsets depends on the batch size (cuBLAS); the
// kernel uses the order the probe matched most often, so those values agree only to rounding (DESIGN.md §5g).  The emit table's
// checks, the CTA scan, the grid size and the row range are gsb_common.cuh's, shared with gsb_mcmc.cu and gsb_mercy.cu.
#include "gsb_common.cuh"

namespace gsb {

#define DENS_THREADS 256
#define DENS_ITEMS 4
#define DENS_TILE (DENS_THREADS * DENS_ITEMS)
#define DENS_CH 5              // channels of the scan: kept originals, clones, kept clones, split parents, kept children
#define DENS_LB_STRIDE 8
#define DENS_FIELD 12          // bits per channel in the packed per-thread / per-CTA counts (a tile has at most 1024 rows)

struct DensifyWorkspace {
	int4* rows;                // per source row: rank of the kept row, the kept clone, the split parent, the kept children; -1 = none
	float* split_std;          // [P, 3]: exp(scaling) of the split parents, by split rank
	uint32_t* lookback;        // [n_tiles, DENS_LB_STRIDE]
	uint32_t* ticket;
	uint32_t n_tiles;
	size_t bytes, std_offset;
};
static DensifyWorkspace densify_carve(char* base, int P)
{
	Carver c(base);
	DensifyWorkspace w;
	const size_t n = P > 0 ? (size_t)P : 1;
	w.n_tiles = (uint32_t)((n + DENS_TILE - 1) / DENS_TILE);
	w.rows = c.take<int4>(n);
	w.split_std = c.take<float>(3 * n);
	w.std_offset = (size_t)(reinterpret_cast<char*>(w.split_std) - base);
	w.lookback = c.take<uint32_t>((size_t)w.n_tiles * DENS_LB_STRIDE);
	w.ticket = c.take<uint32_t>(1);
	w.bytes = c.off + 256;
	return w;
}

struct PlanArgs {
	const float *accum, *denom, *scaling, *opacity, *max_radii2D;
	const uint8_t* mask;
	float max_grad, clone_max_scale, min_opacity, max_screen_size, big_scale, split_factor;
	const float* accum_abs;    // non-NULL: the split test reads accum_abs / denom against max_grad_abs (AbsGS)
	float max_grad_abs;
	int P, mode, screen_test;
};

// torch.max(t, dim=1).values of a row: NaN if any element is NaN
__device__ __forceinline__ float max3_torch(float a, float b, float c)
{
	if (isnan(a) || isnan(b) || isnan(c)) return __int_as_float(0x7fc00000);
	return fmaxf(fmaxf(a, b), c);
}
// prune()'s test of one row (gaussian_model.py:685-689)
__device__ __forceinline__ bool pruned(const PlanArgs& a, float opacity_logit, float radius, float max_scale)
{
	return sigmoid_torch(opacity_logit) < a.min_opacity || (a.screen_test && (radius > a.max_screen_size || max_scale > a.big_scale));
}

// bit c of the result = row r counts in channel c
__device__ __forceinline__ unsigned row_flags(const PlanArgs& a, long long r)
{
	if (a.mode == GSB_DENSIFY_PRUNE_MASK) return a.mask[r] ? 0u : 1u;
	const float e0 = exp_ref(a.scaling[3 * r]), e1 = exp_ref(a.scaling[3 * r + 1]), e2 = exp_ref(a.scaling[3 * r + 2]);
	const float ms = max3_torch(e0, e1, e2), op = a.opacity[r];
	if (a.mode == GSB_DENSIFY_PRUNE) return pruned(a, op, a.max_radii2D[r], ms) ? 0u : 1u;
	float g = __fdiv_rn(a.accum[r], a.denom[r]);
	if (isnan(g)) g = 0.0f;
	// densify_and_clone (:653-655) and densify_and_split (:626-630).  A clone's padded grad is 0 and its scaling is the parent's,
	// which passed max <= clone_max_scale, so its split test (0 >= max_grad && max > clone_max_scale) is false for every max_grad:
	// clones are never split.
	const bool hot = g >= a.max_grad;
	const bool clone = hot && ms <= a.clone_max_scale;
	bool split = hot && ms > a.clone_max_scale;
	if (a.accum_abs)
	{
		// AbsGS (DESIGN.md §5m): the split test takes the absolute gradient; a clone's padded value is 0 and its scale passed the
		// clone test, so clones are still never split
		float ga = __fdiv_rn(a.accum_abs[r], a.denom[r]);
		if (isnan(ga)) ga = 0.0f;
		split = ga >= a.max_grad_abs && ms > a.clone_max_scale;
	}
	// prune() after both (:685-689): max_radii2D was reset to zeros by densification_postfix (:620)
	const bool gone = pruned(a, op, 0.0f, ms);
	unsigned f = (!split && !gone ? 1u : 0u) | (clone ? 2u : 0u) | (clone && !gone ? 4u : 0u);
	if (split)
	{
		// a child's scaling: log(exp(s) / (0.8 * N)); its prune test reads exp() of that
		const float c0 = exp_ref(logf(__fmul_rn(e0, a.split_factor))), c1 = exp_ref(logf(__fmul_rn(e1, a.split_factor)));
		const float c2 = exp_ref(logf(__fmul_rn(e2, a.split_factor)));
		f |= 8u | (!pruned(a, op, 0.0f, max3_torch(c0, c1, c2)) ? 16u : 0u);
	}
	return f;
}

__device__ __forceinline__ unsigned long long pack_flags(unsigned f)
{
	unsigned long long p = 0;
#pragma unroll
	for (int c = 0; c < DENS_CH; c++) p |= (unsigned long long)((f >> c) & 1u) << (DENS_FIELD * c);
	return p;
}
__device__ __forceinline__ uint32_t field(unsigned long long p, int c) { return (uint32_t)(p >> (DENS_FIELD * c)) & ((1u << DENS_FIELD) - 1u); }

__global__ void __launch_bounds__(DENS_THREADS) densify_plan_kernel(const PlanArgs a, DensifyWorkspace w, long long* __restrict__ counts)
{
	__shared__ uint32_t s_tile;
	__shared__ unsigned long long s_warp[DENS_THREADS / 32];
	__shared__ uint32_t s_excl[DENS_CH], s_total[DENS_CH];
	const int tid = threadIdx.x;
	if (tid == 0) s_tile = atomicAdd(w.ticket, 1u);
	__syncthreads();
	const uint32_t tile = s_tile;
	const long long row0 = (long long)tile * DENS_TILE + (long long)tid * DENS_ITEMS;
	unsigned flags[DENS_ITEMS];
	unsigned long long mine = 0;
#pragma unroll
	for (int i = 0; i < DENS_ITEMS; i++)
	{
		flags[i] = row0 + i < a.P ? row_flags(a, row0 + i) : 0u;
		mine += pack_flags(flags[i]);
	}
	unsigned long long cta_total;
	unsigned long long run = cta_exclusive<DENS_THREADS>(mine, s_warp, &cta_total);
	if (tid < DENS_CH)
	{
		const uint32_t total = field(cta_total, tid);
		s_total[tid] = total;
		s_excl[tid] = lookback_exclusive(w.lookback, tile, DENS_LB_STRIDE, tid, total);
	}
	__syncthreads();
	if (tid == 0 && tile == w.n_tiles - 1)
	{
		long long n[DENS_CH];
		for (int c = 0; c < DENS_CH; c++) { n[c] = (long long)s_excl[c] + s_total[c]; counts[c] = n[c]; }
		const long long out = n[0] + n[2] + 2 * n[4];
		counts[5] = out;
		counts[6] = (a.mode == GSB_DENSIFY_CLONE_SPLIT ? (long long)a.P + n[1] + n[3] : (long long)a.P) - out;
		counts[7] = 0;
	}
#pragma unroll
	for (int i = 0; i < DENS_ITEMS; i++)
	{
		const long long r = row0 + i;
		if (r >= a.P) break;
		const unsigned f = flags[i];
		int4 rec;
		rec.x = (f & 1u) ? (int)(s_excl[0] + field(run, 0)) : -1;
		rec.y = (f & 4u) ? (int)(s_excl[2] + field(run, 2)) : -1;
		rec.z = (f & 8u) ? (int)(s_excl[3] + field(run, 3)) : -1;
		rec.w = (f & 16u) ? (int)(s_excl[4] + field(run, 4)) : -1;
		w.rows[r] = rec;
		if (f & 8u)
		{
			float* s = w.split_std + 3 * (size_t)rec.z;
			s[0] = exp_ref(a.scaling[3 * r]); s[1] = exp_ref(a.scaling[3 * r + 1]); s[2] = exp_ref(a.scaling[3 * r + 2]);
		}
		run += pack_flags(f);
	}
}

// build_rotation (general_utils.py:78-99) row c of the normalised quaternion's matrix, every torch op rounded on its own
__device__ __forceinline__ void rotation_row(const float* q4, int c, float R[3])
{
	const float q0 = q4[0], q1 = q4[1], q2 = q4[2], q3 = q4[3];
	const float nrm = __fsqrt_rn(__fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(q0, q0), __fmul_rn(q1, q1)), __fmul_rn(q2, q2)), __fmul_rn(q3, q3)));
	const float r = __fdiv_rn(q0, nrm), x = __fdiv_rn(q1, nrm), y = __fdiv_rn(q2, nrm), z = __fdiv_rn(q3, nrm);
	if (c == 0)
	{
		R[0] = __fsub_rn(1.0f, __fmul_rn(2.0f, __fadd_rn(__fmul_rn(y, y), __fmul_rn(z, z))));
		R[1] = __fmul_rn(2.0f, __fsub_rn(__fmul_rn(x, y), __fmul_rn(r, z)));
		R[2] = __fmul_rn(2.0f, __fadd_rn(__fmul_rn(x, z), __fmul_rn(r, y)));
	}
	else if (c == 1)
	{
		R[0] = __fmul_rn(2.0f, __fadd_rn(__fmul_rn(x, y), __fmul_rn(r, z)));
		R[1] = __fsub_rn(1.0f, __fmul_rn(2.0f, __fadd_rn(__fmul_rn(x, x), __fmul_rn(z, z))));
		R[2] = __fmul_rn(2.0f, __fsub_rn(__fmul_rn(y, z), __fmul_rn(r, x)));
	}
	else
	{
		R[0] = __fmul_rn(2.0f, __fsub_rn(__fmul_rn(x, z), __fmul_rn(r, y)));
		R[1] = __fmul_rn(2.0f, __fadd_rn(__fmul_rn(y, z), __fmul_rn(r, x)));
		R[2] = __fsub_rn(1.0f, __fmul_rn(2.0f, __fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y))));
	}
}
// bmm(rots, samples)[c] + xyz[c]: (R0 s0 + R1 s1) + R2 s2, unfused (the probe's closest candidate), then the add
__device__ __forceinline__ float child_xyz(const float* q4, const float* smp, float mu, int c)
{
	float R[3];
	rotation_row(q4, c, R);
	const float d = __fadd_rn(__fadd_rn(__fmul_rn(R[0], smp[0]), __fmul_rn(R[1], smp[1])), __fmul_rn(R[2], smp[2]));
	return __fadd_rn(d, mu);
}

// grid.y = table entry; grid.x strides over its P * row_width elements.  Each source element is read once and written to the
// kept row, the kept clone and the two kept children of its row (a -1 rank skips the destination).
__global__ void __launch_bounds__(DENS_THREADS) densify_emit_kernel(const __grid_constant__ RowTable tab, const int4* __restrict__ rows,
	long long P, long long clone_base, long long child1_base, long long child2_base, long long S, const float* __restrict__ rotation,
	const float* __restrict__ samples, float split_factor)
{
	const GsbDensifyTensor& k = tab.t[blockIdx.y];
	const int w = k.row_width;
	const long long total = P * w, stride = (long long)gridDim.x * DENS_THREADS;
	const uint32_t* __restrict__ src = static_cast<const uint32_t*>(k.src);
	uint32_t* __restrict__ dst = static_cast<uint32_t*>(k.dst);
	for (long long e = (long long)blockIdx.x * DENS_THREADS + threadIdx.x; e < total; e += stride)
	{
		long long r;
		int c;
		row_col(e, w, tab.inv_width[blockIdx.y], r, c);
		const int4 rec = __ldg(rows + r);
		if ((rec.x & rec.y & rec.w) < 0) continue;           // all three destinations are -1 (the split rank alone writes nothing)
		const uint32_t v = __ldcs(src + e);
		if (rec.x >= 0)
		{
			const long long d = (long long)rec.x * w + c;
			__stcs(dst + d, v);
			if (k.exp_avg_src)
			{
				__stcs(k.exp_avg_dst + d, __ldcs(k.exp_avg_src + e));
				__stcs(k.exp_avg_sq_dst + d, __ldcs(k.exp_avg_sq_src + e));
			}
			if (k.grad_src) __stcs(k.grad_dst + d, __ldcs(k.grad_src + e));
		}
		if (rec.y >= 0)
		{
			const long long d = (clone_base + rec.y) * w + c;
			__stcs(dst + d, v);
			if (k.exp_avg_src) { __stcs(k.exp_avg_dst + d, 0.0f); __stcs(k.exp_avg_sq_dst + d, 0.0f); }
			if (k.grad_src) __stcs(k.grad_dst + d, 0.0f);
		}
		if (rec.w >= 0)
		{
			const long long d1 = (child1_base + rec.w) * w + c, d2 = (child2_base + rec.w) * w + c;
			uint32_t v1 = v, v2 = v;
			if (k.kind == GSB_DENSIFY_XYZ)
			{
				const float mu = __uint_as_float(v);
				v1 = __float_as_uint(child_xyz(rotation + 4 * r, samples + 3 * (long long)rec.z, mu, c));
				v2 = __float_as_uint(child_xyz(rotation + 4 * r, samples + 3 * (S + rec.z), mu, c));
			}
			else if (k.kind == GSB_DENSIFY_SCALING)
				v1 = v2 = __float_as_uint(logf(__fmul_rn(exp_ref(__uint_as_float(v)), split_factor)));
			__stcs(dst + d1, v1);
			__stcs(dst + d2, v2);
			if (k.exp_avg_src)
			{
				__stcs(k.exp_avg_dst + d1, 0.0f); __stcs(k.exp_avg_sq_dst + d1, 0.0f);
				__stcs(k.exp_avg_dst + d2, 0.0f); __stcs(k.exp_avg_sq_dst + d2, 0.0f);
			}
			if (k.grad_src) { __stcs(k.grad_dst + d1, 0.0f); __stcs(k.grad_dst + d2, 0.0f); }
		}
	}
}

// the per-iteration statistics: train.py:134 and add_densification_stats (gaussian_model.py:693-695); ABS also adds the norm of
// the absolute gradient's first two columns to accum_abs
template <bool ABS>
__global__ void __launch_bounds__(DENS_THREADS) densify_stats_kernel(long long P, const float* __restrict__ grad, int grad_stride,
	const uint8_t* __restrict__ visibility, const int32_t* __restrict__ radii, float* __restrict__ accum, float* __restrict__ denom,
	float* __restrict__ max_radii2D, const float* __restrict__ grad_abs = nullptr, int abs_stride = 0, float* __restrict__ accum_abs = nullptr)
{
	const long long stride = (long long)gridDim.x * DENS_THREADS;
	for (long long i = (long long)blockIdx.x * DENS_THREADS + threadIdx.x; i < P; i += stride)
	{
		const float g0 = grad[i * grad_stride], g1 = grad[i * grad_stride + 1];
		accum[i] = __fadd_rn(accum[i], __fsqrt_rn(__fadd_rn(__fmul_rn(g0, g0), __fmul_rn(g1, g1))));
		if (ABS)
		{
			const float a0 = grad_abs[i * abs_stride], a1 = grad_abs[i * abs_stride + 1];
			accum_abs[i] = __fadd_rn(accum_abs[i], __fsqrt_rn(__fadd_rn(__fmul_rn(a0, a0), __fmul_rn(a1, a1))));
		}
		const bool vis = visibility[i] != 0;
		denom[i] = __fadd_rn(denom[i], vis ? 1.0f : 0.0f);
		if (radii && vis)
		{
			const float m = max_radii2D[i];
			max_radii2D[i] = isnan(m) ? m : fmaxf(m, (float)radii[i]);   // torch.maximum: NaN propagates
		}
	}
}

static const TableRules kEmitRules = {"densify_emit", "n",
	(1u << GSB_DENSIFY_COPY) | (1u << GSB_DENSIFY_XYZ) | (1u << GSB_DENSIFY_SCALING),
	"%s: tensor %d: unknown kind %d", "%s: tensor %d: an xyz / scaling entry needs row_width 3, got %d", true};

} // namespace gsb

using namespace gsb;

extern "C" size_t gsb_densify_workspace_bytes(int32_t P) { return densify_carve(nullptr, P).bytes; }
extern "C" size_t gsb_densify_split_std_offset(int32_t P) { return densify_carve(nullptr, P).std_offset; }

extern "C" int gsb_densify_stats(int32_t P, const float* viewspace_grad, int32_t grad_row_stride, const float* viewspace_grad_abs,
	int32_t abs_row_stride, const uint8_t* visibility, const int32_t* radii, float* xyz_gradient_accum, float* xyz_gradient_accum_abs,
	float* denom, float* max_radii2D, void* stream)
{
	if (P < 0) { set_error("densify_stats: P < 0"); return GSB_EINVAL; }
	if (grad_row_stride < 2) { set_error("densify_stats: grad_row_stride %d < 2", grad_row_stride); return GSB_EINVAL; }
	const bool abs = viewspace_grad_abs != nullptr;
	if (abs != (xyz_gradient_accum_abs != nullptr))
	{ set_error("densify_stats: viewspace_grad_abs and xyz_gradient_accum_abs must be both NULL or both set"); return GSB_EINVAL; }
	if (abs && abs_row_stride < 2) { set_error("densify_stats: abs_row_stride %d must be >= 2", abs_row_stride); return GSB_EINVAL; }
	if (radii && !max_radii2D) { set_error("densify_stats: radii given without max_radii2D"); return GSB_EINVAL; }
	if (P == 0) return GSB_OK;
	if (!viewspace_grad || !visibility || !xyz_gradient_accum || !denom)
	{ set_error("densify_stats: NULL viewspace_grad / visibility / xyz_gradient_accum / denom"); return GSB_EINVAL; }
	const cudaStream_t st = (cudaStream_t)stream;
	ProfScope prof(K_TOOLS, st);
	if (abs)
		densify_stats_kernel<true><<<grid_stride_ctas(P, DENS_THREADS, 8), DENS_THREADS, 0, st>>>(P, viewspace_grad, grad_row_stride, visibility, radii,
			xyz_gradient_accum, denom, max_radii2D, viewspace_grad_abs, abs_row_stride, xyz_gradient_accum_abs);
	else
		densify_stats_kernel<false><<<grid_stride_ctas(P, DENS_THREADS, 8), DENS_THREADS, 0, st>>>(P, viewspace_grad, grad_row_stride, visibility, radii,
			xyz_gradient_accum, denom, max_radii2D);
	GSB_LAUNCHED();
	GSB_CUDA_OK(cudaGetLastError());
	return GSB_OK;
}

// xyz_gradient_accum_abs non-NULL: the AbsGS split test (GSB_DENSIFY_CLONE_SPLIT only)
extern "C" int gsb_densify_plan(int32_t P, int32_t mode, const float* xyz_gradient_accum, const float* xyz_gradient_accum_abs,
	const float* denom, const float* scaling, const float* opacity, const float* max_radii2D, const uint8_t* prune_mask, float max_grad,
	float max_grad_abs, float clone_max_scale, float min_opacity, int32_t screen_test, float max_screen_size, float big_scale,
	float split_scale_factor, void* workspace, int64_t* counts, void* stream)
{
	if (!rows_ok("densify_plan", P)) return GSB_EINVAL;
	if (mode != GSB_DENSIFY_CLONE_SPLIT && mode != GSB_DENSIFY_PRUNE && mode != GSB_DENSIFY_PRUNE_MASK)
	{ set_error("densify_plan: unknown mode %d", mode); return GSB_EINVAL; }
	if (xyz_gradient_accum_abs && mode != GSB_DENSIFY_CLONE_SPLIT)
	{ set_error("densify_plan: xyz_gradient_accum_abs given with mode %d; only GSB_DENSIFY_CLONE_SPLIT reads it", mode); return GSB_EINVAL; }
	if (!workspace || !counts) { set_error("densify_plan: NULL workspace / counts"); return GSB_EINVAL; }
	if (P > 0)
	{
		if (mode == GSB_DENSIFY_PRUNE_MASK && !prune_mask) { set_error("densify_plan: NULL prune_mask"); return GSB_EINVAL; }
		if (mode != GSB_DENSIFY_PRUNE_MASK && (!scaling || !opacity)) { set_error("densify_plan: NULL scaling / opacity"); return GSB_EINVAL; }
		if (mode == GSB_DENSIFY_PRUNE && screen_test && !max_radii2D) { set_error("densify_plan: NULL max_radii2D"); return GSB_EINVAL; }
		if (mode == GSB_DENSIFY_CLONE_SPLIT && (!xyz_gradient_accum || !denom))
		{ set_error("densify_plan: NULL xyz_gradient_accum / denom"); return GSB_EINVAL; }
	}
	const cudaStream_t st = (cudaStream_t)stream;
	ProfScope prof(K_TOOLS, st);
	if (P == 0)
	{
		GSB_CUDA_OK(cudaMemsetAsync(counts, 0, sizeof(int64_t) * GSB_DENSIFY_COUNTS, st));
		return GSB_OK;
	}
	const DensifyWorkspace w = densify_carve(static_cast<char*>(workspace), P);
	GSB_CUDA_OK(cudaMemsetAsync(w.lookback, 0, sizeof(uint32_t) * ((size_t)w.n_tiles * DENS_LB_STRIDE), st));
	GSB_CUDA_OK(cudaMemsetAsync(w.ticket, 0, sizeof(uint32_t), st));
	PlanArgs a;
	a.accum = xyz_gradient_accum; a.denom = denom; a.scaling = scaling; a.opacity = opacity; a.max_radii2D = max_radii2D; a.mask = prune_mask;
	a.max_grad = max_grad; a.clone_max_scale = clone_max_scale; a.min_opacity = min_opacity; a.max_screen_size = max_screen_size;
	a.big_scale = big_scale; a.split_factor = split_scale_factor; a.P = P; a.mode = mode; a.screen_test = screen_test ? 1 : 0;
	a.accum_abs = xyz_gradient_accum_abs; a.max_grad_abs = max_grad_abs;
	densify_plan_kernel<<<w.n_tiles, DENS_THREADS, 0, st>>>(a, w, reinterpret_cast<long long*>(counts));
	GSB_LAUNCHED();
	GSB_CUDA_OK(cudaGetLastError());
	return GSB_OK;
}

extern "C" int gsb_densify_emit(const GsbDensifyTensor* tensors, int32_t n, int32_t P, const void* workspace, int64_t n_kept,
	int64_t n_clones_kept, int64_t n_split, int64_t n_children_kept, const float* rotation, const float* samples,
	float split_scale_factor, void* stream)
{
	if (!rows_ok("densify_emit", P)) return GSB_EINVAL;
	if (n_kept < 0 || n_clones_kept < 0 || n_split < 0 || n_children_kept < 0 || n_kept > P || n_clones_kept > P || n_split > P ||
		n_children_kept > n_split)
	{ set_error("densify_emit: inconsistent counts"); return GSB_EINVAL; }
	if (!workspace) { set_error("densify_emit: NULL workspace"); return GSB_EINVAL; }
	// an empty output has no storage (NULL destinations): only a call that writes rows needs its pointers
	const bool rows_out = n_kept + n_clones_kept + n_children_kept > 0;
	RowTable tab{};
	int max_w;
	if (!fill_row_table(kEmitRules, tensors, n, rows_out, rows_out, tab, max_w)) return GSB_EINVAL;
	for (int i = 0; i < n; i++)
		if (tensors[i].kind == GSB_DENSIFY_XYZ && n_children_kept > 0 && (!rotation || !samples))
		{ set_error("densify_emit: split children need rotation and samples"); return GSB_EINVAL; }
	if (n == 0 || P == 0 || !rows_out) return GSB_OK;
	const DensifyWorkspace w = densify_carve(static_cast<char*>(const_cast<void*>(workspace)), P);
	const cudaStream_t st = (cudaStream_t)stream;
	ProfScope prof(K_TOOLS, st);
	const dim3 grid((unsigned)grid_stride_ctas((long long)P * max_w, DENS_THREADS, 8), (unsigned)n);
	densify_emit_kernel<<<grid, DENS_THREADS, 0, st>>>(tab, w.rows, P, n_kept, n_kept + n_clones_kept, n_kept + n_clones_kept + n_children_kept,
		n_split, rotation, samples, split_scale_factor);
	GSB_LAUNCHED();
	GSB_CUDA_OK(cudaGetLastError());
	return GSB_OK;
}
