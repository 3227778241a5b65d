// gsb_mcmc.cu — 3DGS-MCMC densification (Kheradmand et al. 2024; gs_b200.mcmc, DESIGN.md §5n): the position noise, the
// opacity-weighted sampler and the relocation of dead Gaussians / growth to a budget, with the model's Adam moments.
//
//   mcmc_noise_kernel        xyz += R diag(s)^2 R^T v per row, v = draws * gate * noise_lr * xyz_lr, in double (one launch);
//   mcmc_reduce_kernel       plan, first phase: per 1024-row tile the sum of the fixed-point weights and the dead rows;
//   mcmc_tile_scan_kernel    one CTA: the exclusive prefix of the tile sums and the totals (counts);
//   mcmc_scan_kernel         the inclusive weight prefix per row and the list of dead rows in row order;
//   mcmc_sample_kernel       plan, second phase: each draw's source row (integer inverse CDF), its histogram and the first draw
//                            that picked each source (its owner, which alone writes the source row);
//   mcmc_values_kernel       the relocated opacity and scales of every distinct source (paper eq. 9, in double);
//   mcmc_emit_*_kernel       the rows: in place over the dead rows (relocate), or into [P + n] copies (add).
// Every step of the sampler is integer arithmetic and every histogram count is exact, so the same draws give the same bytes.
#include "gsb_common.cuh"

namespace gsb {

#define MC_THREADS 256
#define MC_ITEMS 4
#define MC_TILE (MC_THREADS * MC_ITEMS)
#define MC_SCAN_THREADS 1024
#define MC_DEAD_BITS 11            // a tile's dead count (<= 1024) sits below its weight sum (< 2^43) in one packed word
#define MC_N_MAX 50                // N = min(count + 1, MC_N_MAX)

struct McmcWorkspace {
	float4* values;                // [P] per sampled source: (o', s'0, s'1, s'2) before the logit / log; at offset 0
	unsigned long long* prefix;    // [P] inclusive prefix of the weights
	int32_t* dead_rows;            // [P] the dead rows in row order
	uint32_t* count;               // [P] draws per source row
	uint32_t* owner;               // [P] the first draw that picked the row (0xffffffff: none)
	int32_t* source;               // [P] source row of each draw
	unsigned long long* tile_sum;  // [n_tiles] packed (weight << MC_DEAD_BITS | dead)
	unsigned long long* tile_w;    // [n_tiles] exclusive weight prefix
	uint32_t* tile_d;              // [n_tiles] exclusive dead prefix
	unsigned long long* totals;    // [2] total weight, dead rows
	uint32_t n_tiles;
	size_t bytes;
};
static McmcWorkspace mcmc_carve(char* base, int P)
{
	Carver c(base);
	McmcWorkspace w;
	const size_t n = P > 0 ? (size_t)P : 1;
	w.n_tiles = (uint32_t)((n + MC_TILE - 1) / MC_TILE);
	w.values = c.take<float4>(n);
	w.prefix = c.take<unsigned long long>(n);
	w.dead_rows = c.take<int32_t>(n);
	w.count = c.take<uint32_t>(n);
	w.owner = c.take<uint32_t>(n);
	w.source = c.take<int32_t>(n);
	w.tile_sum = c.take<unsigned long long>(w.n_tiles);
	w.tile_w = c.take<unsigned long long>(w.n_tiles);
	w.tile_d = c.take<uint32_t>(w.n_tiles);
	w.totals = c.take<unsigned long long>(2);
	w.bytes = c.off + 256;
	return w;
}

// ------------------------------------------------------------------------------------------------ position noise
// build_rotation of a normalised quaternion (general_utils.py), in double: it divides by the norm once more
__device__ __forceinline__ void rotation_d(float r0, float x0, float y0, float z0, double R[3][3])
{
	const double n = sqrt((double)r0 * r0 + (double)x0 * x0 + (double)y0 * y0 + (double)z0 * z0);
	const double r = r0 / n, x = x0 / n, y = y0 / n, z = z0 / n;
	R[0][0] = 1 - 2 * (y * y + z * z); R[0][1] = 2 * (x * y - r * z);     R[0][2] = 2 * (x * z + r * y);
	R[1][0] = 2 * (x * y + r * z);     R[1][1] = 1 - 2 * (x * x + z * z); R[1][2] = 2 * (y * z - r * x);
	R[2][0] = 2 * (x * z - r * y);     R[2][1] = 2 * (y * z + r * x);     R[2][2] = 1 - 2 * (x * x + y * y);
}

__global__ void __launch_bounds__(MC_THREADS) mcmc_noise_kernel(long long P, float* __restrict__ xyz, const float* __restrict__ scaling,
	const float* __restrict__ rotation, const float* __restrict__ logits, const float* __restrict__ draws, float noise_lr, float xyz_lr)
{
	const long long stride = (long long)gridDim.x * MC_THREADS;
	for (long long i = (long long)blockIdx.x * MC_THREADS + threadIdx.x; i < P; i += stride)
	{
		const float o = sigmoid_torch(logits[i]);
		// the gate as torch evaluates it in fp32: where exp(-100 ((1 - o) - 0.995)) overflows the gate is 0 and the row keeps its bytes
		if (isinf(exp_ref(__fmul_rn(-100.0f, __fsub_rn(__fsub_rn(1.0f, o), 0.995f))))) continue;
		const double gate = 1.0 / (1.0 + exp(-100.0 * ((1.0 - (double)o) - 0.995)));
		const double k = gate * (double)noise_lr * (double)xyz_lr;
		float q0 = rotation[4 * i], q1 = rotation[4 * i + 1], q2 = rotation[4 * i + 2], q3 = rotation[4 * i + 3];
		normalize_quat(q0, q1, q2, q3);
		double R[3][3];
		rotation_d(q0, q1, q2, q3, R);
		double v[3], w[3];
#pragma unroll
		for (int c = 0; c < 3; c++) v[c] = (double)draws[3 * i + c] * k;
#pragma unroll
		for (int c = 0; c < 3; c++)
		{
			const double s = exp_ref(scaling[3 * i + c]);
			w[c] = (R[0][c] * v[0] + R[1][c] * v[1] + R[2][c] * v[2]) * (s * s);
		}
#pragma unroll
		for (int c = 0; c < 3; c++) xyz[3 * i + c] = (float)((double)xyz[3 * i + c] + (R[c][0] * w[0] + R[c][1] * w[1] + R[c][2] * w[2]));
	}
}

// ------------------------------------------------------------------------------------------------ plan, first phase
struct McmcPlanArgs {
	const float* logits;
	const uint8_t* dead_mask;
	float min_opacity;
	int P, mode;
};

// (weight << MC_DEAD_BITS) | dead of row r.  W = floor(o * 2^32) (exact: o <= 1 and the scale is a power of two); dead rows, and a
// NaN opacity, weigh 0.
__device__ __forceinline__ unsigned long long packed_row(const McmcPlanArgs& a, long long r)
{
	const float o = sigmoid_torch(a.logits[r]);
	const bool dead = a.mode == GSB_MCMC_RELOCATE && (a.dead_mask ? a.dead_mask[r] != 0 : o <= a.min_opacity);
	const unsigned long long w = dead || !(o > 0.0f) ? 0ull : (unsigned long long)__fmul_rn(o, 4294967296.0f);
	return (w << MC_DEAD_BITS) | (dead ? 1ull : 0ull);
}

// exclusive scan of v over the CTA (blockDim.x a multiple of 32, at most 1024); *total = the CTA's sum
__device__ __forceinline__ unsigned long long cta_exclusive(unsigned long long v, unsigned long long* s_warp, unsigned long long* total)
{
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
	unsigned long long incl = v;
#pragma unroll
	for (int o = 1; o < 32; o <<= 1) { const unsigned long long u = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += u; }
	__syncthreads();                                   // s_warp may still be read by a previous call
	if (lane == 31) s_warp[warp] = incl;
	__syncthreads();
	if (warp == 0)
	{
		unsigned long long x = lane < nw ? s_warp[lane] : 0ull;
#pragma unroll
		for (int o = 1; o < 32; o <<= 1) { const unsigned long long u = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += u; }
		if (lane < nw) s_warp[lane] = x;
	}
	__syncthreads();
	*total = s_warp[nw - 1];
	return (warp ? s_warp[warp - 1] : 0ull) + incl - v;
}

__global__ void __launch_bounds__(MC_THREADS) mcmc_reduce_kernel(const McmcPlanArgs a, McmcWorkspace w)
{
	__shared__ unsigned long long s_warp[32];
	const long long row0 = (long long)blockIdx.x * MC_TILE + (long long)threadIdx.x * MC_ITEMS;
	unsigned long long mine = 0;
#pragma unroll
	for (int i = 0; i < MC_ITEMS; i++)
		if (row0 + i < a.P) mine += packed_row(a, row0 + i);
	unsigned long long total;
	cta_exclusive(mine, s_warp, &total);
	if (threadIdx.x == 0) w.tile_sum[blockIdx.x] = total;
}

__global__ void __launch_bounds__(MC_SCAN_THREADS) mcmc_tile_scan_kernel(McmcWorkspace w, long long* __restrict__ counts)
{
	__shared__ unsigned long long s_warp[32];
	unsigned long long run_w = 0, run_d = 0;
	for (uint32_t base = 0; base < w.n_tiles; base += MC_SCAN_THREADS)
	{
		const uint32_t t = base + threadIdx.x;
		const unsigned long long s = t < w.n_tiles ? w.tile_sum[t] : 0ull;
		unsigned long long tw, td;
		const unsigned long long ew = cta_exclusive(s >> MC_DEAD_BITS, s_warp, &tw);
		const unsigned long long ed = cta_exclusive(s & ((1ull << MC_DEAD_BITS) - 1), s_warp, &td);
		if (t < w.n_tiles) { w.tile_w[t] = run_w + ew; w.tile_d[t] = (uint32_t)(run_d + ed); }
		run_w += tw;
		run_d += td;
	}
	if (threadIdx.x == 0)
	{
		w.totals[0] = run_w;
		w.totals[1] = run_d;
		counts[0] = (long long)run_d;
		counts[1] = (long long)run_w;
		counts[2] = 0;
		counts[3] = 0;
	}
}

__global__ void __launch_bounds__(MC_THREADS) mcmc_scan_kernel(const McmcPlanArgs a, McmcWorkspace w)
{
	__shared__ unsigned long long s_warp[32];
	const long long row0 = (long long)blockIdx.x * MC_TILE + (long long)threadIdx.x * MC_ITEMS;
	unsigned long long p[MC_ITEMS], mine = 0;
#pragma unroll
	for (int i = 0; i < MC_ITEMS; i++)
	{
		p[i] = row0 + i < a.P ? packed_row(a, row0 + i) : 0ull;
		mine += p[i];
	}
	unsigned long long total;
	const unsigned long long excl = cta_exclusive(mine, s_warp, &total);
	unsigned long long run_w = w.tile_w[blockIdx.x] + (excl >> MC_DEAD_BITS);
	uint32_t run_d = w.tile_d[blockIdx.x] + (uint32_t)(excl & ((1ull << MC_DEAD_BITS) - 1));
#pragma unroll
	for (int i = 0; i < MC_ITEMS; i++)
	{
		const long long r = row0 + i;
		if (r >= a.P) break;
		run_w += p[i] >> MC_DEAD_BITS;
		w.prefix[r] = run_w;
		if (p[i] & 1ull) w.dead_rows[run_d++] = (int32_t)r;
	}
}

// ------------------------------------------------------------------------------------------------ plan, second phase
// draws used: relocate pairs draw j with the j-th dead row and so uses min(n, dead rows); add uses all n
__device__ __forceinline__ long long draws_used(const McmcWorkspace& w, int mode, long long n)
{
	return mode == GSB_MCMC_RELOCATE ? min(n, (long long)w.totals[1]) : n;
}

__global__ void __launch_bounds__(MC_THREADS) mcmc_sample_kernel(McmcWorkspace w, int P, int mode, long long n,
	const long long* __restrict__ draws)
{
	const long long used = draws_used(w, mode, n);
	const unsigned long long total = w.totals[0];
	const long long stride = (long long)gridDim.x * MC_THREADS;
	for (long long j = (long long)blockIdx.x * MC_THREADS + threadIdx.x; j < used; j += stride)
	{
		// t = floor(d * total / 2^62) from the 128-bit product (d < 2^62, total < 2^62); the source is the first row whose
		// inclusive prefix exceeds t, which exists because t < total
		const unsigned long long d = (unsigned long long)draws[j] & ((1ull << 62) - 1);
		const unsigned long long t = (__umul64hi(d, total) << 2) | ((d * total) >> 62);
		int lo = 0, hi = P - 1;
		while (lo < hi)
		{
			const int mid = (lo + hi) >> 1;
			if (w.prefix[mid] > t) hi = mid; else lo = mid + 1;
		}
		w.source[j] = lo;
		atomicAdd(w.count + lo, 1u);
		atomicMin(w.owner + lo, (uint32_t)j);
	}
}

// paper eq. 9 for one source: o' = 1 - (1 - o)^(1/N), D = sum_{i=1..N} sum_{k<i} C(i-1, k) (-1)^k o'^(k+1) / sqrt(k+1), evaluated
// as sum_{k<N} C(N, k+1) (-1)^k o'^(k+1) / sqrt(k+1) (sum_{i>k}^{N} C(i-1, k) = C(N, k+1)), every operation rounded on its own in
// double; s' = (o / D) s.  The binomials are exact integers in double (C(50, 25) < 2^53).
__device__ __forceinline__ float4 relocated(float o, float s0, float s1, float s2, int N)
{
	const double od = o;
	const double op = __dsub_rn(1.0, pow(__dsub_rn(1.0, od), __ddiv_rn(1.0, (double)N)));
	double D = 0.0, pw = 1.0, binom = N;                           // binom = C(N, k + 1)
	for (int k = 0; k < N; k++)
	{
		pw = __dmul_rn(pw, op);
		const double term = __ddiv_rn(__dmul_rn(binom, pw), __dsqrt_rn((double)(k + 1)));
		D = (k & 1) ? __dsub_rn(D, term) : __dadd_rn(D, term);
		binom = __ddiv_rn(__dmul_rn(binom, (double)(N - k - 1)), (double)(k + 2));
	}
	const double coeff = __ddiv_rn(od, D);
	const float oc = fminf(fmaxf((float)op, 0.005f), 1.0f - 0x1p-23f);   // torch.clamp(min=0.005, max=1 - eps)
	return make_float4(oc, (float)__dmul_rn(coeff, (double)s0), (float)__dmul_rn(coeff, (double)s1), (float)__dmul_rn(coeff, (double)s2));
}

__global__ void __launch_bounds__(MC_THREADS) mcmc_values_kernel(McmcWorkspace w, int mode, long long n, const float* __restrict__ logits,
	const float* __restrict__ scaling)
{
	const long long used = draws_used(w, mode, n);
	const long long stride = (long long)gridDim.x * MC_THREADS;
	for (long long j = (long long)blockIdx.x * MC_THREADS + threadIdx.x; j < used; j += stride)
	{
		const int r = w.source[j];
		if (w.owner[r] != (uint32_t)j) continue;
		const int N = (int)min(w.count[r] + 1u, (uint32_t)MC_N_MAX);
		w.values[r] = relocated(sigmoid_torch(logits[r]), exp_ref(scaling[3 * (long long)r]), exp_ref(scaling[3 * (long long)r + 1]),
			exp_ref(scaling[3 * (long long)r + 2]), N);
	}
}

// ------------------------------------------------------------------------------------------------ emit
struct McmcTable {
	GsbDensifyTensor t[GSB_DENSIFY_MAX_TENSORS];
	double inv_width[GSB_DENSIFY_MAX_TENSORS];
};

// the stored value of a relocated row: inverse_sigmoid(o') = log(o' / (1 - o')) and log(s'), in fp32 as torch evaluates them
__device__ __forceinline__ uint32_t stored(int kind, const float4& v, int c)
{
	if (kind == GSB_MCMC_OPACITY) return __float_as_uint(logf(__fdiv_rn(v.x, __fsub_rn(1.0f, v.x))));
	return __float_as_uint(logf(c == 0 ? v.y : c == 1 ? v.z : v.w));
}
__device__ __forceinline__ bool relocates(int kind) { return kind == GSB_MCMC_OPACITY || kind == GSB_DENSIFY_SCALING; }

// relocate, in place: element (j, c) of the n_used dead rows.  Dead row j takes its source's row (the relocated value in an opacity
// / scaling entry); the source's owner draw writes the source's relocated value and zeroes its moments.
__global__ void __launch_bounds__(MC_THREADS) mcmc_emit_relocate_kernel(const __grid_constant__ McmcTable tab, McmcWorkspace w, long long n)
{
	const GsbDensifyTensor& k = tab.t[blockIdx.y];
	const int wd = k.row_width;
	const long long total = draws_used(w, GSB_MCMC_RELOCATE, n) * wd, stride = (long long)gridDim.x * MC_THREADS;
	uint32_t* __restrict__ p = static_cast<uint32_t*>(k.dst);
	for (long long e = (long long)blockIdx.x * MC_THREADS + threadIdx.x; e < total; e += stride)
	{
		long long j;
		int c;
		row_col(e, wd, tab.inv_width[blockIdx.y], j, c);
		const long long r = w.source[j], d = w.dead_rows[j];
		if (relocates(k.kind))
		{
			const uint32_t v = stored(k.kind, w.values[r], c);
			p[d * wd + c] = v;
			if (w.owner[r] == (uint32_t)j) p[r * wd + c] = v;
		}
		else
			p[d * wd + c] = p[r * wd + c];
		if (k.exp_avg_dst && w.owner[r] == (uint32_t)j) { k.exp_avg_dst[r * wd + c] = 0.0f; k.exp_avg_sq_dst[r * wd + c] = 0.0f; }
	}
}

// add: every element of the [P + n, row_width] destination.  Rows < P copy the source tensor (a sampled row's opacity / scaling
// takes its relocated value and its moments are zeroed); row P + j copies draw j's source row (relocated opacity / scaling) with
// zero moments, or is zero in a GSB_MCMC_FRESH entry.
__global__ void __launch_bounds__(MC_THREADS) mcmc_emit_add_kernel(const __grid_constant__ McmcTable tab, McmcWorkspace w, long long P,
	long long n)
{
	const GsbDensifyTensor& k = tab.t[blockIdx.y];
	const int wd = k.row_width;
	const long long total = (P + n) * wd, stride = (long long)gridDim.x * MC_THREADS;
	const uint32_t* __restrict__ src = static_cast<const uint32_t*>(k.src);
	uint32_t* __restrict__ dst = static_cast<uint32_t*>(k.dst);
	for (long long e = (long long)blockIdx.x * MC_THREADS + threadIdx.x; e < total; e += stride)
	{
		long long r;
		int c;
		row_col(e, wd, tab.inv_width[blockIdx.y], r, c);
		if (r < P)
		{
			const bool sampled = w.count[r] != 0;
			dst[e] = sampled && relocates(k.kind) ? stored(k.kind, w.values[r], c) : src[e];
			if (k.exp_avg_dst)
			{
				k.exp_avg_dst[e] = sampled ? 0.0f : k.exp_avg_src[e];
				k.exp_avg_sq_dst[e] = sampled ? 0.0f : k.exp_avg_sq_src[e];
			}
		}
		else
		{
			const long long s = w.source[r - P];
			dst[e] = k.kind == GSB_MCMC_FRESH ? 0u : relocates(k.kind) ? stored(k.kind, w.values[s], c) : src[s * wd + c];
			if (k.exp_avg_dst) { k.exp_avg_dst[e] = 0.0f; k.exp_avg_sq_dst[e] = 0.0f; }
		}
	}
}

static int mcmc_grid(long long work)
{
	const long long want = (work + MC_THREADS - 1) / MC_THREADS, cap = (long long)GSB_NUM_SMS * 8;
	return (int)(want < cap ? (want > 0 ? want : 1) : cap);
}

} // namespace gsb

using namespace gsb;

extern "C" int gsb_mcmc_noise(int32_t P, float* xyz, const float* scaling, const float* rotation, const float* opacity_logits,
	const float* draws, float noise_lr, float xyz_lr, void* stream)
{
	if (P < 0 || P >= (1 << 30)) { set_error("mcmc_noise: P = %d is outside 0..2^30 - 1", P); return GSB_EINVAL; }
	if (!isfinite(noise_lr) || !isfinite(xyz_lr)) { set_error("mcmc_noise: noise_lr and xyz_lr must be finite"); return GSB_EINVAL; }
	if (P == 0) return GSB_OK;
	if (!xyz || !scaling || !rotation || !opacity_logits || !draws)
	{ set_error("mcmc_noise: NULL xyz / scaling / rotation / opacity_logits / draws"); return GSB_EINVAL; }
	const cudaStream_t st = (cudaStream_t)stream;
	ProfScope prof(K_TOOLS, st);
	mcmc_noise_kernel<<<mcmc_grid(P), MC_THREADS, 0, st>>>(P, xyz, scaling, rotation, opacity_logits, draws, noise_lr, xyz_lr);
	GSB_LAUNCHED();
	GSB_CUDA_OK(cudaGetLastError());
	return GSB_OK;
}

extern "C" size_t gsb_mcmc_workspace_bytes(int32_t P) { return mcmc_carve(nullptr, P).bytes; }

extern "C" int gsb_mcmc_plan(int32_t P, int32_t mode, const float* opacity_logits, const float* scaling, const uint8_t* dead_mask,
	float min_opacity, int64_t n, const int64_t* draws, void* workspace, int64_t* counts, void* stream)
{
	if (P < 0 || P >= (1 << 30)) { set_error("mcmc_plan: P = %d is outside 0..2^30 - 1", P); return GSB_EINVAL; }
	if (mode != GSB_MCMC_RELOCATE && mode != GSB_MCMC_ADD) { set_error("mcmc_plan: unknown mode %d", mode); return GSB_EINVAL; }
	if (dead_mask && mode != GSB_MCMC_RELOCATE) { set_error("mcmc_plan: dead_mask given with GSB_MCMC_ADD"); return GSB_EINVAL; }
	if (!workspace) { set_error("mcmc_plan: NULL workspace"); return GSB_EINVAL; }
	if (draws ? (n <= 0 || n > P) : n != 0)
	{ set_error("mcmc_plan: n = %lld: with draws it must be 1..P (= %d), without draws 0", (long long)n, P); return GSB_EINVAL; }
	if (!draws && !counts) { set_error("mcmc_plan: NULL counts"); return GSB_EINVAL; }
	if (P > 0 && !opacity_logits) { set_error("mcmc_plan: NULL opacity_logits"); return GSB_EINVAL; }
	if (draws && !scaling) { set_error("mcmc_plan: NULL scaling"); return GSB_EINVAL; }
	const cudaStream_t st = (cudaStream_t)stream;
	ProfScope prof(K_TOOLS, st);
	if (P == 0)
	{
		GSB_CUDA_OK(cudaMemsetAsync(counts, 0, sizeof(int64_t) * GSB_MCMC_COUNTS, st));
		return GSB_OK;
	}
	const McmcWorkspace w = mcmc_carve(static_cast<char*>(workspace), P);
	McmcPlanArgs a;
	a.logits = opacity_logits; a.dead_mask = dead_mask; a.min_opacity = min_opacity; a.P = P; a.mode = mode;
	if (!draws)
	{
		mcmc_reduce_kernel<<<w.n_tiles, MC_THREADS, 0, st>>>(a, w);
		GSB_LAUNCHED();
		mcmc_tile_scan_kernel<<<1, MC_SCAN_THREADS, 0, st>>>(w, reinterpret_cast<long long*>(counts));
		GSB_LAUNCHED();
		mcmc_scan_kernel<<<w.n_tiles, MC_THREADS, 0, st>>>(a, w);
		GSB_LAUNCHED();
		GSB_CUDA_OK(cudaGetLastError());
		return GSB_OK;
	}
	GSB_CUDA_OK(cudaMemsetAsync(w.count, 0, sizeof(uint32_t) * (size_t)P, st));
	GSB_CUDA_OK(cudaMemsetAsync(w.owner, 0xff, sizeof(uint32_t) * (size_t)P, st));
	mcmc_sample_kernel<<<mcmc_grid(n), MC_THREADS, 0, st>>>(w, P, mode, n, reinterpret_cast<const long long*>(draws));
	GSB_LAUNCHED();
	mcmc_values_kernel<<<mcmc_grid(n), MC_THREADS, 0, st>>>(w, mode, n, opacity_logits, scaling);
	GSB_LAUNCHED();
	GSB_CUDA_OK(cudaGetLastError());
	return GSB_OK;
}

extern "C" int gsb_mcmc_emit(const GsbDensifyTensor* tensors, int32_t n_tensors, int32_t P, int32_t mode, int64_t n, const void* workspace,
	void* stream)
{
	if (n_tensors < 0 || n_tensors > GSB_DENSIFY_MAX_TENSORS)
	{ set_error("mcmc_emit: n_tensors = %d is outside 0..%d", n_tensors, GSB_DENSIFY_MAX_TENSORS); return GSB_EINVAL; }
	if (n_tensors > 0 && !tensors) { set_error("mcmc_emit: tensor table is NULL"); return GSB_EINVAL; }
	if (P < 0 || P >= (1 << 30)) { set_error("mcmc_emit: P = %d is outside 0..2^30 - 1", P); return GSB_EINVAL; }
	if (mode != GSB_MCMC_RELOCATE && mode != GSB_MCMC_ADD) { set_error("mcmc_emit: unknown mode %d", mode); return GSB_EINVAL; }
	if (n < 0 || n > P) { set_error("mcmc_emit: n = %lld is outside 0..P (= %d)", (long long)n, P); return GSB_EINVAL; }
	if (!workspace) { set_error("mcmc_emit: NULL workspace"); return GSB_EINVAL; }
	McmcTable tab{};
	int max_w = 1;
	for (int i = 0; i < n_tensors; i++)
	{
		const GsbDensifyTensor& k = tensors[i];
		if (k.row_width <= 0) { set_error("mcmc_emit: tensor %d: row_width %d <= 0", i, k.row_width); return GSB_EINVAL; }
		if (k.kind != GSB_DENSIFY_COPY && k.kind != GSB_DENSIFY_SCALING && k.kind != GSB_MCMC_OPACITY && k.kind != GSB_MCMC_FRESH)
		{ set_error("mcmc_emit: tensor %d: kind %d is not COPY, SCALING, MCMC_OPACITY or MCMC_FRESH", i, k.kind); return GSB_EINVAL; }
		if ((k.kind == GSB_DENSIFY_SCALING && k.row_width != 3) || (k.kind == GSB_MCMC_OPACITY && k.row_width != 1))
		{ set_error("mcmc_emit: tensor %d: a scaling entry needs row_width 3, an opacity entry 1; got %d", i, k.row_width); return GSB_EINVAL; }
		if (k.kind == GSB_MCMC_FRESH && (mode != GSB_MCMC_ADD || k.exp_avg_src))
		{ set_error("mcmc_emit: tensor %d: an MCMC_FRESH entry belongs to GSB_MCMC_ADD and has no moments", i); return GSB_EINVAL; }
		if (k.grad_src || k.grad_dst) { set_error("mcmc_emit: tensor %d: grad pointers must be NULL", i); return GSB_EINVAL; }
		if (!k.exp_avg_src != !k.exp_avg_dst || !k.exp_avg_src != !k.exp_avg_sq_src || !k.exp_avg_src != !k.exp_avg_sq_dst)
		{ set_error("mcmc_emit: tensor %d: exp_avg / exp_avg_sq are half given", i); return GSB_EINVAL; }
		if (P > 0 && (!k.src || !k.dst)) { set_error("mcmc_emit: tensor %d: NULL src / dst", i); return GSB_EINVAL; }
		if (mode == GSB_MCMC_RELOCATE && (k.src != k.dst || k.exp_avg_src != k.exp_avg_dst || k.exp_avg_sq_src != k.exp_avg_sq_dst))
		{ set_error("mcmc_emit: tensor %d: GSB_MCMC_RELOCATE works in place (dst == src for the param and both moments)", i); return GSB_EINVAL; }
		const uintptr_t any = reinterpret_cast<uintptr_t>(k.src) | reinterpret_cast<uintptr_t>(k.dst) |
			reinterpret_cast<uintptr_t>(k.exp_avg_src) | reinterpret_cast<uintptr_t>(k.exp_avg_dst) |
			reinterpret_cast<uintptr_t>(k.exp_avg_sq_src) | reinterpret_cast<uintptr_t>(k.exp_avg_sq_dst);
		if (any & 3u) { set_error("mcmc_emit: tensor %d: a pointer is not 4-byte aligned", i); return GSB_EINVAL; }
		tab.t[i] = k;
		tab.inv_width[i] = 1.0 / k.row_width;
		max_w = k.row_width > max_w ? k.row_width : max_w;
	}
	const long long rows = mode == GSB_MCMC_ADD ? (long long)P + n : n;
	if (n_tensors == 0 || rows == 0) return GSB_OK;
	const McmcWorkspace w = mcmc_carve(static_cast<char*>(const_cast<void*>(workspace)), P);
	const cudaStream_t st = (cudaStream_t)stream;
	ProfScope prof(K_TOOLS, st);
	const dim3 grid((unsigned)mcmc_grid(rows * max_w), (unsigned)n_tensors);
	if (mode == GSB_MCMC_ADD) mcmc_emit_add_kernel<<<grid, MC_THREADS, 0, st>>>(tab, w, P, n);
	else mcmc_emit_relocate_kernel<<<grid, MC_THREADS, 0, st>>>(tab, w, n);
	GSB_LAUNCHED();
	GSB_CUDA_OK(cudaGetLastError());
	return GSB_OK;
}
