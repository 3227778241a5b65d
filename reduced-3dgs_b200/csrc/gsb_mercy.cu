// gsb_mercy.cu — the statistics and the prune mask of the reference's GaussianModel.mercy_points (gaussian_model.py:524-551;
// gs_b200.densify.mercy_points, DESIGN.md §5k).
//
// The reference reads mean + lambda * std back to the host, boolean-indexes the opacities twice, sorts for torch.median /
// torch.quantile (the latter refuses more than 2^24 rows) and synchronises on every masked assignment.  Here, all on the stream:
//   mercy_sums_kernel       sum c and sum c^2 of the counts, exactly, in 64-bit integers;
//   mercy_threshold_kernel  one thread: mean and unbiased variance in fp64 from those sums, each rounded to fp32, then the
//                           reference's fp32 ops for mean + lambda * std and Python's max(., mercy_minimum);
//   mercy_hist_kernel       three radix-select passes (11 + 11 + 10 bits) over sigmoid(opacity), one histogram per wanted rank:
//   mercy_select_kernel       the lower median of the redundant rows (torch.median) and the two ranks torch.quantile interpolates;
//   mercy_mask_kernel       the prune mask and its counts; for 'redundancy_random' the redundant rows' ranks in index order
//                           (decoupled look-back) pick their draw.
// Every result is an integer count or an order statistic, so the outputs are the same bytes on every run.  The CTA scan, the grid
// size and the row range are gsb_common.cuh's, shared with gsb_densify.cu and gsb_mcmc.cu.
#include "gsb_common.cuh"

namespace gsb {

#define MERCY_THREADS 256
#define MERCY_ITEMS 4
#define MERCY_TILE (MERCY_THREADS * MERCY_ITEMS)
#define MERCY_BINS 2048
#define MERCY_TARGETS 3        // the median of the redundant rows, the quantile's lower and upper rank over all rows
#define MERCY_PASSES 3

struct MercyState {
	unsigned long long sum, sumsq;   // sum of the counts (two's complement) and of their squares
	float thr;                       // fp32(max(mean + lambda * std, mercy_minimum)): a row is redundant if (float)count > thr
	float median;                    // median opacity of the redundant rows (NaN: none, or one is NaN)
	float opacity_thr;               // the opacity threshold of 'opacity' / 'redundancy_opacity_opacity'
	float weight;                    // the quantile's interpolation weight
	long long rank[MERCY_TARGETS];   // remaining rank inside the current prefix; -1 = nothing to select
	uint32_t prefix[MERCY_TARGETS];  // the key bits selected so far
	uint32_t nan_any[MERCY_TARGETS];
};

struct MercyWorkspace {
	MercyState* state;
	uint32_t* hist;                  // [MERCY_PASSES][MERCY_TARGETS][MERCY_BINS]
	uint32_t* lookback;              // [n_tiles]
	uint32_t* ticket;
	uint32_t n_tiles;
	size_t bytes;
};
static MercyWorkspace mercy_carve(char* base, int P)
{
	Carver c(base);
	MercyWorkspace w;
	const size_t n = P > 0 ? (size_t)P : 1;
	w.n_tiles = (uint32_t)((n + MERCY_TILE - 1) / MERCY_TILE);
	w.state = c.take<MercyState>(1);
	w.hist = c.take<uint32_t>((size_t)MERCY_PASSES * MERCY_TARGETS * MERCY_BINS);
	w.lookback = c.take<uint32_t>(w.n_tiles);
	w.ticket = c.take<uint32_t>(1);
	w.bytes = c.off + 256;
	return w;
}

struct MercyArgs {
	const int32_t* counts;
	const float* logits;
	const float* draws;
	long long n_draws;
	int P, type;
	bool want_median, want_quantile;
};

// float_key with NaN above everything (torch sorts NaN last); key_float decodes it
__device__ __forceinline__ uint32_t float_key_nan_last(float f) { return isnan(f) ? 0xffffffffu : float_key(f); }
__device__ __forceinline__ bool is_redundant(int c, float thr) { return (float)c > thr; }
// torch.minimum: NaN if either is NaN
__device__ __forceinline__ float min_torch(float a, float b) { return isnan(a) || isnan(b) ? __int_as_float(0x7fc00000) : fminf(a, b); }
// torch's CUDA lerp (ATen/native/Lerp.h), contracted to FMA by nvcc (tools/probe_torch_mercy.py)
__device__ __forceinline__ float lerp_torch(float a, float b, float w)
{
	const float d = __fsub_rn(b, a);
	return fabsf(w) < 0.5f ? __fmaf_rn(w, d, a) : __fmaf_rn(-d, __fsub_rn(1.0f, w), b);
}
__device__ __forceinline__ int pass_shift(int p) { return p == 0 ? 21 : (p == 1 ? 10 : 0); }
__device__ __forceinline__ int pass_width(int p) { return p == 2 ? 10 : 11; }

__global__ void __launch_bounds__(MERCY_THREADS) mercy_sums_kernel(int P, const int32_t* __restrict__ counts, MercyState* st)
{
	__shared__ unsigned long long s[2][MERCY_THREADS / 32];
	unsigned long long a = 0, b = 0;
	for (int i = blockIdx.x * MERCY_THREADS + threadIdx.x; i < P; i += gridDim.x * MERCY_THREADS)
	{
		const long long c = counts[i];
		a += (unsigned long long)c;
		b += (unsigned long long)(c * c);
	}
#pragma unroll
	for (int o = 16; o > 0; o >>= 1) { a += __shfl_xor_sync(0xffffffffu, a, o); b += __shfl_xor_sync(0xffffffffu, b, o); }
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	if (lane == 0) { s[0][warp] = a; s[1][warp] = b; }
	__syncthreads();
	if (threadIdx.x == 0)
	{
		for (int k = 1; k < MERCY_THREADS / 32; k++) { a += s[0][k]; b += s[1][k]; }
		atomicAdd(&st->sum, a);
		atomicAdd(&st->sumsq, b);
	}
}

// mean = S / P and var = (P * Q - S^2) / (P (P - 1)) from the exact integer sums (the numerator in 128 bits), each formed in fp64
// and rounded to fp32; then torch's fp32 ops: std = sqrt(var), mean + fp32(lambda) * std.  P = 1 gives var = NaN (torch's
// unbiased variance of one element), P = 0 a NaN mean.  Python's max(x, m) returns x unless m > x, so NaN stays NaN.
__global__ void mercy_threshold_kernel(int P, int type, float lambda, double mercy_minimum, float q, MercyState* st, float* thresholds)
{
	const long long S = (long long)st->sum;
	const unsigned long long Q = st->sumsq;
	const float mean = (float)((double)S / (double)P);
	float var = __int_as_float(0x7fc00000);
	if (P > 1)
	{
		const __int128 num = (__int128)P * (__int128)Q - (__int128)S * (__int128)S;
		var = (float)((double)num / ((double)P * (double)(P - 1)));
	}
	const float red = __fadd_rn(mean, __fmul_rn(lambda, __fsqrt_rn(var)));
	const double x = (double)red;
	st->thr = (float)(mercy_minimum > x ? mercy_minimum : x);
	st->median = __int_as_float(0x7fc00000);
	st->opacity_thr = (type == GSB_MERCY_OPACITY || type == GSB_MERCY_REDUNDANCY_OPACITY_OPACITY) ? __int_as_float(0x7fc00000) : 0.0f;
	// torch.quantile: rank = fp32(q) * fp32(P - 1); below = (int64) rank; weight = rank - below; above = ceil(rank)
	const float r = __fmul_rn(q, (float)(P > 0 ? P - 1 : 0));
	long long lo = (long long)r, hi = (long long)ceilf(r);
	lo = lo < P - 1 ? lo : P - 1;
	hi = hi < P - 1 ? hi : P - 1;
	st->weight = __fsub_rn(r, (float)lo);
	st->rank[0] = -1;
	st->rank[1] = P > 0 ? lo : -1;
	st->rank[2] = P > 0 ? hi : -1;
	for (int t = 0; t < MERCY_TARGETS; t++) { st->prefix[t] = 0; st->nan_any[t] = 0; }
	thresholds[0] = red;
	thresholds[1] = st->opacity_thr;
}

// One pass of the radix select: per target, the histogram of the current digit over the rows whose higher key bits equal the
// target's prefix.  Target 0 counts the redundant rows only; targets 1 and 2 count every row.
__global__ void __launch_bounds__(MERCY_THREADS) mercy_hist_kernel(const MercyArgs a, const MercyState* __restrict__ st,
	uint32_t* __restrict__ hist, int pass)
{
	__shared__ uint32_t s_h[MERCY_TARGETS][MERCY_BINS];
	for (int i = threadIdx.x; i < MERCY_TARGETS * MERCY_BINS; i += MERCY_THREADS) (&s_h[0][0])[i] = 0;
	__syncthreads();
	const int shift = pass_shift(pass), width = pass_width(pass);
	const uint32_t dmask = (1u << width) - 1u;
	const float thr = st->thr;
	bool on[MERCY_TARGETS];
	uint32_t pre[MERCY_TARGETS];
#pragma unroll
	for (int t = 0; t < MERCY_TARGETS; t++)
	{
		on[t] = (t == 0 ? a.want_median : a.want_quantile) && (pass == 0 || st->rank[t] >= 0);
		pre[t] = st->prefix[t];
	}
	for (int i = blockIdx.x * MERCY_THREADS + threadIdx.x; i < a.P; i += gridDim.x * MERCY_THREADS)
	{
		const uint32_t key = float_key_nan_last(sigmoid_torch(a.logits[i]));
		const uint32_t d = (key >> shift) & dmask;
		const uint32_t high = pass == 0 ? 0u : key >> (shift + width);
		if (on[0] && high == pre[0] && is_redundant(a.counts[i], thr)) atomicAdd(&s_h[0][d], 1u);
		if (on[1] && high == pre[1]) atomicAdd(&s_h[1][d], 1u);
		if (on[2] && high == pre[2]) atomicAdd(&s_h[2][d], 1u);
	}
	__syncthreads();
	for (int i = threadIdx.x; i < MERCY_TARGETS * MERCY_BINS; i += MERCY_THREADS)
	{
		const uint32_t v = (&s_h[0][0])[i];
		if (v) atomicAdd(hist + i, v);
	}
}

// One CTA: per target, find the bin that holds its remaining rank, append the bin to the prefix and subtract the rows below.
// After pass 0 the redundant total fixes the median's rank, floor((n - 1) / 2); after the last pass the prefixes are the keys.
__global__ void __launch_bounds__(MERCY_THREADS) mercy_select_kernel(const MercyArgs a, MercyState* st, const uint32_t* __restrict__ hist,
	int pass, float* thresholds)
{
	constexpr int PER = MERCY_BINS / MERCY_THREADS;
	__shared__ unsigned long long s_warp[MERCY_THREADS / 32];
	const int tid = threadIdx.x;
	const int width = pass_width(pass), nbins = 1 << width;
	for (int t = 0; t < MERCY_TARGETS; t++)
	{
		if (!(t == 0 ? a.want_median : a.want_quantile)) continue;
		const uint32_t* h = hist + (size_t)t * MERCY_BINS;
		unsigned long long mine = 0;
		for (int k = 0; k < PER; k++) { const int b = tid * PER + k; mine += b < nbins ? h[b] : 0u; }
		unsigned long long total;
		const unsigned long long before = cta_exclusive<MERCY_THREADS>(mine, s_warp, &total);
		if (pass == 0)
		{
			if (tid == 0)
			{
				st->nan_any[t] = h[MERCY_BINS - 1] > 0;      // bin 0x7ff of the top 11 bits holds only NaN keys
				if (t == 0) st->rank[0] = total > 0 ? (long long)((total - 1) / 2) : -1;
			}
			__syncthreads();
		}
		const long long rank = st->rank[t];
		__syncthreads();
		if (rank >= 0 && (long long)before <= rank && rank < (long long)(before + mine))
		{
			unsigned long long c = before;
			for (int k = 0; k < PER; k++)
			{
				const int b = tid * PER + k;
				const uint32_t v = b < nbins ? h[b] : 0u;
				if ((long long)(c + v) > rank)
				{
					st->prefix[t] = (st->prefix[t] << width) | (uint32_t)b;
					st->rank[t] = rank - (long long)c;
					break;
				}
				c += v;
			}
		}
		__syncthreads();
	}
	if (pass == MERCY_PASSES - 1 && tid == 0)
	{
		const float nan = __int_as_float(0x7fc00000);
		if (a.want_median) st->median = st->rank[0] >= 0 && !st->nan_any[0] ? key_float(st->prefix[0]) : nan;
		if (a.want_quantile)
		{
			float v = nan;
			if (st->rank[1] >= 0 && !st->nan_any[1]) v = lerp_torch(key_float(st->prefix[1]), key_float(st->prefix[2]), st->weight);
			st->opacity_thr = a.type == GSB_MERCY_REDUNDANCY_OPACITY_OPACITY ? min_torch(v, 0.05f) : v;
			thresholds[1] = st->opacity_thr;
		}
	}
}

// The prune mask: one tile of MERCY_TILE rows per CTA, in ticket order.  With draws, a redundant row's draw is the one at its
// rank among the redundant rows.  counts_out[0] += redundant rows, counts_out[1] += pruned rows.  mask == NULL counts only.
__global__ void __launch_bounds__(MERCY_THREADS) mercy_mask_kernel(const MercyArgs a, const MercyState* __restrict__ st,
	uint32_t* __restrict__ lookback, uint32_t* __restrict__ ticket, uint8_t* __restrict__ mask, long long* __restrict__ counts_out)
{
	__shared__ uint32_t s_tile, s_excl;
	__shared__ uint32_t s_warp[MERCY_THREADS / 32];
	const int tid = threadIdx.x;
	if (tid == 0) s_tile = atomicAdd(ticket, 1u);
	__syncthreads();
	const uint32_t tile = s_tile;
	const long long row0 = (long long)tile * MERCY_TILE + (long long)tid * MERCY_ITEMS;
	const float thr = st->thr, med = st->median, othr = st->opacity_thr;
	bool red[MERCY_ITEMS];
	uint32_t n_red = 0;
#pragma unroll
	for (int i = 0; i < MERCY_ITEMS; i++)
	{
		red[i] = row0 + i < a.P && is_redundant(a.counts[row0 + i], thr);
		n_red += red[i] ? 1u : 0u;
	}
	// the redundant rows' ranks (every CTA takes part so that the look-back chain is complete)
	uint32_t cta_total;
	uint32_t run = cta_exclusive<MERCY_THREADS>(n_red, s_warp, &cta_total);
	if (a.draws && tid == 0) s_excl = lookback_exclusive(lookback, tile, 1, 0, cta_total);
	__syncthreads();
	if (a.draws) run += s_excl;
	uint32_t n_pruned = 0;
	if (mask)
	{
#pragma unroll
		for (int i = 0; i < MERCY_ITEMS; i++)
		{
			const long long r = row0 + i;
			if (r >= a.P) break;
			bool m;
			if (a.type == GSB_MERCY_REDUNDANCY_RANDOM) m = red[i] && (long long)run < a.n_draws && a.draws[run] < 0.5f;
			else if (a.type == GSB_MERCY_REDUNDANCY) m = red[i];
			else
			{
				const float op = sigmoid_torch(a.logits[r]);
				if (a.type == GSB_MERCY_REDUNDANCY_OPACITY) m = red[i] && op < med;
				else if (a.type == GSB_MERCY_OPACITY) m = op < othr;
				else m = (red[i] && op < med) || op < othr;
			}
			mask[r] = m ? 1 : 0;
			n_pruned += m ? 1u : 0u;
			run += red[i] ? 1u : 0u;
		}
	}
	uint32_t np;
	cta_exclusive<MERCY_THREADS>(n_pruned, s_warp, &np);
	if (tid == 0)
	{
		if (cta_total) atomicAdd(reinterpret_cast<unsigned long long*>(counts_out), (unsigned long long)cta_total);
		if (np) atomicAdd(reinterpret_cast<unsigned long long*>(counts_out + 1), (unsigned long long)np);
	}
}

} // namespace gsb

using namespace gsb;

extern "C" size_t gsb_mercy_workspace_bytes(int32_t P) { return mercy_carve(nullptr, P).bytes; }

extern "C" int gsb_mercy_plan(int32_t P, const int32_t* counts, const float* opacity_logits, int32_t type, float lambda_mercy,
	double mercy_minimum, float quantile_q, const float* draws, int64_t n_draws, void* workspace, uint8_t* mask, float* thresholds,
	int64_t* counts_out, void* stream)
{
	if (!rows_ok("mercy_plan", P)) return GSB_EINVAL;
	if (type < GSB_MERCY_REDUNDANCY_OPACITY || type > GSB_MERCY_REDUNDANCY) { set_error("mercy_plan: unknown type %d", type); return GSB_EINVAL; }
	if (!workspace || !thresholds || !counts_out) { set_error("mercy_plan: NULL workspace / thresholds / counts_out"); return GSB_EINVAL; }
	if (draws && type != GSB_MERCY_REDUNDANCY_RANDOM) { set_error("mercy_plan: draws are only read by the random type"); return GSB_EINVAL; }
	if (draws && n_draws < 0) { set_error("mercy_plan: draws given without their count"); return GSB_EINVAL; }
	const bool want_median = type == GSB_MERCY_REDUNDANCY_OPACITY || type == GSB_MERCY_REDUNDANCY_OPACITY_OPACITY;
	const bool want_quantile = type == GSB_MERCY_OPACITY || type == GSB_MERCY_REDUNDANCY_OPACITY_OPACITY;
	if (P > 0)
	{
		if (!counts || !mask) { set_error("mercy_plan: NULL counts / mask"); return GSB_EINVAL; }
		if ((want_median || want_quantile) && !opacity_logits) { set_error("mercy_plan: NULL opacity_logits"); return GSB_EINVAL; }
	}
	const cudaStream_t st = (cudaStream_t)stream;
	ProfScope prof(K_TOOLS, st);
	const MercyWorkspace w = mercy_carve(static_cast<char*>(workspace), P);
	GSB_CUDA_OK(cudaMemsetAsync(workspace, 0, w.bytes, st));
	GSB_CUDA_OK(cudaMemsetAsync(counts_out, 0, 2 * sizeof(int64_t), st));
	MercyArgs a;
	a.counts = counts; a.logits = opacity_logits; a.draws = draws; a.n_draws = n_draws; a.P = P; a.type = type;
	a.want_median = want_median; a.want_quantile = want_quantile;
	const int grid = grid_stride_ctas(P, MERCY_THREADS, 2);
	if (P > 0)
	{
		mercy_sums_kernel<<<grid, MERCY_THREADS, 0, st>>>(P, counts, w.state);
		GSB_LAUNCHED();
	}
	mercy_threshold_kernel<<<1, 1, 0, st>>>(P, type, lambda_mercy, mercy_minimum, quantile_q, w.state, thresholds);
	GSB_LAUNCHED();
	if (P == 0) { GSB_CUDA_OK(cudaGetLastError()); return GSB_OK; }
	if (want_median || want_quantile)
		for (int p = 0; p < MERCY_PASSES; p++)
		{
			uint32_t* h = w.hist + (size_t)p * MERCY_TARGETS * MERCY_BINS;
			mercy_hist_kernel<<<grid, MERCY_THREADS, 0, st>>>(a, w.state, h, p);
			GSB_LAUNCHED();
			mercy_select_kernel<<<1, MERCY_THREADS, 0, st>>>(a, w.state, h, p, thresholds);
			GSB_LAUNCHED();
		}
	const bool count_only = type == GSB_MERCY_REDUNDANCY_RANDOM && !draws;
	mercy_mask_kernel<<<w.n_tiles, MERCY_THREADS, 0, st>>>(a, w.state, w.lookback, w.ticket, count_only ? nullptr : mask, reinterpret_cast<long long*>(counts_out));
	GSB_LAUNCHED();
	GSB_CUDA_OK(cudaGetLastError());
	return GSB_OK;
}
