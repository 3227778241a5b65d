// gsb_kmeans.cu — 1-D k-means for the codebook quantisation (SURVEY.md §8(f) row 4).
//
// Replaces Reduced3DGS::kmeans (reference reduced_3dgs.cu:289-338) with updateIdsCUDA / updateCentersCUDA
// (reduced_3dgs/kmeans.cu:13-107).  The reference does, per Lloyd iteration, an N x K brute-force distance scan, a
// serial 256-value loop by one thread per block with 2K global atomics per block, five ATen ops and a blocking .item().
//
// Here the values are sorted ONCE (hand-written 8-bit onesweep radix sort on the order-preserving integer image of the
// floats).  An iteration then is
//   * assign: binary search of every value in the sorted centres + an exact tie resolution that reproduces the reference's
//     rule "smallest sqrt((c - v)^2), first index wins" (kmeans.cu:93-104) bit for bit;
//   * accumulate: neighbouring sorted values share their cluster, so each thread run-length-sums its 16 consecutive
//     values and a warp whose lanes agree on the cluster issues ONE pair of reductions;
//   * update + convergence test on the device: later iterations see the `done` flag and exit immediately, the host only
//     looks at the flag every few iterations (same stopping rule as the reference, without a sync per iteration).
// Cluster ids / sizes are exact; centre values differ from the reference in float summation order only (the reference's own
// order is arbitrary: atomics).
#include "gsb_common.cuh"

namespace gsb {

#define KM_MAX_K 1024
#define KM_TILE 4096
#define KM_ITEMS 16
#define KM_CHUNK 16

struct KmState {
	int done;            // converged (or max_iterations reached)
	int iterations;      // Lloyd iterations executed
	float shift;         // last centre shift
	int pad;
};

struct KmSortPlan {
	uint32_t digit_base[4][256];
	uint32_t skip[4];
	uint32_t src[4];
	uint32_t final_buf;
};

__device__ __forceinline__ uint32_t float_key(float f)
{
	const uint32_t u = __float_as_uint(f);
	return u ^ ((u >> 31) ? 0xffffffffu : 0x80000000u);
}
__device__ __forceinline__ float key_float(uint32_t k)
{
	return __uint_as_float(k ^ ((k >> 31) ? 0x80000000u : 0xffffffffu));
}

// ------------------------------------------------------------------------------------------------ radix sort (keys only)
__global__ void __launch_bounds__(256) km_keys_hist_kernel(const float* __restrict__ values, long long n, uint32_t* __restrict__ keys,
	uint32_t* __restrict__ hist)
{
	__shared__ uint32_t s_h[4 * 256];
	for (int i = threadIdx.x; i < 4 * 256; i += blockDim.x) s_h[i] = 0;
	__syncthreads();
	for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
	{
		const uint32_t k = float_key(values[i]);
		keys[i] = k;
#pragma unroll
		for (int p = 0; p < 4; p++) atomicAdd(&s_h[p * 256 + ((k >> (8 * p)) & 0xff)], 1u);
	}
	__syncthreads();
	for (int i = threadIdx.x; i < 4 * 256; i += blockDim.x) { const uint32_t c = s_h[i]; if (c) atomicAdd(&hist[i], c); }
}

__global__ void __launch_bounds__(256) km_sort_plan_kernel(const uint32_t* __restrict__ hist, long long n, KmSortPlan* plan)
{
	__shared__ uint32_t s_scan[256];
	__shared__ uint32_t s_skip[4];
	const int d = threadIdx.x;
	if (d < 4) s_skip[d] = 0;
	__syncthreads();
	for (int p = 0; p < 4; p++)
	{
		const uint32_t c = hist[p * 256 + d];
		if (c == (uint32_t)n) s_skip[p] = 1;           // every key has this digit: the pass would be the identity
		s_scan[d] = c;
		__syncthreads();
		for (int o = 1; o < 256; o <<= 1)
		{
			const uint32_t t = d >= o ? s_scan[d - o] : 0u;
			__syncthreads();
			s_scan[d] += t;
			__syncthreads();
		}
		plan->digit_base[p][d] = s_scan[d] - c;
		__syncthreads();
	}
	if (d == 0)
	{
		uint32_t cur = 0;
		for (int p = 0; p < 4; p++)
		{
			const uint32_t sk = s_skip[p] == 1;
			plan->skip[p] = sk; plan->src[p] = cur;
			if (!sk) cur ^= 1u;
		}
		plan->final_buf = cur;
	}
}

#define KM_LB_AGG 0x40000000u
#define KM_LB_INC 0x80000000u
#define KM_LB_VAL 0x3fffffffu
// One onesweep pass: tile = 4096 consecutive keys; warp w ranks keys [512 w, 512 (w+1)) in 16 warp-wide steps with match.any
// (stable), digit counts are chained across tiles with decoupled look-back.  PAIRS: a 32-bit value travels with each key
// (the kNN's (Morton code, point index) sort); the k-means sorts keys only.
template <bool PAIRS>
__global__ void __launch_bounds__(256) km_sort_pass_kernel(uint32_t* keys0, uint32_t* keys1, uint32_t* vals0, uint32_t* vals1, long long n,
	int pass, const KmSortPlan* __restrict__ plan, uint32_t* lookback_all, uint32_t* tickets, size_t n_tiles)
{
	if (plan->skip[pass]) return;
	const uint32_t srcb = plan->src[pass];
	const uint32_t* __restrict__ kin = srcb ? keys1 : keys0;
	uint32_t* __restrict__ kout = srcb ? keys0 : keys1;
	const uint32_t* __restrict__ vin = srcb ? vals1 : vals0;
	uint32_t* __restrict__ vout = srcb ? vals0 : vals1;
	uint32_t* lookback = lookback_all + (size_t)pass * n_tiles * 256;

	__shared__ uint32_t s_whist[8][256];
	__shared__ uint32_t s_dstart[256];
	__shared__ uint32_t s_gbase[256];
	__shared__ uint32_t s_keys[KM_TILE];
	__shared__ uint32_t s_vals[PAIRS ? KM_TILE : 1];
	__shared__ uint32_t s_tile;

	const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
	if (tid == 0) s_tile = atomicAdd(&tickets[pass], 1u);
	for (int i = tid; i < 8 * 256; i += 256) (&s_whist[0][0])[i] = 0;
	__syncthreads();
	const uint32_t tile = s_tile;
	const long long tbase = (long long)tile * KM_TILE;
	const int count = (int)min((long long)KM_TILE, n - tbase);
	const int shift = 8 * pass;

	uint32_t key[KM_ITEMS], rank[KM_ITEMS], val[PAIRS ? KM_ITEMS : 1];
	const unsigned lt = (1u << lane) - 1u;
#pragma unroll
	for (int i = 0; i < KM_ITEMS; i++)
	{
		const int local = warp * (32 * KM_ITEMS) + i * 32 + lane;
		const bool valid = local < count;
		key[i] = valid ? kin[tbase + local] : 0xffffffffu;
		if (PAIRS) val[i] = valid ? vin[tbase + local] : 0u;
		const uint32_t d = valid ? ((key[i] >> shift) & 0xff) : 256u;
		const unsigned vmask = __ballot_sync(0xffffffffu, valid);
		const unsigned m = __match_any_sync(0xffffffffu, d) & vmask;
		rank[i] = 0;
		if (valid)
		{
			const int leader = __ffs(m) - 1;
			uint32_t old = 0;
			if (lane == leader) { old = s_whist[warp][d]; s_whist[warp][d] = old + __popc(m); }
			old = __shfl_sync(m, old, leader);
			rank[i] = old + __popc(m & lt);
		}
		__syncwarp();
	}
	__syncthreads();
	uint32_t total = 0;
#pragma unroll
	for (int w = 0; w < 8; w++) { const uint32_t c = s_whist[w][tid]; s_whist[w][tid] = total; total += c; }
	uint32_t excl = 0;
	if (tile == 0) atomicExch(&lookback[tid], KM_LB_INC | total);
	else
	{
		atomicExch(&lookback[(size_t)tile * 256 + tid], KM_LB_AGG | total);
		long long j = (long long)tile - 1;
		while (true)
		{
			uint32_t c;
			do { c = *reinterpret_cast<volatile uint32_t*>(&lookback[(size_t)j * 256 + tid]); } while (c == 0);
			excl += c & KM_LB_VAL;
			if (c & KM_LB_INC) break;
			j--;
		}
		atomicExch(&lookback[(size_t)tile * 256 + tid], KM_LB_INC | (excl + total));
	}
	s_dstart[tid] = total;
	__syncthreads();
	for (int o = 1; o < 256; o <<= 1)
	{
		const uint32_t t = tid >= o ? s_dstart[tid - o] : 0u;
		__syncthreads();
		s_dstart[tid] += t;
		__syncthreads();
	}
	const uint32_t dstart = s_dstart[tid] - total;
	__syncthreads();
	s_dstart[tid] = dstart;
	s_gbase[tid] = plan->digit_base[pass][tid] + excl - dstart;
	__syncthreads();
#pragma unroll
	for (int i = 0; i < KM_ITEMS; i++)
	{
		const int local = warp * (32 * KM_ITEMS) + i * 32 + lane;
		if (local < count)
		{
			const uint32_t d = (key[i] >> shift) & 0xff;
			const uint32_t pos = s_dstart[d] + s_whist[warp][d] + rank[i];
			s_keys[pos] = key[i];
			if (PAIRS) s_vals[pos] = val[i];
		}
	}
	__syncthreads();
#pragma unroll
	for (int i = 0; i < KM_ITEMS; i++)
	{
		const int p = i * 256 + tid;
		if (p < count)
		{
			const uint32_t k = s_keys[p];
			const uint32_t dst = s_gbase[(k >> shift) & 0xff] + p;
			kout[dst] = k;
			if (PAIRS) vout[dst] = s_vals[p];
		}
	}
}

// ------------------------------------------------------------------------------------------------ Lloyd iteration
// Sorted centres in shared memory: value ascending, ties by original index; run_start / run_end delimit runs of EQUAL values.
struct KmCentres {
	float c[KM_MAX_K];
	int idx[KM_MAX_K];
	short run_start[KM_MAX_K];
	short run_end[KM_MAX_K];         // one past the run's last element
};

__device__ void km_load_sorted_centres(KmCentres& S, const float* __restrict__ centres, int K)
{
	__shared__ unsigned long long s_key[KM_MAX_K];
	int Kp = 1;
	while (Kp < K) Kp <<= 1;
	for (int i = threadIdx.x; i < Kp; i += blockDim.x)
		s_key[i] = i < K ? (((unsigned long long)float_key(centres[i]) << 32) | (uint32_t)i) : ~0ull;
	__syncthreads();
	for (int k = 2; k <= Kp; k <<= 1)
		for (int j = k >> 1; j > 0; j >>= 1)
		{
			for (int i = threadIdx.x; i < Kp; i += blockDim.x)
			{
				const int l = i ^ j;
				if (l > i)
				{
					const unsigned long long a = s_key[i], b = s_key[l];
					const bool up = (i & k) == 0;
					if ((a > b) == up) { s_key[i] = b; s_key[l] = a; }
				}
			}
			__syncthreads();
		}
	for (int i = threadIdx.x; i < K; i += blockDim.x)
	{
		S.c[i] = key_float((uint32_t)(s_key[i] >> 32));
		S.idx[i] = (int)(uint32_t)s_key[i];
	}
	__syncthreads();
	for (int i = threadIdx.x; i < K; i += blockDim.x)
	{
		int a = i;
		while (a > 0 && S.c[a - 1] == S.c[i]) a--;
		int b = i + 1;
		while (b < K && S.c[b] == S.c[i]) b++;
		S.run_start[i] = (short)a; S.run_end[i] = (short)b;
	}
	__syncthreads();
}

// kmeans.cu:6-9 distanceCUDA(value, centre) = sqrt((centre - value) * (centre - value))
__device__ __forceinline__ float km_dist(float v, float c)
{
	const float d = __fsub_rn(c, v);
	return __fsqrt_rn(__fmul_rn(d, d));
}

// kmeans.cu:83-104: argmin over the centres in ORIGINAL order with a strict `<`, i.e. the smallest distance and, among equal
// (rounded) distances, the smallest original index; 0 when no distance is below +inf (or the value is NaN).
__device__ __forceinline__ int km_assign(const KmCentres& S, int K, float v)
{
	int lo = 0, hi = K;                                       // lower bound: first centre >= v
	while (lo < hi)
	{
		const int mid = (lo + hi) >> 1;
		if (S.c[mid] < v) lo = mid + 1; else hi = mid;
	}
	const int j = lo;
	const float dl = j > 0 ? km_dist(v, S.c[j - 1]) : INFINITY, dr = j < K ? km_dist(v, S.c[j]) : INFINITY;
	const float dmin = fminf(dl, dr);
	if (!(dmin < INFINITY)) return 0;
	int best = 0x7fffffff;
	for (int p = j - 1; p >= 0 && km_dist(v, S.c[p]) == dmin; p = S.run_start[p] - 1) best = min(best, S.idx[S.run_start[p]]);
	for (int p = j; p < K && km_dist(v, S.c[p]) == dmin; p = S.run_end[p]) best = min(best, S.idx[p]);
	return best;
}

__global__ void __launch_bounds__(256) km_accumulate_kernel(const uint32_t* __restrict__ sorted_keys, long long n, const float* __restrict__ centres,
	int K, float* __restrict__ sums, int* __restrict__ sizes, const KmState* __restrict__ state)
{
	if (state->done) return;
	__shared__ KmCentres S;
	km_load_sorted_centres(S, centres, K);
	const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
	const long long a = t * KM_CHUNK, b = min(n, a + KM_CHUNK);
	int cur = -1, cnt = 0;
	float sum = 0.0f;
	for (long long i = a; i < b; i++)
	{
		const float v = key_float(sorted_keys[i]);
		const int id = km_assign(S, K, v);
		if (id != cur)
		{
			if (cnt) { atomicAdd(&sums[cur], sum); atomicAdd(&sizes[cur], cnt); }
			cur = id; cnt = 0; sum = 0.0f;
		}
		sum += v; cnt++;
	}
	// the open run: lanes of a warp nearly always agree on the cluster (sorted values) -> one pair of reductions per warp
	const unsigned same = __match_any_sync(0xffffffffu, cur);
	if (same == 0xffffffffu)
	{
#pragma unroll
		for (int o = 16; o > 0; o >>= 1) { sum += __shfl_xor_sync(0xffffffffu, sum, o); cnt += __shfl_xor_sync(0xffffffffu, cnt, o); }
		if ((threadIdx.x & 31) == 0 && cnt) { atomicAdd(&sums[cur], sum); atomicAdd(&sizes[cur], cnt); }
	}
	else if (cnt) { atomicAdd(&sums[cur], sum); atomicAdd(&sizes[cur], cnt); }
}

// reduced_3dgs.cu:322-327: new = sums / sizes (NaN -> 0), shift = sum |old - new|, stop when shift < tol; also clears the
// accumulators for the next iteration.  One CTA.
__global__ void __launch_bounds__(256) km_update_kernel(float* __restrict__ centres, int K, float* __restrict__ sums, int* __restrict__ sizes,
	float tol, int max_iterations, KmState* state)
{
	if (state->done) return;
	__shared__ float s_red[256];
	float part = 0.0f;
	for (int i = threadIdx.x; i < K; i += blockDim.x)
	{
		const float old = centres[i];
		float nc = __fdiv_rn(sums[i], (float)sizes[i]);
		if (isnan(nc)) nc = 0.0f;
		centres[i] = nc;
		sums[i] = 0.0f; sizes[i] = 0;
		part += fabsf(old - nc);
	}
	s_red[threadIdx.x] = part;
	__syncthreads();
	for (int o = 128; o > 0; o >>= 1)
	{
		if (threadIdx.x < o) s_red[threadIdx.x] += s_red[threadIdx.x + o];
		__syncthreads();
	}
	if (threadIdx.x == 0)
	{
		const int it = state->iterations + 1;
		state->iterations = it;
		state->shift = s_red[0];
		if (s_red[0] < tol || it >= max_iterations) state->done = 1;
	}
}

// Final ids in the ORIGINAL order of the values (reduced_3dgs.cu:330-335).
__global__ void __launch_bounds__(256) km_ids_kernel(const float* __restrict__ values, long long n, const float* __restrict__ centres, int K,
	int* __restrict__ ids)
{
	__shared__ KmCentres S;
	km_load_sorted_centres(S, centres, K);
	for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
		ids[i] = km_assign(S, K, values[i]);
}

// ------------------------------------------------------------------------------------------------ host
struct KmWorkspace {
	uint32_t* keys0; uint32_t* keys1; uint32_t* hist; KmSortPlan* plan; uint32_t* lookback; uint32_t* tickets;
	float* sums; int* sizes; KmState* state; size_t n_tiles; size_t bytes;
};
static KmWorkspace km_carve(char* base, long long n, int K)
{
	Carver c(base);
	KmWorkspace w;
	const size_t nn = n > 0 ? (size_t)n : 1;
	w.n_tiles = (nn + KM_TILE - 1) / KM_TILE;
	w.keys0 = c.take<uint32_t>(nn); w.keys1 = c.take<uint32_t>(nn);
	w.hist = c.take<uint32_t>(4 * 256);
	w.plan = c.take<KmSortPlan>(1);
	w.lookback = c.take<uint32_t>(4 * w.n_tiles * 256);
	w.tickets = c.take<uint32_t>(4);
	w.sums = c.take<float>(KM_MAX_K); w.sizes = c.take<int>(KM_MAX_K);
	w.state = c.take<KmState>(1);
	w.bytes = c.off + 256;
	(void)K;
	return w;
}

size_t kmeans_workspace_bytes(long long n, int K) { return km_carve(nullptr, n, K).bytes; }

int launch_kmeans(const float* values, long long n, const float* centres_in, int K, float tol, int max_iterations, int* ids, float* centres,
	char* workspace, cudaStream_t stream)
{
	if (K <= 0 || K > KM_MAX_K) { set_error("kmeans: number of centres must be in 1..%d", KM_MAX_K); return GSB_EINVAL; }
	ProfScope prof(K_KMEANS, stream);
	GSB_CUDA_OK(cudaMemcpyAsync(centres, centres_in, sizeof(float) * K, cudaMemcpyDeviceToDevice, stream));
	if (n <= 0) return GSB_OK;
	KmWorkspace w = km_carve(workspace, n, K);
	const int grid_ids = (int)std::min<long long>((n + 255) / 256, GSB_NUM_SMS * 8);
	if (max_iterations > 0)
	{
		// ---- sort the values once
		GSB_CUDA_OK(cudaMemsetAsync(w.hist, 0, sizeof(uint32_t) * 4 * 256, stream));
		GSB_CUDA_OK(cudaMemsetAsync(w.lookback, 0, sizeof(uint32_t) * 4 * w.n_tiles * 256, stream));
		GSB_CUDA_OK(cudaMemsetAsync(w.tickets, 0, sizeof(uint32_t) * 4, stream));
		GSB_CUDA_OK(cudaMemsetAsync(w.sums, 0, sizeof(float) * KM_MAX_K, stream));
		GSB_CUDA_OK(cudaMemsetAsync(w.sizes, 0, sizeof(int) * KM_MAX_K, stream));
		GSB_CUDA_OK(cudaMemsetAsync(w.state, 0, sizeof(KmState), stream));
		km_keys_hist_kernel<<<GSB_NUM_SMS * 4, 256, 0, stream>>>(values, n, w.keys0, w.hist);
		GSB_LAUNCHED();
		km_sort_plan_kernel<<<1, 256, 0, stream>>>(w.hist, n, w.plan);
		GSB_LAUNCHED();
		for (int p = 0; p < 4; p++)
		{
			km_sort_pass_kernel<false><<<(unsigned)w.n_tiles, 256, 0, stream>>>(w.keys0, w.keys1, nullptr, nullptr, n, p, w.plan, w.lookback,
				w.tickets, w.n_tiles);
			GSB_LAUNCHED();
		}
		static thread_local KmSortPlan* h_plan = nullptr;
		static thread_local KmState* h_state = nullptr;
		if (!h_plan) { GSB_CUDA_OK(cudaMallocHost(&h_plan, sizeof(KmSortPlan))); GSB_CUDA_OK(cudaMallocHost(&h_state, sizeof(KmState))); }
		GSB_CUDA_OK(cudaMemcpyAsync(h_plan, w.plan, sizeof(KmSortPlan), cudaMemcpyDeviceToHost, stream));
		GSB_CUDA_OK(cudaStreamSynchronize(stream));
		const uint32_t* sorted = h_plan->final_buf ? w.keys1 : w.keys0;
		// ---- Lloyd iterations; the device decides when to stop, the host polls the flag every 16 iterations
		const long long threads = (n + KM_CHUNK - 1) / KM_CHUNK;
		const unsigned grid_acc = (unsigned)((threads + 255) / 256);
		int launched = 0;
		while (launched < max_iterations)
		{
			const int batch = std::min(16, max_iterations - launched);
			for (int i = 0; i < batch; i++)
			{
				km_accumulate_kernel<<<grid_acc, 256, 0, stream>>>(sorted, n, centres, K, w.sums, w.sizes, w.state);
				GSB_LAUNCHED();
				km_update_kernel<<<1, 256, 0, stream>>>(centres, K, w.sums, w.sizes, tol, max_iterations, w.state);
				GSB_LAUNCHED();
			}
			launched += batch;
			GSB_CUDA_OK(cudaMemcpyAsync(h_state, w.state, sizeof(KmState), cudaMemcpyDeviceToHost, stream));
			GSB_CUDA_OK(cudaStreamSynchronize(stream));
			if (h_state->done) break;
		}
	}
	km_ids_kernel<<<grid_ids, 256, 0, stream>>>(values, n, centres, K, ids);
	GSB_LAUNCHED();
	GSB_CUDA_OK(cudaGetLastError());
	return GSB_OK;
}

// ------------------------------------------------------------------------------------------------ pair sort (gsb_knn.cu)
// The same onesweep sort on (key, value) pairs, keys in keys0 / values in vals0, with the caller's 4 x 256 digit histogram.  Fully
// asynchronous: the sorted pairs end in buffer *final_buf (0: keys0 / vals0, 1: keys1 / vals1), a DEVICE word the consumer reads.
static void sort_pairs_carve(char* base, long long n, KmSortPlan** plan, uint32_t** lookback, uint32_t** tickets, size_t* n_tiles, size_t* bytes)
{
	Carver c(base);
	*n_tiles = ((n > 0 ? (size_t)n : 1) + KM_TILE - 1) / KM_TILE;
	*plan = c.take<KmSortPlan>(1);
	*lookback = c.take<uint32_t>(4 * *n_tiles * 256);
	*tickets = c.take<uint32_t>(4);
	*bytes = c.off + 256;
}

size_t sort_pairs_scratch_bytes(long long n)
{
	KmSortPlan* plan; uint32_t *lookback, *tickets; size_t n_tiles, bytes;
	sort_pairs_carve(nullptr, n, &plan, &lookback, &tickets, &n_tiles, &bytes);
	return bytes;
}

int launch_sort_pairs(uint32_t* keys0, uint32_t* keys1, uint32_t* vals0, uint32_t* vals1, long long n, const uint32_t* hist, char* scratch,
	const uint32_t** final_buf, cudaStream_t stream)
{
	KmSortPlan* plan; uint32_t *lookback, *tickets; size_t n_tiles, bytes;
	sort_pairs_carve(scratch, n, &plan, &lookback, &tickets, &n_tiles, &bytes);
	*final_buf = &plan->final_buf;
	GSB_CUDA_OK(cudaMemsetAsync(lookback, 0, sizeof(uint32_t) * 4 * n_tiles * 256, stream));
	GSB_CUDA_OK(cudaMemsetAsync(tickets, 0, sizeof(uint32_t) * 4, stream));
	km_sort_plan_kernel<<<1, 256, 0, stream>>>(hist, n, plan);
	GSB_LAUNCHED();
	for (int p = 0; p < 4; p++)
	{
		km_sort_pass_kernel<true><<<(unsigned)n_tiles, 256, 0, stream>>>(keys0, keys1, vals0, vals1, n, p, plan, lookback, tickets, n_tiles);
		GSB_LAUNCHED();
	}
	return GSB_OK;
}

} // namespace gsb
