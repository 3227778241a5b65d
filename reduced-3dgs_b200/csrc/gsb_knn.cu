// gsb_knn.cu — exact k nearest neighbours of a point cloud (SURVEY.md §8(f) row 5), the drop-in for the reference's second
// extension simple_knn._C (submodules/simple-knn: distCUDA2, distIndex2, distIndexQ).
//
// The reference sorts the points by Morton code, cuts them into boxes of 128 (1024 for distCUDA2) and lets every query test
// EVERY box (simple_knn.cu:149-185, :422-465, :523-575): P^2 / 128 box tests, K-best lists in global memory, and two blocking
// device-to-host copies of the bounding box per call.  Here:
//   bounds (device, atomics on order-preserving integers) -> 90-bit Morton codes (30 bits per axis, computed in double) -> stable
//   (code, index) sort as three LSD radix sorts of 30-bit words (the k-means onesweep sort of gsb_kmeans.cu with a payload) ->
//   sorted points as float4 (x, y, z, index bits) -> leaf boxes of 32 sorted points -> a 32-ary box tree over the leaves, up to
//   one root.  30 bits per axis is finer than fp32 itself resolves the coordinates of a scene whose bounding box is stretched by
//   far outliers (the cell of a 4000-unit box is 4e-6), so dense clusters still fall into compact leaves (with 10 bits per axis whole
//   blobs shared a cell, in index order, and every query there opened the whole cell);
//   queries: one warp per 32 Morton-consecutive queries (an explicit query list is first sorted by the Morton rank of its points).  The warp walks the tree
//   depth-first, children nearest-first; a node is opened when it may hold a better neighbour for ANY lane; a leaf is staged
//   in shared memory once and every lane tests its 32 points against its own query.  The K best of a lane are u64 keys
//   (float bits of the distance << 32 | index) kept sorted in shared memory: distances are >= 0, so unsigned order is exactly
//   (distance, index) order, and the result is the K smallest keys — a function of the points alone, whatever the visiting
//   order, hence identical bytes from run to run.
//
// Arithmetic (gsb_common.cuh policy): the point distance is the reference's SASS sequence (boxMeanDist, boxKnn2 of its sm_90
// build): FADD x3; FMUL dy,dy; FFMA dx,dx,.; FFMA dz,dz,. — y first — written with explicit intrinsics.  Box distances use the same monotone operations on the box faces, so they never exceed the
// distance of a point inside the box, and pruning "box distance > K-th distance" is exact.  Candidates at a distance >= FLT_MAX
// (overflow, NaN coordinates) are never taken — the reference's `dist >= reject` (reject starts at FLT_MAX) — so unfilled slots
// stay (FLT_MAX, -1).
#include <algorithm>
#include <cfloat>
#include "gsb_common.cuh"

namespace gsb {

#define KNN_LEAF 32
#define KNN_MAX_LEVELS 8                    // P < 2^30 needs at most 6 levels of 32-ary boxes
#define KNN_STACK (32 * KNN_MAX_LEVELS)    // DFS: at most 31 siblings wait per level, plus the 32 children just pushed
#define KNN_WARPS 4
#define KNN_NONE 0xffffffffu                // index of an empty slot / of a padding point
#define KNN_SKIP 0x80000000u                // index bit of a sorted point that is no candidate (padding, or not listed for distIndexQ)
#define KNN_EXCLUDED (1u << 30)             // bit of the most significant code word of a non-candidate: sorts after every candidate
#define KNN_WORDS 3                         // 30-bit words of the Morton code, least significant first
#define KNN_FLT_MAX_BITS 0x7f7fffffu

struct KnnLevels {
	int n;                                   // number of levels (0: no point)
	long long off[KNN_MAX_LEVELS];           // first box of level l in the box arrays (level 0 = leaves)
	long long count[KNN_MAX_LEVELS];         // boxes in level l
};

static KnnLevels knn_levels(long long P)
{
	KnnLevels L{};
	long long c = (P + KNN_LEAF - 1) / KNN_LEAF, off = 0;
	while (c > 0)
	{
		L.off[L.n] = off; L.count[L.n] = c; off += c; L.n++;
		if (c == 1) break;
		c = (c + 31) / 32;
	}
	return L;
}

// simple_knn.cu:137 / :228 / :400 `d = point - ref; d.x*d.x + d.y*d.y + d.z*d.z` as the reference's SASS evaluates it
__device__ __forceinline__ float knn_dist(float px, float py, float pz, float qx, float qy, float qz)
{
	const float dx = __fsub_rn(px, qx), dy = __fsub_rn(py, qy), dz = __fsub_rn(pz, qz);
	return __fmaf_rn(dz, dz, __fmaf_rn(dx, dx, __fmul_rn(dy, dy)));
}
// Lower bound of knn_dist over every point of [lo, hi] seen from q: per axis the rounded distance to the nearer face (rounding is
// monotone, so it is <= every |p - q| rounded), squared and summed with the same operations.  An empty box (lo > hi) gives +inf.
__device__ __forceinline__ float knn_gap(float lo, float hi, float q) { return fmaxf(fmaxf(__fsub_rn(lo, q), __fsub_rn(q, hi)), 0.0f); }
__device__ __forceinline__ float knn_box_point(const float4& lo, const float4& hi, float qx, float qy, float qz)
{
	if (!(lo.x <= hi.x)) return INFINITY;
	const float gx = knn_gap(lo.x, hi.x, qx), gy = knn_gap(lo.y, hi.y, qy), gz = knn_gap(lo.z, hi.z, qz);
	return __fmaf_rn(gz, gz, __fmaf_rn(gx, gx, __fmul_rn(gy, gy)));
}
// Lower bound over every pair (query in the warp's box [wlo, whi], point in [lo, hi]).
__device__ __forceinline__ float knn_box_gap(float lo, float hi, float wlo, float whi)
{
	return fmaxf(fmaxf(__fsub_rn(lo, whi), __fsub_rn(wlo, hi)), 0.0f);
}
__device__ __forceinline__ float knn_box_box(const float4& lo, const float4& hi, const float3& wlo, const float3& whi)
{
	if (!(lo.x <= hi.x)) return INFINITY;
	const float gx = knn_box_gap(lo.x, hi.x, wlo.x, whi.x), gy = knn_box_gap(lo.y, hi.y, wlo.y, whi.y), gz = knn_box_gap(lo.z, hi.z, wlo.z, whi.z);
	return __fmaf_rn(gz, gz, __fmaf_rn(gx, gx, __fmul_rn(gy, gy)));
}

// ------------------------------------------------------------------------------------------------ structure
// bounds[0..2] = min, bounds[3..5] = max of the coordinates as order-preserving integers (NaN ignored); pre-set to 0xff.. / 0.
__global__ void __launch_bounds__(256) knn_bounds_kernel(const float* __restrict__ points, long long P, uint32_t* __restrict__ bounds)
{
	float mn[3] = { INFINITY, INFINITY, INFINITY }, mx[3] = { -INFINITY, -INFINITY, -INFINITY };
	for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < P; i += (long long)gridDim.x * blockDim.x)
#pragma unroll
		for (int a = 0; a < 3; a++) { const float v = points[3 * i + a]; mn[a] = fminf(mn[a], v); mx[a] = fmaxf(mx[a], v); }
#pragma unroll
	for (int a = 0; a < 3; a++) { mn[a] = warp_min(mn[a]); mx[a] = warp_max(mx[a]); }
	if ((threadIdx.x & 31) == 0)
#pragma unroll
		for (int a = 0; a < 3; a++) { atomicMin(&bounds[a], float_key(mn[a])); atomicMax(&bounds[3 + a], float_key(mx[a])); }
}

// distIndexQ's candidate filter: flags[id] = 1 for the first min(N, P) listed ids (simple_knn.cu:577-589 runs P threads); ids
// outside [0, P) are ignored.
__global__ void __launch_bounds__(256) knn_flag_kernel(const int32_t* __restrict__ ids, long long n, long long P, uint8_t* __restrict__ flags)
{
	const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	const int32_t id = ids[i];
	if (id >= 0 && id < P) flags[id] = 1;
}

__device__ __forceinline__ uint32_t knn_spread10(uint32_t x)          // 10 bits -> every third bit
{
	x = (x | (x << 16)) & 0x030000FFu;
	x = (x | (x << 8)) & 0x0300F00Fu;
	x = (x | (x << 4)) & 0x030C30C3u;
	x = (x | (x << 2)) & 0x09249249u;
	return x;
}
// Cell of a coordinate on a 2^30 grid over [lo, lo + ext]; in double so that a far-away lo does not round the offset away.
// NaN -> 0.  A zero extent (all points on a plane / line / one spot) has scale 0: that axis maps to cell 0.
__device__ __forceinline__ uint32_t knn_cell(float v, double lo, double scale)
{
	return (uint32_t)fmin(fmax(((double)v - lo) * scale, 0.0), 1073741823.0);
}
struct KnnGrid { double lo[3], scale[3]; };
__device__ __forceinline__ KnnGrid knn_grid(const uint32_t* __restrict__ bounds)
{
	KnnGrid g;
#pragma unroll
	for (int a = 0; a < 3; a++)
	{
		g.lo[a] = (double)key_float(bounds[a]);
		const double ext = (double)key_float(bounds[3 + a]) - g.lo[a];
		g.scale[a] = (ext > 0.0 && ext <= 1e300) ? 1073741823.0 / ext : 0.0;
	}
	return g;
}
// Word w (bits [30 w, 30 w + 30)) of point i's Morton code; the top word carries KNN_EXCLUDED for a non-candidate.
__device__ __forceinline__ uint32_t knn_word(const float* __restrict__ points, long long i, const KnnGrid& g, const uint8_t* __restrict__ flags, int w)
{
	const int sh = 10 * w;
	uint32_t k = knn_spread10((knn_cell(points[3 * i], g.lo[0], g.scale[0]) >> sh) & 1023u) |
	             (knn_spread10((knn_cell(points[3 * i + 1], g.lo[1], g.scale[1]) >> sh) & 1023u) << 1) |
	             (knn_spread10((knn_cell(points[3 * i + 2], g.lo[2], g.scale[2]) >> sh) & 1023u) << 2);
	if (w == KNN_WORDS - 1 && flags && !flags[i]) k |= KNN_EXCLUDED;
	return k;
}

// keys[i] = the least significant code word of point i, vals[i] = i, and the 4 x 256 digit histograms of ALL words (a histogram
// does not depend on the order, so the later sorts of the permuted words reuse them): hist[w][4][256].
__global__ void __launch_bounds__(256) knn_codes_kernel(const float* __restrict__ points, long long P, const uint32_t* __restrict__ bounds,
	const uint8_t* __restrict__ flags, uint32_t* __restrict__ keys, uint32_t* __restrict__ vals, uint32_t* __restrict__ hist)
{
	__shared__ uint32_t s_h[KNN_WORDS * 4 * 256];
	for (int i = threadIdx.x; i < KNN_WORDS * 4 * 256; i += blockDim.x) s_h[i] = 0;
	__syncthreads();
	const KnnGrid g = knn_grid(bounds);
	for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < P; i += (long long)gridDim.x * blockDim.x)
	{
#pragma unroll
		for (int w = 0; w < KNN_WORDS; w++)
		{
			const uint32_t k = knn_word(points, i, g, flags, w);
			if (w == 0) { keys[i] = k; vals[i] = (uint32_t)i; }
#pragma unroll
			for (int p = 0; p < 4; p++) atomicAdd(&s_h[(w * 4 + p) * 256 + ((k >> (8 * p)) & 0xff)], 1u);
		}
	}
	__syncthreads();
	for (int i = threadIdx.x; i < KNN_WORDS * 4 * 256; i += blockDim.x) { const uint32_t c = s_h[i]; if (c) atomicAdd(&hist[i], c); }
}

// Next LSD step: the points in the order the previous word's sort left them (*final_buf selects its buffer), keyed by word w.
__global__ void __launch_bounds__(256) knn_permute_kernel(const float* __restrict__ points, long long P, const uint32_t* __restrict__ bounds,
	const uint8_t* __restrict__ flags, int w, const uint32_t* vals0, const uint32_t* vals1, const uint32_t* __restrict__ final_buf,
	uint32_t* __restrict__ keys_out, uint32_t* __restrict__ vals_out)
{
	const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
	if (j >= P) return;
	const uint32_t v = (*final_buf ? vals1 : vals0)[j];
	vals_out[j] = v;
	keys_out[j] = knn_word(points, v, knn_grid(bounds), flags, w);
}

// An explicit query list in the Morton order of its points: key = sorted position (rank) of the query's point, ids outside [0, P)
// last; value = the query's slot.  With the 4 x 256 digit histogram.
__global__ void __launch_bounds__(256) knn_query_keys_kernel(const int32_t* __restrict__ query_ids, long long Q, long long P,
	const uint32_t* __restrict__ rank, uint32_t* __restrict__ keys, uint32_t* __restrict__ vals, uint32_t* __restrict__ hist)
{
	__shared__ uint32_t s_h[4 * 256];
	for (int i = threadIdx.x; i < 4 * 256; i += blockDim.x) s_h[i] = 0;
	__syncthreads();
	for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < Q; t += (long long)gridDim.x * blockDim.x)
	{
		const int32_t id = query_ids[t];
		const uint32_t k = (id >= 0 && id < P) ? rank[id] : (1u << 30);
		keys[t] = k;
		vals[t] = (uint32_t)t;
#pragma unroll
		for (int p = 0; p < 4; p++) atomicAdd(&s_h[p * 256 + ((k >> (8 * p)) & 0xff)], 1u);
	}
	__syncthreads();
	for (int i = threadIdx.x; i < 4 * 256; i += blockDim.x) { const uint32_t c = s_h[i]; if (c) atomicAdd(&hist[i], c); }
}

// Sorted points as (x, y, z, index bits); padding up to a whole leaf is KNN_NONE, non-candidates carry KNN_SKIP | index.
// rank (may be NULL): rank[v] = sorted position of point v.
__global__ void __launch_bounds__(256) knn_gather_kernel(const float* __restrict__ points, long long P, long long n_padded,
	const uint32_t* keys0, const uint32_t* keys1, const uint32_t* vals0, const uint32_t* vals1, const uint32_t* __restrict__ final_buf,
	float4* __restrict__ pts, uint32_t* __restrict__ rank)
{
	const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n_padded) return;
	float4 r = make_float4(0.0f, 0.0f, 0.0f, __uint_as_float(KNN_NONE));
	if (i < P)
	{
		const bool b = *final_buf != 0;
		const uint32_t k = (b ? keys1 : keys0)[i], v = (b ? vals1 : vals0)[i];
		r = make_float4(points[3 * (size_t)v], points[3 * (size_t)v + 1], points[3 * (size_t)v + 2], __uint_as_float((k & KNN_EXCLUDED) ? (KNN_SKIP | v) : v));
		if (rank) rank[v] = (uint32_t)i;
	}
	pts[i] = r;
}

// One warp per box: leaves bound their 32 points (excluded / padding points do not count), upper levels their 32 children.
// An empty box is (+inf, -inf).
__global__ void __launch_bounds__(256) knn_box_kernel(const float4* __restrict__ pts, const float4* __restrict__ child_lo,
	const float4* __restrict__ child_hi, long long n_children, long long n_boxes, float4* __restrict__ lo, float4* __restrict__ hi)
{
	const long long box = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
	const int lane = threadIdx.x & 31;
	if (box >= n_boxes) return;
	const long long c = box * 32 + lane;
	float3 a = make_float3(INFINITY, INFINITY, INFINITY), b = make_float3(-INFINITY, -INFINITY, -INFINITY);
	if (pts)
	{
		const float4 p = pts[c];
		if (!(__float_as_uint(p.w) & KNN_SKIP)) { a = make_float3(p.x, p.y, p.z); b = a; }
	}
	else if (c < n_children)
	{
		const float4 l = child_lo[c], h = child_hi[c];
		if (l.x <= h.x) { a = make_float3(l.x, l.y, l.z); b = make_float3(h.x, h.y, h.z); }
	}
	a.x = warp_min(a.x); a.y = warp_min(a.y); a.z = warp_min(a.z);
	b.x = warp_max(b.x); b.y = warp_max(b.y); b.z = warp_max(b.z);
	if (lane == 0) { lo[box] = make_float4(a.x, a.y, a.z, 0.0f); hi[box] = make_float4(b.x, b.y, b.z, 0.0f); }
}

// ------------------------------------------------------------------------------------------------ queries
struct KnnQuery {
	const float* points; long long P;
	const float4* pts;                       // sorted points
	const float4* lo; const float4* hi;      // boxes of every level
	KnnLevels L;
	const int32_t* query_ids; long long n_queries;   // NULL: query t is sorted point t, its row is the point's index
	const uint32_t *order0, *order1, *order_final;   // query list only (may be NULL): slot j takes query (*order_final ? order1 : order0)[j]
	int K;
	float* dists; int32_t* indices; float* mean3;
};

__device__ __forceinline__ uint32_t knn_node(int level, long long i) { return ((uint32_t)level << 27) | (uint32_t)i; }

// Dynamic shared memory per warp: the K-best lists [K][32] u64, the DFS stack, one staged leaf.
__global__ void __launch_bounds__(KNN_WARPS * 32) knn_query_kernel(const KnnQuery a)
{
	extern __shared__ __align__(16) unsigned char knn_smem[];
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, K = a.K;
	unsigned long long* best = reinterpret_cast<unsigned long long*>(knn_smem) + (size_t)warp * K * 32 + lane;
	float4* cand = reinterpret_cast<float4*>(knn_smem + (size_t)KNN_WARPS * K * 32 * 8) + warp * 32;
	uint32_t* stack = reinterpret_cast<uint32_t*>(knn_smem + (size_t)KNN_WARPS * K * 32 * 8 + KNN_WARPS * 32 * 16) + warp * KNN_STACK;

	long long t = ((long long)blockIdx.x * KNN_WARPS + warp) * 32 + lane;
	if (a.order0 && t < a.n_queries) t = (*a.order_final ? a.order1 : a.order0)[t];
	bool active = false;
	long long row = -1;
	uint32_t self = KNN_NONE;
	float qx = 0.0f, qy = 0.0f, qz = 0.0f;
	if (t < a.n_queries)
	{
		if (a.query_ids)
		{
			const int32_t id = a.query_ids[t];
			row = t;
			if (id >= 0 && id < a.P)
			{
				active = true; self = (uint32_t)id;
				qx = a.points[3 * (size_t)id]; qy = a.points[3 * (size_t)id + 1]; qz = a.points[3 * (size_t)id + 2];
			}
		}
		else
		{
			const float4 p = a.pts[t];
			if (__float_as_uint(p.w) != KNN_NONE) { active = true; self = __float_as_uint(p.w) & ~KNN_SKIP; row = self; qx = p.x; qy = p.y; qz = p.z; }
		}
	}
	const unsigned long long EMPTY = ((unsigned long long)KNN_FLT_MAX_BITS << 32) | KNN_NONE;
	for (int k = 0; k < K; k++) best[k * 32] = EMPTY;
	unsigned long long kth = EMPTY;

	if (__any_sync(0xffffffffu, active) && a.L.n > 0)
	{
		float3 wlo, whi;                                 // box of the warp's queries
		wlo.x = warp_min(active ? qx : INFINITY); wlo.y = warp_min(active ? qy : INFINITY); wlo.z = warp_min(active ? qz : INFINITY);
		whi.x = warp_max(active ? qx : -INFINITY); whi.y = warp_max(active ? qy : -INFINITY); whi.z = warp_max(active ? qz : -INFINITY);
		if (lane == 0) stack[0] = knn_node(a.L.n - 1, 0);
		int top = 1;
		__syncwarp();
		while (top > 0)
		{
			top--;
			const uint32_t node = stack[top];
			const int level = (int)(node >> 27);
			const long long i = node & ((1u << 27) - 1);
			// this lane's bound: the K-th distance; a box at exactly that distance may still hold a smaller index
			const float thr = active ? __uint_as_float((uint32_t)(kth >> 32)) : -1.0f;
			const float4 blo = a.lo[a.L.off[level] + i], bhi = a.hi[a.L.off[level] + i];
			const bool need = knn_box_point(blo, bhi, qx, qy, qz) <= thr;
			if (!__any_sync(0xffffffffu, need)) continue;
			if (level == 0)
			{
				cand[lane] = a.pts[i * KNN_LEAF + lane];
				__syncwarp();
				if (need)
				{
					for (int c = 0; c < KNN_LEAF; c++)
					{
						const float4 p = cand[c];
						const uint32_t id = __float_as_uint(p.w);
						const float d = knn_dist(p.x, p.y, p.z, qx, qy, qz);
						const uint32_t db = __float_as_uint(d);
						const unsigned long long key = ((unsigned long long)db << 32) | id;
						if (key < kth && db < KNN_FLT_MAX_BITS && id != self && !(id & KNN_SKIP))
						{
							int pos = K - 1;
							while (pos > 0)
							{
								const unsigned long long prev = best[(pos - 1) * 32];
								if (prev < key) break;
								best[pos * 32] = prev;
								pos--;
							}
							best[pos * 32] = key;
							kth = best[(K - 1) * 32];
						}
					}
				}
				__syncwarp();
			}
			else
			{
				// children nearest-first (distance to the warp's box), pruned against the largest K-th distance of the warp
				const float wthr = warp_max(thr);
				const long long child = i * 32 + lane;
				float d = INFINITY;
				if (child < a.L.count[level - 1])
				{
					const long long o = a.L.off[level - 1] + child;
					d = knn_box_box(a.lo[o], a.hi[o], wlo, whi);
					if (!(d <= wthr)) d = INFINITY;
				}
				uint32_t id = (uint32_t)child;
				for (int size = 2; size <= 32; size <<= 1)           // bitonic sort of (d, child) over the lanes, ascending
					for (int stride = size >> 1; stride > 0; stride >>= 1)
					{
						const float od = __shfl_xor_sync(0xffffffffu, d, stride);
						const uint32_t oid = __shfl_xor_sync(0xffffffffu, id, stride);
						const bool up = (lane & size) == 0, lower = (lane & stride) == 0;
						const bool other_less = od < d || (od == d && oid < id);
						if (lower == up ? other_less : !other_less && !(od == d && oid == id)) { d = od; id = oid; }
					}
				const int nvalid = __popc(__ballot_sync(0xffffffffu, d < INFINITY));
				if (lane < nvalid) stack[top + nvalid - 1 - lane] = knn_node(level - 1, id);
				top += nvalid;
				__syncwarp();
			}
		}
	}
	if (row < 0) return;
	const size_t base = (size_t)row * K;
	if (a.dists || a.indices)
		for (int k = 0; k < K; k++)
		{
			const unsigned long long key = best[k * 32];
			if (a.dists) a.dists[base + k] = __uint_as_float((uint32_t)(key >> 32));
			if (a.indices) a.indices[base + k] = (int32_t)(uint32_t)key;
		}
	if (a.mean3)                                         // simple_knn.cu:184 (best[0] + best[1] + best[2]) / 3.0f
	{
		const float b0 = __uint_as_float((uint32_t)(best[0] >> 32)), b1 = __uint_as_float((uint32_t)(best[32] >> 32)),
		            b2 = __uint_as_float((uint32_t)(best[64] >> 32));
		a.mean3[row] = __fdiv_rn(__fadd_rn(__fadd_rn(b0, b1), b2), 3.0f);
	}
}

// ------------------------------------------------------------------------------------------------ host
// Two sets of (key, value) double buffers: the three word sorts alternate between them (A, B, A), each permute step reading the
// previous sort's result and writing the other set; the query-list sort reuses set B.
struct KnnWorkspace {
	uint32_t* bounds; uint32_t* hist; uint32_t* qhist; char* sort_scratch; uint32_t* buf[2][4]; uint8_t* flags; uint32_t* rank;
	float4* pts; float4* lo; float4* hi; size_t bytes;
};
static KnnWorkspace knn_carve(char* base, long long P, long long Q)
{
	Carver c(base);
	KnnWorkspace w;
	const size_t n = std::max<long long>(std::max(P, Q), 1);
	const KnnLevels L = knn_levels(P);
	const size_t boxes = L.n ? (size_t)(L.off[L.n - 1] + L.count[L.n - 1]) : 1;
	w.bounds = c.take<uint32_t>(8);
	w.hist = c.take<uint32_t>(KNN_WORDS * 4 * 256);
	w.qhist = c.take<uint32_t>(4 * 256);
	w.sort_scratch = c.take<char>(sort_pairs_scratch_bytes((long long)n));
	for (int s = 0; s < 2; s++)
		for (int b = 0; b < 4; b++) w.buf[s][b] = c.take<uint32_t>(n);      // keys0, keys1, vals0, vals1
	w.flags = c.take<uint8_t>(std::max<long long>(P, 1));
	w.rank = c.take<uint32_t>(std::max<long long>(P, 1));
	w.pts = c.take<float4>((n + KNN_LEAF - 1) / KNN_LEAF * KNN_LEAF);
	w.lo = c.take<float4>(boxes); w.hi = c.take<float4>(boxes);
	w.bytes = c.off + 256;
	return w;
}

size_t knn_workspace_bytes(long long P, long long n_queries) { return knn_carve(nullptr, P, n_queries < 0 ? 0 : n_queries).bytes; }

int launch_knn(const float* points, long long P, int K, const int32_t* query_ids, long long n_queries, const int32_t* candidate_ids,
	long long n_candidates, float* mean3, float* dists, int32_t* indices, char* workspace, cudaStream_t stream)
{
	const long long rows = query_ids ? n_queries : P;
	if (rows == 0 || K == 0) return GSB_OK;
	ProfScope prof(K_KNN, stream);
	KnnWorkspace w = knn_carve(workspace, P, query_ids ? rows : 0);
	KnnQuery q{};
	q.points = points; q.P = P; q.pts = w.pts; q.lo = w.lo; q.hi = w.hi;
	q.query_ids = query_ids; q.n_queries = rows; q.K = K; q.dists = dists; q.indices = indices; q.mean3 = mean3;
	if (P > 0)
	{
		q.L = knn_levels(P);
		const long long padded = q.L.count[0] * KNN_LEAF;
		GSB_CUDA_OK(cudaMemsetAsync(w.bounds, 0xff, sizeof(uint32_t) * 3, stream));
		GSB_CUDA_OK(cudaMemsetAsync(w.bounds + 3, 0, sizeof(uint32_t) * 3, stream));
		GSB_CUDA_OK(cudaMemsetAsync(w.hist, 0, sizeof(uint32_t) * KNN_WORDS * 4 * 256, stream));
		const unsigned grid = (unsigned)std::min<long long>((P + 255) / 256, GSB_NUM_SMS * 4);
		knn_bounds_kernel<<<grid, 256, 0, stream>>>(points, P, w.bounds);
		GSB_LAUNCHED();
		const uint8_t* flags = nullptr;
		if (n_candidates >= 0)                           // a candidate list (possibly empty); < 0: every point
		{
			GSB_CUDA_OK(cudaMemsetAsync(w.flags, 0, (size_t)P, stream));
			const long long n = std::min(n_candidates, P);
			if (n > 0)
			{
				knn_flag_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(candidate_ids, n, P, w.flags);
				GSB_LAUNCHED();
			}
			flags = w.flags;
		}
		knn_codes_kernel<<<grid, 256, 0, stream>>>(points, P, w.bounds, flags, w.buf[0][0], w.buf[0][2], w.hist);
		GSB_LAUNCHED();
		const uint32_t* final_buf = nullptr;
		for (int word = 0; word < KNN_WORDS; word++)         // LSD over the 30-bit words: stable, so the result is (code, index) order
		{
			uint32_t** b = w.buf[word & 1];
			if (word > 0)
			{
				uint32_t** prev = w.buf[(word - 1) & 1];
				knn_permute_kernel<<<(unsigned)((P + 255) / 256), 256, 0, stream>>>(points, P, w.bounds, flags, word, prev[2], prev[3], final_buf,
					b[0], b[2]);
				GSB_LAUNCHED();
			}
			if (int st = launch_sort_pairs(b[0], b[1], b[2], b[3], P, w.hist + word * 4 * 256, w.sort_scratch, &final_buf, stream)) return st;
		}
		uint32_t** last = w.buf[(KNN_WORDS - 1) & 1];
		knn_gather_kernel<<<(unsigned)((padded + 255) / 256), 256, 0, stream>>>(points, P, padded, last[0], last[1], last[2], last[3],
			final_buf, w.pts, query_ids ? w.rank : nullptr);
		GSB_LAUNCHED();
		if (query_ids)                                   // the query list in Morton order: warps of spatially close queries
		{
			static_assert(KNN_WORDS % 2 == 1, "the query sort uses set B, free after the last word sort in set A");
			uint32_t** b = w.buf[1];
			GSB_CUDA_OK(cudaMemsetAsync(w.qhist, 0, sizeof(uint32_t) * 4 * 256, stream));
			knn_query_keys_kernel<<<(unsigned)std::min<long long>((rows + 255) / 256, GSB_NUM_SMS * 4), 256, 0, stream>>>(query_ids, rows, P,
				w.rank, b[0], b[2], w.qhist);
			GSB_LAUNCHED();
			const uint32_t* qfinal = nullptr;
			if (int st = launch_sort_pairs(b[0], b[1], b[2], b[3], rows, w.qhist, w.sort_scratch, &qfinal, stream)) return st;
			q.order0 = b[2]; q.order1 = b[3]; q.order_final = qfinal;
		}
		for (int l = 0; l < q.L.n; l++)
		{
			const long long nb = q.L.count[l];
			const float4* clo = l ? w.lo + q.L.off[l - 1] : nullptr;
			const float4* chi = l ? w.hi + q.L.off[l - 1] : nullptr;
			knn_box_kernel<<<(unsigned)((nb * 32 + 255) / 256), 256, 0, stream>>>(l ? nullptr : w.pts, clo, chi, l ? q.L.count[l - 1] : 0, nb,
				w.lo + q.L.off[l], w.hi + q.L.off[l]);
			GSB_LAUNCHED();
		}
	}
	const int smem = KNN_WARPS * (K * 32 * 8 + 32 * 16 + KNN_STACK * 4);
	if (int st = ensure_dyn_smem((const void*)knn_query_kernel, smem)) return st;
	const long long blocks = (rows + KNN_WARPS * 32 - 1) / (KNN_WARPS * 32);
	knn_query_kernel<<<(unsigned)blocks, KNN_WARPS * 32, smem, stream>>>(q);
	GSB_LAUNCHED();
	GSB_CUDA_OK(cudaGetLastError());
	return GSB_OK;
}

} // namespace gsb
