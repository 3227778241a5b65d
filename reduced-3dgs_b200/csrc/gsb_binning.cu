// gsb_binning.cu — tile binning for sm_90a: count -> scan -> scatter -> per-tile sort.
//
// What the reference does (rasterizer_impl.cu:441-482): inclusive scan of tiles_touched, duplicateWithKeys into
// R (tile << 32 | depth bits, gaussian id) pairs, ONE global cub::DeviceRadixSort over all R 64-bit keys
// (6 digit passes = ~150 B of HBM traffic per instance), then identifyTileRanges.
//
// What this file does instead — same result, bit for bit, ~20 B of algorithmic traffic per instance, no global atomics:
//   1. the preprocess kernel counts (Gaussian, tile) pairs into a PER-CTA shared-memory tile histogram; every CTA owns a
//      contiguous chunk of Gaussians (BinPlan) and flushes its histogram as one row of cta_count[ctas][tiles];
//   2. tile_prefix_kernel: per tile, exclusive prefix over the CTA rows (in place) + tile totals;
//      tile_scan_kernel: exclusive scan of the T tile totals -> ranges[t] = (start, end) directly (== identifyTileRanges'
//      output), R, and the lists of tiles too large for the one-CTA sort classes;
//   3. scatter_priv_kernel: the same chunking again; slot = tile start + this CTA's prefix + shared-memory cursor; stores the
//      64-bit composite (depth bits << 32 | gaussian id) with an L2 evict_last policy into a bucket array that was just
//      written once with full-sector stores (the scattered 8-byte stores then hit in L2 instead of filling sectors from DRAM);
//   4. tile_sort_dist_kernel<256>: one CTA per tile, one-pass distribution sort (2048 order-preserving depth bins, then every
//      entry placed by its rank among its bin-mates by (depth bits, id)); tiles of 2049..8192 instances: the same kernel with
//      8192 bins on persistent 1024-thread CTAs; tiles whose depths cluster are queued on a device-side list for the stable
//      8-bit LSD radix sort in shared memory (tile_sort_kernel); beyond 8192 instances a single-CTA global-memory radix sort.
//      The large classes are launched only when non-empty (their sizes ride the R read-back).
//   Steps 3 and the small-tile part of 4 are launched SPECULATIVELY, before the host knows this frame's instance count
//   (gsb_api.cu gsb_forward): they compare the device-side count with the capacity they were given and do nothing if it is larger.
// The global stable sort by (tile, depth) with ties in emission order (ascending Gaussian id) is exactly "per tile, sort
// by (depth bits, id)": a Gaussian appears at most once per tile, so the composites are unique and the order is total.
// When the tile histogram does not fit in shared memory (> 160 KB, i.e. beyond ~8K images) counting and scattering fall
// back to global atomics (tile_count / scatter_kernel).
// (The first version of this file was a hand-written 8-bit onesweep radix sort; see git history and DESIGN.md.)
#include <algorithm>
#include <cstdlib>
#include "gsb_common.cuh"

namespace gsb {

// ------------------------------------------------------------------------------------------------
// Exclusive scan over the tile counters (T <= a few 10^4): one CTA, 1024 threads, sequential chunks.  The scan and the running
// carry are 64-bit: a total beyond 2^32 must not wrap silently.
__global__ void __launch_bounds__(1024) tile_scan_kernel(const uint32_t* __restrict__ tile_count, int T, uint2* __restrict__ ranges,
	uint32_t* __restrict__ counters, uint32_t* __restrict__ cursor, uint32_t* __restrict__ cls_list, uint32_t* __restrict__ cls_count)
{
	__shared__ unsigned long long s_warp[32];
	const int tid = threadIdx.x;
	if (tid == 0) { cls_count[0] = 0; cls_count[1] = 0; cls_count[2] = 0; cls_count[3] = 0; }
	__syncthreads();
	unsigned long long carry = 0;
	for (int base = 0; base < T; base += 1024)
	{
		const int t = base + tid;
		const uint32_t c = t < T ? tile_count[t] : 0u;
		unsigned long long total;
		const unsigned long long start64 = carry + cta_exclusive<1024>((unsigned long long)c, s_warp, &total);
		carry += total;
		const uint32_t start = (uint32_t)start64;       // positions are only used when the total fits 31 bits (checked below)
		if (t < T)
		{
			ranges[t] = c ? make_uint2(start, start + c) : make_uint2(0u, 0u);   // empty tiles stay (0,0) as after the reference's memset (RI:475)
			cursor[t] = 0;
			// tiles too large for the one-CTA-per-tile class are queued for the persistent large-segment kernels
			if (c > GSB_SORT_CAP_A) { const int k = c > GSB_SORT_CAP_B; cls_list[k * T + atomicAdd(&cls_count[k], 1u)] = t; }
		}
	}
	__syncthreads();
	if (tid == 0)
	{
		const bool overflow = carry >= (1ull << 31);
		counters[0] = overflow ? 0xffffffffu : (uint32_t)carry;   // num_rendered; the saturated value also stops every speculative launch
		counters[6] = overflow ? 1u : 0u;
		counters[4] = cls_count[0]; counters[5] = cls_count[1];   // read back with R: the host skips the large-tile launches when both are 0
	}
}

// Per tile: turn the per-CTA histograms into exclusive prefixes over CTAs (in place) and emit the tile total.
// CTA = 32 tiles x 32 row-groups: lanes of a warp read 32 consecutive tiles of one histogram row (128-byte segments), warp g
// owns rows [g*per, (g+1)*per).  The rows of a thread are loaded into registers first (independent loads, all in flight), the
// 32 group totals are combined through shared memory, and the prefixes are written once: one read and one write of the table.
#define PREFIX_GROUPS 32
#define PREFIX_MAXPER 20            // rows per thread: ctas <= 32 * 20 (make_bin_plan caps ctas at 592)
__global__ void __launch_bounds__(1024) tile_prefix_kernel(uint32_t* __restrict__ cta_count, int ctas, int T, uint32_t* __restrict__ tile_count)
{
	__shared__ uint32_t s_part[PREFIX_GROUPS][32];
	const int lane = threadIdx.x & 31, grp = threadIdx.x >> 5;
	const int t = blockIdx.x * 32 + lane;
	const int per = (ctas + PREFIX_GROUPS - 1) / PREFIX_GROUPS, c0 = grp * per;
	uint32_t v[PREFIX_MAXPER];
	uint32_t run = 0;
#pragma unroll
	for (int k = 0; k < PREFIX_MAXPER; k++)
	{
		const int c = c0 + k;
		v[k] = (t < T && k < per && c < ctas) ? cta_count[(size_t)c * T + t] : 0u;
	}
#pragma unroll
	for (int k = 0; k < PREFIX_MAXPER; k++) run += v[k];
	s_part[grp][lane] = run;
	__syncthreads();
	uint32_t off = 0, total = 0;
#pragma unroll
	for (int g = 0; g < PREFIX_GROUPS; g++) { const uint32_t x = s_part[g][lane]; if (g < grp) off += x; total += x; }
	if (t < T)
	{
#pragma unroll
		for (int k = 0; k < PREFIX_MAXPER; k++)
		{
			const int c = c0 + k;
			if (k < per && c < ctas) { cta_count[(size_t)c * T + t] = off; off += v[k]; }
		}
		if (grp == 0) tile_count[t] = total;
	}
}

// The instance stores are 8-byte writes into ~3-entry runs scattered over the whole bucket array: written through to DRAM
// they cost a read-modify-write of a 32-byte sector each.  The array (8 B x R, 96 MB at 3 M Gaussians / 1080p) is written in
// row bands whose slices fit H100's 50 MB L2 (GSB_BAND_BYTES), so the stores carry an evict_last policy (sectors fill up in L2
// and are written back whole, and the per-tile sort that follows reads them from L2), while the one-touch inputs are read with
// the streaming (evict-first) hint.
__device__ __forceinline__ uint64_t l2_policy_evict_last()
{
	uint64_t pol;
	asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
	return pol;
}
__device__ __forceinline__ void st_u64_policy(uint64_t* p, uint64_t v, uint64_t pol)
{
	asm volatile("st.global.L2::cache_hint.b64 [%0], %1, %2;" ::"l"(p), "l"(v), "l"(pol) : "memory");
}

// Row-band launches (bucket array larger than L2): the slice of the bucket array that belongs to the tile rows of one band is
// pre-written with full-sector stores right before that band's scatter (see scatter_prefill).  The slice's bounds are device
// data (`ranges` of the band's first / last non-empty tile), hence a kernel and not a memset.
__global__ void __launch_bounds__(256) band_prefill_kernel(const uint2* __restrict__ ranges, int t0, int t1, uint64_t* __restrict__ bucket,
	const uint32_t* __restrict__ counters, uint32_t cap)
{
	if (counters[0] > cap) return;                   // speculative launch, see scatter_priv_kernel
	__shared__ uint32_t s_lo, s_hi;
	if (threadIdx.x == 0)
	{
		uint32_t lo = 0, hi = 0;
		for (int t = t0; t < t1; t++) { const uint2 r = ranges[t]; if (r.y > r.x) { lo = r.x; break; } }
		for (int t = t1 - 1; t >= t0; t--) { const uint2 r = ranges[t]; if (r.y > r.x) { hi = r.y; break; } }
		s_lo = lo; s_hi = hi;
	}
	__syncthreads();
	const uint32_t lo = (s_lo + 1u) & ~1u, hi = s_hi & ~1u;      // 16-byte aligned interior; the two edge entries are written by the scatter anyway
	if (hi <= lo) return;
	uint4* p = reinterpret_cast<uint4*>(bucket + lo);
	const size_t n16 = (size_t)(hi - lo) / 2;
	for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n16; i += (size_t)gridDim.x * blockDim.x) p[i] = make_uint4(0u, 0u, 0u, 0u);
}

// Scatter with privatised cursors: CTA c (same Gaussian chunk as in the preprocess kernel) starts every tile's cursor at
// tile start + (instances of that tile owned by CTAs < c); slots are then claimed with shared-memory atomics only.
__global__ void __launch_bounds__(1024, 1) scatter_priv_kernel(int P, int chunk, int T, const uint32_t* __restrict__ depth_bits, const uint2* __restrict__ rect,
	const uint2* __restrict__ ranges, const uint32_t* __restrict__ cta_base, int gx, uint32_t y_lo, uint32_t y_hi, uint64_t* __restrict__ bucket,
	const uint32_t* __restrict__ counters, uint32_t cap)
{
	// The launch is speculative: the host sized `bucket` for `cap` instances before the instance count of THIS frame was known
	// (it is still in flight to the host).  More instances than that: do nothing, the host re-launches with a larger blob.
	if (counters[0] > cap) return;
	// One launch handles the tile rows [y_lo, y_hi): when the bucket array is larger than L2 the host splits the image into row
	// bands whose slice of the (tile-major) array fits, so that the scattered 8-byte stores still complete their sectors in L2.
	extern __shared__ uint32_t s_cur[];
	const uint32_t* base = cta_base + (size_t)blockIdx.x * T;
	const int t0 = (int)y_lo * gx, nt = (int)(y_hi - y_lo) * gx;
	for (int t = threadIdx.x; t < nt; t += blockDim.x) s_cur[t] = ranges[t0 + t].x + base[t0 + t];
	__syncthreads();
	const int lane = threadIdx.x & 31;
	const uint64_t pol = l2_policy_evict_last();
	const long long first = (long long)blockIdx.x * chunk, last = min((long long)P, first + chunk);
	// The kernel is latency-bound (long-scoreboard waits on rect -> depth -> store, two DRAM round trips per
	// iteration): the depth bits are loaded together with the rectangle (4 wasted bytes for a culled Gaussian), and the
	// NEXT iteration's pair is requested before this iteration's instances are scattered.
	uint2 rc_n = make_uint2(0, 0); uint32_t db_n = 0;
	if (first + threadIdx.x < last) { rc_n = __ldcs(&rect[first + threadIdx.x]); db_n = __ldcs(&depth_bits[first + threadIdx.x]); }
	for (long long b0 = first; b0 < last; b0 += blockDim.x)
	{
		const long long idx = b0 + threadIdx.x;
		const uint2 rc = rc_n; const uint32_t dbits = db_n;
		{
			const long long nx = idx + blockDim.x;
			rc_n = make_uint2(0, 0); db_n = 0;
			if (nx < last) { rc_n = __ldcs(&rect[nx]); db_n = __ldcs(&depth_bits[nx]); }
		}
		TileRect tr(rc);
		tr.miny = max(tr.miny, y_lo); tr.maxy = min(tr.maxy, y_hi);                          // clipped to this band
		const uint32_t w = tr.width(), t = tr.maxy > tr.miny ? tr.area() : 0u;
		const bool big = t > 32;
		if (t && !big)
		{
			const uint64_t comp = ((uint64_t)dbits << 32) | (uint32_t)idx;
			for (uint32_t y = tr.miny; y < tr.maxy; y++)
				for (uint32_t x = tr.minx; x < tr.maxx; x++) st_u64_policy(&bucket[atomicAdd(&s_cur[(y - y_lo) * gx + x], 1u)], comp, pol);
		}
		unsigned bigmask = __ballot_sync(0xffffffffu, big);
		while (bigmask)
		{
			const int src = __ffs(bigmask) - 1; bigmask &= bigmask - 1;
			const uint32_t bt = __shfl_sync(0xffffffffu, t, src), bw = __shfl_sync(0xffffffffu, w, src);
			const uint32_t bminx = __shfl_sync(0xffffffffu, tr.minx, src), bminy = __shfl_sync(0xffffffffu, tr.miny, src);
			const uint64_t comp = ((uint64_t)__shfl_sync(0xffffffffu, dbits, src) << 32) | (uint32_t)(idx - lane + src);
			for (uint32_t k = lane; k < bt; k += 32)
				st_u64_policy(&bucket[atomicAdd(&s_cur[(bminy - y_lo + k / bw) * gx + bminx + k % bw], 1u)], comp, pol);
		}
	}
}

// ------------------------------------------------------------------------------------------------
// One thread per Gaussian writes its instances; Gaussians covering more than 32 tiles are handled by the whole warp.
__global__ void __launch_bounds__(256) scatter_kernel(int P, const uint32_t* __restrict__ depth_bits, const uint2* __restrict__ rect,
	const uint2* __restrict__ ranges, uint32_t* __restrict__ cursor, int gx, uint64_t* __restrict__ bucket,
	const uint32_t* __restrict__ counters, uint32_t cap)
{
	if (counters[0] > cap) return;                   // speculative launch, see scatter_priv_kernel
	const int idx = blockIdx.x * blockDim.x + threadIdx.x;
	const int lane = threadIdx.x & 31;
	uint2 rc = make_uint2(0, 0); uint32_t dbits = 0;
	if (idx < P)
	{
		rc = rect[idx];
		if (rc.x | rc.y) dbits = depth_bits[idx];
	}
	const TileRect tr(rc);
	const uint32_t w = tr.width(), t = tr.area();
	const bool big = t > 32;
	if (t && !big)
	{
		const uint64_t comp = ((uint64_t)dbits << 32) | (uint32_t)idx;
		for (uint32_t y = tr.miny; y < tr.maxy; y++)
			for (uint32_t x = tr.minx; x < tr.maxx; x++)
			{
				const uint32_t tile = y * gx + x;
				bucket[ranges[tile].x + atomicAdd(&cursor[tile], 1u)] = comp;
			}
	}
	unsigned bigmask = __ballot_sync(0xffffffffu, big);
	while (bigmask)
	{
		const int src = __ffs(bigmask) - 1; bigmask &= bigmask - 1;
		const uint32_t bt = __shfl_sync(0xffffffffu, t, src), bw = __shfl_sync(0xffffffffu, w, src);
		const uint32_t bminx = __shfl_sync(0xffffffffu, tr.minx, src), bminy = __shfl_sync(0xffffffffu, tr.miny, src);
		const uint64_t comp = ((uint64_t)__shfl_sync(0xffffffffu, dbits, src) << 32) | (uint32_t)(idx - lane + src);
		for (uint32_t k = lane; k < bt; k += 32)
		{
			const uint32_t tile = (bminy + k / bw) * gx + bminx + k % bw;
			bucket[ranges[tile].x + atomicAdd(&cursor[tile], 1u)] = comp;
		}
	}
}

// ------------------------------------------------------------------------------------------------
// Per-tile sort in shared memory: stable LSD radix sort of (depth bits, id) pairs on the 32 depth bits, 8 bits per pass.
// Warp w owns positions [w*32*ITEMS, (w+1)*32*ITEMS); ranks inside a warp come from match.any, across warps from a
// per-digit scan of the per-warp counters (the same stable ranking as a onesweep tile, but the whole "array" is the tile).
// Persistent CTAs walk a device-side list of queued tiles: the tiles the distribution sort found too clustered.
template <int CAP, int THREADS>
__global__ void __launch_bounds__(THREADS) tile_sort_kernel(const uint2* __restrict__ ranges, const uint64_t* __restrict__ bucket,
	uint32_t* __restrict__ point_list, const uint32_t* __restrict__ cls_list, const uint32_t* __restrict__ cls_count,
	const uint32_t* __restrict__ counters, uint32_t cap)
{
	if (counters[0] > cap) return;                   // speculative launch, see scatter_priv_kernel
	constexpr int ITEMS = CAP / THREADS, NW = THREADS / 32;
	extern __shared__ __align__(16) unsigned char s_raw[];
	uint32_t* kA = reinterpret_cast<uint32_t*>(s_raw);
	uint32_t* vA = kA + CAP;
	uint32_t* kB = vA + CAP;
	uint32_t* vB = kB + CAP;
	uint32_t* whist = vB + CAP;                 // [NW][256]
	__shared__ uint32_t s_dstart[256];
	__shared__ uint32_t s_wtot[8];
	__shared__ uint32_t s_and, s_or;
	const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
	const unsigned lt = (1u << lane) - 1u;
	const uint32_t n_work = *cls_count;
	for (uint32_t wi = blockIdx.x; wi < n_work; wi += gridDim.x)
	{
		const uint2 r = ranges[cls_list[wi]];
		const uint32_t n = r.y - r.x;
		if (n == 0 || n > (uint32_t)CAP) continue;
		if (n == 1) { if (tid == 0) point_list[r.x] = (uint32_t)bucket[r.x]; continue; }
		if (tid == 0) { s_and = 0xffffffffu; s_or = 0u; }
		__syncthreads();
		uint32_t a_and = 0xffffffffu, a_or = 0u;
		for (uint32_t i = tid; i < n; i += THREADS)
		{
			const uint64_t c = bucket[r.x + i];
			const uint32_t k = (uint32_t)(c >> 32);
			kA[i] = k; vA[i] = (uint32_t)c;
			a_and &= k; a_or |= k;
		}
		a_and = __reduce_and_sync(0xffffffffu, a_and); a_or = __reduce_or_sync(0xffffffffu, a_or);
		if (lane == 0) { atomicAnd(&s_and, a_and); atomicOr(&s_or, a_or); }
		__syncthreads();
		const uint32_t differ = s_and ^ s_or;       // bits in which the tile's keys are not all equal
		uint32_t* ks = kA; uint32_t* vs = vA; uint32_t* kd = kB; uint32_t* vd = vB;
		for (int pass = 0; pass < 4; pass++)
		{
			const int shift = 8 * pass;
			if (((differ >> shift) & 0xffu) == 0) continue;         // every key has the same digit: the pass is the identity
			for (int i = tid; i < NW * 256; i += THREADS) whist[i] = 0;
			__syncthreads();
			uint32_t key[ITEMS], val[ITEMS], rank[ITEMS];
#pragma unroll
			for (int i = 0; i < ITEMS; i++)
			{
				const uint32_t pos = warp * (32 * ITEMS) + i * 32 + lane;
				const bool valid = pos < n;
				key[i] = valid ? ks[pos] : 0u; val[i] = valid ? vs[pos] : 0u;
				const uint32_t d = valid ? (key[i] >> shift) & 0xffu : 256u;
				const unsigned vm = __ballot_sync(0xffffffffu, valid);
				if (vm == 0) { rank[i] = 0; continue; }
				const unsigned m = __match_any_sync(0xffffffffu, d) & vm;
				if (valid)
				{
					const int leader = __ffs(m) - 1;
					uint32_t old = 0;
					if (lane == leader) { old = whist[warp * 256 + d]; whist[warp * 256 + d] = old + __popc(m); }
					old = __shfl_sync(m, old, leader);
					rank[i] = old + __popc(m & lt);
				}
				__syncwarp();
			}
			__syncthreads();
			// digit `tid` (< 256): per-warp exclusive offsets, then an exclusive scan of the digit totals
			uint32_t total = 0;
			if (tid < 256)
			{
#pragma unroll 4
				for (int w = 0; w < NW; w++) { const uint32_t c = whist[w * 256 + tid]; whist[w * 256 + tid] = total; total += c; }
				uint32_t incl = total;
#pragma unroll
				for (int o = 1; o < 32; o <<= 1) { const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += v; }
				if (lane == 31) s_wtot[warp] = incl;
				s_dstart[tid] = incl - total;
			}
			__syncthreads();
			if (tid < 256)
			{
				uint32_t add = 0;
#pragma unroll
				for (int w = 0; w < 8; w++) if (w < warp) add += s_wtot[w];
				s_dstart[tid] += add;
			}
			__syncthreads();
#pragma unroll
			for (int i = 0; i < ITEMS; i++)
			{
				const uint32_t pos = warp * (32 * ITEMS) + i * 32 + lane;
				if (pos < n)
				{
					const uint32_t d = (key[i] >> shift) & 0xffu;
					const uint32_t np = s_dstart[d] + whist[warp * 256 + d] + rank[i];
					kd[np] = key[i]; vd[np] = val[i];
				}
			}
			__syncthreads();
			uint32_t* t0 = ks; ks = kd; kd = t0; t0 = vs; vs = vd; vd = t0;
		}
		// runs of bit-identical depths (rare): ascending Gaussian id, as the reference's stable sort leaves them
		for (uint32_t p = tid; p < n; p += THREADS)
		{
			const uint32_t k = ks[p];
			if ((p == 0 || ks[p - 1] != k) && p + 1 < n && ks[p + 1] == k)
			{
				uint32_t e = p + 1;
				while (e < n && ks[e] == k) e++;
				for (uint32_t i = p + 1; i < e; i++)
				{
					const uint32_t v = vs[i];
					uint32_t j = i;
					while (j > p && vs[j - 1] > v) { vs[j] = vs[j - 1]; j--; }
					vs[j] = v;
				}
			}
		}
		__syncthreads();
		for (uint32_t i = tid; i < n; i += THREADS) point_list[r.x + i] = vs[i];
		__syncthreads();
	}
}

// Fast path for tiles of up to CAP_A instances: ONE-pass distribution sort.  Depth keys inside a tile are spread over a
// narrow range, so binning them by (key - min) >> shift into 2048 order-preserving bins leaves ~1 key per bin; a per-bin
// insertion sort on the full 64-bit composite (depth bits, id) then finishes the total order.  Tiles whose depths cluster
// (some bin > 32 keys) are flagged and handled by the radix kernel below, so the result never depends on the heuristic.
// One template serves both shared-memory classes: THREADS = 256 sorts tiles of up to 2048 instances (one CTA per tile,
// 2048 bins), THREADS = 1024 tiles of up to 8192 instances (persistent CTAs over the queued tile list, 8192 bins).
template <int THREADS>
struct DistSmem {
	static constexpr int CAP = 8 * THREADS, BINS = 8 * THREADS;
	uint64_t out[CAP];                   // entries grouped by bin (unsorted inside a bin)
	uint32_t bin[BINS];                  // counts, then exclusive starts
	uint32_t sorted[CAP];                // the sorted ids, written by rank
	uint32_t wtot[32];
	uint32_t kmin, kmax, big;
};

template <int THREADS>
__device__ __forceinline__ void dist_sort_tile(DistSmem<THREADS>& S, uint32_t tile, const uint2 r, const uint64_t* __restrict__ bucket,
	uint32_t* __restrict__ point_list, uint32_t* __restrict__ fallback_list, uint32_t* __restrict__ fallback_count)
{
	constexpr int BINS = DistSmem<THREADS>::BINS, NW = THREADS / 32;
	constexpr int LOG_BINS = THREADS == 256 ? 11 : 13;
	static_assert(THREADS == 256 || THREADS == 1024, "bin count = 8 * THREADS must be 2^LOG_BINS");
	const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
	const uint32_t n = r.y - r.x;
	if (tid == 0) { S.kmin = 0xffffffffu; S.kmax = 0u; S.big = 0u; }
	for (int i = tid; i < BINS; i += THREADS) S.bin[i] = 0;
	__syncthreads();
	uint64_t c[8];
	uint32_t kmin = 0xffffffffu, kmax = 0u;
#pragma unroll
	for (int i = 0; i < 8; i++)
	{
		const uint32_t p = i * THREADS + tid;
		c[i] = p < n ? bucket[r.x + p] : ~0ull;
		if (p < n) { const uint32_t k = (uint32_t)(c[i] >> 32); kmin = min(kmin, k); kmax = max(kmax, k); }
	}
	kmin = __reduce_min_sync(0xffffffffu, kmin); kmax = __reduce_max_sync(0xffffffffu, kmax);
	if (lane == 0) { atomicMin(&S.kmin, kmin); atomicMax(&S.kmax, kmax); }
	__syncthreads();
	const uint32_t lo = S.kmin, range = S.kmax - lo;
	const int shift = max(0, (32 - __clz(range)) - LOG_BINS);        // (range >> shift) < BINS
	uint32_t slot[8];
	uint32_t worst = 0;
#pragma unroll
	for (int i = 0; i < 8; i++)
	{
		const uint32_t p = i * THREADS + tid;
		if (p < n)
		{
			const uint32_t b = ((uint32_t)(c[i] >> 32) - lo) >> shift;
			const uint32_t q = atomicAdd(&S.bin[b], 1u);
			slot[i] = (b << 16) | q;
			worst = max(worst, q);
		}
	}
	if (__any_sync(0xffffffffu, worst >= 32)) { if (lane == 0) S.big = 1; }
	__syncthreads();
	if (S.big) { if (tid == 0) fallback_list[atomicAdd(fallback_count, 1u)] = tile; return; }   // queued for the radix kernel
	// exclusive scan of the bin counts: thread t owns bins [8t, 8t+8)
	uint32_t cnt[8], local = 0;
#pragma unroll
	for (int i = 0; i < 8; i++) { cnt[i] = S.bin[8 * tid + i]; local += cnt[i]; }
	uint32_t incl = local;
#pragma unroll
	for (int o = 1; o < 32; o <<= 1) { const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += v; }
	if (lane == 31) S.wtot[warp] = incl;
	__syncthreads();
	uint32_t start = incl - local;
#pragma unroll
	for (int w = 0; w < NW; w++) if (w < warp) start += S.wtot[w];
	{
		uint32_t run = start;
#pragma unroll
		for (int i = 0; i < 8; i++) { S.bin[8 * tid + i] = run; run += cnt[i]; }
	}
	__syncthreads();
#pragma unroll
	for (int i = 0; i < 8; i++)
	{
		const uint32_t p = i * THREADS + tid;
		if (p < n) S.out[S.bin[slot[i] >> 16] + (slot[i] & 0xffffu)] = c[i];
	}
	__syncthreads();
	// Finish the bins by RANK, one entry at a time: an entry's final position is its bin's start + the number of bin-mates with a
	// smaller composite (depth bits, then Gaussian id; composites are unique).  The earlier version let each thread insertion-sort
	// the 8 bins it owned: most of the kernel's stalls were the barrier behind that loop (a thread that owns a crowded bin
	// holds up the CTA).  Ranking costs the same comparisons but spreads a crowded bin's work over the threads that hold its
	// entries (entries are dealt round-robin).
#pragma unroll
	for (int i = 0; i < 8; i++)
	{
		const uint32_t p = i * THREADS + tid;
		if (p < n)
		{
			const uint32_t b = slot[i] >> 16;
			const uint32_t bs = S.bin[b], be = (b + 1 < (uint32_t)BINS) ? S.bin[b + 1] : n;
			const uint64_t v = c[i];
			uint32_t rank = 0;
			for (uint32_t k = bs; k < be; k++) rank += S.out[k] < v ? 1u : 0u;
			S.sorted[bs + rank] = (uint32_t)v;
		}
	}
	__syncthreads();
	for (uint32_t i = tid; i < n; i += THREADS) point_list[r.x + i] = S.sorted[i];
}

// LIST == false: one CTA per tile (tiles of 2 .. 8 * THREADS instances; larger ones belong to another class).
// LIST == true: persistent CTAs walk the device-side list of queued tiles.
template <int THREADS, bool LIST>
__global__ void __launch_bounds__(THREADS) tile_sort_dist_kernel(const uint2* __restrict__ ranges, const uint64_t* __restrict__ bucket,
	uint32_t* __restrict__ point_list, const uint32_t* __restrict__ work_list, const uint32_t* __restrict__ work_count,
	uint32_t* __restrict__ fallback_list, uint32_t* __restrict__ fallback_count, const uint32_t* __restrict__ counters, uint32_t cap)
{
	if (counters[0] > cap) return;                   // speculative launch, see scatter_priv_kernel
	extern __shared__ __align__(16) unsigned char s_dist_raw[];
	DistSmem<THREADS>& S = *reinterpret_cast<DistSmem<THREADS>*>(s_dist_raw);
	constexpr uint32_t CAP = DistSmem<THREADS>::CAP;
	if (!LIST)
	{
		const uint32_t tile = blockIdx.x;
		const uint2 r = ranges[tile];
		const uint32_t n = r.y - r.x;
		if (n == 0 || n > CAP) return;
		if (n == 1) { if (threadIdx.x == 0) point_list[r.x] = (uint32_t)bucket[r.x]; return; }
		dist_sort_tile<THREADS>(S, tile, r, bucket, point_list, fallback_list, fallback_count);
	}
	else
	{
		const uint32_t n_work = *work_count;
		for (uint32_t wi = blockIdx.x; wi < n_work; wi += gridDim.x)
		{
			const uint32_t tile = work_list[wi];
			const uint2 r = ranges[tile];
			if (r.y - r.x <= CAP) dist_sort_tile<THREADS>(S, tile, r, bucket, point_list, fallback_list, fallback_count);
			__syncthreads();
		}
	}
}

// Segments beyond the shared-memory classes: single-CTA stable LSD radix sort (8 x 8-bit digits of the 64-bit
// composite) ping-ponging between the bucket and its spare copy in global memory.  Rare (very dense tiles).
__global__ void __launch_bounds__(1024) tile_sort_big_kernel(const uint2* __restrict__ ranges, uint64_t* bucket, uint64_t* alt,
	uint32_t* __restrict__ point_list, const uint32_t* __restrict__ cls_list, const uint32_t* __restrict__ cls_count)
{
	__shared__ uint32_t s_base[256];
	const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
	for (uint32_t wi = blockIdx.x; wi < *cls_count; wi += gridDim.x)
	{
	const uint2 r = ranges[cls_list[wi]];
	const uint32_t n = r.y - r.x;
	uint64_t* src = bucket + r.x;
	uint64_t* dst = alt + r.x;
	__syncthreads();
	for (int pass = 0; pass < 8; pass++)
	{
		const int shift = 8 * pass;
		if (tid < 256) s_base[tid] = 0;
		__syncthreads();
		for (uint32_t i = tid; i < n; i += 1024) atomicAdd(&s_base[(uint32_t)(src[i] >> shift) & 0xff], 1u);
		__syncthreads();
		if (tid == 0) { uint32_t run = 0; for (int d = 0; d < 256; d++) { const uint32_t c = s_base[d]; s_base[d] = run; run += c; } }
		__syncthreads();
		// stable scatter, 1024 elements at a time; warps take turns (ranks inside a warp from match.any)
		for (uint32_t c0 = 0; c0 < n; c0 += 1024)
		{
			const uint32_t i = c0 + tid;
			const bool valid = i < n;
			const uint64_t key = valid ? src[i] : 0ull;
			const uint32_t d = valid ? (uint32_t)(key >> shift) & 0xff : 256u;
			for (int w = 0; w < 32; w++)
			{
				if (warp == w)
				{
					const unsigned vm = __ballot_sync(0xffffffffu, valid);
					const unsigned m = __match_any_sync(0xffffffffu, d) & vm;
					if (valid)
					{
						const int leader = __ffs(m) - 1;
						uint32_t old = 0;
						if (lane == leader) { old = s_base[d]; s_base[d] = old + __popc(m); }
						old = __shfl_sync(m, old, leader);
						dst[old + __popc(m & ((1u << lane) - 1u))] = key;
					}
				}
				__syncthreads();
			}
		}
		__threadfence_block();
		__syncthreads();
		uint64_t* tmp = src; src = dst; dst = tmp;
	}
	// after 8 passes the data is back in `bucket`
	for (uint32_t i = tid; i < n; i += 1024) point_list[r.x + i] = (uint32_t)src[i];
	}
}

// ------------------------------------------------------------------------------------------------
int launch_tile_scan(const ImageState& img, const GeomState& g, const BinPlan& plan, int W, int H, cudaStream_t stream)
{
	const int T = (int)ImageState::tiles(W, H);
	ProfScope prof(K_SCAN, stream);
	if (plan.priv)
	{
		tile_prefix_kernel<<<(T + 31) / 32, 1024, 0, stream>>>(img.cta_count, plan.ctas, T, img.tile_count);
		GSB_LAUNCHED();
	}
	tile_scan_kernel<<<1, 1024, 0, stream>>>(img.tile_count, T, img.ranges, g.counters, img.tile_cursor, img.cls_list, img.cls_count);
	GSB_LAUNCHED();
	GSB_CUDA_OK(cudaGetLastError());
	return GSB_OK;
}

// Scattered 8-byte stores that miss in L2 are partial-sector writes
// // that fill the sector from DRAM first.  The bucket array (or, with several bands, the band's slice of it) is therefore written once
// with full-sector stores right before the scatter, and the scattered stores then hit.  GSB_SCATTER_PREFILL=0 switches it off
// (A/B measurements).
// bucket-array bytes per row band: 40 MB leaves a fifth of the 50 MB L2 to the inputs the scatter streams through it
#define GSB_BAND_BYTES (40ll << 20)
static bool scatter_prefill()
{
	static const bool v = [] { const char* e = getenv("GSB_SCATTER_PREFILL"); return !(e && e[0] == '0'); }();
	return v;
}

// Scatter + the per-tile sort classes that are launched unconditionally.  SPECULATIVE: `cap` is the instance capacity the
// binning blob was carved for; every kernel here compares the device-side instance count with it and exits when it does not
// fit (gsb_forward then repeats the call with the true count).
int launch_scatter_sort(const GeomState& g, const BinningState& b, const ImageState& img, const BinPlan& plan, int P, long long cap, int W, int H,
	cudaStream_t stream)
{
	if (cap <= 0) return GSB_OK;
	const dim3 tiles = tile_grid(W, H);
	const int gx = tiles.x, gy = tiles.y, T = gx * gy;
	const uint32_t cap32 = (uint32_t)std::min<long long>(cap, 0x7fffffffll);
	{
		ProfScope prof(K_SCATTER, stream);
		if (plan.priv)
		{
			if (int e = ensure_dyn_smem((const void*)scatter_priv_kernel, 220 * 1024)) return e;
			// row bands: each band's slice of the bucket array (8 B x its instances, tile-major = contiguous) should fit L2
			const int bands = (int)std::min<long long>(gy, std::max<long long>(1, (cap * 8 + GSB_BAND_BYTES - 1) / GSB_BAND_BYTES));
			const int rows = (gy + bands - 1) / bands;
			for (int y0 = 0; y0 < gy; y0 += rows)
			{
				const int y1 = std::min(gy, y0 + rows);
				if (scatter_prefill())
				{
					if (bands == 1) GSB_CUDA_OK(cudaMemsetAsync(b.bucket, 0, size_t(cap) * 8, stream));
					else { band_prefill_kernel<<<GSB_NUM_SMS * 2, 256, 0, stream>>>(img.ranges, y0 * gx, y1 * gx, b.bucket, g.counters, cap32); GSB_LAUNCHED(); }
				}
				scatter_priv_kernel<<<plan.ctas, plan.threads, size_t(y1 - y0) * gx * sizeof(uint32_t), stream>>>(P, plan.chunk, T, g.dbits, g.rect,
					img.ranges, img.cta_count, gx, (uint32_t)y0, (uint32_t)y1, b.bucket, g.counters, cap32);
				GSB_LAUNCHED();
			}
		}
		else
		{
			scatter_kernel<<<(P + 255) / 256, 256, 0, stream>>>(P, g.dbits, g.rect, img.ranges, img.tile_cursor, gx, b.bucket, g.counters, cap32);
			GSB_LAUNCHED();
		}
	}
	constexpr size_t smemA = size_t(GSB_SORT_CAP_A) * 16 + 8 * 256 * 4;
	if (int e = ensure_dyn_smem((const void*)tile_sort_kernel<GSB_SORT_CAP_A, 256>, (int)smemA)) return e;
	if (int e = ensure_dyn_smem((const void*)tile_sort_dist_kernel<256, false>, (int)sizeof(DistSmem<256>))) return e;
	{
		ProfScope prof(K_TILE_SORT, stream);
		tile_sort_dist_kernel<256, false><<<T, 256, sizeof(DistSmem<256>), stream>>>(img.ranges, b.bucket, b.point_list, nullptr, nullptr,
			img.cls_list + 2 * (size_t)T, img.cls_count + 2, g.counters, cap32);
		GSB_LAUNCHED();
	}
	{
		ProfScope prof(K_SORT_LARGE, stream);
		// radix fallback for the tiles the distribution sort queued (device-side list; normally empty: the CTAs exit at once)
		tile_sort_kernel<GSB_SORT_CAP_A, 256><<<GSB_NUM_SMS * 4, 256, smemA, stream>>>(img.ranges, b.bucket, b.point_list, img.cls_list + 2 * (size_t)T,
			img.cls_count + 2, g.counters, cap32);
		GSB_LAUNCHED();
	}
	GSB_CUDA_OK(cudaGetLastError());
	return GSB_OK;
}

// The two large-tile classes (> GSB_SORT_CAP_A / > GSB_SORT_CAP_B instances): launched after the host has seen the class
// sizes (they ride the instance-count read-back), nothing is launched for an empty class.
int launch_sort_large(const GeomState& g, const BinningState& b, const ImageState& img, int W, int H, uint32_t n_tiles_over_a, uint32_t n_tiles_over_b,
	cudaStream_t stream)
{
	const int T = (int)ImageState::tiles(W, H);
	constexpr size_t smemB = size_t(GSB_SORT_CAP_B) * 16 + 32 * 256 * 4;
	if (n_tiles_over_a)
	{
		// tiles of 2049 .. 8192 instances: the same one-pass distribution sort with 8192 bins on persistent 1024-thread CTAs; a tile
		// whose depths cluster is queued (device-side list, region 3) for the 4-pass shared-memory radix sort that used to take them all
		if (int e = ensure_dyn_smem((const void*)tile_sort_dist_kernel<1024, true>, (int)sizeof(DistSmem<1024>))) return e;
		if (int e = ensure_dyn_smem((const void*)tile_sort_kernel<GSB_SORT_CAP_B, 1024>, (int)smemB)) return e;
		ProfScope prof(K_SORT_LARGE, stream);
		tile_sort_dist_kernel<1024, true><<<GSB_NUM_SMS, 1024, sizeof(DistSmem<1024>), stream>>>(img.ranges, b.bucket, b.point_list, img.cls_list, img.cls_count,
			img.cls_list + 3 * (size_t)T, img.cls_count + 3, g.counters, 0xffffffffu);
		GSB_LAUNCHED();
		tile_sort_kernel<GSB_SORT_CAP_B, 1024><<<GSB_NUM_SMS, 1024, smemB, stream>>>(img.ranges, b.bucket, b.point_list, img.cls_list + 3 * (size_t)T,
			img.cls_count + 3, g.counters, 0xffffffffu);
		GSB_LAUNCHED();
	}
	if (n_tiles_over_b)
	{
		ProfScope prof(K_SORT_LARGE, stream);
		tile_sort_big_kernel<<<GSB_NUM_SMS / 2, 1024, 0, stream>>>(img.ranges, b.bucket, b.alt, b.point_list, img.cls_list + T, img.cls_count + 1);
		GSB_LAUNCHED();
	}
	GSB_CUDA_OK(cudaGetLastError());
	return GSB_OK;
}

// Debug/tooling export in the reference's format: sorted keys (tile << 32 | depth bits) and the sorted id list.
__global__ void export_binning_kernel(int T, const uint2* __restrict__ ranges, const uint32_t* __restrict__ point_list,
	const float4* __restrict__ rec, uint64_t* keys, uint32_t* vals)
{
	const int tile = blockIdx.x;
	if (tile >= T) return;
	const uint2 r = ranges[tile];
	for (uint32_t i = r.x + threadIdx.x; i < r.y; i += blockDim.x)
	{
		const uint32_t id = point_list[i];
		if (keys) keys[i] = ((uint64_t)tile << 32) | __float_as_uint(rec[3 * (size_t)id + 2].z);
		if (vals) vals[i] = id;
	}
}

int launch_export_binning(const GeomState& g, const BinningState& b, const ImageState& img, int W, int H, uint64_t* keys, uint32_t* vals, cudaStream_t stream)
{
	const int T = (int)ImageState::tiles(W, H);
	export_binning_kernel<<<T, 128, 0, stream>>>(T, img.ranges, b.point_list, g.rec, keys, vals);
	GSB_CUDA_OK(cudaGetLastError());
	return GSB_OK;
}

} // namespace gsb
