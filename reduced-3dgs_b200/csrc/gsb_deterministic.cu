// gsb_deterministic.cu — the two small kernels around the deterministic render backward (DESIGN.md §5i).
//
// The R instances have fixed slots, Gaussian-major and then row-major over the Gaussian's tiles (gsb_common.cuh TileRect):
// det_scan_kernel computes each Gaussian's first slot, render_backward_kernel<*, true> stores one partial per instance into its
// slot (the 8 warps of the tile added in warp order), and det_gather_kernel adds each Gaussian's slots in order into the 12-float
// accumulator the preprocess backward reads.  No float atomics anywhere: the same inputs give the same bytes on every run.
#include "gsb_common.cuh"

namespace gsb {

#define DET_SCAN_THREADS 1024
#define DET_SCAN_ITEMS 4                      // Gaussians per thread: 4096 per CTA

// Workspace: [ticket, error flag] | look-back descriptors, one per scan CTA | offset[P] | parts[R * ns] (ns = 10, DET_NS_ABS with absgrad)
struct DetWorkspace {
	uint32_t* head;          // [0] = scan ticket, [1] = error flag (slot total != R)
	uint32_t* lb;            // [scan CTAs] decoupled look-back descriptors (zeroed with head)
	uint32_t* offset;        // [P] first slot of each Gaussian
	float* parts;            // [R][ns] per-instance partials (ns = 10, 9 used without the maps; DET_NS_ABS with absgrad)
	static int scan_ctas(int P) { return (P + DET_SCAN_THREADS * DET_SCAN_ITEMS - 1) / (DET_SCAN_THREADS * DET_SCAN_ITEMS); }
	static DetWorkspace carve(char* blob, int P, long long R, int ns, size_t* bytes = nullptr)
	{
		Carver c(blob); DetWorkspace w;
		w.head = c.take<uint32_t>(64);
		w.lb = c.take<uint32_t>(scan_ctas(P));
		w.offset = c.take<uint32_t>(P);
		w.parts = c.take<float>(size_t(R) * ns);
		if (bytes) *bytes = c.off + 256;
		return w;
	}
	size_t head_bytes() const { return size_t(reinterpret_cast<char*>(offset) - reinterpret_cast<char*>(head)); }
};

size_t det_workspace_bytes(int P, long long R, int ns)
{
	size_t b; DetWorkspace::carve(nullptr, P < 0 ? 0 : P, R < 0 ? 0 : R, ns, &b); return b;
}

// offset = exclusive scan of the TileRect areas; CTAs chain their totals with the decoupled look-back (ticket order).  The CTA
// holding the last Gaussian checks the total against R and raises the error flag on a mismatch.
__global__ void __launch_bounds__(DET_SCAN_THREADS) det_scan_kernel(int P, const uint2* __restrict__ rect, uint32_t* __restrict__ head,
	uint32_t* __restrict__ lb, uint32_t* __restrict__ offset, unsigned long long R)
{
	__shared__ uint32_t s_tile, s_excl, s_warp[DET_SCAN_THREADS / 32];
	const int tid = threadIdx.x;
	if (tid == 0) s_tile = atomicAdd(&head[0], 1u);
	__syncthreads();
	const uint32_t tile = s_tile;
	const long long base = (long long)tile * DET_SCAN_THREADS * DET_SCAN_ITEMS + (long long)tid * DET_SCAN_ITEMS;
	uint32_t a[DET_SCAN_ITEMS], sum = 0;
#pragma unroll
	for (int i = 0; i < DET_SCAN_ITEMS; i++)
	{
		a[i] = base + i < P ? TileRect(rect[base + i]).area() : 0u;
		sum += a[i];
	}
	uint32_t total;
	const uint32_t cta_excl = cta_exclusive<DET_SCAN_THREADS>(sum, s_warp, &total);
	if (tid == 0)
	{
		const uint32_t excl = lookback_exclusive(lb, tile, 1, 0, total);
		s_excl = excl;
		const long long last = (long long)(tile + 1) * DET_SCAN_THREADS * DET_SCAN_ITEMS;
		if (last >= P && (unsigned long long)excl + total != R) atomicExch(&head[1], 1u);
	}
	__syncthreads();
	uint32_t run = s_excl + cta_excl;
#pragma unroll
	for (int i = 0; i < DET_SCAN_ITEMS; i++)
		if (base + i < P) { offset[base + i] = run; run += a[i]; }
}

// 16 threads per Gaussian, thread k writes acc[12 g + k]: the sum of component k over the Gaussian's slots in slot order
// (zero for culled and pruned Gaussians and for components the slot does not carry).  With the error flag set the accumulator is
// filled with NaN, so blobs that do not match R cannot pass for a gradient.
__global__ void __launch_bounds__(256) det_gather_kernel(int P, int ns, const uint2* __restrict__ rect, const uint32_t* __restrict__ offset,
	const float* __restrict__ parts, unsigned long long R, const uint32_t* __restrict__ head, float* __restrict__ acc)
{
	const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
	const long long g = t >> 4;
	const int k = (int)(t & 15);
	if (g >= P) return;
	const uint32_t area = TileRect(rect[g]).area();
	const unsigned long long off = offset[g];
	float s = 0.0f;
	const bool bad = head[1] != 0 || off + area > R;
	if (k < ns && !bad)
	{
		const float* p = parts + off * ns + k;
#pragma unroll 4
		for (uint32_t i = 0; i < area; i++) s += p[(size_t)i * ns];
	}
	if (bad) s = __int_as_float(0x7fffffff);
	if (k < 12) acc[12 * g + k] = s;
}

// scan -> deterministic render backward -> gather: writes all 12 floats of every Gaussian's accumulator.
int launch_render_backward_deterministic(const GsbBackwardRequest& req, const ImageState& img, const BinningState& b, const GeomState& g,
	float* acc)
{
	const int P = req.scene->P; const long long R = req.num_rendered; const cudaStream_t stream = stream_of(req);
	if (R == 0)
	{
		// nothing rendered: every rect is empty and every gradient zero
		GSB_CUDA_OK(cudaMemsetAsync(acc, 0, size_t(P) * 48, stream));
		return GSB_OK;
	}
	const bool abs = req.dL_dmeans2D_abs != nullptr;
	DetWorkspace w = DetWorkspace::carve(req.det_workspace, P, R, abs ? DET_NS_ABS : 10);
	{
		ProfScope prof(K_DET_SCAN, stream);
		GSB_CUDA_OK(cudaMemsetAsync(w.head, 0, w.head_bytes(), stream));
		det_scan_kernel<<<DetWorkspace::scan_ctas(P), DET_SCAN_THREADS, 0, stream>>>(P, g.rect, w.head, w.lb, w.offset,
			(unsigned long long)R);
		GSB_LAUNCHED();
		GSB_CUDA_OK(cudaGetLastError());
	}
	if (int e = launch_render_backward(req, img, b, g, acc, w.parts, w.offset)) return e;
	ProfScope prof(K_DET_GATHER, stream);
	const int ns = abs ? DET_NS_ABS : (req.dL_dinvdepth || req.dL_dalpha) ? 10 : 9;
	det_gather_kernel<<<(unsigned)((16ll * P + 255) / 256), 256, 0, stream>>>(P, ns, g.rect, w.offset, w.parts, (unsigned long long)R, w.head,
		acc);
	GSB_LAUNCHED();
	GSB_CUDA_OK(cudaGetLastError());
	return GSB_OK;
}

} // namespace gsb
