// gsb_adam.cu — one Adam step over the model's parameter tensors (gsb_adam_step, gs_b200.optim.GaussianAdam; DESIGN.md §5f).
//
// torch.optim.Adam's default CUDA path makes seven elementwise passes per step (lerp_, mul_, addcmul_, sqrt, div_, add_,
// addcdiv_: ~72 B per element).  Here one persistent grid-stride launch streams every tensor of the step once: read p, g, m, v,
// write p, m, v (28 B per updated element).  The tensor table travels as a __grid_constant__ kernel parameter.
//
// Arithmetic: each of torch's seven passes rounds its result to fp32, and tools/probe_torch_adam.py established on an H100 which
// of them torch's build contracts into FMA and that its division by a scalar is an IEEE division; adam_update() spells those
// roundings out with __f*_rn intrinsics so that no contraction choice of this compiler can change them.
//
// Work unit: up to 4 consecutive elements of one tensor.  When param, grad and both moments share their 16-byte alignment, a
// tensor is [head: the 0..3 elements before the first aligned address][aligned 16-byte chunks][tail]; the chunks take one 128-bit
// load / store per array.  Otherwise (offset views of different alignment) every unit is four scalar accesses.
// Sparse modes: an element's row and column come from its flat index; a unit whose elements are all skipped reads only the
// visibility / degree words; a partly active unit touches only its active elements, with scalar accesses.
#include <atomic>
#include "gsb_common.cuh"

namespace gsb {

#define ADAM_THREADS 256
#define ADAM_CTAS_PER_SM 4

struct AdamTable {
	GsbAdamTensor t[GSB_ADAM_MAX_TENSORS];
	long long unit_end[GSB_ADAM_MAX_TENSORS];   // inclusive prefix of the tensors' unit counts
	double inv_width[GSB_ADAM_MAX_TENSORS];     // 1 / row_width (sparse modes: row of a flat index without a 64-bit division)
	int head[GSB_ADAM_MAX_TENSORS];             // elements before the first 16-byte aligned chunk; -1 = no 128-bit path
	int n;
};

// torch 2.11 _multi_tensor_adam, non-capturable branch, one element (each line is one of its foreach passes):
//   _foreach_lerp_(m, g, w)        ATen Lerp.h: |w| < 0.5 ? m + w*(g - m) : g - (g - m)*(1 - w)   contracted to one FMA
//   _foreach_mul_(v, beta2)
//   _foreach_addcmul_(v, g, g, c)  v + c*(g*g)                                                    contracted: fma(c, g*g, v)
//   _foreach_sqrt / _foreach_div_(., bc2_sqrt) / _foreach_add_(., eps)                            IEEE sqrt, IEEE division
//   _foreach_addcdiv_(p, m, d, s)  p + s*(m/d)                                                    contracted: fma(s, m/d, p)
__device__ __forceinline__ void adam_update(float& p, float g, float& m, float& v, const GsbAdamTensor& k)
{
	const float w = k.one_minus_beta1, diff = __fsub_rn(g, m);
	m = fabsf(w) < 0.5f ? __fmaf_rn(w, diff, m) : __fmaf_rn(-diff, __fsub_rn(1.0f, w), g);
	v = __fmaf_rn(k.one_minus_beta2, __fmul_rn(g, g), __fmul_rn(v, k.beta2));
	const float d = __fadd_rn(__fdiv_rn(__fsqrt_rn(v), k.bc2_sqrt), k.eps);
	p = __fmaf_rn(k.step_size, __fdiv_rn(m, d), p);
}

template <bool VIS, bool DEG>
__global__ void __launch_bounds__(ADAM_THREADS, ADAM_CTAS_PER_SM) adam_step_kernel(const __grid_constant__ AdamTable tab,
	const uint8_t* __restrict__ visibility, const int32_t* __restrict__ degrees)
{
	const long long total = tab.unit_end[tab.n - 1], stride = (long long)gridDim.x * ADAM_THREADS;
	int t = 0;
	for (long long u = (long long)blockIdx.x * ADAM_THREADS + threadIdx.x; u < total; u += stride)
	{
		while (u >= tab.unit_end[t]) t++;                       // u only grows: the tensor index only moves forward
		const GsbAdamTensor& k = tab.t[t];
		const long long lu = u - (t ? tab.unit_end[t - 1] : 0);
		const int h = tab.head[t];
		long long e0;
		int cnt;
		if (h > 0 && lu == 0) { e0 = 0; cnt = h; }
		else
		{
			e0 = (h > 0 ? h : 0) + 4 * (lu - (h > 0 ? 1 : 0));
			cnt = (int)min(4ll, k.numel - e0);
		}
		unsigned mask = (1u << cnt) - 1u;
		const bool banded = DEG && k.sh_offset >= 0;
		if (VIS || banded)
		{
			long long r;
			int c;
			row_col(e0, k.row_width, tab.inv_width[t], r, c);
			unsigned on = 0;
#pragma unroll
			for (int i = 0; i < 4; i++)
			{
				if (i < cnt)
				{
					bool a = true;
					if (VIS) a = visibility[r] != 0;
					if (banded && a)
					{
						const int d = min(max(degrees[r], 0), 3);
						a = k.sh_offset + c / 3 < (d + 1) * (d + 1);
					}
					on |= (a ? 1u : 0u) << i;
					if (++c == k.row_width) { c = 0; r++; }
				}
			}
			mask = on;
			if (mask == 0u) continue;
		}
		if (h >= 0 && mask == 0xFu)                              // a full chunk: only the body's chunks can be full
		{
			float4* pp = reinterpret_cast<float4*>(k.param + e0);
			float4* mp = reinterpret_cast<float4*>(k.exp_avg + e0);
			float4* vp = reinterpret_cast<float4*>(k.exp_avg_sq + e0);
			float4 p = __ldcs(pp), m = __ldcs(mp), v = __ldcs(vp);
			const float4 g = __ldcs(reinterpret_cast<const float4*>(k.grad + e0));
			adam_update(p.x, g.x, m.x, v.x, k);
			adam_update(p.y, g.y, m.y, v.y, k);
			adam_update(p.z, g.z, m.z, v.z, k);
			adam_update(p.w, g.w, m.w, v.w, k);
			__stcs(pp, p); __stcs(mp, m); __stcs(vp, v);
		}
		else
		{
#pragma unroll
			for (int i = 0; i < 4; i++)
			{
				if ((mask >> i) & 1u)
				{
					const long long e = e0 + i;
					float p = __ldcs(k.param + e), m = __ldcs(k.exp_avg + e), v = __ldcs(k.exp_avg_sq + e);
					adam_update(p, __ldcs(k.grad + e), m, v, k);
					__stcs(k.param + e, p); __stcs(k.exp_avg + e, m); __stcs(k.exp_avg_sq + e, v);
				}
			}
		}
	}
}

// SM count per device, read once (the grid is persistent: a few CTAs per SM, grid-striding over every unit).
static int sm_count()
{
	static std::atomic<int> cached[64];
	int dev = 0;
	if (cudaGetDevice(&dev) != cudaSuccess) return GSB_NUM_SMS;
	if (dev < 0 || dev >= 64) return GSB_NUM_SMS;
	if (cached[dev] == 0)
	{
		int n = 0;
		if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = GSB_NUM_SMS;
		cached[dev] = n;                                          // idempotent: concurrent first calls store the same value
	}
	return cached[dev];
}

} // namespace gsb

using namespace gsb;

extern "C" int gsb_adam_step(const GsbAdamTensor* tensors, int32_t n, int32_t P, const uint8_t* visibility, const int32_t* degrees,
	void* stream)
{
	if (n < 0 || n > GSB_ADAM_MAX_TENSORS) { set_error("adam_step: n = %d is outside 0..%d", n, GSB_ADAM_MAX_TENSORS); return GSB_EINVAL; }
	if (n > 0 && !tensors) { set_error("adam_step: tensor table is NULL"); return GSB_EINVAL; }
	if (P < 0) { set_error("adam_step: P < 0"); return GSB_EINVAL; }
	const bool sparse = visibility || degrees;
	AdamTable tab{};
	tab.n = n;
	long long total = 0;
	for (int i = 0; i < n; i++)
	{
		const GsbAdamTensor& k = tensors[i];
		if (k.numel < 0) { set_error("adam_step: tensor %d: numel < 0", i); return GSB_EINVAL; }
		if (k.numel > 0 && (!k.param || !k.grad || !k.exp_avg || !k.exp_avg_sq))
		{ set_error("adam_step: tensor %d: NULL param / grad / exp_avg / exp_avg_sq", i); return GSB_EINVAL; }
		if (k.sh_offset < -1) { set_error("adam_step: tensor %d: sh_offset %d < -1", i, k.sh_offset); return GSB_EINVAL; }
		if (k.sh_offset >= 0 && (k.row_width <= 0 || k.row_width % 3 != 0))
		{ set_error("adam_step: tensor %d: an SH tensor (sh_offset %d) needs a row width that is a positive multiple of 3, got %d", i,
			k.sh_offset, k.row_width); return GSB_EINVAL; }
		if (sparse && (k.row_width <= 0 || k.numel != (long long)P * k.row_width))
		{ set_error("adam_step: tensor %d: %lld elements is not P = %d rows of %d", i, (long long)k.numel, P, k.row_width); return GSB_EINVAL; }
		const uintptr_t a = reinterpret_cast<uintptr_t>(k.param);
		if (k.numel > 0 && ((a | reinterpret_cast<uintptr_t>(k.grad) | reinterpret_cast<uintptr_t>(k.exp_avg) |
			reinterpret_cast<uintptr_t>(k.exp_avg_sq)) & 3u))
		{ set_error("adam_step: tensor %d: a pointer is not 4-byte aligned", i); return GSB_EINVAL; }
		const bool same = ((a ^ reinterpret_cast<uintptr_t>(k.grad)) & 15u) == 0 && ((a ^ reinterpret_cast<uintptr_t>(k.exp_avg)) & 15u) == 0 &&
			((a ^ reinterpret_cast<uintptr_t>(k.exp_avg_sq)) & 15u) == 0;
		long long units;
		if (same)
		{
			const long long lead = (long long)(((16u - (a & 15u)) & 15u) / 4u), h = lead < k.numel ? lead : k.numel;
			tab.head[i] = (int)h;
			units = (h > 0 ? 1 : 0) + (k.numel - h + 3) / 4;
		}
		else
		{
			tab.head[i] = -1;
			units = (k.numel + 3) / 4;
		}
		total += units;
		tab.t[i] = k;
		tab.unit_end[i] = total;
		tab.inv_width[i] = k.row_width > 0 ? 1.0 / k.row_width : 0.0;
	}
	if (total == 0) return GSB_OK;
	const long long want = (total + ADAM_THREADS - 1) / ADAM_THREADS;
	const long long cap = (long long)sm_count() * ADAM_CTAS_PER_SM;
	const int grid = (int)(want < cap ? want : cap);
	const cudaStream_t st = (cudaStream_t)stream;
	ProfScope prof(K_TOOLS, st);
	if (visibility && degrees) adam_step_kernel<true, true><<<grid, ADAM_THREADS, 0, st>>>(tab, visibility, degrees);
	else if (visibility) adam_step_kernel<true, false><<<grid, ADAM_THREADS, 0, st>>>(tab, visibility, nullptr);
	else if (degrees) adam_step_kernel<false, true><<<grid, ADAM_THREADS, 0, st>>>(tab, nullptr, degrees);
	else adam_step_kernel<false, false><<<grid, ADAM_THREADS, 0, st>>>(tab, nullptr, nullptr);
	GSB_LAUNCHED();
	GSB_CUDA_OK(cudaGetLastError());
	return GSB_OK;
}
