"""GPU probe: does the device's powf(x, 2.0f) equal x * x for every finite fp32 x?

The sphere / ellipsoid test of the redundancy score (gsb_tools.cu sphere_hits) squares with powf(v, 2.0f), as the reference's
glm::pow does; the CPU oracle (oracle/gs_oracle.cpp gso_sphere_ellipsoid) squares with the host libm.  If the two agree on every
input, the oracle's hit decisions are the kernel's bit for bit and the tests need no borderline allowance near dot = 1.

One launch walks all 2^32 bit patterns (compiled with csrc/build.py's NVCC_FLAGS, so powf lowers as it does in the library) and
counts the finite x where the bits of powf(x, 2.0f) and x * x differ, with the largest distance in ulp, how many of them have a
normal (or infinite) x * x, the largest such |x|, how far from a rounding midpoint the exact square of such an x with a
normal finite x * x can lie, and a few such x.

    python tools/probe_powf_square.py
"""
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "reduced-3dgs_b200", "csrc"))
import build  # noqa: E402

SRC = r"""
#include <cstdio>
#include <cstdint>
#include <cstring>
#define SHOW 16
__device__ unsigned long long g_count, g_finite, g_normal;
__device__ unsigned g_maxulp, g_maxabs, g_maxmid, g_shown, g_show[SHOW][3];

__device__ __forceinline__ int ordered(unsigned b) { return (b & 0x80000000u) ? -(int)(b & 0x7fffffffu) : (int)b; }

__global__ void probe()
{
	unsigned long long bad = 0, fin = 0, normal = 0;
	unsigned maxulp = 0, maxabs = 0, maxmid = 0;
	for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < (1ull << 32);
	     i += (unsigned long long)gridDim.x * blockDim.x)
	{
		const unsigned b = (unsigned)i;
		const float x = __uint_as_float(b);
		if (!isfinite(x)) continue;
		fin++;
		const float p = powf(x, 2.0f), s = __fmul_rn(x, x);
		const unsigned pb = __float_as_uint(p), sb = __float_as_uint(s);
		if (pb == sb) continue;
		bad++;
		if (!(fabsf(s) < 1.17549435e-38f)) normal++;          // x * x is a normal number or infinite
		if (fabsf(s) >= 1.17549435e-38f && !isinf(s))
		{
			// how far the exact square lies from the rounding midpoint between x * x and its neighbour, in ulp of that gap
			const double sq = (double)x * (double)x, r = (double)s;
			const double gap = fabs((double)nextafterf(s, sq > r ? INFINITY : -INFINITY) - r);
			maxmid = max(maxmid, __float_as_uint((float)(0.5 - fabs(sq - r) / gap)));
		}
		maxabs = max(maxabs, b & 0x7fffffffu);
		const long long d = (long long)ordered(pb) - (long long)ordered(sb);
		const unsigned u = (unsigned)min(d < 0 ? -d : d, 0xffffffffll);
		maxulp = max(maxulp, u);
		if (*(volatile unsigned*)&g_shown < SHOW)
		{
			const unsigned k = atomicAdd(&g_shown, 1u);
			if (k < SHOW) { g_show[k][0] = b; g_show[k][1] = pb; g_show[k][2] = sb; }
		}
	}
	atomicAdd(&g_count, bad);
	atomicAdd(&g_finite, fin);
	atomicAdd(&g_normal, normal);
	atomicMax(&g_maxulp, maxulp);
	atomicMax(&g_maxabs, maxabs);
	atomicMax(&g_maxmid, maxmid);
}

int main()
{
	probe<<<132 * 16, 256>>>();
	cudaError_t e = cudaDeviceSynchronize();
	if (e != cudaSuccess) { printf("CUDA error: %s\n", cudaGetErrorString(e)); return 1; }
	unsigned long long count = 0, finite = 0, normal = 0;
	unsigned maxulp = 0, maxabs = 0, maxmid = 0, shown = 0, show[SHOW][3];
	cudaMemcpyFromSymbol(&count, g_count, sizeof(count));
	cudaMemcpyFromSymbol(&shown, g_shown, sizeof(shown));
	cudaMemcpyFromSymbol(&finite, g_finite, sizeof(finite));
	cudaMemcpyFromSymbol(&maxulp, g_maxulp, sizeof(maxulp));
	cudaMemcpyFromSymbol(&maxabs, g_maxabs, sizeof(maxabs));
	cudaMemcpyFromSymbol(&normal, g_normal, sizeof(normal));
	cudaMemcpyFromSymbol(&maxmid, g_maxmid, sizeof(maxmid));
	cudaMemcpyFromSymbol(show, g_show, sizeof(show));
	printf("finite inputs: %llu\n", finite);
	printf("powf(x, 2.0f) != x * x: %llu\n", count);
	printf("largest distance: %u ulp\n", maxulp);
	printf("of them with x * x normal or infinite: %llu\n", normal);
	float xm;
	memcpy(&xm, &maxabs, 4);
	printf("largest |x| among them: %.9g (0x%08x)\n", xm, maxabs);
	float mm;
	memcpy(&mm, &maxmid, 4);
	printf("with x * x normal and finite, the exact square lies at most %.9g ulp from a rounding midpoint\n", mm);
	for (unsigned k = 0; k < shown && k < SHOW; k++)
	{
		float x, p, s;
		memcpy(&x, &show[k][0], 4); memcpy(&p, &show[k][1], 4); memcpy(&s, &show[k][2], 4);
		printf("  x = %.9g (0x%08x): powf %.9g (0x%08x), x * x %.9g (0x%08x)\n", x, show[k][0], p, show[k][1], s, show[k][2]);
	}
	return 0;
}
"""


def main():
    with tempfile.TemporaryDirectory() as tmp:
        src, exe = os.path.join(tmp, "probe_powf_square.cu"), os.path.join(tmp, "probe_powf_square")
        with open(src, "w") as f:
            f.write(SRC)
        subprocess.run([build.nvcc(), src, "-o", exe] + build.NVCC_FLAGS, check=True)
        out = subprocess.run([exe], check=True, capture_output=True, text=True).stdout
    print(out, end="")
    return 0


if __name__ == "__main__":
    sys.exit(main())
