// gsb_tools.cu — the reduced-3dgs tools that sit on either side of the rasterizer (SURVEY.md §8(f) rows 2-3):
//   * SH-culling statistics: per-camera update of the transmittance-weighted colour statistics that decide each
//     Gaussian's SH degree (reference reduced_3dgs.cu:41-203 calculateColourVariance + reduced_3dgs/sh_culling.cu)
//   * resolution-aware redundancy score: pixel footprint of a Gaussian centre over all cameras, sphere / ellipsoid
//     intersection count against the k nearest neighbours, minimum score over intersecting neighbours
//     (reference reduced_3dgs/redundancy_score.cu, reduced_3dgs.cu:205-287)
//
// The reference runs these as ~30 ATen element-wise ops per camera (colour statistics) and one kernel launch + one host
// synchronisation per camera (pixel size); here each is ONE fused pass over the Gaussians, bandwidth-bound.
#include <math_constants.h>
#include "gsb_common.cuh"

namespace gsb {

// ------------------------------------------------------------------------------------------------
// One camera's update of the colour statistics (reduced_3dgs.cu:150-201), one thread per Gaussian.
//   t        = transmittance_sum / max(touched_pixels, 1)                                     :154
//   wSum    += t;  wSumSq += t^2                                                              :155-156
//   colours  = SH colour truncated after band 0, 1, 2, 3 (slot k exists only if k <= degree;
//              slots above the Gaussian's degree stay 0; invisible Gaussians are all 0)       :158-165, sh_culling.cu:6-57
//   dist[d] += t * || colours[3] - colours[d] ||_2   (NaN -> 0)            d = 0, 1, 2         :167-181
//   visible Gaussians: weighted running mean of colours[3]; variance += t * (colour - new mean)^2  :183-200
// The colour table has 4 slots per Gaussian (sh_culling.cu:21 hard-codes the stride), i.e. max_sh_degree = 3.
__global__ void __launch_bounds__(256) sh_stats_update_kernel(int P, int M, const int* __restrict__ degrees,
	const float* __restrict__ means3D, const float* __restrict__ campos, const float* __restrict__ shs,
	const int* __restrict__ radii, const int* __restrict__ touched, const float* __restrict__ tsum,
	float* __restrict__ wSum, float* __restrict__ wSumSq, float* __restrict__ dist_accum,
	float* __restrict__ mean, float* __restrict__ variance)
{
	const int idx = blockIdx.x * blockDim.x + threadIdx.x;
	if (idx >= P) return;
	const int tp = touched[idx];
	const float t = tsum[idx] / (float)max(tp, 1);
	const float ws = wSum[idx] + t;
	wSum[idx] = ws;
	wSumSq[idx] += t * t;
	const bool present = radii[idx] > 0;

	float col[4][3];
#pragma unroll
	for (int k = 0; k < 4; k++) col[k][0] = col[k][1] = col[k][2] = 0.0f;
	if (present)
	{
		const float px = means3D[3 * idx], py = means3D[3 * idx + 1], pz = means3D[3 * idx + 2];
		float dx = px - campos[0], dy = py - campos[1], dz = pz - campos[2];
		const float len = sqrtf(dx * dx + dy * dy + dz * dz);
		dx = dx / len; dy = dy / len; dz = dz / len;
		const float* sh = shs + (size_t)idx * M * 3;
		const int deg = degrees[idx];
		float res[3];
#pragma unroll
		for (int c = 0; c < 3; c++)
		{
			res[c] = kSH_C0 * sh[c] + 0.5f;
			col[0][c] = fmaxf(res[c], 0.0f);
		}
		if (deg > 0)
		{
			const float x = dx, y = dy, z = dz;
#pragma unroll
			for (int c = 0; c < 3; c++)
			{
				res[c] = res[c] - kSH_C1 * y * sh[3 + c] + kSH_C1 * z * sh[6 + c] - kSH_C1 * x * sh[9 + c];
				col[1][c] = fmaxf(res[c], 0.0f);
			}
			if (deg > 1)
			{
				const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
#pragma unroll
				for (int c = 0; c < 3; c++)
				{
					res[c] = res[c] + kSH_C2[0] * xy * sh[12 + c] + kSH_C2[1] * yz * sh[15 + c] + kSH_C2[2] * (2.0f * zz - xx - yy) * sh[18 + c] +
						kSH_C2[3] * xz * sh[21 + c] + kSH_C2[4] * (xx - yy) * sh[24 + c];
					col[2][c] = fmaxf(res[c], 0.0f);
				}
				if (deg > 2)
				{
#pragma unroll
					for (int c = 0; c < 3; c++)
					{
						res[c] = res[c] + kSH_C3[0] * y * (3.0f * xx - yy) * sh[27 + c] + kSH_C3[1] * xy * z * sh[30 + c] +
							kSH_C3[2] * y * (4.0f * zz - xx - yy) * sh[33 + c] + kSH_C3[3] * z * (2.0f * zz - 3.0f * xx - 3.0f * yy) * sh[36 + c] +
							kSH_C3[4] * x * (4.0f * zz - xx - yy) * sh[39 + c] + kSH_C3[5] * z * (xx - yy) * sh[42 + c] +
							kSH_C3[6] * x * (xx - 3.0f * yy) * sh[45 + c];
						col[3][c] = fmaxf(res[c], 0.0f);
					}
				}
			}
		}
	}
#pragma unroll
	for (int d = 0; d < 3; d++)
	{
		const float a = col[3][0] - col[d][0], b = col[3][1] - col[d][1], c = col[3][2] - col[d][2];
		float dist = sqrtf(a * a + b * b + c * c);
		if (isnan(dist)) dist = 0.0f;
		dist_accum[3 * idx + d] += t * dist;
	}
	if (present)
	{
		float coef = t / ws;
		if (isnan(coef)) coef = 0.0f;
#pragma unroll
		for (int c = 0; c < 3; c++)
		{
			const float m_old = mean[3 * idx + c];
			const float m_new = m_old + coef * (col[3][c] - m_old);
			mean[3 * idx + c] = m_new;
			// reduced_3dgs.cu:185 `auto mean_old = mean;` is a handle to the SAME tensor, so after the in-place update of `mean`
			// both factors of the variance term (:196-200) see the new mean
			variance[3 * idx + c] += t * (col[3][c] - m_new) * (col[3][c] - m_new);
		}
	}
}

int launch_sh_stats_update(int P, int M, const int* degrees, const float* means3D, const float* campos, const float* shs,
	const int* radii, const int* touched, const float* tsum, float* wSum, float* wSumSq, float* dist_accum, float* mean,
	float* variance, cudaStream_t stream)
{
	if (P <= 0) return GSB_OK;
	ProfScope prof(K_TOOLS, stream);
	sh_stats_update_kernel<<<(P + 255) / 256, 256, 0, stream>>>(P, M, degrees, means3D, campos, shs, radii, touched, tsum, wSum, wSumSq,
		dist_accum, mean, variance);
	GSB_LAUNCHED();
	GSB_CUDA_OK(cudaGetLastError());
	return GSB_OK;
}

// ------------------------------------------------------------------------------------------------
// Minimum world-space size of one pixel at each Gaussian centre over all cameras (redundancy_score.cu:45-101,
// reduced_3dgs.cu:246-268).  The reference launches one kernel per camera (reading H, W back to the host each time) that
// min-updates pixel_sizes in global memory; here one thread walks all cameras with the running minimum in a register.
// Matrices are the reference's flat 4x4 tensors reinterpreted as column-major glm::mat4 (m[c][r] = flat[4c + r]);
// M * v is evaluated as (M[0] v.x + M[1] v.y) + (M[2] v.z + M[3] v.w) like GLM.
// The float operation order is the reference build's (read off its SASS): per row fma(v.x, m0, v.y*m1) + fma(v.z, m2, m3*v.w).
__device__ __forceinline__ void mat4_mul(const float* __restrict__ m, float vx, float vy, float vz, float (&o)[4])
{
#pragma unroll
	for (int r = 0; r < 4; r++)
		o[r] = __fadd_rn(__fmaf_rn(vx, m[r], __fmul_rn(vy, m[4 + r])), __fmaf_rn(vz, m[8 + r], m[12 + r]));     // v.w == 1
}

__global__ void __launch_bounds__(256) pixel_size_kernel(int P, const float* __restrict__ means3D, int n_cams,
	const float* __restrict__ w2ndc, const float* __restrict__ w2ndc_inv, const int* __restrict__ heights, const int* __restrict__ widths,
	float* __restrict__ pixel_sizes)
{
	extern __shared__ float s_mat[];                       // [n_cams][32]: forward | inverse
	for (int i = threadIdx.x; i < n_cams * 32; i += blockDim.x)
	{
		const int cam = i >> 5, k = i & 31;
		s_mat[i] = k < 16 ? w2ndc[16 * cam + k] : w2ndc_inv[16 * cam + k - 16];
	}
	__syncthreads();
	const int idx = blockIdx.x * blockDim.x + threadIdx.x;
	if (idx >= P) return;
	const float cx = means3D[3 * idx], cy = means3D[3 * idx + 1], cz = means3D[3 * idx + 2];
	float best = 10000.0f;                                  // reduced_3dgs.cu:256 initial value
	for (int cam = 0; cam < n_cams; cam++)
	{
		const float* pm = s_mat + 32 * cam;
		const float* im = pm + 16;
		float ph[4];
		mat4_mul(pm, cx, cy, cz, ph);
		float pw = __fdiv_rn(1.0f, __fadd_rn(ph[3], 0.0000001f));
		const float qx = __fmul_rn(ph[0], pw), qy = __fmul_rn(ph[1], pw), qz = __fmul_rn(ph[2], pw);
		const bool inside = qx <= 1.0f && qy <= 1.0f && qz <= 1.0f && qx >= -1.0f && qy >= -1.0f && qz >= 0.0f;
		if (!inside) continue;
		const int W = widths[cam], H = heights[cam];
		float ex = 0.0f, ey = 0.0f;
		if (W > H) ex = __fdiv_rn(2.0f, (float)W); else ey = __fdiv_rn(2.0f, (float)H);
		float e[4], s[4];
		mat4_mul(im, ex, ey, qz, e);
		pw = __fdiv_rn(1.0f, __fadd_rn(e[3], 0.0000001f));
		const float enx = __fmul_rn(e[0], pw), eny = __fmul_rn(e[1], pw), enz = __fmul_rn(e[2], pw);
		mat4_mul(im, 0.0f, 0.0f, qz, s);
		pw = __fdiv_rn(1.0f, __fadd_rn(s[3], 0.0000001f));
		const float dx = __fmaf_rn(-s[0], pw, enx), dy = __fmaf_rn(-s[1], pw, eny), dz = __fmaf_rn(-s[2], pw, enz);
		const float len = __fsqrt_rn(__fmaf_rn(dz, dz, __fmaf_rn(dx, dx, __fmul_rn(dy, dy))));
		best = fminf(best, len);
	}
	pixel_sizes[idx] = best;
}

int launch_pixel_size(int P, const float* means3D, int n_cams, const float* w2ndc, const float* w2ndc_inv, const int* heights,
	const int* widths, float* pixel_sizes, cudaStream_t stream)
{
	if (P <= 0) return GSB_OK;
	if (n_cams > 1024) { set_error("find_minimum_projected_pixel_size: more than 1024 cameras per call"); return GSB_EINVAL; }
	ProfScope prof(K_TOOLS, stream);
	if (int e = ensure_dyn_smem((const void*)pixel_size_kernel, 1024 * 32 * 4)) return e;
	pixel_size_kernel<<<(P + 255) / 256, 256, (size_t)n_cams * 32 * sizeof(float), stream>>>(P, means3D, n_cams, w2ndc, w2ndc_inv, heights, widths,
		pixel_sizes);
	GSB_LAUNCHED();
	GSB_CUDA_OK(cudaGetLastError());
	return GSB_OK;
}

// ------------------------------------------------------------------------------------------------
// Mip-Splatting's compute_3D_filter (DESIGN.md §5o) in two launches and no host read: the torch loop runs about fifteen [P]-wide ops
// per camera.  Pass 1: one thread per centre walks every camera, staged through shared memory in chunks of F3D_CHUNK (no camera
// limit), keeps the smallest depth z of the cameras that see it (z > 0.2 and the projection inside the screen grown by 15 % on
// each side) and adds its depth to the maximum over the seen centres; block 0 also takes the maximum focal length over all cameras.
// Pass 2: unseen centres take that maximum, and f = (dist / F) * sqrt(0.2).  Both maxima are exact (integer max of the
// non-negative float bits), so the result is the same bytes on every run.
#define F3D_CHUNK 256
#define F3D_CAM 20     // view rows 0..2 as xform_row reads them (m[i], m[4+i], m[8+i], m[12+i]), fx, fy, W/2, H/2, the four screen bounds

__device__ __forceinline__ float f3d_row(const float* __restrict__ d, float x, float y, float z)
{
	float t = __fmul_rn(y, d[1]);
	t = __fmaf_rn(x, d[0], t);
	t = __fmaf_rn(z, d[2], t);
	return __fadd_rn(t, d[3]);
}

__global__ void __launch_bounds__(256) filter_3d_dist_kernel(int P, const float* __restrict__ means3D, int n_cams,
	const float* __restrict__ views, const float* __restrict__ focals, const int* __restrict__ sizes, float* __restrict__ dist,
	unsigned* __restrict__ maxima)
{
	__shared__ float s_cam[F3D_CHUNK * F3D_CAM];
	const int idx = blockIdx.x * blockDim.x + threadIdx.x;
	float x = 0.f, y = 0.f, z = 0.f;
	if (idx < P) { x = means3D[3 * idx]; y = means3D[3 * idx + 1]; z = means3D[3 * idx + 2]; }
	float best = CUDART_INF_F;
	for (int c0 = 0; c0 < n_cams; c0 += F3D_CHUNK)
	{
		const int nc = min(F3D_CHUNK, n_cams - c0);
		__syncthreads();
		for (int c = threadIdx.x; c < nc; c += blockDim.x)
		{
			const float* v = views + 16 * (size_t)(c0 + c);
			float* d = s_cam + F3D_CAM * c;
			for (int i = 0; i < 3; i++) { d[4 * i] = v[i]; d[4 * i + 1] = v[4 + i]; d[4 * i + 2] = v[8 + i]; d[4 * i + 3] = v[12 + i]; }
			const float fx = focals[2 * (c0 + c)], fy = focals[2 * (c0 + c) + 1];
			const int W = sizes[2 * (c0 + c)], H = sizes[2 * (c0 + c) + 1];
			d[12] = fx; d[13] = fy; d[14] = 0.5f * (float)W; d[15] = 0.5f * (float)H;
			// torch compares the fp32 tensor with the Python doubles -0.15 * W and W * 1.15 rounded to fp32
			d[16] = (float)(-0.15 * W); d[17] = (float)(W * 1.15); d[18] = (float)(-0.15 * H); d[19] = (float)(H * 1.15);
			if (blockIdx.x == 0) atomicMax(&maxima[1], __float_as_uint(fx));
		}
		__syncthreads();
		if (idx < P)
			for (int c = 0; c < nc; c++)
			{
				const float* d = s_cam + F3D_CAM * c;
				const float tz = f3d_row(d + 8, x, y, z);
				if (!(tz > 0.2f)) continue;
				const float zc = fmaxf(tz, 0.001f);
				const float u = __fadd_rn(__fmul_rn(__fdiv_rn(f3d_row(d, x, y, z), zc), d[12]), d[14]);
				const float w = __fadd_rn(__fmul_rn(__fdiv_rn(f3d_row(d + 4, x, y, z), zc), d[13]), d[15]);
				if (u >= d[16] && u <= d[17] && w >= d[18] && w <= d[19]) best = fminf(best, tz);
			}
	}
	if (idx < P) dist[idx] = best;
	// seen depths are > 0.2, so their bits order as the values; 0 marks "no seen centre"
	const unsigned m = __reduce_max_sync(0xffffffffu, idx < P && best != CUDART_INF_F ? __float_as_uint(best) : 0u);
	if ((threadIdx.x & 31) == 0 && m) atomicMax(&maxima[0], m);
}

__global__ void __launch_bounds__(256) filter_3d_finish_kernel(int P, const unsigned* __restrict__ maxima, float* __restrict__ filter)
{
	const int idx = blockIdx.x * blockDim.x + threadIdx.x;
	if (idx >= P) return;
	const unsigned seen_max = maxima[0];
	if (seen_max == 0u) { filter[idx] = 0.f; return; }        // no centre seen, or no camera: Mip-Splatting raises here
	float d = filter[idx];
	if (d == CUDART_INF_F) d = __uint_as_float(seen_max);
	// F is the largest focal over ALL cameras, not over those that see the centre (Mip-Splatting's choice, kept)
	filter[idx] = __fmul_rn(__fdiv_rn(d, __uint_as_float(maxima[1])), 0.44721359549995793f);   // fp32(sqrt(0.2))
}

int launch_filter_3d(int P, const float* means3D, int n_cams, const float* views, const float* focals, const int* sizes, float* filter,
	unsigned* maxima, cudaStream_t stream)
{
	if (P <= 0) return GSB_OK;
	ProfScope prof(K_TOOLS, stream);
	GSB_CUDA_OK(cudaMemsetAsync(maxima, 0, 2 * sizeof(unsigned), stream));
	filter_3d_dist_kernel<<<(P + 255) / 256, 256, 0, stream>>>(P, means3D, n_cams, views, focals, sizes, filter, maxima);
	GSB_LAUNCHED();
	GSB_CUDA_OK(cudaGetLastError());
	filter_3d_finish_kernel<<<(P + 255) / 256, 256, 0, stream>>>(P, maxima, filter);
	GSB_LAUNCHED();
	GSB_CUDA_OK(cudaGetLastError());
	return GSB_OK;
}

// ------------------------------------------------------------------------------------------------
// Sphere / ellipsoid intersection against the k nearest neighbours (redundancy_score.cu:119-160 + buildRotationMatrixCUDA
// :186-205, fused: the 3x3 rotation is rebuilt from the quaternion in registers instead of a [P,3,3] tensor round trip).
// Reference quirk kept: the rotation used for neighbour i is the CURRENT Gaussian's (`R[idx]`, :143), not the neighbour's.
// The centre, radius and rotation of one Gaussian, and the test of one neighbour against them; sphere_ellipsoid_kernel and
// redundancy_fused_kernel share them.
struct SphereProbe { float cx, cy, cz, rad, m00, m01, m02, m10, m11, m12, m20, m21, m22; };
// The loads are issued in the order centre, radius, rotation (the caller sets s.rad between the two calls).
__device__ __forceinline__ void sphere_centre(SphereProbe& s, const float* __restrict__ means3D, int idx)
{
	s.cx = means3D[3 * idx]; s.cy = means3D[3 * idx + 1]; s.cz = means3D[3 * idx + 2];
}
__device__ __forceinline__ void sphere_rotation(SphereProbe& s, const float* __restrict__ rotations, int idx)
{
	const float4 q = reinterpret_cast<const float4*>(rotations)[idx];
	const float r = q.x, x = q.y, y = q.z, z = q.w;
	// column-major mat3(c0 | c1 | c2) of redundancy_score.cu:201-204, in the operation order of the reference build (its SASS)
	const float rz = __fmul_rn(r, z), ry = __fmul_rn(r, y), yz = __fmul_rn(y, z), yy = __fmul_rn(y, y), zz = __fmul_rn(z, z);
	s.m00 = __fsub_rn(1.f, __fmul_rn(2.f, __fadd_rn(yy, zz)));
	s.m01 = __fmul_rn(2.f, __fmaf_rn(x, y, rz)); s.m02 = __fmul_rn(2.f, __fmaf_rn(x, z, -ry));
	s.m10 = __fmul_rn(2.f, __fmaf_rn(x, y, -rz)); s.m11 = __fsub_rn(1.f, __fmul_rn(2.f, __fmaf_rn(x, x, zz)));
	s.m12 = __fmul_rn(2.f, __fmaf_rn(r, x, yz));
	s.m20 = __fmul_rn(2.f, __fmaf_rn(x, z, ry)); s.m21 = __fmul_rn(2.f, __fmaf_rn(-r, x, yz));
	s.m22 = __fsub_rn(1.f, __fmul_rn(2.f, __fmaf_rn(x, x, yy)));
}
// true if the centre lies inside neighbour n's ellipsoid with its scales grown by the sphere radius
__device__ __forceinline__ bool sphere_hits(const SphereProbe& s, const float* __restrict__ means3D, const float* __restrict__ scales, int n)
{
	const float dx = __fsub_rn(s.cx, means3D[3 * n]), dy = __fsub_rn(s.cy, means3D[3 * n + 1]), dz = __fsub_rn(s.cz, means3D[3 * n + 2]);
	const float sx = __fadd_rn(scales[3 * n], s.rad), sy = __fadd_rn(scales[3 * n + 1], s.rad), sz = __fadd_rn(scales[3 * n + 2], s.rad);
	// row vector times matrix: component c = dot(column c, d), contracted as fma(d.z, m2, fma(d.x, m0, d.y*m1))
	const float lx = __fmaf_rn(dz, s.m02, __fmaf_rn(dx, s.m00, __fmul_rn(dy, s.m01)));
	const float ly = __fmaf_rn(dz, s.m12, __fmaf_rn(dx, s.m10, __fmul_rn(dy, s.m11)));
	const float lz = __fmaf_rn(dz, s.m22, __fmaf_rn(dx, s.m20, __fmul_rn(dy, s.m21)));
	// glm::pow(v, vec3(2)) is the full powf (the reference build does not reduce it to a product)
	const float bx = __frcp_rn(powf(sx, 2.0f)), by = __frcp_rn(powf(sy, 2.0f)), bz = __frcp_rn(powf(sz, 2.0f));
	const float dot = __fmaf_rn(bz, powf(lz, 2.0f), __fmaf_rn(bx, powf(lx, 2.0f), __fmul_rn(by, powf(ly, 2.0f))));
	return dot < 1.0f;
}

// One thread per Gaussian; the neighbour list row is [knn] int32.
__global__ void __launch_bounds__(256) sphere_ellipsoid_kernel(int P, const float* __restrict__ means3D, const float* __restrict__ scales,
	const float* __restrict__ rotations, const int* __restrict__ neighbours, const float* __restrict__ sphere_radius, int knn,
	int* __restrict__ redundancy_values, uint8_t* __restrict__ intersection_mask)
{
	const int idx = blockIdx.x * blockDim.x + threadIdx.x;
	if (idx >= P) return;
	SphereProbe s;
	sphere_centre(s, means3D, idx);
	s.rad = sphere_radius[idx];
	sphere_rotation(s, rotations, idx);
	const int* nb = neighbours + (size_t)idx * knn;
	uint8_t* mk = intersection_mask + (size_t)idx * knn;
	int count = 0;
	for (int i = 0; i < knn; i++)
	{
		const bool hit = sphere_hits(s, means3D, scales, nb[i]);
		mk[i] = hit ? 1 : 0;
		count += hit ? 1 : 0;
	}
	redundancy_values[idx] = count;
}

int launch_sphere_ellipsoid(int P, const float* means3D, const float* scales, const float* rotations, const int* neighbours,
	const float* sphere_radius, int knn, int* redundancy_values, uint8_t* intersection_mask, cudaStream_t stream)
{
	if (P <= 0) return GSB_OK;
	ProfScope prof(K_TOOLS, stream);
	sphere_ellipsoid_kernel<<<(P + 255) / 256, 256, 0, stream>>>(P, means3D, scales, rotations, neighbours, sphere_radius, knn,
		redundancy_values, intersection_mask);
	GSB_LAUNCHED();
	GSB_CUDA_OK(cudaGetLastError());
	return GSB_OK;
}

// ------------------------------------------------------------------------------------------------
// minimum_redundancy[n] = min over Gaussians i that intersect neighbour n of redundancy[i] (redundancy_score.cu:6-27);
// initial value P (reduced_3dgs.cu:279).  Integer atomicMin: the result does not depend on the order.
__global__ void __launch_bounds__(256) fill_int_kernel(int n, int v, int* __restrict__ out)
{
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i < n) out[i] = v;
}
__global__ void __launch_bounds__(256) min_redundancy_kernel(int P, const int* __restrict__ redundancy_values, const int* __restrict__ neighbours,
	const uint8_t* __restrict__ intersection_mask, int knn, int* __restrict__ minimum)
{
	const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;   // one thread per (Gaussian, neighbour slot): coalesced
	if (e >= (long long)P * knn) return;
	if (intersection_mask[e]) atomicMin(&minimum[neighbours[e]], redundancy_values[e / knn]);
}

int launch_min_redundancy(int P, const int* redundancy_values, const int* neighbours, const uint8_t* intersection_mask, int knn,
	int* minimum, cudaStream_t stream)
{
	if (P <= 0) return GSB_OK;
	ProfScope prof(K_TOOLS, stream);
	fill_int_kernel<<<(P + 255) / 256, 256, 0, stream>>>(P, P, minimum);
	GSB_LAUNCHED();
	const long long E = (long long)P * knn;
	if (E > 0)
	{
		min_redundancy_kernel<<<(unsigned)((E + 255) / 256), 256, 0, stream>>>(P, redundancy_values, neighbours, intersection_mask, knn, minimum);
		GSB_LAUNCHED();
	}
	GSB_CUDA_OK(cudaGetLastError());
	return GSB_OK;
}

// ------------------------------------------------------------------------------------------------
// The whole of Scene.calculate_redundancy_metric after the kNN (scene/__init__.py:153-173) in one pass, one thread per Gaussian i:
//   radius  = ((cube_size[i] * pixel_scale) * sqrt(3)) / 2        torch's fp32 order (division by 2 is exact)
//   hits    = the neighbours k whose grown ellipsoid contains centre i (sphere_hits); slots holding -1 (missing) are skipped
//   red_i   = |hits| + 1                                           the "+1" for the Gaussian itself
//   minimum[i]   = min(minimum[i], red_i)                          the self column the reference concatenates
//   minimum[n_k] = min(minimum[n_k], red_i) for each hit k         allocate_minimum_redundancy_value
// `minimum` is filled with P before.  Integer minima do not depend on the order, so the result is deterministic.  The hit bits
// stay in a register: no [P, K] mask and no [P, K + 1] copies.
__global__ void __launch_bounds__(256) redundancy_fused_kernel(int P, const float* __restrict__ means3D, const float* __restrict__ scales,
	const float* __restrict__ rotations, const int* __restrict__ neighbours, const float* __restrict__ cube_size, float pixel_scale, int knn,
	int* __restrict__ minimum)
{
	const int idx = blockIdx.x * blockDim.x + threadIdx.x;
	if (idx >= P) return;
	SphereProbe s;
	sphere_centre(s, means3D, idx);
	s.rad = __fdiv_rn(__fmul_rn(__fmul_rn(cube_size[idx], pixel_scale), __fsqrt_rn(3.0f)), 2.0f);
	sphere_rotation(s, rotations, idx);
	const int* nb = neighbours + (size_t)idx * knn;
	unsigned long long hits = 0;
	for (int i = 0; i < knn; i++)
	{
		const int n = nb[i];
		if (n >= 0 && sphere_hits(s, means3D, scales, n)) hits |= 1ull << i;
	}
	const int red = __popcll(hits) + 1;
	atomicMin(&minimum[idx], red);
	while (hits)
	{
		const int i = __ffsll((long long)hits) - 1;
		hits &= hits - 1;
		atomicMin(&minimum[nb[i]], red);
	}
}

int launch_redundancy_fused(int P, const float* means3D, const float* scales, const float* rotations, const int* neighbours,
	const float* cube_size, float pixel_scale, int knn, int* minimum, cudaStream_t stream)
{
	if (P <= 0) return GSB_OK;
	ProfScope prof(K_TOOLS, stream);
	fill_int_kernel<<<(P + 255) / 256, 256, 0, stream>>>(P, P, minimum);
	GSB_LAUNCHED();
	redundancy_fused_kernel<<<(P + 255) / 256, 256, 0, stream>>>(P, means3D, scales, rotations, neighbours, cube_size, pixel_scale, knn, minimum);
	GSB_LAUNCHED();
	GSB_CUDA_OK(cudaGetLastError());
	return GSB_OK;
}

} // namespace gsb
