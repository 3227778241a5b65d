// gsb_backward.cu — per-Gaussian backward of the preprocess stage (sm_90a).
//
// One fused kernel replaces reference backward.cu:177-307 computeCov2DCUDA + backward.cu:380-434 preprocessCUDA
// (with :20-172 computeColorFromSH and :311-374 computeCov3D), the nonZeroMask/cub::DeviceReduce/cudaMalloc/D2H
// sequence of rasterizer_impl.cu:549-571 (the visible count was produced by the forward preprocess), and the nine
// torch::zeros of rasterize_points.cu:259-267: every output element is written exactly once (zeros for culled
// Gaussians and inactive SH bands), so the caller allocates with torch.empty and nothing is memset.  The Gaussian's inputs are
// read and activated here, not through the forward's GaussianReader: the scale / rotation chain below is contractible fp32, and
// its FMA contraction (so its bits) follows how the activated values reach it.
// Gradients are fp32 and tolerance-compared (the reference's atomicAdd order makes its own bits non-deterministic).
#include "gsb_common.cuh"

namespace gsb {

struct BwdArgs {
	SceneArgs s;              // M: with raw parameters 1 + C, or 0 without SH
	float lambda;
	const int32_t* radii;
	GeomState g; const float* acc;
	GsbGrads out;
	float* cam_rows;          // CAM: one row of GSB_CAM_SLOTS partial sums per CTA (the caller's workspace)
	// IN_RAW: out.dL_dscales / dL_drotations receive the gradients of _scaling / _rotation, dL_ddc / dL_drest those of the SH rows
	// (either may be NULL: not written); raw_vec4: every SH pointer is 16-byte aligned
	float* dL_ddc; float* dL_drest; int raw_vec4;
	// 16-byte alignment of the caller's SH pointers (a contiguous view may start at any float): shs for the M == 16 staging, dL_dsh
	// (an accumulate_into tensor) for its write-back; the scalar loops take the others.  Rotations are read as one float4: the
	// Python layer hands over 16-byte aligned rows (lib.aligned16)
	int sh_vec4, dsh_vec4;
};

// Camera gradient slots (CAM): 0..11 view[4r+c] (r = 0..3, c = 0..2) at 3r+c; 12..23 proj[4r+j] (j = 0, 1, 3) at 12+3r+{0,1,2};
// 24..26 campos.  view[3,7,11,15] and proj[2,6,10,14] have no slot: the preprocess never reads them.
#define GSB_CAM_SLOTS 27
#define GSB_CAM_ROW 32

// ACC (view-batch accumulation): the sums are formed by the L2 with fire-and-forget reductions (RED.ADD, no value returns to
// the SM): a load-add-store in the kernel serialises one DRAM round trip per output element behind the previous store.
// One kernel per view runs at a time on the stream, so every
// element receives exactly one addition per view, in view order: the result is deterministic.  Adding zero is skipped — culled
// Gaussians and inactive SH bands are most of the rows; the overwrite mode stores them (every element written once, no memset).
template <bool ACC> __device__ __forceinline__ void put(float* p, float v) { if (ACC) { if (v != 0.0f) atomicAdd(p, v); } else *p = v; }

// Coalesced store of one small per-Gaussian output ([P,WD]) for the 32 Gaussians of a warp: lanes park their WD values in
// shared memory, then the warp writes the 32*WD contiguous floats with unit-stride stores.
template <int WD, bool ACC>
__device__ __forceinline__ void warp_store(float* __restrict__ dst, long long base, int n_valid, const float* v, float* tmp, int lane)
{
#pragma unroll
	for (int k = 0; k < WD; k++) tmp[lane * WD + k] = v[k];
	__syncwarp();
#pragma unroll
	for (int i = 0; i < WD; i++)
	{
		const int f = i * 32 + lane;
		if (f < n_valid * WD) put<ACC>(dst + base * WD + f, tmp[f]);
	}
	__syncwarp();
}

// backward.cu:250-255: dL/dSigma (the 6 entries of the symmetric 3D covariance) from dL/d(a, b, c) of the 2D covariance
// (a, b, c) = (T0 Sigma T0, T0 Sigma T1, T1 Sigma T1), T0 / T1 the rows of T = W J
__device__ __forceinline__ void cov2d_to_cov3d_grad(const float* T0, const float* T1, float dL_da, float dL_db, float dL_dc, float* dcov)
{
	dcov[0] = (T0[0] * T0[0] * dL_da + T0[0] * T1[0] * dL_db + T1[0] * T1[0] * dL_dc);
	dcov[3] = (T0[1] * T0[1] * dL_da + T0[1] * T1[1] * dL_db + T1[1] * T1[1] * dL_dc);
	dcov[5] = (T0[2] * T0[2] * dL_da + T0[2] * T1[2] * dL_db + T1[2] * T1[2] * dL_dc);
	dcov[1] = 2 * T0[0] * T0[1] * dL_da + (T0[0] * T1[1] + T0[1] * T1[0]) * dL_db + 2 * T1[0] * T1[1] * dL_dc;
	dcov[2] = 2 * T0[0] * T0[2] * dL_da + (T0[0] * T1[2] + T0[2] * T1[0]) * dL_db + 2 * T1[0] * T1[2] * dL_dc;
	dcov[4] = 2 * T0[2] * T0[1] * dL_da + (T0[1] * T1[2] + T0[2] * T1[1]) * dL_db + 2 * T1[1] * T1[2] * dL_dc;
}

// RAW: moves the warp's SH rows between the padded shared-memory rows (row r: coefficient 0 in columns 0..2, coefficients 1..C in
// columns 3..3C+2) and the two tensors, whose 32-row blocks are contiguous: [base, base + n) rows of _features_dc (3 floats each)
// and of _features_rest (3C floats each).  STORE = false stages the values; STORE = true writes the gradients (zeros when !have)
// to dL_ddc / dL_drest, whichever is non-NULL, adding them in accumulate mode.  Full warps of 16-byte aligned tensors move float4.
template <bool STORE, bool ACC>
__device__ __forceinline__ void raw_block(const float* src, float* dst, int width, int col0, long long base, int n_valid, float* s_row,
	int RS, int lane, bool have, bool vec4)
{
	if (vec4 && n_valid == 32)
	{
		const int n4 = 8 * width;                                        // 32 rows * width floats / 4
		for (int i = lane; i < n4; i += 32)
		{
			const int f = 4 * i;
			int row = f / width, col = f - row * width;
			if (!STORE)
			{
				const float4 v = reinterpret_cast<const float4*>(src + base * width)[i];
				const float e[4] = { v.x, v.y, v.z, v.w };
#pragma unroll
				for (int j = 0; j < 4; j++)
				{
					s_row[row * RS + col0 + col] = e[j];
					if (++col == width) { col = 0; row++; }
				}
			}
			else
			{
				float e[4];
#pragma unroll
				for (int j = 0; j < 4; j++)
				{
					e[j] = have ? s_row[row * RS + col0 + col] : 0.f;
					if (++col == width) { col = 0; row++; }
				}
				float* p = dst + base * width + f;
				if (ACC)
				{
					if (e[0] != 0.f || e[1] != 0.f || e[2] != 0.f || e[3] != 0.f) red_add_v4(p, e[0], e[1], e[2], e[3]);
				}
				else *reinterpret_cast<float4*>(p) = make_float4(e[0], e[1], e[2], e[3]);
			}
		}
		return;
	}
	int row = 0, col = lane;
	while (col >= width) { col -= width; row++; }
	for (int f = lane; f < n_valid * width; f += 32)
	{
		if (!STORE) s_row[row * RS + col0 + col] = src[base * width + f];
		else put<ACC>(dst + base * width + f, have ? s_row[row * RS + col0 + col] : 0.f);
		col += 32;
		while (col >= width) { col -= width; row++; }
	}
}

// One warp per 32 consecutive Gaussians (lane = Gaussian).  The SH rows of the warp (32 x 3M floats, contiguous in HBM) are
// staged through shared memory with unit-stride loads, overwritten in place by the SH gradients and written back with
// unit-stride stores; the seven small outputs go through warp_store.  Every output element is written exactly once.
// MAPS: the render backward also left sum alpha*T*dL/dinvdepth in accumulator slot 9; invdepth = 1/tz adds -slot9/tz^2 to dL/dtz.
// CAM: also the gradient w.r.t. the camera (DESIGN.md §5d).  Each visible Gaussian keeps the 16 intermediates the camera chain
// needs (dL/dt, dL/dT, J, the projection terms, the SH direction term of dmean); after the write-back the warp forms the 27 products
// one at a time and reduces each with an xor butterfly (every lane ends with the same bits), and lane k adds slot k to its running
// sum.  At the end the CTA sums its 8 warps in warp order into its row of a.cam_rows: no atomics, the same bytes on every run.
// AA: the forward scaled the opacity by s(cov2D) (DESIGN.md §5e); dL/do^ (accumulator slot 3) also reaches the cov2D through s,
// before dcov and dL/dT are formed, and from there the 3D covariance, the means through J and, with CAM, the camera.
// RAW (IN == IN_RAW, DESIGN.md §5h): the inputs are the model's leaf parameters.  Their activations are recomputed exactly as the
// forward applied them, and the gradients are chained back through them in torch's CUDA roundings: dL/d_scaling = dL/ds * s
// (ExpBackward0), dL/d_rotation = autograd's F.normalize chain (tools/probe_torch_activations.py), the SH gradient row split
// into its dc and rest parts.  A warp's 32 dc rows (96 floats) and 32 rest rows (96 C floats) are each contiguous and a multiple
// of 16 bytes: they are staged into the padded rows and written back with 128-bit accesses.
// F3D (Mip-Splatting's 3D filter, DESIGN.md §5o): the scales are filtered again as the forward filtered them (filter_3d), the
// covariance chain runs on the filtered scales s', and a row with f != 0 then maps the scale gradient g (w.r.t. mod * s') back to s,
// g s / s' + dL/do^ a sigmoid dc3/ds, and takes dL/dlogit = dL/do^ a c3 sigmoid (1 - sigmoid), with the sigmoid of the logit
// (not o^ / c3, which is 0 / 0 on a flat splat).  A row with f == 0 keeps the unfiltered arithmetic.
template <int IN, bool ACC, bool MAPS, bool CAM, bool AA, bool F3D>
__global__ void __launch_bounds__(256) preprocess_backward_kernel(const BwdArgs a)
{
	constexpr bool QUANT = IN == IN_QUANT, RAW = IN == IN_RAW;
	extern __shared__ float s_dyn[];
	float* s_cb = s_dyn;                                                  // QUANT: [20][256]
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	const int RL = 3 * a.s.M, RS = RL + 1;                                  // row length / padded stride (conflict-free per-lane rows)
	float* s_row = s_dyn + (QUANT ? GSB_NUM_CODEBOOKS * GSB_CODEBOOK_SIZE : 0) + warp * (32 * RS + 32 * 6);
	float* s_tmp = s_row + 32 * RS;
	if (QUANT) stage_codebooks(a.s.q.centers, s_cb);
	// rasterizer_impl.cu:549-571: sh_sparsity_multiplier = lambda / (n_visible * 15 * 3)
	const float mult = a.lambda != 0.0f ? a.lambda / (float)((int)a.g.counters[1] * 15 * 3) : 0.0f;
	// colours given by the caller (override_color): the SH coefficients were not used by the forward, their gradient is zero
	const bool have_sh = RAW ? (a.s.sh_dc != nullptr && a.s.colors_precomp == nullptr)
	                         : ((QUANT || a.s.shs != nullptr) && a.out.dL_dsh != nullptr && a.s.colors_precomp == nullptr);
	const bool have_scales = QUANT || a.s.scales != nullptr;
	float cam_sum = 0.f;                                                  // CAM: this warp's running sum of slot `lane`
	for (long long base = ((long long)blockIdx.x * 8 + warp) * 32; base < a.s.P; base += (long long)gridDim.x * 8 * 32)
	{
		const long long idx = base + lane;
		const int n_valid = (int)min((long long)32, a.s.P - base);
		const bool valid = lane < n_valid;
		const bool vis = valid && a.radii[idx] > 0;
		// ---- stage the warp's SH rows -------------------------------------------------------------
		if (RAW)
		{
			if (have_sh)
			{
				raw_block<false, ACC>(a.s.sh_dc, nullptr, 3, 0, base, n_valid, s_row, RS, lane, true, a.raw_vec4);
				if (a.s.n_rest) raw_block<false, ACC>(a.s.sh_rest, nullptr, 3 * a.s.n_rest, 3, base, n_valid, s_row, RS, lane, true, a.raw_vec4);
			}
		}
		else if (have_sh && !QUANT && RL == 48 && n_valid == 32 && a.sh_vec4)
		{
			// M == 16 fast path: 12 independent 128-bit loads per lane (6 KB contiguous per warp), then scatter to padded rows
			const float4* src4 = reinterpret_cast<const float4*>(a.s.shs + base * 48);
			float4 v[12];
#pragma unroll
			for (int i = 0; i < 12; i++) v[i] = src4[i * 32 + lane];
#pragma unroll
			for (int i = 0; i < 12; i++)
			{
				const int f = (i * 32 + lane) * 4, row = f / 48, col = f - row * 48;
				float* d = s_row + row * RS + col;
				d[0] = v[i].x; d[1] = v[i].y; d[2] = v[i].z; d[3] = v[i].w;
			}
		}
		else if (have_sh && !QUANT)
		{
			const float* src = a.s.shs + base * RL;
			int row = 0, col = lane;
			while (col >= RL) { col -= RL; row++; }
			for (int f = lane; f < n_valid * RL; f += 32)
			{
				s_row[row * RS + col] = src[f];
				col += 32;
				while (col >= RL) { col -= RL; row++; }
			}
		}
		__syncwarp();
		float o_m2[3] = { 0, 0, 0 }, o_col[3] = { 0, 0, 0 }, o_m3[3] = { 0, 0, 0 }, o_cov[6] = { 0, 0, 0, 0, 0, 0 };
		float o_sc[3] = { 0, 0, 0 }, o_rot[4] = { 0, 0, 0, 0 }, o_con[4] = { 0, 0, 0, 0 }, o_op[1] = { 0 };
		float* myrow = s_row + lane * RS;
		// every per-Gaussian input is requested before the visibility flag is known (the flag is itself a load): radius -> accumulator
		// -> position -> ids used to be a chain of DRAM round trips; a culled Gaussian now costs ~90 wasted bytes
		float4 acc0 = make_float4(0.f, 0.f, 0.f, 0.f), acc1 = acc0; float cyy = 0.f, dinvd = 0.f, mx = 0.f, my = 0.f, mz = 0.f, opac = 0.f;
		float sc[3] = { 0, 0, 0 }, qr = 1, qx = 0, qy = 0, qz = 0;
		uint32_t isb[3] = { 0, 0, 0 }, irw = 0; int deg_in = 0; unsigned cl_in = 0;
		float f3d = 0.f, logit = 0.f; uint32_t iop = 0;
		if (valid)
		{
			if (F3D)
			{
				f3d = a.s.filter_3D[idx];
				if (QUANT) iop = a.s.q.ids_opacity[idx]; else logit = a.s.opacities[idx];
			}
			acc0 = reinterpret_cast<const float4*>(a.acc)[3 * idx];
			acc1 = reinterpret_cast<const float4*>(a.acc)[3 * idx + 1];
			if (MAPS) { const float2 c = reinterpret_cast<const float2*>(a.acc)[6 * idx + 4]; cyy = c.x; dinvd = c.y; }
			else cyy = a.acc[12 * idx + 8];
			mx = a.s.means3D[3 * idx]; my = a.s.means3D[3 * idx + 1]; mz = a.s.means3D[3 * idx + 2];
			opac = a.g.rec[3 * idx + 1].z;
			if (QUANT)
			{
				const uint8_t* is = a.s.q.ids_scaling + 3 * idx;
				isb[0] = is[0]; isb[1] = is[1]; isb[2] = is[2];
				irw = reinterpret_cast<const uint32_t*>(a.s.q.ids_rot)[idx];
			}
			else if (!a.s.cov3D_precomp)
			{
				for (int k = 0; k < 3; k++) sc[k] = a.s.scales[3 * idx + k];
				const float4 q = reinterpret_cast<const float4*>(a.s.rotations)[idx];
				qr = q.x; qx = q.y; qy = q.z; qz = q.w;
			}
			if (have_sh) { deg_in = a.s.degrees[idx]; cl_in = a.g.clamped[idx]; }
		}
		// CAM intermediates (zero for culled / invalid lanes): dL/dt, dL/dT0[r], dL/dT1[r], (J00, J02, J11, J12), projection
		// (g2x*m_w, g2y*m_w, -(g2x*mul1 + g2y*mul2)), SH direction term of dmean
		float cg_dt[3] = { 0, 0, 0 }, cg_T0[3] = { 0, 0, 0 }, cg_T1[3] = { 0, 0, 0 }, cg_J[4] = { 0, 0, 0, 0 }, cg_p[3] = { 0, 0, 0 };
		float cg_dir[3] = { 0, 0, 0 };
		if (!vis)
		{
			if (have_sh) for (int k = 0; k < RL; k++) myrow[k] = 0.f;
		}
		else
		{
			// constant factors of backward.cu:498-499, 583-589 applied once per Gaussian
			const float g2x = acc1.x * (0.5f * a.s.W), g2y = acc1.y * (0.5f * a.s.H);
			const float dconx = -0.5f * acc1.z, dcony = -0.5f * acc1.w, dconz = -0.5f * cyy;
			float cov3D[6];
			// F3D: s_act keeps the activated scales, sc becomes the filtered s' the covariance was built from
			float s_act[3] = { 0, 0, 0 }, c3 = 1.f; Filter3DSquares f3sq;
			const float sig = F3D ? sigmoid_ref(QUANT ? quant_value(s_cb, CB_OPACITY, iop) : logit) : 0.f;   // F3D: the logit's sigmoid
			auto filter = [&] {
				if constexpr (F3D)
				{
					for (int k = 0; k < 3; k++) s_act[k] = sc[k];
					c3 = filter_3d(sc[0], sc[1], sc[2], f3d, &f3sq);
				}
			};
			if (QUANT)
			{
				for (int k = 0; k < 3; k++) sc[k] = quant_value(s_cb, CB_SCALING, isb[k]);
				quant_rotation(s_cb, irw, qr, qx, qy, qz);
				filter();
				compute_cov3D(sc[0], sc[1], sc[2], a.s.mod, qr, qx, qy, qz, cov3D);
			}
			else if (RAW)
			{
				normalize_quat(qr, qx, qy, qz);
				for (int k = 0; k < 3; k++) sc[k] = exp_ref(sc[k]);
				filter();
				compute_cov3D(sc[0], sc[1], sc[2], a.s.mod, qr, qx, qy, qz, cov3D);      // bit-identical to the forward's
			}
			else if (a.s.cov3D_precomp) { for (int k = 0; k < 6; k++) cov3D[k] = a.s.cov3D_precomp[6 * idx + k]; }
			else
			{
				filter();
				compute_cov3D(sc[0], sc[1], sc[2], a.s.mod, qr, qx, qy, qz, cov3D);   // the forward computed exactly this; recomputing is bit-identical
			}
			float dmean[3], dcov[6];
			float aa_s = 1.f, aa_q = 0.f;                                     // AA: the forward's opacity factor s and ratio q
			// AA: s and the clamp decision are the forward's own bits: q is formed again from the same inputs with the forward's
			// operation order (compute_cov2D_undilated, aa_det_ratio), not from the cov2D products below, whose association differs
			// (on a needle-thin splat det0 cancels, and an unfused CPU emulation of those products moves s by up to 11 %).  Formed here,
			// ahead of the cov2D chain; only q and s are kept (CAM + AA, IN = 0, ACC = false still spills 16 bytes, DESIGN.md §5e).
			if constexpr (AA)
			{
				const float* v = a.s.view;
				const float3 u = compute_cov2D_undilated(xform_row(v, 0, mx, my, mz), xform_row(v, 1, mx, my, mz), xform_row(v, 2, mx, my, mz),
					a.s.focal_x, a.s.focal_y, a.s.tan_fovx, a.s.tan_fovy, cov3D, v);
				const float3 d1 = dilate_cov2D(u);
				aa_q = aa_det_ratio(u, __fmaf_rn(d1.x, d1.z, -__fmul_rn(d1.y, d1.y)));
				aa_s = __fsqrt_rn(fmaxf(GSB_AA_MIN_RATIO, aa_q));
			}
			// ---------------- computeCov2DCUDA, backward.cu:177-307 ----------------
			{
				const float* v = a.s.view;
				float tx = v[0] * mx + v[4] * my + v[8] * mz + v[12];
				float ty = v[1] * mx + v[5] * my + v[9] * mz + v[13];
				const float tz = v[2] * mx + v[6] * my + v[10] * mz + v[14];
				const float limx = 1.3f * a.s.tan_fovx, limy = 1.3f * a.s.tan_fovy;
				const float txtz = tx / tz, tytz = ty / tz;
				tx = fminf(limx, fmaxf(-limx, txtz)) * tz;
				ty = fminf(limy, fmaxf(-limy, tytz)) * tz;
				const float x_grad_mul = (txtz < -limx || txtz > limx) ? 0.f : 1.f;
				const float y_grad_mul = (tytz < -limy || tytz > limy) ? 0.f : 1.f;
				const float h_x = a.s.focal_x, h_y = a.s.focal_y;
				const float J00 = h_x / tz, J02 = -(h_x * tx) / (tz * tz), J11 = h_y / tz, J12 = -(h_y * ty) / (tz * tz);
				// T = W*J (column-major): T[0][r] = W[0][r]*J00 + W[2][r]*J02 ; T[1][r] = W[1][r]*J11 + W[2][r]*J12 ; W[k][r] = view[4r+k]
				float T0[3], T1[3];
				for (int r = 0; r < 3; r++) { T0[r] = v[4 * r] * J00 + v[4 * r + 2] * J02; T1[r] = v[4 * r + 1] * J11 + v[4 * r + 2] * J12; }
				const float V[3][3] = { { cov3D[0], cov3D[1], cov3D[2] }, { cov3D[1], cov3D[3], cov3D[4] }, { cov3D[2], cov3D[4], cov3D[5] } };
				float TV0[3], TV1[3];      // (T[0] . V[c]), (T[1] . V[c])
				for (int c = 0; c < 3; c++) { TV0[c] = T0[0] * V[c][0] + T0[1] * V[c][1] + T0[2] * V[c][2]; TV1[c] = T1[0] * V[c][0] + T1[1] * V[c][1] + T1[2] * V[c][2]; }
				const float ca = TV0[0] * T0[0] + TV0[1] * T0[1] + TV0[2] * T0[2] + 0.3f;
				const float cb = TV1[0] * T0[0] + TV1[1] * T0[1] + TV1[2] * T0[2];
				const float cc = TV1[0] * T1[0] + TV1[1] * T1[1] + TV1[2] * T1[2] + 0.3f;
				const float denom = ca * cc - cb * cb;
				float dL_da = 0, dL_db = 0, dL_dc = 0;
				const float denom2inv = 1.0f / ((denom * denom) + 0.0000001f);
				if (denom2inv != 0)
				{
					dL_da = denom2inv * (-cc * cc * dconx + 2 * cb * cc * dcony + (denom - ca * cc) * dconz);
					dL_dc = denom2inv * (-ca * ca * dconz + 2 * ca * cb * dcony + (denom - ca * cc) * dconx);
					dL_db = denom2inv * 2 * (cb * cc * dconx - (denom + 2 * cb * cb) * dcony + ca * cb * dconz);
					cov2d_to_cov3d_grad(T0, T1, dL_da, dL_db, dL_dc, dcov);
				}
				else { for (int i = 0; i < 6; i++) dcov[i] = 0; }
				// AA:  o^ = sigmoid * s, s = sqrt(q),
				// q = det0 / det1, clamped below at 2.5e-5 (no gradient through q there).  With h = 0.3 and (a, b, c) the UNDILATED
				// cov2D (b the single off-diagonal parameter): dq/da = h (c^2 + h c + b^2) / det1^2, dq/dc = h (a^2 + h a + b^2) / det1^2,
				// dq/db = -2 b h (a + c + h) / det1^2, and dL/dq = dL/do^ * sigmoid / (2 s) with sigmoid = o^ / s.  The terms are added
				// whether or not the conic branch above was taken, and dcov (linear in dL/da, dL/db, dL/dc) is formed again from the sums.
				// s and the clamp decision (aa_s, aa_q) were taken above from the forward's arithmetic.
				if constexpr (AA)
				{
					const float ua = TV0[0] * T0[0] + TV0[1] * T0[1] + TV0[2] * T0[2];
					const float uc = TV1[0] * T1[0] + TV1[1] * T1[1] + TV1[2] * T1[2];
					if (aa_q > GSB_AA_MIN_RATIO)
					{
						const float k = acc0.w * (opac / aa_s) * 0.3f / (2.f * aa_s * denom * denom);
						dL_da += k * (uc * uc + 0.3f * uc + cb * cb);
						dL_dc += k * (ua * ua + 0.3f * ua + cb * cb);
						dL_db -= 2.f * cb * k * (ua + uc + 0.3f);
					}
					cov2d_to_cov3d_grad(T0, T1, dL_da, dL_db, dL_dc, dcov);
				}
				const float dL_dT00 = 2 * TV0[0] * dL_da + TV1[0] * dL_db, dL_dT01 = 2 * TV0[1] * dL_da + TV1[1] * dL_db, dL_dT02 = 2 * TV0[2] * dL_da + TV1[2] * dL_db;
				const float dL_dT10 = 2 * TV1[0] * dL_dc + TV0[0] * dL_db, dL_dT11 = 2 * TV1[1] * dL_dc + TV0[1] * dL_db, dL_dT12 = 2 * TV1[2] * dL_dc + TV0[2] * dL_db;
				// W[c][r] = view[4r + c]
				const float dL_dJ00 = v[0] * dL_dT00 + v[4] * dL_dT01 + v[8] * dL_dT02;
				const float dL_dJ02 = v[2] * dL_dT00 + v[6] * dL_dT01 + v[10] * dL_dT02;
				const float dL_dJ11 = v[1] * dL_dT10 + v[5] * dL_dT11 + v[9] * dL_dT12;
				const float dL_dJ12 = v[2] * dL_dT10 + v[6] * dL_dT11 + v[10] * dL_dT12;
				const float itz = 1.f / tz, tz2 = itz * itz, tz3 = tz2 * itz;
				const float dL_dtx = x_grad_mul * -h_x * tz2 * dL_dJ02;
				const float dL_dty = y_grad_mul * -h_y * tz2 * dL_dJ12;
				float dL_dtz = -h_x * tz2 * dL_dJ00 - h_y * tz2 * dL_dJ11 + (2 * h_x * tx) * tz3 * dL_dJ02 + (2 * h_y * ty) * tz3 * dL_dJ12;
				if (MAPS) dL_dtz -= dinvd * tz2;                                          // d(1/tz)/dtz = -1/tz^2
				dmean[0] = v[0] * dL_dtx + v[1] * dL_dty + v[2] * dL_dtz;                // transformVec4x3Transpose
				dmean[1] = v[4] * dL_dtx + v[5] * dL_dty + v[6] * dL_dtz;
				dmean[2] = v[8] * dL_dtx + v[9] * dL_dty + v[10] * dL_dtz;
				if (CAM)
				{
					cg_dt[0] = dL_dtx; cg_dt[1] = dL_dty; cg_dt[2] = dL_dtz;
					cg_T0[0] = dL_dT00; cg_T0[1] = dL_dT01; cg_T0[2] = dL_dT02; cg_T1[0] = dL_dT10; cg_T1[1] = dL_dT11; cg_T1[2] = dL_dT12;
					cg_J[0] = J00; cg_J[1] = J02; cg_J[2] = J11; cg_J[3] = J12;
				}
			}
			// ---------------- preprocessCUDA, backward.cu:406-423 ----------------
			{
				const float* p = a.s.proj;
				const float m_hw = p[3] * mx + p[7] * my + p[11] * mz + p[15];
				const float m_w = 1.0f / (m_hw + 0.0000001f);
				const float mul1 = (p[0] * mx + p[4] * my + p[8] * mz + p[12]) * m_w * m_w;
				const float mul2 = (p[1] * mx + p[5] * my + p[9] * mz + p[13]) * m_w * m_w;
				dmean[0] += (p[0] * m_w - p[3] * mul1) * g2x + (p[1] * m_w - p[3] * mul2) * g2y;
				dmean[1] += (p[4] * m_w - p[7] * mul1) * g2x + (p[5] * m_w - p[7] * mul2) * g2y;
				dmean[2] += (p[8] * m_w - p[11] * mul1) * g2x + (p[9] * m_w - p[11] * mul2) * g2y;
				if (CAM) { cg_p[0] = g2x * m_w; cg_p[1] = g2y * m_w; cg_p[2] = -(g2x * mul1 + g2y * mul2); }
			}
			// ---------------- SH backward, backward.cu:20-172 ----------------
			if (have_sh)
			{
				const int deg = deg_in;
				const uint8_t* idc = QUANT ? a.s.q.ids_dc + 3 * idx : nullptr;
				const uint8_t* irest = QUANT ? a.s.q.ids_rest + 45 * idx : nullptr;
				auto sh = [&](int k, int c) -> float {
					if (QUANT) return quant_sh(s_cb, s_cb[idc[c]], irest, k, c);
					return myrow[3 * k + c];
				};
				const float dox = mx - a.s.campos[0], doy = my - a.s.campos[1], doz = mz - a.s.campos[2];
				const float len = sqrtf(dox * dox + doy * doy + doz * doz);
				const float x = dox / len, y = doy / len, z = doz / len;
				const unsigned cl = cl_in;
				const float dRGB[3] = { (cl & 1u) ? 0.f : acc0.x, (cl & 2u) ? 0.f : acc0.y, (cl & 4u) ? 0.f : acc0.z };
				// gradient of coefficient k (in place over the staged value; the sparsity term needs the value's sign first)
				auto wr = [&](int k, float w) {
#pragma unroll
					for (int c = 0; c < 3; c++)
					{
						float g = w * dRGB[c];
						if (mult != 0.f && k > 0) { const float sv = sh(k, c); g += mult * (float)((0.f < sv) - (sv < 0.f)); }
						myrow[3 * k + c] = g;
					}
				};
				float dRx[3] = { 0, 0, 0 }, dRy[3] = { 0, 0, 0 }, dRz[3] = { 0, 0, 0 };
				if (deg > 0)
				{
					for (int c = 0; c < 3; c++) { dRx[c] = -kSH_C1 * sh(3, c); dRy[c] = -kSH_C1 * sh(1, c); dRz[c] = kSH_C1 * sh(2, c); }
					wr(1, -kSH_C1 * y); wr(2, kSH_C1 * z); wr(3, -kSH_C1 * x);
					if (deg > 1)
					{
						const float C20 = kSH_C2[0], C21 = kSH_C2[1], C22 = kSH_C2[2], C23 = kSH_C2[3], C24 = kSH_C2[4];
						const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
						for (int c = 0; c < 3; c++)
						{
							const float s4 = sh(4, c), s5 = sh(5, c), s6 = sh(6, c), s7 = sh(7, c), s8 = sh(8, c);
							dRx[c] += C20 * y * s4 + C22 * 2.f * -x * s6 + C23 * z * s7 + C24 * 2.f * x * s8;
							dRy[c] += C20 * x * s4 + C21 * z * s5 + C22 * 2.f * -y * s6 + C24 * 2.f * -y * s8;
							dRz[c] += C21 * y * s5 + C22 * 2.f * 2.f * z * s6 + C23 * x * s7;
						}
						wr(4, C20 * xy); wr(5, C21 * yz); wr(6, C22 * (2.f * zz - xx - yy)); wr(7, C23 * xz); wr(8, C24 * (xx - yy));
						if (deg > 2)
						{
							const float C30 = kSH_C3[0], C31 = kSH_C3[1], C32 = kSH_C3[2], C33 = kSH_C3[3], C34 = kSH_C3[4], C35 = kSH_C3[5],
								C36 = kSH_C3[6];
							for (int c = 0; c < 3; c++)
							{
								const float s9 = sh(9, c), s10 = sh(10, c), s11 = sh(11, c), s12 = sh(12, c), s13 = sh(13, c), s14 = sh(14, c), s15 = sh(15, c);
								dRx[c] += (C30 * s9 * 3.f * 2.f * xy + C31 * s10 * yz + C32 * s11 * -2.f * xy + C33 * s12 * -3.f * 2.f * xz +
									C34 * s13 * (-3.f * xx + 4.f * zz - yy) + C35 * s14 * 2.f * xz + C36 * s15 * 3.f * (xx - yy));
								dRy[c] += (C30 * s9 * 3.f * (xx - yy) + C31 * s10 * xz + C32 * s11 * (-3.f * yy + 4.f * zz - xx) + C33 * s12 * -3.f * 2.f * yz +
									C34 * s13 * -2.f * xy + C35 * s14 * -2.f * yz + C36 * s15 * -3.f * 2.f * xy);
								dRz[c] += (C31 * s10 * xy + C32 * s11 * 4.f * 2.f * yz + C33 * s12 * 3.f * (2.f * zz - xx - yy) + C34 * s13 * 4.f * 2.f * xz +
									C35 * s14 * (xx - yy));
							}
							wr(9, C30 * y * (3.f * xx - yy)); wr(10, C31 * xy * z); wr(11, C32 * y * (4.f * zz - xx - yy));
							wr(12, C33 * z * (2.f * zz - 3.f * xx - 3.f * yy)); wr(13, C34 * x * (4.f * zz - xx - yy));
							wr(14, C35 * z * (xx - yy)); wr(15, C36 * x * (xx - 3.f * yy));
						}
					}
				}
				wr(0, kSH_C0);
				{ const int nact = (deg + 1) * (deg + 1); for (int k = 3 * nact; k < RL; k++) myrow[k] = 0.f; }
				const float ddx = dRx[0] * dRGB[0] + dRx[1] * dRGB[1] + dRx[2] * dRGB[2];
				const float ddy = dRy[0] * dRGB[0] + dRy[1] * dRGB[1] + dRy[2] * dRGB[2];
				const float ddz = dRz[0] * dRGB[0] + dRz[1] * dRGB[1] + dRz[2] * dRGB[2];
				const float sum2 = dox * dox + doy * doy + doz * doz;                       // dnormvdv, auxiliary.h:107-117
				const float invsum32 = 1.0f / sqrtf(sum2 * sum2 * sum2);
				const float n0 = (+sum2 - dox * dox) * ddx - doy * dox * ddy - doz * dox * ddz;
				const float n1 = -dox * doy * ddx + (sum2 - doy * doy) * ddy - doz * doy * ddz;
				const float n2 = -dox * doz * ddx - doy * doz * ddy + (sum2 - doz * doz) * ddz;
				dmean[0] += n0 * invsum32;
				dmean[1] += n1 * invsum32;
				dmean[2] += n2 * invsum32;
				// dir = mean - campos.  A product of its own: a second use of n*invsum32 would change how the compiler fuses the
				// additions above (dL_dmeans3D of the CAM variant then still agrees with CAM = false to rounding only, see gs_b200.h)
				if (CAM) { cg_dir[0] = __fmul_rn(n0, invsum32); cg_dir[1] = __fmul_rn(n1, invsum32); cg_dir[2] = __fmul_rn(n2, invsum32); }
			}
			// ---------------- cov3D -> scale / rotation, backward.cu:311-374 ----------------
			if (have_scales)
			{
				const float r = qr, x = qx, y = qy, z = qz;
				const float Rm[3][3] = { { 1.f - 2.f * (y * y + z * z), 2.f * (x * y - r * z), 2.f * (x * z + r * y) },
					{ 2.f * (x * y + r * z), 1.f - 2.f * (x * x + z * z), 2.f * (y * z - r * x) },
					{ 2.f * (x * z - r * y), 2.f * (y * z + r * x), 1.f - 2.f * (x * x + y * y) } };     // Rm[c][r]
				const float s[3] = { a.s.mod * sc[0], a.s.mod * sc[1], a.s.mod * sc[2] };
				float Mm[3][3];
				for (int c = 0; c < 3; c++) for (int rr = 0; rr < 3; rr++) Mm[c][rr] = s[rr] * Rm[c][rr];
				const float dSig[3][3] = { { dcov[0], 0.5f * dcov[1], 0.5f * dcov[2] }, { 0.5f * dcov[1], dcov[3], 0.5f * dcov[4] }, { 0.5f * dcov[2], 0.5f * dcov[4], dcov[5] } };
				float dMt[3][3];   // dL_dMt[c][r] = dL_dM[r][c], dL_dM = 2 * M * dL_dSigma
				for (int c = 0; c < 3; c++) for (int rr = 0; rr < 3; rr++)
					dMt[rr][c] = 2.f * (Mm[0][rr] * dSig[c][0] + Mm[1][rr] * dSig[c][1] + Mm[2][rr] * dSig[c][2]);
				for (int k = 0; k < 3; k++) o_sc[k] = Rm[0][k] * dMt[k][0] + Rm[1][k] * dMt[k][1] + Rm[2][k] * dMt[k][2];   // Rt[k][j] = Rm[j][k]
				for (int k = 0; k < 3; k++) for (int rr = 0; rr < 3; rr++) dMt[k][rr] *= s[k];
				o_rot[0] = 2 * z * (dMt[0][1] - dMt[1][0]) + 2 * y * (dMt[2][0] - dMt[0][2]) + 2 * x * (dMt[1][2] - dMt[2][1]);
				o_rot[1] = 2 * y * (dMt[1][0] + dMt[0][1]) + 2 * z * (dMt[2][0] + dMt[0][2]) + 2 * r * (dMt[1][2] - dMt[2][1]) - 4 * x * (dMt[2][2] + dMt[1][1]);
				o_rot[2] = 2 * x * (dMt[1][0] + dMt[0][1]) + 2 * r * (dMt[2][0] - dMt[0][2]) + 2 * z * (dMt[1][2] + dMt[2][1]) - 4 * y * (dMt[2][2] + dMt[0][0]);
				o_rot[3] = 2 * r * (dMt[0][1] - dMt[1][0]) + 2 * x * (dMt[2][0] + dMt[0][2]) + 2 * y * (dMt[1][2] + dMt[2][1]) - 4 * z * (dMt[1][1] + dMt[0][0]);
				if constexpr (F3D)
				{
					if (f3d != 0.f)
					{
						// s'_k = sqrt(s_k^2 + f^2): ds'_k/ds_k = s_k / s'_k.  c3 = prod_k s_k / s'_k, so with r = s^2 / s'^2
						// dc3/ds_k = sqrt(r_i r_j) (1 - r_k) / s'_k, finite at s_k = 0 (flat splats)
						const float gs = acc0.w * (AA ? aa_s : 1.f) * sig;
						float rr[3];
						for (int k = 0; k < 3; k++) rr[k] = __fdiv_rn(f3sq.a[k], f3sq.b[k]);
						for (int k = 0; k < 3; k++)
						{
							const float dc3 = __fsqrt_rn(rr[(k + 1) % 3] * rr[(k + 2) % 3]) * (1.f - rr[k]) / sc[k];
							o_sc[k] = o_sc[k] * (s_act[k] / sc[k]) + gs * dc3;
						}
					}
				}
				if (RAW)
				{
					// ExpBackward0: grad * result
					for (int k = 0; k < 3; k++) o_sc[k] = __fmul_rn(o_sc[k], F3D ? s_act[k] : sc[k]);
					// F.normalize = q / expand(clamp_min(norm(q), 1e-12)).  DivBackward0: g / d and -g * ((q / d) / d), where q / d is
					// the normalised (r, x, y, z) above; ExpandBackward0 sums the four as (0 + 2) + (1 + 3); ClampMinBackward0 passes
					// it where norm >= 1e-12; LinalgVectorNormBackward0: gn * (q / norm), 0 where norm == 0
					// the unnormalised rotation is read again here (an L1 / L2 hit) rather than kept live through the covariance
					const float4 q4 = reinterpret_cast<const float4*>(a.s.rotations)[idx];
					const float rq[4] = { q4.x, q4.y, q4.z, q4.w };
					const float rq_n = quat_norm(q4.x, q4.y, q4.z, q4.w);
					const float d = fmaxf(rq_n, 1e-12f);
					const float qn[4] = { r, x, y, z };
					float go[4];
					for (int k = 0; k < 4; k++) go[k] = __fmul_rn(-o_rot[k], __fdiv_rn(qn[k], d));
					const float gsum = __fadd_rn(__fadd_rn(go[0], go[2]), __fadd_rn(go[1], go[3]));
					const float gn = rq_n >= 1e-12f ? gsum : 0.f;
					for (int k = 0; k < 4; k++)
						o_rot[k] = __fadd_rn(__fdiv_rn(o_rot[k], d), rq_n == 0.f ? 0.f : __fmul_rn(gn, __fdiv_rn(rq[k], rq_n)));
				}
			}
			o_m2[0] = g2x; o_m2[1] = g2y;
			o_col[0] = acc0.x; o_col[1] = acc0.y; o_col[2] = acc0.z;
			o_op[0] = acc0.w * (opac * (1.0f - opac));                                    // backward.cu:433
			// AA: the record holds o^ = sigmoid * s, so dL/dlogit = dL/do^ * s * sigmoid (1 - sigmoid) = dL/do^ * o^ (1 - o^ / s)
			if constexpr (AA) o_op[0] = acc0.w * (opac * (1.0f - opac / aa_s));
			// F3D: o^ = sigmoid * c3 (* s with AA), the sigmoid taken from the logit
			if constexpr (F3D)
			{
				if (f3d != 0.f) o_op[0] = acc0.w * (AA ? aa_s : 1.f) * c3 * (sig * (1.0f - sig));
			}
			for (int k = 0; k < 3; k++) o_m3[k] = dmean[k];
			for (int k = 0; k < 6; k++) o_cov[k] = dcov[k];
			o_con[0] = dconx; o_con[1] = dcony; o_con[3] = dconz;
		}
		__syncwarp();
		// ---- unit-stride write-back ------------------------------------------------------------------
		if (RAW)
		{
			if (a.dL_ddc) raw_block<true, ACC>(nullptr, a.dL_ddc, 3, 0, base, n_valid, s_row, RS, lane, have_sh, a.raw_vec4);
			if (a.dL_drest && a.s.n_rest)
				raw_block<true, ACC>(nullptr, a.dL_drest, 3 * a.s.n_rest, 3, base, n_valid, s_row, RS, lane, have_sh, a.raw_vec4);
		}
		else if (a.out.dL_dsh && RL == 48 && n_valid == 32 && a.dsh_vec4)
		{
			float4* dst4 = reinterpret_cast<float4*>(a.out.dL_dsh + base * 48);
#pragma unroll
			for (int i = 0; i < 12; i++)
			{
				const int f = (i * 32 + lane) * 4, row = f / 48, col = f - row * 48;
				const float* sp = s_row + row * RS + col;
				float4 o = have_sh ? make_float4(sp[0], sp[1], sp[2], sp[3]) : make_float4(0.f, 0.f, 0.f, 0.f);
				if (ACC)
				{
					if (o.x != 0.f || o.y != 0.f || o.z != 0.f || o.w != 0.f) red_add_v4(reinterpret_cast<float*>(dst4 + i * 32 + lane), o.x, o.y, o.z, o.w);
				}
				else dst4[i * 32 + lane] = o;
			}
		}
		else if (a.out.dL_dsh)
		{
			float* dst = a.out.dL_dsh + base * RL;
			int row = 0, col = lane;
			while (col >= RL) { col -= RL; row++; }
			for (int f = lane; f < n_valid * RL; f += 32)
			{
				put<ACC>(dst + f, have_sh ? s_row[row * RS + col] : 0.f);
				col += 32;
				while (col >= RL) { col -= RL; row++; }
			}
		}
		warp_store<3, ACC>(a.out.dL_dmeans2D, base, n_valid, o_m2, s_tmp, lane);
		// accumulate mode: THIS view's screen-space gradient on its own (densification statistics are ||.|| per view, gaussian_model.py:693-695)
		if (ACC && a.out.dL_dmeans2D_view) warp_store<3, false>(a.out.dL_dmeans2D_view, base, n_valid, o_m2, s_tmp, lane);
		if (!RAW || a.out.dL_dcolors) warp_store<3, ACC>(a.out.dL_dcolors, base, n_valid, o_col, s_tmp, lane);
		warp_store<1, ACC>(a.out.dL_dopacity, base, n_valid, o_op, s_tmp, lane);
		warp_store<3, ACC>(a.out.dL_dmeans3D, base, n_valid, o_m3, s_tmp, lane);
		if (!RAW || a.out.dL_dcov3D) warp_store<6, ACC>(a.out.dL_dcov3D, base, n_valid, o_cov, s_tmp, lane);
		warp_store<3, ACC>(a.out.dL_dscales, base, n_valid, o_sc, s_tmp, lane);
		warp_store<4, ACC>(a.out.dL_drotations, base, n_valid, o_rot, s_tmp, lane);
		if (a.out.dL_dconic) warp_store<4, ACC>(a.out.dL_dconic, base, n_valid, o_con, s_tmp, lane);
		__syncwarp();
		if (CAM && __any_sync(0xffffffffu, vis))
		{
			const float m[4] = { vis ? mx : 0.f, vis ? my : 0.f, vis ? mz : 0.f, vis ? 1.f : 0.f };
			float mine = 0.f;
#pragma unroll
			for (int k = 0; k < GSB_CAM_SLOTS; k++)
			{
				float c;
				if (k < 12)
				{
					const int r = k / 3, cc = k % 3;
					c = cg_dt[cc] * m[r];                                             // through t_c = sum_r view[4r+c] m_r
					if (r < 3)                                                        // direct, through T = W J
					{
						if (cc == 0) c += cg_T0[r] * cg_J[0];
						else if (cc == 1) c += cg_T1[r] * cg_J[2];
						else c += cg_T0[r] * cg_J[1] + cg_T1[r] * cg_J[3];
					}
				}
				else if (k < 24) c = cg_p[(k - 12) % 3] * m[(k - 12) / 3];
				else c = -cg_dir[k - 24];
#pragma unroll
				for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
				if (lane == k) mine = c;
			}
			cam_sum += mine;
		}
	}
	if (CAM)
	{
		// every warp is past its last warp_store: its s_tmp is free
		s_tmp[lane] = cam_sum;
		__syncthreads();
		if (threadIdx.x < GSB_CAM_SLOTS)
		{
			const float* s0 = s_dyn + (QUANT ? GSB_NUM_CODEBOOKS * GSB_CODEBOOK_SIZE : 0) + 32 * RS + threadIdx.x;
			float s = 0.f;
			for (int w = 0; w < 8; w++) s += s0[w * (32 * RS + 32 * 6)];
			a.cam_rows[(size_t)blockIdx.x * GSB_CAM_ROW + threadIdx.x] = s;
		}
	}
}

// One CTA: the per-CTA rows of preprocess_backward_kernel<.., CAM = true> summed in double, in row order within 8 strided parts and
// then part order, and scattered into the 4x4 layouts (zeros where the preprocess does not read the matrix).
__global__ void __launch_bounds__(256) camera_grad_finish_kernel(const float* __restrict__ rows, int n_rows, float* dview, float* dproj,
	float* dcampos)
{
	__shared__ double s_part[8][GSB_CAM_ROW];
	const int k = threadIdx.x & 31, part = threadIdx.x >> 5;
	double s = 0.0;
	if (k < GSB_CAM_SLOTS)
		for (int r = part; r < n_rows; r += 8) s += (double)rows[(size_t)r * GSB_CAM_ROW + k];
	s_part[part][k] = s;
	__syncthreads();
	if (threadIdx.x < 16)
	{
		const int t = threadIdx.x, r = t >> 2, c = t & 3;
		auto total = [&](int slot) { double v = 0.0; for (int p = 0; p < 8; p++) v += s_part[p][slot]; return (float)v; };
		if (dview) dview[t] = c == 3 ? 0.f : total(3 * r + c);
		if (dproj) dproj[t] = c == 2 ? 0.f : total(12 + 3 * r + (c == 3 ? 2 : c));
		if (dcampos && t < 3) dcampos[t] = total(24 + t);
	}
}

static int preprocess_backward_grid(int P)
{
	const int need = (P + 255) / 256;
	return need < GSB_NUM_SMS * 4 ? need : GSB_NUM_SMS * 4;
}

size_t camera_grad_workspace_bytes(int P)
{
	const int rows = P > 0 ? preprocess_backward_grid(P) : 1;
	return size_t(rows) * GSB_CAM_ROW * sizeof(float);
}

int launch_camera_grad_finish(int P, const float* rows, float* dview, float* dproj, float* dcampos, cudaStream_t stream)
{
	ProfScope prof(K_CAMERA_GRAD, stream);
	camera_grad_finish_kernel<<<1, 256, 0, stream>>>(rows, P > 0 ? preprocess_backward_grid(P) : 0, dview, dproj, dcampos);
	GSB_LAUNCHED();
	GSB_CUDA_OK(cudaGetLastError());
	return GSB_OK;
}

int launch_preprocess_backward(const GsbBackwardRequest& req, const GeomState& g, const float* acc)
{
	const GsbScene* s = req.scene; const GsbRawParams* raw = req.raw;
	BwdArgs a{};
	a.s = scene_args(s, req.cam, raw);
	a.lambda = req.lambda_sh_sparsity;
	a.radii = req.radii;
	a.g = g; a.acc = acc; a.out = *req.grads; a.cam_rows = want_cam(req) ? reinterpret_cast<float*>(req.camera_workspace) : nullptr;
	auto al = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
	if (raw)
	{
		a.s.M = raw->features_dc && !s->colors_precomp ? 1 + raw->C : 0;
		a.out.dL_dscales = req.raw_grads->dL_dscaling; a.out.dL_drotations = req.raw_grads->dL_drotation;
		a.dL_ddc = req.raw_grads->dL_dfeatures_dc; a.dL_drest = req.raw_grads->dL_dfeatures_rest;
		a.raw_vec4 = al(s->colors_precomp ? nullptr : a.s.sh_dc) && al(a.s.sh_rest) && al(a.dL_ddc) && al(a.dL_drest);   // sh_dc is not read with colours
	}
	a.sh_vec4 = al(a.s.shs); a.dsh_vec4 = al(a.out.dL_dsh);
	const int grid = preprocess_backward_grid(s->P);
	const size_t smem = (a.s.quant ? GSB_NUM_CODEBOOKS * GSB_CODEBOOK_SIZE : 0) * sizeof(float) + 8 * (32 * (3 * a.s.M + 1) + 32 * 6) * sizeof(float);
	const cudaStream_t stream = stream_of(req);
	ProfScope prof(K_PREPROCESS_BWD, stream);
	const InputMode in = a.s.quant ? IN_QUANT : (raw ? IN_RAW : IN_ACTIVATED);
	return dispatch([&](auto in, auto accumulate, auto maps, auto cam_grad, auto aa, auto f3d) -> int {
		auto kernel = preprocess_backward_kernel<in, accumulate, maps, cam_grad, aa, f3d>;
		if (int e = ensure_dyn_smem((const void*)kernel, 160 * 1024)) return e;
		kernel<<<grid, 256, smem, stream>>>(a);
		GSB_LAUNCHED();
		GSB_CUDA_OK(cudaGetLastError());
		return GSB_OK;
	}, in, req.grads->accumulate != 0, req.dL_dinvdepth != nullptr, a.cam_rows != nullptr, req.antialiasing != 0, s->filter_3D != nullptr);
}

} // namespace gsb
