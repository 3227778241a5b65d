// gsb_api.cu — the C ABI (include/gs_b200.h): orchestration of the forward / backward pipelines.
//
// Forward replaces CudaRasterizer::Rasterizer::forward (rasterizer_impl.cu:359-504):
//   preprocess (+ per-CTA tile histograms) -> tile prefix / scan -> [R travels to the host in the background] -> scatter ->
//   per-tile sort (both launched speculatively against the capacity recent frames needed) -> [host waits for R's event] -> render
//                                                (the reference: preprocess -> scan -> D2H of R, device stalled -> emit keys ->
//                                                 global radix sort -> ranges -> render)
// Backward replaces Rasterizer::backward (rasterizer_impl.cu:508-630): render backward -> preprocess backward.
// The entry points of the reduced-3dgs tools around the rasterizer (statistics forward, redundancy score, k-means, loss) are
// thin argument checks in front of the launchers in gsb_tools.cu / gsb_kmeans.cu / gsb_loss.cu.
#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>
#include <utility>
#include <vector>
#include "gsb_common.cuh"

namespace gsb {

// ---- process-wide state: all of it is either atomic, mutex-guarded or per thread; per-device facts are keyed by device ----
static std::atomic<unsigned long long> g_launch_count{0};
void count_launch() { g_launch_count.fetch_add(1, std::memory_order_relaxed); }
static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...)
{
	va_list ap; va_start(ap, fmt);
	vsnprintf(g_err, sizeof(g_err), fmt, ap);
	va_end(ap);
}

// cudaFuncAttributeMaxDynamicSharedMemorySize is a per-device (per-context) attribute: remember the largest opt-in made for
// each (kernel, device) pair instead of a process-wide "done" flag, so a second GPU driven from the same process gets its own.
int ensure_dyn_smem(const void* kernel, int bytes)
{
	static std::mutex mu;
	static std::map<std::pair<const void*, int>, int> done;
	int dev = 0;
	GSB_CUDA_OK(cudaGetDevice(&dev));
	std::lock_guard<std::mutex> lk(mu);
	int& have = done[std::make_pair(kernel, dev)];
	if (have >= bytes) return GSB_OK;
	GSB_CUDA_OK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
	have = bytes;
	return GSB_OK;
}

int bin_plan_per_sm_override()
{
	static const int v = [] { const char* e = getenv("GSB_BIN_PER_SM"); const int x = e ? atoi(e) : 0; return x >= 1 && x <= 4 ? x : 0; }();
	return v;
}

// ---- per-kernel profiling (events are created on the device that is current when they are first needed; the bench drives
// one device per process).  The record list and the event pool are shared by all host threads: mutex-guarded; the "open"
// event of a ProfScope belongs to the thread that opened it.
static std::atomic<bool> g_prof_on{false};
struct ProfRec { int kid; cudaEvent_t a, b; };
static std::mutex g_prof_mu;
static std::vector<ProfRec> g_prof_recs;
static std::vector<cudaEvent_t> g_prof_pool;
static thread_local cudaEvent_t t_prof_cur = nullptr;
static cudaEvent_t prof_event()
{
	{
		std::lock_guard<std::mutex> lk(g_prof_mu);
		if (!g_prof_pool.empty()) { cudaEvent_t e = g_prof_pool.back(); g_prof_pool.pop_back(); return e; }
	}
	cudaEvent_t e; cudaEventCreate(&e); return e;
}
void prof_begin(int kid, cudaStream_t stream)
{
	(void)kid;
	if (!g_prof_on.load(std::memory_order_relaxed)) return;
	t_prof_cur = prof_event();
	cudaEventRecord(t_prof_cur, stream);
}
void prof_end(int kid, cudaStream_t stream)
{
	if (!g_prof_on.load(std::memory_order_relaxed) || !t_prof_cur) return;
	cudaEvent_t b = prof_event();
	cudaEventRecord(b, stream);
	{
		std::lock_guard<std::mutex> lk(g_prof_mu);
		g_prof_recs.push_back({ kid, t_prof_cur, b });
	}
	t_prof_cur = nullptr;
}
static const char* kKernelNames[K_COUNT] = { "preprocess", "tile_scan", "scatter", "tile_sort_large", "tile_sort", "render_forward", "render_backward", "preprocess_backward", "mark_visible", "tools", "kmeans", "knn", "camera_grad", "det_scan",
	"det_gather", "det_clear", "features_forward", "features_backward", "absgrad_finish", "contributions" };

int launch_debug_dequant(const GsbQuant*, int, float*, float*, cudaStream_t);
int launch_mark_visible(int, const float*, const float*, uint8_t*, cudaStream_t);
int launch_tile_scan(const ImageState&, const GeomState&, const BinPlan&, int, int, cudaStream_t);
int launch_scatter_sort(const GeomState&, const BinningState&, const ImageState&, const BinPlan&, int, long long, int, int, cudaStream_t);
int launch_sort_large(const GeomState&, const BinningState&, const ImageState&, int, int, uint32_t, uint32_t, cudaStream_t);
int launch_export_binning(const GeomState&, const BinningState&, const ImageState&, int, int, uint64_t*, uint32_t*, cudaStream_t);
int launch_sh_stats_update(int, int, const int*, const float*, const float*, const float*, const int*, const int*, const float*, float*, float*,
	float*, float*, float*, cudaStream_t);
int launch_pixel_size(int, const float*, int, const float*, const float*, const int*, const int*, float*, cudaStream_t);
int launch_filter_3d(int, const float*, int, const float*, const float*, const int*, float*, unsigned*, cudaStream_t);
int launch_sphere_ellipsoid(int, const float*, const float*, const float*, const int*, const float*, int, int*, uint8_t*, cudaStream_t);
int launch_min_redundancy(int, const int*, const int*, const uint8_t*, int, int*, cudaStream_t);
int launch_redundancy_fused(int, const float*, const float*, const float*, const int*, const float*, float, int, int*, cudaStream_t);
int launch_l1_ssim_forward(const float*, const float*, int, int, int, float*, float*, cudaStream_t);
int launch_l1_ssim_backward(const float*, const float*, int, int, int, const float*, float, const float*, float, const float*, float*, cudaStream_t);
size_t kmeans_workspace_bytes(long long, int, bool);
int launch_kmeans(const float*, long long, const float*, int, float, int, int*, float*, char*, bool, cudaStream_t);
size_t knn_workspace_bytes(long long, long long);
int launch_knn(const float*, long long, int, const int32_t*, long long, const int32_t*, long long, float*, float*, int32_t*, char*, cudaStream_t);
size_t det_workspace_bytes(int, long long, int);
size_t camera_grad_workspace_bytes(int);
int launch_camera_grad_finish(int, const float*, float*, float*, float*, cudaStream_t);

// geometry blob = GeomState followed by the backward's gradient accumulator (12 floats per Gaussian)
static size_t geom_state_bytes(int P) { size_t b; GeomState::carve(nullptr, P, &b); return (b + 255) & ~size_t(255); }

// The request checks: check_forward / check_backward validate a request before gsb_forward / gsb_backward make any CUDA call, in
// the order include/gs_b200.h lists under "Request checks".  Every message starts with the direction, `dir`.

// With raw parameters: what the scene and the raw struct hold.
static int check_raw(const char* dir, const GsbScene* s, const GsbRawParams* raw)
{
	if (raw->C != 0 && raw->C != 3 && raw->C != 8 && raw->C != 15)
	{ set_error("%s: raw parameters: C = %d rest coefficients; only 0, 3, 8 or 15 (max SH degree 0..3) exist", dir, raw->C); return GSB_EINVAL; }
	if (s->scales || s->rotations || s->shs || s->cov3D_precomp || s->quant || s->sh_packed)
	{ set_error("%s: raw parameters: the scene's scales, rotations, shs, cov3D_precomp and quant must be NULL and sh_packed 0", dir); return GSB_EINVAL; }
	if (s->P == 0) return GSB_OK;
	if (!raw->scaling || !raw->rotation) { set_error("%s: raw parameters: scaling / rotation missing", dir); return GSB_EINVAL; }
	if (s->colors_precomp)
	{
		if (raw->features_dc || raw->features_rest) { set_error("%s: raw parameters: SH given together with colors_precomp", dir); return GSB_EINVAL; }
	}
	else if (!raw->features_dc || !s->degrees || (raw->features_rest == nullptr) != (raw->C == 0))
	{ set_error("%s: raw parameters: features_dc, degrees and (for C > 0) features_rest are required without colors_precomp", dir); return GSB_EINVAL; }
	return GSB_OK;
}

// The camera and the scene's tensors; the scene itself is non-NULL with P >= 0.  raw: check_raw replaces the checks of the
// activated inputs.
static int check_scene(const char* dir, const GsbScene* s, const GsbCamera* c, bool raw)
{
	if (!c) { set_error("%s: camera is NULL", dir); return GSB_EINVAL; }
	if (c->width <= 0 || c->height <= 0) { set_error("%s: bad image size %dx%d", dir, c->width, c->height); return GSB_EINVAL; }
	if (!c->viewmatrix || !c->projmatrix || !c->campos || !c->background) { set_error("%s: camera tensors missing", dir); return GSB_EINVAL; }
	if (s->P == 0) return GSB_OK;
	if (!s->means3D) { set_error("%s: means3D missing", dir); return GSB_EINVAL; }
	if (s->quant)
	{
		const GsbQuant* q = s->quant;
		if (!q->ids_dc || !q->ids_rest || !q->ids_opacity || !q->ids_scaling || !q->ids_rot || !q->centers || !s->degrees)
		{ set_error("%s: quantised scene: id planes / centres / degrees missing", dir); return GSB_EINVAL; }
		if (s->M != 16) { set_error("%s: quantised scene needs M == 16", dir); return GSB_EINVAL; }
		return GSB_OK;
	}
	if (!s->opacities) { set_error("%s: opacities missing", dir); return GSB_EINVAL; }
	if (raw) return GSB_OK;
	// diff_gaussian_rasterization/__init__.py:203-207
	if ((s->shs == nullptr) == (s->colors_precomp == nullptr)) { set_error("%s: Please provide excatly one of either SHs or precomputed colors!", dir); return GSB_EINVAL; }
	const bool sr = s->scales != nullptr && s->rotations != nullptr;
	if (sr == (s->cov3D_precomp != nullptr) || ((s->scales != nullptr) != (s->rotations != nullptr)))
	{ set_error("%s: Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!", dir); return GSB_EINVAL; }
	if (s->shs && !s->sh_packed && (!s->degrees || s->M <= 0)) { set_error("%s: dense SH needs degrees and M > 0", dir); return GSB_EINVAL; }
	if (s->filter_3D && s->cov3D_precomp)
	{ set_error("%s: filter_3D filters the scales; it does not go with cov3D_precomp", dir); return GSB_EINVAL; }
	return GSB_OK;
}

// The feature pass's own fields (a request with features).
static int check_features(const char* dir, const GsbFeatures* f, int P, bool backward)
{
	if (f->F < 1 || f->F > GSB_FEATURES_MAX) { set_error("%s: F = %d channels; 1..%d are supported", dir, f->F, GSB_FEATURES_MAX); return GSB_EINVAL; }
	if (P > 0 && !f->features) { set_error("%s: features->features is NULL", dir); return GSB_EINVAL; }
	if (backward && P > 0 && (!f->dL_dout || !f->dL_dfeatures)) { set_error("%s: features->dL_dout / dL_dfeatures is NULL", dir); return GSB_EINVAL; }
	if (!backward && !f->out) { set_error("%s: features->out is NULL", dir); return GSB_EINVAL; }
	return GSB_OK;
}

static int check_forward(const GsbForwardRequest& r)
{
	const GsbScene* s = r.scene; const GsbCamera* c = r.cam;
	if (!s || s->P < 0) { set_error("forward: scene is NULL or P < 0"); return GSB_EINVAL; }
	if (r.features) if (int e = check_features("forward", r.features, s->P, false)) return e;
	if ((r.out_invdepth == nullptr) != (r.out_alpha == nullptr))
	{ set_error("forward: give both map outputs (invdepth and alpha) or neither"); return GSB_EINVAL; }
	if (statistics(r))
	{
		if (!r.touched_pixels || !r.transmittance_sum) { set_error("forward: statistics output pointers missing"); return GSB_EINVAL; }
		if (r.out_invdepth || r.antialiasing || r.raw)
		{ set_error("forward: statistics go without the maps, antialiasing and raw parameters"); return GSB_EINVAL; }
		if (s->filter_3D) { set_error("forward: statistics go without filter_3D (they keep the reference's definition)"); return GSB_EINVAL; }
		if (r.deterministic)
		{
			if (s->P > 0 && !r.workspace) { set_error("forward: workspace is NULL"); return GSB_EINVAL; }
			if (c && (long long)c->width * c->height >= (1ll << 28))
			{ set_error("forward: %d x %d pixels; the 64-bit fixed-point sums need W * H < 2^28", c->width, c->height); return GSB_ERANGE; }
		}
	}
	if (r.raw) if (int e = check_raw("forward", s, r.raw)) return e;
	if (int e = check_scene("forward", s, c, r.raw != nullptr)) return e;
	if (!r.out_color || !r.num_rendered || (s->P > 0 && !r.radii)) { set_error("forward: output pointers missing"); return GSB_EINVAL; }
	return GSB_OK;
}

static int check_backward(const GsbBackwardRequest& r)
{
	const GsbScene* s = r.scene; const GsbGrads* grads = r.grads;
	if (!s || s->P < 0) { set_error("backward: scene is NULL or P < 0"); return GSB_EINVAL; }
	if (r.features)
	{
		if (r.deterministic) { set_error("backward: the feature backward has no deterministic form; deterministic must be 0"); return GSB_EINVAL; }
		if (int e = check_features("backward", r.features, s->P, true)) return e;
	}
	if (r.dL_dmeans2D_abs)
	{
		if (r.features) { set_error("backward: the absolute gradient has no feature form; give features or dL_dmeans2D_abs"); return GSB_EINVAL; }
		if (grads && grads->accumulate)
		{ set_error("backward: grads->accumulate is set; the absolute gradient has no view-batch accumulation form"); return GSB_EINVAL; }
	}
	if (r.num_rendered < 0) { set_error("backward: num_rendered < 0"); return GSB_EINVAL; }
	if (r.deterministic)
	{
		if (r.num_rendered >= (1ll << 30))
		{ set_error("backward: 2^30 or more instances (the slot scan's look-back descriptors carry 30-bit counts)"); return GSB_ERANGE; }
		if (s->P > 0 && r.num_rendered > 0 && !r.det_workspace) { set_error("backward: det_workspace is NULL"); return GSB_EINVAL; }
	}
	if (want_cam(r) && !r.camera_workspace) { set_error("backward: a camera gradient is requested but the workspace is NULL"); return GSB_EINVAL; }
	if (r.raw_grads && !r.raw) { set_error("backward: raw_grads given without raw"); return GSB_EINVAL; }
	if (r.raw)
	{
		if (int e = check_raw("backward", s, r.raw)) return e;
		const GsbRawGrads* rg = r.raw_grads;
		if (!rg || !grads) { set_error("backward: grads / raw_grads are NULL"); return GSB_EINVAL; }
		if (grads->dL_dsh || grads->dL_dscales || grads->dL_drotations)
		{ set_error("backward: grads->dL_dsh, dL_dscales and dL_drotations must be NULL (raw_grads replaces them)"); return GSB_EINVAL; }
		if (s->colors_precomp && (rg->dL_dfeatures_dc || rg->dL_dfeatures_rest))
		{ set_error("backward: SH gradients requested together with colors_precomp"); return GSB_EINVAL; }
		if (r.raw->C == 0 && rg->dL_dfeatures_rest) { set_error("backward: dL_dfeatures_rest given with C == 0"); return GSB_EINVAL; }
	}
	if (int e = check_scene("backward", s, r.cam, r.raw != nullptr)) return e;
	if (!grads) { set_error("backward: grads is NULL"); return GSB_EINVAL; }
	if (s->P == 0) return GSB_OK;
	if (!r.geom_blob || !r.binning_blob || !r.image_blob || !r.dL_dout_color || !r.radii) { set_error("backward: backward inputs missing"); return GSB_EINVAL; }
	if (r.raw)
	{
		if (!grads->dL_dmeans2D || !grads->dL_dopacity || !grads->dL_dmeans3D || !r.raw_grads->dL_dscaling || !r.raw_grads->dL_drotation)
		{ set_error("backward: gradient output pointers missing"); return GSB_EINVAL; }
	}
	else if (!grads->dL_dmeans2D || !grads->dL_dcolors || !grads->dL_dopacity || !grads->dL_dmeans3D || !grads->dL_dcov3D ||
		!grads->dL_dscales || !grads->dL_drotations || (s->M > 0 && !grads->dL_dsh))
	{ set_error("backward: gradient output pointers missing"); return GSB_EINVAL; }
	return GSB_OK;
}

} // namespace gsb

using namespace gsb;

extern "C" {

size_t gsb_geom_bytes(int32_t P) { return geom_state_bytes(P) + size_t(P) * 48 + 512; }
// upper bound for callers that pre-allocate without knowing the scene (the largest per-CTA histogram table: 592 rows) ...
size_t gsb_image_bytes(int32_t W, int32_t H) { size_t b; ImageState::carve(nullptr, W, H, &b, GSB_NUM_SMS * 4); return b + 256; }
// ... and what the forward actually requests: the histogram rows of THIS scene's plan (none at all beyond the shared-memory limit)
size_t gsb_image_bytes_for(int32_t P, int32_t W, int32_t H, int32_t quantised)
{
	const BinPlan plan = make_bin_plan(P, W, H, quantised != 0);
	size_t b; ImageState::carve(nullptr, W, H, &b, plan.priv ? plan.ctas : 0); return b + 256;
}
size_t gsb_binning_bytes(int64_t R) { size_t b; BinningState::carve(nullptr, R, &b); return b + 256; }
uint64_t gsb_launch_count(void) { return g_launch_count.load(); }
const char* gsb_last_error(void) { return g_err; }
const char* gsb_version(void) { return "gs_b200 0.3 (sm_90a)"; }

void gsb_profile_enable(int on)
{
	g_prof_on.store(on != 0);
	// cudaEventCreate costs tens of microseconds: create the pool up front so the timed region only records
	std::lock_guard<std::mutex> lk(g_prof_mu);
	if (on) while (g_prof_pool.size() < 4096) { cudaEvent_t e; if (cudaEventCreate(&e) != cudaSuccess) break; g_prof_pool.push_back(e); }
}

int gsb_profile_read(int max_entries, const char** names, double* total_ms, uint64_t* launches)
{
	double ms[K_COUNT] = { 0 }; uint64_t n[K_COUNT] = { 0 };
	std::vector<ProfRec> recs;
	{
		std::lock_guard<std::mutex> lk(g_prof_mu);
		recs.swap(g_prof_recs);
	}
	for (auto& r : recs)
	{
		cudaEventSynchronize(r.b);
		float t = 0.f;
		if (cudaEventElapsedTime(&t, r.a, r.b) == cudaSuccess) { ms[r.kid] += t; n[r.kid]++; }
		std::lock_guard<std::mutex> lk(g_prof_mu);
		g_prof_pool.push_back(r.a); g_prof_pool.push_back(r.b);
	}
	int k = 0;
	for (int i = 0; i < K_COUNT && k < max_entries; i++)
		if (n[i]) { names[k] = kKernelNames[i]; total_ms[k] = ms[i]; launches[k] = n[i]; k++; }
	return k;
}

// Host side of the instance-count read-back, per (host thread, device): a pinned landing buffer, the event that marks its
// arrival, and the largest instance count seen recently (the capacity the next frame's binning blob is speculatively carved for).
namespace {
struct HostSide {
	uint32_t* counters = nullptr;
	cudaEvent_t arrived = nullptr;
	long long r_hint = 0;
	~HostSide()
	{
		if (counters) cudaFreeHost(counters);             // thread exit; errors (runtime already unloading) are irrelevant here
		if (arrived) cudaEventDestroy(arrived);
	}
};
static thread_local std::map<int, HostSide> t_host;
}

int gsb_forward(const GsbForwardRequest* req)
{
	if (!req) { set_error("forward: request is NULL"); return GSB_EINVAL; }
	const GsbForwardRequest& r = *req;
	if (int e = check_forward(r)) return e;
	const GsbScene* scene = r.scene; const cudaStream_t stream = stream_of(r);
	*r.num_rendered = 0;
	const int P = scene->P, W = r.cam->width, H = r.cam->height;
	const size_t N = size_t(W) * H;
	if (P == 0)
	{
		// rasterize_points.cu:170,184-185: P == 0 returns the zero-initialised image (no background); the maps are zero too
		GSB_CUDA_OK(cudaMemsetAsync(r.out_color, 0, 3 * N * sizeof(float), stream));
		if (r.out_invdepth) GSB_CUDA_OK(cudaMemsetAsync(r.out_invdepth, 0, N * sizeof(float), stream));
		if (r.out_alpha) GSB_CUDA_OK(cudaMemsetAsync(r.out_alpha, 0, N * sizeof(float), stream));
		// the forward of an empty scene allocates no blobs; its feature image is zero like its colour image
		if (r.features) GSB_CUDA_OK(cudaMemsetAsync(r.features->out, 0, size_t(r.features->F) * N * sizeof(float), stream));
		return GSB_OK;
	}
	if (statistics(r))
	{
		// reduced_3dgs.cu:117-118: both statistics start from zero for every camera
		GSB_CUDA_OK(cudaMemsetAsync(r.touched_pixels, 0, size_t(P) * sizeof(int32_t), stream));
		if (stats_fixed(r)) GSB_CUDA_OK(cudaMemsetAsync(transmittance_fixed(r), 0, size_t(P) * sizeof(unsigned long long), stream));
		else GSB_CUDA_OK(cudaMemsetAsync(r.transmittance_sum, 0, size_t(P) * sizeof(float), stream));
	}
	const BinPlan plan = make_bin_plan(P, W, H, scene->quant != nullptr);
	char* geom_blob = r.geom_alloc(r.geom_user, gsb_geom_bytes(P));
	char* img_blob = r.image_alloc(r.image_user, gsb_image_bytes_for(P, W, H, scene->quant != nullptr));
	if (!geom_blob || !img_blob) { set_error("forward: scratch allocation failed"); return GSB_ENOMEM; }
	GeomState g = GeomState::carve(geom_blob, P);
	ImageState img = ImageState::carve(img_blob, W, H, nullptr, plan.priv ? plan.ctas : 0);
	GSB_CUDA_OK(cudaMemsetAsync(g.counters, 0, 16 * sizeof(uint32_t), stream));
	if (!plan.priv) GSB_CUDA_OK(cudaMemsetAsync(img.tile_count, 0, ImageState::tiles(W, H) * sizeof(uint32_t), stream));
	if (int e = launch_preprocess(r, g, img, plan)) return e;
	if (int e = launch_tile_scan(img, g, plan, W, H, stream)) return e;

	// The instance count R sizes the binning blob (rasterizer_impl.cu:445-450 reads it back and stalls the device meanwhile).
	// Here it travels to the host in the background (32 bytes: R, error flags, large-tile class sizes) while the scatter and the
	// per-tile sort are ALREADY queued behind it, carved for the capacity recent frames needed; the host then waits for the
	// copy's event only — the stream keeps running — and re-launches in the rare case that R outgrew the speculation.
	int dev = 0;
	GSB_CUDA_OK(cudaGetDevice(&dev));
	HostSide& hs = t_host[dev];
	if (!hs.counters) GSB_CUDA_OK(cudaMallocHost(&hs.counters, 16 * sizeof(uint32_t)));
	if (!hs.arrived) GSB_CUDA_OK(cudaEventCreateWithFlags(&hs.arrived, cudaEventDisableTiming));
	GSB_CUDA_OK(cudaMemcpyAsync(hs.counters, g.counters, 8 * sizeof(uint32_t), cudaMemcpyDeviceToHost, stream));
	GSB_CUDA_OK(cudaEventRecord(hs.arrived, stream));
	long long cap = hs.r_hint > 0 ? hs.r_hint + hs.r_hint / 16 + 4096 : 0;
	if (cap > 0x7fffffffll) cap = 0x7fffffffll;
	BinningState b{};
	if (cap > 0)
	{
		char* bin_blob = r.binning_alloc(r.binning_user, gsb_binning_bytes(cap));
		if (!bin_blob) { set_error("forward: binning allocation failed"); return GSB_ENOMEM; }
		b = BinningState::carve(bin_blob, cap);
		if (int e = launch_scatter_sort(g, b, img, plan, P, cap, W, H, stream)) return e;
	}
	GSB_CUDA_OK(cudaEventSynchronize(hs.arrived));
	const uint32_t* hc = hs.counters;
	if (hc[3]) { set_error("forward: Point is filtered although prefiltered is set. This shouldn't happen!"); return GSB_ECUDA; }
	if (hc[6]) { set_error("forward: the (Gaussian, tile) instance count does not fit 31 bits"); return GSB_ERANGE; }
	const long long R = hc[0];
	if (R > hs.r_hint || 2 * R < hs.r_hint) hs.r_hint = R;       // grows with the workload, restarts when a much smaller one begins
	*r.num_rendered = R;
	if (cap == 0 || R > cap)
	{
		// first frame of this thread on this device, or more instances than speculated (the guarded kernels above did nothing)
		char* bin_blob = r.binning_alloc(r.binning_user, gsb_binning_bytes(R));
		if (!bin_blob) { set_error("forward: binning allocation failed"); return GSB_ENOMEM; }
		b = BinningState::carve(bin_blob, R);
		if (int e = launch_scatter_sort(g, b, img, plan, P, R, W, H, stream)) return e;
	}
	if (R > 0) if (int e = launch_sort_large(g, b, img, W, H, hc[4], hc[5], stream)) return e;
	if (int e = launch_render_forward(r, img, b, g)) return e;
	if (stats_fixed(r)) if (int e = launch_stats_fixed_to_float(P, transmittance_fixed(r), r.transmittance_sum, stream)) return e;
	return r.features ? launch_features_forward(img, b, g, W, H, *r.features, stream) : GSB_OK;
}

size_t gsb_statistics_workspace_bytes(int32_t P) { return (P > 0 ? size_t(P) * sizeof(unsigned long long) : 0) + 256; }

int gsb_sh_statistics_update(int32_t P, int32_t M, const int32_t* degrees, const float* means3D, const float* campos, const float* shs,
	const int32_t* radii, const int32_t* touched_pixels, const float* transmittance_sum, float* weight_sum, float* weight_sq_sum,
	float* distance_accum, float* mean, float* variance, void* stream)
{
	if (P < 0 || M < 16) { set_error("sh_statistics_update: needs P >= 0 and the full 16-coefficient SH layout (max_sh_degree 3)"); return GSB_EINVAL; }
	if (P > 0 && (!degrees || !means3D || !campos || !shs || !radii || !touched_pixels || !transmittance_sum || !weight_sum || !weight_sq_sum ||
		!distance_accum || !mean || !variance)) { set_error("sh_statistics_update: NULL argument"); return GSB_EINVAL; }
	return launch_sh_stats_update(P, M, degrees, means3D, campos, shs, radii, touched_pixels, transmittance_sum, weight_sum, weight_sq_sum,
		distance_accum, mean, variance, (cudaStream_t)stream);
}

int gsb_min_projected_pixel_size(int32_t P, const float* means3D, int32_t n_cameras, const float* w2ndc, const float* w2ndc_inverse,
	const int32_t* image_heights, const int32_t* image_widths, float* pixel_sizes, void* stream)
{
	if (P < 0 || n_cameras < 0) { set_error("min_projected_pixel_size: negative size"); return GSB_EINVAL; }
	if (P > 0 && (!means3D || !pixel_sizes || (n_cameras > 0 && (!w2ndc || !w2ndc_inverse || !image_heights || !image_widths))))
	{ set_error("min_projected_pixel_size: NULL argument"); return GSB_EINVAL; }
	return launch_pixel_size(P, means3D, n_cameras, w2ndc, w2ndc_inverse, image_heights, image_widths, pixel_sizes, (cudaStream_t)stream);
}

size_t gsb_filter_3d_workspace_bytes(void) { return 256; }

int gsb_filter_3d(int32_t P, const float* means3D, int32_t n_cameras, const float* viewmatrices, const float* focals, const int32_t* sizes,
	float* filter, void* workspace, void* stream)
{
	if (!rows_ok("filter_3d", P)) return GSB_EINVAL;
	if (n_cameras < 0) { set_error("filter_3d: n_cameras < 0"); return GSB_EINVAL; }
	if (P == 0) return GSB_OK;
	if (!means3D || !filter || !workspace || (n_cameras > 0 && (!viewmatrices || !focals || !sizes)))
	{ set_error("filter_3d: NULL argument"); return GSB_EINVAL; }
	return launch_filter_3d(P, means3D, n_cameras, viewmatrices, focals, sizes, filter, static_cast<unsigned*>(workspace), (cudaStream_t)stream);
}

int gsb_sphere_ellipsoid_intersection(int32_t P, const float* means3D, const float* scales, const float* rotations, const int32_t* neighbours,
	const float* sphere_radius, int32_t knn, int32_t* redundancy_values, uint8_t* intersection_mask, void* stream)
{
	if (P < 0 || knn < 0) { set_error("sphere_ellipsoid_intersection: negative size"); return GSB_EINVAL; }
	if (P > 0 && (!means3D || !scales || !rotations || !sphere_radius || !redundancy_values || (knn > 0 && (!neighbours || !intersection_mask))))
	{ set_error("sphere_ellipsoid_intersection: NULL argument"); return GSB_EINVAL; }
	return launch_sphere_ellipsoid(P, means3D, scales, rotations, neighbours, sphere_radius, knn, redundancy_values, intersection_mask, (cudaStream_t)stream);
}

int64_t gsb_l1_ssim_blocks(int32_t channels, int32_t height, int32_t width)
{
	return (int64_t)channels * ((height + 15) / 16) * ((width + 15) / 16);
}

int gsb_l1_ssim_forward(const float* image, const float* gt, int32_t channels, int32_t height, int32_t width, float* maps, float* partial_sums,
	void* stream)
{
	if (channels <= 0 || height <= 0 || width <= 0 || !image || !gt || !maps || !partial_sums) { set_error("l1_ssim_forward: bad arguments"); return GSB_EINVAL; }
	return launch_l1_ssim_forward(image, gt, channels, height, width, maps, partial_sums, (cudaStream_t)stream);
}

int gsb_l1_ssim_backward(const float* image, const float* gt, int32_t channels, int32_t height, int32_t width, const float* maps,
	float coef_l1, const float* upstream_l1, float coef_ssim, const float* upstream_ssim, float* dL_dimage, void* stream)
{
	if (channels <= 0 || height <= 0 || width <= 0 || !image || !gt || !maps || !dL_dimage) { set_error("l1_ssim_backward: bad arguments"); return GSB_EINVAL; }
	return launch_l1_ssim_backward(image, gt, channels, height, width, maps, coef_l1, upstream_l1, coef_ssim, upstream_ssim, dL_dimage,
		(cudaStream_t)stream);
}

size_t gsb_kmeans_workspace_bytes(int64_t n_values, int32_t n_centers, int32_t deterministic)
{
	return kmeans_workspace_bytes(n_values, n_centers, deterministic != 0);
}

int gsb_kmeans(const float* values, int64_t n_values, const float* centers_in, int32_t n_centers, float tol, int32_t max_iterations,
	int32_t deterministic, int32_t* ids, float* centers_out, char* workspace, void* stream)
{
	if (n_values < 0 || n_centers <= 0 || max_iterations < 0) { set_error("kmeans: bad sizes"); return GSB_EINVAL; }
	if (!centers_in || !centers_out || (n_values > 0 && (!values || !ids || !workspace))) { set_error("kmeans: NULL argument"); return GSB_EINVAL; }
	if (deterministic && (reinterpret_cast<uintptr_t>(workspace) & 15)) { set_error("kmeans: workspace is not 16-byte aligned"); return GSB_EINVAL; }
	if (n_values >= (1ll << 30)) { set_error("kmeans: 2^30 or more values (the look-back descriptors carry 30-bit counts)"); return GSB_ERANGE; }
	return launch_kmeans(values, n_values, centers_in, n_centers, tol, max_iterations, ids, centers_out, workspace, deterministic != 0,
		(cudaStream_t)stream);
}

size_t gsb_knn_workspace_bytes(int32_t P, int32_t n_queries) { return knn_workspace_bytes(P < 0 ? 0 : P, n_queries); }

int gsb_knn(const float* points, int32_t P, int32_t K, const int32_t* query_ids, int32_t n_queries, const int32_t* candidate_ids,
	int32_t n_candidates, float* mean3, float* dists, int32_t* indices, char* workspace, void* stream)
{
	if (P < 0) { set_error("knn: P < 0"); return GSB_EINVAL; }
	if (K < 0) { set_error("knn: K < 0"); return GSB_EINVAL; }
	if (K > GSB_KNN_MAX_K) { set_error("knn: K = %d is above the supported maximum of %d neighbours", K, GSB_KNN_MAX_K); return GSB_EINVAL; }
	if (mean3 && K != 3) { set_error("knn: the mean of the 3 nearest needs K == 3 (got %d)", K); return GSB_EINVAL; }
	if (P >= (1 << 30) || n_queries >= (1 << 30))
	{ set_error("knn: 2^30 or more points or queries (the sort's look-back descriptors carry 30-bit counts)"); return GSB_ERANGE; }
	const long long rows = n_queries < 0 ? P : n_queries;
	if (rows == 0 || K == 0) return GSB_OK;
	if (n_queries >= 0 && !query_ids) { set_error("knn: query_ids is NULL"); return GSB_EINVAL; }
	if (n_candidates > 0 && !candidate_ids) { set_error("knn: candidate_ids is NULL"); return GSB_EINVAL; }
	if (!mean3 && !dists && !indices) { set_error("knn: no output"); return GSB_EINVAL; }
	if (P > 0 && (!points || !workspace)) { set_error("knn: NULL points / workspace"); return GSB_EINVAL; }
	return launch_knn(points, P, K, n_queries < 0 ? nullptr : query_ids, rows, candidate_ids, n_candidates, mean3, dists, indices, workspace,
		(cudaStream_t)stream);
}

int gsb_min_redundancy_value(int32_t P, const int32_t* redundancy_values, const int32_t* neighbours, const uint8_t* intersection_mask,
	int32_t knn, int32_t* minimum_redundancy_values, void* stream)
{
	if (P < 0 || knn < 0) { set_error("min_redundancy_value: negative size"); return GSB_EINVAL; }
	if (P > 0 && (!redundancy_values || !minimum_redundancy_values || (knn > 0 && (!neighbours || !intersection_mask))))
	{ set_error("min_redundancy_value: NULL argument"); return GSB_EINVAL; }
	return launch_min_redundancy(P, redundancy_values, neighbours, intersection_mask, knn, minimum_redundancy_values, (cudaStream_t)stream);
}

int gsb_backward(const GsbBackwardRequest* req)
{
	if (!req) { set_error("backward: request is NULL"); return GSB_EINVAL; }
	const GsbBackwardRequest& r = *req;
	if (int e = check_backward(r)) return e;
	const cudaStream_t stream = stream_of(r);
	const int P = r.scene->P, W = r.cam->width, H = r.cam->height;
	if (P == 0)
	{
		// no Gaussian, no camera gradient (the camera outputs are always written, also in accumulate mode)
		if (r.dL_dviewmatrix) GSB_CUDA_OK(cudaMemsetAsync(r.dL_dviewmatrix, 0, 16 * sizeof(float), stream));
		if (r.dL_dprojmatrix) GSB_CUDA_OK(cudaMemsetAsync(r.dL_dprojmatrix, 0, 16 * sizeof(float), stream));
		if (r.dL_dcampos) GSB_CUDA_OK(cudaMemsetAsync(r.dL_dcampos, 0, 3 * sizeof(float), stream));
		return GSB_OK;
	}
	GeomState g = GeomState::carve(const_cast<char*>(r.geom_blob), P);
	ImageState img = ImageState::carve(const_cast<char*>(r.image_blob), W, H);
	BinningState b = BinningState::carve(const_cast<char*>(r.binning_blob), r.num_rendered);
	float* acc = reinterpret_cast<float*>(const_cast<char*>(r.geom_blob) + geom_state_bytes(P));
	if (int e = r.deterministic ? launch_render_backward_deterministic(r, img, b, g, acc) : launch_render_backward(r, img, b, g, acc, nullptr, nullptr))
		return e;
	if (r.features) if (int e = launch_features_backward(img, b, g, P, W, H, *r.features, acc, stream)) return e;
	if (int e = launch_preprocess_backward(r, g, acc)) return e;
	if (r.dL_dmeans2D_abs) if (int e = launch_absgrad_finish(r, acc)) return e;
	if (want_cam(r))
		if (int e = launch_camera_grad_finish(P, reinterpret_cast<float*>(r.camera_workspace), r.dL_dviewmatrix, r.dL_dprojmatrix, r.dL_dcampos,
			stream)) return e;
	return GSB_OK;
}

size_t gsb_camera_grad_workspace_bytes(int32_t P) { return camera_grad_workspace_bytes(P); }
size_t gsb_deterministic_workspace_bytes(int32_t P, int64_t num_rendered, int32_t absgrad)
{
	return det_workspace_bytes(P, num_rendered, absgrad ? DET_NS_ABS : 10);
}

int gsb_mark_visible(int32_t P, const float* means3D, const float* viewmatrix, const float* projmatrix, uint8_t* present, void* stream)
{
	(void)projmatrix;
	if (P < 0 || (P > 0 && (!means3D || !viewmatrix || !present))) { set_error("mark_visible: bad arguments"); return GSB_EINVAL; }
	return launch_mark_visible(P, means3D, viewmatrix, present, (cudaStream_t)stream);
}

int gsb_debug_dequant(const GsbQuant* quant, int32_t P, float* scales, float* rotations, void* stream)
{
	if (!quant || !scales || !rotations) { set_error("gsb_debug_dequant: NULL argument"); return GSB_EINVAL; }
	return launch_debug_dequant(quant, P, scales, rotations, (cudaStream_t)stream);
}

int gsb_export_binning(const char* geom_blob, int32_t P, const char* binning_blob, int64_t R, const char* image_blob, int32_t W, int32_t H,
	uint64_t* keys_sorted, uint32_t* point_list, void* stream)
{
	if (R <= 0) return GSB_OK;
	GeomState g = GeomState::carve(const_cast<char*>(geom_blob), P);
	BinningState b = BinningState::carve(const_cast<char*>(binning_blob), R);
	ImageState img = ImageState::carve(const_cast<char*>(image_blob), W, H);
	return launch_export_binning(g, b, img, W, H, keys_sorted, point_list, (cudaStream_t)stream);
}

size_t gsb_contributions_workspace_bytes(int32_t P) { return (P > 0 ? size_t(P) * sizeof(unsigned long long) : 0) + 256; }

// Every refusal of gsb_contributions, before any CUDA call (the order of include/gs_b200.h).
static int check_contributions(const char* geom_blob, int P, const char* binning_blob, long long R, const char* image_blob, int W, int H,
	const float* weight_sum, const float* weight_max, const int32_t* pixels, const int32_t* top_id, const void* workspace)
{
	if (P < 0 || R < 0) { set_error("contributions: negative size (P = %d, num_rendered = %lld)", P, R); return GSB_EINVAL; }
	if (W <= 0 || H <= 0) { set_error("contributions: bad image size %dx%d", W, H); return GSB_EINVAL; }
	if ((long long)W * H >= (1ll << 28))
	{ set_error("contributions: %d x %d pixels; the 64-bit fixed-point sums need W * H < 2^28", W, H); return GSB_ERANGE; }
	if (!top_id || (P > 0 && (!weight_sum || !weight_max || !pixels))) { set_error("contributions: an output is NULL"); return GSB_EINVAL; }
	if ((P > 0 || R > 0) && (!geom_blob || !binning_blob || !image_blob)) { set_error("contributions: a blob is NULL"); return GSB_EINVAL; }
	if (P > 0 && (!workspace || (reinterpret_cast<uintptr_t>(workspace) & 7)))
	{ set_error("contributions: the workspace is NULL or not 8-byte aligned"); return GSB_EINVAL; }
	return GSB_OK;
}

int gsb_contributions(const char* geom_blob, int32_t P, const char* binning_blob, int64_t R, const char* image_blob, int32_t W, int32_t H,
	const float* pixel_weights, float* weight_sum, float* weight_max, int32_t* pixels, int32_t* top_id, void* workspace, void* stream)
{
	if (int e = check_contributions(geom_blob, P, binning_blob, R, image_blob, W, H, weight_sum, weight_max, pixels, top_id, workspace))
		return e;
	GeomState g{}; BinningState b{}; ImageState img{};
	if (P > 0 && R > 0)
	{
		g = GeomState::carve(const_cast<char*>(geom_blob), P);
		b = BinningState::carve(const_cast<char*>(binning_blob), R);
		img = ImageState::carve(const_cast<char*>(image_blob), W, H);
	}
	return launch_contributions(g, b, img, P, R, W, H, pixel_weights, weight_sum, weight_max, pixels, top_id,
		static_cast<unsigned long long*>(workspace), (cudaStream_t)stream);
}

int gsb_export_image(const char* image_blob, int32_t W, int32_t H, float* final_T, uint32_t* n_contrib, uint32_t* ranges, void* stream_)
{
	cudaStream_t stream = (cudaStream_t)stream_;
	ImageState img = ImageState::carve(const_cast<char*>(image_blob), W, H);
	const size_t N = size_t(W) * H, T = ImageState::tiles(W, H);
	if (final_T) GSB_CUDA_OK(cudaMemcpyAsync(final_T, img.final_T, N * 4, cudaMemcpyDeviceToDevice, stream));
	if (n_contrib) GSB_CUDA_OK(cudaMemcpyAsync(n_contrib, img.n_contrib, N * 4, cudaMemcpyDeviceToDevice, stream));
	if (ranges) GSB_CUDA_OK(cudaMemcpyAsync(ranges, img.ranges, T * 8, cudaMemcpyDeviceToDevice, stream));
	return GSB_OK;
}

// [P, K] int32 neighbour indices, then the kNN's own workspace
static size_t redundancy_knn_offset(int P, int K) { return ((size_t)P * K * sizeof(int32_t) + 255) & ~size_t(255); }

size_t gsb_redundancy_workspace_bytes(int32_t P, int32_t K)
{
	const int p = P < 0 ? 0 : P, k = K < 0 ? 0 : K;
	return redundancy_knn_offset(p, k) + knn_workspace_bytes(p, -1);
}

int gsb_redundancy_score(int32_t P, const float* means3D, const float* scales, const float* rotations, int32_t n_cameras,
	const float* w2ndc, const float* w2ndc_inverse, const int32_t* image_heights, const int32_t* image_widths, float pixel_scale,
	int32_t K, int32_t* min_redundancy, float* pixel_sizes, void* workspace, void* stream)
{
	if (!rows_ok("redundancy_score", P)) return GSB_EINVAL;
	if (K < 1 || K > GSB_KNN_MAX_K) { set_error("redundancy_score: K = %d is outside 1..%d", K, GSB_KNN_MAX_K); return GSB_EINVAL; }
	if (n_cameras < 0 || n_cameras > 1024) { set_error("redundancy_score: n_cameras = %d is outside 0..1024", n_cameras); return GSB_EINVAL; }
	if (P == 0) return GSB_OK;
	if (!means3D || !scales || !rotations || !min_redundancy || !pixel_sizes || !workspace ||
		(n_cameras > 0 && (!w2ndc || !w2ndc_inverse || !image_heights || !image_widths)))
	{ set_error("redundancy_score: NULL argument"); return GSB_EINVAL; }
	const cudaStream_t st = (cudaStream_t)stream;
	int32_t* nb = static_cast<int32_t*>(workspace);
	char* knn_ws = static_cast<char*>(workspace) + redundancy_knn_offset(P, K);
	if (int e = launch_pixel_size(P, means3D, n_cameras, w2ndc, w2ndc_inverse, image_heights, image_widths, pixel_sizes, st)) return e;
	if (int e = launch_knn(means3D, P, K, nullptr, P, nullptr, -1, nullptr, nullptr, nb, knn_ws, st)) return e;
	return launch_redundancy_fused(P, means3D, scales, rotations, nb, pixel_sizes, pixel_scale, K, min_redundancy, st);
}

} // extern "C"
