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
static const char* kKernelNames[K_COUNT] = { "preprocess", "tile_scan", "scatter", "tile_sort_large", "unused4", "tile_sort", "unused6",
	"render_forward", "render_backward", "preprocess_backward", "mark_visible", "tools", "kmeans", "knn" };

int launch_debug_dequant(const GsbQuant*, int, float*, float*, cudaStream_t);
int launch_preprocess(const GsbScene*, const GsbCamera*, const GeomState&, const ImageState&, const BinPlan&, int32_t*, const GsbDebug*, cudaStream_t);
int launch_mark_visible(int, const float*, const float*, uint8_t*, cudaStream_t);
int launch_tile_scan(const ImageState&, const GeomState&, const BinPlan&, int, int, cudaStream_t);
int launch_scatter_sort(const GeomState&, const BinningState&, const ImageState&, const BinPlan&, int, long long, int, int, cudaStream_t);
int launch_sort_large(const GeomState&, const BinningState&, const ImageState&, int, int, uint32_t, uint32_t, cudaStream_t);
int launch_export_binning(const GeomState&, const BinningState&, const ImageState&, int, int, uint64_t*, uint32_t*, cudaStream_t);
int launch_render_forward(const ImageState&, const BinningState&, const GeomState&, int, int, const float*, float*, int32_t*, float*, cudaStream_t);
int launch_sh_stats_update(int, int, const int*, const float*, const float*, const float*, const int*, const int*, const float*, float*, float*,
	float*, float*, float*, cudaStream_t);
int launch_pixel_size(int, const float*, int, const float*, const float*, const int*, const int*, float*, cudaStream_t);
int launch_sphere_ellipsoid(int, const float*, const float*, const float*, const int*, const float*, int, int*, uint8_t*, cudaStream_t);
int launch_min_redundancy(int, const int*, const int*, const uint8_t*, int, int*, cudaStream_t);
int launch_l1_ssim_forward(const float*, const float*, int, int, int, float*, float*, cudaStream_t);
int launch_l1_ssim_backward(const float*, const float*, int, int, int, const float*, float, const float*, float, const float*, float*, cudaStream_t);
size_t kmeans_workspace_bytes(long long, int);
int launch_kmeans(const float*, long long, const float*, int, float, int, int*, float*, char*, cudaStream_t);
size_t knn_workspace_bytes(long long, long long);
int launch_knn(const float*, long long, int, const int32_t*, long long, const int32_t*, long long, float*, float*, int32_t*, char*, cudaStream_t);
int launch_render_backward(const ImageState&, const BinningState&, const GeomState&, int, int, int, const float*, const float*, float*, cudaStream_t);
int launch_preprocess_backward(const GsbScene*, const GsbCamera*, const GeomState&, const int32_t*, const float*, const GsbGrads*, float, cudaStream_t);

// geometry blob = GeomState followed by the backward's gradient accumulator (12 floats per Gaussian)
static size_t geom_state_bytes(int P) { size_t b; GeomState::carve(nullptr, P, &b); return (b + 255) & ~size_t(255); }

static int check_scene(const GsbScene* s, const GsbCamera* c)
{
	if (!s || !c) { set_error("scene / camera is NULL"); return GSB_EINVAL; }
	if (s->P < 0) { set_error("P < 0"); return GSB_EINVAL; }
	if (c->width <= 0 || c->height <= 0) { set_error("bad image size %dx%d", c->width, c->height); return GSB_EINVAL; }
	if (!c->viewmatrix || !c->projmatrix || !c->campos || !c->background) { set_error("camera tensors missing"); return GSB_EINVAL; }
	if (s->P == 0) return GSB_OK;
	if (!s->means3D) { set_error("means3D missing"); return GSB_EINVAL; }
	if (s->quant)
	{
		const GsbQuant* q = s->quant;
		if (!q->ids_dc || !q->ids_rest || !q->ids_opacity || !q->ids_scaling || !q->ids_rot || !q->centers || !s->degrees)
		{ set_error("quantised scene: id planes / centres / degrees missing"); return GSB_EINVAL; }
		if (s->M != 16) { set_error("quantised scene needs M == 16"); return GSB_EINVAL; }
		return GSB_OK;
	}
	if (!s->opacities) { set_error("opacities missing"); return GSB_EINVAL; }
	// diff_gaussian_rasterization/__init__.py:203-207
	if ((s->shs == nullptr) == (s->colors_precomp == nullptr)) { set_error("Please provide excatly one of either SHs or precomputed colors!"); return GSB_EINVAL; }
	const bool sr = s->scales != nullptr && s->rotations != nullptr;
	if (sr == (s->cov3D_precomp != nullptr) || ((s->scales != nullptr) != (s->rotations != nullptr)))
	{ set_error("Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!"); return GSB_EINVAL; }
	if (s->shs && !s->sh_packed && (!s->degrees || s->M <= 0)) { set_error("dense SH needs degrees and M > 0"); return GSB_EINVAL; }
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
const char* gsb_version(void) { return "gs_b200 0.1 (sm_90a)"; }

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

static int forward_impl(const GsbScene* scene, const GsbCamera* cam, gsb_alloc_fn geom_alloc, void* geom_user,
	gsb_alloc_fn binning_alloc, void* binning_user, gsb_alloc_fn image_alloc, void* image_user,
	float* out_color, int32_t* radii, int64_t* num_rendered, const GsbDebug* debug, int32_t* touched_pixels, float* transmittance,
	void* stream_)
{
	cudaStream_t stream = (cudaStream_t)stream_;
	if (int e = check_scene(scene, cam)) return e;
	if (!out_color || !num_rendered || (scene->P > 0 && !radii)) { set_error("output pointers missing"); return GSB_EINVAL; }
	*num_rendered = 0;
	const int P = scene->P, W = cam->width, H = cam->height;
	const size_t N = size_t(W) * H;
	if (P == 0)
	{
		// rasterize_points.cu:170,184-185: P == 0 returns the zero-initialised image (no background)
		GSB_CUDA_OK(cudaMemsetAsync(out_color, 0, 3 * N * sizeof(float), stream));
		return GSB_OK;
	}
	const BinPlan plan = make_bin_plan(P, W, H, scene->quant != nullptr);
	char* geom_blob = geom_alloc(geom_user, gsb_geom_bytes(P));
	char* img_blob = image_alloc(image_user, gsb_image_bytes_for(P, W, H, scene->quant != nullptr));
	if (!geom_blob || !img_blob) { set_error("scratch allocation failed"); return GSB_ENOMEM; }
	GeomState g = GeomState::carve(geom_blob, P);
	ImageState img = ImageState::carve(img_blob, W, H, nullptr, plan.priv ? plan.ctas : 0);
	GSB_CUDA_OK(cudaMemsetAsync(g.counters, 0, 16 * sizeof(uint32_t), stream));
	if (!plan.priv) GSB_CUDA_OK(cudaMemsetAsync(img.tile_count, 0, ImageState::tiles(W, H) * sizeof(uint32_t), stream));
	if (int e = launch_preprocess(scene, cam, g, img, plan, radii, debug, stream)) return e;
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
		char* bin_blob = binning_alloc(binning_user, gsb_binning_bytes(cap));
		if (!bin_blob) { set_error("binning allocation failed"); return GSB_ENOMEM; }
		b = BinningState::carve(bin_blob, cap);
		if (int e = launch_scatter_sort(g, b, img, plan, P, cap, W, H, stream)) return e;
	}
	GSB_CUDA_OK(cudaEventSynchronize(hs.arrived));
	const uint32_t* hc = hs.counters;
	if (hc[3]) { set_error("Point is filtered although prefiltered is set. This shouldn't happen!"); return GSB_ECUDA; }
	if (hc[6]) { set_error("the (Gaussian, tile) instance count does not fit 31 bits"); return GSB_ERANGE; }
	const long long R = hc[0];
	if (R > hs.r_hint || 2 * R < hs.r_hint) hs.r_hint = R;       // grows with the workload, restarts when a much smaller one begins
	*num_rendered = R;
	if (cap == 0 || R > cap)
	{
		// first frame of this thread on this device, or more instances than speculated (the guarded kernels above did nothing)
		char* bin_blob = binning_alloc(binning_user, gsb_binning_bytes(R));
		if (!bin_blob) { set_error("binning allocation failed"); return GSB_ENOMEM; }
		b = BinningState::carve(bin_blob, R);
		if (int e = launch_scatter_sort(g, b, img, plan, P, R, W, H, stream)) return e;
	}
	if (R > 0) if (int e = launch_sort_large(g, b, img, W, H, hc[4], hc[5], stream)) return e;
	if (int e = launch_render_forward(img, b, g, W, H, cam->background, out_color, touched_pixels, transmittance, stream)) return e;
	return GSB_OK;
}

int gsb_forward(const GsbScene* scene, const GsbCamera* cam, gsb_alloc_fn geom_alloc, void* geom_user,
	gsb_alloc_fn binning_alloc, void* binning_user, gsb_alloc_fn image_alloc, void* image_user,
	float* out_color, int32_t* radii, int64_t* num_rendered, const GsbDebug* debug, void* stream)
{
	return forward_impl(scene, cam, geom_alloc, geom_user, binning_alloc, binning_user, image_alloc, image_user, out_color, radii,
		num_rendered, debug, nullptr, nullptr, stream);
}

int gsb_forward_statistics(const GsbScene* scene, const GsbCamera* cam, gsb_alloc_fn geom_alloc, void* geom_user,
	gsb_alloc_fn binning_alloc, void* binning_user, gsb_alloc_fn image_alloc, void* image_user,
	float* out_color, int32_t* radii, int64_t* num_rendered, int32_t* touched_pixels, float* transmittance_sum, void* stream)
{
	if (!scene || scene->P < 0) { set_error("scene is NULL"); return GSB_EINVAL; }
	if (scene->P > 0 && (!touched_pixels || !transmittance_sum)) { set_error("statistics output pointers missing"); return GSB_EINVAL; }
	if (scene->P > 0)
	{
		// reduced_3dgs.cu:117-118: both statistics start from zero for every camera
		GSB_CUDA_OK(cudaMemsetAsync(touched_pixels, 0, size_t(scene->P) * sizeof(int32_t), (cudaStream_t)stream));
		GSB_CUDA_OK(cudaMemsetAsync(transmittance_sum, 0, size_t(scene->P) * sizeof(float), (cudaStream_t)stream));
	}
	return forward_impl(scene, cam, geom_alloc, geom_user, binning_alloc, binning_user, image_alloc, image_user, out_color, radii,
		num_rendered, nullptr, touched_pixels, transmittance_sum, stream);
}

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

size_t gsb_kmeans_workspace_bytes(int64_t n_values, int32_t n_centers) { return kmeans_workspace_bytes(n_values, n_centers); }

int gsb_kmeans(const float* values, int64_t n_values, const float* centers_in, int32_t n_centers, float tol, int32_t max_iterations,
	int32_t* ids, float* centers_out, char* workspace, void* stream)
{
	if (n_values < 0 || n_centers <= 0 || max_iterations < 0) { set_error("kmeans: bad sizes"); return GSB_EINVAL; }
	if (!centers_in || !centers_out || (n_values > 0 && (!values || !ids || !workspace))) { set_error("kmeans: NULL argument"); return GSB_EINVAL; }
	if (n_values >= (1ll << 30)) { set_error("kmeans: 2^30 or more values (the look-back descriptors carry 30-bit counts)"); return GSB_ERANGE; }
	return launch_kmeans(values, n_values, centers_in, n_centers, tol, max_iterations, ids, centers_out, workspace, (cudaStream_t)stream);
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

int gsb_backward(const GsbScene* scene, const GsbCamera* cam, int64_t R, const int32_t* radii,
	const char* geom_blob, const char* binning_blob, const char* image_blob, const float* dL_dout_color,
	const GsbGrads* grads, float lambda_sh_sparsity, void* stream_)
{
	cudaStream_t stream = (cudaStream_t)stream_;
	if (int e = check_scene(scene, cam)) return e;
	if (!grads) { set_error("grads is NULL"); return GSB_EINVAL; }
	const int P = scene->P, W = cam->width, H = cam->height;
	if (P == 0) return GSB_OK;
	if (!geom_blob || !binning_blob || !image_blob || !dL_dout_color || !radii) { set_error("backward inputs missing"); return GSB_EINVAL; }
	if (!grads->dL_dmeans2D || !grads->dL_dcolors || !grads->dL_dopacity || !grads->dL_dmeans3D || !grads->dL_dcov3D ||
		!grads->dL_dscales || !grads->dL_drotations || (scene->M > 0 && !grads->dL_dsh))
	{ set_error("gradient output pointers missing"); return GSB_EINVAL; }
	GeomState g = GeomState::carve(const_cast<char*>(geom_blob), P);
	ImageState img = ImageState::carve(const_cast<char*>(image_blob), W, H);
	BinningState b = BinningState::carve(const_cast<char*>(binning_blob), R);
	float* acc = reinterpret_cast<float*>(const_cast<char*>(geom_blob) + geom_state_bytes(P));
	if (int e = launch_render_backward(img, b, g, P, W, H, cam->background, dL_dout_color, acc, stream)) return e;
	if (int e = launch_preprocess_backward(scene, cam, g, radii, acc, grads, lambda_sh_sparsity, stream)) return e;
	return GSB_OK;
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

int gsb_export_image(const char* image_blob, int32_t W, int32_t H, float* final_T, uint32_t* n_contrib, uint32_t* ranges, void* stream_)
{
	cudaStream_t stream = (cudaStream_t)stream_;
	ImageState img = ImageState::carve(const_cast<char*>(image_blob), W, H);
	const size_t N = size_t(W) * H, T = size_t((W + 15) / 16) * ((H + 15) / 16);
	if (final_T) GSB_CUDA_OK(cudaMemcpyAsync(final_T, img.final_T, N * 4, cudaMemcpyDeviceToDevice, stream));
	if (n_contrib) GSB_CUDA_OK(cudaMemcpyAsync(n_contrib, img.n_contrib, N * 4, cudaMemcpyDeviceToDevice, stream));
	if (ranges) GSB_CUDA_OK(cudaMemcpyAsync(ranges, img.ranges, T * 8, cudaMemcpyDeviceToDevice, stream));
	return GSB_OK;
}

} // extern "C"
