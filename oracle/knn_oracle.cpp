// knn_oracle.cpp — brute-force CPU oracle of the k nearest neighbours (the reference's simple_knn._C: distCUDA2, distIndex2,
// distIndexQ).  TEST INFRASTRUCTURE ONLY.  Compiled with -ffp-contract=off so that the only fused multiply-adds are the explicit
// fmaf calls: the distance is the reference's SASS sequence FADD x3; FMUL dy,dy; FFMA dx,dx,.; FFMA dz,dz,. (simple_knn.cu:137,
// :400 as its sm_90 build evaluates them: y first).
//
// Every row lists its K smallest (distance, index) pairs in that order; a candidate at a distance >= FLT_MAX (or NaN) never counts
// (the reference's `dist >= reject` with reject starting at FLT_MAX), so missing neighbours are (FLT_MAX, -1).  The query itself
// is excluded by index, not by value.  The reference's visiting order is not restated: the set of the K smallest distances does not
// depend on it, only which of several candidates tied at the K-th distance is kept.
#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>

#define KO_API extern "C" __attribute__((visibility("default")))

static inline float ko_dist(const float* p, const float* q)
{
	const float dx = p[0] - q[0], dy = p[1] - q[1], dz = p[2] - q[2];
	return fmaf(dz, dz, fmaf(dx, dx, dy * dy));
}

// n_queries < 0: every point is a query (row i = point i); else row t = query_ids[t] (ids outside [0, P) give an empty row).
// n_candidates < 0: every point is a candidate; else those listed in the first min(n_candidates, P) entries of candidate_ids.
KO_API void ko_knn(const float* points, int P, int K, const int32_t* query_ids, int n_queries, const int32_t* candidate_ids, int n_candidates,
	float* dists, int32_t* indices, float* mean3)
{
	const long long rows = n_queries < 0 ? P : n_queries;
	std::vector<int32_t> cand;
	if (n_candidates < 0)
		for (int i = 0; i < P; i++) cand.push_back(i);
	else
	{
		std::vector<uint8_t> flag(P > 0 ? P : 1, 0);
		for (int i = 0; i < std::min(n_candidates, P); i++)
			if (candidate_ids[i] >= 0 && candidate_ids[i] < P) flag[candidate_ids[i]] = 1;
		for (int i = 0; i < P; i++)
			if (flag[i]) cand.push_back(i);
	}
	const uint64_t empty = ((uint64_t)0x7f7fffffu << 32) | 0xffffffffu;
#pragma omp parallel for schedule(dynamic, 64)
	for (long long r = 0; r < rows; r++)
	{
		const long long q = n_queries < 0 ? r : query_ids[r];
		std::vector<uint64_t> best(K > 0 ? K : 1, empty);
		if (q >= 0 && q < P)
			for (int c : cand)
			{
				if (c == q || K == 0) continue;
				const float d = ko_dist(points + 3 * (size_t)c, points + 3 * (size_t)q);
				uint32_t db;
				std::memcpy(&db, &d, 4);
				if (db >= 0x7f7fffffu) continue;                 // >= FLT_MAX, or NaN
				const uint64_t key = ((uint64_t)db << 32) | (uint32_t)c;
				if (key >= best[K - 1]) continue;
				int pos = K - 1;
				while (pos > 0 && best[pos - 1] > key) { best[pos] = best[pos - 1]; pos--; }
				best[pos] = key;
			}
		for (int k = 0; k < K; k++)
		{
			const uint32_t db = (uint32_t)(best[k] >> 32);
			float d;
			std::memcpy(&d, &db, 4);
			if (dists) dists[r * K + k] = d;
			if (indices) indices[r * K + k] = (int32_t)(uint32_t)best[k];
		}
		if (mean3 && K == 3)                                   // simple_knn.cu:184
		{
			float b[3];
			for (int k = 0; k < 3; k++) { const uint32_t db = (uint32_t)(best[k] >> 32); std::memcpy(&b[k], &db, 4); }
			mean3[r] = ((b[0] + b[1]) + b[2]) / 3.0f;
		}
	}
}
