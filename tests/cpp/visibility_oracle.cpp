// visibility_oracle.cpp — the exhaustive CPU restatement of Scene::PointCloudFilter (libs/MVS/SceneDensify.cpp:2226-2360) the
// tests hold the library's visibility counts and removal order against.  Built by the tests with -O2 -ffp-contract=off, so every
// float expression below is evaluated as written, one correctly rounded operation at a time.
//  - Every (point X, view v of X) cone classifies EVERY point of the cloud: the reference's octree only skips cells whose
//    circumscribed sphere misses the cone, which is conservative in exact arithmetic (DESIGN.md §8).
//  - The sums of three terms are Eigen's order for a 3-vector (Redux.h: redux_novec_unroller halves the range): a0 + (a1 + a2).
//  - The counts are the sequential build's: threads take disjoint sets of cones into their own int arrays, summed at the end.
#include <cmath>
#include <cstdint>
#include <thread>
#include <vector>

namespace {

inline float sum3(float a0, float a1, float a2) { return a0 + (a1 + a2); }

struct Collector {
	float orig[3], cosAngleSq;
};

} // namespace

extern "C" {

// K: 9 doubles per image (row-major), C: 3 doubles per image, width: per image.  visibility: n ints, overwritten.
int vis_oracle(const float* pts, uint64_t n, const uint32_t* off, const uint32_t* views, int nImages, const double* K, const double* C,
	const int* width, int threads, int32_t* visibility)
{
	std::vector<Collector> col(nImages);
	for (int i = 0; i < nImages; ++i) {
		for (int a = 0; a < 3; ++a) col[i].orig[a] = (float)C[3*i+a];
		// Image::ComputeFOV(0) (libs/MVS/Image.cpp:209-216) over width, cast to float; TConeIntersect's SQUARE(COS(angle))
		const double fov = 2*std::atan((double)width[i]/(K[9*i]*2));
		const float angle = (float)(fov/width[i]);
		const float c = std::cos(angle);
		col[i].cosAngleSq = c*c;
	}
	if (threads < 1) threads = 1;
	std::vector<std::vector<int32_t>> part(threads, std::vector<int32_t>(n, 0));
	auto work = [&](int t) {
		int32_t* vis = part[t].data();
		for (uint64_t i = t; i < n; i += threads) {
			const float* X = pts + 3*i;
			const int weight = (int)(off[i+1] - off[i]);
			for (uint32_t k = off[i]; k < off[i+1]; ++k) {
				const Collector& cl = col[views[k]];
				// Collector::Init
				const float D[3] = {X[0] - cl.orig[0], X[1] - cl.orig[1], X[2] - cl.orig[2]};
				const float distance = std::sqrt(sum3(D[0]*D[0], D[1]*D[1], D[2]*D[2]));
				const float dir[3] = {D[0]/distance, D[1]/distance, D[2]/distance};
				const float maxHeight = distance*1.02f;
				// Collector::operator() over every point
				for (uint64_t j = 0; j < n; ++j) {
					const float* P = pts + 3*j;
					const float E[3] = {P[0] - cl.orig[0], P[1] - cl.orig[1], P[2] - cl.orig[2]};
					const float dist = sum3(dir[0]*E[0], dir[1]*E[1], dir[2]*E[2]);
					// TConeIntersect::Classify (libs/Common/Ray.inl:905-920), minHeight 0
					if (std::fabs(dist) < 0.0001f) continue;   // PLANAR
					if (dist < 0.f) continue;                   // BACK
					if (dist > maxHeight) continue;             // FRONT
					const float tSq = dist*dist;
					const float dSq = cl.cosAngleSq*sum3(E[0]*E[0], E[1]*E[1], E[2]*E[2]);
					if (!(tSq > dSq)) continue;                 // CULLED or PLANAR
					// IsDepthSimilar(distance, dist, 0.01f) (libs/Common/Util.inl:797-809)
					if (std::fabs(distance - dist)/distance < 0.01f) continue;
					if (dist > distance) vis[j] += (int32_t)(off[j+1] - off[j]);
					else vis[j] -= weight;
				}
			}
		}
	};
	std::vector<std::thread> pool;
	for (int t = 1; t < threads; ++t) pool.emplace_back(work, t);
	work(0);
	for (std::thread& th: pool) th.join();
	for (uint64_t j = 0; j < n; ++j) {
		int32_t s = 0;
		for (int t = 0; t < threads; ++t) s += part[t][j];
		visibility[j] = s;
	}
	return 0;
}

// The reference's removal loop, literally: RFOREACH(idxPoint, points) if (visibility[idxPoint] <= thRemove) RemovePoint(idxPoint),
// on an array of original indices; RemovePoint is cList::RemoveAt (libs/Common/List.h:1129-1136).  -> the number kept; order holds
// the kept original indices in their final slots.
uint64_t vis_oracle_filter(const int32_t* visibility, uint64_t n, int thRemove, uint32_t* order) {
	std::vector<uint32_t> points(n);
	for (uint64_t i = 0; i < n; ++i) points[i] = (uint32_t)i;
	uint64_t size = n;
	for (uint64_t idxPoint = size; idxPoint-- > 0; ) {
		if (visibility[idxPoint] <= thRemove) {
			if (idxPoint+1 == size) --size;                       // RemoveLast
			else points[idxPoint] = points[--size];               // _ArrayMoveCopy of the last element
		}
	}
	for (uint64_t i = 0; i < size; ++i) order[i] = points[i];
	return size;
}

} // extern "C"
