// sgm_fuse_oracle.cpp — sequential restatement of fusion-mode -2 (TEST INFRASTRUCTURE, like the rest of oracle/): the pairs'
// disparity maps projected into an image and fused (SemiGlobalMatcher::ProjectDisparity2DepthMap and ::Fuse,
// libs/MVS/SemiGlobalMatcher.cpp:1925-2039 and :739-859), the Q of a reversed pair (:770-779) and EstimateNormalMap
// (libs/MVS/DepthMap.cpp:1522-1613).  Loops in the reference's order; built with -ffp-contract=off.
//
// The three places where the engine departs from the reference on purpose are restated the engine's way:
//  - rejected pixels get range and conf 0 (the reference leaves them uninitialised);
//  - a pixel whose agreeing entries have total weight 0 (0/0 in the reference) gets depth 0;
//  - a source whose projected position puts its 3x3 block outside the image is skipped before the float -> int conversion (the
//    reference writes nothing for it either, but converts the position first, which is undefined for huge values).
#include <cfloat>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>

namespace {

const int HW = 3;                 // halfWindowSizeX / Y
const int NO_DISP = 32767;

// Image::Disparity2Depth(Q, u, d) (Image.cpp:373-381)
float disparity2depth(const double* Q, int ux, int uy, float d) {
	const double w = Q[12]*ux + Q[13]*uy - Q[14]*d + Q[15];
	if (std::fabs(w) < 1e-7) return 0;
	const double z = Q[8]*ux + Q[9]*uy - Q[10]*d + Q[11];
	const float depth = (float)(z/w);
	return depth < 0.0001f ? 0.f : depth;
}

// the same, also returning the position in the image (Image.cpp:392-404)
float disparity2depth(const double* Q, int ux, int uy, float d, float& px, float& py) {
	const double w = Q[12]*ux + Q[13]*uy - Q[14]*d + Q[15];
	if (std::fabs(w) < 1e-7) return 0;
	const double z = (Q[8]*ux + Q[9]*uy - Q[10]*d + Q[11])/w;
	if (z < 1e-7) return 0;
	const double nrm = 1.0/(w*z);
	px = (float)((Q[0]*ux + Q[1]*uy - Q[2]*d + Q[3])*nrm);
	py = (float)((Q[4]*ux + Q[5]*uy - Q[6]*d + Q[7])*nrm);
	return (float)z;
}

bool depth_similar(float d0, float d1, float th) { return std::fabs(d0-d1)/d0 < th; }

} // namespace

extern "C" {

// ProjectDisparity2DepthMap of one pair into a W x H image: depth, range (2 floats per pixel), conf (nullable) -> numDepths
int oracle_sgmf_project(const int16_t* disparity, const uint16_t* cost, int vw, int vh, int steps, const double* Q, int W, int H,
	float* depth, float* range, float* conf)
{
	const size_t n = (size_t)W*H;
	struct Buf { std::vector<float> dist, depth, lo, hi, conf; } bufs[4];
	for (Buf& b: bufs) { b.dist.assign(n, 0.f); b.depth.assign(n, 0.f); b.lo.assign(n, 0.f); b.hi.assign(n, 0.f); b.conf.assign(n, 0.f); }
	const float overlapBorder = 0.5f+0.25f;
	for (int r = 0; r < vh; ++r) {
		for (int c = 0; c < vw; ++c) {
			const int dint = disparity[(size_t)r*vw+c];
			if (dint == NO_DISP) continue;
			const float d = (float)dint/(float)steps;
			const int ux = c+HW, uy = r+HW;
			float px = 0, py = 0;
			const float dep = disparity2depth(Q, ux, uy, d, px, py);
			if (dep <= 0) continue;
			const float fx = std::floor(px), fy = std::floor(py);
			if (!(fx >= -1.f && fx <= (float)W && fy >= -1.f && fy <= (float)H)) continue;
			const int dc = (int16_t)(int)std::floor(d);
			const float lo = disparity2depth(Q, ux, uy, (float)(dc-1)), hi = disparity2depth(Q, ux, uy, (float)(dc+1));
			const float cf = cost ? 1.f/(float)(cost[(size_t)r*vw+c]+1) : 0.f;
			const int x0 = (int)fx, y0 = (int)fy;
			px -= 0.5f; py -= 0.5f;
			for (int i = -1; i <= 1; ++i) {
				for (int j = -1; j <= 1; ++j) {
					const int nx = x0+j, ny = y0+i;
					if (nx < 0 || ny < 0 || nx >= W || ny >= H) continue;
					const float dx = (float)nx-px, dy = (float)ny-py;
					if (std::fabs(dx) > overlapBorder || std::fabs(dy) > overlapBorder) continue;
					Buf& b = bufs[(dx < 0 ? 1 : 0)+(dy < 0 ? 2 : 0)];
					const float dsq = dx*dx+dy*dy;
					const size_t k = (size_t)ny*W+nx;
					if (b.depth[k] > 0 && b.dist[k] <= dsq) continue;
					b.dist[k] = dsq; b.depth[k] = dep; b.lo[k] = lo; b.hi[k] = hi; b.conf[k] = cf;
				}
			}
		}
	}
	const float thDist = 0.75f*0.75f, thDepth = 0.02f;
	int numDepths = 0;
	for (size_t k = 0; k < n; ++k) {
		float distCenter = FLT_MAX, depthCenter = 0;
		for (int i = 0; i < 4; ++i) {
			if (bufs[i].depth[k] <= 0) continue;
			if (distCenter > bufs[i].dist[k]) { distCenter = bufs[i].dist[k]; depthCenter = bufs[i].depth[k]; }
		}
		float v[4] = {0, 0, 0, 0}, weight = 0;
		if (!(distCenter > thDist)) {
			for (int i = 0; i < 4; ++i) {
				const Buf& b = bufs[i];
				if (b.depth[k] <= 0 || !depth_similar(depthCenter, b.depth[k], thDepth)) continue;
				const float w = std::sqrt(b.dist[k]);
				v[0] += b.depth[k]*w; v[1] += b.lo[k]*w; v[2] += b.hi[k]*w; v[3] += b.conf[k]*w;
				weight += w;
			}
		}
		if (weight > 0) {
			const float inv = 1.f/weight;
			for (float& x: v) x = x*inv;
			++numDepths;
		} else {
			v[0] = v[1] = v[2] = v[3] = 0;
		}
		depth[k] = v[0]; range[2*k] = v[1]; range[2*k+1] = v[2];
		if (conf) conf[k] = v[3];
	}
	return numDepths;
}

// the cluster vote of Fuse (:795-848) over nPairs projected maps (pair p at offset p x W x H; ranges 2 floats per pixel)
void oracle_sgmf_fuse(int nPairs, const float* depths, const float* ranges, const float* confs, int W, int H, unsigned minViews,
	float* depth, float* conf)
{
	const size_t n = (size_t)W*H;
	struct Cluster { std::vector<int> views; float lo, hi; };
	for (size_t k = 0; k < n; ++k) {
		std::vector<Cluster> clusters;
		for (int p = 0; p < nPairs; ++p) {
			const float d = depths[p*n+k];
			if (d <= 0) continue;
			const float rlo = ranges[2*(p*n+k)], rhi = ranges[2*(p*n+k)+1];
			unsigned numClusters = 0;
			for (Cluster& cl: clusters) {
				if (!(cl.lo <= d && d < cl.hi)) continue;
				cl.views.push_back(p);
				if (cl.lo < rlo) cl.lo = rlo;
				if (cl.hi > rhi) cl.hi = rhi;
				++numClusters;
			}
			if (numClusters == 0) clusters.push_back(Cluster{{p}, rlo, rhi});
		}
		depth[k] = 0; if (conf) conf[k] = 0;
		if (clusters.empty()) continue;
		size_t best = 0;
		for (size_t i = 1; i < clusters.size(); ++i)
			if (clusters[best].views.size() < clusters[i].views.size()) best = i;
		const Cluster& cl = clusters[best];
		if (cl.views.size() < minViews) continue;
		float sd = 0, sc = 0;
		unsigned num = 0;
		for (int p: cl.views) { sd += depths[p*n+k]; sc += confs[p*n+k]; ++num; }
		depth[k] = sd/num;
		if (conf) conf[k] = sc/num;
	}
}

// Q' = P invK Q of a reversed pair (:770-779)
void oracle_sgmf_pair_q(const double* Q, const double* Kl, const double* Rl, const double* Cl, const double* K, const double* R,
	const double* C, double* Qout)
{
	double Rr[9], Cr[3], dC[3] = {C[0]-Cl[0], C[1]-Cl[1], C[2]-Cl[2]};
	for (int i = 0; i < 3; ++i) {
		for (int j = 0; j < 3; ++j) { double s = 0; for (int k = 0; k < 3; ++k) s += R[i*3+k]*Rl[j*3+k]; Rr[i*3+j] = s; }
		double s = 0; for (int k = 0; k < 3; ++k) s += Rl[i*3+k]*dC[k]; Cr[i] = s;
	}
	double P[16] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 1};
	for (int i = 0; i < 3; ++i) {
		for (int j = 0; j < 3; ++j) { double s = 0; for (int k = 0; k < 3; ++k) s += K[i*3+k]*Rr[k*3+j]; P[i*4+j] = s; }
		double s = 0; for (int k = 0; k < 3; ++k) s += P[i*4+k]*(-Cr[k]); P[i*4+3] = s;
	}
	double iK[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
	iK[0] = 1.0/Kl[0]; iK[5] = 1.0/Kl[4]; iK[2] = -Kl[2]*iK[0]; iK[6] = -Kl[5]*iK[5];
	double T[16], O[16];
	for (int i = 0; i < 4; ++i) for (int j = 0; j < 4; ++j) { double s = 0; for (int k = 0; k < 4; ++k) s += P[i*4+k]*iK[k*4+j]; T[i*4+j] = s; }
	for (int i = 0; i < 4; ++i) for (int j = 0; j < 4; ++j) { double s = 0; for (int k = 0; k < 4; ++k) s += T[i*4+k]*Q[k*4+j]; O[i*4+j] = s; }
	std::memcpy(Qout, O, sizeof(O));
}

// EstimateNormalMap(Matrix3x3f(K), depth, normal); normal: 3 floats per pixel
void oracle_sgmf_normals(const float* D, int W, int H, const double* Kd, float* N) {
	const float fx = (float)Kd[0], fy = (float)Kd[4], cx = (float)Kd[2], cy = (float)Kd[5];
	for (int r = 0; r < H; ++r) {
		for (int c = 0; c < W; ++c) {
			float* n = N+3*((size_t)r*W+c);
			n[0] = n[1] = n[2] = 0;
			const float w = D[(size_t)r*W+c];
			if (w <= 0) continue;
			int whxx = 0, whxy = 0, whyy = 0, cnt = 0;
			float wgx = 0, wgy = 0;
			for (int y = -1; y <= 1; ++y) {
				for (int x = -1; x <= 1; ++x) {
					if (x == 0 && y == 0) continue;
					const int px = c+x, py = r+y;
					if (px < 0 || py < 0 || px >= W || py >= H) continue;
					const float wi = D[(size_t)py*W+px];
					if (!(wi > 0 && depth_similar(w, wi, 0.03f))) continue;
					whxx += x*x; whxy += x*y; whyy += y*y;
					wgx += (wi-w)*x; wgy += (wi-w)*y;
					++cnt;
				}
			}
			if (cnt < 3) continue;
			const int det = whxx*whyy - whxy*whxy;
			if (det == 0) continue;
			const float invDet = 1.f/float(det);
			const float wx = (float(whyy)*wgx - float(whxy)*wgy)*invDet;
			const float wy = (float(-whxy)*wgx + float(whxx)*wgy)*invDet;
			const float ax = fx*wx, ay = fy*wy, az = (cx-float(c))*wx + (cy-float(r))*wy - w;
			// cv::normalize(Vec3f): v * (1/norm(v)), the norm accumulated in double
			double s = 0; s += (double)ax*ax; s += (double)ay*ay; s += (double)az*az;
			const double nv = std::sqrt(s);
			const double k = nv ? 1./nv : 0.;
			n[0] = (float)(ax*k); n[1] = (float)(ay*k); n[2] = (float)(az*k);
		}
	}
}

} // extern "C"
