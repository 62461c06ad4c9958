/*
 * oracle.h — C interface of the CPU oracle (TEST INFRASTRUCTURE, not product code).
 *
 * The oracle is a dependency-free CPU restatement of the reference's dense depth
 * estimation path (cdcseacave/openMVS, libs/MVS/DepthMap.{h,cpp},
 * libs/MVS/SceneDensify.cpp:490-805, libs/MVS/SemiGlobalMatcher.cpp:863-1302).
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference
 * legs may load it.  The product path (openmvs_b200/csrc) never links or calls it.
 *
 * PARITY UNPINNED: the reference ships no golden vectors for this path
 * (apps/Tests/Tests.cpp:87 only asserts a fused point count) and the reference itself
 * cannot be compiled in this image (OpenCV/Eigen/Boost/CGAL absent), so this
 * restatement is validated against hand-derived known answers and analytic ground
 * truth only.
 */
#ifndef B200MVS_ORACLE_H_
#define B200MVS_ORACLE_H_
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* one view: gray float image in [0,1], pinhole camera (K scaled to the image size),
 * optional known depth-map + its camera for the geometric-consistency pass
 * (DepthData::ViewData, libs/MVS/DepthMap.h:158-185) */
typedef struct {
	const float* image;
	int width, height;
	double K[9], R[9], C[3];
	const float* depth; /* nullable */
	int dwidth, dheight;
	double Kd[9], Rd[9], Cd[3];
} oracle_view;

/* OPTDENSE knobs consumed by the estimator (libs/MVS/DepthMap.cpp:69-114) + schedule */
typedef struct {
	int nEstimationIters;          /* 3 */
	int nEstimationGeometricIters; /* 2 */
	int nRandomIters;              /* 6 */
	float fNCCThresholdKeep;       /* 0.9 */
	float fDescriptorMinMagnitudeThreshold; /* 0.02 */
	float fRandomDepthRatio;       /* 0.003 */
	float fRandomAngle1Range;      /* 16 deg */
	float fRandomAngle2Range;      /* 10 deg */
	float fRandomSmoothDepth;      /* 0.02 */
	float fRandomSmoothNormal;     /* 13 deg */
	float fRandomSmoothBonus;      /* 0.93 */
	float fEstimationGeometricWeight; /* 0.1 */
	int nSubResolutionLevels;      /* 2 */
	int schedule;    /* 0 = ZZ: reference zig-zag order, sequential Gauss-Seidel, mt19937
	                    1 = RB: red-black half-sweeps, Philox4x32-10 counter RNG */
	int propagation; /* RB only (the engine's schedule): bits 0-3: 2 = the two causal neighbours of the reference
	                    direction, 4 = all four 4-neighbours; bits 4-7: F far rings, the candidate of a direction is the
	                    lowest-cost pixel at distance 1, 3, .. 2F+1; bit 8 (0x100): a direction whose candidates kept
	                    their plane in their last update is not re-tested; bits 12-15: E > 0 = a pixel that scored c
	                    candidates spends at most max(1, E - c) refinement tries in the sweep */
	uint32_t seed;
	int threads;     /* ZZ: number of worker threads pulling from the shared counter */
} oracle_params;

void oracle_default_params(oracle_params* p);

/* Philox4x32-10 block (known-answer testable) */
void oracle_philox4x32(const uint32_t ctr[4], const uint32_t key[2], uint32_t out[4]);

/* pass A only (ScoreDepthMapTmp): depth/normal are in/out (random init where invalid),
 * conf receives the raw cost in [0,2]. lowres (nullable) is the low-resolution depth prior. */
int oracle_pm_score(const oracle_view* views, int nViews, const oracle_params* prm,
	float dMin, float dMax, const float* lowres,
	float* depth, float* normal, float* conf);

/* one PatchMatch iteration `iter` (EstimateDepthMapTmp) on an existing state. RB: both
 * half-sweeps unless half >= 0, in which case only colour `half` (0/1) is processed. */
int oracle_pm_iterate(const oracle_view* views, int nViews, const oracle_params* prm,
	float dMin, float dMax, const float* lowres, int iter, int half,
	float* depth, float* normal, float* conf);

/* oracle_pm_iterate carrying the memory of the RB changed-flag rule (propagation & 0x100): changed = width x height bytes,
 * 1 = the pixel's plane changed in its last update (or was never tested); read and updated.  NULL: rule off. */
int oracle_pm_iterate_flags(const oracle_view* views, int nViews, const oracle_params* prm,
	float dMin, float dMax, const float* lowres, int iter, int half,
	float* depth, float* normal, float* conf, uint8_t* changed);

/* pass C (EndDepthMapTmp): threshold + cost -> confidence */
int oracle_pm_finalize(int width, int height, float keepThreshold,
	float* depth, float* normal, float* conf);

/* whole DepthMapsData::EstimateDepthMap (scale loop, passes A/B/C).
 * nGeometricIter < 0: photometric pass; >= 0: geometric pass (views need depth). */
int oracle_pm_estimate(const oracle_view* views, int nViews, const oracle_params* prm,
	float dMin, float dMax, int nGeometricIter,
	float* depth, float* normal, float* conf);

/* RB changed-flag rule (propagation & 0x100): {directions tested, directions skipped} since the last call */
void oracle_pm_counters(long long out[2]);

/* oracle_pm_estimate with an explicit range [iterBegin, iterEnd) of pass-B iterations (RB: sweeps) and an optional
 * ignore-mask of the reference view (width x height bytes, 0 = ignored; DepthMap.cpp:215-230,300-323,343; the depth is then
 * up-sampled NEAREST between the levels, SceneDensify.cpp:661).  geometric != 0: no scale loop, keep threshold x1. */
int oracle_pm_estimate_range(const oracle_view* views, int nViews, const oracle_params* prm,
	float dMin, float dMax, int geometric, int iterBegin, int iterEnd, const uint8_t* mask,
	float* depth, float* normal, float* conf);

/* single hypothesis score at pixel (x,y) with explicit smoothing neighbours
 * (known-answer helper for ScorePixel); close = n x {depth, nx,ny,nz, X,Y,Z} */
float oracle_pm_score_pixel(const oracle_view* views, int nViews, const oracle_params* prm,
	float dMin, float dMax, const float* lowres, int x, int y,
	float depth, const float normal[3], const float* close, int nClose, float* viewScores);

/* geometry helpers exposed for known-answer tests */
void oracle_dir2normal(float a, float b, float n[3]);
void oracle_normal2dir(const float n[3], float* a, float* b);
void oracle_correct_normal(const double X0[3], float n[3]);
float oracle_interpolate_pixel(const double K[9], int x0, int y0, int nx, int ny,
	float depth, const float normal[3], float dMin, float dMax);
void oracle_zigzag(int width, int height, int rawStride, uint16_t* coordsXY);

/* cv::resize restatements used by the scale loop (third-party arithmetic, OpenCV) */
/* scx/scy: source/destination scale (1/fx for the factor form of cv::resize); <= 0: sw/dw */
void oracle_resize_area(const float* src, int sw, int sh, float* dst, int dw, int dh, double scx, double scy);
void oracle_resize_linear(const float* src, int sw, int sh, float* dst, int dw, int dh);
void oracle_resize_nearest(const float* src, int sw, int sh, int channels, float* dst, int dw, int dh);
void oracle_scale_K(const double K[9], int sw, int sh, int dw, int dh, double Kout[9]);

/* ---- SGM (SemiGlobalMatcher::Match, libs/MVS/SemiGlobalMatcher.cpp:863-1302) ---- */
typedef struct {
	uint64_t idx;      /* offset of the first cost of this pixel in the ragged volume */
	int16_t dmin, dmax;/* disparity range [dmin, dmax); invalid pixel: dmin >= dmax */
	int32_t reserved;
} oracle_sgm_pixel;

void oracle_sgm_p2s(uint16_t P2, float alpha, float beta, uint16_t out[256]);
/* stage & 7: 1 costs, 2 + aggregation, 3 + WTA; stage & 8: costs[] is supplied, skip stage 1 */
int oracle_sgm_match(const float* leftGray, const uint8_t* leftBGR, const float* rightGray, int width, int height,
	const oracle_sgm_pixel* pixels, uint64_t numCosts, uint16_t P1, uint16_t P2, float P2alpha, float P2beta, int stage,
	uint8_t* costs, uint16_t* accums, int16_t* disparity, uint16_t* cost);

void oracle_sgm_cross_check(int16_t* l2r, const int16_t* r2l, int width, int height, int thCross);
void oracle_sgm_refine(const oracle_sgm_pixel* pixels, const uint16_t* accums, int16_t* disparity, int nPixels, int subpixelSteps);

/* ---- helpers of the hierarchical (tSGM) level loop of SemiGlobalMatcher::Match(scene, ...) (tsgm_oracle.cpp) ---- */
/* Disparity2RangeMap: pixels of the mw x mh 2x grid from the cols x rows disparity map; returns numCosts */
uint64_t oracle_tsgm_range_map(const int16_t* disparityMap, int cols, int rows, const uint8_t* maskMap, int mw, int mh,
	int minNumDisp, int minNumDispInvalid, oracle_sgm_pixel* pixels);
void oracle_tsgm_flip_direction(const int16_t* l2r, int16_t* r2l, int width, int height);
void oracle_tsgm_upscale_mask(const uint8_t* maskMap, int width, int height, uint8_t* maskMap2x, int w2, int h2);
void oracle_tsgm_extract_mask(const int16_t* disparityMap, uint8_t* maskMap, int width, int height, int thValid);

/* ---- fusion-mode -2 (SemiGlobalMatcher::ProjectDisparity2DepthMap and ::Fuse, libs/MVS/SemiGlobalMatcher.cpp:1925-2039 and
 * :739-859; sgm_fuse_oracle.cpp) ---- */
/* ProjectDisparity2DepthMap of one pair into a W x H image: depth, range (2 floats per pixel), conf (nullable) -> numDepths */
int oracle_sgmf_project(const int16_t* disparity, const uint16_t* cost, int vw, int vh, int steps, const double* Q, int W, int H,
	float* depth, float* range, float* conf);
/* the cluster vote of Fuse (:795-848) over nPairs projected maps (pair p at offset p x W x H; ranges 2 floats per pixel) */
void oracle_sgmf_fuse(int nPairs, const float* depths, const float* ranges, const float* confs, int W, int H, unsigned minViews,
	float* depth, float* conf);
/* Q' = P invK Q of a reversed pair (:770-779) */
void oracle_sgmf_pair_q(const double* Q, const double* Kl, const double* Rl, const double* Cl, const double* K, const double* R,
	const double* C, double* Qout);
/* EstimateNormalMap(Matrix3x3f(K), depth, normal) (libs/MVS/DepthMap.cpp:1522-1613); normal: 3 floats per pixel */
void oracle_sgmf_normals(const float* D, int W, int H, const double* Kd, float* N);

/* ---- depth-map post-processing (libs/MVS/SceneDensify.cpp:810-1299) ---- */
/* one estimated depth-map with its camera (DepthData of a view: depthMap, confMap, images[0].camera) */
typedef struct {
	const float* depth; const float* conf; /* conf may be NULL when unused (bAdjust = 0 neighbours) */
	int width, height;
	double K[9], R[9], C[3];
} oracle_dmap;

/* z-buffered forward projection of a neighbour depth-map into the reference view (4-pixel splat) */
void oracle_filter_project(const oracle_dmap* ref, const oracle_dmap* nbr, float* projDepth, float* projConf /*nullable*/);
/* DepthMapsData::FilterDepthMap; nMinViews / nMinViewsAdjust already min(..., nCalibratedImages-1).
 * returns 0 when the map can not be filtered (too few neighbours). projected: nullable, N x H x W */
int oracle_filter_depth_map(const oracle_dmap* ref, const oracle_dmap* nbrs, int nNbrs, int nMinViews, int nMinViewsAdjust,
	float fDepthDiffThreshold, int bAdjust, float dMin, float dMax, float* outDepth, float* outConf, float* projected);
/* DepthMapsData::RemoveSmallSegments; th = fDepthDiffThreshold*0.7; normal/conf nullable; in place */
void oracle_remove_small_segments(float* depth, float* normal, float* conf, int width, int height, float th, unsigned speckle);
int oracle_count_asymmetric_edges(const float* depth, int width, int height, float th);
/* DepthMapsData::GapInterpolation; th = fDepthDiffThreshold*2.5; normal/conf nullable; in place */
void oracle_gap_interpolation(float* depth, float* normal, float* conf, int width, int height, float th, unsigned gap);
/* TImage<Pixel8U>::toGray(..., bNormalize = true) (libs/Common/Types.inl:2377-2431); stride in bytes */
void oracle_to_gray(const uint8_t* src, int width, int height, int stride, int channels, int bgr, float* dst);

/* ---- Scene::PointCloudFilter (libs/MVS/SceneDensify.cpp:2226-2360; visibility_oracle.cpp) ---- */
/* the visibility counts of every (point, view) cone over every point.  pts: 3 floats per point; off: n + 1 view offsets, views:
 * the image IDs; K: 9 doubles per image (row-major), C: 3 doubles per image, width: per image.  visibility: n ints, overwritten */
int oracle_visibility(const float* pts, uint64_t n, const uint32_t* off, const uint32_t* views, int nImages, const double* K,
	const double* C, const int* width, int threads, int32_t* visibility);
/* The reference's removal loop, literally: RFOREACH(idxPoint, points) if (visibility[idxPoint] <= thRemove) RemovePoint(idxPoint),
 * on an array of original indices; RemovePoint is cList::RemoveAt (libs/Common/List.h:1129-1136).  -> the number kept; order
 * holds the kept original indices in their final slots */
uint64_t oracle_visibility_filter(const int32_t* visibility, uint64_t n, int thRemove, uint32_t* order);

#ifdef __cplusplus
}
#endif
#endif
