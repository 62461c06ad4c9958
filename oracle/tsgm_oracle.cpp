// tsgm_oracle.cpp — CPU restatement of the helpers of the hierarchical (tSGM) level loop of
// SemiGlobalMatcher::Match(scene, ...) (TEST INFRASTRUCTURE, see oracle.h).  Sequential, in the reference's loop order.
// Part of liboracle.so; oracle/tsgm.py binds it.
#include "oracle.h"
#include <algorithm>
#include <vector>

namespace {
typedef int16_t Disparity;
const Disparity NO_DISP = 32767;
const uint8_t INVALID = 0;
const int halfWindowSizeX = 3, halfWindowSizeY = 3;

// cList::GetMedian<Disparity> (libs/Common/List.h:668-678): nth_element, for an even count the mean of the two middle values
// in the Disparity type (int arithmetic, truncated toward zero)
Disparity median(std::vector<Disparity>& v) {
	const size_t n = v.size();
	if (n % 2) {
		std::nth_element(v.begin(), v.begin()+(n>>1), v.end());
		return v[n>>1];
	}
	std::nth_element(v.begin(), v.begin()+(n>>1), v.end());
	const Disparity b = v[n>>1];
	std::nth_element(v.begin(), v.begin()+(n>>1)-1, v.begin()+(n>>1));
	const Disparity a = v[(n>>1)-1];
	return (Disparity)((a+b)/(Disparity)2);
}
} // namespace

// SemiGlobalMatcher::Disparity2RangeMap (libs/MVS/SemiGlobalMatcher.cpp:1350-1444)
uint64_t oracle_tsgm_range_map(const int16_t* disparityMap, int cols, int rows, const uint8_t* maskMap, int mw, int mh,
	int minNumDisp, int minNumDispInvalid, oracle_sgm_pixel* imagePixels)
{
	uint64_t numCosts = 0;
	std::vector<Disparity> disps;
	auto D = [&](int r, int c) { return disparityMap[(size_t)r*cols+c]; };
	for (int r = 0; r < rows; ++r) {
		const int r2 = r == 0 ? 0 : r*2+halfWindowSizeY;
		const int offset = r2*mw;
		int c2e = halfWindowSizeX;
		const uint8_t* pm = maskMap + (size_t)(r*2+halfWindowSizeY)*mw + halfWindowSizeX;
		for (int c = 0, c2 = 0; c < cols; ++c, pm += 2) {
			Disparity numDisp, minDisp, maxDisp;
			if (*pm == INVALID) {
				minDisp = maxDisp = NO_DISP;
				numDisp = 0;
			} else {
				const bool bInvalid = D(r, c) == NO_DISP;
				disps.clear();
				const int hw = bInvalid ? 20 : 3;
				for (int i = -hw; i <= hw; ++i)
					for (int j = -hw; j <= hw; ++j) {
						const int x = c+j, y = r+i;
						if (x >= 0 && y >= 0 && x < cols && y < rows) {
							const Disparity d = D(y, x);
							if (d != NO_DISP) disps.push_back(d);
						}
					}
				if (disps.size() < 3) {
					maxDisp = std::min((Disparity)(cols*2/3), (Disparity)minNumDispInvalid);
					minDisp = (Disparity)-maxDisp;
					numDisp = (Disparity)(maxDisp-minDisp);
				} else {
					const Disparity disp = (Disparity)(median(disps)*2);
					const Disparity mn = *std::min_element(disps.begin(), disps.end()), mx = *std::max_element(disps.begin(), disps.end());
					numDisp = (Disparity)((mx-mn)*2);
					if (numDisp < minNumDisp) {
						numDisp = (Disparity)minNumDisp;
						minDisp = (Disparity)(disp-numDisp/2);
						maxDisp = (Disparity)(disp+(numDisp+1)/2);
					} else {
						const Disparity maxNumDisp = bInvalid ? 64 : 32;
						if (numDisp > maxNumDisp) {
							minDisp = (Disparity)(disp-(maxNumDisp*(disp-mn*2)+1)/numDisp);
							maxDisp = (Disparity)(disp+(maxNumDisp*(mx*2+1-disp)+1)/numDisp);
							numDisp = (Disparity)(maxDisp-minDisp);
						} else {
							minDisp = (Disparity)(disp-numDisp/2);
							maxDisp = (Disparity)(disp+(numDisp+1)/2);
						}
					}
				}
			}
			c2e += 2;
			do {
				oracle_sgm_pixel& pixel = imagePixels[offset+c2];
				pixel.dmin = minDisp; pixel.dmax = maxDisp; pixel.reserved = 0;
				pixel.idx = numCosts;
				numCosts += (uint64_t)numDisp;
			} while (++c2 < c2e);
		}
		do {
			const oracle_sgm_pixel& pixel = imagePixels[offset+c2e-1];
			oracle_sgm_pixel& _pixel = imagePixels[offset+c2e];
			_pixel.dmin = pixel.dmin; _pixel.dmax = pixel.dmax; _pixel.reserved = 0;
			_pixel.idx = numCosts;
			numCosts += (uint64_t)(Disparity)(pixel.dmax-pixel.dmin);
		} while (++c2e < mw);
		const int _offsete = (r+1 == rows ? mh : r*2+halfWindowSizeY+2)*mw;
		for (int _offset = offset+mw; _offset < _offsete; _offset += mw) {
			for (int c2 = 0; c2 < mw; ++c2) {
				const oracle_sgm_pixel& pixel = imagePixels[offset+c2];
				oracle_sgm_pixel& _pixel = imagePixels[_offset+c2];
				_pixel.dmin = pixel.dmin; _pixel.dmax = pixel.dmax; _pixel.reserved = 0;
				_pixel.idx = numCosts;
				numCosts += (uint64_t)(Disparity)(pixel.dmax-pixel.dmin);
			}
		}
	}
	return numCosts;
}

// SemiGlobalMatcher::FlipDirection (libs/MVS/SemiGlobalMatcher.cpp:1630-1657)
void oracle_tsgm_flip_direction(const int16_t* l2r, int16_t* r2l, int width, int height) {
	std::fill(r2l, r2l+(size_t)width*height, NO_DISP);
	for (int r = 0; r < height; ++r)
		for (int c = 0; c < width; ++c) {
			const Disparity d = l2r[(size_t)r*width+c];
			if (d == NO_DISP) continue;
			for (int x = std::max(c+d-1, 0), xe = std::min(c+d+2, width); x < xe; ++x)
				r2l[(size_t)r*width+x] = (Disparity)-d;
		}
}

// SemiGlobalMatcher::UpscaleMask (libs/MVS/SemiGlobalMatcher.cpp:1662-1690)
void oracle_tsgm_upscale_mask(const uint8_t* maskMap, int width, int height, uint8_t* maskMap2x, int w2, int h2) {
	std::fill(maskMap2x, maskMap2x+(size_t)w2*h2, INVALID);
	for (int r = 0; r < height; ++r)
		for (int c = 0; c < width; ++c) {
			const int r2 = r*2+halfWindowSizeY, c2 = c*2+halfWindowSizeX;
			const uint8_t m = maskMap[(size_t)r*width+c];
			for (int i = 0; i < 2; ++i)
				for (int j = 0; j < 2; ++j) {
					const int x = c2+j, y = r2+i;
					if (x >= 0 && y >= 0 && x < w2 && y < h2) maskMap2x[(size_t)y*w2+x] = m;
				}
		}
}

// SemiGlobalMatcher::ExtractMask (libs/MVS/SemiGlobalMatcher.cpp:1518-1576), maskMap of the disparity map's size, in place
void oracle_tsgm_extract_mask(const int16_t* disparityMap, uint8_t* maskMap, int width, int height, int thValid) {
	for (int r = 0; r < height; ++r) {
		int numValid = 0;
		for (int c = 0; c < width; ++c) {
			uint8_t& m = maskMap[(size_t)r*width+c];
			if (m == INVALID) continue;
			m = INVALID;
			if (disparityMap[(size_t)r*width+c] == NO_DISP) continue;
			if (++numValid >= thValid) break;
		}
	}
	for (int r = 0; r < height; ++r) {
		int numValid = 0;
		for (int c = width; --c >= 0; ) {
			uint8_t& m = maskMap[(size_t)r*width+c];
			if (m == INVALID) continue;
			m = INVALID;
			if (disparityMap[(size_t)r*width+c] == NO_DISP) continue;
			if (++numValid >= thValid) break;
		}
	}
}
