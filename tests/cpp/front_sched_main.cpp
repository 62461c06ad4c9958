// CPU simulation of the wave-front SGM aggregation schedule (openmvs_b200/csrc/sgm_front_sched.h): builds the same work items
// as the host driver, walks them in queue order the way the kernel's warps do — dependency checks, per-path state hand-over
// between segments, store-or-add of the sum volume — with the path recursion in plain scalar code, and writes the summed path
// costs.  tests/test_sgm_front_schedule.py compares them with the oracle: every (pixel, direction) is processed exactly once, in
// an order that respects every dependency, for every block size / lag / sub-cell width.  (The CUDA arithmetic itself is covered
// on the GPU.)
#include "../../openmvs_b200/csrc/sgm_front_sched.h"
#include <cstdio>
#include <cstdlib>
#include <cmath>
#include <cstring>

int main(int argc, char** argv) {
	if (argc < 3) { fprintf(stderr, "usage: front_sched in.bin out.bin\n"); return 64; }
	FILE* f = fopen(argv[1], "rb");
	if (!f) return 65;
	int hdr[7]; // w, h, num, FB, lag, P1, sub-cell width (0: the driver's)
	if (fread(hdr, 4, 7, f) != 7) return 66;
	const int w = hdr[0], h = hdr[1], num = hdr[2], FB = hdr[3], lag = hdr[4], P1 = hdr[5];
	const int vw = w-6, vh = h-6;
	std::vector<uint16_t> P2s(256);
	std::vector<float> gray((size_t)w*h);
	const size_t n = (size_t)vw*vh*num;
	std::vector<uint8_t> costs(n);
	if (fread(P2s.data(), 2, 256, f) != 256 || fread(gray.data(), 4, gray.size(), f) != gray.size() || fread(costs.data(), 1, n, f) != n) return 66;
	fclose(f);
	std::vector<uint16_t> S[2] = {std::vector<uint16_t>(n, 0xABCD), std::vector<uint16_t>(n, 0xABCD)};   // garbage: phase 0 of a pass must store every entry
	std::vector<uint32_t> touched(n/num*8, 0);
	const int maxPaths = vw+vh+8;
	std::vector<uint16_t> state((size_t)8*maxPaths*num);
	std::vector<float> metaI((size_t)8*maxPaths); std::vector<int> metaH((size_t)8*maxPaths);
	FrontLaunch LA;
	sgm_front_build_launch(vw, vh, FB, lag, hdr[6] ? hdr[6] : sgm_front_sub_cell(vw), LA);
	std::vector<int> progress((size_t)LA.nChains, 0), cellDone((size_t)LA.nCells, 0);
	for (const FrontItem& it: LA.items) {
		const int dir = it.dir & 0xFF, pass = (it.dir >> 8) & 1;
		const FrontPassDesc& pd = FRONT_PASSES[pass];
		// in-order execution: every dependency must already be complete, or the queue order would deadlock a single worker
		if (progress[it.chain] < it.seq) { printf("FAIL: band dependency not met (dir %d k0 %d fb %d)\n", dir, it.k0, it.fb); return 2; }
		const int nDep = it.depCell >= 0 ? (it.depNeed & 0xFF) : 0, nOwn = (it.depNeed >> 8) & 0xFF;
		if (nOwn > 31 || nDep > 31) { printf("FAIL: an item touches %d sub-cells (one lane polls one counter)\n", nOwn); return 2; }
		for (int i = 0; i < nDep; ++i)
			if (cellDone[it.depCell+i] < LA.cellNeed[it.depCell+i]) { printf("FAIL: phase dependency not met (ph %d fb %d sub-cell %d)\n", it.ph, it.fb, i); return 2; }
		if (nOwn == 0) { printf("FAIL: an item touches no sub-cell\n"); return 2; }
		const bool add = it.ph != 0;
		std::vector<uint16_t>& V = S[pass];
		for (int g = 0; g < 4; ++g) {
			int xs, ys, dx, dy;
			if (!front_path_start(dir, it.k0+g, vw, vh, xs, ys, dx, dy)) continue;
			const int len = front_path_len(xs, ys, dx, dy, vw, vh);
			const int f0 = pd.fa*xs + pd.fb*ys + LA.fc[pass], df = std::max(1, pd.fa*dx + pd.fb*dy);
			const int s0 = std::min(len, front_first_step(it.fb*LA.FB, f0, df)), s1 = std::min(len, front_first_step((it.fb+1)*LA.FB, f0, df));
			if (s1 <= s0) continue;
			const size_t slot = (size_t)(pass*4+it.ph)*maxPaths + (it.k0+g);
			std::vector<unsigned> A(num, 0xFFFFu); float Ip = 0.5f; bool havePrev = false;
			if (s0 > 0) { for (int d = 0; d < num; ++d) A[d] = state[slot*num+d]; Ip = metaI[slot]; havePrev = metaH[slot] != 0; }
			for (int s = s0; s < s1; ++s) {
				const int x = xs+s*dx, y = ys+s*dy;
				const size_t idx = ((size_t)y*vw + x)*num;
				const float I = gray[(size_t)y*w + x];
				int di = std::abs((int)std::floor(255.f*(I-Ip)+.5f)); if (di > 255) di = 255;
				const unsigned P2 = P2s[di];
				std::vector<unsigned> L(num);
				unsigned m = 0xFFFFFFFFu;
				for (int d = 0; d < num; ++d) {
					unsigned best = P2;
					if (havePrev) {
						const unsigned lm = d > 0 ? A[d-1] : 0xFFFFu, lq = d+1 < num ? A[d+1] : 0xFFFFu;
						const unsigned nb = std::min(0xFFFFu, std::min(lm, lq)+(unsigned)P1);
						best = std::min(std::min(A[d], nb), P2);
					}
					L[d] = costs[idx+d]+best;
					m = std::min(m, L[d]);
				}
				for (int d = 0; d < num; ++d) {
					V[idx+d] = (uint16_t)(add ? V[idx+d]+L[d] : L[d]);
					A[d] = L[d]-m;
				}
				touched[((size_t)y*vw+x)*8 + dir] += 1;
				// the counters this item bumps must include the sub-cell of every pixel it writes
				const int nSX = (vw+LA.subCell-1)/LA.subCell, sx = x/LA.subCell, first = it.cell % nSX;
				if (sx < first || sx >= first+nOwn) { printf("FAIL: pixel outside the item's sub-cells\n"); return 2; }
				Ip = I; havePrev = true;
			}
			if (s1 < len) { for (int d = 0; d < num; ++d) state[slot*num+d] = (uint16_t)A[d]; metaI[slot] = Ip; metaH[slot] = havePrev; }
		}
		progress[it.chain] = it.seq+1;
		for (int i = 0; i < nOwn; ++i) cellDone[it.cell+i] += 1;
	}
	for (size_t i = 0; i < n; ++i) S[0][i] = (uint16_t)(S[0][i]+S[1][i]);
	for (size_t i = 0; i < touched.size(); ++i)
		if (touched[i] != 1) { printf("FAIL: pixel %zu direction %zu processed %u times\n", i/8, i%8, touched[i]); return 3; }
	f = fopen(argv[2], "wb");
	fwrite(S[0].data(), 2, n, f);
	fclose(f);
	printf("ok: %zu items\n", LA.items.size());
	return 0;
}
