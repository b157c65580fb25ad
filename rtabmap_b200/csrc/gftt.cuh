// gftt.cuh — GFTT corners for the GFTT/ORB detector (Kp/DetectorStrategy=8, RTAB-Map's default).
//
// Replaces: rtabmap::GFTT::generateKeypointsImpl (corelib/src/Features2d.cpp:2141-2178), i.e. cv::GFTTDetector::detect =
// cv::goodFeaturesToTrack with the min-eigenvalue corner map (cv::cornerMinEigenVal, block 3, Sobel aperture 3), then the image-border
// filter of cv::ORB::compute on the kept corners (GFTT_ORB::generateDescriptorsImpl, :2352-2356).  The level-0 gray image and depth mask
// come from orb_prepare*, the descriptors and 3-D points from the ORB kernels (orb.cuh) unchanged.
//
// Bit-exactness (the arithmetic of oracle/gftt_py.py, pinned to opencv-python 4.13 by tests/test_oracle_gftt.py):
//   * Sobel with s = 1/3060: dx = fma(U + D, s, C * 2s) on the row differences above / at / below; row pass of column c
//     fma(R, s, fma(M, 2s, L * s)) for c < (w & ~31), ((L * s + M * 2s) + R * s) without fused multiply-add in the last w % 32 columns
//     (OpenCV's x86 AVX2 row filter fuses in its 32-pixel vector body, not in its scalar tail); dy = the row pass's difference between
//     the rows below and above; reflect-101 border;
//   * the 3x3 box filter of the products sums each row in double and keeps a RUNNING column sum in double from the top of the image
//     down, as OpenCV's column filter does: that sum is not exact, so the corner kernel walks every column from row 0;
//   * lambda = (a + c) - sqrt((a - c)^2 + b^2) in float, a = 0.5 xx, c = 0.5 yy, no fused multiply-add;
//   * candidates: interior, inside the mask, above float(max * quality) and equal to their 3x3 dilation; key (lambda descending, raster
//     index descending) reproduces std::sort with greaterThanPtr (equal values: the higher address first);
//   * the cvRound(minDistance) grid test only looks at the 3x3 neighbouring cells, with the squared distance in float.
#pragma once
#include "orb.cuh"

namespace lcd {

constexpr int kGfttCandCap = 65536;     // local maxima kept per frame before the sort
constexpr int kGfttSortChunk = 8192;    // keys per shared-memory pass of the sort (64 KB)
constexpr int kGfttColTile = 126;       // output columns per CTA of the corner kernel (128 threads, one halo column each side)
constexpr int kGfttBitmapSmem = 200 * 1024; // largest occupancy bitmap kept in shared memory; larger images use a global one

// order-preserving key of a float: larger float, larger unsigned (0 sorts below every float)
__device__ __forceinline__ unsigned gftt_ord(float f)
{
	const unsigned u = __float_as_uint(f);
	return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__device__ __forceinline__ float gftt_unord(unsigned k)
{
	return k == 0u ? 0.0f : __uint_as_float((k & 0x80000000u) ? (k & 0x7FFFFFFFu) : ~k);
}

struct GfttEigArgs
{
	const uint8_t * gray;  // level 0 of each frame's pyramid
	const uint8_t * mask;  // level 0 of each frame's mask pyramid, or nullptr
	int w, h, frame_stride;
	float * eig;           // [frame][h][w]
	unsigned * max_key;    // [frame] gftt_ord of the largest lambda inside the mask
};

// One CTA per 126 columns of a frame, one thread per column, walking the rows from the top: Sobel, products, the 3x3 box (row sums of
// the three columns exchanged through shared memory, running column sum in registers) and the minimum eigenvalue.
__global__ void __launch_bounds__(128)
gftt_eig_kernel(const GfttEigArgs a)
{
	__shared__ float s_p[3][128];
	const int frame = blockIdx.y, t = threadIdx.x;
	const int w = a.w, h = a.h;
	const uint8_t * img = a.gray + static_cast<size_t>(frame) * a.frame_stride;
	const uint8_t * msk = a.mask ? a.mask + static_cast<size_t>(frame) * a.frame_stride : nullptr;
	float * eig = a.eig + static_cast<size_t>(frame) * w * h;
	const int x = blockIdx.x * kGfttColTile + t - 1;
	const bool out_col = t >= 1 && t <= kGfttColTile && x < w;
	const int xc = reflect101(min(x, w), w);
	const int xm = reflect101(xc - 1, w), xp = reflect101(xc + 1, w);
	const float s = static_cast<float>(1.0 / 3060.0), s2 = static_cast<float>(2.0 / 3060.0);
	const bool fused = xc < (w & ~31); // xc, not x: the halo thread at x = w stands for column w - 2
	auto row_d = [&](int r) { return static_cast<float>(img[r * w + xp]) - static_cast<float>(img[r * w + xm]); };
	auto row_s = [&](int r) {
		const float L = static_cast<float>(img[r * w + xm]), M = static_cast<float>(img[r * w + xc]), R = static_cast<float>(img[r * w + xp]);
		return fused ? __fmaf_rn(R, s, __fmaf_rn(M, s2, __fmul_rn(L, s))) : __fadd_rn(__fadd_rn(__fmul_rn(L, s), __fmul_rn(M, s2)), __fmul_rn(R, s));
	};
	// row sums (double) of the products of image row r
	auto row_sums = [&](int r, double & sxx, double & sxy, double & syy) {
		const int ru = reflect101(r - 1, h), rd = reflect101(r + 1, h);
		const float dx = __fmaf_rn(__fadd_rn(row_d(ru), row_d(rd)), s, __fmul_rn(row_d(r), s2));
		const float dy = __fsub_rn(row_s(rd), row_s(ru));
		__syncthreads(); // the previous row's sums have been read
		s_p[0][t] = __fmul_rn(dx, dx);
		s_p[1][t] = __fmul_rn(dx, dy);
		s_p[2][t] = __fmul_rn(dy, dy);
		__syncthreads();
		if (out_col)
		{
			sxx = (static_cast<double>(s_p[0][t - 1]) + static_cast<double>(s_p[0][t])) + static_cast<double>(s_p[0][t + 1]);
			sxy = (static_cast<double>(s_p[1][t - 1]) + static_cast<double>(s_p[1][t])) + static_cast<double>(s_p[1][t + 1]);
			syy = (static_cast<double>(s_p[2][t - 1]) + static_cast<double>(s_p[2][t])) + static_cast<double>(s_p[2][t + 1]);
		}
	};
	// ring of the row sums of rows y - 1, y, y + 1 (reflected)
	double rxx[3] = {0, 0, 0}, rxy[3] = {0, 0, 0}, ryy[3] = {0, 0, 0};
	row_sums(reflect101(-1, h), rxx[0], rxy[0], ryy[0]);
	row_sums(0, rxx[1], rxy[1], ryy[1]);
	double axx = (0.0 + rxx[0]) + rxx[1], axy = (0.0 + rxy[0]) + rxy[1], ayy = (0.0 + ryy[0]) + ryy[1];
	unsigned best = 0u;
	for (int y = 0; y < h; ++y)
	{
		const int in = (y + 2) % 3, leave = y % 3; // ring slots of rows y + 1 and y - 1
		row_sums(reflect101(y + 1, h), rxx[in], rxy[in], ryy[in]);
		if (!out_col) continue;
		const double sxx = axx + rxx[in], sxy = axy + rxy[in], syy = ayy + ryy[in];
		axx = sxx - rxx[leave];
		axy = sxy - rxy[leave];
		ayy = syy - ryy[leave];
		const float ea = __fmul_rn(static_cast<float>(sxx), 0.5f), eb = static_cast<float>(sxy), ec = __fmul_rn(static_cast<float>(syy), 0.5f);
		const float d = __fsub_rn(ea, ec);
		const float lam = __fsub_rn(__fadd_rn(ea, ec), __fsqrt_rn(__fadd_rn(__fmul_rn(d, d), __fmul_rn(eb, eb))));
		eig[static_cast<size_t>(y) * w + x] = lam;
		if (!msk || msk[static_cast<size_t>(y) * w + x]) best = max(best, gftt_ord(lam));
	}
	best = __reduce_max_sync(0xFFFFFFFFu, best);
	if ((t & 31) == 0 && best) atomicMax(a.max_key + frame, best);
}

struct GfttCandArgs
{
	const float * eig;
	const uint8_t * mask;
	int w, h, frame_stride;
	const unsigned * max_key;
	double quality;
	unsigned long long * keys; // [frame][kGfttCandCap]
	int * count;               // [frame]
	int * overflow;
};

// 3x3 local maxima of the thresholded map (THRESH_TOZERO, then dilate), interior pixels inside the mask, appended to the frame's list
__global__ void __launch_bounds__(256)
gftt_cand_kernel(const GfttCandArgs a)
{
	const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y, frame = blockIdx.z;
	const int w = a.w;
	if (x < 1 || y < 1 || x >= w - 1 || y >= a.h - 1) return;
	if (a.mask && !a.mask[static_cast<size_t>(frame) * a.frame_stride + static_cast<size_t>(y) * w + x]) return;
	const float thr = static_cast<float>(static_cast<double>(gftt_unord(a.max_key[frame])) * a.quality);
	const float * e = a.eig + static_cast<size_t>(frame) * w * a.h;
	auto tz = [&](int yy, int xx) { const float v = e[static_cast<size_t>(yy) * w + xx]; return v > thr ? v : 0.0f; };
	const float v = tz(y, x);
	if (v == 0.0f) return;
#pragma unroll
	for (int dy = -1; dy <= 1; ++dy)
#pragma unroll
		for (int dx = -1; dx <= 1; ++dx)
			if ((dy | dx) && tz(y + dy, x + dx) > v) return;
	const int pos = atomicAdd(a.count + frame, 1);
	if (pos < kGfttCandCap)
		a.keys[static_cast<size_t>(frame) * kGfttCandCap + pos] = (static_cast<unsigned long long>(gftt_ord(v)) << 32) | static_cast<unsigned>(y * w + x);
	else
		*a.overflow = 1;
}

// Descending bitonic sort of each frame's keys, one CTA per frame: stages with a distance below kGfttSortChunk run in shared memory,
// the longer ones in global memory.
__global__ void __launch_bounds__(1024)
gftt_sort_kernel(unsigned long long * __restrict__ keys_all, const int * __restrict__ count)
{
	extern __shared__ __align__(16) unsigned char smem_raw[];
	unsigned long long * sk = reinterpret_cast<unsigned long long *>(smem_raw);
	const int frame = blockIdx.x, tid = threadIdx.x;
	unsigned long long * keys = keys_all + static_cast<size_t>(frame) * kGfttCandCap;
	const int n = min(count[frame], kGfttCandCap);
	if (n <= 1) return;
	int pad = 2;
	while (pad < n) pad <<= 1;
	for (int i = n + tid; i < pad; i += blockDim.x) keys[i] = 0ull; // sorts last
	__syncthreads();
	const int chunk = min(pad, kGfttSortChunk);
	auto cmpx = [](unsigned long long * k, int i, int j, bool desc_block) {
		const unsigned long long x = k[i], y = k[j];
		if ((x < y) == desc_block)
		{
			k[i] = y;
			k[j] = x;
		}
	};
	// all stages of distance j < chunk for the merge size kk (kk <= chunk: the whole sort of the chunk up to kk)
	auto chunk_pass = [&](int kk_from, int kk_to, int j_from) {
		for (int c0 = 0; c0 < pad; c0 += chunk)
		{
			for (int i = tid; i < chunk; i += blockDim.x) sk[i] = keys[c0 + i];
			__syncthreads();
			for (int kk = kk_from; kk <= kk_to; kk <<= 1)
				for (int j = (kk == kk_from ? j_from : kk >> 1); j > 0; j >>= 1)
				{
					for (int i = tid; i < chunk; i += blockDim.x)
					{
						const int ixj = i ^ j;
						if (ixj > i) cmpx(sk, i, ixj, ((c0 + i) & kk) == 0);
					}
					__syncthreads();
				}
			for (int i = tid; i < chunk; i += blockDim.x) keys[c0 + i] = sk[i];
			__syncthreads();
		}
	};
	chunk_pass(2, chunk, 1);
	for (int kk = chunk << 1; kk <= pad; kk <<= 1)
	{
		for (int j = kk >> 1; j >= chunk; j >>= 1)
		{
			for (int i = tid; i < pad; i += blockDim.x)
			{
				const int ixj = i ^ j;
				if (ixj > i) cmpx(keys, i, ixj, (i & kk) == 0);
			}
			__syncthreads();
		}
		chunk_pass(kk, kk, chunk >> 1);
	}
}

struct GfttSelectArgs
{
	const unsigned long long * keys;
	const int * count;
	int w, h;
	double min_distance;  // GFTT/MinDistance
	int max_corners;      // Kp/MaxFeatures
	int edge;             // ORB/EdgeThreshold (cv::ORB::compute drops corners closer to the border)
	int bitmap_words;     // 32-bit words per row of the occupancy bitmap
	uint32_t * bitmap;    // [frame][h][bitmap_words] when the bitmap does not fit in shared memory, else nullptr
	OrbKeypoint * kps;    // [frame][cap]
	int * n_kp;
	int cap;
};

// The greedy minDistance walk over the sorted candidates, one CTA per frame.  Warp 0 takes 32 candidates at a time: each lane tests its
// candidate against the corners kept so far (a bitmap of kept pixels, read over the 3x3 neighbouring grid cells), then the lanes are
// resolved in order with shuffles, so the result is the sequential walk's.
__global__ void __launch_bounds__(256)
gftt_select_kernel(const GfttSelectArgs a)
{
	extern __shared__ __align__(16) unsigned char smem_raw[];
	const int frame = blockIdx.x, tid = threadIdx.x;
	const int w = a.w, h = a.h;
	const bool grid = a.min_distance >= 1.0;
	const size_t bm_n = static_cast<size_t>(a.bitmap_words) * h;
	uint32_t * bm = a.bitmap ? a.bitmap + static_cast<size_t>(frame) * bm_n : reinterpret_cast<uint32_t *>(smem_raw);
	if (grid)
	{
		for (size_t i = tid; i < bm_n; i += blockDim.x) bm[i] = 0u;
		__syncthreads();
	}
	if (tid >= 32) return;
	const int lane = tid;
	const volatile uint32_t * vbm = bm;
	const int n = min(a.count[frame], kGfttCandCap);
	const unsigned long long * keys = a.keys + static_cast<size_t>(frame) * kGfttCandCap;
	const int cell = grid ? __double2int_rn(a.min_distance) : 1;
	const int gw = (w + cell - 1) / cell, gh = (h + cell - 1) / cell;
	const double md2 = a.min_distance * a.min_distance;
	const unsigned lt = (1u << lane) - 1u;
	auto near = [&](int x, int y, int px, int py) {
		const float dx = static_cast<float>(x - px), dy = static_cast<float>(y - py);
		return static_cast<double>(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy))) < md2;
	};
	int kept = 0, n_out = 0;
	OrbKeypoint * out = a.kps + static_cast<size_t>(frame) * a.cap;
	for (int base = 0; base < n && kept < a.max_corners; base += 32)
	{
		const int i = base + lane;
		const bool valid = i < n;
		const unsigned long long key = valid ? keys[i] : 0ull;
		const int idx = static_cast<int>(key & 0xFFFFFFFFull);
		const int y = idx / w, x = idx - y * w;
		bool good = valid;
		if (grid)
		{
			const int xc = x / cell, yc = y / cell;
			if (good)
			{
				const int X0 = max(0, xc - 1) * cell, X1 = min(min(gw - 1, xc + 1) * cell + cell - 1, w - 1);
				const int Y0 = max(0, yc - 1) * cell, Y1 = min(min(gh - 1, yc + 1) * cell + cell - 1, h - 1);
				for (int yy = Y0; yy <= Y1 && good; ++yy)
					for (int wd = X0 >> 5; wd <= (X1 >> 5) && good; ++wd)
					{
						uint32_t bits = vbm[static_cast<size_t>(yy) * a.bitmap_words + wd];
						const int lo = max(X0 - wd * 32, 0), hi = min(X1 - wd * 32, 31);
						bits &= (0xFFFFFFFFu >> (31 - hi)) & (0xFFFFFFFFu << lo);
						while (bits && good)
						{
							const int b = __ffs(bits) - 1;
							bits &= bits - 1;
							if (near(x, y, wd * 32 + b, yy)) good = false;
						}
					}
			}
			// earlier lanes of this group that are kept suppress later ones in their neighbouring cells
			for (int j = 0; j < 31; ++j)
			{
				const bool gj = __shfl_sync(0xFFFFFFFFu, good, j);
				const int xj = __shfl_sync(0xFFFFFFFFu, x, j), yj = __shfl_sync(0xFFFFFFFFu, y, j);
				if (gj && good && lane > j && abs(x / cell - xj / cell) <= 1 && abs(y / cell - yj / cell) <= 1 && near(x, y, xj, yj)) good = false;
			}
		}
		const unsigned acc = __ballot_sync(0xFFFFFFFFu, good);
		const bool take = good && kept + __popc(acc & lt) < a.max_corners;
		if (take && grid) atomicOr(bm + static_cast<size_t>(y) * a.bitmap_words + (x >> 5), 1u << (x & 31));
		const bool inb = take && x >= a.edge && y >= a.edge && x < w - a.edge && y < h - a.edge;
		const unsigned ob = __ballot_sync(0xFFFFFFFFu, inb);
		if (inb)
		{
			const int pos = n_out + __popc(ob & lt);
			if (pos < a.cap)
			{
				OrbKeypoint k;
				k.x = static_cast<float>(x);
				k.y = static_cast<float>(y);
				k.size = 3.0f;
				k.angle = -1.0f;
				k.response = gftt_unord(static_cast<unsigned>(key >> 32));
				k.octave = 0;
				out[pos] = k;
			}
		}
		n_out += __popc(ob);
		kept += __popc(__ballot_sync(0xFFFFFFFFu, take));
		__syncwarp();
	}
	if (lane == 0) a.n_kp[frame] = min(n_out, a.cap);
}

} // namespace lcd
