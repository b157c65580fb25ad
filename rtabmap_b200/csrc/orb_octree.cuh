// orb_octree.cuh — the ORB-OCTREE detector (Kp/DetectorStrategy=10): RTAB-Map's ORB-SLAM2 extractor (corelib/src/opencv/ORBextractor.cc)
// behind rtabmap::ORBOctree (corelib/src/Features2d.cpp:2479-2566).
//
// Stages, one launch each (engine.cu: octree_run):
//   resize    level l from level l-1 at cvRound(size / scale_l) (ComputePyramid, :1114-1139): cv::resize INTER_LINEAR on 8-bit images,
//             i.e. the 2x2 mean (OpenCV's area-fast path) at an exact factor of 2 and 11-bit fixed-point bilinear otherwise;
//   fast      one CTA per cell of ComputeKeyPointsOctTree (:772-855, cells computed on the host): FAST-9/16 with non-max suppression
//             local to the cell (neighbours outside the cell's [3, n-3) window score 0), FAST/MinThreshold when FAST/Threshold finds
//             nothing; keys in raster order into the cell's own slot (room for every possible survivor: no overflow);
//   tree      DistributeOctTree (:546-770), one CTA per (frame, level): a node's keys are a contiguous segment of a per-level index array
//             and a division is a stable four-way partition of that segment (one warp per node, ballots); the list is kept in order
//             as node storage order; phase 2 sorts (size, creation rank), the later-created node counting as the larger pointer;
//   blur      GaussianBlur(7x7, sigma 2, REFLECT_101) of a clone of each level: OpenCV's 8-bit fixed-point path, taps
//             (18, 34, 48, 56, 48, 34, 18) / 256 per pass, (sum + 2^15) >> 16;
//   describe  one warp per kept key: IC angle on the unblurred level (integer moments, fastAtan2), steered BRIEF on the blurred one with
//             cos/sin of the float angle equal to glibc's cosf/sinf (oct_sincosf below), coordinates scaled by the float scale chain;
//   finish    per frame: the level-0 mask at the truncated coordinates, then Feature2D::limitKeypoints (limit_key / block_sort_desc).
#pragma once
#include "orb.cuh"

namespace lcd {

constexpr int kOctMaxLevels = 8;
constexpr int kOctTreeThreads = 512;

struct OctGeom
{
	int n_levels;
	int w[kOctMaxLevels], h[kOctMaxLevels];
	int off[kOctMaxLevels]; // plane offset of each level inside one frame's pyramid
	int frame_stride;       // bytes of one frame's pyramid
	float scale[kOctMaxLevels];
	int n_per_level[kOctMaxLevels];
	int size[kOctMaxLevels];       // (int)(patchSize * scale)
	int n_ini[kOctMaxLevels];      // round((maxX - minX) / (maxY - minY))
	float hx[kOctMaxLevels];       // (maxX - minX) / nIni
	int span_w[kOctMaxLevels], span_h[kOctMaxLevels]; // maxX - minX, maxY - minY
	int cell0[kOctMaxLevels + 1];  // first cell of each level in the cell table
	int key0[kOctMaxLevels + 1];   // first key slot of each level in a frame's key workspace
	int node0[kOctMaxLevels + 1];  // first node of each level in a frame's node workspace
	int raw_cap;                   // keypoints one frame can produce before the mask and the limit
	int edge;
	int thr_ini, thr_min;
	int umax[16];
};

struct OctCell
{
	int x0, y0, x1, y1; // level coordinates of the cell's sub-image [x0, x1) x [y0, y1)
	int dx, dy;         // j * wCell, i * hCell: added to the cell's keypoints
	int slot;           // first key slot of the cell inside the frame's key workspace
	int level;
};

struct OctNode
{
	int x0, y0, x1, y1; // UL = (x0, y0), BR = (x1, y1)
	int lo, hi;         // segment of the level's index array
	int rank;           // creation order (the phase-2 tie rule)
	int no_more;
};

// ---- glibc's sinf / cosf on [0, 2 pi] -----------------------------------------------------------------------------------------------
// The sincosf of glibc 2.28+ (reduction by a double pi/2 and double polynomials, rounded once to float), restated: computeOrbDescriptor
// calls cos/sin on a float, which is cosf/sinf.  glibc picks an FMA build of these functions when the CPU has FMA; on [0, 2 pi] the FMA
// and non-FMA builds give the same floats (both checked against the host libm over every float of the range), and this restatement uses
// the fused form.
__device__ __constant__ double kOctSinCos[2][8] = {
	{0x1p0, -0x1.ffffffd0c621cp-2, 0x1.55553e1068f19p-5, -0x1.6c087e89a359dp-10, 0x1.99343027bf8c3p-16, -0x1.555545995a603p-3, 0x1.1107605230bc4p-7,
	 -0x1.994eb3774cf24p-13},
	{-0x1p0, 0x1.ffffffd0c621cp-2, -0x1.55553e1068f19p-5, 0x1.6c087e89a359dp-10, -0x1.99343027bf8c3p-16, -0x1.555545995a603p-3, 0x1.1107605230bc4p-7,
	 -0x1.994eb3774cf24p-13}};

__device__ __forceinline__ float oct_sincos_poly(double x, double x2, const double * p, int n)
{
	if ((n & 1) == 0)
	{
		const double x3 = __dmul_rn(x, x2);
		const double s1 = __fma_rn(x2, p[7], p[6]);
		const double x7 = __dmul_rn(x3, x2);
		const double s = __fma_rn(x3, p[5], x);
		return __double2float_rn(__fma_rn(x7, s1, s));
	}
	const double x4 = __dmul_rn(x2, x2);
	const double c2 = __fma_rn(x2, p[4], p[3]);
	const double c1 = __fma_rn(x2, p[1], p[0]);
	const double x6 = __dmul_rn(x4, x2);
	const double c = __fma_rn(x4, p[2], c1);
	return __double2float_rn(__fma_rn(x6, c2, c));
}

// cosine = 1: cosf(y), 0: sinf(y), for 0 <= y < 120 (the descriptor's angles lie in [0, 2 pi])
__device__ __forceinline__ float oct_sincosf(float y, int cosine)
{
	const uint32_t top = (__float_as_uint(y) >> 20) & 0x7FFu;
	double x = y;
	if (top < ((__float_as_uint(0x1.921FB6p-1f) >> 20) & 0x7FFu))
	{
		if (top < ((__float_as_uint(0x1p-12f) >> 20) & 0x7FFu)) return cosine ? 1.0f : y;
		return oct_sincos_poly(x, __dmul_rn(x, x), kOctSinCos[0], cosine);
	}
	const double r = __dmul_rn(x, 0x1.45F306DC9C883p+23);
	const int n = (static_cast<int>(r) + 0x800000) >> 24;
	x = __fma_rn(-static_cast<double>(n), 0x1.921FB54442D18p0, x);
	const double s = ((n & 3) == 1 || (n & 3) == 2) ? -1.0 : 1.0;
	return oct_sincos_poly(__dmul_rn(x, s), __dmul_rn(x, x), kOctSinCos[(n & 2) ? 1 : 0], cosine ? (n ^ 1) : n);
}

// every float x in [0, x_max] from bit pattern `first` on: cosf and sinf (the test of the restatement against the host libm)
__global__ void orb_oct_sincos_kernel(uint32_t first, uint32_t count, float * __restrict__ c, float * __restrict__ s)
{
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= count) return;
	const float x = __uint_as_float(first + i);
	c[i] = oct_sincosf(x, 1);
	s[i] = oct_sincosf(x, 0);
}

// ---- gray + level-0 depth mask of every frame, one thread per pixel (any width and height) ---------------------------------------
__global__ void orb_oct_prepare_kernel(const OrbPrepArgs a)
{
	const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y, frame = blockIdx.z;
	const int w = a.g.w[0], h = a.g.h[0];
	if (x >= w || y >= h) return;
	const size_t px = static_cast<size_t>(y) * w + x;
	const uint8_t * p = a.images + (static_cast<size_t>(frame) * w * h + px) * a.channels;
	const int gv = a.channels == 1 ? p[0] : (p[0] * 3735 + p[1] * 19235 + p[2] * 9798 + (1 << 14)) >> 15;
	a.gray[static_cast<size_t>(frame) * a.g.frame_stride + px] = static_cast<uint8_t>(gv);
	if (a.mask)
		a.mask[static_cast<size_t>(frame) * a.g.frame_stride + px] =
			depth_to_mask(a.depth, a.depth_type, static_cast<size_t>(frame) * w * h + px, a.min_depth, a.max_depth);
}

// ---- resize: level l from level l-1 --------------------------------------------------------------------------------------------------
__global__ void orb_oct_resize_kernel(uint8_t * __restrict__ pyr, const OctGeom g, int level)
{
	const int dx = blockIdx.x * blockDim.x + threadIdx.x, dy = blockIdx.y * blockDim.y + threadIdx.y;
	const int dw = g.w[level], dh = g.h[level], sw = g.w[level - 1], sh = g.h[level - 1];
	if (dx >= dw || dy >= dh) return;
	uint8_t * frame = pyr + static_cast<size_t>(blockIdx.z) * g.frame_stride;
	const uint8_t * src = frame + g.off[level - 1];
	uint8_t * dst = frame + g.off[level];
	if (sw == 2 * dw && sh == 2 * dh)
	{
		// cv::resize turns INTER_LINEAR at an exact factor of 2 into its area-fast path
		const uint8_t * p = src + static_cast<size_t>(2 * dy) * sw + 2 * dx;
		dst[static_cast<size_t>(dy) * dw + dx] = static_cast<uint8_t>((p[0] + p[1] + p[sw] + p[sw + 1] + 2) >> 2);
		return;
	}
	// resizeGeneric_ coefficients: f = (float)((d + 0.5) * scale - 0.5) in double, s = floor(f), alpha = saturate_cast<short>(w * 2048)
	auto coef = [](int d, int n_dst, int n_src, int & i0, int & i1, int & a0, int & a1) {
		const double scale = 1.0 / (static_cast<double>(n_dst) / n_src);
		float f = static_cast<float>((d + 0.5) * scale - 0.5);
		int si = static_cast<int>(floorf(f));
		f -= static_cast<float>(si);
		if (si < 0) f = 0.f, si = 0;
		if (si >= n_src - 1) f = 0.f, si = n_src - 1;
		i0 = si;
		i1 = min(si + 1, n_src - 1);
		a0 = __float2int_rn((1.f - f) * 2048.f);
		a1 = __float2int_rn(f * 2048.f);
	};
	int x0, x1, xa0, xa1, y0, y1, ya0, ya1;
	coef(dx, dw, sw, x0, x1, xa0, xa1);
	coef(dy, dh, sh, y0, y1, ya0, ya1);
	const uint8_t * r0 = src + static_cast<size_t>(y0) * sw;
	const uint8_t * r1 = src + static_cast<size_t>(y1) * sw;
	const int h0 = r0[x0] * xa0 + r0[x1] * xa1, h1 = r1[x0] * xa0 + r1[x1] * xa1;
	// VResizeLinear<uchar, int, short>: ((b0 * (S0 >> 4)) >> 16) + ((b1 * (S1 >> 4)) >> 16), then (v + 2) >> 2 saturated
	const int v = (((ya0 * (h0 >> 4)) >> 16) + ((ya1 * (h1 >> 4)) >> 16) + 2) >> 2;
	dst[static_cast<size_t>(dy) * dw + dx] = static_cast<uint8_t>(min(max(v, 0), 255));
}

// ---- FAST per cell ------------------------------------------------------------------------------------------------------------------
constexpr int kOctCellMax = 72; // wCell, hCell < 60 (nCols = floor(span / 30)) plus the 6-pixel overlap

__global__ void __launch_bounds__(256)
orb_oct_fast_kernel(const uint8_t * __restrict__ pyr, const OctGeom g, const OctCell * __restrict__ cells, int n_cells, int key_stride,
                    uint32_t * __restrict__ keys, int * __restrict__ cell_n)
{
	__shared__ uint8_t s_img[kOctCellMax * kOctCellMax];
	__shared__ int16_t s_score[kOctCellMax * kOctCellMax];
	__shared__ int s_warp[8];
	const OctCell c = cells[blockIdx.x];
	const int frame = blockIdx.y, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
	const int cw = c.x1 - c.x0, ch = c.y1 - c.y0, lw = g.w[c.level];
	const uint8_t * img = pyr + static_cast<size_t>(frame) * g.frame_stride + g.off[c.level];
	for (int i = tid; i < cw * ch; i += 256) s_img[i] = img[static_cast<size_t>(c.y0 + i / cw) * lw + c.x0 + i % cw];
	uint32_t * out = keys + static_cast<size_t>(frame) * key_stride + c.slot;
	int total = 0;
	for (int pass = 0; pass < 2 && total == 0; ++pass)
	{
		const int thr = pass == 0 ? g.thr_ini : g.thr_min;
		__syncthreads();
		for (int i = tid; i < cw * ch; i += 256)
		{
			const int x = i % cw, y = i / cw;
			s_score[i] = (x >= 3 && x < cw - 3 && y >= 3 && y < ch - 3) ? static_cast<int16_t>(fast_score(s_img + i, cw, thr)) : int16_t(0);
		}
		__syncthreads();
		// non-max suppression in raster order, appended in order: 256 positions per step, ballots inside a warp, warp totals across
		for (int base = 0; base < cw * ch; base += 256)
		{
			const int i = base + tid;
			bool keep = false;
			int sc = 0;
			if (i < cw * ch)
			{
				const int x = i % cw, y = i / cw;
				sc = s_score[i];
				if (sc > 0)
				{
					keep = true;
					for (int ddy = -1; ddy <= 1 && keep; ++ddy)
						for (int ddx = -1; ddx <= 1; ++ddx)
						{
							if (!ddx && !ddy) continue;
							if (s_score[(y + ddy) * cw + x + ddx] >= sc)
							{
								keep = false;
								break;
							}
						}
				}
			}
			const unsigned b = __ballot_sync(0xFFFFFFFFu, keep);
			if (lane == 0) s_warp[warp] = __popc(b);
			__syncthreads();
			int before = 0, step = 0;
			for (int k = 0; k < 8; ++k)
			{
				before += k < warp ? s_warp[k] : 0;
				step += s_warp[k];
			}
			if (keep)
			{
				const int x = i % cw, y = i / cw;
				const int pos = (c.y0 + y) * lw + c.x0 + x;
				out[total + before + __popc(b & ((1u << lane) - 1u))] = (static_cast<uint32_t>(pos) << 8) | static_cast<uint32_t>(sc);
			}
			total += step;
			__syncthreads();
		}
	}
	if (tid == 0) cell_n[static_cast<size_t>(frame) * n_cells + blockIdx.x] = total;
}

// ---- DistributeOctTree --------------------------------------------------------------------------------------------------------------
struct OctTreeArgs
{
	OctGeom g;
	const uint32_t * keys;   // [frame][key_stride]
	const int * cell_n;      // [frame][n_cells]
	const OctCell * cells;
	int n_cells, key_stride, node_stride;
	uint32_t * kk;           // [frame][key_stride] the level's keys, compacted in cell order
	int * perm, * scratch;   // [frame][key_stride] index arrays
	OctNode * nodes;         // [frame][2][node_stride]: the list, in list order, and the next one
	int * cand;              // [frame][node_stride] the nodes divided this round, in division order
	int4 * cnt;              // [frame][node_stride] their children's key counts
	int * expand;            // [frame][node_stride] children with more than one key, in push order
	uint32_t * sel;          // [frame][node_stride] the kept key of each node, in list order
	int * sel_n;             // [frame][n_levels]
};

__device__ __forceinline__ int oct_child(uint32_t key, int w, int min_b, int mx, int my)
{
	const int pos = static_cast<int>(key >> 8);
	const int x = pos % w - min_b, y = pos / w - min_b;
	return (y < my ? 0 : 2) + (x < mx ? 0 : 1);
}

__global__ void __launch_bounds__(kOctTreeThreads)
orb_oct_tree_kernel(const OctTreeArgs a)
{
	extern __shared__ __align__(16) unsigned long long s_sort[]; // phase-2 sort keys
	__shared__ int s_n, s_len, s_n_cand, s_j, s_phase, s_done, s_n_exp, s_buf;
	const OctGeom & g = a.g;
	const int level = blockIdx.x, frame = blockIdx.y, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, n_warps = blockDim.x >> 5;
	const int w = g.w[level], min_b = g.edge - 3, N = g.n_per_level[level];
	const size_t kbase = static_cast<size_t>(frame) * a.key_stride + g.key0[level];
	const size_t nbase = static_cast<size_t>(frame) * a.node_stride + g.node0[level];
	uint32_t * kk = a.kk + kbase;
	int * perm = a.perm + kbase;
	int * scratch = a.scratch + kbase;
	// the two node lists of this (frame, level): list `b` starts at nodes + b * node_stride
	OctNode * const nodes = a.nodes + 2 * static_cast<size_t>(frame) * a.node_stride + g.node0[level];
	int * cand = a.cand + nbase;
	int4 * cnt = a.cnt + nbase;
	int * expand = a.expand + nbase;
	// the level's keys in cell order (cells row-major, raster order inside a cell)
	if (tid == 0)
	{
		int n = 0;
		for (int ci = g.cell0[level]; ci < g.cell0[level + 1]; ++ci) n += a.cell_n[static_cast<size_t>(frame) * a.n_cells + ci];
		s_n = n;
	}
	__syncthreads();
	for (int ci = g.cell0[level] + warp; ci < g.cell0[level + 1]; ci += n_warps)
	{
		int before = 0;
		for (int k = g.cell0[level] + lane; k < ci; k += 32) before += a.cell_n[static_cast<size_t>(frame) * a.n_cells + k];
		before = __reduce_add_sync(0xFFFFFFFFu, before);
		const int m = a.cell_n[static_cast<size_t>(frame) * a.n_cells + ci];
		const OctCell & c = a.cells[ci];
		const uint32_t * src = a.keys + static_cast<size_t>(frame) * a.key_stride + c.slot;
		for (int i = lane; i < m; i += 32) kk[before + i] = src[i];
	}
	__syncthreads();
	const int n = s_n;
	// initial nodes: keys binned by (int)(x / hX), stably, by warp 0; empty nodes dropped
	const int n_ini = g.n_ini[level];
	const float hx = g.hx[level];
	if (warp == 0)
	{
		int at = 0, len = 0;
		for (int b = 0; b < n_ini; ++b)
		{
			const int lo = at;
			for (int base = 0; base < n; base += 32)
			{
				const int i = base + lane;
				bool in = false;
				if (i < n)
				{
					const int x = static_cast<int>(kk[i] >> 8) % w - min_b;
					in = static_cast<int>(__fdiv_rn(static_cast<float>(x), hx)) == b;
				}
				const unsigned m = __ballot_sync(0xFFFFFFFFu, in);
				if (in) perm[at + __popc(m & ((1u << lane) - 1u))] = i;
				at += __popc(m);
			}
			if (at > lo && lane == 0)
			{
				OctNode nd;
				nd.x0 = static_cast<int>(__fmul_rn(hx, static_cast<float>(b)));
				nd.x1 = static_cast<int>(__fmul_rn(hx, static_cast<float>(b + 1)));
				nd.y0 = 0;
				nd.y1 = g.span_h[level];
				nd.lo = lo;
				nd.hi = at;
				nd.rank = b;
				nd.no_more = at - lo == 1;
				nodes[len] = nd;
			}
			if (at > lo) ++len;
		}
		if (lane == 0)
		{
			s_len = len;
			s_phase = 1;
			s_done = 0;
			s_n_exp = 0;
			s_buf = 0;
		}
	}
	__syncthreads();
	int rank = n_ini; // creation counter (thread 0's copy is the one used)
	while (!s_done)
	{
		const int buf = s_buf, len = s_len;
		OctNode * cur = nodes + buf * a.node_stride;
		OctNode * nxt = nodes + (buf ^ 1) * a.node_stride;
		// candidates: phase 1 every node that can be divided, in list order; phase 2 the last round's children with more than one key,
		// largest (size, rank) first
		if (s_phase == 1)
		{
			if (tid == 0)
			{
				int k = 0;
				for (int i = 0; i < len; ++i)
					if (!cur[i].no_more) cand[k++] = i;
				s_n_cand = k;
			}
		}
		else
		{
			const int m = s_n_exp;
			int pad = 1;
			while (pad < m) pad <<= 1;
			for (int i = tid; i < pad; i += blockDim.x)
			{
				unsigned long long key = 0ull;
				if (i < m)
				{
					const OctNode & nd = cur[expand[i]];
					key = (static_cast<unsigned long long>(nd.hi - nd.lo) << 40) | (static_cast<unsigned long long>(nd.rank) << 16) |
					      static_cast<unsigned long long>(expand[i]);
				}
				s_sort[i] = key;
			}
			block_sort_desc(s_sort, pad);
			for (int i = tid; i < m; i += blockDim.x) cand[i] = static_cast<int>(s_sort[i] & 0xFFFFull);
			if (tid == 0) s_n_cand = m;
		}
		__syncthreads();
		const int n_cand = s_n_cand;
		// children's key counts, one warp per candidate
		for (int k = warp; k < n_cand; k += n_warps)
		{
			const OctNode nd = cur[cand[k]];
			const int mx = nd.x0 + (nd.x1 - nd.x0 + 1) / 2, my = nd.y0 + (nd.y1 - nd.y0 + 1) / 2;
			int c4[4] = {0, 0, 0, 0};
			for (int base = nd.lo; base < nd.hi; base += 32) // the same trip count on every lane: the ballots need the whole warp
			{
				const int i = base + lane;
				const int ch = i < nd.hi ? oct_child(kk[perm[i]], w, min_b, mx, my) : -1;
#pragma unroll
				for (int q = 0; q < 4; ++q) c4[q] += __popc(__ballot_sync(0xFFFFFFFFu, ch == q));
			}
			if (lane == 0) cnt[k] = make_int4(c4[0], c4[1], c4[2], c4[3]);
		}
		__syncthreads();
		// how many candidates divide (phase 2 stops once the list reaches N), then the next list: the children pushed to the front (the
		// last pushed first), then the nodes that were not divided, in order
		if (tid == 0)
		{
			int j = n_cand;
			if (s_phase == 2)
			{
				int size = len;
				for (int k = 0; k < n_cand; ++k)
				{
					const int4 q = cnt[k];
					size += (q.x > 0) + (q.y > 0) + (q.z > 0) + (q.w > 0) - 1;
					if (size >= N)
					{
						j = k + 1;
						break;
					}
				}
			}
			int pushed = 0;
			for (int k = 0; k < j; ++k)
			{
				const int4 q = cnt[k];
				pushed += (q.x > 0) + (q.y > 0) + (q.z > 0) + (q.w > 0);
			}
			int at = pushed, n_exp = 0;
			for (int k = 0; k < j; ++k)
			{
				const OctNode nd = cur[cand[k]];
				const int mx = nd.x0 + (nd.x1 - nd.x0 + 1) / 2, my = nd.y0 + (nd.y1 - nd.y0 + 1) / 2;
				const int4 q = cnt[k];
				const int qc[4] = {q.x, q.y, q.z, q.w};
				const int rx0[4] = {nd.x0, mx, nd.x0, mx}, rx1[4] = {mx, nd.x1, mx, nd.x1};
				const int ry0[4] = {nd.y0, nd.y0, my, my}, ry1[4] = {my, my, nd.y1, nd.y1};
				int lo = nd.lo;
#pragma unroll
				for (int c = 0; c < 4; ++c)
				{
					if (qc[c] == 0) continue;
					OctNode ch;
					ch.x0 = rx0[c];
					ch.x1 = rx1[c];
					ch.y0 = ry0[c];
					ch.y1 = ry1[c];
					ch.lo = lo;
					ch.hi = lo + qc[c];
					ch.rank = rank++;
					ch.no_more = qc[c] == 1;
					nxt[--at] = ch;
					if (qc[c] > 1) expand[n_exp++] = at;
					lo += qc[c];
				}
				cur[cand[k]].no_more = -1; // divided: leaves the list
			}
			int out = pushed;
			for (int i = 0; i < len; ++i)
				if (cur[i].no_more >= 0) nxt[out++] = cur[i];
			s_j = j;
			s_n_exp = n_exp;
			s_len = out;
			s_buf = buf ^ 1;
			if (out >= N || out == len) s_done = 1;
			else if (s_phase == 1 && out + 3 * n_exp > N) s_phase = 2;
		}
		__syncthreads();
		// the divided segments: a stable four-way partition by child, one warp per node
		for (int k = warp; k < s_j; k += n_warps)
		{
			const OctNode nd = cur[cand[k]];
			const int mx = nd.x0 + (nd.x1 - nd.x0 + 1) / 2, my = nd.y0 + (nd.y1 - nd.y0 + 1) / 2;
			const int4 q = cnt[k];
			int base[4] = {nd.lo, nd.lo + q.x, nd.lo + q.x + q.y, nd.lo + q.x + q.y + q.z};
			for (int b0 = nd.lo; b0 < nd.hi; b0 += 32)
			{
				const int i = b0 + lane;
				const int p = i < nd.hi ? perm[i] : 0;
				const int ch = i < nd.hi ? oct_child(kk[p], w, min_b, mx, my) : -1;
#pragma unroll
				for (int c = 0; c < 4; ++c)
				{
					const unsigned m = __ballot_sync(0xFFFFFFFFu, ch == c);
					if (ch == c) scratch[base[c] + __popc(m & ((1u << lane) - 1u))] = p;
					base[c] += __popc(m);
				}
			}
			__syncwarp();
			for (int i = nd.lo + lane; i < nd.hi; i += 32) perm[i] = scratch[i];
			__syncwarp();
		}
		__syncthreads();
	}
	// the strongest key of each node, the first one in the node's order among equals; list order
	const OctNode * fin = nodes + s_buf * a.node_stride;
	const int len = s_len;
	for (int k = warp; k < len; k += n_warps)
	{
		const OctNode nd = fin[k];
		unsigned long long best = 0ull;
		for (int i = nd.lo + lane; i < nd.hi; i += 32)
		{
			const uint32_t key = kk[perm[i]];
			const unsigned long long v = (static_cast<unsigned long long>(key & 0xFFu) << 32) | static_cast<unsigned>(0x7FFFFFFF - (i - nd.lo));
			best = v > best ? v : best;
		}
		for (int o = 16; o > 0; o >>= 1)
		{
			const unsigned long long v = __shfl_xor_sync(0xFFFFFFFFu, best, o);
			best = v > best ? v : best;
		}
		if (lane == 0) a.sel[nbase + k] = kk[perm[nd.lo + (0x7FFFFFFF - static_cast<int>(best & 0xFFFFFFFFull))]];
	}
	if (tid == 0) a.sel_n[frame * g.n_levels + level] = len;
}

// ---- blur: cv::GaussianBlur(7x7, sigma 2) on a contiguous 8-bit level (fixed point) --------------------------------------------------
__global__ void orb_oct_blur_kernel(const uint8_t * __restrict__ pyr, uint8_t * __restrict__ blur, const OctGeom g, int level)
{
	const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
	const int w = g.w[level], h = g.h[level];
	if (x >= w || y >= h) return;
	const size_t base = static_cast<size_t>(blockIdx.z) * g.frame_stride + g.off[level];
	const uint8_t * img = pyr + base;
	constexpr int k[7] = {18, 34, 48, 56, 48, 34, 18};
	int col[7];
#pragma unroll
	for (int i = 0; i < 7; ++i) col[i] = reflect101(x + i - 3, w);
	unsigned acc = 0;
#pragma unroll
	for (int j = 0; j < 7; ++j)
	{
		const uint8_t * row = img + static_cast<size_t>(reflect101(y + j - 3, h)) * w;
		unsigned r = 0;
#pragma unroll
		for (int i = 0; i < 7; ++i) r += k[i] * row[col[i]];
		acc += k[j] * r;
	}
	blur[base + static_cast<size_t>(y) * w + x] = static_cast<uint8_t>(min((acc + 32768u) >> 16, 255u));
}

// ---- angle + descriptor of every kept key, one warp per key --------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
orb_oct_describe_kernel(const uint8_t * __restrict__ pyr, const uint8_t * __restrict__ blur, const OctGeom g, const uint32_t * __restrict__ sel,
                        const int * __restrict__ sel_n, int node_stride, OrbKeypoint * __restrict__ raw_kp, uint8_t * __restrict__ raw_desc)
{
	const int level = blockIdx.y, frame = blockIdx.z, lane = threadIdx.x & 31;
	const int k = blockIdx.x * 8 + (threadIdx.x >> 5);
	if (k >= sel_n[frame * g.n_levels + level]) return;
	int at = k;
	for (int l = 0; l < level; ++l) at += sel_n[frame * g.n_levels + l];
	const int w = g.w[level];
	const size_t plane = static_cast<size_t>(frame) * g.frame_stride + g.off[level];
	const uint8_t * img = pyr + plane;
	const uint8_t * blr = blur + plane;
	const uint32_t key = sel[static_cast<size_t>(frame) * node_stride + g.node0[level] + k];
	const int pos = static_cast<int>(key >> 8);
	const int x0 = pos % w, y0 = pos / w;
	// IC_Angle: lane = column u = lane - 15 of the circular patch, rows |v| <= the last v whose umax reaches |u|
	const int u = lane - 15;
	int m01 = 0, m10 = 0;
	if (u <= 15)
	{
		const int au = u < 0 ? -u : u;
		int sum = 0;
		for (int v = -15; v <= 15; ++v)
		{
			const int av = v < 0 ? -v : v;
			if ((av == 0 ? 15 : g.umax[av]) >= au)
			{
				const int val = img[static_cast<size_t>(y0 + v) * w + x0 + u];
				sum += val;
				m01 += v * val;
			}
		}
		m10 = u * sum;
	}
	m10 = __reduce_add_sync(0xFFFFFFFFu, m10);
	m01 = __reduce_add_sync(0xFFFFFFFFu, m01);
	const float angle = fast_atan2_deg(static_cast<float>(m01), static_cast<float>(m10));
	const float ar = __fmul_rn(angle, static_cast<float>(3.141592653589793238462643383279502884197169399375 / 180.0));
	const float ca = oct_sincosf(ar, 1), sa = oct_sincosf(ar, 0);
	// computeOrbDescriptor: byte = lane; every tap lies inside the level (ORB/EdgeThreshold >= 19)
	int val = 0;
#pragma unroll
	for (int b = 0; b < 8; ++b)
	{
		const int t = 8 * lane + b;
		const float px0 = kOrbPattern31[4 * t], py0 = kOrbPattern31[4 * t + 1], px1 = kOrbPattern31[4 * t + 2], py1 = kOrbPattern31[4 * t + 3];
		const int c0 = __float2int_rn(__fsub_rn(__fmul_rn(px0, ca), __fmul_rn(py0, sa)));
		const int r0 = __float2int_rn(__fadd_rn(__fmul_rn(px0, sa), __fmul_rn(py0, ca)));
		const int c1 = __float2int_rn(__fsub_rn(__fmul_rn(px1, ca), __fmul_rn(py1, sa)));
		const int r1 = __float2int_rn(__fadd_rn(__fmul_rn(px1, sa), __fmul_rn(py1, ca)));
		const int t0 = blr[static_cast<size_t>(y0 + r0) * w + x0 + c0], t1 = blr[static_cast<size_t>(y0 + r1) * w + x0 + c1];
		val |= (t0 < t1) << b;
	}
	const size_t row = static_cast<size_t>(frame) * g.raw_cap + at;
	raw_desc[row * 32 + lane] = static_cast<uint8_t>(val);
	if (lane == 0)
	{
		OrbKeypoint kp;
		const float sf = g.scale[level];
		kp.x = level ? __fmul_rn(static_cast<float>(x0), sf) : static_cast<float>(x0);
		kp.y = level ? __fmul_rn(static_cast<float>(y0), sf) : static_cast<float>(y0);
		kp.size = static_cast<float>(g.size[level]);
		kp.angle = angle;
		kp.response = static_cast<float>(key & 0xFFu);
		kp.octave = level;
		raw_kp[row] = kp;
	}
}

// ---- the wrapper: level-0 mask at the truncated coordinates, then Feature2D::limitKeypoints -------------------------------------------
__global__ void __launch_bounds__(1024)
orb_oct_finish_kernel(const OrbKeypoint * __restrict__ raw_kp, const uint8_t * __restrict__ raw_desc, const int * __restrict__ sel_n, const OctGeom g,
                      const uint8_t * __restrict__ mask, int max_features, OrbKeypoint * __restrict__ out, uint8_t * __restrict__ out_desc,
                      int * __restrict__ out_n, int out_cap)
{
	extern __shared__ __align__(16) unsigned long long skey[]; // [pad]
	__shared__ int s_warp[32];
	const int frame = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
	int total = 0;
	for (int l = 0; l < g.n_levels; ++l) total += sel_n[frame * g.n_levels + l];
	const OrbKeypoint * kp = raw_kp + static_cast<size_t>(frame) * g.raw_cap;
	const uint8_t * mk = mask ? mask + static_cast<size_t>(frame) * g.frame_stride : nullptr;
	int pad = 1;
	while (pad < total) pad <<= 1;
	// index of each kept keypoint, in order: skey[i] = raw index (the mask compaction), then sorted when the limit cuts
	int kept = 0;
	for (int base = 0; base < total; base += blockDim.x)
	{
		const int i = base + tid;
		bool keep = i < total;
		if (keep && mk)
			keep = mk[static_cast<size_t>(static_cast<int>(kp[i].y)) * g.w[0] + static_cast<int>(kp[i].x)] != 0;
		const unsigned b = __ballot_sync(0xFFFFFFFFu, keep);
		if (lane == 0) s_warp[warp] = __popc(b);
		__syncthreads();
		int before = 0, step = 0;
		for (int k = 0; k < static_cast<int>(blockDim.x >> 5); ++k)
		{
			before += k < warp ? s_warp[k] : 0;
			step += s_warp[k];
		}
		if (keep) skey[kept + before + __popc(b & ((1u << lane) - 1u))] = static_cast<unsigned long long>(i);
		kept += step;
		__syncthreads();
	}
	const bool cut = max_features > 0 && kept > max_features;
	if (cut)
	{
		// multimap<fabs(response), index> walked in reverse (limit_key's order), index = position after the mask; the raw index rides in
		// the low 16 bits (raw_cap < 65536)
		for (int i = tid; i < pad; i += blockDim.x)
			skey[i] = i < kept ? ((limit_key(kp[skey[i]].response, 0) & ~0xFFFFFFFFull) | (static_cast<unsigned long long>(i) << 16) | skey[i]) : 0ull;
		block_sort_desc(skey, pad);
		kept = max_features;
	}
	__syncthreads();
	const int n = min(kept, out_cap);
	for (int i = tid; i < n * 32; i += blockDim.x)
	{
		const int r = i >> 5;
		const int src = static_cast<int>(cut ? (skey[r] & 0xFFFFull) : skey[r]);
		if ((i & 31) == 0) out[static_cast<size_t>(frame) * out_cap + r] = kp[src];
		out_desc[(static_cast<size_t>(frame) * out_cap + r) * 32 + (i & 31)] = raw_desc[(static_cast<size_t>(frame) * g.raw_cap + src) * 32 + (i & 31)];
	}
	if (tid == 0) out_n[frame] = n;
}

} // namespace lcd
