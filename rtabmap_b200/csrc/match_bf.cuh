// match_bf.cuh — brute-force descriptor matching of two descriptor sets (lcd_match_bf).
//
// Replaces cv::BFMatcher as RTAB-Map's registration uses it on a signature pair:
//   mode LCD_MATCH_KNN2        cv::BFMatcher(norm).knnMatch(query, train, k = 2)           (RegistrationVis.cpp:1128-1141, :1280-1300)
//   mode LCD_MATCH_CROSSCHECK  cv::BFMatcher(norm, crossCheck = true).match(query, train)  (RegistrationVis.cpp:1452-1453, Vis/CorNNType=5)
// norm = NORM_HAMMING for CV_8U rows, NORM_L2SQR for CV_32F rows.  cv::BFMatcher is third-party (OpenCV features2d, not under
// /root/reference); its published behaviour restated here:
//   knnMatch   : per query the k nearest train rows, ties -> lowest train index (cv::batchDistance keeps the first minimum);
//   crossCheck : a query q is matched to its nearest train row t (ties -> lowest t) only if q is in turn the nearest query of t
//                (ties -> lowest q); other queries get no DMatch.  Verified against cv2 4.13 on tie-heavy random sets
//                (tests/test_gpu_boundary.py).
// Sizes are those of one signature pair (<= 4096 rows each), so one thread scans one row of one side against a shared-memory
// tile of the other.
#pragma once
#include "common.cuh"
#include "nn_hamming.cuh"
#include "l2_path.cuh"

namespace lcd {

constexpr int kBfThreads = 128;
constexpr int kBfTile = 64; // rows of the scanned side staged per shared-memory tile

struct BfAsFloat
{
	const uint32_t * p;
	__device__ __forceinline__ float operator[](int i) const { return __uint_as_float(p[i]); }
};

template <int NW, bool F32>
__device__ __forceinline__ unsigned long long bf_key(const uint32_t (&q)[NW], const uint32_t * row, uint32_t idx)
{
	if constexpr (F32)
	{
		const float d = l2_rtflann<NW>(BfAsFloat{q}, BfAsFloat{row});
		return pack64(d, idx);
	}
	else
	{
		uint32_t w[NW];
#pragma unroll
		for (int v = 0; v < NW; ++v) w[v] = row[v];
		const uint32_t d = hamming<NW, (NW == 8 ? 2 : 0)>(q, w);
		return (static_cast<unsigned long long>(d) << 32) | idx;
	}
}

// For every row i of A (n_a rows): the two nearest rows of B as packed keys (distance bits << 32 | index of B); kKey64None = none.
// grid = (ceil(n_a / kBfThreads), n_pairs); A and B hold `cap` rows per pair.
template <int NW, bool F32>
__global__ void __launch_bounds__(kBfThreads)
bf_knn2_kernel(const uint32_t * __restrict__ A, const int * __restrict__ n_a, const uint32_t * __restrict__ B, const int * __restrict__ n_b, int cap,
               ulonglong2 * __restrict__ keys /* [n_pairs][cap] */)
{
	__shared__ __align__(16) uint32_t s_rows[kBfTile * NW];
	const int pair = blockIdx.y, tid = threadIdx.x;
	const int na = min(n_a[pair], cap), nb = min(n_b[pair], cap);
	const int i = blockIdx.x * kBfThreads + tid;
	if (blockIdx.x * kBfThreads >= na) return;
	const uint32_t * a = A + static_cast<size_t>(pair) * cap * NW;
	const uint32_t * b = B + static_cast<size_t>(pair) * cap * NW;
	uint32_t q[NW];
#pragma unroll
	for (int v = 0; v < NW; ++v) q[v] = i < na ? a[static_cast<size_t>(i) * NW + v] : 0u;
	unsigned long long k1 = kKey64None, k2 = kKey64None;
	for (int r0 = 0; r0 < nb; r0 += kBfTile)
	{
		const int nr = min(kBfTile, nb - r0);
		__syncthreads();
		for (int t = tid; t < nr * NW; t += kBfThreads) s_rows[t] = b[static_cast<size_t>(r0) * NW + t];
		__syncthreads();
		for (int r = 0; r < nr; ++r) top2_insert64(k1, k2, bf_key<NW, F32>(q, s_rows + r * NW, static_cast<uint32_t>(r0 + r)));
	}
	if (i < na) keys[static_cast<size_t>(pair) * cap + i] = make_ulonglong2(k1, k2);
}

// bf_knn2_kernel for 256-D float rows, whose query does not fit in registers: it is read a chunk at a time (l2_chunked_rows,
// l2_path.cuh), with kBfTile / 2 rows per tile so that the rows (32 KB) and their running totals (16 KB) fit the static shared memory.
template <int DIM>
__global__ void __launch_bounds__(kBfThreads)
bf_knn2_l2_chunked_kernel(const uint32_t * __restrict__ A, const int * __restrict__ n_a, const uint32_t * __restrict__ B, const int * __restrict__ n_b,
                          int cap, ulonglong2 * __restrict__ keys /* [n_pairs][cap] */)
{
	constexpr int kTile = kBfTile / 2;
	__shared__ __align__(16) float s_rows[kTile * DIM];
	__shared__ float s_acc[kTile * kBfThreads];
	const int pair = blockIdx.y, tid = threadIdx.x;
	const int na = min(n_a[pair], cap), nb = min(n_b[pair], cap);
	const int i = blockIdx.x * kBfThreads + tid;
	if (blockIdx.x * kBfThreads >= na) return;
	const float * q = reinterpret_cast<const float *>(A) + (static_cast<size_t>(pair) * cap + min(i, na - 1)) * DIM;
	const float4 * b4 = reinterpret_cast<const float4 *>(B) + static_cast<size_t>(pair) * cap * (DIM / 4);
	unsigned long long k1 = kKey64None, k2 = kKey64None;
	for (int r0 = 0; r0 < nb; r0 += kTile)
	{
		const int nr = min(kTile, nb - r0);
		__syncthreads();
		for (int t = tid; t < nr * (DIM / 4); t += kBfThreads) reinterpret_cast<float4 *>(s_rows)[t] = b4[static_cast<size_t>(r0) * (DIM / 4) + t];
		__syncthreads();
		l2_chunked_rows<DIM, kBfThreads>(q, s_rows, nr, s_acc, tid);
		for (int r = 0; r < nr; ++r) top2_insert64(k1, k2, pack64(s_acc[r * kBfThreads + tid], static_cast<uint32_t>(r0 + r)));
	}
	if (i < na) keys[static_cast<size_t>(pair) * cap + i] = make_ulonglong2(k1, k2);
}

// cross check: query q keeps its nearest train row t only if q is also the nearest query of t (ties -> lowest index on both sides).
// query_keys[pair][q].x = (distance, t), train_keys[pair][t].x = (distance, q).
__global__ void bf_cross_kernel(const ulonglong2 * __restrict__ query_keys, const ulonglong2 * __restrict__ train_keys, const int * __restrict__ n_query,
                                int cap, unsigned long long * __restrict__ best)
{
	const int pair = blockIdx.y;
	const int q = blockIdx.x * blockDim.x + threadIdx.x;
	if (q >= cap) return;
	unsigned long long out = kKey64None;
	if (q < min(n_query[pair], cap))
	{
		const unsigned long long k = query_keys[static_cast<size_t>(pair) * cap + q].x;
		if (k != kKey64None)
		{
			const unsigned long long kt = train_keys[static_cast<size_t>(pair) * cap + static_cast<uint32_t>(k)].x;
			if (kt != kKey64None && static_cast<uint32_t>(kt) == static_cast<uint32_t>(q)) out = k;
		}
	}
	best[static_cast<size_t>(pair) * cap + q] = out;
}

// decode packed keys into (index, distance as float); index -1 / distance -1 = none
template <bool F32>
__global__ void bf_decode_kernel(const unsigned long long * __restrict__ keys, int stride_keys /* 1 or 2 keys per row */, int which, int n,
                                 int * __restrict__ idx, float * __restrict__ dist)
{
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	const unsigned long long k = keys[static_cast<size_t>(i) * stride_keys + which];
	if (k == kKey64None)
	{
		idx[i] = -1;
		dist[i] = -1.0f;
		return;
	}
	idx[i] = static_cast<int>(static_cast<uint32_t>(k));
	dist[i] = F32 ? __uint_as_float(static_cast<uint32_t>(k >> 32)) : static_cast<float>(static_cast<uint32_t>(k >> 32));
}

} // namespace lcd
