// l2_path.cuh — the quantiser for FLOAT descriptors (SURF-64 / SURF-128 / SIFT, LCD_DESC_F32): exact squared-L2 2-NN and the
// NNDR / new-word loop, kept apart from the binary path (nn_tensor.cuh / nn_hamming.cuh / resolve.cuh), which it does not touch.
//
// Replaces, for CV_32F descriptors: FlannIndex::knnSearch on a LinearIndex (corelib/src/FlannIndex.cpp:701-745 ->
// rtflann/algorithms/linear_index.h:129-146, rtflann::L2<float>::operator() rtflann/algorithms/dist.h:133-180,
// KNNSimpleResultSet::addPoint rtflann/util/result_set.h:151-172) and the "Process results" loop of
// VWDictionary::addNewWords / findNN (corelib/src/VWDictionary.cpp:1088-1219, :1476-1546).
//
// Bit-exactness: rtflann's L2 sums the squared differences in groups of four (each group left to right, then added to the
// running total); l2_rtflann below performs the same additions in the same order without FMA contraction, so distances — and
// with them every tie-break and every NNDR decision — equal the CPU's.  Keys are 64-bit: (float bits of the distance << 32) |
// row; distances are >= 0, so unsigned order of the key is (distance, lowest row) order.
//
// knn2_l2_kernel is the exact CUDA-core scan (one query per thread, rows staged through shared memory), used for small dictionaries
// and as the cross-check of the tensor-core filter + exact re-rank of nn_tensor_f32.cuh (dictionaries of >= 4096 rows).
// resolve_l2_kernel settles the new-word loop with the chunked scheme of the binary path (parallel inside a frame, exact).
#pragma once
#include "common.cuh"
#include "resolve.cuh"

namespace lcd {

constexpr unsigned long long kKey64None = ~0ull;
constexpr int kL2Threads = 128;   // queries per CTA of the 2-NN kernel
constexpr int kL2TileRows = 32;   // vocabulary rows staged per shared-memory tile
constexpr int kL2ResolveThreads = 256;

__device__ __forceinline__ unsigned long long pack64(float d, uint32_t row)
{
	return (static_cast<unsigned long long>(__float_as_uint(d)) << 32) | row;
}
__device__ __forceinline__ float key64_dist(unsigned long long k) { return __uint_as_float(static_cast<uint32_t>(k >> 32)); }
__device__ __forceinline__ uint32_t key64_row(unsigned long long k) { return static_cast<uint32_t>(k); }
__device__ __forceinline__ void top2_insert64(unsigned long long & k1, unsigned long long & k2, unsigned long long key)
{
	const unsigned long long m = max(k1, key);
	k1 = min(k1, key);
	k2 = min(k2, m);
}

// rtflann::L2<float>::operator()(a, b, size): groups of four, each summed left to right, then added to the total
template <int DIM, class PA, class PB>
__device__ __forceinline__ float l2_rtflann(PA a, PB b)
{
	float result = 0.0f;
#pragma unroll
	for (int i = 0; i < DIM; i += 4)
	{
		const float d0 = __fsub_rn(a[i], b[i]), d1 = __fsub_rn(a[i + 1], b[i + 1]), d2 = __fsub_rn(a[i + 2], b[i + 2]),
		            d3 = __fsub_rn(a[i + 3], b[i + 3]);
		float g = __fadd_rn(__fmul_rn(d0, d0), __fmul_rn(d1, d1));
		g = __fadd_rn(g, __fmul_rn(d2, d2));
		g = __fadd_rn(g, __fmul_rn(d3, d3));
		result = __fadd_rn(result, g);
	}
	return result;
}

// Descriptors too wide to keep in registers (256-D): thread tid's distances from its own vector q (global, 16-byte aligned) to the nr
// rows staged in s_rows (DIM floats each), accumulated kL2Chunk dimensions at a time.  rtflann adds the groups of four to one running
// total from left to right, so carrying each row's total across the chunks (in s_acc[r * kThreads + tid]) gives its bits exactly.
constexpr int kL2Chunk = 64; // dimensions of q held in registers at a time
template <int DIM, int kThreads>
__device__ __forceinline__ void l2_chunked_rows(const float * __restrict__ q, const float * s_rows, int nr, float * s_acc, int tid)
{
	static_assert(DIM % kL2Chunk == 0, "whole chunks");
#pragma unroll 1
	for (int c = 0; c < DIM; c += kL2Chunk)
	{
		float qc[kL2Chunk];
		const float4 * q4 = reinterpret_cast<const float4 *>(q + c);
#pragma unroll
		for (int v = 0; v < kL2Chunk / 4; ++v)
		{
			const float4 x = q4[v];
			qc[4 * v] = x.x;
			qc[4 * v + 1] = x.y;
			qc[4 * v + 2] = x.z;
			qc[4 * v + 3] = x.w;
		}
#pragma unroll 1
		for (int r = 0; r < nr; ++r)
		{
			const float4 * b4 = reinterpret_cast<const float4 *>(s_rows + r * DIM + c);
			float result = c == 0 ? 0.0f : s_acc[r * kThreads + tid];
#pragma unroll
			for (int i = 0; i < kL2Chunk; i += 4)
			{
				const float4 v = b4[i >> 2];
				const float d0 = __fsub_rn(qc[i], v.x), d1 = __fsub_rn(qc[i + 1], v.y), d2 = __fsub_rn(qc[i + 2], v.z), d3 = __fsub_rn(qc[i + 3], v.w);
				float g = __fadd_rn(__fmul_rn(d0, d0), __fmul_rn(d1, d1));
				g = __fadd_rn(g, __fmul_rn(d2, d2));
				g = __fadd_rn(g, __fmul_rn(d3, d3));
				result = __fadd_rn(result, g);
			}
			s_acc[r * kThreads + tid] = result;
		}
	}
}

// partial[split * nq + query] = (best key, second key) over the rows [split * rows_per_split, ...) of the vocabulary
template <int DIM>
__global__ void __launch_bounds__(kL2Threads)
knn2_l2_kernel(const float * __restrict__ vocab, int n_rows, int row_offset, const float * __restrict__ queries, int nq,
               ulonglong2 * __restrict__ partial, int rows_per_split)
{
	__shared__ __align__(16) float s_rows[kL2TileRows * DIM];
	const int tid = threadIdx.x;
	const int qi = blockIdx.x * kL2Threads + tid;
	const int r_begin = blockIdx.y * rows_per_split, r_end = min(n_rows, r_begin + rows_per_split);
	if constexpr (DIM > 128)
	{
		// the query stays in global memory (L1) and is read a chunk at a time; 32 KB of rows + 16 KB of running totals
		__shared__ float s_acc[kL2TileRows * kL2Threads];
		const float * q = queries + static_cast<size_t>(min(qi, max(nq - 1, 0))) * DIM;
		unsigned long long k1 = kKey64None, k2 = kKey64None;
		for (int r0 = r_begin; r0 < r_end; r0 += kL2TileRows)
		{
			const int nr = min(kL2TileRows, r_end - r0);
			__syncthreads();
			for (int i = tid; i < nr * (DIM / 4); i += kL2Threads)
				reinterpret_cast<float4 *>(s_rows)[i] = reinterpret_cast<const float4 *>(vocab + static_cast<size_t>(r0) * DIM)[i];
			__syncthreads();
			if (qi < nq)
			{
				l2_chunked_rows<DIM, kL2Threads>(q, s_rows, nr, s_acc, tid);
				for (int r = 0; r < nr; ++r) top2_insert64(k1, k2, pack64(s_acc[r * kL2Threads + tid], static_cast<uint32_t>(row_offset + r0 + r)));
			}
		}
		if (qi < nq) partial[static_cast<size_t>(blockIdx.y) * nq + qi] = make_ulonglong2(k1, k2);
	}
	else
	{
		float q[DIM];
#pragma unroll
		for (int i = 0; i < DIM; ++i) q[i] = qi < nq ? queries[static_cast<size_t>(qi) * DIM + i] : 0.0f;
		unsigned long long k1 = kKey64None, k2 = kKey64None;
		for (int r0 = r_begin; r0 < r_end; r0 += kL2TileRows)
		{
			const int nr = min(kL2TileRows, r_end - r0);
			__syncthreads();
			for (int i = tid; i < nr * DIM; i += kL2Threads) s_rows[i] = vocab[static_cast<size_t>(r0) * DIM + i];
			__syncthreads();
			for (int r = 0; r < nr; ++r)
			{
				const float d = l2_rtflann<DIM>(q, s_rows + r * DIM);
				top2_insert64(k1, k2, pack64(d, static_cast<uint32_t>(row_offset + r0 + r)));
			}
		}
		if (qi < nq) partial[static_cast<size_t>(blockIdx.y) * nq + qi] = make_ulonglong2(k1, k2);
	}
}

// lcd_dict_knn2 for float descriptors: merge the splits, decode to (word id, squared distance)
__global__ void knn2_l2_decode_kernel(const ulonglong2 * __restrict__ partial, int n_splits, int nq, const int * __restrict__ row_ids,
                                      int * __restrict__ id1, float * __restrict__ d1, int * __restrict__ id2, float * __restrict__ d2)
{
	const int qi = blockIdx.x * blockDim.x + threadIdx.x;
	if (qi >= nq) return;
	unsigned long long k1 = kKey64None, k2 = kKey64None;
	for (int c = 0; c < n_splits; ++c)
	{
		const ulonglong2 p = partial[static_cast<size_t>(c) * nq + qi];
		top2_insert64(k1, k2, p.x);
		top2_insert64(k1, k2, p.y);
	}
	id1[qi] = k1 == kKey64None ? 0 : row_ids[key64_row(k1)];
	d1[qi] = k1 == kKey64None ? -1.0f : key64_dist(k1);
	id2[qi] = k2 == kKey64None ? 0 : row_ids[key64_row(k2)];
	d2[qi] = k2 == kKey64None ? -1.0f : key64_dist(k2);
}

// lcd_shard_knn2_keys_dev for float descriptors: merge the splits (n_splits of the exact kernel, 1 of the fp16 filter path) into one
// key pair per query, in the order of the unsharded merge, so that ties go to the lowest global row
__global__ void knn2_merge64_kernel(const ulonglong2 * __restrict__ partial, int n_splits, int nq, ulonglong2 * __restrict__ out)
{
	const int qi = blockIdx.x * blockDim.x + threadIdx.x;
	if (qi >= nq) return;
	unsigned long long k1 = kKey64None, k2 = kKey64None;
	for (int c = 0; c < n_splits; ++c)
	{
		const ulonglong2 p = partial[static_cast<size_t>(c) * nq + qi];
		top2_insert64(k1, k2, p.x);
		top2_insert64(k1, k2, p.y);
	}
	out[qi] = make_ulonglong2(k1, k2);
}

// The decision on the multimap<float,int> fullResults of one descriptor (VWDictionary.cpp:1162-1219): candidates in insertion
// order a1, a2 (index hits), n1, n2 (hits among this frame's new words); strict '<' keeps the earlier entry on ties.
__device__ __forceinline__ bool nndr_decide64(unsigned long long a1, unsigned long long a2, unsigned long long n1, unsigned long long n2,
                                              float nndr, int & best_tag)
{
	float bd = INFINITY, sd = INFINITY;
	int bt = -1, cnt = 0;
	const unsigned long long keys[4] = {a1, a2, n1, n2};
#pragma unroll
	for (int t = 0; t < 4; ++t)
	{
		if (keys[t] != kKey64None)
		{
			const float d = key64_dist(keys[t]);
			++cnt;
			if (d < bd)
			{
				sd = bd;
				bd = d;
				bt = t;
			}
			else if (d < sd) sd = d;
		}
	}
	best_tag = bt;
	return cnt < 2 || bd > __fmul_rn(nndr, sd);
}

// Intra-frame new-word resolution for one frame of FLOAT descriptors: the chunked scheme of resolve_rounds (resolve.cuh) with exact
// squared-L2 distances in rtflann's order.  The reference decides descriptor i after descriptors 0..i-1 (VWDictionary.cpp:1139-1219);
// here the frame is walked in chunks of 32: (A) one warp per descriptor of the chunk finds its two nearest among the words created by
// EARLIER chunks (already final) and its distances to the 32 chunk-mates, all warps in parallel; (B) one warp settles the dependencies
// inside the chunk by fixed-point iteration over a ballot mask; (C) the chunk's new words join the list.
// sa1 / sa2: each descriptor's two best index hits (64-bit keys).  Returns the number of created words; flag / rank / L / res as in
// resolve_rounds.
// exact rtflann-order distance between a descriptor held in registers and a vector streamed with 16-byte loads (all lanes of a
// warp read the same address: one transaction per load)
template <int DIM>
__device__ __forceinline__ float l2_reg_vs_stream(const float (&a)[DIM], const float * __restrict__ b)
{
	const float4 * b4 = reinterpret_cast<const float4 *>(b);
	float result = 0.0f;
#pragma unroll
	for (int i = 0; i < DIM; i += 4)
	{
		const float4 v = b4[i >> 2];
		const float d0 = __fsub_rn(a[i], v.x), d1 = __fsub_rn(a[i + 1], v.y), d2 = __fsub_rn(a[i + 2], v.z), d3 = __fsub_rn(a[i + 3], v.w);
		float g = __fadd_rn(__fmul_rn(d0, d0), __fmul_rn(d1, d1));
		g = __fadd_rn(g, __fmul_rn(d2, d2));
		g = __fadd_rn(g, __fmul_rn(d3, d3));
		result = __fadd_rn(result, g);
	}
	return result;
}

// the same with the descriptor in (shared) memory: a[i] is read per element
template <int DIM>
__device__ __forceinline__ float l2_ptr_vs_stream(const float * a, const float * __restrict__ b)
{
	const float4 * b4 = reinterpret_cast<const float4 *>(b);
	float result = 0.0f;
#pragma unroll 16
	for (int i = 0; i < DIM; i += 4)
	{
		const float4 v = b4[i >> 2];
		const float d0 = __fsub_rn(a[i], v.x), d1 = __fsub_rn(a[i + 1], v.y), d2 = __fsub_rn(a[i + 2], v.z), d3 = __fsub_rn(a[i + 3], v.w);
		float g = __fadd_rn(__fmul_rn(d0, d0), __fmul_rn(d1, d1));
		g = __fadd_rn(g, __fmul_rn(d2, d2));
		g = __fadd_rn(g, __fmul_rn(d3, d3));
		result = __fadd_rn(result, g);
	}
	return result;
}

template <int DIM>
__device__ int resolve_rounds_l2(const float * __restrict__ fq, int nq, const unsigned long long * sa1, const unsigned long long * sa2, int * res,
                                 uint16_t * L, uint16_t * rank, uint8_t * flag, int * s_nL, float nndr, int cmp_new)
{
	constexpr int kWarps = kL2ResolveThreads / 32;
	__shared__ __align__(16) unsigned long long s_wk[kWarps][32][2]; // per warp, per descriptor of the chunk: best two among the created words it scanned
	__shared__ float s_dl[32][33];                     // s_dl[e][j] = distance between descriptors c0+e and c0+j of the current chunk
	const int tid = threadIdx.x;
	const int warp = tid >> 5, lane = tid & 31;
	if (!cmp_new)
	{
		if (tid < 32)
		{
			const int n = warp0_compact(flag, nq, L, rank);
			if (tid == 0) *s_nL = n;
		}
		__syncthreads();
		return *s_nL;
	}
	if (tid == 0) *s_nL = 0;
	__syncthreads();
	for (int c0 = 0; c0 < nq; c0 += 32)
	{
		const int nL = *s_nL;
		// (A) lane j of EVERY warp holds descriptor c0 + j in registers; the warps share out the vectors it is compared with (the 32
		// chunk-mates and the nL words created so far), each streamed once per warp with broadcast loads.  256-D: the descriptor does
		// not fit in registers, so the chunk's 32 descriptors are staged in shared memory (row stride DIM + 1: lane j reads bank j + i)
		if constexpr (DIM > 128)
		{
			__shared__ float s_cq[32 * (DIM + 1)]; // the previous chunk's readers passed the barrier at the end of the loop
			for (int v = tid; v < 32 * DIM; v += blockDim.x)
				s_cq[(v / DIM) * (DIM + 1) + v % DIM] = fq[static_cast<size_t>(min(c0 + v / DIM, nq - 1)) * DIM + v % DIM];
			__syncthreads();
			const float * q = s_cq + lane * (DIM + 1);
			for (int e = warp; e < 32; e += kWarps)
			{
				const int m = c0 + e;
				s_dl[e][lane] = m < nq ? l2_ptr_vs_stream<DIM>(q, fq + static_cast<size_t>(m) * DIM) : INFINITY;
			}
			unsigned long long k1 = kKey64None, k2 = kKey64None;
			for (int k = warp; k < nL; k += kWarps)
			{
				const float d = l2_ptr_vs_stream<DIM>(q, fq + static_cast<size_t>(L[k]) * DIM);
				top2_insert64(k1, k2, pack64(d, static_cast<uint32_t>(k)));
			}
			s_wk[warp][lane][0] = k1;
			s_wk[warp][lane][1] = k2;
		}
		else
		{
			const int i = min(c0 + lane, nq - 1);
			float q[DIM];
			const float4 * q4 = reinterpret_cast<const float4 *>(fq + static_cast<size_t>(i) * DIM);
#pragma unroll
			for (int v = 0; v < DIM / 4; ++v)
			{
				const float4 x = q4[v];
				q[4 * v] = x.x;
				q[4 * v + 1] = x.y;
				q[4 * v + 2] = x.z;
				q[4 * v + 3] = x.w;
			}
			for (int e = warp; e < 32; e += kWarps)
			{
				const int m = c0 + e;
				s_dl[e][lane] = m < nq ? l2_reg_vs_stream<DIM>(q, fq + static_cast<size_t>(m) * DIM) : INFINITY;
			}
			unsigned long long k1 = kKey64None, k2 = kKey64None;
			for (int k = warp; k < nL; k += kWarps)
			{
				const float d = l2_reg_vs_stream<DIM>(q, fq + static_cast<size_t>(L[k]) * DIM);
				top2_insert64(k1, k2, pack64(d, static_cast<uint32_t>(k)));
			}
			s_wk[warp][lane][0] = k1;
			s_wk[warp][lane][1] = k2;
		}
		__syncthreads();
		if (warp == 0)
		{
			const int i = c0 + lane;
			const bool valid = i < nq;
			float dl[32];
#pragma unroll
			for (int jl = 0; jl < 32; ++jl) dl[jl] = s_dl[jl][lane]; // the matrix is symmetric; this read is conflict-free
			const unsigned long long a1 = valid ? sa1[i] : kKey64None, a2 = valid ? sa2[i] : kKey64None;
			unsigned long long e1 = kKey64None, e2 = kKey64None;
#pragma unroll
			for (int w = 0; w < kWarps; ++w)
			{
				top2_insert64(e1, e2, s_wk[w][lane][0]);
				top2_insert64(e1, e2, s_wk[w][lane][1]);
			}
			int bt;
			bool bad = valid && nndr_decide64(a1, a2, e1, e2, nndr, bt);
			unsigned long long n1 = e1;
			uint32_t mask = __ballot_sync(0xFFFFFFFFu, bad);
			for (int r = 0; r < 33; ++r)
			{
				n1 = e1;
				unsigned long long n2 = e2;
#pragma unroll
				for (int jl = 0; jl < 32; ++jl)
				{
					if (jl < lane && ((mask >> jl) & 1u))
					{
						const uint32_t kidx = static_cast<uint32_t>(nL) + __popc(mask & ((1u << jl) - 1u));
						top2_insert64(n1, n2, pack64(dl[jl], kidx));
					}
				}
				bad = valid && nndr_decide64(a1, a2, n1, n2, nndr, bt);
				const uint32_t nm = __ballot_sync(0xFFFFFFFFu, bad);
				if (nm == mask) break;
				mask = nm;
			}
			if (valid)
			{
				flag[i] = bad ? 1 : 0;
				if (bad)
				{
					const int k = nL + __popc(mask & ((1u << lane) - 1u));
					rank[i] = static_cast<uint16_t>(k);
					L[k] = static_cast<uint16_t>(i);
				}
				else res[i] = bt >= 2 ? -1 - static_cast<int>(key64_row(n1)) : static_cast<int>(key64_row(a1));
			}
			if (lane == 0) *s_nL = nL + __popc(mask);
		}
		__syncthreads();
	}
	return *s_nL;
}

__host__ __device__ inline size_t resolve_l2_smem_bytes(int cap)
{
	int nq_pad = 32;
	while (nq_pad < cap) nq_pad <<= 1;
	return static_cast<size_t>(cap) * (8 + 8 + 4 + 2 + 2 + 1) + static_cast<size_t>(nq_pad) * 4 + 64;
}

// One CTA per frame.  Dynamic shared memory: resolve_l2_smem_bytes(a.nq).
template <int DIM>
__global__ void __launch_bounds__(kL2ResolveThreads)
resolve_l2_kernel(const ResolveArgs a, const ulonglong2 * __restrict__ partial64)
{
	extern __shared__ __align__(128) unsigned char smem_raw[];
	const int cap = a.nq;
	int nq_pad = 32;
	while (nq_pad < cap) nq_pad <<= 1;
	unsigned long long * sa1 = reinterpret_cast<unsigned long long *>(smem_raw);
	unsigned long long * sa2 = sa1 + cap;
	uint32_t * sbuf = reinterpret_cast<uint32_t *>(sa2 + cap); // [nq_pad]
	int * res = reinterpret_cast<int *>(sbuf + nq_pad);        // >=0 row, -1-k new word k, INT_MIN none
	uint16_t * L = reinterpret_cast<uint16_t *>(res + cap);
	uint16_t * rank = L + cap;
	uint8_t * flag = reinterpret_cast<uint8_t *>(rank + cap);
	__shared__ int s_nL;

	const int tid = threadIdx.x;
	const int frame = blockIdx.x;
	const int nq = a.nq_frame ? min(max(a.nq_frame[frame], 0), cap) : cap;
	const float * fq = reinterpret_cast<const float *>(a.queries) + static_cast<size_t>(frame) * cap * DIM;
	const size_t pbase = static_cast<size_t>(frame) * cap;

	// 1. merge the per-split top-2 keys (FlannIndex::knnSearch result of this descriptor) and take the index-only decision
	for (int i = tid; i < nq; i += blockDim.x)
	{
		unsigned long long k1 = kKey64None, k2 = kKey64None;
		for (int c = 0; c < a.n_chunks; ++c)
		{
			const ulonglong2 p = partial64[static_cast<size_t>(c) * a.nq_total + pbase + i];
			top2_insert64(k1, k2, p.x);
			top2_insert64(k1, k2, p.y);
		}
		sa1[i] = k1;
		sa2[i] = k2;
		int bt;
		const bool bad = nndr_decide64(k1, k2, kKey64None, kKey64None, a.nndr, bt);
		if (a.incremental)
		{
			flag[i] = bad ? 1 : 0;
			res[i] = static_cast<int>(key64_row(k1));
		}
		else
		{
			// fixed dictionary: nearest word, no NNDR (VWDictionary.cpp:1211-1218)
			flag[i] = 0;
			res[i] = k1 != kKey64None ? static_cast<int>(key64_row(k1)) : INT_MIN;
		}
	}
	__syncthreads();

	int n_new = 0;
	if (a.incremental)
	{
		// 2. intra-frame dependency among the words this frame creates (findNN creates none: every descriptor stands alone)
		n_new = resolve_rounds_l2<DIM>(fq, nq, sa1, sa2, res, L, rank, flag, &s_nL, a.nndr, a.find_only ? 0 : a.cmp_new);
	}

	// 3. word ids in creation order, and the created words into the not-indexed tail of the vocabulary (single-frame quantise)
	int n_valid = 0;
	for (int i = tid; i < nq; i += blockDim.x)
	{
		int wid;
		uint32_t sv = kSortNone;
		if (flag[i]) wid = a.find_only ? 0 : a.last_word_id + 1 + rank[i];
		else if (res[i] == INT_MIN) wid = 0;
		else if (res[i] < 0) wid = a.last_word_id + 1 + (-1 - res[i]);
		else
		{
			wid = a.row_ids[res[i]];
			sv = static_cast<uint32_t>(wid);
		}
		if (a.word_ids_out) a.word_ids_out[pbase + i] = wid;
		sbuf[i] = sv;
		n_valid += wid > 0;
	}
	for (int i = nq + tid; i < nq_pad; i += blockDim.x)
	{
		sbuf[i] = kSortNone;
		if (i < cap && a.word_ids_out) a.word_ids_out[pbase + i] = 0; // padding rows of a short frame
	}
	if (a.pending_desc && !a.find_only)
	{
		float * dst = reinterpret_cast<float *>(a.pending_desc);
		const int lane = tid & 31, warp = tid >> 5;
		for (int k = warp; k < n_new; k += static_cast<int>(blockDim.x >> 5))
		{
			for (int v = lane; v < DIM; v += 32) dst[static_cast<size_t>(k) * DIM + v] = fq[static_cast<size_t>(L[k]) * DIM + v];
			if (lane == 0) a.pending_ids[k] = a.last_word_id + 1 + k;
		}
	}
	if (tid == 0 && a.n_new_out) a.n_new_out[frame] = (a.find_only ? 0 : n_new);
	if (a.q_valid) cta_count_store(n_valid, a.q_valid + frame);
	__syncthreads();
	if (a.do_prep) score_prep(sbuf, nq_pad, cap, a, frame);
}

} // namespace lcd
