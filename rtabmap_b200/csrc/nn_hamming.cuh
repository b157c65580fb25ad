// nn_hamming.cuh — exact 2-nearest-neighbour search of binary descriptors over the
// device-resident vocabulary (the "dictionary NN" kernel of the hot path).
//
// Replaces: FlannIndex::knnSearch(k=2) -> rtflann::LinearIndex::findNeighbors
// (corelib/src/rtflann/algorithms/linear_index.h:129-146) with rtflann::Hamming
// (dist.h:533-580) and KNNSimpleResultSet::addPoint (util/result_set.h:151-172), as
// called from VWDictionary::addNewWords (corelib/src/VWDictionary.cpp:1015-1024).
//
// Design (H100): the vocabulary is split into contiguous row chunks, one per CTA.  A CTA
// pulls its chunk from L2/HBM into shared memory ONCE with 1-D bulk async copies (TMA
// engine, mbarrier completion), so the vocabulary is read exactly once per launch
// (algorithmic bytes W*D).  Each thread keeps TQ query descriptors in registers and walks
// the chunk with warp-uniform (broadcast) LDS.128 reads: per (query,word) pair the work is
// NW XOR + popcount + adds and a branch-free top-2 update on a packed (dist<<22|row) key.
// Per-chunk top-2 keys go to a [chunk][query] scratch array; the resolve kernel merges
// them.  The kernel is integer-pipe (POPC/LOP3) bound, not HBM bound: the vocabulary of
// every BASELINE config fits in the 126 MB L2 (SURVEY.md F9).
#pragma once
#include "common.cuh"

namespace lcd {

constexpr int kNnThreads = 256;

// ---- distance variants ------------------------------------------------------------
// 0: plain        NW x (LOP3 + POPC) + adds
// 1: Harley-Seal  carry-save adders trade POPC (16 lanes/clk/SM) for LOP3 (64 lanes/clk/SM):
//                 8 words -> 4 POPC
// 2: partial CSA  8 words -> 5 POPC, fewer LOP3 than variant 1
__device__ __forceinline__ void csa(uint32_t a, uint32_t b, uint32_t c, uint32_t & s, uint32_t & cy)
{
	s = a ^ b ^ c;
	cy = (a & b) | (c & (a ^ b));
}

template <int NW, int VARIANT>
__device__ __forceinline__ uint32_t hamming(const uint32_t (&q)[NW], const uint32_t (&w)[NW])
{
	if constexpr (NW == 8 && VARIANT == 1)
	{
		uint32_t x[8];
#pragma unroll
		for (int i = 0; i < 8; ++i) x[i] = q[i] ^ w[i];
		uint32_t sA, cA, sB, cB, sC, cC, sD, cD;
		csa(x[0], x[1], x[2], sA, cA);
		csa(x[3], x[4], x[5], sB, cB);
		csa(x[6], x[7], sA, sC, cC);
		csa(cA, cB, cC, sD, cD);
		return __popc(sB) + __popc(sC) + 2 * __popc(sD) + 4 * __popc(cD);
	}
	else if constexpr (NW == 8 && VARIANT == 2)
	{
		uint32_t x[8];
#pragma unroll
		for (int i = 0; i < 8; ++i) x[i] = q[i] ^ w[i];
		uint32_t sA, cA, sB, cB, sC, cC;
		csa(x[0], x[1], x[2], sA, cA);
		csa(x[3], x[4], x[5], sB, cB);
		csa(x[6], x[7], sA, sC, cC);
		return __popc(sB) + __popc(sC) + 2 * (__popc(cA) + __popc(cB) + __popc(cC));
	}
	else
	{
		uint32_t d = 0;
#pragma unroll
		for (int i = 0; i < NW; ++i) d += __popc(q[i] ^ w[i]);
		return d;
	}
}

// partial[chunk * nq + query] = (best key, second key) of `query` over the chunk's rows.
// Shared memory: 16 B (mbarrier) + rows_per_cta * NW * 4 B.
template <int NW, int TQ, int VARIANT>
__global__ void __launch_bounds__(kNnThreads)
knn2_hamming_kernel(const uint32_t * __restrict__ vocab, int n_rows, int row_offset,
                    const uint32_t * __restrict__ queries, int nq,
                    uint2 * __restrict__ partial, int rows_per_cta)
{
	extern __shared__ __align__(128) unsigned char smem_raw[];
	uint64_t * bar = reinterpret_cast<uint64_t *>(smem_raw);
	const uint4 * s_rows = reinterpret_cast<const uint4 *>(smem_raw + 16);

	const int tid = threadIdx.x;
	const int row_begin = blockIdx.x * rows_per_cta;
	const int row_end = min(n_rows, row_begin + rows_per_cta);
	const int nr = max(0, row_end - row_begin);

	if (tid == 0)
	{
		mbar_init(bar, 1);
		mbar_fence_init();
	}
	__syncthreads();
	if (tid == 0 && nr > 0)
	{
		const uint32_t bytes = static_cast<uint32_t>(nr) * NW * 4u;
		mbar_arrive_expect_tx(bar, bytes);
		const unsigned char * src = reinterpret_cast<const unsigned char *>(vocab + static_cast<size_t>(row_begin) * NW);
		unsigned char * dst = smem_raw + 16;
		for (uint32_t off = 0; off < bytes; off += 32768u)
		{
			bulk_g2s(dst + off, src + off, min(32768u, bytes - off), bar);
		}
	}

	bool waited = false;
	for (int qbase = 0; qbase < nq; qbase += kNnThreads * TQ)
	{
		uint32_t q[TQ][NW];
		uint32_t k1[TQ], k2[TQ];
#pragma unroll
		for (int t = 0; t < TQ; ++t)
		{
			const int qi = qbase + t * kNnThreads + tid;
			k1[t] = kKeyNone;
			k2[t] = kKeyNone;
			if (qi < nq)
			{
				const uint4 * src = reinterpret_cast<const uint4 *>(queries + static_cast<size_t>(qi) * NW);
#pragma unroll
				for (int v = 0; v < NW / 4; ++v)
				{
					uint4 x = __ldg(src + v);
					q[t][4 * v + 0] = x.x;
					q[t][4 * v + 1] = x.y;
					q[t][4 * v + 2] = x.z;
					q[t][4 * v + 3] = x.w;
				}
			}
			else
			{
#pragma unroll
				for (int v = 0; v < NW; ++v) q[t][v] = 0u;
			}
		}
		if (!waited)
		{
			if (nr > 0) mbar_wait(bar, 0);
			waited = true;
		}

		uint32_t rowkey = static_cast<uint32_t>(row_offset + row_begin);
#pragma unroll 2
		for (int r = 0; r < nr; ++r, ++rowkey)
		{
			uint32_t w[NW];
#pragma unroll
			for (int v = 0; v < NW / 4; ++v)
			{
				uint4 x = s_rows[r * (NW / 4) + v]; // warp-uniform address: broadcast
				w[4 * v + 0] = x.x;
				w[4 * v + 1] = x.y;
				w[4 * v + 2] = x.z;
				w[4 * v + 3] = x.w;
			}
#pragma unroll
			for (int t = 0; t < TQ; ++t)
			{
				const uint32_t d = hamming<NW, VARIANT>(q[t], w);
				top2_insert(k1[t], k2[t], (d << kKeyShift) + rowkey);
			}
		}
#pragma unroll
		for (int t = 0; t < TQ; ++t)
		{
			const int qi = qbase + t * kNnThreads + tid;
			if (qi < nq)
			{
				partial[static_cast<size_t>(blockIdx.x) * nq + qi] = make_uint2(k1[t], k2[t]);
			}
		}
	}
}

// Merge per-chunk top-2 keys: out[2*q], out[2*q+1] (used by lcd_dict_knn2 and the sharded path).
__global__ void knn2_merge_kernel(const uint2 * __restrict__ partial, int n_chunks, int nq, uint32_t * __restrict__ out)
{
	const int qi = blockIdx.x * blockDim.x + threadIdx.x;
	if (qi >= nq) return;
	uint32_t k1 = kKeyNone, k2 = kKeyNone;
	for (int c = 0; c < n_chunks; ++c)
	{
		const uint2 p = partial[static_cast<size_t>(c) * nq + qi];
		top2_insert(k1, k2, p.x);
		top2_insert(k1, k2, p.y);
	}
	out[2 * qi] = k1;
	out[2 * qi + 1] = k2;
}

// Decode packed keys into (word id, distance) pairs for lcd_dict_knn2.
__global__ void knn2_decode_kernel(const uint32_t * __restrict__ keys, int nq, const int * __restrict__ row_ids,
                                   int * __restrict__ id1, float * __restrict__ d1, int * __restrict__ id2, float * __restrict__ d2)
{
	const int qi = blockIdx.x * blockDim.x + threadIdx.x;
	if (qi >= nq) return;
	const uint32_t a = keys[2 * qi], b = keys[2 * qi + 1];
	id1[qi] = a == kKeyNone ? 0 : row_ids[a & kKeyRowMask];
	d1[qi] = a == kKeyNone ? -1.0f : static_cast<float>(a >> kKeyShift);
	id2[qi] = b == kKeyNone ? 0 : row_ids[b & kKeyRowMask];
	d2[qi] = b == kKeyNone ? -1.0f : static_cast<float>(b >> kKeyShift);
}

} // namespace lcd
