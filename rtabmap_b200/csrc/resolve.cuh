// resolve.cuh — per-frame word assignment: merge of per-chunk top-2, NNDR test,
// intra-frame new-word resolution, word-id assignment and TF-IDF preparation.
//
// Replaces: the "Process results" loop of VWDictionary::addNewWords
// (corelib/src/VWDictionary.cpp:1088-1219) and the read-only variant in
// VWDictionary::findNN (VWDictionary.cpp:1476-1546).
//
// The reference loop is sequential: descriptor i is also matched against the words
// created by descriptors 0..i-1 of the same frame (Kp/NewWordsComparedTogether,
// VWDictionary.cpp:1139-1160) and ties in the std::multimap<float,int> keep insertion
// order (index hits first, then new-word hits; lower row / earlier new word first).
// Here one CTA owns one frame and walks it in chunks of 32 descriptors (resolve_rounds below):
// words created by earlier chunks are searched by all warps in parallel, the dependencies inside
// a chunk are settled by one warp with a ballot-mask fixed point (new[i] = f_i(new[0..i-1]) has a
// unique fixed point = the sequential answer), so the result is exact and the cost does not depend
// on how long the chains of mutually-near descriptors are.
#pragma once
#include "common.cuh"
#include "nn_hamming.cuh"
#include <math.h>
#include <limits.h>

namespace lcd {

constexpr int kResolveThreads = 1024;
constexpr int kMaxFrameQueries = 4096;
constexpr uint32_t kSortNone = 0x7FFFFFFFu;

struct ResolveArgs
{
	const uint32_t * queries; // [n_frames*nq][NW]
	int nq;                   // descriptor rows per frame (stride of every per-frame array)
	const int * nq_frame;     // valid descriptors of each frame (<= nq), or nullptr (= nq for all)
	int nq_total;             // n_frames*nq (stride of `partial`)
	const uint2 * partial;    // [n_chunks][nq_total] top-2 keys per vocabulary chunk / per rank
	const ulonglong2 * partial64; // the same for float descriptors: 64-bit keys (l2_path.cuh)
	int n_chunks;
	const int * row_ids; // global row -> word id
	int incremental;     // Kp/IncrementalDictionary
	float nndr;          // Kp/NndrRatio
	int cmp_new;         // Kp/NewWordsComparedTogether
	int last_word_id;    // _lastWordId before this frame
	int find_only;       // findNN semantics: rejected descriptors get id 0, nothing is created
	int * word_ids_out;  // [nq_total] or nullptr
	int * n_new_out;     // [n_frames] or nullptr
	// commit of created words into the not-indexed tail of the vocabulary (single frame) or nullptr
	uint32_t * pending_desc;
	int * pending_ids;
	// TF-IDF preparation (Memory::computeLikelihood, Memory.cpp:2238-2266)
	int do_prep;
	const int * post_len; // posting-list length by word id
	int id_cap;           // entries of post_len
	float n_total;        // N
	int self_ref;         // 1: count the query signature itself in nw (its refs are not in the index)
	int * uq_count;       // [n_frames]
	int * uq_word;        // [n_frames][nq]    unique matched word ids, ascending
	int * uq_prefix;      // [n_frames][nq+1]  exclusive scan of posting lengths to walk
	float * uq_idf;       // [n_frames][nq]    log10(N/nw)
	// similarity likelihood (Memory.cpp:2179-2214): the per-word payload is the query's multiplicity of the word instead of the idf,
	// and every posting is walked (TF-IDF skips the words whose idf is 0)
	int pairs;
	int * uq_mult;        // [n_frames][nq]    multiplicity of each unique word (pairs only)
	int * q_valid;        // [n_frames]        valid(q): the frame's word ids > 0 (pairs only, else nullptr)
};

// Writes the CTA-wide sum of every thread's `mine` to *out (thread 0).  All threads of the CTA must call it.
__device__ inline void cta_count_store(int mine, int * out)
{
	__shared__ int s_count;
	if (threadIdx.x == 0) s_count = 0;
	__syncthreads();
	if (mine) atomicAdd(&s_count, mine);
	__syncthreads();
	if (threadIdx.x == 0) *out = s_count;
}

// Outcome of the multimap<float,int> fullResults of one descriptor.
// a1,a2: index hits (packed keys), n1,n2: hits among this frame's new words (dist<<22|k).
// Returns badDist; best_tag: 0/1 = a1/a2, 2/3 = n1/n2, -1 none.
__device__ __forceinline__ bool nndr_decide(uint32_t a1, uint32_t a2, uint32_t n1, uint32_t n2, float nndr, int & best_tag)
{
	float bd = INFINITY, sd = INFINITY;
	int bt = -1, cnt = 0;
	const uint32_t keys[4] = {a1, a2, n1, n2};
#pragma unroll
	for (int t = 0; t < 4; ++t)
	{
		if (keys[t] != kKeyNone)
		{
			const float d = static_cast<float>(keys[t] >> kKeyShift);
			++cnt;
			if (d < bd)
			{
				sd = bd;
				bd = d;
				bt = t;
			}
			else if (d < sd)
			{
				sd = d;
			}
		}
	}
	best_tag = bt;
	return cnt < 2 || bd > __fmul_rn(nndr, sd); // VWDictionary.cpp:1170-1183
}

// warp 0 only: stable compaction of flagged indices; L[k] = k-th flagged index, rank[i] = k.
__device__ __forceinline__ int warp0_compact(const uint8_t * flag, int n, uint16_t * L, uint16_t * rank)
{
	const int lane = threadIdx.x & 31;
	int base = 0;
	for (int c = 0; c < n; c += 32)
	{
		const int i = c + lane;
		const bool f = i < n && flag[i] != 0;
		const uint32_t m = __ballot_sync(0xFFFFFFFFu, f);
		if (f)
		{
			const int k = base + __popc(m & ((1u << lane) - 1u));
			L[k] = static_cast<uint16_t>(i);
			rank[i] = static_cast<uint16_t>(k);
		}
		base += __popc(m);
	}
	return base;
}

template <int NW>
__device__ __forceinline__ void load_desc(const uint32_t * __restrict__ base, int idx, uint32_t (&q)[NW])
{
	const uint4 * src = reinterpret_cast<const uint4 *>(base + static_cast<size_t>(idx) * NW);
#pragma unroll
	for (int v = 0; v < NW / 4; ++v)
	{
		const uint4 x = src[v]; // plain load: callers pass global or shared memory
		q[4 * v + 0] = x.x;
		q[4 * v + 1] = x.y;
		q[4 * v + 2] = x.z;
		q[4 * v + 3] = x.w;
	}
}

// Shared-memory carve-up for one frame of nq descriptors (nq_pad = next pow2 >= nq).
__host__ __device__ inline size_t resolve_smem_bytes(int nq)
{
	int nq_pad = 32;
	while (nq_pad < nq) nq_pad <<= 1;
	return static_cast<size_t>(nq) * (4 + 4 + 4 + 2 + 2 + 1 + 1) + static_cast<size_t>(nq_pad) * 4 + 64;
}

// TF-IDF preparation from a list of candidate word ids in sbuf[0..n_pad) (kSortNone = skip):
// sort, unique, per-word posting length + idf, exclusive scan.  Used by both entry kernels.
// With a.pairs the payload is the word's multiplicity in the list and the whole posting list is walked.
__device__ void score_prep(uint32_t * sbuf, int n_pad, int nq, const ResolveArgs & a, int frame)
{
	const int tid = threadIdx.x;
	// bitonic sort, ascending
	for (int k = 2; k <= n_pad; k <<= 1)
	{
		for (int j = k >> 1; j > 0; j >>= 1)
		{
			for (int idx = tid; idx < n_pad; idx += blockDim.x)
			{
				const int ixj = idx ^ j;
				if (ixj > idx)
				{
					const uint32_t x = sbuf[idx], y = sbuf[ixj];
					const bool asc = (idx & k) == 0;
					if ((x > y) == asc)
					{
						sbuf[idx] = y;
						sbuf[ixj] = x;
					}
				}
			}
			__syncthreads();
		}
	}
	// unique + compaction + per-word idf / length (warp 0, in order)
	if (tid < 32)
	{
		const int lane = tid;
		int base = 0;
		int run = 0; // running exclusive prefix of posting lengths
		int * uqw = a.uq_word + static_cast<size_t>(frame) * nq;
		int * uqp = a.uq_prefix + static_cast<size_t>(frame) * (nq + 1);
		float * uqi = a.uq_idf + static_cast<size_t>(frame) * nq;
		int * uqm = a.pairs ? a.uq_mult + static_cast<size_t>(frame) * nq : nullptr;
		for (int c = 0; c < n_pad; c += 32)
		{
			const int i = c + lane;
			const uint32_t v = sbuf[i];
			const bool f = v != kSortNone && (i == 0 || sbuf[i - 1] != v);
			const uint32_t m = __ballot_sync(0xFFFFFFFFu, f);
			int len = 0;
			float idf = 0.0f;
			int mult = 0;
			if (f)
			{
				const int id = static_cast<int>(v);
				const int plen = id < a.id_cap ? a.post_len[id] : 0;
				if (a.pairs)
				{
					int j = i + 1;
					while (j < n_pad && sbuf[j] == v) ++j;
					mult = j - i;
					len = plen;
				}
				else
				{
					const float nw = static_cast<float>(plen + a.self_ref);
					// the reference computes nothing when N is 0 (Memory.cpp:2250 `if(N)`): idf 0, the word adds nothing
					if (nw > 0.0f && a.n_total != 0.0f)
					{
						// logNnw = log10(N/nw) on floats (Memory.cpp:2266)
						idf = static_cast<float>(log10(static_cast<double>(__fdiv_rn(a.n_total, nw))));
					}
					len = idf != 0.0f ? plen : 0;
				}
			}
			// inclusive scan of len across the warp
			int incl = len;
#pragma unroll
			for (int o = 1; o < 32; o <<= 1)
			{
				const int t = __shfl_up_sync(0xFFFFFFFFu, incl, o);
				if (lane >= o) incl += t;
			}
			if (f)
			{
				const int k = base + __popc(m & ((1u << lane) - 1u));
				uqw[k] = static_cast<int>(v);
				if (uqm) uqm[k] = mult;
				else uqi[k] = idf;
				uqp[k] = run + incl - len;
			}
			run += __shfl_sync(0xFFFFFFFFu, incl, 31);
			base += __popc(m);
		}
		if (lane == 0)
		{
			uqp[base] = run;
			a.uq_count[frame] = base;
		}
	}
	__syncthreads();
}

// Intra-frame new-word resolution for ONE frame held by the calling CTA (exact, bounded time).
// The reference decides descriptor i after descriptors 0..i-1 (VWDictionary.cpp:1139-1219).  Here the
// frame is walked in chunks of 32 descriptors: (A) one warp per descriptor of the chunk scans the words
// created by all EARLIER chunks (already final) for its two nearest, all warps in parallel; (B) one warp
// resolves the dependencies INSIDE the chunk by fixed-point iteration over a ballot mask (at most 32
// rounds, each descriptor of the chunk in one lane, chunk-mate distances in registers); (C) the chunk's
// new words are appended to the list.  Cost is O(nq * n_new / 32) per warp regardless of how long the
// chains of mutually-near descriptors are.
// On entry sa1/sa2 hold each descriptor's two best index hits.  On return flag[i] = 1 for descriptors
// that create a word (rank[i] = creation order, L[k] = descriptor of the k-th created word), res[i] >= 0 =
// matched index row, res[i] = -1-k = matched the k-th word created by this frame.  Returns the number of
// created words.  All threads of the CTA must call it.
template <int NW>
__device__ int resolve_rounds(const uint32_t * __restrict__ fq, int nq, const uint32_t * sa1, const uint32_t * sa2, int * res,
                              uint16_t * L, uint16_t * rank, uint8_t * flag, uint8_t * flag2, int * s_nL, float nndr, int cmp_new)
{
	__shared__ uint32_t s_ext[64];
	__shared__ uint16_t s_dl[32][34]; // s_dl[e][j] = distance between descriptors c0+e and c0+j of the current chunk
	const int tid = threadIdx.x;
	const int warp = tid >> 5, lane = tid & 31, nwarps = blockDim.x >> 5;
	(void)flag2;
	if (!cmp_new)
	{
		// no comparison among the frame's own new words: the index-only decision in flag[] is final
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
		// (A) nearest two among the words created by earlier chunks
		for (int e = warp; e < 32; e += nwarps)
		{
			const int i = c0 + e;
			if (i >= nq) continue;
			uint32_t k1 = kKeyNone, k2 = kKeyNone;
			uint32_t qi[NW];
			load_desc<NW>(fq, i, qi);
			{
				// distances to the chunk-mates (one per lane), for the dependency pass of warp 0 below: computed here by
				// 32 warps in parallel instead of 1024 shuffled distances by one warp
				uint32_t qm[NW];
				const int jm = c0 + lane;
				if (jm < nq) load_desc<NW>(fq, jm, qm);
				else
				{
#pragma unroll
					for (int v = 0; v < NW; ++v) qm[v] = 0u;
				}
				s_dl[e][lane] = static_cast<uint16_t>(hamming<NW, 2>(qi, qm));
			}
			if (nL > 0)
			{
				for (int k = lane; k < nL; k += 32)
				{
					uint32_t qj[NW];
					load_desc<NW>(fq, L[k], qj);
					const uint32_t d = hamming<NW, 2>(qi, qj);
					top2_insert(k1, k2, (d << kKeyShift) + static_cast<uint32_t>(k));
				}
#pragma unroll
				for (int o = 16; o > 0; o >>= 1)
				{
					const uint32_t o1 = __shfl_down_sync(0xFFFFFFFFu, k1, o);
					const uint32_t o2 = __shfl_down_sync(0xFFFFFFFFu, k2, o);
					top2_insert(k1, k2, o1);
					top2_insert(k1, k2, o2);
				}
			}
			if (lane == 0)
			{
				s_ext[2 * e] = k1;
				s_ext[2 * e + 1] = k2;
			}
		}
		__syncthreads();
		// (B) dependencies inside the chunk, (C) append its new words
		if (warp == 0)
		{
			const int i = c0 + lane;
			const bool valid = i < nq;
			uint32_t dl[32]; // distance to chunk-mate j (only j < lane is used)
#pragma unroll
			for (int jl = 0; jl < 32; ++jl) dl[jl] = s_dl[lane][jl];
			const uint32_t a1 = valid ? sa1[i] : kKeyNone, a2 = valid ? sa2[i] : kKeyNone;
			const uint32_t e1 = s_ext[2 * lane], e2 = s_ext[2 * lane + 1];
			int bt;
			bool bad = valid && nndr_decide(a1, a2, e1, e2, nndr, bt);
			uint32_t n1 = e1;
			uint32_t mask = __ballot_sync(0xFFFFFFFFu, bad);
			for (int r = 0; r < 33; ++r)
			{
				n1 = e1;
				uint32_t n2 = e2;
#pragma unroll
				for (int jl = 0; jl < 32; ++jl)
				{
					if (jl < lane && ((mask >> jl) & 1u))
					{
						const uint32_t kidx = static_cast<uint32_t>(nL) + __popc(mask & ((1u << jl) - 1u));
						top2_insert(n1, n2, (dl[jl] << kKeyShift) + kidx);
					}
				}
				bad = valid && nndr_decide(a1, a2, n1, n2, nndr, bt);
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
				else
				{
					res[i] = bt >= 2 ? -1 - static_cast<int>(n1 & kKeyRowMask) : static_cast<int>(a1 & kKeyRowMask);
				}
			}
			if (lane == 0) *s_nL = nL + __popc(mask);
		}
		__syncthreads();
	}
	return *s_nL;
}

// One CTA per frame.
template <int NW>
__global__ void __launch_bounds__(kResolveThreads)
resolve_kernel(const ResolveArgs a)
{
	extern __shared__ __align__(128) unsigned char smem_raw[];
	const int cap = a.nq; // rows per frame
	int nq_pad = 32;
	while (nq_pad < cap) nq_pad <<= 1;
	uint32_t * sa1 = reinterpret_cast<uint32_t *>(smem_raw);
	uint32_t * sa2 = sa1 + cap;
	int * res = reinterpret_cast<int *>(sa2 + cap);              // >=0 row, -1-k new word k, INT_MIN none
	uint32_t * sbuf = reinterpret_cast<uint32_t *>(res + cap);   // [nq_pad]
	uint16_t * L = reinterpret_cast<uint16_t *>(sbuf + nq_pad);  // [cap]
	uint16_t * rank = L + cap;                                   // [cap]
	uint8_t * flag = reinterpret_cast<uint8_t *>(rank + cap);    // [cap]
	uint8_t * flag2 = flag + cap;                                // [cap]
	__shared__ int s_nL;

	const int tid = threadIdx.x;
	const int frame = blockIdx.x;
	const int nq = a.nq_frame ? min(max(a.nq_frame[frame], 0), cap) : cap; // valid descriptors of this frame
	const uint32_t * fq = a.queries + static_cast<size_t>(frame) * cap * NW;
	const size_t pbase = static_cast<size_t>(frame) * cap;

	// 1. merge the per-chunk top-2 keys (FlannIndex::knnSearch result of this descriptor)
	for (int i = tid; i < nq; i += blockDim.x)
	{
		uint32_t k1 = kKeyNone, k2 = kKeyNone;
		for (int c = 0; c < a.n_chunks; ++c)
		{
			const uint2 p = a.partial[static_cast<size_t>(c) * a.nq_total + pbase + i];
			top2_insert(k1, k2, p.x);
			top2_insert(k1, k2, p.y);
		}
		sa1[i] = k1;
		sa2[i] = k2;
		int bt;
		const bool bad = nndr_decide(k1, k2, kKeyNone, kKeyNone, a.nndr, bt);
		if (a.incremental)
		{
			flag[i] = bad ? 1 : 0;
			res[i] = static_cast<int>(k1 & kKeyRowMask);
		}
		else
		{
			// fixed dictionary: nearest word, no NNDR (VWDictionary.cpp:1211-1218)
			flag[i] = 0;
			res[i] = k1 != kKeyNone ? static_cast<int>(k1 & kKeyRowMask) : INT_MIN;
		}
	}
	__syncthreads();

	int n_new = 0;
	if (a.incremental)
	{
		// 2. intra-frame dependency among the words this frame creates
		n_new = resolve_rounds<NW>(fq, nq, sa1, sa2, res, L, rank, flag, flag2, &s_nL, a.nndr, a.cmp_new);
	}

	// 3. word ids (VWDictionary::getNextId = ++_lastWordId in creation order)
	int n_valid = 0;
	for (int i = tid; i < nq; i += blockDim.x)
	{
		int wid;
		uint32_t sv = kSortNone;
		if (flag[i])
		{
			wid = a.find_only ? 0 : a.last_word_id + 1 + rank[i];
			if (a.pending_desc && !a.find_only)
			{
				uint32_t qi[NW];
				load_desc<NW>(fq, i, qi);
#pragma unroll
				for (int v = 0; v < NW; ++v) a.pending_desc[static_cast<size_t>(rank[i]) * NW + v] = qi[v];
				a.pending_ids[rank[i]] = wid;
			}
		}
		else if (res[i] == INT_MIN)
		{
			wid = 0;
		}
		else if (res[i] < 0)
		{
			wid = a.last_word_id + 1 + (-1 - res[i]);
		}
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
	if (tid == 0 && a.n_new_out) a.n_new_out[frame] = n_new;
	if (a.q_valid) cta_count_store(n_valid, a.q_valid + frame); // new words count too: they are ids > 0 of the query signature
	__syncthreads();

	// 4. unique matched words -> idf + posting extents for the scoring kernel
	if (a.do_prep) score_prep(sbuf, nq_pad, cap, a, frame);
}

// TF-IDF preparation from host-provided word ids (lcd_index_score): applies uUniqueKeys and
// the "*i > 0" filter of Memory::computeLikelihood (Memory.cpp:2238, :2256).
__global__ void __launch_bounds__(kResolveThreads)
prep_from_ids_kernel(const int * __restrict__ word_ids, const ResolveArgs a)
{
	extern __shared__ __align__(128) unsigned char smem_raw[];
	const int nq = a.nq;
	int nq_pad = 32;
	while (nq_pad < nq) nq_pad <<= 1;
	uint32_t * sbuf = reinterpret_cast<uint32_t *>(smem_raw);
	const int frame = blockIdx.x;
	int n_valid = 0;
	for (int i = threadIdx.x; i < nq_pad; i += blockDim.x)
	{
		int w = i < nq ? word_ids[static_cast<size_t>(frame) * nq + i] : 0;
		sbuf[i] = w > 0 ? static_cast<uint32_t>(w) : kSortNone;
		n_valid += w > 0;
	}
	if (a.q_valid) cta_count_store(n_valid, a.q_valid + frame);
	__syncthreads();
	score_prep(sbuf, nq_pad, nq, a, frame);
}

// Sharded scoring (lcd_shard_process_frames_dev): a rank scores EVERY rank's frames over its own word range, so only the ids that have
// postings on this rank matter (no postings = nothing added to any sum).  They are compacted before the sort, which keeps the preparation
// of G ranks' frames at the cost of one rank's frames unsharded instead of growing with G.
__global__ void __launch_bounds__(kResolveThreads)
prep_local_ids_kernel(const int * __restrict__ word_ids, const ResolveArgs a, int frames_per_rank, int part_f0, int part_frames)
{
	// block b prepares frame part_f0 + b % part_frames of rank b / part_frames; word_ids is [rank][frames_per_rank][nq]
	extern __shared__ __align__(128) unsigned char smem_raw[];
	__shared__ int s_n;
	const int nq = a.nq;
	int nq_pad = 32;
	while (nq_pad < nq) nq_pad <<= 1;
	uint32_t * sbuf = reinterpret_cast<uint32_t *>(smem_raw);
	const int frame = blockIdx.x;
	const int src_frame = (frame / part_frames) * frames_per_rank + part_f0 + frame % part_frames;
	const int lane = threadIdx.x & 31;
	if (threadIdx.x == 0) s_n = 0;
	__syncthreads();
	for (int i = threadIdx.x; i < nq_pad; i += blockDim.x) // nq_pad and blockDim are multiples of 32: whole warps iterate together
	{
		const int w = i < nq ? word_ids[static_cast<size_t>(src_frame) * nq + i] : 0;
		const bool keep = w > 0 && w < a.id_cap && a.post_len[w] > 0;
		const uint32_t m = __ballot_sync(0xFFFFFFFFu, keep);
		int base = 0;
		if (lane == 0 && m) base = atomicAdd(&s_n, __popc(m));
		base = __shfl_sync(0xFFFFFFFFu, base, 0);
		if (keep) sbuf[base + __popc(m & ((1u << lane) - 1u))] = static_cast<uint32_t>(w);
	}
	__syncthreads();
	const int n = s_n;
	int n_pad = 32;
	while (n_pad < n) n_pad <<= 1;
	for (int i = n + threadIdx.x; i < n_pad; i += blockDim.x) sbuf[i] = kSortNone;
	__syncthreads();
	score_prep(sbuf, n_pad, nq, a, frame);
}

} // namespace lcd
