// score.cuh — TF-IDF likelihood of every signature through the inverted index.
//
// Replaces: the TF-IDF branch of Memory::computeLikelihood
// (corelib/src/Memory.cpp:2215-2291) walking VisualWord::_references
// (corelib/include/rtabmap/core/VisualWord.h:62) with Memory::getNi (Memory.cpp:4955-4968).
//
// The inverted index is a word -> posting-list table in HBM: post_off[word] / post_len[word]
// locate a contiguous run of (signature id, count) pairs in one arena.  A frame touches the
// posting lists of its unique matched words (prepared by resolve.cuh): the kernel flattens
// those lists into one index space (segmented by the exclusive scan uq_prefix) so that every
// thread handles one posting regardless of how skewed the list lengths are, computes the
// reference's float term (nwi*logNnw)/ni, and accumulates it into a per-signature 2^-40
// fixed-point int64 accumulator.  Integer accumulation is associative, so the result is
// deterministic and independent of traversal order (and of how words are sharded across
// GPUs), and tests/tfidf_model.py reproduces it bit for bit.  It differs from the reference's
// sequential float sum by the idf (log10f against the correctly rounded double log10: up to
// 2 ulps with glibc), the float rounding of the reference's running sum and 2^-41 per term;
// tests/tfidf_model.py derives that bound per signature (below the smallest single term in
// nearly every signature at bench scale).  The int prefix of a frame's postings limits one
// frame's query words to 2^31 postings in total; the arena itself holds up to 2^32.
#pragma once
#include "common.cuh"

namespace lcd {

constexpr int kScoreThreads = 256;
constexpr double kScoreScale = 1099511627776.0; // 2^40
constexpr double kScoreInvScale = 1.0 / 1099511627776.0;

struct ScoreArgs
{
	int nq;                 // stride of the uq_* arrays
	const int * uq_count;   // [n_frames]
	const int * uq_word;    // [n_frames][nq]
	const int * uq_prefix;  // [n_frames][nq+1]
	const float * uq_idf;   // [n_frames][nq]
	const int * uq_mult;    // [n_frames][nq] query multiplicity of each word (PAIRS)
	const uint32_t * post_off; // by word id
	const int2 * postings;     // (signature id, count)
	const int * ni;            // by signature id
	int sig_cap;               // entries of ni / of one accumulator row
	long long * acc;           // [n_frames][acc_stride]
	int acc_stride;
};

// grid = (blocks_per_frame, n_frames)
// PAIRS = false: the TF-IDF term of every posting.  PAIRS = true: the word pairs of Signature::compareTo (Signature.cpp:278-284),
// acc[frame][sig] += min(count in the query, count in the signature) = EpipolarGeometry::findPairs summed over the shared ids
// (EpipolarGeometry.h:119-151); integer, hence exact and independent of the order.
template <bool PAIRS>
__global__ void __launch_bounds__(kScoreThreads)
score_kernel(const ScoreArgs a)
{
	extern __shared__ int s_prefix[]; // [nuq+1]
	const int frame = blockIdx.y;
	const int nuq = a.uq_count[frame];
	if (nuq == 0) return;
	const int * uqp = a.uq_prefix + static_cast<size_t>(frame) * (a.nq + 1);
	const int total = uqp[nuq];
	// every block takes one contiguous slice of the frame's postings, its threads consecutive postings: a thread's next posting is 256
	// further on, i.e. in the same or one of the next few words, so ONE binary search per thread and then a short forward walk replaces
	// a 10-step search per posting (59 % of the kernel's instructions before).  Integer atomics: the result does not depend on the order.
	const int chunk = (total + static_cast<int>(gridDim.x) - 1) / static_cast<int>(gridDim.x);
	const int begin = blockIdx.x * chunk, end = min(total, begin + chunk);
	if (begin >= end) return;
	for (int i = threadIdx.x; i <= nuq; i += kScoreThreads) s_prefix[i] = uqp[i];
	__syncthreads();
	const int * uqw = a.uq_word + static_cast<size_t>(frame) * a.nq;
	const float * uqi = a.uq_idf + static_cast<size_t>(frame) * a.nq;
	const int * uqm = a.uq_mult + static_cast<size_t>(frame) * a.nq;
	long long * acc = a.acc + static_cast<size_t>(frame) * a.acc_stride;

	int p = begin + threadIdx.x;
	if (p >= end) return;
	int lo = 0;
	{
		// largest k with prefix[k] <= p
		int hi = nuq;
		while (hi - lo > 1)
		{
			const int mid = (lo + hi) >> 1;
			if (s_prefix[mid] <= p) lo = mid;
			else hi = mid;
		}
	}
	for (; p < end; p += kScoreThreads)
	{
		while (s_prefix[lo + 1] <= p) ++lo; // p < total = prefix[nuq]: stops at lo < nuq
		const int word = uqw[lo];
		const int2 ref = a.postings[static_cast<size_t>(a.post_off[word]) + (p - s_prefix[lo])];
		if constexpr (PAIRS)
		{
			if (ref.x > 0 && ref.x < a.sig_cap)
				atomicAdd(reinterpret_cast<unsigned long long *>(acc + ref.x), static_cast<unsigned long long>(min(uqm[lo], ref.y)));
		}
		else if (ref.x > 0 && ref.x < a.sig_cap)
		{
			const float idf = uqi[lo];
			const float ni = static_cast<float>(a.ni[ref.x]);
			if (ni != 0.0f)
			{
				// iter->second += (nwi * logNnw) / ni   (Memory.cpp:2279)
				const float term = __fdiv_rn(__fmul_rn(static_cast<float>(ref.y), idf), ni);
				const long long fx = __double2ll_rn(static_cast<double>(term) * kScoreScale);
				atomicAdd(reinterpret_cast<unsigned long long *>(acc + ref.x), static_cast<unsigned long long>(fx));
			}
		}
	}
}

// likelihood[f][k] = acc[f][sig_ids[k]] (0 for ids <= 0 or unknown: likelihood starts at 0 for
// every requested id, Memory.cpp:2232-2235)
__global__ void gather_likelihood_kernel(const long long * __restrict__ acc, int acc_stride, int sig_cap,
                                         const int * __restrict__ sig_ids, int ns, float * __restrict__ out)
{
	const int k = blockIdx.x * blockDim.x + threadIdx.x;
	const int frame = blockIdx.y;
	if (k >= ns) return;
	const int s = sig_ids[k];
	float v = 0.0f;
	if (s > 0 && s < sig_cap)
	{
		v = static_cast<float>(static_cast<double>(acc[static_cast<size_t>(frame) * acc_stride + s]) * kScoreInvScale);
	}
	out[static_cast<size_t>(frame) * ns + k] = v;
}

// plain fixed-point -> float conversion of an (all-reduced) score vector
__global__ void fixed_to_float_kernel(const long long * __restrict__ in, int n, float * __restrict__ out)
{
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i < n) out[i] = static_cast<float>(static_cast<double>(in[i]) * kScoreInvScale);
}

// gather of raw fixed-point scores for the requested ids (sharded path: all-reduce these)
__global__ void gather_fixed_kernel(const long long * __restrict__ acc, int acc_stride, int sig_cap,
                                    const int * __restrict__ sig_ids, int ns, long long * __restrict__ out)
{
	const int k = blockIdx.x * blockDim.x + threadIdx.x;
	const int frame = blockIdx.y;
	if (k >= ns) return;
	const int s = sig_ids[k];
	long long v = 0;
	if (s > 0 && s < sig_cap) v = acc[static_cast<size_t>(frame) * acc_stride + s];
	out[static_cast<size_t>(frame) * ns + k] = v;
}

// ---- inverted-index maintenance ---------------------------------------------------------
struct RefOp
{
	int word;   // word id
	int sig;    // signature id
	int cnt;    // references to add
	int pos;    // >= 0: write a new posting at this position; -1: find `sig` and add cnt
	int newlen; // posting-list length after the op
};

// VisualWord::addRef (VisualWord.cpp:51-63), one thread per (word, signature)
__global__ void index_apply_kernel(const RefOp * __restrict__ ops, int n, const uint32_t * __restrict__ post_off,
                                   int * __restrict__ post_len, int2 * __restrict__ postings)
{
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	const RefOp op = ops[i];
	int2 * list = postings + post_off[op.word];
	if (op.pos >= 0)
	{
		list[op.pos] = make_int2(op.sig, op.cnt);
	}
	else
	{
		const int len = post_len[op.word];
		for (int k = 0; k < len; ++k)
		{
			if (list[k].x == op.sig)
			{
				list[k].y += op.cnt;
				break;
			}
		}
	}
	post_len[op.word] = op.newlen;
}

// VisualWord::removeAllRef (VisualWord.cpp:65-70): one warp per (word, signature); the posting
// is replaced by the list's last entry (posting order carries no meaning here).
__global__ void index_remove_kernel(const RefOp * __restrict__ ops, int n, const uint32_t * __restrict__ post_off,
                                    int * __restrict__ post_len, int2 * __restrict__ postings)
{
	const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
	const int lane = threadIdx.x & 31;
	if (w >= n) return;
	const RefOp op = ops[w];
	int2 * list = postings + post_off[op.word];
	const int len = post_len[op.word];
	int found = -1;
	for (int k = lane; k < len && found < 0; k += 32)
	{
		if (list[k].x == op.sig) found = k;
	}
	const uint32_t m = __ballot_sync(0xFFFFFFFFu, found >= 0);
	if (m)
	{
		const int src = __ffs(m) - 1;
		const int k = __shfl_sync(0xFFFFFFFFu, found, src);
		if (lane == 0)
		{
			list[k] = list[len - 1];
			post_len[op.word] = len - 1;
		}
	}
}

// relocation of a posting list to a larger extent
struct MoveOp
{
	int word;
	uint32_t old_off;
	uint32_t new_off;
	int len;
};
__global__ void index_move_kernel(const MoveOp * __restrict__ ops, int n, uint32_t * __restrict__ post_off, int2 * __restrict__ postings)
{
	const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
	const int lane = threadIdx.x & 31;
	if (w >= n) return;
	const MoveOp op = ops[w];
	for (int k = lane; k < op.len; k += 32) postings[op.new_off + k] = postings[op.old_off + k];
	if (lane == 0) post_off[op.word] = op.new_off;
}

// gather rows of a descriptor matrix: dst[r] = src[src_row[r]]  (vocabulary compaction / reorder)
__global__ void gather_rows_kernel(const uint32_t * __restrict__ src, const int * __restrict__ src_row, int n_rows, int nw,
                                   uint32_t * __restrict__ dst)
{
	const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
	if (i >= static_cast<size_t>(n_rows) * nw) return;
	const int r = static_cast<int>(i / nw), c = static_cast<int>(i % nw);
	dst[i] = src[static_cast<size_t>(src_row[r]) * nw + c];
}

// ---- Rtabmap::adjustLikelihood (Rtabmap.cpp:5691-5760), one CTA per frame ------------------------------------
// in: like[frame][ns] raw likelihood of the ids the caller listed (ascending id order, as the std::map iterates);
// out: adj[frame][ns + 1], element 0 = the virtual place.  uMean / uVariance (UMath.h:419-431, :512-526) are float sums in
// list order over the values > 0: the positive values are compacted chunk by chunk (order preserved) and thread 0 adds each
// chunk sequentially, so mean, standard deviation and every adjusted value are bit-identical to the reference arithmetic.
constexpr int kAdjustThreads = 256;
constexpr int kAdjustChunk = 2048;

__device__ inline int adjust_compact_chunk(const float * __restrict__ row, int c0, int n, float * s_val, int * s_cnt,
                                           const unsigned char * __restrict__ listed = nullptr)
{
	// stable compaction of row[c0 .. c0+n) > 0 (and listed, when a list is given) into s_val; returns the count (valid in all threads)
	const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
	__shared__ int s_warp[kAdjustThreads / 32];
	int base = 0;
	for (int i0 = 0; i0 < n; i0 += kAdjustThreads)
	{
		const int i = i0 + tid;
		const float v = i < n ? row[c0 + i] : 0.f;
		const bool keep = i < n && v > 0.f && (!listed || listed[c0 + i]);
		const unsigned m = __ballot_sync(0xFFFFFFFFu, keep);
		if (lane == 0) s_warp[warp] = __popc(m);
		__syncthreads();
		int off = base;
		for (int w = 0; w < warp; ++w) off += s_warp[w];
		int tot = 0;
		for (int w = 0; w < kAdjustThreads / 32; ++w) tot += s_warp[w];
		if (keep) s_val[off + __popc(m & ((1u << lane) - 1u))] = v;
		base += tot;
		__syncthreads();
	}
	if (tid == 0) *s_cnt = base;
	__syncthreads();
	return *s_cnt;
}

// listed[ns] (nullptr: every place): the places the frame compares; the others are left out of the mean, the deviation and the
// maximum, as if absent from the likelihood map, and their adjusted value is 0 (they add exact zeros to the posterior after it)
__device__ __forceinline__ void adjust_likelihood_row(const float * __restrict__ row, int ns, int virtual_place_ratio, float * __restrict__ out,
                                                      const unsigned char * __restrict__ listed)
{
	__shared__ float s_val[kAdjustChunk];
	__shared__ int s_cnt;
	__shared__ float s_acc, s_mean, s_std, s_max[kAdjustThreads / 32];
	__shared__ long long s_n;
	const int tid = threadIdx.x;
	if (tid == 0)
	{
		s_acc = 0.f;
		s_n = 0;
	}
	__syncthreads();
	// pass 1: mean of the values > 0
	for (int c0 = 0; c0 < ns; c0 += kAdjustChunk)
	{
		const int cnt = adjust_compact_chunk(row, c0, min(kAdjustChunk, ns - c0), s_val, &s_cnt, listed);
		if (tid == 0)
		{
			float m = s_acc;
			for (int i = 0; i < cnt; ++i) m = __fadd_rn(m, s_val[i]);
			s_acc = m;
			s_n += cnt;
		}
		__syncthreads();
	}
	if (tid == 0)
	{
		s_mean = s_n ? __fdiv_rn(s_acc, static_cast<float>(static_cast<unsigned long long>(s_n))) : 0.f;
		s_acc = 0.f;
	}
	__syncthreads();
	const float mean = s_mean;
	const long long n_pos = s_n;
	// pass 2: variance (n - 1 in the denominator)
	if (n_pos > 1)
	{
		for (int c0 = 0; c0 < ns; c0 += kAdjustChunk)
		{
			const int cnt = adjust_compact_chunk(row, c0, min(kAdjustChunk, ns - c0), s_val, &s_cnt, listed);
			if (tid == 0)
			{
				float sum = s_acc;
				for (int i = 0; i < cnt; ++i)
				{
					const float d = __fsub_rn(s_val[i], mean);
					sum = __fadd_rn(sum, __fmul_rn(d, d));
				}
				s_acc = sum;
			}
			__syncthreads();
		}
	}
	if (tid == 0)
	{
		const float var = n_pos > 1 ? __fdiv_rn(s_acc, static_cast<float>(static_cast<unsigned long long>(n_pos - 1))) : 0.f;
		s_std = sqrtf(var);
	}
	__syncthreads();
	const float sd = s_std;
	const float epsilon = 0.0001f;
	const float thr = __fadd_rn(mean, sd);
	float mx = 0.f;
	for (int i = tid; i < ns; i += kAdjustThreads)
	{
		if (listed && !listed[i])
		{
			out[1 + i] = 0.f;
			continue;
		}
		const float value = row[i];
		float r = 1.0f;
		if (value > thr)
		{
			if (virtual_place_ratio == 0 && mean != 0.f) r = __fdiv_rn(__fsub_rn(value, __fsub_rn(sd, epsilon)), mean);
			else if (virtual_place_ratio != 0 && sd != 0.f) r = __fdiv_rn(__fsub_rn(value, mean), sd);
		}
		out[1 + i] = r;
		mx = fmaxf(mx, value);
	}
	for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_down_sync(0xFFFFFFFFu, mx, o));
	if ((tid & 31) == 0) s_max[tid >> 5] = mx;
	__syncthreads();
	if (tid == 0)
	{
		float m = 0.f;
		for (int w = 0; w < kAdjustThreads / 32; ++w) m = fmaxf(m, s_max[w]);
		float vp = 2.0f;
		if (virtual_place_ratio == 0 && sd > epsilon && m != 0.f) vp = __fadd_rn(__fdiv_rn(mean, sd), 1.0f);
		else if (virtual_place_ratio != 0 && m > mean) vp = __fadd_rn(__fdiv_rn(sd, __fsub_rn(m, mean)), 1.0f);
		out[0] = vp;
	}
}

__global__ void __launch_bounds__(kAdjustThreads)
adjust_likelihood_kernel(const float * __restrict__ like, int ns, int virtual_place_ratio, float * __restrict__ adj)
{
	adjust_likelihood_row(like + static_cast<size_t>(blockIdx.x) * ns, ns, virtual_place_ratio, adj + static_cast<size_t>(blockIdx.x) * (ns + 1),
	                      nullptr);
}

// the same over the places of listed[frame][ns + 1] (element 0 the virtual place); a row that lists every place gives the bits above
__global__ void __launch_bounds__(kAdjustThreads)
adjust_likelihood_listed_kernel(const float * __restrict__ like, int ns, int virtual_place_ratio, float * __restrict__ adj,
                                const unsigned char * __restrict__ listed)
{
	const size_t f = blockIdx.x;
	adjust_likelihood_row(like + f * ns, ns, virtual_place_ratio, adj + f * (ns + 1), listed + f * (ns + 1) + 1);
}

} // namespace lcd
