// similarity.cuh — the similarity likelihood: Memory::computeLikelihood with Kp/TfIdfLikelihoodUsed=false
// (corelib/src/Memory.cpp:2179-2214), i.e. Signature::compareTo (Signature.cpp:250-288) of the query against every listed signature.
//
// Two sources feed it:
//   - word pairs: score_kernel<true> (score.cuh) accumulates, per (frame, signature), the sum over the shared word ids of
//     min(count in the query, count in the signature) into the integer accumulator; valid(q) comes from the preparation
//     (resolve.cuh) and valid(s) = nvalid[s] from the engine, so the quotient is exact.
//   - global descriptors (SensorData::globalDescriptors(), type 1, one per signature): gdesc_dot_kernel below, the dense
//     B x ns product of the frames' descriptors with the listed signatures' rows.
// similarity_finalize_kernel applies the rules of compareTo per (frame, k).
//
// Word-range-sharded step (lcd_shard_*similarity*): a word's postings live on one rank, so the pair count of (frame, place) and
// valid(s) are exact integer sums of per-rank parts.  Every rank counts the pairs of every rank's frames over its own words
// (gather_pairs_kernel) and its own valid(s) of the listed places (gather_valid_kernel); the summed rows are read by list position
// (similarity_finalize_kernel<true>), valid(q) comes from the frame's own word ids (valid_ids_kernel), and the dot products of a rank's
// local frames need no exchange at all.
//
// Word ids <= 0 never pair here.  EpipolarGeometry::findPairs (EpipolarGeometry.h:119-151) tests id >= 0, so it would pair id 0;
// the quantiser never puts id 0 into a signature (new and matched words are > 0, VWDictionary.cpp:1190-1216; unquantised features
// get distinct negative ids, Memory.cpp:6029-6057), and the inverted index holds positive ids only.
#pragma once
#include "common.cuh"

namespace lcd {

// ---- global-descriptor dot products -----------------------------------------------------------------------------------------
// Register-tiled fp32 SIMT GEMM.  A CTA owns kGdBM frames x kGdBN listed signatures; the signature rows are gathered through
// slot_of_sig and streamed through shared memory in kGdBK-wide slices, so at B <= kGdBM every row is read from HBM once per batch.
// Each thread holds kGdTM x kGdTN outputs.  Order of the arithmetic (this is what makes the value deterministic): every output is
// ONE fused multiply-add chain  acc = 0; for k = 0 .. dim-1: acc = fma(q[k], s[k], acc)  in ascending k, whatever the tile, the
// batch size, the frame's position or ns.  Zero padding past dim adds fma(0, 0, acc) = acc.  The error of such a chain is within
// gamma_dim * sum |q_k s_k| of the exact dot product (recursive summation bound).  Tensor cores would need a multi-term split to
// keep that bound, so they are not used here.
constexpr int kGdBM = 128, kGdBN = 32, kGdBK = 16;
constexpr int kGdTM = 8, kGdTN = 4;
constexpr int kGdThreads = (kGdBM / kGdTM) * (kGdBN / kGdTN); // 128
constexpr int kGdPadM = kGdBM + 4, kGdPadN = kGdBN + 4;        // shared-memory strides (fewer bank conflicts, rows stay 16-byte aligned)

struct GdescArgs
{
	const float * q;           // [n_frames][dim] the frames' descriptors
	int n_frames;
	const float * rows;        // [slot][dim] descriptor store
	int dim;
	const int * slot_of_sig;   // by signature id, -1 = none
	int gd_cap;                // entries of slot_of_sig
	const int * sig_ids;       // [ns]
	int ns;
	float * dot;               // [n_frames][ns] (written where the signature has a descriptor)
	const int * row_of_k;      // [ns] row of each listed place (-1 = none) in place of slot_of_sig, or nullptr
};

// grid = (ceil(ns / kGdBN), ceil(n_frames / kGdBM))
__global__ void __launch_bounds__(kGdThreads)
gdesc_dot_kernel(const GdescArgs a)
{
	__shared__ __align__(16) float sq[2][kGdBK][kGdPadM];
	__shared__ __align__(16) float ss[2][kGdBK][kGdPadN];
	__shared__ int s_slot[kGdBN];
	const int tid = threadIdx.x;
	const int n0 = blockIdx.x * kGdBN, f0 = blockIdx.y * kGdBM;
	if (tid < kGdBN)
	{
		const int k = n0 + tid;
		int slot = -1;
		if (k < a.ns)
		{
			const int s = a.sig_ids[k];
			if (a.row_of_k) slot = a.row_of_k[k];
			else if (s > 0 && s < a.gd_cap) slot = a.slot_of_sig[s];
		}
		s_slot[tid] = slot;
	}
	__syncthreads();

	// loader mapping: 16 consecutive threads read 16 consecutive floats of one row
	const int lk = tid % kGdBK, lr = tid / kGdBK; // lr in [0, 8)
	constexpr int kRowsPerPass = kGdThreads / kGdBK;  // 8
	constexpr int kQLoads = kGdBM / kRowsPerPass;     // 16
	constexpr int kSLoads = kGdBN / kRowsPerPass;     // 4
	float rq[kQLoads], rs[kSLoads];
	auto load = [&](int k0) {
		const int k = k0 + lk;
#pragma unroll
		for (int i = 0; i < kQLoads; ++i)
		{
			const int f = f0 + lr + i * kRowsPerPass;
			rq[i] = (f < a.n_frames && k < a.dim) ? a.q[static_cast<size_t>(f) * a.dim + k] : 0.0f;
		}
#pragma unroll
		for (int i = 0; i < kSLoads; ++i)
		{
			const int slot = s_slot[lr + i * kRowsPerPass];
			rs[i] = (slot >= 0 && k < a.dim) ? a.rows[static_cast<size_t>(slot) * a.dim + k] : 0.0f;
		}
	};
	auto store = [&](int buf) {
#pragma unroll
		for (int i = 0; i < kQLoads; ++i) sq[buf][lk][lr + i * kRowsPerPass] = rq[i];
#pragma unroll
		for (int i = 0; i < kSLoads; ++i) ss[buf][lk][lr + i * kRowsPerPass] = rs[i];
	};

	const int tx = tid % (kGdBN / kGdTN), ty = tid / (kGdBN / kGdTN);
	const bool active = f0 + ty * kGdTM < a.n_frames; // threads whose frames are all past the batch skip the arithmetic
	float acc[kGdTM][kGdTN];
#pragma unroll
	for (int i = 0; i < kGdTM; ++i)
#pragma unroll
		for (int j = 0; j < kGdTN; ++j) acc[i][j] = 0.0f;

	const int n_tiles = (a.dim + kGdBK - 1) / kGdBK;
	load(0);
	store(0);
	__syncthreads();
	for (int t = 0; t < n_tiles; ++t)
	{
		const int buf = t & 1;
		if (t + 1 < n_tiles) load((t + 1) * kGdBK); // global loads of the next slice in flight under the arithmetic
		if (active)
		{
#pragma unroll
			for (int kk = 0; kk < kGdBK; ++kk)
			{
				const float4 qa = *reinterpret_cast<const float4 *>(&sq[buf][kk][ty * kGdTM]);
				const float4 qb = *reinterpret_cast<const float4 *>(&sq[buf][kk][ty * kGdTM + 4]);
				const float4 sv = *reinterpret_cast<const float4 *>(&ss[buf][kk][tx * kGdTN]);
				const float qv[kGdTM] = {qa.x, qa.y, qa.z, qa.w, qb.x, qb.y, qb.z, qb.w};
				const float svv[kGdTN] = {sv.x, sv.y, sv.z, sv.w};
#pragma unroll
				for (int i = 0; i < kGdTM; ++i)
#pragma unroll
					for (int j = 0; j < kGdTN; ++j) acc[i][j] = __fmaf_rn(qv[i], svv[j], acc[i][j]);
			}
		}
		if (t + 1 < n_tiles) store(buf ^ 1); // buf ^ 1 was last read in iteration t - 1, before the barrier that ended it
		__syncthreads();
	}
	if (!active) return;
#pragma unroll
	for (int i = 0; i < kGdTM; ++i)
	{
		const int f = f0 + ty * kGdTM + i;
		if (f >= a.n_frames) break;
#pragma unroll
		for (int j = 0; j < kGdTN; ++j)
		{
			const int n = tx * kGdTN + j;
			if (n0 + n < a.ns && s_slot[n] >= 0) a.dot[static_cast<size_t>(f) * a.ns + n0 + n] = acc[i][j];
		}
	}
}

// ---- Signature::compareTo per (frame, k) ---------------------------------------------------------------------------------------
struct SimilarityArgs
{
	const long long * acc;   // [n_frames][acc_stride] word pairs by signature id (score_kernel<true>)
	int acc_stride;
	const int * pairs;       // LISTED: [n_frames][ns] word pairs by list position (the sharded step's cross-rank sums)
	const int * nvalid;      // valid(s) = sum of the signature's posting counts: by signature id, or by list position (LISTED)
	int sig_cap;             // entries of nvalid by signature id
	const int * q_valid;     // [n_frames] valid(q)
	const float * dot;       // [n_frames][ns] or nullptr when the frames carry no global descriptor
	const int * slot_of_sig; // global-descriptor slot (-1 = none): by signature id, or by list position (LISTED)
	int gd_cap;              // entries of slot_of_sig by signature id
	const int * sig_ids;     // [ns]
	int ns;
	float * out;             // [n_frames][ns]
};

// grid = (ceil(ns / 256), n_frames).  LISTED = false: one engine's arrays, indexed by signature id; true: the sharded step's rows,
// indexed by list position.
template <bool LISTED>
__global__ void similarity_finalize_kernel(const SimilarityArgs a)
{
	const int k = blockIdx.x * blockDim.x + threadIdx.x;
	const int frame = blockIdx.y;
	if (k >= a.ns) return;
	const int s = a.sig_ids[k];
	const size_t o = static_cast<size_t>(frame) * a.ns + k;
	const int key = LISTED ? k : s; // index of the per-place arrays
	float v = 0.0f; // the virtual place (s <= 0) and bad signatures
	if (s > 0)
	{
		if (a.dot && (LISTED || s < a.gd_cap) && a.slot_of_sig[key] >= 0)
		{
			// (dot + 1.0f) / 2.0f on the double cv::Mat::dot returns, then the float of compareTo (Signature.cpp:263)
			v = static_cast<float>((static_cast<double>(a.dot[o]) + 1.0) / 2.0);
		}
		else
		{
			const int nq = a.q_valid[frame];
			const int nsig = LISTED || s < a.sig_cap ? a.nvalid[key] : 0;
			if (nq > 0 && nsig > 0) // isBadSignature on either side (Signature.cpp:341-344) gives 0
			{
				const long long pairs = LISTED ? a.pairs[o] : a.acc[static_cast<size_t>(frame) * a.acc_stride + s];
				v = __fdiv_rn(static_cast<float>(pairs), static_cast<float>(max(nq, nsig))); // float(pairs) / float(totalWords)
			}
		}
	}
	a.out[o] = v;
}

// ---- the word-range-sharded step ---------------------------------------------------------------------------------------------
// A pair count is at most valid(q) <= kMaxFrameQueries, and valid(s) a signature's reference count, so both are exchanged as int32.
// Pair counts of `frame` by list position, from the accumulator rows score_kernel<true> filled: row frame + frame / rows_per_seg of
// out[..][ns], i.e. one row is left free after every rows_per_seg frames (the reduce-scatter segment of a rank carries its valid(s)
// there; rows_per_seg = n_frames leaves none).  grid = (ceil(ns / 256), n_frames)
__global__ void gather_pairs_kernel(const long long * __restrict__ acc, int acc_stride, int sig_cap, const int * __restrict__ sig_ids, int ns,
                                    int rows_per_seg, int * __restrict__ out)
{
	const int k = blockIdx.x * blockDim.x + threadIdx.x;
	const int frame = blockIdx.y;
	if (k >= ns) return;
	const int s = sig_ids[k];
	int v = 0;
	if (s > 0 && s < sig_cap) v = static_cast<int>(acc[static_cast<size_t>(frame) * acc_stride + s]);
	out[(static_cast<size_t>(frame) + frame / rows_per_seg) * ns + k] = v;
}

// this rank's valid(s) of the listed places, written to out + c * stride for c < gridDim.y.  grid = (ceil(ns / 256), copies)
__global__ void gather_valid_kernel(const int * __restrict__ nvalid, int sig_cap, const int * __restrict__ sig_ids, int ns, int * __restrict__ out,
                                    size_t stride)
{
	const int k = blockIdx.x * blockDim.x + threadIdx.x;
	if (k >= ns) return;
	const int s = sig_ids[k];
	out[blockIdx.y * stride + k] = s > 0 && s < sig_cap ? nvalid[s] : 0;
}

// valid(q) of each frame from its word ids [n_frames][nq]: the ids > 0, new words included (the rule of the unsharded preparation).
// grid = n_frames, block = kValidThreads
constexpr int kValidThreads = 128;
__global__ void __launch_bounds__(kValidThreads)
valid_ids_kernel(const int * __restrict__ word_ids, int nq, int * __restrict__ out)
{
	__shared__ int s_warp[kValidThreads / 32];
	const int * w = word_ids + static_cast<size_t>(blockIdx.x) * nq;
	int n = 0;
	for (int i = threadIdx.x; i < nq; i += kValidThreads) n += w[i] > 0;
	n = __reduce_add_sync(0xFFFFFFFFu, n);
	if ((threadIdx.x & 31) == 0) s_warp[threadIdx.x >> 5] = n;
	__syncthreads();
	if (threadIdx.x == 0)
	{
		int t = 0;
		for (int i = 0; i < kValidThreads / 32; ++i) t += s_warp[i];
		out[blockIdx.x] = t;
	}
}

} // namespace lcd
