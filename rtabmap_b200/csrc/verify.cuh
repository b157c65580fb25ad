// verify.cuh — geometric verification of loop-closure hypotheses: descriptor matching of a
// signature pair and PnP/RANSAC with refinement, batched one CTA per pair.
//
// Replaces, for Vis/CorNNType in {0,3} (exact matching), Vis/EstimationType=1 (PnP), single camera:
//   pair_match_kernel  RegistrationVis::computeTransformationImpl global matching through a temporary
//                      VWDictionary (corelib/src/RegistrationVis.cpp:1482-1546) and the correspondence
//                      assembly of util3d::estimateMotion3DTo2D (util3d_motion_estimation.cpp:88-110)
//   pnp_ransac_kernel  util3d::solvePnPRansac (util3d_motion_estimation.cpp:843-990) =
//                      cv3::solvePnPRansac / RANSACPointSetRegistrator::run (opencv/solvepnp.cpp:112-417)
//                      + the PCL-style refinement loop, and the pose -> Transform conversion (:121-154)
//
// RANSAC is sequential in the reference (adaptive iteration count, strict-best update) but its random
// samples depend only on the point count (cv::RNG seeded with (uint64)-1 on every run), so all
// Vis/Iterations hypotheses are evaluated in parallel (one thread each: EPnP on 6 points + inlier count
// over all points) and one thread then replays the sequential best/niters bookkeeping over the counts.
#pragma once
#include "common.cuh"
#include "l2_path.cuh"
#include "pnp_device.cuh"
#include "ransac.cuh"
#include "resolve.cuh"

namespace lcd {

constexpr int kPnpChunk = 128;      // sizes two areas of the PnP kernel's shared memory (pnp_smem_bytes)
constexpr int kPnpWave = 16;        // RANSAC hypotheses of the first wave (one thread each for EPnP)
constexpr int kPnpWaveMax = 256;    // hypotheses of every later wave
constexpr int kVerifyThreads = 256; // threads of the CTA: RANSAC waves after the first, inlier counts, LM sums and error passes
constexpr int kMaxRansacIters = 320;

// What a signature-store row's cached FROM dictionary was built for.  The temporary dictionary of addNewWords(descriptorsFrom) is a
// function of the row's first nf descriptors and Vis/CorNNDR alone, so the matching kernel reuses it while both are those of the call.
struct FromDictTag
{
	int nf;             // -1: stale (the row was written or freed since)
	int n_dict;
	uint32_t nndr_bits; // Vis/CorNNDR as float bits
	int unused;
};

// Where the two signatures of each pair are read, for both matching passes.
struct PairSource
{
	struct
	{
		const uint32_t * desc; // [n_from_rows][cap][NW]
		const float * xyz;     // [n_from_rows][cap][3]   NaN = no depth
		const int * n;         // [n_from_rows]
		const int * slot;      // nullptr: FROM row = pair; else row of the signature store for each pair (-1 = none)
		int cap;               // row stride of the FROM arrays
	} from;
	struct
	{
		const uint32_t * desc; // [n_to_rows][cap][NW]
		const float * uv;      // [n_to_rows][cap][2]
		const float * xyz;     // [n_to_rows][cap][3] or nullptr: Signature::getWords3 of the TO side (words3B of estimateMotion3DTo2D)
		const int * n;         // [n_pairs] or nullptr (= n_all)
		int n_all;
		int cap;               // row stride of the TO arrays
		const int * row;       // nullptr: TO row = pair; else the TO row of each pair
		const FrameCam * cam;  // [n_to_rows] the TO camera of each TO row (set = 0: the call's lcd_verify_params) or nullptr
	} to;

	__device__ __forceinline__ int from_row(int pair) const { return from.slot ? from.slot[pair] : pair; }
	// the pair's own TO camera, nullptr when it takes the call's parameters
	__device__ __forceinline__ const FrameCam * to_cam(int pair) const
	{
		if (!to.cam) return nullptr;
		const FrameCam * c = to.cam + (to.row ? to.row[pair] : pair);
		return c->set ? c : nullptr;
	}
	// TO descriptors of the pair, at most cap (the call's) and the TO row stride
	__device__ __forceinline__ int to_count(int pair, int cap) const { return min(to.n ? to.n[pair] : to.n_all, min(cap, to.cap)); }
	__device__ __forceinline__ size_t to_base(int pair) const { return static_cast<size_t>(to.row ? to.row[pair] : pair) * to.cap; }
};

// words3B: the 3-D point of TO descriptor ti (TO row at tbase) to output row m of obj_to; nothing when obj_to is nullptr (no TO points)
__device__ __forceinline__ void gather_obj_to(const PairSource & src, float * obj_to, size_t m, size_t tbase, int ti)
{
	if (!obj_to) return;
	const float * r = src.to.xyz + (tbase + ti) * 3;
	obj_to[m * 3 + 0] = r[0];
	obj_to[m * 3 + 1] = r[1];
	obj_to[m * 3 + 2] = r[2];
}

struct MatchArgs
{
	PairSource src;
	int cap;                    // stride of the outputs and size of the shared-memory arrays (>= both row strides)
	float nndr; // Vis/CorNNDR
	// FROM dictionaries cached per signature-store row (src.from.slot only, else nullptr): see from_dict_build_kernel
	const FromDictTag * from_tag;  // [n_from_rows]
	const uint16_t * from_kof;     // [n_from_rows][src.from.cap]
	const uint16_t * from_creator; // [n_from_rows][src.from.cap]
	// outputs
	float * obj;       // [n_pairs][cap][3]
	float * img;       // [n_pairs][cap][2]
	float * obj_to;    // [n_pairs][cap][3] 3-D point of the TO side for each correspondence (NaN = none); nullptr when src.to.xyz is
	int * match_id;    // [n_pairs][cap]  word id of the correspondence (ascending)
	int * match_from;  // [n_pairs][cap]  descriptor index in FROM
	int * match_to;    // [n_pairs][cap]  descriptor index in TO
	int * n_match;     // [n_pairs]
	int * from_ids;    // [n_pairs][cap] or nullptr
	int * to_ids;      // [n_pairs][cap] or nullptr
};

// ---- TO x dictionary 2-NN of the matching kernel on the tensor cores ------------------------------------------------------------
// A descriptor bit b is the s8 value 1 - 2b, so the s32 dot product of two descriptors is 32*NW - 2*hamming: exact integers, as in
// nn_tensor.cuh.  mma.m16n8k32 gives each thread (group g = lane / 4, tig = lane % 4) the k positions 4*tig..4*tig+3 (a0, a1, b0) and
// 16+4*tig..19+4*tig (a2, a3, b1) of a k-step.  The order of k inside a dot product is free as long as A and B agree, so those eight
// positions are the eight bits of byte 4*ks + tig of the packed descriptor: low nibble -> a0/a1/b0, high nibble -> a2/a3/b1.  The
// queries (A) are expanded in registers per k-step; the dictionary (B) is expanded to s8 in shared memory, kScanWords words at a time.
constexpr int kScanNJ = 4;                 // n8 tiles (dictionary words / 8) per accumulator set of a warp: 16 registers (1024 threads: 64 each)
constexpr int kScanWords = 64;             // dictionary words expanded per pass
// 32-bit words per expanded dictionary word: 32*NW s8 + 32 bytes of padding, so the lds.64 of the 8 groups x 4 threads of a warp
// fall on 32 different banks in each half-warp
__host__ __device__ constexpr int scan_stride_words(int nw) { return 8 * nw + 8; }
__host__ __device__ constexpr size_t scan_tile_bytes(int nw) { return static_cast<size_t>(kScanWords) * scan_stride_words(nw) * 4; }

__host__ __device__ inline size_t match_smem_bytes(int cap, int nw)
{
	return scan_tile_bytes(nw) + static_cast<size_t>(cap) * (4 + 4 + 4 + 2 + 2 + 1 + 1 + 4 + 4 + 2 + 2) + 2 * static_cast<size_t>(cap) * nw * 4 + 128;
}

// the four bits of a nibble as four s8 values 1 - 2b (byte j = bit j)
__device__ __forceinline__ uint32_t pm1_nibble(uint32_t n)
{
	return ((n * 0x00204081u) & 0x01010101u) * 0xFEu + 0x01010101u;
}

__device__ __forceinline__ void mma_s8_m16n8k32(int (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1)
{
	asm("mma.sync.aligned.m16n8k32.row.col.s32.s8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
	    : "+r"(c[0]), "+r"(c[1]), "+r"(c[2]), "+r"(c[3])
	    : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

// For every query j < nt: merges the two nearest dictionary words, as keys (d << kKeyShift) + k, into sa1[j] / sa2[j].  The keys are
// the ones a scan of k = 0..n_dict-1 with top2_insert produces: distinct per k, so the smaller k wins a tie whatever the order.
// Warp w owns the 16-query tiles w, w + 32, ...; per pass it multiplies them by kScanWords expanded words.  All threads must call it.
// Not inlined: with the matching kernel's live values around it, the 64 registers of a 1024-thread CTA spill.
template <int NW>
__device__ __noinline__ void to_dict_knn2_mma(const uint32_t * __restrict__ q, int nt, const uint32_t * __restrict__ dict, int n_dict, uint32_t * __restrict__ stile,
                                 uint32_t * sa1, uint32_t * sa2)
{
	constexpr int S = scan_stride_words(NW);
	const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = blockDim.x >> 5;
	const int g = lane >> 2, tig = lane & 3;
	const int n_mt = (nt + 15) >> 4;
	for (int w0 = 0; w0 < n_dict; w0 += kScanWords)
	{
		__syncthreads(); // the previous pass is consumed
		for (int i = tid; i < kScanWords * NW; i += blockDim.x)
		{
			const int w = i / NW, v = i % NW;
			const uint32_t x = w0 + w < n_dict ? dict[static_cast<size_t>(w0 + w) * NW + v] : 0u;
			uint4 * dst = reinterpret_cast<uint4 *>(stile + w * S + v * 8); // packed byte 4v + b -> s8 bytes 8(4v + b) .. +7
			dst[0] = make_uint4(pm1_nibble(x & 0xFu), pm1_nibble((x >> 4) & 0xFu), pm1_nibble((x >> 8) & 0xFu), pm1_nibble((x >> 12) & 0xFu));
			dst[1] = make_uint4(pm1_nibble((x >> 16) & 0xFu), pm1_nibble((x >> 20) & 0xFu), pm1_nibble((x >> 24) & 0xFu), pm1_nibble(x >> 28));
		}
		__syncthreads();
		const int n_valid = min(kScanWords, n_dict - w0);
		for (int mt = warp; mt < n_mt; mt += nwarps)
		{
			const int r0 = mt * 16 + g, r1 = r0 + 8;
			const uint32_t * q0 = q + static_cast<size_t>(min(r0, nt - 1)) * NW; // rows past nt compute on a real row; dropped below
			const uint32_t * q1 = q + static_cast<size_t>(min(r1, nt - 1)) * NW;
			uint32_t k1a = kKeyNone, k2a = kKeyNone, k1b = kKeyNone, k2b = kKeyNone;
#pragma unroll 1
			for (int n0 = 0; n0 < n_valid; n0 += 8 * kScanNJ)
			{
				int acc[kScanNJ][4];
#pragma unroll
				for (int j = 0; j < kScanNJ; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0;
#pragma unroll 4
				for (int ks = 0; ks < NW; ++ks)
				{
					const uint32_t x0 = q0[ks] >> (8 * tig), x1 = q1[ks] >> (8 * tig);
					const uint32_t a0 = pm1_nibble(x0 & 0xFu), a1 = pm1_nibble(x1 & 0xFu), a2 = pm1_nibble((x0 >> 4) & 0xFu), a3 = pm1_nibble((x1 >> 4) & 0xFu);
#pragma unroll
					for (int j = 0; j < kScanNJ; ++j)
					{
						const uint2 b = *reinterpret_cast<const uint2 *>(stile + (n0 + j * 8 + g) * S + ks * 8 + tig * 2);
						mma_s8_m16n8k32(acc[j], a0, a1, a2, a3, b.x, b.y);
					}
				}
				// c0 / c1: row r0, words 2 tig and 2 tig + 1 of the n8 tile; c2 / c3: row r1.  key = ((32 NW - dot) / 2 << kKeyShift) + k
#pragma unroll
				for (int j = 0; j < kScanNJ; ++j)
				{
#pragma unroll
					for (int e = 0; e < 2; ++e)
					{
						const int kl = n0 + j * 8 + tig * 2 + e;
						if (kl < n_valid)
						{
							const uint32_t base = (static_cast<uint32_t>(32 * NW) << (kKeyShift - 1)) + static_cast<uint32_t>(w0 + kl);
							top2_insert(k1a, k2a, base - (static_cast<uint32_t>(acc[j][e]) << (kKeyShift - 1)));
							top2_insert(k1b, k2b, base - (static_cast<uint32_t>(acc[j][2 + e]) << (kKeyShift - 1)));
						}
					}
				}
			}
#pragma unroll
			for (int o = 1; o < 4; o <<= 1)
			{
				const uint32_t oa1 = __shfl_xor_sync(0xFFFFFFFFu, k1a, o), oa2 = __shfl_xor_sync(0xFFFFFFFFu, k2a, o);
				const uint32_t ob1 = __shfl_xor_sync(0xFFFFFFFFu, k1b, o), ob2 = __shfl_xor_sync(0xFFFFFFFFu, k2b, o);
				top2_insert(k1a, k2a, oa1);
				top2_insert(k1a, k2a, oa2);
				top2_insert(k1b, k2b, ob1);
				top2_insert(k1b, k2b, ob2);
			}
			if (tig == 0)
			{
				// the same warp owns these rows in every pass: no barrier between the passes' merges
				if (r0 < nt)
				{
					uint32_t u1 = sa1[r0], u2 = sa2[r0];
					top2_insert(u1, u2, k1a);
					top2_insert(u1, u2, k2a);
					sa1[r0] = u1;
					sa2[r0] = u2;
				}
				if (r1 < nt)
				{
					uint32_t u1 = sa1[r1], u2 = sa2[r1];
					top2_insert(u1, u2, k1b);
					top2_insert(u1, u2, k2b);
					sa1[r1] = u1;
					sa2[r1] = u2;
				}
			}
		}
	}
}

// phase clocks of the matching kernel: diagnostics only, compiled in with -DLCD_DEBUG_PHASES
#ifdef LCD_DEBUG_PHASES
__device__ long long g_match_dbg[8];
#define MATCH_PHASE(k) do { if (blockIdx.x == 0 && threadIdx.x == 0) g_match_dbg[k] = clock64(); } while (0)
#else
#define MATCH_PHASE(k) do { } while (0)
#endif

// FROM side: addNewWords(descriptorsFrom, 1) on an empty dictionary.  Copies the nf descriptors of F to sdesc; on return L[k] is the
// descriptor that created word k and rank[i] the word of descriptor i.  Returns the number of words.  All threads must call it.
template <int NW>
__device__ int from_dictionary(const uint32_t * F, int nf, uint32_t * sdesc, uint32_t * sa1, uint32_t * sa2, int * res, uint16_t * L,
                               uint16_t * rank, uint8_t * flag, uint8_t * flag2, int * s_nL, float nndr)
{
	const int tid = threadIdx.x;
	for (int i = tid; i < nf * NW; i += blockDim.x) sdesc[i] = F[i]; // the scans re-read every descriptor ~nf/32 times
	for (int i = tid; i < nf; i += blockDim.x)
	{
		sa1[i] = kKeyNone;
		sa2[i] = kKeyNone;
		flag[i] = 1;
		res[i] = 0;
	}
	__syncthreads();
	int n_dict = 0;
	if (nf > 0) n_dict = resolve_rounds<NW>(sdesc, nf, sa1, sa2, res, L, rank, flag, flag2, s_nL, nndr, 1);
	__syncthreads();
	for (int i = tid; i < nf; i += blockDim.x)
		if (!flag[i]) rank[i] = static_cast<uint16_t>(-1 - res[i]);
	__syncthreads();
	return n_dict;
}

struct FromDictArgs
{
	const uint32_t * desc;  // signature store [slots][cap_from][NW]
	const int * n;          // [slots]
	const int * slot;       // [n_pairs] row of each pair (-1 = none)
	int cap_from;
	int rows;               // min(cap of the call, cap_from): size of the shared-memory arrays
	float nndr;
	FromDictTag * tag;      // [slots]
	uint16_t * kof;         // [slots][cap_from]
	uint16_t * creator;     // [slots][cap_from]
};

__host__ __device__ inline size_t from_dict_smem_bytes(int rows, int nw)
{
	return static_cast<size_t>(rows) * (static_cast<size_t>(nw) * 4 + 4 + 4 + 4 + 2 + 2 + 1 + 1) + 128;
}

// Builds the FROM dictionary of each pair's store row unless it is cached for this nf and NNDR already or an earlier pair of the batch
// has the same row (frames often share a hypothesis).  One CTA per pair, launched before pair_match_kernel on the same stream.
template <int NW>
__global__ void __launch_bounds__(kResolveThreads)
from_dict_build_kernel(const FromDictArgs a)
{
	extern __shared__ __align__(128) unsigned char smem_raw[];
	const int rows = a.rows;
	uint32_t * sdesc = reinterpret_cast<uint32_t *>(smem_raw); // [rows][NW]
	uint32_t * sa1 = sdesc + static_cast<size_t>(rows) * NW;
	uint32_t * sa2 = sa1 + rows;
	int * res = reinterpret_cast<int *>(sa2 + rows);
	uint16_t * L = reinterpret_cast<uint16_t *>(res + rows);
	uint16_t * rank = L + rows;
	uint8_t * flag = reinterpret_cast<uint8_t *>(rank + rows);
	uint8_t * flag2 = flag + rows;
	__shared__ int s_nL, s_build;
	const int pair = blockIdx.x, slot = a.slot[pair];
	if (slot < 0) return;
	const int nf = min(a.n[slot], rows);
	const uint32_t nndr_bits = __float_as_uint(a.nndr);
	if (threadIdx.x == 0)
	{
		const FromDictTag t = a.tag[slot];
		int build = t.nf != nf || t.nndr_bits != nndr_bits;
		for (int p = 0; p < pair && build; ++p)
			if (a.slot[p] == slot) build = 0;
		s_build = build;
	}
	__syncthreads();
	if (!s_build) return;
	const size_t base = static_cast<size_t>(slot) * a.cap_from;
	const int n_dict = from_dictionary<NW>(a.desc + base * NW, nf, sdesc, sa1, sa2, res, L, rank, flag, flag2, &s_nL, a.nndr);
	for (int i = threadIdx.x; i < nf; i += blockDim.x) a.kof[base + i] = rank[i];
	for (int k = threadIdx.x; k < n_dict; k += blockDim.x) a.creator[base + k] = L[k];
	__threadfence();
	__syncthreads();
	if (threadIdx.x == 0) a.tag[slot] = FromDictTag{nf, n_dict, nndr_bits, 0};
}

template <int NW>
__global__ void __launch_bounds__(kResolveThreads)
pair_match_kernel(const MatchArgs a)
{
	MATCH_PHASE(0);
	extern __shared__ __align__(128) unsigned char smem_raw[];
	const int cap = a.cap;
	uint32_t * stile = reinterpret_cast<uint32_t *>(smem_raw);           // [kScanWords][scan_stride_words(NW)] s8 words of the TO scan
	uint32_t * dict = stile + scan_tile_bytes(NW) / 4;                    // [cap][NW] words of the temporary dictionary
	uint32_t * sdesc = dict + static_cast<size_t>(cap) * NW;              // [cap][NW] the side being quantised (FROM, then TO)
	uint32_t * sa1 = sdesc + static_cast<size_t>(cap) * NW;               // [cap]
	uint32_t * sa2 = sa1 + cap;
	int * res = reinterpret_cast<int *>(sa2 + cap);
	int * cntF = res + cap;
	int * cntT = cntF + cap;
	uint16_t * L = reinterpret_cast<uint16_t *>(cntT + cap);
	uint16_t * rank = L + cap;
	uint16_t * idxF = rank + cap;
	uint16_t * idxT = idxF + cap;
	uint8_t * flag = reinterpret_cast<uint8_t *>(idxT + cap);
	uint8_t * flag2 = flag + cap;
	__shared__ int s_nL;

	const int tid = threadIdx.x;
	const int pair = blockIdx.x;
	const int frow = a.src.from_row(pair);
	const int nf = frow >= 0 ? min(a.src.from.n[frow], min(cap, a.src.from.cap)) : 0;
	const int nt = a.src.to_count(pair, cap);
	const size_t base = static_cast<size_t>(pair) * cap;
	const size_t fbase = static_cast<size_t>(frow >= 0 ? frow : 0) * a.src.from.cap;
	const size_t tbase = a.src.to_base(pair);
	const uint32_t * F = a.src.from.desc + fbase * NW;
	const uint32_t * T = a.src.to.desc + tbase * NW;

	// ---- FROM side: addNewWords(descriptorsFrom, 1) on an empty dictionary, or the store row's cached result -------------------
	__shared__ int s_cached;
	if (tid == 0)
	{
		const FromDictTag * t = a.from_tag && frow >= 0 ? a.from_tag + frow : nullptr;
		s_cached = t && t->nf == nf && t->nndr_bits == __float_as_uint(a.nndr) ? t->n_dict : -1;
	}
	__syncthreads();
	const bool cached = s_cached >= 0;
	int n_dict;
	if (cached)
	{
		n_dict = s_cached;
		for (int i = tid; i < nf; i += blockDim.x) rank[i] = a.from_kof[fbase + i];
		for (int k = tid; k < n_dict; k += blockDim.x) L[k] = a.from_creator[fbase + k];
		__syncthreads();
	}
	else n_dict = from_dictionary<NW>(F, nf, sdesc, sa1, sa2, res, L, rank, flag, flag2, &s_nL, a.nndr);
	MATCH_PHASE(1);
	for (int k = tid; k < n_dict; k += blockDim.x)
	{
		cntF[k] = 0;
		cntT[k] = 0;
		uint32_t q[NW];
		load_desc<NW>(cached ? F : sdesc, L[k], q);
#pragma unroll
		for (int v = 0; v < NW; ++v) dict[static_cast<size_t>(k) * NW + v] = q[v];
	}
	__syncthreads();
	for (int i = tid; i < nf; i += blockDim.x)
	{
		const int k = rank[i];
		atomicAdd(&cntF[k], 1);
		idxF[k] = static_cast<uint16_t>(i);
		if (a.from_ids) a.from_ids[base + i] = k + 1;
	}
	__syncthreads();

	MATCH_PHASE(2);
	// ---- TO side: update(); addNewWords(descriptorsTo, 2) --------------------------------------
	__syncthreads();
	for (int i = tid; i < nt * NW; i += blockDim.x) sdesc[i] = T[i];
	for (int j = tid; j < nt; j += blockDim.x)
	{
		sa1[j] = kKeyNone;
		sa2[j] = kKeyNone;
	}
	__syncthreads();
	to_dict_knn2_mma<NW>(sdesc, nt, dict, n_dict, stile, sa1, sa2);
	__syncthreads();
	for (int j = tid; j < nt; j += blockDim.x)
	{
		const uint32_t k1 = sa1[j], k2 = sa2[j];
		int bt;
		flag[j] = nndr_decide(k1, k2, kKeyNone, kKeyNone, a.nndr, bt) ? 1 : 0;
		res[j] = static_cast<int>(k1 & kKeyRowMask);
	}
	__syncthreads();
	MATCH_PHASE(3);
	if (nt > 0) resolve_rounds<NW>(sdesc, nt, sa1, sa2, res, L, rank, flag, flag2, &s_nL, a.nndr, 1);
	__syncthreads();
	MATCH_PHASE(4);
	for (int j = tid; j < nt; j += blockDim.x)
	{
		int id;
		if (flag[j]) id = n_dict + 1 + rank[j];
		else if (res[j] >= 0)
		{
			id = res[j] + 1;
			atomicAdd(&cntT[res[j]], 1);
			idxT[res[j]] = static_cast<uint16_t>(j);
		}
		else id = n_dict + 1 + (-1 - res[j]);
		if (a.to_ids) a.to_ids[base + j] = id;
	}
	__syncthreads();

	// ---- correspondences: ids seen exactly once on each side, finite 3D, ascending id ------------
	for (int k = tid; k < n_dict; k += blockDim.x)
	{
		bool ok = cntF[k] == 1 && cntT[k] == 1;
		if (ok)
		{
			const float * p = a.src.from.xyz + (fbase + idxF[k]) * 3;
			ok = isfinite(p[0]) && isfinite(p[1]) && isfinite(p[2]);
		}
		flag[k] = ok ? 1 : 0;
	}
	__syncthreads();
	if (tid < 32)
	{
		const int n = warp0_compact(flag, n_dict, L, rank);
		if (tid == 0)
		{
			s_nL = n;
			a.n_match[pair] = n;
		}
	}
	__syncthreads();
	const int nm = s_nL;
	for (int m = tid; m < nm; m += blockDim.x)
	{
		const int k = L[m];
		const int fi = idxF[k], ti = idxT[k];
		const float * p = a.src.from.xyz + (fbase + fi) * 3;
		const float * q = a.src.to.uv + (tbase + ti) * 2;
		a.obj[(base + m) * 3 + 0] = p[0];
		a.obj[(base + m) * 3 + 1] = p[1];
		a.obj[(base + m) * 3 + 2] = p[2];
		a.img[(base + m) * 2 + 0] = q[0];
		a.img[(base + m) * 2 + 1] = q[1];
		gather_obj_to(a.src, a.obj_to, base + m, tbase, ti);
		a.match_id[base + m] = k + 1;
		a.match_from[base + m] = fi;
		a.match_to[base + m] = ti;
	}
	MATCH_PHASE(5);
}

// ---- pair matching of float descriptors (LCD_DESC_F32, 64-D / 128-D) ---------------------------------------------------------
// The same temporary dictionary as from_dict_build_kernel + pair_match_kernel, with squared L2 summed in rtflann's order
// (l2_path.cuh) in place of Hamming (VWDictionary.cpp:1020-1028: NORM_L2SQR / rtflann L2 for CV_32F).  A float row is 256 or 512
// bytes, so both sides stay in global memory (L2-resident per pair) and shared memory holds per-row scalars only; the work is split
// into three launches of at most 256 threads (the new-word loop, resolve_rounds_l2, is written for kL2ResolveThreads):
//   from_dict_l2_kernel      FROM side, addNewWords(descriptorsFrom, 1): kof[i] = word of descriptor i, creator[k] = descriptor
//                            that created word k, tag.n_dict.  Store rows: cached per row as the binary build; host pairs: per pair.
//   to_dict_knn2_l2_kernel   TO side, the 2-NN of every TO descriptor over the FROM words, exact, keys pack64(d, k) (ties -> lowest k)
//   pair_match_l2_kernel     TO side, the NNDR decision and the new-word loop of addNewWords(descriptorsTo, 2), then the
//                            correspondences into exactly the outputs pair_match_kernel writes
constexpr int kL2ScanThreads = 128; // TO descriptors per CTA of the 2-NN scan, one per thread (DIM floats in registers up to 128-D)
constexpr int kL2ScanWords = 32;    // dictionary words staged per shared-memory tile of the scan

__host__ __device__ inline size_t from_dict_l2_smem_bytes(int rows)
{
	return static_cast<size_t>(rows) * (8 + 8 + 4 + 2 + 2 + 1) + 128;
}

__host__ __device__ inline size_t match_l2_smem_bytes(int cap)
{
	return static_cast<size_t>(cap) * (8 + 8 + 4 + 4 + 4 + 2 + 2 + 2 + 2 + 1) + 128;
}

// One CTA per pair.  a.slot set: store rows, built unless cached for this nf and NNDR or built by an earlier pair of the batch (as
// from_dict_build_kernel).  a.slot == nullptr: row = pair, always built (the host pairs of lcd_verify_batch).
template <int DIM>
__global__ void __launch_bounds__(kL2ResolveThreads)
from_dict_l2_kernel(const FromDictArgs a)
{
	extern __shared__ __align__(128) unsigned char smem_raw[];
	const int rows = a.rows;
	unsigned long long * sa1 = reinterpret_cast<unsigned long long *>(smem_raw); // [rows] no index hits: the dictionary starts empty
	unsigned long long * sa2 = sa1 + rows;
	int * res = reinterpret_cast<int *>(sa2 + rows);
	uint16_t * L = reinterpret_cast<uint16_t *>(res + rows);
	uint16_t * rank = L + rows;
	uint8_t * flag = reinterpret_cast<uint8_t *>(rank + rows);
	__shared__ int s_nL, s_build;
	const int pair = blockIdx.x, slot = a.slot ? a.slot[pair] : pair;
	if (slot < 0) return;
	const int nf = min(a.n[slot], rows);
	const uint32_t nndr_bits = __float_as_uint(a.nndr);
	if (threadIdx.x == 0)
	{
		int build = 1;
		if (a.slot)
		{
			const FromDictTag t = a.tag[slot];
			build = t.nf != nf || t.nndr_bits != nndr_bits;
			for (int p = 0; p < pair && build; ++p)
				if (a.slot[p] == slot) build = 0;
		}
		s_build = build;
	}
	__syncthreads();
	if (!s_build) return;
	const size_t base = static_cast<size_t>(slot) * a.cap_from;
	for (int i = threadIdx.x; i < nf; i += blockDim.x)
	{
		sa1[i] = kKey64None;
		sa2[i] = kKey64None;
		flag[i] = 1;
		res[i] = 0;
	}
	__syncthreads();
	const int n_dict = resolve_rounds_l2<DIM>(reinterpret_cast<const float *>(a.desc) + base * DIM, nf, sa1, sa2, res, L, rank, flag, &s_nL, a.nndr, 1);
	__syncthreads();
	for (int i = threadIdx.x; i < nf; i += blockDim.x) a.kof[base + i] = flag[i] ? rank[i] : static_cast<uint16_t>(-1 - res[i]);
	for (int k = threadIdx.x; k < n_dict; k += blockDim.x) a.creator[base + k] = L[k];
	__threadfence();
	__syncthreads();
	if (threadIdx.x == 0) a.tag[slot] = FromDictTag{nf, n_dict, nndr_bits, 0};
}

// grid (n_pairs, ceil(cap / kL2ScanThreads)): pairs on x, which has no 65 535 limit, as in the other matching kernels.  keys[pair][j] = the two nearest FROM words of TO descriptor j.  The words are read
// through a.from_creator from the FROM row, kL2ScanWords at a time into shared memory, and every thread compares its descriptor
// with each of them (broadcast reads).
template <int DIM>
__global__ void __launch_bounds__(kL2ScanThreads)
to_dict_knn2_l2_kernel(const MatchArgs a, ulonglong2 * __restrict__ keys)
{
	__shared__ __align__(16) float s_w[kL2ScanWords * DIM];
	const int pair = blockIdx.x, tid = threadIdx.x;
	const int nt = a.src.to_count(pair, a.cap);
	const int j = blockIdx.y * kL2ScanThreads + tid;
	if (blockIdx.y * kL2ScanThreads >= nt) return;
	const int frow = a.src.from_row(pair);
	const int n_dict = frow >= 0 ? a.from_tag[frow].n_dict : 0;
	const size_t fbase = static_cast<size_t>(frow >= 0 ? frow : 0) * a.src.from.cap;
	const float4 * F4 = reinterpret_cast<const float4 *>(a.src.from.desc + fbase * DIM);
	const uint16_t * creator = a.from_creator + fbase;
	const float * tq = reinterpret_cast<const float *>(a.src.to.desc + (a.src.to_base(pair) + min(j, nt - 1)) * DIM);
	unsigned long long k1 = kKey64None, k2 = kKey64None;
	float4 * s_w4 = reinterpret_cast<float4 *>(s_w);
	if constexpr (DIM > 128)
	{
		// 256-D: the TO descriptor is read a chunk at a time (l2_chunked_rows); 32 KB of words + 16 KB of running totals
		__shared__ float s_acc[kL2ScanWords * kL2ScanThreads];
		for (int w0 = 0; w0 < n_dict; w0 += kL2ScanWords)
		{
			const int nw = min(kL2ScanWords, n_dict - w0);
			__syncthreads();
			for (int i = tid; i < nw * (DIM / 4); i += kL2ScanThreads)
				s_w4[i] = F4[static_cast<size_t>(creator[w0 + i / (DIM / 4)]) * (DIM / 4) + i % (DIM / 4)];
			__syncthreads();
			l2_chunked_rows<DIM, kL2ScanThreads>(tq, s_w, nw, s_acc, tid);
			for (int r = 0; r < nw; ++r) top2_insert64(k1, k2, pack64(s_acc[r * kL2ScanThreads + tid], static_cast<uint32_t>(w0 + r)));
		}
	}
	else
	{
		float q[DIM];
		{
			const float4 * t4 = reinterpret_cast<const float4 *>(tq);
#pragma unroll
			for (int v = 0; v < DIM / 4; ++v)
			{
				const float4 x = t4[v];
				q[4 * v] = x.x;
				q[4 * v + 1] = x.y;
				q[4 * v + 2] = x.z;
				q[4 * v + 3] = x.w;
			}
		}
		for (int w0 = 0; w0 < n_dict; w0 += kL2ScanWords)
		{
			const int nw = min(kL2ScanWords, n_dict - w0);
			__syncthreads();
			for (int i = tid; i < nw * (DIM / 4); i += kL2ScanThreads)
				s_w4[i] = F4[static_cast<size_t>(creator[w0 + i / (DIM / 4)]) * (DIM / 4) + i % (DIM / 4)];
			__syncthreads();
			for (int r = 0; r < nw; ++r) top2_insert64(k1, k2, pack64(l2_reg_vs_stream<DIM>(q, s_w + r * DIM), static_cast<uint32_t>(w0 + r)));
		}
	}
	if (j < nt) keys[static_cast<size_t>(pair) * a.cap + j] = make_ulonglong2(k1, k2);
}

// One CTA per pair, after to_dict_knn2_l2_kernel.  Dynamic shared memory: match_l2_smem_bytes(cap).
template <int DIM>
__global__ void __launch_bounds__(kL2ResolveThreads)
pair_match_l2_kernel(const MatchArgs a, const ulonglong2 * __restrict__ keys)
{
	extern __shared__ __align__(128) unsigned char smem_raw[];
	const int cap = a.cap;
	unsigned long long * sa1 = reinterpret_cast<unsigned long long *>(smem_raw); // [cap] the TO descriptors' two nearest FROM words
	unsigned long long * sa2 = sa1 + cap;
	int * res = reinterpret_cast<int *>(sa2 + cap);
	int * cntF = res + cap;
	int * cntT = cntF + cap;
	uint16_t * L = reinterpret_cast<uint16_t *>(cntT + cap);
	uint16_t * rank = L + cap;
	uint16_t * idxF = rank + cap;
	uint16_t * idxT = idxF + cap;
	uint8_t * flag = reinterpret_cast<uint8_t *>(idxT + cap);
	__shared__ int s_nL;

	const int tid = threadIdx.x;
	const int pair = blockIdx.x;
	const int frow = a.src.from_row(pair);
	const int nf = frow >= 0 ? min(a.src.from.n[frow], min(cap, a.src.from.cap)) : 0;
	const int nt = a.src.to_count(pair, cap);
	const int n_dict = frow >= 0 ? a.from_tag[frow].n_dict : 0;
	const size_t base = static_cast<size_t>(pair) * cap;
	const size_t fbase = static_cast<size_t>(frow >= 0 ? frow : 0) * a.src.from.cap;
	const size_t tbase = a.src.to_base(pair);

	for (int k = tid; k < n_dict; k += blockDim.x)
	{
		cntF[k] = 0;
		cntT[k] = 0;
	}
	for (int j = tid; j < nt; j += blockDim.x)
	{
		const ulonglong2 kk = keys[base + j];
		sa1[j] = kk.x;
		sa2[j] = kk.y;
		int bt;
		flag[j] = nndr_decide64(kk.x, kk.y, kKey64None, kKey64None, a.nndr, bt) ? 1 : 0;
		res[j] = static_cast<int>(key64_row(kk.x));
	}
	__syncthreads();
	for (int i = tid; i < nf; i += blockDim.x)
	{
		const int k = a.from_kof[fbase + i];
		atomicAdd(&cntF[k], 1);
		idxF[k] = static_cast<uint16_t>(i);
	}
	resolve_rounds_l2<DIM>(reinterpret_cast<const float *>(a.src.to.desc) + tbase * DIM, nt, sa1, sa2, res, L, rank, flag, &s_nL, a.nndr, 1);
	__syncthreads();
	for (int j = tid; j < nt; j += blockDim.x)
	{
		if (!flag[j] && res[j] >= 0)
		{
			atomicAdd(&cntT[res[j]], 1);
			idxT[res[j]] = static_cast<uint16_t>(j);
		}
	}
	__syncthreads();

	// ---- correspondences: ids seen exactly once on each side, finite 3D, ascending id (as pair_match_kernel) ------------
	for (int k = tid; k < n_dict; k += blockDim.x)
	{
		bool ok = cntF[k] == 1 && cntT[k] == 1;
		if (ok)
		{
			const float * p = a.src.from.xyz + (fbase + idxF[k]) * 3;
			ok = isfinite(p[0]) && isfinite(p[1]) && isfinite(p[2]);
		}
		flag[k] = ok ? 1 : 0;
	}
	__syncthreads();
	if (tid < 32)
	{
		const int n = warp0_compact(flag, n_dict, L, rank);
		if (tid == 0)
		{
			s_nL = n;
			a.n_match[pair] = n;
		}
	}
	__syncthreads();
	const int nm = s_nL;
	for (int m = tid; m < nm; m += blockDim.x)
	{
		const int k = L[m];
		const int fi = idxF[k], ti = idxT[k];
		const float * p = a.src.from.xyz + (fbase + fi) * 3;
		const float * q = a.src.to.uv + (tbase + ti) * 2;
		a.obj[(base + m) * 3 + 0] = p[0];
		a.obj[(base + m) * 3 + 1] = p[1];
		a.obj[(base + m) * 3 + 2] = p[2];
		a.img[(base + m) * 2 + 0] = q[0];
		a.img[(base + m) * 2 + 1] = q[1];
		gather_obj_to(a.src, a.obj_to, base + m, tbase, ti);
		a.match_id[base + m] = k + 1;
		a.match_from[base + m] = fi;
		a.match_to[base + m] = ti;
	}
}

// ------------------------------------------------------------------- second pass: matching with a guess
// Reg/RepeatOnce (Registration.cpp:221-229): when the first registration succeeded, RegistrationVis runs again with that transform
// as the guess (RegistrationVis.cpp:1017-1070, :1225-1370, Vis/CorGuessMatchToProjection = false): the 3-D points of FROM are
// projected into TO's image, the TO keypoints within Vis/CorGuessWinSize pixels of a projection are its candidates, ranked by
// cv::BFMatcher::knnMatch(k = 2) + the strict Vis/CorNNDR test (a single candidate is accepted as it is); a TO keypoint goes to the
// first FROM point (ascending index) that selects it; correspondences in ascending FROM index.  The reference finds the candidates
// with a randomised kd-tree limited to 32 checks — approximate and unordered (SURVEY App. C.3); this kernel does the EXACT radius
// search (squared distance < r^2, rtflann/util/result_set.h:475-479) with candidates in ascending TO index, like the oracle.
// Pairs whose first pass failed (or whose pose is the identity: "guess not set") keep their first-pass correspondences.
struct GuessMatchArgs
{
	PairSource src;
	int cap;
	const int * ok1;        // [n_pairs] first pass accepted
	const double * rvec;    // [n_pairs][3] first-pass pose
	const double * tvec;
	CamK cam;               // the call's TO camera; a pair with its own (src.to_cam) uses that one
	int img_w, img_h;
	float win;              // Vis/CorGuessWinSize
	float nndr;
	// outputs (overwritten only for pairs that run the second pass)
	float * obj;
	float * img;
	float * obj_to;
	int * match_id;         // FROM index of every correspondence (the reference's ids of this pass)
	int * match_from;
	int * match_to;
	int * n_match;
};

__host__ __device__ inline size_t guess_smem_bytes(int cap) { return static_cast<size_t>(cap) * (8 + 4 + 4 + 2 + 2 + 1) + 64; }

// Descriptor kinds of the guess pass: the distance cv::BFMatcher ranks a FROM point's candidates by.  kWords: 32-bit words per row.
template <int NW>
struct HammingDesc // NORM_HAMMING; the FROM descriptor is held in registers
{
	static constexpr int kWords = NW;
	using Dist = uint32_t;
	static constexpr Dist kFar = 0xFFFFFFFFu;
	struct Query
	{
		uint32_t w[NW];
	};
	__device__ __forceinline__ static void load(const uint32_t * base, int i, Query & q) { load_desc<NW>(base, i, q.w); }
	__device__ __forceinline__ static Dist dist(const Query & q, const uint32_t * base, int j)
	{
		uint32_t w[NW];
		load_desc<NW>(base, j, w);
		return hamming<NW, 0>(q.w, w);
	}
};

template <int DIM>
struct L2Desc // NORM_L2SQR in rtflann's order; a 256 / 512-byte FROM descriptor is streamed from memory, not held in registers
{
	static constexpr int kWords = DIM;
	using Dist = float;
	static constexpr Dist kFar = INFINITY;
	struct Query
	{
		const float * p;
	};
	__device__ __forceinline__ static void load(const uint32_t * base, int i, Query & q)
	{
		q.p = reinterpret_cast<const float *>(base) + static_cast<size_t>(i) * DIM;
	}
	__device__ __forceinline__ static Dist dist(const Query & q, const uint32_t * base, int j)
	{
		return l2_rtflann<DIM>(q.p, reinterpret_cast<const float *>(base) + static_cast<size_t>(j) * DIM);
	}
};

template <class D>
__global__ void __launch_bounds__(256)
guess_match_kernel(const GuessMatchArgs a)
{
	extern __shared__ __align__(16) unsigned char smem_raw[];
	const int cap = a.cap;
	float * s_uv = reinterpret_cast<float *>(smem_raw);            // [cap][2] TO keypoints
	int * sel = reinterpret_cast<int *>(s_uv + 2 * cap);           // [cap] TO index chosen by FROM i
	int * claim = sel + cap;                                       // [cap] smallest FROM index that chose TO j
	uint16_t * L = reinterpret_cast<uint16_t *>(claim + cap);      // [cap]
	uint16_t * rank = L + cap;                                     // [cap]
	uint8_t * flag = reinterpret_cast<uint8_t *>(rank + cap);      // [cap]
	__shared__ double s_R[9], s_t[3];
	__shared__ CamK s_cam;
	__shared__ int s_n;
	const int tid = threadIdx.x, pair = blockIdx.x;
	if (!a.ok1[pair]) return;
	const double * rv = a.rvec + pair * 3;
	const double * tv = a.tvec + pair * 3;
	if (rv[0] == 0.0 && rv[1] == 0.0 && rv[2] == 0.0 && tv[0] == 0.0 && tv[1] == 0.0 && tv[2] == 0.0) return; // guess.isIdentity(): global matching again
	const int frow = a.src.from_row(pair);
	if (frow < 0) return;
	const FrameCam * fc = a.src.to_cam(pair);
	const int img_w = fc ? fc->w : a.img_w, img_h = fc ? fc->h : a.img_h;
	if (img_w <= 0 || img_h <= 0) return; // no image size: the reference has no guess pass for this camera
	const int nf = min(a.src.from.n[frow], min(cap, a.src.from.cap));
	const int nt = a.src.to_count(pair, cap);
	const size_t base = static_cast<size_t>(pair) * cap;
	const size_t fbase = static_cast<size_t>(frow) * a.src.from.cap, tbase = a.src.to_base(pair);
	if (tid == 0)
	{
		rodrigues_v2m(rv, s_R, nullptr);
		s_t[0] = tv[0];
		s_t[1] = tv[1];
		s_t[2] = tv[2];
		s_cam = fc ? CamK{fc->fx, fc->fy, fc->cx, fc->cy} : a.cam;
	}
	for (int j = tid; j < nt; j += blockDim.x)
	{
		s_uv[2 * j] = a.src.to.uv[(tbase + j) * 2];
		s_uv[2 * j + 1] = a.src.to.uv[(tbase + j) * 2 + 1];
		claim[j] = 0x7FFFFFFF;
	}
	__syncthreads();
	const float r2 = __fmul_rn(a.win, a.win);
	const float wmax = static_cast<float>(img_w - 1), hmax = static_cast<float>(img_h - 1);
	for (int i = tid; i < nf; i += blockDim.x)
	{
		int m = -1;
		const float * X = a.src.from.xyz + (fbase + i) * 3;
		double pu, pv;
		// the first pass's PnP pose is (guess * localTransform)^-1 of the reference's projection (RegistrationVis.cpp:1034)
		project_point(s_R, s_t, s_cam, X, pu, pv);
		const float px = static_cast<float>(pu), py = static_cast<float>(pv);
		const float zc = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(static_cast<float>(s_R[6]), X[0]), __fmul_rn(static_cast<float>(s_R[7]), X[1])),
		                                     __fmul_rn(static_cast<float>(s_R[8]), X[2])), static_cast<float>(s_t[2]));
		const bool inb = isfinite(px) && !(px < 0.0f) && !(px >= wmax) && isfinite(py) && !(py < 0.0f) && !(py >= hmax);
		if (inb && zc > 0.0f && isfinite(X[0]) && isfinite(X[1]) && isfinite(X[2]))
		{
			typename D::Query q;
			D::load(a.src.from.desc + fbase * D::kWords, i, q);
			int cnt = 0, b1 = -1;
			typename D::Dist d1 = D::kFar, d2 = D::kFar;
			for (int j = 0; j < nt; ++j)
			{
				const float dx = __fsub_rn(px, s_uv[2 * j]), dy = __fsub_rn(py, s_uv[2 * j + 1]);
				const float dist = __fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy));
				if (!(dist < r2)) continue;
				++cnt;
				const typename D::Dist d = D::dist(q, a.src.to.desc + tbase * D::kWords, j);
				if (d < d1)
				{
					d2 = d1;
					d1 = d;
					b1 = j;
				}
				else if (d < d2) d2 = d;
			}
			if (cnt >= 2)
			{
				if (static_cast<float>(d1) < __fmul_rn(a.nndr, static_cast<float>(d2))) m = b1;
			}
			else if (cnt == 1) m = b1;
			if (m >= 0) atomicMin(&claim[m], i);
		}
		sel[i] = m;
	}
	__syncthreads();
	for (int i = tid; i < nf; i += blockDim.x) flag[i] = (sel[i] >= 0 && claim[sel[i]] == i) ? 1 : 0;
	__syncthreads();
	if (tid < 32)
	{
		const int n = warp0_compact(flag, nf, L, rank);
		if (tid == 0)
		{
			s_n = n;
			a.n_match[pair] = n;
		}
	}
	__syncthreads();
	const int nm = s_n;
	for (int m = tid; m < nm; m += blockDim.x)
	{
		const int fi = L[m], ti = sel[fi];
		const float * p = a.src.from.xyz + (fbase + fi) * 3;
		a.obj[(base + m) * 3 + 0] = p[0];
		a.obj[(base + m) * 3 + 1] = p[1];
		a.obj[(base + m) * 3 + 2] = p[2];
		a.img[(base + m) * 2 + 0] = s_uv[2 * ti];
		a.img[(base + m) * 2 + 1] = s_uv[2 * ti + 1];
		gather_obj_to(a.src, a.obj_to, base + m, tbase, ti);
		a.match_id[base + m] = fi;
		a.match_from[base + m] = fi;
		a.match_to[base + m] = ti;
	}
}

// ------------------------------------------------------------------------------------ PnP RANSAC
struct PnpArgs
{
	const float * obj;   // [n_pairs][cap][3]
	const float * img;   // [n_pairs][cap][2]
	const int * n_pts;   // [n_pairs]
	int cap;
	CamK cam;
	int iterations;        // Vis/Iterations (<= kMaxRansacIters)
	float reproj;          // Vis/PnPReprojError
	int min_inliers;       // Vis/MinInliers
	int refine_iterations; // Vis/PnPRefineIterations
	float refine_sigma;    // 3.0
	int gate_min_matches;  // 1: util3d::estimateMotion3DTo2D semantics (PnP only with >= min_inliers correspondences, :111);
	                       // 0: util3d::solvePnPRansac alone (lcd_pnp_ransac)
	// covariance of util3d::estimateMotion3DTo2D (util3d_motion_estimation.cpp:156-258); cov6 == nullptr: skipped
	const float * obj_to;  // [n_pairs][cap][3] words3B of each correspondence (NaN = none) or nullptr (words3B empty)
	int var_median_ratio;  // Vis/PnPVarianceMedianRatio (> 1)
	float max_variance;    // Vis/PnPMaxVariance (0 = off)
	int split_linear;      // Vis/PnPSplitLinearCovComponents
	int img_w, img_h;      // CameraModel::imageSize() of the TO camera (0 x 0 = not set)
	// each pair's own TO camera (K, image size and local transform in place of cam, img_w, img_h and identity) where it has one
	const FrameCam * cam_tab; // nullptr: every pair takes the fields above
	const int * cam_row;      // nullptr: cam_tab[pair]; else cam_tab[cam_row[pair]]
	double * cov6;         // [n_pairs][6] diagonal of the 6x6 covariance (the reference only ever scales the identity)
	// outputs
	double * rvec;      // [n_pairs][3]
	double * tvec;      // [n_pairs][3]
	int * inliers;      // [n_pairs][cap] indices into the correspondence list
	int * n_inliers;    // [n_pairs]
	int * iters_run;    // [n_pairs]
	int * ok;           // [n_pairs] 1 = accepted (inliers >= min_inliers)
	float * transform;  // [n_pairs][12] (localTransform * pnp)^-1
	long long * phase_clk; // [n_pairs][16] clock64() at the phase boundaries (diagnostics; may be null)
};

__host__ __device__ inline size_t pnp_smem_bytes(int cap)
{
	return static_cast<size_t>(cap) * (12 + 8 + 4 + 4 + 2 + 2 + 1) + kMaxRansacIters * (6 * 2) + kPnpChunk * (4 + 6 * 8) + (28 * 32 + 32) * 8 + 1024;
}

// block-wide sum of NV doubles per thread; result valid in all threads (via smem)
template <int NV>
__device__ inline void block_sum(double (&v)[NV], double * s_red /* [NV * 32] */, double * s_out /* [NV] */)
{
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
#pragma unroll
	for (int k = 0; k < NV; ++k)
	{
		double x = v[k];
#pragma unroll
		for (int o = 16; o > 0; o >>= 1) x += __shfl_down_sync(0xFFFFFFFFu, x, o);
		if (lane == 0) s_red[k * 32 + warp] = x;
	}
	__syncthreads();
	if (threadIdx.x < NV)
	{
		double x = 0;
		for (int w = 0; w < nwarps; ++w) x += s_red[threadIdx.x * 32 + w];
		s_out[threadIdx.x] = x;
	}
	__syncthreads();
#pragma unroll
	for (int k = 0; k < NV; ++k) v[k] = s_out[k];
	__syncthreads();
}

struct LmState
{
	double param[6], prev[6], JtJ[36], JtErr[6];
	double R[9], dRdr[27];
	double prevErrNorm;
	int lambdaLg10, iters, done, cont;
};

// LM step: param = prev - (JtJ with diag*(1+lambda))^-1 JtErr   (CvLevMarq::step)
__device__ inline void lm_step(LmState & s)
{
	const double lambda = exp(s.lambdaLg10 * log(10.0));
	double A[36], v[36], dx[6] = {0, 0, 0, 0, 0, 0};
	int ord[6];
	for (int i = 0; i < 36; ++i) A[i] = s.JtJ[i];
	for (int i = 0; i < 6; ++i) A[i * 6 + i] *= 1.0 + lambda;
	if (chol_solve<6>(A, s.JtErr, dx))
	{
		for (int i = 0; i < 6; ++i) s.param[i] = s.prev[i] - dx[i];
		return;
	}
	for (int i = 0; i < 6; ++i) dx[i] = 0;
	sym_eigen<6>(A, v, ord);
	const double wmax = A[ord[0] * 6 + ord[0]];
	for (int kk = 0; kk < 6; ++kk)
	{
		const int k = ord[kk];
		const double w = A[k * 6 + k];
		if (w <= 2.220446049250313e-16 * 6 * wmax) continue;
		double c = 0;
		for (int i = 0; i < 6; ++i) c += v[i * 6 + k] * s.JtErr[i];
		c /= w;
		for (int i = 0; i < 6; ++i) dx[i] += c * v[i * 6 + k];
	}
	for (int i = 0; i < 6; ++i) s.param[i] = s.prev[i] - dx[i];
}

// cv::solvePnP(SOLVEPNP_ITERATIVE, useExtrinsicGuess = true) on the points X[list[0..m)], cooperatively by the CTA.
__device__ inline void lm_refine_block(const float * X, const float * uv, const uint16_t * list, int m, const CamK & cam, LmState & s,
                                       double * s_red, double * s_out)
{
	const int tid = threadIdx.x;
	if (tid == 0)
	{
		s.lambdaLg10 = -3;
		s.iters = 0;
		s.done = 0;
		s.prevErrNorm = 1.7976931348623157e308;
	}
	__syncthreads();
	for (;;)
	{
		if (tid == 0) rodrigues_v2m(s.param, s.R, s.dRdr);
		__syncthreads();
		// JtJ (upper 21) + JtErr (6) + |err|^2
		double acc[28];
#pragma unroll
		for (int k = 0; k < 28; ++k) acc[k] = 0;
		for (int p = tid; p < m; p += blockDim.x)
		{
			const float * P = X + 3 * list[p];
			const double Xx = P[0], Xy = P[1], Xz = P[2];
			const double x = s.R[0] * Xx + s.R[1] * Xy + s.R[2] * Xz + s.param[3];
			const double y = s.R[3] * Xx + s.R[4] * Xy + s.R[5] * Xz + s.param[4];
			double z = s.R[6] * Xx + s.R[7] * Xy + s.R[8] * Xz + s.param[5];
			z = z ? 1. / z : 1;
			const double xn = x * z, yn = y * z;
			double j0[6], j1[6];
			j0[3] = cam.fu * z;
			j0[4] = 0;
			j0[5] = -cam.fu * xn * z;
			j1[3] = 0;
			j1[4] = cam.fv * z;
			j1[5] = -cam.fv * yn * z;
			for (int k = 0; k < 3; ++k)
			{
				const double * d = s.dRdr + 9 * k;
				const double dx = d[0] * Xx + d[1] * Xy + d[2] * Xz;
				const double dy = d[3] * Xx + d[4] * Xy + d[5] * Xz;
				const double dz = d[6] * Xx + d[7] * Xy + d[8] * Xz;
				j0[k] = cam.fu * (dx * z - xn * z * dz);
				j1[k] = cam.fv * (dy * z - yn * z * dz);
			}
			const double e0 = xn * cam.fu + cam.uc - static_cast<double>(uv[2 * list[p]]);
			const double e1 = yn * cam.fv + cam.vc - static_cast<double>(uv[2 * list[p] + 1]);
			int q = 0;
#pragma unroll
			for (int a = 0; a < 6; ++a)
#pragma unroll
				for (int b = a; b < 6; ++b) acc[q++] += j0[a] * j0[b] + j1[a] * j1[b];
#pragma unroll
			for (int a = 0; a < 6; ++a) acc[21 + a] += j0[a] * e0 + j1[a] * e1;
			acc[27] += e0 * e0 + e1 * e1;
		}
		block_sum<28>(acc, s_red, s_out);
		if (tid == 0)
		{
			int q = 0;
			for (int a = 0; a < 6; ++a)
				for (int b = a; b < 6; ++b)
				{
					s.JtJ[a * 6 + b] = acc[q];
					s.JtJ[b * 6 + a] = acc[q];
					++q;
				}
			for (int a = 0; a < 6; ++a)
			{
				s.JtErr[a] = acc[21 + a];
				s.prev[a] = s.param[a];
			}
			lm_step(s);
			if (s.iters == 0) s.prevErrNorm = sqrt(acc[27]);
		}
		__syncthreads();
		// CHECK_ERR
		for (;;)
		{
			if (tid == 0) rodrigues_v2m(s.param, s.R, nullptr);
			__syncthreads();
			double e[1] = {0};
			for (int p = tid; p < m; p += blockDim.x)
			{
				double u, v;
				project_point(s.R, s.param + 3, cam, X + 3 * list[p], u, v);
				const double e0 = u - static_cast<double>(uv[2 * list[p]]), e1 = v - static_cast<double>(uv[2 * list[p] + 1]);
				e[0] += e0 * e0 + e1 * e1;
			}
			block_sum<1>(e, s_red, s_out);
			if (tid == 0)
			{
				const double errNorm = sqrt(e[0]);
				s.cont = 0;
				if (errNorm > s.prevErrNorm && ++s.lambdaLg10 <= 16)
				{
					lm_step(s);
					s.cont = 1;
				}
				else
				{
					s.lambdaLg10 = max(s.lambdaLg10 - 1, -16);
					double num = 0, den = 0;
					for (int i = 0; i < 6; ++i)
					{
						num += (s.param[i] - s.prev[i]) * (s.param[i] - s.prev[i]);
						den += s.prev[i] * s.prev[i];
					}
					if (++s.iters >= 20 || sqrt(num) < 1.1920928955078125e-07 * sqrt(den)) s.done = 1;
					s.prevErrNorm = errNorm;
				}
			}
			__syncthreads();
			if (!s.cont) break;
		}
		if (s.done) break;
	}
}

__global__ void __launch_bounds__(kVerifyThreads)
pnp_ransac_kernel(const PnpArgs a)
{
	extern __shared__ __align__(128) unsigned char smem_raw[];
	const int cap = a.cap;
	double * h_rt = reinterpret_cast<double *>(smem_raw);                    // [kPnpChunk][6]
	double * s_red = h_rt + kPnpChunk * 6;                              // [28*32]
	double * s_out = s_red + 28 * 32;                                        // [32]
	float * X = reinterpret_cast<float *>(s_out + 32);                       // [cap][3]
	float * uv = X + static_cast<size_t>(cap) * 3;                           // [cap][2]
	float * errs = uv + static_cast<size_t>(cap) * 2;                        // [cap]
	float * cbuf = errs + cap;                                               // [cap] covariance pass: per-inlier error values
	// [kPnpChunk] ints after cbuf are not used since a wave's counts moved into h_rt + s_red; pnp_smem_bytes keeps its size unchanged
	uint16_t * sidx = reinterpret_cast<uint16_t *>(reinterpret_cast<int *>(cbuf + cap) + kPnpChunk); // [kMaxRansacIters][6]
	uint16_t * listA = sidx + kMaxRansacIters * 6;                           // [cap]
	uint16_t * listB = listA + cap;                                          // [cap]
	uint8_t * flag = reinterpret_cast<uint8_t *>(listB + cap);               // [cap]
	__shared__ LmState lm;
	__shared__ int s_best, s_nA, s_nB, s_ctrl, s_sizes[64];
	__shared__ float s_thr;
	// the pair's TO camera, loaded once per CTA from the pair table (or the call's parameters)
	__shared__ CamK s_cam;
	__shared__ int s_img_w, s_img_h, s_local;
	__shared__ float s_L[12];

	const int tid = threadIdx.x;
	const int pair = blockIdx.x;
	const int n = min(a.n_pts[pair], cap);
	const size_t base = static_cast<size_t>(pair) * cap;
	const int iterations = min(max(a.iterations, 1), kMaxRansacIters);
	const int min_inliers = max(a.min_inliers, 4);
#define PNP_PHASE(k) do { if (a.phase_clk && tid == 0) a.phase_clk[pair * 16 + (k)] = clock64(); } while (0)
	PNP_PHASE(0);

	if (tid < 3)
	{
		a.rvec[pair * 3 + tid] = 0;
		a.tvec[pair * 3 + tid] = 0;
	}
	if (tid < 12) a.transform[pair * 12 + tid] = 0.f;
	if (tid == 0)
	{
		a.n_inliers[pair] = 0;
		a.iters_run[pair] = 0;
		a.ok[pair] = 0;
	}
	if (a.cov6 && tid < 6) a.cov6[pair * 6 + tid] = 1.0; // *covariance = cv::Mat::eye(6,6,CV_64FC1) (:83)
	// util3d::estimateMotion3DTo2D runs PnP only with >= Vis/MinInliers correspondences; RANSAC needs >= 6
	if ((a.gate_min_matches && n < a.min_inliers) || n < 6) return;

	if (tid == 0)
	{
		const FrameCam * fc = a.cam_tab ? a.cam_tab + (a.cam_row ? a.cam_row[pair] : pair) : nullptr;
		if (fc && !fc->set) fc = nullptr;
		s_cam = fc ? CamK{fc->fx, fc->fy, fc->cx, fc->cy} : a.cam;
		s_img_w = fc ? fc->w : a.img_w;
		s_img_h = fc ? fc->h : a.img_h;
		s_local = fc ? fc->local : 0;
		if (fc)
			for (int k = 0; k < 12; ++k) s_L[k] = fc->L[k];
	}
	for (int i = tid; i < n * 3; i += blockDim.x) X[i] = a.obj[base * 3 + i];
	for (int i = tid; i < n * 2; i += blockDim.x) uv[i] = a.img[base * 2 + i];
	__syncthreads();
	PNP_PHASE(1);
	// each thread's copy of the camera, as the kernel always had (a reference to s_cam costs spills): the same registers and stack frame
	const CamK cam = s_cam;

	// ---- hypotheses in waves, one thread per hypothesis: EPnP on the sample, then the inlier counts; thread 0 then replays the
	//      sequential bookkeeping of RANSACPointSetRegistrator::run (solvepnp.cpp:358-399) and decides whether the run goes on.
	//      The adaptive iteration count of the reference usually ends the run within the first few hypotheses (a 90 % inlier ratio
	//      needs 7 iterations at 0.99 confidence), so the first wave solves only kPnpWave hypotheses: 16 EPnP threads finish much
	//      sooner than 128 (less stack-frame traffic, a shorter wait for the slowest hypothesis).  A run that goes past them (no good
	//      model yet) takes the rest in waves of up to kPnpWaveMax, every thread of the CTA, so that a full 300-iteration run is
	//      three waves (16, 256, 28), as many as the 128-hypothesis chunks it replaces.
	//      A wave's poses and counts use the h_rt and s_red areas; s_red is the refinement's and is not in use yet.
	double * w_rt = h_rt;                                                    // [kPnpWaveMax][6]
	int * w_cnt = reinterpret_cast<int *>(w_rt + kPnpWaveMax * 6);            // [kPnpWaveMax]
	static_assert(kPnpWaveMax * (6 * 8 + 4) <= (kPnpChunk * 6 + 28 * 32) * 8, "a wave's poses and counts must fit in h_rt + s_red");
	static_assert(kPnpWaveMax <= kVerifyThreads, "one thread per hypothesis of a wave");
	const float thr2 = static_cast<float>(static_cast<double>(a.reproj) * static_cast<double>(a.reproj));
	__shared__ int s_niters, s_maxgood, s_it;
	if (tid == 0)
	{
		s_best = -1;
		s_maxgood = 0;
		s_it = 0;
		s_niters = (n == 6) ? 1 : iterations;
	}
	__syncthreads();
	__shared__ unsigned long long s_rng;
	if (tid == 0) s_rng = 0xFFFFFFFFFFFFFFFFull;
	__syncthreads();
	for (int w0 = 0; w0 < s_niters;)
	{
		const int w1 = min(w0 + (w0 == 0 ? kPnpWave : kPnpWaveMax), s_niters);
		if (tid == 0 && n != 6)
		{
			// RANSACPointSetRegistrator::getSubset with cv::RNG((uint64)-1): the draws depend only on n and are
			// consumed in iteration order, so the samples of a wave are generated when the wave is reached
			unsigned long long state = s_rng;
			for (int it = w0; it < w1; ++it)
			{
				for (int i = 0; i < 6;)
				{
					int idx_i;
					for (;;)
					{
						idx_i = cv_rng_uniform(state, n);
						int j;
						for (j = 0; j < i; ++j)
							if (idx_i == sidx[it * 6 + j]) break;
						if (j == i) break;
					}
					sidx[it * 6 + i] = static_cast<uint16_t>(idx_i);
					++i;
				}
			}
			s_rng = state;
		}
		__syncthreads();
		// EPnP (the first wave runs on lanes 0..kPnpWave-1 of warp 0; spread over four warps it measured slower)
		if (tid < w1 - w0)
		{
			const int it = w0 + tid;
			int idx[6];
			for (int k = 0; k < 6; ++k) idx[k] = (n == 6) ? k : sidx[it * 6 + k];
			double rv[3], tv[3];
			long long * clk = (a.phase_clk && it == 0) ? a.phase_clk + pair * 16 + 8 : nullptr;
			int c = -1;
			if (solve_pnp_epnp6(X, uv, idx, cam, rv, tv, clk))
			{
				if (clk) clk[4] = clock64();
				c = 0;
				for (int k = 0; k < 3; ++k)
				{
					w_rt[tid * 6 + k] = rv[k];
					w_rt[tid * 6 + 3 + k] = tv[k];
				}
			}
			w_cnt[tid] = c;
		}
		__syncthreads();
		// Inlier counts + the bookkeeping in sub-chunks of kPnpWave hypotheses, so that the run can end inside a wave without counting
		// the rest of it.  Every hypothesis of a sub-chunk is counted by blockDim.x / size threads, each over a slice of the points.
		for (int s0 = w0; s0 < w1;)
		{
			const int s1 = min(s0 + kPnpWave, w1);
			const int nh = s1 - s0, parts = blockDim.x / nh;
			const int h = s0 - w0 + tid % nh, part = tid / nh; // h: index in the wave
			if (part < parts && w_cnt[h] >= 0)
			{
				double R[9];
				rodrigues_v2m(w_rt + h * 6, R, nullptr);
				const double tv[3] = {w_rt[h * 6 + 3], w_rt[h * 6 + 4], w_rt[h * 6 + 5]};
				const int i0 = static_cast<int>(static_cast<long long>(n) * part / parts), i1 = static_cast<int>(static_cast<long long>(n) * (part + 1) / parts);
				int c = 0;
				int i = i0;
				for (; i + 4 <= i1; i += 4)
				{
					// four independent points per trip: the fp64 divide and square root of each projection are long dependent
					// chains, and a warp here has at most one neighbour on its scheduler to hide them
					const float e0 = reproj_err(R, tv, cam, X + 3 * i, uv + 2 * i);
					const float e1 = reproj_err(R, tv, cam, X + 3 * i + 3, uv + 2 * i + 2);
					const float e2 = reproj_err(R, tv, cam, X + 3 * i + 6, uv + 2 * i + 4);
					const float e3 = reproj_err(R, tv, cam, X + 3 * i + 9, uv + 2 * i + 6);
					c += (e0 <= thr2 ? 1 : 0) + (e1 <= thr2 ? 1 : 0) + (e2 <= thr2 ? 1 : 0) + (e3 <= thr2 ? 1 : 0);
				}
				for (; i < i1; ++i) c += reproj_err(R, tv, cam, X + 3 * i, uv + 2 * i) <= thr2 ? 1 : 0;
				if (c) atomicAdd(&w_cnt[h], c);
			}
			if (a.phase_clk && tid == 0 && s0 == 0) a.phase_clk[pair * 16 + 8 + 5] = clock64();
			__syncthreads();
			if (tid == 0)
			{
				int it0 = s_it, niters = s_niters, maxGood = s_maxgood;
				if (n == 6)
				{
					if (w_cnt[0] >= 0)
					{
						s_best = 0;
						for (int k = 0; k < 6; ++k) lm.param[k] = w_rt[k];
					}
					it0 = 0;
				}
				else
				{
					for (; it0 < niters && it0 < s1; ++it0)
					{
						const int c = w_cnt[it0 - w0];
						if (c < 0) continue;
						if (c > max(maxGood, 5))
						{
							s_best = it0;
							maxGood = c;
							for (int k = 0; k < 6; ++k) lm.param[k] = w_rt[(it0 - w0) * 6 + k];
							niters = ransac_update_num_iters(0.99, static_cast<double>(n - c) / n, 6, niters);
						}
					}
				}
				s_it = it0;
				s_niters = niters;
				s_maxgood = maxGood;
			}
			__syncthreads();
			if (s_niters <= s1) break; // the run ended inside this sub-chunk (uniform: shared state read after the barrier)
			s0 = s1;
		}
		if (w0 == 0) PNP_PHASE(5);
		if (w0 == 0 ? s_niters <= w1 : w0 == kPnpWave) PNP_PHASE(2); // end of the first two waves
		w0 = w1;
	}
	const int best = s_best;
	PNP_PHASE(3);
	if (tid == 0) a.iters_run[pair] = s_it;
	if (best < 0) return; // rvec/tvec keep the (identity) guess

	// ---- inliers of the best minimal-sample model ----------------------------------------------
	if (tid == 0) rodrigues_v2m(lm.param, lm.R, nullptr);
	__syncthreads();
	for (int i = tid; i < n; i += blockDim.x)
		flag[i] = (n == 6) ? 1 : (reproj_err(lm.R, lm.param + 3, cam, X + 3 * i, uv + 2 * i) <= thr2 ? 1 : 0);
	__syncthreads();
	if (tid < 32)
	{
		const int c = warp0_compact(flag, n, listA, listB /* scratch ranks */);
		if (tid == 0) s_nA = c;
	}
	__syncthreads();
	// listA = inliers (RANSAC).  From here on: prev = listA / new = listB as in util3d::solvePnPRansac.
	uint16_t * prev = listA;
	uint16_t * nw = listB;
	int n_prev = s_nA, n_new = 0;
	uint16_t * fin = prev; // list that ends up in `inliers`
	int n_fin = n_prev;

	if (n_prev >= min_inliers && a.refine_iterations > 0)
	{
		if (tid == 0)
		{
			s_thr = a.reproj;
			s_ctrl = 0;
		}
		int refine_it = 0, n_sizes = 0;
		bool inlier_changed = false;
		__syncthreads();
		for (;;) // do { ... } while (inlier_changed && ++refine_it < refineIterations)
		{
			bool leave = false;
			lm_refine_block(X, uv, prev, n_prev, cam, lm, s_red, s_out);
			if (tid == 0 && n_sizes < 64) s_sizes[n_sizes] = n_prev;
			++n_sizes;
			// computeReprojErrors under the refined model, threshold NOT squared (util3d_motion_estimation.cpp:829-837)
			if (tid == 0) rodrigues_v2m(lm.param, lm.R, nullptr);
			__syncthreads();
			const float thr = s_thr;
			for (int i = tid; i < n; i += blockDim.x)
			{
				const float e = reproj_err(lm.R, lm.param + 3, cam, X + 3 * i, uv + 2 * i);
				errs[i] = e;
				flag[i] = e <= thr ? 1 : 0;
			}
			__syncthreads();
			if (tid < 32)
			{
				const int lane = tid;
				int basec = 0;
				for (int c0 = 0; c0 < n; c0 += 32)
				{
					const int i = c0 + lane;
					const bool f = i < n && flag[i] != 0;
					const uint32_t mk = __ballot_sync(0xFFFFFFFFu, f);
					if (f) nw[basec + __popc(mk & ((1u << lane) - 1u))] = static_cast<uint16_t>(i);
					basec += __popc(mk);
				}
				if (lane == 0) s_nB = basec;
			}
			__syncthreads();
			n_new = s_nB;
			if (n_new < min_inliers)
			{
				// "continue" of a do-while: falls to the loop condition with inlier_changed unchanged
				++refine_it;
				if (refine_it >= a.refine_iterations) leave = true;
			}
			else
			{
				if (tid == 0)
				{
					// uMean / uVariance over the new inliers' errors, sequential float arithmetic (UMath.h:419-431, :512-526)
					float mean = 0.f;
					for (int k = 0; k < n_new; ++k) mean += errs[nw[k]];
					mean /= static_cast<float>(n_new);
					float variance = 0.f;
					if (n_new > 1)
					{
						float sum = 0.f;
						for (int k = 0; k < n_new; ++k) sum += (errs[nw[k]] - mean) * (errs[nw[k]] - mean);
						variance = sum / static_cast<float>(n_new - 1);
					}
					s_thr = fminf(a.reproj, a.refine_sigma * static_cast<float>(sqrt(static_cast<double>(variance))));
					int changed = 0;
					if (n_new != n_prev) changed = 1;
					else
						for (int k = 0; k < n_new; ++k)
							if (prev[k] != nw[k])
							{
								changed = 1;
								break;
							}
					s_ctrl = changed;
				}
				__syncthreads();
				// std::swap(prev_inliers, new_inliers)
				{
					uint16_t * t = prev;
					prev = nw;
					nw = t;
					const int tn = n_prev;
					n_prev = n_new;
					n_new = tn;
				}
				inlier_changed = s_ctrl != 0;
				if (n_new != n_prev && n_sizes >= min_inliers && n_sizes >= 4 && n_sizes <= 64 &&
				    s_sizes[n_sizes - 1] == s_sizes[n_sizes - 3] && s_sizes[n_sizes - 2] == s_sizes[n_sizes - 4])
					leave = true; // oscillating
				__syncthreads();
			}
			if (leave) break;
			if (!(inlier_changed && ++refine_it < a.refine_iterations)) break;
		}
		// std::swap(inliers, new_inliers); rvec/tvec = refined model
		fin = nw;
		n_fin = n_new;
	}
	__syncthreads();
	PNP_PHASE(4);

	if (tid < 3)
	{
		a.rvec[pair * 3 + tid] = lm.param[tid];
		a.tvec[pair * 3 + tid] = lm.param[3 + tid];
	}
	for (int k = tid; k < n_fin; k += blockDim.x) a.inliers[base + k] = fin[k];
	// transform = (localTransform * pnp)^-1, transformCameraFrame = transform * localTransform and its inverse, 3x4 float; with an identity
	// local transform the last two are transform and pnp itself
	__shared__ float s_T[12], s_C[12], s_P[12];
	__shared__ int s_acc;
	__shared__ double s_med[5];
	if (tid == 0)
	{
		a.n_inliers[pair] = n_fin;
		const int accepted = n_fin >= a.min_inliers ? 1 : 0;
		s_acc = accepted;
		if (accepted)
		{
			double R[9];
			rodrigues_v2m(lm.param, R, nullptr);
			float Rf[9], tf[3];
			for (int i = 0; i < 9; ++i) Rf[i] = static_cast<float>(R[i]);
			for (int i = 0; i < 3; ++i) tf[i] = static_cast<float>(lm.param[3 + i]);
			for (int i = 0; i < 3; ++i)
			{
				for (int j = 0; j < 3; ++j)
				{
					s_T[4 * i + j] = Rf[3 * j + i];
					s_P[4 * i + j] = Rf[3 * i + j];
				}
				s_T[4 * i + 3] = -(Rf[0 + i] * tf[0] + Rf[3 + i] * tf[1] + Rf[6 + i] * tf[2]);
				s_P[4 * i + 3] = tf[i];
			}
			if (s_local)
			{
				transform_mul_f(s_L, s_P, s_C); // localTransform * pnp, in s_C until the last two steps
				transform_inv_f(s_C, s_T);
				transform_mul_f(s_T, s_L, s_C);
				transform_inv_f(s_C, s_P);
			}
			else
				for (int k = 0; k < 12; ++k) s_C[k] = s_T[k];
		}
	}
	__syncthreads();
	int accepted = s_acc;
	if (accepted && a.cov6)
	{
		// ---- covariance (util3d_motion_estimation.cpp:156-258) --------------------
		const bool have3B = a.obj_to != nullptr;
		if (have3B || s_img_w != 0 || s_img_h != 0)
		{
			// channels: 0 squared 3-D distance, 1 angle (pcl::getAngle3D), 2..4 squared x / y / z error (split components)
			const int n_ch = a.split_linear ? 5 : 2;
			const int kth = n_fin / max(a.var_median_ratio, 2);
			for (int ch = 0; ch < n_ch; ++ch)
			{
				for (int k = tid; k < n_fin; k += blockDim.x)
				{
					const int i = fin[k];
					const float ox = X[3 * i], oy = X[3 * i + 1], oz = X[3 * i + 2];
					float nx, ny, nz;
					bool from3B = false;
					if (have3B)
					{
						const float * p = a.obj_to + (base + i) * 3;
						if (isfinite(p[0]) && isfinite(p[1]) && isfinite(p[2]))
						{
							// util3d::transformPoint(words3B, transform) (util3d_transforms.cpp:211-220), float, left to right
							nx = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(s_T[0], p[0]), __fmul_rn(s_T[1], p[1])), __fmul_rn(s_T[2], p[2])), s_T[3]);
							ny = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(s_T[4], p[0]), __fmul_rn(s_T[5], p[1])), __fmul_rn(s_T[6], p[2])), s_T[7]);
							nz = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(s_T[8], p[0]), __fmul_rn(s_T[9], p[1])), __fmul_rn(s_T[10], p[2])), s_T[11]);
							from3B = true;
						}
					}
					if (!from3B)
					{
						// depth of the object point in camera B, ray through the image point, 10 % error (:186-203)
						const float zc = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(s_P[8], ox), __fmul_rn(s_P[9], oy)), __fmul_rn(s_P[10], oz)), s_P[11]);
						const float fx = static_cast<float>(cam.fu), fy = static_cast<float>(cam.fv);
						float cx = static_cast<float>(cam.uc), cy = static_cast<float>(cam.vc);
						cx = cx > 0.0f ? cx : static_cast<float>(s_img_w / 2) - 0.5f;
						cy = cy > 0.0f ? cy : static_cast<float>(s_img_h / 2) - 0.5f;
						const float rx = __fdiv_rn(__fsub_rn(uv[2 * i], cx), fx), ry = __fdiv_rn(__fsub_rn(uv[2 * i + 1], cy), fy);
						// cv::Point3f * (float * double): the scale is a double product converted back to float per component
						const double sc = static_cast<double>(zc) * 1.1;
						const float px = static_cast<float>(static_cast<double>(rx) * sc), py = static_cast<float>(static_cast<double>(ry) * sc),
						            pz = static_cast<float>(sc);
						nx = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(s_C[0], px), __fmul_rn(s_C[1], py)), __fmul_rn(s_C[2], pz)), s_C[3]);
						ny = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(s_C[4], px), __fmul_rn(s_C[5], py)), __fmul_rn(s_C[6], pz)), s_C[7]);
						nz = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(s_C[8], px), __fmul_rn(s_C[9], py)), __fmul_rn(s_C[10], pz)), s_C[11]);
					}
					const float dx = __fsub_rn(ox, nx), dy = __fsub_rn(oy, ny), dz = __fsub_rn(oz, nz);
					float v;
					if (ch == 0) v = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
					else if (ch == 1)
					{
						// pcl::getAngle3D(v1, v2): acos of the clamped dot product of the normalised vectors (Eigen::Vector4f, w = 0)
						const float n1 = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(ox, ox), __fmul_rn(oz, oz)), __fmul_rn(oy, oy)));
						const float n2 = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(nx, nx), __fmul_rn(nz, nz)), __fmul_rn(ny, ny)));
						const float ax = __fdiv_rn(ox, n1), ay = __fdiv_rn(oy, n1), az = __fdiv_rn(oz, n1);
						const float bx = __fdiv_rn(nx, n2), by = __fdiv_rn(ny, n2), bz = __fdiv_rn(nz, n2);
						double rad = static_cast<double>(__fadd_rn(__fadd_rn(__fmul_rn(ax, bx), __fmul_rn(az, bz)), __fmul_rn(ay, by)));
						rad = rad < -1.0 ? -1.0 : (rad > 1.0 ? 1.0 : rad);
						v = static_cast<float>(acos(rad));
					}
					else
					{
						const double e = static_cast<double>(ch == 2 ? dx : (ch == 3 ? dy : dz));
						v = static_cast<float>(e * e);
					}
					cbuf[k] = v;
				}
				__syncthreads();
				// the element std::sort would leave at index kth: rank by (value, position)
				for (int k = tid; k < n_fin; k += blockDim.x)
				{
					const float v = cbuf[k];
					int r = 0;
					for (int j = 0; j < n_fin; ++j)
					{
						const float w = cbuf[j];
						r += (w < v || (w == v && j < k)) ? 1 : 0;
					}
					if (r == kth) s_med[ch] = 2.1981 * static_cast<double>(v);
				}
				__syncthreads();
			}
			if (tid == 0)
			{
				double lin = s_med[0];
				double d[6] = {lin, lin, lin, s_med[1], s_med[1], s_med[1]};
				if (a.split_linear)
				{
					d[0] = s_med[2];
					d[1] = s_med[3];
					d[2] = s_med[4];
					lin = fmax(fmax(s_med[2], s_med[3]), s_med[4]);
				}
				if (a.max_variance > 0.f && lin > static_cast<double>(a.max_variance))
				{
					// "Rejected PnP transform, variance is too high": covariance back to identity, transform null (:246-251)
					for (int k = 0; k < 6; ++k) d[k] = 1.0;
					s_acc = 0;
				}
				for (int k = 0; k < 6; ++k) a.cov6[pair * 6 + k] = d[k];
			}
		}
		else
		{
			// no 3-D points of B and no image size: covariance *= sqrt(mean squared reprojection error of the inliers) (:253-266);
			// cv::projectPoints with the final pose, K and no distortion; float accumulation in inlier order
			if (tid == 0) rodrigues_v2m(lm.param, lm.R, nullptr);
			__syncthreads();
			for (int k = tid; k < n_fin; k += blockDim.x)
			{
				const int i = fin[k];
				double pu, pv;
				project_point(lm.R, lm.param + 3, cam, X + 3 * i, pu, pv);
				const float ex = __fsub_rn(uv[2 * i], static_cast<float>(pu)), ey = __fsub_rn(uv[2 * i + 1], static_cast<float>(pv));
				cbuf[k] = __fadd_rn(__fmul_rn(ex, ex), __fmul_rn(ey, ey));
			}
			__syncthreads();
			if (tid == 0)
			{
				float err = 0.0f;
				for (int k = 0; k < n_fin; ++k) err = __fadd_rn(err, cbuf[k]);
				const double sc = static_cast<double>(sqrtf(__fdiv_rn(err, static_cast<float>(n_fin))));
				for (int k = 0; k < 6; ++k) a.cov6[pair * 6 + k] = sc;
			}
		}
		__syncthreads();
		accepted = s_acc;
	}
	if (tid == 0) a.ok[pair] = accepted;
	if (accepted && tid < 12) a.transform[pair * 12 + tid] = s_T[tid];
}

// Pack the per-pair verification outputs into lcd_verify_result records (one device->host copy instead of seven).
struct PackedVerifyResult // layout of lcd_verify_result (include/lcd_b200.h)
{
	int ok, n_matches, n_inliers, iterations_run;
	double rvec[3], tvec[3];
	float transform[12];
	double covariance[36];
};
__global__ void pack_verify_results_kernel(int n_pairs, const int * __restrict__ ok, const int * __restrict__ n_match, const int * __restrict__ n_inl,
                                           const int * __restrict__ iters, const double * __restrict__ rvec, const double * __restrict__ tvec,
                                           const float * __restrict__ T, const double * __restrict__ cov6, PackedVerifyResult * __restrict__ out)
{
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n_pairs) return;
	PackedVerifyResult r;
	r.ok = ok[i];
	r.n_matches = n_match[i];
	r.n_inliers = n_inl[i];
	r.iterations_run = iters[i];
	for (int k = 0; k < 3; ++k)
	{
		r.rvec[k] = rvec[3 * i + k];
		r.tvec[k] = tvec[3 * i + k];
	}
	for (int k = 0; k < 12; ++k) r.transform[k] = T[12 * i + k];
	for (int k = 0; k < 36; ++k) r.covariance[k] = 0.0;
	for (int k = 0; k < 6; ++k)
	{
		// Registration::computeTransformationMod floors the diagonal (COVARIANCE_LINEAR / ANGULAR_EPSILON, Registration.cpp:36-37, :239-250)
		const double floor_v = k < 3 ? 0.00000001 : 0.00000003;
		const double c = cov6 ? cov6[6 * i + k] : 1.0;
		r.covariance[7 * k] = c <= floor_v ? floor_v : c;
	}
	out[i] = r;
}

// Hypothesis selection for the fused query: the signature with the highest likelihood of each frame
// (first maximum; a zero / negative maximum selects nothing).  The reference selects through the Bayes
// filter (Rtabmap.cpp:2133-2226, out of scope here, SURVEY.md §8(f)); the raw-likelihood arg-max is what
// the benchmark verifies.  hyp_id[frame] = signature id or 0, hyp_slot[frame] = row of the signature store or -1.
__global__ void argmax_hypothesis_kernel(const float * __restrict__ like, int ns, const int * __restrict__ sig_ids,
                                         const int * __restrict__ sig_slot, int slot_cap, int * __restrict__ hyp_id, int * __restrict__ hyp_slot)
{
	__shared__ float s_v[32];
	__shared__ int s_i[32];
	const int frame = blockIdx.x;
	const float * row = like + static_cast<size_t>(frame) * ns;
	float bv = -1.0f;
	int bi = 0x7FFFFFFF;
	for (int k = threadIdx.x; k < ns; k += blockDim.x)
	{
		const float v = row[k];
		if (v > bv || (v == bv && k < bi))
		{
			bv = v;
			bi = k;
		}
	}
	for (int o = 16; o > 0; o >>= 1)
	{
		const float ov = __shfl_down_sync(0xFFFFFFFFu, bv, o);
		const int oi = __shfl_down_sync(0xFFFFFFFFu, bi, o);
		if (ov > bv || (ov == bv && oi < bi))
		{
			bv = ov;
			bi = oi;
		}
	}
	if ((threadIdx.x & 31) == 0)
	{
		s_v[threadIdx.x >> 5] = bv;
		s_i[threadIdx.x >> 5] = bi;
	}
	__syncthreads();
	if (threadIdx.x == 0)
	{
		for (int w = 1; w < (blockDim.x >> 5); ++w)
			if (s_v[w] > bv || (s_v[w] == bv && s_i[w] < bi))
			{
				bv = s_v[w];
				bi = s_i[w];
			}
		int id = 0, slot = -1;
		if (bv > 0.0f && bi < ns)
		{
			id = sig_ids[bi];
			if (id > 0 && id < slot_cap) slot = sig_slot[id];
		}
		hyp_id[frame] = id;
		hyp_slot[frame] = slot;
	}
}

// out[pair][k] = values[pair][index[pair][k]] for k < count[pair]  (inlier word ids = matches[inliers[k]])
__global__ void gather_by_index_kernel(const int * __restrict__ values, const int * __restrict__ index, const int * __restrict__ count,
                                       int cap, int * __restrict__ out)
{
	const int k = blockIdx.x * blockDim.x + threadIdx.x;
	const int pair = blockIdx.y;
	if (k >= cap) return;
	const size_t base = static_cast<size_t>(pair) * cap;
	out[base + k] = k < count[pair] ? values[base + index[base + k]] : 0;
}

} // namespace lcd
