// nn_tensor_f32.cuh — exact squared-L2 2-NN of FLOAT descriptors (SURF-64 / SIFT-128 sized rows) with the distance matrix on the
// Hopper tensor cores (sm_90a, wgmma): BASELINE configs[3], "tensor cores ... if SURF/float descriptors make it a true dense GEMM".
//
// Replaces, for CV_32F descriptors: FlannIndex::knnSearch(k = 2) on a LinearIndex (corelib/src/FlannIndex.cpp:701-745 ->
// rtflann::L2<float>::operator(), rtflann/algorithms/dist.h:133-180, KNNSimpleResultSet, rtflann/util/result_set.h:151-172), whose
// result — ids AND fp32 distances in rtflann's summation order — must be reproduced bit for bit.  A tensor-core GEMM cannot reproduce
// an fp32 summation order, so it is used as a FILTER with a proven bound, followed by an exact re-rank:
//
//   1. operands rounded to fp16 (round to nearest, no scaling; |x| < 65504 is checked) in pre-tiled, 128-byte-swizzled K-major
//      images: the word image is built once per dictionary change and CACHED (half the bytes of the fp32 rows: the 1M x 64
//      vocabulary streams as 128 MB), the query image per call;
//   2. knn2_tensor_f32_kernel: wgmma .f32.f16.f16 (M64 N256 K16 per warpgroup, fp32 accumulators in registers).  The word image holds -2 w and one
//      extra K-step holds |w|^2 (as an fp16 hi + lo pair against a constant column of the query image), so the accumulator IS
//      v = |w|^2 - 2 q.w (= approximate squared distance minus |q|^2): the epilogue is a running minimum over the columns
//      and appends to the query's CANDIDATE LIST every row with v <= t2 + 2 eps, where t2 is the
//      second-smallest v this thread has seen so far (initialised from a shared per-query bound);
//   3. rerank_l2_kernel computes the exact rtflann-order distance of every candidate from the fp32 rows and keeps the best two by
//      (distance, row) — the same packed 64-bit keys as the exact kernel of l2_path.cuh, consumed by the same resolve kernel;
//   4. a query whose list overflowed (or whose values do not fit fp16) is redone by an exact scan (knn2_l2_fallback_kernel).
//
// Why the filter cannot lose a true neighbour.  Let d(w) be the distance rtflann computes, e1, e2 the true two nearest rows, and
// |v(w) + |q|^2 - d(w)| <= eps for every row w.  t2 is always the larger of the v's of two DISTINCT rows, hence
// t2 + |q|^2 >= d(e2) - eps; and v(e_i) + |q|^2 <= d(e_i) + eps <= d(e2) + eps.  So v(e_i) <= t2 + 2 eps whenever e_i is examined:
// both true neighbours (and every row tying with them) reach the list, and the exact re-rank then orders them as rtflann does.
// eps bounds (a) fp16 rounding of both operands: |q^.w^ - q.w| <= 2^-10 (1 + 2^-11) |q| |w| + subnormal terms (Cauchy-Schwarz on the
// element-wise relative errors 2^-11), doubled by the factor 2 in the distance; (b) fp32 accumulation in the tensor core, the fma
// the fp16 hi + lo split of |w|^2 (relative 2^-21, plus 2^-19 absolute for its subnormal tail), the float norms and rtflann's own
// rounding, all far below 2^-15 (|q|^2 + |w|^2) + 4e-6:
//     eps(q) = 1.02 * 2^-9 * |q| * Wmax + 2^-15 * (|q|^2 + Wmax^2) + 4e-6,      Wmax = largest |w| in the dictionary.
// For unit-length descriptors eps ~ 2.1e-3 against nearest-neighbour distances of 1e-2 .. 1: the lists stay a few dozen rows long.
//
// D = 256 (SuperPoint).  Term (a) does not depend on D.  The terms of (b) grow with the length of the sums, and at 256 the lumped
// 2^-15 is no longer shown to cover them, so 256 has its own constant (64 and 128 keep theirs: lcd_nn_f32_stats counts are observable).
// Model: each of the K = 256 + 16 = 272 products of the tensor core's chain enters the fp32 accumulator with at most one rounding of
// relative 2^-23 (truncation allowed) of a partial sum bounded by the sum of the terms' magnitudes, sum |2 q_i w_i| + |w|^2
// <= 2 |q| Wmax + Wmax^2 (fp16 products are exact in fp32).  So the accumulation error is at most
//     271 * 2^-23 * (2 |q| Wmax + Wmax^2) <= 6.5e-5 |q| Wmax + 3.3e-5 Wmax^2.
// rtflann sums 4 squares per group and 64 groups: its distance d <= (|q| + Wmax)^2 carries at most 67 * 2^-24 * d <= 4.0e-6 (|q|^2 + Wmax^2)
// + 8.0e-6 |q| Wmax.  The fp32 norm |w|^2 (67 * 2^-24 relative) and its hi + lo split (2^-22 relative) add 4.3e-6 Wmax^2.  In total
// 7.3e-5 |q| Wmax + 4.2e-5 Wmax^2 + 4.0e-6 |q|^2, which the 256 constant covers with room for the subnormal terms:
//     eps256(q) = (1.02 * 2^-9 + 2^-13) * |q| * Wmax + 2^-14 * (|q|^2 + Wmax^2) + 4e-6          (2^-13 = 1.2e-4, 2^-14 = 6.1e-5)
// For unit-length rows eps256 ~ 2.24e-3 against 2.06e-3 with the 64 / 128 constant.
//
// Tiling at D = 256.  A 256-word tile is 128 KB of fp16, so two whole tiles per stage no longer fit: 64 KB query tile + 4 KB query slab
// + 2 x (128 KB + 8 KB) = 340 KB against the H100's 227 KB per block.  The word tile is streamed in K slices instead: the image is
// [tile][atom][rows][128 B], so one 128-byte swizzle atom (64 halves) of all 256 rows is one contiguous 32 KB bulk copy, and a ring of
// 4 such stages holds one whole tile: 1 KB (alignment) + 64 KB + 4 KB + 4 x 32 KB + 8 KB word slab (with the last slice) + 512 B of
// barriers = 205.5 KB.  The accumulators carry over the four slices of a tile; a stage is released as soon as the MMAs of the next
// slice are issued and its own have completed, so the slices of the next tile stream in under the current tile's MMAs and epilogue.
// The N = 256 epilogue is the one of 64 / 128.
#pragma once
#include "common.cuh"
#include "l2_path.cuh"
#include "nn_tensor.cuh"
#include <cuda_fp16.h>

namespace lcd {

constexpr int kTfBM = 128;          // queries per CTA tile (two consumer warpgroups of M64)
constexpr int kTfBN = 256;          // words per tile (wgmma N)
constexpr int kTfThreads = 384;     // producer warpgroup + two consumer warpgroups
constexpr int kTfCandCap = 96;      // candidate rows kept per query; more -> exact fallback for that query
constexpr int kTfMinRows = 4096;    // below this the exact CUDA-core kernel is used
constexpr int kTfPrepassTiles = 16; // rows [0, 4096): the bound-only pre-pass that initialises the per-query bound
constexpr float kTfAugScale = 64.0f; // the constant of the query image's augmentation columns; |w|^2 is stored divided by it
constexpr float kTfMaxAbs = 32752.0f; // -2 w must fit fp16
constexpr float kTfMaxNorm2 = 65504.0f * kTfAugScale;

template <int DIM>
struct TfCfg
{
	static constexpr int atoms = DIM / 64;                 // 64 halves = one 128-byte swizzle atom
	static constexpr uint32_t a_bytes = kTfBM * DIM * 2;
	static constexpr uint32_t b_bytes = kTfBN * DIM * 2;
	static constexpr uint32_t a_aug_bytes = kTfBM * 32;    // one K-step (16 halves) per row, un-swizzled core-matrix layout
	static constexpr uint32_t b_aug_bytes = kTfBN * 32;
	// 64 / 128: a stage holds a whole word tile and its augmentation slab.  256: a word tile is 128 KB, so a stage holds one K slice
	// (one swizzle atom of all 256 rows, 32 KB, contiguous in the image) and the tile's slab sits beside the ring, written with the last
	// slice; stages == slices, so slice k of every tile lands in stage k and the slab is covered by the last stage's barriers.
	static constexpr int slices = DIM == 256 ? atoms : 1;
	static constexpr uint32_t slice_bytes = b_bytes / slices;
	static constexpr int stages = DIM == 64 ? 5 : DIM == 128 ? 2 : slices;
	static constexpr uint32_t stage_bytes = slices == 1 ? b_bytes + b_aug_bytes : slice_bytes;
	static constexpr uint32_t ring_bytes = stages * stage_bytes + (slices == 1 ? 0 : b_aug_bytes);
	static constexpr size_t smem = 1024 + a_bytes + a_aug_bytes + ring_bytes + 512;
	static_assert(slices == 1 || stages == slices, "the augmentation slab travels with the last stage");
};

// dynamic shared memory of the filter kernel at a descriptor width (0: the width has no filter)
inline size_t tf_smem_bytes(int dim)
{
	return dim == 64 ? TfCfg<64>::smem : dim == 128 ? TfCfg<128>::smem : dim == 256 ? TfCfg<256>::smem : 0;
}

// order-preserving float <-> uint mapping (v can be negative), for atomicMin on the shared per-query bound
__device__ __forceinline__ uint32_t f2ord(float f)
{
	const uint32_t b = __float_as_uint(f);
	return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float ord2f(uint32_t u)
{
	return __uint_as_float((u & 0x80000000u) ? (u & 0x7FFFFFFFu) : ~u);
}

// ---- operand images ----------------------------------------------------------------------------------------------
// One thread converts 8 consecutive floats of a row into one 16-byte chunk.  Rows >= n_rows of the last tile are zero.
// Layout: [tile][atom][tile_rows][128 B], chunk c of row r at c ^ (r & 7) (canonical K-major SWIZZLE_128B).
// bad_row[row] (may be null) is set when a value is not finite or does not fit fp16.
template <int DIM>
__global__ void tf_expand_kernel(const float * __restrict__ src, int row_begin, int n_rows, int tile_rows, uint4 * __restrict__ dst,
                                 int * __restrict__ bad_flag, float scale)
{
	constexpr int chunks = DIM / 8;
	const size_t gid = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
	const int tile0 = row_begin / tile_rows;
	const size_t row = static_cast<size_t>(tile0) * tile_rows + gid / chunks;
	const int chunk = static_cast<int>(gid % chunks);
	const size_t row_end = (static_cast<size_t>(n_rows) + tile_rows - 1) / tile_rows * tile_rows;
	if (row >= row_end) return;
	uint4 o = make_uint4(0, 0, 0, 0);
	if (row < static_cast<size_t>(n_rows))
	{
		const float4 a = *reinterpret_cast<const float4 *>(src + row * DIM + chunk * 8);
		const float4 b = *reinterpret_cast<const float4 *>(src + row * DIM + chunk * 8 + 4);
		const float m = fmaxf(fmaxf(fmaxf(fabsf(a.x), fabsf(a.y)), fmaxf(fabsf(a.z), fabsf(a.w))),
		                      fmaxf(fmaxf(fabsf(b.x), fabsf(b.y)), fmaxf(fabsf(b.z), fabsf(b.w))));
		if (!(m < kTfMaxAbs) && bad_flag) *bad_flag = 1; // also true for NaN
		// scale = -2 for the word image (exact in fp16), 1 for the query image
		const __half2 h0 = __floats2half2_rn(a.x * scale, a.y * scale), h1 = __floats2half2_rn(a.z * scale, a.w * scale),
		              h2 = __floats2half2_rn(b.x * scale, b.y * scale), h3 = __floats2half2_rn(b.z * scale, b.w * scale);
		o.x = *reinterpret_cast<const uint32_t *>(&h0);
		o.y = *reinterpret_cast<const uint32_t *>(&h1);
		o.z = *reinterpret_cast<const uint32_t *>(&h2);
		o.w = *reinterpret_cast<const uint32_t *>(&h3);
	}
	const int tile = static_cast<int>(row / tile_rows), r = static_cast<int>(row % tile_rows);
	const int atom = chunk >> 3, c = chunk & 7;
	const size_t off16 = static_cast<size_t>(tile) * (static_cast<size_t>(tile_rows) * chunks) + static_cast<size_t>(atom) * (tile_rows * 8) +
	                     static_cast<size_t>(r) * 8 + static_cast<size_t>(c ^ (r & 7));
	dst[off16] = o;
}

// The augmentation K-step of rows [row_begin rounded down to a tile, n_rows rounded up): 16 halves per row in the un-swizzled K-major
// core-matrix layout ([8-row group][k-chunk 0..1][8 rows][8 halves], 256 B per group), image = [tile][tile_rows / 8 groups].
//   words  : (hi, lo, 0...) with hi + lo = |w|^2 / kTfAugScale (+inf in the padding rows); the largest |w|^2 into *wmax2_bits
//   queries: (kTfAugScale, kTfAugScale, 0...)
template <int DIM>
__global__ void tf_aug_kernel(const float * __restrict__ src, int row_begin, int n_rows, int tile_rows, uint4 * __restrict__ aug, int is_query,
                              uint32_t * __restrict__ wmax2_bits, int * __restrict__ bad_flag)
{
	const size_t row = static_cast<size_t>(row_begin / tile_rows) * tile_rows + static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
	const size_t row_end = (static_cast<size_t>(n_rows) + tile_rows - 1) / tile_rows * tile_rows;
	if (row >= row_end) return;
	__half h0, h1;
	if (is_query)
	{
		h0 = __float2half_rn(kTfAugScale);
		h1 = h0;
	}
	else
	{
		float s = INFINITY;
		if (row < static_cast<size_t>(n_rows))
		{
			s = 0.0f;
			for (int i = 0; i < DIM; i += 4)
			{
				const float4 a = *reinterpret_cast<const float4 *>(src + row * DIM + i);
				s += a.x * a.x + a.y * a.y + a.z * a.z + a.w * a.w;
			}
			if (!(s < kTfMaxNorm2) && bad_flag) *bad_flag = 1;
			if (wmax2_bits && s == s) atomicMax(wmax2_bits, __float_as_uint(s)); // s >= 0: unsigned order of the bits = float order
		}
		const float t = s / kTfAugScale;
		h0 = __float2half_rn(t);
		h1 = (t < INFINITY) ? __float2half_rn(t - __half2float(h0)) : __float2half_rn(0.0f);
	}
	// row r of the image: group r / 8, core-matrix row r % 8; k-chunk 0 holds halves 0..7 (hi, lo, 0 x 6), k-chunk 1 is zero
	const size_t grp = row / 8;
	const int rr = static_cast<int>(row % 8);
	uint4 c0 = make_uint4(0, 0, 0, 0);
	c0.x = static_cast<uint32_t>(__half_as_ushort(h0)) | (static_cast<uint32_t>(__half_as_ushort(h1)) << 16);
	aug[grp * 16 + rr] = c0;
	aug[grp * 16 + 8 + rr] = make_uint4(0, 0, 0, 0);
}

// per-query state of one search: norm, empty candidate list (or "overflowed" for queries that do not fit fp16), loose bound
template <int DIM>
__global__ void tf_query_init_kernel(const float * __restrict__ q, int nq, float * __restrict__ qn, int * __restrict__ cand_count,
                                     uint32_t * __restrict__ tau)
{
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= nq) return;
	float s = 0.0f, m = 0.0f;
	for (int k = 0; k < DIM; k += 4)
	{
		const float4 a = *reinterpret_cast<const float4 *>(q + static_cast<size_t>(i) * DIM + k);
		s += a.x * a.x + a.y * a.y + a.z * a.z + a.w * a.w;
		m = fmaxf(m, fmaxf(fmaxf(fabsf(a.x), fabsf(a.y)), fmaxf(fabsf(a.z), fabsf(a.w))));
	}
	const bool ok = (m < 65504.0f) && (s == s) && (s < INFINITY);
	qn[i] = ok ? s : 0.0f;
	cand_count[i] = ok ? 0 : (kTfCandCap + 1);
	tau[i] = 0xFF800000u; // f2ord(+inf): no bound yet
}

// D[regs] (+)= A[smem] * B[smem]^T, f16 x f16 -> f32, M64 x N256 x K16 over one warpgroup (same fragment layout as wg_mma_b1)
__device__ __forceinline__ void wg_mma_f16(float (&d)[128], uint64_t adesc, uint64_t bdesc, uint32_t accumulate)
{
	asm volatile(
		"{\n"
		".reg .pred p;\n"
		"setp.ne.b32 p, %130, 0;\n"
		"wgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 "
		"{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
		"%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
		"%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
		"%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
		"%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "
		"%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, "
		"%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, "
		"%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, "
		"%128, %129, p, 1, 1, 0, 0;\n"
		"}\n"
		: "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
		  "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
		  "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
		  "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
		  "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
		  "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
		  "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
		  "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
		  "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
		  "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
		  "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
		  "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]),
		  "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]),
		  "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]),
		  "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]),
		  "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
		: "l"(adesc), "l"(bdesc), "r"(accumulate)
		: "memory");
}

// wait until at most N commit groups of this warpgroup's MMAs are pending
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

struct TfArgs
{
	const uint4 * word_img;      // fp16 image of -2 w
	const uint4 * word_aug;      // augmentation K-step of the words (|w|^2 as hi + lo)
	int n_rows;                  // rows of this search
	const uint4 * query_img;
	const uint4 * query_aug;
	const float * qn;            // [nq] |q|^2
	int nq;
	int tile_begin, tile_end;    // tile range of the whole launch; blockIdx.y * tiles_per_split selects the CTA's share
	int tiles_per_split;
	const uint32_t * wmax2_bits; // largest |w|^2 of the dictionary (float bits)
	uint32_t * tau;              // [nq] shared bound on the second-smallest v (ordered-uint encoding)
	uint32_t * cand;             // [nq][kTfCandCap] candidate rows (local to this engine)
	int * cand_count;            // [nq]
	int emit;                    // 0: bound-only pre-pass
};

// grid = (query tiles, splits).  Roles as in knn2_tensor_kernel (nn_tensor.cuh): warpgroup 0 producer (bulk copies of the query tile and
// of the word tiles with their augmentation slabs), warpgroups 1-2 consumers (wgmma M64 per warpgroup, accumulators in registers; a
// thread holds two query rows of 64 columns each).
template <int DIM>
__global__ void __launch_bounds__(kTfThreads, 1)
knn2_tensor_f32_kernel(const TfArgs a)
{
	using Cfg = TfCfg<DIM>;
	constexpr int kStages = Cfg::stages;
	constexpr uint32_t kStageBytes = Cfg::stage_bytes;
	extern __shared__ unsigned char smem_dyn[];
	unsigned char * smem = reinterpret_cast<unsigned char *>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~static_cast<uintptr_t>(1023));
	unsigned char * sA = smem;                                   // query tile, then its augmentation slab
	unsigned char * sB = smem + Cfg::a_bytes + Cfg::a_aug_bytes; // stages of (word tile, augmentation slab)
	unsigned char * sBaug = sB + kStages * kStageBytes;          // 256: the word tile's augmentation slab
	uint64_t * bars = reinterpret_cast<uint64_t *>(sB + Cfg::ring_bytes);
	uint64_t * full = bars;                     // [kStages] word tile landed
	uint64_t * empty = full + kStages;          // [kStages] word tile consumed by both consumer warpgroups
	uint64_t * afull = empty + kStages;         // [1] query tile landed

	const int tid = threadIdx.x, wg = tid >> 7, lane = tid & 31;
	const int tile_begin = a.tile_begin + blockIdx.y * a.tiles_per_split;
	const int tile_end = min(a.tile_end, tile_begin + a.tiles_per_split);
	const int n_tiles = max(0, tile_end - tile_begin);
	const int qtile = blockIdx.x;

	if (tid == 0)
	{
		for (int s = 0; s < kStages; ++s)
		{
			mbar_init(&full[s], 1);
			mbar_init(&empty[s], 2);
		}
		mbar_init(afull, 1);
		mbar_fence_init();
	}
	__syncthreads();

	if (wg == 0)
	{
		if (tid == 0 && n_tiles > 0)
		{
			mbar_arrive_expect_tx(afull, Cfg::a_bytes + Cfg::a_aug_bytes);
			bulk_g2s(sA, reinterpret_cast<const unsigned char *>(a.query_img) + static_cast<size_t>(qtile) * Cfg::a_bytes, Cfg::a_bytes, afull);
			bulk_g2s(sA + Cfg::a_bytes, reinterpret_cast<const unsigned char *>(a.query_aug) + static_cast<size_t>(qtile) * Cfg::a_aug_bytes,
			         Cfg::a_aug_bytes, afull);
			if constexpr (Cfg::slices == 1)
			{
				for (int t = 0; t < n_tiles; ++t)
				{
					const int s = t % kStages;
					if (t >= kStages) mbar_wait(&empty[s], ((t / kStages) - 1) & 1);
					mbar_arrive_expect_tx(&full[s], kStageBytes);
					const unsigned char * src = reinterpret_cast<const unsigned char *>(a.word_img) + static_cast<size_t>(tile_begin + t) * Cfg::b_bytes;
					unsigned char * dst = sB + s * kStageBytes;
					bulk_g2s(dst, src, Cfg::b_bytes / 2, &full[s]);
					bulk_g2s(dst + Cfg::b_bytes / 2, src + Cfg::b_bytes / 2, Cfg::b_bytes / 2, &full[s]);
					bulk_g2s(dst + Cfg::b_bytes, reinterpret_cast<const unsigned char *>(a.word_aug) + static_cast<size_t>(tile_begin + t) * Cfg::b_aug_bytes,
					         Cfg::b_aug_bytes, &full[s]);
				}
			}
			else
			{
				// slice g of the launch = K slice g % slices of word tile g / slices; the image is [tile][atom][rows][128 B], so a slice
				// is one contiguous copy
				for (int g = 0; g < n_tiles * Cfg::slices; ++g)
				{
					const int s = g % kStages, t = g / Cfg::slices, k = g % Cfg::slices;
					const bool last = k == Cfg::slices - 1;
					if (g >= kStages) mbar_wait(&empty[s], ((g / kStages) - 1) & 1);
					mbar_arrive_expect_tx(&full[s], Cfg::slice_bytes + (last ? Cfg::b_aug_bytes : 0u));
					bulk_g2s(sB + s * kStageBytes,
					         reinterpret_cast<const unsigned char *>(a.word_img) + static_cast<size_t>(tile_begin + t) * Cfg::b_bytes + static_cast<size_t>(k) * Cfg::slice_bytes,
					         Cfg::slice_bytes, &full[s]);
					if (last)
						bulk_g2s(sBaug, reinterpret_cast<const unsigned char *>(a.word_aug) + static_cast<size_t>(tile_begin + t) * Cfg::b_aug_bytes, Cfg::b_aug_bytes,
						         &full[s]);
				}
			}
		}
		return;
	}

	// consumer warpgroup c: query rows [64 c, 64 c + 64) of the tile
	const int c = wg - 1;
	const int et = tid - 128 * wg;
	const int quad = lane & 3;
	const int r_lo = c * 64 + (et >> 5) * 16 + (lane >> 2); // tile rows of this thread: r_lo and r_lo + 8
	int qi[2];
	bool live[2];
	float margin[2], t1[2], t2[2];
#pragma unroll
	for (int h = 0; h < 2; ++h)
	{
		qi[h] = qtile * kTfBM + r_lo + 8 * h;
		live[h] = qi[h] < a.nq;
		margin[h] = 0.0f;
		t1[h] = INFINITY;
		t2[h] = INFINITY;
		if (live[h])
		{
			const float q2 = a.qn[qi[h]], w2 = __uint_as_float(*a.wmax2_bits);
			float eps;
			if constexpr (DIM == 256)
				eps = (1.02f * 0.001953125f + 1.220703125e-04f) * sqrtf(q2) * sqrtf(w2) + 6.103515625e-05f * (q2 + w2) + 4.0e-6f;
			else
				eps = 1.02f * 0.001953125f * sqrtf(q2) * sqrtf(w2) + 3.0517578125e-05f * (q2 + w2) + 4.0e-6f;
			margin[h] = 2.0f * eps;
			t2[h] = ord2f(a.tau[qi[h]]);
		}
	}
	if (n_tiles == 0) return;
	const int emit = a.emit;
	const uint32_t a_base = smem_u32(sA) + static_cast<uint32_t>(c * 64 * 128);
	const uint64_t a_aug = wg_smem_desc_noswz(smem_u32(sA + Cfg::a_bytes) + static_cast<uint32_t>(c * 8 * 256));
	float acc[128];
#pragma unroll
	for (int i = 0; i < 128; ++i) acc[i] = 0.0f;
	mbar_wait(afull, 0);
	for (int t = 0; t < n_tiles; ++t)
	{
		if constexpr (Cfg::slices == 1)
		{
			const int s = t % kStages;
			mbar_wait(&full[s], (t / kStages) & 1);
			__syncwarp(); // wgmma is .aligned: the warp issues it converged
			const uint32_t b_base = smem_u32(sB + s * kStageBytes);
			wg_fence();
#pragma unroll
			for (int ks = 0; ks < DIM / 16; ++ks)
			{
				const uint32_t atom = ks >> 2, koff = (ks & 3) * 32; // 16 halves = 32 bytes per K step, 4 steps per 128-byte atom
				wg_mma_f16(acc, wg_smem_desc(a_base + atom * (kTfBM * 128) + koff), wg_smem_desc(b_base + atom * (kTfBN * 128) + koff), ks > 0 ? 1u : 0u);
			}
			// the augmentation K-step: + kTfAugScale * (hi + lo) = + |w|^2
			wg_mma_f16(acc, a_aug, wg_smem_desc_noswz(b_base + Cfg::b_bytes), 1u);
			wg_commit();
			wg_wait_all();
			// the stage is free as soon as the MMAs have completed: the accumulators are in registers
			if (et == 0) mbar_arrive(&empty[s]);
		}
		else
		{
			// the accumulators carry over the K slices of the tile; a slice's stage is released as soon as the MMAs of the next slice
			// are issued and its own have completed (one commit group per slice)
#pragma unroll
			for (int k = 0; k < Cfg::slices; ++k)
			{
				const int g = t * Cfg::slices + k, s = g % kStages;
				mbar_wait(&full[s], (g / kStages) & 1);
				__syncwarp();
				const uint32_t b_base = smem_u32(sB + s * kStageBytes);
				wg_fence();
#pragma unroll
				for (int ks = 0; ks < 4; ++ks)
					wg_mma_f16(acc, wg_smem_desc(a_base + k * (kTfBM * 128) + ks * 32), wg_smem_desc(b_base + ks * 32), (k > 0 || ks > 0) ? 1u : 0u);
				if (k == Cfg::slices - 1) wg_mma_f16(acc, a_aug, wg_smem_desc_noswz(smem_u32(sBaug)), 1u);
				wg_commit();
				if (k > 0)
				{
					wg_wait<1>();
					if (et == 0) mbar_arrive(&empty[(g - 1) % kStages]);
				}
			}
			wg_wait<0>();
			if (et == 0) mbar_arrive(&empty[(t * Cfg::slices + Cfg::slices - 1) % kStages]);
		}
		const int row0 = (tile_begin + t) * kTfBN;
#pragma unroll
		for (int h = 0; h < 2; ++h)
		{
			float m = INFINITY;
#pragma unroll
			for (int i = 0; i < 32; ++i) m = fminf(m, fminf(acc[4 * i + 2 * h], acc[4 * i + 2 * h + 1]));
			if (live[h] && m <= t2[h] + margin[h])
			{
				// rare: some column of this tile may belong to the two nearest rows
#pragma unroll
				for (int lc = 0; lc < 64; ++lc)
				{
					const float x = acc[4 * (lc >> 1) + 2 * h + (lc & 1)];
					const int row = row0 + 8 * (lc >> 1) + 2 * quad + (lc & 1);
					// rows past n_rows of the cached image are words that are not searchable in this call (not indexed yet)
					if (x <= t2[h] + margin[h] && x < INFINITY && row < a.n_rows)
					{
						if (emit)
						{
							const int pos = atomicAdd(&a.cand_count[qi[h]], 1);
							if (pos < kTfCandCap) a.cand[static_cast<size_t>(qi[h]) * kTfCandCap + pos] = static_cast<uint32_t>(row);
						}
						// t2 only ever tightens: it starts as the shared bound while t1 is still unknown (+inf)
						if (x < t1[h])
						{
							t2[h] = fminf(t2[h], t1[h]);
							t1[h] = x;
						}
						else if (x < t2[h]) t2[h] = x;
					}
				}
			}
		}
	}
#pragma unroll
	for (int h = 0; h < 2; ++h)
		if (live[h] && t2[h] < INFINITY) atomicMin(&a.tau[qi[h]], f2ord(t2[h]));
}

// ---- exact re-rank of the candidate lists: one warp per query -----------------------------------------------------------------
// partial[q] = (best key, second key) with keys (float bits of rtflann's distance << 32 | row_offset + row); queries whose list
// overflowed go to the fallback list instead.
template <int DIM>
__global__ void rerank_l2_kernel(const float * __restrict__ vocab, int row_offset, const float * __restrict__ queries, int nq,
                                 const uint32_t * __restrict__ cand, const int * __restrict__ cand_count, ulonglong2 * __restrict__ partial,
                                 int * __restrict__ fb_list, int * __restrict__ fb_count)
{
	const int qi = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
	const int lane = threadIdx.x & 31;
	if (qi >= nq) return;
	const int n = cand_count[qi];
	if (n > kTfCandCap)
	{
		if (lane == 0) fb_list[atomicAdd(fb_count, 1)] = qi;
		return;
	}
	unsigned long long k1 = kKey64None, k2 = kKey64None;
	const float * q = queries + static_cast<size_t>(qi) * DIM;
	for (int c = lane; c < n; c += 32)
	{
		const uint32_t row = cand[static_cast<size_t>(qi) * kTfCandCap + c];
		float d;
		if constexpr (DIM > 128) d = l2_ptr_vs_stream<DIM>(q, vocab + static_cast<size_t>(row) * DIM); // fully unrolled, 256-D spills
		else d = l2_rtflann<DIM>(q, vocab + static_cast<size_t>(row) * DIM);
		top2_insert64(k1, k2, pack64(d, static_cast<uint32_t>(row_offset) + row));
	}
#pragma unroll
	for (int o = 16; o > 0; o >>= 1)
	{
		const unsigned long long o1 = __shfl_down_sync(0xFFFFFFFFu, k1, o);
		const unsigned long long o2 = __shfl_down_sync(0xFFFFFFFFu, k2, o);
		top2_insert64(k1, k2, o1);
		top2_insert64(k1, k2, o2);
	}
	if (lane == 0) partial[qi] = make_ulonglong2(k1, k2);
}

// exact scan for the queries of the fallback list (list overflow, values outside fp16), spread over the whole machine: the CTAs form
// S row-splits x G query-group slots (S as large as the scratch allows: one overflowing query still uses every SM).  A CTA takes
// kFbQueries queries at a time and streams its share of the vocabulary once for all of them: 256-row tiles are loaded coalesced
// into (padded) shared memory, thread t then computes row t against every query in rtflann's summation order.  The per-split results
// are merged by knn2_l2_fallback_merge_kernel.  Dynamic shared memory: R * (DIM + 1) + kFbQueries * DIM floats, R = fallback_rows<DIM>()
// rows per tile and threads per CTA (256; 128 at 256-D, where 256 rows would need 267 KB).
constexpr int kFbQueries = 4;
template <int DIM>
__host__ __device__ constexpr int fallback_rows() { return DIM == 256 ? 128 : 256; }
template <int DIM>
__host__ __device__ constexpr size_t fallback_smem_bytes() { return (fallback_rows<DIM>() * (DIM + 1) + kFbQueries * DIM) * sizeof(float); }

__device__ __forceinline__ int fallback_splits(int n_fb, int n_ctas, int slots) { return max(1, min(n_ctas, slots / max(n_fb, 1))); }

template <int DIM>
__global__ void __launch_bounds__(fallback_rows<DIM>())
knn2_l2_fallback_kernel(const float * __restrict__ vocab, int n_rows, int row_offset, const float * __restrict__ queries,
                        const int * __restrict__ fb_list, const int * __restrict__ fb_count, ulonglong2 * __restrict__ scratch, int slots)
{
	extern __shared__ __align__(16) float fb_smem[];
	constexpr int kRows = fallback_rows<DIM>();
	float * s_rows = fb_smem;                    // [kRows][DIM + 1]
	float * s_q = fb_smem + kRows * (DIM + 1);   // [kFbQueries][DIM]
	__shared__ unsigned long long s_k1[kFbQueries][8], s_k2[kFbQueries][8];
	const int n_fb = *fb_count;
	if (n_fb <= 0) return;
	const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
	const int S = fallback_splits(n_fb, gridDim.x, slots);
	const int split = blockIdx.x % S, gslot = blockIdx.x / S, n_gslots = gridDim.x / S;
	if (gslot >= n_gslots) return;
	const int n_groups = (n_fb + kFbQueries - 1) / kFbQueries;
	const int n_tiles = (n_rows + kRows - 1) / kRows;
	for (int g = gslot; g < n_groups; g += n_gslots)
	{
		const int nqg = min(kFbQueries, n_fb - g * kFbQueries);
		__syncthreads();
		for (int i = tid; i < nqg * DIM; i += kRows) s_q[i] = queries[static_cast<size_t>(fb_list[g * kFbQueries + i / DIM]) * DIM + (i % DIM)];
		unsigned long long k1[kFbQueries], k2[kFbQueries];
#pragma unroll
		for (int j = 0; j < kFbQueries; ++j) k1[j] = k2[j] = kKey64None;
		for (int t = split; t < n_tiles; t += S)
		{
			const int r0 = t * kRows;
			const int nr = min(kRows, n_rows - r0);
			__syncthreads();
			for (int i = tid; i < nr * (DIM / 4); i += kRows)
			{
				const int r = i / (DIM / 4), c = (i % (DIM / 4)) * 4;
				const float4 v = *reinterpret_cast<const float4 *>(vocab + static_cast<size_t>(r0 + r) * DIM + c);
				float * d = s_rows + r * (DIM + 1) + c;
				d[0] = v.x;
				d[1] = v.y;
				d[2] = v.z;
				d[3] = v.w;
			}
			__syncthreads();
			if (tid < nr)
			{
#pragma unroll
				for (int j = 0; j < kFbQueries; ++j)
				{
					if (j < nqg)
					{
						const float d = l2_rtflann<DIM>(s_q + j * DIM, s_rows + tid * (DIM + 1));
						top2_insert64(k1[j], k2[j], pack64(d, static_cast<uint32_t>(row_offset + r0 + tid)));
					}
				}
			}
		}
#pragma unroll
		for (int j = 0; j < kFbQueries; ++j)
		{
#pragma unroll
			for (int o = 16; o > 0; o >>= 1)
			{
				const unsigned long long o1 = __shfl_down_sync(0xFFFFFFFFu, k1[j], o);
				const unsigned long long o2 = __shfl_down_sync(0xFFFFFFFFu, k2[j], o);
				top2_insert64(k1[j], k2[j], o1);
				top2_insert64(k1[j], k2[j], o2);
			}
			if (lane == 0)
			{
				s_k1[j][warp] = k1[j];
				s_k2[j][warp] = k2[j];
			}
		}
		__syncthreads();
		if (tid < nqg)
		{
			unsigned long long a1 = kKey64None, a2 = kKey64None;
			for (int w = 0; w < kRows / 32; ++w)
			{
				top2_insert64(a1, a2, s_k1[tid][w]);
				top2_insert64(a1, a2, s_k2[tid][w]);
			}
			scratch[static_cast<size_t>(g * kFbQueries + tid) * S + split] = make_ulonglong2(a1, a2);
		}
	}
}

__global__ void knn2_l2_fallback_merge_kernel(const int * __restrict__ fb_list, const int * __restrict__ fb_count, const ulonglong2 * __restrict__ scratch,
                                              int slots, int n_ctas, ulonglong2 * __restrict__ partial)
{
	const int n_fb = *fb_count;
	const int S = fallback_splits(n_fb, n_ctas, slots);
	for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < n_fb; k += gridDim.x * blockDim.x)
	{
		unsigned long long a1 = kKey64None, a2 = kKey64None;
		for (int sp = 0; sp < S; ++sp)
		{
			const ulonglong2 p = scratch[static_cast<size_t>(k) * S + sp];
			top2_insert64(a1, a2, p.x);
			top2_insert64(a1, a2, p.y);
		}
		partial[fb_list[k]] = make_ulonglong2(a1, a2);
	}
}

} // namespace lcd
