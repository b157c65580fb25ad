// nn_tensor.cuh — exact Hamming 2-NN of 256-bit descriptors on the Hopper tensor cores (sm_90a, wgmma).
//
// The all-pairs distance matrix of VWDictionary::addNewWords / findNN (reference: corelib/src/VWDictionary.cpp:1004-1118,
// the brute-force branch, and rtflann's LinearIndex::findNeighbors, rtflann/algorithms/linear_index.h:113-123) is
// GEMM-shaped: with every descriptor bit b encoded as the signed byte 2b-1 the dot product of two descriptors is
//     a . w = 256 - 2 * hamming(a, w),
// an integer the tensor cores accumulate exactly in s32 (wgmma .s32.s8.s8).  The packed key order of
// common.cuh, (distance << 22) | row, is recovered in the epilogue as ((256 - acc) << 21) + row, so the result is
// bit-identical to the POPC kernel of nn_hamming.cuh (and to the oracle).
//
// One CTA owns a tile of 128 queries and a contiguous range of 256-word tiles.  Roles (three warpgroups):
//   warpgroup 0  producer : one thread issues cp.async.bulk (TMA engine) of the pre-tiled, pre-swizzled word image into a ring of
//                           shared-memory stages (the image is cached with the dictionary)
//   warpgroups 1-2 consumers: warpgroup c owns queries [64 (c-1), 64 c) of the tile.  It expands its half of the query tile in place
//                           from the packed form, issues 8 x wgmma.mma_async (M64 N256 K32) per word tile with the accumulators in
//                           registers, releases the stage and runs the top-2 epilogue while the other consumer's MMAs use the
//                           tensor cores.  Each query row is spread over the 4 threads of a lane quad (64 columns each), and each
//                           thread keeps its own running top-2, written out as one of kTcEpiGroups partial results.
//
// Operand images (written by the expand kernels below): K-major, 128-byte swizzle (the canonical GMMA/TMA layout:
// 16-byte chunk c of row r of every 8-row x 128-byte block sits at chunk c ^ (r & 7)), split in K/128 "atoms":
//   query tile : [atom][128 rows][128 B]            (32 KB for 256-bit descriptors)
//   word tile  : [atom][256 rows][128 B]            (64 KB)
// so a tile is ONE contiguous bulk copy and no tensor map is needed.
#pragma once
#include "common.cuh"

namespace lcd {

constexpr int kTcBM = 128;       // queries per CTA tile (two consumer warpgroups of M64)
constexpr int kTcBN = 256;       // words per tile (wgmma N)
constexpr int kTcK = 256;        // descriptor bits = int8 K extent
constexpr int kTcAtoms = kTcK / 128;
constexpr int kTcStages = 3;     // word-tile smem stages (3 x 64 KB + the 32 KB query tile fit the 227 KB a block may use)
constexpr int kTcEpiGroups = 4;  // partial results per query and split: the 4 threads of a lane quad that share a query row
constexpr int kTcThreads = 384;  // producer warpgroup + two consumer warpgroups
constexpr uint32_t kTcABytes = kTcBM * kTcK;
constexpr uint32_t kTcBBytes = kTcBN * kTcK;
constexpr size_t kTcSmemBytes = 1024 /* alignment slack */ + kTcABytes + kTcStages * kTcBBytes + 256 /* barriers */;

// ---- operand expansion: bit b -> int8 (2b - 1), tiled + swizzled ---------------------------------
// One thread writes one 16-byte chunk (16 descriptor bits).  rows >= n_rows of the last tile are written as 0.
__device__ __forceinline__ uint32_t expand4(uint32_t nibble)
{
	const uint32_t t = (nibble * 0x00204081u) & 0x01010101u; // bit i -> byte i (0 / 1)
	const uint32_t m = t * 0xFFu;                            // 0x00 / 0xFF per byte
	return (~m) | t;                                         // 0 -> 0xFF (-1), 1 -> 0x01 (+1)
}

__global__ void tc_expand_kernel(const uint32_t * __restrict__ src /* [n_rows][8] */, int n_rows, int tile_rows, int tile0, int n_tiles,
                                 uint4 * __restrict__ dst)
{
	// tiles [tile0, n_tiles): the image of a frozen dictionary is built once and kept; only tiles that gained rows are rewritten
	const size_t gid = static_cast<size_t>(tile0) * tile_rows * 16 + static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
	const size_t total = static_cast<size_t>(n_tiles) * tile_rows * 16;
	if (gid >= total) return;
	const int chunk = static_cast<int>(gid & 15);           // 16-byte chunk of the 256-byte expanded row
	const size_t row = gid >> 4;
	const int tile = static_cast<int>(row / tile_rows), r = static_cast<int>(row % tile_rows);
	uint4 v = make_uint4(0, 0, 0, 0);
	if (row < static_cast<size_t>(n_rows))
	{
		const uint32_t w = src[row * 8 + (chunk >> 1)];
		const uint32_t bits = (w >> ((chunk & 1) * 16)) & 0xFFFFu;
		v.x = expand4(bits & 15u);
		v.y = expand4((bits >> 4) & 15u);
		v.z = expand4((bits >> 8) & 15u);
		v.w = expand4((bits >> 12) & 15u);
	}
	const int atom = chunk >> 3, c = chunk & 7;
	const size_t off16 = static_cast<size_t>(tile) * (static_cast<size_t>(tile_rows) * 16) + static_cast<size_t>(atom) * (tile_rows * 8) +
	                     static_cast<size_t>(r) * 8 + static_cast<size_t>(c ^ (r & 7));
	dst[off16] = v;
}

// ---- Hopper mbarrier / wgmma helpers ---------------------------------------------------------------
__device__ __forceinline__ void mbar_arrive(uint64_t * bar)
{
	asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// named barrier over the 128 threads of one warpgroup (id 0 is __syncthreads)
__device__ __forceinline__ void wg_bar_sync(int id) { asm volatile("bar.sync %0, 128;" ::"r"(id) : "memory"); }
// shared-memory matrix descriptor (GMMA): K-major, SWIZZLE_128B, 8-row groups 1024 B apart
__device__ __forceinline__ uint64_t wg_smem_desc(uint32_t saddr)
{
	uint64_t d = 0;
	d |= static_cast<uint64_t>((saddr & 0x3FFFFu) >> 4);        // start address  [0,14)
	d |= static_cast<uint64_t>(1) << 16;                         // leading byte offset (unused for swizzled K-major)
	d |= static_cast<uint64_t>(1024 >> 4) << 32;                 // stride byte offset [32,46)
	d |= static_cast<uint64_t>(1) << 62;                         // layout type [62,64): SWIZZLE_128B
	return d;
}
// D[regs] (+)= A[smem] * B[smem]^T, s8 x s8 -> s32, M64 x N256 x K32 over one warpgroup.  Accumulator fragment: thread (warp w,
// lane l) holds rows 16 w + l / 4 (d[4 i], d[4 i + 1]) and 16 w + l / 4 + 8 (d[4 i + 2], d[4 i + 3]) at columns 8 i + 2 (l % 4) + {0, 1}.
__device__ __forceinline__ void wg_mma_i8(int (&d)[128], uint64_t adesc, uint64_t bdesc, uint32_t accumulate)
{
	asm volatile(
		"{\n"
		".reg .pred p;\n"
		"setp.ne.b32 p, %130, 0;\n"
		"wgmma.mma_async.sync.aligned.m64n256k32.s32.s8.s8 "
		"{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
		"%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
		"%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
		"%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
		"%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "
		"%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, "
		"%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, "
		"%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, "
		"%128, %129, p;\n"
		"}\n"
		: "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]),
		  "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]),
		  "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]),
		  "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]),
		  "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]),
		  "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]),
		  "+r"(d[48]), "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55]),
		  "+r"(d[56]), "+r"(d[57]), "+r"(d[58]), "+r"(d[59]), "+r"(d[60]), "+r"(d[61]), "+r"(d[62]), "+r"(d[63]),
		  "+r"(d[64]), "+r"(d[65]), "+r"(d[66]), "+r"(d[67]), "+r"(d[68]), "+r"(d[69]), "+r"(d[70]), "+r"(d[71]),
		  "+r"(d[72]), "+r"(d[73]), "+r"(d[74]), "+r"(d[75]), "+r"(d[76]), "+r"(d[77]), "+r"(d[78]), "+r"(d[79]),
		  "+r"(d[80]), "+r"(d[81]), "+r"(d[82]), "+r"(d[83]), "+r"(d[84]), "+r"(d[85]), "+r"(d[86]), "+r"(d[87]),
		  "+r"(d[88]), "+r"(d[89]), "+r"(d[90]), "+r"(d[91]), "+r"(d[92]), "+r"(d[93]), "+r"(d[94]), "+r"(d[95]),
		  "+r"(d[96]), "+r"(d[97]), "+r"(d[98]), "+r"(d[99]), "+r"(d[100]), "+r"(d[101]), "+r"(d[102]), "+r"(d[103]),
		  "+r"(d[104]), "+r"(d[105]), "+r"(d[106]), "+r"(d[107]), "+r"(d[108]), "+r"(d[109]), "+r"(d[110]), "+r"(d[111]),
		  "+r"(d[112]), "+r"(d[113]), "+r"(d[114]), "+r"(d[115]), "+r"(d[116]), "+r"(d[117]), "+r"(d[118]), "+r"(d[119]),
		  "+r"(d[120]), "+r"(d[121]), "+r"(d[122]), "+r"(d[123]), "+r"(d[124]), "+r"(d[125]), "+r"(d[126]), "+r"(d[127])
		: "l"(adesc), "l"(bdesc), "r"(accumulate)
		: "memory");
}

// ---- the kernel ------------------------------------------------------------------------------------
// neg32 = (uint32_t)-32, passed as an argument so that the key arithmetic stays an IMAD on the FMA pipe instead of being
// strength-reduced to a shift-add on the ALU pipe, which the min/max network needs.
// Work items = (query tile, word split) pairs, item = split * n_qtiles + qtile.  The grid is PERSISTENT: CTA b runs items b, b + gridDim.x,
// ... with one set of barriers; the word-tile stream runs on across item boundaries (all barrier phases are functions of a CTA-wide
// running tile count), and the packed queries of the next item are loaded into registers while the current item runs.  What an item
// boundary costs is the in-place expansion of the query tile instead of a CTA launch and a pipeline fill — which is what a word-range
// shard with few tiles per item was paying.
// partial[(split * kTcEpiGroups + quad) * nq + query] = (best key, second key) over the rows of that split that fall in the 64 columns of
// each tile owned by lane quad position `quad` (columns 8 i + 2 quad + {0, 1}).
__global__ void __launch_bounds__(kTcThreads, 1)
knn2_tensor_kernel(const uint4 * __restrict__ word_img, int n_rows, int row_offset, const uint32_t * __restrict__ queries /* [nq][8] packed */, int nq,
                   uint2 * __restrict__ partial, int tiles_per_split, uint32_t neg32, int n_qtiles, int n_splits)
{
	extern __shared__ unsigned char smem_dyn[];
	unsigned char * smem = reinterpret_cast<unsigned char *>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~static_cast<uintptr_t>(1023));
	unsigned char * sA = smem;
	unsigned char * sB = smem + kTcABytes;
	uint64_t * bars = reinterpret_cast<uint64_t *>(sB + kTcStages * kTcBBytes);
	uint64_t * full = bars;                    // [kTcStages] word tile landed
	uint64_t * empty = bars + kTcStages;       // [kTcStages] word tile consumed by both consumer warpgroups

	const int tid = threadIdx.x, wg = tid >> 7, lane = tid & 31;
	const int n_tiles_total = (n_rows + kTcBN - 1) / kTcBN;
	const int n_items = n_qtiles * n_splits;
	// tiles of an item (every role walks the same item sequence and keeps the same running tile count)
	auto item_tiles = [&](int item, int & tile_begin) {
		tile_begin = (item / n_qtiles) * tiles_per_split;
		return max(0, min(n_tiles_total, tile_begin + tiles_per_split) - tile_begin);
	};

	if (tid == 0)
	{
		for (int s = 0; s < kTcStages; ++s)
		{
			mbar_init(&full[s], 1);
			mbar_init(&empty[s], 2); // one arrival per consumer warpgroup
		}
		mbar_fence_init();
	}
	__syncthreads();

	if (wg == 0)
	{
		if (tid == 0)
		{
			int g = 0; // running tile count of this CTA
			for (int item = blockIdx.x; item < n_items; item += gridDim.x)
			{
				int tile_begin;
				const int n_tiles = item_tiles(item, tile_begin);
				for (int t = 0; t < n_tiles; ++t, ++g)
				{
					const int s = g % kTcStages;
					if (g >= kTcStages) mbar_wait(&empty[s], ((g / kTcStages) - 1) & 1);
					mbar_arrive_expect_tx(&full[s], kTcBBytes);
					const unsigned char * src = reinterpret_cast<const unsigned char *>(word_img) + static_cast<size_t>(tile_begin + t) * kTcBBytes;
					bulk_g2s(sB + s * kTcBBytes, src, kTcBBytes / 2, &full[s]);
					bulk_g2s(sB + s * kTcBBytes + kTcBBytes / 2, src + kTcBBytes / 2, kTcBBytes / 2, &full[s]);
				}
			}
		}
		return;
	}

	// consumer warpgroup c: query rows [64 c, 64 c + 64) of the tile
	const int c = wg - 1;
	const int et = tid - 128 * wg;
	const int quad = lane & 3;
	const int r_lo = c * 64 + (et >> 5) * 16 + (lane >> 2); // tile rows of this thread's accumulators: r_lo and r_lo + 8
	// The query half goes from its packed form (32 B per descriptor) straight into the swizzled +-1 byte image in shared memory:
	// no expanded copy of the queries ever touches HBM.  One 16-byte chunk (16 descriptor bits) per thread and step.
	uint4 * sA4 = reinterpret_cast<uint4 *>(sA);
	constexpr int kItems = 64 * 16 / 128; // chunks per thread: same chunk column, rows 8 apart
	const int chunk = et & 15, er0 = c * 64 + (et >> 4);
	uint32_t w[kItems];
	auto load_packed = [&](int qtile) { // all loads in flight before the first use: one memory round trip
#pragma unroll
		for (int j = 0; j < kItems; ++j)
		{
			const int q = qtile * kTcBM + er0 + 8 * j;
			w[j] = q < nq ? __ldg(queries + static_cast<size_t>(q) * 8 + (chunk >> 1)) : 0u;
		}
	};
	auto expand_tile = [&](int qtile) {
#pragma unroll
		for (int j = 0; j < kItems; ++j)
		{
			const int r = er0 + 8 * j;
			uint4 v = make_uint4(0, 0, 0, 0);
			if (qtile * kTcBM + r < nq)
			{
				const uint32_t bits = (w[j] >> ((chunk & 1) * 16)) & 0xFFFFu;
				v.x = expand4(bits & 15u);
				v.y = expand4((bits >> 4) & 15u);
				v.z = expand4((bits >> 8) & 15u);
				v.w = expand4((bits >> 12) & 15u);
			}
			const int atom = chunk >> 3, cc = chunk & 7;
			sA4[atom * (kTcBM * 8) + r * 8 + (cc ^ (r & 7))] = v;
		}
		asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); // generic-proxy writes -> visible to the tensor core's async proxy
		wg_bar_sync(1 + c);
	};
	const uint32_t a_base = smem_u32(sA) + static_cast<uint32_t>(c * 64 * 128);
	int acc[128];
#pragma unroll
	for (int i = 0; i < 128; ++i) acc[i] = 0;
	int g = 0;
	if (static_cast<int>(blockIdx.x) < n_items) load_packed(static_cast<int>(blockIdx.x) % n_qtiles);
	for (int item = blockIdx.x; item < n_items; item += gridDim.x)
	{
		int tile_begin;
		const int n_tiles = item_tiles(item, tile_begin);
		const int qtile = item % n_qtiles, split = item / n_qtiles;
		wg_bar_sync(1 + c); // every warp of this warpgroup is past the MMAs that read the previous query tile
		expand_tile(qtile);
		const int next = item + static_cast<int>(gridDim.x);
		if (next < n_items) load_packed(next % n_qtiles); // in registers long before the boundary
		uint32_t k1[2] = {kKeyNone, kKeyNone}, k2[2] = {kKeyNone, kKeyNone};
		int thr[2] = {-100000, -100000}; // accumulator value a candidate has to exceed to enter the top-2
		for (int t = 0; t < n_tiles; ++t, ++g)
		{
			const int s = g % kTcStages;
			mbar_wait(&full[s], (g / kTcStages) & 1);
			__syncwarp(); // wgmma is .aligned: the warp issues it converged
			const uint32_t b_base = smem_u32(sB + s * kTcBBytes);
			wg_fence();
#pragma unroll
			for (int ks = 0; ks < kTcK / 32; ++ks)
			{
				const uint32_t atom = ks >> 2, koff = (ks & 3) * 32;
				wg_mma_i8(acc, wg_smem_desc(a_base + atom * (kTcBM * 128) + koff), wg_smem_desc(b_base + atom * (kTcBN * 128) + koff), ks > 0 ? 1u : 0u);
			}
			wg_commit();
			wg_wait_all();
			// the stage is free as soon as the MMAs have completed: the accumulators are in registers
			if (et == 0) mbar_arrive(&empty[s]);
			const int row0 = (tile_begin + t) * kTcBN;
			const int valid = n_rows - row0; // columns of this tile that are real words
#pragma unroll
			for (int h = 0; h < 2; ++h)
			{
				if (valid >= kTcBN)
				{
					// Branch-free top-2 over this thread's 64 columns of the row with 16-bit keys, two columns per register:
					//   key16 = distance * 64 + j = acc * (-32) + (8192 + j)   (distance = (256 - acc) / 2 <= 256, j < 32)
					// The low half-word carries local column j, the high half-word local column j + 32; S = acc_hi * 65536 + acc_lo and
					// K = S * (-32) + (8192 + j) * 65537 is that pair of keys exactly (every field stays in [0, 65536), so no
					// carry crosses the halves).  Two IMADs (FMA pipe) and three VIMNMX.U16x2 (ALU pipe) per column pair.
					uint32_t p1 = 0xFFFFFFFFu, p2 = 0xFFFFFFFFu;
#pragma unroll
					for (int j = 0; j < 32; ++j)
					{
						const int lo = 4 * (j >> 1) + 2 * h + (j & 1); // local column j; local column j + 32 is lo + 64
						const uint32_t sp = static_cast<uint32_t>(acc[lo + 64]) * 65536u + static_cast<uint32_t>(acc[lo]);
						const uint32_t kp = sp * neg32 + static_cast<uint32_t>(8192 + j) * 65537u;
						const uint32_t mx = __vmaxu2(p1, kp);
						p1 = __vminu2(p1, kp);
						p2 = __vminu2(p2, mx);
					}
					// the four survivors (two per half) go into the running packed keys only if they can improve them
					const uint32_t best16 = min(p1 & 0xFFFFu, p1 >> 16);
					if (static_cast<int>(best16 >> 6) * 2 < kTcK - thr[h])
					{
						const uint32_t base = static_cast<uint32_t>(row_offset + row0 + 2 * quad);
						const uint32_t cand[4] = {p1 & 0xFFFFu, p2 & 0xFFFFu, p1 >> 16, p2 >> 16};
#pragma unroll
						for (int u = 0; u < 4; ++u)
						{
							const uint32_t lc = (cand[u] & 63u) + (u >= 2 ? 32u : 0u); // local column -> tile column 8 (lc / 2) + 2 quad + lc % 2
							const uint32_t key = ((cand[u] >> 6) << kKeyShift) + base + 8u * (lc >> 1) + (lc & 1u);
							top2_insert(k1[h], k2[h], key);
						}
						thr[h] = k2[h] == kKeyNone ? -100000 : kTcK - 2 * static_cast<int>(k2[h] >> kKeyShift);
					}
				}
				else if (valid > 0)
				{
					// last, partly filled tile: plain insertion of the real columns
#pragma unroll
					for (int lc = 0; lc < 64; ++lc)
					{
						const int col = 8 * (lc >> 1) + 2 * quad + (lc & 1);
						if (col < valid)
						{
							const int a = acc[4 * (lc >> 1) + 2 * h + (lc & 1)];
							const uint32_t key = (static_cast<uint32_t>(kTcK - a) << (kKeyShift - 1)) + static_cast<uint32_t>(row_offset + row0 + col);
							top2_insert(k1[h], k2[h], key);
						}
					}
					thr[h] = k2[h] == kKeyNone ? -100000 : kTcK - 2 * static_cast<int>(k2[h] >> kKeyShift);
				}
			}
		}
#pragma unroll
		for (int h = 0; h < 2; ++h)
		{
			const int qi = qtile * kTcBM + r_lo + 8 * h;
			if (qi < nq) partial[(static_cast<size_t>(split) * kTcEpiGroups + quad) * nq + qi] = make_uint2(k1[h], k2[h]);
		}
	}
}

} // namespace lcd
