// nn_tensor.cuh — exact Hamming 2-NN of 256-bit descriptors on the Hopper binary tensor cores (sm_90a, wgmma .b1).
//
// The all-pairs distance matrix of VWDictionary::addNewWords / findNN (reference: corelib/src/VWDictionary.cpp:1004-1118,
// the brute-force branch, and rtflann's LinearIndex::findNeighbors, rtflann/algorithms/linear_index.h:113-123) is
// GEMM-shaped: one wgmma m64n128k256 .b1.and.popc (BGMMA) gives, for 64 queries a x 128 words w, c = popc(a AND w) over the whole
// descriptor, and
//     hamming(a, w) = pa + pw - 2 c,          pa = popc(a), pw = popc(w).
// Within a query row pa is a constant, so the epilogue orders the words by pw - 2 c and adds pa back only when a survivor becomes a
// packed key of common.cuh, (distance << 22) | row: the result is bit-identical to the POPC kernel of nn_hamming.cuh (and to the
// oracle).  pw is cached with the word image (below), folded into the per-column constants of the epilogue.
//
// One CTA owns a tile of 256 queries and a contiguous range of 256-word tiles.  Roles (five warpgroups, 640 threads):
//   warpgroup 0  producer : one thread issues cp.async.bulk (TMA engine) of the pre-tiled word image into a ring of shared-memory
//                           stages (the image is cached with the dictionary).  The warpgroup gives its registers away (setmaxnreg
//                           24), so the four consumers may hold 112 each where the launch gives every thread 96.
//   warpgroups 1-4 consumers: warpgroup c owns queries [64 (c-1), 64 c) of the tile.  It copies its quarter of the packed query tile
//                           into the operand layout and, per word tile, issues one BGMMA (M64 N128 K256) on columns [0, 128), waits,
//                           runs that half's top-2 epilogue, then does the same for columns [128, 256).  The accumulators are 64
//                           registers.  Nothing orders the consumers against each other: while one waits for its MMA, the warp
//                           schedulers issue the epilogues of the other three (four consumer warps per scheduler).  Each query row is
//                           spread over the 4 threads of a lane quad (64 columns of the tile each), and each thread keeps its own
//                           running top-2, written out as one of kTcEpiGroups partial results.
//
// Operand layout: K-major, no swizzle, 32-byte rows (the 256 descriptor bits, in the order of the packed descriptor) cut into 8-row x
// 16-byte core matrices: byte b of row r sits at (r / 8) * 256 + (b / 16) * 128 + (r % 8) * 16 + b % 16.  A and B share it, so
// popc(a AND w) sees the same bit at the same k in both.
//   query tile : [256 rows] 8 KB, two of them (the next item's queries are copied in while the current item runs)
//   word tile  : [256 rows] 8 KB, followed by the 512-byte epilogue constants T of that tile (tc_pack_kernel)
// so a word tile is ONE contiguous bulk copy and no tensor map is needed.  Its second half-tile (rows [128, 256)) starts 4 KB in.
#pragma once
#include "common.cuh"

namespace lcd {

constexpr int kTcBM = 256;       // queries per CTA tile (four consumer warpgroups of M64)
constexpr int kTcBN = 256;       // words per tile (two wgmma N128 half-tiles)
constexpr int kTcHalfN = kTcBN / 2;
constexpr int kTcK = 256;        // descriptor bits = b1 K extent
constexpr int kTcRowBytes = kTcK / 8;
constexpr int kTcStages = 8;     // word-tile smem stages; a choice, not swept: 7 tiles in flight behind the one in use
constexpr int kTcEpiGroups = 4;  // partial results per query and split: the 4 threads of a lane quad that share a query row
constexpr int kTcConsumers = 4;  // consumer warpgroups
constexpr int kTcThreads = 128 * (1 + kTcConsumers);
// setmaxnreg moves registers within the CTA's pool, which is what the launch gave it: 640 x 96 = 61 440.  128 * 24 + 512 * 112 =
// 60 416 fits; a consumer budget of 120 (64 512) would never be granted and its setmaxnreg.inc would wait forever.
constexpr uint32_t kTcProducerRegs = 24, kTcConsumerRegs = 112;
constexpr uint32_t kTcABytes = kTcBM * kTcRowBytes;
constexpr uint32_t kTcWordBytes = kTcBN * kTcRowBytes;
constexpr uint32_t kTcHalfBytes = kTcHalfN * kTcRowBytes;  // the rows of one half-tile
constexpr uint32_t kTcBBytes = kTcWordBytes + kTcBN * 2;  // packed rows + T (one 16-bit field per word)
constexpr size_t kTcSmemBytes = 1024 /* alignment slack */ + 2 * kTcABytes + kTcStages * kTcBBytes + 256 /* barriers */;

// byte offset of the 16-byte chunk `half` (descriptor bits [128 half, 128 half + 128)) of row r in the operand layout
__host__ __device__ __forceinline__ uint32_t tc_chunk_off(int r, int half) { return (r >> 3) * 256 + half * 128 + (r & 7) * 16; }

// ---- the cached word image: packed rows in the operand layout + the epilogue constants, per 256-row tile ----------------------
// T of a tile is the uint32 array [hf = 0..1][k = 0..3][quad = 0..3][e = 0..3]: for the lane quad `quad`, half-tile hf and its local
// column pair j = 4 k + e (tile columns col = 128 hf + 8 (j / 2) + 2 quad + j % 2 and col + 64, fragment columns i = j / 2 and i + 8
// of the N128 accumulators) it holds the two 16-bit fields
//     64 (pw(col) + 256) + 32 hf + j   |   (64 (pw(col + 64) + 256) + 32 hf + 16 + j) << 16
// which the epilogue adds to -128 c of both columns to get its 16-bit keys (see knn2_tensor_kernel).  The low 6 bits, lc, are the
// thread's local column over the whole tile: tile column 8 (lc / 2) + 2 quad + lc % 2, in the order of the rows.  Stored so that the 4
// quads of a warp read 64 consecutive bytes with one LDS.128 each.  One thread writes one 16-byte chunk; rows >= n_rows are written as
// 0.
__global__ void tc_pack_kernel(const uint4 * __restrict__ src /* [n_rows][2] */, int n_rows, int tile0, int n_tiles, uint4 * __restrict__ dst)
{
	// tiles [tile0, n_tiles): the image of a frozen dictionary is built once and kept; only tiles that gained rows are rewritten
	constexpr int kChunks = kTcBBytes / 16, kRowChunks = kTcWordBytes / 16;
	const size_t gid = static_cast<size_t>(tile0) * kChunks + static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
	if (gid >= static_cast<size_t>(n_tiles) * kChunks) return;
	const int tile = static_cast<int>(gid / kChunks), o = static_cast<int>(gid % kChunks);
	const int row0 = tile * kTcBN;
	uint4 v = make_uint4(0, 0, 0, 0);
	if (o < kRowChunks)
	{
		// chunk o = (r / 8) * 16 + half * 8 + r % 8, the inverse of tc_chunk_off
		const int r = (o >> 4) * 8 + (o & 7), half = (o >> 3) & 1;
		if (row0 + r < n_rows) v = src[static_cast<size_t>(row0 + r) * 2 + half];
	}
	else
	{
		const int t = o - kRowChunks, hf = t >> 4, k = (t >> 2) & 3, quad = t & 3;
		auto pw = [&](int col) {
			if (row0 + col >= n_rows) return 0;
			const uint4 a = src[static_cast<size_t>(row0 + col) * 2], b = src[static_cast<size_t>(row0 + col) * 2 + 1];
			return __popc(a.x) + __popc(a.y) + __popc(a.z) + __popc(a.w) + __popc(b.x) + __popc(b.y) + __popc(b.z) + __popc(b.w);
		};
		uint32_t f[4];
#pragma unroll
		for (int e = 0; e < 4; ++e)
		{
			const int j = 4 * k + e, col = kTcHalfN * hf + 8 * (j >> 1) + 2 * quad + (j & 1);
			f[e] = static_cast<uint32_t>(64 * (pw(col) + 256) + 32 * hf + j) | (static_cast<uint32_t>(64 * (pw(col + 64) + 256) + 32 * hf + 16 + j) << 16);
		}
		v = make_uint4(f[0], f[1], f[2], f[3]);
	}
	dst[gid] = v;
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
// shared-memory matrix descriptor (GMMA) of an UN-swizzled K-major operand with 32-byte rows: 8 x 16-byte core matrices, the two
// 16-byte chunks of a row group 128 B apart (leading byte offset), row groups 256 B apart (stride byte offset)
__device__ __forceinline__ uint64_t wg_smem_desc_noswz(uint32_t saddr)
{
	uint64_t d = 0;
	d |= static_cast<uint64_t>((saddr & 0x3FFFFu) >> 4);        // start address  [0,14)
	d |= static_cast<uint64_t>(128 >> 4) << 16;                  // leading byte offset [16,30): next core matrix along K
	d |= static_cast<uint64_t>(256 >> 4) << 32;                  // stride byte offset [32,46): next 8-row group
	return d;                                                    // layout type 0: no swizzle
}
// D[regs] = popc(A[smem] AND B[smem]^T), b1 x b1 -> s32, M64 x N128 x K256 over one warpgroup (BGMMA): half a word tile.
// D is overwritten, not accumulated (scale-d = 0), so it is an output only: its registers are free from the last read of one half-tile's
// epilogue to the next MMA.
// Accumulator fragment: thread (warp w, lane l) holds rows 16 w + l / 4 (d[4 i], d[4 i + 1]) and 16 w + l / 4 + 8 (d[4 i + 2],
// d[4 i + 3]) at columns 8 i + 2 (l % 4) + {0, 1}, i < 16.
__device__ __forceinline__ void wg_mma_b1(int (&d)[64], uint64_t adesc, uint64_t bdesc)
{
	asm volatile(
		"{\n"
		".reg .pred p;\n"
		"setp.ne.b32 p, 0, 0;\n"
		"wgmma.mma_async.sync.aligned.m64n128k256.s32.b1.b1.and.popc "
		"{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
		"%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
		"%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
		"%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
		"%64, %65, p;\n"
		"}\n"
		: "=r"(d[0]), "=r"(d[1]), "=r"(d[2]), "=r"(d[3]), "=r"(d[4]), "=r"(d[5]), "=r"(d[6]), "=r"(d[7]),
		  "=r"(d[8]), "=r"(d[9]), "=r"(d[10]), "=r"(d[11]), "=r"(d[12]), "=r"(d[13]), "=r"(d[14]), "=r"(d[15]),
		  "=r"(d[16]), "=r"(d[17]), "=r"(d[18]), "=r"(d[19]), "=r"(d[20]), "=r"(d[21]), "=r"(d[22]), "=r"(d[23]),
		  "=r"(d[24]), "=r"(d[25]), "=r"(d[26]), "=r"(d[27]), "=r"(d[28]), "=r"(d[29]), "=r"(d[30]), "=r"(d[31]),
		  "=r"(d[32]), "=r"(d[33]), "=r"(d[34]), "=r"(d[35]), "=r"(d[36]), "=r"(d[37]), "=r"(d[38]), "=r"(d[39]),
		  "=r"(d[40]), "=r"(d[41]), "=r"(d[42]), "=r"(d[43]), "=r"(d[44]), "=r"(d[45]), "=r"(d[46]), "=r"(d[47]),
		  "=r"(d[48]), "=r"(d[49]), "=r"(d[50]), "=r"(d[51]), "=r"(d[52]), "=r"(d[53]), "=r"(d[54]), "=r"(d[55]),
		  "=r"(d[56]), "=r"(d[57]), "=r"(d[58]), "=r"(d[59]), "=r"(d[60]), "=r"(d[61]), "=r"(d[62]), "=r"(d[63])
		: "l"(adesc), "l"(bdesc)
		: "memory");
}
// Register budget of a warpgroup's threads (setmaxnreg): every warp of the warpgroup executes it, with the same count.
template <uint32_t kRegs> __device__ __forceinline__ void wg_regs_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kRegs)); }
template <uint32_t kRegs> __device__ __forceinline__ void wg_regs_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kRegs)); }

// ---- the kernel ------------------------------------------------------------------------------------
// neg128 = (uint32_t)-128, passed as an argument so that the key arithmetic stays an IMAD on the FMA pipe instead of being
// strength-reduced to a shift-add on the ALU pipe, which the min/max network needs.
// Work items = (query tile, word split) pairs, item = split * n_qtiles + qtile.  The grid is PERSISTENT: CTA b runs items b, b + gridDim.x,
// ... with one set of barriers; the word-tile stream runs on across item boundaries (all barrier phases are functions of a CTA-wide
// running tile count), and the packed queries of the next item are copied into the other query buffer while the current item runs.
// What an item boundary costs is one warpgroup barrier instead of a CTA launch and a pipeline fill — which is what a word-range shard
// with few tiles per item was paying.
// partial[(split * kTcEpiGroups + quad) * nq + query] = (best key, second key) over the rows of that split that fall in the 64 columns of
// each tile owned by lane quad position `quad` (columns 8 i + 2 quad + {0, 1}).
__global__ void __launch_bounds__(kTcThreads, 1)
knn2_tensor_kernel(const uint4 * __restrict__ word_img, int n_rows, int row_offset, const uint32_t * __restrict__ queries /* [nq][8] packed */, int nq,
                   uint2 * __restrict__ partial, int tiles_per_split, uint32_t neg128, int n_qtiles, int n_splits)
{
	extern __shared__ unsigned char smem_dyn[];
	// aligned by offsetting smem_dyn itself, not through an integer round trip, so that the compiler keeps the shared address space and
	// reads T and the queries with LDS (a generic load costs an address-space check on every read of the epilogue)
	unsigned char * smem = smem_dyn + ((1024u - (smem_u32(smem_dyn) & 1023u)) & 1023u);
	unsigned char * sA = smem;
	unsigned char * sB = smem + 2 * kTcABytes;        // after the two query buffers
	uint64_t * bars = reinterpret_cast<uint64_t *>(sB + kTcStages * kTcBBytes);
	uint64_t * full = bars;                    // [kTcStages] word tile landed
	uint64_t * empty = bars + kTcStages;       // [kTcStages] word tile consumed by every consumer warp

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
			mbar_init(&empty[s], 4 * kTcConsumers); // one arrival per consumer warp: each reads T of the stage in its epilogues
		}
		mbar_fence_init();
	}
	__syncthreads();

	if (wg == 0)
	{
		wg_regs_dec<kTcProducerRegs>();
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
					bulk_g2s(sB + s * kTcBBytes, reinterpret_cast<const unsigned char *>(word_img) + static_cast<size_t>(tile_begin + t) * kTcBBytes,
					         kTcBBytes, &full[s]);
				}
			}
		}
		return;
	}

	// consumer warpgroup c: query rows [64 c, 64 c + 64) of the tile
	wg_regs_inc<kTcConsumerRegs>();
	const int c = wg - 1;
	const int et = tid - 128 * wg;
	const int quad = lane & 3;
	const int r_lo = c * 64 + (et >> 5) * 16 + (lane >> 2); // tile rows of this thread's accumulators: r_lo and r_lo + 8
	// The query half goes from its packed form straight into the operand layout in shared memory, by cp.async, one item ahead into the
	// other of two query buffers: one 16-byte chunk per thread (row er, descriptor bits [128 half, 128 half + 128)), copied as 32-bit
	// words because the caller's query pointer is only 4-byte aligned.  Rows >= nq are zero-filled.
	const int er = c * 64 + (et >> 1), half = et & 1;
	auto prefetch = [&](int qtile, int buf) {
		const int q = qtile * kTcBM + er;
		const uint32_t dst = smem_u32(sA + buf * kTcABytes + tc_chunk_off(er, half));
		const uint32_t * src = q < nq ? queries + static_cast<size_t>(q) * 8 + 4 * half : queries;
		const uint32_t n = q < nq ? 4u : 0u;
#pragma unroll
		for (int j = 0; j < 4; ++j) asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(dst + 4 * j), "l"(src + j), "r"(n) : "memory");
		asm volatile("cp.async.commit_group;" ::: "memory");
	};
	int acc[64];
	int g = 0, buf = 0;
	if (static_cast<int>(blockIdx.x) < n_items) prefetch(static_cast<int>(blockIdx.x) % n_qtiles, 0);
	for (int item = blockIdx.x; item < n_items; item += gridDim.x, buf ^= 1)
	{
		int tile_begin;
		const int n_tiles = item_tiles(item, tile_begin);
		const int qtile = item % n_qtiles, split = item / n_qtiles;
		asm volatile("cp.async.wait_all;" ::: "memory");
		asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); // generic-proxy writes -> visible to the tensor core's async proxy
		// every copy of this warpgroup into buffer `buf` has landed, and every warp is past the MMAs of the previous item, which read
		// the other buffer: that one can take the next item's queries
		wg_bar_sync(1 + c);
		const int next = item + static_cast<int>(gridDim.x);
		if (next < n_items) prefetch(next % n_qtiles, buf ^ 1);
		const unsigned char * sAq = sA + buf * kTcABytes;
		const uint32_t a_base = smem_u32(sAq) + static_cast<uint32_t>(c * 64 * kTcRowBytes);
		// Within a query row pa is a constant: during the item the running keys carry the distance minus pa, plus 256 (in [0, 512]),
		// ((pw - 2 c + 256) << 22) | row, and pa - 256 is added back when they are written out.
		uint32_t k1[2] = {kKeyNone, kKeyNone}, k2[2] = {kKeyNone, kKeyNone};
		for (int t = 0; t < n_tiles; ++t, ++g)
		{
			const int s = g % kTcStages;
			mbar_wait(&full[s], (g / kTcStages) & 1);
			__syncwarp(); // wgmma is .aligned: the warp issues it converged
			const unsigned char * stage = sB + s * kTcBBytes;
			// T of this tile and lane quad: uint4 16 hf + 4 k holds the column pairs j = 4 k .. 4 k + 3 of half-tile hf
			const uint4 * sT = reinterpret_cast<const uint4 *>(stage + kTcWordBytes) + quad;
			const int row0 = (tile_begin + t) * kTcBN;
			const int valid = n_rows - row0; // columns of this tile that are real words (>= 1)
			const bool full_tile = valid >= kTcBN;
			// Branch-free top-2 of a full tile over this thread's 64 columns of each of its two rows with 16-bit keys, two columns per
			// register, carried across both half-tiles:
			//   key16 = 64 (pw - 2 c + 256) + lc = c * (-128) + T   (pw - 2 c + 256 = hamming - pa + 256 lies in [0, 512], lc < 64)
			// The low half-word carries fragment column i = j / 2 of the half, the high half-word column i + 8; S = c_hi * 65536 + c_lo
			// and K = S * (-128) + T is that pair of keys exactly (every field stays in [0, 65536), so no carry crosses the halves).
			// Two IMADs (FMA pipe) and three VIMNMX.U16x2 (ALU pipe) per column pair; T is shared by both rows.
			uint32_t p1[2] = {0xFFFFFFFFu, 0xFFFFFFFFu}, p2[2] = {0xFFFFFFFFu, 0xFFFFFFFFu};
#pragma unroll
			for (int hf = 0; hf < 2; ++hf)
			{
				if (hf * kTcHalfN >= valid) break; // no real word in this half of the last tile
				wg_fence();
				wg_mma_b1(acc, wg_smem_desc_noswz(a_base), wg_smem_desc_noswz(smem_u32(stage) + hf * kTcHalfBytes));
				wg_commit();
				wg_wait_all();
				if (full_tile)
				{
#pragma unroll
					for (int k = 0; k < 4; ++k)
					{
						const uint4 t4 = sT[16 * hf + 4 * k];
						const uint32_t tv[4] = {t4.x, t4.y, t4.z, t4.w};
#pragma unroll
						for (int e = 0; e < 4; ++e)
						{
							const int j = 4 * k + e;
#pragma unroll
							for (int h = 0; h < 2; ++h)
							{
								const int lo = 4 * (j >> 1) + 2 * h + (j & 1); // fragment column i = j / 2; column i + 8 is lo + 32
								const uint32_t sp = static_cast<uint32_t>(acc[lo + 32]) * 65536u + static_cast<uint32_t>(acc[lo]);
								const uint32_t kp = sp * neg128 + tv[e];
								const uint32_t mx = __vmaxu2(p1[h], kp);
								p1[h] = __vminu2(p1[h], kp);
								p2[h] = __vminu2(p2[h], mx);
							}
						}
					}
				}
				else
				{
					// last, partly filled tile: plain insertion of the real columns of this half, pw - 2 c + 256 read back from T
					const uint32_t * sT32 = reinterpret_cast<const uint32_t *>(sT) + 64 * hf;
#pragma unroll
					for (int h = 0; h < 2; ++h)
					{
#pragma unroll
						for (int m = 0; m < 32; ++m)
						{
							const int col = kTcHalfN * hf + 8 * (m >> 1) + 2 * quad + (m & 1);
							if (col < valid)
							{
								const int j = m & 15;
								const uint32_t tj = sT32[16 * (j >> 2) + (j & 3)];
								const int pw256 = static_cast<int>(((m < 16 ? tj : tj >> 16) & 0xFFFFu) >> 6);
								const int d = pw256 - 2 * acc[4 * (m >> 1) + 2 * h + (m & 1)];
								const uint32_t key = (static_cast<uint32_t>(d) << kKeyShift) + static_cast<uint32_t>(row_offset + row0 + col);
								top2_insert(k1[h], k2[h], key);
							}
						}
					}
				}
			}
			if (full_tile)
			{
#pragma unroll
				for (int h = 0; h < 2; ++h)
				{
					// the four survivors (two per half-word) go into the running keys only if they can improve them (an empty k2 reads
					// as 1023, above every distance)
					const uint32_t best16 = min(p1[h] & 0xFFFFu, p1[h] >> 16);
					if ((best16 >> 6) < (k2[h] >> kKeyShift))
					{
						const uint32_t base = static_cast<uint32_t>(row_offset + row0 + 2 * quad);
						const uint32_t cand[4] = {p1[h] & 0xFFFFu, p2[h] & 0xFFFFu, p1[h] >> 16, p2[h] >> 16};
#pragma unroll
						for (int u = 0; u < 4; ++u)
						{
							const uint32_t lc = cand[u] & 63u; // local column -> tile column 8 (lc / 2) + 2 quad + lc % 2
							const uint32_t key = ((cand[u] >> 6) << kKeyShift) + base + 8u * (lc >> 1) + (lc & 1u);
							top2_insert(k1[h], k2[h], key);
						}
					}
				}
			}
			// the stage (rows and T) is free once every consumer warp's epilogue has read T
			__syncwarp();
			if (lane == 0) mbar_arrive(&empty[s]);
		}
#pragma unroll
		for (int h = 0; h < 2; ++h)
		{
			const int qi = qtile * kTcBM + r_lo + 8 * h;
			const uint4 x = *reinterpret_cast<const uint4 *>(sAq + tc_chunk_off(r_lo + 8 * h, 0));
			const uint4 y = *reinterpret_cast<const uint4 *>(sAq + tc_chunk_off(r_lo + 8 * h, 1));
			const uint32_t pa = __popc(x.x) + __popc(x.y) + __popc(x.z) + __popc(x.w) + __popc(y.x) + __popc(y.y) + __popc(y.z) + __popc(y.w);
			const uint32_t bias = (pa - 256u) << kKeyShift; // turns pw - 2 c + 256 into pa + pw - 2 c = hamming
			if (qi < nq)
				partial[(static_cast<size_t>(split) * kTcEpiGroups + quad) * nq + qi] =
					make_uint2(k1[h] == kKeyNone ? kKeyNone : k1[h] + bias, k2[h] == kKeyNone ? kKeyNone : k2[h] + bias);
		}
	}
}

} // namespace lcd
