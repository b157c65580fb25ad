// common.cuh — shared device helpers for the loop-closure hot-path kernels (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace lcd {

// Packed nearest-neighbour key: (distance << 22) | global_row.
// Hamming-256 distances need 9 bits, rows 22 bits (< 4 194 304 indexed words), so the
// lexicographic (distance, row) order that rtflann's KNNSimpleResultSet produces when it
// scans rows in ascending order (reference: rtflann/util/result_set.h:151-172, strict '>'
// shift, reject on '>=') is exactly the unsigned order of the packed key.
constexpr int kKeyShift = 22;
constexpr uint32_t kKeyRowMask = (1u << kKeyShift) - 1u;
constexpr uint32_t kKeyNone = 0xFFFFFFFFu;
constexpr int kMaxRowsPacked = 1 << kKeyShift;

__device__ __forceinline__ void top2_insert(uint32_t & k1, uint32_t & k2, uint32_t key)
{
	uint32_t m = max(k1, key);
	k1 = min(k1, key);
	k2 = min(k2, m);
}

__device__ __forceinline__ uint32_t smem_u32(const void * p)
{
	return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ---- mbarrier + 1-D bulk async copy (TMA engine, UBLKCP in SASS) -------------------
__device__ __forceinline__ void mbar_init(uint64_t * bar, uint32_t count)
{
	asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init()
{
	asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t * bar, uint32_t bytes)
{
	asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t * bar, uint32_t phase)
{
	asm volatile(
		"{\n"
		".reg .pred p;\n"
		"WAIT_%=:\n"
		"mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
		"@p bra DONE_%=;\n"
		"bra WAIT_%=;\n"
		"DONE_%=:\n"
		"}\n" ::"r"(smem_u32(bar)),
		"r"(phase)
		: "memory");
}
// global -> shared bulk copy, completion signalled on an mbarrier (bytes % 16 == 0,
// both addresses 16-byte aligned).
__device__ __forceinline__ void bulk_g2s(void * smem_dst, const void * gmem_src, uint32_t bytes, uint64_t * bar)
{
	asm volatile(
		"cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem_dst)),
		"l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
		: "memory");
}

} // namespace lcd
