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

// A localisation client's camera as one decision call took it (lcd_clients_set_cameras), one record per frame of the call.  A frame
// whose client has no camera has set = 0 and is computed with the call's parameters.
struct FrameCam
{
	double fx, fy, cx, cy; // CameraModel::K()
	float L[12];           // CameraModel::localTransform(), 3x4 row-major
	int w, h;              // CameraModel::imageSize() (0 x 0 = not set)
	int set;               // 1: the client has a camera
	int local;             // 1: L is not identity (Transform::isIdentity, Transform.cpp:156-170)
};
static_assert(sizeof(FrameCam) == 96, "FrameCam is staged as 12 64-bit words per frame");

// util3d::transformPoint (util3d_transforms.cpp:211-220): float, r0 x + r1 y + r2 z + t, left to right, each operation rounded on its own
__device__ __forceinline__ void transform_point_f(const float * T, float x, float y, float z, float & ox, float & oy, float & oz)
{
	ox = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(T[0], x), __fmul_rn(T[1], y)), __fmul_rn(T[2], z)), T[3]);
	oy = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(T[4], x), __fmul_rn(T[5], y)), __fmul_rn(T[6], z)), T[7]);
	oz = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(T[8], x), __fmul_rn(T[9], y)), __fmul_rn(T[10], z)), T[11]);
}

// rtabmap::Transform A * B of two 3x4 float transforms (Eigen's 4x4 product, the implicit last row 0 0 0 1), left to right
__device__ __forceinline__ void transform_mul_f(const float * A, const float * B, float * out)
{
	for (int i = 0; i < 3; ++i)
		for (int j = 0; j < 4; ++j)
		{
			float v = __fadd_rn(__fadd_rn(__fmul_rn(A[4 * i], B[j]), __fmul_rn(A[4 * i + 1], B[4 + j])), __fmul_rn(A[4 * i + 2], B[8 + j]));
			if (j == 3) v = __fadd_rn(v, A[4 * i + 3]);
			out[4 * i + j] = v;
		}
}

// the inverse of a rigid 3x4 float transform as [R^T | -R^T t]
__device__ __forceinline__ void transform_inv_f(const float * A, float * out)
{
	for (int i = 0; i < 3; ++i)
	{
		for (int j = 0; j < 3; ++j) out[4 * i + j] = A[4 * j + i];
		out[4 * i + 3] = -__fadd_rn(__fadd_rn(__fmul_rn(A[i], A[3]), __fmul_rn(A[4 + i], A[7])), __fmul_rn(A[8 + i], A[11]));
	}
}

} // namespace lcd
