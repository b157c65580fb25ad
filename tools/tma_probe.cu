// tma_probe.cu — diagnostic: which way of handing a CUtensorMap to cp.async.bulk.tensor works on this driver / GPU.
//   nvcc -gencode arch=compute_90a,code=sm_90a -o /tmp/tma_probe tools/tma_probe.cu && /tmp/tma_probe
#include <cuda.h>
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdint>
#include <vector>

struct alignas(64) TMap { unsigned long long o[16]; };
__constant__ TMap c_map;

__device__ __forceinline__ uint32_t s32(const void * p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

__device__ void load_tile(const void * tmap, uint8_t * s_tile, uint64_t * bar, int x, int y, int z, int bytes)
{
	if (threadIdx.x == 0)
	{
		asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(s32(bar)) : "memory");
		asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
	}
	__syncthreads();
	if (threadIdx.x == 0)
	{
		asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(s32(bar)), "r"(bytes) : "memory");
		asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];" ::"r"(s32(s_tile)),
		             "l"(tmap), "r"(x), "r"(y), "r"(z), "r"(s32(bar))
		             : "memory");
	}
	asm volatile("{\n.reg .pred p;\nW: mbarrier.try_wait.parity.shared::cta.b64 p, [%0], 0;\n@p bra D;\nbra W;\nD:\n}\n" ::"r"(s32(bar)) : "memory");
}

template <int BW, int BH>
__global__ void k_param(const __grid_constant__ TMap tmap, int x, int y, int z, uint8_t * out)
{
	__shared__ __align__(128) uint8_t s_tile[BW * BH];
	__shared__ __align__(8) uint64_t bar;
	load_tile(&tmap, s_tile, &bar, x, y, z, BW * BH);
	for (int i = threadIdx.x; i < BW * BH; i += blockDim.x) out[i] = s_tile[i];
}
template <int BW, int BH>
__global__ void k_global(const TMap * tmap, int x, int y, int z, uint8_t * out)
{
	__shared__ __align__(128) uint8_t s_tile[BW * BH];
	__shared__ __align__(8) uint64_t bar;
	load_tile(tmap, s_tile, &bar, x, y, z, BW * BH);
	for (int i = threadIdx.x; i < BW * BH; i += blockDim.x) out[i] = s_tile[i];
}
template <int BW, int BH>
__global__ void k_const(int x, int y, int z, uint8_t * out)
{
	__shared__ __align__(128) uint8_t s_tile[BW * BH];
	__shared__ __align__(8) uint64_t bar;
	load_tile(&c_map, s_tile, &bar, x, y, z, BW * BH);
	for (int i = threadIdx.x; i < BW * BH; i += blockDim.x) out[i] = s_tile[i];
}

typedef CUresult (*Enc)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *, const cuuint32_t *, const cuuint32_t *,
                        CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

template <int BW, int BH>
void run(Enc enc, uint8_t * d_img, const std::vector<uint8_t> & h, int w, int hgt, int nf, int x, int y, int z)
{
	TMap tm;
	const cuuint64_t dims[3] = {(cuuint64_t)w, (cuuint64_t)hgt, (cuuint64_t)nf};
	const cuuint64_t str[2] = {(cuuint64_t)w, (cuuint64_t)w * hgt};
	const cuuint32_t box[3] = {BW, BH, 1};
	const cuuint32_t es[3] = {1, 1, 1};
	CUresult r = enc((CUtensorMap *)&tm, CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, d_img, dims, str, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
	                 CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
	printf("box %dx%d at (%d,%d,%d): encode rc=%d\n", BW, BH, x, y, z, (int)r);
	if (r != CUDA_SUCCESS) return;
	uint8_t * d_out;
	cudaMalloc(&d_out, BW * BH);
	std::vector<uint8_t> o(BW * BH);
	auto check = [&](const char * name) {
		cudaError_t e = cudaDeviceSynchronize();
		if (e != cudaSuccess)
		{
			printf("  %-8s FAILED: %s\n", name, cudaGetErrorString(e));
			return false;
		}
		cudaMemcpy(o.data(), d_out, BW * BH, cudaMemcpyDeviceToHost);
		int bad = 0;
		for (int r2 = 0; r2 < BH; ++r2)
			for (int c = 0; c < BW; ++c)
			{
				const int gx = x + c, gy = y + r2;
				const uint8_t want = (gx >= 0 && gx < w && gy >= 0 && gy < hgt) ? h[(size_t)z * w * hgt + (size_t)gy * w + gx] : 0;
				bad += o[r2 * BW + c] != want;
			}
		printf("  %-8s ok, %d wrong bytes\n", name, bad);
		return true;
	};
	k_param<BW, BH><<<1, 128>>>(tm, x, y, z, d_out);
	if (!check("param")) return;
	TMap * d_map;
	cudaMalloc(&d_map, sizeof(TMap));
	cudaMemcpy(d_map, &tm, sizeof(TMap), cudaMemcpyHostToDevice);
	k_global<BW, BH><<<1, 128>>>(d_map, x, y, z, d_out);
	if (!check("global")) return;
	cudaMemcpyToSymbol(c_map, &tm, sizeof(TMap));
	k_const<BW, BH><<<1, 128>>>(x, y, z, d_out);
	check("constant");
}

int main()
{
	void * p = nullptr;
	cudaDriverEntryPointQueryResult q;
	cudaFree(0);
	if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || !p) { printf("no encoder\n"); return 1; }
	Enc enc = (Enc)p;
	const int w = 320, h = 240, nf = 2;
	std::vector<uint8_t> img((size_t)w * h * nf);
	for (size_t i = 0; i < img.size(); ++i) img[i] = (uint8_t)(i * 131 + (i >> 8));
	uint8_t * d_img;
	cudaMalloc(&d_img, img.size());
	cudaMemcpy(d_img, img.data(), img.size(), cudaMemcpyHostToDevice);
	run<64, 32>(enc, d_img, img, w, h, nf, 64, 32, 0);
	run<80, 40>(enc, d_img, img, w, h, nf, 56, 28, 1);
	run<80, 40>(enc, d_img, img, w, h, nf, -8, -4, 0);
	run<80, 40>(enc, d_img, img, w, h, nf, 248, 220, 1);
	run<128, 40>(enc, d_img, img, w, h, nf, 48, 28, 0);
	return 0;
}
