// gmma_rate_probe.cu — issue rate of the two warpgroup MMAs a 256-bit binary descriptor can be matched with on an H100:
//   IGMMA  wgmma m64n256k32  .s32.s8.s8          (one k32 step of the +-1 byte encoding; 8 per 256-bit descriptor)
//   BGMMA  wgmma m64n256k256 .s32.b1.b1.and.popc (the whole 256-bit descriptor at once)
// One persistent CTA per SM; each of its two warpgroups issues a long chain of back-to-back MMAs on shared-memory operands (their
// contents do not matter: zeros) and times it with clock64.  Prints cycles per instruction per SM, the rate that implies at the SM
// clock measured over the same run, and the card's name, power limit and clocks.
// It also times ONE BGMMA issued, committed and waited for by a lone warpgroup: what a consumer warpgroup of the 2-NN kernel
// (nn_tensor.cuh) waits per word tile before its epilogue can start.
//   nvcc -gencode arch=compute_90a,code=sm_90a -o /tmp/gmma_rate_probe tools/gmma_rate_probe.cu -ldl && /tmp/gmma_rate_probe
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <vector>

constexpr int kWarpgroups = 2;
constexpr int kBatch = 16;    // MMAs per commit group
constexpr int kBatches = 512; // per warpgroup and timed chain

__device__ __forceinline__ uint32_t s32(const void * p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

// K-major, no swizzle, 32-byte rows (k32 of s8 and k256 of b1 are both 32 bytes): 8 x 16-byte core matrices, the two along K
// 128 B apart, 8-row groups 256 B apart
__device__ __forceinline__ uint64_t desc32(uint32_t saddr)
{
	return static_cast<uint64_t>((saddr & 0x3FFFFu) >> 4) | (static_cast<uint64_t>(128 >> 4) << 16) | (static_cast<uint64_t>(256 >> 4) << 32);
}

#define ACC128                                                                                                                          \
	"{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, "    \
	"%27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, " \
	"%53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, " \
	"%79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, " \
	"%104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, "    \
	"%125, %126, %127}"
#define R8(i) "+r"(d[i]), "+r"(d[i + 1]), "+r"(d[i + 2]), "+r"(d[i + 3]), "+r"(d[i + 4]), "+r"(d[i + 5]), "+r"(d[i + 6]), "+r"(d[i + 7])
#define OUT128 R8(0), R8(8), R8(16), R8(24), R8(32), R8(40), R8(48), R8(56), R8(64), R8(72), R8(80), R8(88), R8(96), R8(104), R8(112), R8(120)

template <bool kBinary>
__device__ __forceinline__ void mma(int (&d)[128], uint64_t a, uint64_t b)
{
	if (kBinary)
		asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, 1, 0;\n"
		             "wgmma.mma_async.sync.aligned.m64n256k256.s32.b1.b1.and.popc " ACC128 ", %128, %129, p;\n}\n"
		             : OUT128 : "l"(a), "l"(b) : "memory");
	else
		asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, 1, 0;\n"
		             "wgmma.mma_async.sync.aligned.m64n256k32.s32.s8.s8 " ACC128 ", %128, %129, p;\n}\n"
		             : OUT128 : "l"(a), "l"(b) : "memory");
}

template <bool kBinary>
__global__ void __launch_bounds__(128 * kWarpgroups, 1) chain(long long * cycles, int * sink)
{
	__shared__ __align__(1024) unsigned char sA[kWarpgroups][64 * 32];
	__shared__ __align__(1024) unsigned char sB[256 * 32];
	for (int i = threadIdx.x; i < static_cast<int>(sizeof(sA) / 4); i += blockDim.x) reinterpret_cast<uint32_t *>(sA)[i] = 0;
	for (int i = threadIdx.x; i < static_cast<int>(sizeof(sB) / 4); i += blockDim.x) reinterpret_cast<uint32_t *>(sB)[i] = 0;
	asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
	__syncthreads();
	const int wg = threadIdx.x >> 7;
	const uint64_t a = desc32(s32(sA[wg])), b = desc32(s32(sB));
	int d[128];
#pragma unroll
	for (int i = 0; i < 128; ++i) d[i] = 0;
	__syncthreads();
	const long long t0 = clock64();
	for (int it = 0; it < kBatches; ++it)
	{
		asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
#pragma unroll
		for (int k = 0; k < kBatch; ++k) mma<kBinary>(d, a, b);
		asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
		asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
	}
	const long long t1 = clock64();
	__shared__ long long span[kWarpgroups];
	if ((threadIdx.x & 127) == 0) span[wg] = t1 - t0;
	int s = 0;
#pragma unroll
	for (int i = 0; i < 128; ++i) s += d[i];
	if (s != 0) sink[blockIdx.x] = s; // zeros in, zeros out: keeps the chain live without a store per thread
	__syncthreads();
	if (threadIdx.x == 0)
	{
		long long m = 0;
		for (int w = 0; w < kWarpgroups; ++w) m = span[w] > m ? span[w] : m;
		cycles[blockIdx.x] = m;
	}
}

// one warpgroup per SM: fence, one BGMMA, commit, wait — kIters times
constexpr int kIters = 2048;
__global__ void __launch_bounds__(128, 1) latency(long long * cycles, int * sink)
{
	__shared__ __align__(1024) unsigned char sA[64 * 32];
	__shared__ __align__(1024) unsigned char sB[256 * 32];
	for (int i = threadIdx.x; i < static_cast<int>(sizeof(sA) / 4); i += blockDim.x) reinterpret_cast<uint32_t *>(sA)[i] = 0;
	for (int i = threadIdx.x; i < static_cast<int>(sizeof(sB) / 4); i += blockDim.x) reinterpret_cast<uint32_t *>(sB)[i] = 0;
	asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
	__syncthreads();
	const uint64_t a = desc32(s32(sA)), b = desc32(s32(sB));
	int d[128];
#pragma unroll
	for (int i = 0; i < 128; ++i) d[i] = 0;
	const long long t0 = clock64();
	for (int it = 0; it < kIters; ++it)
	{
		asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
		mma<true>(d, a, b);
		asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
		asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
	}
	const long long t1 = clock64();
	int s = 0;
#pragma unroll
	for (int i = 0; i < 128; ++i) s += d[i];
	if (s != 0) sink[blockIdx.x] = s;
	if (threadIdx.x == 0) cycles[blockIdx.x] = t1 - t0;
}

static void run_latency(const char * name, int sms)
{
	long long * d_cycles;
	int * d_sink;
	cudaMalloc(&d_cycles, sms * sizeof(long long));
	cudaMalloc(&d_sink, sms * sizeof(int));
	for (int rep = 0; rep < 2; ++rep) latency<<<sms, 128>>>(d_cycles, d_sink); // first launch: warm-up
	const cudaError_t err = cudaDeviceSynchronize();
	if (err != cudaSuccess) { printf("%s: %s\n", name, cudaGetErrorString(err)); return; }
	std::vector<long long> c(sms);
	cudaMemcpy(c.data(), d_cycles, sms * sizeof(long long), cudaMemcpyDeviceToHost);
	std::sort(c.begin(), c.end());
	printf("%-58s cycles per BGMMA: median %.1f (min %.1f, max %.1f)\n", name, c[sms / 2] / double(kIters), c[0] / double(kIters),
	       c[sms - 1] / double(kIters));
	cudaFree(d_cycles);
	cudaFree(d_sink);
}

typedef int (*NvmlInit)();
typedef int (*NvmlHandle)(unsigned, void **);
typedef int (*NvmlUint)(void *, unsigned *);
typedef int (*NvmlClock)(void *, int, unsigned *);

static void print_card()
{
	cudaDeviceProp p;
	cudaGetDeviceProperties(&p, 0);
	int clk_khz = 0;
	cudaDeviceGetAttribute(&clk_khz, cudaDevAttrClockRate, 0);
	printf("device: %s, %d SMs, max SM clock %d MHz (CUDA attribute)\n", p.name, p.multiProcessorCount, clk_khz / 1000);
	void * h = dlopen("libnvidia-ml.so.1", RTLD_NOW);
	if (!h) { printf("NVML not available: power limit not read\n"); return; }
	auto init = reinterpret_cast<NvmlInit>(dlsym(h, "nvmlInit_v2"));
	auto handle = reinterpret_cast<NvmlHandle>(dlsym(h, "nvmlDeviceGetHandleByIndex_v2"));
	auto limit = reinterpret_cast<NvmlUint>(dlsym(h, "nvmlDeviceGetPowerManagementLimit"));
	auto clock = reinterpret_cast<NvmlClock>(dlsym(h, "nvmlDeviceGetClockInfo"));
	auto maxclock = reinterpret_cast<NvmlClock>(dlsym(h, "nvmlDeviceGetMaxClockInfo"));
	void * dev = nullptr;
	unsigned mw = 0, sm = 0, smmax = 0;
	if (init && handle && init() == 0 && handle(0, &dev) == 0)
	{
		if (limit && limit(dev, &mw) == 0) printf("power limit: %.0f W\n", mw / 1000.0);
		if (clock && clock(dev, 1 /* NVML_CLOCK_SM */, &sm) == 0 && maxclock && maxclock(dev, 1, &smmax) == 0)
			printf("SM clock now: %u MHz, max %u MHz (NVML)\n", sm, smmax);
	}
	dlclose(h);
}

template <bool kBinary>
static void run(const char * name, double ops_per_inst, int sms)
{
	long long * d_cycles;
	int * d_sink;
	cudaMalloc(&d_cycles, sms * sizeof(long long));
	cudaMalloc(&d_sink, sms * sizeof(int));
	chain<kBinary><<<sms, 128 * kWarpgroups>>>(d_cycles, d_sink); // warm-up: module load, clocks up
	cudaEvent_t e0, e1;
	cudaEventCreate(&e0);
	cudaEventCreate(&e1);
	cudaEventRecord(e0);
	chain<kBinary><<<sms, 128 * kWarpgroups>>>(d_cycles, d_sink);
	cudaEventRecord(e1);
	const cudaError_t err = cudaDeviceSynchronize();
	if (err != cudaSuccess) { printf("%s: %s\n", name, cudaGetErrorString(err)); return; }
	float ms = 0.0f;
	cudaEventElapsedTime(&ms, e0, e1);
	std::vector<long long> c(sms);
	cudaMemcpy(c.data(), d_cycles, sms * sizeof(long long), cudaMemcpyDeviceToHost);
	std::sort(c.begin(), c.end());
	const double n_inst = static_cast<double>(kWarpgroups) * kBatch * kBatches; // per SM
	const double med = static_cast<double>(c[sms / 2]);
	const double mhz = static_cast<double>(c[sms - 1]) / (ms * 1e3);            // slowest SM's cycles over the launch's wall time
	printf("%-40s cycles/instruction per SM: median %.1f (min %.1f, max %.1f); launch %.3f ms, SM clock over the chain >= %.0f MHz, "
	       "%.0f T ops/s at that clock\n",
	       name, med / n_inst, c[0] / n_inst, c[sms - 1] / n_inst, ms, mhz, ops_per_inst * n_inst / (med / (mhz * 1e6)) * sms / 1e12);
	cudaFree(d_cycles);
	cudaFree(d_sink);
}

int main()
{
	print_card();
	int sms = 0;
	cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
	run<false>("IGMMA m64n256k32 .s8 (2*64*256*32 ops)", 2.0 * 64 * 256 * 32, sms);
	run<true>("BGMMA m64n256k256 .b1.and.popc (bit ops)", 2.0 * 64 * 256 * 256, sms);
	run_latency("one BGMMA issued + waited by a lone warpgroup (latency)", sms);
	print_card();
	return 0;
}
