// limit.cuh — the keypoint split of Memory::createSignature (corelib/src/Memory.cpp:5945-6100) on the device.
//
// A frame keeps every detected keypoint (registration matches them all), but only the Kp/MaxFeatures strongest are quantised:
//   * bad-signature gate (:5945-5947, :6051-6058): a frame with fewer than int(Kp/BadSignRatio * meanWordsPerLocation) keypoints
//     quantises nothing;
//   * Feature2D::limitKeypoints(keypoints, inliers, Kp/MaxFeatures) (Features2d.cpp:412-477) flags the strongest, and only the flagged
//     rows go to addNewWords, in ascending keypoint order (quantizedToRawIndices, Memory.cpp:5954-6048);
//   * every other keypoint gets a negative word id: -1, -2, ... in keypoint order (:6070-6100).
#pragma once
#include "orb.cuh"
#include "resolve.cuh"

namespace lcd {

constexpr int kLimitThreads = 1024;

// One CTA per frame: n = n_in[frame] rows of kp / desc [cap] are split.  gate: the host-computed int(ratio * mean_words) (0 = none);
// max_features <= 0 or n <= max_features: every row is quantised.  Writes the quantised rows in ascending keypoint order to
// desc_out [k][row_words] (zeros past the frame's count: padding rows feed the 2-NN), their keypoint index to index_out [k] (-1 past
// the count) and the count to n_out.  Dynamic shared memory: 8 bytes per row of the padded power of two >= cap.
__global__ void __launch_bounds__(kLimitThreads)
limit_keypoints_kernel(const OrbKeypoint * __restrict__ kp, const int * __restrict__ n_in, const uint32_t * __restrict__ desc, int cap, int row_words,
                       int max_features, int k, int gate, uint32_t * __restrict__ desc_out, int * __restrict__ index_out, int * __restrict__ n_out)
{
	extern __shared__ __align__(16) unsigned char smem_raw[];
	unsigned long long * skey = reinterpret_cast<unsigned long long *>(smem_raw); // [pad] sort keys, then int s_idx[k]
	int * s_idx = reinterpret_cast<int *>(smem_raw);
	__shared__ unsigned char s_flag[kMaxFrameQueries];
	__shared__ int s_warp[32];
	const int frame = blockIdx.x, tid = threadIdx.x;
	const int n = min(max(n_in[frame], 0), cap);
	const bool all = max_features <= 0 || n <= max_features;
	const int q = n < gate ? 0 : (all ? n : min(max_features, k));
	if (q > 0 && !all)
	{
		int pad = 1;
		while (pad < n) pad <<= 1;
		const OrbKeypoint * fk = kp + static_cast<size_t>(frame) * cap;
		for (int i = tid; i < pad; i += blockDim.x) skey[i] = i < n ? limit_key(fk[i].response, i) : 0ull;
		for (int i = tid; i < n; i += blockDim.x) s_flag[i] = 0;
		block_sort_desc(skey, pad);
		for (int r = tid; r < q; r += blockDim.x) s_flag[limit_key_index(skey[r])] = 1;
		__syncthreads(); // the keys are dead from here on: s_idx reuses their space
		// block exclusive scan of the flags: each thread owns `per` consecutive keypoints
		const int per = (n + blockDim.x - 1) / blockDim.x, i0 = min(tid * per, n), i1 = min(i0 + per, n);
		int cnt = 0;
		for (int i = i0; i < i1; ++i) cnt += s_flag[i];
		const int lane = tid & 31, warp = tid >> 5, n_warps = blockDim.x >> 5;
		int x = cnt;
		for (int o = 1; o < 32; o <<= 1)
		{
			const int y = __shfl_up_sync(0xFFFFFFFFu, x, o);
			if (lane >= o) x += y;
		}
		if (lane == 31) s_warp[warp] = x;
		__syncthreads();
		if (warp == 0)
		{
			int w = lane < n_warps ? s_warp[lane] : 0;
			for (int o = 1; o < 32; o <<= 1)
			{
				const int y = __shfl_up_sync(0xFFFFFFFFu, w, o);
				if (lane >= o) w += y;
			}
			s_warp[lane] = w;
		}
		__syncthreads();
		int pos = x - cnt + (warp > 0 ? s_warp[warp - 1] : 0);
		for (int i = i0; i < i1; ++i)
			if (s_flag[i]) s_idx[pos++] = i;
	}
	else
	{
		for (int r = tid; r < q; r += blockDim.x) s_idx[r] = r;
	}
	__syncthreads();
	const size_t f = static_cast<size_t>(frame);
	for (int r = tid; r < k; r += blockDim.x) index_out[f * k + r] = r < q ? s_idx[r] : -1;
	const uint32_t * fd = desc + f * cap * row_words;
	uint32_t * od = desc_out + f * k * row_words;
	for (int t = tid; t < k * row_words; t += blockDim.x)
	{
		const int r = t / row_words;
		od[t] = r < q ? fd[static_cast<size_t>(s_idx[r]) * row_words + (t - r * row_words)] : 0u;
	}
	if (tid == 0) n_out[frame] = q;
}

// Per-keypoint word ids of a frame from the ids of its quantised rows: words_q [k] (k-strided), index [k] ascending, n_q of them.
// Keypoint i < n takes its row's id when it was quantised, else -(1 + i - (quantised keypoints before i)); rows >= n get 0.
__global__ void word_ids_expand_kernel(int cap, int k, const int * __restrict__ n_in, const int * __restrict__ index, const int * __restrict__ n_q,
                                       const int * __restrict__ words_q, int * __restrict__ words_out)
{
	const int frame = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= cap) return;
	const int n = min(max(n_in[frame], 0), cap);
	const int q = min(max(n_q[frame], 0), min(k, n));
	const int * idx = index + static_cast<size_t>(frame) * k;
	int out = 0;
	if (i < n)
	{
		int lo = 0, hi = q; // lower_bound of i in idx[0, q)
		while (lo < hi)
		{
			const int mid = (lo + hi) >> 1;
			if (idx[mid] < i) lo = mid + 1;
			else hi = mid;
		}
		out = lo < q && idx[lo] == i ? words_q[static_cast<size_t>(frame) * k + lo] : -(1 + i - lo);
	}
	words_out[static_cast<size_t>(frame) * cap + i] = out;
}

} // namespace lcd
