// epipolar.cuh — EpipolarGeometry::check (corelib/src/EpipolarGeometry.cpp:65-102) of (new, old) signature pairs, one CTA per pair.
//
//   pairs      findPairsUnique (EpipolarGeometry.h:157-186): the word ids >= 0 found exactly once on each side, in ascending id order,
//              each side's (id, row) keys sorted in shared memory and merge-joined; row i of a side is word i and keypoint i
//   F          cv::findFundamentalMat(FM_RANSAC, VhEp/RansacParam1, VhEp/RansacParam2) as OpenCV 4.13 runs it (findFFromWords,
//              :298-379): 7 points -> the 7-point kernel alone, mask all ones; 8-14 -> LMeDS; >= 15 -> RANSAC with 7-point samples,
//              maxIters 1000.  The registrators are the vendored OpenCV-3 ones (opencv/solvepnp.cpp:213-557).
//
// RANSAC is sequential in the reference, but its samples depend only on the points (cv::RNG((uint64)-1), checkSubset rejects
// collinear samples), so thread 0 draws the samples of a chunk, one thread per sample runs the 7-point solver in fp64 (up to three
// models each), the CTA counts the inliers of every model, and thread 0 replays the strict-best / adaptive-niters bookkeeping in
// iteration and model order.  LMeDS (at most 14 points) has each sample's thread compute its models' medians itself.
// The fundamental-matrix arithmetic is fm_solver.h, which the CPU oracle compiles too: both compute the same bits.
#pragma once
#include "common.cuh"
#include "fm_solver.h"
#include "ransac.cuh"

namespace lcd {

constexpr int kEpiThreads = 256;
constexpr int kEpiChunk = 128; // samples per chunk (one thread each for the 7-point solver)
constexpr int kEpiMaxIters = 1000;

struct EpiArgs
{
	const int * ids_a;   // [n_pairs][cap]  new frame
	const float * uv_a;  // [n_pairs][cap][2]
	const int * n_a;     // [n_pairs]
	const int * ids_b;   // [n_pairs][cap]  hypothesis
	const float * uv_b;  // [n_pairs][cap][2]
	const int * n_b;     // [n_b rows]
	const int * slot_b;  // nullptr: B row = pair; else the B row of each pair (-1: a signature without words)
	const int * skip;    // nullptr, or [n_pairs] nonzero: the pair is not checked (checked = 0)
	int cap_a, cap_b;
	int match_count_min;
	double thr, conf;    // after findFundamentalMat's resets
	int * res;           // [n_pairs][8] checked, ok, n_pairs, n_inliers, method, found, iterations_run, raised
	double * F;          // [n_pairs][9]
	uint8_t * status;    // [n_pairs][status_cap] in pair order, or nullptr
	int status_cap;
};

__host__ __device__ inline size_t epi_smem_bytes(int cap)
{
	int p2 = 1;
	while (p2 < cap) p2 <<= 1;
	return static_cast<size_t>(p2) * 2 * sizeof(unsigned long long) + static_cast<size_t>(cap) * 2 * sizeof(FmPt) +
	       kEpiChunk * (27 * sizeof(double) + 3 * sizeof(double) + 3 * sizeof(int) + sizeof(int) + 7 * sizeof(uint16_t)) + 256 * sizeof(int) + 64;
}


// ascending (id, row) keys; the sign bit is flipped so that negative ids sort first as unsigned
__device__ inline void epi_sort_keys(unsigned long long * k, int p2)
{
	for (int size = 2; size <= p2; size <<= 1)
		for (int stride = size >> 1; stride > 0; stride >>= 1)
		{
			__syncthreads();
			for (int i = threadIdx.x; i < p2; i += blockDim.x)
			{
				const int j = i ^ stride;
				if (j > i)
				{
					const bool up = (i & size) == 0;
					const unsigned long long x = k[i], y = k[j];
					if ((x > y) == up)
					{
						k[i] = y;
						k[j] = x;
					}
				}
			}
		}
	__syncthreads();
}

__device__ inline int epi_key_id(unsigned long long k) { return static_cast<int>(static_cast<unsigned>(k >> 32) ^ 0x80000000u); }

__global__ void __launch_bounds__(kEpiThreads) epipolar_check_kernel(const EpiArgs a)
{
	extern __shared__ __align__(16) unsigned char smem_raw[];
	const int cap = max(a.cap_a, a.cap_b);
	int p2 = 1;
	while (p2 < cap) p2 <<= 1;
	unsigned long long * kA = reinterpret_cast<unsigned long long *>(smem_raw);
	unsigned long long * kB = kA + p2;
	FmPt * P1 = reinterpret_cast<FmPt *>(kB + p2);
	FmPt * P2 = P1 + cap;
	double * models = reinterpret_cast<double *>(P2 + cap);   // [kEpiChunk][27]
	double * meds = models + kEpiChunk * 27;                 // [kEpiChunk][3] LMeDS medians
	int * cnt = reinterpret_cast<int *>(meds + kEpiChunk * 3); // [kEpiChunk][3] RANSAC inlier counts
	int * nmod = cnt + kEpiChunk * 3;                          // [kEpiChunk]
	int * scan = nmod + kEpiChunk;                             // [256]
	uint16_t * sidx = reinterpret_cast<uint16_t *>(scan + 256); // [kEpiChunk][7]
	__shared__ double s_best[9];
	__shared__ double s_min_median;
	__shared__ int s_np, s_niters, s_max_good, s_draw_end, s_fail_at, s_done, s_raised, s_iters, s_have_best, s_total;
	__shared__ unsigned long long s_rng;

	const int tid = threadIdx.x, pair = blockIdx.x;
	int * res = a.res + pair * 8;
	if (tid < 8) res[tid] = 0;
	if (tid < 9) a.F[pair * 9 + tid] = 0.;
	if (a.skip && a.skip[pair]) return;
	const int na = min(max(a.n_a[pair], 0), a.cap_a);
	const int slot = a.slot_b ? a.slot_b[pair] : pair;
	const int nb = slot < 0 ? 0 : min(max(a.n_b[slot], 0), a.cap_b);
	if (a.status)
		for (int i = tid; i < a.status_cap; i += blockDim.x) a.status[static_cast<size_t>(pair) * a.status_cap + i] = 0;

	// ---- findPairsUnique
	const int * ida = a.ids_a + static_cast<size_t>(pair) * a.cap_a;
	const int * idb = a.ids_b + static_cast<size_t>(max(slot, 0)) * a.cap_b;
	for (int i = tid; i < p2; i += blockDim.x)
	{
		kA[i] = i < na ? (static_cast<unsigned long long>(static_cast<unsigned>(ida[i]) ^ 0x80000000u) << 32) | static_cast<unsigned>(i) : ~0ull;
		kB[i] = i < nb ? (static_cast<unsigned long long>(static_cast<unsigned>(idb[i]) ^ 0x80000000u) << 32) | static_cast<unsigned>(i) : ~0ull;
	}
	epi_sort_keys(kA, p2);
	epi_sort_keys(kB, p2);
	// each thread takes a contiguous run of A's sorted keys, so the pairs come out in ascending id order after a scan of the counts
	const int per = (na + blockDim.x - 1) / blockDim.x;
	const int i0 = min(tid * per, na), i1 = min(i0 + per, na);
	auto match = [&](int i) -> int {
		const int id = epi_key_id(kA[i]);
		if (id < 0 || (i > 0 && epi_key_id(kA[i - 1]) == id) || (i + 1 < na && epi_key_id(kA[i + 1]) == id)) return -1;
		int lo = 0, hi = nb;
		while (lo < hi)
		{
			const int mid = (lo + hi) >> 1;
			if (epi_key_id(kB[mid]) < id) lo = mid + 1;
			else hi = mid;
		}
		if (lo >= nb || epi_key_id(kB[lo]) != id || (lo + 1 < nb && epi_key_id(kB[lo + 1]) == id)) return -1;
		return lo;
	};
	int c = 0;
	for (int i = i0; i < i1; ++i) c += match(i) >= 0;
	scan[tid] = c;
	__syncthreads();
	if (tid == 0)
	{
		int s = 0;
		for (int t = 0; t < blockDim.x; ++t)
		{
			const int v = scan[t];
			scan[t] = s;
			s += v;
		}
		s_np = s;
	}
	__syncthreads();
	{
		const float * uva = a.uv_a + static_cast<size_t>(pair) * a.cap_a * 2;
		const float * uvb = a.uv_b + static_cast<size_t>(max(slot, 0)) * a.cap_b * 2;
		int o = scan[tid];
		for (int i = i0; i < i1; ++i)
		{
			const int j = match(i);
			if (j < 0) continue;
			const int ra = static_cast<int>(kA[i] & 0xFFFFFFFFu), rb = static_cast<int>(kB[j] & 0xFFFFFFFFu);
			P1[o] = FmPt{uva[2 * ra], uva[2 * ra + 1]};
			P2[o] = FmPt{uvb[2 * rb], uvb[2 * rb + 1]};
			++o;
		}
	}
	__syncthreads();
	const int np = s_np;
	if (tid == 0)
	{
		res[0] = 1;
		res[2] = np;
	}
	if (np < a.match_count_min || np < 7) return;

	// ---- findFundamentalMat
	const int method = np == 7 ? 1 : np < 15 ? 2 : 3;
	if (method == 1)
	{
		if (tid == 0)
		{
			uint16_t idx[7] = {0, 1, 2, 3, 4, 5, 6};
			const int k = fm_run_7point(P1, P2, idx, models);
			res[4] = 1;
			res[7] = k < 0;
			if (k > 0)
			{
				res[5] = 1;
				res[3] = 7;
				res[1] = 7 >= a.match_count_min;
				for (int q = 0; q < 9; ++q) a.F[pair * 9 + q] = models[q];
				if (a.status)
					for (int q = 0; q < 7; ++q) a.status[static_cast<size_t>(pair) * a.status_cap + q] = 1;
			}
		}
		return;
	}
	const bool lmeds = method == 2;
	if (tid == 0)
	{
		s_rng = 0xFFFFFFFFFFFFFFFFull;
		s_niters = lmeds ? max(ransac_update_num_iters(a.conf, 0.45, 7, kEpiMaxIters), 3) : kEpiMaxIters;
		s_max_good = 0;
		s_min_median = 1.7976931348623157e308;
		s_fail_at = -1;
		s_done = 0;
		s_raised = 0;
		s_iters = 0;
		s_have_best = 0;
	}
	__syncthreads();
	const int max_attempts = lmeds ? 1000 : 10000;
	for (int c0 = 0;; c0 += kEpiChunk)
	{
		if (tid == 0)
		{
			// getSubset (checkPartialSubsets = false): 7 distinct indices, redrawn whole while the 7th point of either image is collinear
			// with two earlier ones; a run of max_attempts rejections ends the sampling
			unsigned long long st = s_rng;
			const int end = min(c0 + kEpiChunk, s_niters);
			int it = c0;
			for (; it < end; ++it)
			{
				uint16_t * idx = sidx + (it - c0) * 7;
				int i = 0, iters = 0;
				for (; iters < max_attempts; ++iters)
				{
					for (i = 0; i < 7 && iters < max_attempts;)
					{
						int v;
						for (;;)
						{
							v = cv_rng_uniform(st, np);
							int j;
							for (j = 0; j < i; ++j)
								if (v == idx[j]) break;
							if (j == i) break;
						}
						idx[i++] = static_cast<uint16_t>(v);
					}
					if (i == 7 && (fm_collinear(P1, idx) || fm_collinear(P2, idx))) continue;
					break;
				}
				if (!(i == 7 && iters < max_attempts))
				{
					s_fail_at = it;
					break;
				}
			}
			s_draw_end = it;
			s_rng = st;
		}
		__syncthreads();
		const int draw_end = s_draw_end;
		if (tid < kEpiChunk)
		{
			const int it = c0 + tid;
			int k = 0;
			if (it < draw_end)
			{
				k = fm_run_7point(P1, P2, sidx + tid * 7, models + tid * 27);
				if (lmeds)
					for (int m = 0; m < k; ++m)
					{
						// the median of the errors, sorted as int32 bit patterns (std::sort(errf.ptr<int>(), ...))
						int e[14];
						for (int q = 0; q < np; ++q) e[q] = __float_as_int(fm_error(models + tid * 27 + m * 9, P1[q], P2[q]));
						for (int q = 1; q < np; ++q)
						{
							const int v = e[q];
							int r = q - 1;
							while (r >= 0 && e[r] > v)
							{
								e[r + 1] = e[r];
								--r;
							}
							e[r + 1] = v;
						}
						meds[tid * 3 + m] = np % 2 != 0 ? static_cast<double>(__int_as_float(e[np / 2]))
						                                : static_cast<double>(__fadd_rn(__int_as_float(e[np / 2 - 1]), __int_as_float(e[np / 2]))) * 0.5;
					}
			}
			nmod[tid] = k;
			for (int m = 0; m < 3; ++m) cnt[tid * 3 + m] = 0;
		}
		__syncthreads();
		if (!lmeds)
		{
			// inlier counts: one warp per model
			const float t2 = static_cast<float>(a.thr * a.thr);
			const int warp = tid >> 5, lane = tid & 31;
			for (int slot_m = warp; slot_m < kEpiChunk * 3; slot_m += kEpiThreads / 32)
			{
				const int h = slot_m / 3, m = slot_m % 3;
				if (c0 + h >= draw_end || m >= nmod[h]) continue;
				const double * Fm = models + h * 27 + m * 9;
				int cc = 0;
				for (int q = lane; q < np; q += 32) cc += fm_error(Fm, P1[q], P2[q]) <= t2;
				for (int o = 16; o > 0; o >>= 1) cc += __shfl_down_sync(0xFFFFFFFFu, cc, o);
				if (lane == 0) cnt[slot_m] = cc;
			}
			__syncthreads();
		}
		if (tid == 0)
		{
			int niters = s_niters;
			int it = c0;
			for (; it < c0 + kEpiChunk && it < niters; ++it)
			{
				if (it == s_fail_at)
				{
					s_done = 1;
					break;
				}
				const int h = it - c0, k = nmod[h];
				s_iters = it + 1;
				if (k < 0)
				{
					s_raised = 1; // runKernel copies F.rowRange(0, n*3) for n < 0: OpenCV asserts
					s_done = 1;
					break;
				}
				for (int m = 0; m < k; ++m)
				{
					const double * Fm = models + h * 27 + m * 9;
					bool take;
					if (lmeds)
					{
						take = meds[h * 3 + m] < s_min_median;
						if (take) s_min_median = meds[h * 3 + m];
					}
					else
					{
						const int g = cnt[h * 3 + m];
						take = g > max(s_max_good, 6);
						if (take)
						{
							s_max_good = g;
							niters = ransac_update_num_iters(a.conf, static_cast<double>(np - g) / np, 7, niters);
						}
					}
					if (take)
					{
						s_have_best = 1;
						for (int q = 0; q < 9; ++q) s_best[q] = Fm[q];
					}
				}
			}
			if (it >= niters) s_done = 1;
			s_niters = niters;
		}
		__syncthreads();
		if (s_done) break;
	}

	// ---- the mask of the best model
	const bool raised = s_raised != 0;
	double thr_mask = a.thr;
	if (lmeds && s_have_best)
	{
		double sigma = 2.5 * 1.4826 * (1 + 5. / (np - 7)) * sqrt(s_min_median);
		thr_mask = fmax(sigma, 0.001);
	}
	const float t2 = static_cast<float>(thr_mask * thr_mask);
	if (tid == 0) s_total = 0;
	__syncthreads();
	int good = 0;
	if (!raised && s_have_best)
		for (int q = tid; q < np; q += blockDim.x) good += fm_error(s_best, P1[q], P2[q]) <= t2;
	for (int o = 16; o > 0; o >>= 1) good += __shfl_down_sync(0xFFFFFFFFu, good, o);
	if ((tid & 31) == 0 && good) atomicAdd(&s_total, good);
	__syncthreads();
	const int total = s_total;
	const bool found = !raised && s_have_best && (!lmeds || total >= 7);
	if (found && a.status)
		for (int q = tid; q < np; q += blockDim.x)
			a.status[static_cast<size_t>(pair) * a.status_cap + q] = fm_error(s_best, P1[q], P2[q]) <= t2;
	if (tid == 0)
	{
		res[4] = method;
		res[6] = s_iters;
		res[7] = raised;
		if (found)
		{
			res[5] = 1;
			res[3] = total;
			res[1] = total >= a.match_count_min;
			for (int q = 0; q < 9; ++q) a.F[pair * 9 + q] = s_best[q];
		}
	}
}

// Rtabmap.cpp:2186-2196 on the last decision: a frame that reached the epipolar check (ACCEPTED, RATIO, LAST_NULL) is checked against
// its highest hypothesis, looked up in the word store (-1: not stored, checked as a signature without words)
__global__ void epi_decide_prep_kernel(int n_frames, const Decision * __restrict__ dec, const int * __restrict__ slot_of_sig, int n_ids,
                                       int * __restrict__ slot_b, int * __restrict__ skip)
{
	const int f = blockIdx.x * blockDim.x + threadIdx.x;
	if (f >= n_frames) return;
	const int st = dec[f].status, id = dec[f].highest_id;
	skip[f] = !(st == 8 || st == 6 || st == 7); // LCD_DECIDE_ACCEPTED, _RATIO, _LAST_NULL
	slot_b[f] = (id > 0 && id < n_ids) ? slot_of_sig[id] : -1;
}

// a failed check: LCD_DECIDE_EPIPOLAR_REJECTED, no loop closure, and no hypothesis left for lcd_verify_decided_dev; highest untouched
__global__ void epi_decide_apply_kernel(int n_frames, const int * __restrict__ res, Decision * __restrict__ dec, int * __restrict__ hyp_id,
                                        int * __restrict__ hyp_slot)
{
	const int f = blockIdx.x * blockDim.x + threadIdx.x;
	if (f >= n_frames || !res[f * 8] || res[f * 8 + 1]) return;
	dec[f].status = 11; // LCD_DECIDE_EPIPOLAR_REJECTED
	dec[f].loop_id = 0;
	if (hyp_id) hyp_id[f] = 0;
	if (hyp_slot) hyp_slot[f] = -1;
}

} // namespace lcd
