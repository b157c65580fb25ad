// ransac.cuh — the pieces of OpenCV's RANSACPointSetRegistrator that every RANSAC kernel replays (opencv/solvepnp.cpp:213-228 and
// cv::RNG): the random stream the samples are drawn from, and the adaptive iteration count.
#pragma once
#include <cuda_runtime.h>
#include <math.h>

namespace lcd {

// cv::RNG::next (multiply-with-carry); every registrator run starts from the state (uint64)-1
__host__ __device__ inline unsigned cv_rng_next(unsigned long long & state)
{
	state = static_cast<unsigned long long>(static_cast<unsigned>(state)) * 4164903690ull + static_cast<unsigned>(state >> 32);
	return static_cast<unsigned>(state);
}

// cv::RNG::uniform(0, n) for n > 0
__host__ __device__ inline int cv_rng_uniform(unsigned long long & state, int n)
{
	return static_cast<int>(cv_rng_next(state) % static_cast<unsigned>(n));
}

// RANSACUpdateNumIters
__device__ inline int ransac_update_num_iters(double p, double ep, int modelPoints, int maxIters)
{
	p = fmax(p, 0.);
	p = fmin(p, 1.);
	ep = fmax(ep, 0.);
	ep = fmin(ep, 1.);
	double num = fmax(1. - p, 2.2250738585072014e-308);
	double denom = 1. - pow(1. - ep, static_cast<double>(modelPoints));
	if (denom < 2.2250738585072014e-308) return 0;
	num = log(num);
	denom = log(denom);
	return denom >= 0 || -num >= maxIters * (-denom) ? maxIters : static_cast<int>(nearbyint(num / denom));
}

} // namespace lcd
