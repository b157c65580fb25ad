// oracle_epipolar.cpp — CPU restatement of rtabmap::EpipolarGeometry::check (TEST INFRASTRUCTURE, never linked by the product).
//
//   findPairsUnique          corelib/include/rtabmap/core/EpipolarGeometry.h:157-186 (A = new signature, B = hypothesis)
//   EpipolarGeometry::check  corelib/src/EpipolarGeometry.cpp:65-102, findFFromWords :298-379
//   cv::findFundamentalMat(points1, points2, status, FM_RANSAC, param1, param2) as OpenCV 4.13 runs it: < 7 points -> no matrix;
//   7 points -> the 7-point kernel alone (mask all ones); 8-14 points -> LMeDSPointSetRegistrator; >= 15 -> RANSACPointSetRegistrator
//   with 7-point samples, maxIters 1000.  The registrators are those vendored in corelib/src/opencv/solvepnp.cpp:213-557; the
//   fundamental-matrix callback (7-point kernel, computeError, checkSubset) is OpenCV's calib3d fundam.cpp, restated here and pinned
//   to cv2 by tests/test_oracle_epipolar.py.
//
// The callback's arithmetic (the 7-point kernel with OpenCV's Jacobi SVD and its random completion of the two missing null-space rows,
// solveCubic, computeError, haveCollinearPoints) is rtabmap_b200/csrc/fm_solver.h, the code the GPU kernel runs, so that the two
// compute the same bits; this file restates the rest (findPairsUnique, the path selection, both registrators) on its own, and
// tests/test_oracle_epipolar.py pins the whole against cv2.
// The PnP oracle's cv::RNG (CvRng) and RANSACUpdateNumIters (ransac_update_num_iters) are used as they are: its translation unit is
// compiled into this library (with oracle.cpp, which it calls).
#include "oracle_verify.cpp"
#include "../rtabmap_b200/csrc/fm_solver.h"

#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <map>
#include <vector>

namespace {

using P2 = lcd::FmPt;

const uint16_t kIdx7[7] = {0, 1, 2, 3, 4, 5, 6};

// run7Point: up to 3 models in F[27], the count (-1 when the determinant polynomial vanishes identically)
int run_7point(const P2 * m1, const P2 * m2, double * fmatrix) { return lcd::fm_run_7point(m1, m2, kIdx7, fmatrix); }

// FMEstimatorCallback::computeError over all points
void compute_error(const P2 * m1, const P2 * m2, int count, const double * F, float * err)
{
	for (int i = 0; i < count; ++i) err[i] = lcd::fm_error(F, m1[i], m2[i]);
}

// haveCollinearPoints on a full sample of 7
bool have_collinear_points(const P2 * p) { return lcd::fm_collinear(p, kIdx7); }

struct Ctx
{
	const P2 *m1, *m2;
	int count;
	int check_subset;
	int raised = 0;
	int iterations = 0;
};

// getSubset of the vendored registrator (checkPartialSubsets = false)
bool get_subset(Ctx & cx, CvRng & rng, P2 * ms1, P2 * ms2, int max_attempts)
{
	int idx[7], i = 0, iters = 0;
	for (; iters < max_attempts; ++iters)
	{
		for (i = 0; i < 7 && iters < max_attempts;)
		{
			int idx_i;
			for (;;)
			{
				idx_i = idx[i] = rng.uniform(0, cx.count);
				int j;
				for (j = 0; j < i; ++j)
					if (idx_i == idx[j]) break;
				if (j == i) break;
			}
			ms1[i] = cx.m1[idx_i];
			ms2[i] = cx.m2[idx_i];
			++i;
		}
		if (i == 7 && cx.check_subset && (have_collinear_points(ms1) || have_collinear_points(ms2))) continue;
		break;
	}
	return i == 7 && iters < max_attempts;
}

int find_inliers(const Ctx & cx, const double * F, double thresh, std::vector<float> & err, uint8_t * mask)
{
	compute_error(cx.m1, cx.m2, cx.count, F, err.data());
	const float t = (float)(thresh * thresh);
	int nz = 0;
	for (int i = 0; i < cx.count; ++i)
	{
		const int f = err[i] <= t;
		mask[i] = (uint8_t)f;
		nz += f;
	}
	return nz;
}

// runKernel: OpenCV copies F.rowRange(0, n*3) for any n != 0, which asserts for n < 0
int run_kernel(Ctx & cx, const P2 * a, const P2 * b, double * F)
{
	const int n = run_7point(a, b, F);
	if (n < 0) cx.raised = 1;
	return n;
}

bool ransac_run(Ctx & cx, double threshold, double confidence, int max_iters, double * best, uint8_t * mask)
{
	std::vector<float> err(cx.count);
	std::vector<uint8_t> m(cx.count);
	int niters = std::max(max_iters, 1), max_good = 0;
	CvRng rng;
	P2 ms1[7], ms2[7];
	double F[27];
	int iter;
	for (iter = 0; iter < niters; ++iter)
	{
		if (!get_subset(cx, rng, ms1, ms2, 10000))
		{
			if (iter == 0) return false;
			break;
		}
		const int nmodels = run_kernel(cx, ms1, ms2, F);
		if (cx.raised)
		{
			cx.iterations = iter + 1;
			return false;
		}
		if (nmodels <= 0) continue;
		for (int i = 0; i < nmodels; ++i)
		{
			const int good = find_inliers(cx, F + 9 * i, threshold, err, m.data());
			if (good > std::max(max_good, 6))
			{
				std::memcpy(mask, m.data(), cx.count);
				std::memcpy(best, F + 9 * i, sizeof(double) * 9);
				max_good = good;
				niters = ransac_update_num_iters(confidence, (double)(cx.count - good) / cx.count, 7, niters);
			}
		}
	}
	cx.iterations = iter;
	return max_good > 0;
}

bool lmeds_run(Ctx & cx, double confidence, int max_iters, double * best, uint8_t * mask)
{
	std::vector<float> err(cx.count);
	double min_median = DBL_MAX;
	CvRng rng;
	P2 ms1[7], ms2[7];
	double F[27];
	int niters = std::max(ransac_update_num_iters(confidence, 0.45, 7, max_iters), 3), iter;
	for (iter = 0; iter < niters; ++iter)
	{
		if (!get_subset(cx, rng, ms1, ms2, 1000))
		{
			if (iter == 0) return false;
			break;
		}
		const int nmodels = run_kernel(cx, ms1, ms2, F);
		if (cx.raised)
		{
			cx.iterations = iter + 1;
			return false;
		}
		if (nmodels <= 0) continue;
		for (int i = 0; i < nmodels; ++i)
		{
			compute_error(cx.m1, cx.m2, cx.count, F + 9 * i, err.data());
			std::vector<int32_t> bits(cx.count);
			std::memcpy(bits.data(), err.data(), sizeof(float) * cx.count);
			std::sort(bits.begin(), bits.end()); // std::sort(errf.ptr<int>(), ...): float errors ordered by their int32 bit patterns
			std::memcpy(err.data(), bits.data(), sizeof(float) * cx.count);
			const int c = cx.count;
			const double median = c % 2 != 0 ? err[c / 2] : (err[c / 2 - 1] + err[c / 2]) * 0.5;
				if (median < min_median)
			{
				min_median = median;
				std::memcpy(best, F + 9 * i, sizeof(double) * 9);
			}
		}
	}
	cx.iterations = iter;
	if (min_median < DBL_MAX)
	{
		double sigma = 2.5 * 1.4826 * (1 + 5. / (cx.count - 7)) * std::sqrt(min_median);
		sigma = std::max(sigma, 0.001);
		const int good = find_inliers(cx, best, sigma, err, mask);
		return good >= 7;
	}
	return false;
}

} // namespace

extern "C" {

// run7Point on 7 correspondences: the models in F[27] (as findFundamentalMat returns them for 7 points), their count
int epo_run_7point(const float * p1, const float * p2, double * F)
{
	return run_7point(reinterpret_cast<const P2 *>(p1), reinterpret_cast<const P2 *>(p2), F);
}

// findPairsUnique(A, B): rows_a / rows_b / ids_out [min(na, nb)] in ascending word id order; returns the number of pairs
int epo_find_pairs_unique(const int * ids_a, int na, const int * ids_b, int nb, int * rows_a, int * rows_b, int * ids_out)
{
	std::multimap<int, int> A, B;
	for (int i = 0; i < na; ++i) A.insert(std::make_pair(ids_a[i], i));
	for (int i = 0; i < nb; ++i) B.insert(std::make_pair(ids_b[i], i));
	int n = 0;
	for (auto it = A.begin(); it != A.end(); it = A.upper_bound(it->first))
	{
		const int id = it->first;
		if (id < 0) continue;
		if (A.count(id) == 1 && B.count(id) == 1)
		{
			rows_a[n] = it->second;
			rows_b[n] = B.find(id)->second;
			ids_out[n] = id;
			++n;
		}
	}
	return n;
}

// cv::findFundamentalMat(p1, p2, mask, FM_RANSAC, param1, param2) as OpenCV 4.13 runs it.  info[0] method (0 none, 1 7-point,
// 2 LMeDS, 3 RANSAC), info[1] found (a matrix was returned), info[2] iterations run, info[3] OpenCV raises; F[9] the returned matrix
// (7 points: the first solution); mask[n].  Returns the number of inliers (0 when no matrix).
int epo_find_fundamental(const float * p1, const float * p2, int n, double param1, double param2, int check_subset, uint8_t * mask,
                         double * Fout, int * info)
{
	Ctx cx;
	cx.m1 = reinterpret_cast<const P2 *>(p1);
	cx.m2 = reinterpret_cast<const P2 *>(p2);
	cx.count = n;
	cx.check_subset = check_subset;
	std::memset(mask, 0, n);
	for (int i = 0; i < 9; ++i) Fout[i] = 0;
	info[0] = info[1] = info[2] = info[3] = 0;
	if (n < 7) return 0;
	double F[27];
	bool ok;
	if (n == 7)
	{
		info[0] = 1;
		const int k = run_kernel(cx, cx.m1, cx.m2, F);
		std::memset(mask, 1, n);
		ok = k > 0;
	}
	else
	{
		if (param1 <= 0) param1 = 3;
		if (param2 < DBL_EPSILON || param2 > 1 - DBL_EPSILON) param2 = 0.99;
		if (n >= 15)
		{
			info[0] = 3;
			ok = ransac_run(cx, param1, param2, 1000, F, mask);
		}
		else
		{
			info[0] = 2;
			ok = lmeds_run(cx, param2, 1000, F, mask);
		}
		info[2] = cx.iterations;
	}
	info[3] = cx.raised;
	if (cx.raised || !ok)
	{
		if (cx.raised) std::memset(mask, 0, n);
		return 0;
	}
	info[1] = 1;
	std::memcpy(Fout, F, sizeof(double) * 9);
	int s = 0;
	for (int i = 0; i < n; ++i) s += mask[i];
	return s;
}

} // extern "C"
