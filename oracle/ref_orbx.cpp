// C wrapper over the reference's own rtabmap::ORBextractor (corelib/src/opencv/ORBextractor.cc compiled against the stand-ins of
// oracle/refstubs/orbx/ into _ref/libref_orbx.so by orbx.mk).  TEST INFRASTRUCTURE ONLY: the constructor's tables and
// DistributeOctTree, which oracle/orb_octree_py.py and the CUDA quadtree are compared against.  No image operation is called.
#include <exception>
#include <vector>

#include "ORBextractor.h"

namespace {
struct RefOrbx : rtabmap::ORBextractor
{
	using ORBextractor::ORBextractor;
	using ORBextractor::DistributeOctTree;
	using ORBextractor::mnFeaturesPerLevel;
	using ORBextractor::mvInvScaleFactor;
	using ORBextractor::mvScaleFactor;
	using ORBextractor::umax;
};
} // namespace

extern "C" {

// mvScaleFactor, mvInvScaleFactor, mnFeaturesPerLevel [nlevels] and umax [patch/2 + 1]
int ref_orbx_tables(int nfeatures, float scale_factor, int nlevels, int patch, float * scale, float * inv, int * per, int * umax)
{
	try
	{
		RefOrbx o(nfeatures, scale_factor, nlevels, 20, 7, patch, 19);
		for (int l = 0; l < nlevels; ++l)
		{
			scale[l] = o.mvScaleFactor[l];
			inv[l] = o.mvInvScaleFactor[l];
			per[l] = o.mnFeaturesPerLevel[l];
		}
		for (size_t v = 0; v < o.umax.size(); ++v) umax[v] = o.umax[v];
		return 0;
	}
	catch (const std::exception &)
	{
		return -1;
	}
}

// DistributeOctTree(keys, 0, w, 0, h, n, 0) on keys[n_keys] = (x, y, response) relative to the level's border, in the order
// ComputeKeyPointsOctTree hands them over; writes the kept keys' indices in list order, returns their count (-1 past cap)
int ref_orbx_distribute(const float * keys, int n_keys, int w, int h, int n, int * out, int cap)
{
	RefOrbx o(1000, 1.2f, 1, 20, 7, 31, 19);
	std::vector<cv::KeyPoint> in(n_keys);
	for (int i = 0; i < n_keys; ++i)
	{
		in[i].pt = cv::Point2f(keys[3 * i], keys[3 * i + 1]);
		in[i].response = keys[3 * i + 2];
		in[i].class_id = i; // DistributeOctTree copies keypoints whole: the index travels with them
	}
	const int min_x = 0, max_x = w, min_y = 0, max_y = h, level = 0;
	const std::vector<cv::KeyPoint> kept = o.DistributeOctTree(in, min_x, max_x, min_y, max_y, n, level);
	if (static_cast<int>(kept.size()) > cap) return -1;
	for (size_t i = 0; i < kept.size(); ++i) out[i] = kept[i].class_id;
	return static_cast<int>(kept.size());
}
}
