// Stand-in (oracle/refstubs/orbx/opencv2/core/core.hpp): declared, aborts if called
#pragma once
#include <vector>
#include "../core/core.hpp"
namespace cv {
inline void FAST(const Mat &, std::vector<KeyPoint> &, int, bool) { stub_abort(); }
struct KeyPointsFilter
{
	static void retainBest(std::vector<KeyPoint> &, int) { stub_abort(); }
};
} // namespace cv
