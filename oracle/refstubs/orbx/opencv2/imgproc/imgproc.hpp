// Stand-in (oracle/refstubs/orbx/opencv2/core/core.hpp): declared, aborts if called
#pragma once
#include "../core/core.hpp"
namespace cv {
inline void resize(const Mat &, Mat &, Size, double, double, int) { stub_abort(); }
inline void copyMakeBorder(const Mat &, Mat &, int, int, int, int, int) { stub_abort(); }
inline void GaussianBlur(const Mat &, Mat &, Size, double, double, int) { stub_abort(); }
} // namespace cv
