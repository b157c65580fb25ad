// Stand-in for the OpenCV types the reference's corelib/src/opencv/ORBextractor.cc names (TEST INFRASTRUCTURE ONLY, oracle/orbx.mk).
// Only what the ORBextractor constructor and DistributeOctTree execute is real: cv::Point_, cv::KeyPoint, cvRound / cvFloor / cvCeil.
// Every image operation (Mat access, FAST, resize, copyMakeBorder, GaussianBlur, fastAtan2, retainBest) is declared so that the file
// compiles, and aborts if it is ever called: the wrapper (ref_orbx.cpp) never calls them.
#pragma once
#include <cassert>
#include <cmath>
#include <cstdlib>
#include <vector>

#define CV_PI 3.1415926535897932384626433832795
#define CV_8U 0
#define CV_8UC1 0

inline int cvRound(double v) { return static_cast<int>(std::nearbyint(v)); }
inline int cvRound(float v) { return static_cast<int>(std::nearbyint(v)); }
inline int cvFloor(double v) { return static_cast<int>(std::floor(v)); }
inline int cvCeil(double v) { return static_cast<int>(std::ceil(v)); }

typedef unsigned char uchar;

namespace cv {
[[noreturn]] inline void stub_abort() { std::abort(); }

template <typename T>
struct Point_
{
	T x, y;
	Point_() : x(0), y(0) {}
	Point_(T x_, T y_) : x(x_), y(y_) {}
	Point_ & operator*=(float s)
	{
		x = static_cast<T>(x * s);
		y = static_cast<T>(y * s);
		return *this;
	}
};
typedef Point_<int> Point2i;
typedef Point_<int> Point;
typedef Point_<float> Point2f;

struct KeyPoint
{
	Point2f pt;
	float size = 0, angle = -1, response = 0;
	int octave = 0, class_id = -1;
};

struct Size
{
	int width, height;
	Size(int w, int h) : width(w), height(h) {}
};
struct Rect
{
	int x, y, width, height;
	Rect(int x_, int y_, int w, int h) : x(x_), y(y_), width(w), height(h) {}
};
struct Range
{
};

struct Mat
{
	int rows = 0, cols = 0;
	size_t step = 0;
	Mat() {}
	Mat(Size, int) { stub_abort(); }
	Mat operator()(const Rect &) const { stub_abort(); }
	template <typename T> const T & at(int, int) const { stub_abort(); }
	template <typename T> T & at(int, int) { stub_abort(); }
	size_t step1() const { stub_abort(); }
	Mat rowRange(int, int) const { stub_abort(); }
	Mat colRange(int, int) const { stub_abort(); }
	Mat clone() const { stub_abort(); }
	bool empty() const { stub_abort(); }
	int type() const { stub_abort(); }
	unsigned char * ptr(int) { stub_abort(); }
	static Mat zeros(int, int, int) { stub_abort(); }
};

struct InputArray
{
	InputArray(const Mat &) {}
	Mat getMat() const { stub_abort(); }
	bool empty() const { stub_abort(); }
};
struct OutputArray
{
	OutputArray(Mat &) {}
	Mat getMat() const { stub_abort(); }
	void create(int, int, int) const { stub_abort(); }
	void release() const { stub_abort(); }
};

struct Point3f
{
};

enum { INTER_LINEAR = 1, BORDER_REFLECT_101 = 4, BORDER_ISOLATED = 16 };

inline float fastAtan2(float, float) { stub_abort(); }
} // namespace cv
