// Stand-in for the part of OpenCV that the reference's GeodeticCoords.h / GeodeticCoords.cpp use (cv::Point3d, cv::Point3f, cv::Vec3d,
// cv::normalize), so that file compiles into oracle/_ref/libref_geodetic.so without OpenCV.  TEST INFRASTRUCTURE ONLY.
//
// Point3d's difference is a component-wise double subtraction, as OpenCV's.  Vec3d, normalize and cross only serve
// ENU_WGS84ToGeocentric_WGS84, which the oracle does not call.
#pragma once
#include <cmath>

namespace cv {

template <typename T>
struct Point3_
{
	Point3_() : x(0), y(0), z(0) {}
	Point3_(T x_, T y_, T z_) : x(x_), y(y_), z(z_) {}
	template <typename U>
	Point3_(const Point3_<U> & p) : x(static_cast<T>(p.x)), y(static_cast<T>(p.y)), z(static_cast<T>(p.z)) {}
	T x, y, z;
};
typedef Point3_<double> Point3d;
typedef Point3_<float> Point3f;

template <typename T>
inline Point3_<T> operator-(const Point3_<T> & a, const Point3_<T> & b) { return Point3_<T>(a.x - b.x, a.y - b.y, a.z - b.z); }

struct Vec3d
{
	Vec3d() : v{0, 0, 0} {}
	Vec3d(double a, double b, double c) : v{a, b, c} {}
	double & operator[](int i) { return v[i]; }
	double operator[](int i) const { return v[i]; }
	Vec3d cross(const Vec3d & o) const { return Vec3d(v[1] * o[2] - v[2] * o[1], v[2] * o[0] - v[0] * o[2], v[0] * o[1] - v[1] * o[0]); }
	double v[3];
};

inline Vec3d normalize(const Vec3d & a)
{
	const double n = std::sqrt(a[0] * a[0] + a[1] * a[1] + a[2] * a[2]);
	return n > 0 ? Vec3d(a[0] / n, a[1] / n, a[2] / n) : a;
}

} // namespace cv
