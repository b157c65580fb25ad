// Stand-in for the part of OpenCV's cv::Mat that the reference's BayesFilter.cpp uses, so that file compiles into
// oracle/_ref/libref_bayes.so without OpenCV.  TEST INFRASTRUCTURE ONLY.
//
// Covered: CV_32FC1 matrices (zeros, rows/cols/data, empty, total, elemSize), shared-storage views (Mat, Range, Range) with
// copyTo, and operator* as a matrix product.  The product accumulates in double in ascending column order: OpenCV's gemm
// blocking and summation order are not what the oracle pins, and the double sum is the high-precision reference of it.
#pragma once
#include <cstddef>
#include <cstring> // the real header brings in memcmp, which BayesFilter.cpp uses
#include <memory>
#include <vector>

#define CV_32FC1 5

namespace cv {

typedef unsigned char uchar;

struct Range
{
	Range(int s, int e) : start(s), end(e) {}
	int start, end;
};

class Mat
{
public:
	Mat() {}
	Mat(int r, int c, int /*type: CV_32FC1 only*/) : rows(r), cols(c), step_(c), buf_(std::make_shared<std::vector<float> >(static_cast<size_t>(r) * c))
	{
		data = reinterpret_cast<uchar *>(buf_->data());
	}
	Mat(const Mat & m, const Range & rr, const Range & cr) : rows(rr.end - rr.start), cols(cr.end - cr.start), step_(m.step_), buf_(m.buf_)
	{
		data = reinterpret_cast<uchar *>(m.at_ptr(rr.start, cr.start));
	}
	static Mat zeros(int r, int c, int type) { return Mat(r, c, type); }

	bool empty() const { return !data || rows == 0 || cols == 0; }
	size_t total() const { return static_cast<size_t>(rows) * cols; }
	size_t elemSize() const { return sizeof(float); }

	void copyTo(const Mat & dst) const
	{
		for (int r = 0; r < rows; ++r)
			for (int c = 0; c < cols; ++c) *dst.at_ptr(r, c) = *at_ptr(r, c);
	}

	int rows = 0;
	int cols = 0;
	uchar * data = nullptr;

	float * at_ptr(int r, int c) const { return reinterpret_cast<float *>(data) + static_cast<size_t>(r) * step_ + c; }

private:
	size_t step_ = 0;
	std::shared_ptr<std::vector<float> > buf_;
};

inline Mat operator*(const Mat & a, const Mat & b)
{
	Mat out(a.rows, b.cols, CV_32FC1);
	for (int r = 0; r < a.rows; ++r)
		for (int c = 0; c < b.cols; ++c)
		{
			double acc = 0.0;
			for (int k = 0; k < a.cols; ++k) acc += static_cast<double>(*a.at_ptr(r, k)) * static_cast<double>(*b.at_ptr(k, c));
			*out.at_ptr(r, c) = static_cast<float>(acc);
		}
	return out;
}

} // namespace cv
