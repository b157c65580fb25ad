// fm_solver.h — the fundamental-matrix arithmetic of OpenCV's FMEstimatorCallback (calib3d fundam.cpp: run7Point with the null space
// of cv::SVDecomp, cv::solveCubic, computeError, and the haveCollinearPoints test of checkSubset), written once for the device
// (epipolar.cuh) and the host (the CPU oracle, oracle/oracle_epipolar.cpp).
//
// Every operation is an IEEE-rounded +, -, *, / or sqrt, built without contraction on both sides (--fmad=false, -ffp-contract=off),
// so the kernel and the oracle compute the same bits.  Where OpenCV calls hypot, acos, cos and pow(x, 1/3), whose device and host
// libraries differ in the last bit, the routines below stand in: they are accurate to a few ulp, and the models they give match
// cv2's to ~1e-13 relative (the SVD is OpenCV's one-sided Jacobi, step for step; its rotation's hypot is sqrt(a*a + b*b)).
#pragma once
#include <math.h>
#include <stdint.h>

#ifdef __CUDACC__
#define FM_HD __host__ __device__
#else
#define FM_HD
#endif

namespace lcd {

struct FmPt
{
	float x, y;
};

// cv::RNG::next (multiply-with-carry)
FM_HD inline unsigned fm_rng_next(unsigned long long & state)
{
	state = static_cast<unsigned long long>(static_cast<unsigned>(state)) * 4164903690ull + static_cast<unsigned>(state >> 32);
	return static_cast<unsigned>(state);
}

FM_HD inline double fm_hypot(double a, double b) { return sqrt(a * a + b * b); }

// cos(x) for |x| < 8: x - k pi/2 (two-part pi/2), then the sine or cosine series on |r| <= pi/4
FM_HD inline double fm_cos(double x)
{
	const double pio2_hi = 1.5707963267948966, pio2_lo = 6.123233995736766e-17;
	const double k = floor(x / pio2_hi + 0.5);
	const double r = (x - k * pio2_hi) - k * pio2_lo, r2 = r * r;
	double c = 1, s = 1;
	for (int n = 11; n >= 1; --n)
	{
		c = 1 - r2 / ((2. * n - 1) * (2. * n)) * c;
		s = 1 - r2 / ((2. * n) * (2. * n + 1)) * s;
	}
	s *= r;
	switch (static_cast<int>(k) & 3)
	{
	case 0: return c;
	case 1: return -s;
	case 2: return -c;
	default: return s;
	}
}

// asin(y) for |y| <= 0.5 by its series (terms fall by at least 4x)
FM_HD inline double fm_asin_small(double y)
{
	const double y2 = y * y;
	double term = y, s = y;
	for (int n = 1; n <= 30; ++n)
	{
		term *= y2 * ((2. * n - 1) * (2. * n - 1)) / ((2. * n) * (2. * n + 1));
		s += term;
	}
	return s;
}

FM_HD inline double fm_acos(double x)
{
	const double pi = 3.141592653589793, pio2 = 1.5707963267948966;
	if (!(fabs(x) <= 1)) return (x - x) / (x - x); // NaN, as acos outside [-1, 1]
	if (fabs(x) <= 0.5) return pio2 - fm_asin_small(x);
	if (x > 0) return 2 * fm_asin_small(sqrt((1 - x) * 0.5));
	return pi - 2 * fm_asin_small(sqrt((1 + x) * 0.5));
}

// pow(x, 1/3) for x >= 0: Newton's iteration on the mantissa, scaled back by an exact power of two
FM_HD inline double fm_cbrt(double x)
{
	if (x == 0 || !(x < 1.7976931348623157e308)) return x;
	int e;
	double m = frexp(x, &e);
	while (((e % 3) + 3) % 3 != 0)
	{
		m *= 2;
		--e;
	}
	double y = 1;
	for (int i = 0; i < 12; ++i) y = y - (y * y * y - m) / (3 * y * y);
	return ldexp(y, e / 3);
}

// JacobiSVDImpl_ on A (7x9, row-major, OpenCV works on it as At since m < n) with the completion of the two missing rows of V^T
// (random +-1/9 vectors from cv::RNG(0x12345678), orthogonalised twice, normalised): rows 7 and 8, the null space
FM_HD inline void fm_null_space(const double * a, double * f1, double * f2)
{
	constexpr int m = 9, n = 7;
	const double eps = 2.220446049250313e-16 * 10, minval = 2.2250738585072014e-308;
	double At[81], W[7];
	for (int i = 0; i < 63; ++i) At[i] = a[i];
	for (int i = 0; i < n; ++i)
	{
		double sd = 0;
		for (int k = 0; k < m; ++k) sd += At[i * m + k] * At[i * m + k];
		W[i] = sd;
	}
	for (int iter = 0; iter < 30; ++iter)
	{
		bool changed = false;
		for (int i = 0; i < n - 1; ++i)
			for (int j = i + 1; j < n; ++j)
			{
				double * Ai = At + i * m;
				double * Aj = At + j * m;
				double aa = W[i], p = 0, bb = W[j];
				for (int k = 0; k < m; ++k) p += Ai[k] * Aj[k];
				if (fabs(p) <= eps * sqrt(aa * bb)) continue;
				p *= 2;
				const double beta = aa - bb, gamma = fm_hypot(p, beta);
				double c, s;
				if (beta < 0)
				{
					const double delta = (gamma - beta) * 0.5;
					s = sqrt(delta / gamma);
					c = p / (gamma * s * 2);
				}
				else
				{
					c = sqrt((gamma + beta) / (gamma * 2));
					s = p / (gamma * c * 2);
				}
				aa = bb = 0;
				for (int k = 0; k < m; ++k)
				{
					const double t0 = c * Ai[k] + s * Aj[k];
					const double t1 = -s * Ai[k] + c * Aj[k];
					Ai[k] = t0;
					Aj[k] = t1;
					aa += t0 * t0;
					bb += t1 * t1;
				}
				W[i] = aa;
				W[j] = bb;
				changed = true;
			}
		if (!changed) break;
	}
	for (int i = 0; i < n; ++i)
	{
		double sd = 0;
		for (int k = 0; k < m; ++k) sd += At[i * m + k] * At[i * m + k];
		W[i] = sqrt(sd);
	}
	for (int i = 0; i < n - 1; ++i)
	{
		int j = i;
		for (int k = i + 1; k < n; ++k)
			if (W[j] < W[k]) j = k;
		if (i != j)
		{
			const double t = W[i];
			W[i] = W[j];
			W[j] = t;
			for (int k = 0; k < m; ++k)
			{
				const double u = At[i * m + k];
				At[i * m + k] = At[j * m + k];
				At[j * m + k] = u;
			}
		}
	}
	unsigned long long rng = 0x12345678ull;
	for (int i = 0; i < m; ++i)
	{
		double sd = i < n ? W[i] : 0;
		for (int ii = 0; ii < 100 && sd <= minval; ++ii)
		{
			for (int k = 0; k < m; ++k) At[i * m + k] = (fm_rng_next(rng) & 256) != 0 ? 1. / m : -1. / m;
			for (int it = 0; it < 2; ++it)
				for (int j = 0; j < i; ++j)
				{
					sd = 0;
					for (int k = 0; k < m; ++k) sd += At[i * m + k] * At[j * m + k];
					double asum = 0;
					for (int k = 0; k < m; ++k)
					{
						const double t = At[i * m + k] - sd * At[j * m + k];
						At[i * m + k] = t;
						asum += fabs(t);
					}
					asum = asum > eps * 100 ? 1 / asum : 0;
					for (int k = 0; k < m; ++k) At[i * m + k] *= asum;
				}
			sd = 0;
			for (int k = 0; k < m; ++k) sd += At[i * m + k] * At[i * m + k];
			sd = sqrt(sd);
		}
		const double s = sd > minval ? 1 / sd : 0.;
		for (int k = 0; k < m; ++k) At[i * m + k] *= s;
	}
	for (int k = 0; k < 9; ++k)
	{
		f1[k] = At[7 * 9 + k];
		f2[k] = At[8 * 9 + k];
	}
}

// cv::solveCubic, c[0] x^3 + ... + c[3]; -1 when every x is a root
FM_HD inline int fm_solve_cubic(const double * c, double * r)
{
	double a0 = c[0], a1 = c[1], a2 = c[2], a3 = c[3], x0 = 0, x1 = 0, x2 = 0;
	int n = 0;
	if (a0 == 0)
	{
		if (a1 == 0)
		{
			if (a2 == 0)
				n = a3 == 0 ? -1 : 0;
			else
			{
				x0 = -a3 / a2;
				n = 1;
			}
		}
		else
		{
			double d = a2 * a2 - 4 * a1 * a3;
			if (d >= 0)
			{
				d = sqrt(d);
				const double q1 = (-a2 + d) * 0.5, q2 = (a2 + d) * -0.5;
				if (fabs(q1) > fabs(q2))
				{
					x0 = q1 / a1;
					x1 = a3 / q1;
				}
				else
				{
					x0 = q2 / a1;
					x1 = a3 / q2;
				}
				n = d > 0 ? 2 : 1;
			}
		}
	}
	else
	{
		a0 = 1. / a0;
		a1 *= a0;
		a2 *= a0;
		a3 *= a0;
		const double Q = (a1 * a1 - 3 * a2) * (1. / 9);
		const double R = (a1 * (2 * a1 * a1 - 9 * a2) + 27 * a3) * (1. / 54);
		const double Qcubed = Q * Q * Q;
		double d = (a1 * a1 * (a2 * a2 - 4 * a1 * a3) + 2 * a2 * (9 * a1 * a3 - 2 * a2 * a2) - 27 * a3 * a3) * (1. / 108);
		if (d > 0)
		{
			const double theta = fm_acos(R / sqrt(Qcubed));
			const double t0 = -2 * sqrt(Q), t1 = theta * (1. / 3), t2 = a1 * (1. / 3);
			x0 = t0 * fm_cos(t1) - t2;
			x1 = t0 * fm_cos(t1 + (2. * 3.141592653589793 / 3)) - t2;
			x2 = t0 * fm_cos(t1 + (4. * 3.141592653589793 / 3)) - t2;
			n = 3;
		}
		else if (d == 0)
		{
			if (R >= 0)
			{
				x0 = -2 * fm_cbrt(R) - a1 / 3;
				x1 = fm_cbrt(R) - a1 / 3;
			}
			else
			{
				x0 = 2 * fm_cbrt(-R) - a1 / 3;
				x1 = -fm_cbrt(-R) - a1 / 3;
			}
			x2 = 0;
			n = x0 == x1 ? 1 : 2;
			x1 = x0 == x1 ? 0 : x1;
		}
		else
		{
			d = sqrt(-d);
			double e = fm_cbrt(d + fabs(R));
			if (R > 0) e = -e;
			x0 = (e + Q / e) - a1 * (1. / 3);
			n = 1;
		}
	}
	r[0] = x0;
	r[1] = x1;
	r[2] = x2;
	return n;
}

// run7Point (calib3d fundam.cpp) on the points p1[idx[k]], p2[idx[k]]: up to 3 models in F[27], their count (-1: OpenCV raises)
FM_HD inline int fm_run_7point(const FmPt * p1, const FmPt * p2, const uint16_t * idx, double * F)
{
	double m1cx = 0, m1cy = 0, m2cx = 0, m2cy = 0, scale1 = 0, scale2 = 0;
	for (int i = 0; i < 7; ++i)
	{
		m1cx += p1[idx[i]].x;
		m1cy += p1[idx[i]].y;
		m2cx += p2[idx[i]].x;
		m2cy += p2[idx[i]].y;
	}
	const double t = 1. / 7;
	m1cx *= t;
	m1cy *= t;
	m2cx *= t;
	m2cy *= t;
	for (int i = 0; i < 7; ++i)
	{
		const double dx1 = p1[idx[i]].x - m1cx, dy1 = p1[idx[i]].y - m1cy, dx2 = p2[idx[i]].x - m2cx, dy2 = p2[idx[i]].y - m2cy;
		scale1 += sqrt(dx1 * dx1 + dy1 * dy1);
		scale2 += sqrt(dx2 * dx2 + dy2 * dy2);
	}
	scale1 *= t;
	scale2 *= t;
	if (scale1 < 1.1920928955078125e-07 || scale2 < 1.1920928955078125e-07) return 0;
	scale1 = sqrt(2.) / scale1;
	scale2 = sqrt(2.) / scale2;
	double a[63];
	for (int i = 0; i < 7; ++i)
	{
		const double x0 = (p1[idx[i]].x - m1cx) * scale1, y0 = (p1[idx[i]].y - m1cy) * scale1;
		const double x1 = (p2[idx[i]].x - m2cx) * scale2, y1 = (p2[idx[i]].y - m2cy) * scale2;
		double * ai = a + i * 9;
		ai[0] = x1 * x0;
		ai[1] = x1 * y0;
		ai[2] = x1;
		ai[3] = y1 * x0;
		ai[4] = y1 * y0;
		ai[5] = y1;
		ai[6] = x0;
		ai[7] = y0;
		ai[8] = 1;
	}
	double f1[9], f2[9], c[4], r[3];
	fm_null_space(a, f1, f2);
	for (int i = 0; i < 9; ++i) f1[i] -= f2[i];
	double t0 = f2[4] * f2[8] - f2[5] * f2[7];
	double t1 = f2[3] * f2[8] - f2[5] * f2[6];
	double t2 = f2[3] * f2[7] - f2[4] * f2[6];
	c[3] = f2[0] * t0 - f2[1] * t1 + f2[2] * t2;
	c[2] = f1[0] * t0 - f1[1] * t1 + f1[2] * t2 - f1[3] * (f2[1] * f2[8] - f2[2] * f2[7]) + f1[4] * (f2[0] * f2[8] - f2[2] * f2[6]) -
	       f1[5] * (f2[0] * f2[7] - f2[1] * f2[6]) + f1[6] * (f2[1] * f2[5] - f2[2] * f2[4]) - f1[7] * (f2[0] * f2[5] - f2[2] * f2[3]) +
	       f1[8] * (f2[0] * f2[4] - f2[1] * f2[3]);
	t0 = f1[4] * f1[8] - f1[5] * f1[7];
	t1 = f1[3] * f1[8] - f1[5] * f1[6];
	t2 = f1[3] * f1[7] - f1[4] * f1[6];
	c[1] = f2[0] * t0 - f2[1] * t1 + f2[2] * t2 - f2[3] * (f1[1] * f1[8] - f1[2] * f1[7]) + f2[4] * (f1[0] * f1[8] - f1[2] * f1[6]) -
	       f2[5] * (f1[0] * f1[7] - f1[1] * f1[6]) + f2[6] * (f1[1] * f1[5] - f1[2] * f1[4]) - f2[7] * (f1[0] * f1[5] - f1[2] * f1[3]) +
	       f2[8] * (f1[0] * f1[4] - f1[1] * f1[3]);
	c[0] = f1[0] * t0 - f1[1] * t1 + f1[2] * t2;
	const int n = fm_solve_cubic(c, r);
	if (n < 1 || n > 3) return n;
	const double T1[9] = {scale1, 0, -scale1 * m1cx, 0, scale1, -scale1 * m1cy, 0, 0, 1};
	const double T2[9] = {scale2, 0, -scale2 * m2cx, 0, scale2, -scale2 * m2cy, 0, 0, 1};
	for (int k = 0; k < n; ++k)
	{
		double fm[9], G[9];
		double lambda = r[k], mu = 1.;
		const double s = f1[8] * r[k] + f2[8];
		if (fabs(s) > 2.220446049250313e-16)
		{
			mu = 1. / s;
			lambda *= mu;
			fm[8] = 1.;
		}
		else
			fm[8] = 0.;
		for (int i = 0; i < 8; ++i) fm[i] = f1[i] * lambda + f2[i] * mu;
		// F = T2^T * F * T1, then F(3,3) = 1
		for (int i = 0; i < 3; ++i)
			for (int j = 0; j < 3; ++j)
			{
				double acc = 0;
				for (int q = 0; q < 3; ++q) acc += T2[q * 3 + i] * fm[q * 3 + j];
				G[i * 3 + j] = acc;
			}
		double * H = F + 9 * k;
		for (int i = 0; i < 3; ++i)
			for (int j = 0; j < 3; ++j)
			{
				double acc = 0;
				for (int q = 0; q < 3; ++q) acc += G[i * 3 + q] * T1[q * 3 + j];
				H[i * 3 + j] = acc;
			}
		if (fabs(H[8]) > 1.1920928955078125e-07)
		{
			const double sc = 1. / H[8];
			for (int i = 0; i < 9; ++i) H[i] *= sc;
		}
	}
	return n;
}

// FMEstimatorCallback::computeError
FM_HD inline float fm_error(const double * F, FmPt m1, FmPt m2)
{
	double a = F[0] * m1.x + F[1] * m1.y + F[2];
	double b = F[3] * m1.x + F[4] * m1.y + F[5];
	double c = F[6] * m1.x + F[7] * m1.y + F[8];
	const double s2 = 1. / (a * a + b * b);
	const double d2 = m2.x * a + m2.y * b + c;
	a = F[0] * m2.x + F[3] * m2.y + F[6];
	b = F[1] * m2.x + F[4] * m2.y + F[7];
	c = F[2] * m2.x + F[5] * m2.y + F[8];
	const double s1 = 1. / (a * a + b * b);
	const double d1 = m1.x * a + m1.y * b + c;
	const double e1 = d1 * d1 * s1, e2 = d2 * d2 * s2;
	return static_cast<float>(e1 < e2 ? e2 : e1); // std::max(e1, e2)
}

// haveCollinearPoints on the last of 7 sampled points
FM_HD inline bool fm_collinear(const FmPt * p, const uint16_t * idx)
{
	const FmPt pi = p[idx[6]];
	for (int j = 0; j < 6; ++j)
	{
		const double dx1 = p[idx[j]].x - pi.x, dy1 = p[idx[j]].y - pi.y;
		for (int k = 0; k < j; ++k)
		{
			const double dx2 = p[idx[k]].x - pi.x, dy2 = p[idx[k]].y - pi.y;
			if (fabs(dx2 * dy1 - dy2 * dx1) <= 1.1920928955078125e-07 * (fabs(dx1) + fabs(dy1) + fabs(dx2) + fabs(dy2))) return true;
		}
	}
	return false;
}

} // namespace lcd
