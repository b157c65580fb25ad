// pnp_device.cuh — thread-local fp64 building blocks of the geometric verification kernels:
// EPnP on a minimal sample, Rodrigues, projection with jacobian, small dense solvers.
//
// Replaces (third-party arithmetic the reference calls, SURVEY.md §8(c)): cv::solvePnP(SOLVEPNP_EPNP)
// [EPnP, Lepetit/Moreno-Noguer/Fua, IJCV 2009, as implemented in OpenCV calib3d epnp.cpp],
// cv::Rodrigues, cv::projectPoints — reached from PnPRansacCallback::runKernel / computeError
// (corelib/src/opencv/solvepnp.cpp:63-101).  The library is built with --fmad=false so that every
// double operation rounds exactly like the host's (results match the CPU oracle to ~1e-12).
//
// EPnP's answer on noisy minimal samples depends on the SIGN of the PCA axes that define its
// control points; OpenCV obtains them from its internal one-sided Jacobi SVD (used for every
// matrix smaller than 25x25), so that routine is reproduced step for step in svd_rows_jacobi().
#pragma once
#include <cuda_runtime.h>
#include <math.h>

namespace lcd {

struct CamK
{
	double fu, fv, uc, vc;
};

// One-sided Jacobi SVD, OpenCV JacobiSVDImpl_ semantics: At is n x m (row i = column i of A); on return
// rows of At = left singular vectors (unit), W descending.  m, n <= 3 here (control points).
__device__ inline void svd_rows_jacobi3(double * At, double * W)
{
	const int m = 3, n = 3;
	const double eps = 2.220446049250313e-16 * 10, minval = 2.2250738585072014e-308;
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
				double a = W[i], p = 0, b = W[j];
				for (int k = 0; k < m; ++k) p += Ai[k] * Aj[k];
				if (fabs(p) <= eps * sqrt(a * b)) continue;
				p *= 2;
				const double beta = a - b, gamma = hypot(p, beta);
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
				a = b = 0;
				for (int k = 0; k < m; ++k)
				{
					const double t0 = c * Ai[k] + s * Aj[k];
					const double t1 = -s * Ai[k] + c * Aj[k];
					Ai[k] = t0;
					Aj[k] = t1;
					a += t0 * t0;
					b += t1 * t1;
				}
				W[i] = a;
				W[j] = b;
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
			double t = W[i];
			W[i] = W[j];
			W[j] = t;
			for (int k = 0; k < m; ++k)
			{
				t = At[i * m + k];
				At[i * m + k] = At[j * m + k];
				At[j * m + k] = t;
			}
		}
	}
	for (int i = 0; i < n; ++i)
	{
		const double s = W[i] > minval ? 1 / W[i] : 0.;
		for (int k = 0; k < m; ++k) At[i * m + k] *= s;
	}
}

// Eigen-decomposition of a symmetric N x N matrix held in a[] (destroyed; the eigenvalues are left on its
// diagonal): Householder reduction to tridiagonal form, then the implicit-shift QL iteration — the same operation
// sequence as the CPU oracle's sym_eigen_desc (oracle/pnp_math.h), every sum in ascending index order.  v[] receives
// the eigenvectors as COLUMNS; ord[] the column order of descending eigenvalue.  About 15x fewer dependent
// operations than the cyclic Jacobi sweeps this replaces (one thread per RANSAC hypothesis is latency-bound).
__device__ long long g_pnp_dbg[8];

template <int N>
__device__ inline void sym_eigen(double * a, double * z, int * ord, long long * dbg = nullptr)
{
	const long long t_start = dbg ? clock64() : 0;
	const unsigned mask = __activemask();
	double d[N], e[N], hv[N], hp[N], hw[N];
#pragma unroll
	for (int i = 0; i < N; ++i)
#pragma unroll
		for (int j = 0; j < N; ++j) z[i * N + j] = i == j ? 1.0 : 0.0;
	// fully unrolled: every index below is a compile-time constant, so the compiler is free to keep the matrix in
	// registers / schedule its spills instead of chasing dynamically indexed local memory one load at a time
#pragma unroll
	for (int k = 0; k + 2 < N; ++k)
	{
		double sigma = 0;
#pragma unroll
		for (int i = k + 2; i < N; ++i) sigma += a[i * N + k] * a[i * N + k];
		if (sigma == 0.0) continue;
		const double x0 = a[(k + 1) * N + k];
		const double nrm = sqrt(x0 * x0 + sigma);
		const double alpha = x0 > 0 ? -nrm : nrm;
		hv[k + 1] = x0 - alpha;
#pragma unroll
		for (int i = k + 2; i < N; ++i) hv[i] = a[i * N + k];
		const double beta = 2.0 / (hv[k + 1] * hv[k + 1] + sigma);
#pragma unroll
		for (int i = k + 1; i < N; ++i)
		{
			double s = 0;
#pragma unroll
			for (int j = k + 1; j < N; ++j) s += a[i * N + j] * hv[j];
			hp[i] = beta * s;
		}
		double vp = 0;
#pragma unroll
		for (int i = k + 1; i < N; ++i) vp += hv[i] * hp[i];
		const double K = 0.5 * beta * vp;
#pragma unroll
		for (int i = k + 1; i < N; ++i) hw[i] = hp[i] - K * hv[i];
#pragma unroll
		for (int i = k + 1; i < N; ++i)
#pragma unroll
			for (int j = k + 1; j < N; ++j) a[i * N + j] -= hv[i] * hw[j] + hw[i] * hv[j];
		a[(k + 1) * N + k] = alpha;
		a[k * N + k + 1] = alpha;
#pragma unroll
		for (int i = k + 2; i < N; ++i)
		{
			a[i * N + k] = 0.0;
			a[k * N + i] = 0.0;
		}
#pragma unroll
		for (int r = 0; r < N; ++r)
		{
			double s = 0;
#pragma unroll
			for (int j = k + 1; j < N; ++j) s += z[r * N + j] * hv[j];
			s *= beta;
#pragma unroll
			for (int j = k + 1; j < N; ++j) z[r * N + j] -= s * hv[j];
		}
	}
#pragma unroll
	for (int i = 0; i < N; ++i)
	{
		d[i] = a[i * N + i];
		e[i] = i + 1 < N ? a[(i + 1) * N + i] : 0.0;
	}
	if (dbg) dbg[0] = clock64() - t_start;
	// The QL sweeps are data dependent (iterations per eigenvalue, deflation point m).  Lanes of a warp that drift apart
	// here would serialise, so every iteration starts from a warp vote: lanes that have converged on this l idle through
	// the iteration instead of running ahead.  The arithmetic of each lane is untouched.
	//
	// d[] and e[] stay in registers: every access below has a compile-time index.  The rotation sweep i = m-1 .. l is unrolled over
	// all N-1 positions, each guarded by l <= i < m, and the reads and writes at the run-time positions l and m go through
	// select loops (sel / put).  Column i+1 of z that the previous rotation produced is carried in zc[] instead of being stored
	// and loaded back (zc is stored once the sweep ends), and column i is loaded one rotation ahead, so z's local-memory traffic is
	// off the rotation chain.
	const auto sel = [](const double (&v)[N], int i) {
		double r = v[0];
#pragma unroll
		for (int k = 1; k < N; ++k)
			if (k == i) r = v[k];
		return r;
	};
	const auto put = [](double (&v)[N], int i, double x) {
#pragma unroll
		for (int k = 0; k < N; ++k)
			if (k == i) v[k] = x;
	};
	for (int l = 0; l < N; ++l)
	{
		for (int iter = 0; iter < 60; ++iter)
		{
			int m = N - 1;
			bool found = false;
#pragma unroll
			for (int k = 0; k + 1 < N; ++k)
				if (!found && k >= l && fabs(e[k]) <= 2.220446049250313e-16 * (fabs(d[k]) + fabs(d[k + 1])))
				{
					m = k;
					found = true;
				}
			const bool done = m == l;
			if (__all_sync(mask, done)) break;
			if (!done)
			{
				double g = (sel(d, l + 1) - sel(d, l)) / (2.0 * sel(e, l));
				double r = sqrt(g * g + 1.0);
				g = sel(d, m) - sel(d, l) + sel(e, l) / (g + (g >= 0 ? r : -r));
				double sn = 1.0, cs = 1.0, pp = 0.0;
				bool underflow = false;
				double zc[N], zp[N];
				int cz = m; // the column of z that zc holds
#pragma unroll
				for (int k = 0; k < N; ++k)
				{
					zc[k] = z[k * N + m];
					zp[k] = z[k * N + m - 1];
				}
#pragma unroll
				for (int i = N - 2; i >= 0; --i)
				{
					if (underflow || i >= m || i < l) continue;
					double zi[N]; // column i of z, loaded one rotation ahead; column i-1 is loaded now for the next rotation
#pragma unroll
					for (int k = 0; k < N; ++k)
					{
						zi[k] = zp[k];
						if (i > 0) zp[k] = z[k * N + i - 1];
					}
					double f = sn * e[i];
					const double b = cs * e[i];
					r = sqrt(f * f + g * g);
					e[i + 1] = r;
					if (r == 0.0)
					{
						d[i + 1] -= pp;
						put(e, m, 0.0);
						underflow = true;
						continue;
					}
					sn = f / r;
					cs = g / r;
					g = d[i + 1] - pp;
					r = (d[i] - g) * sn + 2.0 * cs * b;
					pp = sn * r;
					d[i + 1] = g + pp;
					g = cs * r - b;
					// columns i, i+1 of z (off the critical chain): column i is loaded, column i+1 is the carried one
#pragma unroll
					for (int k = 0; k < N; ++k)
					{
						z[k * N + i + 1] = sn * zi[k] + cs * zc[k];
						zc[k] = cs * zi[k] - sn * zc[k];
					}
					cz = i;
				}
#pragma unroll
				for (int k = 0; k < N; ++k) z[k * N + cz] = zc[k];
				if (!underflow)
				{
					put(d, l, sel(d, l) - pp);
					put(e, l, g);
					put(e, m, 0.0);
				}
			}
		}
	}
#pragma unroll
	for (int i = 0; i < N; ++i) a[i * N + i] = d[i];
	int o[N];
#pragma unroll
	for (int i = 0; i < N; ++i) o[i] = i;
#pragma unroll
	for (int i = 0; i < N - 1; ++i) // selection sort, descending, stable
	{
		int j = i;
		double dj = sel(d, o[i]);
#pragma unroll
		for (int k = i + 1; k < N; ++k)
		{
			const double dk = sel(d, o[k]);
			if (dk > dj)
			{
				j = k;
				dj = dk;
			}
		}
		int t = o[i];
#pragma unroll
		for (int k = i + 1; k < N; ++k)
			if (k == j) t = o[k];
#pragma unroll
		for (int k = N - 1; k > i; --k)
			if (k <= j) o[k] = o[k - 1];
		o[i] = t;
	}
#pragma unroll
	for (int i = 0; i < N; ++i) ord[i] = o[i];
}

// minimum-norm least squares of A x = b, A is M x N row-major (cvSolve(..., CV_SVD))
template <int M, int N>
__device__ inline void solve_ls(const double * A, const double * b, double * x)
{
	double ata[N * N], v[N * N], atb[N];
	int ord[N];
	for (int i = 0; i < N; ++i)
	{
		for (int j = 0; j < N; ++j)
		{
			double s = 0;
			for (int k = 0; k < M; ++k) s += A[k * N + i] * A[k * N + j];
			ata[i * N + j] = s;
		}
		double s = 0;
		for (int k = 0; k < M; ++k) s += A[k * N + i] * b[k];
		atb[i] = s;
	}
	sym_eigen<N>(ata, v, ord);
	for (int i = 0; i < N; ++i) x[i] = 0;
	const double wmax = ata[ord[0] * N + ord[0]];
	const double tol = wmax * 1e-14 * N;
	for (int kk = 0; kk < N; ++kk)
	{
		const int k = ord[kk];
		const double w = ata[k * N + k];
		if (w <= tol) continue;
		double c = 0;
		for (int i = 0; i < N; ++i) c += v[i * N + k] * atb[i];
		c /= w;
		for (int i = 0; i < N; ++i) x[i] += c * v[i * N + k];
	}
}

// x = A^-1 b for a symmetric positive definite N x N matrix by Cholesky — same operation sequence as the oracle's chol_solve
// (oracle/pnp_math.h).  false: a pivot is not safely positive, the caller falls back to the eigen pseudo-inverse.
template <int N>
__device__ inline bool chol_solve(const double * A, const double * b, double * x)
{
	double L[N * N], y[N];
	double dmax = 0;
#pragma unroll
	for (int i = 0; i < N; ++i) dmax = fmax(dmax, A[i * N + i]);
#pragma unroll
	for (int j = 0; j < N; ++j)
	{
		double d = A[j * N + j];
#pragma unroll
		for (int k = 0; k < j; ++k) d -= L[j * N + k] * L[j * N + k];
		if (!(d > 1e-12 * dmax)) return false;
		const double ljj = sqrt(d);
		L[j * N + j] = ljj;
#pragma unroll
		for (int i = j + 1; i < N; ++i)
		{
			double s = A[i * N + j];
#pragma unroll
			for (int k = 0; k < j; ++k) s -= L[i * N + k] * L[j * N + k];
			L[i * N + j] = s / ljj;
		}
	}
#pragma unroll
	for (int i = 0; i < N; ++i)
	{
		double s = b[i];
#pragma unroll
		for (int k = 0; k < i; ++k) s -= L[i * N + k] * y[k];
		y[i] = s / L[i * N + i];
	}
#pragma unroll
	for (int i = N - 1; i >= 0; --i)
	{
		double s = y[i];
#pragma unroll
		for (int k = i + 1; k < N; ++k) s -= L[k * N + i] * x[k];
		x[i] = s / L[i * N + i];
	}
	return true;
}

// Least squares of A x = b (A is M x N row-major, full column rank) by Householder QR — EPnP's Gauss-Newton step
// (OpenCV epnp.cpp, epnp::qr_solve).  Same operation sequence as the oracle's qr_solve_ls (oracle/pnp_math.h); every
// index is a compile-time constant, so it runs out of registers with uniform control flow.
template <int M, int N>
__device__ inline bool qr_solve(double * A, double * b, double * x, double rel_tol = 0.0)
{
	double rdiag[N], v[M];
	double amax = 0;
#pragma unroll
	for (int k = 0; k < N; ++k)
	{
		double sigma = 0;
#pragma unroll
		for (int i = k; i < M; ++i) sigma += A[i * N + k] * A[i * N + k];
		if (sigma == 0.0) return false;
		const double akk = A[k * N + k];
		const double alpha = akk > 0 ? -sqrt(sigma) : sqrt(sigma);
		if (!(fabs(alpha) > rel_tol * amax)) return false;
		amax = fmax(amax, fabs(alpha));
		const double beta = 1.0 / (sigma - akk * alpha);
		v[k] = akk - alpha;
#pragma unroll
		for (int i = k + 1; i < M; ++i) v[i] = A[i * N + k];
#pragma unroll
		for (int j = k + 1; j < N; ++j)
		{
			double s = 0;
#pragma unroll
			for (int i = k; i < M; ++i) s += v[i] * A[i * N + j];
			s *= beta;
#pragma unroll
			for (int i = k; i < M; ++i) A[i * N + j] -= s * v[i];
		}
		double s = 0;
#pragma unroll
		for (int i = k; i < M; ++i) s += v[i] * b[i];
		s *= beta;
#pragma unroll
		for (int i = k; i < M; ++i) b[i] -= s * v[i];
		rdiag[k] = alpha;
	}
#pragma unroll
	for (int k = N - 1; k >= 0; --k)
	{
		double s = b[k];
#pragma unroll
		for (int j = k + 1; j < N; ++j) s -= A[k * N + j] * x[j];
		x[k] = s / rdiag[k];
	}
	return true;
}

// cvSolve(A, b, x, CV_SVD) of EPnP's find_betas_approx_*: guarded QR, eigen pseudo-inverse as the fallback (oracle: ls_solve)
template <int M, int N>
__device__ inline void ls_solve(const double * A, const double * b, double * x)
{
	double Ac[M * N], bc[M];
#pragma unroll
	for (int i = 0; i < M * N; ++i) Ac[i] = A[i];
#pragma unroll
	for (int i = 0; i < M; ++i) bc[i] = b[i];
	if (qr_solve<M, N>(Ac, bc, x, 1e-8)) return;
	solve_ls<M, N>(A, b, x);
}

// SVD of a 3x3 matrix M = U diag(w) V^T; U, V row-major with singular vectors as columns
__device__ inline void svd3(const double * M, double * U, double * w, double * V)
{
	double mtm[9], vv[9];
	int ord[3];
	for (int i = 0; i < 3; ++i)
		for (int j = 0; j < 3; ++j)
		{
			double s = 0;
			for (int k = 0; k < 3; ++k) s += M[k * 3 + i] * M[k * 3 + j];
			mtm[i * 3 + j] = s;
		}
	sym_eigen<3>(mtm, vv, ord);
	for (int k = 0; k < 3; ++k)
	{
		const double e = mtm[ord[k] * 3 + ord[k]];
		w[k] = sqrt(e > 0.0 ? e : 0.0);
		for (int i = 0; i < 3; ++i) V[i * 3 + k] = vv[i * 3 + ord[k]];
	}
	for (int k = 0; k < 3; ++k)
	{
		double u[3];
		for (int i = 0; i < 3; ++i) u[i] = M[i * 3 + 0] * V[0 * 3 + k] + M[i * 3 + 1] * V[1 * 3 + k] + M[i * 3 + 2] * V[2 * 3 + k];
		const double nrm = sqrt(u[0] * u[0] + u[1] * u[1] + u[2] * u[2]);
		if (nrm > 1e-12 * (w[0] + 1e-300))
		{
			for (int i = 0; i < 3; ++i) U[i * 3 + k] = u[i] / nrm;
		}
		else
		{
			const int a = (k + 1) % 3, b = (k + 2) % 3;
			U[0 * 3 + k] = U[1 * 3 + a] * U[2 * 3 + b] - U[2 * 3 + a] * U[1 * 3 + b];
			U[1 * 3 + k] = U[2 * 3 + a] * U[0 * 3 + b] - U[0 * 3 + a] * U[2 * 3 + b];
			U[2 * 3 + k] = U[0 * 3 + a] * U[1 * 3 + b] - U[1 * 3 + a] * U[0 * 3 + b];
		}
	}
}

__device__ inline void mat3_inv(const double * m, double * inv)
{
	const double det = m[0] * (m[4] * m[8] - m[5] * m[7]) - m[1] * (m[3] * m[8] - m[5] * m[6]) + m[2] * (m[3] * m[7] - m[4] * m[6]);
	const double id = 1.0 / det;
	inv[0] = (m[4] * m[8] - m[5] * m[7]) * id;
	inv[1] = (m[2] * m[7] - m[1] * m[8]) * id;
	inv[2] = (m[1] * m[5] - m[2] * m[4]) * id;
	inv[3] = (m[5] * m[6] - m[3] * m[8]) * id;
	inv[4] = (m[0] * m[8] - m[2] * m[6]) * id;
	inv[5] = (m[2] * m[3] - m[0] * m[5]) * id;
	inv[6] = (m[3] * m[7] - m[4] * m[6]) * id;
	inv[7] = (m[1] * m[6] - m[0] * m[7]) * id;
	inv[8] = (m[0] * m[4] - m[1] * m[3]) * id;
}

// cv::Rodrigues vector -> matrix (+ optional jacobian J[3][9] = dR(k)/dr(i))
__device__ inline void rodrigues_v2m(const double * r, double * R, double * J)
{
	const double theta = sqrt(r[0] * r[0] + r[1] * r[1] + r[2] * r[2]);
	if (theta < 2.220446049250313e-16)
	{
		for (int k = 0; k < 9; ++k) R[k] = (k % 4 == 0) ? 1.0 : 0.0;
		if (J)
		{
			for (int k = 0; k < 27; ++k) J[k] = 0;
			J[5] = J[15] = J[19] = -1;
			J[7] = J[11] = J[21] = 1;
		}
		return;
	}
	const double c = cos(theta), s = sin(theta), c1 = 1.0 - c, itheta = 1.0 / theta;
	const double rx = r[0] * itheta, ry = r[1] * itheta, rz = r[2] * itheta;
	const double rrt[9] = {rx * rx, rx * ry, rx * rz, rx * ry, ry * ry, ry * rz, rx * rz, ry * rz, rz * rz};
	const double r_x[9] = {0, -rz, ry, rz, 0, -rx, -ry, rx, 0};
	for (int k = 0; k < 9; ++k) R[k] = c * ((k % 4 == 0) ? 1.0 : 0.0) + c1 * rrt[k] + s * r_x[k];
	if (J)
	{
		const double drrt[27] = {rx + rx, ry, rz, ry, 0, 0, rz, 0, 0, 0, rx, 0, rx, ry + ry, rz, 0, rz, 0, 0, 0, rx, 0, 0, ry, rx, ry, rz + rz};
		const double d_r_x[27] = {0, 0, 0, 0, 0, -1, 0, 1, 0, 0, 0, 1, 0, 0, 0, -1, 0, 0, 0, -1, 0, 1, 0, 0, 0, 0, 0};
		for (int i = 0; i < 3; ++i)
		{
			const double ri = i == 0 ? rx : i == 1 ? ry : rz;
			const double a0 = -s * ri, a1 = (s - 2 * c1 * itheta) * ri, a2 = c1 * itheta;
			const double a3 = (c - s * itheta) * ri, a4 = s * itheta;
			for (int k = 0; k < 9; ++k)
				J[i * 9 + k] = a0 * ((k % 4 == 0) ? 1.0 : 0.0) + a1 * rrt[k] + a2 * drrt[i * 9 + k] + a3 * r_x[k] + a4 * d_r_x[i * 9 + k];
		}
	}
}

// cv::Rodrigues matrix -> vector (re-orthonormalised by SVD first)
__device__ inline void rodrigues_m2v(const double * Rin, double * r)
{
	double U[9], w[3], V[9], R[9];
	svd3(Rin, U, w, V);
	for (int i = 0; i < 3; ++i)
		for (int j = 0; j < 3; ++j) R[i * 3 + j] = U[i * 3 + 0] * V[j * 3 + 0] + U[i * 3 + 1] * V[j * 3 + 1] + U[i * 3 + 2] * V[j * 3 + 2];
	double rx = R[7] - R[5], ry = R[2] - R[6], rz = R[3] - R[1];
	const double s = sqrt((rx * rx + ry * ry + rz * rz) * 0.25);
	double c = (R[0] + R[4] + R[8] - 1) * 0.5;
	c = c > 1. ? 1. : c < -1. ? -1. : c;
	const double theta = acos(c);
	if (s < 1e-5)
	{
		if (c > 0)
		{
			r[0] = r[1] = r[2] = 0;
		}
		else
		{
			double t;
			t = (R[0] + 1) * 0.5;
			rx = sqrt(t > 0. ? t : 0.);
			t = (R[4] + 1) * 0.5;
			ry = sqrt(t > 0. ? t : 0.) * (R[1] < 0 ? -1. : 1.);
			t = (R[8] + 1) * 0.5;
			rz = sqrt(t > 0. ? t : 0.) * (R[2] < 0 ? -1. : 1.);
			if (fabs(rx) < fabs(ry) && fabs(rx) < fabs(rz) && (R[5] > 0) != (ry * rz > 0)) rz = -rz;
			const double k = theta / sqrt(rx * rx + ry * ry + rz * rz);
			r[0] = rx * k;
			r[1] = ry * k;
			r[2] = rz * k;
		}
	}
	else
	{
		const double vth = 1 / (2 * s) * theta;
		r[0] = rx * vth;
		r[1] = ry * vth;
		r[2] = rz * vth;
	}
}

// ------------------------------------------------------------------------------------- EPnP (n = 6)
struct Epnp6
{
	CamK cam;
	double pws[18], us[12], alphas[24], pcs[18];
	double cws[4][3], ccs[4][3];

	__device__ void choose_control_points()
	{
		const int n = 6;
		cws[0][0] = cws[0][1] = cws[0][2] = 0;
		for (int i = 0; i < n; ++i)
			for (int j = 0; j < 3; ++j) cws[0][j] += pws[3 * i + j];
		for (int j = 0; j < 3; ++j) cws[0][j] /= n;
		double ptp[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
		for (int i = 0; i < n; ++i)
		{
			double d[3];
			for (int j = 0; j < 3; ++j) d[j] = pws[3 * i + j] - cws[0][j];
			for (int a = 0; a < 3; ++a)
				for (int b = 0; b < 3; ++b) ptp[3 * a + b] += d[a] * d[b];
		}
		double dc[3], uct[9];
		for (int a = 0; a < 3; ++a)
			for (int b = 0; b < 3; ++b) uct[3 * a + b] = ptp[3 * b + a];
		svd_rows_jacobi3(uct, dc);
		for (int i = 1; i < 4; ++i)
		{
			const double k = sqrt((dc[i - 1] > 0.0 ? dc[i - 1] : 0.0) / n);
			for (int j = 0; j < 3; ++j) cws[i][j] = cws[0][j] + k * uct[3 * (i - 1) + j];
		}
	}

	__device__ void compute_barycentric_coordinates()
	{
		double cc[9], cci[9];
		for (int i = 0; i < 3; ++i)
			for (int j = 1; j < 4; ++j) cc[3 * i + j - 1] = cws[j][i] - cws[0][i];
		mat3_inv(cc, cci);
		for (int i = 0; i < 6; ++i)
		{
			const double * pi = &pws[3 * i];
			double * a = &alphas[4 * i];
			for (int j = 0; j < 3; ++j)
				a[1 + j] = cci[3 * j] * (pi[0] - cws[0][0]) + cci[3 * j + 1] * (pi[1] - cws[0][1]) + cci[3 * j + 2] * (pi[2] - cws[0][2]);
			a[0] = 1.0 - a[1] - a[2] - a[3];
		}
	}

	// v[i] = the eigenvector of the (i+1)-th SMALLEST eigenvalue (12 values)
	__device__ double compute_R_and_t(const double * vecs, const int * ord, const double * betas, double * R, double * t)
	{
		for (int i = 0; i < 4; ++i) ccs[i][0] = ccs[i][1] = ccs[i][2] = 0;
		for (int i = 0; i < 4; ++i)
		{
			const int col = ord[11 - i];
			for (int j = 0; j < 4; ++j)
				for (int k = 0; k < 3; ++k) ccs[j][k] += betas[i] * vecs[(3 * j + k) * 12 + col];
		}
		for (int i = 0; i < 6; ++i)
		{
			const double * a = &alphas[4 * i];
			for (int j = 0; j < 3; ++j) pcs[3 * i + j] = a[0] * ccs[0][j] + a[1] * ccs[1][j] + a[2] * ccs[2][j] + a[3] * ccs[3][j];
		}
		if (pcs[2] < 0.0)
		{
			for (int i = 0; i < 4; ++i)
				for (int j = 0; j < 3; ++j) ccs[i][j] = -ccs[i][j];
			for (int i = 0; i < 18; ++i) pcs[i] = -pcs[i];
		}
		// estimate_R_and_t
		double pc0[3] = {0, 0, 0}, pw0[3] = {0, 0, 0};
		for (int i = 0; i < 6; ++i)
			for (int j = 0; j < 3; ++j)
			{
				pc0[j] += pcs[3 * i + j];
				pw0[j] += pws[3 * i + j];
			}
		for (int j = 0; j < 3; ++j)
		{
			pc0[j] /= 6;
			pw0[j] /= 6;
		}
		double abt[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
		for (int i = 0; i < 6; ++i)
			for (int j = 0; j < 3; ++j)
				for (int k = 0; k < 3; ++k) abt[3 * j + k] += (pcs[3 * i + j] - pc0[j]) * (pws[3 * i + k] - pw0[k]);
		double U[9], w[3], V[9];
		svd3(abt, U, w, V);
		for (int i = 0; i < 3; ++i)
			for (int j = 0; j < 3; ++j) R[3 * i + j] = U[3 * i] * V[3 * j] + U[3 * i + 1] * V[3 * j + 1] + U[3 * i + 2] * V[3 * j + 2];
		const double det = R[0] * R[4] * R[8] + R[1] * R[5] * R[6] + R[2] * R[3] * R[7] - R[2] * R[4] * R[6] - R[1] * R[3] * R[8] - R[0] * R[5] * R[7];
		if (det < 0)
		{
			R[6] = -R[6];
			R[7] = -R[7];
			R[8] = -R[8];
		}
		for (int i = 0; i < 3; ++i) t[i] = pc0[i] - (R[3 * i] * pw0[0] + R[3 * i + 1] * pw0[1] + R[3 * i + 2] * pw0[2]);
		// reprojection_error
		double sum2 = 0.0;
		for (int i = 0; i < 6; ++i)
		{
			const double * pw = &pws[3 * i];
			const double Xc = R[0] * pw[0] + R[1] * pw[1] + R[2] * pw[2] + t[0];
			const double Yc = R[3] * pw[0] + R[4] * pw[1] + R[5] * pw[2] + t[1];
			const double inv_Zc = 1.0 / (R[6] * pw[0] + R[7] * pw[1] + R[8] * pw[2] + t[2]);
			const double ue = cam.uc + cam.fu * Xc * inv_Zc, ve = cam.vc + cam.fv * Yc * inv_Zc;
			const double u = us[2 * i], v = us[2 * i + 1];
			sum2 += sqrt((u - ue) * (u - ue) + (v - ve) * (v - ve));
		}
		return sum2 / 6;
	}

	__device__ static void gauss_newton(const double * l, const double * rho, double * betas)
	{
		for (int it = 0; it < 5; ++it)
		{
			double A[24], b[6], x[4];
			for (int i = 0; i < 6; ++i)
			{
				const double * rl = l + 10 * i;
				double * ra = A + 4 * i;
				ra[0] = 2 * rl[0] * betas[0] + rl[1] * betas[1] + rl[3] * betas[2] + rl[6] * betas[3];
				ra[1] = rl[1] * betas[0] + 2 * rl[2] * betas[1] + rl[4] * betas[2] + rl[7] * betas[3];
				ra[2] = rl[3] * betas[0] + rl[4] * betas[1] + 2 * rl[5] * betas[2] + rl[8] * betas[3];
				ra[3] = rl[6] * betas[0] + rl[7] * betas[1] + rl[8] * betas[2] + 2 * rl[9] * betas[3];
				b[i] = rho[i] - (rl[0] * betas[0] * betas[0] + rl[1] * betas[0] * betas[1] + rl[2] * betas[1] * betas[1] +
				                 rl[3] * betas[0] * betas[2] + rl[4] * betas[1] * betas[2] + rl[5] * betas[2] * betas[2] +
				                 rl[6] * betas[0] * betas[3] + rl[7] * betas[1] * betas[3] + rl[8] * betas[2] * betas[3] +
				                 rl[9] * betas[3] * betas[3]);
			}
			if (!qr_solve<6, 4>(A, b, x)) return;
			for (int i = 0; i < 4; ++i) betas[i] += x[i];
		}
	}

	// returns false when the pose is not finite
	long long * clk = nullptr; // diagnostics: clock64() after each stage
	__device__ bool compute_pose(double * R, double * t)
	{
		if (clk) clk[0] = clock64();
		choose_control_points();
		compute_barycentric_coordinates();
		double mtm[144], vecs[144];
		int ord[12];
		for (int k = 0; k < 144; ++k) mtm[k] = 0;
		for (int i = 0; i < 6; ++i)
		{
			const double * as = &alphas[4 * i];
			double m1[12], m2[12];
			for (int k = 0; k < 4; ++k)
			{
				m1[3 * k] = as[k] * cam.fu;
				m1[3 * k + 1] = 0.0;
				m1[3 * k + 2] = as[k] * (cam.uc - us[2 * i]);
				m2[3 * k] = 0.0;
				m2[3 * k + 1] = as[k] * cam.fv;
				m2[3 * k + 2] = as[k] * (cam.vc - us[2 * i + 1]);
			}
			for (int a = 0; a < 12; ++a)
				for (int b = 0; b < 12; ++b) mtm[a * 12 + b] += m1[a] * m1[b] + m2[a] * m2[b];
		}
		if (clk) clk[1] = clock64();
		sym_eigen<12>(mtm, vecs, ord, clk ? g_pnp_dbg : nullptr);
		if (clk) clk[2] = clock64();
		// L_6x10 and rho
		double l[60], rho[6];
		{
			double dv[4][6][3];
			for (int i = 0; i < 4; ++i)
			{
				const int col = ord[11 - i];
				int a = 0, b = 1;
				for (int j = 0; j < 6; ++j)
				{
					for (int k = 0; k < 3; ++k) dv[i][j][k] = vecs[(3 * a + k) * 12 + col] - vecs[(3 * b + k) * 12 + col];
					if (++b > 3)
					{
						++a;
						b = a + 1;
					}
				}
			}
#define LCD_DOT3(x, y) ((x)[0] * (y)[0] + (x)[1] * (y)[1] + (x)[2] * (y)[2])
			for (int i = 0; i < 6; ++i)
			{
				double * row = l + 10 * i;
				row[0] = LCD_DOT3(dv[0][i], dv[0][i]);
				row[1] = 2.0 * LCD_DOT3(dv[0][i], dv[1][i]);
				row[2] = LCD_DOT3(dv[1][i], dv[1][i]);
				row[3] = 2.0 * LCD_DOT3(dv[0][i], dv[2][i]);
				row[4] = 2.0 * LCD_DOT3(dv[1][i], dv[2][i]);
				row[5] = LCD_DOT3(dv[2][i], dv[2][i]);
				row[6] = 2.0 * LCD_DOT3(dv[0][i], dv[3][i]);
				row[7] = 2.0 * LCD_DOT3(dv[1][i], dv[3][i]);
				row[8] = 2.0 * LCD_DOT3(dv[2][i], dv[3][i]);
				row[9] = LCD_DOT3(dv[3][i], dv[3][i]);
			}
#undef LCD_DOT3
			int a = 0, b = 1;
			for (int j = 0; j < 6; ++j)
			{
				rho[j] = (cws[a][0] - cws[b][0]) * (cws[a][0] - cws[b][0]) + (cws[a][1] - cws[b][1]) * (cws[a][1] - cws[b][1]) +
				         (cws[a][2] - cws[b][2]) * (cws[a][2] - cws[b][2]);
				if (++b > 3)
				{
					++a;
					b = a + 1;
				}
			}
		}
		double best_rep = 0;
		bool have = false;
		for (int approx = 1; approx <= 3; ++approx)
		{
			double betas[4];
			if (approx == 1)
			{
				double A[24], b4[4];
				for (int i = 0; i < 6; ++i)
				{
					A[4 * i] = l[10 * i];
					A[4 * i + 1] = l[10 * i + 1];
					A[4 * i + 2] = l[10 * i + 3];
					A[4 * i + 3] = l[10 * i + 6];
				}
				ls_solve<6, 4>(A, rho, b4);
				if (b4[0] < 0)
				{
					betas[0] = sqrt(-b4[0]);
					betas[1] = -b4[1] / betas[0];
					betas[2] = -b4[2] / betas[0];
					betas[3] = -b4[3] / betas[0];
				}
				else
				{
					betas[0] = sqrt(b4[0]);
					betas[1] = b4[1] / betas[0];
					betas[2] = b4[2] / betas[0];
					betas[3] = b4[3] / betas[0];
				}
			}
			else if (approx == 2)
			{
				double A[18], b3[3];
				for (int i = 0; i < 6; ++i)
				{
					A[3 * i] = l[10 * i];
					A[3 * i + 1] = l[10 * i + 1];
					A[3 * i + 2] = l[10 * i + 2];
				}
				ls_solve<6, 3>(A, rho, b3);
				if (b3[0] < 0)
				{
					betas[0] = sqrt(-b3[0]);
					betas[1] = (b3[2] < 0) ? sqrt(-b3[2]) : 0.0;
				}
				else
				{
					betas[0] = sqrt(b3[0]);
					betas[1] = (b3[2] > 0) ? sqrt(b3[2]) : 0.0;
				}
				if (b3[1] < 0) betas[0] = -betas[0];
				betas[2] = 0.0;
				betas[3] = 0.0;
			}
			else
			{
				double A[30], b5[5];
				for (int i = 0; i < 6; ++i)
					for (int j = 0; j < 5; ++j) A[5 * i + j] = l[10 * i + j];
				ls_solve<6, 5>(A, rho, b5);
				if (b5[0] < 0)
				{
					betas[0] = sqrt(-b5[0]);
					betas[1] = (b5[2] < 0) ? sqrt(-b5[2]) : 0.0;
				}
				else
				{
					betas[0] = sqrt(b5[0]);
					betas[1] = (b5[2] > 0) ? sqrt(b5[2]) : 0.0;
				}
				if (b5[1] < 0) betas[0] = -betas[0];
				betas[2] = b5[3] / betas[0];
				betas[3] = 0.0;
			}
			const long long t_a = clk ? clock64() : 0;
			gauss_newton(l, rho, betas);
			const long long t_b = clk ? clock64() : 0;
			double Rc[9], tc[3];
			const double rep = compute_R_and_t(vecs, ord, betas, Rc, tc);
			if (clk)
			{
				g_pnp_dbg[1 + approx] = t_b - t_a;
				g_pnp_dbg[4 + approx] = clock64() - t_b;
			}
			// N = 1; if (rep[2] < rep[1]) N = 2; if (rep[3] < rep[N]) N = 3;
			if (!have || rep < best_rep)
			{
				have = true;
				best_rep = rep;
				for (int k = 0; k < 9; ++k) R[k] = Rc[k];
				for (int k = 0; k < 3; ++k) t[k] = tc[k];
			}
		}
		return isfinite(t[0]) && isfinite(t[1]) && isfinite(t[2]);
	}
};

// cv::solvePnP(SOLVEPNP_EPNP) on six correspondences (object float xyz, image float pixels, no distortion):
// undistortPoints stores the normalised coordinates as float before EPnP multiplies them back.
__device__ inline bool solve_pnp_epnp6(const float * X, const float * uv, const int * idx, const CamK & cam, double * rvec, double * tvec,
                                       long long * clk = nullptr)
{
	Epnp6 e;
	e.cam = cam;
	e.clk = clk;
	for (int i = 0; i < 6; ++i)
	{
		const float * p = X + 3 * idx[i];
		const float * q = uv + 2 * idx[i];
		e.pws[3 * i] = p[0];
		e.pws[3 * i + 1] = p[1];
		e.pws[3 * i + 2] = p[2];
		const float xn = static_cast<float>((static_cast<double>(q[0]) - cam.uc) / cam.fu);
		const float yn = static_cast<float>((static_cast<double>(q[1]) - cam.vc) / cam.fv);
		e.us[2 * i] = static_cast<double>(xn) * cam.fu + cam.uc;
		e.us[2 * i + 1] = static_cast<double>(yn) * cam.fv + cam.vc;
	}
	double R[9], t[3];
	if (!e.compute_pose(R, t)) return false;
	if (clk) clk[3] = clock64();
	rodrigues_m2v(R, rvec);
	tvec[0] = t[0];
	tvec[1] = t[1];
	tvec[2] = t[2];
	return isfinite(rvec[0]) && isfinite(rvec[1]) && isfinite(rvec[2]);
}

// projection of one point (cv::projectPoints, no distortion): uv double
__device__ inline void project_point(const double * R, const double * t, const CamK & cam, const float * X, double & u, double & v)
{
	const double x = R[0] * X[0] + R[1] * X[1] + R[2] * X[2] + t[0];
	const double y = R[3] * X[0] + R[4] * X[1] + R[5] * X[2] + t[1];
	double z = R[6] * X[0] + R[7] * X[1] + R[8] * X[2] + t[2];
	z = z ? 1. / z : 1;
	u = x * z * cam.fu + cam.uc;
	v = y * z * cam.fv + cam.vc;
}

// PnPRansacCallback::computeError for one point: (float)norm(ipt - (Point2f)proj)
__device__ inline float reproj_err(const double * R, const double * t, const CamK & cam, const float * X, const float * uv)
{
	double u, v;
	project_point(R, t, cam, X, u, v);
	const float dx = uv[0] - static_cast<float>(u), dy = uv[1] - static_cast<float>(v);
	return static_cast<float>(sqrt(static_cast<double>(dx) * dx + static_cast<double>(dy) * dy));
}

} // namespace lcd
