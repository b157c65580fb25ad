// bayes.cuh — the discrete Bayes filter over loop-closure hypotheses, prediction matrix in sparse form.
//
// Replaces rtabmap::BayesFilter::computePosterior (corelib/src/BayesFilter.cpp:145-270) with the prediction of generatePrediction
// (:301-420) / addNeighborProb (:272-299) / normalize (:437-505), SURVEY.md §8(f) #1.  The reference materialises a dense S x S float
// matrix (400 MB at 10 000 places) and multiplies it with the last posterior on the CPU.  A column of that matrix is
//     the LC value of every graph neighbour of the place (by margin)  +  one uniform value in every other row  +  the virtual-place row,
// i.e. sparse + rank one, so the product is   prior[r] = U + P[r][0] post[0] + sum over columns c that list r of (P[r][c] - u_c) post[c]
// with U = sum_c u_c post[c]: O(neighbours) instead of O(S^2).  Every column (its listed values, delta, uniform value, scale and
// epsilon cut) is bit-equal to the reference's float statements, including normalize's column sum, which adds the uniform value to a
// float once per filled row (repeated_fadd reproduces that loop without running it).  Only the product with the last posterior and
// the posterior sum are evaluated in double, so results agree with the dense float product to ~1e-6 relative (tolerance for float
// work: 1e-4).
#pragma once
#include "common.cuh"

namespace lcd {

struct BayesArgs
{
	int n;                    // places of this call (ids ascending, ids[0] < 0 = virtual place)
	int vp_used;              // ids[0] < 0
	const int * ids;
	const float * like;       // [n] (adjusted) likelihood
	const int * col_ptr;      // [n+1] neighbour lists per column (empty for the virtual place)
	const int * nbr_row;      // [nnz] row index (position in ids) of the neighbour, ascending inside a column
	const int * nbr_level;    // [nnz] graph margin 0..n_lc-2
	const double * lc;        // [n_lc] Bayes/PredictionLC {virtual place, loop closure, level 1, ...}
	int n_lc;
	float total;              // _totalPredictionLCValues (float sum of lc)
	float eps;                // _predictionEpsilon (smallest lc)
	float vpp;                // Bayes/VirtualPlacePriorThr
	const int * prev_ids;     // [n_prev] ids of the last posterior, ascending
	const float * prev_post;  // [n_prev]
	int n_prev;
	// work
	float * last;             // [n] last posterior re-keyed to ids (updatePosterior, :712-737)
	float * col_u;            // [n] uniform value of the column after scaling / epsilon cut
	float * col_scale;        // [n]
	float * col_delta;        // [n] mass added to the diagonal
	double * prior;           // [n]
	double * sums;            // [0] U, [1] sum of the real places' last posterior (for the virtual-place row), [2] posterior sum
	float * post;             // [n] output
};

// updatePosterior (:712-737) for one place: its value in the last posterior (ids ascending), 0 for a place the last posterior did not
// have, 1 for every place when the last posterior is empty
__device__ inline float bayes_rekey(const int * prev_ids, const float * prev_post, int n_prev, int id)
{
	float v = n_prev == 0 ? 1.0f : 0.0f;
	int lo = 0, hi = n_prev;
	while (lo < hi)
	{
		const int mid = (lo + hi) >> 1;
		if (prev_ids[mid] < id) lo = mid + 1;
		else hi = mid;
	}
	if (lo < n_prev && prev_ids[lo] == id) v = prev_post[lo];
	return v;
}

__global__ void bayes_last_kernel(const BayesArgs a)
{
	const int r = blockIdx.x * blockDim.x + threadIdx.x;
	if (r < 3) a.sums[r] = 0.0; // before the bound check: with fewer than 3 places the sums would keep the last call's values
	if (r >= a.n) return;
	a.last[r] = bayes_rekey(a.prev_ids, a.prev_post, a.n_prev, a.ids[r]);
	a.prior[r] = 0.0;
}

// s + value + value + ... (times adds, each rounded to nearest float) as normalize's fill loop computes it (BayesFilter.cpp:457-464),
// in a few steps per binade of s instead of one per add.  Inside one binade every add moves s by the same number of ulps, once one add
// inside the binade has been made: a round-half-even tie leaves the last bit even, and from an even s every later tie resolves the
// same way.  So after a literal add that stays in its binade, the run of adds that keeps s below the next power of two is one step.
// Adds that cross a binade, and sums below FLT_MIN, are made literally.  When an add leaves s unchanged (value under half an ulp, or a
// tie onto the even s) no later add can move it.
__host__ __device__ inline float repeated_fadd(float s, const float value, int times)
{
	while (times > 0)
	{
		const float before = s;
		s = s + value;
		--times;
		if (s == before) break;
		if (times == 0 || !(before >= 1.17549435e-38f) || ilogbf(s) != ilogbf(before)) continue;
		const int e = ilogbf(s);
		const int m = static_cast<int>(ldexpf(s, 23 - e));              // significand as an integer in [2^23, 2^24)
		const int d = static_cast<int>(ldexpf((s + value) - s, 23 - e)); // ulps of the next add (exact difference)
		if (d == 0) break;
		const int fit = (0xFFFFFF - m) / d;                              // adds whose result stays below 2^(e+1)
		const int k = times < fit ? times : fit;
		s = ldexpf(static_cast<float>(m + k * d), e - 23);
		times -= k;
	}
	return s;
}

// addNeighborProb + normalize of column c without materialising it: the uniform value of its unlisted rows (after scaling and the
// epsilon cut), its scale (negative: renormalised, the epsilon cut applies to the listed entries too) and the mass added to its diagonal
struct BayesColumn
{
	float u, scale, delta;
};

// listed (nullptr: every row): the rows of the places in this call's matrix; a.n then counts those places (the prediction of a frame
// whose place list was cut, Rtabmap.cpp:2046-2115: generatePrediction only sees the listed neighbours, BayesFilter.cpp:352-372)
__device__ inline BayesColumn bayes_column(const BayesArgs & a, int c, const unsigned char * listed = nullptr)
{
	if (a.ids[c] < 0) return BayesColumn{0.f, 1.f, 0.f};
	const int first = a.vp_used ? 1 : 0;
	float s = 0.f;
	int n_nonzero = 0;
	bool diag_zero = false;
	for (int e = a.col_ptr[c]; e < a.col_ptr[c + 1]; ++e)
	{
		if (listed && !listed[a.nbr_row[e]]) continue;
		const float v = static_cast<float>(a.lc[a.nbr_level[e] + 1]);
		s = __fadd_rn(s, v);
		if (a.nbr_row[e] < first) continue;
		if (v != 0.f) ++n_nonzero;
		else if (a.nbr_row[e] == c) diag_zero = true;
	}
	float delta = 0.f;
	const double lc0 = a.lc[0];
	if (static_cast<double>(s) < static_cast<double>(a.total) - lc0)
	{
		delta = static_cast<float>(static_cast<double>(a.total) - lc0 - static_cast<double>(s));
		s = __fadd_rn(s, delta);
	}
	// the fill below sees the diagonal after delta: a place whose own (margin-0) value is 0 is not filled once delta made it non-zero
	if (diag_zero && delta != 0.f) ++n_nonzero;
	float other = 0.f;
	if (a.total < 1.f) other = __fsub_rn(1.0f, a.total);
	float value = 0.f;
	if (other > 0.f && a.n > 1)
	{
		value = __fdiv_rn(other, static_cast<float>(a.n - 1));
		const int zeros = (a.n - first) - n_nonzero;
		s = repeated_fadd(s, value, zeros);
	}
	const float max_norm = static_cast<float>(1.0 - (a.vp_used ? lc0 : 0.0));
	float scale = 1.f;
	if (static_cast<double>(s) < static_cast<double>(max_norm) - 0.0001 || static_cast<double>(s) > static_cast<double>(max_norm) + 0.0001)
	{
		scale = __fdiv_rn(max_norm, s);
		value = __fmul_rn(value, scale);
		if (value < a.eps) value = 0.f;
		return BayesColumn{value, -scale, delta};
	}
	return BayesColumn{value, 1.f, delta};
}

// P[r][c] of a listed entry with LC value v (float) in column col (the diagonal gets the column's delta)
__device__ inline float bayes_entry_pv(float v, bool diag, const BayesColumn & col, float eps)
{
	if (diag) v = __fadd_rn(v, col.delta);
	float pv = v;
	if (v == 0.f) pv = col.u; // a listed neighbour with a zero LC value is filled like any other zero row (already scaled)
	else if (col.scale < 0.f)
	{
		pv = __fmul_rn(v, -col.scale);
		if (pv < eps) pv = 0.f;
	}
	return pv;
}

// P[r][c] of listed entry e (row r of column c), the columns' values already in col_u / col_scale / col_delta
__device__ inline float bayes_entry_value(const BayesArgs & a, int e, int c, int r)
{
	return bayes_entry_pv(static_cast<float>(a.lc[a.nbr_level[e] + 1]), r == c, BayesColumn{a.col_u[c], a.col_scale[c], a.col_delta[c]}, a.eps);
}

// the virtual-place row and column (:375-411, :482-487): P[0][0], and P[r][0] of every real place r
__device__ inline float bayes_vp_p00(float vpp, int n) { return vpp > 0.f ? (n > 1 ? vpp : 1.0f) : (n > 1 ? static_cast<float>(1.0 / n) : 1.0f); }
__device__ inline float bayes_vp_pr0(float vpp, int n)
{
	return vpp > 0.f ? static_cast<float>((1.0 - static_cast<double>(vpp)) / (n - 1)) : static_cast<float>(1.0 / n);
}

// one thread per column: the column's values, and its share of U and of the real places' last-posterior sum
__global__ void bayes_columns_kernel(const BayesArgs a)
{
	const int c = blockIdx.x * blockDim.x + threadIdx.x;
	if (c >= a.n) return;
	const BayesColumn col = bayes_column(a, c);
	a.col_u[c] = col.u;
	a.col_scale[c] = col.scale;
	a.col_delta[c] = col.delta;
	if (a.ids[c] < 0) return;
	// U: the uniform part of this column reaches every row >= first
	const double up = static_cast<double>(col.u) * static_cast<double>(a.last[c]);
	if (up != 0.0) atomicAdd(&a.sums[0], up);
	atomicAdd(&a.sums[1], static_cast<double>(a.last[c]));
}

// one thread per listed entry: (P[r][c] - u_c) * last[c] onto prior[r]
__global__ void bayes_scatter_kernel(const BayesArgs a, int nnz, const int * __restrict__ entry_col)
{
	const int e = blockIdx.x * blockDim.x + threadIdx.x;
	if (e >= nnz) return;
	const int c = entry_col[e];
	const int r = a.nbr_row[e];
	const int first = a.vp_used ? 1 : 0;
	if (r < first) return; // the virtual-place row is set by the model, not by neighbours
	const float pv = bayes_entry_value(a, e, c, r);
	const double d = (static_cast<double>(pv) - static_cast<double>(a.col_u[c])) * static_cast<double>(a.last[c]);
	if (d != 0.0) atomicAdd(&a.prior[r], d);
}

// prior -> unnormalised posterior, and its sum
__global__ void bayes_update_kernel(const BayesArgs a)
{
	__shared__ double s_part[8];
	const int r = blockIdx.x * blockDim.x + threadIdx.x;
	double pv = 0.0;
	if (r < a.n)
	{
		double prior;
		const int first = a.vp_used ? 1 : 0;
		const double last0 = a.vp_used ? static_cast<double>(a.last[0]) : 0.0;
		if (a.vp_used && r == 0)
		{
			// row 0: P[0][0] = vpp (or 1 for a single place, or 1/n when vpp == 0), P[0][c] = lc[0] for every real place
			const float p00 = bayes_vp_p00(a.vpp, a.n);
			prior = static_cast<double>(p00) * last0 + static_cast<double>(static_cast<float>(a.lc[0])) * a.sums[1]; // sums[1]: real places only
		}
		else
		{
			prior = a.prior[r] + a.sums[0];
			if (a.vp_used)
			{
				const float pr0 = bayes_vp_pr0(a.vpp, a.n);
				prior += static_cast<double>(pr0) * last0;
			}
			(void)first;
		}
		const float pf = static_cast<float>(prior);
		const float post = __fmul_rn(a.like[r], pf);
		a.post[r] = post;
		pv = static_cast<double>(post);
	}
#pragma unroll
	for (int o = 16; o > 0; o >>= 1) pv += __shfl_down_sync(0xFFFFFFFFu, pv, o);
	if ((threadIdx.x & 31) == 0) s_part[threadIdx.x >> 5] = pv;
	__syncthreads();
	if (threadIdx.x == 0)
	{
		double t = 0.0;
		for (int w = 0; w < (blockDim.x >> 5); ++w) t += s_part[w];
		if (t != 0.0) atomicAdd(&a.sums[2], t);
	}
}

__global__ void bayes_normalize_kernel(const BayesArgs a, int * __restrict__ state_ids, float * __restrict__ state_post)
{
	const int r = blockIdx.x * blockDim.x + threadIdx.x;
	if (r >= a.n) return;
	const float sum = static_cast<float>(a.sums[2]);
	float v = a.post[r];
	if (sum != 0.f) v = __fdiv_rn(v, sum);
	a.post[r] = v;
	state_ids[r] = a.ids[r];
	state_post[r] = v;
}

} // namespace lcd
