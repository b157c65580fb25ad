// decide.cuh — Rtabmap::process's loop-closure decision for many localisation clients against one shared map.
//
// Replaces, per client, BayesFilter::computePosterior (corelib/src/BayesFilter.cpp:145-270) and the hypothesis selection and checks of
// Rtabmap::process (Rtabmap.cpp:2143-2226), then turns the verification of the accepted hypothesis into the decision (:3156-3191).
// Every client is one Rtabmap in localisation mode with its own Bayes filter state and its own last highest hypothesis; the map, and
// so the prediction matrix, is shared.  The prediction's columns are computed once per map by bayes_column (bayes.cuh), bit-equal to
// lcd_bayes_compute_posterior's; what is left per frame is
//     prior[r][b] = U[b] + sum over the columns c that list r of (P[r][c] - u_c) last[c][b]  (+ the virtual-place column),
// with the listed entries stored by ROW (transposed at set_map), so each row gathers its entries without atomics, and the batch's
// last posteriors stored [place][frame], so an entry reads B contiguous values.  Every sum over places (U, the real places' last
// posterior, the posterior sum) runs in a fixed order that depends on the number of places only: a frame's posterior is the same
// bits whatever the batch size, its position in the batch and the other clients in it.
#pragma once
#include "bayes.cuh"

namespace lcd {

constexpr int kDcColChunk = 256;   // columns per partial sum of U and of the last posterior
constexpr int kDcRowChunk = 32;    // rows per partial posterior sum
constexpr int kDcThreads = 128;    // frames per CTA in the column and row passes (more frames: the CTA loops)

// decision statuses and frame flags (lcd_b200.h)
constexpr int kDcSkipped = 0, kDcHeld = 1, kDcNoHypothesis = 2, kDcUnderThreshold = 3, kDcUnderRatio = 4, kDcSingle = 5, kDcRatio = 6,
              kDcLastNull = 7, kDcAccepted = 8, kDcVerifyRejected = 9, kDcDistanceRejected = 10;
constexpr int kDcFlagSkip = 1, kDcFlagHold = 2, kDcFlagAggressive = 4;

struct Decision
{
	int highest_id;
	float highest_value;
	int loop_id;
	int status;
};

// the map's shared tables (lcd_clients_set_map)
struct DecideMap
{
	int n;                  // places, ids[0] = the virtual place
	const int * ids;        // [n] ascending
	const float * col_u;    // [n] uniform value of each column
	const int * t_ptr;      // [n+1] listed entries by row (row 0, the virtual place, has none)
	const int * t_col;      // [nt] column of each entry, ascending inside a row
	const double * t_val;   // [nt] P[r][c] - u_c
	double lc0;             // Bayes/PredictionLC[0] (P[0][c] of every real place, as a float)
	float vpp;              // Bayes/VirtualPlacePriorThr
};

// set_map: the listed entries in row order, k -> (entry e of column c, row r); t_val[k] = P[r][c] - u_c in double
__global__ void decide_entry_values_kernel(const BayesArgs a, int nt, const int * __restrict__ t_entry, const int * __restrict__ t_col,
                                           double * __restrict__ t_val)
{
	const int k = blockIdx.x * blockDim.x + threadIdx.x;
	if (k >= nt) return;
	const int e = t_entry[k], c = t_col[k];
	const float pv = bayes_entry_value(a, e, c, a.nbr_row[e]);
	t_val[k] = static_cast<double>(pv) - static_cast<double>(a.col_u[c]);
}

// set_map: the columns (u, scale, delta) once per map, bit-equal to bayes_columns_kernel's
__global__ void decide_map_columns_kernel(const BayesArgs a)
{
	const int c = blockIdx.x * blockDim.x + threadIdx.x;
	if (c >= a.n) return;
	const BayesColumn col = bayes_column(a, c);
	a.col_u[c] = col.u;
	a.col_scale[c] = col.scale;
	a.col_delta[c] = col.delta;
}

// per-call tables of the B frames that compute a posterior (frames without LCD_FRAME_SKIP / HOLD)
struct DecideBatch
{
	int B;
	const long long * frame;    // [B] frame index in the call
	const long long * client;   // [B]
	const long long * prev_n;   // [B] places of the client's last posterior (0 = empty state)
	const long long * prev_ids; // [B] device address of the ids the client's last posterior is keyed to
	const float * cl_post;      // [client][stride] the clients' last posteriors
	long long stride;
	const float * adj;          // [n_frames][n] adjusted likelihood (element 0 = the virtual place)
	float * last_t;             // [n][B] last posterior re-keyed to the map (updatePosterior)
	float * post_t;             // [n][B] unnormalised posterior
	double * part_u;            // [col chunks][B]
	double * part_s1;           // [col chunks][B]
	double * part_p;            // [row chunks][B]
	double * u;                 // [B] U
	double * s1;                // [B] sum of the real places' last posterior
	double * psum;              // [B] posterior sum (normalised by it as a float, as the reference does)
};

__global__ void decide_last_kernel(const DecideMap m, const DecideBatch d)
{
	const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
	if (i >= static_cast<long long>(m.n) * d.B) return;
	const int r = static_cast<int>(i / d.B), b = static_cast<int>(i % d.B);
	const int * prev_ids = reinterpret_cast<const int *>(d.prev_ids[b]);
	const float * prev = d.cl_post + d.client[b] * d.stride;
	d.last_t[i] = bayes_rekey(prev_ids, prev, static_cast<int>(d.prev_n[b]), m.ids[r]);
}

// partial U and last-posterior sums over a chunk of columns, each frame's columns added in ascending order
__global__ void __launch_bounds__(kDcThreads) decide_columns_kernel(const DecideMap m, const DecideBatch d)
{
	const int c0 = blockIdx.x * kDcColChunk, c1 = min(m.n, c0 + kDcColChunk);
	for (int b = threadIdx.x; b < d.B; b += blockDim.x)
	{
		double u = 0.0, s1 = 0.0;
		for (int c = c0; c < c1; ++c)
		{
			if (m.ids[c] < 0) continue;
			const float last = d.last_t[static_cast<size_t>(c) * d.B + b];
			const double up = static_cast<double>(m.col_u[c]) * static_cast<double>(last);
			if (up != 0.0) u += up;
			s1 += static_cast<double>(last);
		}
		d.part_u[static_cast<size_t>(blockIdx.x) * d.B + b] = u;
		d.part_s1[static_cast<size_t>(blockIdx.x) * d.B + b] = s1;
	}
}

// out[b] = sum over the chunks in ascending order of part[chunk][b]
__global__ void decide_sum_chunks_kernel(const double * __restrict__ part, int n_chunks, int B, double * __restrict__ out)
{
	const int b = blockIdx.x * blockDim.x + threadIdx.x;
	if (b >= B) return;
	double t = 0.0;
	for (int k = 0; k < n_chunks; ++k) t += part[static_cast<size_t>(k) * B + b];
	out[b] = t;
}

// prior -> unnormalised posterior of a chunk of rows, and the chunk's posterior sum; each frame's rows in ascending order
__global__ void __launch_bounds__(kDcThreads) decide_rows_kernel(const DecideMap m, const DecideBatch d)
{
	const int r0 = blockIdx.x * kDcRowChunk, r1 = min(m.n, r0 + kDcRowChunk);
	const float p00 = bayes_vp_p00(m.vpp, m.n);
	const float pr0 = m.n > 1 ? bayes_vp_pr0(m.vpp, m.n) : 0.f;
	const double lc0f = static_cast<double>(static_cast<float>(m.lc0));
	for (int b = threadIdx.x; b < d.B; b += blockDim.x)
	{
		const double last0 = static_cast<double>(d.last_t[b]);
		const double u = d.u[b];
		const float * like = d.adj + d.frame[b] * m.n;
		double psum = 0.0;
		for (int r = r0; r < r1; ++r)
		{
			double prior;
			if (r == 0) prior = static_cast<double>(p00) * last0 + lc0f * d.s1[b];
			else
			{
				double acc = 0.0;
				for (int k = m.t_ptr[r]; k < m.t_ptr[r + 1]; ++k)
					acc += m.t_val[k] * static_cast<double>(d.last_t[static_cast<size_t>(m.t_col[k]) * d.B + b]);
				prior = acc + u;
				prior += static_cast<double>(pr0) * last0;
			}
			const float post = __fmul_rn(like[r], static_cast<float>(prior));
			d.post_t[static_cast<size_t>(r) * d.B + b] = post;
			psum += static_cast<double>(post);
		}
		d.part_p[static_cast<size_t>(blockIdx.x) * d.B + b] = psum;
	}
}

// normalisation, transposed through shared memory: the client's new state [client][r] and the optional output [frame][r]
__global__ void decide_normalize_kernel(const DecideMap m, const DecideBatch d, float * __restrict__ cl_post, float * __restrict__ out)
{
	__shared__ float tile[32][33];
	const int r0 = blockIdx.x * 32, b0 = blockIdx.y * 32;
	for (int j = threadIdx.y; j < 32; j += blockDim.y)
	{
		const int r = r0 + j, b = b0 + threadIdx.x;
		if (r < m.n && b < d.B)
		{
			float v = d.post_t[static_cast<size_t>(r) * d.B + b];
			const float sum = static_cast<float>(d.psum[b]);
			if (sum != 0.f) v = __fdiv_rn(v, sum);
			tile[j][threadIdx.x] = v;
		}
	}
	__syncthreads();
	for (int j = threadIdx.y; j < 32; j += blockDim.y)
	{
		const int b = b0 + j, r = r0 + threadIdx.x;
		if (r < m.n && b < d.B)
		{
			const float v = tile[threadIdx.x][j];
			cl_post[d.client[b] * d.stride + r] = v;
			if (out) out[d.frame[b] * m.n + r] = v;
		}
	}
}

struct DecideSelect
{
	int n_frames;
	const long long * client;  // [n_frames]
	const long long * flags;   // [n_frames]
	const float * cl_post;     // [client][stride]
	long long stride;
	int * hi_id;               // [client] last highest hypothesis
	float * hi_val;
	float loop_thr, aggressive_loop_thr, loop_ratio;
	const int * sig_slot;      // signature store row of each id (nullptr: no store)
	int slot_cap;
	Decision * dec;            // [n_frames]
	int * hyp_id;              // [n_frames] accepted id or 0
	int * hyp_slot;            // [n_frames] its store row or -1
};

// Rtabmap.cpp:2143-2233 for one frame per CTA: the highest real-place posterior (scanned in descending id order with a strict '>', so
// ties go to the highest id), its value replaced by 1 - posterior(virtual place), then the threshold / single-hypothesis / ratio checks
__global__ void decide_select_kernel(const DecideMap m, const DecideSelect a)
{
	__shared__ float s_v[32];
	__shared__ int s_r[32];
	const int f = blockIdx.x;
	const int client = static_cast<int>(a.client[f]);
	const int flags = static_cast<int>(a.flags[f]);
	const bool compute = (flags & (kDcFlagSkip | kDcFlagHold)) == 0;
	float bv = 0.f;
	int br = -1;
	if (compute)
	{
		const float * post = a.cl_post + client * a.stride;
		for (int r = 1 + threadIdx.x; r < m.n; r += blockDim.x)
		{
			const float v = post[r];
			if (v > bv || (v == bv && br >= 0 && r > br))
			{
				bv = v;
				br = r;
			}
		}
	}
	for (int o = 16; o > 0; o >>= 1)
	{
		const float ov = __shfl_down_sync(0xFFFFFFFFu, bv, o);
		const int orr = __shfl_down_sync(0xFFFFFFFFu, br, o);
		if (orr >= 0 && (ov > bv || (ov == bv && orr > br)))
		{
			bv = ov;
			br = orr;
		}
	}
	if ((threadIdx.x & 31) == 0)
	{
		s_v[threadIdx.x >> 5] = bv;
		s_r[threadIdx.x >> 5] = br;
	}
	__syncthreads();
	if (threadIdx.x != 0) return;
	for (int w = 1; w < (blockDim.x >> 5); ++w)
		if (s_r[w] >= 0 && (s_v[w] > bv || (s_v[w] == bv && s_r[w] > br)))
		{
			bv = s_v[w];
			br = s_r[w];
		}
	const int last_id = a.hi_id[client];
	const float last_val = a.hi_val[client];
	Decision d{0, 0.f, 0, kDcSkipped};
	if (flags & kDcFlagSkip) d.status = kDcSkipped; // bad signature / intermediate node / empty working memory: highest = (0, 0)
	else if (flags & kDcFlagHold)
	{
		d.highest_id = last_id; // small displacement / too fast movement: highest = the last one (:2229-2233)
		d.highest_value = last_val;
		d.status = kDcHeld;
	}
	else
	{
		d.highest_id = br >= 0 ? m.ids[br] : 0;
		d.highest_value = __fsub_rn(1.0f, a.cl_post[client * a.stride]);
		d.status = kDcNoHypothesis;
		if (d.highest_id > 0)
		{
			float thr = a.loop_thr;
			if ((flags & kDcFlagAggressive) && thr > a.aggressive_loop_thr) thr = a.aggressive_loop_thr;
			if (d.highest_value >= thr)
			{
				if (m.n <= 2 && thr > 0.f) d.status = kDcSingle;
				else if (a.loop_ratio > 0.f && last_val != 0.f && d.highest_value < __fmul_rn(a.loop_ratio, last_val)) d.status = kDcRatio;
				else if (a.loop_ratio > 0.f && last_val == 0.f) d.status = kDcLastNull;
				else
				{
					d.status = kDcAccepted;
					d.loop_id = d.highest_id;
				}
			}
			else if (d.highest_value < __fmul_rn(a.loop_ratio, last_val)) d.status = kDcUnderRatio;
			else d.status = kDcUnderThreshold;
		}
	}
	a.hi_id[client] = d.highest_id;
	a.hi_val[client] = d.highest_value;
	a.dec[f] = d;
	int slot = -1;
	if (d.loop_id > 0 && a.sig_slot && d.loop_id < a.slot_cap) slot = a.sig_slot[d.loop_id];
	a.hyp_id[f] = d.loop_id;
	a.hyp_slot[f] = slot;
}

// Rtabmap.cpp:3156-3167 after the verification of the accepted hypotheses: a failed registration, or (max_dist > 0) a transform longer
// than RGBD/MaxLoopClosureDistance, rejects the loop closure (the last highest hypothesis is left as it is).  skip (may be null): frames
// whose hypothesis a proximity detection already registered (proximity.cuh), which keep their decision.
__global__ void decide_verified_kernel(int n_frames, const int * __restrict__ ok, const float * __restrict__ T, float max_dist,
                                       Decision * __restrict__ dec, int * __restrict__ hyp_id, const unsigned char * __restrict__ skip)
{
	const int f = blockIdx.x * blockDim.x + threadIdx.x;
	if (f >= n_frames || dec[f].status != kDcAccepted || (skip && skip[f])) return;
	int status = kDcAccepted;
	if (!ok[f]) status = kDcVerifyRejected;
	else if (max_dist > 0.f)
	{
		// Transform::getNorm = uNorm(x, y, z) in float; the inverse has the same norm
		const float x = T[12 * f + 3], y = T[12 * f + 7], z = T[12 * f + 11];
		const float norm = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)), __fmul_rn(z, z)));
		if (norm > max_dist) status = kDcDistanceRejected;
	}
	if (status != kDcAccepted)
	{
		dec[f].status = status;
		dec[f].loop_id = 0;
		hyp_id[f] = 0;
	}
}

__global__ void decide_reset_clients_kernel(const int * __restrict__ clients, int n, int * __restrict__ hi_id, float * __restrict__ hi_val)
{
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	hi_id[clients[i]] = 0;
	hi_val[clients[i]] = 0.f;
}

} // namespace lcd
