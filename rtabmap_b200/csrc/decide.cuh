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
//
// A frame with a GPS fix (lcd_decide_gps_batch_dev) compares only the places within RGBD/LocalRadius of it (Rtabmap.cpp:2046-2115).
// Such a "gated" frame keeps the map's layout: its places that are not compared get a last posterior and an adjusted likelihood of
// exactly 0, so they add exact zeros to every fixed-order sum, and its prediction columns are recomputed over the compared rows only
// (decide_gps_columns_kernel).  A gate that keeps every place therefore gives the ungated bits.
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
	const float * t_lv;     // [nt] LC value of each listed entry, as a float (for the columns of gated frames)
	float eps;              // _predictionEpsilon
};

// the GPS filter of the place list (Rtabmap/LoopGPS, Rtabmap.cpp:2046-2115).  A place's geocentric point (GeodeticCoords::toGeocentric_WGS84, computed on the host) and the x, y, z of its offsetENU (Memory::getGPS).
struct GpsPlace
{
	double x, y, z;
	float ox, oy, oz;
	int fix; // stamp > 0: otherwise the place has no cache entry and is always compared (:2077)
};

// a frame's place list: kGpsNone computes nothing (skipped / held), kGpsAll compares every place, kGpsGated runs the filter with the
// frame's geocentric origin and the sines and cosines of its latitude and longitude (computed on the host)
constexpr int kGpsNone = 0, kGpsAll = 1, kGpsGated = 2;
struct GpsFrame
{
	double x, y, z, slat, clat, slon, clon, error;
	int mode;
	int pad;
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
	const int * key_n;          // [client] places of the client's last posterior (0 = empty state)
	const long long * key_ids;  // [client] device address of the ids the client's last posterior is keyed to
	const int * qn;             // [n_frames] quantised words of each frame, or nullptr: a frame with none is a bad signature
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
	// gated frames (nullptr in lcd_decide_batch_dev: no frame is gated)
	const GpsFrame * gps;       // [n_frames] kGpsGated: the frame compares only the places of listed
	const int * count;          // [n_frames] real places a gated frame compares
	const unsigned char * listed; // [n_frames][n] 1 = compared
	float * fu;                 // [n][B] columns of the gated frames: uniform value, scale, delta
	float * fscale;
	float * fdelta;
};

__device__ __forceinline__ bool decide_gated(const DecideBatch & d, int f) { return d.gps && d.gps[f].mode == kGpsGated; }

__global__ void decide_last_kernel(const DecideMap m, const DecideBatch d)
{
	const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
	if (i >= static_cast<long long>(m.n) * d.B) return;
	const int r = static_cast<int>(i / d.B), b = static_cast<int>(i % d.B);
	const long long c = d.client[b];
	const int * prev_ids = reinterpret_cast<const int *>(d.key_ids[c]);
	const float * prev = d.cl_post + c * d.stride;
	const int f = static_cast<int>(d.frame[b]);
	float v = bayes_rekey(prev_ids, prev, d.key_n[c], m.ids[r]);
	if (decide_gated(d, f) && !d.listed[static_cast<size_t>(f) * m.n + r]) v = 0.f; // updatePosterior over the compared ids only
	d.last_t[i] = v;
}

// the prediction's columns of every gated frame over its compared places (generatePrediction + normalize with cols = compared + 1);
// a column that is not compared gets (0, 1, 0), which its zero last posterior makes inert.  a: the map's columns (set_map's BayesArgs).
__global__ void decide_gps_columns_kernel(BayesArgs a, const DecideBatch d)
{
	const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
	if (i >= static_cast<long long>(a.n) * d.B) return;
	const int c = static_cast<int>(i / d.B), b = static_cast<int>(i % d.B);
	const int f = static_cast<int>(d.frame[b]);
	if (d.gps[f].mode != kGpsGated) return;
	const unsigned char * listed = d.listed + static_cast<size_t>(f) * a.n;
	BayesColumn col{0.f, 1.f, 0.f};
	if (listed[c])
	{
		a.n = d.count[f] + 1;
		col = bayes_column(a, c, listed);
	}
	d.fu[i] = col.u;
	d.fscale[i] = col.scale;
	d.fdelta[i] = col.delta;
}

// partial U and last-posterior sums over a chunk of columns, each frame's columns added in ascending order
__global__ void __launch_bounds__(kDcThreads) decide_columns_kernel(const DecideMap m, const DecideBatch d)
{
	const int c0 = blockIdx.x * kDcColChunk, c1 = min(m.n, c0 + kDcColChunk);
	for (int b = threadIdx.x; b < d.B; b += blockDim.x)
	{
		const float * col_u = decide_gated(d, static_cast<int>(d.frame[b])) ? d.fu : nullptr;
		double u = 0.0, s1 = 0.0;
		for (int c = c0; c < c1; ++c)
		{
			if (m.ids[c] < 0) continue;
			const float last = d.last_t[static_cast<size_t>(c) * d.B + b];
			const float cu = col_u ? col_u[static_cast<size_t>(c) * d.B + b] : m.col_u[c];
			const double up = static_cast<double>(cu) * static_cast<double>(last);
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
	const double lc0f = static_cast<double>(static_cast<float>(m.lc0));
	for (int b = threadIdx.x; b < d.B; b += blockDim.x)
	{
		const bool gated = decide_gated(d, static_cast<int>(d.frame[b]));
		const int n = gated ? d.count[d.frame[b]] + 1 : m.n; // places of the frame's matrix
		const float p00 = bayes_vp_p00(m.vpp, n);
		const float pr0 = n > 1 ? bayes_vp_pr0(m.vpp, n) : 0.f;
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
				if (!gated)
					for (int k = m.t_ptr[r]; k < m.t_ptr[r + 1]; ++k)
						acc += m.t_val[k] * static_cast<double>(d.last_t[static_cast<size_t>(m.t_col[k]) * d.B + b]);
				else
					for (int k = m.t_ptr[r]; k < m.t_ptr[r + 1]; ++k)
					{
						// decide_entry_values_kernel's P[r][c] - u_c, from the frame's own column c
						const int c = m.t_col[k];
						const size_t ci = static_cast<size_t>(c) * d.B + b;
						const BayesColumn col{d.fu[ci], d.fscale[ci], d.fdelta[ci]};
						const double tv = static_cast<double>(bayes_entry_pv(m.t_lv[k], r == c, col, m.eps)) - static_cast<double>(col.u);
						acc += tv * static_cast<double>(d.last_t[ci]);
					}
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

// a frame without quantised words (Signature::isBadSignature, Signature.cpp:341-344) is skipped as LCD_FRAME_SKIP skips it (Rtabmap.cpp:
// 1994-1999), even when the host put it into the batch: its columns are computed but nothing of it is written
__device__ __forceinline__ bool decide_bad(const int * qn, long long f) { return qn && qn[f] == 0; }

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
		if (r < m.n && b < d.B && !decide_bad(d.qn, d.frame[b]))
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
	const GpsFrame * gps;      // [n_frames] or nullptr (DecideBatch::gps)
	const int * count;         // [n_frames] real places a gated frame compares
	const int * qn;            // [n_frames] or nullptr (DecideBatch::qn)
	int * key_n;               // [client] what each client's last posterior is keyed to (DecideBatch::key_n / key_ids)
	long long * key_ids;
};

// Rtabmap.cpp:2143-2233 for one frame per CTA: the highest real-place posterior (scanned in descending id order with a strict '>', so
// ties go to the highest id), its value replaced by 1 - posterior(virtual place), then the threshold / single-hypothesis / ratio checks
__global__ void decide_select_kernel(const DecideMap m, const DecideSelect a)
{
	__shared__ float s_v[32];
	__shared__ int s_r[32];
	const int f = blockIdx.x;
	const int client = static_cast<int>(a.client[f]);
	const int flags = static_cast<int>(a.flags[f]) | (decide_bad(a.qn, f) ? kDcFlagSkip : 0);
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
				const int n = a.gps && a.gps[f].mode == kGpsGated ? a.count[f] + 1 : m.n; // entries of the posterior map
				if (n <= 2 && thr > 0.f) d.status = kDcSingle;
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
	if (compute)
	{
		// the posterior decide_normalize_kernel wrote is keyed to the current map
		a.key_n[client] = m.n;
		a.key_ids[client] = static_cast<long long>(reinterpret_cast<uintptr_t>(m.ids));
	}
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

// listed[f][r] for every frame f and place r (r = 0 the virtual place, always listed by a frame that computes), and count[f] += the real
// places a gated frame compares.  Geocentric_WGS84ToENU_WGS84 (GeodeticCoords.cpp:119-149), the offset, the altitude tolerance of
// :2087-2099 and uNormSquared(...) < r2, in the reference's double statements, each operation rounded on its own (no FMA).
__global__ void decide_gps_gate_kernel(int n, const GpsPlace * __restrict__ places, const GpsFrame * __restrict__ frames, double r2,
                                       unsigned char * __restrict__ listed, int * __restrict__ count)
{
	const int r = blockIdx.x * blockDim.x + threadIdx.x, f = blockIdx.y;
	const int mode = frames[f].mode;
	bool keep = mode != kGpsNone;
	if (mode == kGpsGated && r > 0 && r < n && places[r - 1].fix)
	{
		const GpsFrame g = frames[f];
		const GpsPlace p = places[r - 1];
		const double rx = __dsub_rn(p.x, g.x), ry = __dsub_rn(p.y, g.y), rz = __dsub_rn(p.z, g.z);
		double x = __dadd_rn(__dmul_rn(-g.slon, rx), __dmul_rn(g.clon, ry));
		double y = __dadd_rn(__dsub_rn(__dmul_rn(__dmul_rn(-g.clon, g.slat), rx), __dmul_rn(__dmul_rn(g.slon, g.slat), ry)), __dmul_rn(g.clat, rz));
		double z = __dadd_rn(__dadd_rn(__dmul_rn(__dmul_rn(g.clon, g.clat), rx), __dmul_rn(__dmul_rn(g.slon, g.clat), ry)), __dmul_rn(g.slat, rz));
		x = __dadd_rn(x, static_cast<double>(p.ox)); // offsetENU.x() - originOffsetENU.x() (identity in localisation mode), a float
		y = __dadd_rn(y, static_cast<double>(p.oy));
		z = __dadd_rn(z, static_cast<double>(p.oz));
		if (z > g.error) z = __dsub_rn(z, g.error);
		else if (z < -g.error) z = __dadd_rn(z, g.error);
		else z = 0.0;
		keep = __dadd_rn(__dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y)), __dmul_rn(z, z)) < r2;
	}
	if (r < n) listed[static_cast<size_t>(f) * n + r] = keep ? 1 : 0;
	if (mode == kGpsGated)
	{
		const unsigned m = __ballot_sync(0xFFFFFFFFu, keep && r > 0 && r < n);
		if ((threadIdx.x & 31) == 0 && m) atomicAdd(&count[f], __popc(m));
	}
}

__global__ void decide_reset_clients_kernel(const int * __restrict__ clients, int n, int * __restrict__ hi_id, float * __restrict__ hi_val,
                                            int * __restrict__ key_n, long long * __restrict__ key_ids)
{
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	hi_id[clients[i]] = 0;
	hi_val[clients[i]] = 0.f;
	key_n[clients[i]] = 0;
	key_ids[clients[i]] = 0;
}

} // namespace lcd
