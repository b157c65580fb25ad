// proximity.cuh — proximity detection by space (RGBD/ProximityBySpace) for many localisation clients, one CTA per frame.
//
// Replaces, per frame, the candidate search of Rtabmap::process in localisation mode (Rtabmap.cpp:2698-2934):
//   graph::findNearestNodes over the map's optimised poses (Graph.cpp:2239-2325; the radius rule of rtflann's result sets, dist < r^2),
//   Rtabmap::getPaths (Rtabmap.cpp:5303-5382) with Memory::getNeighborsId (Memory.cpp:1703-1870) over the neighbour links,
//   the NearestPathKey of every path (:1147-1176, :2796-2816) and the walk over the paths in descending key order (:2827-2934).
// The registrations the walk attempts do not depend on each other, so they are all known when this kernel ends and are verified in one
// launch of the existing matching and PnP kernels; proximity_apply_kernel then turns the results into the links and the suppression of
// the global hypothesis (:2894-2911, :3193-3196).
#pragma once
#include "decide.cuh"

namespace lcd {

constexpr int kPxThreads = 256;
constexpr int kPxMaxCand = 1024; // places inside RGBD/LocalRadius one frame can segment; more: kPxCapacity, nothing else is done
constexpr int kPxMaxPaths = 16;  // RGBD/ProximityMaxPaths
constexpr int kPxOff = 0, kPxRan = 1, kPxCapacity = 2;       // lcd_proximity_result.status
constexpr int kPxLinkLocal = 1, kPxLinkGlobal = 2;           // Link::kLocalSpaceClosure, Link::kGlobalClosure
constexpr int kDcProximitySuppressed = 12;

struct ProxPath
{
	float likelihood; // NearestPathKey
	int id;
	float distance;
	int candidate;    // the place the registration was attempted with
};

struct ProxRecord
{
	int status, n_nearest, n_paths, n_attempts, loop_in_radius, suppressed;
	ProxPath path[kPxMaxPaths];
	int accepted[kPxMaxPaths];
	int link_type[kPxMaxPaths];
};

struct ProxArgs
{
	int n;                      // real places of the map
	const int * ids;            // [n] ascending
	const float * poses;        // [n][12] rtabmap::Transform 3x4
	const int * nbr_ptr;        // [n+1] neighbour links by row
	const int * nbr_row;        // their target rows
	const float * frame_pose;   // [n_frames][12]
	const int * enabled;        // [n_frames]
	const long long * flags;    // [n_frames] the decision's frame flags: skipped / held frames have no likelihood (all 0)
	const float * adj;          // [n_frames][n+1] adjusted likelihood of the decision, element 0 the virtual place
	const Decision * dec;       // [n_frames]
	const int * sig_slot;       // signature store row of each id (nullptr: no store)
	int slot_cap;
	float radius, angle, filter_radius;
	int max_paths, max_depth;
	int nq;                     // descriptors per frame
	const int * n_frame;        // [n_frames] descriptors of each frame (nullptr: nq each)
	const int * qn;             // [n_frames] quantised words of each frame (nullptr: none is a bad signature), decide.cuh's decide_bad
	ProxRecord * rec;           // [n_frames]
	int * pair_slot;            // [n_frames][max_paths] store row of each attempted registration, -1 = none
	int * pair_row;             // [n_frames][max_paths] its frame row
	int * pair_n_to;            // [n_frames][max_paths] the frame's descriptors to register, 0 for slots not attempted
};

// squared distance of two positions as FLANN's L2_Simple sums it: x, y, z
__device__ inline float px_d2(float ax, float ay, float az, float bx, float by, float bz)
{
	const float dx = __fsub_rn(ax, bx), dy = __fsub_rn(ay, by), dz = __fsub_rn(az, bz);
	return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
}

// (A^-1 * B).getNormSquared() with A^-1 = [R^T | -R^T t] (the reference inverts the 4x4 with Eigen; the last bits are not pinned)
__device__ inline float px_rel_norm2(const float * A, const float * B)
{
	float v[3];
	for (int i = 0; i < 3; ++i)
	{
		const float ti = __fadd_rn(__fadd_rn(__fmul_rn(A[i], A[3]), __fmul_rn(A[4 + i], A[7])), __fmul_rn(A[8 + i], A[11]));
		const float bi = B ? __fadd_rn(__fadd_rn(__fmul_rn(A[i], B[3]), __fmul_rn(A[4 + i], B[7])), __fmul_rn(A[8 + i], B[11])) : 0.f;
		v[i] = __fsub_rn(bi, ti);
	}
	return __fadd_rn(__fadd_rn(__fmul_rn(v[0], v[0]), __fmul_rn(v[1], v[1])), __fmul_rn(v[2], v[2]));
}

// pcl::getAngle3D of the two x axes (Eigen::Vector4f, w = 0: Eigen sums (x + z) + y), compared with the angle as the reference does
__device__ inline bool px_angle_ok(const float * A, const float * B, float angle)
{
	if (!(angle > 0.f)) return true;
	const float ox = A[0], oy = A[4], oz = A[8], nx = B[0], ny = B[4], nz = B[8];
	const float n1 = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(ox, ox), __fmul_rn(oz, oz)), __fmul_rn(oy, oy)));
	const float n2 = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(nx, nx), __fmul_rn(nz, nz)), __fmul_rn(ny, ny)));
	const float ax = __fdiv_rn(ox, n1), ay = __fdiv_rn(oy, n1), az = __fdiv_rn(oz, n1);
	const float bx = __fdiv_rn(nx, n2), by = __fdiv_rn(ny, n2), bz = __fdiv_rn(nz, n2);
	double rad = static_cast<double>(__fadd_rn(__fadd_rn(__fmul_rn(ax, bx), __fmul_rn(az, bz)), __fmul_rn(ay, by)));
	rad = rad < -1.0 ? -1.0 : (rad > 1.0 ? 1.0 : rad);
	return acos(rad) <= static_cast<double>(angle);
}

// NearestPathKey::operator< (Rtabmap.cpp:1154-1172)
__device__ inline bool px_key_less(float la, float da, int ia, float lb, float db, int ib)
{
	if (la < lb) return true;
	if (la == lb) return da > db || (da == db && ia < ib);
	return false;
}

// block-wide arg-min of (value, index); index -1 = none.  Every thread gets the result.
__device__ inline int px_block_argmin(float v, int i, float * s_v, int * s_i)
{
	for (int o = 16; o > 0; o >>= 1)
	{
		const float ov = __shfl_down_sync(0xFFFFFFFFu, v, o);
		const int oi = __shfl_down_sync(0xFFFFFFFFu, i, o);
		if (oi >= 0 && (i < 0 || ov < v || (ov == v && oi < i)))
		{
			v = ov;
			i = oi;
		}
	}
	const int w = threadIdx.x >> 5;
	__syncthreads();
	if ((threadIdx.x & 31) == 0)
	{
		s_v[w] = v;
		s_i[w] = i;
	}
	__syncthreads();
	if (threadIdx.x == 0)
	{
		for (int k = 1; k < kPxThreads / 32; ++k)
			if (s_i[k] >= 0 && (s_i[0] < 0 || s_v[k] < s_v[0] || (s_v[k] == s_v[0] && s_i[k] < s_i[0])))
			{
				s_v[0] = s_v[k];
				s_i[0] = s_i[k];
			}
	}
	__syncthreads();
	return s_i[0];
}

// candidate index of map row r (s_row ascending), -1 when r is not a candidate
__device__ inline int px_find(const int * s_row, int K, int r)
{
	int lo = 0, hi = K - 1;
	while (lo <= hi)
	{
		const int mid = (lo + hi) >> 1;
		if (s_row[mid] == r) return mid;
		if (s_row[mid] < r) lo = mid + 1;
		else hi = mid - 1;
	}
	return -1;
}

__global__ void __launch_bounds__(kPxThreads) proximity_paths_kernel(const ProxArgs a)
{
	__shared__ int s_row[kPxMaxCand];   // candidates: map rows in ascending id order
	__shared__ float s_d2[kPxMaxCand];  // their squared distance to the frame
	__shared__ int s_path[kPxMaxCand];  // path of each candidate (-1: not segmented yet)
	__shared__ int s_mark[kPxMaxCand];  // stamp of the last graph search that reached it
	__shared__ int s_q[kPxMaxCand];     // graph search queue, then "path walked" flags
	__shared__ float s_kl[kPxMaxCand], s_kd[kPxMaxCand];
	__shared__ int s_kid[kPxMaxCand];
	__shared__ int s_start[kPxMaxCand]; // the nearest place each path started from
	__shared__ float s_rv[32];
	__shared__ int s_ri[32], s_wc[kPxThreads / 32];
	__shared__ int s_count, s_np, s_attempts, s_done;
	const int f = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
	ProxRecord & rec = a.rec[f];
	const float * P = a.frame_pose + 12 * static_cast<size_t>(f);
	const bool enabled = a.enabled[f] && !decide_bad(a.qn, f); // a bad signature's frame is not a proximity candidate
	for (int j = tid; j < a.max_paths; j += blockDim.x)
	{
		a.pair_slot[f * a.max_paths + j] = -1;
		a.pair_row[f * a.max_paths + j] = f;
		a.pair_n_to[f * a.max_paths + j] = 0;
	}
	if (tid == 0)
	{
		rec.status = enabled ? kPxRan : kPxOff;
		rec.n_nearest = rec.n_paths = rec.n_attempts = rec.loop_in_radius = rec.suppressed = 0;
		for (int j = 0; j < kPxMaxPaths; ++j)
		{
			rec.path[j] = ProxPath{0.f, 0, 0.f, 0};
			rec.accepted[j] = rec.link_type[j] = 0;
		}
		s_count = 0;
	}
	if (!enabled) return;
	__syncthreads();
	// 1) graph::findNearestNodes(signature->id(), _optimizedPoses, radius): every place with d2 < radius^2, compacted in id order
	const float r2 = __fmul_rn(a.radius, a.radius);
	for (int base = 0; base < a.n; base += blockDim.x)
	{
		const int i = base + tid;
		float d2 = 0.f;
		bool in = false;
		if (i < a.n)
		{
			const float * Q = a.poses + 12 * static_cast<size_t>(i);
			d2 = px_d2(P[3], P[7], P[11], Q[3], Q[7], Q[11]);
			in = d2 < r2;
		}
		const unsigned bal = __ballot_sync(0xFFFFFFFFu, in);
		if (lane == 0) s_wc[warp] = __popc(bal);
		__syncthreads();
		int off = s_count;
		for (int w = 0; w < warp; ++w) off += s_wc[w];
		off += __popc(bal & ((1u << lane) - 1u));
		if (in && off < kPxMaxCand)
		{
			s_row[off] = i;
			s_d2[off] = d2;
		}
		__syncthreads();
		if (tid == 0)
			for (int w = 0; w < kPxThreads / 32; ++w) s_count += s_wc[w];
		__syncthreads();
	}
	const int K = s_count;
	const int loop_id = a.dec[f].loop_id;
	if (tid == 0)
	{
		rec.n_nearest = K;
		if (K > kPxMaxCand) rec.status = kPxCapacity;
	}
	if (K > kPxMaxCand || K == 0) return;
	for (int k = tid; k < K; k += blockDim.x)
	{
		s_path[k] = -1;
		s_mark[k] = -1;
		if (a.ids[s_row[k]] == loop_id) rec.loop_in_radius = 1;
	}
	if (tid == 0) s_np = 0;
	__syncthreads();
	const bool use_like = (a.flags[f] & (kDcFlagSkip | kDcFlagHold)) == 0;
	const float * like = a.adj + static_cast<size_t>(f) * (a.n + 1) + 1;
	// 2) Rtabmap::getPaths: the nearest place not in a path yet, Memory::getNeighborsId(nearest, maxGraphDepth) through candidates only,
	// then the reached places not in a path yet, in ascending id order, each admitted when it is the first or links to one already admitted
	int round = 0; // graph searches so far (thread 0): the stamp of s_mark
	for (;;)
	{
		float v = INFINITY;
		int best = -1;
		for (int k = tid; k < K; k += blockDim.x)
			if (s_path[k] < 0 && (best < 0 || s_d2[k] < v))
			{
				v = s_d2[k];
				best = k;
			}
		best = px_block_argmin(v, best, s_rv, s_ri);
		if (best < 0) break;
		if (tid == 0)
		{
			const int p = s_np, stamp = round++;
			int head = 0, tail = 0, level = 0, layer_end = 1;
			s_q[tail++] = best;
			s_mark[best] = stamp;
			while (head < tail)
			{
				if (head == layer_end)
				{
					++level;
					layer_end = tail;
				}
				const int k = s_q[head++];
				if (a.max_depth > 0 && level + 1 >= a.max_depth) continue; // margins 0 .. maxGraphDepth-1
				const int r = s_row[k];
				for (int e = a.nbr_ptr[r]; e < a.nbr_ptr[r + 1]; ++e)
				{
					const int j = px_find(s_row, K, a.nbr_row[e]);
					if (j >= 0 && s_mark[j] != stamp)
					{
						s_mark[j] = stamp;
						s_q[tail++] = j;
					}
				}
			}
			// ascending id order of the reached set (candidate order is id order)
			if (tail <= 64)
			{
				for (int i = 1; i < tail; ++i)
				{
					const int x = s_q[i];
					int j = i - 1;
					while (j >= 0 && s_q[j] > x)
					{
						s_q[j + 1] = s_q[j];
						--j;
					}
					s_q[j + 1] = x;
				}
			}
			else
			{
				tail = 0;
				for (int k = 0; k < K; ++k)
					if (s_mark[k] == stamp) s_q[tail++] = k;
			}
			float hl = 0.f, sd = -1.f;
			int hid = 0, size = 0;
			for (int i = 0; i < tail; ++i)
			{
				const int k = s_q[i];
				if (s_path[k] >= 0) continue;
				bool valid = size == 0;
				const int r = s_row[k];
				for (int e = a.nbr_ptr[r]; e < a.nbr_ptr[r + 1] && !valid; ++e)
				{
					const int j = px_find(s_row, K, a.nbr_row[e]);
					valid = j >= 0 && s_path[j] == p;
				}
				if (!valid) continue;
				s_path[k] = p;
				++size;
				// the path's key: highest likelihood, ties to the smaller distance, scanned in ascending id order (:2804-2814)
				const float lv = use_like ? like[r] : 0.f;
				const float dist = px_rel_norm2(P, a.poses + 12 * static_cast<size_t>(r));
				if (lv > hl || (lv == hl && (sd < 0.f || dist < sd)))
				{
					hl = lv;
					hid = a.ids[r];
					sd = dist;
				}
			}
			// paths.insert(nearestId, path) keeps the first path of a start: when the start itself was not admitted (it links only to
			// higher ids than the first admitted place), the next round starts from it again and its path is lost
			bool dup = false;
			for (int q = 0; q < p && !dup; ++q) dup = s_start[q] == best;
			if (dup)
				for (int k = 0; k < K; ++k)
					if (s_path[k] == p) s_path[k] = kPxMaxCand; // segmented, in no path
			if (!dup)
			{
				s_kl[p] = hl;
				s_kd[p] = sd;
				s_kid[p] = hid;
				s_start[p] = best;
				s_np = p + 1;
			}
		}
		__syncthreads();
	}
	const int np = s_np;
	for (int k = tid; k < np; k += blockDim.x) s_q[k] = 0;
	if (tid == 0)
	{
		rec.n_paths = np;
		s_attempts = 0;
	}
	__syncthreads();
	// 3) the paths in descending NearestPathKey order until max_paths registrations were attempted (:2827-2934)
	const float fr2 = __fmul_rn(a.filter_radius, a.filter_radius);
	for (int step = 0; step < np && s_attempts < a.max_paths; ++step)
	{
		// the largest key not walked yet: one thread per path, reduced by warp 0
		int best = -1;
		for (int p = tid; p < np; p += blockDim.x)
			if (!s_q[p] && (best < 0 || px_key_less(s_kl[best], s_kd[best], s_kid[best], s_kl[p], s_kd[p], s_kid[p]))) best = p;
		for (int o = 16; o > 0; o >>= 1)
		{
			const int ob = __shfl_down_sync(0xFFFFFFFFu, best, o);
			if (ob >= 0 && (best < 0 || px_key_less(s_kl[best], s_kd[best], s_kid[best], s_kl[ob], s_kd[ob], s_kid[ob]))) best = ob;
		}
		if (lane == 0) s_ri[warp] = best;
		__syncthreads();
		if (tid == 0)
		{
			best = s_ri[0];
			for (int w = 1; w < kPxThreads / 32; ++w)
			{
				const int ob = s_ri[w];
				if (ob >= 0 && (best < 0 || px_key_less(s_kl[best], s_kd[best], s_kid[best], s_kl[ob], s_kd[ob], s_kid[ob]))) best = ob;
			}
			s_q[best] = 1;
			s_done = best;
			s_rv[31] = 0.f;
			s_ri[31] = 0; // the key's id survived the filter
		}
		__syncthreads();
		const int p = s_done;
		// graph::findNearestPoses(signature, path + signature, radius, angle), then findNearestNode of what is left
		float v = INFINITY;
		int nb = -1;
		for (int k = tid; k < K; k += blockDim.x)
		{
			if (s_path[k] != p || !(s_d2[k] < r2)) continue;
			const float * Q = a.poses + 12 * static_cast<size_t>(s_row[k]);
			if (!px_angle_ok(P, Q, a.angle)) continue;
			if (a.ids[s_row[k]] == s_kid[p]) s_ri[31] = 1;
			if (nb < 0 || s_d2[k] < v)
			{
				v = s_d2[k];
				nb = k;
			}
		}
		__syncthreads();
		const int key_ok = s_ri[31];
		nb = px_block_argmin(v, nb, s_rv, s_ri);
		if (tid == 0)
		{
			int k = -1;
			if (s_kl[p] > 0.f && key_ok)
			{
				for (int j = 0; j < K; ++j)
					if (s_path[j] == p && a.ids[s_row[j]] == s_kid[p]) k = j;
			}
			else k = nb;
			// the nearest place must be closer than the filtering radius (RGBD/ProximityPathFilteringRadius capped by MaxLoopClosureDistance)
			if (k >= 0 && (!(a.filter_radius > 0.f) || s_d2[k] < fr2))
			{
				const int t = s_attempts;
				const int id = a.ids[s_row[k]];
				rec.path[t] = ProxPath{s_kl[p], s_kid[p], s_kd[p], id};
				a.pair_slot[f * a.max_paths + t] = (a.sig_slot && id < a.slot_cap) ? a.sig_slot[id] : -1;
				a.pair_n_to[f * a.max_paths + t] = a.n_frame ? a.n_frame[f] : a.nq;
				s_attempts = t + 1;
			}
		}
		__syncthreads();
	}
	if (tid == 0) rec.n_attempts = s_attempts;
}

// the registrations' outcome (:2866-2911) and its effect on the global hypothesis (:3193-3196), one thread per frame
__global__ void proximity_apply_kernel(int n_frames, int max_paths, float filter_radius, const int * __restrict__ ok, const float * __restrict__ T,
                                       ProxRecord * __restrict__ rec, Decision * __restrict__ dec, int * __restrict__ hyp_id,
                                       int * __restrict__ hyp_slot, unsigned char * __restrict__ skip)
{
	const int f = blockIdx.x * blockDim.x + threadIdx.x;
	if (f >= n_frames) return;
	ProxRecord & r = rec[f];
	const int loop_id = dec[f].loop_id;
	const float fr2 = __fmul_rn(filter_radius, filter_radius);
	int suppressed = 0;
	for (int j = 0; j < r.n_attempts; ++j)
	{
		const int pr = f * max_paths + j;
		const bool acc = ok[pr] && (!(filter_radius > 0.f) || px_rel_norm2(T + 12 * static_cast<size_t>(pr), nullptr) <= fr2);
		r.accepted[j] = acc ? 1 : 0;
		r.link_type[j] = acc ? kPxLinkLocal : 0;
		if (!acc || loop_id <= 0 || !r.loop_in_radius) continue;
		const int id = r.path[j].candidate;
		if (id == loop_id)
		{
			r.link_type[j] = kPxLinkGlobal;
			suppressed = id;
		}
		else if (suppressed == 0) suppressed = id;
	}
	r.suppressed = suppressed;
	skip[f] = 0;
	if (loop_id > 0 && suppressed != 0)
	{
		skip[f] = 1; // the global hypothesis is not registered again (:3134)
		hyp_slot[f] = -1;
		if (suppressed != loop_id)
		{
			dec[f].status = kDcProximitySuppressed;
			dec[f].loop_id = 0;
			hyp_id[f] = 0;
		}
	}
}

} // namespace lcd
