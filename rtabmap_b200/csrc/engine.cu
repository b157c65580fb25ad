// engine.cu — host side of the loop-closure engine and the C ABI (include/lcd_b200.h).
//
// One lcd_engine = the device-resident state of one rtabmap::VWDictionary
// (corelib/include/rtabmap/core/VWDictionary.h:46-160): the vocabulary matrix in search
// order (_dataTree + _mapIndexId), the not-indexed tail (_notIndexedWords), and the inverted
// index (VisualWord::_references of every word) as an arena of posting lists.  The host keeps
// only the bookkeeping the reference keeps in std::map's (id -> row, list extents, the words
// of each signature); all descriptor and posting data lives in HBM and every distance,
// decision and score is computed by the kernels in nn_hamming.cuh / resolve.cuh / score.cuh.
// There is deliberately no CPU fallback: every entry point fails with LCD_ERR_CUDA if the
// device is missing.
#include "../../include/lcd_b200.h"
#include "common.cuh"
#include "nn_hamming.cuh"
#include "nn_tensor.cuh"
#include "l2_path.cuh"
#include "nn_tensor_f32.cuh"
#include "resolve.cuh"
#include "score.cuh"
#include "similarity.cuh"
#include "bayes.cuh"
#include "decide.cuh"
#include "verify.cuh"
#include "epipolar.cuh"
#include "proximity.cuh"
#include "match_bf.cuh"
#include "orb.cuh"
#include "gftt.cuh"
#include "orb_octree.cuh"
#include "limit.cuh"

#include <cuda.h>
#include <dlfcn.h>
#include <nccl.h>

#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <unordered_map>
#include <unordered_set>
#include <utility>
#include <chrono>
#include <type_traits>
#include <vector>

using namespace lcd;

namespace {

thread_local std::string g_create_error;

template <typename T>
struct DevBuf
{
	T * p = nullptr;
	size_t cap = 0; // elements
	~DevBuf() { release(); }
	void release()
	{
		if (p) cudaFree(p);
		p = nullptr;
		cap = 0;
	}
	void swap(DevBuf & o)
	{
		std::swap(p, o.p);
		std::swap(cap, o.cap);
	}
	// grow to at least n elements; keep the first `keep` elements; zero the rest if asked.
	// A re-growth replaces a buffer that kernels on ANY stream of the engine (caller streams of the _dev entry points, the ORB side
	// streams) may still be reading or writing: the device is drained first, so the copy sees final data and the free is safe.
	cudaError_t reserve(size_t n, size_t keep, bool zero_new, cudaStream_t s)
	{
		if (n <= cap) return cudaSuccess;
		size_t ncap = std::max(n, cap + cap / 2 + 16);
		T * np = nullptr;
		cudaError_t err = cudaMalloc(&np, ncap * sizeof(T));
		if (err != cudaSuccess) return err;
		if (p) err = cudaDeviceSynchronize();
		if (err == cudaSuccess && zero_new) err = cudaMemsetAsync(np, 0, ncap * sizeof(T), s);
		if (err == cudaSuccess && p && keep) err = cudaMemcpyAsync(np, p, keep * sizeof(T), cudaMemcpyDeviceToDevice, s);
		if (err == cudaSuccess && p) err = cudaStreamSynchronize(s);
		if (err != cudaSuccess)
		{
			cudaFree(np);
			return err;
		}
		if (p) cudaFree(p);
		p = np;
		cap = ncap;
		return cudaSuccess;
	}
};

// Signature id -> row ("slot") of a per-signature store in HBM, on the host and as the device copy the kernels read through
// (d.p, n_ids).  Freed slots are reused first, the last freed first: the WM -> LTM transfer adds and removes one signature per
// frame, and the store must not grow.
struct SlotMap
{
	std::vector<int> h;     // by id, -1: none
	std::vector<int> freed;
	int slots = 0;          // handed out, freed ones included
	DevBuf<int> d;
	int n_ids = 0;          // ids the device copy holds

	int count() const { return slots - static_cast<int>(freed.size()); }
	// the slot of each id: the one it has, else a freed one, else a new one.  false: an id is not > 0, and nothing changed.
	bool assign(const int * ids, int n, std::vector<int> & slot)
	{
		int max_id = 0;
		for (int i = 0; i < n; ++i)
		{
			if (ids[i] <= 0) return false;
			max_id = std::max(max_id, ids[i]);
		}
		if (static_cast<size_t>(max_id) >= h.size()) h.resize(std::max<size_t>(max_id + 1, h.size() + h.size() / 2 + 1024), -1);
		slot.resize(n);
		for (int i = 0; i < n; ++i)
		{
			int & s = h[ids[i]];
			if (s < 0 && !freed.empty())
			{
				s = freed.back();
				freed.pop_back();
			}
			else if (s < 0)
				s = slots++;
			slot[i] = s;
		}
		return true;
	}
	// the slot id held, now free; -1: it held none
	int release(int id)
	{
		if (id <= 0 || id >= static_cast<int>(h.size()) || h[id] < 0) return -1;
		const int s = h[id];
		h[id] = -1;
		freed.push_back(s);
		return s;
	}
	cudaError_t upload(cudaStream_t s)
	{
		cudaError_t err = d.reserve(h.size(), 0, false, s);
		if (err == cudaSuccess) err = cudaMemcpyAsync(d.p, h.data(), h.size() * sizeof(int), cudaMemcpyHostToDevice, s);
		if (err == cudaSuccess) n_ids = static_cast<int>(h.size());
		return err;
	}
	// the entry of one id
	cudaError_t upload(int id, cudaStream_t s)
	{
		return id < n_ids ? cudaMemcpyAsync(d.p + id, &h[id], sizeof(int), cudaMemcpyHostToDevice, s) : cudaSuccess;
	}
};

// Rows i of a batch to rows slot[i] of a store: put(slot, i, k) writes k rows from row i on; one call when the slots are
// consecutive, else one per row.
template <typename Put>
cudaError_t write_rows(const std::vector<int> & slot, Put put)
{
	const size_t n = slot.size();
	size_t i = 1;
	while (i < n && slot[i] == slot[0] + static_cast<int>(i)) ++i;
	if (i == n) return put(static_cast<size_t>(slot[0]), 0, n);
	for (i = 0; i < n; ++i)
		if (cudaError_t err = put(static_cast<size_t>(slot[i]), i, 1)) return err;
	return cudaSuccess;
}

template <typename T>
struct PinBuf
{
	T * p = nullptr;
	size_t cap = 0;
	~PinBuf()
	{
		if (p) cudaFreeHost(p);
	}
	cudaError_t reserve(size_t n)
	{
		if (n <= cap) return cudaSuccess;
		if (p) cudaFreeHost(p);
		p = nullptr;
		cap = 0;
		size_t ncap = n + n / 2 + 16;
		cudaError_t err = cudaMallocHost(&p, ncap * sizeof(T));
		if (err == cudaSuccess) cap = ncap;
		return err;
	}
};

// Zero-fill on the SMs.  cudaMemsetAsync may be scheduled on a copy engine, where it queues behind the (much longer) host ->
// device upload of the NEXT batch and stalls the kernels of the current one (measured: 1.8 ms per step in the pipelined path).
__global__ void zero_fill_kernel(uint4 * __restrict__ p16, size_t n16, unsigned char * __restrict__ tail, size_t n_tail)
{
	const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
	if (i < n16) p16[i] = make_uint4(0, 0, 0, 0);
	if (i < n_tail) tail[i] = 0;
}
static cudaError_t zero_fill_async(void * p, size_t bytes, cudaStream_t s)
{
	if (!bytes) return cudaSuccess;
	if (reinterpret_cast<uintptr_t>(p) & 15) return cudaMemsetAsync(p, 0, bytes, s);
	const size_t n16 = bytes / 16, n_tail = bytes % 16;
	const size_t n = std::max(n16, n_tail);
	zero_fill_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, s>>>(static_cast<uint4 *>(p), n16, static_cast<unsigned char *>(p) + n16 * 16, n_tail);
	return cudaGetLastError();
}

size_t depth_elem_bytes(int depth_type) { return depth_type == LCD_DEPTH_U16_MM ? 2 : (depth_type == LCD_DEPTH_MASK_U8 ? 1 : 4); }

// NCCL is loaded at run time (dlopen): single-GPU users of liblcd_b200.so need no NCCL, and a host that already carries one
// (PyTorch's bundled libnccl.so.2, or the system's) shares it with the library.
struct NcclApi
{
	ncclResult_t (*GetUniqueId)(ncclUniqueId *) = nullptr;
	ncclResult_t (*CommInitRank)(ncclComm_t *, int, ncclUniqueId, int) = nullptr;
	ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
	ncclResult_t (*AllGather)(const void *, void *, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
	ncclResult_t (*ReduceScatter)(const void *, void *, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
	ncclResult_t (*Send)(const void *, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
	ncclResult_t (*Recv)(void *, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
	ncclResult_t (*GroupStart)() = nullptr;
	ncclResult_t (*GroupEnd)() = nullptr;
	const char * (*GetErrorString)(ncclResult_t) = nullptr;
	bool ok = false;
	std::string why;
};
const NcclApi & nccl_api()
{
	static NcclApi api = []() {
		NcclApi a;
		void * h = nullptr;
		for (const char * name : {"libnccl.so.2", "libnccl.so"})
		{
			h = dlopen(name, RTLD_NOW | RTLD_GLOBAL);
			if (h) break;
		}
		if (!h)
		{
			a.why = std::string("libnccl.so.2 not found: ") + (dlerror() ? dlerror() : "");
			return a;
		}
#define LCD_NCCL_SYM(field, sym)                                         \
	a.field = reinterpret_cast<decltype(a.field)>(dlsym(h, sym));       \
	if (!a.field)                                                        \
	{                                                                    \
		a.why = std::string("NCCL symbol missing: ") + sym;              \
		return a;                                                        \
	}
		LCD_NCCL_SYM(GetUniqueId, "ncclGetUniqueId")
		LCD_NCCL_SYM(CommInitRank, "ncclCommInitRank")
		LCD_NCCL_SYM(CommDestroy, "ncclCommDestroy")
		LCD_NCCL_SYM(AllGather, "ncclAllGather")
		LCD_NCCL_SYM(ReduceScatter, "ncclReduceScatter")
		LCD_NCCL_SYM(Send, "ncclSend")
		LCD_NCCL_SYM(Recv, "ncclRecv")
		LCD_NCCL_SYM(GroupStart, "ncclGroupStart")
		LCD_NCCL_SYM(GroupEnd, "ncclGroupEnd")
		LCD_NCCL_SYM(GetErrorString, "ncclGetErrorString")
#undef LCD_NCCL_SYM
		a.ok = true;
		return a;
	}();
	return api;
}

// cuTensorMapEncodeTiled through the runtime's driver entry point (the library does not link libcuda)
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *, const cuuint32_t *,
                                  const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn tensor_map_encoder()
{
	static EncodeTiledFn fn = []() -> EncodeTiledFn {
		void * p = nullptr;
		cudaDriverEntryPointQueryResult q;
		if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) return nullptr;
		return reinterpret_cast<EncodeTiledFn>(p);
	}();
	return fn;
}

// 3-D tensor map over the u8 planes [frames][h][w] of one pyramid level (frame pitch `frame_stride` bytes), box = box_w x box_h x 1,
// zero fill outside.  false: the geometry does not meet the TMA alignment rules (or the driver lacks the call): plain loads instead.
static_assert(sizeof(CUtensorMap) == sizeof(lcd::OrbTensorMap), "tensor map size");
bool make_plane_tensor_map(lcd::OrbTensorMap * out, const uint8_t * base, int w, int h, int n_frames, size_t frame_stride, int box_w, int box_h)
{
	EncodeTiledFn enc = tensor_map_encoder();
	if (!enc || (w % 16) || (frame_stride % 16) || (reinterpret_cast<uintptr_t>(base) % 16) || n_frames <= 0) return false;
	const cuuint64_t dims[3] = {static_cast<cuuint64_t>(w), static_cast<cuuint64_t>(h), static_cast<cuuint64_t>(n_frames)};
	const cuuint64_t strides[2] = {static_cast<cuuint64_t>(w), static_cast<cuuint64_t>(frame_stride)};
	const cuuint32_t box[3] = {static_cast<cuuint32_t>(box_w), static_cast<cuuint32_t>(box_h), 1u};
	const cuuint32_t estr[3] = {1u, 1u, 1u};
	return enc(reinterpret_cast<CUtensorMap *>(out), CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, const_cast<uint8_t *>(base), dims, strides, box, estr,
	           CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

int env_int(const char * name, int def)
{
	const char * v = getenv(name);
	return v && *v ? atoi(v) : def;
}

} // namespace

struct lcd_engine
{
	lcd_config cfg{};
	int nw = 0; // 32-bit words per descriptor
	mutable std::string err;
	mutable std::mutex err_mu;                // lcd_orb_* may fail on another thread than the dictionary calls
	cudaStream_t stream = nullptr;
	cudaStream_t orb_stream = nullptr;        // host-buffer lcd_orb_detect_describe: its own stream, so that it overlaps lcd_dict_update
	cudaStream_t copy_stream = nullptr;       // host -> device images of lcd_process_frames and lcd_process_frames_submit
	cudaEvent_t copy_fence = nullptr;
	cudaStream_t aux_stream[4] = {nullptr, nullptr, nullptr, nullptr}; // fork/join side streams (coarse pyramid levels of the ORB selection)
	cudaEvent_t aux_fork = nullptr, aux_blur_done = nullptr, aux_join[4] = {nullptr, nullptr, nullptr, nullptr};
	// lcd_process_frames_submit / _wait: two batches in flight
	struct Flight
	{
		DevBuf<uint8_t> img;
		DevBuf<unsigned char> depth;
		DevBuf<int> sig_ids;
		PinBuf<PackedVerifyResult> res;
		PinBuf<int> overflow;                  // candidate overflow flag of the batch
		int detector = LCD_DETECTOR_ORB;       // and the detector that set it
		cudaEvent_t uploaded = nullptr, done = nullptr;
		lcd_verify_result * user_results = nullptr;
		int n_frames = 0;
		// lcd_process_frames_decide_submit: the batch's own staging of the decision's host tables (decide_prepare), the proximity poses
		// and flags, and the downloads of its decisions and epipolar and proximity records, so that no batch waits for another's copies
		PinBuf<long long> h_tab;
		PinBuf<float> h_pose;
		PinBuf<int> h_enabled, h_ep_res;
		PinBuf<double> h_ep_F;
		PinBuf<Decision> h_dec;
		PinBuf<ProxRecord> h_px_rec;
		PinBuf<PackedVerifyResult> h_px_res;
		lcd_decision * user_dec = nullptr;
		lcd_epipolar_result * user_ep = nullptr;
		lcd_proximity_result * user_px = nullptr;
		int px_max_paths = 0;
		cudaEvent_t t_h0 = nullptr, t_h1 = nullptr, t_c0 = nullptr, t_c1 = nullptr; // LCD_DEBUG_TIMELINE
	};
	cudaEvent_t t_base = nullptr;
	Flight flights[2];
	int flight_head = 0, flights_busy = 0;
	DevBuf<PackedVerifyResult> v_packed;
	PinBuf<PackedVerifyResult> h_packed;
	PinBuf<int> h_overflow;
	std::atomic<long long> launches{0};
	int sm_count = 132;
	int smem_optin = 0;

	// --- vocabulary: rows [0,n_indexed) searchable, [n_indexed, n_indexed+n_pending) not indexed
	DevBuf<uint32_t> vocab, vocab_alt;
	DevBuf<int> row_ids, row_ids_alt;
	std::vector<int> h_row_ids;
	std::unordered_map<int, int> id2row;
	std::unordered_set<int> removed_rows; // indexed rows leaving at the next update
	int n_indexed = 0, n_pending = 0;
	bool pending_sorted = true;
	int last_word_id = 0;
	int row_offset = 0;

	// --- inverted index
	DevBuf<uint32_t> post_off;
	DevBuf<int> post_len;
	std::vector<uint32_t> h_off;
	std::vector<int> h_len, h_cap;
	DevBuf<int2> postings;
	size_t post_used = 0;
	DevBuf<int> ni;
	std::vector<int> h_ni;
	std::unordered_map<int, std::vector<std::pair<int, int>>> sig_words; // sig -> sorted (word,count)
	DevBuf<int> nvalid;      // by signature id: valid(s) of Signature::compareTo = sum of the signature's posting counts
	std::vector<int> h_nvalid; // = the sum of its sig_words counts; same size as h_ni
	long long total_refs = 0;

	// --- scratch
	DevBuf<uint32_t> d_queries;
	DevBuf<uint2> d_partial;
	DevBuf<uint4> tc_words;             // cached packed image of the vocabulary rows [0, tc_rows) for the tensor-core 2-NN (tc_pack_kernel)
	int tc_rows = 0;
	DevBuf<uint32_t> d_keys;
	DevBuf<int> d_word_ids, d_n_new, d_in_ids;
	DevBuf<int> uq_count, uq_word, uq_prefix;
	DevBuf<float> uq_idf;
	DevBuf<int> uq_mult, q_valid; // similarity likelihood: query multiplicity of each unique word, valid(q) of each frame
	DevBuf<long long> acc;
	int acc_stride = 0;
	DevBuf<int> d_sig_ids;
	DevBuf<float> d_like;
	DevBuf<int> d_i1, d_i2;
	DevBuf<float> d_f1, d_f2;
	DevBuf<RefOp> d_ops;
	DevBuf<MoveOp> d_moves;
	DevBuf<int> d_perm;
	// Bayes filter (bayes.cuh): the last posterior by place id + per-call scratch
	DevBuf<int> by_ids, by_colptr, by_row, by_level, by_entry_col, by_state_ids;
	DevBuf<float> by_like, by_last, by_u, by_scale, by_delta, by_post, by_state_post;
	DevBuf<double> by_lc, by_prior, by_sums;
	int by_n_state = 0;
	// the loop-closure decision of many localisation clients against one map (lcd_clients_* / lcd_decide_*, decide.cuh)
	struct MapVersion
	{
		DevBuf<int> ids; // ascending place ids, ids[0] = the virtual place
		int n = 0;
	};
	std::map<int, std::unique_ptr<MapVersion>> dc_versions; // the current map and every map whose ids a client's last posterior is keyed to
	int dc_map_ver = -1, dc_next_ver = 0, dc_n = 0;
	struct MapTables
	{
		DevBuf<float> u;      // [n] uniform value of every column of the prediction
		DevBuf<int> tptr;     // [n+1] listed entries by row
		DevBuf<int> tcol;     // [nt] their columns
		DevBuf<double> tval;  // [nt] P[r][c] - u_c
		// what the columns of a frame with a cut place list are computed from (lcd_decide_gps_batch_dev)
		DevBuf<float> tlv;    // [nt] LC value of each listed entry as a float
		DevBuf<int> cptr;     // [n+1] neighbour lists by column, as lcd_clients_set_map received them
		DevBuf<int> crow, clev;
		DevBuf<double> lc;    // [n_lc] Bayes/PredictionLC
		int n_lc = 0;
		float total = 0.f, eps = 0.f;
	};
	std::unique_ptr<MapTables> dc_tables; // the current map's; replaced as a whole by lcd_clients_set_map
	std::unique_ptr<DevBuf<GpsPlace>> gps_places; // the current map's GPS table (lcd_clients_set_map_gps); dropped by lcd_clients_set_map
	DevBuf<unsigned char> gps_listed;     // [n_frames][n] the places each frame of the last GPS call compared
	DevBuf<int> gps_count;                // [n_frames]
	DevBuf<float> gps_fu, gps_fscale, gps_fdelta; // [n][B] the gated frames' columns
	double dc_lc0 = 0.0;
	float dc_vpp = 0.f;
	int dc_clients = 0;
	DevBuf<int> dc_key_n;                 // [client] places of the ids its last posterior is keyed to (0 = empty state), and
	DevBuf<long long> dc_key_ids;         // [client] their device address: kept on the device, where a bad signature is found
	DevBuf<float> dc_post;                // [client][dc_stride] last posterior of every client
	size_t dc_stride = 0;
	DevBuf<int> dc_hi_id;                 // [client] last highest hypothesis
	DevBuf<float> dc_hi_val;
	PinBuf<long long> dc_h_tab;           // per-call frame tables, staged for the upload
	cudaEvent_t dc_h_ev = nullptr;        // the last upload from dc_h_tab
	DevBuf<long long> dc_tab;
	std::vector<int> dc_active;           // frames the call being launched computes a posterior for (unless they are bad signatures)
	DevBuf<float> dc_adj, dc_last_t, dc_post_t;
	DevBuf<double> dc_part_u, dc_part_s1, dc_part_p, dc_sums;
	DevBuf<Decision> dc_dec;
	int dc_last_frames = 0;               // frames of the last decision (0: none)
	bool dc_hyp_valid = false;            // d_hyp_id / d_hyp_slot hold the last decision's accepted hypotheses
	float dc_max_dist = 0.f;              // RGBD/MaxLoopClosureDistance of the last decision
	std::vector<int> dc_h_ids;            // the current map's ids (host copy)
	std::vector<FrameCam> dc_cams;        // [client] each client's camera (lcd_clients_set_cameras; set = 0: none)
	const FrameCam * dc_frame_cam = nullptr; // [frame] the last decision's snapshot of its frames' cameras in dc_tab, nullptr when none had one
	bool dc_cam_sized = false;            // a camera of that snapshot has an image size
	// proximity detection by space (lcd_clients_set_map_poses / lcd_decide_proximity_dev, proximity.cuh)
	struct MapPoses
	{
		DevBuf<float> poses;  // [n][12] optimised pose of every real place
		DevBuf<int> nbr_ptr;  // [n+1] neighbour links by row
		DevBuf<int> nbr_row;  // their target rows
	};
	std::unique_ptr<MapPoses> px_map;     // the poses of map version px_ver
	int px_ver = -1;
	DevBuf<float> px_frame_pose;
	DevBuf<int> px_enabled, px_slot, px_row, px_nto;
	DevBuf<ProxRecord> px_rec;
	DevBuf<PackedVerifyResult> px_res;
	DevBuf<unsigned char> px_skip;
	int px_last_frames = 0, px_max_paths = 0;
	bool px_valid = false;                // px_skip belongs to the last decision
	bool dc_verified = false;             // the last decision went through lcd_verify_decided_dev
	// verification scratch
	DevBuf<uint32_t> v_df, v_dt;
	DevBuf<float> v_xyz, v_uv, v_obj, v_img, v_T, v_xyz_to, v_obj_to;
	// epipolar check scratch
	DevBuf<int> ep_ids_a, ep_ids_b, ep_n, ep_res;
	DevBuf<float> ep_uv_a, ep_uv_b;
	DevBuf<double> ep_F;
	DevBuf<uint8_t> ep_status;
	DevBuf<int> ep_slot, ep_skip;
	int ep_last_frames = 0; // frames of the last lcd_decide_epipolar_dev (0: none)
	// word store of the stored places for the epipolar check: Signature::getWords() / getWordsKpts() by row
	DevBuf<int> ws_ids, ws_n;
	DevBuf<float> ws_uv;
	int ws_cap = 0;
	SlotMap ws_map;
	DevBuf<double> v_cov6;
	DevBuf<ulonglong2> bf_keys_a, bf_keys_b;
	DevBuf<unsigned long long> bf_best;
	DevBuf<long long> v_clk;
	DevBuf<int> v_nf, v_nt, v_mid, v_mfrom, v_mto, v_nm, v_fid, v_tid, v_inl, v_ninl, v_iters, v_ok, v_inl_ids;
	DevBuf<double> v_rvec, v_tvec;
	// signature store (Signature::getWordsDescriptors / getWords3 of the nodes in working memory)
	DevBuf<uint32_t> st_desc;
	DevBuf<float> st_xyz;
	DevBuf<int> st_n;
	// each row's temporary FROM dictionary of the matching kernel (verify.cuh, from_dict_build_kernel), built on first use for the
	// (nf, Vis/CorNNDR) of the call: word of each descriptor, creator of each word [slot][st_cap], and what it was built for [slot]
	DevBuf<uint16_t> st_kof, st_creator;
	DevBuf<FromDictTag> st_ftag;
	// float engines: the FROM dictionaries of host pairs [pair][cap] (stored rows use st_*) and the TO descriptors' two nearest words
	DevBuf<uint16_t> v_kof, v_creator;
	DevBuf<FromDictTag> v_ftag;
	DevBuf<ulonglong2> v_keys64;
	int st_cap = 0;
	SlotMap st_map;
	// global descriptors (SensorData::globalDescriptors(), type 1, one per signature): rows [slot][gd_dim]
	DevBuf<float> gd_rows, gd_query, gd_dot;
	int gd_dim = 0;
	SlotMap gd_map;
	DevBuf<int> d_hyp_id, d_hyp_slot;
	// ORB workspace
	DevBuf<uint8_t> o_img, o_gray, o_mask, o_blur, o_desc;
	DevBuf<unsigned char> o_depth, o_rank_ws;
	DevBuf<uint32_t> o_cand;
	DevBuf<int> o_cand_count, o_surv_n, o_level_n, o_n, o_overflow;
	DevBuf<OrbKeypoint> o_level_kp, o_kp;
	DevBuf<float> o_xyz, o_uv;
	float gauss_sigma_loaded = -1.f;
	int orb_tma_used = 0; // the last FAST launch staged its tiles through a tensor map
	int orb_path = 0;     // lcd_orb_last_path flags of the last detection
	int detector = LCD_DETECTOR_ORB; // lcd_detector_set: what orb_run detects
	lcd_gftt_params gftt{0.001, 7.0, 3, 0, 0.04};
	int oct_min_threshold = 7; // lcd_detector_set_orb_octree: FAST/MinThreshold
	// ORB-OCTREE workspace (orb_octree.cuh)
	DevBuf<OctCell> oc_cells;
	std::vector<OctCell> oc_cells_host; // what oc_cells holds (uploaded again only when the geometry changes)
	const OctCell * oc_cells_at = nullptr;
	DevBuf<uint32_t> oc_keys, oc_kk, oc_sel;
	DevBuf<int> oc_cell_n, oc_perm, oc_scratch, oc_cand, oc_expand, oc_sel_n;
	DevBuf<OctNode> oc_nodes;
	DevBuf<int4> oc_cnt;
	DevBuf<OrbKeypoint> oc_raw_kp;
	DevBuf<uint8_t> oc_raw_desc, oc_desc;
	// lcd_quantize_limit_set: the split of Memory::createSignature for every image-level call (limit.cuh); ql_gate = int(ratio * mean_words)
	lcd_quantize_limit ql{0, 0.0f, 0};
	int ql_gate = 0;
	DevBuf<uint32_t> ql_desc;          // [frame][k] the quantised rows
	DevBuf<int> ql_index, ql_n, ql_words; // [frame][k] their keypoint index, [frame] their count, [frame][k] their word ids
	DevBuf<float> g_eig;
	DevBuf<unsigned> g_max_key;
	DevBuf<unsigned long long> g_keys;
	DevBuf<int> g_count;
	DevBuf<uint32_t> g_bitmap;
	DevBuf<float> d_uv;

	// measurement hooks (lcd_profile_*)
	bool prof_on = false;
	struct Prof
	{
		std::vector<cudaEvent_t> ev; // start/stop pairs
		size_t used = 0;
	} prof[8];

	// tuning knobs (env: LCD_NN_CTAS_PER_SM, LCD_NN_TQ, LCD_NN_VARIANT, LCD_SCORE_BLOCKS)
	int nn_ctas_per_sm = 2, nn_tq = 8, nn_variant = 2, score_blocks = 32;
	bool f32 = false;    // LCD_DESC_F32: squared-L2 path (l2_path.cuh)
	DevBuf<ulonglong2> d_partial64, tf_fb_scratch;
	// float descriptors on the tensor cores (nn_tensor_f32.cuh): cached fp16 image of rows [0, tf_rows) + their norms
	DevBuf<uint4> tf_words, tf_queries, tf_words_aug, tf_queries_aug;
	DevBuf<float> tf_qn;
	DevBuf<uint32_t> tf_tau, tf_cand, tf_wmax2;  // tf_wmax2[0] = bits of the largest |w|^2 seen
	DevBuf<int> tf_cand_count, tf_fb_list, tf_flags; // tf_flags[0] = fallback count, tf_flags[1] = "a row does not fit fp16"
	int tf_rows = 0;            // rows of the vocabulary whose image is current
	bool tf_disabled = false;   // a dictionary row does not fit fp16: exact CUDA-core path from then on
	int nn_f32_tensor = 1;      // LCD_NN_F32_TENSOR=0 forces the exact CUDA-core kernel
	int nn_last_f32_tensor = 0;
	long long tf_img_builds = 0; // rows expanded so far (diagnostics: the image is built once per dictionary change)
	int nn_tensor = 1;   // 256-bit descriptors: wgmma int8 path (nn_tensor.cuh); 0 = POPC kernel (nn_hamming.cuh)
	int nn_last_tensor = 0; // which kernel the last run_knn used (bench / diagnostics)
	// mapping mode (lcd_map_*): detection of frame t+1 on the ORB stream while frame t is quantised and scored
	struct MapSlot
	{
		DevBuf<uint8_t> img, desc;
		DevBuf<unsigned char> depth;
		DevBuf<OrbKeypoint> kp;
		DevBuf<float> xyz;
		DevBuf<int> n;
		PinBuf<int> h_n, h_overflow;
		int detector = LCD_DETECTOR_ORB;       // the detector that ran (h_overflow names its limit)
		cudaEvent_t done = nullptr;
		int cap = 0;
		bool busy = false;
	};
	MapSlot map_slots[2];
	int map_head = 0, map_busy = 0;
	PinBuf<int> map_h_words, map_h_scalars;
	// word-range sharding across GPUs (lcd_shard_*): NCCL communicator + exchange buffers of the fused sharded step
	ncclComm_t comm = nullptr;
	bool comm_owned = false;
	int sh_rank = 0, sh_ranks = 1;
	cudaStream_t comm_stream = nullptr;
	cudaEvent_t sh_ev[2][8] = {};
	cudaEvent_t sh_tr[2] = {};         // LCD_SHARD_TRACE=1: first / last kernel of the step on the compute stream
	int sh_trace = 0, sh_ring_step = 0;
	bool sh_trace_armed = false;
	std::vector<cudaEvent_t> sh_ring;  // [step][half][8 stage events + 1 begin/end]
	DevBuf<uint8_t> sh_desc_all[2];
	DevBuf<int> sh_n_all, sh_words_loc, sh_words_all;
	DevBuf<uint32_t> sh_keys[2], sh_keys_mine;
	DevBuf<long long> sh_scores[2], sh_scores_loc[2];
	DevBuf<int> sh_pairs[2], sh_pairs_loc[2]; // similarity variant: [rank][frames + 1][ns] pair counts + valid(s), and the local sums
};

#define LCD_FAIL(e, code, ...)                          \
	do                                                  \
	{                                                   \
		char _b[512];                                   \
		snprintf(_b, sizeof(_b), __VA_ARGS__);          \
		{                                               \
			std::lock_guard<std::mutex> _g((e)->err_mu); \
			(e)->err = _b;                              \
		}                                               \
		return (code);                                  \
	} while (0)

#define LCD_CUDA(e, call)                                                                          \
	do                                                                                             \
	{                                                                                              \
		cudaError_t _c = (call);                                                                   \
		if (_c != cudaSuccess)                                                                     \
		{                                                                                          \
			LCD_FAIL(e, LCD_ERR_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(_c), __FILE__, __LINE__); \
		}                                                                                          \
	} while (0)

#define LCD_NCCL(e, call)                                                                                     \
	do                                                                                                        \
	{                                                                                                         \
		ncclResult_t _n = (call);                                                                             \
		if (_n != ncclSuccess) LCD_FAIL(e, LCD_ERR_CUDA, "%s failed: %s", #call, nccl_api().GetErrorString(_n)); \
	} while (0)

#define LCD_CHECK_LAUNCH(e)                 \
	do                                      \
	{                                       \
		++(e)->launches;                    \
		LCD_CUDA(e, cudaGetLastError());    \
	} while (0)

#define LCD_TRY(expr)              \
	do                             \
	{                              \
		int _r = (expr);           \
		if (_r != LCD_OK) return _r; \
	} while (0)

namespace {

int total_rows(const lcd_engine * e) { return e->n_indexed + e->n_pending; }

int set_device(lcd_engine * e)
{
	LCD_CUDA(e, cudaSetDevice(e->cfg.device));
	return LCD_OK;
}

int ensure_rows(lcd_engine * e, int rows)
{
	const size_t keep = static_cast<size_t>(total_rows(e));
	LCD_CUDA(e, e->vocab.reserve(static_cast<size_t>(rows) * e->nw, keep * e->nw, false, e->stream));
	LCD_CUDA(e, e->row_ids.reserve(static_cast<size_t>(rows), keep, false, e->stream));
	return LCD_OK;
}

int ensure_ids(lcd_engine * e, int max_id)
{
	const size_t need = static_cast<size_t>(max_id) + 1;
	if (need > e->h_len.size())
	{
		const size_t old = e->h_len.size();
		const size_t ncap = std::max(need, old + old / 2 + 1024);
		LCD_CUDA(e, e->post_off.reserve(ncap, old, true, e->stream));
		LCD_CUDA(e, e->post_len.reserve(ncap, old, true, e->stream));
		e->h_off.resize(e->post_off.cap, 0u);
		e->h_len.resize(e->post_off.cap, 0);
		e->h_cap.resize(e->post_off.cap, 0);
	}
	return LCD_OK;
}

int ensure_sigs(lcd_engine * e, int max_sig)
{
	const size_t need = static_cast<size_t>(max_sig) + 1;
	if (need > e->h_ni.size())
	{
		const size_t old = e->h_ni.size();
		const size_t ncap = std::max(need, old + old / 2 + 1024);
		LCD_CUDA(e, e->ni.reserve(ncap, old, true, e->stream));
		LCD_CUDA(e, e->nvalid.reserve(e->ni.cap, old, true, e->stream));
		e->h_ni.resize(e->ni.cap, 0);
		e->h_nvalid.resize(e->ni.cap, 0);
	}
	return LCD_OK;
}

int ensure_postings(lcd_engine * e, size_t extra)
{
	if (e->post_used + extra > 0xFFFFFFF0ull) LCD_FAIL(e, LCD_ERR_CAPACITY, "posting arena exceeds 2^32 entries");
	LCD_CUDA(e, e->postings.reserve(e->post_used + extra, e->post_used, false, e->stream));
	return LCD_OK;
}

// ---- measurement hooks ------------------------------------------------------------------
void prof_mark(lcd_engine * e, int which, cudaStream_t s)
{
	if (!e->prof_on) return;
	auto & p = e->prof[which];
	if (p.used == p.ev.size())
	{
		cudaEvent_t ev;
		if (cudaEventCreate(&ev) != cudaSuccess) return;
		p.ev.push_back(ev);
	}
	cudaEventRecord(p.ev[p.used++], s);
}

// ---- kernel launch helpers --------------------------------------------------------------
template <int NW, int TQ, int VARIANT>
int launch_knn_t(lcd_engine * e, const uint32_t * d_q, int nq_total, int n_rows, int n_chunks, int rows_per_cta,
                 uint2 * d_partial, cudaStream_t s)
{
	auto kern = knn2_hamming_kernel<NW, TQ, VARIANT>;
	const size_t smem = 16 + static_cast<size_t>(rows_per_cta) * NW * 4;
	if (smem > 48 * 1024)
	{
		LCD_CUDA(e, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
	}
	prof_mark(e, LCD_PROF_NN, s);
	kern<<<n_chunks, kNnThreads, smem, s>>>(e->vocab.p, n_rows, e->row_offset, d_q, nq_total, d_partial, rows_per_cta);
	prof_mark(e, LCD_PROF_NN, s);
	LCD_CHECK_LAUNCH(e);
	return LCD_OK;
}

template <int NW>
int launch_knn_nw(lcd_engine * e, const uint32_t * d_q, int nq_total, int n_rows, int n_chunks, int rows_per_cta,
                  uint2 * d_partial, cudaStream_t s)
{
	const int tq = e->nn_tq, var = (NW == 8) ? e->nn_variant : 0;
#define LCD_KNN_CASE(TQ_, V_) \
	if (tq == TQ_ && var == V_) return launch_knn_t<NW, TQ_, V_>(e, d_q, nq_total, n_rows, n_chunks, rows_per_cta, d_partial, s);
	LCD_KNN_CASE(4, 0)
	LCD_KNN_CASE(2, 0)
	LCD_KNN_CASE(8, 0)
	if constexpr (NW == 8)
	{
		LCD_KNN_CASE(4, 1)
		LCD_KNN_CASE(2, 1)
		LCD_KNN_CASE(8, 1)
		LCD_KNN_CASE(4, 2)
		LCD_KNN_CASE(2, 2)
		LCD_KNN_CASE(8, 2)
	}
#undef LCD_KNN_CASE
	return launch_knn_t<NW, 4, 0>(e, d_q, nq_total, n_rows, n_chunks, rows_per_cta, d_partial, s);
}

// ---- float descriptors on the tensor cores ------------------------------------------------------------------------
// rows of the vocabulary changed from `row` on (compaction, re-sorted tail): their image is stale
void tf_invalidate_from(lcd_engine * e, int row)
{
	e->tf_rows = std::min(e->tf_rows, std::max(row, 0));
	e->tc_rows = std::min(e->tc_rows, std::max(row, 0));
}

// (1) the cached word image: only rows that are new since the last search are converted.  When rows were converted, the "does not
// fit fp16" flag is read back at once (a synchronisation that only happens right after the dictionary changed): such a dictionary
// stays on the exact kernel.
template <int DIM>
int tf_prepare_words(lcd_engine * e, int n_rows, cudaStream_t s)
{
	if (e->tf_rows >= n_rows) return LCD_OK;
	const int n_tiles = (n_rows + kTfBN - 1) / kTfBN;
	const float * vocab = reinterpret_cast<const float *>(e->vocab.p);
	LCD_CUDA(e, e->tf_flags.reserve(4, 0, true, s));
	LCD_CUDA(e, e->tf_wmax2.reserve(1, 0, true, s));
	const size_t tile16 = static_cast<size_t>(kTfBN) * (DIM / 8);
	const int old_tiles = static_cast<int>(e->tf_words.cap / tile16);
	if (n_tiles > old_tiles)
	{
		const int want = std::max(n_tiles, old_tiles + old_tiles / 2 + 64);
		LCD_CUDA(e, e->tf_words.reserve(static_cast<size_t>(want) * tile16, static_cast<size_t>(e->tf_rows / kTfBN) * tile16, false, s));
		LCD_CUDA(e, e->tf_words_aug.reserve(static_cast<size_t>(want) * kTfBN * 2, static_cast<size_t>(e->tf_rows / kTfBN) * kTfBN * 2, false, s));
	}
	const int t0 = e->tf_rows / kTfBN;
	const size_t rows_todo = static_cast<size_t>(n_tiles - t0) * kTfBN, chunks = rows_todo * (DIM / 8);
	tf_expand_kernel<DIM><<<static_cast<unsigned>((chunks + 255) / 256), 256, 0, s>>>(vocab, t0 * kTfBN, n_rows, kTfBN, e->tf_words.p, e->tf_flags.p + 1, -2.0f);
	LCD_CHECK_LAUNCH(e);
	tf_aug_kernel<DIM><<<static_cast<unsigned>((rows_todo + 255) / 256), 256, 0, s>>>(vocab, t0 * kTfBN, n_rows, kTfBN, e->tf_words_aug.p, 0, e->tf_wmax2.p,
	                                                                                  e->tf_flags.p + 1);
	LCD_CHECK_LAUNCH(e);
	e->tf_img_builds += n_rows - e->tf_rows;
	e->tf_rows = n_rows;
	int bad = 0;
	LCD_CUDA(e, cudaMemcpyAsync(&bad, e->tf_flags.p + 1, sizeof(int), cudaMemcpyDeviceToHost, s));
	LCD_CUDA(e, cudaStreamSynchronize(s));
	if (bad) e->tf_disabled = true;
	return LCD_OK;
}

template <int DIM>
int tf_search(lcd_engine * e, const float * d_q, int nq, int n_rows, cudaStream_t s)
{
	using Cfg = TfCfg<DIM>;
	const int n_tiles = (n_rows + kTfBN - 1) / kTfBN, n_qtiles = (nq + kTfBM - 1) / kTfBM;
	const float * vocab = reinterpret_cast<const float *>(e->vocab.p);
	// (2) per-call query image and per-query state
	const size_t qtile16 = static_cast<size_t>(kTfBM) * (DIM / 8);
	LCD_CUDA(e, e->tf_queries.reserve(static_cast<size_t>(n_qtiles) * qtile16, 0, false, s));
	LCD_CUDA(e, e->tf_qn.reserve(nq, 0, false, s));
	LCD_CUDA(e, e->tf_tau.reserve(nq, 0, false, s));
	LCD_CUDA(e, e->tf_cand_count.reserve(nq, 0, false, s));
	LCD_CUDA(e, e->tf_cand.reserve(static_cast<size_t>(nq) * kTfCandCap, 0, false, s));
	LCD_CUDA(e, e->tf_fb_list.reserve(nq, 0, false, s));
	LCD_CUDA(e, e->d_partial64.reserve(nq, 0, false, s));
	LCD_CUDA(e, zero_fill_async(e->tf_flags.p, sizeof(int), s)); // fallback count
	{
		const size_t chunks = static_cast<size_t>(n_qtiles) * kTfBM * (DIM / 8);
		tf_expand_kernel<DIM><<<static_cast<unsigned>((chunks + 255) / 256), 256, 0, s>>>(d_q, 0, nq, kTfBM, e->tf_queries.p, nullptr, 1.0f);
		LCD_CHECK_LAUNCH(e);
		LCD_CUDA(e, e->tf_queries_aug.reserve(static_cast<size_t>(n_qtiles) * kTfBM * 2, 0, false, s));
		tf_aug_kernel<DIM><<<(n_qtiles * kTfBM + 255) / 256, 256, 0, s>>>(d_q, 0, nq, kTfBM, e->tf_queries_aug.p, 1, nullptr, nullptr);
		LCD_CHECK_LAUNCH(e);
		tf_query_init_kernel<DIM><<<(nq + 255) / 256, 256, 0, s>>>(d_q, nq, e->tf_qn.p, e->tf_cand_count.p, e->tf_tau.p);
		LCD_CHECK_LAUNCH(e);
	}
	// (3) bound-only pre-pass over the first rows, then the emitting pass over all rows
	LCD_CUDA(e, cudaFuncSetAttribute(knn2_tensor_f32_kernel<DIM>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(Cfg::smem)));
	TfArgs a{};
	a.word_img = e->tf_words.p;
	a.word_aug = e->tf_words_aug.p;
	a.query_aug = e->tf_queries_aug.p;
	a.n_rows = n_rows;
	a.query_img = e->tf_queries.p;
	a.qn = e->tf_qn.p;
	a.nq = nq;
	a.wmax2_bits = e->tf_wmax2.p;
	a.tau = e->tf_tau.p;
	a.cand = e->tf_cand.p;
	a.cand_count = e->tf_cand_count.p;
	prof_mark(e, LCD_PROF_NN, s);
	a.tile_begin = 0;
	a.tile_end = std::min(n_tiles, kTfPrepassTiles);
	a.tiles_per_split = a.tile_end;
	a.emit = 0;
	knn2_tensor_f32_kernel<DIM><<<dim3(n_qtiles, 1), kTfThreads, Cfg::smem, s>>>(a);
	LCD_CHECK_LAUNCH(e);
	// splits: a split's slice of the word image should sit in L2 while the query tiles of that split stream it (CTAs with the same
	// blockIdx.y are scheduled together), and small query batches still have to fill the machine
	const int tiles_l2 = std::max(1, static_cast<int>((24u << 20) / Cfg::b_bytes));
	int splits = std::max((n_tiles + tiles_l2 - 1) / tiles_l2, (2 * e->sm_count + n_qtiles - 1) / n_qtiles);
	splits = std::max(1, std::min(splits, n_tiles));
	const int tps = (n_tiles + splits - 1) / splits;
	splits = (n_tiles + tps - 1) / tps;
	a.tile_begin = 0;
	a.tile_end = n_tiles;
	a.tiles_per_split = tps;
	a.emit = 1;
	knn2_tensor_f32_kernel<DIM><<<dim3(n_qtiles, splits), kTfThreads, Cfg::smem, s>>>(a);
	LCD_CHECK_LAUNCH(e);
	// (4) exact re-rank of the candidates; overflowed lists are redone by an exact scan
	rerank_l2_kernel<DIM><<<(nq + 7) / 8, 256, 0, s>>>(vocab, e->row_offset, d_q, nq, e->tf_cand.p, e->tf_cand_count.p, e->d_partial64.p, e->tf_fb_list.p,
	                                                   e->tf_flags.p);
	LCD_CHECK_LAUNCH(e);
	const int fb_slots = std::max(4 * nq, 1 << 18), fb_ctas = 2 * e->sm_count;
	LCD_CUDA(e, e->tf_fb_scratch.reserve(static_cast<size_t>(fb_slots), 0, false, s));
	LCD_CUDA(e, cudaFuncSetAttribute(knn2_l2_fallback_kernel<DIM>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(fallback_smem_bytes<DIM>())));
	knn2_l2_fallback_kernel<DIM><<<fb_ctas, fallback_rows<DIM>(), fallback_smem_bytes<DIM>(), s>>>(vocab, n_rows, e->row_offset, d_q, e->tf_fb_list.p, e->tf_flags.p,
	                                                                              e->tf_fb_scratch.p, fb_slots);
	LCD_CHECK_LAUNCH(e);
	knn2_l2_fallback_merge_kernel<<<64, 256, 0, s>>>(e->tf_fb_list.p, e->tf_flags.p, e->tf_fb_scratch.p, fb_slots, fb_ctas, e->d_partial64.p);
	prof_mark(e, LCD_PROF_NN, s);
	LCD_CHECK_LAUNCH(e);
	return LCD_OK;
}

// exact 2-NN of nq_total queries over rows [0,n_rows): fills e->d_partial, returns chunk count
int run_knn(lcd_engine * e, const uint32_t * d_q, int nq_total, int n_rows, int * n_chunks_out, cudaStream_t s)
{
	if (e->row_offset + n_rows > kMaxRowsPacked) LCD_FAIL(e, LCD_ERR_CAPACITY, "more than %d indexed words", kMaxRowsPacked);
	e->nn_last_tensor = 0;
	e->nn_last_f32_tensor = 0;
	if (e->f32 && e->nn_f32_tensor && !e->tf_disabled && n_rows >= kTfMinRows && nq_total > 0 &&
	    tf_smem_bytes(e->nw) <= static_cast<size_t>(e->smem_optin))
		LCD_TRY(e->nw == 64 ? tf_prepare_words<64>(e, n_rows, s) : e->nw == 128 ? tf_prepare_words<128>(e, n_rows, s) : tf_prepare_words<256>(e, n_rows, s));
	if (e->f32 && e->nn_f32_tensor && !e->tf_disabled && n_rows >= kTfMinRows && nq_total > 0 &&
	    tf_smem_bytes(e->nw) <= static_cast<size_t>(e->smem_optin))
	{
		// float descriptors, large dictionary: distance matrix on the tensor cores as a filter + exact re-rank (nn_tensor_f32.cuh)
		const float * q = reinterpret_cast<const float *>(d_q);
		e->nn_last_f32_tensor = 1;
		*n_chunks_out = 1;
		return e->nw == 64 ? tf_search<64>(e, q, nq_total, n_rows, s) : e->nw == 128 ? tf_search<128>(e, q, nq_total, n_rows, s) : tf_search<256>(e, q, nq_total, n_rows, s);
	}
	if (e->f32)
	{
		// float descriptors: exact squared-L2 2-NN, one query per thread, rows split over blockIdx.y to fill the machine
		const int q_blocks = (nq_total + kL2Threads - 1) / kL2Threads;
		int splits = std::max(1, std::min((2 * e->sm_count + q_blocks - 1) / q_blocks, std::max(1, n_rows / (4 * kL2TileRows))));
		const int rps = std::max(1, (n_rows + splits - 1) / splits);
		splits = std::max(1, (n_rows + rps - 1) / rps);
		LCD_CUDA(e, e->d_partial64.reserve(static_cast<size_t>(splits) * nq_total, 0, false, s));
		const float * v = reinterpret_cast<const float *>(e->vocab.p);
		const float * q = reinterpret_cast<const float *>(d_q);
		prof_mark(e, LCD_PROF_NN, s);
		if (e->nw == 64) knn2_l2_kernel<64><<<dim3(q_blocks, splits), kL2Threads, 0, s>>>(v, n_rows, e->row_offset, q, nq_total, e->d_partial64.p, rps);
		else if (e->nw == 128) knn2_l2_kernel<128><<<dim3(q_blocks, splits), kL2Threads, 0, s>>>(v, n_rows, e->row_offset, q, nq_total, e->d_partial64.p, rps);
		else knn2_l2_kernel<256><<<dim3(q_blocks, splits), kL2Threads, 0, s>>>(v, n_rows, e->row_offset, q, nq_total, e->d_partial64.p, rps);
		prof_mark(e, LCD_PROF_NN, s);
		LCD_CHECK_LAUNCH(e);
		*n_chunks_out = splits;
		return LCD_OK;
	}
	if (e->nn_tensor && e->nw == 8 && n_rows > 0 && nq_total > 0 && kTcSmemBytes <= static_cast<size_t>(e->smem_optin))
	{
		// tensor-core path: the cached packed word image, then one CTA per (query tile, word split)
		const int n_wtiles = (n_rows + kTcBN - 1) / kTcBN, n_qtiles = (nq_total + kTcBM - 1) / kTcBM;
		int best_split = 1;
		long best_cost = -1;
		for (int sp = 1; sp <= std::min(n_wtiles, 16); ++sp)
		{
			const int tps = (n_wtiles + sp - 1) / sp;
			const int real_sp = (n_wtiles + tps - 1) / tps;
			if (real_sp != sp) continue;
			const long waves = (static_cast<long>(n_qtiles) * sp + e->sm_count - 1) / e->sm_count;
			// +2: prologue (barrier init, first loads) and drain, in tile times.  That fixed cost was 3 tiles of 128 queries; a tile of
			// 256 queries takes 1.65 of those (1.09 ms per launch at the bench shape where 128-query tiles took 1.32 ms, H100 80GB HBM3
			// at 700 W), so 3 / 1.65 = 1.8, rounded to 2.
			const long cost = waves * (tps + 2);
			if (best_cost < 0 || cost < best_cost)
			{
				best_cost = cost;
				best_split = sp;
			}
		}
		const int tps = (n_wtiles + best_split - 1) / best_split;
		LCD_CUDA(e, e->d_partial.reserve(static_cast<size_t>(best_split) * kTcEpiGroups * nq_total, 0, false, s));
		static const int tc_recache = env_int("LCD_TC_RECACHE", 0); // experiment: rebuild the word image on every search (as r01 did)
		if (tc_recache) e->tc_rows = 0;
		if (e->tc_rows < n_rows)
		{
			// the packed word image (operand layout + per-word popcounts) is cached with the dictionary: only tiles that gained rows since
			// the last search are written
			const int t0 = e->tc_rows / kTcBN;
			const size_t tile16 = kTcBBytes / 16;
			const int old_tiles = static_cast<int>(e->tc_words.cap / tile16);
			if (n_wtiles > old_tiles)
				LCD_CUDA(e, e->tc_words.reserve(static_cast<size_t>(std::max(n_wtiles, old_tiles + old_tiles / 2 + 16)) * tile16, static_cast<size_t>(t0) * tile16, false, s));
			const size_t todo = static_cast<size_t>(n_wtiles - t0) * tile16;
			tc_pack_kernel<<<static_cast<unsigned>((todo + 255) / 256), 256, 0, s>>>(reinterpret_cast<const uint4 *>(e->vocab.p), n_rows, t0, n_wtiles,
			                                                                      e->tc_words.p);
			LCD_CHECK_LAUNCH(e);
			e->tc_rows = n_rows;
		}
		LCD_CUDA(e, cudaFuncSetAttribute(knn2_tensor_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(kTcSmemBytes)));
		prof_mark(e, LCD_PROF_NN, s);
		// A CTA walks several (query tile, word split) items with one set of barriers and a running pipeline (LCD_NN_PERSIST=0: one CTA
		// per item, as r01).  Unsharded: one CTA per SM takes them all.  Inside the sharded step the search runs beside NCCL kernels that
		// need a few SMs now and then: a grid that holds every SM until the end starves them and then waits for them (measured at 4 ranks:
		// 1.35 -> 1.48 ms), so there a CTA takes only enough items for ~48 word tiles of 256 queries (the time ~96 tiles of 128 queries
		// took) and the grid stays several waves deep.
		static const int nn_persist = env_int("LCD_NN_PERSIST", 1);
		const int n_items = n_qtiles * best_split;
		int grid = n_items;
		if (nn_persist && e->comm)
		{
			const int per_cta = std::max(1, std::min(8, (48 + tps - 1) / std::max(tps, 1))); // items per CTA
			grid = (n_items + per_cta - 1) / per_cta;
		}
		else if (nn_persist)
			grid = std::min(n_items, e->sm_count);
		knn2_tensor_kernel<<<grid, kTcThreads, kTcSmemBytes, s>>>(e->tc_words.p, n_rows, e->row_offset, d_q, nq_total, e->d_partial.p, tps,
		                                                        static_cast<uint32_t>(-128), n_qtiles, best_split);
		prof_mark(e, LCD_PROF_NN, s);
		LCD_CHECK_LAUNCH(e);
		e->nn_last_tensor = 1;
		*n_chunks_out = best_split * kTcEpiGroups;
		return LCD_OK;
	}
	const int max_rows_smem = static_cast<int>((static_cast<size_t>(e->smem_optin) - 16 - 1024) / (e->nw * 4));
	int n_chunks = e->sm_count * e->nn_ctas_per_sm;
	n_chunks = std::min(n_chunks, std::max(1, (n_rows + 31) / 32));
	n_chunks = std::max(n_chunks, (n_rows + max_rows_smem - 1) / max_rows_smem);
	n_chunks = std::max(n_chunks, 1);
	int rows_per_cta = (n_rows + n_chunks - 1) / n_chunks;
	if (rows_per_cta < 1) rows_per_cta = 1;
	n_chunks = std::max(1, (n_rows + rows_per_cta - 1) / rows_per_cta);
	LCD_CUDA(e, e->d_partial.reserve(static_cast<size_t>(n_chunks) * nq_total, 0, false, s));
	int r;
	switch (e->nw)
	{
	case 4: r = launch_knn_nw<4>(e, d_q, nq_total, n_rows, n_chunks, rows_per_cta, e->d_partial.p, s); break;
	case 8: r = launch_knn_nw<8>(e, d_q, nq_total, n_rows, n_chunks, rows_per_cta, e->d_partial.p, s); break;
	case 16: r = launch_knn_nw<16>(e, d_q, nq_total, n_rows, n_chunks, rows_per_cta, e->d_partial.p, s); break;
	default: LCD_FAIL(e, LCD_ERR_INVALID, "unsupported descriptor size %d bytes", e->nw * 4);
	}
	*n_chunks_out = n_chunks;
	return r;
}

int launch_resolve(lcd_engine * e, const ResolveArgs & a, int n_frames, cudaStream_t s)
{
	if (e->f32)
	{
		const size_t smem32 = resolve_l2_smem_bytes(a.nq);
		// 256: resolve_rounds_l2 adds 32 staged descriptors (32 896 B) of static shared memory, so any dynamic size needs the opt-in
		if (smem32 > 48 * 1024 || e->nw == 256)
		{
			if (e->nw == 64) LCD_CUDA(e, cudaFuncSetAttribute(resolve_l2_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem32)));
			else if (e->nw == 128) LCD_CUDA(e, cudaFuncSetAttribute(resolve_l2_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem32)));
			else LCD_CUDA(e, cudaFuncSetAttribute(resolve_l2_kernel<256>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem32)));
		}
		prof_mark(e, LCD_PROF_RESOLVE, s);
		if (e->nw == 64) resolve_l2_kernel<64><<<n_frames, kL2ResolveThreads, smem32, s>>>(a, a.partial64);
		else if (e->nw == 128) resolve_l2_kernel<128><<<n_frames, kL2ResolveThreads, smem32, s>>>(a, a.partial64);
		else resolve_l2_kernel<256><<<n_frames, kL2ResolveThreads, smem32, s>>>(a, a.partial64);
		prof_mark(e, LCD_PROF_RESOLVE, s);
		LCD_CHECK_LAUNCH(e);
		return LCD_OK;
	}
	const size_t smem = resolve_smem_bytes(a.nq);
#define LCD_RES_CASE(NW_)                                                                                               \
	case NW_:                                                                                                           \
	{                                                                                                                   \
		auto kern = resolve_kernel<NW_>;                                                                                \
		if (smem > 48 * 1024)                                                                                           \
			LCD_CUDA(e, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem))); \
		prof_mark(e, LCD_PROF_RESOLVE, s);                                                                              \
		kern<<<n_frames, kResolveThreads, smem, s>>>(a);                                                                \
		prof_mark(e, LCD_PROF_RESOLVE, s);                                                                              \
		break;                                                                                                          \
	}
	switch (e->nw)
	{
		LCD_RES_CASE(4)
		LCD_RES_CASE(8)
		LCD_RES_CASE(16)
	default: LCD_FAIL(e, LCD_ERR_INVALID, "unsupported descriptor size");
	}
#undef LCD_RES_CASE
	LCD_CHECK_LAUNCH(e);
	return LCD_OK;
}

// The NNDR resolve of n_frames frames of nq descriptor rows (d_q) from the n_chunks top-2 key sets of nq_total queries each that run_knn
// left in e->d_partial / e->d_partial64.  The sharded callers point the keys at the gathered sets (shard_set_keys).
ResolveArgs resolve_args(const lcd_engine * e, const uint32_t * d_q, int nq, int nq_total, const int * d_nq_frame, int n_chunks, const int * row_ids,
                         int incremental, float nndr, int cmp_new, int last_word_id, int * word_ids_out)
{
	ResolveArgs a{};
	a.queries = d_q;
	a.nq = nq;
	a.nq_frame = d_nq_frame;
	a.nq_total = nq_total;
	a.partial = e->d_partial.p;
	a.partial64 = e->d_partial64.p;
	a.n_chunks = n_chunks;
	a.row_ids = row_ids;
	a.incremental = incremental;
	a.nndr = nndr;
	a.cmp_new = cmp_new;
	a.last_word_id = last_word_id;
	a.word_ids_out = word_ids_out;
	return a;
}

// The set-up of the likelihood of n_frames frames of a.nq words each: the unique-word arrays (with `pairs`, the similarity likelihood's
// word-pair arrays too) and the accumulator get their size, the accumulator is zeroed, and the preparation fields of `a` point at them.
int score_begin(lcd_engine * e, ResolveArgs & a, int n_frames, int n_total, int self_ref, bool pairs, cudaStream_t s)
{
	const int nq = a.nq;
	LCD_CUDA(e, e->uq_count.reserve(n_frames, 0, false, s));
	LCD_CUDA(e, e->uq_word.reserve(static_cast<size_t>(n_frames) * nq, 0, false, s));
	LCD_CUDA(e, e->uq_prefix.reserve(static_cast<size_t>(n_frames) * (nq + 1), 0, false, s));
	LCD_CUDA(e, e->uq_idf.reserve(static_cast<size_t>(n_frames) * nq, 0, false, s));
	if (pairs)
	{
		LCD_CUDA(e, e->uq_mult.reserve(static_cast<size_t>(n_frames) * nq, 0, false, s));
		LCD_CUDA(e, e->q_valid.reserve(n_frames, 0, false, s));
	}
	const int stride = static_cast<int>(e->h_ni.size());
	if (stride != e->acc_stride || e->acc.cap < static_cast<size_t>(stride) * n_frames)
	{
		LCD_CUDA(e, e->acc.reserve(static_cast<size_t>(std::max(stride, 1)) * n_frames, 0, false, e->stream));
		e->acc_stride = stride;
	}
	LCD_CUDA(e, zero_fill_async(e->acc.p, static_cast<size_t>(e->acc_stride) * n_frames * sizeof(long long), s));
	a.do_prep = 1;
	a.post_len = e->post_len.p;
	a.id_cap = static_cast<int>(e->h_len.size());
	a.n_total = static_cast<float>(n_total);
	a.self_ref = self_ref;
	a.uq_count = e->uq_count.p;
	a.uq_word = e->uq_word.p;
	a.uq_prefix = e->uq_prefix.p;
	a.uq_idf = e->uq_idf.p;
	if (pairs)
	{
		a.pairs = 1;
		a.uq_mult = e->uq_mult.p;
		a.q_valid = e->q_valid.p;
	}
	return LCD_OK;
}

// The word-id layout of the sharded step, [rank][frames_per_rank][nq], of which frames [part_f0, part_f0 + part_frames) of every rank are
// prepared
struct ShardIds
{
	int frames_per_rank, part_f0, part_frames;
};

// The preparation of n_frames frames from their word ids d_ids [n_frames][nq], one CTA per frame after score_begin: prep_from_ids_kernel,
// or with `local` (the sharded layout) prep_local_ids_kernel, which keeps only the ids with postings on this rank.
int prep_ids(lcd_engine * e, const int * d_ids, int n_frames, int nq, int n_total, int self_ref, bool pairs, cudaStream_t s, const ShardIds * local = nullptr)
{
	ResolveArgs a{};
	a.nq = nq;
	LCD_TRY(score_begin(e, a, n_frames, n_total, self_ref, pairs, s));
	int nq_pad = 32;
	while (nq_pad < nq) nq_pad <<= 1;
	const size_t smem = nq_pad * sizeof(uint32_t);
	prof_mark(e, LCD_PROF_RESOLVE, s);
	if (local) prep_local_ids_kernel<<<n_frames, kResolveThreads, smem, s>>>(d_ids, a, local->frames_per_rank, local->part_f0, local->part_frames);
	else prep_from_ids_kernel<<<n_frames, kResolveThreads, smem, s>>>(d_ids, a);
	prof_mark(e, LCD_PROF_RESOLVE, s);
	LCD_CHECK_LAUNCH(e);
	return LCD_OK;
}

int launch_score(lcd_engine * e, int n_frames, int nq, cudaStream_t s, bool pairs = false)
{
	ScoreArgs sa;
	sa.nq = nq;
	sa.uq_count = e->uq_count.p;
	sa.uq_word = e->uq_word.p;
	sa.uq_prefix = e->uq_prefix.p;
	sa.uq_idf = e->uq_idf.p;
	sa.uq_mult = e->uq_mult.p;
	sa.post_off = e->post_off.p;
	sa.postings = e->postings.p;
	sa.ni = e->ni.p;
	sa.sig_cap = static_cast<int>(e->h_ni.size());
	sa.acc = e->acc.p;
	sa.acc_stride = e->acc_stride;
	dim3 grid(e->score_blocks, n_frames);
	prof_mark(e, LCD_PROF_SCORE, s);
	if (pairs) score_kernel<true><<<grid, kScoreThreads, (nq + 1) * sizeof(int), s>>>(sa);
	else score_kernel<false><<<grid, kScoreThreads, (nq + 1) * sizeof(int), s>>>(sa);
	prof_mark(e, LCD_PROF_SCORE, s);
	LCD_CHECK_LAUNCH(e);
	return LCD_OK;
}

// The TF-IDF sums of n_frames prepared frames over the ns listed places, d_out [n_frames][ns]: the likelihood (float), or the exact
// fixed-point sums (long long) that the sharded callers add up across ranks
template <typename T>
int score_tfidf(lcd_engine * e, int n_frames, int nq, const int * d_sig_ids, int ns, T * d_out, cudaStream_t s)
{
	LCD_TRY(launch_score(e, n_frames, nq, s));
	const dim3 grid((ns + 255) / 256, n_frames);
	const int sig_cap = static_cast<int>(e->h_ni.size());
	if constexpr (std::is_same_v<T, float>) gather_likelihood_kernel<<<grid, 256, 0, s>>>(e->acc.p, e->acc_stride, sig_cap, d_sig_ids, ns, d_out);
	else gather_fixed_kernel<<<grid, 256, 0, s>>>(e->acc.p, e->acc_stride, sig_cap, d_sig_ids, ns, d_out);
	LCD_CHECK_LAUNCH(e);
	return LCD_OK;
}

// The word pairs of n_frames prepared frames over the ns listed places: their counts into d_pairs (one free row after every rows_per_seg
// frames, see gather_pairs_kernel), and this engine's valid(s) once per segment, at d_valid + segment * valid_stride
int score_pairs(lcd_engine * e, int n_frames, int nq, const int * d_sig_ids, int ns, int rows_per_seg, int * d_pairs, int * d_valid, size_t valid_stride,
                cudaStream_t s)
{
	LCD_TRY(launch_score(e, n_frames, nq, s, true));
	gather_pairs_kernel<<<dim3((ns + 255) / 256, n_frames), 256, 0, s>>>(e->acc.p, e->acc_stride, static_cast<int>(e->h_ni.size()), d_sig_ids, ns,
	                                                                  rows_per_seg, d_pairs);
	LCD_CHECK_LAUNCH(e);
	gather_valid_kernel<<<dim3((ns + 255) / 256, n_frames / rows_per_seg), 256, 0, s>>>(e->nvalid.p, static_cast<int>(e->h_nvalid.size()), d_sig_ids, ns,
	                                                                                 d_valid, valid_stride);
	LCD_CHECK_LAUNCH(e);
	return LCD_OK;
}

// make the not-indexed tail ascending in id (std::set<int> _notIndexedWords iteration order)
int sort_pending(lcd_engine * e)
{
	if (e->pending_sorted || e->n_pending < 2)
	{
		e->pending_sorted = true;
		return LCD_OK;
	}
	const int base = e->n_indexed, n = e->n_pending;
	std::vector<int> order(n);
	for (int i = 0; i < n; ++i) order[i] = base + i;
	std::stable_sort(order.begin(), order.end(), [&](int x, int y) { return e->h_row_ids[x] < e->h_row_ids[y]; });
	LCD_CUDA(e, e->d_perm.reserve(n, 0, false, e->stream));
	LCD_CUDA(e, cudaMemcpyAsync(e->d_perm.p, order.data(), n * sizeof(int), cudaMemcpyHostToDevice, e->stream));
	LCD_CUDA(e, e->vocab_alt.reserve(static_cast<size_t>(n) * e->nw, 0, false, e->stream));
	const size_t elems = static_cast<size_t>(n) * e->nw;
	gather_rows_kernel<<<static_cast<unsigned>((elems + 255) / 256), 256, 0, e->stream>>>(e->vocab.p, e->d_perm.p, n, e->nw, e->vocab_alt.p);
	LCD_CHECK_LAUNCH(e);
	LCD_CUDA(e, cudaMemcpyAsync(e->vocab.p + static_cast<size_t>(base) * e->nw, e->vocab_alt.p, elems * sizeof(uint32_t),
	                            cudaMemcpyDeviceToDevice, e->stream));
	std::vector<int> ids(n);
	for (int i = 0; i < n; ++i) ids[i] = e->h_row_ids[order[i]];
	for (int i = 0; i < n; ++i)
	{
		e->h_row_ids[base + i] = ids[i];
		e->id2row[ids[i]] = base + i;
	}
	LCD_CUDA(e, cudaMemcpyAsync(e->row_ids.p + base, ids.data(), n * sizeof(int), cudaMemcpyHostToDevice, e->stream));
	LCD_CUDA(e, cudaStreamSynchronize(e->stream));
	e->pending_sorted = true;
	tf_invalidate_from(e, base);
	return LCD_OK;
}

// VWDictionary::addWordRef for the words of one signature (host bookkeeping + device ops)
int add_refs_impl(lcd_engine * e, int sig_id, const int * word_ids, int n)
{
	if (sig_id <= 0) LCD_FAIL(e, LCD_ERR_INVALID, "signature id must be positive");
	LCD_TRY(ensure_sigs(e, sig_id));
	std::vector<int> ids;
	ids.reserve(n);
	for (int i = 0; i < n; ++i)
	{
		if (word_ids[i] > 0) ids.push_back(word_ids[i]);
	}
	std::sort(ids.begin(), ids.end());
	std::vector<RefOp> ops;
	std::vector<MoveOp> moves;
	auto & sw = e->sig_words[sig_id];
	std::vector<std::pair<int, int>> merged;
	merged.reserve(sw.size() + ids.size());
	size_t si = 0;
	size_t extra = 0;
	int added = 0; // references that reach the index (words the dictionary holds)
	for (size_t i = 0; i < ids.size();)
	{
		size_t j = i;
		while (j < ids.size() && ids[j] == ids[i]) ++j;
		const int word = ids[i], cnt = static_cast<int>(j - i);
		i = j;
		if (e->id2row.find(word) == e->id2row.end())
		{
			// reference: UWARN("Not found word %d"), VWDictionary.cpp:893
			continue;
		}
		LCD_TRY(ensure_ids(e, word));
		while (si < sw.size() && sw[si].first < word) merged.push_back(sw[si++]);
		RefOp op{word, sig_id, cnt, -1, 0};
		if (si < sw.size() && sw[si].first == word)
		{
			merged.emplace_back(word, sw[si].second + cnt);
			++si;
			op.pos = -1;
			op.newlen = e->h_len[word];
		}
		else
		{
			merged.emplace_back(word, cnt);
			if (e->h_len[word] == e->h_cap[word])
			{
				const int ncap = std::max(4, e->h_cap[word] * 2);
				MoveOp mv{word, e->h_off[word], static_cast<uint32_t>(e->post_used + extra), e->h_len[word]};
				extra += ncap;
				e->h_off[word] = mv.new_off;
				e->h_cap[word] = ncap;
				moves.push_back(mv);
			}
			op.pos = e->h_len[word];
			op.newlen = ++e->h_len[word];
		}
		e->total_refs += cnt;
		added += cnt;
		ops.push_back(op);
	}
	while (si < sw.size()) merged.push_back(sw[si++]);
	sw.swap(merged);
	e->h_ni[sig_id] += n;
	LCD_CUDA(e, cudaMemcpyAsync(e->ni.p + sig_id, &e->h_ni[sig_id], sizeof(int), cudaMemcpyHostToDevice, e->stream));
	e->h_nvalid[sig_id] += added;
	LCD_CUDA(e, cudaMemcpyAsync(e->nvalid.p + sig_id, &e->h_nvalid[sig_id], sizeof(int), cudaMemcpyHostToDevice, e->stream));
	if (extra)
	{
		LCD_TRY(ensure_postings(e, extra));
		e->post_used += extra;
	}
	if (!moves.empty())
	{
		LCD_CUDA(e, e->d_moves.reserve(moves.size(), 0, false, e->stream));
		LCD_CUDA(e, cudaMemcpyAsync(e->d_moves.p, moves.data(), moves.size() * sizeof(MoveOp), cudaMemcpyHostToDevice, e->stream));
		const int nm = static_cast<int>(moves.size());
		index_move_kernel<<<(nm * 32 + 255) / 256, 256, 0, e->stream>>>(e->d_moves.p, nm, e->post_off.p, e->postings.p);
		LCD_CHECK_LAUNCH(e);
	}
	if (!ops.empty())
	{
		LCD_CUDA(e, e->d_ops.reserve(ops.size(), 0, false, e->stream));
		LCD_CUDA(e, cudaMemcpyAsync(e->d_ops.p, ops.data(), ops.size() * sizeof(RefOp), cudaMemcpyHostToDevice, e->stream));
		const int no = static_cast<int>(ops.size());
		index_apply_kernel<<<(no + 255) / 256, 256, 0, e->stream>>>(e->d_ops.p, no, e->post_off.p, e->post_len.p, e->postings.p);
		LCD_CHECK_LAUNCH(e);
	}
	// the op vectors are pageable: make sure the copies completed before they go out of scope
	LCD_CUDA(e, cudaStreamSynchronize(e->stream));
	return LCD_OK;
}

int require_binary(lcd_engine * e, const char * what)
{
	if (e->f32) LCD_FAIL(e, LCD_ERR_INVALID, "%s works on binary descriptors only (this engine holds float descriptors)", what);
	return LCD_OK;
}

// entry points that translate local rows through e->row_ids are only valid on an unsharded engine
int require_unsharded(lcd_engine * e, const char * what)
{
	if (e->row_offset != 0)
		LCD_FAIL(e, LCD_ERR_STATE, "%s needs an unsharded engine (lcd_shard_set_row_offset(%d) is set: use the lcd_shard_* calls)", what, e->row_offset);
	return LCD_OK;
}

int check_queries(lcd_engine * e, const void * q, int nq)
{
	if (!q || nq <= 0) LCD_FAIL(e, LCD_ERR_INVALID, "Descriptors size is null!");
	if (nq > kMaxFrameQueries) LCD_FAIL(e, LCD_ERR_CAPACITY, "at most %d descriptors per frame", kMaxFrameQueries);
	return LCD_OK;
}

// n_total is N = Memory::getSignatures().size(), a count: a negative one would give NaN idf terms, which the fixed-point sum turns into 0
int check_n_total(lcd_engine * e, int n_total)
{
	if (n_total < 0) LCD_FAIL(e, LCD_ERR_INVALID, "n_total (the number of signatures, N) must be >= 0, got %d", n_total);
	return LCD_OK;
}

// The similarity likelihood (Memory::computeLikelihood with Kp/TfIdfLikelihoodUsed=false) of n_frames frames whose word pairs the
// resolve / prep kernel prepared (score_begin with pairs): word pairs, the global-descriptor dot products where the frames carry a descriptor
// (d_gdesc [n_frames][gd_dim], or nullptr), then Signature::compareTo per (frame, k) into d_like [n_frames][ns].
int launch_similarity(lcd_engine * e, int n_frames, int nq, const float * d_gdesc, const int * d_sig_ids, int ns, float * d_like, cudaStream_t s)
{
	LCD_TRY(launch_score(e, n_frames, nq, s, true));
	const bool gd = d_gdesc && e->gd_map.count() > 0;
	if (gd)
	{
		LCD_CUDA(e, e->gd_dot.reserve(static_cast<size_t>(n_frames) * ns, 0, false, s));
		GdescArgs g{d_gdesc, n_frames, e->gd_rows.p, e->gd_dim, e->gd_map.d.p, e->gd_map.n_ids, d_sig_ids, ns, e->gd_dot.p, nullptr};
		prof_mark(e, LCD_PROF_SCORE, s);
		gdesc_dot_kernel<<<dim3((ns + kGdBN - 1) / kGdBN, (n_frames + kGdBM - 1) / kGdBM), kGdThreads, 0, s>>>(g);
		prof_mark(e, LCD_PROF_SCORE, s);
		LCD_CHECK_LAUNCH(e);
	}
	SimilarityArgs f{e->acc.p, e->acc_stride, nullptr, e->nvalid.p, static_cast<int>(e->h_nvalid.size()), e->q_valid.p, gd ? e->gd_dot.p : nullptr,
	                 e->gd_map.d.p, e->gd_map.n_ids, d_sig_ids, ns, d_like};
	similarity_finalize_kernel<false><<<dim3((ns + 255) / 256, n_frames), 256, 0, s>>>(f);
	LCD_CHECK_LAUNCH(e);
	return LCD_OK;
}

// The resolve of n_frames frames (a from resolve_args) and, when d_out and ns > 0 are given, the likelihood of the listed places from the
// words it found: the TF-IDF sums (score_tfidf), or with `sim` (T = float) the similarity likelihood (launch_similarity, d_gdesc)
template <typename T>
int resolve_score(lcd_engine * e, ResolveArgs & a, int n_frames, int n_total, bool sim, const float * d_gdesc, const int * d_sig_ids, int ns, T * d_out,
                  cudaStream_t s)
{
	const bool score = d_out != nullptr && ns > 0;
	if (score) LCD_TRY(score_begin(e, a, n_frames, n_total, 1, sim, s));
	LCD_TRY(launch_resolve(e, a, n_frames, s));
	if (!score) return LCD_OK;
	if constexpr (std::is_same_v<T, float>)
	{
		if (sim) return launch_similarity(e, n_frames, a.nq, d_gdesc, d_sig_ids, ns, d_out, s);
	}
	return score_tfidf(e, n_frames, a.nq, d_sig_ids, ns, d_out, s);
}

// which branch of Memory::computeLikelihood localize_dev scores with (Kp/TfIdfLikelihoodUsed)
enum class LikelihoodKind
{
	TfIdf,
	Similarity
};

// quantise + score of n_frames independent frames on device buffers, no mutation.  kind = Similarity: d_gdesc [n_frames][gd_dim] are
// the frames' global descriptors (nullptr = none) and n_total is not used.
int localize_dev(lcd_engine * e, const uint32_t * d_q, int n_frames, int nq, int incremental, float nndr, int cmp_new,
                 const int * d_sig_ids, int ns, int n_total, int * d_word_ids_out, float * d_like_out, cudaStream_t s,
                 const int * d_nq_frame = nullptr, LikelihoodKind kind = LikelihoodKind::TfIdf, const float * d_gdesc = nullptr)
{
	if (e->n_indexed == 0 && !incremental) LCD_FAIL(e, LCD_ERR_STATE, "Dictionary mode is set to fixed but no words are in it!");
	LCD_TRY(require_unsharded(e, "localisation on one engine"));
	const int nq_total = n_frames * nq;
	int n_chunks = 0;
	LCD_TRY(run_knn(e, d_q, nq_total, e->n_indexed, &n_chunks, s));
	ResolveArgs a = resolve_args(e, d_q, nq, nq_total, d_nq_frame, n_chunks, e->row_ids.p, incremental, nndr, cmp_new, e->last_word_id, d_word_ids_out);
	return resolve_score(e, a, n_frames, n_total, kind == LikelihoodKind::Similarity, d_gdesc, d_sig_ids, ns, d_like_out, s);
}

} // namespace

// ============================================================================ C ABI ====
extern "C" {

int lcd_abi_version(void) { return 2; }
const char * lcd_build_arch(void) { return "sm_90a"; }

const char * lcd_last_error(const lcd_engine * e) { return e ? e->err.c_str() : g_create_error.c_str(); }
long long lcd_launch_count(const lcd_engine * e) { return e ? e->launches.load() : 0; }

int lcd_nn_select(lcd_engine * e, int kernel)
{
	if (!e) return LCD_ERR_INVALID;
	if (kernel != 0 && kernel != 1) LCD_FAIL(e, LCD_ERR_INVALID, "kernel must be 0 (popcount / exact L2 on the CUDA cores) or 1 (tensor)");
	if (e->f32) e->nn_f32_tensor = kernel;
	else e->nn_tensor = kernel;
	return LCD_OK;
}

int lcd_nn_f32_stats(lcd_engine * e, int nq, int * n_fallback, long long * n_candidates, long long * rows_converted)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(set_device(e));
	if (n_fallback) *n_fallback = 0;
	if (n_candidates) *n_candidates = 0;
	if (rows_converted) *rows_converted = e->tf_img_builds;
	if (!e->f32 || !e->tf_flags.p || !e->tf_cand_count.p || nq <= 0) return LCD_OK;
	LCD_CUDA(e, cudaDeviceSynchronize());
	int fb = 0;
	LCD_CUDA(e, cudaMemcpy(&fb, e->tf_flags.p, sizeof(int), cudaMemcpyDeviceToHost));
	std::vector<int> cnt(std::min<size_t>(nq, e->tf_cand_count.cap));
	LCD_CUDA(e, cudaMemcpy(cnt.data(), e->tf_cand_count.p, cnt.size() * sizeof(int), cudaMemcpyDeviceToHost));
	long long tot = 0;
	for (int c : cnt) tot += std::min(c, kTfCandCap);
	if (n_fallback) *n_fallback = fb;
	if (n_candidates) *n_candidates = tot;
	return LCD_OK;
}

int lcd_nn_last_kernel(const lcd_engine * e) { return e ? (e->f32 ? e->nn_last_f32_tensor : e->nn_last_tensor) : LCD_ERR_INVALID; }
void * lcd_stream(lcd_engine * e) { return e ? static_cast<void *>(e->stream) : nullptr; }

lcd_engine * lcd_create(const lcd_config * cfg)
{
	if (!cfg)
	{
		g_create_error = "null config";
		return nullptr;
	}
	if (cfg->desc_type != LCD_DESC_U8 && cfg->desc_type != LCD_DESC_F32)
	{
		g_create_error = "desc_type must be LCD_DESC_U8 (binary, Hamming) or LCD_DESC_F32 (float, squared L2)";
		return nullptr;
	}
	if (cfg->desc_type == LCD_DESC_U8 && cfg->desc_dim != 16 && cfg->desc_dim != 32 && cfg->desc_dim != 64)
	{
		g_create_error = "binary descriptor size must be 16, 32 or 64 bytes";
		return nullptr;
	}
	if (cfg->desc_type == LCD_DESC_F32 && cfg->desc_dim != 64 && cfg->desc_dim != 128 && cfg->desc_dim != 256)
	{
		g_create_error = "float descriptors must have 64, 128 or 256 dimensions (SURF-64, SURF-128 / SIFT, SuperPoint)";
		return nullptr;
	}
	int ndev = 0;
	cudaError_t err = cudaGetDeviceCount(&ndev);
	if (err != cudaSuccess || ndev <= cfg->device || cfg->device < 0)
	{
		g_create_error = std::string("no usable CUDA device: ") + (err != cudaSuccess ? cudaGetErrorString(err) : "device ordinal out of range");
		return nullptr;
	}
	lcd_engine * e = new lcd_engine();
	e->cfg = *cfg;
	e->f32 = cfg->desc_type == LCD_DESC_F32;
	e->nw = e->f32 ? cfg->desc_dim : cfg->desc_dim / 4; // 32-bit words per descriptor row
	if ((err = cudaSetDevice(cfg->device)) != cudaSuccess || (err = cudaStreamCreateWithFlags(&e->stream, cudaStreamNonBlocking)) != cudaSuccess ||
	    (err = cudaStreamCreateWithFlags(&e->orb_stream, cudaStreamNonBlocking)) != cudaSuccess)
	{
		g_create_error = std::string("CUDA init failed: ") + cudaGetErrorString(err);
		delete e;
		return nullptr;
	}
	cudaDeviceGetAttribute(&e->sm_count, cudaDevAttrMultiProcessorCount, cfg->device);
	cudaDeviceGetAttribute(&e->smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, cfg->device);
	e->nn_ctas_per_sm = std::max(1, env_int("LCD_NN_CTAS_PER_SM", e->nn_ctas_per_sm));
	e->nn_tq = env_int("LCD_NN_TQ", e->nn_tq);
	e->nn_variant = env_int("LCD_NN_VARIANT", e->nn_variant);
	e->nn_tensor = env_int("LCD_NN_TENSOR", e->nn_tensor);
	e->nn_f32_tensor = env_int("LCD_NN_F32_TENSOR", e->nn_f32_tensor);
	e->score_blocks = std::max(1, env_int("LCD_SCORE_BLOCKS", e->score_blocks));
	if (ensure_rows(e, std::max(cfg->max_words, 1024)) != LCD_OK || ensure_ids(e, std::max(cfg->max_words, 1024)) != LCD_OK ||
	    ensure_sigs(e, std::max(cfg->max_signatures, 1024)) != LCD_OK)
	{
		g_create_error = e->err;
		lcd_destroy(e);
		return nullptr;
	}
	return e;
}

void lcd_destroy(lcd_engine * e)
{
	if (!e) return;
	cudaSetDevice(e->cfg.device);
	if (e->stream)
	{
		cudaStreamSynchronize(e->stream);
		for (auto & ms : e->map_slots)
			if (ms.done) cudaEventDestroy(ms.done);
		if (e->comm && e->comm_owned && nccl_api().ok) nccl_api().CommDestroy(e->comm);
		if (e->comm_stream) cudaStreamDestroy(e->comm_stream);
		for (auto & half : e->sh_ev)
			for (cudaEvent_t ev : half)
				if (ev) cudaEventDestroy(ev);
		for (cudaEvent_t ev : e->sh_tr)
			if (ev) cudaEventDestroy(ev);
		for (cudaEvent_t ev : e->sh_ring)
			if (ev) cudaEventDestroy(ev);
		if (e->orb_stream)
		{
			cudaStreamSynchronize(e->orb_stream);
			cudaStreamDestroy(e->orb_stream);
		}
		if (e->copy_stream) cudaStreamDestroy(e->copy_stream);
		if (e->copy_fence) cudaEventDestroy(e->copy_fence);
		if (e->dc_h_ev) cudaEventDestroy(e->dc_h_ev);
		for (int i = 0; i < 4; ++i)
		{
			if (e->aux_stream[i]) cudaStreamDestroy(e->aux_stream[i]);
			if (e->aux_join[i]) cudaEventDestroy(e->aux_join[i]);
		}
		if (e->aux_fork) cudaEventDestroy(e->aux_fork);
		if (e->aux_blur_done) cudaEventDestroy(e->aux_blur_done);
		for (auto & f : e->flights)
		{
			if (f.uploaded) cudaEventDestroy(f.uploaded);
			if (f.done) cudaEventDestroy(f.done);
		}
		cudaStreamDestroy(e->stream);
	}
	for (auto & p : e->prof)
		for (auto ev : p.ev) cudaEventDestroy(ev);
	delete e;
}

int lcd_profile_enable(lcd_engine * e, int on)
{
	if (!e) return LCD_ERR_INVALID;
	e->prof_on = on != 0;
	return LCD_OK;
}

int lcd_profile_reset(lcd_engine * e)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(set_device(e));
	LCD_CUDA(e, cudaDeviceSynchronize());
	for (auto & p : e->prof) p.used = 0;
	return LCD_OK;
}

int lcd_profile_read(lcd_engine * e, int which, double * total_ms, long long * launches)
{
	if (!e || which < 0 || which > 7) return LCD_ERR_INVALID;
	LCD_TRY(set_device(e));
	LCD_CUDA(e, cudaDeviceSynchronize());
	auto & p = e->prof[which];
	double tot = 0.0;
	for (size_t i = 0; i + 1 < p.used; i += 2)
	{
		float ms = 0.f;
		LCD_CUDA(e, cudaEventElapsedTime(&ms, p.ev[i], p.ev[i + 1]));
		tot += ms;
	}
	if (total_ms) *total_ms = tot;
	if (launches) *launches = static_cast<long long>(p.used / 2);
	return LCD_OK;
}

int lcd_synchronize(lcd_engine * e)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(set_device(e));
	LCD_CUDA(e, cudaStreamSynchronize(e->stream));
	return LCD_OK;
}

// ---- dictionary ---------------------------------------------------------------------------
int lcd_dict_add_words(lcd_engine * e, const int * ids, const void * desc, int n)
{
	if (!e) return LCD_ERR_INVALID;
	if (n <= 0) return LCD_OK;
	if (!ids || !desc) LCD_FAIL(e, LCD_ERR_INVALID, "null ids/descriptors");
	LCD_TRY(set_device(e));
	int max_id = 0;
	for (int i = 0; i < n; ++i)
	{
		if (ids[i] <= 0) LCD_FAIL(e, LCD_ERR_INVALID, "word ids must be positive (got %d)", ids[i]);
		if (e->id2row.count(ids[i])) LCD_FAIL(e, LCD_ERR_INVALID, "word %d already in the dictionary", ids[i]);
		max_id = std::max(max_id, ids[i]);
	}
	const int base = total_rows(e);
	LCD_TRY(ensure_rows(e, base + n));
	LCD_TRY(ensure_ids(e, max_id));
	LCD_CUDA(e, cudaMemcpyAsync(e->vocab.p + static_cast<size_t>(base) * e->nw, desc, static_cast<size_t>(n) * e->nw * 4, cudaMemcpyHostToDevice, e->stream));
	LCD_CUDA(e, cudaMemcpyAsync(e->row_ids.p + base, ids, static_cast<size_t>(n) * sizeof(int), cudaMemcpyHostToDevice, e->stream));
	LCD_CUDA(e, cudaStreamSynchronize(e->stream));
	for (int i = 0; i < n; ++i)
	{
		if (!e->h_row_ids.empty() && e->n_pending + i > 0 && ids[i] < e->h_row_ids.back()) e->pending_sorted = false;
		e->h_row_ids.push_back(ids[i]);
		e->id2row[ids[i]] = base + i;
	}
	e->n_pending += n;
	// the reference does not touch _lastWordId in addWord; the caller sets it (Memory.cpp:431)
	return LCD_OK;
}

int lcd_dict_remove_words(lcd_engine * e, const int * ids, int n)
{
	if (!e) return LCD_ERR_INVALID;
	if (n <= 0) return LCD_OK;
	LCD_TRY(set_device(e));
	bool pending_hit = false;
	std::vector<int> zero_ids;
	std::unordered_set<int> nvalid_changed;
	for (int i = 0; i < n; ++i)
	{
		auto it = e->id2row.find(ids[i]);
		if (it == e->id2row.end()) continue;
		const int row = it->second;
		if (row < e->n_indexed) e->removed_rows.insert(row);
		else pending_hit = true;
		e->id2row.erase(it);
		if (ids[i] < static_cast<int>(e->h_len.size()) && e->h_len[ids[i]] > 0)
		{
			// The reference only removes unused words (VWDictionary::deleteUnusedWords, VWDictionary.cpp:1595-1607); a word that still
			// has references takes them with it here: its posting list is read back once so that the per-signature word lists and
			// the reference total stay consistent with the device (a later lcd_index_remove_sig must not count them again).
			const int len = e->h_len[ids[i]];
			std::vector<int2> post(len);
			LCD_CUDA(e, cudaMemcpyAsync(post.data(), e->postings.p + e->h_off[ids[i]], len * sizeof(int2), cudaMemcpyDeviceToHost, e->stream));
			LCD_CUDA(e, cudaStreamSynchronize(e->stream));
			for (const int2 & pc : post)
			{
				e->total_refs -= pc.y;
				auto sw = e->sig_words.find(pc.x);
				if (sw == e->sig_words.end()) continue;
				auto & v = sw->second;
				auto pos = std::lower_bound(v.begin(), v.end(), std::make_pair(ids[i], 0));
				if (pos != v.end() && pos->first == ids[i])
				{
					e->h_nvalid[pc.x] -= pos->second;
					nvalid_changed.insert(pc.x);
					v.erase(pos);
				}
			}
			e->h_len[ids[i]] = 0;
			zero_ids.push_back(ids[i]);
		}
	}
	for (int id : zero_ids)
	{
		LCD_CUDA(e, cudaMemsetAsync(e->post_len.p + id, 0, sizeof(int), e->stream));
	}
	for (int sig : nvalid_changed)
	{
		LCD_CUDA(e, cudaMemcpyAsync(e->nvalid.p + sig, &e->h_nvalid[sig], sizeof(int), cudaMemcpyHostToDevice, e->stream));
	}
	if (pending_hit)
	{
		// compact the not-indexed tail on the spot (it is small)
		const int base = e->n_indexed, np = e->n_pending;
		std::vector<int> keep;
		for (int r = base; r < base + np; ++r)
		{
			auto it = e->id2row.find(e->h_row_ids[r]);
			if (it != e->id2row.end() && it->second == r) keep.push_back(r);
		}
		const int nk = static_cast<int>(keep.size());
		if (nk)
		{
			LCD_CUDA(e, e->d_perm.reserve(nk, 0, false, e->stream));
			LCD_CUDA(e, cudaMemcpyAsync(e->d_perm.p, keep.data(), nk * sizeof(int), cudaMemcpyHostToDevice, e->stream));
			LCD_CUDA(e, e->vocab_alt.reserve(static_cast<size_t>(nk) * e->nw, 0, false, e->stream));
			const size_t elems = static_cast<size_t>(nk) * e->nw;
			gather_rows_kernel<<<static_cast<unsigned>((elems + 255) / 256), 256, 0, e->stream>>>(e->vocab.p, e->d_perm.p, nk, e->nw, e->vocab_alt.p);
			LCD_CHECK_LAUNCH(e);
			LCD_CUDA(e, cudaMemcpyAsync(e->vocab.p + static_cast<size_t>(base) * e->nw, e->vocab_alt.p, elems * 4, cudaMemcpyDeviceToDevice, e->stream));
		}
		std::vector<int> kid(nk);
		for (int i = 0; i < nk; ++i) kid[i] = e->h_row_ids[keep[i]];
		e->h_row_ids.resize(base);
		for (int i = 0; i < nk; ++i)
		{
			e->h_row_ids.push_back(kid[i]);
			e->id2row[kid[i]] = base + i;
		}
		if (nk) LCD_CUDA(e, cudaMemcpyAsync(e->row_ids.p + base, kid.data(), nk * sizeof(int), cudaMemcpyHostToDevice, e->stream));
		e->n_pending = nk;
		tf_invalidate_from(e, base);
	}
	LCD_CUDA(e, cudaStreamSynchronize(e->stream));
	return LCD_OK;
}

int lcd_dict_update(lcd_engine * e)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(set_device(e));
	LCD_TRY(sort_pending(e));
	if (!e->removed_rows.empty())
	{
		const int tot = total_rows(e);
		std::vector<int> keep;
		keep.reserve(tot);
		int kept_indexed = 0;
		for (int r = 0; r < tot; ++r)
		{
			if (r < e->n_indexed && e->removed_rows.count(r)) continue;
			keep.push_back(r);
			if (r < e->n_indexed) ++kept_indexed;
		}
		const int nk = static_cast<int>(keep.size());
		LCD_CUDA(e, e->vocab_alt.reserve(std::max<size_t>(e->vocab.cap, 1), 0, false, e->stream));
		LCD_CUDA(e, e->row_ids_alt.reserve(std::max<size_t>(e->row_ids.cap, 1), 0, false, e->stream));
		std::vector<int> kid(nk);
		for (int i = 0; i < nk; ++i) kid[i] = e->h_row_ids[keep[i]];
		if (nk)
		{
			LCD_CUDA(e, e->d_perm.reserve(nk, 0, false, e->stream));
			LCD_CUDA(e, cudaMemcpyAsync(e->d_perm.p, keep.data(), nk * sizeof(int), cudaMemcpyHostToDevice, e->stream));
			const size_t elems = static_cast<size_t>(nk) * e->nw;
			gather_rows_kernel<<<static_cast<unsigned>((elems + 255) / 256), 256, 0, e->stream>>>(e->vocab.p, e->d_perm.p, nk, e->nw, e->vocab_alt.p);
			LCD_CHECK_LAUNCH(e);
			LCD_CUDA(e, cudaMemcpyAsync(e->row_ids_alt.p, kid.data(), nk * sizeof(int), cudaMemcpyHostToDevice, e->stream));
		}
		LCD_CUDA(e, cudaStreamSynchronize(e->stream));
		e->vocab.swap(e->vocab_alt);
		e->row_ids.swap(e->row_ids_alt);
		e->h_row_ids.swap(kid);
		e->id2row.clear();
		for (int i = 0; i < nk; ++i) e->id2row[e->h_row_ids[i]] = i;
		e->n_pending = nk - kept_indexed;
		e->n_indexed = kept_indexed;
		e->removed_rows.clear();
		tf_invalidate_from(e, 0); // rows moved: the fp16 image is rebuilt at the next search
	}
	e->n_indexed += e->n_pending;
	e->n_pending = 0;
	e->pending_sorted = true;
	return LCD_OK;
}

int lcd_dict_clear(lcd_engine * e)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(set_device(e));
	LCD_CUDA(e, cudaStreamSynchronize(e->stream));
	e->h_row_ids.clear();
	e->id2row.clear();
	e->removed_rows.clear();
	e->n_indexed = e->n_pending = 0;
	e->pending_sorted = true;
	e->last_word_id = 0;
	std::fill(e->h_off.begin(), e->h_off.end(), 0u);
	std::fill(e->h_len.begin(), e->h_len.end(), 0);
	std::fill(e->h_cap.begin(), e->h_cap.end(), 0);
	std::fill(e->h_ni.begin(), e->h_ni.end(), 0);
	std::fill(e->h_nvalid.begin(), e->h_nvalid.end(), 0);
	if (e->post_len.p) LCD_CUDA(e, cudaMemsetAsync(e->post_len.p, 0, e->post_len.cap * sizeof(int), e->stream));
	if (e->post_off.p) LCD_CUDA(e, cudaMemsetAsync(e->post_off.p, 0, e->post_off.cap * sizeof(uint32_t), e->stream));
	if (e->ni.p) LCD_CUDA(e, cudaMemsetAsync(e->ni.p, 0, e->ni.cap * sizeof(int), e->stream));
	if (e->nvalid.p) LCD_CUDA(e, cudaMemsetAsync(e->nvalid.p, 0, e->nvalid.cap * sizeof(int), e->stream));
	e->post_used = 0;
	e->sig_words.clear();
	e->total_refs = 0;
	e->tf_rows = 0;
	e->tc_rows = 0;
	e->tf_disabled = false;
	if (e->tf_wmax2.p) LCD_CUDA(e, cudaMemsetAsync(e->tf_wmax2.p, 0, sizeof(uint32_t), e->stream));
	if (e->tf_flags.p) LCD_CUDA(e, cudaMemsetAsync(e->tf_flags.p, 0, 4 * sizeof(int), e->stream));
	LCD_CUDA(e, cudaStreamSynchronize(e->stream));
	return LCD_OK;
}

int lcd_dict_size(const lcd_engine * e) { return e ? static_cast<int>(e->id2row.size()) : 0; }
int lcd_dict_indexed_size(const lcd_engine * e) { return e ? e->n_indexed : 0; }
int lcd_dict_not_indexed_size(const lcd_engine * e) { return e ? e->n_pending : 0; }
int lcd_dict_last_word_id(const lcd_engine * e) { return e ? e->last_word_id : 0; }
int lcd_dict_set_last_word_id(lcd_engine * e, int id)
{
	if (!e || id < 0) return LCD_ERR_INVALID;
	e->last_word_id = id;
	return LCD_OK;
}

int lcd_dict_has_word(const lcd_engine * e, int word_id) { return e && e->id2row.count(word_id) ? 1 : 0; }

int lcd_dict_get_indexed(lcd_engine * e, int * ids, void * desc, int cap_rows)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(set_device(e));
	const int n = std::min(cap_rows, e->n_indexed);
	if (n <= 0) return 0;
	if (ids) memcpy(ids, e->h_row_ids.data(), n * sizeof(int));
	if (desc)
	{
		LCD_CUDA(e, cudaMemcpyAsync(desc, e->vocab.p, static_cast<size_t>(n) * e->nw * 4, cudaMemcpyDeviceToHost, e->stream));
		LCD_CUDA(e, cudaStreamSynchronize(e->stream));
	}
	return n;
}

int lcd_dict_knn2(lcd_engine * e, const void * queries, int nq, int * id1, float * d1, int * id2, float * d2)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(set_device(e));
	if (!queries || nq <= 0 || !id1 || !d1 || !id2 || !d2) LCD_FAIL(e, LCD_ERR_INVALID, "null argument");
	LCD_TRY(require_unsharded(e, "lcd_dict_knn2"));
	cudaStream_t s = e->stream;
	LCD_CUDA(e, e->d_queries.reserve(static_cast<size_t>(nq) * e->nw, 0, false, s));
	LCD_CUDA(e, cudaMemcpyAsync(e->d_queries.p, queries, static_cast<size_t>(nq) * e->nw * 4, cudaMemcpyHostToDevice, s));
	int n_chunks = 0;
	LCD_TRY(run_knn(e, e->d_queries.p, nq, e->n_indexed, &n_chunks, s));
	LCD_CUDA(e, e->d_i1.reserve(nq, 0, false, s));
	LCD_CUDA(e, e->d_i2.reserve(nq, 0, false, s));
	LCD_CUDA(e, e->d_f1.reserve(nq, 0, false, s));
	LCD_CUDA(e, e->d_f2.reserve(nq, 0, false, s));
	if (e->f32)
	{
		knn2_l2_decode_kernel<<<(nq + 255) / 256, 256, 0, s>>>(e->d_partial64.p, n_chunks, nq, e->row_ids.p, e->d_i1.p, e->d_f1.p, e->d_i2.p, e->d_f2.p);
		LCD_CHECK_LAUNCH(e);
	}
	else
	{
		LCD_CUDA(e, e->d_keys.reserve(2 * static_cast<size_t>(nq), 0, false, s));
		knn2_merge_kernel<<<(nq + 255) / 256, 256, 0, s>>>(e->d_partial.p, n_chunks, nq, e->d_keys.p);
		LCD_CHECK_LAUNCH(e);
		knn2_decode_kernel<<<(nq + 255) / 256, 256, 0, s>>>(e->d_keys.p, nq, e->row_ids.p, e->d_i1.p, e->d_f1.p, e->d_i2.p, e->d_f2.p);
		LCD_CHECK_LAUNCH(e);
	}
	LCD_CUDA(e, cudaMemcpyAsync(id1, e->d_i1.p, nq * sizeof(int), cudaMemcpyDeviceToHost, s));
	LCD_CUDA(e, cudaMemcpyAsync(id2, e->d_i2.p, nq * sizeof(int), cudaMemcpyDeviceToHost, s));
	LCD_CUDA(e, cudaMemcpyAsync(d1, e->d_f1.p, nq * sizeof(float), cudaMemcpyDeviceToHost, s));
	LCD_CUDA(e, cudaMemcpyAsync(d2, e->d_f2.p, nq * sizeof(float), cudaMemcpyDeviceToHost, s));
	LCD_CUDA(e, cudaStreamSynchronize(s));
	return LCD_OK;
}

} // extern "C"

// VWDictionary::addNewWords on descriptors that are already on the device: d_q holds `rows` descriptor rows of which the first
// n_valid (host value, or the device counter d_n_valid when n_valid < 0) are real.  Word ids of all rows -> word_ids_out (host),
// *n_new_out = words created, *n_valid_out = the device counter's value.
static int quantize_dev(lcd_engine * e, const uint32_t * d_q, int rows, int n_valid, const int * d_n_valid, int sig_id, int incremental, float nndr,
                        int cmp_new, int * word_ids_out, int * n_new_out, int * n_valid_out, cudaStream_t s)
{
	if (!incremental && e->id2row.empty()) LCD_FAIL(e, LCD_ERR_STATE, "Dictionary mode is set to fixed but no words are in it!");
	LCD_TRY(require_unsharded(e, "lcd_dict_quantize"));
	const int rows0 = total_rows(e);
	LCD_TRY(ensure_rows(e, rows0 + rows));
	int n_chunks = 0;
	LCD_TRY(run_knn(e, d_q, rows, e->n_indexed, &n_chunks, s));
	LCD_CUDA(e, e->d_word_ids.reserve(rows, 0, false, s));
	LCD_CUDA(e, e->d_n_new.reserve(1, 0, false, s));
	ResolveArgs a = resolve_args(e, d_q, rows, rows, n_valid < 0 ? d_n_valid : nullptr, n_chunks, e->row_ids.p, incremental, nndr, cmp_new, e->last_word_id,
	                             e->d_word_ids.p);
	a.n_new_out = e->d_n_new.p;
	a.pending_desc = e->vocab.p + static_cast<size_t>(rows0) * e->nw;
	a.pending_ids = e->row_ids.p + rows0;
	LCD_TRY(launch_resolve(e, a, 1, s));
	int n_new = 0, nv = n_valid;
	LCD_CUDA(e, cudaMemcpyAsync(word_ids_out, e->d_word_ids.p, rows * sizeof(int), cudaMemcpyDeviceToHost, s));
	LCD_CUDA(e, cudaMemcpyAsync(&n_new, e->d_n_new.p, sizeof(int), cudaMemcpyDeviceToHost, s));
	if (n_valid < 0) LCD_CUDA(e, cudaMemcpyAsync(&nv, d_n_valid, sizeof(int), cudaMemcpyDeviceToHost, s));
	LCD_CUDA(e, cudaStreamSynchronize(s));
	if (n_new > 0)
	{
		LCD_TRY(ensure_ids(e, e->last_word_id + n_new));
		for (int k = 0; k < n_new; ++k)
		{
			const int id = e->last_word_id + 1 + k;
			e->h_row_ids.push_back(id);
			e->id2row[id] = rows0 + k;
		}
		e->n_pending += n_new;
		e->last_word_id += n_new;
	}
	if (n_new_out) *n_new_out = n_new;
	if (n_valid_out) *n_valid_out = nv;
	if (sig_id > 0) LCD_TRY(add_refs_impl(e, sig_id, word_ids_out, std::min(std::max(nv, 0), rows)));
	return LCD_OK;
}

extern "C" {

int lcd_dict_quantize(lcd_engine * e, const void * queries, int nq, int sig_id, int incremental, float nndr,
                      int new_words_compared_together, int * word_ids_out, int * n_new_out)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(set_device(e));
	LCD_TRY(check_queries(e, queries, nq));
	if (!word_ids_out) LCD_FAIL(e, LCD_ERR_INVALID, "null output");
	cudaStream_t s = e->stream;
	LCD_CUDA(e, e->d_queries.reserve(static_cast<size_t>(nq) * e->nw, 0, false, s));
	LCD_CUDA(e, cudaMemcpyAsync(e->d_queries.p, queries, static_cast<size_t>(nq) * e->nw * 4, cudaMemcpyHostToDevice, s));
	return quantize_dev(e, e->d_queries.p, nq, nq, nullptr, sig_id, incremental, nndr, new_words_compared_together, word_ids_out, n_new_out, nullptr, s);
}

int lcd_dict_find_nn(lcd_engine * e, const void * queries, int nq, int incremental, float nndr, int * word_ids_out)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(set_device(e));
	LCD_TRY(check_queries(e, queries, nq));
	if (!word_ids_out) LCD_FAIL(e, LCD_ERR_INVALID, "null output");
	if (e->id2row.empty())
	{
		memset(word_ids_out, 0, nq * sizeof(int));
		return LCD_OK;
	}
	LCD_TRY(require_unsharded(e, "lcd_dict_find_nn"));
	LCD_TRY(sort_pending(e));
	cudaStream_t s = e->stream;
	LCD_CUDA(e, e->d_queries.reserve(static_cast<size_t>(nq) * e->nw, 0, false, s));
	LCD_CUDA(e, cudaMemcpyAsync(e->d_queries.p, queries, static_cast<size_t>(nq) * e->nw * 4, cudaMemcpyHostToDevice, s));
	int n_chunks = 0;
	// index rows first, then the not-indexed tail: (dist,row) order = index hits before
	// not-indexed hits at equal distance, as the multimap insertion order (VWDictionary.cpp:1476-1517)
	LCD_TRY(run_knn(e, e->d_queries.p, nq, total_rows(e), &n_chunks, s));
	LCD_CUDA(e, e->d_word_ids.reserve(nq, 0, false, s));
	LCD_CUDA(e, e->d_n_new.reserve(1, 0, false, s));
	ResolveArgs a = resolve_args(e, e->d_queries.p, nq, nq, nullptr, n_chunks, e->row_ids.p, incremental, nndr, 0, e->last_word_id, e->d_word_ids.p);
	a.find_only = 1;
	a.n_new_out = e->d_n_new.p;
	LCD_TRY(launch_resolve(e, a, 1, s));
	LCD_CUDA(e, cudaMemcpyAsync(word_ids_out, e->d_word_ids.p, nq * sizeof(int), cudaMemcpyDeviceToHost, s));
	LCD_CUDA(e, cudaStreamSynchronize(s));
	return LCD_OK;
}

// ---- inverted index ---------------------------------------------------------------------
int lcd_index_add_refs(lcd_engine * e, int sig_id, const int * word_ids, int n)
{
	if (!e) return LCD_ERR_INVALID;
	if (n < 0 || (n > 0 && !word_ids)) LCD_FAIL(e, LCD_ERR_INVALID, "bad word list");
	LCD_TRY(set_device(e));
	return add_refs_impl(e, sig_id, word_ids, n);
}

int lcd_index_remove_sig(lcd_engine * e, int sig_id)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(set_device(e));
	auto it = e->sig_words.find(sig_id);
	if (it == e->sig_words.end()) return LCD_OK;
	std::vector<RefOp> ops;
	for (auto & wc : it->second)
	{
		const int word = wc.first;
		if (e->id2row.find(word) == e->id2row.end() || e->h_len[word] == 0) continue;
		ops.push_back(RefOp{word, sig_id, wc.second, -1, 0});
		--e->h_len[word];
		e->total_refs -= wc.second;
	}
	e->sig_words.erase(it);
	if (sig_id < static_cast<int>(e->h_ni.size()))
	{
		e->h_ni[sig_id] = 0;
		LCD_CUDA(e, cudaMemsetAsync(e->ni.p + sig_id, 0, sizeof(int), e->stream));
		e->h_nvalid[sig_id] = 0;
		LCD_CUDA(e, cudaMemsetAsync(e->nvalid.p + sig_id, 0, sizeof(int), e->stream));
	}
	if (!ops.empty())
	{
		const int no = static_cast<int>(ops.size());
		LCD_CUDA(e, e->d_ops.reserve(no, 0, false, e->stream));
		LCD_CUDA(e, cudaMemcpyAsync(e->d_ops.p, ops.data(), no * sizeof(RefOp), cudaMemcpyHostToDevice, e->stream));
		index_remove_kernel<<<(no * 32 + 255) / 256, 256, 0, e->stream>>>(e->d_ops.p, no, e->post_off.p, e->post_len.p, e->postings.p);
		LCD_CHECK_LAUNCH(e);
	}
	LCD_CUDA(e, cudaStreamSynchronize(e->stream));
	return LCD_OK;
}

int lcd_index_set_ni(lcd_engine * e, const int * sig_ids, const int * ni, int n)
{
	if (!e) return LCD_ERR_INVALID;
	if (n <= 0) return LCD_OK;
	LCD_TRY(set_device(e));
	int mx = 0;
	for (int i = 0; i < n; ++i)
	{
		if (sig_ids[i] <= 0) LCD_FAIL(e, LCD_ERR_INVALID, "signature id must be positive");
		mx = std::max(mx, sig_ids[i]);
	}
	LCD_TRY(ensure_sigs(e, mx));
	for (int i = 0; i < n; ++i) e->h_ni[sig_ids[i]] = ni[i];
	LCD_CUDA(e, cudaMemcpyAsync(e->ni.p, e->h_ni.data(), (static_cast<size_t>(mx) + 1) * sizeof(int), cudaMemcpyHostToDevice, e->stream));
	LCD_CUDA(e, cudaStreamSynchronize(e->stream));
	return LCD_OK;
}

int lcd_index_load_csr(lcd_engine * e, const int * word_ids, int nw, const int64_t * row_ptr, const int * sig, const int * cnt)
{
	if (!e) return LCD_ERR_INVALID;
	if (nw <= 0) return LCD_OK;
	if (!word_ids || !row_ptr || !sig || !cnt) LCD_FAIL(e, LCD_ERR_INVALID, "null argument");
	LCD_TRY(set_device(e));
	const int64_t total = row_ptr[nw] - row_ptr[0];
	int max_word = 0, max_sig = 0;
	// the whole input is validated before any state changes
	if (total < 0) LCD_FAIL(e, LCD_ERR_INVALID, "row_ptr must be non-decreasing");
	for (int k = 0; k < nw; ++k)
	{
		if (e->id2row.find(word_ids[k]) == e->id2row.end()) LCD_FAIL(e, LCD_ERR_INVALID, "word %d is not in the dictionary", word_ids[k]);
		if (row_ptr[k + 1] < row_ptr[k]) LCD_FAIL(e, LCD_ERR_INVALID, "row_ptr must be non-decreasing");
		if (word_ids[k] < static_cast<int>(e->h_len.size()) && e->h_len[word_ids[k]] != 0)
			LCD_FAIL(e, LCD_ERR_STATE, "word %d already has references; bulk load needs empty lists", word_ids[k]);
		max_word = std::max(max_word, word_ids[k]);
	}
	{
		std::unordered_set<int> seen;
		for (int k = 0; k < nw; ++k)
			if (!seen.insert(word_ids[k]).second) LCD_FAIL(e, LCD_ERR_INVALID, "word %d appears twice in the table", word_ids[k]);
	}
	for (int64_t p = row_ptr[0]; p < row_ptr[nw]; ++p)
	{
		if (sig[p] <= 0 || cnt[p] <= 0) LCD_FAIL(e, LCD_ERR_INVALID, "postings need positive signature ids and counts");
		max_sig = std::max(max_sig, sig[p]);
	}
	LCD_TRY(ensure_ids(e, max_word));
	LCD_TRY(ensure_sigs(e, max_sig));
	LCD_TRY(ensure_postings(e, static_cast<size_t>(total)));
	std::vector<int2> buf(static_cast<size_t>(total));
	size_t w = 0;
	for (int k = 0; k < nw; ++k)
	{
		const int word = word_ids[k];
		const int len = static_cast<int>(row_ptr[k + 1] - row_ptr[k]);
		e->h_off[word] = static_cast<uint32_t>(e->post_used + w);
		e->h_len[word] = len;
		e->h_cap[word] = len;
		for (int64_t p = row_ptr[k]; p < row_ptr[k + 1]; ++p)
		{
			buf[w++] = make_int2(sig[p], cnt[p]);
			e->sig_words[sig[p]].emplace_back(word, cnt[p]);
			e->h_ni[sig[p]] += cnt[p];
			e->h_nvalid[sig[p]] += cnt[p];
			e->total_refs += cnt[p];
		}
	}
	// keep the per-signature word lists sorted by word id (add_refs_impl merges against them)
	for (auto & kv : e->sig_words) std::sort(kv.second.begin(), kv.second.end());
	LCD_CUDA(e, cudaMemcpyAsync(e->postings.p + e->post_used, buf.data(), buf.size() * sizeof(int2), cudaMemcpyHostToDevice, e->stream));
	e->post_used += static_cast<size_t>(total);
	LCD_CUDA(e, cudaMemcpyAsync(e->post_off.p, e->h_off.data(), (static_cast<size_t>(max_word) + 1) * sizeof(uint32_t), cudaMemcpyHostToDevice, e->stream));
	LCD_CUDA(e, cudaMemcpyAsync(e->post_len.p, e->h_len.data(), (static_cast<size_t>(max_word) + 1) * sizeof(int), cudaMemcpyHostToDevice, e->stream));
	LCD_CUDA(e, cudaMemcpyAsync(e->ni.p, e->h_ni.data(), (static_cast<size_t>(max_sig) + 1) * sizeof(int), cudaMemcpyHostToDevice, e->stream));
	LCD_CUDA(e, cudaMemcpyAsync(e->nvalid.p, e->h_nvalid.data(), (static_cast<size_t>(max_sig) + 1) * sizeof(int), cudaMemcpyHostToDevice, e->stream));
	LCD_CUDA(e, cudaStreamSynchronize(e->stream));
	return LCD_OK;
}

int lcd_index_word_nw(lcd_engine * e, int word_id)
{
	if (!e) return LCD_ERR_INVALID;
	if (word_id <= 0 || word_id >= static_cast<int>(e->h_len.size()) || !e->id2row.count(word_id)) return 0;
	return e->h_len[word_id];
}

long long lcd_index_total_refs(const lcd_engine * e) { return e ? e->total_refs : 0; }

int lcd_index_get_refs(lcd_engine * e, int word_id, int * sig, int * cnt, int cap)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(set_device(e));
	if (word_id <= 0 || word_id >= static_cast<int>(e->h_len.size()) || !e->id2row.count(word_id)) return 0;
	const int len = e->h_len[word_id];
	if (len == 0) return 0;
	std::vector<int2> buf(len);
	LCD_CUDA(e, cudaMemcpyAsync(buf.data(), e->postings.p + e->h_off[word_id], len * sizeof(int2), cudaMemcpyDeviceToHost, e->stream));
	LCD_CUDA(e, cudaStreamSynchronize(e->stream));
	std::sort(buf.begin(), buf.end(), [](const int2 & x, const int2 & y) { return x.x < y.x; });
	for (int i = 0; i < len && i < cap; ++i)
	{
		if (sig) sig[i] = buf[i].x;
		if (cnt) cnt[i] = buf[i].y;
	}
	return len;
}

int lcd_index_score(lcd_engine * e, const int * query_word_ids, int nq, const int * sig_ids, int ns, int n_total, float * likelihood_out)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(set_device(e));
	if (!query_word_ids || nq <= 0) LCD_FAIL(e, LCD_ERR_INVALID, "The signature is null");
	if (!sig_ids || ns <= 0 || !likelihood_out) LCD_FAIL(e, LCD_ERR_INVALID, "ids list is empty");
	LCD_TRY(check_n_total(e, n_total));
	if (nq > kMaxFrameQueries) LCD_FAIL(e, LCD_ERR_CAPACITY, "at most %d words per signature", kMaxFrameQueries);
	cudaStream_t s = e->stream;
	LCD_CUDA(e, e->d_in_ids.reserve(nq, 0, false, s));
	LCD_CUDA(e, e->d_sig_ids.reserve(ns, 0, false, s));
	LCD_CUDA(e, e->d_like.reserve(ns, 0, false, s));
	LCD_CUDA(e, cudaMemcpyAsync(e->d_in_ids.p, query_word_ids, nq * sizeof(int), cudaMemcpyHostToDevice, s));
	LCD_CUDA(e, cudaMemcpyAsync(e->d_sig_ids.p, sig_ids, ns * sizeof(int), cudaMemcpyHostToDevice, s));
	LCD_TRY(prep_ids(e, e->d_in_ids.p, 1, nq, n_total, 0, false, s));
	LCD_TRY(score_tfidf(e, 1, nq, e->d_sig_ids.p, ns, e->d_like.p, s));
	LCD_CUDA(e, cudaMemcpyAsync(likelihood_out, e->d_like.p, ns * sizeof(float), cudaMemcpyDeviceToHost, s));
	LCD_CUDA(e, cudaStreamSynchronize(s));
	return LCD_OK;
}

int lcd_adjust_likelihood_dev(lcd_engine * e, const float * d_likelihood, int n_frames, int ns, int virtual_place_ratio, float * d_adjusted_out,
                              void * stream)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(set_device(e));
	if (!d_likelihood || !d_adjusted_out || n_frames <= 0 || ns <= 0) LCD_FAIL(e, LCD_ERR_INVALID, "likelihood is empty");
	cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : e->stream;
	adjust_likelihood_kernel<<<n_frames, kAdjustThreads, 0, s>>>(d_likelihood, ns, virtual_place_ratio, d_adjusted_out);
	LCD_CHECK_LAUNCH(e);
	return LCD_OK;
}

int lcd_adjust_likelihood(lcd_engine * e, const float * likelihood, int n_frames, int ns, int virtual_place_ratio, float * adjusted_out)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(set_device(e));
	if (!likelihood || !adjusted_out || n_frames <= 0 || ns <= 0) LCD_FAIL(e, LCD_ERR_INVALID, "likelihood is empty");
	cudaStream_t s = e->stream;
	const size_t n_in = static_cast<size_t>(n_frames) * ns, n_out = static_cast<size_t>(n_frames) * (ns + 1);
	LCD_CUDA(e, e->d_f1.reserve(n_in, 0, false, s));
	LCD_CUDA(e, e->d_f2.reserve(n_out, 0, false, s));
	LCD_CUDA(e, cudaMemcpyAsync(e->d_f1.p, likelihood, n_in * sizeof(float), cudaMemcpyHostToDevice, s));
	LCD_TRY(lcd_adjust_likelihood_dev(e, e->d_f1.p, n_frames, ns, virtual_place_ratio, e->d_f2.p, s));
	LCD_CUDA(e, cudaMemcpyAsync(adjusted_out, e->d_f2.p, n_out * sizeof(float), cudaMemcpyDeviceToHost, s));
	LCD_CUDA(e, cudaStreamSynchronize(s));
	return LCD_OK;
}

// ---- Bayes filter over the loop-closure hypotheses ----------------------------------------------------
int lcd_bayes_reset(lcd_engine * e)
{
	if (!e) return LCD_ERR_INVALID;
	e->by_n_state = 0;
	return LCD_OK;
}

// The checks lcd_bayes_compute_posterior and lcd_clients_set_map share, and what they derive: cp = col_ptr as int, ecol = the column of every
// listed entry, total / eps = _totalPredictionLCValues / _predictionEpsilon.
static int check_bayes_tables(lcd_engine * e, const int * ids, int n, const int64_t * col_ptr, const int * nbr_row, const int * nbr_level,
                              const double * prediction_lc, int n_lc, float virtual_place_prior, std::vector<int> & cp, std::vector<int> & ecol,
                              float & total, double & eps)
{
	if (!prediction_lc || n_lc < 2) LCD_FAIL(e, LCD_ERR_INVALID, "Prediction is not valid!");
	if (!col_ptr) LCD_FAIL(e, LCD_ERR_INVALID, "null neighbour table");
	if (!(virtual_place_prior >= 0.f && virtual_place_prior <= 1.f)) LCD_FAIL(e, LCD_ERR_INVALID, "Bayes/VirtualPlacePriorThr must be in [0, 1]");
	for (int i = 1; i < n; ++i)
		if (ids[i] <= ids[i - 1] || ids[i] <= 0) LCD_FAIL(e, LCD_ERR_INVALID, "ids must ascend and only ids[0] may be the (negative) virtual place");
	if (ids[0] == 0) LCD_FAIL(e, LCD_ERR_INVALID, "id 0 is invalid");
	const int64_t nnz = col_ptr[n];
	if (col_ptr[0] != 0 || nnz < 0 || nnz > 0x7FFFFFFF) LCD_FAIL(e, LCD_ERR_INVALID, "bad neighbour table");
	cp.assign(n + 1, 0);
	ecol.assign(static_cast<size_t>(nnz), 0);
	for (int c = 0; c < n; ++c)
	{
		if (col_ptr[c + 1] < col_ptr[c]) LCD_FAIL(e, LCD_ERR_INVALID, "col_ptr must be non-decreasing");
		cp[c] = static_cast<int>(col_ptr[c]);
		bool diag = ids[c] < 0;
		for (int64_t k = col_ptr[c]; k < col_ptr[c + 1]; ++k)
		{
			if (nbr_row[k] < 0 || nbr_row[k] >= n || nbr_level[k] < 0 || nbr_level[k] + 1 >= n_lc)
				LCD_FAIL(e, LCD_ERR_INVALID, "neighbour %lld of column %d is out of range", static_cast<long long>(k - col_ptr[c]), c);
			if (k > col_ptr[c] && nbr_row[k] <= nbr_row[k - 1]) LCD_FAIL(e, LCD_ERR_INVALID, "neighbours of a column must ascend");
			diag = diag || nbr_row[k] == c;
			ecol[static_cast<size_t>(k)] = c;
		}
		// generatePrediction: "No 0 margin neighbor for signature" is fatal in the reference (BayesFilter.cpp:371-374)
		if (!diag) LCD_FAIL(e, LCD_ERR_INVALID, "column %d (place %d) does not list the place itself", c, ids[c]);
	}
	cp[n] = static_cast<int>(nnz);
	// _totalPredictionLCValues / _predictionEpsilon as setPredictionLC computes them (float sum of the doubles, smallest value)
	eps = prediction_lc[0];
	for (int j = 0; j < n_lc; ++j)
	{
		if (prediction_lc[j] < 0.0 || prediction_lc[j] > 1.0) LCD_FAIL(e, LCD_ERR_INVALID, "The prediction is not valid (values must be between >0 && <=1)");
		if (prediction_lc[j] < eps) eps = prediction_lc[j];
	}
	total = 0.f;
	for (int j = 0; j < n_lc; ++j) total = static_cast<float>(static_cast<double>(total) + prediction_lc[j]); // float += double
	return LCD_OK;
}

int lcd_bayes_compute_posterior(lcd_engine * e, const int * ids, const float * likelihood, int n, const int64_t * col_ptr, const int * nbr_row,
                                const int * nbr_level, const double * prediction_lc, int n_lc, float virtual_place_prior, float * posterior_out)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(set_device(e));
	if (!ids || !likelihood || n <= 0 || !posterior_out) LCD_FAIL(e, LCD_ERR_INVALID, "likelihood is empty!");
	std::vector<int> cp, ecol;
	float total = 0.f;
	double eps = 0.0;
	LCD_TRY(check_bayes_tables(e, ids, n, col_ptr, nbr_row, nbr_level, prediction_lc, n_lc, virtual_place_prior, cp, ecol, total, eps));
	const int64_t nnz = col_ptr[n];
	cudaStream_t s = e->stream;
	const size_t nz = static_cast<size_t>(std::max<int64_t>(nnz, 1));
	LCD_CUDA(e, e->by_ids.reserve(n, 0, false, s));
	LCD_CUDA(e, e->by_like.reserve(n, 0, false, s));
	LCD_CUDA(e, e->by_colptr.reserve(n + 1, 0, false, s));
	LCD_CUDA(e, e->by_row.reserve(nz, 0, false, s));
	LCD_CUDA(e, e->by_level.reserve(nz, 0, false, s));
	LCD_CUDA(e, e->by_entry_col.reserve(nz, 0, false, s));
	LCD_CUDA(e, e->by_lc.reserve(n_lc, 0, false, s));
	LCD_CUDA(e, e->by_last.reserve(n, 0, false, s));
	LCD_CUDA(e, e->by_u.reserve(n, 0, false, s));
	LCD_CUDA(e, e->by_scale.reserve(n, 0, false, s));
	LCD_CUDA(e, e->by_delta.reserve(n, 0, false, s));
	LCD_CUDA(e, e->by_post.reserve(n, 0, false, s));
	LCD_CUDA(e, e->by_prior.reserve(n, 0, false, s));
	LCD_CUDA(e, e->by_sums.reserve(4, 0, false, s));
	// the previous state is read while the new one is written: double-buffer by size (state arrays hold max(n, n_state) entries twice)
	const size_t st_need = static_cast<size_t>(std::max(n, e->by_n_state)) * 2;
	LCD_CUDA(e, e->by_state_ids.reserve(st_need, static_cast<size_t>(e->by_n_state), false, s));
	LCD_CUDA(e, e->by_state_post.reserve(st_need, static_cast<size_t>(e->by_n_state), false, s));
	LCD_CUDA(e, cudaMemcpyAsync(e->by_ids.p, ids, n * sizeof(int), cudaMemcpyHostToDevice, s));
	LCD_CUDA(e, cudaMemcpyAsync(e->by_like.p, likelihood, n * sizeof(float), cudaMemcpyHostToDevice, s));
	LCD_CUDA(e, cudaMemcpyAsync(e->by_colptr.p, cp.data(), (n + 1) * sizeof(int), cudaMemcpyHostToDevice, s));
	if (nnz)
	{
		LCD_CUDA(e, cudaMemcpyAsync(e->by_row.p, nbr_row, nnz * sizeof(int), cudaMemcpyHostToDevice, s));
		LCD_CUDA(e, cudaMemcpyAsync(e->by_level.p, nbr_level, nnz * sizeof(int), cudaMemcpyHostToDevice, s));
		LCD_CUDA(e, cudaMemcpyAsync(e->by_entry_col.p, ecol.data(), nnz * sizeof(int), cudaMemcpyHostToDevice, s));
	}
	LCD_CUDA(e, cudaMemcpyAsync(e->by_lc.p, prediction_lc, n_lc * sizeof(double), cudaMemcpyHostToDevice, s));
	BayesArgs a{};
	a.n = n;
	a.vp_used = ids[0] < 0 ? 1 : 0;
	a.ids = e->by_ids.p;
	a.like = e->by_like.p;
	a.col_ptr = e->by_colptr.p;
	a.nbr_row = e->by_row.p;
	a.nbr_level = e->by_level.p;
	a.lc = e->by_lc.p;
	a.n_lc = n_lc;
	a.total = total;
	a.eps = static_cast<float>(eps);
	a.vpp = virtual_place_prior;
	// the state lives in the first half of the state arrays, the new one is written to the second half and copied down
	a.prev_ids = e->by_state_ids.p;
	a.prev_post = e->by_state_post.p;
	a.n_prev = e->by_n_state;
	a.last = e->by_last.p;
	a.col_u = e->by_u.p;
	a.col_scale = e->by_scale.p;
	a.col_delta = e->by_delta.p;
	a.prior = e->by_prior.p;
	a.sums = e->by_sums.p;
	a.post = e->by_post.p;
	const int nb = (n + 255) / 256;
	bayes_last_kernel<<<nb, 256, 0, s>>>(a);
	LCD_CHECK_LAUNCH(e);
	bayes_columns_kernel<<<nb, 256, 0, s>>>(a);
	LCD_CHECK_LAUNCH(e);
	if (nnz)
	{
		bayes_scatter_kernel<<<static_cast<unsigned>((nnz + 255) / 256), 256, 0, s>>>(a, static_cast<int>(nnz), e->by_entry_col.p);
		LCD_CHECK_LAUNCH(e);
	}
	bayes_update_kernel<<<nb, 256, 0, s>>>(a);
	LCD_CHECK_LAUNCH(e);
	int * st_i = e->by_state_ids.p + std::max(n, e->by_n_state);
	float * st_p = e->by_state_post.p + std::max(n, e->by_n_state);
	bayes_normalize_kernel<<<nb, 256, 0, s>>>(a, st_i, st_p);
	LCD_CHECK_LAUNCH(e);
	LCD_CUDA(e, cudaMemcpyAsync(e->by_state_ids.p, st_i, n * sizeof(int), cudaMemcpyDeviceToDevice, s));
	LCD_CUDA(e, cudaMemcpyAsync(e->by_state_post.p, st_p, n * sizeof(float), cudaMemcpyDeviceToDevice, s));
	LCD_CUDA(e, cudaMemcpyAsync(posterior_out, e->by_post.p, n * sizeof(float), cudaMemcpyDeviceToHost, s));
	LCD_CUDA(e, cudaStreamSynchronize(s));
	e->by_n_state = n;
	return LCD_OK;
}

// ---- batched localisation ------------------------------------------------------------------
int lcd_localize_batch_dev(lcd_engine * e, const void * d_queries, int n_frames, int nq_per_frame, int incremental, float nndr,
                           int new_words_compared_together, const int * d_sig_ids, int ns, int n_total,
                           int * d_word_ids_out, float * d_likelihood_out, void * stream)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(set_device(e));
	if (!d_queries || n_frames <= 0) LCD_FAIL(e, LCD_ERR_INVALID, "Descriptors size is null!");
	if (nq_per_frame <= 0 || nq_per_frame > kMaxFrameQueries) LCD_FAIL(e, LCD_ERR_CAPACITY, "1..%d descriptors per frame", kMaxFrameQueries);
	LCD_TRY(check_n_total(e, n_total));
	cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : e->stream;
	return localize_dev(e, static_cast<const uint32_t *>(d_queries), n_frames, nq_per_frame, incremental, nndr, new_words_compared_together,
	                    d_sig_ids, ns, n_total, d_word_ids_out, d_likelihood_out, s);
}

int lcd_localize_batch(lcd_engine * e, const void * queries, int n_frames, int nq_per_frame, int incremental, float nndr,
                       int new_words_compared_together, const int * sig_ids, int ns, int n_total,
                       int * word_ids_out, float * likelihood_out)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(set_device(e));
	if (!queries || n_frames <= 0) LCD_FAIL(e, LCD_ERR_INVALID, "Descriptors size is null!");
	if (nq_per_frame <= 0 || nq_per_frame > kMaxFrameQueries) LCD_FAIL(e, LCD_ERR_CAPACITY, "1..%d descriptors per frame", kMaxFrameQueries);
	if (likelihood_out && (!sig_ids || ns <= 0)) LCD_FAIL(e, LCD_ERR_INVALID, "ids list is empty");
	LCD_TRY(check_n_total(e, n_total));
	cudaStream_t s = e->stream;
	const size_t nq_total = static_cast<size_t>(n_frames) * nq_per_frame;
	LCD_CUDA(e, e->d_queries.reserve(nq_total * e->nw, 0, false, s));
	LCD_CUDA(e, cudaMemcpyAsync(e->d_queries.p, queries, nq_total * e->nw * 4, cudaMemcpyHostToDevice, s));
	if (word_ids_out) LCD_CUDA(e, e->d_word_ids.reserve(nq_total, 0, false, s));
	if (likelihood_out)
	{
		LCD_CUDA(e, e->d_sig_ids.reserve(ns, 0, false, s));
		LCD_CUDA(e, e->d_like.reserve(static_cast<size_t>(n_frames) * ns, 0, false, s));
		LCD_CUDA(e, cudaMemcpyAsync(e->d_sig_ids.p, sig_ids, ns * sizeof(int), cudaMemcpyHostToDevice, s));
	}
	LCD_TRY(localize_dev(e, e->d_queries.p, n_frames, nq_per_frame, incremental, nndr, new_words_compared_together,
	                     e->d_sig_ids.p, likelihood_out ? ns : 0, n_total, word_ids_out ? e->d_word_ids.p : nullptr,
	                     likelihood_out ? e->d_like.p : nullptr, s));
	if (word_ids_out) LCD_CUDA(e, cudaMemcpyAsync(word_ids_out, e->d_word_ids.p, nq_total * sizeof(int), cudaMemcpyDeviceToHost, s));
	if (likelihood_out)
		LCD_CUDA(e, cudaMemcpyAsync(likelihood_out, e->d_like.p, static_cast<size_t>(n_frames) * ns * sizeof(float), cudaMemcpyDeviceToHost, s));
	LCD_CUDA(e, cudaStreamSynchronize(s));
	return LCD_OK;
}

// ---- similarity likelihood: Memory::computeLikelihood with Kp/TfIdfLikelihoodUsed=false ----------------------------------------
int lcd_gdesc_count(const lcd_engine * e) { return e ? e->gd_map.count() : 0; }
int lcd_gdesc_dim(const lcd_engine * e) { return e ? e->gd_dim : 0; }

int lcd_gdesc_add(lcd_engine * e, const int * sig_ids, int n, int dim, const float * data)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(require_unsharded(e, "lcd_gdesc_add"));
	if (n <= 0) return LCD_OK;
	if (!sig_ids || !data) LCD_FAIL(e, LCD_ERR_INVALID, "null global descriptors");
	if (dim <= 0) LCD_FAIL(e, LCD_ERR_INVALID, "global descriptors need at least one dimension, got %d", dim);
	if (e->gd_dim != 0 && dim != e->gd_dim) LCD_FAIL(e, LCD_ERR_INVALID, "global descriptors of this engine have %d dimensions, got %d", e->gd_dim, dim);
	LCD_TRY(set_device(e));
	cudaStream_t s = e->stream;
	// a signature that has a descriptor keeps its slot (replace)
	const size_t prev_slots = static_cast<size_t>(e->gd_map.slots);
	std::vector<int> slots;
	if (!e->gd_map.assign(sig_ids, n, slots)) LCD_FAIL(e, LCD_ERR_INVALID, "signature id must be positive");
	e->gd_dim = dim;
	const size_t row = static_cast<size_t>(dim);
	LCD_CUDA(e, e->gd_rows.reserve(static_cast<size_t>(e->gd_map.slots) * row, prev_slots * row, false, s));
	LCD_CUDA(e, write_rows(slots, [&](size_t slot, size_t i, size_t k) {
		return cudaMemcpyAsync(e->gd_rows.p + slot * row, data + i * row, k * row * sizeof(float), cudaMemcpyHostToDevice, s);
	}));
	LCD_CUDA(e, e->gd_map.upload(s));
	LCD_CUDA(e, cudaStreamSynchronize(s));
	return LCD_OK;
}

int lcd_gdesc_remove(lcd_engine * e, const int * sig_ids, int n)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(require_unsharded(e, "lcd_gdesc_remove"));
	if (n <= 0) return LCD_OK;
	if (!sig_ids) LCD_FAIL(e, LCD_ERR_INVALID, "null signature ids");
	LCD_TRY(set_device(e));
	bool changed = false;
	for (int i = 0; i < n; ++i) changed |= e->gd_map.release(sig_ids[i]) >= 0;
	if (!changed) return LCD_OK;
	LCD_CUDA(e, e->gd_map.upload(e->stream));
	LCD_CUDA(e, cudaStreamSynchronize(e->stream));
	return LCD_OK;
}

// UASSERT_MSG(dotProd>=0, ...) of Signature::compareTo (Signature.cpp:264); word-pair values are never negative
static int check_normalized(lcd_engine * e, const float * like, size_t n)
{
	for (size_t i = 0; i < n; ++i)
		if (!(like[i] >= 0.0f)) LCD_FAIL(e, LCD_ERR_INVALID, "Global descriptors should be normalized!");
	return LCD_OK;
}

int lcd_index_similarity(lcd_engine * e, const int * query_word_ids, int nq, const float * query_gdesc, const int * sig_ids, int ns,
                         float * likelihood_out)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(set_device(e));
	LCD_TRY(require_unsharded(e, "lcd_index_similarity"));
	if (nq < 0 || (nq > 0 && !query_word_ids)) LCD_FAIL(e, LCD_ERR_INVALID, "The signature is null");
	if (!sig_ids || ns <= 0 || !likelihood_out) LCD_FAIL(e, LCD_ERR_INVALID, "ids list is empty");
	if (nq > kMaxFrameQueries) LCD_FAIL(e, LCD_ERR_CAPACITY, "at most %d words per signature", kMaxFrameQueries);
	cudaStream_t s = e->stream;
	const int nq1 = std::max(nq, 1); // a signature without words (global descriptor only) is prepared as one invalid id
	LCD_CUDA(e, e->d_in_ids.reserve(nq1, 0, false, s));
	LCD_CUDA(e, e->d_sig_ids.reserve(ns, 0, false, s));
	LCD_CUDA(e, e->d_like.reserve(ns, 0, false, s));
	if (nq > 0) LCD_CUDA(e, cudaMemcpyAsync(e->d_in_ids.p, query_word_ids, nq * sizeof(int), cudaMemcpyHostToDevice, s));
	else LCD_CUDA(e, cudaMemsetAsync(e->d_in_ids.p, 0, sizeof(int), s));
	LCD_CUDA(e, cudaMemcpyAsync(e->d_sig_ids.p, sig_ids, ns * sizeof(int), cudaMemcpyHostToDevice, s));
	const float * d_g = nullptr;
	if (query_gdesc && e->gd_dim > 0)
	{
		LCD_CUDA(e, e->gd_query.reserve(e->gd_dim, 0, false, s));
		LCD_CUDA(e, cudaMemcpyAsync(e->gd_query.p, query_gdesc, e->gd_dim * sizeof(float), cudaMemcpyHostToDevice, s));
		d_g = e->gd_query.p;
	}
	LCD_TRY(prep_ids(e, e->d_in_ids.p, 1, nq1, 0, 0, true, s));
	LCD_TRY(launch_similarity(e, 1, nq1, d_g, e->d_sig_ids.p, ns, e->d_like.p, s));
	LCD_CUDA(e, cudaMemcpyAsync(likelihood_out, e->d_like.p, ns * sizeof(float), cudaMemcpyDeviceToHost, s));
	LCD_CUDA(e, cudaStreamSynchronize(s));
	return check_normalized(e, likelihood_out, static_cast<size_t>(ns));
}

int lcd_localize_similarity_batch_dev(lcd_engine * e, const void * d_queries, int n_frames, int nq_per_frame, int incremental, float nndr,
                                      int new_words_compared_together, const float * d_gdesc, const int * d_sig_ids, int ns,
                                      int * d_word_ids_out, float * d_likelihood_out, void * stream)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(set_device(e));
	LCD_TRY(require_unsharded(e, "lcd_localize_similarity_batch_dev"));
	if (!d_queries || n_frames <= 0) LCD_FAIL(e, LCD_ERR_INVALID, "Descriptors size is null!");
	if (nq_per_frame <= 0 || nq_per_frame > kMaxFrameQueries) LCD_FAIL(e, LCD_ERR_CAPACITY, "1..%d descriptors per frame", kMaxFrameQueries);
	if (d_likelihood_out && (!d_sig_ids || ns <= 0)) LCD_FAIL(e, LCD_ERR_INVALID, "ids list is empty");
	cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : e->stream;
	return localize_dev(e, static_cast<const uint32_t *>(d_queries), n_frames, nq_per_frame, incremental, nndr, new_words_compared_together,
	                    d_sig_ids, ns, 0, d_word_ids_out, d_likelihood_out, s, nullptr, LikelihoodKind::Similarity, e->gd_dim > 0 ? d_gdesc : nullptr);
}

int lcd_localize_similarity_batch(lcd_engine * e, const void * queries, int n_frames, int nq_per_frame, int incremental, float nndr,
                                  int new_words_compared_together, const float * gdesc, const int * sig_ids, int ns,
                                  int * word_ids_out, float * likelihood_out)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(set_device(e));
	LCD_TRY(require_unsharded(e, "lcd_localize_similarity_batch"));
	if (!queries || n_frames <= 0) LCD_FAIL(e, LCD_ERR_INVALID, "Descriptors size is null!");
	if (nq_per_frame <= 0 || nq_per_frame > kMaxFrameQueries) LCD_FAIL(e, LCD_ERR_CAPACITY, "1..%d descriptors per frame", kMaxFrameQueries);
	if (likelihood_out && (!sig_ids || ns <= 0)) LCD_FAIL(e, LCD_ERR_INVALID, "ids list is empty");
	cudaStream_t s = e->stream;
	const size_t nq_total = static_cast<size_t>(n_frames) * nq_per_frame;
	LCD_CUDA(e, e->d_queries.reserve(nq_total * e->nw, 0, false, s));
	LCD_CUDA(e, cudaMemcpyAsync(e->d_queries.p, queries, nq_total * e->nw * 4, cudaMemcpyHostToDevice, s));
	if (word_ids_out) LCD_CUDA(e, e->d_word_ids.reserve(nq_total, 0, false, s));
	const float * d_g = nullptr;
	if (likelihood_out)
	{
		LCD_CUDA(e, e->d_sig_ids.reserve(ns, 0, false, s));
		LCD_CUDA(e, e->d_like.reserve(static_cast<size_t>(n_frames) * ns, 0, false, s));
		LCD_CUDA(e, cudaMemcpyAsync(e->d_sig_ids.p, sig_ids, ns * sizeof(int), cudaMemcpyHostToDevice, s));
		if (gdesc && e->gd_dim > 0)
		{
			const size_t ng = static_cast<size_t>(n_frames) * e->gd_dim;
			LCD_CUDA(e, e->gd_query.reserve(ng, 0, false, s));
			LCD_CUDA(e, cudaMemcpyAsync(e->gd_query.p, gdesc, ng * sizeof(float), cudaMemcpyHostToDevice, s));
			d_g = e->gd_query.p;
		}
	}
	LCD_TRY(localize_dev(e, e->d_queries.p, n_frames, nq_per_frame, incremental, nndr, new_words_compared_together, e->d_sig_ids.p,
	                     likelihood_out ? ns : 0, 0, word_ids_out ? e->d_word_ids.p : nullptr, likelihood_out ? e->d_like.p : nullptr, s, nullptr,
	                     LikelihoodKind::Similarity, d_g));
	if (word_ids_out) LCD_CUDA(e, cudaMemcpyAsync(word_ids_out, e->d_word_ids.p, nq_total * sizeof(int), cudaMemcpyDeviceToHost, s));
	if (likelihood_out)
		LCD_CUDA(e, cudaMemcpyAsync(likelihood_out, e->d_like.p, static_cast<size_t>(n_frames) * ns * sizeof(float), cudaMemcpyDeviceToHost, s));
	LCD_CUDA(e, cudaStreamSynchronize(s));
	return likelihood_out ? check_normalized(e, likelihood_out, static_cast<size_t>(n_frames) * ns) : LCD_OK;
}

// ---- detect (ORB) ------------------------------------------------------------------------------
static int orb_geometry(lcd_engine * e, int width, int height, const lcd_orb_params * p, OrbGeom & g)
{
	if (!p) LCD_FAIL(e, LCD_ERR_INVALID, "null ORB parameters");
	if (p->n_levels < 1 || p->n_levels > kOrbMaxLevels) LCD_FAIL(e, LCD_ERR_INVALID, "ORB/NLevels must be 1..%d", kOrbMaxLevels);
	if (p->scale_factor != 2.0f) LCD_FAIL(e, LCD_ERR_INVALID, "only ORB/ScaleFactor=2 is implemented");
	if (p->patch_size != 31) LCD_FAIL(e, LCD_ERR_INVALID, "only ORB/PatchSize=31 is implemented");
	if (width <= 0 || height <= 0 || (width % (1 << (p->n_levels - 1))) || (height % (1 << (p->n_levels - 1))))
		LCD_FAIL(e, LCD_ERR_INVALID, "image size must be a multiple of 2^(levels-1)");
	if (static_cast<long long>(width) * height >= (1 << 24)) LCD_FAIL(e, LCD_ERR_CAPACITY, "image too large");
	if (p->n_features <= 0) LCD_FAIL(e, LCD_ERR_INVALID, "Kp/MaxFeatures must be positive");
	// FAST compares 8-bit differences; cv::ORB wraps other values modulo 256 rather than clamping them
	if (p->fast_threshold < 0 || p->fast_threshold > 255) LCD_FAIL(e, LCD_ERR_INVALID, "FAST/Threshold must be 0..255");
	g.n_levels = p->n_levels;
	int off = 0;
	for (int l = 0; l < p->n_levels; ++l)
	{
		g.w[l] = width >> l;
		g.h[l] = height >> l;
		g.off[l] = off;
		off += g.w[l] * g.h[l];
	}
	g.frame_stride = off;
	g.edge = p->edge_threshold;
	g.fast_thr = p->fast_threshold;
	g.patch = p->patch_size;
	// ORB computeKeyPoints: features per level (float arithmetic as in OpenCV)
	const float factor = static_cast<float>(1.0 / static_cast<double>(p->scale_factor));
	float nd = p->n_features * (1 - factor) / (1 - static_cast<float>(pow(static_cast<double>(factor), static_cast<double>(p->n_levels))));
	int sum = 0;
	for (int l = 0; l < p->n_levels - 1; ++l)
	{
		g.n_per_level[l] = static_cast<int>(nearbyint(nd));
		sum += g.n_per_level[l];
		nd *= factor;
	}
	g.n_per_level[p->n_levels - 1] = std::max(p->n_features - sum, 0);
	return LCD_OK;
}

// cv::getGaussianKernel(7, 2, CV_32F) into the blur kernels' constant taps, once per engine
static int load_gauss7(lcd_engine * e, cudaStream_t s)
{
	if (e->gauss_sigma_loaded == 2.0f) return LCD_OK;
	// exp(-x^2 / (2 sigma^2)) normalised in double, stored as float
	double t[7], sum = 0;
	for (int i = 0; i < 7; ++i)
	{
		t[i] = exp(-0.5 * (i - 3) * (i - 3) / 4.0);
		sum += t[i];
	}
	float kf[7];
	for (int i = 0; i < 7; ++i) kf[i] = static_cast<float>(t[i] / sum);
	LCD_CUDA(e, cudaMemcpyToSymbolAsync(kOrbGauss7, kf, sizeof(kf), 0, cudaMemcpyHostToDevice, s));
	LCD_CUDA(e, cudaStreamSynchronize(s));
	e->gauss_sigma_loaded = 2.0f;
	return LCD_OK;
}

// 3-D points and plain coordinates of the detected keypoints; d_cam[n_frames] (may be null) the frames' client cameras
static int orb_lift(lcd_engine * e, int n_frames, int width, int height, const void * d_depth, int depth_type, const lcd_orb_params * p, int cap,
                    const OrbKeypoint * d_kp, const int * d_n, float * d_xyz, float * d_uv, cudaStream_t s, const FrameCam * d_cam)
{
	if (d_xyz)
	{
		OrbXyzArgs a{};
		a.depth = (depth_type != LCD_DEPTH_NONE && depth_type != LCD_DEPTH_MASK_U8) ? d_depth : nullptr;
		a.depth_type = depth_type;
		a.w = width;
		a.h = height;
		a.fx = p->fx;
		a.fy = p->fy;
		a.cx = p->cx;
		a.cy = p->cy;
		a.min_depth = p->min_depth;
		a.max_depth = p->max_depth;
		a.cam = d_cam;
		a.kps = d_kp;
		a.n_kp = d_n;
		a.cap = cap;
		a.xyz = d_xyz;
		dim3 grd((cap + 255) / 256, n_frames);
		orb_xyz_kernel<<<grd, 256, 0, s>>>(a);
		LCD_CHECK_LAUNCH(e);
	}
	if (d_uv)
	{
		dim3 grd((cap + 255) / 256, n_frames);
		orb_uv_kernel<<<grd, 256, 0, s>>>(d_kp, d_n, cap, d_uv);
		LCD_CHECK_LAUNCH(e);
	}
	return LCD_OK;
}

// Gray + mask of every frame (orb_prepare*): the vectorised kernel where rows are whole 16-byte vectors and the height is even
static int orb_prepare(lcd_engine * e, int n_frames, const OrbPrepArgs & a, cudaStream_t s)
{
	const int width = a.g.w[0], height = a.g.h[0];
	const bool aligned = ((reinterpret_cast<uintptr_t>(a.images) | reinterpret_cast<uintptr_t>(a.depth) | reinterpret_cast<uintptr_t>(a.gray) |
	                       reinterpret_cast<uintptr_t>(a.mask)) & 15u) == 0 && a.g.frame_stride % 16 == 0;
	if (width % 8 == 0 && height % 2 == 0 && aligned && env_int("LCD_ORB_PREP_VEC", 1) != 0)
	{
		e->orb_path |= 4;
		dim3 blk(16, 16), grd((width / 8 + 15) / 16, (height / 2 + 15) / 16, n_frames);
		orb_prepare_vec_kernel<<<grd, blk, 0, s>>>(a);
	}
	else
	{
		dim3 blk(32, 8), grd(((width + 1) / 2 + 31) / 32, ((height + 1) / 2 + 7) / 8, n_frames);
		orb_prepare_kernel<<<grd, blk, 0, s>>>(a);
	}
	LCD_CHECK_LAUNCH(e);
	return LCD_OK;
}

static int fit_smem(lcd_engine * e, const void * kern, size_t dyn, int cap);

// ORB's keypoints: gray + mask, the coarser pyramid levels, FAST + selection per level, merged into n_features keypoints per frame.  With
// `blur`, the blurred pyramid that feeds the descriptors runs on a side stream under them and s waits for it before returning.
static int fast_pyramid(lcd_engine * e, int n_frames, const OrbPrepArgs & prep, int n_features, bool blur, OrbKeypoint * d_kp, int * d_n, int cap,
                        cudaStream_t s)
{
	const OrbGeom & g = prep.g;
	const int slots = n_frames * g.n_levels;
	// a level stores at most Kp/MaxFeatures keypoints (orb_rank_kernel), and the merge sorts the stored keypoints of all levels of a
	// frame in shared memory: 128 KB for 4 levels at the image-level calls' largest Kp/MaxFeatures; fit_smem checks any other size
	static_assert(kOrbMaxLevels * kMaxFrameQueries * sizeof(unsigned long long) <= 128 * 1024, "merge keys of the largest frame");
	const int level_cap = n_features;
	int pad = 1;
	while (pad < g.n_levels * level_cap) pad <<= 1;
	LCD_TRY(fit_smem(e, reinterpret_cast<const void *>(orb_merge_kernel), pad * sizeof(unsigned long long), n_features));
	LCD_CUDA(e, e->o_cand.reserve(static_cast<size_t>(slots) * kOrbCandCap, 0, false, s));
	LCD_CUDA(e, e->o_cand_count.reserve(slots, 0, false, s));
	LCD_CUDA(e, e->o_surv_n.reserve(slots, 0, false, s));
	LCD_CUDA(e, e->o_rank_ws.reserve(static_cast<size_t>(slots) * kOrbRankWsBytes, 0, false, s));
	LCD_CUDA(e, e->o_level_n.reserve(slots, 0, false, s));
	LCD_CUDA(e, e->o_level_kp.reserve(static_cast<size_t>(slots) * level_cap, 0, false, s));
	uint8_t * const w_gray = prep.gray;
	uint8_t * const w_blur = e->o_blur.p;
	uint8_t * const w_mask = prep.mask;
	uint32_t * const w_cand = e->o_cand.p;
	int * const w_cand_count = e->o_cand_count.p;
	int * const w_surv_n = e->o_surv_n.p;
	unsigned char * const w_rank_ws = e->o_rank_ws.p;
	int * const w_level_n = e->o_level_n.p;
	OrbKeypoint * const w_level_kp = e->o_level_kp.p;
	LCD_CUDA(e, zero_fill_async(w_cand_count, slots * sizeof(int), s));
	LCD_TRY(orb_prepare(e, n_frames, prep, s));
	for (int l = 2; l < g.n_levels; ++l)
	{
		dim3 blk(32, 8), grd((g.w[l] + 31) / 32, (g.h[l] + 7) / 8, n_frames);
		orb_down_kernel<<<grd, blk, 0, s>>>(w_gray, w_mask, g, l);
		LCD_CHECK_LAUNCH(e);
	}
	if (!e->aux_fork)
	{
		LCD_CUDA(e, cudaEventCreateWithFlags(&e->aux_fork, cudaEventDisableTiming));
		LCD_CUDA(e, cudaEventCreateWithFlags(&e->aux_blur_done, cudaEventDisableTiming));
		for (int i = 0; i < 4; ++i)
		{
			LCD_CUDA(e, cudaStreamCreateWithFlags(&e->aux_stream[i], cudaStreamNonBlocking));
			LCD_CUDA(e, cudaEventCreateWithFlags(&e->aux_join[i], cudaEventDisableTiming));
		}
	}
	// one tensor map per pyramid level ([frame][y][x], 96 x 40 boxes): shared by the FAST and the blur kernels
	const int orb_tma = env_int("LCD_ORB_TMA", 1);
	OrbTensorMap tmaps[kOrbMaxLevels];
	bool tma_ok = orb_tma != 0;
	for (int l = 0; l < g.n_levels && tma_ok; ++l)
		tma_ok = make_plane_tensor_map(&tmaps[l], w_gray + g.off[l], g.w[l], g.h[l], n_frames, static_cast<size_t>(g.frame_stride), kFastTmaGW, kFastTmaGH);
	e->orb_tma_used = tma_ok ? 1 : 0;
	if (tma_ok) e->orb_path |= 1;
	LCD_CUDA(e, cudaEventRecord(e->aux_fork, s));
	if (blur)
	{
		// the blurred pyramid only feeds the descriptors: it runs on a side stream under FAST and the (latency-bound) selection
		cudaStream_t bs = e->aux_stream[3];
		LCD_CUDA(e, cudaStreamWaitEvent(bs, e->aux_fork, 0));
		for (int l = 0; l < g.n_levels; ++l)
		{
			if (tma_ok)
			{
				dim3 grd((g.w[l] + kFastTmaTW - 1) / kFastTmaTW, (g.h[l] + kFastTmaTH - 1) / kFastTmaTH, n_frames);
				orb_blur_tma_kernel<<<grd, 256, 0, bs>>>(tmaps[l], w_blur, g, l);
			}
			else
			{
				dim3 grd((g.w[l] + kBlurTW - 1) / kBlurTW, (g.h[l] + kBlurTH - 1) / kBlurTH, n_frames);
				orb_blur_kernel<<<grd, 256, 0, bs>>>(w_gray, w_blur, g, l);
			}
			LCD_CHECK_LAUNCH(e);
		}
		LCD_CUDA(e, cudaEventRecord(e->aux_blur_done, bs));
	}
	{
		OrbSelectArgs a{};
		a.gray = w_gray;
		a.g = g;
		a.cand = w_cand;
		a.cand_count = w_cand_count;
		a.surv_n = w_surv_n;
		a.rank_ws = w_rank_ws;
		a.level_kp = w_level_kp;
		a.level_n = w_level_n;
		a.level_cap = level_cap;
		a.overflow = e->o_overflow.p;
		// The levels are independent: level 0 (the long one) stays on the caller's stream, the coarser ones run FAST + selection on side
		// streams beside it and join before the merge.  The order and rank kernels are one CTA per (frame, level), latency-bound: level l
		// holds at most kOrbCandCap >> l candidates in shared memory (96 KB, 48 KB, 24 KB, ...: two level-0 CTAs per SM), so the FAST / blur
		// CTAs of other levels share its SMs; Harris and the IC angle run over all survivors / keypoints of the level at once.
		LCD_CUDA(e, cudaFuncSetAttribute(orb_order_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
		                                 static_cast<int>(static_cast<size_t>(kOrbCandCap) * (4 + 2))));
		for (int l = g.n_levels - 1; l >= 0; --l)
		{
			cudaStream_t ls = s;
			if (l > 0)
			{
				ls = e->aux_stream[(l - 1) % 3];
				LCD_CUDA(e, cudaStreamWaitEvent(ls, e->aux_fork, 0));
			}
			if (tma_ok)
			{
				// gray tile + halo staged by the TMA engine (one cp.async.bulk.tensor per CTA), byte-SIMD compass test and suppression
				dim3 grd((g.w[l] + kFastTmaTW - 1) / kFastTmaTW, (g.h[l] + kFastTmaTH - 1) / kFastTmaTH, n_frames);
				orb_fast_tma_kernel<<<grd, 256, 0, ls>>>(tmaps[l], w_mask, g, l, w_cand, w_cand_count);
			}
			else
			{
				dim3 grd((g.w[l] + kFastTW - 1) / kFastTW, (g.h[l] + kFastTH - 1) / kFastTH, n_frames);
				orb_fast_kernel<<<grd, 256, 0, ls>>>(w_gray, w_mask, g, l, w_cand, w_cand_count);
			}
			LCD_CHECK_LAUNCH(e);
			a.level = l;
			a.cand_cap = std::max(2048, kOrbCandCap >> l);
			orb_order_kernel<<<n_frames, kOrbSelectThreads, static_cast<size_t>(a.cand_cap) * (4 + 2), ls>>>(a);
			LCD_CHECK_LAUNCH(e);
			// the grids cover the expected survivors (2N) and keypoints (N) of a frame; their blocks stride over the ties beyond
			const int n_level = std::min(g.n_per_level[l], level_cap);
			const dim3 hgrd(std::max(1, (std::min(2 * g.n_per_level[l], a.cand_cap) + kOrbHarrisThreads - 1) / kOrbHarrisThreads), n_frames);
			orb_harris_kernel<<<hgrd, kOrbHarrisThreads, 0, ls>>>(a);
			LCD_CHECK_LAUNCH(e);
			orb_rank_kernel<<<n_frames, kOrbSelectThreads, 0, ls>>>(a);
			LCD_CHECK_LAUNCH(e);
			const int wpb = kOrbAngleThreads / 32;
			orb_angle_kernel<<<dim3(std::max(1, (n_level + wpb - 1) / wpb), n_frames), kOrbAngleThreads, 0, ls>>>(a);
			LCD_CHECK_LAUNCH(e);
			if (l > 0 && l <= 3) LCD_CUDA(e, cudaEventRecord(e->aux_join[l - 1], ls));
		}
		for (int l = 1; l < g.n_levels && l <= 3; ++l) LCD_CUDA(e, cudaStreamWaitEvent(s, e->aux_join[l - 1], 0));
	}
	orb_merge_kernel<<<n_frames, 1024, pad * sizeof(unsigned long long), s>>>(w_level_kp, w_level_n, g.n_levels, level_cap, n_features, d_kp, d_n,
	                                                                          cap);
	LCD_CHECK_LAUNCH(e);
	if (blur) LCD_CUDA(e, cudaStreamWaitEvent(s, e->aux_blur_done, 0));
	return LCD_OK;
}

// GFTT/ORB's keypoints (lcd_detector_set, Kp/DetectorStrategy=8) on one pyramid level: gray + mask, the level-0 blur (with `blur`), the corner
// map with the per-frame maximum, local maxima, per-frame sort, then the minDistance walk + ORB's border filter
static int gftt_corners(lcd_engine * e, int n_frames, const OrbPrepArgs & prep, int n_features, bool blur, OrbKeypoint * d_kp, int * d_n, int cap,
                        cudaStream_t s)
{
	const OrbGeom & g = prep.g;
	const int width = g.w[0], height = g.h[0];
	const int bitmap_words = (width + 31) / 32;
	const size_t bitmap_bytes = static_cast<size_t>(bitmap_words) * height * sizeof(uint32_t);
	const bool bitmap_smem = bitmap_bytes <= static_cast<size_t>(kGfttBitmapSmem);
	LCD_CUDA(e, e->g_eig.reserve(static_cast<size_t>(n_frames) * width * height, 0, false, s));
	LCD_CUDA(e, e->g_max_key.reserve(n_frames, 0, false, s));
	LCD_CUDA(e, e->g_count.reserve(n_frames, 0, false, s));
	LCD_CUDA(e, e->g_keys.reserve(static_cast<size_t>(n_frames) * kGfttCandCap, 0, false, s));
	if (!bitmap_smem) LCD_CUDA(e, e->g_bitmap.reserve(static_cast<size_t>(n_frames) * bitmap_words * height, 0, false, s));
	LCD_CUDA(e, zero_fill_async(e->g_max_key.p, n_frames * sizeof(unsigned), s));
	LCD_CUDA(e, zero_fill_async(e->g_count.p, n_frames * sizeof(int), s));
	LCD_TRY(orb_prepare(e, n_frames, prep, s));
	if (blur)
	{
		dim3 grd((width + kBlurTW - 1) / kBlurTW, (height + kBlurTH - 1) / kBlurTH, n_frames);
		orb_blur_kernel<<<grd, 256, 0, s>>>(prep.gray, e->o_blur.p, g, 0);
		LCD_CHECK_LAUNCH(e);
	}
	{
		GfttEigArgs a{prep.gray, prep.mask, width, height, g.frame_stride, e->g_eig.p, e->g_max_key.p};
		gftt_eig_kernel<<<dim3((width + kGfttColTile - 1) / kGfttColTile, n_frames), 128, 0, s>>>(a);
		LCD_CHECK_LAUNCH(e);
	}
	{
		GfttCandArgs a{e->g_eig.p, prep.mask, width, height, g.frame_stride, e->g_max_key.p, e->gftt.quality_level, e->g_keys.p, e->g_count.p, e->o_overflow.p};
		gftt_cand_kernel<<<dim3((width + 31) / 32, (height + 7) / 8, n_frames), dim3(32, 8), 0, s>>>(a);
		LCD_CHECK_LAUNCH(e);
	}
	{
		const int smem = kGfttSortChunk * static_cast<int>(sizeof(unsigned long long));
		LCD_CUDA(e, cudaFuncSetAttribute(gftt_sort_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
		gftt_sort_kernel<<<n_frames, 1024, smem, s>>>(e->g_keys.p, e->g_count.p);
		LCD_CHECK_LAUNCH(e);
	}
	{
		GfttSelectArgs a{};
		a.keys = e->g_keys.p;
		a.count = e->g_count.p;
		a.w = width;
		a.h = height;
		a.min_distance = e->gftt.min_distance;
		a.max_corners = n_features;
		a.edge = g.edge;
		a.bitmap_words = bitmap_words;
		a.bitmap = bitmap_smem ? nullptr : e->g_bitmap.p;
		a.kps = d_kp;
		a.n_kp = d_n;
		a.cap = cap;
		const int smem = (bitmap_smem && a.min_distance >= 1.0) ? static_cast<int>(bitmap_bytes) : 0;
		LCD_CUDA(e, cudaFuncSetAttribute(gftt_select_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kGfttBitmapSmem));
		gftt_select_kernel<<<n_frames, 256, smem, s>>>(a);
		LCD_CHECK_LAUNCH(e);
	}
	return LCD_OK;
}

// dynamic shared memory of orb_oct_tree_kernel (phase-2 sort keys of the largest level's nodes) and orb_oct_finish_kernel (a frame's keys)
static size_t octree_tree_smem(const OctGeom & g)
{
	int max_nodes = 0;
	for (int l = 0; l < g.n_levels; ++l) max_nodes = std::max(max_nodes, g.node0[l + 1] - g.node0[l]);
	size_t pad = 1;
	while (pad < static_cast<size_t>(max_nodes)) pad <<= 1;
	return pad * sizeof(unsigned long long);
}
static size_t octree_finish_smem(const OctGeom & g)
{
	size_t pad = 1;
	while (pad < static_cast<size_t>(g.raw_cap)) pad <<= 1;
	return pad * sizeof(unsigned long long);
}

// ORB-OCTREE's pyramid, cells and quadtree workspaces (ORBextractor.cc:416-477, :772-855, :1114-1139) on the host, with the inputs on which
// the reference divides by zero, indexes out of range or reads outside a level refused
static int octree_geometry(lcd_engine * e, int width, int height, const lcd_orb_params * p, OctGeom & g, std::vector<OctCell> & cells)
{
	if (p->n_levels < 1 || p->n_levels > kOctMaxLevels) LCD_FAIL(e, LCD_ERR_INVALID, "ORB/NLevels must be 1..%d for ORB-OCTREE", kOctMaxLevels);
	if (!std::isfinite(p->scale_factor) || !(p->scale_factor > 1.0f)) LCD_FAIL(e, LCD_ERR_INVALID, "ORB/ScaleFactor must be finite and > 1");
	if (p->patch_size != 31) LCD_FAIL(e, LCD_ERR_INVALID, "only ORB/PatchSize=31 is implemented");
	// keypoints lie ORB/EdgeThreshold pixels inside a level and the rotated pattern reaches 18: the blurred clone has no border
	if (p->edge_threshold < 19) LCD_FAIL(e, LCD_ERR_INVALID, "ORB-OCTREE needs ORB/EdgeThreshold >= 19");
	if (p->fast_threshold < 0 || p->fast_threshold > 255) LCD_FAIL(e, LCD_ERR_INVALID, "FAST/Threshold must be 0..255");
	// the reference runs Kp/MaxFeatures = 0 (every level's N is 0, no limit); the engine refuses it as it does for the other detectors,
	// whose outputs are sized by it
	if (p->n_features <= 0) LCD_FAIL(e, LCD_ERR_INVALID, "Kp/MaxFeatures must be positive");
	if (width <= 0 || height <= 0) LCD_FAIL(e, LCD_ERR_INVALID, "null image");
	if (static_cast<long long>(width) * height >= (1 << 24)) LCD_FAIL(e, LCD_ERR_CAPACITY, "image too large");
	g = OctGeom{};
	g.n_levels = p->n_levels;
	g.edge = p->edge_threshold;
	g.thr_ini = p->fast_threshold;
	g.thr_min = e->oct_min_threshold;
	// the constructor's tables: float scale chain, float per-level counts
	float scale[kOctMaxLevels], inv[kOctMaxLevels];
	scale[0] = 1.0f;
	for (int l = 1; l < p->n_levels; ++l) scale[l] = scale[l - 1] * p->scale_factor;
	for (int l = 0; l < p->n_levels; ++l) inv[l] = 1.0f / scale[l];
	const float factor = 1.0f / p->scale_factor;
	float nd = p->n_features * (1 - factor) / (1 - static_cast<float>(pow(static_cast<double>(factor), static_cast<double>(p->n_levels))));
	int sum = 0;
	for (int l = 0; l < p->n_levels - 1; ++l)
	{
		g.n_per_level[l] = static_cast<int>(nearbyintf(nd));
		sum += g.n_per_level[l];
		nd *= factor;
	}
	g.n_per_level[p->n_levels - 1] = std::max(p->n_features - sum, 0);
	{
		const int half = 15;
		const int vmax = static_cast<int>(floorf(half * sqrtf(2.f) / 2 + 1)), vmin = static_cast<int>(ceilf(half * sqrtf(2.f) / 2));
		for (int v = 0; v <= vmax; ++v) g.umax[v] = static_cast<int>(nearbyint(sqrt(static_cast<double>(half * half - v * v))));
		for (int v = half, v0 = 0; v >= vmin; --v)
		{
			while (g.umax[v0] == g.umax[v0 + 1]) ++v0;
			g.umax[v] = v0;
			++v0;
		}
	}
	const int min_b = p->edge_threshold - 3;
	int off = 0, key = 0, node = 0;
	cells.clear();
	for (int l = 0; l < p->n_levels; ++l)
	{
		const int w = static_cast<int>(nearbyintf(static_cast<float>(width) * inv[l])), h = static_cast<int>(nearbyintf(static_cast<float>(height) * inv[l]));
		const int max_bx = w - p->edge_threshold + 3, max_by = h - p->edge_threshold + 3;
		const int sw = max_bx - min_b, sh = max_by - min_b;
		// nCols = (maxX - minX) / 30 and nRows must not be 0 (the cell size divides by them)
		if (sw < 30 || sh < 30)
			LCD_FAIL(e, LCD_ERR_INVALID, "ORB-OCTREE level %d is %dx%d: under 30 pixels remain inside ORB/EdgeThreshold", l, w, h);
		// DistributeOctTree's initial node count round(w / h) must not be 0 (a level more than twice as tall as wide)
		const int n_ini = static_cast<int>(roundf(static_cast<float>(sw) / static_cast<float>(sh)));
		if (n_ini == 0) LCD_FAIL(e, LCD_ERR_INVALID, "ORB-OCTREE level %d is %dx%d: more than twice as tall as wide", l, w, h);
		g.w[l] = w;
		g.h[l] = h;
		g.off[l] = off;
		off += w * h;
		g.scale[l] = scale[l];
		g.size[l] = static_cast<int>(31 * scale[l]);
		g.span_w[l] = sw;
		g.span_h[l] = sh;
		g.n_ini[l] = n_ini;
		g.hx[l] = static_cast<float>(sw) / n_ini;
		// ComputeKeyPointsOctTree's cells, in float arithmetic as the reference
		const float W = 30, width_f = static_cast<float>(sw), height_f = static_cast<float>(sh);
		const int n_cols = static_cast<int>(width_f / W), n_rows = static_cast<int>(height_f / W);
		const int w_cell = static_cast<int>(ceilf(width_f / n_cols)), h_cell = static_cast<int>(ceilf(height_f / n_rows));
		g.cell0[l] = static_cast<int>(cells.size());
		g.key0[l] = key;
		for (int i = 0; i < n_rows; ++i)
		{
			const float ini_y = static_cast<float>(min_b + i * h_cell);
			float max_y = ini_y + h_cell + 6;
			if (ini_y >= max_by - 3) continue;
			if (max_y > max_by) max_y = static_cast<float>(max_by);
			for (int j = 0; j < n_cols; ++j)
			{
				const float ini_x = static_cast<float>(min_b + j * w_cell);
				float max_x = ini_x + w_cell + 6;
				if (ini_x >= max_bx - 6) continue;
				if (max_x > max_bx) max_x = static_cast<float>(max_bx);
				OctCell c{static_cast<int>(ini_x), static_cast<int>(ini_y), static_cast<int>(max_x), static_cast<int>(max_y), j * w_cell, i * h_cell, key, l};
				// strict 3x3 maxima of the cell's [3, n-3) window are never 8-adjacent
				const int iw = std::max(c.x1 - c.x0 - 6, 0), ih = std::max(c.y1 - c.y0 - 6, 0);
				key += ((iw + 1) / 2) * ((ih + 1) / 2);
				cells.push_back(c);
			}
		}
		g.node0[l] = node;
		node += std::max(g.n_per_level[l] + 3, 4 * n_ini) + 4;
	}
	g.cell0[p->n_levels] = static_cast<int>(cells.size());
	g.key0[p->n_levels] = key;
	g.node0[p->n_levels] = node;
	g.raw_cap = node;
	g.frame_stride = (off + 15) & ~15;
	if (g.raw_cap >= 65536) LCD_FAIL(e, LCD_ERR_CAPACITY, "ORB-OCTREE keeps at most 65535 keypoints per frame before Kp/MaxFeatures");
	// the shared memory of the quadtree's phase-2 sort and of the final limit, checked before anything is launched
	LCD_TRY(fit_smem(e, reinterpret_cast<const void *>(orb_oct_tree_kernel), octree_tree_smem(g), p->n_features));
	LCD_TRY(fit_smem(e, reinterpret_cast<const void *>(orb_oct_finish_kernel), octree_finish_smem(g), p->n_features));
	return LCD_OK;
}

// ORB-OCTREE (lcd_detector_set_orb_octree, Kp/DetectorStrategy=10): gray + mask, pyramid, FAST per cell, quadtree per level, angle, blur,
// descriptors, then the mask and Kp/MaxFeatures of rtabmap::ORBOctree, and the 3-D points
static int octree_run(lcd_engine * e, int n_frames, const uint8_t * d_images, int width, int height, int channels, const void * d_depth, int depth_type,
                      const lcd_orb_params * p, int cap, OrbKeypoint * d_kp, uint8_t * d_desc, float * d_xyz, float * d_uv, int * d_n, cudaStream_t s,
                      const FrameCam * d_cam)
{
	OctGeom g{};
	std::vector<OctCell> cells;
	LCD_TRY(octree_geometry(e, width, height, p, g, cells));
	if (channels != 1 && channels != 3) LCD_FAIL(e, LCD_ERR_INVALID, "images must be 8UC1 or 8UC3 (BGR)");
	if (cap <= 0 || cap > kMaxFrameQueries) LCD_FAIL(e, LCD_ERR_CAPACITY, "cap must be 1..%d", kMaxFrameQueries);
	if (!d_depth) depth_type = LCD_DEPTH_NONE;
	if (depth_type < LCD_DEPTH_NONE || depth_type > LCD_DEPTH_MASK_U8) LCD_FAIL(e, LCD_ERR_INVALID, "unknown depth type %d", depth_type);
	const bool use_mask = depth_type == LCD_DEPTH_MASK_U8 || (depth_type != LCD_DEPTH_NONE && p->depth_as_mask);
	const int n_cells = static_cast<int>(cells.size());
	const int key_stride = g.key0[g.n_levels], node_stride = g.node0[g.n_levels];
	const size_t pyr = static_cast<size_t>(n_frames) * g.frame_stride;
	LCD_CUDA(e, e->o_gray.reserve(pyr, 0, false, s));
	LCD_CUDA(e, e->o_blur.reserve(pyr, 0, false, s));
	if (use_mask) LCD_CUDA(e, e->o_mask.reserve(pyr, 0, false, s));
	LCD_CUDA(e, e->o_overflow.reserve(1, 0, true, s));
	LCD_CUDA(e, zero_fill_async(e->o_overflow.p, sizeof(int), s)); // no cell can overflow its slot: the flag stays clear
	if (!d_kp)
	{
		LCD_CUDA(e, e->o_kp.reserve(static_cast<size_t>(n_frames) * cap, 0, false, s));
		d_kp = e->o_kp.p;
	}
	if (!d_n)
	{
		LCD_CUDA(e, e->o_n.reserve(n_frames, 0, false, s));
		d_n = e->o_n.p;
	}
	if (!d_desc)
	{
		LCD_CUDA(e, e->oc_desc.reserve(static_cast<size_t>(n_frames) * cap * 32, 0, false, s));
		d_desc = e->oc_desc.p;
	}
	const size_t keys = static_cast<size_t>(n_frames) * key_stride, nodes = static_cast<size_t>(n_frames) * node_stride;
	LCD_CUDA(e, e->oc_cells.reserve(n_cells, 0, false, s));
	LCD_CUDA(e, e->oc_cell_n.reserve(static_cast<size_t>(n_frames) * n_cells, 0, false, s));
	LCD_CUDA(e, e->oc_keys.reserve(keys, 0, false, s));
	LCD_CUDA(e, e->oc_kk.reserve(keys, 0, false, s));
	LCD_CUDA(e, e->oc_perm.reserve(keys, 0, false, s));
	LCD_CUDA(e, e->oc_scratch.reserve(keys, 0, false, s));
	LCD_CUDA(e, e->oc_nodes.reserve(2 * nodes, 0, false, s));
	LCD_CUDA(e, e->oc_cand.reserve(nodes, 0, false, s));
	LCD_CUDA(e, e->oc_cnt.reserve(nodes, 0, false, s));
	LCD_CUDA(e, e->oc_expand.reserve(nodes, 0, false, s));
	LCD_CUDA(e, e->oc_sel.reserve(nodes, 0, false, s));
	LCD_CUDA(e, e->oc_sel_n.reserve(static_cast<size_t>(n_frames) * g.n_levels, 0, false, s));
	LCD_CUDA(e, e->oc_raw_kp.reserve(static_cast<size_t>(n_frames) * g.raw_cap, 0, false, s));
	LCD_CUDA(e, e->oc_raw_desc.reserve(static_cast<size_t>(n_frames) * g.raw_cap * 32, 0, false, s));
	if (e->oc_cells_at != e->oc_cells.p || e->oc_cells_host.size() != cells.size() ||
	    std::memcmp(e->oc_cells_host.data(), cells.data(), cells.size() * sizeof(OctCell)) != 0)
	{
		// a new geometry (or a regrown buffer): the table is a few KB, copied once from the engine's own host copy, which outlives the copy
		e->oc_cells_host = cells;
		e->oc_cells_at = e->oc_cells.p;
		LCD_CUDA(e, cudaMemcpyAsync(e->oc_cells.p, e->oc_cells_host.data(), n_cells * sizeof(OctCell), cudaMemcpyHostToDevice, s));
	}
	prof_mark(e, LCD_PROF_ORB, s);
	e->orb_path = 16;
	{
		OrbPrepArgs prep{};
		prep.images = d_images;
		prep.channels = channels;
		prep.depth = use_mask ? d_depth : nullptr;
		prep.depth_type = depth_type;
		prep.min_depth = p->min_depth;
		prep.max_depth = p->max_depth;
		prep.gray = e->o_gray.p;
		prep.mask = use_mask ? e->o_mask.p : nullptr;
		prep.g.n_levels = 1;
		prep.g.w[0] = width;
		prep.g.h[0] = height;
		prep.g.frame_stride = g.frame_stride;
		orb_oct_prepare_kernel<<<dim3((width + 31) / 32, (height + 7) / 8, n_frames), dim3(32, 8), 0, s>>>(prep);
		LCD_CHECK_LAUNCH(e);
	}
	for (int l = 1; l < g.n_levels; ++l)
	{
		orb_oct_resize_kernel<<<dim3((g.w[l] + 31) / 32, (g.h[l] + 7) / 8, n_frames), dim3(32, 8), 0, s>>>(e->o_gray.p, g, l);
		LCD_CHECK_LAUNCH(e);
	}
	orb_oct_fast_kernel<<<dim3(n_cells, n_frames), 256, 0, s>>>(e->o_gray.p, g, e->oc_cells.p, n_cells, key_stride, e->oc_keys.p, e->oc_cell_n.p);
	LCD_CHECK_LAUNCH(e);
	{
		OctTreeArgs a{};
		a.g = g;
		a.keys = e->oc_keys.p;
		a.cell_n = e->oc_cell_n.p;
		a.cells = e->oc_cells.p;
		a.n_cells = n_cells;
		a.key_stride = key_stride;
		a.node_stride = node_stride;
		a.kk = e->oc_kk.p;
		a.perm = e->oc_perm.p;
		a.scratch = e->oc_scratch.p;
		a.nodes = e->oc_nodes.p;
		a.cand = e->oc_cand.p;
		a.cnt = e->oc_cnt.p;
		a.expand = e->oc_expand.p;
		a.sel = e->oc_sel.p;
		a.sel_n = e->oc_sel_n.p;
		orb_oct_tree_kernel<<<dim3(g.n_levels, n_frames), kOctTreeThreads, octree_tree_smem(g), s>>>(a);
		LCD_CHECK_LAUNCH(e);
	}
	for (int l = 0; l < g.n_levels; ++l)
	{
		orb_oct_blur_kernel<<<dim3((g.w[l] + 31) / 32, (g.h[l] + 7) / 8, n_frames), dim3(32, 8), 0, s>>>(e->o_gray.p, e->o_blur.p, g, l);
		LCD_CHECK_LAUNCH(e);
	}
	{
		int max_nodes = 0;
		for (int l = 0; l < g.n_levels; ++l) max_nodes = std::max(max_nodes, g.node0[l + 1] - g.node0[l]);
		orb_oct_describe_kernel<<<dim3((max_nodes + 7) / 8, g.n_levels, n_frames), 256, 0, s>>>(e->o_gray.p, e->o_blur.p, g, e->oc_sel.p, e->oc_sel_n.p,
		                                                                                      node_stride, e->oc_raw_kp.p, e->oc_raw_desc.p);
		LCD_CHECK_LAUNCH(e);
	}
	{
		orb_oct_finish_kernel<<<n_frames, 1024, octree_finish_smem(g), s>>>(e->oc_raw_kp.p, e->oc_raw_desc.p, e->oc_sel_n.p, g,
		                                                                               use_mask ? e->o_mask.p : nullptr, p->n_features, d_kp, d_desc, d_n, cap);
		LCD_CHECK_LAUNCH(e);
	}
	LCD_TRY(orb_lift(e, n_frames, width, height, d_depth, depth_type, p, cap, d_kp, d_n, d_xyz, d_uv, s, d_cam));
	prof_mark(e, LCD_PROF_ORB, s);
	return LCD_OK;
}

// Detect + describe a batch of frames with the engine's detector (lcd_detector_set): the FAST pyramid or GFTT's corners between the
// shared preparation and the steered BRIEF descriptors and 3-D points.  A null d_kp / d_n detects into the engine's own buffers.
// d_cam[n_frames] (may be null): the frames' client cameras the 3-D points are lifted with.
static int orb_run(lcd_engine * e, int n_frames, const uint8_t * d_images, int width, int height, int channels, const void * d_depth,
                   int depth_type, const lcd_orb_params * p, int cap, OrbKeypoint * d_kp, uint8_t * d_desc, float * d_xyz, float * d_uv,
                   int * d_n, cudaStream_t s, const FrameCam * d_cam = nullptr)
{
	if (!p) LCD_FAIL(e, LCD_ERR_INVALID, "null ORB parameters");
	if (e->detector == LCD_DETECTOR_ORB_OCTREE)
		return octree_run(e, n_frames, d_images, width, height, channels, d_depth, depth_type, p, cap, d_kp, d_desc, d_xyz, d_uv, d_n, s, d_cam);
	const bool gftt = e->detector == LCD_DETECTOR_GFTT_ORB;
	lcd_orb_params pl = *p;
	if (gftt) pl.n_levels = 1; // cv::ORB::compute builds the levels its keypoints use: GFTT corners are all octave 0
	OrbGeom g{};
	LCD_TRY(orb_geometry(e, width, height, &pl, g));
	if (gftt && (width % 2 || height % 2)) LCD_FAIL(e, LCD_ERR_INVALID, "GFTT/ORB needs an even image width and height");
	if (channels != 1 && channels != 3) LCD_FAIL(e, LCD_ERR_INVALID, "images must be 8UC1 or 8UC3 (BGR)");
	if (cap <= 0 || cap > kMaxFrameQueries) LCD_FAIL(e, LCD_ERR_CAPACITY, "cap must be 1..%d", kMaxFrameQueries);
	if (!d_depth) depth_type = LCD_DEPTH_NONE;
	if (depth_type < LCD_DEPTH_NONE || depth_type > LCD_DEPTH_MASK_U8) LCD_FAIL(e, LCD_ERR_INVALID, "unknown depth type %d", depth_type);
	const bool use_mask = depth_type == LCD_DEPTH_MASK_U8 || (depth_type != LCD_DEPTH_NONE && p->depth_as_mask);
	const size_t pyr = static_cast<size_t>(n_frames) * g.frame_stride;
	LCD_CUDA(e, e->o_gray.reserve(pyr, 0, false, s));
	LCD_CUDA(e, e->o_blur.reserve(pyr, 0, false, s));
	if (use_mask) LCD_CUDA(e, e->o_mask.reserve(pyr, 0, false, s));
	// the "candidate list truncated" flag of this batch: cleared here, read back by the host entry points
	LCD_CUDA(e, e->o_overflow.reserve(1, 0, true, s));
	LCD_CUDA(e, zero_fill_async(e->o_overflow.p, sizeof(int), s));
	if (!d_kp)
	{
		LCD_CUDA(e, e->o_kp.reserve(static_cast<size_t>(n_frames) * cap, 0, false, s));
		d_kp = e->o_kp.p;
	}
	if (!d_n)
	{
		LCD_CUDA(e, e->o_n.reserve(n_frames, 0, false, s));
		d_n = e->o_n.p;
	}
	LCD_TRY(load_gauss7(e, s));
	prof_mark(e, LCD_PROF_ORB, s);
	OrbPrepArgs prep{};
	prep.images = d_images;
	prep.channels = channels;
	prep.depth = use_mask ? d_depth : nullptr;
	prep.depth_type = depth_type;
	prep.min_depth = p->min_depth;
	prep.max_depth = p->max_depth;
	prep.gray = e->o_gray.p;
	prep.mask = use_mask ? e->o_mask.p : nullptr;
	prep.g = g;
	e->orb_path = gftt ? 8 : 0;
	if (gftt)
		LCD_TRY(gftt_corners(e, n_frames, prep, p->n_features, d_desc != nullptr, d_kp, d_n, cap, s));
	else
		LCD_TRY(fast_pyramid(e, n_frames, prep, p->n_features, d_desc != nullptr, d_kp, d_n, cap, s));
	if (d_desc)
	{
		dim3 grd((cap + kOrbDescribeKp - 1) / kOrbDescribeKp, n_frames);
		bool patch_ok = g.edge >= kOrbPatchR && env_int("LCD_ORB_PATCH", 1) != 0;
		for (int l = 0; l < g.n_levels; ++l) patch_ok = patch_ok && g.w[l] % 4 == 0;
		if (patch_ok)
		{
			e->orb_path |= 2;
			orb_describe_patch_kernel<<<grd, 256, 0, s>>>(e->o_blur.p, g, d_kp, d_n, cap, d_desc);
		}
		else
			orb_describe_kernel<<<grd, 256, 0, s>>>(e->o_gray.p, e->o_blur.p, g, d_kp, d_n, cap, d_desc);
		LCD_CHECK_LAUNCH(e);
	}
	LCD_TRY(orb_lift(e, n_frames, width, height, d_depth, depth_type, p, cap, d_kp, d_n, d_xyz, d_uv, s, d_cam));
	prof_mark(e, LCD_PROF_ORB, s);
	return LCD_OK;
}

// LCD_ERR_CAPACITY when orb_run's overflow flag is set: a frame had more candidates than `detector` keeps, and the message names its limit
static int overflow_report(lcd_engine * e, int overflow, int detector)
{
	if (overflow && detector == LCD_DETECTOR_GFTT_ORB)
		LCD_FAIL(e, LCD_ERR_CAPACITY, "more than %d GFTT candidates in a frame: raise GFTT/QualityLevel", kGfttCandCap);
	if (overflow) LCD_FAIL(e, LCD_ERR_CAPACITY, "more than %d FAST corners in pyramid level 0 (half as many per further level): raise FAST/Threshold", kOrbCandCap);
	return LCD_OK;
}

// The detection outputs of the image-level calls whose descriptors feed the dictionary search: a 32-byte binary engine, Kp/MaxFeatures
// (cap) in 1..kMaxFrameQueries, room for n_frames frames and zeroed descriptors, so that the padding rows of short frames hold defined
// bytes for the NN kernel.  uv may be null.
static int frame_front_end(lcd_engine * e, int n_frames, int cap, DevBuf<OrbKeypoint> & kp, DevBuf<uint8_t> & desc, DevBuf<float> & xyz,
                           DevBuf<float> * uv, DevBuf<int> & n, cudaStream_t s)
{
	if (e->cfg.desc_type != LCD_DESC_U8 || e->cfg.desc_dim != 32) LCD_FAIL(e, LCD_ERR_INVALID, "ORB descriptors need an engine with 32-byte binary descriptors");
	if (cap <= 0 || cap > kMaxFrameQueries) LCD_FAIL(e, LCD_ERR_CAPACITY, "Kp/MaxFeatures must be 1..%d", kMaxFrameQueries);
	const size_t rows = static_cast<size_t>(n_frames) * cap;
	LCD_CUDA(e, kp.reserve(rows, 0, false, s));
	LCD_CUDA(e, desc.reserve(rows * 32, 0, false, s));
	LCD_CUDA(e, xyz.reserve(rows * 3, 0, false, s));
	if (uv) LCD_CUDA(e, uv->reserve(rows * 2, 0, false, s));
	LCD_CUDA(e, n.reserve(n_frames, 0, false, s));
	LCD_CUDA(e, zero_fill_async(desc.p, rows * 32, s));
	return LCD_OK;
}

// n_frames host frames, and their depth when there is one (depth_type becomes LCD_DEPTH_NONE without), into device buffers on s
static int upload_frames(lcd_engine * e, int n_frames, int width, int height, int channels, const uint8_t * images, const void * depth, int & depth_type,
                         DevBuf<uint8_t> & d_images, DevBuf<unsigned char> & d_depth, cudaStream_t s)
{
	const size_t px = static_cast<size_t>(n_frames) * width * height;
	if (!depth) depth_type = LCD_DEPTH_NONE;
	LCD_CUDA(e, d_images.reserve(px * channels, 0, false, s));
	LCD_CUDA(e, cudaMemcpyAsync(d_images.p, images, px * channels, cudaMemcpyHostToDevice, s));
	if (depth_type != LCD_DEPTH_NONE)
	{
		const size_t bytes = px * depth_elem_bytes(depth_type);
		LCD_CUDA(e, d_depth.reserve(bytes, 0, false, s));
		LCD_CUDA(e, cudaMemcpyAsync(d_depth.p, depth, bytes, cudaMemcpyHostToDevice, s));
	}
	return LCD_OK;
}

int lcd_orb_detect_describe_dev(lcd_engine * e, int n_frames, const uint8_t * d_images, int width, int height, int channels, const void * d_depth,
                                int depth_type, const lcd_orb_params * params, int cap, lcd_keypoint * d_kp_out, uint8_t * d_desc_out,
                                float * d_xyz_out, float * d_uv_out, int * d_n_out, void * stream)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(set_device(e));
	if (!d_images || n_frames <= 0) LCD_FAIL(e, LCD_ERR_INVALID, "null image");
	static_assert(sizeof(lcd_keypoint) == sizeof(OrbKeypoint), "keypoint layout");
	cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : e->stream;
	return orb_run(e, n_frames, d_images, width, height, channels, d_depth, depth_type, params, cap, reinterpret_cast<OrbKeypoint *>(d_kp_out),
	               d_desc_out, d_xyz_out, d_uv_out, d_n_out, s);
}

int lcd_orb_detect_describe(lcd_engine * e, int n_frames, const uint8_t * images, int width, int height, int channels, const void * depth,
                            int depth_type, const lcd_orb_params * params, int cap, lcd_keypoint * kp_out, uint8_t * desc_out, float * xyz_out,
                            int * n_out)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(set_device(e));
	if (!images || n_frames <= 0 || width <= 0 || height <= 0) LCD_FAIL(e, LCD_ERR_INVALID, "null image");
	if (cap <= 0 || cap > kMaxFrameQueries) LCD_FAIL(e, LCD_ERR_CAPACITY, "cap must be 1..%d", kMaxFrameQueries);
	cudaStream_t s = e->orb_stream; // not the dictionary's stream: this call may overlap lcd_dict_update (Memory.cpp:5284)
	LCD_TRY(upload_frames(e, n_frames, width, height, channels, images, depth, depth_type, e->o_img, e->o_depth, s));
	const size_t rows = static_cast<size_t>(n_frames) * cap;
	LCD_CUDA(e, e->o_kp.reserve(rows, 0, false, s));
	LCD_CUDA(e, e->o_desc.reserve(rows * 32, 0, false, s));
	LCD_CUDA(e, e->o_xyz.reserve(rows * 3, 0, false, s));
	LCD_CUDA(e, e->o_n.reserve(n_frames, 0, false, s));
	LCD_TRY(orb_run(e, n_frames, e->o_img.p, width, height, channels, depth_type != LCD_DEPTH_NONE ? e->o_depth.p : nullptr, depth_type, params, cap,
	                e->o_kp.p, desc_out ? e->o_desc.p : nullptr, xyz_out ? e->o_xyz.p : nullptr, nullptr, e->o_n.p, s));
	if (kp_out) LCD_CUDA(e, cudaMemcpyAsync(kp_out, e->o_kp.p, rows * sizeof(OrbKeypoint), cudaMemcpyDeviceToHost, s));
	if (desc_out) LCD_CUDA(e, cudaMemcpyAsync(desc_out, e->o_desc.p, rows * 32, cudaMemcpyDeviceToHost, s));
	if (xyz_out) LCD_CUDA(e, cudaMemcpyAsync(xyz_out, e->o_xyz.p, rows * 3 * sizeof(float), cudaMemcpyDeviceToHost, s));
	if (n_out) LCD_CUDA(e, cudaMemcpyAsync(n_out, e->o_n.p, n_frames * sizeof(int), cudaMemcpyDeviceToHost, s));
	int overflow = 0;
	LCD_CUDA(e, cudaMemcpyAsync(&overflow, e->o_overflow.p, sizeof(int), cudaMemcpyDeviceToHost, s));
	LCD_CUDA(e, cudaStreamSynchronize(s));
	return overflow_report(e, overflow, e->detector);
}

int lcd_detector_set(lcd_engine * e, int detector, const lcd_gftt_params * params)
{
	if (!e) return LCD_ERR_INVALID;
	if (detector == LCD_DETECTOR_ORB)
	{
		e->detector = detector;
		return LCD_OK;
	}
	if (detector == LCD_DETECTOR_ORB_OCTREE) LCD_FAIL(e, LCD_ERR_INVALID, "ORB-OCTREE is selected with lcd_detector_set_orb_octree");
	if (detector != LCD_DETECTOR_GFTT_ORB) LCD_FAIL(e, LCD_ERR_INVALID, "unknown detector %d", detector);
	const lcd_gftt_params q = params ? *params : lcd_gftt_params{0.001, 7.0, 3, 0, 0.04};
	if (q.use_harris != 0) LCD_FAIL(e, LCD_ERR_INVALID, "GFTT/UseHarrisDetector is not implemented");
	if (q.block_size != 3) LCD_FAIL(e, LCD_ERR_INVALID, "only GFTT/BlockSize=3 is implemented");
	if (!(q.quality_level > 0.0) || !std::isfinite(q.quality_level)) LCD_FAIL(e, LCD_ERR_INVALID, "GFTT/QualityLevel must be positive");
	if (!(q.min_distance >= 0.0) || !std::isfinite(q.min_distance)) LCD_FAIL(e, LCD_ERR_INVALID, "GFTT/MinDistance must not be negative");
	e->gftt = q;
	e->detector = detector;
	return LCD_OK;
}

int lcd_detector_set_orb_octree(lcd_engine * e, int fast_min_threshold)
{
	if (!e) return LCD_ERR_INVALID;
	if (fast_min_threshold < 0 || fast_min_threshold > 255) LCD_FAIL(e, LCD_ERR_INVALID, "FAST/MinThreshold must be 0..255");
	e->oct_min_threshold = fast_min_threshold;
	e->detector = LCD_DETECTOR_ORB_OCTREE;
	return LCD_OK;
}

int lcd_debug_orb_sincos(lcd_engine * e, unsigned first, unsigned count, float * d_cos, float * d_sin)
{
	if (!e || !d_cos || !d_sin) return LCD_ERR_INVALID;
	LCD_TRY(set_device(e));
	if (count == 0) return LCD_OK;
	orb_oct_sincos_kernel<<<(count + 255) / 256, 256, 0, e->stream>>>(first, count, d_cos, d_sin);
	LCD_CHECK_LAUNCH(e);
	LCD_CUDA(e, cudaStreamSynchronize(e->stream));
	return LCD_OK;
}

int lcd_detector_get(const lcd_engine * e, lcd_gftt_params * params)
{
	if (!e) return LCD_ERR_INVALID;
	if (params) *params = e->gftt;
	return e->detector;
}

// ---- the quantisation limit of Memory::createSignature (limit.cuh) ----------------------------------------------------------------
int lcd_quantize_limit_set(lcd_engine * e, const lcd_quantize_limit * p)
{
	if (!e) return LCD_ERR_INVALID;
	const lcd_quantize_limit q = p ? *p : lcd_quantize_limit{0, 0.0f, 0};
	if (q.max_features < 0) LCD_FAIL(e, LCD_ERR_INVALID, "Kp/MaxFeatures must not be negative");
	if (q.mean_words < 0) LCD_FAIL(e, LCD_ERR_INVALID, "meanWordsPerLocation must not be negative");
	if (!(q.bad_sign_ratio >= 0.0f) || !std::isfinite(q.bad_sign_ratio)) LCD_FAIL(e, LCD_ERR_INVALID, "Kp/BadSignRatio must be finite and not negative");
	e->ql = q;
	e->ql_gate = static_cast<int>(q.bad_sign_ratio * static_cast<float>(q.mean_words)); // Memory.cpp:5947
	return LCD_OK;
}

int lcd_quantize_limit_get(const lcd_engine * e, lcd_quantize_limit * p)
{
	if (!e || !p) return LCD_ERR_INVALID;
	*p = e->ql;
	return LCD_OK;
}

// rows a frame of `cap` keypoints quantises at most under the engine's limit
static int limit_rows(const lcd_engine * e, int cap) { return e->ql.max_features > 0 ? std::min(e->ql.max_features, cap) : cap; }
// whether the image-level calls split their frames (the default {0, 0, 0} does not: today's path, bit for bit)
static bool limit_active(const lcd_engine * e) { return e->ql.max_features > 0 || e->ql_gate > 0; }

static int launch_limit(lcd_engine * e, int n_frames, int cap, const OrbKeypoint * d_kp, const int * d_n, const uint32_t * d_desc, uint32_t * d_desc_out,
                        int * d_index_out, int * d_n_out, cudaStream_t s)
{
	int pad = 1;
	while (pad < cap) pad <<= 1;
	limit_keypoints_kernel<<<n_frames, kLimitThreads, pad * sizeof(unsigned long long), s>>>(d_kp, d_n, d_desc, cap, e->nw, e->ql.max_features,
	                                                                                         limit_rows(e, cap), e->ql_gate, d_desc_out, d_index_out, d_n_out);
	LCD_CHECK_LAUNCH(e);
	return LCD_OK;
}

static int launch_expand(lcd_engine * e, int n_frames, int cap, int k, const int * d_n, const int * d_index, const int * d_nq, const int * d_words_q,
                         int * d_words_out, cudaStream_t s)
{
	word_ids_expand_kernel<<<dim3((cap + 255) / 256, n_frames), 256, 0, s>>>(cap, k, d_n, d_index, d_nq, d_words_q, d_words_out);
	LCD_CHECK_LAUNCH(e);
	return LCD_OK;
}

// the quantised rows of n_frames detected frames in the engine's ql_* buffers
static int limit_to_engine(lcd_engine * e, int n_frames, int cap, const OrbKeypoint * d_kp, const int * d_n, const uint32_t * d_desc, cudaStream_t s)
{
	const size_t rows = static_cast<size_t>(n_frames) * limit_rows(e, cap);
	LCD_CUDA(e, e->ql_desc.reserve(rows * e->nw, 0, false, s));
	LCD_CUDA(e, e->ql_index.reserve(rows, 0, false, s));
	LCD_CUDA(e, e->ql_words.reserve(rows, 0, false, s));
	LCD_CUDA(e, e->ql_n.reserve(n_frames, 0, false, s));
	return launch_limit(e, n_frames, cap, d_kp, d_n, d_desc, e->ql_desc.p, e->ql_index.p, e->ql_n.p, s);
}

int lcd_limit_keypoints_dev(lcd_engine * e, int n_frames, int cap, const lcd_keypoint * d_kp, const int * d_n, const void * d_desc, void * d_desc_out,
                            int * d_index_out, int * d_n_out, void * stream)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(set_device(e));
	if (n_frames <= 0 || !d_kp || !d_n || !d_desc || !d_desc_out || !d_index_out || !d_n_out) LCD_FAIL(e, LCD_ERR_INVALID, "null argument");
	if (cap <= 0 || cap > kMaxFrameQueries) LCD_FAIL(e, LCD_ERR_CAPACITY, "cap must be 1..%d", kMaxFrameQueries);
	cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : e->stream;
	return launch_limit(e, n_frames, cap, reinterpret_cast<const OrbKeypoint *>(d_kp), d_n, static_cast<const uint32_t *>(d_desc),
	                    static_cast<uint32_t *>(d_desc_out), d_index_out, d_n_out, s);
}

int lcd_word_ids_expand_dev(lcd_engine * e, int n_frames, int cap, int k, const int * d_n, const int * d_index, const int * d_n_quantised,
                            const int * d_words_q, int * d_words_out, void * stream)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(set_device(e));
	if (n_frames <= 0 || !d_n || !d_index || !d_n_quantised || !d_words_q || !d_words_out) LCD_FAIL(e, LCD_ERR_INVALID, "null argument");
	if (cap <= 0 || cap > kMaxFrameQueries) LCD_FAIL(e, LCD_ERR_CAPACITY, "cap must be 1..%d", kMaxFrameQueries);
	if (k <= 0 || k > cap) LCD_FAIL(e, LCD_ERR_INVALID, "k must be 1..cap");
	cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : e->stream;
	return launch_expand(e, n_frames, cap, k, d_n, d_index, d_n_quantised, d_words_q, d_words_out, s);
}

int lcd_orb_overflow(lcd_engine * e)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(set_device(e));
	if (!e->o_overflow.p) return 0;
	int flag = 0;
	LCD_CUDA(e, cudaDeviceSynchronize());
	LCD_CUDA(e, cudaMemcpy(&flag, e->o_overflow.p, sizeof(int), cudaMemcpyDeviceToHost));
	return flag ? 1 : 0;
}

int lcd_orb_last_path(const lcd_engine * e)
{
	return e ? e->orb_path : LCD_ERR_INVALID;
}

long long lcd_debug_orb_buffer(lcd_engine * e, int which, void * out, long long cap_bytes)
{
	if (!e || !out) return LCD_ERR_INVALID;
	if (set_device(e) != LCD_OK) return LCD_ERR_CUDA;
	const void * src = nullptr;
	size_t bytes = 0;
	switch (which)
	{
	case 0: src = e->o_gray.p; bytes = e->o_gray.cap; break;
	case 1: src = e->o_mask.p; bytes = e->o_mask.cap; break;
	case 2: src = e->o_blur.p; bytes = e->o_blur.cap; break;
	case 3: src = e->o_cand.p; bytes = e->o_cand.cap * sizeof(uint32_t); break;
	case 4: src = e->o_cand_count.p; bytes = e->o_cand_count.cap * sizeof(int); break;
	case 5: src = e->o_level_n.p; bytes = e->o_level_n.cap * sizeof(int); break;
	case 6: src = e->o_surv_n.p; bytes = e->o_surv_n.cap * sizeof(int); break;
	case 7: src = e->v_clk.p; bytes = e->v_clk.cap * sizeof(long long); break;
#ifdef LCD_DEBUG_PHASES
	case 9:
	{
		void * sym = nullptr;
		if (cudaGetSymbolAddress(&sym, g_match_dbg) != cudaSuccess) return LCD_ERR_CUDA;
		src = sym;
		bytes = sizeof(long long) * 8;
		break;
	}
#endif
	case 8:
	{
		void * sym = nullptr;
		if (cudaGetSymbolAddress(&sym, g_pnp_dbg) != cudaSuccess) return LCD_ERR_CUDA;
		src = sym;
		bytes = sizeof(long long) * 8;
		break;
	}
	default: return LCD_ERR_INVALID;
	}
	if (!src) return 0;
	bytes = std::min<size_t>(bytes, static_cast<size_t>(cap_bytes));
	if (cudaMemcpy(out, src, bytes, cudaMemcpyDeviceToHost) != cudaSuccess) return LCD_ERR_CUDA;
	return static_cast<long long>(bytes);
}

// ---- geometric verification ------------------------------------------------------------------
// Stages the host's pairs in the engine's verification buffers; src: those buffers, FROM and TO row = pair.
static int verify_upload(lcd_engine * e, int n_pairs, int cap, const void * desc_from, const float * xyz_from, const int * n_from,
                         const void * desc_to, const float * uv_to, const float * xyz_to, const int * n_to, cudaStream_t s, PairSource & src)
{
	const size_t rows = static_cast<size_t>(n_pairs) * cap;
	LCD_CUDA(e, e->v_df.reserve(rows * e->nw, 0, false, s));
	LCD_CUDA(e, e->v_dt.reserve(rows * e->nw, 0, false, s));
	LCD_CUDA(e, e->v_xyz.reserve(rows * 3, 0, false, s));
	LCD_CUDA(e, e->v_uv.reserve(rows * 2, 0, false, s));
	LCD_CUDA(e, e->v_nf.reserve(n_pairs, 0, false, s));
	LCD_CUDA(e, e->v_nt.reserve(n_pairs, 0, false, s));
	LCD_CUDA(e, cudaMemcpyAsync(e->v_df.p, desc_from, rows * e->nw * 4, cudaMemcpyHostToDevice, s));
	LCD_CUDA(e, cudaMemcpyAsync(e->v_dt.p, desc_to, rows * e->nw * 4, cudaMemcpyHostToDevice, s));
	if (xyz_from) LCD_CUDA(e, cudaMemcpyAsync(e->v_xyz.p, xyz_from, rows * 3 * sizeof(float), cudaMemcpyHostToDevice, s));
	else LCD_CUDA(e, cudaMemsetAsync(e->v_xyz.p, 0, rows * 3 * sizeof(float), s));
	if (uv_to) LCD_CUDA(e, cudaMemcpyAsync(e->v_uv.p, uv_to, rows * 2 * sizeof(float), cudaMemcpyHostToDevice, s));
	else LCD_CUDA(e, cudaMemsetAsync(e->v_uv.p, 0, rows * 2 * sizeof(float), s));
	LCD_CUDA(e, cudaMemcpyAsync(e->v_nf.p, n_from, n_pairs * sizeof(int), cudaMemcpyHostToDevice, s));
	LCD_CUDA(e, cudaMemcpyAsync(e->v_nt.p, n_to, n_pairs * sizeof(int), cudaMemcpyHostToDevice, s));
	if (xyz_to)
	{
		LCD_CUDA(e, e->v_xyz_to.reserve(rows * 3, 0, false, s));
		LCD_CUDA(e, cudaMemcpyAsync(e->v_xyz_to.p, xyz_to, rows * 3 * sizeof(float), cudaMemcpyHostToDevice, s));
	}
	src = PairSource{{e->v_df.p, e->v_xyz.p, e->v_nf.p, nullptr, cap},
	                 {e->v_dt.p, e->v_uv.p, xyz_to ? e->v_xyz_to.p : nullptr, e->v_nt.p, 0, cap, nullptr}};
	return LCD_OK;
}

// Shared memory of one verification launch: LCD_ERR_CAPACITY unless the kernel's static shared memory plus dyn fits the device's
// opt-in limit per block; raises the kernel's dynamic limit when the default 48 KB is exceeded.  A failed runtime call is taken off
// the runtime's last error too, so the next launch check of the engine does not report it again.
static int fit_smem(lcd_engine * e, const void * kern, size_t dyn, int cap)
{
	cudaFuncAttributes fa{};
	cudaError_t c = cudaFuncGetAttributes(&fa, kern);
	if (c != cudaSuccess)
	{
		cudaGetLastError();
		LCD_FAIL(e, LCD_ERR_CUDA, "cudaFuncGetAttributes failed: %s", cudaGetErrorString(c));
	}
	const size_t need = fa.sharedSizeBytes + dyn;
	if (need > static_cast<size_t>(e->smem_optin))
		LCD_FAIL(e, LCD_ERR_CAPACITY, "cap %d needs %zu B of shared memory (%zu B static), the device allows %d", cap, need, fa.sharedSizeBytes, e->smem_optin);
	if (need > 48 * 1024)
	{
		c = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(dyn));
		if (c != cudaSuccess)
		{
			cudaGetLastError();
			LCD_FAIL(e, LCD_ERR_CUDA, "cudaFuncSetAttribute(%zu B) failed: %s", dyn, cudaGetErrorString(c));
		}
	}
	return LCD_OK;
}

// Float descriptors: FROM dictionaries (cached per store row, or built per host pair), the TO x dictionary scan, then the TO new-word
// loop and the correspondences (verify.cuh).  a: launch_match's arguments, with the store's FROM-dictionary cache when from_store.
static int launch_match_l2(lcd_engine * e, const PairSource & src, int n_pairs, int cap, float nndr, bool from_store, MatchArgs a, cudaStream_t s)
{
	const int d = e->nw; // 64, 128 or 256
	const auto kern_fd = d == 64 ? from_dict_l2_kernel<64> : d == 128 ? from_dict_l2_kernel<128> : from_dict_l2_kernel<256>;
	const auto kern_scan = d == 64 ? to_dict_knn2_l2_kernel<64> : d == 128 ? to_dict_knn2_l2_kernel<128> : to_dict_knn2_l2_kernel<256>;
	const auto kern = d == 64 ? pair_match_l2_kernel<64> : d == 128 ? pair_match_l2_kernel<128> : pair_match_l2_kernel<256>;
	FromDictArgs fa{src.from.desc, src.from.n, src.from.slot, src.from.cap, std::min(cap, src.from.cap), nndr, e->st_ftag.p, e->st_kof.p, e->st_creator.p};
	if (!from_store)
	{
		// host pairs: FROM row = pair (src.from.slot is nullptr), built on every call
		const size_t frows = static_cast<size_t>(n_pairs) * src.from.cap;
		LCD_CUDA(e, e->v_kof.reserve(frows, 0, false, s));
		LCD_CUDA(e, e->v_creator.reserve(frows, 0, false, s));
		LCD_CUDA(e, e->v_ftag.reserve(n_pairs, 0, false, s));
		fa.tag = e->v_ftag.p;
		fa.kof = e->v_kof.p;
		fa.creator = e->v_creator.p;
		a.from_tag = fa.tag;
		a.from_kof = fa.kof;
		a.from_creator = fa.creator;
	}
	LCD_CUDA(e, e->v_keys64.reserve(static_cast<size_t>(n_pairs) * cap, 0, false, s));
	const size_t smem_fd = from_dict_l2_smem_bytes(fa.rows), smem = match_l2_smem_bytes(cap);
	LCD_TRY(fit_smem(e, reinterpret_cast<const void *>(kern_fd), smem_fd, cap));
	LCD_TRY(fit_smem(e, reinterpret_cast<const void *>(kern), smem, cap));
	prof_mark(e, LCD_PROF_MATCH, s);
	kern_fd<<<n_pairs, kL2ResolveThreads, smem_fd, s>>>(fa);
	kern_scan<<<dim3(n_pairs, (cap + kL2ScanThreads - 1) / kL2ScanThreads), kL2ScanThreads, 0, s>>>(a, e->v_keys64.p);
	kern<<<n_pairs, kL2ResolveThreads, smem, s>>>(a, e->v_keys64.p);
	prof_mark(e, LCD_PROF_MATCH, s);
	LCD_CHECK_LAUNCH(e);
	return LCD_OK;
}

static int launch_match(lcd_engine * e, const PairSource & src, int n_pairs, int cap, float nndr, bool want_ids, cudaStream_t s)
{
	const size_t rows = static_cast<size_t>(n_pairs) * cap;
	LCD_CUDA(e, e->v_obj.reserve(rows * 3, 0, false, s));
	LCD_CUDA(e, e->v_img.reserve(rows * 2, 0, false, s));
	LCD_CUDA(e, e->v_mid.reserve(rows, 0, false, s));
	LCD_CUDA(e, e->v_mfrom.reserve(rows, 0, false, s));
	LCD_CUDA(e, e->v_mto.reserve(rows, 0, false, s));
	LCD_CUDA(e, e->v_nm.reserve(n_pairs, 0, false, s));
	if (want_ids)
	{
		LCD_CUDA(e, e->v_fid.reserve(rows, 0, false, s));
		LCD_CUDA(e, e->v_tid.reserve(rows, 0, false, s));
	}
	MatchArgs a{};
	a.src = src;
	if (src.to.xyz) LCD_CUDA(e, e->v_obj_to.reserve(rows * 3, 0, false, s));
	a.obj_to = src.to.xyz ? e->v_obj_to.p : nullptr;
	a.cap = cap;
	a.nndr = nndr;
	a.obj = e->v_obj.p;
	a.img = e->v_img.p;
	a.match_id = e->v_mid.p;
	a.match_from = e->v_mfrom.p;
	a.match_to = e->v_mto.p;
	a.n_match = e->v_nm.p;
	a.from_ids = want_ids ? e->v_fid.p : nullptr;
	a.to_ids = want_ids ? e->v_tid.p : nullptr;
	// FROM rows of the signature store: their temporary dictionaries are cached next to the store (from_dict_build_kernel)
	const bool from_store = src.from.slot && src.from.desc == e->st_desc.p;
	FromDictArgs fa{};
	if (from_store)
	{
		a.from_tag = e->st_ftag.p;
		a.from_kof = e->st_kof.p;
		a.from_creator = e->st_creator.p;
		fa = FromDictArgs{src.from.desc, src.from.n, src.from.slot, src.from.cap, std::min(cap, src.from.cap), nndr, e->st_ftag.p, e->st_kof.p, e->st_creator.p};
	}
	if (e->f32) return launch_match_l2(e, src, n_pairs, cap, nndr, from_store, a, s);
	const size_t smem = match_smem_bytes(cap, e->nw), smem_fd = from_dict_smem_bytes(fa.rows, e->nw);
#define LCD_MATCH_CASE(NW_)                                                                                                 \
	case NW_:                                                                                                               \
	{                                                                                                                       \
		auto kern = pair_match_kernel<NW_>;                                                                                 \
		auto kern_fd = from_dict_build_kernel<NW_>;                                                                         \
		LCD_TRY(fit_smem(e, reinterpret_cast<const void *>(kern), smem, cap));                                              \
		if (from_store) LCD_TRY(fit_smem(e, reinterpret_cast<const void *>(kern_fd), smem_fd, cap));                        \
		prof_mark(e, LCD_PROF_MATCH, s);                                                                                    \
		if (from_store) kern_fd<<<n_pairs, kResolveThreads, smem_fd, s>>>(fa);                                              \
		kern<<<n_pairs, kResolveThreads, smem, s>>>(a);                                                                     \
		prof_mark(e, LCD_PROF_MATCH, s);                                                                                    \
		break;                                                                                                              \
	}
	switch (e->nw)
	{
		LCD_MATCH_CASE(4)
		LCD_MATCH_CASE(8)
		LCD_MATCH_CASE(16)
	default: LCD_FAIL(e, LCD_ERR_INVALID, "unsupported descriptor size");
	}
#undef LCD_MATCH_CASE
	LCD_CHECK_LAUNCH(e);
	return LCD_OK;
}

// obj_to: words3B of each correspondence (launch_match's v_obj_to) or nullptr; src (may be null): the pairs' TO cameras (src->to.cam)
static int launch_pnp(lcd_engine * e, int n_pairs, int cap, const lcd_verify_params * p, const float * obj_to, cudaStream_t s,
                      bool gate_min_matches = true, bool want_cov = true, const PairSource * src = nullptr)
{
	const size_t rows = static_cast<size_t>(n_pairs) * cap;
	if (want_cov && p->var_median_ratio <= 1) LCD_FAIL(e, LCD_ERR_INVALID, "Vis/PnPVarianceMedianRatio must be > 1 (UASSERT in estimateMotion3DTo2D)");
	LCD_CUDA(e, e->v_cov6.reserve(n_pairs * 6, 0, false, s));
	LCD_CUDA(e, e->v_rvec.reserve(n_pairs * 3, 0, false, s));
	LCD_CUDA(e, e->v_tvec.reserve(n_pairs * 3, 0, false, s));
	LCD_CUDA(e, e->v_inl.reserve(rows, 0, false, s));
	LCD_CUDA(e, e->v_ninl.reserve(n_pairs, 0, false, s));
	LCD_CUDA(e, e->v_iters.reserve(n_pairs, 0, false, s));
	LCD_CUDA(e, e->v_ok.reserve(n_pairs, 0, false, s));
	LCD_CUDA(e, e->v_T.reserve(n_pairs * 12, 0, false, s));
	LCD_CUDA(e, e->v_clk.reserve(n_pairs * 16, 0, false, s));
	PnpArgs a{};
	a.obj = e->v_obj.p;
	a.img = e->v_img.p;
	a.n_pts = e->v_nm.p;
	a.cap = cap;
	a.cam = CamK{p->fx, p->fy, p->cx, p->cy};
	a.iterations = p->iterations;
	a.reproj = p->reproj_error;
	a.min_inliers = p->min_inliers;
	a.refine_iterations = p->refine_iterations;
	a.refine_sigma = p->refine_sigma;
	a.gate_min_matches = gate_min_matches ? 1 : 0;
	a.obj_to = obj_to;
	a.var_median_ratio = p->var_median_ratio;
	a.max_variance = p->max_variance;
	a.split_linear = p->split_linear_cov;
	a.img_w = p->image_width;
	a.img_h = p->image_height;
	a.cam_tab = src ? src->to.cam : nullptr;
	a.cam_row = src ? src->to.row : nullptr;
	a.cov6 = want_cov ? e->v_cov6.p : nullptr;
	a.rvec = e->v_rvec.p;
	a.tvec = e->v_tvec.p;
	a.inliers = e->v_inl.p;
	a.n_inliers = e->v_ninl.p;
	a.iters_run = e->v_iters.p;
	a.ok = e->v_ok.p;
	a.transform = e->v_T.p;
	static const int pnp_clocks = env_int("LCD_PNP_CLOCKS", 0); // diagnostics: phase clocks of the RANSAC kernel (lcd_debug_orb_buffer 7)
	a.phase_clk = pnp_clocks ? e->v_clk.p : nullptr;
	const size_t smem = pnp_smem_bytes(cap);
	LCD_TRY(fit_smem(e, reinterpret_cast<const void *>(pnp_ransac_kernel), smem, cap));
	prof_mark(e, LCD_PROF_PNP, s);
	pnp_ransac_kernel<<<n_pairs, kVerifyThreads, smem, s>>>(a);
	prof_mark(e, LCD_PROF_PNP, s);
	LCD_CHECK_LAUNCH(e);
	return LCD_OK;
}

// Reg/RepeatOnce: the second registration pass of the pairs whose first pass succeeded (guess_match_kernel), then PnP again on all pairs
// (pairs that keep their first-pass correspondences reproduce their first-pass result).  src and obj_to: those of the first pass.
// cam_sized: a pair's own TO camera (src.to.cam) has an image size; the pass needs one, the call's or the pair's.
static int launch_second_pass(lcd_engine * e, const PairSource & src, int n_pairs, int cap, const lcd_verify_params * p, float * obj_to, cudaStream_t s,
                              bool cam_sized)
{
	if (!p->repeat_once || p->guess_win_size <= 0 || ((p->image_width <= 0 || p->image_height <= 0) && !cam_sized)) return LCD_OK;
	GuessMatchArgs a{};
	a.src = src;
	a.cap = cap;
	a.ok1 = e->v_ok.p;
	a.rvec = e->v_rvec.p;
	a.tvec = e->v_tvec.p;
	a.cam = CamK{p->fx, p->fy, p->cx, p->cy};
	a.img_w = p->image_width;
	a.img_h = p->image_height;
	a.win = static_cast<float>(p->guess_win_size);
	a.nndr = p->nndr;
	a.obj = e->v_obj.p;
	a.img = e->v_img.p;
	a.obj_to = obj_to;
	a.match_id = e->v_mid.p;
	a.match_from = e->v_mfrom.p;
	a.match_to = e->v_mto.p;
	a.n_match = e->v_nm.p;
	const size_t smem = guess_smem_bytes(cap);
#define LCD_GUESS_CASE(NW_, DESC_)                                                                                       \
	case NW_:                                                                                                            \
	{                                                                                                                    \
		auto kern = guess_match_kernel<DESC_>;                                                                           \
		LCD_TRY(fit_smem(e, reinterpret_cast<const void *>(kern), smem, cap));                                           \
		prof_mark(e, LCD_PROF_MATCH, s);                                                                                 \
		kern<<<n_pairs, 256, smem, s>>>(a);                                                                              \
		prof_mark(e, LCD_PROF_MATCH, s);                                                                                 \
		break;                                                                                                           \
	}
	switch (e->nw) // 32-bit words per row: 4, 8, 16 binary; 64, 128, 256 float
	{
		LCD_GUESS_CASE(4, HammingDesc<4>)
		LCD_GUESS_CASE(8, HammingDesc<8>)
		LCD_GUESS_CASE(16, HammingDesc<16>)
		LCD_GUESS_CASE(64, L2Desc<64>)
		LCD_GUESS_CASE(128, L2Desc<128>)
		LCD_GUESS_CASE(256, L2Desc<256>)
	default: LCD_FAIL(e, LCD_ERR_INVALID, "unsupported descriptor size");
	}
#undef LCD_GUESS_CASE
	LCD_CHECK_LAUNCH(e);
	return launch_pnp(e, n_pairs, cap, p, obj_to, s, true, true, &src);
}

// Memory::computeTransform of every pair: global matching, PnP, then the Reg/RepeatOnce pass.  cap: stride of the outputs, at least
// both row strides of src.  The covariance takes words3B from src.to.xyz when it is set.  A pair whose TO row has a camera in src.to.cam
// registers with it; cam_sized: one of those cameras has an image size.
static int register_pairs(lcd_engine * e, const PairSource & src, int n_pairs, int cap, const lcd_verify_params * vp, cudaStream_t s,
                          bool cam_sized = false)
{
	LCD_TRY(launch_match(e, src, n_pairs, cap, vp->nndr, false, s));
	float * obj_to = src.to.xyz ? e->v_obj_to.p : nullptr;
	LCD_TRY(launch_pnp(e, n_pairs, cap, vp, obj_to, s, true, true, &src));
	return launch_second_pass(e, src, n_pairs, cap, vp, obj_to, s, cam_sized);
}

static int check_verify_params(lcd_engine * e, const lcd_verify_params * vp, bool need_store)
{
	if (!vp) LCD_FAIL(e, LCD_ERR_INVALID, "null verification parameters");
	if (vp->iterations > kMaxRansacIters) LCD_FAIL(e, LCD_ERR_CAPACITY, "Vis/Iterations > %d", kMaxRansacIters);
	if (need_store && e->st_cap == 0) LCD_FAIL(e, LCD_ERR_STATE, "the signature store is empty: nothing to verify against");
	return LCD_OK;
}

// the per-pair verification outputs of the last registration as lcd_verify_result rows
static int pack_verify_results(lcd_engine * e, int n, PackedVerifyResult * d_out, cudaStream_t s)
{
	static_assert(sizeof(PackedVerifyResult) == sizeof(lcd_verify_result), "PackedVerifyResult must mirror lcd_verify_result");
	pack_verify_results_kernel<<<(n + 127) / 128, 128, 0, s>>>(n, e->v_ok.p, e->v_nm.p, e->v_ninl.p, e->v_iters.p, e->v_rvec.p, e->v_tvec.p, e->v_T.p,
	                                                          e->v_cov6.p, d_out);
	LCD_CHECK_LAUNCH(e);
	return LCD_OK;
}

// copy the per-pair verification outputs back (cap = 0: skip the id arrays)
static int verify_download(lcd_engine * e, int n_pairs, int cap, lcd_verify_result * results, int * match_ids, int * inlier_ids, cudaStream_t s)
{
	const size_t rows = static_cast<size_t>(n_pairs) * cap;
	if (cap > 0 && inlier_ids)
	{
		LCD_CUDA(e, e->v_inl_ids.reserve(rows, 0, false, s));
		gather_by_index_kernel<<<dim3((cap + 255) / 256, n_pairs), 256, 0, s>>>(e->v_mid.p, e->v_inl.p, e->v_ninl.p, cap, e->v_inl_ids.p);
		LCD_CHECK_LAUNCH(e);
	}
	LCD_CUDA(e, e->v_packed.reserve(n_pairs, 0, false, s));
	LCD_CUDA(e, e->h_packed.reserve(n_pairs));
	LCD_TRY(pack_verify_results(e, n_pairs, e->v_packed.p, s));
	LCD_CUDA(e, cudaMemcpyAsync(e->h_packed.p, e->v_packed.p, n_pairs * sizeof(PackedVerifyResult), cudaMemcpyDeviceToHost, s));
	if (cap > 0 && match_ids) LCD_CUDA(e, cudaMemcpyAsync(match_ids, e->v_mid.p, rows * sizeof(int), cudaMemcpyDeviceToHost, s));
	if (cap > 0 && inlier_ids) LCD_CUDA(e, cudaMemcpyAsync(inlier_ids, e->v_inl_ids.p, rows * sizeof(int), cudaMemcpyDeviceToHost, s));
	LCD_CUDA(e, cudaStreamSynchronize(s));
	memcpy(results, e->h_packed.p, n_pairs * sizeof(lcd_verify_result));
	return LCD_OK;
}

static int check_verify_args(lcd_engine * e, int n_pairs, int cap, const void * a, const void * b, const int * na, const int * nb)
{
	if (n_pairs <= 0 || cap <= 0 || !a || !b || !na || !nb) LCD_FAIL(e, LCD_ERR_INVALID, "null or empty verification input");
	if (cap > kMaxFrameQueries) LCD_FAIL(e, LCD_ERR_CAPACITY, "at most %d features per signature", kMaxFrameQueries);
	return LCD_OK;
}

int lcd_match_pairs(lcd_engine * e, int n_pairs, int cap, const void * desc_from, const int * n_from, const void * desc_to,
                    const int * n_to, float nndr, int * from_ids, int * to_ids)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(require_binary(e, "lcd_match_pairs"));
	LCD_TRY(set_device(e));
	LCD_TRY(check_verify_args(e, n_pairs, cap, desc_from, desc_to, n_from, n_to));
	cudaStream_t s = e->stream;
	PairSource src;
	LCD_TRY(verify_upload(e, n_pairs, cap, desc_from, nullptr, n_from, desc_to, nullptr, nullptr, n_to, s, src));
	LCD_TRY(launch_match(e, src, n_pairs, cap, nndr, true, s));
	const size_t rows = static_cast<size_t>(n_pairs) * cap;
	if (from_ids) LCD_CUDA(e, cudaMemcpyAsync(from_ids, e->v_fid.p, rows * sizeof(int), cudaMemcpyDeviceToHost, s));
	if (to_ids) LCD_CUDA(e, cudaMemcpyAsync(to_ids, e->v_tid.p, rows * sizeof(int), cudaMemcpyDeviceToHost, s));
	LCD_CUDA(e, cudaStreamSynchronize(s));
	return LCD_OK;
}

int lcd_verify_batch(lcd_engine * e, int n_pairs, int cap, const void * desc_from, const float * xyz_from, const int * n_from,
                     const void * desc_to, const float * uv_to, const float * xyz_to, const int * n_to, const lcd_verify_params * params,
                     lcd_verify_result * results, int * match_ids, int * inlier_ids)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(set_device(e));
	LCD_TRY(check_verify_args(e, n_pairs, cap, desc_from, desc_to, n_from, n_to));
	if (!xyz_from || !uv_to || !params || !results) LCD_FAIL(e, LCD_ERR_INVALID, "null verification argument");
	LCD_TRY(check_verify_params(e, params, false));
	cudaStream_t s = e->stream;
	PairSource src;
	LCD_TRY(verify_upload(e, n_pairs, cap, desc_from, xyz_from, n_from, desc_to, uv_to, xyz_to, n_to, s, src));
	LCD_TRY(register_pairs(e, src, n_pairs, cap, params, s));
	return verify_download(e, n_pairs, cap, results, match_ids, inlier_ids, s);
}

long long lcd_verify_static_smem(lcd_engine * e, int which)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(set_device(e));
	const void * kern = nullptr;
	switch (which * 1000 + e->nw) // nw: 4, 8, 16 binary; 64, 128, 256 float
	{
	case 4: kern = reinterpret_cast<const void *>(pair_match_kernel<4>); break;
	case 8: kern = reinterpret_cast<const void *>(pair_match_kernel<8>); break;
	case 16: kern = reinterpret_cast<const void *>(pair_match_kernel<16>); break;
	case 1004: kern = reinterpret_cast<const void *>(guess_match_kernel<HammingDesc<4>>); break;
	case 1008: kern = reinterpret_cast<const void *>(guess_match_kernel<HammingDesc<8>>); break;
	case 1016: kern = reinterpret_cast<const void *>(guess_match_kernel<HammingDesc<16>>); break;
	case 2004: case 2008: case 2016: kern = reinterpret_cast<const void *>(pnp_ransac_kernel); break;
	case 3004: kern = reinterpret_cast<const void *>(from_dict_build_kernel<4>); break;
	case 3008: kern = reinterpret_cast<const void *>(from_dict_build_kernel<8>); break;
	case 3016: kern = reinterpret_cast<const void *>(from_dict_build_kernel<16>); break;
	// float engines (nw = 64, 128, 256 floats)
	case 64: kern = reinterpret_cast<const void *>(pair_match_l2_kernel<64>); break;
	case 128: kern = reinterpret_cast<const void *>(pair_match_l2_kernel<128>); break;
	case 256: kern = reinterpret_cast<const void *>(pair_match_l2_kernel<256>); break;
	case 1064: kern = reinterpret_cast<const void *>(guess_match_kernel<L2Desc<64>>); break;
	case 1128: kern = reinterpret_cast<const void *>(guess_match_kernel<L2Desc<128>>); break;
	case 1256: kern = reinterpret_cast<const void *>(guess_match_kernel<L2Desc<256>>); break;
	case 2064: case 2128: case 2256: kern = reinterpret_cast<const void *>(pnp_ransac_kernel); break;
	case 3064: kern = reinterpret_cast<const void *>(from_dict_l2_kernel<64>); break;
	case 3128: kern = reinterpret_cast<const void *>(from_dict_l2_kernel<128>); break;
	case 3256: kern = reinterpret_cast<const void *>(from_dict_l2_kernel<256>); break;
	default: LCD_FAIL(e, LCD_ERR_INVALID, "no verification kernel %d", which);
	}
	cudaFuncAttributes fa{};
	LCD_CUDA(e, cudaFuncGetAttributes(&fa, kern));
	return static_cast<long long>(fa.sharedSizeBytes);
}

// ---- stand-alone PnP RANSAC: util3d::solvePnPRansac ------------------------------------------------
static int check_pnp_camera(lcd_engine * e, const double K[9], const double * dist_coeffs, int n_dist, int flags)
{
	if (!K) LCD_FAIL(e, LCD_ERR_INVALID, "null camera matrix");
	if (K[1] != 0.0 || K[3] != 0.0 || K[6] != 0.0 || K[7] != 0.0 || K[8] != 1.0 || !(K[0] > 0.0) || !(K[4] > 0.0))
		LCD_FAIL(e, LCD_ERR_INVALID, "camera matrix must be [fx 0 cx; 0 fy cy; 0 0 1]");
	for (int i = 0; i < n_dist; ++i)
		if (dist_coeffs && dist_coeffs[i] != 0.0)
			LCD_FAIL(e, LCD_ERR_INVALID, "distortion coefficients are not supported: rectify first (CameraModel::D() is zero for rectified images, CameraModel.h:111)");
	if (flags != 0) LCD_FAIL(e, LCD_ERR_INVALID, "Vis/PnPFlags=%d is not implemented (0 = cv::SOLVEPNP_ITERATIVE only)", flags);
	return LCD_OK;
}

int lcd_pnp_ransac_batch(lcd_engine * e, int n_sets, int cap, const float * object_points, const float * image_points, const int * n_points,
                         const double K[9], const double * dist_coeffs, int n_dist, double * rvec, double * tvec, int use_extrinsic_guess,
                         int iterations, float reproj_error, int min_inliers, int flags, int refine_iterations, float refine_sigma,
                         int * inliers_out, int * n_inliers_out, int * iterations_run_out)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(set_device(e));
	if (n_sets <= 0 || cap <= 0 || !object_points || !image_points || !n_points || !rvec || !tvec) LCD_FAIL(e, LCD_ERR_INVALID, "null or empty PnP input");
	if (cap > kMaxFrameQueries) LCD_FAIL(e, LCD_ERR_CAPACITY, "at most %d correspondences per set", kMaxFrameQueries);
	LCD_TRY(check_pnp_camera(e, K, dist_coeffs, n_dist, flags));
	if (iterations > kMaxRansacIters) LCD_FAIL(e, LCD_ERR_CAPACITY, "iterationsCount > %d", kMaxRansacIters);
	for (int i = 0; i < n_sets; ++i)
	{
		if (n_points[i] < 0 || n_points[i] > cap) LCD_FAIL(e, LCD_ERR_INVALID, "set %d has %d points (cap %d)", i, n_points[i], cap);
		// cv3::solvePnPRansac switches to P3P on exactly four points (opencv/solvepnp.cpp:150-154): not implemented
		if (n_points[i] == 4) LCD_FAIL(e, LCD_ERR_INVALID, "set %d has exactly 4 points: the reference solves it with P3P, which is not implemented", i);
	}
	(void)use_extrinsic_guess; // the RANSAC kernel is EPnP on 6 points, which ignores the guess; on failure rvec / tvec are left untouched
	cudaStream_t s = e->stream;
	const size_t rows = static_cast<size_t>(n_sets) * cap;
	LCD_CUDA(e, e->v_obj.reserve(rows * 3, 0, false, s));
	LCD_CUDA(e, e->v_img.reserve(rows * 2, 0, false, s));
	LCD_CUDA(e, e->v_nm.reserve(n_sets, 0, false, s));
	LCD_CUDA(e, cudaMemcpyAsync(e->v_obj.p, object_points, rows * 3 * sizeof(float), cudaMemcpyHostToDevice, s));
	LCD_CUDA(e, cudaMemcpyAsync(e->v_img.p, image_points, rows * 2 * sizeof(float), cudaMemcpyHostToDevice, s));
	LCD_CUDA(e, cudaMemcpyAsync(e->v_nm.p, n_points, n_sets * sizeof(int), cudaMemcpyHostToDevice, s));
	lcd_verify_params vp{};
	vp.min_inliers = min_inliers;
	vp.iterations = iterations;
	vp.reproj_error = reproj_error;
	vp.refine_iterations = refine_iterations;
	vp.refine_sigma = refine_sigma;
	vp.fx = K[0];
	vp.fy = K[4];
	vp.cx = K[2];
	vp.cy = K[5];
	vp.var_median_ratio = 2;
	LCD_TRY(launch_pnp(e, n_sets, cap, &vp, nullptr, s, false, false));
	std::vector<double> hr(static_cast<size_t>(n_sets) * 3), ht(static_cast<size_t>(n_sets) * 3);
	std::vector<int> hn(n_sets), hit(n_sets);
	LCD_CUDA(e, cudaMemcpyAsync(hr.data(), e->v_rvec.p, hr.size() * sizeof(double), cudaMemcpyDeviceToHost, s));
	LCD_CUDA(e, cudaMemcpyAsync(ht.data(), e->v_tvec.p, ht.size() * sizeof(double), cudaMemcpyDeviceToHost, s));
	LCD_CUDA(e, cudaMemcpyAsync(hn.data(), e->v_ninl.p, n_sets * sizeof(int), cudaMemcpyDeviceToHost, s));
	LCD_CUDA(e, cudaMemcpyAsync(hit.data(), e->v_iters.p, n_sets * sizeof(int), cudaMemcpyDeviceToHost, s));
	if (inliers_out) LCD_CUDA(e, cudaMemcpyAsync(inliers_out, e->v_inl.p, rows * sizeof(int), cudaMemcpyDeviceToHost, s));
	LCD_CUDA(e, cudaStreamSynchronize(s));
	for (int i = 0; i < n_sets; ++i)
	{
		// a model was found (the kernel zeroes the pose first and writes the final model last): rvec / tvec of the (refined) model;
		// otherwise the caller's values stay, as when cv3::solvePnPRansac returns false (solvepnp.cpp:183-192)
		bool found = hn[i] > 0;
		for (int k = 0; k < 3; ++k) found = found || hr[3 * i + k] != 0.0 || ht[3 * i + k] != 0.0;
		if (found)
		{
			for (int k = 0; k < 3; ++k)
			{
				rvec[3 * i + k] = hr[3 * i + k];
				tvec[3 * i + k] = ht[3 * i + k];
			}
		}
		if (n_inliers_out) n_inliers_out[i] = hn[i];
		if (iterations_run_out) iterations_run_out[i] = hit[i];
	}
	return LCD_OK;
}

int lcd_pnp_ransac(lcd_engine * e, const float * object_points, const float * image_points, int n, const double K[9], const double * dist_coeffs,
                   int n_dist, double rvec[3], double tvec[3], int use_extrinsic_guess, int iterations, float reproj_error, int min_inliers,
                   int flags, int refine_iterations, float refine_sigma, int * inliers_out, int * n_inliers_out)
{
	if (!e) return LCD_ERR_INVALID;
	if (n <= 0)
	{
		if (n_inliers_out) *n_inliers_out = 0;
		return LCD_OK;
	}
	return lcd_pnp_ransac_batch(e, 1, n, object_points, image_points, &n, K, dist_coeffs, n_dist, rvec, tvec, use_extrinsic_guess, iterations,
	                            reproj_error, min_inliers, flags, refine_iterations, refine_sigma, inliers_out, n_inliers_out, nullptr);
}

// ---- EpipolarGeometry::check of explicit signature pairs ------------------------------------------------
} // extern "C"
static int launch_epipolar(lcd_engine * e, int n_pairs, EpiArgs & a, const lcd_epipolar_params * p, cudaStream_t s)
{
	const size_t smem = epi_smem_bytes(std::max(a.cap_a, a.cap_b));
	LCD_TRY(fit_smem(e, reinterpret_cast<const void *>(epipolar_check_kernel), smem, std::max(a.cap_a, a.cap_b)));
	LCD_CUDA(e, e->ep_res.reserve(static_cast<size_t>(n_pairs) * 8, 0, false, s));
	LCD_CUDA(e, e->ep_F.reserve(static_cast<size_t>(n_pairs) * 9, 0, false, s));
	a.match_count_min = p->match_count_min;
	// findFundamentalMat's own resets of a threshold <= 0 and of a confidence outside (DBL_EPSILON, 1 - DBL_EPSILON)
	a.thr = p->ransac_param1 <= 0 ? 3. : p->ransac_param1;
	a.conf = (p->ransac_param2 < 2.220446049250313e-16 || p->ransac_param2 > 1 - 2.220446049250313e-16) ? 0.99 : p->ransac_param2;
	a.res = e->ep_res.p;
	a.F = e->ep_F.p;
	prof_mark(e, LCD_PROF_EPIPOLAR, s);
	epipolar_check_kernel<<<n_pairs, kEpiThreads, smem, s>>>(a);
	prof_mark(e, LCD_PROF_EPIPOLAR, s);
	LCD_CHECK_LAUNCH(e);
	return LCD_OK;
}

static void epipolar_results(int n, const int * hr, const double * hF, lcd_epipolar_result * out)
{
	for (int i = 0; i < n; ++i)
	{
		const int * r = hr + static_cast<size_t>(i) * 8;
		lcd_epipolar_result & o = out[i];
		o.checked = r[0];
		o.ok = r[1];
		o.n_pairs = r[2];
		o.n_inliers = r[3];
		o.method = r[4];
		o.found = r[5];
		o.iterations_run = r[6];
		o.raised = r[7];
		for (int k = 0; k < 9; ++k) o.F[k] = hF[static_cast<size_t>(i) * 9 + k];
	}
}

// lcd_proximity_result records of n frames from their device records and registrations [frame][mp]
static void proximity_results(int n, int mp, const ProxRecord * rec, const PackedVerifyResult * res, lcd_proximity_result * out)
{
	for (int f = 0; f < n; ++f)
	{
		const ProxRecord & r = rec[f];
		lcd_proximity_result & o = out[f];
		memset(&o, 0, sizeof(o));
		o.status = r.status;
		o.n_nearest = r.n_nearest;
		o.n_paths = r.n_paths;
		o.n_attempts = r.n_attempts;
		o.suppressed_id = r.suppressed;
		for (int j = 0; j < r.n_attempts; ++j)
		{
			lcd_proximity_path & p = o.paths[j];
			p.likelihood = r.path[j].likelihood;
			p.id = r.path[j].id;
			p.distance = r.path[j].distance;
			p.candidate_id = r.path[j].candidate;
			p.accepted = r.accepted[j];
			p.link_type = r.link_type[j];
			memcpy(&p.result, &res[static_cast<size_t>(f) * mp + j], sizeof(lcd_verify_result));
		}
	}
}
extern "C" {
int lcd_epipolar_check_batch(lcd_engine * e, int n_pairs, int cap, const int * ids_a, const float * uv_a, const int * n_a, const int * ids_b,
                             const float * uv_b, const int * n_b, const lcd_epipolar_params * p, lcd_epipolar_result * out, uint8_t * status_out)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(set_device(e));
	if (n_pairs <= 0 || cap <= 0 || !ids_a || !uv_a || !n_a || !ids_b || !uv_b || !n_b || !p || !out)
		LCD_FAIL(e, LCD_ERR_INVALID, "null or empty epipolar input");
	if (cap > kMaxFrameQueries) LCD_FAIL(e, LCD_ERR_CAPACITY, "at most %d words per signature", kMaxFrameQueries);
	for (int i = 0; i < n_pairs; ++i)
		if (n_a[i] < 0 || n_a[i] > cap || n_b[i] < 0 || n_b[i] > cap)
			LCD_FAIL(e, LCD_ERR_INVALID, "pair %d has %d / %d words (cap %d)", i, n_a[i], n_b[i], cap);
	cudaStream_t s = e->stream;
	const size_t rows = static_cast<size_t>(n_pairs) * cap;
	LCD_CUDA(e, e->ep_ids_a.reserve(rows, 0, false, s));
	LCD_CUDA(e, e->ep_ids_b.reserve(rows, 0, false, s));
	LCD_CUDA(e, e->ep_uv_a.reserve(rows * 2, 0, false, s));
	LCD_CUDA(e, e->ep_uv_b.reserve(rows * 2, 0, false, s));
	LCD_CUDA(e, e->ep_n.reserve(static_cast<size_t>(n_pairs) * 2, 0, false, s));
	if (status_out) LCD_CUDA(e, e->ep_status.reserve(rows, 0, false, s));
	LCD_CUDA(e, cudaMemcpyAsync(e->ep_ids_a.p, ids_a, rows * sizeof(int), cudaMemcpyHostToDevice, s));
	LCD_CUDA(e, cudaMemcpyAsync(e->ep_ids_b.p, ids_b, rows * sizeof(int), cudaMemcpyHostToDevice, s));
	LCD_CUDA(e, cudaMemcpyAsync(e->ep_uv_a.p, uv_a, rows * 2 * sizeof(float), cudaMemcpyHostToDevice, s));
	LCD_CUDA(e, cudaMemcpyAsync(e->ep_uv_b.p, uv_b, rows * 2 * sizeof(float), cudaMemcpyHostToDevice, s));
	LCD_CUDA(e, cudaMemcpyAsync(e->ep_n.p, n_a, n_pairs * sizeof(int), cudaMemcpyHostToDevice, s));
	LCD_CUDA(e, cudaMemcpyAsync(e->ep_n.p + n_pairs, n_b, n_pairs * sizeof(int), cudaMemcpyHostToDevice, s));
	EpiArgs a{};
	a.ids_a = e->ep_ids_a.p;
	a.uv_a = e->ep_uv_a.p;
	a.n_a = e->ep_n.p;
	a.ids_b = e->ep_ids_b.p;
	a.uv_b = e->ep_uv_b.p;
	a.n_b = e->ep_n.p + n_pairs;
	a.cap_a = a.cap_b = cap;
	a.status = status_out ? e->ep_status.p : nullptr;
	a.status_cap = cap;
	LCD_TRY(launch_epipolar(e, n_pairs, a, p, s));
	std::vector<int> hr(static_cast<size_t>(n_pairs) * 8);
	std::vector<double> hF(static_cast<size_t>(n_pairs) * 9);
	LCD_CUDA(e, cudaMemcpyAsync(hr.data(), e->ep_res.p, hr.size() * sizeof(int), cudaMemcpyDeviceToHost, s));
	LCD_CUDA(e, cudaMemcpyAsync(hF.data(), e->ep_F.p, hF.size() * sizeof(double), cudaMemcpyDeviceToHost, s));
	if (status_out) LCD_CUDA(e, cudaMemcpyAsync(status_out, e->ep_status.p, rows, cudaMemcpyDeviceToHost, s));
	LCD_CUDA(e, cudaStreamSynchronize(s));
	epipolar_results(n_pairs, hr.data(), hF.data(), out);
	return LCD_OK;
}

int lcd_sig_words_add_batch(lcd_engine * e, const int * sig_ids, int n_sigs, int cap, const int * word_ids, const float * uv, const int * n)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(set_device(e));
	if (n_sigs <= 0 || cap <= 0 || !sig_ids || !word_ids || !uv || !n) LCD_FAIL(e, LCD_ERR_INVALID, "null or empty word store input");
	if (cap > kMaxFrameQueries) LCD_FAIL(e, LCD_ERR_CAPACITY, "at most %d words per signature", kMaxFrameQueries);
	for (int i = 0; i < n_sigs; ++i)
		if (n[i] < 0 || n[i] > cap) LCD_FAIL(e, LCD_ERR_INVALID, "signature %d has %d words (cap %d)", sig_ids[i], n[i], cap);
	cudaStream_t s = e->stream;
	const size_t prev_rows = static_cast<size_t>(e->ws_map.slots);
	std::vector<int> slots;
	if (!e->ws_map.assign(sig_ids, n_sigs, slots)) LCD_FAIL(e, LCD_ERR_INVALID, "signature ids must be > 0");
	const size_t rows = static_cast<size_t>(e->ws_map.slots), wc = std::max(e->ws_cap, cap);
	if (cap > e->ws_cap && prev_rows > 0)
	{
		// wider rows: re-lay the stored rows out at the new stride
		DevBuf<int> ids2;
		DevBuf<float> uv2;
		LCD_CUDA(e, ids2.reserve(rows * wc, 0, false, s));
		LCD_CUDA(e, uv2.reserve(rows * wc * 2, 0, false, s));
		// kernels on any stream may still read the rows being copied and freed
		LCD_CUDA(e, cudaDeviceSynchronize());
		LCD_CUDA(e, cudaMemcpy2DAsync(ids2.p, wc * sizeof(int), e->ws_ids.p, e->ws_cap * sizeof(int), e->ws_cap * sizeof(int), prev_rows,
		                              cudaMemcpyDeviceToDevice, s));
		LCD_CUDA(e, cudaMemcpy2DAsync(uv2.p, wc * 2 * sizeof(float), e->ws_uv.p, e->ws_cap * 2 * sizeof(float), e->ws_cap * 2 * sizeof(float),
		                              prev_rows, cudaMemcpyDeviceToDevice, s));
		LCD_CUDA(e, cudaStreamSynchronize(s));
		e->ws_ids.swap(ids2);
		e->ws_uv.swap(uv2);
	}
	e->ws_cap = static_cast<int>(wc);
	LCD_CUDA(e, e->ws_ids.reserve(rows * wc, e->ws_ids.cap, false, s));
	LCD_CUDA(e, e->ws_uv.reserve(rows * wc * 2, e->ws_uv.cap, false, s));
	LCD_CUDA(e, e->ws_n.reserve(rows, e->ws_n.cap, false, s));
	for (int i = 0; i < n_sigs; ++i)
	{
		const size_t r = slots[i];
		LCD_CUDA(e, cudaMemcpyAsync(e->ws_ids.p + r * wc, word_ids + static_cast<size_t>(i) * cap, n[i] * sizeof(int), cudaMemcpyHostToDevice, s));
		LCD_CUDA(e, cudaMemcpyAsync(e->ws_uv.p + r * wc * 2, uv + static_cast<size_t>(i) * cap * 2, n[i] * 2 * sizeof(float), cudaMemcpyHostToDevice, s));
		LCD_CUDA(e, cudaMemcpyAsync(e->ws_n.p + r, n + i, sizeof(int), cudaMemcpyHostToDevice, s));
	}
	LCD_CUDA(e, e->ws_map.upload(s));
	LCD_CUDA(e, cudaStreamSynchronize(s));
	return LCD_OK;
}

int lcd_sig_words_remove(lcd_engine * e, int sig_id)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(set_device(e));
	if (e->ws_map.release(sig_id) < 0) return LCD_OK;
	LCD_CUDA(e, e->ws_map.upload(sig_id, e->stream));
	LCD_CUDA(e, cudaStreamSynchronize(e->stream));
	return LCD_OK;
}

int lcd_sig_words_count(const lcd_engine * e) { return e ? e->ws_map.count() : 0; }

} // extern "C"
// VhEp/Enabled on the last decision (checked by the callers): the frames' words d_word_ids[n_frames][nq] against the word store
static int epipolar_decide(lcd_engine * e, const int * d_word_ids, const float * d_uv, const int * d_n_per_frame, int n_frames, int nq_per_frame,
                           const lcd_epipolar_params * p, cudaStream_t s)
{
	LCD_CUDA(e, e->ep_slot.reserve(n_frames, 0, false, s));
	LCD_CUDA(e, e->ep_skip.reserve(n_frames, 0, false, s));
	LCD_CUDA(e, e->ws_n.reserve(1, 0, true, s)); // an empty store: every hypothesis is a signature without words
	LCD_CUDA(e, e->ws_ids.reserve(1, 0, false, s));
	LCD_CUDA(e, e->ws_uv.reserve(2, 0, false, s));
	epi_decide_prep_kernel<<<(n_frames + 127) / 128, 128, 0, s>>>(n_frames, e->dc_dec.p, e->ws_map.d.p, e->ws_map.n_ids, e->ep_slot.p,
	                                                                 e->ep_skip.p);
	LCD_CHECK_LAUNCH(e);
	EpiArgs a{};
	a.ids_a = d_word_ids;
	a.uv_a = d_uv;
	a.n_a = d_n_per_frame;
	a.ids_b = e->ws_ids.p;
	a.uv_b = e->ws_uv.p;
	a.n_b = e->ws_n.p;
	a.slot_b = e->ep_slot.p;
	a.skip = e->ep_skip.p;
	a.cap_a = nq_per_frame;
	a.cap_b = std::max(e->ws_cap, 1);
	LCD_TRY(launch_epipolar(e, n_frames, a, p, s));
	epi_decide_apply_kernel<<<(n_frames + 127) / 128, 128, 0, s>>>(n_frames, e->ep_res.p, e->dc_dec.p, e->dc_hyp_valid ? e->d_hyp_id.p : nullptr,
	                                                                  e->dc_hyp_valid ? e->d_hyp_slot.p : nullptr);
	LCD_CHECK_LAUNCH(e);
	e->ep_last_frames = n_frames;
	return LCD_OK;
}
extern "C" {

int lcd_decide_epipolar_dev(lcd_engine * e, const int * d_word_ids, const float * d_uv, const int * d_n_per_frame, int n_frames, int nq_per_frame,
                            const lcd_epipolar_params * p, void * stream)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(set_device(e));
	if (e->dc_last_frames == 0) LCD_FAIL(e, LCD_ERR_STATE, "no decision to check: run lcd_decide_batch_dev first");
	if (!d_word_ids || !d_uv || !d_n_per_frame || !p) LCD_FAIL(e, LCD_ERR_INVALID, "null epipolar input");
	if (n_frames != e->dc_last_frames) LCD_FAIL(e, LCD_ERR_INVALID, "the last decision has %d frames, not %d", e->dc_last_frames, n_frames);
	if (nq_per_frame <= 0) LCD_FAIL(e, LCD_ERR_INVALID, "nq_per_frame %d", nq_per_frame);
	if (nq_per_frame > kMaxFrameQueries) LCD_FAIL(e, LCD_ERR_CAPACITY, "at most %d words per frame", kMaxFrameQueries);
	cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : e->stream;
	return epipolar_decide(e, d_word_ids, d_uv, d_n_per_frame, n_frames, nq_per_frame, p, s);
}

int lcd_epipolar_fetch(lcd_engine * e, int n_frames, lcd_epipolar_result * out)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(set_device(e));
	if (!out || n_frames <= 0) LCD_FAIL(e, LCD_ERR_INVALID, "null output");
	if (e->ep_last_frames == 0) LCD_FAIL(e, LCD_ERR_STATE, "no epipolar decision: run lcd_decide_epipolar_dev first");
	if (n_frames > e->ep_last_frames) LCD_FAIL(e, LCD_ERR_INVALID, "the last epipolar decision has %d frames", e->ep_last_frames);
	std::vector<int> hr(static_cast<size_t>(n_frames) * 8);
	std::vector<double> hF(static_cast<size_t>(n_frames) * 9);
	LCD_CUDA(e, cudaDeviceSynchronize());
	LCD_CUDA(e, cudaMemcpy(hr.data(), e->ep_res.p, hr.size() * sizeof(int), cudaMemcpyDeviceToHost));
	LCD_CUDA(e, cudaMemcpy(hF.data(), e->ep_F.p, hF.size() * sizeof(double), cudaMemcpyDeviceToHost));
	epipolar_results(n_frames, hr.data(), hF.data(), out);
	return LCD_OK;
}

// ---- brute-force matching of two descriptor sets: cv::BFMatcher ----------------------------------------
} // extern "C"
template <int NW, bool F32>
static int launch_bf(lcd_engine * e, int n_pairs, int cap, const uint32_t * A, const int * nA, const uint32_t * B, const int * nB, ulonglong2 * keys,
                     cudaStream_t s)
{
	dim3 grid((cap + kBfThreads - 1) / kBfThreads, n_pairs);
	prof_mark(e, LCD_PROF_MATCH, s);
	if constexpr (F32 && NW == 256) bf_knn2_l2_chunked_kernel<NW><<<grid, kBfThreads, 0, s>>>(A, nA, B, nB, cap, keys);
	else bf_knn2_kernel<NW, F32><<<grid, kBfThreads, 0, s>>>(A, nA, B, nB, cap, keys);
	prof_mark(e, LCD_PROF_MATCH, s);
	LCD_CHECK_LAUNCH(e);
	return LCD_OK;
}

static int launch_bf_any(lcd_engine * e, int n_pairs, int cap, const uint32_t * A, const int * nA, const uint32_t * B, const int * nB,
                         ulonglong2 * keys, cudaStream_t s)
{
	if (e->f32)
		return e->nw == 64    ? launch_bf<64, true>(e, n_pairs, cap, A, nA, B, nB, keys, s)
		       : e->nw == 128 ? launch_bf<128, true>(e, n_pairs, cap, A, nA, B, nB, keys, s)
		                      : launch_bf<256, true>(e, n_pairs, cap, A, nA, B, nB, keys, s);
	switch (e->nw)
	{
	case 4: return launch_bf<4, false>(e, n_pairs, cap, A, nA, B, nB, keys, s);
	case 8: return launch_bf<8, false>(e, n_pairs, cap, A, nA, B, nB, keys, s);
	case 16: return launch_bf<16, false>(e, n_pairs, cap, A, nA, B, nB, keys, s);
	default: LCD_FAIL(e, LCD_ERR_INVALID, "unsupported descriptor size");
	}
}

extern "C" {
int lcd_match_bf(lcd_engine * e, int n_pairs, int cap, const void * desc_query, const int * n_query, const void * desc_train, const int * n_train,
                 int mode, int * idx1, float * dist1, int * idx2, float * dist2)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(set_device(e));
	LCD_TRY(check_verify_args(e, n_pairs, cap, desc_query, desc_train, n_query, n_train));
	if (mode != LCD_MATCH_KNN2 && mode != LCD_MATCH_CROSSCHECK) LCD_FAIL(e, LCD_ERR_INVALID, "mode must be LCD_MATCH_KNN2 or LCD_MATCH_CROSSCHECK");
	if (!idx1 || !dist1 || (mode == LCD_MATCH_KNN2 && (!idx2 || !dist2))) LCD_FAIL(e, LCD_ERR_INVALID, "null output");
	cudaStream_t s = e->stream;
	const size_t rows = static_cast<size_t>(n_pairs) * cap;
	// FROM buffers hold the train side, TO buffers the query side (cv::BFMatcher::match(queryDescriptors = TO, trainDescriptors = FROM))
	PairSource staged;
	LCD_TRY(verify_upload(e, n_pairs, cap, desc_train, nullptr, n_train, desc_query, nullptr, nullptr, n_query, s, staged));
	LCD_CUDA(e, e->bf_keys_a.reserve(rows, 0, false, s));
	LCD_CUDA(e, e->d_i1.reserve(rows, 0, false, s));
	LCD_CUDA(e, e->d_f1.reserve(rows, 0, false, s));
	const int nb = static_cast<int>((rows + 255) / 256);
	if (mode == LCD_MATCH_KNN2)
	{
		LCD_TRY(launch_bf_any(e, n_pairs, cap, e->v_dt.p, e->v_nt.p, e->v_df.p, e->v_nf.p, e->bf_keys_a.p, s));
		LCD_CUDA(e, e->d_i2.reserve(rows, 0, false, s));
		LCD_CUDA(e, e->d_f2.reserve(rows, 0, false, s));
		const unsigned long long * k = reinterpret_cast<const unsigned long long *>(e->bf_keys_a.p);
		if (e->f32)
		{
			bf_decode_kernel<true><<<nb, 256, 0, s>>>(k, 2, 0, static_cast<int>(rows), e->d_i1.p, e->d_f1.p);
			bf_decode_kernel<true><<<nb, 256, 0, s>>>(k, 2, 1, static_cast<int>(rows), e->d_i2.p, e->d_f2.p);
		}
		else
		{
			bf_decode_kernel<false><<<nb, 256, 0, s>>>(k, 2, 0, static_cast<int>(rows), e->d_i1.p, e->d_f1.p);
			bf_decode_kernel<false><<<nb, 256, 0, s>>>(k, 2, 1, static_cast<int>(rows), e->d_i2.p, e->d_f2.p);
		}
		LCD_CHECK_LAUNCH(e);
		++e->launches;
		LCD_CUDA(e, cudaMemcpyAsync(idx2, e->d_i2.p, rows * sizeof(int), cudaMemcpyDeviceToHost, s));
		LCD_CUDA(e, cudaMemcpyAsync(dist2, e->d_f2.p, rows * sizeof(float), cudaMemcpyDeviceToHost, s));
	}
	else
	{
		// nearest train row of every query, nearest query of every train row, then the mutual test
		LCD_TRY(launch_bf_any(e, n_pairs, cap, e->v_dt.p, e->v_nt.p, e->v_df.p, e->v_nf.p, e->bf_keys_a.p, s));
		LCD_CUDA(e, e->bf_keys_b.reserve(rows, 0, false, s));
		LCD_TRY(launch_bf_any(e, n_pairs, cap, e->v_df.p, e->v_nf.p, e->v_dt.p, e->v_nt.p, e->bf_keys_b.p, s));
		LCD_CUDA(e, e->bf_best.reserve(rows, 0, false, s));
		bf_cross_kernel<<<dim3((cap + 255) / 256, n_pairs), 256, 0, s>>>(e->bf_keys_a.p, e->bf_keys_b.p, e->v_nt.p, cap, e->bf_best.p);
		LCD_CHECK_LAUNCH(e);
		if (e->f32) bf_decode_kernel<true><<<nb, 256, 0, s>>>(e->bf_best.p, 1, 0, static_cast<int>(rows), e->d_i1.p, e->d_f1.p);
		else bf_decode_kernel<false><<<nb, 256, 0, s>>>(e->bf_best.p, 1, 0, static_cast<int>(rows), e->d_i1.p, e->d_f1.p);
		LCD_CHECK_LAUNCH(e);
	}
	LCD_CUDA(e, cudaMemcpyAsync(idx1, e->d_i1.p, rows * sizeof(int), cudaMemcpyDeviceToHost, s));
	LCD_CUDA(e, cudaMemcpyAsync(dist1, e->d_f1.p, rows * sizeof(float), cudaMemcpyDeviceToHost, s));
	LCD_CUDA(e, cudaStreamSynchronize(s));
	if (mode == LCD_MATCH_KNN2)
	{
		// rows past a pair's query count were not written by the kernel: report them as "no match"
		for (int p = 0; p < n_pairs; ++p)
			for (int i = std::max(0, std::min(n_query[p], cap)); i < cap; ++i)
			{
				const size_t r = static_cast<size_t>(p) * cap + i;
				idx1[r] = idx2[r] = -1;
				dist1[r] = dist2[r] = -1.0f;
			}
	}
	return LCD_OK;
}

// ---- signature store + fused query -------------------------------------------------------------
int lcd_sig_count(const lcd_engine * e) { return e ? e->st_map.count() : 0; }
int lcd_sig_slots(const lcd_engine * e) { return e ? e->st_map.slots : 0; }

int lcd_sig_add_batch(lcd_engine * e, const int * sig_ids, int n_sigs, int cap, const void * desc, const float * xyz, const int * n)
{
	if (!e) return LCD_ERR_INVALID;
	if (n_sigs <= 0) return LCD_OK;
	if (!sig_ids || !desc || !xyz || !n || cap <= 0) LCD_FAIL(e, LCD_ERR_INVALID, "null signature data");
	if (cap > kMaxFrameQueries) LCD_FAIL(e, LCD_ERR_CAPACITY, "at most %d features per signature", kMaxFrameQueries);
	if (e->st_cap != 0 && cap != e->st_cap) LCD_FAIL(e, LCD_ERR_INVALID, "signature store was created with %d rows per signature, got %d", e->st_cap, cap);
	LCD_TRY(set_device(e));
	cudaStream_t s = e->stream;
	const size_t prev_slots = static_cast<size_t>(e->st_map.slots);
	std::vector<int> slots;
	if (!e->st_map.assign(sig_ids, n_sigs, slots)) LCD_FAIL(e, LCD_ERR_INVALID, "signature id must be positive");
	e->st_cap = cap;
	const size_t nst = static_cast<size_t>(e->st_map.slots), drow = static_cast<size_t>(cap) * e->nw, xrow = static_cast<size_t>(cap) * 3;
	LCD_CUDA(e, e->st_desc.reserve(nst * drow, prev_slots * drow, false, s));
	LCD_CUDA(e, e->st_xyz.reserve(nst * xrow, prev_slots * xrow, false, s));
	LCD_CUDA(e, e->st_n.reserve(nst, prev_slots, true, s));
	LCD_CUDA(e, e->st_kof.reserve(nst * cap, prev_slots * cap, false, s));
	LCD_CUDA(e, e->st_creator.reserve(nst * cap, prev_slots * cap, false, s));
	LCD_CUDA(e, e->st_ftag.reserve(nst, prev_slots, false, s));
	// a written row's cached FROM dictionary is stale (0xFF..: nf = -1 matches no call)
	const auto put = [&](size_t slot, size_t i, size_t k) {
		const uint32_t * src = static_cast<const uint32_t *>(desc) + i * drow;
		cudaError_t err = cudaMemcpyAsync(e->st_desc.p + slot * drow, src, k * drow * sizeof(uint32_t), cudaMemcpyHostToDevice, s);
		if (err == cudaSuccess) err = cudaMemcpyAsync(e->st_xyz.p + slot * xrow, xyz + i * xrow, k * xrow * sizeof(float), cudaMemcpyHostToDevice, s);
		if (err == cudaSuccess) err = cudaMemcpyAsync(e->st_n.p + slot, n + i, k * sizeof(int), cudaMemcpyHostToDevice, s);
		if (err == cudaSuccess) err = cudaMemsetAsync(e->st_ftag.p + slot, 0xFF, k * sizeof(FromDictTag), s);
		return err;
	};
	LCD_CUDA(e, write_rows(slots, put));
	LCD_CUDA(e, e->st_map.upload(s));
	LCD_CUDA(e, cudaStreamSynchronize(s));
	return LCD_OK;
}

int lcd_sig_remove(lcd_engine * e, int sig_id)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(set_device(e));
	const int slot = e->st_map.release(sig_id);
	if (slot < 0) return LCD_OK;
	LCD_CUDA(e, e->st_map.upload(sig_id, e->stream));
	LCD_CUDA(e, cudaMemsetAsync(e->st_n.p + slot, 0, sizeof(int), e->stream));
	LCD_CUDA(e, cudaMemsetAsync(e->st_ftag.p + slot, 0xFF, sizeof(FromDictTag), e->stream));
	LCD_CUDA(e, cudaStreamSynchronize(e->stream));
	return LCD_OK;
}

// d_nq_frame: descriptors of each frame (nullptr: nq each); d_xyz_to: the frames' 3-D points (words3B) or nullptr
static int verify_top_dev(lcd_engine * e, const uint32_t * d_q, const float * d_uv, int n_frames, int nq, const float * d_like,
                          const int * d_sig_ids, int ns, const lcd_verify_params * vp, cudaStream_t s, const int * d_nq_frame, const float * d_xyz_to)
{
	LCD_TRY(check_verify_params(e, vp, true));
	LCD_CUDA(e, e->d_hyp_id.reserve(n_frames, 0, false, s));
	LCD_CUDA(e, e->d_hyp_slot.reserve(n_frames, 0, false, s));
	e->dc_hyp_valid = false; // the arg-max replaces the hypotheses of the last decision
	argmax_hypothesis_kernel<<<n_frames, 256, 0, s>>>(d_like, ns, d_sig_ids, e->st_map.d.p, e->st_map.n_ids, e->d_hyp_id.p, e->d_hyp_slot.p);
	LCD_CHECK_LAUNCH(e);
	const PairSource src{{e->st_desc.p, e->st_xyz.p, e->st_n.p, e->d_hyp_slot.p, e->st_cap}, {d_q, d_uv, d_xyz_to, d_nq_frame, nq, nq, nullptr}};
	return register_pairs(e, src, n_frames, std::max(e->st_cap, nq), vp, s);
}

static int process_dev(lcd_engine * e, const uint32_t * d_q, const float * d_uv, int n_frames, int nq, int incremental, float nndr, int cmp_new,
                       const int * d_sig_ids, int ns, int n_total, const lcd_verify_params * vp, int * d_words, float * d_like, cudaStream_t s)
{
	LCD_TRY(check_verify_params(e, vp, true));
	if (!d_sig_ids || ns <= 0) LCD_FAIL(e, LCD_ERR_INVALID, "ids list is empty");
	if (!d_like)
	{
		LCD_CUDA(e, e->d_like.reserve(static_cast<size_t>(n_frames) * ns, 0, false, s));
		d_like = e->d_like.p;
	}
	LCD_TRY(localize_dev(e, d_q, n_frames, nq, incremental, nndr, cmp_new, d_sig_ids, ns, n_total, d_words, d_like, s));
	return verify_top_dev(e, d_q, d_uv, n_frames, nq, d_like, d_sig_ids, ns, vp, s, nullptr, nullptr);
}

int lcd_process_batch_dev(lcd_engine * e, const void * d_queries, const float * d_uv, int n_frames, int nq_per_frame, int incremental, float nndr,
                          int new_words_compared_together, const int * d_sig_ids, int ns, int n_total, const lcd_verify_params * vp,
                          int * d_word_ids_out, float * d_likelihood_out, void * stream)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(set_device(e));
	if (!d_queries || !d_uv || n_frames <= 0) LCD_FAIL(e, LCD_ERR_INVALID, "Descriptors size is null!");
	if (nq_per_frame <= 0 || nq_per_frame > kMaxFrameQueries) LCD_FAIL(e, LCD_ERR_CAPACITY, "1..%d descriptors per frame", kMaxFrameQueries);
	LCD_TRY(check_n_total(e, n_total));
	cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : e->stream;
	return process_dev(e, static_cast<const uint32_t *>(d_queries), d_uv, n_frames, nq_per_frame, incremental, nndr, new_words_compared_together,
	                   d_sig_ids, ns, n_total, vp, d_word_ids_out, d_likelihood_out, s);
}

// images -> detect -> quantise -> score -> verify, all on device buffers
static int process_frames_dev(lcd_engine * e, int n_frames, const uint8_t * d_images, int width, int height, int channels, const void * d_depth,
                              int depth_type, const lcd_orb_params * op, int incremental, float nndr, int cmp_new, const int * d_sig_ids, int ns,
                              int n_total, const lcd_verify_params * vp, int * d_words, float * d_like, cudaStream_t s)
{
	if (!op) LCD_FAIL(e, LCD_ERR_INVALID, "null ORB parameters");
	const int cap = op->n_features;
	LCD_TRY(frame_front_end(e, n_frames, cap, e->o_kp, e->o_desc, e->o_xyz, &e->o_uv, e->o_n, s));
	LCD_TRY(orb_run(e, n_frames, d_images, width, height, channels, d_depth, depth_type, op, cap, e->o_kp.p, e->o_desc.p, e->o_xyz.p, e->o_uv.p,
	                e->o_n.p, s));
	if (!d_like)
	{
		LCD_CUDA(e, e->d_like.reserve(static_cast<size_t>(n_frames) * ns, 0, false, s));
		d_like = e->d_like.p;
	}
	const uint32_t * d_q = reinterpret_cast<const uint32_t *>(e->o_desc.p);
	if (limit_active(e))
	{
		// Memory::createSignature's split: quantise the strongest rows only, verify with every detected row
		const int k = limit_rows(e, cap);
		LCD_TRY(limit_to_engine(e, n_frames, cap, e->o_kp.p, e->o_n.p, d_q, s));
		LCD_TRY(localize_dev(e, e->ql_desc.p, n_frames, k, incremental, nndr, cmp_new, d_sig_ids, ns, n_total, d_words ? e->ql_words.p : nullptr, d_like,
		                     s, e->ql_n.p));
		if (d_words) LCD_TRY(launch_expand(e, n_frames, cap, k, e->o_n.p, e->ql_index.p, e->ql_n.p, e->ql_words.p, d_words, s));
	}
	else
		LCD_TRY(localize_dev(e, d_q, n_frames, cap, incremental, nndr, cmp_new, d_sig_ids, ns, n_total, d_words, d_like, s, e->o_n.p));
	if (vp) LCD_TRY(verify_top_dev(e, d_q, e->o_uv.p, n_frames, cap, d_like, d_sig_ids, ns, vp, s, e->o_n.p, e->o_xyz.p));
	return LCD_OK;
}

int lcd_process_frames_dev(lcd_engine * e, int n_frames, const uint8_t * d_images, int width, int height, int channels, const void * d_depth,
                           int depth_type, const lcd_orb_params * op, int incremental, float nndr, int new_words_compared_together,
                           const int * d_sig_ids, int ns, int n_total, const lcd_verify_params * vp, int * d_word_ids_out,
                           float * d_likelihood_out, void * stream)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(set_device(e));
	if (!d_images || n_frames <= 0) LCD_FAIL(e, LCD_ERR_INVALID, "null image");
	if (!d_sig_ids || ns <= 0) LCD_FAIL(e, LCD_ERR_INVALID, "ids list is empty");
	LCD_TRY(check_n_total(e, n_total));
	cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : e->stream;
	return process_frames_dev(e, n_frames, d_images, width, height, channels, d_depth, depth_type, op, incremental, nndr, new_words_compared_together,
	                          d_sig_ids, ns, n_total, vp, d_word_ids_out, d_likelihood_out, s);
}

// the host -> device stream of lcd_process_frames and lcd_process_frames_submit, and the event that orders it against the engine stream
static int copy_stream_ready(lcd_engine * e)
{
	if (e->copy_stream) return LCD_OK;
	LCD_CUDA(e, cudaStreamCreateWithFlags(&e->copy_stream, cudaStreamNonBlocking));
	LCD_CUDA(e, cudaEventCreateWithFlags(&e->copy_fence, cudaEventDisableTiming));
	return LCD_OK;
}

// the per-frame results of lcd_process_frames / _submit that the caller asked for, queued on s: keypoint counts, word ids ([frame][rows /
// n_frames]), likelihoods and, with verification, the hypotheses
static int download_frames(lcd_engine * e, int n_frames, size_t rows, int ns, const lcd_verify_params * vp, int * n_kp_out, int * word_ids_out,
                           float * likelihood_out, int * hypothesis_out, cudaStream_t s)
{
	if (n_kp_out) LCD_CUDA(e, cudaMemcpyAsync(n_kp_out, e->o_n.p, n_frames * sizeof(int), cudaMemcpyDeviceToHost, s));
	if (word_ids_out) LCD_CUDA(e, cudaMemcpyAsync(word_ids_out, e->d_word_ids.p, rows * sizeof(int), cudaMemcpyDeviceToHost, s));
	if (likelihood_out)
		LCD_CUDA(e, cudaMemcpyAsync(likelihood_out, e->d_like.p, static_cast<size_t>(n_frames) * ns * sizeof(float), cudaMemcpyDeviceToHost, s));
	if (vp && hypothesis_out) LCD_CUDA(e, cudaMemcpyAsync(hypothesis_out, e->d_hyp_id.p, n_frames * sizeof(int), cudaMemcpyDeviceToHost, s));
	return LCD_OK;
}

int lcd_process_frames(lcd_engine * e, int n_frames, const uint8_t * images, int width, int height, int channels, const void * depth, int depth_type,
                       const lcd_orb_params * op, int incremental, float nndr, int new_words_compared_together, const int * sig_ids, int ns,
                       int n_total, const lcd_verify_params * vp, int * n_kp_out, int * word_ids_out, float * likelihood_out, int * hypothesis_out,
                       lcd_verify_result * results)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(set_device(e));
	if (!images || n_frames <= 0 || width <= 0 || height <= 0) LCD_FAIL(e, LCD_ERR_INVALID, "null image");
	if (!sig_ids || ns <= 0) LCD_FAIL(e, LCD_ERR_INVALID, "ids list is empty");
	if (!op) LCD_FAIL(e, LCD_ERR_INVALID, "null ORB parameters");
	LCD_TRY(check_n_total(e, n_total));
	cudaStream_t s = e->stream;
	const int cap = op->n_features;
	const size_t rows = static_cast<size_t>(n_frames) * std::max(cap, 1);
	LCD_CUDA(e, e->d_sig_ids.reserve(ns, 0, false, s));
	LCD_CUDA(e, e->d_like.reserve(static_cast<size_t>(n_frames) * ns, 0, false, s));
	LCD_CUDA(e, e->d_word_ids.reserve(rows, 0, false, s));
	LCD_CUDA(e, cudaMemcpyAsync(e->d_sig_ids.p, sig_ids, ns * sizeof(int), cudaMemcpyHostToDevice, s));
	// the frames go up on the copy stream.  The device images may still be read by work queued on s (a previous call), so the copies
	// wait for it; s waits for the copies.  Each wait binds to the fence's latest record, so one event serves both directions.
	LCD_TRY(copy_stream_ready(e));
	LCD_CUDA(e, cudaEventRecord(e->copy_fence, s));
	LCD_CUDA(e, cudaStreamWaitEvent(e->copy_stream, e->copy_fence, 0));
	LCD_TRY(upload_frames(e, n_frames, width, height, channels, images, depth, depth_type, e->o_img, e->o_depth, e->copy_stream));
	LCD_CUDA(e, cudaEventRecord(e->copy_fence, e->copy_stream));
	LCD_CUDA(e, cudaStreamWaitEvent(s, e->copy_fence, 0));
	LCD_TRY(process_frames_dev(e, n_frames, e->o_img.p, width, height, channels, depth_type != LCD_DEPTH_NONE ? e->o_depth.p : nullptr, depth_type, op,
	                           incremental, nndr, new_words_compared_together, e->d_sig_ids.p, ns, n_total, vp, e->d_word_ids.p, e->d_like.p, s));
	LCD_TRY(download_frames(e, n_frames, rows, ns, vp, n_kp_out, word_ids_out, likelihood_out, hypothesis_out, s));
	LCD_CUDA(e, e->h_overflow.reserve(1));
	LCD_CUDA(e, cudaMemcpyAsync(e->h_overflow.p, e->o_overflow.p, sizeof(int), cudaMemcpyDeviceToHost, s));
	if (vp && results) LCD_TRY(verify_download(e, n_frames, 0, results, nullptr, nullptr, s));
	LCD_CUDA(e, cudaStreamSynchronize(s));
	return overflow_report(e, *e->h_overflow.p, e->detector);
}

// ---- pipelined host path: two batches in flight ------------------------------------------------------------
int lcd_process_frames_submit(lcd_engine * e, int n_frames, const uint8_t * images, int width, int height, int channels, const void * depth,
                              int depth_type, const lcd_orb_params * op, int incremental, float nndr, int new_words_compared_together,
                              const int * sig_ids, int ns, int n_total, const lcd_verify_params * vp, int * n_kp_out, int * word_ids_out,
                              float * likelihood_out, int * hypothesis_out, lcd_verify_result * results)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(set_device(e));
	if (!images || n_frames <= 0 || width <= 0 || height <= 0) LCD_FAIL(e, LCD_ERR_INVALID, "null image");
	if (!sig_ids || ns <= 0) LCD_FAIL(e, LCD_ERR_INVALID, "ids list is empty");
	if (!op) LCD_FAIL(e, LCD_ERR_INVALID, "null ORB parameters");
	if (e->flights_busy >= 2) LCD_FAIL(e, LCD_ERR_INVALID, "two batches are already in flight: call lcd_process_frames_wait first");
	LCD_TRY(check_n_total(e, n_total));
	cudaStream_t s = e->stream;
	const int slot = (e->flight_head + e->flights_busy) & 1;
	lcd_engine::Flight & f = e->flights[slot];
	LCD_TRY(copy_stream_ready(e));
	if (!f.uploaded)
	{
		LCD_CUDA(e, cudaEventCreateWithFlags(&f.uploaded, cudaEventDisableTiming));
		LCD_CUDA(e, cudaEventCreateWithFlags(&f.done, cudaEventDisableTiming));
	}
	// upload on the copy stream: the slot's previous batch was waited for, so its staging buffers are free
	static const int dbg_tl = env_int("LCD_DEBUG_TIMELINE", 0); // diagnostics: print each batch's upload / compute window at _wait
	if (dbg_tl && !f.t_h0)
	{
		cudaEventCreate(&f.t_h0);
		cudaEventCreate(&f.t_h1);
		cudaEventCreate(&f.t_c0);
		cudaEventCreate(&f.t_c1);
		if (!e->t_base)
		{
			cudaEventCreate(&e->t_base);
			cudaEventRecord(e->t_base, e->copy_stream);
		}
	}
	if (dbg_tl) cudaEventRecord(f.t_h0, e->copy_stream);
	LCD_TRY(upload_frames(e, n_frames, width, height, channels, images, depth, depth_type, f.img, f.depth, e->copy_stream));
	// the signature id list rides on the copy stream too: a host -> device copy queued on the compute stream would sit in the
	// same copy-engine queue as the next batch's images and serialise the two batches (measured)
	LCD_CUDA(e, f.sig_ids.reserve(ns, 0, false, e->copy_stream));
	LCD_CUDA(e, cudaMemcpyAsync(f.sig_ids.p, sig_ids, ns * sizeof(int), cudaMemcpyHostToDevice, e->copy_stream));
	if (dbg_tl) cudaEventRecord(f.t_h1, e->copy_stream);
	LCD_CUDA(e, cudaEventRecord(f.uploaded, e->copy_stream));
	// compute on the engine stream, behind the previous batch
	const int cap = op->n_features;
	const size_t rows = static_cast<size_t>(n_frames) * std::max(cap, 1);
	LCD_CUDA(e, e->d_like.reserve(static_cast<size_t>(n_frames) * ns, 0, false, s));
	LCD_CUDA(e, e->d_word_ids.reserve(rows, 0, false, s));
	LCD_CUDA(e, cudaStreamWaitEvent(s, f.uploaded, 0));
	if (dbg_tl) cudaEventRecord(f.t_c0, s);
	LCD_TRY(process_frames_dev(e, n_frames, f.img.p, width, height, channels, depth_type != LCD_DEPTH_NONE ? f.depth.p : nullptr, depth_type, op,
	                           incremental, nndr, new_words_compared_together, f.sig_ids.p, ns, n_total, vp, e->d_word_ids.p, e->d_like.p, s));
	LCD_TRY(download_frames(e, n_frames, rows, ns, vp, n_kp_out, word_ids_out, likelihood_out, hypothesis_out, s));
	f.user_results = nullptr;
	if (vp && results)
	{
		LCD_CUDA(e, e->v_packed.reserve(n_frames, 0, false, s));
		LCD_CUDA(e, f.res.reserve(n_frames));
		LCD_TRY(pack_verify_results(e, n_frames, e->v_packed.p, s));
		LCD_CUDA(e, cudaMemcpyAsync(f.res.p, e->v_packed.p, n_frames * sizeof(PackedVerifyResult), cudaMemcpyDeviceToHost, s));
		f.user_results = results;
	}
	f.n_frames = n_frames;
	f.detector = e->detector;
	LCD_CUDA(e, f.overflow.reserve(1));
	LCD_CUDA(e, cudaMemcpyAsync(f.overflow.p, e->o_overflow.p, sizeof(int), cudaMemcpyDeviceToHost, s));
	if (dbg_tl) cudaEventRecord(f.t_c1, s);
	LCD_CUDA(e, cudaEventRecord(f.done, s));
	++e->flights_busy;
	return LCD_OK;
}

int lcd_process_frames_wait(lcd_engine * e)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(set_device(e));
	if (e->flights_busy <= 0) LCD_FAIL(e, LCD_ERR_INVALID, "no batch in flight");
	lcd_engine::Flight & f = e->flights[e->flight_head];
	LCD_CUDA(e, cudaEventSynchronize(f.done));
	if (f.t_h0 && e->t_base)
	{
		float a = 0, b = 0, c = 0, d = 0;
		cudaEventElapsedTime(&a, e->t_base, f.t_h0);
		cudaEventElapsedTime(&b, e->t_base, f.t_h1);
		cudaEventElapsedTime(&c, e->t_base, f.t_c0);
		cudaEventElapsedTime(&d, e->t_base, f.t_c1);
		fprintf(stderr, "[lcd timeline] upload %.2f..%.2f  compute %.2f..%.2f ms\n", a, b, c, d);
	}
	if (f.user_results) memcpy(f.user_results, f.res.p, f.n_frames * sizeof(lcd_verify_result));
	if (f.user_dec) memcpy(f.user_dec, f.h_dec.p, f.n_frames * sizeof(lcd_decision));
	if (f.user_ep) epipolar_results(f.n_frames, f.h_ep_res.p, f.h_ep_F.p, f.user_ep);
	if (f.user_px) proximity_results(f.n_frames, f.px_max_paths, f.h_px_rec.p, f.h_px_res.p, f.user_px);
	f.user_results = nullptr;
	f.user_dec = nullptr;
	f.user_ep = nullptr;
	f.user_px = nullptr;
	e->flight_head ^= 1;
	--e->flights_busy;
	return overflow_report(e, f.overflow.p ? *f.overflow.p : 0, f.detector);
}

int lcd_verify_top_dev(lcd_engine * e, const void * d_queries, const float * d_uv, int n_frames, int nq_per_frame, const float * d_likelihood,
                       const int * d_sig_ids, int ns, const lcd_verify_params * vp, void * stream)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(set_device(e));
	if (!d_queries || !d_uv || !d_likelihood || !d_sig_ids || n_frames <= 0 || ns <= 0) LCD_FAIL(e, LCD_ERR_INVALID, "null argument");
	if (nq_per_frame <= 0 || nq_per_frame > kMaxFrameQueries) LCD_FAIL(e, LCD_ERR_CAPACITY, "1..%d descriptors per frame", kMaxFrameQueries);
	cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : e->stream;
	return verify_top_dev(e, static_cast<const uint32_t *>(d_queries), d_uv, n_frames, nq_per_frame, d_likelihood, d_sig_ids, ns, vp, s, nullptr, nullptr);
}

int lcd_process_fetch(lcd_engine * e, int n_frames, int * hypothesis_out, lcd_verify_result * results)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(set_device(e));
	if (n_frames <= 0) return LCD_OK;
	cudaStream_t s = e->stream;
	LCD_CUDA(e, cudaDeviceSynchronize());
	if (hypothesis_out) LCD_CUDA(e, cudaMemcpyAsync(hypothesis_out, e->d_hyp_id.p, n_frames * sizeof(int), cudaMemcpyDeviceToHost, s));
	if (results) return verify_download(e, n_frames, 0, results, nullptr, nullptr, s);
	LCD_CUDA(e, cudaStreamSynchronize(s));
	return LCD_OK;
}

int lcd_process_fetch_async(lcd_engine * e, int n_frames, int * hypothesis_out, lcd_verify_result * results, void * stream)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(set_device(e));
	if (n_frames <= 0) return LCD_OK;
	cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : e->stream;
	if (hypothesis_out) LCD_CUDA(e, cudaMemcpyAsync(hypothesis_out, e->d_hyp_id.p, n_frames * sizeof(int), cudaMemcpyDeviceToHost, s));
	if (results)
	{
		if (!e->v_ok.p || !e->d_hyp_id.p) LCD_FAIL(e, LCD_ERR_STATE, "no verification results on the device: run a step with verify parameters first");
		LCD_CUDA(e, e->v_packed.reserve(n_frames, 0, false, s));
		LCD_TRY(pack_verify_results(e, n_frames, e->v_packed.p, s));
		LCD_CUDA(e, cudaMemcpyAsync(results, e->v_packed.p, n_frames * sizeof(PackedVerifyResult), cudaMemcpyDeviceToHost, s));
	}
	return LCD_OK;
}

int lcd_process_batch(lcd_engine * e, const void * queries, const float * uv, int n_frames, int nq_per_frame, int incremental, float nndr,
                      int new_words_compared_together, const int * sig_ids, int ns, int n_total, const lcd_verify_params * vp,
                      int * word_ids_out, float * likelihood_out, int * hypothesis_out, lcd_verify_result * results)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(set_device(e));
	if (!queries || !uv || n_frames <= 0) LCD_FAIL(e, LCD_ERR_INVALID, "Descriptors size is null!");
	if (nq_per_frame <= 0 || nq_per_frame > kMaxFrameQueries) LCD_FAIL(e, LCD_ERR_CAPACITY, "1..%d descriptors per frame", kMaxFrameQueries);
	if (!sig_ids || ns <= 0) LCD_FAIL(e, LCD_ERR_INVALID, "ids list is empty");
	LCD_TRY(check_n_total(e, n_total));
	cudaStream_t s = e->stream;
	const size_t nq_total = static_cast<size_t>(n_frames) * nq_per_frame;
	LCD_CUDA(e, e->d_queries.reserve(nq_total * e->nw, 0, false, s));
	LCD_CUDA(e, e->d_uv.reserve(nq_total * 2, 0, false, s));
	LCD_CUDA(e, e->d_sig_ids.reserve(ns, 0, false, s));
	LCD_CUDA(e, e->d_like.reserve(static_cast<size_t>(n_frames) * ns, 0, false, s));
	if (word_ids_out) LCD_CUDA(e, e->d_word_ids.reserve(nq_total, 0, false, s));
	LCD_CUDA(e, cudaMemcpyAsync(e->d_queries.p, queries, nq_total * e->nw * 4, cudaMemcpyHostToDevice, s));
	LCD_CUDA(e, cudaMemcpyAsync(e->d_uv.p, uv, nq_total * 2 * sizeof(float), cudaMemcpyHostToDevice, s));
	LCD_CUDA(e, cudaMemcpyAsync(e->d_sig_ids.p, sig_ids, ns * sizeof(int), cudaMemcpyHostToDevice, s));
	LCD_TRY(process_dev(e, e->d_queries.p, e->d_uv.p, n_frames, nq_per_frame, incremental, nndr, new_words_compared_together, e->d_sig_ids.p, ns,
	                    n_total, vp, word_ids_out ? e->d_word_ids.p : nullptr, e->d_like.p, s));
	if (word_ids_out) LCD_CUDA(e, cudaMemcpyAsync(word_ids_out, e->d_word_ids.p, nq_total * sizeof(int), cudaMemcpyDeviceToHost, s));
	if (likelihood_out)
		LCD_CUDA(e, cudaMemcpyAsync(likelihood_out, e->d_like.p, static_cast<size_t>(n_frames) * ns * sizeof(float), cudaMemcpyDeviceToHost, s));
	if (hypothesis_out) LCD_CUDA(e, cudaMemcpyAsync(hypothesis_out, e->d_hyp_id.p, n_frames * sizeof(int), cudaMemcpyDeviceToHost, s));
	if (results) return verify_download(e, n_frames, 0, results, nullptr, nullptr, s);
	LCD_CUDA(e, cudaStreamSynchronize(s));
	return LCD_OK;
}

// ---- the loop-closure decision of many localisation clients (decide.cuh) -----------------------------------------
static_assert(sizeof(Decision) == sizeof(lcd_decision), "decision layout");

// drop the map versions that neither the current map nor any client's last posterior uses (the device must be idle)
static int prune_map_versions(lcd_engine * e)
{
	std::vector<long long> keys(e->dc_clients);
	if (e->dc_clients > 0) LCD_CUDA(e, cudaMemcpy(keys.data(), e->dc_key_ids.p, keys.size() * sizeof(long long), cudaMemcpyDeviceToHost));
	for (auto it = e->dc_versions.begin(); it != e->dc_versions.end();)
	{
		const long long ids = static_cast<long long>(reinterpret_cast<uintptr_t>(it->second->ids.p));
		const bool held = it->first == e->dc_map_ver || std::find(keys.begin(), keys.end(), ids) != keys.end();
		it = held ? std::next(it) : e->dc_versions.erase(it);
	}
	return LCD_OK;
}

int lcd_clients_create(lcd_engine * e, int n_clients)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(set_device(e));
	if (n_clients <= 0) LCD_FAIL(e, LCD_ERR_INVALID, "n_clients must be > 0");
	LCD_CUDA(e, cudaDeviceSynchronize());
	cudaStream_t s = e->stream;
	const size_t n = static_cast<size_t>(n_clients);
	if (e->dc_hi_id.reserve(n, 0, false, s) != cudaSuccess || e->dc_hi_val.reserve(n, 0, false, s) != cudaSuccess ||
	    e->dc_key_n.reserve(n, 0, false, s) != cudaSuccess || e->dc_key_ids.reserve(n, 0, false, s) != cudaSuccess ||
	    (e->dc_stride && e->dc_post.reserve(n * e->dc_stride, 0, false, s) != cudaSuccess))
	{
		cudaGetLastError();
		e->dc_clients = 0;
		LCD_FAIL(e, LCD_ERR_CAPACITY, "no device memory for the state of %d clients", n_clients);
	}
	LCD_CUDA(e, cudaMemsetAsync(e->dc_hi_id.p, 0, n * sizeof(int), s));
	LCD_CUDA(e, cudaMemsetAsync(e->dc_hi_val.p, 0, n * sizeof(float), s));
	LCD_CUDA(e, cudaMemsetAsync(e->dc_key_n.p, 0, n * sizeof(int), s));
	LCD_CUDA(e, cudaMemsetAsync(e->dc_key_ids.p, 0, n * sizeof(long long), s));
	LCD_CUDA(e, cudaStreamSynchronize(s));
	e->dc_clients = n_clients;
	e->dc_cams.assign(n, FrameCam{});
	e->dc_last_frames = 0;
	e->dc_hyp_valid = false;
	return prune_map_versions(e);
}

int lcd_clients_set_cameras(lcd_engine * e, const int * clients, int n, const lcd_camera * cams)
{
	if (!e) return LCD_ERR_INVALID;
	if (e->dc_clients <= 0) LCD_FAIL(e, LCD_ERR_STATE, "no clients: call lcd_clients_create first");
	if (n <= 0) return LCD_OK;
	if (!clients) LCD_FAIL(e, LCD_ERR_INVALID, "null client list");
	std::vector<FrameCam> rec(n, FrameCam{});
	for (int i = 0; i < n; ++i)
	{
		if (clients[i] < 0 || clients[i] >= e->dc_clients) LCD_FAIL(e, LCD_ERR_INVALID, "client %d is out of range [0, %d)", clients[i], e->dc_clients);
		if (!cams) continue;
		const lcd_camera & c = cams[i];
		bool finite = std::isfinite(c.fx) && std::isfinite(c.fy) && std::isfinite(c.cx) && std::isfinite(c.cy);
		for (int k = 0; k < 12; ++k) finite = finite && std::isfinite(c.local_transform[k]);
		if (!finite) LCD_FAIL(e, LCD_ERR_INVALID, "the camera of client %d has a value that is not finite", clients[i]);
		if (!(c.fx > 0.0) || !(c.fy > 0.0)) LCD_FAIL(e, LCD_ERR_INVALID, "the camera of client %d needs fx, fy > 0", clients[i]);
		if (c.image_width < 0 || c.image_height < 0 || (c.image_width == 0) != (c.image_height == 0))
			LCD_FAIL(e, LCD_ERR_INVALID, "the image size of client %d must be 0 x 0 or positive", clients[i]);
		// the engine inverts transforms as [R^T | -R^T t]: R R^T must be the identity
		const float * L = c.local_transform;
		for (int r = 0; r < 3; ++r)
			for (int q = 0; q < 3; ++q)
			{
				const double d = static_cast<double>(L[4 * r]) * L[4 * q] + static_cast<double>(L[4 * r + 1]) * L[4 * q + 1] +
				                 static_cast<double>(L[4 * r + 2]) * L[4 * q + 2];
				if (std::fabs(d - (r == q ? 1.0 : 0.0)) > 1e-5)
					LCD_FAIL(e, LCD_ERR_INVALID, "the local transform of client %d is not a rotation within 1e-5", clients[i]);
			}
		FrameCam & f = rec[i];
		f.fx = c.fx;
		f.fy = c.fy;
		f.cx = c.cx;
		f.cy = c.cy;
		std::memcpy(f.L, L, sizeof(f.L));
		f.w = c.image_width;
		f.h = c.image_height;
		f.set = 1;
		// Transform::isIdentity compares the values (-0 is 0)
		static const float kIdentity[12] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0};
		for (int k = 0; k < 12; ++k) f.local |= L[k] != kIdentity[k] ? 1 : 0;
	}
	// checked as a whole: a refused call changes nothing
	for (int i = 0; i < n; ++i) e->dc_cams[clients[i]] = rec[i];
	return LCD_OK;
}

int lcd_clients_reset(lcd_engine * e, const int * clients, int n)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(set_device(e));
	if (e->dc_clients <= 0) LCD_FAIL(e, LCD_ERR_STATE, "no clients: call lcd_clients_create first");
	if (n <= 0) return LCD_OK;
	if (!clients) LCD_FAIL(e, LCD_ERR_INVALID, "null client list");
	for (int i = 0; i < n; ++i)
		if (clients[i] < 0 || clients[i] >= e->dc_clients) LCD_FAIL(e, LCD_ERR_INVALID, "client %d is out of range [0, %d)", clients[i], e->dc_clients);
	LCD_CUDA(e, cudaDeviceSynchronize());
	cudaStream_t s = e->stream;
	LCD_CUDA(e, e->d_i1.reserve(n, 0, false, s));
	LCD_CUDA(e, cudaMemcpyAsync(e->d_i1.p, clients, n * sizeof(int), cudaMemcpyHostToDevice, s));
	decide_reset_clients_kernel<<<(n + 255) / 256, 256, 0, s>>>(e->d_i1.p, n, e->dc_hi_id.p, e->dc_hi_val.p, e->dc_key_n.p, e->dc_key_ids.p);
	LCD_CHECK_LAUNCH(e);
	LCD_CUDA(e, cudaStreamSynchronize(s));
	return prune_map_versions(e);
}

int lcd_clients_set_map(lcd_engine * e, const int * ids, int n, const int64_t * col_ptr, const int * nbr_row, const int * nbr_level,
                        const double * prediction_lc, int n_lc, float virtual_place_prior)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(set_device(e));
	if (!ids || n <= 0) LCD_FAIL(e, LCD_ERR_INVALID, "ids list is empty");
	if (ids[0] >= 0) LCD_FAIL(e, LCD_ERR_INVALID, "ids[0] must be the virtual place (a negative id): the working memory always holds it");
	std::vector<int> cp, ecol;
	float total = 0.f;
	double eps = 0.0;
	LCD_TRY(check_bayes_tables(e, ids, n, col_ptr, nbr_row, nbr_level, prediction_lc, n_lc, virtual_place_prior, cp, ecol, total, eps));
	const int64_t nnz = col_ptr[n];
	// the listed entries by row: row r gathers (P[r][c] - u_c) last[c] over the columns c that list it, in ascending c
	std::vector<int> tptr(n + 1, 0);
	for (int64_t k = 0; k < nnz; ++k)
		if (nbr_row[k] >= 1) ++tptr[nbr_row[k] + 1];
	for (int r = 0; r < n; ++r) tptr[r + 1] += tptr[r];
	const int nt = tptr[n];
	std::vector<int> tentry(std::max(nt, 1)), tcol(std::max(nt, 1)), fill(tptr.begin(), tptr.end() - 1);
	for (int64_t k = 0; k < nnz; ++k)
	{
		const int r = nbr_row[k];
		if (r < 1) continue;
		tentry[fill[r]] = static_cast<int>(k);
		tcol[fill[r]++] = ecol[static_cast<size_t>(k)];
	}
	// Everything the new map needs is built in new buffers; the engine switches to it only after the last step that can fail, so a failed
	// call leaves the previous map (or no map) in place.  The single-client path's per-call buffers serve as scratch for the column pass.
	cudaStream_t s = e->stream;
	auto ver = std::make_unique<lcd_engine::MapVersion>();
	auto tab = std::make_unique<lcd_engine::MapTables>();
	ver->n = n;
	DevBuf<int> d_tentry;
	const size_t nz = static_cast<size_t>(std::max<int64_t>(nnz, 1)), ntz = static_cast<size_t>(std::max(nt, 1));
	std::vector<float> tlv(ntz, 0.f);
	for (int k = 0; k < nt; ++k) tlv[k] = static_cast<float>(prediction_lc[nbr_level[tentry[k]] + 1]);
	// the scratch buffers below may be in use by queued work of the single-client path
	LCD_CUDA(e, cudaStreamSynchronize(s));
	if (ver->ids.reserve(n, 0, false, s) != cudaSuccess || tab->cptr.reserve(n + 1, 0, false, s) != cudaSuccess ||
	    tab->crow.reserve(nz, 0, false, s) != cudaSuccess || tab->clev.reserve(nz, 0, false, s) != cudaSuccess ||
	    e->by_scale.reserve(n, 0, false, s) != cudaSuccess || e->by_delta.reserve(n, 0, false, s) != cudaSuccess ||
	    tab->lc.reserve(n_lc, 0, false, s) != cudaSuccess || d_tentry.reserve(ntz, 0, false, s) != cudaSuccess ||
	    tab->u.reserve(n, 0, false, s) != cudaSuccess || tab->tptr.reserve(n + 1, 0, false, s) != cudaSuccess ||
	    tab->tcol.reserve(ntz, 0, false, s) != cudaSuccess || tab->tval.reserve(ntz, 0, false, s) != cudaSuccess ||
	    tab->tlv.reserve(ntz, 0, false, s) != cudaSuccess)
	{
		cudaGetLastError();
		LCD_FAIL(e, LCD_ERR_CAPACITY, "no device memory for a map of %d places and %d listed entries", n, nt);
	}
	LCD_CUDA(e, cudaMemcpyAsync(ver->ids.p, ids, n * sizeof(int), cudaMemcpyHostToDevice, s));
	LCD_CUDA(e, cudaMemcpyAsync(tab->cptr.p, cp.data(), (n + 1) * sizeof(int), cudaMemcpyHostToDevice, s));
	if (nnz)
	{
		LCD_CUDA(e, cudaMemcpyAsync(tab->crow.p, nbr_row, nnz * sizeof(int), cudaMemcpyHostToDevice, s));
		LCD_CUDA(e, cudaMemcpyAsync(tab->clev.p, nbr_level, nnz * sizeof(int), cudaMemcpyHostToDevice, s));
	}
	LCD_CUDA(e, cudaMemcpyAsync(tab->lc.p, prediction_lc, n_lc * sizeof(double), cudaMemcpyHostToDevice, s));
	LCD_CUDA(e, cudaMemcpyAsync(tab->tptr.p, tptr.data(), (n + 1) * sizeof(int), cudaMemcpyHostToDevice, s));
	if (nt)
	{
		LCD_CUDA(e, cudaMemcpyAsync(d_tentry.p, tentry.data(), nt * sizeof(int), cudaMemcpyHostToDevice, s));
		LCD_CUDA(e, cudaMemcpyAsync(tab->tcol.p, tcol.data(), nt * sizeof(int), cudaMemcpyHostToDevice, s));
		LCD_CUDA(e, cudaMemcpyAsync(tab->tlv.p, tlv.data(), nt * sizeof(float), cudaMemcpyHostToDevice, s));
	}
	tab->n_lc = n_lc;
	tab->total = total;
	tab->eps = static_cast<float>(eps);
	BayesArgs a{};
	a.n = n;
	a.vp_used = 1;
	a.ids = ver->ids.p;
	a.col_ptr = tab->cptr.p;
	a.nbr_row = tab->crow.p;
	a.nbr_level = tab->clev.p;
	a.lc = tab->lc.p;
	a.n_lc = n_lc;
	a.total = total;
	a.eps = static_cast<float>(eps);
	a.vpp = virtual_place_prior;
	a.col_u = tab->u.p;
	a.col_scale = e->by_scale.p;
	a.col_delta = e->by_delta.p;
	decide_map_columns_kernel<<<(n + 255) / 256, 256, 0, s>>>(a);
	LCD_CHECK_LAUNCH(e);
	if (nt)
	{
		decide_entry_values_kernel<<<(nt + 255) / 256, 256, 0, s>>>(a, nt, d_tentry.p, tab->tcol.p, tab->tval.p);
		LCD_CHECK_LAUNCH(e);
	}
	// the clients' posteriors keep their ids (re-keyed when each client next computes); their rows grow to the largest map
	DevBuf<float> grown;
	const size_t stride = std::max(e->dc_stride, static_cast<size_t>(n));
	if (stride > e->dc_stride && e->dc_clients > 0)
	{
		if (grown.reserve(static_cast<size_t>(e->dc_clients) * stride, 0, false, s) != cudaSuccess)
		{
			cudaGetLastError();
			LCD_FAIL(e, LCD_ERR_CAPACITY, "no device memory for the posteriors of %d clients over %d places", e->dc_clients, n);
		}
		// kernels of the last decision (on any stream) may still write the posteriors being copied
		LCD_CUDA(e, cudaDeviceSynchronize());
		if (e->dc_stride)
			LCD_CUDA(e, cudaMemcpy2DAsync(grown.p, stride * sizeof(float), e->dc_post.p, e->dc_stride * sizeof(float), e->dc_stride * sizeof(float),
			                              e->dc_clients, cudaMemcpyDeviceToDevice, s));
	}
	LCD_CUDA(e, cudaStreamSynchronize(s));
	// kernels of the last decision may still read the tables this call replaces
	LCD_CUDA(e, cudaDeviceSynchronize());
	// commit: nothing below can fail
	if (grown.p) e->dc_post.swap(grown);
	e->dc_stride = stride;
	e->dc_tables = std::move(tab);
	e->gps_places.reset();
	e->dc_map_ver = e->dc_next_ver++;
	e->dc_versions[e->dc_map_ver] = std::move(ver);
	e->dc_n = n;
	e->dc_h_ids.assign(ids, ids + n);
	e->dc_lc0 = prediction_lc[0];
	e->dc_vpp = virtual_place_prior;
	return prune_map_versions(e);
}

static int check_decide_params(lcd_engine * e, const lcd_decide_params * dp)
{
	if (!dp) LCD_FAIL(e, LCD_ERR_INVALID, "null decision parameters");
	if (dp->virtual_place_ratio != 0 && dp->virtual_place_ratio != 1) LCD_FAIL(e, LCD_ERR_INVALID, "Rtabmap/VirtualPlaceLikelihoodRatio must be 0 or 1");
	if (!(dp->loop_thr >= 0.f && dp->loop_thr <= 1.f)) LCD_FAIL(e, LCD_ERR_INVALID, "Rtabmap/LoopThr must be in [0, 1]");
	if (!(dp->aggressive_loop_thr >= 0.f && dp->aggressive_loop_thr <= 1.f)) LCD_FAIL(e, LCD_ERR_INVALID, "RGBD/AggressiveLoopThr must be in [0, 1]");
	if (!(dp->loop_ratio >= 0.f && dp->loop_ratio <= 1.f)) LCD_FAIL(e, LCD_ERR_INVALID, "Rtabmap/LoopRatio must be in [0, 1]");
	if (!(dp->max_loop_closure_distance >= 0.f && std::isfinite(dp->max_loop_closure_distance)))
		LCD_FAIL(e, LCD_ERR_INVALID, "RGBD/MaxLoopClosureDistance must be >= 0");
	return LCD_OK;
}

// checks of one decision call and the upload of its frame tables (before any kernel of the call is queued); gps[n_frames] (may be null)
// is uploaded behind them, then the snapshot of the frames' cameras when a frame's client has one.  stage: pinned staging the caller owns
// and knows to be free (null: the engine's, once its last upload is done).  width x height: the call's image size (0 x 0: no images),
// which a camera's image size must match when it is set.
static int decide_prepare(lcd_engine * e, int n_frames, int ns, const int * clients, const int * frame_flags, const lcd_decide_params * dp,
                          cudaStream_t s, const GpsFrame * gps = nullptr, PinBuf<long long> * stage = nullptr, int width = 0, int height = 0)
{
	if (e->dc_clients <= 0) LCD_FAIL(e, LCD_ERR_STATE, "no clients: call lcd_clients_create first");
	if (e->dc_map_ver < 0) LCD_FAIL(e, LCD_ERR_STATE, "no map: call lcd_clients_set_map first");
	LCD_TRY(check_decide_params(e, dp));
	if (n_frames <= 0 || !clients || !frame_flags) LCD_FAIL(e, LCD_ERR_INVALID, "no frames");
	if (ns <= 0 || ns != e->dc_n - 1) LCD_FAIL(e, LCD_ERR_INVALID, "ns = %d, but the map holds %d real places", ns, e->dc_n - 1);
	std::vector<char> seen(e->dc_clients, 0);
	e->dc_active.clear();
	for (int f = 0; f < n_frames; ++f)
	{
		const int c = clients[f];
		if (c < 0 || c >= e->dc_clients) LCD_FAIL(e, LCD_ERR_INVALID, "client %d of frame %d is out of range [0, %d)", c, f, e->dc_clients);
		if (seen[c]) LCD_FAIL(e, LCD_ERR_INVALID, "client %d appears more than once in one call", c);
		seen[c] = 1;
		if (!(frame_flags[f] & (kDcFlagSkip | kDcFlagHold))) e->dc_active.push_back(f);
	}
	bool any_cam = false, cam_sized = false;
	for (int f = 0; f < n_frames; ++f)
	{
		const FrameCam & c = e->dc_cams[clients[f]];
		if (!c.set) continue;
		any_cam = true;
		cam_sized = cam_sized || c.w > 0;
		if (width > 0 && c.w > 0 && (c.w != width || c.h != height))
			LCD_FAIL(e, LCD_ERR_INVALID, "the camera of client %d is %d x %d, the images of the call %d x %d", clients[f], c.w, c.h, width, height);
	}
	const int B = static_cast<int>(e->dc_active.size());
	static_assert(sizeof(GpsFrame) % sizeof(long long) == 0, "GPS frame table layout");
	const size_t gps_words = gps ? n_frames * (sizeof(GpsFrame) / sizeof(long long)) : 0;
	const size_t cam0 = 2 * static_cast<size_t>(n_frames) + 2 * static_cast<size_t>(B) + gps_words;
	const size_t words = cam0 + (any_cam ? n_frames * (sizeof(FrameCam) / sizeof(long long)) : 0);
	if (!stage)
	{
		if (!e->dc_h_ev) LCD_CUDA(e, cudaEventCreateWithFlags(&e->dc_h_ev, cudaEventDisableTiming));
		else LCD_CUDA(e, cudaEventSynchronize(e->dc_h_ev)); // the staging buffer of the last call has been copied
		stage = &e->dc_h_tab;
	}
	LCD_CUDA(e, stage->reserve(words));
	long long * h = stage->p;
	for (int f = 0; f < n_frames; ++f)
	{
		h[f] = clients[f];
		h[n_frames + f] = frame_flags[f];
	}
	long long * hb = h + 2 * n_frames;
	for (int b = 0; b < B; ++b)
	{
		const int f = e->dc_active[b];
		hb[b] = f;
		hb[B + b] = clients[f];
	}
	if (gps) std::memcpy(hb + 2 * B, gps, n_frames * sizeof(GpsFrame));
	FrameCam * hc = reinterpret_cast<FrameCam *>(h + cam0);
	if (any_cam)
		for (int f = 0; f < n_frames; ++f) hc[f] = e->dc_cams[clients[f]];
	LCD_CUDA(e, e->dc_tab.reserve(words, 0, false, s));
	LCD_CUDA(e, cudaMemcpyAsync(e->dc_tab.p, h, words * sizeof(long long), cudaMemcpyHostToDevice, s));
	if (stage == &e->dc_h_tab) LCD_CUDA(e, cudaEventRecord(e->dc_h_ev, s));
	e->dc_frame_cam = any_cam ? reinterpret_cast<const FrameCam *>(e->dc_tab.p + cam0) : nullptr;
	e->dc_cam_sized = cam_sized;
	return LCD_OK;
}

// adjustLikelihood, the posterior of every frame that computes one, the hypothesis selection and checks.  r2 >= 0 (a call with a GPS
// table uploaded by decide_prepare): the GPS filter of each frame's place list first, with RGBD/LocalRadius squared.  d_qn[n_frames]
// (may be null): each frame's quantised words; a frame with none is decided as LCD_FRAME_SKIP decides it (decide.cuh, decide_bad)
static int decide_launch(lcd_engine * e, const float * d_like, int n_frames, int ns, const lcd_decide_params * dp, float * d_post_out, cudaStream_t s,
                         double r2 = -1.0, const int * d_qn = nullptr)
{
	const int n = e->dc_n, B = static_cast<int>(e->dc_active.size());
	const lcd_engine::MapTables & t = *e->dc_tables;
	DecideMap m{n, e->dc_versions.at(e->dc_map_ver)->ids.p, t.u.p, t.tptr.p, t.tcol.p, t.tval.p, e->dc_lc0, e->dc_vpp, t.tlv.p, t.eps};
	const long long * tab = e->dc_tab.p;
	const GpsFrame * gps = r2 >= 0.0 ? reinterpret_cast<const GpsFrame *>(tab + 2 * n_frames + 2 * B) : nullptr;
	LCD_CUDA(e, e->dc_adj.reserve(static_cast<size_t>(n_frames) * n, 0, false, s));
	if (gps)
	{
		LCD_CUDA(e, e->gps_listed.reserve(static_cast<size_t>(n_frames) * n, 0, false, s));
		LCD_CUDA(e, e->gps_count.reserve(n_frames, 0, false, s));
		LCD_CUDA(e, cudaMemsetAsync(e->gps_count.p, 0, n_frames * sizeof(int), s));
		// without a table no frame is gated (lcd_decide_gps_batch_dev refuses fixes then), and the kernel reads no place
		decide_gps_gate_kernel<<<dim3((n + 255) / 256, n_frames), 256, 0, s>>>(n, e->gps_places ? e->gps_places->p : nullptr, gps, r2, e->gps_listed.p,
		                                                                         e->gps_count.p);
		LCD_CHECK_LAUNCH(e);
		adjust_likelihood_listed_kernel<<<n_frames, kAdjustThreads, 0, s>>>(d_like, ns, dp->virtual_place_ratio, e->dc_adj.p, e->gps_listed.p);
	}
	else adjust_likelihood_kernel<<<n_frames, kAdjustThreads, 0, s>>>(d_like, ns, dp->virtual_place_ratio, e->dc_adj.p);
	LCD_CHECK_LAUNCH(e);
	if (B > 0)
	{
		const int n_cc = (n + kDcColChunk - 1) / kDcColChunk, n_rc = (n + kDcRowChunk - 1) / kDcRowChunk;
		const size_t nb = static_cast<size_t>(n) * B;
		LCD_CUDA(e, e->dc_last_t.reserve(nb, 0, false, s));
		LCD_CUDA(e, e->dc_post_t.reserve(nb, 0, false, s));
		LCD_CUDA(e, e->dc_part_u.reserve(static_cast<size_t>(n_cc) * B, 0, false, s));
		LCD_CUDA(e, e->dc_part_s1.reserve(static_cast<size_t>(n_cc) * B, 0, false, s));
		LCD_CUDA(e, e->dc_part_p.reserve(static_cast<size_t>(n_rc) * B, 0, false, s));
		LCD_CUDA(e, e->dc_sums.reserve(3 * static_cast<size_t>(B), 0, false, s));
		DecideBatch d{};
		d.B = B;
		d.frame = tab + 2 * n_frames;
		d.client = d.frame + B;
		d.key_n = e->dc_key_n.p;
		d.key_ids = e->dc_key_ids.p;
		d.qn = d_qn;
		d.cl_post = e->dc_post.p;
		d.stride = static_cast<long long>(e->dc_stride);
		d.adj = e->dc_adj.p;
		d.last_t = e->dc_last_t.p;
		d.post_t = e->dc_post_t.p;
		d.part_u = e->dc_part_u.p;
		d.part_s1 = e->dc_part_s1.p;
		d.part_p = e->dc_part_p.p;
		d.u = e->dc_sums.p;
		d.s1 = e->dc_sums.p + B;
		d.psum = e->dc_sums.p + 2 * B;
		if (gps)
		{
			LCD_CUDA(e, e->gps_fu.reserve(nb, 0, false, s));
			LCD_CUDA(e, e->gps_fscale.reserve(nb, 0, false, s));
			LCD_CUDA(e, e->gps_fdelta.reserve(nb, 0, false, s));
			d.gps = gps;
			d.count = e->gps_count.p;
			d.listed = e->gps_listed.p;
			d.fu = e->gps_fu.p;
			d.fscale = e->gps_fscale.p;
			d.fdelta = e->gps_fdelta.p;
			BayesArgs a{};
			a.n = n;
			a.vp_used = 1;
			a.ids = m.ids;
			a.col_ptr = t.cptr.p;
			a.nbr_row = t.crow.p;
			a.nbr_level = t.clev.p;
			a.lc = t.lc.p;
			a.n_lc = t.n_lc;
			a.total = t.total;
			a.eps = t.eps;
			a.vpp = e->dc_vpp;
			decide_gps_columns_kernel<<<static_cast<unsigned>((nb + 255) / 256), 256, 0, s>>>(a, d);
			LCD_CHECK_LAUNCH(e);
		}
		const int threads = std::min(kDcThreads, (B + 31) / 32 * 32);
		decide_last_kernel<<<static_cast<unsigned>((nb + 255) / 256), 256, 0, s>>>(m, d);
		LCD_CHECK_LAUNCH(e);
		decide_columns_kernel<<<n_cc, threads, 0, s>>>(m, d);
		LCD_CHECK_LAUNCH(e);
		decide_sum_chunks_kernel<<<(B + 127) / 128, 128, 0, s>>>(d.part_u, n_cc, B, d.u);
		LCD_CHECK_LAUNCH(e);
		decide_sum_chunks_kernel<<<(B + 127) / 128, 128, 0, s>>>(d.part_s1, n_cc, B, d.s1);
		LCD_CHECK_LAUNCH(e);
		decide_rows_kernel<<<n_rc, threads, 0, s>>>(m, d);
		LCD_CHECK_LAUNCH(e);
		decide_sum_chunks_kernel<<<(B + 127) / 128, 128, 0, s>>>(d.part_p, n_rc, B, d.psum);
		LCD_CHECK_LAUNCH(e);
		decide_normalize_kernel<<<dim3((n + 31) / 32, (B + 31) / 32), dim3(32, 8), 0, s>>>(m, d, e->dc_post.p, d_post_out);
		LCD_CHECK_LAUNCH(e);
	}
	LCD_CUDA(e, e->dc_dec.reserve(n_frames, 0, false, s));
	LCD_CUDA(e, e->d_hyp_id.reserve(n_frames, 0, false, s));
	LCD_CUDA(e, e->d_hyp_slot.reserve(n_frames, 0, false, s));
	DecideSelect a{};
	a.n_frames = n_frames;
	a.client = tab;
	a.flags = tab + n_frames;
	a.cl_post = e->dc_post.p;
	a.stride = static_cast<long long>(e->dc_stride);
	a.hi_id = e->dc_hi_id.p;
	a.hi_val = e->dc_hi_val.p;
	a.loop_thr = dp->loop_thr;
	a.aggressive_loop_thr = dp->aggressive_loop_thr;
	a.loop_ratio = dp->loop_ratio;
	a.sig_slot = e->st_map.d.p;
	a.slot_cap = e->st_map.n_ids;
	a.dec = e->dc_dec.p;
	a.hyp_id = e->d_hyp_id.p;
	a.hyp_slot = e->d_hyp_slot.p;
	a.gps = gps;
	a.count = gps ? e->gps_count.p : nullptr;
	a.qn = d_qn;
	a.key_n = e->dc_key_n.p;
	a.key_ids = e->dc_key_ids.p;
	decide_select_kernel<<<n_frames, 256, 0, s>>>(m, a);
	LCD_CHECK_LAUNCH(e);
	e->dc_last_frames = n_frames;
	e->dc_hyp_valid = true;
	e->px_valid = false;
	e->px_last_frames = 0;
	e->dc_verified = false;
	e->dc_max_dist = dp->max_loop_closure_distance;
	return LCD_OK;
}

int lcd_decide_batch_dev(lcd_engine * e, const float * d_likelihood, int n_frames, int ns, const int * clients, const int * frame_flags,
                         const lcd_decide_params * dp, float * d_posterior_out, void * stream)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(set_device(e));
	if (!d_likelihood) LCD_FAIL(e, LCD_ERR_INVALID, "likelihood is empty");
	cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : e->stream;
	LCD_TRY(decide_prepare(e, n_frames, ns, clients, frame_flags, dp, s));
	return decide_launch(e, d_likelihood, n_frames, ns, dp, d_posterior_out, s);
}

// ---- the GPS filter of the place list (Rtabmap/LoopGPS) ----------------------------------------------------------------
static_assert(sizeof(GpsFrame) == 72 && sizeof(GpsPlace) == 40, "GPS table layout");

// GeodeticCoords::toGeocentric_WGS84 (GeodeticCoords.cpp:75-102): the same double statements, glibc's trigonometry
static void geocentric_wgs84(const lcd_gps & g, double & x, double & y, double & z)
{
	static const double a = 6378137;
	static const double b = 6356752.3142;
	static const double ae = std::acos(b / a);
	static const double cos2_ae_earth = std::cos(ae) * std::cos(ae);
	static const double sin2_ae_earth = std::sin(ae) * std::sin(ae);
	const double lon = g.longitude * M_PI / 180.0;
	const double lat = g.latitude * M_PI / 180.0;
	const double sin_lat = std::sin(lat);
	const double N = a / std::sqrt(1.0 - sin2_ae_earth * (sin_lat * sin_lat));
	x = (N + g.altitude) * std::cos(lat) * std::cos(lon);
	y = (N + g.altitude) * std::cos(lat) * std::sin(lon);
	z = (cos2_ae_earth * N + g.altitude) * sin_lat;
}

static bool gps_finite(const lcd_gps & g)
{
	return std::isfinite(g.stamp) && std::isfinite(g.longitude) && std::isfinite(g.latitude) && std::isfinite(g.altitude) && std::isfinite(g.error);
}

int lcd_clients_set_map_gps(lcd_engine * e, const int * ids, int n, const lcd_gps * gps, const float * offset_enu)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(set_device(e));
	if (e->dc_map_ver < 0) LCD_FAIL(e, LCD_ERR_STATE, "no map: call lcd_clients_set_map first");
	if (!ids || !gps || n != e->dc_n - 1) LCD_FAIL(e, LCD_ERR_INVALID, "n = %d, but the map holds %d real places", n, e->dc_n - 1);
	for (int i = 0; i < n; ++i)
	{
		if (ids[i] != e->dc_h_ids[i + 1]) LCD_FAIL(e, LCD_ERR_INVALID, "ids[%d] = %d differs from the map's %d", i, ids[i], e->dc_h_ids[i + 1]);
		if (!gps_finite(gps[i])) LCD_FAIL(e, LCD_ERR_INVALID, "the GPS of place %d is not finite", ids[i]);
		if (offset_enu && !(std::isfinite(offset_enu[3 * i]) && std::isfinite(offset_enu[3 * i + 1]) && std::isfinite(offset_enu[3 * i + 2])))
			LCD_FAIL(e, LCD_ERR_INVALID, "the ENU offset of place %d is not finite", ids[i]);
	}
	std::vector<GpsPlace> h(std::max(n, 1));
	for (int i = 0; i < n; ++i)
	{
		GpsPlace & p = h[i];
		p = GpsPlace{};
		p.fix = gps[i].stamp > 0.0;
		if (p.fix) geocentric_wgs84(gps[i], p.x, p.y, p.z);
		if (offset_enu)
		{
			p.ox = offset_enu[3 * i];
			p.oy = offset_enu[3 * i + 1];
			p.oz = offset_enu[3 * i + 2];
		}
	}
	cudaStream_t s = e->stream;
	auto buf = std::make_unique<DevBuf<GpsPlace>>();
	if (buf->reserve(h.size(), 0, false, s) != cudaSuccess)
	{
		cudaGetLastError();
		LCD_FAIL(e, LCD_ERR_CAPACITY, "no device memory for the GPS of %d places", n);
	}
	LCD_CUDA(e, cudaMemcpyAsync(buf->p, h.data(), h.size() * sizeof(GpsPlace), cudaMemcpyHostToDevice, s));
	LCD_CUDA(e, cudaStreamSynchronize(s));
	// kernels of the last GPS decision may still read the table this call replaces
	LCD_CUDA(e, cudaDeviceSynchronize());
	e->gps_places = std::move(buf);
	return LCD_OK;
}

} // extern "C"
// the GPS frame table of a decision call (frame_gps may be null: no fixes): the frames that compute a posterior and carry a fix (the block
// of Rtabmap.cpp:1994 does not run for the others) are gated
static int gps_frames(lcd_engine * e, int n_frames, const int * frame_flags, const lcd_gps * frame_gps, float local_radius, std::vector<GpsFrame> & g)
{
	if (n_frames <= 0 || !frame_flags) LCD_FAIL(e, LCD_ERR_INVALID, "no frames");
	if (!(local_radius >= 0.f) || !std::isfinite(local_radius)) LCD_FAIL(e, LCD_ERR_INVALID, "RGBD/LocalRadius must be >= 0");
	g.assign(n_frames, GpsFrame{});
	bool any_fix = false;
	for (int f = 0; f < n_frames; ++f)
	{
		const bool compute = !(frame_flags[f] & (kDcFlagSkip | kDcFlagHold));
		g[f].mode = compute ? kGpsAll : kGpsNone;
		if (!frame_gps) continue;
		if (!gps_finite(frame_gps[f])) LCD_FAIL(e, LCD_ERR_INVALID, "the GPS of frame %d is not finite", f);
		if (!compute || !(frame_gps[f].stamp > 0.0)) continue;
		any_fix = true;
		const lcd_gps & o = frame_gps[f];
		geocentric_wgs84(o, g[f].x, g[f].y, g[f].z);
		// Geocentric_WGS84ToENU_WGS84's rotation (GeodeticCoords.cpp:134-135)
		g[f].clat = std::cos(o.latitude * M_PI / 180.0);
		g[f].slat = std::sin(o.latitude * M_PI / 180.0);
		g[f].clon = std::cos(o.longitude * M_PI / 180.0);
		g[f].slon = std::sin(o.longitude * M_PI / 180.0);
		g[f].error = o.error;
		g[f].mode = kGpsGated;
	}
	if (any_fix && (e->dc_map_ver < 0 || !e->gps_places))
		LCD_FAIL(e, LCD_ERR_STATE, "frames carry a GPS fix but the map has no GPS table: call lcd_clients_set_map_gps");
	return LCD_OK;
}
extern "C" {

int lcd_decide_gps_batch_dev(lcd_engine * e, const float * d_likelihood, int n_frames, int ns, const int * clients, const int * frame_flags,
                             const lcd_gps * frame_gps, float local_radius, const lcd_decide_params * dp, float * d_posterior_out,
                             unsigned char * d_compared_out, void * stream)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(set_device(e));
	if (!d_likelihood) LCD_FAIL(e, LCD_ERR_INVALID, "likelihood is empty");
	if (!clients) LCD_FAIL(e, LCD_ERR_INVALID, "no frames");
	std::vector<GpsFrame> g;
	LCD_TRY(gps_frames(e, n_frames, frame_flags, frame_gps, local_radius, g));
	cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : e->stream;
	LCD_TRY(decide_prepare(e, n_frames, ns, clients, frame_flags, dp, s, g.data()));
	const float r2 = local_radius * local_radius; // _localRadius*_localRadius: a float, compared in double
	LCD_TRY(decide_launch(e, d_likelihood, n_frames, ns, dp, d_posterior_out, s, static_cast<double>(r2)));
	if (d_compared_out)
		LCD_CUDA(e, cudaMemcpy2DAsync(d_compared_out, ns, e->gps_listed.p + 1, e->dc_n, ns, n_frames, cudaMemcpyDeviceToDevice, s));
	return LCD_OK;
}

int lcd_decide_fetch(lcd_engine * e, int n_frames, lcd_decision * out)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(set_device(e));
	if (!out || n_frames <= 0) LCD_FAIL(e, LCD_ERR_INVALID, "null output");
	if (e->dc_last_frames == 0) LCD_FAIL(e, LCD_ERR_STATE, "no decision: run lcd_decide_batch_dev first");
	if (n_frames > e->dc_last_frames) LCD_FAIL(e, LCD_ERR_INVALID, "the last decision has %d frames", e->dc_last_frames);
	LCD_CUDA(e, cudaDeviceSynchronize());
	LCD_CUDA(e, cudaMemcpy(out, e->dc_dec.p, n_frames * sizeof(lcd_decision), cudaMemcpyDeviceToHost));
	return LCD_OK;
}

// Memory::computeTransform of every accepted hypothesis of the last decision (store slot -1: not verified), then the rejections of
// Rtabmap.cpp:3156-3167.  d_nq_frame / d_xyz_to as verify_top_dev takes them.
static int verify_decided(lcd_engine * e, const uint32_t * d_q, const float * d_uv, int n_frames, int nq, const lcd_verify_params * vp, cudaStream_t s,
                          const int * d_nq_frame = nullptr, const float * d_xyz_to = nullptr)
{
	LCD_TRY(check_verify_params(e, vp, true));
	if (e->dc_last_frames == 0 || !e->dc_hyp_valid) LCD_FAIL(e, LCD_ERR_STATE, "no decision to verify: run lcd_decide_batch_dev first");
	if (n_frames != e->dc_last_frames) LCD_FAIL(e, LCD_ERR_INVALID, "the last decision has %d frames, not %d", e->dc_last_frames, n_frames);
	const PairSource src{{e->st_desc.p, e->st_xyz.p, e->st_n.p, e->d_hyp_slot.p, e->st_cap},
	                     {d_q, d_uv, d_xyz_to, d_nq_frame, nq, nq, nullptr, e->dc_frame_cam}};
	LCD_TRY(register_pairs(e, src, n_frames, std::max(e->st_cap, nq), vp, s, e->dc_cam_sized));
	decide_verified_kernel<<<(n_frames + 127) / 128, 128, 0, s>>>(n_frames, e->v_ok.p, e->v_T.p, e->dc_max_dist, e->dc_dec.p, e->d_hyp_id.p,
	                                                             e->px_valid ? e->px_skip.p : nullptr);
	LCD_CHECK_LAUNCH(e);
	e->dc_verified = true;
	return LCD_OK;
}

int lcd_verify_decided_dev(lcd_engine * e, const void * d_queries, const float * d_uv, int n_frames, int nq_per_frame, const lcd_verify_params * vp,
                           void * stream)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(set_device(e));
	if (!d_queries || !d_uv || n_frames <= 0) LCD_FAIL(e, LCD_ERR_INVALID, "Descriptors size is null!");
	if (nq_per_frame <= 0 || nq_per_frame > kMaxFrameQueries) LCD_FAIL(e, LCD_ERR_CAPACITY, "1..%d descriptors per frame", kMaxFrameQueries);
	cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : e->stream;
	return verify_decided(e, static_cast<const uint32_t *>(d_queries), d_uv, n_frames, nq_per_frame, vp, s);
}

int lcd_process_decide_batch_dev(lcd_engine * e, const void * d_queries, const float * d_uv, int n_frames, int nq_per_frame, int incremental,
                                 float nndr, int new_words_compared_together, int ns, int n_total, const lcd_verify_params * vp, const int * clients,
                                 const int * frame_flags, const lcd_decide_params * dp, int * d_word_ids_out, float * d_likelihood_out,
                                 float * d_posterior_out, void * stream)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(require_binary(e, "lcd_process_decide_batch_dev"));
	LCD_TRY(require_unsharded(e, "lcd_process_decide_batch_dev"));
	LCD_TRY(set_device(e));
	if (!d_queries || !d_uv || n_frames <= 0) LCD_FAIL(e, LCD_ERR_INVALID, "Descriptors size is null!");
	if (nq_per_frame <= 0 || nq_per_frame > kMaxFrameQueries) LCD_FAIL(e, LCD_ERR_CAPACITY, "1..%d descriptors per frame", kMaxFrameQueries);
	LCD_TRY(check_n_total(e, n_total));
	LCD_TRY(check_verify_params(e, vp, true));
	cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : e->stream;
	LCD_TRY(decide_prepare(e, n_frames, ns, clients, frame_flags, dp, s));
	float * d_like = d_likelihood_out;
	if (!d_like)
	{
		LCD_CUDA(e, e->d_like.reserve(static_cast<size_t>(n_frames) * ns, 0, false, s));
		d_like = e->d_like.p;
	}
	const uint32_t * d_q = static_cast<const uint32_t *>(d_queries);
	const int * d_sig_ids = e->dc_versions.at(e->dc_map_ver)->ids.p + 1; // the map's real places, ascending
	LCD_TRY(localize_dev(e, d_q, n_frames, nq_per_frame, incremental, nndr, new_words_compared_together, d_sig_ids, ns, n_total, d_word_ids_out,
	                     d_like, s));
	LCD_TRY(decide_launch(e, d_like, n_frames, ns, dp, d_posterior_out, s));
	return verify_decided(e, d_q, d_uv, n_frames, nq_per_frame, vp, s);
}

// ---- proximity detection by space (proximity.cuh) ---------------------------------------------------------------------
static_assert(sizeof(ProxPath) == 16, "lcd_proximity_path key layout");

int lcd_clients_set_map_poses(lcd_engine * e, const int * ids, int n, const float * poses, const int64_t * nbr_ptr, const int * nbr_ids)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(set_device(e));
	if (e->dc_map_ver < 0) LCD_FAIL(e, LCD_ERR_STATE, "no map: call lcd_clients_set_map first");
	if (!ids || !poses || !nbr_ptr || n != e->dc_n - 1) LCD_FAIL(e, LCD_ERR_INVALID, "n = %d, but the map holds %d real places", n, e->dc_n - 1);
	for (int i = 0; i < n; ++i)
		if (ids[i] != e->dc_h_ids[i + 1]) LCD_FAIL(e, LCD_ERR_INVALID, "ids[%d] = %d differs from the map's %d", i, ids[i], e->dc_h_ids[i + 1]);
	for (size_t k = 0; k < 12 * static_cast<size_t>(n); ++k)
		if (!std::isfinite(poses[k])) LCD_FAIL(e, LCD_ERR_INVALID, "the pose of place %d is not finite", ids[k / 12]);
	if (nbr_ptr[0] != 0) LCD_FAIL(e, LCD_ERR_INVALID, "nbr_ptr[0] must be 0");
	for (int i = 0; i < n; ++i)
		if (nbr_ptr[i + 1] < nbr_ptr[i]) LCD_FAIL(e, LCD_ERR_INVALID, "nbr_ptr must not decrease");
	if (nbr_ptr[n] > INT32_MAX || (nbr_ptr[n] > 0 && !nbr_ids)) LCD_FAIL(e, LCD_ERR_INVALID, "bad neighbour links");
	// links to places outside the map (not in the working memory) can never join a path: they are dropped here
	std::vector<int> ptr(n + 1, 0), row;
	row.reserve(static_cast<size_t>(nbr_ptr[n]));
	for (int i = 0; i < n; ++i)
	{
		for (int64_t k = nbr_ptr[i]; k < nbr_ptr[i + 1]; ++k)
		{
			const int * it = std::lower_bound(ids, ids + n, nbr_ids[k]);
			if (it != ids + n && *it == nbr_ids[k]) row.push_back(static_cast<int>(it - ids));
		}
		ptr[i + 1] = static_cast<int>(row.size());
	}
	cudaStream_t s = e->stream;
	auto m = std::make_unique<lcd_engine::MapPoses>();
	if (m->poses.reserve(12 * static_cast<size_t>(n), 0, false, s) != cudaSuccess || m->nbr_ptr.reserve(n + 1, 0, false, s) != cudaSuccess ||
	    m->nbr_row.reserve(std::max<size_t>(row.size(), 1), 0, false, s) != cudaSuccess)
	{
		cudaGetLastError();
		LCD_FAIL(e, LCD_ERR_CAPACITY, "no device memory for the poses and links of %d places", n);
	}
	LCD_CUDA(e, cudaMemcpyAsync(m->poses.p, poses, 12 * static_cast<size_t>(n) * sizeof(float), cudaMemcpyHostToDevice, s));
	LCD_CUDA(e, cudaMemcpyAsync(m->nbr_ptr.p, ptr.data(), (n + 1) * sizeof(int), cudaMemcpyHostToDevice, s));
	if (!row.empty()) LCD_CUDA(e, cudaMemcpyAsync(m->nbr_row.p, row.data(), row.size() * sizeof(int), cudaMemcpyHostToDevice, s));
	LCD_CUDA(e, cudaStreamSynchronize(s));
	// kernels of the last proximity step may still read the poses this call replaces
	LCD_CUDA(e, cudaDeviceSynchronize());
	e->px_map = std::move(m);
	e->px_ver = e->dc_map_ver;
	return LCD_OK;
}

} // extern "C"
// the checks of a proximity step's parameters
static int check_proximity_params(lcd_engine * e, const lcd_proximity_params * pp)
{
	if (!pp || !pp->verify) LCD_FAIL(e, LCD_ERR_INVALID, "null proximity or verification parameters");
	const lcd_verify_params * vp = pp->verify;
	LCD_TRY(check_verify_params(e, vp, false));
	if (!(pp->local_radius > 0.f) || !std::isfinite(pp->local_radius)) LCD_FAIL(e, LCD_ERR_INVALID, "RGBD/LocalRadius must be > 0");
	if (!(pp->angle >= 0.f) || !std::isfinite(pp->angle)) LCD_FAIL(e, LCD_ERR_INVALID, "RGBD/ProximityAngle must be >= 0");
	if (pp->max_graph_depth < 0) LCD_FAIL(e, LCD_ERR_INVALID, "RGBD/ProximityMaxGraphDepth must be >= 0");
	if (!std::isfinite(pp->path_filtering_radius) || !(pp->max_loop_closure_distance >= 0.f) || !std::isfinite(pp->max_loop_closure_distance))
		LCD_FAIL(e, LCD_ERR_INVALID, "bad RGBD/ProximityPathFilteringRadius or RGBD/MaxLoopClosureDistance");
	// <= 0 is "no limit" in the reference (Rtabmap.cpp:2829); at most kPxMaxPaths attempts per frame are supported
	if (pp->max_paths <= 0 || pp->max_paths > kPxMaxPaths) LCD_FAIL(e, LCD_ERR_CAPACITY, "RGBD/ProximityMaxPaths must be 1..%d", kPxMaxPaths);
	if (e->st_cap == 0) LCD_FAIL(e, LCD_ERR_STATE, "the signature store is empty: nothing to verify against");
	return LCD_OK;
}

static int check_proximity_poses(lcd_engine * e)
{
	if (!e->px_map || e->px_ver != e->dc_map_ver) LCD_FAIL(e, LCD_ERR_STATE, "no poses for the current map: call lcd_clients_set_map_poses");
	return LCD_OK;
}

static int check_frame_poses(lcd_engine * e, int n_frames, const float * frame_poses)
{
	for (int k = 0; k < 12 * n_frames; ++k)
		if (!std::isfinite(frame_poses[k])) LCD_FAIL(e, LCD_ERR_INVALID, "the pose of frame %d is not finite", k / 12);
	return LCD_OK;
}

// proximity detection on the last decision (checked by the callers); frame_poses / enabled: host arrays.  d_n_frame[n_frames] (may be
// null: nq_per_frame each) the frames' rows to register, with d_xyz_to their 3-D points (may be null); d_qn as decide_launch takes it.
static int proximity_decide(lcd_engine * e, const uint32_t * d_q, const float * d_uv, int n_frames, int nq_per_frame, const float * frame_poses,
                            const int * enabled, const lcd_proximity_params * pp, cudaStream_t s, const int * d_n_frame = nullptr,
                            const float * d_xyz_to = nullptr, const int * d_qn = nullptr)
{
	const lcd_verify_params * vp = pp->verify;
	const int mp = pp->max_paths, n_pairs = n_frames * mp;
	LCD_CUDA(e, e->px_frame_pose.reserve(12 * static_cast<size_t>(n_frames), 0, false, s));
	LCD_CUDA(e, e->px_enabled.reserve(n_frames, 0, false, s));
	LCD_CUDA(e, e->px_rec.reserve(n_frames, 0, false, s));
	LCD_CUDA(e, e->px_skip.reserve(n_frames, 0, false, s));
	LCD_CUDA(e, e->px_slot.reserve(n_pairs, 0, false, s));
	LCD_CUDA(e, e->px_row.reserve(n_pairs, 0, false, s));
	LCD_CUDA(e, e->px_nto.reserve(n_pairs, 0, false, s));
	LCD_CUDA(e, e->px_res.reserve(n_pairs, 0, false, s));
	LCD_CUDA(e, cudaMemcpyAsync(e->px_frame_pose.p, frame_poses, 12 * static_cast<size_t>(n_frames) * sizeof(float), cudaMemcpyHostToDevice, s));
	LCD_CUDA(e, cudaMemcpyAsync(e->px_enabled.p, enabled, n_frames * sizeof(int), cudaMemcpyHostToDevice, s));
	// RGBD/ProximityPathFilteringRadius, capped by RGBD/MaxLoopClosureDistance (Rtabmap.cpp:2822-2826)
	float fr = pp->path_filtering_radius;
	if (pp->max_loop_closure_distance > 0.f && (fr <= 0.f || pp->max_loop_closure_distance < fr)) fr = pp->max_loop_closure_distance;
	ProxArgs a{};
	a.n = e->dc_n - 1;
	a.ids = e->dc_versions.at(e->dc_map_ver)->ids.p + 1;
	a.poses = e->px_map->poses.p;
	a.nbr_ptr = e->px_map->nbr_ptr.p;
	a.nbr_row = e->px_map->nbr_row.p;
	a.frame_pose = e->px_frame_pose.p;
	a.enabled = e->px_enabled.p;
	a.flags = e->dc_tab.p + n_frames;
	a.adj = e->dc_adj.p;
	a.dec = e->dc_dec.p;
	a.sig_slot = e->st_map.d.p;
	a.slot_cap = e->st_map.n_ids;
	a.radius = pp->local_radius;
	// _proximityAngle *= M_PI/180.0f, a float (Rtabmap.cpp:609-612)
	a.angle = static_cast<float>(static_cast<double>(pp->angle) * (M_PI / 180.0));
	a.filter_radius = fr;
	a.max_paths = mp;
	a.max_depth = pp->max_graph_depth;
	a.rec = e->px_rec.p;
	a.pair_slot = e->px_slot.p;
	a.pair_row = e->px_row.p;
	a.pair_n_to = e->px_nto.p;
	a.nq = nq_per_frame;
	a.n_frame = d_n_frame;
	a.qn = d_qn;
	prof_mark(e, LCD_PROF_PROXIMITY, s);
	proximity_paths_kernel<<<n_frames, kPxThreads, 0, s>>>(a);
	prof_mark(e, LCD_PROF_PROXIMITY, s);
	LCD_CHECK_LAUNCH(e);
	// Memory::computeTransform(place, frame) of every attempted pair in one launch, with a null guess (RGBD/ProximityOdomGuess = false):
	// FROM = the store row px_slot[i] (-1: none) with its cached dictionary, TO = row px_row[i] of the frames' descriptors, px_nto[i] of
	// them (0: the pair is not registered)
	const PairSource src{{e->st_desc.p, e->st_xyz.p, e->st_n.p, e->px_slot.p, e->st_cap},
	                     {d_q, d_uv, d_xyz_to, e->px_nto.p, 0, nq_per_frame, e->px_row.p, e->dc_frame_cam}};
	LCD_TRY(register_pairs(e, src, n_pairs, std::max(e->st_cap, nq_per_frame), vp, s, e->dc_cam_sized));
	LCD_TRY(pack_verify_results(e, n_pairs, e->px_res.p, s));
	proximity_apply_kernel<<<(n_frames + 127) / 128, 128, 0, s>>>(n_frames, mp, fr, e->v_ok.p, e->v_T.p, e->px_rec.p, e->dc_dec.p, e->d_hyp_id.p,
	                                                             e->d_hyp_slot.p, e->px_skip.p);
	LCD_CHECK_LAUNCH(e);
	e->px_last_frames = n_frames;
	e->px_max_paths = mp;
	e->px_valid = true;
	return LCD_OK;
}

extern "C" {

int lcd_decide_proximity_dev(lcd_engine * e, const void * d_queries, const float * d_uv, int n_frames, int nq_per_frame, const float * frame_poses,
                             const int * enabled, const lcd_proximity_params * pp, void * stream)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(set_device(e));
	if (!d_queries || !d_uv || !frame_poses || !enabled || n_frames <= 0) LCD_FAIL(e, LCD_ERR_INVALID, "null or empty frame input");
	if (nq_per_frame <= 0 || nq_per_frame > kMaxFrameQueries) LCD_FAIL(e, LCD_ERR_CAPACITY, "1..%d descriptors per frame", kMaxFrameQueries);
	LCD_TRY(check_proximity_params(e, pp));
	if (e->dc_last_frames == 0 || !e->dc_hyp_valid) LCD_FAIL(e, LCD_ERR_STATE, "no decision: run lcd_decide_batch_dev first");
	if (e->dc_verified) LCD_FAIL(e, LCD_ERR_STATE, "the decision was already verified: run proximity detection before lcd_verify_decided_dev");
	if (n_frames != e->dc_last_frames) LCD_FAIL(e, LCD_ERR_INVALID, "the last decision has %d frames, not %d", e->dc_last_frames, n_frames);
	LCD_TRY(check_proximity_poses(e));
	if (e->px_last_frames) LCD_FAIL(e, LCD_ERR_STATE, "proximity detection already ran on this decision");
	LCD_TRY(check_frame_poses(e, n_frames, frame_poses));
	cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : e->stream;
	return proximity_decide(e, static_cast<const uint32_t *>(d_queries), d_uv, n_frames, nq_per_frame, frame_poses, enabled, pp, s);
}

int lcd_proximity_fetch(lcd_engine * e, int n_frames, lcd_proximity_result * out)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(set_device(e));
	if (!out || n_frames <= 0) LCD_FAIL(e, LCD_ERR_INVALID, "null output");
	if (e->px_last_frames == 0) LCD_FAIL(e, LCD_ERR_STATE, "no proximity detection: run lcd_decide_proximity_dev first");
	if (n_frames > e->px_last_frames) LCD_FAIL(e, LCD_ERR_INVALID, "the last proximity detection has %d frames", e->px_last_frames);
	LCD_CUDA(e, cudaDeviceSynchronize());
	const int mp = e->px_max_paths;
	std::vector<ProxRecord> rec(n_frames);
	std::vector<PackedVerifyResult> res(static_cast<size_t>(n_frames) * mp);
	LCD_CUDA(e, cudaMemcpy(rec.data(), e->px_rec.p, n_frames * sizeof(ProxRecord), cudaMemcpyDeviceToHost));
	LCD_CUDA(e, cudaMemcpy(res.data(), e->px_res.p, res.size() * sizeof(PackedVerifyResult), cudaMemcpyDeviceToHost));
	proximity_results(n_frames, mp, rec.data(), res.data(), out);
	return LCD_OK;
}

// ---- the localisation step of Rtabmap::process from images (lcd_process_frames_decide_*) --------------------------------------------
static_assert(sizeof(lcd_decide_stages) == 48 && offsetof(lcd_decide_stages, local_radius) == 8 && offsetof(lcd_decide_stages, epipolar) == 16 &&
                  offsetof(lcd_decide_stages, proximity_enabled) == 40,
              "lcd_decide_stages layout (rtabmap_b200/capi.py DecideStages)");
} // extern "C"

// the checks of lcd_process_frames_decide_*, before anything is queued (decide_prepare makes the decision's own); g: the GPS frame
// table of the call, empty without the GPS filter
static int frames_decide_check(lcd_engine * e, const char * what, int n_frames, const lcd_orb_params * op, int n_total, const lcd_verify_params * vp,
                               const int * frame_flags, const lcd_decide_stages * st, std::vector<GpsFrame> & g)
{
	LCD_TRY(require_binary(e, what));
	LCD_TRY(require_unsharded(e, what));
	if (e->cfg.desc_type != LCD_DESC_U8 || e->cfg.desc_dim != 32) LCD_FAIL(e, LCD_ERR_INVALID, "ORB descriptors need an engine with 32-byte binary descriptors");
	if (!op) LCD_FAIL(e, LCD_ERR_INVALID, "null ORB parameters");
	if (op->n_features <= 0 || op->n_features > kMaxFrameQueries) LCD_FAIL(e, LCD_ERR_CAPACITY, "Kp/MaxFeatures must be 1..%d", kMaxFrameQueries);
	if (n_frames <= 0 || !frame_flags) LCD_FAIL(e, LCD_ERR_INVALID, "no frames");
	LCD_TRY(check_n_total(e, n_total));
	LCD_TRY(check_verify_params(e, vp, true));
	g.clear();
	if (!st) return LCD_OK;
	if (st->frame_gps) LCD_TRY(gps_frames(e, n_frames, frame_flags, st->frame_gps, st->local_radius, g));
	if (st->epipolar)
	{
		// epipolar_decide's launch limit, checked before the decision changes any client state
		const int cap = std::max(op->n_features, std::max(e->ws_cap, 1));
		LCD_TRY(fit_smem(e, reinterpret_cast<const void *>(epipolar_check_kernel), epi_smem_bytes(cap), cap));
	}
	if (st->proximity)
	{
		if (!st->frame_poses || !st->proximity_enabled) LCD_FAIL(e, LCD_ERR_INVALID, "proximity detection needs the frames' poses and enabled flags");
		LCD_TRY(check_proximity_params(e, st->proximity));
		LCD_TRY(check_proximity_poses(e));
		LCD_TRY(check_frame_poses(e, n_frames, st->frame_poses));
	}
	return LCD_OK;
}

// the device work of lcd_process_frames_decide_* on s, behind decide_prepare: detection, the likelihood against the map's real places,
// the decision with its optional stages, and the verification of what it accepted.  poses / enabled: the proximity step's host arrays.
static int frames_decide_dev(lcd_engine * e, int n_frames, const uint8_t * d_images, int width, int height, int channels, const void * d_depth,
                             int depth_type, const lcd_orb_params * op, int incremental, float nndr, int cmp_new, int ns, int n_total,
                             const lcd_verify_params * vp, const lcd_decide_params * dp, const lcd_decide_stages * st, const float * poses,
                             const int * enabled, int * d_words, float * d_like, float * d_post, cudaStream_t s)
{
	const int cap = op->n_features;
	LCD_TRY(frame_front_end(e, n_frames, cap, e->o_kp, e->o_desc, e->o_xyz, &e->o_uv, e->o_n, s));
	LCD_TRY(orb_run(e, n_frames, d_images, width, height, channels, d_depth, depth_type, op, cap, e->o_kp.p, e->o_desc.p, e->o_xyz.p, e->o_uv.p,
	                e->o_n.p, s, e->dc_frame_cam));
	const uint32_t * d_q = reinterpret_cast<const uint32_t *>(e->o_desc.p);
	const int * d_sig_ids = e->dc_versions.at(e->dc_map_ver)->ids.p + 1; // the map's real places, ascending
	const int * d_qn = e->o_n.p;                                         // quantised words of each frame: Signature::isBadSignature
	if (limit_active(e))
	{
		const int k = limit_rows(e, cap);
		LCD_TRY(limit_to_engine(e, n_frames, cap, e->o_kp.p, e->o_n.p, d_q, s));
		LCD_TRY(localize_dev(e, e->ql_desc.p, n_frames, k, incremental, nndr, cmp_new, d_sig_ids, ns, n_total, e->ql_words.p, d_like, s, e->ql_n.p));
		LCD_TRY(launch_expand(e, n_frames, cap, k, e->o_n.p, e->ql_index.p, e->ql_n.p, e->ql_words.p, d_words, s));
		d_qn = e->ql_n.p;
	}
	else
		LCD_TRY(localize_dev(e, d_q, n_frames, cap, incremental, nndr, cmp_new, d_sig_ids, ns, n_total, d_words, d_like, s, e->o_n.p));
	const double r2 = st && st->frame_gps ? static_cast<double>(st->local_radius * st->local_radius) : -1.0;
	LCD_TRY(decide_launch(e, d_like, n_frames, ns, dp, d_post, s, r2, d_qn));
	if (st && st->epipolar) LCD_TRY(epipolar_decide(e, d_words, e->o_uv.p, e->o_n.p, n_frames, cap, st->epipolar, s));
	if (st && st->proximity)
		LCD_TRY(proximity_decide(e, d_q, e->o_uv.p, n_frames, cap, poses, enabled, st->proximity, s, e->o_n.p, e->o_xyz.p, d_qn));
	return verify_decided(e, d_q, e->o_uv.p, n_frames, cap, vp, s, e->o_n.p, e->o_xyz.p);
}
extern "C" {

int lcd_process_frames_decide_dev(lcd_engine * e, int n_frames, const uint8_t * d_images, int width, int height, int channels, const void * d_depth,
                                  int depth_type, const lcd_orb_params * op, int incremental, float nndr, int new_words_compared_together, int ns,
                                  int n_total, const lcd_verify_params * vp, const int * clients, const int * frame_flags, const lcd_decide_params * dp,
                                  const lcd_decide_stages * stages, int * d_word_ids_out, float * d_likelihood_out, float * d_posterior_out,
                                  void * stream)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(set_device(e));
	if (!d_images) LCD_FAIL(e, LCD_ERR_INVALID, "null image");
	std::vector<GpsFrame> g;
	LCD_TRY(frames_decide_check(e, "lcd_process_frames_decide_dev", n_frames, op, n_total, vp, frame_flags, stages, g));
	cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : e->stream;
	LCD_TRY(decide_prepare(e, n_frames, ns, clients, frame_flags, dp, s, g.empty() ? nullptr : g.data(), nullptr, width, height));
	int * d_words = d_word_ids_out;
	if (!d_words)
	{
		LCD_CUDA(e, e->d_word_ids.reserve(static_cast<size_t>(n_frames) * op->n_features, 0, false, s));
		d_words = e->d_word_ids.p;
	}
	float * d_like = d_likelihood_out;
	if (!d_like)
	{
		LCD_CUDA(e, e->d_like.reserve(static_cast<size_t>(n_frames) * ns, 0, false, s));
		d_like = e->d_like.p;
	}
	return frames_decide_dev(e, n_frames, d_images, width, height, channels, d_depth, depth_type, op, incremental, nndr, new_words_compared_together, ns,
	                         n_total, vp, dp, stages, stages ? stages->frame_poses : nullptr, stages ? stages->proximity_enabled : nullptr, d_words,
	                         d_like, d_posterior_out, s);
}

int lcd_process_frames_decide_submit(lcd_engine * e, int n_frames, const uint8_t * images, int width, int height, int channels, const void * depth,
                                     int depth_type, const lcd_orb_params * op, int incremental, float nndr, int new_words_compared_together, int ns,
                                     int n_total, const lcd_verify_params * vp, const int * clients, const int * frame_flags,
                                     const lcd_decide_params * dp, const lcd_decide_stages * stages, int * n_kp_out, int * word_ids_out,
                                     float * likelihood_out, lcd_decision * decisions_out, lcd_verify_result * results_out,
                                     lcd_epipolar_result * epipolar_out, lcd_proximity_result * proximity_out)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(set_device(e));
	if (!images || n_frames <= 0 || width <= 0 || height <= 0) LCD_FAIL(e, LCD_ERR_INVALID, "null image");
	if (e->flights_busy >= 2) LCD_FAIL(e, LCD_ERR_INVALID, "two batches are already in flight: call lcd_process_frames_wait first");
	std::vector<GpsFrame> g;
	LCD_TRY(frames_decide_check(e, "lcd_process_frames_decide_submit", n_frames, op, n_total, vp, frame_flags, stages, g));
	cudaStream_t s = e->stream;
	const int slot = (e->flight_head + e->flights_busy) & 1;
	lcd_engine::Flight & f = e->flights[slot];
	LCD_TRY(copy_stream_ready(e));
	if (!f.uploaded)
	{
		LCD_CUDA(e, cudaEventCreateWithFlags(&f.uploaded, cudaEventDisableTiming));
		LCD_CUDA(e, cudaEventCreateWithFlags(&f.done, cudaEventDisableTiming));
	}
	// the slot's previous batch was waited for, so its staging buffers are free: nothing here waits for the batch in flight
	LCD_TRY(decide_prepare(e, n_frames, ns, clients, frame_flags, dp, s, g.empty() ? nullptr : g.data(), &f.h_tab, width, height));
	const float * poses = nullptr;
	const int * enabled = nullptr;
	if (stages && stages->proximity)
	{
		LCD_CUDA(e, f.h_pose.reserve(12 * static_cast<size_t>(n_frames)));
		LCD_CUDA(e, f.h_enabled.reserve(n_frames));
		std::memcpy(f.h_pose.p, stages->frame_poses, 12 * static_cast<size_t>(n_frames) * sizeof(float));
		std::memcpy(f.h_enabled.p, stages->proximity_enabled, n_frames * sizeof(int));
		poses = f.h_pose.p;
		enabled = f.h_enabled.p;
	}
	LCD_TRY(upload_frames(e, n_frames, width, height, channels, images, depth, depth_type, f.img, f.depth, e->copy_stream));
	LCD_CUDA(e, cudaEventRecord(f.uploaded, e->copy_stream));
	const int cap = op->n_features;
	const size_t rows = static_cast<size_t>(n_frames) * cap;
	LCD_CUDA(e, e->d_like.reserve(static_cast<size_t>(n_frames) * ns, 0, false, s));
	LCD_CUDA(e, e->d_word_ids.reserve(rows, 0, false, s));
	LCD_CUDA(e, cudaStreamWaitEvent(s, f.uploaded, 0));
	LCD_TRY(frames_decide_dev(e, n_frames, f.img.p, width, height, channels, depth_type != LCD_DEPTH_NONE ? f.depth.p : nullptr, depth_type, op,
	                          incremental, nndr, new_words_compared_together, ns, n_total, vp, dp, stages, poses, enabled, e->d_word_ids.p, e->d_like.p,
	                          nullptr, s));
	LCD_TRY(download_frames(e, n_frames, rows, ns, nullptr, n_kp_out, word_ids_out, likelihood_out, nullptr, s));
	f.user_results = nullptr;
	f.user_dec = nullptr;
	f.user_ep = nullptr;
	f.user_px = nullptr;
	if (results_out)
	{
		LCD_CUDA(e, e->v_packed.reserve(n_frames, 0, false, s));
		LCD_CUDA(e, f.res.reserve(n_frames));
		LCD_TRY(pack_verify_results(e, n_frames, e->v_packed.p, s));
		LCD_CUDA(e, cudaMemcpyAsync(f.res.p, e->v_packed.p, n_frames * sizeof(PackedVerifyResult), cudaMemcpyDeviceToHost, s));
		f.user_results = results_out;
	}
	if (decisions_out)
	{
		LCD_CUDA(e, f.h_dec.reserve(n_frames));
		LCD_CUDA(e, cudaMemcpyAsync(f.h_dec.p, e->dc_dec.p, n_frames * sizeof(Decision), cudaMemcpyDeviceToHost, s));
		f.user_dec = decisions_out;
	}
	if (epipolar_out && stages && stages->epipolar)
	{
		LCD_CUDA(e, f.h_ep_res.reserve(static_cast<size_t>(n_frames) * 8));
		LCD_CUDA(e, f.h_ep_F.reserve(static_cast<size_t>(n_frames) * 9));
		LCD_CUDA(e, cudaMemcpyAsync(f.h_ep_res.p, e->ep_res.p, static_cast<size_t>(n_frames) * 8 * sizeof(int), cudaMemcpyDeviceToHost, s));
		LCD_CUDA(e, cudaMemcpyAsync(f.h_ep_F.p, e->ep_F.p, static_cast<size_t>(n_frames) * 9 * sizeof(double), cudaMemcpyDeviceToHost, s));
		f.user_ep = epipolar_out;
	}
	if (proximity_out && stages && stages->proximity)
	{
		const size_t n_pairs = static_cast<size_t>(n_frames) * e->px_max_paths;
		LCD_CUDA(e, f.h_px_rec.reserve(n_frames));
		LCD_CUDA(e, f.h_px_res.reserve(n_pairs));
		LCD_CUDA(e, cudaMemcpyAsync(f.h_px_rec.p, e->px_rec.p, n_frames * sizeof(ProxRecord), cudaMemcpyDeviceToHost, s));
		LCD_CUDA(e, cudaMemcpyAsync(f.h_px_res.p, e->px_res.p, n_pairs * sizeof(PackedVerifyResult), cudaMemcpyDeviceToHost, s));
		f.user_px = proximity_out;
		f.px_max_paths = e->px_max_paths;
	}
	f.n_frames = n_frames;
	f.detector = e->detector;
	LCD_CUDA(e, f.overflow.reserve(1));
	LCD_CUDA(e, cudaMemcpyAsync(f.overflow.p, e->o_overflow.p, sizeof(int), cudaMemcpyDeviceToHost, s));
	LCD_CUDA(e, cudaEventRecord(f.done, s));
	++e->flights_busy;
	return LCD_OK;
}

// ---- word-range sharding ---------------------------------------------------------------------
int lcd_shard_set_row_offset(lcd_engine * e, int global_row_offset)
{
	if (!e || global_row_offset < 0) return LCD_ERR_INVALID;
	e->row_offset = global_row_offset;
	return LCD_OK;
}

// Sharded key sets: per query two u32 keys (dist << 22 | global row) for binary descriptors, two u64 keys (float bits of the distance
// << 32 | global row) for float descriptors; all-ones = none.  Buffers stay typed uint32_t: a float key pair is four words.
static int shard_key_words(const lcd_engine * e) { return e->f32 ? 4 : 2; }

// merge of the n_chunks partial top-2 sets run_knn left behind into one key pair per query
static int shard_merge_keys(lcd_engine * e, int n_chunks, int nq, uint32_t * d_keys_out, cudaStream_t s)
{
	if (e->f32) knn2_merge64_kernel<<<(nq + 255) / 256, 256, 0, s>>>(e->d_partial64.p, n_chunks, nq, reinterpret_cast<ulonglong2 *>(d_keys_out));
	else knn2_merge_kernel<<<(nq + 255) / 256, 256, 0, s>>>(e->d_partial.p, n_chunks, nq, d_keys_out);
	LCD_CHECK_LAUNCH(e);
	return LCD_OK;
}

// the resolve reads its keys from `keys` (gathered key sets), starting at query `q0`
static void shard_set_keys(const lcd_engine * e, ResolveArgs & a, const uint32_t * keys, size_t q0)
{
	if (e->f32) a.partial64 = reinterpret_cast<const ulonglong2 *>(keys) + q0;
	else a.partial = reinterpret_cast<const uint2 *>(keys) + q0;
}

int lcd_shard_knn2_keys_dev(lcd_engine * e, const void * d_queries, int nq, uint32_t * d_keys_out, void * stream)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(set_device(e));
	if (!d_queries || nq <= 0 || !d_keys_out) LCD_FAIL(e, LCD_ERR_INVALID, "null argument");
	cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : e->stream;
	int n_chunks = 0;
	LCD_TRY(run_knn(e, static_cast<const uint32_t *>(d_queries), nq, e->n_indexed, &n_chunks, s));
	return shard_merge_keys(e, n_chunks, nq, d_keys_out, s);
}

int lcd_shard_resolve_score_dev(lcd_engine * e, const void * d_queries, int n_frames, int nq_per_frame,
                                const uint32_t * d_keys_gathered, int n_ranks, const int * d_row_ids, int total_rows_, int last_word_id,
                                int incremental, float nndr, int new_words_compared_together, const int * d_sig_ids, int ns, int n_total,
                                int * d_word_ids_out, long long * d_scores_out, void * stream)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(set_device(e));
	if (!d_queries || !d_keys_gathered || !d_row_ids || n_frames <= 0 || n_ranks <= 0) LCD_FAIL(e, LCD_ERR_INVALID, "null argument");
	if (nq_per_frame <= 0 || nq_per_frame > kMaxFrameQueries) LCD_FAIL(e, LCD_ERR_CAPACITY, "1..%d descriptors per frame", kMaxFrameQueries);
	LCD_TRY(check_n_total(e, n_total));
	(void)total_rows_;
	cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : e->stream;
	ResolveArgs a = resolve_args(e, static_cast<const uint32_t *>(d_queries), nq_per_frame, n_frames * nq_per_frame, nullptr, n_ranks, d_row_ids, incremental,
	                             nndr, new_words_compared_together, last_word_id, d_word_ids_out);
	shard_set_keys(e, a, d_keys_gathered, 0);
	return resolve_score(e, a, n_frames, n_total, false, nullptr, d_sig_ids, ns, d_scores_out, s);
}

int lcd_shard_resolve_frames_dev(lcd_engine * e, const void * d_queries_all, int frame0, int n_frames, int n_frames_total, int nq_per_frame,
                                 const uint32_t * d_keys_gathered, int n_ranks, const int * d_row_ids, int last_word_id, int incremental,
                                 float nndr, int new_words_compared_together, const int * d_n_per_frame, int * d_word_ids_out, void * stream)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(set_device(e));
	if (!d_queries_all || !d_keys_gathered || !d_row_ids || !d_word_ids_out || n_frames <= 0 || n_ranks <= 0 || frame0 < 0 ||
	    frame0 + n_frames > n_frames_total)
		LCD_FAIL(e, LCD_ERR_INVALID, "null argument or frame range outside the job");
	if (nq_per_frame <= 0 || nq_per_frame > kMaxFrameQueries) LCD_FAIL(e, LCD_ERR_CAPACITY, "1..%d descriptors per frame", kMaxFrameQueries);
	cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : e->stream;
	// nq_total = n_frames_total * nq_per_frame: the stride between the gathered key sets
	ResolveArgs a = resolve_args(e, static_cast<const uint32_t *>(d_queries_all) + static_cast<size_t>(frame0) * nq_per_frame * e->nw, nq_per_frame,
	                             n_frames_total * nq_per_frame, d_n_per_frame ? d_n_per_frame + frame0 : nullptr, n_ranks, d_row_ids, incremental, nndr,
	                             new_words_compared_together, last_word_id, d_word_ids_out);
	shard_set_keys(e, a, d_keys_gathered, static_cast<size_t>(frame0) * nq_per_frame);
	return launch_resolve(e, a, n_frames, s);
}

int lcd_shard_score_ids_dev(lcd_engine * e, const int * d_word_ids_all, int n_frames, int nq_per_frame, const int * d_sig_ids, int ns, int n_total,
                            long long * d_scores_out, void * stream)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(set_device(e));
	if (!d_word_ids_all || !d_sig_ids || !d_scores_out || n_frames <= 0 || ns <= 0) LCD_FAIL(e, LCD_ERR_INVALID, "null argument");
	if (nq_per_frame <= 0 || nq_per_frame > kMaxFrameQueries) LCD_FAIL(e, LCD_ERR_CAPACITY, "1..%d words per signature", kMaxFrameQueries);
	LCD_TRY(check_n_total(e, n_total));
	cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : e->stream;
	LCD_TRY(prep_ids(e, d_word_ids_all, n_frames, nq_per_frame, n_total, 1, false, s));
	return score_tfidf(e, n_frames, nq_per_frame, d_sig_ids, ns, d_scores_out, s);
}

// ---- the similarity likelihood over word-range shards ----------------------------------------------------------------------
// Global descriptors of the sharded similarity step: the local frames' own (frames [n_frames][dim] or nullptr), and the map's, given by
// the caller because the descriptor store refuses sharded engines (rows [n_rows][dim], row_of_k [ns] the row of each listed place or -1).
struct ShardGdesc
{
	const float * frames;
	const float * rows;
	const int * row_of_k;
	int n_rows;
	int dim;
};

// The row indices are read back (one synchronisation of `s`) so that an index outside the table is refused before any kernel reads it.
static int shard_check_gdesc(lcd_engine * e, const ShardGdesc & g, int ns, cudaStream_t s)
{
	if (!g.frames && !g.rows && !g.row_of_k) return LCD_OK;
	if (g.dim <= 0) LCD_FAIL(e, LCD_ERR_INVALID, "global descriptors need dim > 0, got %d", g.dim);
	if (!g.rows != !g.row_of_k) LCD_FAIL(e, LCD_ERR_INVALID, "the map's global descriptors need both the table and the row of each listed place");
	if (!g.rows) return LCD_OK;
	if (g.n_rows <= 0) LCD_FAIL(e, LCD_ERR_INVALID, "the global-descriptor table needs at least one row, got %d", g.n_rows);
	std::vector<int> h(ns);
	LCD_CUDA(e, cudaMemcpyAsync(h.data(), g.row_of_k, static_cast<size_t>(ns) * sizeof(int), cudaMemcpyDeviceToHost, s));
	LCD_CUDA(e, cudaStreamSynchronize(s));
	for (int k = 0; k < ns; ++k)
		if (h[k] < -1 || h[k] >= g.n_rows)
			LCD_FAIL(e, LCD_ERR_INVALID, "global-descriptor row %d of listed place %d is outside the table of %d rows", h[k], k, g.n_rows);
	return LCD_OK;
}

// valid(q) of n_frames local frames from their word ids [n_frames][nq] into e->q_valid, and their dot products with the listed places'
// descriptors into e->gd_dot when both sides carry descriptors.  Returns whether the dot products exist through *gd.
static int shard_similarity_prepare(lcd_engine * e, int n_frames, int nq, const int * d_word_ids, const ShardGdesc & g, const int * d_sig_ids, int ns,
                                    bool * gd, cudaStream_t s)
{
	LCD_CUDA(e, e->q_valid.reserve(n_frames, 0, false, s));
	valid_ids_kernel<<<n_frames, kValidThreads, 0, s>>>(d_word_ids, nq, e->q_valid.p);
	LCD_CHECK_LAUNCH(e);
	*gd = g.frames && g.rows;
	if (*gd)
	{
		LCD_CUDA(e, e->gd_dot.reserve(static_cast<size_t>(n_frames) * ns, 0, false, s));
		GdescArgs a{g.frames, n_frames, g.rows, g.dim, nullptr, 0, d_sig_ids, ns, e->gd_dot.p, g.row_of_k};
		prof_mark(e, LCD_PROF_SCORE, s);
		gdesc_dot_kernel<<<dim3((ns + kGdBN - 1) / kGdBN, (n_frames + kGdBM - 1) / kGdBM), kGdThreads, 0, s>>>(a);
		prof_mark(e, LCD_PROF_SCORE, s);
		LCD_CHECK_LAUNCH(e);
	}
	return LCD_OK;
}

// compareTo of the local frames [f0, f0 + n_frames) from the summed pair counts d_pairs [n_frames][ns] and valid(s) d_valid [ns], after
// shard_similarity_prepare of all local frames
static int shard_similarity_finalize(lcd_engine * e, int f0, int n_frames, const int * d_pairs, const int * d_valid, const ShardGdesc & g, bool gd,
                                     const int * d_sig_ids, int ns, float * d_likelihood_out, cudaStream_t s)
{
	const size_t o = static_cast<size_t>(f0) * ns;
	SimilarityArgs a{nullptr, 0, d_pairs, d_valid, 0, e->q_valid.p + f0, gd ? e->gd_dot.p + o : nullptr, g.row_of_k, 0, d_sig_ids, ns, d_likelihood_out + o};
	similarity_finalize_kernel<true><<<dim3((ns + 255) / 256, n_frames), 256, 0, s>>>(a);
	LCD_CHECK_LAUNCH(e);
	return LCD_OK;
}

int lcd_shard_similarity_ids_dev(lcd_engine * e, const int * d_word_ids_all, int n_frames, int nq_per_frame, const int * d_sig_ids, int ns,
                                 int * d_pairs_out, int * d_valid_out, void * stream)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(set_device(e));
	if (!d_word_ids_all || !d_sig_ids || !d_pairs_out || !d_valid_out || n_frames <= 0 || ns <= 0) LCD_FAIL(e, LCD_ERR_INVALID, "null argument");
	if (nq_per_frame <= 0 || nq_per_frame > kMaxFrameQueries) LCD_FAIL(e, LCD_ERR_CAPACITY, "1..%d words per signature", kMaxFrameQueries);
	cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : e->stream;
	const ShardIds local{n_frames, 0, n_frames};
	LCD_TRY(prep_ids(e, d_word_ids_all, n_frames, nq_per_frame, 0, 1, true, s, &local));
	return score_pairs(e, n_frames, nq_per_frame, d_sig_ids, ns, n_frames, d_pairs_out, d_valid_out, 0, s);
}

int lcd_shard_similarity_finalize_dev(lcd_engine * e, const int * d_pairs, const int * d_valid, const int * d_word_ids, int n_frames, int nq_per_frame,
                                      const float * d_frame_gdesc, const float * d_map_gdesc, const int * d_map_gdesc_row, int n_map_rows, int dim,
                                      const int * d_sig_ids, int ns, float * d_likelihood_out, void * stream)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(set_device(e));
	if (!d_pairs || !d_valid || !d_word_ids || !d_sig_ids || !d_likelihood_out || n_frames <= 0 || ns <= 0) LCD_FAIL(e, LCD_ERR_INVALID, "null argument");
	if (nq_per_frame <= 0 || nq_per_frame > kMaxFrameQueries) LCD_FAIL(e, LCD_ERR_CAPACITY, "1..%d words per signature", kMaxFrameQueries);
	cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : e->stream;
	const ShardGdesc g{d_frame_gdesc, d_map_gdesc, d_map_gdesc_row, n_map_rows, dim};
	LCD_TRY(shard_check_gdesc(e, g, ns, s));
	bool gd = false;
	LCD_TRY(shard_similarity_prepare(e, n_frames, nq_per_frame, d_word_ids, g, d_sig_ids, ns, &gd, s));
	return shard_similarity_finalize(e, 0, n_frames, d_pairs, d_valid, g, gd, d_sig_ids, ns, d_likelihood_out, s);
}

// ---- mapping mode: Memory::update for a stream of frames ------------------------------------------------------------------
int lcd_map_detect_async(lcd_engine * e, const uint8_t * image, int width, int height, int channels, const void * depth, int depth_type,
                         const lcd_orb_params * params)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(set_device(e));
	if (!image || width <= 0 || height <= 0 || !params) LCD_FAIL(e, LCD_ERR_INVALID, "null image");
	if (e->map_busy >= 2) LCD_FAIL(e, LCD_ERR_STATE, "two detections are already in flight: call lcd_map_frame first");
	const int cap = params->n_features;
	lcd_engine::MapSlot & ms = e->map_slots[(e->map_head + e->map_busy) & 1];
	cudaStream_t s = e->orb_stream;
	if (!ms.done) LCD_CUDA(e, cudaEventCreateWithFlags(&ms.done, cudaEventDisableTiming));
	LCD_TRY(frame_front_end(e, 1, cap, ms.kp, ms.desc, ms.xyz, nullptr, ms.n, s));
	LCD_TRY(upload_frames(e, 1, width, height, channels, image, depth, depth_type, ms.img, ms.depth, s));
	LCD_CUDA(e, ms.h_n.reserve(1));
	LCD_CUDA(e, ms.h_overflow.reserve(1));
	LCD_TRY(orb_run(e, 1, ms.img.p, width, height, channels, depth_type != LCD_DEPTH_NONE ? ms.depth.p : nullptr, depth_type, params, cap, ms.kp.p, ms.desc.p,
	                ms.xyz.p, nullptr, ms.n.p, s));
	LCD_CUDA(e, cudaMemcpyAsync(ms.h_n.p, ms.n.p, sizeof(int), cudaMemcpyDeviceToHost, s));
	LCD_CUDA(e, cudaMemcpyAsync(ms.h_overflow.p, e->o_overflow.p, sizeof(int), cudaMemcpyDeviceToHost, s));
	LCD_CUDA(e, cudaEventRecord(ms.done, s));
	ms.cap = cap;
	ms.detector = e->detector;
	ms.busy = true;
	++e->map_busy;
	return LCD_OK;
}

int lcd_map_frame(lcd_engine * e, int sig_id, int incremental, float nndr, int new_words_compared_together, const int * wm_sig_ids, int ns,
                  int n_total, int * n_kp_out, lcd_keypoint * kp_out, uint8_t * desc_out, float * xyz_out, int * word_ids_out, int * n_new_out,
                  float * likelihood_out)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(set_device(e));
	if (e->map_busy <= 0) LCD_FAIL(e, LCD_ERR_STATE, "no detection in flight: call lcd_map_detect_async first");
	if (!word_ids_out) LCD_FAIL(e, LCD_ERR_INVALID, "null output");
	LCD_TRY(check_n_total(e, n_total)); // before the detection is taken: the call can be repeated with a valid N
	lcd_engine::MapSlot & ms = e->map_slots[e->map_head];
	cudaStream_t s = e->stream;
	// Memory::preUpdate: the words of the previous frame join the index (VWDictionary::update)
	LCD_TRY(lcd_dict_update(e));
	LCD_CUDA(e, cudaStreamWaitEvent(s, ms.done, 0));
	const int cap = ms.cap;
	int n_new = 0, n_kp = 0;
	bool bad = false;
	int rc = LCD_OK;
	if (!limit_active(e))
	{
		// Memory::createSignature: quantise the frame's descriptors (they never leave the device), references for sig_id
		rc = quantize_dev(e, reinterpret_cast<const uint32_t *>(ms.desc.p), cap, -1, ms.n.p, sig_id, incremental, nndr, new_words_compared_together,
		                  word_ids_out, &n_new, &n_kp, s);
	}
	else
	{
		// the same with the split (limit.cuh): the strongest rows are quantised, the others get -1, -2, ...; the references are those of
		// the quantised words, ni grows by the keypoint count (Memory::getNi counts every word of the signature)
		auto split = [&]() -> int {
			LCD_CUDA(e, cudaEventSynchronize(ms.done));
			n_kp = std::min(std::max(*ms.h_n.p, 0), cap);
			bad = n_kp < e->ql_gate;
			if (bad)
			{
				for (int i = 0; i < cap; ++i) word_ids_out[i] = i < n_kp ? -(1 + i) : 0;
			}
			else
			{
				const int k = limit_rows(e, cap);
				LCD_TRY(limit_to_engine(e, 1, cap, ms.kp.p, ms.n.p, reinterpret_cast<const uint32_t *>(ms.desc.p), s));
				LCD_CUDA(e, e->ql_words.reserve(cap, 0, false, s));
				std::vector<int> words_q(k);
				LCD_TRY(quantize_dev(e, e->ql_desc.p, k, -1, e->ql_n.p, 0, incremental, nndr, new_words_compared_together, words_q.data(), &n_new, nullptr, s));
				LCD_TRY(launch_expand(e, 1, cap, k, ms.n.p, e->ql_index.p, e->ql_n.p, e->d_word_ids.p, e->ql_words.p, s));
				LCD_CUDA(e, cudaMemcpyAsync(word_ids_out, e->ql_words.p, cap * sizeof(int), cudaMemcpyDeviceToHost, s));
				LCD_CUDA(e, cudaStreamSynchronize(s));
			}
			return sig_id > 0 ? add_refs_impl(e, sig_id, word_ids_out, n_kp) : LCD_OK;
		};
		rc = split();
	}
	e->map_head ^= 1;
	--e->map_busy;
	ms.busy = false;
	if (rc != LCD_OK) return rc;
	LCD_TRY(overflow_report(e, *ms.h_overflow.p, ms.detector));
	if (n_kp_out) *n_kp_out = n_kp;
	if (n_new_out) *n_new_out = n_new;
	if (kp_out) LCD_CUDA(e, cudaMemcpyAsync(kp_out, ms.kp.p, static_cast<size_t>(n_kp) * sizeof(OrbKeypoint), cudaMemcpyDeviceToHost, s));
	if (desc_out) LCD_CUDA(e, cudaMemcpyAsync(desc_out, ms.desc.p, static_cast<size_t>(n_kp) * 32, cudaMemcpyDeviceToHost, s));
	if (xyz_out) LCD_CUDA(e, cudaMemcpyAsync(xyz_out, ms.xyz.p, static_cast<size_t>(n_kp) * 3 * sizeof(float), cudaMemcpyDeviceToHost, s));
	// Memory::computeLikelihood against the working memory (Rtabmap::process computes none for a bad signature: zeros)
	if (bad && likelihood_out && wm_sig_ids && ns > 0) std::fill(likelihood_out, likelihood_out + ns, 0.0f);
	else if (likelihood_out && wm_sig_ids && ns > 0 && n_kp > 0) return lcd_index_score(e, word_ids_out, n_kp, wm_sig_ids, ns, n_total, likelihood_out);
	LCD_CUDA(e, cudaStreamSynchronize(s));
	return LCD_OK;
}

// ---- NCCL inside the library: communicator + the fused sharded step ------------------------------------------------
int lcd_shard_unique_id(char id_out[128])
{
	static_assert(sizeof(ncclUniqueId) == 128, "ncclUniqueId is 128 bytes");
	if (!id_out) return LCD_ERR_INVALID;
	if (!nccl_api().ok)
	{
		g_create_error = nccl_api().why;
		return LCD_ERR_STATE;
	}
	ncclUniqueId id;
	if (nccl_api().GetUniqueId(&id) != ncclSuccess)
	{
		g_create_error = "ncclGetUniqueId failed";
		return LCD_ERR_CUDA;
	}
	memcpy(id_out, &id, 128);
	return LCD_OK;
}

// LCD_SHARD_TRACE=2: sixteen steps of per-stage events recorded without any synchronisation, printed after the sixteenth
static int shard_record(lcd_engine * e, int h, int k, cudaStream_t st)
{
	LCD_CUDA(e, cudaEventRecord(e->sh_ev[h][k], st));
	if (e->sh_trace == 2 && e->sh_ring_step < 16) LCD_CUDA(e, cudaEventRecord(e->sh_ring[(e->sh_ring_step * 2 + h) * 9 + k], st));
	return LCD_OK;
}

static int shard_comm_common(lcd_engine * e, int rank, int n_ranks)
{
	if (!e->comm_stream) LCD_CUDA(e, cudaStreamCreateWithFlags(&e->comm_stream, cudaStreamNonBlocking));
	e->sh_trace = env_int("LCD_SHARD_TRACE", 0);
	if (e->sh_trace == 2 && e->sh_ring.empty())
	{
		e->sh_ring.assign(16 * 2 * 9, nullptr);
		for (cudaEvent_t & ev : e->sh_ring) LCD_CUDA(e, cudaEventCreate(&ev));
	}
	for (auto & half : e->sh_ev)
		for (cudaEvent_t & ev : half)
			if (!ev) LCD_CUDA(e, cudaEventCreateWithFlags(&ev, e->sh_trace ? cudaEventDefault : cudaEventDisableTiming));
	for (cudaEvent_t & ev : e->sh_tr)
		if (e->sh_trace && !ev) LCD_CUDA(e, cudaEventCreate(&ev));
	e->sh_rank = rank;
	e->sh_ranks = n_ranks;
	return LCD_OK;
}

int lcd_shard_comm_init(lcd_engine * e, const char id[128], int rank, int n_ranks)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(set_device(e));
	if (!id || n_ranks < 1 || rank < 0 || rank >= n_ranks) LCD_FAIL(e, LCD_ERR_INVALID, "bad rank %d of %d", rank, n_ranks);
	if (!nccl_api().ok) LCD_FAIL(e, LCD_ERR_STATE, "%s", nccl_api().why.c_str());
	if (e->comm) LCD_FAIL(e, LCD_ERR_STATE, "the engine already has a communicator");
	ncclUniqueId uid;
	memcpy(&uid, id, 128);
	LCD_NCCL(e, nccl_api().CommInitRank(&e->comm, n_ranks, uid, rank));
	e->comm_owned = true;
	return shard_comm_common(e, rank, n_ranks);
}

int lcd_shard_comm_adopt(lcd_engine * e, void * nccl_comm, int rank, int n_ranks)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(set_device(e));
	if (!nccl_comm || n_ranks < 1 || rank < 0 || rank >= n_ranks) LCD_FAIL(e, LCD_ERR_INVALID, "bad communicator / rank");
	if (!nccl_api().ok) LCD_FAIL(e, LCD_ERR_STATE, "%s", nccl_api().why.c_str());
	if (e->comm) LCD_FAIL(e, LCD_ERR_STATE, "the engine already has a communicator");
	e->comm = static_cast<ncclComm_t>(nccl_comm);
	e->comm_owned = false;
	return shard_comm_common(e, rank, n_ranks);
}

int lcd_shard_comm_destroy(lcd_engine * e)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(set_device(e));
	if (e->comm)
	{
		LCD_CUDA(e, cudaDeviceSynchronize());
		if (e->comm_owned) nccl_api().CommDestroy(e->comm);
		e->comm = nullptr;
	}
	e->sh_ranks = 1;
	e->sh_rank = 0;
	return LCD_OK;
}

// The exchange body of one sharded step, shared by lcd_shard_process_frames_dev, lcd_shard_localize_batch_dev and
// lcd_shard_localize_similarity_batch_dev.  desc: the n_frames local frames of `cap` descriptor rows each (e->nw * 4 bytes per row); n_local:
// valid rows of each local frame, or nullptr (full frames).  `detect` runs first on the compute stream and produces desc / n_local (ORB);
// `finish` runs after the likelihood of the local frames (verification).  Either may be empty.  Keys are exchanged as two u32 (binary) or
// two u64 (float) per query.  sim: nullptr = the TF-IDF likelihood; else the similarity likelihood, whose phase 4 counts word pairs instead
// of TF-IDF terms and reduce-scatters int32 counts with this rank's valid(s) row folded into every rank's segment.
using ShardHook = std::function<int(cudaStream_t)>;

static int shard_step(lcd_engine * e, int n_frames, int cap, const uint8_t * desc, const int * n_local, const ShardHook & detect, const ShardHook & finish,
                      int incremental, float nndr, int new_words_compared_together, const int * d_sig_ids, int ns, int n_total,
                      const int * d_row_ids_global, int last_word_id, int * d_word_ids_out, float * d_likelihood_out, cudaStream_t s,
                      const ShardGdesc * sim = nullptr)
{
	const NcclApi & nc = nccl_api();
	cudaStream_t c = e->comm_stream;
	const int G = e->sh_ranks, R = e->sh_rank;
	const size_t row_bytes = static_cast<size_t>(e->nw) * 4;
	const size_t kw = shard_key_words(e);                               // u32 words of one query's key pair
	const ncclDataType_t key_type = e->f32 ? ncclUint64 : ncclUint32; // two keys of this type per query
	// The dictionary search runs on two halves of the local batch, so that the descriptor all-gather of the second half and the key
	// exchange of the first run under a search kernel.  The merge + NNDR stage is a one-CTA-per-frame kernel that takes as long for half a
	// batch as for a whole one, so it runs once on the whole batch and its exchange (word ids) is exposed: measured cheaper than splitting.
	const int n_parts = n_frames >= 2 && env_int("LCD_SHARD_NN_PARTS", 2) >= 2 ? 2 : 1;
	const int part_frames[2] = {n_parts == 2 ? (n_frames + 1) / 2 : n_frames, n_parts == 2 ? n_frames / 2 : 0};
	const int part_f0[2] = {0, part_frames[0]};
	// merge + NNDR always runs on the whole batch; the TF-IDF stage scores G x n_frames frames, so from 4 ranks on it is no longer a
	// single-wave kernel and is split in two halves of every rank's frames: the reduce-scatter of the first half runs under the scoring of
	// the second (LCD_SHARD_SCORE_PARTS=1|2 overrides)
	const int s_parts_env = env_int("LCD_SHARD_SCORE_PARTS", 0);
	const int s_parts = n_frames >= 2 && (s_parts_env ? s_parts_env >= 2 : G >= 4) ? 2 : 1;
	const int score_frames[2] = {s_parts == 2 ? (n_frames + 1) / 2 : n_frames, s_parts == 2 ? n_frames / 2 : 0};
	const int score_f0[2] = {0, score_frames[0]};
	const size_t rows = static_cast<size_t>(n_frames) * cap;
	if (n_local) LCD_CUDA(e, e->sh_n_all.reserve(static_cast<size_t>(G) * n_frames, 0, false, s));
	for (int h = 0; h < n_parts; ++h)
	{
		const size_t pr = static_cast<size_t>(part_frames[h]) * cap; // descriptor rows of this part on one rank
		LCD_CUDA(e, e->sh_desc_all[h].reserve(pr * row_bytes * G, 0, false, s));
		LCD_CUDA(e, e->sh_keys[h].reserve(pr * kw * G, 0, false, s));
	}
	LCD_CUDA(e, e->sh_keys_mine.reserve(rows * kw * G, 0, false, s)); // [rank][local frame][feature]: both halves land in one array
	LCD_CUDA(e, e->sh_words_loc.reserve(rows, 0, false, s));
	LCD_CUDA(e, e->sh_words_all.reserve(rows * G, 0, false, s));
	for (int h = 0; h < s_parts; ++h)
	{
		if (sim)
		{
			LCD_CUDA(e, e->sh_pairs[h].reserve(static_cast<size_t>(score_frames[h] + 1) * G * ns, 0, false, s));
			LCD_CUDA(e, e->sh_pairs_loc[h].reserve(static_cast<size_t>(score_frames[h] + 1) * ns, 0, false, s));
			continue;
		}
		LCD_CUDA(e, e->sh_scores[h].reserve(static_cast<size_t>(score_frames[h]) * G * ns, 0, false, s));
		LCD_CUDA(e, e->sh_scores_loc[h].reserve(static_cast<size_t>(score_frames[h]) * ns, 0, false, s));
	}
	std::chrono::steady_clock::time_point host_t[6];
	const auto host_begin = std::chrono::steady_clock::now();
	if (e->sh_trace == 1 && e->sh_trace_armed)
	{
		// timeline of the PREVIOUS step, in ms after its first kernel: per half, the end of each compute stage (s) and exchange (c)
		LCD_CUDA(e, cudaEventSynchronize(e->sh_tr[1]));
		LCD_CUDA(e, cudaStreamSynchronize(c));
		static const char * names[8] = {"orb", "ag_desc", "nn", "a2a_keys", "resolve", "ag_words", "score", "rs_scores"};
		float ms = 0.f;
		fprintf(stderr, "[lcd shard trace rank %d]", R);
		for (int h = 0; h < n_parts; ++h)
			for (int k = 0; k < 8; ++k)
				if ((k < 4 || (k < 6 ? h == 0 : h < s_parts)) && cudaEventElapsedTime(&ms, e->sh_tr[0], e->sh_ev[h][k]) == cudaSuccess) fprintf(stderr, " %s%d=%.3f", names[k], h, ms);
		if (cudaEventElapsedTime(&ms, e->sh_tr[0], e->sh_tr[1]) == cudaSuccess) fprintf(stderr, " end=%.3f", ms);
		fprintf(stderr, "\n");
	}
	if (e->sh_trace) LCD_CUDA(e, cudaEventRecord(e->sh_tr[0], s));
	if (e->sh_trace == 2 && e->sh_ring_step < 16) LCD_CUDA(e, cudaEventRecord(e->sh_ring[(e->sh_ring_step * 2 + 0) * 9 + 8], s));
	// the communication stream starts behind everything already queued on the compute stream
	LCD_CUDA(e, cudaEventRecord(e->sh_ev[0][7], s));
	LCD_CUDA(e, cudaStreamWaitEvent(c, e->sh_ev[0][7], 0));

	host_t[0] = std::chrono::steady_clock::now();
	// phase 1: the local descriptors (detected here in one pass when `detect` is given: splitting detection costs more than the 30-50 us
	// all-gather it would hide), then all-gather of the descriptors part by part (and of the per-frame counts): the second part's exchange
	// runs under the first part's search
	if (detect) LCD_TRY(detect(s));
	for (int h = 0; h < n_parts; ++h)
	{
		LCD_TRY(shard_record(e, h, 0, s));
		LCD_CUDA(e, cudaStreamWaitEvent(c, e->sh_ev[h][0], 0));
		const size_t pr = static_cast<size_t>(part_frames[h]) * cap;
		LCD_NCCL(e, nc.GroupStart());
		LCD_NCCL(e, nc.AllGather(desc + static_cast<size_t>(part_f0[h]) * cap * row_bytes, e->sh_desc_all[h].p, pr * row_bytes, ncclUint8, e->comm, c));
		if (h == n_parts - 1 && n_local) LCD_NCCL(e, nc.AllGather(n_local, e->sh_n_all.p, n_frames, ncclInt32, e->comm, c));
		LCD_NCCL(e, nc.GroupEnd());
		LCD_TRY(shard_record(e, h, 1, c));
	}
	host_t[1] = std::chrono::steady_clock::now();
	// phase 2: top-2 keys of every rank's descriptors over the local word range; every rank gets back the keys of ITS frames
	for (int h = 0; h < n_parts; ++h)
	{
		const size_t pr = static_cast<size_t>(part_frames[h]) * cap;
		const int nq_all = static_cast<int>(pr) * G;
		LCD_CUDA(e, cudaStreamWaitEvent(s, e->sh_ev[h][1], 0));
		int n_chunks = 0;
		LCD_TRY(run_knn(e, reinterpret_cast<const uint32_t *>(e->sh_desc_all[h].p), nq_all, e->n_indexed, &n_chunks, s));
		LCD_TRY(shard_merge_keys(e, n_chunks, nq_all, e->sh_keys[h].p, s));
		LCD_TRY(shard_record(e, h, 2, s));
		LCD_CUDA(e, cudaStreamWaitEvent(c, e->sh_ev[h][2], 0));
		LCD_NCCL(e, nc.GroupStart());
		for (int p = 0; p < G; ++p)
		{
			LCD_NCCL(e, nc.Send(e->sh_keys[h].p + static_cast<size_t>(p) * pr * kw, pr * 2, key_type, p, e->comm, c));
			LCD_NCCL(e, nc.Recv(e->sh_keys_mine.p + (static_cast<size_t>(p) * rows + static_cast<size_t>(part_f0[h]) * cap) * kw, pr * 2, key_type, p, e->comm, c));
		}
		LCD_NCCL(e, nc.GroupEnd());
		LCD_TRY(shard_record(e, h, 3, c));
	}
	host_t[2] = std::chrono::steady_clock::now();
	// phase 3: merge + NNDR / new-word pass of the local frames, all-gather of their word ids
	LCD_CUDA(e, cudaStreamWaitEvent(s, e->sh_ev[n_parts - 1][3], 0));
	// nq_total = rows: the stride between the G key sets
	ResolveArgs a = resolve_args(e, reinterpret_cast<const uint32_t *>(desc), cap, static_cast<int>(rows), n_local, G, d_row_ids_global, incremental, nndr,
	                             new_words_compared_together, last_word_id, e->sh_words_loc.p);
	shard_set_keys(e, a, e->sh_keys_mine.p, 0);
	LCD_TRY(launch_resolve(e, a, n_frames, s));
	if (d_word_ids_out) LCD_CUDA(e, cudaMemcpyAsync(d_word_ids_out, e->sh_words_loc.p, rows * sizeof(int), cudaMemcpyDeviceToDevice, s));
	LCD_TRY(shard_record(e, 0, 4, s));
	LCD_CUDA(e, cudaStreamWaitEvent(c, e->sh_ev[0][4], 0));
	LCD_NCCL(e, nc.AllGather(e->sh_words_loc.p, e->sh_words_all.p, rows, ncclInt32, e->comm, c));
	LCD_TRY(shard_record(e, 0, 5, c));
	host_t[3] = std::chrono::steady_clock::now();
	// phase 4: TF-IDF (or word pairs) of every rank's frames over the local word range, reduce-scatter of the exact integer sums
	for (int h = 0; h < s_parts; ++h)
	{
		const int nf_all = score_frames[h] * G; // frames [score_f0, +score_frames) of every rank, rank-major
		LCD_CUDA(e, cudaStreamWaitEvent(s, e->sh_ev[0][5], 0));
		const ShardIds local{n_frames, score_f0[h], score_frames[h]};
		LCD_TRY(prep_ids(e, e->sh_words_all.p, nf_all, cap, n_total, 1, sim != nullptr, s, &local));
		if (sim)
		{
			// [rank][score_frames + 1][ns]: the pair counts of the rank's frames, then this rank's valid(s) in every segment, so that the
			// reduce-scatter that sums the counts sums valid(s) across ranks too (no collective of its own)
			const size_t seg = static_cast<size_t>(score_frames[h] + 1) * ns;
			LCD_TRY(score_pairs(e, nf_all, cap, d_sig_ids, ns, score_frames[h], e->sh_pairs[h].p, e->sh_pairs[h].p + static_cast<size_t>(score_frames[h]) * ns, seg,
			                    s));
			LCD_TRY(shard_record(e, h, 6, s));
			LCD_CUDA(e, cudaStreamWaitEvent(c, e->sh_ev[h][6], 0));
			LCD_NCCL(e, nc.ReduceScatter(e->sh_pairs[h].p, e->sh_pairs_loc[h].p, seg, ncclInt32, ncclSum, e->comm, c));
		}
		else
		{
			LCD_TRY(score_tfidf(e, nf_all, cap, d_sig_ids, ns, e->sh_scores[h].p, s));
			LCD_TRY(shard_record(e, h, 6, s));
			LCD_CUDA(e, cudaStreamWaitEvent(c, e->sh_ev[h][6], 0));
			LCD_NCCL(e, nc.ReduceScatter(e->sh_scores[h].p, e->sh_scores_loc[h].p, static_cast<size_t>(score_frames[h]) * ns, ncclInt64, ncclSum, e->comm, c));
		}
		LCD_TRY(shard_record(e, h, 7, c));
	}
	host_t[4] = std::chrono::steady_clock::now();
	// phase 5: likelihood of the local frames (then `finish`: verification of their top hypothesis).  The similarity variant first
	// counts valid(q) of the local frames and takes their dot products, under the last reduce-scatter.
	bool gd = false;
	if (sim) LCD_TRY(shard_similarity_prepare(e, n_frames, cap, e->sh_words_loc.p, *sim, d_sig_ids, ns, &gd, s));
	for (int h = 0; h < s_parts; ++h)
	{
		const int n = score_frames[h] * ns;
		LCD_CUDA(e, cudaStreamWaitEvent(s, e->sh_ev[h][7], 0));
		if (sim)
		{
			LCD_TRY(shard_similarity_finalize(e, score_f0[h], score_frames[h], e->sh_pairs_loc[h].p, e->sh_pairs_loc[h].p + n, *sim, gd, d_sig_ids, ns,
			                                  d_likelihood_out, s));
			continue;
		}
		fixed_to_float_kernel<<<(n + 255) / 256, 256, 0, s>>>(e->sh_scores_loc[h].p, n, d_likelihood_out + static_cast<size_t>(score_f0[h]) * ns);
		LCD_CHECK_LAUNCH(e);
	}
	if (finish) LCD_TRY(finish(s));
	if (e->sh_trace)
	{
		LCD_CUDA(e, cudaEventRecord(e->sh_tr[1], s));
		e->sh_trace_armed = true;
	}
	host_t[5] = std::chrono::steady_clock::now();
	if (e->sh_trace == 2 && e->sh_ring_step == 9)
	{
		auto us = [](std::chrono::steady_clock::time_point a, std::chrono::steady_clock::time_point b) {
			return std::chrono::duration<double, std::micro>(b - a).count();
		};
		fprintf(stderr, "[lcd shard host rank %d] us: reserve=%.0f orb+ag_desc=%.0f nn+a2a=%.0f resolve+ag_words=%.0f score+rs=%.0f verify=%.0f\n", R,
		        us(host_begin, host_t[0]), us(host_t[0], host_t[1]), us(host_t[1], host_t[2]), us(host_t[2], host_t[3]), us(host_t[3], host_t[4]),
		        us(host_t[4], host_t[5]));
	}
	if (e->sh_trace == 2 && e->sh_ring_step < 16)
	{
		LCD_CUDA(e, cudaEventRecord(e->sh_ring[(e->sh_ring_step * 2 + 1) * 9 + 8], s));
		if (++e->sh_ring_step == 16)
		{
			LCD_CUDA(e, cudaStreamSynchronize(s));
			LCD_CUDA(e, cudaStreamSynchronize(c));
			static const char * names[8] = {"orb", "ag_desc", "nn", "a2a_keys", "resolve", "ag_words", "score", "rs_scores"};
			const cudaEvent_t origin = e->sh_ring[(8 * 2 + 0) * 9 + 8]; // begin of step 8
			for (int st = 8; st < 12; ++st)
			{
				float ms = 0.f;
				fprintf(stderr, "[lcd shard ring rank %d step %d]", R, st);
				if (cudaEventElapsedTime(&ms, origin, e->sh_ring[(st * 2 + 0) * 9 + 8]) == cudaSuccess) fprintf(stderr, " begin=%.3f", ms);
				for (int h = 0; h < n_parts; ++h)
					for (int k = 0; k < 8; ++k)
						if ((k < 4 || (k < 6 ? h == 0 : h < s_parts)) && cudaEventElapsedTime(&ms, origin, e->sh_ring[(st * 2 + h) * 9 + k]) == cudaSuccess) fprintf(stderr, " %s%d=%.3f", names[k], h, ms);
				if (cudaEventElapsedTime(&ms, origin, e->sh_ring[(st * 2 + 1) * 9 + 8]) == cudaSuccess) fprintf(stderr, " end=%.3f", ms);
				fprintf(stderr, "\n");
			}
		}
	}
	return LCD_OK;
}

int lcd_shard_process_frames_dev(lcd_engine * e, int n_frames, const uint8_t * d_images, int width, int height, int channels, const void * d_depth,
                                 int depth_type, const lcd_orb_params * op, int incremental, float nndr, int new_words_compared_together,
                                 const int * d_sig_ids, int ns, int n_total, const int * d_row_ids_global, int last_word_id,
                                 const lcd_verify_params * vp, int * d_word_ids_out, float * d_likelihood_out, void * stream)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(require_binary(e, "lcd_shard_process_frames_dev"));
	LCD_TRY(set_device(e));
	if (!e->comm) LCD_FAIL(e, LCD_ERR_STATE, "no communicator: call lcd_shard_comm_init first");
	if (!d_images || n_frames <= 0 || !op || !d_sig_ids || ns <= 0 || !d_row_ids_global || !d_likelihood_out)
		LCD_FAIL(e, LCD_ERR_INVALID, "null argument");
	LCD_TRY(check_n_total(e, n_total));
	const int cap = op->n_features;
	cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : e->stream;
	LCD_TRY(frame_front_end(e, n_frames, cap, e->o_kp, e->o_desc, e->o_xyz, &e->o_uv, e->o_n, s));
	LCD_CUDA(e, e->d_like.reserve(static_cast<size_t>(n_frames) * ns, 0, false, s));
	// detect + describe the local frames, and after the likelihood verify their top hypothesis
	const ShardHook orb = [&](cudaStream_t st) {
		return orb_run(e, n_frames, d_images, width, height, channels, d_depth, depth_type, op, cap, e->o_kp.p, e->o_desc.p, e->o_xyz.p, e->o_uv.p, e->o_n.p,
		               st);
	};
	const ShardHook verify = [&](cudaStream_t st) {
		return vp ? verify_top_dev(e, reinterpret_cast<const uint32_t *>(e->o_desc.p), e->o_uv.p, n_frames, cap, d_likelihood_out, d_sig_ids, ns, vp, st,
		                           e->o_n.p, e->o_xyz.p)
		          : LCD_OK;
	};
	if (!limit_active(e))
		return shard_step(e, n_frames, cap, e->o_desc.p, e->o_n.p, orb, verify, incremental, nndr, new_words_compared_together, d_sig_ids, ns, n_total,
		                  d_row_ids_global, last_word_id, d_word_ids_out, d_likelihood_out, s);
	// Memory::createSignature's split (limit.cuh): the exchanges and the search carry the k quantised rows of every frame; the word ids
	// are expanded to every detected row and the verification matches them all
	const int k = limit_rows(e, cap);
	// shard_step takes the buffers' addresses before the detect hook runs: they get their size here (the hook's reserve is then a no-op)
	LCD_CUDA(e, e->ql_desc.reserve(static_cast<size_t>(n_frames) * k * e->nw, 0, false, s));
	LCD_CUDA(e, e->ql_index.reserve(static_cast<size_t>(n_frames) * k, 0, false, s));
	LCD_CUDA(e, e->ql_words.reserve(static_cast<size_t>(n_frames) * k, 0, false, s));
	LCD_CUDA(e, e->ql_n.reserve(n_frames, 0, false, s));
	const ShardHook orb_limit = [&](cudaStream_t st) {
		LCD_TRY(orb(st));
		return limit_to_engine(e, n_frames, cap, e->o_kp.p, e->o_n.p, reinterpret_cast<const uint32_t *>(e->o_desc.p), st);
	};
	const ShardHook expand_verify = [&](cudaStream_t st) {
		if (d_word_ids_out) LCD_TRY(launch_expand(e, n_frames, cap, k, e->o_n.p, e->ql_index.p, e->ql_n.p, e->ql_words.p, d_word_ids_out, st));
		return verify(st);
	};
	return shard_step(e, n_frames, k, reinterpret_cast<const uint8_t *>(e->ql_desc.p), e->ql_n.p, orb_limit, expand_verify, incremental, nndr,
	                  new_words_compared_together, d_sig_ids, ns, n_total, d_row_ids_global, last_word_id, d_word_ids_out ? e->ql_words.p : nullptr,
	                  d_likelihood_out, s);
}

int lcd_shard_localize_batch_dev(lcd_engine * e, const void * d_queries, int n_frames, int nq_per_frame, int incremental, float nndr,
                                 int new_words_compared_together, const int * d_sig_ids, int ns, int n_total, const int * d_row_ids_global,
                                 int last_word_id, int * d_word_ids_out, float * d_likelihood_out, void * stream)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(set_device(e));
	if (!e->comm) LCD_FAIL(e, LCD_ERR_STATE, "no communicator: call lcd_shard_comm_init first");
	if (!d_queries || n_frames <= 0 || !d_sig_ids || ns <= 0 || !d_row_ids_global || !d_likelihood_out)
		LCD_FAIL(e, LCD_ERR_INVALID, "null argument");
	if (nq_per_frame <= 0 || nq_per_frame > kMaxFrameQueries) LCD_FAIL(e, LCD_ERR_CAPACITY, "1..%d descriptors per frame", kMaxFrameQueries);
	LCD_TRY(check_n_total(e, n_total));
	cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : e->stream;
	return shard_step(e, n_frames, nq_per_frame, static_cast<const uint8_t *>(d_queries), nullptr, ShardHook(), ShardHook(), incremental, nndr,
	                  new_words_compared_together, d_sig_ids, ns, n_total, d_row_ids_global, last_word_id, d_word_ids_out, d_likelihood_out, s);
}

int lcd_shard_localize_similarity_batch_dev(lcd_engine * e, const void * d_queries, int n_frames, int nq_per_frame, int incremental, float nndr,
                                            int new_words_compared_together, const float * d_frame_gdesc, const float * d_map_gdesc,
                                            const int * d_map_gdesc_row, int n_map_rows, int dim, const int * d_sig_ids, int ns,
                                            const int * d_row_ids_global, int last_word_id, int * d_word_ids_out, float * d_likelihood_out, void * stream)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(set_device(e));
	if (!e->comm) LCD_FAIL(e, LCD_ERR_STATE, "no communicator: call lcd_shard_comm_init first");
	if (!d_queries || n_frames <= 0 || !d_sig_ids || ns <= 0 || !d_row_ids_global || !d_likelihood_out)
		LCD_FAIL(e, LCD_ERR_INVALID, "null argument");
	if (nq_per_frame <= 0 || nq_per_frame > kMaxFrameQueries) LCD_FAIL(e, LCD_ERR_CAPACITY, "1..%d descriptors per frame", kMaxFrameQueries);
	cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : e->stream;
	const ShardGdesc g{d_frame_gdesc, d_map_gdesc, d_map_gdesc_row, n_map_rows, dim};
	LCD_TRY(shard_check_gdesc(e, g, ns, s));
	return shard_step(e, n_frames, nq_per_frame, static_cast<const uint8_t *>(d_queries), nullptr, ShardHook(), ShardHook(), incremental, nndr,
	                  new_words_compared_together, d_sig_ids, ns, 0, d_row_ids_global, last_word_id, d_word_ids_out, d_likelihood_out, s, &g);
}

int lcd_shard_finalize_dev(lcd_engine * e, const long long * d_scores, int n, float * d_likelihood_out, void * stream)
{
	if (!e) return LCD_ERR_INVALID;
	LCD_TRY(set_device(e));
	if (!d_scores || !d_likelihood_out || n <= 0) LCD_FAIL(e, LCD_ERR_INVALID, "null argument");
	cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : e->stream;
	fixed_to_float_kernel<<<(n + 255) / 256, 256, 0, s>>>(d_scores, n, d_likelihood_out);
	LCD_CHECK_LAUNCH(e);
	return LCD_OK;
}

} // extern "C"
