/*
 * lcd_b200.h — C ABI of the H100-native loop-closure hot path
 * (detect -> quantise -> score -> verify) that drops in behind
 * rtabmap::Memory / VWDictionary / Signature / Feature2D.
 *
 * RTAB-Map has no C ABI or plugin loader for this path (SURVEY.md §8(b)); its
 * seams are C++ virtuals owned by rtabmap::Memory.  Every entry point below
 * names the reference member function (file:line under corelib/) whose work it
 * replaces.  INTEGRATION.md shows the two shim classes (VWDictionaryB200,
 * ORB_B200) a maintainer adds on the reference side to bind these symbols.
 *
 * Conventions (mirroring the reference's, SURVEY.md §8(b)):
 *   - all functions return 0 on success, <0 on error (never throw); the message
 *     is available through lcd_last_error(engine)  [reference: UERROR + empty
 *     return, VWDictionary.cpp:920-957];
 *   - all buffers are caller-owned HOST pointers, row-major, unless the function
 *     name ends in _dev (device pointers valid on the engine's device);
 *   - word ids are positive ints, 0 = invalid / no match; signature ids are
 *     positive ints (VWDictionary.cpp:875-878, Memory.cpp:6040-6058);
 *   - one engine = one VWDictionary instance + its inverted index on one GPU;
 *     several engines may coexist (RegistrationVis builds temporary
 *     dictionaries, RegistrationVis.cpp:1482-1503);
 *   - calls on one engine must be serialised by the caller, with ONE exception:
 *     the host-buffer lcd_orb_detect_describe may run on a second thread while
 *     lcd_dict_update runs (the reference runs VWDictionary::update() on
 *     PreUpdateThread beside feature extraction, Memory.cpp:5284, :5926).  The two
 *     calls share no buffers, run on different CUDA streams, and the counters they
 *     both touch are atomic (tests/test_gpu_concurrency.py).  lcd_profile_enable(1)
 *     suspends that exception (its event lists are not thread-safe);
 *   - the *_dev entry points of one engine must all be given the same stream (or
 *     NULL): scratch buffers are shared between them.
 */
#ifndef LCD_B200_H
#define LCD_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define LCD_OK 0
#define LCD_ERR_INVALID (-1)  /* bad argument / size or type mismatch            */
#define LCD_ERR_CUDA (-2)     /* CUDA runtime failure (message has the detail)   */
#define LCD_ERR_CAPACITY (-3) /* a configured capacity would be exceeded         */
#define LCD_ERR_STATE (-4)    /* call not valid in the current state             */

/* descriptor types: cv::Mat type()/cols of VisualWord::getDescriptor()
 * (VWDictionary.cpp:933-957 checks) */
#define LCD_DESC_U8 0  /* CV_8U rows, desc_dim bytes (ORB/BRIEF: 32)  -> Hamming   */
#define LCD_DESC_F32 1 /* CV_32F rows, desc_dim floats (SURF: 64/128, SIFT: 128, SuperPoint: 256) -> squared L2 */

typedef struct lcd_engine lcd_engine;

typedef struct lcd_config {
	int device;         /* CUDA device ordinal                                          */
	int desc_type;      /* LCD_DESC_U8 | LCD_DESC_F32                                   */
	int desc_dim;       /* bytes (U8: 16/32/64) or floats (F32: 64/128/256)             */
	int max_words;      /* initial capacity hint for vocabulary rows (grows)            */
	int max_signatures; /* initial capacity hint for signature ids (grows)              */
	int max_queries;    /* max descriptors per lcd_dict_* call / per frame (<= 4096)    */
	int max_batch;      /* max frames per lcd_localize_batch call                       */
} lcd_config;

/* ---- lifetime ---------------------------------------------------------------- */
/* replaces: VWDictionary::VWDictionary / ~VWDictionary (VWDictionary.cpp:56-120) */
lcd_engine * lcd_create(const lcd_config * cfg);
void lcd_destroy(lcd_engine * e);
/* last error text of this engine (e may be NULL: error of the last failed lcd_create) */
const char * lcd_last_error(const lcd_engine * e);
/* library/ABI version, and the name of the CUDA arch the kernels were built for */
int lcd_abi_version(void); /* 2: lcd_verify_params / lcd_verify_result grew (covariance), lcd_verify_batch takes xyz_to */
const char * lcd_build_arch(void);
/* number of kernels this engine has launched since creation (bench "gpu_launches") */
long long lcd_launch_count(const lcd_engine * e);

/* ---- detect: Feature2D (ORB) ---------------------------------------------------------------
 * cv::KeyPoint fields the reference uses (Signature keypoints, Features2d.cpp:1657). */
typedef struct lcd_keypoint {
	float x, y;      /* pt, level-0 pixel coordinates */
	float size;      /* patchSize * scale of the level */
	float angle;     /* degrees, intensity-centroid orientation */
	float response;  /* Harris response */
	int octave;      /* pyramid level */
} lcd_keypoint;

typedef struct lcd_orb_params {
	int n_features;       /* Kp/MaxFeatures: nfeatures of cv::ORB and the limit of Feature2D::limitKeypoints */
	int n_levels;         /* ORB/NLevels (1..4) */
	float scale_factor;   /* ORB/ScaleFactor: 2.0 (the reference default) is the only value implemented */
	int edge_threshold;   /* ORB/EdgeThreshold (19) */
	int fast_threshold;   /* FAST/Threshold (20), 0..255 (cv::ORB wraps other values modulo 256; they are rejected here) */
	int patch_size;       /* ORB/PatchSize: 31 (the learned rBRIEF pattern) */
	float min_depth;      /* Kp/MinDepth */
	float max_depth;      /* Kp/MaxDepth (0 = unlimited) */
	int depth_as_mask;    /* Mem/DepthAsMask */
	float fx, fy, cx, cy; /* CameraModel of the frame (depth registered to the image, same size) */
} lcd_orb_params;

#define LCD_DEPTH_NONE 0
#define LCD_DEPTH_U16_MM 1 /* CV_16UC1, millimetres */
#define LCD_DEPTH_F32_M 2  /* CV_32FC1, metres     */
#define LCD_DEPTH_MASK_U8 3 /* not a depth image: the CV_8UC1 mask (0 / 255) Feature2D::generateKeypoints hands to
                               generateKeypointsImpl (Features2d.cpp:783-857); no 3-D points are produced */

/* replaces, for Kp/DetectorStrategy=2: cv::cvtColor(BGR2GRAY) (Memory.cpp:5447),
 * Feature2D::generateKeypoints incl. the depth mask and limitKeypoints (Features2d.cpp:775-878, :356-399)
 * -> cv::ORB::detect, Feature2D::generateDescriptors -> cv::ORB::compute (Features2d.cpp:1663-1718) and
 * Feature2D::generateKeypoints3D -> util3d::generateKeypoints3DDepth (util3d_features.cpp:67-120), for
 * n_frames images [n_frames][height][width][channels] (channels 1 = gray, 3 = BGR) with optional depth
 * [n_frames][height][width].  Outputs hold `cap` rows per frame: kp_out[n_frames*cap],
 * desc_out[n_frames*cap*32], xyz_out[n_frames*cap*3] (NaN = no depth), n_out[n_frames] valid rows. */
int lcd_orb_detect_describe(lcd_engine * e, int n_frames, const uint8_t * images, int width, int height, int channels,
                            const void * depth, int depth_type, const lcd_orb_params * params, int cap,
                            lcd_keypoint * kp_out, uint8_t * desc_out, float * xyz_out, int * n_out);
/* same with device-resident inputs and outputs (any output may be NULL), asynchronous on `stream`;
 * d_uv_out[n_frames*cap*2] optionally receives the keypoint coordinates as a plain float2 array. */
int lcd_orb_detect_describe_dev(lcd_engine * e, int n_frames, const uint8_t * d_images, int width, int height, int channels,
                                const void * d_depth, int depth_type, const lcd_orb_params * params, int cap,
                                lcd_keypoint * d_kp_out, uint8_t * d_desc_out, float * d_xyz_out, float * d_uv_out,
                                int * d_n_out, void * stream);
/* 1 if the last lcd_orb_* / lcd_process_frames* call on this engine truncated a FAST candidate list (more than 16 384 corners in
 * level 0, half as many per further level), else 0; synchronises the device.  The host-buffer entry points report the condition
 * themselves (LCD_ERR_CAPACITY); the *_dev variants return before the kernels ran, so their callers ask here. */
int lcd_orb_overflow(lcd_engine * e);
/* Which kernels the last detection used (bit flags; diagnostics for tests and benchmarks): 1 = FAST and blur tiles staged by TMA with a
 * tensor map (rows a multiple of 16 bytes), 2 = descriptors from shared-memory patches (rows a multiple of 4 bytes on every level, edge
 * threshold >= 19), 4 = vectorised gray / mask preparation (rows a multiple of 8 pixels, even height), 8 = the GFTT/ORB detector
 * (lcd_detector_set), 16 = the ORB-OCTREE detector (lcd_detector_set_orb_octree; no other bit is set then).  0 = the general kernels. */
int lcd_orb_last_path(const lcd_engine * e);

/* ---- detect: the detector of every image-level call -----------------------------------------
 * LCD_DETECTOR_ORB (the default): Kp/DetectorStrategy=2, FAST corners on the ORB pyramid, as above.
 * LCD_DETECTOR_GFTT_ORB: Kp/DetectorStrategy=8 (RTAB-Map's default), rtabmap::GFTT_ORB (Features2d.cpp:2141-2178, :2352-2356):
 * cv::GFTTDetector(Kp/MaxFeatures, GFTT/QualityLevel, GFTT/MinDistance, GFTT/BlockSize, GFTT/UseHarrisDetector, GFTT/K) on the
 * level-0 gray image and depth mask, then cv::ORB::compute on the kept corners (corners within ORB/EdgeThreshold of the border are
 * dropped, the order is kept, descriptors are steered by the corners' angle of -1 degree).  Keypoints carry size = GFTT/BlockSize,
 * angle = -1, response = the minimum eigenvalue, octave = 0.  lcd_orb_params still supplies n_features, edge_threshold, patch_size and
 * the depth fields.  Once selected, lcd_orb_detect_describe[_dev], lcd_process_frames[_submit|_dev], lcd_map_detect_async and
 * lcd_shard_process_frames_dev all detect GFTT/ORB.  Width and height must be even; more than 65 536 local maxima above the quality
 * threshold in a frame truncate its candidate list, reported as for FAST (lcd_orb_overflow, LCD_ERR_CAPACITY). */
#define LCD_DETECTOR_ORB 2
#define LCD_DETECTOR_GFTT_ORB 8
typedef struct lcd_gftt_params {
	double quality_level; /* GFTT/QualityLevel (0.001): must be > 0 */
	double min_distance;  /* GFTT/MinDistance (7): must be >= 0; below 1 no distance filter */
	int block_size;       /* GFTT/BlockSize: 3 is the only value implemented */
	int use_harris;       /* GFTT/UseHarrisDetector: 0 is the only value implemented */
	double k;             /* GFTT/K (0.04): unused without the Harris detector */
} lcd_gftt_params;
/* Select the detector.  `params` is read for LCD_DETECTOR_GFTT_ORB (NULL = the defaults above) and ignored for LCD_DETECTOR_ORB.
 * LCD_ERR_INVALID for an unknown detector, use_harris != 0, block_size != 3, quality_level <= 0 or a negative min_distance; the
 * previous selection then stays. */
int lcd_detector_set(lcd_engine * e, int detector, const lcd_gftt_params * params);
/* The selected detector; `params` (may be NULL) receives its GFTT parameters. */
int lcd_detector_get(const lcd_engine * e, lcd_gftt_params * params);

/* LCD_DETECTOR_ORB_OCTREE: Kp/DetectorStrategy=10, rtabmap::ORBOctree (Features2d.cpp:2479-2566) around RTAB-Map's ORB-SLAM2 extractor
 * (corelib/src/opencv/ORBextractor.cc).  lcd_orb_params supplies n_features (nfeatures and Kp/MaxFeatures), n_levels (1..8), scale_factor
 * (any finite value > 1), edge_threshold (>= 19), fast_threshold (the initial FAST threshold), patch_size (31) and the depth fields.
 *   pyramid   level l = cv::resize(level l-1, cvRound(size / scale_factor^l), INTER_LINEAR)          ORBextractor.cc:1114-1139
 *   keypoints FAST per 30-pixel cell with FAST/MinThreshold as fallback, spread by a quadtree      :772-855, :546-770
 *             (DistributeOctTree) to the per-level counts of the constructor                      :416-477
 *   describe  IC angle, GaussianBlur(7x7, 2) of each level, steered BRIEF                          :83-153, :1066-1111
 *   wrapper   detection ignores the mask; keypoints whose level-0 mask byte at the truncated      Features2d.cpp:2527-2549
 *             coordinates is 0 are dropped, then limitKeypoints(Kp/MaxFeatures)
 * Phase 2 of DistributeOctTree orders nodes of equal size by their heap addresses, which the reference leaves undefined; the engine treats
 * the node created later as the larger one (DESIGN.md §2).  LCD_ERR_INVALID, before any launch, for n_levels outside 1..8, a scale factor
 * <= 1 or not finite, patch_size != 31, edge_threshold < 19, and a level whose span inside edge_threshold - 3 is under 30 pixels or more
 * than twice as tall as wide (the reference divides by zero or indexes out of range there).  n_features <= 0 is refused as for the other
 * detectors (the reference would run it with every level's count at 0 and no limit). */
#define LCD_DETECTOR_ORB_OCTREE 10
/* Select ORB-OCTREE with FAST/MinThreshold (7 in RTAB-Map, 0..255; LCD_ERR_INVALID otherwise, the previous selection then stays).
 * lcd_detector_set(e, LCD_DETECTOR_ORB_OCTREE, ...) is refused: this call selects it.  lcd_detector_get then returns 10. */
int lcd_detector_set_orb_octree(lcd_engine * e, int fast_min_threshold);
/* Test hook: cosf and sinf as the ORB-OCTREE descriptor computes them on the device, for the `count` floats whose bit patterns start at
 * `first` (d_cos, d_sin: device arrays of `count` floats).  Synchronous. */
int lcd_debug_orb_sincos(lcd_engine * e, unsigned first, unsigned count, float * d_cos, float * d_sin);

/* ---- detect: which keypoints of a frame are quantised (Memory::createSignature, Memory.cpp:5945-6100) ---------------------------
 * With Mem/RawDescriptorsKept, an odometry pose and Kp/MaxFeatures < Vis/MaxFeatures, the reference detects Vis/MaxFeatures keypoints
 * (Memory.cpp:5516-5538, :5725-5745) and keeps all of them in the signature (registration matches them all, Memory::getNi counts them,
 * :4955-4968), but quantises only the Kp/MaxFeatures strongest:
 *   gate   a frame with descriptors.rows < int(Kp/BadSignRatio * meanWordsPerLocation) (:5945-5947, :6051-6058) quantises nothing: a bad
 *          signature, for which Rtabmap::process computes no likelihood;
 *   limit  with more rows than Kp/MaxFeatures, Feature2D::limitKeypoints(keypoints, inliers, Kp/MaxFeatures, imageSize, ssc = false)
 *          (Features2d.cpp:412-477) picks the rows: a std::multimap<fabs(response), index> walked in reverse, so the strongest first and,
 *          among equal responses, the later index first (responses compared as bit patterns of their absolute value);
 *   words  the picked rows go to addNewWords in ascending keypoint order (quantizedToRawIndices, :5954-6048); every other keypoint gets
 *          a negative id, -1, -2, ... in keypoint order (:6070-6100).
 * The limit is engine state, as lcd_detector_set.  Once set, every image-level call applies it to each frame: lcd_process_frames[_submit|
 * _wait|_dev], lcd_map_detect_async + lcd_map_frame and lcd_shard_process_frames_dev.  lcd_orb_params.n_features stays the detection count
 * (Vis/MaxFeatures when the caller's condition above holds).  word_ids_out keeps its [n_frames * n_features] shape: quantised rows carry
 * their word ids, the other rows -1, -2, ..., padding rows 0.  The likelihood comes from the quantised words only; verification uses
 * every detected row (descriptors, uv, xyz).  A bad frame gets a likelihood row of zeros, no hypothesis (0) and no registration (ok = 0,
 * no matches).  In lcd_map_frame only quantised rows add references, ni(sig_id) grows by the keypoint count, and a bad frame creates
 * no words and adds no references. */
typedef struct lcd_quantize_limit {
	int max_features;     /* Kp/MaxFeatures: quantise at most this many keypoints of a frame, the strongest (0 = all, the default) */
	float bad_sign_ratio; /* Kp/BadSignRatio (0.5) */
	int mean_words;       /* meanWordsPerLocation of Memory::update (Memory.cpp:5269-5278): Kp/MaxFeatures when > 0, the caller's
	                         totalActiveReferences / treeSize otherwise, 0 with Mem/UseOdomFeatures.  0 = no bad-signature gate */
} lcd_quantize_limit;
/* Set the limit (NULL = {0, 0, 0}: every row quantised, no gate, every call as without this setting).  The gate's threshold is
 * computed here once, as the reference does: (int)(bad_sign_ratio * (float)mean_words).  LCD_ERR_INVALID for a negative max_features or
 * mean_words and for a bad_sign_ratio that is negative or not finite; the previous setting then stays.  A new engine holds {0, 0, 0}. */
int lcd_quantize_limit_set(lcd_engine * e, const lcd_quantize_limit * p);
int lcd_quantize_limit_get(const lcd_engine * e, lcd_quantize_limit * p);
/* replaces: the gate and Feature2D::limitKeypoints(keypoints, inliers, ...) of Memory::createSignature (Memory.cpp:5945-6048,
 * Features2d.cpp:412-477; tie rule above) for n_frames detected frames under the engine's limit: d_kp[n_frames][cap] (lcd_keypoint, as
 * lcd_orb_detect_describe_dev writes them), d_n[n_frames], d_desc[n_frames][cap][row] (bytes of a binary engine, floats of a float
 * engine).  Writes the quantised rows in ascending keypoint order, d_desc_out[n_frames][k][row] (zeros past a frame's count), their
 * keypoint index d_index_out[n_frames][k] (quantizedToRawIndices; -1 past the count) and d_n_out[n_frames] (0 for a bad signature), with
 * k = max_features > 0 ? min(max_features, cap) : cap.  lcd_localize_batch_dev has no per-frame counts: it quantises the zero rows of
 * a frame with fewer than k quantised rows too, so a caller with such frames reads d_n_out (a bad signature is LCD_FRAME_SKIP for
 * lcd_decide_batch_dev).  Asynchronous on `stream`.  LCD_ERR_INVALID for a null pointer or n_frames <= 0, LCD_ERR_CAPACITY for cap
 * outside 1..4096. */
int lcd_limit_keypoints_dev(lcd_engine * e, int n_frames, int cap, const lcd_keypoint * d_kp, const int * d_n, const void * d_desc,
                            void * d_desc_out, int * d_index_out, int * d_n_out, void * stream);
/* replaces: the word list assembly of Memory::createSignature (Memory.cpp:6070-6100).  Per-keypoint word ids d_words_out[n_frames][cap]
 * from the k-strided ids of the quantised rows d_words_q[n_frames][k] (e.g. lcd_localize_batch_dev's output on d_desc_out): quantised
 * rows take their id, the other rows of a frame -(1 + i - (quantised rows before i)), i.e. -1, -2, ... in keypoint order, padding rows
 * (i >= d_n[f]) 0.  d_index / d_n_quantised as lcd_limit_keypoints_dev wrote them.  This is what lcd_decide_epipolar_dev needs beside
 * the frame's full uv.  Asynchronous on `stream`.  LCD_ERR_INVALID for a null pointer, n_frames <= 0 or k outside 1..cap,
 * LCD_ERR_CAPACITY for cap outside 1..4096. */
int lcd_word_ids_expand_dev(lcd_engine * e, int n_frames, int cap, int k, const int * d_n, const int * d_index, const int * d_n_quantised,
                            const int * d_words_q, int * d_words_out, void * stream);

/* ---- dictionary: VWDictionary ------------------------------------------------ */
/* replaces: VWDictionary::addWord (VWDictionary.cpp:1554-1580) for n words whose ids
 * the caller chose (DB load, LTM reactivation).  Words become "not indexed" until
 * lcd_dict_update, exactly like _notIndexedWords. */
int lcd_dict_add_words(lcd_engine * e, const int * ids, const void * desc, int n);
/* replaces: VWDictionary::removeWords / deleteUnusedWords (VWDictionary.cpp:1582-1607).
 * Indexed words leave the search structure at the next lcd_dict_update
 * (_removedIndexedWords); their posting lists are dropped immediately. */
int lcd_dict_remove_words(lcd_engine * e, const int * ids, int n);
/* replaces: VWDictionary::update (VWDictionary.cpp:475-701), Kp/NNStrategy=0 row order:
 * not-indexed words are appended in ascending id, removed rows are compacted out. */
int lcd_dict_update(lcd_engine * e);
/* replaces: VWDictionary::clear (VWDictionary.cpp:842-873) */
int lcd_dict_clear(lcd_engine * e);
/* _visualWords.size(), rows of the search index, _notIndexedWords.size(), _lastWordId */
int lcd_dict_size(const lcd_engine * e);
int lcd_dict_indexed_size(const lcd_engine * e);
int lcd_dict_not_indexed_size(const lcd_engine * e);
int lcd_dict_last_word_id(const lcd_engine * e);
int lcd_dict_set_last_word_id(lcd_engine * e, int id);
/* 1 if the word is in _visualWords (uContains), else 0 */
int lcd_dict_has_word(const lcd_engine * e, int word_id);
/* copy back the indexed rows in search order: ids[rows], desc[rows*dim] (either may be NULL).
 * Mirrors what _dataTree/_mapIndexId hold (VWDictionary.cpp:650-676). */
int lcd_dict_get_indexed(lcd_engine * e, int * ids, void * desc, int cap_rows);

/* The 2-NN of 32-byte binary descriptors has two bit-identical implementations: kernel 1 (default) computes the Hamming
 * distances as an exact s8 GEMM on the tensor cores (nn_tensor.cuh), kernel 0 with XOR + POPC on the integer pipes
 * (nn_hamming.cuh; the only one for other descriptor sizes).  Mirrors choosing Kp/NNStrategy in the reference
 * (VWDictionary::setNNStrategy, VWDictionary.cpp:316-338).  lcd_nn_last_kernel: which one the last search used. */
int lcd_nn_select(lcd_engine * e, int kernel);
int lcd_nn_last_kernel(const lcd_engine * e);
/* Float engines (LCD_DESC_F32) with >= 4096 rows search through the fp16 tensor-core filter + exact re-rank (kernel 1; kernel 0 = the
 * exact CUDA-core scan; results are bit-identical).  Diagnostics of the LAST search of nq queries: how many queries were redone by
 * the exact fallback scan, how many candidate rows the filter passed to the re-rank in total, and how many dictionary rows have been
 * converted to the cached fp16 image since the engine was created (it is converted once per dictionary change, not per search). */
int lcd_nn_f32_stats(lcd_engine * e, int nq, int * n_fallback, long long * n_candidates, long long * rows_converted);

/* replaces: FlannIndex::knnSearch(k=2) on a LinearIndex (FlannIndex.cpp:701-745 ->
 * rtflann linear_index.h:129-146 + result_set.h:151-172): exact 2-NN of every query
 * row over the INDEXED words; ties -> lowest row.  id = 0 and dist = -1 where fewer
 * than 1 (2) indexed words exist.  dist: Hamming count, or squared L2, as float. */
int lcd_dict_knn2(lcd_engine * e, const void * queries, int nq,
                  int * id1, float * d1, int * id2, float * d2);

/* replaces: VWDictionary::addNewWords (VWDictionary.cpp:913-1229) incl. the NNDR test,
 * intra-frame new-word comparison (Kp/NewWordsComparedTogether) and addWordRef for
 * sig_id (VWDictionary.cpp:880-897).  incremental = Kp/IncrementalDictionary,
 * nndr = Kp/NndrRatio.  word_ids_out[nq]; *n_new_out = words created.
 * sig_id <= 0: quantise only, add no references. */
int lcd_dict_quantize(lcd_engine * e, const void * queries, int nq, int sig_id,
                      int incremental, float nndr, int new_words_compared_together,
                      int * word_ids_out, int * n_new_out);

/* replaces: VWDictionary::findNN(cv::Mat) (VWDictionary.cpp:1273-1552): read-only,
 * also searches the not-indexed words; 0 where NNDR rejects. */
int lcd_dict_find_nn(lcd_engine * e, const void * queries, int nq, int incremental,
                     float nndr, int * word_ids_out);

/* ---- inverted index: VisualWord::_references + Memory::computeLikelihood ------ */
/* replaces: VWDictionary::addWordRef (VWDictionary.cpp:880-897) / VisualWord::addRef
 * (VisualWord.cpp:51-63) for the n words of one signature (duplicates count). */
int lcd_index_add_refs(lcd_engine * e, int sig_id, const int * word_ids, int n);
/* replaces: VWDictionary::removeAllWordRef (VWDictionary.cpp:899-911) for every word of
 * sig_id (what Memory::disableWordsRef does, Memory.cpp:6871-6897). */
int lcd_index_remove_sig(lcd_engine * e, int sig_id);
/* ni of Memory::getNi (Memory.cpp:4955-4968): total words of the signature, including
 * un-quantised (<=0) ones.  lcd_index_add_refs / lcd_dict_quantize add n to it; this
 * overrides it. */
int lcd_index_set_ni(lcd_engine * e, const int * sig_ids, const int * ni, int n);
/* bulk load of a word->(signature,count) table in CSR form (cold start from a database,
 * Memory::loadDataFromDb, Memory.cpp:410-438): word_ids[nw], row_ptr[nw+1],
 * sig[row_ptr[nw]], cnt[row_ptr[nw]].  Words must exist in the dictionary. */
int lcd_index_load_csr(lcd_engine * e, const int * word_ids, int nw, const int64_t * row_ptr,
                       const int * sig, const int * cnt);
/* number of signatures referencing word (VisualWord::getReferences().size()), total refs */
int lcd_index_word_nw(lcd_engine * e, int word_id);
long long lcd_index_total_refs(const lcd_engine * e);
/* copy back the posting list of one word sorted by signature id (cap entries max);
 * returns the list length or <0. */
int lcd_index_get_refs(lcd_engine * e, int word_id, int * sig, int * cnt, int cap);

/* replaces: the TF-IDF branch of Memory::computeLikelihood (Memory.cpp:2215-2291):
 * query_word_ids = the new signature's words (any order, duplicates and ids <= 0
 * allowed: uUniqueKeys + the *i>0 test are applied), sig_ids[ns] = the ids to score,
 * n_total = N = Memory::getSignatures().size().  likelihood_out[ns] float.
 * Every call that takes n_total (this one, the localize, process, map and shard families) returns LCD_ERR_INVALID when
 * n_total < 0; n_total = 0 gives 0 for every listed id, as the reference computes nothing when N is 0 (Memory.cpp:2250). */
int lcd_index_score(lcd_engine * e, const int * query_word_ids, int nq,
                    const int * sig_ids, int ns, int n_total, float * likelihood_out);

/* ---- Bayes filter over the loop-closure hypotheses (SURVEY.md 8(f) #1) ---------------------------
 * replaces: BayesFilter::computePosterior (BayesFilter.cpp:145-270): prior = prediction x last posterior, posterior = likelihood .* prior,
 * normalised; the prediction is the matrix of generatePrediction / addNeighborProb / normalize (:272-505) kept in its sparse form (the
 * reference builds it dense: S x S floats).  The engine keeps the last posterior by place id between calls (updatePosterior, :712-737);
 * lcd_bayes_reset = BayesFilter::reset.
 *   ids[n]         uKeys(likelihood): ascending place ids, ids[0] < 0 = the virtual place (Rtabmap::adjustLikelihood adds it)
 *   likelihood[n]  the adjusted likelihood of each id
 *   col_ptr[n+1], nbr_row[nnz], nbr_level[nnz]   for every place (column) the places its probability mass spreads to:
 *                  Memory::getNeighborsId(id, n_lc - 1, ...) restricted to the places of this call and outside the short-term memory,
 *                  as (position in ids, graph margin) pairs in ascending id order; the place itself (margin 0) must be listed — the
 *                  graph walk is the caller's (Memory), the probability model is computed here.  Columns of loop-closure partners that
 *                  share a neighbour tree (BayesFilter.cpp:378-391) simply carry the same list.  The virtual place has an empty list.
 *   prediction_lc[n_lc]  Bayes/PredictionLC {virtual place, loop closure, level 1, level 2, ...}, virtual_place_prior = Bayes/VirtualPlacePriorThr
 *   posterior_out[n]
 * Float results agree with the reference's dense float product to ~1e-6 relative. */
int lcd_bayes_compute_posterior(lcd_engine * e, const int * ids, const float * likelihood, int n, const int64_t * col_ptr, const int * nbr_row,
                                const int * nbr_level, const double * prediction_lc, int n_lc, float virtual_place_prior, float * posterior_out);
int lcd_bayes_reset(lcd_engine * e);

/* ---- fused, batched localisation query (frozen dictionary + frozen map) ---------
 * One call = B independent queries of the quantise -> score half of the hot path with
 * NO mutation of the engine (SURVEY.md App. C.5): for each frame b
 *   addNewWords(desc_b, sigId) -> computeLikelihood(sig, sig_ids) -> roll back.
 * queries: B*nq_per_frame descriptors (frame-major); n_total = N including the query
 * itself; word_ids_out[B*nq] (new words get ids last_word_id+1.. per frame, not kept);
 * likelihood_out[B*ns]. Either output may be NULL. */
int lcd_localize_batch(lcd_engine * e, const void * queries, int n_frames, int nq_per_frame,
                       int incremental, float nndr, int new_words_compared_together,
                       const int * sig_ids, int ns, int n_total,
                       int * word_ids_out, float * likelihood_out);

/* Same work on device-resident inputs/outputs, asynchronous on `stream` (a cudaStream_t
 * passed as void*; NULL = the engine's stream).  d_queries as above; d_sig_ids[ns];
 * outputs may be NULL.  Used by bench.py for the HBM-resident timing and by the
 * word-range-sharded multi-GPU path. */
int lcd_localize_batch_dev(lcd_engine * e, const void * d_queries, int n_frames, int nq_per_frame,
                           int incremental, float nndr, int new_words_compared_together,
                           const int * d_sig_ids, int ns, int n_total,
                           int * d_word_ids_out, float * d_likelihood_out, void * stream);

/* ---- similarity likelihood: Memory::computeLikelihood with Kp/TfIdfLikelihoodUsed=false --------------------------
 * The other branch of computeLikelihood (Memory.cpp:2179-2214): Signature::compareTo (Signature.cpp:250-288) of the query
 * against every listed id, in list order.  Global-descriptor pipelines (Mem/GlobalDescriptorStrategy, PyDescriptor), the
 * memory of OdometryMono and rehearsal (Mem/RehearsalSimilarity, Memory.cpp:4218-4266) use it.  For each id s:
 *   s <= 0 (the virtual place)                          -> 0
 *   query and s both carry a global descriptor          -> (float)(((double)dot(q, s) + 1.0f) / 2.0f)
 *   otherwise, valid(x) = number of x's word ids > 0:
 *     valid(q) == 0 or valid(s) == 0 (bad signature)    -> 0
 *     else                                              -> (float)pairs / (float)max(valid(q), valid(s))
 * pairs = sum over the shared word ids of min(count in q, count in s), what EpipolarGeometry::findPairs counts
 * (EpipolarGeometry.h:119-151); valid(s) = the references the index holds for s (lcd_index_get_refs counts).  The word-pair value
 * is exact.  Word ids <= 0 never pair: findPairs tests id >= 0 and would pair id 0, which the quantiser never puts into a
 * signature (new and matched words are > 0, unquantised features get distinct negative ids).
 * The dot product is one fp32 fused multiply-add chain in ascending dimension order: the same bits for a (query, signature)
 * whatever the batch, the frame's position, ns or the entry point, within gamma_D * sum |q_i s_i| of the exact value
 * (gamma_D = D u / (1 - D u), u = 2^-24).  OpenCV's cv::Mat::dot is dispatched per CPU, so no single reference bit pattern exists.
 * Sharded engines (lcd_shard_set_row_offset != 0) get LCD_ERR_STATE from every call of this group: they use
 * lcd_shard_localize_similarity_batch_dev and its stages (word-range sharding, below).
 *
 * Global descriptors: Signature::sensorData().globalDescriptors(), type 1, one per signature, fp32 [n][dim] row-major.  The
 * dimension is fixed by the first add; a later add with another dimension is LCD_ERR_INVALID.  Adding an id that has a
 * descriptor replaces it; freed rows are reused before the store grows. */
int lcd_gdesc_add(lcd_engine * e, const int * sig_ids, int n, int dim, const float * data);
int lcd_gdesc_remove(lcd_engine * e, const int * sig_ids, int n);
int lcd_gdesc_count(const lcd_engine * e);
int lcd_gdesc_dim(const lcd_engine * e); /* 0 before the first add */
/* Memory::computeLikelihood with Kp/TfIdfLikelihoodUsed=false for one query signature (with ns = 1 also Memory::rehearsal's
 * compareTo, Memory.cpp:4245): query_word_ids[nq] its words (any order, duplicates and ids <= 0 allowed; nq may be 0),
 * query_gdesc[lcd_gdesc_dim(e)] its global descriptor or NULL, sig_ids[ns], likelihood_out[ns].  Returns LCD_ERR_INVALID
 * ("Global descriptors should be normalized!", the reference's UASSERT) when a global-descriptor value is < 0; the values are
 * written all the same. */
int lcd_index_similarity(lcd_engine * e, const int * query_word_ids, int nq, const float * query_gdesc,
                         const int * sig_ids, int ns, float * likelihood_out);
/* lcd_localize_batch semantics (quantise n_frames frames without mutation) followed by the similarity likelihood of every frame
 * against sig_ids[ns]: gdesc[n_frames][lcd_gdesc_dim(e)] the frames' global descriptors or NULL, word_ids_out[n_frames*nq_per_frame],
 * likelihood_out[n_frames*ns] (either output may be NULL).  LCD_ERR_INVALID as lcd_index_similarity when a value is < 0. */
int lcd_localize_similarity_batch(lcd_engine * e, const void * queries, int n_frames, int nq_per_frame, int incremental, float nndr,
                                  int new_words_compared_together, const float * gdesc, const int * sig_ids, int ns,
                                  int * word_ids_out, float * likelihood_out);
/* The same on device pointers, asynchronous on `stream` (NULL = the engine's stream).  It does not check the values: a caller
 * that needs the UASSERT looks for values < 0 itself.  Similarity followed by verification is this call, then lcd_verify_top_dev
 * on d_likelihood_out (any likelihood rows work there), then lcd_process_fetch. */
int lcd_localize_similarity_batch_dev(lcd_engine * e, const void * d_queries, int n_frames, int nq_per_frame, int incremental,
                                      float nndr, int new_words_compared_together, const float * d_gdesc, const int * d_sig_ids,
                                      int ns, int * d_word_ids_out, float * d_likelihood_out, void * stream);

/* ---- geometric verification: Memory::computeTransform ----------------------------------
 * Batched verification of n_pairs (FROM = old signature with 3-D points, TO = new signature with
 * 2-D keypoints) hypotheses.  Buffers are [n_pairs][cap] row-major; n_from/n_to give the valid
 * rows of each pair.  Single camera, identity local transform, rectified (no distortion); the decision calls of localisation clients
 * take each client's own camera instead (lcd_clients_set_cameras). */
typedef struct lcd_verify_params {
	float nndr;            /* Vis/CorNNDR (0.8)                                             */
	int min_inliers;       /* Vis/MinInliers (20)                                           */
	int iterations;        /* Vis/Iterations (300, <= 320)                                  */
	float reproj_error;    /* Vis/PnPReprojError (2): RANSAC compares the error with its square */
	int refine_iterations; /* Vis/PnPRefineIterations (1)                                   */
	float refine_sigma;    /* refineSigma of util3d::solvePnPRansac (3.0)                   */
	double fx, fy, cx, cy; /* CameraModel::K() of the TO signature                          */
	int var_median_ratio;  /* Vis/PnPVarianceMedianRatio (4, must be > 1)                   */
	float max_variance;    /* Vis/PnPMaxVariance (0 = off): reject when the linear variance exceeds it */
	int split_linear_cov;  /* Vis/PnPSplitLinearCovComponents (0)                           */
	int image_width, image_height; /* CameraModel::imageSize() of the TO camera (0, 0 = not set) */
	int repeat_once;       /* Reg/RepeatOnce (1 in the reference): after a successful first pass, register again with its transform as
	                          the guess (projection + window matching); needs the image size */
	int guess_win_size;    /* Vis/CorGuessWinSize (40 pixels; 0 = no second pass) */
} lcd_verify_params;

typedef struct lcd_verify_result {
	int ok;               /* 1: inliers >= min_inliers (and variance accepted), transform valid */
	int n_matches;        /* correspondences given to PnP                                    */
	int n_inliers;
	int iterations_run;   /* RANSAC iterations the sequential reference would have executed  */
	double rvec[3];       /* PnP pose (object -> camera), Rodrigues vector                   */
	double tvec[3];
	float transform[12];  /* (localTransform * pnp)^-1 as rtabmap::Transform 3x4             */
	double covariance[36]; /* RegistrationInfo::covariance, 6x6 row-major (util3d_motion_estimation.cpp:156-258): identity scaled by
	                          2.1981 x the [n/ratio]-th smallest squared 3-D error (rows 0-2) and angular error (rows 3-5) of the inliers */
} lcd_verify_result;

/* replaces: the global matching of RegistrationVis::computeTransformationImpl through a temporary
 * VWDictionary (RegistrationVis.cpp:1482-1503), Vis/CorNNType 0/3: from_ids/to_ids[n_pairs*cap] word
 * ids of every descriptor (ids start at 1 per pair).  Binary engines only (LCD_ERR_INVALID on a float engine); the float matching is
 * observable through lcd_verify_batch's match_ids / inlier_ids. */
int lcd_match_pairs(lcd_engine * e, int n_pairs, int cap, const void * desc_from, const int * n_from,
                    const void * desc_to, const int * n_to, float nndr, int * from_ids, int * to_ids);

/* replaces: Memory::computeTransform -> RegistrationVis (global matching, RegistrationVis.cpp:1482-1546)
 * -> util3d::estimateMotion3DTo2D (util3d_motion_estimation.cpp:59-289, incl. the covariance :156-258) -> util3d::solvePnPRansac
 * (:843-990) -> cv3::solvePnPRansac (opencv/solvepnp.cpp:112-417).  xyz_from: NaN where a keypoint has no depth.  xyz_to: the 3-D
 * points of the TO signature (words3B; NaN = none) or NULL when it has none — the covariance then comes from the 10 %-depth ray
 * model (image size set) or from the reprojection RMS (image size 0 x 0), as in the reference.
 * match_ids / inlier_ids [n_pairs*cap] (word ids, ascending / in inlier order) may be NULL.
 * cap (here, and max(store row size, nq) in the store-backed calls) is bounded by the matching kernel's shared memory, not by 4096:
 * LCD_ERR_CAPACITY when its dynamic size (DESIGN.md §6) plus its static size exceeds the device's opt-in limit per block.  On an H100
 * (232 448 B per block) the largest cap is 3540 for 16-byte descriptors, 2248 for 32-byte and 1233 for 64-byte ones (2560 B static).
 * The refusal leaves the engine usable.
 * Float engines (LCD_DESC_F32, 64, 128 or 256 floats; every registration call below, the store-backed ones included): the same temporary
 * dictionary with squared L2 in place of Hamming (VWDictionary.cpp:1020-1028, NORM_L2SQR / rtflann L2), summed in rtflann's order
 * (dist.h:158-166) for the dictionary and for the Reg/RepeatOnce pass's cv::BFMatcher(NORM_L2SQR) ranking, whose OpenCV SIMD order can
 * differ in the last ulp (as lcd_match_bf).  Ties go to the first-created word.  Both sides are read from global memory and shared
 * memory holds per-row scalars only, so every cap up to 4096 is accepted at 64-D, 128-D and 256-D (largest dynamic size 37 B per row;
 * at 256-D the new-word loop stages 32 descriptors in 32 896 B of static shared memory). */
int lcd_verify_batch(lcd_engine * e, int n_pairs, int cap, const void * desc_from, const float * xyz_from, const int * n_from,
                     const void * desc_to, const float * uv_to, const float * xyz_to, const int * n_to,
                     const lcd_verify_params * params, lcd_verify_result * results, int * match_ids, int * inlier_ids);

/* Static shared memory in bytes of a verification kernel at the engine's descriptor size: which = 0 pair matching, 1 matching with a
 * guess (Reg/RepeatOnce), 2 PnP RANSAC, 3 FROM-dictionary build; on a float engine 0 is the kernel that resolves the TO side and assembles the
 * correspondences (the TO x dictionary scan before it has only static shared memory).  Float engines have all four at 64, 128 and 256
 * floats.  < 0 on error. */
long long lcd_verify_static_smem(lcd_engine * e, int which);

/* replaces: util3d::solvePnPRansac (util3d_motion_estimation.cpp:843-990; argument for argument: objectPoints, imagePoints,
 * cameraMatrix, distCoeffs, rvec, tvec, useExtrinsicGuess, iterationsCount, reprojectionError, minInliersCount, inliers, flags,
 * refineIterations, refineSigma) = cv3::solvePnPRansac (opencv/solvepnp.cpp:112-211: EPnP on 6-point samples drawn with
 * cv::RNG(-1), strict-best model, adaptive iteration count at confidence 0.99, returned pose = best minimal-sample model) followed
 * by the PCL-style refinement loop (:882-989).  object_points[n*3], image_points[n*2] float; K[9] row-major 3x3 double;
 * dist_coeffs[n_dist] must be all zero (or NULL): RTAB-Map passes CameraModel::D(), zeros for rectified images — anything else is
 * rejected with LCD_ERR_INVALID, as are flags != 0 (SOLVEPNP_ITERATIVE) and n == 4 (the reference switches to P3P).
 * rvec / tvec: in = the extrinsic guess (EPnP ignores it, exactly as in the reference), out = the refined pose; left untouched when
 * RANSAC finds no model.  inliers_out[n] (indices into the input, ascending), *n_inliers_out. */
int lcd_pnp_ransac(lcd_engine * e, const float * object_points, const float * image_points, int n, const double K[9],
                   const double * dist_coeffs, int n_dist, double rvec[3], double tvec[3], int use_extrinsic_guess,
                   int iterations, float reproj_error, int min_inliers, int flags, int refine_iterations, float refine_sigma,
                   int * inliers_out, int * n_inliers_out);
/* n_sets independent problems in one launch (one CTA each): object_points[n_sets][cap][3], image_points[n_sets][cap][2],
 * n_points[n_sets], rvec / tvec [n_sets][3], inliers_out[n_sets][cap], n_inliers_out / iterations_run_out [n_sets] (may be NULL). */
int lcd_pnp_ransac_batch(lcd_engine * e, int n_sets, int cap, const float * object_points, const float * image_points, const int * n_points,
                         const double K[9], const double * dist_coeffs, int n_dist, double * rvec, double * tvec, int use_extrinsic_guess,
                         int iterations, float reproj_error, int min_inliers, int flags, int refine_iterations, float refine_sigma,
                         int * inliers_out, int * n_inliers_out, int * iterations_run_out);

/* replaces: cv::BFMatcher on the descriptors of a signature pair (NORM_HAMMING for LCD_DESC_U8 engines, NORM_L2SQR for LCD_DESC_F32):
 *   LCD_MATCH_KNN2       knnMatch(query, train, k = 2)          (RegistrationVis.cpp:1128-1141, :1280-1300; VWDictionary.cpp:1027-1028)
 *   LCD_MATCH_CROSSCHECK BFMatcher(norm, crossCheck = true).match(query, train)   (RegistrationVis.cpp:1452-1453, Vis/CorNNType = 5)
 * for n_pairs independent pairs, [n_pairs][cap] rows each.  idx1 / dist1 [n_pairs*cap]: train index and distance of the best match of
 * every query row (-1 / -1 = none: in cross-check mode the queries OpenCV returns no DMatch for); idx2 / dist2: second neighbour
 * (KNN2 only; may be NULL in cross-check mode).  Ties resolve to the lowest index, as in cv::batchDistance.  Float distances are summed in
 * rtflann's order (dist.h:158-166), which can differ from OpenCV's SIMD order in the last ulp. */
#define LCD_MATCH_KNN2 0
#define LCD_MATCH_CROSSCHECK 1
int lcd_match_bf(lcd_engine * e, int n_pairs, int cap, const void * desc_query, const int * n_query, const void * desc_train,
                 const int * n_train, int mode, int * idx1, float * dist1, int * idx2, float * dist2);

/* ---- signature store + fused query ----------------------------------------------------------
 * The per-node data Memory keeps for verification (Signature::getWordsDescriptors / getWords3,
 * corelib/include/rtabmap/core/Signature.h:155-164), resident in HBM so that the hypothesis picked
 * from the likelihood can be verified without a host round trip.
 * desc [n_sigs][cap][dim] (bytes of a binary engine, floats of a float engine), xyz [n_sigs][cap][3] (NaN = no depth), n[n_sigs]
 * valid rows. */
int lcd_sig_add_batch(lcd_engine * e, const int * sig_ids, int n_sigs, int cap, const void * desc,
                      const float * xyz, const int * n);
int lcd_sig_remove(lcd_engine * e, int sig_id);
int lcd_sig_count(const lcd_engine * e);
/* rows the store has allocated so far (freed rows are reused before it grows) */
int lcd_sig_slots(const lcd_engine * e);

/* One call = n_frames independent loop-closure queries through quantise -> score -> verify:
 * lcd_localize_batch, then for every frame the signature with the highest likelihood (first maximum,
 * > 0) is verified against the frame (Memory::computeTransform(hypothesis, frame), FROM = hypothesis
 * with its stored 3-D points, TO = the frame's descriptors + keypoints uv[n_frames][nq][2]).
 * hypothesis_out[n_frames] = verified signature id (0 = none).  Outputs may be NULL. */
int lcd_process_batch(lcd_engine * e, const void * queries, const float * uv, int n_frames, int nq_per_frame,
                      int incremental, float nndr, int new_words_compared_together,
                      const int * sig_ids, int ns, int n_total, const lcd_verify_params * vp,
                      int * word_ids_out, float * likelihood_out, int * hypothesis_out,
                      lcd_verify_result * results);
/* replaces: Rtabmap::adjustLikelihood (Rtabmap.cpp:5691-5760; uMean / uVariance of the values > 0, UMath.h:419-431, :512-526),
 * the step between Memory::computeLikelihood and the Bayes filter.  likelihood[n_frames*ns] are rows in ascending signature id
 * order (as lcd_index_score / lcd_localize_batch return them); adjusted_out[n_frames*(ns+1)]: element 0 of every row is the virtual
 * place, then the ns adjusted values.  virtual_place_ratio = Rtabmap/VirtualPlaceLikelihoodRatio (0 or 1).  Bit-identical to the
 * reference's float arithmetic (the sums run in list order). */
int lcd_adjust_likelihood(lcd_engine * e, const float * likelihood, int n_frames, int ns, int virtual_place_ratio,
                          float * adjusted_out);
int lcd_adjust_likelihood_dev(lcd_engine * e, const float * d_likelihood, int n_frames, int ns, int virtual_place_ratio,
                              float * d_adjusted_out, void * stream);
/* Same on device-resident inputs, asynchronous on `stream`; results stay in engine buffers until
 * lcd_process_fetch copies them back (hypothesis ids, verification results). */
int lcd_process_batch_dev(lcd_engine * e, const void * d_queries, const float * d_uv, int n_frames, int nq_per_frame,
                          int incremental, float nndr, int new_words_compared_together,
                          const int * d_sig_ids, int ns, int n_total, const lcd_verify_params * vp,
                          int * d_word_ids_out, float * d_likelihood_out, void * stream);
int lcd_process_fetch(lcd_engine * e, int n_frames, int * hypothesis_out, lcd_verify_result * results);
/* The same download queued on `stream` (NULL: the engine's stream) behind the step that produced the results, without any
 * synchronisation: a caller that keeps steps in flight (pinned output buffers, one set per step in flight) reads them after its own
 * event / stream synchronisation, while the next step already runs. */
int lcd_process_fetch_async(lcd_engine * e, int n_frames, int * hypothesis_out, lcd_verify_result * results, void * stream);
/* The whole hot path for n_frames frames: Memory::update (detect + quantise, Rtabmap.cpp:1470) ->
 * Memory::computeLikelihood (:2117) -> Memory::computeTransform of the top hypothesis (:3143), as
 * independent localisation queries (no mutation).  Host buffers in, host results out: n_kp_out[n_frames]
 * keypoints found, word_ids_out[n_frames * params->n_features] (0 in the padding rows of short frames),
 * likelihood_out[n_frames*ns], hypothesis_out / results as lcd_process_batch (vp may be NULL: no verify). */
int lcd_process_frames(lcd_engine * e, int n_frames, const uint8_t * images, int width, int height, int channels,
                       const void * depth, int depth_type, const lcd_orb_params * params,
                       int incremental, float nndr, int new_words_compared_together,
                       const int * sig_ids, int ns, int n_total, const lcd_verify_params * vp,
                       int * n_kp_out, int * word_ids_out, float * likelihood_out, int * hypothesis_out,
                       lcd_verify_result * results);
/* Pipelined form of lcd_process_frames for a stream of batches (a relocalisation service): _submit queues the upload
 * and the kernels of a batch and returns; _wait blocks until the OLDEST submitted batch is complete and its output
 * arrays are filled.  Two batches may be in flight, so the PCIe upload of batch k+1 runs under the kernels of batch k.
 * Input and output host arrays must stay valid (and should be pinned) until the matching _wait returns. */
int lcd_process_frames_submit(lcd_engine * e, int n_frames, const uint8_t * images, int width, int height, int channels,
                              const void * depth, int depth_type, const lcd_orb_params * params,
                              int incremental, float nndr, int new_words_compared_together,
                              const int * sig_ids, int ns, int n_total, const lcd_verify_params * vp,
                              int * n_kp_out, int * word_ids_out, float * likelihood_out, int * hypothesis_out,
                              lcd_verify_result * results);
int lcd_process_frames_wait(lcd_engine * e);
int lcd_process_frames_dev(lcd_engine * e, int n_frames, const uint8_t * d_images, int width, int height, int channels,
                           const void * d_depth, int depth_type, const lcd_orb_params * params,
                           int incremental, float nndr, int new_words_compared_together,
                           const int * d_sig_ids, int ns, int n_total, const lcd_verify_params * vp,
                           int * d_word_ids_out, float * d_likelihood_out, void * stream);

/* ---- mapping mode: Memory::update + Memory::computeLikelihood for a STREAM of frames (Rtabmap.cpp:1470, :2117) --------------------------
 * Frame t+1 depends on frame t (its new words, its references), so the frames of one map cannot be batched; what can overlap is the
 * detection of the next frame.  lcd_map_detect_async uploads one image (+ depth) and runs ORB detect + describe + 3-D lifting on the
 * engine's ORB stream and returns at once (two detections may be in flight; host buffers must stay valid until the matching
 * lcd_map_frame).  lcd_map_frame takes the OLDEST detection and does, in the reference's order: VWDictionary::update (Memory::preUpdate,
 * Memory.cpp:1004-1016), addNewWords of the frame's descriptors for sig_id incl. the references (the descriptors never leave the device),
 * and — when wm_sig_ids is given — the TF-IDF likelihood against those signatures (n_total = Memory::getSignatures().size()).
 * Outputs: *n_kp_out, kp_out / desc_out / xyz_out [n_kp] (any may be NULL), word_ids_out[Kp/MaxFeatures] (first n_kp valid), *n_new_out,
 * likelihood_out[ns].  Identical, call for call, to lcd_orb_detect_describe + lcd_dict_update + lcd_dict_quantize + lcd_index_score. */
int lcd_map_detect_async(lcd_engine * e, const uint8_t * image, int width, int height, int channels, const void * depth, int depth_type,
                         const lcd_orb_params * params);
int lcd_map_frame(lcd_engine * e, int sig_id, int incremental, float nndr, int new_words_compared_together, const int * wm_sig_ids, int ns,
                  int n_total, int * n_kp_out, lcd_keypoint * kp_out, uint8_t * desc_out, float * xyz_out, int * word_ids_out, int * n_new_out,
                  float * likelihood_out);

/* The verification half alone, for likelihood rows that already exist on the device (the sharded
 * multi-GPU path all-reduces the scores first, then every rank verifies its share of the frames):
 * arg-max hypothesis of each of the n_frames rows of d_likelihood[n_frames][ns], then
 * Memory::computeTransform(hypothesis, frame).  Results via lcd_process_fetch. */
int lcd_verify_top_dev(lcd_engine * e, const void * d_queries, const float * d_uv, int n_frames, int nq_per_frame,
                       const float * d_likelihood, const int * d_sig_ids, int ns, const lcd_verify_params * vp, void * stream);

/* ---- the loop-closure decision of many localisation clients (Mem/IncrementalMemory=false) -----------------------------------
 * A relocalisation service runs one rtabmap::Rtabmap per camera (a client) against one frozen map.  Each client has its own Bayes
 * filter state (BayesFilter::_posterior) and its own last highest hypothesis (Rtabmap::_highestHypothesis); the map, and with it the
 * prediction matrix, is shared.  These calls replace, for B clients at once, what Rtabmap::process does with one frame's raw
 * likelihood in localisation mode: adjustLikelihood (Rtabmap.cpp:2119-2121), BayesFilter::computePosterior (:2133), the hypothesis
 * selection and its checks (:2143-2233), and the verification of the accepted hypothesis with its rejections (:3133-3191).
 * The epipolar check (VhEp/Enabled) is lcd_decide_epipolar_dev, run between the decision and its verification; proximity detection by
 * space is lcd_decide_proximity_dev, run after it.  Retrieval and the graph optimisation stay the caller's.
 *
 * replaces: BayesFilter::BayesFilter + BayesFilter::reset (BayesFilter.cpp:43-68, :140-143) and Rtabmap's _highestHypothesis = (0, 0)
 * (Rtabmap.cpp:467, :1094) for n_clients clients at once; calling it again resets every client.  LCD_ERR_CAPACITY when the device
 * cannot hold the state. */
int lcd_clients_create(lcd_engine * e, int n_clients);
/* BayesFilter::reset + _highestHypothesis = (0, 0) of the listed clients; their cameras stay */
int lcd_clients_reset(lcd_engine * e, const int * clients, int n);

/* A client's camera: SensorData::cameraModels()[0] of the frames it sends (rectified, depth registered to the image). */
typedef struct lcd_camera {
	double fx, fy, cx, cy;          /* CameraModel::K(); fx, fy > 0; cx, cy read as lcd_orb_params / lcd_verify_params read them */
	int image_width, image_height;  /* CameraModel::imageSize(): 0 x 0 = not set, otherwise the image size of the calls that decide it */
	float local_transform[12];      /* CameraModel::localTransform(), 3x4 row-major rtabmap::Transform (base -> optical frame) */
} lcd_camera;
/* Sets the cameras of the listed clients (cams NULL: the listed clients go back to the parameters of each call).  For the frames of a
 * client with a camera, the decision calls (lcd_decide_batch_dev, lcd_decide_gps_batch_dev, lcd_process_decide_batch_dev,
 * lcd_process_frames_decide_*) take the camera as the call is made, and lcd_decide_proximity_dev and lcd_verify_decided_dev use that
 * snapshot; a submitted batch keeps the cameras it was submitted with.  Such a frame is lifted with the camera's fx..cy (as floats, as
 * projectDepthTo3D receives them) and its local transform (util3d::transformPoint, applied when it is not identity, util3d_features.cpp:
 * 110-114) in lcd_process_frames_decide_*, and every registration of its decision uses the camera's K and image size in place of
 * lcd_verify_params': transform = (localTransform * pnp)^-1, the covariance with transformCameraFrame = transform * localTransform
 * (util3d_motion_estimation.cpp:154-258), and RGBD/MaxLoopClosureDistance and the proximity radius read that base-frame transform.
 * Frames of clients without a camera are computed exactly as before.  LCD_ERR_STATE without clients; LCD_ERR_INVALID, changing nothing,
 * for a client out of range, a value that is not finite, fx or fy <= 0, a negative image size or only one side set, and a rotation that
 * is not orthonormal within 1e-5 (transforms are inverted as [R^T | -R^T t]).  lcd_process_frames_decide_* refuse (LCD_ERR_INVALID,
 * before any state changes) a camera whose image size is set and differs from the images'.  A registration with a client camera of
 * image size 0 x 0 has no Reg/RepeatOnce pass and takes the covariance from the reprojection RMS when the TO side has no 3-D points.
 * Not read by lcd_process_frames*, lcd_process_batch*, lcd_verify_batch, the sharded step or mapping mode. */
int lcd_clients_set_cameras(lcd_engine * e, const int * clients, int n, const lcd_camera * cams);
/* The working memory the clients localise against: ids[n] ascending, ids[0] the virtual place (a negative id: Memory keeps it in the
 * working memory, Memory.cpp:592), and the neighbour tables, Bayes/PredictionLC and Bayes/VirtualPlacePriorThr exactly as
 * lcd_bayes_compute_posterior takes them (same checks).  The prediction's columns are computed here, once per map, bit-equal to
 * lcd_bayes_compute_posterior's.  A client's last posterior is re-keyed to the current places when that client next computes
 * (updatePosterior, BayesFilter.cpp:712-737), not when the map changes: a place it did not have starts from 0 (from 1 for every place
 * when its state is empty), a place that left is dropped, and a place that left and came back while the client computed nothing keeps
 * its value, as in the reference.  A call that fails (bad tables: LCD_ERR_INVALID; no device memory for the tables or for the clients'
 * posteriors over the new map: LCD_ERR_CAPACITY) changes nothing: the previous map, or no map, stays in place. */
int lcd_clients_set_map(lcd_engine * e, const int * ids, int n, const int64_t * col_ptr, const int * nbr_row, const int * nbr_level,
                        const double * prediction_lc, int n_lc, float virtual_place_prior);

typedef struct lcd_decide_params {
	int virtual_place_ratio;         /* Rtabmap/VirtualPlaceLikelihoodRatio (0; 0 or 1)                                       */
	float loop_thr;                  /* Rtabmap/LoopThr (0.11; [0, 1])                                                        */
	float aggressive_loop_thr;       /* RGBD/AggressiveLoopThr (0.05; [0, 1]): used by LCD_FRAME_AGGRESSIVE frames when lower   */
	float loop_ratio;                /* Rtabmap/LoopRatio (0; [0, 1])                                                         */
	float max_loop_closure_distance; /* RGBD/MaxLoopClosureDistance (0 = off; >= 0, metres)                                   */
} lcd_decide_params;

/* frame flags: conditions the caller evaluates, because it owns the signature and the odometry cache */
#define LCD_FRAME_SKIP 1       /* bad signature, intermediate node or empty working memory (Rtabmap.cpp:1994-1999): the likelihood row
                                  is ignored, the posterior is untouched, highest = (0, 0) */
#define LCD_FRAME_HOLD 2       /* small displacement or too fast movement (:2229-2233): the posterior is untouched, highest = the
                                  client's last highest hypothesis */
#define LCD_FRAME_AGGRESSIVE 4 /* the conditions of :2173-2177 hold (not localised yet, RGB-D SLAM mode, old map present) */

/* decision statuses */
#define LCD_DECIDE_SKIPPED 0            /* LCD_FRAME_SKIP */
#define LCD_DECIDE_HELD 1               /* LCD_FRAME_HOLD */
#define LCD_DECIDE_NO_HYPOTHESIS 2      /* no real place has a posterior > 0 (:2162) */
#define LCD_DECIDE_UNDER_THRESHOLD 3    /* value < threshold */
#define LCD_DECIDE_UNDER_RATIO 4        /* value < threshold and value < loop_ratio x last value (:2215-2222) */
#define LCD_DECIDE_SINGLE_HYPOTHESIS 5  /* the posterior has <= 2 entries and the threshold is > 0 (:2188-2192) */
#define LCD_DECIDE_RATIO 6              /* value < loop_ratio x last value (:2197-2201) */
#define LCD_DECIDE_LAST_NULL 7          /* loop_ratio > 0 and the last value is 0 (:2202-2205) */
#define LCD_DECIDE_ACCEPTED 8           /* _loopClosureHypothesis = highest (:2206-2210) */
#define LCD_DECIDE_VERIFY_REJECTED 9    /* accepted, then Memory::computeTransform failed (:3156-3161) */
#define LCD_DECIDE_DISTANCE_REJECTED 10 /* accepted and registered, transform norm > max_loop_closure_distance (:3162-3167) */

typedef struct lcd_decision {
	int highest_id;      /* _highestHypothesis.first after this frame (the client's new last highest hypothesis) */
	float highest_value; /* _highestHypothesis.second: 1 - posterior(virtual place) */
	int loop_id;         /* _loopClosureHypothesis.first: the accepted (and, after verification, registered) place, else 0 */
	int status;          /* LCD_DECIDE_* */
} lcd_decision;

/* For each of n_frames frames, on the device: Rtabmap::adjustLikelihood of d_likelihood[n_frames][ns] (raw likelihood rows over the
 * map's real places in ascending id order, as lcd_localize_batch_dev, lcd_localize_similarity_batch_dev and
 * lcd_shard_localize_batch_dev write them; ns must equal the map's real places), BayesFilter::computePosterior of the frame's client
 * (the client's state becomes the new posterior; d_posterior_out[n_frames][ns+1], element 0 the virtual place, may be NULL; rows of
 * skipped or held frames are not written), then the hypothesis selection of Rtabmap.cpp:2143-2226: the real place with the largest
 * posterior, scanned in descending id order with a strict '>' from (0, 0) (ties go to the highest id), its value replaced by
 * 1 - posterior(virtual place); if its id is > 0, threshold loop_thr (aggressive_loop_thr for LCD_FRAME_AGGRESSIVE frames when lower);
 * at or over the threshold the single-hypothesis, ratio and last-null rejections in that order, else accepted.  clients[n_frames] and
 * frame_flags[n_frames] are host arrays, read before the call returns; a client appears at most once per call.  A client's posterior
 * is the same bits whatever the batch size, its position in the batch and the other clients in it.  Results stay on the device:
 * lcd_decide_fetch copies the decisions back, lcd_process_fetch the accepted ids (0 = none), lcd_verify_decided_dev verifies them. */
int lcd_decide_batch_dev(lcd_engine * e, const float * d_likelihood, int n_frames, int ns, const int * clients, const int * frame_flags,
                         const lcd_decide_params * dp, float * d_posterior_out, void * stream);
/* decisions of the first n_frames frames of the last decision call (and its verification, when it ran): out[n_frames]; synchronises */
int lcd_decide_fetch(lcd_engine * e, int n_frames, lcd_decision * out);
/* replaces: Memory::computeTransform(_loopClosureHypothesis.first, signature) (Rtabmap.cpp:3133-3191) for the frames whose last
 * decision was accepted (the other frames are not verified: ok = 0, no matches).  A failed registration becomes
 * LCD_DECIDE_VERIFY_REJECTED, a transform longer than max_loop_closure_distance (> 0) LCD_DECIDE_DISTANCE_REJECTED; both clear loop_id,
 * and the client's last highest hypothesis is left as it is.  d_queries / d_uv as lcd_process_batch_dev; n_frames must be the last
 * decision's.  Results through lcd_process_fetch (hypothesis = the final loop id) and lcd_decide_fetch.  After lcd_decide_proximity_dev,
 * a frame whose accepted place a proximity detection registered keeps LCD_DECIDE_ACCEPTED but is not registered again: lcd_process_fetch
 * reports it with ok = 0 and no matches, and its transform is that of the lcd_proximity_fetch path with link_type
 * LCD_PROXIMITY_LINK_GLOBAL (the reference adds that link with the proximity transform, Rtabmap.cpp:2902-2913, :3134). */
int lcd_verify_decided_dev(lcd_engine * e, const void * d_queries, const float * d_uv, int n_frames, int nq_per_frame,
                           const lcd_verify_params * vp, void * stream);
/* lcd_process_batch_dev with the decision: quantise + score against the map's real places (word ids and likelihood bit-identical to
 * lcd_localize_batch_dev with those ids), lcd_decide_batch_dev, lcd_verify_decided_dev.  Binary engines only; sharded engines get
 * LCD_ERR_STATE (a sharded rank calls lcd_decide_batch_dev on the rows lcd_shard_localize_batch_dev wrote). */
int lcd_process_decide_batch_dev(lcd_engine * e, const void * d_queries, const float * d_uv, int n_frames, int nq_per_frame,
                                 int incremental, float nndr, int new_words_compared_together, int ns, int n_total,
                                 const lcd_verify_params * vp, const int * clients, const int * frame_flags, const lcd_decide_params * dp,
                                 int * d_word_ids_out, float * d_likelihood_out, float * d_posterior_out, void * stream);

/* ---- the GPS filter of the place list (Rtabmap/LoopGPS, on by default) -------------------------------------------------------
 * replaces: the construction of signaturesToCompare in Rtabmap::process (Rtabmap.cpp:2046-2115) in localisation mode.  A frame with a
 * GPS fix compares only the places whose GPS position lies within RGBD/LocalRadius of its own (altitude differences under the frame's
 * GPS error ignored) and every place without a fix; adjustLikelihood, the prediction and the posterior then run over those places only,
 * as the reference's do over the shorter likelihood map.  Mapping mode (the nearest node's fix for a frame without one, a non-identity
 * originOffsetENU, Rtabmap.cpp:2014-2038) is not covered. */
typedef struct lcd_gps { /* the fields of rtabmap::GPS (GPS.h:68-72) the filter reads */
	double stamp;            /* > 0: a fix; otherwise none */
	double longitude, latitude, altitude, error; /* degrees, degrees, metres, metres */
} lcd_gps;

/* The GPS of every real place of the current map: ids[n] ascending exactly as lcd_clients_set_map received them after the virtual place,
 * gps[n] each place's sensorData().gps() (or what Memory::getGPS found for it, Memory.cpp:4507-4553), offset_enu[n][3] the x, y, z of
 * getGPS's offsetENU (NULL = zeros).  A place whose stamp is not > 0 is always compared (Rtabmap.cpp:2077: no cache entry -> accept).
 * Each place's geocentric point (GeodeticCoords::toGeocentric_WGS84, GeodeticCoords.cpp:75-102) is computed here, once per map, with
 * the host's libm.  LCD_ERR_STATE without a map; LCD_ERR_INVALID for other ids or a value that is not finite (nothing changes then).
 * lcd_clients_set_map drops the table. */
int lcd_clients_set_map_gps(lcd_engine * e, const int * ids, int n, const lcd_gps * gps, const float * offset_enu);

/* lcd_decide_batch_dev where a frame that computes a posterior and has frame_gps[f].stamp > 0 compares only the places of
 * Rtabmap.cpp:2046-2115 with radius local_radius (RGBD/LocalRadius, 10 by default; >= 0).  Frames without a fix, skipped and held frames
 * (which ignore their fix, as the reference does), and every frame when frame_gps is NULL are decided exactly as lcd_decide_batch_dev
 * decides them.  A gated frame's posterior row, and its client's state, hold 0 for the places it did not compare; the single-hypothesis
 * check counts its compared places.  d_compared_out[n_frames][ns] (device, may be NULL): 1 where the frame compared the place (every
 * place of a frame without a fix, none of a skipped or held frame).  lcd_decide_fetch, lcd_process_fetch, lcd_decide_epipolar_dev,
 * lcd_decide_proximity_dev and lcd_verify_decided_dev take this decision as they take lcd_decide_batch_dev's.  LCD_ERR_INVALID (nothing
 * changes) for a negative or non-finite radius, a frame GPS value that is not finite and lcd_decide_batch_dev's cases; LCD_ERR_STATE when
 * a frame that computes has a fix and the current map has no GPS table.  Device scratch: n_frames x (ns + 1) bytes for the compared
 * places and 12 bytes per (place, frame that computes) for the gated frames' prediction columns. */
int lcd_decide_gps_batch_dev(lcd_engine * e, const float * d_likelihood, int n_frames, int ns, const int * clients, const int * frame_flags,
                             const lcd_gps * frame_gps, float local_radius, const lcd_decide_params * dp, float * d_posterior_out,
                             unsigned char * d_compared_out, void * stream);

/* ---- word-range sharding across GPUs (SURVEY.md §8(e)) ---------------------------
 * Each rank owns the words whose row (in ascending id order) falls in its range; rows
 * are numbered globally: set the global row offset of this shard so that packed top-2
 * keys from different ranks merge with the reference's tie-break (lowest row = lowest id).
 * The key width is a property of the engine:
 *   binary (LCD_DESC_U8):  2 x u32 per query, (dist << 22) | global_row, 0xFFFFFFFF = none;
 *   float (LCD_DESC_F32):  2 x u64 per query, (float bits of the squared distance << 32) | global_row,
 *                          0xFFFFFFFFFFFFFFFF = none (4 u32 words per query behind the uint32_t pointers).
 * Unsigned order of a key is (distance, lowest global row) order in both layouts. */
int lcd_shard_set_row_offset(lcd_engine * e, int global_row_offset);
/* stage 1: local top-2 keys of every query over this rank's rows -> d_keys_out (2*nq u32 for
 * binary engines, 2*nq u64 for float engines).  All-gather these across ranks, then call stage 2 on every rank. */
int lcd_shard_knn2_keys_dev(lcd_engine * e, const void * d_queries, int nq, uint32_t * d_keys_out,
                            void * stream);
/* stage 2, sharded by FRAME (what scales): every rank resolves only its own frames [frame0, frame0+n_frames) of the job's
 * n_frames_total — merge of the G gathered key sets [G][n_frames_total * nq] key pairs + NNDR / new-word pass — and writes their
 * word ids (d_word_ids_out[n_frames*nq], 0 in padding rows; d_n_per_frame[n_frames_total] valid descriptors per frame or NULL).
 * All-gather the word ids, then lcd_shard_score_ids_dev on every rank accumulates this rank's share (its word range) of the
 * TF-IDF scores of ALL frames from the ids (uUniqueKeys + "id > 0" filter of Memory::computeLikelihood, Memory.cpp:2238-2256)
 * into d_scores_out[n_frames*ns]; all-reduce(sum), then lcd_shard_finalize_dev. */
int lcd_shard_resolve_frames_dev(lcd_engine * e, const void * d_queries_all, int frame0, int n_frames, int n_frames_total,
                                 int nq_per_frame, const uint32_t * d_keys_gathered, int n_ranks, const int * d_row_ids,
                                 int last_word_id, int incremental, float nndr, int new_words_compared_together,
                                 const int * d_n_per_frame, int * d_word_ids_out, void * stream);
int lcd_shard_score_ids_dev(lcd_engine * e, const int * d_word_ids_all, int n_frames, int nq_per_frame,
                            const int * d_sig_ids, int ns, int n_total, long long * d_scores_out, void * stream);
/* stage 2: merge G gathered key sets [G][nq] key pairs, run the replicated NNDR / new-word pass,
 * and accumulate this rank's share of the TF-IDF scores into d_scores_out[n_frames*ns]
 * (fixed-point int64, exact and order-independent; all-reduce(sum) them, then call
 * lcd_shard_finalize_dev).  d_row_ids: global row -> word id table [total_rows]. */
int lcd_shard_resolve_score_dev(lcd_engine * e, const void * d_queries, int n_frames, int nq_per_frame,
                                const uint32_t * d_keys_gathered, int n_ranks,
                                const int * d_row_ids, int total_rows, int last_word_id,
                                int incremental, float nndr, int new_words_compared_together,
                                const int * d_sig_ids, int ns, int n_total,
                                int * d_word_ids_out, long long * d_scores_out, void * stream);
int lcd_shard_finalize_dev(lcd_engine * e, const long long * d_scores, int n, float * d_likelihood_out,
                           void * stream);
/* The similarity likelihood (Kp/TfIdfLikelihoodUsed=false, see lcd_localize_similarity_batch_dev) in the same stages.  A word's
 * postings live on one rank, so the pair count of (frame, place) and valid(s) are exact sums of per-rank parts, and the result equals
 * the unsharded engine's bit for bit.
 * lcd_shard_similarity_ids_dev: from the word ids of ALL frames d_word_ids_all[n_frames*nq_per_frame] (the all-gathered output of
 * lcd_shard_resolve_frames_dev), this rank's pair counts over its word range d_pairs_out[n_frames*ns] int32, by position in
 * d_sig_ids, and this rank's valid(s) of the listed places d_valid_out[ns] int32.  All-reduce(sum) both across ranks (exact: a pair
 * count is at most nq_per_frame), then call lcd_shard_similarity_finalize_dev on every rank for its own frames.
 * lcd_shard_similarity_finalize_dev: compareTo of n_frames frames from the summed counts d_pairs[n_frames*ns], the summed valid(s)
 * d_valid[ns] and the frames' own word ids d_word_ids[n_frames*nq_per_frame] (valid(q) = their ids > 0, new words included) into
 * d_likelihood_out[n_frames*ns].  Global descriptors (all may be NULL): d_frame_gdesc[n_frames][dim] the frames' own, and the map's
 * as a table d_map_gdesc[n_map_rows][dim] with d_map_gdesc_row[ns] the row of each listed place or -1 for none (the descriptor store
 * of lcd_gdesc_add refuses sharded engines).  A (frame, place) pair takes the descriptor value when both sides carry one.  Returns
 * LCD_ERR_INVALID when dim <= 0 while descriptors are given, or when a row index lies outside [-1, n_map_rows): the row indices are
 * read back to check them, which synchronises `stream` once. */
int lcd_shard_similarity_ids_dev(lcd_engine * e, const int * d_word_ids_all, int n_frames, int nq_per_frame, const int * d_sig_ids,
                                 int ns, int * d_pairs_out, int * d_valid_out, void * stream);
int lcd_shard_similarity_finalize_dev(lcd_engine * e, const int * d_pairs, const int * d_valid, const int * d_word_ids, int n_frames,
                                      int nq_per_frame, const float * d_frame_gdesc, const float * d_map_gdesc,
                                      const int * d_map_gdesc_row, int n_map_rows, int dim, const int * d_sig_ids, int ns,
                                      float * d_likelihood_out, void * stream);

/* ---- the exchanges behind the C ABI: one engine = one rank of a word-range-sharded job ----------------------------------
 * NCCL is loaded at run time (dlopen of libnccl.so.2: the host's own copy when it has one).  Bootstrap as any NCCL program: rank 0 calls
 * lcd_shard_unique_id, the host sends the 128 bytes to the other ranks over whatever channel it has (MPI, sockets, a file), every rank
 * calls lcd_shard_comm_init; or hand over a communicator the host already owns with lcd_shard_comm_adopt (ncclComm_t as void *). */
int lcd_shard_unique_id(char id_out[128]);
int lcd_shard_comm_init(lcd_engine * e, const char id[128], int rank, int n_ranks);
int lcd_shard_comm_adopt(lcd_engine * e, void * nccl_comm, int rank, int n_ranks);
int lcd_shard_comm_destroy(lcd_engine * e);
/* One step of the sharded job on this rank, entirely on the device: detect + describe the n_frames LOCAL frames, all-gather of the
 * descriptors, top-2 keys of every rank's descriptors over the local word range (lcd_shard_set_row_offset), all-to-all so that every rank
 * receives the keys of ITS frames, merge + NNDR / new-word pass of the local frames, all-gather of their word ids, TF-IDF of all frames
 * over the local word range, reduce-scatter of the exact 64-bit fixed-point sums, likelihood + verification of the local frames'
 * top hypotheses (results through lcd_process_fetch).  The dictionary search runs as two halves of the local batch so that the
 * descriptor and key exchanges (on the engine's communication stream) overlap a search kernel; the later stages run once on the whole
 * batch.  LCD_SHARD_TRACE=1|2 (environment) prints a per-stage timeline of the step to stderr.  d_row_ids_global: global row -> word id of the WHOLE dictionary
 * (rows of all ranks in ascending id order); d_word_ids_out[n_frames * n_features] (may be NULL), d_likelihood_out[n_frames * ns].
 * Every rank must call it with the same n_frames.  Results equal the unsharded engine's: word ids bit for bit, likelihood from the same
 * exact sums. */
int lcd_shard_process_frames_dev(lcd_engine * e, int n_frames, const uint8_t * d_images, int width, int height, int channels, const void * d_depth,
                                 int depth_type, const lcd_orb_params * params, int incremental, float nndr, int new_words_compared_together,
                                 const int * d_sig_ids, int ns, int n_total, const int * d_row_ids_global, int last_word_id,
                                 const lcd_verify_params * vp, int * d_word_ids_out, float * d_likelihood_out, void * stream);
/* The same step on descriptors the caller already has on the device, for binary and float engines alike: lcd_localize_batch_dev
 * semantics (quantise + score of n_frames independent LOCAL frames of nq_per_frame descriptors each, no mutation) with the dictionary and
 * the inverted index sharded by word range over the engine's communicator.  All-gather of the descriptors, top-2 keys over the local
 * word range, all-to-all of the keys (2 x u32 or 2 x u64 per query, see above), merge + NNDR / new-word pass of the local frames,
 * all-gather of their word ids, TF-IDF of all frames over the local word range, reduce-scatter of the exact fixed-point sums, likelihood
 * of the local frames.  No verification.  Every rank must call it with the same n_frames and nq_per_frame.  d_word_ids_out[n_frames *
 * nq_per_frame] (may be NULL), d_likelihood_out[n_frames * ns]: equal to lcd_localize_batch_dev on one unsharded engine (word ids bit
 * for bit, likelihood from the same exact sums). */
int lcd_shard_localize_batch_dev(lcd_engine * e, const void * d_queries, int n_frames, int nq_per_frame,
                                 int incremental, float nndr, int new_words_compared_together,
                                 const int * d_sig_ids, int ns, int n_total, const int * d_row_ids_global, int last_word_id,
                                 int * d_word_ids_out, float * d_likelihood_out, void * stream);
/* lcd_shard_localize_batch_dev with the similarity likelihood: equal bit for bit to lcd_localize_similarity_batch_dev on one unsharded
 * engine.  The exchanges of the descriptors, keys and word ids are those of lcd_shard_localize_batch_dev; then every rank counts the
 * word pairs of all frames over its word range and a reduce-scatter of int32 counts returns each rank the sums of its own frames, with
 * the ranks' valid(s) of the listed places summed in the same collective.  The dot products of the local frames' global descriptors
 * need no exchange.  Global descriptors as lcd_shard_similarity_finalize_dev (d_frame_gdesc of the LOCAL frames; the checks of the
 * row indices synchronise `stream` once per call when d_map_gdesc is given).  n_total has no role in the similarity likelihood and
 * is not taken. */
int lcd_shard_localize_similarity_batch_dev(lcd_engine * e, const void * d_queries, int n_frames, int nq_per_frame, int incremental,
                                            float nndr, int new_words_compared_together, const float * d_frame_gdesc,
                                            const float * d_map_gdesc, const int * d_map_gdesc_row, int n_map_rows, int dim,
                                            const int * d_sig_ids, int ns, const int * d_row_ids_global, int last_word_id,
                                            int * d_word_ids_out, float * d_likelihood_out, void * stream);

/* ---- epipolar verification of loop-closure hypotheses (VhEp/Enabled) ---------------------------------------------------------
 * EpipolarGeometry::check(A, B) (corelib/src/EpipolarGeometry.cpp:65-102) of a new signature A and a hypothesis B, from word ids and
 * keypoints alone (no depth, any descriptor type): findPairsUnique, the word ids >= 0 found exactly once in A and once in B, in
 * ascending id order; then cv::findFundamentalMat(FM_RANSAC, ransac_param1, ransac_param2) on their keypoints as OpenCV 4.13 runs it
 * (7 points: the 7-point kernel alone, mask all ones; 8-14: LMeDS; >= 15: RANSAC with 7-point samples, 1000 iterations at most); the
 * check passes with at least match_count_min inliers.  Where the reference itself fails, the check is a rejection: findFundamentalMat
 * returns no matrix (the reference asserts on the empty Mat), or OpenCV raises.  OpenCV raises when its 7-point kernel returns -1
 * models: the four coefficients of the determinant polynomial are exactly zero, which collinear points can cause.  raised flags the
 * inputs where the coefficients as computed here are exactly zero; they are not OpenCV's bits, so OpenCV raises on some inputs that
 * raised does not flag (53 of the 640 sets of the test corpus, all with many collinear points). */
typedef struct lcd_epipolar_params {
	int match_count_min;  /* VhEp/MatchCountMin (8) */
	double ransac_param1; /* VhEp/RansacParam1 (3): distance threshold, compared squared; <= 0 -> 3 as in findFundamentalMat */
	double ransac_param2; /* VhEp/RansacParam2 (0.99): confidence; outside (DBL_EPSILON, 1 - DBL_EPSILON) -> 0.99 */
} lcd_epipolar_params;

#define LCD_EPIPOLAR_NONE 0   /* fewer than 7 pairs or fewer than match_count_min: no fundamental matrix */
#define LCD_EPIPOLAR_7POINT 1 /* exactly 7 pairs */
#define LCD_EPIPOLAR_LMEDS 2  /* 8-14 pairs */
#define LCD_EPIPOLAR_RANSAC 3 /* 15 pairs or more */

typedef struct lcd_epipolar_result {
	int checked;        /* 1: the pair was checked */
	int ok;             /* EpipolarGeometry::check */
	int n_pairs;        /* findPairsUnique pairs */
	int n_inliers;      /* uSum(status) (0 when no matrix) */
	int method;         /* LCD_EPIPOLAR_* */
	int found;          /* findFundamentalMat returned a matrix (0 also where OpenCV raises) */
	int iterations_run; /* registrator iterations executed (0 for 7 pairs) */
	int raised;         /* a sample's 7-point kernel returned -1 models, where OpenCV raises (see above); a rejection here */
	double F[9];        /* the returned matrix, row-major (7 pairs: the first solution); zeros when none */
} lcd_epipolar_result;

/* EpipolarGeometry::check for n_pairs explicit (A = new, B = old) signatures.  ids_*[n_pairs][cap] word ids, uv_*[n_pairs][cap][2]
 * keypoints (row i = word i), n_*[n_pairs] rows used; out[n_pairs]; status_out[n_pairs][cap] (optional) the inlier mask in pair order.
 * LCD_ERR_INVALID for a count outside [0, cap]; LCD_ERR_CAPACITY for cap > 4096. */
int lcd_epipolar_check_batch(lcd_engine * e, int n_pairs, int cap, const int * ids_a, const float * uv_a, const int * n_a,
                             const int * ids_b, const float * uv_b, const int * n_b, const lcd_epipolar_params * p,
                             lcd_epipolar_result * out, uint8_t * status_out);

/* The stored places' words for the check inside the decision: Signature::getWords() / getWordsKpts() of each signature, word_ids[n_sigs][cap]
 * and uv[n_sigs][cap][2] (row i = word i), n[n_sigs] rows used.  A store of its own (no descriptors, no depth), so RGB-only callers and
 * float engines can fill it; adding an id again replaces its row, and slots of removed ids are reused.  LCD_ERR_INVALID for an id <= 0
 * or a count outside [0, cap]; LCD_ERR_CAPACITY for cap > 4096. */
int lcd_sig_words_add_batch(lcd_engine * e, const int * sig_ids, int n_sigs, int cap, const int * word_ids, const float * uv, const int * n);
int lcd_sig_words_remove(lcd_engine * e, int sig_id);
int lcd_sig_words_count(const lcd_engine * e);

#define LCD_DECIDE_EPIPOLAR_REJECTED 11 /* value over the threshold, EpipolarGeometry::check failed (Rtabmap.cpp:2193-2196) */

/* VhEp/Enabled on the last decision (Rtabmap.cpp:2193, between the single-hypothesis and the ratio rejections): every frame whose status
 * is ACCEPTED, RATIO or LAST_NULL is checked against its highest hypothesis in the word store (a hypothesis not stored is a signature
 * without words: 0 pairs).  A failed check makes the frame LCD_DECIDE_EPIPOLAR_REJECTED with loop id 0 and no hypothesis left for
 * lcd_verify_decided_dev; highest_id / highest_value stay.  A frame that passes keeps its status.  d_word_ids[n_frames][nq_per_frame]
 * (the frame's words, e.g. from lcd_localize_batch_dev), d_uv[n_frames][nq_per_frame][2], d_n_per_frame[n_frames]: device pointers.
 * Composition: a likelihood call, lcd_decide_batch_dev, lcd_decide_epipolar_dev, then optionally lcd_verify_decided_dev.
 * LCD_ERR_STATE without a decision; LCD_ERR_INVALID when n_frames differs from the last decision's; LCD_ERR_CAPACITY for
 * nq_per_frame > 4096. */
int lcd_decide_epipolar_dev(lcd_engine * e, const int * d_word_ids, const float * d_uv, const int * d_n_per_frame, int n_frames,
                            int nq_per_frame, const lcd_epipolar_params * p, void * stream);
/* the per-frame check results of the last lcd_decide_epipolar_dev (checked = 0: the frame did not reach the check) */
int lcd_epipolar_fetch(lcd_engine * e, int n_frames, lcd_epipolar_result * out);

/* ---- proximity detection by space (RGBD/ProximityBySpace) of many localisation clients --------------------------------------------
 * Rtabmap::process, Rtabmap.cpp:2698-2934, in localisation mode, for every frame of the last decision at once.
 *
 * The optimised poses of the map set by lcd_clients_set_map (Rtabmap::_optimizedPoses): ids[n] the map's real places in the same ascending
 * order (anything else: LCD_ERR_INVALID), poses[n][12] each place's rtabmap::Transform 3x4 row-major (a value that is not finite:
 * LCD_ERR_INVALID, the reference asserts there, Graph.cpp:2278), and each place's neighbour links in CSR form: nbr_ids[nbr_ptr[i] ..
 * nbr_ptr[i+1]) the places its kNeighbor / kNeighborMerged links point to (Signature::getLinks of those types, the links
 * Memory::getNeighborsId follows with ignoreLoopIds, Memory.cpp:1824-1845, and Memory::getNeighborLinks returns, :1521-1560).  Links to
 * places that are not in the map cannot join a path and are dropped.  Intermediate nodes (weight -1, Rtabmap/CreateIntermediateNodes)
 * are not supported.  A failed call (LCD_ERR_CAPACITY: no device memory) keeps the previous poses; a later lcd_clients_set_map makes
 * them stale and lcd_decide_proximity_dev returns LCD_ERR_STATE until poses are set for the new map. */
int lcd_clients_set_map_poses(lcd_engine * e, const int * ids, int n, const float * poses, const int64_t * nbr_ptr, const int * nbr_ids);

typedef struct lcd_proximity_params {
	float local_radius;              /* RGBD/LocalRadius (10 m; > 0) */
	float angle;                     /* RGBD/ProximityAngle (45 degrees; 0 = no angle filter) */
	int max_paths;                   /* RGBD/ProximityMaxPaths (3; 1..16: <= 0, unlimited in the reference, is LCD_ERR_CAPACITY) */
	int max_graph_depth;             /* RGBD/ProximityMaxGraphDepth (50; 0 = unlimited) */
	float path_filtering_radius;     /* RGBD/ProximityPathFilteringRadius (1 m; <= 0 = off) */
	float max_loop_closure_distance; /* RGBD/MaxLoopClosureDistance (0 = off): caps the filtering radius (Rtabmap.cpp:2822-2826) */
	const lcd_verify_params * verify; /* the registrations' parameters */
} lcd_proximity_params;

#define LCD_PROXIMITY_OFF 0      /* the frame's enabled flag was 0 */
#define LCD_PROXIMITY_RAN 1
#define LCD_PROXIMITY_CAPACITY 2 /* more than 1024 places inside RGBD/LocalRadius: the frame was not segmented, its decision is untouched */
#define LCD_PROXIMITY_LINK_LOCAL 1  /* Link::kLocalSpaceClosure */
#define LCD_PROXIMITY_LINK_GLOBAL 2 /* Link::kGlobalClosure: the accepted place is the global hypothesis (:2902-2906) */
#define LCD_DECIDE_PROXIMITY_SUPPRESSED 12 /* accepted, then a proximity detection was made near it on another place (:3193-3196) */

typedef struct lcd_proximity_path {
	float likelihood;  /* NearestPathKey (Rtabmap.cpp:1147-1176) of the path: its highest adjusted likelihood, */
	int id;            /*   the place that has it (ties: the smaller distance), */
	float distance;    /*   and (currentPoseInv * pose).getNormSquared() of that place */
	int candidate_id;  /* the place the registration was attempted with */
	int accepted;      /* registered, and the inverted transform's norm within the filtering radius */
	int link_type;     /* LCD_PROXIMITY_LINK_* of the link the reference adds, 0 when not accepted */
	lcd_verify_result result; /* Memory::computeTransform(candidate, frame) */
} lcd_proximity_path;

typedef struct lcd_proximity_result {
	int status;        /* LCD_PROXIMITY_* */
	int n_nearest;     /* places inside RGBD/LocalRadius (graph::findNearestNodes) */
	int n_paths;       /* paths of Rtabmap::getPaths */
	int n_attempts;    /* registrations attempted (localVisualPathsChecked) */
	int suppressed_id; /* loopIdSuppressedByProximity (0: none) */
	lcd_proximity_path paths[16]; /* the first n_attempts, in the order they were attempted */
} lcd_proximity_result;

/* Proximity detection on the last decision, after lcd_decide_batch_dev (and lcd_decide_epipolar_dev) and before lcd_verify_decided_dev.
 * Per frame with enabled[f] != 0 (the caller's check of Rtabmap.cpp:2698-2723: RGBD/ProximityBySpace, RGB-D SLAM mode, weight >= 0,
 * Rtabmap/StartNewMapOnLoopClosure, optimiser iterations, small displacement / too fast movement), frame_poses[f][12] the frame's
 * optimised pose (host arrays):
 *  1. graph::findNearestNodes(frame, poses, local_radius) (Graph.cpp:2239-2325): squared distances in float, x + y then + z, places with
 *     a squared distance < local_radius^2 (rtflann's radius result sets), ids >= 1.  In localisation mode the graph-depth filter of
 *     Rtabmap.cpp:2740-2789 does not run (Memory::isIncremental() is false) and no map place is in the short-term memory (:2773): the
 *     map's places are loaded into the working memory (Memory.cpp:262-272), the short-term memory holds the session's own frames (:1263).
 *  2. Rtabmap::getPaths (Rtabmap.cpp:5303-5382): the nearest place not in a path yet, Memory::getNeighborsId(it, max_graph_depth, ...)
 *     over neighbour links and through places within the radius only, then the reached places not in a path yet, in ascending id order,
 *     each admitted when it is the first or links to a place already admitted (one reachable only through a higher id waits for a later
 *     path).
 *  3. The paths' NearestPathKey from the decision's adjusted likelihood (0 for skipped or held frames, which computed none).
 *  4. The paths in descending key order (:2827-2934): graph::findNearestPoses with the radius and RGBD/ProximityAngle, the key's place
 *     when its likelihood is > 0 and it passed, else the nearest place left; attempted when closer than the filtering radius, until
 *     max_paths attempts.  The frame is never linked to a map place, so signature->hasLink does not fire.
 * All attempts of the batch are then registered in one launch (store rows as FROM, the frame's d_queries / d_uv rows as TO, as
 * lcd_verify_decided_dev takes them, null guess: RGBD/ProximityOdomGuess = false).  A registration is accepted when it succeeds and the
 * inverted transform's norm is within the filtering radius.  When the frame's decision is accepted and its place lies within the radius,
 * an accepted detection on it keeps the decision (its transform is the proximity path's; lcd_verify_decided_dev skips the frame), one on
 * another place makes it LCD_DECIDE_PROXIMITY_SUPPRESSED with loop id 0 (:2894-2911, :3193-3196).  Float transform inverses are
 * computed as [R^T | -R^T t]; the reference's Eigen inverse may differ in the last bits.
 * The registrations read row f of d_queries / d_uv for frame f in place (no copy); slots not attempted register nothing.
 * Binary engines only.  LCD_ERR_STATE without a decision, without poses for the current map, with an empty signature store, when the
 * decision already had its proximity step, or when it was already verified (lcd_verify_decided_dev, lcd_process_decide_batch_dev: the
 * proximity step comes first, as in the reference); LCD_ERR_INVALID for n_frames other than the decision's, bad parameters or a pose that
 * is not finite; LCD_ERR_CAPACITY for max_paths outside 1..16 or nq_per_frame > 4096. */
int lcd_decide_proximity_dev(lcd_engine * e, const void * d_queries, const float * d_uv, int n_frames, int nq_per_frame, const float * frame_poses,
                             const int * enabled, const lcd_proximity_params * pp, void * stream);
/* the per-frame results of the last lcd_decide_proximity_dev; synchronises */
int lcd_proximity_fetch(lcd_engine * e, int n_frames, lcd_proximity_result * out);

/* ---- the localisation step of Rtabmap::process from images, for many clients -------------------------------------------------
 * The optional stages of the decision inside lcd_process_frames_decide_*; a NULL member turns its stage off.  Host arrays, read before
 * the call returns. */
typedef struct lcd_decide_stages {
	const lcd_gps * frame_gps;              /* [n_frames]: Rtabmap/LoopGPS as lcd_decide_gps_batch_dev takes it (NULL: no GPS filter) */
	float local_radius;                     /* RGBD/LocalRadius of the GPS filter (>= 0) */
	const lcd_epipolar_params * epipolar;   /* VhEp/Enabled: lcd_decide_epipolar_dev (NULL: off) */
	const lcd_proximity_params * proximity; /* RGBD/ProximityBySpace: lcd_decide_proximity_dev (NULL: off), with */
	const float * frame_poses;              /*   [n_frames][12] each frame's optimised pose and */
	const int * proximity_enabled;          /*   [n_frames] the caller's conditions of Rtabmap.cpp:2698-2723 */
} lcd_decide_stages;

/* replaces: the localisation step of Rtabmap::process (Mem/IncrementalMemory=false) for n_frames frames of distinct clients, from their
 * device images (and depth), asynchronous on `stream`:
 *  1. Memory::update's detection with the engine's detector (lcd_detector_*) and its quantisation limit (lcd_quantize_limit_set), then
 *     Memory::computeLikelihood (Rtabmap.cpp:2117) against the map's real places (lcd_clients_set_map; ns must equal their number):
 *     word ids and likelihood rows bit-identical to lcd_process_frames with those ids as sig_ids;
 *  2. with stages->frame_gps, the GPS filter of the place list (:2046-2115), then adjustLikelihood, the client's Bayes posterior and the
 *     hypothesis selection (:2119-2226) as lcd_decide_gps_batch_dev (lcd_decide_batch_dev without GPS) decides them;
 *  3. with stages->epipolar, the epipolar check (:2193) on the frame's expanded word ids and keypoints, as lcd_decide_epipolar_dev;
 *  4. with stages->proximity, proximity detection by space (:2698-2934), as lcd_decide_proximity_dev, with each frame's own rows;
 *  5. Memory::computeTransform of the accepted hypotheses and its rejections (:3133-3191), as lcd_verify_decided_dev.
 * Registrations (steps 4 and 5) take each frame's n_kp detected rows as TO, with their depth (words3) when there is depth: the rows a
 * short frame pads with are never matched.  A frame without a quantised word is a bad signature (Signature::isBadSignature,
 * Signature.cpp:341-344): it is decided as LCD_FRAME_SKIP decides it (Rtabmap.cpp:1994-1999), found on the device, so the caller needs no
 * synchronisation to learn it: LCD_DECIDE_SKIPPED, highest (0, 0), its client's posterior untouched, no epipolar check, no proximity
 * detection (status LCD_PROXIMITY_OFF) and no registration.  clients[n_frames] and frame_flags[n_frames] as lcd_decide_batch_dev takes
 * them.  d_word_ids_out[n_frames][params->n_features] (expanded ids, negative for rows the limit did not quantise),
 * d_likelihood_out[n_frames][ns] and d_posterior_out[n_frames][ns+1] (not written for skipped, held and bad-signature frames) may be NULL.
 * This decision becomes the last decision: lcd_decide_fetch, lcd_process_fetch, lcd_epipolar_fetch and lcd_proximity_fetch read it.
 * Binary 32-byte engines only: float engines get LCD_ERR_INVALID (no image detector builds float descriptors), sharded engines
 * LCD_ERR_STATE.  LCD_ERR_STATE without clients or a map, with proximity but no poses for the current map, and for a GPS fix on a frame
 * that computes while the map has no GPS table; LCD_ERR_INVALID for a client listed twice and for bad parameters or arrays; these
 * refusals, and the epipolar check's shared-memory limit (LCD_ERR_CAPACITY), come before the decision changes any client state.  A
 * detector refusal of the image geometry (as lcd_orb_detect_describe_dev's) comes before it too, once the frame tables are uploaded.  The
 * registrations' own capacity limit (LCD_ERR_CAPACITY, as lcd_process_decide_batch_dev's) is met after the decision: the clients' state
 * has then advanced, as it has after a refused lcd_verify_decided_dev.  Not covered: the similarity likelihood (Kp/TfIdfLikelihoodUsed=false), mapping
 * mode, retrieval and intermediate nodes. */
int lcd_process_frames_decide_dev(lcd_engine * e, int n_frames, const uint8_t * d_images, int width, int height, int channels,
                                  const void * d_depth, int depth_type, const lcd_orb_params * params,
                                  int incremental, float nndr, int new_words_compared_together, int ns, int n_total,
                                  const lcd_verify_params * vp, const int * clients, const int * frame_flags, const lcd_decide_params * dp,
                                  const lcd_decide_stages * stages, int * d_word_ids_out, float * d_likelihood_out, float * d_posterior_out,
                                  void * stream);
/* The same from host images for a relocalisation service: _submit queues the batch and returns, lcd_process_frames_wait completes it.
 * It shares the two batches in flight of lcd_process_frames_submit (the two kinds may be interleaved; _wait always completes the oldest
 * batch, LCD_ERR_INVALID for a third).  Host outputs, each may be NULL, filled when the matching _wait returns: n_kp_out, word_ids_out and
 * likelihood_out shaped as lcd_process_frames' (word ids as lcd_process_frames_decide_dev's), decisions_out[n_frames],
 * results_out[n_frames] (the verification of the accepted hypotheses, as lcd_process_fetch), epipolar_out[n_frames] and
 * proximity_out[n_frames] (when those stages run, as lcd_epipolar_fetch / lcd_proximity_fetch).  Each batch stages its decision tables,
 * poses and flags in pinned buffers of its own, so a submit never waits for the batch in flight. */
int lcd_process_frames_decide_submit(lcd_engine * e, int n_frames, const uint8_t * images, int width, int height, int channels,
                                     const void * depth, int depth_type, const lcd_orb_params * params,
                                     int incremental, float nndr, int new_words_compared_together, int ns, int n_total,
                                     const lcd_verify_params * vp, const int * clients, const int * frame_flags, const lcd_decide_params * dp,
                                     const lcd_decide_stages * stages, int * n_kp_out, int * word_ids_out, float * likelihood_out,
                                     lcd_decision * decisions_out, lcd_verify_result * results_out, lcd_epipolar_result * epipolar_out,
                                     lcd_proximity_result * proximity_out);

/* ---- measurement hooks ---------------------------------------------------------------
 * Optional per-kernel timing with CUDA events recorded on the launching stream around
 * every launch of kernel class `which` (0 = dictionary NN, 1 = resolve, 2 = score, 3 = pair
 * matching, 4 = PnP RANSAC, 5 = all ORB kernels, 6 = the epipolar check, 7 = the proximity candidate kernel).
 * lcd_profile_read synchronises, returns the summed device time and the launch count
 * since the last reset. */
#define LCD_PROF_NN 0
#define LCD_PROF_RESOLVE 1
#define LCD_PROF_SCORE 2
#define LCD_PROF_MATCH 3
#define LCD_PROF_PNP 4
#define LCD_PROF_ORB 5
#define LCD_PROF_EPIPOLAR 6
#define LCD_PROF_PROXIMITY 7
int lcd_profile_enable(lcd_engine * e, int on);
int lcd_profile_read(lcd_engine * e, int which, double * total_ms, long long * launches);
int lcd_profile_reset(lcd_engine * e);

/* copy an internal ORB buffer of the last lcd_orb_* call back to the host (diagnostics / tests):
 * which = 0 gray pyramid, 1 mask pyramid, 2 blurred pyramid, 3 FAST candidate keys (after the selection: the survivors of the
 * first retainBest, in its order), 4 candidate counts, 5 keypoints per level counts, 6 survivors of the first retainBest per
 * level.  Returns the number of bytes copied (<= cap_bytes) or <0. */
long long lcd_debug_orb_buffer(lcd_engine * e, int which, void * out, long long cap_bytes);

/* engine stream (cudaStream_t as void*) and a full device sync, for harnesses */
void * lcd_stream(lcd_engine * e);
int lcd_synchronize(lcd_engine * e);

#ifdef __cplusplus
}
#endif
#endif /* LCD_B200_H */
