/*
 * bundletrack_b200.h — C-ABI of the H100-native (sm_90a) pose-graph optimizer + feature matcher that drops in behind
 * BundleTrack's C++ surface.  Plain pointers and sizes only; no C++/torch types.  Every entry point returns
 * BT_OK (0) or a negative bt_status — it never exits, throws or hangs (the reference does all three, SURVEY.md §5).
 *
 * The reference has no plugin/FFI layer; the "boundary" is the three C++ call sites where BundleTrack's host code
 * hands device work to something replaceable (SURVEY.md §8b).  Each entry point below names the call it replaces.
 * INTEGRATION.md shows the reference-side shim a maintainer adds at each site.
 *
 * Threading: a bt_ctx may be used by one host thread at a time.  All work is enqueued on the cudaStream_t passed
 * in (as void*); entry points that return host data synchronise that stream before returning.
 */
#ifndef BUNDLETRACK_B200_H
#define BUNDLETRACK_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif
#if defined(__GNUC__)
#define BT_API __attribute__((visibility("default")))
#else
#define BT_API
#endif

typedef enum {
	BT_OK = 0,
	BT_ERR_INVALID_ARG = -1,
	BT_ERR_CAPACITY = -2,     /* more windows / frames / correspondences / features than the context was created for */
	BT_ERR_CUDA = -3,         /* a CUDA runtime call failed; bt_last_error() has the string */
	BT_ERR_NO_DEVICE = -4,    /* no CUDA device, or not an sm_90 part: there is NO CPU fallback */
	BT_ERR_UNSUPPORTED = -5
} bt_status;

typedef struct bt_ctx bt_ctx;

/* One 3D-3D feature correspondence.  Layout-identical to the reference's `struct EntryJ`
 * (/root/reference/src/cuda/SIFTImageManager.h:44-59): 32 bytes, invalid <=> imgIdx_i == 0xFFFFFFFF. */
typedef struct {
	uint32_t imgIdx_i;
	uint32_t imgIdx_j;
	float pos_i[3];   /* camera-frame point in frame i, metres */
	float pos_j[3];
} bt_entryj;

/* Solver parameters, filled from the UNCHANGED config_*.yml keys (SURVEY.md §5):
 *   num_iter_outer  <- bundle.num_iter_outter      (Solver/CUDASolverBundling.cpp:193)
 *   num_iter_inner  <- bundle.num_iter_inner       (:210)
 *   robust_delta    <- bundle.robust_delta         (:214)
 *   image_downscale <- bundle.image_downscale      (LossGPU.cu:55)
 *   dense_dist_thresh        <- p2p.max_dist                       (CUDASolverBundling.cpp:93)
 *   dense_cos_normal_thresh  <- cos(p2p.max_normal_angle * pi/180) (:94)
 *   depth_min / depth_max    =  0.1 / 9999 (hard-wired, :97-98)
 *   w_sparse / w_dense       =  1 / 1      (hard-wired, SBA.cpp:28-30)                                   */
typedef struct {
	int num_iter_outer;
	int num_iter_inner;
	float robust_delta;
	float image_downscale;
	float dense_dist_thresh;
	float dense_cos_normal_thresh;
	float depth_min;
	float depth_max;
	float w_sparse;
	float w_dense;
} bt_solver_params;

/* One tracking window = one OptimizerGpu::optimizeFrames call (/root/reference/src/cuda/LossGPU.cu:53). */
typedef struct {
	int n_frames;                     /* N, frame 0 is the gauge (never moves) */
	int H, W;                         /* full-resolution image size */
	int n_corr;
	const bt_entryj* corr;            /* HOST pointer, n_corr entries (std::vector<EntryJ>::data()).  Pageable memory is copied
	                                   * during the call.  PAGE-LOCKED memory (cudaHostAlloc / cudaHostRegister /
	                                   * bt_host_alloc_pinned) is read in place by the copy engine - windows whose buffers follow
	                                   * each other share one transfer - and must stay unchanged until bt_solve_windows returns
	                                   * (split API: until bt_solve_fetch). */
	const float* const* depth_dev;    /* HOST array of N DEVICE pointers: Frame::_depth_gpu, float[H*W], metres, 0 = invalid */
	const float* const* normal_dev;   /* HOST array of N DEVICE pointers: Frame::_normal_gpu, float4[H*W], (nx,ny,nz,0) */
	float fx, fy, cx, cy;             /* K at full resolution */
	/* Dense point-to-plane pair list as (target, source) frame indices.  NULL => every unordered pair once with
	 * target = the larger index, which is what the reference's FindImageImageCorr_Kernel produces when the
	 * per-frame d_num_valid_points allocations have ascending addresses (SURVEY.md Q1).  n_dense_pairs == 0 with a
	 * non-NULL pointer disables the dense term for this window. */
	const uint32_t* dense_pairs;
	int n_dense_pairs;
	/* 1 => reproduce the reference's FlipJtJ behaviour: a pair's cross block survives only when target < source
	 * (SURVEY.md Q2).  0 => keep every cross block (the mathematically complete Gauss-Newton system). */
	int compat_flip;
	/* Optional: N slots of the context's frame cache (bt_frame_cache_store).  When non-NULL, depth_dev / normal_dev are not
	 * read: the quarter-resolution maps CUDACache::storeFrame (CUDACache.cpp:76-88) would rebuild for this call were built
	 * once per keyframe.  Results are bit-identical either way. */
	const int32_t* cache_slots;
	/* Optional: correspondences that are ALREADY ON THE DEVICE, as bt_match_pairs leaves them (SURVEY.md 8f rank 2): no entry
	 * crosses the PCIe bus.  corr_dev: DEVICE EntryJ array holding n_blocks blocks back to back; block b has block_n[b]
	 * entries that all carry (imgIdx_i, imgIdx_j) = (block_i[b], block_j[b]) and starts at block_off[b] (entries), with
	 * block_off[b+1] == block_off[b] + block_n[b].  block_* are HOST arrays - bt_match_pairs' n_entry_out / entry_off_out read
	 * back (a few dozen ints) and the pair list the caller gave it.  When corr_dev is non-NULL, corr / n_corr are ignored. */
	const bt_entryj* corr_dev;
	/* With HOST correspondences (corr_dev == NULL) block_n / n_blocks are optional too: the caller states that `corr` is n_blocks blocks
	 * back to back, block b holding block_n[b] entries of ONE (imgIdx_i, imgIdx_j) pair (read from the block's first entry, or from
	 * block_i / block_j when given) - what Bundler::optimizeGPU's n_match_per_pair describes (Bundler.cpp:298-351).  The library then
	 * skips its own grouping pass over the entries.  block_off is not read for host correspondences. */
	int n_blocks;
	const int32_t* block_off;
	const int32_t* block_n;
	const uint32_t* block_i;
	const uint32_t* block_j;
} bt_window;

typedef struct {
	int max_windows;        /* windows per bt_solve_* call */
	int max_frames;         /* frames per window (<= 32) */
	int max_corr;           /* correspondences per window */
	int H, W;               /* largest full-resolution frame */
	float image_downscale;  /* bundle.image_downscale */
} bt_solver_limits;

BT_API const char* bt_last_error(void);
BT_API int bt_version(void);

/* Create / destroy.  `device` is a CUDA ordinal.  The context owns every scratch buffer, so the per-call path does
 * no cudaMalloc/cudaFree (the reference does ~110 per call, SURVEY.md Q10).  A *_reserve refused for its arguments changes nothing; one
 * that fails while allocating (BT_ERR_CUDA) leaves its module refusing every call with BT_ERR_INVALID_ARG until a reserve succeeds. */
BT_API int bt_ctx_create(bt_ctx** out, int device);
BT_API void bt_ctx_destroy(bt_ctx* ctx);
BT_API int bt_solver_reserve(bt_ctx* ctx, const bt_solver_limits* lim);

/* Replaces OptimizerGpu::optimizeFrames (/root/reference/src/cuda/LossGPU.cu:53-139; caller
 * /root/reference/src/Bundler.cpp:350-351) for a BATCH of independent windows.
 * poses_inout: HOST, row-major 4x4 cam->model per frame, windows concatenated (sum of n_frames * 16 floats);
 * overwritten with the optimised poses of EVERY frame of the window, exactly like the reference's in-out vector.
 * Equivalent to bt_solve_stage + bt_solve_run + bt_solve_fetch. */
BT_API int bt_solve_windows(bt_ctx* ctx, int n_windows, const bt_window* windows, const bt_solver_params* params,
                     float* poses_inout, void* stream);

/* Streaming form: `begin` stages + launches a batch and queues the download of its poses, `end` waits for the OLDEST batch begun and
 * copies its poses (same layout as bt_solve_windows) to poses_out.  At most two batches may be in flight: the host side of batch k+1
 * then overlaps the GPU side of batch k.  The windows' host arrays (corr, pointer tables, block arrays) may be reused as soon as
 * `begin` returns unless they are page-locked and read in place (then: until the matching `end`). */
BT_API int bt_solve_windows_begin(bt_ctx* ctx, int n_windows, const bt_window* windows, const bt_solver_params* params,
                           const float* poses_in, void* stream);
BT_API int bt_solve_windows_end(bt_ctx* ctx, float* poses_out);

/* The same call split at the host<->device boundary, so a caller (and bench.py) can keep inputs resident:
 *   stage : host -> device copies of correspondences, poses, window tables (async on `stream`)
 *   run   : the kernels only (frame cache, plan, persistent GN/PCG solve); asynchronous
 *   fetch : device -> host copy of the poses + stream synchronise                                       */
BT_API int bt_solve_stage(bt_ctx* ctx, int n_windows, const bt_window* windows, const bt_solver_params* params,
                   const float* poses_in, void* stream);
BT_API int bt_solve_run(bt_ctx* ctx, void* stream);
BT_API int bt_solve_fetch(bt_ctx* ctx, float* poses_out, void* stream);

/* Introspection used by tests / bench (device pointers stay owned by the context). */
typedef struct {
	int n_windows;
	int n_tiles_total;         /* dense tiles per GN iteration over the batch */
	int n_kernel_launches;     /* kernels enqueued by the last bt_solve_run */
	long long n_src_pixels;    /* valid quarter-res source pixels summed over (window, pair) */
} bt_solve_stats;
BT_API int bt_solve_get_stats(bt_ctx* ctx, bt_solve_stats* out);
/* Copies the dense system (6N x 6N JtJ, row-major, reference ordering trans 0-2 / rot 3-5, and 6N Jtr) that the
 * LAST Gauss-Newton iteration of window `w` assembled; debugging/parity aid. */
/* Per-kernel device time of the last bt_solve_run (ms3 = {frame preparation incl. the tile plan, gap to the solve, persistent
 * solve}), from device-timer stamps the kernels write; opt-in.  bt_solve_get_timing synchronises the device. */
BT_API int bt_solve_enable_timing(bt_ctx* ctx, int on);
BT_API int bt_solve_get_timing(bt_ctx* ctx, float* ms3);
/* Host-side time of the last bt_solve_windows call, microseconds: us6 = {window tables + first upload, frame-preparation launch,
 * correspondence scan + staging + uploads, k_solve launch, pose download + wait for the GPU, whole call}. */
BT_API int bt_solve_get_host_timing(bt_ctx* ctx, double* us6);
/* Developer aid: in-kernel phase timestamps (clock64) of every tile and tail of the next runs; 12 int64 per record:
 * {kind<<32|cta, ids, t[10]}.  bt_solve_get_profile returns the number of records copied (>= 0) or a negative status. */
BT_API int bt_solve_enable_profile(bt_ctx* ctx, int max_records);
BT_API int bt_solve_get_profile(bt_ctx* ctx, long long* out, int max_records);
BT_API int bt_solve_enable_debug(bt_ctx* ctx, int on);
BT_API int bt_solve_debug_dense(bt_ctx* ctx, int w, float* JtJ_out, float* Jtr_out);
/* Number of dense correspondences each pair found in the last GN iteration of window `w` (gating parity aid). */
BT_API int bt_solve_debug_counts(bt_ctx* ctx, int w, int n_pairs, float* counts_out);
/* The system the PCG of the LAST Gauss-Newton iteration of window `w` solved, over the free frames 1..N-1 (dim = 6(N-1), per frame
 * trans 0-2 / rot 3-5): A (dim x dim, row-major, sparse + dense), the right-hand side, the Jacobi preconditioner (inverse diagonal)
 * and the PCG result delta before the Lie update.  `n_frames` is the frame count the outputs are sized for and must equal the
 * window's (BT_ERR_INVALID_ARG otherwise).  Any output may be NULL. */
BT_API int bt_solve_debug_system(bt_ctx* ctx, int w, int n_frames, float* A_out, float* rhs_out, float* minv_out, float* delta_out);

/* ------------------------------------------------------------------------------------------------------------
 * Matcher.  Replaces the two cv::cuda::DescriptorMatcher::knnMatch calls in SiftManager::findCorresbyNN
 * (/root/reference/src/FeatureManager.cpp:271-273) for a batch of frame pairs.
 * Distances are sqrt(sum d^2) like cv::NORM_L2, ascending; ties -> lower train index first.                  */
typedef struct {
	const float* dev;      /* DEVICE pointer, row-major n x dim (cv::cuda::GpuMat data), fp32 */
	int n;
	int dim;               /* 256 for LF-Net; must be a multiple of 32 */
	size_t pitch_bytes;    /* GpuMat::step; 0 => dim*4 */
} bt_desc_view;

BT_API int bt_matcher_reserve(bt_ctx* ctx, int max_pairs, int max_feats, int dim);
/* idxAB/distAB: DEVICE [sum_p nA_p * k] results for queries in A against train B; idxBA/distBA the reverse
 * direction.  ONE tensor-core contraction per pair serves both directions (rows of its accumulator tile are reduced for
 * A->B, columns for B->A).  Pair p's block starts at k * (sum of nA over pairs < p) (resp. nB).  Rows with fewer than k
 * candidates are padded with idx -1 / dist +inf. */
BT_API int bt_knn_match_pairs(bt_ctx* ctx, int n_pairs, const bt_desc_view* A, const bt_desc_view* B, int k,
                       int32_t* idxAB, float* distAB, int32_t* idxBA, float* distBA, void* stream);
/* Persistent descriptor pool (SURVEY.md 8f rank 3).  Lfnet::detectFeature uploads a frame's descriptors once
 * (/root/reference/src/FeatureManager.cpp:876-908); bt_desc_pool_store converts them ONCE into pool slot `slot` (fp16 rows for the
 * tensor pass, fp32 copy for the exact stage, norms, measured rounding errors - the caller's buffer is not referenced afterwards) and
 * bt_knn_match_slots / bt_match_pairs_pool then name slots: no per-call conversion.  Slots stay valid until overwritten or until
 * bt_matcher_reserve / bt_desc_pool_reserve re-size the pool.  The pool shares its blocks with the matcher's per-call slots: after a
 * bt_desc_pool_reserve that fails, every matcher call is refused until bt_matcher_reserve (then bt_desc_pool_reserve) succeeds. */
BT_API int bt_desc_pool_reserve(bt_ctx* ctx, int n_slots);
BT_API int bt_desc_pool_store(bt_ctx* ctx, int slot, const bt_desc_view* desc, void* stream);
BT_API int bt_knn_match_slots(bt_ctx* ctx, int n_pairs, const int32_t* slotA, const int32_t* slotB, int k,
                       int32_t* idxAB, float* distAB, int32_t* idxBA, float* distBA, void* stream);
/* Device time of the last kNN call: ms4 = {descriptor conversion, tensor-core pass, candidate selection + exact re-rank, exact
 * fallback}, info3 = {tensor-pass units (128 x 256 tiles), query rows, rows that needed the exact fallback}. */
BT_API int bt_knn_enable_timing(bt_ctx* ctx, int on);
/* Test knob: send every n-th query row through the exact brute-force fallback (0 = off).  Results do not change. */
BT_API int bt_knn_debug_force_fallback(bt_ctx* ctx, int every_nth);
BT_API int bt_knn_get_timing(bt_ctx* ctx, float* ms4, int* info3);

/* ------------------------------------------------------------------------------------------------------------
 * RANSAC.  Replaces ransacMultiPairGPU (/root/reference/src/cuda/cuda_ransac.cu:1228-1323; caller
 * /root/reference/src/FeatureManager.cpp:713).  ptsA/ptsB: HOST arrays of n_pairs DEVICE pointers to float4[n]
 * model-frame points (w ignored).  seed 0 => the reference's sampling sequence (XORWOW, curand_init(0, trial, 0)).
 * Winner = max inlier count, ties -> lowest trial id (the reference's findBestTrial is racy, SURVEY.md Q8).
 * inlier_ids_out: DEVICE int32 [sum n_pts] (pair p's list starts at sum of n_pts over pairs < p);
 * n_inliers_out: DEVICE int32 [n_pairs]. */
BT_API int bt_ransac_reserve(bt_ctx* ctx, int max_pairs, int max_pts, int max_trials);
BT_API int bt_ransac_pairs(bt_ctx* ctx, int n_pairs, const float* const* ptsA, const float* const* ptsB, const int* n_pts,
                    int n_trials, float dist_thresh, uint64_t seed, int32_t* inlier_ids_out, int32_t* n_inliers_out,
                    void* stream);
/* Parity aid: the three uniforms per trial the sampler used (same values as curand_uniform after
 * curand_init(seed, trial, 0)) and the winning trial id of every pair of the last call. */
BT_API int bt_ransac_debug(bt_ctx* ctx, float* u3_out, int n_trials, int32_t* best_trial_out, int n_pairs);
/* Parity aid: for pair `pair` of the last call (bt_ransac_pairs or the matcher chain), every trial's pose (poses_out [n_trials][12],
 * row-major [R | t]; a trial that is not good leaves its row as it was) and good flag (a model was fitted) of the first n_trials trials,
 * and the inlier count the winner was chosen with (-1 when no trial finished).  n_trials above the last call's is refused (BT_ERR_INVALID_ARG).  NULL outputs are skipped. */
BT_API int bt_ransac_debug_trials(bt_ctx* ctx, int pair, int n_trials, float* poses_out, int32_t* good_out, int32_t* best_count_out);

/* ------------------------------------------------------------------------------------------------------------
 * Geometric pruning + "mutual" union + the fused matcher pipeline.  Replaces SiftManager::pruneMatches and
 * collectMutualMatches (/root/reference/src/FeatureManager.cpp:290-368) and, fused, everything findCorres does
 * between the descriptors and the EntryJ loop of Bundler::optimizeGPU (/root/reference/src/Bundler.cpp:298-324). */
typedef struct {
	const float* kpts_dev;     /* DEVICE float2[n]: cv::KeyPoint::pt (x = column, y = row), Frame::_keypts */
	int n;
	const float* depth_dev;    /* DEVICE float[H*W]:  Frame::_depth_gpu */
	const float* normal_dev;   /* DEVICE float4[H*W]: Frame::_normal_gpu */
	float pose[16];            /* Frame::_pose_in_model, row-major cam->model */
	int frame_id;              /* Frame::_id; |idA - idB| == 1 selects the *_neighbor thresholds */
	int window_index;          /* index of this frame in the sorted BA window (EntryJ::imgIdx_*) */
} bt_match_frame;

typedef struct {               /* feature_corres.* of config_*.yml, angles already as cosines (FeatureManager.cpp:292-295) */
	float max_dist_no_neighbor, cos_max_normal_no_neighbor, max_dist_neighbor, cos_max_normal_neighbor;
} bt_prune_params;

typedef struct {               /* the reference's `Correspondence` (uA,vA,uB,vB,ptA_cam,ptB_cam), 40 bytes */
	float uA, vA, uB, vB;
	float ptA_cam[3];
	float ptB_cam[3];
} bt_correspondence;

BT_API int bt_pipeline_reserve(bt_ctx* ctx, int max_pairs, int max_feats, int dim, int max_trials);
/* A[p] is the NEWER frame of pair p (frameA->_id > frameB->_id, FeatureManager.cpp:175).  idxAB/idxBA: DEVICE kNN indices
 * as produced by bt_knn_match_pairs for the same pairs.  corr_out: DEVICE, pair p's block starts at sum_{q<p}(nA_q+nB_q)
 * and holds n_corr_out[p] entries: survivors of A->B in query order, then those of B->A (duplicates kept). */
BT_API int bt_prune_mutual_pairs(bt_ctx* ctx, int n_pairs, const bt_match_frame* A, const bt_match_frame* B, int H, int W,
                          float fx, float fy, float cx, float cy, const int32_t* idxAB, const int32_t* idxBA, int k,
                          const bt_prune_params* prm, bt_correspondence* corr_out, int32_t* n_corr_out, void* stream);
/* kNN -> prune -> mutual -> RANSAC -> EntryJ without leaving the device.  entry_out: DEVICE, pairs back to back
 * (entry_off_out[p], n_entry_out[p]; *total_out entries in all).  Pairs with <= 5 pruned matches or < 5 RANSAC
 * inliers contribute nothing (FeatureManager.cpp:575-579,233-241).  The list never exceeds entry_capacity: a pair that does not
 * fit is cut and (offset, count) describe what was written, so they can be handed on as bt_window::block_off / block_n as they
 * are; entry_capacity = sum over pairs of (nA + nB) can never truncate. */
BT_API int bt_match_pairs(bt_ctx* ctx, int n_pairs, const bt_match_frame* A, const bt_match_frame* B,
                   const bt_desc_view* dA, const bt_desc_view* dB, int H, int W, float fx, float fy, float cx, float cy,
                   const bt_prune_params* prune, int ransac_trials, float ransac_inlier_dist, uint64_t ransac_seed,
                   bt_entryj* entry_out, int entry_capacity, int32_t* n_entry_out, int32_t* entry_off_out,
                   int32_t* total_out, void* stream);
/* The same chain on descriptor sets stored with bt_desc_pool_store (slotA[p] / slotB[p] instead of descriptor views). */
BT_API int bt_match_pairs_pool(bt_ctx* ctx, int n_pairs, const bt_match_frame* A, const bt_match_frame* B,
                        const int32_t* slotA, const int32_t* slotB, int H, int W, float fx, float fy, float cx, float cy,
                        const bt_prune_params* prune, int ransac_trials, float ransac_inlier_dist, uint64_t ransac_seed,
                        bt_entryj* entry_out, int entry_capacity, int32_t* n_entry_out, int32_t* entry_off_out,
                        int32_t* total_out, void* stream);

/* The rest of SiftManager::findCorres (/root/reference/src/FeatureManager.cpp:173-242) around the same chain:
 *  - extra[p]: the matches findCorresByMapPoints (:489-520) would APPEND for a NON-neighbour pair - bt_tracks_propagate's output for
 *    (A[p].frame_id, B[p].frame_id) called with n_existing = 0; the device drops the ones whose (uA,vA) or (uB,vB) already occurs among
 *    the pair's mutual matches, looks the 3-D points up at round(u), round(v) and appends the rest before RANSAC.  Ignored for
 *    neighbour pairs (|idA - idB| == 1), as in the reference.
 *  - status_out[p] (DEVICE, optional): BT_PAIR_OK (>= 5 inliers), BT_PAIR_EMPTY (matches cleared, frame status unchanged) or
 *    BT_PAIR_FAIL (a neighbour pair ended with fewer than 5 matches: the reference marks frame A Frame::FAIL, :233-241,282-286).  The
 *    status is the match's outcome: a pair that entry_capacity cuts keeps it, and only n_entry_out[p] shows the cut.
 *  - uv_out (DEVICE float4 per emitted entry, optional): (uA, vA, uB, vB) of the entry - what updateFramePairMapPoints (:448-485) is fed
 *    through bt_tracks_update_pair. */
typedef struct { const float* uv; int n; } bt_match_extra;   /* HOST: n x (uA, vA, uB, vB) */
enum { BT_PAIR_OK = 0, BT_PAIR_EMPTY = 1, BT_PAIR_FAIL = 2 };
BT_API int bt_match_pairs_ex(bt_ctx* ctx, int n_pairs, const bt_match_frame* A, const bt_match_frame* B,
                      const bt_desc_view* dA, const bt_desc_view* dB, const int32_t* slotA, const int32_t* slotB,
                      int H, int W, float fx, float fy, float cx, float cy, const bt_prune_params* prune,
                      int ransac_trials, float ransac_inlier_dist, uint64_t ransac_seed, const bt_match_extra* extra,
                      bt_entryj* entry_out, int entry_capacity, int32_t* n_entry_out, int32_t* entry_off_out, int32_t* total_out,
                      int32_t* status_out, float* uv_out, void* stream);

/* Per-pair result cache: SiftManager::_matches (findCorres returns at once for a pair it has seen, FeatureManager.cpp:176;
 * forgetFrame drops a frame's pairs, :131-148).  Entries stay on the device; frames are named by Frame::_id.
 *   put     stores the blocks a bt_match_pairs* call produced (host copies of its n_entry / entry_off / status arrays).
 *   has     1 / 0 (BT_ERR_INVALID_ARG for a NULL ctx).
 *   gather  writes the cached blocks of the listed pairs back to back into dst_dev with imgIdx_i / imgIdx_j rewritten to the given
 *           window indices (a frame's index changes from window to window) and fills block_off / block_n for bt_window::corr_dev;
 *           pairs with no cached matches contribute empty blocks.
 *   usage   the pairs cached now and the entries their blocks hold.
 * The blocks live in one device arena of 32-B entries; each takes exactly its pair's entry count.  forget_frame gives a pair's block back.  A put
 * that finds no room behind the last block first moves the live blocks to the arena's start (a device-to-device copy on the put's stream, no
 * host synchronisation; gather's output does not change).  put returns BT_ERR_CAPACITY, and changes nothing, only when the pairs cached would
 * exceed max_pairs_cached, the live entries would exceed the arena, or a block is longer than the per-pair limit.
 *   bt_match_cache_reserve          arena of max_pairs_cached x max_entries_per_pair entries, per-pair limit max_entries_per_pair.
 *   bt_match_cache_reserve_entries  arena of max_entries_total entries (<= INT_MAX), no per-pair limit beyond that.
 * Both empty the cache; the arena takes 32 B per entry. */
BT_API int bt_match_cache_reserve(bt_ctx* ctx, int max_pairs_cached, int max_entries_per_pair);
BT_API int bt_match_cache_reserve_entries(bt_ctx* ctx, int max_pairs_cached, long long max_entries_total);
BT_API int bt_match_cache_usage(bt_ctx* ctx, int* n_pairs, long long* n_entries);
BT_API int bt_match_cache_put(bt_ctx* ctx, int n_pairs, const int32_t* idA, const int32_t* idB, const bt_entryj* entry_dev,
                       const int32_t* n_entry_host, const int32_t* entry_off_host, const int32_t* status_host, void* stream);
BT_API int bt_match_cache_has(bt_ctx* ctx, int idA, int idB);
BT_API int bt_match_cache_status(bt_ctx* ctx, int idA, int idB, int* n_entry, int* status);
BT_API int bt_match_cache_gather(bt_ctx* ctx, int n_pairs, const int32_t* idA, const int32_t* idB, const uint32_t* win_i, const uint32_t* win_j,
                          bt_entryj* dst_dev, int capacity, int32_t* block_off_host, int32_t* block_n_host, void* stream);
BT_API int bt_match_cache_forget_frame(bt_ctx* ctx, int frame_id);

/* ---- frame front end (SURVEY.md 8f rank 1): Frame::processDepth + Frame::depthToCloudAndNormals -------------------------
 * /root/reference/src/Frame.cpp:152-233 -> CUDAImageUtil::erodeDepthMap, gaussFilterDepthMap x2,
 * convertDepthFloatToCameraSpaceFloat4, computeNormals (src/cuda/CUDAImageUtil.cu:676-806,310-336,342-423), fused into
 * one kernel per batch of frames.  Parameters are config_*.yml "depth_processing" (erode.radius/diff/ratio,
 * bilateral_filter.radius/sigma_D/sigma_R). */
typedef struct {
	int erode_radius; float erode_diff, erode_ratio;
	int bf_radius; float sigma_D, sigma_R;
} bt_depth_params;
/* All map pointers are DEVICE memory; the pointer ARRAYS are host memory.  depth_raw/depth_out: H*W float (metres);
 * xyz_out (may be NULL: not wanted) and normal_out: H*W float4 = 4 floats per pixel ((x,y,z,1) / (nx,ny,nz,0), zeros
 * where undefined) - depth_out and normal_out are exactly Frame::_depth_gpu / _normal_gpu as the solver reads them.
 * Out of place: depth_out[f] must differ from depth_raw[f]. */
BT_API int bt_frames_preprocess(bt_ctx* ctx, int n_frames, const float* const* depth_raw_dev, int H, int W,
                         float fx, float fy, float cx, float cy, const bt_depth_params* prm,
                         float* const* depth_out_dev, float* const* xyz_out_dev, float* const* normal_out_dev, void* stream);

/* ---- object mask: Frame::segmentationByMaskFile + Frame::invalidatePixelsByMask (reference src/Frame.cpp:267-374) -----------
 * mask_dev: DEVICE uint8 H*W per frame as cv::imread(IMREAD_UNCHANGED) returns the mask PNG, non-zero = object.
 * BT_MASK_LARGEST_HULL (the reference's NOCS datasets): the largest 8-connected component of mask != 0 (ties: the component whose
 * first pixel in row-major order comes first), replaced by cv::fillConvexPoly of its convex hull (0/1); an empty mask stays empty.
 * BT_MASK_AS_IS (every other dataset): the mask as given.  Then fg = cv::dilate(mask, 5 x 5 rectangle) = Frame::_fg_mask, written to
 * fg_out_dev (DEVICE uint8 H*W per frame; must not alias mask_dev), and roi_out_dev (DEVICE int32 [n_frames][4]) = Frame::_roi =
 * (umin, umax, vmin, vmax) of fg != 0, (9999, 0, 9999, 0) when fg is empty.  The maps are exactly bt_frames_preprocess's with depth,
 * xyz and normal zeroed where fg == 0 (computed from the unmasked depth first, as in the reference).  Asynchronous like
 * bt_frames_preprocess: the ROI stays on the device for bt_lfnet_request; read it back when the tracker's gate needs it
 * (umax - umin < 10 || vmax - vmin < 10 -> Frame::FAIL, Bundler.cpp:88-93).  Largest-hull mode keeps label scratch in the context,
 * grown on the first call at a size. */
enum { BT_MASK_AS_IS = 0, BT_MASK_LARGEST_HULL = 1 };
BT_API int bt_frames_preprocess_masked(bt_ctx* ctx, int n_frames, const float* const* depth_raw_dev, const uint8_t* const* mask_dev, int mask_mode,
                         int H, int W, float fx, float fy, float cx, float cy, const bt_depth_params* prm, float* const* depth_out_dev,
                         float* const* xyz_out_dev, float* const* normal_out_dev, uint8_t* const* fg_out_dev, int32_t* roi_out_dev, void* stream);
/* bt_frames_preprocess_masked on the depth PNG's samples: depth_mm_dev is DEVICE uint16 H*W per frame as cv::imread(path, IMREAD_ANYDEPTH)
 * returns a 16-bit depth PNG (millimetres).  The kernel converts each sample as Utils::readDepthImage does (Utils.cpp:57-66):
 * d = (float)((double)s * 0.001), 0 where (double)d < 0.1.  Every output is bit for bit what bt_frames_preprocess_masked gives on that float
 * image; the upload is half the bytes and the host does no per-pixel work. */
BT_API int bt_frames_preprocess_masked_u16(bt_ctx* ctx, int n_frames, const uint16_t* const* depth_mm_dev, const uint8_t* const* mask_dev, int mask_mode,
                         int H, int W, float fx, float fy, float cx, float cy, const bt_depth_params* prm, float* const* depth_out_dev,
                         float* const* xyz_out_dev, float* const* normal_out_dev, uint8_t* const* fg_out_dev, int32_t* roi_out_dev, void* stream);
/* Lfnet::detectFeature's request image (src/FeatureManager.cpp:813-873, rot_deg = 0): the colour zeroed where fg == 0, cropped to
 * [vmin, vmax) x [umin, umax) of roi_dev (the reference's crop drops the last row and column), padded with zeros to a square and
 * resized to 400 x 400 as cv::resize(INTER_LINEAR) does on 8-bit images.  colour_dev: DEVICE uint8 H*W*3 BGR (cv::Mat CV_8UC3 data);
 * fg_dev / roi_dev: bt_frames_preprocess_masked's outputs; request_out_dev: DEVICE uint8 400*400*3 per frame, the bytes of the second
 * message part of the request.  Frames whose roi fails the tracker's 10-pixel gate are left untouched.  Asynchronous. */
BT_API int bt_lfnet_request(bt_ctx* ctx, int n_frames, const uint8_t* const* colour_dev, const uint8_t* const* fg_dev, const int32_t* roi_dev,
                         int H, int W, uint8_t* const* request_out_dev, void* stream);

/* Frame cache (SURVEY.md 8f rank 1, second half).  The reference re-creates a CUDACache and re-downsamples every keyframe of
 * the window in EVERY optimizeFrames call (/root/reference/src/cuda/LossGPU.cu:74-101, CUDACache.cpp:76-88); a keyframe
 * takes part in many windows, so its quarter-resolution point/normal texel map and compacted source list are built here
 * once, when the keyframe enters the pool, and referenced by slot from bt_window::cache_slots.  The cache belongs to the
 * solver of this context: call bt_solver_reserve first.  Slots stay valid until overwritten.  depth_min/depth_max:
 * bt_solver_params::depth_min/max (they define which pixels enter the source list). */
BT_API int bt_frame_cache_reserve(bt_ctx* ctx, int capacity, int H, int W, float image_downscale);
BT_API int bt_frame_cache_store(bt_ctx* ctx, int n_frames, const int32_t* slots, const float* const* depth_dev, const float* const* normal_dev,
                         int H, int W, float fx, float fy, float cx, float cy, float depth_min, float depth_max, void* stream);

/* ---- host-side policy around the path (SURVEY.md 8f rank 4): plain host code, callable without a GPU -----------------------------
 * Poses are row-major 4x4 cam->model.  keyframe_poses: n_keyframes consecutive 4x4 matrices. */
/* Utils::rotationGeodesicDistance (/root/reference/src/Utils.cpp:42-47): angle between the two rotations, radians. */
BT_API float bt_rotation_geodesic(const float* pose_a, const float* pose_b);
/* Bundler::checkAndAddKeyframe (/root/reference/src/Bundler.cpp:185-221): 1 = the frame becomes a keyframe (frame 0 always; otherwise
 * enough keypoints and at least min_rot_deg degrees away from EVERY existing keyframe), 0 = not.  The caller applies the
 * reference's `_status == OTHER` test. */
BT_API int bt_keyframe_check(const float* pose_new, int frame_id, int n_keypts, const float* keyframe_poses, int n_keyframes,
                      int min_feat_num, float min_rot_deg);
/* Bundler::selectKeyFramesForBA, method "greedy_rot" (Bundler.cpp:224-274): indices (ascending) of the keyframes that join the new
 * frame in the window; at most max_BA_frames - 1 of them.  chosen_out needs room for n_keyframes entries. */
BT_API int bt_select_keyframes(const float* pose_new, const float* keyframe_poses, int n_keyframes, int max_BA_frames,
                        int32_t* chosen_out, int* n_chosen_out);
/* Utils::solveRigidTransformBetweenPoints (Utils.cpp:180-214), the closed form behind SiftManager::procrustesByCorrespondence
 * (FeatureManager.cpp:523-557): pose_out (row-major 4x4) maps pts1 onto pts2 (n x 3 each) in the least-squares sense; identity when
 * the fit degenerates, as in the reference. */
BT_API int bt_rigid_transform(const float* pts1, const float* pts2, int n, float* pose_out);

/* The gate in front of the optimizer in Bundler::optimizeGPU (/root/reference/src/Bundler.cpp:343-347): bundle adjustment runs only when
 * the new frame takes part in MORE than min_fm_edges_newframe correspondences of the window; otherwise the frame's status becomes
 * Frame::NO_BA and the poses stay as they are.  n_edges_newframe = number of EntryJ records with the new frame on either side
 * (bt_match_cache_gather / FindCorres report it).  Returns 1 = run bt_solve_windows, 0 = NO_BA. */
BT_API int bt_ba_gate(int n_edges_newframe, int min_fm_edges_newframe);
/* Bundler::saveNewframeResult's pose record (/root/reference/src/Bundler.cpp:362-378): ob_in_cam = inverse(cur_in_model) as text, the 4 x 4
 * matrix printed the way `ofstream << std::setprecision(10) << Eigen::Matrix4f` prints it (10 significant digits, columns right-aligned
 * to the widest coefficient, one row per line).  bt_pose_format writes at most `cap` bytes incl. the terminating 0 into `text` and
 * returns BT_ERR_CAPACITY when it does not fit (1024 is always enough); bt_pose_write_txt writes `path` (the caller creates
 * <debug_dir>/poses/ as the reference does). */
BT_API int bt_pose_format(const float* cur_in_model, char* text, int cap);
BT_API int bt_pose_write_txt(const char* path, const float* cur_in_model);

/* Lfnet::detectFeature's reply handling (/root/reference/src/FeatureManager.cpp:876-907; rot_deg = 0, the only value the tracker uses):
 * validates the three message parts of the LF-Net server's reply (int32 (n, dim) | float32 n x 2 keypoints in the 400 x 400 network
 * input | float32 n x dim descriptors) and maps the keypoints back to image pixels through the crop / pad-to-square / resize
 * transform of `roi` = Frame::_roi (umin, umax, vmin, vmax).  kpts_out: n x 2 floats (x, y).  The descriptor part is already the
 * row-major matrix bt_knn_match_pairs takes: upload it as it is (bt_memcpy_h2d). */
BT_API int bt_lfnet_parse_reply(const void* info, size_t info_bytes, const void* kpts, size_t kpts_bytes, size_t desc_bytes, const int* roi,
                         float* kpts_out, int kpts_capacity, int* n_out, int* dim_out);

/* Map-point bookkeeping between matching and RANSAC (SURVEY.md 8f rank 2; host code, no GPU):
 * SiftManager::updateFramePairMapPoints / findCorresByMapPoints / the map-point part of forgetFrame
 * (/root/reference/src/FeatureManager.cpp:448-520,163-169).  Frames are named by Frame::_id; uv arrays hold (uA, vA, uB, vB) per
 * match, A = the newer frame.  bt_tracks_propagate returns the matches findCorresByMapPoints would APPEND for the pair (map points
 * seen in both frames whose (uA,vA) and (uB,vB) are not matched yet), in the reference's order; the caller looks the 3-D points up
 * at round(u), round(v) of its point maps exactly as the reference does and hands them to RANSAC with the rest. */
typedef struct bt_tracks bt_tracks;
BT_API int bt_tracks_create(bt_tracks** out);
BT_API void bt_tracks_destroy(bt_tracks* t);
BT_API int bt_tracks_update_pair(bt_tracks* t, int frame_a, int frame_b, const float* uv, const unsigned char* is_inlier, int n);
BT_API int bt_tracks_propagate(bt_tracks* t, int frame_a, int frame_b, const float* existing_uv, int n_existing,
                        float* out_uv, int capacity, int* n_out);
BT_API int bt_tracks_forget_frame(bt_tracks* t, int frame);
BT_API int bt_tracks_stats(const bt_tracks* t, int* n_points, int* n_observations);

/* The same table on the device, owned by the context, with the same results as bt_tracks (output bits and order included).  Everything is
 * asynchronous on `stream` except stats; use one stream for a context's table.
 *   reserve       capacities: frames alive (<= 64), keys per frame (<= 8192), map points alive.  Empties the table.  Nothing is allocated
 *                 later.  The table takes max_points x max_frames x 8 B of observations plus max_frames x max_keys_per_frame x 48 B of frame maps
 *                 (and 20 B per point).
 *   reserve_ex    the same with max_frames up to 64 + 1024 (BT_ERR_INVALID_ARG above that).  A call that would exceed a capacity changes nothing and latches a flag: the next bt_tracks_dev_stats returns
 *                 BT_ERR_CAPACITY (and clears it).  Frames are mapped to slots on the host; a frame past the limit fails at once.
 *   update_pair   uv_dev: DEVICE (uA, vA, uB, vB) per match, *n_dev (DEVICE) of them, at most uv_capacity; so it can follow an emit without
 *                 a synchronisation.  Keys must not be NaN.
 *   propagate     bt_tracks_propagate with existing_uv_dev / out_uv_dev DEVICE and the count written to *n_out_dev.
 *   stats         synchronises the stream; n_points counts every map point ever created, as bt_tracks_stats does. */
BT_API int bt_tracks_dev_reserve(bt_ctx* ctx, int max_frames, int max_keys_per_frame, int max_points);
BT_API int bt_tracks_dev_reserve_ex(bt_ctx* ctx, int max_frames, int max_keys_per_frame, int max_points);
BT_API int bt_tracks_dev_update_pair(bt_ctx* ctx, int frame_a, int frame_b, const float* uv_dev, const int32_t* n_dev, int uv_capacity, void* stream);
BT_API int bt_tracks_dev_propagate(bt_ctx* ctx, int frame_a, int frame_b, const float* existing_uv_dev, int n_existing,
                            float* out_uv_dev, int capacity, int32_t* n_out_dev, void* stream);
BT_API int bt_tracks_dev_forget_frame(bt_ctx* ctx, int frame, void* stream);
BT_API int bt_tracks_dev_stats(bt_ctx* ctx, int* n_points, int* n_observations, void* stream);

/* SiftManager::findCorres for an ORDERED list of pairs on the context's device table (Bundler::optimizeGPU's loop, Bundler.cpp:298-305):
 * bt_match_pairs_ex's arguments without `extra` - a non-neighbour pair's propagated matches come from the table as the earlier pairs of
 * the same call left it, and every pair with status BT_PAIR_OK updates the table with its emitted entries.  The outputs equal those of
 * calling bt_match_pairs_ex one pair at a time in the same order (propagated matches from bt_tracks_propagate, bt_tracks_update_pair fed
 * from uv_out), with the pairs back to back in entry_out.  Needs bt_pipeline_reserve and bt_tracks_dev_reserve; A[p].frame_id >
 * B[p].frame_id.  No device-to-host copy and no synchronisation inside the call. */
BT_API int bt_find_corres_pairs(bt_ctx* ctx, int n_pairs, const bt_match_frame* A, const bt_match_frame* B,
                         const bt_desc_view* dA, const bt_desc_view* dB, const int32_t* slotA, const int32_t* slotB,
                         int H, int W, float fx, float fy, float cx, float cy, const bt_prune_params* prune,
                         int ransac_trials, float ransac_inlier_dist, uint64_t ransac_seed,
                         bt_entryj* entry_out, int entry_capacity, int32_t* n_entry_out, int32_t* entry_off_out, int32_t* total_out,
                         int32_t* status_out, float* uv_out, void* stream);

/* SiftManager::procrustesByCorrespondence (the reference's src/FeatureManager.cpp:523-557) plus the pose update after it (Bundler.cpp:134-135)
 * on the device, for one pair as bt_find_corres_pairs leaves it: entry_dev / n_entry_dev / status_dev are the pair's EntryJ block (pos_j =
 * the newer frame A's camera point, pos_i = the older frame B's), its count and its BT_PAIR_* status, all DEVICE memory.  pose_a / pose_b:
 * HOST row-major cam->model poses of A and B.  src = pose_a * pos_j and dst = pose_b * pos_i per entry, each coordinate
 * ((m0 x + m1 y) + m2 z) + m3 in float; offset = bt_rigid_transform(src, dst) bit for bit, or the identity when the status is not BT_PAIR_OK;
 * pose_out_dev (DEVICE, 16 floats) = offset * pose_a, each element ((o0 p0 + o1 p1) + o2 p2) + o3 p3 in float.  Asynchronous; one CTA. */
BT_API int bt_pose_init(bt_ctx* ctx, const bt_entryj* entry_dev, const int32_t* n_entry_dev, const int32_t* status_dev, const float* pose_a,
                        const float* pose_b, float* pose_out_dev, void* stream);

/* ---- the whole tracking step: Bundler::processNewFrame (the reference's src/Bundler.cpp:56-183) as one object -------------------------
 * A tracker owns its own bt_ctx and reserves everything in bt_tracker_create, for frames of H x W with at most max_feats keypoints and
 * 256-dimensional descriptors.  With S = max_frames_alive + max_keyframes frame slots: S + 1 sets of full-resolution maps (depth, normals,
 * foreground mask: 25 B per pixel) with their keypoints and descriptor-pool slots (1 KB per feature), S frame-cache slots, the device map-point
 * table (S frames, 16 x max_feats x ceil(S / 64) points: S x points x 8 B of observations), the match cache and the matcher and solver for
 * windows of max_BA_frames frames.  The match cache holds every pair of S frames at 3 x max_feats entries of 32 B each when max_keyframes = 0,
 * and S x max_BA_frames x 3 x max_feats / 2 entries in all (max_BA_frames / 2 worst-case blocks per frame slot) otherwise.
 * At 640 x 480, 2000 features, max_frames_alive = 32 and max_BA_frames = 15 that is roughly 0.6 GB: 0.25 GB of frame maps, 0.1 GB each of
 * descriptor pool and match cache, the rest matcher and solver scratch.  One frame slot costs about 11.7 MB at 640 x 480 with 2000 features
 * (7.7 MB of maps, 3.1 MB of descriptor pool, 0.9 MB of frame cache), plus 0.26 MB x ceil(S / 64) of map-point observations and 1.4 MB of
 * match cache at max_BA_frames = 15: max_frames_alive = 8 with max_keyframes = 256 reserved 4.65 GB in all (DESIGN.md §9.5).
 * A frame's step is split where the reference calls the LF-Net server: begin_frame (id, pose, segmentation, the 10-pixel ROI gate and the
 * request image) and end_frame (descriptors, findCorres on the neighbour pair, the initial pose on the device, the frame deque, keyframe
 * selection, findCorres on the window, the BA gate, the solve, keyframe admission).  Poses are row-major 4 x 4 cam->model. */
typedef struct bt_tracker bt_tracker;
typedef struct {
	int H, W; float fx, fy, cx, cy;
	int max_feats;                 /* keypoints per frame */
	int max_frames_alive;          /* 2..64.  max_keyframes = 0: the frames held at once during a step, keyframes + the recent-frame deque + the
	                                * new frame.  max_keyframes > 0: the same without the keyframes.  The oldest recent frame is released only after
	                                * the new frame's neighbour pair is matched, as in the reference, so it counts too. */
	int mask_mode;                 /* BT_MASK_AS_IS / BT_MASK_LARGEST_HULL */
	bt_depth_params depth; bt_solver_params solver; bt_prune_params prune;
	int ransac_trials; float ransac_inlier_dist;
	int window_size, max_BA_frames, min_fm_edges_newframe, min_feat_num; float min_rot_deg;
	int max_keyframes;             /* 0..1024.  0: keyframes count against max_frames_alive (at most 64 frames alive in all).  > 0: a keyframe pool of
	                                * this many, held apart from max_frames_alive; the reference never releases a keyframe, so this bounds the
	                                * sequence's keyframes.  Value-initialise the struct (= {0}) so older callers get 0. */
} bt_tracker_params;
enum { BT_FRAME_OTHER = 0, BT_FRAME_FAIL = 1, BT_FRAME_NO_BA = 2 };   /* Frame::_status */
/* BT_ERR_NO_DEVICE without an sm_90 GPU; BT_ERR_INVALID_ARG for parameters out of range (max_BA_frames 2..32, max_frames_alive 2..64,
 * max_keyframes 0..1024), checked before the device is looked at. */
BT_API int bt_tracker_create(bt_tracker** out, int device, const bt_tracker_params* p);
BT_API void bt_tracker_destroy(bt_tracker* t);
/* The new frame's id and pose: the last frame's id + 1 and its pose when the tracker holds frames, else loader_id and first_pose (identity when
 * NULL).  depth_raw_dev (float H*W, metres), mask_dev (uint8 H*W, the mask PNG's bytes), colour_dev (uint8 H*W*3 BGR): DEVICE.  Writes the ROI
 * (umin, umax, vmin, vmax) to roi_out (host, optional) after one synchronisation.  A frame that fails the 10-pixel gate gets BT_FRAME_FAIL: the
 * tracker keeps nothing of it, so the next frame gets the same id.  Otherwise request_out_dev (DEVICE uint8 400*400*3) receives the LF-Net
 * request image and *status_out = BT_FRAME_OTHER; finish the frame with end_frame or drop_frame. */
BT_API int bt_tracker_begin_frame(bt_tracker* t, int loader_id, const float* first_pose, const float* depth_raw_dev, const uint8_t* mask_dev,
                                  const uint8_t* colour_dev, uint8_t* request_out_dev, int32_t* roi_out, int* status_out, void* stream);
/* bt_tracker_begin_frame on the depth PNG's uint16 millimetres (DEVICE H*W; converted as bt_frames_preprocess_masked_u16 does).  Also writes
 * the new frame's id to id_out and its initial pose (cam->model, 16 floats) to pose_out, for every status (both host, optional).  A frame
 * that fails the ROI gate still has that pose: Bundler::saveNewframeResult records it (Bundler.cpp:362-377). */
BT_API int bt_tracker_begin_frame_u16(bt_tracker* t, int loader_id, const float* first_pose, const uint16_t* depth_mm_dev, const uint8_t* mask_dev,
                                      const uint8_t* colour_dev, uint8_t* request_out_dev, int32_t* roi_out, int* id_out, float* pose_out, int* status_out,
                                      void* stream);
/* kpts_host: n_kpts x (x, y) image pixels (bt_lfnet_parse_reply's output); desc: the n_kpts x 256 descriptors on the device.  Writes the frame's
 * pose as Bundler::saveNewframeResult would record it and its status.  BT_ERR_INVALID_ARG without a pending begin_frame, for n_kpts > max_feats
 * or a NULL argument.  BT_ERR_CAPACITY when max_keyframes = 0 and the frames alive plus the new one exceed max_frames_alive, or when
 * max_keyframes > 0 and either the frames alive that are not keyframes plus the new one exceed max_frames_alive or the keyframe pool is full
 * (the new frame might be admitted).  Both change nothing: the frame stays pending. */
BT_API int bt_tracker_end_frame(bt_tracker* t, const float* kpts_host, int n_kpts, const bt_desc_view* desc, float* pose_out, int* status_out, void* stream);
/* Lfnet::detectFeature threw: the pending frame becomes FAIL and is forgotten (Bundler.cpp:108-116).  pose_out (optional): its pose. */
BT_API int bt_tracker_drop_frame(bt_tracker* t, float* pose_out);
/* Every frame alive (the deque and the keyframes), oldest first: ids, poses (16 floats each) and whether it is a keyframe.  *n = the count;
 * BT_ERR_CAPACITY when it exceeds cap (the arrays may be NULL when cap is 0). */
BT_API int bt_tracker_state(bt_tracker* t, int32_t* ids, float* poses, int32_t* is_keyframe, int cap, int* n);
/* What the tracker's tables hold now: map points alive, pairs in the match cache and the entries of their blocks.  Synchronises `stream`. */
BT_API int bt_tracker_usage(bt_tracker* t, int* n_points, int* n_pairs_cached, long long* n_entries_cached, void* stream);
/* Frame::_fg_mask (DEVICE uint8 H*W, 0 = background) of the frame the last begin_frame segmented, whatever became of it: a frame that failed
 * the ROI gate or was dropped included.  Valid until the next begin_frame on the tracker's stream; read it with work enqueued on that stream
 * before then (bt_pose_overlay for the reference's LOG frames).  BT_ERR_INVALID_ARG before the first begin_frame. */
BT_API int bt_tracker_last_fg(bt_tracker* t, const uint8_t** fg_dev);
/* The processed depth (DEVICE float32 H*W, metres, 0 = none or masked out: what the solver reads) of frame frame_id, which must be alive
 * (bt_tracker_state lists it).  Valid until the frame is released: for a keyframe, until the tracker is destroyed; otherwise until a later
 * end_frame slides it out of the deque.  Read it with work enqueued on the tracker's stream (bt_tsdf_fuse for an object model).
 * BT_ERR_INVALID_ARG for a NULL argument or an id that is not alive. */
BT_API int bt_tracker_frame_depth(bt_tracker* t, int frame_id, const float** depth_dev);

/* ---- pose accuracy: the reference's evaluation (scripts/Utils.py add / adi, scripts/eval_ycbineoat.py VOCap) -------------------------
 * bt_pose_metrics: per frame f, ADD = mean_i |gt_f p_i - pred_f p_i| and ADD-S = mean_i min_j |gt_f p_i - pred_f p_j| over the model points p,
 * in metres, float64.  ADD-S is the exact nearest neighbour (brute force on the device, an fp32 filter whose rounding is bounded, then the
 * candidates it keeps in float64; DESIGN.md §3.7): equal to a float64 k-d tree query up to float64 rounding.
 *   model_pts_dev  DEVICE float64 n_pts x 3 (the rows of points.xyz), finite.
 *   pred / gt      HOST row-major 4 x 4 ob_in_cam per frame (model -> camera: what poses/<id>.txt and bt_pose_write_txt hold), n_frames
 *                  of each back to back.  The last row is not read.
 *   add_out / adds_out  DEVICE float64 [n_frames].
 * Asynchronous on `stream`: the poses are copied before the call returns (the host arrays may be reused at once), the results are ready
 * when the stream is.  BT_ERR_INVALID_ARG for n_pts < 1, n_frames < 1, a NULL pointer, a non-finite pose element, or a context without
 * bt_metrics_reserve; BT_ERR_CAPACITY above the reserved sizes.
 * bt_metrics_reserve: scratch for up to max_pts model points (<= 67,107,840) and max_frames frames per call: 16 B per point, 304 B per
 * frame (device and pinned host) and 16 B per frame per 1024 points. */
BT_API int bt_metrics_reserve(bt_ctx* ctx, int max_pts, int max_frames);
BT_API int bt_pose_metrics(bt_ctx* ctx, const double* model_pts_dev, int n_pts, const double* pred_ob_in_cam, const double* gt_ob_in_cam, int n_frames,
                           double* add_out, double* adds_out, void* stream);
/* VOCap (eval_ycbineoat.py): the area under the accuracy-threshold curve of n errors up to max_err (the reference's 0.1 m), divided by
 * max_err; the paper's tables print it x 100.  Host code, no GPU.  n = 0 or no error below max_err gives 0; NaN errors count in n but never
 * as below max_err.  BT_ERR_INVALID_ARG for n < 0, err NULL with n > 0, auc_out NULL or max_err not positive and finite. */
BT_API int bt_vocap(const double* err, int n, double max_err, double* auc_out);

/* ---- NOCS-REAL275 scoring: the reference's 6-PACK benchmark (scripts/benchmark.py) -----------------------------------------------------
 * bt_nocs_metrics: per record i, theta (degrees), shift and IoU as compute_RT_degree_cm_symmetry(pred, gt) and compute_3d_iou_new(gt, pred)
 * return them, in float64, with the benchmark's quirks kept (DESIGN.md §3.8): columns normalised over all four rows, a bottom row other
 * than [0,0,0,1] gives theta = shift = 10000, the rotation is divided by cbrt(det), arccos is not clipped (an argument beyond +-1 gives a
 * NaN theta), the "box" extents are taken per corner over x, y and z, and for a symmetric record theta uses the y axes and the IoU is the
 * maximum (from 0, NaN skipped) over 20 rotations of gt about its y axis.  The operation order is fixed, so results do not depend on n.
 *   pred / gt   HOST row-major 4 x 4 per record, translations in mm, as the benchmark compares them (before normalizeRotation).
 *   corners     HOST n x 8 x 3: the rows of model_scales/<model>.txt.
 *   symmetric   HOST n flags: the y-axis rule (bottle, bowl and can; the benchmark never applies it to mugs).
 *   theta_deg_out / shift_out / iou_out  DEVICE float64 [n].
 * Asynchronous on `stream`: the inputs are copied before the call returns, the results are ready when the stream is.  BT_ERR_INVALID_ARG
 * for n < 1, a NULL pointer, a non-finite input element, or a context without bt_nocs_reserve; BT_ERR_CAPACITY above max_records.
 * bt_nocs_reserve: room for max_records records per call, 456 B each on the device and in pinned host memory. */
BT_API int bt_nocs_reserve(bt_ctx* ctx, int max_records);
BT_API int bt_nocs_metrics(bt_ctx* ctx, const double* pred, const double* gt, const double* corners, const int32_t* symmetric, int n,
                           double* theta_deg_out, double* shift_out, double* iou_out, void* stream);
/* The benchmark's aggregation (benchmark.py main), host code, no GPU.  Records in the order given; cls[i] in 1..6 (bottle, bowl, camera, can,
 * laptop, mug); scored[i] = 0 for a record that is counted but not scored.  per_class_out[4 c + k] for class c + 1 and overall_out[k]:
 *   k = 0  5 deg 5 cm fraction: theta < 5 and shift < 50, over the class's record count
 *   k = 1  IoU25 fraction: IoU > 0.25, over the same count
 *   k = 2  mean theta over IoU > 0.25 and theta < 360 (NaN when empty)
 *   k = 3  mean shift over IoU > 0.25 (NaN when empty)
 * Means are numpy's (pairwise sum, then / count); overall is x += v / 6 in class order, so NaN class means reach it.  Fed the benchmark's
 * own per-record values, every number equals what it prints (x 100 for fractions, / 10 for the shift in cm).  BT_ERR_INVALID_ARG for
 * n < 1, a NULL pointer, a class outside 1..6 or a class without records. */
BT_API int bt_nocs_score(const int32_t* cls, const int32_t* scored, const double* theta_deg, const double* shift, const double* iou, int n,
                         double* per_class_out, double* overall_out);

/* ---- object model accuracy: a mesh against a reference mesh, in the frame both are given in (no alignment; DESIGN.md §3.15) ----------
 * bt_mesh_sample: n_samples points on the mesh, uniform by area and reproducible bit for bit (oracle/surface_oracle.py restates it):
 * per face w = |(B - A) x (C - A)| in float64, the integer weight q = floor(w / max w * 2^32), the exact 64-bit prefix sum of q as the CDF,
 * and sample k at CDF position ((k 2^32 + (h_3k >> 32)) * total) / (n_samples 2^32) in integer arithmetic, where h_i is splitmix64 output i
 * from state `seed`; its face is the first whose CDF exceeds the position (a face with q = 0, area 0 included, is never chosen).  The point is
 * ((1 - s) A + s (1 - u2) B) + s u2 C with s = sqrt(u1), u1, u2 = (h_3k+1 >> 11, h_3k+2 >> 11) * 2^-53, every operation rounded on its own.
 *   verts_dev     DEVICE float64 n_verts x 3.   faces_dev  DEVICE int32 n_faces x 3 (vertex indices).
 *   pts_out_dev   DEVICE float64 n_samples x 3, in CDF order (sample k lies on a face no later than sample k + 1's).
 * Synchronises `stream` once, to read back the face check and the CDF's total; the samples are then written on `stream`.  BT_ERR_INVALID_ARG,
 * with the output untouched, for a NULL pointer, sizes < 1, a face index outside [0, n_verts) or a non-finite vertex on a face (the message
 * names the lowest such face), a mesh whose weights are all 0, or a context without bt_surface_reserve; BT_ERR_CAPACITY for more faces or
 * samples than reserved.
 * bt_surface_distances: d_ab[i] = min_j |a_i - b_j| and d_ba[j] = min_i |b_j - a_i|, float64 and exact: the ADD-S scan (an fp32 filter with
 * a proven bound, then |a_i - b_j| = sqrt((dx dx + dy dy) + dz dz) in float64 for every candidate it keeps).
 *   a_dev / b_dev DEVICE float64 n_a x 3 / n_b x 3, finite.   d_ab_out / d_ba_out  DEVICE float64 [n_a] / [n_b].
 * Asynchronous on `stream`.  BT_ERR_INVALID_ARG for a NULL pointer, sizes < 1 or a context without bt_surface_reserve; BT_ERR_CAPACITY for
 * more than max_samples points on either side.
 * bt_surface_reserve: room for meshes of up to max_faces faces (1..2^27) and point sets of up to max_samples points (1..2^27): 16 B per face
 * and 32 B per sample on the device. */
BT_API int bt_surface_reserve(bt_ctx* ctx, int max_faces, int max_samples);
BT_API int bt_mesh_sample(bt_ctx* ctx, const double* verts_dev, int n_verts, const int32_t* faces_dev, int n_faces, int n_samples, uint64_t seed,
                          double* pts_out_dev, void* stream);
BT_API int bt_surface_distances(bt_ctx* ctx, const double* a_dev, int n_a, const double* b_dev, int n_b, double* d_ab_out, double* d_ba_out, void* stream);
/* The scores of the two directions' distances, host code, no GPU (d_ab: model -> reference, d_ba: reference -> model).  out[0..6]: accuracy
 * = mean d_ab, completeness = mean d_ba, chamfer = (accuracy + completeness) / 2, then the median and p95 of d_ab and of d_ba; then per
 * threshold t: out[7 + 3 t] precision = #{d_ab < tau} / n_a, out[8 + 3 t] recall = #{d_ba < tau} / n_b (strictly less), out[9 + 3 t]
 * F = 2 P R / (P + R), 0 when P + R = 0.  Means sum in index order; a quantile p is x[lo] + (pos - lo) (x[lo + 1] - x[lo]) at pos = p (n - 1)
 * of the sorted values, lo = floor(pos).  BT_ERR_INVALID_ARG for a NULL pointer (taus may be NULL when n_taus = 0), n_a or n_b < 1,
 * n_taus < 0, a distance that is negative or not finite, or a tau that is not positive and finite. */
BT_API int bt_surface_score(const double* d_ab, int n_a, const double* d_ba, int n_b, const double* taus, int n_taus, double* out);

/* ---- mask accuracy: the DAVIS region similarity J and boundary accuracy F per frame, and their per-sequence statistics (DESIGN.md §3.16) --
 * These restate the DAVIS toolkit's metrics (davis2017-evaluation metrics.py / utils.py); oracle/mask_oracle.py restates them in numpy.
 * P is the prediction and G the ground truth, H x W uint8 each, foreground = value != 0.
 *   J = |P & G| / |P | G| in float64, 1 when the union is 0.
 *   b(S), the boundary map (_seg2bmap): with e(y,x) = S(y,x+1), s(y,x) = S(y+1,x), se(y,x) = S(y+1,x+1), each 0 outside the image,
 *     b = (S ^ e) | (S ^ s) | (S ^ se) for y < H-1 and x < W-1;  b = S ^ e on the last row (x < W-1);  b = S ^ s on the last column
 *     (y < H-1);  b = 0 at the corner (H-1, W-1).  So a full-frame mask has no boundary, nor does foreground along the top or left edge.
 *   r = ceil(bound_th sqrt(H^2 + W^2)) in float64 (bound_th 0.008: r = 7 at 480 x 640, 8 at 480 x 854, 12 at 720 x 1280, 18 at 1080 x 1920);
 *     the disk is every offset with dx^2 + dy^2 <= r^2 (skimage disk(r) under cv2.dilate, nothing dilating in from outside the image).
 *   m_P = #{pixels of b(P) with a pixel of b(G) within the disk}, m_G the same with P and G swapped, n_P = |b(P)|, n_G = |b(G)|.
 *   precision, recall = (1, 0) when n_P = 0 < n_G;  (0, 1) when n_G = 0 < n_P;  (1, 1) when both are 0;  else m_P / n_P, m_G / n_G.
 *   F = 0 when precision + recall = 0, else 2 precision recall / (precision + recall), left to right in float64.
 * bt_mask_metrics: J and F of n_frames frame pairs.
 *   pred_dev / gt_dev  DEVICE uint8 [n_frames][h][w], contiguous, any alignment.  The kernel reads the whole 16-byte blocks that hold a pixel
 *                      of the arrays, so it may read up to 15 bytes before or after them (never across a 16-byte boundary).
 *   j_dev / f_dev      DEVICE float64 [n_frames].
 *   counts_dev         DEVICE int64 [n_frames][6] or NULL: |P & G|, |P | G|, n_P, n_G, m_P, m_G of each frame.
 * Asynchronous on `stream`, with no host synchronisation.  BT_ERR_INVALID_ARG for a NULL input or output, sizes < 1, bound_th outside
 * (0, 1), r > 64, or a context without a successful bt_mask_reserve; BT_ERR_CAPACITY above the reserved sizes.  A refused call writes nothing.
 * bt_mask_reserve: room for calls of up to max_frames frames of up to max_h x max_w.  One CTA holds a band of 64 rows of both masks plus
 * r rows above and r + 1 below as bit rows, 16 B per 64 pixels of a row; the reserve refuses (BT_ERR_INVALID_ARG) sizes whose band at r = 64
 * does not fit in the device's shared memory per block (on an H100, 227 KB: widths up to 4800, so 4K UHD, r = 36, fits).  24 B per frame
 * and 64-row band on the device. */
BT_API int bt_mask_reserve(bt_ctx* ctx, int max_frames, int max_h, int max_w);
BT_API int bt_mask_metrics(bt_ctx* ctx, const uint8_t* pred_dev, const uint8_t* gt_dev, int n_frames, int h, int w, double bound_th,
                           double* j_dev, double* f_dev, int64_t* counts_dev, void* stream);
/* Per-object mask accuracy of label maps with void pixels (DESIGN.md §3.17), DAVIS 2017's multi-object scoring: the toolkit's db_eval_iou and
 * f_measure with void_pixels.  pred and gt hold object ids per pixel (0 is background).  For object k in 1..n_objects of a frame pair:
 *   V = (gt == void_value), the void pixels (none when void_value is -1);
 *   P = (pred == k) & ~V and G = (gt == k) & ~V, so void is removed from both masks before the counts and before the boundary maps;
 *   then the six counts, J and F of P and G exactly as bt_mask_metrics defines them above.  An object in neither mask has an empty union
 *   and no boundary pixels, so J = 1 and F = 1.
 * bt_mask_metrics_objects: J and F of every object of n_frames frame pairs.
 *   pred_dev / gt_dev  DEVICE uint8 [n_frames][h][w] object ids, contiguous, any alignment; read as bt_mask_metrics reads its masks.
 *   n_objects          1 to 255; void_value -1, or 0 to 255 and not in 1..n_objects.
 *   j_dev / f_dev      DEVICE float64 [n_frames][n_objects], object k of frame i at i * n_objects + k - 1.
 *   counts_dev         DEVICE int64 [n_frames][n_objects][6] or NULL, the counts of bt_mask_metrics per object.
 * Each (frame, object) pair is one row of the reservation: n_frames * n_objects above bt_mask_reserve's max_frames is BT_ERR_CAPACITY.
 * Asynchronous on `stream`; the other refusals are bt_mask_metrics's, and a refused call writes nothing. */
BT_API int bt_mask_metrics_objects(bt_ctx* ctx, const uint8_t* pred_dev, const uint8_t* gt_dev, int n_frames, int h, int w, int n_objects,
                                   int void_value, double bound_th, double* j_dev, double* f_dev, int64_t* counts_dev, void* stream);
/* db_statistics of one sequence's per-frame J and F (host code, no GPU).  For X = J and then X = F: the mean, np.mean(X) (numpy's pairwise
 * sum); the recall, mean(X > 0.5), strictly greater; the decay, mean(bin 0) - mean(bin 3), bin i = X[ids[i] .. ids[i + 1]] inclusive, with
 * ids = round_half_even(linspace(1, n, 5) + 1e-10) - 1 and linspace's points i ((n - 1) / 4) + 1 for i < 4 and exactly n for i = 4.
 * out[7] = J&F = (J mean + F mean) / 2, J mean, J recall, J decay, F mean, F recall, F decay (the toolkit's CSV order).  The library scores
 * the frames it is given: the DAVIS semi-supervised protocol's leaving out of the first and last frames is the caller's.  BT_ERR_INVALID_ARG
 * for a NULL pointer or n < 1. */
BT_API int bt_mask_score(const double* j, const double* f, int n, double* out);

/* ---- tracking overlays: the reference's LOG frames (Bundler::saveNewframeResult, Bundler.cpp:379-411) ---------------------------------
 * bt_voxel_downsample: PCL's VoxelGrid (Utils::downsamplePointCloud, Utils.cpp:134-140; pcl::VoxelGrid::applyFilter with every field
 * averaged and no minimum count) of n_clouds clouds in one call, float32 (DESIGN.md §3.10): the voxel bounds from each cloud's finite
 * points, one centroid per occupied voxel in ascending voxel index, non-finite points skipped, and a cloud whose grid would exceed INT32_MAX
 * cells returned unchanged (non-finite points included).  Deliberate difference: the points of a voxel are summed in input order (PCL's
 * std::sort leaves that order open; DESIGN.md §4).  Results do not depend on how clouds are batched.
 *   pts_dev    HOST array of n_clouds DEVICE pointers, float32 n_pts[c] x 3 each.  n_pts: HOST, each >= 1.
 *   leaf       the voxel side (metres), positive and finite; the same for every cloud.
 *   out_dev    HOST array of n_clouds DEVICE pointers with room for n_pts[c] x 3 floats; n_out_dev: DEVICE int32 [n_clouds], the counts.
 * Asynchronous on `stream`: no host synchronisation; the counts stay on the device.  BT_ERR_INVALID_ARG for a NULL pointer, n_clouds < 1,
 * an empty cloud, a bad leaf or a context without bt_overlay_reserve; BT_ERR_CAPACITY for more than max_frames clouds or more than
 * max_pts x max_frames points in all. */
BT_API int bt_voxel_downsample(bt_ctx* ctx, int n_clouds, const float* const* pts_dev, const int* n_pts, float leaf, float* const* out_dev, int32_t* n_out_dev,
                               void* stream);
/* bt_pose_overlay: Bundler::saveNewframeResult's color_viz without the label, for n_frames frames in one call (Utils::drawProjectPoints,
 * Utils.cpp:216-226): the model moved by ob_in_cam = inverse(cur_in_model) (the float inverse bt_pose_format prints; each coordinate
 * ((m0 x + m1 y) + m2 z) + m3, every operation rounded), voxel-gridded at 0.01 as bt_voxel_downsample does, each centroid projected to
 * u = roundf(x fx / z + cx), v = roundf(y fy / z + cy) and, inside the image, stamped as cv::circle(r = 1, filled) in BGR (0, 255, 255): the
 * pixel and its four neighbours, clipped.  Under the stamps: the colour, each channel (uint8)(c * 0.2) where fg == 0.  raw: the colour with
 * fg == 0 pixels zeroed (the color_raw image, Frame::_color after invalidatePixelsByMask).
 *   model_dev   DEVICE float32 n_model x 3 (the model as the loader keeps it, voxel-gridded at 0.015).
 *   cur_in_model HOST row-major 4 x 4 cam->model per frame (the tracker's pose), n_frames back to back.
 *   colour_dev / fg_dev / viz_out_dev / raw_out_dev  HOST arrays of n_frames DEVICE pointers: uint8 H*W*3 BGR, H*W, H*W*3, H*W*3.  raw_out_dev
 *               may be NULL.
 * Asynchronous on `stream`.  BT_ERR_INVALID_ARG for a NULL pointer, sizes < 1, a singular pose or a context without bt_overlay_reserve;
 * BT_ERR_CAPACITY for more than max_frames frames or max_pts model points.
 * bt_overlay_reserve: scratch for max_frames clouds of max_pts points (max_pts x max_frames <= 2^30): 44 B per point on the device, about
 * 1 KB per 2048 points in pinned host memory. */
BT_API int bt_overlay_reserve(bt_ctx* ctx, int max_pts, int max_frames);
BT_API int bt_pose_overlay(bt_ctx* ctx, int n_frames, const float* model_dev, int n_model, const float* cur_in_model, float fx, float fy, float cx, float cy,
                           const uint8_t* const* colour_dev, const uint8_t* const* fg_dev, int H, int W, uint8_t* const* viz_out_dev,
                           uint8_t* const* raw_out_dev, void* stream);

/* ---- match images: the reference's LOG correspondence drawings (SiftManager::vizCorresBetween, FeatureManager.cpp:760-796) ----------
 * One image per desc, exactly as cv::drawMatches(NOT_DRAW_SINGLE_POINTS) of OpenCV 4.x draws it (DESIGN.md §3.11): the two ROI crops,
 * each resized by scale = min(900 / rows_a, 900 / rows_b) (integer division; 8-bit INTER_LINEAR, a copy at 1) and placed side by side on a
 * zero canvas of max(rows) x (cols_a + cols_b) pixels; then per match, in list order, a colour from cv::RNG, an anti-aliased circle of
 * radius 3 at the A keypoint clipped to the A half, one at the B keypoint clipped to the B half, and an anti-aliased line between them
 * (LINE_AA, 1/16-pixel coordinates).  Keypoints are ((u - umin) scale, (v - vmin) scale) in float32.
 *   colour_a / colour_b  DEVICE uint8 H x W x 3 BGR (the masked colour); roi_*: umin, umax, vmin, vmax, the crop is rows [vmin, vmax) and
 *               columns [umin, umax) and must lie inside the image, at most 900 rows tall.
 *   uv          DEVICE float4 (uA, vA, uB, vB) per match in full-image pixels, 16-byte aligned; may be NULL when n == 0.
 *   rng_state   cv::theRNG()'s state before the image (OpenCV's default is 0xffffffff).  A match draws three values, so the next image
 *               of a run starts from the state advanced by 3 n draws. */
typedef struct {
	const uint8_t* colour_a;
	int H_a, W_a;
	int32_t roi_a[4];
	const uint8_t* colour_b;
	int H_b, W_b;
	int32_t roi_b[4];
	const float* uv;
	int n;
	uint64_t rng_state;
} bt_match_viz_desc;
/* bt_match_viz_shape: the output rows and cols of the image of two ROIs (each at least 1 x 1 and at most 900 rows tall). */
BT_API int bt_match_viz_shape(const int32_t* roi_a, const int32_t* roi_b, int* rows, int* cols);
/* bt_match_viz_reserve: scratch for max_images images (1 to 65535) and max_matches matches over a call: 2052 B of device memory and 4 B
 * of pinned host memory per match (25 segment records of 80 B, 3 boxes, a colour), 112 B per image on each side. */
BT_API int bt_match_viz_reserve(bt_ctx* ctx, int max_images, int max_matches);
/* bt_match_viz: draws n_images images in one asynchronous call on `stream`; out_dev is a HOST array of n_images DEVICE pointers to
 * rows x cols x 3 uint8 (bt_match_viz_shape).  Results do not depend on how images are batched.  BT_ERR_INVALID_ARG for a NULL pointer,
 * a bad ROI, n < 0, more than 2^31 - 1 tiles of 32 x 32 output pixels in all, or a context without bt_match_viz_reserve;
 * BT_ERR_CAPACITY beyond the reserved images or matches. */
BT_API int bt_match_viz(bt_ctx* ctx, int n_images, const bt_match_viz_desc* desc, uint8_t* const* out_dev, void* stream);

/* ---- object model from a tracking run: a TSDF of depth maps in the model frame, and its zero surface (DESIGN.md §3.14) -----------------
 * bt_tsdf_fuse: fuses n_frames depth maps into a truncated signed distance field on a grid in the model frame, float32 with every operation
 * rounded on its own, so the grid is bit-reproducible (oracle/recon_oracle.py restates it):
 *   - the grid spans the axis-aligned box of every valid pixel (finite depth > 0) of every frame, back-projected and moved into the model frame,
 *     with m = ceil(trunc / voxel) + 1 samples of margin on every side: origin = lo - m voxel, n_a = ceil((hi_a - lo_a) / voxel) + 1 + 2 m,
 *     sample i at origin + i voxel;
 *   - per sample, frames in the order given: c = R^T (p - t); skipped when c_z <= 0, when the nearest pixel (floor(u + 0.5), floor(v + 0.5))
 *     is outside the image or has depth d <= 0 (masked-out pixels are 0 and never carve), or when sdf = d - c_z < -trunc; otherwise
 *     sum += min(1, sdf / trunc) and count += 1.
 *   depth_dev     HOST array of n_frames DEVICE pointers to float32 H*W depth (metres, 0 = none), e.g. bt_tracker_frame_depth's.
 *   cam_in_model  HOST row-major 4 x 4 cam->model per frame (bt_tracker_state's poses), n_frames back to back, finite.
 *   p             voxel (the sample spacing) and trunc, in metres, positive and finite.
 * Synchronises `stream` once, to read the bounds back (the grid's size decides what runs); the integration is then enqueued on `stream`.
 * BT_ERR_INVALID_ARG for a NULL pointer, n_frames < 1, sizes < 1, bad params or intrinsics, a non-finite pose element, no valid pixel in any
 * frame, or a context without bt_recon_reserve.  BT_ERR_CAPACITY for more frames or a larger image than reserved, or a grid of more than
 * max_voxels samples (the message names the dims and the bounds); both leave the previous grid as it was.
 * bt_tsdf_mesh: the zero surface of f = sum / count over the samples with count >= 1 (f < 0 inside), by marching tetrahedra: every cube split
 * into the six tets of its (0,0,0)-(1,1,1) diagonal, so the surface is closed wherever it is observed; a tet takes part when its four corners
 * are observed.  A vertex lies on one of the 7 edge directions {x, y, z, xy, xz, yz, xyz} of its edge's lower sample and is stored once, at
 * t = fa / (fa - fb) from that sample; vertices come in (sample, direction) order, faces in (cube, tet, triangle) order, wound so that their
 * normals point to f > 0 (free space).  Two calls on one grid give the same bytes.
 *   verts_dev     DEVICE float32 [max_vertices x 3]; faces_dev DEVICE int32 [max_faces x 3] (indices into verts).
 *   n_verts / n_faces  HOST: the counts, written also when they exceed the reserve.
 * Synchronises `stream` once, to read the counts back; the outputs are written on `stream` after it.  BT_ERR_INVALID_ARG for a NULL pointer
 * or before a successful bt_tsdf_fuse; BT_ERR_CAPACITY, with the outputs untouched, for more than max_vertices vertices or max_faces faces.
 * bt_tsdf_grid: the last fused grid (a parity aid): dims (3 ints), origin (3 floats), the bounds of the valid pixels (min x y z, max x y z)
 * and the DEVICE sum (float32) and count (int32) arrays, sample (i, j, k) at i + n_x (j + n_y k), valid until the next fuse or reserve on the
 * context.  Any output may be NULL.  BT_ERR_INVALID_ARG before a successful bt_tsdf_fuse.
 * bt_recon_reserve: room for max_frames frames (1..65535) of up to H x W per fuse and a grid of max_voxels samples (8..2^27): 24 B per sample
 * on the device.  max_vertices / max_faces bound a mesh call's outputs. */
typedef struct { float voxel, trunc; } bt_tsdf_params;
BT_API int bt_recon_reserve(bt_ctx* ctx, int max_frames, int H, int W, long long max_voxels, int max_vertices, int max_faces);
BT_API int bt_tsdf_fuse(bt_ctx* ctx, int n_frames, const float* const* depth_dev, const float* cam_in_model, float fx, float fy, float cx, float cy,
                        int H, int W, const bt_tsdf_params* p, void* stream);
BT_API int bt_tsdf_mesh(bt_ctx* ctx, float* verts_dev, int32_t* faces_dev, int* n_verts, int* n_faces, void* stream);
BT_API int bt_tsdf_grid(bt_ctx* ctx, int* dims, float* origin, float* bounds, const float** sum_dev, const int32_t** count_dev);

/* ---- LF-Net on the device: Lfnet::detectFeature's feature server (lf-net-release/run_server.py) without TensorFlow ----------------------
 * The network run_server.py builds at train_lfnet.py's defaults (DESIGN.md §3.12): mso_resnet_detector with use_nms3d, soft_scale and
 * soft_kpts, simple_desc on photo patches, l2-normalised descriptors, FP32 throughout.  bt_lfnet_params holds its numeric hyper-parameters;
 * the kernels take net_channel 16 and conv_ksize 5 only (the orientation conv uses conv_ksize as the reference's does).
 * bt_lfnet_weights_size: the float count of the weight blob for `p` (host code, no GPU).  Blob layout, float32, in this order (TF weight
 * layouts [kh][kw][cin][cout] and [in][out]; BN = (scale, shift) with scale = gamma / sqrt(moving_variance + 1e-5), shift = beta -
 * moving_mean scale, folded in float64 and rounded once; C = net_channel, k = conv_ksize):
 *   init_conv W[k][k][1][C] b[C]; per block: pre-bn scale[C] shift[C], conv1 W[k][k][C][C] b[C], mid-bn scale shift, conv2 W b;
 *   fin-bn scale[C] shift[C]; per scale i: score_conv_i W[k][k][C][1] b[1]; ori_conv W[k][k][C][2] b[2];
 *   per descriptor conv l: W[kd][kd][cin][cout] scale[cout] shift[cout] (shift also holds the conv bias times scale);
 *   fc1 W[F][512] scale[512] shift[512] (F = the flattened last conv output, HWC); fc2 W[512][desc_dim] b[desc_dim].
 * bt_lfnet_reserve: everything bt_lfnet_detect uses for up to max_images requests per call (about 46 MB per image for the maps plus
 * 122 KB per keypoint row at the defaults); a later call with other parameters drops the loaded weights.  BT_ERR_INVALID_ARG names a
 * parameter the kernels do not take.
 * bt_lfnet_load_weights: copies the blob (synchronously); refuses a size other than bt_lfnet_weights_size's and non-finite floats.
 * bt_lfnet_detect: n requests (HOST array of DEVICE pointers to 400 x 400 x 3 uint8, bt_lfnet_request's output) in one asynchronous call:
 *   kpts_out   DEVICE float [n][top_k][2]: (x, y) in the 400 x 400 input, the server's reply keypoints, row-major pixel order of the
 *              integer peaks (tf.where); rows past n_out[i] are zero.
 *   desc_out   DEVICE float [n][top_k][desc_dim]: the reply's descriptor rows (a bt_desc_view with pitch desc_dim * 4); rows past n_out[i]
 *              are zero.
 *   n_out      DEVICE int32 [n]: keypoints per request (top_k, or fewer when fewer NMS peaks are selected).
 * Results do not depend on how requests are batched.  BT_ERR_CAPACITY above max_images.
 * bt_lfnet_enable_timing / bt_lfnet_get_timing: device time of the last call per stage, ms5 = {trunk, score maps, detection, keypoints and
 * patches, descriptor}; get_timing waits for that call.
 * bt_lfnet_debug_maps (test aid): image `image` of the last call's max_heatmaps and max_scales (400 x 400 floats each), its integer
 * keypoints (top_k x (x, y) int32) and orientations (top_k x (cos, sin)), each output optional; synchronises `stream`.
 * Weights file (lfnet.write_weights_file, scripts/lfnet_export_blob.py), so a host without Python can load a network; byte order of the
 * host that wrote it (little-endian on x86-64 and aarch64), no padding:
 *   offset 0        char     magic[8] = "BTLFNETW"
 *   offset 8        uint32   format version = 1
 *   offset 12       uint32   sizeof(bt_lfnet_params) = P (104 on x86-64 and aarch64)
 *   offset 16       bt_lfnet_params, P bytes, as the struct is laid out in memory
 *   offset 16 + P   uint64   n_floats = bt_lfnet_weights_size of those parameters
 *   offset 24 + P   float32  the blob above, n_floats of them, and nothing after it.
 * bt_lfnet_file_info (host code, no GPU): checks the file and writes its parameters and float count (each output optional).
 *   BT_ERR_INVALID_ARG, naming what differs, for a file it cannot open, a bad magic, another format version or struct size, a truncated
 *   file or trailing bytes, parameters bt_lfnet_weights_size refuses and a float count other than its.
 * bt_lfnet_load_file: bt_lfnet_file_info's checks, then bt_lfnet_reserve(ctx, params, max_images) and bt_lfnet_load_weights with the
 *   file's blob; their refusals come through unchanged.  params_out (optional) receives the file's parameters. */
typedef struct {
	int top_k;                 /* run_server.py --top_k (500) */
	int net_channel, net_block, conv_ksize, net_num_scales;
	double net_min_scale, net_max_scale;
	float leaky_alpha;
	int sm_ksize;
	float com_strength, score_com_strength, scale_com_strength;
	int kp_loc_size;
	float kp_com_strength;
	int nms_ksize;
	float nms_thresh;
	int crop_radius, patch_size;
	int desc_net_channel, desc_net_depth, desc_conv_ksize, desc_dim;
} bt_lfnet_params;
BT_API int bt_lfnet_weights_size(const bt_lfnet_params* p, size_t* n_floats);
BT_API int bt_lfnet_reserve(bt_ctx* ctx, const bt_lfnet_params* params, int max_images);
BT_API int bt_lfnet_load_weights(bt_ctx* ctx, const float* blob, size_t n_floats);
BT_API int bt_lfnet_detect(bt_ctx* ctx, int n, const uint8_t* const* request_dev, float* kpts_out, float* desc_out, int32_t* n_out, void* stream);
BT_API int bt_lfnet_enable_timing(bt_ctx* ctx, int on);
BT_API int bt_lfnet_get_timing(bt_ctx* ctx, float* ms5);
BT_API int bt_lfnet_debug_maps(bt_ctx* ctx, int image, float* heat_host, float* scale_host, int32_t* kpts_int_host, float* ori_host, void* stream);
BT_API int bt_lfnet_file_info(const char* path, bt_lfnet_params* params_out, size_t* n_floats_out);
BT_API int bt_lfnet_load_file(bt_ctx* ctx, const char* path, int max_images, bt_lfnet_params* params_out);

/* ---- Object masks on the device: transductive-vos.pytorch's run_video.py (resnet50) without PyTorch ----------------------------------
 * The first frame's mask is propagated through the video (DESIGN.md §3.13): a ResNet-50 to stride 8 (layer3 and layer4 at stride 1,
 * layer4 with 256 planes) plus adjust_dim and bn256 gives 256 features per pixel of the (ceil(H / 8), ceil(W / 8)) grid; each frame's
 * labels are a softmax over the selected earlier frames' pixels, spatially weighted, times their labels.  FP32 results from 3xTF32
 * tensor-core products.  bt_vos_params holds run_video.py's --ref_num (5 to 64), --range (0 to 10000), --sigma1, --sigma2 (> 0) and
 * --temperature.
 * bt_vos_schedule (host code, no GPU): the history frames frame k >= 1 reads (lib/predict.py's sample_frames), n_out <= ref_num of them.
 * bt_vos_weights_size: the float count of the weight blob (the same for every params).  Blob layout, float32: per conv, in the network's
 * order, W[cout][ky][kx][cin] then BN scale[cout] and shift[cout] (scale = weight / sqrt(running_var + 1e-5), shift = bias - running_mean
 * scale, folded in float64 and rounded once).  The order: conv1 (3 -> 64, 7 x 7) with bn1; for each bottleneck of layer1..layer4 (3, 4,
 * 6, 3 blocks; planes 64, 128, 256, 256) conv1 (1 x 1) bn1, conv2 (3 x 3) bn2, conv3 (1 x 1) bn3, then, in the first block of layer1,
 * layer2 and layer3, downsample.0 with downsample.1; last adjust_dim (1024 -> 256, 1 x 1) with bn256.
 * bt_vos_reserve: the history ring of max(range + 5, ref_num + 1) frames of features (1 KB per low-resolution pixel) and labels, and the
 * network's scratch, for H x W frames (8 to 4096 each).  It ends any sequence begun.
 * bt_vos_load_weights: copies the blob (synchronously); refuses a size other than bt_vos_weights_size's and non-finite floats.
 * bt_vos_begin: frame 0.  colour_dev DEVICE H x W x 3 uint8 BGR (cv2.imread's order), init_mask_dev DEVICE H x W uint8 label values,
 *   mask_out_dev DEVICE H x W uint8 (the mask with > 0 -> 255).  The mask's distinct values become consecutive label channels, value 0
 *   being channel 0 even when absent; more than 8 channels is BT_ERR_INVALID_ARG, naming the count.  Reads the value set back, so it
 *   synchronises `stream`.
 * bt_vos_next: the next frame, asynchronous on `stream`: mask_out_dev DEVICE H x W uint8, 255 where the label is not channel 0.
 *   BT_ERR_INVALID_ARG before bt_vos_begin.  Both take frames of the reserved size.
 * bt_vos_labels: the label map of the last frame bt_vos_begin or bt_vos_next processed, asynchronous on `stream`: labels_out_dev DEVICE
 *   H x W uint8.  After bt_vos_next each pixel holds the initial mask's value of its label channel (the channel bt_vos_next's mask takes,
 *   the first of equal maxima of the bilinearly upsampled prediction), so a pixel is non-zero exactly where that mask is 255.  After
 *   bt_vos_begin it is the initial mask as given.  bt_vos_next overwrites the prediction this reads: call it before the next bt_vos_next
 *   in stream order.  BT_ERR_INVALID_ARG before bt_vos_begin.
 * bt_vos_enable_timing / bt_vos_get_timing: device time of the last call, ms3 = {backbone, propagation, mask}; get_timing waits for it.
 * bt_vos_debug (test aid): ring slot `slot`'s features (Hd x Wd x 256 floats) and label (Hd x Wd x 8 floats), the last bt_vos_next's
 *   low-resolution prediction (8 x Hd x Wd floats, channels past the label count zero) and info5 = {frame index, label channels, ring
 *   slots, Hd, Wd}; frame k lives in slot k mod ring slots.  Each output optional; synchronises `stream`. */
typedef struct {
	int ref_num, range;
	double sigma1, sigma2, temperature;
} bt_vos_params;
BT_API int bt_vos_schedule(int k, int ref_num, int range, int32_t* idx_out, int* n_out);
BT_API int bt_vos_weights_size(const bt_vos_params* p, size_t* n_floats);
BT_API int bt_vos_reserve(bt_ctx* ctx, const bt_vos_params* params, int H, int W);
BT_API int bt_vos_load_weights(bt_ctx* ctx, const float* blob, size_t n_floats);
BT_API int bt_vos_begin(bt_ctx* ctx, const uint8_t* colour_dev, const uint8_t* init_mask_dev, uint8_t* mask_out_dev, void* stream);
BT_API int bt_vos_next(bt_ctx* ctx, const uint8_t* colour_dev, uint8_t* mask_out_dev, void* stream);
BT_API int bt_vos_labels(bt_ctx* ctx, uint8_t* labels_out_dev, void* stream);
BT_API int bt_vos_enable_timing(bt_ctx* ctx, int on);
BT_API int bt_vos_get_timing(bt_ctx* ctx, float* ms3);
BT_API int bt_vos_debug(bt_ctx* ctx, int slot, float* feat_host, float* label_host, float* pred_host, int32_t* info5, void* stream);

/* Small device-memory helpers so non-CUDA hosts (ctypes, cgo, JNI) can drive the library without another runtime. */
BT_API int bt_dev_alloc(void** out, size_t bytes);
BT_API int bt_dev_free(void* p);
BT_API int bt_memcpy_h2d(void* dst_dev, const void* src_host, size_t bytes, void* stream);
BT_API int bt_memcpy_d2h(void* dst_host, const void* src_dev, size_t bytes, void* stream);
BT_API int bt_host_alloc_pinned(void** out, size_t bytes);
BT_API int bt_host_free_pinned(void* p);
BT_API int bt_stream_sync(void* stream);

/* Test aid: what the contexts and trackers of this process hold right now - device bytes, page-locked host bytes, and CUDA events plus
 * streams.  Destroying a context or tracker returns all three to their values from before it was created.  Memory from bt_dev_alloc /
 * bt_host_alloc_pinned is the caller's and is not counted. */
BT_API int bt_debug_live_resources(long long* device_bytes, long long* pinned_bytes, int* handles);
/* Test aid: the nth allocation of a device or page-locked block by the library from now (a reserve's, typically) fails with BT_ERR_CUDA
 * without calling CUDA, as an out-of-memory would; 0 disarms.  BT_ERR_INVALID_ARG for nth < 0. */
BT_API int bt_debug_fail_alloc(int nth);

#ifdef __cplusplus
}
#endif
#endif /* BUNDLETRACK_B200_H */
