// tracker.cu — the whole tracking step, Bundler::processNewFrame (the reference's src/Bundler.cpp:56-183), as one library object over the
// existing entry points, plus k_pose_init: SiftManager::procrustesByCorrespondence (FeatureManager.cpp:523-557) on the device.
//
// The tracker is host code: it calls bt_frames_preprocess_masked (or _u16), bt_lfnet_request, bt_desc_pool_store, bt_find_corres_pairs, bt_pose_init,
// bt_match_cache_*, bt_tracks_dev_forget_frame, bt_select_keyframes, bt_ba_gate, bt_frame_cache_store, bt_solve_windows and bt_keyframe_check
// in the reference's order.  Its own state is the frame deque, the keyframe list and which slot of its reserved buffers each frame holds.
// Synchronisations per frame: the ROI read-back in begin_frame; in end_frame the initial pose (with the neighbour pair's count and status),
// the window pairs' counts when any pair of the window was not matched before, and the poses of the solve when bundle adjustment runs.
// Compiled with -fmad=false: rigid_solve (rigid.cuh) must give the bits bt_rigid_transform gives on the host.
#include <algorithm>
#include <deque>
#include <map>
#include <vector>
#include "bt_common.cuh"
#include "rigid.cuh"

namespace bt {

constexpr int kPoseInitThreads = 256;
constexpr int kDescDim = 256;          // LF-Net descriptors
constexpr int kMaxKeyframes = 1024;    // bt_tracker_params::max_keyframes; with max_frames_alive <= 64 the map-point table's bt_tracks_dev_reserve_ex limit
struct PoseInitArgs { float A[16], B[16]; };

// pcl::transformPointWithNormal's point part, ((m0 x + m1 y) + m2 z) + m3 per coordinate, each operation rounded on its own
__device__ __forceinline__ void xform_point(const float* P, const float* p, float* o) {
#pragma unroll
	for (int r = 0; r < 3; r++)
		o[r] = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(P[r * 4], p[0]), __fmul_rn(P[r * 4 + 1], p[1])), __fmul_rn(P[r * 4 + 2], p[2])), P[r * 4 + 3]);
}

// One CTA.  The threads transform a chunk of entries into shared memory; thread 0 adds them to the sums in entry order (the host's serial order:
// a parallel reduction would round differently), once for the means and once more for S, then solves and composes offset * pose_A.
__global__ void __launch_bounds__(kPoseInitThreads) k_pose_init(const bt_entryj* __restrict__ entries, const int32_t* __restrict__ n_dev,
                                                               const int32_t* __restrict__ status_dev, PoseInitArgs a, float* __restrict__ pose_out) {
	__shared__ float s1[kPoseInitThreads][3], s2[kPoseInitThreads][3];
	const int n = *n_dev;
	const bool ok = *status_dev == BT_PAIR_OK && n >= 3;       // block-uniform
	RigidSums r;
	rigid_init(r);
	if (ok) {
		for (int pass = 0; pass < 2; pass++) {
			for (int base = 0; base < n; base += kPoseInitThreads) {
				const int i = base + threadIdx.x;
				if (i < n) {
					const bt_entryj e = entries[i];
					xform_point(a.A, e.pos_j, s1[threadIdx.x]);      // src: the newer frame's point in the model frame
					xform_point(a.B, e.pos_i, s2[threadIdx.x]);      // dst: the older frame's
				}
				__syncthreads();
				if (threadIdx.x == 0) {
					const int m = min(kPoseInitThreads, n - base);
					if (pass == 0) for (int k = 0; k < m; k++) rigid_add_means(r, s1[k], s2[k]);
					else for (int k = 0; k < m; k++) rigid_add_cov(r, s1[k], s2[k]);
				}
				__syncthreads();
			}
			if (pass == 0 && threadIdx.x == 0) rigid_means(r, n);
		}
	}
	if (threadIdx.x != 0) return;
	float O[16];
	if (ok) rigid_solve(r, O);
	else for (int i = 0; i < 16; i++) O[i] = (i % 5 == 0) ? 1.f : 0.f;
	for (int i = 0; i < 4; i++)
		for (int j = 0; j < 4; j++)
			pose_out[i * 4 + j] = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(O[i * 4], a.A[j]), __fmul_rn(O[i * 4 + 1], a.A[4 + j])), __fmul_rn(O[i * 4 + 2], a.A[8 + j])),
			                                __fmul_rn(O[i * 4 + 3], a.A[12 + j]));
}

}  // namespace bt

using namespace bt;

extern "C" int bt_pose_init(bt_ctx* ctx, const bt_entryj* entry_dev, const int32_t* n_entry_dev, const int32_t* status_dev, const float* pose_a,
                            const float* pose_b, float* pose_out_dev, void* stream) {
	BT_REQUIRE(ctx && entry_dev && n_entry_dev && status_dev && pose_a && pose_b && pose_out_dev, BT_ERR_INVALID_ARG, "bt_pose_init: NULL argument");
	BT_CUDA(cudaSetDevice(ctx->device));
	PoseInitArgs a;
	memcpy(a.A, pose_a, sizeof a.A);
	memcpy(a.B, pose_b, sizeof a.B);
	k_pose_init<<<1, kPoseInitThreads, 0, (cudaStream_t)stream>>>(entry_dev, n_entry_dev, status_dev, a, pose_out_dev);
	BT_CUDA(cudaGetLastError());
	return BT_OK;
}

// ------------------------------------------------------------------------------------------------ the tracker
namespace {
struct TFrame {
	int id = 0, slot = -1, cslot = -1;     // map / descriptor-pool slot, frame-cache slot (-1: none)
	int n_kpts = 0;
	bool keyframe = false;
	float pose[16];
};
struct TPair { const TFrame *a, *b; int wa, wb; };   // a findCorres pair (a newer) and the two frames' window indices
// device scratch in int32 units: the neighbour pair's initial pose and (count, offset, status), then the window call's counts
enum { M_POSE = 0, M_N = 16, M_OFF = 17, M_STATUS = 18, M_TOTAL = 20, M_WIN = 24 };
}  // namespace

struct bt_tracker {
	bt_ctx* ctx = nullptr;
	bt_tracker_params p;
	int n_slots = 0, max_pairs = 0, slot_entries = 0, win_entries = 0;
	size_t hw = 0;
	DevBuf depth, normal, fg, kpts, roi, entries, gather, meta;
	PinnedBuf h_meta;
	std::vector<int> free_slots, free_cslots;
	std::map<int, TFrame> alive;           // the deque's frames and the keyframes, by id
	std::deque<int> frames;                // Bundler::_frames (ids)
	std::vector<int> keyframes;            // Bundler::_keyframes (ids, admission order = id order)
	bool pending = false;
	TFrame pend;
	int last_fg_slot = -1;                 // the slot whose fg map the last begin_frame wrote (bt_tracker_last_fg)
};

static int tr_forget(bt_tracker* t, const TFrame& f, cudaStream_t stream) {
	BT_TRY(bt_match_cache_forget_frame(t->ctx, f.id));
	BT_TRY(bt_tracks_dev_forget_frame(t->ctx, f.id, stream));
	t->free_slots.push_back(f.slot);
	if (f.cslot >= 0) t->free_cslots.push_back(f.cslot);
	return BT_OK;
}
static float* tr_depth(bt_tracker* t, int slot) { return t->depth.as<float>() + t->hw * slot; }
static float* tr_normal(bt_tracker* t, int slot) { return t->normal.as<float>() + 4 * t->hw * slot; }
static uint8_t* tr_fg(bt_tracker* t, int slot) { return t->fg.as<uint8_t>() + t->hw * slot; }
static float* tr_kpts(bt_tracker* t, int slot) { return t->kpts.as<float>() + 2 * (size_t)t->p.max_feats * slot; }

static bt_match_frame tr_match_frame(bt_tracker* t, const TFrame& f, int window_index) {
	bt_match_frame m{};
	m.kpts_dev = tr_kpts(t, f.slot); m.n = f.n_kpts;
	m.depth_dev = tr_depth(t, f.slot); m.normal_dev = tr_normal(t, f.slot);
	memcpy(m.pose, f.pose, sizeof m.pose);
	m.frame_id = f.id; m.window_index = window_index;
	return m;
}
// the frame's quarter-resolution maps in the frame cache (CUDACache::storeFrame), once
static int tr_cache(bt_tracker* t, TFrame& f, cudaStream_t stream) {
	if (f.cslot >= 0) return BT_OK;
	BT_REQUIRE(!t->free_cslots.empty(), BT_ERR_CAPACITY, "bt_tracker: no frame-cache slot left");
	const int cs = t->free_cslots.back();
	const float* d[1] = { tr_depth(t, f.slot) };
	const float* n[1] = { tr_normal(t, f.slot) };
	const bt_tracker_params& p = t->p;
	BT_TRY(bt_frame_cache_store(t->ctx, 1, &cs, d, n, p.H, p.W, p.fx, p.fy, p.cx, p.cy, p.solver.depth_min, p.solver.depth_max, stream));
	t->free_cslots.pop_back();
	f.cslot = cs;
	return BT_OK;
}
static int tr_read(void* dst, const void* src, size_t bytes, cudaStream_t stream) {
	BT_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, stream));
	BT_CUDA(cudaStreamSynchronize(stream));
	return BT_OK;
}
// findCorres on an ordered pair list (A newer) in one asynchronous call: (count, offset, status) of the n pairs go to meta_dev[0, 3n)
static int tr_find_corres(bt_tracker* t, const std::vector<TPair>& prs, int32_t* meta_dev, cudaStream_t stream) {
	const int n = (int)prs.size();
	std::vector<bt_match_frame> A(n), B(n);
	std::vector<int32_t> sa(n), sb(n);
	int cap = n * t->p.max_feats;                         // room for every propagated match: never truncates
	for (int k = 0; k < n; k++) {
		A[k] = tr_match_frame(t, *prs[k].a, prs[k].wa); B[k] = tr_match_frame(t, *prs[k].b, prs[k].wb);
		sa[k] = prs[k].a->slot; sb[k] = prs[k].b->slot;
		cap += A[k].n + B[k].n;
	}
	const bt_tracker_params& p = t->p;
	return bt_find_corres_pairs(t->ctx, n, A.data(), B.data(), nullptr, nullptr, sa.data(), sb.data(), p.H, p.W, p.fx, p.fy, p.cx, p.cy, &p.prune, p.ransac_trials,
	                            p.ransac_inlier_dist, 0, t->entries.as<bt_entryj>(), cap, meta_dev, meta_dev + n, t->meta.as<int32_t>() + M_TOTAL, meta_dev + 2 * n,
	                            nullptr, stream);
}
// after the counts are read back: the table's overflow flag, then the _matches cache (SiftManager::_matches) for the same pairs
static int tr_put(bt_tracker* t, const std::vector<TPair>& prs, const int32_t* h, cudaStream_t stream) {
	const int n = (int)prs.size();
	int pts, obs;
	BT_TRY(bt_tracks_dev_stats(t->ctx, &pts, &obs, stream));     // (the stream is idle: reports a map-point table overflow)
	std::vector<int32_t> ia(n), ib(n);
	for (int k = 0; k < n; k++) { ia[k] = prs[k].a->id; ib[k] = prs[k].b->id; }
	return bt_match_cache_put(t->ctx, n, ia.data(), ib.data(), t->entries.as<bt_entryj>(), h, h + n, h + 2 * n, stream);
}
// the keyframes' poses, 16 floats each in admission order, for the policy calls (one row at least)
static std::vector<float> tr_keyframe_poses(const bt_tracker* t) {
	const int K = (int)t->keyframes.size();
	std::vector<float> kp(16 * (size_t)std::max(K, 1));
	for (int k = 0; k < K; k++) memcpy(&kp[16 * (size_t)k], t->alive.at(t->keyframes[k]).pose, 64);
	return kp;
}

// the tracker's own context and every buffer and table it uses; the caller destroys the tracker when one of them fails
static int tr_reserve(bt_tracker* t, int device, const bt_tracker_params* p) {
	BT_TRY(bt_ctx_create(&t->ctx, device));
	const int F = p->max_frames_alive + p->max_keyframes;    // frames with maps at once (max_keyframes = 0: max_frames_alive counts keyframes too)
	t->n_slots = F + 1;                                    // + the frame between begin_frame and end_frame
	t->max_pairs = p->max_BA_frames * (p->max_BA_frames - 1) / 2;
	t->slot_entries = 3 * p->max_feats;
	t->win_entries = t->max_pairs * t->slot_entries;
	t->hw = (size_t)p->H * p->W;
	const bt_solver_limits lim = { 1, p->max_BA_frames, t->win_entries, p->H, p->W, p->solver.image_downscale };
	BT_TRY(bt_solver_reserve(t->ctx, &lim));
	BT_TRY(bt_frame_cache_reserve(t->ctx, F, p->H, p->W, p->solver.image_downscale));
	BT_TRY(bt_pipeline_reserve(t->ctx, t->max_pairs, p->max_feats, kDescDim, p->ransac_trials));
	BT_TRY(bt_desc_pool_reserve(t->ctx, t->n_slots));
	BT_TRY(bt_tracks_dev_reserve_ex(t->ctx, F, p->max_feats, 16 * p->max_feats * ((F + 63) / 64)));
	// the keyframe pool's match-cache budget (the header states it): max_BA_frames / 2 worst-case blocks of 3 x max_feats entries per frame slot.
	// A frame's cached pairs are those of the windows it was new in, with at most max_BA_frames - 1 older frames each.
	BT_TRY(p->max_keyframes == 0 ? bt_match_cache_reserve(t->ctx, F * (F - 1) / 2, t->slot_entries)
	                             : bt_match_cache_reserve_entries(t->ctx, F * (F - 1) / 2, (long long)F * p->max_BA_frames * 3 * p->max_feats / 2));
	BT_TRY(t->depth.alloc(sizeof(float) * t->hw * t->n_slots));
	BT_TRY(t->normal.alloc(4 * sizeof(float) * t->hw * t->n_slots));
	BT_TRY(t->fg.alloc(t->hw * t->n_slots));
	BT_TRY(t->kpts.alloc(2 * sizeof(float) * (size_t)p->max_feats * t->n_slots));
	BT_TRY(t->roi.alloc(4 * sizeof(int32_t)));
	BT_TRY(t->entries.alloc(sizeof(bt_entryj) * (size_t)t->win_entries));
	BT_TRY(t->gather.alloc(sizeof(bt_entryj) * (size_t)t->win_entries));
	BT_TRY(t->meta.alloc(sizeof(int32_t) * (M_WIN + 3 * (size_t)t->max_pairs)));
	BT_TRY(t->h_meta.alloc(sizeof(int32_t) * (M_WIN + 3 * (size_t)t->max_pairs)));
	for (int s = t->n_slots - 1; s >= 0; s--) t->free_slots.push_back(s);
	for (int s = F - 1; s >= 0; s--) t->free_cslots.push_back(s);
	return BT_OK;
}

extern "C" int bt_tracker_create(bt_tracker** out, int device, const bt_tracker_params* p) {
	BT_REQUIRE(out && p, BT_ERR_INVALID_ARG, "bt_tracker_create: NULL argument");
	*out = nullptr;
	BT_REQUIRE(p->H > 0 && p->W > 0 && p->max_feats > 0 && p->max_feats <= 8192 && p->max_frames_alive >= 2 && p->max_frames_alive <= 64, BT_ERR_INVALID_ARG,
	           "bt_tracker_create: bad sizes (max_feats 1..8192, max_frames_alive 2..64)");
	BT_REQUIRE(p->max_keyframes >= 0 && p->max_keyframes <= kMaxKeyframes, BT_ERR_INVALID_ARG, "bt_tracker_create: max_keyframes 0..%d", kMaxKeyframes);
	BT_REQUIRE(p->max_BA_frames >= 2 && p->max_BA_frames <= 32 && p->window_size >= 0 && p->ransac_trials >= 1 &&
	           (p->mask_mode == BT_MASK_AS_IS || p->mask_mode == BT_MASK_LARGEST_HULL), BT_ERR_INVALID_ARG,
	           "bt_tracker_create: bad parameters (max_BA_frames 2..32, window_size >= 0, ransac_trials >= 1, mask_mode)");
	bt_tracker* t = new bt_tracker();
	t->p = *p;
	const int rc = tr_reserve(t, device, p);
	if (rc == BT_OK) *out = t;
	else bt_tracker_destroy(t);
	return rc;
}

extern "C" void bt_tracker_destroy(bt_tracker* t) {
	if (!t) return;
	bt_ctx* ctx = t->ctx;
	if (ctx) cudaSetDevice(ctx->device);
	delete t;
	bt_ctx_destroy(ctx);
}

// both begin_frame entry points: depth_raw_dev is float metres, or uint16 millimetres when u16
static int tr_begin(bt_tracker* t, const char* who, int loader_id, const float* first_pose, const void* depth_raw_dev, bool u16, const uint8_t* mask_dev,
                    const uint8_t* colour_dev, uint8_t* request_out_dev, int32_t* roi_out, int* id_out, float* pose_out, int* status_out, void* stream_) {
	BT_REQUIRE(t && depth_raw_dev && mask_dev && colour_dev && request_out_dev && status_out, BT_ERR_INVALID_ARG, "%s: NULL argument", who);
	BT_REQUIRE(!t->pending, BT_ERR_INVALID_ARG, "%s: frame %d is pending: finish it with end_frame or drop_frame first", who, t->pend.id);
	cudaStream_t stream = (cudaStream_t)stream_;
	BT_CUDA(cudaSetDevice(t->ctx->device));
	const bt_tracker_params& p = t->p;
	TFrame f;
	if (!t->frames.empty()) {                              // Bundler.cpp:74-81
		const TFrame& last = t->alive.at(t->frames.back());
		f.id = last.id + 1;
		memcpy(f.pose, last.pose, sizeof f.pose);
	} else {
		f.id = loader_id;
		for (int i = 0; i < 16; i++) f.pose[i] = first_pose ? first_pose[i] : ((i % 5 == 0) ? 1.f : 0.f);
	}
	if (id_out) *id_out = f.id;
	if (pose_out) memcpy(pose_out, f.pose, sizeof f.pose);
	f.slot = t->free_slots.back();                         // (one slot more than frames alive: never empty here)
	const uint8_t* msk[1] = { mask_dev };
	float* dout[1] = { tr_depth(t, f.slot) };
	float* nout[1] = { tr_normal(t, f.slot) };
	uint8_t* fg[1] = { tr_fg(t, f.slot) };
	const uint16_t* din_mm[1] = { static_cast<const uint16_t*>(depth_raw_dev) };
	const float* din[1] = { static_cast<const float*>(depth_raw_dev) };
	BT_TRY(u16 ? bt_frames_preprocess_masked_u16(t->ctx, 1, din_mm, msk, p.mask_mode, p.H, p.W, p.fx, p.fy, p.cx, p.cy, &p.depth, dout, nullptr, nout, fg, t->roi.as<int32_t>(), stream)
	           : bt_frames_preprocess_masked(t->ctx, 1, din, msk, p.mask_mode, p.H, p.W, p.fx, p.fy, p.cx, p.cy, &p.depth, dout, nullptr, nout, fg, t->roi.as<int32_t>(), stream));
	t->last_fg_slot = f.slot;
	int32_t* roi = t->h_meta.as<int32_t>();
	BT_TRY(tr_read(roi, t->roi.p, 4 * sizeof(int32_t), stream));
	if (roi_out) memcpy(roi_out, roi, 4 * sizeof(int32_t));
	if (roi[1] - roi[0] < 10 || roi[3] - roi[2] < 10) {   // Bundler.cpp:88-93: FAIL, nothing is kept or forgotten
		*status_out = BT_FRAME_FAIL;
		return BT_OK;
	}
	const uint8_t* col[1] = { colour_dev };
	const uint8_t* fgc[1] = { fg[0] };
	uint8_t* req[1] = { request_out_dev };
	BT_TRY(bt_lfnet_request(t->ctx, 1, col, fgc, t->roi.as<int32_t>(), p.H, p.W, req, stream));
	t->free_slots.pop_back();
	t->pend = f;
	t->pending = true;
	*status_out = BT_FRAME_OTHER;
	return BT_OK;
}

extern "C" int bt_tracker_begin_frame(bt_tracker* t, int loader_id, const float* first_pose, const float* depth_raw_dev, const uint8_t* mask_dev,
                                      const uint8_t* colour_dev, uint8_t* request_out_dev, int32_t* roi_out, int* status_out, void* stream) {
	return tr_begin(t, "bt_tracker_begin_frame", loader_id, first_pose, depth_raw_dev, false, mask_dev, colour_dev, request_out_dev, roi_out, nullptr, nullptr,
	                status_out, stream);
}

extern "C" int bt_tracker_begin_frame_u16(bt_tracker* t, int loader_id, const float* first_pose, const uint16_t* depth_mm_dev, const uint8_t* mask_dev,
                                          const uint8_t* colour_dev, uint8_t* request_out_dev, int32_t* roi_out, int* id_out, float* pose_out, int* status_out,
                                          void* stream) {
	return tr_begin(t, "bt_tracker_begin_frame_u16", loader_id, first_pose, depth_mm_dev, true, mask_dev, colour_dev, request_out_dev, roi_out, id_out, pose_out,
	                status_out, stream);
}

extern "C" int bt_tracker_drop_frame(bt_tracker* t, float* pose_out) {
	BT_REQUIRE(t, BT_ERR_INVALID_ARG, "bt_tracker_drop_frame: NULL tracker");
	BT_REQUIRE(t->pending, BT_ERR_INVALID_ARG, "bt_tracker_drop_frame: no frame is pending");
	BT_CUDA(cudaSetDevice(t->ctx->device));
	BT_TRY(tr_forget(t, t->pend, nullptr));
	t->pending = false;
	if (pose_out) memcpy(pose_out, t->pend.pose, sizeof t->pend.pose);
	return BT_OK;
}

// Bundler.cpp:119-138: findCorres on (new, last), the initial pose from its inliers, the pair into the match cache; a FAIL pair fails the frame
static int tr_neighbour(bt_tracker* t, TFrame& f, int* status, cudaStream_t stream) {
	if (t->frames.empty()) return BT_OK;
	int32_t* md = t->meta.as<int32_t>();
	int32_t* mh = t->h_meta.as<int32_t>();
	const TFrame& last = t->alive.at(t->frames.back());
	const std::vector<TPair> prs = { { &f, &last, 1, 0 } };
	BT_TRY(tr_find_corres(t, prs, md + M_N, stream));
	BT_TRY(bt_pose_init(t->ctx, t->entries.as<bt_entryj>(), md + M_N, md + M_STATUS, f.pose, last.pose, reinterpret_cast<float*>(md + M_POSE), stream));
	BT_TRY(tr_read(mh, md, sizeof(int32_t) * (M_STATUS + 1), stream));     // the pose, count, offset and status
	BT_TRY(tr_put(t, prs, mh + M_N, stream));
	if (mh[M_STATUS] == BT_PAIR_FAIL) *status = BT_FRAME_FAIL;
	else memcpy(f.pose, mh + M_POSE, sizeof f.pose);
	return BT_OK;
}
// Bundler.cpp:149-157: the oldest frame leaves a full deque (a keyframe stays alive), the new one joins
static int tr_slide(bt_tracker* t, const TFrame& f, cudaStream_t stream) {
	if ((int)t->frames.size() >= t->p.window_size + 3) {
		const TFrame& o = t->alive.at(t->frames.front());
		if (!o.keyframe) {
			BT_TRY(tr_forget(t, o, stream));
			t->alive.erase(t->frames.front());
		}
		t->frames.pop_front();
	}
	t->frames.push_back(f.id);
	t->alive[f.id] = f;
	return BT_OK;
}
// selectKeyFramesForBA + optimizeGPU (Bundler.cpp:222-358): the uncached pairs matched, all gathered, the BA gate, the solve
static int tr_window(bt_tracker* t, TFrame& nf, int* status, cudaStream_t stream) {
	const bt_tracker_params& p = t->p;
	const int K = (int)t->keyframes.size();
	std::vector<int32_t> chosen(std::max(K, 1));
	int n_chosen = 0;
	BT_TRY(bt_select_keyframes(nf.pose, tr_keyframe_poses(t).data(), K, p.max_BA_frames, chosen.data(), &n_chosen));
	std::vector<TFrame*> win;
	for (int k = 0; k < n_chosen; k++) win.push_back(&t->alive.at(t->keyframes[chosen[k]]));
	win.push_back(&nf);                                    // the newest frame sorts last
	const int N = (int)win.size();
	std::vector<TPair> todo;
	std::vector<int32_t> ga, gb;
	std::vector<uint32_t> wi, wj;
	for (int i = 0; i < N; i++)
		for (int j = i + 1; j < N; j++) {
			ga.push_back(win[j]->id); gb.push_back(win[i]->id); wi.push_back(i); wj.push_back(j);
			if (!bt_match_cache_has(t->ctx, win[j]->id, win[i]->id)) todo.push_back({ win[j], win[i], j, i });
		}
	if (!todo.empty()) {
		const int n = (int)todo.size();
		int32_t* md = t->meta.as<int32_t>() + M_WIN;
		int32_t* mh = t->h_meta.as<int32_t>() + M_WIN;
		BT_TRY(tr_find_corres(t, todo, md, stream));
		BT_TRY(tr_read(mh, md, sizeof(int32_t) * 3 * n, stream));
		BT_TRY(tr_put(t, todo, mh, stream));
		for (int k = 0; k < n; k++)
			if (mh[2 * n + k] == BT_PAIR_FAIL && todo[k].a == &nf) *status = BT_FRAME_FAIL;
	}
	int n_edges = 0;
	const int np = (int)ga.size();
	std::vector<int32_t> boff(std::max(np, 1)), bn(std::max(np, 1));
	if (np > 0) BT_TRY(bt_match_cache_gather(t->ctx, np, ga.data(), gb.data(), wi.data(), wj.data(), t->gather.as<bt_entryj>(), t->win_entries, boff.data(), bn.data(), stream));
	for (int k = 0; k < np; k++) if ((int)wj[k] == N - 1) n_edges += bn[k];
	if (*status != BT_FRAME_FAIL && !bt_ba_gate(n_edges, p.min_fm_edges_newframe)) *status = BT_FRAME_NO_BA;
	if (*status != BT_FRAME_OTHER || N < 2) return BT_OK;
	BT_TRY(tr_cache(t, nf, stream));
	std::vector<const float*> dptr(N), nptr(N);
	std::vector<int32_t> cs(N);
	std::vector<float> poses(16 * (size_t)N);
	for (int k = 0; k < N; k++) {
		dptr[k] = tr_depth(t, win[k]->slot); nptr[k] = tr_normal(t, win[k]->slot); cs[k] = win[k]->cslot;
		memcpy(&poses[16 * (size_t)k], win[k]->pose, 64);
	}
	bt_window w{};
	w.n_frames = N; w.H = p.H; w.W = p.W;
	w.depth_dev = dptr.data(); w.normal_dev = nptr.data();
	w.fx = p.fx; w.fy = p.fy; w.cx = p.cx; w.cy = p.cy;
	w.compat_flip = 1;
	w.cache_slots = cs.data();
	w.corr_dev = t->gather.as<bt_entryj>();
	w.n_blocks = np; w.block_off = boff.data(); w.block_n = bn.data(); w.block_i = wi.data(); w.block_j = wj.data();
	BT_TRY(bt_solve_windows(t->ctx, 1, &w, &p.solver, poses.data(), stream));
	for (int k = 0; k < N; k++) memcpy(win[k]->pose, &poses[16 * (size_t)k], 64);     // every frame of the window, keyframes included
	return BT_OK;
}
// a FAIL frame is forgotten, and popped when the deque holds it (Bundler.cpp:173-179); the reported pose is the one the frame has
static int tr_fail(bt_tracker* t, TFrame f, bool in_deque, float* pose_out, int* status_out, cudaStream_t stream) {
	BT_TRY(tr_forget(t, f, stream));
	if (in_deque) { t->frames.pop_back(); t->alive.erase(f.id); }
	memcpy(pose_out, f.pose, sizeof f.pose);
	*status_out = BT_FRAME_FAIL;
	return BT_OK;
}
// closing the frame (Bundler.cpp:173-221): FAIL, or checkAndAddKeyframe
static int tr_close(bt_tracker* t, TFrame& nf, int status, float* pose_out, int* status_out, cudaStream_t stream) {
	if (status == BT_FRAME_FAIL) return tr_fail(t, nf, true, pose_out, status_out, stream);
	if (status == BT_FRAME_OTHER && bt_keyframe_check(nf.pose, nf.id, nf.n_kpts, tr_keyframe_poses(t).data(), (int)t->keyframes.size(), t->p.min_feat_num,
	                                                  t->p.min_rot_deg) == 1) {
		BT_TRY(tr_cache(t, nf, stream));
		nf.keyframe = true;
		t->keyframes.push_back(nf.id);
	} else if (nf.cslot >= 0) {                            // only keyframes take part in later windows
		t->free_cslots.push_back(nf.cslot);
		nf.cslot = -1;
	}
	memcpy(pose_out, nf.pose, sizeof nf.pose);
	*status_out = status;
	return BT_OK;
}

extern "C" int bt_tracker_end_frame(bt_tracker* t, const float* kpts_host, int n_kpts, const bt_desc_view* desc, float* pose_out, int* status_out, void* stream_) {
	BT_REQUIRE(t && desc && pose_out && status_out, BT_ERR_INVALID_ARG, "bt_tracker_end_frame: NULL argument");
	BT_REQUIRE(t->pending, BT_ERR_INVALID_ARG, "bt_tracker_end_frame: no frame is pending (begin_frame first; a frame that failed the ROI gate is done)");
	const bt_tracker_params& p = t->p;
	BT_REQUIRE(n_kpts >= 0 && n_kpts <= p.max_feats, BT_ERR_INVALID_ARG, "bt_tracker_end_frame: %d keypoints, the tracker was created for %d", n_kpts, p.max_feats);
	BT_REQUIRE((n_kpts == 0 || (kpts_host && desc->dev)) && desc->n == n_kpts && desc->dim == kDescDim, BT_ERR_INVALID_ARG,
	           "bt_tracker_end_frame: the descriptor view must hold n_kpts rows of %d floats", kDescDim);
	if (p.max_keyframes == 0) {
		BT_REQUIRE((int)t->alive.size() + 1 <= p.max_frames_alive, BT_ERR_CAPACITY, "bt_tracker_end_frame: %d frames alive + the new one > max_frames_alive %d",
		           (int)t->alive.size(), p.max_frames_alive);
	} else {                                               // the new frame may become a keyframe: the pool must have room for it
		const int n_kf = (int)t->keyframes.size(), n_other = (int)t->alive.size() - n_kf;
		BT_REQUIRE(n_other + 1 <= p.max_frames_alive, BT_ERR_CAPACITY, "bt_tracker_end_frame: %d frames alive that are not keyframes + the new one > max_frames_alive %d",
		           n_other, p.max_frames_alive);
		BT_REQUIRE(n_kf < p.max_keyframes, BT_ERR_CAPACITY, "bt_tracker_end_frame: the keyframe pool is full (%d keyframes)", n_kf);
	}
	cudaStream_t stream = (cudaStream_t)stream_;
	BT_CUDA(cudaSetDevice(t->ctx->device));
	TFrame f = t->pend;
	f.n_kpts = n_kpts;
	if (n_kpts) BT_CUDA(cudaMemcpyAsync(tr_kpts(t, f.slot), kpts_host, 2 * sizeof(float) * (size_t)n_kpts, cudaMemcpyHostToDevice, stream));
	BT_TRY(bt_desc_pool_store(t->ctx, f.slot, desc, stream));
	t->pending = false;                                    // from here on the frame is the tracker's
	int status = BT_FRAME_OTHER;
	BT_TRY(tr_neighbour(t, f, &status, stream));
	if (status == BT_FRAME_FAIL) return tr_fail(t, f, false, pose_out, status_out, stream);
	BT_TRY(tr_slide(t, f, stream));
	TFrame& nf = t->alive.at(f.id);
	if (nf.id != 0) BT_TRY(tr_window(t, nf, &status, stream));
	return tr_close(t, nf, status, pose_out, status_out, stream);
}

extern "C" int bt_tracker_state(bt_tracker* t, int32_t* ids, float* poses, int32_t* is_keyframe, int cap, int* n) {
	BT_REQUIRE(t && n && cap >= 0, BT_ERR_INVALID_ARG, "bt_tracker_state: NULL argument");
	*n = (int)t->alive.size();
	BT_REQUIRE(*n <= cap, BT_ERR_CAPACITY, "bt_tracker_state: %d frames alive > cap %d", *n, cap);
	int k = 0;
	for (const auto& kv : t->alive) {
		if (ids) ids[k] = kv.first;
		if (poses) memcpy(poses + 16 * (size_t)k, kv.second.pose, 64);
		if (is_keyframe) is_keyframe[k] = kv.second.keyframe ? 1 : 0;
		k++;
	}
	return BT_OK;
}

// Frame::_fg_mask of the frame the last begin_frame segmented.  Its slot is taken again only by a later begin_frame: a frame that failed the
// ROI gate never took it, a dropped or failed frame gave it back, a tracked frame keeps it until a later step forgets the frame.
extern "C" int bt_tracker_last_fg(bt_tracker* t, const uint8_t** fg_dev) {
	BT_REQUIRE(t && fg_dev, BT_ERR_INVALID_ARG, "bt_tracker_last_fg: NULL argument");
	BT_REQUIRE(t->last_fg_slot >= 0, BT_ERR_INVALID_ARG, "bt_tracker_last_fg: no frame has been segmented yet");
	*fg_dev = tr_fg(t, t->last_fg_slot);
	return BT_OK;
}

extern "C" int bt_tracker_frame_depth(bt_tracker* t, int frame_id, const float** depth_dev) {
	BT_REQUIRE(t && depth_dev, BT_ERR_INVALID_ARG, "bt_tracker_frame_depth: NULL argument");
	const auto it = t->alive.find(frame_id);
	BT_REQUIRE(it != t->alive.end(), BT_ERR_INVALID_ARG, "bt_tracker_frame_depth: frame %d is not alive", frame_id);
	*depth_dev = tr_depth(t, it->second.slot);
	return BT_OK;
}

extern "C" int bt_tracker_usage(bt_tracker* t, int* n_points, int* n_pairs_cached, long long* n_entries_cached, void* stream) {
	BT_REQUIRE(t && n_points && n_pairs_cached && n_entries_cached, BT_ERR_INVALID_ARG, "bt_tracker_usage: NULL argument");
	BT_CUDA(cudaSetDevice(t->ctx->device));
	BT_TRY(tracks_points_alive(t->ctx, (cudaStream_t)stream, n_points));
	return bt_match_cache_usage(t->ctx, n_pairs_cached, n_entries_cached);
}
