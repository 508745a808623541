// bt_common.cuh — shared declarations for the sm_90a hot-path library (no torch, no third-party headers).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <vector>
#include "../../include/bundletrack_b200.h"

namespace bt {

void set_error(const char* fmt, ...);

#define BT_CUDA(x)                                                                                   \
	do {                                                                                             \
		cudaError_t e_ = (x);                                                                        \
		if (e_ != cudaSuccess) {                                                                     \
			bt::set_error("%s:%d %s -> %s", __FILE__, __LINE__, #x, cudaGetErrorString(e_));         \
			return BT_ERR_CUDA;                                                                      \
		}                                                                                            \
	} while (0)

#define BT_REQUIRE(cond, code, ...)                                                                  \
	do {                                                                                             \
		if (!(cond)) { bt::set_error(__VA_ARGS__); return (code); }                                  \
	} while (0)

// A growable device buffer owned by the context (allocation happens in *_reserve, never on the per-call path
// unless a call exceeds what was reserved, in which case the call fails with BT_ERR_CAPACITY).
struct DevBuf {
	void* p = nullptr;
	size_t bytes = 0;
	int alloc(size_t n) {
		if (n <= bytes) return BT_OK;
		if (p) cudaFree(p);
		p = nullptr; bytes = 0;
		BT_CUDA(cudaMalloc(&p, n));
		bytes = n;
		return BT_OK;
	}
	void release() { if (p) cudaFree(p); p = nullptr; bytes = 0; }
	template <class T> T* as() const { return reinterpret_cast<T*>(p); }
};
struct PinnedBuf {
	void* p = nullptr;
	size_t bytes = 0;
	int alloc(size_t n) {
		if (n <= bytes) return BT_OK;
		if (p) cudaFreeHost(p);
		p = nullptr; bytes = 0;
		BT_CUDA(cudaMallocHost(&p, n));
		bytes = n;
		return BT_OK;
	}
	void release() { if (p) cudaFreeHost(p); p = nullptr; bytes = 0; }
	template <class T> T* as() const { return reinterpret_cast<T*>(p); }
};

struct SolverState;   // solver.cu
struct MatcherState;  // knn.cu
struct RansacState;   // ransac.cu
struct FrontState;    // frontend.cu
struct PruneState;    // prune.cu
struct MatchCache;    // prune.cu
struct TracksDev;     // tracks_dev.cu
struct MetricsState;  // metrics.cu

}  // namespace bt

struct bt_ctx {
	int device = 0;
	int sm_count = 0;
	int cc_major = 0, cc_minor = 0;
	bt::SolverState* solver = nullptr;
	bt::MatcherState* matcher = nullptr;
	bt::RansacState* ransac = nullptr;
	bt::FrontState* front = nullptr;
	bt::PruneState* prune = nullptr;
	bt::MatchCache* mcache = nullptr;
	bt::TracksDev* tracks = nullptr;
	bt::MetricsState* metrics = nullptr;
};

namespace bt {
void solver_destroy(bt_ctx* ctx);
void matcher_destroy(bt_ctx* ctx);
void ransac_destroy(bt_ctx* ctx);
void prune_destroy(bt_ctx* ctx);
void mcache_destroy(bt_ctx* ctx);
void front_destroy(bt_ctx* ctx);
void metrics_destroy(bt_ctx* ctx);
// segment.cu: largest-hull mode for the masked front end, and the LF-Net request
size_t hull_fill_smem(int H);
int segment_largest_hull(const uint8_t* const* mask_tbl_dev, int n, int H, int W, int32_t* label, int32_t* count, unsigned long long* best,
                         uint8_t* fill, cudaStream_t stream);
int launch_lfnet_request(const void* const* tbl_dev, const int32_t* roi_dev, int n, int H, int W, cudaStream_t stream);
// tracks_dev.cu: the device map-point table, driven pair by pair from bt_find_corres_pairs (prune.cu).  Frames are named by slot;
// tracks_slot maps a frame id to its slot (-1: the frame has no map yet, unless create is set).
void tracks_dev_destroy(bt_ctx* ctx);
int tracks_slot(bt_ctx* ctx, int frame_id, bool create, int* slot);
int tracks_free_slots(bt_ctx* ctx);
// map points alive now (created and not freed by forgets); synchronises `stream`
int tracks_points_alive(bt_ctx* ctx, cudaStream_t stream, int* n);
// where an update takes its (uA, vA, uB, vB) list from: entry i = base + stride * (ids ? ids[i] : i) floats.  The count is *n_dev, or, when
// n_inl is set, pair `pair`'s emitted count (n_inl[pair] < 5 -> 0, clamped to `capacity` behind the earlier pairs) as k_emit_entryj writes it.
struct TrkSrc { const float* base; int stride; const int32_t* ids; const int32_t* n_dev; int max_n; const int32_t* n_inl; int pair; int capacity; };
int tracks_launch_update(bt_ctx* ctx, int slot_a, int slot_b, const TrkSrc& src, cudaStream_t stream);
int tracks_launch_propagate(bt_ctx* ctx, int slot_a, int slot_b, const float4* existing, int n_existing, float4* out, int capacity, int32_t* n_out,
                            cudaStream_t stream);
}
