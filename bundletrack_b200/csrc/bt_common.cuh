// bt_common.cuh — shared declarations for the sm_90a hot-path library (no torch, no third-party headers).
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <atomic>
#include <memory>
#include <utility>
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

#define BT_TRY(x)                                                                                    \
	do {                                                                                             \
		const int rc_ = (x);                                                                         \
		if (rc_ != BT_OK) return rc_;                                                                \
	} while (0)

// Largest float d2max with `sqrtf(d2) <= th` <=> `d2 <= d2max` for every float d2 (sqrtf is correctly rounded and monotonic), so a
// kernel can compare squared distances.  -1 when no d2 qualifies (th < 0 or NaN); +inf for th = +inf.
inline float sqrt_le_max(float th) {
	if (!(th > 0.f)) return (th == 0.f) ? 0.f : -1.f;
	auto nextf = [](float v, int d) { int32_t b; memcpy(&b, &v, 4); b += d; float r; memcpy(&r, &b, 4); return r; };
	float d2max = th * th;
	while (d2max > 0.f && sqrtf(d2max) > th) d2max = nextf(d2max, -1);
	while (sqrtf(nextf(d2max, 1)) <= th) d2max = nextf(d2max, 1);
	return d2max;
}

// What the handle types below hold right now, across the process (bt_debug_live_resources).
struct LiveResources { std::atomic<long long> dev_bytes{0}, pinned_bytes{0}; std::atomic<int> handles{0}; };
inline LiveResources g_live;

// A growable block of device memory (DevBuf) or page-locked host memory (PinnedBuf), freed with its owner.  `alloc` only grows: a block
// that is large enough is kept, a larger one replaces it (contents are not kept).  The contexts allocate in *_reserve, never on the
// per-call path unless a call exceeds what was reserved, in which case the call fails with BT_ERR_CAPACITY.
template <bool Pinned>
struct Block {
	void* p = nullptr;
	size_t bytes = 0;
	Block() = default;
	Block(const Block&) = delete;
	Block& operator=(const Block&) = delete;
	Block(Block&& o) noexcept : p(o.p), bytes(o.bytes) { o.p = nullptr; o.bytes = 0; }
	Block& operator=(Block&& o) noexcept { std::swap(p, o.p); std::swap(bytes, o.bytes); return *this; }
	~Block() { free(); }
	int alloc(size_t n) {
		if (n <= bytes) return BT_OK;
		free();
		if (Pinned) BT_CUDA(cudaMallocHost(&p, n));
		else BT_CUDA(cudaMalloc(&p, n));
		bytes = n;
		live() += (long long)n;
		return BT_OK;
	}
	template <class T> T* as() const { return reinterpret_cast<T*>(p); }
private:
	static std::atomic<long long>& live() { return Pinned ? g_live.pinned_bytes : g_live.dev_bytes; }
	void free() {
		if (!p) return;
		if (Pinned) cudaFreeHost(p);
		else cudaFree(p);
		live() -= (long long)bytes;
		p = nullptr; bytes = 0;
	}
};
using DevBuf = Block<false>;
using PinnedBuf = Block<true>;

// A CUDA event created on first use and destroyed with its owner.  Timing events are created with create(true) before they are
// recorded; record() creates the others without timing.
struct Event {
	cudaEvent_t e = nullptr;
	Event() = default;
	Event(const Event&) = delete;
	Event& operator=(const Event&) = delete;
	~Event() { if (e) { cudaEventDestroy(e); g_live.handles--; } }
	int create(bool timing = false) {
		if (e) return BT_OK;
		BT_CUDA(cudaEventCreateWithFlags(&e, timing ? cudaEventDefault : cudaEventDisableTiming));
		g_live.handles++;
		return BT_OK;
	}
	int record(cudaStream_t stream) { BT_TRY(create()); BT_CUDA(cudaEventRecord(e, stream)); return BT_OK; }
	int sync() const { if (e) BT_CUDA(cudaEventSynchronize(e)); return BT_OK; }     // (an event never recorded has nothing to wait for)
	operator cudaEvent_t() const { return e; }
};

// A non-blocking CUDA stream created on first use and destroyed with its owner.
struct Stream {
	cudaStream_t s = nullptr;
	Stream() = default;
	Stream(const Stream&) = delete;
	Stream& operator=(const Stream&) = delete;
	~Stream() { if (s) { cudaStreamDestroy(s); g_live.handles--; } }
	int create() {
		if (s) return BT_OK;
		BT_CUDA(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
		g_live.handles++;
		return BT_OK;
	}
	operator cudaStream_t() const { return s; }
};

// A page-locked block the host fills for an asynchronous upload, and the event recorded behind the copies that read it.  The entry
// points return before those copies run, so the block is rewritten (acquire) or regrown (reserve) only once the event has passed.
struct UploadBuf {
	PinnedBuf buf;
	Event ev;
	// the block, at least `bytes` large (0: as reserved), once the last upload from it is done
	template <class T> int acquire(size_t bytes, T** host) {
		BT_TRY(ev.sync());
		BT_TRY(buf.alloc(bytes));
		*host = buf.as<T>();
		return BT_OK;
	}
	int reserve(size_t bytes) {
		if (bytes > buf.bytes) BT_TRY(ev.sync());
		return buf.alloc(bytes);
	}
	// the copies from the block are queued on `stream`
	int in_flight(cudaStream_t stream) { return ev.record(stream); }
};

struct SolverState;   // solver.cu
struct MatcherState;  // knn.cu
struct RansacState;   // ransac.cu
struct FrontState;    // frontend.cu
struct PruneState;    // prune.cu
struct MatchCache;    // prune.cu
struct TracksDev;     // tracks_dev.cu
struct MetricsState;  // metrics.cu
struct NocsState;     // metrics.cu
struct OverlayState;  // overlay.cu
struct MatchVizState; // matchviz.cu
struct LfnetState;    // lfnet.cu
struct VosState;      // vos.cu

// The context owns the module states; each module defines the deleter of its state next to it, so the states stay private to their files.
struct StateDeleter {
	void operator()(SolverState*) const;
	void operator()(MatcherState*) const;
	void operator()(RansacState*) const;
	void operator()(FrontState*) const;
	void operator()(PruneState*) const;
	void operator()(MatchCache*) const;
	void operator()(TracksDev*) const;
	void operator()(MetricsState*) const;
	void operator()(NocsState*) const;
	void operator()(OverlayState*) const;
	void operator()(MatchVizState*) const;
	void operator()(LfnetState*) const;
	void operator()(VosState*) const;
};
template <class T> using StatePtr = std::unique_ptr<T, StateDeleter>;

}  // namespace bt

struct bt_ctx {
	int device = 0;
	int sm_count = 0;
	int cc_major = 0, cc_minor = 0;
	bt::StatePtr<bt::SolverState> solver;
	bt::StatePtr<bt::MatcherState> matcher;
	bt::StatePtr<bt::RansacState> ransac;
	bt::StatePtr<bt::FrontState> front;
	bt::StatePtr<bt::PruneState> prune;
	bt::StatePtr<bt::MatchCache> mcache;
	bt::StatePtr<bt::TracksDev> tracks;
	bt::StatePtr<bt::MetricsState> metrics;
	bt::StatePtr<bt::NocsState> nocs;
	bt::StatePtr<bt::OverlayState> overlay;
	bt::StatePtr<bt::MatchVizState> matchviz;
	bt::StatePtr<bt::LfnetState> lfnet;
	bt::StatePtr<bt::VosState> vos;
};

namespace bt {
// policy.cu: the float cofactor inverse of a row-major 4 x 4 (Eigen's Matrix4f::inverse()); false when it is singular
bool inverse4(const float* m, float* inv);
// segment.cu: largest-hull mode for the masked front end, and the LF-Net request
size_t hull_fill_smem(int H);
int segment_largest_hull(const uint8_t* const* mask_tbl_dev, int n, int H, int W, int32_t* label, int32_t* count, unsigned long long* best,
                         uint8_t* fill, cudaStream_t stream);
int launch_lfnet_request(const void* const* tbl_dev, const int32_t* roi_dev, int n, int H, int W, cudaStream_t stream);
// tracks_dev.cu: the device map-point table, driven pair by pair from bt_find_corres_pairs (prune.cu).  Frames are named by slot;
// tracks_slot maps a frame id to its slot (-1: the frame has no map yet, unless create is set).
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
