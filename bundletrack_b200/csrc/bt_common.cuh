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

// Reports a failed runtime call and consumes it as the runtime's last error, so that a later, unrelated cudaGetLastError() does not
// report it again (a sticky error stays sticky regardless).
#define BT_CUDA(x)                                                                                   \
	do {                                                                                             \
		cudaError_t e_ = (x);                                                                        \
		if (e_ != cudaSuccess) {                                                                     \
			bt::set_error("%s:%d %s -> %s", __FILE__, __LINE__, #x, cudaGetErrorString(e_));         \
			(void)cudaGetLastError();                                                                \
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
// Test aid (bt_debug_fail_alloc): when positive, the allocation that counts it down to 0 fails without calling CUDA.
inline std::atomic<int> g_fail_alloc{0};

// A growable block of device memory (DevBuf) or page-locked host memory (PinnedBuf), freed with its owner.  `alloc` only grows: a block
// that is large enough is kept, a larger one replaces it (contents are not kept).  The contexts allocate in *_reserve, never on the
// per-call path unless a call exceeds what was reserved, in which case the call fails with BT_ERR_CAPACITY.  The old block is freed
// before the new one is allocated, so a failed alloc leaves the block empty.
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
		BT_REQUIRE(!(g_fail_alloc > 0 && --g_fail_alloc == 0), BT_ERR_CUDA, "Block::alloc: %zu bytes refused by bt_debug_fail_alloc", n);
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

// The tables a call builds on the host for its kernels: typed slices of one block, added in order, each at a multiple of 256 bytes.
// A module lays out each call shape in one function of its counts; its reserve calls that function with the worst-case counts and every
// call with its real ones, so whether a call fits its reservation is decided by one piece of arithmetic (TableBlock::begin checks it).
template <class T> struct Slice {
	size_t off = 0, n = 0;
	size_t end() const { return off + sizeof(T) * n; }
};
struct TableLayout {
	size_t total = 0;
	template <class T> Slice<T> add(size_t n) {
		const Slice<T> s{total, n};
		total += (sizeof(T) * n + 255) & ~(size_t)255;
		return s;
	}
};

// The block a call's tables are built in and its device mirror.  NH page-locked blocks used in turn (with 2, a call waits only for the
// upload of the call before last), each with the event recorded behind the copies that read it, and NM device blocks at the same
// offsets.  The entry points return before those copies run, so a pinned block is rewritten (begin) or regrown (reserve) only once its
// event has passed.  The device blocks are allocated first: a reservation too large for the device fails there, before any pinning.
template <int NH = 1, int NM = 1> struct TableBlock {
	int reserve(size_t bytes) {
		for (DevBuf& d : mirror) BT_TRY(d.alloc(bytes));
		for (int k = 0; k < NH; k++) {
			if (bytes > pinned[k].bytes) BT_TRY(ev[k].sync());
			BT_TRY(pinned[k].alloc(bytes));
		}
		return BT_OK;
	}
	// the next pinned block, once its last upload is done, for tables laid out as L; BT_ERR_CAPACITY when L exceeds the reservation
	int begin(const char* who, const TableLayout& L) {
		cur = (cur + 1) % NH;
		BT_TRY(ev[cur].sync());
		size_t have = pinned[cur].bytes;
		for (const DevBuf& d : mirror) have = d.bytes < have ? d.bytes : have;
		BT_REQUIRE(L.total <= have, BT_ERR_CAPACITY, "%s: tables of %zu bytes exceed the %zu reserved", who, L.total, have);
		return BT_OK;
	}
	template <class T> T* host(const Slice<T>& s) const { return reinterpret_cast<T*>(pinned[cur].template as<char>() + s.off); }
	template <class T> T* dev(const Slice<T>& s, int m = 0) const { return reinterpret_cast<T*>(mirror[m].template as<char>() + s.off); }
	// bytes [from, to) of the current pinned block to device block m
	int send(size_t from, size_t to, cudaStream_t stream, int m = 0) {
		BT_CUDA(cudaMemcpyAsync(mirror[m].template as<char>() + from, pinned[cur].template as<char>() + from, to - from, cudaMemcpyHostToDevice, stream));
		return BT_OK;
	}
	// the copies from the current pinned block are queued on `stream`
	int in_flight(cudaStream_t stream) { return ev[cur].record(stream); }
	cudaEvent_t uploaded() const { return ev[cur]; }
private:
	PinnedBuf pinned[NH];
	Event ev[NH];
	DevBuf mirror[NM];
	int cur = 0;
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
struct ReconState;    // recon.cu
struct SurfaceState;  // metrics.cu
struct MaskState;     // metrics.cu

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
	void operator()(ReconState*) const;
	void operator()(SurfaceState*) const;
	void operator()(MaskState*) const;
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
	bt::StatePtr<bt::ReconState> recon;
	bt::StatePtr<bt::SurfaceState> surface;
	bt::StatePtr<bt::MaskState> mask;
};

namespace bt {
// Every module state has `bool ready`.  A reserve checks its arguments, then takes its state with take_state (ready = false), allocates,
// and sets its capacities and ready = true last; every other entry point looks its state up with state_of, which refuses a state that is
// not ready.  So after a reserve fails partway, nothing runs on the blocks it freed until a later reserve succeeds.
template <class T> int take_state(bt_ctx* ctx, StatePtr<T> bt_ctx::*member, T** out) {
	BT_CUDA(cudaSetDevice(ctx->device));
	StatePtr<T>& s = ctx->*member;
	if (!s) s.reset(new T());
	s->ready = false;
	*out = s.get();
	return BT_OK;
}
template <class T> int state_of(bt_ctx* ctx, StatePtr<T> bt_ctx::*member, const char* who, const char* reserve, T** out) {
	BT_REQUIRE(ctx, BT_ERR_INVALID_ARG, "%s: ctx is NULL", who);
	T* s = (ctx->*member).get();
	BT_REQUIRE(s && s->ready, BT_ERR_INVALID_ARG, "%s: call %s (successfully) first", who, reserve);
	BT_CUDA(cudaSetDevice(ctx->device));
	*out = s;
	return BT_OK;
}

// knn.cu: the argument checks of bt_matcher_reserve, which bt_pipeline_reserve makes before it changes any state
int matcher_reserve_args(int max_pairs, int max_feats, int dim);
// policy.cu: the float cofactor inverse of a row-major 4 x 4 (Eigen's Matrix4f::inverse()); false when it is singular
bool inverse4(const float* m, float* inv);
// segment.cu: largest-hull mode for the masked front end, and the LF-Net request
size_t hull_fill_smem(int H);
int segment_largest_hull(const uint8_t* const* mask_tbl_dev, int n, int H, int W, int32_t* label, int32_t* count, unsigned long long* best,
                         uint8_t* fill, cudaStream_t stream);
int launch_lfnet_request(const void* const* tbl_dev, const int32_t* roi_dev, int n, int H, int W, cudaStream_t stream);
// tracks_dev.cu: the device map-point table, driven pair by pair from bt_find_corres_pairs (prune.cu).  Frames are named by slot;
// tracks_slot maps a frame id to its slot (-1: the frame has no map yet, unless create is set).  tracks_state is state_of for the table.
int tracks_state(bt_ctx* ctx, const char* who);
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
