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
};

namespace bt {
void solver_destroy(bt_ctx* ctx);
void matcher_destroy(bt_ctx* ctx);
void ransac_destroy(bt_ctx* ctx);
void prune_destroy(bt_ctx* ctx);
void mcache_destroy(bt_ctx* ctx);
void front_destroy(bt_ctx* ctx);
// segment.cu: largest-hull mode for the masked front end, and the LF-Net request
size_t hull_fill_smem(int H);
int segment_largest_hull(const uint8_t* const* mask_tbl_dev, int n, int H, int W, int32_t* label, int32_t* count, unsigned long long* best,
                         uint8_t* fill, cudaStream_t stream);
int launch_lfnet_request(const void* const* tbl_dev, const int32_t* roi_dev, int n, int H, int W, cudaStream_t stream);
}
