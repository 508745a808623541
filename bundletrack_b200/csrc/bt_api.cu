// bt_api.cu — context lifetime, error string, raw device-memory helpers of the C-ABI (include/bundletrack_b200.h).
#include <stdarg.h>
#include "bt_common.cuh"

namespace bt {
static thread_local char g_err[512] = "";
void set_error(const char* fmt, ...) {
	va_list ap;
	va_start(ap, fmt);
	vsnprintf(g_err, sizeof g_err, fmt, ap);
	va_end(ap);
}
}  // namespace bt

extern "C" const char* bt_last_error(void) { return bt::g_err; }
extern "C" int bt_version(void) { return 101; }

extern "C" int bt_ctx_create(bt_ctx** out, int device) {
	BT_REQUIRE(out != nullptr, BT_ERR_INVALID_ARG, "bt_ctx_create: out is NULL");
	*out = nullptr;
	int n = 0;
	cudaError_t e = cudaGetDeviceCount(&n);
	if (e != cudaSuccess || n <= 0) {
		bt::set_error("bt_ctx_create: no CUDA device (%s); this library has no CPU fallback", cudaGetErrorString(e));
		return BT_ERR_NO_DEVICE;
	}
	BT_REQUIRE(device >= 0 && device < n, BT_ERR_INVALID_ARG, "bt_ctx_create: device %d out of range [0,%d)", device, n);
	BT_CUDA(cudaSetDevice(device));
	cudaDeviceProp prop;
	BT_CUDA(cudaGetDeviceProperties(&prop, device));
	if (prop.major != 9 || prop.minor != 0) {
		bt::set_error("bt_ctx_create: device %d is sm_%d%d; this library is built for sm_90a only", device, prop.major, prop.minor);
		return BT_ERR_NO_DEVICE;
	}
	bt_ctx* c = new bt_ctx();
	c->device = device;
	c->sm_count = prop.multiProcessorCount;
	c->cc_major = prop.major;
	c->cc_minor = prop.minor;
	*out = c;
	return BT_OK;
}

extern "C" void bt_ctx_destroy(bt_ctx* ctx) {
	if (!ctx) return;
	cudaSetDevice(ctx->device);
	delete ctx;
}

// Test aid: what the handle types of bt_common.cuh hold right now, across the process.  Memory from bt_dev_alloc / bt_host_alloc_pinned
// is the caller's and is not counted.
extern "C" int bt_debug_live_resources(long long* device_bytes, long long* pinned_bytes, int* handles) {
	BT_REQUIRE(device_bytes && pinned_bytes && handles, BT_ERR_INVALID_ARG, "bt_debug_live_resources: NULL argument");
	*device_bytes = bt::g_live.dev_bytes; *pinned_bytes = bt::g_live.pinned_bytes; *handles = bt::g_live.handles;
	return BT_OK;
}

// Test aid: the nth allocation of a library-owned block from now fails with BT_ERR_CUDA without calling CUDA (0 disarms).
extern "C" int bt_debug_fail_alloc(int nth) {
	BT_REQUIRE(nth >= 0, BT_ERR_INVALID_ARG, "bt_debug_fail_alloc: nth %d < 0", nth);
	bt::g_fail_alloc = nth;
	return BT_OK;
}

extern "C" int bt_dev_alloc(void** out, size_t bytes) {
	BT_REQUIRE(out != nullptr, BT_ERR_INVALID_ARG, "bt_dev_alloc: out is NULL");
	BT_CUDA(cudaMalloc(out, bytes ? bytes : 1));
	return BT_OK;
}
extern "C" int bt_dev_free(void* p) { BT_CUDA(cudaFree(p)); return BT_OK; }
extern "C" int bt_memcpy_h2d(void* d, const void* s, size_t bytes, void* stream) {
	BT_CUDA(cudaMemcpyAsync(d, s, bytes, cudaMemcpyHostToDevice, (cudaStream_t)stream));
	return BT_OK;
}
extern "C" int bt_memcpy_d2h(void* d, const void* s, size_t bytes, void* stream) {
	BT_CUDA(cudaMemcpyAsync(d, s, bytes, cudaMemcpyDeviceToHost, (cudaStream_t)stream));
	BT_CUDA(cudaStreamSynchronize((cudaStream_t)stream));
	return BT_OK;
}
extern "C" int bt_host_alloc_pinned(void** out, size_t bytes) {
	BT_REQUIRE(out != nullptr, BT_ERR_INVALID_ARG, "bt_host_alloc_pinned: out is NULL");
	BT_CUDA(cudaMallocHost(out, bytes ? bytes : 1));
	return BT_OK;
}
extern "C" int bt_host_free_pinned(void* p) { BT_CUDA(cudaFreeHost(p)); return BT_OK; }
extern "C" int bt_stream_sync(void* stream) { BT_CUDA(cudaStreamSynchronize((cudaStream_t)stream)); return BT_OK; }
