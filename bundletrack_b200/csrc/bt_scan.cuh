// bt_scan.cuh — the library's integer scans and its order-preserving float key.  Device code: bt_common.cuh stays plain C++.
// The scans add integers, so their results do not depend on the order of the additions.
#pragma once
#include <cuda_runtime.h>
#include <string.h>

namespace bt {

// int, unsigned, and int2: the mesh scans its (vertex, face) counts together, component-wise
__device__ __forceinline__ int2 operator+(int2 a, int2 b) { return make_int2(a.x + b.x, a.y + b.y); }
__device__ __forceinline__ int2 operator-(int2 a, int2 b) { return make_int2(a.x - b.x, a.y - b.y); }
template <typename T> __device__ __forceinline__ T shfl_up(T v, int o) { return __shfl_up_sync(0xffffffffu, v, o); }
template <typename T> __device__ __forceinline__ T shfl_idx(T v, int lane) { return __shfl_sync(0xffffffffu, v, lane); }
__device__ __forceinline__ int2 shfl_up(int2 v, int o) { return make_int2(shfl_up(v.x, o), shfl_up(v.y, o)); }
__device__ __forceinline__ int2 shfl_idx(int2 v, int lane) { return make_int2(shfl_idx(v.x, lane), shfl_idx(v.y, lane)); }

// Inclusive prefix sum over the lanes of a warp; all 32 lanes call it.
template <typename T>
__device__ __forceinline__ T warp_incl_scan(T v) {
	const int lane = threadIdx.x & 31;
#pragma unroll
	for (int o = 1; o < 32; o <<= 1) { const T u = shfl_up(v, o); if (lane >= o) v = v + u; }
	return v;
}

// Exclusive prefix sum over the CTA in thread order; *total = the CTA's sum.  Every thread calls it; blockDim.x is a multiple of 32,
// at most 1024.  s: blockDim.x / 32 elements of shared memory, free again on return, so calls may follow one another.  Every warp
// scans the warp totals itself, so there are two barriers: one before the totals are read and one after.
template <typename T>
__device__ __forceinline__ T block_excl_scan(T v, T* s, T* total) {
	const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
	const T x = warp_incl_scan(v);
	if (lane == 31) s[wid] = x;
	__syncthreads();
	const T t = lane < (int)(blockDim.x >> 5) ? s[lane] : T{};
	__syncthreads();
	const T w = warp_incl_scan(t);
	*total = shfl_idx(w, 31);
	return x - v + shfl_idx(w - t, wid);
}

// A float's order-preserving image in int, and back: the integer min / max of the keys order the floats (-0 below +0).
__host__ __device__ __forceinline__ int ordered_key(float f) {
	int i;
	memcpy(&i, &f, sizeof i);
	return i >= 0 ? i : i ^ 0x7fffffff;
}
__host__ __device__ __forceinline__ float ordered_float(int k) {
	k = k >= 0 ? k : k ^ 0x7fffffff;
	float f;
	memcpy(&f, &k, sizeof f);
	return f;
}

}  // namespace bt
