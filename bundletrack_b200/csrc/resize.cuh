// resize.cuh — OpenCV's 8-bit INTER_LINEAR resize sampled one output pixel at a time (cv::resize, resize.cpp), shared by the LF-Net
// request (segment.cu) and the match images (matchviz.cu).
#pragma once
#include <stdint.h>

namespace bt {

// cv::resize's INTER_LINEAR source index and 11-bit weights for destination index d of a dst-long axis over a src-long one (resize.cpp:
// fx = (float)((d + 0.5) * scale - 0.5), scale = 1 / (dst / src) in double; the weights are saturate_cast<short>(w * 2048), i.e. rounded
// half to even).  Only the horizontal direction moves the weight onto the edge sample; both clamp the indices.
// lin_coeffs_at takes that scale precomputed.
__device__ __forceinline__ void lin_coeffs_at(int d, double scale, int src, bool clamp_weights, int& s0, int& s1, int& w0, int& w1) {
	float fx = __double2float_rn(__dadd_rn(__dmul_rn((double)d + 0.5, scale), -0.5));
	int s = (int)floorf(fx);
	fx = __fsub_rn(fx, (float)s);
	if (clamp_weights) {
		if (s < 0) { fx = 0.f; s = 0; }
		if (s >= src - 1) { fx = 0.f; s = src - 1; }
	}
	w0 = __float2int_rn(__fmul_rn(__fsub_rn(1.f, fx), 2048.f));
	w1 = __float2int_rn(__fmul_rn(fx, 2048.f));
	s0 = min(max(s, 0), src - 1); s1 = min(max(s + 1, 0), src - 1);
}

__device__ __forceinline__ void lin_coeffs(int d, int dst, int src, bool clamp_weights, int& s0, int& s1, int& w0, int& w1) {
	lin_coeffs_at(d, __ddiv_rn(1.0, __ddiv_rn((double)dst, (double)src)), src, clamp_weights, s0, s1, w0, w1);
}

// one channel from its four taps: the horizontal pass exact, the vertical pass as OpenCV's vector path rounds it:
// ((b0 * (h0 >> 4)) >> 16) + ((b1 * (h1 >> 4)) >> 16), then (t + 2) >> 2
__device__ __forceinline__ uint8_t lin_blend(int p00, int p01, int p10, int p11, int a0, int a1, int b0, int b1) {
	const int h0 = p00 * a0 + p01 * a1, h1 = p10 * a0 + p11 * a1;
	const int t = ((b0 * (h0 >> 4)) >> 16) + ((b1 * (h1 >> 4)) >> 16);
	return (uint8_t)min(max((t + 2) >> 2, 0), 255);
}

}  // namespace bt
