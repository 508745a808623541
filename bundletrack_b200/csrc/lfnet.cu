// lfnet.cu — LF-Net inference on the device: the network lf-net-release/run_server.py builds (mso_resnet_detector + simple_desc,
// desc_inputs = photos, use_nms3d), from the 400 x 400 request image to the keypoints and descriptors of the server's reply.
// FP32 throughout; every reduction has a fixed order, so results do not depend on scheduling or on how requests are batched.
// oracle/lfnet_oracle.py is the float64 statement of the same graph, written from the reference's Python.  DESIGN.md §3.12.
#include <errno.h>
#include <math.h>
#include "bt_common.cuh"
#include "bt_scan.cuh"

namespace bt {
namespace {

constexpr int SIDE = 400;                 // the request image (segment.cu)
constexpr int HW = SIDE * SIDE;
constexpr int TC = 16, TK = 5;            // trunk channels and kernel; bt_lfnet_reserve refuses other values
constexpr int MAX_SCALES = 8, MAX_BLOCKS = 8, MAX_DESC = 6;
constexpr int FC_HIDDEN = 512;            // simple_desc.py:44
constexpr float IN_EPS = 1e-3f;           // instance_normalization (det_tools.py:793)

__device__ __forceinline__ float leaky(float v, float a) { return v > 0.f ? v : v * a; }   // tf.nn.leaky_relu

// ---- trunk ---------------------------------------------------------------------------------------------------------------------------
// run_server.py:155-157: cv2.cvtColor(request, COLOR_RGB2GRAY) on BGR bytes, so byte 0 takes the red weight; OpenCV's uint8 path is
// OpenCV 4's fixed point (9798 R + 19235 G + 3735 B + 2^14) >> 15.  Then / 255 in float32.
__global__ void __launch_bounds__(256) k_grey(const uint8_t* const* req, float* grey) {
	const int f = blockIdx.y, p = blockIdx.x * 256 + threadIdx.x;
	if (p >= HW) return;
	const uint8_t* r = req[f] + 3 * (size_t)p;
	const int g = ((int)r[0] * 9798 + (int)r[1] * 19235 + (int)r[2] * 3735 + (1 << 14)) >> 15;
	grey[(size_t)f * HW + p] = (float)g / 255.0f;
}

// conv2d_fixed_padding at stride 1 (SAME, 5 x 5) of CIN -> 16 channels on CHW maps, one 32 x 16 output tile per CTA, each thread two
// pixels (rows ty and ty + 8) x 16 channels.  The input is taken through the BN + leaky ReLU that precedes the conv (s == nullptr: as it
// is), zero outside the image; res != nullptr adds the residual block's shortcut.  w is TF's [ky][kx][ci][co].
constexpr int CT_W = 32, CT_H = 16, CT_CH = 4;
template <int CIN>
__global__ void __launch_bounds__(256) k_trunk_conv(const float* __restrict__ in, const float* __restrict__ w, const float* __restrict__ b,
                                                    const float* __restrict__ s, const float* __restrict__ t, float alpha,
                                                    const float* __restrict__ res, float* __restrict__ out) {
	constexpr int CH = CIN < CT_CH ? CIN : CT_CH;
	__shared__ __align__(16) float ws[TK * TK * CIN * TC];
	__shared__ float tile[CH][CT_H + TK - 1][CT_W + TK - 1];
	const int f = blockIdx.z, x0 = blockIdx.x * CT_W, y0 = blockIdx.y * CT_H;
	const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
	for (int i = threadIdx.x; i < TK * TK * CIN * TC; i += 256) ws[i] = w[i];
	const float* src = in + (size_t)f * CIN * HW;
	float acc0[TC], acc1[TC];
#pragma unroll
	for (int c = 0; c < TC; c++) { acc0[c] = 0.f; acc1[c] = 0.f; }
	for (int c0 = 0; c0 < CIN; c0 += CH) {
		__syncthreads();
		for (int i = threadIdx.x; i < CH * (CT_H + TK - 1) * (CT_W + TK - 1); i += 256) {
			const int c = i / ((CT_H + TK - 1) * (CT_W + TK - 1)), r = i % ((CT_H + TK - 1) * (CT_W + TK - 1));
			const int yy = y0 + r / (CT_W + TK - 1) - TK / 2, xx = x0 + r % (CT_W + TK - 1) - TK / 2;
			float v = 0.f;
			if (yy >= 0 && yy < SIDE && xx >= 0 && xx < SIDE) {
				v = src[(size_t)(c0 + c) * HW + yy * SIDE + xx];
				if (s) v = leaky(fmaf(v, s[c0 + c], t[c0 + c]), alpha);
			}
			tile[c][r / (CT_W + TK - 1)][r % (CT_W + TK - 1)] = v;
		}
		__syncthreads();
#pragma unroll 1
		for (int c = 0; c < CH; c++)
#pragma unroll 1
			for (int ky = 0; ky < TK; ky++)
#pragma unroll
				for (int kx = 0; kx < TK; kx++) {
					const float v0 = tile[c][ty + ky][tx + kx], v1 = tile[c][ty + 8 + ky][tx + kx];
					const float4* wp = reinterpret_cast<const float4*>(ws + ((ky * TK + kx) * CIN + c0 + c) * TC);
#pragma unroll
					for (int q = 0; q < TC / 4; q++) {
						const float4 wq = wp[q];
						acc0[4 * q] = fmaf(v0, wq.x, acc0[4 * q]); acc0[4 * q + 1] = fmaf(v0, wq.y, acc0[4 * q + 1]);
						acc0[4 * q + 2] = fmaf(v0, wq.z, acc0[4 * q + 2]); acc0[4 * q + 3] = fmaf(v0, wq.w, acc0[4 * q + 3]);
						acc1[4 * q] = fmaf(v1, wq.x, acc1[4 * q]); acc1[4 * q + 1] = fmaf(v1, wq.y, acc1[4 * q + 1]);
						acc1[4 * q + 2] = fmaf(v1, wq.z, acc1[4 * q + 2]); acc1[4 * q + 3] = fmaf(v1, wq.w, acc1[4 * q + 3]);
					}
				}
	}
	const int x = x0 + tx;
	if (x >= SIDE) return;
	float* dst = out + (size_t)f * TC * HW;
	const float* rs = res ? res + (size_t)f * TC * HW : nullptr;
#pragma unroll
	for (int h = 0; h < 2; h++) {
		const int y = y0 + ty + 8 * h;
		if (y >= SIDE) continue;
#pragma unroll
		for (int c = 0; c < TC; c++) {
			const size_t q = (size_t)c * HW + y * SIDE + x;
			float v = (h ? acc1[c] : acc0[c]) + b[c];
			if (rs) v += rs[q];
			dst[q] = v;
		}
	}
}

// fin-bn + activation: the trunk's feat_maps (mso_resnet_detector.py:97-104)
__global__ void __launch_bounds__(256) k_bn_act(const float* __restrict__ in, const float* __restrict__ s, const float* __restrict__ t, float alpha,
                                                float* __restrict__ out, int n) {
	const size_t i = (size_t)blockIdx.x * 256 + threadIdx.x;
	if (i >= (size_t)n * TC * HW) return;
	const int c = (int)((i / HW) % TC);
	out[i] = leaky(fmaf(in[i], s[c], t[c]), alpha);
}

// ---- per scale -----------------------------------------------------------------------------------------------------------------------
// TF1 resize_bilinear, align_corners = False, no half-pixel centres: src = dst * (in / out) in float, lower = floor, upper =
// min(ceil, in - 1), lerp = src - floor; top / bottom lerps in x, then y.
struct Lerp { int lo, hi; float f; };
__device__ __forceinline__ Lerp lerp_of(int d, float scale, int in) {
	const float sx = (float)d * scale, fl = floorf(sx);
	Lerp l; l.lo = max((int)fl, 0); l.hi = min((int)ceilf(sx), in - 1); l.f = sx - fl;
	return l;
}
__device__ __forceinline__ float blerp(float tl, float tr, float bl, float br, float xf, float yf) {
	const float top = tl + (tr - tl) * xf, bot = bl + (br - bl) * xf;
	return top + (bot - top) * yf;
}

struct ScaleArgs {
	int n_scales;
	int size[MAX_SCALES];
	size_t logit_off[MAX_SCALES];        // floats into one image's logits block
	const float* w[MAX_SCALES];          // score_conv_i weights [5][5][16][1] and bias
	const float* b[MAX_SCALES];
	float factor[MAX_SCALES];            // scale_factors as the float32 constant (inference.py:171)
};

// score_conv_i on the feature maps resized to S_i x S_i (mso_resnet_detector.py:129-137); the resize is evaluated while the tile loads.
// One 32 x 8 tile of one scale of one image per CTA.
__global__ void __launch_bounds__(256) k_score_conv(const float* __restrict__ feat, ScaleArgs a, float* __restrict__ logits, size_t logit_stride) {
	const int f = blockIdx.z / a.n_scales, si = blockIdx.z % a.n_scales, S = a.size[si];
	const int x0 = blockIdx.x * 32, y0 = blockIdx.y * 8;
	if (x0 >= S || y0 >= S) return;
	__shared__ float tile[TC][8 + TK - 1][32 + TK - 1];
	__shared__ float ws[TK * TK * TC];
	for (int i = threadIdx.x; i < TK * TK * TC; i += 256) ws[i] = a.w[si][i];
	const float scale = (float)SIDE / (float)S;
	const float* src = feat + (size_t)f * TC * HW;
	for (int i = threadIdx.x; i < (8 + TK - 1) * (32 + TK - 1); i += 256) {
		const int yy = y0 + i / (32 + TK - 1) - TK / 2, xx = x0 + i % (32 + TK - 1) - TK / 2;
		if (yy < 0 || yy >= S || xx < 0 || xx >= S) {
			for (int c = 0; c < TC; c++) tile[c][i / (32 + TK - 1)][i % (32 + TK - 1)] = 0.f;
			continue;
		}
		const Lerp ly = lerp_of(yy, scale, SIDE), lx = lerp_of(xx, scale, SIDE);
		for (int c = 0; c < TC; c++) {
			const float* m = src + (size_t)c * HW;
			tile[c][i / (32 + TK - 1)][i % (32 + TK - 1)] =
				blerp(m[ly.lo * SIDE + lx.lo], m[ly.lo * SIDE + lx.hi], m[ly.hi * SIDE + lx.lo], m[ly.hi * SIDE + lx.hi], lx.f, ly.f);
		}
	}
	__syncthreads();
	const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5, x = x0 + tx, y = y0 + ty;
	if (x >= S || y >= S) return;
	float acc = 0.f;
	for (int ky = 0; ky < TK; ky++)
		for (int kx = 0; kx < TK; kx++)
#pragma unroll
			for (int c = 0; c < TC; c++) acc = fmaf(tile[c][ty + ky][tx + kx], ws[(ky * TK + kx) * TC + c], acc);
	logits[(size_t)f * logit_stride + a.logit_off[si] + (size_t)y * S + x] = acc + a.b[si][0];
}

// Instance-norm moments of one score map per CTA (det_tools.py:789-803): mean, then the mean squared deviation, each a float64 sum in a
// fixed order (per thread strided, then a fixed tree).  stats = (mean, 1 / sqrt(var + 1e-3)).
constexpr int MOM_THREADS = 1024;
__device__ double block_sum_fixed(double v, double* sh) {
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
	if (lane == 0) sh[warp] = v;
	__syncthreads();
	if (warp == 0) {
		v = lane < MOM_THREADS / 32 ? sh[lane] : 0.0;
		for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
		if (lane == 0) sh[32] = v;
	}
	__syncthreads();
	const double r = sh[32];
	__syncthreads();
	return r;
}
__global__ void __launch_bounds__(MOM_THREADS) k_moments(const float* __restrict__ logits, ScaleArgs a, size_t logit_stride, float2* __restrict__ stats) {
	__shared__ double sh[33];
	const int f = blockIdx.x / a.n_scales, si = blockIdx.x % a.n_scales, n = a.size[si] * a.size[si];
	const float* l = logits + (size_t)f * logit_stride + a.logit_off[si];
	double s = 0.0;
	for (int i = threadIdx.x; i < n; i += MOM_THREADS) s += l[i];
	const double mean = block_sum_fixed(s, sh) / n;
	double q = 0.0;
	for (int i = threadIdx.x; i < n; i += MOM_THREADS) { const double d = l[i] - mean; q += d * d; }
	const double var = block_sum_fixed(q, sh) / n;
	if (threadIdx.x == 0) stats[blockIdx.x] = make_float2((float)mean, (float)(1.0 / sqrt(var + (double)IN_EPS)));
}

// ---- detection -----------------------------------------------------------------------------------------------------------------------
// The normalised logits resized back to 400 x 400 (build_multi_scale_deep_detector_3DNMS, inference.py:176-180) as L[s][p], and the
// maximum over scales per pixel (the 3-D max pool's scale axis, det_tools.py:778).
__global__ void __launch_bounds__(256) k_upsample(const float* __restrict__ logits, const float2* __restrict__ stats, ScaleArgs a, size_t logit_stride,
                                                  float* __restrict__ L, float* __restrict__ Lmax) {
	const int f = blockIdx.y, p = blockIdx.x * 256 + threadIdx.x;
	if (p >= HW) return;
	const int y = p / SIDE, x = p % SIDE;
	float m = -INFINITY;
	for (int si = 0; si < a.n_scales; si++) {
		const int S = a.size[si];
		const float scale = (float)S / (float)SIDE;
		const Lerp ly = lerp_of(y, scale, S), lx = lerp_of(x, scale, S);
		const float* l = logits + (size_t)f * logit_stride + a.logit_off[si];
		const float2 st = stats[f * a.n_scales + si];
		auto nv = [&](int yy, int xx) { return (l[(size_t)yy * S + xx] - st.x) * st.y; };
		const float v = blerp(nv(ly.lo, lx.lo), nv(ly.lo, lx.hi), nv(ly.hi, lx.lo), nv(ly.hi, lx.hi), lx.f, ly.f);
		L[((size_t)f * a.n_scales + si) * HW + p] = v;
		m = fmaxf(m, v);
	}
	Lmax[(size_t)f * HW + p] = m;
}

// A 1-D box of radius r along x or y, clipped at the border: the maximum (SAME max pooling ignores padding) or the sum in a fixed order
// (SAME conv pads zeros).  The 15 x 15 windows of soft_nms_3d are two such passes.
__global__ void __launch_bounds__(256) k_box(const float* __restrict__ in, float* __restrict__ out, int r, int vertical, int is_sum) {
	const int f = blockIdx.y, p = blockIdx.x * 256 + threadIdx.x;
	if (p >= HW) return;
	const int y = p / SIDE, x = p % SIDE, c = vertical ? y : x;
	const float* m = in + (size_t)f * HW;
	float acc = is_sum ? 0.f : -INFINITY;
	for (int d = max(c - r, 0); d <= min(c + r, SIDE - 1); d++) {
		const float v = m[vertical ? d * SIDE + x : y * SIDE + d];
		acc = is_sum ? acc + v : fmaxf(acc, v);
	}
	out[(size_t)f * HW + p] = acc;
}

// exp_maps = exp(com_strength (L - max_maps)) per scale (det_tools.py:780) and their sum over scales, which the box sum then spreads.
__global__ void __launch_bounds__(256) k_exp(float* __restrict__ L, const float* __restrict__ M, float* __restrict__ Es, int n_scales, float com) {
	const int f = blockIdx.y, p = blockIdx.x * 256 + threadIdx.x;
	if (p >= HW) return;
	const float m = M[(size_t)f * HW + p];
	float s = 0.f;
	for (int si = 0; si < n_scales; si++) {
		float* l = L + ((size_t)f * n_scales + si) * HW + p;
		const float e = expf(com * (*l - m));
		*l = e;
		s += e;
	}
	Es[(size_t)f * HW + p] = s;
}

// probs = exp_maps / (sum_ex + 1e-6) (det_tools.py:785); soft_max_and_argmax_1d over the scales (det_tools.py:1707-1725) gives
// max_heatmaps and max_scales; max_heatmaps times the pad mask (inference.py:201-202).
__global__ void __launch_bounds__(256) k_soft_scale(const float* __restrict__ E, const float* __restrict__ S, ScaleArgs a, float c1, float c2, int pad,
                                                    float* __restrict__ heat, float* __restrict__ scl) {
	const int f = blockIdx.y, p = blockIdx.x * 256 + threadIdx.x;
	if (p >= HW) return;
	const int y = p / SIDE, x = p % SIDE;
	float pr[MAX_SCALES], pm = -INFINITY;
	const float den = S[(size_t)f * HW + p] + 1e-6f;
#pragma unroll
	for (int si = 0; si < MAX_SCALES; si++)
		if (si < a.n_scales) { pr[si] = E[((size_t)f * a.n_scales + si) * HW + p] / den; pm = fmaxf(pm, pr[si]); }
	float s1 = 0.f, s2 = 0.f;
#pragma unroll
	for (int si = 0; si < MAX_SCALES; si++)
		if (si < a.n_scales) { s1 += expf(c1 * (pr[si] - pm)); s2 += expf(c2 * (pr[si] - pm)); }
	float h = 0.f, sc = 0.f;
#pragma unroll
	for (int si = 0; si < MAX_SCALES; si++)
		if (si < a.n_scales) {
			h += pr[si] * (expf(c1 * (pr[si] - pm)) / (s1 + 1e-8f));
			sc += a.factor[si] * (expf(c2 * (pr[si] - pm)) / (s2 + 1e-8f));
		}
	const bool in = y >= pad && y < SIDE - pad && x >= pad && x < SIDE - pad;
	heat[(size_t)f * HW + p] = in ? h : 0.f;
	scl[(size_t)f * HW + p] = sc;
}

// non_max_suppression (det_tools.py:806-834): values below thresh count as 0, zero padding, and the centre must be strictly greater
// than every other pixel of the k x k window.  nms_scores = max_heatmaps * nms_maps * crop mask (inference.py:205-207).
__global__ void __launch_bounds__(256) k_nms(const float* __restrict__ heat, float thresh, int hk, int crop, float* __restrict__ score,
                                             uint8_t* __restrict__ peak) {
	const int f = blockIdx.y, p = blockIdx.x * 256 + threadIdx.x;
	if (p >= HW) return;
	const int y = p / SIDE, x = p % SIDE;
	const float* m = heat + (size_t)f * HW;
	auto wk = [&](int yy, int xx) { if (yy < 0 || yy >= SIDE || xx < 0 || xx >= SIDE) return 0.f; const float v = m[yy * SIDE + xx]; return v < thresh ? 0.f : v; };
	const float c = wk(y, x);
	bool pk = true;
	for (int dy = -hk; dy <= hk; dy++)
		for (int dx = -hk; dx <= hk; dx++)
			if ((dy || dx) && !(c > wk(y + dy, x + dx))) pk = false;
	const bool in = y >= crop && y < SIDE - crop && x >= crop && x < SIDE - crop;
	score[(size_t)f * HW + p] = (pk && in) ? m[p] : 0.f;
	peak[(size_t)f * HW + p] = pk;
}

// make_top_k_sparse_tensor + "* nms_maps" + extract_keypoints (inference.py:208-214, det_tools.py:681-693, 848-861), one CTA per image:
// a radix select of the k-th largest score (ties at it: lower flat index first), then the selected pixels that are NMS peaks in
// row-major order (tf.where).  Each thread owns one contiguous run of pixels, so thread order is pixel order for both scans.
constexpr int TOPK_THREADS = 1024;
__device__ __forceinline__ unsigned okey(float v) { const unsigned u = __float_as_uint(v); return (u & 0x80000000u) ? ~u : (u | 0x80000000u); }
__global__ void __launch_bounds__(TOPK_THREADS) k_topk(const float* __restrict__ score, const uint8_t* __restrict__ peak, int k, int2* __restrict__ kint,
                                                       int32_t* __restrict__ n_out) {
	__shared__ int hist[256];
	__shared__ int sh[TOPK_THREADS / 32];
	__shared__ unsigned s_prefix;
	__shared__ int s_remaining;
	const int f = blockIdx.x;
	const float* sc = score + (size_t)f * HW;
	if (threadIdx.x == 0) { s_prefix = 0u; s_remaining = k; }
	unsigned mask = 0u;
	for (int shift = 24; shift >= 0; shift -= 8) {
		for (int i = threadIdx.x; i < 256; i += TOPK_THREADS) hist[i] = 0;
		__syncthreads();
		const unsigned prefix = s_prefix;
		for (int p = threadIdx.x; p < HW; p += TOPK_THREADS) {
			const unsigned u = okey(sc[p]);
			if ((u & mask) == prefix) atomicAdd(&hist[(u >> shift) & 255u], 1);
		}
		__syncthreads();
		if (threadIdx.x == 0) {
			int rem = s_remaining, d = 255;
			for (; d > 0 && hist[d] < rem; d--) rem -= hist[d];
			s_prefix = prefix | ((unsigned)d << shift);
			s_remaining = rem;
		}
		mask |= 255u << shift;
		__syncthreads();
	}
	const unsigned T = s_prefix;
	const int need_eq = s_remaining;           // pixels equal to the k-th value that are still taken, lowest index first
	constexpr int RUN = (HW + TOPK_THREADS - 1) / TOPK_THREADS;
	const int p0 = threadIdx.x * RUN, p1 = min(p0 + RUN, HW);
	int n_eq = 0, total;
	for (int p = p0; p < p1; p++) n_eq += okey(sc[p]) == T;
	int eq_rank = block_excl_scan(n_eq, sh, &total);
	const uint8_t* pk = peak + (size_t)f * HW;
	int n_kp = 0;
	for (int p = p0, r = eq_rank; p < p1; p++) {
		const unsigned u = okey(sc[p]);
		const bool sel = u > T || (u == T && r++ < need_eq);
		n_kp += sel && pk[p];
	}
	int pos = block_excl_scan(n_kp, sh, &total);
	for (int p = p0, r = eq_rank; p < p1; p++) {
		const unsigned u = okey(sc[p]);
		const bool sel = u > T || (u == T && r++ < need_eq);
		if (sel && pk[p]) kint[(size_t)f * k + pos++] = make_int2(p % SIDE, p / SIDE);
	}
	if (threadIdx.x == 0) n_out[f] = total;
}

// ---- refinement, orientation, patches ------------------------------------------------------------------------------------------------
// transformer_crop's sampler (spatial_transformer.py:97-136): floor, +1, both clipped, weights from the clipped corners.
__device__ __forceinline__ float st_sample(const float* img, float x, float y) {
	int x0 = (int)floorf(x), y0 = (int)floorf(y), x1 = x0 + 1, y1 = y0 + 1;
	x0 = min(max(x0, 0), SIDE - 1); x1 = min(max(x1, 0), SIDE - 1); y0 = min(max(y0, 0), SIDE - 1); y1 = min(max(y1, 0), SIDE - 1);
	const float x0f = (float)x0, x1f = (float)x1, y0f = (float)y0, y1f = (float)y1;
	const float wa = (x1f - x) * (y1f - y), wb = (x1f - x) * (y - y0f), wc = (x - x0f) * (y1f - y), wd = (x - x0f) * (y - y0f);
	return wa * img[y0 * SIDE + x0] + wb * img[y1 * SIDE + x0] + wc * img[y0 * SIDE + x1] + wd * img[y1 * SIDE + x1];
}
__device__ __forceinline__ float lin(int i, int n) { const float step = 2.0f / (float)(n - 1); return -1.0f + step * (float)i; }   // tf.linspace(-1, 1, n)

struct KpArgs {
	const float* heat; const float* scl; const float* feat; const float* grey;
	const int2* kint; const int32_t* n_kp;
	const float* ori_w; const float* ori_b;
	int top_k, loc, patch;
	float kp_com;
	float* kpts_out;          // [n][top_k][2], the refined keypoints
	float2* ori;              // [n * top_k] (cos, sin)
	float* patches;           // [n * top_k][patch][patch]
};

// One warp per keypoint: ori_conv at the integer keypoint only (mso_resnet_detector.py:144-148, l2-normalised), the kp_loc_size crop of
// max_heatmaps scaled by the keypoint's scale and its soft-argmax (inference.py:218-230), then the photo patch scaled and rotated about
// the refined keypoint (inference.py:259-260).  Rows past the image's keypoint count get zeros.
__global__ void __launch_bounds__(128) k_keypoints(KpArgs a, int n_rows) {
	const int g = blockIdx.x * 4 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
	if (g >= n_rows) return;
	const int f = g / a.top_k, j = g % a.top_k;
	const int PP = a.patch * a.patch;
	float* pt = a.patches + (size_t)g * PP;
	if (j >= a.n_kp[f]) {
		for (int i = lane; i < PP; i += 32) pt[i] = 0.f;
		if (lane == 0) { a.kpts_out[2 * (size_t)g] = 0.f; a.kpts_out[2 * (size_t)g + 1] = 0.f; a.ori[g] = make_float2(0.f, 0.f); }
		return;
	}
	const int2 k = a.kint[g];
	// orientation: 2 x (16 x 5 x 5) taps, lane-strided, then a fixed shuffle tree
	const float* fm = a.feat + (size_t)f * TC * HW;
	float o0 = 0.f, o1 = 0.f;
	for (int i = lane; i < TK * TK * TC; i += 32) {
		const int c = i % TC, kk = i / TC, ky = kk / TK, kx = kk % TK;
		const int yy = k.y + ky - TK / 2, xx = k.x + kx - TK / 2;
		if (yy < 0 || yy >= SIDE || xx < 0 || xx >= SIDE) continue;
		const float v = fm[(size_t)c * HW + yy * SIDE + xx];
		o0 = fmaf(v, a.ori_w[2 * i], o0); o1 = fmaf(v, a.ori_w[2 * i + 1], o1);
	}
	for (int o = 16; o > 0; o >>= 1) { o0 += __shfl_xor_sync(0xffffffffu, o0, o); o1 += __shfl_xor_sync(0xffffffffu, o1, o); }
	o0 += a.ori_b[0]; o1 += a.ori_b[1];
	const float inv = 1.0f / sqrtf(fmaxf(o0 * o0 + o1 * o1, 1e-12f));     // tf.nn.l2_normalize
	const float cs = o0 * inv, sn = o1 * inv;
	// refinement: the loc x loc crop (no rotation), softmax with kp_com_strength, soft-argmax on the [-1, 1] grid
	const float s = a.scl[(size_t)f * HW + k.y * SIDE + k.x];
	const float* hm = a.heat + (size_t)f * HW;
	const int LL = a.loc * a.loc;
	const float half = (float)a.loc / 2.0f;
	float vmax = -INFINITY;
	for (int i = lane; i < LL; i += 32) {
		const float xt = lin(i % a.loc, a.loc), yt = lin(i / a.loc, a.loc);
		vmax = fmaxf(vmax, st_sample(hm, s * xt * half + (float)k.x, s * yt * half + (float)k.y));
	}
	for (int o = 16; o > 0; o >>= 1) vmax = fmaxf(vmax, __shfl_xor_sync(0xffffffffu, vmax, o));
	float se = 0.f, sx = 0.f, sy = 0.f;
	for (int i = lane; i < LL; i += 32) {
		const float xt = lin(i % a.loc, a.loc), yt = lin(i / a.loc, a.loc);
		const float e = expf(a.kp_com * (st_sample(hm, s * xt * half + (float)k.x, s * yt * half + (float)k.y) - vmax));
		se += e; sx += xt * e; sy += yt * e;
	}
	for (int o = 16; o > 0; o >>= 1) {
		se += __shfl_xor_sync(0xffffffffu, se, o); sx += __shfl_xor_sync(0xffffffffu, sx, o); sy += __shfl_xor_sync(0xffffffffu, sy, o);
	}
	const float kx = (float)k.x + sx / (se + 1e-8f) * s * (float)a.loc / 2.0f;
	const float ky = (float)k.y + sy / (se + 1e-8f) * s * (float)a.loc / 2.0f;
	if (lane == 0) { a.kpts_out[2 * (size_t)g] = kx; a.kpts_out[2 * (size_t)g + 1] = ky; a.ori[g] = make_float2(cs, sn); }
	// the patch: theta = s * R(cos, sin), x = (theta00 xt + theta01 yt) * P / 2 + kx
	const float* gm = a.grey + (size_t)f * HW;
	const float t00 = s * cs, t01 = s * -sn, t10 = s * sn, t11 = s * cs, hp = (float)a.patch / 2.0f;
	for (int i = lane; i < PP; i += 32) {
		const float xt = lin(i % a.patch, a.patch), yt = lin(i / a.patch, a.patch);
		pt[i] = st_sample(gm, (t00 * xt + t01 * yt) * hp + kx, (t10 * xt + t11 * yt) * hp + ky);
	}
}

// ---- descriptor ----------------------------------------------------------------------------------------------------------------------
// simple_desc's layers as implicit GEMMs on NHWC activations: out[m][n] = act(s[n] * sum_k A[m][k] W[k][n] + t[n]), m = (row, oy, ox),
// k = (ky, kx, ci) in TF's weight order, A gathered from the input with SAME padding (pad_before, the rest after).  fc layers are the
// 1 x 1 case on the flattened (HWC, tf.layers.flatten) input.  64 x 64 output tiles, K in steps of 16, 4 x 4 outputs per thread.
struct Gemm {
	const float* in; const float* w; const float* s; const float* t; float* out;
	int M, Hin, Win, Cin, Hout, Wout, Cout, ks, stride, pad, relu;
};
constexpr int GB_M = 64, GB_N = 64, GB_K = 16;
__global__ void __launch_bounds__(256) k_gemm(Gemm g) {
	__shared__ __align__(16) float As[GB_K][GB_M + 4];
	__shared__ __align__(16) float Bs[GB_K][GB_N];
	const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
	const int m0 = blockIdx.x * GB_M, n0 = blockIdx.y * GB_N;
	const int K = g.ks * g.ks * g.Cin, HWo = g.Hout * g.Wout;
	float acc[4][4] = {};
	for (int k0 = 0; k0 < K; k0 += GB_K) {
#pragma unroll
		for (int i = 0; i < 4; i++) {
			const int e = tid + i * 256, kk = e % GB_K, ml = e / GB_K, m = m0 + ml, k = k0 + kk;
			float v = 0.f;
			if (m < g.M && k < K) {
				const int r = m / HWo, q = m % HWo, oy = q / g.Wout, ox = q % g.Wout;
				const int ky = k / (g.ks * g.Cin), rem = k % (g.ks * g.Cin), kx = rem / g.Cin, ci = rem % g.Cin;
				const int iy = oy * g.stride + ky - g.pad, ix = ox * g.stride + kx - g.pad;
				if (iy >= 0 && iy < g.Hin && ix >= 0 && ix < g.Win) v = g.in[(((size_t)r * g.Hin + iy) * g.Win + ix) * g.Cin + ci];
			}
			As[kk][ml] = v;
		}
#pragma unroll
		for (int i = 0; i < 4; i++) {
			const int e = tid + i * 256, kk = e / GB_N, nl = e % GB_N, k = k0 + kk, n = n0 + nl;
			Bs[kk][nl] = (k < K && n < g.Cout) ? g.w[(size_t)k * g.Cout + n] : 0.f;
		}
		__syncthreads();
#pragma unroll
		for (int kk = 0; kk < GB_K; kk++) {
			const float4 av = *reinterpret_cast<const float4*>(&As[kk][ty * 4]);
			const float4 bv = *reinterpret_cast<const float4*>(&Bs[kk][tx * 4]);
			const float ar[4] = {av.x, av.y, av.z, av.w}, br[4] = {bv.x, bv.y, bv.z, bv.w};
#pragma unroll
			for (int i = 0; i < 4; i++)
#pragma unroll
				for (int j = 0; j < 4; j++) acc[i][j] = fmaf(ar[i], br[j], acc[i][j]);
		}
		__syncthreads();
	}
#pragma unroll
	for (int i = 0; i < 4; i++) {
		const int m = m0 + ty * 4 + i;
		if (m >= g.M) continue;
#pragma unroll
		for (int j = 0; j < 4; j++) {
			const int n = n0 + tx * 4 + j;
			if (n >= g.Cout) continue;
			float v = g.s ? fmaf(acc[i][j], g.s[n], g.t[n]) : acc[i][j] + g.t[n];
			if (g.relu) v = fmaxf(v, 0.f);
			g.out[(size_t)m * g.Cout + n] = v;
		}
	}
}

// feat_norm = l2norm (simple_desc.py:55-56): one warp per row; rows past the image's keypoint count are zero.
__global__ void __launch_bounds__(128) k_l2norm(const float* __restrict__ raw, const int32_t* __restrict__ n_kp, int top_k, int D, int n_rows,
                                                float* __restrict__ out) {
	const int g = blockIdx.x * 4 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
	if (g >= n_rows) return;
	const bool live = (g % top_k) < n_kp[g / top_k];
	const float* r = raw + (size_t)g * D;
	float ss = 0.f;
	for (int i = lane; i < D; i += 32) ss = fmaf(r[i], r[i], ss);
	for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
	const float inv = 1.0f / sqrtf(fmaxf(ss, 1e-12f));
	for (int i = lane; i < D; i += 32) out[(size_t)g * D + i] = live ? r[i] * inv : 0.f;
}

// ---- weight blob ---------------------------------------------------------------------------------------------------------------------
struct DescLayer { int Hin, Cin, Hout, Cout, ks, pad; };
struct Layout {
	size_t init_w, init_b, fin_s, fin_t, ori_w, ori_b, fc2_w, fc2_b, total;
	size_t blk[MAX_BLOCKS][8];       // pre_s, pre_t, conv1_w, conv1_b, mid_s, mid_t, conv2_w, conv2_b
	size_t sc_w[MAX_SCALES], sc_b[MAX_SCALES];
	size_t dw[MAX_DESC + 1], ds[MAX_DESC + 1], dt[MAX_DESC + 1];   // desc conv layers, then fc1 at [depth]
	DescLayer dl[MAX_DESC];
	int feat_dim;                    // fc1's input: the flattened last conv output
};

Layout layout_of(const bt_lfnet_params& p) {
	Layout L = {};
	size_t o = 0;
	auto take = [&](size_t n) { const size_t r = o; o += n; return r; };
	const size_t kk = (size_t)p.conv_ksize * p.conv_ksize, C = (size_t)p.net_channel;
	L.init_w = take(kk * C); L.init_b = take(C);
	for (int b = 0; b < p.net_block; b++) {
		L.blk[b][0] = take(C); L.blk[b][1] = take(C); L.blk[b][2] = take(kk * C * C); L.blk[b][3] = take(C);
		L.blk[b][4] = take(C); L.blk[b][5] = take(C); L.blk[b][6] = take(kk * C * C); L.blk[b][7] = take(C);
	}
	L.fin_s = take(C); L.fin_t = take(C);
	for (int s = 0; s < p.net_num_scales; s++) { L.sc_w[s] = take(kk * C); L.sc_b[s] = take(1); }
	L.ori_w = take(kk * C * 2); L.ori_b = take(2);
	int h = p.patch_size, cin = 1;
	for (int l = 0; l < p.desc_net_depth; l++) {
		DescLayer& d = L.dl[l];
		d.Hin = h; d.Cin = cin; d.Cout = p.desc_net_channel << l; d.ks = p.desc_conv_ksize;
		d.Hout = (h + 1) / 2;                                           // TF SAME at stride 2: ceil(in / 2)
		const int pad_total = std::max((d.Hout - 1) * 2 + d.ks - h, 0);
		d.pad = pad_total / 2;                                          // the rest goes after: 32 wide, 3 x 3 -> 0 before, 1 after
		L.dw[l] = take((size_t)d.ks * d.ks * d.Cin * d.Cout); L.ds[l] = take(d.Cout); L.dt[l] = take(d.Cout);
		h = d.Hout; cin = d.Cout;
	}
	L.feat_dim = h * h * cin;
	L.dw[p.desc_net_depth] = take((size_t)L.feat_dim * FC_HIDDEN);
	L.ds[p.desc_net_depth] = take(FC_HIDDEN); L.dt[p.desc_net_depth] = take(FC_HIDDEN);
	L.fc2_w = take((size_t)FC_HIDDEN * p.desc_dim); L.fc2_b = take(p.desc_dim);
	L.total = o;
	return L;
}

constexpr int N_STAGES = 5;     // trunk, scales, detection, keypoints + patches, descriptor

}  // namespace

struct LfnetState {
	bt_lfnet_params p = {};
	bool ready = false;
	int max_images = 0;
	bool loaded = false;            // the weights in w are those of the network p
	Layout L = {};
	ScaleArgs sa = {};
	size_t logit_stride = 0;
	DevBuf w, grey, fa, fb, fc, logits, stats, Lm, Lmax, t1, t2, Es, heat, scl, nms, peak, kint, ori, patches, act, raw;
	TableBlock<> requests;          // the request pointers of a bt_lfnet_detect call
	bool timing = false;
	Event ev[N_STAGES + 1];
	bool timed = false;
};
void StateDeleter::operator()(LfnetState* s) const { delete s; }
struct RequestTable : TableLayout { Slice<const uint8_t*> req; };
static RequestTable request_table(size_t n) { RequestTable t; t.req = t.add<const uint8_t*>(n); return t; }

}  // namespace bt

using namespace bt;

extern "C" int bt_lfnet_weights_size(const bt_lfnet_params* p, size_t* n_floats) {
	BT_REQUIRE(p && n_floats, BT_ERR_INVALID_ARG, "bt_lfnet_weights_size: NULL argument");
	BT_REQUIRE(p->net_block >= 0 && p->net_block <= MAX_BLOCKS && p->net_num_scales >= 1 && p->net_num_scales <= MAX_SCALES &&
	           p->desc_net_depth >= 1 && p->desc_net_depth <= MAX_DESC && p->net_channel > 0 && p->conv_ksize > 0 && p->patch_size > 0 &&
	           p->desc_net_channel > 0 && p->desc_conv_ksize > 0 && p->desc_dim > 0, BT_ERR_INVALID_ARG, "bt_lfnet_weights_size: parameters out of range");
	*n_floats = layout_of(*p).total;
	return BT_OK;
}

// ---- the weights file (layout: include/bundletrack_b200.h): plain host code, no GPU --------------------------------------------------------
namespace {
constexpr char kFileMagic[8] = {'B', 'T', 'L', 'F', 'N', 'E', 'T', 'W'};
constexpr uint32_t kFileVersion = 1;
struct FileCloser { void operator()(FILE* f) const { fclose(f); } };
using File = std::unique_ptr<FILE, FileCloser>;

// Opens `path` and checks its header against this library and its size against the header; on success `f` stands at the first float.
// Refusals are BT_ERR_INVALID_ARG with a message that starts with `who` and names what differs.
int open_weights_file(const char* who, const char* path, File& f, bt_lfnet_params* p, size_t* n_floats) {
	BT_REQUIRE(path, BT_ERR_INVALID_ARG, "%s: path is NULL", who);
	f.reset(fopen(path, "rb"));
	BT_REQUIRE(f, BT_ERR_INVALID_ARG, "%s: %s: cannot open it: %s", who, path, strerror(errno));
	BT_REQUIRE(fseek(f.get(), 0, SEEK_END) == 0, BT_ERR_INVALID_ARG, "%s: %s: cannot seek in it", who, path);
	const long long size = ftell(f.get());
	BT_REQUIRE(size >= 0 && fseek(f.get(), 0, SEEK_SET) == 0, BT_ERR_INVALID_ARG, "%s: %s: cannot seek in it", who, path);
	const long long head = (long long)(sizeof kFileMagic + 2 * sizeof(uint32_t) + sizeof(bt_lfnet_params) + sizeof(uint64_t));
	char magic[sizeof kFileMagic];
	BT_REQUIRE(fread(magic, 1, sizeof magic, f.get()) == sizeof magic, BT_ERR_INVALID_ARG, "%s: %s: truncated: %lld bytes, the header takes %lld",
	           who, path, size, head);
	BT_REQUIRE(memcmp(magic, kFileMagic, sizeof magic) == 0, BT_ERR_INVALID_ARG, "%s: %s: bad magic: not an LF-Net weights file (lfnet.write_weights_file)",
	           who, path);
	uint32_t version = 0, params_bytes = 0;
	uint64_t count = 0;
	const bool whole = fread(&version, sizeof version, 1, f.get()) == 1 && fread(&params_bytes, sizeof params_bytes, 1, f.get()) == 1;
	BT_REQUIRE(!whole || version == kFileVersion, BT_ERR_INVALID_ARG, "%s: %s: format version %u, this library reads version %u", who, path, version,
	           kFileVersion);
	BT_REQUIRE(!whole || params_bytes == sizeof(bt_lfnet_params), BT_ERR_INVALID_ARG,
	           "%s: %s: a bt_lfnet_params struct size of %u bytes, this library's is %zu", who, path, params_bytes, sizeof(bt_lfnet_params));
	BT_REQUIRE(whole && fread(p, sizeof *p, 1, f.get()) == 1 && fread(&count, sizeof count, 1, f.get()) == 1, BT_ERR_INVALID_ARG,
	           "%s: %s: truncated: %lld bytes, the header takes %lld", who, path, size, head);
	size_t want = 0;
	BT_REQUIRE(bt_lfnet_weights_size(p, &want) == BT_OK, BT_ERR_INVALID_ARG, "%s: %s: its parameters are out of range", who, path);
	BT_REQUIRE(count == want, BT_ERR_INVALID_ARG, "%s: %s: a float count of %llu, bt_lfnet_weights_size gives %zu for its parameters", who, path,
	           (unsigned long long)count, want);
	const long long total = head + (long long)(sizeof(float) * want);
	BT_REQUIRE(size >= total, BT_ERR_INVALID_ARG, "%s: %s: truncated: %lld bytes, the header and %zu floats take %lld", who, path, size, want, total);
	BT_REQUIRE(size == total, BT_ERR_INVALID_ARG, "%s: %s: %lld bytes, %lld more than the header and %zu floats take", who, path, size, size - total, want);
	*n_floats = want;
	return BT_OK;
}
}  // namespace

extern "C" int bt_lfnet_file_info(const char* path, bt_lfnet_params* params_out, size_t* n_floats_out) {
	File f;
	bt_lfnet_params p;
	size_t n = 0;
	BT_TRY(open_weights_file("bt_lfnet_file_info", path, f, &p, &n));
	if (params_out) *params_out = p;
	if (n_floats_out) *n_floats_out = n;
	return BT_OK;
}

extern "C" int bt_lfnet_load_file(bt_ctx* ctx, const char* path, int max_images, bt_lfnet_params* params_out) {
	BT_REQUIRE(ctx, BT_ERR_INVALID_ARG, "bt_lfnet_load_file: ctx is NULL");
	File f;
	bt_lfnet_params p;
	size_t n = 0;
	BT_TRY(open_weights_file("bt_lfnet_load_file", path, f, &p, &n));
	std::vector<float> blob(n);
	BT_REQUIRE(fread(blob.data(), sizeof(float), n, f.get()) == n, BT_ERR_INVALID_ARG, "bt_lfnet_load_file: %s: reading the floats failed", path);
	f.reset();
	BT_TRY(bt_lfnet_reserve(ctx, &p, max_images));
	BT_TRY(bt_lfnet_load_weights(ctx, blob.data(), n));
	if (params_out) *params_out = p;
	return BT_OK;
}

#define LF_FIELD(cond, name, fmt, val) BT_REQUIRE(cond, BT_ERR_INVALID_ARG, "bt_lfnet_reserve: " name " = " fmt " is not supported here", val)

extern "C" int bt_lfnet_reserve(bt_ctx* ctx, const bt_lfnet_params* p, int max_images) {
	BT_REQUIRE(ctx, BT_ERR_INVALID_ARG, "bt_lfnet_reserve: ctx is NULL");
	BT_REQUIRE(p, BT_ERR_INVALID_ARG, "bt_lfnet_reserve: params is NULL");
	BT_REQUIRE(max_images >= 1 && max_images <= 65535, BT_ERR_INVALID_ARG, "bt_lfnet_reserve: max_images %d outside [1, 65535]", max_images);
	LF_FIELD(p->net_channel == TC, "net_channel", "%d", p->net_channel);
	LF_FIELD(p->conv_ksize == TK, "conv_ksize", "%d", p->conv_ksize);
	LF_FIELD(p->net_block >= 0 && p->net_block <= MAX_BLOCKS, "net_block", "%d", p->net_block);
	LF_FIELD(p->net_num_scales >= 1 && p->net_num_scales <= MAX_SCALES, "net_num_scales", "%d", p->net_num_scales);
	LF_FIELD(p->net_min_scale > 0 && p->net_max_scale >= p->net_min_scale && isfinite(p->net_max_scale), "net_min_scale / net_max_scale", "%g", p->net_min_scale);
	LF_FIELD(p->top_k >= 1 && p->top_k <= HW, "top_k", "%d", p->top_k);
	LF_FIELD(p->sm_ksize >= 1 && p->sm_ksize % 2 == 1 && p->sm_ksize <= SIDE, "sm_ksize", "%d", p->sm_ksize);
	LF_FIELD(p->nms_ksize >= 3 && p->nms_ksize % 2 == 1 && p->nms_ksize <= 31, "nms_ksize", "%d", p->nms_ksize);
	LF_FIELD(p->kp_loc_size >= 2 && p->kp_loc_size <= 64, "kp_loc_size", "%d", p->kp_loc_size);
	LF_FIELD(p->crop_radius >= 0 && 2 * p->crop_radius < SIDE, "crop_radius", "%d", p->crop_radius);
	LF_FIELD(p->patch_size >= 2 && p->patch_size <= 128, "patch_size", "%d", p->patch_size);
	LF_FIELD(p->desc_net_depth >= 1 && p->desc_net_depth <= MAX_DESC, "desc_net_depth", "%d", p->desc_net_depth);
	LF_FIELD(p->desc_net_channel >= 1 && (p->desc_net_channel << (p->desc_net_depth - 1)) <= 4096, "desc_net_channel", "%d", p->desc_net_channel);
	LF_FIELD(p->desc_conv_ksize >= 1 && p->desc_conv_ksize <= 7, "desc_conv_ksize", "%d", p->desc_conv_ksize);
	LF_FIELD(p->desc_dim >= 32 && p->desc_dim % 32 == 0 && p->desc_dim <= 4096, "desc_dim", "%d", p->desc_dim);
	LF_FIELD(isfinite(p->leaky_alpha) && isfinite(p->com_strength) && isfinite(p->score_com_strength) && isfinite(p->scale_com_strength) &&
	         isfinite(p->kp_com_strength) && isfinite(p->nms_thresh), "a strength, alpha or threshold", "%s", "non-finite");
	// scale_factors = exp(linspace(log(max), log(min), n)) in float64 (mso_resnet_detector.py:106-110), numpy's linspace (start + i step,
	// the last element set to stop); sizes int(float32(400) * float32(1 / s) + 0.5) (mso_resnet_detector.py:130-132)
	ScaleArgs a = {};
	a.n_scales = p->net_num_scales;
	size_t off = 0;
	for (int i = 0; i < a.n_scales; i++) {
		double lg;
		if (a.n_scales == 1) lg = 0.0;
		else if (i == a.n_scales - 1) lg = log(p->net_min_scale);
		else lg = log(p->net_max_scale) + i * ((log(p->net_min_scale) - log(p->net_max_scale)) / (a.n_scales - 1));
		const double sf = a.n_scales == 1 ? 1.0 : exp(lg);
		a.factor[i] = (float)sf;
		const float inv = (float)(1.0 / sf);
		a.size[i] = (int)((float)SIDE * inv + 0.5f);
		LF_FIELD(a.size[i] >= 1 && a.size[i] <= 4 * SIDE, "net_min_scale", "%g", p->net_min_scale);
		a.logit_off[i] = off;
		off += (size_t)a.size[i] * a.size[i];
	}
	LfnetState* s;
	BT_TRY(take_state(ctx, &bt_ctx::lfnet, &s));
	s->loaded = s->loaded && memcmp(&s->p, p, sizeof *p) == 0;      // (the same network keeps its weights: w is not reallocated)
	const Layout L = layout_of(*p);
	const size_t n = (size_t)max_images, rows = n * p->top_k, ns = (size_t)a.n_scales;
	size_t act = 0;
	for (int l = 0; l < p->desc_net_depth; l++) act = std::max(act, (size_t)L.dl[l].Hout * L.dl[l].Hout * L.dl[l].Cout);
	BT_TRY(s->w.alloc(sizeof(float) * L.total));
	BT_TRY(s->requests.reserve(request_table(n).total));
	BT_TRY(s->grey.alloc(sizeof(float) * n * HW));
	for (DevBuf* b : {&s->fa, &s->fb, &s->fc}) BT_TRY(b->alloc(sizeof(float) * n * TC * HW));
	BT_TRY(s->logits.alloc(sizeof(float) * n * off));
	BT_TRY(s->stats.alloc(sizeof(float2) * n * ns));
	BT_TRY(s->Lm.alloc(sizeof(float) * n * ns * HW));
	for (DevBuf* b : {&s->Lmax, &s->t1, &s->t2, &s->Es, &s->heat, &s->scl, &s->nms}) BT_TRY(b->alloc(sizeof(float) * n * HW));
	BT_TRY(s->peak.alloc(n * HW));
	BT_TRY(s->kint.alloc(sizeof(int2) * rows));
	BT_TRY(s->ori.alloc(sizeof(float2) * rows));
	BT_TRY(s->patches.alloc(sizeof(float) * rows * p->patch_size * p->patch_size));
	// two activation blocks, ping-pong: the widest conv output, fc1 and fc2
	const size_t per_row = std::max(std::max(act, (size_t)FC_HIDDEN), (size_t)p->desc_dim);
	BT_TRY(s->act.alloc(sizeof(float) * rows * per_row));
	BT_TRY(s->raw.alloc(sizeof(float) * rows * per_row));
	s->p = *p; s->L = L; s->sa = a; s->logit_stride = off;
	s->max_images = max_images;
	s->ready = true;
	return BT_OK;
}

extern "C" int bt_lfnet_load_weights(bt_ctx* ctx, const float* blob, size_t n_floats) {
	LfnetState* s;
	BT_TRY(state_of(ctx, &bt_ctx::lfnet, "bt_lfnet_load_weights", "bt_lfnet_reserve", &s));
	BT_REQUIRE(blob, BT_ERR_INVALID_ARG, "bt_lfnet_load_weights: blob is NULL");
	BT_REQUIRE(n_floats == s->L.total, BT_ERR_INVALID_ARG, "bt_lfnet_load_weights: %zu floats, the network of these parameters has %zu", n_floats, s->L.total);
	for (size_t i = 0; i < n_floats; i++)
		BT_REQUIRE(isfinite(blob[i]), BT_ERR_INVALID_ARG, "bt_lfnet_load_weights: float %zu is not finite", i);
	BT_CUDA(cudaMemcpy(s->w.p, blob, sizeof(float) * n_floats, cudaMemcpyHostToDevice));
	s->loaded = true;
	return BT_OK;
}

extern "C" int bt_lfnet_detect(bt_ctx* ctx, int n, const uint8_t* const* request_dev, float* kpts_out, float* desc_out, int32_t* n_out, void* stream_) {
	LfnetState* s;
	BT_TRY(state_of(ctx, &bt_ctx::lfnet, "bt_lfnet_detect", "bt_lfnet_reserve", &s));
	BT_REQUIRE(s->loaded, BT_ERR_INVALID_ARG, "bt_lfnet_detect: call bt_lfnet_load_weights first");
	BT_REQUIRE(n >= 1 && request_dev && kpts_out && desc_out && n_out, BT_ERR_INVALID_ARG, "bt_lfnet_detect: n %d < 1 or a NULL pointer", n);
	for (int i = 0; i < n; i++) BT_REQUIRE(request_dev[i], BT_ERR_INVALID_ARG, "bt_lfnet_detect: request %d is NULL", i);
	BT_REQUIRE(n <= s->max_images, BT_ERR_CAPACITY, "bt_lfnet_detect: %d images > the reserved %d", n, s->max_images);
	cudaStream_t st = (cudaStream_t)stream_;
	const bt_lfnet_params& p = s->p;
	const Layout& L = s->L;
	const float* W = s->w.as<float>();
	const float alpha = p.leaky_alpha;
	const size_t N = (size_t)n;
	const int rows = n * p.top_k;
	if (s->timing) for (auto& e : s->ev) BT_TRY(e.create(true));
	auto mark = [&](int i) -> int { if (s->timing) BT_CUDA(cudaEventRecord(s->ev[i], st)); return BT_OK; };
	BT_TRY(mark(0));
	// request pointers
	const RequestTable rt = request_table(N);
	BT_TRY(s->requests.begin("bt_lfnet_detect", rt));
	memcpy(s->requests.host(rt.req), request_dev, sizeof(void*) * N);
	BT_TRY(s->requests.send(0, rt.req.end(), st));
	BT_TRY(s->requests.in_flight(st));
	const dim3 gp((HW + 255) / 256, n);
	k_grey<<<gp, 256, 0, st>>>(s->requests.dev(rt.req), s->grey.as<float>());
	// trunk: init conv, then per block x -> t = conv1(act(bn_pre x)) -> x' = conv2(act(bn_mid t)) + x, then act(bn_fin x)
	const dim3 gc((SIDE + CT_W - 1) / CT_W, (SIDE + CT_H - 1) / CT_H, n);
	float *x = s->fa.as<float>(), *t = s->fb.as<float>(), *y = s->fc.as<float>();
	k_trunk_conv<1><<<gc, 256, 0, st>>>(s->grey.as<float>(), W + L.init_w, W + L.init_b, nullptr, nullptr, alpha, nullptr, x);
	for (int b = 0; b < p.net_block; b++) {
		const size_t* o = L.blk[b];
		k_trunk_conv<TC><<<gc, 256, 0, st>>>(x, W + o[2], W + o[3], W + o[0], W + o[1], alpha, nullptr, t);
		k_trunk_conv<TC><<<gc, 256, 0, st>>>(t, W + o[6], W + o[7], W + o[4], W + o[5], alpha, x, y);
		std::swap(x, y);
	}
	float* feat = t;
	k_bn_act<<<(unsigned)((N * TC * HW + 255) / 256), 256, 0, st>>>(x, W + L.fin_s, W + L.fin_t, alpha, feat, n);
	BT_CUDA(cudaGetLastError());
	BT_TRY(mark(1));
	// per scale: resize + score conv, instance-norm moments
	ScaleArgs a = s->sa;
	int smax = 0;
	for (int i = 0; i < a.n_scales; i++) { a.w[i] = W + L.sc_w[i]; a.b[i] = W + L.sc_b[i]; smax = std::max(smax, a.size[i]); }
	k_score_conv<<<dim3((smax + 31) / 32, (smax + 7) / 8, n * a.n_scales), 256, 0, st>>>(feat, a, s->logits.as<float>(), s->logit_stride);
	k_moments<<<n * a.n_scales, MOM_THREADS, 0, st>>>(s->logits.as<float>(), a, s->logit_stride, s->stats.as<float2>());
	BT_CUDA(cudaGetLastError());
	BT_TRY(mark(2));
	// detection: soft 3-D NMS, soft scale, masks, NMS, top-k
	const int r = p.sm_ksize / 2;
	k_upsample<<<gp, 256, 0, st>>>(s->logits.as<float>(), s->stats.as<float2>(), a, s->logit_stride, s->Lm.as<float>(), s->Lmax.as<float>());
	k_box<<<gp, 256, 0, st>>>(s->Lmax.as<float>(), s->t1.as<float>(), r, 0, 0);
	k_box<<<gp, 256, 0, st>>>(s->t1.as<float>(), s->t2.as<float>(), r, 1, 0);
	k_exp<<<gp, 256, 0, st>>>(s->Lm.as<float>(), s->t2.as<float>(), s->Es.as<float>(), a.n_scales, p.com_strength);
	k_box<<<gp, 256, 0, st>>>(s->Es.as<float>(), s->t1.as<float>(), r, 0, 1);
	k_box<<<gp, 256, 0, st>>>(s->t1.as<float>(), s->t2.as<float>(), r, 1, 1);
	// end_of_frame_masks' pad radius: pad_size = num_conv * (conv_ksize // 2), num_conv counting the init conv, two per block and the
	// score conv (mso_resnet_detector.py:85,96,139,171): 8 x 2 = 16 at the defaults
	const int pad = (2 + 2 * p.net_block) * (p.conv_ksize / 2);
	k_soft_scale<<<gp, 256, 0, st>>>(s->Lm.as<float>(), s->t2.as<float>(), a, p.score_com_strength, p.scale_com_strength, pad, s->heat.as<float>(), s->scl.as<float>());
	k_nms<<<gp, 256, 0, st>>>(s->heat.as<float>(), p.nms_thresh, p.nms_ksize / 2, p.crop_radius, s->nms.as<float>(), s->peak.as<uint8_t>());
	k_topk<<<n, TOPK_THREADS, 0, st>>>(s->nms.as<float>(), s->peak.as<uint8_t>(), p.top_k, s->kint.as<int2>(), n_out);
	BT_CUDA(cudaGetLastError());
	BT_TRY(mark(3));
	// keypoints: orientation, refinement, patches
	KpArgs ka;
	ka.heat = s->heat.as<float>(); ka.scl = s->scl.as<float>(); ka.feat = feat; ka.grey = s->grey.as<float>();
	ka.kint = s->kint.as<int2>(); ka.n_kp = n_out; ka.ori_w = W + L.ori_w; ka.ori_b = W + L.ori_b;
	ka.top_k = p.top_k; ka.loc = p.kp_loc_size; ka.patch = p.patch_size; ka.kp_com = p.kp_com_strength;
	ka.kpts_out = kpts_out; ka.ori = s->ori.as<float2>(); ka.patches = s->patches.as<float>();
	k_keypoints<<<(rows + 3) / 4, 128, 0, st>>>(ka, rows);
	BT_CUDA(cudaGetLastError());
	BT_TRY(mark(4));
	// descriptor
	const float* in = s->patches.as<float>();
	float* bufs[2] = {s->act.as<float>(), s->raw.as<float>()};
	int cur = 0;
	auto gemm = [&](Gemm g) -> int {
		k_gemm<<<dim3((unsigned)((g.M + GB_M - 1) / GB_M), (unsigned)((g.Cout + GB_N - 1) / GB_N)), 256, 0, st>>>(g);
		BT_CUDA(cudaGetLastError());
		return BT_OK;
	};
	for (int l = 0; l < p.desc_net_depth; l++) {
		const DescLayer& d = L.dl[l];
		Gemm g = {in, W + L.dw[l], W + L.ds[l], W + L.dt[l], bufs[cur], rows * d.Hout * d.Hout, d.Hin, d.Hin, d.Cin, d.Hout, d.Hout, d.Cout, d.ks, 2, d.pad, 1};
		BT_TRY(gemm(g));
		in = bufs[cur]; cur ^= 1;
	}
	const int dd = p.desc_net_depth;
	BT_TRY(gemm(Gemm{in, W + L.dw[dd], W + L.ds[dd], W + L.dt[dd], bufs[cur], rows, 1, 1, L.feat_dim, 1, 1, FC_HIDDEN, 1, 1, 0, 1}));
	in = bufs[cur]; cur ^= 1;
	BT_TRY(gemm(Gemm{in, W + L.fc2_w, nullptr, W + L.fc2_b, bufs[cur], rows, 1, 1, FC_HIDDEN, 1, 1, p.desc_dim, 1, 1, 0, 0}));
	k_l2norm<<<(rows + 3) / 4, 128, 0, st>>>(bufs[cur], n_out, p.top_k, p.desc_dim, rows, desc_out);
	BT_CUDA(cudaGetLastError());
	BT_TRY(mark(5));
	s->timed = s->timing;
	return BT_OK;
}

extern "C" int bt_lfnet_enable_timing(bt_ctx* ctx, int on) {
	LfnetState* s;
	BT_TRY(state_of(ctx, &bt_ctx::lfnet, "bt_lfnet_enable_timing", "bt_lfnet_reserve", &s));
	s->timing = on != 0;
	return BT_OK;
}

extern "C" int bt_lfnet_get_timing(bt_ctx* ctx, float* ms5) {
	LfnetState* s;
	BT_TRY(state_of(ctx, &bt_ctx::lfnet, "bt_lfnet_get_timing", "bt_lfnet_reserve", &s));
	BT_REQUIRE(s->timed && ms5, BT_ERR_INVALID_ARG, "bt_lfnet_get_timing: no timed call (bt_lfnet_enable_timing) or ms5 is NULL");
	BT_CUDA(cudaEventSynchronize(s->ev[N_STAGES]));
	for (int i = 0; i < N_STAGES; i++) BT_CUDA(cudaEventElapsedTime(ms5 + i, s->ev[i], s->ev[i + 1]));
	return BT_OK;
}

extern "C" int bt_lfnet_debug_maps(bt_ctx* ctx, int image, float* heat_host, float* scale_host, int32_t* kpts_int_host, float* ori_host, void* stream) {
	LfnetState* s;
	BT_TRY(state_of(ctx, &bt_ctx::lfnet, "bt_lfnet_debug_maps", "bt_lfnet_reserve", &s));
	BT_REQUIRE(s->loaded, BT_ERR_INVALID_ARG, "bt_lfnet_debug_maps: call bt_lfnet_load_weights first");
	BT_REQUIRE(image >= 0 && image < s->max_images, BT_ERR_INVALID_ARG, "bt_lfnet_debug_maps: image %d outside [0, %d)", image, s->max_images);
	cudaStream_t st = (cudaStream_t)stream;
	const size_t k = (size_t)s->p.top_k, f = (size_t)image;
	if (heat_host) BT_CUDA(cudaMemcpyAsync(heat_host, s->heat.as<float>() + f * HW, sizeof(float) * HW, cudaMemcpyDeviceToHost, st));
	if (scale_host) BT_CUDA(cudaMemcpyAsync(scale_host, s->scl.as<float>() + f * HW, sizeof(float) * HW, cudaMemcpyDeviceToHost, st));
	if (kpts_int_host) BT_CUDA(cudaMemcpyAsync(kpts_int_host, s->kint.as<int2>() + f * k, sizeof(int2) * k, cudaMemcpyDeviceToHost, st));
	if (ori_host) BT_CUDA(cudaMemcpyAsync(ori_host, s->ori.as<float2>() + f * k, sizeof(float2) * k, cudaMemcpyDeviceToHost, st));
	BT_CUDA(cudaStreamSynchronize(st));
	return BT_OK;
}
