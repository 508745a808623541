// vos.cu — transductive video object segmentation on the device (transductive-vos.pytorch's run_video.py at its defaults, resnet50):
// a ResNet-50 feature network to stride 8 and label propagation from a ring of earlier frames.  DESIGN.md §3.13, §9.14.
//
//   k_vos_stem       7 x 7 / 2 conv of the normalised RGB (read from BGR bytes) + BN + ReLU, FP32, 64 output channels per thread
//   k_vos_pool       3 x 3 / 2 max pool, padding 1
//   k_vos_conv       implicit-GEMM convolution (NHWC, weights [co][ky][kx][ci]) on the 3xTF32 tensor-core mainloop, with the folded BN,
//                    an optional residual and ReLU in the epilogue: every 1 x 1, 3 x 3, shortcut and adjust_dim conv
//   k_vos_propagate  fused propagation, flash-attention style: a CTA owns 64 target pixels and one selected reference frame, computes
//                    S = ref . target on the same mainloop (K = 256) key tile by key tile, and keeps per target pixel the running maximum,
//                    the unweighted exponential sum and one spatially weighted numerator per label.  S is never stored.
//   k_vos_merge      combines the per-reference partial softmax states into the low-resolution prediction, and writes the one-hot of its
//                    argmax into the history ring
//   k_vos_mask       bilinear upsample of the prediction to full resolution, argmax, one output byte per channel: 0 / 255 for the mask,
//                    the initial mask's values for the label map
//
// 3xTF32: each FP32 operand x is split into hi = tf32(x) and lo = tf32(x - hi); a product is accumulated as lo.hi + hi.lo + hi.hi in
// FP32 (the lo.lo term is below FP32's rounding).  The MMA is the warp-level mma.sync.m16n8k8.tf32.
#include "bt_common.cuh"

#include <algorithm>
#include <cmath>
#include <vector>

namespace bt {
namespace {

constexpr int FEAT = 256;               // the feature dimension (bn256)
constexpr int MAX_LABELS = 8;           // label channels the kernels carry (channel 0 included)
constexpr int MAX_REFS = 64;            // ref_num's upper bound (the per-call reference table)

// ---- the 3xTF32 mainloop pieces ---------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t tf32(float x) {
	uint32_t r;
	asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
	return r;
}
__device__ __forceinline__ void split(float x, uint32_t& hi, uint32_t& lo) {
	hi = tf32(x);
	lo = tf32(x - __uint_as_float(hi));
}
__device__ __forceinline__ void mma_tf32(float (&d)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
	asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
	             : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
	             : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}
// One k8 step of a warp tile MT x NT of m16n8 blocks.  A is row-major [m][k] and B is [n][k] in shared memory (pitch P floats, P = 4 mod 32
// so the fragment reads are conflict-free); a0 / b0 point at the warp's first row and the step's first k.
template <int MT, int NT, int P>
__device__ __forceinline__ void mma_step_3x(float (&acc)[MT][NT][4], const float* a0, const float* b0) {
	const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
	uint32_t ah[MT][4], al[MT][4], bh[NT][2], bl[NT][2];
#pragma unroll
	for (int i = 0; i < MT; i++) {
		const float* a = a0 + (i * 16 + g) * P + t;
		split(a[0], ah[i][0], al[i][0]);
		split(a[8 * P], ah[i][1], al[i][1]);
		split(a[4], ah[i][2], al[i][2]);
		split(a[8 * P + 4], ah[i][3], al[i][3]);
	}
#pragma unroll
	for (int j = 0; j < NT; j++) {
		const float* b = b0 + (j * 8 + g) * P + t;
		split(b[0], bh[j][0], bl[j][0]);
		split(b[4], bh[j][1], bl[j][1]);
	}
#pragma unroll
	for (int i = 0; i < MT; i++)
#pragma unroll
		for (int j = 0; j < NT; j++) {
			mma_tf32(acc[i][j], al[i], bh[j]);
			mma_tf32(acc[i][j], ah[i], bl[j]);
			mma_tf32(acc[i][j], ah[i], bh[j]);
		}
}

// A KT-deep slice of the product, accumulated by the tensor cores into a zeroed tile and then added to `sum` on the FP32 pipe.  The
// tensor cores' FP32 accumulation truncates where an FADD rounds to nearest, so a running accumulator that took every MMA of the whole K
// (up to 864 of them in a 3 x 3 conv) drifts by a bias; promoting every 32-deep slice keeps the results FP32-grade (DESIGN.md §9.14).
template <int MT, int NT, int P, int KT>
__device__ __forceinline__ void mma_slice_3x(float (&sum)[MT][NT][4], const float* a0, const float* b0) {
	float acc[MT][NT][4];
#pragma unroll
	for (int i = 0; i < MT; i++)
#pragma unroll
		for (int j = 0; j < NT; j++)
#pragma unroll
			for (int e = 0; e < 4; e++) acc[i][j][e] = 0.f;
#pragma unroll
	for (int kk = 0; kk < KT; kk += 8) mma_step_3x<MT, NT, P>(acc, a0 + kk, b0 + kk);
#pragma unroll
	for (int i = 0; i < MT; i++)
#pragma unroll
		for (int j = 0; j < NT; j++)
#pragma unroll
			for (int e = 0; e < 4; e++) sum[i][j][e] = __fadd_rn(sum[i][j][e], acc[i][j][e]);
}

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
// 16-byte cp.async; src_bytes 0 fills the destination with zeros (padding and rows past the end)
__device__ __forceinline__ void cp16(void* dst, const void* src, int src_bytes) {
	asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(dst)), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// ---- stem: normalise while loading, 7 x 7 / 2 conv, BN, ReLU ---------------------------------------------------------------------------
constexpr int STEM_K = 7 * 7 * 3;
// ToTensor then Normalize in float32: (v / 255 - mean) / std, RGB order, read from BGR bytes
__constant__ float c_mean[3] = {0.485f, 0.456f, 0.406f};
__constant__ float c_std[3] = {0.229f, 0.224f, 0.225f};

__global__ void __launch_bounds__(128) k_vos_stem(const uint8_t* __restrict__ bgr, int H, int W, const float* __restrict__ w,
                                                  const float* __restrict__ scale, const float* __restrict__ shift, float* __restrict__ out,
                                                  int Ho, int Wo) {
	__shared__ float sw[STEM_K][64];       // [ky][kx][c] x co: every thread reads the same tap, a broadcast
	for (int i = threadIdx.x; i < STEM_K * 64; i += blockDim.x) {
		const int co = i / STEM_K, k = i % STEM_K;
		sw[k][co] = w[i];
	}
	__syncthreads();
	const int p = blockIdx.x * blockDim.x + threadIdx.x;
	if (p >= Ho * Wo) return;
	const int oy = p / Wo, ox = p % Wo;
	float acc[64];
#pragma unroll
	for (int c = 0; c < 64; c++) acc[c] = 0.f;
	for (int ky = 0; ky < 7; ky++) {
		const int iy = oy * 2 - 3 + ky;
		if (iy < 0 || iy >= H) continue;
		for (int kx = 0; kx < 7; kx++) {
			const int ix = ox * 2 - 3 + kx;
			if (ix < 0 || ix >= W) continue;
			const uint8_t* px = bgr + ((size_t)iy * W + ix) * 3;
#pragma unroll
			for (int c = 0; c < 3; c++) {
				const float v = __fdiv_rn(__fsub_rn(__fdiv_rn((float)px[2 - c], 255.f), c_mean[c]), c_std[c]);
				const float* wk = sw[(ky * 7 + kx) * 3 + c];
#pragma unroll
				for (int co = 0; co < 64; co++) acc[co] = fmaf(v, wk[co], acc[co]);
			}
		}
	}
	float4* o = reinterpret_cast<float4*>(out + (size_t)p * 64);
#pragma unroll
	for (int c = 0; c < 64; c += 4) {
		float4 r;
		r.x = fmaxf(fmaf(acc[c], scale[c], shift[c]), 0.f);
		r.y = fmaxf(fmaf(acc[c + 1], scale[c + 1], shift[c + 1]), 0.f);
		r.z = fmaxf(fmaf(acc[c + 2], scale[c + 2], shift[c + 2]), 0.f);
		r.w = fmaxf(fmaf(acc[c + 3], scale[c + 3], shift[c + 3]), 0.f);
		o[c / 4] = r;
	}
}

__global__ void k_vos_pool(const float* __restrict__ in, int H, int W, int C, float* __restrict__ out, int Ho, int Wo) {
	const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= (size_t)Ho * Wo * C) return;
	const int c = (int)(i % C), p = (int)(i / C), oy = p / Wo, ox = p % Wo;
	float m = -INFINITY;
	for (int dy = 0; dy < 3; dy++) {
		const int iy = oy * 2 - 1 + dy;
		if (iy < 0 || iy >= H) continue;
		for (int dx = 0; dx < 3; dx++) {
			const int ix = ox * 2 - 1 + dx;
			if (ix >= 0 && ix < W) m = fmaxf(m, in[((size_t)iy * W + ix) * C + c]);
		}
	}
	out[i] = m;
}

// ---- implicit-GEMM convolution ----------------------------------------------------------------------------------------------------------
constexpr int CB_M = 128, CB_N = 64, CB_K = 32, CB_P = CB_K + 4, CB_THREADS = 128;   // 4 warps, 2 x 2, warp tile 64 x 32
constexpr int CB_STAGE = (CB_M + CB_N) * CB_P;                                           // floats per pipeline stage
constexpr size_t CB_SMEM = 2 * CB_STAGE * sizeof(float);

struct ConvArgs {
	const float* in; int H, W, Cin;
	const float* w; const float* scale; const float* shift;
	const float* res;                    // residual [M][Cout] or nullptr
	float* out; int Ho, Wo, Cout;
	int ks, stride, pad, relu;
};

__global__ void __launch_bounds__(CB_THREADS) k_vos_conv(const ConvArgs a) {
	extern __shared__ __align__(16) float smem[];
	const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
	const int M = a.Ho * a.Wo, K = a.ks * a.ks * a.Cin;
	const int m0 = blockIdx.x * CB_M, n0 = blockIdx.y * CB_N;
	// this thread's A rows (tid / 8 + 16 i) and 16-byte chunk (tid % 8), fixed over the K loop
	const int chunk = tid & 7;
	int row_y[8], row_x[8];
#pragma unroll
	for (int i = 0; i < 8; i++) {
		const int m = m0 + (tid >> 3) + 16 * i;
		row_y[i] = m < M ? (m / a.Wo) * a.stride - a.pad : -(1 << 20);
		row_x[i] = m < M ? (m % a.Wo) * a.stride - a.pad : -(1 << 20);
	}
	auto load = [&](int kt, int stage) {
		float* As = smem + stage * CB_STAGE;
		float* Bs = As + CB_M * CB_P;
		const int k0 = kt * CB_K, tap = k0 / a.Cin, ci = k0 % a.Cin + chunk * 4;
		const int ky = tap / a.ks, kx = tap % a.ks;
#pragma unroll
		for (int i = 0; i < 8; i++) {
			const int r = (tid >> 3) + 16 * i, iy = row_y[i] + ky, ix = row_x[i] + kx;
			const bool ok = iy >= 0 && iy < a.H && ix >= 0 && ix < a.W;
			const float* src = ok ? a.in + ((size_t)iy * a.W + ix) * a.Cin + ci : a.in;
			cp16(As + r * CB_P + chunk * 4, src, ok ? 16 : 0);
		}
#pragma unroll
		for (int i = 0; i < 4; i++) {
			const int r = (tid >> 3) + 16 * i;
			cp16(Bs + r * CB_P + chunk * 4, a.w + (size_t)(n0 + r) * K + k0 + chunk * 4, 16);
		}
		cp_commit();
	};
	float acc[4][4][4];
#pragma unroll
	for (int i = 0; i < 4; i++)
#pragma unroll
		for (int j = 0; j < 4; j++)
#pragma unroll
			for (int e = 0; e < 4; e++) acc[i][j][e] = 0.f;
	const int wm = (warp >> 1) * 64, wn = (warp & 1) * 32;
	const int n_kt = K / CB_K;
	load(0, 0);
	for (int kt = 0; kt < n_kt; kt++) {
		if (kt + 1 < n_kt) { load(kt + 1, (kt + 1) & 1); cp_wait<1>(); }
		else cp_wait<0>();
		__syncthreads();
		const float* As = smem + (kt & 1) * CB_STAGE;
		const float* Bs = As + CB_M * CB_P;
		mma_slice_3x<4, 4, CB_P, CB_K>(acc, As + wm * CB_P, Bs + wn * CB_P);
		__syncthreads();
	}
	// epilogue: thread holds rows g, g + 8 and columns 2t, 2t + 1 of each m16n8 block
	const int g = lane >> 2, t = lane & 3;
#pragma unroll
	for (int j = 0; j < 4; j++) {
		const int n = n0 + wn + j * 8 + 2 * t;
		const float s0 = a.scale[n], s1 = a.scale[n + 1], h0 = a.shift[n], h1 = a.shift[n + 1];
#pragma unroll
		for (int i = 0; i < 4; i++)
#pragma unroll
			for (int hh = 0; hh < 2; hh++) {
				const int m = m0 + wm + i * 16 + g + 8 * hh;
				if (m >= M) continue;
				float2 v = make_float2(fmaf(acc[i][j][2 * hh], s0, h0), fmaf(acc[i][j][2 * hh + 1], s1, h1));
				const size_t o = (size_t)m * a.Cout + n;
				if (a.res) { const float2 r = *reinterpret_cast<const float2*>(a.res + o); v.x += r.x; v.y += r.y; }
				if (a.relu) { v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); }
				*reinterpret_cast<float2*>(a.out + o) = v;
			}
	}
}

// ---- propagation ------------------------------------------------------------------------------------------------------------------------
constexpr int PB_T = 64, PB_R = 32, PB_P = FEAT + 4, PB_THREADS = 128;     // 64 targets (4 warps x 16 rows), 32-key tiles
constexpr size_t PB_SMEM = sizeof(float) * ((size_t)PB_T * PB_P + 2 * (size_t)PB_R * PB_P + 2 * (size_t)PB_R * MAX_LABELS);

struct PropArgs {
	const float* feat;                   // ring [slots][HW][FEAT]
	const float* label;                  // ring [slots][HW][MAX_LABELS]
	int target_slot, Hd, Wd;
	float temperature;
	int slot[MAX_REFS];
	float sig2[MAX_REFS];                // sigma^2 of each selected reference, float32
	float* part;                         // [n_ref][HW][2 + MAX_LABELS]: max, exp sum, numerators
};

__global__ void __launch_bounds__(PB_THREADS) k_vos_propagate(const PropArgs a) {
	extern __shared__ __align__(16) float smem[];
	float* Qs = smem;
	float* Ks = Qs + PB_T * PB_P;                 // two stages of PB_R x PB_P
	float* Ls = Ks + 2 * PB_R * PB_P;             // two stages of PB_R x MAX_LABELS
	const int HW = a.Hd * a.Wd, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
	const int t0 = blockIdx.x * PB_T, j = blockIdx.y;
	const float* tf = a.feat + (size_t)a.target_slot * HW * FEAT;
	const float* rf = a.feat + (size_t)a.slot[j] * HW * FEAT;
	const float* rl = a.label + (size_t)a.slot[j] * HW * MAX_LABELS;
	for (int i = tid; i < PB_T * (FEAT / 4); i += PB_THREADS) {
		const int r = i / (FEAT / 4), c = i % (FEAT / 4);
		const bool ok = t0 + r < HW;
		cp16(Qs + r * PB_P + c * 4, ok ? tf + (size_t)(t0 + r) * FEAT + c * 4 : tf, ok ? 16 : 0);
	}
	auto load = [&](int kt, int stage) {
		const int r0 = kt * PB_R;
		float* K = Ks + stage * PB_R * PB_P;
		for (int i = tid; i < PB_R * (FEAT / 4); i += PB_THREADS) {
			const int r = i / (FEAT / 4), c = i % (FEAT / 4);
			const bool ok = r0 + r < HW;
			cp16(K + r * PB_P + c * 4, ok ? rf + (size_t)(r0 + r) * FEAT + c * 4 : rf, ok ? 16 : 0);
		}
		float* L = Ls + stage * PB_R * MAX_LABELS;
		for (int i = tid; i < PB_R * MAX_LABELS / 4; i += PB_THREADS) {
			const bool ok = r0 + i / 2 < HW;
			cp16(L + i * 4, ok ? rl + (size_t)r0 * MAX_LABELS + i * 4 : rl, ok ? 16 : 0);
		}
		cp_commit();
	};
	// per thread: rows g and g + 8 of the warp's 16 targets; m is the row's running max (equal across the quad), l and num partial sums
	// over this thread's columns, folded across the quad at the end
	const int ty[2] = {(t0 + warp * 16 + g) / a.Wd, (t0 + warp * 16 + g + 8) / a.Wd};
	const int tx[2] = {(t0 + warp * 16 + g) % a.Wd, (t0 + warp * 16 + g + 8) % a.Wd};
	float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f}, num[2][MAX_LABELS];
#pragma unroll
	for (int h = 0; h < 2; h++)
#pragma unroll
		for (int c = 0; c < MAX_LABELS; c++) num[h][c] = 0.f;
	const float nsig = -1.f;
	const float sig2 = a.sig2[j];
	const int n_kt = (HW + PB_R - 1) / PB_R;
	load(0, 0);
	for (int kt = 0; kt < n_kt; kt++) {
		if (kt + 1 < n_kt) { load(kt + 1, (kt + 1) & 1); cp_wait<1>(); }
		else cp_wait<0>();
		__syncthreads();
		const float* K = Ks + (kt & 1) * PB_R * PB_P;
		const float* L = Ls + (kt & 1) * PB_R * MAX_LABELS;
		float s[1][4][4];
#pragma unroll
		for (int jj = 0; jj < 4; jj++)
#pragma unroll
			for (int e = 0; e < 4; e++) s[0][jj][e] = 0.f;
#pragma unroll 2
		for (int kk = 0; kk < FEAT; kk += 32) mma_slice_3x<1, 4, PB_P, 32>(s, Qs + warp * 16 * PB_P + kk, K + kk);
		// s[0][jj][2 h + e]: target row g + 8 h, key column kt * PB_R + jj * 8 + 2 t + e
		const int r0 = kt * PB_R;
#pragma unroll
		for (int h = 0; h < 2; h++) {
			float mx = -INFINITY;
#pragma unroll
			for (int jj = 0; jj < 4; jj++)
#pragma unroll
				for (int e = 0; e < 2; e++) {
					const int r = r0 + jj * 8 + 2 * t + e;
					const float v = __fmul_rn(s[0][jj][2 * h + e], a.temperature);
					s[0][jj][2 * h + e] = v;
					if (r < HW) mx = fmaxf(mx, v);
				}
			mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
			mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
			const float mn = fmaxf(m[h], mx);
			const float corr = expf(m[h] - mn);       // m = -inf on the first tile: exp(-inf) = 0 scales the empty sums
			m[h] = mn;
			l[h] *= corr;
#pragma unroll
			for (int c = 0; c < MAX_LABELS; c++) num[h][c] *= corr;
#pragma unroll
			for (int jj = 0; jj < 4; jj++)
#pragma unroll
				for (int e = 0; e < 2; e++) {
					const int rc = jj * 8 + 2 * t + e, r = r0 + rc;
					if (r >= HW) continue;
					const float p = expf(s[0][jj][2 * h + e] - mn);
					const int dy = r / a.Wd - ty[h], dx = r % a.Wd - tx[h];
					const float w = expf(__fdiv_rn(nsig * (float)(dy * dy + dx * dx), sig2));
					const float pw = p * w;
					l[h] += p;
					const float4 la = *reinterpret_cast<const float4*>(L + rc * MAX_LABELS);
					const float4 lb = *reinterpret_cast<const float4*>(L + rc * MAX_LABELS + 4);
					num[h][0] = fmaf(la.x, pw, num[h][0]); num[h][1] = fmaf(la.y, pw, num[h][1]);
					num[h][2] = fmaf(la.z, pw, num[h][2]); num[h][3] = fmaf(la.w, pw, num[h][3]);
					num[h][4] = fmaf(lb.x, pw, num[h][4]); num[h][5] = fmaf(lb.y, pw, num[h][5]);
					num[h][6] = fmaf(lb.z, pw, num[h][6]); num[h][7] = fmaf(lb.w, pw, num[h][7]);
				}
		}
		__syncthreads();
	}
#pragma unroll
	for (int h = 0; h < 2; h++) {
#pragma unroll
		for (int o = 1; o <= 2; o <<= 1) {
			l[h] += __shfl_xor_sync(0xffffffffu, l[h], o);
#pragma unroll
			for (int c = 0; c < MAX_LABELS; c++) num[h][c] += __shfl_xor_sync(0xffffffffu, num[h][c], o);
		}
		const int tp = t0 + warp * 16 + g + 8 * h;
		if (t == 0 && tp < HW) {
			float* o = a.part + ((size_t)j * HW + tp) * (2 + MAX_LABELS);
			o[0] = m[h]; o[1] = l[h];
#pragma unroll
			for (int c = 0; c < MAX_LABELS; c++) o[2 + c] = num[h][c];
		}
	}
}

// the references' partial states -> pred [MAX_LABELS][HW]; its argmax (first channel wins ties) as a one-hot into the ring
__global__ void k_vos_merge(const float* __restrict__ part, int n_ref, int HW, int d, float* __restrict__ pred, float* __restrict__ label_out) {
	const int tp = blockIdx.x * blockDim.x + threadIdx.x;
	if (tp >= HW) return;
	float M = -INFINITY;
	for (int j = 0; j < n_ref; j++) M = fmaxf(M, part[((size_t)j * HW + tp) * (2 + MAX_LABELS)]);
	float l = 0.f, num[MAX_LABELS] = {};
	for (int j = 0; j < n_ref; j++) {
		const float* p = part + ((size_t)j * HW + tp) * (2 + MAX_LABELS);
		const float f = expf(p[0] - M);
		l = fmaf(p[1], f, l);
#pragma unroll
		for (int c = 0; c < MAX_LABELS; c++) num[c] = fmaf(p[2 + c], f, num[c]);
	}
	int best = 0;
	float bv = 0.f;
#pragma unroll
	for (int c = 0; c < MAX_LABELS; c++) {
		const float v = c < d ? num[c] / l : 0.f;
		pred[(size_t)c * HW + tp] = v;
		if (c < d && (c == 0 || v > bv)) { bv = v; best = c; }
	}
	float* lo = label_out + (size_t)tp * MAX_LABELS;
#pragma unroll
	for (int c = 0; c < MAX_LABELS; c++) lo[c] = c == best ? 1.f : 0.f;
}

// PyTorch's bilinear source index, align_corners = False: src = max((dst + 0.5) scale - 0.5, 0), scale = in / out in float
__device__ __forceinline__ void lin_src(int dst, float scale, int in, int& i0, int& i1, float& l0, float& l1) {
	const float s = fmaxf((dst + 0.5f) * scale - 0.5f, 0.f);
	i0 = (int)s;
	i1 = i0 + (i0 < in - 1 ? 1 : 0);
	l1 = s - (float)i0;
	l0 = 1.f - l1;
}

// the byte k_vos_mask writes for each label channel
struct ChanBytes { uint8_t v[MAX_LABELS]; };
constexpr ChanBytes kMaskBytes = {{0, 255, 255, 255, 255, 255, 255, 255}};

__global__ void k_vos_mask(const float* __restrict__ pred, int Hd, int Wd, int d, ChanBytes out, uint8_t* __restrict__ mask, int H, int W) {
	const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
	if (x >= W) return;
	int y0, y1, x0, x1;
	float ly0, ly1, lx0, lx1;
	lin_src(y, (float)Hd / (float)H, Hd, y0, y1, ly0, ly1);
	lin_src(x, (float)Wd / (float)W, Wd, x0, x1, lx0, lx1);
	const int HW = Hd * Wd;
	int best = 0;
	float bv = 0.f;
	for (int c = 0; c < d; c++) {
		const float* p = pred + (size_t)c * HW;
		const float v = ly0 * (lx0 * p[y0 * Wd + x0] + lx1 * p[y0 * Wd + x1]) + ly1 * (lx0 * p[y1 * Wd + x0] + lx1 * p[y1 * Wd + x1]);
		if (c == 0 || v > bv) { bv = v; best = c; }
	}
	mask[(size_t)y * W + x] = out.v[best];
}

// frame 0: which of the 256 values the initial mask holds
__global__ void k_vos_values(const uint8_t* __restrict__ m, int n, int32_t* __restrict__ present) {
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i < n) present[m[i]] = 1;
}

// frame 0's history label: the one-hot of the compressed initial mask, bilinearly resized to (Hd, Wd); its output mask: > 0 -> 255
__global__ void k_vos_init_label(const uint8_t* __restrict__ m, int H, int W, const int32_t* __restrict__ chan, float* __restrict__ label,
                                 int Hd, int Wd) {
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= Hd * Wd) return;
	int y0, y1, x0, x1;
	float ly0, ly1, lx0, lx1;
	lin_src(i / Wd, (float)H / (float)Hd, H, y0, y1, ly0, ly1);
	lin_src(i % Wd, (float)W / (float)Wd, W, x0, x1, lx0, lx1);
	const int c00 = chan[m[y0 * W + x0]], c01 = chan[m[y0 * W + x1]], c10 = chan[m[y1 * W + x0]], c11 = chan[m[y1 * W + x1]];
	float* o = label + (size_t)i * MAX_LABELS;
#pragma unroll
	for (int c = 0; c < MAX_LABELS; c++)
		o[c] = ly0 * (lx0 * (float)(c00 == c) + lx1 * (float)(c01 == c)) + ly1 * (lx0 * (float)(c10 == c) + lx1 * (float)(c11 == c));
}

__global__ void k_vos_binarise(const uint8_t* __restrict__ m, int n, uint8_t* __restrict__ out) {
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i < n) out[i] = m[i] > 0 ? 255 : 0;
}

// ---- the network's layout -----------------------------------------------------------------------------------------------------------
struct ConvW { size_t w, s, t; int cin, cout, ks, stride; };
struct Bottleneck { ConvW c1, c2, c3, down; bool has_down; };
constexpr int N_BLOCKS = 3 + 4 + 6 + 3;
struct Net { ConvW stem; Bottleneck b[N_BLOCKS]; ConvW adjust; size_t total; };

Net net_layout() {
	Net n = {};
	size_t o = 0;
	auto conv = [&](int cin, int cout, int ks, int stride) {
		ConvW c;
		c.cin = cin; c.cout = cout; c.ks = ks; c.stride = stride;
		c.w = o; o += (size_t)cout * ks * ks * cin;
		c.s = o; o += cout;
		c.t = o; o += cout;
		return c;
	};
	n.stem = conv(3, 64, 7, 2);
	const int blocks[4] = {3, 4, 6, 3}, planes[4] = {64, 128, 256, 256}, strides[4] = {1, 2, 1, 1};
	int inp = 64, bi = 0;
	for (int L = 0; L < 4; L++)
		for (int k = 0; k < blocks[L]; k++) {
			Bottleneck& b = n.b[bi++];
			const int s = k == 0 ? strides[L] : 1, p = planes[L];
			b.c1 = conv(inp, p, 1, 1);
			b.c2 = conv(p, p, 3, s);
			b.c3 = conv(p, 4 * p, 1, 1);
			b.has_down = k == 0 && (s != 1 || inp != 4 * p);
			if (b.has_down) b.down = conv(inp, 4 * p, 1, s);
			inp = 4 * p;
		}
	n.adjust = conv(1024, FEAT, 1, 1);
	n.total = o;
	return n;
}

constexpr int N_STAGES = 3;     // backbone, propagation, mask

}  // namespace

struct VosState {
	bt_vos_params p = {};
	int H = 0, W = 0, Hd = 0, Wd = 0, slots = 0;
	bool ready = false;
	bool loaded = false;
	int frame = -1;                 // frames seen since bt_vos_begin; -1 before it
	int n_labels = 0;
	ChanBytes values = {};          // label channel -> the initial mask's value
	Net net = {};
	DevBuf w, act[5], feat, label, part, pred, chan, init;       // init: the initial mask, bt_vos_labels' output for frame 0
	PinnedBuf present;
	bool timing = false;
	Event ev[N_STAGES + 1];
	bool timed = false;
};
void StateDeleter::operator()(VosState* s) const { delete s; }

}  // namespace bt

using namespace bt;

namespace {

int conv_out(int in, int ks, int stride) { return (in + 2 * (ks / 2) - ks) / stride + 1; }

int launch_conv(const float* W, const ConvW& c, const float* in, int H, int Wd, const float* res, bool relu, float* out, int& Ho, int& Wo,
                cudaStream_t st) {
	Ho = conv_out(H, c.ks, c.stride); Wo = conv_out(Wd, c.ks, c.stride);
	ConvArgs a = {in, H, Wd, c.cin, W + c.w, W + c.s, W + c.t, res, out, Ho, Wo, c.cout, c.ks, c.stride, c.ks / 2, relu ? 1 : 0};
	const dim3 grid((unsigned)((Ho * Wo + CB_M - 1) / CB_M), (unsigned)(c.cout / CB_N));
	k_vos_conv<<<grid, CB_THREADS, CB_SMEM, st>>>(a);
	BT_CUDA(cudaGetLastError());
	return BT_OK;
}

// the backbone of one frame into ring slot `slot`
int run_backbone(VosState* s, const uint8_t* colour, int slot, cudaStream_t st) {
	const float* W = s->w.as<float>();
	const Net& n = s->net;
	float* b[5];
	for (int i = 0; i < 5; i++) b[i] = s->act[i].as<float>();
	const int H1 = conv_out(s->H, 7, 2), W1 = conv_out(s->W, 7, 2);
	k_vos_stem<<<(H1 * W1 + 127) / 128, 128, 0, st>>>(colour, s->H, s->W, W + n.stem.w, W + n.stem.s, W + n.stem.t, b[0], H1, W1);
	int H = conv_out(H1, 3, 2), Wd = conv_out(W1, 3, 2);
	k_vos_pool<<<(unsigned)(((size_t)H * Wd * 64 + 255) / 256), 256, 0, st>>>(b[0], H1, W1, 64, b[1], H, Wd);
	BT_CUDA(cudaGetLastError());
	float *x = b[1], *t1 = b[2], *t2 = b[3], *sc = b[4], *y = b[0];
	for (int i = 0; i < N_BLOCKS; i++) {
		const Bottleneck& k = n.b[i];
		int h1, w1, h2, w2, h3, w3;
		BT_TRY(launch_conv(W, k.c1, x, H, Wd, nullptr, true, t1, h1, w1, st));
		BT_TRY(launch_conv(W, k.c2, t1, h1, w1, nullptr, true, t2, h2, w2, st));
		const float* res = x;
		if (k.has_down) { int hs, ws; BT_TRY(launch_conv(W, k.down, x, H, Wd, nullptr, false, sc, hs, ws, st)); res = sc; }
		BT_TRY(launch_conv(W, k.c3, t2, h2, w2, res, true, y, h3, w3, st));
		std::swap(x, y);
		H = h3; Wd = w3;
	}
	int ho, wo;
	return launch_conv(W, n.adjust, x, H, Wd, nullptr, false, s->feat.as<float>() + (size_t)slot * s->Hd * s->Wd * FEAT, ho, wo, st);
}

}  // namespace

// run_video.py's sample_frames: frames 0..k-1 up to ref_num, then numpy's linspace(ref_start, ref_end, ref_num - 3) truncated to int
// (start + i * step in double, the last sample set to stop) and the three frames before k
extern "C" int bt_vos_schedule(int k, int ref_num, int range, int32_t* idx_out, int* n_out) {
	BT_REQUIRE(idx_out && n_out, BT_ERR_INVALID_ARG, "bt_vos_schedule: NULL argument");
	BT_REQUIRE(k >= 1 && ref_num >= 5 && ref_num <= MAX_REFS && range >= 0, BT_ERR_INVALID_ARG,
	           "bt_vos_schedule: k %d < 1, ref_num %d outside [5, %d] or range %d < 0", k, ref_num, MAX_REFS, range);
	if (k <= ref_num) {
		for (int i = 0; i < k; i++) idx_out[i] = i;
		*n_out = k;
		return BT_OK;
	}
	const int dense = 3, sparse = ref_num - dense, end = k - dense - 1, start = std::max(end - range, 0);
	const double step = (double)(end - start) / (double)(sparse - 1);
	for (int i = 0; i < sparse; i++) idx_out[i] = i == sparse - 1 ? end : (int)(i * step + (double)start);
	for (int i = 0; i < dense; i++) idx_out[sparse + i] = k - dense + i;
	*n_out = ref_num;
	return BT_OK;
}

extern "C" int bt_vos_weights_size(const bt_vos_params* p, size_t* n_floats) {
	BT_REQUIRE(p && n_floats, BT_ERR_INVALID_ARG, "bt_vos_weights_size: NULL argument");
	*n_floats = net_layout().total;
	return BT_OK;
}

extern "C" int bt_vos_reserve(bt_ctx* ctx, const bt_vos_params* p, int H, int W) {
	BT_REQUIRE(ctx && p, BT_ERR_INVALID_ARG, "bt_vos_reserve: NULL argument");
	BT_REQUIRE(p->ref_num >= 5 && p->ref_num <= MAX_REFS, BT_ERR_INVALID_ARG, "bt_vos_reserve: ref_num %d outside [5, %d]", p->ref_num, MAX_REFS);
	BT_REQUIRE(p->range >= 0 && p->range <= 10000, BT_ERR_INVALID_ARG, "bt_vos_reserve: range %d outside [0, 10000]", p->range);
	BT_REQUIRE(p->sigma1 > 0 && p->sigma2 > 0 && std::isfinite(p->sigma1) && std::isfinite(p->sigma2) && std::isfinite(p->temperature),
	           BT_ERR_INVALID_ARG, "bt_vos_reserve: sigma1 %g, sigma2 %g must be finite and positive, temperature %g finite", p->sigma1, p->sigma2,
	           p->temperature);
	BT_REQUIRE(H >= 8 && W >= 8 && H <= 4096 && W <= 4096, BT_ERR_INVALID_ARG, "bt_vos_reserve: size %d x %d outside [8, 4096]", H, W);
	VosState* s;
	BT_TRY(take_state(ctx, &bt_ctx::vos, &s));
	const int Hd = (H + 7) / 8, Wd = (W + 7) / 8, slots = std::max(p->range + 5, p->ref_num + 1);
	const Net net = net_layout();
	const size_t HW = (size_t)Hd * Wd;
	const int H1 = conv_out(H, 7, 2), W1 = conv_out(W, 7, 2), H2 = conv_out(H1, 3, 2), W2 = conv_out(W1, 3, 2);
	const size_t act = std::max({(size_t)H1 * W1 * 64, (size_t)H2 * W2 * 256, HW * 1024});
	BT_TRY(s->w.alloc(sizeof(float) * net.total));
	for (DevBuf& b : s->act) BT_TRY(b.alloc(sizeof(float) * act));
	BT_TRY(s->feat.alloc(sizeof(float) * slots * HW * FEAT));
	BT_TRY(s->label.alloc(sizeof(float) * slots * HW * MAX_LABELS));
	BT_TRY(s->part.alloc(sizeof(float) * p->ref_num * HW * (2 + MAX_LABELS)));
	BT_TRY(s->pred.alloc(sizeof(float) * MAX_LABELS * HW));
	BT_TRY(s->chan.alloc(sizeof(int32_t) * 512));
	BT_TRY(s->init.alloc((size_t)H * W));
	BT_TRY(s->present.alloc(sizeof(int32_t) * 256));
	BT_CUDA(cudaFuncSetAttribute(k_vos_conv, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)CB_SMEM));
	BT_CUDA(cudaFuncSetAttribute(k_vos_propagate, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)PB_SMEM));
	s->p = *p;
	s->H = H; s->W = W; s->Hd = Hd; s->Wd = Wd; s->slots = slots;
	s->net = net;
	s->frame = -1;
	s->ready = true;
	return BT_OK;
}

extern "C" int bt_vos_load_weights(bt_ctx* ctx, const float* blob, size_t n_floats) {
	VosState* s;
	BT_TRY(state_of(ctx, &bt_ctx::vos, "bt_vos_load_weights", "bt_vos_reserve", &s));
	BT_REQUIRE(blob, BT_ERR_INVALID_ARG, "bt_vos_load_weights: blob is NULL");
	BT_REQUIRE(n_floats == s->net.total, BT_ERR_INVALID_ARG, "bt_vos_load_weights: %zu floats, the network has %zu", n_floats, s->net.total);
	for (size_t i = 0; i < n_floats; i++) BT_REQUIRE(std::isfinite(blob[i]), BT_ERR_INVALID_ARG, "bt_vos_load_weights: float %zu is not finite", i);
	BT_CUDA(cudaMemcpy(s->w.p, blob, sizeof(float) * n_floats, cudaMemcpyHostToDevice));
	s->loaded = true;
	return BT_OK;
}

extern "C" int bt_vos_begin(bt_ctx* ctx, const uint8_t* colour_dev, const uint8_t* init_mask_dev, uint8_t* mask_out_dev, void* stream_) {
	VosState* s;
	BT_TRY(state_of(ctx, &bt_ctx::vos, "bt_vos_begin", "bt_vos_reserve", &s));
	BT_REQUIRE(s->loaded, BT_ERR_INVALID_ARG, "bt_vos_begin: call bt_vos_load_weights first");
	BT_REQUIRE(colour_dev && init_mask_dev && mask_out_dev, BT_ERR_INVALID_ARG, "bt_vos_begin: NULL pointer");
	cudaStream_t st = (cudaStream_t)stream_;
	const int n = s->H * s->W, HW = s->Hd * s->Wd;
	// the mask's distinct values, read back once: value 0 -> channel 0 (kept when absent), the others in increasing order
	int32_t* present = s->present.as<int32_t>();
	BT_CUDA(cudaMemsetAsync(s->chan.p, 0, sizeof(int32_t) * 256, st));
	k_vos_values<<<(n + 255) / 256, 256, 0, st>>>(init_mask_dev, n, s->chan.as<int32_t>());
	BT_CUDA(cudaGetLastError());
	BT_CUDA(cudaMemcpyAsync(present, s->chan.p, sizeof(int32_t) * 256, cudaMemcpyDeviceToHost, st));
	BT_CUDA(cudaStreamSynchronize(st));
	int distinct = 0, d = 1;
	for (int v = 0; v < 256; v++) distinct += present[v] != 0;
	int32_t* chan = present;        // rewritten in place as the value -> channel map
	ChanBytes values = {};
	for (int v = 0; v < 256; v++) {
		if (v > 0 && present[v] && d < MAX_LABELS) values.v[d] = (uint8_t)v;
		chan[v] = v == 0 ? 0 : (present[v] ? d++ : 0);
	}
	BT_REQUIRE(d <= MAX_LABELS, BT_ERR_INVALID_ARG, "bt_vos_begin: the initial mask has %d distinct values (%d label channels with channel 0); at most %d channels are supported",
	           distinct, d, MAX_LABELS);
	BT_CUDA(cudaMemcpyAsync(s->chan.as<int32_t>() + 256, chan, sizeof(int32_t) * 256, cudaMemcpyHostToDevice, st));
	if (s->timing) for (auto& e : s->ev) BT_TRY(e.create(true));
	auto mark = [&](int i) -> int { if (s->timing) BT_CUDA(cudaEventRecord(s->ev[i], st)); return BT_OK; };
	BT_TRY(mark(0));
	BT_TRY(run_backbone(s, colour_dev, 0, st));
	BT_TRY(mark(1));
	BT_TRY(mark(2));
	k_vos_init_label<<<(HW + 127) / 128, 128, 0, st>>>(init_mask_dev, s->H, s->W, s->chan.as<int32_t>() + 256, s->label.as<float>(), s->Hd, s->Wd);
	k_vos_binarise<<<(n + 255) / 256, 256, 0, st>>>(init_mask_dev, n, mask_out_dev);
	BT_CUDA(cudaGetLastError());
	BT_TRY(mark(3));
	BT_CUDA(cudaMemcpyAsync(s->init.p, init_mask_dev, (size_t)n, cudaMemcpyDeviceToDevice, st));
	// the chan upload reads the pinned block: wait for it before a later begin rewrites it
	BT_CUDA(cudaStreamSynchronize(st));
	s->n_labels = d;
	s->values = values;
	s->frame = 0;
	s->timed = s->timing;
	return BT_OK;
}

extern "C" int bt_vos_next(bt_ctx* ctx, const uint8_t* colour_dev, uint8_t* mask_out_dev, void* stream_) {
	VosState* s;
	BT_TRY(state_of(ctx, &bt_ctx::vos, "bt_vos_next", "bt_vos_reserve", &s));
	BT_REQUIRE(s->loaded, BT_ERR_INVALID_ARG, "bt_vos_next: call bt_vos_load_weights first");
	BT_REQUIRE(s->frame >= 0, BT_ERR_INVALID_ARG, "bt_vos_next: no sequence begun (bt_vos_begin)");
	BT_REQUIRE(colour_dev && mask_out_dev, BT_ERR_INVALID_ARG, "bt_vos_next: NULL pointer");
	BT_REQUIRE(s->frame < (1 << 30), BT_ERR_CAPACITY, "bt_vos_next: sequence too long");
	cudaStream_t st = (cudaStream_t)stream_;
	const int k = s->frame + 1, HW = s->Hd * s->Wd, slot = k % s->slots;
	PropArgs a = {};
	int32_t idx[MAX_REFS];
	int n_ref = 0;
	BT_TRY(bt_vos_schedule(k, s->p.ref_num, s->p.range, idx, &n_ref));
	const float sig1 = (float)(s->p.sigma1 * s->p.sigma1), sig2 = (float)(s->p.sigma2 * s->p.sigma2);
	for (int j = 0; j < n_ref; j++) {
		a.slot[j] = idx[j] % s->slots;
		a.sig2[j] = (k > 15 && j < n_ref - 4) ? sig2 : sig1;
	}
	a.feat = s->feat.as<float>(); a.label = s->label.as<float>();
	a.target_slot = slot; a.Hd = s->Hd; a.Wd = s->Wd;
	a.temperature = (float)s->p.temperature;
	a.part = s->part.as<float>();
	if (s->timing) for (auto& e : s->ev) BT_TRY(e.create(true));
	auto mark = [&](int i) -> int { if (s->timing) BT_CUDA(cudaEventRecord(s->ev[i], st)); return BT_OK; };
	BT_TRY(mark(0));
	BT_TRY(run_backbone(s, colour_dev, slot, st));
	BT_TRY(mark(1));
	k_vos_propagate<<<dim3((unsigned)((HW + PB_T - 1) / PB_T), (unsigned)n_ref), PB_THREADS, PB_SMEM, st>>>(a);
	k_vos_merge<<<(HW + 127) / 128, 128, 0, st>>>(s->part.as<float>(), n_ref, HW, s->n_labels, s->pred.as<float>(),
	                                               s->label.as<float>() + (size_t)slot * HW * MAX_LABELS);
	BT_CUDA(cudaGetLastError());
	BT_TRY(mark(2));
	k_vos_mask<<<dim3((s->W + 127) / 128, s->H), 128, 0, st>>>(s->pred.as<float>(), s->Hd, s->Wd, s->n_labels, kMaskBytes, mask_out_dev, s->H, s->W);
	BT_CUDA(cudaGetLastError());
	BT_TRY(mark(3));
	s->frame = k;
	s->timed = s->timing;
	return BT_OK;
}

extern "C" int bt_vos_labels(bt_ctx* ctx, uint8_t* labels_out_dev, void* stream_) {
	VosState* s;
	BT_TRY(state_of(ctx, &bt_ctx::vos, "bt_vos_labels", "bt_vos_reserve", &s));
	BT_REQUIRE(s->frame >= 0, BT_ERR_INVALID_ARG, "bt_vos_labels: no sequence begun (bt_vos_begin)");
	BT_REQUIRE(labels_out_dev, BT_ERR_INVALID_ARG, "bt_vos_labels: NULL pointer");
	cudaStream_t st = (cudaStream_t)stream_;
	if (s->frame == 0) {
		BT_CUDA(cudaMemcpyAsync(labels_out_dev, s->init.p, (size_t)s->H * s->W, cudaMemcpyDeviceToDevice, st));
		return BT_OK;
	}
	// the same upsample and argmax as bt_vos_next's mask, with each channel's value in place of 255
	k_vos_mask<<<dim3((s->W + 127) / 128, s->H), 128, 0, st>>>(s->pred.as<float>(), s->Hd, s->Wd, s->n_labels, s->values, labels_out_dev, s->H, s->W);
	BT_CUDA(cudaGetLastError());
	return BT_OK;
}

extern "C" int bt_vos_enable_timing(bt_ctx* ctx, int on) {
	VosState* s;
	BT_TRY(state_of(ctx, &bt_ctx::vos, "bt_vos_enable_timing", "bt_vos_reserve", &s));
	s->timing = on != 0;
	return BT_OK;
}

extern "C" int bt_vos_get_timing(bt_ctx* ctx, float* ms3) {
	VosState* s;
	BT_TRY(state_of(ctx, &bt_ctx::vos, "bt_vos_get_timing", "bt_vos_reserve", &s));
	BT_REQUIRE(ms3, BT_ERR_INVALID_ARG, "bt_vos_get_timing: NULL argument");
	BT_REQUIRE(s->timed, BT_ERR_INVALID_ARG, "bt_vos_get_timing: no timed call (bt_vos_enable_timing)");
	BT_CUDA(cudaEventSynchronize(s->ev[N_STAGES]));
	for (int i = 0; i < N_STAGES; i++) BT_CUDA(cudaEventElapsedTime(ms3 + i, s->ev[i], s->ev[i + 1]));
	return BT_OK;
}

extern "C" int bt_vos_debug(bt_ctx* ctx, int slot, float* feat_host, float* label_host, float* pred_host, int32_t* info5, void* stream) {
	VosState* s;
	BT_TRY(state_of(ctx, &bt_ctx::vos, "bt_vos_debug", "bt_vos_reserve", &s));
	BT_REQUIRE(s->loaded, BT_ERR_INVALID_ARG, "bt_vos_debug: call bt_vos_load_weights first");
	BT_REQUIRE(slot >= 0 && slot < s->slots, BT_ERR_INVALID_ARG, "bt_vos_debug: slot %d outside [0, %d)", slot, s->slots);
	cudaStream_t st = (cudaStream_t)stream;
	const size_t HW = (size_t)s->Hd * s->Wd;
	if (feat_host) BT_CUDA(cudaMemcpyAsync(feat_host, s->feat.as<float>() + slot * HW * FEAT, sizeof(float) * HW * FEAT, cudaMemcpyDeviceToHost, st));
	if (label_host) BT_CUDA(cudaMemcpyAsync(label_host, s->label.as<float>() + slot * HW * MAX_LABELS, sizeof(float) * HW * MAX_LABELS, cudaMemcpyDeviceToHost, st));
	if (pred_host) BT_CUDA(cudaMemcpyAsync(pred_host, s->pred.p, sizeof(float) * HW * MAX_LABELS, cudaMemcpyDeviceToHost, st));
	BT_CUDA(cudaStreamSynchronize(st));
	if (info5) { info5[0] = s->frame; info5[1] = s->n_labels; info5[2] = s->slots; info5[3] = s->Hd; info5[4] = s->Wd; }
	return BT_OK;
}
