// metrics.cu — pose accuracy on the device: ADD and ADD-S per frame (the reference's scripts/Utils.py add / adi) and the host-side
// VOCap area under the accuracy curve (scripts/eval_ycbineoat.py), as BundleTrack's YCBInEOAT table reports them.
//
// ADD(f)   = mean_i |gt_f p_i - pred_f p_i|
// ADD-S(f) = mean_i min_j |gt_f p_i - pred_f p_j|          (exact nearest neighbour; the reference uses a cKDTree per frame)
//
// ADD-S is a brute-force scan over the model, tiled through shared memory, in two precisions (DESIGN.md §3.7):
//  - filter, fp32: the query gt p_i is moved into the model frame, q_i = pred^-1 gt p_i, so every frame compares against the SAME
//    untransformed model, converted to fp32 once per call.  For a rigid pred |q_i - p_j| = |gt p_i - pred p_j|; for a pred whose rotation
//    block A is only nearly orthonormal (10-digit text, float32 tracker poses) |q_i - p_j| = |A^-1 w_ij| with w_ij = gt p_i - pred p_j,
//    which lies within the singular values of A^-1 of |w_ij|.  Their ratio kappa bounds how far the filter's order can differ from the
//    true one.
//  - rerank, fp64: a candidate whose fp32 squared distance is within the threshold T(m) of the running fp32 minimum m is evaluated as
//    |gt p_i - pred p_j| in float64, the reference's expression.  T covers the fp32 rounding of q, p and the distance, and kappa, so the
//    true nearest neighbour is always reranked; the result is the float64 minimum over all candidates.
// ADD is the same block's queries against themselves, so one kernel gives both; each block writes one partial sum per metric and a
// second kernel adds a frame's partials in chunk order: the result depends on n_pts only, not on the grid or the number of frames.
#include <math.h>
#include <stddef.h>
#include <algorithm>
#include <vector>
#include "bt_common.cuh"

namespace bt {

namespace {

constexpr int kThreads = 256;
constexpr int kQpt = 4;                            // queries per thread: one shared-memory load serves four distance tests
constexpr int kChunk = kThreads * kQpt;            // queries per block
constexpr int kTile = 1024;                        // model points per shared-memory tile (16 KB of float4)
constexpr double kU = 1.0 / 16777216.0;            // fp32 unit roundoff 2^-24
constexpr double kGamma = 8.0 * kU;                // relative error of the fp32 squared distance of two rounded points (5 roundings, with slack)

// one frame's constants, row-major 3 x 4 (the last row of a pose is not read)
struct FrameConst {
	double pred[12], gt[12];
	double M[12];          // pred^-1 gt: the query's transform into the model frame
	double kappa;          // ratio of the singular values of pred's rotation block (INFINITY: every candidate is reranked)
	double a_abs;          // float64 slack of q, absolute (metres)
};
constexpr int kFrameDoubles = sizeof(FrameConst) / sizeof(double);

template <class Ptr>
__device__ __forceinline__ void xform(Ptr T, double x, double y, double z, double& ox, double& oy, double& oz) {
	ox = T[0] * x + T[1] * y + T[2] * z + T[3];
	oy = T[4] * x + T[5] * y + T[6] * z + T[7];
	oz = T[8] * x + T[9] * y + T[10] * z + T[11];
}

// Largest fp32 squared distance a candidate may show and still be the nearest neighbour, given the running fp32 minimum m:
//   f_k <= sqrt(m / (1 - gamma)) + a for the candidate k that gave m, the true nearest neighbour j* has f_j* <= kappa f_k,
//   and its fp32 value is at most (1 + gamma) (f_j* + a)^2.  1 + 2 gamma > 1 / (1 - gamma), and the last factor covers the at most seven
//   roundings of the expression (each <= 2^-24 relative, every term non-negative).
__device__ __forceinline__ float rerank_threshold(float m, float a, float kappa_ru) {
	const float r = sqrtf(m * (1.0f + 2.0f * (float)kGamma)) + a;
	const float f = kappa_ru * r + a;
	return f * f * (1.0f + (float)kGamma) * (1.0f + 0x1p-19f);
}

__device__ __forceinline__ float dist2_f32(float qx, float qy, float qz, float4 c) {
	const float dx = qx - c.x, dy = qy - c.y, dz = qz - c.z;
	return fmaf(dz, dz, fmaf(dy, dy, dx * dx));
}

// fp32 copy of the model and the largest |p| (as the bits of a non-negative double, so an integer max orders them)
__global__ void __launch_bounds__(kThreads) k_metrics_prep(const double* __restrict__ pts, int n, float4* __restrict__ pts32,
                                                           unsigned long long* __restrict__ pmax_bits) {
	const int i = blockIdx.x * kThreads + threadIdx.x;
	double r = 0.0;
	if (i < n) {
		const double x = pts[3 * (size_t)i], y = pts[3 * (size_t)i + 1], z = pts[3 * (size_t)i + 2];
		pts32[i] = make_float4((float)x, (float)y, (float)z, 0.f);
		r = sqrt(x * x + y * y + z * z);
	}
	for (int o = 16; o > 0; o >>= 1) r = fmax(r, __shfl_xor_sync(0xffffffffu, r, o));
	if ((threadIdx.x & 31) == 0) atomicMax(pmax_bits, (unsigned long long)__double_as_longlong(r));
}

// grid (n_frames, ceil(n / kChunk)): block (f, c) takes queries [c kChunk, (c + 1) kChunk) of frame f against the whole model
__global__ void __launch_bounds__(kThreads) k_pose_metrics(const double* __restrict__ pts, const float4* __restrict__ pts32, int n,
                                                           const FrameConst* __restrict__ frames, const unsigned long long* __restrict__ pmax_bits,
                                                           double* __restrict__ part_add, double* __restrict__ part_adds) {
	__shared__ float4 s_tile[kTile];
	static_assert(kTile >= kChunk, "the queries pass through the tile buffer");
	__shared__ double s_fr[kFrameDoubles];
	__shared__ double s_red[2][kThreads / 32];
	__shared__ double s_best[kQpt][kThreads];
	__shared__ float s_m[kQpt][kThreads], s_a[kQpt][kThreads];
	const int f = blockIdx.x, chunk = blockIdx.y, tid = threadIdx.x;
	const double* src = reinterpret_cast<const double*>(frames + f);
	for (int t = tid; t < kFrameDoubles; t += kThreads) s_fr[t] = src[t];
	__syncthreads();
	const FrameConst& fr = *reinterpret_cast<const FrameConst*>(s_fr);
	const double pmax = __longlong_as_double((long long)*pmax_bits);
	const float kappa = __double2float_ru(fr.kappa);
	// Only the fp32 query and its threshold stay in registers through the scan.  What the rerank alone needs - the poses, the running minima,
	// the rounding slack and the best squared float64 distance - lives in shared memory, one slot per thread and query.
	const volatile double* v_pred = s_fr + offsetof(FrameConst, pred) / sizeof(double);
	const volatile double* v_gt = s_fr + offsetof(FrameConst, gt) / sizeof(double);

	double sa = 0.0;
#pragma unroll 1
	for (int k = 0; k < kQpt; k++) {
		const int i = chunk * kChunk + k * kThreads + tid;
		const int ii = min(i, n - 1);          // queries past n repeat the last point and are left out of the sums
		const double x = pts[3 * (size_t)ii], y = pts[3 * (size_t)ii + 1], z = pts[3 * (size_t)ii + 2];
		double gx, gy, gz, cx, cy, cz, ux, uy, uz;
		xform(fr.gt, x, y, z, gx, gy, gz);
		xform(fr.pred, x, y, z, cx, cy, cz);
		xform(fr.M, x, y, z, ux, uy, uz);
		const double d2 = (gx - cx) * (gx - cx) + (gy - cy) * (gy - cy) + (gz - cz) * (gz - cz);
		if (i < n) sa += sqrt(d2);                         // ADD, in k order
		// the query's own point is a candidate too: it seeds the running minima
		s_best[k][tid] = d2;
		const float4 q = make_float4((float)ux, (float)uy, (float)uz, 0.f);
		s_tile[k * kThreads + tid] = q;         // the tile is loaded after the queries are in registers
		s_a[k][tid] = __double2float_ru(2.0 * kU * (sqrt(ux * ux + uy * uy + uz * uz) + pmax) + fr.a_abs);
		s_m[k][tid] = dist2_f32(q.x, q.y, q.z, pts32[ii]);
	}
	float qx[kQpt], qy[kQpt], qz[kQpt], T[kQpt];
#pragma unroll
	for (int k = 0; k < kQpt; k++) {
		const float4 q = s_tile[k * kThreads + tid];
		qx[k] = q.x; qy[k] = q.y; qz[k] = q.z;
		T[k] = rerank_threshold(s_m[k][tid], s_a[k][tid], kappa);
	}

	for (int base = 0; base < n; base += kTile) {
		const int cnt = min(kTile, n - base);
		__syncthreads();
		for (int t = tid; t < cnt; t += kThreads) s_tile[t] = pts32[base + t];
		__syncthreads();
#pragma unroll 1
		for (int t = 0; t < cnt; t++) {
			const float4 c = s_tile[t];
			float s[kQpt];
			bool hit = false;
#pragma unroll
			for (int k = 0; k < kQpt; k++) {
				s[k] = dist2_f32(qx[k], qy[k], qz[k], c);
				hit |= s[k] <= T[k];
			}
			if (hit) {
				const int j = base + t;
				const double x = pts[3 * (size_t)j], y = pts[3 * (size_t)j + 1], z = pts[3 * (size_t)j + 2];
				double cx, cy, cz;
				xform(v_pred, x, y, z, cx, cy, cz);
#pragma unroll
				for (int k = 0; k < kQpt; k++) {
					if (s[k] <= T[k]) {
						const int ii = min(chunk * kChunk + k * kThreads + tid, n - 1);
						const double px = pts[3 * (size_t)ii], py = pts[3 * (size_t)ii + 1], pz = pts[3 * (size_t)ii + 2];
						double gx, gy, gz;
						xform(v_gt, px, py, pz, gx, gy, gz);
						s_best[k][tid] = fmin(s_best[k][tid], (gx - cx) * (gx - cx) + (gy - cy) * (gy - cy) + (gz - cz) * (gz - cz));
						if (s[k] < s_m[k][tid]) { s_m[k][tid] = s[k]; T[k] = rerank_threshold(s[k], s_a[k][tid], kappa); }
					}
				}
			}
		}
	}

	// fixed-order sums: the thread's queries in k order, then a shuffle tree per warp, then the warps in order
	double ss = 0.0;
#pragma unroll
	for (int k = 0; k < kQpt; k++)
		if (chunk * kChunk + k * kThreads + tid < n) ss += sqrt(s_best[k][tid]);      // sqrt is monotone: the root of the smallest square
	for (int o = 16; o > 0; o >>= 1) {
		sa += __shfl_down_sync(0xffffffffu, sa, o);
		ss += __shfl_down_sync(0xffffffffu, ss, o);
	}
	if ((tid & 31) == 0) { s_red[0][tid >> 5] = sa; s_red[1][tid >> 5] = ss; }
	__syncthreads();
	if (tid == 0) {
		double ta = 0.0, ts = 0.0;
		for (int w = 0; w < kThreads / 32; w++) { ta += s_red[0][w]; ts += s_red[1][w]; }
		part_add[(size_t)f * gridDim.y + chunk] = ta;
		part_adds[(size_t)f * gridDim.y + chunk] = ts;
	}
}

__global__ void k_metrics_final(const double* __restrict__ part_add, const double* __restrict__ part_adds, int n_chunks, int n, int n_frames,
                                double* __restrict__ add_out, double* __restrict__ adds_out) {
	const int f = blockIdx.x * blockDim.x + threadIdx.x;
	if (f >= n_frames) return;
	double sa = 0.0, ss = 0.0;
	for (int c = 0; c < n_chunks; c++) { sa += part_add[(size_t)f * n_chunks + c]; ss += part_adds[(size_t)f * n_chunks + c]; }
	add_out[f] = sa / n;
	adds_out[f] = ss / n;
}

// pred^-1 gt and the filter's constants for one frame, in float64 on the host
void frame_const(const double* pred, const double* gt, FrameConst& fc) {
	for (int k = 0; k < 12; k++) { fc.pred[k] = pred[k]; fc.gt[k] = gt[k]; }
	const double* P = pred;
	// e = ||A^T A - I||_F bounds the spectral norm, so the squared singular values of A lie in [1 - e, 1 + e]
	double e2 = 0.0;
	for (int r = 0; r < 3; r++)
		for (int c = 0; c < 3; c++) {
			const double g = P[r] * P[c] + P[4 + r] * P[4 + c] + P[8 + r] * P[8 + c] - (r == c ? 1.0 : 0.0);
			e2 += g * g;
		}
	const double e = sqrt(e2) + 1e-12;
	const double det = P[0] * (P[5] * P[10] - P[6] * P[9]) - P[1] * (P[4] * P[10] - P[6] * P[8]) + P[2] * (P[4] * P[9] - P[5] * P[8]);
	for (int k = 0; k < 12; k++) fc.M[k] = (k % 5 == 0) ? 1.0 : 0.0;
	fc.kappa = INFINITY;
	if (e < 0.5 && det != 0.0) {
		double inv[9] = {
			(P[5] * P[10] - P[6] * P[9]) / det, (P[2] * P[9] - P[1] * P[10]) / det, (P[1] * P[6] - P[2] * P[5]) / det,
			(P[6] * P[8] - P[4] * P[10]) / det, (P[0] * P[10] - P[2] * P[8]) / det, (P[2] * P[4] - P[0] * P[6]) / det,
			(P[4] * P[9] - P[5] * P[8]) / det,  (P[1] * P[8] - P[0] * P[9]) / det,  (P[0] * P[5] - P[1] * P[4]) / det };
		const double d[3] = { gt[3] - P[3], gt[7] - P[7], gt[11] - P[11] };
		for (int r = 0; r < 3; r++) {
			for (int c = 0; c < 3; c++) fc.M[4 * r + c] = inv[3 * r] * gt[c] + inv[3 * r + 1] * gt[4 + c] + inv[3 * r + 2] * gt[8 + c];
			fc.M[4 * r + 3] = inv[3 * r] * d[0] + inv[3 * r + 1] * d[1] + inv[3 * r + 2] * d[2];
		}
		fc.kappa = sqrt((1.0 + e) / (1.0 - e));
	}
	// the float64 rounding of M and of q = M p is far below the fp32 terms; this bounds it by the poses' own scale
	const double tp = fabs(P[3]) + fabs(P[7]) + fabs(P[11]), tg = fabs(gt[3]) + fabs(gt[7]) + fabs(gt[11]);
	fc.a_abs = 1e-13 * (1.0 + tp + tg);
}

}  // namespace

struct MetricsState {
	int max_pts = 0, max_frames = 0;
	DevBuf pts32, frames, part, pmax;
	UploadBuf h_frames;
};
void StateDeleter::operator()(MetricsState* s) const { delete s; }

}  // namespace bt

using namespace bt;

extern "C" int bt_metrics_reserve(bt_ctx* ctx, int max_pts, int max_frames) {
	BT_REQUIRE(ctx, BT_ERR_INVALID_ARG, "bt_metrics_reserve: ctx is NULL");
	BT_REQUIRE(max_pts >= 1 && max_frames >= 1, BT_ERR_INVALID_ARG, "bt_metrics_reserve: max_pts %d / max_frames %d must be >= 1", max_pts, max_frames);
	BT_REQUIRE((max_pts + kChunk - 1) / kChunk <= 65535, BT_ERR_INVALID_ARG, "bt_metrics_reserve: max_pts %d > %d", max_pts, 65535 * kChunk);
	BT_CUDA(cudaSetDevice(ctx->device));
	if (!ctx->metrics) ctx->metrics.reset(new MetricsState());
	MetricsState* s = ctx->metrics.get();
	const size_t n_chunks = (size_t)(max_pts + kChunk - 1) / kChunk;
	BT_TRY(s->pts32.alloc(sizeof(float4) * (size_t)max_pts));
	BT_TRY(s->frames.alloc(sizeof(FrameConst) * (size_t)max_frames));
	BT_TRY(s->part.alloc(2 * sizeof(double) * n_chunks * max_frames));
	BT_TRY(s->pmax.alloc(sizeof(unsigned long long)));
	BT_TRY(s->h_frames.reserve(sizeof(FrameConst) * (size_t)max_frames));
	s->max_pts = max_pts; s->max_frames = max_frames;
	return BT_OK;
}

extern "C" int bt_pose_metrics(bt_ctx* ctx, const double* model_pts_dev, int n_pts, const double* pred_ob_in_cam, const double* gt_ob_in_cam, int n_frames,
                               double* add_out, double* adds_out, void* stream_) {
	BT_REQUIRE(n_pts >= 1 && n_frames >= 1, BT_ERR_INVALID_ARG, "bt_pose_metrics: n_pts %d / n_frames %d must be >= 1", n_pts, n_frames);
	BT_REQUIRE(model_pts_dev && pred_ob_in_cam && gt_ob_in_cam && add_out && adds_out, BT_ERR_INVALID_ARG, "bt_pose_metrics: NULL argument");
	for (size_t k = 0; k < 16 * (size_t)n_frames; k++)
		BT_REQUIRE(isfinite(pred_ob_in_cam[k]) && isfinite(gt_ob_in_cam[k]), BT_ERR_INVALID_ARG, "bt_pose_metrics: frame %d has a non-finite pose element", (int)(k / 16));
	BT_REQUIRE(ctx, BT_ERR_INVALID_ARG, "bt_pose_metrics: ctx is NULL");
	MetricsState* s = ctx->metrics.get();
	BT_REQUIRE(s, BT_ERR_INVALID_ARG, "bt_pose_metrics: call bt_metrics_reserve first");
	BT_REQUIRE(n_pts <= s->max_pts && n_frames <= s->max_frames, BT_ERR_CAPACITY, "bt_pose_metrics: %d points / %d frames exceed the reserved %d / %d",
	           n_pts, n_frames, s->max_pts, s->max_frames);
	cudaStream_t stream = (cudaStream_t)stream_;
	BT_CUDA(cudaSetDevice(ctx->device));
	FrameConst* hf;
	BT_TRY(s->h_frames.acquire(0, &hf));
	for (int f = 0; f < n_frames; f++) frame_const(pred_ob_in_cam + 16 * (size_t)f, gt_ob_in_cam + 16 * (size_t)f, hf[f]);
	BT_CUDA(cudaMemcpyAsync(s->frames.p, hf, sizeof(FrameConst) * (size_t)n_frames, cudaMemcpyHostToDevice, stream));
	BT_TRY(s->h_frames.in_flight(stream));
	BT_CUDA(cudaMemsetAsync(s->pmax.p, 0, sizeof(unsigned long long), stream));
	k_metrics_prep<<<(n_pts + kThreads - 1) / kThreads, kThreads, 0, stream>>>(model_pts_dev, n_pts, s->pts32.as<float4>(), s->pmax.as<unsigned long long>());
	const int n_chunks = (n_pts + kChunk - 1) / kChunk;
	double* part_add = s->part.as<double>();
	double* part_adds = part_add + (size_t)n_chunks * n_frames;
	k_pose_metrics<<<dim3(n_frames, n_chunks), kThreads, 0, stream>>>(model_pts_dev, s->pts32.as<float4>(), n_pts, s->frames.as<FrameConst>(),
	                                                                  s->pmax.as<unsigned long long>(), part_add, part_adds);
	k_metrics_final<<<(n_frames + 127) / 128, 128, 0, stream>>>(part_add, part_adds, n_chunks, n_pts, n_frames, add_out, adds_out);
	BT_CUDA(cudaGetLastError());
	return BT_OK;
}

// VOCap (scripts/eval_ycbineoat.py): sort the errors, keep those below max_err, precision k / n at the k-th, the monotone envelope over
// recall points [0, rec..., max_err], and the area divided by max_err.  NaN errors count in n and are never below max_err.
extern "C" int bt_vocap(const double* err, int n, double max_err, double* auc_out) {
	BT_REQUIRE(auc_out && n >= 0 && (err || n == 0), BT_ERR_INVALID_ARG, "bt_vocap: bad arguments");
	BT_REQUIRE(max_err > 0.0 && isfinite(max_err), BT_ERR_INVALID_ARG, "bt_vocap: max_err must be positive and finite");
	*auc_out = 0.0;
	std::vector<double> rec;
	rec.reserve(n);
	for (int i = 0; i < n; i++) if (err[i] < max_err) rec.push_back(err[i]);
	if (rec.empty()) return BT_OK;
	std::sort(rec.begin(), rec.end());
	const int m = (int)rec.size();
	std::vector<double> mrec(m + 2), mpre(m + 2);
	mrec[0] = 0.0; mpre[0] = 0.0;
	for (int k = 0; k < m; k++) { mrec[k + 1] = rec[k]; mpre[k + 1] = (double)(k + 1) / (double)n; }
	mrec[m + 1] = max_err; mpre[m + 1] = mpre[m];
	for (int k = 1; k < m + 2; k++) mpre[k] = std::max(mpre[k], mpre[k - 1]);
	double area = 0.0;
	for (int k = 1; k < m + 2; k++)
		if (mrec[k] != mrec[k - 1]) area += (mrec[k] - mrec[k - 1]) * mpre[k];
	*auc_out = area * (1.0 / max_err);      // the reference multiplies by 10 for its 0.1 m; 1.0 / 0.1 rounds to exactly 10
	return BT_OK;
}
