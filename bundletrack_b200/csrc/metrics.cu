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

// ---- NOCS-REAL275: the 6-PACK benchmark (the reference's scripts/benchmark.py) -------------------------------------------------------
// Per record, in float64, statement by statement as compute_RT_degree_cm_symmetry and compute_3d_iou_new state it (DESIGN.md §3.8):
//  - columns 0..2 of both 4 x 4 poses are divided by their norms over all four rows (normalizeRotation);
//  - a bottom row other than [0,0,0,1] on either pose gives theta = shift = 10000;
//  - R = M[:3,:3] / cbrt(det M[:3,:3]), negative determinants included;
//  - theta = arccos of the y-axis cosine (symmetric classes) or of (trace(R1 R2^T) - 1) / 2, NOT clipped: an argument beyond +-1 is NaN;
//  - shift = |T1 - T2|;
//  - IoU of the two transformed corner sets, with the box extents taken PER CORNER over x, y and z (np.amax(bbox, axis=0) of a [3, 8]
//    array) and the division by the homogeneous row; for symmetric classes the maximum over 20 rotations of the ground truth about its y
//    axis (gt @ Y(2 pi i / 20)), starting at 0 and skipping NaN as Python's max(max_iou, v) does.
// Operation order, pinned (numpy's dot / norm / det / matmul go through BLAS and LAPACK, whose rounding is not): every sum of products is
// ((a0 b0 + a1 b1) + a2 b2) + a3 b3 left to right, without fused multiply-adds (__dmul_rn / __dadd_rn); det = a(ei - fh) - b(di - fg) +
// c(dh - eg); products over the 8 corners run in corner order.  cbrt and acos are CUDA's (1 ulp / 2 ulp), the 20 (cos, sin) pairs are the
// host's libm of ((2 pi) i) / 20.0.
namespace bt {
namespace {

constexpr int kNocsWarps = 4;                      // records per block
constexpr int kNocsRot = 20;                       // the benchmark's rotations about y
constexpr double kRadToDeg = 180.0 / 3.141592653589793;

struct NocsRecord {
	double pred[16], gt[16];     // row-major 4 x 4, translations in mm
	double corners[24];          // 8 rows x, y, z of model_scales/<model>.txt
	int32_t sym, pad;
};

__device__ __forceinline__ double mul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double add(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double sub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double dot3(double a0, double a1, double a2, double b0, double b1, double b2) {
	return add(add(mul(a0, b0), mul(a1, b1)), mul(a2, b2));
}
// numpy's maximum / minimum: a NaN on either side is the result
__device__ __forceinline__ double nmax(double a, double b) { return (a > b || isnan(a)) ? a : b; }
__device__ __forceinline__ double nmin(double a, double b) { return (a < b || isnan(a)) ? a : b; }

__device__ __forceinline__ void normalize_columns(double* M) {
#pragma unroll
	for (int c = 0; c < 3; c++) {
		const double n = sqrt(add(add(add(mul(M[c], M[c]), mul(M[4 + c], M[4 + c])), mul(M[8 + c], M[8 + c])), mul(M[12 + c], M[12 + c])));
#pragma unroll
		for (int r = 0; r < 4; r++) M[4 * r + c] = __ddiv_rn(M[4 * r + c], n);
	}
}

__device__ __forceinline__ double det3(const double* M) {
	const double a = mul(M[0], sub(mul(M[5], M[10]), mul(M[6], M[9])));
	const double b = mul(M[1], sub(mul(M[4], M[10]), mul(M[6], M[8])));
	const double c = mul(M[2], sub(mul(M[4], M[9]), mul(M[5], M[8])));
	return add(sub(a, b), c);
}

// transform_coordinates_3d of one corner: row r of M [x y z 1]^T over the homogeneous row, then the corner's max / min over x, y, z
__device__ __forceinline__ void corner_extent(const double* M, double x, double y, double z, double& hi, double& lo) {
	double w[4];
#pragma unroll
	for (int r = 0; r < 4; r++) w[r] = add(add(add(mul(M[4 * r], x), mul(M[4 * r + 1], y)), mul(M[4 * r + 2], z)), M[4 * r + 3]);
	const double u0 = __ddiv_rn(w[0], w[3]), u1 = __ddiv_rn(w[1], w[3]), u2 = __ddiv_rn(w[2], w[3]);
	hi = nmax(nmax(u0, u1), u2);
	lo = nmin(nmin(u0, u1), u2);
}

// grid ceil(n / kNocsWarps) x (32 kNocsWarps): one warp per record.  Lane r < 20 of a symmetric record evaluates rotation r, lane 0 of any
// other record the asymmetric IoU (rotation 0: cos 1, sin 0 reproduces gt exactly).
__global__ void __launch_bounds__(32 * kNocsWarps) k_nocs_metrics(const NocsRecord* __restrict__ recs, const double2* __restrict__ rot, int n,
                                                                  double* __restrict__ theta_out, double* __restrict__ shift_out,
                                                                  double* __restrict__ iou_out) {
	const int lane = threadIdx.x & 31;
	const int i = blockIdx.x * kNocsWarps + (threadIdx.x >> 5);
	if (i >= n) return;                                // whole warps leave together
	const NocsRecord& rec = recs[i];
	double P[16], G[16];
#pragma unroll
	for (int k = 0; k < 16; k++) { P[k] = rec.pred[k]; G[k] = rec.gt[k]; }
	const bool sym = rec.sym != 0;
	normalize_columns(P);
	normalize_columns(G);

	if (lane == 0) {
		double theta = 10000.0, shift = 10000.0;
		const bool bottom = P[12] == 0.0 && P[13] == 0.0 && P[14] == 0.0 && P[15] == 1.0 && G[12] == 0.0 && G[13] == 0.0 && G[14] == 0.0 && G[15] == 1.0;
		if (bottom) {
			const double c1 = cbrt(det3(P)), c2 = cbrt(det3(G));
			double R1[9], R2[9];
#pragma unroll
			for (int r = 0; r < 3; r++)
#pragma unroll
				for (int c = 0; c < 3; c++) { R1[3 * r + c] = __ddiv_rn(P[4 * r + c], c1); R2[3 * r + c] = __ddiv_rn(G[4 * r + c], c2); }
			double arg;
			if (sym) {
				// y1 = R1 [0 1 0]^T, y2 = R2 [0 1 0]^T: the middle columns
				const double d = dot3(R1[1], R1[4], R1[7], R2[1], R2[4], R2[7]);
				const double n1 = sqrt(dot3(R1[1], R1[4], R1[7], R1[1], R1[4], R1[7]));
				const double n2 = sqrt(dot3(R2[1], R2[4], R2[7], R2[1], R2[4], R2[7]));
				arg = __ddiv_rn(d, mul(n1, n2));
			} else {
				// trace(R1 R2^T) = sum_r R1[r,:] . R2[r,:]
				const double t0 = dot3(R1[0], R1[1], R1[2], R2[0], R2[1], R2[2]);
				const double t1 = dot3(R1[3], R1[4], R1[5], R2[3], R2[4], R2[5]);
				const double t2 = dot3(R1[6], R1[7], R1[8], R2[6], R2[7], R2[8]);
				arg = __ddiv_rn(sub(add(add(t0, t1), t2), 1.0), 2.0);
			}
			theta = mul(acos(arg), kRadToDeg);
			const double dx = sub(P[3], G[3]), dy = sub(P[7], G[7]), dz = sub(P[11], G[11]);
			shift = sqrt(dot3(dx, dy, dz, dx, dy, dz));
		}
		theta_out[i] = theta;
		shift_out[i] = shift;
	}

	double iou = 0.0;
	if (lane < (sym ? kNocsRot : 1)) {
		// gt @ Y(t): columns 0 and 2 mix, 1 and 3 stay
		const double2 cs = rot[lane];
#pragma unroll
		for (int r = 0; r < 4; r++) {
			const double g0 = G[4 * r], g2 = G[4 * r + 2];
			G[4 * r] = add(mul(g0, cs.x), mul(g2, -cs.y));
			G[4 * r + 2] = add(mul(g0, cs.y), mul(g2, cs.x));
		}
		double dmin = INFINITY, inter = 1.0, v1 = 1.0, v2 = 1.0;
#pragma unroll 1
		for (int c = 0; c < 8; c++) {
			const double x = rec.corners[3 * c], y = rec.corners[3 * c + 1], z = rec.corners[3 * c + 2];
			double hi1, lo1, hi2, lo2;
			corner_extent(G, x, y, z, hi1, lo1);
			corner_extent(P, x, y, z, hi2, lo2);
			const double d = sub(nmin(hi1, hi2), nmax(lo1, lo2));
			dmin = c == 0 ? d : nmin(dmin, d);
			inter = c == 0 ? d : mul(inter, d);
			v1 = c == 0 ? sub(hi1, lo1) : mul(v1, sub(hi1, lo1));
			v2 = c == 0 ? sub(hi2, lo2) : mul(v2, sub(hi2, lo2));
		}
		if (dmin < 0.0) inter = 0.0;
		iou = __ddiv_rn(inter, sub(add(v1, v2), inter));
	}
	if (sym) {
		// max(max_iou, v) from 0 in rotation order: a value enters only if it is greater, so NaN never does
		double best = (iou > 0.0) ? iou : 0.0;
		for (int o = 16; o > 0; o >>= 1) {
			const double v = __shfl_xor_sync(0xffffffffu, best, o);
			if (v > best) best = v;
		}
		iou = best;
	}
	if (lane == 0) iou_out[i] = iou;
}

}  // namespace

struct NocsState {
	int max_records = 0;
	DevBuf recs;
	UploadBuf h_recs;
};
void StateDeleter::operator()(NocsState* s) const { delete s; }

}  // namespace bt

extern "C" int bt_nocs_reserve(bt_ctx* ctx, int max_records) {
	BT_REQUIRE(ctx, BT_ERR_INVALID_ARG, "bt_nocs_reserve: ctx is NULL");
	BT_REQUIRE(max_records >= 1, BT_ERR_INVALID_ARG, "bt_nocs_reserve: max_records %d must be >= 1", max_records);
	BT_CUDA(cudaSetDevice(ctx->device));
	if (!ctx->nocs) ctx->nocs.reset(new NocsState());
	NocsState* s = ctx->nocs.get();
	const size_t bytes = kNocsRot * sizeof(double2) + sizeof(NocsRecord) * (size_t)max_records;
	BT_TRY(s->recs.alloc(bytes));
	BT_TRY(s->h_recs.reserve(bytes));
	s->max_records = max_records;
	return BT_OK;
}

extern "C" int bt_nocs_metrics(bt_ctx* ctx, const double* pred, const double* gt, const double* corners, const int32_t* symmetric, int n,
                               double* theta_deg_out, double* shift_out, double* iou_out, void* stream_) {
	BT_REQUIRE(n >= 1, BT_ERR_INVALID_ARG, "bt_nocs_metrics: n %d must be >= 1", n);
	BT_REQUIRE(pred && gt && corners && symmetric && theta_deg_out && shift_out && iou_out, BT_ERR_INVALID_ARG, "bt_nocs_metrics: NULL argument");
	for (size_t k = 0; k < 16 * (size_t)n; k++)
		BT_REQUIRE(isfinite(pred[k]) && isfinite(gt[k]), BT_ERR_INVALID_ARG, "bt_nocs_metrics: record %d has a non-finite pose element", (int)(k / 16));
	for (size_t k = 0; k < 24 * (size_t)n; k++)
		BT_REQUIRE(isfinite(corners[k]), BT_ERR_INVALID_ARG, "bt_nocs_metrics: record %d has a non-finite corner", (int)(k / 24));
	BT_REQUIRE(ctx, BT_ERR_INVALID_ARG, "bt_nocs_metrics: ctx is NULL");
	NocsState* s = ctx->nocs.get();
	BT_REQUIRE(s, BT_ERR_INVALID_ARG, "bt_nocs_metrics: call bt_nocs_reserve first");
	BT_REQUIRE(n <= s->max_records, BT_ERR_CAPACITY, "bt_nocs_metrics: %d records exceed the reserved %d", n, s->max_records);
	cudaStream_t stream = (cudaStream_t)stream_;
	BT_CUDA(cudaSetDevice(ctx->device));
	char* h;
	BT_TRY(s->h_recs.acquire(0, &h));
	double2* hrot = reinterpret_cast<double2*>(h);
	for (int r = 0; r < kNocsRot; r++) {
		const double t = ((2.0 * 3.141592653589793) * r) / 20.0;      // 2 * math.pi * i / float(n), Python's order
		hrot[r] = make_double2(cos(t), sin(t));
	}
	NocsRecord* hr = reinterpret_cast<NocsRecord*>(h + kNocsRot * sizeof(double2));
	for (int i = 0; i < n; i++) {
		memcpy(hr[i].pred, pred + 16 * (size_t)i, sizeof(hr[i].pred));
		memcpy(hr[i].gt, gt + 16 * (size_t)i, sizeof(hr[i].gt));
		memcpy(hr[i].corners, corners + 24 * (size_t)i, sizeof(hr[i].corners));
		hr[i].sym = symmetric[i] != 0;
		hr[i].pad = 0;
	}
	const size_t bytes = kNocsRot * sizeof(double2) + sizeof(NocsRecord) * (size_t)n;
	BT_CUDA(cudaMemcpyAsync(s->recs.p, h, bytes, cudaMemcpyHostToDevice, stream));
	BT_TRY(s->h_recs.in_flight(stream));
	const double2* d_rot = s->recs.as<double2>();
	const NocsRecord* d_recs = reinterpret_cast<const NocsRecord*>(s->recs.as<char>() + kNocsRot * sizeof(double2));
	k_nocs_metrics<<<(n + kNocsWarps - 1) / kNocsWarps, 32 * kNocsWarps, 0, stream>>>(d_recs, d_rot, n, theta_deg_out, shift_out, iou_out);
	BT_CUDA(cudaGetLastError());
	return BT_OK;
}

// numpy's pairwise summation (pairwise_sum in loops_utils.h): below 8 terms in order, up to 128 through 8 accumulators, above that split
// at a multiple of 8 near the middle.  np.add.reduce feeds it all terms of a contiguous array, np.mean divides the result by the count.
static double np_pairwise_sum(const double* a, size_t n) {
	if (n < 8) {
		double res = -0.0;
		for (size_t i = 0; i < n; i++) res += a[i];
		return res;
	}
	if (n <= 128) {
		double r[8];
		for (int j = 0; j < 8; j++) r[j] = a[j];
		size_t i = 8;
		for (; i < n - (n % 8); i += 8)
			for (int j = 0; j < 8; j++) r[j] += a[i + j];
		double res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]));
		for (; i < n; i++) res += a[i];
		return res;
	}
	size_t n2 = n / 2;
	n2 -= n2 % 8;
	return np_pairwise_sum(a, n2) + np_pairwise_sum(a + n2, n - n2);
}

static double np_mean(const std::vector<double>& v) {
	if (v.empty()) return NAN;                       // np.mean([])
	return np_pairwise_sum(v.data(), v.size()) / (double)v.size();
}

// benchmark.py main's aggregation: per class the 5 deg 5 cm and IoU25 fractions of all its records, the mean theta over IoU > 0.25 and
// theta < 360, the mean shift over IoU > 0.25; overall x += v / 6 in class order.
extern "C" int bt_nocs_score(const int32_t* cls, const int32_t* scored, const double* theta_deg, const double* shift, const double* iou, int n,
                             double* per_class_out, double* overall_out) {
	BT_REQUIRE(n >= 1, BT_ERR_INVALID_ARG, "bt_nocs_score: n %d must be >= 1", n);
	BT_REQUIRE(cls && scored && theta_deg && shift && iou && per_class_out && overall_out, BT_ERR_INVALID_ARG, "bt_nocs_score: NULL argument");
	int cls_num[6] = {0, 0, 0, 0, 0, 0};
	for (int i = 0; i < n; i++) {
		BT_REQUIRE(cls[i] >= 1 && cls[i] <= 6, BT_ERR_INVALID_ARG, "bt_nocs_score: record %d has class %d outside 1..6", i, cls[i]);
		cls_num[cls[i] - 1]++;
	}
	for (int c = 0; c < 6; c++)
		BT_REQUIRE(cls_num[c] > 0, BT_ERR_INVALID_ARG, "bt_nocs_score: class %d has no record (the benchmark divides by its count)", c + 1);
	double overall[4] = {0.0, 0.0, 0.0, 0.0};
	std::vector<double> rot, trans;
	for (int c = 0; c < 6; c++) {
		int in55 = 0, iou25 = 0;
		rot.clear();
		trans.clear();
		for (int i = 0; i < n; i++) {
			if (cls[i] != c + 1 || !scored[i]) continue;
			if (iou[i] > 0.25 && theta_deg[i] < 360) rot.push_back(theta_deg[i]);
			if (iou[i] > 0.25) { trans.push_back(shift[i]); iou25++; }
			if (theta_deg[i] < 5 && shift[i] < 50) in55++;
		}
		const double v[4] = {(double)in55 / (double)cls_num[c], (double)iou25 / (double)cls_num[c], np_mean(rot), np_mean(trans)};
		for (int k = 0; k < 4; k++) {
			per_class_out[4 * c + k] = v[k];
			overall[k] += v[k] / 6;
		}
	}
	for (int k = 0; k < 4; k++) overall_out[k] = overall[k];
	return BT_OK;
}
