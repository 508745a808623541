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
// The scan itself (nearest_scan) also serves the object model's surface distances, at the end of this file.
#include <math.h>
#include <stddef.h>
#include <algorithm>
#include <vector>
#include "bt_common.cuh"
#include "bt_scan.cuh"

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

// The exact nearest-distance scan that ADD-S and the surface distances share.  On entry each thread has seeded its kQpt queries: slot
// k * kThreads + tid of s_tile holds query k in fp32, s_a[k][tid] its rounding slack a, and s_m[k][tid] / s_best[k][tid] the fp32 and float64
// squared distances to one candidate.  The scan runs every target of pts32 through the fp32 filter and hands each survivor to `rr`:
//   rr.target(j, cx, cy, cz)   target j's float64 point, as the rerank compares it;
//   rr.dist2(k, cx, cy, cz)    the float64 squared distance from query k to that point.
// On return s_best[k][tid] is the smallest rerank over all candidates.  The whole block calls it.
template <class Rerank>
__device__ __forceinline__ void nearest_scan(const float4* __restrict__ pts32, int n, float kappa, float4* s_tile, double (*s_best)[kThreads],
                                             float (*s_m)[kThreads], float (*s_a)[kThreads], const Rerank& rr) {
	const int tid = threadIdx.x;
	// Only the fp32 query and its threshold stay in registers through the scan.  What the rerank alone needs - the running minima, the
	// rounding slack and the best squared float64 distance - lives in shared memory, one slot per thread and query.
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
				double cx, cy, cz;
				rr.target(base + t, cx, cy, cz);
#pragma unroll
				for (int k = 0; k < kQpt; k++) {
					if (s[k] <= T[k]) {
						s_best[k][tid] = fmin(s_best[k][tid], rr.dist2(k, cx, cy, cz));
						if (s[k] < s_m[k][tid]) { s_m[k][tid] = s[k]; T[k] = rerank_threshold(s[k], s_a[k][tid], kappa); }
					}
				}
			}
		}
	}
}

// ADD-S's rerank: |gt p_i - pred p_j|, the reference's expression, with the poses read from shared memory
struct PoseRerank {
	const double* pts;
	const volatile double* pred;
	const volatile double* gt;
	int first, n;            // query k of this thread is point min(first + k kThreads, n - 1)
	__device__ __forceinline__ void target(int j, double& cx, double& cy, double& cz) const {
		const double x = pts[3 * (size_t)j], y = pts[3 * (size_t)j + 1], z = pts[3 * (size_t)j + 2];
		xform(pred, x, y, z, cx, cy, cz);
	}
	__device__ __forceinline__ double dist2(int k, double cx, double cy, double cz) const {
		const int ii = min(first + k * kThreads, n - 1);
		const double px = pts[3 * (size_t)ii], py = pts[3 * (size_t)ii + 1], pz = pts[3 * (size_t)ii + 2];
		double gx, gy, gz;
		xform(gt, px, py, pz, gx, gy, gz);
		return (gx - cx) * (gx - cx) + (gy - cy) * (gy - cy) + (gz - cz) * (gz - cz);
	}
};

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
	const PoseRerank rr{pts, s_fr + offsetof(FrameConst, pred) / sizeof(double), s_fr + offsetof(FrameConst, gt) / sizeof(double), chunk * kChunk + tid, n};
	nearest_scan(pts32, n, kappa, s_tile, s_best, s_m, s_a, rr);

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
	bool ready = false;
	int max_pts = 0, max_frames = 0;
	DevBuf pts32, part, pmax;
	TableBlock<> frames;
};
struct FrameTable : TableLayout { Slice<FrameConst> frames; };
static FrameTable frame_table(size_t n_frames) { FrameTable t; t.frames = t.add<FrameConst>(n_frames); return t; }
void StateDeleter::operator()(MetricsState* s) const { delete s; }

}  // namespace bt

using namespace bt;

extern "C" int bt_metrics_reserve(bt_ctx* ctx, int max_pts, int max_frames) {
	BT_REQUIRE(ctx, BT_ERR_INVALID_ARG, "bt_metrics_reserve: ctx is NULL");
	BT_REQUIRE(max_pts >= 1 && max_frames >= 1, BT_ERR_INVALID_ARG, "bt_metrics_reserve: max_pts %d / max_frames %d must be >= 1", max_pts, max_frames);
	BT_REQUIRE((max_pts + kChunk - 1) / kChunk <= 65535, BT_ERR_INVALID_ARG, "bt_metrics_reserve: max_pts %d > %d", max_pts, 65535 * kChunk);
	MetricsState* s;
	BT_TRY(take_state(ctx, &bt_ctx::metrics, &s));
	const size_t n_chunks = (size_t)(max_pts + kChunk - 1) / kChunk;
	BT_TRY(s->pts32.alloc(sizeof(float4) * (size_t)max_pts));
	BT_TRY(s->part.alloc(2 * sizeof(double) * n_chunks * max_frames));
	BT_TRY(s->pmax.alloc(sizeof(unsigned long long)));
	BT_TRY(s->frames.reserve(frame_table(max_frames).total));
	s->max_pts = max_pts; s->max_frames = max_frames;
	s->ready = true;
	return BT_OK;
}

extern "C" int bt_pose_metrics(bt_ctx* ctx, const double* model_pts_dev, int n_pts, const double* pred_ob_in_cam, const double* gt_ob_in_cam, int n_frames,
                               double* add_out, double* adds_out, void* stream_) {
	BT_REQUIRE(n_pts >= 1 && n_frames >= 1, BT_ERR_INVALID_ARG, "bt_pose_metrics: n_pts %d / n_frames %d must be >= 1", n_pts, n_frames);
	BT_REQUIRE(model_pts_dev && pred_ob_in_cam && gt_ob_in_cam && add_out && adds_out, BT_ERR_INVALID_ARG, "bt_pose_metrics: NULL argument");
	for (size_t k = 0; k < 16 * (size_t)n_frames; k++)
		BT_REQUIRE(isfinite(pred_ob_in_cam[k]) && isfinite(gt_ob_in_cam[k]), BT_ERR_INVALID_ARG, "bt_pose_metrics: frame %d has a non-finite pose element", (int)(k / 16));
	MetricsState* s;
	BT_TRY(state_of(ctx, &bt_ctx::metrics, "bt_pose_metrics", "bt_metrics_reserve", &s));
	BT_REQUIRE(n_pts <= s->max_pts && n_frames <= s->max_frames, BT_ERR_CAPACITY, "bt_pose_metrics: %d points / %d frames exceed the reserved %d / %d",
	           n_pts, n_frames, s->max_pts, s->max_frames);
	cudaStream_t stream = (cudaStream_t)stream_;
	const FrameTable t = frame_table(n_frames);
	BT_TRY(s->frames.begin("bt_pose_metrics", t));
	FrameConst* hf = s->frames.host(t.frames);
	for (int f = 0; f < n_frames; f++) frame_const(pred_ob_in_cam + 16 * (size_t)f, gt_ob_in_cam + 16 * (size_t)f, hf[f]);
	BT_TRY(s->frames.send(0, t.frames.end(), stream));
	BT_TRY(s->frames.in_flight(stream));
	BT_CUDA(cudaMemsetAsync(s->pmax.p, 0, sizeof(unsigned long long), stream));
	k_metrics_prep<<<(n_pts + kThreads - 1) / kThreads, kThreads, 0, stream>>>(model_pts_dev, n_pts, s->pts32.as<float4>(), s->pmax.as<unsigned long long>());
	const int n_chunks = (n_pts + kChunk - 1) / kChunk;
	double* part_add = s->part.as<double>();
	double* part_adds = part_add + (size_t)n_chunks * n_frames;
	k_pose_metrics<<<dim3(n_frames, n_chunks), kThreads, 0, stream>>>(model_pts_dev, s->pts32.as<float4>(), n_pts, s->frames.dev(t.frames),
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
	bool ready = false;
	int max_records = 0;
	TableBlock<> recs;
};
// the rotation table (kNocsRot angles), then the records
struct NocsTables : TableLayout { Slice<double2> rot; Slice<NocsRecord> recs; };
static NocsTables nocs_tables(size_t n) { NocsTables t; t.rot = t.add<double2>(kNocsRot); t.recs = t.add<NocsRecord>(n); return t; }
void StateDeleter::operator()(NocsState* s) const { delete s; }

}  // namespace bt

extern "C" int bt_nocs_reserve(bt_ctx* ctx, int max_records) {
	BT_REQUIRE(ctx, BT_ERR_INVALID_ARG, "bt_nocs_reserve: ctx is NULL");
	BT_REQUIRE(max_records >= 1, BT_ERR_INVALID_ARG, "bt_nocs_reserve: max_records %d must be >= 1", max_records);
	NocsState* s;
	BT_TRY(take_state(ctx, &bt_ctx::nocs, &s));
	BT_TRY(s->recs.reserve(nocs_tables(max_records).total));
	s->max_records = max_records;
	s->ready = true;
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
	NocsState* s;
	BT_TRY(state_of(ctx, &bt_ctx::nocs, "bt_nocs_metrics", "bt_nocs_reserve", &s));
	BT_REQUIRE(n <= s->max_records, BT_ERR_CAPACITY, "bt_nocs_metrics: %d records exceed the reserved %d", n, s->max_records);
	cudaStream_t stream = (cudaStream_t)stream_;
	const NocsTables t = nocs_tables(n);
	BT_TRY(s->recs.begin("bt_nocs_metrics", t));
	double2* hrot = s->recs.host(t.rot);
	for (int r = 0; r < kNocsRot; r++) {
		const double t = ((2.0 * 3.141592653589793) * r) / 20.0;      // 2 * math.pi * i / float(n), Python's order
		hrot[r] = make_double2(cos(t), sin(t));
	}
	NocsRecord* hr = s->recs.host(t.recs);
	for (int i = 0; i < n; i++) {
		memcpy(hr[i].pred, pred + 16 * (size_t)i, sizeof(hr[i].pred));
		memcpy(hr[i].gt, gt + 16 * (size_t)i, sizeof(hr[i].gt));
		memcpy(hr[i].corners, corners + 24 * (size_t)i, sizeof(hr[i].corners));
		hr[i].sym = symmetric[i] != 0;
		hr[i].pad = 0;
	}
	BT_TRY(s->recs.send(0, t.recs.end(), stream));
	BT_TRY(s->recs.in_flight(stream));
	const double2* d_rot = s->recs.dev(t.rot);
	const NocsRecord* d_recs = s->recs.dev(t.recs);
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

// ---- object model accuracy: surface samples and exact nearest distances both ways (DESIGN.md §3.15) --------------------------------------
// Sampling, pinned so that oracle/surface_oracle.py restates it bit for bit:
//  - per face, w = |(B - A) x (C - A)| (twice the area) in float64, every operation rounded on its own, sums left to right;
//  - the weight q = floor(w / w_max 2^32), an integer, with w_max the largest w (an integer max of the bits of non-negative doubles);
//  - the CDF is the 64-bit inclusive prefix sum of q, exact, so its order does not matter; total = the last entry;
//  - sample k draws h_i = splitmix64 output i from state `seed`, i = 3k, 3k + 1, 3k + 2.  Its position in [0, total) is
//    ((k 2^32 + (h_3k >> 32)) total) / (N 2^32), integer division, one per stratum of the CDF; its face is the first whose CDF exceeds it,
//    so a face with q = 0 is never chosen;
//  - u1, u2 = (h >> 11) 2^-53 of the other two, s = sqrt(u1), and the point is ((1 - s) A + s (1 - u2) B) + s u2 C per coordinate.
// Distances: the ADD-S scan with the identity as the pose (kappa = 1), reranking |a_i - b_j| as sqrt(((dx dx + dy dy) + dz dz)).
namespace bt {
namespace {

constexpr int kFaceThreads = 1024;                 // faces per CDF block
constexpr int kMaxSurfaceFaces = 1 << 27;          // q <= 2^32 per face, so the total stays below 2^59
constexpr int kMaxSurfaceSamples = 1 << 27;

// what one sampling call reads back: the CDF's total, and n_faces - f of the lowest face f with a bad index or a non-finite vertex (0: none)
struct SampleStatus {
	unsigned long long total, wmax_bits;
	int bad, pad;
};

__device__ __forceinline__ unsigned long long splitmix64(unsigned long long seed, unsigned long long i) {
	unsigned long long z = seed + (i + 1) * 0x9E3779B97F4A7C15ull;
	z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
	z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
	return z ^ (z >> 31);
}

__device__ __forceinline__ double3 vert(const double* v, int i) { return make_double3(v[3 * (size_t)i], v[3 * (size_t)i + 1], v[3 * (size_t)i + 2]); }

__global__ void __launch_bounds__(kThreads) k_face_weight(const double* __restrict__ verts, int n_verts, const int32_t* __restrict__ faces, int n_faces,
                                                          double* __restrict__ w_out, SampleStatus* __restrict__ st) {
	const int f = blockIdx.x * kThreads + threadIdx.x;
	if (f >= n_faces) return;
	const int i0 = faces[3 * (size_t)f], i1 = faces[3 * (size_t)f + 1], i2 = faces[3 * (size_t)f + 2];
	double w = 0.0;
	bool ok = i0 >= 0 && i0 < n_verts && i1 >= 0 && i1 < n_verts && i2 >= 0 && i2 < n_verts;
	if (ok) {
		const double3 A = vert(verts, i0), B = vert(verts, i1), C = vert(verts, i2);
		const double ux = sub(B.x, A.x), uy = sub(B.y, A.y), uz = sub(B.z, A.z);
		const double vx = sub(C.x, A.x), vy = sub(C.y, A.y), vz = sub(C.z, A.z);
		const double cx = sub(mul(uy, vz), mul(uz, vy)), cy = sub(mul(uz, vx), mul(ux, vz)), cz = sub(mul(ux, vy), mul(uy, vx));
		w = sqrt(dot3(cx, cy, cz, cx, cy, cz));
		ok = isfinite(w) && isfinite(A.x + A.y + A.z + B.x + B.y + B.z + C.x + C.y + C.z);
	}
	if (!ok) { atomicMax(&st->bad, n_faces - f); w = 0.0; }
	w_out[f] = w;
	atomicMax(&st->wmax_bits, (unsigned long long)__double_as_longlong(w));
}

// per block of kFaceThreads faces: q and its inclusive prefix within the block, and the block's total
__global__ void __launch_bounds__(kFaceThreads) k_face_cdf(const double* __restrict__ w, int n_faces, const SampleStatus* __restrict__ st,
                                                           unsigned long long* __restrict__ cdf, unsigned long long* __restrict__ block_tot) {
	__shared__ unsigned long long s[kFaceThreads / 32];
	const int f = blockIdx.x * kFaceThreads + threadIdx.x;
	const double wmax = __longlong_as_double((long long)st->wmax_bits);
	unsigned long long q = 0;
	if (f < n_faces && wmax > 0.0) q = __double2ull_rz(__dmul_rn(__ddiv_rn(w[f], wmax), 4294967296.0));
	unsigned long long tot;
	const unsigned long long ex = block_excl_scan(q, s, &tot);
	if (f < n_faces) cdf[f] = ex + q;
	if (threadIdx.x == 0) block_tot[blockIdx.x] = tot;
}

// one block: the blocks' offsets (exclusive prefix of their totals, in rounds of kFaceThreads) and the CDF's total
__global__ void __launch_bounds__(kFaceThreads) k_face_cdf_top(unsigned long long* __restrict__ block_tot, int n_blocks, SampleStatus* __restrict__ st) {
	__shared__ unsigned long long s[kFaceThreads / 32];
	unsigned long long carry = 0;
	for (int base = 0; base < n_blocks; base += kFaceThreads) {
		const int b = base + threadIdx.x;
		const unsigned long long v = b < n_blocks ? block_tot[b] : 0;
		unsigned long long tot;
		const unsigned long long ex = block_excl_scan(v, s, &tot);
		if (b < n_blocks) block_tot[b] = carry + ex;
		carry += tot;
	}
	if (threadIdx.x == 0) st->total = carry;
}

__global__ void __launch_bounds__(kFaceThreads) k_face_cdf_add(unsigned long long* __restrict__ cdf, int n_faces, const unsigned long long* __restrict__ block_off) {
	const int f = blockIdx.x * kFaceThreads + threadIdx.x;
	if (f < n_faces) cdf[f] += block_off[blockIdx.x];
}

__global__ void __launch_bounds__(kThreads) k_mesh_sample(const double* __restrict__ verts, const int32_t* __restrict__ faces,
                                                          const unsigned long long* __restrict__ cdf, int n_faces, const SampleStatus* __restrict__ st,
                                                          int n_samples, unsigned long long seed, double* __restrict__ out) {
	const int k = blockIdx.x * kThreads + threadIdx.x;
	if (k >= n_samples) return;
	const unsigned long long total = st->total;
	const unsigned long long h0 = splitmix64(seed, 3ull * k), h1 = splitmix64(seed, 3ull * k + 1), h2 = splitmix64(seed, 3ull * k + 2);
	const unsigned long long x = ((unsigned long long)k << 32) + (h0 >> 32);
	const unsigned long long pos = (unsigned long long)(((unsigned __int128)x * total) / ((unsigned __int128)n_samples << 32));
	int lo = 0, hi = n_faces - 1;
	while (lo < hi) {                                  // the first face whose CDF exceeds pos
		const int mid = (lo + hi) >> 1;
		if (cdf[mid] > pos) hi = mid;
		else lo = mid + 1;
	}
	const double u1 = (double)(h1 >> 11) * 0x1p-53, u2 = (double)(h2 >> 11) * 0x1p-53;
	const double s = sqrt(u1);
	const double b0 = sub(1.0, s), b1 = mul(s, sub(1.0, u2)), b2 = mul(s, u2);
	const double3 A = vert(verts, faces[3 * (size_t)lo]), B = vert(verts, faces[3 * (size_t)lo + 1]), C = vert(verts, faces[3 * (size_t)lo + 2]);
	out[3 * (size_t)k] = add(add(mul(b0, A.x), mul(b1, B.x)), mul(b2, C.x));
	out[3 * (size_t)k + 1] = add(add(mul(b0, A.y), mul(b1, B.y)), mul(b2, C.y));
	out[3 * (size_t)k + 2] = add(add(mul(b0, A.z), mul(b1, B.z)), mul(b2, C.z));
}

// The surface's rerank: |q_i - t_j| of two float64 point sets, every operation rounded on its own
struct PointRerank {
	const double* q;
	const double* t;
	int first, n;            // query k of this thread is point min(first + k kThreads, n - 1)
	__device__ __forceinline__ void target(int j, double& cx, double& cy, double& cz) const {
		cx = t[3 * (size_t)j]; cy = t[3 * (size_t)j + 1]; cz = t[3 * (size_t)j + 2];
	}
	__device__ __forceinline__ double dist2(int k, double cx, double cy, double cz) const {
		const int ii = min(first + k * kThreads, n - 1);
		const double dx = sub(q[3 * (size_t)ii], cx), dy = sub(q[3 * (size_t)ii + 1], cy), dz = sub(q[3 * (size_t)ii + 2], cz);
		return dot3(dx, dy, dz, dx, dy, dz);
	}
};

// grid ceil(n_q / kChunk): d_out[i] = min_j |q_i - t_j| for the block's kChunk queries
__global__ void __launch_bounds__(kThreads) k_surface_nearest(const double* __restrict__ q, int n_q, const double* __restrict__ t,
                                                              const float4* __restrict__ t32, int n_t, const unsigned long long* __restrict__ pmax_bits,
                                                              double* __restrict__ d_out) {
	__shared__ float4 s_tile[kTile];
	__shared__ double s_best[kQpt][kThreads];
	__shared__ float s_m[kQpt][kThreads], s_a[kQpt][kThreads];
	const int tid = threadIdx.x, first = blockIdx.x * kChunk + tid;
	const double pmax = __longlong_as_double((long long)*pmax_bits);
	const PointRerank rr{q, t, first, n_q};
#pragma unroll 1
	for (int k = 0; k < kQpt; k++) {
		const int ii = min(first + k * kThreads, n_q - 1);
		const double x = q[3 * (size_t)ii], y = q[3 * (size_t)ii + 1], z = q[3 * (size_t)ii + 2];
		// target min(i, n_t - 1) seeds the running minima (the same index of a set sampled alike lies close by)
		const int js = min(ii, n_t - 1);
		double cx, cy, cz;
		rr.target(js, cx, cy, cz);
		s_best[k][tid] = rr.dist2(k, cx, cy, cz);
		const float4 qf = make_float4((float)x, (float)y, (float)z, 0.f);
		s_tile[k * kThreads + tid] = qf;
		s_a[k][tid] = __double2float_ru(2.0 * kU * (sqrt(x * x + y * y + z * z) + pmax));
		s_m[k][tid] = dist2_f32(qf.x, qf.y, qf.z, t32[js]);
	}
	nearest_scan(t32, n_t, 1.0f, s_tile, s_best, s_m, s_a, rr);
#pragma unroll
	for (int k = 0; k < kQpt; k++) {
		const int i = first + k * kThreads;
		if (i < n_q) d_out[i] = sqrt(s_best[k][tid]);
	}
}

}  // namespace

struct SurfaceState {
	bool ready = false;
	int max_faces = 0, max_samples = 0;
	DevBuf w, cdf, block, status, pts32, pmax;
	PinnedBuf h_status;
};
void StateDeleter::operator()(SurfaceState* s) const { delete s; }

}  // namespace bt

extern "C" int bt_surface_reserve(bt_ctx* ctx, int max_faces, int max_samples) {
	BT_REQUIRE(ctx, BT_ERR_INVALID_ARG, "bt_surface_reserve: ctx is NULL");
	BT_REQUIRE(max_faces >= 1 && max_faces <= kMaxSurfaceFaces && max_samples >= 1 && max_samples <= kMaxSurfaceSamples, BT_ERR_INVALID_ARG,
	           "bt_surface_reserve: max_faces %d / max_samples %d must be in 1..%d / 1..%d", max_faces, max_samples, kMaxSurfaceFaces, kMaxSurfaceSamples);
	SurfaceState* s;
	BT_TRY(take_state(ctx, &bt_ctx::surface, &s));
	const size_t nb = (size_t)(max_faces + kFaceThreads - 1) / kFaceThreads;
	BT_TRY(s->w.alloc(sizeof(double) * (size_t)max_faces));
	BT_TRY(s->cdf.alloc(sizeof(unsigned long long) * (size_t)max_faces));
	BT_TRY(s->block.alloc(sizeof(unsigned long long) * nb));
	BT_TRY(s->status.alloc(sizeof(SampleStatus)));
	BT_TRY(s->pts32.alloc(2 * sizeof(float4) * (size_t)max_samples));
	BT_TRY(s->pmax.alloc(2 * sizeof(unsigned long long)));
	BT_TRY(s->h_status.alloc(sizeof(SampleStatus)));
	s->max_faces = max_faces; s->max_samples = max_samples;
	s->ready = true;
	return BT_OK;
}

extern "C" int bt_mesh_sample(bt_ctx* ctx, const double* verts_dev, int n_verts, const int32_t* faces_dev, int n_faces, int n_samples, uint64_t seed,
                              double* pts_out_dev, void* stream_) {
	BT_REQUIRE(verts_dev && faces_dev && pts_out_dev, BT_ERR_INVALID_ARG, "bt_mesh_sample: NULL argument");
	BT_REQUIRE(n_verts >= 1 && n_faces >= 1 && n_samples >= 1, BT_ERR_INVALID_ARG, "bt_mesh_sample: n_verts %d / n_faces %d / n_samples %d must be >= 1",
	           n_verts, n_faces, n_samples);
	SurfaceState* s;
	BT_TRY(state_of(ctx, &bt_ctx::surface, "bt_mesh_sample", "bt_surface_reserve", &s));
	BT_REQUIRE(n_faces <= s->max_faces && n_samples <= s->max_samples, BT_ERR_CAPACITY, "bt_mesh_sample: %d faces / %d samples exceed the reserved %d / %d",
	           n_faces, n_samples, s->max_faces, s->max_samples);
	cudaStream_t stream = (cudaStream_t)stream_;
	SampleStatus* st = s->status.as<SampleStatus>();
	const int nb = (n_faces + kFaceThreads - 1) / kFaceThreads;
	BT_CUDA(cudaMemsetAsync(st, 0, sizeof(SampleStatus), stream));
	k_face_weight<<<(n_faces + kThreads - 1) / kThreads, kThreads, 0, stream>>>(verts_dev, n_verts, faces_dev, n_faces, s->w.as<double>(), st);
	k_face_cdf<<<nb, kFaceThreads, 0, stream>>>(s->w.as<double>(), n_faces, st, s->cdf.as<unsigned long long>(), s->block.as<unsigned long long>());
	k_face_cdf_top<<<1, kFaceThreads, 0, stream>>>(s->block.as<unsigned long long>(), nb, st);
	k_face_cdf_add<<<nb, kFaceThreads, 0, stream>>>(s->cdf.as<unsigned long long>(), n_faces, s->block.as<unsigned long long>());
	BT_CUDA(cudaGetLastError());
	SampleStatus* h = s->h_status.as<SampleStatus>();
	BT_CUDA(cudaMemcpyAsync(h, st, sizeof(SampleStatus), cudaMemcpyDeviceToHost, stream));
	BT_CUDA(cudaStreamSynchronize(stream));                 // the call's one synchronisation: a bad mesh is refused before the output is touched
	BT_REQUIRE(h->bad == 0, BT_ERR_INVALID_ARG, "bt_mesh_sample: face %d has a vertex index outside [0, %d) or a non-finite vertex", n_faces - h->bad, n_verts);
	BT_REQUIRE(h->total > 0, BT_ERR_INVALID_ARG, "bt_mesh_sample: the mesh's %d faces have no area", n_faces);
	k_mesh_sample<<<(n_samples + kThreads - 1) / kThreads, kThreads, 0, stream>>>(verts_dev, faces_dev, s->cdf.as<unsigned long long>(), n_faces, st,
	                                                                              n_samples, seed, pts_out_dev);
	BT_CUDA(cudaGetLastError());
	return BT_OK;
}

extern "C" int bt_surface_distances(bt_ctx* ctx, const double* a_dev, int n_a, const double* b_dev, int n_b, double* d_ab_out, double* d_ba_out, void* stream_) {
	BT_REQUIRE(a_dev && b_dev && d_ab_out && d_ba_out, BT_ERR_INVALID_ARG, "bt_surface_distances: NULL argument");
	BT_REQUIRE(n_a >= 1 && n_b >= 1, BT_ERR_INVALID_ARG, "bt_surface_distances: n_a %d / n_b %d must be >= 1", n_a, n_b);
	SurfaceState* s;
	BT_TRY(state_of(ctx, &bt_ctx::surface, "bt_surface_distances", "bt_surface_reserve", &s));
	BT_REQUIRE(n_a <= s->max_samples && n_b <= s->max_samples, BT_ERR_CAPACITY, "bt_surface_distances: %d / %d points exceed the reserved %d",
	           n_a, n_b, s->max_samples);
	cudaStream_t stream = (cudaStream_t)stream_;
	float4* a32 = s->pts32.as<float4>();
	float4* b32 = a32 + s->max_samples;
	unsigned long long* pmax = s->pmax.as<unsigned long long>();
	BT_CUDA(cudaMemsetAsync(pmax, 0, 2 * sizeof(unsigned long long), stream));
	k_metrics_prep<<<(n_a + kThreads - 1) / kThreads, kThreads, 0, stream>>>(a_dev, n_a, a32, pmax);
	k_metrics_prep<<<(n_b + kThreads - 1) / kThreads, kThreads, 0, stream>>>(b_dev, n_b, b32, pmax + 1);
	k_surface_nearest<<<(n_a + kChunk - 1) / kChunk, kThreads, 0, stream>>>(a_dev, n_a, b_dev, b32, n_b, pmax + 1, d_ab_out);
	k_surface_nearest<<<(n_b + kChunk - 1) / kChunk, kThreads, 0, stream>>>(b_dev, n_b, a_dev, a32, n_a, pmax, d_ba_out);
	BT_CUDA(cudaGetLastError());
	return BT_OK;
}

// the p-quantile of sorted x: linear interpolation at position p (n - 1), x[lo] + (pos - lo) (x[lo + 1] - x[lo])
static double quantile_sorted(const std::vector<double>& x, double p) {
	const double pos = p * (double)(x.size() - 1);
	const size_t lo = (size_t)pos;
	if (lo + 1 >= x.size()) return x.back();
	return x[lo] + (pos - (double)lo) * (x[lo + 1] - x[lo]);
}

extern "C" int bt_surface_score(const double* d_ab, int n_a, const double* d_ba, int n_b, const double* taus, int n_taus, double* out) {
	BT_REQUIRE(d_ab && d_ba && out && (taus || n_taus == 0), BT_ERR_INVALID_ARG, "bt_surface_score: NULL argument");
	BT_REQUIRE(n_a >= 1 && n_b >= 1 && n_taus >= 0, BT_ERR_INVALID_ARG, "bt_surface_score: n_a %d / n_b %d must be >= 1, n_taus %d >= 0", n_a, n_b, n_taus);
	for (int t = 0; t < n_taus; t++)
		BT_REQUIRE(taus[t] > 0.0 && isfinite(taus[t]), BT_ERR_INVALID_ARG, "bt_surface_score: tau %d (%g) must be positive and finite", t, taus[t]);
	const double* d[2] = {d_ab, d_ba};
	const int n[2] = {n_a, n_b};
	double mean[2], med[2], p95[2];
	for (int s = 0; s < 2; s++) {
		std::vector<double> x(d[s], d[s] + n[s]);
		double sum = 0.0;
		for (int i = 0; i < n[s]; i++) {
			BT_REQUIRE(x[i] >= 0.0 && isfinite(x[i]), BT_ERR_INVALID_ARG, "bt_surface_score: distance %d of %s (%g) must be finite and >= 0", i,
			           s ? "d_ba" : "d_ab", x[i]);
			sum += x[i];
		}
		mean[s] = sum / (double)n[s];
		std::sort(x.begin(), x.end());
		med[s] = quantile_sorted(x, 0.5);
		p95[s] = quantile_sorted(x, 0.95);
	}
	out[0] = mean[0];
	out[1] = mean[1];
	out[2] = (mean[0] + mean[1]) / 2.0;
	out[3] = med[0]; out[4] = p95[0]; out[5] = med[1]; out[6] = p95[1];
	for (int t = 0; t < n_taus; t++) {
		long long c[2] = {0, 0};
		for (int s = 0; s < 2; s++)
			for (int i = 0; i < n[s]; i++) c[s] += d[s][i] < taus[t];
		const double P = (double)c[0] / (double)n_a, R = (double)c[1] / (double)n_b;
		out[7 + 3 * t] = P;
		out[8 + 3 * t] = R;
		out[9 + 3 * t] = P + R > 0.0 ? 2.0 * P * R / (P + R) : 0.0;
	}
	return BT_OK;
}

// ---- mask accuracy: the DAVIS region similarity J and boundary accuracy F per frame (DESIGN.md §3.16) ----------------------------------
// J = |P & G| / |P | G| (1 for an empty union).  F: the boundary maps b(P), b(G) with _seg2bmap's edge rules, the tolerance radius
// r = ceil(bound_th sqrt(H^2 + W^2)), the matches m_P = #{boundary pixels of P with a boundary pixel of G at dx^2 + dy^2 <= r^2} and m_G the
// same the other way, then precision m_P / n_P, recall m_G / n_G and F = 2 P R / (P + R), with the toolkit's rules for empty boundaries.
// One CTA per (frame, band of kMaskBand rows) holds both masks as bit rows in shared memory, 64 pixels to a word (bit j of word c is pixel
// 64 c + j): the band plus r rows above it and r + 1 below, clipped to the image.  The six counts are integers, so summing them per frame
// in any order is exact, and k_mask_final forms J and F from them in float64.
namespace bt {
namespace {

constexpr int kMaskThreads = 256;
constexpr int kMaskBand = 64;                      // rows per CTA
constexpr int kMaxMaskRadius = 64;                 // r: a row is dilated from its two neighbouring words at most
constexpr int kMaskCounts = 6;                     // |P & G|, |P | G|, n_P, n_G, m_P, m_G
constexpr int kMaxMaskBands = 65535;               // grid.y
typedef unsigned long long u64;

__host__ __device__ __forceinline__ int mask_words(int w) { return (w + 63) / 64; }
// shared bit rows of one mask for a band: at most the band, r rows above and r + 1 below
__host__ __device__ __forceinline__ int mask_rows(int h, int r) { return min(kMaskBand + 2 * r + 1, h); }

// bit j set when byte j of x is 0xff (the byte compares of __vcmp*4): the multiply gathers the bytes' low bits into bits 28..31
__device__ __forceinline__ unsigned bytes4(unsigned m) { return ((m & 0x01010101u) * 0x10204080u) >> 28; }
__device__ __forceinline__ unsigned nonzero4(unsigned x) { return bytes4(__vcmpne4(x, 0u)); }
__device__ __forceinline__ unsigned nonzero16(uint4 v) { return nonzero4(v.x) | nonzero4(v.y) << 4 | nonzero4(v.z) << 8 | nonzero4(v.w) << 12; }
// bit j set when byte j of v equals the byte that k4 holds four times (ne: does not equal it)
__device__ __forceinline__ unsigned equal16(uint4 v, unsigned k4) {
	return bytes4(__vcmpeq4(v.x, k4)) | bytes4(__vcmpeq4(v.y, k4)) << 4 | bytes4(__vcmpeq4(v.z, k4)) << 8 | bytes4(__vcmpeq4(v.w, k4)) << 12;
}
__device__ __forceinline__ unsigned differ16(uint4 v, unsigned k4) { return ~equal16(v, k4) & 0xffffu; }

// How pack_row turns block b of a row (16 bytes, aligned) into 16 bits, bit j for byte j.
// The binary masks: the byte is not 0.
struct NonZeroBits {
	__device__ __forceinline__ unsigned operator()(const uint4* blk, int b) const { return nonzero16(__ldg(blk + b)); }
};
// Object k of a label map: the byte equals k (k4 = k times 0x01010101).  With gt set, also the ground-truth byte of the same pixel is not
// the void value: byte j of block b is pixel 16 b + j - d of the row, and that pixel is byte s + j of the ground-truth row's blocks gb, gb + 1
// with gb = b + q, where q (0 or -1) and s (0..15) come from the two rows' offsets in their first blocks.  Only blocks that hold a pixel of
// the ground-truth row are read; a pixel of the row always lies in one.
struct ObjectBits {
	unsigned k4, void4;
	const uint4* gt;                 // the ground-truth row's first block, or NULL: no void
	int q, s, n_gt;                  // n_gt: the blocks that hold a pixel of the ground-truth row
	__device__ __forceinline__ unsigned operator()(const uint4* blk, int b) const {
		unsigned m = equal16(__ldg(blk + b), k4);
		if (gt) {
			const int gb = b + q;
			const unsigned lo = gb >= 0 && gb < n_gt ? differ16(__ldg(gt + gb), void4) : 0u;
			const unsigned hi = s && gb + 1 < n_gt ? differ16(__ldg(gt + gb + 1), void4) : 0u;
			m &= (lo | hi << 16) >> s;
		}
		return m;
	}
};

__device__ __forceinline__ const uint4* first_block(const uint8_t* src) {
	return reinterpret_cast<const uint4*>(reinterpret_cast<uintptr_t>(src) & ~(uintptr_t)15);
}

// One warp packs row `src` (w bytes at any alignment) into dst[0, nw): it reads the whole 16-byte blocks that hold a pixel of the row, one
// per lane, turns each into 16 bits with `bits`, and word c takes the 64 bits that start d = src & 15 bits into blocks 4c .. 4c + 4.  Bits
// past the row's end are 0.
template <class Bits>
__device__ void pack_row(const uint8_t* src, int w, u64* dst, int nw, int lane, const Bits& bits) {
	const uint4* blk = first_block(src);
	const int d = (int)(reinterpret_cast<uintptr_t>(src) & 15);
	const int n_blk = (d + w + 15) >> 4;
	for (int c0 = 0; c0 < nw; c0 += 8) {                // 8 words, 32 blocks (plus the next round's first) per round
		const int k = 4 * c0 + lane;
		const unsigned m = k < n_blk ? bits(blk, k) : 0u;
		const unsigned next = (lane == 31 && k + 1 < n_blk) ? bits(blk, k + 1) : 0u;
		const int i = lane & 7;
		const u64 m0 = __shfl_sync(0xffffffffu, m, 4 * i), m1 = __shfl_sync(0xffffffffu, m, 4 * i + 1);
		const u64 m2 = __shfl_sync(0xffffffffu, m, 4 * i + 2), m3 = __shfl_sync(0xffffffffu, m, 4 * i + 3);
		const unsigned m4a = __shfl_sync(0xffffffffu, m, (4 * i + 4) & 31), m4b = __shfl_sync(0xffffffffu, next, 31);
		const u64 m4 = i == 7 ? m4b : m4a;
		u64 v = m0 | m1 << 16 | m2 << 32 | m3 << 48;
		if (d) v = (v >> d) | (m4 << (64 - d));
		const int c = c0 + i, valid = w - 64 * c;
		if (lane < 8 && c < nw) dst[c] = valid >= 64 ? v : v & ((1ull << valid) - 1);
	}
}

// Pixels of word c of bit row R that have a set pixel of R within h columns (0 <= h <= 64): the 192 bits of words c - 1 .. c + 1 are
// spread h columns one way and then h the other, each by doubling.  Words outside [0, nw) are 0.
__device__ __forceinline__ u64 dilate_word(const u64* R, int c, int nw, int h) {
	u64 lo = c > 0 ? R[c - 1] : 0, mid = R[c], hi = c + 1 < nw ? R[c + 1] : 0;
	if ((lo | mid | hi) == 0) return 0;
	// every bit takes the OR of itself and the h bits above it (steps of at most 32, so no shift reaches 64)
	for (int cover = 1; cover <= h;) {
		const int s = min(cover, h + 1 - cover);
		lo |= (lo >> s) | (mid << (64 - s));
		mid |= (mid >> s) | (hi << (64 - s));
		hi |= hi >> s;
		cover += s;
	}
	// then of itself and the h bits below it
	for (int cover = 1; cover <= h;) {
		const int s = min(cover, h + 1 - cover);
		mid |= (mid << s) | (lo >> (64 - s));
		lo |= lo << s;
		cover += s;
	}
	return mid;
}

__device__ __forceinline__ int isqrt(int n) {
	int v = (int)sqrt((double)n);
	while (v * v > n) v--;
	while ((v + 1) * (v + 1) <= n) v++;
	return v;
}

// Which masks a k_mask_band row scores.  frame(x): the frame of grid row x; pack(): one warp packs row y of that frame's prediction
// (map 0) or ground truth (map 1), given both rows.
// bt_mask_metrics: row x is frame x, foreground is non-zero.
struct BinaryMasks {
	__device__ __forceinline__ int frame(int x) const { return x; }
	__device__ __forceinline__ void pack(int map, int, const uint8_t* p, const uint8_t* g, int w, u64* dst, int nw, int lane) const {
		pack_row(map ? g : p, w, dst, nw, lane, NonZeroBits());
	}
};
// bt_mask_metrics_objects: row x is object k = x % n_objects + 1 of frame x / n_objects; P = (pred == k) & ~V, G = (gt == k), which
// excludes V = (gt == void_value) since void_value is not an object id.
struct ObjectMasks {
	int n_objects, void_value;       // -1: no void
	__device__ __forceinline__ int frame(int x) const { return x / n_objects; }
	__device__ __forceinline__ void pack(int map, int x, const uint8_t* p, const uint8_t* g, int w, u64* dst, int nw, int lane) const {
		ObjectBits bits = {(unsigned)(x % n_objects + 1) * 0x01010101u, (unsigned)void_value * 0x01010101u, nullptr, 0, 0, 0};
		if (map == 0 && void_value >= 0) {
			const int e = (int)(reinterpret_cast<uintptr_t>(g) & 15) - (int)(reinterpret_cast<uintptr_t>(p) & 15);
			bits.gt = first_block(g);
			bits.q = e >> 4;
			bits.s = e & 15;
			bits.n_gt = ((int)(reinterpret_cast<uintptr_t>(g) & 15) + w + 15) >> 4;
		}
		pack_row(map ? g : p, w, dst, nw, lane, bits);
	}
};

// grid (rows, n_bands): block (x, band) writes band_counts[x][band][0..5] for rows [y0, y0 + kMaskBand) of grid row x (Select::frame)
template <class Select>
__global__ void __launch_bounds__(kMaskThreads) k_mask_band(const uint8_t* __restrict__ pred, const uint8_t* __restrict__ gt, int h, int w, int r,
                                                            unsigned* __restrict__ band_counts, Select sel) {
	extern __shared__ u64 s_bits[];                    // [2][n_rows][nw]: the prediction's rows, then the ground truth's
	__shared__ int s_h[2 * kMaxMaskRadius + 1];        // s_h[dy + r] = isqrt(r^2 - dy^2): the disk's half-width on row dy
	__shared__ unsigned s_cnt[kMaskCounts];
	const int f = blockIdx.x, band = blockIdx.y, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
	const size_t frame = (size_t)sel.frame(f);
	const int nw = mask_words(w);
	const int y0 = band * kMaskBand, y1 = min(y0 + kMaskBand, h);
	const int ylo = max(0, y0 - r), yhi = min(h, y1 + r + 1);        // the rows held
	const int n_rows = yhi - ylo, n_brows = min(h, y1 + r) - ylo;      // the first n_brows become boundary rows
	for (int k = tid; k <= 2 * r; k += kMaskThreads) s_h[k] = isqrt(r * r - (k - r) * (k - r));
	if (tid < kMaskCounts) s_cnt[tid] = 0;

	for (int t = warp; t < 2 * n_rows; t += kMaskThreads / 32) {
		const int map = t & 1, row = t >> 1;
		const size_t at = (frame * h + ylo + row) * (size_t)w;
		sel.pack(map, f, pred + at, gt + at, w, s_bits + ((size_t)map * n_rows + row) * nw, nw, lane);
	}
	__syncthreads();

	u64* const P = s_bits;
	u64* const G = s_bits + (size_t)n_rows * nw;
	unsigned inter = 0, uni = 0;
	for (int k = tid; k < (y1 - y0) * nw; k += kMaskThreads) {
		const int i = (y0 - ylo) * nw + k;
		inter += __popcll(P[i] & G[i]);
		uni += __popcll(P[i] | G[i]);
	}

	// The boundary maps, in place: b at (y, x) reads S at (y, x), (y, x + 1), (y + 1, x) and (y + 1, x + 1), all at or after its own word in
	// row-major order.  So each round reads its words before the barrier and writes them after it, and no round reads a word an earlier
	// round has written.
	const int per_map = n_brows * nw;
	for (int base = 0; base < 2 * per_map; base += kMaskThreads) {
		const int k = base + tid;
		const bool mine = k < 2 * per_map;
		u64 b = 0;
		int at = 0;
		if (mine) {
			const int map = k >= per_map, rem = k - map * per_map, row = rem / nw, c = rem - row * nw, y = ylo + row;
			const u64* S = s_bits + (size_t)map * n_rows * nw;
			at = map * n_rows * nw + rem;
			const u64 s = S[rem], e = (s >> 1) | ((c + 1 < nw ? S[rem + 1] : 0) << 63);
			const int n_in = w - 1 - 64 * c;              // pixels of this word left of the last column
			const u64 inner = n_in >= 64 ? ~0ull : n_in <= 0 ? 0 : (1ull << n_in) - 1;
			const u64 last = (n_in >= 0 && n_in < 64) ? 1ull << n_in : 0;
			if (y < h - 1) {
				const u64 so = S[rem + nw], se = (so >> 1) | ((c + 1 < nw ? S[rem + nw + 1] : 0) << 63);
				b = (((s ^ e) | (s ^ so) | (s ^ se)) & inner) | ((s ^ so) & last);
			} else {
				b = (s ^ e) & inner;                        // the last row; its last pixel is the corner, 0
			}
		}
		__syncthreads();
		if (mine) s_bits[at] = b;
		__syncthreads();
	}

	// matches: a boundary word of one map against the other map's boundary rows y - r .. y + r, each dilated by the disk's half-width
	unsigned n_p = 0, n_g = 0, m_p = 0, m_g = 0;
	const int band_words = (y1 - y0) * nw;
	for (int k = tid; k < 2 * band_words; k += kMaskThreads) {
		const int map = k >= band_words, rem = k - map * band_words, row = (y0 - ylo) + rem / nw, c = rem % nw;
		const u64* Q = s_bits + (size_t)map * n_rows * nw;
		const u64* O = s_bits + (size_t)(1 - map) * n_rows * nw;
		const u64 q = Q[(size_t)row * nw + c];
		if (!q) continue;
		const int dy0 = max(-r, -row), dy1 = min(r, n_brows - 1 - row);
		u64 hit = 0;
		for (int dy = dy0; dy <= dy1 && (hit & q) != q; dy++) hit |= dilate_word(O + (size_t)(row + dy) * nw, c, nw, s_h[dy + r]);
		const unsigned n = __popcll(q), m = __popcll(hit & q);
		if (map) { n_g += n; m_g += m; }
		else { n_p += n; m_p += m; }
	}

	const unsigned v[kMaskCounts] = {inter, uni, n_p, n_g, m_p, m_g};
#pragma unroll
	for (int i = 0; i < kMaskCounts; i++) {
		const unsigned s = __reduce_add_sync(0xffffffffu, v[i]);
		if (lane == 0 && s) atomicAdd(&s_cnt[i], s);
	}
	__syncthreads();
	if (tid < kMaskCounts) band_counts[((size_t)f * gridDim.y + band) * kMaskCounts + tid] = s_cnt[tid];
}

// one thread per grid row of k_mask_band: the bands' counts in band order, then J and F in float64
__global__ void k_mask_final(const unsigned* __restrict__ band_counts, int n_bands, int n_frames, double* __restrict__ j_out,
                             double* __restrict__ f_out, long long* __restrict__ counts_out) {
	const int f = blockIdx.x * blockDim.x + threadIdx.x;
	if (f >= n_frames) return;
	long long c[kMaskCounts] = {0, 0, 0, 0, 0, 0};
	for (int b = 0; b < n_bands; b++)
		for (int i = 0; i < kMaskCounts; i++) c[i] += band_counts[((size_t)f * n_bands + b) * kMaskCounts + i];
	const long long inter = c[0], uni = c[1], n_p = c[2], n_g = c[3], m_p = c[4], m_g = c[5];
	double precision, recall;
	if (n_p == 0 && n_g > 0) { precision = 1.0; recall = 0.0; }
	else if (n_p > 0 && n_g == 0) { precision = 0.0; recall = 1.0; }
	else if (n_p == 0 && n_g == 0) { precision = 1.0; recall = 1.0; }
	else { precision = __ddiv_rn((double)m_p, (double)n_p); recall = __ddiv_rn((double)m_g, (double)n_g); }
	const double pr = add(precision, recall);
	j_out[f] = uni == 0 ? 1.0 : __ddiv_rn((double)inter, (double)uni);
	f_out[f] = pr == 0.0 ? 0.0 : __ddiv_rn(mul(mul(2.0, precision), recall), pr);
	if (counts_out)
		for (int i = 0; i < kMaskCounts; i++) counts_out[(size_t)f * kMaskCounts + i] = c[i];
}

// bytes of shared bit rows a band needs
size_t mask_smem(int h, int w, int r) { return 2 * sizeof(u64) * (size_t)mask_rows(h, r) * (size_t)mask_words(w); }

}  // namespace

struct MaskState {
	bool ready = false;
	int max_frames = 0, max_h = 0, max_w = 0;
	DevBuf band;
};
void StateDeleter::operator()(MaskState* s) const { delete s; }

}  // namespace bt

extern "C" int bt_mask_reserve(bt_ctx* ctx, int max_frames, int max_h, int max_w) {
	BT_REQUIRE(ctx, BT_ERR_INVALID_ARG, "bt_mask_reserve: ctx is NULL");
	BT_REQUIRE(max_frames >= 1 && max_h >= 1 && max_w >= 1, BT_ERR_INVALID_ARG, "bt_mask_reserve: max_frames %d / max_h %d / max_w %d must be >= 1",
	           max_frames, max_h, max_w);
	const int max_bands = (max_h + kMaskBand - 1) / kMaskBand;
	BT_REQUIRE(max_bands <= kMaxMaskBands, BT_ERR_INVALID_ARG, "bt_mask_reserve: max_h %d > %d", max_h, kMaxMaskBands * kMaskBand);
	BT_CUDA(cudaSetDevice(ctx->device));
	int optin = 0;
	cudaFuncAttributes fa, fo;
	BT_CUDA(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, ctx->device));
	BT_CUDA(cudaFuncGetAttributes(&fa, k_mask_band<BinaryMasks>));
	BT_CUDA(cudaFuncGetAttributes(&fo, k_mask_band<ObjectMasks>));
	const size_t smem = mask_smem(max_h, max_w, kMaxMaskRadius), room = (size_t)optin - std::max(fa.sharedSizeBytes, fo.sharedSizeBytes);
	BT_REQUIRE(smem <= room, BT_ERR_INVALID_ARG,
	           "bt_mask_reserve: a band of %d x %d masks needs %zu bytes of shared memory at r = %d, the device has %zu per block", max_h, max_w, smem,
	           kMaxMaskRadius, room);
	MaskState* s;
	BT_TRY(take_state(ctx, &bt_ctx::mask, &s));
	// the kernel's limit is the device's, not this reservation's: it is one setting for every context in the process
	BT_CUDA(cudaFuncSetAttribute(k_mask_band<BinaryMasks>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)room));
	BT_CUDA(cudaFuncSetAttribute(k_mask_band<ObjectMasks>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)room));
	BT_TRY(s->band.alloc(sizeof(unsigned) * kMaskCounts * (size_t)max_bands * (size_t)max_frames));
	s->max_frames = max_frames; s->max_h = max_h; s->max_w = max_w;
	s->ready = true;
	return BT_OK;
}

extern "C" int bt_mask_metrics(bt_ctx* ctx, const uint8_t* pred_dev, const uint8_t* gt_dev, int n_frames, int h, int w, double bound_th,
                               double* j_dev, double* f_dev, int64_t* counts_dev, void* stream_) {
	BT_REQUIRE(pred_dev && gt_dev && j_dev && f_dev, BT_ERR_INVALID_ARG, "bt_mask_metrics: NULL argument");
	BT_REQUIRE(n_frames >= 1 && h >= 1 && w >= 1, BT_ERR_INVALID_ARG, "bt_mask_metrics: n_frames %d / h %d / w %d must be >= 1", n_frames, h, w);
	BT_REQUIRE(bound_th > 0.0 && bound_th < 1.0, BT_ERR_INVALID_ARG, "bt_mask_metrics: bound_th %g must be in (0, 1)", bound_th);
	const double rr = ceil(bound_th * sqrt((double)h * h + (double)w * w));
	BT_REQUIRE(rr <= kMaxMaskRadius, BT_ERR_INVALID_ARG, "bt_mask_metrics: the tolerance radius %.0f of bound_th %g at %d x %d exceeds %d", rr, bound_th, h, w,
	           kMaxMaskRadius);
	const int r = (int)rr;
	MaskState* s;
	BT_TRY(state_of(ctx, &bt_ctx::mask, "bt_mask_metrics", "bt_mask_reserve", &s));
	BT_REQUIRE(n_frames <= s->max_frames && h <= s->max_h && w <= s->max_w, BT_ERR_CAPACITY,
	           "bt_mask_metrics: %d frames of %d x %d exceed the reserved %d of %d x %d", n_frames, h, w, s->max_frames, s->max_h, s->max_w);
	cudaStream_t stream = (cudaStream_t)stream_;
	const int n_bands = (h + kMaskBand - 1) / kMaskBand;
	unsigned* band = s->band.as<unsigned>();
	k_mask_band<<<dim3(n_frames, n_bands), kMaskThreads, mask_smem(h, w, r), stream>>>(pred_dev, gt_dev, h, w, r, band, BinaryMasks());
	k_mask_final<<<(n_frames + 127) / 128, 128, 0, stream>>>(band, n_bands, n_frames, j_dev, f_dev, reinterpret_cast<long long*>(counts_dev));
	BT_CUDA(cudaGetLastError());
	return BT_OK;
}

extern "C" int bt_mask_metrics_objects(bt_ctx* ctx, const uint8_t* pred_dev, const uint8_t* gt_dev, int n_frames, int h, int w, int n_objects,
                                       int void_value, double bound_th, double* j_dev, double* f_dev, int64_t* counts_dev, void* stream_) {
	BT_REQUIRE(pred_dev && gt_dev && j_dev && f_dev, BT_ERR_INVALID_ARG, "bt_mask_metrics_objects: NULL argument");
	BT_REQUIRE(n_frames >= 1 && h >= 1 && w >= 1, BT_ERR_INVALID_ARG, "bt_mask_metrics_objects: n_frames %d / h %d / w %d must be >= 1", n_frames,
	           h, w);
	BT_REQUIRE(n_objects >= 1 && n_objects <= 255, BT_ERR_INVALID_ARG, "bt_mask_metrics_objects: n_objects %d outside [1, 255]", n_objects);
	BT_REQUIRE(void_value == -1 || (void_value >= 0 && void_value <= 255 && !(void_value >= 1 && void_value <= n_objects)), BT_ERR_INVALID_ARG,
	           "bt_mask_metrics_objects: void_value %d must be -1 (no void) or in [0, 255] outside the object ids 1..%d", void_value, n_objects);
	BT_REQUIRE(bound_th > 0.0 && bound_th < 1.0, BT_ERR_INVALID_ARG, "bt_mask_metrics_objects: bound_th %g must be in (0, 1)", bound_th);
	const double rr = ceil(bound_th * sqrt((double)h * h + (double)w * w));
	BT_REQUIRE(rr <= kMaxMaskRadius, BT_ERR_INVALID_ARG, "bt_mask_metrics_objects: the tolerance radius %.0f of bound_th %g at %d x %d exceeds %d", rr,
	           bound_th, h, w, kMaxMaskRadius);
	const int r = (int)rr;
	MaskState* s;
	BT_TRY(state_of(ctx, &bt_ctx::mask, "bt_mask_metrics_objects", "bt_mask_reserve", &s));
	const long long rows = (long long)n_frames * n_objects;
	BT_REQUIRE(rows <= s->max_frames && h <= s->max_h && w <= s->max_w, BT_ERR_CAPACITY,
	           "bt_mask_metrics_objects: %d frames x %d objects = %lld rows of %d x %d exceed the reserved %d of %d x %d", n_frames, n_objects, rows, h, w,
	           s->max_frames, s->max_h, s->max_w);
	cudaStream_t stream = (cudaStream_t)stream_;
	const int n_bands = (h + kMaskBand - 1) / kMaskBand;
	unsigned* band = s->band.as<unsigned>();
	k_mask_band<<<dim3((unsigned)rows, n_bands), kMaskThreads, mask_smem(h, w, r), stream>>>(pred_dev, gt_dev, h, w, r, band,
	                                                                                          ObjectMasks{n_objects, void_value});
	k_mask_final<<<(unsigned)((rows + 127) / 128), 128, 0, stream>>>(band, n_bands, (int)rows, j_dev, f_dev, reinterpret_cast<long long*>(counts_dev));
	BT_CUDA(cudaGetLastError());
	return BT_OK;
}

// db_statistics of one sequence's per-frame values: the mean (numpy's pairwise sum), the recall mean(x > 0.5), and the decay, the mean of
// the first of four bins minus that of the last, bin i = x[ids[i] .. ids[i + 1]] with ids = round_half_even(linspace(1, n, 5) + 1e-10) - 1.
static void db_statistics(const double* x, int n, double* mean, double* recall, double* decay) {
	*mean = np_pairwise_sum(x, n) / (double)n;
	int above = 0;
	for (int i = 0; i < n; i++) above += x[i] > 0.5;
	*recall = (double)above / (double)n;
	long long ids[5];
	const double step = (double)(n - 1) / 4.0;
	for (int i = 0; i < 5; i++) {
		const double at = i < 4 ? (double)i * step + 1.0 : (double)n;      // numpy's linspace: its last point is exactly `stop`
		ids[i] = (long long)nearbyint(at + 1e-10) - 1;                     // round half to even, the default rounding mode
	}
	const double first = np_pairwise_sum(x + ids[0], (size_t)(ids[1] + 1 - ids[0])) / (double)(ids[1] + 1 - ids[0]);
	const double last = np_pairwise_sum(x + ids[3], (size_t)(ids[4] + 1 - ids[3])) / (double)(ids[4] + 1 - ids[3]);
	*decay = first - last;
}

extern "C" int bt_mask_score(const double* j, const double* f, int n, double* out) {
	BT_REQUIRE(j && f && out, BT_ERR_INVALID_ARG, "bt_mask_score: NULL argument");
	BT_REQUIRE(n >= 1, BT_ERR_INVALID_ARG, "bt_mask_score: n %d must be >= 1", n);
	double jm, jr, jd, fm, fr, fd;
	db_statistics(j, n, &jm, &jr, &jd);
	db_statistics(f, n, &fm, &fr, &fd);
	out[0] = (jm + fm) / 2.0;
	out[1] = jm; out[2] = jr; out[3] = jd;
	out[4] = fm; out[5] = fr; out[6] = fd;
	return BT_OK;
}
