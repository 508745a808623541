/*
 * oracle/solver_oracle.c — TEST INFRASTRUCTURE ONLY.
 *
 * CPU restatement ("Oracle A", SURVEY.md §7 step 2 / §8c) of the reference's Gauss-Newton x PCG pose-graph solve:
 * OptimizerGpu::optimizeFrames -> CUDACache -> SBA::align -> CUDASolverBundling::solve -> solveBundlingStub.
 * The reference has NO CPU optimizer (SURVEY.md §0 D5); this file restates, statement by statement and in a fixed
 * sequential summation order, what the reference's CUDA kernels compute.  Only tests/, __graft_entry__.smoke() and
 * bench.py's cpu_baseline / --impl reference legs may load it.  The product path never does.
 *
 * Parity status: the reference ships no tests or golden vectors for this path (SURVEY.md §4), so this restatement is
 * pinned against the reference's own kernels compiled verbatim (oracle/_ref, "Oracle B", run on the GPU box:
 * tests/test_solver_gpu.py::test_oracle_a_vs_reference_kernels) — not against published vectors.
 *
 * Build:  gcc -O2 -fPIC -shared [-DORACLE_REAL=double] -ffp-contract=off  -> liboracle_f32.so / liboracle_f64.so
 * `real` is the arithmetic type: float = literal restatement; double = same algorithm at higher precision
 * (used to bound how much of a CUDA-vs-oracle difference is plain fp32 rounding).
 *
 * Reference citations are relative to /root/reference/src/cuda/.
 */
#include <math.h>
#include <stdlib.h>
#include <string.h>
#include <stdint.h>

#ifndef ORACLE_REAL
#define ORACLE_REAL float
#endif
typedef ORACLE_REAL real;

#define R_(x) ((real)(x))
#define FLOAT_EPSILON R_(0.000001)        /* SolverUtil.h:10 */
#define ONE_TWENTIETH R_(0.05)            /* Solver/LieDerivUtil.h:14 */
#define ONE_SIXTH R_(0.16666667)          /* Solver/LieDerivUtil.h:15 */

static real rsqrt_(real x) { return (real)sqrt((double)x); }
static real rsin(real x) { return (real)sin((double)x); }
static real rcos(real x) { return (real)cos((double)x); }
static real rasin(real x) { return (real)asin((double)x); }
static real racos(real x) { return (real)acos((double)x); }

typedef struct { uint32_t imgIdx_i, imgIdx_j; float pos_i[3]; float pos_j[3]; } EntryJ; /* SIFTImageManager.h:44-59 */

typedef struct {
	int num_iter_outer;        /* bundle.num_iter_outter  (Solver/CUDASolverBundling.cpp:193) */
	int num_iter_inner;        /* bundle.num_iter_inner   (:210) */
	float robust_delta;        /* bundle.robust_delta     (:214) */
	float image_downscale;     /* bundle.image_downscale  (LossGPU.cu:55) */
	float dense_dist_thresh;   /* p2p.max_dist            (CUDASolverBundling.cpp:93) */
	float dense_cos_normal_thresh; /* cos(p2p.max_normal_angle) (:94) */
	float depth_min;           /* 0.1   (:97) */
	float depth_max;           /* 9999  (:98) */
	float w_sparse;            /* 1     (SBA.cpp:28) */
	float w_dense;             /* 1     (SBA.cpp:30) */
} oracle_params;

typedef struct { real m[16]; } mat4; /* row-major like float4x4 (cuda_SimpleMatrixUtil.h:853) */
typedef struct { real x, y, z; } vec3;

static vec3 v3(real x, real y, real z) { vec3 v = { x, y, z }; return v; }
static vec3 vadd(vec3 a, vec3 b) { return v3(a.x + b.x, a.y + b.y, a.z + b.z); }
static vec3 vsub(vec3 a, vec3 b) { return v3(a.x - b.x, a.y - b.y, a.z - b.z); }
static vec3 vscale(vec3 a, real s) { return v3(a.x * s, a.y * s, a.z * s); }
static real vdot(vec3 a, vec3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
static vec3 vcross(vec3 a, vec3 b) { return v3(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x); }
static real vlen(vec3 a) { return rsqrt_(vdot(a, a)); }

#define M(A, r, c) ((A).m[(r) * 4 + (c)])

static mat4 mat_identity(void) { mat4 A; memset(&A, 0, sizeof A); M(A,0,0)=M(A,1,1)=M(A,2,2)=M(A,3,3)=1; return A; }
static mat4 mat_mul(const mat4* A, const mat4* B) {
	mat4 C;
	for (int r = 0; r < 4; r++) for (int c = 0; c < 4; c++) {
		real s = 0;
		for (int k = 0; k < 4; k++) s += M(*A, r, k) * M(*B, k, c);
		M(C, r, c) = s;
	}
	return C;
}
/* float4x4 * float3 assumes w = 1 (cuda_SimpleMatrixUtil.h:935-942) */
static vec3 mat_mul_p(const mat4* A, vec3 v) {
	return v3(M(*A,0,0)*v.x + M(*A,0,1)*v.y + M(*A,0,2)*v.z + M(*A,0,3) * R_(1),
	          M(*A,1,0)*v.x + M(*A,1,1)*v.y + M(*A,1,2)*v.z + M(*A,1,3) * R_(1),
	          M(*A,2,0)*v.x + M(*A,2,1)*v.y + M(*A,2,2)*v.z + M(*A,2,3) * R_(1));
}
/* general 4x4 inverse by cofactors, like float4x4::getInverse (cuda_SimpleMatrixUtil.h:978-1100) */
static real det3(real a, real b, real c, real d, real e, real f, real g, real h, real i) {
	return a * (e * i - f * h) - b * (d * i - f * g) + c * (d * h - e * g);
}
static mat4 mat_inverse(const mat4* A) {
	mat4 cof;
	for (int r = 0; r < 4; r++) for (int c = 0; c < 4; c++) {
		real s[9]; int n = 0;
		for (int rr = 0; rr < 4; rr++) if (rr != r) for (int cc = 0; cc < 4; cc++) if (cc != c) s[n++] = M(*A, rr, cc);
		real d = det3(s[0], s[1], s[2], s[3], s[4], s[5], s[6], s[7], s[8]);
		M(cof, r, c) = ((r + c) & 1) ? -d : d;
	}
	real det = 0;
	for (int c = 0; c < 4; c++) det += M(*A, 0, c) * M(cof, 0, c);
	real detr = R_(1) / det;
	mat4 inv;
	for (int r = 0; r < 4; r++) for (int c = 0; c < 4; c++) M(inv, r, c) = M(cof, c, r) * detr;
	return inv;
}

/* ---- se(3) <-> SE(3): Solver/LieDerivUtil.h:17-194 ---- */
static void rodrigues_so3_exp(vec3 w, real A, real B, real R[9]) { /* :17-44 */
	const real wx2 = w.x * w.x, wy2 = w.y * w.y, wz2 = w.z * w.z;
	R[0] = R_(1) - B * (wy2 + wz2);
	R[4] = R_(1) - B * (wx2 + wz2);
	R[8] = R_(1) - B * (wx2 + wy2);
	real a = A * w.z, b = B * (w.x * w.y);
	R[1] = b - a; R[3] = b + a;
	a = A * w.y; b = B * (w.x * w.z);
	R[2] = b + a; R[6] = b - a;
	a = A * w.x; b = B * (w.y * w.z);
	R[5] = b - a; R[7] = b + a;
}
static void exp_rotation(vec3 w, real R[9]) { /* :46-70 */
	const real theta_sq = vdot(w, w);
	const real theta = rsqrt_(theta_sq);
	real A, B;
	if (theta_sq < R_(1e-8)) { A = R_(1) - ONE_SIXTH * theta_sq; B = R_(0.5); }
	else if (theta_sq < R_(1e-6)) {
		B = R_(0.5) - R_(0.25) * ONE_SIXTH * theta_sq;
		A = R_(1) - theta_sq * ONE_SIXTH * (R_(1) - ONE_TWENTIETH * theta_sq);
	} else {
		const real inv_theta = R_(1) / theta;
		A = rsin(theta) * inv_theta;
		B = (R_(1) - rcos(theta)) * (inv_theta * inv_theta);
	}
	rodrigues_so3_exp(w, A, B, R);
}
static vec3 ln_rotation(const real R[9]) { /* :72-124 */
	vec3 result;
	const real cos_angle = (R[0] + R[4] + R[8] - R_(1)) * R_(0.5);
	result.x = (R[7] - R[5]) * R_(0.5);
	result.y = (R[2] - R[6]) * R_(0.5);
	result.z = (R[3] - R[1]) * R_(0.5);
	real sin_angle_abs = vlen(result);
	if (cos_angle > R_(0.70710678118654752440)) {
		if (sin_angle_abs > 0) result = vscale(result, rasin(sin_angle_abs) / sin_angle_abs);
	} else if (cos_angle > -R_(0.70710678118654752440)) {
		real angle = racos(cos_angle);
		result = vscale(result, angle / sin_angle_abs);
	} else {
		const real angle = R_(3.14159265358979323846) - rasin(sin_angle_abs);
		const real d0 = R[0] - cos_angle, d1 = R[4] - cos_angle, d2 = R[8] - cos_angle;
		vec3 r2;
		if (fabs((double)d0) > fabs((double)d1) && fabs((double)d0) > fabs((double)d2)) {
			r2.x = d0; r2.y = (R[3] + R[1]) * R_(0.5); r2.z = (R[2] + R[6]) * R_(0.5);
		} else if (fabs((double)d1) > fabs((double)d2)) {
			r2.x = (R[3] + R[1]) * R_(0.5); r2.y = d1; r2.z = (R[7] + R[5]) * R_(0.5);
		} else {
			r2.x = (R[2] + R[6]) * R_(0.5); r2.y = (R[7] + R[5]) * R_(0.5); r2.z = d2;
		}
		if (vdot(r2, result) < 0) r2 = vscale(r2, R_(-1));
		result = vscale(r2, angle / vlen(r2));
	}
	return result;
}
static void matrixToPose(const mat4* T, vec3* rot, vec3* trans) { /* :126-148 */
	real R[9] = { M(*T,0,0), M(*T,0,1), M(*T,0,2), M(*T,1,0), M(*T,1,1), M(*T,1,2), M(*T,2,0), M(*T,2,1), M(*T,2,2) };
	const vec3 t = v3(M(*T,0,3), M(*T,1,3), M(*T,2,3));
	*rot = ln_rotation(R);
	const real theta = vlen(*rot);
	real shtot = R_(0.5);
	if (theta > R_(0.00001)) shtot = rsin(theta * R_(0.5)) / theta;
	real H[9];
	exp_rotation(vscale(*rot, R_(-0.5)), H);
	vec3 tr = v3(H[0]*t.x + H[1]*t.y + H[2]*t.z, H[3]*t.x + H[4]*t.y + H[5]*t.z, H[6]*t.x + H[7]*t.y + H[8]*t.z);
	if (theta > R_(0.001)) tr = vsub(tr, vscale(*rot, vdot(t, *rot) * (R_(1) - R_(2) * shtot) / vdot(*rot, *rot)));
	else tr = vsub(tr, vscale(*rot, vdot(t, *rot) / R_(24)));
	*trans = vscale(tr, R_(1) / (R_(2) * shtot));
}
static mat4 poseToMatrix(vec3 rot, vec3 trans) { /* :150-194 */
	mat4 T = mat_identity();
	const real theta_sq = vdot(rot, rot);
	const real theta = rsqrt_(theta_sq);
	real A, B;
	vec3 cr = vcross(rot, trans), translation;
	if (theta_sq < R_(1e-8)) {
		A = R_(1) - ONE_SIXTH * theta_sq; B = R_(0.5);
		translation = vadd(trans, vscale(cr, R_(0.5)));
	} else {
		real C;
		if (theta_sq < R_(1e-6)) {
			C = ONE_SIXTH * (R_(1) - ONE_TWENTIETH * theta_sq);
			A = R_(1) - theta_sq * C;
			B = R_(0.5) - R_(0.25) * ONE_SIXTH * theta_sq;
		} else {
			const real inv_theta = R_(1) / theta;
			A = rsin(theta) * inv_theta;
			B = (R_(1) - rcos(theta)) * (inv_theta * inv_theta);
			C = (R_(1) - A) * (inv_theta * inv_theta);
		}
		vec3 w_cross = vcross(rot, cr);
		translation = vadd(vadd(trans, vscale(cr, B)), vscale(w_cross, C));
	}
	real R[9];
	rodrigues_so3_exp(rot, A, B, R);
	for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) M(T, r, c) = R[r * 3 + c];
	M(T,0,3) = translation.x; M(T,1,3) = translation.y; M(T,2,3) = translation.z;
	return T;
}

/* ---- Huber: Solver/SolverBundlingUtil.h:24-39 (only rho.y, the weight, is consumed) ---- */
static real huber_weight(real e, real delta) {
	real dsqr = delta * delta;
	if (e <= dsqr) return R_(1);
	double sqrte = sqrt((double)e); /* the reference promotes to double here (:34) */
	return (real)((double)delta / sqrte);
}

/* ---- quarter-resolution frame cache: CUDACache.cpp:14-38,76-88 + CUDAImageUtil.cu:50-99,310-326 ---- */
typedef struct {
	int w, h;               /* W/downscale, H/downscale */
	real fx, fy, cx, cy;    /* rescaled intrinsics (CUDACache.cpp:20-24) */
	real* campos;           /* [N][h*w][4]  (x,y,z,1) or zeros */
	real* normal;           /* [N][h*w][4] */
} frame_cache;

static void cache_build(frame_cache* fc, int N, int H, int W, const float* depth, const float* normal,
                        float fx, float fy, float cx, float cy, float downscale) {
	fc->w = (int)(W / downscale); fc->h = (int)(H / downscale);      /* LossGPU.cu:56-57 */
	const int w = fc->w, h = fc->h;
	fc->fx = (real)fx * ((real)w / (real)W);
	fc->fy = (real)fy * ((real)h / (real)H);
	fc->cx = (real)cx * ((real)(w - 1) / (real)(W - 1));
	fc->cy = (real)cy * ((real)(h - 1) / (real)(H - 1));
	fc->campos = (real*)calloc((size_t)N * w * h * 4, sizeof(real));
	fc->normal = (real*)calloc((size_t)N * w * h * 4, sizeof(real));
	/* inverse of the FULL-resolution intrinsics (m_inputIntrinsicsInv, CUDACache.cpp:32-33), analytic form */
	const real ifx = R_(1) / (real)fx, ify = R_(1) / (real)fy;
	const real icx = -(real)cx / (real)fx, icy = -(real)cy / (real)fy;
	const real scaleW = (real)(float)((float)(W - 1) / (float)(w - 1));    /* CUDAImageUtil.cu:57-58: float */
	const real scaleH = (real)(float)((float)(H - 1) / (float)(h - 1));
	for (int f = 0; f < N; f++) for (int y = 0; y < h; y++) for (int x = 0; x < w; x++) {
		const unsigned xi = (unsigned)((float)x * (float)scaleW + 0.5f);
		const unsigned yi = (unsigned)((float)y * (float)scaleH + 0.5f);
		if (xi >= (unsigned)W || yi >= (unsigned)H) continue;
		const size_t src = (size_t)f * H * W + (size_t)yi * W + xi, dst = ((size_t)f * h * w + (size_t)y * w + x) * 4;
		const real d = (real)depth[src];
		if (d >= R_(0.1)) { /* CUDAImageUtil.cu:319-323: K^-1 * (x d, y d, d, d), z := w component */
			fc->campos[dst + 0] = ifx * ((real)xi * d) + icx * d;
			fc->campos[dst + 1] = ify * ((real)yi * d) + icy * d;
			fc->campos[dst + 2] = d;
			fc->campos[dst + 3] = R_(1);
		}
		for (int k = 0; k < 4; k++) fc->normal[dst + k] = (real)normal[src * 4 + k];
	}
}
static void cache_free(frame_cache* fc) { free(fc->campos); free(fc->normal); }

/* bilinearInterpolationFloat4 (Solver/ICPUtil.h:83-110). Invalid texels are ZEROS, never MINF, in this fork
 * (SURVEY.md Q6) so every in-bounds tap contributes; the unsigned compare drops taps at -1. */
static int bilinear4(real x, real y, const real* img, int w, int h, real out[4]) {
	const int x0 = (int)floor((double)x), y0 = (int)floor((double)y);
	const real alpha = x - (real)x0, beta = y - (real)y0;
	const int px[4] = { x0, x0 + 1, x0, x0 + 1 }, py[4] = { y0, y0, y0 + 1, y0 + 1 };
	real s0[4] = { 0, 0, 0, 0 }, s1[4] = { 0, 0, 0, 0 }, w0 = 0, w1 = 0;
	for (int t = 0; t < 4; t++) {
		if ((unsigned)px[t] < (unsigned)w && (unsigned)py[t] < (unsigned)h) {
			const real* v = img + ((size_t)py[t] * w + px[t]) * 4;
			const real wt = (t & 1) ? alpha : (R_(1) - alpha);
			real* s = (t < 2) ? s0 : s1;
			for (int k = 0; k < 4; k++) s[k] += wt * v[k];
			if (t < 2) w0 += wt; else w1 += wt;
		}
	}
	real ss[4] = { 0, 0, 0, 0 }, ww = 0;
	if (w0 > 0) { for (int k = 0; k < 4; k++) ss[k] += (R_(1) - beta) * (s0[k] / w0); ww += (R_(1) - beta); }
	if (w1 > 0) { for (int k = 0; k < 4; k++) ss[k] += beta * (s1[k] / w1); ww += beta; }
	if (ww > 0) { for (int k = 0; k < 4; k++) out[k] = ss[k] / ww; return 1; }
	return 0; /* reference returns MINF -> every later test fails */
}

/* evalLie_derivI / evalLie_derivJ: Solver/LieDerivUtil.h:228-273, restated literally (dense j0*j1 product). */
static void evalLie_derivI(const mat4* A, const mat4* D, vec3 p, real jac[3][6]) {
	real j0[3][12], j1[12][6];
	memset(j0, 0, sizeof j0); memset(j1, 0, sizeof j1);
	const mat4 T = mat_mul(A, D);
	const real pt[3] = { p.x - M(T,0,3), p.y - M(T,1,3), p.z - M(T,2,3) };
	for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) j0[r][3 * r + c] = pt[c];
	for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) { j0[r][c + 9] = -M(T, c, r); j1[r + 9][c] = M(*A, r, c); }
	for (int k = 0; k < 4; k++) {
		const real v[3] = { M(*D,0,k), M(*D,1,k), M(*D,2,k) };
		const real S[3][3] = { { 0, -v[2], v[1] }, { v[2], 0, -v[0] }, { -v[1], v[0], 0 } }; /* :196-206 */
		for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) {
			real s = 0;
			for (int q = 0; q < 3; q++) s += M(*A, r, q) * S[q][c];
			j1[3 * k + r][3 + c] = s * R_(-1);
		}
	}
	for (int r = 0; r < 3; r++) for (int c = 0; c < 6; c++) {
		real s = 0;
		for (int k = 0; k < 12; k++) s += j0[r][k] * j1[k][c];
		jac[r][c] = s;
	}
}
static void evalLie_derivJ(const mat4* A, const mat4* D, vec3 p, real jac[3][6]) {
	const vec3 dr1 = v3(M(*D,0,0), M(*D,0,1), M(*D,0,2)), dr2 = v3(M(*D,1,0), M(*D,1,1), M(*D,1,2)), dr3 = v3(M(*D,2,0), M(*D,2,1), M(*D,2,2));
	const real dtx = M(*D,0,3), dty = M(*D,1,3), dtz = M(*D,2,3);
	real J[3][6] = { { 1, 0, 0, 0, vdot(p, dr3) + dtz, -(vdot(p, dr2) + dty) },
	                 { 0, 1, 0, -(vdot(p, dr3) + dtz), 0, vdot(p, dr1) + dtx },
	                 { 0, 0, 1, vdot(p, dr2) + dty, -(vdot(p, dr1) + dtx), 0 } };
	for (int r = 0; r < 3; r++) for (int c = 0; c < 6; c++) {
		real s = 0;
		for (int k = 0; k < 3; k++) s += M(*A, r, k) * J[k][c];
		jac[r][c] = s;
	}
}

/* ---- dense term: Solver/SolverBundling.cu:129-229 (BuildDenseSystem_Kernel<true,false>), findDenseCorr
 * (SolverBundlingDenseUtil.h:78-110), addToLocalSystem (:217-285), FlipJtJ_Kernel (SolverBundling.cu:49-58) ---- */
/* Optional outputs of build_dense_system beyond the system itself (all NULL for the solve).
 * JtJ_abs / Jtr_abs: the same sums over |term| (what a per-entry float tolerance scales with).
 * margin [n_pairs][w*h]: per (pair, source pixel) the smallest relative distance of any gate quantity to its decision boundary,
 *   over the gates the pixel reached (all of them when accepted); +1 when the source pixel has no valid depth.  Each distance is
 *   divided by the magnitude its float32 rounding error scales with: depths by the depth, the projected pixel position by the image
 *   width / height, the point distance by the length of the transformed source point; the normal cosine is already O(1).
 * accepted [n_pairs][w*h]: 1 when the pixel passed every gate.
 * contrib [n_pairs][w*h]: weight * (|J_i|^2 + |J_j|^2) of an accepted pixel: what it adds to the traces of the pair's diagonal blocks. */
typedef struct { real* JtJ_abs; real* Jtr_abs; float* margin; unsigned char* accepted; float* contrib; int flip; } dense_extra;

static real rel_gap(real v, real edge, real scale) { return (real)fabs((double)(v - edge)) / scale; }
static real rmin(real a, real b) { return a < b ? a : b; }

static void build_dense_system(const frame_cache* fc, int N, const mat4* T, const mat4* Tinv,
                               const uint32_t* pairs, int n_pairs, const oracle_params* prm,
                               real* JtJ /*[6N][6N]*/, real* Jtr /*[6N]*/, int* n_found_per_pair, const dense_extra* ex) {
	const int dim = 6 * N, w = fc->w, h = fc->h, npix = w * h;
	memset(JtJ, 0, sizeof(real) * dim * dim);
	memset(Jtr, 0, sizeof(real) * dim);
	real* JtJa = ex ? ex->JtJ_abs : NULL;
	real* Jtra = ex ? ex->Jtr_abs : NULL;
	if (JtJa) memset(JtJa, 0, sizeof(real) * dim * dim);
	if (Jtra) memset(Jtra, 0, sizeof(real) * dim);
	const real dmin = (real)prm->depth_min, dmax = (real)prm->depth_max;
	for (int pidx = 0; pidx < n_pairs; pidx++) {
		const unsigned i = pairs[2 * pidx], j = pairs[2 * pidx + 1];    /* i = target, j = source */
		const mat4 transform = mat_mul(&Tinv[i], &T[j]);
		const real* tgtCam = fc->campos + (size_t)i * npix * 4, *tgtNrm = fc->normal + (size_t)i * npix * 4;
		const real* srcCam = fc->campos + (size_t)j * npix * 4, *srcNrm = fc->normal + (size_t)j * npix * 4;
		float* marg = (ex && ex->margin) ? ex->margin + (size_t)pidx * npix : NULL;
		unsigned char* acc = (ex && ex->accepted) ? ex->accepted + (size_t)pidx * npix : NULL;
		float* ctb = (ex && ex->contrib) ? ex->contrib + (size_t)pidx * npix : NULL;
		int found = 0;
		for (int idx = 0; idx < npix; idx++) {
			const real* cposj = srcCam + (size_t)idx * 4;
			real m = 1;
			if (acc) acc[idx] = 0;
			if (ctb) ctb[idx] = 0;
			if (marg) { marg[idx] = 1; if (cposj[2] > 0) m = rmin(rel_gap(cposj[2], dmin, cposj[2]), rel_gap(cposj[2], dmax, cposj[2])); }
#define GATE_FAIL(cond) if (cond) { if (marg) marg[idx] = (float)m; continue; }
			GATE_FAIL(!(cposj[2] > (real)prm->depth_min && cposj[2] < (real)prm->depth_max));
			const vec3 camPosSrc = v3(cposj[0], cposj[1], cposj[2]);
			const real* nj = srcNrm + (size_t)idx * 4;
			real nrmj[4];
			for (int r = 0; r < 4; r++) nrmj[r] = M(transform,r,0)*nj[0] + M(transform,r,1)*nj[1] + M(transform,r,2)*nj[2] + M(transform,r,3)*nj[3];
			const vec3 camPosSrcToTgt = mat_mul_p(&transform, camPosSrc);
			const real sx = camPosSrcToTgt.x * fc->fx / camPosSrcToTgt.z + fc->cx;   /* CUDACameraUtil.h:9-14 */
			const real sy = camPosSrcToTgt.y * fc->fy / camPosSrcToTgt.z + fc->cy;
			if (marg) {   /* roundf bounds at -0.5 / size - 0.5; bilinear tap validity switches at 0 / size - 1 */
				m = rmin(m, rmin(rel_gap(sx, R_(-0.5), (real)w), rel_gap(sx, (real)w - R_(0.5), (real)w)));
				m = rmin(m, rmin(rel_gap(sy, R_(-0.5), (real)h), rel_gap(sy, (real)h - R_(0.5), (real)h)));
				m = rmin(m, rmin(rel_gap(sx, R_(0), (real)w), rel_gap(sx, (real)(w - 1), (real)w)));
				m = rmin(m, rmin(rel_gap(sy, R_(0), (real)h), rel_gap(sy, (real)(h - 1), (real)h)));
			}
			const int ix = (int)roundf((float)sx), iy = (int)roundf((float)sy);
			GATE_FAIL(!(ix >= 0 && iy >= 0 && ix < w && iy < h));
			real cposi[4], nrmi[4];
			GATE_FAIL(!bilinear4(sx, sy, tgtCam, w, h, cposi));
			if (marg) { const real sc = cposi[2] > dmin ? cposi[2] : dmin; m = rmin(m, rmin(rel_gap(cposi[2], dmin, sc), rel_gap(cposi[2], dmax, sc))); }
			GATE_FAIL(!(cposi[2] > (real)prm->depth_min && cposi[2] < (real)prm->depth_max));
			GATE_FAIL(!bilinear4(sx, sy, tgtNrm, w, h, nrmi));
			const vec3 camPosTgt = v3(cposi[0], cposi[1], cposi[2]), normalTgt = v3(nrmi[0], nrmi[1], nrmi[2]);
			const real dist = vlen(vsub(camPosSrcToTgt, camPosTgt));
			const real dNormal = nrmj[0]*nrmi[0] + nrmj[1]*nrmi[1] + nrmj[2]*nrmi[2] + nrmj[3]*nrmi[3];
			if (marg) m = rmin(m, rmin(rel_gap(dist, (real)prm->dense_dist_thresh, vlen(camPosSrcToTgt)), rel_gap(dNormal, (real)prm->dense_cos_normal_thresh, R_(1))));
			GATE_FAIL(!(dNormal >= (real)prm->dense_cos_normal_thresh && dist <= (real)prm->dense_dist_thresh));
#undef GATE_FAIL
			if (marg) marg[idx] = (float)m;
			if (acc) acc[idx] = 1;
			found++;
			const real depthRes = vdot(vsub(camPosTgt, camPosSrcToTgt), normalTgt);
			const real weight = (real)prm->w_dense * huber_weight(depthRes * depthRes, (real)prm->robust_delta);
			real Ji[6] = { 0 }, Jj[6] = { 0 }, jac[3][6];
			if (i > 0) { /* computeJacobianBlockRow_i: Solver/SolverBundlingEquationsLie.h:214-221 */
				evalLie_derivI(&Tinv[j], &T[i], camPosSrc, jac);
				for (int c = 0; c < 6; c++) Ji[c] = -(jac[0][c] * normalTgt.x + jac[1][c] * normalTgt.y + jac[2][c] * normalTgt.z);
			}
			if (j > 0) { /* computeJacobianBlockRow_j: :223-230 */
				evalLie_derivJ(&Tinv[i], &T[j], camPosSrc, jac);
				for (int c = 0; c < 6; c++) Jj[c] = -(jac[0][c] * normalTgt.x + jac[1][c] * normalTgt.y + jac[2][c] * normalTgt.z);
			}
			for (int a = 0; a < 6; a++) { /* addToLocalSystem */
				for (int b = a; b < 6; b++) {
					if (i > 0) JtJ[(i * 6 + b) * dim + (i * 6 + a)] += Ji[a] * Ji[b] * weight;
					if (j > 0) JtJ[(j * 6 + b) * dim + (j * 6 + a)] += Jj[a] * Jj[b] * weight;
					if (i > 0 && j > 0) {
						JtJ[(j * 6 + b) * dim + (i * 6 + a)] += Ji[a] * Jj[b] * weight;
						if (a != b) JtJ[(j * 6 + a) * dim + (i * 6 + b)] += Ji[b] * Jj[a] * weight;
					}
					if (JtJa) {
						if (i > 0) JtJa[(i * 6 + b) * dim + (i * 6 + a)] += (real)fabs((double)(Ji[a] * Ji[b] * weight));
						if (j > 0) JtJa[(j * 6 + b) * dim + (j * 6 + a)] += (real)fabs((double)(Jj[a] * Jj[b] * weight));
						if (i > 0 && j > 0) {
							JtJa[(j * 6 + b) * dim + (i * 6 + a)] += (real)fabs((double)(Ji[a] * Jj[b] * weight));
							if (a != b) JtJa[(j * 6 + a) * dim + (i * 6 + b)] += (real)fabs((double)(Ji[b] * Jj[a] * weight));
						}
					}
				}
				if (i > 0) Jtr[i * 6 + a] += Ji[a] * depthRes * weight;
				if (j > 0) Jtr[j * 6 + a] += Jj[a] * depthRes * weight;
				if (Jtra && i > 0) Jtra[i * 6 + a] += (real)fabs((double)(Ji[a] * depthRes * weight));
				if (Jtra && j > 0) Jtra[j * 6 + a] += (real)fabs((double)(Jj[a] * depthRes * weight));
				if (ctb) ctb[idx] += (float)((Ji[a] * Ji[a] + Jj[a] * Jj[a]) * weight);
			}
		}
		if (n_found_per_pair) n_found_per_pair[pidx] = found;
	}
	if (ex && !ex->flip) return;     /* raw addToLocalSystem output: lower triangle of each diagonal block, each cross block where it was written */
	/* FlipJtJ_Kernel: upper := lower (erases cross blocks that were written above the diagonal, SURVEY.md Q2) */
	for (int y = 0; y < dim; y++) for (int x = y + 1; x < dim; x++) JtJ[y * dim + x] = JtJ[x * dim + y];
	if (JtJa) for (int y = 0; y < dim; y++) for (int x = y + 1; x < dim; x++) JtJa[y * dim + x] = JtJa[x * dim + y];
}

/* ---- sparse term + PCG: SolverBundlingEquationsLie.h:60-211, SolverBundling.cu:575-887 ---- */
typedef struct { vec3 rot, trans; } pose6;

static void lie_d(vec3 q, vec3* da, vec3* db, vec3* dc) { /* LieDerivUtil.h:215-226 */
	*da = v3(0, -q.z, q.y); *db = v3(q.z, 0, -q.x); *dc = v3(-q.y, q.x, 0);
}
static vec3 vabs3(vec3 a) { return v3((real)fabs((double)a.x), (real)fabs((double)a.y), (real)fabs((double)a.z)); }

/* evalMinusJTFDevice for frame v, sparse part: r = sum rho sign J^T res (rot, trans) and the Jacobi sums p (rot, trans).
 * aRot / aTrans (optional): the same gradient sums over |term|. */
static void sparse_jtf(int v, const mat4* T, int n_corr, const EntryJ* corr, real robust_delta,
                       vec3* rRot_, vec3* rTrans_, vec3* pRot_, vec3* pTrans_, vec3* aRot, vec3* aTrans) {
	vec3 rRot = v3(0,0,0), rTrans = v3(0,0,0), pRot = v3(0,0,0), pTrans = v3(0,0,0);
	if (aRot) { *aRot = v3(0,0,0); *aTrans = v3(0,0,0); }
	for (int c = 0; c < n_corr; c++) {
		const EntryJ* e = &corr[c];
		if (e->imgIdx_i == 0xFFFFFFFFu) continue;
		if ((int)e->imgIdx_i != v && (int)e->imgIdx_j != v) continue;
		const vec3 pi_ = v3((real)e->pos_i[0], (real)e->pos_i[1], (real)e->pos_i[2]);
		const vec3 pj_ = v3((real)e->pos_j[0], (real)e->pos_j[1], (real)e->pos_j[2]);
		const vec3 wi = mat_mul_p(&T[e->imgIdx_i], pi_), wj = mat_mul_p(&T[e->imgIdx_j], pj_);
		real sign = 1; vec3 worldP = wi;
		if ((unsigned)v != e->imgIdx_i) { sign = -1; worldP = wj; }
		vec3 da, db, dc; lie_d(worldP, &da, &db, &dc);
		const vec3 res = vsub(wi, wj);
		const real rho = huber_weight(vdot(res, res), robust_delta);
		const vec3 gr = vscale(v3(vdot(da, res), vdot(db, res), vdot(dc, res)), rho * sign), gt = vscale(res, rho * sign);
		rRot = vadd(rRot, gr);
		rTrans = vadd(rTrans, gt);
		pRot = vadd(pRot, vscale(v3(vdot(da, da), vdot(db, db), vdot(dc, dc)), rho));
		pTrans = vadd(pTrans, vscale(v3(1, 1, 1), rho));
		if (aRot) { *aRot = vadd(*aRot, vabs3(gr)); *aTrans = vadd(*aTrans, vabs3(gt)); }
	}
	*rRot_ = rRot; *rTrans_ = rTrans; *pRot_ = pRot; *pTrans_ = pTrans;
}

/* PCGStep_Kernel0 / applyJDevice: Jp[c] = wS (J_i p_i - J_j p_j) of every correspondence (zero for invalid entries) */
static void apply_j(const mat4* T, int n_corr, const EntryJ* corr, const pose6* p, real wS, vec3* Jp) {
	for (int c = 0; c < n_corr; c++) {
		const EntryJ* e = &corr[c];
		vec3 b = v3(0,0,0);
		if (e->imgIdx_i != 0xFFFFFFFFu) {
			if (e->imgIdx_i > 0) {
				const vec3 wp = mat_mul_p(&T[e->imgIdx_i], v3((real)e->pos_i[0], (real)e->pos_i[1], (real)e->pos_i[2]));
				vec3 da, db, dc; lie_d(wp, &da, &db, &dc);
				const vec3 pp = p[e->imgIdx_i].rot;
				b = vadd(b, vadd(vadd(vadd(vscale(da, pp.x), vscale(db, pp.y)), vscale(dc, pp.z)), p[e->imgIdx_i].trans));
			}
			if (e->imgIdx_j > 0) {
				const vec3 wp = mat_mul_p(&T[e->imgIdx_j], v3((real)e->pos_j[0], (real)e->pos_j[1], (real)e->pos_j[2]));
				vec3 da, db, dc; lie_d(wp, &da, &db, &dc);
				const vec3 pp = p[e->imgIdx_j].rot;
				b = vsub(b, vadd(vadd(vadd(vscale(da, pp.x), vscale(db, pp.y)), vscale(dc, pp.z)), p[e->imgIdx_j].trans));
			}
			b = vscale(b, wS);
		}
		Jp[c] = b;
	}
}

/* PCGStep_Kernel1a / applyJTDevice: Ap[v] += J_v^T Jp (with the sign of v's side) for frames 1..N-1 */
static void apply_jt(int N, const mat4* T, int n_corr, const EntryJ* corr, const vec3* Jp, pose6* Ap) {
	for (int v = 1; v < N; v++) {
		vec3 oR = v3(0,0,0), oT = v3(0,0,0);
		for (int c = 0; c < n_corr; c++) {
			const EntryJ* e = &corr[c];
			if (e->imgIdx_i == 0xFFFFFFFFu) continue;
			if ((int)e->imgIdx_i != v && (int)e->imgIdx_j != v) continue;
			real sign = 1; vec3 wp;
			if ((unsigned)v != e->imgIdx_i) { sign = -1; wp = mat_mul_p(&T[e->imgIdx_j], v3((real)e->pos_j[0], (real)e->pos_j[1], (real)e->pos_j[2])); }
			else wp = mat_mul_p(&T[e->imgIdx_i], v3((real)e->pos_i[0], (real)e->pos_i[1], (real)e->pos_i[2]));
			vec3 da, db, dc; lie_d(wp, &da, &db, &dc);
			oR = vadd(oR, vscale(v3(vdot(da, Jp[c]), vdot(db, Jp[c]), vdot(dc, Jp[c])), sign));
			oT = vadd(oT, vscale(Jp[c], sign));
		}
		Ap[v].rot = vadd(Ap[v].rot, oR); Ap[v].trans = vadd(Ap[v].trans, oT);
	}
}

int oracle_solve_window(int N, int H, int W, const float* depth, const float* normal,
                        float fx, float fy, float cx, float cy,
                        int n_corr, const EntryJ* corr,
                        const uint32_t* dense_pairs, int n_pairs,
                        const oracle_params* prm, float* poses_inout /*[N][16] row-major*/,
                        double* dbg_JtJ0 /*optional [6N*6N]: dense JtJ of GN iter 0*/,
                        double* dbg_Jtr0 /*optional [6N]*/) {
	if (N < 2 || N > 64) return -1;
	const int dim = 6 * N;
	frame_cache fc;
	const int use_dense_any = prm->w_dense > 0 && n_pairs > 0;
	if (use_dense_any) cache_build(&fc, N, H, W, depth, normal, fx, fy, cx, cy, prm->image_downscale);
	mat4* T = (mat4*)malloc(sizeof(mat4) * N), *Tinv = (mat4*)malloc(sizeof(mat4) * N);
	pose6* x = (pose6*)malloc(sizeof(pose6) * N);
	real* JtJ = (real*)calloc((size_t)dim * dim, sizeof(real)), *Jtr = (real*)calloc(dim, sizeof(real));
	vec3* Jp = (vec3*)malloc(sizeof(vec3) * (n_corr > 0 ? n_corr : 1));
	pose6 *delta = (pose6*)calloc(N, sizeof(pose6)), *r = (pose6*)calloc(N, sizeof(pose6)), *z = (pose6*)calloc(N, sizeof(pose6)),
	      *p = (pose6*)calloc(N, sizeof(pose6)), *Ap = (pose6*)calloc(N, sizeof(pose6)), *Minv = (pose6*)calloc(N, sizeof(pose6));

	for (int f = 0; f < N; f++) { /* convertMatricesToPosesCU (SBA.cu:71-79) */
		mat4 Tm;
		for (int k = 0; k < 16; k++) Tm.m[k] = (real)poses_inout[f * 16 + k];
		matrixToPose(&Tm, &x[f].rot, &x[f].trans);
	}
	const real wS = (real)prm->w_sparse;
	for (int it = 0; it < prm->num_iter_outer; it++) { /* solveBundlingStub loop, SolverBundling.cu:946-1001 */
		for (int f = 0; f < N; f++) { T[f] = poseToMatrix(x[f].rot, x[f].trans); Tinv[f] = mat_inverse(&T[f]); } /* :890-897 */
		int useDense = use_dense_any;
		if (useDense) {
			build_dense_system(&fc, N, T, Tinv, dense_pairs, n_pairs, prm, JtJ, Jtr, NULL, NULL);
			if (it == 0 && dbg_JtJ0) for (int k = 0; k < dim * dim; k++) dbg_JtJ0[k] = (double)JtJ[k];
			if (it == 0 && dbg_Jtr0) for (int k = 0; k < dim; k++) dbg_Jtr0[k] = (double)Jtr[k];
		}
		/* PCGInit_Kernel1 / evalMinusJTFDevice (frames 1..N-1; frame 0 is the gauge) */
		real rDotzOld = 0;
		for (int v = 1; v < N; v++) {
			vec3 rRot, rTrans, pRot, pTrans;
			delta[v].rot = v3(0,0,0); delta[v].trans = v3(0,0,0);
			sparse_jtf(v, T, n_corr, corr, (real)prm->robust_delta, &rRot, &rTrans, &pRot, &pTrans, NULL, NULL);
			vec3 resRot = vscale(rRot, -wS), resTrans = vscale(rTrans, -wS);
			if (useDense) { /* dense ordering: trans 0-2, rot 3-5 (SolverBundlingEquationsLie.h:113-118) */
				resRot = vsub(resRot, v3(Jtr[v * 6 + 3], Jtr[v * 6 + 4], Jtr[v * 6 + 5]));
				resTrans = vsub(resTrans, v3(Jtr[v * 6 + 0], Jtr[v * 6 + 1], Jtr[v * 6 + 2]));
			}
			Minv[v].rot.x = pRot.x > FLOAT_EPSILON ? R_(1) / pRot.x : R_(1);
			Minv[v].rot.y = pRot.y > FLOAT_EPSILON ? R_(1) / pRot.y : R_(1);
			Minv[v].rot.z = pRot.z > FLOAT_EPSILON ? R_(1) / pRot.z : R_(1);
			Minv[v].trans.x = pTrans.x > FLOAT_EPSILON ? R_(1) / pTrans.x : R_(1);
			Minv[v].trans.y = pTrans.y > FLOAT_EPSILON ? R_(1) / pTrans.y : R_(1);
			Minv[v].trans.z = pTrans.z > FLOAT_EPSILON ? R_(1) / pTrans.z : R_(1);
			r[v].rot = resRot; r[v].trans = resTrans;
			p[v].rot = v3(Minv[v].rot.x * resRot.x, Minv[v].rot.y * resRot.y, Minv[v].rot.z * resRot.z);
			p[v].trans = v3(Minv[v].trans.x * resTrans.x, Minv[v].trans.y * resTrans.y, Minv[v].trans.z * resTrans.z);
			rDotzOld += vdot(resRot, p[v].rot) + vdot(resTrans, p[v].trans);
			Ap[v].rot = v3(0,0,0); Ap[v].trans = v3(0,0,0);
		}
		for (int lin = 0; lin < prm->num_iter_inner; lin++) { /* PCGIteration<useSparse,useDense>, :820-887 */
			if (wS > 0) {
				apply_j(T, n_corr, corr, p, wS, Jp);
				apply_jt(N, T, n_corr, corr, Jp, Ap);
			}
			if (useDense) { /* PCGStep_Kernel_Dense / applyJTJDenseDevice (SolverBundlingDenseUtil.h:349-385) */
				for (int v = 1; v < N; v++) {
					vec3 oR = v3(0,0,0), oT = v3(0,0,0);
					for (int k = 1; k < N; k++) {
						const real pv[6] = { p[k].trans.x, p[k].trans.y, p[k].trans.z, p[k].rot.x, p[k].rot.y, p[k].rot.z };
						real o[6] = { 0, 0, 0, 0, 0, 0 };
						for (int a = 0; a < 6; a++) for (int b = 0; b < 6; b++) o[a] += JtJ[(v * 6 + a) * dim + k * 6 + b] * pv[b];
						oT = vadd(oT, v3(o[0], o[1], o[2])); oR = vadd(oR, v3(o[3], o[4], o[5]));
					}
					Ap[v].rot = vadd(Ap[v].rot, oR); Ap[v].trans = vadd(Ap[v].trans, oT);
				}
			}
			real dotProduct = 0; /* PCGStep_Kernel1b */
			for (int v = 1; v < N; v++) dotProduct += vdot(p[v].rot, Ap[v].rot) + vdot(p[v].trans, Ap[v].trans);
			real alpha = 0, rDotzNew = 0; /* PCGStep_Kernel2 */
			if (dotProduct > FLOAT_EPSILON) alpha = rDotzOld / dotProduct;
			for (int v = 1; v < N; v++) {
				delta[v].rot = vadd(delta[v].rot, vscale(p[v].rot, alpha));
				delta[v].trans = vadd(delta[v].trans, vscale(p[v].trans, alpha));
				r[v].rot = vsub(r[v].rot, vscale(Ap[v].rot, alpha));
				r[v].trans = vsub(r[v].trans, vscale(Ap[v].trans, alpha));
				z[v].rot = v3(Minv[v].rot.x * r[v].rot.x, Minv[v].rot.y * r[v].rot.y, Minv[v].rot.z * r[v].rot.z);
				z[v].trans = v3(Minv[v].trans.x * r[v].trans.x, Minv[v].trans.y * r[v].trans.y, Minv[v].trans.z * r[v].trans.z);
				rDotzNew += vdot(z[v].rot, r[v].rot) + vdot(z[v].trans, r[v].trans);
			}
			real beta = 0; /* PCGStep_Kernel3 */
			if (rDotzOld > FLOAT_EPSILON) beta = rDotzNew / rDotzOld;
			rDotzOld = rDotzNew;
			for (int v = 1; v < N; v++) {
				p[v].rot = vadd(z[v].rot, vscale(p[v].rot, beta));
				p[v].trans = vadd(z[v].trans, vscale(p[v].trans, beta));
				Ap[v].rot = v3(0,0,0); Ap[v].trans = v3(0,0,0);
				if (lin == prm->num_iter_inner - 1) { /* computeLieUpdate (LieDerivUtil.h:276-282) */
					const mat4 upd = poseToMatrix(delta[v].rot, delta[v].trans), cur = poseToMatrix(x[v].rot, x[v].trans);
					const mat4 nw = mat_mul(&upd, &cur);
					matrixToPose(&nw, &x[v].rot, &x[v].trans);
				}
			}
		}
	}
	for (int f = 0; f < N; f++) { /* convertPosesToMatricesCU (SBA.cu:97-104) */
		const mat4 Tm = poseToMatrix(x[f].rot, x[f].trans);
		for (int k = 0; k < 16; k++) poses_inout[f * 16 + k] = (float)Tm.m[k];
	}
	if (use_dense_any) cache_free(&fc);
	free(T); free(Tinv); free(x); free(JtJ); free(Jtr); free(Jp);
	free(delta); free(r); free(z); free(p); free(Ap); free(Minv);
	return 0;
}

/* Exposed pieces for unit tests of the CUDA kernels (cache texels, one dense system at given poses). */
int oracle_build_cache(int N, int H, int W, const float* depth, const float* normal, float fx, float fy, float cx, float cy,
                       float downscale, float* campos_out /*[N][h*w][4]*/, float* normal_out, float* intr_out /*[4]*/) {
	frame_cache fc;
	cache_build(&fc, N, H, W, depth, normal, fx, fy, cx, cy, downscale);
	const size_t n = (size_t)N * fc.w * fc.h * 4;
	for (size_t k = 0; k < n; k++) { campos_out[k] = (float)fc.campos[k]; normal_out[k] = (float)fc.normal[k]; }
	intr_out[0] = (float)fc.fx; intr_out[1] = (float)fc.fy; intr_out[2] = (float)fc.cx; intr_out[3] = (float)fc.cy;
	cache_free(&fc);
	return 0;
}

/* the round trip the solver applies to its input poses: matrix -> se(3) -> matrix */
static void load_poses(int N, const float* poses, mat4* T, mat4* Tinv) {
	for (int f = 0; f < N; f++) {
		mat4 Tm; vec3 rot, trans;
		for (int k = 0; k < 16; k++) Tm.m[k] = (real)poses[f * 16 + k];
		matrixToPose(&Tm, &rot, &trans);
		T[f] = poseToMatrix(rot, trans);
		if (Tinv) Tinv[f] = mat_inverse(&T[f]);
	}
}

/* One dense system at given poses.  flip = 0 returns the raw addToLocalSystem sums (no FlipJtJ); the optional outputs are those of
 * dense_extra (JtJ_abs_out / Jtr_abs_out as doubles, margin / accepted / contrib per (pair, quarter-res source pixel)). */
int oracle_dense_system_ex(int N, int H, int W, const float* depth, const float* normal, float fx, float fy, float cx, float cy,
                           const uint32_t* dense_pairs, int n_pairs, const oracle_params* prm, const float* poses /*[N][16]*/, int flip,
                           double* JtJ_out, double* Jtr_out, int* n_found_per_pair, double* JtJ_abs_out, double* Jtr_abs_out,
                           float* margin_out, unsigned char* accepted_out, float* contrib_out) {
	const int dim = 6 * N;
	frame_cache fc;
	cache_build(&fc, N, H, W, depth, normal, fx, fy, cx, cy, prm->image_downscale);
	mat4* T = (mat4*)malloc(sizeof(mat4) * N), *Tinv = (mat4*)malloc(sizeof(mat4) * N);
	load_poses(N, poses, T, Tinv);
	real* JtJ = (real*)calloc((size_t)dim * dim, sizeof(real)), *Jtr = (real*)calloc(dim, sizeof(real));
	real* JtJa = JtJ_abs_out ? (real*)calloc((size_t)dim * dim, sizeof(real)) : NULL, *Jtra = Jtr_abs_out ? (real*)calloc(dim, sizeof(real)) : NULL;
	dense_extra ex = { JtJa, Jtra, margin_out, accepted_out, contrib_out, flip };
	build_dense_system(&fc, N, T, Tinv, dense_pairs, n_pairs, prm, JtJ, Jtr, n_found_per_pair, &ex);
	for (int k = 0; k < dim * dim; k++) JtJ_out[k] = (double)JtJ[k];
	for (int k = 0; k < dim; k++) Jtr_out[k] = (double)Jtr[k];
	if (JtJa) for (int k = 0; k < dim * dim; k++) JtJ_abs_out[k] = (double)JtJa[k];
	if (Jtra) for (int k = 0; k < dim; k++) Jtr_abs_out[k] = (double)Jtra[k];
	cache_free(&fc); free(T); free(Tinv); free(JtJ); free(Jtr); free(JtJa); free(Jtra);
	return 0;
}

int oracle_dense_system(int N, int H, int W, const float* depth, const float* normal, float fx, float fy, float cx, float cy,
                        const uint32_t* dense_pairs, int n_pairs, const oracle_params* prm, const float* poses /*[N][16]*/,
                        double* JtJ_out, double* Jtr_out, int* n_found_per_pair) {
	return oracle_dense_system_ex(N, H, W, depth, normal, fx, fy, cx, cy, dense_pairs, n_pairs, prm, poses, 1, JtJ_out, Jtr_out, n_found_per_pair,
	                              NULL, NULL, NULL, NULL, NULL);
}

/* The sparse term at given poses as the PCG of oracle_solve_window uses it, over the free frames 1..N-1 (dim = 6(N-1), per frame
 * trans 0-2 / rot 3-5 like the dense system): A_out = the explicit matrix of applyJT(applyJ(.)), column by column from unit vectors;
 * rhs_out = -wS J^T F (evalMinusJTF without the dense term); minv_out = the Jacobi preconditioner; rhs_abs_out (optional) = the
 * gradient sums over |term|, scaled by wS. */
int oracle_sparse_system(int N, int n_corr, const EntryJ* corr, const oracle_params* prm, const float* poses /*[N][16]*/,
                         double* A_out, double* rhs_out, double* minv_out, double* rhs_abs_out) {
	if (N < 2) return -1;
	const int dimp = 6 * (N - 1);
	const real wS = (real)prm->w_sparse;
	mat4* T = (mat4*)malloc(sizeof(mat4) * N);
	load_poses(N, poses, T, NULL);
	pose6* p = (pose6*)calloc(N, sizeof(pose6)), *Ap = (pose6*)calloc(N, sizeof(pose6));
	vec3* Jp = (vec3*)malloc(sizeof(vec3) * (n_corr > 0 ? n_corr : 1));
	for (int u = 0; u < dimp; u++) {
		memset(p, 0, sizeof(pose6) * N); memset(Ap, 0, sizeof(pose6) * N);
		const int fu = 1 + u / 6, cu = u % 6;
		real* pu = (cu < 3) ? &p[fu].trans.x : &p[fu].rot.x;
		pu[cu % 3] = R_(1);
		apply_j(T, n_corr, corr, p, wS, Jp);
		apply_jt(N, T, n_corr, corr, Jp, Ap);
		for (int v = 1; v < N; v++) {
			const real col[6] = { Ap[v].trans.x, Ap[v].trans.y, Ap[v].trans.z, Ap[v].rot.x, Ap[v].rot.y, Ap[v].rot.z };
			for (int r = 0; r < 6; r++) A_out[(size_t)((v - 1) * 6 + r) * dimp + u] = (double)col[r];
		}
	}
	for (int v = 1; v < N; v++) {
		vec3 rRot, rTrans, pRot, pTrans, aRot, aTrans;
		sparse_jtf(v, T, n_corr, corr, (real)prm->robust_delta, &rRot, &rTrans, &pRot, &pTrans, &aRot, &aTrans);
		const vec3 resRot = vscale(rRot, -wS), resTrans = vscale(rTrans, -wS);
		const real rr[6] = { resTrans.x, resTrans.y, resTrans.z, resRot.x, resRot.y, resRot.z };
		const real pc[6] = { pTrans.x, pTrans.y, pTrans.z, pRot.x, pRot.y, pRot.z };
		const real ra[6] = { aTrans.x, aTrans.y, aTrans.z, aRot.x, aRot.y, aRot.z };
		for (int r = 0; r < 6; r++) {
			rhs_out[(v - 1) * 6 + r] = (double)rr[r];
			minv_out[(v - 1) * 6 + r] = (double)(pc[r] > FLOAT_EPSILON ? R_(1) / pc[r] : R_(1));
			if (rhs_abs_out) rhs_abs_out[(v - 1) * 6 + r] = (double)(ra[r] * wS);
		}
	}
	free(T); free(p); free(Ap); free(Jp);
	return 0;
}

/* The matrix-free sparse operator itself: y = applyJT(applyJ(x)) over frames 1..N-1, x and y in the layout of oracle_sparse_system. */
int oracle_sparse_apply(int N, int n_corr, const EntryJ* corr, const oracle_params* prm, const float* poses, const double* x, double* y) {
	if (N < 2) return -1;
	mat4* T = (mat4*)malloc(sizeof(mat4) * N);
	load_poses(N, poses, T, NULL);
	pose6* p = (pose6*)calloc(N, sizeof(pose6)), *Ap = (pose6*)calloc(N, sizeof(pose6));
	vec3* Jp = (vec3*)malloc(sizeof(vec3) * (n_corr > 0 ? n_corr : 1));
	for (int v = 1; v < N; v++) {
		const double* xv = x + (v - 1) * 6;
		p[v].trans = v3((real)xv[0], (real)xv[1], (real)xv[2]); p[v].rot = v3((real)xv[3], (real)xv[4], (real)xv[5]);
	}
	apply_j(T, n_corr, corr, p, (real)prm->w_sparse, Jp);
	apply_jt(N, T, n_corr, corr, Jp, Ap);
	for (int v = 1; v < N; v++) {
		const real o[6] = { Ap[v].trans.x, Ap[v].trans.y, Ap[v].trans.z, Ap[v].rot.x, Ap[v].rot.y, Ap[v].rot.z };
		for (int r = 0; r < 6; r++) y[(v - 1) * 6 + r] = (double)o[r];
	}
	free(T); free(p); free(Ap); free(Jp);
	return 0;
}

/* se(3) round trip helpers for tests */
void oracle_matrix_to_pose(const float* T16, float* rot3, float* trans3) {
	mat4 Tm; vec3 r, t;
	for (int k = 0; k < 16; k++) Tm.m[k] = (real)T16[k];
	matrixToPose(&Tm, &r, &t);
	rot3[0] = (float)r.x; rot3[1] = (float)r.y; rot3[2] = (float)r.z;
	trans3[0] = (float)t.x; trans3[1] = (float)t.y; trans3[2] = (float)t.z;
}
void oracle_pose_to_matrix(const float* rot3, const float* trans3, float* T16) {
	const mat4 Tm = poseToMatrix(v3((real)rot3[0], (real)rot3[1], (real)rot3[2]), v3((real)trans3[0], (real)trans3[1], (real)trans3[2]));
	for (int k = 0; k < 16; k++) T16[k] = (float)Tm.m[k];
}
int oracle_sizeof_real(void) { return (int)sizeof(real); }
