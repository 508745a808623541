// rigid.cuh — Utils::solveRigidTransformBetweenPoints (the reference's src/Utils.cpp:180-214) as __host__ __device__ code, shared by
// bt_rigid_transform (policy.cu, host) and k_pose_init (tracker.cu, device) so both give the same bits on the same float points.
// Conditions for that: every double operation is rounded on its own (no fused multiply-add).  The host build has no FMA (x86-64 without
// -mfma); the translation units that call this on the device are compiled with -fmad=false, and the accumulations below use the _rn
// intrinsics on the device besides.  The caller feeds the points in order: rigid_add_means over all points, rigid_means, rigid_add_cov
// over all points in the same order, then rigid_solve.
#pragma once
#include <math.h>

#ifdef __CUDA_ARCH__
#define BT_DADD(a, b) __dadd_rn((a), (b))
#define BT_DSUB(a, b) __dsub_rn((a), (b))
#define BT_DMUL(a, b) __dmul_rn((a), (b))
#else
#define BT_DADD(a, b) ((a) + (b))
#define BT_DSUB(a, b) ((a) - (b))
#define BT_DMUL(a, b) ((a) * (b))
#endif

namespace bt {

struct RigidSums {
	double m1[3], m2[3];      // sums, then means, of the two point sets
	double S[9];              // S = P^T Q with P, Q the centred point sets
};

__host__ __device__ inline void rigid_init(RigidSums& r) {
	for (int k = 0; k < 3; k++) { r.m1[k] = 0; r.m2[k] = 0; }
	for (int k = 0; k < 9; k++) r.S[k] = 0;
}
__host__ __device__ inline void rigid_add_means(RigidSums& r, const float p1[3], const float p2[3]) {
	for (int k = 0; k < 3; k++) { r.m1[k] = BT_DADD(r.m1[k], (double)p1[k]); r.m2[k] = BT_DADD(r.m2[k], (double)p2[k]); }
}
__host__ __device__ inline void rigid_means(RigidSums& r, int n) {
	for (int k = 0; k < 3; k++) { r.m1[k] /= n; r.m2[k] /= n; }
}
__host__ __device__ inline void rigid_add_cov(RigidSums& r, const float p1[3], const float p2[3]) {
	for (int a = 0; a < 3; a++)
		for (int c = 0; c < 3; c++) r.S[a * 3 + c] = BT_DADD(r.S[a * 3 + c], BT_DMUL(BT_DSUB((double)p1[a], r.m1[a]), BT_DSUB((double)p2[c], r.m2[c])));
}

__host__ __device__ inline double dmax(double a, double b) { return (a < b) ? b : a; }     // std::max

// one-sided Jacobi SVD of a 3x3 (double): M = U diag(s) V^T, singular values sorted descending
__host__ __device__ inline void svd3(const double M[9], double U[9], double S[3], double V[9]) {
	double A[9];
	for (int i = 0; i < 9; i++) { A[i] = M[i]; V[i] = (i % 4 == 0) ? 1.0 : 0.0; }
	for (int sweep = 0; sweep < 60; sweep++) {
		double off = 0.0;
		for (int p = 0; p < 2; p++)
			for (int q = p + 1; q < 3; q++) {
				double a = 0, b = 0, g = 0;      // columns p, q of A
				for (int r = 0; r < 3; r++) { a += A[r * 3 + p] * A[r * 3 + p]; b += A[r * 3 + q] * A[r * 3 + q]; g += A[r * 3 + p] * A[r * 3 + q]; }
				off = dmax(off, fabs(g) / (sqrt(a * b) + 1e-300));
				if (fabs(g) < 1e-300) continue;
				const double zeta = (b - a) / (2.0 * g);
				const double t = (zeta >= 0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
				const double c = 1.0 / sqrt(1.0 + t * t), s = c * t;
				for (int r = 0; r < 3; r++) {
					const double ap = A[r * 3 + p], aq = A[r * 3 + q];
					A[r * 3 + p] = c * ap - s * aq; A[r * 3 + q] = s * ap + c * aq;
					const double vp = V[r * 3 + p], vq = V[r * 3 + q];
					V[r * 3 + p] = c * vp - s * vq; V[r * 3 + q] = s * vp + c * vq;
				}
			}
		if (off < 1e-15) break;
	}
	double n[3];
	for (int j = 0; j < 3; j++) n[j] = sqrt(A[j] * A[j] + A[3 + j] * A[3 + j] + A[6 + j] * A[6 + j]);
	// column order by descending norm: libstdc++'s std::sort on three elements, i.e. its insertion sort step for step (ties keep the column order)
	int order[3] = { 0, 1, 2 };
	for (int i = 1; i < 3; i++) {
		const int v = order[i];
		int j = i;
		if (n[v] > n[order[0]]) {
			for (; j > 0; j--) order[j] = order[j - 1];
		} else {
			while (n[v] > n[order[j - 1]]) { order[j] = order[j - 1]; j--; }
		}
		order[j] = v;
	}
	double Vs[9];
	for (int j = 0; j < 3; j++) {
		const int o = order[j];
		S[j] = n[o];
		for (int r = 0; r < 3; r++) { U[r * 3 + j] = n[o] > 1e-300 ? A[r * 3 + o] / n[o] : 0.0; Vs[r * 3 + j] = V[r * 3 + o]; }
	}
	// A singular value that is rounding noise next to the largest one (coplanar points: one column of M V is ~1e-18) carries no
	// direction: normalising that column would give a U that is not orthogonal.  Treat it as zero and complete U below.
	for (int j = 1; j < 3; j++) if (S[j] <= 1e-12 * S[0]) S[j] = 0.0;
	for (int i = 0; i < 9; i++) V[i] = Vs[i];
	// complete U to an orthonormal basis when M is rank deficient (Eigen's thin U is full for a 3x3 as well)
	if (!(S[0] > 1e-300)) { for (int i = 0; i < 9; i++) U[i] = (i % 4 == 0) ? 1.0 : 0.0; return; }      // M = 0
	if (!(S[1] > 1e-300)) {      // rank 1: any unit vector orthogonal to column 0
		const int m = fabs(U[0]) < fabs(U[3]) ? (fabs(U[0]) < fabs(U[6]) ? 0 : 2) : (fabs(U[3]) < fabs(U[6]) ? 1 : 2);
		double e[3] = { 0, 0, 0 }; e[m] = 1.0;
		const double c[3] = { U[3] * e[2] - U[6] * e[1], U[6] * e[0] - U[0] * e[2], U[0] * e[1] - U[3] * e[0] };
		const double cn = sqrt(c[0] * c[0] + c[1] * c[1] + c[2] * c[2]);
		for (int r = 0; r < 3; r++) U[r * 3 + 1] = c[r] / cn;
	}
	if (!(S[2] > 1e-300)) {      // rank <= 2: column 2 = column 0 x column 1
		U[2] = U[3] * U[7] - U[6] * U[4];
		U[5] = U[6] * U[1] - U[0] * U[7];
		U[8] = U[0] * U[4] - U[3] * U[1];
	}
}

__host__ __device__ inline void rigid_vut(const double U[9], const double V[9], double R[9]) {      // R = V U^T
	for (int r = 0; r < 3; r++)
		for (int c = 0; c < 3; c++) { R[r * 3 + c] = 0; for (int k = 0; k < 3; k++) R[r * 3 + c] += V[r * 3 + k] * U[c * 3 + k]; }
}

// T (row-major 4x4): the rigid transform mapping set 1 onto set 2 from the means and S; T is left as the identity when the fit degenerates
__host__ __device__ inline void rigid_solve(const RigidSums& r, float T[16]) {
	for (int i = 0; i < 16; i++) T[i] = (i % 5 == 0) ? 1.f : 0.f;
	double U[9], sv[3], V[9];
	svd3(r.S, U, sv, V);
	double R[9];
	rigid_vut(U, V, R);
	for (int a = 0; a < 3; a++)                          // R^T R must be the identity (isApprox, Utils.cpp:196), else the pose stays identity
		for (int c = 0; c < 3; c++) {
			double d = 0;
			for (int k = 0; k < 3; k++) d += R[k * 3 + a] * R[k * 3 + c];
			if (!(fabs(d - (a == c ? 1.0 : 0.0)) <= 1e-5)) return;
		}
	const double det = R[0] * (R[4] * R[8] - R[5] * R[7]) - R[1] * (R[3] * R[8] - R[5] * R[6]) + R[2] * (R[3] * R[7] - R[4] * R[6]);
	if (det < 0) { for (int a = 0; a < 3; a++) V[a * 3 + 2] = -V[a * 3 + 2]; rigid_vut(U, V, R); }      // reflection: flip the last right singular vector
	float out[16] = { 0 };
	out[15] = 1.f;
	for (int a = 0; a < 3; a++) {
		double t = r.m2[a];
		for (int c = 0; c < 3; c++) { out[a * 4 + c] = (float)R[a * 3 + c]; t -= R[a * 3 + c] * r.m1[c]; }
		out[a * 4 + 3] = (float)t;
	}
	for (int i = 0; i < 16; i++) if (!isfinite(out[i])) return;      // isMatrixFinite, Utils.cpp:209
	for (int i = 0; i < 16; i++) T[i] = out[i];
}

}  // namespace bt
