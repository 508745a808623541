// ransac.cu — batched 3-point RANSAC over frame pairs.
//
// Replaces ransacMultiPairGPU (/root/reference/src/cuda/cuda_ransac.cu:1228-1323: per pair 6 cudaMalloc/cudaFree, a new
// stream, three kernels and an int[n_trials][n_pts] flag matrix — 16 MB at 2000 x 2000 — copied back row by row) with three
// launches for the WHOLE batch and no flag matrix:
//
//   k_ransac_model   one thread per (pair, trial): the reference's sampling (ransacEstimateModelKernel :1145-1181:
//                    curand_init(seed, trial, 0) XORWOW, idx = round(u * (n-1)), repeats rejected) read from a table of
//                    the 3 uniforms per trial that depends only on (seed, trial) and is generated ONCE per context with
//                    the same curand call; 3-point rigid fit (procrustesKernel :998-1102) solved in closed form with
//                    Horn's quaternion method (largest eigenvector of the 4x4 profile matrix, cyclic Jacobi) instead of
//                    the reference's approximate McAdams SVD — same least-squares rotation, always orthonormal.
//   k_ransac_eval    (pair, 256-trial block): points staged through shared memory, every thread scores one trial
//                    (ransacEvalModelKernel :1183-1200: inlier <=> |B - T A| <= dist_thresh); block arg-max, one 64-bit
//                    atomicMax per block on (count << 32 | ~trial)  => max count, ties -> LOWEST trial id (the
//                    reference's findBestTrial :1202-1217 is racy, SURVEY.md Q8).
//   k_ransac_inliers per pair: inlier test of the winning pose, order-preserving compaction of the ids
//                    (host loop :1293-1302).
#include <curand_kernel.h>
#include <algorithm>
#include <vector>
#include <math.h>
#include "bt_common.cuh"

namespace bt {

struct RansacPair { const float4* A; const float4* B; int n; int out_off; };

__global__ void k_ransac_table(float* u3, int n_trials, unsigned long long seed) {
	const int t = blockIdx.x * blockDim.x + threadIdx.x;
	if (t >= n_trials) return;
	curandState st;
	curand_init(seed, (unsigned long long)t, 0ull, &st);
	u3[3 * t + 0] = curand_uniform(&st);
	u3[3 * t + 1] = curand_uniform(&st);
	u3[3 * t + 2] = curand_uniform(&st);
}

// Largest-eigenvalue eigenvector of a symmetric 4x4 (cyclic Jacobi, fp32).
__device__ void sym4_max_eigvec(float Nm[4][4], float q[4]) {
	float V[4][4] = { { 1, 0, 0, 0 }, { 0, 1, 0, 0 }, { 0, 0, 1, 0 }, { 0, 0, 0, 1 } };
	for (int sweep = 0; sweep < 8; sweep++) {
		float off = 0.f;
		for (int p = 0; p < 4; p++) for (int r = p + 1; r < 4; r++) off += Nm[p][r] * Nm[p][r];
		if (off < 1e-22f) break;
		for (int p = 0; p < 3; p++) {
			for (int r = p + 1; r < 4; r++) {
				const float apq = Nm[p][r];
				if (fabsf(apq) < 1e-30f) continue;
				const float theta = (Nm[r][r] - Nm[p][p]) / (2.0f * apq);
				const float t = (theta >= 0.f ? 1.0f : -1.0f) / (fabsf(theta) + sqrtf(theta * theta + 1.0f));
				const float c = rsqrtf(t * t + 1.0f), s = t * c;
				for (int k = 0; k < 4; k++) { const float akp = Nm[k][p], akq = Nm[k][r]; Nm[k][p] = c * akp - s * akq; Nm[k][r] = s * akp + c * akq; }
				for (int k = 0; k < 4; k++) { const float apk = Nm[p][k], aqk = Nm[r][k]; Nm[p][k] = c * apk - s * aqk; Nm[r][k] = s * apk + c * aqk; }
				for (int k = 0; k < 4; k++) { const float vkp = V[k][p], vkq = V[k][r]; V[k][p] = c * vkp - s * vkq; V[k][r] = s * vkp + c * vkq; }
			}
		}
	}
	int best = 0;
	for (int k = 1; k < 4; k++) if (Nm[k][k] > Nm[best][best]) best = k;
	for (int k = 0; k < 4; k++) q[k] = V[k][best];
}

__global__ void __launch_bounds__(256) k_ransac_model(const RansacPair* __restrict__ pairs, int n_trials, const float* __restrict__ u3, float* __restrict__ poses, int* __restrict__ good) {
	const int pair = blockIdx.y, t = blockIdx.x * blockDim.x + threadIdx.x;
	if (t >= n_trials) return;
	const RansacPair pr = pairs[pair];
	float* P = poses + ((size_t)pair * n_trials + t) * 12;
	good[(size_t)pair * n_trials + t] = 0;
	if (pr.n < 3) return;
	int id[3];
	for (int k = 0; k < 3; k++) id[k] = (int)roundf(u3[3 * t + k] * (float)(pr.n - 1));
	if (id[0] == id[1] || id[1] == id[2] || id[0] == id[2]) return;
	if (id[0] < 0 || id[1] < 0 || id[2] < 0 || id[0] >= pr.n || id[1] >= pr.n || id[2] >= pr.n) return;
	float3 s[3], d[3], sm = make_float3(0.f, 0.f, 0.f), dm = make_float3(0.f, 0.f, 0.f);
	for (int k = 0; k < 3; k++) {
		const float4 a = __ldg(pr.A + id[k]), b = __ldg(pr.B + id[k]);
		s[k] = make_float3(a.x, a.y, a.z); d[k] = make_float3(b.x, b.y, b.z);
		sm.x += a.x; sm.y += a.y; sm.z += a.z; dm.x += b.x; dm.y += b.y; dm.z += b.z;
	}
	sm.x /= 3.f; sm.y /= 3.f; sm.z /= 3.f; dm.x /= 3.f; dm.y /= 3.f; dm.z /= 3.f;
	float S[3][3] = { { 0, 0, 0 }, { 0, 0, 0 }, { 0, 0, 0 } };   // S[a][b] = sum src_a * dst_b  (cuda_ransac.cu:1027-1046)
	for (int k = 0; k < 3; k++) {
		const float sx = s[k].x - sm.x, sy = s[k].y - sm.y, sz = s[k].z - sm.z, dx = d[k].x - dm.x, dy = d[k].y - dm.y, dz = d[k].z - dm.z;
		S[0][0] += sx * dx; S[0][1] += sx * dy; S[0][2] += sx * dz;
		S[1][0] += sy * dx; S[1][1] += sy * dy; S[1][2] += sy * dz;
		S[2][0] += sz * dx; S[2][1] += sz * dy; S[2][2] += sz * dz;
	}
	float Nm[4][4];
	Nm[0][0] = S[0][0] + S[1][1] + S[2][2];
	Nm[0][1] = Nm[1][0] = S[1][2] - S[2][1];
	Nm[0][2] = Nm[2][0] = S[2][0] - S[0][2];
	Nm[0][3] = Nm[3][0] = S[0][1] - S[1][0];
	Nm[1][1] = S[0][0] - S[1][1] - S[2][2];
	Nm[1][2] = Nm[2][1] = S[0][1] + S[1][0];
	Nm[1][3] = Nm[3][1] = S[2][0] + S[0][2];
	Nm[2][2] = -S[0][0] + S[1][1] - S[2][2];
	Nm[2][3] = Nm[3][2] = S[1][2] + S[2][1];
	Nm[3][3] = -S[0][0] - S[1][1] + S[2][2];
	float q[4];
	sym4_max_eigvec(Nm, q);
	const float qn = rsqrtf(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
	const float w = q[0] * qn, x = q[1] * qn, y = q[2] * qn, z = q[3] * qn;
	float R[9] = { 1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y),
	               2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x),
	               2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y) };
	if (!(isfinite(R[0]) && isfinite(R[4]) && isfinite(R[8]))) return;
	P[0] = R[0]; P[1] = R[1]; P[2] = R[2]; P[3] = dm.x - (R[0] * sm.x + R[1] * sm.y + R[2] * sm.z);
	P[4] = R[3]; P[5] = R[4]; P[6] = R[5]; P[7] = dm.y - (R[3] * sm.x + R[4] * sm.y + R[5] * sm.z);
	P[8] = R[6]; P[9] = R[7]; P[10] = R[8]; P[11] = dm.z - (R[6] * sm.x + R[7] * sm.y + R[8] * sm.z);
	good[(size_t)pair * n_trials + t] = 1;
}

static constexpr int kEvalPts = 1024;   // points staged per shared-memory chunk (2 x 16 KB)
static constexpr int kEvalCheck = 128;   // points between two looks at the best count found so far

// Counts the inliers of every trial (one thread per trial, the points broadcast from shared memory).  Two things keep the
// instruction count down - the kernel is issue-bound, ~2000 trials x ~1500 points x 45 pairs:
//  * `sqrtf(d2) <= thresh` is evaluated as `d2 <= d2_max` with d2_max the largest float whose correctly rounded square root
//    is <= thresh (computed on the host): same truth value for every float, no square root;
//  * a trial stops as soon as it can no longer reach the best count any trial of this pair has finished with so far
//    (count + points left < best): it cannot win and it cannot tie, so the winner (max count, then lowest trial) is unchanged.
// two points side by side: sm_90 has no packed f32x2 arithmetic, so each helper is two scalar IEEE operations (the _rn intrinsics keep
// nvcc from contracting them into other forms)
__device__ __forceinline__ float2 pk2(float lo, float hi) { return make_float2(lo, hi); }
__device__ __forceinline__ float2 mul2(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ float2 fma2(float2 a, float2 b, float2 c) { return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y)); }
__device__ __forceinline__ float2 add2(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ float2 sub2(float2 a, float2 b) { return make_float2(__fsub_rn(a.x, b.x), __fsub_rn(a.y, b.y)); }

// One thread per trial, the pair's points broadcast from shared memory, two points per loop step (the kernel is issue-bound: 2000
// trials x ~2-3 k candidate points x 45 pairs).  Every point gets exactly the operations, in exactly the order, of the scalar
// expression `pb - (P[0]*pa.x + P[1]*pa.y + P[2]*pa.z + P[3])` as nvcc contracts it (mul y, fma x, fma z, add t; squares: mul dy, fma dx, fma
// dz), so the inlier counts are bit-identical to the scalar version that was pinned against the reference's ransacMultiPairGPU.
__global__ void __launch_bounds__(256) k_ransac_eval(const RansacPair* __restrict__ pairs, int n_trials, const float* __restrict__ poses, const int* __restrict__ good,
                                                      float d2_max, unsigned long long* __restrict__ best) {
	__shared__ float4 sP[3][kEvalPts / 2];      // per PAIR of points: (ax, ax', ay, ay') | (az, az', bx, bx') | (by, by', bz, bz')
	const int pair = blockIdx.y, t = blockIdx.x * blockDim.x + threadIdx.x;
	const RansacPair pr = pairs[pair];
	const bool live = t < n_trials && good[(size_t)pair * n_trials + t] != 0;
	float2 P2[12];
	{
		const float* Pg = poses + ((size_t)pair * n_trials + t) * 12;
		for (int k = 0; k < 12; k++) { const float v = live ? Pg[k] : 0.f; P2[k] = pk2(v, v); }
	}
	int count = 0;
	bool running = live;
	for (int base = 0; base < pr.n; base += kEvalPts) {
		const int m = min(kEvalPts, pr.n - base);
		__syncthreads();
		for (int k = threadIdx.x; k < ((m + 1) & ~1); k += blockDim.x) {
			float4 a4 = make_float4(0.f, 0.f, 0.f, 0.f), b4 = make_float4(NAN, NAN, NAN, 0.f);      // padding point of an odd tail: its squared distance is NaN, never <= d2_max (+inf included)
			if (k < m) { a4 = __ldg(pr.A + base + k); b4 = __ldg(pr.B + base + k); }
			const int j = k >> 1, h = k & 1;
			float* p0 = reinterpret_cast<float*>(&sP[0][j]); float* p1 = reinterpret_cast<float*>(&sP[1][j]); float* p2 = reinterpret_cast<float*>(&sP[2][j]);
			p0[h] = a4.x; p0[2 + h] = a4.y; p1[h] = a4.z; p1[2 + h] = b4.x; p2[h] = b4.y; p2[2 + h] = b4.z;
		}
		__syncthreads();
		for (int k0 = 0; k0 < m && running; k0 += kEvalCheck) {
			const int k1 = min(m, k0 + kEvalCheck);
#pragma unroll 4
			for (int j = k0 >> 1; j < (k1 + 1) >> 1; j++) {
				const float4 u = sP[0][j], v = sP[1][j], w = sP[2][j];
				const float2 ax = pk2(u.x, u.y), ay = pk2(u.z, u.w), az = pk2(v.x, v.y), bx = pk2(v.z, v.w), by = pk2(w.x, w.y), bz = pk2(w.z, w.w);
				const float2 dx = sub2(bx, add2(fma2(P2[2], az, fma2(P2[0], ax, mul2(P2[1], ay))), P2[3]));
				const float2 dy = sub2(by, add2(fma2(P2[6], az, fma2(P2[4], ax, mul2(P2[5], ay))), P2[7]));
				const float2 dz = sub2(bz, add2(fma2(P2[10], az, fma2(P2[8], ax, mul2(P2[9], ay))), P2[11]));
				const float2 d2 = fma2(dz, dz, fma2(dx, dx, mul2(dy, dy)));
				count += (d2.x <= d2_max) ? 1 : 0;
				count += (d2.y <= d2_max) ? 1 : 0;
			}
			// best[pair] only ever holds counts of trials that have seen ALL points
			const int best_cnt = (int)(__ldcg(best + pair) >> 32);
			if (count + (pr.n - base - k1) < best_cnt) running = false;
		}
		if (running && base + m >= pr.n) {     // finished: publish (count, lowest trial) right away so that slower trials can stop early
			atomicMax(best + pair, ((unsigned long long)(unsigned)count << 32) | (unsigned long long)(0xFFFFFFFFu - (unsigned)t));
		}
	}
}

__global__ void __launch_bounds__(256) k_ransac_inliers(const RansacPair* __restrict__ pairs, int n_trials, const float* __restrict__ poses, float thresh,
                                                         const unsigned long long* __restrict__ best, int32_t* __restrict__ inlier_ids, int32_t* __restrict__ n_inliers,
                                                         int32_t* __restrict__ best_trial_out) {
	__shared__ int s_warp[8];
	__shared__ int s_base;
	const int pair = blockIdx.x;
	const RansacPair pr = pairs[pair];
	const unsigned long long key = best[pair];
	const int cnt = (int)(key >> 32);
	const int trial = (key == 0ull) ? -1 : (int)(0xFFFFFFFFu - (unsigned)(key & 0xFFFFFFFFull));
	if (threadIdx.x == 0) { s_base = 0; if (best_trial_out) best_trial_out[pair] = trial; }
	__syncthreads();
	if (trial < 0 || cnt == 0) { if (threadIdx.x == 0) n_inliers[pair] = 0; return; }
	float P[12];
	{ const float* Pg = poses + ((size_t)pair * n_trials + trial) * 12; for (int k = 0; k < 12; k++) P[k] = Pg[k]; }
	const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
	for (int base = 0; base < pr.n; base += blockDim.x) {
		const int k = base + threadIdx.x;
		bool in = false;
		if (k < pr.n) {
			const float4 a = __ldg(pr.A + k), b = __ldg(pr.B + k);
			const float dx = b.x - (P[0] * a.x + P[1] * a.y + P[2] * a.z + P[3]);
			const float dy = b.y - (P[4] * a.x + P[5] * a.y + P[6] * a.z + P[7]);
			const float dz = b.z - (P[8] * a.x + P[9] * a.y + P[10] * a.z + P[11]);
			in = sqrtf(dx * dx + dy * dy + dz * dz) <= thresh;
		}
		const unsigned bal = __ballot_sync(0xffffffffu, in);
		if (lane == 0) s_warp[wid] = __popc(bal);
		__syncthreads();
		int off = s_base;
		for (int w = 0; w < wid; w++) off += s_warp[w];
		if (in) inlier_ids[pr.out_off + off + __popc(bal & ((1u << lane) - 1u))] = k;
		__syncthreads();
		if (threadIdx.x == 0) { int tsum = 0; for (int w = 0; w < (int)(blockDim.x >> 5); w++) tsum += s_warp[w]; s_base += tsum; }
		__syncthreads();
	}
	if (threadIdx.x == 0) n_inliers[pair] = s_base;
}

struct RansacState {
	bool ready = false;
	int max_pairs = 0, max_pts = 0, max_trials = 0;
	DevBuf table, poses, good, best, best_trial;
	TableBlock<> pairs;                       // the pair table of a bt_ransac_pairs call
	unsigned long long table_seed = ~0ull;
	int table_trials = 0;
	int last_pairs = 0, last_trials = 0;      // shape of the last run's per-trial poses, flags and keys (bt_ransac_debug_trials)
};
void StateDeleter::operator()(RansacState* r) const { delete r; }
struct PairTable : TableLayout { Slice<RansacPair> pairs; };
static PairTable pair_table(size_t n_pairs) { PairTable t; t.pairs = t.add<RansacPair>(n_pairs); return t; }

// shared by the host-pointer API below and the fused matcher pipeline (pairs table already on the device)
int ransac_run_device(bt_ctx* ctx, const RansacPair* d_pairs, int n_pairs, int n_trials, float dist_thresh, uint64_t seed,
                      int32_t* inlier_ids_out, int32_t* n_inliers_out, cudaStream_t stream) {
	RansacState* r = ctx->ransac.get();
	BT_REQUIRE(r && r->ready, BT_ERR_INVALID_ARG, "ransac: call bt_ransac_reserve (successfully) first");
	BT_REQUIRE(n_pairs <= r->max_pairs && n_trials <= r->max_trials && n_trials > 0, BT_ERR_CAPACITY, "ransac: %d pairs / %d trials exceed the reserved %d / %d", n_pairs, n_trials, r->max_pairs, r->max_trials);
	if (r->table_seed != seed || r->table_trials < n_trials) {
		k_ransac_table<<<(r->max_trials + 255) / 256, 256, 0, stream>>>(r->table.as<float>(), r->max_trials, (unsigned long long)seed);
		r->table_seed = seed; r->table_trials = r->max_trials;
	}
	BT_CUDA(cudaMemsetAsync(r->best.p, 0, sizeof(unsigned long long) * n_pairs, stream));
	const float d2_max = sqrt_le_max(dist_thresh);      // (sqrtf is correctly rounded on the device too: the kernel compares squares)
	const dim3 grid((n_trials + 255) / 256, n_pairs);
	k_ransac_model<<<grid, 256, 0, stream>>>(d_pairs, n_trials, r->table.as<float>(), r->poses.as<float>(), r->good.as<int>());
	k_ransac_eval<<<grid, 256, 0, stream>>>(d_pairs, n_trials, r->poses.as<float>(), r->good.as<int>(), d2_max, r->best.as<unsigned long long>());
	k_ransac_inliers<<<n_pairs, 256, 0, stream>>>(d_pairs, n_trials, r->poses.as<float>(), dist_thresh, r->best.as<unsigned long long>(), inlier_ids_out, n_inliers_out, r->best_trial.as<int32_t>());
	BT_CUDA(cudaGetLastError());
	r->last_pairs = n_pairs; r->last_trials = n_trials;
	return BT_OK;
}

}  // namespace bt

using namespace bt;

extern "C" int bt_ransac_reserve(bt_ctx* ctx, int max_pairs, int max_pts, int max_trials) {
	BT_REQUIRE(ctx && max_pairs > 0 && max_pts > 0 && max_trials > 0, BT_ERR_INVALID_ARG, "bt_ransac_reserve: bad arguments");
	RansacState* r;
	BT_TRY(take_state(ctx, &bt_ctx::ransac, &r));
	BT_TRY(r->table.alloc(sizeof(float) * 3 * max_trials));
	BT_TRY(r->poses.alloc(sizeof(float) * 12 * (size_t)max_pairs * max_trials));
	BT_TRY(r->good.alloc(sizeof(int) * (size_t)max_pairs * max_trials));
	BT_TRY(r->best.alloc(sizeof(unsigned long long) * max_pairs));
	BT_TRY(r->best_trial.alloc(sizeof(int32_t) * max_pairs));
	BT_TRY(r->pairs.reserve(pair_table(max_pairs).total));
	r->table_seed = ~0ull; r->table_trials = 0; r->last_pairs = r->last_trials = 0;
	r->max_pairs = max_pairs; r->max_pts = max_pts; r->max_trials = max_trials;
	r->ready = true;
	return BT_OK;
}

extern "C" int bt_ransac_pairs(bt_ctx* ctx, int n_pairs, const float* const* ptsA, const float* const* ptsB, const int* n_pts, int n_trials, float dist_thresh,
                               uint64_t seed, int32_t* inlier_ids_out, int32_t* n_inliers_out, void* stream_) {
	RansacState* r;
	BT_TRY(state_of(ctx, &bt_ctx::ransac, "bt_ransac_pairs", "bt_ransac_reserve", &r));
	BT_REQUIRE(ptsA && ptsB && n_pts && inlier_ids_out && n_inliers_out && n_pairs > 0, BT_ERR_INVALID_ARG, "bt_ransac_pairs: NULL argument");
	cudaStream_t stream = (cudaStream_t)stream_;
	BT_REQUIRE(n_pairs <= r->max_pairs, BT_ERR_CAPACITY, "bt_ransac_pairs: %d pairs > reserved %d", n_pairs, r->max_pairs);
	const PairTable t = pair_table(n_pairs);
	BT_TRY(r->pairs.begin("bt_ransac_pairs", t));
	RansacPair* hp = r->pairs.host(t.pairs);
	int off = 0;
	for (int p = 0; p < n_pairs; p++) {
		BT_REQUIRE(n_pts[p] >= 0 && n_pts[p] <= r->max_pts, BT_ERR_CAPACITY, "bt_ransac_pairs: pair %d has %d points > reserved %d", p, n_pts[p], r->max_pts);
		hp[p].A = reinterpret_cast<const float4*>(ptsA[p]); hp[p].B = reinterpret_cast<const float4*>(ptsB[p]); hp[p].n = n_pts[p]; hp[p].out_off = off;
		off += n_pts[p];
	}
	BT_TRY(r->pairs.send(0, t.pairs.end(), stream));
	BT_TRY(r->pairs.in_flight(stream));
	return ransac_run_device(ctx, r->pairs.dev(t.pairs), n_pairs, n_trials, dist_thresh, seed, inlier_ids_out, n_inliers_out, stream);
}

// Debug/parity aid: the 3 uniforms per trial the sampler uses (seed as in bt_ransac_pairs), and the winning trial ids of the last call.
extern "C" int bt_ransac_debug(bt_ctx* ctx, float* u3_out, int n_trials, int32_t* best_trial_out, int n_pairs) {
	RansacState* r;
	BT_TRY(state_of(ctx, &bt_ctx::ransac, "bt_ransac_debug", "bt_ransac_reserve", &r));
	BT_CUDA(cudaDeviceSynchronize());
	if (u3_out) BT_CUDA(cudaMemcpy(u3_out, r->table.p, sizeof(float) * 3 * std::min(n_trials, r->table_trials), cudaMemcpyDeviceToHost));
	if (best_trial_out) BT_CUDA(cudaMemcpy(best_trial_out, r->best_trial.p, sizeof(int32_t) * std::min(n_pairs, r->max_pairs), cudaMemcpyDeviceToHost));
	return BT_OK;
}

// Debug/parity aid: one pair's per-trial poses ([n_trials][12], row-major [R | t]) and good flags of the last call (n_trials at most that
// call's), and the inlier count its winning key holds (-1 when no trial finished).
extern "C" int bt_ransac_debug_trials(bt_ctx* ctx, int pair, int n_trials, float* poses_out, int32_t* good_out, int32_t* best_count_out) {
	RansacState* r;
	BT_TRY(state_of(ctx, &bt_ctx::ransac, "bt_ransac_debug_trials", "bt_ransac_reserve", &r));
	BT_REQUIRE(pair >= 0 && pair < r->last_pairs, BT_ERR_INVALID_ARG, "bt_ransac_debug_trials: pair %d of a last call with %d pairs", pair, r->last_pairs);
	BT_REQUIRE(n_trials >= 0 && n_trials <= r->last_trials, BT_ERR_INVALID_ARG, "bt_ransac_debug_trials: %d trials, the last call ran %d", n_trials, r->last_trials);
	BT_CUDA(cudaDeviceSynchronize());
	const int nt = n_trials;
	const size_t row = (size_t)pair * r->last_trials;
	if (poses_out && nt) BT_CUDA(cudaMemcpy(poses_out, r->poses.as<float>() + row * 12, sizeof(float) * 12 * nt, cudaMemcpyDeviceToHost));
	if (good_out && nt) BT_CUDA(cudaMemcpy(good_out, r->good.as<int>() + row, sizeof(int32_t) * nt, cudaMemcpyDeviceToHost));
	if (best_count_out) {
		unsigned long long key;
		BT_CUDA(cudaMemcpy(&key, r->best.as<unsigned long long>() + pair, sizeof(key), cudaMemcpyDeviceToHost));
		*best_count_out = key == 0ull ? -1 : (int32_t)(key >> 32);
	}
	return BT_OK;
}
