// solver.cu — H100-native Gauss-Newton x PCG pose-graph solve for a BATCH of independent tracking windows.
//
// Replaces (behind the C-ABI in include/bundletrack_b200.h) the reference's OptimizerGpu::optimizeFrames
// (/root/reference/src/cuda/LossGPU.cu:53-139) -> CUDACache::storeFrame (CUDACache.cpp:76-88) -> SBA::align
// (SBA.cpp:81-139) -> CUDASolverBundling::solve (Solver/CUDASolverBundling.cpp:190-288) -> solveBundlingStub
// (Solver/SolverBundling.cu:931-1003): ~260 kernel launches, ~75 memsets, 7 blocking copies and ~110 cudaMalloc per
// window there; THREE launches per BATCH here, none of them allocating:
//
//   k_prep_count   one CTA per 1024 quarter-res pixels of a (window, frame): number of valid pixels of the block.
//   k_prep_frames  same grid: quarter-res cache (one 16-byte texel {depth, normal} per pixel: a bilinear tap is one
//                  128-bit load and rebuilds the camera point) + an order-preserving COMPACTED list of the
//                  valid source pixels (the object mask leaves ~10 % of the image valid), + se(3) of the input pose.
//                  Each block's offset in the ordered list = the counts of the blocks before it.
//   (plan)         the LAST CTA of k_prep_frames to finish: per-window tile counts -> exclusive scan -> flat tile list.
//   k_solve        persistent: tiles are (GN iteration, window, pair, pixel chunk), handed out by a queue (the next tile's 48-byte
//                  record is fetched one tile ahead) or - when one iteration's tiles fit the grid - assigned statically (CTA c =
//                  tile c of every iteration).  A tile evaluates point-to-plane residuals/Jacobians for its chunk and reduces a 6x6
//                  system in the TARGET camera frame; every window also has two SPARSE tiles per iteration (the moment sums of half
//                  of its correspondence groups each: they only need the poses, so they run next to the dense tiles); the CTA that
//                  retires a window's last tile of an iteration runs that window's "tail": table loads as asynchronous copies next
//                  to the per-pair sums, assembly of the (6(N-1))^2 normal equations in shared memory (dense blocks + explicit
//                  sparse blocks from per-pair moment sums), the PCG steps with one thread per unknown, the pose update, and the
//                  release of the window's next iteration.  Tiles of iteration k+1 wait on a per-window flag, so all GN iterations
//                  of all windows flow through ONE launch with no host round trip.
//
// Maths restated from the reference (see oracle/solver_oracle.c for the statement-by-statement CPU version):
//   * dense residual/gates: findDenseCorr (Solver/SolverBundlingDenseUtil.h:78-110), bilinear taps
//     (Solver/ICPUtil.h:83-110, zeros blended - SURVEY.md Q6), Huber weight (Solver/SolverBundlingUtil.h:24-39).
//   * Jacobian rows: computeJacobianBlockRow_i/j (Solver/SolverBundlingEquationsLie.h:214-230) reduce analytically to
//     J_i = [N, q x N], J_j = -J_i with N = R_i n_tgt and q the source point in the model frame (derivation in
//     DESIGN.md), so one symmetric 6x6 + one 6-vector per pair carries all four blocks addToLocalSystem writes
//     (SolverBundlingDenseUtil.h:217-285).  FlipJtJ (SolverBundling.cu:49-58) erases cross blocks with
//     target > source; `compat_flip` reproduces that (SURVEY.md Q2).
//   * sparse term: evalMinusJTFDevice / applyJDevice / applyJTDevice (SolverBundlingEquationsLie.h:60-211) with the
//     Huber weight on the gradient and the Jacobi preconditioner only (SURVEY.md Q3/Q4); J^T J is formed explicitly
//     from per-pair moment sums instead of matrix-free, which changes summation order only.
//   * PCG recurrences and the 1e-6 guards: SolverBundling.cu:575-818; update x <- log(exp(delta) exp(x)):
//     Solver/LieDerivUtil.h:126-194,276-282.
#include <algorithm>
#include <math.h>
#include <stddef.h>
#include <stdlib.h>
#include <chrono>
#include "bt_common.cuh"
#include "bt_scan.cuh"

namespace bt {

#ifndef BT_SOLVE_MIN_CTAS
#define BT_SOLVE_MIN_CTAS 2
#endif
static constexpr int kTileVals = 28;          // 21 (sym 6x6) + 6 (rhs) + 1 (#correspondences found)
static constexpr int kGrpVals = 44;           // sparse moment sums per pair group
static constexpr int kMaxFrames = 32;
static constexpr int kSparseTiles = 2;        // sparse tiles per window and GN iteration: each takes a contiguous share of the window's (i,j) groups (45 groups = 23 + 22: one round of
                                              // 32 eight-lane teams each instead of two; as one tile it was the longest tile of a lone window)
static constexpr size_t kTailSmemMax = 224 * 1024;   // dynamic shared memory a tail may use (227 KB per CTA minus k_solve's static arrays)
static constexpr float kEps = 0.000001f;      // FLOAT_EPSILON, /root/reference/src/cuda/SolverUtil.h:10

// What turns a quarter-res pixel into its full-res sample and camera-space point (texel_sample / texel_coord)
struct TexelGeom {
	float ifx, ify, icx, icy;         // inverse full-res intrinsics (m_inputIntrinsicsInv)
	float scaleW, scaleH;             // (W-1)/(w-1), (H-1)/(h-1)  (CUDAImageUtil.cu:57-58)
};

// What the frame preparation needs of a window: uploaded before k_prep_frames is launched.
struct WinDesc {
	int n_frames, n_pairs, pair_off, frame_off;
	int tile_off, n_tiles;            // per GN iteration; written by the tile plan (last CTA of k_prep_frames)
	int H, W, w, h;                   // full / quarter resolution
	float fx, fy, cx, cy;             // quarter-res intrinsics (CUDACache.cpp:20-24)
	TexelGeom tg;
	int compat_flip;
	int pad[3];
};

// What arrives with a window's correspondences: uploaded AFTER the frame preparation has been launched (the host scans the
// correspondences while the GPU already works).
struct WinSparse {
	int n_corr, n_groups, corr_off, grp_off, mem_off;      // mem_off: per-frame membership CSR of this window (see SolveArgs::mem)
	int unique_blocks, pad0, pad1;    // 1: no two groups / no two dense pairs share an unordered frame pair => cross blocks need no atomics
};

// One unit of work of k_solve.  Everything the tile's prologue needs travels in the record (frame slots, map pointers, the window's
// tile count), so that claiming a tile costs ONE dependent load - and that one is issued a whole tile ahead (k_solve keeps the next
// record in shared memory).  pair == -2 => the window's sparse tile (moment sums of its correspondences).
struct __align__(16) Tile {
	int win; int pair; int start; int count;
	int tgt_slot; int src_slot;          // global frame slots (frame_off + target / source) of the pair
	int n_tiles_win; int pad;            // tiles of the window per GN iteration (dense + the sparse one)
	const float4* src; const float4* tex;   // compacted source list of the source frame, texel map of the target frame
};

struct SolveArgs {
	const WinDesc* wins;
	const WinSparse* wsp;
	int n_windows;
	// frame slots
	const float* const* depth_ptr;
	const float4* const* normal_ptr;
	const int* frame_win;
	float4* texel;        // [F][npix_max]    the context's own maps (frames prepared by this call)
	float4* src;          // [F][2*npix_max]
	int* nsrc;            // [F]
	float* grp_sums;      // [groups of the batch][kGrpVals] sparse moment sums of the current GN iteration (written by the window's sparse tile)
	const float4* const* texel_tab;   // [F] where each frame slot's texel map / source list lives: the arrays above, or a
	const float4* const* src_tab;     //     frame-cache slot built earlier by bt_frame_cache_store
	const int* const* nsrc_cached;    // [F] cached frame: address of its source count, else nullptr
	const float* pose_in; // [F][16]
	float* x;             // [F][6]  rot, trans
	float* T;             // [F][12] row-major 3x4 cam->model
	float* pose_out;      // [F][16]
	int npix_max;
	// correspondences, grouped by (i,j)
	const bt_entryj* corr;
	const int* grp_i; const int* grp_j; const int* grp_start;   // grp_start has n_groups+1 entries per window
	const uint2* pairs;   // (target, source)
	const int* pair_win;  // owning window of every entry of `pairs`
	const int* pair_src_slot;   // global frame slot (frame_off + source) of every entry of `pairs`
	// per-window CSR built on the host: for every frame f, first the correspondence groups touching f, then the dense
	// pairs touching f.  Layout at mem_off: fg_start[N+1], fp_start[N+1], items[2G] (g | role<<16), items[2P] (p | role<<16)
	const int* mem;
	// schedule
	Tile* tiles; int* n_tiles_total; int max_tiles;
	int* pair_tile0; int* pair_ntile;   // per (window, pair): first tile (relative to the window's tile_off) and tile count
	float* partial;       // [max_tiles][kTileVals]
	int* tiles_done;      // [n_windows]
	int* iter_done;       // [n_windows]
	int* queue;           // [1]
	long long* n_src_px;  // [1] stats
	int chunk;
	int grp_in_smem;      // 0: the tail reads the groups' moment sums from global memory (windows too big for shared memory)
	int grid_ctas;        // CTAs k_solve will be launched with (tile planning targets one wave for small batches)
	float d2max;          // largest float whose correctly rounded square root is <= prm.dense_dist_thresh (computed once on the host)
	bt_solver_params prm;
	float* dbg_JtJ; float* dbg_Jtr; int dbg_stride;   // optional dense-system dump (last GN iteration)
	float* dbg_cnt; int dbg_cnt_stride;               // optional per-pair #correspondences found (last GN iteration)
	float* dbg_sys; int dbg_sys_stride;               // optional PCG system dump (last GN iteration): per window A [st][st], rhs, Jacobi diagonal, delta [st] each
	long long* prof; int prof_cap;                    // optional phase timestamps: [0] = record count, then 12 x int64 per record
	// optional device times (bt_solve_enable_timing), %globaltimer ns: [0] prep start (first prep kernel's block 0), [1] prep end (tile
	// plan written), [2] k_solve start (block 0), [3] k_solve end (last CTA).  Stamped inside the kernels: an event recorded between two
	// kernels would cut the step's launch chain.  with_count: k_prep_count runs before k_prep_frames (it stamps [0] then).
	long long* tstamp; int with_count;
};

// ------------------------------------------------------------------------------------------------ device math
struct V3 { float x, y, z; };
__device__ __forceinline__ V3 mk(float x, float y, float z) { V3 v; v.x = x; v.y = y; v.z = z; return v; }
__device__ __forceinline__ V3 operator+(V3 a, V3 b) { return mk(a.x + b.x, a.y + b.y, a.z + b.z); }
__device__ __forceinline__ V3 operator-(V3 a, V3 b) { return mk(a.x - b.x, a.y - b.y, a.z - b.z); }
__device__ __forceinline__ V3 operator*(V3 a, float s) { return mk(a.x * s, a.y * s, a.z * s); }
__device__ __forceinline__ float dot(V3 a, V3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
__device__ __forceinline__ V3 cross(V3 a, V3 b) { return mk(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x); }

// Rodrigues coefficients with the reference's Taylor branches (LieDerivUtil.h:46-70,150-194).
__device__ void so3_coeffs(float theta_sq, float& A, float& B, float& C) {
	if (theta_sq < 1e-8f) { A = 1.0f - 0.16666667f * theta_sq; B = 0.5f; C = 0.16666667f; }
	else if (theta_sq < 1e-6f) {
		C = 0.16666667f * (1.0f - 0.05f * theta_sq);
		A = 1.0f - theta_sq * C;
		B = 0.5f - 0.25f * 0.16666667f * theta_sq;
	} else {
		const float theta = sqrtf(theta_sq), inv = 1.0f / theta;
		A = sinf(theta) * inv;
		B = (1.0f - cosf(theta)) * (inv * inv);
		C = (1.0f - A) * (inv * inv);
	}
}
__device__ void so3_exp_AB(V3 w, float A, float B, float R[9]) {  // rodrigues_so3_exp, LieDerivUtil.h:17-44
	const float wx2 = w.x * w.x, wy2 = w.y * w.y, wz2 = w.z * w.z;
	R[0] = 1.0f - B * (wy2 + wz2); R[4] = 1.0f - B * (wx2 + wz2); R[8] = 1.0f - B * (wx2 + wy2);
	float a = A * w.z, b = B * (w.x * w.y); R[1] = b - a; R[3] = b + a;
	a = A * w.y; b = B * (w.x * w.z); R[2] = b + a; R[6] = b - a;
	a = A * w.x; b = B * (w.y * w.z); R[5] = b - a; R[7] = b + a;
}
// poseToMatrix (LieDerivUtil.h:150-194): T[12] = row-major 3x4 [R | t]
__device__ __forceinline__ void se3_exp(V3 rot, V3 trans, float T[12]) {
	const float theta_sq = dot(rot, rot);
	float A, B, C;
	so3_coeffs(theta_sq, A, B, C);
	const V3 cr = cross(rot, trans);
	V3 t;
	if (theta_sq < 1e-8f) t = trans + cr * 0.5f;
	else t = trans + cr * B + cross(rot, cr) * C;
	float R[9];
	so3_exp_AB(rot, A, B, R);
	T[0] = R[0]; T[1] = R[1]; T[2] = R[2]; T[3] = t.x;
	T[4] = R[3]; T[5] = R[4]; T[6] = R[5]; T[7] = t.y;
	T[8] = R[6]; T[9] = R[7]; T[10] = R[8]; T[11] = t.z;
}
// ln_rotation (LieDerivUtil.h:72-124)
__device__ V3 so3_log(const float R[9]) {
	V3 r = mk((R[7] - R[5]) * 0.5f, (R[2] - R[6]) * 0.5f, (R[3] - R[1]) * 0.5f);
	const float cos_angle = (R[0] + R[4] + R[8] - 1.0f) * 0.5f;
	const float s = sqrtf(dot(r, r));
	if (cos_angle > 0.70710678118654752440f) {
		if (s > 0.0f) r = r * (asinf(s) / s);
	} else if (cos_angle > -0.70710678118654752440f) {
		r = r * (acosf(cos_angle) / s);
	} else {
		const float angle = 3.14159265358979323846f - asinf(s);
		const float d0 = R[0] - cos_angle, d1 = R[4] - cos_angle, d2 = R[8] - cos_angle;
		V3 r2;
		if (fabsf(d0) > fabsf(d1) && fabsf(d0) > fabsf(d2)) r2 = mk(d0, (R[3] + R[1]) * 0.5f, (R[2] + R[6]) * 0.5f);
		else if (fabsf(d1) > fabsf(d2)) r2 = mk((R[3] + R[1]) * 0.5f, d1, (R[7] + R[5]) * 0.5f);
		else r2 = mk((R[2] + R[6]) * 0.5f, (R[7] + R[5]) * 0.5f, d2);
		if (dot(r2, r) < 0.0f) r2 = r2 * -1.0f;
		r = r2 * (angle / sqrtf(dot(r2, r2)));
	}
	return r;
}
// matrixToPose (LieDerivUtil.h:126-148); T = row-major 3x4
__device__ __forceinline__ void se3_log(const float T[12], V3& rot, V3& trans) {
	const float R[9] = { T[0], T[1], T[2], T[4], T[5], T[6], T[8], T[9], T[10] };
	const V3 t = mk(T[3], T[7], T[11]);
	rot = so3_log(R);
	const float theta = sqrtf(dot(rot, rot));
	float shtot = 0.5f;
	if (theta > 0.00001f) shtot = sinf(theta * 0.5f) / theta;
	const V3 half = rot * -0.5f;
	float A, B, C, Hm[9];
	so3_coeffs(dot(half, half), A, B, C);
	so3_exp_AB(half, A, B, Hm);
	V3 tr = mk(Hm[0] * t.x + Hm[1] * t.y + Hm[2] * t.z, Hm[3] * t.x + Hm[4] * t.y + Hm[5] * t.z, Hm[6] * t.x + Hm[7] * t.y + Hm[8] * t.z);
	if (theta > 0.001f) tr = tr - rot * (dot(t, rot) * (1.0f - 2.0f * shtot) / dot(rot, rot));
	else tr = tr - rot * (dot(t, rot) / 24.0f);
	trans = tr * (1.0f / (2.0f * shtot));
}
__device__ __forceinline__ float huber_w(float e, float delta) {  // rho.y of huberLoss, SolverBundlingUtil.h:24-39
	return (e <= delta * delta) ? 1.0f : delta / sqrtf(e);
}
// The dense pixel loop's quotients.  Default: correctly rounded (__frcp_rn, IEEE Huber weight).  -DBT_DENSE_FAST_RCP builds the variant
// with one MUFU reciprocal (1 ulp) per quotient: the reference itself is compiled with -use_fast_math (/root/reference/CMakeLists.txt:7),
// but individual gate-sensitive windows move by ~1e-4 either way between the two variants, so the shipped default keeps the
// arithmetic the committed parity windows were pinned with.
#ifndef BT_DENSE_FAST_RCP      // default: correctly rounded reciprocals / IEEE Huber weight; -DBT_DENSE_FAST_RCP builds the MUFU variant (A/B in DESIGN.md)
__device__ __forceinline__ float rcp_fast(float x) { return __frcp_rn(x); }
__device__ __forceinline__ float huber_w_fast(float e, float delta) { return huber_w(e, delta); }
#else
__device__ __forceinline__ float rcp_fast(float x) { float r; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }
__device__ __forceinline__ float huber_w_fast(float e, float delta) {
	float r; asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(e));
	return (e <= delta * delta) ? 1.0f : delta * r;
}
#endif
// ---- the quarter-resolution texel map, one 16-byte record per pixel: {d', nx, ny, nz}.  d' is the nearest-neighbour depth sample
// when it lies inside the full-resolution image and is >= 0.1, else 0; the normal is the sample's as stored (0 outside the image).
// The camera-space point is not stored: it is rebuilt from the pixel's integer sample position with the operation order
// ifx * (xi * d) + icx * d, pinned (no contraction choice left to the compiler), so the builders' source records and the dense
// tap's rebuilt points are the same floats.  Every writer and reader of the record goes through the helpers below.
// full-resolution sample position of quarter-res coordinate x (resampleFloat4 nearest, CUDAImageUtil.cu:82-99)
__device__ __forceinline__ unsigned texel_sample(int x, float scale) { return __float2uint_rz(__fmaf_rn((float)x, scale, 0.5f)); }
// one camera-space coordinate of the point behind sample position xi at depth d (convertDepthFloatToCameraSpaceFloat4)
__device__ __forceinline__ float texel_coord(unsigned xi, float d, float inv_f, float inv_c) { return __fmaf_rn(inv_c, d, __fmul_rn(inv_f, __fmul_rn((float)xi, d))); }
__device__ __forceinline__ bool texel_sample_xy(const TexelGeom& g, int W, int H, int w, int idx, unsigned& xi, unsigned& yi) {
	xi = texel_sample(idx % w, g.scaleW); yi = texel_sample(idx / w, g.scaleH);
	return xi < (unsigned)W && yi < (unsigned)H;
}
// Loads the sample of quarter-res pixel idx: returns the texel record and sets cp to the camera point ({0,0,0} and w = 0 when d' = 0).
__device__ __forceinline__ float4 texel_build(const TexelGeom& g, int W, int H, int w, const float* __restrict__ depth, const float4* __restrict__ normal,
                                              int idx, float4& cp, float4& nr) {
	unsigned xi, yi;
	float d = 0.f;
	cp = make_float4(0.f, 0.f, 0.f, 0.f); nr = make_float4(0.f, 0.f, 0.f, 0.f);
	if (texel_sample_xy(g, W, H, w, idx, xi, yi)) {
		const size_t sidx = (size_t)yi * W + xi;
		const float ds = __ldg(depth + sidx);
		nr = __ldg(normal + sidx);
		if (ds >= 0.1f) { d = ds; cp = make_float4(texel_coord(xi, d, g.ifx, g.icx), texel_coord(yi, d, g.ify, g.icy), d, 1.0f); }
	}
	return make_float4(d, nr.x, nr.y, nr.z);
}
// Depth of the sample of quarter-res pixel idx as texel_build sees it (0 outside the image or below 0.1): the counting sweeps use
// it so that they agree bit for bit with the build.
__device__ __forceinline__ float texel_depth(const TexelGeom& g, int W, int H, int w, const float* __restrict__ depth, int idx) {
	unsigned xi, yi;
	if (!texel_sample_xy(g, W, H, w, idx, xi, yi)) return 0.f;
	const float d = __ldg(depth + (size_t)yi * W + xi);
	return (d >= 0.1f) ? d : 0.f;
}

struct FrameGeom { int W, H, w, h; TexelGeom tg; };

// Programmatic dependent launch (DESIGN §3.4): a step's kernels are launched as one chain, each one allowed to start while its
// predecessor on the stream finishes.  chain_wait() returns once the predecessor has completed and its writes are visible; before it a
// kernel only reads memory that no kernel still in flight writes.  chain_release() lets the successor's CTAs launch (they then sit in
// their own chain_wait); a grid whose CTAs exit without it releases the successor at exit.  Without a programmatic predecessor (a
// plain launch, a copy or an event wait in between) both are no-ops.
__device__ __forceinline__ void chain_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void chain_release() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ long long global_ns() { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return (long long)t; }

// A frame's maps are built one CTA per 1024 quarter-res pixels (block b, 1024 threads) in two launches.  The compacted source list
// keeps pixel order (fixed summation order downstream), so each block needs the number of valid pixels before it: the first launch
// counts the valid pixels of every block (frame_block_count), the second turns the counts of the blocks before it into the block's
// offset in the list and writes its slice of the texel map and its source records there (frame_block_build).  blk_cnt is the
// frame's row of block counts.
__device__ __forceinline__ void frame_block_count(const FrameGeom& g, const float* __restrict__ depth, float dmin, float dmax, int b, int* __restrict__ blk_cnt) {
	const int npix = g.w * g.h, idx = b * 1024 + threadIdx.x;
	__shared__ int s_w[32];
	bool valid = false;
	if (idx < npix) {
		const float z = texel_depth(g.tg, g.W, g.H, g.w, depth, idx);
		valid = (z > dmin && z < dmax);
	}
	const unsigned bal = __ballot_sync(0xffffffffu, valid);
	if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = __popc(bal);
	__syncthreads();
	if (threadIdx.x < 32) {
		int t = s_w[threadIdx.x];
#pragma unroll
		for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
		if (threadIdx.x == 0) blk_cnt[b] = t;
	}
}
// The frame's last block also writes the source count to *nsrc.  Blocks past the end of the frame do nothing.  The pixel's depth and
// normal samples are loaded before chain_wait(): in k_cache_build that runs under the previous kernels' last CTAs, because the maps
// are the call's inputs, complete before the chain's first kernel passed its own wait.  blk_cnt and every write come after it.
__device__ __forceinline__ void frame_block_build(const FrameGeom& g, const float* __restrict__ depth, const float4* __restrict__ normal, float dmin, float dmax, int b,
                                                  const int* __restrict__ blk_cnt, float4* texel, float4* src, int* nsrc) {
	__shared__ int s_w[32];
	__shared__ int s_base;
	const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
	const int npix = g.w * g.h;
	const int idx = b * 1024 + tid;
	float4 rec, cp, nr;
	if (idx < npix) rec = texel_build(g.tg, g.W, g.H, g.w, depth, normal, idx, cp, nr);
	chain_wait();
	if (b * 1024 >= npix) return;
	if (wid == 0) {      // offset of this block = valid pixels of the blocks before it (at most a few dozen)
		int t = 0;
		for (int q = lane; q < b; q += 32) t += blk_cnt[q];
#pragma unroll
		for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
		if (lane == 0) s_base = t;
	}
	bool valid = false;
	if (idx < npix) {
		texel[idx] = rec;
		valid = (cp.z > dmin && cp.z < dmax);
	}
	const unsigned bal = __ballot_sync(0xffffffffu, valid);
	if (lane == 0) s_w[wid] = __popc(bal);
	__syncthreads();
	int off = (lane < wid) ? s_w[lane] : 0;       // exclusive prefix over the warps of this block
#pragma unroll
	for (int o = 16; o > 0; o >>= 1) off += __shfl_xor_sync(0xffffffffu, off, o);
	if (valid) {
		const int o = s_base + off + __popc(bal & ((1u << lane) - 1u));
		src[2 * o] = make_float4(cp.x, cp.y, cp.z, nr.x);
		src[2 * o + 1] = make_float4(nr.y, nr.z, nr.w, 0.f);
	}
	if ((b + 1) * 1024 >= npix && tid == 1023) *nsrc = s_base + off + __popc(bal);     // last block of the frame, last warp: the total
}

// one 32-byte source record through the read-only path: two 128-bit loads (the widest global load sm_90 has)
struct __align__(32) F8 { float4 lo, hi; };
__device__ __forceinline__ F8 ldg256(const float4* p) {
	F8 r;
	r.lo = __ldg(p);
	r.hi = __ldg(p + 1);
	return r;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
	for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
	return v;
}
__device__ __forceinline__ int ld_acquire(const int* p) {
	int v;
	asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
	return v;
}
// Polling load for the iteration flags: relaxed, i.e. WITHOUT the L1 invalidation (CCTL.IVALL) every ld.acquire.gpu carries - a CTA
// spinning on an acquire load flushed its SM's L1 five million times per launch (ncu), under the feet of the co-resident CTA's
// texel taps.  The waiter confirms with ONE acquire load once the relaxed load has seen the value.
__device__ __forceinline__ int ld_relaxed(const int* p) {
	int v;
	asm volatile("ld.relaxed.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
	return v;
}
// ticket with release (orders this thread's - and, through the preceding __syncwarp / barrier, its warp's / CTA's - earlier writes
// before it) and acquire (the CTA that draws the last ticket sees every other tile's writes) semantics in ONE instruction; a full
// __threadfence() by every writer lane in front of a relaxed atomic costs far more per tile
__device__ __forceinline__ int ticket_acq_rel(int* p) {
	int old;
	asm volatile("atom.add.acq_rel.gpu.global.s32 %0, [%1], 1;" : "=r"(old) : "l"(p) : "memory");
	return old;
}
// asynchronous global -> shared copy of one 48-byte tile record (no registers held while it is in flight)
__device__ __forceinline__ void tile_fetch_async(void* smem_dst, const void* gsrc) {
	const unsigned d = (unsigned)__cvta_generic_to_shared(smem_dst);
	asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n cp.async.cg.shared.global [%2], [%3], 16;\n cp.async.cg.shared.global [%4], [%5], 16;"
	             ::"r"(d), "l"(gsrc), "r"(d + 16), "l"((const char*)gsrc + 16), "r"(d + 32), "l"((const char*)gsrc + 32) : "memory");
}
__device__ __forceinline__ void cp_async4(void* smem_dst, const void* gsrc) {      // 4-byte asynchronous copy (through L1: immutable tables only)
	asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"((unsigned)__cvta_generic_to_shared(smem_dst)), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async16_cg(void* smem_dst, const void* gsrc) {  // 16-byte asynchronous copy from L2 (data other CTAs wrote during this launch)
	asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((unsigned)__cvta_generic_to_shared(smem_dst)), "l"(gsrc) : "memory");
}
// 16-byte shared-memory load the compiler keeps where it is written: the pixel loop re-reads its per-tile constants (transform,
// geometry) at every use instead of holding 24 registers across the loop
__device__ __forceinline__ float4 lds128(const float* p) {
	float4 v;
	asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"((unsigned)__cvta_generic_to_shared(p)));
	return v;
}
__device__ __forceinline__ void tile_fetch_wait() { asm volatile("cp.async.wait_all;" ::: "memory"); }
__device__ __forceinline__ void st_release(int* p, int v) {
	asm volatile("st.release.gpu.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// Optional in-kernel phase profile (developer aid): thread 0 stamps clock64() at phase boundaries.
struct ProfRec { long long kind_cta, tile_win, t[10]; };
__device__ __forceinline__ void prof_emit(const SolveArgs& a, const ProfRec& r) {
	const unsigned long long k = atomicAdd((unsigned long long*)a.prof, 1ull);
	if ((int)k < a.prof_cap) {
		long long* o = a.prof + 1 + k * 12;
		o[0] = r.kind_cta; o[1] = r.tile_win;
		for (int i = 0; i < 10; i++) o[2 + i] = r.t[i];
	}
}
#ifdef BT_PROF_GLOBALTIMER      // (variant build: nanoseconds of the device-wide timer, comparable across SMs, instead of the SM's own cycle counter)
__device__ __forceinline__ long long prof_now() { return global_ns(); }
#else
__device__ __forceinline__ long long prof_now() { return clock64(); }
#endif
#define PROF_T(i) do { if (a.prof && threadIdx.x == 0) prf.t[i] = prof_now(); } while (0)

// ------------------------------------------------------------------------------------------------ k_prep_frames
// CUDACache::storeFrame fused (convertDepthFloatToCameraSpaceFloat4 + 2x resampleFloat4 nearest, CUDAImageUtil.cu:
// 310-326,82-99) + compaction of the source list + matrixToPose/poseToMatrix of the incoming pose (SBA.cu:71-79).
__device__ void plan_body(const SolveArgs& a, WinDesc* wins_rw);

// One CTA per frame.  The compacted source list keeps pixel order (fixed summation order downstream), so the CTA needs
// an ordered prefix over its pixels; instead of one block-wide scan per 1024 pixels (19 x 3 barriers per frame, the loads
// of each round exposed) it runs two sweeps around ONE scan: sweep 1 counts the valid pixels of every (round, warp) from
// the depth map alone, the scan turns the counts into offsets, sweep 2 loads depth + normal, writes the texel map and the
// source records at their final position.  No barrier inside either sweep, so the loads of consecutive rounds overlap.
static constexpr int kPrepRounds = 64;      // rounds of 1024 pixels per scan (one scan covers 65536 quarter-res pixels)

// Builds one frame's quarter-resolution texel map and compacted source list (1024 threads); returns the source count.
__device__ int build_frame_maps(const FrameGeom& g, const float* __restrict__ depth, const float4* __restrict__ normal, float4* texel, float4* src,
                                float dmin, float dmax, int* s_cnt, int* s_wt) {
	const int npix = g.w * g.h;
	const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
	int base = 0;
	for (int sb = 0; sb < npix; sb += kPrepRounds * 1024) {
		const int rounds = min(kPrepRounds, (npix - sb + 1023) >> 10);
		// ---- sweep 1: valid counts per (round, warp)
#pragma unroll 4
		for (int r = 0; r < rounds; r++) {
			const int idx = sb + (r << 10) + tid;
			bool valid = false;
			if (idx < npix) {
				const float z = texel_depth(g.tg, g.W, g.H, g.w, depth, idx);
				valid = (z > dmin && z < dmax);
			}
			const unsigned bal = __ballot_sync(0xffffffffu, valid);
			if (lane == 0) s_cnt[r * 32 + wid] = __popc(bal);
		}
		__syncthreads();
		// ---- exclusive scan of the rounds*32 counts in (round, warp) order: two entries per thread
		const int n = rounds * 32;
		const int v0 = (2 * tid < n) ? s_cnt[2 * tid] : 0, v1 = (2 * tid + 1 < n) ? s_cnt[2 * tid + 1] : 0;
		int total;
		const int excl = base + block_excl_scan(v0 + v1, s_wt, &total);
		if (2 * tid < n) s_cnt[2 * tid] = excl;
		if (2 * tid + 1 < n) s_cnt[2 * tid + 1] = excl + v0;
		base += total;
		__syncthreads();
		// ---- sweep 2: texel map + source records at their final offsets
#pragma unroll 2
		for (int r = 0; r < rounds; r++) {
			const int idx = sb + (r << 10) + tid;
			float4 cp, nr;
			bool valid = false;
			if (idx < npix) {
				texel[idx] = texel_build(g.tg, g.W, g.H, g.w, depth, normal, idx, cp, nr);
				valid = (cp.z > dmin && cp.z < dmax);
			}
			const unsigned bal = __ballot_sync(0xffffffffu, valid);
			if (valid) {
				const int o = s_cnt[r * 32 + wid] + __popc(bal & ((1u << lane) - 1u));
				src[2 * o] = make_float4(cp.x, cp.y, cp.z, nr.x);
				src[2 * o + 1] = make_float4(nr.y, nr.z, nr.w, 0.f);
			}
		}
		__syncthreads();
	}
	return base;
}

// Frame preparation of the frames a call rebuilds itself, one CTA per 1024 quarter-res pixels of a (window, frame) slot:
// frame_block_count, then frame_block_build.  (One CTA per frame would walk 19 rounds serially.)
// Every CTA of a chained kernel passes chain_wait() before it exits, so that the grid's completion orders everything after it behind
// the predecessor.
__global__ void __launch_bounds__(1024, 2) k_prep_count(SolveArgs a, int* __restrict__ blk_cnt) {
	const int fs = blockIdx.y, b = blockIdx.x;
	chain_wait();
	chain_release();
	if (a.tstamp && fs == 0 && b == 0 && threadIdx.x == 0) a.tstamp[0] = global_ns();
	if (a.nsrc_cached[fs] || !(a.prm.w_dense > 0.0f)) return;
	const WinDesc wd = a.wins[a.frame_win[fs]];
	const FrameGeom g = {wd.W, wd.H, wd.w, wd.h, wd.tg};
	frame_block_count(g, a.depth_ptr[fs], a.prm.depth_min, a.prm.depth_max, b, blk_cnt + fs * gridDim.x);
}

__global__ void __launch_bounds__(1024, 2) k_prep_frames(SolveArgs a, WinDesc* wins_rw, int* prep_ticket, const int* __restrict__ blk_cnt) {
	const int fs = blockIdx.y, b = blockIdx.x;
	const int tid = threadIdx.x;
	chain_wait();
	chain_release();
	if (a.tstamp && !a.with_count && fs == 0 && b == 0 && tid == 0) a.tstamp[0] = global_ns();
	const WinDesc wd = a.wins[a.frame_win[fs]];
	const int* cached = a.nsrc_cached[fs];
	if (cached) { if (b == 0 && tid == 0) a.nsrc[fs] = *cached; }      // maps and source list were built by bt_frame_cache_store
	else if (!(a.prm.w_dense > 0.0f)) { if (b == 0 && tid == 0) a.nsrc[fs] = 0; }
	else {
		const FrameGeom g = {wd.W, wd.H, wd.w, wd.h, wd.tg};
		frame_block_build(g, a.depth_ptr[fs], a.normal_ptr[fs], a.prm.depth_min, a.prm.depth_max, b, blk_cnt + fs * gridDim.x,
		                  a.texel + (size_t)fs * a.npix_max, a.src + (size_t)fs * 2 * a.npix_max, a.nsrc + fs);
	}
	if (b == 0 && tid == 1023) {      // pose -> (rot, trans) -> T of iteration 0 (one lane of the frame's first block)
		float Tm[12];
		const float* P = a.pose_in + (size_t)fs * 16;
		for (int k = 0; k < 12; k++) Tm[k] = P[k];
		V3 rot, trans;
		se3_log(Tm, rot, trans);
		float* x = a.x + (size_t)fs * 6;
		x[0] = rot.x; x[1] = rot.y; x[2] = rot.z; x[3] = trans.x; x[4] = trans.y; x[5] = trans.z;
		se3_exp(rot, trans, Tm);
		float* T = a.T + (size_t)fs * 12;
		for (int k = 0; k < 12; k++) T[k] = Tm[k];
	}
	// the last CTA to finish plans the dense tiles of the whole batch (saves a launch and its dependency gap)
	__shared__ int s_last;
	__threadfence();
	__syncthreads();
	if (tid == 0) { const int t = atomicAdd(prep_ticket, 1); s_last = (t == (int)(gridDim.x * gridDim.y) - 1); if (s_last) { *prep_ticket = 0; __threadfence(); } }
	__syncthreads();
	if (s_last) {
		plan_body(a, wins_rw);
		if (a.tstamp && tid == 0) { a.tstamp[1] = global_ns(); a.tstamp[3] = 0; }      // ([3]: k_solve's CTAs take the maximum of their end times)
	}
}

// bt_frame_cache_store: the same maps, built once per keyframe into a slot of the context's frame cache.
// A store of up to kStoreInline frames carries its map pointers and slots in the kernel parameters (no table upload between the
// previous kernel and the store's, which would cut the launch chain); a larger one reads them from the uploaded tables.
static constexpr int kStoreInline = 64;
struct CacheStoreArgs {
	FrameGeom g;
	const float* const* depth; const float4* const* normal; const int* slots;   // the uploaded tables, or nullptr: the arrays below
	float4* texel; float4* src; int* nsrc; size_t slot_npix;   // quarter-res pixels per slot: texel map slot_npix float4, source list 2 * slot_npix
	float dmin, dmax;
	const float* depth_in[kStoreInline]; const float4* normal_in[kStoreInline]; int slot_in[kStoreInline];
};
__device__ __forceinline__ const float* store_depth(const CacheStoreArgs& c, int f) { return c.depth ? c.depth[f] : c.depth_in[f]; }
__device__ __forceinline__ const float4* store_normal(const CacheStoreArgs& c, int f) { return c.normal ? c.normal[f] : c.normal_in[f]; }
__device__ __forceinline__ int store_slot(const CacheStoreArgs& c, int f) { return c.slots ? c.slots[f] : c.slot_in[f]; }
__global__ void __launch_bounds__(1024, 2) k_frame_cache_store(const __grid_constant__ CacheStoreArgs c) {
	__shared__ int s_cnt[kPrepRounds * 32];
	__shared__ int s_wt[32];
	const int slot = store_slot(c, blockIdx.x);
	const int n = build_frame_maps(c.g, store_depth(c, blockIdx.x), store_normal(c, blockIdx.x), c.texel + (size_t)slot * c.slot_npix, c.src + (size_t)slot * 2 * c.slot_npix,
	                               c.dmin, c.dmax, s_cnt, s_wt);
	if (threadIdx.x == 0) c.nsrc[slot] = n;
}

// The same store spread over one CTA per 1024 quarter-res pixels (count + build, like k_prep_count / k_prep_frames): a handful of new
// frames per step - one per tracked window - otherwise runs on a handful of CTAs walking 19 rounds each.
// k_cache_count reads nothing before its wait (the caller's maps may come from the kernel right before the store) and releases
// k_cache_build only after it: k_cache_build then loads its samples while the last count CTAs finish.  k_cache_build's writes wait for
// k_cache_count's completion, which follows the previous kernel's - in a tracking step, the k_solve that read the slot being rewritten.
__global__ void __launch_bounds__(1024, 2) k_cache_count(const __grid_constant__ CacheStoreArgs c, int* __restrict__ blk_cnt) {
	const int f = blockIdx.y;
	chain_wait();
	chain_release();
	frame_block_count(c.g, store_depth(c, f), c.dmin, c.dmax, blockIdx.x, blk_cnt + f * gridDim.x);
}
__global__ void __launch_bounds__(1024, 2) k_cache_build(const __grid_constant__ CacheStoreArgs c, const int* __restrict__ blk_cnt) {
	const int f = blockIdx.y, slot = store_slot(c, f);
	chain_release();      // (the successor waits before it reads anything)
	frame_block_build(c.g, store_depth(c, f), store_normal(c, f), c.dmin, c.dmax, blockIdx.x, blk_cnt + f * gridDim.x,
	                  c.texel + (size_t)slot * c.slot_npix, c.src + (size_t)slot * 2 * c.slot_npix, c.nsrc + slot);
}

// ------------------------------------------------------------------------------------------------ tile plan
__device__ __forceinline__ int chunks_for(int n, int chunk, int& per) {
	if (n <= 0) { per = 0; return 0; }
	const int nch = (n + chunk - 1) / chunk;
	per = (((n + nch - 1) / nch) + 31) & ~31;   // balanced, warp-aligned
	return (n + per - 1) / per;
}
// Runs on the LAST CTA of k_prep_frames to finish (1024 threads): per-window tile counts -> scans -> flat tile list.
__device__ void plan_body(const SolveArgs& a, WinDesc* wins_rw) {
	__shared__ int s_cnt[1024];
	__shared__ int s_wtot[32];
	__shared__ int s_carry;
	__shared__ unsigned long long s_px;
	const int tid = threadIdx.x;
	ProfRec prf; prf.kind_cta = (3ll << 32) | blockIdx.x; prf.tile_win = a.n_windows;
	for (int i = 0; i < 10; i++) prf.t[i] = 0;
	PROF_T(0);
	if (tid == 0) { s_carry = 0; s_px = 0ull; *a.queue = 0; }
	__syncthreads();
	// Small batches: when one GN iteration has only slightly more tiles than k_solve has CTAs, the few CTAs that get two tiles
	// put a whole extra tile on the critical path of every iteration.  Grow the chunk until an iteration fits one wave.
	int chunk = a.chunk;
	if (a.n_windows <= 1024) {
		__shared__ int s_total;
		const WinDesc wl0 = a.wins[a.n_windows - 1];
		const int n_pairs_all = wl0.pair_off + wl0.n_pairs;
		// (a lone window's plan is on its critical path: the pairs' source counts - two dependent global loads - are read once, not per attempt)
		const bool one_each = n_pairs_all <= 1024;
		const int n_mine = (one_each && tid < n_pairs_all) ? a.nsrc[a.pair_src_slot[tid]] : 0;
		for (int attempt = 0; attempt < 4; attempt++) {
			if (tid == 0) s_total = 0;
			__syncthreads();
			int mine = 0;
			if (one_each) { int per; mine = chunks_for(n_mine, chunk, per); }
			else for (int q = tid; q < n_pairs_all; q += 1024) { int per; mine += chunks_for(a.nsrc[a.pair_src_slot[q]], chunk, per); }
#pragma unroll
			for (int o = 16; o > 0; o >>= 1) mine += __shfl_xor_sync(0xffffffffu, mine, o);
			if ((tid & 31) == 0 && mine) atomicAdd(&s_total, mine);
			__syncthreads();
			const int total = s_total + kSparseTiles * a.n_windows;      // + the sparse tiles of every window
			__syncthreads();
			if (total <= a.grid_ctas || total > 2 * a.grid_ctas) break;
			chunk = (int)(((long long)chunk * total / a.grid_ctas + 63) / 32 * 32);     // ~(total/grid) x larger, rounded up to warps
		}
	}
	for (int base = 0; base < a.n_windows; base += 1024) {
		const int nw = min(1024, a.n_windows - base);
		s_cnt[tid] = 0;
		__syncthreads();
		// (1) chunk count of every (window, pair) of this block of windows, in parallel
		const int first_pair = a.wins[base].pair_off;
		const WinDesc wl = a.wins[base + nw - 1];
		const int end_pair = wl.pair_off + wl.n_pairs;
		unsigned long long px = 0;
		for (int q = first_pair + tid; q < end_pair; q += 1024) {
			const int lo = a.pair_win[q];
			const int n = a.nsrc[a.pair_src_slot[q]];
			int per;
			const int nch = chunks_for(n, chunk, per);
			a.pair_ntile[q] = nch;
			atomicAdd(&s_cnt[lo - base], nch);
			px += (unsigned long long)n;
		}
		// one 64-bit shared atomic per warp, not per thread: 1024 threads hammering one 64-bit shared word serialise (a CAS loop in hardware)
#pragma unroll
		for (int o = 16; o > 0; o >>= 1) px += __shfl_xor_sync(0xffffffffu, px, o);
		if ((tid & 31) == 0 && px) atomicAdd(&s_px, px);
		__syncthreads();
		PROF_T(1);
		// (2) exclusive scan of the per-window tile counts: the dense tiles plus ONE sparse tile (the window's moment sums), first in line
		int cnt = 0;
		if (tid < nw) { cnt = s_cnt[tid] + kSparseTiles; a.tiles_done[base + tid] = 0; a.iter_done[base + tid] = 0; }
		int n_tiles;      // the tiles of this block of windows
		const int excl = s_carry + block_excl_scan(cnt, s_wtot, &n_tiles);
		PROF_T(2);
		const bool fits = (s_carry + n_tiles <= a.max_tiles);
		// (3) per-window prefix over its pairs: one warp per window, lanes over pairs
		if (tid < nw) {
			wins_rw[base + tid].tile_off = excl;
			wins_rw[base + tid].n_tiles = cnt;
			s_cnt[tid] = excl;      // reuse: window -> tile_off for step (4)
		}
		__syncthreads();
		if (tid == 0) s_carry += n_tiles;      // (every thread has read s_carry)
		for (int wl = (tid >> 5); wl < nw; wl += 32) {
			const int w = base + wl, lane = tid & 31;
			const int poff = a.wins[w].pair_off, np = a.wins[w].n_pairs;
			int carry = 0;
			for (int p0 = 0; p0 < np; p0 += 32) {
				const int p = p0 + lane;
				const int v = (p < np) ? a.pair_ntile[poff + p] : 0;
				const int incl = warp_incl_scan(v);
				if (p < np) a.pair_tile0[poff + p] = kSparseTiles + carry + incl - v;      // the first slots of the window are its sparse tiles
				carry += __shfl_sync(0xffffffffu, incl, 31);
			}
			if (lane < kSparseTiles && fits) {      // start / count of a sparse tile = its share: part `start` of `count`
				Tile tl; tl.win = w; tl.pair = -2; tl.start = lane; tl.count = kSparseTiles; tl.tgt_slot = tl.src_slot = 0; tl.n_tiles_win = wins_rw[w].n_tiles;
				tl.pad = 0; tl.src = tl.tex = nullptr; a.tiles[s_cnt[wl] + lane] = tl;
			}
		}
		__syncthreads();
		PROF_T(3);
		// (4) tile records, one (window, pair) per thread
		if (fits) {
			for (int q = first_pair + tid; q < end_pair; q += 1024) {
				const int lo = a.pair_win[q];
				const int n = a.nsrc[a.pair_src_slot[q]];
				const int pair_off_w = a.wins[lo].pair_off;
				int per;
				const int nch = chunks_for(n, chunk, per);
				int t = s_cnt[lo - base] + a.pair_tile0[q];
				Tile tl; tl.win = lo; tl.pair = q - pair_off_w; tl.pad = 0;
				tl.src_slot = a.pair_src_slot[q]; tl.tgt_slot = a.wins[lo].frame_off + (int)a.pairs[q].x;
				tl.n_tiles_win = wins_rw[lo].n_tiles;
				tl.src = a.src_tab[tl.src_slot]; tl.tex = a.texel_tab[tl.tgt_slot];
				for (int c = 0; c < nch; c++) { tl.start = c * per; tl.count = min(per, n - c * per); a.tiles[t++] = tl; }
			}
		}
		__syncthreads();
		PROF_T(4);
	}
	if (tid == 0) {
		*a.n_tiles_total = (s_carry <= a.max_tiles && (long long)s_carry * a.prm.num_iter_outer < 0x7fffff00ll) ? s_carry : -1;   // -1 => capacity error reported by the host
		*a.n_src_px = (long long)s_px;
	}
	PROF_T(5);
	if (a.prof && tid == 0) prof_emit(a, prf);
}

// ------------------------------------------------------------------------------------------------ tile (dense term)
// Evaluate one chunk of compacted source pixels of pair (tgt i, src j).  Accumulates, in the TARGET camera frame,
// S' = sum w g' g'^T (upper triangle, 21) and b' = sum w g' r (6) with g' = (n_tgt, p' x n_tgt); the tail maps them to
// the model frame with the 6x6 adjoint of T_i.
struct TileAcc { float v[kTileVals]; };

// One pixel between the issue of its loads and its evaluation: the source point mapped into the target camera, the source normal,
// the projection and the four bilinear taps of the texel map (zeros for a tap outside the map).  in = the pixel projects into the map.
struct PixTaps { float tx, ty, tz, nx, ny, nz, sx, sy; float4 t00, t01, t10, t11; bool in; };

// Software-pipelined over a thread's pixels (stride NT): iteration k issues the projection and taps of pixel k and the source load
// of pixel k + 2 NT, then evaluates pixel k.
// sM: the transform (3 rows of 4); sG: {fx, fy, cx, cy}, {ifx, ify, icx, icy}, {scaleW, scaleH, w, h (int bits)} of the window.
template <int NT> __device__ __forceinline__ void tile_pixels(const SolveArgs& a, const float4* __restrict__ src, const float4* __restrict__ tex,
                                            const float* sM, const float* sG, int start, int count, TileAcc& acc) {
	const float dmin = a.prm.depth_min, dmax = a.prm.depth_max, cos_t = a.prm.dense_cos_normal_thresh;
	const float delta = a.prm.robust_delta, wdense = a.prm.w_dense;
	// `sqrtf(d2) <= dist_t` evaluated as `d2 <= d2max`, d2max = the largest float whose correctly rounded square root is <= dist_t
	// (same truth value for every float, no square root in the loop; found once on the host, make_args)
	const float d2max = a.d2max;
	auto issue = [&](const F8& s, PixTaps& q) {
		const float4 M0 = lds128(sM), M1 = lds128(sM + 4), M2 = lds128(sM + 8), K = lds128(sG), Z = lds128(sG + 8);
		const float m00 = M0.x, m01 = M0.y, m02 = M0.z, m03 = M0.w, m10 = M1.x, m11 = M1.y, m12 = M1.z, m13 = M1.w, m20 = M2.x, m21 = M2.y, m22 = M2.z, m23 = M2.w;
		const float fx = K.x, fy = K.y, cx = K.z, cy = K.w;
		const unsigned W = __float_as_uint(Z.z), Hh = __float_as_uint(Z.w);
		const float px = s.lo.x, py = s.lo.y, pz = s.lo.z;
		q.nx = s.lo.w; q.ny = s.hi.x; q.nz = s.hi.y;
		// camPosSrcToTgt = transform * camPosSrc
		q.tx = m00 * px + m01 * py + m02 * pz + m03;
		q.ty = m10 * px + m11 * py + m12 * pz + m13;
		q.tz = m20 * px + m21 * py + m22 * pz + m23;
		// cameraToDepth, CUDACameraUtil.h:9-14.  One reciprocal serves both quotients (the reference itself is built with
		// -use_fast_math: its divisions are rcp.approx too; either way the result differs from the exact quotient by an ulp or two)
		const float itz = rcp_fast(q.tz);
		q.sx = (q.tx * fx) * itz + cx; q.sy = (q.ty * fy) * itz + cy;
		const int ix = (int)roundf(q.sx), iy = (int)roundf(q.sy);
		q.in = ix >= 0 && iy >= 0 && ix < (int)W && iy < (int)Hh;
		q.t00 = q.t01 = q.t10 = q.t11 = make_float4(0.f, 0.f, 0.f, 0.f);
		if (q.in) {
			const int x0 = (int)floorf(q.sx), y0 = (int)floorf(q.sy);
			const bool inx0 = (unsigned)x0 < W, inx1 = (unsigned)(x0 + 1) < W;
			if ((unsigned)y0 < Hh) { const float4* row = tex + (size_t)y0 * W; if (inx0) q.t00 = __ldg(row + x0); if (inx1) q.t01 = __ldg(row + x0 + 1); }
			if ((unsigned)(y0 + 1) < Hh) { const float4* row = tex + (size_t)(y0 + 1) * W; if (inx0) q.t10 = __ldg(row + x0); if (inx1) q.t11 = __ldg(row + x0 + 1); }
		}
	};
	auto evaluate = [&](const PixTaps& q) {
		if (!q.in) return;
		const float4 I = lds128(sG + 4), Z = lds128(sG + 8);
		TexelGeom tg; tg.ifx = I.x; tg.ify = I.y; tg.icx = I.z; tg.icy = I.w; tg.scaleW = Z.x; tg.scaleH = Z.y;
		const unsigned W = __float_as_uint(Z.z), Hh = __float_as_uint(Z.w);
		const float tx = q.tx, ty = q.ty, tz = q.tz;
		// bilinearInterpolationFloat4 on camera-space points AND normals (same taps, same weights); the tap's point is rebuilt from its
		// depth at the tap's full-res sample position
		const float fx0 = floorf(q.sx), fy0 = floorf(q.sy);
		const int x0 = (int)fx0, y0 = (int)fy0;
		const float al = q.sx - fx0, be = q.sy - fy0;
		const unsigned xs0 = texel_sample(x0, tg.scaleW), xs1 = texel_sample(x0 + 1, tg.scaleW);
		const unsigned ys0 = texel_sample(y0, tg.scaleH), ys1 = texel_sample(y0 + 1, tg.scaleH);
		float a0[3] = { 0.f, 0.f, 0.f }, b0[3] = { 0.f, 0.f, 0.f }, a1[3] = { 0.f, 0.f, 0.f }, b1[3] = { 0.f, 0.f, 0.f };
		float w0 = 0.f, w1 = 0.f;
		auto tap = [&](const float4& t, unsigned xs, unsigned ys, float wt, float* ac, float* bc, float& wsum) {
			ac[0] += wt * texel_coord(xs, t.x, tg.ifx, tg.icx); ac[1] += wt * texel_coord(ys, t.x, tg.ify, tg.icy); ac[2] += wt * t.x;
			bc[0] += wt * t.y; bc[1] += wt * t.z; bc[2] += wt * t.w; wsum += wt;
		};
		const bool inx0 = (unsigned)x0 < W, inx1 = (unsigned)(x0 + 1) < W, iny0 = (unsigned)y0 < Hh, iny1 = (unsigned)(y0 + 1) < Hh;
		if (iny0) {
			if (inx0) tap(q.t00, xs0, ys0, 1.0f - al, a0, b0, w0);
			if (inx1) tap(q.t01, xs1, ys0, al, a0, b0, w0);
		}
		if (iny1) {
			if (inx0) tap(q.t10, xs0, ys1, 1.0f - al, a1, b1, w1);
			if (inx1) tap(q.t11, xs1, ys1, al, a1, b1, w1);
		}
		float ww = 0.f, cxs = 0.f, cys = 0.f, czs = 0.f, nxs = 0.f, nys = 0.f, nzs = 0.f;
		if (w0 > 0.f) { const float r = (1.0f - be) * rcp_fast(w0); cxs += r * a0[0]; cys += r * a0[1]; czs += r * a0[2]; nxs += r * b0[0]; nys += r * b0[1]; nzs += r * b0[2]; ww += (1.0f - be); }
		if (w1 > 0.f) { const float r = be * rcp_fast(w1); cxs += r * a1[0]; cys += r * a1[1]; czs += r * a1[2]; nxs += r * b1[0]; nys += r * b1[1]; nzs += r * b1[2]; ww += be; }
		if (!(ww > 0.f)) return;
		const float rw = rcp_fast(ww);
		const float qx = cxs * rw, qy = cys * rw, qz = czs * rw;        // camPosTgt
		if (!(qz > dmin && qz < dmax)) return;
		const float tnx = nxs * rw, tny = nys * rw, tnz = nzs * rw;     // normalTgt
		// nrmj = transform(3x3) * n  (w of the normal is 0)
		const float4 M0 = lds128(sM), M1 = lds128(sM + 4), M2 = lds128(sM + 8);
		const float m00 = M0.x, m01 = M0.y, m02 = M0.z, m10 = M1.x, m11 = M1.y, m12 = M1.z, m20 = M2.x, m21 = M2.y, m22 = M2.z;
		const float rnx = m00 * q.nx + m01 * q.ny + m02 * q.nz;
		const float rny = m10 * q.nx + m11 * q.ny + m12 * q.nz;
		const float rnz = m20 * q.nx + m21 * q.ny + m22 * q.nz;
		const float dx = tx - qx, dy = ty - qy, dz = tz - qz;
		const float dist2 = dx * dx + dy * dy + dz * dz;
		const float dn = rnx * tnx + rny * tny + rnz * tnz;
		if (!(dn >= cos_t && dist2 <= d2max)) return;
		const float res = -(dx * tnx + dy * tny + dz * tnz);            // dot(camPosTgt - camPosSrcToTgt, normalTgt)
		const float wgt = wdense * huber_w_fast(res * res, delta);
		float g[6];
		g[0] = tnx; g[1] = tny; g[2] = tnz;
		g[3] = ty * tnz - tz * tny; g[4] = tz * tnx - tx * tnz; g[5] = tx * tny - ty * tnx;   // p' x n_tgt
		int e = 0;
#pragma unroll
		for (int r = 0; r < 6; r++) {
			const float wg = wgt * g[r];
#pragma unroll
			for (int c = r; c < 6; c++) acc.v[e++] += wg * g[c];
		}
#pragma unroll
		for (int r = 0; r < 6; r++) acc.v[21 + r] += wgt * g[r] * res;
		acc.v[27] += 1.0f;
	};
	const float4* sp = src + 2 * (size_t)start;
	int k = threadIdx.x;
	F8 c0, c1;      // source records of pixels k and k + NT
	c0.lo = c0.hi = c1.lo = c1.hi = make_float4(0.f, 0.f, 0.f, 0.f);
	if (k < count) c0 = ldg256(sp + 2 * k);
	if (k + NT < count) c1 = ldg256(sp + 2 * (k + NT));
	for (; k < count; k += NT) {
		PixTaps q;
		issue(c0, q);
		c0 = c1;
		if (k + 2 * NT < count) c1 = ldg256(sp + 2 * (k + 2 * NT));
		evaluate(q);
	}
}

// ------------------------------------------------------------------------------------------------ tail (per window, per GN iteration)
__constant__ unsigned char c_sym_r[21] = { 0,0,0,0,0,0, 1,1,1,1,1, 2,2,2,2, 3,3,3, 4,4, 5 };
__constant__ unsigned char c_sym_c[21] = { 0,1,2,3,4,5, 1,2,3,4,5, 2,3,4,5, 3,4,5, 4,5, 5 };
__constant__ unsigned char c_sym_idx[36] = { 0,1,2,3,4,5, 1,6,7,8,9,10, 2,7,11,12,13,14, 3,8,12,15,16,17, 4,9,13,16,18,19, 5,10,14,17,19,20 };

struct TailSmem {
	float* T;      // [N][12]
	float* A;      // [dimp][ld]
	float* rhs; float* Minv; float* r; float* z; float* p; float* Ap; float* delta;   // [dimp] each
	float* pairW;    // [P][28] per-pair sums over the pair's tiles (model frame; 27 used + count)
	float* grp;      // [G][44]
	float* fS;       // [N][20] per-frame sparse sums: n, S(3), Q(6), grad rot(3), grad trans(3), Pw(3), Pn
	float* fD;       // [N][28] per-frame dense sums: S(21) + signed b(6)
	int* gi; int* gj; int* gstart;     // [G], [G], [G+1]
	int* pt; int* ps; int* pt0; int* pnt;   // [P] each: pair target, source, first tile, #tiles
	int* fg_start; int* fp_start; int* fg_items; int* fp_items;   // per-frame membership CSR ([N+1], [N+1], [2G], [2P])
	int dimp, ld;
};
static constexpr int kFS = 20, kFD = 28;
// (grp_in_smem = false: big windows - 30 frames, 435 groups - leave the 44 moment sums per group in global memory and read them
// through L2; with them the tail of such a window would need 279 KB of shared memory)
// Leading dimension of the system matrix: the PCG reads a whole row per THREAD with 16-byte loads, which is conflict-free when the rows
// of eight consecutive threads start in eight different 4-bank groups: ld = 4 (mod 8), ld >= dimp rounded up to a multiple of 4.
__host__ __device__ inline int tail_ld(int dimp) { int ld = (dimp + 3) & ~3; if ((ld & 7) != 4) ld += 4; return ld; }
__host__ __device__ inline size_t tail_smem_floats(int N, int P, int G, bool grp_in_smem = true) {
	const int dimp = 6 * (N - 1), ld = tail_ld(dimp), dimp4 = (dimp + 3) & ~3;
	return (size_t)N * 12 + (size_t)dimp * ld + 7 * (size_t)dimp4 + (size_t)P * kTileVals + (grp_in_smem ? (size_t)G * kGrpVals : 0) +
	       (size_t)N * (kFS + kFD) + (size_t)(3 * G + 1 + 4 * P) + (size_t)(2 * (N + 1) + 2 * G + 2 * P) + 16;
}
__device__ inline void tail_carve(float* base, int N, int P, int G, TailSmem& s, bool grp_in_smem) {
	s.dimp = 6 * (N - 1); s.ld = tail_ld(s.dimp);
	const int dimp4 = (s.dimp + 3) & ~3;      // every vector starts 16-byte aligned (N * 12 and dimp * ld are multiples of 4 floats)
	float* q = base;
	s.T = q; q += N * 12;
	s.A = q; q += s.dimp * s.ld;
	s.rhs = q; q += dimp4; s.Minv = q; q += dimp4; s.r = q; q += dimp4; s.z = q; q += dimp4;
	s.p = q; q += dimp4; s.Ap = q; q += dimp4; s.delta = q; q += dimp4;
	s.pairW = q; q += P * kTileVals;
	s.grp = q; if (grp_in_smem) q += G * kGrpVals;
	s.fS = q; q += N * kFS; s.fD = q; q += N * kFD;
	int* iq = reinterpret_cast<int*>(q);
	s.gi = iq; iq += G; s.gj = iq; iq += G; s.gstart = iq; iq += G + 1;
	s.pt = iq; iq += P; s.ps = iq; iq += P; s.pt0 = iq; iq += P; s.pnt = iq; iq += P;
	s.fg_start = iq; iq += N + 1; s.fp_start = iq; iq += N + 1; s.fg_items = iq; iq += 2 * G; s.fp_items = iq; iq += 2 * P;
}
// index of (r,c), r<=c, in the packed upper triangle of a symmetric 6x6
__device__ __forceinline__ int sym6(int r, int c) { if (r > c) { const int t = r; r = c; c = t; } return r * 6 - (r * (r - 1)) / 2 + (c - r); }
__device__ __forceinline__ float skew(const float* v, int a, int b) {   // [v]x (a,b)
	if (a == b) return 0.f;
	const int k = 3 - a - b;                                // the remaining axis
	const float s = ((b - a + 3) % 3 == 1) ? -1.f : 1.f;    // (0,1):-vz (1,2):-vx (2,0):-vy ; transposed: +
	return s * v[k];
}
// skew() of the vector (x, y, z) without an array: an array indexed at run time would live in local memory, and the compiler may
// then keep other small arrays of the kernel there too (the pixel loop's bilinear sums)
__device__ __forceinline__ float skew3(float x, float y, float z, int a, int b) {
	if (a == b) return 0.f;
	const int k = 3 - a - b;
	const float s = ((b - a + 3) % 3 == 1) ? -1.f : 1.f;
	return s * (k == 0 ? x : (k == 1 ? y : z));
}
__device__ __forceinline__ void unpack_sym(int e, int& r, int& c) {
	r = 0;
	while (e >= 6 - r) { e -= 6 - r; r++; }
	c = r + e;
}

// Sparse moment sums of one window for the CURRENT poses: 8 lanes per (i,j) group of correspondences, loads one iteration
// ahead; 44 sums per group go to a.grp_sums.  This is the window's SPARSE tile: first in the window's slice of the queue, it runs
// on whichever CTA claims it while the dense tiles are in flight, so the window's tail does not wait for it.
template <int NT> __device__ void sparse_sums(const SolveArgs& a, int w, int part, int nparts) {
	const WinDesc wd0 = a.wins[w];
	const WinSparse ws = a.wsp[w];
	const int G = ws.n_groups, tid = threadIdx.x;
	const int sub = tid >> 3, sl = tid & 7, nsub = NT >> 3;
	const int g_lo = (int)(((long long)G * part) / nparts), g_hi = (int)(((long long)G * (part + 1)) / nparts);      // this tile's share of the groups
	for (int g0 = g_lo; g0 < g_hi; g0 += nsub) {
		const int g = g0 + sub;
		float m[kGrpVals];
#pragma unroll
		for (int k = 0; k < kGrpVals; k++) m[k] = 0.f;
		if (g < g_hi) {
			const int c0 = a.grp_start[ws.grp_off + w + g], c1 = a.grp_start[ws.grp_off + w + g + 1];
			const float* Ti = a.T + (size_t)(wd0.frame_off + a.grp_i[ws.grp_off + g]) * 12; const float* Tj = a.T + (size_t)(wd0.frame_off + a.grp_j[ws.grp_off + g]) * 12;
			const float t00 = __ldcg(Ti + 0), t01 = __ldcg(Ti + 1), t02 = __ldcg(Ti + 2), t03 = __ldcg(Ti + 3), t10 = __ldcg(Ti + 4), t11 = __ldcg(Ti + 5), t12 = __ldcg(Ti + 6), t13 = __ldcg(Ti + 7),
			            t20 = __ldcg(Ti + 8), t21 = __ldcg(Ti + 9), t22 = __ldcg(Ti + 10), t23 = __ldcg(Ti + 11);
			const float u00 = __ldcg(Tj + 0), u01 = __ldcg(Tj + 1), u02 = __ldcg(Tj + 2), u03 = __ldcg(Tj + 3), u10 = __ldcg(Tj + 4), u11 = __ldcg(Tj + 5), u12 = __ldcg(Tj + 6), u13 = __ldcg(Tj + 7),
			            u20 = __ldcg(Tj + 8), u21 = __ldcg(Tj + 9), u22 = __ldcg(Tj + 10), u23 = __ldcg(Tj + 11);
			int c = c0 + sl;
			float4 lo = make_float4(0.f, 0.f, 0.f, 0.f), hi = lo;
			if (c < c1) { const float4* e4 = reinterpret_cast<const float4*>(a.corr + ws.corr_off + c); lo = __ldg(e4); hi = __ldg(e4 + 1); }
			while (c < c1) {
				const int cn = c + 8;
				float4 lo_n = lo, hi_n = hi;
				if (cn < c1) { const float4* e4 = reinterpret_cast<const float4*>(a.corr + ws.corr_off + cn); lo_n = __ldg(e4); hi_n = __ldg(e4 + 1); }
				const float pix = lo.z, piy = lo.w, piz = hi.x, pjx = hi.y, pjy = hi.z, pjz = hi.w;   // {i, j, pi.x, pi.y}, {pi.z, pj.x, pj.y, pj.z}
				const V3 q = mk(t00 * pix + t01 * piy + t02 * piz + t03, t10 * pix + t11 * piy + t12 * piz + t13, t20 * pix + t21 * piy + t22 * piz + t23);
				const V3 sp = mk(u00 * pjx + u01 * pjy + u02 * pjz + u03, u10 * pjx + u11 * pjy + u12 * pjz + u13, u20 * pjx + u21 * pjy + u22 * pjz + u23);
				const V3 rr = q - sp;
				const float rho = huber_w(dot(rr, rr), a.prm.robust_delta);
				m[0] += 1.f;
				m[1] += q.x; m[2] += q.y; m[3] += q.z;
				m[4] += sp.x; m[5] += sp.y; m[6] += sp.z;
				m[7] += q.x * q.x; m[8] += q.x * q.y; m[9] += q.x * q.z; m[10] += q.y * q.y; m[11] += q.y * q.z; m[12] += q.z * q.z;
				m[13] += sp.x * sp.x; m[14] += sp.x * sp.y; m[15] += sp.x * sp.z; m[16] += sp.y * sp.y; m[17] += sp.y * sp.z; m[18] += sp.z * sp.z;
				m[19] += sp.x * q.x; m[20] += sp.x * q.y; m[21] += sp.x * q.z;      // Qsq[a][b] = sum s_a q_b
				m[22] += sp.y * q.x; m[23] += sp.y * q.y; m[24] += sp.y * q.z;
				m[25] += sp.z * q.x; m[26] += sp.z * q.y; m[27] += sp.z * q.z;
				const V3 gq = cross(q, rr), gs = cross(sp, rr);
				m[28] += rho * gq.x; m[29] += rho * gq.y; m[30] += rho * gq.z;
				m[31] += rho * gs.x; m[32] += rho * gs.y; m[33] += rho * gs.z;
				m[34] += rho * rr.x; m[35] += rho * rr.y; m[36] += rho * rr.z;
				m[37] += rho * q.x * q.x; m[38] += rho * q.y * q.y; m[39] += rho * q.z * q.z;
				m[40] += rho * sp.x * sp.x; m[41] += rho * sp.y * sp.y; m[42] += rho * sp.z * sp.z;
				m[43] += rho;
				lo = lo_n; hi = hi_n; c = cn;
			}
		}
#pragma unroll
		for (int k = 0; k < kGrpVals; k++) {
			float v = m[k];
			v += __shfl_xor_sync(0xffffffffu, v, 4); v += __shfl_xor_sync(0xffffffffu, v, 2); v += __shfl_xor_sync(0xffffffffu, v, 1);
			if (g < g_hi && sl == 0) __stcg(a.grp_sums + (size_t)(ws.grp_off + g) * kGrpVals + k, v);
		}
	}
}

// (wd and ws by value: every field is loaded once, not again behind each barrier)
template <int NT> __device__ void window_tail(const SolveArgs& a, const WinDesc wd, const WinSparse ws, int w, int it, float* smem_base, int* p2_claim) {
	const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
	static_assert(NT >= 6 * (kMaxFrames - 1), "the PCG runs one thread per unknown");
	const int N = wd.n_frames, P = wd.n_pairs, G = ws.n_groups;
	TailSmem s;
	const bool gsm = a.grp_in_smem != 0;
	tail_carve(smem_base, N, P, G, s, gsm);
	const float* grp_g = a.grp_sums + (size_t)ws.grp_off * kGrpVals;      // the same sums in global memory (written with st.cg by the sparse tile)
	const int dimp = s.dimp, ld = s.ld;
	const float wS = a.prm.w_sparse;
	const bool use_dense = a.prm.w_dense > 0.f && P > 0;
	const bool dbg = a.dbg_JtJ && it == a.prm.num_iter_outer - 1;
	ProfRec prf; prf.kind_cta = (1ll << 32) | blockIdx.x; prf.tile_win = ((long long)it << 32) | w;
	PROF_T(0);

	// ---- P0 || P2.  P0: everything the later phases index repeatedly goes to shared memory once (poses, group / pair tables, membership
	//      CSR, the groups' moment sums): ALL of it as asynchronous copies issued back to back - one L2 round trip instead of one per
	//      table - while the same warps clear the system matrix.  P2: per-pair sums over the pair's tiles (already in the model frame; the
	//      tile epilogue applied X S' X^T): a pair's tiles are consecutive and summed in order (deterministic), 4 tiles x RI items per
	//      thread in flight.  The second half of the CTA starts on P2 at once (it needs nothing from P0: the tile ranges come straight from
	//      global memory), the first half joins when its copies are issued; work is handed out in warp-sized blocks by a shared counter.
	int& s_p2_claim = *p2_claim;
	constexpr int RI = 5;
	const int n_p2 = use_dense ? P * kTileVals : 0;
	auto p2_work = [&]() {
		for (;;) {
			int base = 0;
			if (lane == 0) base = atomicAdd(&s_p2_claim, 32 * RI);
			base = __shfl_sync(0xffffffffu, base, 0);
			if (base >= n_p2) break;
			float v[RI]; const float* src[RI]; int nt[RI]; int mx = 0;
#pragma unroll
			for (int r = 0; r < RI; r++) {
				const int k = base + lane + 32 * r;
				v[r] = 0.f; nt[r] = 0; src[r] = a.partial;
				if (k < n_p2) {
					const int p = k / kTileVals, e = k - p * kTileVals;
					nt[r] = __ldg(a.pair_ntile + wd.pair_off + p);
					src[r] = a.partial + (size_t)(wd.tile_off + __ldg(a.pair_tile0 + wd.pair_off + p)) * kTileVals + e;
					mx = max(mx, nt[r]);
				}
			}
			for (int c = 0; c < mx; c += 4) {      // four tiles x RI items in flight per thread; the adds keep the tile order (x + 0.f == x)
				float t[4][RI];
#pragma unroll
				for (int u = 0; u < 4; u++) {
#pragma unroll
					for (int r = 0; r < RI; r++) t[u][r] = (c + u < nt[r]) ? __ldcg(src[r] + (size_t)(c + u) * kTileVals) : 0.f;
				}
#pragma unroll
				for (int u = 0; u < 4; u++) {
#pragma unroll
					for (int r = 0; r < RI; r++) v[r] += t[u][r];
				}
			}
#pragma unroll
			for (int r = 0; r < RI; r++) {
				const int k = base + lane + 32 * r;
				if (k < n_p2) {
					s.pairW[k] = v[r];
					if (a.dbg_cnt && (k % kTileVals) == 27 && it == a.prm.num_iter_outer - 1) a.dbg_cnt[(size_t)w * a.dbg_cnt_stride + k / kTileVals] = v[r];
				}
			}
		}
	};
	if (tid >= NT / 2) p2_work();
	else {
		constexpr int H = NT / 2;
		{   // poses of this iteration: written by this window's previous tail with st.cg -> read from L2
			const float4* Tg = reinterpret_cast<const float4*>(a.T + (size_t)wd.frame_off * 12);
			for (int k = tid; k < N * 3; k += H) cp_async16_cg(reinterpret_cast<float4*>(s.T) + k, Tg + k);
		}
		if (gsm) {  // the sparse moment sums were computed by sparse_sums() while the window's dense tiles were still running (st.cg)
			const float4* Gg = reinterpret_cast<const float4*>(grp_g);
			for (int k = tid; k < G * (kGrpVals / 4); k += H) cp_async16_cg(reinterpret_cast<float4*>(s.grp) + k, Gg + k);
		}
		for (int k = tid; k < G; k += H) { cp_async4(s.gi + k, a.grp_i + ws.grp_off + k); cp_async4(s.gj + k, a.grp_j + ws.grp_off + k); }
		for (int k = tid; k <= G; k += H) cp_async4(s.gstart + k, a.grp_start + ws.grp_off + w + k);
		for (int k = tid; k < P; k += H) {
			const uint2* pr = a.pairs + wd.pair_off + k;
			cp_async4(s.pt + k, &pr->x); cp_async4(s.ps + k, &pr->y);
			cp_async4(s.pt0 + k, a.pair_tile0 + wd.pair_off + k); cp_async4(s.pnt + k, a.pair_ntile + wd.pair_off + k);
		}
		{
			const int* mem = a.mem + ws.mem_off;     // fg_start[N+1] fp_start[N+1] fg_items[2G] fp_items[2P], contiguous like the smem copy
			const int nmem = 2 * (N + 1) + 2 * G + 2 * P;
			for (int k = tid; k < nmem; k += H) cp_async4(s.fg_start + k, mem + k);
		}
		{
			float4* A4 = reinterpret_cast<float4*>(s.A);      // (dimp * ld is a multiple of four floats)
			for (int k = tid; k < (dimp * ld) >> 2; k += H) A4[k] = make_float4(0.f, 0.f, 0.f, 0.f);
		}
		p2_work();
		asm volatile("cp.async.wait_all;" ::: "memory");
	}
	__syncthreads();
	if (tid == 0) s_p2_claim = 0;      // for this CTA's next tail (nobody touches the counter again before several barriers have passed)
	PROF_T(1);
	PROF_T(2);
	__syncthreads();
	PROF_T(3);
	// ---- P3a: per-frame gathers (no atomics, fixed order).  Every output entry e reads one moment from the q-side or the s-side of each
	//      group touching the frame (offset / sign chosen once, outside the loop).  The loop over the frame's groups is a chain of two
	//      dependent shared-memory loads per step (item -> moment): four steps are loaded at a time, the adds keep the list order.
	for (int k = tid; k < N * (kFS + kFD); k += NT) {
		const int f = k / (kFS + kFD), e = k - f * (kFS + kFD);
		float acc = 0.f;
		if (e < kFS) {
			// fS layout: 0 n | 1-3 S | 4-9 Q | 10-12 grad rot | 13-15 grad trans | 16-18 Pw | 19 Pn
			int oq, os; float sg = 1.f;
			if (e == 0) { oq = 0; os = 0; }
			else if (e < 4) { oq = e; os = 3 + e; }
			else if (e < 10) { oq = 3 + e; os = 9 + e; }
			else if (e < 13) { oq = 18 + e; os = 21 + e; sg = -1.f; }
			else if (e < 16) { oq = 21 + e; os = 21 + e; sg = -1.f; }
			else if (e < 19) { oq = 21 + e; os = 24 + e; }
			else { oq = 43; os = 43; }
			const int q1 = s.fg_start[f + 1];
			for (int q = s.fg_start[f]; q < q1; q += 4) {
				int item[4]; float mv[4];
#pragma unroll
				for (int u = 0; u < 4; u++) item[u] = s.fg_items[min(q + u, q1 - 1)];
#pragma unroll
				for (int u = 0; u < 4; u++) {
					const int mo = (item[u] & 0xffff) * kGrpVals + ((item[u] >> 16) ? os : oq);      // role 0: this frame is the group's i (q side); 1: j (s side)
					mv[u] = gsm ? s.grp[mo] : __ldcg(grp_g + mo);
				}
#pragma unroll
				for (int u = 0; u < 4; u++) if (q + u < q1) acc += (item[u] >> 16) ? sg * mv[u] : mv[u];
			}
			s.fS[f * kFS + e] = acc;
		} else {
			const int d = e - kFS;
			if (use_dense && d < 27) {
				const float sgs = (d >= 21) ? -1.f : 1.f;      // Jtr_i += b, Jtr_j -= b ; S adds to both diagonal blocks
				const int q1 = s.fp_start[f + 1];
				for (int q = s.fp_start[f]; q < q1; q += 4) {
					int item[4]; float v[4];
#pragma unroll
					for (int u = 0; u < 4; u++) item[u] = s.fp_items[min(q + u, q1 - 1)];
#pragma unroll
					for (int u = 0; u < 4; u++) v[u] = s.pairW[(item[u] & 0xffff) * kTileVals + d];
#pragma unroll
					for (int u = 0; u < 4; u++) if (q + u < q1) acc += (item[u] >> 16) ? sgs * v[u] : v[u];             // role 0: target, 1: source
				}
			}
			s.fD[f * kFD + d] = acc;
		}
	}
	__syncthreads();
	PROF_T(4);
	// ---- P3b: diagonal blocks, right-hand side, Jacobi preconditioner from the per-frame sums
	{
		const int per = 21 + 6 + 6;
		for (int k = tid; k < (N - 1) * per; k += NT) {
			const int f = 1 + k / per, e = k % per;
			const int base = (f - 1) * 6;
			const float* F = s.fS + f * kFS;
			const float* D = s.fD + f * kFD;
			if (e < 21) {
				int r, c;
				unpack_sym(e, r, c);
				float sp;
				if (r < 3 && c < 3) sp = (r == c) ? F[0] : 0.f;                                   // TT = n I
				else if (r < 3) sp = -skew(F + 1, r, c - 3);                                       // TR = -[S]x
				else { const int ra = r - 3, cb = c - 3; const float tr = F[4] + F[7] + F[9];
					const int qi = (ra == 0) ? cb : (ra == 1 ? 2 + cb : 5);                          // packed (ra,cb), ra<=cb
					sp = ((ra == cb) ? tr : 0.f) - F[4 + qi]; }
				const float dn = D[e];
				const float v = wS * sp + dn;
				s.A[(base + r) * ld + base + c] = v;
				s.A[(base + c) * ld + base + r] = v;
				if (dbg) { float* Dg = a.dbg_JtJ + (size_t)w * a.dbg_stride * a.dbg_stride; const int dim = 6 * N;
					Dg[(f * 6 + r) * dim + f * 6 + c] = dn; Dg[(f * 6 + c) * dim + f * 6 + r] = dn; }
			} else if (e < 27) {
				const int r = e - 21;
				const float gs = (r < 3) ? F[13 + r] : F[10 + (r - 3)];
				const float dn = D[21 + r];
				s.rhs[base + r] = -wS * gs - dn;
				if (dbg && a.dbg_Jtr) a.dbg_Jtr[(size_t)w * a.dbg_stride + f * 6 + r] = dn;
			} else {
				const int r = e - 27;
				float pc;
				if (r < 3) pc = F[19];
				else { const int ax = r - 3; pc = F[16 + (ax + 1) % 3] + F[16 + (ax + 2) % 3]; }
				s.Minv[base + r] = (pc > kEps) ? 1.0f / pc : 1.0f;
			}
		}
	}
	__syncthreads();
	PROF_T(5);
	// ---- P4a: sparse cross blocks (i,j): J_i^T J_j, both frames free.  One thread per (group, 3x3 sub-block): uniform code per
	//      thread, 9 entries each.  Sub-blocks: 0 = TT (-n I), 1 = TR ([sum s]x), 2 = RT (-[sum q]x), 3 = RR (-((q.s) I - s q^T)).
	const bool uniq = ws.unique_blocks != 0;
	for (int k = tid; k < G * 4; k += NT) {
		const int g = k >> 2, sb = k & 3;
		const int gi = s.gi[g], gj = s.gj[g];
		if (gi < 1 || gj < 1 || gi == gj) continue;
		float ml[28];
#pragma unroll
		for (int q = 0; q < 28; q++) ml[q] = gsm ? s.grp[g * kGrpVals + q] : __ldcg(grp_g + (size_t)g * kGrpVals + q);
		const float* m = ml;
		const int r0 = (sb >> 1) * 3, c0 = (sb & 1) * 3;
		const float tr = m[19] + m[23] + m[27];
#pragma unroll
		for (int a3 = 0; a3 < 3; a3++) {
#pragma unroll
			for (int b3 = 0; b3 < 3; b3++) {
				float v;
				if (sb == 0) v = (a3 == b3) ? -m[0] : 0.f;
				else if (sb == 1) v = skew(m + 4, a3, b3);
				else if (sb == 2) v = -skew(m + 1, a3, b3);
				else v = -(((a3 == b3) ? tr : 0.f) - m[19 + a3 * 3 + b3]);
				v *= wS;
				float* p1 = &s.A[((gi - 1) * 6 + r0 + a3) * ld + (gj - 1) * 6 + c0 + b3];
				float* p2 = &s.A[((gj - 1) * 6 + c0 + b3) * ld + (gi - 1) * 6 + r0 + a3];
				if (uniq) { *p1 = v; *p2 = v; } else { atomicAdd(p1, v); atomicAdd(p2, v); }
			}
		}
	}
	__syncthreads();
	// ---- P4b: dense cross blocks: -S for pairs whose cross block survives FlipJtJ (target < source) or all if !compat
	if (use_dense) {
		for (int k = tid; k < P * 6; k += NT) {
			const int p = k / 6, r = k - p * 6;
			const int ti = s.pt[p], sj = s.ps[p];
			if (ti < 1 || sj < 1) continue;
			if (wd.compat_flip && !(ti < sj)) continue;
#pragma unroll
			for (int c = 0; c < 6; c++) {
				const float v = -s.pairW[p * kTileVals + c_sym_idx[r * 6 + c]];
				float* p1 = &s.A[((sj - 1) * 6 + r) * ld + (ti - 1) * 6 + c];
				float* p2 = &s.A[((ti - 1) * 6 + c) * ld + (sj - 1) * 6 + r];
				if (uniq) { *p1 += v; *p2 += v; } else { atomicAdd(p1, v); atomicAdd(p2, v); }
				if (dbg) {
					float* Dg = a.dbg_JtJ + (size_t)w * a.dbg_stride * a.dbg_stride;
					const int dim = 6 * N;
					atomicAdd(&Dg[(sj * 6 + r) * dim + ti * 6 + c], v);
					atomicAdd(&Dg[(ti * 6 + c) * dim + sj * 6 + r], v);
				}
			}
		}
	}
	__syncthreads();
	PROF_T(6);

	// ---- PCG (PCGInit_Kernel1/2, PCGStep_Kernel*: SolverBundling.cu:575-818).  One THREAD per unknown: thread r reads row r of A
	//      with 16-byte loads (conflict-free, see tail_ld) against p in shared memory (broadcast) - no cross-lane reduction inside the
	//      matrix-vector product; only the two scalar products of a step are reduced (warp shuffle + one word per warp through shared
	//      memory, named barrier among the ceil(dimp / 32) warps that take part).  The first version spread every ROW over the lanes of
	//      a warp: 20 dependent shuffles per four rows.
	{
		__shared__ float s_dot[3][8];
		const int nwp = (dimp + 31) >> 5;      // warps that take part (<= 6)
		if (dimp <= 64) {
			// up to 11 frames (the shipped max_BA_frames is 10): ONE warp, two rows per lane - the scalar products are plain warp shuffles,
			// nothing crosses a barrier
			if (wid == 0) {
				const int r0 = lane, r1 = lane + 32;
				const bool act0 = r0 < dimp, act1 = r1 < dimp;
				const int n4 = (dimp + 3) >> 2;
				float rr0 = act0 ? s.rhs[r0] : 0.f, rr1 = act1 ? s.rhs[r1] : 0.f;
				const float mi0 = act0 ? s.Minv[r0] : 0.f, mi1 = act1 ? s.Minv[r1] : 0.f;
				float pp0 = mi0 * rr0, pp1 = mi1 * rr1, dl0 = 0.f, dl1 = 0.f;
				if (r0 < 4 * n4) s.p[r0] = pp0;      // (inactive rows hold zeros: the padding of p up to a multiple of four is zero, like A's columns there)
				if (r1 < 4 * n4) s.p[r1] = pp1;
				__syncwarp();
				float rz = warp_sum(rr0 * pp0 + rr1 * pp1);
				const float4* A0 = reinterpret_cast<const float4*>(s.A + (act0 ? r0 : 0) * ld);
				const float4* A1 = reinterpret_cast<const float4*>(s.A + (act1 ? r1 : 0) * ld);
				const float4* p4 = reinterpret_cast<const float4*>(s.p);
#pragma unroll 1
				for (int lin = 0; lin < a.prm.num_iter_inner; lin++) {
					float a00 = 0.f, a01 = 0.f, a02 = 0.f, a03 = 0.f, a10 = 0.f, a11 = 0.f, a12 = 0.f, a13 = 0.f;
#pragma unroll 4
					for (int c = 0; c < n4; c++) {
						const float4 pv = p4[c], u = A0[c], v = A1[c];
						a00 += u.x * pv.x; a01 += u.y * pv.y; a02 += u.z * pv.z; a03 += u.w * pv.w;
						a10 += v.x * pv.x; a11 += v.y * pv.y; a12 += v.z * pv.z; a13 += v.w * pv.w;
					}
					const float ap0 = act0 ? (a00 + a01) + (a02 + a03) : 0.f, ap1 = act1 ? (a10 + a11) + (a12 + a13) : 0.f;
					const float pAp = warp_sum(pp0 * ap0 + pp1 * ap1);
					const float alpha = (pAp > kEps) ? rz / pAp : 0.f;
					dl0 += alpha * pp0; dl1 += alpha * pp1;
					rr0 -= alpha * ap0; rr1 -= alpha * ap1;
					const float zz0 = mi0 * rr0, zz1 = mi1 * rr1;
					const float rz_new = warp_sum(zz0 * rr0 + zz1 * rr1);
					const float beta = (rz > kEps) ? rz_new / rz : 0.f;
					rz = rz_new;
					pp0 = zz0 + beta * pp0; pp1 = zz1 + beta * pp1;
					__syncwarp();      // every lane has read the old p
					if (act0) s.p[r0] = pp0;
					if (act1) s.p[r1] = pp1;
					__syncwarp();
				}
				if (act0) s.delta[r0] = dl0;
				if (act1) s.delta[r1] = dl1;
			}
		} else if (wid < nwp) {
			const int r = tid;
			const bool act = r < dimp;
			const int rc = act ? r : dimp - 1;       // idle lanes of the last warp read a valid row
			const int nthr = nwp * 32;
			const int n4 = (dimp + 3) >> 2;
			float rr = act ? s.rhs[r] : 0.f;
			const float mi = act ? s.Minv[r] : 0.f;
			float pp = mi * rr, dl = 0.f;
			if (r < 4 * n4) s.p[r] = act ? pp : 0.f;      // (the padding of p up to a multiple of four is zero, and so are A's columns there)
			{ const float v = warp_sum(rr * pp); if (lane == 0) s_dot[0][wid] = v; }
			asm volatile("bar.sync 1, %0;" ::"r"(nthr) : "memory");
			float rz = 0.f;
			for (int q = 0; q < nwp; q++) rz += s_dot[0][q];
			const float4* Arow = reinterpret_cast<const float4*>(s.A + rc * ld);
			const float4* p4 = reinterpret_cast<const float4*>(s.p);
#pragma unroll 1
			for (int lin = 0; lin < a.prm.num_iter_inner; lin++) {
				float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
#pragma unroll 4
				for (int c = 0; c < n4; c++) { const float4 av = Arow[c], pv = p4[c]; a0 += av.x * pv.x; a1 += av.y * pv.y; a2 += av.z * pv.z; a3 += av.w * pv.w; }
				const float ap = act ? (a0 + a1) + (a2 + a3) : 0.f;
				{ const float v = warp_sum(pp * ap); if (lane == 0) s_dot[1][wid] = v; }
				asm volatile("bar.sync 1, %0;" ::"r"(nthr) : "memory");
				float pAp = 0.f;
				for (int q = 0; q < nwp; q++) pAp += s_dot[1][q];
				const float alpha = (pAp > kEps) ? rz / pAp : 0.f;
				dl += alpha * pp;
				rr -= alpha * ap;
				const float zz = mi * rr;
				{ const float v = warp_sum(zz * rr); if (lane == 0) s_dot[2][wid] = v; }
				asm volatile("bar.sync 1, %0;" ::"r"(nthr) : "memory");
				float rz_new = 0.f;
				for (int q = 0; q < nwp; q++) rz_new += s_dot[2][q];
				const float beta = (rz > kEps) ? rz_new / rz : 0.f;
				rz = rz_new;
				pp = zz + beta * pp;
				if (act) s.p[r] = pp;
				asm volatile("bar.sync 1, %0;" ::"r"(nthr) : "memory");      // p of the next step is complete (and s_dot[1] / [2] may be rewritten)
			}
			if (act) s.delta[r] = dl;
		}
	}
	__syncthreads();
	PROF_T(7);
	if (dbg && a.dbg_sys) {      // what the PCG saw and returned: A, rhs, Jacobi diagonal, delta (bt_solve_debug_system)
		const int st = a.dbg_sys_stride;
		float* Sg = a.dbg_sys + (size_t)w * st * (st + 3);
		for (int k = tid; k < dimp * dimp; k += NT) { const int r = k / dimp; Sg[k] = s.A[r * ld + (k - r * dimp)]; }
		for (int k = tid; k < dimp; k += NT) { Sg[st * st + k] = s.rhs[k]; Sg[st * st + st + k] = s.Minv[k]; Sg[st * st + 2 * st + k] = s.delta[k]; }
	}
	// ---- pose update: x <- log(exp(delta) * exp(x))  (computeLieUpdate), new T for the next iteration
	const bool last = (it == a.prm.num_iter_outer - 1);
	for (int f = tid; f < N; f += NT) {
		float* xg = a.x + (size_t)(wd.frame_off + f) * 6;
		V3 rot = mk(__ldcg(xg + 0), __ldcg(xg + 1), __ldcg(xg + 2)), trans = mk(__ldcg(xg + 3), __ldcg(xg + 4), __ldcg(xg + 5));
		float Tn[12];
		if (f >= 1) {
			const float* dl = s.delta + (f - 1) * 6;
			float U[12];
			se3_exp(mk(dl[3], dl[4], dl[5]), mk(dl[0], dl[1], dl[2]), U);
			const float* Cm = s.T + f * 12;    // exp(x) of this iteration, already in shared memory
			for (int r = 0; r < 3; r++) {
				for (int c = 0; c < 4; c++) {
					float v = U[r * 4 + 0] * Cm[0 * 4 + c] + U[r * 4 + 1] * Cm[1 * 4 + c] + U[r * 4 + 2] * Cm[2 * 4 + c];
					if (c == 3) v += U[r * 4 + 3];
					Tn[r * 4 + c] = v;
				}
			}
			se3_log(Tn, rot, trans);
			__stcg(xg + 0, rot.x); __stcg(xg + 1, rot.y); __stcg(xg + 2, rot.z); __stcg(xg + 3, trans.x); __stcg(xg + 4, trans.y); __stcg(xg + 5, trans.z);
		}
		se3_exp(rot, trans, Tn);
		float* Tg = a.T + (size_t)(wd.frame_off + f) * 12;
		for (int k = 0; k < 12; k++) __stcg(Tg + k, Tn[k]);
		if (last) {   // convertPosesToMatricesCU (SBA.cu:97-104)
			float* Po = a.pose_out + (size_t)(wd.frame_off + f) * 16;
			for (int k = 0; k < 12; k++) Po[k] = Tn[k];
			Po[12] = 0.f; Po[13] = 0.f; Po[14] = 0.f; Po[15] = 1.f;
		}
	}
	__syncthreads();
	PROF_T(8);
	if (a.prof && threadIdx.x == 0) { prf.t[9] = 0; prof_emit(a, prf); }
}

// ------------------------------------------------------------------------------------------------ k_solve
// One step of the tile's transposing butterfly, then the next (HALF = 16, 8, ..., 1): the lanes with bit HALF set keep the upper half
// of v and send the lower one, the others the reverse.  A template parameter, so every index into v is a compile-time constant and
// v stays in registers.
template <int HALF> __device__ __forceinline__ void butterfly_step(float (&v)[32], int lane) {
	const bool up = (lane & HALF) != 0;
#pragma unroll
	for (int k = 0; k < HALF; k++) {
		const float send = up ? v[k] : v[k + HALF];
		const float keep = up ? v[k + HALF] : v[k];
		v[k] = keep + __shfl_xor_sync(0xffffffffu, send, HALF);
	}
	if constexpr (HALF > 1) butterfly_step<HALF / 2>(v, lane);
}
// Entry e of a dense tile's constants, from the current poses of its frames: e < 12: transform = T_i^-1 T_j (rigid inverse), row r,
// col c; 12 <= e < 48: X_i = [[R,0],[[t]x R, R]] of the TARGET frame, which maps the tile's sums to the model frame; e == 48: the
// window's projection / texel geometry, read by the pixel loop where it is used.
__device__ __forceinline__ void tile_const(const SolveArgs& a, const Tile& tl, int e, float* sM, float* sX, float* sG) {
	if (e < 12) {
		const float* Ti = a.T + (size_t)tl.tgt_slot * 12;
		const float* Tj = a.T + (size_t)tl.src_slot * 12;
		const int r = e >> 2, c = e & 3;
		float v = 0.f;
		for (int k = 0; k < 3; k++) {
			const float rik = __ldcg(Ti + k * 4 + r);          // R_i^T (r,k) = R_i(k,r)
			v += rik * ((c < 3) ? __ldcg(Tj + k * 4 + c) : (__ldcg(Tj + k * 4 + 3) - __ldcg(Ti + k * 4 + 3)));
		}
		sM[e] = v;
	} else if (e < 48) {
		const float* Ti = a.T + (size_t)tl.tgt_slot * 12;
		const int x = e - 12, r = x / 6, c = x - r * 6;
		float v;
		if (r < 3) v = (c < 3) ? __ldcg(Ti + r * 4 + c) : 0.f;
		else if (c >= 3) v = __ldcg(Ti + (r - 3) * 4 + (c - 3));
		else { const float tx = __ldcg(Ti + 3), ty = __ldcg(Ti + 7), tz = __ldcg(Ti + 11); v = 0.f; for (int kk = 0; kk < 3; kk++) v += skew3(tx, ty, tz, r - 3, kk) * __ldcg(Ti + kk * 4 + c); }
		sX[x] = v;
	} else if (e == 48) {
		const WinDesc& wd = a.wins[tl.win];
		sG[0] = wd.fx; sG[1] = wd.fy; sG[2] = wd.cx; sG[3] = wd.cy;
		sG[4] = wd.tg.ifx; sG[5] = wd.tg.ify; sG[6] = wd.tg.icx; sG[7] = wd.tg.icy;
		sG[8] = wd.tg.scaleW; sG[9] = wd.tg.scaleH; sG[10] = __int_as_float(wd.w); sG[11] = __int_as_float(wd.h);
	}
}
// Thread tid's entry of tile_const: in the CTA-wide set-up tid < 12, 32..67 and 96; while warp 0 finishes the previous tile the
// transform moves to 128..139.  -1: none.  Each entry takes a few dependent L2 loads, so they are spread over warps.
__device__ __forceinline__ int tile_const_entry(int tid, bool warp0_busy) {
	if (tid >= 32 && tid < 68) return 12 + (tid - 32);
	if (tid == 96) return 48;
	const int m = warp0_busy ? tid - 128 : tid;
	return (m >= 0 && m < 12) ? m : -1;
}
template <int NT, int MINB> __global__ void __launch_bounds__(NT, MINB) k_solve(SolveArgs a) {
	extern __shared__ __align__(16) float dyn_smem[];
	__shared__ int s_tile, s_it, s_idx;
	__shared__ Tile s_tl[2];      // the tile being processed and the one claimed for the next round (thread 0 fetches its record a tile ahead)
	// the tile's constants.  s_pre[] = 1: written (and the tile's iteration flag acquired) by warps 1.. while warp 0 finished the previous
	// tile, so the tile starts on its pixels at once.  Only X, which warp 0's epilogue reads, needs a second buffer; the pixel loop reads
	// s_M and s_G at fixed addresses.
	__shared__ __align__(16) float s_M[12];
	__shared__ __align__(16) float s_G[12];
	__shared__ float s_X[2][36];
	__shared__ int s_pre[2], s_nxt;
	__shared__ float s_red[kTileVals];
	__shared__ float s_part[(NT / 32)][kTileVals];
	__shared__ int s_is_last, s_p2_claim;
	const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
	chain_wait();
	if (a.tstamp && blockIdx.x == 0 && tid == 0) a.tstamp[2] = global_ns();
	const auto stamp_end = [&]() { if (a.tstamp && tid == 0) atomicMax((unsigned long long*)a.tstamp + 3, (unsigned long long)global_ns()); };
	const int total = *a.n_tiles_total;
	if (total <= 0) { stamp_end(); return; }
	const int all = total * a.prm.num_iter_outer;      // (the tile plan reports an overflow when this does not fit 31 bits)
	// One iteration's tiles fit the grid (a single window, a handful of windows): STATIC assignment - CTA c runs tile c of every GN
	// iteration.  With the queue the CTAs claim one tile ahead, i.e. into the NEXT iteration, and then sit on the iteration flag while
	// the current iteration's last tiles wait for a CTA that finishes its first one, and an iteration's tile phase takes up to two tiles' time.
	const bool fixed = total <= (int)gridDim.x;
	if (fixed && (int)blockIdx.x >= total) { stamp_end(); return; }
	if (tid == 0) {
		const int t0 = fixed ? (int)blockIdx.x : atomicAdd(a.queue, 1);
		s_tile = t0; s_p2_claim = 0; s_pre[0] = 0;
		if (t0 < all) { const int it0 = t0 / total; s_it = it0; s_idx = t0 - it0 * total; s_tl[0] = a.tiles[t0 - it0 * total]; }
	}
	int cur = 0;
	for (;;) {
		__syncthreads();
		if (s_tile >= all) break;
		const int it = s_it, tl_idx = s_idx;
		const Tile& tl = s_tl[cur];      // (read from shared memory where it is used: 12 registers less across the pixel loop)
		// claim the NEXT tile now: the atomic's round trip hides behind this tile.  Safe for the iteration dependencies:
		// a CTA only ever waits on tiles with a smaller index than the one it is processing, never on its look-ahead.
		int nxt = 0;
		if (tid == 0) nxt = fixed ? s_tile + total : atomicAdd(a.queue, 1);
		ProfRec prf; PROF_T(0);
		const WinDesc& wd = a.wins[tl.win];      // (fields are read where they are used: geometry in the pixel loop, the rest in the tail)
		const bool pre = s_pre[cur] != 0;
		if (it > 0 && !pre) {   // this window's previous GN iteration must have published its poses
			if (tid == 0) { while (ld_relaxed(a.iter_done + tl.win) < it) __nanosleep(64); (void)ld_acquire(a.iter_done + tl.win); }
			__syncthreads();
		}
		PROF_T(1);
		if (tl.pair == -2) {     // the window's sparse tile: moment sums of all its (i,j) groups for the current poses (CTA-uniform branch)
			PROF_T(2);
			sparse_sums<NT>(a, tl.win, tl.start, tl.count);
			PROF_T(3);
			int itn = 0, idxn = 0;      // thread 0: the record of the tile claimed above (in flight across the barrier and the ticket)
			if (tid == 0 && nxt < all) { itn = nxt / total; idxn = nxt - itn * total; tile_fetch_async(&s_tl[cur ^ 1], a.tiles + idxn); }
			__syncthreads();      // (every thread's sums are written; the barrier orders them before thread 0's release below)
			if (tid == 0) {
				const int done = ticket_acq_rel(a.tiles_done + tl.win) + 1;
				s_is_last = (done == (it + 1) * tl.n_tiles_win);
				s_tile = nxt;
				if (nxt < all) { s_it = itn; s_idx = idxn; }
				s_pre[cur ^ 1] = 0;
				tile_fetch_wait();
			}
			PROF_T(4);
			__syncthreads();
		} else {
		TileAcc acc;
#pragma unroll
		for (int k = 0; k < kTileVals; k++) acc.v[k] = 0.f;
		if (tl.pair >= 0) {
			if (!pre) {
				const int e = tile_const_entry(tid, false);
				if (e >= 0) tile_const(a, tl, e, s_M, s_X[cur], s_G);
			}
			if (!pre) __syncthreads();
			PROF_T(2);
			tile_pixels<NT>(a, tl.src, tl.tex, s_M, s_G, tl.start, tl.count, acc);
		}
		PROF_T(3);
		int itn = 0, idxn = 0;
		if (tid == 0 && nxt < all) { itn = nxt / total; idxn = nxt - itn * total; tile_fetch_async(&s_tl[cur ^ 1], a.tiles + idxn); }   // the next tile's record, in flight behind the reduction
		// block reduction of the 28 sums -> this tile's slot.  Warp level: a transposing butterfly (31 shuffles instead of
		// 28 x 5): after the five steps lane L holds the warp total of value L.
		{
			float v[32];
#pragma unroll
			for (int k = 0; k < 32; k++) v[k] = (k < kTileVals) ? acc.v[k] : 0.f;
			butterfly_step<16>(v, lane);
			if (lane < kTileVals) s_part[wid][lane] = v[0];
		}
		if (tid == 0) { s_nxt = nxt; if (!fixed) tile_fetch_wait(); }      // (warps 1.. read the next tile's record after the barrier)
		__syncthreads();
		if (wid == 0) {   // warp 0 finishes the tile: cross-warp sum, model-frame transform, store, ticket
			float red = 0.f;
			if (lane < kTileVals) {
#pragma unroll
				for (int k = 0; k < (NT / 32); k++) red += s_part[k][lane];
				s_red[lane] = red;
			}
			__syncwarp();
			if (lane < kTileVals) {   // S = X S' X^T, b = X b' (rows 0-2 of X have 3 non-zeros); entry 27 = #correspondences
				float out = red;
				if (tl.pair >= 0 && lane < 27) {
					out = 0.f;
					if (lane < 21) {
						const int r = c_sym_r[lane], c = c_sym_c[lane];
						float xr[6], xc[6];
#pragma unroll
						for (int u = 0; u < 6; u++) { xr[u] = s_X[cur][r * 6 + u]; xc[u] = s_X[cur][c * 6 + u]; }   // zero entries make the short rows exact
#pragma unroll
						for (int u = 0; u < 6; u++) {
							float tsum = 0.f;
#pragma unroll
							for (int v = 0; v < 6; v++) tsum += s_red[c_sym_idx[u * 6 + v]] * xc[v];
							out += xr[u] * tsum;
						}
					} else {
						const int r = lane - 21;
#pragma unroll
						for (int u = 0; u < 6; u++) out += s_X[cur][r * 6 + u] * s_red[21 + u];
					}
				}
				__stcg(a.partial + (size_t)tl_idx * kTileVals + lane, out);
			}
			__syncwarp();             // orders the 28 lanes' stores before lane 0's release
			if (lane == 0) {
				const int done = ticket_acq_rel(a.tiles_done + tl.win) + 1;
				s_is_last = (done == (it + 1) * tl.n_tiles_win);
				s_tile = nxt;
				if (nxt < all) { s_it = itn; s_idx = idxn; }
				if (fixed) tile_fetch_wait();
			}
		} else if (fixed) {   // (the next tile is this window's next iteration: its flag waits for this tile's ticket)
			if (tid == 32) s_pre[cur ^ 1] = 0;
		} else {   // warps 1..: the next tile's set-up while warp 0 finishes this one, when its iteration flag is already set
			const int nx = s_nxt;
			const Tile& tn = s_tl[cur ^ 1];
			if (tid == 32) {
				int ok = 0;
				if (nx < all) {
					const int itx = nx / total;
					ok = itx == 0 || ld_relaxed(a.iter_done + tn.win) >= itx;
					if (ok && itx > 0) (void)ld_acquire(a.iter_done + tn.win);
				}
				s_pre[cur ^ 1] = ok;
			}
			asm volatile("bar.sync 2, %0;" ::"r"(NT - 32) : "memory");      // (barrier 1 belongs to the tail's PCG)
			if (s_pre[cur ^ 1] && tn.pair >= 0) {
				const int e = tile_const_entry(tid, true);
				if (e >= 0) tile_const(a, tn, e, s_M, s_X[cur ^ 1], s_G);      // (every warp is past its pixels)
			}
		}
		PROF_T(4);
		__syncthreads();
		}      // dense tile
		PROF_T(5);
		if (a.prof && tid == 0) { prf.kind_cta = blockIdx.x; prf.tile_win = ((long long)tl_idx << 32) | ((long long)it << 16) | tl.count; prf.t[6] = prf.t[7] = prf.t[8] = prf.t[9] = 0; prof_emit(a, prf); }
		// this CTA's look-ahead claim found no tile left: the next kernel on the stream may launch into the SMs this CTA and the others
		// that are done leave idle, while the windows' last tails run.  It only waits for k_solve's completion, and every CTA of k_solve is
		// resident before any of its CTAs (the grid never exceeds one wave), so the persistent kernel's progress argument holds (DESIGN §3.1).
		if (s_tile >= all) chain_release();
		if (s_is_last) {
			window_tail<NT>(a, wd, a.wsp[tl.win], tl.win, it, dyn_smem, &s_p2_claim);
			__threadfence();
			__syncthreads();
			if (tid == 0) st_release(a.iter_done + tl.win, it + 1);
		}
		cur ^= 1;
	}
	stamp_end();
}

// ------------------------------------------------------------------------------------------------ host side
// Everything bt_solve_stage uploads lives in ONE pinned block mirrored by the device staging blocks (same offsets): the small tables
// first (sized for the worst case of this window count), the correspondences last so that the copy length follows the actual number of
// entries.  [0, wsp.off) is what k_prep_frames needs.
struct StageLayout : TableLayout {
	Slice<WinDesc> wins; Slice<const float*> dp; Slice<const float4*> np; Slice<int> fw; Slice<const float4*> texp, srcp; Slice<const int*> nsrcp;
	Slice<float> pose; Slice<uint2> pairs; Slice<int> pwin, psrc;
	Slice<WinSparse> wsp; Slice<int> gi, gj, gs, mem; Slice<bt_entryj> corr;
};
static StageLayout stage_layout(int n_windows, size_t F, size_t C, int max_frames, size_t maxG, size_t maxP) {
	StageLayout L;
	const size_t nw = (size_t)n_windows;
	L.wins = L.add<WinDesc>(nw); L.dp = L.add<const float*>(F); L.np = L.add<const float4*>(F); L.fw = L.add<int>(F);
	L.texp = L.add<const float4*>(F); L.srcp = L.add<const float4*>(F); L.nsrcp = L.add<const int*>(F);
	L.pose = L.add<float>(16 * F); L.pairs = L.add<uint2>(maxP * nw); L.pwin = L.add<int>(maxP * nw); L.psrc = L.add<int>(maxP * nw);
	L.wsp = L.add<WinSparse>(nw); L.gi = L.add<int>(maxG * nw); L.gj = L.add<int>(maxG * nw); L.gs = L.add<int>((maxG + 1) * nw);
	L.mem = L.add<int>((2 * ((size_t)max_frames + 1) + 2 * maxG + 2 * maxP) * nw);
	L.corr = L.add<bt_entryj>(C + 1);      // (one entry of slack behind the last)
	return L;
}

struct SolverState {
	bool ready = false;
	bt_solver_limits lim{};
	int npix_max = 0, max_pairs = 0, max_frames_total = 0, max_tiles = 0, max_groups = 0;
	DevBuf blk_cnt, grp_sums, texel, src, nsrc, x, T, pose_out, tiles, scalars, partial, tiles_done, iter_done, pair_tile0, pair_ntile, dbgJ, dbgR, dbgC, dbgS, prof;
	StageLayout layout{};
	// frame cache (bt_frame_cache_*): quarter-res maps of keyframes, built once, referenced by bt_window::cache_slots
	struct CacheMeta { bool valid = false; int H = 0, W = 0; float fx = 0, fy = 0, cx = 0, cy = 0, dmin = 0, dmax = 0; };
	DevBuf c_texel, c_src, c_nsrc, c_blk;
	TableBlock<2> c_tables;              // two pinned table blocks, used alternately: a store only waits for the upload of the store before last,
	                                     // so back-to-back stores (one new frame per window per step) never stall the host behind the GPU
	int c_capacity = 0, c_npix = 0;      // (c_capacity 0 until bt_frame_cache_reserve completes)
	float c_downscale = 0.f;
	std::vector<CacheMeta> c_meta;
	int prof_cap = 0;
	TableBlock<1, 2> stage;              // the staging block: read by the uploads on copy_stream into device block stage_cur
	PinnedBuf h_poses;
	// streaming form (bt_solve_windows_begin / _end): two batches may be in flight; each has its own pinned pose block and completion event
	PinnedBuf h_pipe[2];
	Event ev_pipe[2];
	bool pipe_pending[2] = { false, false };
	int pipe_frames[2] = { 0, 0 };
	int pipe_head = 0, pipe_tail = 0;
	// last staged batch
	int n_windows = 0, frames_total = 0, smem_bytes = 0, chunk = 1024;
	bt_solver_params prm{};
	float d2max = 0.f;                   // SolveArgs::d2max of prm.dense_dist_thresh
	std::vector<int> frame_off;
	std::vector<int> n_frames;
	bool staged = false, debug = false, timing = false;
	double host_us[6] = { 0, 0, 0, 0, 0, 0 };   // host time of the last call: tables+early upload, prep launch, correspondence scan+staging, run (launch), fetch (copy + wait), total
	bool grp_in_smem = true;
	int force_chunk = 0;                 // tuning knob (BT_SOLVE_CHUNK): source pixels per dense tile
	int launches = 0;
	int attr_bytes = 0, occ = BT_SOLVE_MIN_CTAS, occ_smem = -1;
	bool prep_launched = false, any_uncached = true;
	Stream copy_stream;
	Event ev_prev, ev_early;
	Event ev_stage_free[2];              // behind the k_solve that last read staging block 0 / 1
	int stage_cur = 0;
	// ev_stage_free of the current block is recorded when the next batch is staged, on the stream of the last bt_solve_run, not right
	// behind k_solve: there it would sit between k_solve and the next step's store and cut the launch chain
	cudaStream_t run_stream = nullptr;
	bool run_pending = false;
	DevBuf tstamp;                       // SolveArgs::tstamp (timing on)
};
void StateDeleter::operator()(SolverState* s) const { delete s; }

}  // namespace bt

using namespace bt;

extern "C" int bt_solver_reserve(bt_ctx* ctx, const bt_solver_limits* lim) {
	BT_REQUIRE(ctx && lim, BT_ERR_INVALID_ARG, "bt_solver_reserve: NULL argument");
	BT_REQUIRE(lim->max_windows > 0 && lim->max_frames >= 2 && lim->max_frames <= kMaxFrames && lim->max_corr >= 0 && lim->H > 0 && lim->W > 0 && lim->image_downscale >= 1.0f,
	           BT_ERR_INVALID_ARG, "bt_solver_reserve: bad limits (max_frames must be 2..%d)", kMaxFrames);
	SolverState* s;
	BT_TRY(take_state(ctx, &bt_ctx::solver, &s));
	{ const char* e = getenv("BT_SOLVE_CHUNK"); const int v = e ? atoi(e) : 0; s->force_chunk = (v >= 256 && v <= 16384) ? (v + 255) / 256 * 256 : 0; }
	const int w = (int)(lim->W / lim->image_downscale), h = (int)(lim->H / lim->image_downscale);
	const int npix_max = w * h;
	const int F = lim->max_windows * lim->max_frames;
	const int max_pairs = lim->max_frames * (lim->max_frames - 1);   // both directions allowed in custom lists
	const int max_groups = lim->max_frames * lim->max_frames;
	const int min_chunk = 256;   // worst case: every pixel valid at the smallest chunk the scheduler ever picks
	const int max_tiles = lim->max_windows * (lim->max_frames * (lim->max_frames - 1) / 2) * ((npix_max + min_chunk - 1) / min_chunk + 1) + kSparseTiles * lim->max_windows;
	{   // worst case over every window count <= max_windows (the table offsets grow with the count, so the maximum is at max_windows)
		const StageLayout L = stage_layout(lim->max_windows, (size_t)F, (size_t)lim->max_corr * lim->max_windows, lim->max_frames, (size_t)max_groups, (size_t)max_pairs);
		BT_TRY(s->stage.reserve(L.total));
	}
	BT_TRY(s->texel.alloc(sizeof(float4) * (size_t)npix_max * F));
	BT_TRY(s->src.alloc(sizeof(float4) * 2 * (size_t)npix_max * F));
	BT_TRY(s->nsrc.alloc(sizeof(int) * F));
	BT_TRY(s->grp_sums.alloc(sizeof(float) * kGrpVals * (size_t)max_groups * lim->max_windows));
	BT_TRY(s->blk_cnt.alloc(sizeof(int) * (size_t)F * ((npix_max + 1023) / 1024)));
	BT_TRY(s->x.alloc(sizeof(float) * 6 * F)); BT_TRY(s->T.alloc(sizeof(float) * 12 * F)); BT_TRY(s->pose_out.alloc(sizeof(float) * 16 * F));
	BT_TRY(s->pair_tile0.alloc(sizeof(int) * (size_t)max_pairs * lim->max_windows));
	BT_TRY(s->pair_ntile.alloc(sizeof(int) * (size_t)max_pairs * lim->max_windows));
	BT_TRY(s->tiles.alloc(sizeof(Tile) * (size_t)max_tiles));
	BT_TRY(s->partial.alloc(sizeof(float) * kTileVals * (size_t)max_tiles));
	BT_TRY(s->scalars.alloc(64));
	BT_CUDA(cudaMemset(s->scalars.p, 0, 64));
	BT_TRY(s->tiles_done.alloc(sizeof(int) * lim->max_windows)); BT_TRY(s->iter_done.alloc(sizeof(int) * lim->max_windows));
	s->lim = *lim;
	s->npix_max = npix_max; s->max_frames_total = F; s->max_pairs = max_pairs; s->max_groups = max_groups; s->max_tiles = max_tiles;
	s->ready = true;
	return BT_OK;
}

extern "C" int bt_solve_enable_debug(bt_ctx* ctx, int on) {
	SolverState* s;
	BT_TRY(state_of(ctx, &bt_ctx::solver, "bt_solve_enable_debug", "bt_solver_reserve", &s));
	s->debug = on != 0;
	return BT_OK;
}

extern "C" int bt_solve_enable_timing(bt_ctx* ctx, int on) {
	SolverState* s;
	BT_TRY(state_of(ctx, &bt_ctx::solver, "bt_solve_enable_timing", "bt_solver_reserve", &s));
	if (on && !s->tstamp.p) { BT_TRY(s->tstamp.alloc(4 * sizeof(long long))); BT_CUDA(cudaMemset(s->tstamp.p, 0, 4 * sizeof(long long))); }
	s->timing = on != 0;
	return BT_OK;
}

// Device time of the LAST bt_solve_run as (prep incl. the tile plan, gap, solve), from %globaltimer stamps the kernels write: prep =
// first prep kernel's start to the tile plan's end, gap = from there to k_solve's start, solve = k_solve's start to its last CTA's end.
// Synchronises the device.
extern "C" int bt_solve_get_timing(bt_ctx* ctx, float* ms3) {
	SolverState* s;
	BT_TRY(state_of(ctx, &bt_ctx::solver, "bt_solve_get_timing", "bt_solver_reserve", &s));
	BT_REQUIRE(s->timing && ms3, BT_ERR_INVALID_ARG, "bt_solve_get_timing: timing not enabled");
	BT_CUDA(cudaDeviceSynchronize());
	long long t[4];
	BT_CUDA(cudaMemcpy(t, s->tstamp.p, sizeof t, cudaMemcpyDeviceToHost));
	for (int k = 0; k < 3; k++) ms3[k] = (float)((double)(t[k + 1] - t[k]) * 1e-6);
	return BT_OK;
}

// Full- and quarter-resolution size and texel geometry of a frame (LossGPU.cu:56-57, CUDACache.cpp:20-24).  The per-call build and the
// frame cache both take it from here: the dense tap rebuilds camera points from these floats, so cached and per-call maps must share them.
static FrameGeom frame_geom(int H, int W, float fx, float fy, float cx, float cy, float image_downscale) {
	FrameGeom g;
	g.W = W; g.H = H; g.w = (int)(W / image_downscale); g.h = (int)(H / image_downscale);
	g.tg.ifx = 1.0f / fx; g.tg.ify = 1.0f / fy; g.tg.icx = -cx / fx; g.tg.icy = -cy / fy;
	g.tg.scaleW = (float)(W - 1) / (float)(g.w - 1); g.tg.scaleH = (float)(H - 1) / (float)(g.h - 1);
	return g;
}

static int launch_prep(bt_ctx* ctx, cudaStream_t stream);
static double us_since(std::chrono::steady_clock::time_point t0) { return std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now() - t0).count(); }

// Every window against what was reserved; F / C = frames / correspondences of the batch.
static int validate_windows(const SolverState* s, int n_windows, const bt_window* windows, const bt_solver_params* params, size_t* F, size_t* C) {
	*F = 0; *C = 0;
	for (int w = 0; w < n_windows; w++) {
		const bt_window& bw = windows[w];
		BT_REQUIRE(bw.n_frames >= 2 && bw.n_frames <= s->lim.max_frames, BT_ERR_CAPACITY, "window %d: n_frames %d outside [2,%d]", w, bw.n_frames, s->lim.max_frames);
		long long nc = bw.n_corr;
		if (bw.corr_dev) {     // device-resident blocks: validate the host-side description
			BT_REQUIRE(bw.n_blocks >= 0 && (bw.n_blocks == 0 || (bw.block_off && bw.block_n && bw.block_i && bw.block_j)), BT_ERR_INVALID_ARG, "window %d: corr_dev given without block arrays", w);
			nc = 0;
			for (int b = 0; b < bw.n_blocks; b++) {
				BT_REQUIRE(bw.block_n[b] >= 0 && bw.block_off[b] >= 0 && (b == 0 || bw.block_off[b] == bw.block_off[b - 1] + bw.block_n[b - 1]), BT_ERR_INVALID_ARG,
				           "window %d: correspondence block %d is not back to back with its predecessor", w, b);
				BT_REQUIRE(bw.block_n[b] == 0 || (bw.block_i[b] < (uint32_t)bw.n_frames && bw.block_j[b] < (uint32_t)bw.n_frames), BT_ERR_INVALID_ARG,
				           "window %d: correspondence block %d references a frame outside [0,%d)", w, b, bw.n_frames);
				nc += bw.block_n[b];
			}
		}
		BT_REQUIRE(nc >= 0 && nc <= s->lim.max_corr, BT_ERR_CAPACITY, "window %d: n_corr %lld > reserved %d", w, nc, s->lim.max_corr);
		BT_REQUIRE(bw.H > 0 && bw.W > 0 && bw.H <= s->lim.H && bw.W <= s->lim.W, BT_ERR_CAPACITY, "window %d: image %dx%d larger than reserved", w, bw.W, bw.H);
		BT_REQUIRE((int)(bw.W / params->image_downscale) >= 2 && (int)(bw.H / params->image_downscale) >= 2, BT_ERR_INVALID_ARG, "window %d: image too small", w);
		BT_REQUIRE(bw.corr_dev || bw.n_corr == 0 || bw.corr, BT_ERR_INVALID_ARG, "window %d: corr is NULL", w);
		BT_REQUIRE(params->w_dense <= 0.f || bw.cache_slots || (bw.depth_dev && bw.normal_dev), BT_ERR_INVALID_ARG, "window %d: depth/normal pointers are NULL and no cache slots given", w);
		*F += bw.n_frames; *C += (size_t)nc;
	}
	return BT_OK;
}

// What the frame preparation needs, with no look at the correspondences: window geometry, where each frame slot's maps live (a cache
// slot or the call's own pointers), poses, the dense pair list with each pair's window and source slot.  *n_pairs = pairs of the batch.
static int fill_frame_tables(SolverState* s, int n_windows, const bt_window* windows, const bt_solver_params* params, const float* poses_in,
                             const StageLayout& L, size_t* n_pairs) {
	const TableBlock<1, 2>& st = s->stage;
	WinDesc* hw = st.host(L.wins);
	const float** hdp = st.host(L.dp); const float4** hnp = st.host(L.np);
	const float4** htex = st.host(L.texp); const float4** hsrc = st.host(L.srcp); const int** hnsrc = st.host(L.nsrcp);
	int* hfw = st.host(L.fw); float* hpose = st.host(L.pose);
	uint2* hpairs = st.host(L.pairs); int* hpwin = st.host(L.pwin); int* hpsrc = st.host(L.psrc);
	const bool dense = params->w_dense > 0.f;
	s->frame_off.assign(n_windows, 0); s->n_frames.assign(n_windows, 0);
	s->any_uncached = false;
	size_t f_off = 0, p_off = 0;
	for (int w = 0; w < n_windows; w++) {
		const bt_window& bw = windows[w];
		const int N = bw.n_frames;
		WinDesc& d = hw[w];
		memset(&d, 0, sizeof d);
		const FrameGeom geom = frame_geom(bw.H, bw.W, bw.fx, bw.fy, bw.cx, bw.cy, params->image_downscale);
		d.n_frames = N; d.H = geom.H; d.W = geom.W; d.w = geom.w; d.h = geom.h; d.tg = geom.tg;
		d.fx = bw.fx * ((float)d.w / (float)bw.W); d.fy = bw.fy * ((float)d.h / (float)bw.H);         // CUDACache.cpp:20-24
		d.cx = bw.cx * ((float)(d.w - 1) / (float)(bw.W - 1)); d.cy = bw.cy * ((float)(d.h - 1) / (float)(bw.H - 1));
		d.compat_flip = bw.compat_flip;
		d.frame_off = (int)f_off; d.pair_off = (int)p_off;
		s->frame_off[w] = (int)f_off; s->n_frames[w] = N;
		for (int f = 0; f < N; f++) {
			const size_t fs = f_off + f;
			if (bw.cache_slots && dense) {     // maps built earlier by bt_frame_cache_store
				const int cs = bw.cache_slots[f];
				BT_REQUIRE(cs >= 0 && cs < s->c_capacity && s->c_meta[cs].valid, BT_ERR_INVALID_ARG, "window %d frame %d: cache slot %d is empty or out of range", w, f, cs);
				const SolverState::CacheMeta& m = s->c_meta[cs];
				BT_REQUIRE(m.H == bw.H && m.W == bw.W && m.fx == bw.fx && m.fy == bw.fy && m.cx == bw.cx && m.cy == bw.cy && m.dmin == params->depth_min && m.dmax == params->depth_max
				               && s->c_downscale == params->image_downscale,
				           BT_ERR_INVALID_ARG, "window %d frame %d: cache slot %d was stored with another image size, K, depth range or downscale", w, f, cs);
				hdp[fs] = nullptr; hnp[fs] = nullptr;
				htex[fs] = s->c_texel.as<float4>() + (size_t)cs * s->c_npix; hsrc[fs] = s->c_src.as<float4>() + (size_t)cs * 2 * s->c_npix;
				hnsrc[fs] = s->c_nsrc.as<int>() + cs;
			} else {
				hdp[fs] = dense ? bw.depth_dev[f] : nullptr; hnp[fs] = dense ? (const float4*)bw.normal_dev[f] : nullptr;
				htex[fs] = s->texel.as<float4>() + fs * (size_t)s->npix_max; hsrc[fs] = s->src.as<float4>() + fs * 2 * (size_t)s->npix_max;
				hnsrc[fs] = nullptr;
				if (dense) s->any_uncached = true;
			}
			hfw[fs] = w;
			memcpy(hpose + fs * 16, poses_in + fs * 16, sizeof(float) * 16);
		}
		int np = 0;
		if (dense) {
			if (bw.dense_pairs) {
				BT_REQUIRE(bw.n_dense_pairs >= 0 && bw.n_dense_pairs <= s->max_pairs, BT_ERR_CAPACITY, "window %d: %d dense pairs > %d", w, bw.n_dense_pairs, s->max_pairs);
				for (int p = 0; p < bw.n_dense_pairs; p++) {
					const uint32_t ti = bw.dense_pairs[2 * p], sj = bw.dense_pairs[2 * p + 1];
					BT_REQUIRE(ti < (uint32_t)N && sj < (uint32_t)N && ti != sj, BT_ERR_INVALID_ARG, "window %d: dense pair %d = (%u,%u) invalid", w, p, ti, sj);
					hpairs[p_off + np++] = make_uint2(ti, sj);
				}
			} else {
				for (int i = 0; i < N; i++) for (int j = 0; j < i; j++) hpairs[p_off + np++] = make_uint2((unsigned)i, (unsigned)j);
			}
		}
		d.n_pairs = np;
		for (int p = 0; p < np; p++) { hpwin[p_off + p] = w; hpsrc[p_off + p] = (int)f_off + (int)hpairs[p_off + p].y; }
		f_off += N; p_off += np;
	}
	*n_pairs = p_off;
	return BT_OK;
}

// How a window's entries reach the device block: through the pinned block (or none to move), in place from page-locked caller memory, from corr_dev
enum class CorrFrom { Staged, InPlace, Device };

// Groups one window's correspondences by (i,j): gi / gj / gs[ng + 1] (starts relative to the window's first entry), *n_valid entries kept,
// and how they reach the device (*src: where they are, unless that is `staged`, the window's slice of the pinned block).  Four input forms:
// blocks on the device; host entries in blocks the caller names; host entries already grouped; anything else.  Issues no CUDA copy.
static int group_window(const bt_window& bw, int w, bt_entryj* staged, int* gi, int* gj, int* gs, std::vector<int>& bin,
                        int* ng_out, int* n_valid_out, CorrFrom* how, const bt_entryj** src) {
	static_assert(offsetof(bt_entryj, imgIdx_i) == 0 && offsetof(bt_entryj, imgIdx_j) == 4, "EntryJ header layout");
	const int N = bw.n_frames;
	int n_valid = 0, ng = 0; bool grouped = true;    // keys (i*N+j) non-decreasing and no invalid entries => groups are runs, the entries stay in their order
	*how = CorrFrom::Staged; *src = nullptr;
	if (bw.corr_dev) {      // every non-empty block is a group
		for (int b = 0; b < bw.n_blocks; b++) {
			if (bw.block_n[b] == 0) continue;
			gi[ng] = (int)bw.block_i[b]; gj[ng] = (int)bw.block_j[b]; gs[ng] = n_valid; ng++;
			n_valid += bw.block_n[b];
		}
		if (n_valid) { *how = CorrFrom::Device; *src = bw.corr_dev + bw.block_off[0]; }      // nothing to copy on the host
	} else if (bw.block_n && bw.n_blocks > 0) {
		// the caller names the blocks (Bundler::optimizeGPU emits the entries pair by pair and hands n_match_per_pair along,
		// /root/reference/src/Bundler.cpp:298-351): only the first entry of every block is read - no pass over the 64 KB of a window
		long long off = 0;
		for (int b = 0; b < bw.n_blocks; b++) {
			const int nb = bw.block_n[b];
			BT_REQUIRE(nb >= 0 && off + nb <= bw.n_corr, BT_ERR_INVALID_ARG, "window %d: correspondence block %d overruns n_corr", w, b);
			if (nb == 0) continue;
			const uint32_t ei = bw.block_i ? bw.block_i[b] : bw.corr[off].imgIdx_i, ej = bw.block_j ? bw.block_j[b] : bw.corr[off].imgIdx_j;
			BT_REQUIRE(ei < (uint32_t)N && ej < (uint32_t)N, BT_ERR_INVALID_ARG, "window %d: correspondence block %d references a frame outside [0,%d)", w, b, N);
			gi[ng] = (int)ei; gj[ng] = (int)ej; gs[ng] = (int)off; ng++;
			off += nb;
		}
		BT_REQUIRE(off == bw.n_corr, BT_ERR_INVALID_ARG, "window %d: the correspondence blocks cover %lld of %d entries", w, off, bw.n_corr);
	} else {
		// one 8-byte compare per entry (imgIdx_i | imgIdx_j << 32, little endian); range and order are only checked where a run ends
		unsigned long long prev_raw = 0ull; long long prev_key = -1; bool have_prev = false;
		for (int c = 0; c < bw.n_corr; c++) {
			unsigned long long raw; memcpy(&raw, &bw.corr[c], sizeof raw);
			if (have_prev && raw == prev_raw) continue;
			const uint32_t ei = (uint32_t)raw, ej = (uint32_t)(raw >> 32);
			if (ei >= (uint32_t)N || ej >= (uint32_t)N) { grouped = false; break; }
			const long long key = (long long)ei * N + ej;
			if (key < prev_key) { grouped = false; break; }
			gi[ng] = (int)ei; gj[ng] = (int)ej; gs[ng] = c; ng++;
			prev_raw = raw; prev_key = key; have_prev = true;
		}
	}
	if (!bw.corr_dev && grouped) {
		n_valid = bw.n_corr;
		if (n_valid) {
			// Caller's buffer page-locked (cudaHostAlloc / cudaHostRegister / bt_host_alloc_pinned)?  Then the copy engine reads it in
			// place - no staging copy - and windows whose buffers follow each other in memory share one transfer.
			cudaPointerAttributes pa;
			if (cudaPointerGetAttributes(&pa, bw.corr) == cudaSuccess && pa.type == cudaMemoryTypeHost) { *how = CorrFrom::InPlace; *src = bw.corr; }
			else memcpy(staged, bw.corr, sizeof(bt_entryj) * (size_t)n_valid);      // the window's entries are still in cache from the scan
		}
	} else if (!bw.corr_dev) {
		// stable counting sort by (i,j) so each pair's entries are contiguous (Bundler::optimizeGPU already emits them that way,
		// /root/reference/src/Bundler.cpp:298-324); invalid entries are dropped
		ng = 0;
		bin.assign((size_t)N * N + 1, 0);
		for (int c = 0; c < bw.n_corr; c++) {
			const bt_entryj& e = bw.corr[c];
			if (e.imgIdx_i == 0xFFFFFFFFu) continue;
			BT_REQUIRE(e.imgIdx_i < (uint32_t)N && e.imgIdx_j < (uint32_t)N, BT_ERR_INVALID_ARG, "window %d: correspondence %d references frame outside [0,%d)", w, c, N);
			bin[(size_t)e.imgIdx_i * N + e.imgIdx_j + 1]++;
			n_valid++;
		}
		for (size_t b = 0; b < (size_t)N * N; b++) {      // counts -> starts; every non-empty bin is a group
			if (bin[b + 1] > 0) { gi[ng] = (int)(b / N); gj[ng] = (int)(b % N); gs[ng] = bin[b]; ng++; }
			bin[b + 1] += bin[b];
		}
		for (int c = 0; c < bw.n_corr; c++) {
			const bt_entryj& e = bw.corr[c];
			if (e.imgIdx_i == 0xFFFFFFFFu) continue;
			staged[bin[(size_t)e.imgIdx_i * N + e.imgIdx_j]++] = e;
		}
	}
	gs[ng] = n_valid;
	// a group that pairs a frame with itself has no counterpart in the moment form of the sparse term (DESIGN.md §4): refused
	for (int g = 0; g < ng; g++) BT_REQUIRE(gi[g] != gj[g], BT_ERR_INVALID_ARG, "window %d: correspondences pair frame %d with itself", w, gi[g]);
	*ng_out = ng; *n_valid_out = n_valid; return BT_OK;
}

// A window's per-frame membership CSR at `mem` (layout: SolveArgs::mem): the groups, then the dense pairs, touching each frame, in increasing index
// order (fixed summation order); returns its length in ints.  *unique_blocks: every unordered frame pair occurs at most once per table.
static size_t window_membership(int N, int ng, int np, const int* gi, const int* gj, const uint2* pairs, int* mem, std::vector<char>& seen, int* unique_blocks) {
	bool uq = true; seen.assign((size_t)N * N, 0);
	for (int g = 0; g < ng && uq; g++) { const int a2 = std::min(gi[g], gj[g]), b2 = std::max(gi[g], gj[g]); if (seen[(size_t)a2 * N + b2]) uq = false; seen[(size_t)a2 * N + b2] = 1; }
	std::fill(seen.begin(), seen.end(), 0);
	for (int p = 0; p < np && uq; p++) { const int a2 = (int)std::min(pairs[p].x, pairs[p].y), b2 = (int)std::max(pairs[p].x, pairs[p].y); if (seen[(size_t)a2 * N + b2]) uq = false; seen[(size_t)a2 * N + b2] = 1; }
	*unique_blocks = uq ? 1 : 0;
	int* fg_start = mem; int* fp_start = fg_start + (N + 1); int* fg_items = fp_start + (N + 1); int* fp_items = fg_items + 2 * ng;
	auto csr = [N](int* start, int* items, int n, auto first, auto second) {      // per frame f: the k with first(k) == f, or (role 1) second(k) == f
		int q = 0;
		for (int f = 0; f < N; f++) {
			start[f] = q;
			for (int k = 0; k < n; k++) {
				if (first(k) == f) items[q++] = k;
				else if (second(k) == f) items[q++] = k | (1 << 16);
			}
		}
		start[N] = q;
	};
	csr(fg_start, fg_items, ng, [gi](int g) { return gi[g]; }, [gj](int g) { return gj[g]; });
	csr(fp_start, fp_items, np, [pairs](int p) { return (int)pairs[p].x; }, [pairs](int p) { return (int)pairs[p].y; });
	return (size_t)(2 * (N + 1) + 2 * ng + 2 * np);
}

// The correspondence uploads of one batch, in order on the copy stream.  Entries staged in the pinned block go up in pieces of >= 256 KB;
// entries in page-locked caller memory are read in place, buffers that follow each other in memory as one transfer; blocks on the device are
// copied device -> device.  The last two leave a hole in the pinned block, so whatever is staged below the hole is flushed first.
struct CorrUpload {
	bt_entryj* dev; const bt_entryj* pinned; cudaStream_t stream;      // entry 0 of the device block and of the pinned block
	size_t sent = 0;                  // entries [0, sent) are uploaded or belong to the pending run
	const bt_entryj* run_src = nullptr; size_t run_dst = 0, run_n = 0;      // pending in-place transfer
	int staged(size_t upto) { return (upto - sent) * sizeof(bt_entryj) >= 256 * 1024 ? flush(upto) : BT_OK; }      // host entries now fill the pinned block up to `upto`
	int in_place(const bt_entryj* src, size_t at, size_t n) {
		BT_TRY(flush(at));
		if (run_n && run_src + run_n == src && run_dst + run_n == at) run_n += n;      // extends the pending run
		else { BT_TRY(send_run()); run_src = src; run_dst = at; run_n = n; }
		sent = at + n; return BT_OK;
	}
	int from_device(const bt_entryj* src, size_t at, size_t n) {
		BT_TRY(flush(at));
		BT_CUDA(cudaMemcpyAsync(dev + at, src, n * sizeof(bt_entryj), cudaMemcpyDeviceToDevice, stream));
		sent = at + n; return BT_OK;
	}
	int finish(size_t upto) { BT_TRY(flush(upto)); return send_run(); }
private:
	int flush(size_t upto) {
		if (upto > sent) BT_CUDA(cudaMemcpyAsync(dev + sent, pinned + sent, (upto - sent) * sizeof(bt_entryj), cudaMemcpyHostToDevice, stream));
		sent = upto; return BT_OK;
	}
	int send_run() {
		if (run_n) BT_CUDA(cudaMemcpyAsync(dev + run_dst, run_src, run_n * sizeof(bt_entryj), cudaMemcpyHostToDevice, stream));
		run_n = 0; return BT_OK;
	}
};

// Staging order (what makes the fused call fast): everything the frame preparation needs (window descriptors, frame
// pointers, poses, pair tables - ~100 KB) is built and uploaded first and, in the fused call, k_prep_frames is launched
// right there; only then are the correspondences (the bulk: 32 B each) grouped and uploaded on a private copy stream,
// overlapping the kernel.  k_solve waits on the last copy's event.
static int stage_impl(bt_ctx* ctx, int n_windows, const bt_window* windows, const bt_solver_params* params,
                      const float* poses_in, void* stream_, bool early_prep) {
	SolverState* s;
	BT_TRY(state_of(ctx, &bt_ctx::solver, "bt_solve_stage", "bt_solver_reserve", &s));
	BT_REQUIRE(windows && params && poses_in, BT_ERR_INVALID_ARG, "bt_solve_stage: NULL argument");
	cudaStream_t stream = (cudaStream_t)stream_;
	BT_REQUIRE(n_windows > 0 && n_windows <= s->lim.max_windows, BT_ERR_CAPACITY, "bt_solve_stage: %d windows > reserved %d", n_windows, s->lim.max_windows);
	BT_REQUIRE(params->num_iter_outer > 0 && params->num_iter_inner > 0 && params->image_downscale == s->lim.image_downscale, BT_ERR_INVALID_ARG,
	           "bt_solve_stage: iteration counts must be positive and image_downscale must equal the reserved value");
	s->staged = false; s->prep_launched = false;
	const auto t_h0 = std::chrono::steady_clock::now();
	size_t F, C, n_pairs;
	BT_TRY(validate_windows(s, n_windows, windows, params, &F, &C));
	// ---- lay out the pinned block (mirrored by one device block) and fill what the frame preparation needs
	const StageLayout L = stage_layout(n_windows, F, C, s->lim.max_frames, (size_t)s->max_groups, (size_t)s->max_pairs);
	BT_TRY(s->stage.begin("bt_solve_stage", L));
	BT_TRY(fill_frame_tables(s, n_windows, windows, params, poses_in, L, &n_pairs));
	s->n_windows = n_windows; s->frames_total = (int)F; s->prm = *params; s->d2max = sqrt_le_max(params->dense_dist_thresh); s->layout = L;
	{   // chunk: aim for >= 4 tiles per SM-resident CTA over the batch, between 256 and 2048 source pixels
		const long long est_px = (long long)n_pairs * (s->npix_max / 8);   // ~12 % valid
		long long c = est_px / ((long long)ctx->sm_count * 2 * 4);
		c = std::max(256LL, std::min(2048LL, c));
		s->chunk = s->force_chunk ? s->force_chunk : (int)((c + 255) / 256 * 256);
	}
	// ---- early upload.  Two device staging blocks, used alternately: every upload of this batch runs on the private copy stream and only waits for
	// the k_solve that last read THIS block (two batches ago), so with the streaming form the 2 MB of batch k+1 cross PCIe while batch k is being solved.
	BT_TRY(s->copy_stream.create());
	if (s->run_pending) { BT_TRY(s->ev_stage_free[s->stage_cur].record(s->run_stream)); s->run_pending = false; }     // behind the runs of the block being left
	s->stage_cur ^= 1;
	if (s->ev_stage_free[s->stage_cur]) BT_CUDA(cudaStreamWaitEvent(s->copy_stream, s->ev_stage_free[s->stage_cur], 0));
	// correspondence blocks produced on the device (bt_match_pairs on the caller's stream) are copied device -> device on the copy stream: order them
	if (std::any_of(windows, windows + n_windows, [](const bt_window& bw) { return bw.corr_dev != nullptr; })) {
		BT_TRY(s->ev_prev.record(stream)); BT_CUDA(cudaStreamWaitEvent(s->copy_stream, s->ev_prev, 0));
	}
	BT_TRY(s->stage.send(0, L.wsp.off, s->copy_stream, s->stage_cur));
	BT_TRY(s->ev_early.record(s->copy_stream));
	BT_CUDA(cudaStreamWaitEvent(stream, s->ev_early, 0));      // the caller's stream (frame prep in the fused call) waits for the early tables only
	s->host_us[0] = us_since(t_h0);
	if (early_prep) BT_TRY(launch_prep(ctx, stream));
	s->host_us[1] = us_since(t_h0) - s->host_us[0];
	// ---- per window (the GPU is already busy in the fused call): group the correspondences, upload them, membership CSR
	const TableBlock<1, 2>& st = s->stage;
	const WinDesc* hw = st.host(L.wins); WinSparse* hws = st.host(L.wsp);
	int* hgi = st.host(L.gi); int* hgj = st.host(L.gj); int* hgs = st.host(L.gs); int* hmem = st.host(L.mem);
	const uint2* hpairs = st.host(L.pairs); bt_entryj* hcorr = st.host(L.corr);
	CorrUpload up{st.dev(L.corr, s->stage_cur), hcorr, s->copy_stream};
	size_t c_off = 0, g_off = 0, m_off = 0, p_off = 0, smem_need = 0, smem_lean = 0;
	std::vector<int> bin; std::vector<char> seen;
	for (int w = 0; w < n_windows; w++) {
		const int N = windows[w].n_frames, np = hw[w].n_pairs;
		int* gi = hgi + g_off; int* gj = hgj + g_off; int* gs = hgs + g_off + w;      // every window's group starts have one extra end entry
		int ng, n_valid; CorrFrom how; const bt_entryj* src;
		BT_TRY(group_window(windows[w], w, hcorr + c_off, gi, gj, gs, bin, &ng, &n_valid, &how, &src));
		if (how == CorrFrom::Device) BT_TRY(up.from_device(src, c_off, (size_t)n_valid));
		else if (how == CorrFrom::InPlace) BT_TRY(up.in_place(src, c_off, (size_t)n_valid));
		WinSparse& ws = hws[w];
		memset(&ws, 0, sizeof ws);
		ws.n_corr = n_valid; ws.n_groups = ng; ws.corr_off = (int)c_off; ws.grp_off = (int)g_off; ws.mem_off = (int)m_off;
		m_off += window_membership(N, ng, np, gi, gj, hpairs + p_off, hmem + m_off, seen, &ws.unique_blocks);
		smem_need = std::max(smem_need, tail_smem_floats(N, np, ng) * sizeof(float));
		smem_lean = std::max(smem_lean, tail_smem_floats(N, np, ng, false) * sizeof(float));
		c_off += n_valid; g_off += ng; p_off += np;
		BT_TRY(up.staged(c_off));
	}
	BT_TRY(up.finish(c_off));
	s->grp_in_smem = smem_need <= kTailSmemMax; if (!s->grp_in_smem) smem_need = smem_lean;
	BT_REQUIRE(smem_need <= kTailSmemMax, BT_ERR_CAPACITY, "bt_solve_stage: window needs %zu bytes of shared memory (> %d KB)", smem_need, (int)(kTailSmemMax / 1024));
	s->smem_bytes = (int)smem_need;
	BT_TRY(s->stage.send(L.wsp.off, L.corr.off, s->copy_stream, s->stage_cur));      // ---- late upload: group tables, CSR, WinSparse
	BT_TRY(s->stage.in_flight(s->copy_stream));
	BT_CUDA(cudaStreamWaitEvent(stream, s->stage.uploaded(), 0));     // everything later on the caller's stream sees the correspondences
	if (s->debug) {
		const int st = 6 * s->lim.max_frames, sp = 6 * (s->lim.max_frames - 1);
		BT_TRY(s->dbgJ.alloc(sizeof(float) * (size_t)st * st * s->lim.max_windows));
		BT_TRY(s->dbgR.alloc(sizeof(float) * (size_t)st * s->lim.max_windows));
		BT_TRY(s->dbgC.alloc(sizeof(float) * (size_t)s->max_pairs * s->lim.max_windows));
		BT_TRY(s->dbgS.alloc(sizeof(float) * (size_t)sp * (sp + 3) * s->lim.max_windows));
	}
	s->staged = true;
	s->host_us[2] = us_since(t_h0) - s->host_us[0] - s->host_us[1];
	return BT_OK;
}

extern "C" int bt_solve_stage(bt_ctx* ctx, int n_windows, const bt_window* windows, const bt_solver_params* params,
                              const float* poses_in, void* stream_) {
	return stage_impl(ctx, n_windows, windows, params, poses_in, stream_, false);
}

static int ensure_occupancy(bt_ctx* ctx) {
	SolverState* s = ctx->solver.get();
	if (s->attr_bytes == 0) {      // the attribute belongs to (function, device), not to the context: set it to the ceiling stage_impl enforces, once,
		s->attr_bytes = (int)kTailSmemMax;   // so that a second context on the same device can never lower what another context's next launch needs
		BT_CUDA(cudaFuncSetAttribute(k_solve<256, BT_SOLVE_MIN_CTAS>, cudaFuncAttributeMaxDynamicSharedMemorySize, s->attr_bytes));
	}
	if (s->occ_smem != s->smem_bytes) {
		int occ_q = 1;
		BT_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ_q, k_solve<256, BT_SOLVE_MIN_CTAS>, 256, s->smem_bytes));
		s->occ = std::max(occ_q, 1); s->occ_smem = s->smem_bytes;
	}
	return BT_OK;
}

// Launches `kern` as the next link of the stream's dependent-launch chain: it may start while the kernel before it on the stream
// finishes, and its chain_wait() orders it behind that kernel (DESIGN §3.4).  Behind a copy or an event wait it starts as a plain launch.
template <typename... KArgs, typename... Args>
static int launch_chained(void (*kern)(KArgs...), dim3 grid, int threads, size_t smem, cudaStream_t stream, Args&&... args) {
	cudaLaunchAttribute attr;
	attr.id = cudaLaunchAttributeProgrammaticStreamSerialization;
	attr.val.programmaticStreamSerializationAllowed = 1;
	cudaLaunchConfig_t cfg = {};
	cfg.gridDim = grid; cfg.blockDim = dim3((unsigned)threads); cfg.dynamicSmemBytes = smem; cfg.stream = stream;
	cfg.attrs = &attr; cfg.numAttrs = 1;
	BT_CUDA(cudaLaunchKernelEx(&cfg, kern, std::forward<Args>(args)...));
	return BT_OK;
}

static SolveArgs make_args(bt_ctx* ctx) {
	SolverState* s = ctx->solver.get();
	SolveArgs a;
	memset(&a, 0, sizeof a);
	const TableBlock<1, 2>& sd = s->stage;
	const int m = s->stage_cur;
	const StageLayout& L = s->layout;
	a.wins = sd.dev(L.wins, m); a.wsp = sd.dev(L.wsp, m); a.n_windows = s->n_windows;
	a.depth_ptr = sd.dev(L.dp, m); a.normal_ptr = sd.dev(L.np, m); a.frame_win = sd.dev(L.fw, m);
	a.texel = s->texel.as<float4>(); a.src = s->src.as<float4>(); a.nsrc = s->nsrc.as<int>(); a.grp_sums = s->grp_sums.as<float>();
	a.texel_tab = sd.dev(L.texp, m); a.src_tab = sd.dev(L.srcp, m); a.nsrc_cached = sd.dev(L.nsrcp, m);
	a.pose_in = sd.dev(L.pose, m); a.x = s->x.as<float>(); a.T = s->T.as<float>(); a.pose_out = s->pose_out.as<float>();
	a.npix_max = s->npix_max;
	a.corr = sd.dev(L.corr, m); a.grp_i = sd.dev(L.gi, m); a.grp_j = sd.dev(L.gj, m); a.grp_start = sd.dev(L.gs, m);
	a.pairs = sd.dev(L.pairs, m); a.pair_win = sd.dev(L.pwin, m); a.pair_src_slot = sd.dev(L.psrc, m); a.mem = sd.dev(L.mem, m);
	a.tiles = s->tiles.as<Tile>(); a.max_tiles = s->max_tiles; a.partial = s->partial.as<float>();
	a.pair_tile0 = s->pair_tile0.as<int>(); a.pair_ntile = s->pair_ntile.as<int>();
	a.n_tiles_total = s->scalars.as<int>(); a.queue = s->scalars.as<int>() + 1; a.n_src_px = (long long*)(s->scalars.as<char>() + 16);
	a.tiles_done = s->tiles_done.as<int>(); a.iter_done = s->iter_done.as<int>();
	a.chunk = s->chunk; a.grp_in_smem = s->grp_in_smem ? 1 : 0; a.prm = s->prm; a.d2max = s->d2max; a.grid_ctas = ctx->sm_count * s->occ;
	if (s->prof_cap > 0) { a.prof = s->prof.as<long long>(); a.prof_cap = s->prof_cap; }
	if (s->timing) a.tstamp = s->tstamp.as<long long>();
	a.with_count = s->any_uncached ? 1 : 0;
	if (s->debug) { a.dbg_JtJ = s->dbgJ.as<float>(); a.dbg_Jtr = s->dbgR.as<float>(); a.dbg_stride = 6 * s->lim.max_frames; a.dbg_cnt = s->dbgC.as<float>(); a.dbg_cnt_stride = s->max_pairs;
	                a.dbg_sys = s->dbgS.as<float>(); a.dbg_sys_stride = 6 * (s->lim.max_frames - 1); }
	return a;
}

static int launch_prep(bt_ctx* ctx, cudaStream_t stream) {
	SolverState* s = ctx->solver.get();
	// make_args again at run time: grid_ctas and grp_in_smem are only final there (in the fused call the tile plan aims at the last batch's occupancy)
	SolveArgs a = make_args(ctx);
	// frames whose maps come from the frame cache need one block each (source count + pose); a batch of cached frames only skips the count kernel
	const dim3 pgrid(s->any_uncached ? (unsigned)((s->npix_max + 1023) / 1024) : 1u, (unsigned)s->frames_total);
	if (s->any_uncached) BT_TRY(launch_chained(k_prep_count, pgrid, 1024, 0, stream, a, s->blk_cnt.as<int>()));
	BT_TRY(launch_chained(k_prep_frames, pgrid, 1024, 0, stream, a, const_cast<WinDesc*>(a.wins), s->scalars.as<int>() + 8, (const int*)s->blk_cnt.as<int>()));
	s->prep_launched = true;
	return BT_OK;
}

extern "C" int bt_solve_run(bt_ctx* ctx, void* stream_) {
	SolverState* s;
	BT_TRY(state_of(ctx, &bt_ctx::solver, "bt_solve_run", "bt_solver_reserve", &s));
	BT_REQUIRE(s->staged, BT_ERR_INVALID_ARG, "bt_solve_run: nothing staged");
	cudaStream_t stream = (cudaStream_t)stream_;
	BT_TRY(ensure_occupancy(ctx));
	SolveArgs a = make_args(ctx);
	if (s->debug) {
		BT_CUDA(cudaMemsetAsync(s->dbgJ.p, 0, s->dbgJ.bytes, stream));
		BT_CUDA(cudaMemsetAsync(s->dbgR.p, 0, s->dbgR.bytes, stream));
		BT_CUDA(cudaMemsetAsync(s->dbgS.p, 0, s->dbgS.bytes, stream));
	}
	if (s->prof_cap > 0) BT_CUDA(cudaMemsetAsync(s->prof.p, 0, 8, stream));
	if (!s->prep_launched) BT_TRY(launch_prep(ctx, stream));
	s->prep_launched = false;       // a second bt_solve_run on the same staged batch prepares again (poses restart from the staged input)
	const int occ = s->occ;
	const int grid = ctx->sm_count * occ;
	BT_TRY(launch_chained(k_solve<256, BT_SOLVE_MIN_CTAS>, dim3((unsigned)grid), 256, (size_t)s->smem_bytes, stream, a));
	s->run_stream = stream; s->run_pending = true;      // (ev_stage_free: see SolverState)
	s->launches = s->any_uncached ? 3 : 2;
	return BT_OK;
}

// Queues, on `stream`, the download of the staged batch's poses and - behind them - the 32 bytes of scalars (tile count first) into `h`.
static int queue_pose_download(SolverState* s, PinnedBuf& h, cudaStream_t stream) {
	const size_t bytes = sizeof(float) * 16 * (size_t)s->frames_total;
	BT_TRY(h.alloc(bytes + 64));
	BT_CUDA(cudaMemcpyAsync(h.p, s->pose_out.p, bytes, cudaMemcpyDeviceToHost, stream));
	BT_CUDA(cudaMemcpyAsync(h.as<char>() + bytes, s->scalars.p, 32, cudaMemcpyDeviceToHost, stream));
	return BT_OK;
}
// Hands out the poses of a completed download, unless the tile plan reported an overflow.
static int take_poses(const PinnedBuf& h, int frames, float* poses_out, const char* who) {
	const size_t bytes = sizeof(float) * 16 * (size_t)frames;
	const int n_tiles_total = *(const int*)(h.as<char>() + bytes);
	BT_REQUIRE(n_tiles_total >= 0, BT_ERR_CAPACITY, "%s: tile list overflow (more dense tiles than reserved)", who);
	memcpy(poses_out, h.p, bytes);
	return BT_OK;
}

extern "C" int bt_solve_fetch(bt_ctx* ctx, float* poses_out, void* stream_) {
	SolverState* s;
	BT_TRY(state_of(ctx, &bt_ctx::solver, "bt_solve_fetch", "bt_solver_reserve", &s));
	BT_REQUIRE(s->staged && poses_out, BT_ERR_INVALID_ARG, "bt_solve_fetch: nothing staged / NULL output");
	BT_TRY(queue_pose_download(s, s->h_poses, (cudaStream_t)stream_));
	BT_CUDA(cudaStreamSynchronize((cudaStream_t)stream_));
	return take_poses(s->h_poses, s->frames_total, poses_out, "bt_solve_fetch");
}

extern "C" int bt_solve_windows(bt_ctx* ctx, int n_windows, const bt_window* windows, const bt_solver_params* params,
                                float* poses_inout, void* stream) {
	const auto t0 = std::chrono::steady_clock::now();
	BT_TRY(stage_impl(ctx, n_windows, windows, params, poses_inout, stream, true));
	const double t1 = us_since(t0);
	BT_TRY(bt_solve_run(ctx, stream));
	const double t2 = us_since(t0);
	const int rc = bt_solve_fetch(ctx, poses_inout, stream);
	SolverState* s = ctx->solver.get();
	s->host_us[3] = t2 - t1; s->host_us[4] = us_since(t0) - t2; s->host_us[5] = us_since(t0);
	return rc;
}

// Streaming form of bt_solve_windows: `begin` stages and launches a batch and queues the download of its poses, `end` waits for the
// OLDEST batch begun and hands its poses out.  Up to two batches may be in flight, so the host side of batch k+1 (tables, grouping,
// uploads, launches) overlaps the GPU side of batch k; everything is ordered on `stream`.
extern "C" int bt_solve_windows_begin(bt_ctx* ctx, int n_windows, const bt_window* windows, const bt_solver_params* params, const float* poses_in, void* stream_) {
	SolverState* s;
	BT_TRY(state_of(ctx, &bt_ctx::solver, "bt_solve_windows_begin", "bt_solver_reserve", &s));
	const int slot = s->pipe_head;
	BT_REQUIRE(!s->pipe_pending[slot], BT_ERR_INVALID_ARG, "bt_solve_windows_begin: two batches are already in flight - call bt_solve_windows_end first");
	BT_TRY(stage_impl(ctx, n_windows, windows, params, poses_in, stream_, true));
	BT_TRY(bt_solve_run(ctx, stream_));
	BT_TRY(queue_pose_download(s, s->h_pipe[slot], (cudaStream_t)stream_));
	BT_TRY(s->ev_pipe[slot].record((cudaStream_t)stream_));
	s->pipe_pending[slot] = true; s->pipe_frames[slot] = s->frames_total; s->pipe_head ^= 1;
	return BT_OK;
}
extern "C" int bt_solve_windows_end(bt_ctx* ctx, float* poses_out) {
	SolverState* s;
	BT_TRY(state_of(ctx, &bt_ctx::solver, "bt_solve_windows_end", "bt_solver_reserve", &s));
	BT_REQUIRE(poses_out, BT_ERR_INVALID_ARG, "bt_solve_windows_end: NULL argument");
	const int slot = s->pipe_tail;
	BT_REQUIRE(s->pipe_pending[slot], BT_ERR_INVALID_ARG, "bt_solve_windows_end: no batch in flight");
	BT_CUDA(cudaEventSynchronize(s->ev_pipe[slot]));
	s->pipe_pending[slot] = false; s->pipe_tail ^= 1;
	return take_poses(s->h_pipe[slot], s->pipe_frames[slot], poses_out, "bt_solve_windows_end");
}

// Host time of the last bt_solve_windows call, microseconds: {window tables + first upload, frame-prep launch, correspondence scan +
// staging + uploads, k_solve launch, pose download + wait for the GPU, whole call}.
extern "C" int bt_solve_get_host_timing(bt_ctx* ctx, double* us6) {
	SolverState* s;
	BT_TRY(state_of(ctx, &bt_ctx::solver, "bt_solve_get_host_timing", "bt_solver_reserve", &s));
	BT_REQUIRE(us6, BT_ERR_INVALID_ARG, "bt_solve_get_host_timing: NULL argument");
	for (int k = 0; k < 6; k++) us6[k] = s->host_us[k];
	return BT_OK;
}

extern "C" int bt_frame_cache_reserve(bt_ctx* ctx, int capacity, int H, int W, float image_downscale) {
	SolverState* s;
	BT_TRY(state_of(ctx, &bt_ctx::solver, "bt_frame_cache_reserve", "bt_solver_reserve", &s));
	BT_REQUIRE(capacity > 0 && H > 0 && W > 0 && image_downscale >= 1.0f, BT_ERR_INVALID_ARG, "bt_frame_cache_reserve: bad arguments");
	const int w = (int)(W / image_downscale), h = (int)(H / image_downscale);
	BT_REQUIRE(w >= 2 && h >= 2, BT_ERR_INVALID_ARG, "bt_frame_cache_reserve: image too small");
	s->c_capacity = 0;
	BT_TRY(s->c_texel.alloc(sizeof(float4) * (size_t)w * h * capacity));
	BT_TRY(s->c_src.alloc(sizeof(float4) * 2 * (size_t)w * h * capacity));
	BT_TRY(s->c_nsrc.alloc(sizeof(int) * (size_t)capacity));
	BT_TRY(s->c_blk.alloc(sizeof(int) * (size_t)capacity * ((w * h + 1023) / 1024)));
	s->c_capacity = capacity; s->c_npix = w * h; s->c_downscale = image_downscale;
	s->c_meta.assign(capacity, SolverState::CacheMeta());
	return BT_OK;
}

extern "C" int bt_frame_cache_store(bt_ctx* ctx, int n_frames, const int32_t* slots, const float* const* depth_dev, const float* const* normal_dev,
                                    int H, int W, float fx, float fy, float cx, float cy, float depth_min, float depth_max, void* stream_) {
	SolverState* s;
	BT_TRY(state_of(ctx, &bt_ctx::solver, "bt_frame_cache_store", "bt_solver_reserve", &s));
	BT_REQUIRE(slots && depth_dev && normal_dev, BT_ERR_INVALID_ARG, "bt_frame_cache_store: NULL argument");
	BT_REQUIRE(s->c_capacity > 0, BT_ERR_INVALID_ARG, "bt_frame_cache_store: call bt_frame_cache_reserve first");
	BT_REQUIRE(n_frames > 0 && n_frames <= s->c_capacity, BT_ERR_CAPACITY, "bt_frame_cache_store: %d frames > capacity %d", n_frames, s->c_capacity);
	const FrameGeom geom = frame_geom(H, W, fx, fy, cx, cy, s->c_downscale);
	BT_REQUIRE(H > 0 && W > 0 && geom.w >= 2 && geom.h >= 2 && geom.w * geom.h <= s->c_npix, BT_ERR_CAPACITY, "bt_frame_cache_store: image %dx%d does not fit the reserved cache", W, H);
	cudaStream_t stream = (cudaStream_t)stream_;
	for (int f = 0; f < n_frames; f++) {
		BT_REQUIRE(slots[f] >= 0 && slots[f] < s->c_capacity, BT_ERR_INVALID_ARG, "bt_frame_cache_store: slot %d out of range [0,%d)", slots[f], s->c_capacity);
		BT_REQUIRE(depth_dev[f] && normal_dev[f], BT_ERR_INVALID_ARG, "bt_frame_cache_store: frame %d has a NULL map", f);
		for (int g = 0; g < f; g++) BT_REQUIRE(slots[g] != slots[f], BT_ERR_INVALID_ARG, "bt_frame_cache_store: slot %d listed twice", slots[f]);
	}
	CacheStoreArgs c;
	memset(&c, 0, sizeof c);
	c.g = geom;
	c.texel = s->c_texel.as<float4>(); c.src = s->c_src.as<float4>(); c.nsrc = s->c_nsrc.as<int>(); c.slot_npix = (size_t)s->c_npix;
	c.dmin = depth_min; c.dmax = depth_max;
	if (n_frames <= kStoreInline) {
		for (int f = 0; f < n_frames; f++) { c.depth_in[f] = depth_dev[f]; c.normal_in[f] = (const float4*)normal_dev[f]; c.slot_in[f] = slots[f]; }
	} else {
		TableLayout L;
		const Slice<const float*> depth = L.add<const float*>(n_frames);
		const Slice<const float4*> normal = L.add<const float4*>(n_frames);
		const Slice<int> slot = L.add<int>(n_frames);
		BT_TRY(s->c_tables.reserve(L.total));
		BT_TRY(s->c_tables.begin("bt_frame_cache_store", L));
		const float** hd = s->c_tables.host(depth); const float4** hn = s->c_tables.host(normal); int* hs = s->c_tables.host(slot);
		for (int f = 0; f < n_frames; f++) { hd[f] = depth_dev[f]; hn[f] = (const float4*)normal_dev[f]; hs[f] = slots[f]; }
		BT_TRY(s->c_tables.send(0, slot.end(), stream));
		BT_TRY(s->c_tables.in_flight(stream));
		c.depth = s->c_tables.dev(depth); c.normal = s->c_tables.dev(normal); c.slots = s->c_tables.dev(slot);
	}
	if (n_frames >= 2 * ctx->sm_count) {      // many frames: one CTA per frame fills the machine (faster than count + build there, DESIGN §9.6)
		k_frame_cache_store<<<n_frames, 1024, 0, stream>>>(c);
		BT_CUDA(cudaGetLastError());
	} else {
		const dim3 grid((unsigned)((geom.w * geom.h + 1023) / 1024), (unsigned)n_frames);
		BT_TRY(launch_chained(k_cache_count, grid, 1024, 0, stream, c, s->c_blk.as<int>()));
		BT_TRY(launch_chained(k_cache_build, grid, 1024, 0, stream, c, (const int*)s->c_blk.as<int>()));
	}
	for (int f = 0; f < n_frames; f++) {
		SolverState::CacheMeta& m = s->c_meta[slots[f]];
		m.valid = true; m.H = H; m.W = W; m.fx = fx; m.fy = fy; m.cx = cx; m.cy = cy; m.dmin = depth_min; m.dmax = depth_max;
	}
	return BT_OK;
}

extern "C" int bt_solve_get_stats(bt_ctx* ctx, bt_solve_stats* out) {
	SolverState* s;
	BT_TRY(state_of(ctx, &bt_ctx::solver, "bt_solve_get_stats", "bt_solver_reserve", &s));
	BT_REQUIRE(out, BT_ERR_INVALID_ARG, "bt_solve_get_stats: NULL argument");
	char h[32];
	BT_CUDA(cudaMemcpy(h, s->scalars.p, 32, cudaMemcpyDeviceToHost));
	out->n_windows = s->n_windows;
	out->n_tiles_total = *(int*)h;
	out->n_kernel_launches = s->launches;
	out->n_src_pixels = *(long long*)(h + 16);
	return BT_OK;
}

extern "C" int bt_solve_enable_profile(bt_ctx* ctx, int max_records) {
	SolverState* s;
	BT_TRY(state_of(ctx, &bt_ctx::solver, "bt_solve_enable_profile", "bt_solver_reserve", &s));
	BT_REQUIRE(max_records >= 0, BT_ERR_INVALID_ARG, "bt_solve_enable_profile: max_records %d < 0", max_records);
	if (max_records > 0) BT_TRY(s->prof.alloc(8 + (size_t)max_records * 96));
	s->prof_cap = max_records;
	return BT_OK;
}
extern "C" int bt_solve_get_profile(bt_ctx* ctx, long long* out, int max_records) {
	SolverState* s;
	BT_TRY(state_of(ctx, &bt_ctx::solver, "bt_solve_get_profile", "bt_solver_reserve", &s));
	BT_REQUIRE(s->prof_cap > 0 && out, BT_ERR_INVALID_ARG, "bt_solve_get_profile: profiling not enabled");
	BT_CUDA(cudaDeviceSynchronize());
	long long n = 0;
	BT_CUDA(cudaMemcpy(&n, s->prof.p, 8, cudaMemcpyDeviceToHost));
	if (n > s->prof_cap) n = s->prof_cap;
	if (n > max_records) n = max_records;
	if (n > 0) BT_CUDA(cudaMemcpy(out, s->prof.as<long long>() + 1, (size_t)n * 96, cudaMemcpyDeviceToHost));
	return (int)n;
}

extern "C" int bt_solve_debug_counts(bt_ctx* ctx, int w, int n_pairs, float* counts_out) {
	SolverState* s;
	BT_TRY(state_of(ctx, &bt_ctx::solver, "bt_solve_debug_counts", "bt_solver_reserve", &s));
	BT_REQUIRE(s->debug && s->staged && counts_out, BT_ERR_INVALID_ARG, "bt_solve_debug_counts: debug not enabled / nothing run");
	BT_REQUIRE(w >= 0 && w < s->n_windows && n_pairs >= 0 && n_pairs <= s->max_pairs, BT_ERR_INVALID_ARG, "bt_solve_debug_counts: bad index");
	BT_CUDA(cudaDeviceSynchronize());
	BT_CUDA(cudaMemcpy(counts_out, s->dbgC.as<float>() + (size_t)w * s->max_pairs, sizeof(float) * n_pairs, cudaMemcpyDeviceToHost));
	return BT_OK;
}

extern "C" int bt_solve_debug_dense(bt_ctx* ctx, int w, float* JtJ_out, float* Jtr_out) {
	SolverState* s;
	BT_TRY(state_of(ctx, &bt_ctx::solver, "bt_solve_debug_dense", "bt_solver_reserve", &s));
	BT_REQUIRE(s->debug && s->staged, BT_ERR_INVALID_ARG, "bt_solve_debug_dense: debug not enabled / nothing run");
	BT_REQUIRE(w >= 0 && w < s->n_windows, BT_ERR_INVALID_ARG, "bt_solve_debug_dense: window %d out of range", w);
	const int st = 6 * s->lim.max_frames, dim = 6 * s->n_frames[w];
	BT_CUDA(cudaDeviceSynchronize());
	if (JtJ_out) BT_CUDA(cudaMemcpy(JtJ_out, s->dbgJ.as<float>() + (size_t)w * st * st, sizeof(float) * dim * dim, cudaMemcpyDeviceToHost));
	if (Jtr_out) BT_CUDA(cudaMemcpy(Jtr_out, s->dbgR.as<float>() + (size_t)w * st, sizeof(float) * dim, cudaMemcpyDeviceToHost));
	return BT_OK;
}

extern "C" int bt_solve_debug_system(bt_ctx* ctx, int w, int n_frames, float* A_out, float* rhs_out, float* minv_out, float* delta_out) {
	SolverState* s;
	BT_TRY(state_of(ctx, &bt_ctx::solver, "bt_solve_debug_system", "bt_solver_reserve", &s));
	BT_REQUIRE(s->debug && s->staged, BT_ERR_INVALID_ARG, "bt_solve_debug_system: debug not enabled / nothing run");
	BT_REQUIRE(w >= 0 && w < s->n_windows, BT_ERR_INVALID_ARG, "bt_solve_debug_system: window %d out of range", w);
	BT_REQUIRE(n_frames == s->n_frames[w], BT_ERR_INVALID_ARG, "bt_solve_debug_system: window %d has %d frames, the outputs are sized for %d", w, s->n_frames[w], n_frames);
	const int st = 6 * (s->lim.max_frames - 1), dim = 6 * (s->n_frames[w] - 1);
	const float* S = s->dbgS.as<float>() + (size_t)w * st * (st + 3);
	BT_CUDA(cudaDeviceSynchronize());
	if (A_out) BT_CUDA(cudaMemcpy(A_out, S, sizeof(float) * dim * dim, cudaMemcpyDeviceToHost));
	if (rhs_out) BT_CUDA(cudaMemcpy(rhs_out, S + (size_t)st * st, sizeof(float) * dim, cudaMemcpyDeviceToHost));
	if (minv_out) BT_CUDA(cudaMemcpy(minv_out, S + (size_t)st * st + st, sizeof(float) * dim, cudaMemcpyDeviceToHost));
	if (delta_out) BT_CUDA(cudaMemcpy(delta_out, S + (size_t)st * st + 2 * st, sizeof(float) * dim, cudaMemcpyDeviceToHost));
	return BT_OK;
}
