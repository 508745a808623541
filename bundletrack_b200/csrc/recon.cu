// recon.cu — an object model from a tracking run: the keyframes' depth maps fused into a truncated signed distance field (TSDF) in the model
// frame, and its zero surface extracted by marching tetrahedra.  Nothing here is called by the tracking step.
//
// bt_tsdf_fuse, float32, every operation rounded on its own (__fmul_rn / __fadd_rn / __fdiv_rn), so oracle/recon_oracle.py restates it bit for bit:
//   - bounds: every valid pixel (finite depth d > 0) of every frame back-projected, X = ((u - cx) d) / fx, Y = ((v - cy) d) / fy, Z = d, and
//     moved into the model frame ((R0 X + R1 Y) + R2 Z) + t per coordinate; min / max per axis over all of them (ordered-int atomics: min and
//     max do not depend on the order, so the bounds are exact);
//   - the grid: m = ceil(trunc / voxel) + 1 voxels of margin, origin_a = lo_a - m voxel, n_a = ceil((hi_a - lo_a) / voxel) + 1 + 2 m samples;
//     sample (i, j, k) sits at p_a = origin_a + i_a voxel.  Reading the bounds back is the call's one host synchronisation;
//   - integration: one thread per sample, the frames in the order given: q = p - t, c_r = ((R0r q0 + R1r q1) + R2r q2) (c = R^T (p - t)),
//     skip z <= 0; u = floor(x fx / z + cx + 0.5), v likewise, skip outside the image or d <= 0 (masked-out pixels are 0 and never carve);
//     sdf = d - z, skip sdf < -trunc; sum += min(1, sdf / trunc), count += 1.  No atomics: each sample is one thread's sequential sum.
// bt_tsdf_mesh: the zero surface of f = sum / count over the samples with count >= 1; f < 0 is inside.  Every cube is cut into the six
// tetrahedra of its (0,0,0)-(1,1,1) diagonal (Kuhn), so neighbouring cubes share their face diagonals and the surface is closed wherever it is
// observed.  A tet takes part when all four corners are observed.  Every tet edge is one of the 7 directions {x, y, z, xy, xz, yz, xyz} from its
// lower corner, so a vertex is named (sample, direction); a pass marks the edges the crossing tets use, scans give each sample its first vertex
// and face, and an emit pass writes vertices in (sample, direction) order and faces in (cube, tet, triangle) order, wound so that their normals
// point towards f > 0 (free space).  Positions: t = fa / (fa - fb), p = pa + t (pb - pa) per coordinate, from the lower corner a.
#include <math.h>
#include <limits.h>
#include "bt_common.cuh"
#include "bt_scan.cuh"

namespace bt {

namespace {

constexpr int kThreads = 256;
constexpr int kScanItems = 4;                           // samples per thread of a scan block
constexpr int kScanBlock = kThreads * kScanItems;       // 1024 samples per scan block
constexpr int kScanTopThreads = 1024;
constexpr long long kMaxVoxels = 1LL << 27;             // 12 faces per cube stay below 2^31

struct FramePose { float R[9], t[3]; };                 // cam_in_model: row-major rotation, translation

struct Grid {
	int n[3];
	float origin[3];
	float voxel, trunc;
	float fx, fy, cx, cy;
	int H, W;
};

__device__ __forceinline__ float coord(const Grid& g, int a, int i) { return __fadd_rn(g.origin[a], __fmul_rn((float)i, g.voxel)); }

__global__ void k_bounds_init(int* __restrict__ b) {
	if (threadIdx.x < 3) { b[threadIdx.x] = INT_MAX; b[3 + threadIdx.x] = INT_MIN; }
}

// grid (pixel blocks, frames): the min / max of the valid pixels in the model frame
__global__ void __launch_bounds__(kThreads) k_bounds(const float* const* __restrict__ depth, const FramePose* __restrict__ poses, Grid g,
                                                     int* __restrict__ bounds) {
	__shared__ int s[6];
	if (threadIdx.x < 3) { s[threadIdx.x] = INT_MAX; s[3 + threadIdx.x] = INT_MIN; }
	__syncthreads();
	const int f = blockIdx.y;
	const int i = blockIdx.x * kThreads + threadIdx.x;
	if (i < g.H * g.W) {
		const float d = depth[f][i];
		if (d > 0.f && isfinite(d)) {
			const FramePose& P = poses[f];
			const float c[3] = { __fdiv_rn(__fmul_rn(__fsub_rn((float)(i % g.W), g.cx), d), g.fx), __fdiv_rn(__fmul_rn(__fsub_rn((float)(i / g.W), g.cy), d), g.fy), d };
#pragma unroll
			for (int a = 0; a < 3; a++) {
				const float p = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(P.R[3 * a], c[0]), __fmul_rn(P.R[3 * a + 1], c[1])), __fmul_rn(P.R[3 * a + 2], c[2])), P.t[a]);
				atomicMin(&s[a], ordered_key(p));
				atomicMax(&s[3 + a], ordered_key(p));
			}
		}
	}
	__syncthreads();
	if (threadIdx.x < 3) {
		if (s[threadIdx.x] != INT_MAX) atomicMin(&bounds[threadIdx.x], s[threadIdx.x]);
		if (s[3 + threadIdx.x] != INT_MIN) atomicMax(&bounds[3 + threadIdx.x], s[3 + threadIdx.x]);
	}
}

__global__ void __launch_bounds__(kThreads) k_integrate(const float* const* __restrict__ depth, const FramePose* __restrict__ poses, int n_frames, Grid g,
                                                        float* __restrict__ sum_out, int32_t* __restrict__ cnt_out) {
	const long long nv = (long long)g.n[0] * g.n[1] * g.n[2];
	const long long v = (long long)blockIdx.x * kThreads + threadIdx.x;
	if (v >= nv) return;
	const int ix = (int)(v % g.n[0]), iy = (int)((v / g.n[0]) % g.n[1]), iz = (int)(v / ((long long)g.n[0] * g.n[1]));
	const float p[3] = { coord(g, 0, ix), coord(g, 1, iy), coord(g, 2, iz) };
	float sum = 0.f;
	int cnt = 0;
	for (int f = 0; f < n_frames; f++) {
		const FramePose& P = poses[f];
		const float q[3] = { __fsub_rn(p[0], P.t[0]), __fsub_rn(p[1], P.t[1]), __fsub_rn(p[2], P.t[2]) };
		float c[3];
#pragma unroll
		for (int r = 0; r < 3; r++) c[r] = __fadd_rn(__fadd_rn(__fmul_rn(P.R[r], q[0]), __fmul_rn(P.R[3 + r], q[1])), __fmul_rn(P.R[6 + r], q[2]));
		if (!(c[2] > 0.f)) continue;
		const float fu = floorf(__fadd_rn(__fadd_rn(__fdiv_rn(__fmul_rn(c[0], g.fx), c[2]), g.cx), 0.5f));
		const float fv = floorf(__fadd_rn(__fadd_rn(__fdiv_rn(__fmul_rn(c[1], g.fy), c[2]), g.cy), 0.5f));
		if (!(fu >= 0.f && fu < (float)g.W && fv >= 0.f && fv < (float)g.H)) continue;     // NaN and infinities are outside too
		const float d = __ldg(depth[f] + (size_t)(int)fv * g.W + (int)fu);
		if (!(d > 0.f)) continue;
		const float sdf = __fsub_rn(d, c[2]);
		if (sdf < -g.trunc) continue;
		sum = __fadd_rn(sum, fminf(1.f, __fdiv_rn(sdf, g.trunc)));
		cnt++;
	}
	sum_out[v] = sum;
	cnt_out[v] = cnt;
}

// ---- marching tetrahedra
// direction k of a vertex as a corner-offset bitmask (bit 0: +x, bit 1: +y, bit 2: +z), in the order {x, y, z, xy, xz, yz, xyz}, and back
__constant__ uint8_t c_dir_code[7] = { 1, 2, 4, 3, 5, 6, 7 };
__constant__ int8_t c_dir_of_code[8] = { -1, 0, 1, 3, 2, 4, 5, 6 };
// tet t of the cube: the path 0 -> e_a -> e_a + e_b -> 7 for the axis permutation (a, b, c) = kPerm[t], its corners as offset codes listed
// in a positively oriented order (an odd permutation has its middle corners swapped)
__constant__ uint8_t c_tet[6][4] = {
	{ 0, 1, 3, 7 },     // (x, y, z)  even
	{ 0, 5, 1, 7 },     // (x, z, y)  odd
	{ 0, 3, 2, 7 },     // (y, x, z)  odd
	{ 0, 2, 6, 7 },     // (y, z, x)  even
	{ 0, 4, 5, 7 },     // (z, x, y)  even
	{ 0, 6, 4, 7 },     // (z, y, x)  odd
};
// even permutations of the tet's corners that start with the one corner on its own side (1 or 3 inside), and with the two inside ones
__constant__ uint8_t c_odd[4][4] = { { 0, 1, 2, 3 }, { 1, 0, 3, 2 }, { 2, 3, 0, 1 }, { 3, 2, 1, 0 } };
__constant__ uint8_t c_pair[16][4] = {    // by the inside mask of two corners
	{}, {}, {}, { 0, 1, 2, 3 }, {}, { 0, 2, 3, 1 }, { 1, 2, 0, 3 }, {}, {}, { 0, 3, 1, 2 }, { 1, 3, 2, 0 }, {}, { 2, 3, 0, 1 }, {}, {}, {},
};

// the field at a sample: sum / count, or NaN where count = 0
__device__ __forceinline__ float field(const float* __restrict__ sum, const int32_t* __restrict__ cnt, long long v) {
	const int c = cnt[v];
	return c > 0 ? __fdiv_rn(sum[v], (float)c) : __int_as_float(0x7fffffff);
}

struct Cube { float f[8]; long long v0; long long stride[3]; };

__device__ __forceinline__ long long corner_index(const Cube& q, int code) {
	return q.v0 + ((code & 1) ? q.stride[0] : 0) + ((code & 2) ? q.stride[1] : 0) + ((code & 4) ? q.stride[2] : 0);
}
// the (owner sample, direction) of the tet edge between corners of offset codes a and b (one contains the other)
__device__ __forceinline__ void edge_of(const Cube& q, int a, int b, long long* owner, int* dir) {
	const int lo = (a & b) == a ? a : b, hi = lo == a ? b : a;
	*owner = corner_index(q, lo);
	*dir = c_dir_of_code[lo ^ hi];
}

// the triangles of tet t: visit(k, (code_a, code_b) x 3) per triangle; returns their count
template <class F> __device__ __forceinline__ int tet_triangles(const Cube& q, int t, F visit) {
	int code[4], in = 0;
#pragma unroll
	for (int k = 0; k < 4; k++) {
		code[k] = c_tet[t][k];
		const float f = q.f[code[k]];
		if (f != f) return 0;                                                     // a corner not observed
		if (f < 0.f) in |= 1 << k;
	}
	const int n_in = __popc(in);
	if (n_in == 0 || n_in == 4) return 0;
	if (n_in != 2) {
		const int a = __ffs(n_in == 1 ? in : (~in & 15)) - 1;
		const uint8_t* P = c_odd[a];
		const int A = code[P[0]], B = code[P[1]], C = code[P[2]], D = code[P[3]];
		if (n_in == 1) visit(0, A, B, A, C, A, D);
		else visit(0, A, B, A, D, A, C);
		return 1;
	}
	const uint8_t* P = c_pair[in];
	const int A = code[P[0]], B = code[P[1]], C = code[P[2]], D = code[P[3]];
	visit(0, A, C, A, D, B, D);
	visit(1, A, C, B, D, B, C);
	return 2;
}

__device__ __forceinline__ bool load_cube(const Grid& g, const float* __restrict__ sum, const int32_t* __restrict__ cnt, long long v, Cube& q) {
	const int ix = (int)(v % g.n[0]), iy = (int)((v / g.n[0]) % g.n[1]), iz = (int)(v / ((long long)g.n[0] * g.n[1]));
	if (ix >= g.n[0] - 1 || iy >= g.n[1] - 1 || iz >= g.n[2] - 1) return false;
	q.v0 = v; q.stride[0] = 1; q.stride[1] = g.n[0]; q.stride[2] = (long long)g.n[0] * g.n[1];
#pragma unroll
	for (int c = 0; c < 8; c++) q.f[c] = field(sum, cnt, corner_index(q, c));
	return true;
}

// per cube: its triangle count, and the edges its triangles use marked on their owners (OR: the result does not depend on the order)
__global__ void __launch_bounds__(kThreads) k_mt_mark(Grid g, const float* __restrict__ sum, const int32_t* __restrict__ cnt, uint32_t* __restrict__ mask,
                                                      int32_t* __restrict__ ntri) {
	const long long nv = (long long)g.n[0] * g.n[1] * g.n[2];
	const long long v = (long long)blockIdx.x * kThreads + threadIdx.x;
	if (v >= nv) return;
	Cube q;
	int n = 0;
	if (load_cube(g, sum, cnt, v, q)) {
		for (int t = 0; t < 6; t++)
			n += tet_triangles(q, t, [&](int, int a0, int b0, int a1, int b1, int a2, int b2) {
				const int e[3][2] = { { a0, b0 }, { a1, b1 }, { a2, b2 } };
				for (int k = 0; k < 3; k++) {
					long long o;
					int d;
					edge_of(q, e[k][0], e[k][1], &o, &d);
					atomicOr(mask + o, 1u << d);
				}
			});
	}
	ntri[v] = n;
}

// a scan block's vertex and face totals
__global__ void __launch_bounds__(kThreads) k_mt_block_sums(const uint32_t* __restrict__ mask, const int32_t* __restrict__ ntri, long long nv,
                                                            int2* __restrict__ blk) {
	__shared__ int s_v[kThreads / 32], s_f[kThreads / 32];
	const long long base = (long long)blockIdx.x * kScanBlock;
	int cv = 0, cf = 0;
	for (int r = 0; r < kScanItems; r++) {
		const long long v = base + r * kThreads + threadIdx.x;
		if (v < nv) { cv += __popc(mask[v]); cf += ntri[v]; }
	}
	for (int o = 16; o > 0; o >>= 1) { cv += __shfl_xor_sync(0xffffffffu, cv, o); cf += __shfl_xor_sync(0xffffffffu, cf, o); }
	if ((threadIdx.x & 31) == 0) { s_v[threadIdx.x >> 5] = cv; s_f[threadIdx.x >> 5] = cf; }
	__syncthreads();
	if (threadIdx.x == 0) {
		int tv = 0, tf = 0;
		for (int w = 0; w < kThreads / 32; w++) { tv += s_v[w]; tf += s_f[w]; }
		blk[blockIdx.x] = make_int2(tv, tf);
	}
}

// exclusive scan of the block totals in one CTA; blk[n] = the totals
__global__ void __launch_bounds__(kScanTopThreads) k_mt_scan_top(int2* __restrict__ blk, int n) {
	__shared__ int2 s_w[kScanTopThreads / 32];
	const int tid = threadIdx.x;
	const int per = (n + kScanTopThreads - 1) / kScanTopThreads;
	const int b = min(n, tid * per), e = min(n, b + per);
	int2 sum = make_int2(0, 0), total;
	for (int i = b; i < e; i++) { sum.x += blk[i].x; sum.y += blk[i].y; }
	int2 run = block_excl_scan(sum, s_w, &total);
	for (int i = b; i < e; i++) { const int2 c = blk[i]; blk[i] = run; run.x += c.x; run.y += c.y; }
	if (tid == kScanTopThreads - 1) blk[n] = run;
}

// each sample's first vertex and first face: the block's offset plus the exclusive scan within the block (rounds, then warps, then lanes)
__global__ void __launch_bounds__(kThreads) k_mt_offsets(const uint32_t* __restrict__ mask, const int32_t* __restrict__ ntri, long long nv,
                                                         const int2* __restrict__ blk, int32_t* __restrict__ voff, int32_t* __restrict__ foff) {
	__shared__ int s_v[kThreads / 32], s_f[kThreads / 32];
	const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
	const long long base = (long long)blockIdx.x * kScanBlock;
	int2 run = blk[blockIdx.x];
	for (int r = 0; r < kScanItems; r++) {
		const long long v = base + r * kThreads + tid;
		const int cv = v < nv ? __popc(mask[v]) : 0, cf = v < nv ? ntri[v] : 0;
		const int2 x = warp_incl_scan(make_int2(cv, cf));
		const int xv = x.x, xf = x.y;
		if (lane == 31) { s_v[w] = xv; s_f[w] = xf; }
		__syncthreads();
		int bv = run.x, bf = run.y, tv = 0, tf = 0;
		for (int k = 0; k < kThreads / 32; k++) {
			if (k < w) { bv += s_v[k]; bf += s_f[k]; }
			tv += s_v[k]; tf += s_f[k];
		}
		if (v < nv) { voff[v] = bv + xv - cv; foff[v] = bf + xf - cf; }
		run.x += tv; run.y += tf;
		__syncthreads();
	}
}

__global__ void __launch_bounds__(kThreads) k_mt_emit(Grid g, const float* __restrict__ sum, const int32_t* __restrict__ cnt, const uint32_t* __restrict__ mask,
                                                      const int32_t* __restrict__ voff, const int32_t* __restrict__ foff, float* __restrict__ verts,
                                                      int32_t* __restrict__ faces) {
	const long long nv = (long long)g.n[0] * g.n[1] * g.n[2];
	const long long v = (long long)blockIdx.x * kThreads + threadIdx.x;
	if (v >= nv) return;
	const int ix = (int)(v % g.n[0]), iy = (int)((v / g.n[0]) % g.n[1]), iz = (int)(v / ((long long)g.n[0] * g.n[1]));
	const int idx[3] = { ix, iy, iz };
	const uint32_t m = mask[v];
	if (m) {
		const long long stride[3] = { 1, g.n[0], (long long)g.n[0] * g.n[1] };
		const float fa = field(sum, cnt, v);
		int o = voff[v];
		for (int k = 0; k < 7; k++) {
			if (!(m & (1u << k))) continue;
			const int code = c_dir_code[k];
			long long w = v;
			for (int a = 0; a < 3; a++) if (code & (1 << a)) w += stride[a];
			const float t = __fdiv_rn(fa, __fsub_rn(fa, field(sum, cnt, w)));
			for (int a = 0; a < 3; a++) {
				const float pa = coord(g, a, idx[a]), pb = coord(g, a, idx[a] + ((code >> a) & 1));
				verts[3 * (size_t)o + a] = __fadd_rn(pa, __fmul_rn(t, __fsub_rn(pb, pa)));
			}
			o++;
		}
	}
	Cube q;
	if (!load_cube(g, sum, cnt, v, q)) return;
	int fo = foff[v];
	for (int t = 0; t < 6; t++)
		fo += tet_triangles(q, t, [&](int k, int a0, int b0, int a1, int b1, int a2, int b2) {
			const int e[3][2] = { { a0, b0 }, { a1, b1 }, { a2, b2 } };
			for (int c = 0; c < 3; c++) {
				long long ow;
				int d;
				edge_of(q, e[c][0], e[c][1], &ow, &d);
				faces[3 * (size_t)(fo + k) + c] = voff[ow] + __popc(mask[ow] & ((1u << d) - 1u));
			}
		});
}

}  // namespace

struct ReconState {
	bool ready = false;
	int max_frames = 0, H = 0, W = 0, max_vertices = 0, max_faces = 0;
	long long max_voxels = 0;
	bool fused = false;                            // a grid is in sum / cnt
	Grid grid{};
	float bounds[6] = {};
	DevBuf sum, cnt, mask, ntri, voff, foff, blk, bnd;
	PinnedBuf h_read;                              // the bounds, then the mesh's totals, read back
	TableBlock<> tables;                           // the poses and the depth pointer table of one call
};
void StateDeleter::operator()(ReconState* s) const { delete s; }

namespace {
struct FuseTables : TableLayout { Slice<FramePose> poses; Slice<const float*> depth; };
FuseTables fuse_tables(size_t n_frames) {
	FuseTables t;
	t.poses = t.add<FramePose>(n_frames); t.depth = t.add<const float*>(n_frames);
	return t;
}
long long n_scan_blocks(long long nv) { return (nv + kScanBlock - 1) / kScanBlock; }
}  // namespace

}  // namespace bt

using namespace bt;

extern "C" int bt_recon_reserve(bt_ctx* ctx, int max_frames, int H, int W, long long max_voxels, int max_vertices, int max_faces) {
	BT_REQUIRE(ctx, BT_ERR_INVALID_ARG, "bt_recon_reserve: ctx is NULL");
	BT_REQUIRE(max_frames >= 1 && H >= 1 && W >= 1 && max_vertices >= 1 && max_faces >= 1, BT_ERR_INVALID_ARG,
	           "bt_recon_reserve: max_frames %d, %d x %d, max_vertices %d, max_faces %d must be >= 1", max_frames, W, H, max_vertices, max_faces);
	BT_REQUIRE(max_frames <= 65535, BT_ERR_INVALID_ARG, "bt_recon_reserve: max_frames %d exceeds 65535", max_frames);
	BT_REQUIRE(max_voxels >= 8 && max_voxels <= kMaxVoxels, BT_ERR_INVALID_ARG, "bt_recon_reserve: max_voxels %lld must be in 8..%lld", max_voxels, kMaxVoxels);
	BT_REQUIRE((long long)H * W <= INT_MAX, BT_ERR_INVALID_ARG, "bt_recon_reserve: %d x %d pixels exceed 2^31 - 1", W, H);
	ReconState* s;
	BT_TRY(take_state(ctx, &bt_ctx::recon, &s));
	s->fused = false;
	const size_t nv = (size_t)max_voxels;
	BT_TRY(s->sum.alloc(sizeof(float) * nv));
	BT_TRY(s->cnt.alloc(sizeof(int32_t) * nv));
	BT_TRY(s->mask.alloc(sizeof(uint32_t) * nv));
	BT_TRY(s->ntri.alloc(sizeof(int32_t) * nv));
	BT_TRY(s->voff.alloc(sizeof(int32_t) * nv));
	BT_TRY(s->foff.alloc(sizeof(int32_t) * nv));
	BT_TRY(s->blk.alloc(sizeof(int2) * ((size_t)n_scan_blocks(max_voxels) + 1)));
	BT_TRY(s->tables.reserve(fuse_tables(max_frames).total));
	BT_TRY(s->bnd.alloc(6 * sizeof(int)));
	BT_TRY(s->h_read.alloc(6 * sizeof(int)));
	s->max_frames = max_frames; s->H = H; s->W = W; s->max_voxels = max_voxels; s->max_vertices = max_vertices; s->max_faces = max_faces;
	s->ready = true;
	return BT_OK;
}

extern "C" int bt_tsdf_fuse(bt_ctx* ctx, int n_frames, const float* const* depth_dev, const float* cam_in_model, float fx, float fy, float cx, float cy,
                            int H, int W, const bt_tsdf_params* p, void* stream_) {
	BT_REQUIRE(depth_dev && cam_in_model && p, BT_ERR_INVALID_ARG, "bt_tsdf_fuse: NULL argument");
	BT_REQUIRE(n_frames >= 1 && H >= 1 && W >= 1, BT_ERR_INVALID_ARG, "bt_tsdf_fuse: n_frames %d / %d x %d must be >= 1", n_frames, W, H);
	BT_REQUIRE(p->voxel > 0.f && isfinite(p->voxel) && p->trunc > 0.f && isfinite(p->trunc), BT_ERR_INVALID_ARG,
	           "bt_tsdf_fuse: voxel %g and trunc %g must be positive and finite", p->voxel, p->trunc);
	BT_REQUIRE(isfinite(fx) && isfinite(fy) && isfinite(cx) && isfinite(cy) && fx != 0.f && fy != 0.f, BT_ERR_INVALID_ARG,
	           "bt_tsdf_fuse: the intrinsics must be finite, fx and fy non-zero");
	for (int f = 0; f < n_frames; f++) {
		BT_REQUIRE(depth_dev[f], BT_ERR_INVALID_ARG, "bt_tsdf_fuse: frame %d's depth is NULL", f);
		for (int k = 0; k < 16; k++)
			BT_REQUIRE(isfinite(cam_in_model[16 * (size_t)f + k]), BT_ERR_INVALID_ARG, "bt_tsdf_fuse: frame %d's pose has a non-finite element", f);
	}
	ReconState* s;
	BT_TRY(state_of(ctx, &bt_ctx::recon, "bt_tsdf_fuse", "bt_recon_reserve", &s));
	BT_REQUIRE(n_frames <= s->max_frames && H <= s->H && W <= s->W, BT_ERR_CAPACITY, "bt_tsdf_fuse: %d frames of %d x %d exceed the reserved %d frames of %d x %d",
	           n_frames, W, H, s->max_frames, s->W, s->H);
	cudaStream_t stream = (cudaStream_t)stream_;
	const FuseTables t = fuse_tables(n_frames);
	BT_TRY(s->tables.begin("bt_tsdf_fuse", t));
	FramePose* fp = s->tables.host(t.poses);
	for (int f = 0; f < n_frames; f++) {
		const float* P = cam_in_model + 16 * (size_t)f;
		for (int r = 0; r < 3; r++) {
			for (int c = 0; c < 3; c++) fp[f].R[3 * r + c] = P[4 * r + c];
			fp[f].t[r] = P[4 * r + 3];
		}
	}
	memcpy(s->tables.host(t.depth), depth_dev, sizeof(void*) * n_frames);
	BT_TRY(s->tables.send(0, t.depth.end(), stream));
	BT_TRY(s->tables.in_flight(stream));
	const FramePose* d_pose = s->tables.dev(t.poses);
	const float* const* d_depth = s->tables.dev(t.depth);
	Grid g{};
	g.voxel = p->voxel; g.trunc = p->trunc;
	g.fx = fx; g.fy = fy; g.cx = cx; g.cy = cy; g.H = H; g.W = W;
	int* bnd = s->bnd.as<int>();
	k_bounds_init<<<1, 32, 0, stream>>>(bnd);
	k_bounds<<<dim3((H * W + kThreads - 1) / kThreads, n_frames), kThreads, 0, stream>>>(d_depth, d_pose, g, bnd);
	BT_CUDA(cudaGetLastError());
	int* hb = s->h_read.as<int>();
	BT_CUDA(cudaMemcpyAsync(hb, bnd, 6 * sizeof(int), cudaMemcpyDeviceToHost, stream));
	BT_CUDA(cudaStreamSynchronize(stream));                 // the call's one synchronisation: the grid's size decides what runs next
	BT_REQUIRE(hb[0] != INT_MAX, BT_ERR_INVALID_ARG, "bt_tsdf_fuse: no frame has a valid depth pixel");
	float lo[3], hi[3];
	for (int a = 0; a < 3; a++) { lo[a] = ordered_float(hb[a]); hi[a] = ordered_float(hb[3 + a]); }
	// float32 on the host, one rounding per operation (oracle/recon_oracle.py: grid)
	const int m = (int)ceilf(p->trunc / p->voxel) + 1;
	long long n[3], total = 1;
	bool fits = true;
	for (int a = 0; a < 3; a++) {
		const float span = ceilf((hi[a] - lo[a]) / p->voxel);
		fits = fits && span < 1e9f;
		n[a] = fits ? (long long)span + 1 + 2LL * m : 0;
		total = fits && total <= kMaxVoxels ? total * n[a] : kMaxVoxels + 1;
	}
	BT_REQUIRE(fits && total <= s->max_voxels, BT_ERR_CAPACITY, "bt_tsdf_fuse: a grid of %lld x %lld x %lld samples (bounds [%g, %g] x [%g, %g] x [%g, %g], voxel %g) "
	           "exceeds the reserved %lld", n[0], n[1], n[2], lo[0], hi[0], lo[1], hi[1], lo[2], hi[2], p->voxel, s->max_voxels);
	for (int a = 0; a < 3; a++) {
		g.n[a] = (int)n[a];
		g.origin[a] = lo[a] - (float)m * p->voxel;
		s->bounds[a] = lo[a]; s->bounds[3 + a] = hi[a];
	}
	k_integrate<<<(unsigned)((total + kThreads - 1) / kThreads), kThreads, 0, stream>>>(d_depth, d_pose, n_frames, g, s->sum.as<float>(), s->cnt.as<int32_t>());
	BT_CUDA(cudaGetLastError());
	s->grid = g;
	s->fused = true;
	return BT_OK;
}

extern "C" int bt_tsdf_grid(bt_ctx* ctx, int* dims, float* origin, float* bounds, const float** sum_dev, const int32_t** count_dev) {
	ReconState* s;
	BT_TRY(state_of(ctx, &bt_ctx::recon, "bt_tsdf_grid", "bt_recon_reserve", &s));
	BT_REQUIRE(s->fused, BT_ERR_INVALID_ARG, "bt_tsdf_grid: no grid: call bt_tsdf_fuse (successfully) first");
	for (int a = 0; a < 3; a++) {
		if (dims) dims[a] = s->grid.n[a];
		if (origin) origin[a] = s->grid.origin[a];
	}
	if (bounds) memcpy(bounds, s->bounds, sizeof s->bounds);
	if (sum_dev) *sum_dev = s->sum.as<float>();
	if (count_dev) *count_dev = s->cnt.as<int32_t>();
	return BT_OK;
}

extern "C" int bt_tsdf_mesh(bt_ctx* ctx, float* verts_dev, int32_t* faces_dev, int* n_verts, int* n_faces, void* stream_) {
	BT_REQUIRE(verts_dev && faces_dev && n_verts && n_faces, BT_ERR_INVALID_ARG, "bt_tsdf_mesh: NULL argument");
	ReconState* s;
	BT_TRY(state_of(ctx, &bt_ctx::recon, "bt_tsdf_mesh", "bt_recon_reserve", &s));
	BT_REQUIRE(s->fused, BT_ERR_INVALID_ARG, "bt_tsdf_mesh: no grid: call bt_tsdf_fuse (successfully) first");
	cudaStream_t stream = (cudaStream_t)stream_;
	const Grid& g = s->grid;
	const long long nv = (long long)g.n[0] * g.n[1] * g.n[2];
	const unsigned blocks = (unsigned)((nv + kThreads - 1) / kThreads);
	const int nb = (int)n_scan_blocks(nv);
	uint32_t* mask = s->mask.as<uint32_t>();
	int32_t* ntri = s->ntri.as<int32_t>();
	int2* blk = s->blk.as<int2>();
	BT_CUDA(cudaMemsetAsync(mask, 0, sizeof(uint32_t) * (size_t)nv, stream));
	k_mt_mark<<<blocks, kThreads, 0, stream>>>(g, s->sum.as<float>(), s->cnt.as<int32_t>(), mask, ntri);
	k_mt_block_sums<<<nb, kThreads, 0, stream>>>(mask, ntri, nv, blk);
	k_mt_scan_top<<<1, kScanTopThreads, 0, stream>>>(blk, nb);
	k_mt_offsets<<<nb, kThreads, 0, stream>>>(mask, ntri, nv, blk, s->voff.as<int32_t>(), s->foff.as<int32_t>());
	BT_CUDA(cudaGetLastError());
	int* ht = s->h_read.as<int>();
	BT_CUDA(cudaMemcpyAsync(ht, blk + nb, sizeof(int2), cudaMemcpyDeviceToHost, stream));
	BT_CUDA(cudaStreamSynchronize(stream));                 // the counts decide whether the outputs have room
	*n_verts = ht[0];
	*n_faces = ht[1];
	BT_REQUIRE(ht[0] <= s->max_vertices && ht[1] <= s->max_faces, BT_ERR_CAPACITY, "bt_tsdf_mesh: the mesh has %d vertices and %d faces, the reserved "
	           "%d / %d", ht[0], ht[1], s->max_vertices, s->max_faces);
	k_mt_emit<<<blocks, kThreads, 0, stream>>>(g, s->sum.as<float>(), s->cnt.as<int32_t>(), mask, s->voff.as<int32_t>(), s->foff.as<int32_t>(), verts_dev, faces_dev);
	BT_CUDA(cudaGetLastError());
	return BT_OK;
}
