// overlay.cu — the tracking overlay of the reference's LOG frames (Bundler::saveNewframeResult, src/Bundler.cpp:379-411): the model voxel-gridded
// as PCL's VoxelGrid does (Utils::downsamplePointCloud, Utils.cpp:134-140), moved under the tracked pose, gridded again at 1 cm, projected and
// stamped onto the frame's colour dimmed outside the object mask (Utils::drawProjectPoints, Utils.cpp:216-226).
//
// VoxelGrid (PCL 1.9 applyFilter, downsample_all_data_, min_points_per_voxel_ = 0), float32 throughout:
//   inv = 1 / leaf; min_p / max_p over the finite points; d_a = (int64)((max_p_a - min_p_a) inv) + 1, and d_x d_y d_z > INT32_MAX returns the
//   input unchanged; min_b_a = (int)floorf(min_p_a inv), div_a = (int)floorf(max_p_a inv) - min_b_a + 1; per point
//   ijk_a = (int)(floorf(p_a inv) - (float)min_b_a), idx = ijk_x + ijk_y div_x + ijk_z div_x div_y (unsigned, as PCL stores it); one point per
//   occupied voxel in ascending idx, the float sum of its points from 0 in INPUT order divided by (float)count (DESIGN.md §3.10, §4).
//
// The grid of many clouds runs in one asynchronous call, without a host synchronisation:
//   - the clouds lie back to back in scratch as float4 (x, y, z, key) and are cut into tiles of kTile points that never straddle two clouds;
//   - per-cloud min / max (ordered-int atomics), then the grid constants and the overflow rule per cloud, then the keys;
//   - a stable LSD radix sort of the keys, 8 bits per pass, segmented by cloud: per pass a tile histogram, one exclusive scan over all
//     (cloud, digit, tile) counts laid out cloud-major, digit-major, and a stable scatter (warp match + per-warp digit counts, warps and rounds
//     in order).  Non-finite points take the key 0xffffffff and sort to their cloud's end; an overflowing cloud has every key 0, so the sort
//     keeps its input order and the emit step copies it;
//   - run heads counted per tile, scanned, and each head sums its run sequentially: the centroid's bits depend on the input order only.
// So the results depend neither on how clouds are batched nor on the grid.
#include <math.h>
#include <limits.h>
#include "bt_common.cuh"
#include "bt_scan.cuh"

namespace bt {

namespace {

constexpr int kThreads = 256;
constexpr int kItems = 8;                          // points per thread per tile (rounds)
constexpr int kTile = kThreads * kItems;           // 2048 points per tile
constexpr int kScanThreads = 1024;
constexpr uint32_t kInvalid = 0xffffffffu;         // the key of a non-finite point
enum { kModeGrid = 0, kModeCopy = 1, kModeEmpty = 2 };

struct Tile { int start, count, t0, nt, cloud, local; };       // local: the tile's first point within its cloud

struct CloudGrid {
	int mn[3], mx[3];                              // ordered-int images of min_p / max_p (atomics)
	int min_b[3];
	uint32_t div_x, div_xy;
	int mode;
};

struct OverlayFrame { float P[12]; };              // ob_in_cam rows 0..2

__device__ __forceinline__ bool finite3(float x, float y, float z) { return isfinite(x) && isfinite(y) && isfinite(z); }

__global__ void k_vox_init(CloudGrid* __restrict__ g, int n_clouds) {
	const int c = blockIdx.x * blockDim.x + threadIdx.x;
	if (c >= n_clouds) return;
	for (int a = 0; a < 3; a++) { g[c].mn[a] = INT_MAX; g[c].mx[a] = INT_MIN; }
}

// per-block min / max of the finite points into the cloud's slot (a tile belongs to one cloud)
__device__ __forceinline__ void minmax_tile(float x, float y, float z, bool valid, CloudGrid* g) {
	__shared__ int s[6];
	if (threadIdx.x < 3) { s[threadIdx.x] = INT_MAX; s[3 + threadIdx.x] = INT_MIN; }
	__syncthreads();
	if (valid && finite3(x, y, z)) {
		const int ox = ordered_key(x), oy = ordered_key(y), oz = ordered_key(z);
		atomicMin(&s[0], ox); atomicMin(&s[1], oy); atomicMin(&s[2], oz);
		atomicMax(&s[3], ox); atomicMax(&s[4], oy); atomicMax(&s[5], oz);
	}
	__syncthreads();
	if (threadIdx.x < 3) {
		if (s[threadIdx.x] != INT_MAX) atomicMin(&g->mn[threadIdx.x], s[threadIdx.x]);
		if (s[3 + threadIdx.x] != INT_MIN) atomicMax(&g->mx[threadIdx.x], s[3 + threadIdx.x]);
	}
}

// bt_voxel_downsample's input: cloud c's float32 x, y, z rows into the scratch
__global__ void __launch_bounds__(kThreads) k_vox_gather(const Tile* __restrict__ tiles, const float* const* __restrict__ src, float4* __restrict__ buf,
                                                         CloudGrid* __restrict__ grid) {
	const Tile tl = tiles[blockIdx.x];
	const float* p = src[tl.cloud];
	for (int r = 0; r < kItems; r++) {
		const int j = r * kThreads + threadIdx.x;
		const bool valid = j < tl.count;
		float x = 0.f, y = 0.f, z = 0.f;
		if (valid) {
			const size_t q = 3 * (size_t)(tl.local + j);
			x = p[q]; y = p[q + 1]; z = p[q + 2];
			buf[tl.start + j] = make_float4(x, y, z, 0.f);
		}
		minmax_tile(x, y, z, valid, grid + tl.cloud);
	}
}

// bt_pose_overlay's input: the model under frame c's ob_in_cam, ((m0 x + m1 y) + m2 z) + m3 per coordinate, each operation rounded on its own
__global__ void __launch_bounds__(kThreads) k_ovl_transform(const Tile* __restrict__ tiles, const float* __restrict__ model, const OverlayFrame* __restrict__ frames,
                                                            float4* __restrict__ buf, CloudGrid* __restrict__ grid) {
	const Tile tl = tiles[blockIdx.x];
	__shared__ float P[12];
	if (threadIdx.x < 12) P[threadIdx.x] = frames[tl.cloud].P[threadIdx.x];
	__syncthreads();
	for (int r = 0; r < kItems; r++) {
		const int j = r * kThreads + threadIdx.x;
		const bool valid = j < tl.count;
		float o[3] = { 0.f, 0.f, 0.f };
		if (valid) {
			const size_t q = 3 * (size_t)(tl.local + j);
			const float x = model[q], y = model[q + 1], z = model[q + 2];
#pragma unroll
			for (int a = 0; a < 3; a++)
				o[a] = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(P[4 * a], x), __fmul_rn(P[4 * a + 1], y)), __fmul_rn(P[4 * a + 2], z)), P[4 * a + 3]);
			buf[tl.start + j] = make_float4(o[0], o[1], o[2], 0.f);
		}
		minmax_tile(o[0], o[1], o[2], valid, grid + tl.cloud);
	}
}

// the grid constants and the overflow rule of every cloud
__global__ void k_vox_grid(CloudGrid* __restrict__ g, int n_clouds, float inv) {
	const int c = blockIdx.x * blockDim.x + threadIdx.x;
	if (c >= n_clouds) return;
	CloudGrid& G = g[c];
	if (G.mn[0] == INT_MAX) { G.mode = kModeEmpty; return; }          // no finite point
	double cells = 1.0;
	int div[3];
	for (int a = 0; a < 3; a++) {
		const float lo = ordered_float(G.mn[a]), hi = ordered_float(G.mx[a]);
		const float span = __fmul_rn(__fsub_rn(hi, lo), inv);
		cells *= (span >= 9.2e18f ? 9.2e18 : (double)((long long)span + 1));
		G.min_b[a] = (int)floorf(__fmul_rn(lo, inv));
		div[a] = (int)floorf(__fmul_rn(hi, inv)) - G.min_b[a] + 1;
	}
	G.mode = cells > (double)INT_MAX ? kModeCopy : kModeGrid;
	G.div_x = (uint32_t)div[0];
	G.div_xy = (uint32_t)div[0] * (uint32_t)div[1];
}

__global__ void __launch_bounds__(kThreads) k_vox_keys(const Tile* __restrict__ tiles, float4* __restrict__ buf, const CloudGrid* __restrict__ grid, float inv) {
	const Tile tl = tiles[blockIdx.x];
	const CloudGrid& G = grid[tl.cloud];
	const int mode = G.mode;
	for (int r = 0; r < kItems; r++) {
		const int j = r * kThreads + threadIdx.x;
		if (j >= tl.count) break;
		float4 e = buf[tl.start + j];
		uint32_t key = 0;
		if (mode == kModeGrid) {
			if (!finite3(e.x, e.y, e.z)) key = kInvalid;
			else {
				const int i = (int)__fsub_rn(floorf(__fmul_rn(e.x, inv)), (float)G.min_b[0]);
				const int k = (int)__fsub_rn(floorf(__fmul_rn(e.y, inv)), (float)G.min_b[1]);
				const int l = (int)__fsub_rn(floorf(__fmul_rn(e.z, inv)), (float)G.min_b[2]);
				key = (uint32_t)i + (uint32_t)k * G.div_x + (uint32_t)l * G.div_xy;
			}
		}
		e.w = __uint_as_float(key);
		buf[tl.start + j] = e;
	}
}

__device__ __forceinline__ uint32_t key_of(const float4& e) { return __float_as_uint(e.w); }

// where (tile, digit) sits in the scan: cloud-major, then digit, then the cloud's tiles in order
__device__ __forceinline__ size_t hist_at(const Tile& tl, int t, int d) { return (size_t)tl.t0 * 256 + (size_t)d * tl.nt + (t - tl.t0); }

__global__ void __launch_bounds__(kThreads) k_vox_hist(const Tile* __restrict__ tiles, const float4* __restrict__ buf, int shift, uint32_t* __restrict__ hist) {
	__shared__ uint32_t s[256];
	const int t = blockIdx.x;
	const Tile tl = tiles[t];
	s[threadIdx.x] = 0;
	__syncthreads();
	for (int r = 0; r < kItems; r++) {
		const int j = r * kThreads + threadIdx.x;
		if (j < tl.count) atomicAdd(&s[(key_of(buf[tl.start + j]) >> shift) & 255], 1u);
	}
	__syncthreads();
	hist[hist_at(tl, t, threadIdx.x)] = s[threadIdx.x];
}

// exclusive scan of n counts in one block; out[n] = the total
__global__ void __launch_bounds__(kScanThreads) k_scan(const uint32_t* __restrict__ in, uint32_t* __restrict__ out, int n) {
	__shared__ uint32_t s_w[kScanThreads / 32];
	const int tid = threadIdx.x;
	const int per = (n + kScanThreads - 1) / kScanThreads;
	const int b = min(n, tid * per), e = min(n, b + per);
	uint32_t sum = 0, total;
	for (int i = b; i < e; i++) sum += in[i];
	uint32_t run = block_excl_scan(sum, s_w, &total);
	for (int i = b; i < e; i++) { const uint32_t c = in[i]; out[i] = run; run += c; }
	if (tid == kScanThreads - 1) out[n] = run;
}

// stable scatter of one tile: rounds in order, warps in order within a round, lanes in order within a warp
__global__ void __launch_bounds__(kThreads) k_vox_scatter(const Tile* __restrict__ tiles, const float4* __restrict__ in, float4* __restrict__ out, int shift,
                                                          const uint32_t* __restrict__ offs) {
	__shared__ uint32_t s_run[256];
	__shared__ uint32_t s_wc[kThreads / 32][256];
	const int t = blockIdx.x, tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
	const Tile tl = tiles[t];
	s_run[tid] = offs[hist_at(tl, t, tid)];
	const unsigned lt = (1u << lane) - 1u;
	for (int r = 0; r < kItems; r++) {
		if (r * kThreads >= tl.count) break;                            // block-uniform
		const int j = r * kThreads + tid;
		const bool valid = j < tl.count;
		for (int k = 0; k < kThreads / 32; k++) s_wc[k][tid] = 0;
		__syncthreads();
		float4 e = make_float4(0.f, 0.f, 0.f, 0.f);
		uint32_t d = 0x100u + lane;                                    // a value no digit has, distinct per lane
		if (valid) { e = in[tl.start + j]; d = (key_of(e) >> shift) & 255; }
		const unsigned peers = __match_any_sync(0xffffffffu, d);
		const int rank = __popc(peers & lt);
		if (valid && rank == 0) s_wc[w][d] = __popc(peers);
		__syncthreads();
		uint32_t run = s_run[tid];
		for (int k = 0; k < kThreads / 32; k++) { const uint32_t c = s_wc[k][tid]; s_wc[k][tid] = run; run += c; }
		s_run[tid] = run;
		__syncthreads();
		if (valid) out[s_wc[w][d] + rank] = e;
		__syncthreads();
	}
}

__device__ __forceinline__ bool is_head(const Tile& tl, const float4* buf, int j) {
	const uint32_t k = key_of(buf[tl.start + j]);
	if (k == kInvalid) return false;
	return tl.local + j == 0 || key_of(buf[tl.start + j - 1]) != k;
}

__global__ void __launch_bounds__(kThreads) k_vox_heads(const Tile* __restrict__ tiles, const float4* __restrict__ buf, const CloudGrid* __restrict__ grid,
                                                        uint32_t* __restrict__ cnt) {
	__shared__ uint32_t s;
	const Tile tl = tiles[blockIdx.x];
	const int mode = grid[tl.cloud].mode;
	if (threadIdx.x == 0) s = 0;
	__syncthreads();
	uint32_t c = 0;
	for (int r = 0; r < kItems; r++) {
		const int j = r * kThreads + threadIdx.x;
		if (j < tl.count) c += mode == kModeCopy ? 1u : (mode == kModeGrid && is_head(tl, buf, j)) ? 1u : 0u;
	}
	for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
	if ((threadIdx.x & 31) == 0) atomicAdd(&s, c);
	__syncthreads();
	if (threadIdx.x == 0) cnt[blockIdx.x] = s;
}

// each run head sums its run in order and writes the centroid at its ordinal; an overflowing cloud is copied as it came in
__global__ void __launch_bounds__(kThreads, 4) k_vox_emit(const Tile* __restrict__ tiles, const float4* __restrict__ buf, const CloudGrid* __restrict__ grid,
                                                       const uint32_t* __restrict__ tscan, float* const* __restrict__ out_tbl, float* __restrict__ out_flat,
                                                       int32_t* __restrict__ n_out) {
	__shared__ uint32_t s_w[kThreads / 32];
	const int t = blockIdx.x, tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
	const Tile tl = tiles[t];
	const int mode = grid[tl.cloud].mode;
	const uint32_t base = tscan[t] - tscan[tl.t0];
	if (tid == 0 && t == tl.t0) n_out[tl.cloud] = (int32_t)(tscan[tl.t0 + tl.nt] - tscan[tl.t0]);
	float* out = out_tbl ? out_tbl[tl.cloud] : out_flat + 3 * (size_t)(tl.start - tl.local);
	const Tile last = tiles[tl.t0 + tl.nt - 1];
	const int end = last.start + last.count;                               // the cloud's end in the scratch
	uint32_t run = base;
	for (int r = 0; r < kItems; r++) {
		if (r * kThreads >= tl.count) break;                              // block-uniform
		const int j = r * kThreads + tid;
		const bool head = j < tl.count && (mode == kModeCopy || (mode == kModeGrid && is_head(tl, buf, j)));
		const unsigned b = __ballot_sync(0xffffffffu, head);
		if (lane == 0) s_w[w] = __popc(b);
		__syncthreads();
		uint32_t before = run;
		for (int k = 0; k < w; k++) before += s_w[k];
		uint32_t total = 0;
		for (int k = 0; k < kThreads / 32; k++) total += s_w[k];
		if (head) {
			const uint32_t o = before + __popc(b & ((1u << lane) - 1u));
			const int q = tl.start + j;
			float4 e = buf[q];
			if (mode == kModeGrid) {
				const uint32_t key = key_of(e);
				float sx = 0.f, sy = 0.f, sz = 0.f;
				int n = 0;
				for (int p = q; p < end; p++) {
					const float4 v = buf[p];
					if (key_of(v) != key) break;
					sx = __fadd_rn(sx, v.x); sy = __fadd_rn(sy, v.y); sz = __fadd_rn(sz, v.z);
					n++;
				}
				const float fn = (float)n;
				e = make_float4(__fdiv_rn(sx, fn), __fdiv_rn(sy, fn), __fdiv_rn(sz, fn), 0.f);
			}
			out[3 * (size_t)o] = e.x; out[3 * (size_t)o + 1] = e.y; out[3 * (size_t)o + 2] = e.z;
		}
		run += total;
		__syncthreads();
	}
}

// viz: the colour, each channel (uint8)(c * 0.2) in double where fg == 0; raw: the colour, 0 where fg == 0
__global__ void k_ovl_pixels(const uint8_t* const* __restrict__ colour, const uint8_t* const* __restrict__ fg, uint8_t* const* __restrict__ viz,
                             uint8_t* const* __restrict__ raw, int hw) {
	const int f = blockIdx.y;
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= hw) return;
	const uint8_t* c = colour[f] + 3 * (size_t)i;
	const bool on = fg[f][i] != 0;
	uint8_t* v = viz[f] + 3 * (size_t)i;
	uint8_t* o = raw ? raw[f] + 3 * (size_t)i : nullptr;
#pragma unroll
	for (int k = 0; k < 3; k++) {
		const uint8_t x = c[k];
		v[k] = on ? x : (uint8_t)__dmul_rn((double)x, 0.2);
		if (o) o[k] = on ? x : 0;
	}
}

// u = roundf(x fx / z + cx), v likewise, in that order; a centre inside the image stamps cv::circle(r = 1, filled): itself and its four
// neighbours, clipped.  Every stamp writes the same bytes, so overlapping stamps need no order.
__global__ void k_ovl_stamp(const float* __restrict__ cent, int stride, const int32_t* __restrict__ n_cent, uint8_t* const* __restrict__ viz, int H, int W,
                            float fx, float fy, float cx, float cy) {
	const int f = blockIdx.y;
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n_cent[f]) return;
	const float* p = cent + 3 * ((size_t)f * stride + i);
	const float x = p[0], y = p[1], z = p[2];
	const float fu = roundf(__fadd_rn(__fdiv_rn(__fmul_rn(x, fx), z), cx));
	const float fv = roundf(__fadd_rn(__fdiv_rn(__fmul_rn(y, fy), z), cy));
	if (!(fu >= 0.f && fu < (float)W && fv >= 0.f && fv < (float)H)) return;     // NaN, infinities and out-of-int values are outside too
	const int u = (int)fu, v = (int)fv;
	uint8_t* img = viz[f];
	const int du[5] = { 0, -1, 1, 0, 0 }, dv[5] = { 0, 0, 0, -1, 1 };
#pragma unroll
	for (int k = 0; k < 5; k++) {
		const int uu = u + du[k], vv = v + dv[k];
		if (uu < 0 || uu >= W || vv < 0 || vv >= H) continue;
		uint8_t* px = img + 3 * ((size_t)vv * W + uu);
		px[0] = 0; px[1] = 255; px[2] = 255;                              // BGR (0, 255, 255)
	}
}

}  // namespace

struct OverlayState {
	bool ready = false;
	int max_pts = 0, max_frames = 0, max_tiles = 0;
	DevBuf a, b, cent, grid, hist, scan, cnt, tscan, nout;
	TableBlock<> tables;                           // tiles, pointer tables and poses of one call
};
void StateDeleter::operator()(OverlayState* s) const { delete s; }

namespace {

// the tiles of clouds of n[0 .. n_clouds) points: how many, and the tile table
int n_tiles_of(const int* n, int n_clouds) {
	int k = 0;
	for (int c = 0; c < n_clouds; c++) k += (n[c] + kTile - 1) / kTile;
	return k;
}
void plan_tiles(const int* n, int n_clouds, Tile* t) {
	int k = 0, start = 0;
	for (int c = 0; c < n_clouds; c++) {
		const int nt = (n[c] + kTile - 1) / kTile;
		for (int j = 0; j < nt; j++) t[k + j] = Tile{ start + j * kTile, min(kTile, n[c] - j * kTile), k, nt, c, j * kTile };
		k += nt;
		start += n[c];
	}
}

// the tables of a bt_voxel_downsample call and of a bt_pose_overlay call
struct DownsampleTables : TableLayout { Slice<Tile> tiles; Slice<const float*> src; Slice<float*> out; };
DownsampleTables downsample_tables(size_t n_tiles, size_t n_clouds) {
	DownsampleTables t;
	t.tiles = t.add<Tile>(n_tiles); t.src = t.add<const float*>(n_clouds); t.out = t.add<float*>(n_clouds);
	return t;
}
struct OverlayTables : TableLayout { Slice<Tile> tiles; Slice<OverlayFrame> frames; Slice<const uint8_t*> colour, fg; Slice<uint8_t*> viz, raw; };
OverlayTables overlay_tables(size_t n_tiles, size_t n_frames) {
	OverlayTables t;
	t.tiles = t.add<Tile>(n_tiles); t.frames = t.add<OverlayFrame>(n_frames);
	t.colour = t.add<const uint8_t*>(n_frames); t.fg = t.add<const uint8_t*>(n_frames); t.viz = t.add<uint8_t*>(n_frames); t.raw = t.add<uint8_t*>(n_frames);
	return t;
}

// the grid of the clouds already in s->a (after the gather / transform and min / max): keys, sort, centroids
int grid_and_emit(OverlayState* s, const Tile* d_tiles, int n_tiles, int n_clouds, float inv, float* const* out_tbl, float* out_flat, int32_t* n_out,
                  cudaStream_t stream) {
	CloudGrid* g = s->grid.as<CloudGrid>();
	k_vox_grid<<<(n_clouds + 127) / 128, 128, 0, stream>>>(g, n_clouds, inv);
	k_vox_keys<<<n_tiles, kThreads, 0, stream>>>(d_tiles, s->a.as<float4>(), g, inv);
	float4* src = s->a.as<float4>();
	float4* dst = s->b.as<float4>();
	for (int pass = 0; pass < 4; pass++) {
		k_vox_hist<<<n_tiles, kThreads, 0, stream>>>(d_tiles, src, 8 * pass, s->hist.as<uint32_t>());
		k_scan<<<1, kScanThreads, 0, stream>>>(s->hist.as<uint32_t>(), s->scan.as<uint32_t>(), 256 * n_tiles);
		k_vox_scatter<<<n_tiles, kThreads, 0, stream>>>(d_tiles, src, dst, 8 * pass, s->scan.as<uint32_t>());
		std::swap(src, dst);
	}
	// four passes: the sorted points are back in s->a
	k_vox_heads<<<n_tiles, kThreads, 0, stream>>>(d_tiles, src, g, s->cnt.as<uint32_t>());
	k_scan<<<1, kScanThreads, 0, stream>>>(s->cnt.as<uint32_t>(), s->tscan.as<uint32_t>(), n_tiles);
	k_vox_emit<<<n_tiles, kThreads, 0, stream>>>(d_tiles, src, g, s->tscan.as<uint32_t>(), out_tbl, out_flat, n_out);
	BT_CUDA(cudaGetLastError());
	return BT_OK;
}

}  // namespace
}  // namespace bt

using namespace bt;

extern "C" int bt_overlay_reserve(bt_ctx* ctx, int max_pts, int max_frames) {
	BT_REQUIRE(ctx, BT_ERR_INVALID_ARG, "bt_overlay_reserve: ctx is NULL");
	BT_REQUIRE(max_pts >= 1 && max_frames >= 1, BT_ERR_INVALID_ARG, "bt_overlay_reserve: max_pts %d / max_frames %d must be >= 1", max_pts, max_frames);
	const long long total = (long long)max_pts * max_frames;
	const long long tiles = total / kTile + max_frames;
	BT_REQUIRE(total <= (1LL << 30), BT_ERR_INVALID_ARG, "bt_overlay_reserve: max_pts x max_frames = %lld > 2^30", total);
	OverlayState* s;
	BT_TRY(take_state(ctx, &bt_ctx::overlay, &s));
	BT_TRY(s->a.alloc(sizeof(float4) * (size_t)total));
	BT_TRY(s->b.alloc(sizeof(float4) * (size_t)total));
	BT_TRY(s->cent.alloc(3 * sizeof(float) * (size_t)total));
	BT_TRY(s->grid.alloc(sizeof(CloudGrid) * (size_t)max_frames));
	BT_TRY(s->hist.alloc(sizeof(uint32_t) * 256 * (size_t)tiles));
	BT_TRY(s->scan.alloc(sizeof(uint32_t) * (256 * (size_t)tiles + 1)));
	BT_TRY(s->cnt.alloc(sizeof(uint32_t) * (size_t)tiles));
	BT_TRY(s->tscan.alloc(sizeof(uint32_t) * ((size_t)tiles + 1)));
	BT_TRY(s->nout.alloc(sizeof(int32_t) * (size_t)max_frames));
	BT_TRY(s->tables.reserve(std::max(downsample_tables(tiles, max_frames).total, overlay_tables(tiles, max_frames).total)));
	s->max_pts = max_pts; s->max_frames = max_frames; s->max_tiles = (int)tiles;
	s->ready = true;
	return BT_OK;
}

extern "C" int bt_voxel_downsample(bt_ctx* ctx, int n_clouds, const float* const* pts_dev, const int* n_pts, float leaf, float* const* out_dev, int32_t* n_out_dev,
                                   void* stream_) {
	BT_REQUIRE(pts_dev && n_pts && out_dev && n_out_dev, BT_ERR_INVALID_ARG, "bt_voxel_downsample: NULL argument");
	BT_REQUIRE(n_clouds >= 1, BT_ERR_INVALID_ARG, "bt_voxel_downsample: n_clouds %d must be >= 1", n_clouds);
	BT_REQUIRE(leaf > 0.f && isfinite(leaf), BT_ERR_INVALID_ARG, "bt_voxel_downsample: leaf must be positive and finite");
	OverlayState* s;
	BT_TRY(state_of(ctx, &bt_ctx::overlay, "bt_voxel_downsample", "bt_overlay_reserve", &s));
	long long total = 0;
	for (int c = 0; c < n_clouds; c++) {
		BT_REQUIRE(n_pts[c] >= 1 && pts_dev[c] && out_dev[c], BT_ERR_INVALID_ARG, "bt_voxel_downsample: cloud %d has %d points or a NULL pointer", c, n_pts[c]);
		total += n_pts[c];
	}
	BT_REQUIRE(n_clouds <= s->max_frames && total <= (long long)s->max_pts * s->max_frames, BT_ERR_CAPACITY,
	           "bt_voxel_downsample: %d clouds / %lld points exceed the reserved %d clouds / %lld points", n_clouds, total, s->max_frames,
	           (long long)s->max_pts * s->max_frames);
	cudaStream_t stream = (cudaStream_t)stream_;
	const int n_tiles = n_tiles_of(n_pts, n_clouds);
	const DownsampleTables t = downsample_tables(n_tiles, n_clouds);
	BT_TRY(s->tables.begin("bt_voxel_downsample", t));
	plan_tiles(n_pts, n_clouds, s->tables.host(t.tiles));
	memcpy(s->tables.host(t.src), pts_dev, sizeof(void*) * n_clouds);
	memcpy(s->tables.host(t.out), out_dev, sizeof(void*) * n_clouds);
	BT_TRY(s->tables.send(0, t.out.end(), stream));
	BT_TRY(s->tables.in_flight(stream));
	const Tile* d_tiles = s->tables.dev(t.tiles);
	const float* const* d_src = s->tables.dev(t.src);
	float* const* d_out = s->tables.dev(t.out);
	k_vox_init<<<(n_clouds + 127) / 128, 128, 0, stream>>>(s->grid.as<CloudGrid>(), n_clouds);
	k_vox_gather<<<n_tiles, kThreads, 0, stream>>>(d_tiles, d_src, s->a.as<float4>(), s->grid.as<CloudGrid>());
	return grid_and_emit(s, d_tiles, n_tiles, n_clouds, 1.0f / leaf, d_out, nullptr, n_out_dev, stream);
}

extern "C" int bt_pose_overlay(bt_ctx* ctx, int n_frames, const float* model_dev, int n_model, const float* cur_in_model, float fx, float fy, float cx, float cy,
                               const uint8_t* const* colour_dev, const uint8_t* const* fg_dev, int H, int W, uint8_t* const* viz_out_dev,
                               uint8_t* const* raw_out_dev, void* stream_) {
	BT_REQUIRE(model_dev && cur_in_model && colour_dev && fg_dev && viz_out_dev, BT_ERR_INVALID_ARG, "bt_pose_overlay: NULL argument");
	BT_REQUIRE(n_frames >= 1 && n_model >= 1 && H >= 1 && W >= 1, BT_ERR_INVALID_ARG, "bt_pose_overlay: n_frames %d / n_model %d / %d x %d must be >= 1",
	           n_frames, n_model, W, H);
	for (int f = 0; f < n_frames; f++)
		BT_REQUIRE(colour_dev[f] && fg_dev[f] && viz_out_dev[f] && (!raw_out_dev || raw_out_dev[f]), BT_ERR_INVALID_ARG, "bt_pose_overlay: frame %d has a NULL image", f);
	OverlayState* s;
	BT_TRY(state_of(ctx, &bt_ctx::overlay, "bt_pose_overlay", "bt_overlay_reserve", &s));
	BT_REQUIRE(n_frames <= s->max_frames && n_model <= s->max_pts, BT_ERR_CAPACITY, "bt_pose_overlay: %d frames / %d model points exceed the reserved %d / %d",
	           n_frames, n_model, s->max_frames, s->max_pts);
	cudaStream_t stream = (cudaStream_t)stream_;
	std::vector<int> n(n_frames, n_model);
	const OverlayTables t = overlay_tables(n_tiles_of(n.data(), n_frames), n_frames);
	BT_TRY(s->tables.begin("bt_pose_overlay", t));
	OverlayFrame* fr = s->tables.host(t.frames);
	for (int f = 0; f < n_frames; f++) {
		float ob[16];
		BT_REQUIRE(inverse4(cur_in_model + 16 * (size_t)f, ob), BT_ERR_INVALID_ARG, "bt_pose_overlay: frame %d's pose is singular", f);
		memcpy(fr[f].P, ob, sizeof fr[f].P);
	}
	memcpy(s->tables.host(t.colour), colour_dev, sizeof(void*) * n_frames);
	memcpy(s->tables.host(t.fg), fg_dev, sizeof(void*) * n_frames);
	memcpy(s->tables.host(t.viz), viz_out_dev, sizeof(void*) * n_frames);
	if (raw_out_dev) memcpy(s->tables.host(t.raw), raw_out_dev, sizeof(void*) * n_frames);
	plan_tiles(n.data(), n_frames, s->tables.host(t.tiles));
	BT_TRY(s->tables.send(0, t.raw.end(), stream));
	BT_TRY(s->tables.in_flight(stream));
	const int n_tiles = (int)t.tiles.n;
	const OverlayFrame* d_fr = s->tables.dev(t.frames);
	const Tile* d_tiles = s->tables.dev(t.tiles);
	k_vox_init<<<(n_frames + 127) / 128, 128, 0, stream>>>(s->grid.as<CloudGrid>(), n_frames);
	k_ovl_transform<<<n_tiles, kThreads, 0, stream>>>(d_tiles, model_dev, d_fr, s->a.as<float4>(), s->grid.as<CloudGrid>());
	int32_t* n_cent = s->nout.as<int32_t>();
	BT_TRY(grid_and_emit(s, d_tiles, n_tiles, n_frames, 1.0f / 0.01f, nullptr, s->cent.as<float>(), n_cent, stream));
	const int hw = H * W;
	k_ovl_pixels<<<dim3((hw + 255) / 256, n_frames), 256, 0, stream>>>(s->tables.dev(t.colour), s->tables.dev(t.fg), s->tables.dev(t.viz),
	                                                                   raw_out_dev ? s->tables.dev(t.raw) : nullptr, hw);
	k_ovl_stamp<<<dim3((n_model + 255) / 256, n_frames), 256, 0, stream>>>(s->cent.as<float>(), n_model, n_cent, s->tables.dev(t.viz), H, W, fx, fy, cx, cy);
	BT_CUDA(cudaGetLastError());
	return BT_OK;
}
