// segment.cu — the object mask on the device (reference src/Frame.cpp:267-313, src/FeatureManager.cpp:813-873):
//   largest-hull mode (NOCS): the 8-connected components of mask != 0, the largest one (ties: the component whose first pixel in
//     row-major order comes first), its convex hull and cv::fillConvexPoly of that hull -> a 0/1 map the masked front end dilates;
//   the LF-Net request: the masked colour cropped to the ROI, padded to a square and resized to 400 x 400 (cv::resize, INTER_LINEAR).
// Everything is integer arithmetic (the resize's coefficients come from the same double -> float expressions as OpenCV's, with no
// contraction), so the results do not depend on scheduling.  oracle/segment_oracle.py is the CPU statement of the same rules.
#include "bt_common.cuh"

namespace bt {

static constexpr int SEG_THREADS = 256, HULL_THREADS = 1024;

// ---- connected components: lock-free union-find over the frame's label map (label = row-major index, -1 = background).  A root
// only ever hooks under a smaller index, so every root is its component's first pixel in row-major order.
__global__ void __launch_bounds__(SEG_THREADS) k_ccl_init(const uint8_t* const* mask, int32_t* label, int32_t* count, unsigned long long* best, int HW) {
	const int f = blockIdx.y, p = blockIdx.x * SEG_THREADS + threadIdx.x;
	if (p == 0) best[f] = 0ull;
	if (p >= HW) return;
	label[(size_t)f * HW + p] = mask[f][p] ? p : -1;
	count[(size_t)f * HW + p] = 0;
}

__device__ __forceinline__ int uf_find(const int32_t* L, int x) {
	int p;
	while ((p = __ldcg(L + x)) != x) x = p;       // L2 reads: other CTAs hook roots while this kernel runs
	return x;
}
__device__ __forceinline__ void uf_unite(int32_t* L, int a, int b) {
	for (;;) {
		a = uf_find(L, a); b = uf_find(L, b);
		if (a == b) return;
		if (a > b) { const int t = a; a = b; b = t; }
		const int old = atomicMin(L + b, a);
		if (old == b) return;                     // b was a root and now hangs under a
		b = old;                                  // b was hooked elsewhere meanwhile: unite a with b's new parent
	}
}

// 8-connectivity from the four neighbours earlier in raster order (W, NW, N, NE).  By induction on that order every pixel ends up
// joined to each foreground one of its four: when N is foreground, NW is N's W, N is NE's W and N is W's NE, so joining N covers all
// four; otherwise, when W is foreground, NW is W's N.
__global__ void __launch_bounds__(SEG_THREADS) k_ccl_merge(const uint8_t* const* mask, int32_t* label, int H, int W) {
	const int f = blockIdx.z, x = blockIdx.x * 32 + threadIdx.x, y = blockIdx.y * 8 + threadIdx.y;
	if (x >= W || y >= H) return;
	const uint8_t* m = mask[f];
	const int p = y * W + x;
	if (!m[p]) return;
	int32_t* L = label + (size_t)f * H * W;
	if (y > 0 && m[p - W]) { uf_unite(L, p, p - W); return; }
	if (x > 0 && m[p - 1]) uf_unite(L, p, p - 1);
	else if (y > 0 && x > 0 && m[p - W - 1]) uf_unite(L, p, p - W - 1);
	if (y > 0 && x < W - 1 && m[p - W + 1]) uf_unite(L, p, p - W + 1);
}

// Every pixel points at its root; pixels per root, one atomic per (warp, root).
__global__ void __launch_bounds__(SEG_THREADS) k_ccl_flatten(int32_t* label, int32_t* count, int HW) {
	const int f = blockIdx.y, p = blockIdx.x * SEG_THREADS + threadIdx.x;
	int32_t* L = label + (size_t)f * HW;
	int r = -1;
	if (p < HW) {
		const int l = L[p];
		if (l >= 0) { r = uf_find(L, l); if (r != l) L[p] = r; }
	}
	const unsigned act = __ballot_sync(0xffffffffu, r >= 0);
	if (r >= 0) {
		const unsigned peers = __match_any_sync(act, r);
		if ((int)(threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(count + (size_t)f * HW + r, __popc(peers));
	}
}

// The winner per frame: the largest count, then the smallest root (key = count << 32 | ~root).
__global__ void __launch_bounds__(SEG_THREADS) k_ccl_best(const int32_t* label, const int32_t* count, unsigned long long* best, int HW) {
	const int f = blockIdx.y, p = blockIdx.x * SEG_THREADS + threadIdx.x;
	if (p >= HW || label[(size_t)f * HW + p] != p) return;
	atomicMax(best + f, ((unsigned long long)(unsigned)count[(size_t)f * HW + p] << 32) | (unsigned)~p);
}

__device__ __forceinline__ long long cross2(int2 o, int2 a, int2 b) {
	return (long long)(a.x - o.x) * (b.y - o.y) - (long long)(a.y - o.y) * (b.x - o.x);
}

// cv::line(LINE_8) between two points inside the image; the LineIterator runs left to right, so the pixel set is the same either way.
__device__ void line8(uint8_t* img, int W, int2 p0, int2 p1) {
	if (p1.x < p0.x) { const int2 t = p0; p0 = p1; p1 = t; }
	const int dx = p1.x - p0.x, sy = p1.y < p0.y ? -1 : 1, dy = abs(p1.y - p0.y);
	const bool vert = dy > dx;
	const int major = vert ? dy : dx, minor = vert ? dx : dy;
	int err = major - 2 * minor, x = p0.x, y = p0.y;
	for (int i = 0; i <= major; i++) {
		img[(size_t)y * W + x] = 1;
		const bool step = err < 0;
		err += -2 * minor + (step ? 2 * major : 0);
		if (vert) { y += sy; x += step; } else { x++; y += step ? sy : 0; }
	}
}

// One CTA per frame: per-row extreme columns of the winning component (their hull is the hull of all its pixels), the monotone-chain
// hull without collinear points, then cv::fillConvexPoly(shift 0, LINE_8): the scanline spans of its 16.16 fixed-point edge walk
// plus the Bresenham outline of every edge.  Writes the 0/1 map (all zero without foreground).
__global__ void __launch_bounds__(HULL_THREADS) k_hull_fill(const int32_t* label, const unsigned long long* best, uint8_t* fill, int H, int W) {
	extern __shared__ int hs[];
	int* rmin = hs;                       // [H] per-row min column, later the span's left end
	int* rmax = hs + H;                   // [H] per-row max column, later the span's right end
	int2* P = reinterpret_cast<int2*>(hs + 2 * H);   // [2H] points, (y, x)-sorted
	int2* V = P + 2 * H;                  // [4H] monotone-chain stack, then the hull
	__shared__ int s_nh, s_y0, s_y1;
	const int f = blockIdx.x, HW = H * W;
	const int32_t* L = label + (size_t)f * HW;
	uint8_t* out = fill + (size_t)f * HW;
	const unsigned long long key = best[f];
	if (key == 0ull) {
		for (int p = threadIdx.x; p < HW; p += HULL_THREADS) out[p] = 0;
		return;
	}
	const int root = (int)~(unsigned)(key & 0xffffffffull);
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	for (int y = warp; y < H; y += HULL_THREADS / 32) {
		int mn = 0x7fffffff, mx = -1;
		for (int x = lane; x < W; x += 32)
			if (L[(size_t)y * W + x] == root) { mn = min(mn, x); mx = max(mx, x); }
		mn = __reduce_min_sync(0xffffffffu, mn); mx = __reduce_max_sync(0xffffffffu, mx);
		if (lane == 0) { rmin[y] = mn; rmax[y] = mx; }
	}
	__syncthreads();
	if (threadIdx.x == 0) {
		int np = 0;
		for (int y = 0; y < H; y++)
			if (rmax[y] >= 0) { P[np++] = make_int2(rmin[y], y); if (rmax[y] != rmin[y]) P[np++] = make_int2(rmax[y], y); }
		// Andrew's monotone chain on the (y, x) order; cross <= 0 pops collinear points
		int k = 0;
		for (int i = 0; i < np; i++) { while (k >= 2 && cross2(V[k - 2], V[k - 1], P[i]) <= 0) k--; V[k++] = P[i]; }
		for (int i = np - 2, t = k + 1; i >= 0; i--) { while (k >= t && cross2(V[k - 2], V[k - 1], P[i]) <= 0) k--; V[k++] = P[i]; }
		const int n = np == 1 ? 1 : k - 1;
		// fillConvexPoly's scanline walk (drawing.cpp FillConvexPoly, shift 0): spans into rmin / rmax
		int ymin = V[0].y, ymax = V[0].y, imin = 0;
		for (int i = 1; i < n; i++) { if (V[i].y < ymin) { ymin = V[i].y; imin = i; } ymax = max(ymax, V[i].y); }
		ymax = min(ymax, H - 1);
		for (int y = ymin; y <= ymax; y++) { rmin[y] = 1; rmax[y] = 0; }
		if (n >= 3) {
			int e_idx[2] = {imin, imin}, e_di[2] = {1, n - 1}, e_ye[2] = {ymin, ymin};
			long long e_x[2] = {-65536, -65536}, e_dx[2] = {0, 0};
			int edges = n, y = ymin;
			for (;;) {
				for (int i = 0; i < 2; i++) {
					if (y < e_ye[i]) continue;
					int idx0 = e_idx[i], idx = idx0 + e_di[i];
					if (idx >= n) idx -= n;
					while (edges-- > 0) {
						const int ty = V[idx].y;
						if (ty > y) {
							const long long xs = (long long)V[idx0].x << 16, xe = (long long)V[idx].x << 16;
							e_ye[i] = ty; e_dx[i] = ((xe - xs) * 2 + (ty - y)) / (2 * (long long)(ty - y)); e_x[i] = xs; e_idx[i] = idx;
							break;
						}
						idx0 = idx; idx += e_di[i];
						if (idx >= n) idx -= n;
					}
				}
				if (edges < 0) break;
				const int l = e_x[0] > e_x[1] ? 1 : 0;
				const int x1 = (int)((e_x[l] + 32768) >> 16), x2 = (int)((e_x[1 - l] + 32768) >> 16);
				if (x2 >= 0 && x1 < W) { rmin[y] = max(x1, 0); rmax[y] = min(x2, W - 1); }
				e_x[0] += e_dx[0]; e_x[1] += e_dx[1];
				if (++y > ymax) break;
			}
		}
		s_nh = n; s_y0 = ymin; s_y1 = ymax;
	}
	__syncthreads();
	const int y0 = s_y0, y1 = s_y1, nh = s_nh;
	for (int p = threadIdx.x; p < HW; p += HULL_THREADS) {
		const int y = p / W, x = p - y * W;
		out[p] = (y >= y0 && y <= y1 && x >= rmin[y] && x <= rmax[y]) ? 1 : 0;
	}
	__syncthreads();
	for (int i = threadIdx.x; i < nh; i += HULL_THREADS) line8(out, W, V[i == 0 ? nh - 1 : i - 1], V[i]);
}

size_t hull_fill_smem(int H) { return sizeof(int) * 2 * (size_t)H + sizeof(int2) * 6 * (size_t)H; }

int segment_largest_hull(const uint8_t* const* mask_tbl_dev, int n, int H, int W, int32_t* label, int32_t* count, unsigned long long* best,
                         uint8_t* fill, cudaStream_t stream) {
	const int HW = H * W;
	const dim3 gp((unsigned)((HW + SEG_THREADS - 1) / SEG_THREADS), (unsigned)n);
	k_ccl_init<<<gp, SEG_THREADS, 0, stream>>>(mask_tbl_dev, label, count, best, HW);
	k_ccl_merge<<<dim3((unsigned)((W + 31) / 32), (unsigned)((H + 7) / 8), (unsigned)n), dim3(32, 8), 0, stream>>>(mask_tbl_dev, label, H, W);
	k_ccl_flatten<<<gp, SEG_THREADS, 0, stream>>>(label, count, HW);
	k_ccl_best<<<gp, SEG_THREADS, 0, stream>>>(label, count, best, HW);
	const size_t smem = hull_fill_smem(H);
	if (smem > 48 * 1024) BT_CUDA(cudaFuncSetAttribute(k_hull_fill, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
	k_hull_fill<<<n, HULL_THREADS, smem, stream>>>(label, best, fill, H, W);
	BT_CUDA(cudaGetLastError());
	return BT_OK;
}

// ---- the LF-Net request (Lfnet::detectFeature, rot_deg = 0): one thread per output pixel, the masked crop sampled on the fly.
static constexpr int REQ_SIDE = 400;
struct ReqArgs {
	const uint8_t* const* colour;   // [n] H x W x 3
	const uint8_t* const* fg;       // [n] H x W
	const int32_t* roi;             // [n][4]
	uint8_t* const* out;            // [n] 400 x 400 x 3
	int H, W;
};

// cv::resize's INTER_LINEAR source index and 11-bit weights for destination index d (resize.cpp: fx = (float)((d + 0.5) * scale - 0.5),
// scale = 1 / (dst / src) in double; the weights are saturate_cast<short>(w * 2048), i.e. rounded half to even).  Only the horizontal
// direction moves the weight onto the edge sample; both clamp the indices.
__device__ __forceinline__ void lin_coeffs(int d, int src, bool clamp_weights, int& s0, int& s1, int& w0, int& w1) {
	const double scale = __ddiv_rn(1.0, __ddiv_rn((double)REQ_SIDE, (double)src));
	float fx = __double2float_rn(__dadd_rn(__dmul_rn((double)d + 0.5, scale), -0.5));
	int s = (int)floorf(fx);
	fx = __fsub_rn(fx, (float)s);
	if (clamp_weights) {
		if (s < 0) { fx = 0.f; s = 0; }
		if (s >= src - 1) { fx = 0.f; s = src - 1; }
	}
	w0 = __float2int_rn(__fmul_rn(__fsub_rn(1.f, fx), 2048.f));
	w1 = __float2int_rn(__fmul_rn(fx, 2048.f));
	s0 = min(max(s, 0), src - 1); s1 = min(max(s + 1, 0), src - 1);
}

__global__ void __launch_bounds__(256) k_lfnet_request(ReqArgs a) {
	const int f = blockIdx.z, dx = blockIdx.x * 32 + threadIdx.x, dy = blockIdx.y * 8 + threadIdx.y;
	if (dx >= REQ_SIDE || dy >= REQ_SIDE) return;
	const int32_t* r = a.roi + 4 * (size_t)f;
	const int umin = r[0], umax = r[1], vmin = r[2], vmax = r[3];
	if (umax - umin < 10 || vmax - vmin < 10) return;        // the tracker's gate (Bundler.cpp:88-93): no request for this frame
	const int Wr = umax - umin, Hr = vmax - vmin, side = max(Wr, Hr), W = a.W;
	const uint8_t* __restrict__ col = a.colour[f];
	const uint8_t* __restrict__ fg = a.fg[f];
	uint8_t* __restrict__ o = a.out[f] + ((size_t)dy * REQ_SIDE + dx) * 3;
	// pixel (h, w) of the padded square: the colour zeroed where fg == 0 inside the crop [vmin, vmax) x [umin, umax), 0 outside
	auto px = [&](int h, int w, uchar3& c) {
		const size_t q = (size_t)(vmin + h) * W + (umin + w);
		if (h < Hr && w < Wr && fg[q]) c = make_uchar3(col[3 * q], col[3 * q + 1], col[3 * q + 2]);
		else c = make_uchar3(0, 0, 0);
	};
	uchar3 c00;
	if (side == REQ_SIDE) { px(dy, dx, c00); o[0] = c00.x; o[1] = c00.y; o[2] = c00.z; return; }
	int x0, x1, a0, a1, y0, y1, b0, b1;
	lin_coeffs(dx, side, true, x0, x1, a0, a1);
	lin_coeffs(dy, side, false, y0, y1, b0, b1);
	uchar3 c01, c10, c11;
	px(y0, x0, c00); px(y0, x1, c01); px(y1, x0, c10); px(y1, x1, c11);
	// horizontal pass exact; vertical pass as OpenCV's vector path rounds it: ((b0 * (h0 >> 4)) >> 16) + ((b1 * (h1 >> 4)) >> 16), then (t + 2) >> 2
	auto v = [&](int p00, int p01, int p10, int p11) {
		const int h0 = p00 * a0 + p01 * a1, h1 = p10 * a0 + p11 * a1;
		const int t = ((b0 * (h0 >> 4)) >> 16) + ((b1 * (h1 >> 4)) >> 16);
		return (uint8_t)min(max((t + 2) >> 2, 0), 255);
	};
	o[0] = v(c00.x, c01.x, c10.x, c11.x);
	o[1] = v(c00.y, c01.y, c10.y, c11.y);
	o[2] = v(c00.z, c01.z, c10.z, c11.z);
}

int launch_lfnet_request(const void* const* tbl_dev, const int32_t* roi_dev, int n, int H, int W, cudaStream_t stream) {
	ReqArgs a;
	a.colour = (const uint8_t* const*)tbl_dev; a.fg = (const uint8_t* const*)(tbl_dev + n); a.out = (uint8_t* const*)(tbl_dev + 2 * n);
	a.roi = roi_dev; a.H = H; a.W = W;
	k_lfnet_request<<<dim3((REQ_SIDE + 31) / 32, (REQ_SIDE + 7) / 8, (unsigned)n), dim3(32, 8), 0, stream>>>(a);
	BT_CUDA(cudaGetLastError());
	return BT_OK;
}

}  // namespace bt
