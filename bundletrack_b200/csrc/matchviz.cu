// matchviz.cu — the reference's match images (SiftManager::vizCorresBetween, src/FeatureManager.cpp:760-796): two ROI crops resized by an
// integer factor and placed side by side, with cv::drawMatches(NOT_DRAW_SINGLE_POINTS) of OpenCV 4.x drawn over them (DESIGN.md §3.11).
//
// Every match is three primitives in order: the circle at kp1 (clipped to the A half), the circle at kp2 (clipped to the B half) and the
// line.  A circle (radius 3, thickness 1, LINE_AA, shift 4) is EllipseEx's polygon of ellipse2Poly at a 30 degree step, drawn as 12 LineAA
// segments; the line is one LineAA.  So a match is 25 LineAA segments, each set up once by k_mv_setup (clipLine, the 16.16 start and step,
// the end-point correction table).
//
// A LineAA call touches a pixel at most once: it steps one pixel along its major axis and writes three distinct pixels across.  So the
// fragment a segment leaves on a pixel is a closed-form function of the pixel, and the blend, which reads the destination, only needs the
// segments in drawing order.  k_mv_base writes the canvas (the shared INTER_LINEAR of resize.cuh); k_mv_draw gives each 32 x 32 tile of an
// image one block, culls the matches against the tile 256 at a time (an order-keeping compaction), and every thread folds the surviving
// segments over its four pixels in drawing order.  No fragment is stored and nothing is sorted; the result is the same however the images
// are batched.
#include "bt_common.cuh"
#include "resize.cuh"

namespace bt {

namespace {

constexpr int kThreads = 256;
constexpr int kTile = 32;                        // tile side; a thread owns 4 pixels of a column
constexpr int kRows = kTile / (kThreads / kTile);
constexpr int kSegs = 25;                        // 12 + 12 circle segments, 1 line
constexpr int kXYShift = 16;
constexpr long long kXYOne = 1LL << kXYShift;
constexpr int kDrawShift = 4;

// one LineAA call, set up; a pixel (X, Y) of the image is (X - vx, Y) in the call's view of vw x vh pixels
struct MvSeg {
	int4 box;                                     // x0, y0, x1, y1 in image pixels (x0 > x1: empty)
	long long minor0, step;                       // the 16.16 minor coordinate at major0 and its step per pixel
	int major0, ecount;                           // ecount < 0: clipped away
	int vx, vw, vh;
	int xmajor;
	uint16_t ep[9];                               // the end-point correction table (9-bit values)
};
static_assert(sizeof(MvSeg) == 80, "bt_match_viz_reserve's documented footprint assumes an 80-byte segment");

struct MvImage {
	const uint8_t* a;                             // the crops' first pixels
	const uint8_t* b;
	int stride_a, stride_b;                       // bytes per colour row
	int ha, wa, hb, wb, s, rows, cols, tiles_x;
	double inv_s;                                 // 1 / (double)s
	float roi[4];                                // umin_a, vmin_a, umin_b, vmin_b
	const float4* uv;
	int n, match_base, tile_base;
	uint8_t* out;
};
static_assert(sizeof(MvImage) == 112, "bt_match_viz_reserve's documented footprint assumes a 112-byte image record");

__constant__ int c_slope_corr[32] = { 181, 181, 181, 182, 182, 183, 184, 185, 187, 188, 190, 192, 194, 196, 198, 201,
                                      203, 206, 209, 211, 214, 218, 221, 224, 227, 231, 235, 238, 242, 246, 250, 254 };
__constant__ int c_filter[64] = { 168, 177, 185, 194, 202, 210, 218, 224, 231, 236, 241, 246, 249, 252, 254, 254,
                                  254, 254, 252, 249, 246, 241, 236, 231, 224, 218, 210, 202, 194, 185, 177, 168,
                                  158, 149, 140, 131, 122, 114, 105, 97, 89, 82, 75, 68, 62, 56, 50, 45,
                                  40, 36, 32, 28, 25, 22, 19, 16, 14, 12, 11, 9, 8, 7, 5, 5 };
// OpenCV's SinTable at 30 k degrees and at 450 - 30 k (the cosine), as its float literals
__constant__ float c_sin[13] = { 0.f, 0.5f, 0.8660254f, 1.f, 0.8660254f, 0.5f, 0.f, -0.5f, -0.8660254f, -1.f, -0.8660254f, -0.5f, 0.f };
__constant__ float c_cos[13] = { 1.f, 0.8660254f, 0.5f, 0.f, -0.5f, -0.8660254f, -1.f, -0.8660254f, -0.5f, 0.f, 0.5f, 0.8660254f, 1.f };

__device__ __forceinline__ long long div_ll(double a, long long b, long long c) {   // (int64)((double)a * b / c)
	return __double2ll_rz(__ddiv_rn(__dmul_rn(a, __ll2double_rn(b)), __ll2double_rn(c)));
}

// cv::clipLine on a w x h rectangle (16.16 sizes)
__device__ bool clip_line(long long w, long long h, long long& x1, long long& y1, long long& x2, long long& y2) {
	const long long right = w - 1, bottom = h - 1;
	int c1 = (x1 < 0) + (x1 > right) * 2 + (y1 < 0) * 4 + (y1 > bottom) * 8;
	int c2 = (x2 < 0) + (x2 > right) * 2 + (y2 < 0) * 4 + (y2 > bottom) * 8;
	if ((c1 & c2) == 0 && (c1 | c2) != 0) {
		if (c1 & 12) {
			const long long a = c1 < 8 ? 0 : bottom;
			x1 += div_ll(__ll2double_rn(a - y1), x2 - x1, y2 - y1);
			y1 = a;
			c1 = (x1 < 0) + (x1 > right) * 2;
		}
		if (c2 & 12) {
			const long long a = c2 < 8 ? 0 : bottom;
			x2 += div_ll(__ll2double_rn(a - y2), x2 - x1, y2 - y1);
			y2 = a;
			c2 = (x2 < 0) + (x2 > right) * 2;
		}
		if ((c1 & c2) == 0 && (c1 | c2) != 0) {
			if (c1) {
				const long long a = c1 == 1 ? 0 : right;
				y1 += div_ll(__ll2double_rn(a - x1), y2 - y1, x2 - x1);
				x1 = a;
				c1 = 0;
			}
			if (c2) {
				const long long a = c2 == 1 ? 0 : right;
				y2 += div_ll(__ll2double_rn(a - x2), y2 - y1, x2 - x1);
				x2 = a;
				c2 = 0;
			}
		}
	}
	return (c1 | c2) == 0;
}

// cv::LineAA's set-up from p1 to p2 (16.16) in the view (vx, vw, vh)
__device__ void line_setup(long long x1, long long y1, long long x2, long long y2, int vx, int vw, int vh, MvSeg* __restrict__ g) {
	g->vx = vx; g->vw = vw; g->vh = vh;
	g->box = make_int4(1, 0, 0, 0);
	g->ecount = -1;
	if (!clip_line((long long)vw << kXYShift, (long long)vh << kXYShift, x1, y1, x2, y2)) return;
	long long dx = x2 - x1, dy = y2 - y1;
	const long long ax = dx < 0 ? -dx : dx, ay = dy < 0 ? -dy : dy;
	const bool xmajor = ax > ay;
	long long step, major0, minor0, ecount, i, j;
	if (xmajor) {
		if (dx < 0) { dy = -dy; long long t = x1; x1 = x2; x2 = t; t = y1; y1 = y2; y2 = t; }
		step = (dy << kXYShift) / (ax | 1);
		x2 += kXYOne;
		ecount = (x2 >> kXYShift) - (x1 >> kXYShift);
		j = -(x1 & (kXYOne - 1));
		y1 += ((step * j) >> kXYShift) + (kXYOne >> 1);
		i = (x1 >> (kXYShift - 7)) & 0x78; j = (x2 >> (kXYShift - 7)) & 0x78;
		major0 = x1 >> kXYShift; minor0 = y1;
	} else {
		if (dy < 0) { dx = -dx; long long t = x1; x1 = x2; x2 = t; t = y1; y1 = y2; y2 = t; }
		step = (dx << kXYShift) / (ay | 1);
		y2 += kXYOne;
		ecount = (y2 >> kXYShift) - (y1 >> kXYShift);
		j = -(y1 & (kXYOne - 1));
		x1 += ((step * j) >> kXYShift) + (kXYOne >> 1);
		i = (y1 >> (kXYShift - 7)) & 0x78; j = (y2 >> (kXYShift - 7)) & 0x78;
		major0 = y1 >> kXYShift; minor0 = x1;
	}
	int slope = (int)((step >> (kXYShift - 5)) & 0x3f);
	slope ^= step < 0 ? 0x3f : 0;
	slope = (slope & 0x20) ? 0x100 : c_slope_corr[slope];
	const long long t0 = (long long)slope << 7, t1 = ((0x78 - i) | 4) * slope, t2 = (j | 4) * slope;
	g->ep[0] = 0;
	g->ep[8] = (uint16_t)slope;
	g->ep[1] = g->ep[3] = (uint16_t)(((((j - i) & 0x78) | 4) * slope >> 8) & 0x1ff);
	g->ep[2] = (uint16_t)((t1 >> 8) & 0x1ff);
	g->ep[4] = (uint16_t)(((((j - i) + 0x80) | 4) * slope >> 8) & 0x1ff);
	g->ep[5] = (uint16_t)(((t1 + t0) >> 8) & 0x1ff);
	g->ep[6] = (uint16_t)((t2 >> 8) & 0x1ff);
	g->ep[7] = (uint16_t)(((t2 + t0) >> 8) & 0x1ff);
	g->minor0 = minor0; g->step = step; g->major0 = (int)major0; g->ecount = (int)ecount; g->xmajor = xmajor;
	// the pixels it can touch: majors inside the view, minors one pixel either side of the path
	const int n_major = xmajor ? vw : vh, n_minor = xmajor ? vh : vw;
	const long long k0 = max(0LL, -major0), k1 = min(ecount, (long long)n_major - 1 - major0);
	if (k0 > k1) return;
	const long long m0 = minor0 + k0 * step, m1 = minor0 + k1 * step;
	const int lo = max(0, (int)(min(m0, m1) >> kXYShift) - 1), hi = min(n_minor - 1, (int)(max(m0, m1) >> kXYShift) + 1);
	if (lo > hi) return;
	const int a0 = (int)(major0 + k0), a1 = (int)(major0 + k1);
	g->box = xmajor ? make_int4(vx + a0, lo, vx + a1, hi) : make_int4(vx + lo, a0, vx + hi, a1);
}

__device__ __forceinline__ int4 box_union(int4 a, int4 b) {
	if (a.x > a.z) return b;
	if (b.x > b.z) return a;
	return make_int4(min(a.x, b.x), min(a.y, b.y), max(a.z, b.z), max(a.w, b.w));
}

// cvRound(t * 16) of a float keypoint coordinate
__device__ __forceinline__ long long r16(float t) { return (long long)__float2int_rn(__fmul_rn(t, 16.f)); }

// one thread per (image, match, primitive): the circles' 12 segments or the line; the primitive's box for the tile culling
__global__ void __launch_bounds__(128) k_mv_setup(const MvImage* __restrict__ imgs, MvSeg* __restrict__ segs, int4* __restrict__ boxes) {
	const MvImage& I = imgs[blockIdx.y];
	const int t = blockIdx.x * blockDim.x + threadIdx.x;
	if (t >= 3 * I.n) return;
	const int m = t / 3, prim = t % 3;
	const float4 q = I.uv[m];
	const float s = (float)I.s;
	const float xa = __fmul_rn(__fsub_rn(q.x, I.roi[0]), s), ya = __fmul_rn(__fsub_rn(q.y, I.roi[1]), s);
	const float xb = __fmul_rn(__fsub_rn(q.z, I.roi[2]), s), yb = __fmul_rn(__fsub_rn(q.w, I.roi[3]), s);
	const int wa = I.wa * I.s;
	MvSeg* g = segs + (size_t)(I.match_base + m) * kSegs;
	int4 box = make_int4(1, 0, 0, 0);
	if (prim < 2) {
		// EllipseEx(centre, (r, r), 0, 0, 360) with r = 3 pixels: 13 polygon points 30 degrees apart, never two equal after rounding
		const long long sh = kXYShift - kDrawShift;
		const long long cx = (prim == 0 ? r16(xa) : r16(xb)) << sh, cy = (prim == 0 ? r16(ya) : r16(yb)) << sh;
		const double r = (double)((3LL << kDrawShift) << sh);
		const int vx = prim == 0 ? 0 : wa, vw = prim == 0 ? wa : I.wb * I.s, vh = prim == 0 ? I.ha * I.s : I.hb * I.s;
		long long px = 0, py = 0;
#pragma unroll
		for (int k = 0; k <= 12; k++) {
			const double x = __dmul_rn(r, (double)c_cos[k]), y = __dmul_rn(r, (double)c_sin[k]);
			const double fx = __dsub_rn(__dadd_rn((double)cx, __dmul_rn(x, 1.0)), __dmul_rn(y, 0.0));
			const double fy = __dadd_rn(__dadd_rn((double)cy, __dmul_rn(x, 0.0)), __dmul_rn(y, 1.0));
			long long qx = __double2ll_rn(__dmul_rn(fx, 1.0 / kXYOne)) << kXYShift;
			long long qy = __double2ll_rn(__dmul_rn(fy, 1.0 / kXYOne)) << kXYShift;
			qx += __double2ll_rn(__dsub_rn(fx, (double)qx));
			qy += __double2ll_rn(__dsub_rn(fy, (double)qy));
			if (k > 0) {
				MvSeg* gk = g + prim * 12 + (k - 1);
				line_setup(px, py, qx, qy, vx, vw, vh, gk);
				box = box_union(box, gk->box);
			}
			px = qx; py = qy;
		}
	} else {
		const float x2 = __fadd_rn(xb, (float)wa), lim = (float)(I.cols - 1);
		const float dx2 = lim < x2 ? lim : x2;
		const long long sh = kXYShift - kDrawShift;
		MvSeg* gl = g + 24;
		line_setup(r16(xa) << sh, r16(ya) << sh, r16(dx2) << sh, r16(yb) << sh, 0, I.cols, I.rows, gl);
		box = gl->box;
	}
	boxes[3 * (size_t)(I.match_base + m) + prim] = box;
}

// the fragment segment g leaves on image pixel (X, Y): its alpha, or -1
__device__ __forceinline__ int frag_alpha(const MvSeg* __restrict__ g, int X, int Y, const int* s_filter) {
	const int lx = X - g->vx;
	if (lx < 0 || lx >= g->vw || Y >= g->vh) return -1;
	const bool xm = g->xmajor != 0;
	const int k = (xm ? lx : Y) - g->major0;
	if (k < 0 || k > g->ecount) return -1;
	const long long minor = g->minor0 + (long long)k * g->step;
	const int o = (xm ? Y : lx) - ((int)(minor >> kXYShift) - 1);
	if ((unsigned)o > 2u) return -1;
	const int dist = (int)(minor >> (kXYShift - 5)) & 31;
	const int ec = g->ecount - k;
	const int corr = g->ep[(((k >= 2) + 1) & (k | 2)) * 3 + (((ec >= 2) + 1) & (ec | 2))];
	const int f = s_filter[o == 0 ? dist + 32 : o == 1 ? dist : 63 - dist];
	return (corr * f >> 8) & 0xff;
}

// ICV_PUT_POINT of a 3-channel image: each channel blended twice
__device__ __forceinline__ void put(int* p, uchar4 c, int a) {
	const int cc[3] = { c.x, c.y, c.z };
#pragma unroll
	for (int k = 0; k < 3; k++) {
		int v = p[k];
		v += ((cc[k] - v) * a + 127) >> 8;
		v += ((cc[k] - v) * a + 127) >> 8;
		p[k] = v;
	}
}

// pixel (dx, dy) of a crop resized by s (a copy at s = 1); inv_s = 1 / (dst / src) = 1 / s in double, as cv::resize takes it
__device__ __forceinline__ void sample(const uint8_t* __restrict__ src, int stride, int h, int w, int s, double inv_s, int dx, int dy, int* p) {
	if (s == 1) {
		const uint8_t* q = src + (size_t)dy * stride + 3 * dx;
		p[0] = q[0]; p[1] = q[1]; p[2] = q[2];
		return;
	}
	int x0, x1, a0, a1, y0, y1, b0, b1;
	lin_coeffs_at(dx, inv_s, w, true, x0, x1, a0, a1);
	lin_coeffs_at(dy, inv_s, h, false, y0, y1, b0, b1);
	const uint8_t* r0 = src + (size_t)y0 * stride;
	const uint8_t* r1 = src + (size_t)y1 * stride;
#pragma unroll
	for (int k = 0; k < 3; k++) p[k] = lin_blend(r0[3 * x0 + k], r0[3 * x1 + k], r1[3 * x0 + k], r1[3 * x1 + k], a0, a1, b0, b1);
}

// does the line's path come within a pixel of the tile [x0, x0 + 31] x [y0, y0 + 31]?
__device__ __forceinline__ bool line_hits(const MvSeg* __restrict__ g, int x0, int y0) {
	const bool xm = g->xmajor != 0;
	const int t0 = xm ? x0 - g->vx : y0, n0 = xm ? y0 : x0 - g->vx;
	const long long k0 = max(0LL, (long long)t0 - g->major0), k1 = min((long long)g->ecount, (long long)t0 + kTile - 1 - g->major0);
	if (k0 > k1) return false;
	const long long m0 = g->minor0 + k0 * g->step, m1 = g->minor0 + k1 * g->step;
	const long long lo = (min(m0, m1) >> kXYShift) - 1, hi = (max(m0, m1) >> kXYShift) + 1;
	return hi >= n0 && lo <= n0 + kTile - 1;
}

// the image of tile block b: the last one whose first tile is at or before it
__device__ __forceinline__ int image_of(const MvImage* __restrict__ imgs, int n_images, int b) {
	int lo = 0, hi = n_images - 1;
	while (lo < hi) {
		const int mid = (lo + hi + 1) >> 1;
		if (imgs[mid].tile_base <= b) lo = mid; else hi = mid - 1;
	}
	return lo;
}

// the canvas under the matches: zeros, the resized A crop at the left, the resized B crop to its right
__global__ void __launch_bounds__(kThreads) k_mv_base(const MvImage* __restrict__ imgs, int n_images) {
	const MvImage& I = imgs[image_of(imgs, n_images, (int)blockIdx.x)];
	const int t = (int)blockIdx.x - I.tile_base;
	const int X = (t % I.tiles_x) * kTile + (threadIdx.x & (kTile - 1));
	const int wa = I.wa * I.s;
	if (X >= I.cols) return;
	for (int r = 0; r < kRows; r++) {
		const int Y = (t / I.tiles_x) * kTile + (threadIdx.x / kTile) + r * (kThreads / kTile);
		if (Y >= I.rows) return;
		int p[3] = { 0, 0, 0 };
		if (X < wa) { if (Y < I.ha * I.s) sample(I.a, I.stride_a, I.ha, I.wa, I.s, I.inv_s, X, Y, p); }
		else if (Y < I.hb * I.s) sample(I.b, I.stride_b, I.hb, I.wb, I.s, I.inv_s, X - wa, Y, p);
		uint8_t* o = I.out + ((size_t)Y * I.cols + X) * 3;
		o[0] = (uint8_t)p[0]; o[1] = (uint8_t)p[1]; o[2] = (uint8_t)p[2];
	}
}

__global__ void __launch_bounds__(kThreads, 1) k_mv_draw(const MvImage* __restrict__ imgs, int n_images, const MvSeg* __restrict__ segs,
                                                      const int4* __restrict__ boxes, const uchar4* __restrict__ colours) {
	__shared__ int s_filter[64];
	__shared__ int s_hit[kThreads];
	__shared__ int s_wc[kThreads / 32];
	const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
	if (tid < 64) s_filter[tid] = c_filter[tid];
	const MvImage& I = imgs[image_of(imgs, n_images, (int)blockIdx.x)];
	if (I.n == 0) return;                                                  // block-uniform
	const int t = (int)blockIdx.x - I.tile_base;
	const int x0 = (t % I.tiles_x) * kTile, y0 = (t / I.tiles_x) * kTile;
	const int X = x0 + lane;
	int px[kRows][3];
#pragma unroll
	for (int r = 0; r < kRows; r++) {
		const int Y = y0 + w + r * (kThreads / kTile);
		px[r][0] = px[r][1] = px[r][2] = 0;
		if (X >= I.cols || Y >= I.rows) continue;
		const uint8_t* o = I.out + ((size_t)Y * I.cols + X) * 3;
		px[r][0] = o[0]; px[r][1] = o[1]; px[r][2] = o[2];
	}
	bool any = false;
	const int4 tile = make_int4(x0, y0, x0 + kTile - 1, y0 + kTile - 1);
	for (int c0 = 0; c0 < I.n; c0 += kThreads) {
		// the matches of this chunk that reach the tile, in order, each with the mask of its primitives that do
		const int m = c0 + tid;
		int mask = 0;
		if (m < I.n) {
			const size_t gm = (size_t)(I.match_base + m);
#pragma unroll
			for (int p = 0; p < 3; p++) {
				const int4 b = boxes[3 * gm + p];
				bool hit = b.x <= b.z && b.x <= tile.z && b.z >= tile.x && b.y <= tile.w && b.w >= tile.y;
				if (hit && p == 2) hit = line_hits(segs + gm * kSegs + 24, x0, y0);
				mask |= hit << p;
			}
		}
		const unsigned bal = __ballot_sync(0xffffffffu, mask != 0);
		if (lane == 0) s_wc[w] = __popc(bal);
		__syncthreads();
		int before = 0, total = 0;
#pragma unroll
		for (int k = 0; k < kThreads / 32; k++) { const int c = s_wc[k]; before += k < w ? c : 0; total += c; }
		if (mask) s_hit[before + __popc(bal & ((1u << lane) - 1u))] = m | (mask << 28);
		__syncthreads();
		any |= total > 0;
		for (int h = 0; h < total; h++) {
			const int e = s_hit[h];
			const size_t gm = (size_t)(I.match_base + (e & 0x0fffffff));
			const uchar4 col = colours[gm];
			const MvSeg* gs = segs + gm * kSegs;
			for (int p = 0; p < 3; p++) {
				if (!((e >> (28 + p)) & 1)) continue;
				const int n_seg = p < 2 ? 12 : 1;
				for (int k = 0; k < n_seg; k++) {
					const MvSeg* g = gs + p * 12 + k;
					const int4 b = g->box;
					if (b.x > b.z || b.x > tile.z || b.z < tile.x || b.y > tile.w || b.w < tile.y) continue;
#pragma unroll
					for (int r = 0; r < kRows; r++) {
						const int a = frag_alpha(g, X, y0 + w + r * (kThreads / kTile), s_filter);
						if (a >= 0) put(px[r], col, a);
					}
				}
			}
		}
		__syncthreads();
	}
	if (!any) return;                                                      // block-uniform: the tile keeps its canvas
#pragma unroll
	for (int r = 0; r < kRows; r++) {
		const int Y = y0 + w + r * (kThreads / kTile);
		if (X >= I.cols || Y >= I.rows) continue;
		uint8_t* o = I.out + ((size_t)Y * I.cols + X) * 3;
		o[0] = (uint8_t)px[r][0]; o[1] = (uint8_t)px[r][1]; o[2] = (uint8_t)px[r][2];
	}
}

// cv::RNG::next
inline uint64_t rng_next(uint64_t s) { return (uint64_t)(uint32_t)s * 4164903690ull + (s >> 32); }

struct VizTables : TableLayout { Slice<MvImage> images; Slice<uchar4> colours; };
VizTables viz_tables(size_t n_images, size_t n_matches) {
	VizTables t;
	t.images = t.add<MvImage>(n_images); t.colours = t.add<uchar4>(n_matches);
	return t;
}

bool roi_ok(const int32_t* r, int H, int W) { return r[0] >= 0 && r[0] < r[1] && r[1] <= W && r[2] >= 0 && r[2] < r[3] && r[3] <= H && r[3] - r[2] <= 900; }

}  // namespace

struct MatchVizState {
	bool ready = false;
	int max_images = 0, max_matches = 0;
	DevBuf segs, boxes;
	TableBlock<> tables;                           // the image table and the colours of one call
};
void StateDeleter::operator()(MatchVizState* s) const { delete s; }

}  // namespace bt

using namespace bt;

extern "C" int bt_match_viz_shape(const int32_t* roi_a, const int32_t* roi_b, int* rows, int* cols) {
	BT_REQUIRE(roi_a && roi_b && rows && cols, BT_ERR_INVALID_ARG, "bt_match_viz_shape: NULL argument");
	const int ha = roi_a[3] - roi_a[2], wa = roi_a[1] - roi_a[0], hb = roi_b[3] - roi_b[2], wb = roi_b[1] - roi_b[0];
	BT_REQUIRE(ha >= 1 && wa >= 1 && hb >= 1 && wb >= 1 && ha <= 900 && hb <= 900, BT_ERR_INVALID_ARG,
	           "bt_match_viz_shape: crops %d x %d and %d x %d must be at least 1 x 1 and at most 900 rows", wa, ha, wb, hb);
	const int s = min(900 / ha, 900 / hb);
	const long long c = (long long)(wa + wb) * s;
	BT_REQUIRE(c <= INT32_MAX / 3, BT_ERR_INVALID_ARG, "bt_match_viz_shape: %lld columns", c);
	*rows = max(ha, hb) * s;
	*cols = (int)c;
	return BT_OK;
}

extern "C" int bt_match_viz_reserve(bt_ctx* ctx, int max_images, int max_matches) {
	BT_REQUIRE(ctx, BT_ERR_INVALID_ARG, "bt_match_viz_reserve: ctx is NULL");
	// the images of a call are k_mv_setup's grid rows (at most 65535)
	BT_REQUIRE(max_images >= 1 && max_images <= 65535 && max_matches >= 0 && max_matches < (1 << 28), BT_ERR_INVALID_ARG,
	           "bt_match_viz_reserve: max_images %d must be in [1, 65535] and max_matches %d in [0, 2^28)", max_images, max_matches);
	MatchVizState* s;
	BT_TRY(take_state(ctx, &bt_ctx::matchviz, &s));
	const size_t mm = (size_t)max(max_matches, 1);
	BT_TRY(s->segs.alloc(sizeof(MvSeg) * kSegs * mm));
	BT_TRY(s->boxes.alloc(sizeof(int4) * 3 * mm));
	BT_TRY(s->tables.reserve(viz_tables(max_images, mm).total));
	s->max_images = max_images; s->max_matches = max_matches;
	s->ready = true;
	return BT_OK;
}

extern "C" int bt_match_viz(bt_ctx* ctx, int n_images, const bt_match_viz_desc* desc, uint8_t* const* out_dev, void* stream_) {
	BT_REQUIRE(desc && out_dev, BT_ERR_INVALID_ARG, "bt_match_viz: NULL argument");
	BT_REQUIRE(n_images >= 1, BT_ERR_INVALID_ARG, "bt_match_viz: n_images %d must be >= 1", n_images);
	MatchVizState* s;
	BT_TRY(state_of(ctx, &bt_ctx::matchviz, "bt_match_viz", "bt_match_viz_reserve", &s));
	long long total = 0, tiles = 0;
	for (int i = 0; i < n_images; i++) {
		const bt_match_viz_desc& d = desc[i];
		BT_REQUIRE(d.colour_a && d.colour_b && out_dev[i] && d.n >= 0 && (d.n == 0 || d.uv), BT_ERR_INVALID_ARG,
		           "bt_match_viz: image %d has a NULL pointer or n = %d", i, d.n);
		BT_REQUIRE(roi_ok(d.roi_a, d.H_a, d.W_a) && roi_ok(d.roi_b, d.H_b, d.W_b), BT_ERR_INVALID_ARG,
		           "bt_match_viz: image %d's ROIs must lie inside their images and be at most 900 rows", i);
		BT_REQUIRE(((uintptr_t)d.uv & 15) == 0, BT_ERR_INVALID_ARG, "bt_match_viz: image %d's uv list is not 16-byte aligned", i);
		int rows, cols;
		BT_TRY(bt_match_viz_shape(d.roi_a, d.roi_b, &rows, &cols));
		total += d.n;
		tiles += (long long)((cols + kTile - 1) / kTile) * ((rows + kTile - 1) / kTile);
	}
	// one block per tile of every image: k_mv_base's and k_mv_draw's grid
	BT_REQUIRE(tiles <= INT32_MAX, BT_ERR_INVALID_ARG, "bt_match_viz: %lld tiles of 32 x 32 pixels in one call exceed 2^31 - 1", tiles);
	BT_REQUIRE(n_images <= s->max_images && total <= s->max_matches, BT_ERR_CAPACITY,
	           "bt_match_viz: %d images / %lld matches exceed the reserved %d / %d", n_images, total, s->max_images, s->max_matches);
	cudaStream_t stream = (cudaStream_t)stream_;
	const VizTables t = viz_tables(n_images, (size_t)total);
	BT_TRY(s->tables.begin("bt_match_viz", t));
	MvImage* im = s->tables.host(t.images);
	uchar4* col = s->tables.host(t.colours);
	int match_base = 0, tile_base = 0, max_n = 0;
	for (int i = 0; i < n_images; i++) {
		const bt_match_viz_desc& d = desc[i];
		MvImage& I = im[i];
		I.ha = d.roi_a[3] - d.roi_a[2]; I.wa = d.roi_a[1] - d.roi_a[0];
		I.hb = d.roi_b[3] - d.roi_b[2]; I.wb = d.roi_b[1] - d.roi_b[0];
		I.s = min(900 / I.ha, 900 / I.hb);
		I.inv_s = 1.0 / (double)I.s;              // = 1 / ((s src) / src) exactly: s src / src is s in double
		bt_match_viz_shape(d.roi_a, d.roi_b, &I.rows, &I.cols);
		I.stride_a = 3 * d.W_a; I.stride_b = 3 * d.W_b;
		I.a = d.colour_a + (size_t)d.roi_a[2] * I.stride_a + 3 * (size_t)d.roi_a[0];
		I.b = d.colour_b + (size_t)d.roi_b[2] * I.stride_b + 3 * (size_t)d.roi_b[0];
		I.roi[0] = (float)d.roi_a[0]; I.roi[1] = (float)d.roi_a[2]; I.roi[2] = (float)d.roi_b[0]; I.roi[3] = (float)d.roi_b[2];
		I.uv = reinterpret_cast<const float4*>(d.uv);
		I.n = d.n; I.match_base = match_base; I.tile_base = tile_base; I.out = out_dev[i];
		I.tiles_x = (I.cols + kTile - 1) / kTile;
		tile_base += I.tiles_x * ((I.rows + kTile - 1) / kTile);
		// Scalar(rng(256), rng(256), rng(256)) with the arguments evaluated right to left: the first draw is R, the last B
		uint64_t st = d.rng_state;
		for (int m = 0; m < d.n; m++) {
			uint8_t v[3];
			for (int k = 0; k < 3; k++) { st = rng_next(st); v[k] = (uint8_t)((uint32_t)st % 256u); }
			col[match_base + m] = make_uchar4(v[2], v[1], v[0], 255);
		}
		match_base += d.n;
		max_n = max(max_n, d.n);
	}
	BT_TRY(s->tables.send(0, t.colours.end(), stream));
	BT_TRY(s->tables.in_flight(stream));
	const MvImage* d_im = s->tables.dev(t.images);
	if (total) k_mv_setup<<<dim3((3 * max_n + 127) / 128, n_images), 128, 0, stream>>>(d_im, s->segs.as<MvSeg>(), s->boxes.as<int4>());
	k_mv_base<<<tile_base, kThreads, 0, stream>>>(d_im, n_images);
	if (total) k_mv_draw<<<tile_base, kThreads, 0, stream>>>(d_im, n_images, s->segs.as<MvSeg>(), s->boxes.as<int4>(), s->tables.dev(t.colours));
	BT_CUDA(cudaGetLastError());
	return BT_OK;
}
