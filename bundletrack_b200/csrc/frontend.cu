// frontend.cu — the per-frame depth front end that feeds the solver's frame maps (SURVEY.md §8f rank 1):
//   Frame::processDepth          (/root/reference/src/Frame.cpp:152-180)  erode -> bilateral/"gauss" filter x2
//   Frame::depthToCloudAndNormals (Frame.cpp:182-233)                       camera-space points -> normals
// The reference runs five full-image kernels (CUDAImageUtil.cu:676-806, 310-336, 342-423) with a cudaMalloc/cudaFree
// pair around each group and two device->host copies of the maps for PCL.  Here ONE kernel does the whole chain per
// output tile: the raw depth of the tile plus its halo (erode radius + 2 x filter radius + 1 for the normal stencil) is
// staged in shared memory once and the four stencils ping-pong between two shared arrays, so the image is read ~1.6x
// and the three results (filtered depth, points, normals) are written once.  HBM-bound: 4 B in (2 B from a depth PNG), 4 + 16 + 16 B out per
// pixel.  Arithmetic follows the reference statement by statement (loop order of the float accumulations, float vs
// double comparisons, the hole-filling behaviour of the filter on invalid centre pixels).
#include "bt_common.cuh"

namespace bt {

static constexpr int FE_TW = 64, FE_TH = 32, FE_THREADS = 256;
static constexpr int FE_MAX_HALO = 12;

struct FrontArgs {
	const void* const* depth_in;    // [n] device pointers, H x W: float metres, or uint16 millimetres (the _u16 instantiation)
	float* const* depth_out;        // [n]
	float4* const* xyz_out;         // [n] or nullptr entries
	float4* const* normal_out;      // [n]
	int H, W;
	float k00, k11, k02, k12;       // inverse intrinsics as Eigen's 3x3 inverse forms them (cofactor * 1/det)
	int er; float e_diff, e_ratio;  // erode
	int br; float sigD, sigR;       // filter
};

__device__ __forceinline__ float4 to_camera(const FrontArgs& a, int x, int y, float d) {
	// convertDepthFloatToCameraSpaceFloat4_Kernel (CUDAImageUtil.cu:310-326): K^-1 * (x d, y d, d, d), output (x, y, w=d, 1)
	if (!(d >= 0.1f)) return make_float4(0.f, 0.f, 0.f, 0.f);     // (double)d >= 0.1 <=> d >= 0.1f
	const float xd = (float)x * d, yd = (float)y * d;
	return make_float4(a.k00 * xd + 0.f * yd + a.k02 * d + 0.f * d, 0.f * xd + a.k11 * yd + a.k12 * d + 0.f * d, d, 1.0f);
}

// One output pixel of gaussFilterDepthMapDevice (CUDAImageUtil.cu:735-796) from the staged neighbourhood (see the kernel for
// why no bounds tests are needed and how the weight table stays bit-identical to exp(a_tap - q)).  BR > 0: compile-time radius,
// the (2BR+1)^2 taps are read once into registers and serve both loops; BR == 0: run-time radius `rbr`, taps re-read.
template <int BR>
__device__ __forceinline__ float filter_pixel(const float* __restrict__ Sc, int RW, const float* __restrict__ t_a, const float* __restrict__ t_w,
                                              const float* __restrict__ t_q, float inv2sr, float num_total, int rbr = BR) {
	constexpr int SIDE = 2 * BR + 1, NT = BR > 0 ? SIDE * SIDE : 1;
	const int side = BR > 0 ? SIDE : 2 * rbr + 1, ntap = side * side, br = BR > 0 ? BR : rbr;
	const float centre = Sc[0];
	float v[NT];
	float mean = 0.f; int nv = 0;
	if (BR > 0) {
#pragma unroll
		for (int t = 0; t < NT; t++) {         // tap t: x offset outer, y offset inner (the reference's summation order)
			v[t] = Sc[(t % SIDE - BR) * RW + (t / SIDE - BR)];
			if (v[t] >= 0.1f) { nv++; mean += v[t]; }
		}
	} else {
		for (int t = 0; t < ntap; t++) { const float d = Sc[(t % side - br) * RW + (t / side - br)]; if (d >= 0.1f) { nv++; mean += d; } }
	}
	if (nv == 0) return 0.f;
	mean /= nv;
	float s = 0.f, sw = 0.f;
	if (BR > 0) {
#pragma unroll
		for (int t = 0; t < NT; t++) {
			const float d = v[t];
			if (d >= 0.1f && fabsf(d - mean) <= 0.01f) {
				const float dd = (centre - d) * (centre - d);
				const float wgt = (dd < t_q[t]) ? t_w[t] : expf(t_a[t] - dd / inv2sr);
				sw += wgt; s += wgt * d;
			}
		}
	} else {
		for (int t = 0; t < ntap; t++) {
			const float d = Sc[(t % side - br) * RW + (t / side - br)];
			if (d >= 0.1f && fabsf(d - mean) <= 0.01f) {
				const float dd = (centre - d) * (centre - d);
				const float wgt = (dd < t_q[t]) ? t_w[t] : expf(t_a[t] - dd / inv2sr);
				sw += wgt; s += wgt * d;
			}
		}
	}
	return (sw > 0.0f && (float)nv / num_total > 0) ? s / sw : 0.f;
}

// The masked instantiation (bt_frames_preprocess_masked) also stages the tile's pre-dilation mask with a halo of 2, takes its 5 x 5
// maximum (cv::dilate with a 5 x 5 rectangle; cells outside the image hold 0), writes it as fg, zeroes the three maps where fg == 0
// and folds the tile's ROI of fg != 0 into roi with atomics.  The maps are computed from the unmasked depth first, as in the
// reference, where invalidatePixelsByMask runs after the Frame constructor's filtering and normal estimation.
struct MaskArgs {
	const uint8_t* const* mask_in;  // [n] H x W pre-dilation masks
	uint8_t* const* fg_out;         // [n] H x W
	int32_t* roi;                   // [n][4] (umin, umax, vmin, vmax), (9999, 0, 9999, 0) on entry
};
static constexpr int FE_MW = FE_TW + 4, FE_MH = FE_TH + 4;

// One raw depth sample in metres.  uint16: Utils::readDepthImage (Utils.cpp:57-66) on the depth PNG's millimetres: (float)s * 0.001 is a
// double multiply (0.001 is a double literal) rounded to float, and values below 0.1 m (compared in double) become 0.
__device__ __forceinline__ float depth_sample(const float* p) { return __ldg(p); }
__device__ __forceinline__ float depth_sample(const uint16_t* p) {
	const float d = __double2float_rn(__dmul_rn((double)__ldg(p), 0.001));
	return ((double)d < 0.1) ? 0.f : d;
}

template <bool MASKED, class DIn>
__device__ __forceinline__ void frontend_tile(const FrontArgs& a, const MaskArgs& mk) {
	extern __shared__ float fe_smem[];
	const int er = a.er, br = a.br, halo = er + 2 * br + 1;
	const int RW = FE_TW + 2 * halo, RH = FE_TH + 2 * halo;      // staged region (stride RW for every stage)
	float* A = fe_smem;
	float* B = fe_smem + RW * RH;
	const int f = blockIdx.z;
	const int x0 = blockIdx.x * FE_TW - halo, y0 = blockIdx.y * FE_TH - halo;   // image coordinates of region cell (0,0)
	const int W = a.W, H = a.H;
	const DIn* __restrict__ din = static_cast<const DIn*>(a.depth_in[f]);
	// ---- stage 0: raw depth of the region; cells outside the image hold 0 here and after every later stage
	for (int c = threadIdx.x; c < RW * RH; c += FE_THREADS) {
		const int cx = c % RW, cy = c / RW, x = x0 + cx, y = y0 + cy;
		A[c] = (x >= 0 && x < W && y >= 0 && y < H) ? depth_sample(din + (size_t)y * W + x) : 0.f;
	}
	uint8_t* Ms = reinterpret_cast<uint8_t*>(fe_smem + 2 * RW * RH + 3 * (2 * br + 1) * (2 * br + 1));   // [FE_MH][FE_MW] mask, halo 2
	if constexpr (MASKED) {
		const uint8_t* __restrict__ mi = mk.mask_in[f];
		const int mx0 = blockIdx.x * FE_TW - 2, my0 = blockIdx.y * FE_TH - 2;
		for (int c = threadIdx.x; c < FE_MW * FE_MH; c += FE_THREADS) {
			const int x = mx0 + c % FE_MW, y = my0 + c / FE_MW;
			Ms[c] = (x >= 0 && x < W && y >= 0 && y < H) ? mi[(size_t)y * W + x] : (uint8_t)0;
		}
	}
	__syncthreads();
	const float MINF = __int_as_float(0xff800000);
	// ---- stage 1: erodeDepthMapDevice (CUDAImageUtil.cu:676-718) on the region shrunk by er: A -> B
	{
		const int m = er, w = RW - 2 * m, h = RH - 2 * m;
		const unsigned sum = (unsigned)((2 * er + 1) * (2 * er + 1));
		for (int c = threadIdx.x; c < w * h; c += FE_THREADS) {
			const int cx = m + c % w, cy = m + c / w, x = x0 + cx, y = y0 + cy;
			float out = 0.f;
			if (x >= 0 && x < W && y >= 0 && y < H) {
				const float old = A[cy * RW + cx];
				if (!(old <= 0.1f)) {
					unsigned count = 0;
					for (int i = -er; i <= er; i++)
						for (int j = -er; j <= er; j++)
							if (x + j >= 0 && x + j < W && y + i >= 0 && y + i < H) {
								const float d = A[(cy + i) * RW + (cx + j)];
								if (d == MINF || d < 0.1f || fabsf(d - old) > a.e_diff) count++;
							}
					out = ((float)count / (float)sum >= a.e_ratio) ? 0.f : old;
				}
			}
			B[cy * RW + cx] = out;
		}
	}
	__syncthreads();
	// ---- stages 2, 3: gaussFilterDepthMapDevice (CUDAImageUtil.cu:735-796), twice: B -> A (margin er+br), A -> B (margin er+2br).
	//      Cells outside the image hold 0 in every stage, and the filter ignores neighbours below 0.1 m, so the reference's
	//      bounds tests on the neighbours are implied.  The weight exp(a_tap - q), a_tap = -(dx^2+dy^2)/(2 sigD^2), q =
	//      (centre-d)^2/(2 sigR^2): whenever q is too small to change a_tap in float (always, with the shipped sigma_R = 1e5)
	//      the sum rounds to a_tap and the weight IS the tabulated expf(a_tap) - same bits, no exp, no division.
	//      The reference's double comparisons are replaced by their exact float equivalents: (double)x < 0.01 <=> x <= 0.01f
	//      (0.01f is the largest float below 0.01), (double)x >= 0.1 <=> x >= 0.1f (0.1f is the smallest float above 0.1).
	const float inv2sd = 2.0f * a.sigD * a.sigD;
	const float inv2sr = 2 * a.sigR * a.sigR;
	const int side = 2 * br + 1, ntap = side * side;
	float* t_a = B + RW * RH;            // [ntap] a_tap
	float* t_w = t_a + ntap;             // [ntap] expf(a_tap)
	float* t_q = t_w + ntap;             // [ntap] (centre-d)^2 below this leaves a_tap (and the weight) unchanged
	for (int t = threadIdx.x; t < ntap; t += FE_THREADS) {
		const int mm = t / side - br, nn = t % side - br;      // x offset outer, y offset inner: the reference's summation order
		const float at = -(float)(mm * mm + nn * nn) / inv2sd;
		t_a[t] = at; t_w[t] = expf(at);
		t_q[t] = (at != 0.f) ? inv2sr * fabsf(at) * 1.4901161e-8f /* 2^-26 */ : inv2sr * 1.4901161e-8f;
	}
	__syncthreads();
	const float num_total = (float)(side * side);
	for (int pass = 0; pass < 2; pass++) {
		const float* S = pass == 0 ? B : A;
		float* D = pass == 0 ? A : B;
		const int m = er + br * (pass + 1), w = RW - 2 * m, h = RH - 2 * m;
		for (int c = threadIdx.x; c < w * h; c += FE_THREADS) {
			const int cx = m + c % w, cy = m + c / w, x = x0 + cx, y = y0 + cy;
			float out = 0.f;
			if (x >= 0 && x < W && y >= 0 && y < H) {
				const float* Sc = S + cy * RW + cx;
				if (br == 2) out = filter_pixel<2>(Sc, RW, t_a, t_w, t_q, inv2sr, num_total);       // the shipped radius: taps and tables in registers
				else if (br == 1) out = filter_pixel<1>(Sc, RW, t_a, t_w, t_q, inv2sr, num_total);
				else out = filter_pixel<0>(Sc, RW, t_a, t_w, t_q, inv2sr, num_total, br);
			}
			D[cy * RW + cx] = out;
		}
		__syncthreads();
	}
	// ---- stage 4: outputs on the tile (margin halo): filtered depth, camera-space point, normal (computeNormals_Kernel,
	//      CUDAImageUtil.cu:342-413: central / one-sided differences gated by 2 cm, oriented towards the camera)
	float* __restrict__ dout = a.depth_out[f];
	float4* __restrict__ xout = a.xyz_out ? a.xyz_out[f] : nullptr;
	float4* __restrict__ nout = a.normal_out[f];
	const float zth = 0.02f;
	uint8_t* __restrict__ fgo = MASKED ? mk.fg_out[f] : nullptr;
	int umin = 0x7fffffff, umax = -1, vmin = 0x7fffffff, vmax = -1;   // MASKED: this thread's ROI of fg != 0
	for (int c = threadIdx.x; c < FE_TW * FE_TH; c += FE_THREADS) {
		const int cx = halo + c % FE_TW, cy = halo + c / FE_TW, x = x0 + cx, y = y0 + cy;
		if (x >= W || y >= H) continue;
		const size_t o = (size_t)y * W + x;
		if constexpr (MASKED) {
			const uint8_t* mc = Ms + (c / FE_TW) * FE_MW + c % FE_TW;
			uint8_t v = 0;
#pragma unroll
			for (int i = 0; i < 5; i++)
#pragma unroll
				for (int j = 0; j < 5; j++) v = max(v, mc[i * FE_MW + j]);
			fgo[o] = v;
			if (v == 0) {
				const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
				dout[o] = 0.f; nout[o] = z;
				if (xout) xout[o] = z;
				continue;
			}
			umin = min(umin, x); umax = max(umax, x); vmin = min(vmin, y); vmax = max(vmax, y);
		}
		const float d = B[cy * RW + cx];
		dout[o] = d;
		const float4 CC = to_camera(a, x, y, d);
		if (xout) xout[o] = CC;
		float4 nrm = make_float4(0.f, 0.f, 0.f, 0.f);
		if (x > 0 && x < W - 1 && y > 0 && y < H - 1 && !(CC.z < 0.1f)) {
			const float4 PC = to_camera(a, x, y + 1, B[(cy + 1) * RW + cx]);
			const float4 CP = to_camera(a, x + 1, y, B[cy * RW + cx + 1]);
			const float4 MC = to_camera(a, x, y - 1, B[(cy - 1) * RW + cx]);
			const float4 CM = to_camera(a, x - 1, y, B[cy * RW + cx - 1]);
			const bool pc = PC.z >= 0.1f && fabsf(PC.z - CC.z) <= zth, mc = MC.z >= 0.1f && fabsf(MC.z - CC.z) <= zth;
			const bool cp = CP.z >= 0.1f && fabsf(CP.z - CC.z) <= zth, cm = CM.z >= 0.1f && fabsf(CM.z - CC.z) <= zth;
			if ((pc || mc) && (cp || cm)) {
				float ax, ay, az, bx, by, bz;      // "x_dir" (vertical difference) and "y_dir" (horizontal), as named in the reference
				if (pc && mc) { ax = PC.x - MC.x; ay = PC.y - MC.y; az = PC.z - MC.z; }
				else if (pc) { ax = PC.x - CC.x; ay = PC.y - CC.y; az = PC.z - CC.z; }
				else { ax = MC.x - CC.x; ay = MC.y - CC.y; az = MC.z - CC.z; }
				if (cp && cm) { bx = CP.x - CM.x; by = CP.y - CM.y; bz = CP.z - CM.z; }
				else if (cp) { bx = CP.x - CC.x; by = CP.y - CC.y; bz = CP.z - CC.z; }
				else { bx = CM.x - CC.x; by = CM.y - CC.y; bz = CM.z - CC.z; }
				float nx = ay * bz - az * by, ny = az * bx - ax * bz, nz = ax * by - ay * bx;
				const float l = sqrtf(nx * nx + ny * ny + nz * nz);
				nx /= l; ny /= l; nz /= l;
				if (nx * -CC.x + ny * -CC.y + nz * -CC.z < 0) { nx = -nx; ny = -ny; nz = -nz; }
				if (l > 0.0f) nrm = make_float4(nx, ny, nz, 0.0f);
			}
		}
		nout[o] = nrm;
	}
	if constexpr (MASKED) {
		umin = __reduce_min_sync(0xffffffffu, umin); umax = __reduce_max_sync(0xffffffffu, umax);
		vmin = __reduce_min_sync(0xffffffffu, vmin); vmax = __reduce_max_sync(0xffffffffu, vmax);
		if ((threadIdx.x & 31) == 0 && umax >= 0) {
			int32_t* r = mk.roi + 4 * (size_t)f;
			atomicMin(r, umin); atomicMax(r + 1, umax); atomicMin(r + 2, vmin); atomicMax(r + 3, vmax);
		}
	}
}

__global__ void __launch_bounds__(FE_THREADS) k_frame_frontend(FrontArgs a) { frontend_tile<false, float>(a, MaskArgs{}); }
__global__ void __launch_bounds__(FE_THREADS) k_frame_frontend_masked(FrontArgs a, MaskArgs m) { frontend_tile<true, float>(a, m); }
__global__ void __launch_bounds__(FE_THREADS) k_frame_frontend_masked_u16(FrontArgs a, MaskArgs m) { frontend_tile<true, uint16_t>(a, m); }

struct FrontState {
	TableBlock<> tables;
	// largest-hull mode scratch (segment.cu), grown on demand: label / pixel-count maps, per-frame winner, the filled hull maps
	DevBuf seg_label, seg_count, seg_best, seg_fill;
	// bt_lfnet_request's own pointer table, so it never waits on or overwrites the front end's
	TableBlock<> req_tables;
};
void StateDeleter::operator()(FrontState* s) const { delete s; }
static FrontState* g_front(bt_ctx* ctx, bool create) {
	if (!ctx->front && create) ctx->front.reset(new FrontState());
	return ctx->front.get();
}

// The optional mask part of a front-end call (bt_frames_preprocess_masked).
struct MaskSpec {
	const uint8_t* const* mask;     // [n] device pointers
	int mode;                       // BT_MASK_AS_IS / BT_MASK_LARGEST_HULL
	uint8_t* const* fg_out;         // [n]
	int32_t* roi_out;               // device [n][4]
};

// The pointer tables of a front-end call and, when masked, those of the mask and the ROI's initial (9999, 0, 9999, 0) per frame, which
// goes to the caller's roi_out.  mask_in is the mask the front end dilates: the caller's, or the filled hull.
struct FrontTables : TableLayout {
	Slice<const void*> depth_in; Slice<float*> depth_out; Slice<float4*> xyz_out, normal_out;
	Slice<const uint8_t*> mask, mask_in; Slice<uint8_t*> fg_out; Slice<int32_t> roi;
};
static FrontTables front_tables(size_t n_frames, bool masked) {
	const size_t nm = masked ? n_frames : 0;
	FrontTables t;
	t.depth_in = t.add<const void*>(n_frames); t.depth_out = t.add<float*>(n_frames);
	t.xyz_out = t.add<float4*>(n_frames); t.normal_out = t.add<float4*>(n_frames);
	t.mask = t.add<const uint8_t*>(nm); t.fg_out = t.add<uint8_t*>(nm); t.mask_in = t.add<const uint8_t*>(nm);
	t.roi = t.add<int32_t>(4 * nm);
	return t;
}

// depth_raw_dev: float metres, or uint16 millimetres when u16 (masked calls only)
static int frames_preprocess(bt_ctx* ctx, const char* who, int n_frames, const void* const* depth_raw_dev, bool u16, int H, int W, float fx, float fy, float cx, float cy,
                             const bt_depth_params* prm, float* const* depth_out_dev, float* const* xyz_out_dev, float* const* normal_out_dev,
                             const MaskSpec* mask, void* stream_) {
	BT_REQUIRE(ctx && depth_raw_dev && prm && depth_out_dev && normal_out_dev, BT_ERR_INVALID_ARG, "%s: NULL argument", who);
	BT_REQUIRE(n_frames > 0 && n_frames <= 65535 && H > 0 && W > 0, BT_ERR_INVALID_ARG, "%s: bad sizes (n=%d, %dx%d)", who, n_frames, W, H);
	BT_REQUIRE(prm->erode_radius >= 0 && prm->bf_radius >= 0 && prm->erode_radius + 2 * prm->bf_radius + 1 <= FE_MAX_HALO, BT_ERR_UNSUPPORTED,
	           "%s: erode radius %d + 2 x filter radius %d + 1 exceeds the supported halo %d", who, prm->erode_radius, prm->bf_radius, FE_MAX_HALO);
	BT_REQUIRE(fx != 0.f && fy != 0.f && prm->sigma_D != 0.f && prm->sigma_R != 0.f, BT_ERR_INVALID_ARG, "%s: zero focal length or sigma", who);
	const bool hull = mask && mask->mode == BT_MASK_LARGEST_HULL;
	if (mask) {
		BT_REQUIRE(mask->mask && mask->fg_out && mask->roi_out, BT_ERR_INVALID_ARG, "%s: NULL mask, fg or roi argument", who);
		BT_REQUIRE(mask->mode == BT_MASK_AS_IS || mask->mode == BT_MASK_LARGEST_HULL, BT_ERR_INVALID_ARG, "%s: unknown mask mode %d", who, mask->mode);
		BT_REQUIRE((size_t)H * W < (size_t)0x7fffffff, BT_ERR_UNSUPPORTED, "%s: %dx%d pixels do not fit the int32 labels", who, W, H);
		BT_REQUIRE(!hull || hull_fill_smem(H) <= 227 * 1024, BT_ERR_UNSUPPORTED, "%s: largest-hull mode supports at most 4150 rows (%d given)", who, H);
	}
	cudaStream_t stream = (cudaStream_t)stream_;
	BT_CUDA(cudaSetDevice(ctx->device));
	FrontState* s = g_front(ctx, true);
	const FrontTables t = front_tables(n_frames, mask != nullptr);
	const size_t hw = (size_t)H * W * n_frames;
	int rc;
	BT_TRY(s->tables.reserve(t.total));
	if (hull) {
		if ((rc = s->seg_label.alloc(sizeof(int32_t) * hw)) != BT_OK) return rc;
		if ((rc = s->seg_count.alloc(sizeof(int32_t) * hw)) != BT_OK) return rc;
		if ((rc = s->seg_fill.alloc(hw)) != BT_OK) return rc;
		if ((rc = s->seg_best.alloc(sizeof(unsigned long long) * n_frames)) != BT_OK) return rc;
	}
	BT_TRY(s->tables.begin(who, t));
	const void** h_in = s->tables.host(t.depth_in); float** h_out = s->tables.host(t.depth_out);
	float4** h_xyz = s->tables.host(t.xyz_out); float4** h_normal = s->tables.host(t.normal_out);
	bool any_xyz = false;
	for (int f = 0; f < n_frames; f++) {
		BT_REQUIRE(depth_raw_dev[f] && depth_out_dev[f] && normal_out_dev[f], BT_ERR_INVALID_ARG, "%s: frame %d has a NULL map", who, f);
		BT_REQUIRE((const void*)depth_raw_dev[f] != (const void*)depth_out_dev[f], BT_ERR_INVALID_ARG, "%s: frame %d: in-place filtering is not supported (tiles read their neighbours' input)", who, f);
		h_in[f] = depth_raw_dev[f]; h_out[f] = depth_out_dev[f];
		h_xyz[f] = xyz_out_dev ? (float4*)xyz_out_dev[f] : nullptr; h_normal[f] = (float4*)normal_out_dev[f];
		any_xyz = any_xyz || (xyz_out_dev && xyz_out_dev[f]);
		if (mask) {
			BT_REQUIRE(mask->mask[f] && mask->fg_out[f], BT_ERR_INVALID_ARG, "%s: frame %d has a NULL mask or fg map", who, f);
			BT_REQUIRE((const void*)mask->mask[f] != (const void*)mask->fg_out[f], BT_ERR_INVALID_ARG, "%s: frame %d: fg_out aliases the mask (tiles read their neighbours' mask)", who, f);
			s->tables.host(t.mask)[f] = mask->mask[f]; s->tables.host(t.fg_out)[f] = mask->fg_out[f];
			s->tables.host(t.mask_in)[f] = hull ? s->seg_fill.as<uint8_t>() + (size_t)H * W * f : mask->mask[f];
		}
	}
	if (xyz_out_dev) for (int f = 0; f < n_frames; f++) BT_REQUIRE(!any_xyz || xyz_out_dev[f], BT_ERR_INVALID_ARG, "%s: xyz outputs must be given for all frames or none", who);
	BT_TRY(s->tables.send(0, mask ? t.mask_in.end() : t.normal_out.end(), stream));
	if (mask) {
		int32_t* hr = s->tables.host(t.roi);
		for (int f = 0; f < n_frames; f++) { hr[4 * f] = 9999; hr[4 * f + 1] = 0; hr[4 * f + 2] = 9999; hr[4 * f + 3] = 0; }
		BT_CUDA(cudaMemcpyAsync(mask->roi_out, hr, sizeof(int32_t) * 4 * (size_t)n_frames, cudaMemcpyHostToDevice, stream));
	}
	BT_TRY(s->tables.in_flight(stream));
	FrontArgs a;
	a.depth_in = s->tables.dev(t.depth_in); a.depth_out = s->tables.dev(t.depth_out);
	a.xyz_out = any_xyz ? s->tables.dev(t.xyz_out) : nullptr; a.normal_out = s->tables.dev(t.normal_out);
	a.H = H; a.W = W;
	{   // Eigen::Matrix3f::inverse() of [[fx,0,cx],[0,fy,cy],[0,0,1]] (Frame.cpp:189): cofactors times 1/det, in float
		const float det = fx * fy, invdet = 1.0f / det;
		a.k00 = fy * invdet; a.k11 = fx * invdet; a.k02 = (0.f * cy - cx * fy) * invdet; a.k12 = -(fx * cy - cx * 0.f) * invdet;
	}
	a.er = prm->erode_radius; a.e_diff = prm->erode_diff; a.e_ratio = prm->erode_ratio;
	a.br = prm->bf_radius; a.sigD = prm->sigma_D; a.sigR = prm->sigma_R;
	const int halo = a.er + 2 * a.br + 1;
	const int ntap = (2 * a.br + 1) * (2 * a.br + 1);
	const size_t smem = sizeof(float) * (2 * (size_t)(FE_TW + 2 * halo) * (FE_TH + 2 * halo) + 3 * (size_t)ntap) + (mask ? (size_t)FE_MW * FE_MH : 0);
	const dim3 grid((unsigned)((W + FE_TW - 1) / FE_TW), (unsigned)((H + FE_TH - 1) / FE_TH), (unsigned)n_frames);
	if (!mask) {
		if (smem > 48 * 1024) BT_CUDA(cudaFuncSetAttribute(k_frame_frontend, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
		k_frame_frontend<<<grid, FE_THREADS, smem, stream>>>(a);
	} else {
		if (hull && (rc = segment_largest_hull(s->tables.dev(t.mask), n_frames, H, W, s->seg_label.as<int32_t>(), s->seg_count.as<int32_t>(),
		                                       s->seg_best.as<unsigned long long>(), s->seg_fill.as<uint8_t>(), stream)) != BT_OK) return rc;
		MaskArgs m;
		m.mask_in = s->tables.dev(t.mask_in); m.fg_out = s->tables.dev(t.fg_out); m.roi = mask->roi_out;
		auto* k = u16 ? k_frame_frontend_masked_u16 : k_frame_frontend_masked;
		if (smem > 48 * 1024) BT_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
		k<<<grid, FE_THREADS, smem, stream>>>(a, m);
	}
	BT_CUDA(cudaGetLastError());
	return BT_OK;
}

}  // namespace bt

using namespace bt;

extern "C" int bt_frames_preprocess(bt_ctx* ctx, int n_frames, const float* const* depth_raw_dev, int H, int W, float fx, float fy, float cx, float cy,
                                    const bt_depth_params* prm, float* const* depth_out_dev, float* const* xyz_out_dev, float* const* normal_out_dev,
                                    void* stream_) {
	return frames_preprocess(ctx, "bt_frames_preprocess", n_frames, (const void* const*)depth_raw_dev, false, H, W, fx, fy, cx, cy, prm, depth_out_dev, xyz_out_dev, normal_out_dev,
	                         nullptr, stream_);
}

extern "C" int bt_frames_preprocess_masked(bt_ctx* ctx, int n_frames, const float* const* depth_raw_dev, const uint8_t* const* mask_dev, int mask_mode,
                                           int H, int W, float fx, float fy, float cx, float cy, const bt_depth_params* prm, float* const* depth_out_dev,
                                           float* const* xyz_out_dev, float* const* normal_out_dev, uint8_t* const* fg_out_dev, int32_t* roi_out_dev,
                                           void* stream_) {
	const MaskSpec m{mask_dev, mask_mode, fg_out_dev, roi_out_dev};
	return frames_preprocess(ctx, "bt_frames_preprocess_masked", n_frames, (const void* const*)depth_raw_dev, false, H, W, fx, fy, cx, cy, prm, depth_out_dev, xyz_out_dev, normal_out_dev,
	                         &m, stream_);
}

extern "C" int bt_frames_preprocess_masked_u16(bt_ctx* ctx, int n_frames, const uint16_t* const* depth_mm_dev, const uint8_t* const* mask_dev, int mask_mode,
                                               int H, int W, float fx, float fy, float cx, float cy, const bt_depth_params* prm, float* const* depth_out_dev,
                                               float* const* xyz_out_dev, float* const* normal_out_dev, uint8_t* const* fg_out_dev, int32_t* roi_out_dev,
                                               void* stream_) {
	const MaskSpec m{mask_dev, mask_mode, fg_out_dev, roi_out_dev};
	return frames_preprocess(ctx, "bt_frames_preprocess_masked_u16", n_frames, (const void* const*)depth_mm_dev, true, H, W, fx, fy, cx, cy, prm, depth_out_dev,
	                         xyz_out_dev, normal_out_dev, &m, stream_);
}

extern "C" int bt_lfnet_request(bt_ctx* ctx, int n_frames, const uint8_t* const* colour_dev, const uint8_t* const* fg_dev, const int32_t* roi_dev,
                                int H, int W, uint8_t* const* request_out_dev, void* stream_) {
	BT_REQUIRE(ctx && colour_dev && fg_dev && roi_dev && request_out_dev, BT_ERR_INVALID_ARG, "bt_lfnet_request: NULL argument");
	BT_REQUIRE(n_frames > 0 && n_frames <= 65535 && H > 0 && W > 0, BT_ERR_INVALID_ARG, "bt_lfnet_request: bad sizes (n=%d, %dx%d)", n_frames, W, H);
	cudaStream_t stream = (cudaStream_t)stream_;
	BT_CUDA(cudaSetDevice(ctx->device));
	FrontState* s = g_front(ctx, true);
	TableLayout L;
	const Slice<const void*> tbl = L.add<const void*>(3 * (size_t)n_frames);   // [colour | fg | out]
	BT_TRY(s->req_tables.reserve(L.total));
	BT_TRY(s->req_tables.begin("bt_lfnet_request", L));
	const void** ht = s->req_tables.host(tbl);
	for (int f = 0; f < n_frames; f++) {
		BT_REQUIRE(colour_dev[f] && fg_dev[f] && request_out_dev[f], BT_ERR_INVALID_ARG, "bt_lfnet_request: frame %d has a NULL image", f);
		ht[f] = colour_dev[f]; ht[n_frames + f] = fg_dev[f]; ht[2 * n_frames + f] = request_out_dev[f];
	}
	BT_TRY(s->req_tables.send(0, tbl.end(), stream));
	BT_TRY(s->req_tables.in_flight(stream));
	return launch_lfnet_request(s->req_tables.dev(tbl), roi_dev, n_frames, H, W, stream);
}
