// knn.cu — all-pairs L2 k-nearest-neighbour matching of 256-d LF-Net descriptors on the Hopper tensor cores (wgmma).
//
// Replaces the two cv::cuda::DescriptorMatcher::knnMatch(…, k=5) calls of SiftManager::findCorresbyNN
// (/root/reference/src/FeatureManager.cpp:271-273) for a BATCH of frame pairs.  OpenCV's CUDA matcher materialises the nQ x nT
// fp32 distance matrix with a SIMT kernel, once per direction, and runs k row-min passes over it (SURVEY.md §2.2).  Here ONE
// tensor-core contraction per pair serves BOTH directions and the distance matrix is never written:
//
//   k_desc_prep    fp32 (pitched GpuMat rows) -> a pool slot: fp16 rows [rows padded to 256][256] for the tensor pass, an fp32
//                  copy for the exact stage, |x~|^2 of the ROUNDED rows (padding rows: zero data, norm +inf) and the measured
//                  rounding error |x~ - x| of every row.  Done once per descriptor set - once per FRAME with the persistent
//                  pool (bt_desc_pool_store at detectFeature time, FeatureManager.cpp:907), once per call otherwise.
//   k_knn_tc       persistent, warp-specialised wgmma kernel over the flattened list of (pair, 256-row B tile, 128-row A tile)
//                  units, cut into equal contiguous ranges (one per SM: no wave quantisation).  One producer thread keeps the B tile
//                  resident in shared memory (128 KB, reloaded K-chunk by K-chunk while the last unit of the previous tile still
//                  runs) and streams A tiles through a 5-stage ring with TMA (SWIZZLE_128B, K-major); two consumer warpgroups each
//                  own one 128-row half of the B tile and issue wgmma.m64n128k16 (fp16 x fp16 -> fp32) for the A tile's two 64-row
//                  halves into registers, then form d2 = |a~|^2 + |b~|^2 - 2 a~.b~ (scaled into [0,1] by a per-pair power of two)
//                  and reduce it BOTH ways inside the thread (a group is four rows / columns one thread holds, see knn_unpos):
//                    A->B  min over each group of 4 B columns                                      -> G_rowT[B group][A position]
//                    B->A  min over each group of 4 A rows                                         -> G_col [A group][B position]
//                  both stored as fp16 (round to nearest; the bound below carries the half ulp).  No data-dependent branch, no
//                  candidate lists, no shuffles.
//   k_knn_select   per query (lane) over its column of group minima: exact k-th smallest key -> a rigorous threshold (measured
//                  fp16 rounding error of both rows + accumulation slack + storage rounding) -> the groups that can still hold
//                  one of the k nearest; each member of such a group is then checked against the OTHER direction's matrix (the
//                  minimum over the 4-row group that contains the query is a lower bound of the member's own distance: 8 bytes
//                  instead of re-scoring four 512-byte rows) -> candidate list, typically k + 0..1 rows.
//   k_knn_rerank   exact float64 sum of (a-b)^2 on the fp32 rows of the candidates, top k by (distance, index).
//   k_knn_exact    exact brute force for the rows whose candidate set overflowed (degenerate inputs: many equal distances).
// Result == exact brute-force kNN (float64 distances, ties -> lower train index), distances returned as float(sqrt(d2)) like
// cv::NORM_L2.
#include <algorithm>
#include <cuda.h>
#include <cuda_fp16.h>
#include <map>
#include <math.h>
#include <stdlib.h>
#include "bt_common.cuh"

namespace bt {

static constexpr int KD = 256;              // descriptor dimension handled by the tensor path
static constexpr int BM = 128;              // A rows per unit (two wgmma M = 64 row blocks)
static constexpr int BN = 256;              // B rows per unit (two consumer warpgroups)
static constexpr int WN = 128;              // B rows per consumer warpgroup (wgmma N)
static constexpr int BK = 64;               // K elements per smem chunk: 64 fp16 = 128 B = one SWIZZLE_128B atom row
static constexpr int KCH = KD / BK;         // 4 chunks
static constexpr int STAGES = 5;            // A-operand pipeline depth (16 KB each)
static constexpr int GRP = 4;               // rows / columns per group minimum
static constexpr int KNN_THREADS = 128 * 3; // warpgroup 0: TMA producer (one thread); warpgroups 1, 2: wgmma + epilogue
static constexpr uint32_t CONSUMER_WARPS = 8;         // arrivals that free an A stage / a B chunk (lane 0 of every consumer warp)
static constexpr uint32_t SA_BYTES = BM * BK * 2;     // 16 KB per stage: one K-chunk of an A tile
static constexpr uint32_t SB_BYTES = BN * BK * 2;     // 32 KB per K-chunk of the resident B tile
static constexpr uint32_t SMEM_B = KCH * SB_BYTES;    // 128 KB
static constexpr uint32_t SMEM_A = STAGES * SA_BYTES; // 80 KB
static constexpr uint32_t SMEM_NORM = BN * 4;         // 1 KB
static constexpr uint32_t SMEM_BAR = 256;
static constexpr uint32_t SMEM_TOTAL = SMEM_B + SMEM_A + SMEM_NORM + SMEM_BAR + 1024;   // + alignment slack: 210 KB of the 227 KB a block may have
static constexpr int SEL_MAXG = 16;        // groups / candidates kept per query; more => exact fallback
static constexpr int SEL_MAXC = 16;

struct KnnPair {          // one non-empty frame pair: units (B tile tt, A tile qt), qt fastest
	int a_row0, b_row0;   // first pool row of the two descriptor sets
	int nA, nB;
	int n_qt, n_tt;
	int unit0;
	int nA_pad, nB_pad;   // n_qt * 128, n_tt * 256
	int setA, setB;       // pool slots (per-set maxima)
	int pad;
	long long g_row;      // offset (halves) of G_rowT [nB_pad/4][nA_pad]
	long long g_col;      // offset (halves) of G_col  [nA_pad/4][nB_pad]
};
struct PairConst { float s, inv_s, delta, emaxA, emaxB, pad0, pad1, pad2; };

// ------------------------------------------------------------------------------------------------ PTX helpers
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
	asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
	asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
	asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
	asm volatile(
	    "{\n"
	    ".reg .pred p;\n"
	    "WAIT_LOOP:\n"
	    "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
	    "@p bra WAIT_DONE;\n"
	    "bra WAIT_LOOP;\n"
	    "WAIT_DONE:\n"
	    "}\n" ::"r"(smem_u32(bar)),
	    "r"(parity)
	    : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* tmap, uint64_t* bar, int c0, int c1) {
	asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(smem_u32(smem_dst)),
	             "l"(tmap), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
	             : "memory");
}
// wgmma shared-memory matrix descriptor, K-major operand, SWIZZLE_128B, rows at 128-byte pitch, 8-row groups 1024 B apart.
//   [0,14) start address >> 4 | [16,30) leading byte offset >> 4 (unused for swizzled K-major) | [32,46) stride byte offset >> 4
//   (= 1024 >> 4) | [62,64) layout type (1 = SWIZZLE_128B).  A K step of 16 halves inside the 128-byte swizzle row adds 32 B to the start.
__device__ __forceinline__ uint64_t wgmma_desc_k128(uint32_t smem_addr) {
	uint64_t d = 0;
	d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);
	d |= (uint64_t)1 << 16;
	d |= (uint64_t)(1024 >> 4) << 32;
	d |= (uint64_t)1 << 62;
	return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// the accumulator registers are written asynchronously: nothing may read or move them across a wait
__device__ __forceinline__ void wgmma_fence_acc(float (&d)[64]) {
#pragma unroll
	for (int i = 0; i < 64; i++) asm volatile("" : "+f"(d[i])::"memory");
}
// D[64 x 128] (+)= A[smem, 64 x 16] * B[smem, 128 x 16]^T, fp16 inputs, fp32 accumulate, both operands K-major
__device__ __forceinline__ void wgmma_m64n128k16(float (&d)[64], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
	asm volatile(
	    "{\n"
	    ".reg .pred p;\n"
	    "setp.ne.b32 p, %66, 0;\n"
	    "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
	    "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, "
	    "%28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, "
	    "%54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n"
	    "}\n"
	    : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]),
	      "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]),
	      "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]),
	      "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]),
	      "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]),
	      "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]),
	      "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
	    : "l"(a_desc), "l"(b_desc), "r"(accumulate));
}

// ------------------------------------------------------------------------------------------------ k_desc_prep
struct PrepSet { const float* src; size_t pitch_bytes; int n; int row0; int rows_padded; int slot; };

__global__ void __launch_bounds__(256) k_desc_prep(const PrepSet* sets, __half* pool_h, float* pool_f, float* norms, float* errn, int* slot_meta) {
	const PrepSet st = sets[blockIdx.y];
	const int warps_per_block = blockDim.x >> 5, lane = threadIdx.x & 31;
	for (int r = blockIdx.x * warps_per_block + (threadIdx.x >> 5); r < st.rows_padded; r += gridDim.x * warps_per_block) {
		__half* dst = pool_h + (size_t)(st.row0 + r) * KD;
		float4* dstf = reinterpret_cast<float4*>(pool_f + (size_t)(st.row0 + r) * KD);
		float ss = 0.f, ee = 0.f;
		if (r < st.n) {
			const float* src = (const float*)((const char*)st.src + (size_t)r * st.pitch_bytes);
			// each lane converts 8 consecutive floats (two float4 loads, one 16-byte store) and keeps the fp32 copy
			const float4 a = __ldg(reinterpret_cast<const float4*>(src) + lane * 2), b = __ldg(reinterpret_cast<const float4*>(src) + lane * 2 + 1);
			dstf[lane * 2] = a; dstf[lane * 2 + 1] = b;
			const float v[8] = { a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w };
			__half h[8];
#pragma unroll
			for (int k = 0; k < 8; k++) {
				// fp16 range: values beyond +-65504 are clamped, halves that would be subnormal are flushed (whatever the tensor core does
				// with subnormals, it then sees a zero); either way the difference lands in the measured error norm of the row
				float c = fminf(fmaxf(v[k], -65504.f), 65504.f);
				if (fabsf(c) < 6.1035156e-5f) c = 0.f;
				h[k] = __float2half_rn(c);
				const float f = __half2float(h[k]);
				ss += f * f; const float dlt = v[k] - f; ee += dlt * dlt;
			}
			*reinterpret_cast<uint4*>(dst + lane * 8) = *reinterpret_cast<const uint4*>(h);
		} else {
			*reinterpret_cast<uint4*>(dst + lane * 8) = make_uint4(0u, 0u, 0u, 0u);
			dstf[lane * 2] = make_float4(0.f, 0.f, 0.f, 0.f); dstf[lane * 2 + 1] = make_float4(0.f, 0.f, 0.f, 0.f);
		}
#pragma unroll
		for (int o = 16; o > 0; o >>= 1) { ss += __shfl_xor_sync(0xffffffffu, ss, o); ee += __shfl_xor_sync(0xffffffffu, ee, o); }
		if (lane == 0) {
			norms[st.row0 + r] = (r < st.n) ? ss : __int_as_float(0x7f800000);
			const float en = sqrtf(ee) * 1.001f + 1e-7f;     // |x~ - x|, rounded up: the ACTUAL fp16 rounding error of this row
			errn[st.row0 + r] = (r < st.n) ? en : 0.f;
			if (r < st.n) { atomicMax(slot_meta + 2 * st.slot, __float_as_int(ss)); atomicMax(slot_meta + 2 * st.slot + 1, __float_as_int(en)); }   // non-negative floats order like ints
		}
	}
}

// per pair: the power-of-two scale that maps d2 into [0,1] for the fp16 group minima, the slack for the fp32 accumulation of the
// contraction and of the norms, and the largest row rounding errors of the two sets
__global__ void k_knn_pairconst(const KnnPair* __restrict__ pairs, int n_pairs, const int* __restrict__ slot_meta, PairConst* __restrict__ out) {
	const int p = blockIdx.x * blockDim.x + threadIdx.x;
	if (p >= n_pairs) return;
	const KnnPair pr = pairs[p];
	const float m2A = __int_as_float(slot_meta[2 * pr.setA]), m2B = __int_as_float(slot_meta[2 * pr.setB]);
	const float mx = 4.0f * fmaxf(m2A, m2B);          // d2 <= (|a| + |b|)^2 <= 4 max |x|^2
	float s = 1.0f;
	if (mx > 0.f && mx < 1e37f) {
		int e = ((__float_as_int(mx) >> 23) & 255) - 127;          // mx = m * 2^e, 1 <= m < 2
		if (__float_as_int(mx) & 0x7fffff) e++;                    // 2^e >= mx
		e = min(max(e, -100), 100);
		s = __int_as_float((127 - e) << 23);
	}
	PairConst c;
	c.s = s; c.inv_s = 1.0f / s;
	// |computed d2 - exact d2 of the rounded rows|: 272 fp32 accumulation steps of the tensor pipe (<= 2^-22 relative to the sum of
	// |products| <= |a||b| each), the two norms (256 terms each) and the epilogue's fma + add; bounded with room to spare
	c.delta = 1.5e-4f * (m2A + m2B) + 1e-30f;
	c.emaxA = __int_as_float(slot_meta[2 * pr.setA + 1]); c.emaxB = __int_as_float(slot_meta[2 * pr.setB + 1]);
	c.pad0 = c.pad1 = c.pad2 = 0.f;
	out[p] = c;
}

// ------------------------------------------------------------------------------------------------ k_knn_tc
// position in the flattened unit list; every role of the CTA walks the same sequence
struct UnitWalk {
	const KnnPair* pairs; int p; int tt, qt; KnnPair pr;
	__device__ __forceinline__ void init(const KnnPair* pairs_, int n_pairs, int u) {
		pairs = pairs_;
		int lo = 0, hi = n_pairs - 1;
		while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (pairs[mid].unit0 <= u) lo = mid; else hi = mid - 1; }
		p = lo; pr = pairs[p];
		const int l = u - pr.unit0;
		tt = l / pr.n_qt; qt = l - tt * pr.n_qt;
	}
	__device__ __forceinline__ void next() {      // (reads one element past the table after the very last unit: the host pads the table by one entry)
		if (++qt == pr.n_qt) { qt = 0; if (++tt == pr.n_tt) { tt = 0; ++p; pr = pairs[p]; } }
	}
};

__device__ __forceinline__ uint32_t h2_as_u32(__half2 h) { return *reinterpret_cast<uint32_t*>(&h); }
__device__ __forceinline__ uint32_t hmin2_u32(uint32_t a, uint32_t b) {
	const __half2 r = __hmin2(*reinterpret_cast<__half2*>(&a), *reinterpret_cast<__half2*>(&b));
	return h2_as_u32(r);
}

// ---- the consumer's view of the accumulator -----------------------------------------------------------------------------------
// wgmma.m64nNk16 hands thread T of a warpgroup (warp w = T / 32, lane l) register 4j + 2i + e = row 16 w + l / 4 + 8 i, column
// 8 j + 2 (l % 4) + e.  With two such accumulators (A rows 0..63 and 64..127 of the tile) a thread holds FOUR rows r + {0, 8, 64, 72},
// r = 16 w + l / 4, and of each of them the columns c + {0, 8, 64, 72}, c = 16 w' + 2 (l % 4) + e, w' = 0..3.  A "group" of four rows
// (columns) is such a set, so both group minima the matcher needs stay inside the thread:
//   B->A  min over the thread's four rows, per column                      (3 packed-fp16 min per column pair)
//   A->B  min over the four columns of a group, per row                    (3 packed-fp16 min per two groups)
// no shuffle, no select.  In POSITION space a group is four CONSECUTIVE positions: in a block of 128, position p belongs to group
// g = (p / 4) % 32 = 8 w + q and is row 16 w + q + 8 (p & 1) + 64 ((p >> 1) & 1).  Both group-minimum matrices are stored by position,
// and a thread's results land on 8 / 16 contiguous bytes.  k_knn_select works in position space and converts back with knn_unpos()
// where it touches real rows.
__host__ __device__ __forceinline__ int knn_unpos(int p) { return (p & ~127) + 16 * ((p >> 5) & 3) + ((p >> 2) & 7) + 8 * (p & 1) + 64 * ((p >> 1) & 1); }

// d2 (scaled) = |a~|^2 + |b~|^2 - 2 a~.b~ of a column pair, clamped at zero and rounded to an fp16 pair (cvt.rn.relu: a rounding-level
// negative d2 becomes +0, so the halves order like unsigned integers)
__device__ __forceinline__ uint32_t d2_f16x2(float acc_lo, float acc_hi, float2 nb, float na, float m2s) {
	const float lo = __fadd_rn(__fmaf_rn(m2s, acc_lo, nb.x), na), hi = __fadd_rn(__fmaf_rn(m2s, acc_hi, nb.y), na);
	uint32_t h;
	asm("cvt.rn.relu.f16x2.f32 %0, %1, %2;" : "=r"(h) : "f"(hi), "f"(lo));
	return h;
}

// One CTA per SM, persistent over its slice of the unit list.  Warpgroup 0: one thread issues every TMA load (the resident B tile per
// K-chunk, the A tiles through the STAGES ring).  Warpgroups 1 and 2 (consumer c = 0, 1): B rows [128 c, 128 c + 128) of the tile against
// all 128 A rows as two 64 x 128 accumulators in registers, then the epilogue straight from the registers into the two matrices.
__global__ void __launch_bounds__(KNN_THREADS, 1)
k_knn_tc(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b, const KnnPair* __restrict__ pairs, int n_pairs, int total_units,
         const float* __restrict__ norms, const PairConst* __restrict__ pconst, __half* __restrict__ G) {
	extern __shared__ uint8_t smem_raw[];
	uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);   // SWIZZLE_128B needs 1024-B alignment
	uint8_t* sB = smem;
	uint8_t* sA = smem + SMEM_B;
	float* sNorm = reinterpret_cast<float*>(smem + SMEM_B + SMEM_A);
	uint64_t* bars = reinterpret_cast<uint64_t*>(smem + SMEM_B + SMEM_A + SMEM_NORM);
	uint64_t* b_full = bars + 0;               // [KCH]  resident B tile, per K-chunk
	uint64_t* b_empty = bars + KCH;            // [KCH]
	uint64_t* full = bars + 2 * KCH;           // [STAGES]
	uint64_t* empty = full + STAGES;           // [STAGES]

	const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
	if (threadIdx.x == 0) {
		asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap_a) : "memory");
		asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap_b) : "memory");
		for (int s = 0; s < KCH; s++) { mbar_init(b_full + s, 1); mbar_init(b_empty + s, CONSUMER_WARPS); }
		for (int s = 0; s < STAGES; s++) { mbar_init(full + s, 1); mbar_init(empty + s, CONSUMER_WARPS); }
		asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
	}
	__syncthreads();
	// this CTA's contiguous slice of the unit list (balanced to +-1 unit)
	const int u0 = (int)(((long long)blockIdx.x * total_units) / gridDim.x), u1 = (int)(((long long)(blockIdx.x + 1) * total_units) / gridDim.x);
	if (u0 >= u1) return;

	if (warp < 4) {
		// ================================================= TMA producer
		asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory");      // registers go to the consumers: 128 x 40 + 256 x 232 <= 64 K
		if (threadIdx.x == 0) {
			uint32_t stage = 0, sphase = 0, bphase = 0;
			UnitWalk w; w.init(pairs, n_pairs, u0);
			for (int u = u0; u < u1; u++) {
				const bool newb = (u == u0) || (w.qt == 0);
				for (int kc = 0; kc < KCH; kc++) {
					if (newb) {      // the previous B tile's last MMAs of this K-chunk have retired: reload the chunk while the others still run
						mbar_wait(b_empty + kc, bphase ^ 1);
						mbar_expect_tx(b_full + kc, SB_BYTES);
						tma_load_2d(sB + kc * SB_BYTES, &tmap_b, b_full + kc, kc * BK, w.pr.b_row0 + w.tt * BN);
					}
					mbar_wait(empty + stage, sphase ^ 1);
					mbar_expect_tx(full + stage, SA_BYTES);
					tma_load_2d(sA + stage * SA_BYTES, &tmap_a, full + stage, kc * BK, w.pr.a_row0 + w.qt * BM);
					if (++stage == STAGES) { stage = 0; sphase ^= 1; }
				}
				if (newb) bphase ^= 1;
				if (u + 1 < u1) w.next();
			}
		}
		return;
	}
	// ================================================= consumers
	asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory");      // two 64 x 128 fp32 accumulators = 128 registers per thread
	const int c = warp / 4 - 1;                 // B rows [128 c, 128 c + 128) of the tile
	const int wq = warp & 3;                    // warp of the warpgroup: accumulator rows 16 wq .. 16 wq + 15 of each 64-row half
	const int q = lane >> 2, m = lane & 3;      // this thread: tile rows 16 wq + q + {0, 8, 64, 72}, columns 128 c + 8 j + 2 m (+1), j = 0..15
	const int ctid = threadIdx.x - 128;         // 0..255
	uint32_t stage = 0, sphase = 0, bphase = 0;
	UnitWalk w; w.init(pairs, n_pairs, u0);
	int cur_p = -1;
	float s = 1.f;
	float acc0[64], acc1[64];
	for (int u = u0; u < u1; u++) {
		const bool newb = (u == u0) || (w.qt == 0);
		const bool lastb = (u + 1 == u1) || (w.qt == w.pr.n_qt - 1);
		if (w.p != cur_p) { cur_p = w.p; s = pconst[cur_p].s; }
		if (newb) {      // |b~|^2 of the resident B tile (scaled) -> smem, one float per consumer thread
			asm volatile("bar.sync 1, 256;" ::: "memory");       // every consumer is done with the previous tile's norms
			sNorm[ctid] = __ldg(norms + w.pr.b_row0 + w.tt * BN + ctid) * s;
			asm volatile("bar.sync 1, 256;" ::: "memory");
		}
		const int qrow0 = w.qt * BM;                // first A row (within the pair's set) of this tile
		const float* nAp = norms + w.pr.a_row0 + qrow0 + 16 * wq + q;
		const float nA[4] = { __ldg(nAp) * s, __ldg(nAp + 8) * s, __ldg(nAp + 64) * s, __ldg(nAp + 72) * s };
		// ---- four K-chunks; the A stage (and, after a tile's last unit, the B chunk) of chunk kc - 1 is released once chunk kc's MMAs
		//      are issued and kc - 1's have retired
		uint32_t prev = 0;
		for (int kc = 0; kc < KCH; kc++) {
			if (newb) mbar_wait(b_full + kc, bphase);
			mbar_wait(full + stage, sphase);
			wgmma_fence();
			const uint32_t a_base = smem_u32(sA + stage * SA_BYTES), b_base = smem_u32(sB + kc * SB_BYTES + c * WN * 128);
#pragma unroll
			for (int k = 0; k < BK / 16; k++) {      // wgmma K = 16 halves = 32 bytes inside the 128-byte swizzle row
				const uint32_t accumulate = (uint32_t)((kc | k) != 0);
				const uint64_t bd = wgmma_desc_k128(b_base + k * 32);
				wgmma_m64n128k16(acc0, wgmma_desc_k128(a_base + k * 32), bd, accumulate);
				wgmma_m64n128k16(acc1, wgmma_desc_k128(a_base + 64 * 128 + k * 32), bd, accumulate);
			}
			wgmma_commit();
			if (kc > 0) {
				wgmma_wait<1>();
				if (lane == 0) { mbar_arrive(empty + prev); if (lastb) mbar_arrive(b_empty + kc - 1); }
			}
			prev = stage;
			if (++stage == STAGES) { stage = 0; sphase ^= 1; }
		}
		wgmma_wait<0>();
		wgmma_fence_acc(acc0);
		wgmma_fence_acc(acc1);
		if (lane == 0) { mbar_arrive(empty + prev); if (lastb) mbar_arrive(b_empty + KCH - 1); }
		if (newb) bphase ^= 1;
		// ---- epilogue
		const float m2s = -2.0f * s;
		// A->B matrix [B group][A position]: this thread's four rows are positions 4 g .. 4 g + 3, g = 8 wq + q; its B groups are 8 w' + 2 m + e
		__half* rowp = G + w.pr.g_row + (size_t)(w.tt * (BN / GRP) + c * (WN / GRP) + 2 * m) * (size_t)w.pr.nA_pad + (size_t)(qrow0 + 32 * wq + 4 * q);
		// B->A matrix [A group][B position]: A group 8 wq + q of the tile; the members of its B groups 8 w' + 2 m + e are positions 32 w' + 8 m .. + 7
		__half* colp = G + w.pr.g_col + (size_t)(qrow0 / GRP + 8 * wq + q) * (size_t)w.pr.nB_pad + (size_t)(w.tt * BN + c * WN + 8 * m);
		const size_t rstride = (size_t)w.pr.nA_pad;
		const float* nbs = sNorm + c * WN + 2 * m;
#pragma unroll
		for (int gw = 0; gw < 4; gw++) {      // w' = gw: member columns 16 w' + 2 m + e + {0, 8, 64, 72} = accumulator column blocks j = 2 w' + {0, 1, 8, 9}
			uint32_t h[4][4];                 // [row][member column] as (e = 0, e = 1) fp16 pairs
#pragma unroll
			for (int jj = 0; jj < 4; jj++) {
				const int j = 2 * gw + (jj & 1) + 8 * (jj >> 1);
				const float2 nb = *reinterpret_cast<const float2*>(nbs + 8 * j);
				h[0][jj] = d2_f16x2(acc0[4 * j], acc0[4 * j + 1], nb, nA[0], m2s);
				h[1][jj] = d2_f16x2(acc0[4 * j + 2], acc0[4 * j + 3], nb, nA[1], m2s);
				h[2][jj] = d2_f16x2(acc1[4 * j], acc1[4 * j + 1], nb, nA[2], m2s);
				h[3][jj] = d2_f16x2(acc1[4 * j + 2], acc1[4 * j + 3], nb, nA[3], m2s);
			}
			// ---- B->A: minimum over the thread's four rows, per column pair; transposed into position order and stored as 16 bytes
			uint32_t cm[4];
#pragma unroll
			for (int jj = 0; jj < 4; jj++) cm[jj] = hmin2_u32(hmin2_u32(h[0][jj], h[1][jj]), hmin2_u32(h[2][jj], h[3][jj]));
			*reinterpret_cast<uint4*>(colp + 32 * gw) = make_uint4(__byte_perm(cm[0], cm[1], 0x5410), __byte_perm(cm[2], cm[3], 0x5410), __byte_perm(cm[0], cm[1], 0x7632), __byte_perm(cm[2], cm[3], 0x7632));
			// ---- A->B: minimum over the four member columns, per row: (group 8 w' + 2 m, group 8 w' + 2 m + 1) x four rows
			uint32_t r[4];
#pragma unroll
			for (int i = 0; i < 4; i++) r[i] = hmin2_u32(hmin2_u32(h[i][0], h[i][1]), hmin2_u32(h[i][2], h[i][3]));
			__half* rp = rowp + (size_t)(8 * gw) * rstride;
			*reinterpret_cast<uint2*>(rp) = make_uint2(__byte_perm(r[0], r[1], 0x5410), __byte_perm(r[2], r[3], 0x5410));
			*reinterpret_cast<uint2*>(rp + rstride) = make_uint2(__byte_perm(r[0], r[1], 0x7632), __byte_perm(r[2], r[3], 0x7632));
		}
		if (u + 1 < u1) w.next();
	}
}

// ------------------------------------------------------------------------------------------------ select
struct SelJob {           // one per (pair, direction)
	long long g_off;      // this direction's matrix  [n_groups padded][q_stride]  (halves, offset into G)
	long long x_off;      // the other direction's    [queries / 4][x_stride]
	int q_stride, x_stride;
	int nq, nt, n_groups; // n_groups = ceil(nt / 4)
	int q_pool_row0, t_pool_row0;
	int pconst;           // index into the PairConst table, -1: empty pair (no tensor pass ran)
	int dir;              // 0: A->B outputs, 1: B->A outputs
	int out_off;          // rows (x k) into the idx/dist outputs of this direction
	int q_base;           // global query index of this job's row 0
	int blk0;             // first k_knn_select block of this job
	int pad0, pad1;
};
__device__ __forceinline__ int find_by_start(const int* __restrict__ start, int n, int v) {      // largest j with start[j] <= v
	int lo = 0, hi = n - 1;
	while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (start[mid] <= v) lo = mid; else hi = mid - 1; }
	return lo;
}
struct KnnOut { int32_t* idx[2]; float* dist[2]; };

// branch-free insertion into an ascending list that drops its largest entry; half2 = two queries at once (the keys are non-negative
// halves, +inf = empty)
template <int K> __device__ __forceinline__ void kmin_insert2(__half2 (&a)[K], __half2 x) {
	__half2 prev = a[0];
	a[0] = __hmin2(a[0], x);
#pragma unroll
	for (int j = 1; j < K; j++) { const __half2 cur = a[j]; a[j] = __hmin2(cur, __hmax2(prev, x)); prev = cur; }
}
__device__ __forceinline__ __half2 u32_as_h2(unsigned v) { return *reinterpret_cast<__half2*>(&v); }

// 64 queries per block: lane = two adjacent queries (the matrices are [group][query], so a warp reads 128 contiguous bytes per group
// and every min / max of the selection network serves both queries), 8 warps = 8 segments of the group axis.
template <int K> __global__ void __launch_bounds__(256) k_knn_select(const SelJob* __restrict__ jobs, const int* __restrict__ blk_start, int n_jobs,
                                                                     const __half* __restrict__ G, const float* __restrict__ errn, const PairConst* __restrict__ pconst,
                                                                     int k, int32_t* __restrict__ cand, int32_t* __restrict__ cand_cnt, int* __restrict__ qjob) {
	__shared__ unsigned s_top[8][K][32];
	__shared__ unsigned s_hmax[64];
	__shared__ int s_ng[64], s_nc[64];
	__shared__ int s_grp[64][SEL_MAXG];
	__shared__ int s_cand[64][SEL_MAXC];
	const int lane = threadIdx.x & 31, seg = threadIdx.x >> 5;
	const int ji = find_by_start(blk_start, n_jobs, (int)blockIdx.x);
	const SelJob jb = jobs[ji];
	const int q0 = ((int)blockIdx.x - jb.blk0) * 64;
	const bool live = jb.pconst >= 0;
	// Everything here runs in POSITION space (see knn_unpos): the matrices are stored by position, a group is four consecutive positions;
	// real row numbers only appear where a row's data (error norm, bounds, outputs) is touched.
	const int qa = q0 + 2 * lane;                                   // my two query positions: qa, qa + 1 (the matrices are padded to whole tiles: both loads stay inside)
	const bool anyq = live && (knn_unpos(qa) < jb.nq || knn_unpos(qa + 1) < jb.nq);
	const unsigned* Gq = reinterpret_cast<const unsigned*>(G + jb.g_off + qa);
	const size_t gstride = (size_t)jb.q_stride >> 1;                // in 32-bit words
	const int per = (jb.n_groups + 7) >> 3;
	const int g0 = min(seg * per, jb.n_groups), g1 = min(g0 + per, jb.n_groups);
	if (threadIdx.x < 64) { s_ng[threadIdx.x] = 0; s_nc[threadIdx.x] = 0; }
	// ---- pass 1: the K smallest keys of my segment, for both queries
	const __half2 inf2 = u32_as_h2(0x7c007c00u);
	__half2 top[K];
#pragma unroll
	for (int j = 0; j < K; j++) top[j] = inf2;
	if (anyq) {
		int g = g0;
		for (; g + 8 <= g1; g += 8) {      // eight independent loads in flight per lane: the matrices come from L2 / DRAM and this pass is latency-bound
			unsigned kq[8];
#pragma unroll
			for (int u = 0; u < 8; u++) kq[u] = __ldg(Gq + (size_t)(g + u) * gstride);
#pragma unroll
			for (int u = 0; u < 8; u++) kmin_insert2<K>(top, u32_as_h2(kq[u]));
		}
		for (; g + 4 <= g1; g += 4) {
			const unsigned k0 = __ldg(Gq + (size_t)g * gstride), k1 = __ldg(Gq + (size_t)(g + 1) * gstride);
			const unsigned k2 = __ldg(Gq + (size_t)(g + 2) * gstride), k3 = __ldg(Gq + (size_t)(g + 3) * gstride);
			kmin_insert2<K>(top, u32_as_h2(k0)); kmin_insert2<K>(top, u32_as_h2(k1)); kmin_insert2<K>(top, u32_as_h2(k2)); kmin_insert2<K>(top, u32_as_h2(k3));
		}
		for (; g < g1; g++) kmin_insert2<K>(top, u32_as_h2(__ldg(Gq + (size_t)g * gstride)));
	}
#pragma unroll
	for (int j = 0; j < K; j++) s_top[seg][j][lane] = h2_as_u32(top[j]);
	__syncthreads();
	if (seg == 0) {      // merge: the k-th smallest key of each whole column, then its threshold
		__half2 all[K];
#pragma unroll
		for (int j = 0; j < K; j++) all[j] = inf2;
		for (int s2 = 0; s2 < 8; s2++) {
#pragma unroll
			for (int j = 0; j < K; j++) kmin_insert2<K>(all, u32_as_h2(s_top[s2][j][lane]));
		}
		const int kk = min(min(k, jb.nt), K);
		unsigned hk2 = 0x7c007c00u;
#pragma unroll
		for (int j = 0; j < K; j++) if (j == kk - 1) hk2 = h2_as_u32(all[j]);
#pragma unroll
		for (int hq = 0; hq < 2; hq++) {
			const int q = knn_unpos(qa + hq);      // the real query row
			const unsigned hk16 = hq ? (hk2 >> 16) : (hk2 & 0xffffu);
			unsigned hmax = 0u;
			if (live && q < jb.nq) {
				hmax = 0xffffu;
				if (kk > 0 && hk16 < 0x7c00u) {
					const PairConst pc = pconst[jb.pconst];
					const float hk = __half2float(__ushort_as_half((unsigned short)hk16));
					const float eq = __ldg(errn + jb.q_pool_row0 + q);
					const float e = (eq + (jb.dir == 0 ? pc.emaxB : pc.emaxA)) * 1.0001f + 1e-9f;
					// k groups have a member (their minimum) whose stored key is <= hk  =>  the exact k-th distance is <= T:
					//   stored = rn16(s * computed d2): |stored - s d2c| <= 2^-11 stored + 2^-25;  |d2c - d2(rounded rows)| <= delta;  | |a~-b~| - |a-b| | <= e
					const float D2hi = fmaf(hk, 1.0f + 0x1p-10f, 0x1p-22f) * pc.inv_s + pc.delta;
					const float T = sqrtf(D2hi) * (1.0f + 1e-6f) + e;
					// a row whose rounded-row distance exceeds R is farther than T in exact arithmetic; translate R back into a stored key
					const float R = (T + e) * (1.0f + 1e-6f);
					const float hl = fmaf(R * R * (1.0f + 2e-6f) + pc.delta, pc.s * (1.0f + 0x1p-10f), 0x1p-22f);
					if (hl < 65000.f) hmax = (unsigned)__half_as_ushort(__float2half_ru(hl));
				}
			}
			s_hmax[2 * lane + hq] = hmax;
		}
	}
	__syncthreads();
	// ---- pass 2: groups that can still hold one of the k nearest (keys order like their bit patterns)
	const unsigned hm0 = s_hmax[2 * lane], hm1 = s_hmax[2 * lane + 1];
	if (anyq) {
		for (int gb = g0; gb < g1; gb += 8) {      // (second sweep over the same column: eight loads in flight again)
			unsigned kq[8];
#pragma unroll
			for (int u = 0; u < 8; u++) kq[u] = __ldg(Gq + (size_t)min(gb + u, g1 - 1) * gstride);
#pragma unroll
			for (int u = 0; u < 8; u++) {
				const int g = gb + u;
				const unsigned key2 = kq[u];
				const bool p0 = g < g1 && (key2 & 0xffffu) <= hm0 && hm0 != 0u, p1 = g < g1 && (key2 >> 16) <= hm1 && hm1 != 0u;
				if (p0) { const int slot = atomicAdd(&s_ng[2 * lane], 1); if (slot < SEL_MAXG) s_grp[2 * lane][slot] = g; }
				if (p1) { const int slot = atomicAdd(&s_ng[2 * lane + 1], 1); if (slot < SEL_MAXG) s_grp[2 * lane + 1][slot] = g; }
			}
		}
	}
	__syncthreads();
	// ---- members: the other direction's matrix holds, for (my 4-row group, member column), a minimum that includes my own entry
	//      => a lower bound of the member's stored key; 8 bytes per group instead of four descriptor rows
	for (int w2 = threadIdx.x; w2 < 64 * SEL_MAXG; w2 += 256) {
		const int ql = w2 & 63, it = w2 >> 6, q = q0 + ql;      // q: query POSITION
		if (live && it < min(s_ng[ql], SEL_MAXG)) {      // (queries beyond nq have hmax = 0 and therefore no groups)
			const int g = s_grp[ql][it];
			const unsigned hmax = s_hmax[ql];
			const uint2 m = __ldg(reinterpret_cast<const uint2*>(G + jb.x_off + (size_t)(q >> 2) * jb.x_stride + (size_t)g * GRP));
			const unsigned key4[4] = { m.x & 0xffffu, m.x >> 16, m.y & 0xffffu, m.y >> 16 };
#pragma unroll
			for (int j = 0; j < 4; j++) {
				const int t = knn_unpos(g * GRP + j);      // the member's real row
				if (t < jb.nt && key4[j] <= hmax) { const int c = atomicAdd(&s_nc[ql], 1); if (c < SEL_MAXC) s_cand[ql][c] = t; }
			}
		}
	}
	__syncthreads();
	for (int w2 = threadIdx.x; w2 < 64 * SEL_MAXC; w2 += 256) {
		const int ql = w2 & 63, c = w2 >> 6, q = knn_unpos(q0 + ql);      // back to the real query row for the outputs
		if (q < jb.nq) {
			const int ng = s_ng[ql], nc = s_nc[ql];
			const bool over = ng > SEL_MAXG || nc > SEL_MAXC;
			if (c == 0) { cand_cnt[jb.q_base + q] = over ? -1 : nc; qjob[jb.q_base + q] = ji; }
			if (!over && c < nc) cand[(size_t)(jb.q_base + q) * SEL_MAXC + c] = s_cand[ql][c];
		}
	}
}

// ------------------------------------------------------------------------------------------------ exact stage
__device__ __forceinline__ bool dist_less(double da, int ia, double db, int ib) {      // non-negative doubles order like their bit patterns
	const long long a = __double_as_longlong(da), b = __double_as_longlong(db);
	return a < b || (a == b && ia < ib);
}

// one warp per query row: exact float64 distance of every candidate on the fp32 copies of the rows (two rows in flight), top k by
// (distance, index).  The kernel is paced by the float -> double conversions (XU pipe) and the FP64 pipe; a variant with eight lanes per
// candidate and four candidates in flight (three shuffle steps instead of five) is slower: it
// converts the query's slice four times as often and idles on the last round's unused candidate slots.
__global__ void __launch_bounds__(256) k_knn_rerank(const SelJob* __restrict__ jobs, const int* __restrict__ qjob, int total_q,
                                                    const int32_t* __restrict__ cand, const int32_t* __restrict__ cand_cnt, const float* __restrict__ pool_f,
                                                    int k, KnnOut out, int* fallback_rows, int* fallback_count, int force_fallback) {
	const int lane = threadIdx.x & 31;
	const int gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
	if (gw >= total_q) return;
	const SelJob jb = jobs[__ldg(qjob + gw)];      // (k_knn_select wrote the job of every query next to its candidate count: a binary search over the
	                                               //  job table per warp would cost dozens of instructions per query)
	const int r = gw - jb.q_base;
	const int kk = min(k, jb.nt);
	const float INF = __int_as_float(0x7f800000);
	const int nc = (jb.pconst >= 0) ? cand_cnt[gw] : 0;
	bool ok = nc >= kk;      // fewer candidates than neighbours can only mean an overflow (-1) or a broken bound: recompute exactly
	double my_d = 1e300; int my_i = 0x7fffffff;      // lane c keeps candidate c
	if (ok && nc > 0) {
		const int myc = (lane < nc) ? cand[(size_t)gw * SEL_MAXC + lane] : 0;
		const float* qrow = pool_f + (size_t)(jb.q_pool_row0 + r) * KD;
		const float* tbase = pool_f + (size_t)jb.t_pool_row0 * KD;
		const float4 qa = __ldg(reinterpret_cast<const float4*>(qrow) + lane * 2), qb = __ldg(reinterpret_cast<const float4*>(qrow) + lane * 2 + 1);
		const double q0 = qa.x, q1 = qa.y, q2 = qa.z, q3 = qa.w, q4 = qb.x, q5 = qb.y, q6 = qb.z, q7 = qb.w;
		auto d2_exact = [&](const float4& b0, const float4& b1) -> double {
			double s = 0.0, d;
			d = q0 - (double)b0.x; s += d * d; d = q1 - (double)b0.y; s += d * d;
			d = q2 - (double)b0.z; s += d * d; d = q3 - (double)b0.w; s += d * d;
			d = q4 - (double)b1.x; s += d * d; d = q5 - (double)b1.y; s += d * d;
			d = q6 - (double)b1.z; s += d * d; d = q7 - (double)b1.w; s += d * d;
			return s;
		};
		for (int c = 0; c < nc; c += 2) {
			const int t0 = __shfl_sync(0xffffffffu, myc, c), t1 = __shfl_sync(0xffffffffu, myc, min(c + 1, nc - 1));
			const float4* r0 = reinterpret_cast<const float4*>(tbase + (size_t)t0 * KD) + lane * 2;
			const float4* r1 = reinterpret_cast<const float4*>(tbase + (size_t)t1 * KD) + lane * 2;
			const float4 x0 = __ldg(r0), x1 = __ldg(r0 + 1), y0 = __ldg(r1), y1 = __ldg(r1 + 1);
			double sa = d2_exact(x0, x1), sb = d2_exact(y0, y1);
#pragma unroll
			for (int o = 16; o > 0; o >>= 1) { sa += __shfl_xor_sync(0xffffffffu, sa, o); sb += __shfl_xor_sync(0xffffffffu, sb, o); }
			if (lane == c) { my_d = sa; my_i = t0; }
			if (lane == c + 1 && c + 1 < nc) { my_d = sb; my_i = t1; }
		}
	}
	// ---- rank by counting: lane c's output slot = number of candidates that order before it by (distance, index); the indices are
	//      distinct, so the ranks are a permutation (a sorted insertion of doubles cost five times the distance evaluation)
	int rank = 0;
	for (int j = 0; j < nc; j++) {
		const double dj = __shfl_sync(0xffffffffu, my_d, j);
		const int ij = __shfl_sync(0xffffffffu, my_i, j);
		rank += dist_less(dj, ij, my_d, my_i) ? 1 : 0;
	}
	int32_t* io = out.idx[jb.dir] + ((size_t)jb.out_off + r) * k;
	float* dd = out.dist[jb.dir] + ((size_t)jb.out_off + r) * k;
	if (ok && lane < nc && rank < kk) { io[rank] = my_i; dd[rank] = (float)sqrt(my_d); }
	if (lane < k && (!ok || lane >= kk)) { io[lane] = -1; dd[lane] = INF; }      // rows with fewer than k train rows are padded; a row that goes to the fallback is rewritten there
	if (force_fallback > 0 && gw % force_fallback == 0) ok = false;
	if (jb.nt == 0) ok = true;      // nothing to find
	if (lane == 0 && !ok) { const int slot = atomicAdd(fallback_count, 1); fallback_rows[slot] = gw; }
}

// exact brute force for the rows whose candidate set overflowed.  Few rows (the normal case: none or one): each row's train set is
// cut into FB_SEG segments, one CTA per (row, segment), the last CTA of a row (ticket) merges the FB_SEG partial lists.  Many rows:
// one CTA per row.  Every merge is a warp-parallel selection (k rounds of a shuffle arg-min), never a serial walk.
static constexpr int FB_SEG = 64, FB_SPLIT_ROWS = 256;

__device__ __forceinline__ double exact_d2(const float* __restrict__ a, const float* __restrict__ b, int lane) {
	// warp-cooperative sum over KD floats: lane handles 8 consecutive elements; fixed order => deterministic
	const float4 a0 = __ldg(reinterpret_cast<const float4*>(a) + lane * 2), a1 = __ldg(reinterpret_cast<const float4*>(a) + lane * 2 + 1);
	const float4 b0 = __ldg(reinterpret_cast<const float4*>(b) + lane * 2), b1 = __ldg(reinterpret_cast<const float4*>(b) + lane * 2 + 1);
	double s = 0.0, d;
	d = (double)a0.x - (double)b0.x; s += d * d; d = (double)a0.y - (double)b0.y; s += d * d;
	d = (double)a0.z - (double)b0.z; s += d * d; d = (double)a0.w - (double)b0.w; s += d * d;
	d = (double)a1.x - (double)b1.x; s += d * d; d = (double)a1.y - (double)b1.y; s += d * d;
	d = (double)a1.z - (double)b1.z; s += d * d; d = (double)a1.w - (double)b1.w; s += d * d;
#pragma unroll
	for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
	return s;
}
// Every lane brings two (distance, index) entries (index 0x7fffffff = empty; real indices are distinct); lane j < 8 returns the j-th
// smallest of the warp's 64 by (distance, index).
__device__ __forceinline__ void warp_select8(double d0, int i0, double d1, int i1, double& od, int& oi) {
	const int lane = threadIdx.x & 31;
	od = 1e300; oi = 0x7fffffff;
#pragma unroll 1
	for (int r = 0; r < 8; r++) {
		const bool first = dist_less(d0, i0, d1, i1);
		double wd = first ? d0 : d1; int wi = first ? i0 : i1;
#pragma unroll
		for (int o = 16; o > 0; o >>= 1) {
			const double xd = __shfl_xor_sync(0xffffffffu, wd, o); const int xi = __shfl_xor_sync(0xffffffffu, wi, o);
			if (dist_less(xd, xi, wd, wi)) { wd = xd; wi = xi; }
		}
		if (lane == r) { od = wd; oi = wi; }
		if (wi == 0x7fffffff) break;                     // nothing left (uniform: every lane holds the same winner)
		if (i0 == wi) { d0 = 1e300; i0 = 0x7fffffff; } else if (i1 == wi) { d1 = 1e300; i1 = 0x7fffffff; }
	}
}

__global__ void __launch_bounds__(256) k_knn_exact(const SelJob* __restrict__ jobs, const int* __restrict__ q_start, int n_jobs, const float* __restrict__ pool_f,
                                                    const int* __restrict__ fallback_rows, const int* __restrict__ fallback_count, int k, KnnOut out,
                                                    double* part_d, int* part_i, int* tickets) {
	__shared__ double s_d[8][8];
	__shared__ int s_i[8][8];
	__shared__ int s_last;
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	const int n = *fallback_count;
	const bool split = n <= FB_SPLIT_ROWS;
	const int S = split ? FB_SEG : 1;
	for (int w = blockIdx.x; w < n * S; w += gridDim.x) {
		const int f = w / S, seg = w - f * S;
		const int gw = fallback_rows[f];
		const int ji = find_by_start(q_start, n_jobs, gw);
		const SelJob jb = jobs[ji];
		const int r = gw - jb.q_base;
		const float* qrow = pool_f + (size_t)(jb.q_pool_row0 + r) * KD;
		const float* tbase = pool_f + (size_t)jb.t_pool_row0 * KD;
		const int len = (jb.nt + S - 1) / S, t0 = seg * len, t1 = min(jb.nt, t0 + len);
		// ---- every warp: sorted top-8 of its share of the segment (two rows in flight)
		double best_d[8]; int best_i[8];
#pragma unroll
		for (int j = 0; j < 8; j++) { best_d[j] = 1e300; best_i[j] = 0x7fffffff; }
		auto insert = [&](double cd, int ci) {
#pragma unroll
			for (int j = 0; j < 8; j++) {
				if (dist_less(cd, ci, best_d[j], best_i[j])) { const double td = best_d[j]; const int tix = best_i[j]; best_d[j] = cd; best_i[j] = ci; cd = td; ci = tix; }
			}
		};
		for (int ti = t0 + warp; ti < t1; ti += 16) {
			const int tj = ti + 8;
			const double da = exact_d2(qrow, tbase + (size_t)ti * KD, lane);
			const double db = exact_d2(qrow, tbase + (size_t)min(tj, t1 - 1) * KD, lane);
			insert(da, ti);
			if (tj < t1) insert(db, tj);
		}
		__syncthreads();      // (the previous round's readers of s_d are done)
		if (lane < 8) {
			double md = 1e300; int mi = 0x7fffffff;
#pragma unroll
			for (int j = 0; j < 8; j++) if (lane == j) { md = best_d[j]; mi = best_i[j]; }
			s_d[warp][lane] = md; s_i[warp][lane] = mi;
		}
		__syncthreads();
		int32_t* io = out.idx[jb.dir] + ((size_t)jb.out_off + r) * k;
		float* dd = out.dist[jb.dir] + ((size_t)jb.out_off + r) * k;
		if (warp == 0) {      // the CTA's 8 best of its 64 entries
			double od; int oi;
			warp_select8((&s_d[0][0])[2 * lane], (&s_i[0][0])[2 * lane], (&s_d[0][0])[2 * lane + 1], (&s_i[0][0])[2 * lane + 1], od, oi);
			if (lane < 8) {
				if (!split) { if (lane < k) { io[lane] = oi == 0x7fffffff ? -1 : oi; dd[lane] = oi == 0x7fffffff ? __int_as_float(0x7f800000) : (float)sqrt(od); } }
				else { part_d[((size_t)f * FB_SEG + seg) * 8 + lane] = od; part_i[((size_t)f * FB_SEG + seg) * 8 + lane] = oi; }
			}
			if (lane == 0) s_last = 0;
			__syncwarp();
			if (split) { __threadfence(); if (lane == 0) s_last = (atomicAdd(tickets + f, 1) == FB_SEG - 1); }
		}
		__syncthreads();
		if (split && s_last) {     // FB_SEG sorted lists (512 entries, two per thread) -> per-warp 8 best -> the row's k best
			__threadfence();
			const size_t base = (size_t)f * FB_SEG * 8 + 2 * threadIdx.x;
			double od; int oi;
			warp_select8(__ldcg(part_d + base), __ldcg(part_i + base), __ldcg(part_d + base + 1), __ldcg(part_i + base + 1), od, oi);
			__syncthreads();
			if (lane < 8) { s_d[warp][lane] = od; s_i[warp][lane] = oi; }
			__syncthreads();
			if (warp == 0) {
				warp_select8((&s_d[0][0])[2 * lane], (&s_i[0][0])[2 * lane], (&s_d[0][0])[2 * lane + 1], (&s_i[0][0])[2 * lane + 1], od, oi);
				if (lane < k) { io[lane] = oi == 0x7fffffff ? -1 : oi; dd[lane] = oi == 0x7fffffff ? __int_as_float(0x7f800000) : (float)sqrt(od); }
				if (lane == 0) tickets[f] = 0;
			}
		}
		__syncthreads();
	}
}

// ------------------------------------------------------------------------------------------------ host side
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                    const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

struct MatcherState {
	bool ready = false;
	int max_pairs = 0, max_feats = 0, dim = 0;
	int slot_rows = 0;                      // rows per pool slot (max_feats padded to 256)
	int n_transient = 0, n_persist = 0;     // transient slots [0, n_transient) serve bt_knn_match_pairs; persistent ones follow
	std::vector<int> slot_n;                // persistent slots: number of rows stored, -1 = empty
	DevBuf pool_h, pool_f, norms, errn, slot_meta, pconst, G, cand, cand_cnt, qjob, fb_rows, fb_count, fb_part_d, fb_part_i, fb_tickets;
	TableBlock<> tables;                    // the set and work tables of a call (KnnTables)
	PFN_encodeTiled encode = nullptr;
	CUtensorMap tmap_a, tmap_b;
	size_t g_halves_cap = 0;
	int max_q_total = 0, max_blocks = 0;
	int last_units = 0, last_rows = 0;
	Event ev[5];
	bool timing = false;
	int force_fallback = 0;     // test knob: every n-th query row is sent to the exact fallback regardless of its candidates
};
void StateDeleter::operator()(MatcherState* m) const { delete m; }

static int make_tmap(MatcherState* m, CUtensorMap* out, void* base, uint64_t rows, uint32_t box_rows) {
	const cuuint64_t gdim[2] = { (cuuint64_t)KD, rows };
	const cuuint64_t gstride[1] = { (cuuint64_t)KD * 2 };
	const cuuint32_t box[2] = { (cuuint32_t)BK, box_rows };
	const cuuint32_t estr[2] = { 1, 1 };
	const CUresult r = m->encode(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, base, gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
	                             CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
	if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled failed with CUresult %d", (int)r); return BT_ERR_CUDA; }
	return BT_OK;
}

// (re)allocates the descriptor pool for n_transient + n_persist slots and rebuilds the tensor maps over it
static int pool_alloc(MatcherState* m, int n_persist) {
	const size_t rows = (size_t)(m->n_transient + n_persist) * m->slot_rows + BN;
	BT_TRY(m->pool_h.alloc(rows * KD * 2));
	BT_TRY(m->pool_f.alloc(rows * KD * 4));
	BT_TRY(m->norms.alloc(rows * 4));
	BT_TRY(m->errn.alloc(rows * 4));
	BT_TRY(m->slot_meta.alloc(sizeof(int) * 2 * (size_t)(m->n_transient + n_persist)));
	BT_TRY(make_tmap(m, &m->tmap_a, m->pool_h.p, (uint64_t)rows, BM));
	return make_tmap(m, &m->tmap_b, m->pool_h.p, (uint64_t)rows, BN);
}

// timing event i, when timing is on: [ev0, ev1) = descriptor conversion + table upload + per-pair constants, [ev1, ev2) = k_knn_tc alone
static int mark(MatcherState* m, int i, cudaStream_t stream) { if (m->timing) BT_CUDA(cudaEventRecord(m->ev[i], stream)); return BT_OK; }

static size_t desc_pitch(const bt_desc_view& v) { return v.pitch_bytes ? v.pitch_bytes : (size_t)KD * 4; }

// What the matcher requires of a descriptor set.  The error texts begin with `who`, or, for the view of pair `pair` >= 0, with "pair %d".
static int check_desc(const bt_desc_view& v, const MatcherState* m, const char* who, int pair) {
	char at[24];
	auto where = [&]() -> const char* { if (pair < 0) return who; snprintf(at, sizeof at, "pair %d", pair); return at; };
	BT_REQUIRE(v.dim == KD, BT_ERR_UNSUPPORTED, "%s: descriptor dim %d != %d", where(), v.dim, KD);
	BT_REQUIRE(v.n >= 0 && v.n <= m->max_feats, BT_ERR_CAPACITY, "%s: %d features > reserved %d", where(), v.n, m->max_feats);
	BT_REQUIRE(v.n == 0 || v.dev, BT_ERR_INVALID_ARG, "%s: NULL descriptor pointer", where());
	BT_REQUIRE(((uintptr_t)v.dev & 15) == 0 && (desc_pitch(v) & 15) == 0, BT_ERR_INVALID_ARG, "%s: descriptors must be 16-byte aligned", where());
	return BT_OK;
}

// the conversion of a checked descriptor set into pool slot `slot`, padded to whole 256-row B tiles
static PrepSet prep_set(const MatcherState* m, const bt_desc_view& v, int slot) {
	return PrepSet{ v.dev, desc_pitch(v), v.n, slot * m->slot_rows, (std::max(v.n, 1) + BN - 1) / BN * BN, slot };
}

struct PoolSetRef { int slot; int n; };      // a descriptor set in the pool: rows [slot * slot_rows, +n)

// The tables of a call: the descriptor sets it converts, then the work plan (KnnPlan) on n_pairs pairs.  The sets go up first, in a copy
// of their own, so that the conversion runs while the plan is made.
struct KnnTables : TableLayout { Slice<PrepSet> sets; Slice<KnnPair> pairs; Slice<SelJob> jobs; Slice<int> blk_start, q_start; };
static KnnTables knn_tables(size_t n_sets, size_t n_pairs) {
	KnnTables t;
	t.sets = t.add<PrepSet>(n_sets);
	t.pairs = t.add<KnnPair>(n_pairs + 1);      // (the live pairs and the guard entry)
	t.jobs = t.add<SelJob>(2 * n_pairs); t.blk_start = t.add<int>(2 * n_pairs); t.q_start = t.add<int>(2 * n_pairs);
	return t;
}

// uploads the set table.  `sets` take consecutive slots (one call's transient slots 0, 1, ..., or the one slot a store writes): one memset
// clears their counters.
static int launch_prep(MatcherState* m, const KnnTables& t, const std::vector<PrepSet>& sets, cudaStream_t stream) {
	if (sets.empty()) return BT_OK;
	memcpy(m->tables.host(t.sets), sets.data(), sizeof(PrepSet) * sets.size());
	BT_TRY(m->tables.send(t.sets.off, t.sets.end(), stream));
	BT_CUDA(cudaMemsetAsync(m->slot_meta.as<int>() + 2 * sets[0].slot, 0, 2 * sizeof(int) * sets.size(), stream));
	int max_padded = 0;
	for (auto& s : sets) max_padded = std::max(max_padded, s.rows_padded);
	k_desc_prep<<<dim3((unsigned)std::max(1, std::min((max_padded + 7) / 8, 64)), (unsigned)sets.size()), 256, 0, stream>>>(
	    m->tables.dev(t.sets), m->pool_h.as<__half>(), m->pool_f.as<float>(), m->norms.as<float>(), m->errn.as<float>(), m->slot_meta.as<int>());
	return BT_OK;
}

// The work of one call on descriptor sets in the pool, as the kernels walk it.
struct KnnPlan {
	std::vector<KnnPair> pairs;             // the live pairs, then a guard entry: UnitWalk::next() may read one entry past the last pair
	std::vector<SelJob> jobs;               // one per (pair, direction)
	std::vector<int> blk_start, q_start;    // per job: its first k_knn_select block, its first query row
	long long units = 0, g_off = 0;         // tensor-pass units; halves of G in use
	int q_total = 0, blocks = 0;            // query rows; k_knn_select blocks
};

static int plan_work(const MatcherState* m, const char* who, int n_pairs, const PoolSetRef* A, const PoolSetRef* B, KnnPlan& w) {
	size_t off_dir[2] = { 0, 0 };
	for (int p = 0; p < n_pairs; p++) {
		const int nA = A[p].n, nB = B[p].n;
		const bool live = nA > 0 && nB > 0;
		KnnPair pr; memset(&pr, 0, sizeof pr);
		if (live) {
			pr.a_row0 = A[p].slot * m->slot_rows; pr.b_row0 = B[p].slot * m->slot_rows; pr.nA = nA; pr.nB = nB;
			pr.n_qt = (nA + BM - 1) / BM; pr.n_tt = (nB + BN - 1) / BN; pr.unit0 = (int)w.units;      // a unit = 128 A rows x 256 B rows
			pr.nA_pad = pr.n_qt * BM; pr.nB_pad = pr.n_tt * BN; pr.setA = A[p].slot; pr.setB = B[p].slot;
			pr.g_row = w.g_off; w.g_off += (long long)(pr.nB_pad / GRP) * pr.nA_pad;
			pr.g_col = w.g_off; w.g_off += (long long)(pr.nA_pad / GRP) * pr.nB_pad;
			w.units += (long long)pr.n_qt * pr.n_tt;
			w.pairs.push_back(pr);
		}
		for (int dir = 0; dir < 2; dir++) {
			SelJob jb; memset(&jb, 0, sizeof jb);
			jb.nq = dir == 0 ? nA : nB; jb.nt = dir == 0 ? nB : nA; jb.n_groups = (jb.nt + 127) / 128 * (128 / GRP);      // whole blocks of 128 positions: a block's valid rows are spread over all of its groups
			jb.q_pool_row0 = (dir == 0 ? A[p].slot : B[p].slot) * m->slot_rows; jb.t_pool_row0 = (dir == 0 ? B[p].slot : A[p].slot) * m->slot_rows;
			jb.pconst = live ? (int)w.pairs.size() - 1 : -1;
			if (live) {
				jb.g_off = dir == 0 ? pr.g_row : pr.g_col; jb.x_off = dir == 0 ? pr.g_col : pr.g_row;
				jb.q_stride = dir == 0 ? pr.nA_pad : pr.nB_pad; jb.x_stride = dir == 0 ? pr.nB_pad : pr.nA_pad;
			}
			jb.dir = dir; jb.out_off = (int)off_dir[dir]; jb.q_base = w.q_total; jb.blk0 = w.blocks;
			w.jobs.push_back(jb);
			w.blk_start.push_back(w.blocks); w.q_start.push_back(w.q_total);
			w.blocks += (jb.nq + 127) / 128 * 2; w.q_total += jb.nq; off_dir[dir] += (size_t)jb.nq;
		}
	}
	BT_REQUIRE((size_t)w.g_off <= m->g_halves_cap && w.q_total <= m->max_q_total && w.blocks <= m->max_blocks && w.units < (1ll << 31), BT_ERR_CAPACITY, "%s: work list overflow", who);
	KnnPair guard; memset(&guard, 0, sizeof guard); guard.unit0 = (int)w.units; guard.n_qt = guard.n_tt = 1; w.pairs.push_back(guard);
	return BT_OK;
}

// one copy of the plan's tables to the device
static int upload_plan(MatcherState* m, const KnnTables& t, const KnnPlan& w, cudaStream_t stream) {
	memcpy(m->tables.host(t.pairs), w.pairs.data(), sizeof(KnnPair) * w.pairs.size());
	memcpy(m->tables.host(t.jobs), w.jobs.data(), sizeof(SelJob) * w.jobs.size());
	memcpy(m->tables.host(t.blk_start), w.blk_start.data(), sizeof(int) * w.blk_start.size());
	memcpy(m->tables.host(t.q_start), w.q_start.data(), sizeof(int) * w.q_start.size());
	BT_TRY(m->tables.send(t.pairs.off, t.q_start.end(), stream));
	return m->tables.in_flight(stream);
}

// The checks every matching entry point makes (A and B are its two input lists), then the device and the first mark.
static int begin_match(bt_ctx* ctx, const char* who, int n_pairs, const void* A, const void* B, int k, const KnnOut& out, cudaStream_t stream) {
	MatcherState* m;
	BT_TRY(state_of(ctx, &bt_ctx::matcher, who, "bt_matcher_reserve", &m));
	BT_REQUIRE(A && B && out.idx[0] && out.dist[0] && out.idx[1] && out.dist[1], BT_ERR_INVALID_ARG, "%s: NULL argument", who);
	BT_REQUIRE(k >= 1 && k <= 8, BT_ERR_UNSUPPORTED, "%s: k=%d outside [1,8]", who, k);
	BT_REQUIRE(n_pairs > 0 && n_pairs <= m->max_pairs, BT_ERR_CAPACITY, "%s: %d pairs > reserved %d", who, n_pairs, m->max_pairs);
	return mark(m, 0, stream);
}

// the matcher proper, after the conversion of `sets` into the pool
static int knn_run(bt_ctx* ctx, const char* who, int n_pairs, const std::vector<PrepSet>& sets, const PoolSetRef* A, const PoolSetRef* B, int k,
                   const KnnOut& out, cudaStream_t stream) {
	MatcherState* m = ctx->matcher.get();
	const KnnTables t = knn_tables(sets.size(), n_pairs);
	BT_TRY(m->tables.begin(who, t));
	BT_TRY(launch_prep(m, t, sets, stream));
	KnnPlan w;
	BT_TRY(plan_work(m, who, n_pairs, A, B, w));
	BT_TRY(upload_plan(m, t, w, stream));
	const KnnPair* d_pairs = m->tables.dev(t.pairs);
	const SelJob* d_jobs = m->tables.dev(t.jobs);
	const int n_live = (int)w.pairs.size() - 1, n_jobs = (int)w.jobs.size();
	BT_CUDA(cudaMemsetAsync(m->fb_count.p, 0, 16, stream));
	if (n_live > 0) k_knn_pairconst<<<(n_live + 127) / 128, 128, 0, stream>>>(d_pairs, n_live, m->slot_meta.as<int>(), m->pconst.as<PairConst>());
	BT_TRY(mark(m, 1, stream));
	if (n_live > 0) {
		const int grid = (int)std::min<long long>(w.units, ctx->sm_count);
		k_knn_tc<<<grid, KNN_THREADS, SMEM_TOTAL, stream>>>(m->tmap_a, m->tmap_b, d_pairs, n_live, (int)w.units, m->norms.as<float>(), m->pconst.as<PairConst>(), m->G.as<__half>());
	}
	BT_TRY(mark(m, 2, stream));
	if (w.q_total > 0) {
		auto* sel = k <= 5 ? k_knn_select<5> : k_knn_select<8>;
		sel<<<w.blocks, 256, 0, stream>>>(d_jobs, m->tables.dev(t.blk_start), n_jobs, m->G.as<__half>(), m->errn.as<float>(), m->pconst.as<PairConst>(), k, m->cand.as<int32_t>(), m->cand_cnt.as<int32_t>(), m->qjob.as<int>());
		k_knn_rerank<<<(w.q_total + 7) / 8, 256, 0, stream>>>(d_jobs, m->qjob.as<int>(), w.q_total, m->cand.as<int32_t>(), m->cand_cnt.as<int32_t>(), m->pool_f.as<float>(),
		                                                   k, out, m->fb_rows.as<int>(), m->fb_count.as<int>(), m->force_fallback);
		BT_TRY(mark(m, 3, stream));
		k_knn_exact<<<ctx->sm_count * 2, 256, 0, stream>>>(d_jobs, m->tables.dev(t.q_start), n_jobs, m->pool_f.as<float>(), m->fb_rows.as<int>(), m->fb_count.as<int>(), k, out,
		                                              m->fb_part_d.as<double>(), m->fb_part_i.as<int>(), m->fb_tickets.as<int>());
	} else BT_TRY(mark(m, 3, stream));
	BT_TRY(mark(m, 4, stream));
	BT_CUDA(cudaGetLastError());
	m->last_units = (int)w.units; m->last_rows = w.q_total;
	return BT_OK;
}

}  // namespace bt

using namespace bt;

int bt::matcher_reserve_args(int max_pairs, int max_feats, int dim) {
	BT_REQUIRE(dim == KD, BT_ERR_UNSUPPORTED, "bt_matcher_reserve: descriptor dim %d unsupported (the tensor path is built for %d)", dim, KD);
	BT_REQUIRE(max_pairs > 0 && max_feats > 0, BT_ERR_INVALID_ARG, "bt_matcher_reserve: bad limits");
	return BT_OK;
}

extern "C" int bt_matcher_reserve(bt_ctx* ctx, int max_pairs, int max_feats, int dim) {
	BT_REQUIRE(ctx, BT_ERR_INVALID_ARG, "bt_matcher_reserve: NULL ctx");
	BT_TRY(matcher_reserve_args(max_pairs, max_feats, dim));
	MatcherState* m;
	BT_TRY(take_state(ctx, &bt_ctx::matcher, &m));
	if (!m->encode) {
		void* fn = nullptr;
		cudaDriverEntryPointQueryResult qres;
		BT_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres));
		BT_REQUIRE(fn != nullptr && qres == cudaDriverEntryPointSuccess, BT_ERR_CUDA, "cuTensorMapEncodeTiled not available from the driver");
		m->encode = (PFN_encodeTiled)fn;
	}
	const int slot_rows = (max_feats + BN - 1) / BN * BN;
	if (slot_rows != m->slot_rows || std::min(2 * max_pairs, 128) != m->n_transient) std::fill(m->slot_n.begin(), m->slot_n.end(), -1);     // the persistent slots move: what they held is dropped
	m->slot_rows = slot_rows;
	m->n_transient = std::min(2 * max_pairs, 128);       // distinct descriptor sets one bt_knn_match_pairs call may name (all pairs of K frames: K sets)
	BT_TRY(pool_alloc(m, m->n_persist));
	const int pad_a = (max_feats + BM - 1) / BM * BM;      // A sets are padded to whole 128-row tiles
	const size_t g_halves_cap = (size_t)max_pairs * ((size_t)(slot_rows / GRP) * pad_a + (size_t)(pad_a / GRP) * slot_rows);
	const int max_q_total = 2 * max_pairs * max_feats;
	BT_TRY(m->tables.reserve(knn_tables(m->n_transient, max_pairs).total));
	BT_TRY(m->pconst.alloc(sizeof(PairConst) * (size_t)max_pairs));
	BT_TRY(m->G.alloc(g_halves_cap * 2 + 64));
	BT_TRY(m->cand.alloc(sizeof(int32_t) * SEL_MAXC * (size_t)max_q_total));
	BT_TRY(m->cand_cnt.alloc(sizeof(int32_t) * (size_t)max_q_total));
	BT_TRY(m->qjob.alloc(sizeof(int) * (size_t)max_q_total));
	BT_TRY(m->fb_rows.alloc(sizeof(int) * (size_t)max_q_total));
	BT_TRY(m->fb_count.alloc(16));
	BT_TRY(m->fb_part_d.alloc(sizeof(double) * (size_t)FB_SPLIT_ROWS * FB_SEG * 8)); BT_TRY(m->fb_part_i.alloc(sizeof(int) * (size_t)FB_SPLIT_ROWS * FB_SEG * 8));
	BT_TRY(m->fb_tickets.alloc(sizeof(int) * (size_t)FB_SPLIT_ROWS));
	BT_CUDA(cudaMemset(m->fb_tickets.p, 0, sizeof(int) * (size_t)FB_SPLIT_ROWS));
	BT_CUDA(cudaFuncSetAttribute(k_knn_tc, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_TOTAL));
	m->max_pairs = max_pairs; m->max_feats = max_feats; m->dim = dim;
	m->g_halves_cap = g_halves_cap; m->max_q_total = max_q_total;
	m->max_blocks = 2 * max_pairs * ((max_feats + 127) / 128 * 2);      // k_knn_select covers whole 128-position blocks, 64 queries per CTA
	m->ready = true;
	return BT_OK;
}

// Persistent descriptor pool (SURVEY.md 8f rank 3): Lfnet::detectFeature uploads a frame's descriptors once (FeatureManager.cpp:907);
// bt_desc_pool_store converts them once into a slot, bt_knn_match_slots / bt_match_pairs_pool then name slots.
extern "C" int bt_desc_pool_reserve(bt_ctx* ctx, int n_slots) {
	MatcherState* m;
	BT_TRY(state_of(ctx, &bt_ctx::matcher, "bt_desc_pool_reserve", "bt_matcher_reserve", &m));
	BT_REQUIRE(n_slots > 0, BT_ERR_INVALID_ARG, "bt_desc_pool_reserve: bad slot count");
	if (n_slots <= m->n_persist) return BT_OK;
	BT_CUDA(cudaDeviceSynchronize());          // the pool moves: nothing may still be reading the old one
	m->ready = false;                          // (the transient slots move too: until the pool is whole, the matcher refuses every call)
	m->n_persist = 0;
	m->slot_n.assign(n_slots, -1);             // (growing the pool re-allocates it: stored sets are dropped)
	BT_TRY(pool_alloc(m, n_slots));
	m->n_persist = n_slots;
	m->ready = true;
	return BT_OK;
}

extern "C" int bt_desc_pool_store(bt_ctx* ctx, int slot, const bt_desc_view* desc, void* stream_) {
	MatcherState* m;
	BT_TRY(state_of(ctx, &bt_ctx::matcher, "bt_desc_pool_store", "bt_matcher_reserve", &m));
	BT_REQUIRE(desc, BT_ERR_INVALID_ARG, "bt_desc_pool_store: NULL descriptor view");
	BT_REQUIRE(slot >= 0 && slot < m->n_persist, BT_ERR_INVALID_ARG, "bt_desc_pool_store: slot %d outside [0,%d)", slot, m->n_persist);
	BT_TRY(check_desc(*desc, m, __func__, -1));
	cudaStream_t stream = (cudaStream_t)stream_;
	const KnnTables t = knn_tables(1, 0);
	BT_TRY(m->tables.begin("bt_desc_pool_store", t));
	BT_TRY(launch_prep(m, t, { prep_set(m, *desc, m->n_transient + slot) }, stream));
	BT_TRY(m->tables.in_flight(stream));
	BT_CUDA(cudaGetLastError());
	m->slot_n[slot] = desc->n;
	return BT_OK;
}

extern "C" int bt_knn_match_slots(bt_ctx* ctx, int n_pairs, const int32_t* slotA, const int32_t* slotB, int k,
                                  int32_t* idxAB, float* distAB, int32_t* idxBA, float* distBA, void* stream_) {
	const KnnOut out{ { idxAB, idxBA }, { distAB, distBA } };
	cudaStream_t stream = (cudaStream_t)stream_;
	BT_TRY(begin_match(ctx, __func__, n_pairs, slotA, slotB, k, out, stream));
	MatcherState* m = ctx->matcher.get();
	std::vector<PoolSetRef> A(n_pairs), B(n_pairs);
	for (int p = 0; p < n_pairs; p++) {
		for (int s2 = 0; s2 < 2; s2++) {
			const int sl = s2 == 0 ? slotA[p] : slotB[p];
			BT_REQUIRE(sl >= 0 && sl < m->n_persist && m->slot_n[sl] >= 0, BT_ERR_INVALID_ARG, "bt_knn_match_slots: pair %d names slot %d, which is empty or out of range", p, sl);
			(s2 == 0 ? A[p] : B[p]) = PoolSetRef{ m->n_transient + sl, m->slot_n[sl] };
		}
	}
	return knn_run(ctx, __func__, n_pairs, {}, A.data(), B.data(), k, out, stream);
}

extern "C" int bt_knn_debug_force_fallback(bt_ctx* ctx, int every_nth) {
	MatcherState* m;
	BT_TRY(state_of(ctx, &bt_ctx::matcher, "bt_knn_debug_force_fallback", "bt_matcher_reserve", &m));
	m->force_fallback = every_nth > 0 ? every_nth : 0;
	return BT_OK;
}

extern "C" int bt_knn_enable_timing(bt_ctx* ctx, int on) {
	MatcherState* m;
	BT_TRY(state_of(ctx, &bt_ctx::matcher, "bt_knn_enable_timing", "bt_matcher_reserve", &m));
	if (on) for (Event& e : m->ev) BT_TRY(e.create(true));
	m->timing = on != 0;
	return BT_OK;
}
// ms4 = {descriptor prep, tensor-core pass, select + exact re-rank, exact fallback}; info3 = {units, query rows, fallback rows}
extern "C" int bt_knn_get_timing(bt_ctx* ctx, float* ms4, int* info3) {
	MatcherState* m;
	BT_TRY(state_of(ctx, &bt_ctx::matcher, "bt_knn_get_timing", "bt_matcher_reserve", &m));
	BT_REQUIRE(m->timing && ms4 && info3, BT_ERR_INVALID_ARG, "bt_knn_get_timing: timing not enabled");
	BT_CUDA(cudaEventSynchronize(m->ev[4]));
	for (int k = 0; k < 4; k++) BT_CUDA(cudaEventElapsedTime(ms4 + k, m->ev[k], m->ev[k + 1]));
	int fb = 0;
	BT_CUDA(cudaMemcpy(&fb, m->fb_count.p, sizeof(int), cudaMemcpyDeviceToHost));
	info3[0] = m->last_units; info3[1] = m->last_rows; info3[2] = fb;
	return BT_OK;
}

extern "C" int bt_knn_match_pairs(bt_ctx* ctx, int n_pairs, const bt_desc_view* A, const bt_desc_view* B, int k,
                                  int32_t* idxAB, float* distAB, int32_t* idxBA, float* distBA, void* stream_) {
	const KnnOut out{ { idxAB, idxBA }, { distAB, distBA } };
	cudaStream_t stream = (cudaStream_t)stream_;
	BT_TRY(begin_match(ctx, __func__, n_pairs, A, B, k, out, stream));
	MatcherState* m = ctx->matcher.get();
	// ---- unique descriptor sets (a keyframe appears in many pairs) -> transient pool slots, converted once per call
	std::map<std::pair<const float*, int>, int> slot_of;
	std::vector<PrepSet> sets;
	auto slot = [&](const bt_desc_view& v) -> int {
		const auto it = slot_of.emplace(std::make_pair(v.dev, v.n), (int)sets.size());
		if (it.second) sets.push_back(prep_set(m, v, it.first->second));
		return it.first->second;
	};
	std::vector<PoolSetRef> sa(n_pairs), sb(n_pairs);
	for (int p = 0; p < n_pairs; p++) {
		BT_TRY(check_desc(A[p], m, __func__, p));
		BT_TRY(check_desc(B[p], m, __func__, p));
		sa[p] = PoolSetRef{ slot(A[p]), A[p].n }; sb[p] = PoolSetRef{ slot(B[p]), B[p].n };
	}
	BT_REQUIRE((int)sets.size() <= m->n_transient, BT_ERR_CAPACITY, "bt_knn_match_pairs: %d distinct descriptor sets in one call > %d (store them with bt_desc_pool_store and use bt_knn_match_slots)", (int)sets.size(), m->n_transient);
	return knn_run(ctx, __func__, n_pairs, sets, sa.data(), sb.data(), k, out, stream);
}
