// prune.cu — geometric pruning of the kNN candidates, the "mutual" union, and the glue that turns RANSAC inliers into
// EntryJ records — everything SiftManager::findCorres does between the two knnMatch calls and Bundler::optimizeGPU's
// EntryJ loop, kept on the device:
//
//   k_prune_mutual   one CTA per frame pair.  Direction A->B then B->A: for every query feature the FIRST of its k
//                    neighbours passing the gates of SiftManager::pruneMatches (/root/reference/src/FeatureManager.cpp:
//                    290-336: both keypoints round()ed inside the image, both depths >= 0.1, model-frame distance <=
//                    max_dist_*, cos(angle between model-frame normals) >= cos(max_normal_*) or NaN (a zero normal), thresholds chosen by
//                    |idA-idB|==1) is kept; survivors are appended in query order, A->B block first, duplicates NOT
//                    removed — exactly collectMutualMatches (:338-368, a union, SURVEY.md D1).  Also emits the
//                    model-frame points RANSAC consumes (runRansacMultiPairGPU :676-706).
//   k_ransac_table_from_counts / k_emit_entryj
//                    counts -> RANSAC pair table (<= 5 candidates => pair dropped, runRansacBetween :575-579);
//                    inliers -> EntryJ {imgIdx_i = older frame, imgIdx_j = newer frame, pos_i = ptB_cam, pos_j = ptA_cam}
//                    (Bundler::optimizeGPU, /root/reference/src/Bundler.cpp:308-317), < 5 inliers => pair dropped
//                    (FeatureManager.cpp:233-241,727-730); pairs written back to back, which is the grouping the
//                    solver's tail wants.  A list longer than the caller's capacity is cut there; the pair status (OK /
//                    cleared / Frame::FAIL) follows the match outcome, never the cut.
//   tests/test_find_corres_adversarial_gpu.py holds all of these to a float64 restatement (oracle/corres_families.py).
#include <algorithm>
#include <climits>
#include <map>
#include <vector>
#include "bt_common.cuh"
#include "bt_scan.cuh"

namespace bt {

struct RansacPair { const float4* A; const float4* B; int n; int out_off; };   // same layout as in ransac.cu
int ransac_run_device(bt_ctx* ctx, const RansacPair* d_pairs, int n_pairs, int n_trials, float dist_thresh, uint64_t seed,
                      int32_t* inlier_ids_out, int32_t* n_inliers_out, cudaStream_t stream);

struct PruneFrame { const float2* kpts; int n; int frame_id; const float* depth; const float4* normal; float T[12]; };
struct PrunePair { PruneFrame A, B; int idx_off_A, idx_off_B; int out_off; int win_idx_A, win_idx_B; int n_extra, extra_off; };   // extras: propagated (uA,vA,uB,vB) matches, non-neighbour pairs only
struct PruneCam { int H, W; float ifx, ify, icx, icy; };

// One candidate (query q of frame Q, train t of frame Tn).  Returns true when it passes pruneMatches' gates.
__device__ __forceinline__ bool prune_gate(const PruneFrame& Q, const PruneFrame& Tn, int q, int t, const PruneCam& cam, float max_dist, float cos_max,
                                           float (&ptQ)[3], float (&ptT)[3], float (&mQ)[3], float (&mT)[3]) {
	const float2 pq = __ldg(Q.kpts + q), pt = __ldg(Tn.kpts + t);
	const int uq = (int)roundf(pq.x), vq = (int)roundf(pq.y), ut = (int)roundf(pt.x), vt = (int)roundf(pt.y);   // std::round
	if (uq < 0 || vq < 0 || uq >= cam.W || vq >= cam.H || ut < 0 || vt < 0 || ut >= cam.W || vt >= cam.H) return false;   // Utils::isPixelInsideImage
	const float dq = __ldg(Q.depth + (size_t)vq * cam.W + uq), dt = __ldg(Tn.depth + (size_t)vt * cam.W + ut);
	if (!(dq >= 0.1f && dt >= 0.1f)) return false;              // the organised cloud holds zeros wherever !(depth >= 0.1), NaN included
	// Frame::depthToCloudAndNormals: K^-1 (u d, v d, d)   (/root/reference/src/Frame.cpp:199-233, CUDAImageUtil.cu:310-326)
	ptQ[0] = cam.ifx * ((float)uq * dq) + cam.icx * dq; ptQ[1] = cam.ify * ((float)vq * dq) + cam.icy * dq; ptQ[2] = dq;
	ptT[0] = cam.ifx * ((float)ut * dt) + cam.icx * dt; ptT[1] = cam.ify * ((float)vt * dt) + cam.icy * dt; ptT[2] = dt;
	const float4 nq = __ldg(Q.normal + (size_t)vq * cam.W + uq), nt = __ldg(Tn.normal + (size_t)vt * cam.W + ut);
	float wq[3], wt[3];
#pragma unroll
	for (int r = 0; r < 3; r++) {   // pcl::transformPointWithNormal
		mQ[r] = Q.T[r * 4] * ptQ[0] + Q.T[r * 4 + 1] * ptQ[1] + Q.T[r * 4 + 2] * ptQ[2] + Q.T[r * 4 + 3];
		mT[r] = Tn.T[r * 4] * ptT[0] + Tn.T[r * 4 + 1] * ptT[1] + Tn.T[r * 4 + 2] * ptT[2] + Tn.T[r * 4 + 3];
		wq[r] = Q.T[r * 4] * nq.x + Q.T[r * 4 + 1] * nq.y + Q.T[r * 4 + 2] * nq.z;
		wt[r] = Tn.T[r * 4] * nt.x + Tn.T[r * 4 + 1] * nt.y + Tn.T[r * 4 + 2] * nt.z;
	}
	const float dx = mQ[0] - mT[0], dy = mQ[1] - mT[1], dz = mQ[2] - mT[2];
	const float dist = sqrtf(dx * dx + dy * dy + dz * dz);
	// n1.normalized().dot(n2.normalized()): a zero normal normalises to NaN, the `<` test is then false and the
	// candidate is NOT rejected (FeatureManager.cpp:326) — reproduced by the !(dot < cos) form below.
	const float lq = sqrtf(wq[0] * wq[0] + wq[1] * wq[1] + wq[2] * wq[2]), lt = sqrtf(wt[0] * wt[0] + wt[1] * wt[1] + wt[2] * wt[2]);
	const float dotn = (wq[0] / lq) * (wt[0] / lt) + (wq[1] / lq) * (wt[1] / lt) + (wq[2] / lq) * (wt[2] / lt);
	if (dist > max_dist || dotn < cos_max) return false;
	return true;
}

__global__ void __launch_bounds__(512) k_prune_mutual(const PrunePair* __restrict__ pairs, PruneCam cam, const int32_t* __restrict__ idxAB, const int32_t* __restrict__ idxBA,
                                                       int k, bt_prune_params prm, bt_correspondence* __restrict__ corr, float4* __restrict__ PA, float4* __restrict__ PB,
                                                       int32_t* __restrict__ n_corr) {
	__shared__ int s_warp[16];
	__shared__ int s_base;
	const PrunePair pp = pairs[blockIdx.x];
	const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
	const bool neighbor = abs(pp.A.frame_id - pp.B.frame_id) == 1;
	const float max_dist = neighbor ? prm.max_dist_neighbor : prm.max_dist_no_neighbor;
	const float cos_max = neighbor ? prm.cos_max_normal_neighbor : prm.cos_max_normal_no_neighbor;
	if (tid == 0) s_base = 0;
	__syncthreads();
	for (int dir = 0; dir < 2; dir++) {
		const PruneFrame& Q = dir == 0 ? pp.A : pp.B;
		const PruneFrame& Tn = dir == 0 ? pp.B : pp.A;
		const int32_t* idx = (dir == 0 ? idxAB + (size_t)pp.idx_off_A * k : idxBA + (size_t)pp.idx_off_B * k);
		for (int base = 0; base < Q.n; base += blockDim.x) {
			const int q = base + tid;
			bool keep = false;
			float ptQ[3], ptT[3], mQ[3], mT[3];
			int tsel = -1;
			if (q < Q.n && Tn.n > 0) {
				for (int c = 0; c < k; c++) {
					const int t = __ldg(idx + (size_t)q * k + c);
					if (t < 0 || t >= Tn.n) continue;
					if (prune_gate(Q, Tn, q, t, cam, max_dist, cos_max, ptQ, ptT, mQ, mT)) { keep = true; tsel = t; break; }
				}
			}
			const unsigned bal = __ballot_sync(0xffffffffu, keep);
			if (lane == 0) s_warp[wid] = __popc(bal);
			__syncthreads();
			int off = s_base;
			for (int w = 0; w < wid; w++) off += s_warp[w];
			if (keep) {
				const int o = pp.out_off + off + __popc(bal & ((1u << lane) - 1u));
				const float2 kq = __ldg(Q.kpts + q), kt = __ldg(Tn.kpts + tsel);
				bt_correspondence c;
				// Correspondence(uA, vA, uB, vB, ptA, ptB): A is always the pair's first (newer) frame
				if (dir == 0) { c.uA = kq.x; c.vA = kq.y; c.uB = kt.x; c.vB = kt.y; for (int r = 0; r < 3; r++) { c.ptA_cam[r] = ptQ[r]; c.ptB_cam[r] = ptT[r]; } PA[o] = make_float4(mQ[0], mQ[1], mQ[2], 1.f); PB[o] = make_float4(mT[0], mT[1], mT[2], 1.f); }
				else { c.uA = kt.x; c.vA = kt.y; c.uB = kq.x; c.vB = kq.y; for (int r = 0; r < 3; r++) { c.ptA_cam[r] = ptT[r]; c.ptB_cam[r] = ptQ[r]; } PA[o] = make_float4(mT[0], mT[1], mT[2], 1.f); PB[o] = make_float4(mQ[0], mQ[1], mQ[2], 1.f); }
				corr[o] = c;
			}
			__syncthreads();
			if (tid == 0) { int t = 0; for (int w = 0; w < (int)(blockDim.x >> 5); w++) t += s_warp[w]; s_base += t; }
			__syncthreads();
		}
	}
	if (tid == 0) n_corr[blockIdx.x] = s_base;
}

// findCorresByMapPoints (/root/reference/src/FeatureManager.cpp:489-520) on the device, between the mutual union and RANSAC, for the
// NON-neighbour pairs: the caller hands the (uA, vA, uB, vB) of the map points both frames observe (bt_tracks_propagate, in the
// reference's order); a candidate is dropped when an existing match of the pair has the same (uA, vA) or the same (uB, vB), the rest
// are appended in order with the organised-cloud points at round(u), round(v) (zeros where the depth is < 0.1, as the cloud holds them).
__global__ void __launch_bounds__(256) k_append_propagated(const PrunePair* __restrict__ pairs, PruneCam cam, const float4* __restrict__ extra_uv,
                                                            bt_correspondence* __restrict__ corr, float4* __restrict__ PA, float4* __restrict__ PB,
                                                            int32_t* __restrict__ n_corr, int32_t* __restrict__ n_nn, const int32_t* __restrict__ n_extra_dev) {
	__shared__ int s_warp[8];
	__shared__ int s_base;
	const PrunePair pp = pairs[blockIdx.x];
	const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
	const int n0 = n_corr[blockIdx.x];
	if (tid == 0) { n_nn[blockIdx.x] = n0; s_base = n0; }
	__syncthreads();
	const int n_extra = n_extra_dev ? n_extra_dev[blockIdx.x] : pp.n_extra;      // (bt_find_corres_pairs: the count the device table wrote)
	if (n_extra <= 0 || abs(pp.A.frame_id - pp.B.frame_id) == 1) return;
	const bt_correspondence* ex = corr + pp.out_off;
	for (int base = 0; base < n_extra; base += blockDim.x) {
		const int e = base + tid;
		bool keep = false;
		float4 uv = make_float4(0.f, 0.f, 0.f, 0.f);
		if (e < n_extra) {
			uv = __ldg(extra_uv + pp.extra_off + e);
			keep = true;
			for (int i = 0; i < n0; i++) {      // only the matches of the two knnMatch directions are compared: map-point keys are unique per frame
				const bt_correspondence c = ex[i];
				if ((c.uA == uv.x && c.vA == uv.y) || (c.uB == uv.z && c.vB == uv.w)) { keep = false; break; }
			}
		}
		const unsigned bal = __ballot_sync(0xffffffffu, keep);
		if (lane == 0) s_warp[wid] = __popc(bal);
		__syncthreads();
		int off = s_base;
		for (int w = 0; w < wid; w++) off += s_warp[w];
		if (keep) {
			const int o = pp.out_off + off + __popc(bal & ((1u << lane) - 1u));
			bt_correspondence c;
			c.uA = uv.x; c.vA = uv.y; c.uB = uv.z; c.vB = uv.w;
			float pa[3] = { 0.f, 0.f, 0.f }, pb[3] = { 0.f, 0.f, 0.f };
			const int ua = (int)roundf(uv.x), va = (int)roundf(uv.y), ub = (int)roundf(uv.z), vb = (int)roundf(uv.w);
			if (ua >= 0 && va >= 0 && ua < cam.W && va < cam.H) { const float d = __ldg(pp.A.depth + (size_t)va * cam.W + ua); if (d >= 0.1f) { pa[0] = cam.ifx * ((float)ua * d) + cam.icx * d; pa[1] = cam.ify * ((float)va * d) + cam.icy * d; pa[2] = d; } }
			if (ub >= 0 && vb >= 0 && ub < cam.W && vb < cam.H) { const float d = __ldg(pp.B.depth + (size_t)vb * cam.W + ub); if (d >= 0.1f) { pb[0] = cam.ifx * ((float)ub * d) + cam.icx * d; pb[1] = cam.ify * ((float)vb * d) + cam.icy * d; pb[2] = d; } }
			float ma[3], mb[3];
#pragma unroll
			for (int r = 0; r < 3; r++) {
				c.ptA_cam[r] = pa[r]; c.ptB_cam[r] = pb[r];
				ma[r] = pp.A.T[r * 4] * pa[0] + pp.A.T[r * 4 + 1] * pa[1] + pp.A.T[r * 4 + 2] * pa[2] + pp.A.T[r * 4 + 3];
				mb[r] = pp.B.T[r * 4] * pb[0] + pp.B.T[r * 4 + 1] * pb[1] + pp.B.T[r * 4 + 2] * pb[2] + pp.B.T[r * 4 + 3];
			}
			corr[o] = c; PA[o] = make_float4(ma[0], ma[1], ma[2], 1.f); PB[o] = make_float4(mb[0], mb[1], mb[2], 1.f);
		}
		__syncthreads();
		if (tid == 0) { int t = 0; for (int w = 0; w < (int)(blockDim.x >> 5); w++) t += s_warp[w]; s_base += t; }
		__syncthreads();
	}
	if (tid == 0) n_corr[blockIdx.x] = s_base;
}

__global__ void k_ransac_table_from_counts(const PrunePair* __restrict__ pairs, int n_pairs, const int32_t* __restrict__ n_corr, const float4* PA, const float4* PB, RansacPair* out) {
	const int p = blockIdx.x * blockDim.x + threadIdx.x;
	if (p >= n_pairs) return;
	const int n = n_corr[p];
	RansacPair r; r.A = PA + pairs[p].out_off; r.B = PB + pairs[p].out_off;
	r.n = (n <= 5) ? 0 : n;                 // countInlierCorres <= 5 => matches cleared before RANSAC
	r.out_off = pairs[p].out_off;
	out[p] = r;
}

// one CTA: exclusive scan of the kept inlier counts over pairs (pairs stay contiguous in the EntryJ list)
__global__ void __launch_bounds__(1024) k_emit_entryj(const PrunePair* __restrict__ pairs, int n_pairs, const bt_correspondence* __restrict__ corr,
                                                       const int32_t* __restrict__ inlier_ids, const int32_t* __restrict__ n_inliers,
                                                       bt_entryj* __restrict__ entry_out, int32_t* __restrict__ n_entry_out, int32_t* __restrict__ entry_off_out, int32_t* total_out, int capacity,
                                                       int32_t* __restrict__ status_out) {
	__shared__ int s_scan[32];
	__shared__ int s_carry;
	const int tid = threadIdx.x;
	if (tid == 0) s_carry = 0;
	__syncthreads();
	for (int base = 0; base < n_pairs; base += 1024) {
		const int p = base + tid;
		int cnt = 0;
		if (p < n_pairs) { cnt = n_inliers[p]; if (cnt < 5) cnt = 0; }     // fewer than 5 matches => cleared
		int total;
		const int matched = cnt;
		int excl = block_excl_scan(cnt, s_scan, &total) + s_carry;
		// never describe more than the caller's buffer holds: a pair that does not fit is cut (or dropped), so the (offset, count)
		// arrays a caller hands on as bt_window::block_off / block_n always stay inside entry_out
		if (excl > capacity) excl = capacity;
		if (excl + cnt > capacity) cnt = capacity - excl;
		if (p < n_pairs) {
			n_entry_out[p] = cnt; entry_off_out[p] = excl;
			// SiftManager::findCorres' outcome for the pair (FeatureManager.cpp:186-241,282-286): a pair left with fewer than 5 matches is
			// cleared, and when the two frames are neighbours (|idA - idB| == 1) the newer frame is marked Frame::FAIL.  The outcome is the
			// match's, not the buffer's: a pair cut by the capacity keeps its status and shows the cut only in its count
			if (status_out) status_out[p] = matched > 0 ? BT_PAIR_OK : (abs(pairs[p].A.frame_id - pairs[p].B.frame_id) == 1 ? BT_PAIR_FAIL : BT_PAIR_EMPTY);
		}
		__syncthreads();
		if (tid == 1023) s_carry += total;
		__syncthreads();
	}
	if (tid == 0) *total_out = min(s_carry, capacity);
}

// one CTA per pair: its EntryJ block (a lone CTA filling all pairs would serialise the whole list)
__global__ void __launch_bounds__(256) k_emit_fill(const PrunePair* __restrict__ pairs, const bt_correspondence* __restrict__ corr, const int32_t* __restrict__ inlier_ids,
                                                    const int32_t* __restrict__ n_entry, const int32_t* __restrict__ entry_off, bt_entryj* __restrict__ entry_out, int capacity,
                                                    float4* __restrict__ uv_out) {
	const int p = blockIdx.x;
	const int cnt = n_entry[p], off = entry_off[p];
	const PrunePair pp = pairs[p];
	for (int i = threadIdx.x; i < cnt; i += blockDim.x) {
		if (off + i >= capacity) break;
		const bt_correspondence c = corr[pp.out_off + inlier_ids[pp.out_off + i]];
		bt_entryj e;
		e.imgIdx_i = (uint32_t)pp.win_idx_B; e.imgIdx_j = (uint32_t)pp.win_idx_A;          // i = older frame B, j = newer frame A
		for (int r = 0; r < 3; r++) { e.pos_i[r] = c.ptB_cam[r]; e.pos_j[r] = c.ptA_cam[r]; }
		entry_out[off + i] = e;
		if (uv_out) uv_out[off + i] = make_float4(c.uA, c.vA, c.uB, c.vB);
	}
}

struct PruneState {
	bool ready = false;
	int max_pairs = 0, max_feats = 0;
	DevBuf corr, PA, PB, n_corr, n_nn, rpairs, inl, n_inl, idxAB, distAB, idxBA, distBA, entry_off, total, extra, n_prop;
	TableBlock<> pairs;                 // the pair table and the host extras of a call (`extra` holds the ones the device table writes)
	size_t extra_cap = 0;               // propagated matches (float4 each) one call may carry
};
void StateDeleter::operator()(PruneState* s) const { delete s; }
struct PairTables : TableLayout { Slice<PrunePair> pairs; Slice<float4> extra; };
static PairTables pair_tables(size_t n_pairs, size_t n_extra) {
	PairTables t;
	t.pairs = t.add<PrunePair>(n_pairs); t.extra = t.add<float4>(n_extra);
	return t;
}

}  // namespace bt

using namespace bt;

extern "C" int bt_pipeline_reserve(bt_ctx* ctx, int max_pairs, int max_feats, int dim, int max_trials) {
	BT_REQUIRE(ctx && max_pairs > 0 && max_feats > 0 && max_trials > 0, BT_ERR_INVALID_ARG, "bt_pipeline_reserve: bad arguments");
	BT_TRY(matcher_reserve_args(max_pairs, max_feats, dim));
	PruneState* s;
	BT_TRY(take_state(ctx, &bt_ctx::prune, &s));
	BT_TRY(bt_matcher_reserve(ctx, max_pairs, max_feats, dim));
	BT_TRY(bt_ransac_reserve(ctx, max_pairs, 3 * max_feats, max_trials));
	const size_t cap = (size_t)3 * max_feats * max_pairs;      // nA + nB mutual candidates + up to max_feats propagated map-point matches per pair
	const size_t extra_cap = (size_t)max_feats * max_pairs;
	BT_TRY(s->corr.alloc(sizeof(bt_correspondence) * cap));
	BT_TRY(s->PA.alloc(sizeof(float4) * cap)); BT_TRY(s->PB.alloc(sizeof(float4) * cap));
	BT_TRY(s->n_corr.alloc(sizeof(int32_t) * max_pairs)); BT_TRY(s->n_nn.alloc(sizeof(int32_t) * max_pairs));
	BT_TRY(s->extra.alloc(sizeof(float4) * extra_cap));
	BT_TRY(s->rpairs.alloc(sizeof(RansacPair) * max_pairs));
	BT_TRY(s->inl.alloc(sizeof(int32_t) * cap)); BT_TRY(s->n_inl.alloc(sizeof(int32_t) * max_pairs));
	BT_TRY(s->idxAB.alloc(sizeof(int32_t) * 8 * (size_t)max_feats * max_pairs)); BT_TRY(s->distAB.alloc(sizeof(float) * 8 * (size_t)max_feats * max_pairs));
	BT_TRY(s->idxBA.alloc(sizeof(int32_t) * 8 * (size_t)max_feats * max_pairs)); BT_TRY(s->distBA.alloc(sizeof(float) * 8 * (size_t)max_feats * max_pairs));
	BT_TRY(s->entry_off.alloc(sizeof(int32_t) * max_pairs)); BT_TRY(s->total.alloc(16)); BT_TRY(s->n_prop.alloc(sizeof(int32_t) * max_pairs));
	BT_TRY(s->pairs.reserve(pair_tables(max_pairs, extra_cap).total));
	s->max_pairs = max_pairs; s->max_feats = max_feats; s->extra_cap = extra_cap;
	s->ready = true;
	return BT_OK;
}

namespace {
// One findCorres call on the context's scratch: each stage of kNN -> prune -> mutual union (+ propagated matches) -> RANSAC -> EntryJ is
// launched by one method.  prune() reads knn()'s lists and writes corr / n_corr; bt_prune_mutual_pairs points both at the caller's arrays.
struct Chain {
	bt_ctx* ctx;
	PruneState* s;
	const char* who;                    // the entry point, for its messages
	int n, trials;                      // pairs, RANSAC trials
	const bt_match_frame *A, *B;
	PruneCam cam;
	const bt_prune_params* prm;
	float inlier_dist;
	uint64_t seed;
	cudaStream_t stream;
	const int32_t *idxAB = nullptr, *idxBA = nullptr;
	int k = 0;
	bt_correspondence* corr;
	int32_t* n_corr;
	const PrunePair *h_pairs = nullptr, *d_pairs = nullptr;    // the pair table on the host and on the device, once pairs() has uploaded it
	const float4* d_extra = nullptr;                            // the propagated matches on the device
	Chain(bt_ctx* ctx_, const char* who_, int n_pairs, const bt_match_frame* A_, const bt_match_frame* B_, int H, int W, float fx, float fy, float cx, float cy,
	      const bt_prune_params* prm_, int trials_, float inlier_dist_, uint64_t seed_, void* stream_)
	    : ctx(ctx_), s(ctx_->prune.get()), who(who_), n(n_pairs), trials(trials_), A(A_), B(B_), cam{ H, W, 1.0f / fx, 1.0f / fy, -cx / fx, -cy / fy },
	      prm(prm_), inlier_dist(inlier_dist_), seed(seed_), stream((cudaStream_t)stream_), corr(s->corr.as<bt_correspondence>()), n_corr(s->n_corr.as<int32_t>()) {}
	// both directions, from descriptor views or from descriptor-pool slots: exactly one of the two is given
	int knn(const bt_desc_view* dA, const bt_desc_view* dB, const int32_t* slotA, const int32_t* slotB) {
		BT_REQUIRE(((dA && dB) ? 1 : 0) + ((slotA && slotB) ? 1 : 0) == 1, BT_ERR_INVALID_ARG, "%s: give either descriptor views or pool slots", who);
		k = 5;   // k_near, FeatureManager.cpp:264
		idxAB = s->idxAB.as<int32_t>(); idxBA = s->idxBA.as<int32_t>();
		return dA ? bt_knn_match_pairs(ctx, n, dA, dB, k, s->idxAB.as<int32_t>(), s->distAB.as<float>(), s->idxBA.as<int32_t>(), s->distBA.as<float>(), stream)
		          : bt_knn_match_slots(ctx, n, slotA, slotB, k, s->idxAB.as<int32_t>(), s->distAB.as<float>(), s->idxBA.as<int32_t>(), s->distBA.as<float>(), stream);
	}
	// the pair table, uploaded with the host extras.  prop_room > 0 (bt_find_corres_pairs): no host extras; pair p keeps room for prop_room
	// propagated matches behind its mutual ones, and its candidates go to extra[p * prop_room, ...) when the device table writes them
	int pairs(const bt_match_extra* extra, int prop_room) {
		// the host extras pairs carry: counted and checked first, so that the table block can be laid out
		auto n_extra = [&](int p) { return (extra && extra[p].n > 0 && abs(A[p].frame_id - B[p].frame_id) != 1) ? extra[p].n : 0; };
		size_t n_x = 0;
		for (int p = 0; p < n; p++) {
			const int nx = n_extra(p);
			BT_REQUIRE(nx == 0 || extra[p].uv, BT_ERR_INVALID_ARG, "pair %d: NULL propagated-match array", p);
			BT_REQUIRE(nx <= s->max_feats && n_x + nx <= s->extra_cap, BT_ERR_CAPACITY, "pair %d: %d propagated matches exceed the reserved room", p, nx);
			n_x += nx;
		}
		const PairTables t = pair_tables(n, n_x);
		BT_TRY(s->pairs.begin(who, t));
		PrunePair* hp = s->pairs.host(t.pairs);
		float4* hx = s->pairs.host(t.extra);
		int offA = 0, offB = 0, out = 0, xoff = 0;
		for (int p = 0; p < n; p++) {
			const bt_match_frame* fr[2] = { &A[p], &B[p] };
			PruneFrame* dst[2] = { &hp[p].A, &hp[p].B };
			for (int s2 = 0; s2 < 2; s2++) {
				BT_REQUIRE(fr[s2]->n >= 0 && fr[s2]->n <= s->max_feats, BT_ERR_CAPACITY, "pair %d: %d features > reserved %d", p, fr[s2]->n, s->max_feats);
				BT_REQUIRE(fr[s2]->n == 0 || (fr[s2]->kpts_dev && fr[s2]->depth_dev && fr[s2]->normal_dev), BT_ERR_INVALID_ARG, "pair %d: NULL frame pointer", p);
				dst[s2]->kpts = reinterpret_cast<const float2*>(fr[s2]->kpts_dev); dst[s2]->n = fr[s2]->n; dst[s2]->frame_id = fr[s2]->frame_id;
				dst[s2]->depth = fr[s2]->depth_dev; dst[s2]->normal = reinterpret_cast<const float4*>(fr[s2]->normal_dev);
				memcpy(dst[s2]->T, fr[s2]->pose, sizeof(float) * 12);
			}
			hp[p].idx_off_A = offA; hp[p].idx_off_B = offB; hp[p].out_off = out;
			hp[p].win_idx_A = A[p].window_index; hp[p].win_idx_B = B[p].window_index;
			const int nx = n_extra(p);
			hp[p].n_extra = nx; hp[p].extra_off = prop_room ? p * prop_room : xoff;
			if (nx) memcpy(hx + xoff, extra[p].uv, sizeof(float4) * (size_t)nx);
			xoff += nx;
			offA += A[p].n; offB += B[p].n; out += A[p].n + B[p].n + nx + prop_room;
		}
		BT_TRY(s->pairs.send(0, xoff ? t.extra.end() : t.pairs.end(), stream));
		h_pairs = hp; d_pairs = s->pairs.dev(t.pairs);
		d_extra = prop_room ? s->extra.as<float4>() : s->pairs.dev(t.extra);
		return s->pairs.in_flight(stream);
	}
	int prune() {
		k_prune_mutual<<<n, 512, 0, stream>>>(d_pairs, cam, idxAB, idxBA, k, *prm, corr, s->PA.as<float4>(), s->PB.as<float4>(), n_corr);
		BT_CUDA(cudaGetLastError());
		return BT_OK;
	}
	// findCorresByMapPoints for pairs [p0, p0 + np), with the pair table's counts or, given n_extra_dev, the ones the device table wrote
	int append(int p0, int np, const int32_t* n_extra_dev) {
		k_append_propagated<<<np, 256, 0, stream>>>(d_pairs + p0, cam, d_extra, corr, s->PA.as<float4>(), s->PB.as<float4>(), n_corr + p0,
		                                            s->n_nn.as<int32_t>() + p0, n_extra_dev);
		BT_CUDA(cudaGetLastError());
		return BT_OK;
	}
	int ransac(int p0, int np) {
		RansacPair* rp = s->rpairs.as<RansacPair>() + p0;
		k_ransac_table_from_counts<<<(np + 127) / 128, 128, 0, stream>>>(d_pairs + p0, np, n_corr + p0, s->PA.as<float4>(), s->PB.as<float4>(), rp);
		BT_CUDA(cudaGetLastError());
		return ransac_run_device(ctx, rp, np, trials, inlier_dist, seed, s->inl.as<int32_t>(), s->n_inl.as<int32_t>() + p0, stream);
	}
	int emit(bt_entryj* entry_out, int capacity, int32_t* n_entry_out, int32_t* entry_off_out, int32_t* total_out, int32_t* status_out, float* uv_out) {
		k_emit_entryj<<<1, 1024, 0, stream>>>(d_pairs, n, corr, s->inl.as<int32_t>(), s->n_inl.as<int32_t>(), entry_out, n_entry_out, entry_off_out, total_out, capacity, status_out);
		k_emit_fill<<<n, 256, 0, stream>>>(d_pairs, corr, s->inl.as<int32_t>(), n_entry_out, entry_off_out, entry_out, capacity, reinterpret_cast<float4*>(uv_out));
		BT_CUDA(cudaGetLastError());
		return BT_OK;
	}
};
}  // namespace

extern "C" int bt_prune_mutual_pairs(bt_ctx* ctx, int n_pairs, const bt_match_frame* A, const bt_match_frame* B, int H, int W, float fx, float fy, float cx, float cy,
                                     const int32_t* idxAB, const int32_t* idxBA, int k, const bt_prune_params* prm,
                                     bt_correspondence* corr_out, int32_t* n_corr_out, void* stream_) {
	PruneState* s;
	BT_TRY(state_of(ctx, &bt_ctx::prune, "bt_prune_mutual_pairs", "bt_pipeline_reserve", &s));
	BT_REQUIRE(A && B && idxAB && idxBA && prm && corr_out && n_corr_out && n_pairs > 0 && n_pairs <= s->max_pairs && k >= 1 && k <= 8, BT_ERR_INVALID_ARG, "bt_prune_mutual_pairs: bad argument");
	Chain c(ctx, "bt_prune_mutual_pairs", n_pairs, A, B, H, W, fx, fy, cx, cy, prm, 0, 0.f, 0, stream_);
	c.idxAB = idxAB; c.idxBA = idxBA; c.k = k;
	c.corr = corr_out; c.n_corr = n_corr_out;
	BT_TRY(c.pairs(nullptr, 0));
	BT_TRY(c.prune());
	return c.append(0, n_pairs, nullptr);
}

extern "C" int bt_match_pairs(bt_ctx* ctx, int n_pairs, const bt_match_frame* A, const bt_match_frame* B, const bt_desc_view* dA, const bt_desc_view* dB,
                              int H, int W, float fx, float fy, float cx, float cy, const bt_prune_params* prune, int ransac_trials, float ransac_inlier_dist,
                              uint64_t ransac_seed, bt_entryj* entry_out, int entry_capacity, int32_t* n_entry_out, int32_t* entry_off_out, int32_t* total_out, void* stream_) {
	BT_REQUIRE(dA && dB, BT_ERR_INVALID_ARG, "bt_match_pairs: NULL descriptor views");
	return bt_match_pairs_ex(ctx, n_pairs, A, B, dA, dB, nullptr, nullptr, H, W, fx, fy, cx, cy, prune, ransac_trials, ransac_inlier_dist, ransac_seed, nullptr, entry_out, entry_capacity, n_entry_out, entry_off_out, total_out, nullptr, nullptr, stream_);
}

extern "C" int bt_match_pairs_pool(bt_ctx* ctx, int n_pairs, const bt_match_frame* A, const bt_match_frame* B, const int32_t* slotA, const int32_t* slotB,
                                   int H, int W, float fx, float fy, float cx, float cy, const bt_prune_params* prune, int ransac_trials, float ransac_inlier_dist,
                                   uint64_t ransac_seed, bt_entryj* entry_out, int entry_capacity, int32_t* n_entry_out, int32_t* entry_off_out, int32_t* total_out, void* stream_) {
	BT_REQUIRE(slotA && slotB, BT_ERR_INVALID_ARG, "bt_match_pairs_pool: NULL slot arrays");
	return bt_match_pairs_ex(ctx, n_pairs, A, B, nullptr, nullptr, slotA, slotB, H, W, fx, fy, cx, cy, prune, ransac_trials, ransac_inlier_dist, ransac_seed, nullptr, entry_out, entry_capacity, n_entry_out, entry_off_out, total_out, nullptr, nullptr, stream_);
}

// SiftManager::findCorres (FeatureManager.cpp:173-242) for a batch of pairs, device-resident end to end, with the propagated map-point matches
// of the non-neighbour pairs, the pair status (OK / cleared / Frame::FAIL) and the (uA, vA, uB, vB) of every emitted entry (what
// updateFramePairMapPoints needs).  Pair p's entries are contiguous in entry_out.  bt_match_pairs and bt_match_pairs_pool are this call.
extern "C" int bt_match_pairs_ex(bt_ctx* ctx, int n_pairs, const bt_match_frame* A, const bt_match_frame* B, const bt_desc_view* dA, const bt_desc_view* dB,
                                 const int32_t* slotA, const int32_t* slotB, int H, int W, float fx, float fy, float cx, float cy, const bt_prune_params* prune,
                                 int ransac_trials, float ransac_inlier_dist, uint64_t ransac_seed, const bt_match_extra* extra,
                                 bt_entryj* entry_out, int entry_capacity, int32_t* n_entry_out, int32_t* entry_off_out, int32_t* total_out, int32_t* status_out, float* uv_out, void* stream_) {
	PruneState* s;
	BT_TRY(state_of(ctx, &bt_ctx::prune, "bt_match_pairs", "bt_pipeline_reserve", &s));
	BT_REQUIRE(A && B && prune && entry_out && n_entry_out && entry_off_out && total_out && n_pairs > 0 && n_pairs <= s->max_pairs, BT_ERR_INVALID_ARG, "bt_match_pairs: bad argument");
	Chain c(ctx, "bt_match_pairs_ex", n_pairs, A, B, H, W, fx, fy, cx, cy, prune, ransac_trials, ransac_inlier_dist, ransac_seed, stream_);
	BT_TRY(c.knn(dA, dB, slotA, slotB));
	BT_TRY(c.pairs(extra, 0));
	BT_TRY(c.prune());
	BT_TRY(c.append(0, n_pairs, nullptr));
	BT_TRY(c.ransac(0, n_pairs));
	return c.emit(entry_out, entry_capacity, n_entry_out, entry_off_out, total_out, status_out, uv_out);
}

// Bundler::optimizeGPU's findCorres loop (/root/reference/src/Bundler.cpp:298-305) in one asynchronous call: the pairs are matched in the
// given order against the context's device map-point table (bt_tracks_dev_*), so a pair's propagated matches see the map points every
// earlier pair of the call created or extended.  kNN, prune and the mutual union do not read the table and run batched; then per pair:
// propagate (non-neighbour pairs) -> RANSAC -> update the table from the emitted entries.  The EntryJ list is written once at the end.
extern "C" int bt_find_corres_pairs(bt_ctx* ctx, int n_pairs, const bt_match_frame* A, const bt_match_frame* B, const bt_desc_view* dA, const bt_desc_view* dB,
                                    const int32_t* slotA, const int32_t* slotB, int H, int W, float fx, float fy, float cx, float cy, const bt_prune_params* prune,
                                    int ransac_trials, float ransac_inlier_dist, uint64_t ransac_seed, bt_entryj* entry_out, int entry_capacity,
                                    int32_t* n_entry_out, int32_t* entry_off_out, int32_t* total_out, int32_t* status_out, float* uv_out, void* stream_) {
	PruneState* s;
	BT_TRY(state_of(ctx, &bt_ctx::prune, "bt_find_corres_pairs", "bt_pipeline_reserve", &s));
	BT_TRY(tracks_state(ctx, "bt_find_corres_pairs"));
	BT_REQUIRE(A && B && prune && entry_out && entry_capacity >= 0 && n_entry_out && entry_off_out && total_out && n_pairs > 0 && n_pairs <= s->max_pairs,
	           BT_ERR_INVALID_ARG, "bt_find_corres_pairs: bad argument");
	std::vector<int> fresh;   // frame A is the newer frame of every pair; the frames that are new to the table must fit before anything is queued
	for (int p = 0; p < n_pairs; p++) {
		BT_REQUIRE(A[p].frame_id > B[p].frame_id, BT_ERR_INVALID_ARG, "bt_find_corres_pairs: pair %d: frame A must be the newer frame (id %d <= %d)", p, A[p].frame_id, B[p].frame_id);
		for (int id : { A[p].frame_id, B[p].frame_id }) {
			int sl;
			tracks_slot(ctx, id, false, &sl);
			if (sl < 0 && std::find(fresh.begin(), fresh.end(), id) == fresh.end()) fresh.push_back(id);
		}
	}
	BT_REQUIRE((int)fresh.size() <= tracks_free_slots(ctx), BT_ERR_CAPACITY, "bt_find_corres_pairs: %d new frames do not fit the map-point table", (int)fresh.size());
	Chain c(ctx, "bt_find_corres_pairs", n_pairs, A, B, H, W, fx, fy, cx, cy, prune, ransac_trials, ransac_inlier_dist, ransac_seed, stream_);
	BT_TRY(c.knn(dA, dB, slotA, slotB));
	BT_TRY(c.pairs(nullptr, s->max_feats));
	BT_TRY(c.prune());
	for (int p = 0; p < n_pairs; p++) {
		int sa, sb;
		if (abs(A[p].frame_id - B[p].frame_id) != 1) {       // findCorresByMapPoints
			tracks_slot(ctx, A[p].frame_id, false, &sa);
			tracks_slot(ctx, B[p].frame_id, false, &sb);
			if (sa >= 0 && sb >= 0) {
				int32_t* n_prop = s->n_prop.as<int32_t>() + p;
				BT_TRY(tracks_launch_propagate(ctx, sa, sb, nullptr, 0, s->extra.as<float4>() + (size_t)p * s->max_feats, s->max_feats, n_prop, c.stream));
				BT_TRY(c.append(p, 1, n_prop));
			}
		}
		BT_TRY(c.ransac(p, 1));
		// updateFramePairMapPoints on the entries the pair emits (none unless its status is OK)
		BT_TRY(tracks_slot(ctx, A[p].frame_id, true, &sa));
		BT_TRY(tracks_slot(ctx, B[p].frame_id, true, &sb));
		const int off = c.h_pairs[p].out_off;
		BT_TRY(tracks_launch_update(ctx, sa, sb, TrkSrc{ reinterpret_cast<const float*>(c.corr + off), (int)(sizeof(bt_correspondence) / sizeof(float)),
		                                                 s->inl.as<int32_t>() + off, nullptr, 0, s->n_inl.as<int32_t>(), p, entry_capacity }, c.stream));
	}
	return c.emit(entry_out, entry_capacity, n_entry_out, entry_off_out, total_out, status_out, uv_out);
}

// ------------------------------------------------------------------------------------------------ per-pair result cache
// SiftManager::_matches (/root/reference/src/FeatureManager.cpp:176): a pair is matched once; later windows reuse its matches.  The
// EntryJ blocks stay on the device in one arena, each block exactly as long as its pair's entry count; the host keeps {offset, count,
// status} per (idA, idB).  Blocks are placed at the arena's top; a forgotten block's entries leave the live count at once and its room is
// reclaimed when a put finds no room at the top: the live blocks then slide down, in offset order, to the arena's start (k_cache_compact),
// on the put's stream and before the put's own copy.
namespace bt {
struct CacheMove { int src, dst, n; uint32_t wi, wj; };      // entries [src, src+n) -> [dst, dst+n); gather rewrites the frame indices
__global__ void __launch_bounds__(128) k_cache_move(const CacheMove* __restrict__ tab, const bt_entryj* __restrict__ from, bt_entryj* __restrict__ to, int rewrite) {
	const CacheMove m = tab[blockIdx.x];
	for (int i = threadIdx.x; i < m.n; i += blockDim.x) {
		bt_entryj e = from[m.src + i];
		if (rewrite) { e.imgIdx_i = m.wi; e.imgIdx_j = m.wj; }
		to[m.dst + i] = e;
	}
}
// In-place compaction: the moves are in ascending source order and every dst <= src, so a block's destination never reaches a source that is
// still to be read - provided each chunk is read completely before it is written.  One CTA; compaction is rare (only when the top is full).
constexpr int kCompactThreads = 1024, kCompactUnroll = 4;
__global__ void __launch_bounds__(kCompactThreads) k_cache_compact(const CacheMove* __restrict__ tab, int n_moves, bt_entryj* arena) {
	for (int k = 0; k < n_moves; k++) {
		const CacheMove m = tab[k];
		if (m.src == m.dst) continue;
		for (int base = 0; base < m.n; base += kCompactThreads * kCompactUnroll) {
			bt_entryj e[kCompactUnroll];
#pragma unroll
			for (int u = 0; u < kCompactUnroll; u++) {
				const int i = base + u * kCompactThreads + threadIdx.x;
				if (i < m.n) e[u] = arena[m.src + i];
			}
			__syncthreads();
#pragma unroll
			for (int u = 0; u < kCompactUnroll; u++) {
				const int i = base + u * kCompactThreads + threadIdx.x;
				if (i < m.n) arena[m.dst + i] = e[u];
			}
			__syncthreads();
		}
	}
}
struct MatchCache {
	bool ready = false;
	int max_pairs = 0, max_block = 0;  // pairs cached at once; entries per block (the arena size for bt_match_cache_reserve_entries)
	long long cap = 0, top = 0, live = 0;   // arena entries: size, end of the last block placed, entries in live blocks
	DevBuf arena;
	TableBlock<2> moves;                // a call waits only for the upload of the call before last
	struct Rec { long long off; int n, status; };
	std::map<std::pair<int, int>, Rec> recs;
};
void StateDeleter::operator()(MatchCache* c) const { delete c; }
struct MoveTable : TableLayout { Slice<CacheMove> moves; };
static MoveTable move_table(size_t n) { MoveTable t; t.moves = t.add<CacheMove>(n); return t; }
// the moves of a call on the device
static int cache_upload(MatchCache* c, const char* who, const std::vector<CacheMove>& mv, cudaStream_t stream, const CacheMove** dev) {
	const MoveTable t = move_table(mv.size());
	BT_TRY(c->moves.begin(who, t));
	memcpy(c->moves.host(t.moves), mv.data(), sizeof(CacheMove) * mv.size());
	BT_TRY(c->moves.send(0, t.moves.end(), stream));
	*dev = c->moves.dev(t.moves);
	return c->moves.in_flight(stream);
}
static int cache_reserve(bt_ctx* ctx, int max_pairs_cached, int max_block, long long total) {
	MatchCache* c;
	BT_TRY(take_state(ctx, &bt_ctx::mcache, &c));
	BT_TRY(c->arena.alloc(sizeof(bt_entryj) * (size_t)total));
	// a put uploads the compaction (every live block) and its own blocks in one table
	BT_TRY(c->moves.reserve(move_table(2 * (size_t)max_pairs_cached).total));
	c->max_pairs = max_pairs_cached; c->max_block = max_block;
	c->cap = total; c->top = 0; c->live = 0;
	c->recs.clear();
	c->ready = true;
	return BT_OK;
}
}  // namespace bt

extern "C" int bt_match_cache_reserve(bt_ctx* ctx, int max_pairs_cached, int max_entries_per_pair) {
	BT_REQUIRE(ctx && max_pairs_cached > 0 && max_entries_per_pair > 0, BT_ERR_INVALID_ARG, "bt_match_cache_reserve: bad arguments");
	return cache_reserve(ctx, max_pairs_cached, max_entries_per_pair, (long long)max_pairs_cached * max_entries_per_pair);
}

extern "C" int bt_match_cache_reserve_entries(bt_ctx* ctx, int max_pairs_cached, long long max_entries_total) {
	BT_REQUIRE(ctx && max_pairs_cached > 0 && max_entries_total > 0 && max_entries_total <= INT_MAX, BT_ERR_INVALID_ARG,
	           "bt_match_cache_reserve_entries: need max_pairs_cached > 0 and 0 < max_entries_total <= %d", INT_MAX);
	return cache_reserve(ctx, max_pairs_cached, (int)max_entries_total, max_entries_total);
}

extern "C" int bt_match_cache_put(bt_ctx* ctx, int n_pairs, const int32_t* idA, const int32_t* idB, const bt_entryj* entry_dev,
                                  const int32_t* n_entry_host, const int32_t* entry_off_host, const int32_t* status_host, void* stream_) {
	MatchCache* c;
	BT_TRY(state_of(ctx, &bt_ctx::mcache, "bt_match_cache_put", "bt_match_cache_reserve", &c));
	BT_REQUIRE(idA && idB && n_entry_host && entry_off_host && n_pairs > 0, BT_ERR_INVALID_ARG, "bt_match_cache_put: NULL argument");
	BT_REQUIRE(n_pairs <= c->max_pairs, BT_ERR_CAPACITY, "bt_match_cache_put: %d pairs > table of %d", n_pairs, c->max_pairs);
	// check everything before changing anything: a refused put leaves the cache as it was.  A pair listed twice keeps its last block.
	std::map<std::pair<int, int>, int> last;            // pair -> index of its last occurrence in the list
	for (int p = 0; p < n_pairs; p++) {
		BT_REQUIRE(idA[p] > idB[p], BT_ERR_INVALID_ARG, "bt_match_cache_put: pair %d: frame A must be the newer frame", p);
		BT_REQUIRE(n_entry_host[p] >= 0 && n_entry_host[p] <= c->max_block, BT_ERR_CAPACITY, "bt_match_cache_put: pair %d has %d entries > block limit %d", p, n_entry_host[p], c->max_block);
		BT_REQUIRE(n_entry_host[p] == 0 || entry_dev, BT_ERR_INVALID_ARG, "bt_match_cache_put: NULL entry list");
		last[std::make_pair((int)idA[p], (int)idB[p])] = p;
	}
	int new_pairs = 0;
	long long live = c->live, need = 0;
	for (const auto& kv : last) {
		const auto it = c->recs.find(kv.first);
		if (it == c->recs.end()) new_pairs++;
		else live -= it->second.n;
		live += n_entry_host[kv.second];
		need += n_entry_host[kv.second];
	}
	BT_REQUIRE((long long)c->recs.size() + new_pairs <= c->max_pairs, BT_ERR_CAPACITY, "bt_match_cache_put: more than %d pairs cached", c->max_pairs);
	BT_REQUIRE(live <= c->cap, BT_ERR_CAPACITY, "bt_match_cache_put: %lld live entries > the cache's %lld", live, c->cap);
	for (const auto& kv : last) {                       // a re-put pair gives its old block back
		const auto it = c->recs.find(kv.first);
		if (it != c->recs.end()) { c->live -= it->second.n; c->recs.erase(it); }
	}
	std::vector<CacheMove> mv;
	if (c->top + need > c->cap) {                       // no room at the top: slide the live blocks down in offset order
		std::vector<MatchCache::Rec*> by_off;
		by_off.reserve(c->recs.size());
		for (auto& kv : c->recs) if (kv.second.n > 0) by_off.push_back(&kv.second);
		std::sort(by_off.begin(), by_off.end(), [](const MatchCache::Rec* a, const MatchCache::Rec* b) { return a->off < b->off; });
		long long off = 0;
		for (MatchCache::Rec* r : by_off) {
			mv.push_back(CacheMove{ (int)r->off, (int)off, r->n, 0u, 0u });
			r->off = off;
			off += r->n;
		}
		c->top = off;
	}
	const int n_compact = (int)mv.size();
	for (int p = 0; p < n_pairs; p++) {
		const auto key = std::make_pair((int)idA[p], (int)idB[p]);
		if (last[key] != p) continue;
		const int n = n_entry_host[p];
		c->recs[key] = MatchCache::Rec{ c->top, n, status_host ? status_host[p] : (n > 0 ? BT_PAIR_OK : BT_PAIR_EMPTY) };
		if (n > 0) mv.push_back(CacheMove{ entry_off_host[p], (int)c->top, n, 0u, 0u });
		c->top += n;
		c->live += n;
	}
	if (mv.empty()) return BT_OK;
	cudaStream_t stream = (cudaStream_t)stream_;
	const CacheMove* d_mv;
	BT_TRY(cache_upload(c, "bt_match_cache_put", mv, stream, &d_mv));
	if (n_compact > 0) k_cache_compact<<<1, kCompactThreads, 0, stream>>>(d_mv, n_compact, c->arena.as<bt_entryj>());
	if ((int)mv.size() > n_compact)
		k_cache_move<<<(unsigned)mv.size() - n_compact, 128, 0, stream>>>(d_mv + n_compact, entry_dev, c->arena.as<bt_entryj>(), 0);
	BT_CUDA(cudaGetLastError());
	return BT_OK;
}

extern "C" int bt_match_cache_has(bt_ctx* ctx, int idA, int idB) {
	BT_REQUIRE(ctx, BT_ERR_INVALID_ARG, "bt_match_cache_has: ctx is NULL");
	if (!ctx->mcache) return 0;        // (nothing cached before the first reserve)
	MatchCache* c;
	BT_TRY(state_of(ctx, &bt_ctx::mcache, "bt_match_cache_has", "bt_match_cache_reserve", &c));
	return c->recs.count(std::make_pair(idA, idB)) ? 1 : 0;
}

extern "C" int bt_match_cache_status(bt_ctx* ctx, int idA, int idB, int* n_entry, int* status) {
	MatchCache* c;
	BT_TRY(state_of(ctx, &bt_ctx::mcache, "bt_match_cache_status", "bt_match_cache_reserve", &c));
	const auto it = c->recs.find(std::make_pair(idA, idB));
	BT_REQUIRE(it != c->recs.end(), BT_ERR_INVALID_ARG, "bt_match_cache_status: pair (%d, %d) is not cached", idA, idB);
	if (n_entry) *n_entry = it->second.n;
	if (status) *status = it->second.status;
	return BT_OK;
}

extern "C" int bt_match_cache_usage(bt_ctx* ctx, int* n_pairs, long long* n_entries) {
	MatchCache* c;
	BT_TRY(state_of(ctx, &bt_ctx::mcache, "bt_match_cache_usage", "bt_match_cache_reserve", &c));
	BT_REQUIRE(n_pairs && n_entries, BT_ERR_INVALID_ARG, "bt_match_cache_usage: NULL argument");
	*n_pairs = (int)c->recs.size();
	*n_entries = c->live;
	return BT_OK;
}

extern "C" int bt_match_cache_gather(bt_ctx* ctx, int n_pairs, const int32_t* idA, const int32_t* idB, const uint32_t* win_i, const uint32_t* win_j,
                                     bt_entryj* dst_dev, int capacity, int32_t* block_off_host, int32_t* block_n_host, void* stream_) {
	MatchCache* c;
	BT_TRY(state_of(ctx, &bt_ctx::mcache, "bt_match_cache_gather", "bt_match_cache_reserve", &c));
	BT_REQUIRE(idA && idB && win_i && win_j && dst_dev && block_off_host && block_n_host && n_pairs > 0, BT_ERR_INVALID_ARG, "bt_match_cache_gather: NULL argument");
	BT_REQUIRE(n_pairs <= c->max_pairs, BT_ERR_CAPACITY, "bt_match_cache_gather: %d pairs > table of %d", n_pairs, c->max_pairs);
	std::vector<CacheMove> mv;
	int off = 0;
	for (int p = 0; p < n_pairs; p++) {
		const auto it = c->recs.find(std::make_pair((int)idA[p], (int)idB[p]));
		BT_REQUIRE(it != c->recs.end(), BT_ERR_INVALID_ARG, "bt_match_cache_gather: pair (%d, %d) is not cached", idA[p], idB[p]);
		const int n = it->second.n;
		BT_REQUIRE(off + n <= capacity, BT_ERR_CAPACITY, "bt_match_cache_gather: %d entries > capacity %d", off + n, capacity);
		block_off_host[p] = off; block_n_host[p] = n;
		if (n > 0) mv.push_back(CacheMove{ (int)it->second.off, off, n, win_i[p], win_j[p] });
		off += n;
	}
	if (mv.empty()) return BT_OK;
	cudaStream_t stream = (cudaStream_t)stream_;
	const CacheMove* d_mv;
	BT_TRY(cache_upload(c, "bt_match_cache_gather", mv, stream, &d_mv));
	k_cache_move<<<(unsigned)mv.size(), 128, 0, stream>>>(d_mv, c->arena.as<bt_entryj>(), dst_dev, 1);
	BT_CUDA(cudaGetLastError());
	return BT_OK;
}

extern "C" int bt_match_cache_forget_frame(bt_ctx* ctx, int frame_id) {
	MatchCache* c;
	BT_TRY(state_of(ctx, &bt_ctx::mcache, "bt_match_cache_forget_frame", "bt_match_cache_reserve", &c));
	for (auto it = c->recs.begin(); it != c->recs.end();) {
		if (it->first.first == frame_id || it->first.second == frame_id) { c->live -= it->second.n; it = c->recs.erase(it); }
		else ++it;
	}
	return BT_OK;
}
