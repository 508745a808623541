// tracks_dev.cu — the map-point table of tracks.cu on the device, owned by the context, so that SiftManager::findCorres can run a whole
// list of dependent frame pairs without a host round trip (bt_find_corres_pairs in prune.cu).  Same rules, same results as bt_tracks:
//   SiftManager::updateFramePairMapPoints   /root/reference/src/FeatureManager.cpp:448-485
//   SiftManager::findCorresByMapPoints      /root/reference/src/FeatureManager.cpp:489-520
//   SiftManager::forgetFrame (map points)   /root/reference/src/FeatureManager.cpp:163-169
//
// Layout (every capacity fixed by bt_tracks_dev_reserve / _ex; nothing is allocated on the call path):
//   frame slot f (the host maps frame ids to slots):  keys[f][0, n_keys[f])  {u bits, v bits, point id, 0} in insertion order, the bits
//                          the key was FIRST inserted with; an open-addressing hash (normalised key -> index into keys[f]).  A key is
//                          normalised by turning -0 into +0, so keys compare as floats compare, as std::map<std::pair<float,float>> does.
//   point p:               obs[f][p] = (u, v) of its observation in slot f (the bits last assigned), or the all-ones pattern (a NaN key,
//                          which never occurs) where the point is not seen in slot f; n_obs[p] = how many slots see it.  Slot-major, so
//                          forget reads one slot's column contiguously.  A point whose count drops to 0 (forget) is unreferenced - no
//                          frame map can point at it - and its id is reused; `created` still counts every point ever made, as the host's
//                          vector does.  The observations take max_points x max_frames x 8 B.
// A capacity overflow never writes: the kernel leaves the table as it was and latches a flag that bt_tracks_dev_stats reports.
//
// k_trk_update applies one pair's list with the order dependence resolved in closed form.  Walking the list in order, entry i is skipped
// iff kA is in A's map AND kB is in B's map "as of entry i".  A key not in the map at the start is inserted by its FIRST occurrence in the
// list (that entry cannot be skipped), so "present as of i" = present at the start || i is not the key's first occurrence.  B's map only
// gains keys (new points); A's map gets the LAST non-skipped entry's id per key, the key bits of the occurrence that inserted it; a point's
// observation in A is the kA of the last non-skipped entry that names the point.  Every step is then a parallel pass.
#include <map>
#include <vector>
#include "bt_common.cuh"
#include "bt_scan.cuh"

namespace bt {

static constexpr unsigned long long kTrkEmpty = ~0ull;   // normalised (NaN, NaN): never a key
static constexpr int kTrkThreads = 1024;
static constexpr int kTrkMaxFrames = 64;                  // bt_tracks_dev_reserve's documented range
static constexpr int kTrkMaxFramesEx = 64 + 1024;         // bt_tracks_dev_reserve_ex: a tracker's frames alive plus its largest keyframe pool
static constexpr int kTrkMaxKeys = 8192;                  // propagate sorts a frame's keys in shared memory

struct TrkTable {
	int4* keys;                    // [max_frames][max_keys]
	unsigned long long* hkey;      // [max_frames][hcap] normalised key or kTrkEmpty
	int* hidx;                     // [max_frames][hcap] index into keys
	int* n_keys;                   // [max_frames]
	float2* obs;                   // [max_frames][max_points], kTrkEmpty bits where the point is not seen in the slot
	int* n_obs;                    // [max_points] slots that see the point
	unsigned long long* last;      // [max_points] (epoch << 32 | entry) of the last writer of the point's observation in A
	int* free_pts;                 // [max_points] ids of dead points
	int* ctr;                      // created, next unused id, n free, n observations, overflow flag
	int max_frames, max_keys, hcap, max_points;
	int sort_cap;                  // power of two >= max_keys: the length of propagate's shared-memory sort arrays
};
enum { C_CREATED = 0, C_NEXT = 1, C_NFREE = 2, C_NOBS = 3, C_OVERFLOW = 4, C_N = 8 };

struct TrkEnt { int da, idB, sA, sB, flags, rc, ra, id; };   // per list entry: initial A index / B id, scratch slots, outcome
enum { E_SKIP = 1, E_CREATE = 2, E_NEWA = 4 };

__device__ __forceinline__ unsigned norm_bits(float x) { const unsigned b = __float_as_uint(x); return b == 0x80000000u ? 0u : b; }
__device__ __forceinline__ unsigned long long norm_key(float u, float v) { return ((unsigned long long)norm_bits(u) << 32) | norm_bits(v); }
__device__ __forceinline__ unsigned ord_bits(unsigned b) { return (b & 0x80000000u) ? ~b : (b | 0x80000000u); }   // float order as unsigned order
__device__ __forceinline__ unsigned long long ord_key(unsigned long long k) { return ((unsigned long long)ord_bits((unsigned)(k >> 32)) << 32) | ord_bits((unsigned)k); }
__device__ __forceinline__ float2* obs_at(const TrkTable& t, int p, int f) { return t.obs + (size_t)f * t.max_points + p; }
__device__ __forceinline__ bool obs_seen(float2 o) { return !(__float_as_uint(o.x) == 0xffffffffu && __float_as_uint(o.y) == 0xffffffffu); }
__device__ __forceinline__ float2 obs_empty() { return make_float2(__uint_as_float(0xffffffffu), __uint_as_float(0xffffffffu)); }
__device__ __forceinline__ unsigned hmix(unsigned long long k) {
	k ^= k >> 33; k *= 0xff51afd7ed558ccdull; k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ull; k ^= k >> 33;
	return (unsigned)k;
}

__device__ int frame_find(const TrkTable& t, int f, unsigned long long key) {
	const unsigned long long* hk = t.hkey + (size_t)f * t.hcap;
	const unsigned m = (unsigned)t.hcap - 1u;
	for (unsigned h = hmix(key) & m, n = 0; n < (unsigned)t.hcap; h = (h + 1u) & m, n++) {
		const unsigned long long k = hk[h];
		if (k == key) return t.hidx[(size_t)f * t.hcap + h];
		if (k == kTrkEmpty) return -1;
	}
	return -1;
}
__device__ void frame_insert(const TrkTable& t, int f, unsigned long long key, int idx) {
	unsigned long long* hk = t.hkey + (size_t)f * t.hcap;
	const unsigned m = (unsigned)t.hcap - 1u;
	for (unsigned h = hmix(key) & m, n = 0; n < (unsigned)t.hcap; h = (h + 1u) & m, n++) {
		const unsigned long long prev = atomicCAS(hk + h, kTrkEmpty, key);
		if (prev == kTrkEmpty || prev == key) { t.hidx[(size_t)f * t.hcap + h] = idx; return; }
	}
}
// find-or-insert in the per-call scratch table (load factor <= 1/2: a free slot always exists)
__device__ int scratch_slot(unsigned long long* hk, int cap, unsigned long long key) {
	const unsigned m = (unsigned)cap - 1u;
	for (unsigned h = hmix(key) & m;; h = (h + 1u) & m) {
		const unsigned long long prev = atomicCAS(hk + h, kTrkEmpty, key);
		if (prev == kTrkEmpty || prev == key) return (int)h;
	}
}

__device__ __forceinline__ float4 src_uv(const TrkSrc& s, int i) {
	const int j = s.ids ? s.ids[i] : i;
	const float* p = s.base + (size_t)s.stride * j;
	return make_float4(p[0], p[1], p[2], p[3]);
}

__global__ void __launch_bounds__(kTrkThreads) k_trk_update(TrkTable t, int sa, int sb, TrkSrc src, unsigned long long* __restrict__ shk, int* __restrict__ smn,
                                                          int* __restrict__ smx, int scap, TrkEnt* __restrict__ ent, int list_cap, unsigned epoch) {
	__shared__ int s_scan[kTrkThreads / 32];
	__shared__ int s_n, s_S, s_ok, s_nc, s_na, s_nfree, s_next, s_nkA, s_nkB;
	const int tid = threadIdx.x;
	if (tid == 0) {
		int n;
		if (src.n_inl) {        // the pair's emitted count exactly as k_emit_entryj computes it
			int excl = 0;
			for (int q = 0; q < src.pair; q++) { const int c = src.n_inl[q]; excl += c < 5 ? 0 : c; }
			int cnt = src.n_inl[src.pair]; if (cnt < 5) cnt = 0;
			if (excl > src.capacity) excl = src.capacity;
			if (excl + cnt > src.capacity) cnt = src.capacity - excl;
			n = cnt;
		} else {
			n = *src.n_dev;
			if (n < 0 || n > src.max_n) { t.ctr[C_OVERFLOW] = 1; n = 0; }
		}
		if (n > list_cap) { t.ctr[C_OVERFLOW] = 1; n = 0; }
		int S = 64;
		while (S < 2 * n) S <<= 1;
		s_n = n; s_S = S;
	}
	__syncthreads();
	const int n = s_n, S = s_S;
	if (n == 0) return;
	unsigned long long* shkA = shk; unsigned long long* shkB = shk + scap;
	int* smnA = smn; int* smnB = smn + scap;
	for (int h = tid; h < S; h += blockDim.x) { shkA[h] = kTrkEmpty; shkB[h] = kTrkEmpty; smnA[h] = 0x7fffffff; smnB[h] = 0x7fffffff; smx[h] = -1; }
	__syncthreads();
	// 1: where each key stood at the start; first occurrence of each key in the list
	for (int i = tid; i < n; i += blockDim.x) {
		const float4 uv = src_uv(src, i);
		const unsigned long long kA = norm_key(uv.x, uv.y), kB = norm_key(uv.z, uv.w);
		TrkEnt e;
		e.da = frame_find(t, sa, kA);
		const int db = frame_find(t, sb, kB);
		e.idB = db >= 0 ? t.keys[(size_t)sb * t.max_keys + db].z : -1;
		e.sA = scratch_slot(shkA, S, kA); e.sB = scratch_slot(shkB, S, kB);
		atomicMin(smnA + e.sA, i); atomicMin(smnB + e.sB, i);
		e.flags = 0; e.rc = e.ra = 0; e.id = -1;
		ent[i] = e;
	}
	__syncthreads();
	// 2: skip / new point / new key in A, ranks in list order
	int carry_c = 0, carry_a = 0;
	for (int base = 0; base < n; base += blockDim.x) {
		const int i = base + tid;
		int fl = 0;
		if (i < n) {
			const TrkEnt& e = ent[i];
			const bool inA = e.da >= 0 || smnA[e.sA] != i, inB = e.idB >= 0 || smnB[e.sB] != i;
			fl = (inA && inB) ? E_SKIP : ((inB ? 0 : E_CREATE) | (inA ? 0 : E_NEWA));
		}
		int tc, ta;
		const int rc = block_excl_scan((fl & E_CREATE) ? 1 : 0, s_scan, &tc);
		const int ra = block_excl_scan((fl & E_NEWA) ? 1 : 0, s_scan, &ta);
		if (i < n) { ent[i].flags = fl; ent[i].rc = carry_c + rc; ent[i].ra = carry_a + ra; }
		carry_c += tc; carry_a += ta;
	}
	if (tid == 0) {
		const int nkA = t.n_keys[sa], nkB = t.n_keys[sb], nfree = t.ctr[C_NFREE], next = t.ctr[C_NEXT];
		const bool ok = nkA + carry_a <= t.max_keys && nkB + carry_c <= t.max_keys && carry_c <= nfree + (t.max_points - next);
		if (!ok) t.ctr[C_OVERFLOW] = 1;
		s_ok = ok; s_nc = carry_c; s_na = carry_a; s_nfree = nfree; s_next = next; s_nkA = nkA; s_nkB = nkB;
	}
	__syncthreads();
	if (!s_ok) return;
	// 3: new points, anchored at B (a reused id was forgotten in every slot: its column entries are all empty)
	for (int i = tid; i < n; i += blockDim.x) {
		const TrkEnt e = ent[i];
		if (!(e.flags & E_CREATE)) continue;
		const int id = e.rc < s_nfree ? t.free_pts[s_nfree - 1 - e.rc] : s_next + (e.rc - s_nfree);
		ent[i].id = id;
		const float4 uv = src_uv(src, i);
		*obs_at(t, id, sb) = make_float2(uv.z, uv.w);
		t.n_obs[id] = 1;
		t.keys[(size_t)sb * t.max_keys + s_nkB + e.rc] = make_int4(__float_as_int(uv.z), __float_as_int(uv.w), id, 0);
		frame_insert(t, sb, norm_key(uv.z, uv.w), s_nkB + e.rc);
	}
	__syncthreads();
	// 4: every other entry that is not skipped reuses mapB[kB]; last writers of mapA[kA] and of the points' observations in A
	for (int i = tid; i < n; i += blockDim.x) {
		const TrkEnt e = ent[i];
		if (e.flags & E_SKIP) continue;
		int id = e.id;
		if (!(e.flags & E_CREATE)) { id = e.idB >= 0 ? e.idB : ent[smnB[e.sB]].id; ent[i].id = id; }
		atomicMax(smx + e.sA, i);
		atomicMax(t.last + id, ((unsigned long long)epoch << 32) | (unsigned)i);
	}
	__syncthreads();
	// 5: mapA[kA] = id (last writer), img_pt[A] = kA (last writer per point)
	int add_obs = 0;
	for (int i = tid; i < n; i += blockDim.x) {
		const TrkEnt e = ent[i];
		if (e.flags & E_SKIP) continue;
		const float4 uv = src_uv(src, i);
		if (smx[e.sA] == i) {
			if (e.da >= 0) {
				t.keys[(size_t)sa * t.max_keys + e.da].z = e.id;
			} else {                               // inserted by the key's first occurrence, with that occurrence's bits
				const int f = smnA[e.sA];
				const float4 uf = src_uv(src, f);
				const int d = s_nkA + ent[f].ra;
				t.keys[(size_t)sa * t.max_keys + d] = make_int4(__float_as_int(uf.x), __float_as_int(uf.y), e.id, 0);
				frame_insert(t, sa, norm_key(uf.x, uf.y), d);
			}
		}
		if (t.last[e.id] == (((unsigned long long)epoch << 32) | (unsigned)i)) {
			float2* o = obs_at(t, e.id, sa);         // (one last writer per point: no other thread touches the point here)
			if (!obs_seen(*o)) { t.n_obs[e.id]++; add_obs++; }
			*o = make_float2(uv.x, uv.y);
		}
	}
	int tot;
	block_excl_scan(add_obs, s_scan, &tot);
	if (tid == 0) {
		t.n_keys[sa] = s_nkA + s_na; t.n_keys[sb] = s_nkB + s_nc;
		t.ctr[C_CREATED] += s_nc;
		t.ctr[C_NFREE] = s_nfree - min(s_nc, s_nfree);
		t.ctr[C_NEXT] = s_next + max(0, s_nc - s_nfree);
		t.ctr[C_NOBS] += tot + s_nc;
	}
}

// findCorresByMapPoints' candidate list for (A, B): A's keys in ascending (u, v) order whose point is seen in B, without those that share
// (uA, vA) or (uB, vB) with `existing`, and of those with the same (uB, vB) only the first.  One CTA: two bitonic sorts in shared memory.
__global__ void __launch_bounds__(kTrkThreads) k_trk_propagate(TrkTable t, int sa, int sb, const float4* __restrict__ existing, int n_existing,
                                                             float4* __restrict__ out, int capacity, int32_t* __restrict__ n_out) {
	extern __shared__ unsigned long long s_key[];           // [sort_cap] sort keys, then int payload, int A-order index, uint8 drop of the same length
	__shared__ int s_scan[kTrkThreads / 32];
	__shared__ int s_m;
	const int tid = threadIdx.x;
	const int nk = t.n_keys[sa];
	int P = 1;
	while (P < nk) P <<= 1;
	// the sorts run over P = the power of two >= nk, which may exceed max_keys: every array is sort_cap (>= P) long
	int* s_pay = reinterpret_cast<int*>(s_key + t.sort_cap);
	int* s_ord = s_pay + t.sort_cap;
	unsigned char* s_drop = reinterpret_cast<unsigned char*>(s_ord + t.sort_cap);
	if (tid == 0) s_m = 0;
	__syncthreads();
	for (int k = tid; k < P; k += blockDim.x) {
		unsigned long long key = kTrkEmpty;
		if (k < nk) {
			const int4 e = t.keys[(size_t)sa * t.max_keys + k];
			const float2 ob = *obs_at(t, e.z, sb);
			if (obs_seen(ob)) {
				const float uA = __int_as_float(e.x), vA = __int_as_float(e.y);
				bool keep = true;
				for (int j = 0; j < n_existing && keep; j++) {
					const float4 x = existing[j];
					keep = !((x.x == uA && x.y == vA) || (x.z == ob.x && x.w == ob.y));
				}
				if (keep) { key = ord_key(norm_key(uA, vA)); atomicAdd(&s_m, 1); }
			}
		}
		s_key[k] = key; s_pay[k] = k;
	}
	__syncthreads();
	const int m = s_m;
	// sort by (key, payload) ascending; A keys are unique per frame, so (key) alone orders the candidates
	for (int size = 2; size <= P; size <<= 1)
		for (int stride = size >> 1; stride > 0; stride >>= 1) {
			for (int i = tid; i < P; i += blockDim.x) {
				const int j = i ^ stride;
				if (j > i) {
					const unsigned long long ki = s_key[i], kj = s_key[j];
					const bool gt = ki > kj || (ki == kj && s_pay[i] > s_pay[j]);
					if (gt == ((i & size) == 0)) { s_key[i] = kj; s_key[j] = ki; const int p = s_pay[i]; s_pay[i] = s_pay[j]; s_pay[j] = p; }
				}
			}
			__syncthreads();
		}
	// the candidates in A order; now sort their (uB, vB) keys, ties by A position, to find the first of each
	for (int k = tid; k < m; k += blockDim.x) s_ord[k] = s_pay[k];
	__syncthreads();
	for (int k = tid; k < P; k += blockDim.x) {
		unsigned long long key = kTrkEmpty;
		if (k < m) {
			const float2 ob = *obs_at(t, t.keys[(size_t)sa * t.max_keys + s_ord[k]].z, sb);
			key = ord_key(norm_key(ob.x, ob.y));
		}
		s_key[k] = key; s_pay[k] = k; s_drop[k] = 0;
	}
	__syncthreads();
	for (int size = 2; size <= P; size <<= 1)
		for (int stride = size >> 1; stride > 0; stride >>= 1) {
			for (int i = tid; i < P; i += blockDim.x) {
				const int j = i ^ stride;
				if (j > i) {
					const unsigned long long ki = s_key[i], kj = s_key[j];
					const bool gt = ki > kj || (ki == kj && s_pay[i] > s_pay[j]);
					if (gt == ((i & size) == 0)) { s_key[i] = kj; s_key[j] = ki; const int p = s_pay[i]; s_pay[i] = s_pay[j]; s_pay[j] = p; }
				}
			}
			__syncthreads();
		}
	for (int k = tid; k < m; k += blockDim.x)
		if (k > 0 && s_key[k] == s_key[k - 1]) s_drop[s_pay[k]] = 1;
	__syncthreads();
	int carry = 0;
	for (int base = 0; base < m; base += blockDim.x) {
		const int k = base + tid;
		const bool keep = k < m && !s_drop[k];
		int tot;
		const int r = carry + block_excl_scan(keep ? 1 : 0, s_scan, &tot);
		if (keep) {
			if (r < capacity) {
				const int4 e = t.keys[(size_t)sa * t.max_keys + s_ord[k]];
				const float2 ob = *obs_at(t, e.z, sb);
				out[r] = make_float4(__int_as_float(e.x), __int_as_float(e.y), ob.x, ob.y);
			} else {
				t.ctr[C_OVERFLOW] = 1;
			}
		}
		carry += tot;
	}
	if (tid == 0) *n_out = min(carry, capacity);
}

// forgetFrame: the slot's observations leave every point; points left with none are free for reuse; the slot's map is emptied
__global__ void __launch_bounds__(256) k_trk_forget(TrkTable t, int slot) {
	const int next = t.ctr[C_NEXT];
	const int stride = gridDim.x * blockDim.x;
	for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < next; p += stride) {
		float2* o = obs_at(t, p, slot);
		if (!obs_seen(*o)) continue;
		*o = obs_empty();
		atomicSub(t.ctr + C_NOBS, 1);
		const int left = t.n_obs[p] - 1;         // (one thread per point)
		t.n_obs[p] = left;
		if (left == 0) t.free_pts[atomicAdd(t.ctr + C_NFREE, 1)] = p;
	}
	for (int h = blockIdx.x * blockDim.x + threadIdx.x; h < t.hcap; h += stride) t.hkey[(size_t)slot * t.hcap + h] = kTrkEmpty;
	if (blockIdx.x == 0 && threadIdx.x == 0) t.n_keys[slot] = 0;
}

struct TracksDev {
	bool ready = false;
	TrkTable t{};
	int list_cap = 0, scap = 0;
	DevBuf keys, hkey, hidx, n_keys, obs, n_obs, last, free_pts, ctr, shk, smn, smx, ent;
	std::map<int, int> slot_of;          // frame id -> slot
	std::vector<int> free_slots;
	unsigned epoch = 0;
	size_t prop_smem = 0;
};

void StateDeleter::operator()(TracksDev* d) const { delete d; }

int tracks_state(bt_ctx* ctx, const char* who) {
	TracksDev* d;
	return state_of(ctx, &bt_ctx::tracks, who, "bt_tracks_dev_reserve", &d);
}

int tracks_slot(bt_ctx* ctx, int frame_id, bool create, int* slot) {
	TracksDev* d = ctx->tracks.get();
	const auto it = d->slot_of.find(frame_id);
	if (it != d->slot_of.end()) { *slot = it->second; return BT_OK; }
	*slot = -1;
	if (!create) return BT_OK;
	BT_REQUIRE(!d->free_slots.empty(), BT_ERR_CAPACITY, "map-point table: more than %d frames alive", d->t.max_frames);
	*slot = d->free_slots.back();
	d->free_slots.pop_back();
	d->slot_of[frame_id] = *slot;
	return BT_OK;
}

int tracks_free_slots(bt_ctx* ctx) { return (int)ctx->tracks->free_slots.size(); }

int tracks_points_alive(bt_ctx* ctx, cudaStream_t stream, int* n) {
	int c[C_N];
	BT_CUDA(cudaMemcpyAsync(c, ctx->tracks->ctr.p, sizeof(c), cudaMemcpyDeviceToHost, stream));
	BT_CUDA(cudaStreamSynchronize(stream));
	*n = c[C_NEXT] - c[C_NFREE];
	return BT_OK;
}

int tracks_launch_update(bt_ctx* ctx, int slot_a, int slot_b, const TrkSrc& src, cudaStream_t stream) {
	TracksDev* d = ctx->tracks.get();
	d->epoch++;
	k_trk_update<<<1, kTrkThreads, 0, stream>>>(d->t, slot_a, slot_b, src, d->shk.as<unsigned long long>(), d->smn.as<int>(), d->smx.as<int>(), d->scap,
	                                            d->ent.as<TrkEnt>(), d->list_cap, d->epoch);
	BT_CUDA(cudaGetLastError());
	return BT_OK;
}

int tracks_launch_propagate(bt_ctx* ctx, int slot_a, int slot_b, const float4* existing, int n_existing, float4* out, int capacity, int32_t* n_out,
                            cudaStream_t stream) {
	TracksDev* d = ctx->tracks.get();
	k_trk_propagate<<<1, kTrkThreads, d->prop_smem, stream>>>(d->t, slot_a, slot_b, existing, n_existing, out, capacity, n_out);
	BT_CUDA(cudaGetLastError());
	return BT_OK;
}

}  // namespace bt

using namespace bt;

static int tracks_dev_reserve(bt_ctx* ctx, int max_frames, int max_keys_per_frame, int max_points) {
	TracksDev* d;
	BT_TRY(take_state(ctx, &bt_ctx::tracks, &d));
	int hcap = 64;
	while (hcap < 2 * max_keys_per_frame) hcap <<= 1;
	const int list_cap = 4 * max_keys_per_frame;       // one pair's list: mutual matches of both directions plus propagated ones, duplicates kept
	int scap = 64;
	while (scap < 2 * list_cap) scap <<= 1;
	const size_t F = (size_t)max_frames, K = (size_t)max_keys_per_frame, Pn = (size_t)max_points;
	BT_TRY(d->keys.alloc(sizeof(int4) * F * K)); BT_TRY(d->hkey.alloc(sizeof(unsigned long long) * F * hcap)); BT_TRY(d->hidx.alloc(sizeof(int) * F * hcap));
	BT_TRY(d->n_keys.alloc(sizeof(int) * F));
	BT_TRY(d->obs.alloc(sizeof(float2) * Pn * F)); BT_TRY(d->n_obs.alloc(sizeof(int) * Pn)); BT_TRY(d->last.alloc(sizeof(unsigned long long) * Pn));
	BT_TRY(d->free_pts.alloc(sizeof(int) * Pn));
	BT_TRY(d->ctr.alloc(sizeof(int) * C_N));
	BT_TRY(d->shk.alloc(sizeof(unsigned long long) * 2 * scap)); BT_TRY(d->smn.alloc(sizeof(int) * 2 * scap)); BT_TRY(d->smx.alloc(sizeof(int) * scap));
	BT_TRY(d->ent.alloc(sizeof(TrkEnt) * list_cap));
	BT_CUDA(cudaMemset(d->hkey.p, 0xff, sizeof(unsigned long long) * F * hcap));
	BT_CUDA(cudaMemset(d->n_keys.p, 0, sizeof(int) * F));
	BT_CUDA(cudaMemset(d->obs.p, 0xff, sizeof(float2) * Pn * F));        // every observation empty
	BT_CUDA(cudaMemset(d->n_obs.p, 0, sizeof(int) * Pn));
	BT_CUDA(cudaMemset(d->last.p, 0, sizeof(unsigned long long) * Pn));
	BT_CUDA(cudaMemset(d->ctr.p, 0, sizeof(int) * C_N));
	BT_CUDA(cudaDeviceSynchronize());
	TrkTable& t = d->t;
	t.keys = d->keys.as<int4>(); t.hkey = d->hkey.as<unsigned long long>(); t.hidx = d->hidx.as<int>(); t.n_keys = d->n_keys.as<int>();
	t.obs = d->obs.as<float2>(); t.n_obs = d->n_obs.as<int>(); t.last = d->last.as<unsigned long long>(); t.free_pts = d->free_pts.as<int>();
	t.ctr = d->ctr.as<int>();
	t.max_frames = max_frames; t.max_keys = max_keys_per_frame; t.hcap = hcap; t.max_points = max_points;
	t.sort_cap = 1;
	while (t.sort_cap < max_keys_per_frame) t.sort_cap <<= 1;
	d->slot_of.clear(); d->free_slots.clear();
	for (int f = max_frames - 1; f >= 0; f--) d->free_slots.push_back(f);
	d->epoch = 0;
	d->list_cap = list_cap; d->scap = scap;
	d->prop_smem = (size_t)t.sort_cap * (sizeof(unsigned long long) + 2 * sizeof(int) + 1);
	BT_CUDA(cudaFuncSetAttribute(k_trk_propagate, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)d->prop_smem));
	d->ready = true;
	return BT_OK;
}

extern "C" int bt_tracks_dev_reserve(bt_ctx* ctx, int max_frames, int max_keys_per_frame, int max_points) {
	BT_REQUIRE(ctx && max_frames > 0 && max_frames <= kTrkMaxFrames && max_keys_per_frame > 0 && max_keys_per_frame <= kTrkMaxKeys && max_points > 0,
	           BT_ERR_INVALID_ARG, "bt_tracks_dev_reserve: need 0 < max_frames <= %d, 0 < max_keys_per_frame <= %d, max_points > 0", kTrkMaxFrames, kTrkMaxKeys);
	return tracks_dev_reserve(ctx, max_frames, max_keys_per_frame, max_points);
}

extern "C" int bt_tracks_dev_reserve_ex(bt_ctx* ctx, int max_frames, int max_keys_per_frame, int max_points) {
	BT_REQUIRE(ctx && max_frames > 0 && max_frames <= kTrkMaxFramesEx && max_keys_per_frame > 0 && max_keys_per_frame <= kTrkMaxKeys && max_points > 0,
	           BT_ERR_INVALID_ARG, "bt_tracks_dev_reserve_ex: need 0 < max_frames <= %d, 0 < max_keys_per_frame <= %d, max_points > 0", kTrkMaxFramesEx,
	           kTrkMaxKeys);
	return tracks_dev_reserve(ctx, max_frames, max_keys_per_frame, max_points);
}

extern "C" int bt_tracks_dev_update_pair(bt_ctx* ctx, int frame_a, int frame_b, const float* uv_dev, const int32_t* n_dev, int uv_capacity, void* stream_) {
	TracksDev* d;
	BT_TRY(state_of(ctx, &bt_ctx::tracks, "bt_tracks_dev_update_pair", "bt_tracks_dev_reserve", &d));
	BT_REQUIRE(n_dev && uv_capacity >= 0 && (uv_capacity == 0 || uv_dev), BT_ERR_INVALID_ARG, "bt_tracks_dev_update_pair: bad arguments");
	BT_REQUIRE(frame_a > frame_b, BT_ERR_INVALID_ARG, "bt_tracks_dev_update_pair: frame A must be the newer frame (id %d <= %d)", frame_a, frame_b);
	const bool need_a = !d->slot_of.count(frame_a), need_b = !d->slot_of.count(frame_b);
	BT_REQUIRE(tracks_free_slots(ctx) >= (int)need_a + (int)need_b, BT_ERR_CAPACITY, "bt_tracks_dev_update_pair: more than %d frames alive", d->t.max_frames);
	int sa, sb, rc;
	if ((rc = tracks_slot(ctx, frame_a, true, &sa)) != BT_OK) return rc;
	if ((rc = tracks_slot(ctx, frame_b, true, &sb)) != BT_OK) return rc;
	TrkSrc src{ uv_dev, 4, nullptr, n_dev, uv_capacity, nullptr, 0, 0 };
	return tracks_launch_update(ctx, sa, sb, src, (cudaStream_t)stream_);
}

extern "C" int bt_tracks_dev_propagate(bt_ctx* ctx, int frame_a, int frame_b, const float* existing_uv_dev, int n_existing, float* out_uv_dev, int capacity,
                                       int32_t* n_out_dev, void* stream_) {
	TracksDev* d;
	BT_TRY(state_of(ctx, &bt_ctx::tracks, "bt_tracks_dev_propagate", "bt_tracks_dev_reserve", &d));
	BT_REQUIRE(n_out_dev && n_existing >= 0 && (n_existing == 0 || existing_uv_dev) && capacity >= 0 && (capacity == 0 || out_uv_dev), BT_ERR_INVALID_ARG,
	           "bt_tracks_dev_propagate: bad arguments");
	BT_REQUIRE(frame_a > frame_b, BT_ERR_INVALID_ARG, "bt_tracks_dev_propagate: frame A must be the newer frame (id %d <= %d)", frame_a, frame_b);
	cudaStream_t stream = (cudaStream_t)stream_;
	int sa, sb;
	tracks_slot(ctx, frame_a, false, &sa);
	tracks_slot(ctx, frame_b, false, &sb);
	if (sa < 0 || sb < 0) {     // a frame without a map: nothing to propagate
		BT_CUDA(cudaMemsetAsync(n_out_dev, 0, sizeof(int32_t), stream));
		return BT_OK;
	}
	return tracks_launch_propagate(ctx, sa, sb, reinterpret_cast<const float4*>(existing_uv_dev), n_existing, reinterpret_cast<float4*>(out_uv_dev), capacity,
	                               n_out_dev, stream);
}

extern "C" int bt_tracks_dev_forget_frame(bt_ctx* ctx, int frame, void* stream_) {
	TracksDev* d;
	BT_TRY(state_of(ctx, &bt_ctx::tracks, "bt_tracks_dev_forget_frame", "bt_tracks_dev_reserve", &d));
	const auto it = d->slot_of.find(frame);
	if (it == d->slot_of.end()) return BT_OK;
	const int slot = it->second;
	k_trk_forget<<<ctx->sm_count > 0 ? ctx->sm_count : 132, 256, 0, (cudaStream_t)stream_>>>(d->t, slot);
	BT_CUDA(cudaGetLastError());
	d->slot_of.erase(it);
	d->free_slots.push_back(slot);
	return BT_OK;
}

// Synchronises `stream`.  BT_ERR_CAPACITY when an earlier call overflowed a capacity (that call changed nothing); the flag is cleared.
extern "C" int bt_tracks_dev_stats(bt_ctx* ctx, int* n_points, int* n_observations, void* stream_) {
	TracksDev* d;
	BT_TRY(state_of(ctx, &bt_ctx::tracks, "bt_tracks_dev_stats", "bt_tracks_dev_reserve", &d));
	BT_REQUIRE(n_points && n_observations, BT_ERR_INVALID_ARG, "bt_tracks_dev_stats: NULL argument");
	cudaStream_t stream = (cudaStream_t)stream_;
	int c[C_N];
	BT_CUDA(cudaMemcpyAsync(c, d->ctr.p, sizeof(c), cudaMemcpyDeviceToHost, stream));
	BT_CUDA(cudaStreamSynchronize(stream));
	*n_points = c[C_CREATED];
	*n_observations = c[C_NOBS];
	if (c[C_OVERFLOW]) {
		BT_CUDA(cudaMemsetAsync(d->ctr.as<int>() + C_OVERFLOW, 0, sizeof(int), stream));
		BT_CUDA(cudaStreamSynchronize(stream));
		BT_REQUIRE(false, BT_ERR_CAPACITY, "map-point table: a call exceeded the reserved frames / keys per frame / points and was not applied");
	}
	return BT_OK;
}
