"""The tables a tracker with a keyframe pool needs past 64 frames: the device map-point table with more than 64 frame slots
(bt_tracks_dev_reserve_ex) against the host table, and the match cache's entry arena (bt_match_cache_reserve_entries) against a dict model."""
import ctypes

import numpy as np
import pytest

from bundletrack_b200 import _lib
from test_tracks_gpu import _bits, _key_pool

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------ 1. the map-point table past 64 slots
def _run_wide_parity(seed, n_ops, n_frames, max_keys, max_list, pool_u, pool_v, long_every=0, max_points=0):
    """Seeded random updates / propagations / forgets over n_frames frame ids through the host and the device table; every propagation
    byte-identical, stats equal at the end.  Returns event counts, among them the most frames the device table held at once."""
    from bundletrack_b200.matcher import DeviceTracks
    from bundletrack_b200.policy import Tracks
    rng = np.random.default_rng(seed)
    assert len(pool_u) * len(pool_v) <= max_keys
    host, dev = Tracks(), DeviceTracks(max_frames=n_frames, max_keys_per_frame=max_keys, max_points=max_points)
    mapped = set()                                    # frames the device table holds a slot for
    keys = {f: set() for f in range(n_frames)}
    anchors = set()
    c = dict(ops=0, prop=0, nonempty=0, forgot_anchor=0, long_list=0, reused=0, max_mapped=0)
    forgotten = set()
    updated = []                                      # pairs updated together: their propagations are the non-empty ones

    def draw(n):
        uv = np.stack([pool_u[rng.integers(0, len(pool_u), n)], pool_v[rng.integers(0, len(pool_v), n)],
                       pool_u[rng.integers(0, len(pool_u), n)], pool_v[rng.integers(0, len(pool_v), n)]], 1).astype(np.float32)
        if n > 3:
            uv[rng.integers(0, n)][:2] = uv[0][:2]
            uv[rng.integers(0, n)][2:] = uv[1][2:]
        return np.ascontiguousarray(uv)

    for k in range(n_ops):
        r = rng.random()
        alive = sorted(mapped)
        if r < 0.55 or len(alive) < 2:
            a, b = (int(x) for x in sorted(rng.choice(n_frames, 2, replace=False))[::-1])
            n = int(rng.integers(max_list // 2, max_list + 1)) if long_every and k % long_every == 0 else (0 if rng.random() < 0.1 else int(rng.integers(1, 41)))
            uv = draw(n)
            inl = (rng.random(n) < 0.8).astype(np.uint8) if rng.random() < 0.3 else None
            host.update_pair(a, b, uv, inl)
            dev.update_pair(a, b, uv, inl)
            kept = uv if inl is None else uv[inl.astype(bool)]
            keys[a] |= {(float(u) + 0.0, float(v) + 0.0) for u, v in kept[:, :2]}
            keys[b] |= {(float(u) + 0.0, float(v) + 0.0) for u, v in kept[:, 2:]}
            anchors |= {b} if len(kept) else set()
            c["reused"] += len({a, b} & forgotten)
            mapped |= {a, b}
            updated.append((a, b))
            c["long_list"] += len(kept) > 1024
            c["max_mapped"] = max(c["max_mapped"], len(mapped))
        elif r < 0.92:
            live = [p for p in updated[-200:] if p[0] in mapped and p[1] in mapped]
            if live and rng.random() < 0.7:
                a, b = live[int(rng.integers(0, len(live)))]
            else:
                cand = alive if rng.random() < 0.8 else list(range(n_frames))
                a, b = (int(x) for x in sorted(rng.choice(cand, 2, replace=False))[::-1])
            ex = draw(int(rng.integers(0, 6))) if rng.random() < 0.3 else np.zeros((0, 4), np.float32)
            want = host.propagate(a, b, ex)
            got = dev.propagate(a, b, ex)
            assert got.shape == want.shape and np.array_equal(_bits(got), _bits(want)), (k, a, b)
            c["prop"] += 1
            c["nonempty"] += len(want) > 0
        else:
            f = int(rng.choice(alive))
            c["forgot_anchor"] += f in anchors
            host.forget_frame(f)
            dev.forget_frame(f)
            keys[f] = set()
            anchors.discard(f)
            mapped.discard(f)
            forgotten.add(f)
        c["ops"] += 1
    assert host.stats() == dev.stats()
    dev.close()
    return c


@pytest.mark.parametrize("seed", [1, 2])
def test_wide_table_equals_host_table(cuda_device, seed):
    """Up to 200 frames alive: slots 64 and above are in use; short lists over a small key pool (+-0, one-ulp keys, repeats)."""
    rng = np.random.default_rng(300 + seed)
    pool = _key_pool(rng, 24)
    c = _run_wide_parity(seed, 1400, 200, 1024, 40, pool, pool)
    assert c["max_mapped"] >= 150 and c["prop"] >= 400 and c["nonempty"] >= 100 and c["forgot_anchor"] >= 20 and c["reused"] >= 20, c


def test_wide_table_long_lists(cuda_device):
    """Lists longer than one CTA on a table of 160 frames."""
    rng = np.random.default_rng(9)
    pool_u, pool_v = _key_pool(rng, 50), _key_pool(rng, 40)
    c = _run_wide_parity(5, 500, 160, 2000, 1800, pool_u, pool_v, long_every=12, max_points=200000)
    assert c["long_list"] >= 10 and c["max_mapped"] >= 100 and c["nonempty"] >= 20 and c["forgot_anchor"] >= 5, c


def test_reserve_ex_limits(cuda_device):
    lib = _lib.load()
    ctx = ctypes.c_void_p()
    _lib.check(lib.bt_ctx_create(ctypes.byref(ctx), 0), "bt_ctx_create")
    assert lib.bt_tracks_dev_reserve(ctx, 65, 4, 3) == _lib.BT_ERR_INVALID_ARG
    assert lib.bt_tracks_dev_reserve_ex(ctx, 64 + 1024 + 1, 4, 3) == _lib.BT_ERR_INVALID_ARG
    assert lib.bt_tracks_dev_reserve_ex(ctx, 0, 4, 3) == _lib.BT_ERR_INVALID_ARG
    assert lib.bt_tracks_dev_reserve_ex(ctx, 64 + 1024, 8, 16) == _lib.BT_OK
    assert lib.bt_tracks_dev_reserve_ex(ctx, 65, 4, 3) == _lib.BT_OK
    lib.bt_ctx_destroy(ctx)


# ------------------------------------------------------------------------------------------------ 2. the match cache's arena
class CacheModel:
    """The cache as a dict: (idA, idB) -> (entries, status); gather = the blocks back to back with imgIdx rewritten.  `compactions` counts
    the puts that found no room behind the last block (the arena's placement rule, followed only to know which puts compacted)."""

    def __init__(self, max_pairs, budget, max_block):
        self.max_pairs, self.budget, self.max_block = max_pairs, budget, max_block
        self.d = {}
        self.top = self.compactions = 0

    def live(self):
        return sum(len(e) for e, _ in self.d.values())

    def put(self, pairs, blocks, status):
        new = dict(self.d)
        for p, e, s in zip(pairs, blocks, status):
            if len(e) > self.max_block:
                return False
            new[p] = (e, s)
        if len(new) > self.max_pairs or sum(len(e) for e, _ in new.values()) > self.budget:
            return False
        need = sum(len(new[p][0]) for p in set(pairs))
        if self.top + need > self.budget:
            self.compactions += 1
            self.top = sum(len(e) for p, (e, _) in self.d.items() if p not in set(pairs))
        self.top += need
        self.d = new
        return True

    def forget(self, f):
        self.d = {p: v for p, v in self.d.items() if f not in p}

    def gather(self, pairs, wi, wj):
        out = []
        for p, i, j in zip(pairs, wi, wj):
            e = self.d[p][0].copy()
            e[:, 0], e[:, 1] = i, j
            out.append(e)
        return np.concatenate(out) if out else np.zeros((0, 8), np.int32)


class Cache:
    def __init__(self, max_pairs, budget=None, per_pair=None):
        self.lib = _lib.load()
        self.ctx = ctypes.c_void_p()
        _lib.check(self.lib.bt_ctx_create(ctypes.byref(self.ctx), 0), "bt_ctx_create")
        if budget is None:
            _lib.check(self.lib.bt_match_cache_reserve(self.ctx, max_pairs, per_pair), "bt_match_cache_reserve")
        else:
            _lib.check(self.lib.bt_match_cache_reserve_entries(self.ctx, max_pairs, ctypes.c_longlong(budget)), "bt_match_cache_reserve_entries")

    def put(self, pairs, blocks, status):
        import torch
        n = len(pairs)
        cat = np.concatenate(blocks) if sum(len(b) for b in blocks) else np.zeros((1, 8), np.int32)
        dev = torch.from_numpy(np.ascontiguousarray(cat, np.int32)).cuda()
        cnt = np.array([len(b) for b in blocks], np.int32)
        off = np.concatenate([[0], np.cumsum(cnt)[:-1]]).astype(np.int32)
        st = np.asarray(status, np.int32)
        rc = self.lib.bt_match_cache_put(self.ctx, n, (ctypes.c_int32 * n)(*[p[0] for p in pairs]), (ctypes.c_int32 * n)(*[p[1] for p in pairs]),
                                         ctypes.c_void_p(dev.data_ptr()), cnt.ctypes.data_as(ctypes.c_void_p), off.ctypes.data_as(ctypes.c_void_p),
                                         st.ctypes.data_as(ctypes.c_void_p), None)
        torch.cuda.synchronize()          # (the source list must outlive the copy)
        return rc

    def gather(self, pairs, wi, wj, cap):
        import torch
        n = len(pairs)
        dst = torch.full((max(cap, 1), 8), -7, dtype=torch.int32, device="cuda")
        off, cnt = np.zeros(n, np.int32), np.zeros(n, np.int32)
        wi, wj = np.asarray(wi, np.uint32), np.asarray(wj, np.uint32)
        _lib.check(self.lib.bt_match_cache_gather(self.ctx, n, (ctypes.c_int32 * n)(*[p[0] for p in pairs]), (ctypes.c_int32 * n)(*[p[1] for p in pairs]),
                                                  wi.ctypes.data_as(ctypes.c_void_p), wj.ctypes.data_as(ctypes.c_void_p), ctypes.c_void_p(dst.data_ptr()),
                                                  ctypes.c_int(cap), off.ctypes.data_as(ctypes.c_void_p), cnt.ctypes.data_as(ctypes.c_void_p), None),
                   "bt_match_cache_gather")
        total = int(cnt.sum())
        assert np.array_equal(off, np.concatenate([[0], np.cumsum(cnt)[:-1]]))
        return dst[:total].cpu().numpy(), cnt

    def forget(self, f):
        _lib.check(self.lib.bt_match_cache_forget_frame(self.ctx, f), "bt_match_cache_forget_frame")

    def has(self, p):
        return bool(self.lib.bt_match_cache_has(self.ctx, p[0], p[1]))

    def usage(self):
        a, b = ctypes.c_int(0), ctypes.c_longlong(0)
        _lib.check(self.lib.bt_match_cache_usage(self.ctx, ctypes.byref(a), ctypes.byref(b)), "bt_match_cache_usage")
        return a.value, b.value

    def close(self):
        self.lib.bt_ctx_destroy(self.ctx)


def _block(rng, n):
    return rng.integers(-2 ** 31, 2 ** 31 - 1, size=(n, 8), dtype=np.int64).astype(np.int32)


def _check_same(cache, model, rng):
    pairs = list(model.d)
    assert cache.usage() == (len(pairs), model.live())
    for p in pairs:
        assert cache.has(p)
        n, s = ctypes.c_int(0), ctypes.c_int(0)
        _lib.check(cache.lib.bt_match_cache_status(cache.ctx, p[0], p[1], ctypes.byref(n), ctypes.byref(s)), "bt_match_cache_status")
        assert (n.value, s.value) == (len(model.d[p][0]), model.d[p][1])
    if pairs:
        sel = [pairs[i] for i in rng.permutation(len(pairs))[:min(len(pairs), 40)]]
        wi, wj = rng.integers(0, 32, len(sel)), rng.integers(0, 32, len(sel))
        got, _ = cache.gather(sel, wi, wj, sum(len(model.d[p][0]) for p in sel))
        assert got.tobytes() == model.gather(sel, wi, wj).tobytes()


def test_arena_compacts_before_it_refuses(cuda_device):
    """Budget 100: put 40, put 40, forget the first, put 50 fits only once the live block has moved to the arena's start."""
    rng = np.random.default_rng(0)
    cache, model = Cache(8, budget=100), CacheModel(8, 100, 100)
    b1, b2, b3 = _block(rng, 40), _block(rng, 40), _block(rng, 50)
    for p, b in (((2, 1), b1), ((3, 2), b2)):
        assert cache.put([p], [b], [0]) == _lib.BT_OK and model.put([p], [b], [0])
    cache.forget(1); model.forget(1)
    assert cache.put([(4, 3)], [b3], [0]) == _lib.BT_OK and model.put([(4, 3)], [b3], [0]) and model.compactions == 1
    _check_same(cache, model, rng)
    got, cnt = cache.gather([(4, 3), (3, 2)], [1, 0], [2, 1], 90)
    assert list(cnt) == [50, 40] and got.tobytes() == model.gather([(4, 3), (3, 2)], [1, 0], [2, 1]).tobytes()
    # 90 live + 11 > 100: refused, nothing changes; 10 more fits exactly
    assert cache.put([(5, 4)], [_block(rng, 11)], [0]) == _lib.BT_ERR_CAPACITY
    _check_same(cache, model, rng)
    b4 = _block(rng, 10)
    assert cache.put([(5, 4)], [b4], [0]) == _lib.BT_OK and model.put([(5, 4)], [b4], [0])
    _check_same(cache, model, rng)
    cache.close()


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_arena_equals_dict_model(cuda_device, seed):
    """Random puts (several pairs, re-puts, empty blocks, blocks of 0..300 entries), forgets and gathers; the budget is tight enough that
    many puts compact and some are refused."""
    rng = np.random.default_rng(seed)
    budget, max_pairs = 2000, 24
    cache, model = Cache(max_pairs, budget=budget), CacheModel(max_pairs, budget, budget)
    c = dict(put=0, refused=0, forget=0, repeat=0)
    for k in range(400):
        r = rng.random()
        if r < 0.6:
            n = int(rng.integers(1, 4))
            pairs = []
            for _ in range(n):
                a = int(rng.integers(1, 30))
                pairs.append((a, int(rng.integers(0, a))))
            c["repeat"] += any(p in model.d for p in pairs)
            blocks = [_block(rng, int(rng.integers(0, 301)) if rng.random() > 0.1 else 0) for _ in pairs]
            status = [int(rng.integers(0, 3)) for _ in pairs]
            ok = model.put(pairs, blocks, status)
            rc = cache.put(pairs, blocks, status)
            assert rc == (_lib.BT_OK if ok else _lib.BT_ERR_CAPACITY), (k, rc, ok)
            c["put"] += ok
            c["refused"] += not ok
        elif r < 0.8:
            f = int(rng.integers(0, 30))
            cache.forget(f); model.forget(f)
            c["forget"] += 1
        _check_same(cache, model, rng)
    assert c["put"] >= 50 and c["refused"] >= 10 and c["forget"] >= 40 and c["repeat"] >= 10 and model.compactions >= 10, (c, model.compactions)
    cache.close()


def test_per_pair_reserve_keeps_its_limits(cuda_device):
    """bt_match_cache_reserve(P, E): a block longer than E and a pair past P are refused; P full blocks fit whatever was forgotten before."""
    rng = np.random.default_rng(4)
    cache, model = Cache(4, per_pair=50), CacheModel(4, 200, 50)
    assert cache.put([(1, 0)], [_block(rng, 51)], [0]) == _lib.BT_ERR_CAPACITY
    for k in range(12):                       # churn: blocks of every size come and go, then four full blocks must still fit
        p = (k + 1, k)
        b = _block(rng, int(rng.integers(1, 51)))
        assert cache.put([p], [b], [0]) == _lib.BT_OK and model.put([p], [b], [0])
        if k % 2:
            cache.forget(k); model.forget(k)
        while len(model.d) >= 4:
            f = min(a for a, _ in model.d)
            cache.forget(f); model.forget(f)
    _check_same(cache, model, rng)
    full = [_block(rng, 50) for _ in range(4 - len(model.d))]
    pairs = [(100 + k, 99) for k in range(len(full))]
    assert cache.put(pairs, full, [0] * len(full)) == _lib.BT_OK and model.put(pairs, full, [0] * len(full))
    _check_same(cache, model, rng)
    assert cache.put([(200, 199)], [_block(rng, 1)], [0]) == _lib.BT_ERR_CAPACITY       # a fifth pair
    _check_same(cache, model, rng)
    cache.close()
