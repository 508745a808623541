"""bt_match_viz on the device against the numpy oracle (oracle/matchviz_oracle.py) and the cv2-recorded golden images, byte for byte;
batched calls against single calls; the capacity and argument errors; and no resource left behind."""
import ctypes
import hashlib
import os

import numpy as np
import pytest

from bundletrack_b200 import _lib
from bundletrack_b200.overlay import MatchViz, match_image_shape
from oracle import matchviz_oracle as mv
from oracle import segment_oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = np.load(os.path.join(ROOT, "tests", "golden", "ref_matchviz.npz"))
NAMES = [str(n) for n in GOLDEN["names"]]


def _live():
    lib = _lib.load()
    d, p, h = ctypes.c_longlong(), ctypes.c_longlong(), ctypes.c_int()
    assert lib.bt_debug_live_resources(ctypes.byref(d), ctypes.byref(p), ctypes.byref(h)) == 0
    return d.value, p.value, h.value


def _golden_jobs():
    colour = segment_oracle.test_colour(int(GOLDEN["H"]), int(GOLDEN["W"]))
    state = mv.RNG_DEFAULT
    jobs = []
    for name in NAMES:
        seed = int(GOLDEN[f"{name}/seed"])
        if seed:
            state = mv.rng_seed(seed)
        ra, rb, uv = GOLDEN[f"{name}/roi_a"], GOLDEN[f"{name}/roi_b"], GOLDEN[f"{name}/uv"]
        jobs.append((name, (colour, ra, colour, rb, uv, state)))
        state = mv.rng_advance(state, len(uv))
    return jobs


def _random_jobs(seed, n_images, max_n=60):
    rs = np.random.default_rng(seed)
    H, W = 120, 160
    jobs = []
    for _ in range(n_images):
        ca = rs.integers(0, 256, (H, W, 3), dtype=np.uint8)
        cb = rs.integers(0, 256, (H, W, 3), dtype=np.uint8)
        rois = []
        for _ in range(2):
            u0, v0 = int(rs.integers(0, W - 2)), int(rs.integers(0, H - 2))
            rois.append((u0, int(rs.integers(u0 + 1, W + 1)), v0, int(rs.integers(v0 + 1, H + 1))))
        ra, rb = rois
        n = int(rs.integers(0, max_n))
        uv = np.stack([rs.uniform(ra[0] - 2, ra[1] + 2, n), rs.uniform(ra[2] - 2, ra[3] + 2, n),
                       rs.uniform(rb[0] - 2, rb[1] + 2, n), rs.uniform(rb[2] - 2, rb[3] + 2, n)], 1).astype(np.float32)
        jobs.append((ca, ra, cb, rb, uv, int(rs.integers(1, 2 ** 63))))
    return jobs


@pytest.mark.gpu
def test_device_equals_golden_images():
    jobs = _golden_jobs()
    mz = MatchViz(max_images=len(jobs), max_matches=sum(len(j[4]) for _, j in jobs))
    got = mz.draw_host([j for _, j in jobs])
    for (name, _), img in zip(jobs, got):
        assert img.shape == tuple(GOLDEN[f"{name}/shape"]), name
        if f"{name}/image" in GOLDEN.files:
            assert img.tobytes() == GOLDEN[f"{name}/image"].tobytes(), name
        else:
            assert hashlib.sha256(img.tobytes()).hexdigest() == str(GOLDEN[f"{name}/sha256"]), name
    mz.close()


@pytest.mark.gpu
def test_device_equals_oracle_and_batches_equal_single_calls():
    jobs = _random_jobs(7, 40)
    mz = MatchViz(max_images=len(jobs), max_matches=sum(len(j[4]) for j in jobs))
    batch = mz.draw_host(jobs)
    for k, j in enumerate(jobs):
        ref, _ = mv.match_image(*j)
        assert batch[k].tobytes() == ref.tobytes(), k
        assert mz.draw_host([j])[0].tobytes() == batch[k].tobytes(), k
    mz.close()


@pytest.mark.gpu
def test_large_scale_images_and_many_matches():
    """Thin ROIs give scale 90 and images wider than JPEG allows; a dense list crosses many 256-match chunks."""
    rs = np.random.default_rng(3)
    colour = segment_oracle.test_colour(480, 640)
    ra, rb = (0, 640, 100, 110), (0, 640, 300, 310)
    n = 700
    uv = np.stack([rs.uniform(0, 640, n), rs.uniform(100, 110, n), rs.uniform(0, 640, n), rs.uniform(300, 310, n)], 1).astype(np.float32)
    job = (colour, ra, colour, rb, uv, 99)
    assert match_image_shape(ra, rb) == (900, 2 * 640 * 90)
    mz = MatchViz(max_images=1, max_matches=n)
    img = mz.draw_host([job])[0]
    ref, _ = mv.match_image(*job)
    assert img.tobytes() == ref.tobytes()
    mz.close()


@pytest.mark.gpu
def test_errors_and_resources():
    import torch
    before = _live()
    jobs = _random_jobs(1, 3, max_n=30)
    mz = MatchViz(max_images=2, max_matches=1000)
    with pytest.raises(_lib.BtError) as e:
        mz.draw_host(jobs)                                      # 3 images > 2 reserved
    assert e.value.rc == _lib.BT_ERR_CAPACITY
    mz2 = MatchViz(max_images=4, max_matches=5, ctx=mz.ctx)
    big = [(jobs[0][0], jobs[0][1], jobs[0][2], jobs[0][3], np.zeros((6, 4), np.float32), 1)]
    with pytest.raises(_lib.BtError) as e:
        mz2.draw_host(big)                                      # 6 matches > 5 reserved
    assert e.value.rc == _lib.BT_ERR_CAPACITY
    with pytest.raises(_lib.BtError) as e:
        MatchViz(max_images=65536, ctx=mz.ctx)                  # more images than one launch's grid rows
    assert e.value.rc == _lib.BT_ERR_INVALID_ARG
    bad = [(jobs[0][0], (0, 10, 0, 200), jobs[0][2], jobs[0][3], None, 1)]  # ROI below the image
    dev = torch.device("cuda", 0)
    c = torch.from_numpy(jobs[0][0]).to(dev)
    out = torch.empty((*match_image_shape(bad[0][1], jobs[0][3]), 3), dtype=torch.uint8, device=dev)
    with pytest.raises(_lib.BtError) as e:
        mz2.draw([(c, bad[0][1], c, jobs[0][3], None, 1)], [out])
    assert e.value.rc == _lib.BT_ERR_INVALID_ARG
    mz.close()
    assert _live() == before


@pytest.mark.gpu
def test_draw_rejects_tensors_the_kernels_cannot_read():
    """Host tensors, wrong dtypes, strided views and wrong shapes are refused before any pointer reaches the library."""
    import torch
    dev = torch.device("cuda", 0)
    ca, ra, cb, rb, uv, st = _random_jobs(2, 1, max_n=10)[0]
    uv = np.zeros((4, 4), np.float32) + np.array([ra[0], ra[2], rb[0], rb[2]], np.float32)
    good = lambda: [torch.from_numpy(ca).to(dev), ra, torch.from_numpy(cb).to(dev), rb, torch.from_numpy(uv).to(dev), st]
    out = lambda: torch.empty((*match_image_shape(ra, rb), 3), dtype=torch.uint8, device=dev)
    mz = MatchViz(max_images=1, max_matches=16)
    mz.draw([tuple(good())], [out()])                                           # the well-formed call goes through
    bt = mz.lib.bt_stream_sync(mz.stream)
    assert bt == 0
    bad = []
    j = good(); j[0] = torch.from_numpy(ca); bad.append((j, out()))               # host colour
    j = good(); j[2] = j[2].float(); bad.append((j, out()))                      # float colour
    j = good(); j[4] = j[4].double(); bad.append((j, out()))                     # float64 uv
    j = good(); j[4] = torch.zeros((4, 8), device=dev)[:, ::2]; bad.append((j, out()))   # strided uv
    j = good(); j[4] = j[4][:, :3].contiguous(); bad.append((j, out()))          # [n, 3] uv
    j = good(); bad.append((j, out()[:-1]))                                      # output one row short
    j = good(); bad.append((j, out().cpu()))                                     # host output
    for j, o in bad:
        with pytest.raises(ValueError):
            mz.draw([tuple(j)], [o])
    mz.close()
