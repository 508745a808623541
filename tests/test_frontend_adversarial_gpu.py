"""The fused frame front end (bt_frames_preprocess) against its float64 statement (oracle.frame_oracle.preprocess64) on frames built to
sit on its edges (oracle/frame_families.py): every size around the 64 x 32 tile and the image border, every (erode, filter) radius
pair the halo admits, and the gate equalities of erode, the filter and the normals.

No fraction of pixels is allowed to differ.  Every pixel outside preprocess64's taint mask must meet its per-pixel bound
(frame_oracle.device_report; pixels fed by subnormal filter weights must also stay within 2e-6 / 3e-6 / 1e-3 of the float32
restatement), and the number of tainted pixels must be the one the family records: 0 except for filter_marginal, built so that the
float32 mean gate decides some taps the other way from float64."""
import numpy as np
import pytest

from oracle import frame_families as ff
from oracle import frame_oracle as fo

pytestmark = pytest.mark.gpu
FAMILIES = {f["name"]: f for f in ff.families()}


@pytest.fixture(scope="module")
def fe(cuda_device):
    from bundletrack_b200.frontend import FrameFrontEnd
    f = FrameFrontEnd()
    yield f
    f.close()


def run(fe, raws, K, dp, dev, want_xyz=True):
    """One bt_frames_preprocess call over raws (same size); outputs start as the -7 sentinel."""
    import torch
    from bundletrack_b200 import _lib
    full = dict(fo.DEFAULTS, **dp)
    fe.params = _lib.DepthParams(int(full["erode_radius"]), full["erode_diff"], full["erode_ratio"], int(full["bf_radius"]), full["sigma_D"], full["sigma_R"])
    H, W = raws[0].shape
    tin = [torch.from_numpy(np.ascontiguousarray(r)).to(dev) for r in raws]
    dout = [torch.full((H, W), -7.0, device=dev) for _ in raws]
    nout = [torch.full((H, W, 4), -7.0, device=dev) for _ in raws]
    xout = [torch.full((H, W, 4), -7.0, device=dev) for _ in raws] if want_xyz else None
    fe.process(tin, H, W, K, dout, nout, xout)
    torch.cuda.synchronize()
    return [d.cpu().numpy() for d in dout], [n.cpu().numpy() for n in nout], ([x.cpu().numpy() for x in xout] if want_xyz else [None] * len(raws))


@pytest.mark.parametrize("name", list(FAMILIES))
def test_family(fe, cuda_device, name):
    fam = FAMILIES[name]
    d, n, x = run(fe, fam["frames"], fam["K"], fam["dp"], cuda_device)
    for i, raw in enumerate(fam["frames"]):
        r = fo.preprocess64(raw, fam["K"], fam["dp"])
        rep = fo.device_report(d[i], x[i], n[i], r, fo.preprocess(raw, fam["K"], fam["dp"]))
        print(f"{name}[{i}] {raw.shape}: tainted {rep['tainted']}, subnormal-weight {rep['subnormal']}, valid {rep['valid']}, "
              f"worst error / bound: depth {rep['depth_frac']:.3f} "
              f"xyz {rep['xyz_frac']:.3f} normal {rep['normal_frac']:.3f}")
        if rep["tainted"]:
            print("  tainted pixels:", np.argwhere(r.taint).tolist()[:50])
        assert not rep["failures"], f"{name}[{i}]: " + "; ".join(rep["failures"])
        assert rep["tainted"] == fam["taint"][i]


def test_gate_cells_decide_as_claimed(fe, cuda_device):
    """The erode cells, where br = 0 shows erode's decision in the output: each claimed cell is untainted and kept or zeroed as in
    float64, and both outcomes occur in every family.  (The filter's and the normals' gate cells move values, not zeros; test_family
    holds them to their bounds.)"""
    for name in ("erode_diff", "erode_validity", "erode_ratio_eq", "erode_ratio_up", "erode_ratio_down"):
        fam = FAMILIES[name]
        d, _, _ = run(fe, fam["frames"], fam["K"], fam["dp"], cuda_device)
        r = fo.preprocess64(fam["frames"][0], fam["K"], fam["dp"])
        outcomes = set()
        for kind, i, y, x, v in fam["claims"]:
            if kind == "erode_diff":
                y, x = v
            assert not r.taint[y, x]
            outcomes.add(bool(r.depth[y, x] > 0))
            assert (d[i][y, x] > 0) == (r.depth[y, x] > 0), f"{name}: {kind} cell ({y}, {x})"
        assert outcomes == {True, False}, name


def test_batch_equals_single_frames(fe, cuda_device):
    """One call over 40 frames of one size mixing every family built at 33 x 65 (run at the shipped parameters), and one over 300 frames of
    3 x 3: each frame's maps equal, bit for bit, what the frame gets alone."""
    raws = [f["frames"][i] for f in FAMILIES.values() for i in range(len(f["frames"])) if f["frames"][i].shape == (ff.EH, ff.EW)]
    raws = (raws * 4)[:40]
    rng = np.random.default_rng(3)
    small = [np.where(rng.random((3, 3)) < 0.8, rng.uniform(0.3, 0.9, (3, 3)), 0).astype(np.float32) for _ in range(300)]
    for frames in (raws, small):
        d, n, x = run(fe, frames, ff.K, ff.SHIPPED, cuda_device)
        for i in list(range(0, len(frames), 7)) + [len(frames) - 1]:
            d1, n1, x1 = run(fe, [frames[i]], ff.K, ff.SHIPPED, cuda_device)
            assert np.array_equal(d1[0].view(np.uint32), d[i].view(np.uint32))
            assert np.array_equal(n1[0].view(np.uint32), n[i].view(np.uint32))
            assert np.array_equal(x1[0].view(np.uint32), x[i].view(np.uint32))
