"""sqrt_le_max (bt_common.cuh), the squared threshold RANSAC and the solver's dense term compare against, against a float32 restatement
of its rule: the largest float d with sqrtf(d) <= th, -1 when there is none.  Host code only: no library, no GPU."""
import os
import shutil
import subprocess
import textwrap

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _cuda_include():
    nvcc = shutil.which("nvcc")
    home = os.path.dirname(os.path.dirname(nvcc)) if nvcc else os.environ.get("CUDA_HOME", "/usr/local/cuda")
    return os.path.join(home, "include")


def _sqrt_le_max(tmp_path, th):
    """sqrt_le_max of every float32 in th, as the header computes it"""
    src = tmp_path / "sq.cpp"
    src.write_text(textwrap.dedent(r'''
        #include "bundletrack_b200/csrc/bt_common.cuh"
        int main() {
            uint32_t b;
            while (scanf("%x", &b) == 1) { float th; memcpy(&th, &b, 4); const float r = bt::sqrt_le_max(th); memcpy(&b, &r, 4); printf("%08x\n", b); }
            return 0;
        }
    '''))
    exe = tmp_path / "sq"
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-I", ROOT, "-I", _cuda_include(), str(src), "-o", str(exe)])
    bits = np.asarray(th, np.float32).view(np.uint32)
    out = subprocess.run([str(exe)], input="\n".join(f"{b:08x}" for b in bits), capture_output=True, text=True, timeout=120, check=True)
    return np.array([int(x, 16) for x in out.stdout.split()], np.uint32).view(np.float32)


def _rule(th):
    """largest float32 d >= 0 with np.sqrt(d) <= th (+inf included), by bisection over the bit patterns of [0, +inf]; -1 if none"""
    th = np.asarray(th, np.float32)
    f = lambda b: b.astype(np.uint32).view(np.float32)
    with np.errstate(invalid="ignore"):
        has = np.float32(0) <= th
        lo = np.zeros(th.shape, np.int64)                    # sqrt(f(lo)) <= th
        hi = np.full(th.shape, 0x7F800001, np.int64)         # past +inf
        while (hi - lo > 1).any():
            mid = (lo + hi) // 2
            ok = np.sqrt(f(mid)) <= th
            lo, hi = np.where(ok, mid, lo), np.where(ok, hi, mid)
    return np.where(has, f(lo), np.float32(-1))


def test_sqrt_le_max_matches_its_rule(tmp_path):
    fmax = np.finfo(np.float32).max
    named = np.array([0.0, -0.0, np.float32(1e-45), 1e-38, 0.0005, 0.005, 0.02, 1.0, 3e19, fmax], np.float32)
    rng = np.random.default_rng(0)
    bits = rng.integers(0, 0x7F800000, 4000, dtype=np.int64).astype(np.uint32) | (rng.integers(0, 2, 4000, dtype=np.uint32) << 31)
    rand = bits.view(np.float32)                             # finite floats of either sign, uniform over the bit patterns
    th = np.concatenate([named, rand])
    got, want = _sqrt_le_max(tmp_path, th), _rule(th)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), th[got.view(np.uint32) != want.view(np.uint32)][:10]
    assert (got[:2] == 0).all() and got[len(named) - 1] == fmax and (got[len(named):][rand < 0] == -1).all()
    special = np.array([-1.0, np.nan, -np.inf, np.inf], np.float32)
    assert _sqrt_le_max(tmp_path, special).tolist() == [-1.0, -1.0, -1.0, np.inf]
    assert _rule(special).tolist() == [-1.0, -1.0, -1.0, np.inf]
