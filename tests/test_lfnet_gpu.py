"""GPU tests of LF-Net on the device (bt_lfnet_detect) against the float64 restatement of the reference's graph (oracle/lfnet_oracle.py):
dense maps, keypoint sets (marginal pixels listed), refined keypoints and descriptors; batching and repeat determinism; and run_sequence
with the device source against a host callable that returns the same features."""
import os

import numpy as np
import pytest

from bundletrack_b200 import _lib, lfnet, sequence, synth
from oracle import lfnet_oracle as lo

pytestmark = pytest.mark.gpu
HP = dict(lfnet.DEFAULTS)


@pytest.fixture(scope="module")
def weights():
    return lo.random_weights(lfnet.weight_shapes(HP), 11)


@pytest.fixture(scope="module")
def requests(cuda_device):
    """Requests made by bt_lfnet_request from synthetic scenes: largest-hull and as-is masks, and one nearly empty as-is mask (two
    specks far apart: a large ROI around almost nothing, so fewer NMS peaks than top_k are selected)."""
    import torch
    from bundletrack_b200.frontend import FrameFrontEnd
    H, W = 240, 320
    seq = synth.make_sequence(23, 2, H=H, W=W)
    speck = np.zeros((H, W), np.uint8)
    speck[30, 40] = speck[200, 290] = 255
    cases = [(seq.colour[0], seq.mask[0], _lib.BT_MASK_LARGEST_HULL), (seq.colour[1], seq.mask[1], _lib.BT_MASK_AS_IS),
             (seq.colour[1], speck, _lib.BT_MASK_AS_IS)]
    fe = FrameFrontEnd()
    out = []
    for colour, mask, mode in cases:
        dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda_device)
        d, nrm, fg = torch.empty((H, W), device=cuda_device), torch.empty((H, W, 4), device=cuda_device), torch.empty((H, W), dtype=torch.uint8, device=cuda_device)
        req = torch.zeros((400, 400, 3), dtype=torch.uint8, device=cuda_device)
        fe.process_masked([dev(seq.depth_raw[0])], [dev(mask)], H, W, seq.K, [d], [nrm], [fg], mode=mode)
        fe.lfnet_request([dev(colour)], [fg], H, W, [req])
        torch.cuda.synchronize()
        out.append(req)
    fe.close()
    return out


@pytest.fixture(scope="module")
def net(weights, cuda_device):
    n = lfnet.LfnetDevice(weights, HP, max_images=8)
    yield n
    n.close()


def _run(net, reqs):
    import torch
    kp, de, nk = net.detect(reqs)
    torch.cuda.synchronize()
    return kp.cpu().numpy(), de.cpu().numpy(), nk.cpu().numpy()


def _debug(net, image):
    heat, scl = np.zeros((400, 400), np.float32), np.zeros((400, 400), np.float32)
    kint, ori = np.zeros((HP["top_k"], 2), np.int32), np.zeros((HP["top_k"], 2), np.float32)
    _lib.check(net.lib.bt_lfnet_debug_maps(net.ctx, image, _lib.ptr(heat), _lib.ptr(scl), _lib.ptr(kint), _lib.ptr(ori), net.stream))
    return heat, scl, kint, ori


# The dense maps agree to TOL relative (FP32 against float64: the soft scale's exp(100 p) turns the trunk's last-bit differences into
# up to about 1.5e-4 of max_heatmaps, DESIGN.md §9.13), so a comparison between two pixels is decided within rounding when their gap is inside both values' bound.
TOL = 2e-4


def _marginal(o):
    """Pixels whose selection is within rounding: an NMS comparison with a neighbour whose gap is within TOL of the two values, or a score
    within TOL of the k-th value."""
    h = o["max_heatmaps"]
    hk = HP["nms_ksize"] // 2
    hp = np.pad(h, hk)
    H, W = h.shape
    near = np.zeros(h.shape, bool)
    for dy in range(2 * hk + 1):
        for dx in range(2 * hk + 1):
            if dy == hk and dx == hk:
                continue
            nb = hp[dy:dy + H, dx:dx + W]
            near |= (h > 0) & (np.abs(h - nb) <= TOL * (h + nb))
    s = o["nms_scores"].reshape(-1)
    kth = np.sort(s)[::-1][HP["top_k"] - 1]
    near |= (o["nms_maps"] > 0) & (np.abs(o["nms_scores"] - kth) <= TOL * (o["nms_scores"] + kth))
    return near


def test_against_oracle(net, requests, weights):
    kp, de, nk = _run(net, requests)
    for i, req in enumerate(requests):
        o = lo.detect(req.cpu().numpy(), weights, HP)
        heat, scl, kint, ori = _debug(net, i)
        for name, got, ref in (("max_heatmaps", heat, o["max_heatmaps"]), ("max_scales", scl, o["max_scales"])):
            rel = np.abs(got - ref) / np.maximum(np.abs(ref), 1e-3 * np.abs(ref).max())
            print(f"request {i}: {name} max relative error {rel.max():.2e}")
            assert rel.max() <= TOL, (i, name, rel.max())
        n = int(nk[i])
        marg = _marginal(o)
        gi, oi = kint[:n], o["kpts_int"]
        keep_g = ~marg[gi[:, 1], gi[:, 0]]
        keep_o = ~marg[oi[:, 1], oi[:, 0]]
        listed = sorted(set(map(tuple, gi[~keep_g])) | set(map(tuple, oi[~keep_o])))
        print(f"request {i}: {n} keypoints (oracle {len(oi)}), marginal pixels {listed}")
        if not np.array_equal(gi[keep_g], oi[keep_o]):
            h, sc = o["max_heatmaps"], o["nms_scores"]
            kth = np.sort(sc.reshape(-1))[::-1][HP["top_k"] - 1]
            for x, y in sorted(set(map(tuple, gi[keep_g])) ^ set(map(tuple, oi[keep_o]))):
                win = h[max(y - 2, 0):y + 3, max(x - 2, 0):x + 3]
                gap = np.abs(win - h[y, x])[np.abs(win - h[y, x]) > 0].min()
                print(f"request {i} differs at ({x}, {y}): heat {h[y, x]:.9g} device {heat[y, x]:.9g}, nearest neighbour gap {gap:.3g}, "
                      f"score {sc[y, x]:.9g} vs k-th {kth:.9g}")
        assert np.array_equal(gi[keep_g], oi[keep_o]), i
        if not listed:
            assert n == len(oi)
        # the same integer keypoints: refined positions, orientations, descriptors
        pos_o = {tuple(p): j for j, p in enumerate(oi)}
        pairs = [(j, pos_o[tuple(p)]) for j, p in enumerate(gi) if tuple(p) in pos_o]
        assert len(pairs) >= n - len(listed)
        g_idx, o_idx = np.array([a for a, _ in pairs]), np.array([b for _, b in pairs])
        dk = np.abs(kp[i, g_idx] - o["kpts"][o_idx]).max()
        do = np.abs(ori[g_idx] - o["ori"][o_idx]).max()
        dd = np.abs(de[i, g_idx] - o["desc"][o_idx]).max()
        print(f"request {i}: refined keypoints {dk:.2e} px, orientations {do:.2e}, descriptors {dd:.2e}")
        assert dk <= 1e-3 and dd <= 1e-4, (i, dk, dd)
        assert not kp[i, n:].any() and not de[i, n:].any()
    assert nk[2] < HP["top_k"], "the nearly empty mask should select fewer peaks than top_k"


def test_batch_equals_single_calls_and_repeats(net, requests):
    reqs = [requests[k % len(requests)] for k in range(8)]
    kp8, de8, n8 = _run(net, reqs)
    kp8b, de8b, n8b = _run(net, reqs)
    assert np.array_equal(n8, n8b) and np.array_equal(kp8.view(np.uint32), kp8b.view(np.uint32)) and np.array_equal(de8.view(np.uint32), de8b.view(np.uint32))
    for k, r in enumerate(reqs):
        kp1, de1, n1 = _run(net, [r])
        assert n1[0] == n8[k]
        assert np.array_equal(kp1[0].view(np.uint32), kp8[k].view(np.uint32)) and np.array_equal(de1[0].view(np.uint32), de8[k].view(np.uint32)), k


def test_reserve_and_detect_refusals(net, requests):
    import ctypes
    lib = net.lib
    bad = lfnet.params_struct(dict(HP, net_channel=32))
    assert lib.bt_lfnet_reserve(net.ctx, ctypes.byref(bad), 1) == _lib.BT_ERR_INVALID_ARG
    assert b"net_channel" in lib.bt_last_error()
    with pytest.raises(_lib.BtError):
        net.detect(requests * 3)                      # 9 > max_images
    blob = np.zeros(10, np.float32)
    assert lib.bt_lfnet_load_weights(net.ctx, _lib.ptr(blob), blob.size) == _lib.BT_ERR_INVALID_ARG


def test_run_sequence_device_source_equals_host_callable(tmp_path, net, cuda_device):
    """Only the transport differs: the host callable uploads the request, runs the same network and hands back host copies."""
    import torch
    H, W, N = 240, 320, 8
    seq = synth.make_sequence(31, N, H=H, W=W, roi_fail=(3,))
    video = tmp_path / "data" / "synthvideo"
    for k in range(N):
        for sub, img in (("rgb", seq.colour[k]), ("depth", np.round(seq.depth_raw[k] * 1000).astype(np.uint16)), ("masks", seq.mask[k])):
            os.makedirs(video / sub, exist_ok=True)
            synth.write_png(str(video / sub / f"{k:07d}.png"), img)
    K = np.array([[seq.K[0], 0, seq.K[2]], [0, seq.K[1], seq.K[3]], [0, 0, 1]])
    (video / "cam_K.txt").write_text("".join(" ".join(f"{v:.9g}" for v in row) + "\n" for row in K))
    (video / "annotated_poses").mkdir()
    for k in range(N):
        G = np.linalg.inv(np.asarray(seq.poses_gt[k], np.float64))
        (video / "annotated_poses" / f"{k:07d}.txt").write_text("".join(" ".join(f"{v:.9g}" for v in row) + "\n" for row in G))
    loader = sequence.YcbineoatVideo(str(video))

    def host(id_str, request, roi):
        kp, de, nk = net.detect([torch.from_numpy(request).to(cuda_device)])
        n = int(nk[0])
        if n == 0:
            raise sequence.DetectionFailed(id_str)
        from bundletrack_b200 import policy
        return policy.lfnet_reply_keypoints(n, HP["desc_dim"], kp[0, :n].cpu().numpy(), roi), de[0, :n].cpu().numpy()
    res_dev = sequence.run_sequence(loader, None, net, str(tmp_path / "dev"), max_feats=HP["top_k"], device=0)
    res_host = sequence.run_sequence(loader, None, host, str(tmp_path / "host"), max_feats=HP["top_k"], device=0)
    files = [sorted(os.listdir(tmp_path / d / "poses")) for d in ("dev", "host")]
    assert files[0] == files[1] and len(files[0]) == N
    for f in files[0]:
        assert open(tmp_path / "dev" / "poses" / f, "rb").read() == open(tmp_path / "host" / "poses" / f, "rb").read(), f
    assert [r[:2] for r in res_dev] == [r[:2] for r in res_host]
    assert sum(r[1] == _lib.BT_FRAME_OTHER for r in res_dev) >= 2
    print("device source:", sequence.summary(res_dev))
    print("host callable:", sequence.summary(res_host))
