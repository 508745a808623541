"""GPU tests of the LF-Net feature server (bundletrack_b200.lfnet_server) run in-process on a private endpoint: replies equal LfnetDevice.detect
byte for byte in run_server.py's wire layout; concurrent clients get what sequential ones get; run_sequence through an LfnetClient equals the
device source; a malformed request is answered with n = 0 and serving goes on; close() frees everything the server held."""
import ctypes
import os
import threading

import numpy as np
import pytest

from bundletrack_b200 import _lib, lfnet, sequence, synth
from bundletrack_b200.lfnet_server import LfnetServer
from oracle import lfnet_oracle as lo

pytestmark = pytest.mark.gpu
HP = dict(lfnet.DEFAULTS)
zmq = pytest.importorskip("zmq")


def _live():
    d, p, h = ctypes.c_longlong(), ctypes.c_longlong(), ctypes.c_int()
    _lib.check(_lib.load().bt_debug_live_resources(ctypes.byref(d), ctypes.byref(p), ctypes.byref(h)))
    return d.value, p.value, h.value


@pytest.fixture(scope="module")
def weights():
    return lo.random_weights(lfnet.weight_shapes(HP), 11)


@pytest.fixture(scope="module")
def weights_file(weights, tmp_path_factory):
    path = tmp_path_factory.mktemp("srv") / "net.btlfnet"
    path.write_bytes(lfnet.weights_file_bytes(lfnet.make_blob(weights, HP), HP))
    return str(path)


@pytest.fixture(scope="module")
def reference(weights, cuda_device):
    net = lfnet.LfnetDevice(weights, HP)
    yield net
    net.close()


class Running:
    """A server on an inproc endpoint, served by one thread until stop()."""

    def __init__(self, weights_file, name, max_batch=8):
        self.ctx = zmq.Context()
        self.endpoint = f"inproc://lfnet-{name}"
        self.server = LfnetServer(lfnet.LfnetDevice.from_file(weights_file, max_images=max_batch), self.endpoint, context=self.ctx)
        self.batches, self.sockets = [], []
        detect = self.server._detect
        self.server._detect = lambda images: (self.batches.append(len(images)), detect(images))[1]
        self.thread = threading.Thread(target=self.server.serve_forever, kwargs=dict(poll_ms=20))
        self.thread.start()

    def socket(self):
        s = self.ctx.socket(zmq.REQ)
        s.setsockopt(zmq.LINGER, 0)
        s.connect(self.endpoint)
        self.sockets.append(s)
        return s

    def stop(self):
        for s in self.sockets:          # (zmq's term waits for every socket of the context)
            s.close(0)
        self.server.stop()
        self.thread.join()
        self.server.close()
        self.ctx.term()


def _images(n, seed):
    """Request images: synthetic scenes through bt_lfnet_request's shape (a masked object on black) and plain noise."""
    rng = np.random.default_rng(seed)
    out = []
    yy, xx = np.mgrid[0:400, 0:400]
    for k in range(n):
        img = rng.integers(0, 256, (400, 400, 3), dtype=np.uint8)
        if k % 2:
            img[(xx - 200 - 10 * k) ** 2 + (yy - 190) ** 2 > (110 + 5 * k) ** 2] = 0
        out.append(img)
    return out


def _request(img):
    return [np.array([img.shape[1], img.shape[0]], np.int32).tobytes(), np.ascontiguousarray(img).tobytes()]


def _expected(reference, img):
    import torch
    kp, de, nk = reference.detect([torch.from_numpy(img).to(reference.kpts.device)])
    torch.cuda.synchronize()
    n = int(nk[0])
    return [np.array([n, HP["desc_dim"]], np.int32).tobytes(), kp[0, :n].cpu().numpy().tobytes(), de[0, :n].cpu().numpy().tobytes()]


def _ask(sock, parts, timeout_ms=60000):
    sock.send_multipart(parts)
    assert sock.poll(timeout_ms, zmq.POLLIN), "no reply"
    return sock.recv_multipart()


def test_replies_equal_detect_and_the_wire_layout(weights_file, reference):
    srv = Running(weights_file, "replies")
    try:
        s = srv.socket()
        for img in _images(4, 1):
            got = _ask(s, _request(img))
            want = _expected(reference, img)
            assert len(got) == 3 and got == want
            n, dim = np.frombuffer(got[0], np.int32)
            assert n > 0 and dim == HP["desc_dim"] and len(got[1]) == 8 * n and len(got[2]) == 4 * n * dim
    finally:
        srv.stop()


def test_concurrent_clients_get_the_bytes_of_sequential_requests(weights_file, reference):
    """Four LfnetClients on threads of their own send interleaved requests; every reply equals the single request's."""
    imgs = _images(6, 2)
    roi = (40, 290, 30, 220)
    srv = Running(weights_file, "concurrent")
    try:
        seq_cl = sequence.LfnetClient(srv.endpoint, timeout_s=60, context=srv.ctx)
        try:
            want = [seq_cl(str(k), img, roi) for k, img in enumerate(imgs)]
        finally:
            seq_cl.close()
        assert set(srv.batches) == {1}
        srv.batches.clear()
        got, errors = {}, []
        start = threading.Barrier(4)

        def client(c):
            cl = sequence.LfnetClient(srv.endpoint, timeout_s=60, context=srv.ctx)
            try:
                start.wait()
                for r in range(5):
                    k = (c + r) % len(imgs)
                    got[(c, r)] = (k, cl(f"{c}-{r}", imgs[k], roi))
            except Exception as e:       # reported by the main thread
                errors.append(e)
            finally:
                cl.close()
        threads = [threading.Thread(target=client, args=(c,)) for c in range(4)]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
        assert not errors, errors
        assert len(got) == 20
        for (k, (kp, de)) in got.values():
            assert kp.tobytes() == want[k][0].tobytes() and de.tobytes() == want[k][1].tobytes()
        print("batch sizes the server ran:", srv.batches)
        assert sum(srv.batches) == 20 and max(srv.batches) <= 8
    finally:
        srv.stop()


def test_malformed_request_mid_run_gets_n_zero_and_serving_goes_on(weights_file, reference):
    img = _images(1, 3)[0]
    srv = Running(weights_file, "malformed")
    try:
        s = srv.socket()
        want = _expected(reference, img)
        assert _ask(s, _request(img)) == want
        small = np.zeros((240, 320, 3), np.uint8)
        for bad in (_request(small), [_request(img)[0]], [_request(img)[0], _request(img)[1][:-3]], _request(img) + [b"extra"]):
            rep = _ask(s, bad)
            assert rep == [np.array([0, HP["desc_dim"]], np.int32).tobytes(), b"", b""]
        assert _ask(s, _request(img)) == want
    finally:
        srv.stop()


def test_run_sequence_through_the_server_equals_the_device_source(tmp_path, weights_file, reference):
    H, W, N = 240, 320, 8
    seq = synth.make_sequence(31, N, H=H, W=W, roi_fail=(3,))
    video = tmp_path / "video"
    synth.write_ycbineoat_video(seq, str(video))
    loader = sequence.YcbineoatVideo(str(video))
    res_dev = sequence.run_sequence(loader, None, reference, str(tmp_path / "dev"), max_feats=HP["top_k"], device=0)
    srv = Running(weights_file, "sequence")
    try:
        cl = sequence.LfnetClient(srv.endpoint, timeout_s=60, context=srv.ctx)
        try:
            res_srv = sequence.run_sequence(loader, None, cl, str(tmp_path / "srv"), max_feats=HP["top_k"], device=0)
        finally:
            cl.close()
    finally:
        srv.stop()
    assert [r[:2] for r in res_dev] == [r[:2] for r in res_srv]
    files = sorted(os.listdir(tmp_path / "dev" / "poses"))
    assert files == sorted(os.listdir(tmp_path / "srv" / "poses")) and len(files) == N
    for f in files:
        assert (tmp_path / "dev" / "poses" / f).read_bytes() == (tmp_path / "srv" / "poses" / f).read_bytes(), f
    assert sum(r[1] == _lib.BT_FRAME_OTHER for r in res_srv) >= 2
    print("device source:", sequence.summary(res_dev))
    print("server:", sequence.summary(res_srv))


def test_close_frees_what_the_server_held(weights_file, cuda_device):
    before = _live()
    srv = Running(weights_file, "close")
    s = srv.socket()
    assert len(_ask(s, _request(_images(1, 4)[0]))) == 3
    s.close(0)
    assert _live() != before
    srv.stop()
    assert not srv.thread.is_alive()
    assert _live() == before
