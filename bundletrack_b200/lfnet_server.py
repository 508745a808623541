"""LF-Net feature server on the device, speaking lf-net-release/run_server.py's ZMQ protocol, so unmodified clients (the reference's
Lfnet::detectFeature, sequence.LfnetClient) get their features without TensorFlow.  DESIGN.md §3.12.

Request: two message parts, int32 [W, H] and the W x H x 3 request bytes (FeatureManager.cpp:861-874).  Reply: three parts, int32 [n, dim],
float32 n x 2 keypoints in the 400 x 400 input and float32 n x dim descriptors (run_server.py:170-177).  The server binds a ROUTER socket, so
many REQ clients share one network: each turn takes every request already waiting (up to max_batch) and runs them in one bt_lfnet_detect.
It never waits for a batch to fill.  A request that is not 400 x 400 x 3 gets a reply with n = 0 and serving goes on (DESIGN.md §4)."""
from __future__ import annotations

import numpy as np

from .lfnet import SIDE

REQUEST_BYTES = SIDE * SIDE * 3


def request_image(body) -> np.ndarray | None:
    """The [400, 400, 3] uint8 image of a request's message parts (after the envelope), or None when they are not run_server.py's two
    parts with W = H = 400 and W x H x 3 image bytes."""
    if len(body) != 2 or len(body[0]) != 8 or len(body[1]) != REQUEST_BYTES:
        return None
    W, H = (int(v) for v in np.frombuffer(bytes(body[0]), np.int32))
    if W != SIDE or H != SIDE:
        return None
    return np.frombuffer(bytes(body[1]), np.uint8).reshape(SIDE, SIDE, 3)


def reply_parts(kpts: np.ndarray, desc: np.ndarray) -> list:
    """run_server.py's three reply parts for n keypoints (float32 n x 2) and descriptors (float32 n x dim)."""
    n, dim = desc.shape
    return [np.array([n, dim], np.int32).tobytes(), np.ascontiguousarray(kpts, np.float32).tobytes(), np.ascontiguousarray(desc, np.float32).tobytes()]


def empty_reply(dim: int) -> list:
    """The reply to a request the network does not take: n = 0."""
    return reply_parts(np.zeros((0, 2), np.float32), np.zeros((0, dim), np.float32))


def split_envelope(parts) -> tuple:
    """(routing envelope, body) of a message a ROUTER socket received: the envelope runs up to and including the first empty part (a REQ
    client's delimiter); without one, the first part is the peer's identity and the rest is the body."""
    for i, p in enumerate(parts):
        if len(p) == 0:
            return list(parts[:i + 1]), list(parts[i + 1:])
    return list(parts[:1]), list(parts[1:])


class LfnetServer:
    """run_server.py on an LfnetDevice (lfnet.load_lfnet or LfnetDevice.from_file), which the server takes over: close() closes it.

    serve_once(timeout_ms) waits up to timeout_ms for a request, then serves every request already waiting, up to max_batch (default: the
    network's max_images), with one bt_lfnet_detect and returns how many it answered.  serve_forever() repeats it until stop() is called
    from another thread or the process is interrupted.  The requests are staged through one pinned block and read back with one
    synchronisation per batch.  context: a zmq.Context to bind in (an inproc:// endpoint needs the clients'), else the server makes its own."""

    def __init__(self, net, endpoint: str, max_batch: int = None, context=None):
        import threading
        import torch
        import zmq
        self.net, self.endpoint = net, endpoint
        self.max_batch = net.max_images if max_batch is None else int(max_batch)
        if not 1 <= self.max_batch <= net.max_images:
            raise ValueError(f"max_batch {self.max_batch} outside [1, {net.max_images}] (the network's max_images)")
        self.dim, self.top_k = int(net.hp["desc_dim"]), int(net.hp["top_k"])
        dev = net.kpts.device
        self.torch, self.zmq = torch, zmq
        self.stream = torch.cuda.Stream(dev)
        B = self.max_batch
        self._req_host = torch.empty((B, SIDE, SIDE, 3), dtype=torch.uint8, pin_memory=True)
        self._req_dev = torch.empty((B, SIDE, SIDE, 3), dtype=torch.uint8, device=dev)
        self._kp_host = torch.empty((B, self.top_k, 2), dtype=torch.float32, pin_memory=True)
        self._de_host = torch.empty((B, self.top_k, self.dim), dtype=torch.float32, pin_memory=True)
        self._n_host = torch.empty((B,), dtype=torch.int32, pin_memory=True)
        self._stop = threading.Event()
        self._own_ctx = context is None
        self.ctx = zmq.Context() if context is None else context
        self.sock = self.ctx.socket(zmq.ROUTER)
        self.sock.setsockopt(zmq.LINGER, 0)
        self.sock.bind(endpoint)

    def _receive(self, timeout_ms: int) -> list:
        """[(envelope, body)] of every request waiting, up to max_batch; waits up to timeout_ms for the first."""
        zmq = self.zmq
        if not self.sock.poll(timeout_ms, zmq.POLLIN):
            return []
        out = []
        while len(out) < self.max_batch:
            try:
                out.append(split_envelope(self.sock.recv_multipart(zmq.NOBLOCK)))
            except zmq.Again:
                break
        return out

    def _detect(self, images: list) -> list:
        """One bt_lfnet_detect over the images; (kpts [n, 2], desc [n, dim]) host arrays per image."""
        torch = self.torch
        m = len(images)
        for i, img in enumerate(images):
            self._req_host[i].numpy()[...] = img
        with torch.cuda.stream(self.stream):
            self._req_dev[:m].copy_(self._req_host[:m], non_blocking=True)
            kp, de, nk = self.net.detect([self._req_dev[i] for i in range(m)], self.stream.cuda_stream)
            self._kp_host[:m].copy_(kp, non_blocking=True)
            self._de_host[:m].copy_(de, non_blocking=True)
            self._n_host[:m].copy_(nk, non_blocking=True)
        self.stream.synchronize()
        ns = self._n_host[:m].numpy()
        return [(self._kp_host[i, :ns[i]].numpy(), self._de_host[i, :ns[i]].numpy()) for i in range(m)]

    def serve_once(self, timeout_ms: int = 100) -> int:
        reqs = self._receive(timeout_ms)
        if not reqs:
            return 0
        images = [request_image(body) for _, body in reqs]
        good = [img for img in images if img is not None]
        feats = iter(self._detect(good) if good else [])
        for (env, _), img in zip(reqs, images):
            self.sock.send_multipart(env + (empty_reply(self.dim) if img is None else reply_parts(*next(feats))))
        return len(reqs)

    def serve_forever(self, poll_ms: int = 100) -> None:
        while not self._stop.is_set():
            self.serve_once(poll_ms)

    def stop(self) -> None:
        """Ends serve_forever after its current turn (at most poll_ms later); safe to call from any thread."""
        self._stop.set()

    def close(self) -> None:
        """Closes the socket, the zmq context if the server made it, and the network.  Call it after serve_forever has returned."""
        self._stop.set()
        if self.sock is not None:
            self.sock.close(0)
            self.sock = None
            if self._own_ctx:
                self.ctx.term()
        if self.net is not None:
            self.stream.synchronize()
            self.net.close()
            self.net = None
