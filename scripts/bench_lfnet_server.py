"""The LF-Net feature server (bundletrack_b200.lfnet_server) under load: requests per second and median / p90 round-trip latency with 1, 4
and 8 concurrent REQ clients, against LfnetDevice.detect called directly on the same requests (host image in, host reply out: the work a
server turn does for one request, without ZMQ).  The server runs in this process on a thread of its own, on an ipc:// endpoint in a temporary
directory; each client is a thread with its own REQ socket, as sequence.LfnetClient is.  Seeded random weights, 400 x 400 requests from
synthetic scenes.  Prints one JSON object; --out also writes it to a file.

    python scripts/bench_lfnet_server.py [--requests 40] [--out results.json]"""
import argparse
import json
import os
import shutil
import tempfile
import threading
import time

import numpy as np

import benchkit


def stats(lat_s, wall_s, n):
    ms = np.asarray(lat_s) * 1000
    return {"requests": int(n), "requests_per_s": round(n / wall_s, 1), "median_ms": round(float(np.median(ms)), 3),
            "p90_ms": round(float(np.percentile(ms, 90)), 3)}


def direct(net, images, iters):
    """LfnetDevice.detect on one host request per call, the reply read back: iters calls in a row."""
    import torch
    dev = net.kpts.device
    lat = []
    for it in range(iters + 3):
        t0 = time.perf_counter()
        kp, de, nk = net.detect([torch.from_numpy(images[it % len(images)]).to(dev)])
        n = int(nk[0])
        kp[0, :n].cpu().numpy().tobytes(), de[0, :n].cpu().numpy().tobytes()
        if it >= 3:
            lat.append(time.perf_counter() - t0)
    return stats(lat, sum(lat), len(lat))


def direct_batch(net, images, iters):
    """LfnetDevice.detect on 8 host requests per call."""
    import torch
    dev = net.kpts.device
    lat = []
    for it in range(iters + 3):
        t0 = time.perf_counter()
        kp, de, nk = net.detect([torch.from_numpy(im).to(dev) for im in images[:8]])
        kp.cpu(), de.cpu(), nk.cpu()
        if it >= 3:
            lat.append(time.perf_counter() - t0)
    return {"ms_per_call_median": round(float(np.median(lat)) * 1000, 3), "ms_per_request": round(float(np.median(lat)) * 1000 / 8, 3)}


def served(endpoint, ctx, images, n_clients, per_client):
    import zmq
    lat, lock = [], threading.Lock()
    start = threading.Barrier(n_clients + 1)

    def client(c):
        s = ctx.socket(zmq.REQ)
        s.setsockopt(zmq.LINGER, 0)
        s.connect(endpoint)
        mine = []
        try:
            for r in range(2):                           # warm-up round trips
                s.send_multipart(req(images[(c + r) % len(images)]))
                s.recv_multipart()
            start.wait(timeout=300)
            for r in range(per_client):
                t0 = time.perf_counter()
                s.send_multipart(req(images[(c + r) % len(images)]))
                s.recv_multipart()
                mine.append(time.perf_counter() - t0)
        finally:
            s.close(0)
        with lock:
            lat.extend(mine)
    threads = [threading.Thread(target=client, args=(c,)) for c in range(n_clients)]
    for t in threads:
        t.start()
    start.wait(timeout=300)
    t0 = time.perf_counter()
    for t in threads:
        t.join()
    return stats(lat, time.perf_counter() - t0, len(lat))


def req(img):
    return [np.array([img.shape[1], img.shape[0]], np.int32).tobytes(), img.tobytes()]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--requests", type=int, default=40, help="requests per client")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    import zmq
    from bench_lfnet import requests
    from bundletrack_b200 import lfnet
    from bundletrack_b200.lfnet_server import LfnetServer
    from oracle import lfnet_oracle as lo
    dev = torch.device("cuda:0")
    hp = dict(lfnet.DEFAULTS)
    w = lo.random_weights(lfnet.weight_shapes(hp), 11)
    images = [r.cpu().numpy() for r in requests(dev, 8)]
    res = {"card": benchkit.card(), "torch": torch.__version__}
    net = lfnet.LfnetDevice(w, hp, max_images=8)
    res["direct_1"] = direct(net, images, a.requests * 2)
    res["direct_batch_8"] = direct_batch(net, images, a.requests)
    net.close()
    tmp = tempfile.mkdtemp()
    endpoint = f"ipc://{tmp}/lfnet.sock"
    ctx = zmq.Context()
    server = LfnetServer(lfnet.LfnetDevice(w, hp, max_images=8), endpoint, context=ctx)
    batches = []
    detect = server._detect
    server._detect = lambda ims: (batches.append(len(ims)), detect(ims))[1]
    th = threading.Thread(target=server.serve_forever, kwargs=dict(poll_ms=50))
    th.start()
    try:
        for c in (1, 4, 8):
            batches.clear()
            r = served(endpoint, ctx, images, c, a.requests)
            r["mean_batch"] = round(float(np.mean(batches)), 2)
            res[f"server_{c}_clients"] = r
    finally:
        server.stop()
        th.join()
        server.close()
        ctx.term()
        shutil.rmtree(tmp, ignore_errors=True)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
