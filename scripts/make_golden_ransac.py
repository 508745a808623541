"""Generates tests/golden/ref_ransac.npz ON A GPU BOX (run under gpurun): model-frame point pairs pushed through the
REFERENCE'S OWN ransacMultiPairGPU (oracle/_ref/libbt_ref.so = /root/reference/src/cuda/cuda_ransac.cu compiled verbatim:
XORWOW sampling, McAdams-SVD 3-point fit :998-1102, inlier rule :1183-1200, racy arg-max :1202-1217) - the inputs and the
inlier ids it returned.  The CPU suite pins oracle/matcher_oracle.ransac_pair against these vectors without a GPU; the GPU
suite compares bt_ransac_pairs with them (and with the inlier sets scripts/make_golden_live.py records).

    gpurun -- 'python scripts/make_golden_ransac.py gpurun_out/golden'   &&  cp gpurun_out/golden/ref_ransac.npz tests/golden/
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import oracle
from oracle import matcher_oracle as mo
from bundletrack_b200 import synth
from bundletrack_b200.matcher import Ransac

out_dir = sys.argv[1] if len(sys.argv) > 1 else "gpurun_out/golden"
os.makedirs(out_dir, exist_ok=True)
dev = torch.device("cuda:0")
cases = [(8, 0.7, 0.005), (60, 0.7, 0.005), (60, 0.4, 0.01), (400, 0.7, 0.005), (400, 0.5, 0.01), (2000, 0.7, 0.005), (2000, 0.5, 0.01)]
A, B, thr = [], [], []
for k, (n, frac, t) in enumerate(cases):
    a, b, _ = synth.make_ransac_case(900 + k, n, inlier_frac=frac)
    A.append(a); B.append(b); thr.append(t)
ref_ids = []
for t in sorted(set(thr)):       # the reference takes one threshold per call
    sel = [k for k in range(len(cases)) if thr[k] == t]
    ids, _ = oracle.ref_ransac_pairs([A[k] for k in sel], [B[k] for k in sel], 2000, t)
    again, _ = oracle.ref_ransac_pairs([A[k] for k in sel], [B[k] for k in sel], 2000, t)
    for k, i, j in zip(sel, ids, again):
        ref_ids.append((k, i))
        print(f"case {k}: n={cases[k][0]} thr={t}: reference inliers {len(i)}; second run identical: {np.array_equal(i, j)}")
ref_ids = [i for _, i in sorted(ref_ids, key=lambda x: x[0])]
r = Ransac(max_pairs=8, max_pts=4096, max_trials=2000)
u3 = None
for k, (n, frac, t) in enumerate(cases):
    got = r.ransac_pairs([torch.from_numpy(A[k]).to(dev)], [torch.from_numpy(B[k]).to(dev)], 2000, t)[0].cpu().numpy()
    u3, best = r.debug(2000, 1)
    want, wbest, counts = mo.ransac_pair(A[k], B[k], u3, t)
    print(f"case {k}: ours {len(got)} (trial {best[0]})  oracle {len(want)} (trial {wbest})  reference {len(ref_ids[k])}  ours==ref {np.array_equal(got, ref_ids[k])}  oracle==ref {np.array_equal(want, ref_ids[k])}")
save = {"n_cases": len(cases), "thresh": np.asarray(thr, np.float32), "n_trials": 2000}
for k in range(len(cases)):
    save[f"A{k}"], save[f"B{k}"], save[f"ref{k}"] = A[k], B[k], ref_ids[k].astype(np.int32)
np.savez_compressed(os.path.join(out_dir, "ref_ransac.npz"), **save)
print("wrote", os.path.join(out_dir, "ref_ransac.npz"))
