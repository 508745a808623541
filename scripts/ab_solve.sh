#!/bin/bash
# A/B of library builds on the flagship workload: usage  ab_solve.sh OUTDIR RUNS NAME=lib.so [NAME=lib.so ...]
# Runs `bench.py --gpus 1 --steps 200 --warmup 10 --skip-cfg3` RUNS times per build, alternating the builds, each with its own
# --dump-outputs directory; prints the card, its power limit, min/median/max per build of the headline and its companions, and
# whether every build's poses are byte-identical to the first build's.
set -e
out=$1; runs=$2; shift 2
mkdir -p "$out"
cd "$(dirname "$0")/.."
nvidia-smi --query-gpu=name,power.limit,clocks.max.sm --format=csv,noheader | tee "$out/card.txt"
for r in $(seq 1 "$runs"); do
	for spec in "$@"; do
		name=${spec%%=*}; lib=${spec#*=}
		BT_B200_LIB=$lib python bench.py --gpus 1 --steps 200 --warmup 10 --skip-cfg3 --dump-outputs "$out/$name.$r" | tail -1 > "$out/$name.$r.json"
		echo "$name run $r done"
	done
done
python - "$out" "$runs" "$@" <<'EOF'
import json, sys, os
import numpy as np
out, runs, specs = sys.argv[1], int(sys.argv[2]), sys.argv[3:]
names = [s.split("=", 1)[0] for s in specs]
keys = [("value", lambda j: j["value"]), ("kernel_ms.solve", lambda j: j["roofline"]["kernel_ms"]["solve"]), ("e2e.value", lambda j: j["e2e"]["value"]),
        ("rebuild_every_call.value", lambda j: j["keyframe_cache"]["rebuild_every_call"]["value"]), ("single_window.e2e_ms", lambda j: j["single_window"]["e2e_ms"])]
print("card:", open(os.path.join(out, "card.txt")).read().strip())
for n in names:
    js = [json.load(open(os.path.join(out, f"{n}.{r}.json"))) for r in range(1, runs + 1)]
    for k, f in keys:
        v = np.array([f(j) for j in js], dtype=float)
        print(f"{n:10s} {k:26s} min {v.min():10.4f}  median {np.median(v):10.4f}  max {v.max():10.4f}")
for n in names[1:]:
    for fn in ("poses_value.npy", "poses_e2e.npy"):
        same = all(open(os.path.join(out, f"{names[0]}.{r}", fn), "rb").read() == open(os.path.join(out, f"{n}.{r}", fn), "rb").read() for r in range(1, runs + 1))
        print(f"{n} vs {names[0]} {fn}: {'byte-identical' if same else 'DIFFERENT'}")
EOF
