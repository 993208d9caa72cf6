"""Time the lidar terms of NeuRAD's training objective (models/neurad.py:486-520), forward + backward: the library's
kernel pair (neurad_studio_b200.losses.lidar_losses) against the reference's torch lines (tests/objective_cases.py), at
a training batch (16 384 lidar rays) and a full sweep (262 144).  The two alternate in one process; each iteration is
timed by CUDA events (device time) and by the host clock up to a torch.cuda.synchronize() (wall time, which includes the
host waits of the reference's boolean-mask indexing).  Prints one JSON line with the card's name and power limit.

    python tools/objective_probe.py [--iters 200] [--warmup 20]
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from neurad_studio_b200 import losses as L  # noqa: E402
from tests import objective_cases as C  # noqa: E402


def card() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name()


def kernel_step(d):
    leaves = [d["pred"].clone().requires_grad_(True), d["intensity"].clone().requires_grad_(True),
              d["logits"].clone().requires_grad_(True)]
    props = [p.clone().requires_grad_(True) for p in d["props"]]
    r = L.lidar_losses(leaves[0], props, d["distance"], d["did_return"], leaves[1], d["lidar"][..., 3:4], leaves[2])
    sum(r[k] for k in C.SCALAR_KEYS).backward()


def torch_step(d):
    leaves = [d["pred"].clone().requires_grad_(True), d["intensity"].clone().requires_grad_(True),
              d["logits"].clone().requires_grad_(True)]
    props = [p.clone().requires_grad_(True) for p in d["props"]]
    m, _, _ = C.reference_lidar_terms(leaves[0], props, d["distance"], d["did_return"], d["lidar"][..., 3:4], leaves[1],
                                      leaves[2])
    sum(m[k] for k in C.SCALAR_KEYS).backward()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    res = {"what": "lidar terms of get_metrics_dict, forward + backward, median per call", "gpu": card(), "sizes": {}}
    for n in (16384, 262144):
        d = C.lidar_inputs(n=n, seed=1, device=dev)
        fns = {"kernels": kernel_step, "torch": torch_step}
        for f in fns.values():
            for _ in range(a.warmup):
                f(d)
        torch.cuda.synchronize()
        dev_ms = {k: [] for k in fns}
        wall_ms = {k: [] for k in fns}
        for _ in range(a.iters):
            for k, f in fns.items():  # alternating, so both see the same machine state
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                t0 = time.perf_counter()
                e0.record()
                f(d)
                e1.record()
                torch.cuda.synchronize()
                wall_ms[k].append((time.perf_counter() - t0) * 1e3)
                dev_ms[k].append(e0.elapsed_time(e1))
        med = lambda v: sorted(v)[len(v) // 2]  # noqa: E731
        res["sizes"][n] = {k: {"device_ms": round(med(dev_ms[k]), 4), "wall_ms": round(med(wall_ms[k]), 4)} for k in fns}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
