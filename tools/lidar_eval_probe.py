"""Time the lidar chamfer distance on the GPU: the library's all-pairs kernel (b200nerf_chamfer_distance) against the
reference's algorithm -- chunked torch.cdist, utils/math.py:745-798 with chunk_size=1000 and normalize_with_target --
restated here in plain torch on the same GPU as the labelled comparator.

    python tools/lidar_eval_probe.py [--reps 20] [--ref-reps 3] [--json out.json]

Sweeps: 64 x 1800 and 128 x 2048 points, seeded; the prediction drops ~8 % of the returns and moves the rest by a few cm.
Reports the card's name, power limit and SM clock limit from the same call, ms per sweep (median of CUDA-event timed
calls after warm-up), pairs/s (2 N M pairs per sweep), and the fraction of the FP32-issue bound: 7 FP32 instructions per
pair (3 FADD, FMUL, 2 FFMA, FMNMX) over SMs x 128 lanes x the SM clock limit.  Checks that the two paths agree within the
reference's cancellation error.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

INSTR_PER_PAIR = 7
U = 2.0 ** -24


def card_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                       capture_output=True, text=True, check=True).stdout.strip().split(", ")
    return {"name": q[0], "power_limit_w": float(q[1]), "sm_clock_limit_mhz": float(q[2]),
            "sms": torch.cuda.get_device_properties(0).multi_processor_count}


def sweep(beams: int, n_az: int, seed: int):
    g = torch.Generator(device="cuda").manual_seed(seed)
    n = beams * n_az
    el = torch.linspace(-25.0, 3.0, beams, device="cuda").deg2rad().repeat_interleave(n_az)
    az = torch.arange(n_az, device="cuda").repeat(beams) * (2 * torch.pi / n_az)
    r = 2.0 + 78.0 * torch.rand(n, device="cuda", generator=g)
    gt = torch.stack([r * el.cos() * az.cos(), r * el.cos() * az.sin(), r * el.sin() + 1.8], -1)
    keep = torch.rand(n, device="cuda", generator=g) > 0.08
    pred = gt[keep] + 0.03 * torch.randn(int(keep.sum()), 3, device="cuda", generator=g)
    return pred.contiguous(), gt.contiguous()


def reference_chamfer(source_pc, target_pc, chunk_size=1_000):
    """The reference's chunked algorithm (normalize_with_target=True) in plain torch."""
    s2t = torch.tensor(0.0, device=source_pc.device)
    t2s = torch.tensor(0.0, device=source_pc.device)
    source_pc, target_pc = source_pc.view(1, -1, 3), target_pc.view(1, -1, 3)
    m = target_pc.shape[1]

    def first_sum(a, b):
        d = torch.cdist(a, b, p=2, compute_mode="use_mm_for_euclid_dist_if_necessary").pow(2).view(a.shape[1], b.shape[1])
        return torch.min(d, dim=1)[0].sum()

    for i in range(0, source_pc.shape[1], chunk_size):
        s2t += first_sum(source_pc[:, i:i + chunk_size], target_pc) / m
    for i in range(0, m, chunk_size):
        t2s += first_sum(target_pc[:, i:i + chunk_size], source_pc) / m
    return s2t + t2s


def time_ms(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return statistics.median(ts), min(ts), max(ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--ref-reps", type=int, default=3)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("lidar_eval_probe needs a CUDA device")
    from neurad_studio_b200.nerfstudio_api import get_backend

    be = get_backend(torch.device("cuda", 0))
    info = card_info()
    print(f"card: {info['name']}, power limit {info['power_limit_w']:.0f} W, SM clock limit {info['sm_clock_limit_mhz']:.0f} MHz, "
          f"{info['sms']} SMs")
    lanes_per_s = info["sms"] * 128 * info["sm_clock_limit_mhz"] * 1e6
    results = {"card": info, "sweeps": []}
    for beams, n_az, seed in ((64, 1800, 1), (128, 2048, 2)):
        pred, gt = sweep(beams, n_az, seed)
        n, m = pred.shape[0], gt.shape[0]
        pairs = 2 * n * m
        k_val = float(be.chamfer_distance(pred, gt, True))
        k_ms = time_ms(lambda: be.chamfer_distance(pred, gt, True), args.reps, 3)
        be.check_status()
        r_val = float(reference_chamfer(pred, gt))
        r_ms = time_ms(lambda: reference_chamfer(pred, gt), args.ref_reps, 1)
        # the mm form's error: a few u of |a|^2 + |b|^2 per pair, summed over both directions and divided by M
        norm2 = float((pred.double() ** 2).sum() + (gt.double() ** 2).sum())
        tol = 32 * U * 2 * norm2 / m
        agree = abs(k_val - r_val) <= tol
        bound_ms = pairs * INSTR_PER_PAIR / lanes_per_s * 1e3
        row = {"sweep": f"{beams}x{n_az}", "n_pred": n, "n_gt": m, "kernel_ms": k_ms[0], "kernel_ms_min_max": k_ms[1:],
               "reference_cdist_ms": r_ms[0], "reference_cdist_ms_min_max": r_ms[1:], "speedup": r_ms[0] / k_ms[0],
               "kernel_pairs_per_s": pairs / (k_ms[0] * 1e-3), "fp32_issue_bound_ms": bound_ms,
               "fraction_of_fp32_issue_bound": bound_ms / k_ms[0], "kernel_value": k_val, "reference_value": r_val,
               "abs_diff": abs(k_val - r_val), "cancellation_tol": tol, "agree": agree}
        results["sweeps"].append(row)
        print(f"{beams}x{n_az} sweep (N={n}, M={m}): kernel {k_ms[0]:.3f} ms [{k_ms[1]:.3f}-{k_ms[2]:.3f}], "
              f"reference chunked cdist {r_ms[0]:.1f} ms [{r_ms[1]:.1f}-{r_ms[2]:.1f}] ({r_ms[0] / k_ms[0]:.0f}x); "
              f"{pairs / (k_ms[0] * 1e-3) / 1e12:.2f} Tpairs/s, {100 * bound_ms / k_ms[0]:.1f} % of the FP32-issue bound "
              f"({bound_ms:.3f} ms); values {k_val:.7g} vs {r_val:.7g} (|diff| {abs(k_val - r_val):.2e} <= tol {tol:.2e}: {agree})")
        if not agree:
            raise SystemExit("kernel and reference disagree beyond the reference's cancellation error")
        del pred, gt
        torch.cuda.empty_cache()
    print(json.dumps(results))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
