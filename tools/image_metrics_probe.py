"""Time the camera image metrics on the GPU: the library's kernels (b200nerf_image_metrics: PSNR and SSIM of an image pair
in three launches) against a torch restatement of the same SSIM definition on the same GPU -- one grouped F.conv2d over
the five stacked moment images, reflect-padded and cropped, as torchmetrics does it -- and, when it is importable,
torchmetrics' structural_similarity_index_measure itself.

    python tools/image_metrics_probe.py [--rounds 5] [--calls 50] [--json out.json]

Images: 1920 x 1080 x 3 and 640 x 360 x 3, seeded, a smooth image and a noisy copy, channels-last as the renderer leaves
them and handed over as [1, C, H, W] views.  Per path, after warm-up: the median and range over `rounds` rounds of `calls`
calls each, the paths alternating within a round, of (i) device time per call from CUDA events around the round and (ii)
wall time of one call up to the Python floats (`.tolist()` / `float()`: the device-to-host copy included).  The card's
name, power limit and SM clock limit are read in the same run.

Bytes: the kernels read both images once in the statistics pass and once plus the 10-pixel halo of every 32 x 32 tile
(42^2 / 32^2 of the image, less at the borders) in the SSIM pass; those algorithmic bytes over the device time are the
achieved bytes/s, reported as a share of the H100 SXM data sheet's 3.35 TB/s of HBM bandwidth.  HBM is the bound named
here; whether the kernels reach it is what the number says.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet
WIN, TILE = 11, 32


def card_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                       capture_output=True, text=True, check=True).stdout.strip().split(", ")
    return {"name": q[0], "power_limit_w": float(q[1]), "sm_clock_limit_mhz": float(q[2]),
            "sms": torch.cuda.get_device_properties(0).multi_processor_count}


def image_pair(h: int, w: int, seed: int):
    """Channels-last [H, W, 3] in [0, 1]: low-pass noise and a copy with 3 % noise."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.rand(1, 3, h // 8 + 2, w // 8 + 2, device="cuda", generator=g)
    x = F.interpolate(x, size=(h, w), mode="bicubic", align_corners=False).clamp(0, 1)[0].permute(1, 2, 0).contiguous()
    y = (x + 0.03 * torch.randn(x.shape, device="cuda", generator=g)).clamp(0, 1)
    return x, y


def algorithmic_bytes(h: int, w: int, c: int) -> int:
    halo = sum(min(TILE + WIN - 1, h - ty * TILE) * min(TILE + WIN - 1, w - tx * TILE)
               for ty in range(-(-(h - WIN + 1) // TILE)) for tx in range(-(-(w - WIN + 1) // TILE)))
    return 2 * 4 * c * (h * w + halo)


def torch_ssim_psnr(preds: torch.Tensor, target: torch.Tensor, kernel: torch.Tensor):
    """The definition of csrc/image_metrics.cuh in torch ops, in torchmetrics' order: reflect pad, one grouped conv over
    the five stacked moment images, crop, mean.  [1, C, H, W] inputs."""
    c = preds.shape[1]
    pad = (WIN - 1) // 2
    data_range = torch.maximum(preds.max() - preds.min(), target.max() - target.min())
    c1, c2 = (0.01 * data_range) ** 2, (0.03 * data_range) ** 2
    p, t = F.pad(preds, (pad,) * 4, mode="reflect"), F.pad(target, (pad,) * 4, mode="reflect")
    out = F.conv2d(torch.cat((p, t, p * p, t * t, p * t)), kernel, groups=c)
    mu_p, mu_t, e_pp, e_tt, e_pt = out.split(1)
    var_p = torch.clamp(e_pp - mu_p * mu_p, min=0.0)
    var_t = torch.clamp(e_tt - mu_t * mu_t, min=0.0)
    cov = e_pt - mu_p * mu_t
    ssim = ((2 * mu_p * mu_t + c1) * (2 * cov + c2)) / ((mu_p * mu_p + mu_t * mu_t + c1) * (var_p + var_t + c2))
    ssim = ssim[..., pad:-pad, pad:-pad].mean()
    psnr = -10.0 * torch.log10(torch.mean((preds - target) ** 2))
    return torch.stack((psnr, ssim))


def measure(paths, rounds: int, calls: int):
    """paths: name -> (enqueue(), to_floats(result)).  Alternates the paths inside every round."""
    for enqueue, to_floats in paths.values():
        for _ in range(5):
            to_floats(enqueue())
    torch.cuda.synchronize()
    dev = {k: [] for k in paths}
    wall = {k: [] for k in paths}
    for _ in range(rounds):
        for name, (enqueue, to_floats) in paths.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(calls):
                enqueue()
            b.record()
            b.synchronize()
            dev[name].append(a.elapsed_time(b) * 1e3 / calls)
            t0 = time.perf_counter()
            for _ in range(calls):
                to_floats(enqueue())
            wall[name].append((time.perf_counter() - t0) * 1e6 / calls)

    def stat(v):
        return {"median_us": statistics.median(v), "min_us": min(v), "max_us": max(v)}

    return {k: {"device": stat(dev[k]), "wall_to_floats": stat(wall[k])} for k in paths}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--calls", type=int, default=50)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("image_metrics_probe needs a CUDA device")
    from oracle import image_metrics_oracle as IM

    from neurad_studio_b200.nerfstudio_api import get_backend

    be = get_backend(torch.device("cuda", 0))
    info = card_info()
    print(f"card: {info['name']}, power limit {info['power_limit_w']:.0f} W, SM clock limit {info['sm_clock_limit_mhz']:.0f} MHz, "
          f"{info['sms']} SMs")
    try:
        from torchmetrics.functional import structural_similarity_index_measure as tm_ssim
    except ImportError:
        tm_ssim = None
    print("torchmetrics:", "importable" if tm_ssim else "not importable (path iii skipped)")
    g1 = torch.from_numpy(IM.window_f32()).cuda()
    results = {"card": info, "torchmetrics": tm_ssim is not None, "rounds": args.rounds, "calls": args.calls, "images": []}
    for (w, h), seed in (((1920, 1080), 1), ((640, 360), 2)):
        x, y = image_pair(h, w, seed)
        preds, target = torch.moveaxis(x, -1, 0)[None], torch.moveaxis(y, -1, 0)[None]
        kernel = torch.outer(g1, g1).expand(3, 1, WIN, WIN).contiguous()
        paths = {
            "kernels": (lambda: be.image_metrics(preds, target), lambda r: r[0].tolist()),
            "torch_conv2d": (lambda: torch_ssim_psnr(preds, target, kernel), lambda r: r.tolist()),
        }
        if tm_ssim:
            paths["torchmetrics"] = (lambda: tm_ssim(preds, target), lambda r: float(r))
        k = be.image_metrics(preds, target)[0].tolist()
        t = torch_ssim_psnr(preds, target, kernel).tolist()
        be.check_status()
        if abs(k[2] - t[1]) > 1e-4 or abs(k[1] - t[0]) > 1e-3:
            raise SystemExit(f"kernels and the torch restatement disagree: ssim {k[2]} vs {t[1]}, psnr {k[1]} vs {t[0]}")
        m = measure(paths, args.rounds, args.calls)
        nbytes = algorithmic_bytes(h, w, 3)
        rate = nbytes / (m["kernels"]["device"]["median_us"] * 1e-6)
        row = {"image": f"{w}x{h}x3", "algorithmic_bytes": nbytes, "kernels_bytes_per_s": rate,
               "share_of_hbm_data_sheet": rate / HBM_BYTES_PER_S, "hbm_bound_us": nbytes / HBM_BYTES_PER_S * 1e6,
               "kernels_psnr_ssim": k[1:3], "torch_psnr_ssim": t, "paths": m}
        results["images"].append(row)
        print(f"{w}x{h}x3: psnr {k[1]:.4f} dB, ssim {k[2]:.6f} (torch restatement {t[0]:.4f}, {t[1]:.6f})")
        for name, r in m.items():
            d, wl = r["device"], r["wall_to_floats"]
            print(f"  {name:13s} device {d['median_us']:9.1f} us/call [{d['min_us']:.1f}-{d['max_us']:.1f}]   "
                  f"wall to floats {wl['median_us']:9.1f} us/call [{wl['min_us']:.1f}-{wl['max_us']:.1f}]")
        print(f"  kernels: {nbytes / 1e6:.1f} MB algorithmic -> {rate / 1e12:.3f} TB/s achieved, "
              f"{100 * rate / HBM_BYTES_PER_S:.1f} % of the data sheet's 3.35 TB/s (HBM bound {nbytes / HBM_BYTES_PER_S * 1e6:.1f} us)")
    print(json.dumps(results))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
