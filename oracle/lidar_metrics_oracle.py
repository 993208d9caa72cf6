"""TEST INFRASTRUCTURE ONLY -- float64 restatement of NeuRAD's lidar chamfer distance (utils/math.py:745-798) and the
seeded inputs of tests/golden/lidar_metrics.npz.

`min_sq_f64` is the brute-force nearest-neighbour squared distance in float64 from direct differences, so it carries no
cancellation error; the GPU tests bound the kernel's fp32 minima against it.  Pure torch: it runs on the CPU here and
on the GPU machine (it never imports the reference).
"""
from __future__ import annotations

from typing import Dict, Tuple

import torch


def min_sq_f64(src: torch.Tensor, dst: torch.Tensor, chunk: int = 512) -> torch.Tensor:
    """min_j |src_i - dst_j|^2 in float64 for every row i (xyz = the first three columns), NaN-propagating like torch.min."""
    s = src[:, :3].double()
    d = dst[:, :3].double()
    out = []
    for i in range(0, s.shape[0], chunk):
        diff = s[i:i + chunk, None, :] - d[None, :, :]
        out.append((diff * diff).sum(-1).min(dim=1).values)
    return torch.cat(out)


def chamfer_sums_f64(src: torch.Tensor, dst: torch.Tensor) -> Tuple[float, float]:
    """(sum_i min_j |s_i - t_j|^2, sum_j min_i |t_j - s_i|^2) in float64."""
    return float(min_sq_f64(src, dst).sum()), float(min_sq_f64(dst, src).sum())


def chamfer_f64(src: torch.Tensor, dst: torch.Tensor, normalize_with_target: bool = True) -> float:
    """NeuRAD's metric chamfer_distance(pred, gt, 1_000, True) in float64: both sums divided by the target count."""
    a, b = chamfer_sums_f64(src, dst)
    m = dst.shape[0] if normalize_with_target else 1
    return a / m + b / m


# ---- seeded inputs -------------------------------------------------------------------------------------------
def _sweep(n: int, g: torch.Generator, r_min: float, r_max: float) -> torch.Tensor:
    """n lidar-frame points [n,4] = (x, y, z, intensity): ranges in [r_min, r_max], a 40-degree elevation band."""
    az = torch.rand(n, generator=g, dtype=torch.float64) * 2 * torch.pi
    el = (torch.rand(n, generator=g, dtype=torch.float64) - 0.7) * (40.0 * torch.pi / 180.0)
    r = r_min + (r_max - r_min) * torch.rand(n, generator=g, dtype=torch.float64)
    xyz = torch.stack([r * el.cos() * az.cos(), r * el.cos() * az.sin(), r * el.sin()], -1)
    inten = torch.rand(n, 1, generator=g, dtype=torch.float64)
    return torch.cat([xyz, inten], -1).float()


def chamfer_cases() -> Dict[str, Tuple[torch.Tensor, torch.Tensor]]:
    """(pred [N,3], gt [M,3]) pairs: sizes that are not tile multiples, a 100 m-scale cloud, N != M."""
    g = torch.Generator().manual_seed(2024)
    cases = {}
    gt = _sweep(3001, g, 2.0, 40.0)[:, :3]
    cases["ragged"] = (gt[:2999] + 0.05 * torch.randn(2999, 3, generator=g), gt)
    gt = _sweep(2500, g, 80.0, 120.0)[:, :3]
    cases["far100m"] = (gt + 0.02 * torch.randn(2500, 3, generator=g), gt)
    gt = _sweep(4100, g, 1.0, 60.0)[:, :3]
    cases["n_ne_m"] = (_sweep(1500, g, 1.0, 60.0)[:, :3], gt)
    return cases


def metrics_cases() -> Dict[str, Tuple[Dict[str, torch.Tensor], Dict[str, torch.Tensor], float]]:
    """(outputs, batch, ray_drop_loss_mult) of get_image_metrics_and_images on one lidar sweep of 2 000 rays:
    - "ray_drop": ray_drop_loss_mult = 0.01 (predicted returns: sigmoid(logit) < 0.5), is_lidar / did_return absent;
    - "depth": ray_drop_loss_mult = 0 (predicted returns: depth < non_return_lidar_distance), both masks given;
    - "fallback": no predicted return, so the chamfer value is the mean range of the measured returns."""
    g = torch.Generator().manual_seed(7)
    n = 2000
    lidar = _sweep(n, g, 2.0, 90.0)
    dist = lidar[:, :3].norm(dim=-1, keepdim=True)
    did_return = torch.rand(n, 1, generator=g) < 0.85
    dirs = lidar[:, :3] / dist
    depth = (dist + 0.3 * torch.randn(n, 1, generator=g)).abs()
    depth = torch.where(did_return, depth, 160.0 + 20.0 * torch.rand(n, 1, generator=g))
    logits = torch.where(did_return, -2.0, 2.0) + 1.5 * torch.randn(n, 1, generator=g)
    outputs = {"depth": depth, "ray_drop_logits": logits, "intensity": torch.rand(n, 1, generator=g),
               "points": dirs * depth}
    cases = {}
    cases["ray_drop"] = (outputs, {"lidar": lidar, "distance": dist}, 0.01)
    cases["depth"] = (outputs, {"lidar": lidar, "distance": dist, "did_return": did_return,
                                "is_lidar": torch.ones(n, 1, dtype=torch.bool)}, 0.0)
    out_fb = dict(outputs, ray_drop_logits=logits.abs() + 0.5)
    cases["fallback"] = (out_fb, {"lidar": lidar, "distance": dist, "did_return": did_return}, 0.01)
    return cases


METRIC_KEYS = ("depth_median_l2", "depth_mean_rel_l2", "intensity_rmse", "ray_drop_accuracy", "chamfer_distance")
