"""TEST INFRASTRUCTURE ONLY -- float64 restatement of the camera metrics of NeuRADModel.get_image_metrics_and_images
(models/neurad.py:265-266, 585-586): PeakSignalNoiseRatio(data_range=1.0) and structural_similarity_index_measure with
its defaults, and the seeded inputs of tests/golden/image_metrics.npz.

The SSIM definition below is written FROM MEMORY, UNPINNED AGAINST TORCHMETRICS: the package is not part of the reference
tree and is not installed where this fixture is made.  The only place it meets the real thing is the importorskip test
of tests/test_zz_image_metrics_gpu.py.

  window  g[i] = exp(-((i - 5) / 1.5)^2 / 2), i = 0..10, normalised to sum 1 in fp32 (the oracle promotes these fp32
          taps to float64, so it filters with the same window as the kernel); the 2-D window is the outer product,
          applied per channel to a, b, a a, b b, a b
  range   R = max(max a - min a, max b - min b) in fp32 over the whole batch when none is given; c1 = (0.01 R)^2,
          c2 = (0.03 R)^2
  value   var = max(E[x x] - mu^2, 0), cov = E[a b] - mu_a mu_b,
          ssim = (2 mu_a mu_b + c1)(2 cov + c2) / ((mu_a^2 + mu_b^2 + c1)(var_a + var_b + c2))
  mean    reflect-pad by 5, filter, crop 5 from every border, mean over the image and its channels, then over the batch

It is written twice.  `ssim_padded_f64` follows that order literally (np.pad, a full 2-D correlation per channel, the
crop).  `ssim_valid_f64` filters only the (H - 10) x (W - 10) windows that lie inside the unpadded image, separably.  The
two agree to 1e-12 on every case (checked when the fixture is made and by tests/test_image_metrics_cpu.py), which is the
proof that the padding is never read.  numpy / scipy / torch on the CPU; it never imports the reference.
"""
from __future__ import annotations

from typing import Dict, Optional, Tuple

import numpy as np
import torch

WIN, SIGMA, K1, K2 = 11, 1.5, 0.01, 0.03
PAD = (WIN - 1) // 2


def window_f32() -> np.ndarray:
    """The 1-D taps as torch computes them in fp32 (numpy's fp32 exp differs in the last bit of some taps)."""
    dist = torch.arange((1 - WIN) / 2, (1 + WIN) / 2, 1, dtype=torch.float32)
    gauss = torch.exp(-torch.pow(dist / SIGMA, 2) / 2)
    return (gauss / gauss.sum()).numpy()


def data_range_f32(a: np.ndarray, b: np.ndarray) -> np.float32:
    """max(a.max() - a.min(), b.max() - b.min()) in fp32; np.max / np.min keep a NaN, as torch's do."""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return np.maximum(a.max() - a.min(), b.max() - b.min())


def _constants(a, b, data_range) -> Tuple[float, float, float]:
    r = float(data_range_f32(a, b)) if data_range is None or data_range <= 0 else float(np.float32(data_range))
    return r, (K1 * r) ** 2, (K2 * r) ** 2


def _ssim_map(mu_a, mu_b, e_aa, e_bb, e_ab, c1, c2):
    var_a = np.maximum(e_aa - mu_a * mu_a, 0.0)  # np.maximum keeps a NaN, as torch.clamp does
    var_b = np.maximum(e_bb - mu_b * mu_b, 0.0)
    cov = e_ab - mu_a * mu_b
    with np.errstate(invalid="ignore", divide="ignore"):
        return ((2 * mu_a * mu_b + c1) * (2 * cov + c2)) / ((mu_a * mu_a + mu_b * mu_b + c1) * (var_a + var_b + c2))


def ssim_padded_f64(a: np.ndarray, b: np.ndarray, data_range: Optional[float] = None) -> np.ndarray:
    """Per-image SSIM [B] of channels-last a, b [B, H, W, C], in torchmetrics' literal order."""
    from scipy.signal import correlate2d

    _, c1, c2 = _constants(a, b, data_range)
    g = window_f32().astype(np.float64)
    k2d = np.outer(g, g)
    x, y = np.asarray(a, np.float64), np.asarray(b, np.float64)
    out = np.empty(x.shape[0])
    for i in range(x.shape[0]):
        maps = []
        for ch in range(x.shape[3]):
            pa = np.pad(x[i, :, :, ch], PAD, mode="reflect")
            pb = np.pad(y[i, :, :, ch], PAD, mode="reflect")
            f = [correlate2d(m, k2d, mode="valid") for m in (pa, pb, pa * pa, pb * pb, pa * pb)]  # H x W again
            maps.append(_ssim_map(*f, c1, c2)[PAD:-PAD, PAD:-PAD])
        out[i] = np.mean(np.stack(maps))
    return out


def _filter_valid(x: np.ndarray, g: np.ndarray, axis: int) -> np.ndarray:
    n = x.shape[axis] - (WIN - 1)
    acc = np.zeros_like(np.take(x, range(n), axis=axis))
    for i in range(WIN):
        acc = acc + g[i] * np.take(x, range(i, i + n), axis=axis)
    return acc


def ssim_valid_f64(a: np.ndarray, b: np.ndarray, data_range: Optional[float] = None) -> np.ndarray:
    """Per-image SSIM [B]: only the windows inside the image, one separable pass along the columns and one along the rows."""
    _, c1, c2 = _constants(a, b, data_range)
    g = window_f32().astype(np.float64)
    x, y = np.asarray(a, np.float64), np.asarray(b, np.float64)
    f = [_filter_valid(_filter_valid(m, g, 2), g, 1) for m in (x, y, x * x, y * y, x * y)]
    return _ssim_map(*f, c1, c2).mean(axis=(1, 2, 3))


def metrics_f64(a: np.ndarray, b: np.ndarray, data_range: Optional[float] = None, padded: bool = False) -> np.ndarray:
    """[(B + 1), 4] = {mse, psnr, ssim, data_range} of the batch, then of each image: the layout of b200nerf_image_metrics."""
    x, y = np.asarray(a, np.float64), np.asarray(b, np.float64)
    mse = ((x - y) ** 2).mean(axis=(1, 2, 3))
    ssim = (ssim_padded_f64 if padded else ssim_valid_f64)(a, b, data_range)
    mse = np.concatenate([[mse.mean()], mse])
    ssim = np.concatenate([[ssim.mean()], ssim])
    with np.errstate(divide="ignore"):
        psnr = 10.0 * np.log10(1.0 / mse)
    r = _constants(a, b, data_range)[0]
    return np.stack([mse, psnr, ssim, np.full_like(mse, r)], axis=1)


# ---- seeded inputs -------------------------------------------------------------------------------------------
def _render_like(rng: np.random.Generator, b: int, h: int, w: int, c: int, noise: float = 0.03, lo: float = 0.0,
                 hi: float = 1.0) -> Tuple[np.ndarray, np.ndarray]:
    """A smooth image (low-pass noise stretched to [lo, hi]) and a perturbed copy, as a render next to its ground truth."""
    from scipy.ndimage import gaussian_filter

    x = gaussian_filter(rng.standard_normal((b, h, w, c)), sigma=(0, 4, 4, 0))
    x = (x - x.min()) / (x.max() - x.min()) * (hi - lo) + lo
    y = x + noise * (hi - lo) * rng.standard_normal(x.shape)
    if lo == 0.0 and hi == 1.0:
        y = np.clip(y, 0.0, 1.0)
    return x.astype(np.float32), y.astype(np.float32)


def cases() -> Dict[str, Tuple[np.ndarray, np.ndarray, float]]:
    """name -> (a, b [B, H, W, C] fp32 channels-last, data_range; 0 = derive it from the images)."""
    rng = np.random.default_rng(20240613)
    out = {}
    out["smooth"] = _render_like(rng, 1, 72, 100, 3) + (0.0,)
    a, b = _render_like(rng, 1, 50, 70, 3)
    out["identical"] = (a, a.copy(), 0.0)
    out["explicit_range"] = _render_like(rng, 1, 40, 36, 3) + (2.0,)
    out["constant"] = (np.full((1, 20, 24, 3), 0.5, np.float32), np.full((1, 20, 24, 3), 0.25, np.float32), 1.0)
    a, b = _render_like(rng, 1, 40, 44, 3, lo=-1.0, hi=1.0)
    out["negative"] = (a, -a, 0.0)
    out["one_window"] = _render_like(rng, 1, 11, 11, 3) + (0.0,)
    out["wide"] = _render_like(rng, 1, 11, 300, 1) + (0.0,)
    out["tall"] = _render_like(rng, 1, 300, 11, 3) + (0.0,)
    out["odd_37x53"] = _render_like(rng, 1, 37, 53, 3) + (0.0,)
    out["odd_65x97_c1"] = _render_like(rng, 1, 65, 97, 1) + (0.0,)
    out["batch2"] = _render_like(rng, 2, 45, 50, 3) + (0.0,)
    out["outside_unit"] = _render_like(rng, 1, 48, 40, 3, lo=-2.0, hi=3.0) + (0.0,)
    a, b = _render_like(rng, 1, 37, 53, 3)
    b[0, 20, 31, 1] = np.nan
    out["nan"] = (a, b, 0.0)
    return out
