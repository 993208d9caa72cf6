"""NeuRAD's evaluation metrics (models/neurad.py:265-271, 568-621) and the training PSNR of get_metrics_dict.

`chamfer_distance` is the reference's `nerfstudio.utils.math.chamfer_distance` on the library's all-pairs kernel
(csrc/lidar_eval.cuh): exact fp32 per-pair squared distances from direct differences and fp64 sums, without the dense
distance matrices of the reference's chunked `torch.cdist`.  The other four metrics are torch one-liners, as in the
reference.

`ssim` is the reference's `self.ssim`, torchmetrics' `structural_similarity_index_measure`, on the library's tile kernel
(csrc/image_metrics.cuh), where the definition is written out.
"""
from __future__ import annotations

import math
from typing import Optional

import torch
from torch import Tensor


def chamfer_distance(source_pc: Tensor, target_pc: Tensor, chunk_size: Optional[int] = None,
                     normalize_with_target: bool = False) -> Tensor:
    """utils/math.py:745-798 with the same signature and value: sum_i min_j |s_i - t_j|^2 + sum_j min_i |t_j - s_i|^2 as
    a 0-d tensor of the source's dtype.

    Nothing is materialised, so `chunk_size` does not change the memory use.  It keeps its one effect on the value: the
    reference divides the sums by the target count M only on its chunked path, so `normalize_with_target` applies when
    `chunk_size` is not None, and with chunk_size=None both sums stay unnormalised, as in the reference.  NeuRAD's
    metric is `chamfer_distance(pred, gt, 1_000, True)`: both sums divided by the ground-truth count.

    The clouds are [N,3] / [M,3] (or wider rows: x, y, z are the first three columns) on a CUDA device.  Empty clouds
    raise B200NerfError; the reference's own callers never pass one (neurad.py:614 takes a fallback branch instead)."""
    from .nerfstudio_api import get_backend

    normalize = bool(normalize_with_target) and chunk_size is not None
    be = get_backend(source_pc.device)
    with torch.no_grad():
        return be.chamfer_distance(source_pc.reshape(-1, source_pc.shape[-1]), target_pc.reshape(-1, target_pc.shape[-1]),
                                   normalize).to(source_pc.dtype)


def median_l2(pred: Tensor, gt: Tensor) -> Tensor:
    return torch.median((pred - gt) ** 2)


def mean_rel_l2(pred: Tensor, gt: Tensor) -> Tensor:
    return torch.mean(((pred - gt) / gt) ** 2)


def rmse(pred: Tensor, gt: Tensor) -> Tensor:
    return torch.sqrt(torch.mean((pred - gt) ** 2))


def psnr(preds: Tensor, target: Tensor) -> Tensor:
    """torchmetrics' PeakSignalNoiseRatio(data_range=1.0) on one batch (neurad.py:265, 465): 10 log10(1 / mse)."""
    return -torch.log(torch.sum((preds - target) ** 2) / target.numel()) * (10 / math.log(10.0))


def ssim(preds: Tensor, target: Tensor, data_range: Optional[float] = None) -> Tensor:
    """torchmetrics' structural_similarity_index_measure(preds, target) with its defaults, the reference's `self.ssim`
    (neurad.py:266, 586), as a 0-d tensor of the input dtype on the input's CUDA device.

    The definition is written from memory, unpinned against torchmetrics (the package is not a dependency, and the one
    test that compares with it, in tests/test_zz_image_metrics_gpu.py, runs only where it is installed): an 11 x 11
    Gaussian window of sigma 1.5, normalised in fp32 and applied per channel to preds, target, their squares and their
    product; c1 = (0.01 R)^2 and c2 = (0.03 R)^2 with R = `data_range`, or max(preds.max() - preds.min(), target.max() -
    target.min()) when it is None; variances clamped at 0; and the mean of
    (2 mu_p mu_t + c1)(2 cov + c2) / ((mu_p^2 + mu_t^2 + c1)(var_p + var_t + c2)) over the (H - 10) x (W - 10) windows that
    lie inside the image (what torchmetrics keeps after its reflect padding and crop), all channels, then over the batch.

    preds / target are [B, C, H, W] with H, W >= 11; non-contiguous views are read in place.  Other window sizes,
    non-Gaussian windows and multi-scale SSIM are not provided."""
    from .nerfstudio_api import get_backend

    with torch.no_grad():
        return get_backend(preds.device).image_metrics(preds, target, data_range)[0, 2].to(preds.dtype)
