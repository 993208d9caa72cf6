"""NeuRAD's lidar evaluation metrics (models/neurad.py:268-271, 589-621) and the training PSNR of get_metrics_dict.

`chamfer_distance` is the reference's `nerfstudio.utils.math.chamfer_distance` on the library's all-pairs kernel
(csrc/lidar_eval.cuh): exact fp32 per-pair squared distances from direct differences and fp64 sums, without the dense
distance matrices of the reference's chunked `torch.cdist`.  The other four metrics are torch one-liners, as in the
reference.
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
