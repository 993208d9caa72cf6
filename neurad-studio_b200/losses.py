"""The per-ray regularisers NeuRAD trains with, and the lidar terms of its objective.

The regularisers keep the same names and call signatures as nerfstudio/model_components/losses.py
(`distortion_loss`, `zipnerf_interlevel_loss`, `ray_samples_to_sdist`; selected at models/neurad.py:262,524,541-545),
evaluated by the library's loss kernels (one thread per ray: blur, piecewise-quadratic cdf, resampling, and the analytic
gradient in the same pass) instead of ~40 small torch kernels with sorts and gathers per proposal level.

`lidar_losses` is the lidar half of `NeuRADModel.get_metrics_dict` in training mode (models/neurad.py:486-520) on one
forward and one backward kernel sequence: the per-ray depth losses with the non-return targets, the exact
torch.quantile of the depth loss and its mask, and the reductions, with no boolean-mask indexing and so no host
synchronisation.

`weights_list` / `ray_samples_list` are the lists `NeuRADModel.get_nff_outputs` returns in the module walk: proposal
levels first, the final level (without the sky sample) last; weights [N,S,1].
"""
from __future__ import annotations

from typing import Dict, List, Sequence

import torch
from torch import Tensor

from . import autograd as AG
from . import nerfstudio_api as api

PULSE_WIDTHS = (0.03, 0.003)  # losses.py:651


def ray_samples_to_sdist(ray_samples) -> Tensor:
    """losses.py:119-125: the spacing-domain bin edges [N,S+1] of a level."""
    return ray_samples.per_ray_spacing_bins()


def _w(weights: Tensor) -> Tensor:
    return (weights[..., 0] if weights.dim() == 3 else weights).contiguous()


def distortion_loss(weights_list: List[Tensor], ray_samples_list) -> Tensor:
    """losses.py:172-177 (mip-NeRF 360): mean over rays of lossfun_distortion on the final level; differentiable with
    respect to its weights."""
    c = ray_samples_to_sdist(ray_samples_list[-1]).detach()
    w = _w(weights_list[-1])
    be = api.get_backend(w.device)
    if torch.is_grad_enabled() and w.requires_grad:
        return AG.DistortionLossFn.apply(be, c, w).mean()
    with torch.no_grad():
        return be.distortion_loss(c, w)[0].mean()


def zipnerf_interlevel_loss(weights_list: List[Tensor], ray_samples_list) -> Tensor:
    """losses.py:645-705 (Zip-NeRF's anti-aliased interlevel loss): the final level is the detached target, every
    proposal level receives a gradient through its weights."""
    c = ray_samples_to_sdist(ray_samples_list[-1]).detach()
    w = _w(weights_list[-1]).detach()
    be = api.get_backend(w.device)
    loss = 0
    for i, (ray_samples, weights) in enumerate(zip(ray_samples_list[:-1], weights_list[:-1])):
        cp = ray_samples_to_sdist(ray_samples).detach()
        wp = _w(weights)
        if torch.is_grad_enabled() and wp.requires_grad:
            per_ray = AG.InterlevelLossFn.apply(be, c, w, cp, wp, PULSE_WIDTHS[i])
        else:
            with torch.no_grad():
                per_ray = be.zipnerf_interlevel_loss(c, w, cp, wp, PULSE_WIDTHS[i])[0]
        loss = loss + per_ray.mean()
    return loss


def lidar_losses(pred_depth: Tensor, prop_depths: Sequence[Tensor], distance: Tensor, did_return: Tensor, intensity: Tensor,
                 gt_intensity: Tensor, ray_drop_logits: Tensor, non_return_lidar_distance: float = 150.0,
                 non_return_loss_mult: float = 0.1, quantile_threshold: float = 0.95) -> Dict[str, Tensor]:
    """neurad.py:486-520 over the n lidar rays of a batch.  Every input is in lidar rows, [n] or [n,1]: the predicted
    depth (outputs["depth"][is_lidar]), the proposal depths of every round, the measured distance, did_return (bool), the
    predicted intensity, the measured intensity (batch["lidar"][:, 3:4]; a strided column needs no copy) and the ray-drop
    logits.

    Returns 0-d tensors "depth_loss" (mean of the depth loss below its quantile), "intensity_loss" (MSE over that mask
    and did_return), "ray_drop_loss" (BCE with logits, mean over all rays), "depth_loss_<i>" per proposal round (plain
    mean), and "quantile" / "quantile_mask" [n] -- the reference's `torch.quantile(loss, quantile_threshold)` bit for bit
    and `loss < quantile`.  Differentiable with respect to the depths, the intensity and the logits.  n = 0 raises, as
    torch.quantile does."""
    be = api.get_backend(distance.device)
    settings = (float(non_return_lidar_distance), float(non_return_loss_mult), float(quantile_threshold))
    grad_in = (pred_depth, intensity, ray_drop_logits, *prop_depths)
    if torch.is_grad_enabled() and any(t.requires_grad for t in grad_in):
        out, mask = AG.LidarLossesFn.apply(be, settings, distance.detach(), did_return, gt_intensity.detach(), pred_depth,
                                           intensity, ray_drop_logits, *prop_depths)
    else:
        with torch.no_grad():
            out, _, mask = be.lidar_losses(pred_depth, list(prop_depths), distance, did_return, intensity, gt_intensity,
                                           ray_drop_logits, *settings)
    res = {"depth_loss": out[0], "intensity_loss": out[1], "ray_drop_loss": out[2]}
    for i in range(len(prop_depths)):
        res[f"depth_loss_{i}"] = out[4 + i]
    res["quantile"], res["quantile_mask"] = out[3].detach(), mask
    return res
