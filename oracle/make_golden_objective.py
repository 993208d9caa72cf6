"""TEST INFRASTRUCTURE ONLY -- pin NeuRAD's training objective to the real reference.

Run in the build container (needs /root/reference):   python -m oracle.make_golden_objective

The reference's unbound `NeuRADModel.get_metrics_dict` / `get_loss_dict` (models/neurad.py:461-561) run on a stand-in
`self` that carries what those lines read: the real `LossSettings()`, the reference's L1Loss / MSELoss /
BCEWithLogitsLoss, its `zipnerf_interlevel_loss` (its `distortion_loss` is module-level in neurad.py and runs as is), its
camera optimizer (mode "off", ad_model.py's default), the eval-metric lambdas of neurad.py:268-270, a restated psnr
(torchmetrics' PeakSignalNoiseRatio(data_range=1.0) on one batch) and a fixed differentiable stand-in `vgg_loss` that the
tests give the mirror too.  `torch.quantile` is wrapped during the call, so the quantile and its input -- hence the mask
`loss < quantile` -- are the reference's own values.

For every case the file records the inputs, every metric and loss value, and the autograd gradients of the summed loss
dict with respect to depth, the proposal depths, intensity, the ray-drop logits, non_nearby_weights, prop_weights_loss_i,
rgb and every weights_list entry.  Everything is written to tests/golden/objective.npz.
"""
from __future__ import annotations

import math
import os
import sys
from types import SimpleNamespace

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import ref_import  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "objective.npz")
ROUNDS = 2
SDF_BETA = 0.1
PROP_SAMPLES, SAMPLES = 8, 6
# name: (camera patches, lidar rays, training, lidar options).  The camera-only batch carries no weights_list: with one,
# the reference's get_loss_dict reads the lidar-only depth_loss_<i> (neurad.py:548-549) and raises KeyError.
CASES = {
    "mixed": (2, 300, True, dict(seed=1)),
    "repeated": (0, 400, True, dict(seed=2, repeat=True)),
    "n21": (0, 21, True, dict(seed=3)),
    "n41": (0, 41, True, dict(seed=4)),
    "n40": (0, 40, True, dict(seed=5)),
    "n1": (0, 1, True, dict(seed=6, return_frac=1.0)),
    "n2": (0, 2, True, dict(seed=7)),
    "all_returns": (0, 200, True, dict(seed=8, return_frac=1.0)),
    "no_returns": (0, 200, True, dict(seed=9, return_frac=0.0)),
    "nan": (0, 200, True, dict(seed=10, nan_at=(17,))),
    "camera_only": (2, 0, True, None),
    "lidar_only": (0, 500, True, dict(seed=11)),
    "eval": (2, 300, False, dict(seed=12)),
}
GRAD_KEYS = ["depth", "prop_depth_0", "prop_depth_1", "intensity", "ray_drop_logits", "non_nearby_weights",
             "prop_weights_loss_0", "prop_weights_loss_1", "rgb", "weights_list_0", "weights_list_1", "weights_list_2"]


def psnr(preds, target):
    return -torch.log(torch.sum((preds - target) ** 2) / target.numel()) * (10 / math.log(10.0))


def vgg_stand_in(rgb, image):
    """Deterministic, differentiable stand-in for VGGPerceptualLossPix2Pix (no VGG19 weights here)."""
    return (rgb - image).abs().mean() + 0.5 * ((rgb.mean(-1) - image.mean(-1)) ** 2).mean()


class SpacingBins:
    """What the regularisers read of a RaySamples: spacing_starts / spacing_ends [N,S,1] (the reference's
    ray_samples_to_sdist, losses.py:107-112) and per_ray_spacing_bins() [N,S+1] (the mirror's)."""

    def __init__(self, sdist: torch.Tensor):
        self.sdist = sdist
        self.spacing_starts, self.spacing_ends = sdist[:, :-1, None], sdist[:, 1:, None]

    def per_ray_spacing_bins(self):
        return self.sdist


def make_case(n_patches: int, n_lidar: int, lidar_opts):
    """(outputs, batch) of a training batch: camera rays first (2 x 4 x 4 patches, rgb at 3x), lidar rays last."""
    from tests import objective_cases as C

    g = torch.Generator().manual_seed(100 + n_lidar + n_patches)
    n_cam = n_patches * 16
    n = n_cam + n_lidar
    outputs, batch = {}, {}
    if n_patches:
        outputs["rgb"] = torch.rand(n_patches, 12, 12, 3, generator=g)
        batch["image"] = torch.rand(n_patches, 12, 12, 3, generator=g)
    depth = 1 + 79 * torch.rand(n, 1, generator=g)
    props = [1 + 79 * torch.rand(n, 1, generator=g) for _ in range(ROUNDS)]
    if n_lidar:
        d = C.lidar_inputs(n_lidar, **lidar_opts)
        depth[n_cam:] = d["pred"]
        for i in range(ROUNDS):
            props[i][n_cam:] = d["props"][i]
        is_lidar = torch.zeros(n, 1, dtype=torch.bool)
        is_lidar[n_cam:] = True
        did_return = torch.rand(n, 1, generator=g) < 0.5
        did_return[n_cam:, 0] = d["did_return"]
        batch.update(is_lidar=is_lidar, did_return=did_return, distance=d["distance"], lidar=d["lidar"])
        outputs.update(intensity=d["intensity"], ray_drop_logits=d["logits"])
        outputs["non_nearby_weights"] = torch.rand(3 * n_lidar, generator=g) * 0.3
        for i in range(ROUNDS):
            outputs[f"prop_weights_loss_{i}"] = torch.rand((), generator=g) * n_lidar * 0.05
    outputs["depth"] = depth
    for i in range(ROUNDS):
        outputs[f"prop_depth_{i}"] = props[i]
    sdists, weights = [], []
    for s in (PROP_SAMPLES, PROP_SAMPLES, SAMPLES):
        sd = torch.sort(torch.rand(n, s + 1, generator=g), dim=-1).values
        sd[:, 0], sd[:, -1] = 0.0, 1.0
        sdists.append(sd)
        w = torch.rand(n, s, 1, generator=g)
        weights.append(w / w.sum(1, keepdim=True) * 0.9)
    return outputs, batch, sdists, weights


def reference_self(training: bool):
    from nerfstudio.cameras.camera_optimizers import CameraOptimizerConfig
    from nerfstudio.model_components.losses import zipnerf_interlevel_loss
    from nerfstudio.models.neurad import LossSettings
    from torch.nn import BCEWithLogitsLoss, L1Loss, MSELoss

    return SimpleNamespace(
        device=torch.device("cpu"), training=training,
        config=SimpleNamespace(loss=LossSettings(), num_proposal_rounds=ROUNDS, field=SimpleNamespace(use_sdf=True)),
        field=SimpleNamespace(sdf_to_density=SimpleNamespace(beta=torch.tensor(SDF_BETA))),
        psnr=psnr, rgb_loss=MSELoss(), depth_loss=L1Loss(reduction="none"), intensity_loss=MSELoss(reduction="none"),
        vgg_loss=vgg_stand_in, ray_drop_loss=BCEWithLogitsLoss(), interlevel_loss=zipnerf_interlevel_loss,
        median_l2=lambda pred, gt: torch.median((pred - gt) ** 2),
        mean_rel_l2=lambda pred, gt: torch.mean(((pred - gt) / gt) ** 2),
        rmse=lambda pred, gt: torch.sqrt(torch.mean((pred - gt) ** 2)),
        camera_optimizer=CameraOptimizerConfig(mode="off").setup(num_cameras=1, device="cpu"),
    )


def run_reference(outputs, batch, sdists, weights, training):
    """(metrics, losses, grads {key: tensor}, quantile or None, quantile input or None)"""
    from nerfstudio.models.neurad import NeuRADModel

    outs = {k: v.clone().requires_grad_(True) for k, v in outputs.items()}
    wl = [w.clone().requires_grad_(True) for w in weights]
    if wl:
        outs["weights_list"] = wl
        outs["ray_samples_list"] = [SpacingBins(s) for s in sdists]
    seen = []
    quantile = torch.quantile

    def recording_quantile(x, q, *a, **k):
        r = quantile(x, q, *a, **k)
        seen.append((x.detach().clone(), r.detach().clone()))
        return r

    torch.quantile = recording_quantile
    try:
        me = reference_self(training)
        metrics = NeuRADModel.get_metrics_dict(me, outs, dict(batch))
        losses = NeuRADModel.get_loss_dict(me, outs, dict(batch), metrics)
    finally:
        torch.quantile = quantile
    total = sum(losses.values())
    leaves = {k: outs[k] for k in GRAD_KEYS if k in outs}
    leaves.update({f"weights_list_{i}": w for i, w in enumerate(wl)})
    got = torch.autograd.grad(total, list(leaves.values()), allow_unused=True)
    grads = {k: (torch.zeros_like(t) if g is None else g) for (k, t), g in zip(leaves.items(), got)}
    q, qin = (seen[0][1], seen[0][0]) if seen else (None, None)
    return metrics, losses, grads, q, qin


def main():
    ref_import.install()
    out = {}
    for name, (patches, n_lidar, training, opts) in CASES.items():
        outputs, batch, sdists, weights = make_case(patches, n_lidar, opts)
        if n_lidar == 0:
            sdists, weights = [], []
        metrics, losses, grads, q, qin = run_reference(outputs, batch, sdists, weights, training)
        p = f"{name}_"
        out[p + "training"] = np.bool_(training)
        for k, v in outputs.items():
            out[p + "out_" + k] = v.numpy()
        for k, v in batch.items():
            out[p + "in_" + k] = v.numpy()
        for i, (s, w) in enumerate(zip(sdists, weights)):
            out[p + f"sdist_{i}"], out[p + f"weights_{i}"] = s.numpy(), w.numpy()
        out[p + "metric_keys"] = np.array(sorted(metrics))
        out[p + "loss_keys"] = np.array(sorted(losses))
        for k, v in metrics.items():
            out[p + "metric_" + k] = np.float32(float(v))
        for k, v in losses.items():
            out[p + "loss_" + k] = np.float32(float(v))
        for k, v in grads.items():
            out[p + "grad_" + k] = v.numpy()
        if q is not None:
            out[p + "quantile"] = q.numpy()
            out[p + "quantile_mask"] = (qin < q).squeeze(-1).numpy()
        print(f"{name:12s} " + "  ".join(f"{k}={float(v):.6g}" for k, v in losses.items()))
    np.savez_compressed(GOLDEN, **out)
    print("wrote", GOLDEN, f"({os.path.getsize(GOLDEN)} bytes)")


if __name__ == "__main__":
    main()
