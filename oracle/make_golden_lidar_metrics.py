"""TEST INFRASTRUCTURE ONLY -- pin NeuRAD's lidar metrics to the real reference.

Run in the build container (needs /root/reference):   python -m oracle.make_golden_lidar_metrics

- chamfer cases (oracle/lidar_metrics_oracle.py: chamfer_cases): the reference's own
  `nerfstudio.utils.math.chamfer_distance(pred, gt, 1_000, True)` -- the call of neurad.py:271 -- in fp32 on the CPU,
  next to the float64 brute-force sums of the oracle.  The difference is the reference's own rounding and cancellation
  error, which the GPU tests require the kernel to match or beat.
- metrics cases (metrics_cases): the unbound `NeuRADModel.get_image_metrics_and_images` of the reference on a stand-in
  `self` that carries the attributes the lidar branch reads (device, config.loss, the metric callables of
  neurad.py:268-271), with the batch side effects recorded.

Everything is written to tests/golden/lidar_metrics.npz.
"""
from __future__ import annotations

import os
import sys
from types import SimpleNamespace

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import lidar_metrics_oracle as LM  # noqa: E402
from oracle import ref_import  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")
NON_RETURN_LIDAR_DISTANCE = 150.0  # LossSettings default (neurad.py:87)


def reference_self(ray_drop_loss_mult: float):
    """What the lidar branch of get_image_metrics_and_images reads from `self` (neurad.py:268-271, 589-621)."""
    from nerfstudio.utils.math import chamfer_distance

    return SimpleNamespace(
        device=torch.device("cpu"),
        config=SimpleNamespace(loss=SimpleNamespace(ray_drop_loss_mult=ray_drop_loss_mult,
                                                    non_return_lidar_distance=NON_RETURN_LIDAR_DISTANCE)),
        median_l2=lambda pred, gt: torch.median((pred - gt) ** 2),
        mean_rel_l2=lambda pred, gt: torch.mean(((pred - gt) / gt) ** 2),
        rmse=lambda pred, gt: torch.sqrt(torch.mean((pred - gt) ** 2)),
        chamfer_distance=lambda pred, gt: chamfer_distance(pred, gt, 1_000, True),
    )


def main():
    ref_import.install()
    from nerfstudio.models.neurad import NeuRADModel
    from nerfstudio.utils.math import chamfer_distance

    out = {}
    for name, (pred, gt) in LM.chamfer_cases().items():
        with torch.no_grad():
            ref = chamfer_distance(pred, gt, 1_000, True)
        a, b = LM.chamfer_sums_f64(pred, gt)
        f64 = a / gt.shape[0] + b / gt.shape[0]
        rel = abs(float(ref) - f64) / f64
        print(f"chamfer {name:8s} N={pred.shape[0]} M={gt.shape[0]}  ref fp32 {float(ref):.9g}  f64 {f64:.12g}  rel err {rel:.2e}")
        assert rel < 0.5, (name, rel)  # the reference's fp32 error: ~1e-4 at 40 m, several percent at 100 m
        out[f"chamfer_{name}_pred"] = pred.numpy()
        out[f"chamfer_{name}_gt"] = gt.numpy()
        out[f"chamfer_{name}_ref"] = np.float32(ref)
        out[f"chamfer_{name}_sums_f64"] = np.array([a, b], np.float64)
        out[f"chamfer_{name}_f64"] = np.float64(f64)

    for name, (outputs, batch, mult) in LM.metrics_cases().items():
        batch = dict(batch)
        given = sorted(batch)
        metrics, images = NeuRADModel.get_image_metrics_and_images(reference_self(mult), dict(outputs), batch)
        assert images == {} and sorted(metrics) == sorted(LM.METRIC_KEYS), (name, metrics, images)
        print(f"metrics {name:8s} " + "  ".join(f"{k}={float(v):.9g}" for k, v in metrics.items()))
        for k, v in outputs.items():
            out[f"metrics_{name}_out_{k}"] = v.numpy()
        for k in given:
            out[f"metrics_{name}_in_{k}"] = batch[k].numpy()
        for k in ("is_lidar", "did_return"):  # after the call: the side effects of neurad.py:591-594
            out[f"metrics_{name}_after_{k}"] = batch[k].numpy()
        out[f"metrics_{name}_ray_drop_loss_mult"] = np.float64(mult)
        out[f"metrics_{name}_chamfer_is_tensor"] = np.bool_(isinstance(metrics["chamfer_distance"], torch.Tensor))
        for k in LM.METRIC_KEYS:
            v = metrics[k]
            out[f"metrics_{name}_{k}"] = np.float32(v) if isinstance(v, torch.Tensor) else np.float64(v)
        if metrics["chamfer_distance"].__class__ is float:
            pred = outputs["points"][(outputs["ray_drop_logits"].sigmoid() < 0.5)[:, 0]] if mult > 0 else \
                outputs["points"][(outputs["depth"] < NON_RETURN_LIDAR_DISTANCE)[:, 0]]
            gt = batch["lidar"][batch["did_return"][:, 0], :3]
            out[f"metrics_{name}_chamfer_f64"] = np.float64(LM.chamfer_f64(pred, gt))
    path = os.path.join(GOLDEN, "lidar_metrics.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, f"({os.path.getsize(path)} bytes)")


if __name__ == "__main__":
    main()
