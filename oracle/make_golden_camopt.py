"""TEST INFRASTRUCTURE ONLY -- pin the CAMERA-POSE gradients to the real reference.

Run in the build container (needs /root/reference):   python -m oracle.make_golden_camopt

For the committed forward cases tests/golden/nff_static.npz and nff_actors.npz it builds the unmodified reference
``NeuRADModel`` (as oracle/make_golden_grads.py does: implementation="torch", CPU, eval-mode sampling) and a reference
camera optimizer over NUM_CAMERAS cameras (rays are assigned camera i % NUM_CAMERAS; camera NON_TRAINABLE is listed as
non-trainable) with a seeded non-zero ``pose_adjustment`` (~1e-2).  It runs ``apply_to_raybundle`` and then
``get_nff_outputs`` on the first N_RAYS rays, back-propagates the seeded linear loss of make_golden_grads.py and records

  d pose_adjustment, d corrected origins / directions (retain_grad), the correction matrices and the regulariser value.

It asserts that torch autograd through the oracle (same corrected rays) agrees to 1e-5 of each tensor's scale and
writes tests/golden/camopt_<mode>_<case>.npz.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import neurad_studio_b200 as nsb  # noqa: E402
from neurad_studio_b200 import scene  # noqa: E402
from oracle import neurad_oracle as O  # noqa: E402
from oracle import ref_driver  # noqa: E402
from oracle.convert import to_oracle_cfg  # noqa: E402
from oracle.make_golden_grads import N_RAYS, OUT_KEYS, load_case, loss_weights  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")
NUM_CAMERAS = 3
NON_TRAINABLE = 1
ADJ_SEED = 11
# (label, mode, scaled?): SO3xR3, the scaled variant of neurad-scaleopt (method_configs.py:440-442), and SE3
MODES = (("so3xr3", "SO3xR3", False), ("scaled", "SO3xR3", True), ("se3", "SE3", False))
SCALEOPT_WEIGHTS = (1.0, 1.0, 0.01, 0.01, 0.01, 1.0)


def pose_adjustment_init():
    gen = torch.Generator().manual_seed(ADJ_SEED)
    return (torch.rand(NUM_CAMERAS, 6, generator=gen) - 0.5) * 2e-2


def camera_indices(n):
    return (torch.arange(n) % NUM_CAMERAS)[:, None]


def make_reference_optimizer(mode, scaled):
    from nerfstudio.cameras.camera_optimizers import CameraOptimizerConfig, ScaledCameraOptimizerConfig

    cfg = ScaledCameraOptimizerConfig(mode=mode, weights=SCALEOPT_WEIGHTS) if scaled else CameraOptimizerConfig(mode=mode)
    opt = cfg.setup(num_cameras=NUM_CAMERAS, device="cpu", non_trainable_camera_indices=torch.tensor([NON_TRAINABLE]))
    with torch.no_grad():
        opt.pose_adjustment.copy_(pose_adjustment_init())
    return opt


def oracle_grads(cfg, params, rays, origins, directions):
    o, d = origins.clone().requires_grad_(True), directions.clone().requires_grad_(True)
    out = O.nff_outputs(params, to_oracle_cfg(cfg), o, d, rays["pixel_area"], rays["times"], rays["sensor_idx"], rays["is_lidar"])
    G = loss_weights({k: out[k].shape for k in OUT_KEYS})
    sum((out[k] * G[k]).sum() for k in OUT_KEYS).backward()
    return o.grad, d.grad


def camopt_case(name, label, mode, scaled):
    meta, params, rays = load_case(name)
    cfg = nsb.small_config(n_actors=meta["n_actors"], log2_main=meta["log2_main"], log2_prop=meta["log2_prop"],
                           static_scale=meta["static_scale"], duration=meta["duration"], num_sensors=meta["num_sensors"])
    trajs = scene.make_trajectories(meta["n_actors"], cfg.duration, seed=meta["seed"]) if meta["n_actors"] else None
    model = ref_driver.build_reference_model(cfg, params, trajs)
    from nerfstudio.cameras.rays import RayBundle

    opt = make_reference_optimizer(mode, scaled)
    n = rays["origins"].shape[0]
    rb = RayBundle(origins=rays["origins"].clone(), directions=rays["directions"].clone(), pixel_area=rays["pixel_area"].clone(),
                   camera_indices=camera_indices(n), fars=torch.full((n, 1), 1_000_000.0), times=rays["times"].clone(),
                   metadata={"is_lidar": rays["is_lidar"].clone(), "sensor_idxs": rays["sensor_idx"].clone()})
    opt.apply_to_raybundle(rb)
    rb.origins.retain_grad()
    rb.directions.retain_grad()
    corr_o, corr_d = rb.origins.detach().clone(), rb.directions.detach().clone()
    out = model.get_nff_outputs(rb)
    G = loss_weights({k: out[k].shape for k in OUT_KEYS})
    sum((out[k] * G[k]).sum() for k in OUT_KEYS).backward()
    ref = {"pose_adjustment": opt.pose_adjustment.grad.detach().clone(), "origins": rb.origins.grad.detach().clone(),
           "directions": rb.directions.grad.detach().clone()}
    o_g, d_g = oracle_grads(cfg, params, rays, corr_o, corr_d)
    for k, v in (("origins", o_g), ("directions", d_g)):
        err = (ref[k] - v).abs().max().item() / ref[k].abs().max().item()
        assert err < 1e-5, (name, label, k, err)
    losses = {}
    opt.get_loss_dict(losses)
    arrays = {f"grad/{k}": v.numpy() for k, v in ref.items()}
    arrays.update({"pose_adjustment": opt.pose_adjustment.detach().numpy(), "correction_matrices": opt.get_correction_matrices().detach().numpy(),
                   "corrected/origins": corr_o.numpy(), "corrected/directions": corr_d.numpy(),
                   "camera_indices": camera_indices(n).numpy(), "regularizer": losses["camera_opt_regularizer"].detach().numpy()})
    if scaled:
        arrays["weights"] = opt.weights.numpy()
    arrays["__meta__"] = np.array(repr(dict(case=name, mode=mode, scaled=scaled, n_rays=N_RAYS, loss_seed=7, num_cameras=NUM_CAMERAS,
                                            non_trainable=[NON_TRAINABLE], adj_seed=ADJ_SEED, torch=torch.__version__)))
    path = os.path.join(GOLDEN, f"camopt_{label}_{name}")
    np.savez_compressed(path, **arrays)
    print(f"wrote {path}: {os.path.getsize(path)/1e3:.1f} kB")


if __name__ == "__main__":
    for case in ("nff_static.npz", "nff_actors.npz"):
        for label, mode, scaled in MODES:
            if case == "nff_actors.npz" and label == "se3":
                continue  # one SE3 case
            camopt_case(case, label, mode, scaled)
