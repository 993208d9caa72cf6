"""Device-side timing of one TRAINING step of the NFF path (SURVEY 8f row f2; development aid, not the bench):
NeuRAD's train batch (40 960 camera + 16 384 lidar rays, datamanagers/ad_datamanager.py:38-41) through the module walk
with the hand-written backward operators, the two regularisers, loss.backward().  Prints one JSON line with the
per-phase CUDA-event times (forward + losses, backward) and rays/s.  (The CPU reference of a training step -- torch
autograd through the oracle -- belongs to bench.py's cpu_baseline leg once a training metric is benched: only tests/,
smoke() and that leg may execute oracle/.)

  python tools/train_probe.py [--cam-rays 40960] [--lidar-rays 16384] [--actors 0] [--steps 5] [--small-tables]
                              [--camopt {off,so3xr3,scaled}] [--profile]

--camopt trains camera pose corrections as well (CameraOptimizer SO3xR3, or the scaled variant of neurad-scaleopt): rays
of sensor k use camera k, pose_adjustment starts at a seeded ~1e-2.  --profile adds one step under torch.profiler and
prints the device time of the position-gradient kernels.
  ncu --set full --clock-control none -k regex:neurad_encoding_bwd -c 2 python tools/train_probe.py --steps 1

Written without GPU access (round 1 budget was spent): first thing to run in round 2.
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import neurad_studio_b200 as nsb  # noqa: E402
from neurad_studio_b200 import losses as L  # noqa: E402
from neurad_studio_b200 import scene  # noqa: E402
from neurad_studio_b200.config import CameraOptimizerConfig, scaleopt_camera_optimizer  # noqa: E402
from neurad_studio_b200.nerfstudio_api import NeuRADModel, RayBundle  # noqa: E402


def make_batch(cfg, n_cam, n_lidar, trajs, device):
    rays = scene.random_rays(n_cam + n_lidar, cfg, seed=3, trajectories=trajs)
    is_lidar = torch.zeros(n_cam + n_lidar, 1, dtype=torch.bool)
    is_lidar[n_cam:] = True  # camera rays first, lidar rays last (neurad.py:418 relies on this order)
    rays["is_lidar"] = is_lidar
    gen = torch.Generator().manual_seed(4)
    md = {"is_lidar": is_lidar.to(device), "sensor_idxs": rays["sensor_idx"].to(device),
          "directions_norm": (2 + 78 * torch.rand(n_cam + n_lidar, 1, generator=gen)).to(device),
          "did_return": (torch.rand(n_cam + n_lidar, 1, generator=gen) < 0.9).to(device)}
    rb = RayBundle(origins=rays["origins"].to(device), directions=rays["directions"].to(device),
                   pixel_area=rays["pixel_area"].to(device), times=rays["times"].to(device), metadata=md,
                   camera_indices=rays["sensor_idx"].reshape(-1, 1).long().to(device))
    return rays, rb


def step(model, rb, targets):
    if model.camera_optimizer.config.mode != "off":  # what NeuRADModel.get_outputs does in training mode
        rb = rb.flatten()
        model.camera_optimizer.apply_to_raybundle(rb)
    out = model.get_nff_outputs(rb, calc_lidar_losses=True)
    loss = ((out["features"] - targets["features"]) ** 2).mean() + 0.01 * (out["depth"] - targets["depth"]).abs().mean()
    loss = loss + 0.001 * L.zipnerf_interlevel_loss(out["weights_list"], out["ray_samples_list"])
    loss = loss + 0.002 * L.distortion_loss(out["weights_list"], out["ray_samples_list"])
    loss = loss + 0.001 * (out["prop_weights_loss_0"] + out["prop_weights_loss_1"]) / max(int(rb.metadata["is_lidar"].sum()), 1)
    return out, loss


def neurad_batch(cfg, rb, n_cam, patch, device):
    """The supervision of a NeuRAD training batch for get_metrics_dict / get_loss_dict: camera images at the decoder's
    upsampled resolution, the lidar rows' distances and points (intensity in column 3), is_lidar / did_return over all
    rays."""
    gen = torch.Generator().manual_seed(6)
    md = rb.metadata
    up = cfg.rgb_upsample_factor
    n_lidar = len(rb) - n_cam
    return {"image": torch.rand(n_cam // (patch[0] * patch[1]), patch[0] * up, patch[1] * up, 3, generator=gen).to(device),
            "is_lidar": md["is_lidar"], "did_return": md["did_return"], "distance": md["directions_norm"][n_cam:],
            "lidar": torch.cat([50 * (torch.rand(n_lidar, 3, generator=gen) - 0.5), torch.rand(n_lidar, 1, generator=gen)],
                               dim=1).to(device)}


def neurad_step(model, rb, batch, patch):
    """One step on NeuRAD's own objective (neurad.py:461-561): get_outputs (camera optimizer, module walk, lidar head, the
    rgb decoder's torch training path) -> get_metrics_dict -> get_loss_dict, summed."""
    out = model.get_outputs(rb, patch)
    metrics = model.get_metrics_dict(out, batch)
    return out, sum(model.get_loss_dict(out, batch, metrics).values())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cam-rays", type=int, default=40960)
    ap.add_argument("--lidar-rays", type=int, default=16384)
    ap.add_argument("--actors", type=int, default=0)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--small-tables", action="store_true", help="2^14 / 2^13 slot tables instead of NeuRAD's 2^22 / 2^20")
    ap.add_argument("--camopt", choices=("off", "so3xr3", "scaled"), default="off")
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--objective", choices=("synthetic", "neurad"), default="synthetic",
                    help="synthetic: feature / depth targets plus the regularisers; neurad: the mirror's get_metrics_dict / "
                         "get_loss_dict on 32 x 32 camera patches, with a fixed stand-in perceptual loss")
    ap.add_argument("--preset", choices=nsb.PRESETS, default=None,
                    help="the model config and camera optimizer of a reference preset (overrides --camopt and the table sizes)")
    a = ap.parse_args()
    dev = "cuda"
    cfg = nsb.small_config(n_actors=a.actors, log2_main=14, log2_prop=13) if a.small_tables else nsb.NeuRADConfig(n_actors=a.actors)
    preset_copt = None
    if a.preset is not None:
        cfg, preset_copt = nsb.preset(a.preset)
        cfg.n_actors = a.actors
    trajs = scene.make_trajectories(a.actors, cfg.duration) if a.actors else None
    params = scene.make_params(cfg, seed=1, beta=3.0, sdf_bias=0.6, trajectories=trajs)
    copt = {"off": None, "so3xr3": CameraOptimizerConfig(mode="SO3xR3"), "scaled": scaleopt_camera_optimizer()}[a.camopt]
    if preset_copt is not None:
        copt = None if preset_copt.mode == "off" else preset_copt
    model = NeuRADModel(cfg, trajs, camera_optimizer=copt, num_cameras=cfg.num_sensors)
    params.update({"camera_optimizer." + k: v for k, v in model.camera_optimizer.state_dict().items()})
    model.load_reference_state_dict(params)
    if a.camopt != "off":
        with torch.no_grad():
            model.camera_optimizer.pose_adjustment.copy_((torch.rand(cfg.num_sensors, 6, generator=torch.Generator().manual_seed(5)) - 0.5) * 2e-2)
    model = model.to(dev)
    model.requires_grad_(True)
    model.train()
    rays, rb = make_batch(cfg, a.cam_rays, a.lidar_rays, trajs, dev)
    n = len(rb)
    with torch.no_grad():
        ref = model.get_nff_outputs(rb, fused=True)
    targets = {"features": ref["features"] + 0.1, "depth": ref["depth"] * 1.1}
    if a.objective == "neurad":
        patch = (32, 32)
        if a.cam_rays % (patch[0] * patch[1]):
            raise SystemExit("--objective neurad needs --cam-rays in whole 32 x 32 patches")
        batch = neurad_batch(cfg, rb, a.cam_rays, patch, dev)
        model.vgg_loss = lambda rgb, image: (rgb - image).abs().mean()  # fixed stand-in: no VGG19 weights ship
        step_fn = lambda model, rb, targets: neurad_step(model, rb, batch, patch)  # noqa: E731
    else:
        step_fn = step
    ev = lambda: torch.cuda.Event(enable_timing=True)  # noqa: E731
    times = {"forward_and_losses": [], "backward": []}
    for it in range(a.warmup + a.steps):
        model.zero_grad(set_to_none=True)
        e0, e1, e2 = ev(), ev(), ev()
        e0.record()
        out, loss = step_fn(model, rb, targets)
        e1.record()
        loss.backward()
        e2.record()
        torch.cuda.synchronize()
        if it >= a.warmup:
            times["forward_and_losses"].append(e0.elapsed_time(e1))
            times["backward"].append(e1.elapsed_time(e2))
    model._bind().check_status()
    kernels = {}
    if a.profile:
        from torch.profiler import ProfilerActivity, profile

        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            model.zero_grad(set_to_none=True)
            step_fn(model, rb, targets)[1].backward()
            torch.cuda.synchronize()
        for e in prof.key_averages():
            if "mean_bwd" in e.key or "isotropic_gaussian" in e.key or "neurad_encoding_bwd" in e.key:
                kernels[e.key[:80]] = {"calls": e.count, "device_ms": getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0)) / 1e3}
    med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
    total = med["forward_and_losses"] + med["backward"]
    what = "NFF training step (module walk + hand-written backward operators), device time"
    if a.objective == "neurad":
        what = "NFF training step on NeuRAD's objective (get_outputs -> get_metrics_dict -> get_loss_dict), device time"
    res = {"what": what, "rays": n,
           "cam_rays": a.cam_rays, "lidar_rays": a.lidar_rays, "actors": a.actors, "tables": a.preset or ("small" if a.small_tables else "neurad-default"),
           "ms": med, "ms_total": total, "rays_per_s": n / total * 1e3, "loss": float(loss.detach()), "camopt": a.camopt,
           "gpu": torch.cuda.get_device_name(), "kernels": kernels}
    if a.objective == "neurad":
        res["objective"] = "neurad"
    print(json.dumps(res))


if __name__ == "__main__":
    main()
