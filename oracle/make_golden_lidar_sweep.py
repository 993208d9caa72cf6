"""TEST INFRASTRUCTURE ONLY -- tests/golden/lidar_sweep.npz from the REAL reference: the viewer's simulated lidar sweep.

Run in the build container (needs /root/reference):   python -m oracle.make_golden_lidar_sweep

The viewer's lidar render (viewer/render_state_machine.py:391-430) builds a beam x azimuth bundle from its control-panel
values, renders it with the model's get_outputs_for_camera_ray_bundle in eval mode and filters the point cloud with
ray drop on (ray_drop_prob < threshold) or off (depth < max distance).  This script states those lines with the
reference's own RayBundle and runs them on the unmodified reference NeuRADModel (implementation="torch", CPU, built by
oracle/ref_driver.py) over a scene with actors.  The bundle carries no sensor index, so the appearance embedding is the
model's fallback sensor (the viewer slider's default, 0).

The two thresholds are the medians of the render's ray-drop probabilities and depths, so that both filters keep about
half of the sweep; they are stored with the panel values, the reference's bundle, outputs, masks and point clouds.  At
the random init the probabilities lie within 1e-3 of each other, so some lie within 1e-5 of the threshold: a
comparison with another implementation of the render leaves those rays out.
"""
from __future__ import annotations

import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import neurad_studio_b200 as nsb  # noqa: E402
from neurad_studio_b200 import scene  # noqa: E402
from oracle import ref_driver  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "lidar_sweep.npz")
N_ACTORS, SEED = 4, 21
# control-panel values (viewer/control_panel.py: lidar_fov, lidar_beams, lidar_azim_res, lidar_position, time)
FOV = (-20.0, 10.0)
BEAMS = 8
AZIM_RES = 7.5
POSITION = (6.0, 0.5, 1.6)
TIME = 1.0


# hash tables at 0.1 of the unit init: with the viewer's zero pixel area every level has full weight, and at scale 1 the
# fused render's depth on the reference's own bundle is 2.2e-4 of its maximum from the reference's, above the 2e-4
# render tolerance; at 0.1 it is 3.5e-5 (an open item of DESIGN.md section 9)
TABLE_SCALE = 0.1


def make_scene():
    cfg = nsb.small_config(n_actors=N_ACTORS, log2_main=10, log2_prop=10)
    trajs = scene.make_trajectories(N_ACTORS, cfg.duration, seed=SEED)
    params = scene.make_params(cfg, seed=SEED, table_scale=TABLE_SCALE, beta=4.0, trajectories=trajs, sdf_bias=0.5)
    return cfg, trajs, params


def split_threshold(values: torch.Tensor) -> float:
    """The midpoint of the two middle values: about half the rays on either side."""
    v = values.reshape(-1).double().sort().values
    mid = v.numel() // 2
    return float(np.float32(0.5 * (v[mid - 1] + v[mid])))


def main():
    torch.manual_seed(0)
    cfg, trajs, params = make_scene()
    model = ref_driver.build_reference_model(cfg, params, trajs)
    model.fallback_sensor_idx = types.SimpleNamespace(value=0)  # the viewer slider at its default
    from nerfstudio.cameras.rays import RayBundle

    # viewer/render_state_machine.py:395-414, line for line
    v_angles = torch.linspace(*np.deg2rad(FOV), BEAMS)
    h_angles = torch.arange(0, 2 * np.pi, np.deg2rad(AZIM_RES))
    v_angles, h_angles = torch.meshgrid(v_angles, h_angles, indexing="ij")
    v_angles, h_angles = v_angles.flatten(), h_angles.flatten()
    directions = torch.stack(
        [torch.cos(v_angles) * torch.cos(h_angles), torch.cos(v_angles) * torch.sin(h_angles), torch.sin(v_angles)], dim=-1)
    origins = torch.tensor(POSITION, dtype=torch.float32)
    bundle = RayBundle(
        origins=origins,
        directions=directions,
        pixel_area=torch.zeros_like(v_angles, dtype=torch.float32)[..., None],
        metadata={"is_lidar": torch.ones_like(v_angles, dtype=torch.bool)[..., None]},
        times=torch.tensor([TIME], dtype=torch.float32),
    )
    model.eval()
    with torch.no_grad():
        outputs = model.get_outputs_for_camera_ray_bundle(bundle)
    # :416-430
    point_cloud = torch.cat([outputs["depth"] * directions + origins, outputs["intensity"]], dim=-1)
    threshold = split_threshold(outputs["ray_drop_prob"])
    max_dist = split_threshold(outputs["depth"])
    keep_drop = outputs["ray_drop_prob"].squeeze(-1) < threshold
    keep_dist = outputs["depth"].squeeze(-1) < max_dist
    n = directions.shape[0]
    assert 0 < int(keep_drop.sum()) < n and 0 < int(keep_dist.sum()) < n

    arrays = {f"param/{k}": v for k, v in params.items()}
    arrays.update({
        "ray/origins": origins.expand(n, 3).clone(), "ray/directions": directions,
        "out/depth": outputs["depth"], "out/intensity": outputs["intensity"], "out/ray_drop_prob": outputs["ray_drop_prob"],
        "out/accumulation": outputs["accumulation"],
        "keep/ray_drop": keep_drop, "keep/max_distance": keep_dist,
        "points/ray_drop": point_cloud[keep_drop], "points/max_distance": point_cloud[keep_dist],
    })
    out = {k: (v.detach().cpu().numpy() if isinstance(v, torch.Tensor) else np.asarray(v)) for k, v in arrays.items()}
    meta = dict(n_actors=N_ACTORS, log2_main=10, log2_prop=10, seed=SEED, beta=4.0, sdf_bias=0.5, table_scale=TABLE_SCALE,
                static_scale=cfg.static_scale, duration=cfg.duration, num_sensors=cfg.num_sensors,
                fov=FOV, beams=BEAMS, azim_res=AZIM_RES, position=POSITION, time=TIME, fallback_sensor_idx=0,
                ray_drop_threshold=threshold, max_distance=max_dist, torch=torch.__version__)
    out["__meta__"] = np.array(repr(meta))
    np.savez_compressed(GOLDEN, **out)
    print(f"wrote {GOLDEN}: {os.path.getsize(GOLDEN) / 1e6:.2f} MB, {n} rays; ray drop keeps {int(keep_drop.sum())}, "
          f"max distance keeps {int(keep_dist.sum())} (threshold {threshold:.6f}, max distance {max_dist:.4f})")


if __name__ == "__main__":
    main()
