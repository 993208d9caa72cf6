"""CPU: the host side of simulated lidar sweeps (scene.LidarSensor, backend.lidar_columns) and the golden's own
consistency.

- LidarSensor.from_fov gives the viewer's elevation table (torch.linspace of np.deg2rad) bit for bit.  The linspace
  b200nerf_raygen_lidar_grid evaluates on the device (restated in fp32 by lidar_sim_cases.linspace_f32) is within one
  ulp of it but not always equal: torch's CPU kernel rounds differently for some beams.  With one beam torch returns
  the start and the grid kernel the end; the sweep path takes the table and so follows torch.
- lidar_columns gives the column count of the viewer's torch.arange(0, 2 pi, step); the kernel's column azimuths
  float(k * step) are within one ulp of torch's.
- The golden's bundle is the sweep model's rays with the viewer's parameters (float64 restatement, 1e-6).
"""
import math

import numpy as np
import pytest
import torch

from tests import lidar_sim_cases as C

FOVS = [(-25.0, 15.0, 128), (-20.0, 10.0, 8), (-30.67, 10.67, 32), (-15.0, 15.0, 64), (-24.9, 2.0, 33), (-10.0, 10.0, 1),
        (-16.0, 15.0, 2)]


@pytest.mark.parametrize("fov", FOVS, ids=lambda f: f"{f[0]}_{f[1]}_{f[2]}")
def test_from_fov_is_the_viewers_linspace(fov):
    from neurad_studio_b200.scene import LidarSensor

    lo, hi, beams = fov
    s = LidarSensor.from_fov(lo, hi, beams, 0.2)
    viewer = torch.linspace(*np.deg2rad((lo, hi)), beams)
    assert s.elevations.dtype == torch.float32 and torch.equal(s.elevations, viewer)
    e0, e1 = (float(v) for v in np.deg2rad((lo, hi)).astype(np.float32))  # what raygen_lidar_grid passes the kernel
    kernel = C.linspace_f32(e0, e1, beams)
    if beams == 1:  # torch.linspace gives the start, the grid kernel's second-half branch the end
        assert viewer.item() == np.float32(e0) and kernel.item() == np.float32(e1)
    else:
        assert (kernel - viewer).abs().max().item() <= float(np.spacing(np.float32(max(abs(e0), abs(e1)))))
    assert s.beams == beams and s.azimuth_offsets is None


@pytest.mark.parametrize("res", [0.1, 360.0 / 2048, 360.0 / 1800, 7.5, 10.0, 0.33])
def test_lidar_columns_match_torch_arange(res):
    from neurad_studio_b200.backend import lidar_columns

    step, n = lidar_columns(res)
    ref = torch.arange(0, 2 * np.pi, np.deg2rad(res))
    assert n == ref.numel() and step == float(np.deg2rad(res))
    assert (C.column_azimuths(step, n) - ref).abs().max().item() <= float(np.spacing(np.float32(2 * np.pi)))


@pytest.mark.parametrize("res", [0.0, -1.0, float("nan"), float("inf")])
def test_lidar_columns_reject_bad_resolution(res):
    from neurad_studio_b200.backend import lidar_columns

    with pytest.raises(ValueError):
        lidar_columns(res)


def test_golden_bundle_is_the_sweep_model():
    from neurad_studio_b200.backend import lidar_columns

    meta, cfg, params, g = C.golden()
    sensor = C.viewer_sensor(meta)
    step, n_az = lidar_columns(meta["azim_res"])
    o, d, t = C.sweep_rays_f64(sensor, C.viewer_pose(meta)[0], meta["time"], None, step, n_az)
    assert d.shape == g["ray"]["directions"].shape
    assert (d - g["ray"]["directions"].double()).abs().max().item() < 1e-6
    assert torch.equal(o.float(), g["ray"]["origins"])
    assert torch.all(t == np.float32(meta["time"]))


def test_golden_filters_are_the_viewers():
    meta, cfg, params, g = C.golden()
    out = g["out"]
    assert torch.equal(g["keep"]["ray_drop"], out["ray_drop_prob"][:, 0] < meta["ray_drop_threshold"])
    assert torch.equal(g["keep"]["max_distance"], out["depth"][:, 0] < meta["max_distance"])
    pc = torch.cat([out["depth"] * g["ray"]["directions"] + g["ray"]["origins"], out["intensity"]], -1)
    assert torch.equal(pc[g["keep"]["ray_drop"]], g["points"]["ray_drop"])
    assert torch.equal(pc[g["keep"]["max_distance"]], g["points"]["max_distance"])


def test_torch_epilogue_order_is_boolean_indexing():
    """The comparator the GPU tests use: row-major (sweep, beam, column) order, per-sweep counts."""
    s, b, c = 3, 2, 5
    n = s * b * c
    g = torch.Generator().manual_seed(3)
    depth = torch.rand(n, 1, generator=g) * 10
    o, d = torch.zeros(n, 3), torch.nn.functional.normalize(torch.rand(n, 3, generator=g), dim=-1)
    poses = torch.stack([C.pose_yaw(1.0 * k, 2.0, 0.5, 0.3 * k) for k in range(s)])
    ps, pw, idx, counts = C.torch_epilogue(o, d, torch.zeros(n), depth, torch.rand(n, generator=g), None, 5.0, poses,
                                           [0.0] * s, (s, b, c))
    flat = (idx[:, 0] * b + idx[:, 1]) * c + idx[:, 2]
    assert torch.equal(flat, (depth[:, 0] < 5.0).nonzero()[:, 0].int())
    assert int(counts.sum()) == ps.shape[0]
    back = (poses[idx[:, 0].long(), :, :3] @ ps[:, :3, None])[..., 0] + poses[idx[:, 0].long(), :, 3]
    assert (back - pw).abs().max().item() < 1e-5 * max(1.0, math.sqrt(float((pw ** 2).sum(-1).max())))
