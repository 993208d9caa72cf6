"""Shared pieces of the lidar-simulation tests (tests/test_lidar_sim_cpu.py, tests/test_zz_lidar_sim_gpu.py).

A restatement of the sweep model of scene.LidarSensor / b200nerf_raygen_lidar_sweeps (float64 directions and origins,
fp32 times in the kernel's order), the viewer's point filter and the sensor-frame transform in torch, and the golden
tests/golden/lidar_sweep.npz (oracle/make_golden_lidar_sweep.py: the reference's render of the viewer's sweep)."""
import math

import numpy as np
import torch

from tests.helpers import cfg_from_meta, load_golden

TWO_PI_F32 = np.float32(6.283185307179586)


def linspace_f32(e0: float, e1: float, beams: int) -> torch.Tensor:
    """torch.linspace(e0, e1, beams) in fp32, written out (start + step * i for the first half, end - step * (n-1-i)
    for the second), every operation one IEEE fp32 rounding: the elevations of b200nerf_raygen_lidar_grid."""
    e0, e1 = np.float32(e0), np.float32(e1)
    step = (e1 - e0) / np.float32(beams - 1) if beams > 1 else np.float32(0)
    out = [e0 + step * np.float32(b) if b < beams // 2 else e1 - step * np.float32(beams - 1 - b) for b in range(beams)]
    return torch.from_numpy(np.array(out, dtype=np.float32))


def column_azimuths(step: float, n_az: int) -> torch.Tensor:
    """torch.arange(0, 2 pi, step) in fp32: k * step in float64, then cast."""
    return (torch.arange(n_az, dtype=torch.float64) * step).float()


def sweep_rays_f64(sensor, pose, time, velocity, step, n_az):
    """One sweep of scene.LidarSensor `sensor` at `pose` [3,4]: origins, directions [B*C,3] in float64 and times [B*C]
    in fp32 with the kernel's roundings.  Direction = R (cos v cos h, cos v sin h, sin v) with h = column azimuth +
    beam offset; dt = (column azimuth / 2 pi - 0.5) * revolution_time; origin = t + velocity * dt."""
    elev = torch.as_tensor(sensor.elevations, dtype=torch.float32).double()
    b = elev.numel()
    off = torch.zeros(b, dtype=torch.float64) if sensor.azimuth_offsets is None else torch.as_tensor(sensor.azimuth_offsets).double()
    h_col = column_azimuths(step, n_az)
    # the kernel adds the offset to the fp32 column azimuth in fp32
    h = (h_col[None, :] + torch.as_tensor(off, dtype=torch.float32)[:, None]).double()
    v = elev[:, None].expand(b, n_az)
    dl = torch.stack([torch.cos(v) * torch.cos(h), torch.cos(v) * torch.sin(h), torch.sin(v)], -1).reshape(-1, 3)
    pose = torch.as_tensor(pose, dtype=torch.float32).double()
    d = dl @ pose[:3, :3].T
    dt32 = ((h_col / torch.tensor(TWO_PI_F32)) - 0.5) * torch.tensor(np.float32(sensor.revolution_time))
    dt32 = dt32[None, :].expand(b, n_az).reshape(-1)
    times = torch.tensor(np.float32(time)) + dt32
    o = pose[:3, 3][None, :].expand(b * n_az, 3).clone()
    if velocity is not None:
        o = o + dt32.double()[:, None] * torch.as_tensor(velocity, dtype=torch.float32).double()[None, :]
    return o, d, times


def torch_epilogue(origins, directions, times, depth, intensity, prob, threshold, poses, scan_times, shape):
    """The viewer's filter by boolean indexing and ad_model.py's sensor-frame transform, in torch: (points_sensor [M,5],
    points_world [M,3], index [M,3], counts [S])."""
    s, b, c = shape
    keep = (prob.reshape(-1) < threshold) if prob is not None else (depth.reshape(-1) < threshold)
    sweep = torch.arange(s, device=depth.device).repeat_interleave(b * c)
    pw = origins + directions * depth.reshape(-1, 1)
    poses = torch.as_tensor(poses, dtype=torch.float32).to(depth.device)
    rot_t = poses[:, :3, :3].transpose(1, 2)[sweep]
    tinv = -(poses[:, :3, :3].transpose(1, 2) @ poses[:, :3, 3:])[..., 0][sweep]
    ps = (rot_t @ pw[..., None])[..., 0] + tinv
    dt = times.reshape(-1) - torch.as_tensor(scan_times, dtype=torch.float32).to(depth.device)[sweep]
    points = torch.cat([ps, intensity.reshape(-1, 1), dt[:, None]], -1)
    j = torch.arange(s * b * c, device=depth.device)
    index = torch.stack([sweep, (j % (b * c)) // c, j % c], -1).int()
    counts = torch.stack([keep[sweep == k].sum() for k in range(s)]).int()
    return points[keep], pw[keep], index[keep], counts


_G = None


def golden():
    """(meta, cfg, params, arrays) of tests/golden/lidar_sweep.npz."""
    global _G
    if _G is None:
        meta, g = load_golden("lidar_sweep.npz")
        _G = (meta, cfg_from_meta(meta), g["param"], g)
    return _G


def viewer_sensor(meta):
    """The viewer's panel values as a LidarSensor: linspace elevations, no offsets, no rolling shutter, zero pixel area
    and the fallback sensor index."""
    from neurad_studio_b200.scene import LidarSensor

    return LidarSensor.from_fov(meta["fov"][0], meta["fov"][1], meta["beams"], meta["azim_res"], revolution_time=0.0,
                                h_div=0.0, v_div=0.0, sensor_idx=meta["fallback_sensor_idx"])


def viewer_pose(meta):
    pose = torch.zeros(1, 3, 4)
    pose[0, :, :3] = torch.eye(3)
    pose[0, :, 3] = torch.tensor(meta["position"])
    return pose


def rel_to_max(a, b):
    a, b = a.detach().cpu().double(), b.detach().cpu().double()
    return (a.reshape(b.shape) - b).abs().max().item() / (b.abs().max().item() + 1e-30)


def nonuniform_sensor(beams=64, seed=0, **kw):
    """A beam table with uneven spacing, unsorted, and per-beam azimuth offsets (a synthetic table, not a product's)."""
    from neurad_studio_b200.scene import LidarSensor

    g = torch.Generator().manual_seed(seed)
    u = torch.linspace(-1.0, 1.0, beams, dtype=torch.float64)
    elev = torch.deg2rad(-8.0 + 17.0 * torch.sign(u) * u.abs() ** 1.7).float()  # dense near -8 deg
    elev = elev[torch.randperm(beams, generator=g)]
    off = torch.deg2rad((torch.rand(beams, generator=g) - 0.5) * 6.0).float()
    return LidarSensor(elevations=elev, azimuth_resolution_deg=kw.pop("azimuth_resolution_deg", 0.2), azimuth_offsets=off, **kw)


def pose_yaw(x, y, z, yaw, pitch=0.0):
    cy, sy, cp, sp = math.cos(yaw), math.sin(yaw), math.cos(pitch), math.sin(pitch)
    rz = torch.tensor([[cy, -sy, 0.0], [sy, cy, 0.0], [0.0, 0.0, 1.0]])
    ry = torch.tensor([[cp, 0.0, sp], [0.0, 1.0, 0.0], [-sp, 0.0, cp]])
    p = torch.zeros(3, 4)
    p[:, :3] = rz @ ry
    p[:, 3] = torch.tensor([x, y, z])
    return p
