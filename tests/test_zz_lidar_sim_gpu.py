"""GPU: simulated lidar sweeps (NeuRADModel.get_outputs_for_lidar_sweep, b200nerf_raygen_lidar_sweeps,
b200nerf_lidar_sweep_points).

- Ray generation: a uniform table through the sweep path is bit-identical to raygen_lidar_grid; non-uniform tables
  with azimuth offsets, a rolling shutter and several sweeps match a float64 restatement (directions and origins 1e-6
  of scale, times exact), with the sensor index, is_lidar and (sweep, beam, column) outputs.
- Point epilogue against torch on the same render outputs: kept set and order equal, points within 1e-6 of scale,
  counts equal; mixed batches with an all-dropped sweep, an all-returned sweep and a one-beam sensor.
- The reference's viewer sweep (tests/golden/lidar_sweep.npz) with ray drop on and off.
- Kept points fed back through Lidars.generate_rays / get_outputs_for_lidar render the same depths.
- Actor edits and the camera optimizer in eval change the sweep exactly as they change a render of the same rays.
"""
import pytest
import torch

from tests import lidar_sim_cases as C

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.fixture(scope="module")
def backend():
    from neurad_studio_b200.nerfstudio_api import get_backend

    return get_backend(torch.device(DEV, 0))


def _model(extra=None, **kw):
    from neurad_studio_b200.nerfstudio_api import NeuRADModel

    meta, cfg, params, g = C.golden()
    model = NeuRADModel(cfg, **kw)
    model.load_reference_state_dict({**params, **(extra or {})})
    return model.to(DEV).eval()


def _scale(x):
    return max(1.0, x.detach().abs().max().item())


# ------------------------------------------------------------------------------------------------ ray generation
def test_uniform_table_is_bit_identical_to_the_grid(backend):
    import numpy as np

    from neurad_studio_b200.scene import LidarSensor

    l2w = C.pose_yaw(12.0, -3.0, 1.9, 0.4, 0.02)
    vel = torch.tensor([10.0, 1.0, 0.0])
    grid = backend.raygen_lidar_grid(l2w, -25.0, 15.0, 128, 360.0 / 2048, scan_time=3.2, velocity=vel)
    e0, e1 = (float(v) for v in np.deg2rad((-25.0, 15.0)).astype(np.float32))
    sensor = LidarSensor(elevations=C.linspace_f32(e0, e1, 128), azimuth_resolution_deg=360.0 / 2048, revolution_time=0.1)
    sw = backend.raygen_lidar_sweeps(sensor, l2w[None], [3.2], vel[None])
    assert sw["shape"] == (1,) + grid["shape"]
    for k in ("origins", "directions", "pixel_area", "times"):
        assert torch.equal(sw[k], grid[k]), k


def test_sweeps_match_the_float64_model(backend):
    from neurad_studio_b200.backend import lidar_columns

    sensors = [C.nonuniform_sensor(64, seed=1, revolution_time=0.1, sensor_idx=5),
               C.nonuniform_sensor(64, seed=2, revolution_time=0.05, sensor_idx=6, h_div=2e-3, v_div=1e-3),
               C.nonuniform_sensor(64, seed=3, revolution_time=0.0, sensor_idx=6)]
    poses = torch.stack([C.pose_yaw(-30.0, 1.0, 2.0, 0.1), C.pose_yaw(5.0, -2.0, 1.8, -2.0, 0.05), C.pose_yaw(40.0, 0.0, 2.1, 3.0)])
    times = [1.5, 2.25, 6.0]
    vels = torch.tensor([[10.0, 0.0, 0.0], [8.0, -1.0, 0.2], [0.0, 12.0, 0.0]])
    r = backend.raygen_lidar_sweeps(sensors, poses, times, vels)
    step, n_az = lidar_columns(0.2)
    assert r["shape"] == (3, 64, n_az)
    per = 64 * n_az
    for s in range(3):
        sl = slice(s * per, (s + 1) * per)
        o, d, t = C.sweep_rays_f64(sensors[s], poses[s], times[s], vels[s], step, n_az)
        assert (r["directions"][sl].cpu().double() - d).abs().max().item() < 1e-6
        assert (r["origins"][sl].cpu().double() - o).abs().max().item() < 1e-6 * _scale(o)
        assert torch.equal(r["times"][sl].cpu().reshape(-1), t)
        assert torch.all(r["pixel_area"][sl] == torch.tensor(sensors[s].h_div) * torch.tensor(sensors[s].v_div))
        assert torch.all(r["sensor_idx"][sl] == sensors[s].sensor_idx)
    assert bool(r["is_lidar"].all())
    j = torch.arange(3 * per, device=DEV)
    want = torch.stack([j // per, (j % per) // n_az, j % n_az], -1).int()
    assert torch.equal(r["index"], want)


def test_raygen_rejects_bad_input(backend):
    import ctypes

    from neurad_studio_b200.scene import LidarSensor

    s = C.nonuniform_sensor(8)
    pose = C.pose_yaw(0.0, 0.0, 2.0, 0.0)[None]
    with pytest.raises(ValueError):  # sweeps of one call share one beam count
        backend.raygen_lidar_sweeps([s, C.nonuniform_sensor(9)], pose.repeat(2, 1, 1), [0.0, 1.0])
    with pytest.raises(ValueError):  # one time per pose
        backend.raygen_lidar_sweeps(s, pose, [0.0, 1.0])
    with pytest.raises(ValueError):  # empty table
        backend.raygen_lidar_sweeps(LidarSensor(elevations=torch.zeros(0), azimuth_resolution_deg=1.0), pose, [0.0])
    with pytest.raises(ValueError):
        backend.raygen_lidar_sweeps(LidarSensor(elevations=torch.tensor([0.0, float("nan")]), azimuth_resolution_deg=1.0), pose, [0.0])
    buf = torch.empty(64, device=DEV)
    p = ctypes.c_void_p(buf.data_ptr())
    rc = backend.lib.b200nerf_raygen_lidar_sweeps(backend._h, p, 1, 0, 4, 0.1, p, None, p, p, p, p, None, None, None, None)
    assert rc == -1  # B200NERF_ERR_INVALID: empty beam table
    rc = backend.lib.b200nerf_raygen_lidar_sweeps(backend._h, p, 1, 2, 4, 0.1, None, None, p, p, p, p, None, None, None, None)
    assert rc == -1  # no elevation table


# ------------------------------------------------------------------------------------------------ point epilogue
def _synthetic_outputs(n, seed):
    g = torch.Generator().manual_seed(seed)
    depth = (torch.rand(n, 1, generator=g) * 120.0).to(DEV)
    inten = torch.rand(n, 1, generator=g).to(DEV)
    prob = torch.rand(n, 1, generator=g).to(DEV)
    return depth, inten, prob


def _check_epilogue(r, pts, depth, inten, prob, thr, poses, times):
    ps, pw, idx, counts = C.torch_epilogue(r["origins"], r["directions"], r["times"], depth, inten, prob, thr, poses, times,
                                           r["shape"])
    m = int(pts["counts"][-1])
    assert m == ps.shape[0]
    assert torch.equal(pts["index"][:m], idx)
    assert torch.equal(pts["counts"][:-1], counts)
    off = torch.cumsum(counts, 0) - counts
    assert torch.equal(pts["offsets"], off.int())
    if m:
        assert (pts["points_world"][:m] - pw).abs().max().item() <= 1e-6 * _scale(pw)
        assert (pts["points_sensor"][:m, :3] - ps[:, :3]).abs().max().item() <= 1e-6 * _scale(pw)
        assert torch.equal(pts["points_sensor"][:m, 3], ps[:, 3])
        assert torch.equal(pts["points_sensor"][:m, 4], ps[:, 4])


@pytest.mark.parametrize("ray_drop", [True, False])
def test_epilogue_matches_torch_on_mixed_sweeps(backend, ray_drop):
    sensors = [C.nonuniform_sensor(32, seed=k, azimuth_resolution_deg=0.5, sensor_idx=5 + k % 2) for k in range(5)]
    poses = torch.stack([C.pose_yaw(10.0 * k, 1.0 - k, 1.8, 0.7 * k, 0.01 * k) for k in range(5)])
    times = [0.5 * k for k in range(5)]
    r = backend.raygen_lidar_sweeps(sensors, poses, times, torch.tensor([[9.0, 1.0, 0.0]] * 5))
    n = r["origins"].shape[0]
    per = n // 5
    depth, inten, prob = _synthetic_outputs(n, 7)
    thr = 0.4 if ray_drop else 60.0
    key = prob if ray_drop else depth
    key[per:2 * per] = thr + 1.0   # sweep 1: every ray dropped
    key[2 * per:3 * per] = thr - 0.5 if ray_drop else 1.0  # sweep 2: every ray returns
    key[3 * per + 5] = float("nan")  # NaN is never kept, as with torch
    pts = backend.lidar_sweep_points(r, depth, inten, prob if ray_drop else None, thr)
    _check_epilogue(r, pts, depth, inten, prob if ray_drop else None, thr, poses, times)
    assert int(pts["counts"][1]) == 0 and int(pts["counts"][2]) == per
    again = backend.lidar_sweep_points(r, depth, inten, prob if ray_drop else None, thr)
    for k in ("points_sensor", "points_world", "index"):  # deterministic
        m = int(pts["counts"][-1])
        assert torch.equal(again[k][:m], pts[k][:m])


def test_epilogue_one_beam_and_large_sweep(backend):
    from neurad_studio_b200.scene import LidarSensor

    one = LidarSensor(elevations=torch.tensor([0.05]), azimuth_resolution_deg=0.1, azimuth_offsets=torch.tensor([0.01]))
    poses = torch.stack([C.pose_yaw(0.0, 0.0, 2.0, 0.3), C.pose_yaw(3.0, 0.0, 2.0, 0.4)])
    r = backend.raygen_lidar_sweeps(one, poses, [1.0, 1.1])
    assert r["shape"] == (2, 1, 3600)
    depth, inten, prob = _synthetic_outputs(r["origins"].shape[0], 8)
    _check_epilogue(r, backend.lidar_sweep_points(r, depth, inten, prob, 0.5), depth, inten, prob, 0.5, poses, [1.0, 1.1])
    big = C.nonuniform_sensor(128, seed=4, azimuth_resolution_deg=360.0 / 2048)
    r = backend.raygen_lidar_sweeps(big, poses, [1.0, 1.1])
    depth, inten, prob = _synthetic_outputs(r["origins"].shape[0], 9)
    _check_epilogue(r, backend.lidar_sweep_points(r, depth, inten, None, 70.0), depth, inten, None, 70.0, poses, [1.0, 1.1])


def test_epilogue_scan_carries_across_tile_chunks(backend):
    """Sweeps of more than 1024 tiles of 1024 rays: the one-CTA scan walks the tile counts in chunks and carries the
    running offset from chunk to chunk and from sweep to sweep."""
    from neurad_studio_b200.scene import LidarSensor

    one = LidarSensor(elevations=torch.tensor([0.02]), azimuth_resolution_deg=360.0 / 1_100_000)
    poses = torch.stack([C.pose_yaw(0.0, 0.0, 2.0, 0.1), C.pose_yaw(2.0, 1.0, 2.0, -0.2)])
    r = backend.raygen_lidar_sweeps(one, poses, [1.0, 1.1])
    assert r["shape"][2] > 1024 * 1024
    depth, inten, prob = _synthetic_outputs(r["origins"].shape[0], 10)
    _check_epilogue(r, backend.lidar_sweep_points(r, depth, inten, prob, 0.3), depth, inten, prob, 0.3, poses, [1.0, 1.1])


def test_epilogue_rejects_bad_input(backend):
    from neurad_studio_b200 import lib as L

    pose = C.pose_yaw(0.0, 0.0, 2.0, 0.0)[None]
    r = backend.raygen_lidar_sweeps(C.nonuniform_sensor(8, azimuth_resolution_deg=10.0), pose, [0.0])
    n = r["origins"].shape[0]
    depth, inten, prob = _synthetic_outputs(n, 1)
    for thr in (float("inf"), float("nan")):
        with pytest.raises(L.B200NerfError):
            backend.lidar_sweep_points(r, depth, inten, prob, thr)
    with pytest.raises(ValueError):
        backend.lidar_sweep_points(r, depth[:-1], inten, prob, 0.5)


# ------------------------------------------------------------------------------------------------ the model API
@pytest.mark.parametrize("ray_drop", [True, False])
def test_viewer_sweep_matches_reference(ray_drop):
    meta, cfg, params, g = C.golden()
    model = _model()
    thr = meta["ray_drop_threshold"] if ray_drop else None
    out = model.get_outputs_for_lidar_sweep(C.viewer_sensor(meta), C.viewer_pose(meta), [meta["time"]], ray_drop_threshold=thr,
                                            max_distance=None if ray_drop else meta["max_distance"])
    ref = g["out"]
    assert C.rel_to_max(out["depth"], ref["depth"]) < 2e-4
    assert C.rel_to_max(out["intensity"], ref["intensity"]) < 1e-4
    assert C.rel_to_max(out["ray_drop_prob"], ref["ray_drop_prob"]) < 1e-4
    assert out["depth_image"].shape == (1, meta["beams"], ref["depth"].shape[0] // meta["beams"])
    assert out["depth_image"].data_ptr() == out["depth"].data_ptr()  # a view, not a copy
    key, lim = (ref["ray_drop_prob"][:, 0], meta["ray_drop_threshold"]) if ray_drop else (ref["depth"][:, 0], meta["max_distance"])
    want = g["keep"]["ray_drop" if ray_drop else "max_distance"]
    got = torch.zeros_like(want)
    flat = out["point_index"][:, 1].long().cpu() * out["depth_image"].shape[2] + out["point_index"][:, 2].long().cpu()
    got[flat] = True
    near = (key - lim).abs() <= 1e-5
    assert torch.equal(got[~near], want[~near])
    both = got & want
    ref_pts = torch.zeros(want.shape[0], 4)
    ref_pts[want] = g["points"]["ray_drop" if ray_drop else "max_distance"]
    ours = torch.zeros(want.shape[0], 4)
    ours[flat] = torch.cat([out["points_world"], out["points"][:, 3:4]], -1).cpu()
    scale = _scale(ref_pts[both, :3])
    assert (ours[both] - ref_pts[both]).abs().max().item() <= 1e-4 * scale
    position = torch.tensor(meta["position"])
    assert (out["points"][:, :3].cpu() - (out["points_world"].cpu() - position)).abs().max().item() <= 1e-6 * scale
    assert torch.all(out["points"][:, 4] == 0)


def test_sweep_points_render_like_get_outputs_for_lidar():
    from neurad_studio_b200.nerfstudio_api import Lidars
    from neurad_studio_b200.scene import LidarScan

    model = _model()
    sensor = C.nonuniform_sensor(32, seed=5, azimuth_resolution_deg=1.0, revolution_time=0.1, sensor_idx=2)
    pose = C.pose_yaw(6.0, 0.5, 1.6, 0.2)
    vel = torch.tensor([9.0, 0.5, 0.0])
    out = model.get_outputs_for_lidar_sweep(sensor, pose[None], [1.0], vel[None], ray_drop_threshold=None, max_distance=1e3)
    m = out["points"].shape[0]
    assert m > 0
    scan = LidarScan(l2w=pose, points=out["points"].cpu(), time=1.0, velocity=vel, sensor_idx=2)
    lo, batch = model.get_outputs_for_lidar(Lidars([scan], DEV), {"lidar": out["points"], "lidar_idx": 0})
    # the measured-points route sees the kept rays again: same world points, same renders
    world = (pose[:, :3] @ out["points"][:, :3].cpu().T).T + pose[:, 3]
    assert (world - out["points_world"].cpu()).abs().max().item() <= 1e-5 * _scale(world)
    j = out["point_index"][:, 1].long() * out["depth_image"].shape[2] + out["point_index"][:, 2].long()
    assert C.rel_to_max(lo["depth"], out["depth"][j]) < 2e-4
    assert C.rel_to_max(lo["intensity"], out["intensity"][j]) < 1e-4
    assert C.rel_to_max(batch["distance"], out["depth"][j]) < 1e-5


def test_actor_edits_and_camopt_act_as_on_a_render_of_the_same_rays(backend):
    from neurad_studio_b200.config import CameraOptimizerConfig
    from neurad_studio_b200.nerfstudio_api import RayBundle

    meta, cfg, params, g = C.golden()
    adj = torch.tensor([[0.0] * 6, [0.05, -0.02, 0.01, 0.01, -0.02, 0.03], [0.1, 0.0, 0.0, 0.0, 0.0, 0.02]])
    model = _model({"camera_optimizer.pose_adjustment": adj}, camera_optimizer=CameraOptimizerConfig(mode="SO3xR3"),
                   num_cameras=3, use_camopt_in_eval=True)
    model.dynamic_actors.actor_editing.update({"lateral": 1.5, "rotation": 0.4})
    sensor = C.nonuniform_sensor(16, seed=6, azimuth_resolution_deg=2.0, sensor_idx=1)
    poses = torch.stack([C.pose_yaw(6.0, 0.5, 1.6, 0.0), C.pose_yaw(8.0, -0.5, 1.6, 0.1)])
    with pytest.raises(ValueError):
        model.get_outputs_for_lidar_sweep(sensor, poses, [1.0, 1.2])
    model.train()
    out = model.get_outputs_for_lidar_sweep(sensor, poses, [1.0, 1.2], camera_indices=[1, 2])
    assert model.training  # the caller's mode comes back
    model.eval()
    r = backend.raygen_lidar_sweeps(sensor, poses, [1.0, 1.2])
    per = r["origins"].shape[0] // 2
    ci = torch.tensor([1, 2], device=DEV).repeat_interleave(per)[:, None]
    rb = RayBundle(origins=r["origins"], directions=r["directions"], pixel_area=r["pixel_area"], times=r["times"],
                   camera_indices=ci, metadata={"is_lidar": r["is_lidar"], "sensor_idxs": r["sensor_idx"]})
    ref = model.get_outputs_for_camera_ray_bundle(rb)
    for k in ("depth", "intensity", "ray_drop_prob", "features"):
        assert torch.equal(out[k], ref[k]), k
    model.dynamic_actors.actor_editing.update({"lateral": 0.0, "rotation": 0.0})
    model.use_camopt_in_eval = False
    plain = model.get_outputs_for_lidar_sweep(sensor, poses, [1.0, 1.2])
    assert not torch.equal(plain["depth"], out["depth"])


def test_sweep_points_feed_chamfer_distance():
    from neurad_studio_b200 import chamfer_distance

    meta, cfg, params, g = C.golden()
    model = _model()
    out = model.get_outputs_for_lidar_sweep(C.viewer_sensor(meta), C.viewer_pose(meta), [meta["time"]], ray_drop_threshold=None,
                                            max_distance=1e3)
    pts = out["points"][:, :3]
    assert float(chamfer_distance(pts, pts)) == 0.0
    shifted = pts + torch.tensor([0.0, 0.0, 0.01], device=DEV)
    assert float(chamfer_distance(pts, shifted)) > 0.0


def test_sweep_waits_on_the_host_only_to_size_the_points(backend):
    """With a host description the sweep uploads its descriptors and tables without a host wait: ray generation, render
    and point epilogue run under torch's sync debug mode "error", and the whole API call synchronises once, to read the
    kept count."""
    import warnings

    from neurad_studio_b200.config import CameraOptimizerConfig

    adj = torch.tensor([[0.0] * 6, [0.05, -0.02, 0.01, 0.01, -0.02, 0.03]])
    model = _model({"camera_optimizer.pose_adjustment": adj}, camera_optimizer=CameraOptimizerConfig(mode="SO3xR3"),
                   num_cameras=2, use_camopt_in_eval=True)
    sensors = [C.nonuniform_sensor(16, seed=7, azimuth_resolution_deg=2.0, sensor_idx=1),
               C.nonuniform_sensor(16, seed=8, azimuth_resolution_deg=2.0, sensor_idx=3)]
    poses = torch.stack([C.pose_yaw(6.0, 0.5, 1.6, 0.0), C.pose_yaw(8.0, -0.5, 1.6, 0.1)])
    args = (sensors, poses, [1.0, 1.2], torch.tensor([[9.0, 0.0, 0.0], [9.0, 0.5, 0.0]]))
    model.get_outputs_for_lidar_sweep(*args, camera_indices=[0, 1])  # binds the parameters
    torch.cuda.synchronize()
    try:
        torch.cuda.set_sync_debug_mode("error")
        r = backend.raygen_lidar_sweeps(*args)
        o = backend.render(r, want_intensity=True)
        pts = backend.lidar_sweep_points(r, o["depth"], o["intensity"], o["ray_drop_logits"].sigmoid(), 0.5)
        torch.cuda.set_sync_debug_mode("warn")
        with warnings.catch_warnings(record=True) as caught:
            warnings.simplefilter("always")
            out = model.get_outputs_for_lidar_sweep(*args, camera_indices=[0, 1])
    finally:
        torch.cuda.set_sync_debug_mode("default")
    syncs = [w for w in caught if "synchroniz" in str(w.message)]
    assert len(syncs) == 1, [str(w.message) for w in syncs]
    assert out["points"].shape[0] == int(out["counts"].sum())
    assert int(pts["counts"][-1]) >= 0


def test_sensor_index_outside_the_model_is_rejected():
    from neurad_studio_b200.scene import LidarSensor

    meta, cfg, params, g = C.golden()
    model = _model()
    for idx in (-1, cfg.num_sensors):
        s = LidarSensor(elevations=torch.tensor([0.0, 0.1]), azimuth_resolution_deg=10.0, sensor_idx=idx)
        with pytest.raises(ValueError):
            model.get_outputs_for_lidar_sweep(s, C.viewer_pose(meta), [1.0])
