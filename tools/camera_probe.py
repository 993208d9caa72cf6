"""Device time of camera ray generation (raygen_camera_kernel) for the camera models the AD dataparsers build.

  python tools/camera_probe.py [--reps 200]

Prints the card's name, power limit and SM clock limit, then the median [min-max] CUDA-event device time of one call,
warmed, over --reps launches, of:
  pandaset_stride3    the six 1920 x 1080 PandaSet cameras at NeuRAD's render stride through B200Backend.raygen_pinhole
  zod_stride3         a ZOD-sized fisheye (3848 x 1418 after the hood crop, k1..k4 != 0) at stride 3 (607 k rays)
  zod_full            the same camera at full resolution (5.46 M rays)
  zod_torch_ref       a torch restatement, on the GPU, of what the reference does for that camera: Cameras.generate_rays at
                      full resolution (3 x 10 Newton steps of undistortion, fisheye mapping, rotation, normalisation, pixel
                      area, rolling shutter), then [1::3, 1::3] (neurad.py:641-646)
  zod_render_stride3  for context: the fused render of the zod_stride3 bundle with the default NeuRADConfig (random
                      parameters, no actors)
and the largest difference between zod_torch_ref's rays and the kernel's.
"""
import argparse
import math
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import neurad_studio_b200 as nsb  # noqa: E402
from neurad_studio_b200 import scene  # noqa: E402
from neurad_studio_b200.backend import B200Backend  # noqa: E402
from oracle import camera_oracle as CO  # noqa: E402

ZOD_K = torch.tensor([-0.031, 0.0047, -0.0012, 0.00021, 0.0, 0.0])


def zod_camera():
    base = scene.pandaset_rig(width=3848, height=1418)[0]
    return scene.PinholeCamera(c2w=base.c2w, fx=1680.0, fy=1680.0, cx=1923.7, cy=709.2, width=3848, height=1418, time=base.time,
                               velocity=base.velocity, rolling_shutter_time=0.032, time_to_center_pixel=-0.004,
                               camera_type="fisheye", distortion_params=ZOD_K)


def torch_reference_rays(cam, dev):
    """Cameras._generate_rays_from_coords for one fisheye camera, as the reference evaluates it (torch elementwise ops over
    the full-resolution grid), then the render stride."""
    ys, xs = torch.meshgrid(torch.arange(cam.height, device=dev), torch.arange(cam.width, device=dev), indexing="ij")
    y, x = ys.float() + 0.5, xs.float() + 0.5
    coord = torch.stack([(x - cam.cx) / cam.fx, (y - cam.cy) / cam.fy], -1)
    coord_x = torch.stack([(x - cam.cx + 1) / cam.fx, (y - cam.cy) / cam.fy], -1)
    coord_y = torch.stack([(x - cam.cx) / cam.fx, (y - cam.cy + 1) / cam.fy], -1)
    st = CO.undistort_radial_tangential(torch.stack([coord, coord_x, coord_y], 0), cam.distortion_params.to(dev))
    st[..., 1] *= -1
    theta = torch.clip(torch.sqrt(torch.sum(st**2, dim=-1)), 0.0, math.pi)
    s = torch.sin(theta)
    local = torch.stack([st[..., 0] * s / theta, st[..., 1] * s / theta, -torch.cos(theta)], -1)
    c2w = cam.c2w.to(dev)
    d = torch.sum(local[..., None, :] * c2w[:3, :3], dim=-1)
    d = d / torch.maximum(torch.linalg.vector_norm(d, dim=-1, keepdim=True), torch.tensor(8.881784197001252e-16, device=dev))
    dx = torch.sqrt(torch.sum((d[0] - d[1]) ** 2, dim=-1))
    dy = torch.sqrt(torch.sum((d[0] - d[2]) ** 2, dim=-1))
    toff = (y[..., None] / cam.height - 0.5) * cam.rolling_shutter_time + cam.time_to_center_pixel
    out = {"origins": c2w[:3, 3] + cam.velocity.to(dev) * toff, "directions": d[0], "pixel_area": (dx * dy)[..., None],
           "times": cam.time + toff}
    return {k: v[1::3, 1::3] for k, v in out.items()}


def timed(fn, reps):
    for _ in range(5):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        ts.append(e0.elapsed_time(e1))
    return np.array(ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("camera_probe needs a CUDA device")
    dev = torch.device("cuda", 0)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    print(f"device: {torch.cuda.get_device_name(dev)}; nvidia-smi: {q[0] if q else 'n/a'}")
    be = B200Backend(dev)
    rig = scene.pandaset_rig()
    zod = zod_camera()
    rays = {}

    def pandaset():
        for cam in rig:
            be.raygen_pinhole(cam, 1, 3, 1, 3)

    rows = {
        "pandaset_stride3": (6 * 640 * 360, pandaset),
        "zod_stride3": (473 * 1283, lambda: rays.__setitem__("zod", be.raygen_camera(zod, 1, 3, 1, 3))),
        "zod_full": (3848 * 1418, lambda: be.raygen_camera(zod)),
        "zod_torch_ref": (473 * 1283, lambda: rays.__setitem__("ref", torch_reference_rays(zod, dev))),
    }
    res = {}
    for name, (n, fn) in rows.items():
        res[name] = (n, timed(fn, a.reps if name != "zod_torch_ref" else max(a.reps // 10, 10)))
        torch.cuda.empty_cache()
    be.check_status()
    err = {k: (rays["zod"][k].view(473, 1283, -1) - rays["ref"][k]).abs().max().item() for k in ("origins", "directions", "pixel_area", "times")}

    cfg = nsb.NeuRADConfig(n_actors=0)
    be.load_params(cfg, scene.make_params(cfg, seed=1, beta=3.0, sdf_bias=0.6, device="cuda"))
    r = dict(rays["zod"])
    r.pop("shape")
    r["sensor_idx"] = torch.zeros(r["origins"].shape[0], 1, dtype=torch.long, device=dev)
    res["zod_render_stride3"] = (r["origins"].shape[0], timed(lambda: be.render(r, image_width=1283), max(a.reps // 20, 10)))
    be.check_status()

    for name, (n, ts) in res.items():
        print(f"  {name:20s} {n:9d} rays  {np.median(ts) * 1e3:10.1f} us  [{ts.min() * 1e3:.1f}-{ts.max() * 1e3:.1f}]"
              f"  {n / np.median(ts) / 1e6:8.2f} Grays/s" if "render" not in name else
              f"  {name:20s} {n:9d} rays  {np.median(ts) * 1e3:10.1f} us  [{ts.min() * 1e3:.1f}-{ts.max() * 1e3:.1f}]")
    print(f"  torch restatement vs kernel (stride 3): " + ", ".join(f"{k} {v:.2e}" for k, v in err.items()))
    print(f"  zod_torch_ref / zod_stride3 = {np.median(res['zod_torch_ref'][1]) / np.median(res['zod_stride3'][1]):.1f}x")


if __name__ == "__main__":
    main()
