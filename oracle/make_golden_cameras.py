"""TEST INFRASTRUCTURE ONLY -- tests/golden/camera_models.npz from the REAL reference's `Cameras.generate_rays`.

Run in the build container (needs /root/reference):   python -m oracle.make_golden_cameras

Six small (96 x 54) cameras of the kinds the AD dataparsers build besides the undistorted perspective one:
  zod_fisheye          ZOD-like FISHEYE: k1..k4 small, p = 0, corners about 60 degrees off axis, vertical shutter
  zod_fisheye_centred  the same with the principal point on a pixel centre: theta = 0 there -> NaN (0 * 0 / 0)
  fisheye_extreme      strong negative k1 and a short focal length: Newton steps with |det| <= 1e-3 and theta > pi clipped
  perspective_distorted  PERSPECTIVE with k1..k4 and p1, p2 != 0
  waymo_horizontal     PERSPECTIVE, metadata["rs_direction"] = "Horizontal", time_to_center_pixel = 0
  waymo_reversed       "Horizontal_reversed" with time_to_center_pixel != 0 (the reversal negates it too)
For each it asserts that oracle.camera_oracle.generate_rays_camera reproduces the reference bit for bit (NaNs in the same
places) before writing the file.
"""
from __future__ import annotations

import dataclasses
import math
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from neurad_studio_b200 import scene  # noqa: E402
from oracle import camera_oracle as CO  # noqa: E402
from oracle import ref_driver  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")
W, H = 96, 54
KEYS = ("origins", "directions", "pixel_area", "times")


def cases():
    base = scene.pandaset_rig(time=2.3, width=W, height=H)
    zod_k = torch.tensor([-0.031, 0.0047, -0.0012, 0.00021, 0.0, 0.0])
    zod = dataclasses.replace(base[0], fx=52.0, fy=51.6, cx=48.27, cy=27.16, camera_type="fisheye", distortion_params=zod_k,
                              rolling_shutter_time=0.032, time_to_center_pixel=-0.004)
    wod = dataclasses.replace(base[1], fx=80.0, fy=80.0, cx=47.6, cy=26.9, rolling_shutter_time=0.024,
                              time_to_center_pixel=0.0, rs_direction="Horizontal")
    return {
        "zod_fisheye": zod,
        "zod_fisheye_centred": dataclasses.replace(zod, cx=48.5, cy=27.5),
        "fisheye_extreme": dataclasses.replace(base[2], fx=17.0, fy=17.5, cx=47.3, cy=27.4, camera_type="fisheye",
                                               distortion_params=torch.tensor([-0.55, 0.04, 0.0, 0.0, 0.0, 0.0])),
        "perspective_distorted": dataclasses.replace(
            base[3], fx=70.0, fy=71.0, cx=48.9, cy=26.3,
            distortion_params=torch.tensor([-0.12, 0.031, -0.0024, 0.0003, 0.0011, -0.0016])),
        "waymo_horizontal": wod,
        "waymo_reversed": dataclasses.replace(wod, rs_direction="Horizontal_reversed", time_to_center_pixel=-0.0075),
    }


def reference_rays(cam):
    from nerfstudio.cameras.cameras import Cameras, CameraType

    md = {"rolling_shutter_time": torch.tensor([[cam.rolling_shutter_time]]),
          "time_to_center_pixel": torch.tensor([[cam.time_to_center_pixel]]), "velocities": cam.velocity[None]}
    if cam.rs_direction != "Vertical":
        md["rs_direction"] = cam.rs_direction
    rc = Cameras(
        camera_to_worlds=cam.c2w[None], fx=cam.fx, fy=cam.fy, cx=cam.cx, cy=cam.cy, width=cam.width, height=cam.height,
        distortion_params=None if cam.distortion_params is None else cam.distortion_params[None],
        camera_type=CameraType.FISHEYE if cam.camera_type == "fisheye" else CameraType.PERSPECTIVE,
        times=torch.tensor([cam.time]), metadata=md,
    )
    return rc.generate_rays(camera_indices=0, keep_shape=True), rc.get_image_coords()


def oracle_rays(cam, coords, **kw):
    return CO.generate_rays_camera(cam.c2w, cam.fx, cam.fy, cam.cx, cam.cy, cam.height, cam.width, coords, cam.time,
                                   cam.velocity, cam.rolling_shutter_time, cam.time_to_center_pixel, cam.camera_type,
                                   cam.distortion_params, cam.rs_direction, **kw)


def same(a, b):
    return a.shape == b.shape and torch.equal(torch.isnan(a), torch.isnan(b)) and torch.equal(a.nan_to_num(), b.nan_to_num())


def main():
    ref_driver.ref_import.install()
    arrays = {}
    for name, cam in cases().items():
        rb, coords = reference_rays(cam)
        o = oracle_rays(cam, coords)
        for k in KEYS:
            assert same(getattr(rb, k), o[k]), f"{name}: oracle != reference for {k}"
        n_nan = int(torch.isnan(rb.pixel_area).sum())
        note = f"NaN pixel_area at {n_nan} pixels"
        if cam.camera_type == "fisheye":
            k = cam.distortion_params
            st = torch.stack([torch.stack([(coords[..., 1] - cam.cx) / cam.fx, (coords[..., 0] - cam.cy) / cam.fy], -1)])
            und = CO.undistort_radial_tangential(st, k)
            theta = und.norm(dim=-1)
            loose = CO.undistort_radial_tangential(st, k, eps=0.0)
            n_eps = int((~(und == loose).all(-1)).sum())
            note += f"; theta > pi at {int((theta > math.pi).sum())} pixels; |det| <= 1e-3 changes {n_eps} pixels"
        print(f"{name}: oracle == reference bit for bit; {note}")
        arrays[f"{name}/c2w"] = cam.c2w
        arrays[f"{name}/intr"] = torch.tensor([cam.fx, cam.fy, cam.cx, cam.cy])
        arrays[f"{name}/hw"] = torch.tensor([cam.height, cam.width])
        arrays[f"{name}/time"] = torch.tensor(cam.time)
        arrays[f"{name}/velocity"] = cam.velocity
        arrays[f"{name}/rs"] = torch.tensor([cam.rolling_shutter_time, cam.time_to_center_pixel])
        arrays[f"{name}/distortion"] = cam.distortion_params if cam.distortion_params is not None else torch.zeros(6)
        arrays[f"{name}/camera_type"] = np.array(cam.camera_type)
        arrays[f"{name}/rs_direction"] = np.array(cam.rs_direction)
        for k in KEYS:
            arrays[f"{name}/{k}"] = getattr(rb, k)
    out = {k: (v.detach().cpu().numpy() if isinstance(v, torch.Tensor) else np.asarray(v)) for k, v in arrays.items()}
    out["__meta__"] = np.array(repr(dict(torch=torch.__version__, cases=list(cases()))))
    path = os.path.join(GOLDEN, "camera_models.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path}: {os.path.getsize(path) / 1e6:.2f} MB")


if __name__ == "__main__":
    main()
