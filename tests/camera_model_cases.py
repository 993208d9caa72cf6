"""Shared by tests/test_camera_models_cpu.py and tests/test_zz_camera_models_gpu.py: the cases of
tests/golden/camera_models.npz (written by oracle/make_golden_cameras.py from the reference's own Cameras.generate_rays) as
scene.PinholeCamera descriptors, and the comparison the kernel and its host emulation are held to."""
import ast
import os

import numpy as np
import torch

from neurad_studio_b200 import scene

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KEYS = ("origins", "directions", "pixel_area", "times")
# only ray generation is specified for the principal point on a pixel centre (its NaN rays are not rendered)
NAN_CASE = "zod_fisheye_centred"


def load():
    """{case: (PinholeCamera, {key: reference tensor [H, W, C]})}"""
    z = np.load(os.path.join(ROOT, "tests", "golden", "camera_models.npz"), allow_pickle=False)
    meta = ast.literal_eval(str(z["__meta__"]))
    out = {}
    for name in meta["cases"]:
        g = lambda k: z[f"{name}/{k}"]  # noqa: E731
        fx, fy, cx, cy = (float(v) for v in g("intr"))
        h, w = (int(v) for v in g("hw"))
        rs, ttc = (float(v) for v in g("rs"))
        cam = scene.PinholeCamera(
            c2w=torch.from_numpy(g("c2w")), fx=fx, fy=fy, cx=cx, cy=cy, width=w, height=h, time=float(g("time")),
            velocity=torch.from_numpy(g("velocity")), rolling_shutter_time=rs, time_to_center_pixel=ttc,
            camera_type=str(g("camera_type")), distortion_params=torch.from_numpy(g("distortion")),
            rs_direction=str(g("rs_direction")))
        out[name] = (cam, {k: torch.from_numpy(g(k)) for k in KEYS})
    return out


def errors(cam, got, ref):
    """Worst error of each output against the reference, with NaNs required in the same places:
    {key: (error, tolerance)}.  Origins, directions and times: max |a - b| against 1e-6 * max(1, max |ref|) (perspective
    directions are the reference's bits; fisheye ones go through sinf / cosf, which may differ from torch's in the last
    bit); pixel_area: max |a - b| against 1e-4 of the case's largest area."""
    res = {}
    for k in KEYS:
        a, b = got[k].detach().cpu().reshape(-1).float(), ref[k].reshape(-1).float()
        nan_a, nan_b = torch.isnan(a), torch.isnan(b)
        assert torch.equal(nan_a, nan_b), (k, int(nan_a.sum()), int(nan_b.sum()))
        fin = ~nan_b
        err = (a[fin] - b[fin]).abs().max().item() if fin.any() else 0.0
        scale = b[fin].abs().max().item() if fin.any() else 0.0
        tol = 1e-4 * scale if k == "pixel_area" else 1e-6 * max(1.0, scale)
        res[k] = (err, tol)
    return res
