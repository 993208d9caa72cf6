"""GPU: fisheye and distorted camera rays and the horizontal rolling shutter of raygen_camera_kernel (csrc/camera_rays.h).

- B200Backend.raygen_camera against every case of tests/golden/camera_models.npz (the reference's own
  Cameras.generate_rays): origins, directions and times within 1e-6 * max(1, max |ref|), pixel_area within 1e-4 of the
  case's max, NaNs in the same places.  The worst error of each case is printed.
- The strided grid NeuRAD renders is the same slice of the full-resolution call, bit for bit.
- b200nerf_raygen_pinhole and raygen_camera with a default descriptor give the same bits on the six PandaSet cameras.
- A ZOD-sized fisheye (3848 x 1418, stride 3) gives finite unit directions, deterministically, and renders to rgb at 3x
  the ray grid; a small fisheye render matches the oracle's nff_outputs on the oracle's rays.
"""
import ctypes
import dataclasses

import pytest
import torch

from neurad_studio_b200 import scene
from oracle import camera_oracle as CO
from oracle import neurad_oracle as NO
from tests import camera_model_cases as C
from tests.helpers import cfg_from_meta, load_golden

pytestmark = pytest.mark.gpu

CASES = C.load()
ZOD = dataclasses.replace(CASES["zod_fisheye"][0], width=3848, height=1418, fx=1680.0, fy=1680.0, cx=1923.7, cy=709.2)


@pytest.fixture(scope="module")
def backend():
    from neurad_studio_b200.backend import B200Backend

    return B200Backend(torch.device("cuda", 0))


def _grid(r):
    h, w = r["shape"]
    return {k: r[k].view(h, w, -1) for k in C.KEYS}


@pytest.mark.parametrize("name", list(CASES))
def test_raygen_camera_matches_reference_golden(backend, name):
    cam, ref = CASES[name]
    r = backend.raygen_camera(cam)
    backend.check_status()
    errs = C.errors(cam, _grid(r), ref)
    print(f"{name}: " + ", ".join(f"{k} {e:.2e} (tol {t:.2e})" for k, (e, t) in errs.items()))
    for k, (e, t) in errs.items():
        assert e <= t, (name, k, e, t)


@pytest.mark.parametrize("name", ["zod_fisheye", "perspective_distorted", "waymo_reversed"])
def test_strided_grid_is_the_slice_of_the_full_grid(backend, name):
    cam = CASES[name][0]
    full = _grid(backend.raygen_camera(cam))
    sub = _grid(backend.raygen_camera(cam, row0=1, row_step=3, col0=1, col_step=3))
    for k in C.KEYS:
        assert torch.equal(sub[k], full[k][1::3, 1::3].contiguous()), (name, k)


def test_pinhole_entry_point_equals_default_camera(backend):
    """The C ABI's b200nerf_raygen_pinhole is raygen_camera with a perspective, undistorted, vertical descriptor."""
    for cam in scene.pandaset_rig():
        assert (cam.camera_type, cam.distortion_params, cam.rs_direction) == ("perspective", None, "Vertical")
        r = backend.raygen_camera(cam, 1, 3, 1, 3)
        n = r["origins"].shape[0]
        o, d, a, t = (torch.empty(n, w, device="cuda") for w in (3, 3, 1, 1))
        c2w = (ctypes.c_float * 12)(*cam.c2w.reshape(-1).tolist())
        vel = (ctypes.c_float * 3)(*cam.velocity.tolist())
        n_rows, n_cols = r["shape"]
        ptr = lambda x: ctypes.c_void_p(x.data_ptr())  # noqa: E731
        backend._check(backend.lib.b200nerf_raygen_pinhole(
            backend._h, c2w, cam.fx, cam.fy, cam.cx, cam.cy, cam.height, cam.width, 1, 3, n_rows, 1, 3, n_cols, cam.time, vel,
            cam.rolling_shutter_time, cam.time_to_center_pixel, ptr(o), ptr(d), ptr(a), ptr(t), backend._stream))
        torch.cuda.synchronize()
        for k, v in zip(C.KEYS, (o, d, a, t)):
            assert torch.equal(v, r[k]), (cam.sensor_idx, k)


def test_zod_sized_fisheye(backend):
    r = backend.raygen_camera(ZOD, 1, 3, 1, 3)
    assert r["shape"] == (473, 1283) and r["origins"].shape[0] == 473 * 1283
    d = r["directions"]
    assert torch.isfinite(d).all() and torch.isfinite(r["pixel_area"]).all() and torch.isfinite(r["times"]).all()
    assert (d.norm(dim=-1) - 1).abs().max().item() < 1e-6
    r2 = backend.raygen_camera(ZOD, 1, 3, 1, 3)
    for k in C.KEYS:
        assert torch.equal(r[k], r2[k]), k


def _model():
    from neurad_studio_b200.nerfstudio_api import NeuRADModel
    from oracle import decoder_oracle as D

    meta, g = load_golden("nff_static.npz")
    cfg = cfg_from_meta(meta)
    sd = dict(g["param"])
    sd.update(D.random_decoder_params(seed=31))
    model = NeuRADModel(cfg)
    model.load_reference_state_dict(sd)
    return model.cuda().eval(), cfg, g["param"]


def test_zod_sized_fisheye_renders_through_the_mirror():
    from neurad_studio_b200.nerfstudio_api import Cameras

    model, _, _ = _model()
    rb = Cameras([ZOD], "cuda").generate_rays(camera_indices=0, keep_shape=True)
    assert rb.shape == (1418, 3848)
    with torch.no_grad():
        out = model.get_outputs_for_camera_ray_bundle(rb)
    assert out["depth"].shape == (473, 1283, 1) and out["rgb"].shape == (3 * 473, 3 * 1283, 3)
    assert torch.isfinite(out["rgb"]).all() and torch.isfinite(out["depth"]).all()


@pytest.mark.parametrize("name", ["zod_fisheye", "waymo_reversed"])
def test_small_camera_render_matches_oracle(name):
    from neurad_studio_b200.nerfstudio_api import Cameras
    from oracle.convert import to_oracle_cfg

    model, cfg, params = _model()
    cam = CASES[name][0]
    rb = Cameras([cam], "cuda").generate_rays(camera_indices=0, keep_shape=True)
    with torch.no_grad():
        out = model.get_outputs_for_camera_ray_bundle(rb)
    ys, xs = torch.meshgrid(torch.arange(1, cam.height, 3), torch.arange(1, cam.width, 3), indexing="ij")
    coords = (torch.stack([ys, xs], -1).reshape(-1, 2) + 0.5).float()
    r = CO.generate_rays_camera(cam.c2w, cam.fx, cam.fy, cam.cx, cam.cy, cam.height, cam.width, coords, cam.time, cam.velocity,
                                cam.rolling_shutter_time, cam.time_to_center_pixel, cam.camera_type, cam.distortion_params,
                                cam.rs_direction)
    n = coords.shape[0]
    with torch.no_grad():
        ref = NO.nff_outputs(params, to_oracle_cfg(cfg), r["origins"], r["directions"], r["pixel_area"], r["times"],
                            torch.full((n, 1), cam.sensor_idx), None)
    for k, tol in (("features", 1e-4), ("accumulation", 1e-4), ("depth", 2e-4)):
        a, b = out[k].cpu().reshape(n, -1), ref[k].reshape(n, -1)
        err = (a - b).abs().max().item() / (b.abs().max().item() + 1e-30)
        print(f"{name} {k}: max err / max|ref| = {err:.2e}")
        assert err < tol, (name, k, err)
