"""CPU: fisheye and distorted camera rays and the horizontal rolling shutter (csrc/camera_rays.h).

- The oracle's restatement (oracle/camera_oracle.py:generate_rays_camera) reproduces tests/golden/camera_models.npz, the
  reference's own Cameras.generate_rays, bit for bit, NaNs included.
- The device functions of csrc/camera_rays.h, run on the host by tests/host_emul/emul_camera.cpp, meet the same goldens:
  origins and times bit for bit, directions within 1e-6 (torch's CPU vector_norm rounds differently from the kernel's
  sqrt((x^2 + y^2) + z^2); fisheye ones also go through sinf / cosf), pixel_area within 1e-4 of the case's max.
- A default scene.PinholeCamera still reproduces tests/golden/raygen.npz, and generate_rays_camera with its defaults is
  oracle.neurad_oracle.generate_rays_pinhole bit for bit.
- The mirror's Cameras and get_outputs_for_camera_ray_bundle render a fisheye and a horizontal-shutter camera over
  tests/camera_fake_backend.py.
"""
import ctypes
import dataclasses
import os
import subprocess

import pytest
import torch

from oracle import camera_oracle as CO
from oracle import neurad_oracle as O
from tests import camera_model_cases as C
from tests.helpers import load_golden

CASES = C.load()


def _coords(cam, row0=0, row_step=1, col0=0, col_step=1):
    ys, xs = torch.meshgrid(torch.arange(row0, cam.height, row_step), torch.arange(col0, cam.width, col_step), indexing="ij")
    return (torch.stack([ys, xs], -1) + 0.5).float()


def _oracle(cam, coords):
    return CO.generate_rays_camera(cam.c2w, cam.fx, cam.fy, cam.cx, cam.cy, cam.height, cam.width, coords, cam.time, cam.velocity,
                                   cam.rolling_shutter_time, cam.time_to_center_pixel, cam.camera_type, cam.distortion_params,
                                   cam.rs_direction)


def _bit_equal(a, b):
    return a.shape == b.shape and torch.equal(torch.isnan(a), torch.isnan(b)) and torch.equal(a.nan_to_num(), b.nan_to_num())


@pytest.mark.parametrize("name", list(CASES))
def test_oracle_matches_reference_golden_bit_for_bit(name):
    cam, ref = CASES[name]
    o = _oracle(cam, _coords(cam))
    for k in C.KEYS:
        assert _bit_equal(o[k], ref[k]), (name, k)


def test_golden_cases_cover_the_reference_findings():
    """The NaN of a principal point on a pixel centre: that pixel and its left / upper neighbours; nowhere else."""
    _, ref = CASES[C.NAN_CASE]
    nan = torch.isnan(ref["pixel_area"][..., 0])
    assert sorted(map(tuple, nan.nonzero().tolist())) == [(26, 48), (27, 47), (27, 48)]
    assert torch.isnan(ref["directions"]).any(-1).nonzero().tolist() == [[27, 48]]
    for name in CASES:
        if name != C.NAN_CASE:
            assert not any(torch.isnan(v).any() for v in CASES[name][1].values()), name
    # a horizontal shutter runs along the columns, and the reversed one negates time_to_center_pixel too
    cam, fwd = CASES["waymo_horizontal"]
    rcam, rev = CASES["waymo_reversed"]
    assert cam.time_to_center_pixel == 0.0 and rcam.time_to_center_pixel != 0.0
    t = fwd["times"][..., 0]
    assert torch.equal(t, t[:1].expand_as(t)) and (t[:, 1:] > t[:, :-1]).all()
    expect = -(fwd["times"] - cam.time) - rcam.time_to_center_pixel
    assert ((rev["times"] - rcam.time) - expect).abs().max().item() < 1e-6


# ---------------------------------------------------------------------------------------------- host emulation
@pytest.fixture(scope="module")
def emul_lib(tmp_path_factory):
    src = os.path.join(C.ROOT, "tests", "host_emul", "emul_camera.cpp")
    so = str(tmp_path_factory.mktemp("emul_camera") / "libemul_camera.so")
    subprocess.check_call(["g++", "-std=c++20", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-o", so, src])
    lib = ctypes.CDLL(so)
    lib.emul_raygen_camera.restype = ctypes.c_int
    return lib


def emul_rays(lib, cam, row0=0, row_step=1, col0=0, col_step=1):
    from neurad_studio_b200 import lib as L

    n_rows, n_cols = len(range(row0, cam.height, row_step)), len(range(col0, cam.width, col_step))
    dist = torch.zeros(6) if cam.distortion_params is None else cam.distortion_params.float()
    vel = torch.zeros(3) if cam.velocity is None else cam.velocity.float()
    f = cam.c2w.reshape(-1).float().tolist() + [cam.fx, cam.fy, cam.cx, cam.cy] + dist.tolist() + [cam.time] + vel.tolist() + \
        [cam.rolling_shutter_time, cam.time_to_center_pixel]
    iv = [cam.height, cam.width, row0, row_step, n_rows, col0, col_step, n_cols, int(cam.velocity is not None),
          L.RS_DIRECTIONS[cam.rs_direction], L.CAMERA_TYPES[cam.camera_type]]
    n = n_rows * n_cols
    out = {"origins": torch.zeros(n, 3), "directions": torch.zeros(n, 3), "pixel_area": torch.zeros(n, 1), "times": torch.zeros(n, 1)}
    rc = lib.emul_raygen_camera((ctypes.c_float * len(f))(*f), (ctypes.c_int * len(iv))(*iv),
                                *[ctypes.c_void_p(out[k].data_ptr()) for k in C.KEYS])
    assert rc == 0
    return {k: v.view(n_rows, n_cols, -1) for k, v in out.items()}


@pytest.mark.parametrize("name", list(CASES))
def test_host_emulation_matches_reference_golden(emul_lib, name):
    cam, ref = CASES[name]
    got = emul_rays(emul_lib, cam)
    errs = C.errors(cam, got, ref)
    print(name, {k: f"{e:.2e} (tol {t:.2e})" for k, (e, t) in errs.items()})
    # origins and times are the reference's bits; so are the coordinates the directions are made of (the undistortion
    # included), but torch's CPU vector_norm does not round like sqrt((x^2 + y^2) + z^2), so a direction may differ from
    # the reference's in the last bit -- as the pinhole kernel's always have (test_raygen_matches_reference_golden)
    for k in ("origins", "times"):
        assert _bit_equal(got[k], ref[k]), (name, k)
    assert errs["directions"][0] <= 1e-6, (name, errs["directions"])
    assert errs["pixel_area"][0] <= errs["pixel_area"][1], (name, errs["pixel_area"])


def test_host_emulation_default_camera_matches_raygen_golden(emul_lib):
    """The undistorted perspective instance is the pinhole kernel's arithmetic, held to the raygen golden as the GPU test
    holds the kernel."""
    for cam, ref in _raygen_golden():
        got = emul_rays(emul_lib, cam)
        errs = C.errors(cam, got, {k: v.reshape(got[k].shape) for k, v in ref.items()})
        for k in ("origins", "times"):
            assert torch.equal(got[k].reshape(ref[k].shape), ref[k]), k
        assert errs["directions"][0] <= 1e-6 and errs["pixel_area"][0] <= errs["pixel_area"][1], errs


def _raygen_golden():
    from neurad_studio_b200 import scene

    _, g = load_golden("raygen.npz")
    for key in ("cam0", "cam3"):
        c = g[key]
        h, w = (int(v) for v in c["hw"])
        fx, fy, cx, cy = (float(v) for v in c["intr"])
        cam = scene.PinholeCamera(c2w=c["c2w"], fx=fx, fy=fy, cx=cx, cy=cy, width=w, height=h, time=float(c["time"]),
                                  velocity=c["velocity"], rolling_shutter_time=float(c["rs"][0]),
                                  time_to_center_pixel=float(c["rs"][1]))
        yield cam, {k: c[k] for k in C.KEYS}


def test_default_pinhole_camera_reproduces_raygen_golden():
    from tests.camera_fake_backend import CameraFakeBackend

    be = CameraFakeBackend()
    for cam, ref in _raygen_golden():
        assert (cam.camera_type, cam.distortion_params, cam.rs_direction) == ("perspective", None, "Vertical")
        o = _oracle(cam, _coords(cam))
        p = O.generate_rays_pinhole(cam.c2w, cam.fx, cam.fy, cam.cx, cam.cy, cam.height, cam.width, _coords(cam), cam.time,
                                    cam.velocity, cam.rolling_shutter_time, cam.time_to_center_pixel)
        r = be.raygen_camera(cam)
        for k in ("origins", "directions", "pixel_area", "times", "directions_norm"):
            assert torch.equal(o[k], p[k]), k
        for k in C.KEYS:
            assert torch.equal(o[k].reshape(ref[k].shape), ref[k]), k
            assert torch.equal(r[k].reshape(ref[k].shape), ref[k]), k


# ---------------------------------------------------------------------------------------------- validation and the mirror
def test_invalid_descriptors_raise_value_error():
    from neurad_studio_b200.backend import camera_descriptor, is_pinhole_camera
    from tests.camera_fake_backend import CameraFakeBackend

    cam = CASES["zod_fisheye"][0]
    for bad in (dict(camera_type="equirectangular"), dict(camera_type="FISHEYE"), dict(rs_direction="horizontal"),
                dict(rs_direction="Vertical_reversed"), dict(distortion_params=torch.zeros(4)),
                dict(distortion_params=torch.zeros(8))):
        c = dataclasses.replace(cam, **bad)
        with pytest.raises(ValueError):
            camera_descriptor(c)
        with pytest.raises(ValueError):
            CameraFakeBackend().raygen_camera(c)
    d = camera_descriptor(cam)
    assert (d.camera_type, d.rs_direction, d.has_velocity) == (1, 0, 1)
    plain = dataclasses.replace(cam, camera_type="perspective", distortion_params=None)
    assert is_pinhole_camera(plain) and is_pinhole_camera(dataclasses.replace(plain, distortion_params=torch.zeros(6)))
    for other in (cam, dataclasses.replace(plain, rs_direction="Horizontal"),
                  dataclasses.replace(plain, distortion_params=torch.tensor([0.0, 0.0, 0.0, 0.0, 1e-3, 0.0]))):
        assert not is_pinhole_camera(other)
    assert list(d.distortion) == pytest.approx(cam.distortion_params.tolist())
    d = camera_descriptor(dataclasses.replace(cam, camera_type="perspective", distortion_params=None, velocity=None,
                                              rs_direction="Horizontal_reversed"))
    assert (d.camera_type, d.rs_direction, d.has_velocity, list(d.distortion)) == (0, 2, 0, [0.0] * 6)


@pytest.fixture()
def mirror(monkeypatch):
    import neurad_studio_b200 as nsb
    from neurad_studio_b200 import nerfstudio_api, scene
    from tests.camera_fake_backend import CameraFakeBackend

    be = CameraFakeBackend()
    monkeypatch.setattr(nerfstudio_api, "get_backend", lambda device: be)
    cfg = nsb.small_config(n_actors=0, log2_main=10, log2_prop=10)
    params = scene.make_params(cfg, seed=21, beta=3.0, sdf_bias=0.5)
    dec = scene.make_rgb_decoder_params(seed=22)
    model = nerfstudio_api.NeuRADModel(cfg)
    model.load_reference_state_dict(params)
    model.rgb_decoder.load_state_dict({k[len("rgb_decoder."):]: v for k, v in dec.items()}, strict=False)
    return model.eval(), cfg, params, dec


@pytest.mark.parametrize("name", ["zod_fisheye", "waymo_reversed"])
def test_mirror_renders_fisheye_and_horizontal_cameras(mirror, name):
    from oracle import decoder_oracle as D
    from oracle.convert import to_oracle_cfg

    from neurad_studio_b200.nerfstudio_api import Cameras

    model, cfg, params, dec = mirror
    cam = dataclasses.replace(CASES[name][0], width=24, height=15, cx=CASES[name][0].cx / 4, cy=CASES[name][0].cy / 3.6,
                              fx=CASES[name][0].fx / 4, fy=CASES[name][0].fy / 3.6)
    rb = Cameras([cam], "cpu").generate_rays(camera_indices=0, keep_shape=True)
    assert rb.shape == (15, 24)
    full = _oracle(cam, _coords(cam))
    for k in C.KEYS:
        assert torch.equal(getattr(rb, k), full[k]), k
    out = model.get_outputs_for_camera_ray_bundle(rb)
    assert out["rgb"].shape == (15, 24, 3) and out["features"].shape[:2] == (5, 8)
    sub = _oracle(cam, _coords(cam, 1, 3, 1, 3).reshape(-1, 2))
    with torch.no_grad():
        ref = O.nff_outputs(params, to_oracle_cfg(cfg), sub["origins"], sub["directions"], sub["pixel_area"], sub["times"],
                            torch.full((40, 1), cam.sensor_idx), None)
        rgb_ref = D.rgb_decoder(dec, ref["features"].view(1, 5, 8, -1))[0]
    assert torch.equal(out["depth"].reshape(-1), ref["depth"].reshape(-1))
    assert (out["rgb"] - rgb_ref).abs().max().item() < 1e-5
