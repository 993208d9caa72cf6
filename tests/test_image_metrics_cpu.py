"""CPU: the camera image metrics (PSNR / SSIM) of NeuRADModel.get_image_metrics_and_images.

- The float64 oracle (oracle/image_metrics_oracle.py) reproduces tests/golden/image_metrics.npz over both of its routes:
  torchmetrics' literal reflect-pad / filter / crop order and the valid-window filter the kernels implement.
- The device functions of csrc/image_metrics.cuh, run by the host emulation (tests/host_emul/emul_image_metrics.cpp),
  meet the golden values at the tolerances of tests/image_metric_cases.py.
- The mirror's camera branch over a CPU stand-in backend defined here.

The SSIM definition is from memory, unpinned against torchmetrics; tests/test_zz_image_metrics_gpu.py holds the one
comparison with the package, which runs only where it is installed.
"""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

from oracle import image_metrics_oracle as IM
from tests import image_metric_cases as C
from tests.test_lidar_metrics_cpu import ChamferFakeBackend, _case as lidar_case

ROOT = C.ROOT


@pytest.fixture(scope="module")
def golden():
    return C.load_golden()


# ---------------------------------------------------------------------------------------------- oracle vs golden
def test_golden_inputs_are_the_oracles_seeded_cases(golden):
    cases = IM.cases()
    assert sorted(cases) == sorted(C.NAMES)
    for name, (a, b, data_range) in cases.items():
        assert np.array_equal(golden[f"{name}_a"], a, equal_nan=True), name
        assert np.array_equal(golden[f"{name}_b"], b, equal_nan=True), name
        assert float(golden[f"{name}_data_range"]) == data_range


@pytest.mark.parametrize("name", C.NAMES)
def test_both_oracle_routes_match_golden(golden, name):
    """The padded route never lets a padded pixel into a kept window: it equals the valid-window route."""
    a, b, data_range, want = C.case(golden, name)
    for padded in (False, True):
        got = IM.metrics_f64(a.numpy(), b.numpy(), data_range, padded=padded)
        np.testing.assert_allclose(got, want, rtol=0, atol=1e-12, equal_nan=True)


def test_fixture_covers_the_edge_values(golden):
    assert golden["identical_out"][0, 2] == 1.0 and golden["identical_out"][0, 1] == np.inf
    # two flat images: the luminance term alone, but for the 1e-7 by which the fp32-normalised window misses a sum of 1
    assert golden["constant_out"][0, 2] == pytest.approx((2 * 0.125 + 1e-4) / (0.3125 + 1e-4), abs=1e-5)
    assert golden["one_window_a"].shape == (1, 11, 11, 3)
    assert golden["outside_unit_a"].min() < -1 and golden["outside_unit_a"].max() > 2
    assert np.isnan(golden["nan_out"]).all()


# ---------------------------------------------------------------------------------------------- host emulation
@pytest.fixture(scope="module")
def emul_lib(tmp_path_factory):
    src = os.path.join(ROOT, "tests", "host_emul", "emul_image_metrics.cpp")
    so = str(tmp_path_factory.mktemp("emul_image_metrics") / "libemul_image_metrics.so")
    subprocess.check_call(["g++", "-std=c++20", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-o", so, src])
    lib = ctypes.CDLL(so)
    lib.emul_image_metrics.restype = ctypes.c_int
    lib.emul_image_metrics.argtypes = [ctypes.c_void_p, ctypes.c_void_p] + [ctypes.c_int] * 4 + \
        [ctypes.POINTER(ctypes.c_int64)] * 2 + [ctypes.c_float, ctypes.c_void_p]
    return lib


def emul(lib, a, b, data_range=None):
    """a, b [B, C, H, W] fp32 tensors with any strides, as B200Backend.image_metrics takes them."""
    n, ch, h, w = a.shape
    out = torch.empty(n + 1, 4, dtype=torch.float64)
    strides = [(ctypes.c_int64 * 4)(t.stride(0), t.stride(2), t.stride(3), t.stride(1)) for t in (a, b)]
    rc = lib.emul_image_metrics(a.data_ptr(), b.data_ptr(), n, h, w, ch, strides[0], strides[1],
                                0.0 if data_range is None else data_range, out.data_ptr())
    assert rc == 0
    return out


def test_window_taps_are_torchs_fp32_gaussian(emul_lib):
    taps = np.empty(11, np.float32)
    emul_lib.emul_ssim_taps.argtypes = [ctypes.c_void_p]
    emul_lib.emul_ssim_taps(taps.ctypes.data)
    assert np.array_equal(taps, IM.window_f32())
    assert np.float32(taps.sum(dtype=np.float32)) == pytest.approx(1.0, abs=2e-7)


@pytest.mark.parametrize("name", C.NAMES)
def test_emulated_kernels_against_float64(golden, emul_lib, name):
    a, b, data_range, want = C.case(golden, name)
    got = emul(emul_lib, C.nchw(a), C.nchw(b), data_range).numpy()
    C.check_table(got, want, a, b, data_range, name)
    if name == "identical":
        assert (got[:, 2] == 1.0).all()


def test_emulated_layouts_give_the_same_bits(golden, emul_lib):
    """[B, C, H, W] views of channels-last memory are the channels-last images themselves; contiguous NCHW copies (same
    SSIM bits; the squared error is summed in another fp64 order) and a slice of a wider pixel are read in place too."""
    a, b, _, want = C.case(golden, "batch2")
    base = emul(emul_lib, C.nchw(a), C.nchw(b))
    moved = emul(emul_lib, torch.moveaxis(a[1], -1, 0)[None], torch.moveaxis(b[1], -1, 0)[None])
    one = emul(emul_lib, C.nchw(a[1:].clone()), C.nchw(b[1:].clone()))
    assert torch.equal(moved, one) and torch.equal(moved[0, :2], base[2, :2])
    planar = emul(emul_lib, C.nchw(a).contiguous(), C.nchw(b))
    assert torch.equal(planar[:, 2:], base[:, 2:])
    assert torch.allclose(planar[:, :2], base[:, :2], rtol=1e-13, atol=0)
    rgba = torch.cat([a, torch.full_like(a[..., :1], 7.0)], -1)
    sliced = emul(emul_lib, C.nchw(rgba[..., :3]), C.nchw(b))
    assert rgba[..., :3].stride(2) == 4 and torch.equal(sliced[:, 2:], base[:, 2:])
    C.check_table(sliced.numpy(), want, a, b, None, "batch2")


def test_emulation_rejects_small_images(emul_lib):
    x = torch.zeros(1, 3, 10, 40)
    out = torch.empty(2, 4, dtype=torch.float64)
    s = (ctypes.c_int64 * 4)(x.stride(0), x.stride(2), x.stride(3), x.stride(1))
    assert emul_lib.emul_image_metrics(x.data_ptr(), x.data_ptr(), 1, 10, 40, 3, s, s, 0.0, out.data_ptr()) == -1


# ---------------------------------------------------------------------------------------------- the mirror's logic
class ImageMetricsFakeBackend(ChamferFakeBackend):
    """TEST SCAFFOLDING ONLY: B200Backend.image_metrics' contract on the CPU, run by the host emulation."""

    def __init__(self, lib):
        super().__init__()
        self.lib, self.image_calls = lib, []

    def image_metrics(self, a, b, data_range=None):
        self.image_calls.append((tuple(a.shape), a.stride(), b.stride()))
        return emul(self.lib, a.float(), b.float(), data_range)


@pytest.fixture()
def mirror(monkeypatch, emul_lib):
    import neurad_studio_b200 as nsb
    from neurad_studio_b200 import nerfstudio_api

    be = ImageMetricsFakeBackend(emul_lib)
    monkeypatch.setattr(nerfstudio_api, "get_backend", lambda device: be)
    return nerfstudio_api.NeuRADModel(nsb.small_config(ray_drop_loss_mult=0.0)), be


def _camera(golden):
    a, b, _, want = C.case(golden, "smooth")
    return {"rgb": b[0]}, {"image": a[0]}, want


def test_mirror_camera_metrics(golden, mirror):
    from neurad_studio_b200 import metrics as M

    model, be = mirror
    outputs, batch, want = _camera(golden)
    lpips_calls = []

    def lpips(image, rgb):
        lpips_calls.append((tuple(image.shape), tuple(rgb.shape)))
        return torch.tensor(0.25)

    model.lpips = lpips
    metrics, images = model.get_image_metrics_and_images(outputs, batch)
    assert list(metrics) == ["psnr", "ssim", "lpips"] and all(isinstance(v, float) for v in metrics.values())
    assert list(images) == ["img"]
    h, w, _ = batch["image"].shape
    assert images["img"].shape == (h, 2 * w, 3)
    assert torch.equal(images["img"][:, :w], batch["image"]) and torch.equal(images["img"][:, w:], outputs["rgb"])
    assert metrics["ssim"] == pytest.approx(want[0, 2], abs=C.SSIM_ATOL)
    assert metrics["psnr"] == pytest.approx(want[0, 1], abs=C.PSNR_ATOL_DB)
    assert metrics["lpips"] == 0.25 and lpips_calls == [((1, 3, h, w), (1, 3, h, w))]
    # one backend call, on [1, C, H, W] views of the channels-last images (no copy)
    (shape, sa, sb), = be.image_calls
    assert shape == (1, 3, h, w) and sa[1:] == sb[1:] == (1, 3 * w, 3) and be.calls == []
    # metrics.psnr, the training PSNR of get_metrics_dict, is the same quantity in fp32
    assert float(M.psnr(outputs["rgb"], batch["image"])) == pytest.approx(metrics["psnr"], abs=1e-4)


def test_mirror_refuses_camera_batches_until_lpips_is_assigned(golden, mirror):
    model, be = mirror
    outputs, batch, _ = _camera(golden)
    assert model.lpips is None
    with pytest.raises(NotImplementedError, match=r"model\.lpips") as e:
        model.get_image_metrics_and_images(outputs, batch)
    assert "torchmetrics and LPIPS" in str(e.value)
    assert be.image_calls == [] and be.calls == []
    model.lpips = lambda image, rgb: 0.5
    metrics, images = model.get_image_metrics_and_images(outputs, batch)
    assert sorted(metrics) == ["lpips", "psnr", "ssim"] and sorted(images) == ["img"]


def test_mirror_camera_and_lidar_batch_returns_both_halves(golden, mirror):
    from oracle import lidar_metrics_oracle as LM

    model, be = mirror
    lidar_golden = dict(np.load(os.path.join(ROOT, "tests", "golden", "lidar_metrics.npz"), allow_pickle=False))
    outputs, batch, mult = lidar_case(lidar_golden, "depth")
    assert mult == model.config.ray_drop_loss_mult
    cam_outputs, cam_batch, want = _camera(golden)
    outputs.update(cam_outputs)
    batch.update(cam_batch)
    model.lpips = lambda image, rgb: 0.125
    metrics, images = model.get_image_metrics_and_images(outputs, batch)
    assert sorted(metrics) == sorted(("psnr", "ssim", "lpips") + tuple(LM.METRIC_KEYS)) and list(images) == ["img"]
    assert metrics["ssim"] == pytest.approx(want[0, 2], abs=C.SSIM_ATOL)
    assert metrics["depth_median_l2"] == float(lidar_golden["metrics_depth_depth_median_l2"])
    assert len(be.image_calls) == 1 and len(be.calls) == 1


def test_public_names():
    import neurad_studio_b200 as nsb
    from neurad_studio_b200 import metrics as M
    from neurad_studio_b200 import nerfstudio_api

    assert nsb.structural_similarity_index_measure is M.ssim
    model = nerfstudio_api.NeuRADModel(nsb.small_config())
    assert model.ssim is M.ssim and model.lpips is None
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        M.ssim(torch.zeros(1, 3, 16, 16), torch.zeros(1, 3, 16, 16))
