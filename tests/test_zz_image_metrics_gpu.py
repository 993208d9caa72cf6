"""GPU: the camera image metrics kernels (csrc/image_metrics.cuh, b200nerf_image_metrics) against float64 at the
tolerances of tests/image_metric_cases.py, the mirror's camera branch on a rendered image, and -- only where the package
is installed -- torchmetrics itself: the SSIM definition is from memory, unpinned against torchmetrics, and that last
test is the one place where the two meet."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import image_metrics_oracle as IM
from tests import image_metric_cases as C

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)


@pytest.fixture(scope="module")
def golden():
    return C.load_golden()


@pytest.fixture(scope="module")
def be():
    from neurad_studio_b200.nerfstudio_api import get_backend

    return get_backend(DEV)


def run(be, a, b, data_range=None):
    """a, b channels-last [B, H, W, C] host tensors -> the [(B + 1), 4] table, through [B, C, H, W] views on the device."""
    out = be.image_metrics(C.nchw(a.to(DEV)), C.nchw(b.to(DEV)), data_range)
    torch.cuda.synchronize()
    be.check_status()
    return out.cpu()


@pytest.mark.parametrize("name", C.NAMES)
def test_kernels_against_float64(golden, be, name):
    a, b, data_range, want = C.case(golden, name)
    got = run(be, a, b, data_range).numpy()
    C.check_table(got, want, a, b, data_range, name)
    if name == "identical":
        assert (got[:, 2] == 1.0).all()


def test_two_calls_and_a_side_stream_give_the_same_bits(golden, be):
    a, b, _, _ = C.case(golden, "batch2")
    r1, r2 = run(be, a, b), run(be, a, b)
    assert torch.equal(r1, r2)
    da, db = C.nchw(a.to(DEV)), C.nchw(b.to(DEV))
    side = torch.cuda.Stream(device=DEV)
    side.wait_stream(torch.cuda.current_stream(DEV))
    with torch.cuda.stream(side):
        r3 = be.image_metrics(da, db)
    side.synchronize()
    assert torch.equal(r3.cpu(), r1)


def test_layouts_are_read_in_place(golden, be):
    a, b, _, want = C.case(golden, "batch2")
    base = run(be, a, b)
    da, db = a.to(DEV), b.to(DEV)
    planar = be.image_metrics(C.nchw(da).contiguous(), C.nchw(db)).cpu()
    assert torch.equal(planar[:, 2:], base[:, 2:]) and torch.allclose(planar[:, :2], base[:, :2], rtol=1e-13, atol=0)
    rgba = torch.cat([da, torch.full_like(da[..., :1], 7.0)], -1)
    sliced = be.image_metrics(C.nchw(rgba[..., :3]), C.nchw(db)).cpu()
    assert torch.equal(sliced[:, 2:], base[:, 2:])
    C.check_table(sliced.numpy(), want, a, b, None, "batch2")


def test_full_hd_pair_against_float64(be):
    rng = np.random.default_rng(7)
    a, b = IM._render_like(rng, 1, 1080, 1920, 3)
    want = IM.metrics_f64(a, b)
    ta, tb = torch.from_numpy(a), torch.from_numpy(b)
    got = run(be, ta, tb).numpy()
    print(f"1080p: ssim {got[0, 2]:.9f} (float64 {want[0, 2]:.9f}, diff {got[0, 2] - want[0, 2]:+.2e}), psnr {got[0, 1]:.6f}")
    C.check_table(got, want, ta, tb, None, "full_hd")


def test_public_ssim_keeps_the_reference_call_shape(golden, be):
    import neurad_studio_b200 as nsb

    a, b, _, want = C.case(golden, "smooth")
    image = torch.moveaxis(a[0].to(DEV), -1, 0)[None, ...]  # neurad.py:581-582
    rgb = torch.moveaxis(b[0].to(DEV), -1, 0)[None, ...]
    v = nsb.structural_similarity_index_measure(image, rgb)
    assert v.dim() == 0 and v.dtype == torch.float32 and v.device == rgb.device
    assert float(v) == pytest.approx(want[0, 2], abs=1e-6)
    assert float(nsb.structural_similarity_index_measure(image, rgb, data_range=2.0)) > float(v)


def test_rejects_what_it_cannot_compute(be):
    from neurad_studio_b200.lib import B200NerfError

    x = torch.zeros(1, 3, 10, 64, device=DEV)
    with pytest.raises(B200NerfError, match="11 x 11"):
        be.image_metrics(x, x)
    with pytest.raises(ValueError, match="one shape"):
        be.image_metrics(x, x[..., :32])
    # argument validation only: rejected before any launch
    big = torch.zeros(1, 1, 16, 16, device=DEV)
    s = (ctypes.c_int64 * 4)(0, 0, 0, 0)
    out = torch.empty(2, 4, dtype=torch.float64, device=DEV)
    p = ctypes.c_void_p(big.data_ptr())
    rc = be.lib.b200nerf_image_metrics(be._h, p, p, 1, 1 << 15, 1 << 15, 1, s, s, 0.0, ctypes.c_void_p(out.data_ptr()), be._stream)
    assert rc == -1 and b"2^18 tiles" in be.lib.b200nerf_last_error()
    rc = be.lib.b200nerf_image_metrics(be._h, p, p, 257, 16, 16, 1, s, s, 0.0, ctypes.c_void_p(out.data_ptr()), be._stream)
    assert rc == -1 and b"256 images" in be.lib.b200nerf_last_error()


def test_mirror_scores_a_rendered_image():
    import neurad_studio_b200 as nsb
    from neurad_studio_b200 import metrics as M
    from neurad_studio_b200 import scene
    from neurad_studio_b200.nerfstudio_api import Cameras, NeuRADModel

    cfg = nsb.small_config(n_actors=0, log2_main=12, log2_prop=11)
    model = NeuRADModel(cfg)
    model.load_reference_state_dict(scene.make_params(cfg, seed=4, beta=3.0, sdf_bias=0.5))
    dec = scene.make_rgb_decoder_params(seed=5)
    model.rgb_decoder.load_state_dict({k[len("rgb_decoder."):]: v for k, v in dec.items()}, strict=False)
    model = model.to(DEV).eval()
    cam = scene.pandaset_rig(time=2.0, width=48, height=30)[1]
    rb = Cameras([cam], DEV).generate_rays(camera_indices=0, keep_shape=True)
    out = model.get_outputs_for_camera_ray_bundle(rb)
    rgb = out["rgb"]
    assert rgb.shape == (30, 48, 3)
    g = torch.Generator().manual_seed(3)
    gt = (rgb.cpu() + 0.05 * torch.randn(rgb.shape, generator=g)).clamp(0, 1)  # the batch's image arrives on the host
    with pytest.raises(NotImplementedError, match=r"model\.lpips"):
        model.get_image_metrics_and_images(out, {"image": gt})
    model.lpips = lambda image, pred: (image - pred).abs().mean()
    metrics, images = model.get_image_metrics_and_images(out, {"image": gt})
    assert list(metrics) == ["psnr", "ssim", "lpips"] and all(isinstance(v, float) for v in metrics.values())
    assert list(images) == ["img"] and images["img"].shape == (30, 96, 3) and images["img"].device == rgb.device
    want = IM.metrics_f64(gt.numpy()[None], rgb.cpu().numpy()[None])
    assert metrics["ssim"] == pytest.approx(want[0, 2], abs=C.SSIM_ATOL)
    assert metrics["psnr"] == pytest.approx(want[0, 1], abs=C.PSNR_ATOL_DB)
    assert metrics["lpips"] == pytest.approx(float((gt - rgb.cpu()).abs().mean()), rel=1e-5)
    assert float(M.psnr(rgb, gt.to(DEV))) == pytest.approx(metrics["psnr"], abs=1e-4)


@pytest.mark.parametrize("name", ["smooth", "batch2", "explicit_range"])
def test_against_torchmetrics_where_it_is_installed(golden, be, name):
    torchmetrics = pytest.importorskip("torchmetrics")
    from torchmetrics.functional import structural_similarity_index_measure

    a, b, data_range, _ = C.case(golden, name)
    got = run(be, a, b, data_range)
    preds, target = C.nchw(a.to(DEV)).contiguous(), C.nchw(b.to(DEV)).contiguous()
    ssim = structural_similarity_index_measure(preds, target, data_range=data_range)
    psnr = torchmetrics.PeakSignalNoiseRatio(data_range=1.0).to(DEV)(preds, target)
    assert float(got[0, 2]) == pytest.approx(float(ssim), abs=1e-5)
    assert float(got[0, 1]) == pytest.approx(float(psnr), abs=1e-5 * max(1.0, abs(float(psnr))))
