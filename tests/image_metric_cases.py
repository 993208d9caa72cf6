"""TEST SCAFFOLDING ONLY -- the cases and tolerances of the camera image metrics, shared by tests/test_image_metrics_cpu.py
(host emulation of csrc/image_metrics.cuh) and tests/test_zz_image_metrics_gpu.py (the kernels themselves)."""
import os

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "image_metrics.npz")

NAMES = ["smooth", "identical", "explicit_range", "constant", "negative", "one_window", "wide", "tall", "odd_37x53",
         "odd_65x97_c1", "batch2", "outside_unit", "nan"]
SSIM_ATOL = 2e-6     # absolute, against float64
PSNR_ATOL_DB = 1e-5
MSE_RTOL = 1e-12     # the squared differences are taken and summed in fp64


def load_golden():
    return dict(np.load(GOLDEN, allow_pickle=False))


def case(golden, name):
    """(a, b as channels-last [B, H, W, C] fp32 tensors, data_range or None, the float64 table [(B + 1), 4])."""
    r = float(golden[f"{name}_data_range"])
    return torch.from_numpy(golden[f"{name}_a"]), torch.from_numpy(golden[f"{name}_b"]), (r if r > 0 else None), golden[f"{name}_out"]


def nchw(t):
    """The [B, C, H, W] view of a channels-last [B, H, W, C] tensor: what moveaxis gives the reference's metrics."""
    return t.permute(0, 3, 1, 2)


def check_table(got, want, a, b, data_range, name):
    """got / want [(B + 1), 4] = {mse, psnr, ssim, data_range}; the data range must be fp32's own min / max arithmetic."""
    got = np.asarray(got, np.float64)
    assert got.shape == want.shape, name
    if name == "nan":
        assert np.isnan(got).all(), (name, got)
        return
    np.testing.assert_allclose(got[:, 0], want[:, 0], rtol=MSE_RTOL, atol=0, err_msg=f"{name}: mse")
    finite = np.isfinite(want[:, 1])
    assert np.array_equal(got[~finite, 1], want[~finite, 1]), f"{name}: psnr of identical images is +inf"
    np.testing.assert_allclose(got[finite, 1], want[finite, 1], rtol=0, atol=PSNR_ATOL_DB, err_msg=f"{name}: psnr")
    np.testing.assert_allclose(got[:, 2], want[:, 2], rtol=0, atol=SSIM_ATOL, err_msg=f"{name}: ssim")
    if data_range is None:
        a32, b32 = a.numpy(), b.numpy()
        r = np.maximum(a32.max() - a32.min(), b32.max() - b32.min())
        assert r.dtype == np.float32
    else:
        r = np.float32(data_range)
    assert np.array_equal(got[:, 3], np.full(got.shape[0], np.float64(r))), f"{name}: data_range"
