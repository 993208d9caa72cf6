"""TEST INFRASTRUCTURE ONLY -- write tests/golden/image_metrics.npz:   python -m oracle.make_golden_image_metrics

For every seeded case of oracle/image_metrics_oracle.py (cases): the two fp32 images, the data range given (0 = derived)
and the float64 {mse, psnr, ssim, data_range} table of the batch and of each image.  The table is computed over both
routes of the oracle, torchmetrics' literal reflect-pad / filter / crop order and the valid-window separable filter, and
the fixture is only written if they agree to 1e-12: that agreement is why the kernels never read a padded pixel.

The SSIM definition is from memory, unpinned against torchmetrics (see the oracle's docstring); nothing here reads the
reference tree.
"""
from __future__ import annotations

import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import image_metrics_oracle as IM  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")


def main():
    out = {}
    for name, (a, b, data_range) in IM.cases().items():
        valid = IM.metrics_f64(a, b, data_range)
        padded = IM.metrics_f64(a, b, data_range, padded=True)
        np.testing.assert_allclose(valid, padded, rtol=0, atol=1e-12, equal_nan=True, err_msg=name)
        with np.errstate(invalid="ignore"):  # inf - inf of the identical pair's psnr
            gap = np.nanmax(np.abs(valid - padded), initial=0.0)
        print(f"{name:15s} {str(a.shape):18s} mse {valid[0, 0]:.6g}  psnr {valid[0, 1]:.6f}  ssim {valid[0, 2]:.9f}  "
              f"range {valid[0, 3]:.6g}  |padded - valid| {gap:.1e}")
        out[f"{name}_a"] = a
        out[f"{name}_b"] = b
        out[f"{name}_data_range"] = np.float32(data_range)
        out[f"{name}_out"] = valid
    path = os.path.join(GOLDEN, "image_metrics.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, f"({os.path.getsize(path)} bytes)")


if __name__ == "__main__":
    main()
