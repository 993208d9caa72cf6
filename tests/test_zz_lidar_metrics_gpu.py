"""GPU: the chamfer-distance kernel (csrc/lidar_eval.cuh, b200nerf_chamfer_distance) and the mirror's lidar metrics
against float64 and the reference's values recorded in tests/golden/lidar_metrics.npz."""
import ctypes
import os

import numpy as np
import pytest
import torch

from oracle import lidar_metrics_oracle as LM

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "lidar_metrics.npz")
U = 2.0 ** -24
MIN_BOUND = 8 * U  # per-pair value: <= 6 roundings, no cancellation (tests/test_lidar_metrics_cpu.py)
DEV = torch.device("cuda", 0)
NAMES = ["ragged", "far100m", "n_ne_m"]


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(GOLDEN, allow_pickle=False))


@pytest.fixture(scope="module")
def be():
    from neurad_studio_b200.nerfstudio_api import get_backend

    return get_backend(DEV)


def run(be, pred, gt, normalize=True):
    out, ms, md = be.chamfer_distance(pred.to(DEV), gt.to(DEV), normalize, want_minima=True)
    torch.cuda.synchronize()
    be.check_status()
    return float(out), ms.cpu(), md.cpu()


def check_minima(got, want):
    ok = (got.double() - want).abs() <= MIN_BOUND * want + 1e-30
    assert bool(ok.all()), f"{int((~ok).sum())} of {ok.numel()} minima outside {MIN_BOUND / U:.0f} ulp of float64"


@pytest.mark.parametrize("name", NAMES)
def test_chamfer_against_float64_and_the_reference(golden, be, name):
    pred = torch.from_numpy(golden[f"chamfer_{name}_pred"])
    gt = torch.from_numpy(golden[f"chamfer_{name}_gt"])
    val, ms, md = run(be, pred, gt)
    check_minima(ms, LM.min_sq_f64(pred, gt))
    check_minima(md, LM.min_sq_f64(gt, pred))
    f64 = float(golden[f"chamfer_{name}_f64"])
    err, ref_err = abs(val - f64), abs(float(golden[f"chamfer_{name}_ref"]) - f64)
    print(f"{name}: kernel rel err {err / f64:.2e}, reference fp32 rel err {ref_err / f64:.2e}")
    assert err <= 1e-6 * f64
    assert err <= ref_err  # the reference's own noise floor (fp32 cdist), cf. tests/test_reference_noise_floor.py
    a, b = golden[f"chamfer_{name}_sums_f64"]
    unnorm, _, _ = run(be, pred, gt, normalize=False)
    assert abs(unnorm - (a + b)) <= 1e-6 * (a + b)


def test_chamfer_is_bit_reproducible(be):
    g = torch.Generator().manual_seed(11)
    pred = torch.randn(64 * 1800, 3, generator=g) * 40
    gt = torch.randn(64 * 1800 - 77, 3, generator=g) * 40
    r1, r2 = run(be, pred, gt), run(be, pred, gt)
    assert r1[0] == r2[0]
    assert torch.equal(r1[1], r2[1]) and torch.equal(r1[2], r2[2])
    idx = torch.randperm(pred.shape[0], generator=g)[:300]
    check_minima(r1[1][idx], LM.min_sq_f64(pred[idx], gt))


def test_chamfer_nan_propagates(be):
    g = torch.Generator().manual_seed(12)
    src, dst = torch.randn(3000, 3, generator=g), torch.randn(2500, 3, generator=g)
    dst[1234, 0] = float("nan")
    val, ms, md = run(be, src, dst)
    assert val != val and bool(ms.isnan().all()) and md.isnan().nonzero().flatten().tolist() == [1234]
    dst[1234, 0] = 0.0
    src[7, 1] = float("nan")
    val, ms, md = run(be, src, dst)
    assert val != val and ms.isnan().nonzero().flatten().tolist() == [7] and bool(md.isnan().all())


def test_chamfer_single_points_and_strided_rows(be):
    g = torch.Generator().manual_seed(13)
    pts4 = (torch.randn(5000, 4, generator=g) * 50).to(DEV)
    one = (torch.randn(1, 3, generator=g) * 50).to(DEV)
    for src, dst in ((pts4[:, :3], one), (one, pts4[:, :3]), (one, one + 1.0)):
        val, ms, md = run(be, src, dst)
        check_minima(ms, LM.min_sq_f64(src.cpu(), dst.cpu()))
        check_minima(md, LM.min_sq_f64(dst.cpu(), src.cpu()))
        assert val == pytest.approx(LM.chamfer_f64(src.cpu(), dst.cpu()), rel=1e-6)
    strided = pts4[:, :3]
    assert strided.stride(0) == 4
    a = run(be, strided, pts4[:1000, :3])
    b = run(be, strided.contiguous(), pts4[:1000, :3].contiguous())
    assert a[0] == b[0] and torch.equal(a[1], b[1]) and torch.equal(a[2], b[2])


def test_chamfer_rejects_empty_and_oversized_clouds(be):
    from neurad_studio_b200.lib import B200NerfError

    pts = torch.randn(10, 3, device=DEV)
    with pytest.raises(B200NerfError, match="empty"):
        be.chamfer_distance(pts[:0], pts)
    with pytest.raises(B200NerfError, match="empty"):
        be.chamfer_distance(pts, pts[:0])
    # argument validation only: rejected before any launch or memory access
    buf = torch.empty(4, dtype=torch.float64, device=DEV)
    p = ctypes.c_void_p(pts.data_ptr())
    rc = be.lib.b200nerf_chamfer_distance(be._h, p, 1 << 31, 3, p, 10, 3, 1, ctypes.c_void_p(buf.data_ptr()), p, p, be._stream)
    assert rc == -1 and b"2^31" in be.lib.b200nerf_last_error()


def test_public_chamfer_distance_keeps_the_reference_signature(golden):
    import neurad_studio_b200 as nsb

    pred = torch.from_numpy(golden["chamfer_n_ne_m_pred"]).to(DEV)
    gt = torch.from_numpy(golden["chamfer_n_ne_m_gt"]).to(DEV)
    a, b = golden["chamfer_n_ne_m_sums_f64"]
    v = nsb.chamfer_distance(pred, gt, 1_000, True)
    assert v.dim() == 0 and v.dtype == torch.float32 and v.device == pred.device
    assert float(v) == pytest.approx(float(golden["chamfer_n_ne_m_f64"]), rel=1e-6)
    for cs, norm in ((None, True), (None, False), (1_000, False), (17, False)):  # chunk_size=None never normalises
        assert float(nsb.chamfer_distance(pred, gt, cs, norm)) == pytest.approx(a + b, rel=1e-6)


@pytest.mark.parametrize("name", ["ray_drop", "depth", "fallback"])
def test_mirror_metrics_on_the_gpu_match_the_reference(golden, name):
    import neurad_studio_b200 as nsb
    from neurad_studio_b200 import nerfstudio_api

    mult = float(golden[f"metrics_{name}_ray_drop_loss_mult"])
    model = nerfstudio_api.NeuRADModel(nsb.small_config(ray_drop_loss_mult=mult)).to(DEV)
    outputs = {k[len(f"metrics_{name}_out_"):]: torch.from_numpy(v).to(DEV) for k, v in golden.items() if k.startswith(f"metrics_{name}_out_")}
    batch = {k[len(f"metrics_{name}_in_"):]: torch.from_numpy(v).to(DEV) for k, v in golden.items() if k.startswith(f"metrics_{name}_in_")}
    metrics, images = model.get_image_metrics_and_images(outputs, batch)
    assert images == {} and sorted(metrics) == sorted(LM.METRIC_KEYS)
    for k in ("is_lidar", "did_return"):
        assert np.array_equal(batch[k].cpu().numpy(), golden[f"metrics_{name}_after_{k}"])
    did, depth, dist = batch["did_return"][:, 0], outputs["depth"], batch["distance"]
    want = {  # the reference's expressions, evaluated by torch on this device
        "depth_median_l2": float(torch.median((depth[did] - dist[did]) ** 2)),
        "depth_mean_rel_l2": float(torch.mean(((depth[did] - dist[did]) / dist[did]) ** 2)),
        "intensity_rmse": float(torch.sqrt(torch.mean((outputs["intensity"][did] - batch["lidar"][did, 3:4]) ** 2))),
        "ray_drop_accuracy": float(((outputs["ray_drop_logits"].sigmoid() > 0.5).squeeze(-1) == ~did).float().mean()),
    }
    for k, v in want.items():
        assert metrics[k] == v, k
        assert v == pytest.approx(float(golden[f"metrics_{name}_{k}"]), rel=1e-5), k
    cd = metrics["chamfer_distance"]
    if bool(golden[f"metrics_{name}_chamfer_is_tensor"]):
        assert isinstance(cd, torch.Tensor) and cd.dim() == 0
        assert float(cd) == pytest.approx(float(golden[f"metrics_{name}_chamfer_distance"]), rel=1e-6)
    else:
        f64 = float(golden[f"metrics_{name}_chamfer_f64"])
        ref = float(golden[f"metrics_{name}_chamfer_distance"])
        assert isinstance(cd, float)
        assert abs(cd - f64) <= 1e-6 * f64
        assert abs(cd - f64) <= max(abs(ref - f64), 1e-7 * f64)
