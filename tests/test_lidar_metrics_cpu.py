"""CPU: NeuRAD's lidar metrics.

- The float64 oracle (oracle/lidar_metrics_oracle.py) and the golden inputs agree with the real reference.
- The mirror's NeuRADModel.get_image_metrics_and_images, over a CPU stand-in backend defined here, reproduces the
  reference's metrics_dict of every branch, with its batch side effects, and refuses camera batches.
- The per-tile device function of the chamfer kernel (csrc/lidar_eval.cuh), run by the host emulation
  (tests/host_emul/emul_chamfer.cpp), gives per-point minima within a few fp32 ulp of float64.
"""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

from oracle import lidar_metrics_oracle as LM
from oracle import ref_import
from tests.test_reference_plugin import plugin  # noqa: F401  (fixture: the plugin registered through the reference)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "lidar_metrics.npz")
U = 2.0 ** -24  # fp32 unit roundoff
# |dx|, |dy|, |dz| carry one rounding each, the squares one more and the two FMAs one each: <= 6u relative per pair,
# and the min of values that are each within 6u is within 6u of the true min
MIN_BOUND = 8 * U

needs_reference = pytest.mark.skipif(not ref_import.reference_available(), reason="the reference tree is not present")


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(GOLDEN, allow_pickle=False))


# ---------------------------------------------------------------------------------------------- oracle vs reference
def test_golden_inputs_are_the_oracles_seeded_cases(golden):
    for name, (pred, gt) in LM.chamfer_cases().items():
        assert np.array_equal(golden[f"chamfer_{name}_pred"], pred.numpy()), name
        assert np.array_equal(golden[f"chamfer_{name}_gt"], gt.numpy()), name
    for name, (outputs, batch, mult) in LM.metrics_cases().items():
        for k, v in outputs.items():
            assert np.array_equal(golden[f"metrics_{name}_out_{k}"], v.numpy()), (name, k)
        for k, v in batch.items():
            assert np.array_equal(golden[f"metrics_{name}_in_{k}"], v.numpy()), (name, k)
        assert float(golden[f"metrics_{name}_ray_drop_loss_mult"]) == mult


def test_oracle_sums_match_golden(golden):
    for name, (pred, gt) in LM.chamfer_cases().items():
        a, b = LM.chamfer_sums_f64(pred, gt)
        np.testing.assert_allclose([a, b], golden[f"chamfer_{name}_sums_f64"], rtol=1e-12)
        assert LM.chamfer_f64(pred, gt) == pytest.approx(float(golden[f"chamfer_{name}_f64"]), rel=1e-12)


@needs_reference
def test_reference_chamfer_reproduces_golden_and_is_near_the_oracle(golden):
    """The reference's fp32 chunked cdist on the golden inputs: bit-identical to the recorded value, and within its own
    cancellation error of the float64 oracle (about 1e-4 relative at 40 m ranges, several percent at 100 m)."""
    ref_import.install()
    from nerfstudio.utils.math import chamfer_distance

    for name, (pred, gt) in LM.chamfer_cases().items():
        ref = float(chamfer_distance(pred, gt, 1_000, True))
        assert ref == float(golden[f"chamfer_{name}_ref"]), name
        f64 = LM.chamfer_f64(pred, gt)
        assert abs(ref - f64) <= 0.1 * f64, (name, ref, f64)


@needs_reference
def test_reference_unnormalised_path_ignores_normalize_flag():
    """With chunk_size=None the reference never normalises (utils/math.py:777-778); the library keeps that."""
    ref_import.install()
    from nerfstudio.utils.math import chamfer_distance

    pred, gt = LM.chamfer_cases()["n_ne_m"]
    a, b = LM.chamfer_sums_f64(pred, gt)
    assert float(chamfer_distance(pred, gt, None, True)) == pytest.approx(a + b, rel=1e-4)
    assert float(chamfer_distance(pred, gt, 1_000, False)) == pytest.approx(a + b, rel=1e-4)


# ---------------------------------------------------------------------------------------------- the mirror's logic
class ChamferFakeBackend:
    """TEST SCAFFOLDING ONLY: B200Backend.chamfer_distance's contract on the CPU, as the float64 oracle."""

    def __init__(self):
        self.calls = []

    def chamfer_distance(self, pred, gt, normalize_with_target=True, want_minima=False):
        assert not want_minima
        self.calls.append((pred.shape[0], gt.shape[0], normalize_with_target))
        m = gt.shape[0] if normalize_with_target else 1
        a, b = LM.chamfer_sums_f64(pred, gt)
        return torch.tensor(a / m + b / m, dtype=torch.float64)


@pytest.fixture()
def mirror(monkeypatch):
    import neurad_studio_b200 as nsb
    from neurad_studio_b200 import nerfstudio_api

    be = ChamferFakeBackend()
    monkeypatch.setattr(nerfstudio_api, "get_backend", lambda device: be)

    def make(mult):
        model = nerfstudio_api.NeuRADModel(nsb.small_config(ray_drop_loss_mult=mult))
        return model, be

    return make


def _case(golden, name):
    outputs = {k[len(f"metrics_{name}_out_"):]: torch.from_numpy(v) for k, v in golden.items() if k.startswith(f"metrics_{name}_out_")}
    batch = {k[len(f"metrics_{name}_in_"):]: torch.from_numpy(v) for k, v in golden.items() if k.startswith(f"metrics_{name}_in_")}
    return outputs, batch, float(golden[f"metrics_{name}_ray_drop_loss_mult"])


@pytest.mark.parametrize("name", ["ray_drop", "depth", "fallback"])
def test_mirror_metrics_match_reference(golden, mirror, name):
    outputs, batch, mult = _case(golden, name)
    model, be = mirror(mult)
    given = set(batch)
    metrics, images = model.get_image_metrics_and_images(outputs, batch)
    assert images == {}
    assert sorted(metrics) == sorted(LM.METRIC_KEYS)
    for k in ("is_lidar", "did_return"):  # filled in when absent, left alone otherwise
        assert np.array_equal(batch[k].numpy(), golden[f"metrics_{name}_after_{k}"]), k
        if k in given:
            assert np.array_equal(batch[k].numpy(), golden[f"metrics_{name}_in_{k}"])
    for k in LM.METRIC_KEYS[:4]:  # the same torch ops on the same device as the reference's run: identical
        assert isinstance(metrics[k], float)
        assert metrics[k] == float(golden[f"metrics_{name}_{k}"]), k
    cd = metrics["chamfer_distance"]
    if bool(golden[f"metrics_{name}_chamfer_is_tensor"]):
        assert isinstance(cd, torch.Tensor) and cd.dim() == 0 and be.calls == []
        assert float(cd) == float(golden[f"metrics_{name}_chamfer_distance"])
    else:
        assert isinstance(cd, float) and len(be.calls) == 1 and be.calls[0][2] is True
        assert cd == pytest.approx(float(golden[f"metrics_{name}_chamfer_f64"]), rel=1e-6)
        ref = float(golden[f"metrics_{name}_chamfer_distance"])
        assert abs(cd - ref) <= 1e-3 * ref


def test_mirror_refuses_camera_batches(golden, mirror):
    outputs, batch, mult = _case(golden, "depth")
    model, be = mirror(mult)
    batch["image"] = torch.zeros(4, 4, 3)
    with pytest.raises(NotImplementedError, match="torchmetrics and LPIPS"):
        model.get_image_metrics_and_images(outputs, batch)
    assert be.calls == []


def test_config_default_matches_reference_loss_settings():
    import neurad_studio_b200 as nsb

    assert nsb.NeuRADConfig().ray_drop_loss_mult == 0.01


# ---------------------------------------------------------------------------------------------- host emulation
@pytest.fixture(scope="module")
def emul_lib(tmp_path_factory):
    src = os.path.join(ROOT, "tests", "host_emul", "emul_chamfer.cpp")
    so = str(tmp_path_factory.mktemp("emul_chamfer") / "libemul_chamfer.so")
    subprocess.check_call(["g++", "-std=c++20", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-o", so, src])
    lib = ctypes.CDLL(so)
    lib.emul_chamfer_min.restype = ctypes.c_int
    lib.emul_chamfer_min.argtypes = [ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_void_p, ctypes.c_int64, ctypes.c_int,
                                     ctypes.c_void_p]
    return lib


def emul_min(lib, src, dst):
    out = torch.empty(src.shape[0])
    rc = lib.emul_chamfer_min(src.data_ptr(), src.shape[0], src.stride(0), dst.data_ptr(), dst.shape[0], dst.stride(0), out.data_ptr())
    assert rc == 0
    return out


def check_minima(got, want):
    ok = (got.double() - want).abs() <= MIN_BOUND * want + 1e-30
    assert bool(ok.all()), f"{int((~ok).sum())} minima outside {MIN_BOUND / U:.0f} ulp"


@pytest.mark.parametrize("name", ["ragged", "far100m", "n_ne_m"])
def test_emulated_minima_and_scalar_against_float64(golden, emul_lib, name):
    pred = torch.from_numpy(golden[f"chamfer_{name}_pred"])
    gt = torch.from_numpy(golden[f"chamfer_{name}_gt"])
    ms, md = emul_min(emul_lib, pred, gt), emul_min(emul_lib, gt, pred)
    check_minima(ms, LM.min_sq_f64(pred, gt))
    check_minima(md, LM.min_sq_f64(gt, pred))
    m = gt.shape[0]
    val = float(ms.double().sum()) / m + float(md.double().sum()) / m
    f64 = float(golden[f"chamfer_{name}_f64"])
    assert abs(val - f64) <= 1e-6 * f64
    # at least as close to float64 as the reference's own fp32 result
    assert abs(val - f64) <= abs(float(golden[f"chamfer_{name}_ref"]) - f64)


def test_emulated_strided_rows_and_single_points(emul_lib):
    g = torch.Generator().manual_seed(3)
    pts4 = torch.randn(777, 4, generator=g) * 30
    other = torch.randn(1, 3, generator=g) * 30
    a = emul_min(emul_lib, pts4[:, :3], other)
    b = emul_min(emul_lib, pts4[:, :3].contiguous(), other)
    assert torch.equal(a, b)
    check_minima(a, LM.min_sq_f64(pts4, other))
    check_minima(emul_min(emul_lib, other, pts4[:, :3]), LM.min_sq_f64(other, pts4))


def test_emulated_nan_propagates(emul_lib):
    g = torch.Generator().manual_seed(4)
    src, dst = torch.randn(600, 3, generator=g), torch.randn(700, 3, generator=g)
    dst[517, 1] = float("nan")
    ms, md = emul_min(emul_lib, src, dst), emul_min(emul_lib, dst, src)
    assert bool(ms.isnan().all())  # every source point's candidate set contains the NaN point
    assert md.isnan().nonzero().flatten().tolist() == [517]
    src[5, 2] = float("nan")
    dst[517, 1] = 0.0
    ms, md = emul_min(emul_lib, src, dst), emul_min(emul_lib, dst, src)
    assert ms.isnan().nonzero().flatten().tolist() == [5] and bool(md.isnan().all())


def test_keys_order_like_the_minima():
    """chamfer_key is what the grid's target splits meet in: an unsigned min over keys must be the NaN-propagating min."""
    vals = [0.0, 1e-45, 1e-38, 0.5, 1.0, 3.4e38, float("inf")]
    bits = [np.float32(v).view(np.uint32) + 1 for v in vals]
    assert bits == sorted(bits) and len(set(bits)) == len(bits)
    assert 0 < min(bits) and max(bits) < 0xFFFFFFFF  # NaN -> 0 wins; 0xffffffff is the empty min


# ---------------------------------------------------------------------------------------------- the plugin
@needs_reference
def test_plugin_evaluates_lidar_through_the_library_chamfer(golden, plugin, monkeypatch):
    """`ns-eval` with neurad-b200: the inherited get_image_metrics_and_images calls self.chamfer_distance, which the plugin
    points at neurad_studio_b200.chamfer_distance(pred, gt, 1_000, True); the config mapping carries ray_drop_loss_mult."""
    from tests.test_reference_plugin import _build_model

    from neurad_studio_b200 import nerfstudio_api

    from integration.neurad_b200_plugin import config_from_reference

    be = ChamferFakeBackend()
    monkeypatch.setattr(nerfstudio_api, "get_backend", lambda device: be)
    model, _, _ = _build_model(plugin, n_actors=0)
    assert config_from_reference(model).ray_drop_loss_mult == model.config.loss.ray_drop_loss_mult == 0.01
    outputs, batch, _ = _case(golden, "ray_drop")
    metrics, images = model.get_image_metrics_and_images(outputs, batch)
    assert images == {} and be.calls and be.calls[0][2] is True
    for k in LM.METRIC_KEYS[:4]:
        assert metrics[k] == float(golden[f"metrics_ray_drop_{k}"]), k
    assert metrics["chamfer_distance"] == pytest.approx(float(golden["metrics_ray_drop_chamfer_f64"]), rel=1e-6)
