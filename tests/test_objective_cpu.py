"""CPU: the device functions of the lidar losses (csrc/lidar_loss.cuh), run by the host emulation
(tests/host_emul/emul_lidar_loss.cpp), against torch on the CPU.

- The radix select gives torch.quantile / torch.median bit for bit on random and adversarial inputs.
- The forward gives the reference's quantile and mask bit for bit and its scalars within fp32 rounding; the backward
  matches torch autograd of the reference's lines (tests/objective_cases.py).
- The config carries LossSettings' defaults and the plugin maps every field.
"""
import ctypes
import os
import subprocess

import pytest
import torch

from oracle import ref_import
from tests import objective_cases as C

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
needs_reference = pytest.mark.skipif(not ref_import.reference_available(), reason="the reference tree is not present")


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    src = os.path.join(ROOT, "tests", "host_emul", "emul_lidar_loss.cpp")
    so = str(tmp_path_factory.mktemp("emul_lidar_loss") / "libemul_lidar_loss.so")
    subprocess.check_call(["g++", "-std=c++20", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-o", so, src])
    lib = ctypes.CDLL(so)
    lib.emul_quantile.restype = ctypes.c_float
    lib.emul_quantile.argtypes = [ctypes.c_void_p, ctypes.c_int64, ctypes.c_float, ctypes.c_int]
    lib.emul_lidar_losses.restype = ctypes.c_int
    lib.emul_lidar_losses.argtypes = [ctypes.c_int64, ctypes.c_int] + [ctypes.c_void_p] * 6 + [ctypes.c_int64, ctypes.c_void_p] + \
        [ctypes.c_float] * 3 + [ctypes.c_void_p] * 3
    lib.emul_lidar_losses_bwd.restype = ctypes.c_int
    lib.emul_lidar_losses_bwd.argtypes = [ctypes.c_int64, ctypes.c_int] + [ctypes.c_void_p] * 6 + [ctypes.c_int64, ctypes.c_void_p] + \
        [ctypes.c_float] * 2 + [ctypes.c_void_p] * 7
    return lib


def same_bits(a: torch.Tensor, b: torch.Tensor) -> bool:
    a, b = a.reshape(-1).float(), b.reshape(-1).float()
    both_nan = a.isnan() & b.isnan()
    return bool(((a.view(torch.int32) == b.view(torch.int32)) | both_nan).all())


def emul_quantile(lib, x, q, lower=False):
    x = x.contiguous().float()
    return torch.tensor(lib.emul_quantile(x.data_ptr(), x.numel(), q, int(lower)))


def _rows(d):
    p = torch.cat([t.reshape(1, -1) for t in d["props"]]).contiguous()
    ret = d["did_return"].to(torch.uint8).contiguous()
    gt = d["lidar"][:, 3]
    return p, ret, gt


def emul_forward(lib, d):
    n = d["distance"].shape[0]
    p, ret, gt = _rows(d)
    out, mask, counts = torch.empty(4 + C.ROUNDS), torch.empty(n, dtype=torch.uint8), torch.empty(2, dtype=torch.int32)
    rc = lib.emul_lidar_losses(n, C.ROUNDS, d["pred"].data_ptr(), p.data_ptr(), d["distance"].data_ptr(), ret.data_ptr(),
                               d["intensity"].data_ptr(), gt.data_ptr(), gt.stride(0), d["logits"].data_ptr(),
                               C.NON_RETURN_LIDAR_DISTANCE, C.NON_RETURN_LOSS_MULT, C.QUANTILE_THRESHOLD, out.data_ptr(),
                               mask.data_ptr(), counts.data_ptr())
    assert rc == 0
    return out, mask.bool(), counts


def emul_backward(lib, d, mask, counts, grads):
    n = d["distance"].shape[0]
    p, ret, gt = _rows(d)
    m = mask.to(torch.uint8).contiguous()
    dp, di, dl, dprop = torch.empty(n), torch.empty(n), torch.empty(n), torch.empty(C.ROUNDS, n)
    rc = lib.emul_lidar_losses_bwd(n, C.ROUNDS, d["pred"].data_ptr(), p.data_ptr(), d["distance"].data_ptr(), ret.data_ptr(),
                                   d["intensity"].data_ptr(), gt.data_ptr(), gt.stride(0), d["logits"].data_ptr(),
                                   C.NON_RETURN_LIDAR_DISTANCE, C.NON_RETURN_LOSS_MULT, m.data_ptr(), counts.data_ptr(),
                                   grads.contiguous().data_ptr(), dp.data_ptr(), dprop.data_ptr(), di.data_ptr(), dl.data_ptr())
    assert rc == 0
    return dp, dprop, di, dl


# ---------------------------------------------------------------------------------------------- order statistics
@pytest.mark.parametrize("name", sorted(C.order_statistic_inputs()))
def test_select_matches_torch_quantile_and_median(emul, name):
    x = C.order_statistic_inputs()[name]
    for q in C.QS:
        assert same_bits(emul_quantile(emul, x, q), torch.quantile(x, q)), (name, q)
    assert same_bits(emul_quantile(emul, x, 0.0, lower=True), torch.median(x)), name


def test_select_matches_torch_on_random_inputs(emul):
    g = torch.Generator().manual_seed(3)
    for t in range(200):
        n = int(torch.randint(1, 3000, (1,), generator=g))
        x = torch.rand(n, generator=g) * 10 ** float(torch.randint(-3, 4, (1,), generator=g))
        if t % 3 == 0:
            x = (x * 8).round()  # ties
        q = float(torch.rand(1, generator=g))
        assert same_bits(emul_quantile(emul, x, q), torch.quantile(x, q)), (t, n, q)
        assert same_bits(emul_quantile(emul, x, 0.95), torch.quantile(x, 0.95)), (t, n)


# ---------------------------------------------------------------------------------------------- losses
CASES = {"mixed": dict(n=1000, seed=1), "repeated": dict(n=600, seed=2, repeat=True), "n21": dict(n=21, seed=3),
         "n41": dict(n=41, seed=4), "n40": dict(n=40, seed=5), "n1": dict(n=1, seed=6), "n2": dict(n=2, seed=7),
         "all_returns": dict(n=300, seed=8, return_frac=1.0), "no_returns": dict(n=300, seed=9, return_frac=0.0),
         "nan": dict(n=200, seed=10, nan_at=(17,))}


def _reference(d):
    leaves = {k: (d[k].clone().requires_grad_(True)) for k in ("pred", "intensity", "logits")}
    props = [p.clone().requires_grad_(True) for p in d["props"]]
    m, q, mask = C.reference_lidar_terms(leaves["pred"], props, d["distance"], d["did_return"], d["lidar"][..., 3:4],
                                         leaves["intensity"], leaves["logits"])
    return m, q, mask, leaves, props


@pytest.mark.parametrize("name", sorted(CASES))
def test_forward_matches_the_reference_lines(emul, name):
    d = C.lidar_inputs(**CASES[name])
    m, q, mask, _, _ = _reference(d)
    out, got_mask, counts = emul_forward(emul, d)
    assert same_bits(out[3], q), (float(out[3]), float(q))
    assert torch.equal(got_mask, mask)
    assert int(counts[0]) == int(mask.sum()) and int(counts[1]) == int((mask & d["did_return"]).sum())
    got = {"depth_loss": out[0], "intensity_loss": out[1], "ray_drop_loss": out[2],
           **{f"depth_loss_{i}": out[4 + i] for i in range(C.ROUNDS)}}
    for k, v in m.items():
        v = v.detach()
        if v.isnan():
            assert got[k].isnan(), k
        else:
            assert abs(float(got[k]) - float(v)) <= 2e-6 * abs(float(v)) + 1e-30, (k, float(got[k]), float(v))


@pytest.mark.parametrize("name", sorted(CASES))
def test_backward_matches_torch_autograd(emul, name):
    d = C.lidar_inputs(**CASES[name])
    m, _, _, leaves, props = _reference(d)
    g = torch.Generator().manual_seed(11)
    w = {k: float(torch.rand(1, generator=g)) + 0.5 for k in m}
    total = sum(w[k] * v for k, v in m.items() if not v.isnan())
    inputs = [leaves["pred"], leaves["intensity"], leaves["logits"], *props]
    ref = torch.autograd.grad(total, inputs, allow_unused=True) if torch.is_tensor(total) and total.requires_grad else [None] * 5
    ref = [torch.zeros_like(t) if r is None else r for r, t in zip(ref, inputs)]
    out, mask, counts = emul_forward(emul, d)
    grads = torch.tensor([w["depth_loss"], w["intensity_loss"], w["ray_drop_loss"], 0.0,
                          *[w[f"depth_loss_{i}"] for i in range(C.ROUNDS)]])
    for i, k in enumerate(["depth_loss", "intensity_loss"]):  # NaN terms (empty masks) are left out of `total` above
        if m[k].isnan():
            grads[i] = 0.0
    dp, dprop, di, dl = emul_backward(emul, d, mask, counts, grads)
    for got, want in zip([dp, di, dl, *dprop], ref):
        want = want.reshape(-1)
        tol = 1e-6 * max(float(want.abs().max()), 1e-30)
        assert float((got - want).abs().max()) <= tol, (float((got - want).abs().max()), tol)


def test_non_return_beyond_the_distance_gets_exactly_zero(emul):
    d = C.lidar_inputs(n=64, seed=12, return_frac=0.0)
    d["pred"][:] = 150.0
    d["pred"][::2] = 170.0
    _, mask, counts = emul_forward(emul, d)
    mask[:] = True
    counts[0] = 64
    dp, dprop, _, _ = emul_backward(emul, d, mask, counts, torch.ones(4 + C.ROUNDS))
    assert torch.equal(dp, torch.zeros(64))


# ---------------------------------------------------------------------------------------------- config and plugin
def test_config_defaults_are_the_reference_loss_settings():
    import neurad_studio_b200 as nsb

    c = nsb.NeuRADConfig()
    want = {"rgb_mult": 5.0, "vgg_mult": 0.05, "depth_mult": 0.01, "intensity_mult": 0.1, "carving_mult": 0.01,
            "quantile_threshold": 0.95, "interlevel_loss_mult": 0.001, "distortion_loss_mult": 0.002,
            "non_return_loss_mult": 0.1, "prop_lidar_loss_mult": 0.1}
    assert {k: getattr(c, k) for k in want} == want


@needs_reference
def test_config_defaults_match_the_reference_and_the_plugin_maps_them():
    ref_import.install(full=True)
    from nerfstudio.models.neurad import LossSettings

    import neurad_studio_b200 as nsb
    from integration.neurad_b200_plugin import LOSS_SETTINGS

    ref, c = LossSettings(), nsb.NeuRADConfig()
    for k in LOSS_SETTINGS + ("carving_epsilon", "non_return_lidar_distance", "ray_drop_loss_mult"):
        assert getattr(c, k) == getattr(ref, k), k
    assert set(LOSS_SETTINGS) | {"carving_epsilon", "non_return_lidar_distance", "ray_drop_loss_mult"} == \
        set(LossSettings.__dataclass_fields__)
