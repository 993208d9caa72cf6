"""GPU: the lidar-loss operator (csrc/lidar_loss.cuh, b200nerf_lidar_losses_fwd / _bwd / b200nerf_quantile) and the
mirror's get_metrics_dict / get_loss_dict against torch on the same CUDA device.

- The order statistic is torch.quantile / torch.median bit for bit, up to torch's own limit of 2^24 values.
- The forward gives the reference lines' quantile and mask bit for bit, the scalars within 2e-6 relative, and the
  backward torch autograd's gradients within 1e-6 of each tensor's max (tests/objective_cases.py).
- Forward and backward never synchronise the host; two calls give the same bits.
- A training step through get_outputs -> get_metrics_dict -> get_loss_dict -> backward() agrees with the same step whose
  lidar terms come from the torch restatement.
"""
import pytest
import torch

from tests import objective_cases as C

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)


@pytest.fixture(scope="module")
def be():
    from neurad_studio_b200.nerfstudio_api import get_backend

    return get_backend(DEV)


def same_bits(a, b) -> bool:
    a, b = a.reshape(-1).float().cpu(), b.reshape(-1).float().cpu()
    return bool(((a.view(torch.int32) == b.view(torch.int32)) | (a.isnan() & b.isnan())).all())


# ---------------------------------------------------------------------------------------------- order statistics
@pytest.mark.parametrize("n", [1, 2, 3, 21, 16384, 115200, 262144, 1 << 24])
def test_order_statistics_match_torch(be, n):
    g = torch.Generator(device=DEV).manual_seed(n)
    xs = {"uniform": torch.rand(n, device=DEV, generator=g),
          "ties": torch.randint(0, 50, (n,), device=DEV, generator=g).float(),
          "losses": (torch.randn(n, device=DEV, generator=g) * 3).abs() * 0.1}
    for name, x in xs.items():
        for q in C.QS:
            assert same_bits(be.quantile(x, q), torch.quantile(x, q)), (name, q)
        assert same_bits(be.quantile(x, 0.0, lower_median=True), torch.median(x)), name
    be.check_status()


@pytest.mark.parametrize("name", sorted(C.order_statistic_inputs()))
def test_order_statistics_adversarial(be, name):
    x = C.order_statistic_inputs()[name].to(DEV)
    for q in C.QS:
        assert same_bits(be.quantile(x, q), torch.quantile(x, q)), q
    assert same_bits(be.quantile(x, 0.0, lower_median=True), torch.median(x))


def test_order_statistic_rejects_empty_and_oversized(be):
    from neurad_studio_b200.lib import B200NerfError

    with pytest.raises(B200NerfError):
        be.quantile(torch.empty(0, device=DEV), 0.5)
    with pytest.raises(B200NerfError):
        be.quantile(torch.empty((1 << 24) + 1, device=DEV), 0.5)


# ---------------------------------------------------------------------------------------------- the operator
CASES = {"mixed": dict(n=16384, seed=1), "repeated": dict(n=4000, seed=2, repeat=True), "n21": dict(n=21, seed=3),
         "n41": dict(n=41, seed=4), "n40": dict(n=40, seed=5), "n1": dict(n=1, seed=6), "n2": dict(n=2, seed=7),
         "all_returns": dict(n=3000, seed=8, return_frac=1.0), "no_returns": dict(n=3000, seed=9, return_frac=0.0),
         "nan": dict(n=2000, seed=10, nan_at=(17,)), "sweep": dict(n=262144, seed=11)}


def _library(d, requires_grad=True):
    from neurad_studio_b200 import losses as L

    leaves = {k: d[k].clone().requires_grad_(requires_grad) for k in ("pred", "intensity", "logits")}
    props = [p.clone().requires_grad_(requires_grad) for p in d["props"]]
    res = L.lidar_losses(leaves["pred"], props, d["distance"], d["did_return"], leaves["intensity"], d["lidar"][..., 3:4],
                         leaves["logits"])
    return res, leaves, props


def _reference(d):
    leaves = {k: d[k].clone().requires_grad_(True) for k in ("pred", "intensity", "logits")}
    props = [p.clone().requires_grad_(True) for p in d["props"]]
    m, q, mask = C.reference_lidar_terms(leaves["pred"], props, d["distance"], d["did_return"], d["lidar"][..., 3:4],
                                         leaves["intensity"], leaves["logits"])
    return m, q, mask, leaves, props


@pytest.mark.parametrize("name", sorted(CASES))
def test_operator_matches_the_reference_lines(be, name):
    d = C.lidar_inputs(**CASES[name], device=DEV)
    m, q, mask, rl, rp = _reference(d)
    res, ll, lp = _library(d)
    assert same_bits(res["quantile"], q), (float(res["quantile"]), float(q))
    assert torch.equal(res["quantile_mask"], mask)
    for k in C.SCALAR_KEYS:
        want, got = float(m[k]), float(res[k])
        if want != want:
            assert got != got, k
        else:
            assert abs(got - want) <= 2e-6 * abs(want) + 1e-30, (k, got, want)
    g = torch.Generator().manual_seed(12)
    w = {k: float(torch.rand(1, generator=g)) + 0.5 for k in C.SCALAR_KEYS}
    live = [k for k in C.SCALAR_KEYS if not m[k].isnan()]  # an empty mask's NaN mean has no gradient in either
    sum(w[k] * m[k] for k in live).backward()
    sum(w[k] * res[k] for k in live).backward()
    for got, want in zip([ll["pred"], ll["intensity"], ll["logits"], *lp], [rl["pred"], rl["intensity"], rl["logits"], *rp]):
        gw = torch.zeros_like(want) if want.grad is None else want.grad
        tol = 1e-6 * max(float(gw.abs().max()), 1e-30)
        assert float((got.grad - gw).abs().max()) <= tol
    be.check_status()


def test_operator_never_synchronises_and_repeats_bit_for_bit(be):
    d = C.lidar_inputs(n=16384, seed=13, device=DEV)
    runs = []
    torch.cuda.synchronize()
    for _ in range(2):
        torch.cuda.set_sync_debug_mode("error")
        try:
            res, leaves, props = _library(d)
            sum(res[k] for k in C.SCALAR_KEYS).backward()
        finally:
            torch.cuda.set_sync_debug_mode("default")
        runs.append([res[k] for k in C.SCALAR_KEYS] + [res["quantile"], leaves["pred"].grad, leaves["intensity"].grad,
                                                        leaves["logits"].grad, *[p.grad for p in props]])
    for a, b in zip(*runs):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    assert torch.equal(res["quantile_mask"], _library(d, requires_grad=False)[0]["quantile_mask"])


def test_operator_rejects_an_empty_batch(be):
    from neurad_studio_b200.lib import B200NerfError

    d = C.lidar_inputs(n=4, seed=14, device=DEV)
    e = {k: ([t[:0] for t in v] if isinstance(v, list) else v[:0]) for k, v in d.items()}
    with pytest.raises(B200NerfError):
        _library(e)


# ---------------------------------------------------------------------------------------------- end to end
def _model_and_batch(n_cam_patches=4, patch=(4, 4), n_lidar=2048):
    import neurad_studio_b200 as nsb
    from neurad_studio_b200 import scene
    from neurad_studio_b200.nerfstudio_api import NeuRADModel, RayBundle

    cfg = nsb.small_config(log2_main=14, log2_prop=13)
    model = NeuRADModel(cfg)
    model.load_reference_state_dict(scene.make_params(cfg, seed=1, beta=3.0, sdf_bias=0.6))
    model = model.to(DEV)
    model.requires_grad_(True)
    model.train()
    n_cam = n_cam_patches * patch[0] * patch[1]
    n = n_cam + n_lidar
    rays = scene.random_rays(n, cfg, seed=3)
    is_lidar = torch.zeros(n, 1, dtype=torch.bool)
    is_lidar[n_cam:] = True
    gen = torch.Generator().manual_seed(4)
    dist = 2 + 78 * torch.rand(n, 1, generator=gen)
    did_return = torch.rand(n, 1, generator=gen) < 0.9
    md = {"is_lidar": is_lidar.to(DEV), "sensor_idxs": rays["sensor_idx"].to(DEV), "directions_norm": dist.to(DEV),
          "did_return": did_return.to(DEV)}
    rb = RayBundle(origins=rays["origins"].to(DEV), directions=rays["directions"].to(DEV), pixel_area=rays["pixel_area"].to(DEV),
                   times=rays["times"].to(DEV), metadata=md, camera_indices=rays["sensor_idx"].reshape(-1, 1).long().to(DEV))
    up = cfg.rgb_upsample_factor
    batch = {"image": torch.rand(n_cam_patches, patch[0] * up, patch[1] * up, 3, generator=gen).to(DEV),
             "is_lidar": is_lidar.to(DEV), "did_return": did_return.to(DEV), "distance": dist[n_cam:].to(DEV),
             "lidar": torch.cat([torch.randn(n_lidar, 3, generator=gen), torch.rand(n_lidar, 1, generator=gen)], 1).to(DEV)}
    model.vgg_loss = lambda rgb, image: (rgb - image).abs().mean()  # a fixed stand-in perceptual loss
    return model, rb, batch, patch


def test_training_step_matches_the_torch_restatement(monkeypatch):
    from neurad_studio_b200 import losses as L

    model, rb, batch, patch = _model_and_batch()
    torch.manual_seed(0)
    outputs = model.get_outputs(rb, patch)
    params = [p for p in model.parameters() if p.requires_grad]

    def step():
        metrics = model.get_metrics_dict(outputs, batch)
        losses = model.get_loss_dict(outputs, batch, metrics)
        total = sum(losses.values())
        grads = torch.autograd.grad(total, params, retain_graph=True, allow_unused=True)
        return metrics, losses, total.detach(), grads

    m1, l1, t1, g1 = step()

    def torch_lidar_losses(pred, props, distance, did_return, intensity, gt_intensity, logits, nrd, nrm, q):
        m, quantile, mask = C.reference_lidar_terms(pred, list(props), distance, did_return, gt_intensity, intensity, logits,
                                                    nrd, nrm, q)
        return {**m, "quantile": quantile, "quantile_mask": mask}

    monkeypatch.setattr(L, "lidar_losses", torch_lidar_losses)
    m2, l2, t2, g2 = step()
    assert set(m1) == set(m2) and set(l1) == set(l2)
    assert {"depth_loss", "intensity_loss", "ray_drop_loss", "depth_loss_0", "depth_loss_1", "carving_loss", "vgg_loss",
            "rgb_loss", "interlevel_loss", "distortion_loss"} <= set(l1)
    assert abs(float(t1) - float(t2)) <= 1e-5 * abs(float(t2))
    for a, b in zip(g1, g2):
        if b is None:
            assert a is None or float(a.abs().max()) == 0.0
            continue
        assert float((a - b).abs().max()) <= 1e-5 * max(float(b.abs().max()), 1e-12)
    model._bind().check_status()


def test_vgg_mult_without_a_perceptual_loss_raises():
    model, rb, batch, patch = _model_and_batch(n_lidar=256)
    model.vgg_loss = None
    outputs = model.get_outputs(rb, patch)
    metrics = model.get_metrics_dict(outputs, batch)
    with pytest.raises(RuntimeError, match="vgg_loss"):
        model.get_loss_dict(outputs, batch, metrics)


# ---------------------------------------------------------------------------------------------- against the reference
@pytest.fixture(scope="module")
def golden():
    import os

    import numpy as np

    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "objective.npz")
    return dict(np.load(path, allow_pickle=False))


@pytest.mark.parametrize("name", C.GOLDEN_CASES)
def test_mirror_reproduces_the_reference_objective(golden, name):
    """The reference's own get_metrics_dict / get_loss_dict (oracle/make_golden_objective.py) on every case: key sets,
    values within 2e-6, gradients within 1e-6 of each tensor's max, quantile and mask bit for bit."""
    import neurad_studio_b200 as nsb
    from neurad_studio_b200.nerfstudio_api import NeuRADModel
    from oracle.make_golden_objective import SDF_BETA

    model = NeuRADModel(nsb.small_config()).to(DEV)
    with torch.no_grad():
        model._param("field.sdf_to_density.beta").fill_(SDF_BETA)
    C.check_mirror_against_golden(model, golden, name, DEV)
    model._bind().check_status()
