"""Shared bodies of the objective tests (tests/test_objective_cpu.py, tests/test_zz_objective_gpu.py): seeded lidar-row
inputs, adversarial inputs of the order statistic, and the reference's lidar terms (models/neurad.py:486-520) restated
line by line in torch, so that torch autograd gives the gradients the library's backward must reproduce."""
from typing import Dict, List, Sequence, Tuple

import torch
import torch.nn.functional as F
from torch import Tensor

NON_RETURN_LIDAR_DISTANCE = 150.0  # LossSettings defaults (neurad.py:81, 87, 89)
NON_RETURN_LOSS_MULT = 0.1
QUANTILE_THRESHOLD = 0.95
ROUNDS = 2
SCALAR_KEYS = ["depth_loss", "intensity_loss", "ray_drop_loss"] + [f"depth_loss_{i}" for i in range(ROUNDS)]


def lidar_inputs(n: int, seed: int, return_frac: float = 0.9, nan_at: Sequence[int] = (), repeat: bool = False,
                 device="cpu") -> Dict[str, Tensor]:
    """Lidar rows of a training batch: distances 1-80 m, about 10 % non-returns of which about a third are predicted
    beyond the 150 m non-return distance, intensities in [0, 1], ray-drop logits.  `repeat`: depths on a 0.25 m grid,
    so that many loss values are equal and ties straddle the quantile.  `nan_at`: NaN predicted depths."""
    g = torch.Generator().manual_seed(seed)
    u = lambda *s: torch.rand(*s, generator=g)  # noqa: E731
    distance = 1 + 79 * u(n, 1)
    did_return = u(n) < return_frac
    pred = distance + 2 * (u(n, 1) - 0.5)
    nonret = ~did_return
    pred[nonret] = torch.where(u(n, 1)[nonret] < 0.35, 150 + 60 * u(n, 1)[nonret], 20 + 120 * u(n, 1)[nonret])
    props = [pred + 6 * (u(n, 1) - 0.5) for _ in range(ROUNDS)]
    if repeat:
        distance = distance.round()
        pred = (pred * 4).round() / 4
        props = [(p * 4).round() / 4 for p in props]
    for i in nan_at:
        pred[i] = float("nan")
    lidar = torch.cat([50 * (u(n, 3) - 0.5), u(n, 1)], dim=1)  # x, y, z, intensity
    d = {"pred": pred, "props": props, "distance": distance, "did_return": did_return, "lidar": lidar,
         "intensity": u(n, 1), "logits": 3 * torch.randn(n, 1, generator=g)}
    return {k: ([t.to(device) for t in v] if isinstance(v, list) else v.to(device)) for k, v in d.items()}


def reference_lidar_terms(pred_depth: Tensor, prop_depths: List[Tensor], termination_depth: Tensor, did_return: Tensor,
                          points_intensities: Tensor, intensity: Tensor, ray_drop_logits: Tensor,
                          non_return_lidar_distance: float = NON_RETURN_LIDAR_DISTANCE,
                          non_return_loss_mult: float = NON_RETURN_LOSS_MULT,
                          quantile_threshold: float = QUANTILE_THRESHOLD) -> Tuple[Dict[str, Tensor], Tensor, Tensor]:
    """neurad.py:486-520, lidar rows ([n,1] tensors, did_return [n] bool): (metrics, quantile, quantile_mask)."""
    m = {}
    nonret_lid_dist = torch.tensor(non_return_lidar_distance, device=termination_depth.device)
    target_depth = termination_depth.clone()
    target_depth[~did_return] = pred_depth.detach()[~did_return].maximum(nonret_lid_dist)
    unreduced_depth_loss = F.l1_loss(target_depth, pred_depth, reduction="none")
    unreduced_depth_loss[~did_return] *= non_return_loss_mult
    quantile = torch.quantile(unreduced_depth_loss, quantile_threshold)
    quantile_mask = (unreduced_depth_loss < quantile).squeeze(-1)
    m["depth_loss"] = torch.mean(unreduced_depth_loss[quantile_mask])
    quant_and_return = quantile_mask & did_return
    m["intensity_loss"] = F.mse_loss(points_intensities[quant_and_return], intensity[quant_and_return], reduction="none").mean()
    m["ray_drop_loss"] = F.binary_cross_entropy_with_logits(ray_drop_logits, (~did_return).unsqueeze(-1).to(ray_drop_logits))
    for prop_i, p in enumerate(prop_depths):
        target_depth = termination_depth.clone()
        target_depth[~did_return] = p.detach()[~did_return].maximum(nonret_lid_dist)
        unreduced = F.l1_loss(target_depth, p, reduction="none")
        unreduced[~did_return] *= non_return_loss_mult
        m[f"depth_loss_{prop_i}"] = torch.mean(unreduced)
    return m, quantile.detach(), quantile_mask


def order_statistic_inputs() -> Dict[str, Tensor]:
    """Adversarial inputs of the selection: ties, duplicates at the rank, +-inf, NaN, denormals, negative values, ranks
    with and without a fractional part (0.95 (n - 1) is integral at n = 21, 41)."""
    g = torch.Generator().manual_seed(7)
    tiny = torch.finfo(torch.float32).tiny
    cases = {
        "n1": torch.tensor([3.5]),
        "n2": torch.tensor([2.0, -1.0]),
        "n3": torch.tensor([1.0, 1.0, 0.5]),
        "n21": torch.rand(21, generator=g),
        "n41": torch.rand(41, generator=g),
        "n40": torch.rand(40, generator=g),
        "ties": torch.randint(0, 4, (1000,), generator=g).float(),
        "all_equal": torch.full((257,), 0.3),
        "dup_at_rank": torch.cat([torch.rand(95, generator=g), torch.full((10,), 2.0), 3 + torch.rand(5, generator=g)]),
        "inf": torch.cat([torch.rand(50, generator=g), torch.tensor([float("inf")] * 6 + [float("-inf")] * 3)]),
        "nan": torch.cat([torch.rand(60, generator=g), torch.tensor([float("nan")])]),
        "denormal": torch.cat([torch.rand(30, generator=g) * tiny, torch.tensor([0.0, tiny / 8, tiny * 3])]),
        "signed": torch.randn(999, generator=g) * 1e3,
        "prefix_edge": torch.tensor([1.0, 1.0 + 2 ** -23, 1.0009765625, 2.0] * 5),  # keys that end one 10-bit prefix
        "wide": torch.cat([torch.randn(500, generator=g), torch.randn(500, generator=g) * 1e30]),
    }
    return cases


QS = [0.95, 0.0, 0.5, 1.0, 0.3]


# ---------------------------------------------------------------------------------------------- tests/golden/objective.npz
def golden_case(golden, name: str, device):
    """(outputs, batch, sdists, weights, training) of one case of oracle/make_golden_objective.py."""
    p = name + "_"

    def group(tag):
        return {k[len(p + tag):]: torch.from_numpy(v).to(device) for k, v in golden.items() if k.startswith(p + tag)}

    n_levels = sum(1 for k in golden if k.startswith(p + "sdist_"))
    sdists = [torch.from_numpy(golden[p + f"sdist_{i}"]).to(device) for i in range(n_levels)]
    weights = [torch.from_numpy(golden[p + f"weights_{i}"]).to(device) for i in range(n_levels)]
    return group("out_"), group("in_"), sdists, weights, bool(golden[p + "training"])


def _close(got: float, want: float, rel: float) -> bool:
    if want != want:
        return got != got
    return abs(got - want) <= rel * abs(want) + 1e-30


def check_mirror_against_golden(model, golden, name: str, device, scalar_rel: float = 2e-6, grad_rel: float = 1e-6):
    """The mirror's get_metrics_dict / get_loss_dict on a golden case: the reference's key sets, every value within
    `scalar_rel`, every gradient of the summed loss dict within `grad_rel` of its tensor's max, and the lidar losses'
    quantile and mask bit for bit."""
    from neurad_studio_b200 import losses as L
    from oracle.make_golden_objective import GRAD_KEYS, SpacingBins, vgg_stand_in

    p = name + "_"
    outputs, batch, sdists, weights, training = golden_case(golden, name, device)
    model.train(training)
    model.vgg_loss = vgg_stand_in
    outs = {k: v.clone().requires_grad_(True) for k, v in outputs.items()}
    wl = [w.clone().requires_grad_(True) for w in weights]
    if wl:
        outs["weights_list"], outs["ray_samples_list"] = wl, [SpacingBins(s) for s in sdists]
    metrics = model.get_metrics_dict(outs, dict(batch))
    losses = model.get_loss_dict(outs, dict(batch), metrics)
    assert sorted(metrics) == list(golden[p + "metric_keys"])
    assert sorted(losses) == list(golden[p + "loss_keys"])
    for kind, d in (("metric_", metrics), ("loss_", losses)):
        for k, v in d.items():
            want = float(golden[p + kind + k])
            assert _close(float(v), want, scalar_rel), (kind + k, float(v), want)
    leaves = {k: outs[k] for k in GRAD_KEYS if k in outs}
    leaves.update({f"weights_list_{i}": w for i, w in enumerate(wl)})
    got = torch.autograd.grad(sum(losses.values()), list(leaves.values()), allow_unused=True)
    for (k, t), g in zip(leaves.items(), got):
        g = torch.zeros_like(t) if g is None else g
        want = torch.from_numpy(golden[p + "grad_" + k]).to(device)
        tol = grad_rel * max(float(want.abs().max()), 1e-30)
        assert float((g - want).abs().max()) <= tol, (k, float((g - want).abs().max()), tol)
    if p + "quantile" in golden:
        is_lidar = batch["is_lidar"][:, 0]
        with torch.no_grad():
            res = L.lidar_losses(outputs["depth"][is_lidar], [outputs[f"prop_depth_{i}"][is_lidar] for i in range(ROUNDS)],
                                 batch["distance"], batch["did_return"][is_lidar][:, 0], outputs["intensity"],
                                 batch["lidar"][:, 3:4], outputs["ray_drop_logits"])
        want_q = torch.from_numpy(golden[p + "quantile"]).reshape(-1)
        got_q = res["quantile"].reshape(-1).cpu()
        assert torch.equal(got_q.view(torch.int32), want_q.view(torch.int32)) or (got_q.isnan() & want_q.isnan()).all()
        assert torch.equal(res["quantile_mask"].cpu(), torch.from_numpy(golden[p + "quantile_mask"]))
    return metrics, losses


GOLDEN_CASES = ["mixed", "repeated", "n21", "n41", "n40", "n1", "n2", "all_returns", "no_returns", "nan", "camera_only",
                "lidar_only", "eval"]
