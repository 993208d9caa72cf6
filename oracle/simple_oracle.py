"""TEST INFRASTRUCTURE ONLY -- CPU restatement of BASELINE config 1 (the reference's own CPU-runnable case).

Config 1 (SURVEY.md 8(d)): 64x64 pinhole camera -> UniformSampler(32) -> positions normalised by an AABB -> torch-mode
HashEncoding (16 levels x 2 features, 2^19 entries) -> MLP 32 -> 64 -> 4 -> density = trunc_exp(o[0]), rgb =
sigmoid(o[1:4]) -> RaySamples.get_weights -> RGBRenderer("black") / DepthRenderer("expected") / AccumulationRenderer.
Everything here is in-tree reference code (no third-party arithmetic), so the restatement is pinned BIT FOR BIT against
the imported reference by oracle/make_golden_config1.py; the result is committed as tests/golden/config1.npz.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may import this module.
"""
from __future__ import annotations

from typing import Dict, Optional

import torch
from torch import Tensor

from oracle import neurad_oracle as O

SPACING_UNIFORM, SPACING_LINDISP, SPACING_POWER, SPACING_SQRT, SPACING_LOG = 0, 1, 2, 3, 4


def synthetic_table(n_rows: int, n_features: int, scale: float = 1.0) -> Tensor:
    """Deterministic, generator-independent stand-in for the reference's `torch.rand(...) * 2 - 1` table init
    (field_components/encodings.py:382-384; config 1 re-initialises the table ~U(-1,1), SURVEY 8(d)): an integer hash
    of the element index mapped to [-1, 1).  64 MB of table cannot be committed as a fixture; this can be re-created
    bit-identically anywhere."""
    i = torch.arange(n_rows * n_features, dtype=torch.int64) + 1
    x = (i * 0x9E3779B1) & 0xFFFFFFFF
    x = x ^ (x >> 15)
    x = (x * 0x85EBCA77) & 0xFFFFFFFF
    x = x ^ (x >> 13)
    u = x.double() / 4294967296.0
    return ((u * 2 - 1) * scale).float().view(n_rows, n_features)


def spacing_fns(kind: int, lam: float = -1.0, scaling: float = 0.1):
    """spacing_fn / spacing_fn_inv of the SpacedSampler subclasses (model_components/ray_samplers.py:135-156 Uniform,
    :159-180 LinearDisparity, :183-204 Sqrt, :207-228 Log, :838-852 Power)."""
    if kind == SPACING_UNIFORM:
        return (lambda x: x), (lambda x: x)
    if kind == SPACING_LINDISP:
        return (lambda x: 1 / x), (lambda x: 1 / x)
    if kind == SPACING_SQRT:
        return torch.sqrt, (lambda x: x**2)
    if kind == SPACING_LOG:
        return torch.log, torch.exp
    if kind == SPACING_POWER:
        return (lambda x: O.power_fn(x * scaling, lam)), (lambda x: O.inv_power_fn(x, lam) / scaling)
    raise ValueError(kind)


def spaced_sample(nears: Tensor, fars: Tensor, num_samples: int, kind: int = SPACING_UNIFORM, lam: float = -1.0,
                  scaling: float = 0.1, t_rand: Optional[Tensor] = None):
    """SpacedSampler.generate_ray_samples, eval mode (ray_samplers.py:80-132): returns (spacing bins [1,S+1],
    euclidean bins [N,S+1])."""
    fn, inv = spacing_fns(kind, lam, scaling)
    bins = torch.linspace(0.0, 1.0, num_samples + 1)[None, ...]
    if t_rand is not None:  # training mode, train_stratified (ray_samplers.py:107-115); t_rand [N,1] or [N,S+1]
        bin_centers = (bins[..., 1:] + bins[..., :-1]) / 2.0
        bin_upper = torch.cat([bin_centers, bins[..., -1:]], -1)
        bin_lower = torch.cat([bins[..., :1], bin_centers], -1)
        bins = bin_lower + (bin_upper - bin_lower) * t_rand
    s_near, s_far = fn(nears), fn(fars)
    euclid = inv(bins * s_far + (1 - bins) * s_near)
    return bins, euclid


def frustum_positions(origins: Tensor, directions: Tensor, starts: Tensor, ends: Tensor) -> Tensor:
    """Frustums.get_positions (cameras/rays.py:50-59) with [N,1,3] origins/directions and [N,S,1] starts/ends."""
    return origins[:, None, :] + directions[:, None, :] * (starts + ends) / 2


def normalized_positions(positions: Tensor, aabb: Tensor) -> Tensor:
    """SceneBox.get_normalized_positions (data/scene_box.py:63-79)."""
    lengths = aabb[1] - aabb[0]
    return (positions - aabb[0]) / lengths


def mlp_forward(weights, biases, x: Tensor) -> Tensor:
    """MLP.pytorch_fwd (field_components/mlp.py:142-178): ReLU between layers, no output activation."""
    for i, (w, b) in enumerate(zip(weights, biases)):
        x = torch.nn.functional.linear(x, w, b)
        if i < len(weights) - 1:
            x = torch.relu(x)
    return x


def rgb_render(rgb: Tensor, weights: Tensor, background: Optional[Tensor], training: bool = False) -> Tensor:
    """RGBRenderer.forward (model_components/renderers.py:233-268, combine_rgb :103-148): in eval mode nan_to_num of the
    samples' rgb and a clamp of the result to [0, 1]; in training mode neither."""
    if not training:
        rgb = torch.nan_to_num(rgb)
    comp = torch.sum(weights * rgb, dim=-2)
    if background is not None:  # None is "random": as if black, no blending
        comp = comp + background * (1.0 - torch.sum(weights, dim=-2))
    return comp if training else torch.clamp(comp, min=0.0, max=1.0)


def depth_expected(weights: Tensor, starts: Tensor, ends: Tensor) -> Tensor:
    """DepthRenderer("expected") (renderers.py:396-416), including the GLOBAL clip to [steps.min(), steps.max()]."""
    steps = (starts + ends) / 2
    depth = torch.sum(weights * steps, dim=-2) / (torch.sum(weights, -2) + 1e-10)
    return torch.clip(depth, steps.min(), steps.max())


def depth_median(weights: Tensor, starts: Tensor, ends: Tensor) -> Tensor:
    """DepthRenderer("median") (renderers.py:383-394)."""
    steps = (starts + ends) / 2
    cum = torch.cumsum(weights[..., 0], dim=-1)
    split = torch.ones((*weights.shape[:-2], 1)) * 0.5
    idx = torch.searchsorted(cum, split, side="left")
    idx = torch.clamp(idx, 0, steps.shape[-2] - 1)
    return torch.gather(steps[..., 0], dim=-1, index=idx)


def config1_render(p: Dict[str, Tensor], origins: Tensor, directions: Tensor, nears: Tensor, fars: Tensor,
                   num_samples: int = 32, want_trace: bool = False) -> Dict[str, Tensor]:
    """The whole of config 1.  `p`: hash_table [L*T,F], scalings [L], mlp w0,b0,w1,b1, aabb [2,3]; rays [N,3]/[N,1]."""
    bins_s, bins_e = spaced_sample(nears, fars, num_samples)
    starts, ends = bins_e[..., :-1, None], bins_e[..., 1:, None]
    pos = frustum_positions(origins, directions, starts, ends)
    x = normalized_positions(pos, p["aabb"])
    table_size = p["hash_table"].shape[0] // p["scalings"].shape[0]
    enc = O.hash_encode(x.reshape(-1, 3), p["hash_table"], p["scalings"], table_size)
    raw = mlp_forward([p["w0"], p["w1"]], [p["b0"], p["b1"]], enc).view(*x.shape[:-1], -1)
    density = torch.exp(raw[..., 0:1])  # trunc_exp forward (field_components/activations.py:28-35)
    rgb = torch.sigmoid(raw[..., 1:4])
    weights = O.weights_from_density((ends - starts)[..., 0], density[..., 0])[..., None]
    out = {
        "rgb": rgb_render(rgb, weights, torch.zeros(3)),
        "depth": depth_expected(weights, starts, ends),
        "accumulation": torch.sum(weights, dim=-2),
    }
    if want_trace:
        out.update(bins_e=bins_e, positions=x, encoding=enc.view(*x.shape[:-1], -1), raw=raw, density=density,
                   rgb_samples=rgb, weights=weights, depth_median=depth_median(weights, starts, ends))
    return out
