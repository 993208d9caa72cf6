"""TEST INFRASTRUCTURE ONLY -- CPU oracle for NeuRAD's volumetric-rendering hot path.

This file is a restatement, in plain torch-CPU fp32 tensor ops, of the path that
``NeuRADModel.get_nff_outputs`` (reference ``nerfstudio/models/neurad.py:368-421``) executes in eval mode with
``implementation="torch"``.  Every function cites the reference lines it follows and deliberately uses the SAME
torch elementwise op sequence as the reference (no algebraic simplification, no fused multiply-add), so that on a
CPU it reproduces the reference bit for bit wherever the reference itself is deterministic.

Who may use it: ``tests/``, ``__graft_entry__.smoke()`` and the ``cpu_baseline`` / ``--impl reference`` legs of
``bench.py`` -- as the checker or the timed baseline, never as the product.  Nothing under
``neurad-studio_b200/`` imports this module; the product path is the sm_90a CUDA library and it fails loudly
when that library is missing.

Pinning status: the reference's own tests hold NO golden vector for this path (SURVEY.md section 8c), so the
oracle is pinned against outputs of the reference itself: ``oracle/make_golden.py`` imports the unmodified
reference from /root/reference (build container only), runs it on seeded inputs and commits the input/output
vectors under ``tests/golden/``; ``tests/test_oracle_golden.py`` checks this restatement against them.

Third-party arithmetic that is NOT in the reference tree and is therefore restated from its published
definition (nerfacc==0.5.2, ``pyproject.toml:36``):
  * ``nerfacc.render_weight_from_alpha`` (call site neurad.py:717): w_i = alpha_i * prod_{j<i}(1 - alpha_j)
  * ``nerfacc.accumulate_along_rays``    (call site neurad.py:734): sum_i w_i * v_i over the sample axis
These two are PARITY UNPINNED: nerfacc cannot be installed here (no network) and neither the reference's tests nor its
tree hold a vector for them, so they follow nerfacc's documented dense-tensor semantics; the in-tree twins of the same
formulas (cameras/rays.py:188-210, model_components/renderers.py:85,412) agree with them.  Everything else in this file is
pinned against the reference run.  The reference's CPU debugging branch that returns constant 0.5 weights
(neurad.py:713-715) is bypassed.

Backward pass (SURVEY 8f row f2): torch autograd through these functions is pinned against the reference's own autograd
(oracle/make_golden_grads.py -> tests/golden/grads_*.npz); the backward of ``render_weight_from_alpha`` is therefore
autograd of the cumprod restatement above, not nerfacc's CUDA backward (unpinned for the same reason).
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple

import numpy as np
import torch
import torch.nn.functional as F
from torch import Tensor

EPS = 1.0e-7  # neurad_encoding.py:31, neurad_field.py:42
_NORM_EPS = float(np.finfo(float).eps * 4.0)  # cameras/camera_utils.py:30


# ----------------------------------------------------------------------------------------------------------------------
# configuration (defaults = the reference's `neurad` method defaults)
# ----------------------------------------------------------------------------------------------------------------------
@dataclass
class GridCfg:
    """One HashEncoding (field_components/encodings.py:326-352)."""

    num_levels: int
    min_res: int
    max_res: int
    log2_hashmap_size: int
    features_per_level: int

    @property
    def table_size(self) -> int:
        return 2**self.log2_hashmap_size

    def scalings(self) -> Tensor:
        # encodings.py:348-350 -- evaluated with the very same expression so the buffer matches the reference's
        levels = torch.arange(self.num_levels)
        growth = (
            np.exp((np.log(self.max_res) - np.log(self.min_res)) / (self.num_levels - 1))
            if self.num_levels > 1
            else 1.0
        )
        return torch.floor(self.min_res * growth**levels)


@dataclass
class FieldCfg:
    static: GridCfg
    actor: GridCfg
    actor_scale: float = 10.0  # neurad_encoding.py:52


def main_field_cfg() -> FieldCfg:
    # neurad_encoding.py:34-66
    return FieldCfg(static=GridCfg(8, 32, 8192, 22, 4), actor=GridCfg(4, 64, 1024, 17, 4))


def proposal_field_cfg() -> FieldCfg:
    # neurad_field.py:161-179
    return FieldCfg(static=GridCfg(6, 128, 4096, 20, 1), actor=GridCfg(4, 64, 1024, 15, 1))


@dataclass
class NeuRADCfg:
    """Subset of NeuRADModelConfig / SamplingSettings / NeuRADFieldConfig that shapes the forward path."""

    main: FieldCfg = field(default_factory=main_field_cfg)
    prop: Tuple[FieldCfg, FieldCfg] = field(default_factory=lambda: (proposal_field_cfg(), proposal_field_cfg()))
    num_proposal_samples: Tuple[int, int] = (128, 64)  # neurad.py:108
    num_nerf_samples: int = 32  # neurad.py:110
    power_lambda: float = -1.0  # neurad.py:112
    power_scaling: float = 0.1  # neurad.py:114
    sky_distance: float = 20000.0  # neurad.py:116
    appearance_dim: int = 16  # neurad.py:134
    temporal_appearance_freq: float = 1.0  # neurad.py:138
    rgb_upsample_factor: int = 3  # neurad.py:141
    nff_out_dim: int = 32  # neurad_field.py:64
    geo_hidden_dim: int = 32
    nff_hidden_dim: int = 32
    histogram_padding: float = 0.01  # ray_samplers.py:272
    actor_bbox_padding: Tuple[float, float, float] = (0.25, 0.25, 0.1)  # dynamic_actors.py:39
    # scene
    static_scale: float = 100.0  # scene_box.aabb.max(), neurad.py:182
    duration: float = 8.0  # dataset metadata, neurad.py:188
    num_sensors: int = 7
    n_actors: int = 0

    @property
    def embeds_per_sensor(self) -> int:
        return math.ceil(self.duration * self.temporal_appearance_freq)  # neurad.py:191


# ----------------------------------------------------------------------------------------------------------------------
# sampling
# ----------------------------------------------------------------------------------------------------------------------
def power_fn(x: Tensor, lam: float) -> Tensor:
    """utils/math.py:541-558 (general branch)."""
    lam_1 = abs(lam - 1)
    return (lam_1 / lam) * ((x / lam_1 + 1) ** lam - 1)


def inv_power_fn(x: Tensor, lam: float, eps: float = 1e-10) -> Tensor:
    """utils/math.py:561-579 (general branch)."""
    lam_1 = abs(lam - 1)
    return ((x * lam / lam_1 + 1).clamp_min(eps) ** (1 / lam) - 1) * lam_1


class SpacingFns:
    """PowerSampler's spacing_fn / spacing_fn_inv (ray_samplers.py:846-852) bound to a ray batch
    (ray_samplers.py:117-122)."""

    def __init__(self, cfg: NeuRADCfg, nears: Tensor, fars: Tensor):
        self.lam, self.scaling = cfg.power_lambda, cfg.power_scaling
        self.s_near = power_fn(nears * self.scaling, self.lam)
        self.s_far = power_fn(fars * self.scaling, self.lam)

    def to_euclidean(self, x: Tensor) -> Tensor:
        return inv_power_fn(x * self.s_far + (1 - x) * self.s_near, self.lam) / self.scaling


def initial_bins(cfg: NeuRADCfg, sp: SpacingFns, num_samples: int) -> Tuple[Tensor, Tensor]:
    """SpacedSampler.generate_ray_samples in eval mode (ray_samplers.py:80-132).
    Returns (spacing bins [1,S+1], euclidean bins [N,S+1])."""
    bins = torch.linspace(0.0, 1.0, num_samples + 1)[None, ...]
    return bins, sp.to_euclidean(bins)


def pdf_u(num_samples: int) -> Tensor:
    """The eval-mode quantiles of PDFSampler (ray_samplers.py:332-336)."""
    num_bins = num_samples + 1
    u = torch.linspace(0.0, 1.0 - (1.0 / num_bins), steps=num_bins)
    return u + 1.0 / (2 * num_bins)


def pdf_resample(
    weights: Tensor, existing_bins: Tensor, num_samples: int, histogram_padding: float = 0.01, eps: float = 1e-5,
    rand: Optional[Tensor] = None,
) -> Dict[str, Tensor]:
    """PDFSampler.generate_ray_samples, eval mode, include_original=False (ray_samplers.py:280-361).

    weights [N,S]; existing_bins [N,S+1] (spacing domain).  Returns new spacing bins [N,num_samples+1] plus the
    intermediate cdf and searchsorted indices (the bit-exact targets).  `rand` switches to the training-mode
    stratified quantiles."""
    num_bins = num_samples + 1
    weights = weights + histogram_padding
    weights_sum = torch.sum(weights, dim=-1, keepdim=True)
    padding = torch.relu(eps - weights_sum)
    weights = weights + padding / weights.shape[-1]
    weights_sum = weights_sum + padding
    pdf = weights / weights_sum
    cdf = torch.min(torch.ones_like(pdf), torch.cumsum(pdf, dim=-1))
    cdf = torch.cat([torch.zeros_like(cdf[..., :1]), cdf], dim=-1)
    if rand is None:
        u = pdf_u(num_samples).expand(size=(*cdf.shape[:-1], num_bins)).clone().contiguous()
    else:  # training mode, train_stratified (ray_samplers.py:321-329); rand [N,1] (single_jitter) or [N,num_bins] in [0,1)
        u = torch.linspace(0.0, 1.0 - (1.0 / num_bins), steps=num_bins)
        u = u.expand(size=(*cdf.shape[:-1], num_bins)).clone()
        u = (u + rand / num_bins).contiguous()
    inds = torch.searchsorted(cdf, u, side="right")
    below = torch.clamp(inds - 1, 0, existing_bins.shape[-1] - 1)
    above = torch.clamp(inds, 0, existing_bins.shape[-1] - 1)
    cdf_g0 = torch.gather(cdf, -1, below)
    bins_g0 = torch.gather(existing_bins, -1, below)
    cdf_g1 = torch.gather(cdf, -1, above)
    bins_g1 = torch.gather(existing_bins, -1, above)
    t = torch.clip(torch.nan_to_num((u - cdf_g0) / (cdf_g1 - cdf_g0), 0), 0, 1)
    bins = bins_g0 + t * (bins_g1 - bins_g0)
    return {"bins": bins, "cdf": cdf, "inds": inds}


def weights_from_density(deltas: Tensor, densities: Tensor) -> Tensor:
    """RaySamples.get_weights (cameras/rays.py:188-210) on [N,S] tensors."""
    delta_density = deltas * densities
    alphas = 1 - torch.exp(-delta_density)
    transmittance = torch.cumsum(delta_density[..., :-1], dim=-1)
    transmittance = torch.cat([torch.zeros((*transmittance.shape[:1], 1)), transmittance], dim=-1)
    transmittance = torch.exp(-transmittance)
    return torch.nan_to_num(alphas * transmittance)


# ----------------------------------------------------------------------------------------------------------------------
# gaussians, contraction, hash grid
# ----------------------------------------------------------------------------------------------------------------------
def fast_isotropic_gaussian(
    origins: Tensor, directions: Tensor, pixel_area: Tensor, starts: Tensor, ends: Tensor, num_multisamples: int = 1
) -> Tuple[Tensor, Tensor]:
    """Frustums.get_fast_isotropic_gaussian (cameras/rays.py:109-124).

    origins/directions [N,1,3] (broadcast over samples), pixel_area [N,1,1], starts/ends [N,S,1].
    Returns mean [N,S,M,3], std [N,S,M,1]."""
    multisample_dist = (ends - starts) / (num_multisamples + 1)
    ts = torch.arange(1, num_multisamples + 1, dtype=ends.dtype)
    t = starts + ts.unsqueeze(0) * multisample_dist
    mean = origins.unsqueeze(-2) + directions.unsqueeze(-2) * t.unsqueeze(-1)
    frust_crossection_area = pixel_area.unsqueeze(-2) * t.unsqueeze(-1).pow(2)
    std = (frust_crossection_area * multisample_dist.unsqueeze(-2)).pow(1 / 3)
    return mean, std


def scaled_contraction(mean: Tensor, std: Tensor, scale) -> Tuple[Tensor, Tensor]:
    """ScaledSceneContraction(order=inf, normalize=True) on a GaussiansStd
    (field_components/spatial_distortions.py:103-114, 132-136)."""
    means = (mean / scale).clone()
    std = (std / scale).clone()
    mag = torch.linalg.norm(means, ord=float("inf"), dim=-1)[..., None]
    mask = mag < 1
    clamped_mag = mag.clamp_min(1.0)
    means = torch.where(mask, means, (2 - (1 / clamped_mag)) * (means / clamped_mag))
    std_scaling = ((2 * clamped_mag - 1).pow(1 / 3) / clamped_mag) ** 2
    std = torch.where(mask, std, std * std_scaling)
    means = (means + 2.0) / 4.0
    std = std / 4.0
    return means, std


_HASH_PRIMES = (1, 2654435761, 805459861)  # encodings.py:418


def hash_indices(x: Tensor, scalings: Tensor, table_size: int) -> Tuple[Tensor, Tensor]:
    """HashEncoding.hash_fn + corner ordering of pytorch_fwd (encodings.py:406-444).
    x [P,3] in [0,1].  Returns (indices [P,L,8] int64 into the [L*T,F] table, offset [P,L,3])."""
    num_levels = scalings.shape[0]
    x = x[..., None, :]
    scaled = x * scalings.view(-1, 1)
    scaled_c = torch.ceil(scaled).type(torch.int32)
    scaled_f = torch.floor(scaled).type(torch.int32)
    offset = scaled - scaled_f
    hash_offset = torch.arange(num_levels) * table_size

    def hash_fn(t):
        t = t * torch.tensor(_HASH_PRIMES)
        h = torch.bitwise_xor(t[..., 0], t[..., 1])
        h = torch.bitwise_xor(h, t[..., 2])
        h %= table_size
        h += hash_offset
        return h

    c, f = scaled_c, scaled_f
    cx, cy, cz = c[..., 0:1], c[..., 1:2], c[..., 2:3]
    fx, fy, fz = f[..., 0:1], f[..., 1:2], f[..., 2:3]
    hashed = [
        hash_fn(c),  # 0: c c c
        hash_fn(torch.cat([cx, fy, cz], dim=-1)),  # 1
        hash_fn(torch.cat([fx, fy, cz], dim=-1)),  # 2
        hash_fn(torch.cat([fx, cy, cz], dim=-1)),  # 3
        hash_fn(torch.cat([cx, cy, fz], dim=-1)),  # 4
        hash_fn(torch.cat([cx, fy, fz], dim=-1)),  # 5
        hash_fn(f),  # 6
        hash_fn(torch.cat([fx, cy, fz], dim=-1)),  # 7
    ]
    return torch.stack(hashed, dim=-1), offset


def hash_encode(x: Tensor, table: Tensor, scalings: Tensor, table_size: int) -> Tensor:
    """HashEncoding.pytorch_fwd (encodings.py:425-466).  x [P,3] -> [P, L*F]."""
    idx, offset = hash_indices(x, scalings, table_size)
    f_0, f_1, f_2, f_3, f_4, f_5, f_6, f_7 = (table[idx[..., i]] for i in range(8))
    ox, oy, oz = offset[..., 0:1], offset[..., 1:2], offset[..., 2:3]
    f_03 = f_0 * ox + f_3 * (1 - ox)
    f_12 = f_1 * ox + f_2 * (1 - ox)
    f_56 = f_5 * ox + f_6 * (1 - ox)
    f_47 = f_4 * ox + f_7 * (1 - ox)
    f0312 = f_03 * oy + f_12 * (1 - oy)
    f4756 = f_47 * oy + f_56 * (1 - oy)
    encoded_value = f0312 * oz + f4756 * (1 - oz)
    return torch.flatten(encoded_value, start_dim=-2, end_dim=-1)


def rescale_grid_features(grid_features: Tensor, mean: Tensor, std: Tensor, scalings: Tensor, F_: int) -> Tensor:
    """NeuRADHashEncoding._rescale_grid_features (neurad_encoding.py:297-304): anti-aliasing down-weighting."""
    prefix_shape = list(mean.shape[:-1])
    L = scalings.shape[0]
    grid_feats = grid_features.view(prefix_shape + [L * F_]).unflatten(-1, (L, F_))
    weights = 1 / (scalings * 2 * std).clamp_min(1.0)
    return (grid_feats * weights[..., None]).mean(dim=-3).flatten(-2, -1)


# ----------------------------------------------------------------------------------------------------------------------
# dynamic actors
# ----------------------------------------------------------------------------------------------------------------------
def rotation_6d_to_matrix(d6: Tensor) -> Tensor:
    """cameras/camera_utils.py:422-443."""
    a1, a2 = d6[..., :3], d6[..., 3:]
    b1 = F.normalize(a1, dim=-1)
    b2 = a2 - (b1 * a2).sum(-1, keepdim=True) * b1
    b2 = F.normalize(b2, dim=-1)
    b3 = torch.cross(b1, b2, dim=-1)
    return torch.stack((b1, b2, b3), dim=-2)


def interpolate_trajectories_6d(poses: Tensor, pose_times: Tensor, query_times: Tensor, pose_valid_mask: Tensor):
    """utils/poses.py:90-150 with flatten=False.  poses [T,A,9]; returns ([Q,A,9], valid [Q,A])."""
    a1 = F.normalize(poses[..., :3], dim=-1)
    a2 = poses[..., 3:6]
    a2 = a2 - (a1 * a2).sum(-1, keepdim=True) * a1
    a2 = F.normalize(a2, dim=-1)
    positions = poses[..., 6:9]
    poses = torch.cat([a1, a2, positions], dim=-1)
    query_times = query_times.squeeze(-1)
    right_idx = torch.searchsorted(pose_times, query_times)
    left_idx = (right_idx - 1).clamp(min=0)
    right_idx = right_idx.clamp(max=len(pose_times) - 1)
    right_time = pose_times[right_idx]
    left_time = pose_times[left_idx]
    time_diff = right_time - left_time + 1e-6
    fraction = (query_times - left_time) / time_diff
    fraction = fraction.clamp(0.0, 1.0)
    trajs_to_sample = pose_valid_mask[left_idx] | pose_valid_mask[right_idx]
    poses_left = poses[left_idx]
    poses_right = poses[right_idx]
    interpolated = poses_left + (poses_right - poses_left) * fraction.unsqueeze(-1).unsqueeze(-1)
    return interpolated, trajs_to_sample


def boxes2world_at(params: Dict[str, Tensor], query_times: Tensor) -> Tuple[Tensor, Tensor]:
    """DynamicActors.get_boxes2world(flatten=False), eval, no actor editing (dynamic_actors.py:251-268).
    Returns ([Q,A,4,4], valid [Q,A])."""
    poses9 = torch.cat([params["dynamic_actors.actor_rotations_6d"], params["dynamic_actors.actor_positions"]], dim=-1)
    poses, valid = interpolate_trajectories_6d(
        poses9,
        params["dynamic_actors.unique_timestamps"],
        query_times,
        params["dynamic_actors.actor_present_at_time"],
    )
    b2w = torch.cat([rotation_6d_to_matrix(poses[..., :6]), poses[..., 6:].unsqueeze(-1)], dim=-1)
    constants = torch.zeros_like(b2w[..., :1, :])
    constants[..., :, 3] = 1
    return torch.cat([b2w, constants], dim=-2), valid  # utils/poses.py:28-39


def pose_inverse(pose: Tensor) -> Tensor:
    """utils/poses.py:42-55."""
    R = pose[..., :3, :3]
    t = pose[..., :3, 3:]
    R_inverse = R.transpose(-2, -1)
    t_inverse = -R_inverse.matmul(t)
    return torch.cat([R_inverse, t_inverse], dim=-1)


def transform_points_pairwise(points: Tensor, transforms: Tensor, with_translation: bool = True) -> Tensor:
    """cameras/lidars.py:549-564."""
    rotations = transforms[..., :3, :3]
    translations = transforms[..., :3, 3]
    rotated = torch.bmm(rotations.reshape(-1, 3, 3), points.reshape(-1, 3, 1)).reshape(*points.shape[:-1], 3)
    return rotated + translations if with_translation else rotated


def actor_indices(pos: Tensor, boxes2world: Tensor, valid: Tensor, world2boxes: Tensor, actor_bounds: Tensor):
    """NeuRADHashEncoding._get_actor_indices (neurad_encoding.py:225-263).  pos [N,S,M,3]."""
    actor_radii = actor_bounds.norm(dim=-1)
    sample_mean_pos = pos.mean(-2)
    point_on_line = sample_mean_pos[:, 0, :]
    line_direction = sample_mean_pos[:, -1, :] - point_on_line
    line_direction = line_direction / (torch.linalg.norm(line_direction, dim=-1, keepdim=True) + EPS)
    line_direction = line_direction.unsqueeze(-2)
    vec_from_line = boxes2world[..., :3, 3] - point_on_line.unsqueeze(-2)
    cross_prod = torch.cross(vec_from_line, line_direction.expand_as(vec_from_line), dim=-1)
    distance = torch.linalg.norm(cross_prod, dim=-1)
    close = (distance < actor_radii) & valid
    ray_idx, actor_idx = close.nonzero(as_tuple=False).T
    sample_pos = sample_mean_pos[ray_idx]
    actor_pos = boxes2world[ray_idx, actor_idx, :3, 3].unsqueeze(-2).repeat(1, sample_pos.shape[-2], 1)
    distance = torch.linalg.norm(sample_pos - actor_pos, dim=-1)
    within = (distance < actor_radii[actor_idx].unsqueeze(-1)).nonzero(as_tuple=False)
    indices = torch.stack([ray_idx[within[:, 0]], within[:, 1], actor_idx[within[:, 0]]], dim=-1)
    selected_smp = sample_mean_pos[indices[:, 0], indices[:, 1]]
    selected_w2b = world2boxes[indices[:, 0], indices[:, 2]]
    pos_in_box = transform_points_pairwise(selected_smp, selected_w2b)
    inside_box = (pos_in_box.abs() < actor_bounds[indices[:, 2]]).all(dim=-1)
    indices = indices[inside_box]
    return indices[:, 0], indices[:, 1], indices[:, 2]


# ----------------------------------------------------------------------------------------------------------------------
# NeuRADHashEncoding.forward  (static grid + per-actor grids, torch mode)
# ----------------------------------------------------------------------------------------------------------------------
def hashgrid_forward(
    params: Dict[str, Tensor],
    prefix: str,
    fcfg: FieldCfg,
    cfg: NeuRADCfg,
    mean: Tensor,
    std: Tensor,
    times: Tensor,
    directions: Optional[Tensor],
    trace: Optional[dict] = None,
    flip: Optional[Tensor] = None,
    require_actor_grad: bool = True,
) -> Tuple[Tensor, Optional[Tensor]]:
    """neurad_encoding.py:150-223, 265-304.  mean [N,S,M,3], std [N,S,M,1], times [N,S,1], directions [N,S,3] or None.
    `flip` [N] (+1 / -1 per ray) is the training-mode random actor flip (:212-219, drawn with torch.bernoulli there);
    None = eval mode.  Returns (features [N*S, L*F], directions [N,S,3] | None)."""
    sg, ag = fcfg.static, fcfg.actor
    s_scal = params[f"{prefix}.hashgrid.static_grid.scalings"]
    c_mean, c_std = scaled_contraction(mean, std, params["static_scale"])
    tcnn = f"{prefix}.hashgrid.static_grid.tcnn_encoding.params" in params  # SURVEY 8f row f3 (parity unpinned)
    if tcnn:
        from . import tcnn_oracle as T

        def tcnn_grid(g: GridCfg, key: str, x: Tensor, n_dims: int) -> Tensor:
            growth = float(np.exp((np.log(g.max_res) - np.log(g.min_res)) / (g.num_levels - 1))) if g.num_levels > 1 else 1.0
            lay = T.grid_layout(g.num_levels, g.features_per_level, g.log2_hashmap_size, g.min_res, growth, n_dims)
            return T.hashgrid_encode(lay, T.half_round(params[key].reshape(-1)), x)

        feats = tcnn_grid(sg, f"{prefix}.hashgrid.static_grid.tcnn_encoding.params", c_mean.view(-1, 3), 3)
    else:
        feats = hash_encode(c_mean.view(-1, 3), params[f"{prefix}.hashgrid.static_grid.hash_table"], s_scal, sg.table_size)
    feats = rescale_grid_features(feats, c_mean, c_std, s_scal, sg.features_per_level)
    out_dim = sg.num_levels * sg.features_per_level
    features = feats.reshape(*times[..., 0].shape, out_dim)
    if trace is not None:
        trace["static_pos"] = c_mean.view(*times[..., 0].shape, 3).clone()
        trace["static_std"] = c_std.view(*times[..., 0].shape).clone()
        trace["actor_id"] = torch.full(times[..., 0].shape, -1, dtype=torch.int64)

    if cfg.n_actors == 0:
        return features.view(-1, out_dim), directions

    # neurad_encoding.py:174: the actor split runs under no_grad unless `require_actor_grad` (True for the main field's
    # grid, fields/neurad_field.py:50; False for the proposal fields', :177) -- only then do the actor trajectories
    # receive gradients through the box-frame positions and directions
    with torch.enable_grad() if require_actor_grad else torch.no_grad():
        b2w, valid = boxes2world_at(params, times[:, 0].squeeze(-1))
        w2b_all = pose_inverse(b2w)
        bounds = params["dynamic_actors.actor_sizes"] / 2 + params["dynamic_actors.actor_padding"]
        with torch.no_grad():  # _get_actor_indices is decorated @torch.no_grad() (neurad_encoding.py:224)
            ray_idx, sample_idx, actor_idx = actor_indices(mean, b2w, valid, w2b_all, bounds)
        w2b = w2b_all[ray_idx, actor_idx]
        pos = transform_points_pairwise(mean[ray_idx, sample_idx], w2b.unsqueeze(-3))
        if directions is not None:
            directions = directions.clone()
            dirs = transform_points_pairwise(directions[ray_idx, sample_idx], w2b, with_translation=False).squeeze(1)
            dirs = dirs / (torch.linalg.norm(dirs, dim=-1, keepdim=True) + EPS)
            directions[ray_idx, sample_idx] = dirs
        if flip is not None:  # neurad_encoding.py:212-219
            fl = torch.ones_like(pos[..., 0:1, :])
            fl[..., 0] = flip[ray_idx].unsqueeze(-1)
            pos = pos * fl
            if directions is not None:
                directions[ray_idx, sample_idx, 0] = directions[ray_idx, sample_idx, 0] * fl[..., 0].squeeze(-1)
    if actor_idx.shape[0] == 0:
        return features.view(-1, out_dim), directions
    a_mean, a_std = scaled_contraction(pos, std[ray_idx, sample_idx], fcfg.actor_scale)
    a_scal = params[f"{prefix}.hashgrid.actor_grids.0.scalings"]
    if tcnn:
        # _get_actor_features_fast (neurad_encoding.py:270-281): ONE 4-D grid, 4th coordinate = actor index / n_actors
        pos4 = torch.cat([a_mean.view(-1, 3), (actor_idx / cfg.n_actors).view(-1, 1).to(a_mean.dtype)], dim=-1)
        afe = tcnn_grid(ag, f"{prefix}.hashgrid.actor_grids.0.tcnn_encoding.params", pos4, 4)
        afe = rescale_grid_features(afe, a_mean, a_std, a_scal, ag.features_per_level)
        padded = F.pad(afe, (0, out_dim - afe.shape[-1]))
        features[ray_idx, sample_idx] = padded
        if trace is not None:
            trace["actor_id"][ray_idx, sample_idx] = actor_idx
            trace["actor_triples"] = torch.stack([ray_idx, sample_idx, actor_idx], -1)
        return features.view(-1, out_dim), directions
    # _get_actor_features_slow (neurad_encoding.py:283-295): one 3-D grid per actor
    afe = None
    for i_actor in actor_idx.unique():
        m = actor_idx == i_actor
        t = params[f"{prefix}.hashgrid.actor_grids.{int(i_actor)}.hash_table"]
        f_ = hash_encode(a_mean[m].view(-1, 3), t, a_scal, ag.table_size)
        f_ = rescale_grid_features(f_, a_mean[m], a_std[m], a_scal, ag.features_per_level)
        if afe is None:
            afe = torch.zeros((m.shape[0], f_.shape[-1]), dtype=f_.dtype)
        afe[m] = f_
    padded = F.pad(afe, (0, out_dim - afe.shape[-1]))
    features[ray_idx, sample_idx] = padded
    if trace is not None:
        trace["actor_id"][ray_idx, sample_idx] = actor_idx
        trace["actor_triples"] = torch.stack([ray_idx, sample_idx, actor_idx], -1)
    return features.view(-1, out_dim), directions


# ----------------------------------------------------------------------------------------------------------------------
# fields
# ----------------------------------------------------------------------------------------------------------------------
class _TruncExp(torch.autograd.Function):
    """field_components/activations.py:28-41: exp forward, backward g * exp(clamp(x, -15, 15))."""

    @staticmethod
    def forward(ctx, x):
        ctx.save_for_backward(x)
        return torch.exp(x)

    @staticmethod
    def backward(ctx, g):
        return g * torch.exp(ctx.saved_tensors[0].clamp(-15, 15))


def proposal_density(params, k: int, cfg: NeuRADCfg, o, d, area, times, starts, ends, trace=None) -> Tensor:
    """NeuRADProposalField.get_density (neurad_field.py:208-213).  starts/ends [N,S]; returns [N,S]."""
    N, S = starts.shape
    mean, std = fast_isotropic_gaussian(o[:, None, :], d[:, None, :], area[:, None, None], starts[..., None], ends[..., None])
    t = times[:, None, None].expand(N, S, 1)
    feats, _ = hashgrid_forward(params, f"proposal_fields.{k}", cfg.prop[k], cfg, mean, std, t, None, trace, require_actor_grad=False)
    dens = F.linear(feats, params[f"proposal_fields.{k}.density_decoder.weight"])
    return _TruncExp.apply(dens).view(N, S)


def sh_components_l4(directions: Tensor) -> Tensor:
    """components_from_spherical_harmonics(levels=4) (utils/math.py:31-94)."""
    comp = torch.zeros((*directions.shape[:-1], 16))
    x, y, z = directions[..., 0], directions[..., 1], directions[..., 2]
    xx, yy, zz = x**2, y**2, z**2
    comp[..., 0] = 0.28209479177387814
    comp[..., 1] = 0.4886025119029199 * y
    comp[..., 2] = 0.4886025119029199 * z
    comp[..., 3] = 0.4886025119029199 * x
    comp[..., 4] = 1.0925484305920792 * x * y
    comp[..., 5] = 1.0925484305920792 * y * z
    comp[..., 6] = 0.9461746957575601 * zz - 0.31539156525251999
    comp[..., 7] = 1.0925484305920792 * x * z
    comp[..., 8] = 0.5462742152960396 * (xx - yy)
    comp[..., 9] = 0.5900435899266435 * y * (3 * xx - yy)
    comp[..., 10] = 2.890611442640554 * x * y * z
    comp[..., 11] = 0.4570457994644658 * y * (5 * zz - 1)
    comp[..., 12] = 0.3731763325901154 * z * (5 * zz - 3)
    comp[..., 13] = 0.4570457994644658 * x * (5 * zz - 1)
    comp[..., 14] = 1.445305721320277 * z * (xx - yy)
    comp[..., 15] = 0.5900435899266435 * x * (xx - 3 * yy)
    return comp


def mlp_forward(params, prefix: str, n_layers: int, x: Tensor, out_dim: Optional[int] = None, width: int = 32) -> Tensor:
    """MLP.pytorch_fwd with ReLU hidden activations, no output activation (field_components/mlp.py:142-178); with a
    tcnn-layout parameter set (`<prefix>.tcnn_encoding.params`, SURVEY 8f row f3) the bias-free FullyFusedMLP restated in
    oracle/tcnn_oracle.py (parity unpinned)."""
    if f"{prefix}.tcnn_encoding.params" in params:
        from . import tcnn_oracle as T

        ws = T.mlp_unpack(params[f"{prefix}.tcnn_encoding.params"].reshape(-1), x.shape[-1], width, n_layers - 1, out_dim)
        return T.mlp_forward(ws, x)
    for i in range(n_layers):
        x = F.linear(x, params[f"{prefix}.layers.{i}.weight"], params[f"{prefix}.layers.{i}.bias"])
        if i < n_layers - 1:
            x = torch.relu(x)
    return x


def main_field(params, cfg: NeuRADCfg, o, d, area, times, starts, ends, trace=None) -> Dict[str, Tensor]:
    """NeuRADField.forward, use_sdf=True (neurad_field.py:128-152)."""
    N, S = starts.shape
    mean, std = fast_isotropic_gaussian(o[:, None, :], d[:, None, :], area[:, None, None], starts[..., None], ends[..., None])
    t = times[:, None, None].expand(N, S, 1)
    dirs_in = d[:, None, :].expand(N, S, 3)
    feats, dirs = hashgrid_forward(params, "field", cfg.main, cfg, mean, std, t, dirs_in, trace)
    h = mlp_forward(params, "field.mlp_geo", 2, feats, out_dim=cfg.nff_out_dim + 1, width=cfg.geo_hidden_dim)
    geo_out, geo_embedding = torch.split(h, [1, cfg.nff_out_dim], dim=-1)
    sdf = geo_out.view(N, S, 1)
    with torch.no_grad():  # SHEncoding.pytorch_fwd is decorated @torch.no_grad() (encodings.py:797-800): in torch mode
        # no gradient reaches the directions, hence none reaches the actor rotations through this path
        direction_embedding = sh_components_l4(((dirs + 1.0) / 2.0).reshape(-1, 3))  # base_field.py:136-142
        if "field.hashgrid.static_grid.tcnn_encoding.params" in params:  # tcnn's SH: x * 2 - 1 inside, its own signs
            from . import tcnn_oracle as T

            direction_embedding = T.sh4((((dirs + 1.0) / 2.0) * 2.0 - 1.0).reshape(-1, 3))
    feature = geo_embedding + mlp_forward(
        params, "field.mlp_feature", 3, torch.cat([geo_embedding, direction_embedding], dim=-1), out_dim=cfg.nff_out_dim,
        width=cfg.nff_hidden_dim
    )
    feature = feature.view(N, S, cfg.nff_out_dim)
    beta = params["field.sdf_to_density.beta"].abs() + 0.0001  # model_components/utils.py:24-41
    alpha = torch.sigmoid(-sdf * beta)
    if trace is not None:
        trace["grid_features"] = feats.view(N, S, -1).clone()
    return {"feature": feature, "sdf": sdf, "alpha": alpha}


# ----------------------------------------------------------------------------------------------------------------------
# nerfacc restatements + compositing
# ----------------------------------------------------------------------------------------------------------------------
def render_weight_from_alpha(alphas: Tensor) -> Tensor:
    """nerfacc==0.5.2 render_weight_from_alpha on a dense [N,S] tensor (call site neurad.py:717):
    trans_i = prod_{j<i} (1 - alpha_j) (exclusive cumprod along the sample axis); w = alpha * trans."""
    trans = torch.cumprod(torch.cat([torch.ones_like(alphas[..., :1]), 1 - alphas[..., :-1]], dim=-1), dim=-1)
    return alphas * trans


def appearance_embedding(params, cfg: NeuRADCfg, times: Tensor, sensor_idx: Tensor) -> Tensor:
    """NeuRADModel._get_appearance_embedding, temporal branch (neurad.py:423-441).  times [N,1], sensor_idx [N,1]."""
    emb = params["appearance_embedding.weight"]
    eps_ = cfg.embeds_per_sensor
    time_idx = times / cfg.duration * eps_
    before_idx = time_idx.floor().clamp(0, eps_ - 1)
    after_idx = (before_idx + 1).clamp(0, eps_ - 1)
    ratio = time_idx - before_idx
    before_idx, after_idx = (x + sensor_idx * eps_ for x in (before_idx, after_idx))
    before_embed = emb[before_idx.squeeze(-1).long()]
    after_embed = emb[after_idx.squeeze(-1).long()]
    return before_embed * (1 - ratio) + after_embed * ratio


def density_fn_field_index(i_level: int, n_fields: int) -> int:
    """Which proposal field the i-th density function evaluates.

    neurad.py:248 builds ``density_fns = [lambda x: prop_field.get_density(x)[0] for prop_field in
    self.proposal_fields]``.  The lambdas close over the comprehension variable, which Python binds late, so
    EVERY density function calls the LAST proposal field (``proposal_fields[-1]``); ``proposal_fields[0]`` is never
    evaluated in the forward pass.  Verified against the imported reference (oracle/make_golden.py asserts it).
    A drop-in must reproduce the reference's results, so the oracle (and the CUDA path) do the same."""
    return n_fields - 1


def nff_outputs(
    params: Dict[str, Tensor],
    cfg: NeuRADCfg,
    origins: Tensor,
    directions: Tensor,
    pixel_area: Tensor,
    times: Tensor,
    sensor_idx: Tensor,
    is_lidar: Optional[Tensor] = None,
    fars: Optional[Tensor] = None,
    nears: Optional[Tensor] = None,
    want_trace: bool = False,
) -> Dict[str, Tensor]:
    """NeuRADModel.get_nff_outputs in eval mode (neurad.py:368-421) with _scale_pixel_area (:702-709),
    _get_ray_samples (:443-459) and ProposalNetworkSampler.generate_ray_samples (ray_samplers.py:623-666).

    origins/directions [N,3]; pixel_area/times [N,1]; sensor_idx [N,1] int64; is_lidar [N,1] bool or None.
    """
    N = origins.shape[0]
    # _scale_pixel_area
    if is_lidar is not None:
        scaling = torch.ones_like(pixel_area)
        scaling[~is_lidar] = cfg.rgb_upsample_factor**2
    else:
        scaling = cfg.rgb_upsample_factor**2
    area = (pixel_area * scaling)[:, 0]
    # _get_ray_samples
    fars = torch.full_like(pixel_area, 1_000_000.0) if fars is None else fars.clone()
    fars = fars.clamp_max(cfg.sky_distance)
    nears = torch.zeros_like(fars) if nears is None else nears
    sp = SpacingFns(cfg, nears, fars)
    t1 = times[:, 0]
    trace: Dict[str, Tensor] = {}

    prop_weights: List[Tensor] = []
    prop_bins_e: List[Tensor] = []
    S0 = cfg.num_proposal_samples[0]
    bins_s, bins_e = initial_bins(cfg, sp, S0)
    bins_s = bins_s.expand(N, S0 + 1)
    weights = None
    levels = list(cfg.num_proposal_samples) + [cfg.num_nerf_samples]
    for i_level, S in enumerate(levels):
        if i_level > 0:
            r = pdf_resample(weights, bins_s, S, cfg.histogram_padding)  # anneal == 1.0 -> pow is the identity
            bins_s = r["bins"].detach()  # "Stop gradients" (ray_samplers.py:363-364); values unchanged
            bins_e = sp.to_euclidean(bins_s)
            if want_trace:
                trace[f"cdf_{i_level}"] = r["cdf"]
                trace[f"inds_{i_level}"] = r["inds"]
        if want_trace:
            trace[f"bins_s_{i_level}"] = bins_s.clone()
            trace[f"bins_e_{i_level}"] = bins_e.clone()
        if i_level < len(cfg.num_proposal_samples):
            starts, ends = bins_e[..., :-1], bins_e[..., 1:]
            tr = {} if want_trace else None
            k = density_fn_field_index(i_level, len(cfg.num_proposal_samples))
            dens = proposal_density(params, k, cfg, origins, directions, area, t1, starts, ends, tr)
            weights = weights_from_density(ends - starts, dens)
            prop_weights.append(weights)
            prop_bins_e.append(bins_e)
            if want_trace:
                trace[f"density_{i_level}"] = dens
                trace[f"actor_id_{i_level}"] = tr["actor_id"]

    # sky sample (neurad.py:451-455)
    starts, ends = bins_e[..., :-1].clone(), bins_e[..., 1:].clone()
    dist_to_sky = cfg.sky_distance - ends[..., -1]
    ends[..., -1] += dist_to_sky
    tr = {} if want_trace else None
    fo = main_field(params, cfg, origins, directions, area, t1, starts, ends, tr)
    w = render_weight_from_alpha(fo["alpha"].squeeze(-1))
    accumulation = torch.sum(w[..., None], dim=-2)  # renderers.py:349
    w = torch.cat((w[..., :-1], w[..., -1:] + 1 - accumulation), dim=-1).unsqueeze(-1)
    features = torch.sum(fo["feature"] * w, dim=-2)  # renderers.py:85
    appearance = appearance_embedding(params, cfg, times, sensor_idx)
    features = torch.cat([features, appearance], dim=-1)
    w_ns, s_ns, e_ns = w[..., :-1, :], starts[..., :-1], ends[..., :-1]
    steps = (s_ns + e_ns) / 2
    depth = torch.sum(w_ns[..., 0] * steps, dim=-1, keepdim=True)  # render_depth_simple, neurad.py:727-734
    out = {"features": features, "depth": depth, "accumulation": accumulation}
    for i, (pw, pb) in enumerate(zip(prop_weights, prop_bins_e)):
        steps = (pb[..., :-1] + pb[..., 1:]) / 2
        out[f"prop_depth_{i}"] = torch.sum(pw * steps, dim=-1, keepdim=True)
    if want_trace:
        trace.update(
            {
                "prop_weights_0": prop_weights[0],
                "prop_weights_1": prop_weights[1],
                "sdf": fo["sdf"].squeeze(-1),
                "alpha": fo["alpha"].squeeze(-1),
                "field_feature": fo["feature"],
                "weights": w.squeeze(-1),
                "starts": starts,
                "ends": ends,
                "actor_id_main": tr["actor_id"],
                "static_pos_main": tr["static_pos"],
                "static_std_main": tr["static_std"],
                "grid_features_main": tr["grid_features"],
            }
        )
        out["trace"] = trace
    return out


def decode_lidar(params, features: Tensor) -> Tuple[Tensor, Tensor]:
    """decode_features, lidar half (neurad.py:350-357): intensity = sigmoid(o[0]), ray_drop_logit = o[1]."""
    o = mlp_forward(params, "lidar_decoder", 3, features, out_dim=2)
    intensity, ray_drop_logit = o.split(1, dim=-1)
    return intensity.sigmoid(), ray_drop_logit


# ----------------------------------------------------------------------------------------------------------------------
# ray generation
# ----------------------------------------------------------------------------------------------------------------------
def normalize_with_norm(x: Tensor, dim: int) -> Tuple[Tensor, Tensor]:
    """cameras/camera_utils.py:596-610."""
    norm = torch.maximum(torch.linalg.vector_norm(x, dim=dim, keepdim=True), torch.tensor([_NORM_EPS], dtype=x.dtype))
    return x / norm, norm


def generate_rays_pinhole(
    c2w: Tensor,
    fx: float,
    fy: float,
    cx: float,
    cy: float,
    height: int,
    width: int,
    coords: Tensor,
    time: float,
    velocity: Optional[Tensor] = None,
    rolling_shutter_time: float = 0.0,
    time_to_center_pixel: float = 0.0,
) -> Dict[str, Tensor]:
    """Cameras._generate_rays_from_coords, PERSPECTIVE camera without distortion, top-to-bottom rolling shutter
    (cameras/cameras.py:633-667, 793-798, 898-969).  coords [...,2] = (y, x) incl. the 0.5 pixel-centre offset."""
    y, x = coords[..., 0], coords[..., 1]
    fx_, fy_, cx_, cy_ = (torch.full_like(x, v) for v in (fx, fy, cx, cy))
    coord = torch.stack([(x - cx_) / fx_, (y - cy_) / fy_], -1)
    coord_x_offset = torch.stack([(x - cx_ + 1) / fx_, (y - cy_) / fy_], -1)
    coord_y_offset = torch.stack([(x - cx_) / fx_, (y - cy_ + 1) / fy_], -1)
    coord_stack = torch.stack([coord, coord_x_offset, coord_y_offset], dim=0)
    coord_stack[..., 1] *= -1
    directions_stack = torch.empty((3,) + x.shape + (3,))
    directions_stack[..., 0] = coord_stack[..., 0]
    directions_stack[..., 1] = coord_stack[..., 1]
    directions_stack[..., 2] = -1.0
    rotation = c2w[:3, :3]
    directions_stack = torch.sum(directions_stack[..., None, :] * rotation, dim=-1)
    directions_stack, directions_norm = normalize_with_norm(directions_stack, -1)
    origins = c2w[:3, 3].expand(x.shape + (3,))
    directions = directions_stack[0]
    dx = torch.sqrt(torch.sum((directions - directions_stack[1]) ** 2, dim=-1))
    dy = torch.sqrt(torch.sum((directions - directions_stack[2]) ** 2, dim=-1))
    pixel_area = (dx * dy)[..., None]
    times = torch.full(x.shape + (1,), time)
    if velocity is not None:
        rows = coords[..., 0:1]
        heights = torch.full_like(rows, float(height)).long()  # self.height is an int64 tensor in the reference
        time_offsets = (rows / heights - 0.5) * rolling_shutter_time + time_to_center_pixel
        origins = origins + velocity * time_offsets
        times = times + time_offsets
    return {
        "origins": origins,
        "directions": directions,
        "pixel_area": pixel_area,
        "times": times,
        "fars": torch.ones_like(pixel_area) * 1_000_000,
        "directions_norm": directions_norm[0],
    }


def generate_rays_lidar_points(l2w: Tensor, points: Tensor, scan_time: float, velocity: Optional[Tensor] = None):
    """Lidars._generate_rays_from_points, assume_ego_compensated=True (cameras/lidars.py:399-460).
    l2w [3,4]; points [P,>=5] = (x, y, z, intensity, dt)."""
    P = points.shape[0]
    l2w_b = l2w[None].expand(P, 3, 4)
    points_world = transform_points_pairwise(points[..., :3], l2w_b)
    origins = l2w_b[..., :3, 3]
    if velocity is not None:
        origins = origins + points[..., 4:5] * velocity
    directions = points_world - origins
    directions, distance = normalize_with_norm(directions, -1)
    pixel_area = torch.full((P, 1), 3.0e-3) * torch.full((P, 1), 1.5e-3)  # lidars.py:46-47, 432-434
    times = torch.full((P, 1), scan_time) + points[..., 4:5]
    return {
        "origins": origins,
        "directions": directions,
        "pixel_area": pixel_area,
        "times": times,
        "fars": torch.ones_like(pixel_area) * 1_000_000,
        "directions_norm": distance,
        "did_return": distance < 1e3,
    }


def generate_rays_lidar_grid(elev_min_deg: float, elev_max_deg: float, beams: int, azim_res_deg: float):
    """Beam x azimuth direction grid of the viewer's lidar render (viewer/render_state_machine.py:395-407)."""
    v_angles = torch.linspace(*np.deg2rad((elev_min_deg, elev_max_deg)), beams)
    h_angles = torch.arange(0, 2 * np.pi, np.deg2rad(azim_res_deg))
    v_angles, h_angles = torch.meshgrid(v_angles, h_angles, indexing="ij")
    v_angles, h_angles = v_angles.flatten(), h_angles.flatten()
    return torch.stack(
        [torch.cos(v_angles) * torch.cos(h_angles), torch.cos(v_angles) * torch.sin(h_angles), torch.sin(v_angles)],
        dim=-1,
    )


def generate_rays_lidar_grid_rs(l2w: Tensor, elev_min_deg: float, elev_max_deg: float, beams: int, azim_res_deg: float,
                                scan_time: float, revolution_time: float = 0.1, velocity: Optional[Tensor] = None):
    """BASELINE config 4 input (SURVEY.md section 8d): the viewer's beam x azimuth grid (above) swept with a rolling
    shutter -- per-ray time offset linear in azimuth over one revolution and origin shifted by velocity * dt
    (cameras/lidars.py:421-423, 625-639); pixel_area = the lidar beam divergence product (lidars.py:46-47)."""
    v_angles = torch.linspace(*np.deg2rad((elev_min_deg, elev_max_deg)), beams)
    h_angles = torch.arange(0, 2 * np.pi, np.deg2rad(azim_res_deg))
    v, h = torch.meshgrid(v_angles, h_angles, indexing="ij")
    v, h = v.flatten(), h.flatten()
    d_l = torch.stack([torch.cos(v) * torch.cos(h), torch.cos(v) * torch.sin(h), torch.sin(v)], dim=-1)
    directions = d_l @ l2w[:3, :3].T
    dt = ((h / (2 * np.pi) - 0.5) * revolution_time)[:, None]
    origins = l2w[:3, 3].expand(d_l.shape[0], 3)
    if velocity is not None:
        origins = origins + dt * velocity
    return {"origins": origins, "directions": directions, "pixel_area": torch.full((d_l.shape[0], 1), 3.0e-3 * 1.5e-3),
            "times": scan_time + dt}
