"""Synthetic PandaSet-shaped scenes: parameters, actor trajectories and sensor rigs.

There is no dataset and no checkpoint offline, so benchmarks and tests run on random-initialised parameters
of the reference architecture and on synthetic sensor geometry with the shapes the reference's PandaSet
dataparser produces (6 x 1920x1080 pinhole cameras, one 64-beam lidar; SURVEY.md section 8d).

Parameter tensors are keyed with the reference's ``state_dict`` names (e.g.
``field.hashgrid.static_grid.hash_table``, ``proposal_fields.0.density_decoder.weight``,
``dynamic_actors.actor_rotations_6d``) so that a reference checkpoint and these synthetic parameters are
interchangeable for both the oracle and the CUDA path.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, List, Optional

import torch

from .config import HashGridSettings, NeuRADConfig


def _linear(gen: torch.Generator, out_f: int, in_f: int, bias: bool = True, device="cpu"):
    """torch.nn.Linear's default init: U(-1/sqrt(in), 1/sqrt(in)) for weight and bias."""
    bound = 1.0 / math.sqrt(in_f)
    w = (torch.rand(out_f, in_f, generator=gen, device=device) * 2 - 1) * bound
    b = (torch.rand(out_f, generator=gen, device=device) * 2 - 1) * bound if bias else None
    return w, b


def _table(gen: torch.Generator, g: HashGridSettings, scale: float, device="cpu") -> torch.Tensor:
    """HashEncoding.build_nn_modules (encodings.py:380-384) with a configurable init scale."""
    t = torch.rand(g.hash_table_size * g.num_levels, g.hashgrid_dim, generator=gen, device=device) * 2 - 1
    return t * scale


def make_trajectories(n_actors: int, duration: float = 8.0, hz: float = 10.0, seed: int = 0, axis_aligned: bool = False) -> List[dict]:
    """Straight-line rigid actors on four lanes ahead of the ego; padded boxes never overlap (the reference's
    duplicate-hit winner is unspecified, neurad_encoding.py:256-263).  Same dict layout as the dataparsers'
    ``metadata["trajectories"]`` (dynamic_actors.py:109-170): timestamps [T], poses [T,4,4], dims (w,l,h).
    `axis_aligned`: yaw exactly -90 degrees (rotation entries 0 / +-1), so that the world -> box transform is exact in
    fp32 whatever the order of its operations."""
    gen = torch.Generator().manual_seed(seed + 12345)
    n_t = int(round(duration * hz)) + 1
    ts = torch.arange(n_t, dtype=torch.float64) / hz
    trajs = []
    for a in range(n_actors):
        lane, slot = a % 4, a // 4
        y0 = (-5.25, -1.75, 1.75, 5.25)[lane] * 1.6
        x0 = 12.0 + 14.0 * slot + 3.0 * lane
        speed = (8.0, 10.0, 11.0, 9.0)[lane]
        yaw = -math.pi / 2 + 0.05 * (float(torch.rand((), generator=gen)) - 0.5)  # box y-axis (length) along +x
        c, s = (0.0, -1.0) if axis_aligned else (math.cos(yaw), math.sin(yaw))
        poses = torch.eye(4, dtype=torch.float32).repeat(n_t, 1, 1)
        poses[:, 0, 0], poses[:, 0, 1], poses[:, 1, 0], poses[:, 1, 1] = c, -s, s, c
        poses[:, 0, 3] = (x0 + speed * ts).float()
        poses[:, 1, 3] = y0
        poses[:, 2, 3] = 0.8
        trajs.append(
            {
                "timestamps": ts.float().clone(),
                "poses": poses,
                "dims": torch.tensor([2.0, 4.5, 1.6]),
                "symmetric": True,
                "deformable": False,
            }
        )
    return trajs


def matrix_to_rotation_6d(m: torch.Tensor) -> torch.Tensor:
    """First two rows of the rotation matrix (pytorch3d convention used by cameras/camera_utils.py)."""
    return m[..., :2, :].clone().reshape(*m.shape[:-2], 6)


def actors_state_from_trajectories(trajs: List[dict], padding=(0.25, 0.25, 0.1)) -> Dict[str, torch.Tensor]:
    """The buffers/parameters DynamicActors._populate_actors builds (dynamic_actors.py:109-170) for
    trajectories that share one timestamp set."""
    if len(trajs) == 0:
        return {}
    ts = trajs[0]["timestamps"]
    poses = torch.stack([t["poses"] for t in trajs], dim=1)  # [T,A,4,4]
    return {
        "dynamic_actors.unique_timestamps": ts.clone(),
        "dynamic_actors.actor_positions": poses[..., :3, 3].clone(),
        "dynamic_actors.actor_rotations_6d": matrix_to_rotation_6d(poses[..., :3, :3]),
        "dynamic_actors.actor_present_at_time": torch.ones(ts.shape[0], len(trajs), dtype=torch.bool),
        "dynamic_actors.actor_sizes": torch.stack([t["dims"] for t in trajs]).float(),
        "dynamic_actors.actor_padding": torch.tensor(padding),
    }


def make_params(
    cfg: NeuRADConfig,
    seed: int = 0,
    table_scale: float = 1.0,
    beta: float = 20.0,
    device="cpu",
    trajectories: Optional[List[dict]] = None,
    sdf_bias: Optional[float] = None,
) -> Dict[str, torch.Tensor]:
    """Random-init parameters of the NeuRAD architecture under the reference's state_dict names.

    `sdf_bias` overrides the bias of the SDF output neuron: a positive value makes most samples "outside"
    (small alpha), which spreads the compositing weights along the ray instead of saturating at the first few
    samples as a raw random init with beta=20 does."""
    gen = torch.Generator(device=device).manual_seed(seed)
    p: Dict[str, torch.Tensor] = {}

    def grids(prefix: str, gcfg):
        p[f"{prefix}.hashgrid.static_grid.hash_table"] = _table(gen, gcfg.static, table_scale, device)
        p[f"{prefix}.hashgrid.static_grid.scalings"] = gcfg.static.scalings().to(device)
        for a in range(cfg.n_actors):
            p[f"{prefix}.hashgrid.actor_grids.{a}.hash_table"] = _table(gen, gcfg.actor, table_scale, device)
            p[f"{prefix}.hashgrid.actor_grids.{a}.scalings"] = gcfg.actor.scalings().to(device)

    grids("field", cfg.grid)
    d_in = cfg.grid.static.out_dim
    for i, (o, n) in enumerate([(cfg.geo_hidden_dim, d_in), (cfg.nff_out_dim + 1, cfg.geo_hidden_dim)]):
        w, b = _linear(gen, o, n, device=device)
        p[f"field.mlp_geo.layers.{i}.weight"], p[f"field.mlp_geo.layers.{i}.bias"] = w, b
    dims = [(cfg.nff_hidden_dim, 16 + cfg.nff_out_dim), (cfg.nff_hidden_dim, cfg.nff_hidden_dim), (cfg.nff_out_dim, cfg.nff_hidden_dim)]
    for i, (o, n) in enumerate(dims):
        w, b = _linear(gen, o, n, device=device)
        p[f"field.mlp_feature.layers.{i}.weight"], p[f"field.mlp_feature.layers.{i}.bias"] = w, b
    if sdf_bias is not None:
        p["field.mlp_geo.layers.1.bias"][0] = float(sdf_bias)
    p["field.sdf_to_density.beta"] = torch.full((1,), float(beta), device=device)
    for k, g in enumerate(cfg.proposal_grids):
        grids(f"proposal_fields.{k}", g)
        w, _ = _linear(gen, 1, g.static.out_dim, bias=False, device=device)
        p[f"proposal_fields.{k}.density_decoder.weight"] = w
    p["appearance_embedding.weight"] = torch.randn(cfg.num_appearance_embeds, cfg.appearance_dim, generator=gen, device=device)
    for i, (o, n) in enumerate([(32, cfg.feature_dim), (32, 32), (2, 32)]):
        w, b = _linear(gen, o, n, device=device)
        p[f"lidar_decoder.layers.{i}.weight"], p[f"lidar_decoder.layers.{i}.bias"] = w, b
    if cfg.n_actors > 0:
        trajs = trajectories if trajectories is not None else make_trajectories(cfg.n_actors, cfg.duration, seed=seed)
        for k_, v in actors_state_from_trajectories(trajs, cfg.actor_bbox_padding).items():
            p[k_] = v.to(device)
    p["static_scale"] = torch.tensor(float(cfg.static_scale), device=device)
    return p


def make_params_tcnn(cfg: NeuRADConfig, seed: int = 0, table_scale: float = 1.0, beta: float = 20.0, device="cpu",
                     trajectories: Optional[List[dict]] = None, mlp_gain: float = 1.0) -> Dict[str, torch.Tensor]:
    """Random-init parameters of the same architecture under the state_dict names of a checkpoint trained with the
    reference's default `implementation="tcnn"`: one flat `tcnn_encoding.params` per HashEncoding / MLP in tiny-cuda-nn's
    layout (tcnn_compat.py), one 4-D grid shared by the actors, bias-free MLPs with padded widths.  fp32 master values like
    the torch binding stores them (the binding casts to half at forward time; so does `B200Backend.load_params`)."""
    from . import tcnn_compat as T

    gen = torch.Generator(device=device).manual_seed(seed)
    p: Dict[str, torch.Tensor] = {}

    def rnd(n, scale):
        return (torch.rand(n, generator=gen, device=device) * 2 - 1) * scale

    def grids(prefix: str, gcfg):
        ls = T.layout_of(gcfg.static, 3)
        p[f"{prefix}.hashgrid.static_grid.{T.TCNN_SUFFIX}"] = rnd(ls["n_entries"] * ls["n_features"], table_scale)
        p[f"{prefix}.hashgrid.static_grid.scalings"] = gcfg.static.scalings().to(device)
        if cfg.n_actors > 0:
            la = T.layout_of(gcfg.actor, 4)
            p[f"{prefix}.hashgrid.actor_grids.0.{T.TCNN_SUFFIX}"] = rnd(la["n_entries"] * la["n_features"], table_scale)
            p[f"{prefix}.hashgrid.actor_grids.0.scalings"] = gcfg.actor.scalings().to(device)

    def mlp(prefix, in_dim, width, n_layers, out_dim):
        n = sum(o * k for o, k in T.mlp_shapes(in_dim, width, n_layers - 1, out_dim))
        p[f"{prefix}.{T.TCNN_SUFFIX}"] = rnd(n, mlp_gain * (3.0 / width) ** 0.5)

    grids("field", cfg.grid)
    mlp("field.mlp_geo", cfg.grid.static.out_dim, cfg.geo_hidden_dim, 2, cfg.nff_out_dim + 1)
    mlp("field.mlp_feature", 16 + cfg.nff_out_dim, cfg.nff_hidden_dim, 3, cfg.nff_out_dim)
    p["field.sdf_to_density.beta"] = torch.full((1,), float(beta), device=device)
    for k, g in enumerate(cfg.proposal_grids):
        grids(f"proposal_fields.{k}", g)
        w, _ = _linear(gen, 1, g.static.out_dim, bias=False, device=device)
        p[f"proposal_fields.{k}.density_decoder.weight"] = w
    p["appearance_embedding.weight"] = torch.randn(cfg.num_appearance_embeds, cfg.appearance_dim, generator=gen, device=device)
    mlp("lidar_decoder", cfg.feature_dim, 32, 3, 2)
    if cfg.n_actors > 0:
        trajs = trajectories if trajectories is not None else make_trajectories(cfg.n_actors, cfg.duration, seed=seed)
        for k_, v in actors_state_from_trajectories(trajs, cfg.actor_bbox_padding).items():
            p[k_] = v.to(device)
    p["static_scale"] = torch.tensor(float(cfg.static_scale), device=device)
    return p


# ----------------------------------------------------------------------------------------------------------------------
# sensors
# ----------------------------------------------------------------------------------------------------------------------
@dataclass
class PinholeCamera:
    """One PERSPECTIVE camera of a `Cameras` batch (cameras/cameras.py) plus the rolling-shutter metadata the AD
    dataparsers attach (pandaset_dataparser.py:144-146, ad_dataparser.py:361-386)."""

    c2w: torch.Tensor  # [3,4], OpenGL convention (camera looks along -z, +y up)
    fx: float
    fy: float
    cx: float
    cy: float
    width: int
    height: int
    time: float
    velocity: torch.Tensor  # [3] m/s, world frame
    rolling_shutter_time: float = 0.03
    time_to_center_pixel: float = -0.01
    sensor_idx: int = 0


@dataclass
class LidarScan:
    """One lidar sweep (cameras/lidars.py): pose, per-point (x,y,z,intensity,dt) in the lidar frame."""

    l2w: torch.Tensor  # [3,4]
    points: torch.Tensor  # [P,5]
    time: float
    velocity: torch.Tensor  # [3]
    sensor_idx: int = 6


def _look_at_c2w(pos: torch.Tensor, yaw: float, pitch: float = 0.0) -> torch.Tensor:
    """Camera-to-world for a camera at `pos` whose optical axis (-z) points along world yaw (about +z)."""
    fwd = torch.tensor([math.cos(yaw) * math.cos(pitch), math.sin(yaw) * math.cos(pitch), math.sin(pitch)])
    up = torch.tensor([0.0, 0.0, 1.0])
    right = torch.linalg.cross(fwd, up)
    right = right / right.norm()
    true_up = torch.linalg.cross(right, fwd)
    c2w = torch.zeros(3, 4)
    c2w[:, 0], c2w[:, 1], c2w[:, 2], c2w[:, 3] = right, true_up, -fwd, pos
    return c2w


def pandaset_rig(time: float = 4.0, speed: float = 10.0, width: int = 1920, height: int = 1080) -> List[PinholeCamera]:
    """Six pinhole cameras on an ego vehicle driving along +x at `speed` m/s (SURVEY.md section 8d, config 2)."""
    ego = torch.tensor([speed * time - 40.0, 0.0, 1.8])
    vel = torch.tensor([speed, 0.0, 0.0])
    cams = []
    for i, yaw_deg in enumerate((0.0, 55.0, -55.0, 110.0, -110.0, 180.0)):
        f = 1000.0 if i == 0 else 930.0
        f = f * width / 1920.0
        cams.append(
            PinholeCamera(
                c2w=_look_at_c2w(ego, math.radians(yaw_deg)),
                fx=f, fy=f, cx=width / 2.0, cy=height / 2.0, width=width, height=height,
                time=time, velocity=vel, sensor_idx=i,
            )
        )
    return cams


def pandar64_scan(time: float = 4.0, speed: float = 10.0, beams: int = 64, azimuths: int = 1800, seed: int = 0) -> LidarScan:
    """A 64-beam x 1800-azimuth sweep (115 200 points) with ranges U(2,80) m and per-point time offsets linear in
    azimuth over the 0.1 s revolution (cameras/lidars.py:421-450, 625-639)."""
    gen = torch.Generator().manual_seed(seed + 777)
    elev = torch.deg2rad(torch.linspace(-25.0, 15.0, beams))
    azim = torch.arange(azimuths, dtype=torch.float32) * (2 * math.pi / azimuths)
    e, a = torch.meshgrid(elev, azim, indexing="ij")
    rng = 2.0 + 78.0 * torch.rand(beams, azimuths, generator=gen)
    pts = torch.stack([rng * torch.cos(e) * torch.cos(a), rng * torch.cos(e) * torch.sin(a), rng * torch.sin(e)], -1)
    dt = (a / (2 * math.pi) - 0.5) * 0.1
    inten = torch.rand(beams, azimuths, generator=gen)
    points = torch.cat([pts, inten[..., None], dt[..., None]], -1).reshape(-1, 5)
    l2w = torch.zeros(3, 4)
    l2w[:, :3] = torch.eye(3)
    l2w[:, 3] = torch.tensor([speed * time - 40.0, 0.0, 2.0])
    return LidarScan(l2w=l2w, points=points, time=time, velocity=torch.tensor([speed, 0.0, 0.0]))


def random_rays(
    n: int, cfg: NeuRADConfig, seed: int = 0, lidar_fraction: float = 0.25, trajectories: Optional[List[dict]] = None
) -> Dict[str, torch.Tensor]:
    """A flat ray batch (mix of camera and lidar rays) for unit/parity tests.  With `trajectories`, every
    other ray is aimed at (a jittered point inside) an actor box at the ray's own time so that the actor
    branch of the encoding is exercised."""
    gen = torch.Generator().manual_seed(seed + 999)

    def r(*shape):
        return torch.rand(*shape, generator=gen)

    o = torch.stack([r(n) * 10.0 - 5.0, r(n) * 4.0 - 2.0, 1.2 + r(n)], -1)
    yaw = (r(n) - 0.5) * 1.2
    pitch = (r(n) - 0.6) * 0.25
    d = torch.stack([torch.cos(yaw) * torch.cos(pitch), torch.sin(yaw) * torch.cos(pitch), torch.sin(pitch)], -1)
    times = r(n) * cfg.duration
    if trajectories:
        a_pick = torch.randint(0, len(trajectories), (n,), generator=gen)
        jitter = (r(n, 3) - 0.5) * torch.tensor([3.0, 1.5, 1.2])
        for i in range(0, n, 2):
            tr = trajectories[int(a_pick[i])]
            k = int(torch.argmin((tr["timestamps"] - times[i]).abs()))
            target = tr["poses"][k, :3, 3] + jitter[i]
            v = target - o[i]
            d[i] = v / v.norm()
    is_lidar = r(n) < lidar_fraction
    area = torch.where(is_lidar, torch.full((n,), 3.0e-3 * 1.5e-3), torch.full((n,), 1.0e-6) * (0.5 + r(n)))
    sensor = torch.where(
        is_lidar, torch.full((n,), cfg.num_sensors - 1), torch.randint(0, cfg.num_sensors - 1, (n,), generator=gen)
    )
    return {
        "origins": o,
        "directions": d,
        "pixel_area": area[:, None],
        "times": times[:, None],
        "sensor_idx": sensor[:, None].long(),
        "is_lidar": is_lidar[:, None],
    }


def make_rgb_decoder_params(seed: int = 0, in_dim: int = 48, hidden: int = 32, upsample: int = 3, device="cpu",
                            prefix: str = "rgb_decoder") -> Dict[str, torch.Tensor]:
    """Random-init NeuRADModel.rgb_decoder parameters under the reference's state_dict keys (models/neurad.py:201-216,
    model_components/cnns.py:35-46): torch's default Conv2d init bounds, BatchNorm affine / running statistics
    randomised so that the eval-mode folding is exercised.  Synthetic data for the bench and the tests."""
    g = torch.Generator().manual_seed(seed)

    def conv(co, ci, k, gain=1.0):
        bound = 1.0 / (ci * k * k) ** 0.5
        return (torch.rand(co, ci, k, k, generator=g) * 2 - 1) * bound * gain, (torch.rand(co, generator=g) * 2 - 1) * bound

    p: Dict[str, torch.Tensor] = {}
    p[f"{prefix}.0.weight"], p[f"{prefix}.0.bias"] = conv(hidden, in_dim, 1)
    for blk in (2, 3, 5, 6):
        for c, b in ((0, 1), (3, 4)):
            p[f"{prefix}.{blk}.main_branch.{c}.weight"], p[f"{prefix}.{blk}.main_branch.{c}.bias"] = conv(hidden, hidden, 7, 1.7)
            p[f"{prefix}.{blk}.main_branch.{b}.weight"] = torch.rand(hidden, generator=g) * 0.8 + 0.6
            p[f"{prefix}.{blk}.main_branch.{b}.bias"] = torch.randn(hidden, generator=g) * 0.1
            p[f"{prefix}.{blk}.main_branch.{b}.running_mean"] = torch.randn(hidden, generator=g) * 0.1
            p[f"{prefix}.{blk}.main_branch.{b}.running_var"] = torch.rand(hidden, generator=g) * 0.5 + 0.25
    bound = 1.0 / (hidden * upsample * upsample) ** 0.5
    p[f"{prefix}.4.weight"] = (torch.rand(hidden, hidden, upsample, upsample, generator=g) * 2 - 1) * bound * 3
    p[f"{prefix}.4.bias"] = (torch.rand(hidden, generator=g) * 2 - 1) * bound
    p[f"{prefix}.7.weight"], p[f"{prefix}.7.bias"] = conv(3, hidden, 1)
    return {k: v.to(device) for k, v in p.items()}
