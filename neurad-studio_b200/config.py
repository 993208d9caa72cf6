"""Configuration of the NeuRAD neural-feature-field forward path.

Mirrors the subset of the reference's config tree that shapes ``NeuRADModel.get_nff_outputs``:
``NeuRADModelConfig`` / ``SamplingSettings`` (nerfstudio/models/neurad.py:97-162), ``NeuRADFieldConfig`` /
``NeuRADProposalFieldConfig`` (nerfstudio/fields/neurad_field.py:44-75, 155-182) and ``StaticSettings`` /
``ActorSettings`` (nerfstudio/field_components/neurad_encoding.py:34-66), and the camera pose optimizer's
``CameraOptimizerConfig`` / ``ScaledCameraOptimizerConfig`` (nerfstudio/cameras/camera_optimizers.py:43-60,335-357).
Field names follow the reference.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Tuple, Union

import numpy as np
import torch


@dataclass
class HashGridSettings:
    """One multi-resolution hash grid (HashEncoding, field_components/encodings.py:326-352)."""

    hashgrid_dim: int = 4  # features per level
    num_levels: int = 8
    base_res: int = 32
    max_res: int = 8192
    log2_hashmap_size: int = 22

    @property
    def hash_table_size(self) -> int:
        return 2**self.log2_hashmap_size

    @property
    def out_dim(self) -> int:
        return self.num_levels * self.hashgrid_dim

    def scalings(self) -> torch.Tensor:
        """Per-level resolutions; the same expression as encodings.py:348-350 so that the buffer is identical
        (main grid: [32, 70, 156, 344, 760, 1680, 3709, 8191] -- note 8191)."""
        levels = torch.arange(self.num_levels)
        growth = (
            np.exp((np.log(self.max_res) - np.log(self.base_res)) / (self.num_levels - 1))
            if self.num_levels > 1
            else 1.0
        )
        return torch.floor(self.base_res * growth**levels)


def _main_static() -> HashGridSettings:
    return HashGridSettings(4, 8, 32, 8192, 22)


def _main_actor() -> HashGridSettings:
    return HashGridSettings(4, 4, 64, 1024, 17)


def _prop_static() -> HashGridSettings:
    return HashGridSettings(1, 6, 128, 4096, 20)


def _prop_actor() -> HashGridSettings:
    return HashGridSettings(1, 4, 64, 1024, 15)


@dataclass
class NeuRADHashEncodingConfig:
    static: HashGridSettings = field(default_factory=_main_static)
    actor: HashGridSettings = field(default_factory=_main_actor)
    actor_scale: float = 10.0
    # ActorSettings.flip_prob, training mode only: 0.25 for the main field's grid (fields/neurad_field.py:51), the
    # ActorSettings default 0.5 for the proposal fields' grids (field_components/neurad_encoding.py:50)
    flip_prob: float = 0.25


def _prop_grid() -> NeuRADHashEncodingConfig:
    return NeuRADHashEncodingConfig(static=_prop_static(), actor=_prop_actor(), flip_prob=0.5)


@dataclass
class SamplingSettings:
    num_proposal_samples: Tuple[int, int] = (128, 64)
    num_nerf_samples: int = 32
    power_lambda: float = -1.0
    power_scaling: float = 0.1
    sky_distance: float = 20000.0
    histogram_padding: float = 0.01  # PDFSampler default, ray_samplers.py:272
    single_jitter: bool = True  # SamplingSettings.single_jitter (neurad.py:101), training mode only


@dataclass
class NeuRADConfig:
    """Everything the forward path needs to know that is not a learned tensor."""

    grid: NeuRADHashEncodingConfig = field(default_factory=NeuRADHashEncodingConfig)
    proposal_grid_1: NeuRADHashEncodingConfig = field(default_factory=_prop_grid)
    proposal_grid_2: NeuRADHashEncodingConfig = field(default_factory=_prop_grid)
    sampling: SamplingSettings = field(default_factory=SamplingSettings)
    geo_hidden_dim: int = 32
    nff_hidden_dim: int = 32
    nff_out_dim: int = 32
    num_multisamples: int = 1  # NeuRADFieldConfig.num_multisamples, neurad_field.py:67
    appearance_dim: int = 16
    # NeuRADModelConfig.use_temporal_appearance (neurad.py:136): True -> embeds_per_sensor rows per sensor, linearly
    # interpolated in time; False (the paper presets) -> one row per sensor, copied
    use_temporal_appearance: bool = True
    temporal_appearance_freq: float = 1.0
    rgb_upsample_factor: int = 3
    rgb_hidden_dim: int = 32
    actor_bbox_padding: Tuple[float, float, float] = (0.25, 0.25, 0.1)
    carving_epsilon: float = 0.1  # LossSettings (neurad.py:79,87): lidar carving masks of the training outputs
    non_return_lidar_distance: float = 150.0
    # LossSettings.ray_drop_loss_mult (neurad.py:91); the lidar metrics' predicted returns are ray-drop probabilities < 0.5
    # when it is > 0, depths < non_return_lidar_distance otherwise (neurad.py:610-613)
    ray_drop_loss_mult: float = 0.01
    # the rest of LossSettings (neurad.py:66-94), flat, with the reference's defaults: the multipliers and the lidar
    # depth loss's quantile of NeuRADModel.get_metrics_dict / get_loss_dict (neurad.py:461-561)
    rgb_mult: float = 5.0
    vgg_mult: float = 0.05
    depth_mult: float = 0.01
    intensity_mult: float = 0.1
    carving_mult: float = 0.01
    quantile_threshold: float = 0.95
    interlevel_loss_mult: float = 0.001
    distortion_loss_mult: float = 0.002
    non_return_loss_mult: float = 0.1
    prop_lidar_loss_mult: float = 0.1
    # scene-level constants (dataset metadata in the reference)
    static_scale: float = 100.0
    duration: float = 8.0
    num_sensors: int = 7
    n_actors: int = 0

    @property
    def proposal_grids(self):
        return (self.proposal_grid_1, self.proposal_grid_2)

    @property
    def embeds_per_sensor(self) -> int:
        return math.ceil(self.duration * self.temporal_appearance_freq)

    @property
    def num_appearance_embeds(self) -> int:
        """Rows of appearance_embedding (neurad.py:190-195)."""
        return self.num_sensors * self.embeds_per_sensor if self.use_temporal_appearance else self.num_sensors

    @property
    def feature_dim(self) -> int:
        return self.nff_out_dim + self.appearance_dim


@dataclass
class CameraOptimizerConfig:
    """Camera pose optimisation (cameras/camera_optimizers.py:43-60): "off" (NeuRAD's default, models/neurad.py), or a
    per-camera 6-vector [translation | rotation] mapped to a pose correction by exp_map_SO3xR3 / exp_map_SE3
    (cameras/lie_groups.py).  The penalties weight the L2 norms of the two halves in get_loss_dict."""

    mode: str = "off"  # "off" | "SO3xR3" | "SE3"
    trans_l2_penalty: Union[Tuple[float, ...], float] = 1e-2
    rot_l2_penalty: float = 1e-3

    def __post_init__(self):
        if self.mode not in ("off", "SO3xR3", "SE3"):
            raise ValueError(f"camera optimizer mode must be 'off', 'SO3xR3' or 'SE3', not {self.mode!r}")


@dataclass
class ScaledCameraOptimizerConfig(CameraOptimizerConfig):
    """Axis-weighted pose optimisation (camera_optimizers.py:335-357): the 6-vector is multiplied by `weights` before the
    exp map; the translation penalty is per axis and applied to |t| (an L1 term).  neurad-scaleopt and its siblings
    (configs/method_configs.py:438-495) use mode "SO3xR3" with weights (1, 1, 0.01, 0.01, 0.01, 1)."""

    weights: Tuple[float, float, float, float, float, float] = (1.0, 1.0, 1.0, 1.0, 1.0, 1.0)
    trans_l2_penalty: Union[Tuple[float, float, float], float] = (1e-2, 1e-2, 1e-2)


def scaleopt_camera_optimizer() -> ScaledCameraOptimizerConfig:
    """The camera optimizer of neurad-scaleopt / neurader-scaleopt / neuradest-scaleopt (method_configs.py:440-449)."""
    return ScaledCameraOptimizerConfig(mode="SO3xR3", weights=(1.0, 1.0, 0.01, 0.01, 0.01, 1.0), trans_l2_penalty=(1e-2, 1e-2, 1e-3))


PRESETS = ("neurad", "neurad-scaleopt", "neurader", "neurader-scaleopt", "neuradest", "neuradest-scaleopt", "neurad-paper",
           "neurad-2x-paper")


def preset(name: str) -> Tuple[NeuRADConfig, CameraOptimizerConfig]:
    """(model config, camera optimizer config) of one of the reference's NeuRAD method presets (method_configs.py:395-507).

    - neurader / neuradest (+ -scaleopt) and neurad-2x-paper double every grid's static base / max resolution and add one
      bit to every static and actor table (main static grid: levels 64 ... 16383, 2^23 rows).  neuradest only trains
      longer than neurader, which is not part of this config.
    - -scaleopt: the axis-weighted SO3xR3 camera optimizer.
    - neurad-paper / neurad-2x-paper: one appearance embedding per sensor.  Their `f.flip_prob = 0.0` loop sets an
      attribute the field configs do not read (the encoding reads `grid.actor.flip_prob`), so the actor flip probabilities
      stay 0.25 / 0.5 in training, as in the reference."""
    if name not in PRESETS:
        raise ValueError(f"unknown preset {name!r}; known: {', '.join(PRESETS)}")
    cfg = NeuRADConfig()
    if name.startswith(("neurader", "neuradest")) or name == "neurad-2x-paper":
        for g in (cfg.grid, *cfg.proposal_grids):
            g.static.max_res *= 2
            g.static.base_res *= 2
            g.static.log2_hashmap_size += 1
            g.actor.log2_hashmap_size += 1
    if name.endswith("-paper"):
        cfg.use_temporal_appearance = False
    copt = scaleopt_camera_optimizer() if name.endswith("-scaleopt") else CameraOptimizerConfig(mode="off")
    return cfg, copt


def small_config(n_actors: int = 0, log2_main: int = 12, log2_prop: int = 11, **kw) -> NeuRADConfig:
    """A shrunken-table configuration (same levels / resolutions / code path, fewer hash slots) used for
    self-contained golden fixtures and smoke tests."""
    cfg = NeuRADConfig(n_actors=n_actors, **kw)
    cfg.grid.static.log2_hashmap_size = log2_main
    cfg.grid.actor.log2_hashmap_size = max(log2_main - 3, 6)
    for g in cfg.proposal_grids:
        g.static.log2_hashmap_size = log2_prop
        g.actor.log2_hashmap_size = max(log2_prop - 3, 6)
    return cfg
