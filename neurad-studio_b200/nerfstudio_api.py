"""Host-side mirror of the reference's plugin / operator API for the hot path, backed by libb200nerf.so.

Same class names, constructor arguments, parameter names (state_dict keys) and call signatures as the reference
modules, so that the parity tests read like the reference's own tests and a reference checkpoint loads unchanged:

  reference (nerfstudio/...)                                   here
  -----------------------------------------------------------  ---------------------------------------------
  cameras/rays.py:252           RayBundle                      RayBundle
  field_components/encodings.py:311  HashEncoding(implementation=) HashEncoding      (forward -> hashgrid_fwd kernel)
  field_components/encodings.py:760  SHEncoding(levels=4)      SHEncoding        (forward -> sh4_fwd kernel)
  field_components/mlp.py:60    MLP(implementation=)           MLP               (forward -> wgmma mlp_fwd kernel)
  model_components/ray_samplers.py:255  PDFSampler             PDFSampler        (-> pdf_resample kernel)
  model_components/ray_samplers.py:56,135,838  Spaced/Uniform/.../PowerSampler  same names (-> spaced_sample kernel)
  cameras/rays.py:33,127        Frustums, RaySamples           same names (get_positions / get_weights kernels)
  model_components/renderers.py:59,93,322,353  Feature/RGB/Accumulation/DepthRenderer  same names (-> composite kernel)
  cameras/camera_optimizers.py:84,359  CameraOptimizer, ScaledCameraOptimizer  same names (exp maps in torch on [C,6])
  models/neurad.py:165          NeuRADModel.get_nff_outputs /  NeuRADModel       (-> fused nff_render_fwd kernel)
                                get_outputs_for_camera_ray_bundle / decode_features (lidar half)
  field_components/neurad_encoding.py:85  NeuRADHashEncoding   NeuRADHashEncoding (-> neurad_encoding_fwd kernel)
  fields/neurad_field.py:76,186  NeuRADField, NeuRADProposalField  same names (encoding + wgmma MLPs + head kernels)
  model_components/ray_samplers.py:569  ProposalNetworkSampler  ProposalNetworkSampler (stage kernels, density_fns)
                                NeuRADModel.field / .proposal_fields / .sampler / .density_fns as in neurad.py:180-248;
                                get_nff_outputs(fused=False) walks these modules like the reference does

Inference runs the fused kernels; with grad mode on and trainable parameters the per-module walk runs instead, every
stage an autograd node backed by a hand-written backward operator (autograd.py; SURVEY.md section 8f row f2).  The rgb
decoder is inference-only.  There is no CPU path: modules raise at call time if the parameters are not on a CUDA device.
"""
from __future__ import annotations

import itertools

import math
from dataclasses import dataclass, field
from enum import Enum
from typing import Dict, List, Optional, Tuple

import torch
from torch import Tensor, nn

from . import autograd as AG
from . import metrics as M
from .backend import B200Backend, is_pinhole_camera
from .config import CameraOptimizerConfig, HashGridSettings, NeuRADConfig, ScaledCameraOptimizerConfig

_BACKENDS: Dict[int, B200Backend] = {}
_UIDS = itertools.count(1)  # one token per model instance (id() can be reused after garbage collection)


def get_backend(device: torch.device) -> B200Backend:
    """One B200Backend (= one b200nerf_ctx) per CUDA device and process."""
    device = torch.device(device)
    if device.type != "cuda":
        raise RuntimeError("the b200 implementation runs on CUDA (sm_90a) devices only; there is no CPU fallback")
    idx = device.index if device.index is not None else torch.cuda.current_device()
    if idx not in _BACKENDS:
        _BACKENDS[idx] = B200Backend(torch.device("cuda", idx))
    return _BACKENDS[idx]


def _needs_grad(*tensors) -> bool:
    return torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in tensors)


def _no_backward(what: str, *tensors) -> None:
    """Operators without a backward fail loudly rather than detach silently."""
    if _needs_grad(*tensors):
        raise NotImplementedError(f"{what} has no backward operator (NeuRAD does not train through it); detach its inputs "
                                  "or call it under torch.no_grad()")


@dataclass
class RayBundle:
    """cameras/rays.py:252-275 (the tensors the hot path reads; shapes [*batch, k])."""

    origins: Tensor
    directions: Tensor
    pixel_area: Tensor
    camera_indices: Optional[Tensor] = None
    nears: Optional[Tensor] = None
    fars: Optional[Tensor] = None
    metadata: Dict[str, Tensor] = field(default_factory=dict)
    times: Optional[Tensor] = None

    @property
    def shape(self) -> Tuple[int, ...]:
        return tuple(self.origins.shape[:-1])

    def __len__(self) -> int:
        return self.origins.numel() // 3

    def _map(self, fn) -> "RayBundle":
        def m(t):
            return None if t is None else fn(t)

        return RayBundle(
            origins=fn(self.origins), directions=fn(self.directions), pixel_area=fn(self.pixel_area),
            camera_indices=m(self.camera_indices), nears=m(self.nears), fars=m(self.fars),
            metadata={k: fn(v) for k, v in self.metadata.items()}, times=m(self.times),
        )

    def flatten(self) -> "RayBundle":
        return self._map(lambda t: t.reshape(-1, t.shape[-1]))

    def __getitem__(self, idx) -> "RayBundle":
        return self._map(lambda t: t[idx])

    def get_row_major_sliced_ray_bundle(self, start_idx: int, end_idx: int) -> "RayBundle":
        return self.flatten()[start_idx:end_idx]  # rays.py:300-311

    def as_backend_dict(self) -> Dict[str, Tensor]:
        fb = self.flatten()
        d = {"origins": fb.origins, "directions": fb.directions, "pixel_area": fb.pixel_area, "times": fb.times}
        if fb.nears is not None:
            d["nears"] = fb.nears
        if fb.fars is not None:
            d["fars"] = fb.fars
        if "sensor_idxs" in fb.metadata:
            d["sensor_idx"] = fb.metadata["sensor_idxs"]
        if "is_lidar" in fb.metadata:
            d["is_lidar"] = fb.metadata["is_lidar"]
        return d


class Cameras:
    """cameras/cameras.py with the AD rolling-shutter metadata: a batch of cameras (scene.PinholeCamera descriptors:
    PERSPECTIVE or FISHEYE, optional k1..k4, p1, p2 distortion, vertical or horizontal shutter) whose
    `generate_rays(camera_indices, keep_shape=True)` returns the full-resolution [H, W] bundle the evaluation loop feeds to
    `get_outputs_for_camera_ray_bundle` (pipelines/ad_pipeline.py:198-208).  One raygen kernel; constant per-image fields
    (sensor index, camera index) are stride-0 views."""

    def __init__(self, cameras, device: torch.device) -> None:
        self.cameras = list(cameras)  # scene.PinholeCamera descriptors (host side, like the reference's Cameras tensors)
        self.device = torch.device(device)

    def __len__(self) -> int:
        return len(self.cameras)

    def generate_rays(self, camera_indices: int, keep_shape: bool = True) -> RayBundle:
        cam = self.cameras[int(camera_indices)]
        be = get_backend(self.device)
        # the undistorted perspective model keeps its original entry point; on the device both are raygen_camera_kernel
        r = be.raygen_pinhole(cam) if is_pinhole_camera(cam) else be.raygen_camera(cam)
        h, w = r["shape"]
        shape = (h, w) if keep_shape else (h * w,)

        def v(t):
            return t.view(*shape, t.shape[-1])

        def const(val):
            return torch.full((1,), val, dtype=torch.long, device=self.device).expand(*shape, 1)

        return RayBundle(origins=v(r["origins"]), directions=v(r["directions"]), pixel_area=v(r["pixel_area"]), times=v(r["times"]),
                         camera_indices=const(int(camera_indices)), metadata={"sensor_idxs": const(cam.sensor_idx)})


class Lidars:
    """cameras/lidars.py:399-460: `generate_rays(lidar_indices, points, keep_shape)` -- one ray per measured point
    (origin = sensor pose + velocity * dt, unit direction, beam footprint, metadata directions_norm / is_lidar / did_return)."""

    def __init__(self, scans, device: torch.device) -> None:
        self.scans = list(scans)  # scene.LidarScan descriptors
        self.device = torch.device(device)
        self.lidar_to_worlds = torch.stack([s.l2w for s in self.scans]).to(self.device)

    def __len__(self) -> int:
        return len(self.scans)

    def generate_rays(self, lidar_indices, points: Tensor, keep_shape: bool = True) -> RayBundle:
        idx = int(lidar_indices.reshape(-1)[0]) if torch.is_tensor(lidar_indices) else int(lidar_indices)
        scan = self.scans[idx]
        r = get_backend(self.device).raygen_lidar_points(scan, points.to(self.device, non_blocking=True))
        n = r["origins"].shape[0]
        md = {"directions_norm": r["directions_norm"], "did_return": r["did_return"],
              "is_lidar": torch.ones(1, dtype=torch.bool, device=self.device).expand(n, 1),
              "sensor_idxs": torch.full((1,), scan.sensor_idx, dtype=torch.long, device=self.device).expand(n, 1)}
        return RayBundle(origins=r["origins"], directions=r["directions"], pixel_area=r["pixel_area"], times=r["times"],
                         camera_indices=torch.full((1,), idx, dtype=torch.long, device=self.device).expand(n, 1), metadata=md,
                         fars=torch.full((1,), 1_000_000.0, device=self.device).expand(n, 1))


class HashEncoding(nn.Module):
    """field_components/encodings.py:311-471 with `implementation="b200"`.  Parameter `hash_table` [L*T, F] and
    buffer `scalings` exactly as the torch implementation builds them (encodings.py:348-352, 380-384)."""

    def __init__(self, num_levels: int = 16, min_res: int = 16, max_res: int = 1024, log2_hashmap_size: int = 19,
                 features_per_level: int = 2, hash_init_scale: float = 0.001, implementation: str = "b200") -> None:
        super().__init__()
        if implementation != "b200":
            raise ValueError("this module is the 'b200' implementation of HashEncoding")
        self.num_levels, self.min_res, self.max_res = num_levels, min_res, max_res
        self.features_per_level, self.log2_hashmap_size = features_per_level, log2_hashmap_size
        self.hash_table_size = 2**log2_hashmap_size
        self._g = HashGridSettings(features_per_level, num_levels, min_res, max_res, log2_hashmap_size)
        self.register_buffer("scalings", self._g.scalings())
        table = torch.rand(size=(self.hash_table_size * num_levels, features_per_level)) * 2 - 1
        self.hash_table = nn.Parameter(table * hash_init_scale)

    def get_out_dim(self) -> int:
        return self.num_levels * self.features_per_level

    def forward(self, in_tensor: Tensor) -> Tensor:
        assert in_tensor.shape[-1] == 3  # encodings.py:428
        be = get_backend(self.hash_table.device)
        # the reference also differentiates w.r.t. the positions (encodings.py:425-471); this operator only trains the table
        _no_backward("HashEncoding (d / d positions)", in_tensor)
        if torch.is_grad_enabled() and self.hash_table.requires_grad:  # trains the table (hand-written scatter backward)
            return AG.HashGridFn.apply(be, self._g, self.scalings, in_tensor.detach(), self.hash_table)
        with torch.no_grad():
            return be.hashgrid_fwd(self._g, self.hash_table, in_tensor, self.scalings)


class SHEncoding(nn.Module):
    """field_components/encodings.py:760-805 (levels = 4)."""

    def __init__(self, levels: int = 4, implementation: str = "b200") -> None:
        super().__init__()
        if levels != 4:
            raise ValueError("the b200 implementation provides SH levels = 4 (the only one NeuRAD uses)")
        self.levels = levels

    def get_out_dim(self) -> int:
        return self.levels**2

    @torch.no_grad()
    def forward(self, in_tensor: Tensor) -> Tensor:
        return get_backend(in_tensor.device).sh4_fwd(in_tensor)


class MLP(nn.Module):
    """field_components/mlp.py:60-183: `num_layers` Linear layers of width `layer_width`, ReLU in between, no
    output activation.  Parameters are `layers.{i}.weight/bias` like the torch implementation (mlp.py:142-157)."""

    def __init__(self, in_dim: int, num_layers: int, layer_width: int, out_dim: Optional[int] = None,
                 activation: Optional[nn.Module] = None, out_activation: Optional[nn.Module] = None,
                 implementation: str = "b200") -> None:
        super().__init__()
        assert in_dim > 0
        if activation is not None and not isinstance(activation, nn.ReLU):
            raise NotImplementedError("the tensor-core MLP operator has ReLU hidden activations (all NeuRAD uses)")
        self.in_dim, self.num_layers, self.layer_width = in_dim, num_layers, layer_width
        self.out_dim = out_dim if out_dim is not None else layer_width
        self.out_activation = out_activation  # applied on the operator's output (none on NeuRAD's path)
        self.build_nn_modules()

    def build_nn_modules(self) -> None:
        """mlp.py:142-157 (the reference builds its layers here too; calling it again re-initialises them)."""
        dims = [self.in_dim] + [self.layer_width] * (self.num_layers - 1) + [self.out_dim]
        self.layers = nn.ModuleList([nn.Linear(dims[i], dims[i + 1]) for i in range(self.num_layers)])

    def get_out_dim(self) -> int:
        return self.out_dim

    def forward(self, in_tensor: Tensor) -> Tensor:
        be = get_backend(in_tensor.device)
        wb = [t for l in self.layers for t in (l.weight, l.bias)]
        if _needs_grad(in_tensor, *wb):  # MLP backward operators (dX on wgmma, dW / db)
            y = AG.MlpFn.apply(be, in_tensor.reshape(-1, in_tensor.shape[-1]).contiguous(), *wb).reshape(*in_tensor.shape[:-1], self.out_dim)
        else:
            with torch.no_grad():
                y = be.mlp_fwd(in_tensor, wb[0::2], wb[1::2])
        return y if self.out_activation is None else self.out_activation(y)


class NearFarCollider:
    """model_components/scene_colliders.py:169-191: fixed nears / fars on a ray bundle."""

    def __init__(self, near_plane: float, far_plane: float, reset_near_plane: bool = True) -> None:
        self.near_plane, self.far_plane, self.reset_near_plane = near_plane, far_plane, reset_near_plane
        self.training = True  # a freshly constructed nn.Module is in training mode

    def set_nears_and_fars(self, ray_bundle: RayBundle) -> RayBundle:
        ones = torch.ones_like(ray_bundle.origins[..., 0:1])
        near_plane = self.near_plane if (self.training or not self.reset_near_plane) else 0
        ray_bundle.nears = ones * near_plane
        ray_bundle.fars = ones * self.far_plane
        return ray_bundle

    def __call__(self, ray_bundle: RayBundle) -> RayBundle:
        if ray_bundle.nears is not None and ray_bundle.fars is not None:
            return ray_bundle  # scene_colliders.py:35-39
        return self.set_nears_and_fars(ray_bundle)


class PDFSampler:
    """model_components/ray_samplers.py:255-376 (include_original=True, the reference's default, merges the old edges
    into the new ones with a sort; NeuRAD's sampler passes False).

    Reference signature `pdf_sampler(ray_bundle, ray_samples, weights, num_samples=)` -> RaySamples (the resampled
    spacing bins mapped through the existing samples' spacing_to_euclidean_fn, :363-375); the short form
    `pdf_sampler(weights, existing_bins, num_samples)` returns just the new spacing-domain edges."""

    def __init__(self, num_samples: Optional[int] = None, train_stratified: bool = True, single_jitter: bool = False,
                 include_original: bool = True, histogram_padding: float = 0.01) -> None:
        self.include_original = include_original  # NeuRAD's sampler passes False (ray_samplers.py:606)
        self.num_samples, self.histogram_padding = num_samples, histogram_padding
        self.train_stratified, self.single_jitter = train_stratified, single_jitter
        self.training = False  # the reference's samplers are nn.Modules; NeuRADModel.train() propagates the flag

    @torch.no_grad()
    def __call__(self, *args, num_samples: Optional[int] = None, **kw):
        if args and isinstance(args[0], RayBundle) or "ray_bundle" in kw:
            if len(args) > 3:  # (ray_bundle, ray_samples, weights, num_samples) as in tests/model_components/test_ray_sampler.py
                num_samples, args = args[3], args[:3]
            return self.generate_ray_samples(*args, num_samples=num_samples, **kw)
        weights, existing_bins = args[0], args[1]
        n = num_samples or (args[2] if len(args) > 2 else None) or self.num_samples
        assert n is not None
        w = weights[..., 0] if weights.dim() == existing_bins.dim() + 1 else weights
        be = get_backend(w.device)
        return be.pdf_resample(w, existing_bins, n, self.histogram_padding)[0]

    @torch.no_grad()
    def generate_ray_samples(self, ray_bundle: Optional["RayBundle"] = None, ray_samples: Optional["RaySamples"] = None,
                             weights: Optional[Tensor] = None, num_samples: Optional[int] = None) -> "RaySamples":
        if ray_samples is None or ray_bundle is None:
            raise ValueError("ray_samples and ray_bundle must be provided")  # ray_samplers.py:300-301
        assert weights is not None, "weights must be provided"
        n = num_samples or self.num_samples
        assert n is not None
        be = get_backend(weights.device)
        existing = ray_samples.per_ray_spacing_bins()
        w = weights[..., 0] if weights.dim() == 3 else weights
        if self.train_stratified and self.training:  # ray_samplers.py:321-329: the jitter is drawn here, like the reference
            rand = torch.rand((w.shape[0], 1 if self.single_jitter else n + 1), device=w.device)
            bins = be.pdf_resample_stratified(w, existing, n, rand, self.histogram_padding)[0]
        else:
            bins = be.pdf_resample(w, existing, n, self.histogram_padding)[0]
        if self.include_original:  # ray_samplers.py:360-361
            bins, _ = torch.sort(torch.cat([existing, bins], -1), -1)
        fr = ray_samples.frustums
        return RaySamples(Frustums(fr.origins, fr.directions, ray_samples.spacing_to_euclidean_fn(bins), fr.pixel_area), bins,
                          times=ray_samples.times, metadata=ray_samples.metadata, spacing=ray_samples.spacing)


@dataclass
class GaussiansStd:
    """utils/math.py GaussiansStd: isotropic gaussians, mean [N,S,3] and std [N,S] (one multisample)."""

    mean: Tensor
    std: Tensor


class Frustums:
    """cameras/rays.py:33-60 for contiguous samples: per-ray origins/directions [N,3], pixel_area [N,1] and the
    euclidean bin edges [N,S+1] (starts = edges[:, :-1], ends = edges[:, 1:]) -- never expanded to [N,S,3] views.
    The reference's keyword form `Frustums(origins=, directions=, starts=, ends=, pixel_area=)` is accepted when the bins
    are contiguous (ends[i] == starts[i+1], which every sampler of the path produces)."""

    def __init__(self, origins: Tensor, directions: Tensor, bin_edges: Optional[Tensor] = None, pixel_area: Optional[Tensor] = None,
                 starts: Optional[Tensor] = None, ends: Optional[Tensor] = None) -> None:
        if bin_edges is None:
            if starts is None or ends is None:
                raise ValueError("Frustums needs bin_edges or starts + ends")
            st = starts.reshape(origins.reshape(-1, 3).shape[0], -1)
            en = ends.reshape(st.shape)
            if st.shape[1] > 1 and not torch.equal(st[:, 1:], en[:, :-1]):
                raise NotImplementedError("non-contiguous sample bins (ends[i] != starts[i+1])")
            bin_edges = torch.cat([st, en[:, -1:]], dim=1)
        self.origins, self.directions, self.bin_edges, self.pixel_area = origins, directions, bin_edges, pixel_area

    @classmethod
    def get_mock_frustum(cls, device="cpu") -> "Frustums":
        """rays.py:126-139: a size-1 placeholder frustum."""
        one = torch.ones((1, 1), device=device)
        return cls(origins=torch.ones((1, 3), device=device), directions=torch.ones((1, 3), device=device), starts=one, ends=one,
                   pixel_area=one)

    @property
    def starts(self) -> Tensor:
        return self.bin_edges[:, :-1, None]

    @property
    def ends(self) -> Tensor:
        return self.bin_edges[:, 1:, None]

    @torch.no_grad()
    def get_positions(self, normalize_aabb: Optional[Tensor] = None) -> Tensor:
        """Frustums.get_positions (rays.py:50-59); with `normalize_aabb` [2,3] followed by
        SceneBox.get_normalized_positions (data/scene_box.py:63-79)."""
        be = get_backend(self.bin_edges.device)
        return be.frustum_positions(self.origins, self.directions, self.bin_edges, normalize_aabb)

    def get_fast_isotropic_gaussian(self, num_multisamples: int = 1) -> GaussiansStd:
        """rays.py:109-124 (NeuRAD uses one multisample, neurad_field.py:67).  Differentiable with respect to the origins
        and directions when they require grad (camera pose optimisation); the bins are detached as in the reference."""
        if num_multisamples != 1:
            raise NotImplementedError("num_multisamples != 1")
        assert self.pixel_area is not None, "frustums built without pixel_area"
        be = get_backend(self.bin_edges.device)
        if _needs_grad(self.origins, self.directions):
            return GaussiansStd(*AG.IsotropicGaussianFn.apply(be, self.origins, self.directions, self.pixel_area, self.bin_edges.detach()))
        with torch.no_grad():
            return GaussiansStd(*be.isotropic_gaussian(self.origins, self.directions, self.pixel_area, self.bin_edges))


@dataclass
class RaySamples:
    """cameras/rays.py:127-249 (the members the hot path reads).  `spacing_bins` is [S+1] when every ray shares the
    initial sampler's edges and [N,S+1] after PDF resampling; `spacing` = (kind, power_lambda, power_scaling, nears,
    fars) defines spacing_to_euclidean_fn (ray_samplers.py:119-120)."""

    frustums: Frustums
    spacing_bins: Tensor
    times: Optional[Tensor] = None  # [N,1]
    metadata: Dict[str, Tensor] = field(default_factory=dict)
    spacing: Optional[tuple] = None

    @property
    def shape(self) -> Tuple[int, int]:
        return (self.frustums.bin_edges.shape[0], self.frustums.bin_edges.shape[1] - 1)

    def without_last_sample(self) -> "RaySamples":
        """`ray_samples[..., :-1]` (neurad.py:385-386: the sky sample is dropped before depth and the training lists)."""
        fr = self.frustums
        sb = self.spacing_bins
        return RaySamples(Frustums(fr.origins, fr.directions, fr.bin_edges[:, :-1], fr.pixel_area), sb[..., :-1],
                          times=self.times, metadata=self.metadata, spacing=self.spacing)

    def per_ray_spacing_bins(self) -> Tensor:
        b = self.spacing_bins
        return b if b.dim() == 2 else b[None, :].expand(self.shape[0], -1).contiguous()

    @property
    def spacing_starts(self) -> Tensor:
        b = self.spacing_bins
        return b[:, :-1, None] if b.dim() == 2 else b[None, :-1, None]

    @property
    def spacing_ends(self) -> Tensor:
        b = self.spacing_bins
        return b[:, 1:, None] if b.dim() == 2 else b[None, 1:, None]

    @property
    def deltas(self) -> Tensor:
        return self.frustums.ends - self.frustums.starts

    @torch.no_grad()
    def spacing_to_euclidean_fn(self, bins: Tensor) -> Tensor:
        assert self.spacing is not None, "ray samples built without a spacing function"
        kind, lam, scaling, nears, fars = self.spacing
        return get_backend(bins.device).spacing_to_euclidean(bins, nears, fars, kind, lam, scaling)

    def get_weights(self, densities: Tensor) -> Tensor:
        """RaySamples.get_weights (rays.py:188-210): densities [N,S,1] -> weights [N,S,1]; differentiable with respect
        to the densities (hand-written backward operator) when they require grad."""
        be = get_backend(densities.device)
        deltas = self.deltas[..., 0].detach().contiguous()
        if torch.is_grad_enabled() and densities.requires_grad:
            return AG.DensityToWeightsFn.apply(be, deltas, densities[..., 0].contiguous())[..., None]
        with torch.no_grad():
            return be.density_to_weights(deltas, densities[..., 0])[..., None]


class SpacedSampler:
    """model_components/ray_samplers.py:56-132; `.training` + train_stratified select the stratified jitter (:107-115)."""

    spacing = "uniform"

    def __init__(self, num_samples: Optional[int] = None, train_stratified: bool = True, single_jitter: bool = False) -> None:
        self.num_samples = num_samples
        self.train_stratified, self.single_jitter = train_stratified, single_jitter
        self.training = False

    def _power(self) -> Tuple[float, float]:
        return -1.0, 0.1

    @torch.no_grad()
    def __call__(self, ray_bundle: RayBundle, num_samples: Optional[int] = None) -> RaySamples:
        assert ray_bundle.nears is not None and ray_bundle.fars is not None
        n = num_samples or self.num_samples
        assert n is not None
        be = get_backend(ray_bundle.origins.device)
        lam, scaling = self._power()
        if self.train_stratified and self.training:  # ray_samplers.py:107-115
            num_rays = ray_bundle.origins.reshape(-1, 3).shape[0]
            t_rand = torch.rand((num_rays, 1 if self.single_jitter else n + 1), device=ray_bundle.origins.device)
            bins_s, bins_e = be.spaced_sample_stratified(ray_bundle.nears, ray_bundle.fars, n, t_rand, self.spacing, lam, scaling)
        else:
            bins_s, bins_e = be.spaced_sample(ray_bundle.nears, ray_bundle.fars, n, self.spacing, lam, scaling)
        area = None if ray_bundle.pixel_area is None else ray_bundle.pixel_area.reshape(-1, 1)
        times = None if ray_bundle.times is None else ray_bundle.times.reshape(-1, 1)
        # (a view taken under no_grad does not carry the bundle's autograd history: keep [N,3] tensors as they are, so
        # that corrected origins / directions of a camera optimizer stay differentiable)
        o, d = ray_bundle.origins, ray_bundle.directions
        o, d = (o if o.dim() == 2 else o.reshape(-1, 3)), (d if d.dim() == 2 else d.reshape(-1, 3))
        return RaySamples(Frustums(o, d, bins_e, area), bins_s,
                          times=times, metadata=ray_bundle.metadata,
                          spacing=(self.spacing, lam, scaling, ray_bundle.nears, ray_bundle.fars))

    generate_ray_samples = __call__


class UniformSampler(SpacedSampler):
    """ray_samplers.py:135-156."""


class LinearDisparitySampler(SpacedSampler):
    """ray_samplers.py:159-180."""

    spacing = "lindisp"


class SqrtSampler(SpacedSampler):
    """ray_samplers.py:183-204."""

    spacing = "sqrt"


class LogSampler(SpacedSampler):
    """ray_samplers.py:207-228."""

    spacing = "log"


class PowerSampler(SpacedSampler):
    """ray_samplers.py:838-852 (NeuRAD's initial sampler: power_lambda=-1, power_scaling=0.1, neurad.py:232-235)."""

    spacing = "power"

    def __init__(self, num_samples: Optional[int] = None, lambda_: float = -1.5, scaling: float = 2.0, **kw) -> None:
        # the reference's argument names and defaults (ray_samplers.py:845); NeuRAD passes lambda_=-1, scaling=0.1
        if "power_lambda" in kw:
            lambda_ = kw.pop("power_lambda")
        if "power_scaling" in kw:
            scaling = kw.pop("power_scaling")
        super().__init__(num_samples, **kw)
        self.power_lambda, self.power_scaling = lambda_, scaling

    def _power(self) -> Tuple[float, float]:
        return self.power_lambda, self.power_scaling


class FeatureRenderer(nn.Module):
    """model_components/renderers.py:59-90, unpacked branch: sum_s w_s * f_s (differentiable: composite backward operator)."""

    @classmethod
    def forward(cls, features: Tensor, weights: Tensor) -> Tensor:
        be = get_backend(weights.device)
        if _needs_grad(features, weights):
            w = weights.reshape(weights.shape[0], weights.shape[1]).contiguous()
            return AG.CompositeFn.apply(be, w, features.contiguous(), None, None, False, False)[0]
        with torch.no_grad():
            return be.composite(weights, features, want_accumulation=False)["values"]


class RGBRenderer(nn.Module):
    """model_components/renderers.py:93-268: composite and blend a constant background ("random" / None = no blending,
    like black; "last_sample" is not provided).  In eval mode the samples' rgb go through nan_to_num first and the
    result is clamped to [0, 1]; in training mode neither (renderers.py:258-265)."""

    COLORS = {"white": (1.0, 1.0, 1.0), "black": (0.0, 0.0, 0.0), "red": (1.0, 0.0, 0.0), "green": (0.0, 1.0, 0.0),
              "blue": (0.0, 0.0, 1.0)}  # utils/colors.py:21-31

    def __init__(self, background_color="random") -> None:
        super().__init__()
        if isinstance(background_color, str) and background_color not in ("random",) + tuple(self.COLORS):
            raise NotImplementedError(f"background_color={background_color!r}")
        self.background_color = background_color

    @torch.no_grad()
    def _forward(self, rgb: Tensor, weights: Tensor) -> Tensor:
        bg = self.background_color
        if isinstance(bg, str):
            bg = None if bg == "random" else self.COLORS[bg]
        elif isinstance(bg, Tensor):
            bg = [float(v) for v in bg.reshape(-1)]
        be = get_backend(weights.device)
        out = be.composite(weights, rgb, background=bg, value_nan_to_num=not self.training, want_accumulation=False)["values"]
        return out if self.training else out.clamp_(0.0, 1.0)

    def forward(self, rgb: Tensor, weights: Tensor) -> Tensor:
        _no_backward("RGBRenderer", rgb, weights)
        return self._forward(rgb, weights)


class AccumulationRenderer(nn.Module):
    """model_components/renderers.py:322-350, unpacked branch (differentiable: composite backward operator)."""

    @classmethod
    def forward(cls, weights: Tensor) -> Tensor:
        be = get_backend(weights.device)
        if _needs_grad(weights):
            w = weights.reshape(weights.shape[0], weights.shape[1]).contiguous()
            return AG.CompositeFn.apply(be, w, None, None, None, True, False)[1]
        with torch.no_grad():
            return be.composite(weights)["accumulation"]


class DepthRenderer(nn.Module):
    """model_components/renderers.py:353-418: "median" or "expected" (with its batch-global clip)."""

    def __init__(self, method: str = "median") -> None:
        super().__init__()
        if method not in ("median", "expected"):
            raise NotImplementedError(f"Method {method} not implemented")
        self.method = method

    def forward(self, weights: Tensor, ray_samples: RaySamples) -> Tensor:
        _no_backward(f"DepthRenderer({self.method!r})", weights)  # NeuRAD trains with render_depth_simple (NeuRADModel.renderer_depth)
        fr = ray_samples.frustums
        be = get_backend(weights.device)
        with torch.no_grad():
            return be.composite(weights, starts=fr.starts.contiguous(), ends=fr.ends.contiguous(), depth_method=self.method,
                                want_accumulation=False)["depth"]


class ProposalNetworkSampler:
    """model_components/ray_samplers.py:569-666: initial sampler, then per proposal level density_fns[i] ->
    RaySamples.get_weights -> PDFSampler (stratified in training mode, `train()`); `step_cb` / `update_sched` gate the
    proposal networks' gradients.  Every step is one of the library's stage kernels; the fused `b200nerf_nff_render_fwd`
    does the same work (eval mode) without materialising any of these tensors."""

    def __init__(self, num_proposal_samples_per_ray: Tuple[int, ...] = (64,), num_nerf_samples_per_ray: int = 32,
                 num_proposal_network_iterations: int = 2, single_jitter: bool = False, update_sched=lambda x: 1,
                 initial_sampler: Optional[SpacedSampler] = None, pdf_sampler: Optional[PDFSampler] = None) -> None:
        if num_proposal_network_iterations < 1:
            raise ValueError("num_proposal_network_iterations must be >= 1")  # ray_samplers.py:597-598
        if initial_sampler is None:
            raise NotImplementedError("UniformLinDispPiecewiseSampler (the nerfstudio default) is not on NeuRAD's path; "
                                      "pass initial_sampler=PowerSampler(...) as neurad.py:232-235 does")
        self.num_proposal_samples_per_ray = num_proposal_samples_per_ray
        self.num_nerf_samples_per_ray = num_nerf_samples_per_ray
        self.num_proposal_network_iterations = num_proposal_network_iterations
        self.update_sched = update_sched
        self.initial_sampler = initial_sampler
        self.pdf_sampler = pdf_sampler if pdf_sampler is not None else PDFSampler(include_original=False, single_jitter=single_jitter)
        self._anneal, self._steps_since_update, self._step = 1.0, 0, 0
        self.training = False

    def train(self, mode: bool = True) -> "ProposalNetworkSampler":
        self.training = self.initial_sampler.training = self.pdf_sampler.training = mode
        return self

    def set_anneal(self, anneal: float) -> None:
        self._anneal = anneal

    def step_cb(self, step) -> None:
        self._step = step
        self._steps_since_update += 1

    def generate_ray_samples(self, ray_bundle: Optional[RayBundle] = None, density_fns: Optional[list] = None,
                             pass_ray_samples: bool = False) -> Tuple[RaySamples, List[Tensor], List[RaySamples]]:
        assert ray_bundle is not None
        assert density_fns is not None
        if not pass_ray_samples:
            density_fns = [lambda rs, f=f: f(rs.frustums.get_positions()) for f in density_fns]
        ray_bundle = ray_bundle.flatten()
        weights_list, ray_samples_list = [], []
        n = self.num_proposal_network_iterations
        weights = ray_samples = None
        # the proposal networks only receive gradients every update_sched(step) steps (ray_samplers.py:639, 656-661)
        updated = self._steps_since_update > self.update_sched(self._step) or self._step < 10
        for i_level in range(n + 1):
            is_prop = i_level < n
            num_samples = self.num_proposal_samples_per_ray[i_level] if is_prop else self.num_nerf_samples_per_ray
            with torch.no_grad():  # sample placement is not differentiated (bins.detach(), ray_samplers.py:363-364)
                if i_level == 0:
                    ray_samples = self.initial_sampler(ray_bundle, num_samples=num_samples)
                else:
                    annealed = weights if self._anneal == 1.0 else torch.pow(weights, self._anneal)
                    ray_samples = self.pdf_sampler(ray_bundle, ray_samples, annealed.detach(), num_samples=num_samples)
            if is_prop:
                if updated:
                    density = density_fns[i_level](ray_samples)
                else:
                    with torch.no_grad():
                        density = density_fns[i_level](ray_samples)
                weights = ray_samples.get_weights(density)
                weights_list.append(weights)
                ray_samples_list.append(ray_samples)
        if updated:
            self._steps_since_update = 0
        return ray_samples, weights_list, ray_samples_list

    __call__ = generate_ray_samples


class FieldHeadNames(Enum):
    """field_components/field_heads.py:28-44 (the heads NeuRAD's fields return)."""

    DENSITY = "density"
    SDF = "sdf"
    ALPHA = "alpha"
    FEATURE = "feature"


class NeuRADHashEncoding:
    """field_components/neurad_encoding.py:85-187 of one field of a NeuRADModel mirror (the parameters live in the model
    under the reference's names and are bound to the device context by it)."""

    def __init__(self, model: "NeuRADModel", field_index: int) -> None:
        self._model, self._field = model, field_index
        g = [model.config.grid, model.config.proposal_grid_1, model.config.proposal_grid_2][field_index].static
        self.scene_repr_dim = g.num_levels * g.hashgrid_dim

    def get_out_dim(self) -> int:
        return self.scene_repr_dim

    def forward(self, positions: GaussiansStd, times: Tensor, directions: Optional[Tensor] = None) -> Tuple[Tensor, Optional[Tensor]]:
        """(features [N*S, D], directions [N,S,3] in the actor frame where a sample is inside an actor | None); trains the
        tables (and, for the main field's grid, the actor trajectories) when they require grad, and passes a gradient to
        positions.mean when it requires one (camera pose optimisation)."""
        m = self._model
        be = m._bind()
        flip = m._draw_actor_flip(positions.mean.shape[0], self._field)
        tables = m._grid_params("field" if self._field == 0 else f"proposal_fields.{self._field - 1}")
        traj = [None, None]
        if self._field == 0 and m.config.n_actors:  # require_actor_grad: the main field's grid only (neurad_field.py:50,177)
            traj = [m._param("dynamic_actors.actor_rotations_6d"), m._param("dynamic_actors.actor_positions")]
        if _needs_grad(*tables, *traj, positions.mean):
            feats, dirs = AG.EncodingFn.apply(be, self._field, positions.mean, positions.std, times, directions, flip, traj[0], traj[1],
                                              tables[0], *tables[1:])
            return feats, (dirs if directions is not None else None)
        with torch.no_grad():
            out = be.neurad_encoding(self._field, positions.mean, positions.std, times, directions, flip=flip)
        return out["features"], out.get("directions")

    __call__ = forward


class NeuRADProposalField:
    """fields/neurad_field.py:186-216."""

    def __init__(self, model: "NeuRADModel", field_index: int) -> None:
        self._model, self._field = model, field_index
        self.hashgrid = NeuRADHashEncoding(model, field_index)

    def get_density(self, ray_samples: RaySamples) -> Tuple[Tensor, None]:
        """density [N,S,1] = trunc_exp(density_decoder(hashgrid(gaussians))) (neurad_field.py:208-213); with grad mode
        on and trainable parameters the backward operator delivers d/d(hash tables, density_decoder.weight), and d/d mean
        when the frustums' origins / directions require grad (camera pose optimisation)."""
        m = self._model
        pos = ray_samples.frustums.get_fast_isotropic_gaussian(num_multisamples=1)
        be = m._bind()
        flip = m._draw_actor_flip(ray_samples.shape[0], self._field)
        pre = f"proposal_fields.{self._field - 1}"
        tables = m._grid_params(pre)
        dec = m._param(f"{pre}.density_decoder.weight")
        if _needs_grad(*tables, dec, pos.mean):
            dens = AG.DensityFn.apply(be, self._field, pos.mean, pos.std, ray_samples.times, flip, tables[0], dec, *tables[1:])
            return dens[..., None], None
        with torch.no_grad():
            out = be.neurad_encoding(self._field, pos.mean, pos.std, ray_samples.times, None, want_features=False,
                                     want_density=True, flip=flip)
        return out["density"][..., None], None

    def get_outputs(self, ray_samples: RaySamples, density_embedding: Optional[Tensor] = None) -> dict:
        return {}


class NeuRADField:
    """fields/neurad_field.py:76-152 (use_sdf=True)."""

    def __init__(self, model: "NeuRADModel") -> None:
        self._model = model
        self.hashgrid = NeuRADHashEncoding(model, 0)

    def forward(self, ray_samples: RaySamples, compute_normals: bool = False) -> Dict[FieldHeadNames, Tensor]:
        """{FEATURE [N,S,32], SDF [N,S,1], ALPHA [N,S,1]}.  With grad mode on and trainable parameters (or sample means
        that require grad) every stage is an autograd node with a hand-written backward operator (hash tables, both MLPs,
        beta, sample means)."""
        if compute_normals:
            raise NotImplementedError("NeuRADField never computes normals (neurad_field.py:128)")
        m = self._model
        g = ray_samples.frustums.get_fast_isotropic_gaussian(m.config.num_multisamples)
        be = m._bind()
        flip = m._draw_actor_flip(ray_samples.shape[0])
        n, s = ray_samples.shape
        tables = m._grid_params("field")
        geo_wb = m._mlp_params("field.mlp_geo", 2)
        feat_wb = m._mlp_params("field.mlp_feature", 3)
        beta = m._param("field.sdf_to_density.beta")
        # the main field's grid has require_actor_grad (neurad_field.py:50): its features also train the trajectories
        traj = [m._param("dynamic_actors.actor_rotations_6d"), m._param("dynamic_actors.actor_positions")] if m.config.n_actors else [None, None]
        if _needs_grad(*tables, *geo_wb, *feat_wb, beta, *traj, g.mean):
            feats, dirs = AG.EncodingFn.apply(be, 0, g.mean, g.std, ray_samples.times, ray_samples.frustums.directions, flip,
                                              traj[0], traj[1], tables[0], *tables[1:])
            geo = AG.MlpFn.apply(be, feats, *geo_wb)
            h = AG.MlpFn.apply(be, AG.FieldMidFn.apply(be, geo, dirs), *feat_wb)
            feature, sdf, alpha = AG.FieldTailFn.apply(be, geo, h, beta)
            gdim = feature.shape[1]
            out = {"feature": feature.view(n, s, gdim), "sdf": sdf.view(n, s, 1), "alpha": alpha.view(n, s, 1)}
        else:
            with torch.no_grad():
                out = be.field_forward(g.mean, g.std, ray_samples.times, ray_samples.frustums.directions, flip=flip)
        return {FieldHeadNames.FEATURE: out["feature"], FieldHeadNames.SDF: out["sdf"], FieldHeadNames.ALPHA: out["alpha"]}

    __call__ = forward


class BasicBlock(nn.Module):
    """model_components/cnns.py:35-46 as a parameter container (same sub-module names, hence the same state_dict keys:
    `main_branch.0` Conv2d, `.1` BatchNorm2d, `.3` Conv2d, `.4` BatchNorm2d).  The arithmetic runs inside
    RGBDecoder.forward; calling a block on its own is not provided."""

    def __init__(self, in_dim: int, dim: int, kernel_size: int, padding: int, use_bn: bool = False) -> None:
        super().__init__()
        if in_dim != dim or kernel_size != 7 or padding != 3 or not use_bn:
            raise NotImplementedError("the b200 decoder implements NeuRAD's BasicBlock(32, 32, 7, 3, use_bn=True)")
        self.res_branch = nn.Identity()
        self.main_branch = nn.Sequential(
            nn.Conv2d(in_dim, dim, kernel_size=kernel_size, padding=padding), nn.BatchNorm2d(dim), nn.ReLU(inplace=True),
            nn.Conv2d(dim, dim, kernel_size=kernel_size, padding=padding), nn.BatchNorm2d(dim))
        self.final_activation = nn.ReLU(inplace=True)

    def forward(self, x: Tensor) -> Tensor:
        """cnns.py:45-46.  Only reached through RGBDecoder.forward(impl="torch") (training): the inference path evaluates
        the whole decoder with the fused wgmma convolutions and never calls the blocks one by one."""
        return self.final_activation(self.res_branch(x) + self.main_branch(x))


class RGBDecoder(nn.Sequential):
    """NeuRADModel.rgb_decoder (models/neurad.py:201-216): same module indices 0..8 and parameter names as the
    reference's nn.Sequential, so `load_state_dict` takes the reference's `rgb_decoder.*` tensors unchanged.
    forward takes the feature image channels-LAST, [B,H,W,C] (the ray order of get_nff_outputs; the reference permutes
    to NCHW and back, neurad.py:362-365) and returns rgb [B,3H,3W,3] in eval mode (BatchNorm running statistics)."""

    def __init__(self, in_dim: int = 48, hidden_dim: int = 32, upsample: int = 3) -> None:
        super().__init__(
            nn.Conv2d(in_dim, hidden_dim, kernel_size=1, padding=0), nn.ReLU(inplace=True),
            BasicBlock(hidden_dim, hidden_dim, kernel_size=7, padding=3, use_bn=True),
            BasicBlock(hidden_dim, hidden_dim, kernel_size=7, padding=3, use_bn=True),
            nn.ConvTranspose2d(hidden_dim, hidden_dim, kernel_size=upsample, stride=upsample),
            BasicBlock(hidden_dim, hidden_dim, kernel_size=7, padding=3, use_bn=True),
            BasicBlock(hidden_dim, hidden_dim, kernel_size=7, padding=3, use_bn=True),
            nn.Conv2d(hidden_dim, 3, kernel_size=1, padding=0), nn.Sigmoid())
        self._uid = next(_UIDS)

    def forward(self, features: Tensor, impl: str = "tc") -> Tensor:
        """impl "tc" / "tc_ldgsts" / "ref": the library's decoder kernels (inference: BatchNorm folded from its running
        statistics).  impl "torch": the nn.Sequential itself on torch's convolution library, differentiable and with
        BatchNorm batch statistics in training mode -- exactly what the reference runs (neurad.py:362-365).  It exists so
        that a model can TRAIN end to end (the NFF path through this library's backward operators, the decoder through
        torch) until the decoder has a native backward; it is never chosen implicitly."""
        if impl == "torch":
            x = features if features.dim() == 4 else features[None]
            x = x.permute(0, 3, 1, 2)
            for module in self:
                x = module(x)
            return x.permute(0, 2, 3, 1)
        if self.training:
            raise RuntimeError("the b200 rgb decoder kernels are inference-only (BatchNorm in eval mode); call .eval(), "
                               "or pass impl='torch' to train through torch's convolutions")
        with torch.no_grad():
            return self._forward_kernels(features, impl)

    def _forward_kernels(self, features: Tensor, impl: str) -> Tensor:
        be = get_backend(features.device)
        sd = self.state_dict()
        # the context is shared by every model on the device: re-bind unless THIS decoder, at these parameter versions,
        # is what the context holds (two decoders alternating would otherwise run with each other's weights)
        token = (self._uid, tuple(v._version for v in sd.values()), tuple(v.data_ptr() for v in sd.values()))
        if getattr(be, "_dec_owner", None) != token:
            be.set_rgb_decoder(sd, prefix="", bn_eps=self[2].main_branch[1].eps)
            be._dec_owner = token
        return be.rgb_decode(features, impl)


def _skew(v: Tensor) -> Tensor:
    """[C,3] -> the cross-product matrices [C,3,3] ([v]x w = v x w)."""
    z = torch.zeros_like(v[:, 0])
    return torch.stack([torch.stack([z, -v[:, 2], v[:, 1]], -1), torch.stack([v[:, 2], z, -v[:, 0]], -1),
                        torch.stack([-v[:, 1], v[:, 0], z], -1)], -2)


def exp_map_SO3xR3(tangent: Tensor) -> Tensor:
    """cameras/lie_groups.py exp_map_SO3xR3: [C,6] = (translation, rotation vector) -> [C,3,4].  The rotation is Rodrigues'
    formula R = I + sin(a)/a K + (1 - cos(a))/a^2 K^2 with K = [w]x and a = |w|; like the reference, a is taken as
    sqrt(max(|w|^2, 1e-4)) inside the two coefficients (K itself is not clamped); the translation is used as is."""
    w = tangent[:, 3:]
    a = (w * w).sum(dim=1).clamp(min=1e-4).sqrt()
    k = _skew(w)
    eye = torch.eye(3, dtype=tangent.dtype, device=tangent.device)
    rot = eye + (a.sin() / a)[:, None, None] * k + ((1.0 - a.cos()) / (a * a))[:, None, None] * (k @ k)
    return torch.cat([rot, tangent[:, :3, None]], dim=-1)


def exp_map_SE3(tangent: Tensor) -> Tensor:
    """cameras/lie_groups.py exp_map_SE3: [C,6] = (rho, rotation vector w) -> [C,3,4] = [R | V rho] with
    R = I + A K + B K^2, V = I + B K + C K^2, A = sin(a)/a, B = (1 - cos a)/a^2, C = (a - sin a)/a^3 (K = [w]x, a = |w|).
    Below a = 1e-2 the coefficients are their Taylor series (the reference switches at the same angle; the two differ by
    O(a^4) there)."""
    rho, w = tangent[:, :3], tangent[:, 3:]
    a = w.norm(dim=1)
    small = a < 1e-2
    a2 = a * a
    a_nz = torch.where(small, torch.ones_like(a), a)
    ca = torch.where(small, 1.0 - a2 / 6.0, a_nz.sin() / a_nz)
    cb = torch.where(small, 0.5 - a2 / 24.0, (1.0 - a_nz.cos()) / (a_nz * a_nz))
    cc = torch.where(small, 1.0 / 6.0 - a2 / 120.0, (a_nz - a_nz.sin()) / (a_nz * a_nz * a_nz))
    k = _skew(w)
    k2 = k @ k
    eye = torch.eye(3, dtype=tangent.dtype, device=tangent.device)
    rot = eye + ca[:, None, None] * k + cb[:, None, None] * k2
    v = eye + cb[:, None, None] * k + cc[:, None, None] * k2
    return torch.cat([rot, v @ rho[:, :, None]], dim=-1)


class CameraOptimizer(nn.Module):
    """cameras/camera_optimizers.py:84-233: per-camera pose corrections.  With mode "SO3xR3" / "SE3" the parameter
    `pose_adjustment` [num_cameras, 6] (translation | rotation, zero-initialised) maps through the exp map to [R | t];
    `apply_to_raybundle` then sets o' = o + t and d' = R d (not renormalised).  With mode "off" the module holds nothing.

    `non_trainable_camera_indices`: like the reference, forward() sets the correction ROWS at these positions of its
    output to the identity -- rows of the `indices` batch, not rows whose camera index matches (the two agree for
    get_correction_matrices(), whose batch is every camera in order)."""

    def __init__(self, config: CameraOptimizerConfig, num_cameras: int, device="cpu",
                 non_trainable_camera_indices: Optional[Tensor] = None, **kwargs) -> None:
        super().__init__()
        self.config = config
        self.num_cameras = num_cameras
        self.device = device
        self.non_trainable_camera_indices = non_trainable_camera_indices
        if config.mode != "off":
            self.pose_adjustment = nn.Parameter(torch.zeros((num_cameras, 6), device=device))

    def _get_pose_adjustment(self) -> Tensor:
        return self.pose_adjustment

    def forward(self, indices: Tensor) -> Tensor:
        """Correction matrices [len(indices), 3, 4] (identity with mode "off")."""
        if self.config.mode == "off":
            return torch.eye(4, device=indices.device)[None, :3, :4].tile(indices.shape[0], 1, 1)
        adj = self._get_pose_adjustment()[indices, :]
        out = exp_map_SO3xR3(adj) if self.config.mode == "SO3xR3" else exp_map_SE3(adj)
        if self.non_trainable_camera_indices is not None:
            idx = self.non_trainable_camera_indices.to(out.device)
            self.non_trainable_camera_indices = idx
            out[idx] = torch.eye(4, device=out.device)[:3, :4]
        return out

    def apply_to_raybundle(self, raybundle: RayBundle) -> None:
        """Corrects the flattened bundle in place (camera_optimizers.py:173-182): origins += t, directions = R d."""
        if self.config.mode == "off":
            return
        corr = self(raybundle.camera_indices.squeeze())
        raybundle.origins = raybundle.origins + corr[:, :3, 3]
        raybundle.directions = torch.bmm(corr[:, :3, :3], raybundle.directions[..., None]).squeeze().to(raybundle.origins)

    def apply_to_camera(self, camera) -> Tensor:
        """camera_optimizers.py:184-207: the corrected sensor-to-world [C,3,4] of a Cameras / Lidars object whose
        metadata names its camera (`cam_idx`); the rotation multiplies from the left, the translation is added."""
        s2w = camera.camera_to_worlds if hasattr(camera, "camera_to_worlds") else camera.lidar_to_worlds
        md = getattr(camera, "metadata", None)
        if self.config.mode == "off" or md is None or "cam_idx" not in md:
            return s2w
        adj = self(torch.tensor([md["cam_idx"]], dtype=torch.long, device=s2w.device))
        return torch.cat([torch.bmm(adj[..., :3, :3], s2w[..., :3, :3]), s2w[..., :3, 3:] + adj[..., :3, 3:]], dim=-1)

    def get_loss_dict(self, loss_dict: dict) -> None:
        """camera_opt_regularizer = mean |t| * trans_l2_penalty + mean |w| * rot_l2_penalty (:209-216)."""
        if self.config.mode != "off":
            adj = self._get_pose_adjustment()
            loss_dict["camera_opt_regularizer"] = (adj[:, :3].norm(dim=-1).mean() * self.config.trans_l2_penalty
                                                   + adj[:, 3:].norm(dim=-1).mean() * self.config.rot_l2_penalty)

    def get_correction_matrices(self) -> Tensor:
        return self(torch.arange(0, self.num_cameras).long())

    def get_metrics_dict(self, metrics_dict: dict) -> None:
        """Translation max / mean and rotation mean / max in degrees (:222-230)."""
        if self.config.mode != "off":
            trans = self.pose_adjustment[:, :3].detach().norm(dim=-1)
            rot = self.pose_adjustment[:, 3:].detach().norm(dim=-1)
            metrics_dict["camera_opt_translation_max"] = trans.max()
            metrics_dict["camera_opt_translation_mean"] = trans.mean()
            metrics_dict["camera_opt_rotation_mean"] = torch.rad2deg(rot.mean().cpu())
            metrics_dict["camera_opt_rotation_max"] = torch.rad2deg(rot.max().cpu())

    def get_param_groups(self, param_groups: dict) -> None:
        params = list(self.parameters())
        if self.config.mode != "off":
            assert len(params) > 0
            param_groups["camera_opt"] = params
        else:
            assert len(params) == 0


class ScaledCameraOptimizer(CameraOptimizer):
    """camera_optimizers.py:359-383: the pose adjustment is multiplied by the `weights` buffer before the exp map and the
    regulariser; the translation penalty is per axis on |t|."""

    def __init__(self, config: ScaledCameraOptimizerConfig, **kwargs) -> None:
        super().__init__(config, **kwargs)
        self.register_buffer("weights", torch.tensor(config.weights, dtype=torch.float32))
        self.trans_penalty = torch.tensor(config.trans_l2_penalty, dtype=torch.float32, device=self.device)

    def _get_pose_adjustment(self) -> Tensor:
        return self.pose_adjustment * self.weights

    def get_loss_dict(self, loss_dict: dict) -> None:
        if self.config.mode != "off":
            adj = self._get_pose_adjustment()
            self.trans_penalty = self.trans_penalty.to(adj.device)
            loss_dict["camera_opt_regularizer"] = ((adj[:, :3].abs() * self.trans_penalty).mean()
                                                   + adj[:, 3:].norm(dim=-1).mean() * self.config.rot_l2_penalty)


def make_camera_optimizer(config: Optional[CameraOptimizerConfig], num_cameras: int, device="cpu",
                          non_trainable_camera_indices: Optional[Tensor] = None) -> CameraOptimizer:
    """CameraOptimizerConfig.setup(): the scaled variant for a ScaledCameraOptimizerConfig."""
    config = CameraOptimizerConfig() if config is None else config
    cls = ScaledCameraOptimizer if isinstance(config, ScaledCameraOptimizerConfig) else CameraOptimizer
    return cls(config=config, num_cameras=num_cameras, device=device, non_trainable_camera_indices=non_trainable_camera_indices)


ACTOR_EDIT_KEYS = ("lateral", "longitudinal", "height", "rotation", "index")


class DynamicActors:
    """The non-parameter state of model_components/dynamic_actors.py:43-104 that rendering reads: `actor_editing`, the dict
    the viewer sliders and ADPipeline._update_actor_fids write, with the reference's keys and defaults.  In eval mode every
    render renders the actors at the edited poses (B200Backend.set_actor_edit has the semantics); training ignores it.
    The trajectories themselves are the model's `dynamic_actors.*` parameters."""

    def __init__(self) -> None:
        self.actor_editing = {"lateral": 0.0, "longitudinal": 0.0, "rotation": 0.0, "index": -1.0, "height": 0.0}


class NeuRADModel(nn.Module):
    """models/neurad.py:165 with the reference's parameter names: `state_dict()` / `load_state_dict()` speak the reference's
    dotted keys (`field.hashgrid.static_grid.hash_table`, ...; a `_model.` prefix as in `checkpoint["pipeline"]` is accepted),
    so `load_state_dict(reference_checkpoint["pipeline"], strict=False)` binds the tensors the path uses and raises if a
    hot-path tensor is missing.  Internally the tensors are registered under mangled names (dots are not allowed in
    parameter names); hooks translate in both directions.

    `get_nff_outputs` is ONE fused kernel launch (ray sampling, both proposal rounds, main field, compositing); the
    reference's 32 768-ray chunk loop (neurad.py:650-659) is unnecessary because nothing per-sample goes to HBM."""

    def __init__(self, config: NeuRADConfig, trajectories: Optional[List[dict]] = None, implementation: str = "torch",
                 camera_optimizer: Optional[CameraOptimizerConfig] = None, num_cameras: int = 1, use_camopt_in_eval: bool = False,
                 non_trainable_camera_indices: Optional[Tensor] = None) -> None:
        """`implementation`: which of the reference's two parameter layouts the model holds (models/neurad.py:146) --
        "torch" (per-level hashed tables, nn.Linear MLPs; trainable here) or "tcnn" (the reference's default: flat
        `tcnn_encoding.params` vectors in tiny-cuda-nn's layout, so that a tcnn-trained checkpoint loads with
        `load_state_dict`; inference through the fused kernels only -- SURVEY 8f row f3, tcnn_compat.py).

        `camera_optimizer` / `use_camopt_in_eval`: ADModelConfig's fields (models/ad_model.py:40-45); None = mode "off".
        `num_cameras` sizes `camera_optimizer.pose_adjustment` (the reference's num_train_data)."""
        super().__init__()
        from . import scene  # synthetic init = the reference's random init shapes

        if implementation not in ("torch", "tcnn"):
            raise ValueError("implementation must be 'torch' or 'tcnn'")
        self.config = config
        self.implementation = implementation
        make = scene.make_params if implementation == "torch" else scene.make_params_tcnn
        p = make(config, seed=0, table_scale=1e-3, trajectories=trajectories)
        self._names = []
        for k, v in p.items():
            if k == "static_scale":
                continue
            name = k.replace(".", "__")
            self._names.append((name, k))
            trainable = not k.startswith("dynamic_actors.") or k in ("dynamic_actors.actor_positions", "dynamic_actors.actor_rotations_6d")
            if v.dtype.is_floating_point and trainable and not k.endswith("scalings"):  # optimize_trajectories (dynamic_actors.py:37)
                self.register_parameter(name, nn.Parameter(v, requires_grad=False))
            else:
                self.register_buffer(name, v)
        # not part of the reference's state dict (a float passed to field.setup, neurad.py:180-184): non-persistent
        self.register_buffer("static_scale", torch.tensor(float(config.static_scale)), persistent=False)
        self.rgb_decoder = RGBDecoder(config.nff_out_dim + config.appearance_dim, config.rgb_hidden_dim, config.rgb_upsample_factor)
        self._uid = next(_UIDS)
        self.register_state_dict_post_hook(NeuRADModel._state_dict_out_hook)
        self.register_load_state_dict_pre_hook(NeuRADModel._state_dict_in_hook)
        # the reference's sub-modules (neurad.py:180-254), as views onto this model's parameters
        self.field = NeuRADField(self)
        self.proposal_fields = [NeuRADProposalField(self, 1), NeuRADProposalField(self, 2)]
        sp = config.sampling
        self.sampler = ProposalNetworkSampler(
            num_nerf_samples_per_ray=sp.num_nerf_samples, num_proposal_samples_per_ray=tuple(sp.num_proposal_samples),
            num_proposal_network_iterations=len(sp.num_proposal_samples),
            single_jitter=sp.single_jitter,
            initial_sampler=PowerSampler(lambda_=sp.power_lambda, scaling=sp.power_scaling),
            pdf_sampler=PDFSampler(include_original=False, single_jitter=sp.single_jitter, histogram_padding=sp.histogram_padding),
            update_sched=lambda x: 0,
        )
        # neurad.py:248 builds `[lambda x: prop_field.get_density(x)[0] for prop_field in self.proposal_fields]`: the
        # closures bind late, so EVERY entry evaluates the LAST proposal field (DESIGN.md section 2).  Same here.
        last = self.proposal_fields[-1]
        self.density_fns = [lambda ray_samples: last.get_density(ray_samples)[0] for _ in self.proposal_fields]
        self.renderer_feat = FeatureRenderer()
        self.renderer_accumulation = AccumulationRenderer()
        # ad_model.py:70-72; state dict keys camera_optimizer.pose_adjustment (+ .weights) as in the reference
        self.camera_optimizer = make_camera_optimizer(camera_optimizer, num_cameras, non_trainable_camera_indices=non_trainable_camera_indices)
        self.use_camopt_in_eval = use_camopt_in_eval
        # lidar metrics (neurad.py:268-271); the chamfer distance runs on the library's all-pairs kernel
        self.median_l2, self.mean_rel_l2, self.rmse = M.median_l2, M.mean_rel_l2, M.rmse
        self.chamfer_distance = lambda pred, gt: M.chamfer_distance(pred, gt, 1_000, True)
        # camera metrics (neurad.py:265-267).  PSNR and SSIM run on the library's kernels; LPIPS needs network weights the
        # library does not ship, so `lpips` is any callable (image, rgb) -> value on [1, 3, H, W] tensors, e.g. torchmetrics'
        # LearnedPerceptualImagePatchSimilarity(normalize=True), and camera batches are refused until the caller assigns one.
        self.ssim = M.ssim
        self.lpips = None
        # get_loss_dict's perceptual term (neurad.py:260, 537-538): any callable (rgb, image) -> loss, e.g. the reference's
        # VGGPerceptualLossPix2Pix.  The library ships no VGG19 weights, so it is None until the caller assigns one.
        self.vgg_loss = None
        self.dynamic_actors = DynamicActors()

    # -- nn.Module state dict in the reference's key format --------------------------------------------------------
    @staticmethod
    def _state_dict_out_hook(module, state_dict, prefix, local_metadata):
        for name, key in module._names:
            if prefix + name in state_dict:
                state_dict[prefix + key] = state_dict.pop(prefix + name)

    @staticmethod
    def _state_dict_in_hook(module, state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys, error_msgs):
        pipeline_prefix = prefix + "_model."
        if any(k.startswith(pipeline_prefix) for k in state_dict):  # checkpoint["pipeline"]: `_model.<key>` (+ datamanager keys)
            for k in [k for k in state_dict if k.startswith(prefix)]:
                v = state_dict.pop(k)
                if k.startswith(pipeline_prefix):
                    state_dict[prefix + k[len(pipeline_prefix):]] = v
        for name, key in module._names:
            if prefix + key in state_dict:
                state_dict[prefix + name] = state_dict.pop(prefix + key)

    def load_state_dict(self, state_dict, strict: bool = True, assign: bool = False):
        """nn.Module.load_state_dict on the reference's keys.  Even with strict=False a missing tensor of THIS path (grids,
        MLPs, decoders, appearance embedding, actor trajectories) raises: silently keeping a random init is never wanted.
        The rgb decoder stays optional in a hot-path-only state dict; keys of other subsystems are ignored when not strict.
        With a camera optimizer that is on, `camera_optimizer.pose_adjustment` (and `.weights`) are required too."""
        res = super().load_state_dict(dict(state_dict), strict=strict, assign=assign)
        back = {n: k for n, k in self._names}
        # a camera optimizer that is on needs its pose corrections (mode "off" has no tensors, as in the reference)
        missing = [back.get(k, k) for k in res.missing_keys if k in back or k.startswith("camera_optimizer.")]
        if missing:
            raise KeyError(f"state dict lacks hot-path tensors: {missing[:6]}{' ...' if len(missing) > 6 else ''}")
        return res

    def train(self, mode: bool = True) -> "NeuRADModel":
        """nn.Module.train, also reaching the samplers (nn.Modules in the reference): stratified jitter and the random
        actor flip are training-mode behaviour (ray_samplers.py:107-115, 321-329; neurad_encoding.py:212-219)."""
        super().train(mode)
        if hasattr(self, "sampler"):
            self.sampler.train(mode)
        return self

    # -- state dict under the reference's dotted names ----------------------------------------------------------
    def reference_state_dict(self) -> Dict[str, Tensor]:
        return {k: getattr(self, n) for n, k in self._names}

    def load_reference_state_dict(self, sd: Dict[str, Tensor]) -> None:
        """Copy tensors from a reference `NeuRADModel.state_dict()` (keys like
        `field.hashgrid.static_grid.hash_table`, `proposal_fields.1.density_decoder.weight`); unknown keys (rgb
        decoder, losses) are ignored, missing hot-path keys raise; the camera optimizer's tensors are required when its
        mode is not "off" and ignored otherwise."""
        for n, k in self._names:
            if k not in sd:
                raise KeyError(f"reference state dict lacks {k}")
            with torch.no_grad():  # in place on the tensor itself (not .data): bumps _version, which _bind() watches
                getattr(self, n).copy_(sd[k].to(getattr(self, n).dtype))
        for k, t in self.camera_optimizer.state_dict(keep_vars=True).items():
            if "camera_optimizer." + k not in sd:
                raise KeyError(f"reference state dict lacks camera_optimizer.{k}")
            with torch.no_grad():
                t.copy_(sd["camera_optimizer." + k].to(t.dtype))
        dec = {k[len("rgb_decoder."):]: v for k, v in sd.items() if k.startswith("rgb_decoder.")}
        if dec:  # the camera decoder is optional in a hot-path-only state dict
            self.rgb_decoder.load_state_dict(dec, strict=False)

    def _bind(self) -> B200Backend:
        be = get_backend(self.static_scale.device)
        # The backend is a per-device singleton shared by every model of the process (EMA / teacher-student pairs, two
        # checkpoints side by side): the context records WHO bound it, and a model re-binds unless it is the owner at the
        # current parameter versions and storage (in-place updates bump _version; .to() / load_state_dict may swap storage).
        tensors = [getattr(self, n) for n, _ in self._names] + [self.static_scale]
        token = (self._uid, tuple(t._version for t in tensors), tuple(t.data_ptr() for t in tensors))
        if getattr(be, "_owner", None) != token:
            params = self.reference_state_dict()
            params["static_scale"] = self.static_scale
            be.load_params(self.config, params)
            be._owner = token
        # DynamicActors.get_boxes2world edits only when not self.training (dynamic_actors.py:261-265)
        ed = self.dynamic_actors.actor_editing
        be.set_actor_edit(**({} if self.training else {k: ed[k] for k in ACTOR_EDIT_KEYS}))
        return be

    # -- forward API --------------------------------------------------------------------------------------------
    def get_nff_outputs(self, ray_bundle: RayBundle, calc_lidar_losses: bool = False, fused: Optional[bool] = None) -> Dict[str, Tensor]:
        """neurad.py:368-421 (eval): features [N,48], depth, accumulation, prop_depth_0/1 [N,1].

        fused=True (default): ONE kernel pair for the whole function.  fused=False: the reference's own module walk
        (sampler with density_fns -> field -> _render_weights -> renderers -> appearance), every step a stage kernel of
        the library -- the per-module API of SURVEY 8b; additionally returns the reference's training-side extras
        `weights_list` / `ray_samples_list` (neurad.py:404-405)."""
        # only the parameters of THIS path count (the rgb decoder's nn.Conv2d weights require grad by default, but it is
        # evaluated after this function and is inference-only); camera_optimizer.pose_adjustment counts through the
        # bundle: a bundle corrected by a trainable camera optimizer has origins / directions that require grad
        wants_grad = torch.is_grad_enabled() and (any(getattr(self, n).requires_grad for n, _ in self._names)
                                                  or _needs_grad(ray_bundle.origins, ray_bundle.directions))
        if self.implementation == "tcnn" and (wants_grad or fused is False):
            raise NotImplementedError("tiny-cuda-nn-layout parameters render through the fused kernels only (inference of "
                                      "tcnn-trained checkpoints); the module walk and training use the torch layout")
        be = self._bind()
        if fused is None:
            fused = not wants_grad  # the fused kernels are forward-only; training walks the modules (autograd operators)
        if fused:
            if wants_grad:
                raise RuntimeError("the fused renderer has no backward pass: call get_nff_outputs(fused=False) (or None) to train")
            with torch.no_grad():
                return be.render(ray_bundle.as_backend_dict())
        rb = self._scale_pixel_area(ray_bundle.flatten())
        ray_samples, prop_ray_samples, prop_weights = self._get_ray_samples(rb)
        out = self.field(ray_samples)
        weights = self._render_weights(out, ray_samples)
        accumulation = self._composite(weights, want_acc=True)[1]
        # the sky sample takes the remaining transmittance (neurad.py:379-381)
        weights = torch.cat((weights[:, :-1], weights[:, -1:] + 1.0 - accumulation[:, None]), dim=1)
        features = self._composite(weights, values=out[FieldHeadNames.FEATURE])[0]
        features = torch.cat([features, self._get_appearance_embedding(rb, features)], dim=-1)
        res = {"features": features, "accumulation": accumulation,
               "depth": self.renderer_depth(weights[:, :-1], ray_samples, drop_last=True)}  # sky sample left out (neurad.py:386-390)
        lidar_losses = self.training and calc_lidar_losses
        for i, (w, rs) in enumerate(zip(prop_weights, prop_ray_samples)):
            res[f"prop_depth_{i}"] = self.renderer_depth(w, rs)
            if lidar_losses:  # neurad.py:402-404
                weights_mask = (~rs.metadata["is_close_to_lidar"]) & rs.metadata["is_lidar"].reshape(-1, 1, 1).bool()
                res[f"prop_weights_loss_{i}"] = ((w * weights_mask) ** 2).sum()
        if lidar_losses:  # neurad.py:410-419 (the sky sample is already dropped there)
            md = ray_samples.metadata
            weights_mask = ((~md["is_close_to_lidar"][:, :-1]) & md["is_lidar"].reshape(-1, 1, 1).bool()).squeeze(-1)
            weights_idx = weights_mask.nonzero(as_tuple=True)
            res["non_nearby_weights"] = weights[:, :-1][weights_idx]
            lidar_start_ray = md["is_lidar"].reshape(-1).int().argmax()  # argmax gives the first True
            res["non_nearby_lidar_ray_indices"] = weights_idx[0] - lidar_start_ray
        # neurad.py:385-386, 404-405: the sky sample is dropped from the final level before the lists are built
        res["weights_list"] = prop_weights + [weights[:, :-1]]
        res["ray_samples_list"] = prop_ray_samples + [ray_samples.without_last_sample()]
        return res

    def _scale_pixel_area(self, ray_bundle: RayBundle) -> RayBundle:
        """neurad.py:702-709: camera rays cover upsample^2 pixels."""
        area = ray_bundle.pixel_area
        is_lidar = ray_bundle.metadata.get("is_lidar")
        scale = float(self.config.rgb_upsample_factor**2)
        scaled = area * scale if is_lidar is None else torch.where(is_lidar.reshape(area.shape).bool(), area, area * scale)
        out = ray_bundle._map(lambda t: t)
        out.pixel_area = scaled
        return out

    def _get_ray_samples(self, ray_bundle: RayBundle):
        """neurad.py:443-459: far clamp, proposal sampling, the last sample stretched to the sky."""
        sky = self.config.sampling.sky_distance
        n = len(ray_bundle)
        dev = ray_bundle.origins.device
        ray_bundle.fars = torch.full((n, 1), sky, device=dev) if ray_bundle.fars is None else ray_bundle.fars.clamp_max(sky)
        ray_bundle.nears = torch.zeros((n, 1), device=dev) if ray_bundle.nears is None else ray_bundle.nears
        ray_samples, prop_weights, prop_ray_samples = self.sampler(ray_bundle, self.density_fns, pass_ray_samples=True)
        edges = ray_samples.frustums.bin_edges
        edges[:, -1] += sky - edges[:, -1]  # `ends[-1] += sky - ends[-1]`, the reference's exact expression
        ray_samples.spacing_bins[:, -1] = 1 - 1e-7  # "Hacky, but sky is ish at infinity" (neurad.py:455)
        # the reference computes the masks whenever is_lidar is present (and needs directions_norm for it); bundles without
        # the measured distances simply get no masks here, and calc_lidar_losses then fails loudly on the missing key
        if self.training and "is_lidar" in ray_bundle.metadata and "directions_norm" in ray_bundle.metadata:
            self._compute_is_close_to_lidar(ray_samples, *prop_ray_samples)
        return ray_samples, prop_ray_samples, prop_weights

    def _compute_is_close_to_lidar(self, *all_ray_samples: RaySamples) -> None:
        """neurad.py:677-700: metadata["is_close_to_lidar"] [N,S,1] for every level (lidar carving supervision)."""
        be = self._bind()
        for rs in all_ray_samples:
            if rs is None:
                continue
            md = rs.metadata = dict(rs.metadata)  # one dict per level (the reference's metadata is per RaySamples too)
            md["is_close_to_lidar"] = be.lidar_carving_mask(rs.frustums.bin_edges, md["is_lidar"], md["directions_norm"],
                                                            md.get("did_return"), self.config.carving_epsilon,
                                                            self.config.non_return_lidar_distance)[..., None]

    def _render_weights(self, outputs, ray_samples: RaySamples) -> Tensor:
        """neurad.py:711-724, use_sdf branch: nerfacc.render_weight_from_alpha on [N,S]."""
        alphas = outputs[FieldHeadNames.ALPHA][..., 0]
        be = self._bind()
        if torch.is_grad_enabled() and alphas.requires_grad:
            return AG.AlphaToWeightsFn.apply(be, alphas.contiguous())[..., None]
        with torch.no_grad():
            return be.alpha_to_weights(alphas)[..., None]

    def _composite(self, weights: Tensor, values: Optional[Tensor] = None, starts: Optional[Tensor] = None,
                   ends: Optional[Tensor] = None, want_acc: bool = False):
        """(values [N,C], accumulation [N,1], depth [N,1]) through the composite operator; an autograd node when an input
        requires grad."""
        be = self._bind()
        want_depth = starts is not None
        w = weights.reshape(weights.shape[0], weights.shape[1]).contiguous()
        st = None if starts is None else starts.reshape(w.shape).detach().contiguous()
        en = None if ends is None else ends.reshape(w.shape).detach().contiguous()
        v = None if values is None else values.contiguous()
        if torch.is_grad_enabled() and (w.requires_grad or (v is not None and v.requires_grad)):
            return AG.CompositeFn.apply(be, w, v, st, en, want_acc, want_depth)
        with torch.no_grad():
            out = be.composite(w, v, st, en, "simple" if want_depth else None, want_accumulation=want_acc)
        return out.get("values"), out.get("accumulation"), out.get("depth")

    def renderer_depth(self, weights: Tensor, ray_samples: RaySamples, drop_last: bool = False) -> Tensor:
        """render_depth_simple (neurad.py:727-734): sum_i w_i (start_i + end_i) / 2, un-normalised; `drop_last` is the
        `[..., :-1, :]` slice that leaves the sky sample out (neurad.py:389-390)."""
        fr = ray_samples.frustums
        st, en = fr.starts, fr.ends
        if drop_last:
            st, en = st[:, :-1], en[:, :-1]
        return self._composite(weights, starts=st, ends=en)[2]

    # -- parameter access under the reference's names (leaf tensors, so autograd delivers .grad to them) ----------
    def _param(self, key: str) -> Tensor:
        return getattr(self, key.replace(".", "__"))

    def _grid_params(self, prefix: str) -> List[Tensor]:
        """[static table, actor table 0, actor table 1, ...] of `prefix`.hashgrid."""
        tabs = [self._param(f"{prefix}.hashgrid.static_grid.hash_table")]
        return tabs + [self._param(f"{prefix}.hashgrid.actor_grids.{a}.hash_table") for a in range(self.config.n_actors)]

    def _mlp_params(self, prefix: str, n_layers: int) -> List[Tensor]:
        out: List[Tensor] = []
        for i in range(n_layers):
            out += [self._param(f"{prefix}.layers.{i}.weight"), self._param(f"{prefix}.layers.{i}.bias")]
        return out

    def _draw_actor_flip(self, n_rays: int, field_index: int = 0) -> Optional[Tensor]:
        """Training-mode random actor flip, one draw per ray and per encoding call (neurad_encoding.py:212-219):
        -1 with probability flip_prob of that field's grid (0.25 main, 0.5 proposal), else +1.  None in eval mode /
        without actors."""
        p = [self.config.grid, self.config.proposal_grid_1, self.config.proposal_grid_2][field_index].flip_prob
        if not self.training or self.config.n_actors == 0 or p <= 1e-7:
            return None
        return torch.bernoulli(torch.full((n_rays,), p, device=self.static_scale.device)) * -2 + 1

    def _get_appearance_embedding(self, ray_bundle: RayBundle, features: Tensor) -> Tensor:
        """neurad.py:423-441: per-sensor embedding, linearly interpolated in time (temporal_appearance_freq), or with
        use_temporal_appearance = False the sensor's one row."""
        sd = self.reference_state_dict()
        emb = sd["appearance_embedding.weight"]
        n = len(ray_bundle)
        sensor = ray_bundle.metadata.get("sensor_idxs")
        sensor = torch.zeros(n, dtype=torch.long, device=emb.device) if sensor is None else sensor.reshape(-1).long()
        if not self.config.use_temporal_appearance:
            if emb.requires_grad and emb.shape[0] <= 4096:
                # training: a one-hot [N, E] @ [E, 16] product, for the same reason as below; the forward is exact (one
                # nonzero term per row)
                m = torch.zeros(n, emb.shape[0], device=emb.device, dtype=emb.dtype)
                m.scatter_(1, sensor[:, None], 1.0)
                return m @ emb
            return emb[sensor]
        eps = self.config.embeds_per_sensor
        t = ray_bundle.times.reshape(-1) / self.config.duration * eps
        before = t.floor().clamp(0, eps - 1)
        after = (before + 1).clamp(0, eps - 1)
        frac = (t - before)[:, None]
        i0, i1 = (before + sensor * eps).long(), (after + sensor * eps).long()
        if emb.requires_grad and emb.shape[0] <= 4096:
            # training: the same two-term interpolation as one [N, E] @ [E, 16] product (E = sensors x embeds_per_sensor = 56).
            # Autograd's backward of `emb[i]` with ~1000 duplicates per row is a serialised index_put (1.3 ms per step for
            # 57 k rays, profiles/r02_train_step_launches.txt); the product's backward is a 56 x N x 16 GEMM.
            m = torch.zeros(n, emb.shape[0], device=emb.device, dtype=emb.dtype)
            m.scatter_add_(1, i0[:, None], 1 - frac)
            m.scatter_add_(1, i1[:, None], frac)
            return m @ emb
        return emb[i0] * (1 - frac) + emb[i1] * frac

    def decode_features(self, features: Tensor, patch_size: Optional[Tuple[int, int]] = None, is_lidar: Optional[Tensor] = None,
                        intensity_for_cam: bool = False):
        """neurad.py:337-366.  With `patch_size` (the reference's signature) returns (rgb, intensity, ray_drop_logits):
        lidar rays (`is_lidar` [N,1]) go through `lidar_decoder` (MLP 48->32->32->2 on the wgmma operator, intensity =
        sigmoid), camera rays are reshaped to patches [B,ph,pw,C] and decoded by `rgb_decoder` to [B,3ph,3pw,3]
        (channels-last in and out: the reference's two permutes cancel).  Without `patch_size`: the lidar half only,
        (intensity, ray_drop_logits) for all rows."""
        be = self._bind()
        wb = self._mlp_params("lidar_decoder", 3)

        def lidar_head(x):
            if x.shape[0] == 0:
                return x.new_zeros(0, 2)
            if torch.is_grad_enabled() and (x.requires_grad or any(t.requires_grad for t in wb)):
                return AG.MlpFn.apply(be, x.contiguous(), *wb)
            with torch.no_grad():
                return be.mlp_fwd(x, wb[0::2], wb[1::2])

        if patch_size is None:
            o = lidar_head(features)
            return o[..., 0:1].sigmoid(), o[..., 1:2]
        if is_lidar is None:
            lidar_features, cam_features = features[:0], features
        else:
            m = is_lidar.reshape(-1).bool()
            lidar_features, cam_features = features[m], features[~m]
        if intensity_for_cam:
            o = lidar_head(features)
        elif lidar_features.numel() > 0:
            o = lidar_head(lidar_features)
        else:
            o = None
        intensity, ray_drop_logit = (None, None) if o is None else (o[..., 0:1].sigmoid(), o[..., 1:2])
        rgb = None
        if cam_features.numel() > 0:
            patches = cam_features.reshape(-1, *patch_size, cam_features.shape[-1])
            # inference: the wgmma decoder kernels.  Training (BatchNorm batch statistics + autograd): explicitly the torch
            # modules, as the reference does -- the native decoder has no backward yet (DESIGN.md section 8)
            rgb = self.rgb_decoder(patches, impl="torch" if (self.rgb_decoder.training and torch.is_grad_enabled()) else "tc")
        return rgb, intensity, ray_drop_logit

    def get_outputs(self, ray_bundle: RayBundle, patch_size: Tuple[int, int], intensity_for_cam: bool = False,
                    calc_lidar_losses: bool = True) -> Dict[str, Tensor]:
        """neurad.py:311-335: in training mode (or with use_camopt_in_eval) the camera optimizer corrects the flattened
        bundle first (:318-319; a no-op with mode "off"), then get_nff_outputs + decode_features; `features` is dropped
        from the result."""
        if (self.training or self.use_camopt_in_eval) and self.camera_optimizer.config.mode != "off":
            ray_bundle = ray_bundle.flatten()
            self.camera_optimizer.apply_to_raybundle(ray_bundle)
        out = self.get_nff_outputs(ray_bundle, calc_lidar_losses)
        rgb, intensity, ray_drop_logits = self.decode_features(out["features"], patch_size, ray_bundle.flatten().metadata.get("is_lidar"),
                                                               intensity_for_cam)
        out.pop("features", None)
        for k, v in (("rgb", rgb), ("intensity", intensity), ("ray_drop_logits", ray_drop_logits)):
            if v is not None:
                out[k] = v
        return out

    def forward(self, ray_bundle: RayBundle, patch_size: Tuple[int, int] = (1, 1), intensity_for_cam: bool = False,
                calc_lidar_losses: bool = True) -> Dict[str, Tensor]:
        return self.get_outputs(ray_bundle, patch_size, intensity_for_cam, calc_lidar_losses)

    @torch.no_grad()
    def get_outputs_for_lidar(self, lidar: "Lidars", batch: Dict[str, Tensor]) -> Tuple[Dict[str, Tensor], Dict[str, Tensor]]:
        """models/ad_model.py:84-113: rays from the sweep's points, the model outputs, and the predicted points in the
        lidar frame (origin + direction * depth through the inverse sensor pose)."""
        points = batch["lidar"]
        assert isinstance(batch["lidar_idx"], int), "All lidar points are assumed to be from the same scan."
        ray_bundle = lidar.generate_rays(lidar_indices=0, points=points, keep_shape=True)
        md = ray_bundle.metadata
        batch["is_lidar"], batch["distance"], batch["did_return"] = md["is_lidar"], md["directions_norm"], md["did_return"]
        outputs = self.get_outputs_for_camera_ray_bundle(ray_bundle)
        l2w = lidar.lidar_to_worlds[0]
        rot_t = l2w[:3, :3].t()  # pose_inverse (utils/poses.py:42-55): [R^T | -R^T t]
        pts = ray_bundle.origins + ray_bundle.directions * outputs["depth"]
        outputs["points"] = pts @ rot_t.t() - (rot_t @ l2w[:3, 3])
        return outputs, batch

    # -- training objective ---------------------------------------------------------------------------------------
    def get_metrics_dict(self, outputs: Dict[str, Tensor], batch: Dict[str, Tensor]) -> Dict[str, Tensor]:
        """neurad.py:461-529 with the reference's keys and conditions.  Image batches: psnr.  Lidar batches: the four eval
        metrics (the reference's boolean-mask gathers) and, in training mode, the lidar losses on the library's kernels
        (losses.lidar_losses: depth with the non-return targets and the exact 0.95-quantile mask, intensity, ray drop,
        the per-round proposal depths; no host synchronisation) and the carving sums.  Training with `weights_list`:
        distortion.  Always: sdf_to_density and the camera optimizer's metrics.

        The batch is the reference's: is_lidar / did_return [N,1] over all rays, distance [n,1] and lidar [n,>=4] over the
        lidar rays; the outputs those of get_outputs (intensity and ray_drop_logits in lidar rows)."""
        from . import losses as L

        device = self.static_scale.device
        cfg = self.config
        metrics_dict: Dict[str, Tensor] = {}
        if "image" in batch:
            image, rgb = batch["image"].to(device), outputs["rgb"]
            metrics_dict["psnr"] = M.psnr(rgb.detach(), image)
        if "lidar" in batch:
            is_lidar = batch["is_lidar"][:, 0].to(device)
            n_lidar_rays = is_lidar.sum()
            did_return = batch["did_return"][batch["is_lidar"].squeeze(-1)].squeeze(-1).to(device)
            points_intensities = batch["lidar"][..., 3:4].to(device)
            termination_depth = batch["distance"].to(device)
            pred_depth = outputs["depth"][is_lidar]
            ray_drop_logits = outputs["ray_drop_logits"]
            pred_intensity = outputs["intensity"]

            metrics_dict["depth_median_l2"] = self.median_l2(pred_depth[did_return], termination_depth[did_return])
            metrics_dict["depth_mean_rel_l2"] = self.mean_rel_l2(pred_depth[did_return], termination_depth[did_return])
            metrics_dict["intensity_rmse"] = self.rmse(pred_intensity[did_return], points_intensities[did_return])
            metrics_dict["ray_drop_accuracy"] = ((ray_drop_logits.sigmoid() > 0.5).squeeze(-1) == ~did_return).float().mean()

            if self.training:
                rounds = len(cfg.sampling.num_proposal_samples)
                lidar = L.lidar_losses(pred_depth, [outputs[f"prop_depth_{i}"][is_lidar] for i in range(rounds)],
                                       termination_depth, did_return, pred_intensity, points_intensities, ray_drop_logits,
                                       cfg.non_return_lidar_distance, cfg.non_return_loss_mult, cfg.quantile_threshold)
                for k in ("depth_loss", "intensity_loss", "ray_drop_loss"):
                    metrics_dict[k] = lidar[k]
                metrics_dict["carving_loss"] = (outputs["non_nearby_weights"] ** 2).sum() / n_lidar_rays
                for i in range(rounds):
                    metrics_dict[f"depth_loss_{i}"] = lidar[f"depth_loss_{i}"]
                    metrics_dict[f"carving_loss_{i}"] = outputs[f"prop_weights_loss_{i}"] / n_lidar_rays

        if self.training and "weights_list" in outputs:
            metrics_dict["distortion"] = L.distortion_loss(outputs["weights_list"], outputs["ray_samples_list"])
        metrics_dict["sdf_to_density"] = float(self._param("field.sdf_to_density.beta").detach())  # NeuRAD's field is an SDF
        self.camera_optimizer.get_metrics_dict(metrics_dict)
        return metrics_dict

    def get_loss_dict(self, outputs: Dict[str, Tensor], batch: Dict[str, Tensor],
                      metrics_dict: Optional[Dict[str, Tensor]] = None) -> Dict[str, Tensor]:
        """neurad.py:531-561 with the reference's keys, multipliers and conditions.  An image batch with vgg_mult > 0
        needs `self.vgg_loss` (see __init__): without it this raises rather than return a loss dict without the
        perceptual term."""
        from . import losses as L

        cfg = self.config
        loss_dict: Dict[str, Tensor] = {}
        if "image" in batch:
            image, rgb = batch["image"].to(self.static_scale.device), outputs["rgb"]
            if cfg.vgg_mult > 0.0 and self.vgg_loss is None:
                raise RuntimeError("vgg_mult > 0 needs a perceptual loss: assign model.vgg_loss = a callable (rgb, image) -> "
                                   "loss (e.g. the reference's VGGPerceptualLossPix2Pix; no VGG weights ship with "
                                   "neurad_studio_b200) or set vgg_mult = 0")
            loss_dict["rgb_loss"] = torch.nn.functional.mse_loss(image, rgb) * cfg.rgb_mult
            if cfg.vgg_mult > 0.0:
                loss_dict["vgg_loss"] = self.vgg_loss(rgb, image) * cfg.vgg_mult
        if self.training:
            if "weights_list" in outputs:
                loss_dict["interlevel_loss"] = cfg.interlevel_loss_mult * L.zipnerf_interlevel_loss(outputs["weights_list"],
                                                                                                    outputs["ray_samples_list"])
                assert metrics_dict is not None and "distortion" in metrics_dict
                loss_dict["distortion_loss"] = cfg.distortion_loss_mult * metrics_dict["distortion"]
                prop_depth_mult = cfg.prop_lidar_loss_mult * cfg.depth_mult
                prop_carv_mult = cfg.prop_lidar_loss_mult * cfg.carving_mult
                for i in range(len(cfg.sampling.num_proposal_samples)):
                    loss_dict[f"depth_loss_{i}"] = prop_depth_mult * metrics_dict[f"depth_loss_{i}"]
                    loss_dict[f"carving_loss_{i}"] = prop_carv_mult * metrics_dict[f"carving_loss_{i}"]
            assert metrics_dict
            for k, mult in (("depth_loss", cfg.depth_mult), ("intensity_loss", cfg.intensity_mult),
                            ("carving_loss", cfg.carving_mult), ("ray_drop_loss", cfg.ray_drop_loss_mult)):
                if k in metrics_dict:
                    loss_dict[k] = mult * metrics_dict[k]
            self.camera_optimizer.get_loss_dict(loss_dict)
        return loss_dict

    @torch.no_grad()
    def get_image_metrics_and_images(self, outputs: Dict[str, Tensor], batch: Dict[str, Tensor]) -> Tuple[Dict[str, float], Dict[str, Tensor]]:
        """neurad.py:563-621 on the outputs / batch of an evaluation render.

        Lidar batches ("lidar"): depth median L2, depth mean relative L2, intensity RMSE, ray-drop accuracy and chamfer
        distance, with the reference's keys and values.  Like the reference it fills batch["is_lidar"] / batch["did_return"]
        when they are absent, and the chamfer distance is a 0-d tensor (the mean range of the measured returns) when there
        are no predicted or no measured returns, a float otherwise.

        Camera batches ("image", [H, W, 3] next to outputs["rgb"]): psnr, ssim and lpips as floats and images_dict["img"],
        the ground truth beside the render.  PSNR and SSIM come from one call of the library's kernels and one
        device-to-host copy; LPIPS is whatever callable the caller assigned to `self.lpips`.  Without one a camera batch
        raises before any work: LPIPS needs network weights the library does not ship, and a partial camera dict is never
        returned.  A batch with both keys returns both halves.

        Not provided: the colour-mapped entries of the reference's images_dict ("depth", and "accumulation" /
        "prop_depth_i" under config.verbose), which need matplotlib's colour tables."""
        if "image" in batch and self.lpips is None:
            raise NotImplementedError("camera metrics (PSNR / SSIM / LPIPS): the reference takes them from torchmetrics and LPIPS "
                                      "weights, which neurad_studio_b200 does not ship.  PSNR and SSIM run on the library's "
                                      "kernels, but LPIPS needs a callable: assign model.lpips = fn(image, rgb) -> value for "
                                      "[1, 3, H, W] tensors (e.g. torchmetrics' LearnedPerceptualImagePatchSimilarity"
                                      "(normalize=True)) to evaluate camera images")
        metrics_dict: Dict[str, float] = {}
        images_dict: Dict[str, Tensor] = {}
        if "image" in batch:
            image, rgb = batch["image"].to(self.static_scale.device), outputs["rgb"]
            images_dict["img"] = torch.cat([image, rgb], dim=1)
            # [H, W, C] -> [1, C, H, W] views, as the reference hands them to its metrics (neurad.py:581-582)
            image = torch.moveaxis(image, -1, 0)[None, ...]
            rgb = torch.moveaxis(rgb, -1, 0)[None, ...]
            # row 0 = {mse, psnr, ssim, data_range} of the batch: both floats in one device-to-host copy
            _, metrics_dict["psnr"], metrics_dict["ssim"], _ = get_backend(rgb.device).image_metrics(image, rgb)[0].tolist()
            metrics_dict["lpips"] = float(self.lpips(image, rgb))
        if "lidar" in batch:
            device = self.static_scale.device
            points = batch["lidar"].to(device)
            if "is_lidar" not in batch:
                batch["is_lidar"] = torch.ones(*batch["lidar"].shape[:-1], 1, dtype=torch.bool, device=device)
            if "did_return" not in batch:
                batch["did_return"] = torch.ones(*batch["lidar"].shape[:-1], 1, dtype=torch.bool, device=device)
            ray_drop_logits = outputs["ray_drop_logits"]
            pred_depth = outputs["depth"]
            did_return = batch["did_return"][:, 0].to(device)
            is_lidar = batch["is_lidar"][:, 0].to(device)
            # the reference's indexing: [is_lidar] then [did_return], which needs every ray of the batch to be a lidar ray
            metrics_dict["depth_median_l2"] = float(self.median_l2(pred_depth[is_lidar][did_return], batch["distance"][did_return]))
            metrics_dict["depth_mean_rel_l2"] = float(self.mean_rel_l2(pred_depth[is_lidar][did_return], batch["distance"][did_return]))
            metrics_dict["intensity_rmse"] = float(self.rmse(outputs["intensity"][did_return], points[did_return, 3:4]))
            metrics_dict["ray_drop_accuracy"] = float(((ray_drop_logits.sigmoid() > 0.5).squeeze(-1) == ~did_return).float().mean())
            if self.config.ray_drop_loss_mult > 0.0:
                pred_points_did_return = (ray_drop_logits.sigmoid() < 0.5).squeeze(-1)
            else:
                pred_points_did_return = (pred_depth < self.config.non_return_lidar_distance).squeeze(-1)
            if pred_points_did_return.any() and points.shape[0] > 0 and did_return.any():
                pred_points = outputs["points"][is_lidar][pred_points_did_return]
                metrics_dict["chamfer_distance"] = float(self.chamfer_distance(pred_points[..., :3], points[did_return, :3]))
            else:
                metrics_dict["chamfer_distance"] = points[did_return, :3].norm(dim=-1).mean()
        return metrics_dict, images_dict

    @torch.no_grad()
    def get_outputs_for_camera_ray_bundle(self, camera_ray_bundle: RayBundle) -> Dict[str, Tensor]:
        """neurad.py:623-675: in training mode or with use_camopt_in_eval the camera optimizer corrects the bundle first
        (:630-634), and the fused render takes the corrected rays; 2-D bundles are subsampled at [step//2::step] like the
        reference (`compensate_upsampling_when_rendering`), 1-D bundles are lidar rays."""
        if (self.training or self.use_camopt_in_eval) and self.camera_optimizer.config.mode != "off":
            shape = camera_ray_bundle.shape
            camera_ray_bundle = camera_ray_bundle.flatten()
            self.camera_optimizer.apply_to_raybundle(camera_ray_bundle)
            camera_ray_bundle = camera_ray_bundle._map(lambda t: t.reshape(*shape, t.shape[-1]))
        if len(camera_ray_bundle.shape) == 1:
            output_size = (camera_ray_bundle.shape[0],)
        else:
            assert len(camera_ray_bundle.shape) == 2, "Raybundle should be 2d (an image/patch)"
            step = self.config.rgb_upsample_factor
            camera_ray_bundle = camera_ray_bundle[step // 2 :: step, step // 2 :: step]
            output_size = camera_ray_bundle.shape
        be = self._bind()
        # an image is walked in 2-D tiles (a warp = an 8x4 pixel patch: coherent gathers); the output order is unchanged
        out = be.render(camera_ray_bundle.as_backend_dict(), want_intensity=True, image_width=output_size[1] if len(output_size) == 2 else 0)
        res = {k: v.view(*output_size, -1) for k, v in out.items()}
        res["ray_drop_prob"] = res["ray_drop_logits"].sigmoid()
        if len(output_size) == 2:  # camera: decode the feature image to rgb at `step` x the ray resolution
            ds = getattr(self, "decoder_stream", None)
            if ds is None:
                res["rgb"] = self.rgb_decoder(res["features"][None])[0]
            else:
                # opt-in pipelining (set_decoder_stream): this image's decoder runs on `ds` while the caller's stream goes on
                # to the next image's render -- the sampling kernel (CUDA cores, issue-bound) and the convolutions (tensor
                # pipe) use different parts of an SM.  `rgb` is ready when res["rgb_ready"] (a CUDA event) has completed.
                feats = res["features"]
                ev = torch.cuda.Event()
                ev.record()
                with torch.cuda.stream(ds):
                    ds.wait_event(ev)
                    res["rgb"] = self.rgb_decoder(feats[None])[0]
                    feats.record_stream(ds)
                    done = torch.cuda.Event()
                    done.record(ds)
                res["rgb_ready"] = done
        return res

    @torch.no_grad()
    def get_outputs_for_lidar_sweep(self, sensors, poses: Tensor, times, velocities: Optional[Tensor] = None,
                                    ray_drop_threshold: Optional[float] = 0.5, max_distance: Optional[float] = None,
                                    camera_indices=None) -> Dict[str, Tensor]:
        """What a lidar would see from new poses: S simulated sweeps of scene.LidarSensor descriptors, the viewer's lidar
        render (viewer/render_state_machine.py:391-430) generalised to beam tables, per-beam azimuth offsets, a rolling
        shutter and several sweeps per call.

        `sensors`: one LidarSensor or one per sweep, all with one beam count and azimuth resolution; poses [S,3,4]
        sensor-to-world at the scan times; times [S]; velocities [S,3] or None.  The rays render as one 1-D lidar bundle
        through `get_outputs_for_camera_ray_bundle`, in eval mode (the model's mode is restored afterwards), so actor
        edits and, with use_camopt_in_eval, the camera optimizer act as on any render; `camera_indices` [S] names the
        optimizer row of each sweep and is required when the optimizer applies.

        A ray returns when ray_drop_prob < ray_drop_threshold if the threshold is not None and the model has a ray-drop
        head (ray_drop_loss_mult > 0), else when depth < max_distance (None: non_return_lidar_distance); with the
        defaults this is the rule of get_image_metrics_and_images (neurad.py:610-613).

        Returns the render outputs over all N = S x beams x columns rays ([N,1] each), plus
          depth_image / intensity_image / ray_drop_prob_image: [S, beams, columns] views of those outputs;
          points [M,5]: the kept rays' origin + direction * depth in the frame of their sweep's nominal pose
            (pose_inverse, models/ad_model.py:107-113) with intensity and the time offset from the scan time, the
            layout of a measured scan (x, y, z, intensity, dt) -- `points[:, :3]` goes straight into chamfer_distance;
          points_world [M,3]; point_index [M,3] int32 (sweep, beam, column), in that row-major order;
          counts [S] and offsets [S] (int32, device): kept points per sweep and each sweep's first row.
        The points are those of the generated rays, before any camera-optimizer correction, as in get_outputs_for_lidar.
        Reading the kept count to size `points` is the call's one host synchronisation, given host (CPU) poses, times,
        velocities, tables and camera_indices.  Each sensor_idx must lie in [0, config.num_sensors)."""
        be = get_backend(self.static_scale.device)
        for s_ in (sensors if isinstance(sensors, (list, tuple)) else [sensors]):
            # the render indexes the appearance embedding with it unchecked
            if not 0 <= int(s_.sensor_idx) < self.config.num_sensors:
                raise ValueError(f"sensor_idx {s_.sensor_idx} is outside [0, {self.config.num_sensors}) (config.num_sensors)")
        r = be.raygen_lidar_sweeps(sensors, poses, times, velocities)
        n_sw, beams, n_az = r["shape"]
        cam_idx = None
        if camera_indices is not None:
            ci = torch.as_tensor(camera_indices, dtype=torch.long).cpu().reshape(-1)
            if ci.numel() != n_sw:
                raise ValueError(f"camera_indices needs one entry per sweep ({n_sw}), got {ci.numel()}")
            ci = ci.pin_memory().to(be.device, non_blocking=True)
            cam_idx = ci[:, None].expand(n_sw, beams * n_az).reshape(-1, 1)
        elif self.use_camopt_in_eval and self.camera_optimizer.config.mode != "off":
            raise ValueError("the camera optimizer applies in eval (use_camopt_in_eval): pass camera_indices, one per sweep")
        bundle = RayBundle(origins=r["origins"], directions=r["directions"], pixel_area=r["pixel_area"], times=r["times"],
                           camera_indices=cam_idx, metadata={"is_lidar": r["is_lidar"], "sensor_idxs": r["sensor_idx"]})
        was_training = self.training
        self.eval()
        try:
            out = self.get_outputs_for_camera_ray_bundle(bundle)
        finally:
            self.train(was_training)
        use_ray_drop = ray_drop_threshold is not None and self.config.ray_drop_loss_mult > 0.0
        if use_ray_drop:
            thr = float(ray_drop_threshold)
        else:
            thr = float(self.config.non_return_lidar_distance if max_distance is None else max_distance)
        pts = be.lidar_sweep_points(r, out["depth"], out["intensity"], out["ray_drop_prob"] if use_ray_drop else None, thr)
        m = int(pts["counts"][-1])
        for k in ("depth", "intensity", "ray_drop_prob"):
            out[f"{k}_image"] = out[k].view(n_sw, beams, n_az)
        out["points"], out["points_world"], out["point_index"] = pts["points_sensor"][:m], pts["points_world"][:m], pts["index"][:m]
        out["counts"], out["offsets"] = pts["counts"][:n_sw], pts["offsets"]
        return out

    def set_decoder_stream(self, stream: Optional["torch.cuda.Stream"]) -> None:
        """Run the rgb decoder of `get_outputs_for_camera_ray_bundle` on a side stream (None: on the caller's stream, the
        default and the reference's behaviour).  With a stream, outputs["rgb"] must not be consumed before
        outputs["rgb_ready"] has completed (`stream.wait_event(outputs["rgb_ready"])` or `.synchronize()`)."""
        self.decoder_stream = stream
