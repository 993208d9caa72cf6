"""Host side of the sm_90a NeuRAD backend: owns a `b200nerf_ctx`, feeds it torch CUDA tensors by pointer and
launches the kernels on torch's current stream.  PyTorch is plumbing here (device memory, streams); all compute
is in libb200nerf.so.  There is no CPU path: constructing a `B200Backend` without a CUDA device raises.
"""
from __future__ import annotations

import ctypes
import math
import os
from typing import Dict, Optional, Sequence, Tuple

import torch

from . import lib as _lib
from . import tcnn_compat
from .config import HashGridSettings, NeuRADConfig
from .lib import ConvBnParams, ConvParams, RgbDecoderParams, FIELD_MAIN, FIELD_PROP0, FIELD_PROP1, GridDesc, Outputs, PeerOutputs, Rays, Trace, TRACE_FIELDS


def pdf_quantiles(num_samples: int) -> torch.Tensor:
    """PDFSampler's eval-mode `u` (ray_samplers.py:332-336), evaluated with torch.linspace exactly like the
    reference so the searchsorted inputs are bit-identical."""
    num_bins = num_samples + 1
    u = torch.linspace(0.0, 1.0 - (1.0 / num_bins), steps=num_bins)
    return u + 1.0 / (2 * num_bins)


NO_ACTOR_EDIT = (0.0, 0.0, 0.0, 0.0, -1.0)  # (lateral, longitudinal, height, rotation, index): DynamicActors' defaults
_lib_INVALID = -1  # B200NERF_ERR_INVALID


def _ptr(t: Optional[torch.Tensor]):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def is_pinhole_camera(cam) -> bool:
    """True for an undistorted PERSPECTIVE camera with a top-to-bottom shutter: the model of `raygen_pinhole`."""
    dist = getattr(cam, "distortion_params", None)
    return (getattr(cam, "camera_type", "perspective") == "perspective" and getattr(cam, "rs_direction", "Vertical") == "Vertical"
            and (dist is None or not bool((torch.as_tensor(dist) != 0).any())))


def camera_descriptor(cam) -> "_lib.Camera":
    """b200nerf_camera of a scene.PinholeCamera; ValueError for an unknown camera_type or rs_direction, or a distortion
    vector that does not have 6 entries (k1, k2, k3, k4, p1, p2)."""
    # a camera object without the model fields (written before they existed) is the undistorted perspective default
    camera_type = getattr(cam, "camera_type", "perspective")
    rs_direction = getattr(cam, "rs_direction", "Vertical")
    distortion = getattr(cam, "distortion_params", None)
    if camera_type not in _lib.CAMERA_TYPES:
        raise ValueError(f"camera_type {camera_type!r}: expected one of {sorted(_lib.CAMERA_TYPES)}")
    if rs_direction not in _lib.RS_DIRECTIONS:
        raise ValueError(f"rs_direction {rs_direction!r}: expected one of {sorted(_lib.RS_DIRECTIONS)}")
    dist = [0.0] * 6
    if distortion is not None:
        dist = torch.as_tensor(distortion, dtype=torch.float32).reshape(-1).tolist()
        if len(dist) != 6:
            raise ValueError(f"distortion_params must hold 6 values (k1, k2, k3, k4, p1, p2), got {len(dist)}")
    d = _lib.Camera()
    d.c2w[:] = torch.as_tensor(cam.c2w, dtype=torch.float32).reshape(-1).tolist()
    d.fx, d.fy, d.cx, d.cy = cam.fx, cam.fy, cam.cx, cam.cy
    d.width, d.height = cam.width, cam.height
    d.camera_type = _lib.CAMERA_TYPES[camera_type]
    d.distortion[:] = dist
    d.time = cam.time
    if cam.velocity is not None:
        d.velocity[:] = torch.as_tensor(cam.velocity, dtype=torch.float32).reshape(-1).tolist()
        d.has_velocity = 1
    d.rolling_shutter_time, d.time_to_center_pixel = cam.rolling_shutter_time, cam.time_to_center_pixel
    d.rs_direction = _lib.RS_DIRECTIONS[rs_direction]
    return d


def lidar_columns(azim_res_deg: float) -> Tuple[float, int]:
    """(step in radians, column count) of the viewer's `torch.arange(0, 2 pi, np.deg2rad(azim_res_deg))`."""
    import numpy as np

    step = float(np.deg2rad(azim_res_deg))
    if not (math.isfinite(step) and step > 0.0):
        raise ValueError(f"azimuth resolution must be finite and positive, got {azim_res_deg}")
    return step, int(math.ceil((2 * math.pi) / step))  # len(torch.arange(0, 2*pi, step))


def grid_desc(g: HashGridSettings, scalings: Optional[torch.Tensor] = None) -> GridDesc:
    d = GridDesc()
    d.num_levels, d.features_per_level, d.log2_hashmap_size = g.num_levels, g.hashgrid_dim, g.log2_hashmap_size
    sc = (scalings if scalings is not None else g.scalings()).detach().cpu().float().tolist()
    if len(sc) != g.num_levels:
        raise ValueError("scalings buffer does not match num_levels")
    for i, v in enumerate(sc):
        d.scalings[i] = v
    return d


DEFAULT_MODE = "split"


class B200Backend:
    """One context per CUDA device.  `load_params` takes tensors under the reference's state_dict names."""

    def __init__(self, device: Optional[torch.device] = None):
        if not torch.cuda.is_available():
            raise RuntimeError("neurad_studio_b200 requires a CUDA (sm_90a) device; there is no CPU fallback")
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError("neurad_studio_b200 runs on CUDA devices only")
        self.lib = _lib.load()
        h = ctypes.c_void_p()
        _lib.check(self.lib, self.lib.b200nerf_create(self.device.index or 0, ctypes.byref(h)))
        self._h = h
        self._keep: Dict[str, object] = {}  # tensors the library references zero-copy
        self.cfg: Optional[NeuRADConfig] = None
        # Who bound the context last: (model uid, parameter versions).  The backend is a per-device singleton shared by every
        # model in the process, so a model must re-bind whenever ANOTHER model (or a direct load_params call) came in between.
        self._owner = None
        self._dec_owner = None

    # the actor edit the context holds (b200nerf_set_actors clears it), and whether it changes any actor's pose
    _actor_edit = NO_ACTOR_EDIT
    actor_edit_active = False

    def close(self):
        if getattr(self, "_h", None) is not None and self._h.value:
            self.lib.b200nerf_destroy(self._h)
            self._h = ctypes.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ------------------------------------------------------------------------------------------ helpers
    def _dev(self, t: torch.Tensor, dtype=torch.float32) -> torch.Tensor:
        if t.device != self.device or t.dtype != dtype or not t.is_contiguous():
            t = t.detach().to(device=self.device, dtype=dtype).contiguous()
        return t

    def _ray_times(self, times: Optional[torch.Tensor], n: int) -> Optional[torch.Tensor]:
        """Per-ray times [N] from [N], [N,1] or the reference's expanded [N,S,1] (it reads times[:, 0], neurad_encoding.py:194)."""
        if times is None:
            return None
        return self._dev(times.reshape(n, -1)[:, 0] if times.numel() != n else times.reshape(n))

    def _check(self, rc: int):
        _lib.check(self.lib, rc)

    @property
    def _stream(self):
        return ctypes.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    # --------------------------------------------------------------------------------------- parameters
    def load_params(self, cfg: NeuRADConfig, params: Dict[str, torch.Tensor], density_field_of_round: Sequence[int] = (FIELD_PROP1, FIELD_PROP1)):
        """Bind a full parameter set.  `density_field_of_round` defaults to the reference's effective behaviour:
        both proposal rounds evaluate proposal_fields[1] (late-binding closures at models/neurad.py:248)."""
        self.cfg = cfg
        self._owner = None  # a model that binds through NeuRADModel._bind() records itself after this call
        # packing kernels / copies of the set_* calls go on torch's current stream: ordered after the optimizer step that
        # wrote the parameters and before the renders that read the packed copies (no device-wide synchronisation)
        self._check(self.lib.b200nerf_set_param_stream(self._h, self._stream))
        p = params
        n_act = cfg.n_actors
        # dynamic_actors.actor_to_id (dynamic_actors.py:161, read at neurad_encoding.py:181): actor index -> hash-grid index;
        # identity unless a closed-loop server re-assigned it (scripts/closed_loop/server.py:143)
        a2i = p.get("dynamic_actors.actor_to_id")
        grid_of_actor = list(range(n_act)) if a2i is None else [int(v) for v in a2i.detach().cpu().reshape(-1).tolist()]
        if n_act > 0 and (len(grid_of_actor) != n_act or min(grid_of_actor) < 0 or max(grid_of_actor) >= n_act):
            raise ValueError("dynamic_actors.actor_to_id must hold one grid index in [0, n_actors) per actor")
        self.actor_grids_remapped = grid_of_actor != list(range(n_act))
        prefixes = {FIELD_MAIN: "field", FIELD_PROP0: "proposal_fields.0", FIELD_PROP1: "proposal_fields.1"}
        gcfgs = {FIELD_MAIN: cfg.grid, FIELD_PROP0: cfg.proposal_grid_1, FIELD_PROP1: cfg.proposal_grid_2}
        static_scale = float(p["static_scale"]) if "static_scale" in p else float(cfg.static_scale)
        # a tcnn-trained checkpoint (implementation="tcnn", the reference's default): flat `tcnn_encoding.params` vectors in
        # tiny-cuda-nn's layout instead of the torch twins' tensors (tcnn_compat.py; SURVEY 8f row f3)
        tcnn = tcnn_compat.is_tcnn_state(p)
        self.layout = "tcnn" if tcnn else "torch"
        if tcnn and self.actor_grids_remapped:
            raise NotImplementedError("dynamic_actors.actor_to_id re-assignment is not supported with the tiny-cuda-nn layout")
        sizes = tcnn_compat.n_grid_params(cfg) if tcnn else {}
        for f, pre in prefixes.items():
            g = gcfgs[f]
            if f != FIELD_MAIN:
                w = self._dev(p[f"{pre}.density_decoder.weight"]).reshape(-1)
                self._check(self.lib.b200nerf_set_proposal_decoder(self._h, f, _ptr(w), w.numel()))
            if tcnn:
                def flat(key):
                    t = p[key].reshape(-1)
                    if t.numel() != sizes[key]:
                        raise ValueError(f"{key} has {t.numel()} parameters, the configured grid needs {sizes[key]}")
                    return self._dev(tcnn_compat.half_round(t))

                tab = flat(f"{pre}.hashgrid.static_grid.{tcnn_compat.TCNN_SUFFIX}")
                self._keep[f"{pre}.static"] = tab
                sc = p.get(f"{pre}.hashgrid.static_grid.scalings")
                sd = tcnn_compat.grid_desc(tcnn_compat.layout_of(g.static, 3), sc if sc is not None else g.static.scalings())
                ad = atab = None
                if n_act > 0:
                    atab = flat(f"{pre}.hashgrid.actor_grids.0.{tcnn_compat.TCNN_SUFFIX}")
                    self._keep[f"{pre}.actors"] = atab
                    sc = p.get(f"{pre}.hashgrid.actor_grids.0.scalings")
                    ad = tcnn_compat.grid_desc(tcnn_compat.layout_of(g.actor, 4), sc if sc is not None else g.actor.scalings())
                self._check(self.lib.b200nerf_set_field_grids_tcnn(
                    self._h, f, ctypes.byref(sd), _ptr(tab), ctypes.byref(ad) if ad is not None else None, _ptr(atab), n_act,
                    static_scale, float(g.actor_scale)))
                continue
            tab = self._dev(p[f"{pre}.hashgrid.static_grid.hash_table"])
            self._keep[f"{pre}.static"] = tab
            sd = grid_desc(g.static, p.get(f"{pre}.hashgrid.static_grid.scalings"))
            ad, arr = None, None
            if n_act > 0:
                tabs = [self._dev(p[f"{pre}.hashgrid.actor_grids.{grid_of_actor[a]}.hash_table"]) for a in range(n_act)]
                self._keep[f"{pre}.actors"] = tabs
                arr = (ctypes.c_void_p * n_act)(*[t.data_ptr() for t in tabs])
                ad = grid_desc(g.actor, p.get(f"{pre}.hashgrid.actor_grids.0.scalings"))
            self._check(
                self.lib.b200nerf_set_field_grids(
                    self._h, f, ctypes.byref(sd), _ptr(tab), ctypes.byref(ad) if ad is not None else None,
                    arr, n_act, static_scale, float(g.actor_scale),
                )
            )
        if tcnn and f"field.mlp_geo.{tcnn_compat.TCNN_SUFFIX}" in p:
            # FullyFusedMLP: bias-free, widths padded to 16 (field_components/mlp.py:116-140) -> nn.Linear shapes, zero biases
            hid, nff = cfg.geo_hidden_dim, cfg.nff_out_dim
            ts = (tcnn_compat.mlp_tensors(p, "field.mlp_geo", cfg.grid.static.out_dim, hid, 2, nff + 1, self.device)
                  + tcnn_compat.mlp_tensors(p, "field.mlp_feature", nff + 16, cfg.nff_hidden_dim, 3, nff, self.device))
        else:
            names = ["field.mlp_geo.layers.0", "field.mlp_geo.layers.1", "field.mlp_feature.layers.0",
                     "field.mlp_feature.layers.1", "field.mlp_feature.layers.2"]
            ts = []
            for nme in names:
                ts += [self._dev(p[nme + ".weight"]), self._dev(p[nme + ".bias"])]
        beta = float(p["field.sdf_to_density.beta"].abs().item() + 0.0001)  # model_components/utils.py:38-41
        self._check(self.lib.b200nerf_set_main_mlps(self._h, *[_ptr(t) for t in ts], beta))
        # the module-level NeuRADField.forward runs the same MLPs through b200nerf_mlp_fwd
        self._field_mlps = {"geo": (ts[0:4:2], ts[1:4:2]), "feature": (ts[4::2], ts[5::2])}
        self._beta = beta
        if tcnn and f"lidar_decoder.{tcnn_compat.TCNN_SUFFIX}" in p:
            ts = tcnn_compat.mlp_tensors(p, "lidar_decoder", cfg.feature_dim, 32, 3, 2, self.device)
            self._check(self.lib.b200nerf_set_lidar_decoder(self._h, *[_ptr(t) for t in ts]))
        elif "lidar_decoder.layers.0.weight" in p:
            ts = []
            for i in range(3):
                ts += [self._dev(p[f"lidar_decoder.layers.{i}.weight"]), self._dev(p[f"lidar_decoder.layers.{i}.bias"])]
            self._check(self.lib.b200nerf_set_lidar_decoder(self._h, *[_ptr(t) for t in ts]))
        emb = self._dev(p["appearance_embedding.weight"])
        self._keep["appearance"] = emb
        if cfg.use_temporal_appearance:
            self._check(self.lib.b200nerf_set_appearance(self._h, _ptr(emb), emb.shape[0], emb.shape[1], cfg.embeds_per_sensor,
                                                         float(cfg.duration)))
        else:
            self._check(self.lib.b200nerf_set_appearance_per_sensor(self._h, _ptr(emb), emb.shape[0], emb.shape[1]))
        if n_act > 0:
            ts_ = self._dev(p["dynamic_actors.unique_timestamps"])
            rot = self._dev(p["dynamic_actors.actor_rotations_6d"])
            pos = self._dev(p["dynamic_actors.actor_positions"])
            pres = self._dev(p["dynamic_actors.actor_present_at_time"], torch.uint8)
            sizes = self._dev(p["dynamic_actors.actor_sizes"])
            pad = p.get("dynamic_actors.actor_padding")
            pad = list(cfg.actor_bbox_padding) if pad is None else pad.detach().cpu().tolist()
            cpad = (ctypes.c_float * 3)(*pad)
            self._check(
                self.lib.b200nerf_set_actors(self._h, n_act, ts_.shape[0], _ptr(ts_), _ptr(rot), _ptr(pos), _ptr(pres), _ptr(sizes), cpad)
            )
        else:
            self._check(self.lib.b200nerf_set_actors(self._h, 0, 0, None, None, None, None, None, None))
        self._actor_edit, self.actor_edit_active = NO_ACTOR_EDIT, False
        sp = cfg.sampling
        u1, u2 = pdf_quantiles(sp.num_proposal_samples[1]), pdf_quantiles(sp.num_nerf_samples)
        cu1 = (ctypes.c_float * u1.numel())(*u1.tolist())
        cu2 = (ctypes.c_float * u2.numel())(*u2.tolist())
        rounds = (ctypes.c_int * 2)(*density_field_of_round)
        self._check(
            self.lib.b200nerf_set_sampling(
                self._h, sp.num_proposal_samples[0], sp.num_proposal_samples[1], sp.num_nerf_samples,
                sp.power_lambda, sp.power_scaling, sp.sky_distance, sp.histogram_padding, cu1, cu2, rounds,
                float(cfg.rgb_upsample_factor**2),
            )
        )

    def set_actor_edit(self, lateral: float = 0.0, longitudinal: float = 0.0, height: float = 0.0, rotation: float = 0.0,
                       index: float = -1.0) -> None:
        """DynamicActors.actor_editing (dynamic_actors.py:53-59, 181-249) for the following renders and module-level
        encoding forwards, with the reference's semantics (include/b200nerf.h: b200nerf_set_actor_edit).  All zeros clears
        it; load_params clears it too.  Only a change reaches the library.  Raises ValueError for an index that selects no
        actor (below -n_actors), as the reference's indexing does."""
        edit = tuple(float(v) for v in (lateral, longitudinal, height, rotation, index))
        if edit == self._actor_edit:
            return
        rc = self.lib.b200nerf_set_actor_edit(self._h, *edit)
        if rc == _lib_INVALID:  # the library has cleared the edit
            self._actor_edit, self.actor_edit_active = NO_ACTOR_EDIT, False
            raise ValueError(f"actor edit: {self.lib.b200nerf_last_error().decode()}")
        self._check(rc)
        self._actor_edit = edit
        n_act = self.cfg.n_actors if self.cfg is not None else 0
        self.actor_edit_active = n_act > 0 and any(v != 0.0 for v in (edit[0], edit[1], edit[3]))

    # ------------------------------------------------------------------------------------------ fused path
    def render(self, rays: Dict[str, torch.Tensor], want_trace: bool = False, want_intensity: bool = False,
               out: Optional[Dict[str, torch.Tensor]] = None, image_width: int = 0) -> Dict[str, torch.Tensor]:
        """NeuRADModel.get_nff_outputs (models/neurad.py:368-421) for a flat ray batch.

        rays: origins [N,3], directions [N,3], pixel_area [N,1]|[N], times [N,1]|[N] and optionally nears, fars,
        sensor_idx (int64), is_lidar (bool/uint8).  Returns features [N,48], depth/accumulation/prop_depth_i [N,1].
        `out` may supply pre-allocated output tensors (e.g. a slice of an all-gather buffer).  `image_width` > 0
        declares the bundle a row-major image (stack) of that width so that the kernel can walk it in 2-D tiles
        (better gather coherence); it does not change the output order.

        `want_trace`: True records every per-sample trace field (TRACE_FIELDS) next to the outputs; a collection of
        trace names records only those.  Tracing actor ids turns off the proposal rounds' early exit, so a trace
        without them is how the production path itself is observed."""
        cfg = self.cfg
        if cfg is None:
            raise RuntimeError("load_params() must be called before render()")
        o = self._dev(rays["origins"])
        n = o.shape[0]
        r = Rays()
        r.image_width = int(image_width)
        hold = [o]

        def put(name, key, dtype=torch.float32, required=False):
            t = rays.get(key)
            if t is None:
                if required:
                    raise KeyError(key)
                setattr(r, name, None)
                return
            t = self._dev(t.reshape(n, 3) if name in ("origins", "directions") else t.reshape(-1), dtype)
            hold.append(t)
            setattr(r, name, t.data_ptr())

        r.origins = o.data_ptr()
        put("directions", "directions", required=True)
        put("pixel_area", "pixel_area", required=True)
        put("times", "times", required=True)
        put("nears", "nears")
        put("fars", "fars")
        put("sensor_idx", "sensor_idx", torch.int64)
        put("is_lidar", "is_lidar", torch.uint8)
        fdim = cfg.feature_dim
        res = out if out is not None else {}
        shapes = {"features": (n, fdim), "depth": (n, 1), "accumulation": (n, 1), "prop_depth_0": (n, 1), "prop_depth_1": (n, 1)}
        if want_intensity:
            shapes.update({"intensity": (n, 1), "ray_drop_logits": (n, 1)})
        for k, shp in shapes.items():
            if k not in res:
                res[k] = torch.empty(shp, device=self.device, dtype=torch.float32)
            elif not (res[k].is_contiguous() and res[k].device == self.device and res[k].dtype == torch.float32 and res[k].numel() == shp[0] * shp[1]):
                raise ValueError(f"pre-allocated output {k} has the wrong layout")
        oo = Outputs()
        for k in ("features", "depth", "accumulation", "prop_depth_0", "prop_depth_1"):
            setattr(oo, k, res[k].data_ptr())
        oo.intensity = res["intensity"].data_ptr() if want_intensity else None
        oo.ray_drop_logit = res["ray_drop_logits"].data_ptr() if want_intensity else None
        tr = None
        if isinstance(want_trace, (bool, int)) or getattr(want_trace, "dtype", None) == bool:  # incl. numpy / torch bools
            traced = set(TRACE_FIELDS) if want_trace else set()
        else:
            traced = set(want_trace)
            unknown = traced - set(TRACE_FIELDS)
            if unknown:
                raise ValueError(f"unknown trace fields {sorted(unknown)}; known: {list(TRACE_FIELDS)}")
        if traced:
            S0, S1 = cfg.sampling.num_proposal_samples
            S2 = cfg.sampling.num_nerf_samples
            f32, i32 = torch.float32, torch.int32
            tshapes = {
                "prop_weights_0": ((n, S0), f32), "prop_weights_1": ((n, S1), f32),
                "bins_s_1": ((n, S1 + 1), f32), "bins_e_1": ((n, S1 + 1), f32),
                "bins_s_2": ((n, S2 + 1), f32), "bins_e_2": ((n, S2 + 1), f32),
                "inds_1": ((n, S1 + 1), i32), "inds_2": ((n, S2 + 1), i32),
                "sdf": ((n, S2), f32), "alpha": ((n, S2), f32), "field_feature": ((n, S2, cfg.nff_out_dim), f32),
                "weights": ((n, S2), f32),
                "actor_id_0": ((n, S0), i32), "actor_id_1": ((n, S1), i32), "actor_id_main": ((n, S2), i32),
            }
            tr = Trace()
            for k in TRACE_FIELDS:
                if k not in traced:
                    setattr(tr, k, None)
                    continue
                shp, dt = tshapes[k]
                res[k] = torch.empty(shp, device=self.device, dtype=dt)
                setattr(tr, k, res[k].data_ptr())
        self._check(
            self.lib.b200nerf_nff_render_fwd(self._h, ctypes.byref(r), n, ctypes.byref(oo), ctypes.byref(tr) if tr is not None else None, self._stream)
        )
        return res

    # --------------------------------------------------------------------------------------- stage operators
    def hashgrid_fwd(self, g: HashGridSettings, table: torch.Tensor, x: torch.Tensor, scalings: Optional[torch.Tensor] = None, want_indices: bool = False):
        """HashEncoding.forward (encodings.py:425-471): x [...,3] -> [..., L*F] (+ hashed rows [..., L, 8])."""
        d = grid_desc(g, scalings)
        table = self._dev(table)
        xs = self._dev(x).reshape(-1, 3)
        n = xs.shape[0]
        if n == 0:
            out = torch.empty(*x.shape[:-1], g.num_levels * g.hashgrid_dim, device=self.device)
            return (out, torch.empty(*x.shape[:-1], g.num_levels, 8, device=self.device, dtype=torch.int32)) if want_indices else out
        out = torch.empty(n, g.num_levels * g.hashgrid_dim, device=self.device)
        idx = torch.empty(n, g.num_levels, 8, device=self.device, dtype=torch.int32) if want_indices else None
        self._check(self.lib.b200nerf_hashgrid_fwd(self._h, ctypes.byref(d), _ptr(table), _ptr(xs), _ptr(out), _ptr(idx), n, self._stream))
        out = out.reshape(*x.shape[:-1], -1)
        return (out, idx.reshape(*x.shape[:-1], g.num_levels, 8)) if want_indices else out

    def tcnn_hashgrid_fwd(self, layout: Dict[str, list], params: torch.Tensor, x: torch.Tensor, scalings: Optional[torch.Tensor] = None) -> torch.Tensor:
        """tcnn.Encoding{HashGrid}.forward for a tiny-cuda-nn layout (tcnn_compat.grid_layout): flat params (values already
        fp16-rounded), x [P, n_dims] in [0,1] -> [P, L*F] level-major.  Parity unpinned (tcnn_compat.py)."""
        sc = scalings if scalings is not None else torch.ones(layout["n_levels"])
        d = tcnn_compat.grid_desc(layout, sc)
        pr, xs = self._dev(params).reshape(-1), self._dev(x).reshape(-1, layout["n_dims"])
        out = torch.empty(xs.shape[0], layout["n_levels"] * layout["n_features"], device=self.device)
        self._check(self.lib.b200nerf_tcnn_hashgrid_fwd(self._h, ctypes.byref(d), _ptr(pr), _ptr(xs), _ptr(out), xs.shape[0], self._stream))
        return out

    def sh4_fwd(self, dirs: torch.Tensor) -> torch.Tensor:
        """SHEncoding(levels=4).forward (encodings.py:797-805)."""
        d = self._dev(dirs).reshape(-1, 3)
        out = torch.empty(d.shape[0], 16, device=self.device)
        self._check(self.lib.b200nerf_sh4_fwd(self._h, _ptr(d), _ptr(out), d.shape[0], self._stream))
        return out.reshape(*dirs.shape[:-1], 16)

    def mlp_fwd(self, x: torch.Tensor, weights: Sequence[torch.Tensor], biases: Optional[Sequence[Optional[torch.Tensor]]] = None,
                want_hidden: bool = False):
        """MLP.forward (field_components/mlp.py:142-183) on the wgmma tensor cores (3xTF32): ReLU hidden
        activations, no output activation.  weights[i] is nn.Linear's [out_i, in_i].  `want_hidden` (training): returns
        (y, [pre-activation of hidden layer l, [n_rows, out_l]]) -- what the backward needs, stored by the same launch."""
        xs = self._dev(x).reshape(-1, x.shape[-1])
        ws = [self._dev(w) for w in weights]
        bs = [None if (biases is None or b is None) else self._dev(b) for b in (biases if biases is not None else [None] * len(ws))]
        n, nl = xs.shape[0], len(ws)
        out_dims = [w.shape[0] for w in ws]
        y = torch.empty(n, out_dims[-1], device=self.device)
        cw = (ctypes.c_void_p * nl)(*[w.data_ptr() for w in ws])
        cb = (ctypes.c_void_p * nl)(*[(b.data_ptr() if b is not None else None) for b in bs])
        co = (ctypes.c_int * nl)(*out_dims)
        if want_hidden:
            zs = [torch.empty(n, d, device=self.device) for d in out_dims[:-1]]
            ch = (ctypes.c_void_p * max(nl - 1, 1))(*[z.data_ptr() for z in zs])
            self._check(self.lib.b200nerf_mlp_fwd_train(self._h, _ptr(xs), n, xs.shape[1], nl, cw, cb, co, _ptr(y), ch, self._stream))
            return y.reshape(*x.shape[:-1], out_dims[-1]), zs
        self._check(self.lib.b200nerf_mlp_fwd(self._h, _ptr(xs), n, xs.shape[1], nl, cw, cb, co, _ptr(y), self._stream))
        return y.reshape(*x.shape[:-1], out_dims[-1])

    def set_mlp_mode(self, mode: str):
        """Kernel variant of render(): 'split' (default) ray-per-lane in two kernels -- sampling at 32 warps/SM, then
        shading with wgmma MLPs (fp16 three-term split); 'lane' the same code as one fused kernel; 'tc' warp-per-ray +
        wgmma MLPs (3xTF32); 'ffma' warp-per-ray + CUDA-core fp32 MLPs."""
        self._check(self.lib.b200nerf_set_mlp_mode(self._h, {"ffma": 0, "tc": 1, "lane": 2, "split": 3}[mode]))

    def set_peer_outputs(self, peer_ptrs: Optional[Dict[str, Sequence[int]]], self_rank: int = -1, row_offset: int = 0):
        """Fuse the multi-GPU gather into the render epilogue: `peer_ptrs` maps "features" / "depth" / "accumulation"
        to one device pointer per rank (peer-mapped, e.g. symmetric-memory `buffer_ptrs`); every rendered row is also
        stored at `row_offset + ray` of each peer's buffer.  None clears it."""
        if peer_ptrs is None:
            self._check(self.lib.b200nerf_set_peer_outputs(self._h, None))
            return
        po = PeerOutputs()
        n = len(peer_ptrs["features"])
        po.n_peers, po.self_rank, po.row_offset = n, self_rank, row_offset
        for i in range(n):
            po.features[i], po.depth[i], po.accumulation[i] = peer_ptrs["features"][i], peer_ptrs["depth"][i], peer_ptrs["accumulation"][i]
        self._check(self.lib.b200nerf_set_peer_outputs(self._h, ctypes.byref(po)))

    def check_status(self):
        """Raise if a kernel set the device-side failure flag (synchronises)."""
        self._check(self.lib.b200nerf_check_status(self._h))

    def pdf_resample(self, weights: torch.Tensor, bins: torch.Tensor, num_samples: int, histogram_padding: float = 0.01):
        """PDFSampler (eval, include_original=False): weights [N,S], spacing bins [N,S+1] ->
        (new bins [N,S_new+1], cdf [N,S+1], searchsorted indices [N,S_new+1] int32)."""
        w, b = self._dev(weights), self._dev(bins)
        n, s = w.shape
        u = pdf_quantiles(num_samples).to(self.device)
        nb = torch.empty(n, num_samples + 1, device=self.device)
        cdf = torch.empty(n, s + 1, device=self.device)
        inds = torch.empty(n, num_samples + 1, device=self.device, dtype=torch.int32)
        self._check(self.lib.b200nerf_pdf_resample(self._h, _ptr(w), _ptr(b), _ptr(u), n, s, num_samples, histogram_padding, _ptr(nb), _ptr(cdf), _ptr(inds), self._stream))
        return nb, cdf, inds

    def pdf_resample_stratified(self, weights: torch.Tensor, bins: torch.Tensor, num_samples: int, rand: torch.Tensor,
                                histogram_padding: float = 0.01):
        """PDFSampler in training mode (train_stratified, ray_samplers.py:321-329): `rand` [N,1] (single_jitter) or
        [N,S_new+1] uniform numbers drawn by the caller; returns like pdf_resample."""
        w, b, r = self._dev(weights), self._dev(bins), self._dev(rand)
        n, s = w.shape
        nb = num_samples + 1
        u = torch.linspace(0.0, 1.0 - (1.0 / nb), steps=nb).to(self.device)
        out = torch.empty(n, nb, device=self.device)
        cdf = torch.empty(n, s + 1, device=self.device)
        inds = torch.empty(n, nb, device=self.device, dtype=torch.int32)
        self._check(self.lib.b200nerf_pdf_resample_stratified(self._h, _ptr(w), _ptr(b), _ptr(u), _ptr(r), r.shape[1], n, s, num_samples,
                                                              histogram_padding, _ptr(out), _ptr(cdf), _ptr(inds), self._stream))
        return out, cdf, inds

    def spaced_sample_stratified(self, nears: Optional[torch.Tensor], fars: torch.Tensor, num_samples: int, t_rand: torch.Tensor,
                                 spacing: str = "uniform", power_lambda: float = -1.0, power_scaling: float = 0.1):
        """SpacedSampler in training mode (train_stratified, ray_samplers.py:107-115): `t_rand` [N,1] (single_jitter)
        or [N,S+1]; returns (per-ray spacing bins [N,S+1], euclidean edges [N,S+1])."""
        f = self._dev(fars).reshape(-1)
        nr = None if nears is None else self._dev(nears).reshape(-1)
        r = self._dev(t_rand).reshape(f.shape[0], -1)
        n = f.shape[0]
        bins_s = torch.empty(n, num_samples + 1, device=self.device)
        bins_e = torch.empty(n, num_samples + 1, device=self.device)
        self._check(self.lib.b200nerf_spaced_sample_stratified(self._h, self.SPACINGS[spacing], power_lambda, power_scaling, _ptr(nr), _ptr(f),
                                                               _ptr(r), r.shape[1], n, num_samples, _ptr(bins_s), _ptr(bins_e), self._stream))
        return bins_s, bins_e

    def density_to_weights(self, deltas: torch.Tensor, densities: torch.Tensor) -> torch.Tensor:
        """RaySamples.get_weights (cameras/rays.py:188-210) on [N,S]."""
        d, s = self._dev(deltas), self._dev(densities)
        out = torch.empty_like(d)
        self._check(self.lib.b200nerf_density_to_weights(self._h, _ptr(d), _ptr(s), d.shape[0], d.shape[1], _ptr(out), self._stream))
        return out

    def alpha_to_weights(self, alphas: torch.Tensor) -> torch.Tensor:
        """nerfacc.render_weight_from_alpha, dense [N,S] (call site models/neurad.py:717)."""
        a = self._dev(alphas)
        out = torch.empty_like(a)
        self._check(self.lib.b200nerf_alpha_to_weights(self._h, _ptr(a), a.shape[0], a.shape[1], _ptr(out), self._stream))
        return out

    # ------------------------------------------------------------ module-level seams (Field / Sampler / Encoding)
    def isotropic_gaussian(self, origins: torch.Tensor, directions: torch.Tensor, pixel_area: torch.Tensor,
                           bins_e: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
        """Frustums.get_fast_isotropic_gaussian(1) (cameras/rays.py:109-124): per-ray origins / directions [N,3],
        pixel_area [N], euclidean edges [N,S+1] -> (mean [N,S,3], std [N,S])."""
        o, d = self._dev(origins).reshape(-1, 3), self._dev(directions).reshape(-1, 3)
        a, b = self._dev(pixel_area).reshape(-1), self._dev(bins_e)
        n, s = b.shape[0], b.shape[1] - 1
        mean = torch.empty(n, s, 3, device=self.device)
        std = torch.empty(n, s, device=self.device)
        self._check(self.lib.b200nerf_isotropic_gaussian_fwd(self._h, _ptr(o), _ptr(d), _ptr(a), _ptr(b), n, s, _ptr(mean), _ptr(std), self._stream))
        return mean, std

    def neurad_encoding(self, field: int, mean: torch.Tensor, std: torch.Tensor, times: Optional[torch.Tensor],
                        directions: Optional[torch.Tensor] = None, want_features: bool = True, want_density: bool = False,
                        want_actor_id: bool = False, flip: Optional[torch.Tensor] = None) -> Dict[str, torch.Tensor]:
        """NeuRADHashEncoding.forward (field_components/neurad_encoding.py:150-187) of the bound field `field`:
        mean [N,S,3], std [N,S] (or [N,S,1]), times [N] (or [N,1] / [N,S,1]: the reference reads times[:,0]),
        directions [N,3] or [N,S,3] -> {"features" [N*S,D], "directions" [N,S,3], "density" [N,S], "actor_id" [N,S]}.
        `flip` [N] (+1 / -1): the training-mode random actor flip drawn by the caller (:212-219)."""
        m = self._dev(mean)
        n, s = m.shape[0], m.shape[1]
        m = m.reshape(n, s, 3)
        sd = self._dev(std).reshape(n, s)
        t = self._ray_times(times, n)
        d = per_ray = None
        if directions is not None:
            per_ray = directions.numel() == 3 * n and s != 1
            d = self._dev(directions).reshape(n, 3) if per_ray else self._dev(directions).reshape(n, s, 3)
        g = {FIELD_MAIN: self.cfg.grid, FIELD_PROP0: self.cfg.proposal_grid_1, FIELD_PROP1: self.cfg.proposal_grid_2}[field].static
        out: Dict[str, torch.Tensor] = {}
        f = de = do = ai = None
        if want_features:
            f = out["features"] = torch.empty(n * s, g.num_levels * g.hashgrid_dim, device=self.device)
        if want_density:
            de = out["density"] = torch.empty(n, s, device=self.device)
        if d is not None:
            do = out["directions"] = torch.empty(n, s, 3, device=self.device)
        if want_actor_id:
            ai = out["actor_id"] = torch.empty(n, s, device=self.device, dtype=torch.int32)
        fl = None if flip is None else self._dev(flip).reshape(n)
        self._check(self.lib.b200nerf_neurad_encoding_fwd(self._h, field, _ptr(m), _ptr(sd), _ptr(t), _ptr(fl), _ptr(d), int(bool(per_ray)),
                                                          n, s, _ptr(f), _ptr(de), _ptr(do), _ptr(ai), self._stream))
        return out

    def field_forward(self, mean: torch.Tensor, std: torch.Tensor, times: torch.Tensor, directions: torch.Tensor,
                      flip: Optional[torch.Tensor] = None) -> Dict[str, torch.Tensor]:
        """NeuRADField.forward (fields/neurad_field.py:128-152) on gaussians: encoding -> mlp_geo (wgmma) ->
        [geo_embedding | SH] -> mlp_feature (wgmma) -> residual, sdf, alpha.  Five launches, all ours:
        {"feature" [N,S,G], "sdf" [N,S,1], "alpha" [N,S,1]}."""
        n, s = mean.shape[0], mean.shape[1]
        enc = self.neurad_encoding(FIELD_MAIN, mean, std, times, directions, flip=flip)
        gw, gb = self._field_mlps["geo"]
        fw, fb = self._field_mlps["feature"]
        geo = self.mlp_fwd(enc["features"], gw, gb)
        h = self.mlp_fwd(self._field_mid(geo, enc["directions"]), fw, fb)
        feature, sdf, alpha = self._field_tail(geo, h)
        gdim = feature.shape[1]
        return {"feature": feature.view(n, s, gdim), "sdf": sdf.view(n, s, 1), "alpha": alpha.view(n, s, 1)}

    def _field_mid(self, geo: torch.Tensor, directions: torch.Tensor) -> torch.Tensor:
        """geo_out [P,G+1], directions [P,3] -> mlp_feature's input [P,G+16] (neurad_field.py:139-141)."""
        p, gdim = geo.shape[0], geo.shape[1] - 1
        x2 = torch.empty(p, gdim + 16, device=self.device)
        self._check(self.lib.b200nerf_field_mid_fwd(self._h, _ptr(geo), _ptr(self._dev(directions).reshape(p, 3)), p, gdim, _ptr(x2), self._stream))
        return x2

    def _field_tail(self, geo: torch.Tensor, h: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """(feature [P,G] = geo_embedding + mlp_feature_out, sdf [P], alpha [P]) (neurad_field.py:141-149)."""
        p, gdim = geo.shape[0], geo.shape[1] - 1
        feature = torch.empty(p, gdim, device=self.device)
        sdf = torch.empty(p, device=self.device)
        alpha = torch.empty(p, device=self.device)
        self._check(self.lib.b200nerf_field_tail_fwd(self._h, _ptr(geo), _ptr(h), p, gdim, self._beta, _ptr(feature), _ptr(sdf), _ptr(alpha), self._stream))
        return feature, sdf, alpha

    def spacing_to_euclidean(self, bins_s: torch.Tensor, nears: Optional[torch.Tensor], fars: torch.Tensor, spacing: str = "power",
                             power_lambda: float = -1.0, power_scaling: float = 0.1) -> torch.Tensor:
        """spacing_to_euclidean_fn (ray_samplers.py:119-120) on per-ray spacing edges [N,E] -> euclidean edges [N,E]."""
        b = self._dev(bins_s)
        f = self._dev(fars).reshape(-1)
        nr = None if nears is None else self._dev(nears).reshape(-1)
        out = torch.empty_like(b)
        self._check(self.lib.b200nerf_spacing_to_euclidean(self._h, self.SPACINGS[spacing], power_lambda, power_scaling, _ptr(nr), _ptr(f),
                                                           _ptr(b), b.shape[0], b.shape[1], _ptr(out), self._stream))
        return out

    # ------------------------------------------------------------------------- backward operators (SURVEY 8f, f2)
    def neurad_encoding_bwd(self, field: int, mean: torch.Tensor, std: torch.Tensor, times: Optional[torch.Tensor],
                            grads: Dict[str, object], dfeatures: Optional[torch.Tensor] = None, density: Optional[torch.Tensor] = None,
                            ddensity: Optional[torch.Tensor] = None, flip: Optional[torch.Tensor] = None) -> None:
        """Backward of neurad_encoding: scatter-adds into grads["static"] [L*T,F], grads["actors"] (list of per-actor
        [La*Ta,F] tensors or None) and, in density mode (density + ddensity given), grads["decoder"] [L*F]."""
        # the mode is decided from the arguments here: an empty batch's tensors reach the library as NULL pointers
        if (dfeatures is None) == (ddensity is None) or (ddensity is not None and density is None):
            raise ValueError("pass either dfeatures or (density, ddensity)")
        if grads.get("decoder") is not None and ddensity is None:
            raise ValueError('grads["decoder"] belongs to the density mode')
        m = self._dev(mean)
        n, s = m.shape[0], m.shape[1]
        m = m.reshape(n, s, 3)
        sd = self._dev(std).reshape(n, s)
        t = self._ray_times(times, n)
        fl = None if flip is None else self._dev(flip).reshape(n)
        df = None if dfeatures is None else self._dev(dfeatures).reshape(n * s, dfeatures.shape[-1])  # (n * s may be 0)
        de = None if density is None else self._dev(density).reshape(n, s)
        dd = None if ddensity is None else self._dev(ddensity).reshape(n, s)
        for g in [grads.get("static"), grads.get("decoder")] + list(grads.get("actors") or []):
            assert g is None or (g.is_contiguous() and g.dtype == torch.float32 and g.device == self.device)
        acts = grads.get("actors")
        arr = None
        if acts:
            arr = (ctypes.c_void_p * len(acts))(*[None if g is None else g.data_ptr() for g in acts])
        self._check(self.lib.b200nerf_neurad_encoding_bwd(self._h, field, _ptr(m), _ptr(sd), _ptr(t), _ptr(fl), n, s, _ptr(df), _ptr(de), _ptr(dd),
                                                          _ptr(grads.get("static")), arr, _ptr(grads.get("decoder")), self._stream))

    def neurad_encoding_pose_bwd(self, field: int, mean: torch.Tensor, std: torch.Tensor, times: torch.Tensor, dfeatures: torch.Tensor,
                                 rotations_6d: torch.Tensor, positions: torch.Tensor, grad_rotations_6d: torch.Tensor,
                                 grad_positions: torch.Tensor, flip: Optional[torch.Tensor] = None) -> None:
        """Accumulates dL/d(actor_rotations_6d [T,A,6], actor_positions [T,A,3]) of a field's features (the reference
        does this for the main field only: require_actor_grad)."""
        m = self._dev(mean)
        n, s = m.shape[0], m.shape[1]
        m = m.reshape(n, s, 3)
        sd = self._dev(std).reshape(n, s)
        t = self._ray_times(times, n)
        fl = None if flip is None else self._dev(flip).reshape(n)
        df = self._dev(dfeatures).reshape(n * s, dfeatures.shape[-1])
        r6, ps = self._dev(rotations_6d), self._dev(positions)
        for g_ in (grad_rotations_6d, grad_positions):
            assert g_.is_contiguous() and g_.dtype == torch.float32 and g_.device == self.device
        self._check(self.lib.b200nerf_neurad_encoding_pose_bwd(self._h, field, _ptr(m), _ptr(sd), _ptr(t), _ptr(fl), n, s, _ptr(df), _ptr(r6),
                                                               _ptr(ps), _ptr(grad_rotations_6d), _ptr(grad_positions), self._stream))

    def neurad_encoding_mean_bwd(self, field: int, mean: torch.Tensor, std: torch.Tensor, times: Optional[torch.Tensor],
                                 dfeatures: Optional[torch.Tensor] = None, density: Optional[torch.Tensor] = None,
                                 ddensity: Optional[torch.Tensor] = None, flip: Optional[torch.Tensor] = None) -> torch.Tensor:
        """dL/d mean [N,S,3] of neurad_encoding (features mode: dfeatures; density mode: density + ddensity), for camera
        pose optimisation.  Actor samples contribute for the main field only (require_actor_grad); a proposal field's
        actor samples get exactly 0."""
        if (dfeatures is None) == (ddensity is None) or (ddensity is not None and density is None):
            raise ValueError("pass either dfeatures or (density, ddensity)")
        m = self._dev(mean)
        n, s = m.shape[0], m.shape[1]
        m = m.reshape(n, s, 3)
        sd = self._dev(std).reshape(n, s)
        t = self._ray_times(times, n)
        fl = None if flip is None else self._dev(flip).reshape(n)
        df = None if dfeatures is None else self._dev(dfeatures).reshape(n * s, dfeatures.shape[-1])
        de = None if density is None else self._dev(density).reshape(n, s)
        dd = None if ddensity is None else self._dev(ddensity).reshape(n, s)
        dmean = torch.empty(n, s, 3, device=self.device)
        self._check(self.lib.b200nerf_neurad_encoding_mean_bwd(self._h, field, _ptr(m), _ptr(sd), _ptr(t), _ptr(fl), n, s, _ptr(df), _ptr(de),
                                                               _ptr(dd), _ptr(dmean), self._stream))
        return dmean

    def isotropic_gaussian_bwd(self, bins_e: torch.Tensor, dmean: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
        """Backward of isotropic_gaussian: euclidean edges [N,S+1], dmean [N,S,3] -> (d origins [N,3], d directions [N,3])."""
        b = self._dev(bins_e)
        n, s = b.shape[0], b.shape[1] - 1
        dm = self._dev(dmean).reshape(n, s, 3)
        do = torch.empty(n, 3, device=self.device)
        dd = torch.empty(n, 3, device=self.device)
        self._check(self.lib.b200nerf_isotropic_gaussian_bwd(self._h, _ptr(b), n, s, _ptr(dm), _ptr(do), _ptr(dd), self._stream))
        return do, dd

    def hashgrid_bwd(self, g: HashGridSettings, x: torch.Tensor, dout: torch.Tensor, grad_table: torch.Tensor,
                     scalings: Optional[torch.Tensor] = None) -> None:
        """Backward of hashgrid_fwd: accumulates dL/d hash_table [L*T,F] from dL/d out [P, L*F]."""
        xs = self._dev(x).reshape(-1, 3)
        d = self._dev(dout).reshape(xs.shape[0], -1)
        assert grad_table.is_contiguous() and grad_table.dtype == torch.float32 and grad_table.device == self.device
        desc = grid_desc(g, scalings)
        self._check(self.lib.b200nerf_hashgrid_bwd(self._h, ctypes.byref(desc), _ptr(xs), _ptr(d), xs.shape[0], _ptr(grad_table), self._stream))

    def alpha_to_weights_bwd(self, alphas: torch.Tensor, dweights: torch.Tensor) -> torch.Tensor:
        a, dw = self._dev(alphas), self._dev(dweights)
        out = torch.empty_like(a)
        self._check(self.lib.b200nerf_alpha_to_weights_bwd(self._h, _ptr(a), _ptr(dw), a.shape[0], a.shape[1], _ptr(out), self._stream))
        return out

    def density_to_weights_bwd(self, deltas: torch.Tensor, densities: torch.Tensor, dweights: torch.Tensor) -> torch.Tensor:
        d, r, dw = self._dev(deltas), self._dev(densities), self._dev(dweights)
        out = torch.empty_like(d)
        self._check(self.lib.b200nerf_density_to_weights_bwd(self._h, _ptr(d), _ptr(r), _ptr(dw), d.shape[0], d.shape[1], _ptr(out), self._stream))
        return out

    def composite_bwd(self, weights: torch.Tensor, values: Optional[torch.Tensor], starts: Optional[torch.Tensor], ends: Optional[torch.Tensor],
                      dvalues_out: Optional[torch.Tensor], dacc: Optional[torch.Tensor], ddepth: Optional[torch.Tensor],
                      need_dweights: bool = True, need_dvalues: bool = True) -> Tuple[Optional[torch.Tensor], Optional[torch.Tensor]]:
        """Backward of composite(values / accumulation / "simple" depth): returns (dweights [N,S], dvalues [N,S,C])."""
        w = self._dev(weights)
        n, s = w.shape[0], w.shape[1]
        w = w.reshape(n, s)
        c = 0 if values is None else values.shape[-1]
        v = None if values is None else self._dev(values).reshape(n, s, c)
        st = None if starts is None else self._dev(starts).reshape(n, s)
        en = None if ends is None else self._dev(ends).reshape(n, s)
        go = None if dvalues_out is None else self._dev(dvalues_out).reshape(n, c)
        ga = None if dacc is None else self._dev(dacc).reshape(n)
        gd = None if ddepth is None else self._dev(ddepth).reshape(n)
        dw = torch.empty(n, s, device=self.device) if need_dweights else None
        dv = torch.empty(n, s, c, device=self.device) if (need_dvalues and go is not None) else None
        self._check(self.lib.b200nerf_composite_bwd(self._h, _ptr(w), _ptr(v), c, _ptr(st), _ptr(en), _ptr(go), _ptr(ga), _ptr(gd), n, s,
                                                    _ptr(dw), _ptr(dv), self._stream))
        return dw, dv

    def field_heads_bwd(self, geo: torch.Tensor, dfeature: Optional[torch.Tensor], dsdf: Optional[torch.Tensor],
                        dalpha: Optional[torch.Tensor], dx2: Optional[torch.Tensor]) -> Tuple[torch.Tensor, torch.Tensor]:
        """NeuRADField heads backward: returns (dgeo_out [P,G+1], dbeta [1] = dL/d(|beta|+1e-4))."""
        p, gdim = geo.shape[0], geo.shape[1] - 1
        f = lambda t, *shape: None if t is None else self._dev(t).reshape(*shape)  # noqa: E731
        dgeo = torch.empty(p, gdim + 1, device=self.device)
        dbeta = torch.zeros(1, device=self.device)
        self._check(self.lib.b200nerf_field_heads_bwd(self._h, _ptr(geo), _ptr(f(dfeature, p, gdim)), _ptr(f(dsdf, p)), _ptr(f(dalpha, p)),
                                                      _ptr(f(dx2, p, gdim + 16)), p, gdim, self._beta, _ptr(dgeo), _ptr(dbeta), self._stream))
        return dgeo, dbeta

    def linear_wgrad(self, x: torch.Tensor, dy: torch.Tensor, relu_x: bool, dweight: torch.Tensor, dbias: Optional[torch.Tensor],
                     impl: Optional[str] = None) -> None:
        """dweight [out,in] += dY^T act(X); dbias [out] += sum dY (act = ReLU when X is a hidden pre-activation).
        impl "cuda" (default: CUDA cores, GPU-validated) or "tc" (experimental wgmma split-K twin; also selected by the
        environment variable B200NERF_WGRAD=tc)."""
        xs, ds = self._dev(x), self._dev(dy)
        impl = impl or os.environ.get("B200NERF_WGRAD", "cuda")
        fn = {"cuda": self.lib.b200nerf_linear_wgrad, "tc": self.lib.b200nerf_linear_wgrad_tc}[impl]
        self._check(fn(self._h, _ptr(xs), _ptr(ds), xs.shape[0], xs.shape[1], ds.shape[1], int(relu_x), _ptr(dweight), _ptr(dbias),
                       self._stream))

    def mlp_dgrad(self, dy: torch.Tensor, weight: torch.Tensor, relu_z: Optional[torch.Tensor] = None) -> torch.Tensor:
        """dX = dY W of one Linear layer (weight = nn.Linear's [out, in]) on the wgmma operator; with `relu_z` (the
        pre-activation that fed the layer through ReLU) the result is masked by (relu_z > 0) in the same launch."""
        g = self._dev(dy).reshape(-1, dy.shape[-1]).contiguous()
        wt = self._dev(weight).t().contiguous()  # [in, out]
        dx = torch.empty(g.shape[0], wt.shape[0], device=self.device)
        if g.shape[0] == 0:
            return dx
        z = None if relu_z is None else self._dev(relu_z).reshape(g.shape[0], wt.shape[0]).contiguous()
        self._check(self.lib.b200nerf_mlp_dgrad(self._h, _ptr(g), g.shape[0], g.shape[1], _ptr(wt), wt.shape[0], _ptr(z), _ptr(dx), self._stream))
        return dx

    def relu_bwd(self, z: torch.Tensor, dz: torch.Tensor) -> torch.Tensor:
        """dz *= (z > 0), in place."""
        self._check(self.lib.b200nerf_relu_bwd(self._h, _ptr(z), _ptr(dz), dz.numel(), self._stream))
        return dz

    def mlp_bwd(self, x: torch.Tensor, weights: Sequence[torch.Tensor], biases: Optional[Sequence[Optional[torch.Tensor]]], dy: torch.Tensor,
                dweights: Sequence[Optional[torch.Tensor]], dbiases: Sequence[Optional[torch.Tensor]], need_dx: bool = True,
                hidden: Optional[Sequence[torch.Tensor]] = None) -> Optional[torch.Tensor]:
        """MLP.forward backward (field_components/mlp.py:142-178): accumulates into dweights[l] / dbiases[l] (entries may
        be None) and returns dL/dx.  Hidden pre-activations are recomputed with prefix forward passes (wgmma); dX = dY W
        runs through the same tensor-core operator with the transposed weight; dW through linear_wgrad."""
        x2 = self._dev(x).reshape(-1, x.shape[-1])
        nl = len(weights)
        bs = list(biases) if biases is not None else [None] * nl
        # pre-activation of hidden layer l: kept by the training forward (mlp_fwd(want_hidden=True)), else recomputed
        zs = list(hidden) if hidden is not None else [self.mlp_fwd(x2, weights[: l + 1], bs[: l + 1]) for l in range(nl - 1)]
        g = self._dev(dy).reshape(x2.shape[0], -1)
        for l in range(nl - 1, -1, -1):
            inp = x2 if l == 0 else zs[l - 1]
            if dweights[l] is not None:
                self.linear_wgrad(inp, g, l > 0, dweights[l], dbiases[l])
            if l == 0 and not need_dx:
                return None
            g = self.mlp_dgrad(g, weights[l], zs[l - 1] if l > 0 else None)
        return g.reshape(*x.shape)

    def lidar_carving_mask(self, bins_e: torch.Tensor, is_lidar: torch.Tensor, directions_norm: torch.Tensor,
                           did_return: Optional[torch.Tensor], carving_epsilon: float, non_return_distance: float) -> torch.Tensor:
        """NeuRADModel._compute_is_close_to_lidar (models/neurad.py:677-700): bool mask [N,S] of the samples close to the
        measured lidar return (or, for rays without a return, inside the lidar range); False for camera rays."""
        b = self._dev(bins_e)
        n, s = b.shape[0], b.shape[1] - 1
        il = self._dev(is_lidar.reshape(n), torch.uint8)
        dn = self._dev(directions_norm).reshape(n)
        dr = None if did_return is None else self._dev(did_return.reshape(n), torch.uint8)
        mask = torch.empty(n, s, device=self.device, dtype=torch.uint8)
        self._check(self.lib.b200nerf_lidar_carving_mask(self._h, _ptr(b), _ptr(il), _ptr(dn), _ptr(dr), float(carving_epsilon),
                                                         float(non_return_distance), n, s, _ptr(mask), self._stream))
        return mask.bool()

    def distortion_loss(self, sdist: torch.Tensor, weights: torch.Tensor, want_grad: bool = False):
        """lossfun_distortion per ray (model_components/losses.py:160-172): sdist [N,S+1], weights [N,S] ->
        (loss [N], d loss / d weights [N,S] or None)."""
        c, w = self._dev(sdist), self._dev(weights)
        n, s = w.shape
        loss = torch.empty(n, device=self.device)
        dw = torch.empty(n, s, device=self.device) if want_grad else None
        self._check(self.lib.b200nerf_distortion_loss(self._h, _ptr(c), _ptr(w), n, s, _ptr(loss), _ptr(dw), self._stream))
        return loss, dw

    def zipnerf_interlevel_loss(self, sdist: torch.Tensor, weights: torch.Tensor, prop_sdist: torch.Tensor, prop_weights: torch.Tensor,
                                pulse_width: float, want_grad: bool = False):
        """zipnerf_interlevel_loss for one proposal level, per ray (losses.py:645-705): final level sdist [N,S+1] /
        weights [N,S] (detached), proposal level [N,Sp+1] / [N,Sp] -> (loss [N], d loss / d prop_weights [N,Sp] or None)."""
        c, w, cp, wp = self._dev(sdist), self._dev(weights), self._dev(prop_sdist), self._dev(prop_weights)
        n, s, sp = w.shape[0], w.shape[1], wp.shape[1]
        loss = torch.empty(n, device=self.device)
        dwp = torch.empty(n, sp, device=self.device) if want_grad else None
        self._check(self.lib.b200nerf_zipnerf_interlevel_loss(self._h, _ptr(c), _ptr(w), s, _ptr(cp), _ptr(wp), sp, float(pulse_width), n,
                                                              _ptr(loss), _ptr(dwp), self._stream))
        return loss, dwp

    # ------------------------------------------------------------------- generic sampler / renderer operators
    SPACINGS = {"uniform": 0, "lindisp": 1, "power": 2, "sqrt": 3, "log": 4}
    DEPTH_METHODS = {None: 0, "expected": 1, "median": 2, "simple": 3}

    def spaced_sample(self, nears: Optional[torch.Tensor], fars: torch.Tensor, num_samples: int, spacing: str = "uniform",
                      power_lambda: float = -1.0, power_scaling: float = 0.1) -> Tuple[torch.Tensor, torch.Tensor]:
        """SpacedSampler.generate_ray_samples, eval mode (model_components/ray_samplers.py:80-132):
        nears/fars [N] or [N,1] -> (spacing bins [S+1], euclidean bin edges [N,S+1])."""
        f = self._dev(fars).reshape(-1)
        nr = None if nears is None else self._dev(nears).reshape(-1)
        n = f.shape[0]
        bins_s = torch.empty(num_samples + 1, device=self.device)
        bins_e = torch.empty(n, num_samples + 1, device=self.device)
        self._check(self.lib.b200nerf_spaced_sample(self._h, self.SPACINGS[spacing], power_lambda, power_scaling, _ptr(nr), _ptr(f), n,
                                                    num_samples, _ptr(bins_s), _ptr(bins_e), self._stream))
        if n == 0:
            bins_s = torch.linspace(0.0, 1.0, num_samples + 1, device=self.device)
        return bins_s, bins_e

    def frustum_positions(self, origins: torch.Tensor, directions: torch.Tensor, bins_e: torch.Tensor,
                          aabb: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Frustums.get_positions (cameras/rays.py:50-59) for contiguous bins [N,S+1] -> [N,S,3]; with `aabb` [2,3]
        also SceneBox.get_normalized_positions (data/scene_box.py:63-79)."""
        o, d, b = self._dev(origins).reshape(-1, 3), self._dev(directions).reshape(-1, 3), self._dev(bins_e)
        n, s = b.shape[0], b.shape[1] - 1
        out = torch.empty(n, s, 3, device=self.device)
        ab = None if aabb is None else (ctypes.c_float * 6)(*[float(v) for v in aabb.detach().float().cpu().reshape(-1)])
        self._check(self.lib.b200nerf_frustum_positions(self._h, _ptr(o), _ptr(d), _ptr(b), n, s, ab, _ptr(out), self._stream))
        return out

    def density_rgb_heads(self, raw: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
        """raw [*, 1+C] -> (density [*,1] = trunc_exp(raw[...,0]), rgb [*,C] = sigmoid(raw[...,1:]))."""
        r = self._dev(raw)
        c = r.shape[-1] - 1
        flat = r.reshape(-1, c + 1)
        density = torch.empty(flat.shape[0], device=self.device)
        rgb = torch.empty(flat.shape[0], c, device=self.device)
        self._check(self.lib.b200nerf_density_rgb_heads(self._h, _ptr(flat), flat.shape[0], c, _ptr(density), _ptr(rgb), self._stream))
        return density.reshape(*r.shape[:-1], 1), rgb.reshape(*r.shape[:-1], c)

    def composite(self, weights: torch.Tensor, values: Optional[torch.Tensor] = None, starts: Optional[torch.Tensor] = None,
                  ends: Optional[torch.Tensor] = None, depth_method: Optional[str] = None, background: Optional[Sequence[float]] = None,
                  value_nan_to_num: bool = False, want_accumulation: bool = True) -> Dict[str, torch.Tensor]:
        """Feature/RGB/Accumulation/Depth renderers on dense samples (model_components/renderers.py): weights [N,S]
        (or [N,S,1]), values [N,S,C], starts/ends [N,S] -> {"values" [N,C], "accumulation" [N,1], "depth" [N,1]}."""
        w = self._dev(weights)
        n, s = w.shape[0], w.shape[1]
        w = w.reshape(n, s)
        out: Dict[str, torch.Tensor] = {}
        v = ov = None
        c = 0
        if values is not None:
            c = values.shape[-1]
            v = self._dev(values).reshape(n, s, c)
            ov = out["values"] = torch.empty(n, c, device=self.device)
        oa = None
        if want_accumulation:
            oa = out["accumulation"] = torch.empty(n, 1, device=self.device)
        st = en = od = None
        if depth_method is not None:
            st, en = self._dev(starts).reshape(n, s), self._dev(ends).reshape(n, s)
            od = out["depth"] = torch.empty(n, 1, device=self.device)
        bg = None if background is None else (ctypes.c_float * c)(*[float(b) for b in background])
        self._check(self.lib.b200nerf_composite(self._h, _ptr(w), _ptr(v), c, int(value_nan_to_num), bg, _ptr(st), _ptr(en),
                                                self.DEPTH_METHODS[depth_method], n, s, _ptr(ov), _ptr(oa), _ptr(od), self._stream))
        return out

    # ------------------------------------------------------------------------------------- camera rgb decoder
    def set_rgb_decoder(self, sd: Dict[str, torch.Tensor], prefix: str = "rgb_decoder", bn_eps: float = 1e-5) -> None:
        """Bind NeuRADModel.rgb_decoder (models/neurad.py:201-216) from a reference state dict: keys
        `{prefix}.0.weight`, `{prefix}.2.main_branch.0.weight`, `{prefix}.2.main_branch.1.running_mean`, ...
        BatchNorms are folded into the 7x7 convolutions inside the library (eval-mode semantics)."""
        keep = []
        self._dec_owner = None
        self._check(self.lib.b200nerf_set_param_stream(self._h, self._stream))
        pre = prefix + "." if prefix else ""

        def t(key):
            v = self._dev(sd[pre + key])
            keep.append(v)
            return v.data_ptr()

        p = RgbDecoderParams()
        w0 = sd[pre + "0.weight"]
        p.in_dim, p.hidden_dim, p.upsample, p.bn_eps = w0.shape[1], w0.shape[0], sd[pre + "4.weight"].shape[-1], bn_eps
        p.in_conv = ConvParams(t("0.weight"), t("0.bias"))
        for b, blk in enumerate((2, 3, 5, 6)):
            for k, (cv, bn) in enumerate(((0, 1), (3, 4))):
                m = f"{blk}.main_branch"
                p.block[b][k] = ConvBnParams(t(f"{m}.{cv}.weight"), t(f"{m}.{cv}.bias"), t(f"{m}.{bn}.weight"), t(f"{m}.{bn}.bias"),
                                             t(f"{m}.{bn}.running_mean"), t(f"{m}.{bn}.running_var"))
        p.up_conv = ConvParams(t("4.weight"), t("4.bias"))
        p.out_conv = ConvParams(t("7.weight"), t("7.bias"))
        self._check(self.lib.b200nerf_set_rgb_decoder(self._h, ctypes.byref(p)))  # synchronous: `keep` may go now
        self._dec_in_dim = int(w0.shape[1])

    def rgb_decode(self, features: torch.Tensor, impl: str = "tc", out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Camera half of NeuRADModel.decode_features (neurad.py:359-366): features [B,H,W,C] (or [H,W,C]) ->
        rgb [B,3H,3W,3].  impl "tc": wgmma implicit-GEMM convolutions with TMA operand loads; "tc_ldgsts": the same
        with per-thread cp.async loads; "ref": CUDA-core fp32 cross-check."""
        f = self._dev(features)
        if f.dim() == 3:
            f = f[None]
        b, h, w, c = f.shape
        if c != getattr(self, "_dec_in_dim", None):
            raise _lib.B200NerfError(f"feature width {c} does not match the bound rgb decoder")
        need = int(self.lib.b200nerf_rgb_decode_workspace_bytes(b, h, w))
        ws = getattr(self, "_dec_ws", None)
        if ws is None or ws.numel() < need:
            ws = self._dec_ws = torch.empty(max(need, 16), dtype=torch.uint8, device=self.device)
        rgb = out if out is not None else torch.empty(b, 3 * h, 3 * w, 3, device=self.device)
        if rgb.shape != (b, 3 * h, 3 * w, 3) or not rgb.is_contiguous() or rgb.dtype != torch.float32 or rgb.device != f.device:
            raise _lib.B200NerfError("rgb_decode: `out` must be a contiguous fp32 [B,3H,3W,3] tensor on the backend's device")
        self._check(self.lib.b200nerf_rgb_decode_fwd(self._h, _ptr(f), b, h, w, _ptr(rgb), _ptr(ws), ws.numel(),
                                                     {"tc": 0, "ref": 1, "tc_ldgsts": 2}[impl], self._stream))
        return rgb

    def rgb_decode_layer(self, layer: int, x: torch.Tensor, residual: Optional[torch.Tensor] = None, impl: str = "tc",
                         out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """One of rgb_decode's ten launches (b200nerf_rgb_decode_layer).  Activations are ACT tensors: bf16 [B,H,W,64],
        elements 0..31 the hi parts (bf16 of the value) of the 32 channels, 32..63 their lo parts (bf16 of value - hi),
        which is the library's 128-byte ACT pixel.  Layer 0 takes fp32 features [B,H,W,in_dim]; layer 5 returns
        [B,3H,3W,64]; layer 9 returns fp32 rgb [B,H,W,3].  `residual` (ACT) is required for layers 2, 4, 7 and 9."""
        if not 0 <= layer <= 9:
            raise _lib.B200NerfError("layer must be in [0, 9]")
        want = torch.float32 if layer == 0 else torch.bfloat16
        if x.dtype != want or x.device != self.device or not x.is_contiguous() or x.dim() != 4:
            raise _lib.B200NerfError(f"rgb_decode_layer: input must be a contiguous {want} [B,H,W,C] tensor on the backend's device")
        b, h, w, c = x.shape
        if c != (getattr(self, "_dec_in_dim", None) if layer == 0 else 64):
            raise _lib.B200NerfError(f"rgb_decode_layer: layer {layer} input has {c} channels")
        if residual is not None and (residual.dtype != torch.bfloat16 or residual.shape != x.shape or not residual.is_contiguous()
                                     or residual.device != self.device):
            raise _lib.B200NerfError("rgb_decode_layer: residual must be an ACT tensor shaped like the input")
        up = 3 if layer == 5 else 1
        shape = (b, h * up, w * up, 3 if layer == 9 else 64)
        dtype = torch.float32 if layer == 9 else torch.bfloat16
        if out is None:
            out = torch.empty(shape, dtype=dtype, device=self.device)
        if out.shape != shape or out.dtype != dtype or not out.is_contiguous() or out.device != self.device:
            raise _lib.B200NerfError(f"rgb_decode_layer: `out` must be a contiguous {dtype} {list(shape)} tensor")
        self._check(self.lib.b200nerf_rgb_decode_layer(self._h, layer, _ptr(x), _ptr(residual), _ptr(out), b, h, w,
                                                       {"tc": 0, "ref": 1, "tc_ldgsts": 2}[impl], self._stream))
        return out

    # ------------------------------------------------------------------------------------------- ray generation
    def _ray_buffers(self, n: int, out: Optional[Dict[str, torch.Tensor]]):
        if out is None:
            return (torch.empty(n, 3, device=self.device), torch.empty(n, 3, device=self.device),
                    torch.empty(n, 1, device=self.device), torch.empty(n, 1, device=self.device))
        bufs = tuple(out[k] for k in ("origins", "directions", "pixel_area", "times"))
        for b, w in zip(bufs, (3, 3, 1, 1)):
            if not (b.is_contiguous() and b.device == self.device and b.dtype == torch.float32 and b.numel() == n * w):
                raise ValueError("pre-allocated ray buffer has the wrong layout")
        return bufs

    def raygen_camera(self, cam, row0: int = 0, row_step: int = 1, col0: int = 0, col_step: int = 1,
                      out: Optional[Dict[str, torch.Tensor]] = None) -> Dict[str, torch.Tensor]:
        """Cameras.generate_rays for one camera (scene.PinholeCamera: perspective or fisheye, optional k1..k4, p1, p2
        distortion, vertical or horizontal rolling shutter) over a strided pixel grid.
        `out` may hold pre-allocated (slices of) origins/directions/pixel_area/times buffers."""
        desc = camera_descriptor(cam)
        n_rows = len(range(row0, cam.height, row_step))
        n_cols = len(range(col0, cam.width, col_step))
        n = n_rows * n_cols
        o, d, a, t = self._ray_buffers(n, out)
        self._check(
            self.lib.b200nerf_raygen_camera(self._h, ctypes.byref(desc), row0, row_step, n_rows, col0, col_step, n_cols,
                                            _ptr(o), _ptr(d), _ptr(a), _ptr(t), self._stream)
        )
        return {"origins": o, "directions": d, "pixel_area": a, "times": t, "shape": (n_rows, n_cols)}

    def raygen_pinhole(self, cam, row0: int = 0, row_step: int = 1, col0: int = 0, col_step: int = 1,
                       out: Optional[Dict[str, torch.Tensor]] = None) -> Dict[str, torch.Tensor]:
        """raygen_camera under its original name (a default scene.PinholeCamera is an undistorted perspective camera
        with a top-to-bottom shutter)."""
        return self.raygen_camera(cam, row0, row_step, col0, col_step, out)

    def raygen_lidar_points(self, scan, points: Optional[torch.Tensor] = None,
                            out: Optional[Dict[str, torch.Tensor]] = None) -> Dict[str, torch.Tensor]:
        """Lidars.generate_rays(points=...) for one scan (scene.LidarScan)."""
        pts = self._dev(scan.points if points is None else points)
        n = pts.shape[0]
        o, d, a, t = self._ray_buffers(n, out)
        dist = torch.empty(n, 1, device=self.device)
        l2w = (ctypes.c_float * 12)(*scan.l2w.reshape(-1).tolist())
        vel = (ctypes.c_float * 3)(*scan.velocity.tolist()) if scan.velocity is not None else None
        self._check(
            self.lib.b200nerf_raygen_lidar_points(
                self._h, l2w, _ptr(pts), pts.shape[1], n, scan.time, vel, 3.0e-3, 1.5e-3, _ptr(o), _ptr(d), _ptr(a),
                _ptr(t), _ptr(dist), self._stream,
            )
        )
        res = {"origins": o, "directions": d, "pixel_area": a, "times": t, "directions_norm": dist}
        if out is None:  # metadata["did_return"] (lidars.py:447); skipped on the pre-allocated hot path
            res["did_return"] = dist < 1e3
        return res

    def raygen_lidar_grid(self, l2w: torch.Tensor, elev_min_deg: float, elev_max_deg: float, beams: int, azim_res_deg: float,
                          scan_time: float, revolution_time: float = 0.1, velocity: Optional[torch.Tensor] = None,
                          out: Optional[Dict[str, torch.Tensor]] = None) -> Dict[str, torch.Tensor]:
        """Beam x azimuth lidar grid with rolling shutter (BASELINE config 4 input: 128 beams x 2048 azimuths)."""
        import numpy as np

        step, n_az = lidar_columns(azim_res_deg)
        n = beams * n_az
        o, d, a, t = self._ray_buffers(n, out)
        cl2w = (ctypes.c_float * 12)(*l2w.reshape(-1).tolist())
        vel = (ctypes.c_float * 3)(*velocity.tolist()) if velocity is not None else None
        e0, e1 = (float(v) for v in np.deg2rad((elev_min_deg, elev_max_deg)).astype(np.float32))
        self._check(
            self.lib.b200nerf_raygen_lidar_grid(self._h, cl2w, e0, e1, beams, n_az, step, scan_time, revolution_time, vel,
                                                3.0e-3, 1.5e-3, _ptr(o), _ptr(d), _ptr(a), _ptr(t), self._stream)
        )
        return {"origins": o, "directions": d, "pixel_area": a, "times": t, "shape": (beams, n_az)}

    def raygen_lidar_sweeps(self, sensors, poses: torch.Tensor, times, velocities=None) -> Dict[str, torch.Tensor]:
        """Rays of S simulated sweeps in one launch (b200nerf_raygen_lidar_sweeps): `sensors` is one scene.LidarSensor or
        one per sweep, all with the same beam count and azimuth resolution; poses [S,3,4] (or [S,4,4]) sensor-to-world at
        the scan times; times [S]; velocities [S,3] or None (no origin motion).  Returns the flat ray buffers of the
        render (origins, directions, pixel_area, times, sensor_idx int64, is_lidar uint8), index [N,3] int32 (sweep,
        beam, column), `sweeps` (the device descriptors the point epilogue reads) and shape (S, beams, columns).

        The description is host data: it is validated on the host and uploaded without a host wait.  Poses, times or
        tables passed as CUDA tensors are read back to the host first, which waits on the device."""
        poses = torch.as_tensor(poses, dtype=torch.float32).cpu()
        if poses.dim() == 2:
            poses = poses[None]
        if poses.dim() != 3 or poses.shape[-2] not in (3, 4) or poses.shape[-1] != 4:
            raise ValueError(f"poses must be [S, 3, 4] or [S, 4, 4] sensor-to-world matrices, got {tuple(poses.shape)}")
        n_sw = poses.shape[0]
        times = torch.as_tensor(times, dtype=torch.float32).cpu().reshape(-1)
        sensors = list(sensors) if isinstance(sensors, (list, tuple)) else [sensors] * n_sw
        vel = None if velocities is None else torch.as_tensor(velocities, dtype=torch.float32).cpu().reshape(-1, 3)
        if n_sw < 1 or times.numel() != n_sw or len(sensors) != n_sw or (vel is not None and vel.shape[0] != n_sw):
            raise ValueError(f"{n_sw} poses need as many times, sensors and velocities (got {times.numel()}, {len(sensors)}, "
                             f"{None if vel is None else vel.shape[0]})")
        elev = [torch.as_tensor(s_.elevations, dtype=torch.float32).cpu().reshape(-1) for s_ in sensors]
        beams = elev[0].numel()
        res = float(sensors[0].azimuth_resolution_deg)
        if beams < 1 or any(e.numel() != beams for e in elev) or any(float(s_.azimuth_resolution_deg) != res for s_ in sensors):
            raise ValueError("every sweep of one call needs a non-empty beam table of one size and one azimuth resolution")
        step, n_az = lidar_columns(res)
        off = [torch.zeros(beams) if s_.azimuth_offsets is None else torch.as_tensor(s_.azimuth_offsets, dtype=torch.float32).cpu().reshape(-1)
               for s_ in sensors]
        if any(o.numel() != beams for o in off):
            raise ValueError("azimuth_offsets must hold one value per beam")
        elev, off = torch.stack(elev), torch.stack(off)
        desc = (_lib.LidarSweep * n_sw)()
        for i, s_ in enumerate(sensors):
            d = desc[i]
            d.l2w[:] = poses[i, :3].reshape(-1).tolist()
            d.scan_time, d.revolution_time = float(times[i]), float(s_.revolution_time)
            d.h_div, d.v_div, d.sensor_idx = float(s_.h_div), float(s_.v_div), int(s_.sensor_idx)
            if vel is not None:
                d.velocity[:] = vel[i].tolist()
                d.has_velocity = 1
            scal = list(d.l2w) + [d.scan_time, d.revolution_time, d.h_div, d.v_div] + list(d.velocity)
            if not all(math.isfinite(v) for v in scal):
                raise ValueError(f"sweep {i}: pose, time, velocity, revolution time and divergences must be finite")
        if not (torch.isfinite(elev).all() and torch.isfinite(off).all()):
            raise ValueError("beam tables must be finite")
        # descriptors, elevations and (when any is non-zero) offsets go up in one copy from pinned memory that does not
        # wait on the host: the caching host allocator keeps the staging block until the copy has run
        has_off = bool(off.any())
        n_desc, n_tab = ctypes.sizeof(desc), 4 * n_sw * beams
        stage = torch.empty(n_desc + n_tab * (2 if has_off else 1), dtype=torch.uint8, pin_memory=True)
        stage[:n_desc].copy_(torch.frombuffer(bytearray(bytes(desc)), dtype=torch.uint8))
        stage[n_desc:n_desc + n_tab].view(torch.float32).copy_(elev.reshape(-1))
        if has_off:
            stage[n_desc + n_tab:].view(torch.float32).copy_(off.reshape(-1))
        staged = stage.to(self.device, non_blocking=True)
        base = staged.data_ptr()
        sweeps = staged[:n_desc]
        elev_p = ctypes.c_void_p(base + n_desc)
        off_p = ctypes.c_void_p(base + n_desc + n_tab) if has_off else None
        n = n_sw * beams * n_az
        o, d_, a, t = self._ray_buffers(n, None)
        sensor_idx = torch.empty(n, 1, dtype=torch.int64, device=self.device)
        is_lidar = torch.empty(n, 1, dtype=torch.uint8, device=self.device)
        index = torch.empty(n, 3, dtype=torch.int32, device=self.device)
        self._check(self.lib.b200nerf_raygen_lidar_sweeps(
            self._h, _ptr(sweeps), n_sw, beams, n_az, step, elev_p, off_p, _ptr(o), _ptr(d_), _ptr(a), _ptr(t),
            _ptr(sensor_idx), _ptr(is_lidar), _ptr(index), self._stream))
        return {"origins": o, "directions": d_, "pixel_area": a, "times": t, "sensor_idx": sensor_idx,
                "is_lidar": is_lidar.view(torch.bool), "index": index, "sweeps": sweeps, "shape": (n_sw, beams, n_az)}

    def lidar_sweep_points(self, rays: Dict[str, torch.Tensor], depth: torch.Tensor, intensity: torch.Tensor,
                           ray_drop_prob: Optional[torch.Tensor], threshold: float) -> Dict[str, torch.Tensor]:
        """The point epilogue of rendered sweeps (b200nerf_lidar_sweep_points) for the rays of `raygen_lidar_sweeps`:
        kept = ray_drop_prob < threshold, or depth < threshold when ray_drop_prob is None.  Returns capacity-sized [N, ...]
        buffers points_sensor [N,5] (x, y, z, intensity, dt in the sweep's sensor frame), points_world [N,3], index [N,3]
        int32, whose first counts[-1] rows hold the kept rays in (sweep, beam, column) order, and counts [S+1] /
        offsets [S] int32 on the device.  Nothing synchronises the host."""
        n_sw, beams, n_az = rays["shape"]
        n = n_sw * beams * n_az

        def col(t):
            t = self._dev(t.detach().reshape(-1))
            if t.numel() != n:
                raise ValueError(f"lidar sweep points: {t.numel()} values for {n} rays")
            return t

        dep, inten = col(depth), col(intensity)
        prob = None if ray_drop_prob is None else col(ray_drop_prob)
        ps = torch.empty(n, 5, device=self.device)
        pw = torch.empty(n, 3, device=self.device)
        index = torch.empty(n, 3, dtype=torch.int32, device=self.device)
        counts = torch.empty(n_sw + 1, dtype=torch.int32, device=self.device)
        offsets = torch.empty(n_sw, dtype=torch.int32, device=self.device)
        ws = torch.empty(max(int(self.lib.b200nerf_lidar_sweep_workspace_bytes(n_sw, beams * n_az)), 16), dtype=torch.uint8,
                         device=self.device)
        self._check(self.lib.b200nerf_lidar_sweep_points(
            self._h, _ptr(rays["sweeps"]), n_sw, beams, n_az, _ptr(rays["origins"]), _ptr(rays["directions"]),
            _ptr(rays["times"]), _ptr(dep), _ptr(inten), _ptr(prob), int(prob is not None), float(threshold), _ptr(ps),
            _ptr(pw), _ptr(index), _ptr(counts), _ptr(offsets), _ptr(ws), ws.numel(), self._stream))
        return {"points_sensor": ps, "points_world": pw, "index": index, "counts": counts, "offsets": offsets}

    # ------------------------------------------------------------------------------------------ lidar evaluation
    def chamfer_distance(self, pred: torch.Tensor, gt: torch.Tensor, normalize_with_target: bool = True,
                         want_minima: bool = False):
        """Chamfer distance between point clouds pred [N,>=3] and gt [M,>=3] (x, y, z in the first three columns; a row
        stride is fine, so `points[..., :3]` of an [N,4] tensor needs no copy): sum_i min_j |p_i - g_j|^2 +
        sum_j min_i |g_j - p_i|^2, both sums divided by M with `normalize_with_target` (utils/math.py:783-796).
        Exact fp32 per-pair values, fp64 sums in a fixed order; returns a 0-d float64 tensor on the device, and with
        `want_minima` also the per-point minima [N] and [M] (fp32).  Empty clouds raise B200NerfError."""
        def rows(t):
            t = t.detach()
            if t.device != self.device or t.dtype != torch.float32 or t.dim() != 2 or t.shape[1] < 3 or t.stride(1) != 1:
                t = self._dev(t.reshape(-1, t.shape[-1]))
            return t

        p, g = rows(pred), rows(gt)
        n, m = p.shape[0], g.shape[0]
        out = torch.empty((), dtype=torch.float64, device=self.device)
        min_p = torch.empty(max(n, 1), device=self.device)[:n]
        min_g = torch.empty(max(m, 1), device=self.device)[:m]
        self._check(self.lib.b200nerf_chamfer_distance(self._h, _ptr(p), n, p.stride(0), _ptr(g), m, g.stride(0),
                                                       int(bool(normalize_with_target)), _ptr(out), _ptr(min_p), _ptr(min_g),
                                                       self._stream))
        return (out, min_p, min_g) if want_minima else out

    # ------------------------------------------------------------------------------------------ camera image metrics
    def image_metrics(self, a: torch.Tensor, b: torch.Tensor, data_range: Optional[float] = None) -> torch.Tensor:
        """PSNR (data range 1) and SSIM (11 x 11 Gaussian window, sigma 1.5) of image batches a, b [B, C, H, W], the shape
        the reference hands its metrics (neurad.py:581-586).  Any strides are read in place, so `moveaxis(img, -1, 0)[None]`
        of a channels-last [H, W, C] render needs no copy.  `data_range` None derives SSIM's range from the two images on
        the device, max(a.max() - a.min(), b.max() - b.min()), as torchmetrics does.

        Returns a [B + 1, 4] float64 tensor on the device: {mse, psnr, ssim, data_range} of the whole batch in row 0,
        then of each image.  Nothing synchronises the host.  The partial sums live in the context: calls on one backend
        must be ordered on one stream."""
        if a.dim() != 4 or a.shape != b.shape:
            raise ValueError(f"image metrics need two [B, C, H, W] tensors of one shape, got {tuple(a.shape)} and {tuple(b.shape)}")

        def view(t):
            t = t.detach()
            if t.device != self.device or t.dtype != torch.float32:
                t = t.to(device=self.device, dtype=torch.float32)
            return t, (ctypes.c_int64 * 4)(t.stride(0), t.stride(2), t.stride(3), t.stride(1))

        (ta, sa), (tb, sb) = view(a), view(b)
        n, ch, h, w = ta.shape
        out = torch.empty(n + 1, 4, dtype=torch.float64, device=self.device)
        self._check(self.lib.b200nerf_image_metrics(self._h, _ptr(ta), _ptr(tb), n, h, w, ch, sa, sb,
                                                    0.0 if data_range is None else float(data_range), _ptr(out), self._stream))
        return out

    # ------------------------------------------------------------------------------------------ lidar training losses
    def _lidar_loss_rows(self, pred, prop, distance, did_return, intensity, gt_intensity, logits):
        """Flatten the lidar-row inputs of the lidar losses to what the C ABI takes (no host synchronisation)."""
        def row(t):
            return self._dev(t.reshape(-1))

        n = distance.numel()
        gt = gt_intensity.detach().reshape(-1)
        if gt.device != self.device or gt.dtype != torch.float32:
            gt = self._dev(gt)
        p = [row(t) for t in prop]
        p = torch.stack(p) if p else None
        ret = did_return.detach().reshape(-1).to(device=self.device, dtype=torch.uint8)
        rows = (row(pred), p, row(distance), ret, row(intensity), gt, row(logits))
        if any(t is not None and t.shape[-1] != n for t in rows):
            raise ValueError("lidar losses: every per-ray input needs one entry per lidar ray")
        return rows

    def lidar_losses(self, pred, prop, distance, did_return, intensity, gt_intensity, logits, non_return_distance: float,
                     non_return_mult: float, quantile: float):
        """The lidar terms of get_metrics_dict in training mode (neurad.py:486-520) over n lidar rays.  Every input is in
        lidar rows ([n] or [n,1]): predicted depth, a list of proposal depths, measured distance, did_return (bool),
        predicted intensity, measured intensity (a strided column such as `lidar[:, 3]` is fine) and ray-drop logits.

        Returns (out, counts, mask): out [4 + rounds] fp32 = [depth_loss, intensity_loss, ray_drop_loss, quantile,
        depth_loss_0, ...], counts [2] int32 = [|mask|, |mask & did_return|], mask [n] bool = loss < quantile.  Nothing
        synchronises the host; n = 0 raises (torch.quantile of an empty tensor does too)."""
        n = distance.numel()
        if n == 0:
            raise _lib.B200NerfError("lidar losses of a batch without lidar rays (torch.quantile of an empty tensor)")
        pr, pp, d, ret, it, gt, lg = self._lidar_loss_rows(pred, prop, distance, did_return, intensity, gt_intensity, logits)
        r = 0 if pp is None else pp.shape[0]
        out = torch.empty(4 + r, device=self.device)
        counts = torch.empty(2, dtype=torch.int32, device=self.device)
        mask = torch.empty(n, dtype=torch.bool, device=self.device)
        ws = torch.empty(int(self.lib.b200nerf_lidar_losses_workspace_bytes(n)), dtype=torch.uint8, device=self.device)
        self._check(self.lib.b200nerf_lidar_losses_fwd(
            self._h, n, r, _ptr(pr), _ptr(pp), n, _ptr(d), _ptr(ret), _ptr(it), _ptr(gt), gt.stride(0), _ptr(lg),
            float(non_return_distance), float(non_return_mult), float(quantile), _ptr(out), _ptr(counts), _ptr(mask),
            _ptr(ws), ws.numel(), self._stream))
        return out, counts, mask

    def lidar_losses_bwd(self, pred, prop, distance, did_return, intensity, gt_intensity, logits, non_return_distance: float,
                         non_return_mult: float, mask, counts, grad_out):
        """Gradients of `lidar_losses`' out for upstream gradients grad_out [4 + rounds] (device; the quantile's entry is
        not read): (d pred [n], d prop [rounds, n], d intensity [n], d logits [n]).  mask / counts are the forward's."""
        n = distance.numel()
        pr, pp, d, ret, it, gt, lg = self._lidar_loss_rows(pred, prop, distance, did_return, intensity, gt_intensity, logits)
        r = 0 if pp is None else pp.shape[0]
        g = self._dev(grad_out)
        d_pred, d_int, d_lg = (torch.empty(n, device=self.device) for _ in range(3))
        d_prop = torch.empty(r, n, device=self.device)
        self._check(self.lib.b200nerf_lidar_losses_bwd(
            self._h, n, r, _ptr(pr), _ptr(pp), n, _ptr(d), _ptr(ret), _ptr(it), _ptr(gt), gt.stride(0), _ptr(lg),
            float(non_return_distance), float(non_return_mult), _ptr(mask), _ptr(counts), _ptr(g), _ptr(d_pred),
            _ptr(d_prop) if r else None, _ptr(d_int), _ptr(d_lg), self._stream))
        return d_pred, d_prop, d_int, d_lg

    def quantile(self, x: torch.Tensor, q: float, lower_median: bool = False) -> torch.Tensor:
        """torch.quantile(x, q) (linear interpolation), or with `lower_median` torch.median(x), over all of x, bit for bit,
        as a 0-d device tensor and without a host synchronisation; the selection of `lidar_losses`.  1 <= x.numel() <= 2^24.
        -0 and +0 are one key: a zero at the rank comes back as +0 (torch may return -0 there)."""
        v = self._dev(x.reshape(-1))
        out = torch.empty((), device=self.device)
        ws = torch.empty(int(self.lib.b200nerf_lidar_losses_workspace_bytes(0)), dtype=torch.uint8, device=self.device)
        self._check(self.lib.b200nerf_quantile(self._h, _ptr(v), v.numel(), float(q), int(bool(lower_median)), _ptr(out),
                                               _ptr(ws), ws.numel(), self._stream))
        return out
