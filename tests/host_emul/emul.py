"""TEST SCAFFOLDING ONLY -- ctypes driver for the host SIMT emulation of the render kernel (emul.cpp)."""
import ctypes
import os
import subprocess

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
SO = os.path.join(HERE, "libnffemul.so")
SRC = os.path.join(HERE, "emul.cpp")
CSRC = os.path.join(os.path.dirname(os.path.dirname(HERE)), "neurad-studio_b200", "csrc")


def build(force=False):
    deps = [SRC] + [os.path.join(CSRC, f) for f in ("nff_device.h", "nff_lane.h", "nff_modules.h", "nff_params.h", "simt.h")]
    if force or not os.path.exists(SO) or any(os.path.getmtime(d) > os.path.getmtime(SO) for d in deps):
        subprocess.check_call(
            ["g++", "-std=c++20", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-pthread", "-o", SO, SRC]
        )
    return SO


class _Pack:
    """ptrs / ints / floats argument arrays of the emulation entry points."""

    def __init__(self):
        self.keep, self.ptrs, self.ints, self.floats = [], [], [], []

    def P(self, t):
        if t is None:
            self.ptrs.append(None)
            return None
        t = t.contiguous()
        self.keep.append(t)
        self.ptrs.append(ctypes.c_void_p(t.data_ptr()))
        return t

    def c_arrays(self):
        return ((ctypes.c_void_p * len(self.ptrs))(*self.ptrs), (ctypes.c_int * len(self.ints))(*self.ints),
                (ctypes.c_float * len(self.floats))(*self.floats))


def _pack_params(pk, cfg, params, pdf_u, field_of_round):
    """Everything emul.cpp's parse_params() reads: grids, MLPs, actors, sampling, appearance."""
    keep, ptrs, ints, floats, P = pk.keep, pk.ptrs, pk.ints, pk.floats, pk.P
    n_actors = cfg.n_actors
    n_times = int(params["dynamic_actors.unique_timestamps"].shape[0]) if n_actors else 0
    ints += [n_actors, n_times]
    prefixes = ["field", "proposal_fields.0", "proposal_fields.1"]
    gcfgs = [cfg.grid, cfg.proposal_grid_1, cfg.proposal_grid_2]
    for pre, g in zip(prefixes, gcfgs):
        for name, s in (("static_grid", g.static), ("actor_grids.0", g.actor)):
            ints += [s.num_levels, s.hashgrid_dim, s.log2_hashmap_size]
            key = f"{pre}.hashgrid.{name}.scalings"
            sc = params[key].tolist() if key in params else s.scalings().tolist()
            floats += sc + [0.0] * (16 - len(sc))
        P(params[f"{pre}.hashgrid.static_grid.hash_table"])
        if n_actors:
            tabs = [params[f"{pre}.hashgrid.actor_grids.{a}.hash_table"].contiguous() for a in range(n_actors)]
            keep.extend(tabs)
            arr = (ctypes.c_void_p * n_actors)(*[t.data_ptr() for t in tabs])
            keep.append(arr)
            ptrs.append(ctypes.cast(arr, ctypes.c_void_p))
        else:
            ptrs.append(None)
        P(params.get(f"{pre}.density_decoder.weight"))
        floats += [float(params["static_scale"]), g.actor_scale]
    for k in ("field.mlp_geo.layers.0", "field.mlp_geo.layers.1", "field.mlp_feature.layers.0",
              "field.mlp_feature.layers.1", "field.mlp_feature.layers.2"):
        P(params[k + ".weight"])
        P(params[k + ".bias"])
    floats.append(float(params["field.sdf_to_density.beta"].abs() + 0.0001))
    if n_actors:
        P(params["dynamic_actors.unique_timestamps"])
        P(params["dynamic_actors.actor_rotations_6d"])
        P(params["dynamic_actors.actor_positions"])
        P(params["dynamic_actors.actor_present_at_time"].to(torch.uint8))
        P(params["dynamic_actors.actor_sizes"])
    else:
        for _ in range(5):
            ptrs.append(None)
    floats += list(cfg.actor_bbox_padding)
    sp = cfg.sampling
    floats += [sp.power_lambda, sp.power_scaling, sp.sky_distance, sp.histogram_padding, float(cfg.rgb_upsample_factor**2)]
    P(pdf_u(sp.num_proposal_samples[1]))
    P(pdf_u(sp.num_nerf_samples))
    ints += list(field_of_round)
    P(params["appearance_embedding.weight"])
    ints += [int(params["appearance_embedding.weight"].shape[0]), cfg.appearance_dim, cfg.embeds_per_sensor]
    floats.append(cfg.duration)


def _tcnn_level_ints(layout):
    out, dense_bits = [], 0
    for l in range(16):
        if l < layout["n_levels"]:
            dense_bits |= (1 << l) if layout["dense"][l] else 0
            out += [layout["resolution"][l], layout["offset"][l], layout["size"][l] if layout["dense"][l] else layout["size"][l] - 1]
        else:
            out += [0, 0, 0]
    return dense_bits, out


def _torch_shaped_standin(cfg, params):
    """A torch-layout dict with the same non-grid tensors (MLPs unpacked from the tcnn vectors, zero biases) and dummy hash
    tables, so that the ordinary parameter block can be packed; the grids are then overridden with the tcnn layout."""
    from neurad_studio_b200 import tcnn_compat as T

    q = {k: v for k, v in params.items() if T.TCNN_SUFFIX not in k}
    for pre, g in (("field", cfg.grid), ("proposal_fields.0", cfg.proposal_grid_1), ("proposal_fields.1", cfg.proposal_grid_2)):
        q[f"{pre}.hashgrid.static_grid.hash_table"] = torch.zeros(8, g.static.hashgrid_dim)
        for a in range(cfg.n_actors):
            q[f"{pre}.hashgrid.actor_grids.{a}.hash_table"] = torch.zeros(8, g.actor.hashgrid_dim)
    for pre, dims in (("field.mlp_geo", (cfg.grid.static.out_dim, cfg.geo_hidden_dim, 2, cfg.nff_out_dim + 1)),
                      ("field.mlp_feature", (cfg.nff_out_dim + 16, cfg.nff_hidden_dim, 3, cfg.nff_out_dim)),
                      ("lidar_decoder", (cfg.feature_dim, 32, 3, 2))):
        ts = T.mlp_tensors(params, pre, *dims, "cpu")
        for i in range(dims[2]):
            q[f"{pre}.layers.{i}.weight"], q[f"{pre}.layers.{i}.bias"] = ts[2 * i], ts[2 * i + 1]
    return q


def render(cfg, params, rays, pdf_u, field_of_round=(2, 2), lane_mode=False):
    """cfg: neurad_studio_b200.NeuRADConfig; params: reference-named tensors (CPU); rays: dict of CPU tensors.  A
    tcnn-layout parameter set (tcnn_compat.is_tcnn_state) runs the LAYOUT = 1 instantiation of the ray-per-lane code."""
    from neurad_studio_b200 import tcnn_compat as T

    lib = ctypes.CDLL(build())
    lib.emul_render.restype = ctypes.c_int
    pk = _Pack()
    tcnn_keep = None
    if T.is_tcnn_state(params):
        assert lane_mode, "the tcnn layout exists in the ray-per-lane kernels only"
        t_ptrs, t_ints, t_floats, tcnn_keep = [], [], [], []
        for pre, g in (("field", cfg.grid), ("proposal_fields.0", cfg.proposal_grid_1), ("proposal_fields.1", cfg.proposal_grid_2)):
            for name, gs, nd in (("static_grid", g.static, 3), ("actor_grids.0", g.actor, 4)):
                lay = T.layout_of(gs, nd)
                bits, li = _tcnn_level_ints(lay)
                t_ints += [nd, bits] + li
                t_floats += lay["scale"] + [0.0] * (16 - lay["n_levels"])
                key = f"{pre}.hashgrid.{name}.{T.TCNN_SUFFIX}"
                if key in params:
                    t = T.half_round(params[key].reshape(-1)).contiguous()
                    tcnn_keep.append(t)
                    t_ptrs.append(ctypes.c_void_p(t.data_ptr()))
                else:
                    t_ptrs.append(None)
        arrs = ((ctypes.c_void_p * len(t_ptrs))(*t_ptrs), (ctypes.c_int * len(t_ints))(*t_ints), (ctypes.c_float * len(t_floats))(*t_floats))
        tcnn_keep.append(arrs)
        lib.emul_set_tcnn(*arrs)
        params = _torch_shaped_standin(cfg, params)
        lane_mode = 2
    _pack_params(pk, cfg, params, pdf_u, field_of_round)
    keep, P = pk.keep, pk.P
    sp = cfg.sampling
    n = rays["origins"].shape[0]
    P(rays["origins"].float())
    P(rays["directions"].float())
    P(rays["pixel_area"].reshape(-1).float())
    P(rays["times"].reshape(-1).float())
    P(rays["nears"].reshape(-1).float() if "nears" in rays else None)
    P(rays["fars"].reshape(-1).float() if "fars" in rays else None)
    P(rays["sensor_idx"].reshape(-1).long() if "sensor_idx" in rays else None)
    P(rays["is_lidar"].reshape(-1).to(torch.uint8) if "is_lidar" in rays else None)
    S0, S1 = sp.num_proposal_samples
    S2 = sp.num_nerf_samples
    out = {
        "features": torch.zeros(n, cfg.feature_dim), "depth": torch.zeros(n, 1), "accumulation": torch.zeros(n, 1),
        "prop_depth_0": torch.zeros(n, 1), "prop_depth_1": torch.zeros(n, 1),
        "prop_weights_0": torch.zeros(n, S0), "prop_weights_1": torch.zeros(n, S1),
        "bins_s_1": torch.zeros(n, S1 + 1), "bins_e_1": torch.zeros(n, S1 + 1),
        "bins_s_2": torch.zeros(n, S2 + 1), "bins_e_2": torch.zeros(n, S2 + 1),
        "inds_1": torch.zeros(n, S1 + 1, dtype=torch.int32), "inds_2": torch.zeros(n, S2 + 1, dtype=torch.int32),
        "sdf": torch.zeros(n, S2), "alpha": torch.zeros(n, S2), "field_feature": torch.zeros(n, S2, cfg.nff_out_dim),
        "weights": torch.zeros(n, S2),
        "actor_id_0": torch.zeros(n, S0, dtype=torch.int32), "actor_id_1": torch.zeros(n, S1, dtype=torch.int32),
        "actor_id_main": torch.zeros(n, S2, dtype=torch.int32),
    }
    for k in out:
        P(out[k])
        out[k] = keep[-1]
    c_ptrs, c_ints, c_floats = pk.c_arrays()
    rc = lib.emul_render(c_ptrs, c_ints, c_floats, ctypes.c_longlong(n), ctypes.c_int(int(lane_mode)))
    assert rc == 0
    del tcnn_keep
    return out


def tcnn_hashgrid(layout, params, x):
    """tcnn.Encoding{HashGrid}.forward through the device functions: x [P, n_dims] -> [P, L*F]."""
    lib = ctypes.CDLL(build())
    bits, li = _tcnn_level_ints(layout)
    ints = [layout["n_dims"], layout["n_levels"], layout["n_features"], bits] + li[: 3 * layout["n_levels"]]
    c_ints = (ctypes.c_int * len(ints))(*ints)
    c_sc = (ctypes.c_float * layout["n_levels"])(*layout["scale"])
    p, xs = params.contiguous().float(), x.contiguous().float()
    out = torch.zeros(xs.shape[0], layout["n_levels"] * layout["n_features"])
    rc = lib.emul_tcnn_hashgrid(c_ints, c_sc, ctypes.c_void_p(p.data_ptr()), ctypes.c_void_p(xs.data_ptr()), ctypes.c_longlong(xs.shape[0]),
                                ctypes.c_void_p(out.data_ptr()))
    assert rc == 0
    return out


def gaussian(origins, directions, pixel_area, bins_e):
    """sample_gaussian() of csrc/nff_device.h on frustums: (mean [N,S,3], std [N,S])."""
    lib = ctypes.CDLL(build())
    n, s = bins_e.shape[0], bins_e.shape[1] - 1
    ts = [t.float().contiguous() for t in (origins.reshape(-1, 3), directions.reshape(-1, 3), pixel_area.reshape(-1), bins_e)]
    mean, std = torch.zeros(n, s, 3), torch.zeros(n, s)
    rc = lib.emul_gaussian(*[ctypes.c_void_p(t.data_ptr()) for t in ts], ctypes.c_longlong(n), ctypes.c_int(s),
                           ctypes.c_void_p(mean.data_ptr()), ctypes.c_void_p(std.data_ptr()))
    assert rc == 0
    return mean, std


def encoding(cfg, params, pdf_u, field, mean, std, times, directions=None, want_features=True, want_density=False,
             want_actor_id=True, flip=None):
    """The module-level NeuRADHashEncoding.forward device code (csrc/nff_modules.h) of field `field` (0 main, 1 / 2
    proposal): mean [N,S,3], std [N,S], times [N], directions [N,3] / [N,S,3] / None -> {"features" [N*S,D],
    "directions" [N,S,3], "actor_id" [N,S], "density" [N,S]} (same contract as B200Backend.neurad_encoding)."""
    lib = ctypes.CDLL(build())
    lib.emul_encoding.restype = ctypes.c_int
    pk = _Pack()
    _pack_params(pk, cfg, params, pdf_u, (2, 2))
    g = [cfg.grid, cfg.proposal_grid_1, cfg.proposal_grid_2][field].static
    n, s = mean.shape[0], mean.shape[1]
    ex = _Pack()
    ex.P(mean.float().reshape(n, s, 3))
    ex.P(std.float().reshape(n, s))
    ex.P(None if times is None else times.float().reshape(n, -1)[:, 0])
    per_ray = directions is not None and directions.numel() == 3 * n and s != 1
    ex.P(None if directions is None else directions.float().reshape(n, 3) if per_ray else directions.float().reshape(n, s, 3))
    out = {}
    feats = ex.P(torch.zeros(n * s, g.num_levels * g.hashgrid_dim) if want_features else None)
    dens = ex.P(torch.zeros(n, s) if want_density else None)
    dout = ex.P(torch.zeros(n, s, 3) if directions is not None else None)
    aid = ex.P(torch.zeros(n, s, dtype=torch.int32) if want_actor_id else None)
    ex.P(None if flip is None else flip.float().reshape(n))
    for k, v in (("features", feats), ("density", dens), ("directions", dout), ("actor_id", aid)):
        if v is not None:
            out[k] = v
    c_ptrs, c_ints, c_floats = pk.c_arrays()
    c_extra = (ctypes.c_void_p * len(ex.ptrs))(*ex.ptrs)
    rc = lib.emul_encoding(c_ptrs, c_ints, c_floats, c_extra, ctypes.c_longlong(n), ctypes.c_int(s), ctypes.c_int(field),
                           ctypes.c_int(1 if per_ray else 0))
    assert rc == 0
    return out


def set_bwd_generic(on: bool) -> None:
    """Run the generic (any L x F, MODE 0) variant of the scatter backward instead of the register-resident fast paths."""
    ctypes.CDLL(build()).emul_set_bwd_generic(ctypes.c_int(1 if on else 0))


def encoding_bwd(cfg, params, pdf_u, field, mean, std, times, grads, dfeatures=None, density=None, ddensity=None, flip=None):
    """Backward of `encoding` (csrc/nff_modules.h: neurad_encode_point_bwd).  `grads` = {"static": tensor | None,
    "actors": [tensor | None] * n_actors | None, "decoder": tensor | None}, accumulated in place (same contract as
    B200Backend.neurad_encoding_bwd)."""
    lib = ctypes.CDLL(build())
    lib.emul_encoding_bwd.restype = ctypes.c_int
    pk = _Pack()
    _pack_params(pk, cfg, params, pdf_u, (2, 2))
    n, s = mean.shape[0], mean.shape[1]
    ex = _Pack()
    ex.P(mean.float().reshape(n, s, 3))
    ex.P(std.float().reshape(n, s))
    ex.P(None if times is None else times.float().reshape(n) if times.numel() == n else times.float().reshape(n, -1)[:, 0])
    ex.P(None if flip is None else flip.float().reshape(n))
    ex.P(None if dfeatures is None else dfeatures.float().reshape(n * s, dfeatures.shape[-1]))
    ex.P(None if density is None else density.float().reshape(n, s))
    ex.P(None if ddensity is None else ddensity.float().reshape(n, s))
    for t in (grads.get("static"),):
        assert t is None or (t.is_contiguous() and t.dtype == torch.float32)
        ex.ptrs.append(None if t is None else ctypes.c_void_p(t.data_ptr()))
    acts = grads.get("actors")
    if acts:
        arr = (ctypes.c_void_p * len(acts))(*[None if t is None else t.data_ptr() for t in acts])
        ex.keep.append(arr)
        ex.ptrs.append(ctypes.cast(arr, ctypes.c_void_p))
    else:
        ex.ptrs.append(None)
    t = grads.get("decoder")
    ex.ptrs.append(None if t is None else ctypes.c_void_p(t.data_ptr()))
    c_ptrs, c_ints, c_floats = pk.c_arrays()
    c_extra = (ctypes.c_void_p * len(ex.ptrs))(*ex.ptrs)
    rc = lib.emul_encoding_bwd(c_ptrs, c_ints, c_floats, c_extra, ctypes.c_longlong(n), ctypes.c_int(s), ctypes.c_int(field))
    assert rc == 0


def weights_bwd(from_alpha, a, b, dw):
    """alpha_weights_bwd_ray / density_weights_bwd_ray on [N,S] rows."""
    lib = ctypes.CDLL(build())
    a = a.float().contiguous()
    b = None if b is None else b.float().contiguous()
    dw = dw.float().contiguous()
    out = torch.zeros_like(a)
    p = lambda t: None if t is None else ctypes.c_void_p(t.data_ptr())  # noqa: E731
    rc = lib.emul_weights_bwd(ctypes.c_int(int(from_alpha)), p(a), p(b), p(dw), ctypes.c_longlong(a.shape[0]), ctypes.c_int(a.shape[1]), p(out))
    assert rc == 0
    return out


def linear_wgrad(x, dy, relu_x, dW, db, n_ctas=3):
    """linear_wgrad_kernel's tiling: accumulates dY^T act(X) into dW [N,K] and sum dY into db [N]."""
    lib = ctypes.CDLL(build())
    x, dy = x.float().contiguous(), dy.float().contiguous()
    p = lambda t: None if t is None else ctypes.c_void_p(t.data_ptr())  # noqa: E731
    rc = lib.emul_linear_wgrad(p(x), p(dy), ctypes.c_longlong(x.shape[0]), ctypes.c_int(x.shape[1]), ctypes.c_int(dy.shape[1]),
                               ctypes.c_int(int(relu_x)), ctypes.c_int(n_ctas), p(dW), p(db))
    assert rc == 0


def distortion_loss(sdist, weights, want_grad=True):
    """distortion_loss_ray per ray: (loss [N], dweights [N,S])."""
    lib = ctypes.CDLL(build())
    c, w = sdist.float().contiguous(), weights.float().contiguous()
    loss = torch.zeros(c.shape[0])
    dw = torch.zeros_like(w) if want_grad else None
    p = lambda t: None if t is None else ctypes.c_void_p(t.data_ptr())  # noqa: E731
    rc = lib.emul_distortion_loss(p(c), p(w), ctypes.c_longlong(c.shape[0]), ctypes.c_int(w.shape[1]), p(loss), p(dw))
    assert rc == 0
    return loss, dw


def zipnerf_interlevel(sdist, weights, prop_sdist, prop_weights, pulse_width, want_grad=True):
    """zipnerf_interlevel_ray per ray for one proposal level: (loss [N], dprop_weights [N,Sp])."""
    lib = ctypes.CDLL(build())
    c, w = sdist.float().contiguous(), weights.float().contiguous()
    cp, wp = prop_sdist.float().contiguous(), prop_weights.float().contiguous()
    loss = torch.zeros(c.shape[0])
    dwp = torch.zeros_like(wp) if want_grad else None
    p = lambda t: None if t is None else ctypes.c_void_p(t.data_ptr())  # noqa: E731
    rc = lib.emul_zipnerf_interlevel(p(c), p(w), ctypes.c_int(w.shape[1]), p(cp), p(wp), ctypes.c_int(wp.shape[1]),
                                     ctypes.c_float(pulse_width), ctypes.c_longlong(c.shape[0]), p(loss), p(dwp))
    assert rc == 0
    return loss, dwp


def encoding_pose_bwd(cfg, params, pdf_u, field, mean, std, times, dfeatures, grad_rot6, grad_pos, flip=None):
    """Trajectory gradients (csrc/nff_modules.h: neurad_encode_point_pose_bwd): accumulates dL/d(actor_rotations_6d,
    actor_positions) into grad_rot6 [T,A,6] / grad_pos [T,A,3] (same contract as B200Backend.neurad_encoding_pose_bwd)."""
    lib = ctypes.CDLL(build())
    lib.emul_encoding_pose_bwd.restype = ctypes.c_int
    pk = _Pack()
    _pack_params(pk, cfg, params, pdf_u, (2, 2))
    n, s = mean.shape[0], mean.shape[1]
    ex = _Pack()
    ex.P(mean.float().reshape(n, s, 3))
    ex.P(std.float().reshape(n, s))
    ex.P(times.float().reshape(n, -1)[:, 0])
    ex.P(None if flip is None else flip.float().reshape(n))
    ex.P(dfeatures.float().reshape(n * s, -1))
    ex.P(params["dynamic_actors.actor_rotations_6d"].detach().float())
    ex.P(params["dynamic_actors.actor_positions"].detach().float())
    for t in (grad_rot6, grad_pos):
        assert t.is_contiguous() and t.dtype == torch.float32
        ex.ptrs.append(ctypes.c_void_p(t.data_ptr()))
    c_ptrs, c_ints, c_floats = pk.c_arrays()
    c_extra = (ctypes.c_void_p * len(ex.ptrs))(*ex.ptrs)
    rc = lib.emul_encoding_pose_bwd(c_ptrs, c_ints, c_floats, c_extra, ctypes.c_longlong(n), ctypes.c_int(s), ctypes.c_int(field))
    assert rc == 0


def hashgrid_bwd(num_levels, features_per_level, log2_hashmap_size, scalings, x, dout, grad_table):
    """encode_levels_bwd with unit level weights: accumulates dL/d hash_table from dL/d out [P, L*F]."""
    lib = ctypes.CDLL(build())
    sc = scalings.float().contiguous()
    xs, d = x.float().reshape(-1, 3).contiguous(), dout.float().contiguous()
    p = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731
    rc = lib.emul_hashgrid_bwd(ctypes.c_int(num_levels), ctypes.c_int(features_per_level), ctypes.c_int(log2_hashmap_size), p(sc), p(xs),
                               p(d), ctypes.c_longlong(xs.shape[0]), p(grad_table))
    assert rc == 0
