"""Shared bodies of the preset tests: the reference's NeuRAD method presets (method_configs.py:395-507) -- per-sensor
appearance (neurad-paper, neurad-2x-paper) and doubled grids (neurader, neuradest, neurad-2x-paper).

GPU (tests/test_zz_presets_gpu.py) runs them through the C ABI; CPU (tests/test_presets_cpu.py) through the host emulation
and the oracle.  The goldens tests/golden/nff_paper.npz / nff_neurader.npz come from the unmodified reference
(oracle/make_golden_presets.py)."""
import torch

import neurad_studio_b200 as nsb
from oracle import presets_oracle as PO
from tests.helpers import load_golden

GOLDENS = ("nff_paper.npz", "nff_neurader.npz")


def cfg_from_preset_meta(meta):
    cfg = PO.shrink_tables(nsb.preset(meta["preset"])[0], meta["log2_main"], meta["log2_prop"])
    cfg.n_actors, cfg.static_scale = meta["n_actors"], meta["static_scale"]
    cfg.duration, cfg.num_sensors = meta["duration"], meta["num_sensors"]
    return cfg


def load_preset_golden(name):
    meta, g = load_golden(name)
    return meta, cfg_from_preset_meta(meta), g["param"], g["ray"], g["ref"]


def check_appearance_columns(features, ref_features, nff=32):
    """The appearance columns are a copy (per-sensor) or one fp32 lerp evaluated in the reference's order (temporal):
    bit for bit either way."""
    a, b = features.detach().cpu()[:, nff:].contiguous(), ref_features[:, nff:].contiguous()
    assert a.shape == b.shape, (a.shape, b.shape)
    n_diff = int((a.view(torch.int32) != b.view(torch.int32)).sum())
    assert n_diff == 0, f"{n_diff} appearance entries differ from the reference"


def reference_preset_fields(name):
    """The numbers of the reference's `method_configs[name]` that the backend's preset has to carry."""
    from nerfstudio.configs.method_configs import method_configs

    mc = method_configs[name].pipeline.model

    def grid(g):
        s, a = g.static, g.actor
        return {"static": (s.hashgrid_dim, s.num_levels, s.base_res, s.max_res, s.log2_hashmap_size),
                "actor": (a.hashgrid_dim, a.num_levels, a.base_res, a.max_res, a.log2_hashmap_size),
                "actor_scale": a.actor_scale, "flip_prob": a.flip_prob}

    co = mc.camera_optimizer
    copt = {"mode": co.mode, "weights": tuple(getattr(co, "weights", (1.0,) * 6)),
            "trans_l2_penalty": tuple(co.trans_l2_penalty) if isinstance(co.trans_l2_penalty, (tuple, list)) else co.trans_l2_penalty,
            "rot_l2_penalty": co.rot_l2_penalty}
    sp = mc.sampling
    return {"grids": [grid(f.grid) for f in mc.fields], "use_temporal_appearance": mc.use_temporal_appearance,
            "appearance_dim": mc.appearance_dim, "temporal_appearance_freq": mc.temporal_appearance_freq,
            "sampling": (tuple(sp.num_proposal_samples), sp.num_nerf_samples, sp.power_lambda, sp.power_scaling, sp.sky_distance,
                         sp.single_jitter),
            "field": (mc.field.geo_hidden_dim, mc.field.nff_hidden_dim, mc.field.nff_out_dim, mc.field.num_multisamples),
            "camera_optimizer": copt}


def backend_preset_fields(name):
    cfg, co = nsb.preset(name)

    def grid(g):
        s, a = g.static, g.actor
        return {"static": (s.hashgrid_dim, s.num_levels, s.base_res, s.max_res, s.log2_hashmap_size),
                "actor": (a.hashgrid_dim, a.num_levels, a.base_res, a.max_res, a.log2_hashmap_size),
                "actor_scale": g.actor_scale, "flip_prob": g.flip_prob}

    copt = {"mode": co.mode, "weights": tuple(getattr(co, "weights", (1.0,) * 6)),
            "trans_l2_penalty": tuple(co.trans_l2_penalty) if isinstance(co.trans_l2_penalty, (tuple, list)) else co.trans_l2_penalty,
            "rot_l2_penalty": co.rot_l2_penalty}
    sp = cfg.sampling
    return {"grids": [grid(g) for g in (cfg.grid, *cfg.proposal_grids)], "use_temporal_appearance": cfg.use_temporal_appearance,
            "appearance_dim": cfg.appearance_dim, "temporal_appearance_freq": cfg.temporal_appearance_freq,
            "sampling": (tuple(sp.num_proposal_samples), sp.num_nerf_samples, sp.power_lambda, sp.power_scaling, sp.sky_distance,
                         sp.single_jitter),
            "field": (cfg.geo_hidden_dim, cfg.nff_hidden_dim, cfg.nff_out_dim, cfg.num_multisamples),
            "camera_optimizer": copt}
