"""TEST INFRASTRUCTURE ONLY -- the oracle for the reference's NeuRAD method presets (method_configs.py:395-507).

`nff_outputs` extends oracle/neurad_oracle.py's `nff_outputs` with the per-sensor branch of
NeuRADModel._get_appearance_embedding (neurad.py:440, use_temporal_appearance = False, the paper presets): the appearance
columns are `appearance_embedding.weight[sensor_idx]`, copied.  Everything else, the doubled grids of neurader included,
is the unmodified oracle; with temporal appearance the call is that oracle's, bit for bit.
"""
from __future__ import annotations

import copy

import torch

from . import neurad_oracle as O
from .convert import to_oracle_cfg


def shrink_tables(cfg, log2_main: int = 10, log2_prop: int = 10):
    """A copy of `cfg` with small hash tables and unchanged levels / resolutions, the rule of `small_config`: static
    tables 2^log2_main (main) and 2^log2_prop (proposal), actor tables 8 times smaller (at least 2^6)."""
    cfg = copy.deepcopy(cfg)
    cfg.grid.static.log2_hashmap_size = log2_main
    cfg.grid.actor.log2_hashmap_size = max(log2_main - 3, 6)
    for g in cfg.proposal_grids:
        g.static.log2_hashmap_size = log2_prop
        g.actor.log2_hashmap_size = max(log2_prop - 3, 6)
    return cfg


def appearance_per_sensor(params, sensor_idx: torch.Tensor) -> torch.Tensor:
    """neurad.py:440: `self.appearance_embedding(sensor_idx.squeeze(-1))`.  sensor_idx [N,1] int64."""
    return params["appearance_embedding.weight"][sensor_idx.reshape(-1).long()]


def nff_outputs(params, cfg, origins, directions, pixel_area, times, sensor_idx, is_lidar=None, fars=None, nears=None,
                want_trace=False):
    """oracle/neurad_oracle.nff_outputs for a product `NeuRADConfig` of either appearance mode."""
    ocfg = to_oracle_cfg(cfg)
    if cfg.use_temporal_appearance:
        return O.nff_outputs(params, ocfg, origins, directions, pixel_area, times, sensor_idx, is_lidar, fars, nears, want_trace)
    # the temporal oracle on a stand-in table of the temporal shape, then the per-sensor columns in its place
    emb = params["appearance_embedding.weight"]
    stand_in = dict(params)
    stand_in["appearance_embedding.weight"] = torch.zeros(cfg.num_sensors * cfg.embeds_per_sensor, emb.shape[1], dtype=emb.dtype)
    out = O.nff_outputs(stand_in, ocfg, origins, directions, pixel_area, times, torch.zeros_like(sensor_idx), is_lidar, fars,
                        nears, want_trace)
    nff = cfg.nff_out_dim
    out["features"] = torch.cat([out["features"][:, :nff], appearance_per_sensor(params, sensor_idx)], dim=-1)
    return out
