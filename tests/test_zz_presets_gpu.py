"""GPU: the reference's other NeuRAD presets through the C ABI.

- nff_paper.npz (neurad-paper: one appearance row per sensor) and nff_neurader.npz (neurader: doubled resolutions, finest
  main level 16383) in all four kernel modes, to the bounds of the default goldens (tests/test_parity_gpu.py): sample
  indices and actor ids exact, outputs within 1e-4 of their scale, and the appearance columns bit for bit.
- neurader at production size: a 2^23-row main table (1 GB), 2^21-row proposal tables, 16 actors, against the live
  oracle (the existing live-oracle body, called with the doubled grid).
- the module-level mirror of the paper preset (per-sensor embedding in eval mode)."""
import pytest
import torch

import neurad_studio_b200 as nsb
from neurad_studio_b200.backend import DEFAULT_MODE
from tests.preset_cases import GOLDENS, check_appearance_columns, load_preset_golden
from tests.test_parity_gpu import _check_against, _live_case, rel_to_max

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def backend():
    from neurad_studio_b200.backend import B200Backend

    return B200Backend(torch.device("cuda", 0))


@pytest.mark.parametrize("mode", ["lane", "split", "tc", "ffma"])
@pytest.mark.parametrize("name", GOLDENS)
def test_preset_golden_all_modes(backend, name, mode):
    meta, cfg, p, r, ref = load_preset_golden(name)
    backend.load_params(cfg, p)
    backend.set_mlp_mode(mode)
    try:
        out = backend.render(r, want_trace=True, want_intensity=True)
        backend.check_status()
    finally:
        backend.set_mlp_mode(DEFAULT_MODE)
    _check_against(out, ref, meta["beta"])
    check_appearance_columns(out["features"], ref["features"])
    assert rel_to_max(out["intensity"], ref["intensity"]) < 1e-4
    assert rel_to_max(out["ray_drop_logits"], ref["ray_drop_logits"]) < 1e-4


def test_per_sensor_appearance_without_sensor_idx_uses_sensor_0(backend):
    """A bundle without sensor_idx (the viewer's fallback sensor) reads row 0, as the temporal branch does."""
    meta, cfg, p, r, ref = load_preset_golden("nff_paper.npz")
    backend.load_params(cfg, p)
    rays = {k: v for k, v in r.items() if k != "sensor_idx"}
    out = backend.render(rays)
    backend.check_status()
    emb = p["appearance_embedding.weight"]
    assert torch.equal(out["features"][:, 32:].cpu(), emb[0].expand(r["origins"].shape[0], -1))


def test_per_sensor_c_abi_rejects_what_set_appearance_rejects(backend):
    meta, cfg, p, r, ref = load_preset_golden("nff_paper.npz")
    emb = p["appearance_embedding.weight"].cuda()
    lib, h = backend.lib, backend._h
    assert lib.b200nerf_set_appearance_per_sensor(h, emb.data_ptr(), emb.shape[0], 17) != 0
    assert lib.b200nerf_set_appearance_per_sensor(h, None, emb.shape[0], 16) != 0
    assert lib.b200nerf_set_appearance_per_sensor(h, emb.data_ptr(), 0, 16) != 0
    # the temporal entry point still refuses eps <= 0, the per-sensor marker
    assert lib.b200nerf_set_appearance(h, emb.data_ptr(), emb.shape[0], 16, 0, 8.0) != 0


def test_neurader_production_size_vs_oracle(backend):
    """neurader tables as trained: main 8 x 2^23 x 4 floats (1 GB), proposal 6 x 2^21 (48 MB each), actors 2^18 / 2^16
    rows, 16 actors."""
    cfg, _ = nsb.preset("neurader")
    cfg.n_actors = 16
    assert cfg.grid.static.log2_hashmap_size == 23 and cfg.grid.static.scalings()[-1].item() == 16383.0
    out, ref = _live_case(backend, cfg, 512, seed=51, beta=4.0, sdf_bias=0.5)
    assert int((ref["actor_id_main"] >= 0).sum()) > 20  # the actor branch is exercised
    for k in ("actor_id_0", "actor_id_1", "actor_id_main"):
        assert int((out[k].cpu().long() != ref[k].long()).sum()) == 0, k
    for k in ("inds_1", "inds_2"):
        assert (out[k].cpu().long() != ref[k].long()).float().mean().item() <= 1e-3, k
    for k in ("features", "accumulation", "depth", "prop_depth_0", "prop_depth_1"):
        assert rel_to_max(out[k], ref[k]) < 1e-4, (k, rel_to_max(out[k], ref[k]))
    del out, ref
    torch.cuda.empty_cache()


def test_fused_grids_reject_tables_beyond_32_bit_offsets(backend):
    """b200nerf_set_field_grids: a main (F = 4) table of 2^29 rows does not fit 32-bit byte offsets; 2^28 would."""
    import ctypes

    from neurad_studio_b200.backend import grid_desc

    g = nsb.HashGridSettings(4, 8, 64, 16384, 29)
    sd = grid_desc(g, None)
    dummy = torch.zeros(4, device="cuda")
    rc = backend.lib.b200nerf_set_field_grids(backend._h, 0, ctypes.byref(sd), dummy.data_ptr(), None, None, 0, 100.0, 10.0)
    assert rc != 0 and b"32-bit" in backend.lib.b200nerf_last_error()


def test_mirror_model_paper_preset_matches_golden():
    from neurad_studio_b200.nerfstudio_api import NeuRADModel, RayBundle

    meta, cfg, p, r, ref = load_preset_golden("nff_paper.npz")
    model = NeuRADModel(cfg)
    model.load_reference_state_dict(p)
    model = model.cuda().eval()
    rb = RayBundle(origins=r["origins"].cuda(), directions=r["directions"].cuda(), pixel_area=r["pixel_area"].cuda(),
                   times=r["times"].cuda(), metadata={"is_lidar": r["is_lidar"].cuda(), "sensor_idxs": r["sensor_idx"].cuda()})
    out = model.get_nff_outputs(rb)
    for k in ("features", "accumulation", "depth", "prop_depth_0", "prop_depth_1"):
        assert rel_to_max(out[k], ref[k]) < 1e-4, k
    check_appearance_columns(out["features"], ref["features"])


# ---- the neurader grid at production size through the existing per-entry bodies (the grid is their one new parameter)
def _neurader_cfg(n_actors=0, **_):
    cfg, _copt = nsb.preset("neurader")
    cfg.n_actors = n_actors
    return cfg


class _NeuraderNsb:
    """neurad_studio_b200 with NeuRADConfig(...) building the neurader grid: the production-size scenes of
    tests/render_trace_cases.py at the doubled resolutions (finest main level 16383) and tables (main 2^23 rows)."""

    def __getattr__(self, k):
        return _neurader_cfg if k == "NeuRADConfig" else getattr(nsb, k)


def test_neurader_render_trace_sample_by_sample(monkeypatch):
    from tests import render_trace_cases as RT

    monkeypatch.setattr(RT, "nsb", _NeuraderNsb())
    ws, exits, faces, full, idx = RT.check_scene("cuda", "config3", "split")
    print("\n[neurader render trace] config3: worst ratio to bound " + ", ".join(f"{k} {v:.3g}" for k, v in ws.items())
          + f"; actor-id face exceptions {faces}")


@pytest.mark.parametrize("mode", ["features", "density", "pose", "hashgrid"])
def test_neurader_backward_scatters_per_entry(monkeypatch, mode):
    """The scatters into the 1 GB main table (features mode), the 2^21-row proposal table (density mode), the actor
    trajectories (pose mode) and the stand-alone hashgrid_bwd on an 8 x 2^23 x 4 table, with prefilled accumulators."""
    from tests import backward_scatter_cases as BS

    monkeypatch.setattr(BS, "make_cfg", lambda dev, n_actors: _neurader_cfg(n_actors))
    if mode == "features":
        w = BS.features_mode_matches_float64_reference("cuda", 1031, 32, 16, True)
    elif mode == "density":
        w = BS.density_mode_matches_float64_reference("cuda", 1024, 64, 16, True, True)
    elif mode == "pose":
        w = BS.pose_bwd_matches_oracle_per_actor_and_keyframe("cuda", 16, True)
    else:
        w = BS.hashgrid_bwd_matches_float64_reference("cuda", 8, 4, 23, 1 << 16)
    print(f"\n[neurader backward scatter] {mode}: worst ratio to tolerance {w:.3f}")
    torch.cuda.empty_cache()


def test_neurader_tcnn_layout_render_vs_tcnn_oracle(monkeypatch):
    """The tiny-cuda-nn layout at neurader sizes: main grid levels 0-1 dense, 2-7 hashed into 2^23 entries each."""
    from tests import tcnn_cases as TC

    monkeypatch.setattr(TC, "tcnn_test_config", _neurader_cfg)
    TC.fused_render_matches_tcnn_oracle("cuda", n_actors=3, n_rays=96)
    torch.cuda.empty_cache()


def test_tcnn_layout_paper_checkpoint_renders():
    """A tcnn-layout checkpoint of a per-sensor model: the embedding is the same tensor in both layouts."""
    import dataclasses

    from neurad_studio_b200 import scene
    from neurad_studio_b200.nerfstudio_api import get_backend
    from oracle import presets_oracle as PO
    from tests.tcnn_cases import tcnn_test_config

    cfg = dataclasses.replace(tcnn_test_config(3), use_temporal_appearance=False)
    trajs = scene.make_trajectories(3, cfg.duration, seed=2)
    params = scene.make_params_tcnn(cfg, seed=3, beta=1.5, trajectories=trajs, mlp_gain=0.6)
    assert params["appearance_embedding.weight"].shape[0] == cfg.num_sensors
    rays = scene.random_rays(96, cfg, seed=5, trajectories=trajs)
    with torch.no_grad():
        ref = PO.nff_outputs(params, cfg, rays["origins"], rays["directions"], rays["pixel_area"], rays["times"],
                             rays["sensor_idx"], rays["is_lidar"])
    be = get_backend(torch.device("cuda", 0))
    be.load_params(cfg, params)
    assert be.layout == "tcnn"
    out = be.render(rays)
    be.check_status()
    check_appearance_columns(out["features"], ref["features"])
    for k in ("features", "accumulation", "depth", "prop_depth_0", "prop_depth_1"):
        assert rel_to_max(out[k], ref[k]) < 1e-4, (k, rel_to_max(out[k], ref[k]))


def test_paper_preset_module_walk_matches_reference_gradients(monkeypatch):
    """Training through the mirror's module walk on the neurad-paper golden: every trained tensor's gradient, the per-sensor
    appearance_embedding.weight included, against the reference's autograd (tests/golden/grads_paper.npz) within the
    existing 2e-3 per-group bound."""
    from tests import module_seam_cases as MS
    from tests.helpers import load_golden
    from tests.preset_cases import cfg_from_preset_meta

    def grads(name):
        meta, g = load_golden("grads_paper.npz")
        return meta, g["grad"]

    monkeypatch.setattr(MS, "cfg_from_meta", cfg_from_preset_meta)
    monkeypatch.setattr(MS, "load_golden_grads", grads)
    assert "appearance_embedding.weight" in grads("nff_paper.npz")[1]
    MS.training_gradients_match_reference_golden("nff_paper.npz", "cuda")


@pytest.mark.parametrize("name", nsb.PRESETS)
def test_each_preset_trains_through_the_module_walk(name):
    """One training step of every preset at its production table sizes (4 actors, the preset's camera optimizer): the walk
    runs, and every trained group -- the appearance embedding of either mode included -- receives a finite, nonzero gradient."""
    from neurad_studio_b200 import scene
    from neurad_studio_b200.nerfstudio_api import NeuRADModel, RayBundle

    cfg, copt = nsb.preset(name)
    cfg.n_actors = 4
    trajs = scene.make_trajectories(4, cfg.duration, seed=1)
    model = NeuRADModel(cfg, trajs, camera_optimizer=None if copt.mode == "off" else copt, num_cameras=cfg.num_sensors).cuda()
    model.requires_grad_(True)
    model.train()
    rays = scene.random_rays(2048, cfg, seed=2, trajectories=trajs)
    rb = RayBundle(origins=rays["origins"].cuda(), directions=rays["directions"].cuda(), pixel_area=rays["pixel_area"].cuda(),
                   times=rays["times"].cuda(), camera_indices=rays["sensor_idx"].cuda(),
                   metadata={"is_lidar": rays["is_lidar"].cuda(), "sensor_idxs": rays["sensor_idx"].cuda()})
    if model.camera_optimizer.config.mode != "off":
        rb = rb.flatten()
        model.camera_optimizer.apply_to_raybundle(rb)
    out = model.get_nff_outputs(rb)
    assert "weights_list" in out
    (out["features"].square().mean() + 0.01 * out["depth"].mean() + out["prop_depth_1"].mean() * 1e-3).backward()
    sd = model.reference_state_dict()
    for k in ("appearance_embedding.weight", "field.hashgrid.static_grid.hash_table", "field.mlp_geo.layers.0.weight",
              "proposal_fields.1.hashgrid.static_grid.hash_table", "proposal_fields.1.density_decoder.weight"):
        g = sd[k].grad
        assert g is not None and torch.isfinite(g).all() and g.abs().max().item() > 0, k
    assert sd["appearance_embedding.weight"].shape[0] == cfg.num_appearance_embeds
    model._bind().check_status()
    del model
    torch.cuda.empty_cache()
