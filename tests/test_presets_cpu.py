"""CPU: the reference's NeuRAD presets -- configs against the reference's own method_configs, the per-sensor oracle against
the goldens, the per-sensor epilogue in the host emulation, the plugin's config mapping, and comparator self-tests."""
import dataclasses

import pytest
import torch

import neurad_studio_b200 as nsb
from oracle import presets_oracle as PO
from oracle import ref_import
from tests.preset_cases import (GOLDENS, backend_preset_fields, check_appearance_columns, load_preset_golden,
                                reference_preset_fields)

needs_reference = pytest.mark.skipif(not ref_import.reference_available(), reason="the reference tree exists in the build container only")


@pytest.fixture(scope="module")
def reference():
    ref_import.install(full=True)


@needs_reference
@pytest.mark.parametrize("name", nsb.PRESETS)
def test_preset_equals_reference_method_config(reference, name):
    assert backend_preset_fields(name) == reference_preset_fields(name)


@needs_reference
@pytest.mark.parametrize("name", ["neurad-paper", "neurad-2x-paper"])
def test_paper_presets_still_flip_actors(reference, name):
    """method_configs.py:501-507 sets `f.flip_prob = 0.0` on the field configs, which have no such field; the encoding
    reads grid.actor.flip_prob (neurad_encoding.py:212-214), so training still flips actors."""
    from nerfstudio.configs.method_configs import method_configs

    mc = method_configs[name].pipeline.model
    assert [f.grid.actor.flip_prob for f in mc.fields] == [0.25, 0.5, 0.5]
    cfg, _ = nsb.preset(name)
    assert [g.flip_prob for g in (cfg.grid, *cfg.proposal_grids)] == [0.25, 0.5, 0.5]
    assert not cfg.use_temporal_appearance and cfg.num_appearance_embeds == cfg.num_sensors


def test_unknown_preset_raises():
    with pytest.raises(ValueError):
        nsb.preset("neurad-3x")


@pytest.mark.parametrize("name", GOLDENS)
def test_oracle_reproduces_preset_golden(name):
    meta, cfg, p, r, ref = load_preset_golden(name)
    with torch.no_grad():
        out = PO.nff_outputs(p, cfg, r["origins"], r["directions"], r["pixel_area"], r["times"], r["sensor_idx"], r["is_lidar"])
    for k in ("features", "depth", "accumulation", "prop_depth_0", "prop_depth_1"):
        assert torch.equal(out[k], ref[k]), k


@pytest.mark.parametrize("lane_mode", [True, False])
def test_host_emulation_per_sensor_epilogue(lane_mode):
    """Both output epilogues (shade_ray_lane: modes 3 / 2; the warp-per-ray epilogue: modes 1 / 0) on 32 rays of the
    neurad-paper golden: the appearance columns bit for bit, the rest within 1e-4."""
    from oracle import neurad_oracle as O
    from tests.host_emul import emul
    from tests.preset_fake_backend import emul_cfg

    meta, cfg, p, r, ref = load_preset_golden("nff_paper.npz")
    n = 32
    rays = {k: v[:n] for k, v in r.items()}
    out = emul.render(emul_cfg(cfg), p, rays, O.pdf_u, lane_mode=lane_mode)
    check_appearance_columns(out["features"], ref["features"][:n])
    for k in ("features", "depth", "accumulation"):
        b = ref[k][:n]
        assert (out[k].reshape(b.shape) - b).abs().max().item() <= 1e-4 * b.abs().max().item(), k


def test_comparator_rejects_wrong_appearance():
    meta, cfg, p, r, ref = load_preset_golden("nff_paper.npz")
    emb, sens, f = p["appearance_embedding.weight"], r["sensor_idx"].reshape(-1), ref["features"]
    check_appearance_columns(f.clone(), f)
    bad = f.clone()  # a neighbouring sensor's row
    bad[:, 32:] = emb[(sens + 1) % emb.shape[0]]
    with pytest.raises(AssertionError):
        check_appearance_columns(bad, f)
    bad = f.clone()  # a temporal lerp between a sensor's row and the next one in place of the copy
    w = (r["times"] / cfg.duration).reshape(-1, 1)
    bad[:, 32:] = emb[sens] * (1 - w) + emb[(sens + 1) % emb.shape[0]] * w
    with pytest.raises(AssertionError):
        check_appearance_columns(bad, f)
    bad = f.clone()  # one ulp in one appearance column
    bad[5, 40] = torch.nextafter(bad[5, 40], torch.tensor(float("inf")))
    with pytest.raises(AssertionError):
        check_appearance_columns(bad, f)


def test_state_dicts_of_the_two_modes_do_not_mix():
    from neurad_studio_b200.nerfstudio_api import NeuRADModel

    temporal = nsb.small_config(n_actors=0)
    paper = dataclasses.replace(nsb.small_config(n_actors=0), use_temporal_appearance=False)
    a, b = NeuRADModel(temporal), NeuRADModel(paper)
    assert b.reference_state_dict()["appearance_embedding.weight"].shape[0] == paper.num_sensors
    with pytest.raises(RuntimeError, match="size mismatch"):
        b.load_state_dict(a.state_dict())
    with pytest.raises(RuntimeError, match="size mismatch"):
        a.load_state_dict(b.state_dict())
    tc = NeuRADModel(paper, implementation="tcnn")
    assert tc.reference_state_dict()["appearance_embedding.weight"].shape == (paper.num_sensors, paper.appearance_dim)


def test_mirror_per_sensor_gradient_reaches_the_embedding():
    """Training: the per-sensor columns are the sensor's row, and d loss / d weight is the sum of the columns' upstream
    gradients per sensor (the reference's nn.Embedding backward)."""
    from neurad_studio_b200.nerfstudio_api import NeuRADModel, RayBundle

    cfg = dataclasses.replace(nsb.small_config(n_actors=0), use_temporal_appearance=False)
    model = NeuRADModel(cfg)
    emb = model.reference_state_dict()["appearance_embedding.weight"]
    emb.requires_grad_(True)
    n = 64
    sens = torch.randint(0, cfg.num_sensors, (n, 1))
    rb = RayBundle(origins=torch.zeros(n, 3), directions=torch.ones(n, 3), pixel_area=torch.ones(n, 1), times=torch.rand(n, 1),
                   metadata={"sensor_idxs": sens})
    app = model._get_appearance_embedding(rb, torch.zeros(n, 32))
    assert torch.equal(app.detach(), emb.detach()[sens[:, 0]])
    g = torch.randn(n, cfg.appearance_dim)
    (app * g).sum().backward()
    want = torch.zeros_like(emb).index_add_(0, sens[:, 0], g)
    assert torch.allclose(emb.grad, want, rtol=1e-6, atol=1e-6)


@needs_reference
@pytest.mark.parametrize("name", nsb.PRESETS)
def test_plugin_built_from_each_preset_renders_like_the_reference(reference, name, monkeypatch):
    """The plugin's model built by the reference's own config system from each preset (small tables, every level and
    resolution kept): config_from_reference maps it, and its eval get_nff_outputs -- bound through B200Backend's
    load_params contract and rendered by the host emulation of the kernels -- matches the reference's torch walk on the
    same parameters.  Paper presets: the reference has no `_num_embeds_per_sensor`; num_sensors is the embedding's rows."""
    import os
    import sys
    import warnings
    from copy import deepcopy

    warnings.filterwarnings("ignore")
    from nerfstudio.configs.method_configs import method_configs
    from nerfstudio.data.scene_box import SceneBox
    from nerfstudio.field_components.field_heads import FieldHeadNames

    import nerfstudio.models.neurad as ref_neurad
    from neurad_studio_b200 import nerfstudio_api, scene
    from oracle.ref_driver import _install_nerfacc_restatements
    from tests.preset_fake_backend import PresetFakeBackend

    _install_nerfacc_restatements()
    ref_neurad.VGGPerceptualLossPix2Pix = lambda: torch.nn.Identity()
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    if root not in sys.path:
        sys.path.insert(0, root)
    from integration.neurad_b200_plugin import B200NeuRADModel, B200NeuRADModelConfig, config_from_reference

    ref_mc = deepcopy(method_configs[name].pipeline.model)
    fields = {k: v for k, v in vars(ref_mc).items() if k not in ("_target", "implementation", "eval_num_rays_per_chunk")}
    mc = B200NeuRADModelConfig(**fields)
    for f in mc.fields:
        f.grid.static.log2_hashmap_size, f.grid.actor.log2_hashmap_size = 11, 8
    n_actors, n_sensors = 2, 5
    small = nsb.small_config(n_actors=n_actors, num_sensors=n_sensors)
    trajs = scene.make_trajectories(n_actors, small.duration, seed=3)
    metadata = {"duration": small.duration, "sensor_idx_to_name": {i: f"s{i}" for i in range(n_sensors)}, "trajectories": trajs}
    model = mc.setup(scene_box=SceneBox(aabb=torch.tensor([[-100.0, -100.0, -10.0], [100.0, 100.0, 30.0]])), num_train_data=1,
                     metadata=metadata)
    assert isinstance(model, B200NeuRADModel)
    torch.manual_seed(3)
    with torch.no_grad():  # informative outputs: random tables, mostly-outside sdf
        for k, p in model.named_parameters():
            if k.endswith("hash_table"):
                p.uniform_(-1, 1)
        model.field.mlp_geo.layers[1].bias[0] = 0.5
        model.field.sdf_to_density.beta.fill_(4.0)
    model.eval()
    model._render_weights = (lambda self, outputs, ray_samples: __import__("nerfacc").render_weight_from_alpha(
        outputs[FieldHeadNames.ALPHA].squeeze(-1))[0]).__get__(model)

    cfg = config_from_reference(model)
    want = nsb.preset(name)[0]
    assert cfg.use_temporal_appearance == want.use_temporal_appearance
    assert cfg.num_sensors == n_sensors and cfg.num_appearance_embeds == model.appearance_embedding.num_embeddings
    if not want.use_temporal_appearance:
        assert not hasattr(model, "_num_embeds_per_sensor")
    for got_g, want_g in zip((cfg.grid, *cfg.proposal_grids), (want.grid, *want.proposal_grids)):
        assert (got_g.static.base_res, got_g.static.max_res) == (want_g.static.base_res, want_g.static.max_res)
        assert got_g.flip_prob == want_g.flip_prob

    be = PresetFakeBackend()
    monkeypatch.setattr(nerfstudio_api, "get_backend", lambda device: be)
    rays = scene.random_rays(32, small, seed=9, trajectories=trajs)

    def bundle():
        from nerfstudio.cameras.rays import RayBundle

        return RayBundle(origins=rays["origins"].clone(), directions=rays["directions"].clone(), pixel_area=rays["pixel_area"].clone(),
                         times=rays["times"].clone(), camera_indices=torch.zeros_like(rays["sensor_idx"]),
                         metadata={"is_lidar": rays["is_lidar"].clone().bool(), "sensor_idxs": rays["sensor_idx"].clone()})

    with torch.no_grad():
        ours = model.get_nff_outputs(bundle())
        ref = ref_neurad.NeuRADModel.get_nff_outputs(model, bundle())
    check_appearance_columns(ours["features"], ref["features"])
    for k in ("features", "depth", "accumulation", "prop_depth_0", "prop_depth_1"):
        err = (ours[k] - ref[k]).abs().max().item() / (ref[k].abs().max().item() + 1e-30)
        assert err < 1e-4, (k, err)
