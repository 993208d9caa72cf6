"""CPU, build container only (needs /root/reference): the reference-side plugin `integration/neurad_b200_plugin.py` run
against the REAL reference -- its plugin registry finds the method, its own config system builds the model, the model's
real `RayBundle` goes through the overridden `get_nff_outputs` / `decode_features` / `get_outputs_for_camera_ray_bundle`
(libb200nerf.so replaced by tests/fake_backend.py: oracle + host emulation, there is no GPU here), and the results are
compared with the reference's own torch path on the same model.  This proves attribute names, state-dict binding, side
effects on the bundle and dispatch -- the things a doc snippet cannot."""
import os
import sys
import warnings

import pytest
import torch

from oracle import ref_import

pytestmark = pytest.mark.skipif(not ref_import.reference_available(), reason="the reference tree exists in the build container only")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def rel_to_max(a, b):
    return (a - b).abs().max().item() / (b.abs().max().item() + 1e-30)


@pytest.fixture(scope="module")
def plugin():
    ref_import.install(full=True)
    warnings.filterwarnings("ignore")
    from oracle.ref_driver import _install_nerfacc_restatements

    _install_nerfacc_restatements()
    import nerfstudio.models.neurad as ref_neurad

    ref_neurad.VGGPerceptualLossPix2Pix = lambda: torch.nn.Identity()
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    os.environ["NERFSTUDIO_METHOD_CONFIGS"] = "neurad-b200=integration.neurad_b200_plugin:spec"
    from nerfstudio.plugins.registry import discover_methods

    methods, descriptions = discover_methods()
    return methods, descriptions


def _build_model(plugin, n_actors=3, seed=5):
    """The model as `ns-train neurad-b200` would build it (config.pipeline.model.setup), at test-sized hash tables."""
    from copy import deepcopy

    from nerfstudio.data.scene_box import SceneBox
    from nerfstudio.field_components.field_heads import FieldHeadNames

    import neurad_studio_b200 as nsb
    from neurad_studio_b200 import scene

    methods, _ = plugin
    mc = deepcopy(methods["neurad-b200"].pipeline.model)
    for f, (lm, lp) in zip(mc.fields, ((12, 9), (11, 8), (11, 8))):
        f.grid.static.log2_hashmap_size, f.grid.actor.log2_hashmap_size = lm, lp
    small = nsb.small_config(n_actors=n_actors)
    trajs = scene.make_trajectories(n_actors, small.duration, seed=seed)
    scene_box = SceneBox(aabb=torch.tensor([[-100.0, -100.0, -10.0], [100.0, 100.0, 30.0]]))
    metadata = {"duration": small.duration, "sensor_idx_to_name": {i: f"s{i}" for i in range(7)}, "trajectories": trajs}
    model = mc.setup(scene_box=scene_box, num_train_data=1, metadata=metadata)
    torch.manual_seed(seed)
    with torch.no_grad():  # the default 1e-3 table init renders a constant; make the outputs informative
        for k, p in model.named_parameters():
            if k.endswith("hash_table"):
                p.uniform_(-1, 1)
        model.field.mlp_geo.layers[1].bias[0] = 0.5
        model.field.sdf_to_density.beta.fill_(4.0)
    model.eval()

    def _render_weights(self, outputs, ray_samples):  # the reference's CUDA branch (neurad.py:716-717) on CPU tensors
        import nerfacc

        return nerfacc.render_weight_from_alpha(outputs[FieldHeadNames.ALPHA].squeeze(-1))[0]

    model._render_weights = _render_weights.__get__(model)
    return model, trajs, small


def _bundle(rays, sl=slice(None)):
    from nerfstudio.cameras.rays import RayBundle

    return RayBundle(origins=rays["origins"][sl].clone(), directions=rays["directions"][sl].clone(), pixel_area=rays["pixel_area"][sl].clone(),
                     times=rays["times"][sl].clone(), camera_indices=torch.zeros_like(rays["sensor_idx"][sl]),
                     metadata={"is_lidar": rays["is_lidar"][sl].clone().bool(), "sensor_idxs": rays["sensor_idx"][sl].clone()})


def test_registry_discovers_the_method(plugin):
    methods, descriptions = plugin
    from integration.neurad_b200_plugin import B200NeuRADModel, B200NeuRADModelConfig
    from nerfstudio.engine.trainer import TrainerConfig
    from nerfstudio.models.neurad import NeuRADModelConfig

    assert "neurad-b200" in methods and "H100" in descriptions["neurad-b200"]
    cfg = methods["neurad-b200"]
    assert isinstance(cfg, TrainerConfig) and cfg.method_name == "neurad-b200"
    mc = cfg.pipeline.model
    assert isinstance(mc, B200NeuRADModelConfig) and isinstance(mc, NeuRADModelConfig)
    assert mc._target is B200NeuRADModel and mc.implementation == "torch"
    # everything else is the reference's own "neurad" recipe
    from nerfstudio.configs.method_configs import method_configs

    assert set(cfg.optimizers) == set(method_configs["neurad"].optimizers)
    assert mc.sampling.num_proposal_samples == method_configs["neurad"].pipeline.model.sampling.num_proposal_samples


def test_plugin_model_renders_through_the_backend_like_the_reference(plugin, monkeypatch):
    from integration.neurad_b200_plugin import B200NeuRADModel
    from nerfstudio.models.neurad import NeuRADModel

    from neurad_studio_b200 import nerfstudio_api, scene
    from tests.fake_backend import FakeBackend

    model, trajs, small = _build_model(plugin)
    assert isinstance(model, B200NeuRADModel)
    be = FakeBackend()
    calls = []
    orig_render = be.render
    be.render = lambda *a, **k: (calls.append("render"), orig_render(*a, **k))[1]
    monkeypatch.setattr(nerfstudio_api, "get_backend", lambda device: be)
    rays = scene.random_rays(96, small, seed=9, trajectories=trajs)
    rb_ours, rb_ref = _bundle(rays), _bundle(rays)
    with torch.no_grad():
        ours = model.get_nff_outputs(rb_ours)
        ref = NeuRADModel.get_nff_outputs(model, rb_ref)  # the reference's own torch walk on the very same parameters
    assert calls == ["render"]
    assert set(ours) == set(ref) == {"features", "depth", "accumulation", "prop_depth_0", "prop_depth_1"}
    for k in ref:
        assert ours[k].shape == ref[k].shape and rel_to_max(ours[k], ref[k]) < 1e-4, (k, rel_to_max(ours[k], ref[k]))
    # same side effects on the caller's bundle (pixel areas scaled for camera rays, far clamp, nears)
    assert torch.equal(rb_ours.pixel_area, rb_ref.pixel_area) and torch.equal(rb_ours.fars, rb_ref.fars)
    assert torch.equal(rb_ours.nears, rb_ref.nears)
    # the binding follows the reference's parameters: an in-place update is picked up, untouched parameters are not re-bound
    loads = []
    orig_load = be.load_params
    be.load_params = lambda *a, **k: (loads.append(1), orig_load(*a, **k))[1]
    with torch.no_grad():
        model.get_nff_outputs(_bundle(rays))
        assert loads == []
        model.field.hashgrid.static_grid.hash_table.mul_(0.5)
        changed = model.get_nff_outputs(_bundle(rays))
        assert loads == [1] and rel_to_max(changed["features"], ref["features"]) > 1e-3
        ref2 = NeuRADModel.get_nff_outputs(model, _bundle(rays))
    assert rel_to_max(changed["features"], ref2["features"]) < 1e-4
    # training mode falls through to the reference's own walk (training extras present, backend not called)
    model.train()
    calls.clear()
    rb_train = _bundle(rays)
    rb_train.metadata["directions_norm"] = torch.full_like(rb_train.pixel_area, 40.0)  # lidar carving masks (neurad.py:677-700)
    rb_train.metadata["did_return"] = torch.ones_like(rb_train.pixel_area, dtype=torch.bool)
    out = model.get_nff_outputs(rb_train, calc_lidar_losses=False)
    assert "weights_list" in out and calls == []


def test_plugin_image_and_lidar_entry_points(plugin, monkeypatch):
    """get_outputs_for_camera_ray_bundle (neurad.py:623-675), the function the metric is defined on: one backend call per
    image / sweep, decoders on the library's operators, same output dict as the reference."""
    from nerfstudio.models.neurad import NeuRADModel

    from neurad_studio_b200 import nerfstudio_api, scene
    from tests.fake_backend import FakeBackend

    model, trajs, small = _build_model(plugin, n_actors=2, seed=7)
    be = FakeBackend()
    monkeypatch.setattr(nerfstudio_api, "get_backend", lambda device: be)
    rays = scene.random_rays(12 * 9 + 40, small, seed=11, trajectories=trajs)
    rays["is_lidar"][: 12 * 9] = 0
    rays["is_lidar"][12 * 9:] = 1
    cam = _bundle(rays, slice(0, 12 * 9)).reshape((12, 9))
    cam.metadata.pop("is_lidar")  # camera bundles of the eval path carry no is_lidar (cameras.py generate_rays)
    cam_ref = _bundle(rays, slice(0, 12 * 9)).reshape((12, 9))
    cam_ref.metadata.pop("is_lidar")
    ours = model.get_outputs_for_camera_ray_bundle(cam)
    ref = NeuRADModel.get_outputs_for_camera_ray_bundle(model, cam_ref)  # super()'s chunk loop calls the overridden parts too ...
    assert set(ours) == set(ref)
    # ... so compare against the pure reference: parent-class methods bound explicitly
    import types

    pure = types.SimpleNamespace()
    with torch.no_grad():
        sub = cam_ref[1::3, 1::3].reshape((-1,))
        nff = NeuRADModel.get_nff_outputs(model, sub)
        rgb, intensity, drop = NeuRADModel.decode_features(model, nff["features"], patch_size=(4, 3), is_lidar=None, intensity_for_cam=True)
    assert ours["rgb"].shape == (12, 9, 3) and rel_to_max(ours["rgb"], rgb.squeeze(0)) < 1e-4
    assert rel_to_max(ours["depth"].reshape(-1), nff["depth"].reshape(-1)) < 1e-4
    assert rel_to_max(ours["intensity"].reshape(-1), intensity.reshape(-1)) < 1e-4
    # lidar sweep: 1-D bundle
    lid = _bundle(rays, slice(12 * 9, None))
    out = model.get_outputs_for_camera_ray_bundle(lid)
    with torch.no_grad():
        nff = NeuRADModel.get_nff_outputs(model, _bundle(rays, slice(12 * 9, None)))
        _, intensity, drop = NeuRADModel.decode_features(model, nff["features"], patch_size=(1, 1),
                                                         is_lidar=torch.ones(40, 1, dtype=torch.bool), intensity_for_cam=True)
    assert out["depth"].shape == (40, 1) and rel_to_max(out["depth"], nff["depth"]) < 1e-4
    assert rel_to_max(out["intensity"], intensity) < 1e-4 and rel_to_max(out["ray_drop_logits"], drop) < 1e-4
