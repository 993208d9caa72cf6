"""TEST INFRASTRUCTURE ONLY -- golden vectors of the reference's other NeuRAD presets, from the REAL reference.

Run in the build container (needs the reference checkout):   python -m oracle.make_golden_presets

For each case it builds the unmodified reference ``NeuRADModel`` from ``deepcopy(method_configs[name]).pipeline.model``
(``implementation="torch"``, CPU, hash tables shrunk as ``small_config`` does, every level and resolution kept), runs
``get_nff_outputs`` on seeded synthetic inputs, asserts that oracle/presets_oracle.py reproduces every captured tensor
bit for bit, and writes the same groups as oracle/make_golden.py:
  nff_paper.npz      neurad-paper: one appearance row per sensor (7 sensors, distinct rows), 6 actors, times over the
                     whole duration, a quarter lidar rays (intensity / ray-drop read the appearance columns)
  nff_neurader.npz   neurader: the doubled resolutions (main static levels 64 ... 16383), temporal appearance
  grads_paper.npz    gradients of the neurad-paper case, appearance_embedding.weight included: the reference's autograd
                     of oracle/make_golden_grads.py's seeded loss on its first 96 rays (eval-mode sampling), checked
                     against autograd through the oracle before it is written
"""
from __future__ import annotations

import os
import sys
import warnings
from copy import deepcopy

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import neurad_studio_b200 as nsb  # noqa: E402
from neurad_studio_b200 import scene  # noqa: E402
from oracle import neurad_oracle as O  # noqa: E402
from oracle import presets_oracle as PO  # noqa: E402
from oracle import ref_driver  # noqa: E402
from oracle.make_golden import _save  # noqa: E402

LOG2_MAIN, LOG2_PROP = 10, 10


def build_preset_model(name, cfg, params, trajectories):
    """ref_driver.build_reference_model, but from the preset's own model config instead of a default one."""
    ref_driver.ref_import.install(full=True)
    ref_driver._install_nerfacc_restatements()
    warnings.filterwarnings("ignore")
    import nerfstudio.models.neurad as ref_neurad
    from nerfstudio.configs.method_configs import method_configs
    from nerfstudio.data.scene_box import SceneBox
    from nerfstudio.field_components.field_heads import FieldHeadNames

    ref_neurad.VGGPerceptualLossPix2Pix = lambda: torch.nn.Identity()
    mc = deepcopy(method_configs[name].pipeline.model)
    mc.implementation = "torch"
    for f, g in zip(mc.fields, (cfg.grid, *cfg.proposal_grids)):  # shrink the tables only
        assert (f.grid.static.base_res, f.grid.static.max_res) == (g.static.base_res, g.static.max_res)
        f.grid.static.log2_hashmap_size = g.static.log2_hashmap_size
        f.grid.actor.log2_hashmap_size = g.actor.log2_hashmap_size
    s = float(cfg.static_scale)
    metadata = {"duration": cfg.duration, "sensor_idx_to_name": {i: f"sensor{i}" for i in range(cfg.num_sensors)},
                "trajectories": trajectories if trajectories is not None else []}
    model = ref_neurad.NeuRADModel(mc, scene_box=SceneBox(aabb=torch.tensor([[-s, -s, -10.0], [s, s, 30.0]])),
                                   num_train_data=1, metadata=metadata)
    res = model.load_state_dict({k: v for k, v in params.items() if k != "static_scale"}, strict=False)
    assert not res.unexpected_keys, res.unexpected_keys
    missing = [k for k in res.missing_keys if k.split(".")[0] in ("field", "proposal_fields", "lidar_decoder", "appearance_embedding")
               and ".hashgrid.actors." not in k and not k.endswith("beta_min")]
    assert not missing, missing
    model.eval()

    def _render_weights(self, outputs, ray_samples):  # neurad.py:716-717 (the non-CPU branch), as ref_driver does
        import nerfacc

        weights, _ = nerfacc.render_weight_from_alpha(outputs[FieldHeadNames.ALPHA].squeeze(-1))
        return weights

    model._render_weights = _render_weights.__get__(model)
    return model


def preset_case(file_name, preset, n_actors, n_rays, seed, beta, sdf_bias):
    torch.manual_seed(0)
    cfg = PO.shrink_tables(nsb.preset(preset)[0], LOG2_MAIN, LOG2_PROP)
    cfg.n_actors = n_actors
    trajs = scene.make_trajectories(n_actors, cfg.duration, seed=seed) if n_actors else None
    params = scene.make_params(cfg, seed=seed, beta=beta, trajectories=trajs, sdf_bias=sdf_bias)
    rays = scene.random_rays(n_rays, cfg, seed=seed + 1, trajectories=trajs)
    model = build_preset_model(preset, cfg, params, trajs)
    assert model.appearance_embedding.num_embeddings == cfg.num_appearance_embeds
    ref = ref_driver.run_reference_nff(model, rays)
    with torch.no_grad():
        out = PO.nff_outputs(params, cfg, rays["origins"], rays["directions"], rays["pixel_area"], rays["times"],
                             rays["sensor_idx"], rays["is_lidar"], want_trace=True)
        inten, drop = O.decode_lidar(params, out["features"])
    tr = out.pop("trace")
    allo = {**out, **tr, "intensity": inten, "ray_drop_logits": drop}
    n_cmp = 0
    for k, v in ref.items():
        if k in allo:
            assert torch.equal(v.float(), allo[k].float()), f"oracle != reference for {k}"
            n_cmp += 1
    n_sensors = int(rays["sensor_idx"].unique().numel())
    print(f"{file_name}: oracle == reference bit-for-bit on {n_cmp} tensors; sensors = {n_sensors}; "
          f"actor hits (main) = {int((tr['actor_id_main'] >= 0).sum())}")
    for k in ("inds_1", "inds_2", "cdf_1", "cdf_2", "actor_id_main", "actor_id_0", "actor_id_1", "density_0", "density_1"):
        ref[k] = tr[k]
    arrays = {f"param/{k}": v for k, v in params.items()}
    arrays.update({f"ray/{k}": v for k, v in rays.items()})
    arrays.update({f"ref/{k}": v for k, v in ref.items()})
    meta = dict(preset=preset, n_actors=n_actors, log2_main=LOG2_MAIN, log2_prop=LOG2_PROP, seed=seed, beta=beta,
                sdf_bias=sdf_bias, static_scale=cfg.static_scale, duration=cfg.duration, num_sensors=cfg.num_sensors,
                torch=torch.__version__)
    _save(file_name, arrays, meta)


def grads_case(case_name, file_name):
    """oracle/make_golden_grads.py's grads_case for a preset golden."""
    from oracle import make_golden_grads as MG
    from tests.preset_cases import cfg_from_preset_meta

    meta, params, rays = MG.load_case(case_name)
    cfg = cfg_from_preset_meta(meta)
    trajs = scene.make_trajectories(meta["n_actors"], cfg.duration, seed=meta["seed"]) if meta["n_actors"] else None
    model = build_preset_model(meta["preset"], cfg, params, trajs)
    from nerfstudio.cameras.rays import RayBundle

    named = dict(model.named_parameters())
    keys = [k for k in MG.trainable_keys(params) if k in named]
    for k in keys:
        named[k].requires_grad_(True)
    n = rays["origins"].shape[0]
    rb = RayBundle(origins=rays["origins"].clone(), directions=rays["directions"].clone(), pixel_area=rays["pixel_area"].clone(),
                   fars=torch.full((n, 1), 1_000_000.0), times=rays["times"].clone(),
                   metadata={"is_lidar": rays["is_lidar"].clone(), "sensor_idxs": rays["sensor_idx"].clone()})
    out = model.get_nff_outputs(rb)
    G = MG.loss_weights({k: out[k].shape for k in MG.OUT_KEYS})
    sum((out[k] * G[k]).sum() for k in MG.OUT_KEYS).backward()
    ref = {k: named[k].grad.detach().clone() for k in keys if named[k].grad is not None}
    assert ref["appearance_embedding.weight"].abs().max() > 0
    # autograd through the oracle (the per-sensor branch included)
    p = {k: v.clone() for k, v in params.items()}
    for k in keys:
        p[k].requires_grad_(True)
    o = PO.nff_outputs(p, cfg, rays["origins"], rays["directions"], rays["pixel_area"], rays["times"], rays["sensor_idx"],
                       rays["is_lidar"])
    for k in MG.OUT_KEYS:
        assert torch.equal(out[k].detach(), o[k].detach()), f"oracle forward != reference for {k}"
    sum((o[k] * G[k]).sum() for k in MG.OUT_KEYS).backward()
    ora = {k: p[k].grad for k in keys if p[k].grad is not None}
    assert set(ref) == set(ora), sorted(set(ref) ^ set(ora))
    worst = 0.0
    for k in ref:
        scale = ref[k].abs().max().item()
        if scale == 0:
            assert ora[k].abs().max().item() == 0, k
            continue
        err = (ref[k] - ora[k]).abs().max().item() / scale
        worst = max(worst, err)
        assert err < 1e-5, (k, err)
    print(f"{file_name}: reference autograd == oracle autograd on {len(ref)} parameters (worst rel. diff {worst:.1e})")
    arrays = {f"grad/{k}": v for k, v in ref.items()}
    _save(file_name, arrays, dict(case=case_name, n_rays=MG.N_RAYS, loss_seed=7, loss_scale=MG.LOSS_SCALE, torch=torch.__version__))


def main():
    preset_case("nff_paper.npz", "neurad-paper", n_actors=6, n_rays=96, seed=41, beta=4.0, sdf_bias=0.5)
    preset_case("nff_neurader.npz", "neurader", n_actors=6, n_rays=96, seed=43, beta=4.0, sdf_bias=0.5)
    grads_case("nff_paper.npz", "grads_paper.npz")


if __name__ == "__main__":
    main()
