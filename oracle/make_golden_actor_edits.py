"""TEST INFRASTRUCTURE ONLY -- tests/golden/actor_edits.npz from the REAL reference: renders of edited scenes.

Run in the build container (needs /root/reference):   python -m oracle.make_golden_actor_edits

The unmodified reference ``NeuRADModel`` (implementation="torch", CPU, eval mode, built by oracle/ref_driver.py like
make_golden.py's actor case) renders one ray batch under each actor edit of CASES, set through its own
``dynamic_actors.actor_editing`` dict (model_components/dynamic_actors.py:53-59, 181-249).  For every case the script
asserts that the oracle (oracle/actor_edit_oracle.py) reproduces the reference's outputs bit for bit, then
stores the outputs, the oracle's per-sample actor ids and the reference's own edited boxes2world at the ray times.

The scene is make_golden.py's six-actor scene with actor 1 moved beside actor 0 (3 m apart, parallel): unedited their
padded boxes are disjoint, rotated by 90 degrees they overlap.  Besides the random batch the rays hold
  * "onto" rays aimed 4.5 m to the side of actors 2 and 3, at their laterally edited centres, kept only where the
    reference's unedited render has no actor sample and the unedited centre lies outside the ray-line cull radius;
  * "overlap" rays aimed between actors 0 and 1, inside both boxes once they are rotated.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import neurad_studio_b200 as nsb  # noqa: E402
from neurad_studio_b200 import scene  # noqa: E402
from oracle import actor_edit_oracle as AE  # noqa: E402
from oracle import ref_driver  # noqa: E402
from oracle.convert import to_oracle_cfg  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "actor_edits.npz")
N_ACTORS, SEED = 6, 5
ONTO_SHIFT = 4.5  # lateral shift of the "onto" case (box frame x, metres)
OUTPUTS = ("features", "depth", "accumulation", "prop_depth_0", "prop_depth_1")
TRACE = ("actor_id_0", "actor_id_1", "actor_id_main")
NO_EDIT = {"lateral": 0.0, "longitudinal": 0.0, "rotation": 0.0, "index": -1.0, "height": 0.0}

# name -> (edit, rays) ; rays "mixed" = the camera + lidar batch, "lidar" = the same rays as one lidar batch
CASES = {
    "none": ({}, "mixed"),
    "lateral": ({"lateral": 1.5}, "mixed"),
    "longitudinal": ({"longitudinal": -2.0}, "mixed"),
    "rotation": ({"rotation": 0.6}, "mixed"),
    "shift_rotation": ({"lateral": -1.0, "longitudinal": 1.5, "height": 0.3, "rotation": -0.4}, "mixed"),
    "index": ({"lateral": 1.2, "rotation": 0.3, "index": 2.0}, "mixed"),
    "index_float": ({"longitudinal": 1.8, "index": 3.7}, "mixed"),            # truncates to 3
    "index_clamped": ({"lateral": -1.3, "index": 9.0}, "mixed"),              # min(9, 5) = 5
    "index_negative": ({"lateral": 1.1, "rotation": -0.5, "index": -2.0}, "mixed"),   # actor 4
    "index_negative_float": ({"longitudinal": -1.4, "index": -1.5}, "mixed"),  # truncates to -1: actor 5 only
    "height_only": ({"height": 0.7}, "mixed"),                                 # ignored: equals "none"
    "height_lateral": ({"height": 0.5, "lateral": 0.8}, "mixed"),             # the height is applied
    "onto": ({"lateral": ONTO_SHIFT}, "mixed"),
    "overlap": ({"rotation": float(np.pi / 2)}, "mixed"),
    "lidar": ({"lateral": -1.0, "longitudinal": 1.5, "height": 0.3, "rotation": -0.4}, "lidar"),
}


def make_scene():
    cfg = nsb.small_config(n_actors=N_ACTORS, log2_main=10, log2_prop=10)
    trajs = scene.make_trajectories(N_ACTORS, cfg.duration, seed=SEED)
    # actor 1 beside actor 0: same heading, speed and x, 3 m further along world y (padded half widths 1.25 m)
    trajs[1]["poses"] = trajs[0]["poses"].clone()
    trajs[1]["poses"][:, 1, 3] += 3.0
    params = scene.make_params(cfg, seed=SEED, table_scale=1.0, beta=4.0, trajectories=trajs, sdf_bias=0.5)
    return cfg, trajs, params


def aimed_rays(base, targets, times):
    n = targets.shape[0]
    o = base["origins"][:n].clone()
    d = targets - o
    d = d / d.norm(dim=-1, keepdim=True)
    return {"origins": o, "directions": d, "pixel_area": torch.full((n, 1), 1.0e-6), "times": times[:, None].clone(),
            "sensor_idx": torch.zeros(n, 1, dtype=torch.long), "is_lidar": torch.zeros(n, 1, dtype=torch.bool)}


def cat_rays(*rs):
    return {k: torch.cat([r[k] for r in rs]) for k in rs[0]}


def oracle_render(params, cfg, rays, edit):
    with torch.no_grad():
        out = AE.nff_outputs(params, to_oracle_cfg(cfg), rays["origins"], rays["directions"], rays["pixel_area"], rays["times"],
                             rays["sensor_idx"], rays["is_lidar"], want_trace=True, edit=edit or None)
    tr = out.pop("trace")
    return out, tr


def main():
    torch.manual_seed(0)
    cfg, trajs, params = make_scene()
    model = ref_driver.build_reference_model(cfg, params, trajs)
    da = model.dynamic_actors
    base = scene.random_rays(64, cfg, seed=SEED + 1, trajectories=trajs)
    gen = torch.Generator().manual_seed(SEED + 77)

    def b2w_at(times):  # the reference's own (edited) box poses at the ray times
        with torch.no_grad():
            return da.get_boxes2world(times.reshape(-1), flatten=False)[0][..., :3, :].clone()

    # "onto": targets ONTO_SHIFT to the side (box x) of actors 2 and 3 at the ray's time
    da.actor_editing.update(NO_EDIT)
    cand_t = torch.rand(64, generator=gen) * (cfg.duration - 0.5)
    b2w0 = b2w_at(cand_t)
    pick = torch.tensor([2, 3] * 32)
    shift = torch.tensor([ONTO_SHIFT, 0.0, 0.0])
    centre = b2w0[torch.arange(64), pick, :, 3]
    target = centre + b2w0[torch.arange(64), pick, :, :3] @ shift + (torch.rand(64, 3, generator=gen) - 0.5) * torch.tensor([0.6, 1.5, 0.6])
    onto = aimed_rays(cat_rays(base, base), target, cand_t)
    bounds = params["dynamic_actors.actor_sizes"] / 2 + params["dynamic_actors.actor_padding"]
    radius = bounds.norm(dim=-1)
    v = centre - onto["origins"]
    dist = torch.linalg.norm(torch.cross(v, onto["directions"], dim=-1), dim=-1)
    out0, tr0 = oracle_render(params, cfg, onto, {})
    no_hit = (tr0["actor_id_main"] < 0).all(-1) & (tr0["actor_id_0"] < 0).all(-1) & (tr0["actor_id_1"] < 0).all(-1)
    keep = (no_hit & (dist > radius[pick] * 1.05)).nonzero().reshape(-1)[:16]
    assert keep.numel() >= 8, f"only {keep.numel()} 'onto' rays"
    onto = {k: t[keep] for k, t in onto.items()}

    # "overlap": between actors 0 and 1 (1.5 m from each centre across their width)
    ov_t = torch.rand(16, generator=gen) * (cfg.duration - 0.5)
    b2w0 = b2w_at(ov_t)
    mid = 0.5 * (b2w0[:, 0, :, 3] + b2w0[:, 1, :, 3]) + (torch.rand(16, 3, generator=gen) - 0.5) * torch.tensor([0.8, 0.4, 0.4])
    overlap = aimed_rays(base, mid, ov_t)

    mixed = cat_rays(base, onto, overlap)
    n_onto0, n_ov0 = base["origins"].shape[0], base["origins"].shape[0] + onto["origins"].shape[0]
    lidar = dict(mixed)
    n = mixed["origins"].shape[0]
    lidar["is_lidar"] = torch.ones(n, 1, dtype=torch.bool)
    lidar["sensor_idx"] = torch.full((n, 1), cfg.num_sensors - 1, dtype=torch.long)
    lidar["pixel_area"] = torch.full((n, 1), 3.0e-3 * 1.5e-3)
    batches = {"mixed": mixed, "lidar": lidar}

    arrays = {f"param/{k}": v for k, v in params.items()}
    for b, r in batches.items():
        arrays.update({f"ray_{b}/{k}": v for k, v in r.items()})
    hits = {}
    for name, (edit, which) in CASES.items():
        rays = batches[which]
        da.actor_editing.update({**NO_EDIT, **edit})
        ref = ref_driver.run_reference_nff(model, rays)
        b2w = b2w_at(rays["times"])
        out, tr = oracle_render(params, cfg, rays, edit)
        for k in OUTPUTS:
            assert torch.equal(ref[k], out[k]), f"{name}: oracle != reference for {k}"
        for k in OUTPUTS:
            arrays[f"{name}/{k}"] = ref[k]
        for k in TRACE:
            arrays[f"{name}/{k}"] = tr[k].to(torch.int32)
        arrays[f"{name}/boxes2world"] = b2w
        hits[name] = torch.cat([tr[k] for k in TRACE], dim=-1)  # actor ids of all three sampling rounds
        print(f"{name:22s} oracle == reference bit for bit; main-field actor samples = {int((tr['actor_id_main'] >= 0).sum())}")
    # training mode: get_boxes2world ignores the edit
    da.actor_editing.update({**NO_EDIT, **CASES["shift_rotation"][0]})
    da.train()
    arrays["train/boxes2world"] = b2w_at(mixed["times"])
    da.eval()
    da.actor_editing.update(NO_EDIT)
    assert torch.equal(arrays["train/boxes2world"], arrays["none/boxes2world"])

    # the cases do what their names say
    assert torch.equal(arrays["height_only/features"], arrays["none/features"])
    assert not torch.equal(arrays["height_lateral/boxes2world"], arrays["lateral/boxes2world"])
    on = hits["onto"][n_onto0:n_ov0]
    assert (hits["none"][n_onto0:n_ov0] < 0).all() and (on >= 0).any(-1).float().mean() >= 0.5, "'onto' rays"
    ov = hits["overlap"][n_ov0:]
    assert (ov == 1).any(), "'overlap' rays"
    print(f"onto: {int((on >= 0).any(-1).sum())} of {on.shape[0]} rays reach an edited box; overlap: "
          f"{int((ov == 1).sum())} samples in actor 1 (the higher index of the overlap)")
    e = arrays["index_negative_float/boxes2world"] != arrays["none/boxes2world"]
    assert e[:, 5].any() and not e[:, :5].any(), "index -1.5 edits the last actor only"

    out = {k: (v.detach().cpu().numpy() if isinstance(v, torch.Tensor) else np.asarray(v)) for k, v in arrays.items()}
    meta = dict(n_actors=N_ACTORS, log2_main=10, log2_prop=10, seed=SEED, beta=4.0, sdf_bias=0.5, table_scale=1.0,
                static_scale=cfg.static_scale, duration=cfg.duration, num_sensors=cfg.num_sensors,
                cases={k: {**NO_EDIT, **v[0]} for k, v in CASES.items()}, batches={k: v[1] for k, v in CASES.items()},
                onto_rays=[n_onto0, n_ov0], overlap_rays=[n_ov0, n], torch=torch.__version__)
    out["__meta__"] = np.array(repr(meta))
    np.savez_compressed(GOLDEN, **out)
    print(f"wrote {GOLDEN}: {os.path.getsize(GOLDEN) / 1e6:.2f} MB, {n} rays, {len(CASES)} cases")


if __name__ == "__main__":
    main()
