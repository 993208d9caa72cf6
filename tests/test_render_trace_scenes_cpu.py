"""CPU: the sample-by-sample render checks (tests/render_trace_cases.py) on the scenes beyond config 2 / 3 / opaque, over
the host emulation with small tables: zero-area lidar sweeps at unit and 0.1 table scale (the lidar-sweep golden's
scene), the reference's hash_init_scale, tiny activations with bias-free MLPs, an actor edit, and the neurad-paper and
neurader presets.  Then the comparator extensions these scenes need, each rejecting the matching corruption, and the
reference's own noise floor on the unit-scale sweep, which is what the sweep's depth tolerance rests on."""
import pytest
import torch

from tests import render_trace_cases as C

DEV = "cpu"
SCENES = ["sweep_unit", "sweep_tenth", "init_scale", "f16_small", "edits", "paper", "neurader"]


@pytest.mark.parametrize("name", SCENES)
def test_render_trace_scene_sample_by_sample(name):
    C.check_scene(DEV, name)


def _rejects(fn, what):
    try:
        fn()
    except AssertionError:
        return
    raise AssertionError(f"the comparator accepted {what}")


def _render(name):
    cfg, params, rays, _ = C.scene_rays(DEV, name)
    out = C.renderer(DEV, cfg, params, C.scene_edit(name)).render(rays)
    return cfg, params, rays, torch.arange(rays["origins"].shape[0]), out


# ------------------------------------------------------------------------------------------------ per-sensor appearance
def test_appearance_comparator_rejects_the_temporal_row():
    """neurad-paper: one appearance row per sensor, copied.  The row the temporal branch would read (sensor * eps + the
    keyframe before the time) is another row of the table for most rays, and must be rejected."""
    cfg, params, rays, idx, out = _render("paper")
    assert not cfg.use_temporal_appearance
    C.check_shading(out, out, rays, idx, cfg, params)
    emb = params["appearance_embedding.weight"]
    eps = cfg.embeds_per_sensor
    t, s = rays["times"].reshape(-1), rays["sensor_idx"].reshape(-1)
    before = torch.clamp(torch.floor(t / cfg.duration * eps), 0, eps - 1).long()
    row = (s * eps + before).clamp_max(emb.shape[0] - 1)
    assert (row != s).sum() > idx.numel() // 2
    bad = {k: v.clone() for k, v in out.items()}
    bad["features"][:, cfg.nff_out_dim:] = emb[row]
    _rejects(lambda: C.check_shading(bad, out, rays, idx, cfg, params), "the temporal appearance row of a per-sensor table")


# ------------------------------------------------------------------------------------------------ actor edits
@pytest.fixture(scope="module")
def edited():
    return _render("edits")


def _edited_actor_field(cfg, params, rays, idx, out, edit, corrupt=None):
    o, d, area, times = C._ray_inputs(rays, idx, cfg)
    e = C.main_edges(cfg, out["bins_e_2"])
    fr = C.ActorFrames(params, cfg, o, d, times, edit, corrupt)
    fs = C.FieldSamples(params, cfg, fr, o, d, area, times, e, out["actor_id_main"], cfg.grid.actor_scale)
    return C.main_field_reference(params, cfg, fs, d, DEV, C.gamma_ffma)


def test_edited_frames_reject_a_flipped_yaw_and_a_world_frame_shift(edited):
    """The edited actor's box-frame positions (ActorFrames under the edit, fp32 op by op as edit_box_pose) and the
    float64 box test (edit_boxes2world64) accept the edited render, and reject it under the yaw's sign flipped, the
    shift applied in the world frame, and no edit at all."""
    cfg, params, rays, idx, out = edited
    edit = C.scene_edit("edits")
    a = C.edit_selection(cfg.n_actors, edit)
    assert a == [1] and edit["rotation"] != 0.0
    on_edited = out["actor_id_main"] == a[0]
    assert int(on_edited.sum()) >= 10
    sdf, Es, feat, Ef = _edited_actor_field(cfg, params, rays, idx, out, edit)
    C._ratio(out["sdf"][on_edited], sdf[on_edited], Es[on_edited], "edited actor's sdf")
    C._ratio(out["field_feature"][on_edited], feat[on_edited], Ef[on_edited], "edited actor's features")
    C.check_actor_ids(out, rays, idx, cfg, params, edit=edit)
    flipped = dict(edit, rotation=-edit["rotation"])
    for what, ed, corrupt in (("the yaw's sign flipped", flipped, None), ("the shift in the world frame", edit, "world_shift"),
                              ("no edit", None, None)):
        _, _, bad, _ = _edited_actor_field(cfg, params, rays, idx, out, ed, corrupt)
        _rejects(lambda: C._ratio(out["field_feature"][on_edited], bad[on_edited], Ef[on_edited], "x"),
                 f"box-frame features with {what}")
        _rejects(lambda: C.check_actor_ids(out, rays, idx, cfg, params, edit=ed, corrupt=corrupt), f"actor ids with {what}")


def test_edit_cos_sin_are_rounded_once_from_double():
    c, s = C.edit_cos_sin({"rotation": 0.7})
    assert c == float(torch.tensor(0.7, dtype=torch.float64).cos().float())
    assert s == float(torch.tensor(0.7, dtype=torch.float64).sin().float())


# ------------------------------------------------------------------------------------------------ zero pixel area
def test_zero_area_gives_unit_level_weights_and_lidar_area_scale_is_checked():
    """A viewer-style sweep (pixel_area 0) has every level of every sample at weight exactly 1.  And the area scale is
    part of what the proposal comparator checks: config 2's lidar rays (pixel area > 0, area scale 1) rendered by the
    kernel are rejected against a reference that gives them the camera's area scale (rgb_upsample_factor^2)."""
    cfg, params, rays, idx, out = _render("sweep_unit")
    o, d, area, times = C._ray_inputs(rays, idx, cfg)
    assert (area == 0).all()
    e = C.main_edges(cfg, out["bins_e_2"])
    fs = C.FieldSamples(params, cfg, C._frames(params, cfg, o, d, times), o, d, area, times, e, out["actor_id_main"],
                        cfg.grid.actor_scale)
    lw, t = C.level_weights64(params["field.hashgrid.static_grid.scalings"], fs.cs64_s)
    assert lw.numel() > 0 and (lw == 1.0).all() and (t == 0).all()

    cfg, params, rays, idx, out = _render("config2")
    lid = rays["is_lidar"].reshape(-1)
    assert lid.any() and (rays["pixel_area"].reshape(-1)[lid] > 0).all()
    C.check_proposal_weights(out, rays, idx, cfg, params, DEV)
    as_camera = dict(rays, is_lidar=torch.zeros_like(rays["is_lidar"]))
    _rejects(lambda: C.check_proposal_weights(out, as_camera, idx, cfg, params, DEV), "lidar rays with the camera's area scale")


# ------------------------------------------------------------------------------------------------ the MLP constant
def test_check_scene_uses_the_mlp_constant_it_is_given():
    """check_scene bounds every MLP layer (K = 32 and 48 inputs) with the constant it is given (gamma_f16 by default on
    the GPU); gamma_f16 is tighter than the 3xTF32 constant the lane kernels were checked with before."""
    seen = []
    C.check_scene(DEV, "init_scale", gamma=lambda K: seen.append(K) or C.gamma_ffma(K))
    assert set(seen) == {32, 48}
    for K in (32, 48):
        assert C.gamma_ffma(K) < C.gamma_f16(K) < C.gamma_tc(K)


# ------------------------------------------------------------------------------------------------ the sweep's noise floor
def test_unit_scale_sweep_depth_gap_is_the_reference_floor():
    """The lidar-sweep golden's scene with its tables at the unit init (x10 of the golden's).  The reference's math with
    a correctly rounded exp() moves the depth by more (measured 3.6e-4 of its maximum) than the kernel's device code
    (the host emulation) is from the reference (measured 2.6e-4): the 2e-4 render tolerance is below the reference's
    own floor here, and SWEEP_UNIT_DEPTH_TOL is set above it.  At 0.1 of the unit init the floor is 2.8e-5."""
    from tests.host_emul import emul
    from oracle import neurad_oracle as O

    ref = C.sweep_oracle(1.0)
    floor = {k: C.rel_to_max(C.sweep_oracle(1.0, exact_exp=True)[k], ref[k]) for k in ("depth", "accumulation", "features")}
    cfg, params, rays = C.sweep_golden_scene(1.0)
    got = emul.render(cfg, params, rays, O.pdf_u, lane_mode=True)
    gap = {k: C.rel_to_max(got[k], ref[k]) for k in floor}
    tenth = C.rel_to_max(C.sweep_oracle(0.1, exact_exp=True)["depth"], C.sweep_oracle(0.1)["depth"])
    print(f"\n[sweep floor] unit tables: reference floor {floor}, emulated kernel vs reference {gap}; 0.1 tables: depth floor {tenth:.3g}")
    assert 2e-4 < floor["depth"] < C.SWEEP_UNIT_DEPTH_TOL
    assert gap["depth"] < floor["depth"]
    assert gap["accumulation"] < 1e-4 and gap["features"] < 1e-4
    assert tenth < 1e-4
