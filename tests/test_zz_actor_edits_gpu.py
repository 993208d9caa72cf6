"""GPU: actor edits (DynamicActors.actor_editing) through the C ABI, the fused kernels and the module walk.

- Every case of tests/golden/actor_edits.npz (the reference's own renders of edited scenes) is reproduced by the fused
  renderer in all four kernel variants and by the module walk, within the render goldens' tolerances, with bit-exact
  per-sample actor ids.
- Setting and clearing an edit leaves no trace: the next render is bit-identical to one that never saw an edit.
- Training mode ignores the edit; a backward through an edited forward raises; an index below -n_actors raises.
- A property that does not depend on the reference, in both parameter layouts: with time-constant actor rotations, a
  lateral / longitudinal edit renders what an unedited scene with keyframe positions shifted by R d renders.
"""
import pytest
import torch

from tests import actor_edit_cases as C

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.fixture(scope="module")
def backend():
    from neurad_studio_b200.backend import B200Backend

    return B200Backend(torch.device(DEV, 0))


def _render(be, rays, trace=True):
    out = be.render(rays, want_trace=C.TRACE if trace else False)
    be.check_status()
    return out


@pytest.mark.parametrize("mode", ["split", "lane", "tc", "ffma"])
@pytest.mark.parametrize("case", list(C.golden()[5]))
def test_fused_render_matches_reference(backend, case, mode):
    meta, cfg, params, rays, refs, edits, batches = C.golden()
    backend.load_params(cfg, params)
    backend.set_mlp_mode(mode)
    try:
        backend.set_actor_edit(**C.edit_args(edits[case]))
        out = _render(backend, rays[batches[case]])
    finally:
        backend.set_actor_edit()
        backend.set_mlp_mode("split")
    C.check_outputs(out, refs[case])


@pytest.mark.parametrize("case", list(C.golden()[5]))
def test_module_walk_matches_reference(case):
    from neurad_studio_b200.nerfstudio_api import NeuRADModel, RayBundle

    meta, cfg, params, rays, refs, edits, batches = C.golden()
    model = NeuRADModel(cfg)
    model.load_reference_state_dict(params)
    model = model.to(DEV).eval()
    model.dynamic_actors.actor_editing.update(edits[case])
    r = {k: v.to(DEV) for k, v in rays[batches[case]].items()}
    rb = RayBundle(origins=r["origins"], directions=r["directions"], pixel_area=r["pixel_area"], times=r["times"],
                   metadata={"is_lidar": r["is_lidar"], "sensor_idxs": r["sensor_idx"]})
    with torch.no_grad():
        out = model.get_nff_outputs(rb, fused=False)
        fused = model.get_nff_outputs(rb, fused=True)
    C.check_outputs(out, refs[case], ids=False)
    C.check_outputs(fused, refs[case], ids=False)
    model.dynamic_actors.actor_editing.update({k: (-1.0 if k == "index" else 0.0) for k in C.KEYS})
    model._bind()


def test_set_and_clear_leaves_renders_bit_identical(backend):
    meta, cfg, params, rays, refs, edits, batches = C.golden()
    backend.load_params(cfg, params)
    r = {k: v.to(DEV) for k, v in rays["mixed"].items()}
    before = _render(backend, r)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")  # stream-ordered: setting an edit and rendering with it wait for nothing
    try:
        backend.set_actor_edit(**C.edit_args(edits["shift_rotation"]))
        edited = backend.render(r, want_trace=C.TRACE)
        backend.set_actor_edit()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    after = _render(backend, r)
    backend.set_actor_edit(height=0.7)  # a height alone is no edit
    height_only = _render(backend, r)
    backend.set_actor_edit()
    assert not torch.equal(edited["features"], before["features"])
    for k in list(C.OUTPUTS) + list(C.TRACE):
        assert torch.equal(after[k], before[k]), k
        assert torch.equal(height_only[k], before[k]), k


def test_set_actors_clears_the_edit(backend):
    meta, cfg, params, rays, refs, edits, batches = C.golden()
    backend.load_params(cfg, params)
    before = _render(backend, rays["mixed"], trace=False)
    backend.set_actor_edit(lateral=2.0)
    backend.load_params(cfg, params)
    assert not backend.actor_edit_active
    after = _render(backend, rays["mixed"], trace=False)
    assert torch.equal(after["features"], before["features"])


def test_index_below_minus_n_actors_raises(backend):
    meta, cfg, params, rays, refs, edits, batches = C.golden()
    backend.load_params(cfg, params)
    with pytest.raises(ValueError):
        backend.set_actor_edit(lateral=1.0, index=-7)
    assert not backend.actor_edit_active
    backend.set_actor_edit(lateral=1.0, index=-6)  # wraps to actor 0
    assert backend.actor_edit_active
    backend.set_actor_edit()


def _mirror():
    from neurad_studio_b200.nerfstudio_api import NeuRADModel, RayBundle

    meta, cfg, params, rays, refs, edits, batches = C.golden()
    model = NeuRADModel(cfg)
    model.load_reference_state_dict(params)
    model = model.to(DEV)
    r = {k: v.to(DEV) for k, v in rays["mixed"].items()}
    rb = RayBundle(origins=r["origins"], directions=r["directions"], pixel_area=r["pixel_area"], times=r["times"],
                   metadata={"is_lidar": r["is_lidar"], "sensor_idxs": r["sensor_idx"]})
    return model, rb, edits


def test_training_mode_ignores_edits():
    model, rb, edits = _mirror()
    with torch.no_grad():
        ref = model.eval().get_nff_outputs(rb, fused=True)
        model.dynamic_actors.actor_editing.update(edits["shift_rotation"])
        edited = model.get_nff_outputs(rb, fused=True)
        train = model.train().get_nff_outputs(rb, fused=True)
    assert not torch.equal(edited["features"], ref["features"])
    for k in C.OUTPUTS:
        assert torch.equal(train[k], ref[k]), k


def test_backward_through_edited_forward_raises():
    model, rb, edits = _mirror()
    model.eval()
    model.dynamic_actors.actor_editing.update(edits["shift_rotation"])
    for n, k in model._names:
        if k.endswith("hash_table"):
            getattr(model, n).requires_grad_(True)
    out = model.get_nff_outputs(rb)  # grad mode: the module walk with the autograd operators
    with pytest.raises(RuntimeError, match="actor edit"):
        out["features"].sum().backward()
    # unedited, the same backward runs
    model.dynamic_actors.actor_editing.update(lateral=0.0, longitudinal=0.0, rotation=0.0, height=0.0, index=-1.0)
    model.get_nff_outputs(rb)["features"].sum().backward()


@pytest.mark.parametrize("layout", ["torch", "tcnn"])
@pytest.mark.parametrize("edit", [dict(lateral=1.3), dict(longitudinal=-2.1), dict(lateral=-0.7, longitudinal=1.6, index=3)])
def test_translation_edit_equals_shifted_keyframes(backend, layout, edit):
    cfg, params, rays = C.constant_rotation_scene(layout=layout)
    full = {"lateral": 0.0, "longitudinal": 0.0, "height": 0.0, "rotation": 0.0, "index": -1.0, **edit}
    backend.load_params(cfg, params)
    backend.set_actor_edit(**full)
    edited = _render(backend, rays)
    shifted = dict(params)
    shifted["dynamic_actors.actor_positions"] = C.shifted_positions(params, full["lateral"], full["longitudinal"], int(full["index"]))
    backend.load_params(cfg, shifted)
    moved = _render(backend, rays)
    hits = sum(int((moved[k] >= 0).sum()) for k in C.TRACE)
    assert hits > 1000, hits  # the rays do reach the moved actors
    # R d + lerp(t) and lerp(t + R d) differ in the last bits, which can move a sample lying on a box face across it:
    # such rays (at most 1 %) are left out of the value comparison
    same = torch.ones(rays["origins"].shape[0], dtype=torch.bool, device=DEV)
    for k in C.TRACE:
        same &= (edited[k] == moved[k]).all(-1)
    assert same.float().mean().item() >= 0.99, same.float().mean().item()
    for k in C.OUTPUTS:
        err = C.rel_to_max(edited[k][same], moved[k][same])
        assert err < 1e-5, (k, err)
