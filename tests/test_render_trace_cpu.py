"""CPU: the sample-by-sample checks of the ray-per-lane render (tests/render_trace_cases.py) on the host emulation of the
same device code (render_ray_lane with the CUDA-core MlpLaneFfma), small tables; and the comparator self-tests: every
comparator must reject a corrupted copy of a correct result, including corruptions far below 2e-3 of a tensor's max."""
import pytest
import torch

from tests import render_trace_cases as C

DEV = "cpu"


@pytest.mark.parametrize("name", ["config2", "config3", "opaque"])
def test_render_trace_sample_by_sample(name):
    worst, exits, faces, _, _ = C.check_scene(DEV, name)
    if name == "opaque":
        assert exits > 0, "the opaque scene has no warp whose proposal transmittance certainly underflows"


# ------------------------------------------------------------------------------------------------ comparator self-tests
def _rejects(fn, what):
    try:
        fn()
    except AssertionError:
        return
    raise AssertionError(f"the comparator accepted {what}")


@pytest.fixture(scope="module")
def rendered():
    cfg, params, rays, _ = C.scene_rays(DEV, "config2")
    out = C.renderer(DEV, cfg, params).render(rays)
    idx = torch.arange(rays["origins"].shape[0])
    return cfg, params, rays, idx, out


def test_comparators_accept_the_kernel(rendered):
    cfg, params, rays, idx, out = rendered
    C.check_walk(out, rays, idx, cfg)
    C.check_shading(out, out, rays, idx, cfg, params)


def test_feature_comparator_rejects_misplaced_rows(rendered):
    cfg, params, rays, idx, out = rendered
    n = idx.numel()
    for what, src, dst in (("two rows swapped inside one m64 half", (3, 40), (40, 3)),
                           ("a neighbouring ray's row in the ragged group", (n - 2,), (n - 1,))):
        bad = {k: v.clone() for k, v in out.items()}
        bad["features"][list(dst)] = out["features"][list(src)]
        _rejects(lambda: C.check_shading(bad, out, rays, idx, cfg, params), what)


def test_weight_comparators_reject_small_corruptions(rendered):
    cfg, params, rays, idx, out = rendered
    bad = {k: v.clone() for k, v in out.items()}
    bad["weights"][5, -1] = out["alpha"][5, -1] * torch.prod(1 - out["alpha"][5, :-1].double()).float()  # no top-up
    _rejects(lambda: C.check_shading(out, bad, rays, idx, cfg, params), "the sky sample without its top-up")
    for k in ("depth", "accumulation", "prop_depth_1"):
        bad = {kk: v.clone() for kk, v in out.items()}
        bad[k].view(torch.int32)[7] += 1  # one ulp
        _rejects(lambda: C.check_shading(bad, out, rays, idx, cfg, params), f"a one-ulp change of {k}")
    bad = {k: v.clone() for k, v in out.items()}
    bad["features"].view(torch.int32)[9, cfg.nff_out_dim + 3] += 1
    _rejects(lambda: C.check_shading(bad, out, rays, idx, cfg, params), "a one-ulp change of an appearance column")
    bad = {k: v.clone() for k, v in out.items()}
    bad["alpha"][11, 4] *= 1 + 1e-5
    _rejects(lambda: C.check_shading(out, bad, rays, idx, cfg, params), "alpha 1e-5 off at one sample")


def test_walk_comparator_rejects_an_index_off_by_one(rendered):
    cfg, params, rays, idx, out = rendered
    for k in ("inds_1", "inds_2"):
        bad = {kk: v.clone() for kk, v in out.items()}
        bad[k][4, 10] += 1
        _rejects(lambda: C.check_walk(bad, rays, idx, cfg), f"{k} off by one")
    bad = {kk: v.clone() for kk, v in out.items()}
    bad["bins_e_2"].view(torch.int32)[2, 5] += 1
    _rejects(lambda: C.check_walk(bad, rays, idx, cfg), "a one-ulp change of bins_e_2")


def test_proposal_comparator_rejects_a_dropped_grid_level(rendered):
    """One grid level of the proposal density left out at one sample: the weights of that ray change by far less than
    2e-3 of their max, and the comparator must still see it."""
    cfg, params, rays, idx, out = rendered
    C.check_proposal_weights(out, rays, idx, cfg, params, DEV)
    r = torch.tensor([6])
    o, d, area, times = C._ray_inputs(rays, r, cfg)
    e = out["bins_e_1"][r].float()
    aid = torch.full((1, e.shape[1] - 1), -1)
    fs = C.FieldSamples(params, cfg, None, o, d, area, times, e, aid, cfg.proposal_grid_2.actor_scale)
    dens, rel = C.proposal_density_reference(params, cfg, fs, DEV)
    good_w, tol, _ = C.proposal_weights_reference(dens, rel, e)
    s = int((good_w[0] > 1e-3 * good_w.max()).nonzero()[-1])  # a late sample: the change does not reach the others
    dens_b, _ = C.proposal_density_reference(params, cfg, fs, DEV, drop=(s, 5))
    bad_w, _, _ = C.proposal_weights_reference(dens_b, rel, e)
    assert (bad_w - good_w).abs().max() < 2e-3 * good_w.abs().max()
    C._ratio(good_w.float(), good_w, tol, "fp32 rounding of the reference")
    _rejects(lambda: C._ratio(bad_w.float(), good_w, tol, "x"), "a proposal density with one grid level dropped")


@pytest.fixture(scope="module")
def actors_rendered():
    cfg, params, rays, _ = C.scene_rays(DEV, "config3")
    out = C.renderer(DEV, cfg, params).render(rays)
    return cfg, params, rays, torch.arange(rays["origins"].shape[0]), out


def _main_field(cfg, params, rays, idx, out, corrupt, gamma):
    o, d, area, times = C._ray_inputs(rays, idx, cfg)
    e = C.main_edges(cfg, out["bins_e_2"])
    fs = C.FieldSamples(params, cfg, C._frames(params, cfg, o, d, times), o, d, area, times, e, out["actor_id_main"],
                        cfg.grid.actor_scale)
    return C.main_field_reference(params, cfg, fs, d, DEV, gamma, corrupt=corrupt)


@pytest.mark.parametrize("gamma", [C.gamma_ffma, C.gamma_tc], ids=["ffma", "tc"])
def test_main_field_comparator_rejects_corrupted_mlp_and_padding(actors_rendered, gamma):
    """The main-field comparator under both bounds: it accepts the fp32 rounding of its own reference and rejects actor
    samples whose features are not zero-padded; under the FFMA bound it also rejects features whose last layer ran as
    1xTF32 (3xTF32 without its correction), a change far below 2e-3 of the features' max."""
    cfg, params, rays, idx, out = actors_rendered
    sdf, Es, feat, Ef = _main_field(cfg, params, rays, idx, out, None, gamma)
    C._ratio(feat.float(), feat, Ef, "fp32 rounding of the reference")
    C._ratio(sdf.float(), sdf, Es, "fp32 rounding of the reference")
    _, _, bad, _ = _main_field(cfg, params, rays, idx, out, "tf32", gamma)
    assert (bad - feat).abs().max() < 2e-3 * feat.abs().max()
    if gamma is C.gamma_ffma:
        _rejects(lambda: C._ratio(bad.float(), feat, Ef, "x"), "features from a layer without the 3xTF32 correction")
    else:  # the worst-case wgmma constant (truncating accumulation allowed) is too wide to separate one 1xTF32 layer
        print(f"\n[render trace] 1xTF32 last layer under the 3xTF32 bound: ratio {((bad - feat).abs() / Ef).max().item():.3g}")
    bsdf, _, bad, _ = _main_field(cfg, params, rays, idx, out, "unpadded", gamma)
    act = out["actor_id_main"] >= 0
    assert act.any()
    _rejects(lambda: C._ratio(bad.float()[act], feat[act], Ef[act], "x"), "actor samples with unpadded features")


def test_actor_id_comparator_rejects_a_wrong_actor(actors_rendered):
    cfg, params, rays, idx, out = actors_rendered
    C.check_actor_ids(out, rays, idx, cfg, params)
    bad = {k: v.clone() for k, v in out.items()}
    r, s = (out["actor_id_main"] >= 0).nonzero()[0].tolist()
    bad["actor_id_main"][r, s] = -1
    _rejects(lambda: C.check_actor_ids(bad, rays, idx, cfg, params), "an actor sample assigned to the static field")
