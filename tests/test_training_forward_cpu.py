"""CPU: the entry-by-entry checks of the training step's forward operators (tests/training_forward_cases.py).
neurad_encoding and isotropic_gaussian run the device code here through the host emulation (tests/fake_backend.py), so
those tests check the kernels' code.  spaced_sample_stratified, spacing_to_euclidean, pdf_resample_stratified,
_field_mid / _field_tail and the MLPs have torch or oracle stand-ins in the fake backend: on the CPU those tests check
the references and the bounds, not the kernels; the kernels themselves are checked on the GPU
(test_zz_training_forward_gpu.py).  The comparator self-tests below check that every comparator rejects a corrupted copy
of a correct result."""
import pytest
import torch

from neurad_studio_b200.lib import FIELD_MAIN, FIELD_PROP1
from tests import training_forward_cases as C

DEV = "cpu"


def _report(name, worst):
    print(f"\n[training forward] {name}: worst |got - ref| / tol = {worst:.3g}")


@pytest.mark.parametrize("n,S", [(1, 1), (7, 33)])
def test_gaussian_per_entry(n, S):
    _report(f"gaussian n={n} S={S}", C.gaussian_case(DEV, n, S, seed=S))


@pytest.mark.parametrize("kind,lam", [("uniform", -1.0), ("lindisp", -1.0), ("sqrt", -1.0), ("log", -1.0), ("power", -1.0),
                                      ("power", -1.5)])
@pytest.mark.parametrize("with_nears", [True, False])
@pytest.mark.parametrize("rand_cols", ["single", "edges"])
def test_stratified_per_entry(kind, lam, with_nears, rand_cols):
    _report(f"stratified {kind} {lam} nears={with_nears} {rand_cols}",
            C.stratified_case(DEV, 9, 32, kind, lam, with_nears, rand_cols, "random"))


@pytest.mark.parametrize("t_kind", ["zero", "max"])
@pytest.mark.parametrize("rand_cols", ["single", "edges"])
def test_stratified_jitter_extremes(rand_cols, t_kind):
    C.stratified_case(DEV, 5, 31, "power", -1.0, True, rand_cols, t_kind)


@pytest.mark.parametrize("S,S_new,cols", [(31, 32, 1), (33, 64, "edges"), (64, 32, 1)])
@pytest.mark.parametrize("kind", ["random", "degenerate", "unpadded"])
def test_pdf_per_entry(S, S_new, cols, kind):
    _report(f"pdf {kind} S={S}", C.pdf_case(DEV, 12, S, S_new, cols, kind, seed=S))


def test_pdf_dyadic_quantiles_on_cdf_values():
    C.pdf_case(DEV, 6, 32, 31, 1, "dyadic")


@pytest.mark.parametrize("n_actors,flip", [(0, "none"), (6, "mixed"), (6, "minus"), (64, "plus")])
@pytest.mark.parametrize("field", [FIELD_MAIN, FIELD_PROP1])
def test_encoding_per_entry(field, n_actors, flip):
    worst, faces = C.encoding_case(DEV, field, n_actors, 24, 33, flip)
    _report(f"encoding field={field} actors={n_actors} flip={flip} ({faces} face exceptions)", worst)


def test_encoding_directions_per_sample():
    C.encoding_case(DEV, FIELD_MAIN, 6, 18, 5, "mixed", dirs_per_ray=False)


@pytest.mark.parametrize("n,G", [(1, 15), (129, 32)])
def test_field_mid_tail(n, G):
    _report(f"field n={n} G={G}", C.field_case(DEV, n, G))


@pytest.mark.parametrize("which", ["geo", "feature"])
def test_mlp_reference(which):
    C.mlp_case(DEV, which, 129)


def test_recorded_training_step():
    worst, faces, n = C.check_recorded_step(DEV, 48, 24)
    print(f"\n[training forward] recorded step ({n} calls, {faces} face exceptions): "
          + ", ".join(f"{k} {v:.3g}" for k, v in sorted(worst.items())))


# ------------------------------------------------------------------------------------------------ comparator self-tests
def _rejects(fn, what):
    try:
        fn()
    except AssertionError:
        return
    raise AssertionError(f"the comparator accepted {what}")


def _encoding_fixture(field=FIELD_MAIN, n_actors=6, flip="minus"):
    cfg, params = C.encoding_scene(DEV, n_actors)
    be = C.backend(DEV, cfg, params)
    mean, std, times, dirs = C.encoding_samples(cfg, params, 24, 9, 0)
    fl = C.flips(24, flip)
    out = be.neurad_encoding(field, mean, std, times, dirs if field == FIELD_MAIN else None, want_density=field != FIELD_MAIN,
                             want_actor_id=True, flip=fl)
    C.check_encoding(be, params, cfg, field, mean, std, times, dirs if field == FIELD_MAIN else None, fl, out, DEV, "good")
    return cfg, params, be, mean, std, times, dirs, fl, out


def test_comparators_reject_corrupted_encodings():
    cfg, params, be, mean, std, times, dirs, fl, out = _encoding_fixture()
    chk = lambda o: C.check_encoding(be, params, cfg, FIELD_MAIN, mean, std, times, dirs, fl, o, DEV, "x")  # noqa: E731
    f = out["features"].clone()
    f[40] = out["features"][41]  # a neighbouring sample's feature row
    _rejects(lambda: chk(dict(out, features=f)), "a neighbouring sample's feature row")
    aid = out["actor_id"].reshape(-1)
    k = int((aid >= 0).nonzero()[0])
    d = out["directions"].clone().reshape(-1, 3)
    d[k, 0] = -d[k, 0]  # the flip not applied to the direction
    _rejects(lambda: chk(dict(out, directions=d.reshape(out["directions"].shape))), "an actor direction without its flip")
    a = out["actor_id"].clone()
    a.reshape(-1)[k] = -1
    _rejects(lambda: chk(dict(out, actor_id=a)), "an actor sample assigned to the static field")
    # references that are wrong: the flip on the box y axis, the actor frame of the keyframe before the bracket
    n, S = mean.shape[:2]
    x, Ex = C.encoding_reference(params, cfg, FIELD_MAIN, mean, std, times, fl, out["actor_id"], DEV)
    C._ratio(out["features"], x, Ex, "good")
    for corrupt in ("wrong_axis", "wrong_keyframe"):
        xb, _ = C.encoding_reference(params, cfg, FIELD_MAIN, mean, std, times, fl, out["actor_id"], DEV, corrupt=corrupt)
        _rejects(lambda: C._ratio(xb.float(), x, Ex, "x"), f"features from {corrupt}")
    # density of a proposal field: one sample's density from its neighbour
    cfg, params, be, mean, std, times, _, fl, out = _encoding_fixture(FIELD_PROP1, flip="mixed")
    de = out["density"].clone()
    de.reshape(-1)[10] = out["density"].reshape(-1)[11]
    _rejects(lambda: C.check_encoding(be, params, cfg, FIELD_PROP1, mean, std, times, None, fl, dict(out, density=de), DEV, "x"),
             "a neighbouring sample's density")


def test_encoding_mutation_of_actor_order_is_caught():
    """The highest overlapping actor wins: the reference rejects the kernel's ids with the first hit kept instead."""
    cfg, params, be, mean, std, times, dirs, fl, out = _encoding_fixture(flip="plus")
    a = out["actor_id"].clone()
    ov = a == 1
    assert ov.any()
    ref, near = C.actor_id_reference(params, cfg, mean, times)
    both = ov & (ref == 1)
    a[both] = 0  # what a first-hit rule gives inside the overlap of actors 0 and 1
    _rejects(lambda: C.check_actor_ids(a, params, cfg, mean, times, "x"), "first-hit actor ids in an overlap")


def test_comparators_reject_corrupted_samplers():
    S, n = 16, 6
    nears, fars, t = C.stratified_inputs(n, S, S + 1, 3)
    bs = C.stratified_bins_s(S, t)
    be = C.euclid_reference("power", bs, nears, fars, -1.0, C.f32(0.1)).float()
    C.check_stratified(bs, be, nears, fars, S, t, "power", -1.0, C.f32(0.1), "good")
    bad = bs.clone()
    bad.view(torch.int32)[2, 5] += 1  # one ulp
    _rejects(lambda: C.check_stratified(bad, be, nears, fars, S, t, "power", -1.0, C.f32(0.1), "x"), "a one-ulp bins_s")
    tn = t.clone()
    tn[:, 1:] = t[:, :-1]  # every edge jittered with its neighbour's column
    _rejects(lambda: C.check_stratified(C.stratified_bins_s(S, tn), be, nears, fars, S, t, "power", -1.0, C.f32(0.1), "x"),
             "the neighbouring edge's jitter column")
    bad_e = be.clone()
    bad_e[3, 7] = be[3, 8]
    _rejects(lambda: C.check_euclid(bad_e, bs, nears, fars, "power", -1.0, C.f32(0.1), "x"), "a neighbouring euclidean edge")
    # pdf: one searchsorted index off by one, one ulp of a bin, one cdf entry from its neighbour
    w, bins, rand = C.pdf_inputs(n, 32, 31, "random", 32, 5)
    out = C.backend(DEV).pdf_resample_stratified(w, bins, 31, rand)
    C.check_pdf(out, w, bins, 31, rand, 0.01, "good")
    nb, cdf, inds = out
    i2 = inds.clone()
    i2[1, 4] += 1
    _rejects(lambda: C.check_pdf((nb, cdf, i2), w, bins, 31, rand, 0.01, "x"), "an index off by one")
    nb2 = nb.clone()
    nb2.view(torch.int32)[2, 3] += 1
    _rejects(lambda: C.check_pdf((nb2, cdf, inds), w, bins, 31, rand, 0.01, "x"), "a one-ulp new bin")
    c2 = cdf.clone()
    c2[3, 10] = cdf[3, 11]
    _rejects(lambda: C.check_pdf((nb, c2, inds), w, bins, 31, rand, 0.01, "x"), "a neighbouring cdf entry")
    rs = rand.clone()
    rs[:, 1:] = rand[:, :-1]  # the neighbouring edge's jitter column
    _rejects(lambda: C.check_pdf(out, w, bins, 31, rs, 0.01, "x"), "the neighbouring quantile's jitter column")


def test_comparators_reject_corrupted_mlps_and_heads():
    ws, bs = C.neurad_mlps()["feature"]
    x = torch.randn(300, ws[0].shape[1], generator=torch.Generator().manual_seed(1))
    y, zs = C.backend(DEV).mlp_fwd(x, ws, bs, want_hidden=True)
    C.check_mlp((y, zs), x, ws, bs, DEV, "good")
    bad = y.clone()
    bad[130] = y[2]  # one row of the next 128-row tile taken from the previous tile
    _rejects(lambda: C.check_mlp((bad, zs), x, ws, bs, DEV, "x"), "an MLP row from the neighbouring tile")
    z2 = [z.clone() for z in zs]
    z2[1][5] = zs[1][6]
    _rejects(lambda: C.check_mlp((y, z2), x, ws, bs, DEV, "x"), "a neighbouring row's hidden pre-activation")
    dy = torch.randn(300, 32, generator=torch.Generator().manual_seed(2))
    dx = C.backend(DEV).mlp_dgrad(dy, ws[-1], zs[-1])
    C.check_dgrad(dx, dy, ws[-1], zs[-1], DEV, "good")
    d2 = dx.clone()
    d2[200] = dx[72]
    _rejects(lambda: C.check_dgrad(d2, dy, ws[-1], zs[-1], DEV, "x"), "a dX row from another tile")
    geo = torch.randn(20, 16)
    geo[0, 0] = -10.0
    h = torch.randn(20, 15)
    be = C.backend(DEV, *(lambda cfg: (cfg, C.scene.make_params(cfg)))(C.nsb.small_config()))
    out = be._field_tail(geo, h)
    C.check_field_tail(out, geo, h, C.f32(be._beta), "good")
    f2 = out[0].clone()
    f2.view(torch.int32)[4, 4] += 1
    _rejects(lambda: C.check_field_tail((f2, out[1], out[2]), geo, h, C.f32(be._beta), "x"), "a one-ulp feature")
    a2 = out[2].clone()
    a2[3] = out[2][4]
    _rejects(lambda: C.check_field_tail((out[0], out[1], a2), geo, h, C.f32(be._beta), "x"), "a neighbouring row's alpha")
    d = torch.nn.functional.normalize(torch.randn(20, 3), dim=-1)
    x2 = be._field_mid(geo, d)
    C.check_field_mid(x2, geo, d, "good")
    x3 = x2.clone()
    x3[5, 15:] = x2[6, 15:]
    _rejects(lambda: C.check_field_mid(x3, geo, d, "x"), "a neighbouring row's SH columns")
