"""CPU: the entry-by-entry checks of the per-ray training operators (tests/ray_ops_cases.py) for the operators whose device
code runs here through the host emulation (tests/fake_backend.py): the weights backward from alpha and from density, the
distortion loss and the zipnerf interlevel loss.  composite_bwd, field_heads_bwd, relu_bwd, the mlp_dgrad mask and
lidar_carving_mask have torch stand-ins in the fake backend, so on the CPU they would compare torch with itself; they run
on the GPU only (test_zz_ray_ops_gpu.py).  The comparator self-tests below check that every comparator rejects a
corrupted copy of a correct result."""
import numpy as np
import pytest
import torch

from oracle import losses_oracle as LO
from tests import ray_ops_cases as C

DEV = "cpu"


def _report(name, worst):
    print(f"\n[ray ops] {name}: worst |got - ref| / tol = {worst:.3g}")


@pytest.mark.parametrize("n,S", [(1, 1), (33, 32), (70, 64), (19, 128), (5, 256)])
def test_alpha_weights_backward_per_entry(n, S):
    _report(f"dalpha n={n} S={S}", C.alpha_weights_backward_matches_float64(DEV, n, S, seed=S))


def test_alpha_weights_backward_at_alpha_one():
    """Rays with alpha == 1 exactly (once and twice): the occlusion term of a saturated sample is kept."""
    a = torch.tensor([[0.2, 0.5, 1.0, 0.3, 0.6, 0.1], [0.2, 1.0, 0.4, 1.0, 0.6, 0.1], [1.0, 0.0, 0.0, 0.0, 0.0, 0.0]])
    g = torch.randn(3, 6, generator=torch.Generator().manual_seed(0))
    _, ref, T, Rabs = C.alpha_reference(a, g)
    got = C.backend(DEV).alpha_to_weights_bwd(a, g)
    assert ref[0, 2].abs().item() > 1e-3 and ref[2, 0].abs().item() > 1e-3
    C._ratio(got, ref, C.alpha_bwd_tol(g, T, Rabs), "dalpha at alpha = 1")


@pytest.mark.parametrize("n,S", [(1, 1), (37, 32), (4099, 32), (70, 64), (19, 128), (9, 256)])
def test_density_weights_backward_per_entry(n, S):
    worst, excluded = C.density_weights_backward_matches_float64(DEV, n, S, seed=S)
    print(f"\n[ray ops] ddensity n={n} S={S}: worst {worst:.3g}, {excluded} entries with non-finite float64 autograd excluded")


@pytest.mark.parametrize("n,S", [(1, 1), (37, 33), (65, 64)])
def test_distortion_per_entry(n, S):
    _report(f"distortion n={n} S={S}", C.distortion_matches_float64(DEV, n, S, seed=S))


@pytest.mark.parametrize("r", C.PULSE)
@pytest.mark.parametrize("n,S,Sp", [(1, 1, 1), (63, 2, 64), (65, 33, 257), (64, 64, 128), (40, 32, 128)])
def test_interlevel_per_entry(n, S, Sp, r):
    _report(f"interlevel n={n} S={S} Sp={Sp} r={r:.3g}", C.interlevel_matches_float64(DEV, n, S, Sp, r, seed=S + Sp))


@pytest.mark.parametrize("r", C.PULSE)
def test_interlevel_at_the_relu_boundary(r):
    _report(f"interlevel ws == wp r={r:.3g}", C.interlevel_matches_float64(DEV, 40, 32, 64, r, seed=5, kind="tie"))


@pytest.mark.parametrize("Sp", [64, 257])
def test_interlevel_dyadic_is_exact_up_to_the_division(Sp):
    C.interlevel_matches_float64(DEV, 33, 64, Sp, 2.0 ** -7, seed=Sp, kind="dyadic")


def test_interlevel_no_rays():
    C.interlevel_matches_float64(DEV, 0, 32, 64, C.PULSE[0])


# ------------------------------------------------------------------------------------------------ comparator self-tests
def _rejects(fn, what):
    try:
        fn()
    except AssertionError:
        return
    raise AssertionError(f"the comparator accepted {what}")


def test_comparators_reject_corrupted_weights_gradients():
    n, S = 16, 32
    a = C.alpha_cases(S, n, 1)
    g = torch.randn(n, S, generator=torch.Generator().manual_seed(2))
    _, ref, T, Rabs = C.alpha_reference(a, g)
    tol = C.alpha_bwd_tol(g, T, Rabs)
    good = ref.float()
    C._ratio(good, ref, tol, "fp32 rounding of the reference")
    bad = good.clone()
    bad[5] = good[6]  # a neighbouring ray's row
    _rejects(lambda: C._ratio(bad, ref, tol, "x"), "a neighbouring ray's dalpha row")
    # the division formula this operator used before: dalpha_i = dw_i T_i - sum_{k>i} dw_k w_k / max(1 - a_i, 1e-10)
    a64, g64 = a.double(), g.double()
    w = a64 * T
    suf = C._suffix(g64 * w)
    old = (g64 * T - suf / (1 - a64).clamp_min(1e-10)).float()
    _rejects(lambda: C._ratio(old, ref, tol, "x"), "the clamped-division gradient at alpha = 1")
    delta, dens = C.density_cases(S, n, 3)
    r64 = dens.double().requires_grad_(True)
    ref_d, = torch.autograd.grad((C.O.weights_from_density(delta.double(), r64) * g.double()).sum(), r64)
    tol_d = C.density_bwd_tol(delta, dens, g)
    ok = torch.isfinite(ref_d)
    good_d = torch.nan_to_num(ref_d).float()
    C._ratio(good_d, ref_d, tol_d, "fp32 rounding", mask=ok)
    bad_d = good_d.clone()
    bad_d[7, 3] += 0.5 * (delta[7, 3] * g[7, 4] * 0.01).abs().item() + 1e-6  # a small entry nudged by far less than 1 %
    _rejects(lambda: C._ratio(bad_d, ref_d, tol_d, "x", mask=ok), "a nudged ddensity entry")


def test_comparators_reject_corrupted_losses():
    n, S = 12, 33
    c, w = C.distortion_inputs(n, S, 4)
    ref_l, ref_dw = C.distortion_reference(c, w)
    tl, tdw = C.distortion_tol(c, w)
    C._ratio(ref_dw.float(), ref_dw, tdw, "fp32 rounding")
    w2 = w.clone()
    w2[4, 7] = 0.0  # one bin's weight dropped
    bad_l, bad_dw = C.distortion_reference(c, w2)
    _rejects(lambda: C._ratio(bad_dw.float(), ref_dw, tdw, "x"), "dw with one bin dropped")
    _rejects(lambda: C._ratio(bad_l.float(), ref_l, tl, "x"), "a loss with one bin dropped")
    Sp, r = 64, C.PULSE[1]
    c, w, cp, wp = C.interlevel_inputs(n, S, Sp, 6)
    ref_l, ref_g, ws = C.interlevel_reference(c, w, cp, wp, r)
    tl, tg = C.interlevel_tol(ws, wp, C.interlevel_ws_error(c, w, cp, r))
    C._ratio(ref_g.float(), ref_g, tg, "fp32 rounding")
    C._ratio(ref_l.float(), ref_l, tl, "fp32 rounding")
    w2 = w.clone()
    w2[0, S // 3] = 0.0  # one final-level bin's weight dropped
    bad_l, bad_g, _ = C.interlevel_reference(c, w2, cp, wp, r)
    _rejects(lambda: C._ratio(bad_g.float(), ref_g, tg, "x"), "dwp with one bin dropped")
    wp2 = wp.clone()
    e = int((ws[4] - wp[4].double()).argmax())
    wp2[4, e] = wp[4, e] + 0.5 * (ws[4, e].float() - wp[4, e])  # one proposal bin's weight moved halfway towards ws
    bad_l, bad_g, _ = C.interlevel_reference(c, w, cp, wp2, r)
    _rejects(lambda: C._ratio(bad_l.float(), ref_l, tl, "x"), "a loss with one proposal weight changed")

    orig = LO.blur_stepfun

    def swapped(x, y, rr):  # two neighbouring blur knots of ray 0 swapped (each one's pdf value at the other's position)
        xr, yr = orig(x, y, rr)
        yr = yr.clone()
        m = int((yr[0, 1:] - yr[0, :-1]).abs().argmax())
        yr[0, m], yr[0, m + 1] = yr[0, m + 1].clone(), yr[0, m].clone()
        return xr, yr

    LO.blur_stepfun = swapped
    try:
        _, bad_g, _ = C.interlevel_reference(c, w, cp, wp, r)
    finally:
        LO.blur_stepfun = orig
    assert not torch.equal(bad_g, ref_g)
    _rejects(lambda: C._ratio(bad_g.float(), ref_g, tg, "x"), "dwp with two blur knots swapped")


def test_comparators_reject_corrupted_heads_and_composite():
    n, G, b = 129, 15, float(np.float32(20.0001))
    geo, (df, dsdf, dal, dx2) = C.field_heads_inputs(n, G, 1)
    C.set_extreme_sdf(geo, b)
    ins = {"dfeature": df, "dsdf": dsdf, "dalpha": dal, "dx2": dx2}
    g0, _, db, _ = C.field_heads_reference(geo, dsdf, dal, b)
    dgeo = torch.cat([g0.float()[:, None], df + dx2[:, :G]], 1)
    dbeta = db.sum().float().reshape(1)
    C.check_field_heads(dgeo, dbeta, geo, ins, b, "fp32 rounding")
    bad = dgeo.clone()
    bad[40] = dgeo[41]  # one row of dgeo from the neighbouring ray
    _rejects(lambda: C.check_field_heads(bad, dbeta, geo, ins, b, "x"), "a neighbouring ray's dgeo row")
    bad = dgeo.clone()
    bad[40, 0] = dgeo[41, 0]
    _rejects(lambda: C.check_field_heads(bad, dbeta, geo, ins, b, "x"), "a neighbouring ray's dgeo[:, 0]")
    miss = (dbeta.double() - db[32:64].sum()).float()  # dbeta missing one warp
    _rejects(lambda: C.check_field_heads(dgeo, miss, geo, ins, b, "x"), "dbeta missing one warp")
    bits = dgeo.clone()
    bits.view(torch.int32)[3, 5] ^= 1  # one ulp in the bit-exact columns
    _rejects(lambda: C.check_field_heads(bits, dbeta, geo, ins, b, "x"), "a one-ulp change of dgeo[:, 1:]")
    # composite: the comparator against its own fp32-rounded reference, then one sample's dw taken from its neighbour
    gen = torch.Generator().manual_seed(0)
    w, v = torch.rand(7, 9, generator=gen), torch.randn(7, 9, 3, generator=gen)
    go = torch.randn(7, 3, generator=gen)
    ref = (v.double() * go.double()[:, None, :]).sum(-1)
    tol = 7 * C.U * (v.double() * go.double()[:, None, :]).abs().sum(-1)
    C._ratio(ref.float(), ref, tol, "fp32 rounding")
    bad = ref.float().clone()
    bad[2, 4] = bad[2, 5]
    _rejects(lambda: C._ratio(bad, ref, tol, "x"), "a neighbouring sample's dw")
