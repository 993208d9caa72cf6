"""GPU: the per-ray training operators entry by entry against float64 (tests/ray_ops_cases.py) on the real library: the
weights forward and backward from alpha and from density, composite_bwd, field_heads_bwd, relu_bwd and the mlp_dgrad
ReLU mask, distortion_loss, zipnerf_interlevel_loss and lidar_carving_mask, at production shapes and at their edges.  The
weights backward and the two losses also run on the CPU over the host emulation (test_ray_ops_cpu.py)."""
import time

import pytest

from tests import ray_ops_cases as C

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _report(name, t0, worst):
    print(f"\n[ray ops] {name}: worst |got - ref| / tol = {worst:.3g}, {time.perf_counter() - t0:.1f} s")


@pytest.mark.parametrize("n,S", [(1, 1), (4099, 32), (1027, 64), (513, 128), (129, 256)])
def test_alpha_weights_forward_and_backward_per_entry(n, S):
    t0 = time.perf_counter()
    _report(f"alpha weights n={n} S={S}", t0, C.alpha_weights_backward_matches_float64(DEV, n, S, seed=S))


@pytest.mark.parametrize("n,S", [(1, 1), (4099, 32), (1027, 64), (513, 128), (129, 256)])
def test_density_weights_forward_and_backward_per_entry(n, S):
    t0 = time.perf_counter()
    worst, excluded = C.density_weights_backward_matches_float64(DEV, n, S, seed=S)
    _report(f"density weights n={n} S={S} ({excluded} entries with non-finite float64 autograd excluded)", t0, worst)


@pytest.mark.parametrize("n,S", [(1, 1), (4099, 33), (1025, 64)])
def test_distortion_per_entry(n, S):
    t0 = time.perf_counter()
    _report(f"distortion n={n} S={S}", t0, C.distortion_matches_float64(DEV, n, S, seed=S))


@pytest.mark.parametrize("r", C.PULSE)
@pytest.mark.parametrize("n,S,Sp", [(65536 + 3, 32, 128), (65, 64, 64), (64, 33, 257), (63, 2, 1), (1, 1, 64), (0, 32, 64),
                                    (200, 64, 257)])
def test_interlevel_per_entry(n, S, Sp, r):
    t0 = time.perf_counter()
    _report(f"interlevel n={n} S={S} Sp={Sp} r={r:.3g}", t0, C.interlevel_matches_float64(DEV, n, S, Sp, r, seed=S + Sp))


@pytest.mark.parametrize("r", C.PULSE)
def test_interlevel_at_the_relu_boundary(r):
    t0 = time.perf_counter()
    _report(f"interlevel ws == wp r={r:.3g}", t0, C.interlevel_matches_float64(DEV, 1025, 32, 128, r, seed=5, kind="tie"))


@pytest.mark.parametrize("Sp", [64, 257])
def test_interlevel_dyadic_is_exact_up_to_the_division(Sp):
    C.interlevel_matches_float64(DEV, 1025, 64, Sp, 2.0 ** -7, seed=Sp, kind="dyadic")


def test_interlevel_rejects_more_than_64_final_samples():
    from neurad_studio_b200.lib import B200NerfError

    c, w, cp, wp = C.interlevel_inputs(4, 65, 32, 0)
    with pytest.raises(B200NerfError):
        C.backend(DEV).zipnerf_interlevel_loss(c.to(DEV), w.to(DEV), cp.to(DEV), wp.to(DEV), C.PULSE[0], want_grad=True)


@pytest.mark.parametrize("C_", [1, 3, 48])
def test_composite_bwd_every_cotangent_combination(C_):
    t0 = time.perf_counter()
    be = C.backend(DEV)
    worst = 0.0
    for mask in range(32):
        has_v, has_a, has_d, need_dw, need_dv = (bool(mask >> b & 1) for b in range(5))
        worst = max(worst, C.composite_case(DEV, 337, 45, C_, has_v, has_a, has_d, need_dw, need_dv, seed=mask, be=be))
    _report(f"composite_bwd C={C_} (n * S = 337 * 45, all 32 combinations)", t0, worst)


@pytest.mark.parametrize("G,n", [(1, 129), (15, 127), (32, 57344 * 32), (127, 128), (128, 129), (200, 1), (200, 4099)])
def test_field_heads_bwd_per_entry(G, n):
    t0 = time.perf_counter()
    worst = 0.0
    for absent in (None, "dfeature", "dsdf", "dalpha", "dx2"):
        if n > 100000 and absent not in (None, "dalpha"):
            continue
        worst = max(worst, C.field_heads_case(DEV, n, G, absent, seed=G))
    _report(f"field_heads_bwd G={G} n={n}", t0, worst)


def test_field_tail_gradient_of_a_negative_beta():
    t0 = time.perf_counter()
    _report("FieldTailFn beta < 0", t0, C.field_tail_sign_of_negative_beta(DEV))


@pytest.mark.parametrize("n", [1, 7, 255, 4099])
def test_relu_bwd_bit_exact(n):
    C.relu_bwd_bit_exact(DEV, n)


@pytest.mark.parametrize("rows,k,n_out", [(129, 32, 32), (1000, 33, 64), (300, 48, 17)])
def test_mlp_dgrad_relu_mask_bit_exact(rows, k, n_out):
    C.mlp_dgrad_mask_bit_exact(DEV, rows, k, n_out)


@pytest.mark.parametrize("with_did_return", [True, False])
@pytest.mark.parametrize("n,S", [(1027, 48), (31, 8)])
def test_lidar_carving_mask_bit_exact(n, S, with_did_return):
    C.lidar_mask_bit_exact(DEV, n, S, with_did_return, seed=n)
