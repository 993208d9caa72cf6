"""GPU: the hash-grid backward operators entry by entry against float64 autograd through the oracle
(tests/backward_scatter_cases.py), at production table sizes (main field 2^22 with 4 x 2^17 actor grids, proposal field
2^20 with 4 x 2^15) and at 2^12 (heavy collisions); up to 64 actors, i.e. 128 KB of dynamic shared memory in the scatter
kernel; and linear_wgrad, the CUDA-core dW, at 2^20 + 17 rows.  The same bodies (except linear_wgrad's: on the CPU it would
compare the emulation with itself) run on the CPU over the host emulation in test_backward_scatter_cpu.py.

The warp-level merge of pending sums (modules.cuh: warp_merge_pending) exists in the GPU kernel only; the host emulation
flushes every thread's sums itself, so this file is the one that checks it (the "clusters" cases drive its leftover path)."""
import time

import pytest

from tests import backward_scatter_cases as C

pytestmark = pytest.mark.gpu


def _report(name, t0, worst):
    print(f"\n[backward scatter] {name}: worst |got - P - ref| / tol = {worst:.3f}, {time.perf_counter() - t0:.1f} s")


@pytest.mark.parametrize("n,S,n_actors,flip,layout,log2_main,none_actors", [
    (4103, 32, 0, False, "spread", None, ()),
    (4103, 5, 16, True, "steps", None, (3,)),
    (33, 3, 25, True, "spread", None, ()),
    (1, 1, 0, False, "spread", None, ()),
    (33, 1, 64, False, "spread", None, ()),
    (4103, 32, 64, True, "spread", None, (5, 40)),
    (2048, 32, 0, False, "clusters", None, ()),
    (512, 5, 16, False, "clusters", None, ()),
    (4103, 32, 25, True, "steps", 12, ()),
    (33, 5, 0, False, "spread", 12, ()),
])
def test_features_mode_per_entry(n, S, n_actors, flip, layout, log2_main, none_actors):
    t0 = time.perf_counter()
    w = C.features_mode_matches_float64_reference("cuda", n, S, n_actors, flip, layout, log2_main, none_actors)
    _report(f"features n={n} S={S} actors={n_actors} flip={flip} {layout} log2T={log2_main or 22}", t0, w)


@pytest.mark.parametrize("n,S,n_actors,want_decoder,flip", [
    (1024, 128, 0, True, False),
    (2048, 64, 16, False, False),
    (4103, 5, 64, True, True),
])
def test_density_mode_per_entry(n, S, n_actors, want_decoder, flip):
    t0 = time.perf_counter()
    w = C.density_mode_matches_float64_reference("cuda", n, S, n_actors, want_decoder, flip)
    _report(f"density n={n} S={S} actors={n_actors} decoder={want_decoder} flip={flip}", t0, w)


@pytest.mark.parametrize("L,F,log2T", [(16, 2, 19), (6, 1, 20), (8, 4, 22), (4, 8, 12), (16, 4, 12)])
def test_hashgrid_bwd_per_entry(L, F, log2T):
    t0 = time.perf_counter()
    w = C.hashgrid_bwd_matches_float64_reference("cuda", L, F, log2T, 20000)
    _report(f"hashgrid L={L} F={F} log2T={log2T}", t0, w)


@pytest.mark.parametrize("n_actors,flip", [(16, False), (64, True)])
def test_pose_bwd_per_actor_and_keyframe(n_actors, flip):
    t0 = time.perf_counter()
    w = C.pose_bwd_matches_oracle_per_actor_and_keyframe("cuda", n_actors, flip)
    print(f"\n[backward scatter] pose actors={n_actors} flip={flip}: worst per-slice rel error = {w:.2e}, "
          f"{time.perf_counter() - t0:.1f} s")


@pytest.mark.parametrize("K,N,relu", [(32, 33, True), (48, 32, False), (64, 64, True)])
def test_linear_wgrad_per_entry(K, N, relu):
    t0 = time.perf_counter()
    w = C.linear_wgrad_matches_float64("cuda", K, N, relu)
    _report(f"linear_wgrad K={K} N={N} relu={relu} (2^20 + 17 rows; dyadic run exact)", t0, w)


def test_empty_and_zero_cotangent_are_no_ops():
    C.empty_and_zero_cotangent_leave_accumulators_bit_identical("cuda", 25)
