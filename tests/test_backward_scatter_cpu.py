"""CPU: the entry-by-entry checks of the hash-grid backward operators (tests/backward_scatter_cases.py) over
tests/fake_backend.py, i.e. the kernels' device functions run by the host emulation, at small tables and ray counts.  The
same bodies run on the GPU at production table sizes in test_zz_backward_scatter_gpu.py."""
import pytest

from tests import backward_scatter_cases as C


@pytest.mark.parametrize("n,S,n_actors,flip,layout", [
    (1, 1, 0, False, "spread"),
    (33, 3, 2, True, "spread"),
    (33, 5, 0, False, "steps"),
    (40, 32, 3, False, "steps"),
    (64, 5, 4, True, "clusters"),
    (70, 32, 0, False, "clusters"),
])
def test_features_mode_per_entry(n, S, n_actors, flip, layout):
    C.features_mode_matches_float64_reference("cpu", n, S, n_actors, flip, layout, none_actors=(1,) if n_actors > 2 else ())


@pytest.mark.parametrize("n,S,n_actors,want_decoder", [(33, 5, 0, True), (24, 64, 2, False), (9, 128, 3, True)])
def test_density_mode_per_entry(n, S, n_actors, want_decoder):
    C.density_mode_matches_float64_reference("cpu", n, S, n_actors, want_decoder, flip=n_actors > 0)


@pytest.mark.parametrize("L,F,log2T", [(16, 2, 12), (6, 1, 10), (8, 4, 12), (4, 8, 10), (16, 4, 8)])
def test_hashgrid_bwd_per_entry(L, F, log2T):
    C.hashgrid_bwd_matches_float64_reference("cpu", L, F, log2T, 3000)


@pytest.mark.parametrize("flip", [False, True])
def test_pose_bwd_per_actor_and_keyframe(flip):
    C.pose_bwd_matches_oracle_per_actor_and_keyframe("cpu", 4, flip)


def test_empty_and_zero_cotangent_are_no_ops():
    C.empty_and_zero_cotangent_leave_accumulators_bit_identical("cpu", 2)


def test_comparator_rejects_a_lost_or_doubled_sample():
    C.comparator_rejects_a_lost_or_doubled_sample("cpu")
