"""GPU: the camera-pose gradient operators entry by entry against float64 autograd through the oracle
(tests/camera_opt_cases.py) at production table sizes (main field 2^22 with 2^17 actor grids, proposal field 2^20 with
2^15), up to 64 actors; isotropic_gaussian_bwd; loss.backward() through the camera optimizer and the module walk against
the reference's goldens; and the fused render of a use_camopt_in_eval model.  The operator bodies also run on the CPU over
the host emulation in test_camera_opt_cpu.py."""
import time

import pytest

from neurad_studio_b200.lib import FIELD_MAIN, FIELD_PROP1
from tests import camera_opt_cases as C

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("n,S,n_actors,flip,ties", [
    (4103, 32, 0, False, True),
    (4103, 32, 16, True, False),
    (4103, 32, 16, False, False),
    (1025, 32, 64, True, False),
    (1025, 32, 64, False, False),
])
def test_features_mode_dmean_per_entry(n, S, n_actors, flip, ties):
    t0 = time.perf_counter()
    w = C.mean_bwd_matches_float64_reference("cuda", FIELD_MAIN, n, S, n_actors, flip, ties=ties)
    print(f"\n[camera opt] features n={n} S={S} actors={n_actors} flip={flip}: worst |got - ref| / tol = {w:.3f}, "
          f"{time.perf_counter() - t0:.1f} s")


@pytest.mark.parametrize("n,S,n_actors,flip", [(2048, 64, 0, False), (2048, 64, 16, True), (1025, 64, 64, False)])
def test_density_mode_dmean_per_entry(n, S, n_actors, flip):
    t0 = time.perf_counter()
    w = C.mean_bwd_matches_float64_reference("cuda", FIELD_PROP1, n, S, n_actors, flip)
    print(f"\n[camera opt] density n={n} S={S} actors={n_actors} flip={flip}: worst |got - ref| / tol = {w:.3f}, "
          f"{time.perf_counter() - t0:.1f} s")


def test_empty_and_zero_cotangent_give_zeros():
    C.empty_and_zero_cotangent_give_zeros("cuda", 16)


def test_isotropic_gaussian_bwd_per_entry():
    w = C.gaussian_bwd_matches_float64("cuda", 40960, 33)
    print(f"\n[camera opt] isotropic_gaussian_bwd 40960 x 33: worst ratio {w:.3f}")


@pytest.mark.parametrize("label,name", [("so3xr3", "nff_static.npz"), ("scaled", "nff_static.npz"), ("se3", "nff_static.npz"),
                                        ("so3xr3", "nff_actors.npz"), ("scaled", "nff_actors.npz")])
def test_module_walk_pose_gradients_match_reference_golden(label, name):
    w = C.module_walk_pose_gradients_match_reference_golden(label, name, "cuda")
    print(f"\n[camera opt] {label} {name}: " + ", ".join(f"d{k} {v:.2e}" for k, v in w.items()))


def test_camopt_in_eval_renders_the_corrected_bundle():
    C.camopt_in_eval_renders_the_corrected_bundle("cuda")
