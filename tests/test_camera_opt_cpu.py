"""CPU: the camera-pose gradient operators (tests/camera_opt_cases.py) over tests/camopt_fake_backend.py, i.e. the kernels' device
functions run by the host emulation, at small tables; and the camera optimizer mirror.  The same operator bodies run on
the GPU at production table sizes in test_zz_camera_opt_gpu.py."""
import pytest
import torch

from neurad_studio_b200.lib import FIELD_MAIN, FIELD_PROP1
from tests import camera_opt_cases as C


@pytest.mark.parametrize("n,S,n_actors,flip,ties", [(33, 16, 0, False, True), (40, 32, 3, False, False), (64, 8, 4, True, False)])
def test_features_mode_dmean_per_entry(n, S, n_actors, flip, ties):
    C.mean_bwd_matches_float64_reference("cpu", FIELD_MAIN, n, S, n_actors, flip, ties=ties)


@pytest.mark.parametrize("n,S,n_actors,flip", [(33, 64, 0, False), (24, 32, 3, True)])
def test_density_mode_dmean_per_entry(n, S, n_actors, flip):
    C.mean_bwd_matches_float64_reference("cpu", FIELD_PROP1, n, S, n_actors, flip)


def test_cases_reach_both_sides_of_the_contraction_and_the_clamp():
    C.mean_bwd_covers_both_sides("cpu")


def test_empty_and_zero_cotangent_give_zeros():
    C.empty_and_zero_cotangent_give_zeros("cpu", 2)


def test_isotropic_gaussian_bwd_per_entry():
    C.gaussian_bwd_matches_float64("cpu", 50, 33)


def test_exp_maps_match_closed_forms():
    C.exp_maps_match_closed_forms()


def test_comparator_rejects_a_wrong_row():
    ref = torch.randn(4, 5, 3, dtype=torch.float64)
    C.check_dmean(ref.float(), ref)
    bad = ref.clone()
    bad[2, 3, 1] *= 1.01
    with pytest.raises(AssertionError):
        C.check_dmean(bad, ref)


CASES = [("so3xr3", "nff_static.npz"), ("scaled", "nff_static.npz"), ("se3", "nff_static.npz"), ("so3xr3", "nff_actors.npz"),
         ("scaled", "nff_actors.npz")]


@pytest.mark.parametrize("label,name", CASES)
def test_camera_optimizer_mirror_matches_reference_golden(label, name):
    C.mirror_matches_reference_golden(label, name)


def test_mode_off_adds_no_parameters_or_keys():
    C.mode_off_is_unchanged("nff_static.npz")


@pytest.mark.parametrize("label,name", [("so3xr3", "nff_static.npz"), ("scaled", "nff_actors.npz")])
def test_module_walk_pose_gradients_glue(label, name, monkeypatch):
    from neurad_studio_b200 import nerfstudio_api
    from tests.camopt_fake_backend import CamoptFakeBackend

    be = CamoptFakeBackend()
    monkeypatch.setattr(nerfstudio_api, "get_backend", lambda device: be)
    C.module_walk_pose_gradients_match_reference_golden(label, name, "cpu")


def test_reference_direction_gradient_moves_more_than_the_bar_under_one_ulp():
    C.reference_direction_gradient_noise_floor()
