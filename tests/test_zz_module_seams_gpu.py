"""GPU parity tests of the MODULE-LEVEL seams (SURVEY 8b: Field, Sampler, NeuRADHashEncoding as stand-alone operators
through the C ABI) and of the backward operators / training-mode semantics (SURVEY 8f row f2), against the reference's
own per-stage goldens, gradient goldens (its autograd) and stratified-sampling goldens, and against the fused renderer.

The same bodies run in the CPU container over tests/fake_backend.py (tests/test_module_glue_cpu.py)."""
import pytest

from tests import module_seam_cases as C

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", ["nff_static.npz", "nff_actors.npz", "nff_sharp.npz"])
def test_field_forward_matches_reference_golden(name):
    C.field_forward_matches_reference_golden(name, "cuda")


@pytest.mark.parametrize("name", ["nff_static.npz", "nff_actors.npz"])
def test_proposal_density_and_encoding_match_reference_golden(name):
    C.proposal_density_and_encoding_match_reference_golden(name, "cuda")


@pytest.mark.parametrize("name", ["nff_static.npz", "nff_actors.npz", "nff_sharp.npz"])
def test_proposal_sampler_and_module_walk_match_reference_golden(name):
    C.proposal_sampler_and_module_walk_match_reference_golden(name, "cuda")


def test_module_operator_errors_and_empty_inputs():
    C.module_operator_errors_and_empty_inputs("cuda")


@pytest.mark.parametrize("name", ["nff_static.npz", "nff_actors.npz"])
def test_training_gradients_match_reference_golden(name):
    C.training_gradients_match_reference_golden(name, "cuda")


def test_proposal_density_backward_clamps_like_trunc_exp():
    C.proposal_density_backward_clamps_like_trunc_exp("cuda")


def test_backward_stage_operators_match_torch_autograd():
    C.backward_stage_operators_match_torch_autograd("cuda")


def test_stratified_sampling_matches_reference_golden():
    C.stratified_sampling_matches_reference_golden("cuda")


@pytest.mark.parametrize("name", ["nff_static.npz", "nff_actors.npz"])
def test_training_mode_walk_runs(name):
    C.training_mode_walk_runs(name, "cuda")


def test_training_losses_match_reference_golden():
    C.training_losses_match_reference_golden("cuda")


def test_lidar_carving_masks_and_training_outputs():
    C.lidar_carving_masks_and_training_outputs("cuda")


def test_get_outputs_and_decode_features():
    C.get_outputs_and_decode_features("cuda")


def test_train_mode_encoding_matches_reference_golden():
    C.train_mode_encoding_matches_reference_golden("cuda")


def test_metric_entry_points():
    C.metric_entry_points("cuda")
