"""GPU: the reference's own unit tests for the modules on this path, run against the library's mirror (bodies in
tests/reference_compat_cases.py; CPU twins over the fake backend in tests/test_reference_compat_cpu.py)."""
import pytest

from tests import reference_compat_cases as R

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("kind", sorted(R.SPACED))
def test_spaced_sampler(kind):
    R.spaced_sampler(R.SPACED[kind], "cuda")


def test_pdf_sampler():
    R.pdf_sampler("cuda")


def test_rgb_renderer():
    R.rgb_renderer("cuda")


def test_acc_renderer():
    R.acc_renderer("cuda")


def test_frustum_get_position():
    R.frustum_get_position("cuda")


def test_spherical_harmonics():
    R.spherical_harmonics("cuda")


def test_tensor_hash_encoder():
    R.tensor_hash_encoder("cuda")


def test_mlp():
    R.mlp("cuda")


def test_standalone_modules_train():
    R.standalone_modules_train("cuda")
