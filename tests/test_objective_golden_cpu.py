"""CPU: NeuRADModel.get_metrics_dict / get_loss_dict of the mirror, over a CPU stand-in backend whose lidar losses and
regularisers are the host emulation of the library's device code, reproduce the reference's own methods as recorded in
tests/golden/objective.npz (oracle/make_golden_objective.py): key sets, values, gradients, quantile and mask."""
import os

import numpy as np
import pytest

from tests import objective_cases as C

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "objective.npz")


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(GOLDEN, allow_pickle=False))


@pytest.fixture()
def model(monkeypatch):
    import neurad_studio_b200 as nsb
    from neurad_studio_b200 import nerfstudio_api
    from oracle.make_golden_objective import SDF_BETA
    from tests.objective_fake_backend import ObjectiveFakeBackend

    be = ObjectiveFakeBackend()
    monkeypatch.setattr(nerfstudio_api, "get_backend", lambda device: be)
    m = nerfstudio_api.NeuRADModel(nsb.small_config())
    with __import__("torch").no_grad():
        m._param("field.sdf_to_density.beta").fill_(SDF_BETA)
    return m


def test_golden_inputs_are_the_oracles_cases(golden):
    from oracle.make_golden_objective import CASES, make_case

    assert sorted(CASES) == sorted(C.GOLDEN_CASES)
    for name, (patches, n_lidar, _, opts) in CASES.items():
        outputs, batch, _, _ = make_case(patches, n_lidar, opts)
        for k, v in outputs.items():
            assert np.array_equal(golden[f"{name}_out_{k}"], v.numpy(), equal_nan=True), (name, k)
        for k, v in batch.items():
            assert np.array_equal(golden[f"{name}_in_{k}"], v.numpy()), (name, k)


@pytest.mark.parametrize("name", C.GOLDEN_CASES)
def test_mirror_reproduces_the_reference_objective(golden, model, name):
    C.check_mirror_against_golden(model, golden, name, "cpu")
