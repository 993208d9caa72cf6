"""GPU: the wgmma split-K weight-gradient operator (`b200nerf_linear_wgrad_tc`), checked like any other
operator although the CUDA-core twin stays the default.  The file still sorts last (a faulting kernel here cannot disturb the suites before it)."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def rel_to_max(a, b):
    a, b = a.detach().cpu().float(), b.detach().cpu().float()
    return (a.reshape(b.shape) - b).abs().max().item() / (b.abs().max().item() + 1e-30)


@pytest.mark.parametrize("k,n,relu", [(32, 33, False), (32, 32, True), (48, 32, False), (64, 64, True), (6, 1, False), (50, 57, True)])
@pytest.mark.parametrize("rows", [48 * 5, 48 * 300 + 17, 5])
def test_linear_wgrad_tensor_core_twin(k, n, relu, rows):
    """b200nerf_linear_wgrad_tc (wgmma split-K, 3xTF32) against fp64 torch and against the CUDA-core operator."""
    from neurad_studio_b200.backend import B200Backend

    be = B200Backend(torch.device("cuda", 0))
    gen = torch.Generator().manual_seed(k * 1000 + n + rows)
    x, dy = torch.randn(rows, k, generator=gen).cuda(), torch.randn(rows, n, generator=gen).cuda()
    dW, db = torch.zeros(n, k, device="cuda"), torch.zeros(n, device="cuda")
    be.linear_wgrad(x, dy, relu, dW, db, impl="tc")
    torch.cuda.synchronize()
    be.check_status()
    xa = torch.relu(x) if relu else x
    want = (dy.double().t() @ xa.double()).float()
    assert rel_to_max(dW, want) < 2e-5
    # a column sum of N(0,1) draws cancels (|sum| ~ sqrt(rows) while sum|dy| ~ rows): the fp32 bound is relative to sum|dy|,
    # and the atomics' order changes from run to run
    db_err = (db - dy.double().sum(0).float()).abs().max().item()
    assert db_err <= 2e-6 * dy.abs().sum(0).max().item() + 1e-6
    dW2, db2 = torch.zeros_like(dW), torch.zeros_like(db)
    be.linear_wgrad(x, dy, relu, dW2, db2, impl="cuda")
    assert rel_to_max(dW, dW2) < 2e-5
    be.linear_wgrad(x, dy, relu, dW, db, impl="tc")  # accumulates into the same buffers
    assert rel_to_max(dW, 2 * want) < 2e-5
