"""GPU: the tiny-cuda-nn-layout render kernels sample by sample (tests/tcnn_trace_cases.py; MLP bounds with the fp16
split's gamma_f16) at production table sizes: tcnn_test_config with every kind of level, the default NeuRADConfig with
16 actors through a camera's 2-D tile walk, zero-area lidar sweeps, tables at 1e-4, the neurader preset and an actor
edit set through the backend.  The layout runs in the two-stage renderer ("split") only; the fused lane kernel refuses
it with an error.  Then the layout's grid operator, B200Backend.tcnn_hashgrid_fwd, entry by entry against float64.  The
same scenes run over the host emulation in test_tcnn_trace_cpu.py."""
import time

import pytest
import torch

from tests import render_trace_cases as C
from tests import tcnn_trace_cases as TT

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.mark.parametrize("name", TT.GPU_SCENES)
def test_tcnn_trace_scene_sample_by_sample(name):
    t0 = time.perf_counter()
    (ws, exits, faces, _, _), cov = TT.check_tcnn_scene(DEV, name, "split")
    print(f"\n[tcnn trace] {name}: worst ratio to bound " + ", ".join(f"{k} {v:.3g}" for k, v in ws.items())
          + f"; actor-id face exceptions {faces}; coverage: {cov}; {time.perf_counter() - t0:.1f} s")


def test_fused_lane_kernel_refuses_the_tcnn_layout():
    """A tcnn-layout parameter set renders through the sampling / shading kernel pair only: the fused lane kernel has
    no tiny-cuda-nn instance and must say so rather than read the tcnn grids as torch-layout tables."""
    cfg, params, rays, _ = TT.scene_rays(DEV, "tcnn_small")
    r = C.renderer(DEV, cfg, params)
    assert r.be.layout == "tcnn"
    with pytest.raises(Exception, match="tiny-cuda-nn"):
        r.render({k: v[:256].to(DEV) for k, v in rays.items()}, want_trace=False, mode="lane")
    out = r.render({k: v[:256].to(DEV) for k, v in rays.items()}, want_trace=False, mode="split")
    assert torch.isfinite(out["depth"]).all()


def test_tcnn_grid_operator_entry_by_entry():
    TT.grid_operator_entry_by_entry(DEV)
