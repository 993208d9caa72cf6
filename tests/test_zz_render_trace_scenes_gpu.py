"""GPU: the ray-per-lane render kernels sample by sample (tests/render_trace_cases.py, MLP bounds with the fp16 split's
gamma_f16) on the scenes beyond config 2 / 3 / opaque, at production table sizes: zero-area lidar sweeps from
raygen_lidar_sweeps over four actors at unit and 0.1 table scale, tables at the reference's init scale 1e-3, tables at
1e-4 with bias-free MLPs (subnormal lo parts in the fp16 split), config 3's actors under an actor edit set through the
backend, and the neurad-paper and neurader presets (neurader's 2^23-row main table and 16383-cell finest level).  Both
"split" and "lane" get the full check, and their traces must agree bit for bit.  Then the unit-scale lidar-sweep scene
against the live reference at the tolerance its own noise floor justifies.  The same scenes run on the CPU over the
host emulation in test_render_trace_scenes_cpu.py."""
import time

import pytest

from tests import render_trace_cases as C

pytestmark = pytest.mark.gpu
DEV = "cuda"
SCENES = ["sweep_unit", "sweep_tenth", "init_scale", "f16_small", "edits", "paper", "neurader"]


@pytest.mark.parametrize("name", SCENES)
def test_render_trace_scene_sample_by_sample(name):
    t0 = time.perf_counter()
    ws, exits_s, faces, full_s, idx = C.check_scene(DEV, name, "split")
    full_s = C.select(full_s, idx)
    wl, exits_l, _, full_l, _ = C.check_scene(DEV, name, "lane")
    full_l = C.select(full_l, idx)
    for k in full_s:
        C._bits_equal(full_l[k], full_s[k], f"{name}: lane vs split {k}")
    print(f"\n[render trace] {name}: worst ratio to bound split " + ", ".join(f"{k} {v:.3g}" for k, v in ws.items())
          + "; lane " + ", ".join(f"{k} {v:.3g}" for k, v in wl.items())
          + f"; early-exit warps (inferred) {exits_s}; actor-id face exceptions {faces}; {time.perf_counter() - t0:.1f} s")


def test_unit_scale_sweep_against_the_reference():
    """The lidar-sweep golden's viewer sweep over its scene with the tables at the unit init, rendered by the library
    against the live reference (the oracle): depth within SWEEP_UNIT_DEPTH_TOL (set above the reference's own floor there,
    3.6e-4; tests/test_render_trace_scenes_cpu.py; measured 3.9e-4), every other output within the 1e-4 render
    tolerance."""
    import torch

    cfg, params, rays = C.sweep_golden_scene(1.0)
    ref = C.sweep_oracle(1.0)
    out = C.renderer(DEV, cfg, params).render({k: v.to(DEV) for k, v in rays.items()}, want_trace=False, want_intensity=True)
    got = {k: C.rel_to_max(out[k], ref[k]) for k in ("depth", "accumulation", "features", "prop_depth_0", "prop_depth_1")}
    print(f"\n[sweep unit] library vs reference, of each output's maximum: {got}")
    assert got["depth"] < C.SWEEP_UNIT_DEPTH_TOL, got
    for k, v in got.items():
        assert k == "depth" or v < 1e-4, (k, v)
    assert torch.isfinite(out["depth"]).all()
