"""GPU: the ray-per-lane render kernels sample by sample against stage-local float64 references and bit-exact
restatements (tests/render_trace_cases.py), at production table sizes: config 2 (one PandaSet camera at render stride 3
through the 2-D tile walk, a lidar sweep, nears / fars), config 3 (16 actors, a ray count that leaves the last warp
group ragged) and an opaque scene whose proposal transmittance underflows in whole warps.  Both "split" (sampling and
shading kernels) and "lane" (one fused kernel) get the full check, and their traces must agree bit for bit.  A partial
trace without actor ids (the early exit on) and an untraced render must give the full trace's results bit for bit.
The same bodies run on the CPU over the host emulation in test_render_trace_cpu.py."""
import time

import pytest

from tests import render_trace_cases as C

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.mark.parametrize("name", ["config2", "config3", "opaque"])
def test_render_trace_sample_by_sample(name):
    t0 = time.perf_counter()
    ws, exits_s, faces, full_s, idx = C.check_scene(DEV, name, "split")
    full_s = C.select(full_s, idx)
    wl, exits_l, _, full_l, _ = C.check_scene(DEV, name, "lane")
    full_l = C.select(full_l, idx)
    for k in full_s:
        C._bits_equal(full_l[k], full_s[k], f"{name}: lane vs split {k}")
    if name == "opaque":
        assert exits_s > 0, "no warp of the opaque scene takes the proposal round's early exit"
    print(f"\n[render trace] {name}: worst ratio to bound split " + ", ".join(f"{k} {v:.3g}" for k, v in ws.items())
          + "; lane " + ", ".join(f"{k} {v:.3g}" for k, v in wl.items())
          + f"; early-exit warps (inferred) {exits_s}; actor-id face exceptions {faces}; {time.perf_counter() - t0:.1f} s")


@pytest.mark.parametrize("image_width", [0, 640])
def test_sliced_bundle(image_width):
    bounds, dt = C.check_sliced(DEV, image_width)
    print(f"\n[render trace] 2^21 + 4099 rays, image_width {image_width}: slice boundaries {bounds}; {dt:.1f} s")
