"""GPU: the generic stage operators entry by entry against float64 (tests/stage_ops_cases.py) on the real library:
composite_kernel and depth_clip_kernel (values with and without nan_to_num and a background, accumulation, simple /
expected / median depth; ragged 32-sample chunks and 8-channel passes; 2^20 rays feeding the clip's atomics; every
composite call of one training step and of one eval-mode module walk), the RGBRenderer mirror, and the eval-mode
spaced_sample_kernel, pdf_resample_kernel, frustum_positions_kernel, density_rgb_heads_kernel, sh4_fwd_kernel and
mlp_tc_kernel on config 1's and other generic shapes.  Each test prints its worst |got - ref| / tol."""
import time

import pytest
import torch

from tests import stage_ops_cases as C

pytestmark = pytest.mark.gpu
DEV = "cuda"
_T0 = time.perf_counter()
SAMPLES = (1, 7, 31, 32, 33, 64, 100, 128, 129)
CHANNELS = (1, 3, 7, 8, 9, 32, 33, 48, 64)


def _report(name, t0, worst):
    print(f"\n[stage ops] {name}: worst |got - ref| / tol = {worst:.3g}, {time.perf_counter() - t0:.1f} s "
          f"(file wall time so far {time.perf_counter() - _T0:.1f} s)")


@pytest.fixture(scope="module")
def be():
    return C.backend(DEV)


# ====================================================================================== composite
@pytest.mark.parametrize("depth", ["simple", "expected", "median"])
@pytest.mark.parametrize("S", SAMPLES)
def test_composite_samples(be, S, depth):
    t0 = time.perf_counter()
    r = C.composite_case(DEV, 4097, S, 9, depth, bg=S % 2 == 1, nan_to_num=True, seed=S, be=be)
    _report(f"composite n=4097 S={S} C=9 {depth} (clipped {r['clipped']})", t0, r["worst"])


@pytest.mark.parametrize("C_", CHANNELS)
def test_composite_channels(be, C_):
    t0 = time.perf_counter()
    r = C.composite_case(DEV, 517, 33, C_, "expected", bg=True, nan_to_num=C_ % 2 == 0, seed=C_, be=be)
    _report(f"composite n=517 S=33 C={C_}", t0, r["worst"])


@pytest.mark.parametrize("n", [1, 3, 4, 5])
@pytest.mark.parametrize("depth", ["simple", "expected", "median"])
def test_composite_few_rays(be, n, depth):
    t0 = time.perf_counter()
    _report(f"composite n={n} {depth}", t0, C.composite_case(DEV, n, 65 - n, 3 + n, depth, bg=True, seed=n, be=be)["worst"])


def test_composite_many_rays(be):
    """2^20 + 3 rays: 262 145 CTAs feed the clip's atomics."""
    t0 = time.perf_counter()
    r = C.composite_case(DEV, (1 << 20) + 3, 32, 3, "expected", bg=True, nan_to_num=True, seed=1, be=be)
    _report(f"composite n=2^20+3 S=32 C=3 expected (clipped {r['clipped']})", t0, r["worst"])


def test_composite_rejects_65_channels(be):
    from neurad_studio_b200.lib import B200NerfError

    with pytest.raises(B200NerfError):
        be.composite(torch.rand(2, 3, device=DEV), torch.rand(2, 3, 65, device=DEV))


@pytest.mark.parametrize("S", [33, 129])
@pytest.mark.parametrize("bg", [False, True])
@pytest.mark.parametrize("nan_to_num", [False, True])
def test_composite_specials(be, S, bg, nan_to_num):
    t0 = time.perf_counter()
    r = C.composite_case(DEV, 1001, S, 9, "simple", bg=bg, nan_to_num=nan_to_num, kind="specials", seed=S, be=be)
    _report(f"composite specials S={S} bg={bg} nan_to_num={nan_to_num}", t0, r["worst"])


@pytest.mark.parametrize("S", [1, 3, 31, 32, 33, 64, 128, 129])
def test_median_exact(be, S):
    t0 = time.perf_counter()
    _report(f"median S={S}", t0, C.median_case(DEV, S, n_pad=4093, be=be))


@pytest.mark.parametrize("n,S", [(4097, 33), ((1 << 20) + 1, 32)])
def test_expected_depth_clip(be, n, S):
    t0 = time.perf_counter()
    C.clip_case(DEV, n, S, be=be)
    _report(f"expected depth clip n={n} S={S}, two calls", t0, 0.0)


def test_recorded_composites():
    t0 = time.perf_counter()
    worst, shapes = C.check_recorded_composites(DEV, 8192, 4096)
    _report(f"recorded composites {sorted(shapes.items(), key=str)}", t0, worst)
    for tag in ("training", "eval"):
        assert {(tag, 32, None, None), (tag, 31, None, "simple"), (tag, 128, None, "simple"), (tag, 64, None, "simple")} <= set(shapes)


@pytest.mark.parametrize("training", [False, True])
@pytest.mark.parametrize("bg", C.BACKGROUNDS)
def test_rgb_renderer_mirror(bg, training):
    from neurad_studio_b200 import nerfstudio_api as NA

    t0 = time.perf_counter()
    rgb, w = C.rgb_inputs(2049, 32, 5)
    got = NA.RGBRenderer(C.background_arg(bg)).train(training)(rgb.to(DEV), w.to(DEV))
    worst = C.check_rgb_renderer(got, rgb, w, bg, training, f"RGBRenderer {bg} training={training}")
    if not training:
        assert got.max().item() == 1.0 and got.min().item() >= 0.0
    _report(f"RGBRenderer {bg} training={training}", t0, worst)


# ====================================================================================== eval-mode stage operators
@pytest.mark.parametrize("S", [1, 31, 32, 48, 128])
@pytest.mark.parametrize("kind", ["uniform", "lindisp", "power", "sqrt", "log"])
def test_spaced_sample_eval(kind, S):
    t0 = time.perf_counter()
    worst = max(C.spaced_case(DEV, 2049, S, kind, nears, seed=S) for nears in (True, False))
    _report(f"spaced {kind} S={S}", t0, worst)


@pytest.mark.parametrize("kind,S,S_new", [(k, S, Sn) for k in ("random", "degenerate", "unpadded") for S, Sn in ((33, 31), (32, 48), (64, 32), (128, 64))]
                         + [("dyadic", 32, 31), ("dyadic", 64, 63)])
def test_pdf_eval(kind, S, S_new):
    t0 = time.perf_counter()
    _report(f"pdf eval {kind} S={S} S_new={S_new}", t0, C.pdf_eval_case(DEV, 2051, S, S_new, kind, seed=S))


@pytest.mark.parametrize("S", [1, 32, 129])
@pytest.mark.parametrize("normalize", [False, True])
def test_frustum_positions(normalize, S):
    C.frustum_case(DEV, 4097, S, normalize, seed=S)


@pytest.mark.parametrize("C_", [1, 3, 16])
def test_density_rgb_heads(C_):
    t0 = time.perf_counter()
    _report(f"density_rgb_heads C={C_}", t0, C.heads_case(DEV, 65539, C_, seed=C_))


def test_sh4():
    t0 = time.perf_counter()
    _report("sh4", t0, C.sh_case(DEV, 100003))


@pytest.mark.parametrize("rows", [1, 127, 128, 129, 128 * 132 + 1])
@pytest.mark.parametrize("dims", C.MLP_DIMS)
def test_mlp_generic(dims, rows):
    t0 = time.perf_counter()
    _report(f"mlp {dims} rows={rows}", t0, C.mlp_generic_case(DEV, dims, rows))
