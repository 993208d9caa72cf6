"""CPU: the entry-by-entry checks of the generic stage operators (tests/stage_ops_cases.py) over tests/fake_backend.py,
whose stand-ins are torch restatements: here the tests check the references and the bounds; the kernels are checked on
the GPU (test_zz_stage_ops_gpu.py).  Also: the comparator self-tests (each rejects a corrupted copy of a correct
result), the median's semantics pinned to torch's CPU cumsum, PDFSampler's eval quantiles pinned to the reference's
formula, and RGBRenderer (oracle and mirror) pinned bit for bit to the reference's in eval and training mode."""
import re

import numpy as np
import pytest
import torch

from neurad_studio_b200.backend import pdf_quantiles
from oracle import ref_import
from oracle import simple_oracle as SO
from tests import stage_ops_cases as C

DEV = "cpu"
needs_reference = pytest.mark.skipif(not ref_import.reference_available(), reason="the reference tree is not present")


def _report(name, worst):
    print(f"\n[stage ops] {name}: worst |got - ref| / tol = {worst:.3g}")


def _rejected(fn, min_ratio=10.0):
    """fn must fail its comparator: a bit mismatch, or a ratio far above 1."""
    with pytest.raises(AssertionError) as e:
        fn()
    m = re.search(r"/ tol = ([0-9.e+-]+|inf|nan)", str(e.value))
    if m is not None:
        r = float(m.group(1))
        assert not r <= min_ratio, f"rejected with a ratio of only {r}: {e.value}"
    print(f"\n[stage ops] rejected: {str(e.value).splitlines()[0][:160]}")
    return str(e.value)


# ====================================================================================== composite over the stand-in
@pytest.mark.parametrize("S,C_", [(1, 1), (7, 3), (33, 9), (64, 33)])
@pytest.mark.parametrize("depth", ["simple", "expected", "median"])
def test_composite_per_entry(S, C_, depth):
    r = C.composite_case(DEV, 13, S, C_, depth, bg=S % 2 == 1, nan_to_num=True)
    _report(f"composite S={S} C={C_} {depth}", r["worst"])


@pytest.mark.parametrize("nan_to_num", [True, False])
@pytest.mark.parametrize("bg", [True, False])
def test_composite_specials(nan_to_num, bg):
    C.composite_case(DEV, 29, 33, 9, "simple", bg=bg, nan_to_num=nan_to_num, kind="specials")


@pytest.mark.parametrize("S", [1, 3, 32, 33, 129])
def test_median_edges(S):
    C.median_case(DEV, S, n_pad=5)


def test_expected_depth_clip():
    C.clip_case(DEV, 12, 33)


def test_composite_rejects_65_channels():
    with pytest.raises(Exception):
        C.backend(DEV).composite(torch.rand(2, 3), torch.rand(2, 3, 65))


def test_median_matches_torch_cumsum_semantics():
    """The reference's median (oracle/simple_oracle.depth_median: torch.cumsum of fp32 weights, searchsorted left) agrees
    with median_index on every edge case, and the (0.5 - 2^-25, 3 2^-27, 0.25) row gives 1 where a float64
    comparison would give 2."""
    for S in (3, 32, 33, 129):
        rows, want = C.median_cases(S)
        steps = torch.arange(S, dtype=torch.float32)[None].expand(rows.shape[0], S)
        got = SO.depth_median(rows[..., None], steps[..., None], steps[..., None])[:, 0].long()
        assert torch.equal(got, want) and torch.equal(C.median_index(rows), want), S
    w = torch.tensor([[0.5 - 2.0 ** -25, 3 * 2.0 ** -27, 0.25]])
    assert C.median_index(w).item() == 1
    assert int((torch.cumsum(w.double(), 1) < 0.5).sum()) == 2


# ====================================================================================== comparator self-tests
def _correct(S=33, C_=9, depth="simple", bg=True, n=10, seed=5, kind="random"):
    be = C.backend(DEV)
    w, v, st, en = C.composite_inputs(n, S, C_, seed, kind)
    b = [0.25 * (i % 5) - 0.25 for i in range(C_)] if bg else None
    return be, w, v, st, en, b, C.composite_call(be, DEV, w, v, st, en, depth, b, True)


def test_selftest_median_in_float64():
    rows, want = C.median_cases(33)
    st = torch.arange(33, dtype=torch.float32)[None].expand(rows.shape[0], 33).contiguous()
    en = st + 1
    idx64 = ((torch.cumsum(rows.double(), 1) < 0.5).sum(1)).clamp_max(32)
    got = {"depth": C.mids32(st, en).gather(1, idx64[:, None])}
    C.check_composite({"depth": C.mids32(st, en).gather(1, want[:, None])}, rows, None, st, en, "median", None, False, "ok")
    _rejected(lambda: C.check_composite(got, rows, None, st, en, "median", None, False, "median in float64"))


def test_selftest_clip_per_ray_and_previous_range():
    (_, _, st1, en1), (_, w2, st2, en2) = C.clip_case(DEV, 12, 33)
    d, E = C.composite_reference(w2, None, st2, en2, "expected", None, False)["depth"]
    m = C.mids32(st2, en2)
    per_ray = torch.minimum(torch.maximum(d.float(), m.min(1).values), m.max(1).values)
    _rejected(lambda: C.check_expected_depth(per_ray, d, E, m, "clip per ray"))
    m1 = torch.cat([m, C.mids32(st1, en1)])  # a min / max buffer not reset: the union with call 1's range
    prev = torch.minimum(torch.maximum(d.float(), m1.min()), m1.max())
    _rejected(lambda: C.check_expected_depth(prev, d, E, m, "clip from the previous call"))


def test_selftest_background_omitted():
    be, w, v, st, en, b, out = _correct()
    C.check_composite(out, w, v, st, en, "simple", b, True, "ok")
    bad = C.composite_call(be, DEV, w, v, st, en, "simple", None, True)
    _rejected(lambda: C.check_composite(bad, w, v, st, en, "simple", b, True, "background omitted"))


def test_selftest_channel_8_of_9_dropped():
    be, w, v, st, en, b, out = _correct(C_=9, bg=False)
    out["values"][:, 8] = 0.0
    _rejected(lambda: C.check_composite(out, w, v, st, en, "simple", None, True, "channel 8 dropped"))


def test_selftest_sample_32_of_33_dropped():
    be, w, v, st, en, b, out = _correct(S=33, bg=False)
    w2 = w.clone()
    w2[:, 32] = 0.0
    bad = C.composite_call(be, DEV, w2, v, st, en, "simple", None, True)
    _rejected(lambda: C.check_composite(bad, w, v, st, en, "simple", None, True, "sample 32 dropped"))


def test_selftest_nan_to_num_inf_to_zero():
    be, w, v, st, en, b, out = _correct(kind="specials", bg=False, n=29)
    v2 = torch.where(v == float("inf"), torch.zeros_like(v), v)
    bad = C.composite_call(be, DEV, w, v2, st, en, "simple", None, True)
    assert not torch.equal(bad["values"], out["values"])
    _rejected(lambda: C.check_composite(bad, w, v, st, en, "simple", None, True, "+inf to 0"))


def test_selftest_neighbouring_weights():
    be, w, v, st, en, b, out = _correct(bg=False)
    bad = C.composite_call(be, DEV, w.roll(1, 0), v, st, en, "simple", None, True)
    _rejected(lambda: C.check_composite(bad, w, v, st, en, "simple", None, True, "neighbouring weights"))


def test_selftest_missing_eval_clamp():
    rgb, w = C.rgb_inputs(8, 16, 3)
    unclamped = SO.rgb_render(torch.nan_to_num(rgb), w, torch.tensor([1.0, 1.0, 1.0]), training=True)
    C.check_rgb_renderer(SO.rgb_render(rgb, w, torch.tensor([1.0, 1.0, 1.0])), rgb, w, "white", False, "ok")
    _rejected(lambda: C.check_rgb_renderer(unclamped, rgb, w, "white", False, "missing clamp"))


def test_selftest_density_bf16():
    raw = C.heads_inputs(64, 3, 0)
    dens, rgb = C.backend(DEV).density_rgb_heads(raw)
    C.check_heads(dens, rgb, raw, "ok")
    _rejected(lambda: C.check_heads(dens.bfloat16().float(), rgb, raw, "density in bf16"))


def test_selftest_frustum_one_ulp():
    gen = torch.Generator().manual_seed(0)
    o, d = torch.randn(6, 3, generator=gen), torch.nn.functional.normalize(torch.randn(6, 3, generator=gen), dim=-1)
    b_e = torch.cumsum(torch.rand(6, 9, generator=gen), 1)
    p = C.frustum_reference(o, d, b_e).clone()
    p[4, 2, 1] = float(np.nextafter(np.float32(p[4, 2, 1]), np.float32(np.inf)))
    _rejected(lambda: C._bits_equal(p, C.frustum_reference(o, d, b_e), "frustum"))


# ====================================================================================== RGBRenderer vs the reference
@needs_reference
@pytest.mark.parametrize("training", [False, True])
@pytest.mark.parametrize("bg", C.BACKGROUNDS)
def test_rgb_renderer_matches_reference(bg, training):
    """The reference's RGBRenderer clamps to [0, 1] and applies nan_to_num in eval mode only; the oracle and the mirror
    over the stand-in backend give its result bit for bit on out-of-range colours and NaN / inf samples."""
    from neurad_studio_b200 import nerfstudio_api as NA

    ref_import.install()
    from nerfstudio.model_components.renderers import RGBRenderer

    rgb, w = C.rgb_inputs(9, 16, 1)
    ref_r = RGBRenderer(C.background_arg(bg)).train(training)
    ref = ref_r(rgb.clone(), w.clone())
    bgv = C.background_values(bg)
    got_o = SO.rgb_render(rgb, w, None if bgv is None else torch.tensor(bgv), training=training)
    orig = NA.get_backend
    fake = C.backend(DEV)
    NA.get_backend = lambda device: fake
    try:
        got_m = NA.RGBRenderer(C.background_arg(bg)).train(training)(rgb, w)
    finally:
        NA.get_backend = orig
    for got, name in ((got_o, "oracle"), (got_m, "mirror")):
        assert got.shape == ref.shape
        assert torch.equal(got.isnan(), ref.isnan()), name
        C._bits_equal(got.nan_to_num(7.0), ref.nan_to_num(7.0), f"{name} {bg} training={training}")
    if not training:
        assert ref.max().item() == 1.0 and (ref >= 0).all()


# ====================================================================================== eval-mode stage operators
def test_pdf_quantiles_match_reference_formula():
    """PDFSampler's eval u (ray_samplers.py:332-333): linspace(0, 1 - 1/nb, nb) + 1/(2 nb), bit for bit."""
    for S_new in (1, 31, 32, 48, 63, 64, 127, 128):
        nb = S_new + 1
        u = torch.linspace(0.0, 1.0 - (1.0 / nb), steps=nb)
        u = u + 1.0 / (2 * nb)
        C._bits_equal(pdf_quantiles(S_new), u, f"pdf quantiles S_new={S_new}")


@pytest.mark.parametrize("S", [1, 31, 32, 48, 128])
@pytest.mark.parametrize("kind", ["uniform", "lindisp", "power", "sqrt", "log"])
def test_spaced_sample_eval(kind, S):
    for nears in (True, False):
        _report(f"spaced {kind} S={S} nears={nears}", C.spaced_case(DEV, 7, S, kind, nears))


@pytest.mark.parametrize("kind", ["random", "degenerate", "unpadded", "dyadic"])
def test_pdf_eval(kind):
    _report(f"pdf eval {kind}", C.pdf_eval_case(DEV, 12, 32, 31 if kind == "dyadic" else 48, kind))


@pytest.mark.parametrize("normalize", [False, True])
def test_frustum_positions(normalize):
    C.frustum_case(DEV, 9, 33, normalize)


def test_density_rgb_heads():
    _report("density_rgb_heads", C.heads_case(DEV, 64, 3))


def test_sigmoid_underflow_is_zero_on_cpu():
    """Where expf(-v) overflows, the reference's fp32 sigmoid gives exactly 0."""
    v = torch.tensor([-88.73, -89.0, -104.0, -200.0])
    assert (torch.sigmoid(v) == 0).all() and (1 / (1 + torch.exp(-v)) == 0).all()
    assert torch.isinf(torch.exp(torch.tensor([88.73]))).all()


def test_sh4():
    _report("sh4", C.sh_case(DEV, 50))


@pytest.mark.parametrize("dims", C.MLP_DIMS)
def test_mlp_generic(dims):
    _report(f"mlp {dims}", C.mlp_generic_case(DEV, dims, 129))


def test_recorded_composites():
    worst, shapes = C.check_recorded_composites(DEV, 48, 24)
    print(f"\n[stage ops] recorded composites: worst {worst:.3g}, {shapes}")
