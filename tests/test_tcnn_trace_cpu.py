"""CPU: the tiny-cuda-nn-layout render stages sample by sample (tests/tcnn_trace_cases.py) over the host emulation of
the same device code (LAYOUT = 1, MlpLaneFfma), small tables, on every scene including the actor edit; the layout's
grid operator entry by entry; and the comparator's self-tests, each rejecting one deliberately wrong reference."""
import numpy as np
import pytest
import torch

from tests import render_trace_cases as C
from tests import tcnn_trace_cases as TT

DEV = "cpu"


@pytest.mark.parametrize("name", TT.CPU_SCENES)
def test_tcnn_trace_scene_sample_by_sample(name):
    TT.check_tcnn_scene(DEV, name)


def test_tcnn_grid_operator_entry_by_entry():
    TT.grid_operator_entry_by_entry(DEV)


def test_fma_pos_rounds_once():
    """fl32(x s + 0.5) with one rounding: against exact rational arithmetic on random inputs and on inputs whose double
    sum rounds (tiny x s)."""
    from fractions import Fraction

    gen = torch.Generator().manual_seed(5)
    x = torch.cat([torch.rand(400, generator=gen), torch.rand(200, generator=gen) * 1e-9, torch.tensor([0.0, 1.0])]).float()
    for s in (np.float32(7.0), np.float32(8191.0), np.float32(3.3333333)):
        got = TT.fma_pos(x, s)
        for xi, gi in zip(x.tolist(), got.tolist()):
            exact = Fraction(xi) * Fraction(float(s)) + Fraction(1, 2)
            lo = float(np.float32(float(exact)))
            cands = [np.float32(lo), np.nextafter(np.float32(lo), np.float32(-np.inf)), np.nextafter(np.float32(lo), np.float32(np.inf))]
            best = min(cands, key=lambda c: (abs(Fraction(float(c)) - exact), int(np.float32(c).view(np.int32)) & 1))
            assert gi == float(best), (xi, float(s), gi, float(best))


def test_f16_round_is_nearest_even_with_subnormals():
    t = torch.tensor([1e-7, 2.0 ** -25, 3 * 2.0 ** -25, 1.0 + 2.0 ** -11, 1.0 + 3 * 2.0 ** -11, 65504.0, -6e-5])
    got = TT.f16_round(t)
    assert got[0] == 2.0 ** -24 * round(1e-7 / 2.0 ** -24)
    assert got[1] == 0.0 and got[2] == 2 * 2.0 ** -24  # ties to even
    assert got[3] == 1.0 and got[4] == 1.0 + 2.0 ** -9
    assert got[5] == 65504.0 and got[6] == float(np.float16(-6e-5))


@pytest.fixture(scope="module")
def renders():
    out = {}
    for name in sorted(set(TT.CORRUPTIONS.values())):
        cfg, params, rays, _ = TT.scene_rays(DEV, name)
        r = C.renderer(DEV, cfg, params, TT.EDITS.get(name))
        out[name] = (cfg, params, rays, r.render(rays))
    return out


@pytest.mark.parametrize("corrupt", sorted(TT.CORRUPTIONS))
def test_comparator_rejects_a_corrupted_reference(renders, corrupt):
    """The proposal and main-field comparators accept the emulated render against the right reference and reject it,
    with a ratio above 1, against each corruption: the torch twin's SH, level weights from the tcnn grid scale, a dense
    level hashed, the wrap clamped to res - 1, the 4th coordinate a / (A - 1) or a, unrounded fp32 parameters (tables
    at 1e-4), cell-centred positions (no - 1 in the scale, or no + 0.5), level 1's offset one entry late."""
    name = TT.CORRUPTIONS[corrupt]
    cfg, params, rays, out = renders[name]
    assert TT.field_ratio_error(DEV, name, None, out, cfg, params, rays) is None
    ratio = TT.field_ratio_error(DEV, name, corrupt, out, cfg, params, rays)
    assert ratio is not None and ratio > 1.0, (corrupt, ratio)
    print(f"\n[tcnn self-test] {corrupt} on {name}: rejected at ratio {ratio:.3g}")
