"""GPU: the training step's forward operators entry by entry against float64 (tests/training_forward_cases.py) on the real
library at production table sizes: isotropic_gaussian_kernel, spaced_sample_jitter_kernel, spacing_to_euclidean_kernel,
pdf_resample_kernel (training mode), neurad_encoding_fwd_kernel<4> / <1> (features, density, box-frame directions, actor
ids, the per-ray flip; 0 to 64 actors, partial 32-sample blocks), field_mid_kernel / field_tail_kernel and mlp_tc_kernel
(mlp_fwd with hidden pre-activations, mlp_dgrad), and every such call of one recorded training step at NeuRAD's batch
shape (40 960 camera + 16 384 lidar rays).  Each test prints its worst |got - ref| / tol."""
import time

import pytest

from neurad_studio_b200.lib import FIELD_MAIN, FIELD_PROP1
from tests import training_forward_cases as C

pytestmark = pytest.mark.gpu
DEV = "cuda"
_T0 = time.perf_counter()


def _report(name, t0, worst):
    print(f"\n[training forward] {name}: worst |got - ref| / tol = {worst:.3g}, {time.perf_counter() - t0:.1f} s "
          f"(file wall time so far {time.perf_counter() - _T0:.1f} s)")


@pytest.mark.parametrize("n,S", [(1, 1), (4099, 32), (513, 129), (57344, 32)])
def test_gaussian_per_entry(n, S):
    t0 = time.perf_counter()
    _report(f"gaussian n={n} S={S}", t0, C.gaussian_case(DEV, n, S, seed=S))


@pytest.mark.parametrize("kind,lam", [("uniform", -1.0), ("lindisp", -1.0), ("sqrt", -1.0), ("log", -1.0), ("power", -1.0),
                                      ("power", -1.5)])
@pytest.mark.parametrize("with_nears", [True, False])
@pytest.mark.parametrize("rand_cols", ["single", "edges"])
def test_stratified_per_entry(kind, lam, with_nears, rand_cols):
    t0 = time.perf_counter()
    _report(f"stratified {kind} lam={lam} nears={with_nears} {rand_cols}", t0,
            C.stratified_case(DEV, 1027, 128, kind, lam, with_nears, rand_cols, "random", seed=3))


@pytest.mark.parametrize("t_kind", ["zero", "max"])
@pytest.mark.parametrize("rand_cols", ["single", "edges"])
@pytest.mark.parametrize("kind,lam", [("power", -1.0), ("power", -1.5), ("log", -1.0)])
def test_stratified_jitter_extremes(kind, lam, rand_cols, t_kind):
    t0 = time.perf_counter()
    _report(f"stratified {kind} lam={lam} {rand_cols} t={t_kind}", t0, C.stratified_case(DEV, 515, 64, kind, lam, True, rand_cols, t_kind))


@pytest.mark.parametrize("kind,lam", [("uniform", -1.0), ("lindisp", -1.0), ("sqrt", -1.0), ("log", -1.0), ("power", -1.0),
                                      ("power", -1.5)])
@pytest.mark.parametrize("with_nears", [True, False])
def test_spacing_to_euclidean_per_entry(kind, lam, with_nears):
    t0 = time.perf_counter()
    _report(f"spacing_to_euclidean {kind} lam={lam} nears={with_nears}", t0,
            C.spacing_to_euclidean_case(DEV, 2049, 33, kind, lam, with_nears))


@pytest.mark.parametrize("S", [31, 32, 33, 64, 128])
@pytest.mark.parametrize("rand_cols", [1, "edges"])
@pytest.mark.parametrize("kind", ["random", "degenerate", "unpadded"])
def test_pdf_resample_per_entry(S, rand_cols, kind):
    t0 = time.perf_counter()
    _report(f"pdf {kind} S={S} cols={rand_cols}", t0, C.pdf_case(DEV, 2051, S, 64 if S == 128 else 32, rand_cols, kind, seed=S))


@pytest.mark.parametrize("S,S_new", [(32, 31), (64, 63), (128, 31)])
def test_pdf_resample_dyadic_quantiles_on_cdf_values(S, S_new):
    t0 = time.perf_counter()
    _report(f"pdf dyadic S={S} S_new={S_new}", t0, C.pdf_case(DEV, 1025, S, S_new, 1, "dyadic", seed=S))


@pytest.mark.parametrize("S", [1, 31, 32, 33, 128])
@pytest.mark.parametrize("n_actors", [0, 6, 31, 64])
@pytest.mark.parametrize("field", [FIELD_MAIN, FIELD_PROP1])
def test_encoding_per_entry(field, n_actors, S):
    t0 = time.perf_counter()
    n = 2053 if S <= 33 else 517
    worst, faces = C.encoding_case(DEV, field, n_actors, n, S, "mixed" if n_actors else "none", seed=S)
    _report(f"encoding field={field} actors={n_actors} S={S} ({faces} face exceptions)", t0, worst)


@pytest.mark.parametrize("flip", ["plus", "minus", "mixed"])
@pytest.mark.parametrize("dirs_per_ray", [True, False])
def test_encoding_flip_and_directions(flip, dirs_per_ray):
    t0 = time.perf_counter()
    worst, faces = C.encoding_case(DEV, FIELD_MAIN, 31, 1029, 33, flip, dirs_per_ray=dirs_per_ray, seed=7)
    _report(f"encoding flip={flip} dirs_per_ray={dirs_per_ray} ({faces} face exceptions)", t0, worst)


@pytest.mark.parametrize("G", [15, 32, 127])
@pytest.mark.parametrize("n", [1, 127, 128, 129, 1835008])
def test_field_mid_tail_per_entry(n, G):
    if n > 200000 and G != 32:
        pytest.skip("the production row count runs at NeuRAD's width")
    t0 = time.perf_counter()
    _report(f"field mid / tail n={n} G={G}", t0, C.field_case(DEV, n, G, seed=G))


@pytest.mark.parametrize("rows", [1, 127, 128, 129, 1835008])
@pytest.mark.parametrize("which", ["geo", "feature"])
def test_mlp_per_entry(which, rows):
    t0 = time.perf_counter()
    _report(f"mlp_{which} rows={rows}", t0, C.mlp_case(DEV, which, rows))


def test_recorded_training_step():
    t0 = time.perf_counter()
    worst, faces, n = C.check_recorded_step(DEV, 40960, 16384)
    print(f"\n[training forward] recorded step ({n} calls, {faces} face exceptions, {time.perf_counter() - t0:.1f} s): "
          + ", ".join(f"{k} {v:.3g}" for k, v in sorted(worst.items())))
