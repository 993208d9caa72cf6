"""Bodies of the entry-by-entry tests of the generic stage operators behind the C ABI: composite_kernel with
depth_clip_kernel (values, accumulation and the simple / expected / median depth of FeatureRenderer, RGBRenderer,
AccumulationRenderer, DepthRenderer and the module walk's _composite), and the eval-mode operators of the module walk and
of BASELINE config 1: spaced_sample_kernel, pdf_resample_kernel without `rand`, frustum_positions_kernel,
density_rgb_heads_kernel, sh4_fwd_kernel and mlp_tc_kernel on shapes other than NeuRAD's.  Shared by
tests/test_zz_stage_ops_gpu.py (dev = "cuda": the real library) and tests/test_stage_ops_cpu.py (dev = "cpu":
tests/fake_backend.py, whose stand-ins are torch restatements: there the tests check the references and the bounds).

Reference: the same formula in float64 on the kernel's fp32 inputs.  Bounds per entry from the kernel's op sequence
(one fp32 rounding <= U = 2^-24 of its result, expf <= 2 ulp, a sum of n terms in any order <= n U of the sum of
|terms|), first order, in the style of tests/ray_ops_cases.py.  Nothing is scaled to a tensor's maximum.  Results that
are one IEEE operation sequence the test can repeat in fp32 (the sample mids, the median's sample, the clip bounds,
frustum positions) are compared bit for bit."""
import inspect

import numpy as np
import torch

from oracle import simple_oracle as SO
from tests import render_trace_cases as RT
from tests import training_forward_cases as TF
from tests.ray_ops_cases import F32_EXP_MAX, TINY, U, _bits_equal, _ratio

FLT_MAX = float(np.finfo(np.float32).max)
F32_OVERFLOW = 2.0 ** 128 - 2.0 ** 103  # round-to-nearest gives inf from here up
EPS_DEPTH = TF.f32(1e-10)  # DepthRenderer("expected")'s 1e-10, as the kernel's 1e-10f
_dv = TF._dv


def backend(dev):
    return TF.backend(dev)


# ====================================================================================== composite: references
def mids32(starts, ends):
    """fl(fl(start + end) / 2): the kernel's sample mid, and the reference's steps on fp32 frustums."""
    return (starts.float() + ends.float()) / 2


def median_index(w):
    """DepthRenderer("median")'s index: torch's CPU cumsum of fp32 weights accumulates in float64 and rounds each running
    sum to fp32; searchsorted(side="left") of 0.5 counts the running sums below 0.5; clamped to S - 1.  Exact when the
    float64 running sums are (weights on a 2^-k grid)."""
    cs = torch.cumsum(w.double(), 1).float()
    return (cs < 0.5).sum(1).clamp_max(w.shape[1] - 1)


def composite_reference(w, v, starts, ends, depth_method, bg, nan_to_num):
    """float64 outputs on the kernel's fp32 inputs (on their device) with their bounds:
      acc = sum w:                           E_acc = (S - 1) U sum |w|  (lane partials, then the warp tree)
      t = sum fl(w x):                       E_t = S U sum |w x|        (x = nan_to_num(v) in fp32 when asked)
      with a background: fl(t + fl(bg fl(1 - acc))):
                                             E = E_t + |bg| (E_acc + U |1 - acc|) + U |bg (1 - acc)| + U |out|
      simple depth = sum fl(w mid):          S U sum |w mid|
      expected = fl(dsum / fl(acc + 1e-10f)) (training_forward_cases' _E chain), clipped afterwards
      median: the mid at median_index (exact).
    Returns {name: (ref, tol)}, plus "sum_abs" of the values' terms (to tell overflow apart) and "mids"."""
    w64 = w.double()
    n, S = w64.shape
    acc = w64.sum(1)
    E_acc = (S - 1) * U * w64.abs().sum(1)
    out = {"accumulation": (acc, E_acc)}
    if v is not None:
        x = v.reshape(n, S, -1)
        x = (torch.nan_to_num(x) if nan_to_num else x).double()
        terms = w64[..., None] * x
        t = terms.sum(1)
        E = S * U * terms.abs().sum(1)
        out["sum_abs"] = terms.abs().sum(1)
        if bg is not None:
            b = torch.tensor([TF.f32(c) for c in bg], dtype=torch.float64, device=w.device)
            om = (1 - acc)[:, None]
            bt = b * om
            t = t + bt
            E = E + b.abs() * (E_acc[:, None] + U * om.abs()) + U * bt.abs() + U * t.abs()
        out["values"] = (t, E)
    if depth_method is not None:
        m32 = mids32(starts, ends).reshape(n, S)
        m = m32.double()
        out["mids"] = m32
        if depth_method == "median":
            idx = median_index(w.reshape(n, S))
            d = m32.gather(1, idx[:, None])[:, 0]
            out["depth"] = (d.double(), torch.zeros_like(acc))
        else:
            dt = w64 * m
            dsum = TF._E(dt.sum(1), S * U * dt.abs().sum(1))
            if depth_method == "simple":
                out["depth"] = (dsum.v, dsum.e)
            else:
                den = TF.e_add(TF._E(acc, E_acc), TF.const(EPS_DEPTH, acc))
                d = TF.e_div(dsum, den)
                out["depth"] = (d.v, d.e)
    return out


def _same_value(got, ref):
    """Bit for bit, except that a zero may carry either sign (fminf / fmaxf on +-0 may return either)."""
    got, ref = got.contiguous(), ref.contiguous()
    gi, ri = got.view(torch.int32), ref.view(torch.int32)
    return (gi == ri) | ((got == 0) & (ref == 0))


def check_values(got, ref, tol, sum_abs, what):
    """Per entry; a NaN or inf of the float64 reference (an inf or NaN input without nan_to_num, 0 * inf) must come back
    the same; a finite reference beyond fp32's range (|ref| - tol past the overflow threshold) must come back as the
    signed inf; where no partial sum can overflow (sum |w x| and the bound stay below FLT_MAX) the entry is held to its bound.
    Entries between the two (a partial sum may or may not overflow) must not be NaN."""
    g = got.detach().cpu().double().reshape(ref.shape)
    ref, tol, sum_abs = ref.cpu(), tol.cpu(), sum_abs.cpu()
    nf = ~torch.isfinite(ref)
    bad = nf & ~((g.isnan() & ref.isnan()) | (g == ref))
    assert not bad.any(), f"{what}: {int(bad.sum())} non-finite entries differ from the reference, first at {bad.nonzero()[:3].tolist()}"
    ovf = ~nf & (ref.abs() - tol > F32_OVERFLOW)
    bad = ovf & (g != torch.sign(ref) * float("inf"))
    assert not bad.any(), f"{what}: {int(bad.sum())} entries beyond fp32's range did not overflow"
    fin = ~nf & (sum_abs * (1 + 1e-5) + tol < FLT_MAX)
    mid = ~nf & ~ovf & ~fin
    assert not g[mid].isnan().any(), f"{what}: NaN near fp32's overflow threshold"
    return _ratio(g, ref, tol, what, mask=fin)


def check_expected_depth(got, d, E, mids, what):
    """The clip's range is the exact fp32 min / max of all mids of the call.  A ray whose float64 depth +- bound lies
    below / above it must equal the bound bit for bit; a ray inside it is held to its bound; a ray that straddles an edge
    may take the edge or a value within its bound.  Returns (worst, rays clipped low, rays clipped high)."""
    lo, hi = mids.min().cpu(), mids.max().cpu()
    g32 = got.detach().cpu().float().reshape(-1)
    g = g32.double()
    d, E = d.cpu(), E.cpu()
    below, above = d + E < lo.double(), d - E > hi.double()
    inside = (d - E >= lo.double()) & (d + E <= hi.double())
    for m, b, name in ((below, lo, "low"), (above, hi, "high")):
        ok = _same_value(g32[m], b.expand(int(m.sum())))
        assert ok.all(), f"{what}: {int((~ok).sum())} rays outside the batch range not clipped to its {name} end ({b.item():.9g}), e.g. got {g32[m][~ok][:3].tolist()}"
    strad = ~below & ~above & ~inside
    on_edge = (g32 == lo) | (g32 == hi)
    near = (g - d).abs() <= E + TINY
    ok = (g >= lo.double()) & (g <= hi.double()) & (on_edge | near)
    assert ok[strad].all(), f"{what}: a ray at the edge of the batch range took neither the edge nor its own depth"
    return _ratio(g, d, E + TINY, what, mask=inside), int(below.sum()), int(above.sum())


def check_composite(out, w, v, starts, ends, depth_method, bg, nan_to_num, what):
    """Every output of one composite call against composite_reference, from the call's own arguments (tensors on any
    device; the float64 reference runs on theirs).  Returns {"worst": ..., "clipped": (low, high)}."""
    n, S = w.shape[0], w.shape[1]
    w = w.reshape(n, S)
    st = None if starts is None else starts.reshape(n, S)
    en = None if ends is None else ends.reshape(n, S)
    ref = composite_reference(w, v, st, en, depth_method, bg, nan_to_num)
    worst, clipped = 0.0, (0, 0)
    if "accumulation" in out:
        a, Ea = ref["accumulation"]
        worst = max(worst, _ratio(out["accumulation"], a.cpu(), Ea.cpu() + TINY, what + " accumulation"))
    if v is not None:
        t, E = ref["values"]
        worst = max(worst, check_values(out["values"], t, E + TINY, ref["sum_abs"], what + " values"))
    if depth_method is not None:
        d, E = ref["depth"]
        if depth_method == "median":
            _bits_equal(out["depth"].reshape(-1), d.float().cpu(), what + " median depth")
        elif depth_method == "simple":
            worst = max(worst, _ratio(out["depth"], d.cpu(), E.cpu() + TINY, what + " simple depth"))
        else:
            wr, lo, hi = check_expected_depth(out["depth"], d, E, ref["mids"], what + " expected depth")
            worst, clipped = max(worst, wr), (lo, hi)
    return {"worst": worst, "clipped": clipped}


# ====================================================================================== composite: inputs
def grid_weights(n, S, gen, k=24):
    """Weights on the 2^-k grid (torch.rand's for k = 24): every float64 running sum is exact, so the kernel's
    tree-ordered scan and torch's sequential cumsum have one answer."""
    return torch.floor(torch.rand(n, S, generator=gen) * 2.0 ** k) / 2.0 ** k


def composite_inputs(n, S, C, seed, kind="random"):
    """weights [n, S], values [n, S, C], starts / ends [n, S].  Rows cycle through: all-zero weights, a single 1, rows
    summing to more than 1, 1e-30 next to O(1) weights (not on the grid; they cannot move a median: a running sum of
    grid weights is never within 1e-30 of an fp32 rounding boundary), and random grid weights (which reach 0.5 at some
    sample about half the time).  Steps: increasing edges from a random (some negative) start.  kind "specials" puts
    NaN, +-inf (also at weight 0) and FLT_MAX into the values and the median's edge cases into the weights."""
    gen = torch.Generator().manual_seed(seed)
    w = grid_weights(n, S, gen) * (1.0 / S) * 2
    k = torch.arange(n) % 6
    w[k == 0] = 0.0
    if S > 1:
        w[k == 1] = 0.0
        w[k == 1, torch.randint(0, S, (int((k == 1).sum()),), generator=gen)] = 1.0
    w[k == 2] *= 2.5
    tiny = (k == 3)
    if tiny.any():
        w[tiny] = torch.where(torch.rand(int(tiny.sum()), S, generator=gen) < 0.5, torch.full((int(tiny.sum()), S), 1e-30), w[tiny])
    w0 = torch.rand(n, 1, generator=gen) * 200 - 100
    edges = w0 + torch.cumsum(torch.rand(n, S + 1, generator=gen) * 2 + 0.01, 1)
    v = torch.randn(n, S, C, generator=gen) * 2
    if kind == "specials":
        v[0::7, 0, 0] = float("nan")
        v[1::7, S // 2, C - 1] = float("inf")
        v[2::7, S - 1, C // 2] = -float("inf")
        v[3::7, :, 0] = FLT_MAX
        v[4::7, 0, C - 1] = float("inf")
        w[4::7, 0] = 0.0  # inf at weight 0: NaN without nan_to_num, 0 with it
        w[3::7, :] = 0.0
        w[3::7, 0] = 0.5  # FLT_MAX * w: finite
        if S > 1:
            w[3::14, 1] = 0.75  # 1.25 FLT_MAX: overflows
        w[5::7] = 0.0
        w[5::7, S // 2] = 0.5  # the running sum reaches 0.5 exactly at sample S // 2
    if n > 6 and S > 1:  # mids of -0.0 and +0.0
        starts, ends = edges[:, :-1].clone(), edges[:, 1:].clone()
        starts[6, :2], ends[6, :2] = torch.tensor([-0.0, -1.5]), torch.tensor([-0.0, 1.5])
        return w.contiguous(), v.contiguous(), starts, ends
    return w.contiguous(), v.contiguous(), edges[:, :-1].contiguous(), edges[:, 1:].contiguous()


def median_cases(S):
    """Weight rows [m, S] for the median's edges (all on a 2^-k grid) and the index each must give:
      running sum exactly 0.5 at sample k -> k;
      (0.5 - 2^-25, 3 2^-27, 0.25, ...): the float64 running sum after two samples, 0.5 - 2^-27, rounds to 0.5 in fp32 ->
        index 1 (a float64 comparison would give 2);
      a total below 0.5 -> S - 1; a first weight >= 0.5 -> 0; all zeros -> S - 1;
      the crossing at samples 31 and 32 (the seam of the 32-sample chunks)."""
    rows, want = [], []

    def add(vals, idx):
        r = torch.zeros(S)
        r[: len(vals)] = torch.tensor(vals[:S], dtype=torch.float32)
        rows.append(r)
        want.append(min(idx, S - 1))

    add([0.0] * S, S - 1)
    add([0.125] * min(S, 3), S - 1)  # total 0.375
    add([0.5, 0.25], 0)
    add([0.75], 0)
    if S >= 3:
        add([0.5 - 2.0 ** -25, 3 * 2.0 ** -27, 0.25], 1)
        add([0.25, 0.125, 0.125, 0.25][:S], 2)  # exactly 0.5 at sample 2
    g = 2.0 ** -6
    if S > 31:
        add([g] * 32, 31)  # 32 * 2^-6 = 0.5 exactly at the last sample of the first chunk
        add([0.5 - 2.0 ** -25] + [0.0] * 30 + [3 * 2.0 ** -27], 31)  # rounds to 0.5 at sample 31
    if S > 32:
        add([0.0] + [g] * 32, 32)  # 0.5 exactly at the first sample of the second chunk
        add([0.5 - 2.0 ** -25] + [0.0] * 31 + [2.0 ** -25], 32)
        add([0.5 - 2.0 ** -25] + [0.0] * 31 + [3 * 2.0 ** -27], 32)
    return torch.stack(rows), torch.tensor(want)


def composite_call(be, dev, w, v, st, en, depth_method, bg=None, nan_to_num=False, want_acc=True):
    d = _dv(dev)
    return be.composite(w.to(d), None if v is None else v.to(d), None if st is None else st.to(d), None if en is None else en.to(d),
                        depth_method, background=bg, value_nan_to_num=nan_to_num, want_accumulation=want_acc)


def composite_case(dev, n, S, C, depth_method, bg=False, nan_to_num=False, kind="random", seed=0, be=None):
    be = be or backend(dev)
    w, v, st, en = composite_inputs(n, S, C, seed, kind)
    b = [0.25 * (i % 5) - 0.25 for i in range(C)] if bg else None
    out = composite_call(be, dev, w, v, st, en, depth_method, b, nan_to_num)
    d = _dv(dev)
    return check_composite(out, w.to(d), v.to(d), st.to(d), en.to(d), depth_method, b, nan_to_num,
                           f"composite n={n} S={S} C={C} depth={depth_method} bg={bg} nan_to_num={nan_to_num} {kind}")


def median_case(dev, S, n_pad=0, be=None):
    """median_cases' rows (with n_pad random grid rows after them), negative mids on half the rows, each row's index
    checked against its expected value and the whole call through check_composite."""
    be = be or backend(dev)
    rows, want = median_cases(S)
    gen = torch.Generator().manual_seed(S)
    w = torch.cat([rows, grid_weights(n_pad, S, gen) * (2.0 / S)])
    n = w.shape[0]
    edges = torch.cumsum(torch.rand(n, S + 1, generator=gen) + 0.01, 1) - 3.0 * (torch.arange(n) % 2)[:, None] * S
    st, en = edges[:, :-1].contiguous(), edges[:, 1:].contiguous()
    assert torch.equal(median_index(rows), want), "median_cases' expected indices disagree with the reference"
    out = composite_call(be, dev, w, None, st, en, "median", want_acc=True)
    what = f"median S={S}"
    r = check_composite(out, w.to(_dv(dev)), None, st.to(_dv(dev)), en.to(_dv(dev)), "median", None, False, what)
    _bits_equal(out["depth"].reshape(-1)[: rows.shape[0]], mids32(st, en)[torch.arange(rows.shape[0]), want].contiguous(),
                what + " edge cases")
    return r["worst"]


def clip_case(dev, n, S, be=None):
    """Expected depth's batch-global clip: rays of zero weights (depth 0) and of tiny total weight (depth pulled towards
    0) outside the range; the batch minimum on a zero-weight ray; a second call with a disjoint, all-negative range
    (its zero-weight rays must clip to its own high end, not to the first call's).  Returns the clipped counts."""
    be = be or backend(dev)
    gen = torch.Generator().manual_seed(n + S)
    res = []
    for base in (100.0, -400.0):
        w = grid_weights(n, S, gen) * (1.0 / S)
        edges = base + torch.cumsum(torch.rand(n, S + 1, generator=gen) + 0.01, 1)
        w[0::4] = 0.0
        w[1::4] = 2.0 ** -40
        edges[0] -= 50.0  # the batch minimum sits on a zero-weight ray
        st, en = edges[:, :-1].contiguous(), edges[:, 1:].contiguous()
        out = composite_call(be, dev, w, None, st, en, "expected")
        r = check_composite(out, w, None, st, en, "expected", None, False, f"expected clip n={n} S={S} base={base}")
        lo, hi = r["clipped"]
        assert (lo if base > 0 else hi) >= n // 4, f"the case clips too few rays ({r['clipped']})"
        res.append((out, w, st, en))
    return res


# ====================================================================================== RGBRenderer
def rgb_inputs(n, S, seed):
    """rgb = rand * 1.5 (out of [0, 1]) with NaN / +-inf entries, weights summing to more than 1 on some rays."""
    gen = torch.Generator().manual_seed(seed)
    rgb = torch.rand(n, S, 3, generator=gen) * 1.5
    w = torch.rand(n, S, 1, generator=gen) * (3.0 / S)
    w[0::3] *= 0.1
    rgb[1, 2, 0] = float("nan")
    rgb[2, 0, 1] = float("inf")
    rgb[4, 1, 2] = -float("inf")
    return rgb, w


BACKGROUNDS = ("black", "white", "random", "tensor")


def background_arg(name):
    return torch.tensor([0.2, 0.5, 0.9]) if name == "tensor" else name


def background_values(name):
    return {"black": [0.0, 0.0, 0.0], "white": [1.0, 1.0, 1.0], "random": None, "tensor": [0.2, 0.5, 0.9]}[name]


def check_rgb_renderer(got, rgb, w, bg_name, training, what):
    """The mirror's RGBRenderer (eval: nan_to_num, composite, clamp to [0, 1]; training: the composite alone) per entry:
    composite_reference's bound, which the clamp (1-Lipschitz) keeps."""
    n, S = w.shape[0], w.shape[1]
    ref = composite_reference(w.reshape(n, S).to(got.device), rgb.to(got.device), None, None, None, background_values(bg_name), not training)
    t, E = ref["values"]
    if not training:
        t = t.clamp(0.0, 1.0)
    return check_values(got, t, E + TINY, ref["sum_abs"], what)


# ====================================================================================== eval-mode stage operators
def spaced_case(dev, n, S, kind, with_nears, seed=0):
    """SpacedSampler eval: bins_s bit for bit against torch.linspace for power-of-two S (else within linspace01's 3 U);
    bins_e through training_forward_cases.check_euclid on the kernel's bins."""
    be = backend(dev)
    gen = torch.Generator().manual_seed(seed)
    nears = torch.rand(n, generator=gen) * 2 + 0.05
    fars = nears + torch.exp(torch.rand(n, generator=gen) * 9)
    fars[0] = 20000.0
    scaling = TF.f32(0.1)
    v = _dv(dev)
    bs, b_e = be.spaced_sample(nears.to(v) if with_nears else None, fars.to(v), S, kind, -1.0, scaling)
    what = f"spaced {kind} S={S} nears={with_nears}"
    lin = torch.linspace(0.0, 1.0, S + 1)
    if S & (S - 1) == 0:
        _bits_equal(bs, lin, what + " bins_s")
    else:
        _ratio(bs, torch.arange(S + 1, dtype=torch.float64) / S, torch.full((S + 1,), 3 * U), what + " bins_s")
    u = bs.detach().cpu().float()[None].expand(n, S + 1).contiguous()
    return TF.check_euclid(b_e, u, nears if with_nears else None, fars, kind, -1.0, scaling, what + " bins_e")


def pdf_eval_case(dev, n, S, S_new, kind, seed=0):
    """PDFSampler eval (no rand): training_forward_cases.check_pdf with the eval quantiles the kernel receives."""
    from neurad_studio_b200.backend import pdf_quantiles

    be = backend(dev)
    w, bins, _ = TF.pdf_inputs(n, S, S_new, kind, 1, seed)
    hp = 0.0 if kind in ("dyadic", "unpadded") else 0.01
    v = _dv(dev)
    out = be.pdf_resample(w.to(v), bins.to(v), S_new, histogram_padding=hp)
    uu = pdf_quantiles(S_new)[None].expand(n, S_new + 1).contiguous()
    return TF.check_pdf(out, w, bins, S_new, None, hp, f"pdf eval {kind} S={S} S_new={S_new}", u=uu)


def frustum_reference(o, d, b_e, aabb=None):
    """Frustums.get_positions (+ SceneBox.get_normalized_positions) in fp32 IEEE operations: o + fl(fl(d fl(s + e)) / 2),
    then fl(fl(p - lo) / fl(hi - lo)) -- the kernel's sequence (the oracle's restatements)."""
    o, d, b_e = o.float().cpu(), d.float().cpu(), b_e.float().cpu()
    p = SO.frustum_positions(o, d, b_e[:, :-1, None], b_e[:, 1:, None])
    return p if aabb is None else SO.normalized_positions(p, aabb.float().cpu())


def frustum_case(dev, n, S, normalize, seed=0):
    be = backend(dev)
    gen = torch.Generator().manual_seed(seed)
    o = torch.randn(n, 3, generator=gen) * 30
    d = torch.nn.functional.normalize(torch.randn(n, 3, generator=gen), dim=-1)
    b_e = torch.cumsum(torch.rand(n, S + 1, generator=gen) * 3, 1) + 0.05
    aabb = torch.tensor([[-80.0, -60.5, -7.25], [90.0, 61.0, 13.0]]) if normalize else None
    v = _dv(dev)
    got = be.frustum_positions(o.to(v), d.to(v), b_e.to(v), aabb)
    _bits_equal(got, frustum_reference(o, d, b_e, aabb), f"frustum n={n} S={S} aabb={normalize}")
    return 0.0


def heads_reference(raw):
    """density = expf(v): 2 ulp (4 U relative, 2 TINY in the denormal range), inf where exp(v) overflows fp32;
    rgb = fl(1 / fl(1 + expf(-v))): 6 U relative, exactly 0 where expf(-v) overflows (v < -88.72), as the fp32 formula and
    torch.sigmoid on the CPU give.  Returns (density, tol, rgb, tol, entries held exactly to 0 / inf)."""
    r = raw.double().cpu()
    dens = r[:, 0].exp()
    Ed = 4 * U * dens + 2 * TINY
    x = r[:, 1:]
    rgb = 1 / (1 + (-x).exp())
    Er = 6 * U * rgb + TINY
    return dens, Ed, rgb, Er


def check_heads(density, rgb, raw, what):
    dens, Ed, ref, Er = heads_reference(raw)
    r = raw.double().cpu()
    g = density.detach().cpu().reshape(-1)
    ovf = r[:, 0] > F32_EXP_MAX + 1e-5
    fin = r[:, 0] < F32_EXP_MAX - 1e-5
    assert torch.isinf(g[ovf]).all() and (g[ovf] > 0).all(), f"{what}: density of v > 88.72 is not inf"
    worst = _ratio(g, dens, Ed, what + " density", mask=fin)
    gr = rgb.detach().cpu().reshape(ref.shape)
    zero = -r[:, 1:] > F32_EXP_MAX + 1e-5
    assert (gr[zero] == 0).all(), f"{what}: sigmoid where expf(-v) overflows is not exactly 0"
    keep = -r[:, 1:] < F32_EXP_MAX - 1e-5
    return max(worst, _ratio(gr, ref, Er, what + " rgb", mask=keep))


def heads_inputs(n, C, seed):
    gen = torch.Generator().manual_seed(seed)
    raw = torch.randn(n, C + 1, generator=gen) * 8
    ends = torch.tensor([-200.0, -104.0, -89.0, -88.7, -87.5, 0.0, 87.5, 88.7, 88.73, 89.0, 104.0, 200.0])
    raw[: len(ends), 0] = ends[:n]
    for c in range(1, C + 1):
        raw[: len(ends), c] = ends.roll(c)[:n]
    return raw


def heads_case(dev, n, C, seed=0):
    be = backend(dev)
    raw = heads_inputs(n, C, seed)
    density, rgb = be.density_rgb_heads(raw.to(_dv(dev)))
    return check_heads(density, rgb, raw, f"density_rgb_heads n={n} C={C}")


SH_TOL = 72 * U  # render_trace_cases._sh4_64: degree <= 3 polynomials with terms <= 3 in [-1, 1]^3, <= 24 U each


def sh_inputs(n, seed):
    """Unit directions, their (d + 1) / 2, the corners of [-1, 1]^3 and of [0, 1]^3, and the axes."""
    gen = torch.Generator().manual_seed(seed)
    d = torch.nn.functional.normalize(torch.randn(n, 3, generator=gen), dim=-1)
    corners = torch.tensor([[x, y, z] for x in (-1.0, 1.0) for y in (-1.0, 1.0) for z in (-1.0, 1.0)])
    axes = torch.cat([torch.eye(3), -torch.eye(3)])
    return torch.cat([d, (d + 1) / 2, corners, (corners + 1) / 2, axes])


def check_sh(got, dirs, what):
    ref = RT._sh4_64(dirs.double().cpu())
    return _ratio(got.reshape(ref.shape), ref, torch.full_like(ref, SH_TOL), what)


def sh_case(dev, n, seed=0):
    be = backend(dev)
    dirs = sh_inputs(n, seed)
    return check_sh(be.sh4_fwd(dirs.to(_dv(dev))), dirs, f"sh4 n={dirs.shape[0]}")


MLP_DIMS = ((32, 64, 4), (64, 64, 64, 64), (50, 57, 3), (40, 24, 17))


def mlp_generic_case(dev, dims, rows, seed=0):
    """mlp_fwd (output, then want_hidden: the same output and the hidden pre-activations) and mlp_dgrad of the last layer
    with and without the ReLU mask, through training_forward_cases.check_mlp / check_dgrad (gamma_tc)."""
    be = backend(dev)
    gen = torch.Generator().manual_seed(sum(dims) + rows + seed)
    ws, bs = [], []
    for i in range(len(dims) - 1):
        bound = 1.0 / dims[i] ** 0.5
        ws.append((torch.rand(dims[i + 1], dims[i], generator=gen) * 2 - 1) * bound * 3)
        bs.append((torch.rand(dims[i + 1], generator=gen) * 2 - 1) * bound)
    x = torch.randn(rows, dims[0], generator=gen)
    v = _dv(dev)
    ref_dev = "cuda" if dev == "cuda" else "cpu"
    wv, bv = [w.to(v) for w in ws], [b.to(v) for b in bs]
    what = f"mlp {'-'.join(map(str, dims))} rows={rows}"
    y = be.mlp_fwd(x.to(v), wv, bv)
    worst = TF.check_mlp((y, []), x, ws, bs, ref_dev, what)
    y2, zs = be.mlp_fwd(x.to(v), wv, bv, want_hidden=True)
    _bits_equal(y2, y.detach().cpu(), what + " want_hidden output")
    worst = max(worst, TF.check_mlp((y2, zs), x, ws, bs, ref_dev, what + " want_hidden"))
    dy = torch.randn(rows, dims[-1], generator=gen)
    worst = max(worst, TF.check_dgrad(be.mlp_dgrad(dy.to(v), wv[-1]), dy, ws[-1], None, ref_dev, what))
    return max(worst, TF.check_dgrad(be.mlp_dgrad(dy.to(v), wv[-1], zs[-1]), dy, ws[-1], zs[-1], ref_dev, what + " masked"))


# ====================================================================================== recorded calls
def _composite_args(be, a, k):
    sig = inspect.signature(type(be).composite)
    ba = sig.bind(be, *a, **k)
    ba.apply_defaults()
    return ba.arguments


def check_recorded_composite(be, a, k, out, what="recorded composite"):
    """One recorded composite call judged from its own arguments."""
    p = _composite_args(be, a, k)
    w = p["weights"]
    n, S = w.shape[0], w.shape[1]
    r = check_composite(out, w.reshape(n, S), p["values"], p["starts"], p["ends"], p["depth_method"], p["background"],
                        p["value_nan_to_num"], what + f" S={S} C={0 if p['values'] is None else p['values'].shape[-1]} depth={p['depth_method']}")
    return r["worst"], (S, None if p["values"] is None else p["values"].shape[-1], p["depth_method"])


def record_eval_outputs(dev, n_cam, n_lidar, methods, seed=0):
    """model.eval(); get_nff_outputs(fused=False) under no_grad on training_forward_cases' scene; the calls of `methods`."""
    from neurad_studio_b200 import nerfstudio_api as NA
    from neurad_studio_b200 import scene

    cfg, trajs, params = TF.training_scene(dev, seed=seed)
    v = _dv(dev)
    model = NA.NeuRADModel(cfg, trajs).to(v)
    model.load_reference_state_dict(params)
    model.eval()
    rays = scene.random_rays(n_cam + n_lidar, cfg, seed=seed + 3, trajectories=trajs)
    is_lidar = torch.zeros(n_cam + n_lidar, 1, dtype=torch.bool)
    is_lidar[n_cam:] = True
    rb = NA.RayBundle(origins=rays["origins"].to(v), directions=rays["directions"].to(v), pixel_area=rays["pixel_area"].to(v),
                      times=rays["times"].to(v), metadata={"is_lidar": is_lidar.to(v), "sensor_idxs": rays["sensor_idx"].to(v)})
    orig = NA.get_backend
    if dev == "cpu":
        fake = backend(dev)
        NA.get_backend = lambda device: fake
    try:
        be = model._bind()
        with TF.Recorder(be, methods) as rec, torch.no_grad():
            model.get_nff_outputs(rb, fused=False)
    finally:
        NA.get_backend = orig
    return be, rec.calls


def check_recorded_composites(dev, n_cam, n_lidar, seed=0):
    """Every composite call of one training step (forward and backward) and of one eval-mode module walk.  Returns
    (worst, {(S, C, depth_method): count})."""
    _, _, be, calls = TF.record_training_step(dev, n_cam, n_lidar, seed, methods=("composite",))
    _, ecalls = record_eval_outputs(dev, n_cam, n_lidar, ("composite",), seed)
    worst, shapes = 0.0, {}
    for tag, cs in (("training", calls), ("eval", ecalls)):
        assert cs, f"the {tag} module walk made no composite call"
        for _, a, k, out in cs:
            w, shp = check_recorded_composite(be, a, k, out, f"recorded {tag} composite")
            worst = max(worst, w)
            shapes[(tag,) + shp] = shapes.get((tag,) + shp, 0) + 1
    return worst, shapes
