"""Bodies of the entry-by-entry tests of the per-ray training operators (the weights forward and backward from alpha and
from density, composite_bwd, field_heads_bwd, relu_bwd and the mlp_dgrad ReLU mask, distortion_loss,
zipnerf_interlevel_loss, lidar_carving_mask), shared by tests/test_zz_ray_ops_gpu.py (dev = "cuda": the real library) and
tests/test_ray_ops_cpu.py (dev = "cpu": tests/fake_backend.py, whose weights backward and loss operators run the
kernels' device functions through the host emulation).

Reference: the same formula in float64 on the kernel's fp32 inputs (the oracle's functions on .double() tensors,
gradients from float64 autograd), with the fp32 constants the kernel sees (pulse widths, the 1e-5 of the interlevel
denominator, beta).  Every entry is held to its own bound, counted from the kernel's code under the standard rounding
model (one fp32 rounding <= U = 2^-24 of its result, expf <= 2 ulp <= 4 U, a sum of n terms in any order <= n U of the
sum of |terms|), first order in U; ill-conditioned steps carry their condition factor explicitly.  Nothing is scaled to
a tensor's maximum: a lost bin, a misordered knot or a neighbouring ray's row fails however small the entry is.
Operators whose result is one rounding of an exact expression (dvalues, dgeo[:, 1:], relu_bwd, the masks) are compared
bit for bit."""
import numpy as np
import torch

from oracle import losses_oracle as LO
from oracle import neurad_oracle as O

U = 2.0 ** -24
TINY = 2.0 ** -149  # smallest fp32 denormal: the absolute error of one rounding in the denormal range is <= TINY / 2
EPS_IL = float(np.float32(1e-5))  # the interlevel loss's denominator offset, as the kernel's 1e-5f
PULSE = tuple(float(np.float32(r)) for r in LO.PULSE_WIDTHS)  # NeuRAD's pulse widths as the kernel receives them
F32_EXP_MAX = float(np.log(np.finfo(np.float32).max))  # expf overflows above this


def backend(dev):
    if dev == "cpu":
        from tests.fake_backend import FakeBackend

        return FakeBackend()
    from neurad_studio_b200.backend import B200Backend

    return B200Backend(torch.device(dev, 0))


def _ratio(got, ref, tol, what, mask=None):
    """max |got - ref| / tol over the entries in `mask`; asserts <= 1 and names the worst entry."""
    got = got.detach().cpu().double().reshape(ref.shape)
    err = (got - ref).abs()
    if mask is not None:
        err, tol, got, ref = err[mask], tol[mask], got[mask], ref[mask]
    if err.numel() == 0:
        return 0.0
    assert torch.isfinite(got).all(), f"{what}: non-finite result"
    r = torch.where(err == 0, torch.zeros_like(err), err / tol)
    w = int(r.reshape(-1).argmax())
    worst = r.reshape(-1)[w].item()
    assert worst <= 1.0, (f"{what}: |got - ref| / tol = {worst:.3g} at flat entry {w}: got {got.reshape(-1)[w].item():.9g}, "
                          f"ref {ref.reshape(-1)[w].item():.9g}, tol {tol.reshape(-1)[w].item():.3g}")
    return worst


def _bits_equal(got, ref, what):
    got = got.detach().cpu().contiguous()
    ref = ref.contiguous()
    assert got.shape == ref.shape and got.dtype == ref.dtype, (what, got.shape, ref.shape, got.dtype, ref.dtype)
    if got.dtype == torch.float32:
        bad = got.view(torch.int32) != ref.view(torch.int32)
    else:
        bad = got != ref
    assert not bad.any(), f"{what}: {int(bad.sum())} entries differ, first at {bad.nonzero()[:3].tolist()}"


def _suffix(t):
    """sum_{k>i} t_k along dim 1 (a shifted reverse cumsum: no subtraction, so a tiny tail keeps its value)."""
    rc = torch.flip(torch.cumsum(torch.flip(t, [1]), 1), [1])
    return torch.cat([rc[:, 1:], torch.zeros_like(rc[:, :1])], 1)


def _mul0(a, b):
    """a * b with 0 * inf = 0: a bound term whose exact factor is 0 contributes nothing."""
    return torch.where(a == 0, torch.zeros_like(a), a * b)


# ====================================================================================== weights from alpha / density
def alpha_cases(S, n, seed):
    """alphas [n, S]: random (mostly small, so the transmittance does not vanish at once), with rays holding 0, 1 exactly,
    1 - 2^-24, and two saturated samples in one ray."""
    gen = torch.Generator().manual_seed(seed)
    a = torch.rand(n, S, generator=gen) ** 3
    if S > 1:
        a[0::7, S // 3] = 1.0
        a[1::7, S // 2] = 1.0 - 2.0 ** -24
        a[2::7, 0] = 0.0
        a[3::7, S // 4] = 1.0
        a[3::7, (3 * S) // 4] = 1.0
        a[4::7, :] = 0.0
    else:
        a[0::3] = 1.0
        a[1::3] = 0.0
    return a


def alpha_reference(a, g):
    """float64 autograd of the oracle's cumprod restatement, and the pieces of the bound: T_i and the suffix recurrence
    with |dw|, Rabs_i = sum_{k>i} |dw_k| a_k prod_{i<j<k} (1 - a_j)."""
    a64 = a.double().requires_grad_(True)
    w = O.render_weight_from_alpha(a64)
    ref_da, = torch.autograd.grad((w * g.double()).sum(), a64)
    a64 = a64.detach()
    one_m = 1 - a64
    T = torch.cumprod(torch.cat([torch.ones_like(a64[:, :1]), one_m[:, :-1]], 1), 1)
    Rabs = torch.zeros_like(a64)
    R = torch.zeros(a64.shape[0], dtype=torch.float64)
    for i in range(a64.shape[1] - 1, -1, -1):
        Rabs[:, i] = R
        R = g[:, i].double().abs() * a64[:, i] + one_m[:, i] * R
    return w.detach(), ref_da, T, Rabs


def alpha_bwd_tol(g, T, Rabs):
    """alpha_weights_bwd_ray: T_i is i products of (1 - a_j) (each 1 - a_j <= 1 U, each product 1 U: <= 2 i U relative);
    R_i is S - 1 - i steps of dw a + (1 - a) R (<= 4 U per step of the |dw| recurrence: two products, 1 - a, the sum);
    dalpha = T (dw - R): one subtraction, one product.  First order:
      |err| <= (2 S + 4 (S - i) + 2) U T_i (|dw_i| + Rabs_i) <= (6 S + 2) U T_i (|dw_i| + Rabs_i),
    plus the denormal range: every rounding of T or R adds <= TINY / 2 absolutely, S of each, times (|dw_i| + Rabs_i)."""
    S = g.shape[1]
    m = g.double().abs() + Rabs
    return (6 * S + 2) * U * T * m + S * TINY * (m + 1)


def alpha_weights_backward_matches_float64(dev, n, S, seed=0, be=None):
    """alpha_to_weights_bwd per entry, alpha in {0, 1, 1 - 2^-24, random}; on the GPU also the forward."""
    be = be or backend(dev)
    a = alpha_cases(S, n, seed)
    g = torch.randn(n, S, generator=torch.Generator().manual_seed(seed + 1))
    w64, ref, T, Rabs = alpha_reference(a, g)
    got = be.alpha_to_weights_bwd(a.to(dev), g.to(dev))
    worst = _ratio(got, ref, alpha_bwd_tol(g, T, Rabs), f"dalpha n={n} S={S}")
    if dev != "cpu":
        worst = max(worst, _ratio(be.alpha_to_weights(a.to(dev)), w64, alpha_weights_forward_tol(w64), f"alpha weights n={n} S={S}"))
    return worst


def alpha_weights_forward_tol(w64):
    """Forward: w_i = a_i T_i, a warp-scan product of i factors (any order): <= (2 i + 1) U relative."""
    i = torch.arange(w64.shape[1], dtype=torch.float64)
    return (2 * i + 2) * U * w64 + (i + 1) * TINY


def density_weights_forward_tol(delta, dens, w64):
    """Forward, the terms of E_w in density_bwd_tol (the warp-scan sum of A has the same bound as a sequential one)."""
    a = delta.double() * dens.double()
    A = torch.cat([torch.zeros_like(a[:, :1]), torch.cumsum(a, 1)[:, :-1]], 1)
    i = torch.arange(a.shape[1], dtype=torch.float64)
    eA, ea = torch.exp(-A), torch.exp(-a)
    wt = w64.detach()
    tol = eA * (_mul0(ea, (a + 4) * U) + U * (1 - ea)) + _mul0(wt, _mul0(eA, (i + 1) * U * A + 4 * U) / eA.clamp_min(1e-300) + 2 * U)
    return torch.nan_to_num(tol, nan=0.0) + 4 * TINY


def density_cases(S, n, seed):
    """deltas, densities [n, S]: random, plus density 0, delta 0, delta * density large enough that exp underflows, and
    (on rays of their own) inf density."""
    gen = torch.Generator().manual_seed(seed)
    delta = torch.rand(n, S, generator=gen) * 0.2 + 0.01
    dens = torch.exp(torch.randn(n, S, generator=gen) * 1.5)
    dens[0::9, S // 2] = 0.0
    delta[1::9, S // 3] = 0.0
    dens[2::9, S // 2] = 2000.0  # delta * density ~ 200: expf(-a) underflows to 0
    dens[3::9, (2 * S) // 3] = 1.0e9
    dens[4::9, S // 2] = float("inf")
    delta[4::9, S // 2] = 0.5
    return delta, dens


def density_bwd_tol(delta, dens, g):
    """density_weights_bwd_ray: a = fl(delta rho) (1 U); A_i a sequential fp32 sum (<= (i + 1) U A_i); expf(-x) <= 4 U
    plus the argument's error times 1 (d e^-x / e^-x = dx): rel(eA_i) <= (i + 1) U A_i + 4 U, rel(ea_i) <= (a_i + 4) U;
    w_k = (1 - ea_k) eA_k, whose 1 - ea cancels for small a_k (absolute, not relative, error ea_k rel(ea_k) + U);
      E_w_k = eA_k (ea_k rel(ea_k) + U (1 - ea_k)) + w_k (rel(eA_k) + U)
      suffix_i = sum_{k>i} dw_k w_k:  E_suf_i = sum_{k>i} |dw_k| E_w_k + (S - i + 1) U sum_{k>i} |dw_k w_k|
      first_i = dw_i ea_i eA_i:       E_first_i = |first_i| (rel(ea_i) + rel(eA_i) + 2 U)
      ddensity_i = delta_i (first_i - suffix_i):  delta_i (E_first + E_suf + 2 U (|first| + |suffix|))
    plus TINY per rounding in the denormal range (S of them per sum, times the cotangents' magnitude)."""
    d, r, g = delta.double(), dens.double(), g.double()
    a = d * r
    A = torch.cat([torch.zeros_like(a[:, :1]), torch.cumsum(a, 1)[:, :-1]], 1)
    S = a.shape[1]
    i = torch.arange(S, dtype=torch.float64)
    eA, ea = torch.exp(-A), torch.exp(-a)
    relA = _mul0(eA, (i + 1) * U * A + 4 * U) / torch.where(eA == 0, torch.ones_like(eA), eA)
    rela = (a + 4) * U
    w = (1 - ea) * eA
    Ew = eA * (_mul0(ea, rela) + U * (1 - ea)) + _mul0(w, relA + U)
    dwabs = g.abs()
    t = dwabs * Ew
    tw = dwabs * w
    suf_e, suf_w = _suffix(t), _suffix(tw)
    first = dwabs * ea * eA
    E = _mul0(d, _mul0(first, rela + relA + 2 * U) + suf_e + (S - i + 1) * U * suf_w + 2 * U * (first + suf_w))
    return E + S * TINY * (d + 1) * (dwabs.sum(1, keepdim=True) + 1)


def density_weights_backward_matches_float64(dev, n, S, seed=0, be=None):
    """density_to_weights_bwd per entry.  Entries whose float64 autograd is not finite (the inf-density rays) are
    excluded and counted; the kernel's result must be finite everywhere."""
    be = be or backend(dev)
    delta, dens = density_cases(S, n, seed)
    g = torch.randn(n, S, generator=torch.Generator().manual_seed(seed + 2))
    r64 = dens.double().requires_grad_(True)
    w64 = O.weights_from_density(delta.double(), r64)
    ref, = torch.autograd.grad((w64 * g.double()).sum(), r64)
    got = be.density_to_weights_bwd(delta.to(dev), dens.to(dev), g.to(dev))
    assert torch.isfinite(got).all(), "ddensity: non-finite entries"
    ok = torch.isfinite(ref)
    worst = _ratio(got, ref, density_bwd_tol(delta, dens, g), f"ddensity n={n} S={S}", mask=ok)
    excluded = int((~ok).sum())
    if dev != "cpu":
        wt = w64.detach()
        worst = max(worst, _ratio(be.density_to_weights(delta.to(dev), dens.to(dev)), wt, density_weights_forward_tol(delta, dens, wt),
                                  f"density weights n={n} S={S}"))
    return worst, excluded


# ====================================================================================== distortion loss
def distortion_inputs(n, S, seed, dyadic=False):
    """sdist [n, S+1] sorted in [0, 1], weights [n, S]; zero-width bins and all-zero weights on some rays.  dyadic: edges
    k/64 and weights k/1024 with sum <= 1/8, so every product and partial sum is exact in fp32."""
    gen = torch.Generator().manual_seed(seed)
    if dyadic:
        c = torch.sort(torch.randint(0, 65, (n, S + 1), generator=gen), 1).values.float() / 64
        w = torch.randint(0, 3, (n, S), generator=gen).float() / 1024
        return c, w
    c = torch.sort(torch.rand(n, S + 1, generator=gen), 1).values
    c[:, 0], c[:, -1] = 0.0, 1.0
    w = torch.rand(n, S, generator=gen) ** 2
    w = w / w.sum(1, keepdim=True) * torch.rand(n, 1, generator=gen) * 1.2
    if S > 2:
        c[0::5, 2] = c[0::5, 1]  # a zero-width bin
    w[1::5] = 0.0
    return c, w


def distortion_reference(c, w):
    w64 = w.double().requires_grad_(True)
    loss = LO.lossfun_distortion(c.double(), w64)
    dw, = torch.autograd.grad(loss.sum(), w64)
    return loss.detach(), dw


def distortion_tol(c, w):
    """distortion_loss_ray: u_i = (c_i + c_{i+1}) / 2 (1 U), |u_i - u_j| (1 U more): error <= 3 U Cmax per distance
    (Cmax = max |c| of the ray); inner_i = sum_j w_j d_ij: W1 * 3 U Cmax + (S + 1) U sum_j |w_j| d_ij (products and S
    additions); dw_i = 2 inner_i + 2 w_i d_i / 3 (d_i = c_{i+1} - c_i: 1 U; product, division, sum: 3 U more);
    loss = sum_i w_i inner_i + sum_i w_i^2 d_i / 3: sum_i |w_i| E_inner_i + (S + 1) U sum_i |w_i| Iabs_i
    + (S + 4) U sum_i w_i^2 |d_i| / 3 + U |loss|."""
    c, w = c.double(), w.double()
    u = (c[:, 1:] + c[:, :-1]) / 2
    dist = (u[:, :, None] - u[:, None, :]).abs()
    S = w.shape[1]
    wa = w.abs()
    cmax = c.abs().amax(1, keepdim=True)
    Iabs = (wa[:, None, :] * dist).sum(-1)
    Ein = wa.sum(1, keepdim=True) * 3 * U * cmax + (S + 1) * U * Iabs
    dd = (c[:, 1:] - c[:, :-1]).abs()
    tol_dw = 2 * Ein + 2 * wa * dd / 3 * 5 * U + U * (2 * Iabs + 2 * wa * dd / 3)
    intra = (w * w * dd).sum(1) / 3
    tol_loss = (wa * (Ein + (S + 1) * U * Iabs)).sum(1) + (S + 4) * U * intra + U * ((wa * Iabs).sum(1) + intra)
    return tol_loss, tol_dw


def distortion_matches_float64(dev, n, S, seed=0, be=None):
    """distortion_loss per ray and its dw per entry; the loss is bit-identical with and without dw; the dyadic case is
    exact up to the two divisions by 3 and the additions after them."""
    be = be or backend(dev)
    worst = 0.0
    for dyadic in (False, True):
        c, w = distortion_inputs(n, S, seed, dyadic)
        loss, dw = be.distortion_loss(c.to(dev), w.to(dev), want_grad=True)
        loss2, none = be.distortion_loss(c.to(dev), w.to(dev), want_grad=False)
        assert none is None and loss.shape == (n,) and dw.shape == (n, S)
        _bits_equal(loss2, loss.cpu(), f"distortion loss with / without dw, n={n} S={S}")
        ref_l, ref_dw = distortion_reference(c, w)
        if dyadic:  # inter, intra and inner are exact; the kernel rounds intra / 3, the final sum, 2 w d / 3 and the dw sum
            c64, w64 = c.double(), w.double()
            u = (c64[:, 1:] + c64[:, :-1]) / 2
            inner = (w64[:, None, :] * (u[:, :, None] - u[:, None, :]).abs()).sum(-1)
            d = c64[:, 1:] - c64[:, :-1]
            inter, intra = (w64 * inner).sum(1), (w64 * w64 * d).sum(1)
            f = lambda x: x.float()  # noqa: E731  (exact: every one of these is an fp32 number)
            want_l = f(inter) + f(intra) / 3
            want_dw = 2 * f(inner) + (2 * f(w64) * f(d)) / 3
            _bits_equal(loss, want_l, f"dyadic distortion loss n={n} S={S}")
            _bits_equal(dw, want_dw, f"dyadic distortion dw n={n} S={S}")
            continue
        tl, tdw = distortion_tol(c, w)
        worst = max(worst, _ratio(loss, ref_l, tl, f"distortion loss n={n} S={S}"),
                    _ratio(dw, ref_dw, tdw, f"distortion dw n={n} S={S}"))
    return worst


# ====================================================================================== zipnerf interlevel loss
def interlevel_inputs(n, S, Sp, seed, kind="random"):
    """Final level c [n, S+1] (in [0, 1], c_0 = 0 and c_S = 1 on most rays: knots outside [0, 1]), w [n, S]; proposal
    level cp [n, Sp+1] (edges exactly 0 and 1 on most rays), wp [n, Sp] (some exactly 0).  Weights sum to < 1, 0 (the
    last bin takes all the mass), > 1 (the last bin goes negative), or form a one-bin spike, by ray.
    kind "dyadic": c = k/64 (S = 64: every bin 1/64 wide), w = k/1024, cp = k/256, wp = k/1024, r = 2^-7: every c_k + r
    ties with c_{k+1} - r and every step up to the loss's division is exact in fp32."""
    gen = torch.Generator().manual_seed(seed)
    if kind == "dyadic":
        c = torch.arange(S + 1).float().expand(n, S + 1) / S
        w = torch.randint(0, 40, (n, S), generator=gen).float() / 1024
        cp = torch.sort(torch.randint(0, 257, (n, Sp + 1), generator=gen), 1).values.float() / 256
        cp[:, 0], cp[:, -1] = 0.0, 1.0
        wp = torch.randint(0, 64, (n, Sp), generator=gen).float() / 1024
        return c, w, cp, wp
    c = torch.sort(torch.rand(n, S + 1, generator=gen), 1).values
    c = c + 1e-3 * torch.arange(S + 1).float() / S  # no zero-width bins (w / width)
    c = c / c[:, -1:].clamp_min(1.0)
    c[0::4, 0], c[0::4, -1] = 0.0, 1.0
    c[1::4, 0] = 0.0
    w = torch.rand(n, S, generator=gen) ** 3
    w = w / w.sum(1, keepdim=True) * torch.rand(n, 1, generator=gen)
    w[1::6] = 0.0                       # sum 0: the last bin takes all the mass
    w[2::6] *= 1.7                      # may sum to > 1: the last bin goes negative
    w[3::6] = 0.0
    w[3::6, S // 2] = 0.9               # one-bin spike
    cp = torch.sort(torch.rand(n, Sp + 1, generator=gen), 1).values
    cp[0::2, 0], cp[0::2, -1] = 0.0, 1.0
    wp = torch.rand(n, Sp, generator=gen) ** 2 * (2.0 / Sp)
    wp[torch.rand(n, Sp, generator=gen) < 0.1] = 0.0  # den = 1e-5
    return c, w, cp, wp


def interlevel_ws(c, w, cp, r):
    """zipnerf_interlevel_per_ray up to the resampled weights w_s (oracle/losses_oracle.py), in float64."""
    c, w, cp = c.double(), w.double(), cp.double()
    accum_w = torch.sum(w, dim=-1, keepdim=True)
    w = torch.cat([w[..., :-1], w[..., -1:] + (1 - accum_w)], dim=-1)
    w_norm = w / (c[..., 1:] - c[..., :-1])
    c_, w_ = LO.blur_stepfun(c, w_norm, r)
    area = 0.5 * (w_[..., 1:] + w_[..., :-1]) * (c_[..., 1:] - c_[..., :-1])
    cdf = torch.cat([torch.zeros_like(area[..., :1]), torch.cumsum(area, dim=-1)], dim=-1)
    c_ = torch.cat([torch.zeros_like(c_[..., :1]), c_, torch.ones_like(c_[..., :1])], dim=-1)
    w_ = torch.cat([torch.zeros_like(w_[..., :1]), w_, torch.zeros_like(w_[..., :1])], dim=-1)
    cdf = torch.cat([torch.zeros_like(cdf[..., :1]), cdf, torch.ones_like(cdf[..., :1])], dim=-1)
    return torch.diff(LO.sorted_interp_quad(cp, c_, w_, cdf), dim=-1)


def interlevel_reference(c, w, cp, wp, r):
    """(loss [n], dwp [n, Sp], ws [n, Sp]): the oracle's formula with the kernel's fp32 1e-5, float64 autograd."""
    ws = interlevel_ws(c, w, cp, r)
    wp64 = wp.double().requires_grad_(True)
    per = ((ws - wp64).clamp_min(0) ** 2 / (wp64 + EPS_IL)).sum(-1)
    dwp, = torch.autograd.grad(per.sum(), wp64)
    return per.detach(), dwp, ws


def interlevel_ws_error(c, w, cp, r):
    """Bound E_ws [n, Sp] on |ws_kernel - ws_float64|, by forward error analysis of zipnerf_interlevel_ray, step by step
    (first order; E_x is the bound of quantity x; cumulative sums in double add 2^-52 m sum|terms|):
      acc = sum w (fp32, S terms):           E_acc = S U sum|w|
      w_last = w_{S-1} + (1 - acc):          E = E_acc + U |1 - acc| + U |w_last|
      wn_k = w_k / (c_{k+1} - c_k):          E_wn = 2 U |wn| + E_w / width
      y1_k = (wn_k - wn_{k-1}) / (2 r):      E_y1 = (E_wn_k + E_wn_{k-1} + U |wn_k - wn_{k-1}|) / (2 r) + U |y1|
      slope (double sum of +-y1):            E_slope = sum E_y1 (+ double rounding)
      dx_m = x_m - x_{m-1}:                  E_dx = U |dx|
      raw += dx * (float) slope:             E_prod = |dx| (E_slope + U |slope|) + |slope| E_dx + U |prod|
      y_m = max((float) raw, 0):             E_y = sum E_prod + U |raw|          (the clamp is 1-Lipschitz)
      area = 0.5 (y_m + y_{m-1}) dx:         E_area = 0.5 (E_y_m + E_y_{m-1}) |dx| + 0.5 |y_m + y_{m-1}| E_dx + 3 U |area|
      cdf (double sum, cast to fp32):        E_cdf = sum E_area + U |cdf|
    and the interpolation at x = cp_e between padded knots xp0 = xs[left], xp1 = xs[right] (the reference's bracket):
      t = x - xp0:                           E_t = U |t|
      off = clip(t / (xp1 - xp0), 0, 1):     E_off = min(1, E_t / |xp1 - xp0| + 3 U)
      q = y_l + y_r off + y_l (1 - off):     E_q = 2 E_y_l + E_y_r + |y_r - y_l| E_off + 5 U (2 |y_l| + |y_r|)
      v = cdf_l + 0.5 t q:                   E_v = E_cdf_l + 0.5 (|t| E_q + |q| E_t) + 2 U |t q| / 2 + U |v|
      ws_e = v_e - v_{e-1}:                  E_ws = E_v_e + E_v_{e-1} + U |ws| + E_knot_e.
    The steps above run on the kernel's knots fl(c_k -/+ r); the reference's are the exact c_k -/+ r.  The blurred cdf is
    F(x) = sum_k y1_k (h(x - a_k) - h(x - b_k)), h(t) = max(t, 0)^2 / 2, a_k = c_k - r, b_k = c_k + r, continuous in the
    knots (whatever bracket the search picks), with dF/da_k = -y1_k max(x - a_k, 0); so moving every knot by <= U |knot|
    moves ws_e = F(cp_e) - F(cp_{e-1}) by at most
      E_knot_e = sum_k |y1_k| U (|a_k| clamp(cp_e - a_k, 0, cp_e - cp_{e-1}) + |b_k| clamp(cp_e - b_k, 0, cp_e - cp_{e-1}))."""
    c, w, cp = c.double(), w.double(), cp.double()
    n, S = w.shape
    acc = w.sum(1, keepdim=True)
    Ew = torch.zeros_like(w)
    wl = w.clone()
    wl[:, -1:] = w[:, -1:] + (1 - acc)
    Ew[:, -1:] = S * U * w.abs().sum(1, keepdim=True) + U * (1 - acc).abs() + U * wl[:, -1:].abs()
    width = c[:, 1:] - c[:, :-1]
    wn = wl / width
    Ewn = 2 * U * wn.abs() + Ew / width.abs()
    z = torch.zeros(n, 1, dtype=torch.float64)
    wnp, Ewnp = torch.cat([z, wn, z], 1), torch.cat([z, Ewn, z], 1)
    y1 = (wnp[:, 1:] - wnp[:, :-1]) / (2 * r)
    Ey1 = (Ewnp[:, 1:] + Ewnp[:, :-1] + U * (wnp[:, 1:] - wnp[:, :-1]).abs()) / (2 * r) + U * y1.abs()
    X = torch.cat([c - r, c + r], 1)
    X, idx = torch.sort(X, dim=1, stable=True)
    Y = torch.cat([y1, -y1], 1).gather(1, idx)
    EY = torch.cat([Ey1, Ey1], 1).gather(1, idx)
    EX = torch.zeros_like(X)
    M = X.shape[1]
    slope = torch.cumsum(Y, 1)
    Eslope = torch.cumsum(EY, 1) + 2.0 ** -52 * M * torch.cumsum(Y.abs(), 1)
    dx = X[:, 1:] - X[:, :-1]
    Edx = EX[:, 1:] + EX[:, :-1] + U * dx.abs()
    sl, Esl = slope[:, :-1], Eslope[:, :-1]
    prod = dx * sl
    Eprod = dx.abs() * (Esl + U * sl.abs()) + sl.abs() * Edx + U * prod.abs()
    raw = torch.cumsum(prod, 1)
    y = torch.cat([z, raw.clamp_min(0)], 1)
    Ey = torch.cat([z, torch.cumsum(Eprod, 1) + 2.0 ** -52 * M * torch.cumsum(prod.abs(), 1) + U * raw.abs()], 1)
    area = 0.5 * (y[:, 1:] + y[:, :-1]) * dx
    Earea = 0.5 * (Ey[:, 1:] + Ey[:, :-1]) * dx.abs() + 0.5 * (y[:, 1:] + y[:, :-1]).abs() * Edx + 3 * U * area.abs()
    cdf = torch.cat([z, torch.cumsum(area, 1)], 1)
    Ecdf = torch.cat([z, torch.cumsum(Earea, 1) + 2.0 ** -52 * M * torch.cumsum(area.abs(), 1)], 1) + U * cdf.abs()
    one = torch.ones(n, 1, dtype=torch.float64)
    xs, Exs = torch.cat([z, X, one], 1), torch.cat([z, EX, z], 1)
    ys, Eys = torch.cat([z, y, z], 1), torch.cat([z, Ey, z], 1)
    cdfs, Ecdfs = torch.cat([z, cdf, one], 1), torch.cat([z, Ecdf, z], 1)
    L = xs.shape[1]
    right = torch.searchsorted(xs.contiguous(), cp.contiguous())
    left = (right - 1).clamp_min(0)
    right = right.clamp_max(L - 1)
    G = lambda t, i: t.gather(1, i)  # noqa: E731
    xp0, xp1, Exp0, Exp1 = G(xs, left), G(xs, right), G(Exs, left), G(Exs, right)
    yl, yr, Eyl, Eyr = G(ys, left), G(ys, right), G(Eys, left), G(Eys, right)
    cl, Ecl = G(cdfs, left), G(Ecdfs, left)
    t = cp - xp0
    Et = U * t.abs()
    gap = (xp1 - xp0).abs()
    Eoff = torch.where(gap > 0, Et / gap.clamp_min(1e-300) + 3 * U, torch.ones_like(gap)).clamp_max(1.0)
    off = torch.clip(torch.nan_to_num(t / (xp1 - xp0), 0), 0, 1)
    q = yl + yr * off + yl * (1 - off)
    Eq = 2 * Eyl + Eyr + (yr - yl).abs() * Eoff + 5 * U * (2 * yl.abs() + yr.abs())
    v = cl + t * q * 0.5
    Ev = Ecl + 0.5 * (t.abs() * Eq + q.abs() * Et) + U * (t * q).abs() + U * v.abs()
    ws = v[:, 1:] - v[:, :-1]
    knots = torch.cat([c - r, c + r], 1)
    wk = torch.cat([y1, y1], 1).abs() * U * knots.abs()
    Eknot = torch.empty_like(ws)
    for r0 in range(0, n, 2048):  # [rays, Sp, 2 S + 2] in slices
        sl = slice(r0, r0 + 2048)
        lo, hi = cp[sl, :-1, None], cp[sl, 1:, None]
        reach = torch.minimum((hi - knots[sl, None, :]).clamp_min(0), hi - lo)
        Eknot[sl] = (reach * wk[sl, None, :]).sum(-1)
    return Ev[:, 1:] + Ev[:, :-1] + U * ws.abs() + Eknot


def interlevel_tol(ws, wp, Ews):
    """From |ws error| <= E_ws: d = ws - wp (E_d = E_ws + U |d|), den = wp + 1e-5 (U den).  The relu makes both results
    continuous at d = 0, so a sign flip of d within E_d is covered by the same bound:
      dwp = -2 d / den - d^2 / den^2:  (2 / den + (2 |d| + E_d) / den^2) E_d + (2 |d| / den + d^2 / den^2) (2 U + 4 U)
      loss = sum_e d^2 / den:          sum_e [(2 |d| + E_d) / den E_d + d^2 / den (U + 3 U)] + Sp U sum_e d^2 / den
    Entries with d + E_d <= 0 are 0 in the kernel and the reference alike; their bound is 0."""
    wp = wp.double()
    d = ws - wp
    Ed = Ews + U * d.abs()
    den = wp + EPS_IL
    live = (d + Ed > 0).double()
    dpos = d.clamp_min(0)
    tol_g = live * ((2 / den + (2 * dpos + Ed) / den ** 2) * Ed + (2 * dpos / den + dpos ** 2 / den ** 2) * 6 * U)
    term = dpos ** 2 / den
    tol_l = (live * ((2 * dpos + Ed) / den * Ed + term * 4 * U)).sum(1) + wp.shape[1] * U * term.sum(1)
    return tol_l, tol_g


def interlevel_matches_float64(dev, n, S, Sp, r, seed=0, kind="random", be=None):
    """zipnerf_interlevel_loss per ray and dwp per entry against float64; the loss is bit-identical with and without
    dwp.  kind "tie": wp set to fp32(ws) of the reference (the relu boundary); kind "dyadic": ws is exact, so only the
    roundings after ws are allowed."""
    be = be or backend(dev)
    c, w, cp, wp = interlevel_inputs(n, S, Sp, seed, "dyadic" if kind == "dyadic" else "random")
    if kind == "tie":
        wp = interlevel_ws(c, w, cp, r).float().clamp_min(0)
    loss, dwp = be.zipnerf_interlevel_loss(c.to(dev), w.to(dev), cp.to(dev), wp.to(dev), r, want_grad=True)
    loss2, none = be.zipnerf_interlevel_loss(c.to(dev), w.to(dev), cp.to(dev), wp.to(dev), r, want_grad=False)
    assert none is None and loss.shape == (n,) and dwp.shape == (n, Sp)
    _bits_equal(loss2, loss.cpu(), f"interlevel loss with / without dwp n={n} S={S} Sp={Sp}")
    if n == 0:
        return 0.0
    ref_l, ref_g, ws = interlevel_reference(c, w, cp, wp, r)
    Ews = torch.zeros_like(ws) if kind == "dyadic" else interlevel_ws_error(c, w, cp, r)
    tl, tg = interlevel_tol(ws, wp, Ews)
    what = f"interlevel {kind} n={n} S={S} Sp={Sp} r={r:.3g}"
    return max(_ratio(loss, ref_l, tl, what + " loss"), _ratio(dwp, ref_g, tg, what + " dwp"))


# ====================================================================================== composite backward
def composite_case(dev, n, S, C, has_v, has_a, has_d, need_dw, need_dv, seed=0, be=None):
    """composite_bwd with each cotangent present or absent: dw per entry against float64 with the bound (C + 4) U of
    sum |terms| (C + 2 products and their sum, (start + end) 0.5: 1 U of |ddepth| (|start| + |end|) / 2);
    dvalues = fp32(w * go) bit for bit.  Combinations that compute nothing must raise."""
    from neurad_studio_b200.lib import B200NerfError

    be = be or backend(dev)
    gen = torch.Generator().manual_seed(seed)
    w = torch.rand(n, S, generator=gen)
    v = torch.randn(n, S, C, generator=gen)
    st = torch.rand(n, S, generator=gen) * 50
    en = st + torch.rand(n, S, generator=gen)
    go, ga, gd = torch.randn(n, C, generator=gen), torch.randn(n, generator=gen), torch.randn(n, generator=gen)
    args = (w.to(dev), v.to(dev) if has_v else None, st.to(dev) if has_d else None, en.to(dev) if has_d else None,
            go.to(dev) if has_v else None, ga.to(dev) if has_a else None, gd.to(dev) if has_d else None)
    if not need_dw and not (need_dv and has_v):
        try:
            be.composite_bwd(*args, need_dweights=need_dw, need_dvalues=need_dv)
        except B200NerfError:
            return 0.0
        raise AssertionError("composite_bwd with nothing to compute did not raise")
    dw, dv = be.composite_bwd(*args, need_dweights=need_dw, need_dvalues=need_dv)
    assert (dw is None) == (not need_dw) and (dv is None) == (not (need_dv and has_v))
    worst = 0.0
    if need_dw:
        ref = torch.zeros(n, S, dtype=torch.float64)
        ab = torch.zeros(n, S, dtype=torch.float64)
        if has_a:
            ref += ga.double()[:, None]
            ab += ga.double().abs()[:, None]
        if has_d:
            mid = (st.double() + en.double()) / 2
            ref += gd.double()[:, None] * mid
            ab += gd.double().abs()[:, None] * (st.double().abs() + en.double().abs()) / 2
        if has_v:
            ref += (v.double() * go.double()[:, None, :]).sum(-1)
            ab += (v.double() * go.double()[:, None, :]).abs().sum(-1)
        worst = _ratio(dw, ref, (C + 4) * U * ab, f"composite dw n={n} S={S} C={C} v={has_v} a={has_a} d={has_d}")
    if dv is not None:
        _bits_equal(dv, w[..., None] * go[:, None, :], f"composite dvalues n={n} S={S} C={C}")
    return worst


# ====================================================================================== field heads backward
def field_heads_inputs(n, G, seed):
    """geo [n, G+1] with sdf * beta at +-17 and +-90 (and 0) on some rows, and the four cotangents."""
    gen = torch.Generator().manual_seed(seed)
    geo = torch.randn(n, G + 1, generator=gen)
    geo[:, 0] = torch.randn(n, generator=gen) * 0.3
    return geo, (torch.randn(n, G, generator=gen), torch.randn(n, generator=gen), torch.randn(n, generator=gen),
                 torch.randn(n, G + 16, generator=gen))


def set_extreme_sdf(geo, beta):
    """sdf * beta at -90, -17, 0, 17, 90 on rows 0..4 (mod 7): alpha = 1 exactly, the al (1 - al) cancellation, 1/2,
    ~4e-8, and expf overflow (alpha = 0 in fp32 where the float64 sigmoid is ~8e-40)."""
    for j, x in enumerate((-90.0, -17.0, 0.0, 17.0, 90.0)):
        geo[j::7, 0] = x / beta


def field_heads_reference(geo, dsdf, dalpha, beta):
    """dgeo[:, 0] and the per-row dbeta terms in float64 (beta = the fp32 value the kernel receives), and their bounds.
    Kernel: x = fl(sd beta) (1 U), e = expf(x) (rel <= |x| U + 4 U), al = rcp(1 + e) (2 U): rel(al) <= (1 - al)(|x| + 5) U
    + 2 U.  t = dalpha al (1 - al): 1 - al cancels near al = 1 (absolute error al rel(al) + U (1 - al)), so
      E_t = |dalpha| al ((1 - al)(|x| + 10) U + 2 U)        (two products included)
    Where expf overflows (x > ln FLT_MAX) the kernel's al is 0, as torch's fp32 sigmoid is: the reference takes al = 0
    there (the float64 sigmoid, < 1.7e-38 beta-scaled, is not what either fp32 formula computes).  Then
      g0 = dsdf - beta t:   beta E_t + 2 U (|beta t| + |g0|)
      db = -sd t:           |sd| E_t + U |sd t|
    plus TINY per rounding for al in the denormal range."""
    sd = geo[:, 0].double()
    x = sd * beta
    al = torch.where(x > F32_EXP_MAX, torch.zeros_like(x), torch.sigmoid(-x))
    da = torch.zeros_like(sd) if dalpha is None else dalpha.double()
    t = da * al * (1 - al)
    Et = da.abs() * al * ((1 - al) * (x.abs() + 10) * U + 2 * U) + da.abs() * 4 * TINY
    g0 = (torch.zeros_like(sd) if dsdf is None else dsdf.double()) - beta * t
    Eg0 = beta * Et + 2 * U * ((beta * t).abs() + g0.abs())
    db = -sd * t
    Edb = sd.abs() * Et + U * db.abs()
    return g0, Eg0, db, Edb


def field_heads_case(dev, n, G, absent, beta=20.0, seed=0, be=None):
    """field_heads_bwd with one optional input absent (or none): dgeo[:, 0] per entry, dgeo[:, 1:] = fp32(dfeature +
    dx2[:, :G]) bit for bit, dbeta against the float64 sum with (n + 2) U sum |db_i| + sum E_db_i (n terms summed in any
    order: the per-warp shuffles and the atomics)."""
    from neurad_studio_b200 import scene
    import neurad_studio_b200 as nsb

    if be is None:
        be = backend(dev)
        cfg = nsb.small_config()
        be.load_params(cfg, scene.make_params(cfg, beta=beta))
    b = float(np.float32(be._beta))
    geo, (df, dsdf, dal, dx2) = field_heads_inputs(n, G, seed)
    set_extreme_sdf(geo, b)
    ins = {"dfeature": df, "dsdf": dsdf, "dalpha": dal, "dx2": dx2}
    if absent:
        ins[absent] = None
    dgeo, dbeta = be.field_heads_bwd(geo.to(dev), *[None if ins[k] is None else ins[k].to(dev) for k in ("dfeature", "dsdf", "dalpha", "dx2")])
    return check_field_heads(dgeo, dbeta, geo, ins, b, f"field_heads n={n} G={G} absent={absent}")


def check_field_heads(dgeo, dbeta, geo, ins, b, what):
    n, G = geo.shape[0], geo.shape[1] - 1
    z = torch.zeros(n, G)
    want = (ins["dfeature"] if ins["dfeature"] is not None else z) + (ins["dx2"][:, :G] if ins["dx2"] is not None else z)
    _bits_equal(dgeo[:, 1:].contiguous(), want, what + " dgeo[:, 1:]")
    g0, Eg0, db, Edb = field_heads_reference(geo, ins["dsdf"], ins["dalpha"], b)
    worst = _ratio(dgeo[:, 0], g0, Eg0, what + " dgeo[:, 0]")
    ref_b = db.sum().reshape(1)
    tol_b = (Edb.sum() + (n + 2) * U * db.abs().sum()).reshape(1)
    if ins["dalpha"] is None:
        _bits_equal(dbeta, torch.zeros(1), what + " dbeta without dalpha")
        return worst
    return max(worst, _ratio(dbeta, ref_b, tol_b, what + " dbeta"))


def field_tail_sign_of_negative_beta(dev):
    """FieldTailFn (the autograd wrapper): with beta < 0 the parameter's gradient is sign(beta) dL/d(|beta| + 1e-4)."""
    from neurad_studio_b200 import autograd as AG
    from neurad_studio_b200 import scene
    import neurad_studio_b200 as nsb

    be = backend(dev)
    cfg = nsb.small_config()
    beta = -20.0
    be.load_params(cfg, scene.make_params(cfg, beta=beta))
    b = float(np.float32(be._beta))
    n, G = 1000, cfg.nff_out_dim
    geo, (df, dsdf, dal, _) = field_heads_inputs(n, G, 3)
    param = torch.full((1,), beta, device=dev, requires_grad=True)
    feature, sdf, alpha = AG.FieldTailFn.apply(be, geo.to(dev), torch.zeros(n, G, device=dev), param)
    (alpha.reshape(-1) * dal.to(dev)).sum().backward()
    _, _, db, Edb = field_heads_reference(geo, None, dal, b)
    ref = -db.sum().reshape(1)  # sign(beta) = -1
    tol = (Edb.sum() + (n + 2) * U * db.abs().sum()).reshape(1)
    assert ref.abs().item() > 10 * tol.item()
    return _ratio(param.grad, ref, tol, "FieldTailFn beta < 0")


# ====================================================================================== ReLU backward and the dgrad mask
def special_z(n, seed):
    """z with +0, -0, NaN, +-smallest denormal, +-inf and random values; dz random."""
    gen = torch.Generator().manual_seed(seed)
    z = torch.randn(n, generator=gen)
    sp = torch.tensor([0.0, -0.0, float("nan"), TINY, -TINY, float("inf"), -float("inf")])
    k = min(n, 7 * max(n // 14, 1))  # about half the entries special
    z[:k] = sp.repeat(k // 7 + 1)[:k]
    idx = torch.randperm(n, generator=gen)
    return z[idx], torch.randn(n, generator=gen)


def relu_bwd_bit_exact(dev, n):
    be = backend(dev)
    z, dz = special_z(n, n)
    got = be.relu_bwd(z.to(dev), dz.clone().to(dev))
    _bits_equal(got, torch.where(z > 0, dz, torch.zeros_like(dz)), f"relu_bwd n={n}")


def mlp_dgrad_mask_bit_exact(dev, rows, k, n_out):
    """mlp_dgrad with relu_z = the masked result of the same product without a mask, bit for bit."""
    be = backend(dev)
    gen = torch.Generator().manual_seed(rows + k)
    dy = torch.randn(rows, k, generator=gen)
    wgt = torch.randn(k, n_out, generator=gen) / k ** 0.5
    z, _ = special_z(rows * n_out, rows)
    z = z.reshape(rows, n_out)
    plain = be.mlp_dgrad(dy.to(dev), wgt.to(dev)).cpu()
    masked = be.mlp_dgrad(dy.to(dev), wgt.to(dev), z.to(dev))
    _bits_equal(masked, torch.where(z > 0, plain, torch.zeros_like(plain)), f"mlp_dgrad mask rows={rows} {k}->{n_out}")


# ====================================================================================== lidar carving mask
def lidar_mask_bit_exact(dev, n, S, with_did_return, seed=0):
    """lidar_carving_mask against losses_oracle.is_close_to_lidar on the same fp32 inputs (fp32 epsilon), bit for bit.
    Rows place sample midpoints at |d - mid| == eps exactly (dyadic eps), one fp32 step either side of it, at
    float32(0.1) against the float64 0.1, and at mid == non_return_distance; odd rays are camera rays (mask 0)."""
    be = backend(dev)
    gen = torch.Generator().manual_seed(seed)
    edges = torch.sort(torch.rand(n, S + 1, generator=gen) * 200.0, 1).values
    dn = torch.rand(n, generator=gen) * 150.0 + 10
    is_lidar = (torch.arange(n) // 3) % 2 == 0
    did = torch.rand(n, generator=gen) < 0.6
    worst = 0
    for eps, nrd in ((0.125, 64.0), (float(np.float32(0.1)), 150.0)):
        e = edges.clone()
        d = dn.clone()
        # rows r = 1 (mod 3): edges on the grid nrd - 1.75 + 0.5 k, so midpoint k is nrd - 1.5 + 0.5 k exactly
        # (midpoint 3 == non_return_distance), and the measured distance sits at midpoint j +- eps, one fp32 step
        # inside or outside eps, or + 0.1 in float64 rounded to fp32
        offs = [eps, -eps, float(np.nextafter(np.float32(eps), np.float32(1))), float(np.nextafter(np.float32(eps), np.float32(0))),
                -float(np.nextafter(np.float32(eps), np.float32(0))), 0.1]
        rows = torch.arange(1, n, 3)
        e[rows] = nrd - 1.75 + 0.5 * torch.arange(S + 1).float()
        j = torch.arange(rows.numel()) % min(S, 8)
        mid = nrd - 1.5 + 0.5 * j.float()
        d[rows] = (mid.double() + torch.tensor(offs, dtype=torch.float64)[torch.arange(rows.numel()) % len(offs)]).float()
        dr = did if with_did_return else None
        got = be.lidar_carving_mask(e.to(dev), is_lidar.to(dev), d.to(dev), None if dr is None else dr.to(dev), eps, nrd)
        want = LO.is_close_to_lidar(e, is_lidar, d, dr, eps, nrd)
        _bits_equal(got, want, f"lidar mask n={n} S={S} eps={eps} did_return={with_did_return}")
        assert not got.cpu()[~is_lidar].any()
        worst = max(worst, int(want.sum()))
    return worst
