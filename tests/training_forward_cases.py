"""Bodies of the entry-by-entry tests of the training step's forward operators (the module walk of
NeuRADModel.get_nff_outputs(fused=False)): isotropic_gaussian, spaced_sample_stratified, spacing_to_euclidean,
pdf_resample_stratified, neurad_encoding (main field F = 4, proposal fields F = 1 with their density head), _field_mid /
_field_tail and mlp_fwd(want_hidden=True) / mlp_dgrad, shared by tests/test_zz_training_forward_gpu.py (dev = "cuda":
the real library, production table sizes) and tests/test_training_forward_cpu.py (dev = "cpu": tests/fake_backend.py,
whose encoding and gaussian run the device code through the host emulation, small tables).

Every comparator judges one call from that call's own inputs, so errors do not chain: the same comparators run on
synthetic inputs at the kernels' edges and on the calls of one recorded training step (record_training_step).
Reference: the same formula in float64 on the kernel's fp32 inputs, with the fp32 constants the kernel receives.
Bounds are derived per entry from the kernel's op sequence (standard model: one fp32 rounding <= U = 2^-24 of its
result, expf <= 2 ulp, logf <= 1 ulp, powf <= 4 ulp, rcp.approx <= 2 U, cbrtf as in render_trace_cases.STD_REL, a sum of n
terms in any order <= n U of the sum of |terms|), first order in U, condition factors explicit (the _E chains below
carry them through every step).  Nothing is scaled to a tensor's maximum.  Results that are one IEEE operation
sequence the test can repeat in fp32 (gaussian means, stratified spacing bins, searchsorted indices, resampled bins,
copied columns, sdf, feature = geo + mlp_out) are compared bit for bit.

Hash-grid features use the fixed-cells technique of camera_opt_cases._FixedCells: the grid cells and interpolation
offsets are the kernel's fp32 ones (an fp32 restatement of the contraction, and for actor samples of the kernel's
world -> box frame, render_trace_cases.ActorFrames, reproduces them bit for bit), the blend and the level weight are
float64."""
import functools

import numpy as np
import torch

import neurad_studio_b200 as nsb
from neurad_studio_b200 import scene
from neurad_studio_b200.lib import FIELD_MAIN, FIELD_PROP0, FIELD_PROP1
from oracle import neurad_oracle as O
from oracle import simple_oracle as SO
from tests import ray_ops_cases as RO
from tests import render_trace_cases as RT
from tests.ray_ops_cases import TINY, U, _bits_equal, _ratio

F32_MAX_BELOW_1 = float(np.nextafter(np.float32(1.0), np.float32(0.0)))
SPACINGS = ("uniform", "lindisp", "power", "sqrt", "log")
_f = RT._f


def f32(x):
    """The fp32 value a float constant has once the kernel receives it."""
    return float(np.float32(x))


def backend(dev, cfg=None, params=None):
    be = RO.backend(dev)
    if cfg is not None:
        be.load_params(cfg, params)
    return be


def _dv(dev):
    return torch.device(dev, 0) if dev == "cuda" else torch.device("cpu")


# ====================================================================================== first-order error chains
class _E:
    """A float64 value v and a bound e on the absolute error of the kernel's fp32 value of it.  The functions below are
    one fp32 operation each: the result's rounding (U of it, or the function's ulp bound) plus the inputs' errors
    carried by the derivative, so an ill-conditioned step (a cancelling subtraction, 1 / t near t = 0) shows its
    condition factor in e."""

    def __init__(self, v, e=None):
        self.v = v
        self.e = torch.zeros_like(v) if e is None else e


def const(x, like, rounded=False):
    """A constant: exact (an fp32 number, e.g. lam or scaling as received), or `rounded` to fp32 by the host (1 U)."""
    v = torch.full_like(like, float(x))
    return _E(v, U * v.abs() if rounded else None)


def e_add(a, b):
    v = a.v + b.v
    return _E(v, a.e + b.e + U * v.abs())


def e_sub(a, b):
    v = a.v - b.v
    return _E(v, a.e + b.e + U * v.abs())


def e_mul(a, b):
    v = a.v * b.v
    return _E(v, a.v.abs() * b.e + b.v.abs() * a.e + U * v.abs())


def e_div(a, b):
    v = a.v / b.v
    return _E(v, (a.e + v.abs() * b.e) / b.v.abs() + U * v.abs())


def e_sqrt(a):
    v = a.v.sqrt()
    return _E(v, torch.where(a.e == 0, torch.zeros_like(v), a.e / (2 * v)) + U * v)


def e_log(a):  # logf: <= 1 ulp of the result
    v = a.v.log()
    return _E(v, a.e / a.v.abs() + 2 * U * v.abs() + TINY)


def e_exp(a):  # expf: <= 2 ulp
    v = a.v.exp()
    return _E(v, v * a.e + 4 * U * v)


def e_pow(a, p, p_rel=0.0):
    """powf(a, p32) (<= 4 ulp), p32 = p (1 + p_rel): the rounded exponent moves the result by |v ln a p| p_rel."""
    v = a.v ** p
    return _E(v, (v * p / a.v).abs() * a.e + 8 * U * v.abs() + (v * a.v.log() * p).abs() * p_rel)


def e_fmax(a, c):  # 1-Lipschitz
    return _E(torch.clamp_min(a.v, c), a.e)


def spacing_apply(kind, x, lam, scaling):
    """spacing_apply of b200nerf.cu (spacing_fn of nff_device.h for "power")."""
    if kind == "uniform":
        return x
    if kind == "lindisp":
        return e_div(const(1.0, x.v), x)
    if kind == "sqrt":
        return e_sqrt(x)
    if kind == "log":
        return e_log(x)
    lam_1 = abs(lam - 1.0)
    t = e_add(e_div(e_mul(x, const(scaling, x.v)), const(lam_1, x.v, True)), const(1.0, x.v))
    p = e_div(const(1.0, x.v), t) if lam == -1.0 else e_pow(t, lam)
    return e_mul(const(lam_1 / lam, x.v, True), e_sub(p, const(1.0, x.v)))


def spacing_invert(kind, y, lam, scaling):
    """spacing_invert of b200nerf.cu (spacing_fn_inv of nff_device.h for "power", both branches)."""
    if kind == "uniform":
        return y
    if kind == "lindisp":
        return e_div(const(1.0, y.v), y)
    if kind == "sqrt":
        return e_mul(y, y)
    if kind == "log":
        return e_exp(y)
    lam_1 = const(abs(lam - 1.0), y.v, True)
    one = const(1.0, y.v)
    if lam == -1.0:
        t = e_fmax(e_add(e_mul(y, const(-0.5, y.v)), one), 1e-10)
        return e_div(e_mul(e_sub(e_div(one, t), one), lam_1), const(scaling, y.v))
    t = e_fmax(e_add(e_div(e_mul(y, const(lam, y.v)), lam_1), one), 1e-10)
    p32 = f32(1.0 / lam)
    r = e_mul(e_sub(e_pow(t, 1.0 / lam, abs(p32 * lam - 1.0)), one), lam_1)
    return e_div(r, const(scaling, y.v))


def to_euclid_bound(kind, u, nears, fars, lam, scaling):
    """The kernel's bins_e = g^-1(u g(far) + (1 - u) g(near)) as an _E chain on the fp32 u [n, E], nears / fars [n]."""
    u = _E(u.double())
    n = u.v.shape[0]
    nr = torch.zeros(n, 1, dtype=torch.float64) if nears is None else nears.double().reshape(n, 1)
    s_near = spacing_apply(kind, _E(nr.expand_as(u.v).clone()), lam, scaling)
    s_far = spacing_apply(kind, _E(fars.double().reshape(n, 1).expand_as(u.v).clone()), lam, scaling)
    y = e_add(e_mul(u, s_far), e_mul(e_sub(const(1.0, u.v), u), s_near))
    return spacing_invert(kind, y, lam, scaling)


def euclid_reference(kind, u, nears, fars, lam, scaling):
    """spacing_to_euclidean_fn (ray_samplers.py:119-120) in float64 (oracle/simple_oracle.spacing_fns) on the fp32 u."""
    fn, inv = SO.spacing_fns({"uniform": SO.SPACING_UNIFORM, "lindisp": SO.SPACING_LINDISP, "power": SO.SPACING_POWER,
                              "sqrt": SO.SPACING_SQRT, "log": SO.SPACING_LOG}[kind], lam, scaling)
    n = u.shape[0]
    nr = torch.zeros(n, 1, dtype=torch.float64) if nears is None else nears.double().reshape(n, 1)
    u64 = u.double()
    return inv(u64 * fn(fars.double().reshape(n, 1)) + (1 - u64) * fn(nr))


def check_euclid(got, u, nears, fars, kind, lam, scaling, what):
    """bins_e per entry against euclid_reference with the to_euclid_bound chain.  Where the chain has no finite bound (log
    / lindisp spacing of a zero near: g(0) = -inf / inf, so the inverse gives exactly 0, or NaN where u = 1 meets
    0 * inf) the kernel must give exactly the reference's value."""
    ref = euclid_reference(kind, u, nears, fars, lam, scaling)
    tol = to_euclid_bound(kind, u, nears, fars, lam, scaling).e + TINY
    g = got.detach().cpu().double().reshape(ref.shape)
    fin = torch.isfinite(ref) & torch.isfinite(tol)
    bad = ~fin & ~((g.isnan() & ref.isnan()) | (g == ref))
    assert not bad.any(), f"{what}: {int(bad.sum())} entries without a finite bound differ from the reference"
    return _ratio(g[fin], ref[fin], tol[fin], what)


# ====================================================================================== isotropic_gaussian
def gaussian_inputs(n, S, seed):
    gen = torch.Generator().manual_seed(seed)
    o = torch.randn(n, 3, generator=gen) * 20
    d = torch.nn.functional.normalize(torch.randn(n, 3, generator=gen), dim=-1)
    area = torch.rand(n, generator=gen) * 1e-5 + 1e-8
    e = torch.sort(torch.rand(n, S + 1, generator=gen), 1).values ** 2 * 2000.0 + 0.05
    if S > 1:
        e[0::5, 1] = e[0::5, 0]  # a zero-width bin: std 0
    return o, d, area, e


def check_gaussian(mean, std, o, d, area, e, what):
    """mean bit for bit against get_fast_isotropic_gaussian restated in fp32 (render_trace_cases._gauss32: md = fl(e1 -
    e0) / 2, t = fl(e0 + md), fl(o + fl(d t))); std = cbrtf(fl(fl(area fl(t t)) md)) per entry against float64 cbrt of
    the same product of the fp32 inputs: the product's 4 roundings, md's subtraction and t's addition entering twice
    (8 U relative), a third of it through the cube root, plus cbrtf (STD_REL's 3e-7) and nothing else."""
    o, d, area, e = o.float().cpu(), d.float().cpu(), area.float().cpu().reshape(-1), e.float().cpu()
    _bits_equal(mean.reshape(e.shape[0], e.shape[1] - 1, 3), RT._gauss32(o, d, area, e), what + " mean")
    _, ref = RT._gauss64(o, d, area, e)
    return _ratio(std, ref, (8 * U / 3 + 3e-7) * ref + TINY, what + " std")


def gaussian_case(dev, n, S, seed=0):
    be = backend(dev)
    o, d, area, e = gaussian_inputs(n, S, seed)
    v = _dv(dev)
    mean, std = be.isotropic_gaussian(o.to(v), d.to(v), area.to(v), e.to(v))
    return check_gaussian(mean, std, o, d, area, e, f"gaussian n={n} S={S}")


# ====================================================================================== stratified spacing samples
def stratified_bins_s(S, t_rand):
    """train_stratified's spacing bins in fp32 (oracle/simple_oracle.spaced_sample: linspace, midpoints,
    lower + (upper - lower) t) -- the kernel's op sequence."""
    bins, _ = SO.spaced_sample(torch.zeros(1, 1), torch.ones(1, 1), S, t_rand=t_rand.float())
    return bins.expand(t_rand.shape[0], S + 1)


def check_stratified(bins_s, bins_e, nears, fars, S, t_rand, kind, lam, scaling, what):
    _bits_equal(bins_s, stratified_bins_s(S, t_rand.cpu()).contiguous(), what + " bins_s")
    return check_euclid(bins_e, bins_s.cpu().float(), None if nears is None else nears.cpu(), fars.cpu(), kind, lam, scaling,
                        what + " bins_e")


def stratified_inputs(n, S, rand_cols, seed, t_kind="random"):
    gen = torch.Generator().manual_seed(seed)
    nears = torch.rand(n, generator=gen) * 2 + 0.05
    fars = nears + torch.exp(torch.rand(n, generator=gen) * 9)
    fars[0] = 20000.0  # the sky distance
    if t_kind == "zero":
        t = torch.zeros(n, rand_cols)
    elif t_kind == "max":
        t = torch.full((n, rand_cols), F32_MAX_BELOW_1)
    else:
        t = torch.rand(n, rand_cols, generator=gen)
    return nears, fars, t


def stratified_case(dev, n, S, kind, lam, with_nears, rand_cols, t_kind, seed=0):
    be = backend(dev)
    nears, fars, t = stratified_inputs(n, S, 1 if rand_cols in (1, "single") else S + 1, seed, t_kind)
    v = _dv(dev)
    scaling = f32(0.1)
    bs, be_ = be.spaced_sample_stratified(nears.to(v) if with_nears else None, fars.to(v), S, t.to(v), kind, lam, scaling)
    return check_stratified(bs, be_, nears if with_nears else None, fars, S, t, kind, lam, scaling,
                            f"stratified {kind} lam={lam} nears={with_nears} cols={t.shape[1]} t={t_kind} S={S}")


def spacing_to_euclidean_case(dev, n, E, kind, lam, with_nears, seed=0):
    """Arbitrary per-ray spacing edges (sorted uniform numbers, with 0 and 1 and the largest float below 1)."""
    be = backend(dev)
    nears, fars, _ = stratified_inputs(n, E, 1, seed)
    gen = torch.Generator().manual_seed(seed + 1)
    u = torch.sort(torch.rand(n, E, generator=gen), 1).values
    u[:, 0], u[0::3, -1], u[1::3, -1] = 0.0, 1.0, F32_MAX_BELOW_1
    v = _dv(dev)
    scaling = f32(0.1)
    got = be.spacing_to_euclidean(u.to(v), nears.to(v) if with_nears else None, fars.to(v), kind, lam, scaling)
    return check_euclid(got, u, nears if with_nears else None, fars, kind, lam, scaling,
                        f"spacing_to_euclidean {kind} lam={lam} nears={with_nears} E={E}")


# ====================================================================================== pdf resampling
def pdf_quantiles(S_new, rand):
    """The kernel's u: fl(linspace(0, 1 - 1/nb, nb) + fl(rand / nb)) (nb = S_new + 1; rand [n, 1] or [n, nb])."""
    nb = S_new + 1
    base = torch.linspace(0.0, 1.0 - (1.0 / nb), steps=nb)
    return (base[None, :] + rand.float().cpu() / _f(float(nb))).expand(rand.shape[0], nb).contiguous()


def cdf_reference(w, hp):
    """The cdf in float64 (ray_samplers.py:339-349, the kernel's fp32 hist_pad and 1e-5) and its bound:
      a_s = fl(w_s + hp):                         U |a_s|
      tot = any-order sum of the S a_s:           E_tot = S U sum |a| + sum U |a|
      padding = max(1e-5 - tot, 0); pe = fl(padding / S); tot' = fl(tot + padding):  E_tot' = 2 E_tot + U (pad + tot')
      pdf_s = fl(fl(a_s + pe) / tot'):            E_pdf = (U |a| + E_pe + U |a + pe|) / tot' + pdf E_tot' / tot' + U pdf
      cdf_{s+1} = min(1, warp-scan sum of pdf_0..s plus the carry):  sum E_pdf + (s + 2) U sum pdf."""
    w64 = w.double().cpu()
    n, S = w64.shape
    hp32, eps = f32(hp), f32(1e-5)
    a = w64 + hp32
    tot = a.sum(1, keepdim=True)
    E_tot = S * U * a.abs().sum(1, keepdim=True) + U * a.abs().sum(1, keepdim=True)
    pad = torch.relu(eps - tot)
    E_pad = torch.where(eps - tot + E_tot > 0, E_tot + U * pad, torch.zeros_like(pad))
    pe = pad / S
    E_pe = E_pad / S + U * pe
    tot2 = tot + pad
    E_tot2 = E_tot + E_pad + U * tot2
    num = a + pe
    pdf = num / tot2
    E_pdf = (U * a.abs() + E_pe + U * num.abs() + pdf * E_tot2) / tot2 + U * pdf
    k = torch.arange(S, dtype=torch.float64)
    cdf = torch.cat([torch.zeros(n, 1, dtype=torch.float64), torch.cumsum(pdf, 1).clamp_max(1.0)], 1)
    E = torch.cat([torch.zeros(n, 1, dtype=torch.float64), torch.cumsum(E_pdf, 1) + (k + 2) * U * torch.cumsum(pdf, 1)], 1)
    return cdf, E + TINY


def resample_bits(cdf, inds, bins, uu):
    """The new bins from the kernel's own cdf and indices, op by op in fp32 (pdf_resample_kernel)."""
    S = cdf.shape[1] - 1
    lo = inds.long()
    below, above = (lo - 1).clamp(0, S), lo.clamp_max(S)
    c0, c1 = cdf.gather(1, below), cdf.gather(1, above)
    t = torch.clamp(torch.nan_to_num((uu - c0) / (c1 - c0)), 0.0, 1.0)
    b0, b1 = bins.gather(1, below), bins.gather(1, above)
    return b0 + t * (b1 - b0)


def check_pdf(out, w, bins, S_new, rand, hp, what, u=None):
    """cdf per entry (cdf_reference); inds bit for bit = torch.searchsorted(kernel cdf, u, right=True) (the kernel's
    binary search is torch's); new bins bit for bit from the kernel's cdf and indices.  `u` [n, S_new + 1]: the
    quantiles when no `rand` is drawn (eval mode)."""
    nb, cdf, inds = out
    ref, tol = cdf_reference(w, hp)
    worst = _ratio(cdf, ref, tol, what + " cdf")
    kc = cdf.detach().cpu().float().contiguous()
    uu = pdf_quantiles(S_new, rand) if u is None else u
    _bits_equal(inds, torch.searchsorted(kc, uu, right=True).int(), what + " inds")
    _bits_equal(nb, resample_bits(kc, inds.cpu(), bins.float().cpu().reshape(kc.shape), uu), what + " bins")
    return worst


def pdf_inputs(n, S, S_new, kind, rand_cols, seed):
    """weights [n, S], sorted spacing bins [n, S+1], rand.  kind "random"; "degenerate": rays of all-zero weights and
    single spikes; "unpadded" (run with hist_pad 0): rays of all-zero weights and rays whose weights sum to less than
    1e-5, so the padding branch adds max(1e-5 - tot, 0) spread over the bins; "dyadic": weights k/32 summing to 1 with hist_pad 0 and rand 0, so that u = i / nb lands exactly on
    cdf values (nb a power of two)."""
    gen = torch.Generator().manual_seed(seed)
    bins = torch.sort(torch.rand(n, S + 1, generator=gen), 1).values
    bins[:, 0], bins[:, -1] = 0.0, 1.0
    rand = torch.rand(n, rand_cols, generator=gen)
    if kind == "dyadic":
        assert 32 % S == 0 or S % 32 == 0
        w = torch.zeros(n, S)
        for r in range(n):
            k = torch.randint(0, S, (32,), generator=gen)
            w[r].index_add_(0, k, torch.full((32,), 1.0 / 32))
        return w, bins, torch.zeros(n, rand_cols)
    w = torch.rand(n, S, generator=gen) ** 4
    w[torch.rand(n, S, generator=gen) < 0.2] = 0.0
    if kind == "unpadded":
        w[0::3] = 0.0
        w[1::3] *= 1e-8
        return w, bins, rand
    if kind == "degenerate":
        w[0::3] = 0.0
        w[1::3] = 0.0
        w[1::3, S // 2] = 1.0
        w[2::3] *= 1e-6
    return w, bins, rand


def pdf_case(dev, n, S, S_new, rand_cols, kind="random", seed=0):
    be = backend(dev)
    rc = 1 if rand_cols in (1, "single") else S_new + 1
    w, bins, rand = pdf_inputs(n, S, S_new, kind, rc, seed)
    hp = 0.0 if kind in ("dyadic", "unpadded") else 0.01
    v = _dv(dev)
    out = be.pdf_resample_stratified(w.to(v), bins.to(v), S_new, rand.to(v), histogram_padding=hp)
    worst = check_pdf(out, w, bins, S_new, rand, hp, f"pdf {kind} S={S} S_new={S_new} cols={rc}")
    if kind == "dyadic":
        uu = pdf_quantiles(S_new, rand)
        on = (uu[:, :, None] == out[1].cpu()[:, None, :]).any(-1)
        assert on.sum() > n, "the dyadic case puts no u exactly on a cdf value"
    if kind == "unpadded":
        assert (w.double().sum(1) < f32(1e-5)).sum() >= n // 2, "the case does not reach the padding branch"
    return worst


# ====================================================================================== neurad_encoding
FIELDS = {FIELD_MAIN: ("field", 4), FIELD_PROP0: ("proposal_fields.0", 1), FIELD_PROP1: ("proposal_fields.1", 1)}


def grid_cfg(cfg, field):
    return {FIELD_MAIN: cfg.grid, FIELD_PROP0: cfg.proposal_grid_1, FIELD_PROP1: cfg.proposal_grid_2}[field]


ABSENT = (20, 40)  # keyframes [20, 40) at which actor 2 is absent


@functools.lru_cache(maxsize=2)
def encoding_scene(dev, n_actors, small_actor_tables=False, seed=0):
    """Production grids on the GPU (small actor tables for 64 actors), small tables on the CPU; trajectories with a
    jittered yaw.  With >= 2 actors, actor 1 follows actor 0 1.5 m ahead with the same rotation (overlapping padded
    boxes: the higher index wins); with >= 3, actor 2 is absent at keyframes ABSENT."""
    cfg = nsb.NeuRADConfig(n_actors=n_actors) if dev == "cuda" else nsb.small_config(n_actors=n_actors, log2_main=12, log2_prop=11)
    if small_actor_tables:
        for g in (cfg.grid, cfg.proposal_grid_1, cfg.proposal_grid_2):
            g.actor.log2_hashmap_size = 10
    trajs = scene.make_trajectories(n_actors, cfg.duration, seed=seed) if n_actors else None
    params = scene.make_params(cfg, seed=seed, trajectories=trajs)
    if n_actors >= 2:
        params["dynamic_actors.actor_positions"][:, 1] = params["dynamic_actors.actor_positions"][:, 0] + torch.tensor([1.5, 0.0, 0.0])
        params["dynamic_actors.actor_rotations_6d"][:, 1] = params["dynamic_actors.actor_rotations_6d"][:, 0]
    if n_actors >= 3:
        params["dynamic_actors.actor_present_at_time"][ABSENT[0]:ABSENT[1], 2] = False
    return cfg, params


def encoding_samples(cfg, params, n, S, seed, dirs_per_ray=True):
    """mean [n, S, 3], std [n, S], times [n], directions, flip-free.  Rays of an actor scene put their samples in a box
    1.3 times the padded box of one actor around its centre at the ray's time (about half inside); ray k % 6 == 1 runs
    before the first keyframe, 2 after the last, 3 exactly on a keyframe, 4 inside actor 2's absence, 0 at the
    overlapping actors 0 / 1.  Static samples spread to 400 m (inside and outside the contraction's unit cube); sample 0
    of ray 5 sits at the origin (contracted to 0.5: on the lattice of every even-resolution level) and sample 1 at
    (scale / 2, 0, -scale / 2) (3/8 and 5/8: on the lattice of resolutions that are multiples of 8)."""
    gen = torch.Generator().manual_seed(seed)
    A = cfg.n_actors
    scale = float(params["static_scale"])
    d = torch.nn.functional.normalize(torch.randn(n, 3, generator=gen), dim=-1)
    times = torch.rand(n, generator=gen) * cfg.duration
    std = torch.exp(torch.rand(n, S, generator=gen) * 9.0 - 9.0)
    mean = (torch.rand(n, S, 3, generator=gen) * 2 - 1) * torch.tensor([400.0, 400.0, 30.0])
    if A:
        ts = params["dynamic_actors.unique_timestamps"].float()
        k = torch.arange(n) % 6
        times[k == 1] = ts[0] - 0.5
        times[k == 2] = ts[-1] + 0.5
        times[k == 3] = ts[torch.randint(0, ts.numel(), (int((k == 3).sum()),), generator=gen)]
        if A >= 3:
            times[k == 4] = ts[ABSENT[0]] + (ts[ABSENT[1] - 2] - ts[ABSENT[0]]) * torch.rand(int((k == 4).sum()), generator=gen)
        actor = torch.randint(0, A, (n,), generator=gen)
        actor[k == 0] = torch.randint(0, 2, (int((k == 0).sum()),), generator=gen)
        if A >= 3:
            actor[k == 4] = 2
        p64 = {kk: (v.double() if torch.is_tensor(v) and v.is_floating_point() else v) for kk, v in params.items()}
        b2w, _ = O.boxes2world_at(p64, times.double())
        ray = torch.arange(n)
        R, c = b2w[ray, actor, :3, :3], b2w[ray, actor, :3, 3]
        half = (params["dynamic_actors.actor_sizes"].double() * 0.5 + params["dynamic_actors.actor_padding"].double())[actor]
        box = (torch.rand(n, S, 3, generator=gen, dtype=torch.float64) * 2 - 1) * half[:, None, :] * 1.3
        am = (c[:, None, :] + torch.einsum("nij,nsj->nsi", R, box)).float()
        static_rays = torch.arange(n) % 7 == 6
        mean = torch.where(static_rays[:, None, None], mean, am)
    if n > 5:
        mean[5, 0] = 0.0
        if S > 1:
            mean[5, 1] = torch.tensor([scale * 0.5, 0.0, -scale * 0.5])
    dirs = d if dirs_per_ray else torch.nn.functional.normalize(torch.randn(n, S, 3, generator=gen), dim=-1)
    return mean.contiguous(), std.contiguous(), times, dirs.contiguous()


def flips(n, kind, seed=0):
    if kind == "none":
        return None
    if kind == "plus":
        return torch.ones(n)
    if kind == "minus":
        return -torch.ones(n)
    return (torch.randint(0, 2, (n,), generator=torch.Generator().manual_seed(seed)).float() * 2 - 1)


def box_test(params, cfg, mean, times, dev="cpu"):
    """float64 box test of the means [n, S, 3] at the rays' times [n] (float64 DynamicActors.get_boxes2world, the fp32
    padded half sizes): (geometric containment [n, S, A], presence at a bracketing keyframe [n, 1, A], `near` [n, S]: some
    present actor's box coordinate lies within 64 U (|mean| + |box centre| + half size) of a face)."""
    p64 = {k: (v.double() if torch.is_tensor(v) and v.is_floating_point() else v) for k, v in params.items()}
    b2w, valid = O.boxes2world_at(p64, times.double())
    w2b = O.pose_inverse(b2w)
    bnd = RT.ActorFrames(params, cfg, None, None, times).bounds.double().to(dev)
    m = mean.double().to(dev)
    w2b, b2w, valid = w2b.to(dev), b2w.to(dev), valid.to(dev)
    R, t = w2b[..., :3, :3], w2b[..., :3, 3]
    q = torch.einsum("naij,nsj->nsai", R, m) + t[:, None]
    ok = valid[:, None, :]
    sc = m.abs().amax(-1)[..., None] + b2w[:, :, :3, 3].abs().amax(-1)[:, None, :] + bnd.amax(-1)
    near = (ok[..., None] & ((q.abs() - bnd).abs() <= 64 * U * sc[..., None])).any(-1).any(-1)
    return (q.abs() < bnd).all(-1), ok, near


def actor_id_reference(params, cfg, mean, times, dev="cpu"):
    """The highest actor whose padded box strictly contains the float64 mean, among the actors present at a bracketing
    keyframe (box_test); and box_test's `near`."""
    geo, ok, near = box_test(params, cfg, mean, times, dev)
    inside = geo & ok
    ar = torch.arange(inside.shape[-1], device=inside.device)
    ref = torch.where(inside.any(-1), (inside * (ar + 1)).amax(-1) - 1, torch.full(inside.shape[:-1], -1, device=inside.device))
    return ref.cpu(), near.cpu()


def check_actor_ids(aid, params, cfg, mean, times, what, dev="cpu", chunk=256):
    """Mismatches only at a box face, and at most max(2, 1e-5 of the samples) of them.  Returns the face count."""
    aid = aid.detach().cpu().long()
    faces = 0
    for c0 in range(0, aid.shape[0], chunk):
        c = slice(c0, c0 + chunk)
        ref, near = actor_id_reference(params, cfg, mean[c], times[c], dev)
        bad = aid[c] != ref
        assert not (bad & ~near).any(), (f"{what}: {int((bad & ~near).sum())} samples assigned to the wrong actor away "
                                         f"from every box face, first at {(bad & ~near).nonzero()[:3].tolist()}")
        faces += int(bad.sum())
    assert faces <= max(2, aid.numel() // 100000), f"{what}: {faces} of {aid.numel()} actor ids differ at a box face"
    return faces


def encoding_reference(params, cfg, field, mean, std, times, flip, aid, dev, corrupt=None):
    """float64 features [P, D] and their bounds at the kernel's actor assignment aid [n, S]: static samples at the fp32
    contraction of the mean (RT._contract32), actor samples at the kernel's fp32 box position (RT.ActorFrames.box, x
    negated on flipped rays) through the actor's grid, zero padded to D.  Per level RT._level_terms: three blends of two
    rounded products and a sum plus the rounded 1 - offset (<= 9 U of the interpolation of |f|), the level weight
    rcp.approx(fl(2 res std)) (3 U + STD_REL where 2 res std > 1), the product (U).
    `corrupt` (self-tests): "wrong_axis" flips the box y instead of x, "wrong_keyframe" takes every actor frame from
    the keyframe before the bracket."""
    prefix, F = FIELDS[field]
    gc = grid_cfg(cfg, field)
    n, S = mean.shape[0], mean.shape[1]
    D = gc.static.num_levels * F
    P = n * S
    m32 = mean.float().cpu().reshape(n, S, 3)
    sd64 = std.double().cpu().reshape(P, 1)
    aid = aid.cpu().long().reshape(n, S)
    x = torch.zeros(P, D, dtype=torch.float64, device=dev)
    Ex = torch.zeros_like(x)
    st = (aid < 0).reshape(-1)
    scale = float(params["static_scale"])
    if st.any():
        c32 = RT._contract32(m32.reshape(P, 3)[st], scale)
        _, cs = O.scaled_contraction(m32.reshape(P, 3)[st].double(), sd64[st], scale)
        v, vabs, lw, t = RT._grid(params[f"{prefix}.hashgrid.static_grid.hash_table"], F, gc.static.hash_table_size,
                                  params[f"{prefix}.hashgrid.static_grid.scalings"], c32, cs[:, 0], dev)
        xs, Es = RT._level_terms(v, vabs, lw, t)
        x[st.to(dev)], Ex[st.to(dev)] = xs.reshape(-1, D), Es.reshape(-1, D)
    if (~st).any():
        tt = times.float().cpu().reshape(-1)
        if corrupt == "wrong_keyframe":
            ts = params["dynamic_actors.unique_timestamps"].float()
            r = torch.searchsorted(ts, tt).clamp(1, ts.numel() - 1)
            tt = ts[r - 1] - 1e-3  # the keyframe before the bracket
        fr = RT.ActorFrames(params, cfg, None, None, tt)
        q32, _ = fr.box(m32, aid.clamp_min(0))
        if flip is not None:
            ax = 1 if corrupt == "wrong_axis" else 0
            q32[..., ax] = torch.where(flip.cpu().reshape(n, 1) < 0, -q32[..., ax], q32[..., ax])
        q32 = q32.reshape(P, 3)[~st]
        c32 = RT._contract32(q32, float(gc.actor_scale))
        _, cs = O.scaled_contraction(q32.double(), sd64[~st], float(gc.actor_scale))
        La, T = gc.actor.num_levels, gc.actor.hash_table_size
        base = aid.reshape(-1)[~st] * La * T
        v, vabs, lw, t = RT._grid(RT._actor_tables(params, prefix, cfg.n_actors), F, T, params[f"{prefix}.hashgrid.actor_grids.0.scalings"],
                                  c32, cs[:, 0], dev, base)
        xa, Ea = RT._level_terms(v, vabs, lw, t)
        k = La * F
        x[(~st).to(dev), :k], Ex[(~st).to(dev), :k] = xa.reshape(-1, k), Ea.reshape(-1, k)
    return x, Ex


def density_reference(params, field, x, Ex):
    """density = expf(acc), acc the sequential fmaf over the D decoder terms: E_acc = sum |dec| E_x + D U sum |dec x|;
    expf: 4 U relative; first order."""
    prefix, _ = FIELDS[field]
    dec = params[f"{prefix}.density_decoder.weight"].reshape(-1).double().to(x.device)
    terms = x * dec
    acc = terms.sum(-1)
    E = (Ex * dec.abs()).sum(-1) + x.shape[1] * U * terms.abs().sum(-1)
    dens = acc.exp()
    return dens.cpu(), (dens * (E + 4 * U) + TINY).cpu()


def directions_reference(params, cfg, dirs, times, aid, flip, n, S):
    """Static samples: the input direction, bit for bit.  Actor samples: q = R d with the kernel's fp32 frame, float64
    q / (|q| + 1e-7) (fp32 1e-7), x negated on flipped rays: three products and two sums per component, the norm and
    the division, <= 16 U of a unit vector's components."""
    d = dirs.float().cpu()
    d = d[:, None, :].expand(n, S, 3) if d.numel() == 3 * n and S != 1 else d.reshape(n, S, 3)
    aid = aid.cpu().long().reshape(n, S)
    act = aid >= 0
    ref = d.double().clone()
    if act.any():
        fr = RT.ActorFrames(params, cfg, None, None, times.float().cpu().reshape(-1))
        _, R = fr.box(torch.zeros(n, S, 3), aid.clamp_min(0))
        q = (R.double() @ d.double()[..., None])[..., 0]
        r = q / (q.norm(dim=-1, keepdim=True) + f32(1e-7))
        if flip is not None:
            r[..., 0] = torch.where(flip.cpu().reshape(n, 1) < 0, -r[..., 0], r[..., 0])
        ref[act] = r[act]
    return d, ref, act


def check_encoding(be, params, cfg, field, mean, std, times, dirs, flip, out, dev, what, chunk=1 << 17):
    """One neurad_encoding call's outputs (whichever it returned) against the references above, at the kernel's own
    actor assignment (queried from the same kernel with want_actor_id); the assignment against actor_id_reference.
    Returns (worst ratio, face exceptions)."""
    n, S = mean.shape[0], mean.shape[1]
    mean = mean.reshape(n, S, 3)
    t_ray = None if times is None else times.reshape(n, -1)[:, 0].float().cpu()
    if cfg.n_actors:
        aid = out.get("actor_id")
        if aid is None:
            aid = be.neurad_encoding(field, mean, std, times, None, want_features=False, want_actor_id=True, flip=flip)["actor_id"]
        aid = aid.cpu().reshape(n, S)
        faces = check_actor_ids(aid, params, cfg, mean.cpu(), t_ray, what + " actor_id", dev, 256 if dev == "cpu" else 4096)
    else:
        aid = torch.full((n, S), -1, dtype=torch.int32)
        faces = 0
        if "actor_id" in out:
            _bits_equal(out["actor_id"], aid, what + " actor_id (no actors)")
    worst = 0.0
    R = max(1, chunk // S)
    for r0 in range(0, n, R):
        rs = slice(r0, min(n, r0 + R))
        m_, sd_ = mean[rs].cpu(), std.reshape(n, S)[rs].cpu()
        fl_ = None if flip is None else flip.reshape(n)[rs]
        x, Ex = encoding_reference(params, cfg, field, m_, sd_, t_ray[rs] if t_ray is not None else None, fl_, aid[rs], dev)
        P = x.shape[0]
        if "features" in out:
            got = out["features"].reshape(n * S, -1)[r0 * S: r0 * S + P]
            worst = max(worst, _ratio(got, x.cpu(), Ex.cpu(), what + " features"))
        if "density" in out:
            dens, tol = density_reference(params, field, x, Ex)
            worst = max(worst, _ratio(out["density"].reshape(n * S)[r0 * S: r0 * S + P], dens, tol, what + " density"))
    if "directions" in out:
        d, ref, act = directions_reference(params, cfg, dirs, t_ray, aid, flip, n, S)
        got = out["directions"].detach().cpu().reshape(n, S, 3)
        _bits_equal(got[~act], d[~act].contiguous(), what + " static directions")
        if act.any():
            worst = max(worst, _ratio(got[act], ref[act], torch.full_like(ref[act], 16 * U), what + " actor directions"))
    return worst, faces


def encoding_case(dev, field, n_actors, n, S, flip_kind="mixed", dirs_per_ray=True, seed=0):
    cfg, params = encoding_scene(dev, n_actors, small_actor_tables=n_actors > 32)
    be = backend(dev, cfg, params)
    mean, std, times, dirs = encoding_samples(cfg, params, n, S, seed, dirs_per_ray)
    fl = flips(n, flip_kind, seed)
    v = _dv(dev)
    to = (lambda t: None if t is None else t.to(v))  # noqa: E731
    main = field == FIELD_MAIN
    out = be.neurad_encoding(field, to(mean), to(std), to(times), to(dirs) if main else None, want_features=True,
                             want_density=not main, want_actor_id=n_actors > 0, flip=to(fl))
    worst, faces = check_encoding(be, params, cfg, field, mean, std, times, dirs if main else None, fl, out, dev,
                                  f"encoding field={field} actors={n_actors} n={n} S={S} flip={flip_kind}")
    if n_actors:
        aid = out["actor_id"].cpu()
        assert (aid >= 0).any() and (aid < 0).any(), "the case reaches no actor sample or no static sample"
        overlap = absent = 0
        for r0 in range(0, n, 512):
            r = slice(r0, r0 + 512)
            geo, ok, near = box_test(params, cfg, mean[r], times[r], dev)
            geo, ok, far = geo.cpu(), ok.cpu(), ~near.cpu()  # far from every face: the kernel's fp32 test agrees
            if n_actors >= 2:  # inside both padded boxes, actors 0 and 1 present: the higher index must win
                both = geo[..., 0] & geo[..., 1] & ok[..., 0] & ok[..., 1]
                overlap += int((both & (aid[r] == 1)).sum())
                assert not (both & far & (aid[r] != 1)).any(), "a sample in the overlap of actors 0 / 1 did not go to actor 1"
            if n_actors >= 3:  # inside actor 2's box while it is absent at both bracketing keyframes
                gone = geo[..., 2] & ~ok[..., 2]
                absent += int(gone.sum())
                assert not (gone & far & (aid[r] == 2)).any(), "actor 2 was used while absent at both bracketing keyframes"
        if n_actors >= 2:
            assert overlap > 0, "no sample lies in the overlap of actors 0 and 1"
        if n_actors >= 3:
            assert absent > 0, "no sample lies in actor 2's box while it is absent"
    sc = grid_cfg(cfg, field).static.scalings().float()
    p = RT._contract32(mean.reshape(-1, 3), float(params["static_scale"]))[:, None, :] * sc[None, :, None]
    assert (p == torch.floor(p)).all(-1).any(), "no sample on a level's lattice"
    return worst, faces


# ====================================================================================== field mid / tail
def check_field_mid(x2, geo, dirs, what):
    """geo columns bit for bit; SH4((d + 1) / 2) per entry against float64 (RT._sh4_64): polynomials of degree <= 3 on
    [0, 1]^3 with terms <= 3, <= 24 U each after the 3 U of (d + 1) / 2 (Lipschitz <= 10): 72 U + 10 U."""
    G = geo.shape[1] - 1
    x2 = x2.detach().cpu()
    _bits_equal(x2[:, :G].contiguous(), geo.cpu()[:, 1:].contiguous(), what + " geo columns")
    ref = RT._sh4_64((dirs.double().cpu().reshape(-1, 3) + 1) / 2)
    return _ratio(x2[:, G:], ref, torch.full_like(ref, 82 * U), what + " SH columns")


def check_field_tail(out, geo, h, beta, what):
    """feature = fl(geo + h) and sdf bit for bit; alpha = rcp(1 + expf(fl(sdf beta))) per entry (RT.alpha_reference:
    0 where expf overflows, as the fp32 formula gives); sdf beta at +-200: alpha exactly 0 and exactly 1."""
    feature, sdf, alpha = out
    g, hh = geo.float().cpu(), h.float().cpu()
    _bits_equal(feature, g[:, 1:] + hh, what + " feature")
    _bits_equal(sdf.reshape(-1), g[:, 0].contiguous(), what + " sdf")
    a, tol = RT.alpha_reference(g[:, 0], beta)
    worst = _ratio(alpha.reshape(-1), a, tol, what + " alpha")
    x = g[:, 0].double() * beta
    sat = x.abs() > 150
    _bits_equal(alpha.reshape(-1)[sat].contiguous(), (x[sat] < 0).float(), what + " alpha at the overflow ends")
    return worst


def field_case(dev, n, G, seed=0):
    cfg = nsb.small_config()
    params = scene.make_params(cfg, beta=20.0)
    be = backend(dev, cfg, params)
    gen = torch.Generator().manual_seed(seed)
    geo = torch.randn(n, G + 1, generator=gen)
    geo[:, 0] *= 0.3
    geo[0::7, 0] = -200.0 / be._beta
    geo[1::7, 0] = 200.0 / be._beta
    dirs = torch.nn.functional.normalize(torch.randn(n, 3, generator=gen), dim=-1)
    dirs[2::7] = torch.tensor([0.0, 0.0, -1.0])
    h = torch.randn(n, G, generator=gen)
    v = _dv(dev)
    what = f"field n={n} G={G}"
    w = check_field_mid(be._field_mid(geo.to(v), dirs.to(v)), geo, dirs, what)
    return max(w, check_field_tail(be._field_tail(geo.to(v), h.to(v)), geo, h, f32(be._beta), what))


# ====================================================================================== MLPs
def mlp_reference(x, ws, bs, dev, gamma=RT.gamma_tc, corrupt_row=None):
    """Per layer y = W a + b with E_y = gamma(K) (|W| |a| + |b|) + |W| E_a (render_trace_cases.main_field_reference's
    carry), ReLU between layers (1-Lipschitz; a unit below minus its bound carries none).  Returns (y, E_y, [(z_l,
    E_z_l)] of the hidden pre-activations)."""
    a = x.double().to(dev).reshape(-1, x.shape[-1])
    Ea = torch.zeros_like(a)
    hidden = []
    for l, (w, b) in enumerate(zip(ws, bs)):
        w, b = w.double().to(dev), (torch.zeros(w.shape[0]) if b is None else b).double().to(dev)
        y = a @ w.T + b
        E = gamma(w.shape[1]) * (a.abs() @ w.abs().T + b.abs()) + Ea @ w.abs().T
        if l == len(ws) - 1:
            return y, E, hidden
        hidden.append((y, E))
        a, Ea = y.clamp_min(0), torch.where(y + E <= 0, torch.zeros_like(E), E)


def check_mlp(out, x, ws, bs, dev, what, chunk=1 << 18):
    y, zs = out
    worst = 0.0
    n = x.reshape(-1, x.shape[-1]).shape[0]
    xs = x.reshape(n, -1)
    for r0 in range(0, n, chunk):
        r = slice(r0, r0 + chunk)
        ry, Ey, hid = mlp_reference(xs[r], ws, bs, dev)
        assert len(zs) in (0, len(hid)), f"{what}: {len(zs)} hidden outputs for {len(hid)} hidden layers"
        worst = max(worst, _ratio(y.reshape(n, -1)[r], ry.cpu(), Ey.cpu(), what + " output"))
        for l, (z, Ez) in enumerate(hid[:len(zs)]):
            worst = max(worst, _ratio(zs[l].reshape(n, -1)[r], z.cpu(), Ez.cpu(), what + f" hidden {l}"))
    return worst


def check_dgrad(dx, dy, w, relu_z, dev, what):
    """dX = dY W per entry, gamma_tc(out) |dY| |W|; masked by (relu_z > 0) (masked entries exactly 0)."""
    ref = dy.double().to(dev) @ w.double().to(dev)
    tol = RT.gamma_tc(w.shape[0]) * (dy.double().abs().to(dev) @ w.double().abs().to(dev))
    ref, tol = ref.cpu(), tol.cpu()
    if relu_z is not None:
        m = ~(relu_z.cpu().reshape(ref.shape) > 0)
        _bits_equal(dx.detach().cpu()[m].contiguous(), torch.zeros(int(m.sum())), what + " masked entries")
        ref, tol = torch.where(m, torch.zeros_like(ref), ref), torch.where(m, torch.ones_like(tol), tol)
    return _ratio(dx, ref, tol, what + " dX")


def neurad_mlps(seed=0):
    cfg = nsb.small_config()
    p = scene.make_params(cfg, seed=seed)
    geo = [p["field.mlp_geo.layers.0.weight"], p["field.mlp_geo.layers.1.weight"]], [p["field.mlp_geo.layers.0.bias"], p["field.mlp_geo.layers.1.bias"]]
    feat = ([p[f"field.mlp_feature.layers.{i}.weight"] for i in range(3)], [p[f"field.mlp_feature.layers.{i}.bias"] for i in range(3)])
    return {"geo": geo, "feature": feat}


def mlp_case(dev, which, rows, seed=0):
    """NeuRAD's mlp_geo 32-32-33 and mlp_feature 48-32-32-32 with want_hidden, then mlp_dgrad of the last layer (with the
    ReLU mask of the hidden pre-activation) on the same rows."""
    be = backend(dev)
    ws, bs = neurad_mlps(seed)[which]
    gen = torch.Generator().manual_seed(seed + rows)
    x = torch.randn(rows, ws[0].shape[1], generator=gen)
    v = _dv(dev)
    y, zs = be.mlp_fwd(x.to(v), [w.to(v) for w in ws], [b.to(v) for b in bs], want_hidden=True)
    what = f"mlp_{which} rows={rows}"
    worst = check_mlp((y, zs), x, ws, bs, dev, what)
    dy = torch.randn(rows, ws[-1].shape[0], generator=gen)
    dx = be.mlp_dgrad(dy.to(v), ws[-1].to(v), zs[-1])
    return max(worst, check_dgrad(dx, dy, ws[-1], zs[-1], dev, what))


# ====================================================================================== one recorded training step
RECORDED = ("spaced_sample_stratified", "isotropic_gaussian", "neurad_encoding", "pdf_resample_stratified", "spacing_to_euclidean",
            "_field_mid", "_field_tail", "mlp_fwd", "mlp_dgrad", "alpha_to_weights", "density_to_weights")


def _snap(x):
    if torch.is_tensor(x):
        return x.detach().clone()
    if isinstance(x, (list, tuple)):
        return type(x)(_snap(v) for v in x)
    if isinstance(x, dict):
        return {k: _snap(v) for k, v in x.items()}
    return x


class Recorder:
    """Wraps the listed methods of one backend instance; every call's arguments and results are copied (the module walk
    edits some tensors in place afterwards, e.g. the last edge moved to the sky)."""

    def __init__(self, be, methods=RECORDED):
        self.be, self.methods, self.calls = be, tuple(methods), []

    def __enter__(self):
        for name in self.methods:
            orig = getattr(self.be, name)

            def wrap(*a, _orig=orig, _name=name, **k):
                out = _orig(*a, **k)
                self.calls.append((_name, _snap(a), _snap(k), _snap(out)))
                return out

            setattr(self.be, name, wrap)
        return self

    def __exit__(self, *exc):
        for name in self.methods:
            delattr(self.be, name)


def training_scene(dev, n_actors=8, seed=0):
    cfg = nsb.NeuRADConfig(n_actors=n_actors) if dev == "cuda" else nsb.small_config(n_actors=n_actors, log2_main=12, log2_prop=11)
    trajs = scene.make_trajectories(n_actors, cfg.duration, seed=seed)
    return cfg, trajs, scene.make_params(cfg, seed=seed, beta=3.0, sdf_bias=0.6, trajectories=trajs)


def record_training_step(dev, n_cam, n_lidar, seed=0, methods=RECORDED):
    """model.train(); get_nff_outputs(fused=False) on a seeded scene with actors, then backward of a simple loss (so that
    mlp_dgrad is called too); returns (cfg, params, backend, the recorded calls of `methods`)."""
    from neurad_studio_b200 import nerfstudio_api as NA

    cfg, trajs, params = training_scene(dev, seed=seed)
    v = _dv(dev)
    model = NA.NeuRADModel(cfg, trajs).to(v)
    model.load_reference_state_dict(params)
    model.requires_grad_(True)
    model.train()
    rays = scene.random_rays(n_cam + n_lidar, cfg, seed=seed + 3, trajectories=trajs)
    is_lidar = torch.zeros(n_cam + n_lidar, 1, dtype=torch.bool)
    is_lidar[n_cam:] = True
    rb = NA.RayBundle(origins=rays["origins"].to(v), directions=rays["directions"].to(v), pixel_area=rays["pixel_area"].to(v),
                      times=rays["times"].to(v), metadata={"is_lidar": is_lidar.to(v), "sensor_idxs": rays["sensor_idx"].to(v)})
    orig = NA.get_backend
    if dev == "cpu":  # the model binds the fake backend (tests/fake_backend.py)
        fake = backend(dev)
        NA.get_backend = lambda device: fake
    try:
        be = model._bind()
        torch.manual_seed(seed)
        with Recorder(be, methods) as rec:
            out = model.get_nff_outputs(rb, fused=False)
            (out["features"].square().mean() + out["depth"].mean() * 1e-3).backward()
    finally:
        NA.get_backend = orig
    return cfg, params, be, rec.calls


def check_recorded_call(name, a, k, out, be, cfg, params, dev):
    """The comparator of one recorded call, from that call's own arguments.  Returns (worst ratio, face exceptions)."""
    what = f"recorded {name}"
    if name == "isotropic_gaussian":
        o, d, area, e = a
        return check_gaussian(*out, o.reshape(-1, 3), d.reshape(-1, 3), area, e, what), 0
    if name == "spaced_sample_stratified":
        nears, fars, S, t_rand = a[:4]
        kind, lam, scaling = (list(a[4:]) + [k.get("spacing", "uniform"), k.get("power_lambda", -1.0), k.get("power_scaling", 0.1)][len(a[4:]):])
        return check_stratified(out[0], out[1], None if nears is None else nears.reshape(-1), fars.reshape(-1), S,
                                t_rand.reshape(fars.numel(), -1), kind, f32(lam), f32(scaling), what), 0
    if name == "spacing_to_euclidean":
        bins_s, nears, fars = a[:3]
        kind, lam, scaling = (list(a[3:]) + [k.get("spacing", "power"), k.get("power_lambda", -1.0), k.get("power_scaling", 0.1)][len(a[3:]):])
        return check_euclid(out, bins_s.float().cpu(), None if nears is None else nears.reshape(-1).cpu(), fars.reshape(-1).cpu(),
                            kind, f32(lam), f32(scaling), what), 0
    if name == "pdf_resample_stratified":
        w, bins, S_new, rand = a[:4]
        hp = a[4] if len(a) > 4 else k.get("histogram_padding", 0.01)
        return check_pdf(out, w, bins, S_new, rand.reshape(w.shape[0], -1), hp, what), 0
    if name == "neurad_encoding":
        names = ("field", "mean", "std", "times", "directions", "want_features", "want_density", "want_actor_id", "flip")
        kw = dict(zip(names, a))
        kw.update(k)
        return check_encoding(be, params, cfg, kw["field"], kw["mean"], kw["std"], kw.get("times"), kw.get("directions"),
                              kw.get("flip"), out, dev, what + f" field {kw['field']}")
    if name == "_field_mid":
        return check_field_mid(out, a[0], a[1], what), 0
    if name == "_field_tail":
        return check_field_tail(out, a[0], a[1], f32(be._beta), what), 0
    if name == "mlp_fwd":
        x, ws = a[0], a[1]
        bs = a[2] if len(a) > 2 else k.get("biases")
        bs = bs if bs is not None else [None] * len(ws)
        if not (k.get("want_hidden") or (len(a) > 3 and a[3])):
            out = (out, [])
        return check_mlp(out, x, ws, bs, dev, what + f" {len(ws)} layers"), 0
    if name == "mlp_dgrad":
        dy, w = a[0], a[1]
        z = a[2] if len(a) > 2 else k.get("relu_z")
        return check_dgrad(out, dy.reshape(-1, dy.shape[-1]), w, z, dev, what), 0
    if name == "alpha_to_weights":
        al = a[0].reshape(a[0].shape[0], -1)
        w64 = O.render_weight_from_alpha(al.double().cpu())
        return _ratio(out, w64, RO.alpha_weights_forward_tol(w64), what), 0
    if name == "density_to_weights":
        d_, r_ = a[0].cpu(), a[1].cpu()
        w64 = O.weights_from_density(d_.double(), r_.double())
        return _ratio(out, w64, RO.density_weights_forward_tol(d_, r_, w64), what), 0
    raise KeyError(name)


def check_recorded_step(dev, n_cam, n_lidar, seed=0, report=print):
    """Every recorded call judged by its comparator; every operator of the forward reached.  Returns {name: worst}."""
    cfg, params, be, calls = record_training_step(dev, n_cam, n_lidar, seed)
    worst, faces = {}, 0
    for name, a, k, out in calls:
        w, f = check_recorded_call(name, a, k, out, be, cfg, params, dev)
        worst[name] = max(worst.get(name, 0.0), w)
        faces += f
    missing = set(RECORDED) - set(worst)
    assert not missing, f"the training step never called {sorted(missing)}"
    return worst, faces, len(calls)
