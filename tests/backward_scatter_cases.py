"""Bodies of the entry-by-entry tests of the hash-grid backward operators (the table scatters of neurad_encoding_bwd in
features and density mode, neurad_encoding_pose_bwd, hashgrid_bwd), shared by tests/test_zz_backward_scatter_gpu.py
(dev = "cuda": the real library, production table sizes) and tests/test_backward_scatter_cpu.py (dev = "cpu": the same
device code through tests/fake_backend.py and the host emulation, small tables).

Reference: the oracle's own forward with the hash tables (and the density decoder) promoted to float64 leaves.  Positions,
cells, interpolation and anti-aliasing weights stay fp32, exactly as the kernel computes them, so every term of a row's sum
is the kernel's term and autograd adds the terms in float64.  Each table row e is then checked against its own bound:

  * n_e = number of (sample, level, corner) terms that land on row e (recorded from the oracle's hash_indices);
  * absum_e = the same backward with |cotangent| (all interpolation weights are >= 0);
  * accumulators start from a non-zero prefill P: rows with n_e == 0 must still hold P bit for bit (no stray or misdirected
    reductions), every other row |got - P - ref| <= (n_e + TERM_ULPS) * 2^-24 * (absum_e + |P|) -- the worst case of n_e
    fp32 additions onto P in any order, plus the rounding of each term (see TERM_ULPS).  Nothing is scaled to the largest
    entry: a row that lost or doubled one sample's contribution fails however small it is."""
import torch

import neurad_studio_b200 as nsb
from neurad_studio_b200 import scene
from neurad_studio_b200.lib import FIELD_MAIN, FIELD_PROP1
from oracle import neurad_oracle as O
from oracle.convert import to_oracle_cfg

U = 2.0 ** -24
# Relative difference between the kernel's and the reference's value of ONE term, in units of U (one rounding <= 1 U,
# one ulp <= 2 U), counted from the code (nff_device.h, nff_modules.h) rather than measured.  Cells, offsets and corner
# factors are the same fp32 values on both sides; what differs:
#   level weight 1 / max(2 res std, 1): the kernel contracts the std with a reciprocal multiply (2 U vs the reference's
#     division, 1 U) and, outside the unit ball, cbrtf (<= 1 ulp) x reciprocal (4 U), squared (9 U), times std (12 U in
#     all) where the reference takes powf(x, 0.33333334f) (<= 1 ulp, plus <= 1.2 U for the rounded exponent at
#     2 |x| - 1 < 2^10), divides and squares (11.4 U): <= 23.4 U; then 2 res std (1 U each side) and the reciprocal
#     (rcp.approx <= 2 U on the GPU, 1 U in the reference): <= 28.4 U;
#   products: the kernel rounds d * w, the three corner factors' two products and the corner value (4 U), in density mode
#     also ddensity * density and the decoder weight (6 U); the reference multiplies them in float64 (< 0.01 U);
#   decoder terms (density mode) carry the kernel's trilinear blend (<= 6 U of the sum of |corner terms|) and one more
#     product: <= 37 U, next to n = the number of samples.
# Total <= 35 U for a table term, so 40 is a worst-case allowance, not a measured one (on the host emulation, whose
# reciprocal is exact, single-term rows reach ~11 U).
TERM_ULPS = 40
PREFILL = 1.0 / 1024  # exactly representable; small next to most rows' sums, so a lost term is far outside the bound
DENS_LO, DENS_HI = 3.0590232e-07, 3269017.372  # exp(-15), exp(15) in fp32: the trunc_exp backward's clamp


# ------------------------------------------------------------------------------------------------ comparator
def check_scatter(got, ref, absum, n, prefill=PREFILL, what=""):
    """got: accumulator after the operator ([R, F] or [R]); ref / absum: float64, same shape; n: int64 [R] terms per row.
    Returns the largest |got - P - ref| / tol over the touched entries."""
    got = got.detach().cpu().reshape(ref.shape)
    n = n.reshape(n.shape[0], *([1] * (ref.dim() - 1))).expand(ref.shape)
    untouched = n == 0
    pbits = torch.tensor([prefill], dtype=torch.float32).view(torch.int32).item()
    stray = untouched & (got.view(torch.int32) != pbits)
    assert not stray.any(), f"{what}: {int(stray.sum())} entries no sample reaches changed, e.g. {stray.nonzero()[:4].tolist()}"
    t = ~untouched
    if not t.any():
        return 0.0
    err = (got[t].double() - prefill - ref[t]).abs()
    tol = (n[t] + TERM_ULPS).double() * U * (absum[t] + abs(prefill))
    r = err / tol
    worst = int(r.argmax())
    assert r[worst].item() <= 1.0, (f"{what}: |got - P - ref| / tol = {r[worst].item():.3g} at a row with n = {int(n[t][worst])}: "
                                    f"got - P = {got[t][worst].item() - prefill:.9g}, ref = {ref[t][worst].item():.9g}")
    return r[worst].item()


class RowLog:
    """Records, per hash table, the rows every O.hash_encode call reads (one entry per sample, level and corner)."""

    def __enter__(self):
        self.calls, self._orig = [], O.hash_encode

        def wrapped(x, table, scalings, table_size):
            idx, _ = O.hash_indices(x, scalings, table_size)
            self.calls.append((table, idx))
            return self._orig(x, table, scalings, table_size)

        O.hash_encode = wrapped
        return self

    def __exit__(self, *exc):
        O.hash_encode = self._orig

    def counts(self, table):
        n = torch.zeros(table.shape[0], dtype=torch.int64)
        for t, idx in self.calls:
            if t is table:
                n += torch.bincount(idx.reshape(-1), minlength=table.shape[0])
        return n


# ------------------------------------------------------------------------------------------------ scenes and inputs
def make_cfg(dev, n_actors):
    """Production grids on the GPU (main 2^22 / actors 2^17, proposal 2^20 / 2^15); small tables on the CPU."""
    return nsb.NeuRADConfig(n_actors=n_actors) if dev == "cuda" else nsb.small_config(n_actors=n_actors, log2_main=12, log2_prop=11)


def make_scene(cfg, seed=0, axis_aligned=True):
    """Parameters and trajectories.  The table checks use axis-aligned boxes: with a jittered yaw the kernel and the oracle
    round the world -> box transform in different orders, a sample's box-frame position moves by a few ulps of its world
    coordinates (up to ~300 m), and the fine actor levels' corner weights with it -- far outside a per-entry bound.  That
    parity is covered by the forward and whole-tensor gradient tests; here every term must be the kernel's term."""
    trajs = scene.make_trajectories(cfg.n_actors, cfg.duration, seed=seed, axis_aligned=axis_aligned) if cfg.n_actors else None
    return scene.make_params(cfg, seed=seed, trajectories=trajs), trajs


def backend(dev, cfg, params):
    if dev == "cpu":
        from tests.fake_backend import FakeBackend

        be = FakeBackend()
    else:
        from neurad_studio_b200.backend import B200Backend

        be = B200Backend(torch.device(dev, 0))
    be.load_params(cfg, params)
    return be


CLUSTER_OFFSETS = torch.tensor([[0.0, 0.0, 0.0], [35.0, 14.0, 0.0], [-30.0, -16.0, 0.0], [70.0, -12.0, 2.0], [-65.0, 18.0, -1.0],
                                [18.0, -45.0, 3.0], [-20.0, 50.0, 0.0], [52.0, 40.0, 1.0]])


def make_rays(n, S, seed, trajs=None, layout="spread", times=None, duration=8.0):
    """Gaussians of n rays x S samples (fp32, the kernel's and the reference's common input).  Even rays are aimed at an
    actor box at the ray's time.  layout: "spread" (samples along 250 m, quadratic spacing), "steps" (5 cm apart: consecutive
    samples share the coarse cells, so the run-length aggregation engages), "clusters" (the 8 rays of a warp start in 8
    separated places, 12 m+ apart: more distinct pending coarse cells per warp than the kernel's merge rounds)."""
    gen = torch.Generator().manual_seed(seed)

    def r(*shape):
        return torch.rand(*shape, generator=gen)

    o = torch.stack([r(n) * 10.0 - 5.0, r(n) * 4.0 - 2.0, 1.2 + r(n)], -1)
    if layout == "clusters":
        o = o + CLUSTER_OFFSETS[torch.arange(n) % 8]
    yaw, pitch = (r(n) - 0.5) * 1.2, (r(n) - 0.6) * 0.25
    d = torch.stack([torch.cos(yaw) * torch.cos(pitch), torch.sin(yaw) * torch.cos(pitch), torch.sin(pitch)], -1)
    t = r(n) * duration if times is None else times.float().clone()
    if trajs:
        jitter = (r(n, 3) - 0.5) * torch.tensor([3.0, 1.5, 1.2])
        for i in range(0, n, 2):
            tr = trajs[(i // 2 * 7) % len(trajs)]
            k = int(torch.argmin((tr["timestamps"] - t[i].clamp(0, duration)).abs()))
            v = tr["poses"][k, :3, 3] + jitter[i] - o[i]
            d[i] = v / v.norm()
    area = 1.0e-6 * (0.5 + r(n))
    if layout == "spread":
        u = torch.sort(r(n, S + 1), dim=1).values
        edges = 0.5 + u * u * 250.0
    elif layout == "steps":
        edges = 2.0 + r(n, 1) * 40.0 + 0.05 * torch.arange(S + 1).float()[None, :]
    else:
        edges = 0.5 + r(n, 1) * 0.5 + 0.1 * torch.arange(S + 1).float()[None, :]
    mean, std = O.fast_isotropic_gaussian(o[:, None, :], d[:, None, :], area[:, None, None], edges[:, :-1, None], edges[:, 1:, None])
    return mean.contiguous(), std.contiguous(), t  # [n,S,1,3], [n,S,1,1], [n]


def field_keys(prefix, n_actors):
    return [f"{prefix}.hashgrid.static_grid.hash_table"] + [f"{prefix}.hashgrid.actor_grids.{a}.hash_table" for a in range(n_actors)]


# ------------------------------------------------------------------------------------------------ references
def _oracle_features(params, cfg, prefix, mean, std, times, flip, leaves):
    """The oracle's NeuRADHashEncoding.forward with `leaves` (float64 tables) substituted; returns (features, RowLog)."""
    ocfg = to_oracle_cfg(cfg)
    fcfg = ocfg.main if prefix == "field" else ocfg.prop[1]
    q = dict(params)
    q.update(leaves)
    n, s = mean.shape[0], mean.shape[1]
    with RowLog() as log:
        feats, _ = O.hashgrid_forward(q, prefix, fcfg, ocfg, mean, std, times.reshape(n, 1, 1).expand(n, s, 1), None, flip=flip,
                                      require_actor_grad=False)
    return feats, log


def features_reference(params, cfg, mean, std, times, G, flip=None):
    """Main field, features mode: {key: (ref, absum, n)} for the static and every actor table."""
    keys = field_keys("field", cfg.n_actors)
    leaves = {k: params[k].double().requires_grad_(True) for k in keys}
    feats, log = _oracle_features(params, cfg, "field", mean, std, times, flip, leaves)
    lv = [leaves[k] for k in keys]
    g = torch.autograd.grad((feats * G.double()).sum(), lv, retain_graph=True, allow_unused=True)
    ga = torch.autograd.grad((feats * G.abs().double()).sum(), lv, allow_unused=True)
    out = {}
    for k, a, b in zip(keys, g, ga):
        z = torch.zeros_like(leaves[k])
        out[k] = (z if a is None else a, z if b is None else b, log.counts(leaves[k]))
    return out


def density_reference(params, cfg, mean, std, times, density, ddensity, flip=None):
    """Proposal field 1, density mode: tables get g * decoder_k * d feature_k, the decoder g * feature_k, with
    g = ddensity * clamp(density) (trunc_exp backward).  Returns ({key: (ref, absum, n)}, decoder (ref, absum, n))."""
    pre = "proposal_fields.1"
    keys = field_keys(pre, cfg.n_actors)
    dkey = f"{pre}.density_decoder.weight"
    leaves = {k: params[k].double().requires_grad_(True) for k in keys}
    dec = params[dkey].double().requires_grad_(True)  # [1, L]
    feats, log = _oracle_features(params, cfg, pre, mean, std, times, flip, leaves)
    # the trunc_exp backward restated on the stored density, as the kernel takes it; that this clamp is the reference's
    # (g * exp(clamp(x, -15, 15)), field_components/activations.py:38-41) is checked against the oracle's own
    # O.proposal_density autograd by module_seam_cases.proposal_density_backward_clamps_like_trunc_exp and by
    # test_module_bwd_emul.py::test_encoding_backward_density_mode_clamps_like_trunc_exp
    g = (ddensity.reshape(-1, 1) * density.reshape(-1, 1).clamp(DENS_LO, DENS_HI)).double()
    lv = [leaves[k] for k in keys]
    gr = torch.autograd.grad(((feats @ dec.t()) * g).sum(), lv + [dec], retain_graph=True, allow_unused=True)
    ga = torch.autograd.grad(((feats @ dec.detach().abs().t()) * g.abs()).sum(), lv, allow_unused=True)
    with torch.no_grad():  # |feature_k| bound: the interpolation of |table| (weights >= 0)
        abs_leaves = {k: params[k].double().abs() for k in keys}
        feats_abs, _ = _oracle_features(params, cfg, pre, mean, std, times, flip, abs_leaves)
        dec_abs = (feats_abs * g.abs()).sum(0)
    out = {}
    for k, a, b in zip(keys, gr[:-1], ga):
        z = torch.zeros_like(leaves[k])
        out[k] = (z if a is None else a, z if b is None else b, log.counts(leaves[k]))
    n_dec = torch.full((dec.shape[1],), mean.shape[0] * mean.shape[1], dtype=torch.int64)
    return out, (gr[-1].reshape(-1), dec_abs, n_dec)


# ------------------------------------------------------------------------------------------------ operator runs
def _accumulators(params, keys, dev, none_actors=()):
    static = torch.full(params[keys[0]].shape, PREFILL, device=dev)
    actors = [None if a in none_actors else torch.full(params[k].shape, PREFILL, device=dev) for a, k in enumerate(keys[1:])]
    return {"static": static, "actors": actors}


def _gauss_dev(mean, std, times, dev):
    n, s = mean.shape[0], mean.shape[1]
    return mean.reshape(n, s, 3).to(dev), std.reshape(n, s).to(dev), times.to(dev)


def run_features(be, params, cfg, dev, mean, std, times, G, flip=None, none_actors=()):
    keys = field_keys("field", cfg.n_actors)
    grads = _accumulators(params, keys, dev, none_actors)
    m, s, t = _gauss_dev(mean, std, times, dev)
    be.neurad_encoding_bwd(FIELD_MAIN, m, s, t, grads, dfeatures=G.to(dev), flip=None if flip is None else flip.to(dev))
    return grads


def run_density(be, params, cfg, dev, mean, std, times, density, ddensity, want_decoder=True, flip=None):
    keys = field_keys("proposal_fields.1", cfg.n_actors)
    grads = _accumulators(params, keys, dev)
    if want_decoder:
        grads["decoder"] = torch.full((params["proposal_fields.1.density_decoder.weight"].numel(),), PREFILL, device=dev)
    m, s, t = _gauss_dev(mean, std, times, dev)
    be.neurad_encoding_bwd(FIELD_PROP1, m, s, t, grads, density=density.to(dev), ddensity=ddensity.to(dev),
                           flip=None if flip is None else flip.to(dev))
    return grads


def check_tables(grads, ref, keys, what):
    """Every table the operator was given against its per-entry reference; returns the worst ratio."""
    worst = check_scatter(grads["static"], *ref[keys[0]], what=f"{what} static")
    touched = ref[keys[0]][2].sum().item()
    for a, k in enumerate(keys[1:]):
        if grads["actors"][a] is not None:
            worst = max(worst, check_scatter(grads["actors"][a], *ref[k], what=f"{what} actor {a}"))
        touched += ref[k][2].sum().item()
    assert touched > 0
    return worst


def flip_of(n, seed):
    return torch.where(torch.rand(n, generator=torch.Generator().manual_seed(seed)) < 0.5, -1.0, 1.0)


# ------------------------------------------------------------------------------------------------ cases
def features_mode_matches_float64_reference(dev, n, S, n_actors, flip, layout="spread", log2_main=None, none_actors=()):
    """neurad_encoding_bwd, features mode (main field: 8 levels x 4 features): every entry of the static and the actor
    tables.  Returns the worst |got - P - ref| / tol."""
    cfg = make_cfg(dev, n_actors)
    if log2_main is not None:
        cfg.grid.static.log2_hashmap_size = log2_main
    params, trajs = make_scene(cfg, seed=n_actors + S)
    mean, std, times = make_rays(n, S, seed=100 * n + S, trajs=trajs, layout=layout, duration=cfg.duration)
    fl = flip_of(n, S) if flip else None
    D = cfg.grid.static.out_dim
    G = torch.randn(n * S, D, generator=torch.Generator().manual_seed(n + 7 * S))
    if layout == "clusters":  # the 8 rays of each warp end their walk in >= 6 different level-0 cells
        c, _ = O.scaled_contraction(mean[:, -1, 0], std[:, -1, 0], params["static_scale"])
        cells = torch.floor(c * cfg.grid.static.scalings()[0]).long()
        for w0 in range(0, n - 7, 8):
            assert len({tuple(x) for x in cells[w0:w0 + 8].tolist()}) >= 6
    be = backend(dev, cfg, params)
    grads = run_features(be, params, cfg, dev, mean, std, times, G, fl, none_actors)
    be.check_status()
    ref = features_reference(params, cfg, mean, std, times, G, fl)
    keys = field_keys("field", n_actors)
    if n_actors and n > 1 and layout != "clusters":  # the actor branch was exercised (cluster rays stay near their origins)
        assert sum(ref[k][2].sum().item() for k in keys[1:]) > 0
    return check_tables(grads, ref, keys, f"features n={n} S={S} actors={n_actors}")


def density_mode_matches_float64_reference(dev, n, S, n_actors, want_decoder, flip=False):
    """neurad_encoding_bwd, density mode (proposal field: 6 levels x 1 feature, the x-adjacent pair reductions): every table
    entry and, with grads["decoder"], every decoder weight.  Densities span exp(+-20) so the trunc_exp clamp engages."""
    cfg = make_cfg(dev, n_actors)
    params, trajs = make_scene(cfg, seed=3 + n_actors)
    mean, std, times = make_rays(n, S, seed=7 * n + S, trajs=trajs, duration=cfg.duration)
    gen = torch.Generator().manual_seed(S)
    density = torch.exp(torch.randn(n, S, generator=gen) * 8.0)
    ddensity = torch.randn(n, S, generator=gen)
    fl = flip_of(n, S + 1) if flip else None
    be = backend(dev, cfg, params)
    grads = run_density(be, params, cfg, dev, mean, std, times, density, ddensity, want_decoder, fl)
    be.check_status()
    ref, dec = density_reference(params, cfg, mean, std, times, density, ddensity, fl)
    keys = field_keys("proposal_fields.1", n_actors)
    worst = check_tables(grads, ref, keys, f"density n={n} S={S} actors={n_actors}")
    if want_decoder:
        worst = max(worst, check_scatter(grads["decoder"], *dec, what="decoder"))
    return worst


def hashgrid_bwd_matches_float64_reference(dev, L, F, log2T, n_points):
    """The stand-alone HashEncoding backward (no anti-aliasing weights), lattice points (ceil == floor, 0 and 1) included."""
    g = nsb.HashGridSettings(F, L, 16, 2048, log2T)
    gen = torch.Generator().manual_seed(L * 100 + F)
    x = torch.rand(n_points, 3, generator=gen)
    x[:64] = torch.randint(0, 17, (64, 3), generator=gen).float() / 16.0
    dout = torch.randn(n_points, L * F, generator=gen)
    rows = g.hash_table_size * L
    leaf = torch.zeros(rows, F, dtype=torch.float64, requires_grad=True)  # the gradient does not depend on the values
    with RowLog() as log:
        y = O.hash_encode(x, leaf, g.scalings(), g.hash_table_size)
    ref, = torch.autograd.grad((y * dout.double()).sum(), leaf, retain_graph=True)
    absum, = torch.autograd.grad((y * dout.abs().double()).sum(), leaf)
    be = backend(dev, nsb.small_config(), scene.make_params(nsb.small_config()))
    got = torch.full((rows, F), PREFILL, device=dev)
    be.hashgrid_bwd(g, x.to(dev), dout.to(dev), got)
    return check_scatter(got, ref, absum, log.counts(leaf), what=f"hashgrid L={L} F={F} log2T={log2T}")


def pose_bwd_matches_oracle_per_actor_and_keyframe(dev, n_actors, flip):
    """neurad_encoding_pose_bwd against the oracle's fp32 autograd (float64 trajectories would move samples across cells),
    per (keyframe, actor) slice instead of over the whole tensor: a slice that lost its samples fails however small it is.
    Query times on keyframes, before the first, after the last and in between."""
    cfg = make_cfg(dev, n_actors)
    params, trajs = make_scene(cfg, seed=11, axis_aligned=False)
    n, S = 256, 32
    ts = params["dynamic_actors.unique_timestamps"]
    gen = torch.Generator().manual_seed(5)
    pick = torch.randint(0, ts.shape[0], (n,), generator=gen)
    times = torch.where(torch.arange(n) % 4 == 0, ts[pick], torch.rand(n, generator=gen) * cfg.duration)
    times[1::16], times[3::16] = -0.5, cfg.duration + 0.5
    mean, std, times = make_rays(n, S, seed=21, trajs=trajs, layout="spread", times=times, duration=cfg.duration)
    fl = flip_of(n, 3) if flip else None
    G = torch.randn(n * S, cfg.grid.static.out_dim, generator=gen)
    p = dict(params)
    for k in ("dynamic_actors.actor_positions", "dynamic_actors.actor_rotations_6d"):
        p[k] = params[k].clone().requires_grad_(True)
    ocfg = to_oracle_cfg(cfg)
    trace = {}
    feats, _ = O.hashgrid_forward(p, "field", ocfg.main, ocfg, mean, std, times.reshape(n, 1, 1).expand(n, S, 1), None, trace, flip=fl)
    (feats * G).sum().backward()
    hit = set(trace["actor_id"].unique().tolist()) - {-1}  # actors some sample lies in
    assert len(hit) >= n_actors // 2
    want = {"pos": p["dynamic_actors.actor_positions"].grad, "rot": p["dynamic_actors.actor_rotations_6d"].grad}
    be = backend(dev, cfg, params)
    got = {k: torch.full(v.shape, PREFILL, device=dev) for k, v in want.items()}
    m, s, t = _gauss_dev(mean, std, times, dev)
    be.neurad_encoding_pose_bwd(FIELD_MAIN, m, s, t, G.to(dev), params["dynamic_actors.actor_rotations_6d"].to(dev),
                                params["dynamic_actors.actor_positions"].to(dev), got["rot"], got["pos"],
                                flip=None if fl is None else fl.to(dev))
    be.check_status()
    # A query exactly on keyframe k brackets it as (k-1, k) with frac = 0.1 / (0.1 + 1e-6): keyframe k-1 receives the share
    # 1 - frac ~ 1e-5, which fp32 forms by cancellation (~1e-2 relative, in the reference as in the kernel).  A slice that
    # only such shares reach (or a rotation slice of few samples, whose Gram-Schmidt chain cancels similarly) is held to
    # 10 % of its actor's largest entry instead of its own maximum.  The bound is 1e-3 per slice (the whole-tensor checks
    # hold 2e-4 of the global maximum: the same fp32 noise of the world -> box transform, measured here against smaller
    # scales; up to 6e-4 with actors 300 m from the origin).
    worst = 0.0
    for k in ("pos", "rot"):
        checked = set()
        w, gk = want[k], got[k].cpu() - PREFILL
        for a in range(w.shape[1]):
            floor = 0.1 * w[:, a].abs().max().item()
            for ti in range(w.shape[0]):
                scale = max(w[ti, a].abs().max().item(), floor)
                if scale == 0:
                    assert (gk[ti, a] == 0).all(), (k, ti, a)
                    continue
                e = (gk[ti, a] - w[ti, a]).abs().max().item() / scale
                assert e < 1e-3, (k, ti, a, e)
                worst = max(worst, e)
                checked.add(a)
        assert hit <= checked, (k, sorted(hit - checked))  # every actor a sample lies in was compared
    return worst


def empty_and_zero_cotangent_leave_accumulators_bit_identical(dev, n_actors):
    """n_rays == 0 and an all-zero cotangent: no accumulator changes, in either mode."""
    cfg = make_cfg(dev, n_actors)
    params, trajs = make_scene(cfg, seed=2)
    n, S = 40, 5
    mean, std, times = make_rays(n, S, seed=9, trajs=trajs, duration=cfg.duration)
    be = backend(dev, cfg, params)
    D = cfg.grid.static.out_dim
    for m_, s_, t_, G in ((mean[:0], std[:0], times[:0], torch.zeros(0, D)), (mean, std, times, torch.zeros(n * S, D))):
        grads = run_features(be, params, cfg, dev, m_, s_, t_, G)
        for acc in [grads["static"]] + grads["actors"]:
            assert (acc == PREFILL).all() and not torch.signbit(acc).any()
        dn = torch.exp(torch.randn(m_.shape[0], S))
        grads = run_density(be, params, cfg, dev, m_, s_, t_, dn, torch.zeros_like(dn))
        for acc in [grads["static"], grads["decoder"]] + grads["actors"]:
            assert (acc == PREFILL).all() and not torch.signbit(acc).any()
    if dev != "cpu":  # an empty batch still has its mode checked
        import pytest

        g0 = _accumulators(params, field_keys("field", n_actors), dev)
        m0, s0, t0 = _gauss_dev(mean[:0], std[:0], times[:0], dev)
        with pytest.raises(ValueError):
            be.neurad_encoding_bwd(FIELD_MAIN, m0, s0, t0, g0)
        with pytest.raises(ValueError):
            be.neurad_encoding_bwd(FIELD_MAIN, m0, s0, t0, dict(g0, decoder=torch.zeros(8, device=dev)), dfeatures=torch.zeros(0, D, device=dev))
    be.check_status()


def comparator_rejects_a_lost_or_doubled_sample(dev):
    """The per-entry check must fail when the reference drops or doubles ONE sample's cotangent, chosen so that it reaches
    a row that receives at most two terms."""
    cfg = make_cfg(dev, 0)
    params, _ = make_scene(cfg, seed=4)
    n, S = 33, 5
    mean, std, times = make_rays(n, S, seed=4, duration=cfg.duration)
    G = torch.randn(n * S, cfg.grid.static.out_dim, generator=torch.Generator().manual_seed(4))
    be = backend(dev, cfg, params)
    grads = run_features(be, params, cfg, dev, mean, std, times, G)
    key = field_keys("field", 0)[0]
    ref = features_reference(params, cfg, mean, std, times, G)
    assert check_scatter(grads["static"], *ref[key]) <= 1.0
    # a sample with the largest level-0-free contribution on a row with n_e <= 2
    leaf = params[key].double()
    with RowLog() as log:
        _oracle_features(params, cfg, "field", mean, std, times, None, {key: leaf})
    idx = log.calls[0][1].reshape(n * S, -1)  # [P, L*8]
    few = ref[key][2][idx] <= 2
    share = torch.where(few, ref[key][1].abs().amax(-1)[idx], torch.zeros(()))
    p = int(share.amax(-1).argmax())
    assert share[p].max() > 0
    for factor in (0.0, 2.0):
        G2 = G.clone()
        G2[p] *= factor
        bad = features_reference(params, cfg, mean, std, times, G2)
        try:
            check_scatter(grads["static"], *bad[key])
        except AssertionError:
            continue
        raise AssertionError(f"the comparator accepted a reference with sample {p}'s cotangent x {factor}")


def linear_wgrad_matches_float64(dev, K, N, relu, n_rows=2**20 + 17):
    """linear_wgrad (the CUDA-core default dW = dY^T act(X), db = sum dY) at a row count that is not a multiple of the
    32-row tile, accumulating onto a prefill.

    Random data against a float64 matmul, per entry: |got - P - ref| <= (n_rows + 1 + 2) * U * (|dY|^T |act(X)| + |P|)
    (one rounding per product, at most n_rows additions in any order); at a million rows that bound is loose.  So a second
    run uses dyadic data (X in {-2..2} / 8, dY in {-3..3} / 16): every product and every partial sum is an exact fp32
    number (|sum| < 2^24 units of 2^-7), whatever the order of summation, and the result must equal float64 EXACTLY -- a
    lost, repeated or misplaced row, tile or tail fails by at least one unit."""
    from neurad_studio_b200.backend import B200Backend

    be = B200Backend(torch.device(dev, 0))
    gen = torch.Generator().manual_seed(K * 100 + N + relu)
    P = 0.375  # a multiple of 2^-7: keeps the exact run exact
    worst = 0.0
    for exact in (False, True):
        if exact:
            x = torch.randint(-2, 3, (n_rows, K), generator=gen).float() / 8
            dy = torch.randint(-3, 4, (n_rows, N), generator=gen).float() / 16
        else:
            x, dy = torch.randn(n_rows, K, generator=gen), torch.randn(n_rows, N, generator=gen)
        dW = torch.full((N, K), P, device=dev)
        db = torch.full((N,), P, device=dev)
        be.linear_wgrad(x.to(dev), dy.to(dev), relu, dW, db, impl="cuda")
        torch.cuda.synchronize(dev)
        xa = (torch.relu(x) if relu else x).double()
        ref_w, ref_b = dy.double().t() @ xa, dy.double().sum(0)
        if exact:
            assert torch.equal(dW.cpu().double() - P, ref_w), (dW.cpu().double() - P - ref_w).abs().max().item()
            assert torch.equal(db.cpu().double() - P, ref_b)
            continue
        abs_w, abs_b = dy.double().abs().t() @ xa.abs(), dy.double().abs().sum(0)
        for got, ref, ab in ((dW, ref_w, abs_w), (db, ref_b, abs_b)):
            err = (got.cpu().double() - P - ref).abs()
            tol = (n_rows + 3) * U * (ab + P)
            worst = max(worst, (err / tol).max().item())
    assert worst <= 1.0, worst
    be.close()
    return worst
