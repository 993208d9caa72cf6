"""Bodies of the sample-by-sample tests of the ray-per-lane render kernels (nff_sample_lane_kernel + nff_shade_lane_kernel,
mode "split", and nff_render_lane_kernel, mode "lane"), shared by tests/test_zz_render_trace_gpu.py (dev = "cuda": the
real library, production table sizes) and tests/test_render_trace_cpu.py (dev = "cpu": the same device code through the
host emulation, tests/host_emul/emul.py render(..., lane_mode=True), small tables).

Every stage is recomputed from the kernel's OWN traced inputs to that stage (render(..., want_trace=...)), so errors
do not chain from stage to stage and no sample is compared against a sample placed elsewhere:
  1. proposal weights (prop_weights_0 / _1): float64 proposal density at the round's edges (round 0: linspace01 through
     to_euclid, restated in fp32; round 1: the traced bins_e_1), both rounds on proposal_fields.1, static samples on
     the static grid and actor samples on the actor's grid at the kernel's fp32 box position, then the weights with the
     cumulative sum in float64.  Grid cells and interpolation offsets come from the fp32 contracted positions (the
     kernel keeps the reference's IEEE op sequence for positions, so an fp32 torch pass on the CPU reproduces them);
  2. the resampling merge walk (inds, bins_s, bins_e of both rounds): bit for bit against an fp32 restatement of
     lane_proposal_round's walk on the traced weights;
  3. the main field (sdf, field_feature) in float64 at the traced bins_e_2 with the last edge moved to the sky as the
     kernel does, the traced actor assignment (actor samples: 16 grid features padded to 32, the direction rotated into
     the box frame), and a per-entry bound carried through every MLP layer as gamma (|W| |a| + |b|) + |W| E_a: the
     3xTF32 wgmma constant on the GPU (gamma_tc), the FFMA one in the emulation (gamma_ffma);
  4. alpha from the traced sdf (bounded), weights from the traced alpha incl. the sky top-up (bit for bit);
  5. outputs: depth / accumulation / prop_depth_0 / _1 and the 16 appearance columns bit for bit (sequences of single
     IEEE roundings and double products the restatement repeats); features[:, :32] from the traced weights and field
     features, intensity / ray_drop_logits through the lidar decoder in float64 (GPU): per-entry bounds;
  6. actor ids of all three stages against a float64 box test; a sample within a few ulp of a box face may differ
     and is counted.
Bounds are derived per entry from the kernel's code (standard model: one fp32 rounding <= U = 2^-24 of its result,
expf <= 2 ulp <= 4 U, a sum of n terms in any order <= n U of the sum of |terms|), first order in U, condition factors
explicit; nothing is scaled to a tensor's maximum.  Every output row passes through the 8-ray staging store of the
shading kernel, so a misplaced segment or a neighbouring ray's row fails here."""
import time

import numpy as np
import torch

import neurad_studio_b200 as nsb
from neurad_studio_b200 import scene
from neurad_studio_b200.lib import TRACE_FIELDS
from oracle import neurad_oracle as O

U = 2.0 ** -24
TINY = 2.0 ** -149
F32_EXP_MAX = float(np.log(np.finfo(np.float32).max))
# gaussian std through sample_gaussian and contract (NFF_PARITY_STD 0): cbrtf twice (<= 3e-7 relative each; the second,
# cbrt(2 mag - 1), enters squared: 6e-7), and <= 16 single roundings (md, t, t t, area t t, cs md, std / scale by a
# reciprocal multiply (2), 2 mag - 1 (a third of it through the cbrt), 1 / mag (2), q q, sd q q, plus the 4 U relative
# difference of the fp32 mag from the float64 one)
STD_REL = 9e-7 + 16 * U
EXIT_ARG = 106.0  # expf(-x) is 0 in fp32 for x > ~103.97 (below half the smallest denormal); 106 leaves a margin
PARTIAL = tuple(k for k in TRACE_FIELDS if not k.startswith("actor_id"))  # the early exit stays on


# ====================================================================================== renderers and scenes
class EmulRenderer:
    """render() of the host emulation of the ray-per-lane kernel (MlpLaneFfma: CUDA-core fp32 MLP).  The emulation
    always records the full trace and has no lidar head: a partial trace only filters the returned fields, so the
    partial-trace comparisons are meaningful on the GPU only."""

    def __init__(self, cfg, params):
        self.cfg, self.params = cfg, params

    def render(self, rays, want_trace=True, image_width=0, mode=None, want_intensity=False):
        from tests.host_emul import emul

        out = emul.render(self.cfg, self.params, {k: v.cpu() for k, v in rays.items()}, O.pdf_u, lane_mode=True)
        keep = set(TRACE_FIELDS) if want_trace is True else set(want_trace or ())
        return {k: v for k, v in out.items() if k not in TRACE_FIELDS or k in keep}


class GpuRenderer:
    def __init__(self, cfg, params):
        from neurad_studio_b200.backend import B200Backend

        self.cfg, self.params = cfg, params
        self.be = B200Backend(torch.device("cuda", 0))
        self.be.load_params(cfg, params)

    def render(self, rays, want_trace=True, image_width=0, mode="split", want_intensity=False):
        from neurad_studio_b200.backend import DEFAULT_MODE

        self.be.set_mlp_mode(mode)
        try:
            out = self.be.render(rays, want_trace=want_trace, image_width=image_width, want_intensity=want_intensity)
            self.be.check_status()
        finally:
            self.be.set_mlp_mode(DEFAULT_MODE)
        torch.cuda.synchronize()
        return out


def renderer(dev, cfg, params):
    return EmulRenderer(cfg, params) if dev == "cpu" else GpuRenderer(cfg, params)


def _with_near_far(rays, seed):
    """nears / fars on every ray: most at the defaults (0 and 1e6, as without them), a third with fars below the sky
    distance and nears > 0."""
    n = rays["origins"].shape[0]
    gen = torch.Generator().manual_seed(seed)
    nears = torch.zeros(n, 1)
    fars = torch.full((n, 1), 1.0e6)
    sel = torch.rand(n, generator=gen) < 1 / 3
    k = int(sel.sum())
    nears[sel] = torch.rand(k, 1, generator=gen) * 2.0
    fars[sel] = 20.0 + torch.rand(k, 1, generator=gen) * 300.0
    out = dict(rays)
    out["nears"], out["fars"] = nears, fars
    return out


def _cat(*bundles):
    keys = bundles[0].keys()
    return {k: torch.cat([b[k].cpu() for b in bundles]) for k in keys}


def scene_rays(dev, name):
    """(cfg, params, rays, image_width) of one test scene.

    config2: NeuRADConfig(n_actors=0), default tables on the GPU; one PandaSet camera at render stride 3 (640 x 360, the
      2-D tile walk has ragged 16-row tiles at the bottom) followed by a lidar sweep (is_lidar: area scale 1), with
      nears / fars on every ray, some fars below the sky distance.
    config3: 16 actors, rays aimed at the boxes, a ray count that is not a multiple of 32, 128 or 512.
    opaque: a dense proposal field, so that the proposal transmittance underflows within a few samples in whole warps."""
    gpu = dev != "cpu"
    if name == "config2":
        cfg = nsb.NeuRADConfig(n_actors=0) if gpu else nsb.small_config()
        params = scene.make_params(cfg, seed=41, beta=3.0, sdf_bias=0.6)
        if gpu:
            from neurad_studio_b200.backend import B200Backend

            be = B200Backend(torch.device("cuda", 0))
            cam = be.raygen_pinhole(scene.pandaset_rig()[0], row0=1, row_step=3, col0=1, col_step=3)
            lid = be.raygen_lidar_points(scene.pandar64_scan())
            n_cam, n_lid, width = cam["origins"].shape[0], lid["origins"].shape[0] - 77, 640
            keys = ("origins", "directions", "pixel_area", "times")
            cam = {k: cam[k].cpu().reshape(n_cam, -1) for k in keys}
            lid = {k: lid[k].cpu().reshape(-1, cam[k].shape[1])[:n_lid] for k in keys}
            cam["is_lidar"], lid["is_lidar"] = torch.zeros(n_cam, 1, dtype=torch.bool), torch.ones(n_lid, 1, dtype=torch.bool)
            cam["sensor_idx"] = torch.zeros(n_cam, 1, dtype=torch.long)
            lid["sensor_idx"] = torch.full((n_lid, 1), cfg.num_sensors - 1, dtype=torch.long)
            rays = _cat(cam, lid)
        else:
            rays, width = scene.random_rays(333, cfg, seed=42), 0
        return cfg, params, _with_near_far(rays, 43), width
    if name == "config3":
        cfg = nsb.NeuRADConfig(n_actors=16) if gpu else nsb.small_config(n_actors=16)
        trajs = scene.make_trajectories(cfg.n_actors, cfg.duration, seed=21)
        params = scene.make_params(cfg, seed=21, beta=4.0, sdf_bias=0.5, trajectories=trajs)
        rays = scene.random_rays(8227 if gpu else 197, cfg, seed=22, trajectories=trajs)
        return cfg, params, rays, 0
    if name == "opaque":
        cfg = nsb.NeuRADConfig(n_actors=0) if gpu else nsb.small_config()
        params = scene.make_params(cfg, seed=51, beta=3.0, sdf_bias=0.6)
        key = "proposal_fields.1.hashgrid.static_grid.hash_table"
        params[key] = params[key].abs() * 0.5 + 0.5
        params["proposal_fields.1.density_decoder.weight"] = params["proposal_fields.1.density_decoder.weight"].abs() + 2.0
        rays = scene.random_rays(4160 if gpu else 160, cfg, seed=52, lidar_fraction=0.0)
        return cfg, params, rays, 0
    raise KeyError(name)


def pick_groups(n, n_random, seed, extra=()):
    """Whole 128-ray warp groups: the first, the last (ragged when n % 128 != 0), `extra` (e.g. groups with actor hits)
    and n_random others.  Returns the sorted ray indices."""
    n_groups = (n + 127) // 128
    g = {0, n_groups - 1} | {int(x) for x in extra}
    gen = torch.Generator().manual_seed(seed)
    g |= {int(x) for x in torch.randperm(n_groups, generator=gen)[:n_random]}
    idx = torch.cat([torch.arange(128 * k, min(128 * (k + 1), n)) for k in sorted(g)])
    return idx


# ====================================================================================== fp32 restatements (bit exact)
def _f(x):
    return torch.as_tensor(x, dtype=torch.float32)


class Spacing:
    """spacing_fn / spacing_fn_inv / to_euclid / linspace01 of nff_device.h, op by op in fp32 (single IEEE roundings)."""

    def __init__(self, cfg):
        sp = cfg.sampling
        self.lam = _f(sp.power_lambda)
        self.scaling = _f(sp.power_scaling)
        lam1 = abs(sp.power_lambda - 1.0)
        self.lam_1 = _f(lam1)
        self.ratio = _f(lam1 / sp.power_lambda)
        self.sky = _f(sp.sky_distance)
        assert sp.power_lambda == -1.0, "the restatement covers x ** -1 (a correctly rounded reciprocal) only"

    def fn(self, x):
        t = (x * self.scaling) / self.lam_1 + 1.0
        return self.ratio * (1.0 / t - 1.0)

    def inv(self, y):
        t = (y * self.lam) / self.lam_1 + 1.0
        t = torch.clamp_min(t, _f(1e-10))
        return ((1.0 / t - 1.0) * self.lam_1) / self.scaling

    def to_euclid(self, u, s_near, s_far):
        return self.inv(u * s_far + (1.0 - u) * s_near)

    @staticmethod
    def linspace01(n):
        step = _f(1.0) / _f(float(n))
        i = torch.arange(n + 1)
        lo = step * i.float()
        hi = 1.0 - step * (n - i).float()
        return torch.where(i < (n + 1) // 2, lo, hi)

    def near_far(self, rays, idx):
        n = idx.numel()
        fars = rays["fars"].reshape(-1)[idx].float() if "fars" in rays else torch.full((n,), 1.0e6)
        fars = torch.minimum(fars, self.sky)
        nears = rays["nears"].reshape(-1)[idx].float() if "nears" in rays else torch.zeros(n)
        return self.fn(nears)[:, None], self.fn(fars)[:, None]


def merge_walk(w, edges_s, u, hist_pad):
    """lane_proposal_round's resampling on the traced weights w [n, S] (fp32), the round's spacing edges [n, S+1] and
    the quantiles u [S_new+1]: (inds [n, S_new+1] int32, new spacing edges [n, S_new+1])."""
    n, S = w.shape
    wp = w + _f(hist_pad)
    tot = torch.cumsum(wp.double(), 1)[:, -1:].float()  # sequential double sum, rounded once
    padding = torch.clamp_min(_f(1e-5) - tot, 0.0)
    pad_each = padding / _f(float(S))
    tot = tot + padding
    pdf = (wp + pad_each) / tot
    run = torch.cumsum(pdf.double(), 1)  # double running sum, rounded per entry
    cdf = torch.cat([torch.zeros(n, 1), torch.clamp_max(run.float(), 1.0)], 1)
    uu = u.float().expand(n, -1).contiguous()
    k = torch.searchsorted(cdf, uu, side="right")  # the walk's k: number of cdf entries <= u
    c_km1 = cdf.gather(1, k - 1)
    above = k.clamp_max(S)
    c_k = torch.where(k > S, c_km1, cdf.gather(1, above))
    b0, b1 = edges_s.gather(1, k - 1), edges_s.gather(1, above)
    t = torch.nan_to_num((uu - c_km1) / (c_k - c_km1))
    t = torch.clamp(t, 0.0, 1.0)
    nb = b0 + t * (b1 - b0)
    return k.int(), nb


def appearance_bits(cfg, params, times, sensor):
    """The temporal appearance columns, op by op as the kernel evaluates them (fp32, single roundings)."""
    emb = params["appearance_embedding.weight"].float().cpu()
    eps_ = _f(float(cfg.embeds_per_sensor))
    tidx = (times.float() / _f(cfg.duration)) * eps_
    before = torch.clamp(torch.clamp_min(torch.floor(tidx), 0.0), max=eps_ - 1.0)
    after = torch.clamp(torch.clamp_min(before + 1.0, 0.0), max=eps_ - 1.0)
    ratio = tidx - before
    s = sensor.float()
    ib = (before + s * eps_).long()
    ia = (after + s * eps_).long()
    return emb[ib] * (1.0 - ratio)[:, None] + emb[ia] * ratio[:, None]


# ====================================================================================== the comparators
def _bits_equal(got, ref, what):
    got = got.detach().cpu().contiguous()
    ref = ref.detach().cpu().contiguous().reshape(got.shape)
    assert got.dtype == ref.dtype, (what, got.dtype, ref.dtype)
    if got.dtype == torch.float32:
        bad = got.view(torch.int32) != ref.view(torch.int32)
    else:
        bad = got != ref
    assert not bad.any(), f"{what}: {int(bad.sum())} entries differ, first at {bad.nonzero()[:3].tolist()}"


def _ratio(got, ref, tol, what):
    got = got.detach().cpu().double().reshape(ref.shape)
    ref, tol = ref.cpu(), tol.cpu()
    assert torch.isfinite(got).all(), f"{what}: non-finite result"
    err = (got - ref).abs()
    r = torch.where(err == 0, torch.zeros_like(err), err / tol)
    if r.numel() == 0:
        return 0.0
    w = int(r.reshape(-1).argmax())
    worst = r.reshape(-1)[w].item()
    assert worst <= 1.0, (f"{what}: |got - ref| / tol = {worst:.3g} at flat entry {w} of {tuple(ref.shape)}: got "
                          f"{got.reshape(-1)[w].item():.9g}, ref {ref.reshape(-1)[w].item():.9g}, tol {tol.reshape(-1)[w].item():.3g}")
    return worst


def check_walk(tr, rays, idx, cfg):
    """Stage 2, bit for bit: inds, bins_s, bins_e of both rounds from the traced weights."""
    sp = Spacing(cfg)
    s_near, s_far = sp.near_far(rays, idx)
    S0, S1 = cfg.sampling.num_proposal_samples
    S2 = cfg.sampling.num_nerf_samples
    n = idx.numel()
    e0 = Spacing.linspace01(S0).expand(n, -1)
    for rd, (w, edges, S_new) in enumerate(((tr["prop_weights_0"], e0, S1), (tr["prop_weights_1"], tr["bins_s_1"], S2))):
        k, nb = merge_walk(w.float(), edges.float(), O.pdf_u(S_new), cfg.sampling.histogram_padding)
        _bits_equal(tr[f"inds_{rd + 1}"], k, f"inds_{rd + 1}")
        _bits_equal(tr[f"bins_s_{rd + 1}"], nb, f"bins_s_{rd + 1}")
        _bits_equal(tr[f"bins_e_{rd + 1}"], sp.to_euclid(nb, s_near, s_far), f"bins_e_{rd + 1}")


def weights_bits(alpha):
    """Weights from the traced alpha as shade_ray_lane forms them: w = fl(alpha fl(T)), T a double product of the fp32
    fl(1 - alpha); the last (sky) sample gets the top-up fl(fl(w + 1) - acc), acc the sequential fp32 sum of the weights
    before it.  Returns (weights with the top-up, accumulation)."""
    a = alpha.float()
    one_m = (1.0 - a).double()
    T = torch.cumprod(torch.cat([torch.ones_like(one_m[:, :1]), one_m[:, :-1]], 1), 1)  # sequential double products
    w = a * T.float()
    acc = torch.zeros(a.shape[0])
    for s in range(a.shape[1]):
        acc = acc + w[:, s]
    w = w.clone()
    w[:, -1] = (w[:, -1] + 1.0) - acc
    return w, acc


def depth_bits(w, e):
    """Sequential fp32 fl(d + fl(w fl(fl(e0 + e1) 0.5))) over the samples (prop depths; the shading depth over all but
    the sky sample)."""
    mid = (e[:, :-1] + e[:, 1:]) * 0.5
    d = torch.zeros(w.shape[0])
    for s in range(w.shape[1]):
        d = d + w[:, s] * mid[:, s]
    return d


def alpha_reference(sdf, beta):
    """alpha = rcp(1 + expf(fl(sdf beta))): float64 from the traced sdf, with rel(alpha) <= (1 - alpha)(|x| + 5) U + 2 U
    (x = fl(sdf beta): U |x|; expf: 4 U; 1 + e and the correctly rounded reciprocal: U each).  Where expf overflows the
    kernel's alpha is 0, as the fp32 formula gives: the reference takes 0 there too."""
    x = sdf.double() * beta
    a = torch.where(x > F32_EXP_MAX, torch.zeros_like(x), torch.sigmoid(-x))
    tol = a * ((1 - a) * (x.abs() + 5) * U + 2 * U) + TINY
    return a, tol


def features_reference(feat, w):
    """features[:, :32] = sequential fmaf(feat_s, w_s, acc) over the 32 samples (the traced weights include the top-up):
    one rounding per step, <= S U of the sum of |terms|, plus the denormal floor."""
    terms = feat.double() * w.double()[..., None]
    S = w.shape[1]
    return terms.sum(1), S * U * terms.abs().sum(1) + S * TINY


def check_shading(out, tr, rays, idx, cfg, params):
    """Stage 3: alpha (bounded), weights / accumulation / depth / prop depths / appearance (bit for bit), the features'
    first 32 columns (bounded).  Returns the worst ratios."""
    worst = {}
    sp = Spacing(cfg)
    s_near, s_far = sp.near_far(rays, idx)
    beta = float(np.float32(float(params["field.sdf_to_density.beta"].abs().item() + 0.0001)))
    a_ref, a_tol = alpha_reference(tr["sdf"], beta)
    worst["alpha"] = _ratio(tr["alpha"], a_ref, a_tol, "alpha from sdf")
    w, acc = weights_bits(tr["alpha"])
    _bits_equal(tr["weights"], w, "weights from alpha")
    _bits_equal(out["accumulation"].reshape(-1), acc, "accumulation")
    _bits_equal(out["depth"].reshape(-1), depth_bits(w[:, :-1], tr["bins_e_2"].float()), "depth")
    S0 = cfg.sampling.num_proposal_samples[0]
    e0 = sp.to_euclid(Spacing.linspace01(S0).expand(idx.numel(), -1), s_near, s_far)
    _bits_equal(out["prop_depth_0"].reshape(-1), depth_bits(tr["prop_weights_0"].float(), e0), "prop_depth_0")
    _bits_equal(out["prop_depth_1"].reshape(-1), depth_bits(tr["prop_weights_1"].float(), tr["bins_e_1"].float()), "prop_depth_1")
    nff = cfg.nff_out_dim
    sensor = rays["sensor_idx"].reshape(-1)[idx] if "sensor_idx" in rays else torch.zeros(idx.numel(), dtype=torch.long)
    app = appearance_bits(cfg, params, rays["times"].reshape(-1)[idx], sensor)
    _bits_equal(out["features"][:, nff:].contiguous(), app, "appearance columns")
    f_ref, f_tol = features_reference(tr["field_feature"], tr["weights"])
    worst["features"] = _ratio(out["features"][:, :nff], f_ref, f_tol, "features[:, :32]")
    return worst


def check_sliced(dev, image_width):
    """2^21 + 4099 rays in "split" mode: the bundle is rendered in slices of the sampling -> shading hand-over buffer
    (whole 16-row tile bands with an image width), which moves every output and trace pointer (offset_rays).  The bundle
    repeats the config-2 rays, so every ray must equal its first copy bit for bit; the rays on both sides of each slice
    boundary and the ragged end are also checked against the bit-exact restatements (a partial trace, ~1 GB)."""
    t0 = time.perf_counter()
    cfg, params, rays, _ = scene_rays(dev, "config2")
    n0 = rays["origins"].shape[0]
    n = (1 << 21) + 4099
    big = {k: v.repeat(*([n // n0 + 1] + [1] * (v.dim() - 1)))[:n] for k, v in rays.items()}
    r = renderer(dev, cfg, params)
    traced = ("inds_2", "bins_e_2", "alpha", "weights")
    out = r.render({k: v.to(dev) for k, v in big.items()}, want_trace=traced, image_width=image_width, mode="split")
    slice_ = 1 << 21
    if image_width:
        band = image_width * 16
        slice_ = slice_ // band * band
    bounds = list(range(slice_, n, slice_))
    idx = torch.cat([torch.arange(b - 256, b + 256) for b in bounds] + [torch.arange(n - 300, n)])
    sub = select(out, idx)
    first = select(out, idx % n0)
    for k in ("features", "depth", "accumulation", "prop_depth_0", "prop_depth_1") + traced:
        _bits_equal(sub[k], first[k], f"sliced render (image_width {image_width}): {k} of the copies")
    w, acc = weights_bits(sub["alpha"])
    _bits_equal(sub["weights"], w, "sliced: weights from alpha")
    _bits_equal(sub["accumulation"].reshape(-1), acc, "sliced: accumulation")
    _bits_equal(sub["depth"].reshape(-1), depth_bits(w[:, :-1], sub["bins_e_2"].float()), "sliced: depth")
    nff = cfg.nff_out_dim
    app = appearance_bits(cfg, params, big["times"].reshape(-1)[idx], big["sensor_idx"].reshape(-1)[idx])
    _bits_equal(sub["features"][:, nff:].contiguous(), app, "sliced: appearance columns")
    return bounds, time.perf_counter() - t0


# ====================================================================================== stage 1: proposal weights
def _gauss32(o, d, area, e):
    """sample_gaussian's means, op by op in fp32 (fp32 CPU tensors): o, d [n, 3], e [n, S+1] -> [n, S, 3]."""
    e0, e1 = e[:, :-1], e[:, 1:]
    md = (e1 - e0) / 2.0
    t = e0 + md
    return o[:, None, :] + d[:, None, :] * t[..., None]


def _gauss64(o, d, area, e):
    """The same gaussians in float64 from the fp32 edges: means [n, S, 3], std [n, S]."""
    e = e.double()
    e0, e1 = e[:, :-1], e[:, 1:]
    md = (e1 - e0) / 2
    t = e0 + md
    mean = o.double()[:, None, :] + d.double()[:, None, :] * t[..., None]
    std = (area.double()[:, None] * t * t * md).clamp_min(0) ** (1.0 / 3.0)
    return mean, std


def _contract32(mean, scale):
    """contract()'s positions in fp32 (IEEE divisions, the reference's op sequence)."""
    x = mean / _f(scale)
    mag = x.abs().amax(-1, keepdim=True)
    a = 2.0 - 1.0 / mag
    y = torch.where(mag < 1.0, x, a * (x / mag))
    return (y + 2.0) * 0.25


def _normalize3(v):
    """normalize3 (F.normalize): v / max(sqrt((x x + y y) + z z), 1e-12), fp32."""
    n = torch.sqrt((v[..., 0] * v[..., 0] + v[..., 1] * v[..., 1]) + v[..., 2] * v[..., 2])
    return v / torch.clamp_min(n, _f(1e-12))[..., None]


def _dot3(a, b):
    return (a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]


class ActorFrames:
    """The per-ray actor frames of lane_actor_candidates (after the keyframe Gram-Schmidt of actors_prep_kernel), op by
    op in fp32 on the CPU: rotation R [n, A, 3, 3] and translation t [n, A, 3] of world -> box, the padded half sizes
    [A, 3], validity and the ray-line cull.  box() gives the kernel's box-frame position of a sample bit for bit."""

    def __init__(self, params, cfg, o, d, times):
        rot6 = params["dynamic_actors.actor_rotations_6d"].detach().float().cpu()
        pos = params["dynamic_actors.actor_positions"].detach().float().cpu()
        ts = params["dynamic_actors.unique_timestamps"].detach().float().cpu()
        pres = params["dynamic_actors.actor_present_at_time"].cpu().bool()
        a1 = _normalize3(rot6[..., :3])
        a2 = _normalize3(rot6[..., 3:] - _dot3(a1, rot6[..., 3:])[..., None] * a1)
        kf = torch.cat([a1, a2, pos], -1)  # [T, A, 9]
        times = times.float().contiguous()
        right = torch.searchsorted(ts, times)  # first keyframe time >= t
        left = (right - 1).clamp_min(0)
        right = right.clamp_max(ts.numel() - 1)
        tl, tr = ts[left], ts[right]
        frac = torch.clamp((times - tl) / ((tr - tl) + _f(1e-6)), 0.0, 1.0)
        kl, kr = kf[left], kf[right]
        p = kl + (kr - kl) * frac[:, None, None]  # [n, A, 9]
        self.valid = pres[left] | pres[right]
        b1 = _normalize3(p[..., 0:3])
        b2 = _normalize3(p[..., 3:6] - _dot3(b1, p[..., 3:6])[..., None] * b1)
        b3 = torch.stack([b1[..., 1] * b2[..., 2] - b1[..., 2] * b2[..., 1], b1[..., 2] * b2[..., 0] - b1[..., 0] * b2[..., 2],
                          b1[..., 0] * b2[..., 1] - b1[..., 1] * b2[..., 0]], -1)
        self.R = torch.stack([b1, b2, b3], -1)  # R[..., i, j] = b_j[i]: row i of world -> box
        self.t = -_dot3(self.R, p[..., None, 6:9])
        self.pos = p[..., 6:9]
        pad = params.get("dynamic_actors.actor_padding")
        pad = torch.tensor(list(cfg.actor_bbox_padding)) if pad is None else pad.detach().float().cpu()
        self.bounds = params["dynamic_actors.actor_sizes"].detach().float().cpu() * 0.5 + pad.float()

    def box(self, g, aid):
        """Box-frame positions [..., 3] (fp32, the kernel's op order) of samples g [n, S, 3] in actors aid [n, S] >= 0,
        and the rotations [n, S, 3, 3]."""
        ray = torch.arange(g.shape[0])[:, None].expand_as(aid)
        R, t = self.R[ray, aid], self.t[ray, aid]
        return _dot3(R, g[..., None, :]) + t, R


def _grid(tables, F, T, scalings, c32, cs64, dev, base=None):
    """One hash grid at the fp32 cells / offsets of c32 [P, 3] (on the CPU, where the fp32 pass ran), float64
    interpolation: per level and feature v [P, L, F], the interpolation of |f| (V_abs), and the float64 level weight
    1 / max(1, 2 res std) with its argument t [P, L].  `base` [P]: a row offset per sample (the actor's table)."""
    sc = scalings.float().cpu()
    idx, off = O.hash_indices(c32, sc, T)  # [P, L, 8], [P, L, 3]
    if base is not None:
        idx = idx + base[:, None, None]
    f = tables.reshape(-1, F).to(dev)[idx.to(dev)].double()  # [P, L, 8, F]
    off = off.to(dev).double()
    ox, oy, oz = off[..., 0:1], off[..., 1:2], off[..., 2:3]

    def tri(f):
        c = [f[..., k, :] for k in range(8)]
        f03, f12 = c[0] * ox + c[3] * (1 - ox), c[1] * ox + c[2] * (1 - ox)
        f56, f47 = c[5] * ox + c[6] * (1 - ox), c[4] * ox + c[7] * (1 - ox)
        return (f03 * oy + f12 * (1 - oy)) * oz + (f47 * oy + f56 * (1 - oy)) * (1 - oz)

    t = sc.to(dev).double()[None, :] * 2 * cs64.to(dev)[:, None]
    return tri(f), tri(f.abs()), 1.0 / t.clamp_min(1.0), t


def _level_terms(v, vabs, lw, t):
    """Grid feature x = fl(trilerp fl-weights) of one level and its bound: 3 FMA-folded blends, each <= 2 U of its
    |terms| plus U for the rounded 1 - offset (<= 9 U V_abs); the level weight by rcp.approx (<= 1 ulp = 2 U) of
    fl(2 res std) (U) and the std's STD_REL, only where 2 res std > 1 (else exactly 1); the product U."""
    lw_rel = torch.where(t * (1 + STD_REL + U) > 1.0, torch.full_like(t, 3 * U + STD_REL), torch.zeros_like(t))[..., None]
    lw = lw[..., None]
    x = v * lw
    return x, 9 * U * vabs * lw + (v * lw).abs() * (lw_rel + U)


class FieldSamples:
    """The samples of one field evaluation at fp32 edges e [n, S+1] of the rays (o, d, area, times), with the kernel's
    actor assignment aid [n, S]: fp32 gaussian means (op by op), float64 means / std, the fp32 contracted positions that
    fix the grid cells (static: contract(mean, static_scale); actor: contract(box position, actor_scale)) and the
    float64 contracted std."""

    def __init__(self, params, cfg, frames, o, d, area, times, e, aid, actor_scale):
        self.n, self.S = e.shape[0], e.shape[1] - 1
        g32 = _gauss32(o.float(), d.float(), area.float(), e.float())
        self.mean64, std64 = _gauss64(o, d, area, e)
        self.aid = aid.reshape(-1).long()
        self.static = self.aid < 0
        scale = float(params["static_scale"])
        s = self.static
        self.c32_s = _contract32(g32.reshape(-1, 3)[s], scale)
        _, cs = O.scaled_contraction(self.mean64.reshape(-1, 3)[s], std64.reshape(-1, 1)[s], scale)
        self.cs64_s = cs[:, 0]
        self.R_a = None
        if not s.all():
            q32, R = frames.box(g32, aid.long().clamp_min(0))
            a = ~s
            q32, self.R_a = q32.reshape(-1, 3)[a], R.reshape(-1, 3, 3)[a]
            self.c32_a = _contract32(q32, actor_scale)
            _, cs = O.scaled_contraction(q32.double(), std64.reshape(-1, 1)[a], actor_scale)
            self.cs64_a = cs[:, 0]


def _actor_tables(params, prefix, n_actors):
    return torch.stack([params[f"{prefix}.hashgrid.actor_grids.{a}.hash_table"].float() for a in range(n_actors)])


def proposal_density_reference(params, cfg, fs, dev, drop=None):
    """float64 density of proposal_fields.1 at the samples fs (static: 6 levels; actor: the actor's 4-level grid,
    decoder inputs 0..3) and its relative bound: per level _level_terms; acc = sequential fmaf(x, dec, acc) over the L
    levels, <= L U of sum |dec x|, plus U per term already in x; density = expf(acc): relative E_acc + 4 U.
    `drop` = (flat sample, level): that level's term left out at that sample (a corrupted result for the self-tests)."""
    pre = "proposal_fields.1"
    gc = cfg.proposal_grid_2
    dec = params[f"{pre}.density_decoder.weight"].reshape(-1).double().to(dev)
    P = fs.aid.numel()
    acc = torch.zeros(P, dtype=torch.float64, device=dev)
    E = torch.zeros_like(acc)
    parts = [(fs.static, params[f"{pre}.hashgrid.static_grid.hash_table"], gc.static, fs.c32_s, fs.cs64_s, None,
              params[f"{pre}.hashgrid.static_grid.scalings"])]
    if fs.R_a is not None:
        A, T = cfg.n_actors, gc.actor.hash_table_size
        base = fs.aid[~fs.static] * gc.actor.num_levels * T
        parts.append((~fs.static, _actor_tables(params, pre, A), gc.actor, fs.c32_a, fs.cs64_a, base,
                      params[f"{pre}.hashgrid.actor_grids.0.scalings"]))
    for m, tab, g, c32, cs, base, sc in parts:
        v, vabs, lw, t = _grid(tab, 1, g.hash_table_size, sc, c32, cs, dev, base)
        x, Ex = _level_terms(v, vabs, lw, t)
        L = g.num_levels
        terms = dec[:L] * x[..., 0]
        if drop is not None and m[drop[0]]:
            terms[int(m[:drop[0]].sum()), drop[1]] = 0.0
        acc[m.to(dev)] = terms.sum(-1)
        E[m.to(dev)] = (dec[:L].abs() * Ex[..., 0]).sum(-1) + L * U * terms.abs().sum(-1)
    return torch.exp(acc).reshape(fs.n, fs.S).cpu(), (E + 4 * U).reshape(fs.n, fs.S).cpu()


def proposal_weights_reference(dens, rel_dens, e):
    """Weights of one round from the float64 density and its relative bound, with the kernel's fp32 deltas:
      dd = fl(fl(e1 - e0) dens): rel <= rel_dens + 2 U;  alpha = fl(1 - expf(-dd));  T = expf(-(float) excl), excl the
      double sum of the fp32 dd;  w = fl(alpha T).  Multiplicative errors through exp are bounded by expm1 of the
      argument's error (no first-order truncation where dd or excl is large), plus the fp32 denormal floor.
    Returns (w64, tol, excl64 lower bound)."""
    e = e.double()
    delta = e[:, 1:] - e[:, :-1]
    dd = delta * dens
    E_dd = dd * (rel_dens + 2 * U)
    ea = torch.exp(-dd)
    alpha = -torch.expm1(-dd)
    E_alpha = ea * torch.expm1(E_dd + 4 * U) + U * alpha
    excl = torch.cat([torch.zeros_like(dd[:, :1]), torch.cumsum(dd, 1)[:, :-1]], 1)
    S = dd.shape[1]
    E_excl = torch.cat([torch.zeros_like(dd[:, :1]), torch.cumsum(E_dd, 1)[:, :-1]], 1) + (S * 2.0 ** -52 + U) * excl
    T = torch.exp(-excl)
    E_T = T * torch.expm1(E_excl + 4 * U) + 2 * TINY
    w = alpha * T
    tol = alpha * E_T + T * E_alpha + U * w + 2 * TINY
    return w, tol, excl - E_excl


def _ray_inputs(rays, idx, cfg):
    o = rays["origins"].reshape(-1, 3)[idx].float()
    d = rays["directions"].reshape(-1, 3)[idx].float()
    lid = rays["is_lidar"].reshape(-1)[idx].bool() if "is_lidar" in rays else torch.zeros(idx.numel(), dtype=torch.bool)
    area = rays["pixel_area"].reshape(-1)[idx].float() * torch.where(lid, _f(1.0), _f(float(cfg.rgb_upsample_factor ** 2)))
    return o, d, area, rays["times"].reshape(-1)[idx].float()


def _frames(params, cfg, o, d, times):
    return ActorFrames(params, cfg, o, d, times) if cfg.n_actors else None


def round0_edges(cfg, rays, idx):
    sp = Spacing(cfg)
    s_near, s_far = sp.near_far(rays, idx)
    S0 = cfg.sampling.num_proposal_samples[0]
    return sp.to_euclid(Spacing.linspace01(S0).expand(idx.numel(), -1), s_near, s_far)


def main_edges(cfg, bins_e_2):
    """The shading stage's euclidean edges: the last one moved to the sky, fl(e + fl(sky - e))."""
    e = bins_e_2.float().clone()
    sky = _f(cfg.sampling.sky_distance)
    e[:, -1] = e[:, -1] + (sky - e[:, -1])
    return e


def check_proposal_weights(tr, rays, idx, cfg, params, dev, chunk=2048):
    """Stage 1 on every ray (actor samples through the actor's proposal grid, at the kernel's fp32 box positions);
    returns (worst ratio, excl lower bounds of round 0 [n, S0])."""
    o, d, area, times = _ray_inputs(rays, idx, cfg)
    e0 = round0_edges(cfg, rays, idx)
    worst, low0 = 0.0, None
    for rd, e in enumerate((e0, tr["bins_e_1"].float())):
        aid = tr.get(f"actor_id_{rd}", torch.full(e[:, 1:].shape, -1, dtype=torch.int32))
        w_all, tol_all, low_all = [], [], []
        for c0 in range(0, idx.numel(), chunk):
            c = slice(c0, c0 + chunk)
            fs = FieldSamples(params, cfg, _frames(params, cfg, o[c], d[c], times[c]), o[c], d[c], area[c], times[c], e[c],
                              aid[c], cfg.proposal_grid_2.actor_scale)
            dens, rel = proposal_density_reference(params, cfg, fs, dev)
            w, tol, low = proposal_weights_reference(dens, rel, e[c])
            w_all.append(w), tol_all.append(tol), low_all.append(low)
        worst = max(worst, _ratio(tr[f"prop_weights_{rd}"], torch.cat(w_all), torch.cat(tol_all), f"prop_weights_{rd}"))
        if rd == 0:
            low0 = torch.cat(low_all)
    return worst, low0


# ====================================================================================== stage 3: the main field
def gamma_tc(K):
    """Per-term constant of one 3xTF32 wgmma layer with K inputs (the kernel's half_mma): a = hi + lo with hi = a with
    the low 13 mantissa bits cleared (|lo| < 2^-10 |a|), lo passed as a tf32 operand and so truncated (< 2^-10 |lo| <
    2^-20 |a|); the same split of W; lo lo dropped (< 2^-20 |a w|).  Three products per term: < 3 2^-20 |a w|.  The 3 K
    products and the bias are accumulated in fp32 in an unspecified order and rounding mode (truncation allowed): each of
    the 3 K + 1 additions <= 2^-22 of the running sum, <= 2^-22 (3 K + 1) of sum |terms|."""
    return 3 * 2.0 ** -20 + (3 * K + 1) * 2.0 ** -22


def gamma_ffma(K):
    """dense<> on the CUDA cores: the bias then K sequential FMAs, one rounding each: (K + 1) U of sum |terms|."""
    return (K + 1) * U


def _sh4_64(v):
    """components_from_spherical_harmonics(levels=4) in float64, on (dir + 1) / 2 given as v [..., 3]."""
    x, y, z = v[..., 0], v[..., 1], v[..., 2]
    xx, yy, zz = x * x, y * y, z * z
    return torch.stack([torch.full_like(x, 0.28209479177387814), 0.4886025119029199 * y, 0.4886025119029199 * z,
                        0.4886025119029199 * x, 1.0925484305920792 * x * y, 1.0925484305920792 * y * z,
                        0.9461746957575601 * zz - 0.31539156525251999, 1.0925484305920792 * x * z,
                        0.5462742152960396 * (xx - yy), 0.5900435899266435 * y * (3 * xx - yy), 2.890611442640554 * x * y * z,
                        0.4570457994644658 * y * (5 * zz - 1), 0.3731763325901154 * z * (5 * zz - 3),
                        0.4570457994644658 * x * (5 * zz - 1), 1.445305721320277 * z * (xx - yy),
                        0.5900435899266435 * x * (xx - 3 * yy)], -1)


def _tf32(x):
    """x with the low 13 mantissa bits of its fp32 value cleared (a tf32 operand without its lo correction)."""
    return (x.float().view(torch.int32) & -8192).view(torch.float32).double()


def main_field_reference(params, cfg, fs, d, dev, gamma, corrupt=None):
    """float64 sdf [n, S] and field features [n, S, 32] at the samples fs, with per-entry bounds.
    Grid features: static 8 levels x 4, actor 4 levels x 4 padded with 16 zeros (_level_terms per entry).  Direction:
    the ray's, or for an actor sample rotated into the kernel's fp32 box frame and normalised, q / (|q| + 1e-7) (the
    kernel's fp32 rotation and normalisation: <= 16 U per component).  SH of (dir + 1) / 2: polynomials of degree <= 3
    on [0, 1]^3 whose terms are <= 3 in magnitude, <= 24 U each, and Lipschitz <= 10 in the max-norm of the input.
    Each layer y = W a + b carries E_y = gamma(K) (|W| |a| + |b|) + |W| E_a (ReLU is 1-Lipschitz, and a unit below minus its bound
    carries none); the last adds the
    residual geo_embedding into its accumulator (a term of its own, plus E_geo).  The sdf neuron is an fp32 FMA dot
    product over the 32 hidden units reduced over the quad, plus the bias: (32 + 3) U of sum |terms|, plus |w| E_h.
    `corrupt`: "tf32" runs the last layer as 1xTF32 (3xTF32 without its correction), "unpadded" fills an actor
    sample's inputs 16..31 with its own features 0..15 (the self-tests)."""
    P = fs.aid.numel()
    x = torch.zeros(P, 32, dtype=torch.float64, device=dev)
    Ex = torch.zeros_like(x)
    gc = cfg.grid
    m = fs.static.to(dev)
    v, vabs, lw, t = _grid(params["field.hashgrid.static_grid.hash_table"], 4, gc.static.hash_table_size,
                           params["field.hashgrid.static_grid.scalings"], fs.c32_s, fs.cs64_s, dev)
    xs, Es = _level_terms(v, vabs, lw, t)
    x[m], Ex[m] = xs.reshape(-1, 32), Es.reshape(-1, 32)
    dirs = d.double()[:, None, :].expand(fs.n, fs.S, 3).reshape(-1, 3).clone().to(dev)
    E_dir = torch.full((P, 1), U, dtype=torch.float64, device=dev)
    if fs.R_a is not None:
        T = gc.actor.hash_table_size
        base = fs.aid[~fs.static] * gc.actor.num_levels * T
        v, vabs, lw, t = _grid(_actor_tables(params, "field", cfg.n_actors), 4, T, params["field.hashgrid.actor_grids.0.scalings"],
                               fs.c32_a, fs.cs64_a, dev, base)
        xa, Ea = _level_terms(v, vabs, lw, t)
        xa = torch.cat([xa.reshape(-1, 16), torch.zeros_like(xa.reshape(-1, 16))], 1)
        if corrupt == "unpadded":
            xa[:, 16:] = xa[:, :16]
        x[~m], Ex[~m] = xa, torch.cat([Ea.reshape(-1, 16), torch.zeros_like(Ea.reshape(-1, 16))], 1)
        q = (fs.R_a.double().to(dev) @ dirs[~m][..., None])[..., 0]
        dirs[~m] = q / (q.norm(dim=-1, keepdim=True) + 1e-7)
        E_dir[~m] = 16 * U
    sh = _sh4_64((dirs + 1) / 2)
    E_sh = 72 * U + 10 * E_dir

    def W(k):
        return params[k + ".weight"].double().to(dev), params[k + ".bias"].double().to(dev)

    def lin(w, b, a, Ea, extra=0.0):
        return a @ w.T + b, gamma(w.shape[1]) * (a.abs() @ w.abs().T + b.abs() + extra) + Ea @ w.abs().T

    def relu(y, E):  # 1-Lipschitz; a unit below -E is 0 in the kernel and the reference alike, with no error
        return y.clamp_min(0), torch.where(y + E <= 0, torch.zeros_like(E), E)

    w0, b0 = W("field.mlp_geo.layers.0")
    w1, b1 = W("field.mlp_geo.layers.1")
    h0, Eh0 = relu(*lin(w0, b0, x, Ex))
    sdf = h0 @ w1[0] + b1[0]
    E_sdf = 35 * U * (h0.abs() @ w1[0].abs() + b1[0].abs()) + Eh0 @ w1[0].abs()
    geo, Egeo = lin(w1[1:], b1[1:], h0, Eh0)
    in2, Ein2 = torch.cat([geo, sh], 1), torch.cat([Egeo, E_sh.expand(P, 16)], 1)
    f0, fb0 = W("field.mlp_feature.layers.0")
    f1, fb1 = W("field.mlp_feature.layers.1")
    f2, fb2 = W("field.mlp_feature.layers.2")
    h2, Eh2 = relu(*lin(f0, fb0, in2, Ein2))
    h3, Eh3 = relu(*lin(f1, fb1, h2, Eh2))
    if corrupt == "tf32":  # the last layer as 1xTF32: its input and weights rounded to tf32, no lo terms
        out = _tf32(h3) @ _tf32(f2).T + fb2
        Eout = torch.zeros_like(out)
    else:
        out, Eout = lin(f2, fb2, h3, Eh3, extra=geo.abs())
    feat = out + geo
    E_feat = Eout + Egeo + U * feat.abs()
    n, S = fs.n, fs.S
    return sdf.reshape(n, S).cpu(), E_sdf.reshape(n, S).cpu(), feat.reshape(n, S, 32).cpu(), E_feat.reshape(n, S, 32).cpu()


def check_main_field(tr, rays, idx, cfg, params, dev, gamma, chunk=2048):
    """Stage 3: sdf and field_feature of every sample against main_field_reference at the traced bins_e_2 (the last edge
    moved to the sky), with the traced actor assignment.  Returns the worst ratios."""
    o, d, area, times = _ray_inputs(rays, idx, cfg)
    e = main_edges(cfg, tr["bins_e_2"])
    aid = tr.get("actor_id_main", torch.full(e[:, 1:].shape, -1, dtype=torch.int32))
    ws, wf = 0.0, 0.0
    for c0 in range(0, idx.numel(), chunk):
        c = slice(c0, c0 + chunk)
        fs = FieldSamples(params, cfg, _frames(params, cfg, o[c], d[c], times[c]), o[c], d[c], area[c], times[c], e[c], aid[c],
                          cfg.grid.actor_scale)
        sdf, Es, feat, Ef = main_field_reference(params, cfg, fs, d[c], dev, gamma)
        ws = max(ws, _ratio(tr["sdf"][c], sdf, Es, "sdf"))
        wf = max(wf, _ratio(tr["field_feature"][c], feat, Ef, "field_feature"))
    return {"sdf": ws, "field_feature": wf}


# ====================================================================================== stage 6: actor ids
def check_actor_ids(tr, rays, idx, cfg, params, chunk=512):
    """actor_id_0 / _1 / _main against a float64 box test of the float64 sample means at the traced edges: the highest
    actor whose padded box (the fp32 half sizes) strictly contains the mean, among the actors present at a bracketing
    keyframe.  A mismatch is allowed only where the float64 box coordinate of some present actor lies within
    64 U (|mean| + |box centre| + half size) of a face (the kernel's fp32 frame is a few ulp of those magnitudes off).
    Returns (mismatches at a face, samples compared)."""
    o, d, area, times = _ray_inputs(rays, idx, cfg)
    p64 = {k: (v.double() if torch.is_tensor(v) and v.is_floating_point() else v) for k, v in params.items()}
    b2w, valid = O.boxes2world_at(p64, times.double())
    w2b = O.pose_inverse(b2w)  # [n, A, 3, 4]
    fr = ActorFrames(params, cfg, o, d, times)
    bnd = fr.bounds.double()
    edges = {"actor_id_0": round0_edges(cfg, rays, idx), "actor_id_1": tr["bins_e_1"].float(), "actor_id_main": main_edges(cfg, tr["bins_e_2"])}
    faces, total = 0, 0
    for k, e in edges.items():
        mean64, _ = _gauss64(o, d, area, e)
        for c0 in range(0, idx.numel(), chunk):
            c = slice(c0, c0 + chunk)
            R, t = w2b[c, :, :3, :3], w2b[c, :, :3, 3]
            q = torch.einsum("naij,nsj->nsai", R, mean64[c]) + t[:, None]  # [n, S, A, 3]
            ok = valid[c][:, None, :]
            inside = ok & (q.abs() < bnd).all(-1)
            A = inside.shape[-1]
            ar = torch.arange(A)
            ref = torch.where(inside.any(-1), (inside * (ar + 1)).amax(-1) - 1, torch.full(inside.shape[:-1], -1))
            scale = mean64[c].abs().amax(-1)[..., None] + b2w[c, :, :3, 3].abs().amax(-1)[:, None, :] + bnd.amax(-1)
            near = (ok[..., None] & ((q.abs() - bnd).abs() <= 64 * U * scale[..., None])).any(-1).any(-1)
            bad = tr[k][c].long() != ref
            assert not (bad & ~near).any(), (f"{k}: {int((bad & ~near).sum())} samples assigned to the wrong actor away "
                                             f"from every box face, first at {(bad & ~near).nonzero()[:3].tolist()}")
            faces += int(bad.sum())
            total += bad.numel()
    assert faces <= max(2, total // 100000), f"{faces} of {total} actor ids differ at a box face"
    return faces, total


# ====================================================================================== lidar head
def check_lidar(out, cfg, params):
    """intensity / ray_drop_logits from the output features through the lidar decoder in float64 (lidar_decode_kernel:
    dense<> FFMA layers, gamma_ffma; intensity = 1 / (1 + expf(-o0)): relative (1 - i)(4 U) + 2 U, plus i (1 - i) E_o0)."""
    x = out["features"].double()
    E = torch.zeros_like(x)
    for i in range(3):
        w, b = params[f"lidar_decoder.layers.{i}.weight"].double(), params[f"lidar_decoder.layers.{i}.bias"].double()
        y = x @ w.T + b
        E = gamma_ffma(w.shape[1]) * (x.abs() @ w.abs().T + b.abs()) + E @ w.abs().T
        x = y.clamp_min(0) if i < 2 else y
    it = torch.sigmoid(x[:, 0])
    tol_i = it * (1 - it) * E[:, 0] + it * ((1 - it) * 4 * U + 2 * U) + TINY
    return {"intensity": _ratio(out["intensity"].reshape(-1), it, tol_i, "intensity"),
            "ray_drop_logits": _ratio(out["ray_drop_logits"].reshape(-1), x[:, 1], E[:, 1] + TINY, "ray_drop_logits")}


def early_exit_warps(low_excl, idx):
    """Warps (32 consecutive rays of the flat walk, all in idx) whose round-0 transmittance is certainly 0 in fp32 on
    all 32 lanes before the last sample, by the float64 lower bound of the exclusive sum: the kernel's
    vote_all_converged(T == 0) skips the rest of the round there.  The count is inferred from the reference, not read
    from the kernel; that the skip changes no result is checked by the partial-trace comparison."""
    dead = low_excl > EXIT_ARG  # [n, S0]
    first = torch.where(dead.any(1), dead.float().argmax(1), torch.full((dead.shape[0],), dead.shape[1]))
    count = 0
    for wb in range(0, idx.numel() - 31, 32):
        seg = idx[wb:wb + 32]
        if seg[-1] - seg[0] != 31 or seg[0] % 32 != 0:
            continue
        if int(first[wb:wb + 32].max()) < dead.shape[1] - 1:
            count += 1
    return count


# ====================================================================================== whole-scene checks
def select(out, idx):
    return {k: v[idx.to(v.device)].cpu() for k, v in out.items()}


def check_scene(dev, name, mode="split", n_random=127, report=print):
    """Full trace of one scene: every stage on whole 128-ray warp groups (every ray on the CPU); then a render with a
    partial trace (no actor ids: the early exit on) and an untraced render must match the full trace bit for bit.
    Returns (worst ratio per stage, inferred early-exit warps, actor-id face exceptions, full render, referenced rays)."""
    t0 = time.perf_counter()
    cfg, params, rays, width = scene_rays(dev, name)
    r = renderer(dev, cfg, params)
    rd = {k: (v.to(dev) if dev != "cpu" else v) for k, v in rays.items()}
    full = r.render(rd, want_trace=True, image_width=width, mode=mode, want_intensity=True)
    n = rays["origins"].shape[0]
    extra = ()
    if cfg.n_actors:
        hit = (full["actor_id_main"] >= 0).any(1).cpu()
        extra = torch.unique(hit.nonzero()[:, 0] // 128)
    idx = torch.arange(n) if dev == "cpu" else pick_groups(n, n_random, seed=len(name), extra=extra)
    out = select(full, idx)
    worst = {}
    check_walk(out, rays, idx, cfg)
    worst.update(check_shading(out, out, rays, idx, cfg, params))
    fdev = "cpu" if dev == "cpu" else dev
    worst["prop_weights"], low = check_proposal_weights(out, rays, idx, cfg, params, fdev)
    worst.update(check_main_field(out, rays, idx, cfg, params, fdev, gamma_ffma if dev == "cpu" else gamma_tc))
    if "intensity" in out:
        worst.update(check_lidar(out, cfg, params))
    exits = early_exit_warps(low, idx) if width == 0 else 0
    faces = 0
    if cfg.n_actors:
        hits = int((out["actor_id_main"] >= 0).sum())
        assert hits >= max(10, n // 40), f"{name}: only {hits} actor samples: the actor branch is not exercised"
        faces, _ = check_actor_ids(out, rays, idx, cfg, params)
    # the traced fields and outputs do not depend on what else is traced (on the CPU the emulation always traces
    # everything, so these comparisons only bite on the GPU)
    part = r.render(rd, want_trace=PARTIAL, image_width=width, mode=mode)
    none = r.render(rd, want_trace=False, image_width=width, mode=mode)
    for k in PARTIAL:
        _bits_equal(part[k], full[k].cpu(), f"{name} {mode}: partial trace {k}")
    for k in ("features", "depth", "accumulation", "prop_depth_0", "prop_depth_1"):
        _bits_equal(part[k], full[k].cpu(), f"{name} {mode}: partial-trace output {k}")
        _bits_equal(none[k], full[k].cpu(), f"{name} {mode}: untraced output {k}")
    report(f"\n[render trace] {name} {mode}: {idx.numel()} of {n} rays referenced; worst |got - ref| / bound: "
           + ", ".join(f"{k} {v:.3g}" for k, v in worst.items())
           + f"; early-exit warps (inferred) {exits}; actor-id face exceptions {faces}; {time.perf_counter() - t0:.1f} s")
    return worst, exits, faces, full, idx
