"""Bodies of the tests of the camera-pose gradient operators (neurad_encoding_mean_bwd, isotropic_gaussian_bwd) and of the
camera optimizer mirror, shared by tests/test_zz_camera_opt_gpu.py (dev = "cuda": the real library, production table
sizes) and tests/test_camera_opt_cpu.py (dev = "cpu": the same device code through tests/camopt_fake_backend.py and the
host emulation, small tables).

dmean reference: float64 autograd through the oracle's NeuRADHashEncoding.forward (and, in density mode, the proposal
head with its trunc_exp), with the sample means, the tables, the decoder and the actor trajectories promoted to float64.
The grid CELLS, corner rows and interpolation offsets are the fp32 ones the kernel uses: a first fp32 pass records the
contracted positions of every lookup, and the float64 pass takes rows, floor() and offset VALUES from them while the
offsets' derivative (res times the float64 contraction's) is float64.  Offsets from a float64 contraction would differ
by up to res * ulp(x) ~ 2e-4 on the finest level, and the derivative along one axis is a function of the other axes'
offsets; a float64 contraction would also move some fine-level samples to a neighbouring cell.

Per-entry bound, per sample s and coordinate i:  |got - ref| <= REL * max_i |ref_s,i| + ABS_FLOOR * max |ref|.
The kernel sums up to 8 levels x 4 features x 3 trilinear differences of fp32 corner values in fp32 (FMA) and backs the
contraction up with fp32 reciprocals and cbrtf, where the reference rounds once in float64.  The trilinear differences
(f_c - f_f) cancel: on a level whose corner values agree to k bits, the difference keeps 24 - k bits, so a row's error
is relative to the row's largest TERM, not to its sum.  REL = 1e-3 allows 2^14 ulps of the row's largest entry; the
measured worst ratios (printed by the GPU tests) are far below 1."""
import torch
import torch.nn.functional as F

import neurad_studio_b200 as nsb
from neurad_studio_b200.lib import FIELD_MAIN, FIELD_PROP1
from oracle import neurad_oracle as O
from oracle.convert import to_oracle_cfg
from tests import backward_scatter_cases as BS

U = 2.0 ** -24
REL = 1e-3
ABS_FLOOR = 1e-6


# ------------------------------------------------------------------------------------------------ float64 reference
class _FixedCells:
    """Patches O.hash_encode: the fp32 pass records each call's contracted positions; the float64 pass reads its rows
    and floors from the recorded fp32 positions and interpolates with float64 offsets of its own positions."""

    def __init__(self):
        self.recorded, self.replay = [], None

    def __enter__(self):
        self._orig = O.hash_encode

        def enc(x, table, scalings, table_size):
            if self.replay is None:
                self.recorded.append(x.detach().clone())
                return self._orig(x, table, scalings, table_size)
            x32 = self.replay.pop(0)
            assert x32.shape == x.shape, "the float64 pass took a different actor split than the fp32 pass"
            sc32 = scalings.float()
            idx, _ = O.hash_indices(x32, sc32, table_size)
            p32 = x32[..., None, :] * sc32.view(-1, 1)
            p64 = x[..., None, :] * scalings.double().view(-1, 1)
            off = (p32 - torch.floor(p32)).double() + (p64 - p64.detach())  # the fp32 offset, the float64 derivative
            f = [table[idx[..., i]] for i in range(8)]
            ox, oy, oz = off[..., 0:1], off[..., 1:2], off[..., 2:3]
            f03, f12 = f[0] * ox + f[3] * (1 - ox), f[1] * ox + f[2] * (1 - ox)
            f56, f47 = f[5] * ox + f[6] * (1 - ox), f[4] * ox + f[7] * (1 - ox)
            v = (f03 * oy + f12 * (1 - oy)) * oz + (f47 * oy + f56 * (1 - oy)) * (1 - oz)
            return torch.flatten(v, start_dim=-2, end_dim=-1)

        O.hash_encode = enc
        return self

    def __exit__(self, *exc):
        O.hash_encode = self._orig


def dmean_reference(params, cfg, field, mean, std, times, flip=None, dfeatures=None, ddensity=None):
    """float64 dL/d mean [N,S,3] of field `field` (FIELD_MAIN: features mode with cotangent dfeatures [N*S,D];
    FIELD_PROP1: density mode with cotangent ddensity [N,S]).  Also returns the fp32 density (density mode)."""
    ocfg = to_oracle_cfg(cfg)
    prefix = "field" if field == FIELD_MAIN else "proposal_fields.1"
    fcfg = ocfg.main if field == FIELD_MAIN else ocfg.prop[1]
    n, s = mean.shape[0], mean.shape[1]
    m4, s4 = mean.reshape(n, s, 1, 3), std.reshape(n, s, 1, 1)

    def run(q, m, sd, t):
        feats, _ = O.hashgrid_forward(q, prefix, fcfg, ocfg, m, sd, t.reshape(n, 1, 1).expand(n, s, 1), None, flip=flip,
                                      require_actor_grad=field == FIELD_MAIN)
        return feats

    with _FixedCells() as fc:
        with torch.no_grad():
            feats32 = run(params, m4.float(), s4.float(), times.float())
        q64 = {k: (v.double() if torch.is_tensor(v) and v.dtype == torch.float32 else v) for k, v in params.items()}
        m64 = m4.double().requires_grad_(True)
        fc.replay = list(fc.recorded)
        feats = run(q64, m64, s4.double(), times.double())
        assert not fc.replay
    if field == FIELD_MAIN:
        loss = (feats * dfeatures.double().reshape(feats.shape)).sum()
        density32 = None
    else:
        w = params[f"{prefix}.density_decoder.weight"]
        density32 = torch.exp(F.linear(feats32, w)).reshape(n, s)
        dens = O._TruncExp.apply(F.linear(feats, w.double())).reshape(n, s)
        loss = (dens * ddensity.double()).sum()
    (g,) = torch.autograd.grad(loss, [m64], allow_unused=True)
    g = torch.zeros_like(m64) if g is None else g
    return g.reshape(n, s, 3), density32


def check_dmean(got, ref, what=""):
    """Per-entry bound of the module docstring; returns the worst |got - ref| / tol."""
    got = got.detach().cpu().double().reshape(ref.shape)
    row = ref.abs().amax(dim=-1, keepdim=True)
    tol = REL * row + ABS_FLOOR * float(ref.abs().max()) + 1e-30
    r = (got - ref).abs() / tol
    worst = int(r.reshape(-1).argmax())
    assert r.reshape(-1)[worst] <= 1.0, (f"{what}: |got - ref| / tol = {r.reshape(-1)[worst].item():.3g} at flat index {worst}: "
                                         f"got {got.reshape(-1)[worst].item():.9g}, ref {ref.reshape(-1)[worst].item():.9g}")
    return float(r.max())


def _tie_samples(mean, static_scale):
    """Constructed points on a tie of the inf-norm outside the unit cube (|x| = |y| > scale, and |x| = |y| = |z|), as the
    first samples of rays 0 and 1.  Scenes without actors only: the reference's actor cull (_get_actor_indices,
    neurad_encoding.py:225-263) takes each ray's line through its first and last sample, so a moved first sample changes
    which actor the later samples of its ray are assigned to there, but not in the kernel, which has no such cull."""
    m = mean.clone()
    k = min(m.shape[0], 2)
    pts = torch.tensor([[1.5, -1.5, 0.1], [-2.25, 2.25, 2.25]]) * static_scale
    for r in range(k):
        m[r, 0] = pts[r]
    return m


# ------------------------------------------------------------------------------------------------ operator cases
def backend(dev, cfg, params):
    """backward_scatter_cases.backend, with the camera-pose leaves of tests/camopt_fake_backend.py on the CPU."""
    if dev != "cpu":
        return BS.backend(dev, cfg, params)
    from tests.camopt_fake_backend import CamoptFakeBackend

    be = CamoptFakeBackend()
    be.load_params(cfg, params)
    return be


def mean_bwd_matches_float64_reference(dev, field, n, S, n_actors, flip, layout="spread", seed=3, ties=False):
    """neurad_encoding_mean_bwd of the main field (features) or a proposal field (density) against dmean_reference.
    Proposal-field samples inside an actor must get exactly 0."""
    cfg = BS.make_cfg(dev, n_actors)
    params, trajs = BS.make_scene(cfg, seed=seed)
    be = backend(dev, cfg, params)
    mean, std, t = BS.make_rays(n, S, seed, trajs, layout)
    mean, std = mean.reshape(n, S, 3), std.reshape(n, S)
    if ties:
        assert n_actors == 0, "tie samples are constructed in scenes without actors"
        mean = _tie_samples(mean, cfg.static_scale)
    gen = torch.Generator().manual_seed(seed + 1)
    fl = (torch.randint(0, 2, (n,), generator=gen).float() * 2 - 1) if flip else None
    dv = torch.device(dev, 0) if dev == "cuda" else torch.device("cpu")
    to = (lambda x: None if x is None else x.to(dv))  # noqa: E731
    if field == FIELD_MAIN:
        D = cfg.grid.static.out_dim
        G = torch.randn(n * S, D, generator=gen)
        ref, _ = dmean_reference(params, cfg, field, mean, std, t, fl, dfeatures=G)
        got = be.neurad_encoding_mean_bwd(field, to(mean), to(std), to(t), dfeatures=to(G), flip=to(fl))
    else:
        dd = torch.randn(n, S, generator=gen)
        dens = be.neurad_encoding(field, to(mean), to(std), to(t), None, want_features=False, want_density=True, flip=to(fl))["density"]
        ref, _ = dmean_reference(params, cfg, field, mean, std, t, fl, ddensity=dd)
        got = be.neurad_encoding_mean_bwd(field, to(mean), to(std), to(t), density=dens, ddensity=to(dd), flip=to(fl))
        if n_actors:
            aid = be.neurad_encoding(field, to(mean), to(std), to(t), None, want_features=False, want_actor_id=True)["actor_id"].cpu()
            inside = aid >= 0
            assert inside.any(), "no proposal sample inside an actor: the case does not test the zero gradient"
            assert (got.cpu()[inside] == 0).all(), "proposal-field samples inside an actor must get exactly 0"
    what = f"{'features' if field == FIELD_MAIN else 'density'} n={n} S={S} actors={n_actors} flip={flip}"
    return check_dmean(got, ref, what)


def mean_bwd_covers_both_sides(dev):
    """The inputs of the operator cases reach samples inside and outside |x|_inf = 1 and level weights on both sides of
    the clamp 2 res std = 1 (so both backward paths of the contraction and the level-weight term are exercised)."""
    cfg = BS.make_cfg(dev, 0)
    mean, std, _ = BS.make_rays(64, 32, 3, None, "spread")
    c_mean, c_std = O.scaled_contraction(mean, std, cfg.static_scale)
    mag = (mean / cfg.static_scale).abs().amax(-1)
    assert (mag < 1).any() and (mag >= 1).any()
    t = 2 * cfg.grid.static.scalings().view(1, 1, 1, -1) * c_std
    outside = (mag >= 1)[..., None]
    assert (t[outside.expand_as(t)] > 1).any() and (t < 1).any()


def empty_and_zero_cotangent_give_zeros(dev, n_actors):
    cfg = BS.make_cfg(dev, n_actors)
    params, trajs = BS.make_scene(cfg, seed=5)
    be = backend(dev, cfg, params)
    dv = torch.device(dev, 0) if dev == "cuda" else torch.device("cpu")
    D = cfg.grid.static.out_dim
    e = be.neurad_encoding_mean_bwd(FIELD_MAIN, torch.zeros(0, 4, 3, device=dv), torch.zeros(0, 4, device=dv), torch.zeros(0, device=dv),
                                    dfeatures=torch.zeros(0, D, device=dv))
    assert e.shape == (0, 4, 3)
    do, dd = be.isotropic_gaussian_bwd(torch.zeros(0, 5, device=dv), torch.zeros(0, 4, 3, device=dv))
    assert do.shape == (0, 3) and dd.shape == (0, 3)
    n, S = 37, 9
    mean, std, t = BS.make_rays(n, S, 5, trajs, "spread")
    mean, std, t = mean.reshape(n, S, 3).to(dv), std.reshape(n, S).to(dv), t.to(dv)
    g = be.neurad_encoding_mean_bwd(FIELD_MAIN, mean, std, t, dfeatures=torch.zeros(n * S, D, device=dv))
    assert (g == 0).all()
    dens = be.neurad_encoding(FIELD_PROP1, mean, std, t, None, want_features=False, want_density=True)["density"]
    g = be.neurad_encoding_mean_bwd(FIELD_PROP1, mean, std, t, density=dens, ddensity=torch.zeros(n, S, device=dv))
    assert (g == 0).all()


def gaussian_bwd_matches_float64(dev, n, S, seed=7, sky=20000.0):
    """isotropic_gaussian_bwd against float64 sums of the fp32 terms (t_s computed as sample_gaussian does); the last
    edge of every ray is the sky distance (neurad.py:452-455).  Bound per entry: S * 2^-24 * sum |term| * 2."""
    gen = torch.Generator().manual_seed(seed)
    u = torch.sort(torch.rand(n, S + 1, generator=gen), dim=1).values
    edges = 0.5 + u * u * 250.0
    edges[:, -1] = sky
    dmean = torch.randn(n, S, 3, generator=gen)
    dv = torch.device(dev, 0) if dev == "cuda" else torch.device("cpu")
    do, dd = _backend_free(dev).isotropic_gaussian_bwd(edges.to(dv), dmean.to(dv))
    st, en = edges[:, :-1], edges[:, 1:]
    ts = (st + (en - st) / 2.0).double()  # fp32 ops, then exact in float64
    ref_o = dmean.double().sum(1)
    ref_d = (ts[..., None] * dmean.double()).sum(1)
    abs_o = dmean.double().abs().sum(1)
    abs_d = (ts[..., None] * dmean.double()).abs().sum(1)
    worst = 0.0
    for got, ref, ab in ((do, ref_o, abs_o), (dd, ref_d, abs_d)):
        err = (got.cpu().double() - ref).abs()
        tol = 2.0 * (S + 1) * U * ab + 1e-30
        r = err / tol
        assert r.max() <= 1.0, f"isotropic_gaussian_bwd: worst ratio {r.max().item():.3g}"
        worst = max(worst, float(r.max()))
    return worst


def _backend_free(dev):
    """A backend without bound parameters (isotropic_gaussian_bwd needs none)."""
    if dev == "cpu":
        from tests.camopt_fake_backend import CamoptFakeBackend

        return CamoptFakeBackend()
    from neurad_studio_b200.nerfstudio_api import get_backend

    return get_backend(torch.device(dev, 0))


# ------------------------------------------------------------------------------------------------ camera optimizer mirror
def exp_maps_match_closed_forms():
    """exp_map_SO3xR3 / exp_map_SE3 against float64 closed forms: rotations orthonormal, SE3 translation = V rho, and
    the SO3xR3 clamp of the angle at 1e-2 inside the coefficients."""
    from neurad_studio_b200.nerfstudio_api import exp_map_SE3, exp_map_SO3xR3

    gen = torch.Generator().manual_seed(0)
    x = (torch.rand(64, 6, generator=gen, dtype=torch.float64) - 0.5) * 0.4
    x[:4, 3:] *= 1e-3  # below the small-angle switch
    for f in (exp_map_SO3xR3, exp_map_SE3):
        m = f(x)
        r = m[:, :, :3]
        assert torch.allclose(r @ r.transpose(1, 2), torch.eye(3, dtype=x.dtype).expand(64, 3, 3), atol=1e-12 if f is exp_map_SE3 else 1e-7)
        assert torch.allclose(torch.linalg.det(r), torch.ones(64, dtype=x.dtype), atol=1e-7)
    w = x[:, 3:]
    a = w.norm(dim=1)
    k = torch.zeros(64, 3, 3, dtype=x.dtype)
    k[:, 0, 1], k[:, 0, 2], k[:, 1, 2] = -w[:, 2], w[:, 1], -w[:, 0]
    k = k - k.transpose(1, 2)
    big = a >= 1e-2
    rot = torch.matrix_exp(k)
    assert torch.allclose(exp_map_SE3(x)[:, :, :3], rot, atol=1e-12)
    assert torch.allclose(exp_map_SO3xR3(x)[big, :, :3], rot[big], atol=1e-12)
    assert torch.equal(exp_map_SO3xR3(x)[:, :, 3], x[:, :3])
    # SE3 translation: V rho with V = sum_k K^k / (k+1)!
    v = torch.eye(3, dtype=x.dtype).expand(64, 3, 3).clone()
    kk = torch.eye(3, dtype=x.dtype).expand(64, 3, 3).clone()
    fact = 1.0
    for j in range(1, 20):
        kk = kk @ k
        fact *= j + 1
        v = v + kk / fact
    assert torch.allclose(exp_map_SE3(x)[:, :, 3], (v @ x[:, :3, None])[..., 0], atol=1e-12)


# ------------------------------------------------------------------------------------------------ end to end (goldens)
def load_camopt_golden(label, name):
    import ast
    import os

    import numpy as np

    z = np.load(os.path.join(os.path.dirname(__file__), "golden", f"camopt_{label}_{name}"), allow_pickle=False)
    meta = ast.literal_eval(str(z["__meta__"]))
    return meta, {k: torch.from_numpy(z[k]) for k in z.files if k != "__meta__"}


def _optimizer_config(meta):
    from neurad_studio_b200.config import CameraOptimizerConfig, ScaledCameraOptimizerConfig

    if meta["scaled"]:
        return ScaledCameraOptimizerConfig(mode=meta["mode"], weights=(1.0, 1.0, 0.01, 0.01, 0.01, 1.0))
    return CameraOptimizerConfig(mode=meta["mode"])


def _camopt_model(label, name, dev, use_camopt_in_eval=True):
    from neurad_studio_b200.nerfstudio_api import NeuRADModel, RayBundle
    from tests.helpers import cfg_from_meta, load_golden

    cmeta, want = load_camopt_golden(label, name)
    meta, g = load_golden(name)
    cfg = cfg_from_meta(meta)
    model = NeuRADModel(cfg, camera_optimizer=_optimizer_config(cmeta), num_cameras=cmeta["num_cameras"], use_camopt_in_eval=use_camopt_in_eval,
                        non_trainable_camera_indices=torch.tensor(cmeta["non_trainable"]))
    sd = dict(g["param"])
    sd["camera_optimizer.pose_adjustment"] = want["pose_adjustment"]
    if cmeta["scaled"]:
        sd["camera_optimizer.weights"] = want["weights"]
    model.load_reference_state_dict(sd)
    model = model.to(dev).eval()
    r = g["ray"]
    n = cmeta["n_rays"]
    rb = RayBundle(origins=r["origins"][:n].to(dev), directions=r["directions"][:n].to(dev), pixel_area=r["pixel_area"][:n].to(dev),
                   times=r["times"][:n].to(dev), camera_indices=want["camera_indices"].to(dev),
                   metadata={"is_lidar": r["is_lidar"][:n].to(dev), "sensor_idxs": r["sensor_idx"][:n].to(dev)})
    return cmeta, want, model, rb


def module_walk_pose_gradients_match_reference_golden(label, name, dev):
    """loss.backward() through the camera optimizer and the module walk (every stage a hand-written backward operator, the
    new position gradients included) against the reference's autograd: d pose_adjustment and d corrected origins within
    2e-3 of each tensor's scale -- the bar of the parameter gradients (module_seam_cases.check_grads) -- and d corrected
    directions within 1e-2 (see below)."""
    from oracle.make_golden_grads import OUT_KEYS, loss_weights

    cmeta, want, model, rb = _camopt_model(label, name, dev)
    model.camera_optimizer.apply_to_raybundle(rb)
    rb.origins.retain_grad()
    rb.directions.retain_grad()
    assert torch.allclose(rb.origins.detach().cpu(), want["corrected/origins"], rtol=0, atol=1e-5)
    assert torch.allclose(rb.directions.detach().cpu(), want["corrected/directions"], rtol=0, atol=1e-6)
    out = model.get_nff_outputs(rb)  # the bundle requires grad: the module walk
    assert "weights_list" in out
    G = loss_weights({k: out[k].shape for k in OUT_KEYS}, cmeta["loss_seed"])
    sum((out[k] * G[k].to(dev)).sum() for k in OUT_KEYS).backward()
    got = {"pose_adjustment": model.camera_optimizer.pose_adjustment.grad, "origins": rb.origins.grad, "directions": rb.directions.grad}
    # d directions = sum_s t_s dmean_s weights each sample by its distance (up to the 20 km sky sample), and one ray per
    # case carries most of the difference (2 % - 8 % of that ray's own entries).  That is the reference's own conditioning,
    # not an error of the operators: moving every corrected direction by ONE ulp changes the reference's (the oracle's,
    # equal to it bit for bit) d directions by up to 3.9e-2 of its scale (scaled static) and 6.7e-3 (scaled actors, on
    # the same ray 7 that carries our difference there) -- samples change cell on a fine level, and t_s magnifies the
    # jump (reference_direction_gradient_noise_floor).  d origins, which t_s does not weight, moves by <= 5.6e-4 under the
    # same nudge.  Measured here: 5.2e-3 to 7.4e-3 on the host emulation, 6.3e-3 to 9.6e-3 on an H100; this tensor is
    # held to 1e-2, the other two to 2e-3.
    bound = {"pose_adjustment": 2e-3, "origins": 2e-3, "directions": 1e-2}
    worst = {}
    for k, g in got.items():
        ref = want[f"grad/{k}"].double()
        scale = float(ref.abs().max())
        err = float((g.detach().cpu().double() - ref).abs().max()) / scale
        assert err < bound[k], f"{label} {name} d{k}: max |got - ref| / max |ref| = {err:.2e}"
        worst[k] = err
    return worst


def mirror_matches_reference_golden(label, name):
    """Correction matrices, regulariser, state-dict round trip on the reference keys; the non-trainable camera's row of
    the correction matrices is the identity and gets no gradient through them."""
    from neurad_studio_b200.nerfstudio_api import NeuRADModel

    cmeta, want, model, _ = _camopt_model(label, name, "cpu")
    opt = model.camera_optimizer
    assert torch.allclose(opt.get_correction_matrices().detach(), want["correction_matrices"], rtol=0, atol=1e-6)
    losses = {}
    opt.get_loss_dict(losses)
    assert torch.allclose(losses["camera_opt_regularizer"].detach(), want["regularizer"], rtol=1e-6, atol=0)
    sd = model.state_dict()
    keys = {k for k in sd if k.startswith("camera_optimizer.")}
    assert keys == ({"camera_optimizer.pose_adjustment", "camera_optimizer.weights"} if cmeta["scaled"] else {"camera_optimizer.pose_adjustment"})
    assert torch.equal(sd["camera_optimizer.pose_adjustment"], want["pose_adjustment"])
    fresh = NeuRADModel(model.config, camera_optimizer=_optimizer_config(cmeta), num_cameras=cmeta["num_cameras"])
    fresh.load_state_dict(sd)
    assert torch.equal(fresh.camera_optimizer.pose_adjustment.detach(), want["pose_adjustment"])
    missing = {k: v for k, v in sd.items() if k != "camera_optimizer.pose_adjustment"}
    try:
        fresh.load_state_dict(missing, strict=False)
        raise AssertionError("a camera optimizer that is on must require camera_optimizer.pose_adjustment")
    except KeyError:
        pass
    m = opt.get_correction_matrices()
    (m * torch.randn(m.shape, generator=torch.Generator().manual_seed(1))).sum().backward()
    nt = cmeta["non_trainable"][0]
    assert torch.equal(m[nt].detach(), torch.eye(4)[:3, :4])
    assert (opt.pose_adjustment.grad[nt] == 0).all() and (opt.pose_adjustment.grad.abs().sum(1) > 0).sum() == cmeta["num_cameras"] - 1
    metrics, groups = {}, {}
    opt.get_metrics_dict(metrics)
    opt.get_param_groups(groups)
    assert groups["camera_opt"] == [opt.pose_adjustment] and "camera_opt_rotation_max" in metrics


def mode_off_is_unchanged(name):
    """Mode "off": no new parameters or state-dict keys, and the reference's camera_optimizer keys are ignored on load."""
    from neurad_studio_b200.nerfstudio_api import NeuRADModel
    from tests.helpers import cfg_from_meta, load_golden

    meta, g = load_golden(name)
    cfg = cfg_from_meta(meta)
    a, b = NeuRADModel(cfg), NeuRADModel(cfg, num_cameras=5, use_camopt_in_eval=True)
    assert list(a.state_dict()) == list(b.state_dict())
    assert [n for n, _ in a.named_parameters()] == [n for n, _ in b.named_parameters()]
    sd = dict(a.state_dict())
    sd["camera_optimizer.pose_adjustment"] = torch.zeros(5, 6)
    b.load_state_dict(sd, strict=False)
    b.load_reference_state_dict(dict(g["param"], **{"camera_optimizer.pose_adjustment": torch.zeros(5, 6)}))


def camopt_in_eval_renders_the_corrected_bundle(dev, name="nff_static.npz"):
    """use_camopt_in_eval: get_outputs_for_camera_ray_bundle renders (fused) the corrected rays, bit-identical to
    rendering a bundle corrected beforehand; with mode "off" the outputs are bit-identical to a model built without
    the option."""
    from neurad_studio_b200.nerfstudio_api import NeuRADModel

    cmeta, want, model, rb = _camopt_model("so3xr3", name, dev)
    with torch.no_grad():
        got = model.get_outputs_for_camera_ray_bundle(rb)
        pre = rb.flatten()
        model.camera_optimizer.apply_to_raybundle(pre)
        model.use_camopt_in_eval = False
        ref = model.get_outputs_for_camera_ray_bundle(pre)
        plain = model.get_outputs_for_camera_ray_bundle(rb)
    for k in ("features", "depth", "accumulation"):
        assert torch.equal(got[k], ref[k]), k
    assert not torch.equal(got["depth"], plain["depth"])
    base = NeuRADModel(model.config)
    off = NeuRADModel(model.config, num_cameras=3, use_camopt_in_eval=True)
    for m in (base, off):
        m.load_reference_state_dict({k: v for k, v in model.reference_state_dict().items()})
    base, off = base.to(dev).eval(), off.to(dev).eval()
    with torch.no_grad():
        a = base.get_outputs_for_camera_ray_bundle(rb)
        b = off.get_outputs_for_camera_ray_bundle(rb)
    for k in a:
        if torch.is_tensor(a[k]):
            assert torch.equal(a[k], b[k]), k


def reference_direction_gradient_noise_floor(label="scaled", name="nff_static.npz"):
    """Evidence for the d-directions bound above: nudging every corrected direction of the golden case by one ulp moves
    the reference's d directions (torch autograd through the oracle, equal to the golden bit for bit) by more than the
    2e-3 bar, while d origins stays far inside it.  Returns (directions, origins) relative changes."""
    from oracle.make_golden_camopt import load_case, oracle_grads

    meta, params, rays = load_case(name)
    cfg = nsb.small_config(n_actors=meta["n_actors"], log2_main=meta["log2_main"], log2_prop=meta["log2_prop"],
                           static_scale=meta["static_scale"], duration=meta["duration"], num_sensors=meta["num_sensors"])
    _, want = load_camopt_golden(label, name)
    o, d = want["corrected/origins"], want["corrected/directions"]
    go, gd = oracle_grads(cfg, params, rays, o, d)
    for g, k in ((gd, "directions"), (go, "origins")):  # the golden script's own 1e-5 agreement
        assert float((g - want[f"grad/{k}"]).abs().max() / want[f"grad/{k}"].abs().max()) < 1e-5, k
    go1, gd1 = oracle_grads(cfg, params, rays, o, torch.nextafter(d, d + 1.0))
    rd = float((gd1 - gd).abs().max() / gd.abs().max())
    ro = float((go1 - go).abs().max() / go.abs().max())
    assert rd > 2e-3 and ro < 2e-3, (rd, ro)
    return rd, ro
