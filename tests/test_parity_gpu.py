"""GPU parity tests: libb200nerf.so (through the C ABI) vs the reference golden vectors and vs the CPU oracle.

Tolerances (north_star: "within 1e-4 rel fp32, bit-exact for sample indices/counts"):
  * integer work with identical inputs (hash rows, searchsorted indices of the stage operator fed the oracle's own
    weights) is compared bit-exactly;
  * final outputs are compared as  max|a-b| <= 1e-4 * max|ref|  (relative to the tensor's scale);
  * sample indices / actor ids of the fused pipeline are compared EXACTLY on the three reference goldens; only the
    live-oracle cases (fresh random scenes, thousands of rays) keep an agreement rate, because there an index can
    flip when exp/pow differ by an ulp between the CPU's SLEEF and CUDA's libdevice (a flipped index moves a sample
    edge by a few ulp: the inverse cdf is continuous).
  * per-sample traces (sdf / alpha / field_feature) are held to 1e-5 on the samples whose two edges are bit-identical
    to the reference's, and to 2e-3 elsewhere: an edge that differs by one ulp moves the sample by ~1e-7 of the ray
    length, which the finest grid level (8191 cells) turns into a ~1e-4 change of that sample's features -- in the
    reference's own arithmetic too (tests/test_reference_noise_floor.py).
  * `depth` under the raw beta=20 init (d alpha / d sdf = 5) gets 2e-4: the reference's own math evaluated with a
    correctly rounded exp() instead of SLEEF's already sits 0.7e-4 from the golden (same test file).
  "rel" everywhere = max|a-b| / max|ref| (relative to the tensor's scale, not elementwise).
"""
import pytest
import torch

import neurad_studio_b200 as nsb
from neurad_studio_b200 import scene
from neurad_studio_b200.backend import DEFAULT_MODE
from oracle import neurad_oracle as O
from oracle.convert import to_oracle_cfg
from tests.helpers import cfg_from_meta, load_golden

pytestmark = pytest.mark.gpu


def rel_to_max(a, b):
    a, b = a.detach().cpu().float(), b.detach().cpu().float()
    return (a.reshape(b.shape) - b).abs().max().item() / (b.abs().max().item() + 1e-30)


@pytest.fixture(scope="module")
def backend():
    from neurad_studio_b200.backend import B200Backend

    return B200Backend(torch.device("cuda", 0))


def _check_against(out, ref, beta):
    for k in ("inds_1", "inds_2", "actor_id_0", "actor_id_1", "actor_id_main"):
        n_mism = int((out[k].cpu().long() != ref[k].long()).sum())
        assert n_mism == 0, (k, n_mism)  # bit-exact sample indices / actor assignment on the reference goldens
    for k in ("features", "accumulation", "prop_depth_0", "prop_depth_1", "prop_weights_0"):
        assert rel_to_max(out[k], ref[k]) < 1e-4, (k, rel_to_max(out[k], ref[k]))
    assert rel_to_max(out["depth"], ref["depth"]) < (2e-4 if beta >= 20 else 1e-4)
    for k in ("bins_s_1", "bins_s_2"):
        assert (out[k].cpu() - ref[k]).abs().max().item() < 3e-6, k
    # per-sample traces: tight where the sample sits exactly where the reference's does
    edges_equal = out["bins_s_2"].cpu() == ref["bins_s_2"]
    same_sample = edges_equal[:, :-1] & edges_equal[:, 1:]
    assert same_sample.float().mean().item() > 0.005  # a few % on the GPU (CUDA's expf vs SLEEF), ~18 % in the host emulation
    for k in ("sdf", "alpha", "field_feature"):
        a, b = out[k].cpu().float(), ref[k].float()
        a = a.reshape(b.shape)
        scale = b.abs().max().item()
        err = (a - b).abs()
        err = err.reshape(*same_sample.shape, -1).amax(-1)
        assert err[same_sample].max().item() < 1e-5 * scale, (k, err[same_sample].max().item() / scale)
        assert err.max().item() < 2e-3 * scale, (k, err.max().item() / scale)


@pytest.mark.parametrize("mode", ["lane", "split", "tc", "ffma"])
@pytest.mark.parametrize("name", ["nff_static.npz", "nff_actors.npz", "nff_sharp.npz"])
def test_fused_render_matches_reference_golden(backend, name, mode):
    """All kernel variants: ray-per-lane + wgmma (default), warp-per-ray + wgmma, warp-per-ray + CUDA-core fp32."""
    meta, g = load_golden(name)
    cfg = cfg_from_meta(meta)
    p, r, ref = g["param"], g["ray"], g["ref"]
    backend.load_params(cfg, p)
    backend.set_mlp_mode(mode)
    try:
        out = backend.render(r, want_trace=True, want_intensity=True)
        backend.check_status()
    finally:
        backend.set_mlp_mode(DEFAULT_MODE)
    _check_against(out, ref, meta["beta"])
    assert rel_to_max(out["intensity"], ref["intensity"]) < 1e-4
    assert rel_to_max(out["ray_drop_logits"], ref["ray_drop_logits"]) < 1e-4


def _live_case(backend, cfg, n_rays, seed, beta, sdf_bias, table_scale=1.0, n_check=None):
    trajs = scene.make_trajectories(cfg.n_actors, cfg.duration, seed=seed) if cfg.n_actors else None
    params = scene.make_params(cfg, seed=seed, table_scale=table_scale, beta=beta, trajectories=trajs, sdf_bias=sdf_bias)
    rays = scene.random_rays(n_rays, cfg, seed=seed + 1, trajectories=trajs)
    backend.load_params(cfg, params)
    out = backend.render(rays, want_trace=True)
    torch.cuda.synchronize()
    with torch.no_grad():
        ref = O.nff_outputs(params, to_oracle_cfg(cfg), rays["origins"], rays["directions"], rays["pixel_area"],
                            rays["times"], rays["sensor_idx"], rays["is_lidar"], want_trace=True)
    tr = ref.pop("trace")
    ref.update(tr)
    return out, ref


def test_fused_render_vs_oracle_16_actors(backend):
    """Config 3: 16 rigid actors, rays aimed at the boxes.  Fresh random scene vs the live oracle: discrete decisions
    must agree on >= 99.9 % of samples, and the rendered outputs of ALL rays (no agreement mask) must match to 1e-4."""
    cfg = nsb.small_config(n_actors=16, log2_main=16, log2_prop=14)
    out, ref = _live_case(backend, cfg, 2048, seed=21, beta=4.0, sdf_bias=0.5)
    n_hit = int((ref["actor_id_main"] >= 0).sum())
    assert n_hit > 100, n_hit  # the actor branch is really exercised
    for k in ("actor_id_0", "actor_id_1", "actor_id_main"):  # actor assignment: exact
        assert int((out[k].cpu().long() != ref[k].long()).sum()) == 0, k
    for k in ("inds_1", "inds_2"):
        neq = out[k].cpu().long() != ref[k].long()
        assert neq.float().mean().item() <= 1e-3, (k, neq.float().mean().item())
    for k in ("features", "accumulation", "depth", "prop_depth_0", "prop_depth_1"):
        assert rel_to_max(out[k], ref[k]) < 1e-4, (k, rel_to_max(out[k], ref[k]))


def test_fused_render_vs_oracle_default_tables(backend):
    """Config 2 shapes: the reference's default table sizes (main 8 x 2^22 x 4, proposal 6 x 2^20)."""
    cfg = nsb.NeuRADConfig(n_actors=0)
    out, ref = _live_case(backend, cfg, 1024, seed=31, beta=3.0, sdf_bias=0.6)
    for k in ("inds_1", "inds_2"):
        assert (out[k].cpu().long() != ref[k].long()).float().mean().item() <= 1e-3, k
    for k in ("features", "accumulation", "depth", "prop_depth_0", "prop_depth_1"):
        assert rel_to_max(out[k], ref[k]) < 1e-4, (k, rel_to_max(out[k], ref[k]))


def test_density_field_of_round_is_the_reference_quirk(backend):
    """Both rounds must evaluate proposal_fields[1] (late-binding closures, neurad.py:248); binding round 0 to
    proposal_fields[0] must NOT reproduce the golden weights."""
    from neurad_studio_b200.lib import FIELD_PROP0, FIELD_PROP1

    meta, g = load_golden("nff_static.npz")
    cfg = cfg_from_meta(meta)
    backend.load_params(cfg, g["param"], density_field_of_round=(FIELD_PROP0, FIELD_PROP1))
    out = backend.render(g["ray"], want_trace=True)
    assert rel_to_max(out["prop_weights_0"], g["ref"]["prop_weights_0"]) > 1e-2
    backend.load_params(cfg, g["param"])
    out = backend.render(g["ray"], want_trace=True)
    assert rel_to_max(out["prop_weights_0"], g["ref"]["prop_weights_0"]) < 1e-4


# ----------------------------------------------------------------------------------------------- stage operators
def test_hashgrid_rows_bit_exact_and_values(backend):
    meta, g = load_golden("nff_static.npz")
    cfg = cfg_from_meta(meta)
    p, ref = g["param"], g["ref"]
    gs = cfg.grid.static
    out, idx = backend.hashgrid_fwd(gs, p["field.hashgrid.static_grid.hash_table"], ref["hash_in"],
                                    p["field.hashgrid.static_grid.scalings"], want_indices=True)
    oidx, _ = O.hash_indices(ref["hash_in"], p["field.hashgrid.static_grid.scalings"], gs.hash_table_size)
    assert torch.equal(idx.cpu().long(), oidx)  # bit-exact integer work
    assert torch.equal(out.cpu(), ref["hash_out"])  # same single-rounding op sequence -> bit-exact values too


@pytest.mark.parametrize("L,F,log2T", [(16, 2, 19), (6, 1, 20), (8, 4, 22), (4, 8, 12)])
def test_hashgrid_generic_shapes_vs_oracle(backend, L, F, log2T):
    """HashEncoding defaults (16 levels x 2, encodings.py:326-337) and NeuRAD's grids at full table size, at a
    point count the oracle finishes in seconds; includes exact-integer coordinates (ceil == floor) and 0 / 1."""
    g = nsb.HashGridSettings(F, L, 16, 2048, log2T)
    gen = torch.Generator().manual_seed(L * 100 + F)
    table = torch.rand(g.hash_table_size * L, F, generator=gen) * 2 - 1
    x = torch.rand(20000, 3, generator=gen)
    x[:64] = torch.randint(0, 17, (64, 3), generator=gen).float() / 16.0  # lattice points incl. 0 and 1
    out, idx = backend.hashgrid_fwd(g, table, x, want_indices=True)
    oidx, _ = O.hash_indices(x, g.scalings(), g.hash_table_size)
    assert torch.equal(idx.cpu().long(), oidx)
    ref = O.hash_encode(x, table, g.scalings(), g.hash_table_size)
    assert torch.equal(out.cpu(), ref)


def test_hashgrid_empty_input(backend):
    g = nsb.HashGridSettings(2, 4, 16, 128, 10)
    out = backend.hashgrid_fwd(g, torch.zeros(g.hash_table_size * 4, 2), torch.zeros(0, 3))
    assert out.shape == (0, 8)


def test_pdf_resample_indices_bit_exact(backend):
    """Fed the oracle's own weights and bins, the searchsorted indices must be identical wherever the cdf the
    kernel builds equals the oracle's bit for bit, and the new bins must agree to 1e-6."""
    meta, g = load_golden("nff_static.npz")
    ref = g["ref"]
    for w, b, s_new, inds, cdf, nb in (
        (ref["prop_weights_0"], ref["bins_s_0"], 64, ref["inds_1"], ref["cdf_1"], ref["bins_s_1"]),
        (ref["prop_weights_1"], ref["bins_s_1"], 32, ref["inds_2"], ref["cdf_2"], ref["bins_s_2"]),
    ):
        new_bins, cdf_k, inds_k = backend.pdf_resample(w, b.expand(w.shape[0], -1).contiguous(), s_new)
        assert (cdf_k.cpu() - cdf).abs().max().item() < 5e-7
        # searchsorted on the kernel's own cdf, evaluated by torch: must be bit-identical (pure integer result)
        u = O.pdf_u(s_new).expand(w.shape[0], -1).contiguous()
        assert torch.equal(inds_k.cpu().long(), torch.searchsorted(cdf_k.cpu(), u, side="right"))
        assert (inds_k.cpu().long() != inds).float().mean().item() < 2e-3
        assert (new_bins.cpu() - nb).abs().max().item() < 2e-6


def test_pdf_resample_degenerate_rays(backend):
    """All-zero weights (uniform pdf after padding), a single spike, and inf/NaN-free outputs."""
    n, s = 4, 128
    w = torch.zeros(n, s)
    w[1, 5] = 1.0
    w[2, -1] = 1e-12
    w[3] = 1e30
    b = torch.linspace(0, 1, s + 1).expand(n, -1).contiguous()
    nb, cdf, inds = backend.pdf_resample(w, b, 64)
    r = O.pdf_resample(w, b, 64)
    assert torch.isfinite(nb).all()
    assert (nb.cpu() - r["bins"]).abs().max().item() < 1e-5
    assert (nb.cpu()[:, 1:] >= nb.cpu()[:, :-1]).all()


def test_weights_from_density_and_alpha(backend):
    gen = torch.Generator().manual_seed(5)
    for s in (32, 64, 128, 48):
        deltas = torch.rand(300, s, generator=gen) * 2
        dens = torch.exp(torch.randn(300, s, generator=gen) * 2)
        dens[0, 3] = float("inf")
        w = backend.density_to_weights(deltas, dens).cpu()
        ref = O.weights_from_density(deltas, dens)
        assert (w - ref).abs().max().item() < 2e-6
        al = torch.rand(300, s, generator=gen)
        w = backend.alpha_to_weights(al).cpu()
        assert (w - O.render_weight_from_alpha(al)).abs().max().item() < 2e-6


def test_sh4(backend):
    d = torch.rand(1000, 3)
    assert (backend.sh4_fwd(d).cpu() - O.sh_components_l4(d)).abs().max().item() < 2e-6


def test_raygen_matches_reference_golden(backend):
    meta, g = load_golden("raygen.npz")
    for i, cam in ((0, "cam0"), (3, "cam3")):
        c = g[cam]
        h, w = (int(v) for v in c["hw"])
        fx, fy, cx, cy = (float(v) for v in c["intr"])
        pc = scene.PinholeCamera(c2w=c["c2w"], fx=fx, fy=fy, cx=cx, cy=cy, width=w, height=h, time=float(c["time"]),
                                 velocity=c["velocity"], rolling_shutter_time=float(c["rs"][0]),
                                 time_to_center_pixel=float(c["rs"][1]))
        r = backend.raygen_pinhole(pc)
        for k in ("origins", "directions", "pixel_area", "times"):
            a, b = r[k].cpu().reshape(-1), c[k].reshape(-1)
            err, tol = (a - b).abs().max().item(), 1e-6 * max(1.0, b.abs().max().item())
            assert err <= tol, (cam, k, err, tol)
        # the strided grid NeuRAD actually renders ([1::3, 1::3], neurad.py:641-646)
        r3 = backend.raygen_pinhole(pc, row0=1, row_step=3, col0=1, col_step=3)
        full = c["directions"][1::3, 1::3].reshape(-1, 3)
        e3 = (r3["directions"].cpu() - full).abs().max().item()
        assert e3 <= 1e-6, (cam, "strided directions", e3)
        full_a = c["pixel_area"][1::3, 1::3].reshape(-1)
        ea = (r3["pixel_area"].cpu().reshape(-1) - full_a).abs().max().item()
        assert ea <= 1e-4 * full_a.max().item(), (cam, "strided pixel_area", ea, full_a.max().item())
    li = g["lidar"]
    scan = scene.LidarScan(l2w=li["l2w"], points=li["points"], time=float(li["time"]), velocity=li["velocity"])
    r = backend.raygen_lidar_points(scan)
    for k in ("origins", "directions", "pixel_area", "times"):
        a, b = r[k].cpu().reshape(-1), li[k].reshape(-1)
        err, tol = (a - b).abs().max().item(), 1e-6 * max(1.0, b.abs().max().item())
        assert err <= tol, ("lidar", k, err, tol)
    ed = (r["directions_norm"].cpu().reshape(-1) - li["distance"].reshape(-1)).abs().max().item()
    assert ed < 1e-4, ("lidar distance", ed)


# ------------------------------------------------------------------------------- size-independent properties
def test_full_size_properties(backend):
    """BASELINE config-2 scale (one 1920x1080 camera at the render stride = 230 400 rays + lidar), default tables:
    weights partition unity, bins are sorted, results are deterministic and independent of batch composition."""
    cfg = nsb.NeuRADConfig(n_actors=0)
    params = scene.make_params(cfg, seed=41, beta=3.0, sdf_bias=0.6, device="cuda")
    backend.load_params(cfg, params)
    cam = scene.pandaset_rig()[0]
    rays = backend.raygen_pinhole(cam, row0=1, row_step=3, col0=1, col_step=3)
    n = rays["origins"].shape[0]
    assert n == 640 * 360
    rays["sensor_idx"] = torch.zeros(n, 1, dtype=torch.long, device="cuda")
    out = backend.render(rays, want_trace=True)
    out2 = backend.render(rays)
    backend.check_status()
    for k in ("features", "depth", "accumulation", "prop_depth_0", "prop_depth_1"):
        assert torch.isfinite(out[k]).all(), k
        assert torch.equal(out[k], out2[k]), k  # deterministic
    w = out["weights"]
    assert (w >= -1e-6).all()
    assert (w.sum(-1) - 1.0).abs().max().item() < 1e-5  # sky top-up makes the weights partition unity
    assert (out["accumulation"] <= 1.0 + 1e-5).all() and (out["accumulation"] >= 0).all()
    for k in ("bins_s_1", "bins_s_2", "bins_e_1", "bins_e_2"):
        b = out[k]
        assert (b[:, 1:] >= b[:, :-1]).all(), k
    assert (out["inds_1"] >= 1).all() and (out["inds_1"] <= 129).all()
    # batch-composition independence: a sub-range rendered alone equals the slice of the full render
    # (1003 rays: not a multiple of the 8 rays a CTA renders at a time -> exercises the inactive-warp path)
    sub = {k: (v[1000:2003] if isinstance(v, torch.Tensor) else v) for k, v in rays.items() if k != "shape"}
    o3 = backend.render(sub)
    backend.check_status()
    assert torch.equal(o3["features"], out["features"][1000:2003])
    assert torch.equal(o3["depth"], out["depth"][1000:2003])
    # the 2-D tile walk (image_width hint) must not change any result: same rays, same per-ray arithmetic
    o5 = backend.render(rays, image_width=640)
    backend.check_status()
    for k in ("features", "depth", "accumulation", "prop_depth_0", "prop_depth_1"):
        assert torch.equal(o5[k], out[k]), k
    o6 = backend.render(sub, image_width=77)  # ragged: 1003 rays = 13 rows of 77 + 2
    for k in ("features", "depth"):
        assert torch.equal(o6[k], o3[k]), k
    # two-kernel variant (sampling | shading) runs the same arithmetic: identical results, also when the bundle is
    # sliced because it exceeds the 2^21-ray hand-over buffer (with and without the tile walk)
    backend.set_mlp_mode("split")
    try:
        o7 = backend.render(rays, image_width=640)
        big = {k: torch.cat([v] * 10) for k, v in rays.items() if isinstance(v, torch.Tensor)}
        o8 = backend.render(big)
        o9 = backend.render(big, image_width=640)
        backend.check_status()
    finally:
        backend.set_mlp_mode(DEFAULT_MODE)
    n0 = out["depth"].shape[0]
    assert big["origins"].shape[0] > (1 << 21)
    for k in ("features", "depth", "accumulation", "prop_depth_0", "prop_depth_1"):
        assert torch.equal(o7[k], out[k]), k
        for o in (o8, o9):
            for rep in (0, 8, 9):  # first slice, the copy straddling the slice boundary, last slice
                assert torch.equal(o[k][rep * n0 : (rep + 1) * n0], out[k]), (k, rep)
    backend.set_mlp_mode("lane")  # the single-kernel variant of the same code
    try:
        o10 = backend.render(rays, image_width=640)
    finally:
        backend.set_mlp_mode(DEFAULT_MODE)
    for k in ("features", "depth", "accumulation", "prop_depth_0", "prop_depth_1"):
        assert torch.equal(o10[k], out[k]), k
    # the kernel variants agree to fp32 level on the whole image
    for mode in ("ffma", "tc"):
        backend.set_mlp_mode(mode)
        o4 = backend.render(rays)
        backend.set_mlp_mode(DEFAULT_MODE)
        assert rel_to_max(o4["features"], out["features"]) < 1e-4, mode
        assert rel_to_max(o4["depth"], out["depth"]) < 1e-4, mode


def test_errors_are_loud(backend):
    from neurad_studio_b200.backend import B200Backend
    from neurad_studio_b200.lib import B200NerfError

    fresh = B200Backend(torch.device("cuda", 0))
    fresh.cfg = nsb.small_config()
    rays = scene.random_rays(8, fresh.cfg)
    with pytest.raises(B200NerfError):
        fresh.render(rays)  # no parameters bound
    bad = nsb.small_config()
    bad.grid.static.num_levels = 5
    with pytest.raises(B200NerfError):
        fresh.load_params(bad, scene.make_params(bad))
    # zero rays is a no-op, not an error
    cfg = nsb.small_config()
    fresh.load_params(cfg, scene.make_params(cfg))
    empty = {k: v[:0] for k, v in rays.items()}
    assert fresh.render(empty)["features"].shape[0] == 0


# ---------------------------------------------------------------------------------------- tensor-core MLP (wgmma)
@pytest.mark.parametrize("dims", [(32, 32, 33), (48, 32, 32, 32), (48, 32, 32, 2), (32, 32), (40, 24, 17), (32, 64, 4), (64, 64, 64, 64), (50, 57, 3)])
@pytest.mark.parametrize("n_rows", [1000, 128 * 300 + 5])
def test_mlp_fwd_tensor_core_vs_fp32(backend, dims, n_rows):
    """MLP.forward on wgmma with the 3xTF32 split vs a plain fp32 (float64-accumulated) reference of the same op:
    NeuRAD's three MLP shapes (mlp_geo 32-32-33, mlp_feature 48-32-32-32, lidar_decoder 48-32-32-2) on the 48-column
    tile; BASELINE config 1's 32-64-4 and other <= 64-wide shapes on the 64-column tile."""
    gen = torch.Generator().manual_seed(sum(dims) + n_rows)
    x = torch.randn(n_rows, dims[0], generator=gen)
    ws, bs = [], []
    for i in range(len(dims) - 1):
        bound = 1.0 / dims[i] ** 0.5
        ws.append((torch.rand(dims[i + 1], dims[i], generator=gen) * 2 - 1) * bound * 3)
        bs.append((torch.rand(dims[i + 1], generator=gen) * 2 - 1) * bound)
    y = backend.mlp_fwd(x, ws, bs)
    backend.check_status()
    h = x.double()
    for i, (w, b) in enumerate(zip(ws, bs)):
        h = h @ w.double().T + b.double()
        if i < len(ws) - 1:
            h = torch.relu(h)
    err = rel_to_max(y, h.float())
    assert err < 5e-6, err  # fp32-level (plain TF32 would be ~5e-4)
    # and against the oracle's torch fp32 MLP
    p = {}
    for i, (w, b) in enumerate(zip(ws, bs)):
        p[f"m.layers.{i}.weight"], p[f"m.layers.{i}.bias"] = w, b
    assert rel_to_max(y, O.mlp_forward(p, "m", len(ws), x)) < 5e-6
    # the training forward (b200nerf_mlp_fwd_train): the same output bit for bit, plus the hidden pre-activations
    y2, zs = backend.mlp_fwd(x, ws, bs, want_hidden=True)
    backend.check_status()
    assert torch.equal(y2, y) and len(zs) == len(ws) - 1
    h = x.double()
    for i, z in enumerate(zs):
        pre = h @ ws[i].double().T + bs[i].double()
        assert z.shape == (n_rows, dims[i + 1]) and rel_to_max(z, pre.float()) < 5e-6, i
        h = torch.relu(pre)
    # the input gradient of the last layer through the same operator (b200nerf_mlp_dgrad), with and without the ReLU mask
    dy = torch.randn(n_rows, dims[-1], generator=gen)
    want = dy.double() @ ws[-1].double()
    dx = backend.mlp_dgrad(dy, ws[-1])
    assert rel_to_max(dx, want.float()) < 5e-6
    if zs:
        dxm = backend.mlp_dgrad(dy, ws[-1], zs[-1])
        backend.check_status()
        assert torch.equal(dxm, torch.where(zs[-1] > 0, dx, torch.zeros_like(dx)))


def test_mlp_fwd_no_bias_and_empty(backend):
    w = torch.randn(1, 6) * 0.4  # NeuRADProposalField.density_decoder = Linear(6, 1, bias=False)
    x = torch.randn(777, 6)
    y = backend.mlp_fwd(x, [w], None)
    backend.check_status()
    assert rel_to_max(y, x @ w.T) < 2e-6
    assert backend.mlp_fwd(torch.zeros(0, 6), [w], None).shape == (0, 1)


# ------------------------------------------------------------------------------- reference-API mirror (plugin level)
@pytest.mark.parametrize("name", ["nff_static.npz", "nff_actors.npz"])
def test_neurad_model_api_matches_reference_golden(name):
    """The module-level drop-in: NeuRADModel with the reference's state_dict keys, RayBundle in, dict out."""
    from neurad_studio_b200.nerfstudio_api import NeuRADModel, RayBundle

    meta, g = load_golden(name)
    cfg = cfg_from_meta(meta)
    p, r, ref = g["param"], g["ray"], g["ref"]
    model = NeuRADModel(cfg)
    model.load_reference_state_dict(p)
    model = model.cuda().eval()
    rb = RayBundle(origins=r["origins"].cuda(), directions=r["directions"].cuda(), pixel_area=r["pixel_area"].cuda(),
                   times=r["times"].cuda(), metadata={"is_lidar": r["is_lidar"].cuda(), "sensor_idxs": r["sensor_idx"].cuda()})
    out = model.get_nff_outputs(rb)
    for k in ("features", "accumulation", "depth", "prop_depth_0", "prop_depth_1"):
        assert rel_to_max(out[k], ref[k]) < 1e-4, k
    inten, drop = model.decode_features(out["features"])
    assert rel_to_max(inten, ref["intensity"]) < 1e-4 and rel_to_max(drop, ref["ray_drop_logits"]) < 1e-4
    lid = model.get_outputs_for_camera_ray_bundle(rb)  # 1-D bundle = lidar convention (neurad.py:636-638)
    assert lid["intensity"].shape == (rb.shape[0], 1) and rel_to_max(lid["intensity"], ref["intensity"]) < 1e-4


def test_module_mirrors_hashencoding_mlp_sh():
    """HashEncoding / MLP / SHEncoding modules: same constructor arguments and parameter names as the reference's
    (test_encodings.py:142-168 only shape-checks them; here values are checked against the oracle)."""
    from neurad_studio_b200.nerfstudio_api import MLP, HashEncoding, SHEncoding

    enc = HashEncoding(num_levels=4, min_res=16, max_res=128, log2_hashmap_size=10, features_per_level=2, hash_init_scale=1.0).cuda()
    assert enc.get_out_dim() == 8 and set(dict(enc.named_parameters())) == {"hash_table"}
    x = torch.rand(33, 5, 3, device="cuda")
    y = enc(x)
    assert y.shape == (33, 5, 8)
    ref = O.hash_encode(x.cpu().reshape(-1, 3), enc.hash_table.detach().cpu(), enc.scalings.cpu(), 2**10)
    assert torch.equal(y.cpu().reshape(-1, 8), ref)
    mlp = MLP(in_dim=48, num_layers=3, layer_width=32, out_dim=2).cuda()
    assert [n for n, _ in mlp.named_parameters()][:2] == ["layers.0.weight", "layers.0.bias"]
    xin = torch.randn(500, 48, device="cuda")
    want = xin
    for i, l in enumerate(mlp.layers):
        want = torch.nn.functional.linear(want.double(), l.weight.double(), l.bias.double())
        want = torch.relu(want) if i < 2 else want
    assert rel_to_max(mlp(xin), want.float()) < 5e-6
    sh = SHEncoding(levels=4)
    d = torch.rand(10, 3, device="cuda")
    assert (sh(d).cpu() - O.sh_components_l4(d.cpu())).abs().max().item() < 2e-6


def test_config4_lidar_grid_rolling_shutter(backend):
    """BASELINE config 4: 128 beams x 2048 azimuths with a rolling-shutter sweep -> 262 144 rays through the
    volumetric path; ray generation vs the oracle, render vs the oracle on a strided subsample, intensity in (0,1)."""
    l2w = torch.zeros(3, 4)
    l2w[:, :3] = torch.eye(3)
    l2w[:, 3] = torch.tensor([3.0, -1.0, 2.0])
    vel = torch.tensor([10.0, 0.5, 0.0])
    rays = backend.raygen_lidar_grid(l2w, -25.0, 15.0, 128, 360.0 / 2048, scan_time=3.2, velocity=vel)
    assert rays.pop("shape") == (128, 2048)
    ref = O.generate_rays_lidar_grid_rs(l2w, -25.0, 15.0, 128, 360.0 / 2048, 3.2, velocity=vel)
    for k in ("origins", "directions", "pixel_area", "times"):
        assert (rays[k].cpu().reshape(ref[k].shape) - ref[k]).abs().max().item() < 2e-6, k
    cfg = nsb.small_config(n_actors=0, log2_main=16, log2_prop=14)
    params = scene.make_params(cfg, seed=51, beta=3.0, sdf_bias=0.6)
    backend.load_params(cfg, params)
    n = rays["origins"].shape[0]
    rays["sensor_idx"] = torch.full((n, 1), 6, dtype=torch.long, device="cuda")
    rays["is_lidar"] = torch.ones(n, 1, dtype=torch.uint8, device="cuda")
    out = backend.render(rays, want_intensity=True, image_width=2048)
    backend.check_status()
    assert torch.isfinite(out["features"]).all() and ((out["intensity"] > 0) & (out["intensity"] < 1)).all()
    sel = torch.arange(0, n, 257)
    with torch.no_grad():
        o = O.nff_outputs(params, to_oracle_cfg(cfg), ref["origins"][sel], ref["directions"][sel], ref["pixel_area"][sel],
                          ref["times"][sel], torch.full((sel.numel(), 1), 6), torch.ones(sel.numel(), 1, dtype=torch.bool))
        inten, _ = O.decode_lidar(params, o["features"])
    for k in ("features", "depth", "accumulation"):
        assert rel_to_max(out[k][sel.cuda()], o[k]) < 1e-4, (k, rel_to_max(out[k][sel.cuda()], o[k]))
    assert rel_to_max(out["intensity"][sel.cuda()], inten) < 1e-4


def test_peer_outputs_stream_to_pinned_host_memory(backend):
    """set_peer_outputs with a pinned (device-mapped) host buffer as the only "peer": the render epilogue writes every
    finished row to the host while rendering; the host copy must equal the device output bit for bit, for a ray count
    that is not a multiple of the 8-ray output segments or of the 512-ray CTA, with and without the 2-D tile walk."""
    cfg = nsb.small_config(n_actors=0, log2_main=14, log2_prop=13)
    params = scene.make_params(cfg, seed=61, beta=3.0, sdf_bias=0.6)
    backend.load_params(cfg, params)
    n = 3001
    rays = scene.random_rays(n, cfg, seed=62)
    for width in (0, 77):
        host = {"features": torch.zeros(n, cfg.feature_dim).pin_memory(), "depth": torch.zeros(n, 1).pin_memory(),
                "accumulation": torch.zeros(n, 1).pin_memory()}
        backend.set_peer_outputs({k: [v.data_ptr()] for k, v in host.items()}, self_rank=-1, row_offset=0)
        try:
            out = backend.render(rays, image_width=width)
            torch.cuda.synchronize()
            backend.check_status()
        finally:
            backend.set_peer_outputs(None)
        for k, v in host.items():
            assert torch.equal(v, out[k].cpu()), (k, width)


# ------------------------------------------------------------------- BASELINE config 1 + generic sampler / renderers
def test_config1_matches_reference_golden(backend):
    """BASELINE config 1 through the reference-API mirror, stage by stage and end to end, against the outputs of
    the real reference (tests/golden/config1.npz): Cameras -> UniformSampler(32) -> normalised positions ->
    HashEncoding(16x2, 2^19) -> MLP 32->64->4 -> trunc_exp / sigmoid -> get_weights -> RGB / depth / accumulation."""
    from neurad_studio_b200.nerfstudio_api import (MLP, AccumulationRenderer, DepthRenderer, HashEncoding, RayBundle, RGBRenderer,
                                                   UniformSampler)
    from tests.helpers import load_config1

    meta, p, r, ref = load_config1()
    cam = scene.PinholeCamera(c2w=torch.eye(4)[:3], fx=64.0, fy=64.0, cx=32.0, cy=32.0, width=64, height=64, time=0.0,
                              velocity=None, rolling_shutter_time=0.0, time_to_center_pixel=0.0)
    rays = backend.raygen_pinhole(cam)
    assert (rays["origins"].cpu() - r["origins"]).abs().max().item() == 0.0
    assert (rays["directions"].cpu() - r["directions"]).abs().max().item() < 2e-7
    rb = RayBundle(origins=rays["origins"], directions=rays["directions"], pixel_area=rays["pixel_area"],
                   nears=r["nears"].cuda(), fars=r["fars"].cuda())
    enc = HashEncoding(num_levels=16, min_res=16, max_res=1024, log2_hashmap_size=meta["log2_hashmap_size"], features_per_level=2)
    assert torch.equal(enc.scalings, p["scalings"])
    enc.hash_table.data = p["hash_table"]
    mlp = MLP(in_dim=32, num_layers=2, layer_width=64, out_dim=4)
    mlp.load_state_dict({"layers.0.weight": p["w0"], "layers.0.bias": p["b0"], "layers.1.weight": p["w1"], "layers.1.bias": p["b1"]})
    enc, mlp = enc.cuda(), mlp.cuda()
    rs = UniformSampler(num_samples=32)(rb)
    assert (rs.frustums.bin_edges.cpu() - ref["bins_e"]).abs().max().item() < 1e-6
    assert torch.equal(rs.spacing_bins.cpu(), torch.linspace(0.0, 1.0, 33))
    pos = rs.frustums.get_positions(normalize_aabb=p["aabb"])
    assert (pos[::8].cpu() - ref["positions_sub"]).abs().max().item() < 1e-6
    feat = enc(pos.view(-1, 3))
    assert rel_to_max(feat.view(4096, 32, 32)[::8], ref["encoding_sub"]) < 1e-4
    raw = mlp(feat).view(4096, 32, 4)
    backend.check_status()
    assert rel_to_max(raw[::8], ref["raw_sub"]) < 1e-4
    density, rgb_s = backend.density_rgb_heads(raw)
    assert rel_to_max(density[::8], ref["density_sub"]) < 1e-4 and rel_to_max(rgb_s[::8], ref["rgb_samples_sub"]) < 1e-4
    w = rs.get_weights(density)
    assert rel_to_max(w[::8], ref["weights_sub"]) < 1e-4
    out = {"rgb": RGBRenderer("black")(rgb_s, w), "depth": DepthRenderer("expected")(w, rs),
           "depth_median": DepthRenderer("median")(w, rs), "accumulation": AccumulationRenderer()(w)}
    for k, v in out.items():
        assert v.shape == ref[k].shape, k
        assert rel_to_max(v, ref[k]) < 1e-4, (k, rel_to_max(v, ref[k]))
    # the median picks a sample index: it has to be the reference's index for every ray
    assert torch.equal(out["depth_median"].cpu(), ref["depth_median"]) or rel_to_max(out["depth_median"], ref["depth_median"]) < 1e-6


@pytest.mark.parametrize("spacing,kind", [("uniform", 0), ("lindisp", 1), ("power", 2), ("sqrt", 3), ("log", 4)])
def test_spaced_samplers_match_oracle(backend, spacing, kind):
    from oracle import simple_oracle as S

    gen = torch.Generator().manual_seed(kind)
    n = 1000
    nears = torch.rand(n, 1, generator=gen) * 2 + 0.05
    fars = nears + torch.rand(n, 1, generator=gen) * 100 + 1.0
    for s in (1, 32, 48, 128):
        bs_ref, be_ref = S.spaced_sample(nears, fars, s, kind, -1.0, 0.1)
        bs, be = backend.spaced_sample(nears, fars, s, spacing, -1.0, 0.1)
        # torch's CPU linspace evaluates `base + step * lane` per SIMD vector, so for step sizes that are not exact in
        # fp32 (S not a power of two) its last bit depends on the host's vector width; NeuRAD's S (128/64/32) and
        # config 1's (32) are exact
        pow2 = s & (s - 1) == 0
        assert torch.equal(bs.cpu(), bs_ref[0]) if pow2 else (bs.cpu() - bs_ref[0]).abs().max().item() < 2e-7
        assert rel_to_max(be, be_ref) < (1e-6 if kind < 4 else 1e-5), (spacing, s)
        if kind in (0, 1) and pow2:  # only IEEE +,-,*,/: bit-exact
            assert torch.equal(be.cpu(), be_ref)
    lam_ref = S.spaced_sample(nears, fars, 16, S.SPACING_POWER, -1.7, 0.25)[1]
    assert rel_to_max(backend.spaced_sample(nears, fars, 16, "power", -1.7, 0.25)[1], lam_ref) < 1e-5
    assert backend.spaced_sample(None, fars, 4)[1][:, 0].abs().max().item() == 0.0  # nears default to 0
    assert backend.spaced_sample(nears[:0], fars[:0], 4)[1].shape == (0, 5)


@pytest.mark.parametrize("n_samples,n_channels", [(32, 3), (40, 48), (7, 1), (100, 9), (3, 64), (31, 32), (33, 33), (64, 7),
                                                   (129, 8)])
def test_composite_matches_oracle(backend, n_samples, n_channels):
    """The composite operator against the oracle's renderers.  The operator never clamps (FeatureRenderer shares it), so
    its values are compared with RGBRenderer's unclamped training-mode path on nan_to_num'd colours; the median must pick
    the reference's sample on every ray."""
    from oracle import simple_oracle as S
    from tests import stage_ops_cases as C

    gen = torch.Generator().manual_seed(n_samples * 100 + n_channels)
    n = 777
    dens = torch.rand(n, n_samples, generator=gen) * 3
    edges = torch.cumsum(torch.rand(n, n_samples + 1, generator=gen) * 0.3 + 0.01, -1)
    starts, ends = edges[:, :-1, None], edges[:, 1:, None]
    w = O.weights_from_density((ends - starts)[..., 0], dens)[..., None]
    w = torch.floor(w * 2.0 ** 24) / 2.0 ** 24  # on the 2^-24 grid: the median's float64 running sums are exact
    vals = torch.randn(n, n_samples, n_channels, generator=gen)
    vals[3, 2, 0] = float("nan")
    vals[5, 1, -1] = float("inf")
    bg = [0.25 * (i % 4) for i in range(n_channels)]
    ref_rgb = S.rgb_render(torch.nan_to_num(vals), w, torch.tensor(bg), training=True)  # the operator does not clamp
    out = backend.composite(w, vals, starts, ends, "expected", background=bg, value_nan_to_num=True)
    assert rel_to_max(out["values"], ref_rgb) < 1e-5
    assert rel_to_max(out["accumulation"], w.sum(-2)) < 1e-6
    assert rel_to_max(out["depth"], S.depth_expected(w, starts, ends)) < 1e-5
    good = torch.nan_to_num(vals)
    feat = backend.composite(w, good, want_accumulation=False)
    assert set(feat) == {"values"} and rel_to_max(feat["values"], (w * good).sum(-2)) < 1e-5
    med = backend.composite(w, None, starts, ends, "median", want_accumulation=False)["depth"]
    ref_med = S.depth_median(w, starts, ends)
    # exactly the reference's sample: torch's CPU cumsum runs in float64 and rounds each running sum to fp32
    assert torch.equal(med.cpu(), ref_med)
    assert torch.equal(med.cpu()[:, 0], ((starts + ends) / 2)[..., 0].gather(1, C.median_index(w[..., 0])[:, None])[:, 0])
    simple = backend.composite(w, None, starts, ends, "simple")["depth"]
    assert rel_to_max(simple, (w * (starts + ends) / 2).sum(-2)) < 1e-5
    # the "expected" clip is global over the batch: one heavy ray in a second call must not leak into the first
    lo = backend.composite(w[:5], None, starts[:5] * 0 + 1.0, ends[:5] * 0 + 1.0, "expected")["depth"]
    assert (lo - 1.0).abs().max().item() < 1e-6
    assert backend.composite(w[:0], vals[:0])["values"].shape == (0, n_channels)


# ------------------------------------------------------------------------------- camera rgb decoder (SURVEY 8f, f1)
def _decoder_golden():
    meta, g = load_golden("rgb_decoder.npz")
    return g["param"], g["in"]["features"], g["ref"]["rgb"]


@pytest.mark.parametrize("impl", ["ref", "tc", "tc_ldgsts"])
def test_rgb_decoder_matches_reference_golden(backend, impl):
    """NeuRADModel.rgb_decoder (1x1 conv, 4 BasicBlocks with BatchNorm, 3x transposed conv, 1x1 conv + sigmoid) on the
    reference's own output for a 2 x 19 x 45 feature image: CUDA-core fp32 pipeline and wgmma (bf16 hi/lo split)
    pipeline, both within the 1e-4 parity bar."""
    p, feats, ref = _decoder_golden()
    backend.set_rgb_decoder(p)
    rgb = backend.rgb_decode(feats, impl)
    backend.check_status()
    assert rgb.shape == ref.shape == (2, 57, 135, 3)
    err = (rgb.cpu() - ref).abs().max().item()
    assert err < 1e-4, (impl, err)  # rgb is in (0,1): absolute == relative to the output range
    assert rel_to_max(rgb, ref) < 1e-4


def test_rgb_decoder_tensor_core_multi_tile(backend):
    """Several strips / row tiles / images, ragged edges (width 300 -> 900 = 7 x 128 + 4, heights not multiples of 3):
    wgmma path vs the CPU oracle and vs the in-library CUDA-core path."""
    from oracle import decoder_oracle as D

    p = D.random_decoder_params(seed=21)
    gen = torch.Generator().manual_seed(22)
    feats = torch.randn(2, 13, 300, 48, generator=gen) * 0.7
    backend.set_rgb_decoder(p)
    tc = backend.rgb_decode(feats, "tc")
    backend.check_status()
    ref_k = backend.rgb_decode(feats, "ref")
    with torch.no_grad():
        ref = D.rgb_decoder(p, feats)
    assert tc.shape == ref.shape == (2, 39, 900, 3)
    assert (ref_k.cpu() - ref).abs().max().item() < 1e-4
    assert (tc.cpu() - ref).abs().max().item() < 1e-4
    assert torch.equal(tc, backend.rgb_decode(feats, "tc"))  # deterministic
    backend.check_status()
    assert torch.equal(tc, backend.rgb_decode(feats, "tc_ldgsts"))  # TMA and per-thread async copies feed the same MMAs
    backend.check_status()
    # a single image given as [H,W,C] and batch-composition independence
    one = backend.rgb_decode(feats[1], "tc")
    assert torch.equal(one[0], tc[1])


def test_rgb_decoder_api_and_errors(backend):
    from neurad_studio_b200.backend import B200Backend
    from neurad_studio_b200.lib import B200NerfError
    from neurad_studio_b200.nerfstudio_api import RGBDecoder

    p, feats, ref = _decoder_golden()
    dec = RGBDecoder(48, 32, 3)
    dec.load_state_dict({k[len("rgb_decoder."):]: v for k, v in p.items()}, strict=False)
    dec = dec.cuda()
    with pytest.raises(RuntimeError):
        dec(feats.cuda())  # training mode: BatchNorm batch statistics are not provided
    dec.eval()
    rgb = dec(feats.cuda())
    assert (rgb.cpu() - ref).abs().max().item() < 1e-4
    fresh = B200Backend(torch.device("cuda", 0))
    with pytest.raises(B200NerfError):
        fresh.rgb_decode(feats)  # set_rgb_decoder missing (feature width unknown)
    fresh.set_rgb_decoder(p)
    with pytest.raises(B200NerfError):
        fresh.rgb_decode(feats[..., :40])
    assert fresh.rgb_decode(feats[:, :0]).shape == (2, 0, 135, 3)


def test_camera_outputs_include_rgb():
    """get_outputs_for_camera_ray_bundle on a 2-D bundle: rays at [1::3, 1::3], NFF, then the rgb decoder -> an image at
    the full bundle resolution (neurad.py:623-675)."""
    from neurad_studio_b200.nerfstudio_api import NeuRADModel, RayBundle
    from oracle import decoder_oracle as D

    meta, g = load_golden("nff_static.npz")
    cfg = cfg_from_meta(meta)
    sd = dict(g["param"])
    sd.update(D.random_decoder_params(seed=31))
    model = NeuRADModel(cfg)
    model.load_reference_state_dict(sd)
    model = model.cuda().eval()
    cam = scene.pandaset_rig(time=1.0, width=48, height=27)[0]
    be = model._bind()
    r = be.raygen_pinhole(cam)
    shp = r.pop("shape")
    rb = RayBundle(origins=r["origins"].view(*shp, 3), directions=r["directions"].view(*shp, 3),
                   pixel_area=r["pixel_area"].view(*shp, 1), times=r["times"].view(*shp, 1))
    out = model.get_outputs_for_camera_ray_bundle(rb)
    assert out["features"].shape == (9, 16, 48) and out["rgb"].shape == (27, 48, 3)
    with torch.no_grad():
        ref = D.rgb_decoder(sd, out["features"].cpu()[None])[0]
    assert (out["rgb"].cpu() - ref).abs().max().item() < 1e-4
