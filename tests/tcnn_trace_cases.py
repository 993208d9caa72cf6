"""Bodies of the sample-by-sample tests of the tiny-cuda-nn-layout render kernels (sample_lane_kernel<1> and the shading
kernel with sh_tcnn = 1) and of the layout's grid operator, shared by tests/test_zz_tcnn_trace_gpu.py (dev = "cuda": the
library, production table sizes) and tests/test_tcnn_trace_cpu.py (dev = "cpu": the same device code through the host
emulation, small tables).

The stage checks of tests/render_trace_cases.py (walk, weights, depths, appearance, actor ids, partial-trace and untraced
bit identity) run unchanged; TcnnLayout supplies what differs in this layout, restated in float64 from
oracle/tcnn_oracle.py and nothing of the library's host code:
  * positions: the kernel's fp32 contracted positions (static) and box positions (actors), p = fmaf(x, scale_l, 0.5)
    rounded once (fma_pos), the actor grid's 4th coordinate fl(a / n_actors); cells floor(p), fracs p - floor(p) (exact);
    rows from tcnn_oracle.grid_index plus the level offsets (dense levels: linear, modulo the entry count; the "+1"
    vertex of the last cell wraps);
  * interpolation: float64 over the 2^D corners with the kernel's fp32 fracs.  The kernel's corner weight is a product
    of D factors, each 1 - frac rounded once, with D - 1 rounded products, and the corners are summed by 2^D sequential
    FMAs: <= (2^D + 2 D) U sum_c |w_c f_c| per entry, plus the level-weight terms of render_trace_cases._level_terms
    (level weights from HashEncoding.scalings, not from the tcnn grid scale);
  * parameters: the fp32 master vectors rounded to fp16 here (numpy, round to nearest even, subnormals kept); the
    proposal decoder and the appearance embedding are plain tensors and not rounded; bias-free MLPs unpacked by
    tcnn_oracle.mlp_unpack, lidar decoder included;
  * SH: tiny-cuda-nn's basis with the Condon-Shortley signs, at the kernel's fp32 x = fl(fl(d + 1) - 1) (static samples:
    the ray direction, exactly) or at the float64 rotated direction with that rounding bounded (actor samples).
The grid evaluations count what they cover (Coverage): sample-levels on dense and on hashed levels, sample-levels whose
dense-level "+1" vertex wraps, sample-levels on a dense level exactly at the threshold (res^D == 2^log2_hashmap_size, the
share of a hashed level), and main-field samples per actor.

The tiny-cuda-nn layout runs in the two-stage renderer only ("split"); the fused lane kernel refuses it."""
import copy
import dataclasses
import re

import numpy as np
import torch

import neurad_studio_b200 as nsb
from neurad_studio_b200 import scene
from oracle import tcnn_oracle as TO
from tests import render_trace_cases as C
from tests.tcnn_cases import tcnn_test_config

U, TINY = C.U, C.TINY
SUFFIX = "tcnn_encoding.params"
EDITS = {"tcnn_edits": dict(C.EDITS["edits"])}
GPU_SCENES = ["tcnn_small", "tcnn_default", "tcnn_sweep", "tcnn_init", "tcnn_neurader", "tcnn_edits"]
CPU_SCENES = GPU_SCENES
# the reference corruptions the self-tests feed the comparator (each must be rejected) and the scene that shows each
CORRUPTIONS = {"sh_torch": "tcnn_small", "grid_scale_weights": "tcnn_small", "dense_hashed": "tcnn_small",
               "wrap_clamped": "tcnn_small", "fourth_a_over_a_minus_1": "tcnn_small", "fourth_a": "tcnn_small",
               "unrounded": "tcnn_init", "no_minus_one": "tcnn_small", "no_half": "tcnn_small", "offset_shift": "tcnn_small"}


# ====================================================================================== float64 restatement
def f16_round(t):
    """fp32 -> fp16 -> fp32 by numpy (round to nearest even, fp16 subnormals kept)."""
    return torch.from_numpy(t.detach().cpu().float().numpy().astype(np.float16).astype(np.float32))


def growth(g):
    """HashEncoding.growth_factor: exp((log max_res - log base_res) / (levels - 1))."""
    return float(np.exp((np.log(g.max_res) - np.log(g.base_res)) / (g.num_levels - 1))) if g.num_levels > 1 else 1.0


def grid_layout(g, nd):
    return TO.grid_layout(g.num_levels, g.hashgrid_dim, g.log2_hashmap_size, g.base_res, growth(g), nd)


def fma_pos(x32, s32, half=0.5):
    """fl32(x s + half) with one rounding, as fmaf: x s is exact in double (24 x 24 bits); the double sum may round, and
    where it does and lands exactly half-way between two floats, the exact sum's side of the tie (its TwoSum error)
    decides -- the double result is never rounded a second time blindly."""
    m = x32.double() * float(s32)
    s = m + half
    bp = s - m
    err = (m - (s - bp)) + (half - bp)
    r = s.float()
    rd = r.double()
    other = torch.where(rd > s, torch.nextafter(r, torch.tensor(-np.inf)), torch.nextafter(r, torch.tensor(np.inf))).double()
    tie = (rd != s) & ((rd + other) * 0.5 == s) & (err != 0)
    if tie.any():
        fix = torch.where(err > 0, torch.maximum(rd, other), torch.minimum(rd, other)).float()
        r = torch.where(tie, fix, r)
    return r


class Coverage:
    def __init__(self):
        self.dense = self.hashed = self.wrap = self.threshold = 0
        self.actors = {}

    def __str__(self):
        a = ", ".join(f"{k}: {v}" for k, v in sorted(self.actors.items()))
        return (f"sample-levels dense {self.dense}, hashed {self.hashed}, wrapping {self.wrap}, at the dense threshold "
                f"{self.threshold}; main-field samples per actor {{{a}}}")


def tcnn_levels(lay, table, x32, dev, corrupt=None, cov=None, check_rows=True):
    """Every level of a tcnn grid at the fp32 positions x32 [P, D] (CPU) over the fp32 table [n_entries, F] (on dev):
    float64 interpolation v [P, L, F] and sum_c |w_c f_c| [P, L, F].  `corrupt` (the self-tests): "no_minus_one" /
    "no_half" (cell-centred positions), "dense_hashed", "wrap_clamped", "offset_shift" (level 1 one entry late)."""
    D, L = lay.n_dims, lay.n_levels
    bits = torch.tensor([[(c >> d) & 1 for d in range(D)] for c in range(1 << D)])  # [2^D, D]
    hashed = dataclasses.replace(lay, dense=[False] * L)
    vs, vabs = [], []
    for l in range(L):
        s = np.float32(lay.scale[l])
        if corrupt == "no_minus_one":
            s = np.float32(s + np.float32(1.0))
        p = fma_pos(x32, s, 0.0 if corrupt == "no_half" else 0.5)
        base = torch.floor(p)
        frac = (p - base).double()
        pg = base.long()
        cg = pg[:, None, :] + bits[None]  # [P, 2^D, D]
        res, n = lay.resolution[l], lay.size[l]
        if lay.dense[l] and corrupt == "wrap_clamped":
            cg = cg.clamp_max(res - 1)
        idx = TO.grid_index(hashed if corrupt == "dense_hashed" else lay, l, cg)
        rows = idx + lay.offset[l] + (1 if corrupt == "offset_shift" and l == 1 else 0)
        if check_rows and corrupt is None:
            assert int(rows.min()) >= lay.offset[l] and int(rows.max()) < lay.offset[l] + n, f"level {l}: row outside the level"
        f = table[rows.to(dev)].double()  # [P, 2^D, F]
        w = torch.where(bits[None].bool(), frac[:, None, :], 1 - frac[:, None, :]).prod(-1).to(dev)  # [P, 2^D]
        wf = w[..., None] * f
        vs.append(wf.sum(1))
        vabs.append(wf.abs().sum(1))
        if cov is not None:
            P = x32.shape[0]
            if lay.dense[l]:
                cov.dense += P
                cov.wrap += int((pg >= res - 1).any(-1).sum())
                cov.threshold += P if res**D == n == max(lay.size) else 0  # res^D fills the hashed levels' share exactly
            else:
                cov.hashed += P
    return torch.stack(vs, 1), torch.stack(vabs, 1)


def interp_bound(D):
    """Per-entry constant of the kernel's interpolation: 2 D roundings in a corner weight, 2^D sequential FMAs."""
    return (1 << D) + 2 * D


def sh_tcnn64(v):
    """tiny-cuda-nn's degree-4 SH at v [P, 3] (float64): values [P, 16] and sum |terms| per component [P, 16]."""
    x, y, z = v[:, 0], v[:, 1], v[:, 2]
    ax, ay, az = x.abs(), y.abs(), z.abs()
    xx, yy, zz = x * x, y * y, z * z
    val = torch.stack([torch.full_like(x, 0.28209479177387814), -0.48860251190291987 * y, 0.48860251190291987 * z,
                       -0.48860251190291987 * x, 1.0925484305920792 * x * y, -1.0925484305920792 * y * z,
                       0.94617469575755997 * zz - 0.31539156525251999, -1.0925484305920792 * x * z,
                       0.54627421529603959 * xx - 0.54627421529603959 * yy, 0.59004358992664352 * y * (-3.0 * xx + yy),
                       2.8906114426405538 * x * y * z, 0.45704579946446572 * y * (1.0 - 5.0 * zz),
                       0.3731763325901154 * z * (5.0 * zz - 3.0), 0.45704579946446572 * x * (1.0 - 5.0 * zz),
                       1.4453057213202769 * z * (xx - yy), 0.59004358992664352 * x * (-xx + 3.0 * yy)], -1)
    ab = torch.stack([torch.full_like(x, 0.28209479177387814), 0.48860251190291987 * ay, 0.48860251190291987 * az,
                      0.48860251190291987 * ax, 1.0925484305920792 * ax * ay, 1.0925484305920792 * ay * az,
                      0.94617469575755997 * zz + 0.31539156525251999, 1.0925484305920792 * ax * az,
                      0.54627421529603959 * (xx + yy), 0.59004358992664352 * ay * (3.0 * xx + yy),
                      2.8906114426405538 * ax * ay * az, 0.45704579946446572 * ay * (1.0 + 5.0 * zz),
                      0.3731763325901154 * az * (5.0 * zz + 3.0), 0.45704579946446572 * ax * (1.0 + 5.0 * zz),
                      1.4453057213202769 * az * (xx + yy), 0.59004358992664352 * ax * (xx + 3.0 * yy)], -1)
    return val, ab


class TcnnLayout:
    """The tiny-cuda-nn layout's field stages for render_trace_cases.check_scene (see the module docstring).  One
    instance per scene: it caches the fp16-rounded tables and counts coverage.  `corrupt` names a deliberately wrong
    reference (CORRUPTIONS, the self-tests)."""

    name = "tcnn"

    def __init__(self, corrupt=None):
        self.corrupt = corrupt
        self.cov = Coverage()
        self._tables = {}

    def scene_rays(self, dev, name):
        return scene_rays(dev, name)

    def scene_edit(self, name):
        return EDITS.get(name)

    def _table(self, params, key, F, dev):
        if key not in self._tables:
            t = params[key].reshape(-1).float()
            t = t if self.corrupt == "unrounded" else f16_round(t)
            self._tables[key] = t.reshape(-1, F).to(dev)
        return self._tables[key]

    def _grid(self, params, cfg, pre, g, static, fs, dev, count_actors=False):
        """Level terms (x, bound) [P_m, L, F] of one grid of field `pre` at the static or the actor samples of fs."""
        F = g.hashgrid_dim
        which = "static_grid" if static else "actor_grids.0"
        lay = grid_layout(g, 3 if static else 4)
        if static:
            x32, cs64 = fs.c32_s, fs.cs64_s
        else:
            aid = fs.aid[~fs.static]
            A = cfg.n_actors
            a = aid.float()
            fourth = {"fourth_a_over_a_minus_1": a / float(max(A - 1, 1)), "fourth_a": a}.get(self.corrupt, a / float(A))
            x32, cs64 = torch.cat([fs.c32_a, fourth[:, None]], 1), fs.cs64_a
            if count_actors:
                for k, v in zip(*torch.unique(aid, return_counts=True)):
                    self.cov.actors[int(k)] = self.cov.actors.get(int(k), 0) + int(v)
        tab = self._table(params, f"{pre}.hashgrid.{which}.{SUFFIX}", F, dev)
        v, vabs = tcnn_levels(lay, tab, x32, dev, self.corrupt, self.cov)
        sc = params[f"{pre}.hashgrid.{which}.scalings"]
        if self.corrupt == "grid_scale_weights":
            sc = torch.tensor(lay.scale, dtype=torch.float64)
        lw, t = C.level_weights64(sc, cs64.to(dev))
        return C._level_terms(v, vabs, lw, t, k_interp=interp_bound(lay.n_dims))

    def prop_levels(self, params, cfg, fs, dev):
        pre, gc = "proposal_fields.1", cfg.proposal_grid_2
        x, Ex = self._grid(params, cfg, pre, gc.static, True, fs, dev)
        out = [(fs.static, x[..., 0], Ex[..., 0])]
        if fs.R_a is not None:
            x, Ex = self._grid(params, cfg, pre, gc.actor, False, fs, dev)
            out.append((~fs.static, x[..., 0], Ex[..., 0]))
        return out

    def main_grid(self, params, cfg, fs, dev):
        xs, Es = self._grid(params, cfg, "field", cfg.grid.static, True, fs, dev)
        actor = None
        if fs.R_a is not None:
            xa, Ea = self._grid(params, cfg, "field", cfg.grid.actor, False, fs, dev, count_actors=True)
            actor = (xa.reshape(-1, 16), Ea.reshape(-1, 16))
        return (xs.reshape(-1, 32), Es.reshape(-1, 32)), actor

    def sh(self, dirs, E_dir, static):
        """Static samples: at the kernel's own fp32 x = fl(fl(d + 1) - 1) of the ray direction (exact input).  Actor
        samples: at the float64 rotated direction, whose fp32 value in the kernel is E_dir off, plus <= 2 U for
        fl(d + 1) and <= U for the - 1.  Each component is a sum of monomials of degree <= 3 computed with <= 8
        roundings (fp32 constants included): 8 U sum |terms|; Lipschitz <= 10 in the max-norm of the input on [-1, 1]^3."""
        if self.corrupt == "sh_torch":  # the torch twin's basis: at (d + 1) / 2, without the signs
            return C._sh4_64((dirs + 1) / 2), 72 * U + 10 * E_dir
        x32 = (dirs.float() + 1.0) - 1.0
        v = torch.where(static[:, None], x32.double(), dirs)
        E_x = torch.where(static[:, None], torch.zeros_like(E_dir), E_dir + 3 * U)
        val, ab = sh_tcnn64(v)
        return val, 8 * U * ab + 10 * E_x

    def _mlps(self, params, cfg, dev):
        if "mlps" not in self._tables:
            nff = cfg.nff_out_dim
            geo = TO.mlp_unpack(params[f"field.mlp_geo.{SUFFIX}"].reshape(-1).float(), cfg.grid.static.out_dim,
                                cfg.geo_hidden_dim, 1, nff + 1)
            feat = TO.mlp_unpack(params[f"field.mlp_feature.{SUFFIX}"].reshape(-1).float(), nff + 16, cfg.nff_hidden_dim, 2, nff)
            ws = {"field.mlp_geo.layers.0": geo[0], "field.mlp_geo.layers.1": geo[1]}
            ws.update({f"field.mlp_feature.layers.{i}": w for i, w in enumerate(feat)})
            self._tables["mlps"] = {k: (w.double().to(dev), torch.zeros(w.shape[0], dtype=torch.float64, device=dev))
                                    for k, w in ws.items()}
        return self._tables["mlps"]

    def linear(self, params, cfg, name, dev):
        return self._mlps(params, cfg, dev)[name]

    def lidar_layers(self, params, cfg):
        ws = TO.mlp_unpack(params[f"lidar_decoder.{SUFFIX}"].reshape(-1).float(), cfg.feature_dim, 32, 2, 2)
        return [(w.double(), torch.zeros(w.shape[0], dtype=torch.float64)) for w in ws]

    def describe(self):
        return f"; coverage: {self.cov}"


# ====================================================================================== scenes
def _tcnn_params(cfg, seed, **kw):
    return scene.make_params_tcnn(cfg, seed=seed, beta=kw.pop("beta", 4.0), mlp_gain=kw.pop("mlp_gain", 0.6), **kw)


def _aimed(cfg, n, seed, trajs):
    return C._with_near_far(scene.random_rays(n, cfg, seed=seed, trajectories=trajs), seed + 1)


def scene_rays(dev, name):
    """(cfg, params, rays, image_width) of one tcnn-layout scene.

    tcnn_small: tcnn_test_config(3) (dense and hashed levels in every grid, a dense 4-D level, the main grid's level 2 at
      the dense threshold 32^3 = 2^15), rays aimed at the boxes, nears and fars.
    tcnn_default: NeuRADConfig(n_actors=16); GPU: production sizes (main levels 0-2 dense with 32 768, 357 912 and
      3 869 896 entries, finer levels hashed into 2^22 rows), a PandaSet camera at stride 3 through the 2-D tile walk, a
      lidar sweep and rays aimed at the boxes; CPU: main table 2^16 (level 0 dense), aimed rays.
    tcnn_sweep: zero-area lidar sweeps over four actors (render_trace_cases._sweep_scene's rays; every level at weight 1).
    tcnn_init: tables at 1e-4, tiny-cuda-nn's grid init scale (most values are fp16 subnormals once rounded).
    tcnn_neurader: the neurader preset (GPU: production size; CPU: main table 2^18, level 0 dense at the threshold 64^3).
    tcnn_edits: tcnn_small's scene under the actor edit EDITS["tcnn_edits"], rays aimed at the edited boxes."""
    gpu = dev != "cpu"
    if name in ("tcnn_small", "tcnn_edits"):
        cfg = tcnn_test_config(3)
        trajs = scene.make_trajectories(3, cfg.duration, seed=31)
        params = _tcnn_params(cfg, 32, trajectories=trajs)
        aim = trajs
        if name == "tcnn_edits":
            aim = C.edited_trajectories(trajs, EDITS[name])
            aim = aim + [aim[a] for a in C.edit_selection(3, EDITS[name])] * 3
        return cfg, params, _aimed(cfg, 4100 if gpu else 240, 33, aim), 0
    if name == "tcnn_default":
        cfg = nsb.NeuRADConfig(n_actors=16)
        if not gpu:
            cfg = C._small_tables(cfg, log2_main=16)
        trajs = scene.make_trajectories(16, cfg.duration, seed=41)
        params = _tcnn_params(cfg, 42, trajectories=trajs)
        aimed = _aimed(cfg, 8192 if gpu else 200, 43, trajs)
        if not gpu:
            return cfg, params, aimed, 0
        rays, width = C.camera_and_lidar_rays(cfg)
        rays = C._with_near_far(rays, 44)
        return cfg, params, C._cat(rays, aimed), width
    if name == "tcnn_sweep":
        cfg, tparams, rays, _ = C._sweep_scene(dev, 1.0 if gpu else 0.1)
        cfg = copy.deepcopy(cfg)  # the golden's configuration is shared with the torch-layout sweep scenes
        if not gpu:
            cfg.grid.static.log2_hashmap_size = 16  # main level 0 dense
        params = _tcnn_params(cfg, 21, table_scale=1.0 if gpu else 0.1)
        for k, v in tparams.items():
            if k.startswith("dynamic_actors.") or k == "static_scale":
                params[k] = v
        return cfg, params, rays, 0
    if name == "tcnn_init":
        cfg = nsb.NeuRADConfig(n_actors=0) if gpu else C._small_tables(nsb.NeuRADConfig(n_actors=0), log2_main=16)
        params = _tcnn_params(cfg, 71, table_scale=1e-4)
        return cfg, params, scene.random_rays(4100 if gpu else 160, cfg, seed=72), 0
    if name == "tcnn_neurader":
        cfg, _ = nsb.preset("neurader")
        if not gpu:
            cfg = C._small_tables(cfg, log2_main=18)
        params = _tcnn_params(cfg, 81)
        return cfg, params, C._with_near_far(scene.random_rays(8200 if gpu else 200, cfg, seed=82), 83), 0
    raise KeyError(name)


# coverage each scene must reach: dense / wrap / threshold sample-levels, and main-field samples on every actor
# (tcnn_default's actors stand 12 to 150 m down the road; the far ones get few main-field samples, or none: every actor,
# the last included, is required of tcnn_small and tcnn_edits)
COVERAGE = {"tcnn_small": ("dense", "wrap", "threshold", "actors"), "tcnn_default": ("dense", "wrap"),
            "tcnn_sweep": ("dense", "wrap"), "tcnn_init": ("dense", "wrap"), "tcnn_neurader": ("dense", "wrap"),
            "tcnn_edits": ("dense", "wrap", "threshold", "actors")}
COVERAGE_GPU = {"tcnn_neurader": ("dense", "wrap")}
COVERAGE_CPU = {"tcnn_neurader": ("dense", "wrap", "threshold")}


def check_tcnn_scene(dev, name, mode="split", report=print):
    """check_scene on the tcnn layout, then the scene's coverage.  Returns check_scene's result and the coverage."""
    lay = TcnnLayout()
    res = C.check_scene(dev, name, mode, report=report, layout=lay)
    cov = lay.cov
    need = (COVERAGE_GPU if dev != "cpu" else COVERAGE_CPU).get(name, COVERAGE[name])
    assert cov.hashed > 0, f"{name}: no hashed level evaluated"
    for k in ("dense", "wrap", "threshold"):
        assert k not in need or getattr(cov, k) > 0, f"{name}: no sample-level {k}: {cov}"
    if "actors" in need:
        assert all(cov.actors.get(a, 0) > 0 for a in range(n_actors(name))), f"{name}: an actor is never hit: {cov}"
    return res, cov


def n_actors(name):
    return {"tcnn_small": 3, "tcnn_edits": 3}[name]


# ====================================================================================== self-tests
RATIO = re.compile(r"\|got - ref\| / tol = ([0-9.eE+-]+|inf|nan)")


def field_ratio_error(dev, name, corrupt, out, cfg, params, rays):
    """Run the proposal and main-field comparators with the corrupted reference `corrupt` on a render `out` of every
    ray; returns the worst ratio reported by the first failing comparator (None: the corruption was accepted)."""
    lay = TcnnLayout(corrupt)
    idx = torch.arange(rays["origins"].shape[0])
    edit = lay.scene_edit(name)
    gamma = C.gamma_ffma if dev == "cpu" else C.gamma_f16
    for fn in (lambda: C.check_proposal_weights(out, rays, idx, cfg, params, dev, edit=edit, layout=lay),
               lambda: C.check_main_field(out, rays, idx, cfg, params, dev, gamma, edit=edit, layout=lay)):
        try:
            fn()
        except AssertionError as e:
            m = RATIO.search(str(e))
            assert m is not None, f"{corrupt}: rejected for another reason: {e}"
            return float(m.group(1))
    return None


# ====================================================================================== the grid operator
def _grid_fn(dev):
    """(tcnn_compat layout dict, flat params, x) -> [P, L F] through the library or the host emulation."""
    from neurad_studio_b200 import tcnn_compat as T

    if dev == "cuda":
        from neurad_studio_b200.nerfstudio_api import get_backend

        be = get_backend(torch.device("cuda", 0))
        return lambda g, nd, p, x: be.tcnn_hashgrid_fwd(T.layout_of(g, nd), p.cuda(), x.cuda()).cpu()
    from tests.host_emul import emul

    return lambda g, nd, p, x: emul.tcnn_hashgrid(T.layout_of(g, nd), p, x)


def grid_layouts(dev):
    """(name, HashGridSettings, n_dims) of the operator tests: the default main / proposal / actor grids, neurader's main
    grid (GPU only: 214 M parameters), tcnn_test_config's grids, and a 3-level grid whose dense level 0 has
    res^3 = 512 entries exactly (a multiple of 8: its "+1" vertex wraps to the level's first row) and level 1 at the
    threshold 16^3 = 2^12."""
    d = nsb.NeuRADConfig(n_actors=16)
    t = tcnn_test_config(3)
    out = [("default main", d.grid.static, 3), ("default proposal", d.proposal_grid_2.static, 3),
           ("default main actor", d.grid.actor, 4), ("default proposal actor", d.proposal_grid_2.actor, 4),
           ("test main", t.grid.static, 3), ("test main actor", t.grid.actor, 4),
           ("test proposal", t.proposal_grid_2.static, 3), ("test proposal actor", t.proposal_grid_2.actor, 4),
           ("dense multiple of 8", nsb.HashGridSettings(2, 3, 8, 32, 12), 3)]
    if dev == "cuda":
        out.append(("neurader main", nsb.preset("neurader")[0].grid.static, 3))
    return out


def grid_points(lay, seed, n_actors_4d=(16, 3)):
    """x = 0; x = 1 on each axis alone and on all axes; one ulp either side of (and at) cell boundaries of the finest
    dense level on every axis; for D = 4 the 4th coordinate fl(k / A) for every k of A actors; random points."""
    D = lay.n_dims
    gen = torch.Generator().manual_seed(seed)
    pts = [torch.zeros(1, D), torch.ones(1, D)]
    for d in range(D):
        p = torch.rand(1, D, generator=gen)
        p[0, d] = 1.0
        pts.append(p)
    dense = [l for l in range(lay.n_levels) if lay.dense[l]]
    if dense:
        l = dense[-1]
        s = np.float32(lay.scale[l])
        for k in torch.randint(1, lay.resolution[l], (8,), generator=gen).tolist():
            xb = torch.tensor(np.float32((k - 0.5) / float(s)))
            for xv in (torch.nextafter(xb, torch.tensor(0.0)), xb, torch.nextafter(xb, torch.tensor(1.0))):
                for d in range(D):
                    p = torch.rand(1, D, generator=gen)
                    p[0, d] = xv
                    pts.append(p)
    if D == 4:
        for A in n_actors_4d:
            p = torch.rand(A, 4, generator=gen)
            p[:, 3] = torch.arange(A).float() / float(A)
            pts.append(p)
    pts.append(torch.rand(600, D, generator=gen))
    return torch.cat(pts).clamp(0.0, 1.0).float()


def grid_operator_entry_by_entry(dev, report=print):
    """The grid operator at every entry against tcnn_levels (float64, its per-entry bound (2^D + 2 D) U sum |w f| plus a
    subnormal floor), with the reference's rows inside their level and dense-level wraps reached."""
    grid = _grid_fn(dev)
    gen = torch.Generator().manual_seed(11)
    for i, (nm, g, nd) in enumerate(grid_layouts(dev)):
        lay = grid_layout(g, nd)
        n = (lay.offset[-1] + lay.size[-1]) * lay.n_features
        params = f16_round(torch.rand(n, generator=gen) * 2 - 1)
        x = grid_points(lay, 100 + i)
        cov = Coverage()
        v, vabs = tcnn_levels(lay, params.reshape(-1, lay.n_features), x, "cpu", cov=cov)
        got = grid(g, nd, params, x).reshape(v.shape)
        tol = interp_bound(nd) * U * vabs + (1 << nd) * TINY
        worst = C._ratio(got, v, tol, f"tcnn grid {nm} (D = {nd})")
        if any(lay.dense):
            assert cov.wrap > 0, f"{nm}: no dense-level wrap reached"
        report(f"\n[tcnn grid] {nm} (D = {nd}, {x.shape[0]} points): worst |got - ref| / bound {worst:.3g}; {cov}")
