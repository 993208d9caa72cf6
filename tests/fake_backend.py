"""TEST SCAFFOLDING ONLY -- a CPU stand-in for B200Backend's LEAF operators, so that the Python glue of the reference-API
mirror (RaySamples / PDFSampler / ProposalNetworkSampler / NeuRADField / the per-module walk of get_nff_outputs, and
B200Backend.field_forward's composition) can be executed in the GPU-less container.

Leaves map onto the oracle (already GPU-validated operators) or onto the host emulation of the new device code
(tests/host_emul: the module-level encoding).  Nothing here is importable from the product package; the product has
no CPU path (tests/test_cabi.py::test_no_cpu_fallback)."""
from typing import Dict, Optional

import torch

from neurad_studio_b200.backend import B200Backend
from neurad_studio_b200.lib import FIELD_MAIN
from oracle import neurad_oracle as O
from oracle import simple_oracle as S
from oracle.convert import to_oracle_cfg
from tests.host_emul import emul


class FakeBackend(B200Backend):
    def __init__(self):  # no library, no context
        self.device = torch.device("cpu")
        self.cfg = None
        self.params: Dict[str, torch.Tensor] = {}

    def close(self):
        pass

    def check_status(self):
        pass

    def load_params(self, cfg, params, density_field_of_round=(2, 2)):
        self.cfg, self.params = cfg, {k: v.detach().cpu() for k, v in params.items()}
        p = self.params
        names = ["field.mlp_geo.layers.0", "field.mlp_geo.layers.1", "field.mlp_feature.layers.0",
                 "field.mlp_feature.layers.1", "field.mlp_feature.layers.2"]
        ts = []
        for nme in names:
            ts += [p[nme + ".weight"], p[nme + ".bias"]]
        self._field_mlps = {"geo": (ts[0:4:2], ts[1:4:2]), "feature": (ts[4::2], ts[5::2])}
        self._beta = float(p["field.sdf_to_density.beta"].abs().item() + 0.0001)

    # ---- leaves backed by the host emulation of the NEW device code
    def isotropic_gaussian(self, origins, directions, pixel_area, bins_e):
        return emul.gaussian(origins, directions, pixel_area, bins_e)

    def neurad_encoding(self, field, mean, std, times, directions=None, want_features=True, want_density=False,
                        want_actor_id=False, flip=None):
        return emul.encoding(self.cfg, self.params, O.pdf_u, field, mean.detach(), std.detach(), times, directions,
                             want_features, want_density, want_actor_id, flip)

    def neurad_encoding_bwd(self, field, mean, std, times, grads, dfeatures=None, density=None, ddensity=None, flip=None):
        emul.encoding_bwd(self.cfg, self.params, O.pdf_u, field, mean, std, times, grads, dfeatures, density, ddensity, flip)

    def neurad_encoding_pose_bwd(self, field, mean, std, times, dfeatures, rotations_6d, positions, grad_rotations_6d, grad_positions,
                                 flip=None):
        emul.encoding_pose_bwd(self.cfg, self.params, O.pdf_u, field, mean, std, times, dfeatures, grad_rotations_6d, grad_positions, flip)

    def alpha_to_weights_bwd(self, alphas, dweights):
        return emul.weights_bwd(True, alphas, None, dweights)

    def density_to_weights_bwd(self, deltas, densities, dweights):
        return emul.weights_bwd(False, deltas, densities, dweights)

    def linear_wgrad(self, x, dy, relu_x, dweight, dbias):
        emul.linear_wgrad(x.detach(), dy.detach(), relu_x, dweight, dbias)

    # backward leaves whose kernels are a few lines each (modules.cuh): the same formulas in torch
    def relu_bwd(self, z, dz):
        dz[~(z > 0)] = 0
        return dz

    @torch.no_grad()
    def mlp_dgrad(self, dy, weight, relu_z=None):
        dx = dy.reshape(-1, dy.shape[-1]) @ weight
        if relu_z is not None:
            dx[~(relu_z.reshape(dx.shape) > 0)] = 0
        return dx

    def field_heads_bwd(self, geo, dfeature, dsdf, dalpha, dx2):
        p, gdim = geo.shape[0], geo.shape[1] - 1
        dgeo = torch.zeros(p, gdim + 1)
        dbeta = torch.zeros(1)
        sd = geo[:, 0]
        if dsdf is not None:
            dgeo[:, 0] += dsdf.reshape(p)
        if dalpha is not None:
            al = torch.sigmoid(-sd * self._beta)
            t = dalpha.reshape(p) * al * (1 - al)
            dgeo[:, 0] -= self._beta * t
            dbeta += (-sd * t).sum()
        if dfeature is not None:
            dgeo[:, 1:] += dfeature.reshape(p, gdim)
        if dx2 is not None:
            dgeo[:, 1:] += dx2.reshape(p, gdim + 16)[:, :gdim]
        return dgeo, dbeta

    def composite_bwd(self, weights, values, starts, ends, dvalues_out, dacc, ddepth, need_dweights=True, need_dvalues=True):
        n, s = weights.shape[0], weights.shape[1]
        w = weights.reshape(n, s)
        dw = torch.zeros(n, s)
        dv = None
        if dacc is not None:
            dw += dacc.reshape(n, 1)
        if ddepth is not None:
            dw += ddepth.reshape(n, 1) * (starts.reshape(n, s) + ends.reshape(n, s)) * 0.5
        if dvalues_out is not None:
            c = values.shape[-1]
            dw += (values.reshape(n, s, c) * dvalues_out.reshape(n, 1, c)).sum(-1)
            dv = w[..., None] * dvalues_out.reshape(n, 1, c)
        return (dw if need_dweights else None), (dv if need_dvalues else None)

    @torch.no_grad()
    def _field_mid(self, geo, directions):
        return torch.cat([geo[:, 1:], O.sh_components_l4((directions.reshape(-1, 3) + 1.0) / 2.0)], dim=-1)

    @torch.no_grad()
    def _field_tail(self, geo, h):
        sdf = geo[:, 0]
        return geo[:, 1:] + h, sdf, torch.sigmoid(-sdf * self._beta)

    # ---- leaves that exist (and are GPU-validated) since earlier commits: the oracle's restatements
    @torch.no_grad()
    def mlp_fwd(self, x, weights, biases=None, want_hidden=False):
        y = x.reshape(-1, x.shape[-1])
        zs = []
        for i, w in enumerate(weights):
            y = torch.nn.functional.linear(y, w, None if biases is None else biases[i])
            if i < len(weights) - 1:
                zs.append(y)
                y = torch.relu(y)
        y = y.reshape(*x.shape[:-1], y.shape[-1])
        return (y, zs) if want_hidden else y

    @torch.no_grad()
    def frustum_positions(self, origins, directions, bins_e, aabb=None):
        n = bins_e.shape[0]
        p = S.frustum_positions(origins.reshape(n, 3), directions.reshape(n, 3), bins_e[:, :-1, None], bins_e[:, 1:, None])
        return p if aabb is None else S.normalized_positions(p, aabb.float())

    @torch.no_grad()
    def density_rgb_heads(self, raw):
        return torch.exp(raw[..., :1]), torch.sigmoid(raw[..., 1:])

    @torch.no_grad()
    def hashgrid_fwd(self, g, table, x, scalings=None, want_indices=False):
        sc = g.scalings() if scalings is None else scalings
        y = O.hash_encode(x.reshape(-1, 3), table, sc, 2 ** g.log2_hashmap_size)
        return y.reshape(*x.shape[:-1], y.shape[-1])

    def hashgrid_bwd(self, g, x, dout, grad_table, scalings=None):
        sc = g.scalings() if scalings is None else scalings
        emul.hashgrid_bwd(g.num_levels, g.hashgrid_dim, g.log2_hashmap_size, sc, x.detach(), dout, grad_table)

    @torch.no_grad()
    def sh4_fwd(self, dirs):
        return O.sh_components_l4(dirs)

    def spaced_sample(self, nears, fars, num_samples, spacing="uniform", power_lambda=-1.0, power_scaling=0.1):
        f = fars.reshape(-1, 1)
        nr = torch.zeros_like(f) if nears is None else nears.reshape(-1, 1)
        bins, euclid = S.spaced_sample(nr, f, num_samples, self.SPACINGS[spacing], power_lambda, power_scaling)
        return bins[0], euclid

    def spacing_to_euclidean(self, bins_s, nears, fars, spacing="power", power_lambda=-1.0, power_scaling=0.1):
        fn, inv = S.spacing_fns(self.SPACINGS[spacing], power_lambda, power_scaling)
        f = fars.reshape(-1, 1)
        nr = torch.zeros_like(f) if nears is None else nears.reshape(-1, 1)
        return inv(bins_s * fn(f) + (1 - bins_s) * fn(nr))

    def spaced_sample_stratified(self, nears, fars, num_samples, t_rand, spacing="uniform", power_lambda=-1.0, power_scaling=0.1):
        f = fars.reshape(-1, 1)
        nr = torch.zeros_like(f) if nears is None else nears.reshape(-1, 1)
        bins, euclid = S.spaced_sample(nr, f, num_samples, self.SPACINGS[spacing], power_lambda, power_scaling, t_rand=t_rand)
        return bins.expand_as(euclid).contiguous(), euclid

    def pdf_resample_stratified(self, weights, bins, num_samples, rand, histogram_padding=0.01):
        r = O.pdf_resample(weights, bins, num_samples, histogram_padding, rand=rand)
        return r["bins"], r["cdf"], r["inds"].int()

    def lidar_carving_mask(self, bins_e, is_lidar, directions_norm, did_return, carving_epsilon, non_return_distance):
        from oracle import losses_oracle as LO

        n = bins_e.shape[0]
        return LO.is_close_to_lidar(bins_e, is_lidar.reshape(n).bool(), directions_norm.reshape(n),
                                    None if did_return is None else did_return.reshape(n).bool(), carving_epsilon, non_return_distance)

    def set_rgb_decoder(self, sd, prefix="rgb_decoder", bn_eps=1e-5):
        pre = prefix + "." if prefix else ""
        self._dec = {"rgb_decoder." + k[len(pre):]: v.detach().cpu() for k, v in sd.items() if k.startswith(pre)}

    @torch.no_grad()
    def rgb_decode(self, features, impl="tc", out=None):
        from oracle import decoder_oracle as D

        f = features if features.dim() == 4 else features[None]
        return D.rgb_decoder(self._dec, f)

    def distortion_loss(self, sdist, weights, want_grad=False):
        return emul.distortion_loss(sdist, weights.detach(), want_grad)

    def zipnerf_interlevel_loss(self, sdist, weights, prop_sdist, prop_weights, pulse_width, want_grad=False):
        return emul.zipnerf_interlevel(sdist, weights, prop_sdist, prop_weights.detach(), pulse_width, want_grad)

    def pdf_resample(self, weights, bins, num_samples, histogram_padding=0.01):
        r = O.pdf_resample(weights, bins, num_samples, histogram_padding)
        return r["bins"], r["cdf"], r["inds"].int()

    @torch.no_grad()
    def density_to_weights(self, deltas, densities):
        return O.weights_from_density(deltas, densities)

    @torch.no_grad()
    def alpha_to_weights(self, alphas):
        return O.render_weight_from_alpha(alphas)

    @torch.no_grad()
    def composite(self, weights, values=None, starts=None, ends=None, depth_method=None, background=None,
                  value_nan_to_num=False, want_accumulation=True):
        n, s = weights.shape[0], weights.shape[1]
        w = weights.reshape(n, s, 1)
        out = {}
        if values is not None:
            if values.shape[-1] > 64:
                raise ValueError("at most 64 value channels")
            v = values.reshape(n, s, values.shape[-1])
            out["values"] = (w * (torch.nan_to_num(v) if value_nan_to_num else v)).sum(dim=-2)
            if background is not None:
                out["values"] = out["values"] + torch.tensor(background, dtype=torch.float32) * (1.0 - w.sum(dim=-2))
        if want_accumulation:
            out["accumulation"] = w.sum(dim=-2)
        if depth_method == "simple":
            out["depth"] = (w * (starts.reshape(n, s, 1) + ends.reshape(n, s, 1)) / 2).sum(dim=-2)
        elif depth_method == "median":
            out["depth"] = S.depth_median(w, starts.reshape(n, s, 1), ends.reshape(n, s, 1))
        elif depth_method == "expected":
            out["depth"] = S.depth_expected(w, starts.reshape(n, s, 1), ends.reshape(n, s, 1))
        elif depth_method is not None:
            raise NotImplementedError(depth_method)
        return out

    # ---- ray generation (GPU-validated kernels; the oracle's restatement of Cameras / Lidars.generate_rays here)
    def raygen_pinhole(self, cam, row0=0, row_step=1, col0=0, col_step=1, out=None):
        ys, xs = torch.meshgrid(torch.arange(row0, cam.height, row_step), torch.arange(col0, cam.width, col_step), indexing="ij")
        coords = (torch.stack([ys, xs], -1).reshape(-1, 2) + 0.5).float()
        r = O.generate_rays_pinhole(cam.c2w, cam.fx, cam.fy, cam.cx, cam.cy, cam.height, cam.width, coords, cam.time, cam.velocity,
                                    cam.rolling_shutter_time, cam.time_to_center_pixel)
        return {"origins": r["origins"].contiguous(), "directions": r["directions"], "pixel_area": r["pixel_area"], "times": r["times"],
                "shape": tuple(ys.shape)}

    def raygen_lidar_points(self, scan, points=None, out=None):
        r = O.generate_rays_lidar_points(scan.l2w, scan.points if points is None else points, scan.time, scan.velocity)
        return {k: r[k] for k in ("origins", "directions", "pixel_area", "times", "directions_norm", "did_return")}

    def render(self, rays, want_trace=False, want_intensity=False, out=None, image_width=0):
        n = rays["origins"].shape[0]
        col = lambda t: t.reshape(n, 1)  # noqa: E731
        with torch.no_grad():
            res = O.nff_outputs(self.params, to_oracle_cfg(self.cfg), rays["origins"].reshape(n, 3), rays["directions"].reshape(n, 3),
                                col(rays["pixel_area"]), col(rays["times"]),
                                col(rays.get("sensor_idx", torch.zeros(n, dtype=torch.long))),
                                col(rays["is_lidar"]).bool() if "is_lidar" in rays else None)
            if want_intensity:
                res["intensity"], res["ray_drop_logits"] = O.decode_lidar(self.params, res["features"])
            return res
