"""torch.autograd bindings of the module-level operators (SURVEY.md 8f, row f2): every forward operator of the library
that sits on the training path gets its hand-written backward operator, so `loss.backward()` through the reference-API
mirror (NeuRADField / NeuRADProposalField / RaySamples.get_weights / renderers, `get_nff_outputs(fused=False)`) reaches
the hash tables, density decoders, MLPs and beta without any torch reference math in between.

The reference gets these gradients from torch autograd (implementation="torch") or tiny-cuda-nn's backward kernels
(field_components/encodings.py:386-404, mlp.py:116-140).  Sample bins carry no gradient (PDFSampler detaches them,
ray_samplers.py:363-364); the actor trajectories do, through the main field's box-frame positions
(require_actor_grad, neurad_encoding.py:174; EncodingFn); the box-frame directions do not (torch-mode SHEncoding is
no_grad, encodings.py:797-800).  With a camera optimizer the ray origins and directions require grad: the sample means
then receive a gradient from EncodingFn / DensityFn, and IsotropicGaussianFn passes it on to the rays
(cameras/camera_optimizers.py:173-182, cameras/rays.py:109-124)."""
from __future__ import annotations

from typing import List, Optional

import torch
from torch import Tensor
from torch.autograd import Function

# The reference trains under AMP (mixed_precision, configs/method_configs.py:401).  The operators here are fp32: under
# autocast their tensor arguments are cast to fp32 and autocast is switched off inside forward / backward.
_fwd = torch.amp.custom_fwd(device_type="cuda", cast_inputs=torch.float32)
_bwd = torch.amp.custom_bwd(device_type="cuda")


def _refuse_edited(ctx) -> None:
    """The backward operators differentiate the unedited actor poses, so a forward that rendered an actor edit
    (eval mode, DynamicActors.actor_editing) has no backward here: raise instead of returning the wrong gradients."""
    if ctx.edited:
        raise RuntimeError("backward through a forward with an active actor edit: the gradients would be those of the "
                           "unedited actor poses; clear dynamic_actors.actor_editing (or train in training mode)")


class EncodingFn(Function):
    """NeuRADHashEncoding.forward: (features [N*S,D], directions [N,S,3]); gradients go to the hash tables, the sample
    means (when they require grad: camera optimisation) and -- for a field built with require_actor_grad (the main
    field, fields/neurad_field.py:50) -- to the actor trajectories `actor_rotations_6d` [T,A,6] / `actor_positions`
    [T,A,3] (pass None for a field without trajectory gradients)."""

    @staticmethod
    @_fwd
    def forward(ctx, be, field: int, mean, std, times, directions, flip, rotations_6d, positions, static_table, *actor_tables):
        out = be.neurad_encoding(field, mean, std, times, directions, flip=flip)
        ctx.be, ctx.field, ctx.edited = be, field, be.actor_edit_active
        ctx.table_shapes = [static_table.shape] + [t.shape for t in actor_tables]
        ctx.save_for_backward(mean, std, times, flip, rotations_6d, positions)
        dirs = out.get("directions")
        if dirs is None:
            dirs = mean.new_zeros(0)
        ctx.mark_non_differentiable(dirs)
        return out["features"], dirs

    @staticmethod
    @_bwd
    def backward(ctx, dfeatures, _ddirs):
        _refuse_edited(ctx)
        mean, std, times, flip, rot6, pos = ctx.saved_tensors
        needs = ctx.needs_input_grad[9:]
        shapes, dev = ctx.table_shapes, dfeatures.device
        dfeatures = dfeatures.contiguous()
        g_static = torch.zeros(shapes[0], device=dev) if needs[0] else None
        g_actors: List[Optional[Tensor]] = [torch.zeros(shapes[1 + a], device=dev) if nd else None for a, nd in enumerate(needs[1:])]
        if g_static is not None or any(g is not None for g in g_actors):
            ctx.be.neurad_encoding_bwd(ctx.field, mean, std, times, {"static": g_static, "actors": g_actors}, dfeatures=dfeatures, flip=flip)
        g_rot = g_pos = None
        if rot6 is not None and pos is not None and (ctx.needs_input_grad[7] or ctx.needs_input_grad[8]):
            g_rot, g_pos = torch.zeros_like(rot6), torch.zeros_like(pos)
            ctx.be.neurad_encoding_pose_bwd(ctx.field, mean, std, times, dfeatures, rot6, pos, g_rot, g_pos, flip=flip)
        g_mean = None
        if ctx.needs_input_grad[2]:
            g_mean = ctx.be.neurad_encoding_mean_bwd(ctx.field, mean, std, times, dfeatures=dfeatures, flip=flip).reshape(mean.shape)
        return (None, None, g_mean) + (None,) * 4 + (g_rot if ctx.needs_input_grad[7] else None, g_pos if ctx.needs_input_grad[8] else None, g_static, *g_actors)


class DensityFn(Function):
    """NeuRADProposalField.get_density: density [N,S]; gradients go to the hash tables, the density decoder and (when
    they require grad: camera optimisation) the sample means."""

    @staticmethod
    @_fwd
    def forward(ctx, be, field: int, mean, std, times, flip, static_table, decoder_weight, *actor_tables):
        # the decoder's gradient is sum_i g_i * features_i: keep the forward's features ([N*S, 6] floats) instead of
        # re-gathering 48 table entries per sample in the backward kernel
        want_feats = bool(ctx.needs_input_grad[7])
        out = be.neurad_encoding(field, mean, std, times, None, want_features=want_feats, want_density=True, flip=flip)
        ctx.be, ctx.field, ctx.edited = be, field, be.actor_edit_active
        ctx.save_for_backward(mean, std, times, flip, out["density"], out.get("features"))
        ctx.decoder_shape = decoder_weight.shape
        ctx.table_shapes = [static_table.shape] + [t.shape for t in actor_tables]
        return out["density"]

    @staticmethod
    @_bwd
    def backward(ctx, ddensity):
        _refuse_edited(ctx)
        mean, std, times, flip, density, feats = ctx.saved_tensors
        needs = ctx.needs_input_grad[6:]
        shapes, dev = ctx.table_shapes, ddensity.device
        ddensity = ddensity.contiguous()
        g_static = torch.zeros(shapes[0], device=dev) if needs[0] else None
        g_actors = [torch.zeros(shapes[1 + a], device=dev) if nd else None for a, nd in enumerate(needs[2:])]
        g_dec = None
        if needs[1]:
            # trunc_exp backward (field_components/activations.py:38-41): g * exp(clamp(x, -15, 15)), density = exp(x)
            g = ddensity.reshape(1, -1) * density.reshape(1, -1).clamp(3.0590232e-07, 3269017.372)
            g_dec = (g @ feats).reshape(ctx.decoder_shape)
        if g_static is not None or any(t is not None for t in g_actors):
            ctx.be.neurad_encoding_bwd(ctx.field, mean, std, times, {"static": g_static, "actors": g_actors, "decoder": None},
                                       density=density, ddensity=ddensity, flip=flip)
        g_mean = None
        if ctx.needs_input_grad[2]:
            g_mean = ctx.be.neurad_encoding_mean_bwd(ctx.field, mean, std, times, density=density, ddensity=ddensity,
                                                     flip=flip).reshape(mean.shape)
        return (None, None, g_mean) + (None,) * 3 + (g_static, g_dec, *g_actors)


class IsotropicGaussianFn(Function):
    """Frustums.get_fast_isotropic_gaussian (cameras/rays.py:109-124): (mean [N,S,3], std [N,S]); gradients go to the
    per-ray origins and directions [N,3] through the mean (the bins are detached; std depends on neither)."""

    @staticmethod
    @_fwd
    def forward(ctx, be, origins, directions, pixel_area, bins_e):
        mean, std = be.isotropic_gaussian(origins, directions, pixel_area, bins_e)
        ctx.be = be
        ctx.shapes = (origins.shape, directions.shape)
        ctx.save_for_backward(bins_e)
        ctx.mark_non_differentiable(std)
        return mean, std

    @staticmethod
    @_bwd
    def backward(ctx, dmean, _dstd):
        (bins_e,) = ctx.saved_tensors
        do, dd = ctx.be.isotropic_gaussian_bwd(bins_e, dmean.contiguous())
        return (None, do.reshape(ctx.shapes[0]) if ctx.needs_input_grad[1] else None,
                dd.reshape(ctx.shapes[1]) if ctx.needs_input_grad[2] else None, None, None)


class MlpFn(Function):
    """MLP.forward (ReLU hidden layers, linear output) on the wgmma operator; args: x, then weight_0, bias_0, ..."""

    @staticmethod
    @_fwd
    def forward(ctx, be, x, *wb):
        ws, bs = list(wb[0::2]), list(wb[1::2])
        ctx.be = be
        if any(ctx.needs_input_grad[1:]) and len(ws) > 1:
            # like autograd keeps them for MLP.forward: the hidden pre-activations, stored by the same launch
            y, zs = be.mlp_fwd(x, ws, bs, want_hidden=True)
        else:
            y, zs = be.mlp_fwd(x, ws, bs), []
        ctx.n_hidden = len(zs)
        ctx.save_for_backward(x, *wb, *zs)
        return y

    @staticmethod
    @_bwd
    def backward(ctx, dy):
        x, *rest = ctx.saved_tensors
        wb = rest[: len(rest) - ctx.n_hidden]
        zs = rest[len(rest) - ctx.n_hidden:] if ctx.n_hidden else None
        ws, bs = list(wb[0::2]), list(wb[1::2])
        needs = ctx.needs_input_grad
        dws = [torch.zeros_like(w) if needs[2 + 2 * l] or needs[3 + 2 * l] else None for l, w in enumerate(ws)]
        dbs = [torch.zeros_like(b) if dws[l] is not None else None for l, b in enumerate(bs)]
        dx = ctx.be.mlp_bwd(x, ws, bs, dy.contiguous(), dws, dbs, need_dx=needs[1], hidden=zs)
        grads = []
        for l in range(len(ws)):
            grads += [dws[l] if needs[2 + 2 * l] else None, dbs[l] if needs[3 + 2 * l] else None]
        return (None, dx, *grads)


class FieldMidFn(Function):
    """[geo_embedding | SH4((d+1)/2)] (fields/neurad_field.py:139-141); gradient to geo_out only."""

    @staticmethod
    @_fwd
    def forward(ctx, be, geo_out, directions):
        ctx.be = be
        ctx.save_for_backward(geo_out)
        return be._field_mid(geo_out, directions)

    @staticmethod
    @_bwd
    def backward(ctx, dx2):
        (geo,) = ctx.saved_tensors
        dgeo, _ = ctx.be.field_heads_bwd(geo, None, None, None, dx2.contiguous())
        return None, dgeo, None


class FieldTailFn(Function):
    """feature = geo_embedding + mlp_feature_out, sdf, alpha = sigmoid(-sdf (|beta| + 1e-4)) (neurad_field.py:141-149)."""

    @staticmethod
    @_fwd
    def forward(ctx, be, geo_out, mlp_out, beta_param):
        ctx.be = be
        ctx.save_for_backward(geo_out, beta_param)
        return be._field_tail(geo_out, mlp_out)

    @staticmethod
    @_bwd
    def backward(ctx, dfeature, dsdf, dalpha):
        geo, beta_param = ctx.saved_tensors
        dgeo, dbeta = ctx.be.field_heads_bwd(geo, dfeature.contiguous(), dsdf, dalpha, None)
        # d(|beta| + 1e-4) / d beta = sign(beta)  (model_components/utils.py:38-41)
        g_beta = (dbeta.reshape(beta_param.shape) * torch.sign(beta_param)) if ctx.needs_input_grad[3] else None
        return None, dgeo, dfeature, g_beta


class AlphaToWeightsFn(Function):
    """nerfacc.render_weight_from_alpha on dense [N,S] (models/neurad.py:717)."""

    @staticmethod
    @_fwd
    def forward(ctx, be, alphas):
        ctx.be = be
        ctx.save_for_backward(alphas)
        return be.alpha_to_weights(alphas)

    @staticmethod
    @_bwd
    def backward(ctx, dw):
        (alphas,) = ctx.saved_tensors
        return None, ctx.be.alpha_to_weights_bwd(alphas, dw.contiguous())


class DensityToWeightsFn(Function):
    """RaySamples.get_weights (cameras/rays.py:188-210); gradient to the densities (bin widths are detached)."""

    @staticmethod
    @_fwd
    def forward(ctx, be, deltas, densities):
        ctx.be = be
        ctx.save_for_backward(deltas, densities)
        return be.density_to_weights(deltas, densities)

    @staticmethod
    @_bwd
    def backward(ctx, dw):
        deltas, densities = ctx.saved_tensors
        return None, None, ctx.be.density_to_weights_bwd(deltas, densities, dw.contiguous())


class CompositeFn(Function):
    """FeatureRenderer / AccumulationRenderer / render_depth_simple in one pass: returns (values [N,C], accumulation
    [N,1], depth [N,1]); tensors that were not asked for come back empty."""

    @staticmethod
    @_fwd
    def forward(ctx, be, weights, values, starts, ends, want_acc: bool, want_depth: bool):
        out = be.composite(weights, values, starts, ends, "simple" if want_depth else None, want_accumulation=want_acc)
        ctx.be = be
        ctx.save_for_backward(weights, values if values is not None else weights.new_zeros(0),
                              starts if starts is not None else weights.new_zeros(0),
                              ends if ends is not None else weights.new_zeros(0))
        ctx.has = (values is not None, want_acc, want_depth)
        e = weights.new_zeros(0)
        return out.get("values", e), out.get("accumulation", e), out.get("depth", e)

    @staticmethod
    @_bwd
    def backward(ctx, dvalues_out, dacc, ddepth):
        weights, values, starts, ends = ctx.saved_tensors
        has_v, has_a, has_d = ctx.has
        dw, dv = ctx.be.composite_bwd(weights, values if has_v else None, starts if has_d else None, ends if has_d else None,
                                      dvalues_out.contiguous() if has_v else None, dacc.contiguous() if has_a else None,
                                      ddepth.contiguous() if has_d else None,
                                      need_dweights=ctx.needs_input_grad[1], need_dvalues=has_v and ctx.needs_input_grad[2])
        if dw is not None:
            dw = dw.reshape(weights.shape)
        if dv is not None:
            dv = dv.reshape(values.shape)
        return None, dw, dv, None, None, None, None


class DistortionLossFn(Function):
    """lossfun_distortion per ray (losses.py:160-172): gradient to the weights; the spacing edges are detached."""

    @staticmethod
    @_fwd
    def forward(ctx, be, sdist, weights):
        loss, dw = be.distortion_loss(sdist, weights, want_grad=True)
        ctx.save_for_backward(dw)
        return loss

    @staticmethod
    @_bwd
    def backward(ctx, dloss):
        (dw,) = ctx.saved_tensors
        return None, None, dw * dloss[:, None]


class InterlevelLossFn(Function):
    """zipnerf_interlevel_loss for one proposal level, per ray (losses.py:645-705): gradient to the proposal weights."""

    @staticmethod
    @_fwd
    def forward(ctx, be, sdist, weights, prop_sdist, prop_weights, pulse_width: float):
        loss, dwp = be.zipnerf_interlevel_loss(sdist, weights, prop_sdist, prop_weights, pulse_width, want_grad=True)
        ctx.save_for_backward(dwp)
        return loss

    @staticmethod
    @_bwd
    def backward(ctx, dloss):
        (dwp,) = ctx.saved_tensors
        return None, None, None, None, dwp * dloss[:, None], None


class LidarLossesFn(Function):
    """The lidar terms of get_metrics_dict in training mode (neurad.py:486-520) over the lidar rows: out [4 + rounds] =
    [depth_loss, intensity_loss, ray_drop_loss, quantile, depth_loss_0, ...] and the quantile mask.  Gradients go to the
    predicted depth, the proposal depths, the intensity and the ray-drop logits; none flows through the mask, the quantile
    or the non-return targets.  `settings` = (non_return_lidar_distance, non_return_loss_mult, quantile_threshold)."""

    @staticmethod
    @_fwd
    def forward(ctx, be, settings, distance, did_return, gt_intensity, pred, intensity, logits, *prop):
        out, counts, mask = be.lidar_losses(pred, prop, distance, did_return, intensity, gt_intensity, logits, *settings)
        ctx.be, ctx.settings = be, settings
        ctx.save_for_backward(distance, did_return, gt_intensity, pred, intensity, logits, mask, counts, *prop)
        ctx.mark_non_differentiable(mask)
        return out, mask

    @staticmethod
    @_bwd
    def backward(ctx, d_out, _d_mask):
        distance, did_return, gt, pred, intensity, logits, mask, counts, *prop = ctx.saved_tensors
        dp, dprop, di, dl = ctx.be.lidar_losses_bwd(pred, prop, distance, did_return, intensity, gt, logits, *ctx.settings[:2],
                                                    mask, counts, d_out)
        return (None, None, None, None, None, dp.view(pred.shape), di.view(intensity.shape), dl.view(logits.shape),
                *(dprop[i].view(p.shape) for i, p in enumerate(prop)))


class HashGridFn(Function):
    """HashEncoding.forward (the stand-alone grid, encodings.py:425-471): gradient to the hash table (the reference also
    differentiates with respect to the positions; NeuRAD's path never asks for that on a stand-alone grid -- its position
    gradients go through NeuRADHashEncoding: EncodingFn / DensityFn)."""

    @staticmethod
    @_fwd
    def forward(ctx, be, settings, scalings, x, table):
        ctx.be, ctx.settings, ctx.scalings = be, settings, scalings
        ctx.save_for_backward(x)
        ctx.table_shape = table.shape
        return be.hashgrid_fwd(settings, table, x, scalings)

    @staticmethod
    @_bwd
    def backward(ctx, dout):
        (x,) = ctx.saved_tensors
        g = torch.zeros(ctx.table_shape, device=dout.device)
        ctx.be.hashgrid_bwd(ctx.settings, x, dout.contiguous(), g, ctx.scalings)
        return None, None, None, None, g
