"""Float64 references, exact predictors and per-entry bounds for the camera rgb decoder's ten layers
(csrc/rgb_decoder.cuh, b200nerf_rgb_decode_layer).  Device-agnostic torch: the GPU tests run them on the kernels' own
inputs, the CPU tests on small tensors (comparator self-tests).

ACT tensors are bf16 [B,H,W,64]: elements 0..31 are the hi parts (bf16 of the value, round to nearest even) of the 32
channels, 32..63 the lo parts (bf16 of value - hi) -- the library's 128-byte ACT pixel (include/b200nerf.h).

Two families:
* exact: parameters and inputs chosen so every fp32 operation the kernels issue is exact (integers / dyadics, every
  partial sum below 2^24 quanta, BatchNorm fold with fl(var + eps) = 1 and gamma a power of two).  Then the tensor-core
  kernels compute conv(A_hi, W_hi) + conv(A_lo, W_hi) + conv(A_hi, W_lo) = conv(A, W) - conv(A_lo, W_lo) and the CUDA-core
  kernel conv(A, W), plus bias and residual, ReLU and the round-to-nearest-even hi/lo split: predicted bit for bit.
* bounded: realistic parameters; float64 with the BatchNorm folded in float64 from the state dict, and one bound per
  entry derived from the code (see conv7_bound_terms).  No bound is scaled to a tensor's maximum.
"""
from __future__ import annotations

import math
from typing import Dict, Iterator, Optional, Tuple

import torch

U = 2.0 ** -24          # fp32 unit roundoff
SPLIT = 2.0 ** -16      # |v - hi - lo| <= 2^-16 |v| for the RN bf16 hi/lo split (hi within 2^-8, lo within 2^-8 of the rest)
N_MMA = 49 * 2 * 3      # wgmma instructions accumulating into one output entry: 49 taps x 2 k-steps x 3 products
MMA_ADD = 2.0 ** -22    # error of one wgmma accumulation, relative to |acc| + sum |its 16 products| (see conv7_bound_terms)
N_FFMA = 49 * 32        # dec_conv7_ref_kernel: the folded bias, then at most 1568 sequential FMAs
SLOP = 1.0 + 2.0 ** -10  # second-order terms of the first-order bounds below
BLOCKS = (2, 3, 5, 6)
CONV_LAYERS = (1, 2, 3, 4, 6, 7, 8, 9)
RES_LAYERS = (2, 4, 7, 9)
IMPLS = ("tc", "tc_ldgsts", "ref")
PREFIX = "rgb_decoder"


def conv_index(layer: int) -> int:
    """The library's folded-conv slot (0..7) of a 7x7 layer."""
    return layer - 1 if layer < 5 else layer - 2


def conv_bn_keys(layer: int) -> Tuple[str, str]:
    i = conv_index(layer)
    cv, bn = ((0, 1), (3, 4))[i % 2]
    m = f"{PREFIX}.{BLOCKS[i // 2]}.main_branch"
    return f"{m}.{cv}", f"{m}.{bn}"


# ------------------------------------------------------------------------------------------------------ ACT layout
def pack_act(v: torch.Tensor) -> torch.Tensor:
    """float32 [...,32] -> ACT [...,64]: split_pack2 (hi = bf16_rn(v), lo = bf16_rn(v - hi); v - hi is exact in fp32)."""
    v = v.float()
    hi = v.to(torch.bfloat16)
    lo = (v - hi.float()).to(torch.bfloat16)
    return torch.cat([hi, lo], -1)


def act_hi_lo(a: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    return a[..., :32].double(), a[..., 32:].double()


def unpack_act(a: torch.Tensor) -> torch.Tensor:
    """ACT -> float64 hi + lo (unpack2 adds them in fp32, which is exact for every split the kernels produce)."""
    hi, lo = act_hi_lo(a)
    return hi + lo


def act_bits(a: torch.Tensor) -> torch.Tensor:
    return a.contiguous().view(torch.int16)


# ------------------------------------------------------------------------------------------------- BatchNorm fold
def fold64(p: Dict[str, torch.Tensor], layer: int, eps: float, dev=None):
    """Conv + BatchNorm (eval) folded in float64 from the state dict: w' [co,ci,7,7], b' [co], and the bound on the fp32
    fold of b' (dec_fold_conv_kernel :119-120: s = gamma / sqrtf(var + eps) carries <= 2.5 U (add, sqrt, divide), then
    (b - mean) * s + beta: one subtraction, one multiply, one rounding of the (possibly fused) add)."""
    cv, bn = conv_bn_keys(layer)
    d = lambda k: p[k].to(dev).double()
    s = d(f"{bn}.weight") / torch.sqrt(d(f"{bn}.running_var") + eps)
    w = d(f"{cv}.weight") * s[:, None, None, None]
    bm = (d(f"{cv}.bias") - d(f"{bn}.running_mean")) * s
    b = bm + d(f"{bn}.bias")
    berr = 5.5 * U * bm.abs() + U * b.abs()
    return w, b, berr


def fold32(p: Dict[str, torch.Tensor], layer: int, eps: float, dev=None):
    """dec_fold_conv_kernel's fp32 result for an exact-family parameter set: fl(var + eps) = 1, gamma a power of two,
    mean = beta = 0, so s = gamma exactly and w' = w gamma, b' = b gamma with no rounding (asserted).  Returns w'
    [co,ci,7,7] float64, its bf16 hi / lo parts, b' [co]."""
    cv, bn = conv_bn_keys(layer)
    d = lambda k: p[k].to(dev).float()
    s32 = d(f"{bn}.weight") / torch.sqrt(d(f"{bn}.running_var") + torch.tensor(eps, dtype=torch.float32))
    assert torch.equal(s32, d(f"{bn}.weight")) and not d(f"{bn}.running_mean").any() and not d(f"{bn}.bias").any()
    w64 = d(f"{cv}.weight").double() * s32.double()[:, None, None, None]
    b64 = d(f"{cv}.bias").double() * s32.double()
    w32 = d(f"{cv}.weight") * s32[:, None, None, None]
    assert torch.equal(w32.double(), w64) and torch.equal(b64.float().double(), b64), "exact-family fold is not exact"
    hi = w32.to(torch.bfloat16)
    lo = (w32 - hi.float()).to(torch.bfloat16)
    assert torch.equal(hi.double() + lo.double(), w64), "exact-family weights must split exactly into two bf16"
    return w64, hi.double(), lo.double(), b64


def tap_matrix(w: torch.Tensor) -> torch.Tensor:
    """[co,ci,7,7] -> [7(dy),7(dx),ci,co]"""
    return w.permute(2, 3, 1, 0)


# ------------------------------------------------------------------------------ 7x7 conv in float64, by row bands
def conv7_bands(act: torch.Tensor, feats, mats: torch.Tensor, rows: Optional[Tuple[int, int]] = None,
                budget: int = 1 << 18) -> Iterator[Tuple[slice, slice, torch.Tensor]]:
    """out[b,y,x] = sum_{dy,dx} feats(act[b, y+dy-3, x+dx-3]) @ mats[dy,dx], zero outside the image (feats(0) = 0).
    act ACT [B,H,W,64]; feats(hi64, lo64) -> [...,K]; mats [7,7,K,N] float64.  Yields (images, rows, out [nb,R,W,N])
    over groups of whole small images or row bands of large ones (~`budget` output pixels each), so the float64
    working set stays small at any image size.  `rows` restricts the output to rows [y0, y1) of every image."""
    B, H, W, _ = act.shape
    y_lo, y_hi = rows if rows is not None else (0, H)
    span = y_hi - y_lo
    nb = max(1, min(B, budget // max(1, span * W)))
    R = span if nb > 1 else max(1, min(span, budget // W))
    for b0 in range(0, B, nb):
        b1 = min(B, b0 + nb)
        for y0 in range(y_lo, y_hi, R):
            y1 = min(y_hi, y0 + R)
            s0, s1 = max(0, y0 - 3), min(H, y1 + 3)
            hi, lo = act_hi_lo(act[b0:b1, s0:s1])
            f = feats(hi, lo)
            fp = f.new_zeros(b1 - b0, y1 - y0 + 6, W + 6, f.shape[-1])
            fp[:, s0 - (y0 - 3):s1 - (y0 - 3), 3:3 + W] = f
            out = f.new_zeros(b1 - b0, y1 - y0, W, mats.shape[-1])
            for dy in range(7):
                for dx in range(7):
                    out += fp[:, dy:dy + y1 - y0, dx:dx + W] @ mats[dy, dx]
            yield slice(b0, b1), slice(y0, y1), out


def _block_diag(*ms):
    """[7,7,k_i,n_i] blocks -> [7,7,sum k,sum n]"""
    K, N = sum(m.shape[2] for m in ms), sum(m.shape[3] for m in ms)
    out = ms[0].new_zeros(7, 7, K, N)
    k = n = 0
    for m in ms:
        out[:, :, k:k + m.shape[2], n:n + m.shape[3]] = m
        k, n = k + m.shape[2], n + m.shape[3]
    return out


# --------------------------------------------------------------------------------------------- bounded family
def conv7_bound_terms(impl: str, b64, berr, S, SL):
    """Bound on |conv + b' computed by the kernel - the float64 value|, before the residual, per entry.
    S = sum |a| |w'| and SL = sum |a_lo| |w'| over the entry's 49 x 32 terms (a = the input ACT's hi + lo, w' float64).
      fold      w_f32 = w' (1 + <= 3.5 U) (var + eps, sqrtf, divide, multiply: :124-125)          -> 4 U S
      tc only:  weight split |w_f32 - w_hi - w_lo| <= 2^-16 |w_f32|                               -> 2^-16 S
                dropped a_lo w_lo: |w_lo| <= 2^-8 (1 + 2^-8) |w_f32|                             -> 2^-8 (1 + 2^-7) SL
                accumulation: the accumulator starts at b' and receives 294 wgmma results (49 taps x 2 k-steps x 3
                products).  Assumed: one wgmma adds its 16 exact bf16 products to the fp32 accumulator with an error
                <= 2^-22 (|acc| + sum |products|) (any internal order, alignment and truncation: two fp32 ulps).  Every
                partial sum is <= |b'| + sum |a_hi w_hi| + |a_lo w_hi| + |a_hi w_lo| <= |b'| + (1 + 2^-6) S
                                                                                          -> 294 2^-22 (|b'| + 1.02 S)
      ref:      b' then <= 1568 sequential FMAs, one rounding each              -> 1568 U (|b'| + S)
      bias fold (fold64's berr)."""
    if impl == "ref":
        acc = N_FFMA * U * (b64.abs() + S * (1 + 4 * U))
        return 4 * U * S + acc + berr
    acc = N_MMA * MMA_ADD * (b64.abs() + 1.02 * S)
    return 4 * U * S + SPLIT * S * (1 + 4 * U) + 2.0 ** -8 * (1 + 2.0 ** -7) * SL + acc + berr


def sigmoid_bound(s64: torch.Tensor, bs: torch.Tensor) -> torch.Tensor:
    """|1 / (1 + expf(-s')) - sigmoid(s)| for |s' - s| <= bs: max sigmoid' over [s - bs, s + bs] times bs, plus expf
    (<= 2 ulp: relative 2^-22, moves sigma by sigma (1 - sigma) 2^-22), the add 1 + e and the correctly rounded
    division (2^-24 sigma each)."""
    lo, hi = s64 - bs, s64 + bs
    near0 = torch.where((lo <= 0) & (hi >= 0), torch.zeros_like(s64), torch.minimum(lo.abs(), hi.abs()))
    sg = torch.sigmoid(near0)
    dmax = sg * (1 - sg)
    sig = torch.sigmoid(s64)
    return (dmax * bs + 2.0 ** -22 * sig * (1 - sig) * (1 + bs) + 2.0 ** -23 * sig) * SLOP


def ratio(diff: torch.Tensor, bound: torch.Tensor) -> float:
    r = torch.where(bound > 0, diff / bound.clamp_min(1e-300), torch.where(diff > 0, math.inf, 0.0))
    return float(r.max()) if r.numel() else 0.0


class Worst:
    """Worst ratio of |got - float64| to the per-entry bound over the bands of one layer."""

    def __init__(self):
        self.r = 0.0
        self.n = 0

    def add(self, diff, bound):
        self.r = max(self.r, ratio(diff, bound))
        self.n += diff.numel()


def check_conv7_bounded(p, eps, layer, impl, x_act, res_act, got, rows=None, corrupt=None) -> Worst:
    """The 7x7 layer `layer` run by `impl` on its own input x_act (and residual res_act) produced `got` (ACT, or fp32 rgb
    for layer 9): every entry within its bound of float64.  `corrupt` (self-tests only) perturbs the float64 side."""
    dev = x_act.device
    w64, b64, berr = fold64(p, layer, eps, dev)
    if corrupt and corrupt.get("fold"):
        w64, b64, berr = corrupt["fold"](p, layer, eps, dev)
    m = tap_matrix(w64)
    if corrupt and corrupt.get("taps"):
        m = corrupt["taps"](m)
    mats = _block_diag(m, m.abs(), m.abs())
    feats = lambda hi, lo: torch.cat([hi + lo, (hi + lo).abs(), lo.abs()], -1)
    src = corrupt["input"](x_act) if corrupt and corrupt.get("input") else x_act
    worst = Worst()
    for bs, ys, out in conv7_bands(src, feats, mats, rows):
        v, S, SL = out[..., :32] + b64, out[..., 32:64], out[..., 64:]
        err = conv7_bound_terms(impl, b64, berr, S, SL)
        if layer in RES_LAYERS and not (corrupt and corrupt.get("no_residual")):
            v = v + unpack_act(res_act[bs, ys])
            err = err + U * (v.abs() + err)  # the residual add: one fp32 rounding
        y = v.clamp_min(0)
        if layer == 9:
            ow = p[f"{PREFIX}.7.weight"].to(dev).double().reshape(3, 32)
            ob = p[f"{PREFIX}.7.bias"].to(dev).double()
            if corrupt and corrupt.get("no_out_bias"):
                ob = ob * 0
            s = y @ ow.T + ob
            # the per-lane FMA chains, two shuffle adds and + out_b (tc) or out_b then 32 FMAs (ref): <= 33 roundings
            bs_ = err @ ow.abs().T
            bs_ = (bs_ + 33 * U * (ob.abs() + (y + err) @ ow.abs().T)) * SLOP
            worst.add((got[bs, ys].double() - torch.sigmoid(s)).abs(), sigmoid_bound(s, bs_))
        else:
            bound = (err + SPLIT * (y.abs() + err)) * SLOP
            worst.add((unpack_act(got[bs, ys]) - y).abs(), bound)
    return worst


def _row_chunks(n_rows: int, per_row: int, budget: int = 1 << 18):
    step = max(1, budget // max(1, per_row))
    for r0 in range(0, n_rows, step):
        yield slice(r0, min(n_rows, r0 + step))


def check_input_bounded(p, feats: torch.Tensor, got: torch.Tensor, corrupt=None) -> Worst:
    """Layer 0 (dec_input_kernel): v = b + sum_c x_c w_kc as b then in_dim FMAs, ReLU, split."""
    dev = feats.device
    w = p[f"{PREFIX}.0.weight"].to(dev).double().reshape(32, -1)
    b = p[f"{PREFIX}.0.bias"].to(dev).double()
    if corrupt and corrupt.get("no_bias"):
        b = b * 0
    x, g = feats.reshape(-1, feats.shape[-1]), got.reshape(-1, 64)
    worst = Worst()
    for sl in _row_chunks(x.shape[0], 1):
        xd = x[sl].double()
        v, S = xd @ w.T + b, xd.abs() @ w.abs().T
        err = (w.shape[1] + 1) * U * (b.abs() + S)
        y = v.clamp_min(0)
        worst.add((unpack_act(g[sl]) - y).abs(), (err + SPLIT * (y + err)) * SLOP)
    return worst


def upsample64(p, a: torch.Tensor, dev):
    """ConvTranspose2d k = s = 3 on input pixels a [n,32] float64 -> value and sum |terms|, [n,3,3,32] (i, j, co)."""
    w = p[f"{PREFIX}.4.weight"].to(dev).double()  # [ci,co,3,3]
    b = p[f"{PREFIX}.4.bias"].to(dev).double()
    wm = w.permute(0, 2, 3, 1).reshape(32, 9 * 32)
    v = (a @ wm).reshape(-1, 3, 3, 32) + b
    S = (a.abs() @ wm.abs()).reshape(-1, 3, 3, 32) + b.abs()
    return v, S


def check_upsample_bounded(p, x_act: torch.Tensor, got: torch.Tensor, corrupt=None) -> Worst:
    """Layer 5 (dec_upsample_kernel): b then 32 FMAs per output entry, no ReLU, split."""
    dev = x_act.device
    B, H, W, _ = x_act.shape
    worst = Worst()
    for b in range(B):
        for ys in _row_chunks(H, W):
            a = unpack_act(x_act[b, ys]).reshape(-1, 32)
            v, S = upsample64(p, a, dev)
            n = ys.stop - ys.start
            v = v.reshape(n, W, 3, 3, 32).permute(0, 2, 1, 3, 4).reshape(3 * n, 3 * W, 32)
            S = S.reshape(n, W, 3, 3, 32).permute(0, 2, 1, 3, 4).reshape(3 * n, 3 * W, 32)
            if corrupt and corrupt.get("transpose"):
                v = v.reshape(n, 3, W, 3, 32).transpose(1, 3).reshape(3 * n, 3 * W, 32)
            err = 33 * U * S
            g = unpack_act(got[b, 3 * ys.start:3 * ys.stop])
            worst.add((g - v).abs(), (err + SPLIT * (v.abs() + err)) * SLOP)
    return worst


# ------------------------------------------------------------------------------------------------ exact family
def exact_act_ok(v: torch.Tensor) -> torch.Tensor:
    return v.float().double() == v


def predict_conv7_exact(p, eps, layer, impl, x_act, res_act, quantum: float, rows=None, drop_chunk=None):
    """Bit-exact prediction of layer `layer` by `impl` (ACT, or the exact fp32 logits [..,3] for layer 9), band by band:
    yields (images, rows, prediction).  tc / tc_ldgsts: conv(A, W') - conv(A_lo, W'_lo); ref: conv(A, W').
    Asserts the case is exact: every |partial sum| < 2^24 quantum (quantum: a power of two dividing every term).
    `drop_chunk` = c predicts a kernel that also drops a_lo*w_hi of input channels 8c..8c+7 (self-tests)."""
    dev = x_act.device
    w64, whi, wlo, b64 = fold32(p, layer, eps, dev)
    m, mlo, mabs = tap_matrix(w64), tap_matrix(wlo), tap_matrix(whi.abs() + wlo.abs())
    # features [a, a_lo, |a_hi|, |a_lo|] -> columns [value | sum of |terms| (the exactness certificate)]
    mats = w64.new_zeros(7, 7, 128, 64)
    mats[:, :, 0:32, 0:32] = m
    if impl != "ref":
        mats[:, :, 32:64, 0:32] = -mlo
    if drop_chunk is not None:
        mh = tap_matrix(whi)
        mats[:, :, 32 + 8 * drop_chunk:40 + 8 * drop_chunk, 0:32] -= mh[:, :, 8 * drop_chunk:8 * drop_chunk + 8]
    mats[:, :, 64:96, 32:64] = mabs
    mats[:, :, 96:128, 32:64] = mabs
    feats = lambda hi, lo: torch.cat([hi + lo, lo, hi.abs(), lo.abs()], -1)
    for bs, ys, out in conv7_bands(x_act, feats, mats, rows):
        v, cert = out[..., :32] + b64, out[..., 32:] + b64.abs()
        if layer in RES_LAYERS:
            r = unpack_act(res_act[bs, ys])
            v, cert = v + r, cert + r.abs()
        assert bool((cert < 2.0 ** 24 * quantum).all()), "exact case leaves the exact range"
        assert bool(exact_act_ok(v).all())
        y = v.clamp_min(0)
        if layer == 9:
            ow = p[f"{PREFIX}.7.weight"].to(dev).double().reshape(3, 32)
            ob = p[f"{PREFIX}.7.bias"].to(dev).double()
            s = y @ ow.T + ob
            assert bool(exact_act_ok(s).all()) and bool(((y @ ow.abs().T + ob.abs()) < 2.0 ** 24 * 2.0 ** -18).all())
            yield bs, ys, s
        else:
            yield bs, ys, pack_act(y.float())


def predict_input_exact(p, feats: torch.Tensor) -> torch.Tensor:
    w = p[f"{PREFIX}.0.weight"].to(feats.device).double().reshape(32, -1)
    b = p[f"{PREFIX}.0.bias"].to(feats.device).double()
    x = feats.double()
    v = x @ w.T + b
    assert bool(((x.abs() @ w.abs().T + b.abs()) < 2.0 ** 24).all()) and bool(exact_act_ok(v).all())
    return pack_act(v.clamp_min(0).float())


def predict_upsample_exact(p, x_act: torch.Tensor) -> torch.Tensor:
    B, H, W, _ = x_act.shape
    v, S = upsample64(p, unpack_act(x_act).reshape(-1, 32), x_act.device)
    assert bool((S < 2.0 ** 24).all()) and bool(exact_act_ok(v).all())
    v = v.reshape(B, H, W, 3, 3, 32).permute(0, 1, 3, 2, 4, 5).reshape(B, 3 * H, 3 * W, 32)
    return pack_act(v.float())
