"""CPU: the ACT helpers of tests/rgb_decoder_cases.py against a bit-level numpy model of split_pack2 / unpack2, the exact
predictor's three- vs four-product forms, and comparator self-tests: every comparator of the GPU file
(tests/test_zz_rgb_decoder_stages_gpu.py) accepts a correct fp32 result and rejects corrupted ones."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import decoder_oracle as D
from tests import rgb_decoder_cases as R

EXACT_EPS = 2.0 ** -30


# --------------------------------------------------------------------------------------------------- ACT helpers
def np_bf16_rn(f32):
    """bf16 bits of fp32 values, round to nearest even (what __floats2bfloat162_rn does for finite values)."""
    u = f32.astype(np.float32).view(np.uint32).astype(np.uint64)
    return ((u + 0x7FFF + ((u >> 16) & 1)) >> 16).astype(np.uint16)


def np_split_pack2(v):
    hi = np_bf16_rn(v)
    rest = (v.astype(np.float32) - (hi.astype(np.uint32) << 16).view(np.float32)).astype(np.float32)
    return hi, np_bf16_rn(rest)


def np_unpack2(hi, lo):
    return (hi.astype(np.uint32) << 16).view(np.float32) + (lo.astype(np.uint32) << 16).view(np.float32)


def test_act_pack_matches_split_pack2_model():
    g = np.random.default_rng(0)
    v = np.concatenate([
        g.standard_normal(4096).astype(np.float32) * 10.0 ** g.integers(-6, 6, 4096),
        # ties of the hi rounding: 1 + 2^-8 rounds to 1 (even), 1 + 3 2^-8 to 1 + 2^-6; and of the lo rounding
        np.array([1 + 2 ** -8, 1 + 3 * 2 ** -8, -(1 + 2 ** -8), 256 + 1, 256 + 3, 1 + 2 ** -8 + 2 ** -17, 1 + 2 ** -16 + 2 ** -24,
                  1 + 3 * 2 ** -16 + 2 ** -23, 0.0, -0.0, 2.0 ** -130, 65504.0, 3.0e38], dtype=np.float32)])
    v = np.resize(v, (v.size + 31) // 32 * 32).reshape(-1, 32)
    act = R.pack_act(torch.from_numpy(v))
    hi, lo = np_split_pack2(v)
    bits = act.view(torch.int16).numpy().view(np.uint16)
    assert np.array_equal(bits[:, :32], hi) and np.array_equal(bits[:, 32:], lo)
    assert np.array_equal(R.unpack_act(act).numpy(), np_unpack2(hi, lo).astype(np.float64))
    # the tie cases landed where round-to-nearest-even puts them
    t = R.pack_act(torch.tensor([[1 + 2 ** -8, 1 + 3 * 2 ** -8] + [0.0] * 30]))
    assert t[0, 0].item() == 1.0 and t[0, 1].item() == 1 + 2 ** -6
    # |v - hi - lo| <= 2^-16 |v|
    rel = np.abs(R.unpack_act(act).numpy() - v.astype(np.float64)) / np.maximum(np.abs(v.astype(np.float64)), 1e-300)
    assert rel[np.isfinite(v) & (np.abs(v) > 2.0 ** -100)].max() <= R.SPLIT


# ------------------------------------------------------------------------------------------------ small fixtures
def exact_params_cpu(seed, wmax=300, gamma=1.0):
    g = torch.Generator().manual_seed(seed)
    ri = lambda lo, hi, shape: torch.randint(lo, hi + 1, shape, generator=g).float()
    p = D.random_decoder_params(seed)
    for blk in R.BLOCKS:
        for cv, bn in ((0, 1), (3, 4)):
            m = f"{R.PREFIX}.{blk}.main_branch"
            p[f"{m}.{cv}.weight"] = ri(-wmax, wmax, (32, 32, 7, 7)) * (torch.rand(32, 32, 7, 7, generator=g) < 0.05)
            p[f"{m}.{cv}.bias"] = ri(-8, 8, (32,))
            p[f"{m}.{bn}.weight"] = torch.full((32,), gamma)
            p[f"{m}.{bn}.bias"] = torch.zeros(32)
            p[f"{m}.{bn}.running_mean"] = torch.zeros(32)
            p[f"{m}.{bn}.running_var"] = torch.ones(32)
    p[f"{R.PREFIX}.7.weight"] = ri(-2, 2, (3, 32, 1, 1)) * 2.0 ** -18
    p[f"{R.PREFIX}.7.bias"] = ri(-2 ** 16, 2 ** 16, (3,)) * 2.0 ** -18
    return p


def exact_act_cpu(seed, shape):
    g = torch.Generator().manual_seed(seed)
    n = tuple(shape) + (32,)
    hi = torch.randint(-16, 17, n, generator=g).float() * 16
    lo = torch.randint(-7, 8, n, generator=g).float()
    return torch.cat([hi.bfloat16(), lo.bfloat16()], -1)


def predicted(p, layer, impl, x, res, **kw):
    out = None
    for bs, ys, pred in R.predict_conv7_exact(p, EXACT_EPS, layer, impl, x, res, 1.0, **kw):
        if out is None:
            out = torch.empty(x.shape[:3] + pred.shape[-1:], dtype=pred.dtype)
        out[bs, ys] = pred
    return out


def test_exact_predictor_three_vs_four_products():
    """Both operands with lo parts: the tensor-core form (a_lo w_lo dropped) and the CUDA-core form really differ,
    and the difference is exactly conv(A_lo, W_lo)."""
    p = exact_params_cpu(1)
    x, res = exact_act_cpu(2, (2, 6, 10)), exact_act_cpu(3, (2, 6, 10))
    tc, ref = predicted(p, 2, "tc", x, res), predicted(p, 2, "ref", x, res)
    assert not torch.equal(R.act_bits(tc), R.act_bits(ref))
    _, _, wlo, _ = R.fold32(p, 2, EXACT_EPS)
    xl = x[..., 32:].double().permute(0, 3, 1, 2)
    lolo = F.conv2d(xl, wlo, padding=3).permute(0, 2, 3, 1)
    v_tc, v_ref = R.unpack_act(tc), R.unpack_act(ref)
    both = (v_tc > 0) & (v_ref > 0) & (v_ref.abs() < 256)  # exact ACT (8 + 8 bits) and ReLU inactive
    assert bool(both.any()) and torch.equal(v_ref[both] - v_tc[both], lolo[both])


def fp32_conv_layer(p, layer, x, res, eps=1e-5, fold=None, shift_tap=False, seam=False, no_res=False):
    """A correct (or deliberately wrong) fp32 computation of a 7x7 layer on the CPU -> ACT."""
    cv, bn = R.conv_bn_keys(layer)
    if fold is None:
        s = p[f"{bn}.weight"] / torch.sqrt(p[f"{bn}.running_var"] + eps)
        w = p[f"{cv}.weight"] * s[:, None, None, None]
        b = (p[f"{cv}.bias"] - p[f"{bn}.running_mean"]) * s + p[f"{bn}.bias"]
    else:
        w, b = fold
    if shift_tap:
        w = torch.roll(w, 1, dims=3)
    a = R.unpack_act(x).float().permute(0, 3, 1, 2)
    if seam:  # images stacked vertically: image b's bottom padding rows read image b + 1
        B, C, H, W = a.shape
        v = F.conv2d(a.permute(1, 0, 2, 3).reshape(1, C, B * H, W), w, b, padding=3)
        v = v.reshape(C, B, H, W).permute(1, 0, 2, 3)
    else:
        v = F.conv2d(a, w, b, padding=3)
    v = v.permute(0, 2, 3, 1)
    if layer in R.RES_LAYERS and not no_res:
        v = v + R.unpack_act(res).float()
    return v.clamp_min(0)


@pytest.fixture(scope="module")
def tiny_var_params():
    p = D.random_decoder_params(7)
    g = torch.Generator().manual_seed(8)
    for blk in R.BLOCKS:
        for cv, bn in ((0, 1), (3, 4)):
            m = f"{R.PREFIX}.{blk}.main_branch"
            p[f"{m}.{cv}.weight"] = p[f"{m}.{cv}.weight"] * 0.01
            p[f"{m}.{cv}.bias"] = p[f"{m}.{cv}.bias"] * 0.01
            p[f"{m}.{bn}.running_var"] = torch.rand(32, generator=g) * 1e-4 + 5e-5
            p[f"{m}.{bn}.running_mean"] = torch.randn(32, generator=g) * 0.02
            p[f"{m}.{bn}.weight"] = -(torch.rand(32, generator=g) * 0.8 + 0.6)
    return p


def layer_input(seed, shape=(3, 6, 12)):
    g = torch.Generator().manual_seed(seed)
    return R.pack_act(torch.randn(*shape, 32, generator=g).clamp_min(0)), R.pack_act(torch.randn(*shape, 32, generator=g).clamp_min(0))


@pytest.mark.parametrize("pset", ["random", "tiny_var"])
@pytest.mark.parametrize("layer", [1, 2])
def test_bounded_conv_comparator_accepts_fp32_and_rejects_corruptions(tiny_var_params, pset, layer):
    p = D.random_decoder_params(5) if pset == "random" else tiny_var_params
    x, res = layer_input(9)
    r = res if layer in R.RES_LAYERS else None
    check = lambda got, impl="tc", **c: R.check_conv7_bounded(p, 1e-5, layer, impl, x, r, got, corrupt=c or None).r
    good = R.pack_act(fp32_conv_layer(p, layer, x, r))
    for impl in R.IMPLS:
        assert check(good, impl) <= 1.0, impl
    assert check(R.pack_act(fp32_conv_layer(p, layer, x, r, shift_tap=True))) > 1.0
    assert check(R.pack_act(fp32_conv_layer(p, layer, x, r, seam=True))) > 1.0
    if layer in R.RES_LAYERS:
        assert check(R.pack_act(fp32_conv_layer(p, layer, x, r, no_res=True))) > 1.0
    cv, bn = R.conv_bn_keys(layer)
    if pset == "tiny_var":  # the BatchNorm statistics matter at this scale
        s = p[f"{bn}.weight"] / torch.sqrt(p[f"{bn}.running_var"] + 1e-5)
        no_mean = (p[f"{cv}.weight"] * s[:, None, None, None], p[f"{cv}.bias"] * s + p[f"{bn}.bias"])
        assert check(R.pack_act(fp32_conv_layer(p, layer, x, r, fold=no_mean))) > 1.0
        s0 = p[f"{bn}.weight"] / torch.sqrt(p[f"{bn}.running_var"])
        no_eps = (p[f"{cv}.weight"] * s0[:, None, None, None], (p[f"{cv}.bias"] - p[f"{bn}.running_mean"]) * s0 + p[f"{bn}.bias"])
        assert check(R.pack_act(fp32_conv_layer(p, layer, x, r, fold=no_eps))) > 1.0


def test_bounded_rgb_comparator(tiny_var_params):
    p = D.random_decoder_params(5)
    x, res = layer_input(10)
    v = fp32_conv_layer(p, 9, x, res)
    ow, ob = p[f"{R.PREFIX}.7.weight"].reshape(3, 32), p[f"{R.PREFIX}.7.bias"]
    good = torch.sigmoid(v @ ow.T + ob)
    for impl in R.IMPLS:
        assert R.check_conv7_bounded(p, 1e-5, 9, impl, x, res, good).r <= 1.0
    assert R.check_conv7_bounded(p, 1e-5, 9, "tc", x, res, torch.sigmoid(v @ ow.T)).r > 1.0  # out-conv bias missing
    assert R.check_conv7_bounded(p, 1e-5, 9, "tc", x, res, torch.sigmoid(fp32_conv_layer(p, 9, x, res, no_res=True) @ ow.T + ob)).r > 1.0


def test_bounded_input_and_upsample_comparators():
    p = D.random_decoder_params(5)
    g = torch.Generator().manual_seed(11)
    f = torch.randn(2, 5, 7, 48, generator=g)
    w, b = p[f"{R.PREFIX}.0.weight"].reshape(32, 48), p[f"{R.PREFIX}.0.bias"]
    good = R.pack_act((f @ w.T + b).clamp_min(0))
    assert R.check_input_bounded(p, f, good).r <= 1.0
    assert R.check_input_bounded(p, f, R.pack_act((f @ w.T).clamp_min(0))).r > 1.0  # bias missing
    x, _ = layer_input(12, (2, 5, 7))
    a = R.unpack_act(x).float().permute(0, 3, 1, 2)
    up = F.conv_transpose2d(a, p[f"{R.PREFIX}.4.weight"], p[f"{R.PREFIX}.4.bias"], stride=3).permute(0, 2, 3, 1)
    assert R.check_upsample_bounded(p, x, R.pack_act(up)).r <= 1.0
    assert R.check_upsample_bounded(p, x, R.pack_act(up.transpose(1, 2).reshape(up.shape).contiguous())).r > 1.0
    upt = F.conv_transpose2d(a, p[f"{R.PREFIX}.4.weight"].transpose(2, 3), p[f"{R.PREFIX}.4.bias"], stride=3).permute(0, 2, 3, 1)
    assert R.check_upsample_bounded(p, x, R.pack_act(upt)).r > 1.0  # kernel taps (i, j) swapped


def test_exact_comparator_rejects_one_ulp_and_a_dropped_chunk():
    p = exact_params_cpu(13)
    x, res = exact_act_cpu(14, (2, 6, 10)), exact_act_cpu(15, (2, 6, 10))
    tc = predicted(p, 2, "tc", x, res)
    bits = R.act_bits(tc).clone()
    nz = (bits[..., :32] != 0).nonzero()[0].tolist()
    bits[tuple(nz)] += 1  # one ulp of one hi entry
    assert not torch.equal(bits, R.act_bits(tc))
    for c in range(4):  # the a_lo * w_hi products of one 8-channel chunk dropped: visible in the exact family
        assert not torch.equal(R.act_bits(predicted(p, 2, "tc", x, res, drop_chunk=c)), R.act_bits(tc)), c


def test_bounded_comparator_sees_a_dropped_chunk_on_realistic_data():
    """One chunk's a_lo * w_hi dropped on realistic data.  It is ~3e-5 of sum |a||w|, under the accumulation term, but
    the bound's lo * lo term is taken from the input's actual |a_lo| (2^-8 of it), and the dropped products are 2^8
    times that: the bounded comparator rejects it too (the exact family carries the detection in any case)."""
    p = D.random_decoder_params(5)
    x, _ = layer_input(16)
    cv, bn = R.conv_bn_keys(1)
    s = p[f"{bn}.weight"] / torch.sqrt(p[f"{bn}.running_var"] + 1e-5)
    w = p[f"{cv}.weight"] * s[:, None, None, None]
    b = (p[f"{cv}.bias"] - p[f"{bn}.running_mean"]) * s + p[f"{bn}.bias"]
    whi = w.bfloat16().float()
    lo = x[..., 32:].float().permute(0, 3, 1, 2)
    lo[:, 8:] = 0
    a = R.unpack_act(x).float().permute(0, 3, 1, 2)
    dropped = (F.conv2d(a, w, b, padding=3) - F.conv2d(lo, whi, padding=3)).permute(0, 2, 3, 1).clamp_min(0)
    assert R.check_conv7_bounded(p, 1e-5, 1, "tc", x, None, R.pack_act(dropped)).r > 1.0
