"""GPU: the camera rgb decoder layer by layer (b200nerf_rgb_decode_layer), every entry of every layer of all three
implementations:
* exact family: integer / dyadic parameters and host-built ACT inputs, predicted bit for bit (tests/rgb_decoder_cases.py);
* bounded family: realistic parameters, each layer on the ACT the previous layer call produced from real features,
  against float64 with one bound per entry derived from the code;
* composition: rgb_decode == the ten layer calls, tc == tc_ldgsts, batch-composition independence, and the output of
  rgb_decode on seeded inputs pinned to its SHA-256 (the kernels' results must not move)."""
import hashlib

import pytest
import torch

from oracle import decoder_oracle as D
from tests import rgb_decoder_cases as R

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
EXACT_EPS = 2.0 ** -30  # fl(1 + eps) = 1 in fp32: the BatchNorm fold is exact
WORST = {}  # (param set, layer, impl) -> worst ratio to the bound, printed by test_zzz_report


@pytest.fixture(scope="module")
def be():
    from neurad_studio_b200.nerfstudio_api import get_backend

    b = get_backend(DEV)
    yield b
    b._dec_ws = None
    torch.cuda.empty_cache()


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _ri(g, lo, hi, shape, scale=1.0):
    return torch.randint(lo, hi + 1, shape, generator=g, device=DEV).float() * scale


# ------------------------------------------------------------------------------------------------ exact family
def exact_params(seed, wkind, gamma=1.0, in_dim=48):
    """Integer parameters: BatchNorm gamma a power of two, beta = mean = 0, var = 1 (with EXACT_EPS: s = gamma)."""
    g = _gen(seed)
    p = {}
    p[f"{R.PREFIX}.0.weight"] = _ri(g, -1, 1, (32, in_dim, 1, 1))
    p[f"{R.PREFIX}.0.bias"] = _ri(g, -2, 2, (32,))
    for blk in R.BLOCKS:
        for cv, bn in ((0, 1), (3, 4)):
            m = f"{R.PREFIX}.{blk}.main_branch"
            if wkind == "small":  # A carries the lo parts
                w = _ri(g, -2, 2, (32, 32, 7, 7))
            elif wkind == "lo":  # 11-bit integers: W' has hi and lo parts; A is small
                w = _ri(g, -1000, 1000, (32, 32, 7, 7))
            elif wkind == "sparse_lo":  # both have lo parts, W only on 4 taps per output channel
                w = _ri(g, -300, 300, (32, 32, 7, 7))
                taps = torch.rand(32, 49, generator=g, device=DEV).argsort(1)[:, :4]
                mask = torch.zeros(32, 49, device=DEV).scatter_(1, taps, 1.0)
                w = w * mask.reshape(32, 1, 7, 7)
            elif wkind == "pos":  # large positive outputs: more than 16 significant bits
                w = _ri(g, 0, 2, (32, 32, 7, 7))
            elif wkind == "chain":  # two nonzero taps per output channel: the ten-layer chain stays exact
                w = torch.zeros(32, 32 * 49, device=DEV)
                idx = torch.rand(32, 32 * 49, generator=g, device=DEV).argsort(1)[:, :2]
                w.scatter_(1, idx, _ri(g, 1, 2, (32, 2)) * (_ri(g, 0, 1, (32, 2)) * 2 - 1))
                w = w.reshape(32, 32, 7, 7)
            p[f"{m}.{cv}.weight"], p[f"{m}.{cv}.bias"] = w, _ri(g, -8, 8, (32,))
            p[f"{m}.{bn}.weight"] = torch.full((32,), gamma, device=DEV)
            p[f"{m}.{bn}.bias"] = torch.zeros(32, device=DEV)
            p[f"{m}.{bn}.running_mean"] = torch.zeros(32, device=DEV)
            p[f"{m}.{bn}.running_var"] = torch.ones(32, device=DEV)
    up = _ri(g, -1, 1, (32, 32, 3, 3))
    p[f"{R.PREFIX}.4.weight"] = up * (torch.rand(up.shape, generator=g, device=DEV) < 0.15) if wkind == "chain" else up
    p[f"{R.PREFIX}.4.bias"] = _ri(g, -2, 2, (32,))
    p[f"{R.PREFIX}.7.weight"] = _ri(g, -2, 2, (3, 32, 1, 1), 2.0 ** -18)  # dyadic logits, |logit| < 64
    p[f"{R.PREFIX}.7.bias"] = _ri(g, -2 ** 16, 2 ** 16, (3,), 2.0 ** -18)
    return p


def exact_act(g, shape, kind):
    """Host-built ACT [*shape, 64] whose hi and lo are exact bf16 integers (not necessarily an RN split)."""
    n = tuple(shape) + (32,)
    hi, lo = {"lo": (_ri(g, -255, 255, n, 4.0), _ri(g, -3, 3, n)),
              "small": (_ri(g, -3, 3, n), torch.zeros(n, device=DEV)),
              "sparse_lo": (_ri(g, -16, 16, n, 16.0), _ri(g, -7, 7, n)),
              "pos": (_ri(g, 0, 255, n, 4.0), _ri(g, 0, 3, n))}[kind]
    return torch.cat([hi.bfloat16(), lo.bfloat16()], -1)


# (weight kind, input kind, gamma, quantum of every term)
EXACT_CASES = {"a_lo_w_small": ("small", "lo", 1.0, 1.0), "w_lo_a_small": ("lo", "small", 2.0, 1.0),
               "both_lo_sparse": ("sparse_lo", "sparse_lo", 1.0, 1.0), "wide_outputs": ("pos", "pos", 1.0, 1.0),
               "half_gamma": ("small", "lo", 0.5, 0.5)}
# layer-input (H, W, batch); (76, 100, 7) is 133 tiles: one more than the H100's 132 SMs, a ragged second round
SHAPES = [(1, 1, 4096), (2, 3, 1), (4, 4, 2), (5, 7, 3), (11, 11, 64), (32, 32, 16), (3, 127, 2), (4, 128, 2), (4, 129, 2),
          (5, 257, 2), (19, 45, 2), (13, 300, 2), (76, 100, 7)]


def run_layer(be, layer, x, res, impl):
    out = be.rgb_decode_layer(layer, x, res, impl)
    torch.cuda.synchronize()
    be.check_status()
    return out


def assert_exact(p, eps, layer, impl, x, res, got, quantum, what):
    n = 0
    for bs, ys, pred in R.predict_conv7_exact(p, eps, layer, impl, x, res, quantum):
        if layer == 9:
            s = pred
            bound = R.sigmoid_bound(s, torch.zeros_like(s))
            r = R.ratio((got[bs, ys].double() - torch.sigmoid(s)).abs(), bound)
            assert r <= 1.0, (what, layer, impl, r)
        else:
            bad = R.act_bits(got[bs, ys]) != R.act_bits(pred)
            assert not bool(bad.any()), (what, layer, impl, int(bad.sum()), bad.nonzero()[:4].tolist())
        n += pred.numel()
    return n


@pytest.mark.parametrize("case", list(EXACT_CASES))
def test_conv7_exact_bit_for_bit(be, case):
    wkind, akind, gamma, q = EXACT_CASES[case]
    p = exact_params(11, wkind, gamma)
    be.set_rgb_decoder(p, bn_eps=EXACT_EPS)
    g = _gen(12)
    for (h, w, b) in SHAPES:
        x = exact_act(g, (b, h, w), akind)
        res = exact_act(g, (b, h, w), "small")
        # the rgb head's logit cannot stay exact on activations with more than 16 significant bits
        for layer in (1, 2) if case == "wide_outputs" else (1, 2, 9):
            r = res if layer in R.RES_LAYERS else None
            outs = {impl: run_layer(be, layer, x, r, impl) for impl in R.IMPLS}
            assert torch.equal(outs["tc"], outs["tc_ldgsts"]), (case, h, w, b, layer)
            for impl in R.IMPLS:
                assert_exact(p, EXACT_EPS, layer, impl, x, r, outs[impl], q, (case, h, w, b))
    WORST[("exact " + case, "1,2" if case == "wide_outputs" else "1,2,9", "all")] = "bit-exact"


def test_conv7_exact_deltas(be):
    """One-hot inputs: corners, x = 127 / 128 / 129, tile rows y = 3 / 4, the last row of image b next to image b + 1
    (its taps must not reach image b + 1's first row).  Pins tap orientation, zero padding and image seams."""
    p = exact_params(21, "lo", 1.0)
    be.set_rgb_decoder(p, bn_eps=EXACT_EPS)
    H, W = 9, 260
    pos = [(0, 0), (0, W - 1), (H - 1, 0), (H - 1, W - 1), (5, 127), (5, 128), (5, 129), (3, 60), (4, 60), (H - 1, 128),
           (H - 1, 200), (0, 255), (0, 256)]
    g = _gen(22)
    x = torch.zeros(len(pos), H, W, 64, dtype=torch.bfloat16, device=DEV)
    for i, (y, xx) in enumerate(pos):
        x[i, y, xx] = exact_act(g, (1,), "sparse_lo")[0]
    res = exact_act(g, (len(pos), H, W), "small")
    for layer in (1, 2, 9):
        r = res if layer in R.RES_LAYERS else None
        for impl in R.IMPLS:
            assert_exact(p, EXACT_EPS, layer, impl, x, r, run_layer(be, layer, x, r, impl), 1.0, "delta")
    WORST[("exact deltas", "1,2,9", "all")] = "bit-exact"


@pytest.mark.parametrize("in_dim", [1, 17, 48, 64])
def test_input_and_upsample_exact(be, in_dim):
    p = exact_params(31 + in_dim, "small", 1.0, in_dim)
    be.set_rgb_decoder(p, bn_eps=EXACT_EPS)
    g = _gen(32)
    for (h, w, b) in SHAPES:
        f = _ri(g, -3, 3, (b, h, w, in_dim))
        a0 = run_layer(be, 0, f, None, "tc")
        assert torch.equal(R.act_bits(a0), R.act_bits(R.predict_input_exact(p, f))), (in_dim, h, w, b)
        x = exact_act(g, (b, h, w), "lo")
        up = run_layer(be, 5, x, None, "tc")
        assert up.shape == (b, 3 * h, 3 * w, 64)
        assert torch.equal(R.act_bits(up), R.act_bits(R.predict_upsample_exact(p, x))), (in_dim, h, w, b)
    WORST[(f"exact in_dim {in_dim}", "0,5", "all")] = "bit-exact"


@pytest.mark.parametrize("impl", R.IMPLS)
def test_ten_layer_chain_exact(be, impl):
    """The whole chain on exact parameters: every layer bit for bit on the kernel's own input (so the chain of
    predictions is the kernels' chain), and rgb_decode equal to the ten calls."""
    p = exact_params(41, "chain", 1.0)
    be.set_rgb_decoder(p, bn_eps=EXACT_EPS)
    g = _gen(42)
    for (h, w, b) in [(19, 45, 2), (4, 129, 2), (1, 1, 64), (76, 100, 7)]:
        f = _ri(g, 0, 3, (b, h, w, 48))
        acts = [run_layer(be, 0, f, None, impl)]
        assert torch.equal(R.act_bits(acts[0]), R.act_bits(R.predict_input_exact(p, f)))
        for layer in range(1, 10):
            x = acts[-1]
            res = acts[-2] if layer in R.RES_LAYERS else None
            out = run_layer(be, layer, x, res, impl)
            if layer == 5:
                assert torch.equal(R.act_bits(out), R.act_bits(R.predict_upsample_exact(p, x)))
            else:
                assert_exact(p, EXACT_EPS, layer, impl, x, res, out, 1.0, ("chain", h, w, b))
            acts.append(out)
        rgb = be.rgb_decode(f, impl)
        torch.cuda.synchronize()
        assert torch.equal(rgb, acts[-1]), (impl, h, w, b)
    WORST[("exact chain", "0-9", impl)] = "bit-exact"


# ---------------------------------------------------------------------------------------------- bounded family
def extreme_params(seed):
    """Tiny running_var (s ~ 100), means large against the conv outputs, mixed-sign gamma; conv weights scaled down
    by the same 100 so the activations stay O(1) through the chain."""
    p = D.random_decoder_params(seed)
    g = torch.Generator().manual_seed(seed + 1)
    for blk in R.BLOCKS:
        for cv, bn in ((0, 1), (3, 4)):
            m = f"{R.PREFIX}.{blk}.main_branch"
            p[f"{m}.{cv}.weight"] = p[f"{m}.{cv}.weight"] * 0.01
            p[f"{m}.{cv}.bias"] = p[f"{m}.{cv}.bias"] * 0.01
            p[f"{m}.{bn}.running_var"] = torch.rand(32, generator=g) * 1e-4 + 5e-5
            p[f"{m}.{bn}.running_mean"] = torch.randn(32, generator=g) * 0.02
            p[f"{m}.{bn}.weight"] = (torch.rand(32, generator=g) * 0.8 + 0.6) * torch.where(torch.rand(32, generator=g) < 0.5, -1.0, 1.0)
    return p


PARAM_SETS = {"random": lambda: D.random_decoder_params(seed=51), "tiny_var": lambda: extreme_params(52)}
BOUNDED_SHAPES = SHAPES + [(360, 640, 6)]


def _features(h, w, b, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(b, h, w, 48, generator=g) * 0.7).to(DEV)


def bounded_chain(be, p, feats, pset, rows=None):
    """Each impl's own chain from the features; tc and tc_ldgsts in lockstep (bit-equal at every layer), every layer
    against float64 on its own input.  Returns each impl's chained rgb."""
    rgb = {}
    for impl in ("tc", "ref"):
        acts = [run_layer(be, 0, feats, None, impl)]
        WORST[(pset, 0, "all")] = max(WORST.get((pset, 0, "all"), 0.0), R.check_input_bounded(p, feats, acts[0]).r)
        for layer in range(1, 10):
            x = acts[-1]
            res = acts[-2] if layer in R.RES_LAYERS else None
            out = run_layer(be, layer, x, res, impl)
            if impl == "tc" and layer != 5:
                assert torch.equal(out, run_layer(be, layer, x, res, "tc_ldgsts")), (pset, layer, tuple(feats.shape))
            if layer == 5:
                wr = R.check_upsample_bounded(p, x, out)
                key = (pset, 5, "all")
            else:
                wr = R.check_conv7_bounded(p, 1e-5, layer, impl, x, res, out)
                key = (pset, layer, "tc+tc_ldgsts" if impl == "tc" else impl)
            WORST[key] = max(WORST.get(key, 0.0), wr.r)
            assert wr.r <= 1.0, (pset, layer, impl, tuple(feats.shape), wr.r)
            acts.append(out)
            if len(acts) > 3:
                acts[-4] = None  # keep the working set at three activations
        rgb[impl] = acts[-1]
    return rgb


@pytest.mark.parametrize("pset", list(PARAM_SETS))
@pytest.mark.parametrize("shape", BOUNDED_SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_layers_bounded_against_float64(be, pset, shape):
    h, w, b = shape
    p = PARAM_SETS[pset]()
    be.set_rgb_decoder(p)
    feats = _features(h, w, b, seed=h * 1000 + w + b)
    rgb = bounded_chain(be, p, feats, pset)
    for impl in ("tc", "ref"):  # rgb_decode is exactly the ten layer calls
        assert torch.equal(be.rgb_decode(feats, impl), rgb[impl]), (impl, shape)
    assert torch.equal(be.rgb_decode(feats, "tc_ldgsts"), rgb["tc"])
    if b >= 2:  # batch-composition independence
        assert torch.equal(be.rgb_decode(feats[1:2], "tc")[0], rgb["tc"][1])
    torch.cuda.synchronize()
    be.check_status()
    del rgb
    be._dec_ws = None
    torch.cuda.empty_cache()


def test_single_layer_past_2_gib(be):
    """One 7x7 layer whose ACT input and output are 2.15e9 bytes (> 2^31): the rows past the 2^31-byte offset (and a
    band in the middle) against float64, all three impls."""
    p = D.random_decoder_params(seed=61)
    be.set_rgb_decoder(p)
    B, H, W = 1, 4104, 4096
    assert B * H * W * 128 > 2 ** 31
    x = torch.empty(B, H, W, 64, dtype=torch.bfloat16, device=DEV)
    g = _gen(62)
    for y0 in range(0, H, 256):
        x[:, y0:y0 + 256] = R.pack_act(torch.randn(B, min(256, H - y0), W, 32, generator=g, device=DEV).clamp_min(0))
    out = torch.empty_like(x)
    for impl in R.IMPLS:
        be.rgb_decode_layer(1, x, None, impl, out=out)
        torch.cuda.synchronize()
        be.check_status()
        for rows in ((H - 16, H), (2048, 2056)):
            wr = R.check_conv7_bounded(p, 1e-5, 1, impl, x, None, out, rows=rows)
            assert wr.r <= 1.0, (impl, rows, wr.r)
            WORST[("random >2GiB", 1, impl)] = max(WORST.get(("random >2GiB", 1, impl), 0.0), wr.r)
    del x, out
    torch.cuda.empty_cache()


# --------------------------------------------------------------------------------------- pinned rgb_decode output
# SHA-256 of rgb_decode's fp32 output on seeded inputs (golden params / features; random_decoder_params(71) with
# features torch.randn(6, 360, 640, 48, seed 72) * 0.7), recorded on an H100 80GB HBM3 from the build before
# b200nerf_rgb_decode_layer existed: splitting rgb_decode into layer calls changed no bit.
PINNED = {
    ("golden", "tc"): "dd0265409aaf0f095c23f5528a14a21563a7a12002a5d9374c66fd950d4d3ec1",
    ("golden", "tc_ldgsts"): "dd0265409aaf0f095c23f5528a14a21563a7a12002a5d9374c66fd950d4d3ec1",
    ("golden", "ref"): "b8094d8412520aa77a16a9d67daf8c1a7910eb9e102d9bf5ed317be024928f94",
    ("production", "tc"): "6d8e12feb39d927f972ea42a4041a4c999a1f13b1ecb5e08c49b194ac1e9144d",
    ("production", "tc_ldgsts"): "6d8e12feb39d927f972ea42a4041a4c999a1f13b1ecb5e08c49b194ac1e9144d",
    ("production", "ref"): "71bf17a7f0c4e8bfaaa109c5a4df203b0b276688f1ffe8a02f553762a26102b9",
}


def pinned_inputs(which):
    if which == "golden":
        from tests.helpers import load_golden

        meta, g = load_golden("rgb_decoder.npz")
        return g["param"], g["in"]["features"]
    g = torch.Generator().manual_seed(72)
    return D.random_decoder_params(seed=71), torch.randn(6, 360, 640, 48, generator=g) * 0.7


def rgb_sha256(rgb):
    return hashlib.sha256(rgb.contiguous().cpu().numpy().tobytes()).hexdigest()


@pytest.mark.parametrize("which", ["golden", "production"])
def test_rgb_decode_output_pinned(be, which):
    p, feats = pinned_inputs(which)
    be.set_rgb_decoder(p)
    for impl in R.IMPLS:
        rgb = be.rgb_decode(feats, impl)
        torch.cuda.synchronize()
        assert rgb_sha256(rgb) == PINNED[(which, impl)], (which, impl)
    be._dec_ws = None
    torch.cuda.empty_cache()


def test_layer_entry_rejects_bad_calls(be):
    from neurad_studio_b200.lib import B200NerfError

    p = D.random_decoder_params(seed=81)
    be.set_rgb_decoder(p)
    x = R.pack_act(torch.rand(1, 4, 8, 32, device=DEV))
    lib, h = be.lib, be._h
    ptr = lambda t, off=0: None if t is None else t.data_ptr() + off
    call = lambda layer, i, r, o, impl=0: lib.b200nerf_rgb_decode_layer(h, layer, i, r, o, 1, 4, 8, impl, None)
    out = torch.empty_like(x)
    assert call(1, ptr(x), None, ptr(out)) == 0
    assert call(2, ptr(x), ptr(x), ptr(out)) == 0
    assert call(2, ptr(x), None, ptr(out)) != 0  # residual required
    assert call(1, ptr(x), ptr(x), ptr(out)) != 0  # residual rejected
    assert call(5, ptr(x), ptr(x), ptr(out)) != 0
    assert call(10, ptr(x), None, ptr(out)) != 0 and call(-1, ptr(x), None, ptr(out)) != 0
    assert call(1, ptr(x), None, ptr(x)) != 0  # in place
    big = torch.empty(x.numel() + 64, dtype=torch.bfloat16, device=DEV)
    for impl in (0, 1, 2):
        assert call(1, ptr(big, 8), None, ptr(out), impl) != 0  # 8-byte aligned input
        assert call(1, ptr(x), None, ptr(big, 8), impl) != 0
        assert call(2, ptr(x), ptr(big, 8), ptr(out), impl) != 0
        assert call(1, ptr(x), None, ptr(out), 3) != 0
    torch.cuda.synchronize()
    with pytest.raises(B200NerfError):
        be.rgb_decode_layer(1, x.float()[..., :32])
    with pytest.raises(B200NerfError):
        be.rgb_decode_layer(2, x)
    assert be.rgb_decode_layer(1, x[:, :0]).shape == (1, 0, 8, 64)


def test_zzz_report():
    """Worst ratio of |kernel - float64| to its per-entry bound, per parameter set, layer and impl."""
    for k in sorted(WORST, key=str):
        v = WORST[k]
        print("rgb-decoder-bound", *k, v if isinstance(v, str) else f"{v:.4f}")
