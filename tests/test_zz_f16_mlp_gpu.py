"""The shading kernels' field MLP on fp16 tensor cores (MlpLaneTc, csrc/nff_lane.h): three-term hi / lo split of
power-of-two scaled operands, fp32 accumulation.

  * on the GPU, the traced sdf and field features of both lane kernels stay inside the per-entry float64 bounds of
    tests/render_trace_cases.py with the fp16 split's own constant gamma_f16, which is tighter than gamma_tc;
  * on the CPU, a float64 emulation of the scaled split shows that the three-term split meets gamma_f16 and that a
    two-term split (without a_hi * w_lo) does not;
  * on the GPU, parameters that push an activation beyond the fp16 operand range raise the device status instead of
    rendering inf or NaN."""
import pytest
import torch

import neurad_studio_b200 as nsb
from neurad_studio_b200 import scene
from tests import render_trace_cases as C

A_EXP = 6  # kLaneTcA: A operands are 2^6 times the activations


def gamma_f16(K):
    """Per-term constant of one fp16 three-term layer with K inputs (DESIGN section 4): the split's representation
    and dropped lo * lo terms, <= 3.0001 2^-22 |a w| (rounded up to 4 2^-22, which also covers the subnormal absolute
    term at the kernel's scales), plus the same fp32 accumulation term as gamma_tc, (3 K + 1) 2^-22."""
    return 4 * 2.0 ** -22 + (3 * K + 1) * 2.0 ** -22


def test_gamma_f16_is_tighter_than_gamma_tc():
    for K in (32, 48):
        assert gamma_f16(K) < C.gamma_tc(K)


def _split(x):
    hi = x.half()
    lo = (x - hi.float()).half()
    return hi.double(), lo.double()


def _layer(a, w, terms):
    """float64 value of the kernel's split product a @ w.T with a scaled by 2^A_EXP and w by the layer's 2^e (largest
    scaled |w| below 2^15), every fp16 product exact, the sum exact."""
    e = 15 - int(torch.frexp(w.abs().max())[1])
    ah, al = _split(a * 2.0 ** A_EXP)
    wh, wl = _split(w * 2.0 ** e)
    y = ah @ wh.T + al @ wh.T
    if terms == 3:
        y = y + ah @ wl.T
    return y / 2.0 ** (A_EXP + e)


@pytest.mark.parametrize("K", [32, 48])
def test_split_emulation_meets_gamma_f16_and_two_terms_do_not(K):
    gen = torch.Generator().manual_seed(K)
    n = 4096
    mag = torch.exp2(torch.rand(n, K, generator=gen) * 19 - 10)  # 2^-10 .. 2^9
    a = (mag * (torch.rand(n, K, generator=gen) > 0.3)).float()  # ReLU outputs: non-negative, some zero
    w = ((torch.rand(32, K, generator=gen) * 2 - 1) / K ** 0.5).float()
    ref = a.double() @ w.double().T
    tol = gamma_f16(K) * (a.double().abs() @ w.double().abs().T)
    worst = C._ratio(_layer(a, w, 3), ref, tol, f"three-term split, K = {K}")
    assert worst < 0.5, worst
    try:
        C._ratio(_layer(a, w, 2), ref, tol, f"two-term split, K = {K}")
    except AssertionError:
        return
    raise AssertionError("gamma_f16 accepted a two-term split")


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["split", "lane"])
@pytest.mark.parametrize("name", ["config2", "config3"])
def test_main_field_within_gamma_f16(name, mode):
    cfg, params, rays, width = C.scene_rays("cuda", name)
    r = C.renderer("cuda", cfg, params)
    full = r.render({k: v.to("cuda") for k, v in rays.items()}, want_trace=True, image_width=width, mode=mode)
    n = rays["origins"].shape[0]
    extra = ()
    if cfg.n_actors:
        extra = torch.unique((full["actor_id_main"] >= 0).any(1).cpu().nonzero()[:, 0] // 128)[:16]
    idx = C.pick_groups(n, 31, seed=len(name), extra=extra)
    out = C.select(full, idx)
    worst = C.check_main_field(out, rays, idx, cfg, params, "cuda", gamma_f16)
    print(f"\n[f16 mlp] {name} {mode}: worst |got - ref| / bound with gamma_f16: {worst}")


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["split", "lane"])
def test_activation_beyond_fp16_range_raises(mode):
    from neurad_studio_b200.backend import B200Backend, DEFAULT_MODE
    from neurad_studio_b200.lib import B200NerfError

    cfg = nsb.small_config()
    params = scene.make_params(cfg, seed=61, beta=3.0, sdf_bias=0.6)
    rays = scene.random_rays(512, cfg, seed=62)
    be = B200Backend(torch.device("cuda", 0))
    be.load_params(cfg, params)
    be.set_mlp_mode(mode)
    try:
        be.render(rays)
        be.check_status()  # in range: no error
        # geo_embedding (layer 1's output, layer 2's A operand) beyond 2^16 / 2^6 for most samples
        big = dict(params)
        big["field.mlp_geo.layers.1.weight"] = params["field.mlp_geo.layers.1.weight"] * 1.0e5
        be.load_params(cfg, big)
        be.render(rays)
        with pytest.raises(B200NerfError, match="fp16 operand range"):
            be.check_status()
        be.check_status()  # the flag is cleared once reported
    finally:
        be.set_mlp_mode(DEFAULT_MODE)
