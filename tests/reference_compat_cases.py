"""The reference's own unit tests for the modules on this path (tests/model_components/test_ray_sampler.py,
test_renderers.py, tests/cameras/test_rays.py, tests/utils/test_math.py, tests/field_components/test_encodings.py,
test_mlp.py), with the imports switched to the library's mirror -- same names, same bodies, `dev` added.  SURVEY.md 8c lists
them as the closest thing to fixtures the reference has ("API smoke"); the value checks live in the parity suites."""
import pytest
import torch
from torch import nn

from neurad_studio_b200.nerfstudio_api import (MLP, AccumulationRenderer, Frustums, HashEncoding, LinearDisparitySampler, LogSampler,
                                               NearFarCollider, PDFSampler, RayBundle, RGBRenderer, SHEncoding, SqrtSampler,
                                               UniformSampler)


def _bundle(dev):
    origins = torch.zeros((10, 3), device=dev)
    directions = torch.ones_like(origins)
    radius = torch.ones((10, 1), device=dev)
    ray_bundle = RayBundle(origins=origins, directions=directions, pixel_area=radius)
    collider = NearFarCollider(near_plane=2, far_plane=4)
    return collider(ray_bundle)


def spaced_sampler(cls, dev):
    """test_uniform_sampler / test_lin_disp_sampler / test_sqrt_sampler / test_log_sampler"""
    num_samples = 15
    sampler = cls(num_samples=num_samples)
    ray_bundle = _bundle(dev)
    assert torch.all(ray_bundle.nears == 2) and torch.all(ray_bundle.fars == 4)
    ray_samples = sampler(ray_bundle)
    pos = ray_samples.frustums.get_positions()
    assert pos.shape[-2] == num_samples
    t = pos[..., 0]  # origins 0, directions (1,1,1): the coordinate is the bin midpoint
    assert torch.all(t[:, 1:] > t[:, :-1]) and t.min().item() > 2 and t.max().item() < 4


def pdf_sampler(dev):
    """test_pdf_sampler"""
    num_samples = 15
    ray_bundle = _bundle(dev)
    uniform_sampler = UniformSampler(num_samples=num_samples)
    coarse_ray_samples = uniform_sampler(ray_bundle)
    weights = torch.ones((10, num_samples, 1), device=dev)
    pdf_sampler = PDFSampler(num_samples)
    fine = pdf_sampler(ray_bundle, coarse_ray_samples, weights, num_samples)
    # include_original=True (the default): the 16 old edges merged into the 16 new ones
    assert fine.frustums.bin_edges.shape == (10, 2 * (num_samples + 1))
    e = fine.frustums.bin_edges
    assert torch.all(e[:, 1:] >= e[:, :-1]) and abs(e.min().item() - 2) < 1e-5 and abs(e.max().item() - 4) < 1e-5
    only_new = PDFSampler(num_samples, include_original=False)(ray_bundle, coarse_ray_samples, weights, num_samples)
    assert only_new.frustums.bin_edges.shape == (10, num_samples + 1)


def rgb_renderer(dev):
    """test_rgb_renderer"""
    num_samples = 10
    rgb_samples = torch.ones((3, num_samples, 3), device=dev)
    weights = torch.ones((3, num_samples, 1), device=dev)
    weights /= torch.sum(weights, dim=-2, keepdim=True)
    rgb_renderer = RGBRenderer()
    rgb = rgb_renderer(rgb=rgb_samples, weights=weights)
    assert torch.max(rgb) > 0.9
    rgb = rgb_renderer(rgb=rgb_samples * 0, weights=weights)
    assert torch.max(rgb).item() == pytest.approx(0, abs=1e-6)


def acc_renderer(dev):
    """test_acc_renderer"""
    num_samples = 10
    weights = torch.ones((3, num_samples, 1), device=dev)
    weights /= torch.sum(weights, dim=-2, keepdim=True)
    acc_renderer = AccumulationRenderer()
    accumulation = acc_renderer(weights=weights)
    assert torch.max(accumulation) > 0.9


def frustum_get_position(dev):
    """test_frustum_get_position"""
    origin = torch.Tensor([0, 1, 2])[None, ...].to(dev)
    direction = torch.Tensor([0, 1, 0])[None, ...].to(dev)
    frustum_start = torch.Tensor([2])[None, ...].to(dev)
    frustum_end = torch.Tensor([3])[None, ...].to(dev)
    target_position = torch.Tensor([0, 3.5, 2])[None, ...]
    frustum = Frustums(origins=origin, directions=direction, starts=frustum_start, ends=frustum_end,
                       pixel_area=torch.ones((1, 1), device=dev))
    positions = frustum.get_positions()
    assert positions.cpu().reshape(1, 3) == pytest.approx(target_position, abs=1e-6)
    mock = Frustums.get_mock_frustum(dev)
    assert mock.origins.shape == (1, 3) and mock.starts.shape == (1, 1, 1)


def spherical_harmonics(dev):
    """test_spherical_harmonics, components = 4 (the degree the path uses): the basis is orthonormal on the sphere."""
    torch.manual_seed(0)
    N = 1000000
    dx = torch.normal(0, 1, size=(N, 3))
    dx = (dx / torch.linalg.norm(dx, dim=-1, keepdim=True)).to(dev)
    with pytest.raises(ValueError):
        SHEncoding(levels=5)
    encoder = SHEncoding(levels=4)
    assert encoder.get_out_dim() == 16
    sh = encoder(dx).cpu()
    matrix = (sh.T @ sh) / N * 4 * torch.pi
    torch.testing.assert_close(matrix, torch.eye(16), rtol=0, atol=1.5e-2)


def tensor_hash_encoder(dev):
    """test_tensor_hash_encoder"""
    num_levels = 4
    features_per_level = 4
    out_dim = num_levels * features_per_level
    encoder = HashEncoding(num_levels=num_levels, features_per_level=features_per_level, log2_hashmap_size=5, implementation="b200").to(dev)
    assert encoder.get_out_dim() == out_dim
    in_tensor = torch.rand((10, 3), device=dev)
    encoded = encoder(in_tensor)
    assert encoded.shape == (10, out_dim)
    with pytest.raises(ValueError):
        HashEncoding(implementation="tcnn")


def mlp(dev):
    """test_mlp"""
    in_dim = 6
    out_dim = 10
    num_layers = 2
    layer_width = 32
    out_activation = nn.ReLU()
    m = MLP(in_dim=in_dim, out_dim=out_dim, num_layers=num_layers, layer_width=layer_width, out_activation=out_activation)
    assert m.get_out_dim() == out_dim
    x = torch.ones((9, in_dim), device=dev)
    m.build_nn_modules()
    m = m.to(dev)
    y = m(x)
    assert y.shape[-1] == out_dim and y.min().item() >= 0


SPACED = {"uniform": UniformSampler, "lin_disp": LinearDisparitySampler, "sqrt": SqrtSampler, "log": LogSampler}


def standalone_modules_train(dev):
    """The stand-alone HashEncoding / MLP mirrors are differentiable like the reference's torch modules (hand-written
    backward operators), FeatureRenderer / AccumulationRenderer too; operators without a backward refuse to run on
    inputs that require grad instead of detaching them silently."""
    from neurad_studio_b200.nerfstudio_api import DepthRenderer, FeatureRenderer, RaySamples
    from oracle import neurad_oracle as O

    torch.manual_seed(0)
    enc = HashEncoding(num_levels=4, min_res=16, max_res=128, log2_hashmap_size=8, features_per_level=4, hash_init_scale=1.0).to(dev)
    m = MLP(in_dim=16, num_layers=2, layer_width=32, out_dim=3).to(dev)
    x = torch.rand(200, 3, device=dev)
    g = torch.randn(200, 3, device=dev)
    (m(enc(x)) * g).sum().backward()
    table = enc.hash_table.detach().cpu().clone().requires_grad_(True)
    ws = [l.weight.detach().cpu().clone().requires_grad_(True) for l in m.layers]
    bs = [l.bias.detach().cpu().clone().requires_grad_(True) for l in m.layers]
    f = O.hash_encode(x.cpu(), table, enc.scalings.cpu(), 2**8)
    y = torch.nn.functional.linear(torch.relu(torch.nn.functional.linear(f, ws[0], bs[0])), ws[1], bs[1])
    (y * g.cpu()).sum().backward()

    def rel(a, b):
        return (a.detach().cpu() - b).abs().max().item() / (b.abs().max().item() + 1e-30)

    assert rel(enc.hash_table.grad, table.grad) < 1e-4
    for l, w, b in zip(m.layers, ws, bs):
        assert rel(l.weight.grad, w.grad) < 1e-4 and rel(l.bias.grad, b.grad) < 1e-4
    w = torch.rand(6, 10, 1, device=dev).requires_grad_(True)
    v = torch.randn(6, 10, 5, device=dev).requires_grad_(True)
    (FeatureRenderer()(v, w).sum() + 2 * AccumulationRenderer()(w).sum()).backward()
    assert rel(w.grad, (v.detach().cpu().sum(-1, keepdim=True) + 2)) < 1e-5 and rel(v.grad, w.detach().cpu().expand(6, 10, 5)) < 1e-6
    rs = RaySamples(Frustums(torch.zeros(6, 3, device=dev), torch.ones(6, 3, device=dev), torch.linspace(0, 1, 11, device=dev).repeat(6, 1)),
                    torch.linspace(0, 1, 11, device=dev))
    with pytest.raises(NotImplementedError):
        DepthRenderer("median")(w, rs)
    assert DepthRenderer("median")(w.detach(), rs).shape == (6, 1)
