"""p3d_decoder_mlp_fwd / _bwd (the OSG decoders of the gradient-requiring passes) against the decoder modules' own torch formulation
(training/triplane.py:112-135, triplane_cond.py:859-970) evaluated by ATen + autograd on the same CUDA tensors, and in float64."""
import numpy as np
import pytest
import torch

from conftest import rel_err

pytestmark = pytest.mark.gpu


def _decoders():
    from pix2pix3d_b200.training import triplane, triplane_cond as tc
    base = {'decoder_lr_mul': 1.0, 'decoder_output_dim': 32}
    return [
        ('osg', lambda: triplane.OSGDecoder(32, dict(base))),
        ('semantic_sigmoid', lambda: tc.OSGDecoder_semantic(32, dict(base, sigmoid=True))),
        ('semantic_raw', lambda: tc.OSGDecoder_semantic(32, dict(base, sigmoid=False))),
        ('entangle_6', lambda: tc.OSGDecoder_semantic_entangle(32, dict(base, sigmoid=False, semantic_channels=6, decoder_lr_mul=0.5))),
        ('entangle_sigmoid', lambda: tc.OSGDecoder_semantic_entangle(32, dict(base, sigmoid=True, semantic_channels=19))),
        ('late_separate', lambda: tc.OSGDecoder_semantic_lateSeparate(32, dict(base, sigmoid=False))),
    ]


def _torch_path(dec, feats, monkeypatch):
    from pix2pix3d_b200 import native
    with monkeypatch.context() as mp:
        mp.setattr(native, 'decoder_mlp_supported', lambda *a, **k: False)
        return dec(feats, None)


@pytest.mark.parametrize('name', [n for n, _ in _decoders()])
@pytest.mark.parametrize('n,m', [(2, 1000), (1, 77)])
def test_decoder_mlp_forward_and_gradients_match_the_module(name, n, m, monkeypatch):
    from pix2pix3d_b200 import _lib
    torch.manual_seed(11)
    dec = dict(_decoders())[name]().cuda()
    for p in dec.parameters():      # biases start at zero in the reference's init: give every parameter a value and a gradient
        p.data.normal_(0, 0.7)
    feats = (torch.randn(n, 3, m, 32, device='cuda') * 2).requires_grad_(True)
    params = list(dec.parameters())
    before = _lib.launch_count
    out = dec(feats, None)
    assert _lib.launch_count > before, 'the module must take the libp3d path on CUDA'
    ref = _torch_path(dec, feats, monkeypatch)
    assert out['rgb'].shape == ref['rgb'].shape and out['sigma'].shape == ref['sigma'].shape
    assert rel_err(out['rgb'].detach().cpu().numpy(), ref['rgb'].detach().cpu().numpy()) < 2e-6
    assert rel_err(out['sigma'].detach().cpu().numpy(), ref['sigma'].detach().cpu().numpy()) < 2e-6
    ct_rgb, ct_sigma = torch.randn_like(ref['rgb']), torch.randn_like(ref['sigma'])
    got = torch.autograd.grad((out['rgb'] * ct_rgb).sum() + (out['sigma'] * ct_sigma).sum(), [feats] + params)
    want = torch.autograd.grad((ref['rgb'] * ct_rgb).sum() + (ref['sigma'] * ct_sigma).sum(), [feats] + params)
    for g, w, nm in zip(got, want, ['feats'] + [k for k, _ in dec.named_parameters()]):
        assert g.shape == w.shape
        assert rel_err(g.cpu().numpy(), w.cpu().numpy()) < 2e-5, nm


def test_decoder_mlp_many_tiles_against_float64(monkeypatch):
    """More tiles than CTAs (several tiles per CTA, a ragged last tile), sigma-only and rgb-only cotangents, large activations
    (softplus threshold branch)."""
    from pix2pix3d_b200 import native
    from pix2pix3d_b200.training import triplane_cond as tc
    torch.manual_seed(12)
    dec = tc.OSGDecoder_semantic_entangle(32, {'decoder_lr_mul': 1.0, 'decoder_output_dim': 32, 'sigmoid': False, 'semantic_channels': 6}).cuda()
    for p in dec.parameters():
        p.data.normal_(0, 1.0)
    n, m = 3, 132 * 128 * 2 // 3 + 5
    feats = (torch.randn(n, 3, m, 32, device='cuda') * 6).requires_grad_(True)
    params = list(dec.parameters())
    out = dec(feats, None)
    dec64 = tc.OSGDecoder_semantic_entangle(32, {'decoder_lr_mul': 1.0, 'decoder_output_dim': 32, 'sigmoid': False, 'semantic_channels': 6}).cuda().double()
    dec64.load_state_dict({k: v.double() for k, v in dec.state_dict().items()})
    f64 = feats.detach().double().requires_grad_(True)
    ref = _torch_path(dec64, f64, monkeypatch)
    assert rel_err(out['rgb'].detach().cpu().numpy(), ref['rgb'].detach().cpu().numpy()) < 1e-5
    assert rel_err(out['sigma'].detach().cpu().numpy(), ref['sigma'].detach().cpu().numpy()) < 1e-5
    for use_rgb, use_sigma in ((True, False), (False, True)):
        loss = (out['rgb'].square().sum() if use_rgb else 0) + (out['sigma'].square().sum() if use_sigma else 0)
        loss64 = (ref['rgb'].square().sum() if use_rgb else 0) + (ref['sigma'].square().sum() if use_sigma else 0)
        got = torch.autograd.grad(loss, [feats] + params, retain_graph=True)
        want = torch.autograd.grad(loss64, [f64] + list(dec64.parameters()), retain_graph=True)
        for g, w in zip(got, want):
            assert rel_err(g.cpu().numpy(), w.cpu().numpy()) < 2e-4      # fp32 sums over 37 k points vs float64


def test_decoder_mlp_refuses_double_backward():
    from pix2pix3d_b200.training import triplane
    dec = triplane.OSGDecoder(32, {'decoder_lr_mul': 1.0, 'decoder_output_dim': 32}).cuda()
    feats = torch.randn(1, 3, 50, 32, device='cuda', requires_grad=True)
    out = dec(feats, None)
    (g,) = torch.autograd.grad(out['sigma'].sum(), [feats], create_graph=True)
    with pytest.raises(RuntimeError):
        g.square().sum().backward()
