"""The staged-chain restatement that tests/test_gpu_render_grad.py uses as its float64 reference (`ref_chain`) agrees with
autograd through ImportanceRenderer._forward_staged on CPU in float64, on the same sorted depths (one merged pass, no
importance draw)."""
import torch

from test_gpu_render_grad import _decoder, _grads, _loss, _rays, ref_chain


def test_reference_chain_matches_forward_staged_on_cpu():
    from pix2pix3d_b200.training.volumetric_rendering.renderer import ImportanceRenderer, generate_planes
    gen = torch.Generator().manual_seed(0)
    B, R, S = 2, 20, 24
    for name, white_back in (('osg', False), ('late_sigmoid', True), ('entangle_raw', False)):
        decoder = _decoder(name, 0.5).double()
        planes = 0.5 * torch.randn(B, 3, 32, 12, 10, generator=gen, dtype=torch.float64)
        o, d = (t.double() for t in _rays(B, R, gen, 'cpu'))
        ds = torch.sort(torch.linspace(2.0, 3.4, S).expand(B, R, S) + 0.05 * torch.rand(B, R, S, generator=gen), -1)[0].double()
        g = (torch.randn(B, R, 32 * (2 if name.startswith('late') else 1), generator=gen), torch.randn(B, R, generator=gen),
             torch.randn(B, R, generator=gen))
        opts = dict(box_warp=0.8, white_back=white_back, clamp_mode='softplus')
        r = ImportanceRenderer()
        r.plane_axes = r.plane_axes.double()                    # the projection in float64 too
        coords = (o.unsqueeze(-2) + ds.unsqueeze(-1) * d.unsqueeze(-2)).reshape(B, R * S, 3)
        ref = _grads(planes, decoder, lambda p: _loss(ref_chain(p, decoder, coords, ds, 0.8, white_back, generate_planes()), *g))
        staged = _grads(planes, decoder, lambda p: _loss(r._forward_staged(p, decoder, o, d, ds.unsqueeze(-1), 0, opts), *g))
        for a, b in zip(ref, staged):
            assert a.dtype == torch.float64 and (a - b).abs().max() <= 1e-12 * b.abs().max(), name
