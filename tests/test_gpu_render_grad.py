"""The gradient-requiring fused renderer (`_FusedRender`: p3d_render_fwd under autograd, p3d_render_bwd backward) against a
float64 restatement of the staged chain (grid_sample -> decoder module -> _march_torch) on the kernel's own sorted depths and
fp32 sample coordinates. Each gradient's error must stay within twice the staged fp32 chain's (_SamplePlanes,
native.decoder_mlp, _RayMarch) on the same depths, with a floor of 1e-5. Shapes come from the SM count and a mirror of the
backward's grid rule (render_fused_bwd.cu)."""
import copy

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

TPB = 128            # kRbThreads: a tile holds floor(128 / S) whole rays
CTAS_PER_SM = 2      # kRbCtasPerSm


def bwd_grid(n_rays, S, sms):
    """(rays per tile, tiles, CTAs) of p3d_render_bwd, where two CTAs fit an SM (S >= 16 with two nets)."""
    rt = TPB // S
    tiles = -(-n_rays // rt)
    return rt, tiles, min(tiles, CTAS_PER_SM * sms)


def _decoder(name, lr_mul=1.0):
    from pix2pix3d_b200.training import triplane, triplane_cond as tc
    base = {'decoder_lr_mul': lr_mul, 'decoder_output_dim': 32}
    return {
        'osg': lambda: triplane.OSGDecoder(32, dict(base)),
        'semantic_sigmoid': lambda: tc.OSGDecoder_semantic(32, dict(base, sigmoid=True)),
        'semantic_raw': lambda: tc.OSGDecoder_semantic(32, dict(base, sigmoid=False)),
        'late_sigmoid': lambda: tc.OSGDecoder_semantic_lateSeparate(32, dict(base, sigmoid=True)),
        'late_raw': lambda: tc.OSGDecoder_semantic_lateSeparate(32, dict(base, sigmoid=False)),
        'entangle_sigmoid': lambda: tc.OSGDecoder_semantic_entangle(32, dict(base, sigmoid=True, semantic_channels=19)),
        'entangle_raw': lambda: tc.OSGDecoder_semantic_entangle(32, dict(base, sigmoid=False, semantic_channels=6)),
    }[name]()


def _rays(B, R, gen, dev, radius=2.7):
    o = torch.randn(B, R, 3, generator=gen)
    o = o / o.norm(dim=-1, keepdim=True) * radius
    d = -o + 0.3 * torch.randn(B, R, 3, generator=gen)
    d = d / d.norm(dim=-1, keepdim=True)
    return o.to(dev), d.to(dev)


def ref_chain(planes, decoder, coords, depths, box_warp, white_back, axes):
    """feat [B,R,C], depth [B,R,1], wsum [B,R,1] of the staged chain at given sample coordinates [B,R*S,3] and sorted depths
    [B,R,S], in the dtype of `planes` (grid_sample, the decoder module's own torch formulation, _march_torch)."""
    from pix2pix3d_b200.training.volumetric_rendering.ray_marcher import _march_torch
    from pix2pix3d_b200.training.volumetric_rendering.renderer import project_onto_planes
    B, _, C, H, W = planes.shape
    R, S = depths.shape[1], depths.shape[2]
    grid = project_onto_planes(axes.to(planes), (2 / box_warp) * coords.to(planes)).unsqueeze(1)
    f = F.grid_sample(planes.reshape(B * 3, C, H, W), grid, mode='bilinear', padding_mode='zeros', align_corners=False)
    feats = f.permute(0, 3, 2, 1).reshape(B, 3, R * S, C)
    out = decoder(feats, None)
    colors = out['rgb'].reshape(B, R, S, -1)
    sigma = out['sigma'].reshape(B, R, S, 1)
    rgb, depth, weights = _march_torch(colors, sigma, depths.to(planes).unsqueeze(-1), white_back)
    return rgb, depth, weights.sum(2)


def _loss(outs, g_feat, g_depth, g_wsum):
    feat, depth, wsum = outs
    loss = (feat * g_feat.to(feat)).sum()
    if g_depth is not None:
        loss = loss + (depth.reshape(g_depth.shape) * g_depth.to(depth)).sum()
    if g_wsum is not None:
        loss = loss + (wsum.reshape(g_wsum.shape) * g_wsum.to(wsum)).sum()
    return loss


def _grads(planes, decoder, fn):
    planes = planes.detach().clone().requires_grad_(True)
    decoder.zero_grad(set_to_none=True)
    fn(planes).backward()
    return [planes.grad] + [p.grad if p.grad is not None else torch.zeros_like(p) for p in decoder.parameters()]


def _fused_case(B, R, Sc, Sf, dec_name, white_back=False, lr_mul=1.0, H=32, W=32, box_warp=1.0, grads=('feat',), impl=None,
                seed=0, zero_rays=None):
    """Run the fused forward + backward through native.render_fwd / render_bwd and return everything the checks need."""
    from pix2pix3d_b200 import native
    dev = torch.device('cuda')
    gen = torch.Generator().manual_seed(seed)
    decoder = _decoder(dec_name, lr_mul).to(dev)
    with torch.no_grad():
        for p in decoder.parameters():
            p.add_(0.3 * torch.randn(p.shape, generator=gen).to(dev))
    planes = (0.5 * torch.randn(B, 3, 32, H, W, generator=gen)).to(dev)
    o, d = _rays(B, R, gen, dev)
    dc = torch.sort(torch.linspace(2.0, 3.4, Sc).expand(B, R, Sc) + 0.05 * torch.rand(B, R, Sc, generator=gen), -1)[0].to(dev)
    if zero_rays is not None:
        dc[zero_rays] = 2.5          # every interval has zero length (the fine samples land on the same depth): zero weights
    u = torch.rand(B * R, Sf, generator=gen).to(dev) if Sf > 0 else None
    S = Sc + Sf
    ds = torch.empty(B, R, S, device=dev)
    dec = native.pack_decoder(decoder)
    feat, depth, wsum = native.render_fwd(native.planes_to_channels_last(planes), dec, o, d, dc, u, box_warp, white_back=white_back,
                                          impl=impl, out={'depths_sorted': ds})
    g_feat = torch.randn(B, R, feat.shape[-1], generator=gen).to(dev) if 'feat' in grads else torch.zeros_like(feat)
    g_depth = torch.randn(B, R, generator=gen).to(dev) if 'depth' in grads else None
    g_wsum = torch.randn(B, R, generator=gen).to(dev) if 'wsum' in grads else None
    return dict(decoder=decoder, planes=planes, o=o, d=d, dc=dc, u=u, impl=impl, ds=ds, dec=dec, Sc=Sc, Sf=Sf, box_warp=box_warp, white_back=white_back,
                g_feat=g_feat, g_depth=g_depth, g_wsum=g_wsum, feat=feat, depth=depth, wsum=wsum)


def _fused_grads(c):
    from pix2pix3d_b200 import native
    nets, sigma_net, masks = native.describe_decoder(c['decoder'])
    params = [[*native._effective_fc(n[0]), *native._effective_fc(n[2])] for n in nets]
    rng = None
    if c['g_depth'] is not None:
        lo, hi = torch.aminmax(c['ds'])
        rng = torch.stack([lo, hi])
    g_cl, g_par = native.render_bwd(native.planes_to_channels_last(c['planes']), params, sigma_net, masks, c['o'], c['d'], c['ds'],
                                    c['Sc'], c['Sf'], c['box_warp'], c['g_feat'], c['g_depth'], c['g_wsum'], rng,
                                    white_back=c['white_back'])
    # chain rule to the raw module parameters (effective = raw * gain), through autograd
    flat = [t for net in params for t in net]
    leaves = list(c['decoder'].parameters())
    g_flat = []
    for i in range(len(nets)):
        gw1, gb1, gw2, gb2 = torch.split(g_par[i], [64 * 32, 64, 33 * 64, 33])
        g_flat += [gw1.view(64, 32), gb1, gw2.view(33, 64), gb2]
    g_raw = torch.autograd.grad(flat, leaves, g_flat, allow_unused=True)
    g_planes = g_cl.permute(0, 1, 4, 2, 3)
    return [g_planes] + [g if g is not None else torch.zeros_like(p) for g, p in zip(g_raw, leaves)], g_par


def _reference_grads(c, dtype):
    """Gradients of the staged chain at the kernel's fp32 coordinates and sorted depths: float64 modules (the reference), or
    the fp32 staged kernels (_SamplePlanes, native.decoder_mlp, _RayMarch)."""
    from pix2pix3d_b200.training.volumetric_rendering import renderer as rmod
    B, R, S = c['ds'].shape
    coords = (c['o'].unsqueeze(-2) + c['ds'].unsqueeze(-1) * c['d'].unsqueeze(-2)).reshape(B, R * S, 3)     # fp32, as the kernel
    if dtype == torch.float64:
        dec = copy.deepcopy(c['decoder']).double()
        return _grads(c['planes'].double(), dec, lambda p: _loss(ref_chain(p, dec, coords.double(), c['ds'].double(), c['box_warp'],
                                                                           c['white_back'], rmod.generate_planes()),
                                                             c['g_feat'], c['g_depth'], c['g_wsum']))
    r = rmod.ImportanceRenderer().cuda()
    opts = dict(box_warp=c['box_warp'], white_back=c['white_back'], clamp_mode='softplus')

    def staged(p):
        feats = rmod.sample_from_planes(r.plane_axes.cuda(), p, coords, box_warp=c['box_warp'])
        out = c['decoder'](feats, None)
        colors, sigma = out['rgb'].reshape(B, R, S, -1), out['sigma'].reshape(B, R, S, 1)
        rgb, depth, w = r.ray_marcher(colors, sigma, c['ds'].unsqueeze(-1), opts)
        return _loss((rgb, depth, w.sum(2)), c['g_feat'], c['g_depth'], c['g_wsum'])
    return _grads(c['planes'], c['decoder'], staged)


def _err(got, ref):
    ref = ref.double()
    scale = ref.abs().max().item()
    return (got.double() - ref).abs().max().item() / max(scale, 1e-30)


def _check_against_float64(c):
    ref = _reference_grads(c, torch.float64)
    staged = _reference_grads(c, torch.float32)
    fused, _ = _fused_grads(c)
    names = ['planes'] + [n for n, _ in c['decoder'].named_parameters()]
    for name, g, s, r in zip(names, fused, staged, ref):
        if r.abs().max().item() == 0:
            assert g.abs().max().item() == 0, name
            continue
        e_fused, e_staged = _err(g, r), _err(s, r)
        assert e_fused <= max(2 * e_staged, 1e-5), (name, e_fused, e_staged)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.parametrize('Sc,Sf,impl', [(8, 8, None), (48, 48, None), (64, 64, None), (40, 24, None), (16, 0, None), (13, 11, 'simt')])
@pytest.mark.parametrize('dec_name', ['osg', 'late_sigmoid'])
def test_sample_counts_against_float64(Sc, Sf, impl, dec_name):
    _check_against_float64(_fused_case(2, 37, Sc, Sf, dec_name, impl=impl, grads=('feat', 'depth', 'wsum')))


@pytest.mark.parametrize('which', ['one', 'tiles-1', 'tiles', 'tiles+1', '3sm+2'])
def test_tile_edges_against_float64(which):
    S = 96
    rt, _, _ = bwd_grid(1, S, _sms())
    sms_tiles = CTAS_PER_SM * _sms()
    tiles = {'one': None, 'tiles-1': sms_tiles - 1, 'tiles': sms_tiles, 'tiles+1': sms_tiles + 1, '3sm+2': 3 * _sms() + 2}[which]
    n = 1 if tiles is None else tiles * rt
    B = 2 if n % 2 == 0 else 1
    c = _fused_case(B, n // B, 48, 48, 'late_raw', grads=('feat', 'wsum'))
    assert bwd_grid(n, S, _sms())[1] == (1 if tiles is None else tiles)
    _check_against_float64(c)


@pytest.mark.parametrize('dec_name', ['osg', 'semantic_sigmoid', 'semantic_raw', 'late_sigmoid', 'late_raw', 'entangle_sigmoid',
                                      'entangle_raw'])
@pytest.mark.parametrize('white_back', [False, True])
def test_decoders_and_white_back_against_float64(dec_name, white_back):
    _check_against_float64(_fused_case(2, 50, 16, 16, dec_name, white_back=white_back, grads=('feat', 'depth')))


@pytest.mark.parametrize('grads', [('feat',), ('feat', 'depth'), ('feat', 'wsum'), ('depth', 'wsum')])
def test_upstream_gradients_and_lr_mul_against_float64(grads):
    _check_against_float64(_fused_case(1, 64, 24, 24, 'entangle_raw', lr_mul=0.3, grads=grads))


def test_small_planes_with_samples_outside_the_box():
    _check_against_float64(_fused_case(2, 40, 16, 8, 'late_sigmoid', H=12, W=10, box_warp=0.6, grads=('feat', 'depth', 'wsum')))


def test_zero_weight_rays_have_no_depth_term():
    """All samples of image 0 sit at one depth, so its weights vanish. Its depth gradient must change nothing."""
    c = _fused_case(2, 30, 16, 16, 'osg', grads=('feat', 'depth'), zero_rays=0)
    assert c['wsum'][0].abs().max().item() == 0 and c['wsum'][1].abs().min().item() > 0
    c['g_depth'][1] = 0                                  # depth gradient on the zero-weight rays only
    with_depth, par_a = _fused_grads(c)
    without, par_b = _fused_grads(dict(c, g_depth=None))
    assert torch.equal(par_a, par_b)
    assert all(torch.allclose(x, y, rtol=0, atol=1e-6 * max(y.abs().max().item(), 1e-30)) for x, y in zip(with_depth, without))


@pytest.mark.parametrize('impl', ['tc', 'simt', 'tc_pairs'])
def test_sorted_depth_output_changes_nothing_else(impl):
    """out_depths_sorted leaves every other output bit-identical and holds the depths at the sort permutation."""
    from pix2pix3d_b200 import native
    c = _fused_case(2, 33, 64, 64 if impl == 'tc_pairs' else 32, 'late_sigmoid', impl=impl)
    pcl = native.planes_to_channels_last(c['planes'])
    feat, depth, wsum, dbg = native.render_fwd(pcl, c['dec'], c['o'], c['d'], c['dc'], c['u'], c['box_warp'], impl=impl, debug=True)
    ds = torch.empty_like(c['ds'])
    f2, d2, w2, dbg2 = native.render_fwd(pcl, c['dec'], c['o'], c['d'], c['dc'], c['u'], c['box_warp'], impl=impl, debug=True,
                                         out={'depths_sorted': ds})
    assert torch.equal(feat, f2) and torch.equal(depth, d2) and torch.equal(wsum, w2)
    assert all(torch.equal(dbg[k], dbg2[k]) for k in dbg)
    merged = torch.cat([c['dc'], dbg['depths_fine']], -1)
    assert torch.equal(ds, torch.gather(merged, -1, dbg['perm'].long()))
    assert torch.equal(ds, c['ds'])


def _renderer_case(B, R, Sc, Sf, dec_name, seed=0, **extra):
    from pix2pix3d_b200.training.volumetric_rendering.renderer import ImportanceRenderer
    dev = torch.device('cuda')
    gen = torch.Generator().manual_seed(seed)
    decoder = _decoder(dec_name).to(dev)
    planes = (0.5 * torch.randn(B, 3, 32, 64, 64, generator=gen)).to(dev).requires_grad_(True)
    o, d = _rays(B, R, gen, dev)
    opts = dict(dict(depth_resolution=Sc, depth_resolution_importance=Sf, ray_start=2.0, ray_end=3.4, box_warp=1.0,
                     disparity_space_sampling=False, clamp_mode='softplus', white_back=False), **extra)
    return ImportanceRenderer().to(dev), decoder, planes, o, d, opts


def _render_and_grads(r, decoder, planes, o, d, opts, seed=1):
    torch.manual_seed(seed)
    feat, depth, wsum = r(planes, decoder, o, d, opts)
    loss = (feat * torch.linspace(-1, 1, feat.shape[-1], device=feat.device)).sum() + depth.sum() + wsum.sum()
    gs = torch.autograd.grad(loss, [planes] + list(decoder.parameters()))
    return (feat, depth, wsum), gs


def test_renderer_forward_under_grad_is_bit_identical_to_no_grad():
    r, decoder, planes, o, d, opts = _renderer_case(2, 300, 48, 48, 'late_sigmoid')
    (feat, depth, wsum), _ = _render_and_grads(r, decoder, planes, o, d, opts)
    torch.manual_seed(1)
    with torch.no_grad():
        f0, d0, w0 = r(planes, decoder, o, d, opts)
    assert torch.equal(feat, f0) and torch.equal(depth, d0) and torch.equal(wsum, w0)


def test_renderer_routing(monkeypatch):
    from pix2pix3d_b200 import native
    from pix2pix3d_b200.training.volumetric_rendering import renderer as rmod
    calls = []
    real_bwd, real_staged = native.render_bwd, rmod.ImportanceRenderer._forward_staged
    monkeypatch.setattr(native, 'render_bwd', lambda *a, **k: calls.append('bwd') or real_bwd(*a, **k))
    monkeypatch.setattr(rmod.ImportanceRenderer, '_forward_staged', lambda *a, **k: calls.append('staged') or real_staged(*a, **k))
    r, decoder, planes, o, d, opts = _renderer_case(1, 200, 16, 16, 'osg')
    _render_and_grads(r, decoder, planes, o, d, opts)
    assert calls == ['bwd']
    calls.clear()
    _render_and_grads(r, decoder, planes, o, d, dict(opts, density_noise=0.5))
    assert calls == ['staged']
    calls.clear()
    feat, _, _ = r(planes, decoder, o.clone().requires_grad_(True), d, opts)
    assert calls == ['staged']


def test_renderer_gradients_match_the_staged_path(monkeypatch):
    """The same ImportanceRenderer call with the fused grad path switched off: same draws, gradients within fp32 noise."""
    from pix2pix3d_b200.training.volumetric_rendering import renderer as rmod
    r, decoder, planes, o, d, opts = _renderer_case(2, 500, 48, 48, 'late_sigmoid', white_back=True)
    out_f, g_f = _render_and_grads(r, decoder, planes, o, d, opts)
    monkeypatch.setattr(rmod, 'fused_grad', False)
    out_s, g_s = _render_and_grads(r, decoder, planes, o, d, opts)
    for a, b in zip(out_f, out_s):
        assert _err(a, b) < 1e-4
    for a, b in zip(g_f, g_s):
        assert _err(a, b) < 2e-3


def test_memory_at_config5_shapes(monkeypatch):
    """4 images, 128^2 rays, 48 + 48 samples, OSGDecoder_semantic_lateSeparate: the fused path's peak rise over one forward +
    backward stays below 1 GB (the staged path's is printed)."""
    from pix2pix3d_b200.training.volumetric_rendering import renderer as rmod
    r, decoder, planes, o, d, opts = _renderer_case(4, 128 * 128, 48, 48, 'late_raw')
    peaks = {}
    for name, flag in (('fused', True), ('staged', False)):
        monkeypatch.setattr(rmod, 'fused_grad', flag)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        _render_and_grads(r, decoder, planes, o, d, opts)
        torch.cuda.synchronize()
        peaks[name] = (torch.cuda.max_memory_allocated() - base) / 1e9
    print(f"peak rise over one forward + backward: fused {peaks['fused']:.3f} GB, staged {peaks['staged']:.3f} GB")
    assert peaks['fused'] < 1.0


def test_parameter_gradients_are_deterministic():
    c = _fused_case(4, 700, 48, 48, 'late_raw', grads=('feat', 'depth', 'wsum'))
    _, a = _fused_grads(c)
    _, b = _fused_grads(c)
    assert torch.equal(a, b)


def test_importance_renderer_forward_against_float64(monkeypatch):
    """The whole _FusedRender path (forward draws, saved tensors, aminmax range, parameter split, NCHW plane gradient, gains
    through autograd) through ImportanceRenderer.forward, against float64 on the depths and coordinates of that very call."""
    from pix2pix3d_b200 import native
    seen = {}
    real = native.render_fwd

    def spy(*a, **k):
        res = real(*a, **k)
        seen.update(ds=k['out']['depths_sorted'].clone())
        return res
    monkeypatch.setattr(native, 'render_fwd', spy)
    r, decoder, planes, o, d, opts = _renderer_case(2, 300, 48, 48, 'late_sigmoid', white_back=True)
    gen = torch.Generator().manual_seed(7)
    B, R = o.shape[:2]
    g_feat, g_depth, g_wsum = (torch.randn(*shp, generator=gen).cuda() for shp in ((B, R, 64), (B, R), (B, R)))
    torch.manual_seed(1)
    feat, depth, wsum = r(planes, decoder, o, d, opts)
    decoder.zero_grad(set_to_none=True)
    _loss((feat, depth, wsum), g_feat, g_depth, g_wsum).backward()
    fused = [planes.grad] + [p.grad for p in decoder.parameters()]
    c = dict(decoder=decoder, planes=planes.detach(), o=o, d=d, ds=seen['ds'], box_warp=opts['box_warp'], white_back=True,
             g_feat=g_feat, g_depth=g_depth, g_wsum=g_wsum)
    ref = _reference_grads(c, torch.float64)
    staged = _reference_grads(c, torch.float32)
    for g, st, rf in zip(fused, staged, ref):
        assert _err(g, rf) <= max(2 * _err(st, rf), 1e-5)


def _count_paths(monkeypatch):
    from pix2pix3d_b200 import native
    from pix2pix3d_b200.training.volumetric_rendering import renderer as rmod
    calls = []
    real_bwd, real_staged = native.render_bwd, rmod.ImportanceRenderer._forward_staged
    monkeypatch.setattr(native, 'render_bwd', lambda *a, **k: calls.append('bwd') or real_bwd(*a, **k))
    monkeypatch.setattr(rmod.ImportanceRenderer, '_forward_staged', lambda *a, **k: calls.append('staged') or real_staged(*a, **k))
    return calls


@pytest.mark.parametrize('case_name', ['seg_tiny', 'withbg_tiny'])
def test_synthesis_with_gradients_takes_the_fused_path(case_name, monkeypatch):
    """A gradient-requiring G.synthesis of a tiny TriPlaneSemanticEntangleGenerator, and of the _withBG generator (which
    composites with the weight sum), launches p3d_render_bwd and never the staged chain; its gradients match the same call with
    the fused gradient path switched off."""
    import pix2pix3d_b200.training.triplane_cond as tc
    from conftest import load_golden, rel_err
    from make_golden import EXTRA_CASES, SYNTH_CASES, build_generator
    from pix2pix3d_b200.training.volumetric_rendering import renderer as rmod
    case = dict(SYNTH_CASES, **EXTRA_CASES)[case_name]
    g = load_golden(('extra_' if case_name in EXTRA_CASES else 'synthesis_') + case_name)
    G = build_generator(tc, case).cuda().train().requires_grad_(True)
    ws, cam = torch.from_numpy(g['ws']).cuda(), torch.from_numpy(g['c']).cuda()
    calls = _count_paths(monkeypatch)

    def run():
        G.zero_grad(set_to_none=True)
        torch.manual_seed(11)
        out = G.synthesis(ws, cam, noise_mode='const', neural_rendering_resolution=case['nrr'], force_fp32=True)
        loss = sum((v.float() * torch.linspace(-1, 1, v.shape[-1], device=v.device)).mean() for v in out.values())
        loss.backward()
        return {n: p.grad.clone() for n, p in G.named_parameters() if p.grad is not None}
    fused = run()
    assert 'bwd' in calls and 'staged' not in calls, calls
    calls.clear()
    monkeypatch.setattr(rmod, 'fused_grad', False)
    staged = run()
    assert 'bwd' not in calls and 'staged' in calls
    assert set(fused) == set(staged)
    for n in staged:
        assert rel_err(fused[n].cpu().numpy(), staged[n].cpu().numpy()) < 2e-3, n


WHOLE_STEP = """
import json, sys
sys.path.insert(0, {root!r}); sys.path.insert(0, {root!r} + '/baseline')
import torch
import pix2pix3d_b200
pix2pix3d_b200.install(reference_root={ref!r})
from pix2pix3d_b200 import configs, native, train_step as ts
from pix2pix3d_b200.training.volumetric_rendering import renderer as rmod
cfg = dict(ts.TINY_TRAIN)
dev = torch.device('cuda')
st = ts.build(cfg, dev)
batch = ts.synthetic_batch(cfg, dev, 5)
phase = st.phases[0]
assert phase.name == 'Gmain'
calls = []
real_bwd, real_staged = native.render_bwd, rmod.ImportanceRenderer._forward_staged
native.render_bwd = lambda *a, **k: calls.append('bwd') or real_bwd(*a, **k)
rmod.ImportanceRenderer._forward_staged = lambda *a, **k: calls.append('staged') or real_staged(*a, **k)
b = cfg['batch_gpu']
gen_z = torch.randn([b, st.G.z_dim], generator=torch.Generator().manual_seed(1)).to(dev)
gen_c = configs.camera_labels(b, 1000).to(dev)
res = {{}}
for flag in (True, False):
    rmod.fused_grad = flag
    calls.clear()
    torch.manual_seed(3)
    st.G.zero_grad(set_to_none=True)
    st.G.requires_grad_(True)
    st.loss.accumulate_gradients(phase='Gmain', batch=batch, gen_z=gen_z, gen_c=gen_c, gain=1, cur_nimg=0)
    st.G.requires_grad_(False)
    grads = {{n: p.grad.double() for n, p in st.G.named_parameters() if p.grad is not None}}
    res[flag] = (list(calls), grads)
(calls_f, gf), (calls_s, gs) = res[True], res[False]
worst = max(((gf[n] - gs[n]).abs().max() / gs[n].abs().max().clamp_min(1e-30)).item() for n in gs)
print('RESULT ' + json.dumps(dict(calls_fused=calls_f, calls_staged=calls_s, names_equal=set(gf) == set(gs), n=len(gs), worst=worst)))
"""


def test_tiny_training_gmain_phase_matches_the_staged_path():
    """One Gmain phase of the tiny training recipe (the reference's own loss class driving this package's modules): every G
    gradient with the fused gradient path on is within rel_err 2e-3 of the same phase with it off, and the renderer calls of
    the phase take p3d_render_bwd, never the staged chain. Runs in a subprocess because install() re-maps module names."""
    import json
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    ref = os.path.join(root, 'oracle', '_ref')
    if not os.path.isdir(os.path.join(ref, 'training')):
        pytest.skip('the reference copy under oracle/_ref is made by build()')
    p = subprocess.run([sys.executable, '-c', WHOLE_STEP.format(root=root, ref=ref)], capture_output=True, text=True, timeout=900)
    line = [ln for ln in p.stdout.splitlines() if ln.startswith('RESULT ')]
    assert p.returncode == 0 and line, p.stdout[-3000:] + p.stderr[-3000:]
    r = json.loads(line[0][7:])
    assert 'bwd' in r['calls_fused'] and 'staged' not in r['calls_fused'], r
    assert 'bwd' not in r['calls_staged'], r
    assert r['names_equal'] and r['n'] > 0
    assert r['worst'] < 2e-3, r
