"""The oracle (oracle/p3d_oracle, numpy) against fixtures produced by the REFERENCE implementation
(oracle/make_golden.py, run against a reference checkout). This is what pins the oracle."""
import numpy as np
import pytest
import torch

import p3d_oracle as O
from conftest import load_golden, rel_err
from make_golden import SEMGEN_CASES, SYNTH_CASES

RENDER_CASES = ['seg', 'seg48', 'car', 'rgb_only', 'coarse_only', 'far_outside', 'seg16', 'rgb24', 'coarse8', 'car64']
TC_RENDER_CASES = ['seg48', 'car', 'seg16', 'rgb24', 'coarse8', 'car64']     # Sc and Sf multiples of 8


def oracle_decoder(g):
    kind = str(g['decoder'])
    sd = {k[4:]: v for k, v in g.items() if k.startswith('dec.')}
    nets = [dict(w1=sd['net.0.weight'], b1=sd['net.0.bias'], w2=sd['net.2.weight'], b2=sd['net.2.bias'])]
    if kind == 'osg':
        return dict(kind='OSGDecoder', nets=nets, lr_mul=1.0)
    nets.append(dict(w1=sd['net_semantic.0.weight'], b1=sd['net_semantic.0.bias'], w2=sd['net_semantic.2.weight'],
                     b2=sd['net_semantic.2.bias']))
    return dict(kind='OSGDecoder_semantic_lateSeparate', nets=nets, sigmoid=(kind == 'late1'), lr_mul=1.0)


def render_opts(g):
    return dict(ray_start=float(g['opt_ray_start']), ray_end=float(g['opt_ray_end']), box_warp=float(g['opt_box_warp']),
                white_back=bool(g['opt_white_back']) if 'opt_white_back' in g else False,
                depth_resolution=int(g['Sc']), depth_resolution_importance=int(g['Sf']))


@pytest.mark.parametrize('case', RENDER_CASES)
def test_renderer_matches_reference(case):
    g = load_golden('renderer_' + case)
    o, d = O.renderer.ray_sampler(g['cam2world'], g['intrinsics'], int(g['nrr']))
    assert np.abs(o - g['ray_origins']).max() == 0
    assert np.abs(d - g['ray_dirs']).max() < 2e-7
    opts = render_opts(g)
    b, m = g['ray_origins'].shape[:2]
    dc = O.renderer.sample_stratified(b, m, opts['ray_start'], opts['ray_end'], opts['depth_resolution'], g['jitter'])
    u = g['u'] if int(g['Sf']) > 0 else None
    feat, depth, wsum, dbg = O.renderer.importance_renderer(g['planes'], oracle_decoder(g), g['ray_origins'], g['ray_dirs'],
                                                            dc, u, opts, return_debug=True)
    assert rel_err(feat, g['feat']) < 1e-5
    assert rel_err(depth, g['depth']) < 1e-5
    # sums of alpha = 1 - exp(-x) with tiny x carry ~6e-8 absolute noise per interval
    assert rel_err(wsum[..., 0] if wsum.ndim == 3 else wsum, g['wsum'][..., 0]) < 1e-4
    # per-interval weights amplify 1-ulp differences of nearly coincident depths (delta ~ 1e-3): looser bound
    assert rel_err(dbg['weights_final'], g['weights_final']) < 1e-4
    if u is not None:
        assert rel_err(dbg['weights_coarse'], g['weights_coarse']) < 1e-4   # alpha = 1 - exp(-x) cancels for small x
        assert np.abs(dbg['depths_fine'] - g['depths_fine']).max() < 1e-5
        # integer bookkeeping: the sort permutation must agree exactly wherever the reference's own depth gaps
        # exceed float noise; here it agrees everywhere
        assert (dbg['perm'] == g['perm']).mean() > 0.999


def test_importance_indices_exact_given_reference_weights():
    """searchsorted indices are bit-exact when the oracle is fed the reference's own coarse weights."""
    g = load_golden('renderer_seg48')
    opts = render_opts(g)
    b, m = g['ray_origins'].shape[:2]
    sc = opts['depth_resolution']
    dc = O.renderer.sample_stratified(b, m, opts['ray_start'], opts['ray_end'], sc, g['jitter'])
    fine, dbg = O.renderer.sample_importance(dc.reshape(b * m, sc), g['weights_coarse'].reshape(b * m, -1), g['u'],
                                             return_debug=True)
    # the reference's fine depths follow from its indices; equality to 1 ulp of the bin width implies equal indices
    assert np.abs(fine.reshape(g['depths_fine'].shape) - g['depths_fine']).max() < 2e-6
    assert dbg['inds'].min() >= 1 and dbg['inds'].max() <= sc - 2


def test_bias_act_forward_and_gradients():
    g = load_golden('ops')
    x, b = g['ba_x'], g['ba_b']
    for act in O.ops.ACT:
        for tag, kw in (('d', {}), ('c', dict(gain=1.7, clamp=0.9, alpha=0.3))):
            y = O.ops.bias_act(x, b, act=act, **kw)
            assert rel_err(y, g[f'ba_{act}_{tag}_y']) < 2e-6, (act, tag)
            x64, b64 = x.astype(np.float64), b.astype(np.float64)
            y64 = O.ops.bias_act(x64, b64, act=act, **kw)
            gy, ggx = g[f'ba_{act}_{tag}_gy'], g[f'ba_{act}_{tag}_ggx']
            gx = O.ops.bias_act_grad(gy, x64, b64, y64, act=act, order=1, **kw)
            assert rel_err(gx, g[f'ba_{act}_{tag}_gx']) < 1e-9, (act, tag, 'grad1')
            if O.ops.ACT[act][4]:
                g2 = O.ops.bias_act_grad(ggx, x64, b64, y64, act=act, order=2, dy1=gy, **kw)
                ref = g[f'ba_{act}_{tag}_g2x']
                assert np.abs(g2 - ref).max() < 1e-9 * max(1.0, np.abs(ref).max()), (act, tag, 'grad2')


@pytest.mark.parametrize('numpy_conv', ['0', '1'])
def test_upfirdn2d_variants(numpy_conv, monkeypatch):
    monkeypatch.setenv('P3D_ORACLE_NUMPY_CONV', numpy_conv)
    g = load_golden('ops')
    x = g['up_x']
    fm = dict(f4=g['up_f4'], f8=g['up_f8'], f35=g['up_f35'])
    cfgs = {
        'post_tconv': dict(f='f4', up=1, down=1, padding=[1, 1, 1, 1], gain=4),
        'skip_up': dict(f='f4', up=2, down=1, padding=[2, 1, 2, 1], gain=4),
        'down2': dict(f='f4', up=1, down=2, padding=[1, 1, 1, 1], gain=1),
        'pre_sconv': dict(f='f4', up=1, down=1, padding=[2, 2, 2, 2], gain=1),
        'sep8_up2': dict(f='f8', up=2, down=1, padding=[4, 3, 4, 3], gain=4),
        'odd': dict(f='f35', up=[3, 2], down=[2, 1], padding=[2, 0, -1, 3], gain=0.7, flip_filter=True),
        'crop': dict(f='f4', up=1, down=1, padding=[-1, 2, 0, -2], gain=1),
        'identity': dict(f=None, up=1, down=1, padding=0, gain=1),
    }
    assert np.allclose(O.ops.setup_filter([1, 3, 3, 1]), g['up_f4'])
    assert np.allclose(O.ops.setup_filter([1, 2, 3, 4, 4, 3, 2, 1]), g['up_f8'])
    for name, kw in cfgs.items():
        kw = dict(kw)
        f = fm.get(kw.pop('f'))
        y = O.ops.upfirdn2d(x, f, **kw)
        assert y.shape == g[f'up_{name}_y'].shape, name
        assert rel_err(y, g[f'up_{name}_y']) < 2e-6, name


@pytest.mark.parametrize('numpy_conv', ['0', '1'])
def test_conv_resample_and_modconv(numpy_conv, monkeypatch):
    monkeypatch.setenv('P3D_ORACLE_NUMPY_CONV', numpy_conv)
    g = load_golden('ops')
    x, w3, w1, st, nz, f4 = g['mc_x'], g['mc_w3'], g['mc_w1'], g['mc_styles'], g['mc_noise16'], g['up_f4']
    assert rel_err(O.ops.conv2d_resample(x, w3, f=f4, up=2, padding=1, flip_weight=False), g['cr_up2']) < 1e-5
    assert rel_err(O.ops.conv2d_resample(x, w3, f=f4, down=2, padding=1), g['cr_down2']) < 1e-5
    assert rel_err(O.ops.conv2d_resample(x, w1, f=f4, down=2), g['cr_1x1_down2']) < 1e-5
    assert rel_err(O.ops.conv2d_resample(x, w1, f=f4, up=2), g['cr_1x1_up2']) < 1e-5
    assert rel_err(O.ops.conv2d_resample(x, w3, padding=1), g['cr_plain']) < 1e-5
    for fused in (True, False):
        t = 'f' if fused else 'n'
        y = O.ops.modulated_conv2d(x, w3, st, noise=nz, up=2, padding=1, resample_filter=f4, flip_weight=False, fused_modconv=fused)
        assert rel_err(y, g[f'mc_up2_{t}']) < 1e-5
        y = O.ops.modulated_conv2d(x, w3, st, noise=nz[:, :, :8, :8], padding=1, fused_modconv=fused)
        assert rel_err(y, g[f'mc_plain_{t}']) < 1e-5
        y = O.ops.modulated_conv2d(x, w1, st, demodulate=False, fused_modconv=fused)
        assert rel_err(y, g[f'mc_torgb_{t}']) < 1e-5


@pytest.mark.parametrize('name', list(SYNTH_CASES))
def test_generator_synthesis_matches_reference(name):
    """Whole G.synthesis in the oracle (backbone + renderer + super-resolution) vs the reference's outputs.
    Weights are rebuilt from the seed through the host-side mirror and checked against the fixture's digest."""
    import pix2pix3d_b200.training.triplane_cond as tc
    from make_golden import build_generator, state_digest
    case = SYNTH_CASES[name]
    g = load_golden('synthesis_' + name)
    G = build_generator(tc, case)
    assert state_digest(G) == bytes(g['state_digest']).decode(), 'mirror and reference initialise differently'
    sd = {k: v.numpy() for k, v in G.state_dict().items()}
    rk = dict(G.rendering_kwargs)
    cfg = dict(nrr=case['nrr'], rendering_kwargs=rk, semantic_channels=case['semantic_channels'],
               sr_kind='SuperresolutionHybrid2X', sr_kind_semantic='SuperresolutionHybrid2X_semantic', sr_fp16=True)
    out = O.networks.generator_synthesis(g['ws'], g['c'], sd, cfg, g['jitter'], g['u'])
    assert rel_err(out['planes'].reshape(g['ws'].shape[0], 96, 256, 256)[:, :, 3::16, 5::16], g['planes_sub']) < 1e-4
    for k in ('image_raw', 'image_depth', 'image', 'semantic_raw', 'semantic'):
        if 'out_' + k in g:
            assert rel_err(out[k], g['out_' + k]) < 1e-3, k


@pytest.mark.parametrize('name', list(SEMGEN_CASES))
def test_semantic_generator_synthesis_matches_reference(name):
    """TriPlaneSemanticGenerator.synthesis (two backbones + ImportanceSemanticRenderer, SURVEY 8 a10) in the oracle."""
    import pix2pix3d_b200.training.triplane_cond as tc
    from make_golden import build_generator, state_digest
    case = SEMGEN_CASES[name]
    g = load_golden('synthesis_' + name)
    G = build_generator(tc, case)
    assert state_digest(G) == bytes(g['state_digest']).decode(), 'mirror and reference initialise differently'
    sd = {k: v.numpy() for k, v in G.state_dict().items()}
    cfg = dict(nrr=case['nrr'], rendering_kwargs=dict(G.rendering_kwargs), semantic_channels=case['semantic_channels'],
               w_dim=case['w_dim'], sr_kind='SuperresolutionHybrid2X', sr_kind_semantic='SuperresolutionHybrid2X_semantic', sr_fp16=True)
    out = O.networks.generator_synthesis_semantic(g['ws'], g['c'], sd, cfg, g['jitter'], g['u'])
    n = g['ws'].shape[0]
    assert rel_err(out['planes_texture'].reshape(n, 96, 256, 256)[:, :, 3::16, 5::16], g['planes_texture_sub']) < 1e-4
    assert rel_err(out['planes_semantic'].reshape(n, 96, 256, 256)[:, :, 3::16, 5::16], g['planes_semantic_sub']) < 1e-4
    for k in ('image_raw', 'image_depth', 'image', 'semantic_raw', 'semantic'):
        assert rel_err(out[k], g['out_' + k]) < 1e-3, k
    # run_model at free points (G.sample_mixed)
    rk = G.rendering_kwargs
    dec_t = O.networks.decoder_from_state_dict(sd, 'decoder', 'OSGDecoder')
    dec_s = O.networks.decoder_from_state_dict(sd, 'decoder_semantic', 'OSGDecoder_semantic',
                                               semantic_sigmoid=case['semantic_channels'] == 1)
    rgb, sigma, sem = O.renderer.run_model_semantic(out['planes_texture'], out['planes_semantic'], dec_t, dec_s, g['pts'], rk['box_warp'])
    assert rel_err(rgb, g['sample_rgb']) < 1e-4 and rel_err(sigma, g['sample_sigma']) < 1e-4
    assert rel_err(sem, g['sample_semantic']) < 1e-4


def test_filtered_lrelu_composition():
    g = load_golden('ops')
    y = O.ops.filtered_lrelu(g['fl_x'], g['up_f4'], g['fl_fd'], g['fl_b'], up=2, down=2, padding=[3, 2, 3, 2], clamp=0.8)
    assert y.shape == g['fl_up2_down2'].shape and rel_err(y, g['fl_up2_down2']) < 2e-6
    y = O.ops.filtered_lrelu(g['fl_x'], None, g['up_f4'], g['fl_b'], up=1, down=1, padding=2, gain=1.3, slope=0.1)
    assert rel_err(y, g['fl_up1']) < 2e-6
