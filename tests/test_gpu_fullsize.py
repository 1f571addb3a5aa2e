"""Parity at the METRIC'S scale against reference-generated fixtures (tests/golden/full_*.npz, oracle/make_golden.py fullsize):
BASELINE.json configs[1] (seg2cat 512^2 / 128^2 rays / 48+48 samples), configs[2] as released (seg2face, 19 classes) and
configs[3] (edge2car 128^2 / 64^2 rays / 64+64 samples, white background, Hybrid2X). The reference ran G.synthesis on CPU in
fp32 with seeded weights and seeded inputs; the engine path (wgmma convolutions + fused renderer) must reproduce its outputs
within 1e-3 relative (north-star tolerance), and the fused kernel's importance-sampling indices, fine depths and sort
permutation are scored against the reference's own (torch.searchsorted / torch.sort results) on every 61st ray."""
import json

import numpy as np
import pytest
import torch

from conftest import load_golden, rel_err
from make_golden import FULLSIZE_CASES, fullsize_inputs, state_digest

pytestmark = pytest.mark.gpu


def _run(case, force_fp32, sink=None):
    from pix2pix3d_b200 import _lib, configs, native
    w = configs.WORKLOADS[case['workload']]
    G = configs.build_generator(case['workload'], seed=case['seed'], device='cpu', with_mapping=False)
    digest = state_digest(G)
    G = G.cuda()
    rk = G.rendering_kwargs
    ws, c, jitter, u = fullsize_inputs(case, G.backbone.num_ws, w['nrr'], rk['depth_resolution'], rk['depth_resolution_importance'])
    dev = torch.device('cuda')
    it = iter([jitter.to(dev), u.to(dev)])
    o_like, o_rand = torch.rand_like, torch.rand
    torch.rand_like, torch.rand = (lambda x, *a, **k: next(it)), (lambda *a, **k: next(it))
    native.render_debug_sink = sink
    before = _lib.launch_count
    try:
        with torch.no_grad():
            out = G.synthesis(ws.to(dev), c.to(dev), noise_mode='const', neural_rendering_resolution=w['nrr'], force_fp32=force_fp32)
    finally:
        torch.rand_like, torch.rand = o_like, o_rand
        native.render_debug_sink = None
    assert _lib.launch_count - before > 40, 'the whole-generator tensor-core path was expected'
    return out, digest, w['nrr']


@pytest.mark.parametrize('name', list(FULLSIZE_CASES))
def test_engine_matches_reference_at_full_size(name):
    case = FULLSIZE_CASES[name]
    g = load_golden(name)
    sink = {}
    out, digest, nrr = _run(case, True, sink)
    assert digest == bytes(g['state_digest']).decode(), 'seeded weights differ from the reference run'
    errs = {
        'image': rel_err(out['image'][:, :, 3::8, 5::8].cpu().numpy(), g['out_image_sub']),
        'semantic': rel_err(out['semantic'][:, :, 3::8, 5::8].cpu().numpy(), g['out_semantic_sub']),
        'image_raw': rel_err(out['image_raw'].cpu().numpy(), g['out_image_raw']),
        'image_depth': rel_err(out['image_depth'].cpu().numpy(), g['out_image_depth']),
        'semantic_raw': rel_err(out['semantic_raw'][:, :, ::2, ::2].cpu().numpy(), g['out_semantic_raw']),
    }
    # bookkeeping of the fused kernel vs the reference's own torch.searchsorted / torch.sort results
    B, R = case['B'], nrr * nrr
    rays = torch.arange(0, R, int(g['ray_stride']))
    inds = sink['inds'].reshape(B, R, -1)[:, rays].cpu().numpy()
    perm = sink['perm'].reshape(B, R, -1)[:, rays].cpu().numpy()
    dfine = sink['depths_fine'].reshape(B, R, -1)[:, rays].cpu().numpy()
    feat = sink['feat'].reshape(B, R, -1)[:, rays].cpu().numpy()
    wc = sink['weights_coarse'].reshape(B, R, -1)[:, rays].cpu().numpy()
    rates = {
        'inds_exact': float((inds == g['inds_rays']).mean()),
        'perm_exact': float((perm == g['perm_rays']).mean()),
        'depths_fine_bitexact': float((dfine.view(np.int32) == g['depths_fine_rays'].reshape(dfine.shape).view(np.int32)).mean()),
        'depths_fine_rel_err': rel_err(dfine, g['depths_fine_rays'].reshape(dfine.shape)),
        'rays_with_all_inds_exact': float((inds == g['inds_rays']).all(-1).mean()),
        'feat_rel_err': rel_err(feat, g['feat_rays']),
        'weights_coarse_abs_err': float(np.abs(wc - g['weights_coarse_rays'].reshape(wc.shape)).max()),
        'n_rays_scored': int(inds.shape[0] * inds.shape[1]), 'n_indices_scored': int(inds.size),
    }
    report = {'case': name, 'workload': case['workload'], 'rel_err': errs, 'bookkeeping_vs_reference': rates}
    print('FULLSIZE-PARITY ' + json.dumps(report))
    for k, e in errs.items():
        assert e < 1e-3, (k, e, errs)
    assert rates['feat_rel_err'] < 1e-3
    # the reference's indices come from ATen CPU reductions whose order the kernel cannot replicate bit for bit (DESIGN.md 2);
    # a mismatch moves one fine sample into the neighbouring bin. Floor the rates so that a regression is caught.
    assert rates['inds_exact'] >= 0.999 and rates['perm_exact'] >= 0.995, rates
    assert rates['depths_fine_rel_err'] < 1e-3


@pytest.mark.parametrize('name', ['full_seg2cat'])
def test_fp16_superresolution_at_full_size(name):
    """Default dtype policy (SR stacks in fp16 as the reference on CUDA, superresolution.py:304) vs the fp32 CPU reference:
    raw outputs unchanged (renderer fp32), SR outputs within fp16's own distance."""
    case = FULLSIZE_CASES[name]
    g = load_golden(name)
    out, _, _ = _run(case, False)
    assert rel_err(out['image_raw'].cpu().numpy(), g['out_image_raw']) < 1e-3
    assert rel_err(out['image_depth'].cpu().numpy(), g['out_image_depth']) < 1e-3
    assert rel_err(out['image'][:, :, 3::8, 5::8].cpu().numpy(), g['out_image_sub']) < 2e-2
    assert rel_err(out['semantic'][:, :, 3::8, 5::8].cpu().numpy(), g['out_semantic_sub']) < 2e-2
