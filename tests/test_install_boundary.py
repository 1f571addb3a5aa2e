"""`pix2pix3d_b200.install()` must leave the reference's host-side callers startable: the module lists of train.py:24-28 and
applications/generate_samples.py:9-24 import with the mirror active, reference siblings the mirror does not own
(training_loop, dataset, augment, utils, crosssection_utils, metrics) come from the reference checkout, and they run on
the mirror's classes. Runs in a subprocess so the aliasing does not leak into other tests."""
import os
import subprocess
import sys
import textwrap

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# the reference (pix2pix3D): the copy build() makes in oracle/_ref (oracle/vendor_reference.py), or $P3D_REFERENCE_ROOT
REF = next((p for p in (os.path.join(ROOT, 'oracle', '_ref'), os.environ.get('P3D_REFERENCE_ROOT', ''))
            if p and os.path.isdir(os.path.join(p, 'training'))), None)

SCRIPT = textwrap.dedent('''
    import sys, types
    sys.path.insert(0, {root!r}); sys.path.insert(0, {oracle!r}); sys.path.insert(1, {ref!r})
    import pix2pix3d_b200
    pix2pix3d_b200.install({explicit})
    # lpips (training/loss.py:20) is not installed offline: SURVEY 8c prescribes a stub module
    lp = types.ModuleType('lpips'); lp.LPIPS = lambda **k: (lambda a, b: 0); sys.modules['lpips'] = lp
    import torch

    # train.py:24-28
    import dnnlib
    from training import training_loop
    from metrics import metric_main
    from torch_utils import training_stats
    from torch_utils import custom_ops
    # generate_samples.py:9,16,24 and what training_loop pulls in
    import legacy
    from training.utils import color_mask, color_list
    from camera_utils import LookAtPoseSampler
    import training.dataset, training.augment, training.networks_stylegan3, training.loss
    from training.crosssection_utils import sample_cross_section

    import pix2pix3d_b200.torch_utils.training_stats as ts
    import pix2pix3d_b200.training.networks_stylegan2 as ns2
    assert training_stats is ts and custom_ops.__name__.startswith('pix2pix3d_b200.')
    assert training_loop.__file__.startswith({ref!r}) and training.dataset.__file__.startswith({ref!r})
    assert training_loop.misc.__name__ == 'pix2pix3d_b200.torch_utils.misc'           # siblings run on the mirror's ops
    assert training.augment.upfirdn2d.__name__ == 'pix2pix3d_b200.torch_utils.ops.upfirdn2d'
    assert training.networks_stylegan3.bias_act.__name__ == 'pix2pix3d_b200.torch_utils.ops.bias_act'
    import training.networks_stylegan2
    assert training.networks_stylegan2 is ns2
    assert training.loss.Pix2Pix3DLoss is not None

    # a reference-side helper driving the mirror generator (training_loop.py:31 -> crosssection_utils.py:13-24)
    from make_golden import SYNTH_CASES, build_generator
    import training.triplane_cond as tc
    G = build_generator(tc, SYNTH_CASES['seg_tiny'])
    assert type(G).__module__ == 'pix2pix3d_b200.training.triplane_cond'
    ws = torch.randn(1, G.backbone.num_ws, 512)
    with torch.no_grad():
        sig = sample_cross_section(G, ws, resolution=8)
    assert tuple(sig.shape) == (1, 1, 8, 8) and torch.isfinite(sig).all()

    # training_stats surface used by training_loop.py:323,551,756
    c = training_stats.Collector(regex='Loss/.*')
    training_stats.report('Loss/G', [1.0, 3.0]); training_stats.report0('Loss/D', torch.tensor([2.0])); training_stats.report('Other', 5)
    c.update()
    assert c.names() == ['Loss/G', 'Loss/D'] and c.mean('Loss/G') == 2.0 and abs(c.std('Loss/G') - 1.0) < 1e-12 and c.num('Loss/D') == 1
    assert c.as_dict()['Loss/D'].mean == 2.0 and c['Loss/G'] == 2.0
    c.update()
    assert c.mean('Loss/G') == 2.0          # keep_previous
    print('BOUNDARY-OK')
''')


@pytest.mark.skipif(REF is None, reason='needs the reference copy build() makes in oracle/_ref')
@pytest.mark.parametrize('explicit', [True, False])
def test_reference_callers_import_with_install_active(explicit):
    code = SCRIPT.format(root=ROOT, oracle=os.path.join(ROOT, 'oracle'), ref=REF,
                         explicit=f'reference_root={REF!r}' if explicit else '')
    env = dict(os.environ, CUDA_VISIBLE_DEVICES='')
    r = subprocess.run([sys.executable, '-c', code], capture_output=True, text=True, timeout=600, env=env)
    assert r.returncode == 0 and 'BOUNDARY-OK' in r.stdout, (r.stdout[-1500:], r.stderr[-3000:])


def test_dummy_dual_discriminator_fades_raw_image():
    import torch
    from pix2pix3d_b200.training.dual_discriminator import DualDiscriminator, DummyDualDiscriminator
    kw = dict(c_dim=25, img_resolution=32, img_channels=3, channel_base=512, channel_max=16, mapping_kwargs={},
              epilogue_kwargs={'mbstd_group_size': 2})
    torch.manual_seed(3)
    D = DualDiscriminator(**kw).eval().requires_grad_(False)
    torch.manual_seed(3)
    Dd = DummyDualDiscriminator(**kw).eval().requires_grad_(False)
    assert [k for k, _ in D.state_dict().items()] == [k for k, _ in Dd.state_dict().items()]
    assert all(torch.equal(a, b) for a, b in zip(D.state_dict().values(), Dd.state_dict().values()))
    img = {'image': torch.randn(2, 3, 32, 32), 'image_raw': torch.randn(2, 3, 16, 16)}
    c = torch.randn(2, 25)
    fade = 1 - 32 / 500000
    ref = D({'image': img['image'], 'image_raw': img['image_raw'] * fade}, c.clone())
    out = Dd(img, c.clone())
    assert Dd.raw_fade == fade and torch.allclose(out, ref, rtol=1e-5, atol=1e-6)
    Dd.raw_fade = 1e-9
    out0 = Dd(img, c.clone())
    assert Dd.raw_fade == 0 and torch.allclose(out0, D({'image': img['image'], 'image_raw': img['image_raw'] * 0}, c.clone()), rtol=1e-5, atol=1e-6)
