"""Network pickles written by the reference load through this package (`legacy.load_network_pkl`, reference legacy.py:24-59,
torch_utils/persistence.py:181-204) as mirror classes and reproduce the reference's outputs.

The pickle is produced at test time by the reference itself in a subprocess (it embeds the reference's module sources, so it
is never committed); it reads the reference from the copy build() makes in oracle/_ref (oracle/vendor_reference.py)."""
import io
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest
import torch

from conftest import load_golden, rel_err
from make_golden import SYNTH_CASES

ORACLE_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), '..', 'oracle')
REF = os.path.abspath(os.path.join(ORACLE_DIR, '_ref'))

WRITER = textwrap.dedent('''
    import pickle, sys
    sys.path.insert(0, {ref!r}); sys.path.insert(0, {oracle!r})
    import torch
    from make_golden import SYNTH_CASES, build_generator
    import training.triplane_cond as tc
    import training.dual_discriminator as dd
    G = build_generator(tc, SYNTH_CASES[{case!r}])
    G.neural_rendering_resolution = 40          # training_loop.py:558 mutates this before every snapshot
    G.rendering_kwargs['density_reg'] = 0.125
    torch.manual_seed(5)
    D = dd.DualDiscriminator(c_dim=25, img_resolution=128, img_channels=3, channel_base=1024, channel_max=16,
                             mapping_kwargs={{}}, epilogue_kwargs={{'mbstd_group_size': 2}})
    with open({out!r}, 'wb') as f:
        pickle.dump(dict(G=G, D=D, G_ema=G, training_set_kwargs=dict(path='none')), f)
''')


@pytest.fixture
def install():
    """pix2pix3d_b200.install() for one test: the aliases are removed again afterwards, so that later tests in the process can
    import the reference's own modules under the same names."""
    import pix2pix3d_b200
    try:
        yield pix2pix3d_b200.install
    finally:
        pix2pix3d_b200.uninstall()


@pytest.mark.skipif(not os.path.isdir(os.path.join(REF, 'training')), reason='needs the reference copy build() makes in oracle/_ref')
@pytest.mark.parametrize('case_name', ['seg_tiny', 'rgb_tiny'])
def test_reference_pickle_loads_as_mirror_classes(tmp_path, case_name, install):
    pkl = str(tmp_path / 'network.pkl')
    code = WRITER.format(ref=REF, oracle=os.path.abspath(ORACLE_DIR), case=case_name, out=pkl)
    r = subprocess.run([sys.executable, '-c', code], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    with open(pkl, 'rb') as f:
        raw = f.read()
    assert b'_reconstruct_persistent_obj' in raw and b'class SynthesisLayer' in raw      # reference format: embedded source

    # the reference's calling sequence (generate_samples.py:93-95) through the aliased import paths
    install()
    import dnnlib
    import legacy
    with dnnlib.util.open_url(pkl) as f:
        data = legacy.load_network_pkl(f)
    with dnnlib.util.open_url('file://' + pkl) as f:
        assert f.read(16) == raw[:16]
    G = data['G_ema']
    assert type(G).__module__ == 'pix2pix3d_b200.training.triplane_cond' and type(G).__name__ == SYNTH_CASES[case_name]['cls']
    assert type(data['D']).__module__ == 'pix2pix3d_b200.training.dual_discriminator'
    assert data['augment_pipe'] is None and data['training_set_kwargs'] == dict(path='none')
    assert not G.training and not any(p.requires_grad for p in G.parameters())             # pickled in eval / frozen state
    assert G.init_kwargs['rendering_kwargs']['depth_resolution'] == SYNTH_CASES[case_name]['Sc']
    # attributes mutated after construction come back as pickled (reference persistence.py:197-203 restores __dict__)
    assert G.neural_rendering_resolution == 40 and G.rendering_kwargs['density_reg'] == 0.125

    # same outputs as the reference computed for this seed (tests/golden/synthesis_<case>.npz)
    g = load_golden('synthesis_' + case_name)
    case = SYNTH_CASES[case_name]
    z, c, mask = (torch.from_numpy(g[k]) for k in ('z', 'c', 'mask'))
    with torch.no_grad():
        ws = G.mapping(z, c, {'mask': mask, 'pose': c})
        assert rel_err(ws.numpy(), g['ws']) < 1e-5
        it = iter([torch.from_numpy(g['jitter']), torch.from_numpy(g['u'])])
        o_like, o_rand = torch.rand_like, torch.rand
        torch.rand_like = lambda x, *a, **k: next(it)
        torch.rand = lambda *a, **k: next(it)
        try:
            out = G.synthesis(ws, c, noise_mode='const', neural_rendering_resolution=case['nrr'])
        finally:
            torch.rand_like, torch.rand = o_like, o_rand
    for k, v in out.items():
        assert rel_err(v.numpy(), g['out_' + k]) < 1e-4, k

    # force_fp16 rebuilds the networks with fp16 settings and carries the weights over (legacy.py:47-58)
    data16 = legacy.load_network_pkl(io.BytesIO(raw), force_fp16=True)
    assert data16['G_ema'].init_kwargs['num_fp16_res'] == 4 and data16['G_ema'].init_kwargs['conv_clamp'] == 256
    sd, sd16 = G.state_dict(), data16['G_ema'].state_dict()
    assert all(torch.equal(sd[k], sd16[k]) for k in sd)


def test_unknown_persistent_class_is_refused_without_opt_in():
    from pix2pix3d_b200.torch_utils import persistence
    meta = dict(type='class', version=6, module_src='class Foo:\n    pass\n', class_name='Foo', state={})
    with pytest.raises(ModuleNotFoundError):
        persistence._reconstruct_persistent_obj(meta)
    persistence.allow_embedded_source = True
    try:
        obj = persistence._reconstruct_persistent_obj(meta)
        assert type(obj).__name__ == 'Foo'
    finally:
        persistence.allow_embedded_source = False


def test_mirror_networks_pickle_by_reference_and_deepcopy():
    """Objects of this package pickle without embedded source (by reference to the package) and survive copy.deepcopy, as
    training_loop.py does for G_ema and the snapshot pickles (training_loop.py:197, 603-615)."""
    import copy
    import pickle
    import pix2pix3d_b200.training.triplane_cond as tc
    from make_golden import build_generator
    G = build_generator(tc, SYNTH_CASES['rgb_tiny'])
    blob = pickle.dumps(dict(G_ema=G))
    assert b'class SynthesisLayer' not in blob
    G2 = pickle.loads(blob)['G_ema']
    assert type(G2) is type(G) and G2.init_kwargs == G.init_kwargs
    sd, sd2 = G.state_dict(), G2.state_dict()
    assert sd.keys() == sd2.keys() and all(torch.equal(sd[k], sd2[k]) for k in sd)
    G3 = copy.deepcopy(G).eval().requires_grad_(False)
    assert all(torch.equal(a, b) for a, b in zip(G.state_dict().values(), G3.state_dict().values()))
