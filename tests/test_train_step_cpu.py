"""BASELINE.json configs[4] on CPU at toy size: one training iteration (G main + density reg, D main + R1, D_semantic main + R1,
flat gradient handling, Adam, G_ema) driven by the reference's own loss class, once against the unmodified reference and once
against this package through `install()` -- the parameters of all three networks must come out the same. Each arm runs in a
subprocess (the two resolve the same import names differently)."""
import json
import os
import subprocess
import sys
import textwrap

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# the reference (pix2pix3D): the copy build() makes in oracle/_ref (oracle/vendor_reference.py), or $P3D_REFERENCE_ROOT
REF = next((p for p in (os.path.join(ROOT, 'oracle', '_ref'), os.environ.get('P3D_REFERENCE_ROOT', ''))
            if p and os.path.isdir(os.path.join(p, 'training'))), None)

ARM = textwrap.dedent('''
    import json, sys
    sys.path.insert(0, {root!r}); sys.path.insert(0, {root!r} + '/baseline')
    import torch
    torch.set_num_threads(4)
    if {ours}:
        import pix2pix3d_b200
        pix2pix3d_b200.install(reference_root={ref!r})
    else:
        sys.path.insert(0, {ref!r})
    from pix2pix3d_b200 import train_step as ts
    cfg = dict(ts.TINY_TRAIN, nrr=16, depth_resolution=8)
    cfg['loss'] = dict(cfg['loss'], neural_rendering_resolution_initial=16)
    st = ts.build(cfg, torch.device('cpu'))
    import training.loss, training.triplane_cond
    assert training.loss.__file__.startswith({ref!r})
    assert type(st.G).__module__.startswith('pix2pix3d_b200.') == bool({ours})
    batch = ts.synthetic_batch(cfg, 'cpu', 5)
    torch.manual_seed(3)
    ts.run_iteration(st, batch)
    print('DIGEST ' + json.dumps(dict(ts.grads_digest(st), bytes=st.flat_bytes, phases=[p.name for p in st.phases])))
''')


def _start(ours):
    env = dict(os.environ, CUDA_VISIBLE_DEVICES='')
    return subprocess.Popen([sys.executable, '-c', ARM.format(root=ROOT, ref=REF, ours=ours)], stdout=subprocess.PIPE, stderr=subprocess.PIPE,
                            text=True, env=env)


def _finish(p):
    out, err = p.communicate(timeout=1500)
    assert p.returncode == 0, err[-3000:]
    line = [ln for ln in out.splitlines() if ln.startswith('DIGEST ')][-1]
    return json.loads(line[7:])


@pytest.mark.skipif(REF is None, reason='needs the reference copy build() makes in oracle/_ref')
def test_training_iteration_matches_reference_on_cpu():
    procs = _start(False), _start(True)                      # the two arms run side by side (4 torch threads each)
    ref, ours = _finish(procs[0]), _finish(procs[1])
    assert ref['phases'] == ours['phases'] == ['Gmain', 'Greg', 'Dmain', 'Dreg', 'D_semanticmain', 'D_semanticreg']
    assert ref['bytes'] == ours['bytes']                       # same flat-gradient size per phase = same parameter sets with grads
    for k in ('G', 'D', 'D_semantic'):
        assert abs(ref[k] - ours[k]) <= 1e-6 * abs(ref[k]), (k, ref[k], ours[k])
