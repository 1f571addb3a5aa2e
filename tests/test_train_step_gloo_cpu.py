"""BASELINE.json configs[4], the N > 1 path on CPU: two gloo ranks run one training iteration of the toy configuration on DIFFERENT
data shards through `pix2pix3d_b200.train_step` (the reference's loss class on this package's networks, one flat all-reduce per
phase, training_loop.py:532-541). Data-parallel invariant: after the step every rank holds the same parameters (what the
reference asserts with `misc.check_ddp_consistency`), and they differ from a single-rank step on rank 0's shard alone."""
import json
import os
import socket
import subprocess
import sys
import textwrap

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# the reference (pix2pix3D): the copy build() makes in oracle/_ref (oracle/vendor_reference.py), or $P3D_REFERENCE_ROOT
REF = next((p for p in (os.path.join(ROOT, 'oracle', '_ref'), os.environ.get('P3D_REFERENCE_ROOT', ''))
            if p and os.path.isdir(os.path.join(p, 'training'))), None)

RANK = textwrap.dedent('''
    import json, os, sys
    sys.path.insert(0, {root!r}); sys.path.insert(0, {root!r} + '/baseline')
    import torch, torch.distributed as dist
    torch.set_num_threads(3)
    world, rank = {world}, int(sys.argv[1])
    if world > 1:
        os.environ['MASTER_ADDR'], os.environ['MASTER_PORT'] = '127.0.0.1', '{port}'
        dist.init_process_group('gloo', rank=rank, world_size=world)
    import pix2pix3d_b200
    pix2pix3d_b200.install(reference_root={ref!r})
    from pix2pix3d_b200 import train_step as ts
    cfg = dict(ts.TINY_TRAIN, img_resolution=128, nrr=16, depth_resolution=8)      # 128^2: the 2X super-resolution stacks (cheap on CPU)
    cfg['loss'] = dict(cfg['loss'], neural_rendering_resolution_initial=16)
    st = ts.build(cfg, torch.device('cpu'), rank=rank, num_gpus=world)
    batch = ts.synthetic_batch(cfg, 'cpu', 5 + 10 * rank)            # every rank its own shard
    torch.manual_seed(3 + rank)
    ts.run_iteration(st, batch)
    vec = torch.cat([p.detach().double().flatten() for m in (st.G, st.D, st.D_semantic) for p in m.parameters()])
    print('DIGEST ' + json.dumps(dict(sumsq=float(vec.square().sum()), head=vec[:: max(1, vec.numel() // 64)].tolist(), bytes=st.flat_bytes)))
    if world > 1:
        dist.destroy_process_group()
''')


def _free_port():
    with socket.socket() as s:
        s.bind(('127.0.0.1', 0))
        return s.getsockname()[1]


def _start(world, rank, port):
    env = dict(os.environ, CUDA_VISIBLE_DEVICES='')
    return subprocess.Popen([sys.executable, '-c', RANK.format(root=ROOT, ref=REF, world=world, port=port), str(rank)],
                            stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, env=env)


def _finish(p):
    out, err = p.communicate(timeout=1500)
    assert p.returncode == 0, err[-3000:]
    return json.loads([ln for ln in out.splitlines() if ln.startswith('DIGEST ')][-1][7:])


@pytest.mark.skipif(REF is None, reason='needs the reference copy build() makes in oracle/_ref')
def test_two_gloo_ranks_end_the_iteration_with_identical_parameters():
    port = _free_port()
    procs = [_start(2, 0, port), _start(2, 1, port), _start(1, 0, port)]        # two ranks + a single-rank step on rank 0's shard
    r0, r1, solo = (_finish(p) for p in procs)
    assert r0['bytes'] == r1['bytes'] == solo['bytes']
    assert r0['head'] == r1['head'] and r0['sumsq'] == r1['sumsq']               # bit-identical after the flat all-reduce + Adam
    assert r0['head'] != solo['head']                                            # ... and not what one shard alone would give
