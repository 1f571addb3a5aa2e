"""Comparison with the reference on the GPU.

* G.synthesis on the configurations behind BASELINE.json configs 1 and 3: the reference ran once on CPU in fp32 with the same
  seeded weights, seeded inputs and injected renderer noise (oracle/make_golden.py vs_reference); its outputs are stored at a
  fixed sub-sampling in tests/golden/vsref_*.npz.
* The reference's own op wrappers (torch_utils/ops/{bias_act,upfirdn2d,filtered_lrelu}.py, from the byte-identical copy that
  build() makes in oracle/_ref) run once on their stock plugins, JIT-built by the reference's custom_ops.get_plugin into a
  temporary directory, and once on this package's plugin objects."""
import os
import sys

import pytest
import torch

from conftest import ROOT, load_golden, rel_err
from make_golden import VSREF_CASES, VSREF_SUB, fullsize_inputs, state_digest

sys.path.insert(0, os.path.join(ROOT, 'baseline'))
import ref_harness as rh  # noqa: E402

pytestmark = pytest.mark.gpu


def _ours(name, force_fp32):
    from pix2pix3d_b200 import configs
    case = VSREF_CASES[name]
    dev = torch.device('cuda')
    w = configs.WORKLOADS[case['workload']]
    G = configs.build_generator(case['workload'], seed=0, device='cpu', with_mapping=False)
    digest = state_digest(G)
    G = G.to(dev)
    rk = G.rendering_kwargs
    nrr, Sc, Sf = w['nrr'], rk['depth_resolution'], rk['depth_resolution_importance']
    ws, c, jitter, u = fullsize_inputs(case, G.backbone.num_ws, nrr, Sc, Sf)
    it = iter([jitter.to(dev), u.to(dev)])
    o_like, o_rand = torch.rand_like, torch.rand
    torch.rand_like, torch.rand = (lambda x, *a, **k: next(it)), (lambda *a, **k: next(it))
    try:
        with torch.no_grad():
            out = G.synthesis(ws.to(dev), c.to(dev), noise_mode='const', neural_rendering_resolution=nrr, force_fp32=force_fp32)
    finally:
        torch.rand_like, torch.rand = o_like, o_rand
    g = load_golden(name)
    assert digest == bytes(g['state_digest']).decode(), 'arms must hold identical weights'
    return {k: rel_err(out[k][VSREF_SUB[k]].float().cpu().numpy(), g['out_' + k]) for k in VSREF_SUB}


@pytest.mark.parametrize('workload,batch', [('seg2cat_512', 2), ('edge2car_128', 3)])
def test_synthesis_matches_reference_fp32(workload, batch):
    """fp32 on both sides."""
    name = f'vsref_{workload}'
    assert VSREF_CASES[name]['B'] == batch
    errs = _ours(name, True)
    print('VS-REFERENCE fp32', name, errs)
    for k, e in errs.items():
        assert e < 1e-3, (k, errs)


def test_synthesis_matches_reference_default_dtypes():
    """SR in fp16 (superresolution.py:304) against the fp32 reference: the fp16 path rounds, so the bound is fp16-sized."""
    errs = _ours('vsref_seg2cat_512', False)
    print('VS-REFERENCE default dtypes', errs)
    for k in ('image_raw', 'image_depth', 'semantic_raw'):
        assert errs[k] < 1e-3, (k, errs)
    for k in ('image', 'semantic'):
        assert errs[k] < 2e-2, (k, errs)


needs_ref = pytest.mark.skipif(not rh.available(), reason='oracle/_ref (the reference copy build() makes) is missing')
REFERENCE_ROOTS = ('training', 'torch_utils', 'dnnlib', 'metrics', 'legacy', 'camera_utils')


@pytest.fixture
def reference():
    """The reference's modules under their own names for one test; removed again afterwards so that later tests resolve those
    names to this package (pix2pix3d_b200.install())."""
    saved_path, saved_modules = list(sys.path), set(sys.modules)
    try:
        yield rh.import_reference()
    finally:
        sys.path[:] = saved_path
        for name in set(sys.modules) - saved_modules:
            if name.split('.', 1)[0] in REFERENCE_ROOTS:
                del sys.modules[name]




@needs_ref
def test_reference_op_wrappers_run_on_libp3d_plugins(reference):
    """INTEGRATION.md section 2: the reference's own torch_utils/ops/{bias_act,upfirdn2d}.py, unmodified, with this package's
    `custom_ops.get_plugin` objects in place of the JIT-built pybind modules -- compared with the same wrappers on the
    reference's stock plugins (forward and first-order gradients; e.g. the stock CUDA path does not clamp the gradient of a
    clamped `linear` activation, bias_act.py:164-167 saves no `y` for it, and neither may the replacement)."""
    import torch_utils.ops.bias_act as r_ba
    import torch_utils.ops.upfirdn2d as r_up
    from pix2pix3d_b200.torch_utils import custom_ops as ours
    dev = torch.device('cuda')
    assert r_ba._init() and r_up._init()                       # JIT-build / load the stock plugins
    stock = (r_ba._plugin, r_up._plugin)
    mine = (ours.get_plugin('bias_act_plugin', sources=['bias_act.cpp', 'bias_act.cu']),
            ours.get_plugin('upfirdn2d_plugin', sources=['upfirdn2d.cpp', 'upfirdn2d.cu']))
    torch.manual_seed(0)
    x = torch.randn(3, 8, 33, 31, device=dev, requires_grad=True)
    b = torch.randn(8, device=dev, requires_grad=True)
    f = r_up.setup_filter([1, 3, 3, 1], device=dev)

    def run_all():
        res = []
        for act in ('lrelu', 'swish', 'linear', 'sigmoid', 'softplus'):
            y = r_ba.bias_act(x, b, act=act, clamp=1.5, impl='cuda')
            gx, gb = torch.autograd.grad(y.square().sum(), [x, b], create_graph=True)
            (ggx,) = torch.autograd.grad(gx.square().sum() + gb.square().sum(), [x], allow_unused=True)
            res += [('bias_act ' + act, y), ('bias_act dx ' + act, gx), ('bias_act db ' + act, gb)]
            if ggx is not None:
                res.append(('bias_act d2 ' + act, ggx))
        for kw in (dict(up=2, padding=[2, 1, 2, 1], gain=4), dict(down=2, padding=[1, 1, 1, 1]), dict(padding=[1, 1, 1, 1], gain=4)):
            y = r_up.upfirdn2d(x, f, impl='cuda', **kw)
            (gx,) = torch.autograd.grad(y.square().sum(), [x])
            res += [(f'upfirdn2d {kw}', y), (f'upfirdn2d dx {kw}', gx)]
        return [(n, t.detach().float().cpu().numpy()) for n, t in res]

    try:
        want = run_all()
        r_ba._plugin, r_up._plugin = mine
        got = run_all()
    finally:
        r_ba._plugin, r_up._plugin = stock
    assert len(want) == len(got)
    for (n, w), (_, g) in zip(want, got):
        assert rel_err(g, w) < 2e-6, n


@needs_ref
def test_reference_filtered_lrelu_wrapper_runs_on_libp3d_plugin(reference):
    """The reference's torch_utils/ops/filtered_lrelu.py (autograd class, sign-tensor hand-off between forward and backward,
    fallback on rc = -1) unmodified, once on its stock JIT-built plugin and once on this package's `filtered_lrelu_plugin`."""
    import scipy.signal
    import torch_utils.ops.filtered_lrelu as r_fl
    from pix2pix3d_b200.torch_utils import custom_ops as ours
    dev = torch.device('cuda')
    assert r_fl._init()
    stock = r_fl._plugin
    mine = ours.get_plugin('filtered_lrelu_plugin', sources=['filtered_lrelu.cpp'])
    torch.manual_seed(0)
    k12 = torch.as_tensor(scipy.signal.firwin(numtaps=12, cutoff=0.25, width=0.3, fs=2.0), dtype=torch.float32, device=dev)
    f4 = torch.tensor([1., 3., 3., 1.], device=dev)
    f4 = torch.outer(f4, f4) / 64
    cases = [dict(fu=k12, fd=k12, up=2, down=2, padding=[10, 9, 10, 9], gain=1.4, slope=0.2, clamp=256),
             dict(fu=f4, fd=f4, up=2, down=2, padding=[3, 2, 3, 2], gain=1.0, slope=0.2, clamp=0.8),
             dict(fu=k12, fd=None, up=2, down=1, padding=[5, 6, 5, 6], gain=2 ** 0.5, slope=0.2, clamp=None, flip_filter=True)]

    def run_all():
        res = []
        for kw in cases:
            # the stock plugin has no fused kernel for 2-D filters at up = down = 2 (filtered_lrelu.cu:1252-1259 lists none):
            # it composes upfirdn2d + act + upfirdn2d, which in fp16 rounds the up-sampled tensor and so takes other lrelu /
            # clamp branches than a kernel that keeps fp32 inside; compare that case in fp32 only
            for dtype in ((torch.float32, torch.float16) if kw['fu'].ndim == 1 else (torch.float32,)):
                x = torch.randn(2, 6, 25, 20, device=dev, generator=torch.Generator(dev).manual_seed(1)).to(dtype).requires_grad_(True)
                b = torch.randn(6, device=dev, generator=torch.Generator(dev).manual_seed(2)).to(dtype).requires_grad_(True)
                y = r_fl.filtered_lrelu(x, b=b, impl='cuda', **kw)
                gx, gb = torch.autograd.grad(y.float().square().sum(), [x, b])
                res += [(dtype, y), (dtype, gx), (dtype, gb)]
        return [(d, t.detach().float().cpu().numpy()) for d, t in res]

    import warnings
    try:
        with warnings.catch_warnings():
            warnings.simplefilter('ignore', RuntimeWarning)
            want = run_all()
            r_fl._plugin = mine
            got = run_all()
    finally:
        r_fl._plugin = stock
    for i, ((d, w), (_, g)) in enumerate(zip(want, got)):
        # fp16: both kernels hold fp32 inside but sum in different orders; an element within rounding of 0 / the clamp may
        # take the other branch, which moves single gradient entries
        tol = 2e-5 if d == torch.float32 else 2e-2
        assert rel_err(g, w) < tol, (i, d, rel_err(g, w))
