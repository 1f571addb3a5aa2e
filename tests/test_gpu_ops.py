"""bias_act / upfirdn2d CUDA kernels through the reference-facing functions (torch_utils.ops.*) and the C-ABI,
against the oracle and the reference fixtures."""
import numpy as np
import pytest
import torch

import p3d_oracle as O
from conftest import load_golden, rel_err

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('dtype', [torch.float32, torch.float64, torch.float16])
def test_bias_act_forward_all_activations(dtype):
    from pix2pix3d_b200.torch_utils.ops import bias_act
    g = load_golden('ops')
    x = torch.from_numpy(g['ba_x']).cuda().to(dtype)
    b = torch.from_numpy(g['ba_b']).cuda().to(dtype)
    tol = {torch.float32: 2e-6, torch.float64: 1e-12, torch.float16: 2e-3}[dtype]
    # the plugin ABI carries alpha/gain/clamp as C floats (bias_act.cpp:36), so fp64 sees them rounded to fp32
    r32 = lambda v: float(np.float32(v))
    for act in bias_act.activation_funcs:
        for kw in ({}, dict(gain=r32(1.7), clamp=r32(0.9), alpha=r32(0.3))):
            y = bias_act.bias_act(x, b, act=act, **kw)
            assert y.dtype == dtype and y.shape == x.shape
            kw = dict(kw, gain=r32(kw.get('gain', bias_act.activation_funcs[act].def_gain)),
                      alpha=r32(kw.get('alpha', bias_act.activation_funcs[act].def_alpha)))   # defaults cross the ABI as floats too
            ref = O.ops.bias_act(x.cpu().numpy().astype(np.float64 if dtype == torch.float64 else np.float32),
                                 b.cpu().numpy().astype(np.float64 if dtype == torch.float64 else np.float32), act=act, **kw)
            assert rel_err(y.float().cpu().numpy() if dtype != torch.float64 else y.cpu().numpy(), ref) < tol, (act, kw)
        # channels_last keeps its layout and values
        xc = x.contiguous(memory_format=torch.channels_last)
        yc = bias_act.bias_act(xc, b, act=act)
        assert yc.is_contiguous(memory_format=torch.channels_last)
        assert torch.equal(yc.contiguous(), bias_act.bias_act(x, b, act=act))
    # bias along another dim, no bias, no-op
    y = bias_act.bias_act(x, torch.arange(6, device='cuda', dtype=dtype), dim=3, act='relu')
    ref = O.ops.bias_act(x.double().cpu().numpy(), np.arange(6, dtype=np.float64), dim=3, act='relu', gain=r32(np.sqrt(2)))
    assert rel_err(y.double().cpu().numpy(), ref) < max(tol, 1e-3 if dtype == torch.float16 else 0)
    assert bias_act.bias_act(x, None, act='linear', gain=1) is not None


def test_bias_act_gradients_first_and_second_order():
    from pix2pix3d_b200.torch_utils.ops import bias_act
    g = load_golden('ops')
    # fixtures were produced with double-precision alpha/gain/clamp; the C-ABI rounds them to fp32 (as the reference
    # plugin does), so the fixture comparison is at 1e-6 and the exact comparison is against the oracle evaluated
    # with the rounded parameters
    r32 = lambda v: float(np.float32(v))
    for act in bias_act.activation_funcs:
        for tag, kw in (('d', {}), ('c', dict(gain=1.7, clamp=0.9, alpha=0.3))):
            kw32 = {k: r32(v) for k, v in kw.items()}
            kw32['gain'] = r32(kw.get('gain', bias_act.activation_funcs[act].def_gain))
            kw32['alpha'] = r32(kw.get('alpha', bias_act.activation_funcs[act].def_alpha))
            plugin_only = (act == 'linear' and tag == 'c')   # reference CUDA path ignores the clamp in linear's gradient
            x = torch.from_numpy(g['ba_x']).cuda().double().requires_grad_(True)
            b = torch.from_numpy(g['ba_b']).cuda().double().requires_grad_(True)
            y = bias_act.bias_act(x, b, act=act, **kw)
            x64, b64 = g['ba_x'].astype(np.float64), g['ba_b'].astype(np.float64)
            y_or = O.ops.bias_act(x64, b64, act=act, **kw32)
            assert rel_err(y.detach().cpu().numpy(), y_or) < 1e-12, (act, tag)
            assert rel_err(y.detach().cpu().numpy(), g[f'ba_{act}_{tag}_y64']) < 1e-6
            gy_np, ggx_np = g[f'ba_{act}_{tag}_gy'], g[f'ba_{act}_{tag}_ggx']
            gy = torch.from_numpy(gy_np).cuda()
            gx, gb = torch.autograd.grad(y, [x, b], gy, create_graph=True)
            gx_or = O.ops.bias_act_grad(gy_np, x64, b64, y_or, act=act, order=1, plugin_semantics=True, **kw32)
            assert rel_err(gx.detach().cpu().numpy(), gx_or) < 1e-10, (act, tag)
            if not plugin_only:
                assert rel_err(gx.detach().cpu().numpy(), g[f'ba_{act}_{tag}_gx']) < 1e-6, (act, tag)
            assert rel_err(gb.detach().cpu().numpy(), gx_or.sum((0, 2, 3))) < 1e-10
            ggx = torch.from_numpy(ggx_np).cuda()
            if gx.requires_grad:
                g2x, = torch.autograd.grad(gx, x, ggx, allow_unused=True)
                g2x = torch.zeros_like(x) if g2x is None else g2x
                if O.ops.ACT[act][4]:
                    ref = O.ops.bias_act_grad(ggx_np, x64, b64, y_or, act=act, order=2, dy1=gy_np, plugin_semantics=True, **kw32)
                else:
                    ref = np.zeros_like(x64)
                assert np.abs(g2x.cpu().numpy() - ref).max() < 1e-10 * max(1.0, np.abs(ref).max()), (act, tag)
                assert np.abs(g2x.cpu().numpy() - g[f'ba_{act}_{tag}_g2x']).max() < 1e-5 * max(1.0, np.abs(ref).max())


def test_bias_act_large_and_unaligned():
    from pix2pix3d_b200.torch_utils.ops import bias_act
    torch.manual_seed(0)
    x = torch.randn(3, 7, 33, 31, device='cuda')          # numel not a multiple of 4, step_b odd
    b = torch.randn(7, device='cuda')
    y = bias_act.bias_act(x, b, act='lrelu', clamp=1.5)
    ref = bias_act.bias_act(x.cpu(), b.cpu(), act='lrelu', clamp=1.5)
    assert rel_err(y.cpu().numpy(), ref.numpy()) < 1e-6
    xs = x.flatten()[1:].reshape(-1)                       # misaligned base pointer
    y2 = bias_act.bias_act(xs, None, act='tanh')
    assert rel_err(y2.cpu().numpy(), torch.tanh(xs).cpu().numpy()) < 2e-6
    h = torch.randn(4, 128, 65, 65, device='cuda', dtype=torch.float16)
    bh = torch.randn(128, device='cuda', dtype=torch.float16)
    yh = bias_act.bias_act(h, bh, act='lrelu', gain=1.2, clamp=256)
    rh = bias_act.bias_act(h.float().cpu(), bh.float().cpu(), act='lrelu', gain=1.2, clamp=256)
    assert rel_err(yh.float().cpu().numpy(), rh.numpy()) < 2e-3


UP_CFGS = {
    'post_tconv': dict(f='f4', up=1, down=1, padding=[1, 1, 1, 1], gain=4),
    'skip_up': dict(f='f4', up=2, down=1, padding=[2, 1, 2, 1], gain=4),
    'down2': dict(f='f4', up=1, down=2, padding=[1, 1, 1, 1], gain=1),
    'pre_sconv': dict(f='f4', up=1, down=1, padding=[2, 2, 2, 2], gain=1),
    'sep8_up2': dict(f='f8', up=2, down=1, padding=[4, 3, 4, 3], gain=4),
    'odd': dict(f='f35', up=[3, 2], down=[2, 1], padding=[2, 0, -1, 3], gain=0.7, flip_filter=True),
    'crop': dict(f='f4', up=1, down=1, padding=[-1, 2, 0, -2], gain=1),
    'identity': dict(f=None, up=1, down=1, padding=0, gain=1),
}


@pytest.mark.parametrize('dtype', [torch.float32, torch.float16, torch.float64])
def test_upfirdn2d_variants(dtype):
    from pix2pix3d_b200.torch_utils.ops import upfirdn2d
    g = load_golden('ops')
    fm = {k: torch.from_numpy(g['up_' + k]).cuda() for k in ('f4', 'f8', 'f35')}
    x = torch.from_numpy(g['up_x']).cuda().to(dtype)
    tol = {torch.float32: 2e-6, torch.float64: 2e-6, torch.float16: 2e-3}[dtype]
    for name, kw in UP_CFGS.items():
        kw = dict(kw)
        f = fm.get(kw.pop('f'))
        y = upfirdn2d.upfirdn2d(x, f, **kw)
        assert y.dtype == dtype and tuple(y.shape) == g[f'up_{name}_y'].shape, name
        assert rel_err(y.double().cpu().numpy(), g[f'up_{name}_y']) < tol, (name, dtype)
        if dtype == torch.float32:
            yc = upfirdn2d.upfirdn2d(x.contiguous(memory_format=torch.channels_last), f, **kw)
            assert rel_err(yc.cpu().numpy(), g[f'up_{name}_y']) < tol, name + ' channels_last'


def test_upfirdn2d_hot_shapes_and_gradient():
    from pix2pix3d_b200.torch_utils.ops import upfirdn2d
    torch.manual_seed(0)
    f = upfirdn2d.setup_filter([1, 3, 3, 1]).cuda()
    for (n, c, h) in ((2, 16, 65), (1, 96, 32), (2, 5, 129)):
        x = torch.randn(n, c, h, h, device='cuda')
        y = upfirdn2d.upfirdn2d(x, f, padding=[1, 1, 1, 1], gain=4)
        ref = O.ops.upfirdn2d(x.cpu().numpy(), f.cpu().numpy(), padding=[1, 1, 1, 1], gain=4)
        assert rel_err(y.cpu().numpy(), ref) < 2e-6
        y = upfirdn2d.upsample2d(x, f)
        ref = O.ops.upsample2d(x.cpu().numpy(), f.cpu().numpy())
        assert rel_err(y.cpu().numpy(), ref) < 2e-6
        y = upfirdn2d.downsample2d(x, f)
        ref = O.ops.downsample2d(x.cpu().numpy(), f.cpu().numpy())
        assert rel_err(y.cpu().numpy(), ref) < 2e-6
    x = torch.randn(1, 2, 6, 7, device='cuda', dtype=torch.float64, requires_grad=True)
    f64 = f
    assert torch.autograd.gradcheck(lambda a: upfirdn2d.upfirdn2d(a, f64, up=2, padding=[2, 1, 2, 1], gain=4), (x,))
    assert torch.autograd.gradcheck(lambda a: upfirdn2d.upfirdn2d(a, f64, down=2, padding=[1, 1, 1, 1]), (x,))
    assert torch.autograd.gradgradcheck(lambda a: upfirdn2d.upfirdn2d(a, f64, padding=[1, 1, 1, 1]), (x,))


def test_filtered_lrelu_cuda_matches_oracle_and_reference():
    from pix2pix3d_b200.torch_utils.ops import filtered_lrelu
    g = load_golden('ops')
    t = lambda k: torch.from_numpy(g[k]).cuda()
    y = filtered_lrelu.filtered_lrelu(t('fl_x'), t('up_f4'), t('fl_fd'), t('fl_b'), up=2, down=2, padding=[3, 2, 3, 2], clamp=0.8)
    assert rel_err(y.cpu().numpy(), g['fl_up2_down2']) < 2e-6
    ref = O.ops.filtered_lrelu(g['fl_x'], g['up_f4'], g['fl_fd'], g['fl_b'], up=2, down=2, padding=[3, 2, 3, 2], clamp=0.8)
    assert rel_err(y.cpu().numpy(), ref) < 2e-6
    x = t('fl_x').double().requires_grad_(True)
    assert torch.autograd.gradcheck(lambda a: filtered_lrelu.filtered_lrelu(a, t('up_f4'), t('fl_fd'), None, up=2, down=2, padding=[3, 2, 3, 2]), (x,))


def test_dual_discriminator_cuda_forward():
    from pix2pix3d_b200.training.dual_discriminator import DualDiscriminator
    g = load_golden('ops')
    t = lambda k: torch.from_numpy(g[k]).cuda()
    torch.manual_seed(31)
    D = DualDiscriminator(c_dim=25, img_resolution=64, img_channels=3, channel_base=1024, channel_max=32, mapping_kwargs={},
                          epilogue_kwargs={'mbstd_group_size': 2}).eval().requires_grad_(False).cuda()
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    with torch.no_grad():
        out = D({'image': t('dd_image'), 'image_raw': t('dd_image_raw')}, t('dd_c').clone(), force_fp32=True)
    assert rel_err(out.cpu().numpy(), g['dd_logits']) < 1e-3


@pytest.mark.parametrize('dtype', [torch.float16, torch.float32, torch.float64])
@pytest.mark.parametrize('shapes', [
    ((2, 16, 8, 8), (2, 16, 1, 1), (2, 1, 8, 8)),        # modulated_conv2d: x * dcoefs + noise (networks_stylegan2.py:79-82), vector path
    ((3, 5, 7, 9), (3, 5, 1, 1), (7, 9)),                # odd sizes: scalar path, lower-rank noise
    ((2, 4, 6, 8), (2, 4, 6, 8), ()),                    # the gradient form: dout * b + 0
    ((1, 1, 4, 16), (2, 3, 1, 1), (2, 1, 4, 1)),         # every operand broadcast somewhere
    ((5, 12), (12,), (5, 1)),
])
def test_fma_kernel_matches_addcmul(dtype, shapes):
    from pix2pix3d_b200 import _lib
    from pix2pix3d_b200.torch_utils.ops import fma
    torch.manual_seed(3)
    a, b, c = (torch.randn(s, device='cuda', dtype=torch.float64).to(dtype) for s in shapes)
    before = _lib.launch_count
    y = fma.fma(a, b, c)
    assert _lib.launch_count == before + 1
    ref = torch.addcmul(c, a, b)
    assert y.shape == ref.shape and y.dtype == ref.dtype
    tol = {torch.float16: 1e-3, torch.float32: 2e-7, torch.float64: 1e-15}[dtype]
    assert rel_err(y.double().cpu().numpy(), ref.double().cpu().numpy()) <= tol
    if dtype == torch.float16:       # fp32 arithmetic, one rounding
        exact = (a.double() * b.double() + c.double()).half()
        assert (y != exact).float().mean().item() < 1e-3


def test_fma_gradients_first_and_second_order():
    from pix2pix3d_b200.torch_utils.ops import fma
    torch.manual_seed(4)
    a = torch.randn(2, 3, 4, 4, device='cuda', dtype=torch.float64, requires_grad=True)
    b = torch.randn(2, 3, 1, 1, device='cuda', dtype=torch.float64, requires_grad=True)
    c = torch.randn(2, 1, 4, 4, device='cuda', dtype=torch.float64, requires_grad=True)
    assert torch.autograd.gradcheck(fma.fma, (a, b, c))
    assert torch.autograd.gradgradcheck(fma.fma, (a, b, c))


@pytest.mark.parametrize('act', ['linear', 'lrelu', 'relu'])
@pytest.mark.parametrize('b,fin,fout,bias', [(4, 512, 512, True), (1, 25, 512, True), (17, 96, 33, False), (64, 512, 100, True)])
def test_fully_connected_layer_small_batch_kernel(act, b, fin, fout, bias):
    """FullyConnectedLayer.forward on p3d_fc_bias_act (no gradients, batch <= 64) against its torch formulation in float64."""
    from pix2pix3d_b200 import _lib
    from pix2pix3d_b200.training.networks_stylegan2 import FullyConnectedLayer
    torch.manual_seed(9)
    fc = FullyConnectedLayer(fin, fout, bias=bias, activation=act, lr_multiplier=0.01, bias_init=0.3).cuda()
    x = torch.randn(b, fin, device='cuda')
    before = _lib.launch_count
    with torch.no_grad():
        y = fc(x)
    assert _lib.launch_count == before + 1
    w = fc.weight.detach().double() * fc.weight_gain
    ref = x.double() @ w.t()
    if bias:
        ref = ref + fc.bias.detach().double() * fc.bias_gain
    if act == 'lrelu':
        ref = torch.nn.functional.leaky_relu(ref, 0.2) * np.sqrt(2)
    if act == 'relu':
        ref = torch.relu(ref) * np.sqrt(2)
    assert rel_err(y.cpu().numpy(), ref.cpu().numpy()) < 1e-5
    # gradients required -> the autograd formulation (cuBLAS + p3d_bias_act), same values
    x2 = x.clone().requires_grad_(True)
    y2 = fc(x2)
    assert y2.requires_grad and rel_err(y2.detach().cpu().numpy(), ref.cpu().numpy()) < 1e-5
