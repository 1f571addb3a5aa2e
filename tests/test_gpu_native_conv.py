"""fp32 training convolutions on the wgmma implicit GEMM (torch_utils/ops/native_conv.py): forward and both gradients against
fp64 ATen convolutions; dispatch rules of conv2d_gradfix (only inside first_order() regions, only the shapes the node covers)."""
import pytest
import torch

from conftest import rel_err

pytestmark = pytest.mark.gpu

CASES = [
    # B, Cin, Cout, H, W, k
    (4, 64, 64, 32, 32, 3),
    (2, 128, 96, 64, 64, 3),
    (3, 6, 64, 40, 24, 1),          # fromrgb-like: few input channels, non-square, not a multiple of the tile
    (2, 512, 512, 16, 16, 3),
    (2, 128, 3, 64, 64, 1),         # ToRGB-like
    (1, 96, 104, 17, 19, 3),        # ragged spatial size, padded input channels, ragged output channels
]


@pytest.mark.parametrize('b,cin,cout,h,w,k', CASES)
def test_forward_and_gradients_match_fp64(b, cin, cout, h, w, k):
    from pix2pix3d_b200 import _lib
    from pix2pix3d_b200.torch_utils.ops import conv2d_gradfix, native_conv
    dev = torch.device('cuda')
    torch.backends.cudnn.allow_tf32 = False                 # the weight gradient is ATen's: keep it true fp32
    torch.manual_seed(0)
    x = torch.randn(b, cin, h, w, device=dev, requires_grad=True)
    wt = (torch.randn(cout, cin, k, k, device=dev) / (cin * k * k) ** 0.5).requires_grad_(True)
    n0 = _lib.launch_count
    with native_conv.first_order():
        y = conv2d_gradfix.conv2d(x, wt, padding=k // 2)
    assert _lib.launch_count - n0 >= 3, 'the native node was expected'
    gy = torch.randn_like(y) * 1e-6                         # gradients are tiny in practice: the node must not lose them in fp16
    dx, dw = torch.autograd.grad((y * gy).sum(), [x, wt])
    xr, wr = x.detach().double().requires_grad_(True), wt.detach().double().requires_grad_(True)
    yr = torch.nn.functional.conv2d(xr, wr, padding=k // 2)
    dxr, dwr = torch.autograd.grad((yr * gy.double()).sum(), [xr, wr])
    assert rel_err(y.detach().cpu().numpy(), yr.detach().cpu().numpy()) < 2e-5
    assert rel_err(dx.cpu().numpy(), dxr.cpu().numpy()) < 2e-5
    assert rel_err(dw.cpu().numpy(), dwr.cpu().numpy()) < 1e-4          # ATen fp32 weight gradient (TF32 may be on in this process)


def test_dispatch_rules():
    """(also: more than 128 channels must come in whole 128-channel tiles -- 208 goes to ATen)"""
    from pix2pix3d_b200 import _lib
    from pix2pix3d_b200.torch_utils.ops import conv2d_gradfix, native_conv
    dev = torch.device('cuda')
    x = torch.randn(2, 64, 32, 32, device=dev, requires_grad=True)
    w = torch.randn(64, 64, 3, 3, device=dev, requires_grad=True)

    def launches(fn):
        n0 = _lib.launch_count
        fn()
        return _lib.launch_count - n0

    assert launches(lambda: conv2d_gradfix.conv2d(x, w, padding=1)) == 0                        # outside first_order(): ATen
    with native_conv.first_order():
        assert launches(lambda: conv2d_gradfix.conv2d(x, w, padding=1)) > 0
        assert launches(lambda: conv2d_gradfix.conv2d(x, w, padding=1, stride=2)) == 0          # strided: not covered
        w208 = torch.randn(208, 64, 3, 3, device=dev, requires_grad=True)
        assert launches(lambda: conv2d_gradfix.conv2d(x, w208, padding=1)) == 0                # ragged beyond one channel tile
        assert launches(lambda: conv2d_gradfix.conv2d(x.half(), w.half(), padding=1)) == 0      # fp16 layers stay on cuDNN
        assert launches(lambda: conv2d_gradfix.conv2d(x, w, bias=torch.zeros(64, device=dev), padding=1)) == 0
        with torch.no_grad():
            assert launches(lambda: conv2d_gradfix.conv2d(x, w, padding=1)) == 0                # no gradient needed: generic path
        # double backward is refused loudly, not computed wrongly
        y = conv2d_gradfix.conv2d(x, w, padding=1)
        (g,) = torch.autograd.grad(y.sum(), [x], create_graph=True)
        with pytest.raises(RuntimeError):
            g.sum().backward()
    assert native_conv._depth == 0


def test_generator_training_gradients_use_the_native_node():
    """A training-mode G.synthesis with gradients: same parameter gradients with the native convolutions as with ATen's."""
    import pix2pix3d_b200.training.triplane_cond as tc
    from make_golden import SYNTH_CASES, build_generator
    from conftest import load_golden
    from pix2pix3d_b200 import _lib
    from pix2pix3d_b200.torch_utils.ops import native_conv
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    case = SYNTH_CASES['seg_nrr64']
    g = load_golden('synthesis_seg_nrr64')
    G = build_generator(tc, case).cuda().train().requires_grad_(True)
    ws, c = torch.from_numpy(g['ws']).cuda(), torch.from_numpy(g['c']).cuda()
    grads = []
    for on in (True, False):
        native_conv.enabled = on
        try:
            G.zero_grad(set_to_none=True)
            torch.manual_seed(5)
            n0 = _lib.launch_count
            out = G.synthesis(ws, c, noise_mode='const', neural_rendering_resolution=case['nrr'])
            (out['image'].square().mean() + out['semantic'].square().mean() + out['image_raw'].mean()).backward()
            grads.append(({k: p.grad.detach().clone() for k, p in G.named_parameters() if p.grad is not None}, _lib.launch_count - n0))
        finally:
            native_conv.enabled = True
    (ga, na), (gb, nb) = grads
    assert na > nb                                            # more libp3d launches with the native node
    assert ga.keys() == gb.keys()
    worst = max(rel_err(ga[k].float().cpu().numpy(), gb[k].float().cpu().numpy()) for k in ga if gb[k].abs().max() > 0)
    assert worst < 2e-3, worst



@pytest.mark.parametrize('b,cin,cout,h,w', [(4, 64, 64, 16, 16), (2, 256, 128, 32, 32), (1, 512, 512, 16, 16), (2, 96, 104, 17, 19)])
def test_transposed_convolution_and_gradients_match_fp64(b, cin, cout, h, w):
    """conv_transpose2d(stride 2, padding 0) of the up=2 layers (conv2d_resample.py:114-128): forward on the merged phase GEMMs,
    input gradient on the stride-2 convolution, weight gradient on ATen."""
    from pix2pix3d_b200 import _lib
    from pix2pix3d_b200.torch_utils.ops import conv2d_gradfix, native_conv
    dev = torch.device('cuda')
    torch.backends.cudnn.allow_tf32 = False
    torch.manual_seed(1)
    x = torch.randn(b, cin, h, w, device=dev, requires_grad=True)
    wt = (torch.randn(cin, cout, 3, 3, device=dev) / (cin * 9) ** 0.5).requires_grad_(True)
    n0 = _lib.launch_count
    with native_conv.first_order():
        y = conv2d_gradfix.conv_transpose2d(x, wt, stride=2, padding=0)
    assert _lib.launch_count - n0 >= 3, 'the native node was expected'
    assert tuple(y.shape) == (b, cout, 2 * h + 1, 2 * w + 1)
    gy = torch.randn_like(y) * 1e-6
    dx, dw = torch.autograd.grad((y * gy).sum(), [x, wt])
    xr, wr = x.detach().double().requires_grad_(True), wt.detach().double().requires_grad_(True)
    yr = torch.nn.functional.conv_transpose2d(xr, wr, stride=2)
    dxr, dwr = torch.autograd.grad((yr * gy.double()).sum(), [xr, wr])
    assert rel_err(y.detach().cpu().numpy(), yr.detach().cpu().numpy()) < 2e-5
    assert rel_err(dx.cpu().numpy(), dxr.cpu().numpy()) < 2e-5
    assert rel_err(dw.cpu().numpy(), dwr.cpu().numpy()) < 1e-4
    # outside a first_order() region (the discriminators' R1 differentiates twice) the ATen node is used
    n1 = _lib.launch_count
    conv2d_gradfix.conv_transpose2d(x, wt, stride=2, padding=0)
    assert _lib.launch_count == n1
