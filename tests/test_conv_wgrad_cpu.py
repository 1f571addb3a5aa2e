"""Geometry of the tensor-core weight gradient (tcconv.wgrad_plan, run by p3d_conv_wgrad) checked on the CPU in float64: the
operands are laid out on the planned zero-bordered grid exactly as p3d_wgrad_operand writes them, every tap is a shifted
flattened GEMM over the planned split-K ranges, and the result must equal torch's weight gradient of each node. Also: which
shapes the strided node (native_conv.applies_strided) takes."""
import pytest
import torch

from pix2pix3d_b200 import tcconv


def place_p(x, plan):
    """P [B,C,H,W] -> [B,C,H*Wp] on its grid (p3d_wgrad_operand, stride 1, one phase), in float64."""
    b, c, h, w = x.shape
    g = torch.zeros(b, c, h, plan['wp'], dtype=torch.float64)
    g[..., :w] = x
    return g.reshape(b, c, -1)


def place_q(x, plan):
    """Q -> [B,phases,C,Hq*Wp]: the phases p3d_wgrad_operand writes, built with plain slicing, in float64."""
    b, c, hh, ww = x.shape
    wp, hq, top = plan['wp'], plan['hq'], plan['q_top']
    g = torch.zeros(b, plan['q_phases'], c, hq, wp, dtype=torch.float64)
    for ph in range(plan['q_phases']):
        if plan['stride'] == 1:
            dx = ph - (plan['q_phases'] - 1) // 2                   # phase = Q shifted left by dx columns
            src = x[..., max(dx, 0):ww + min(dx, 0)]
            g[:, ph, :, top:top + hh, max(-dx, 0):max(-dx, 0) + src.shape[-1]] = src
        else:
            ry, kx = divmod(ph, 3)
            src = x[:, :, ry::2, (kx & 1) + 2 * (kx >> 1)::2]          # rows 2 gy + ry, columns 2 (gx + (kx >> 1)) + (kx & 1)
            src = src[..., :hq, :wp]                                     # columns past W pair with P's zero columns only
            g[:, ph, :, :src.shape[2], :src.shape[3]] = src
    return g.reshape(b, plan['q_phases'], c, -1)


def planned_wgrad(p, q, k, stride, splits=None, sms=132):
    """dW as p3d_conv_wgrad computes it: per tap, per split-K range of 64-pixel k-steps, A[m, K] . B[n, K + off]; the splits
    summed in order."""
    b, m, h, w = p.shape
    n = q.shape[1]
    plan = tcconv.wgrad_plan(b, m, n, (h, w), k, stride, sms, splits=splits)
    for ph, off in plan['taps']:
        assert off >= 0 and off % 8 == 0 and 0 <= ph < plan['q_phases']      # aligned, non-negative TMA box starts
    lp, lq, nc = plan['Lp'], plan['Lq'], plan['nchunks']
    pg, qg = place_p(p, plan), place_q(q, plan)
    kk = nc * tcconv.WGRAD_BK
    a = torch.zeros(b, m, kk, dtype=torch.float64)
    a[..., :lp] = pg
    a = a.permute(1, 0, 2).reshape(m, -1)
    dw = torch.zeros(m, n, len(plan['taps']), dtype=torch.float64)
    for t, (ph, off) in enumerate(plan['taps']):
        bq = torch.zeros(b, n, kk, dtype=torch.float64)
        hi = min(kk, lq - off)                                   # B reads g + off; past Lq is the TMA's zero fill
        if hi > 0:
            bq[..., :hi] = qg[:, ph, :, off:off + hi]
        bq = bq.permute(1, 0, 2).reshape(n, -1)
        for k0, k1 in plan['ranges']:
            sl = slice(k0 * tcconv.WGRAD_BK, k1 * tcconv.WGRAD_BK)
            dw[:, :, t] += a[:, sl] @ bq[:, sl].T
    return dw.reshape(m, n, k, k), plan


SHAPES = [
    # B, P channels, Q channels, H, W
    (2, 64, 64, 16, 16),
    (1, 96, 104, 17, 19),
    (3, 64, 6, 40, 24),
    (2, 3, 96, 12, 10),
    (1, 1, 3, 9, 7),
    (2, 104, 1, 5, 13),
]


@pytest.mark.parametrize('b,m,n,h,w', SHAPES)
@pytest.mark.parametrize('k', [1, 3])
def test_stride1_plan_equals_conv2d_weight(b, m, n, h, w, k):
    torch.manual_seed(0)
    dy = torch.randn(b, m, h, w, dtype=torch.float64)          # P = dY [B, Cout, H, W]
    x = torch.randn(b, n, h, w, dtype=torch.float64)           # Q = X  [B, Cin, H, W]
    got, _ = planned_wgrad(dy, x, k, 1)
    ref = torch.nn.grad.conv2d_weight(x, (m, n, k, k), dy, padding=k // 2)
    torch.testing.assert_close(got, ref, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize('b,m,n,h,w', SHAPES)
def test_strided_plan_equals_conv2d_weight(b, m, n, h, w):
    """Encoder down layers: y = conv2d(x [B,I,2H+1,2W+1], w [O,I,3,3], stride 2); P = dY, Q = the four phases of x."""
    torch.manual_seed(1)
    dy = torch.randn(b, m, h, w, dtype=torch.float64)
    x = torch.randn(b, n, 2 * h + 1, 2 * w + 1, dtype=torch.float64)
    got, plan = planned_wgrad(dy, x, 3, 2)
    assert plan['q_phases'] == 6 and plan['hq'] == h + 1
    ref = torch.nn.grad.conv2d_weight(x, (m, n, 3, 3), dy, stride=2)
    torch.testing.assert_close(got, ref, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize('b,m,n,h,w', SHAPES)
def test_transposed_plan_equals_autograd(b, m, n, h, w):
    """Up layers: y = conv_transpose2d(x [B,I,H,W], w [I,O,3,3], stride 2) -> [B,O,2H+1,2W+1]; P = x, Q = the phases of dY,
    dW in torch's [in, out, 3, 3] order."""
    torch.manual_seed(2)
    x = torch.randn(b, m, h, w, dtype=torch.float64)
    wt = torch.randn(m, n, 3, 3, dtype=torch.float64, requires_grad=True)
    y = torch.nn.functional.conv_transpose2d(x, wt, stride=2)
    dy = torch.randn_like(y)
    (ref,) = torch.autograd.grad((y * dy).sum(), [wt])
    got, _ = planned_wgrad(x, dy, 3, 2)
    torch.testing.assert_close(got, ref, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize('splits', [1, 2, 3, 5, 'max'])
def test_split_k_ranges_cover_the_reduction(splits):
    torch.manual_seed(3)
    dy, x = torch.randn(2, 64, 11, 13, dtype=torch.float64), torch.randn(2, 96, 11, 13, dtype=torch.float64)
    total = tcconv.wgrad_plan(2, 64, 96, (11, 13), 3, 1, 132)['total_k']
    s = total if splits == 'max' else splits
    got, plan = planned_wgrad(dy, x, 3, 1, splits=s)
    assert plan['splits'] == s and plan['ranges'][0][0] == 0 and plan['ranges'][-1][1] == total
    assert all(a[1] == b[0] for a, b in zip(plan['ranges'], plan['ranges'][1:]))
    ref = torch.nn.grad.conv2d_weight(x, (64, 96, 3, 3), dy, padding=1)
    torch.testing.assert_close(got, ref, rtol=1e-12, atol=1e-12)


def test_plan_rows_and_scratch():
    """TMA row strides are multiples of 16 bytes; the scratch holds every split's padded tiles; the chosen split count fills the
    machine for the few-tile layers and stays 1-3 for the many-tile ones."""
    for (b, m, n, h, w, k, s) in [(4, 64, 64, 256, 256, 3, 2), (4, 512, 512, 16, 16, 3, 1), (4, 3, 128, 128, 128, 1, 1),
                                  (4, 256, 256, 33, 33, 3, 2), (4, 64, 19, 512, 512, 1, 1)]:
        p = tcconv.wgrad_plan(b, m, n, (h, w), k, s, 132)
        assert p['Lp'] == h * p['wp'] and p['wp'] % 8 == 0 and p['Lq'] == p['hq'] * p['wp']
        mp = p['m_tiles'] * tcconv.WGRAD_BM
        np_ = p['n_tiles'] * p['bn']
        assert p['scratch_floats'] == p['splits'] * k * k * mp * np_
        assert p['units'] == p['m_tiles'] * p['n_tiles'] * k * k * p['splits']
        assert 1 <= p['splits'] <= min(p['total_k'], tcconv.WGRAD_MAX_SPLITS)
    few = tcconv.wgrad_plan(4, 64, 64, (256, 256), 3, 2, 132)           # 9 tiles, ~16 k k-steps: split until the waves are full
    assert few['units'] / (-(-few['units'] // 132) * 132) >= 0.9
    many = tcconv.wgrad_plan(4, 512, 512, (16, 16), 3, 1, 132)          # 144 tiles, 76 k-steps
    assert many['splits'] <= 3


def _fake_cuda(t):
    """A CPU tensor that reports is_cuda (applies_strided only looks at shapes, dtypes and flags)."""
    class T(torch.Tensor):
        @property
        def is_cuda(self):
            return True
    return t.as_subclass(T)


@pytest.mark.parametrize('res', [512, 256, 128, 64, 32])
def test_applies_strided_takes_the_encoder_shapes(res):
    """The Encoder's DiscriminatorBlock.conv1 (down=2) after its FIR: x [B,C,res+1,res+1] -> [B,C',res/2,res/2], 3x3, stride 2,
    padding 0. padding=1 (the generic strided call) and even inputs are refused."""
    from pix2pix3d_b200.torch_utils.ops import native_conv
    x = _fake_cuda(torch.zeros(4, 64, res + 1, res + 1, requires_grad=True))
    w = torch.zeros(128, 64, 3, 3, requires_grad=True)
    args = ((2, 2), (0, 0), (1, 1), 1)
    with native_conv.first_order():
        big = (res // 2) ** 2 >= native_conv.min_pixels
        assert native_conv.applies_strided(x, w, None, *args) == big
        assert not native_conv.applies_strided(x, w, None, (2, 2), (1, 1), (1, 1), 1)
        xe = _fake_cuda(torch.zeros(4, 64, res, res, requires_grad=True))
        assert not native_conv.applies_strided(xe, w, None, *args)
        assert not native_conv.applies_strided(x, w, torch.zeros(128), *args)
        assert not native_conv.applies_strided(x, torch.zeros(208, 64, 3, 3), None, *args)
        with torch.no_grad():
            assert not native_conv.applies_strided(x, w, None, *args)
    assert not native_conv.applies_strided(x, w, None, *args)              # outside first_order()
