"""p3d_conv_wgrad (tcconv.conv_wgrad) against a float64 model of each launch, element by element:

    |dW - dW64| <= eps_acc(k16 slices per split + split-K partials) * S + floor

dW64 is torch's float64 weight gradient of the node and S the same on absolute values. Per 64-pixel k-step a CTA adds 4 k16
slices of each of the three passes (hi*hi, hi*lo, lo*hi); the missing lo*lo term and the lo rounding are 2^-22 of |p q| each,
inside the per-slice allowance. `floor` covers the fp16 subnormal spacing of the lo halves (2^-24 of the scaled operands per
product). Cases: split-K schedules whose unit counts land on the SM count's edges, every layer shape of the full-size afhq
training generator at batch 4, magnitudes 1e-9..1e3 and an all-zero dY, the ragged shapes of test_gpu_native_conv,
bit-reproducibility, a planted fault, and a replay of a generator training step (G.mapping with its Encoder, then
G.synthesis) in which every weight-gradient launch is checked while its inputs are alive.
"""
import pytest
import torch
import torch.nn.functional as F

from test_gpu_conv_persistent import eps_acc

pytestmark = pytest.mark.gpu


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def model(p, q, k, stride):
    """float64 dW[m, n, ky, kx] = sum P[b,m,y,x] Q[b,n,s*y+ky-pad, s*x+kx-pad] and the same on absolute values."""
    def f(a, b):
        a, b = a.double(), b.double()
        m, n = a.shape[1], b.shape[1]
        if stride == 1:
            return torch.nn.grad.conv2d_weight(b, (m, n, k, k), a, padding=k // 2)
        return torch.nn.grad.conv2d_weight(b, (m, n, 3, 3), a, stride=2)
    return f(p, q), f(p.abs(), q.abs())


def worst_ratio(dw, p, q, k, stride, splits, p_scale=None, q_scale=None, drop=None):
    """max |dW - dW64| / tol over the elements of one launch (drop: remove a term from the MODEL, for the planted-fault test)."""
    from pix2pix3d_b200 import tcconv
    ref, s = model(p, q, k, stride)
    if drop == 'hi*lo':
        # the model without the hi*lo pass: P_hi * Q_hi + P_lo * Q_hi
        sp = tcconv.pow2_scale(p) if p_scale is None else p_scale
        sq = tcconv.pow2_scale(q) if q_scale is None else q_scale
        ph = (p * sp).half().float()
        qh = (q * sq).half().float()
        ref = (model(ph, qh, k, stride)[0] + model(p * sp - ph, qh, k, stride)[0]) / (sp.double() * sq.double())
    b, m, h, w = p.shape
    plan = tcconv.wgrad_plan(b, m, q.shape[1], (h, w), k, stride, _sms(), splits=splits)
    steps = max(r[1] - r[0] for r in plan['ranges'])
    sp = (tcconv.pow2_scale(p) if p_scale is None else p_scale).double()
    sq = (tcconv.pow2_scale(q) if q_scale is None else q_scale).double()
    floor = b * h * w * 2.0 ** -24 * 2.0 ** 12 / (sp * sq)
    tol = eps_acc(3 * 4 * steps + splits) * s + floor
    return float(((dw.double() - ref).abs() / tol).max())


def run(p, q, k, stride, splits=None):
    from pix2pix3d_b200 import tcconv
    b, m, h, w = p.shape
    plan = tcconv.wgrad_plan(b, m, q.shape[1], (h, w), k, stride, _sms(), splits=splits)
    dw = tcconv.conv_wgrad(p, q, k, stride, splits=plan['splits'])
    torch.cuda.synchronize()
    return dw, plan


def operands(b, m, n, h, w, stride, seed=0, scale=1.0):
    g = torch.Generator(device='cuda').manual_seed(seed)
    p = torch.randn(b, m, h, w, device='cuda', generator=g) * scale
    qh, qw = (h, w) if stride == 1 else (2 * h + 1, 2 * w + 1)
    q = torch.randn(b, n, qh, qw, device='cuda', generator=g)
    return p, q


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('target', ['1', 'SMs-1', 'SMs', 'SMs+1', '3.5 waves'])
def test_unit_counts_around_the_sm_count(target):
    """One 128 x 64 output tile of a 1x1 layer (4 images of 96^2: 576 k-steps), split into exactly as many CTAs as the
    schedule edge asks for; and a 3x3 layer whose 9 tiles x splits land just past one wave."""
    sms = _sms()
    want = {'1': 1, 'SMs-1': sms - 1, 'SMs': sms, 'SMs+1': sms + 1, '3.5 waves': 7 * sms // 2}[target]
    p, q = operands(4, 128, 64, 96, 96, 1, seed=want)
    dw, plan = run(p, q, 1, 1, splits=want)
    print(f'{target}: units {plan["units"]} ({plan["units"] / sms:.2f} SMs), {plan["total_k"]} k-steps')
    assert plan['units'] == want
    assert worst_ratio(dw, p, q, 1, 1, want) <= 1.0
    splits = sms // 9 + 1
    dw, plan = run(p, q, 3, 1, splits=splits)
    assert plan['units'] == 9 * splits > sms
    assert worst_ratio(dw, p, q, 3, 1, splits) <= 1.0


# every weight-gradient shape of the afhq / seg2cat_512 training generator at batch 4 (backbone, ToRGB, up layers, Encoder)
AFHQ_LAYERS = [
    # name, P channels, Q channels, H, W, k, stride
    ('backbone 3x3 4^2', 512, 512, 4, 4, 3, 1), ('backbone 3x3 8^2', 512, 512, 8, 8, 3, 1),
    ('backbone 3x3 16^2', 512, 512, 16, 16, 3, 1), ('backbone 3x3 32^2', 512, 512, 32, 32, 3, 1),
    ('backbone 3x3 64^2', 256, 256, 64, 64, 3, 1), ('backbone 3x3 128^2', 128, 128, 128, 128, 3, 1),
    ('backbone 3x3 256^2', 64, 64, 256, 256, 3, 1),
    ('ToRGB 1x1 64^2', 96, 256, 64, 64, 1, 1), ('ToRGB 1x1 256^2', 96, 64, 256, 256, 1, 1),
    ('up 3x3 s2 32->65', 512, 512, 32, 32, 3, 2), ('up 3x3 s2 128->257', 128, 128, 128, 128, 3, 2),
    ('Encoder fromrgb 1x1 512^2', 64, 19, 512, 512, 1, 1), ('Encoder conv0 3x3 512^2', 64, 64, 512, 512, 3, 1),
    ('Encoder skip 1x1 256^2', 128, 64, 256, 256, 1, 1), ('Encoder conv1 s2 513->256', 128, 64, 256, 256, 3, 2),
    ('Encoder conv1 s2 65->32', 512, 512, 32, 32, 3, 2),
]


@pytest.mark.parametrize('layer', AFHQ_LAYERS, ids=[l[0] for l in AFHQ_LAYERS])
def test_full_size_training_layers(layer):
    name, m, n, h, w, k, s = layer
    p, q = operands(4, m, n, h, w, s, seed=m + n + h)
    p = p * 1e-6                                            # dY-sized gradients
    dw, plan = run(p, q, k, s)
    r = worst_ratio(dw, p, q, k, s, plan['splits'])
    print(f'{name}: units {plan["units"]}, splits {plan["splits"]}, worst err/tol {r:.3g}')
    assert r <= 1.0


@pytest.mark.parametrize('scale', [1e-9, 1e-6, 1e-3, 1.0, 1e3])
@pytest.mark.parametrize('stride', [1, 2])
def test_magnitudes(scale, stride):
    p, q = operands(2, 96, 104, 17, 19, stride, seed=7, scale=scale)
    dw, plan = run(p, q, 3, stride)
    assert worst_ratio(dw, p, q, 3, stride, plan['splits']) <= 1.0


def test_all_zero_gradient():
    p, q = operands(2, 64, 64, 20, 20, 1)
    dw, _ = run(torch.zeros_like(p), q, 3, 1)
    assert torch.count_nonzero(dw) == 0


@pytest.mark.parametrize('b,m,n,h,w,k', [(4, 64, 64, 32, 32, 3), (2, 96, 128, 64, 64, 3), (3, 64, 6, 40, 24, 1),
                                         (2, 512, 512, 16, 16, 3), (2, 3, 128, 64, 64, 1), (1, 104, 96, 17, 19, 3)])
def test_ragged_shapes_of_the_native_node(b, m, n, h, w, k):
    p, q = operands(b, m, n, h, w, 1, seed=b * h)
    dw, plan = run(p, q, k, 1)
    assert worst_ratio(dw, p, q, k, 1, plan['splits']) <= 1.0


def test_bit_reproducible():
    """Same dW bits on a second run, with the planned split count and with one k-step per split."""
    p, q = operands(2, 128, 64, 33, 31, 2, seed=3)
    a, _ = run(p, q, 3, 2)
    b, _ = run(p, q, 3, 2)
    assert torch.equal(a, b)
    p1, q1 = operands(1, 64, 64, 7, 8, 1, seed=4)                     # 1 image, 100 grid pixels: 2 k-steps
    total = run(p1, q1, 3, 1, splits=1)[1]['total_k']
    x1, _ = run(p1, q1, 3, 1, splits=total)
    x2, _ = run(p1, q1, 3, 1, splits=total)
    assert torch.equal(x1, x2)


def test_bound_rejects_planted_faults():
    """The model without the hi*lo pass is rejected (at about 4x the bound; the real model stays near 0.01 of it)."""
    p, q = operands(2, 64, 64, 24, 24, 1, seed=9)
    dw, plan = run(p, q, 3, 1)
    assert worst_ratio(dw, p, q, 3, 1, plan['splits']) <= 1.0
    r = worst_ratio(dw, p, q, 3, 1, plan['splits'], drop='hi*lo')
    print(f'dropped hi*lo: worst err/tol {r:.3g}')
    assert r > 2.0


# ---------------------------------------------------------------------------------------------------------------------
def test_strided_node_matches_fp64():
    """conv2d(stride 2, padding 0) of the Encoder's down layers: forward, input and weight gradients on libp3d."""
    from pix2pix3d_b200 import _lib
    from pix2pix3d_b200.torch_utils.ops import conv2d_gradfix, native_conv
    from conftest import rel_err
    torch.manual_seed(2)
    for b, cin, cout, h in [(4, 64, 128, 32), (2, 96, 104, 17)]:
        x = torch.randn(b, cin, 2 * h + 1, 2 * h + 1, device='cuda', requires_grad=True)
        w = (torch.randn(cout, cin, 3, 3, device='cuda') / (cin * 9) ** 0.5).requires_grad_(True)
        n0 = _lib.launch_count
        with native_conv.first_order():
            y = conv2d_gradfix.conv2d(x, w, stride=2, padding=0)
        assert _lib.launch_count - n0 >= 3 and tuple(y.shape) == (b, cout, h, h)
        gy = torch.randn_like(y) * 1e-6
        dx, dw = torch.autograd.grad((y * gy).sum(), [x, w])
        xr, wr = x.detach().double().requires_grad_(True), w.detach().double().requires_grad_(True)
        yr = F.conv2d(xr, wr, stride=2)
        dxr, dwr = torch.autograd.grad((yr * gy.double()).sum(), [xr, wr])
        assert rel_err(y.detach().cpu().numpy(), yr.detach().cpu().numpy()) < 2e-5
        assert rel_err(dx.cpu().numpy(), dxr.cpu().numpy()) < 2e-5
        assert rel_err(dw.cpu().numpy(), dwr.cpu().numpy()) < 2e-5
        with native_conv.first_order():
            y = conv2d_gradfix.conv2d(x, w, stride=2, padding=0)
        (g,) = torch.autograd.grad(y.sum(), [x], create_graph=True)
        with pytest.raises(RuntimeError):                       # first-order only
            g.sum().backward()


def test_encoder_training_gradients_use_the_native_node():
    """G.mapping with a label map (the Encoder: fromrgb, conv0, the strided conv1, skips) and G.synthesis, differentiated as in a
    Gmain phase: every weight-gradient launch against the float64 model while its inputs are alive (and ATen's fp32 weight
    gradient of the same operands against the same bound, for scale). Then the mapping network's parameter gradients three
    ways: native nodes, ATen, and native nodes with ATen's weight gradients, which isolates p3d_conv_wgrad. (A float64 run of
    the whole mapping network is not available: its modules cast activations to fp32.)"""
    from make_golden import SYNTH_CASES, build_generator
    import pix2pix3d_b200.training.triplane_cond as tc
    from conftest import load_golden, rel_err
    from pix2pix3d_b200 import _lib
    from pix2pix3d_b200.torch_utils.ops import native_conv
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    case = dict(SYNTH_CASES['seg_tiny'], in_res=64)              # Encoder at 64^2: its strided layers reach the native node
    G = build_generator(tc, case).cuda().train().requires_grad_(True)
    c = torch.from_numpy(load_golden('synthesis_seg_tiny')['c']).cuda()
    g = torch.Generator().manual_seed(4)
    z = torch.randn(c.shape[0], 32, generator=g).cuda()
    blocks = torch.randint(0, case['semantic_channels'], (c.shape[0], 1, 4, 4), generator=g)
    mask = blocks.repeat_interleave(case['in_res'] // 4, 2).repeat_interleave(case['in_res'] // 4, 3).cuda()
    from pix2pix3d_b200 import tcconv
    orig, rows = tcconv.conv_wgrad, []

    def checked(p, q, k, stride, p_scale=None, q_scale=None, splits=None):
        dw = orig(p, q, k, stride, p_scale=p_scale, q_scale=q_scale, splits=splits)
        torch.cuda.synchronize()
        b, m, h, w = p.shape
        plan = tcconv.wgrad_plan(b, m, q.shape[1], (h, w), k, stride, _sms(), splits=splits)
        r = worst_ratio(dw, p, q, k, stride, plan['splits'], p_scale=p_scale, q_scale=q_scale)
        # ATen's fp32 weight gradient of the same operands, held to the same bound (for scale)
        m, n = p.shape[1], q.shape[1]
        kw = dict(padding=k // 2) if stride == 1 else dict(stride=2)
        aten = torch.nn.grad.conv2d_weight(q.detach().float(), (m, n, k, k), p.detach().float(), **kw)
        ra = worst_ratio(aten, p, q, k, stride, plan['splits'], p_scale=p_scale, q_scale=q_scale)
        rows.append(f'P {tuple(p.shape)} Q {tuple(q.shape)} k {k} stride {stride} splits {plan["splits"]} worst err/tol {r:.3g} '
                    f'(ATen fp32 {ra:.3g})')
        assert r <= 1.0, rows[-1]
        return dw

    strided, orig_s2 = [], native_conv.conv2d_stride2

    def counted(x, w):
        strided.append(tuple(x.shape))
        return orig_s2(x, w)

    # a Gmain-shaped pass, mapping (Encoder) and synthesis both differentiated: every weight-gradient launch checked
    try:
        tcconv.conv_wgrad = checked
        native_conv.conv2d_stride2 = counted
        torch.manual_seed(5)
        ws = G.mapping(z, c, {'mask': mask, 'pose': c})
        out = G.synthesis(ws, c, noise_mode='const', neural_rendering_resolution=case['nrr'])
        (ws.square().mean() + out['image'].square().mean() + out['image_raw'].mean()).backward()
    finally:
        tcconv.conv_wgrad = orig
        native_conv.conv2d_stride2 = orig_s2
    print('\n'.join(rows))
    print('strided node inputs:', strided)
    assert strided and sum(' stride 2 ' in r for r in rows) > len(strided)   # Encoder down layers and synthesis up layers
    # the mapping network alone (no renderer, whose importance sampling turns fp32-level differences in the planes into
    # different sample depths): the same parameter gradients with the native nodes as with ATen's
    def aten_wgrad(p, q, k, stride, p_scale=None, q_scale=None, splits=None):
        kw = dict(padding=k // 2) if stride == 1 else dict(stride=2)
        return torch.nn.grad.conv2d_weight(q, (p.shape[1], q.shape[1], k, k), p, **kw)

    grads = []
    for on, wg in ((True, orig), (False, orig), (True, aten_wgrad)):
        native_conv.enabled = on
        try:
            tcconv.conv_wgrad = wg
            G.zero_grad(set_to_none=True)
            n0 = _lib.launch_count
            G.mapping(z, c, {'mask': mask, 'pose': c}).square().mean().backward()
            grads.append(({k: p.grad.detach().clone() for k, p in G.named_parameters() if p.grad is not None}, _lib.launch_count - n0))
        finally:
            native_conv.enabled = True
            tcconv.conv_wgrad = orig
    (ga, na), (gb, nb), (gc, _) = grads
    # the weight-gradient kernel alone: native nodes with p3d_conv_wgrad against the same nodes with ATen's weight gradients
    errs_w = sorted(((rel_err(ga[k].float().cpu().numpy(), gc[k].float().cpu().numpy()), k) for k in ga if gc[k].abs().max() > 0),
                    reverse=True)
    print('p3d_conv_wgrad vs ATen weight gradients under the native nodes:', ', '.join(f'{k} {e:.3g}' for e, k in errs_w[:4]))
    assert errs_w[0][0] < 1e-4, errs_w[0]
    assert na > nb
    assert ga.keys() == gb.keys() and any('conv1' in k for k in ga)
    errs = sorted(((rel_err(ga[k].float().cpu().numpy(), gb[k].float().cpu().numpy()), k) for k in ga if gb[k].abs().max() > 0),
                  reverse=True)
    print('native vs ATen, mapping network:', ', '.join(f'{k} {e:.3g}' for e, k in errs[:4]))
    # the whole chain (native forward and input gradients too) differs from ATen's at the level the synthesis test allows
    assert errs[0][0] < 2e-3, errs[0]

