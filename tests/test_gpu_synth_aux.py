"""The memory-bound helpers of a synthesis step (synth_aux.cu) against a float64 model of each launch.

Every step makes three kinds of launch besides the convolutions and the renderer: the FIR + noise + bias + lrelu + clamp tail
after each up=2 layer (`p3d_fir_act_nhwc*`), the weight modulation of every layer (`p3d_modulate_weights_batch`) and every
style affine (`p3d_affine_batch`). The convolution model takes the modulated weights as an input, so it cannot see an error in
them; this file holds each of these launches, and the upsampler and layout converters, to its own model.

- FIR tail, an interval model. Each output element is an interval [lo, hi] in float64, carried through the kernel's steps in
  its order: the exact FIR (the taps of setup_filter filters are dyadic, so float64 holds every product), widened by the fp32
  accumulation bound; the fp16 rounding of the FIR output (fp16 input) and again after the noise add; bias, lrelu, gain and
  clamp, each fp32 operation widening the interval by one unit roundoff; the final fp16 rounding. Rounding is monotone, so the
  rounded ends bound the result: `rn16(lo) <= got <= rn16(hi)`. Most intervals have width zero after the last rounding, so
  most elements are pinned bit for bit.
- Modulation: `v = w s pre_scale d out_scale`, `d = rsqrt(sum_i (s_i pre_scale)^2 sum_t w_it^2 + 1e-8)`, within a relative
  bound; `hi` is an fp16 rounding of a value within it, and hi + lo lies within it plus lo's own rounding.
- Affine, upsample: a gamma bound on the sum of absolute terms. Converters: bit for bit.

Every launch writes into a NaN-prefilled buffer longer than it needs, and nothing outside its own elements may change.
"""
import math
from collections import Counter

import numpy as np
import pytest
import torch
import torch.nn.functional as F

gpu = pytest.mark.gpu

U32 = 2.0 ** -24               # fp32 unit roundoff
TINY32 = 2.0 ** -149           # fp32 subnormal spacing: absolute floor of one fp32 rounding
LO_REL = 2.0 ** -22            # lo = rn16(v - hi): |v - hi| <= 2^-11 |v| is rounded to 11 bits
LO_ABS = 2.0 ** -25            # ... or to fp16's subnormal spacing 2^-24 (half of it)
PAD = 256                      # NaN elements before and after every output region
SQRT2 = math.sqrt(2.0)


def gamma(n):
    """Bound on the relative error of n fp32 roundings in a chain of sums of non-negative magnitudes (Higham's gamma_n)."""
    return n * U32 / (1 - n * U32)


# Accumulation bounds of the FIR, relative to S (the same FIR on |x| and |f|). A partial sum never exceeds S, and each
# rounding errs by at most U32 of its result:
#   separable kernel: per window row a horizontal 4-tap sum (one mul + 3 fma), then 4 vertical fma -> 4 + 4 roundings;
#   16-tap kernel: one chain of 16 fma; with a hi/lo input one more rounding of hi + lo per input element.
G_FIR = {'sep': gamma(8), 'gen': gamma(16), 'split': gamma(17)}


def f32(v):
    return float(np.float32(v))


def f16_of(v):
    """fp16(v) of an fp32 number (one rounding, as __float2half_rn)."""
    return float(np.float16(np.float32(v)))


def _ulp16(v):
    """fp16 spacing at |v| (subnormals share 2^-24), float64."""
    _, e = torch.frexp(v.abs())
    e = torch.clamp(e - 1, min=-14)
    return torch.ldexp(torch.ones_like(v), e - 10)


def rn16(v):
    """Round-half-even of float64 values to fp16, in float64. `.half()` on float64 can go through fp32 and round twice."""
    q = torch.round(v / _ulp16(v)) * _ulp16(v)
    return torch.where(q.abs() > 65504.0, torch.sign(v) * math.inf, q)


def _widen(lo, hi, exact=False):
    """One fp32 rounding of each end."""
    if exact:
        return lo, hi
    return lo - U32 * lo.abs() - TINY32, hi + U32 * hi.abs() + TINY32


def _pow2(g):
    return g != 0 and math.frexp(abs(g))[0] == 0.5


def _bits(t):
    return t.view({2: torch.int16, 4: torch.int32, 8: torch.int64}[t.element_size()])


def nan_buffer(shape, dtype, device='cuda', offset=PAD, misalign=0):
    """(buffer, view): a NaN-filled flat buffer and a contiguous view of `shape` at element `offset + misalign`."""
    n = int(np.prod(shape))
    buf = torch.full((offset + misalign + n + PAD,), float('nan'), dtype=dtype, device=device)
    return buf, buf[offset + misalign:offset + misalign + n].view(shape)


def untouched(buf, view):
    """Nothing outside `view` changed (bitwise, NaN-safe)."""
    start = (view.data_ptr() - buf.data_ptr()) // buf.element_size()
    rest = torch.cat([buf[:start], buf[start + view.numel():]])
    return torch.equal(_bits(rest), _bits(torch.full_like(rest, float('nan'))))


# ---------------------------------------------------------------------------------------------------------------------
# host rules, mirrored
# ---------------------------------------------------------------------------------------------------------------------
def fir_route(x, f, out_planes, act=3, alpha=0.2, clamp=-1.0, noise=None, variant=None):
    """Which kernel instance tcconv.fir_act_nhwc launches (p3d_fir_act_nhwc_sep's instance rule, or the 16-tap kernels)."""
    from pix2pix3d_b200 import tcconv
    variant = tcconv.FIR_VARIANT if variant is None else variant
    split_in = x.ndim == 5
    dt = 'f16' if x.dtype == torch.float16 else 'f32'
    if variant == 3 and not split_in and tcconv.separable_factors(f) is not None:
        so, nz = out_planes == 2, noise is not None
        c = f32(clamp)
        fast = act == 3 and 0.0 <= f32(alpha) <= 1.0 and (c < 0 or so or f16_of(c) == c)
        return ('sep', dt, so, nz, fast)
    return ('split',) if split_in else ('gen', dt)


FIR_INSTANCES = {('sep', dt, so, nz, fa) for dt in ('f16', 'f32') for so in (False, True) for nz in (False, True)
                 for fa in (False, True)} | {('gen', 'f16'), ('gen', 'f32'), ('split',)}


def modulate_paths(B, Cin, Cin_p, cin_off, ktaps):
    """modulate_row's path per 64-sample chunk: 'fast' (weights in registers) or 'general'."""
    nchunk = Cin_p // 8
    tstep = 256 // nchunk
    out = []
    for b0 in range(0, B, 64):
        nb = min(64, B - b0)
        out.append('fast' if cin_off == 0 and Cin % 8 == 0 and nb <= 8 and ktaps <= 3 * tstep else 'general')
    return out


def modulate_kernel(Cin_p, prepared):
    """tcconv.modulate_weights' choice: the streaming kernel (modulate_row) or the one-CTA-per-row kernel."""
    nchunk = Cin_p // 8
    return 't' if prepared and Cin_p % 8 == 0 and nchunk <= 256 and 256 % nchunk == 0 else 'plain'


# ---------------------------------------------------------------------------------------------------------------------
# FIR tail: interval model
# ---------------------------------------------------------------------------------------------------------------------
def fir_exact(x, f, pad0, out_hw, fir_gain, mirror=True):
    """x [B,ih,iw,C] float64 -> [B,oh,ow,C]: y[py,px] = sum f[3-j,3-i] fir_gain x[py+j-pady0, px+i-padx0], zero outside the
    image (upfirdn2d with flip_filter=False is a true convolution)."""
    b, ih, iw, c = x.shape
    oh, ow = out_hw
    padx, pady = pad0
    k = f.double() * fir_gain
    if mirror:
        k = k.flip([0, 1])
    xn = x.permute(0, 3, 1, 2)
    xp = F.pad(xn, [padx, max(0, ow + 3 - padx - iw), pady, max(0, oh + 3 - pady - ih)])[:, :, :oh + 3, :ow + 3]
    return F.conv2d(xp, k.to(x.device).expand(c, 1, 4, 4).contiguous(), groups=c).permute(0, 2, 3, 1)


def _lrelu_iv(lo, hi, alpha, max_form=False):
    """Image of [lo, hi] under lrelu (v > 0 ? v : fp32(alpha v)); piecewise linear with its kink at 0, so the extremes lie at
    the ends or at 0. max_form: max(v, alpha v), which equals lrelu only for 0 <= alpha <= 1."""
    def g(e):
        m = alpha * e
        y = torch.maximum(e, m) if max_form else torch.where(e > 0, e, m)
        w = torch.where(y == m, U32 * m.abs() + TINY32, torch.zeros_like(m))
        return y - w, y + w
    a0, a1 = g(lo)
    b0, b1 = g(hi)
    nlo, nhi = torch.minimum(a0, b0), torch.maximum(a1, b1)
    straddle = (lo < 0) & (hi > 0)
    return torch.where(straddle, torch.minimum(nlo, torch.zeros_like(nlo)), nlo), torch.where(straddle, torch.maximum(nhi, torch.zeros_like(nhi)), nhi)


def fir_model(x, f, noise, bias, out_planes, out_hw, pad0=(1, 1), fir_gain=4.0, act=3, alpha=0.2, act_gain=1.0, clamp=-1.0,
              kind=None, b0=0, b1=None, fault=None):
    """Intervals of one launch of tcconv.fir_act_nhwc (its arguments), samples b0..b1: {'lo16', 'hi16'}: bounds of the fp16
    output (hi plane), {'vlo', 'vhi'}: bounds of the fp32 value before the final rounding. `kind`: 'sep', 'gen' or 'split'
    (the accumulation bound); `fault` plants one error in the model (test_fir_bound_rejects_planted_faults)."""
    assert fir_gain in (1.0, 4.0)           # powers of two: the kernels' f * fir_gain is exact
    split_in = x.ndim == 5
    b1 = (x.shape[1] if split_in else x.shape[0]) if b1 is None else b1
    if split_in:
        xv = x[0, b0:b1].double() + x[1, b0:b1].double()
    else:
        xv = x[b0:b1].double()
    round16 = x.dtype == torch.float16 and not split_in
    if fault == 'pad_shift':
        pad0 = (pad0[0] + 1, pad0[1])
    mirror = fault != 'no_mirror'
    v = fir_exact(xv, f, pad0, out_hw, fir_gain, mirror)
    s = fir_exact(xv.abs(), f.abs(), pad0, out_hw, fir_gain, mirror)
    e = G_FIR[kind] * s
    lo, hi = v - e, v + e
    if round16 and fault != 'no_round16':
        lo, hi = rn16(lo), rn16(hi)
    if noise is not None:
        if noise.ndim == 2:
            nz = noise.double()[None, :, :, None]
        elif fault == 'noise_sample0':
            nz = noise[:1].double()[..., None]
        else:
            nz = noise[b0:b1].double()[..., None]
        lo, hi = _widen(lo + nz, hi + nz)
        if round16:
            lo, hi = rn16(lo), rn16(hi)
    if bias is not None:
        c = v.shape[-1]
        bv = bias[:c].double()
        if fault == 'bias_block':
            bv = bv.roll(-(64 if x.dtype == torch.float16 else 32))
        lo, hi = _widen(lo + bv, hi + bv)
    if act == 3:
        lo, hi = _lrelu_iv(lo, hi, f32(alpha), max_form=fault == 'max_form')
    g = f32(act_gain)
    lo, hi = _widen(torch.minimum(lo * g, hi * g), torch.maximum(lo * g, hi * g), exact=_pow2(g))
    c = f32(clamp)
    if c >= 0 and fault != 'round_then_clamp':
        lo, hi = lo.clamp(-c, c), hi.clamp(-c, c)
    lo16, hi16 = rn16(lo), rn16(hi)
    if c >= 0 and fault == 'round_then_clamp':
        # clamped after the final rounding, against the fp32 bound: saturated elements would have to come out at the clamp
        lo16, hi16, lo, hi = lo16.clamp(-c, c), hi16.clamp(-c, c), lo.clamp(-c, c), hi.clamp(-c, c)
    return dict(lo16=lo16, hi16=hi16, vlo=lo, vhi=hi)


def fir_check(y, m, out_planes, fault=None):
    """(elements outside the bound, worst err / tol) of the launch's output y [planes,n,oh,ow,C] against fir_model's m.

    hi plane: inside [rn16(vlo), rn16(vhi)]; its err / tol is the distance to [vlo, vhi] over half an fp16 ulp. hi + lo:
    within LO_REL |v| + LO_ABS of [vlo, vhi]."""
    hi = y[0].double()
    vlo, vhi = m['vlo'], m['vhi']
    bad = ~((hi >= m['lo16']) & (hi <= m['hi16']))
    dist = lambda t: torch.clamp(vlo - t, min=0) + torch.clamp(t - vhi, min=0)      # noqa: E731
    ratio = dist(hi) / (0.5 * _ulp16(hi))
    if out_planes == 2:
        lo = torch.zeros_like(hi) if fault == 'lo_zero' else y[1].double()
        tol = LO_REL * torch.maximum(vlo.abs(), vhi.abs()) + LO_ABS
        r2 = dist(hi + lo) / tol
        bad |= ~(r2 <= 1.0)
        ratio = torch.maximum(ratio, r2)
    ratio = torch.nan_to_num(ratio, nan=math.inf)
    return int(bad.sum()), float(ratio.max()) if ratio.numel() else 0.0


def fir_launch_check(x, f, noise, bias, out_planes, out_hw, kind, **kw):
    """Launch tcconv.fir_act_nhwc into a NaN buffer and check it against the model, a few samples at a time.
    Returns (outside, worst err / tol, zero-width fraction)."""
    from pix2pix3d_b200 import tcconv
    b = x.shape[1] if x.ndim == 5 else x.shape[0]
    c = x.shape[-1]
    buf, y = nan_buffer((out_planes, b, out_hw[0], out_hw[1], c), torch.float16, device=x.device)
    tcconv.fir_act_nhwc(x, f, noise, bias, out_planes, out_hw, out=y, **kw)
    torch.cuda.synchronize()
    assert untouched(buf, y), 'the launch wrote outside its output'
    return fir_check_all(y, x, f, noise, bias, out_planes, out_hw, kind, **kw)


def fir_check_all(y, x, f, noise, bias, out_planes, out_hw, kind, fault=None, **kw):
    b = x.shape[1] if x.ndim == 5 else x.shape[0]
    step = max(1, (1 << 22) // max(1, out_hw[0] * out_hw[1] * x.shape[-1]))
    bad, worst, zw, n = 0, 0.0, 0, 0
    for b0 in range(0, b, step):
        b1 = min(b, b0 + step)
        m = fir_model(x, f, noise, bias, out_planes, out_hw, kind=kind, b0=b0, b1=b1, fault=fault, **kw)
        k, r = fir_check(y[:, b0:b1], m, out_planes, fault=fault)
        bad, worst = bad + k, max(worst, r)
        zw += int((m['lo16'] == m['hi16']).sum())
        n += m['lo16'].numel()
    return bad, worst, zw / max(n, 1)


# ---------------------------------------------------------------------------------------------------------------------
# modulation model
# ---------------------------------------------------------------------------------------------------------------------
def modw_eps(Cin, ktaps):
    """Relative bound of one modulated weight. The demodulation sum has positive terms only: sum_t w^2 (ktaps roundings),
    (s pre)^2 (3), the per-lane fma chain (Cin / 32, or Cin ktaps / 256 in the one-CTA-per-row kernel) and the 5 + 8 adds of
    the reductions; d = rsqrt halves that error and adds 2 ulp (4 U32) for rsqrtf; s pre, x d and x w are three more. The bound
    below is about twice that sum."""
    return (ktaps + math.ceil(Cin / 32) + math.ceil(Cin * ktaps / 256) + 24) * U32


def modw_model(weight, styles, demodulate=True, pre_scale=1.0, cin_padded=None, out_scale=128.0, cin_offset=0, fault=None):
    """float64 [B, Op, ktaps, Ip] of one modulation launch (tcconv.modulate_weights' arguments), zero in padding rows and
    columns. It rounds nothing: the kernel rounds v (out_scale included) to hi and lo, where the reference rounds the
    unscaled weight; with a power-of-two out_scale the two differ only below 2^-14."""
    from pix2pix3d_b200 import tcconv
    o, i, kh, kw = weight.shape
    kk = kh * kw
    b = styles.shape[0]
    op, ip = tcconv.pad_to(o, 16), (cin_padded or tcconv.pad_to(i, 64))
    w = weight.detach().double().reshape(o, i, kk)
    s = styles.detach().double()
    if fault == 'styles_b8':
        s = s.roll(-8, 0)
    sp = s * f32(pre_scale)
    v = w[None] * sp[:, None, :, None]                                  # [B, O, I, kk]
    if demodulate:
        wsq = (w[:, :, 1:] if fault == 'tap_missing' else w).square().sum(-1)        # [O, I]
        d = (sp.square() @ wsq.t() + 1e-8).rsqrt()                      # [B, O]
        v = v * d[:, :, None, None]
    v = v * f32(out_scale)
    out = torch.zeros(b, op, kk, ip, dtype=torch.float64, device=weight.device)
    off = cin_offset + (8 if fault == 'cin_off8' else 0)
    out[:, :o, :, off:off + i] = v.permute(0, 1, 3, 2)
    return out


def modw_check(got, ref, eps, planes, fault=None):
    """(elements outside, worst err / tol) of a modulation output got [planes, B, Op, kk*Ip] against ref [B, Op, kk, Ip]."""
    hi = got[0].reshape(ref.shape).double()
    a = ref.abs()
    lo_b, hi_b = rn16(ref - eps * a), rn16(ref + eps * a)
    bad = ~((hi >= lo_b) & (hi <= hi_b))
    tol_h = eps * a + 0.5 * _ulp16(ref)
    ratio = (hi - ref).abs() / tol_h
    if planes == 2:
        lo = torch.zeros_like(hi) if fault == 'lo_zero' else got[1].reshape(ref.shape).double()
        tol = eps * a + LO_REL * a + LO_ABS
        r2 = (hi + lo - ref).abs() / tol
        bad |= ~(r2 <= 1.0)
        ratio = torch.maximum(ratio, r2)
    return int(bad.sum()), float(torch.nan_to_num(ratio, nan=math.inf).max())


def modulate_launch(weight, styles, demodulate=True, pre_scale=1.0, planes=1, cin_padded=None, cin_offset=0, prepared=None,
                    misalign=0):
    """tcconv.modulate_weights' launch, into a NaN buffer (view at `misalign` fp16 elements past a 16-byte boundary).
    Returns (buffer, output view, status)."""
    from pix2pix3d_b200 import _lib, tcconv
    s = styles.detach().float().contiguous()
    o, i, kh, kw = weight.shape
    b = s.shape[0]
    op, ip = tcconv.pad_to(o, 16), (cin_padded or tcconv.pad_to(i, 64))
    buf, out = nan_buffer((planes, b, op, kh * kw * ip), torch.float16, device=s.device, misalign=misalign)
    L = _lib.lib()
    if modulate_kernel(ip, prepared is not None) == 't':
        wt, wsq = prepared
        st = L.p3d_modulate_weights_t(_lib.ptr(wt), _lib.ptr(wsq), _lib.ptr(s), b, o, i, kh * kw, op, ip, cin_offset,
                                      int(demodulate), float(pre_scale), float(tcconv.WEIGHT_SCALE), planes, _lib.ptr(out),
                                      _lib.stream_ptr())
    else:
        w = weight.detach().float().contiguous()
        st = L.p3d_modulate_weights(_lib.ptr(w), _lib.ptr(s), b, o, i, kh * kw, op, ip, cin_offset, int(demodulate),
                                    float(pre_scale), float(tcconv.WEIGHT_SCALE), planes, _lib.ptr(out), _lib.stream_ptr())
    return buf, out, st


# ---------------------------------------------------------------------------------------------------------------------
# affine, upsample
# ---------------------------------------------------------------------------------------------------------------------
def affine_model(ws, weight, bias, meta, out_numel):
    """(expected, tol, written) of p3d_affine_batch: out[m.y + b m.z] = bias[r] + <ws[b, m.x], weight[r]>. Each lane runs
    w_dim / 32 fma, then 5 shuffle adds and the bias add: gamma(w_dim / 32 + 6) of the sum of absolute terms."""
    b, _, w_dim = ws.shape
    m = meta.long()
    x = ws.double()[:, m[:, 0]]                                          # [B, rows, w_dim]
    dot = (x * weight.double()[None]).sum(-1) + bias.double()[None]
    s = (x.abs() * weight.double().abs()[None]).sum(-1) + bias.double().abs()[None]
    idx = (m[:, 1][None] + torch.arange(b, device=ws.device)[:, None] * m[:, 2][None]).reshape(-1)
    exp = torch.zeros(out_numel, dtype=torch.float64, device=ws.device)
    tol = torch.zeros_like(exp)
    wr = torch.zeros(out_numel, dtype=torch.bool, device=ws.device)
    exp[idx], tol[idx], wr[idx] = dot.reshape(-1), gamma(math.ceil(w_dim / 32) + 6) * s.reshape(-1), True
    return exp, tol, wr


def upsample_model(x, f):
    """upfirdn2d.upsample2d(x, f) in float64 (NHWC) and its bound: every output is 4 fma of taps f * 4 (exact here)."""
    from test_gpu_conv_persistent import _upsample2d
    return _upsample2d(x.double(), f), gamma(4) * _upsample2d(x.double().abs(), f.abs())


# ---------------------------------------------------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------------------------------------------------
def asym_filter():
    """setup_filter([1, 2, 4, 1]): separable, asymmetric (a missing mirror shows), taps sum to a power of two (exact fp32
    factors, so separable_factors accepts it)."""
    from pix2pix3d_b200.torch_utils.ops import upfirdn2d
    return upfirdn2d.setup_filter([1, 2, 4, 1])


def rand_filter(seed=5):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(4, 4, generator=g) / 8


def fir_inputs(case, device='cuda', seed=0):
    """(x, f, noise, bias, kwargs) of one sweep case."""
    g = torch.Generator(device=device).manual_seed(seed)
    b, c = case['B'], case['C']
    ih, iw = case['in_hw']
    oh, ow = case['out_hw']
    x = torch.randn(b, ih, iw, c, device=device, generator=g) * case.get('scale', 1.5)
    if case['dt'] == 'f16':
        x = x.half()
    elif case['dt'] == 'split':
        hi = x.half()
        x = torch.stack([hi, (x - hi.float()).half()]).contiguous()
    f = (rand_filter() if case.get('filt') == 'rand' else asym_filter()).to(device)
    noise = None
    if case.get('noise') == 'shared':
        noise = torch.randn(oh, ow, device=device, generator=g) * 0.5
    elif case.get('noise') == 'sample':
        noise = torch.randn(b, oh, ow, device=device, generator=g) * 0.5
    bias = torch.randn(c, device=device, generator=g) * 0.3 if case.get('bias', True) else None
    kw = dict(pad0=case.get('pad0', (1, 1)), fir_gain=case.get('fir_gain', 4.0), act=case.get('act', 3), alpha=case.get('alpha', 0.2),
              act_gain=case.get('gain', 1.0), clamp=case.get('clamp', -1.0))
    return x, f, noise, bias, kw


def _c(dt, B, C, out_hw, planes, in_hw=None, **kw):
    return dict(dt=dt, B=B, C=C, out_hw=out_hw, in_hw=in_hw or (out_hw[0] + 1, out_hw[1] + 1), planes=planes, **kw)


# Tiles are 8 x 16 outputs; the 16 separable instances are input dtype x hi/lo output x noise x kFast, plus the 16-tap kernel
# for fp16, fp32 and a hi/lo input.
FIR_CASES = {
    'f16-1x1': _c('f16', 1, 64, (1, 1), 1, noise='shared', clamp=256.0, gain=SQRT2),
    'f16-1x17-so': _c('f16', 2, 128, (1, 17), 2, noise='sample', gain=SQRT2),
    'f16-7x15-clamp0.7': _c('f16', 3, 192, (7, 15), 1, clamp=0.7, scale=3.0),
    'f16-8x16-linear-so': _c('f16', 1, 64, (8, 16), 2, act=1, bias=False),
    'f16-9x17-alpha1.5': _c('f16', 5, 64, (9, 17), 1, noise='sample', alpha=1.5, clamp=256.0),
    'f16-h4-alpha-0.3-so': _c('f16', 4, 128, (8, 8), 2, noise='shared', alpha=-0.3, gain=SQRT2),
    'f16-h33': _c('f16', 2, 64, (66, 66), 1, clamp=256.0, gain=SQRT2),
    'f16-h256': _c('f16', 1, 64, (512, 512), 1, noise='shared', clamp=256.0, gain=SQRT2),
    'f16-so-alpha0-clamp0.7': _c('f16', 2, 64, (9, 17), 2, alpha=0.0, clamp=0.7, scale=3.0),
    'f16-so-alpha1-clamp0': _c('f16', 3, 64, (7, 15), 2, noise='sample', alpha=1.0, clamp=0.0),
    'f32-1x1-so': _c('f32', 1, 32, (1, 1), 2, noise='shared'),
    'f32-7x15-clamp0.7': _c('f32', 3, 96, (7, 15), 1, noise='sample', clamp=0.7, scale=3.0, gain=SQRT2),
    'f32-9x17': _c('f32', 2, 32, (9, 17), 1, gain=SQRT2),
    'f32-8x16-linear-so': _c('f32', 4, 32, (8, 16), 2, act=1),
    'f32-h33': _c('f32', 2, 96, (66, 66), 1, noise='sample', clamp=256.0, gain=SQRT2),
    'f32-encoder-pad2': _c('f32', 2, 64, (17, 17), 2, in_hw=(16, 16), pad0=(2, 2), fir_gain=1.0, act=1, bias=False),
    'f32-alpha-0.3-so': _c('f32', 5, 32, (8, 16), 2, noise='shared', alpha=-0.3),
    'f32-alpha1.5': _c('f32', 1, 64, (9, 17), 1, alpha=1.5, clamp=256.0),
    'f32-so-clamp0.7': _c('f32', 2, 32, (7, 15), 2, clamp=0.7, scale=3.0),
    'f16-crop-pad0': _c('f16', 2, 64, (9, 17), 1, in_hw=(20, 30), pad0=(0, 0), noise='shared', clamp=256.0),
    'f16-pad2': _c('f16', 2, 64, (17, 17), 1, in_hw=(16, 16), pad0=(2, 2), noise='shared'),
    'gen-f16-random-filter': _c('f16', 2, 128, (9, 17), 1, filt='rand', noise='shared', clamp=0.7, scale=3.0),
    'gen-f32-random-filter': _c('f32', 3, 32, (7, 15), 2, filt='rand', noise='sample', alpha=-0.3, gain=SQRT2),
    'split-encoder-pad2': _c('split', 2, 64, (17, 17), 2, in_hw=(16, 16), pad0=(2, 2), fir_gain=1.0, act=1, bias=False),
    'split-noise': _c('split', 3, 64, (9, 17), 2, noise='sample', clamp=256.0, gain=SQRT2),
    'variant1-f16': _c('f16', 2, 64, (9, 17), 2, noise='sample', variant=1),
    'variant1-f32': _c('f32', 2, 32, (7, 15), 1, clamp=256.0, variant=1, gain=SQRT2),
}


def _case_route(case, device='cpu'):
    x, f, noise, bias, kw = fir_inputs(case, device=device)
    return fir_route(x, f, case['planes'], kw['act'], kw['alpha'], kw['clamp'], noise, case.get('variant', 3))


def _kind(route):
    return route[0]


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the models against the oracle, planted faults, the mirrors
# ---------------------------------------------------------------------------------------------------------------------
def test_fir_model_reproduces_the_oracle():
    """fir_model's interval holds the oracle's upfirdn2d + bias_act (float64) of the golden inputs; with an fp32 input and
    no rounding steps the interval is within G_FIR of it, and the oracle's fp32 result lies inside the rounded interval."""
    import p3d_oracle as O
    from conftest import load_golden
    g = load_golden('ops')
    x = g['up_x'].astype(np.float64)                       # [2,3,9,11] -> outputs 8 x 10
    f = g['up_f4']
    b = np.array([0.3, -0.2, 0.1])
    for act, alpha, gain, clamp in ((3, 0.2, SQRT2, 0.9), (1, 0.0, 1.0, -1.0), (3, -0.3, 1.0, -1.0)):
        name = 'lrelu' if act == 3 else 'linear'
        ref = O.ops.upfirdn2d(x, f, padding=[1, 1, 1, 1], gain=4)
        ref = O.ops.bias_act(ref, b, act=name, alpha=alpha, gain=gain, clamp=None if clamp < 0 else clamp)
        xt = torch.from_numpy(x).permute(0, 2, 3, 1).float()
        m = fir_model(xt, torch.from_numpy(f), None, torch.from_numpy(b).float(), 2, (8, 10), act=act, alpha=alpha,
                      act_gain=gain, clamp=clamp, kind='sep')
        r = torch.from_numpy(ref).permute(0, 2, 3, 1)
        tol = 1e-6 * (r.abs() + 1)
        assert ((m['vlo'] <= r + tol) & (r - tol <= m['vhi'])).all()
        assert float((m['vhi'] - m['vlo']).max()) < 1e-5
        # the fp32 oracle, rounded to fp16, is one of the values the interval allows
        r32 = torch.from_numpy(O.ops.bias_act(O.ops.upfirdn2d(x.astype(np.float32), f, padding=[1, 1, 1, 1], gain=4), b.astype(np.float32),
                                              act=name, alpha=alpha, gain=gain, clamp=None if clamp < 0 else clamp)).permute(0, 2, 3, 1)
        h = rn16(r32.double())
        assert ((m['lo16'] <= h) & (h <= m['hi16'])).all()
    # fp16 input: the reference rounds the FIR output, and after the in-place noise add
    xh = torch.from_numpy(x).half().permute(0, 2, 3, 1).contiguous()
    nz = torch.from_numpy(np.linspace(-1, 1, 80).reshape(8, 10)).float()
    m = fir_model(xh, torch.from_numpy(f), nz, torch.from_numpy(b).float().half().float(), 1, (8, 10), act=3, alpha=0.2,
                  act_gain=SQRT2, clamp=256.0, kind='sep')
    y = O.ops.upfirdn2d(x.astype(np.float16).astype(np.float32), f, padding=[1, 1, 1, 1], gain=4).astype(np.float16)
    y = (y.astype(np.float32) + nz.numpy()).astype(np.float16)
    y = O.ops.bias_act(y.astype(np.float32), b.astype(np.float16).astype(np.float32), act='lrelu', clamp=256.0).astype(np.float16)
    h = torch.from_numpy(y.astype(np.float64)).permute(0, 2, 3, 1)
    assert ((m['lo16'] <= h) & (h <= m['hi16'])).all()
    assert float((m['lo16'] == m['hi16']).double().mean()) > 0.9


def _modulated_by_oracle(w, st, demodulate=True):
    """The oracle's modulated weights [B, O, I, kh, kw]: modulated_conv2d of one-hot images (each output reads one weight)."""
    import p3d_oracle as O
    b, (o, i, kh, kw) = st.shape[0], w.shape
    out = np.zeros((b, o, i, kh, kw), np.float32)
    for c in range(i):
        x = np.zeros((b, i, kh, kw), np.float32)
        x[:, c, kh // 2, kw // 2] = 1
        y = O.ops.modulated_conv2d(x, w, st, padding=kh // 2, demodulate=demodulate)       # y[p] = w[2c - p] (correlation)
        out[:, :, c] = y[:, :, ::-1, ::-1]
    return out


def test_modulation_model_reproduces_the_oracle():
    """modw_model matches the oracle's modulated_conv2d weights (golden inputs) within the relative bound."""
    from conftest import load_golden
    g = load_golden('ops')
    for w, demod, pre in ((g['mc_w3'], True, 1.0), (g['mc_w1'], False, 1 / math.sqrt(6))):
        st = g['mc_styles'] * np.float32(pre)
        ref = _modulated_by_oracle(w, st, demod).astype(np.float64)      # [B, O, I, kh, kw]
        b, o, i, kh, kw = ref.shape
        got = modw_model(torch.from_numpy(w), torch.from_numpy(g['mc_styles']), demod, pre, cin_padded=8, out_scale=1.0)
        want = torch.zeros_like(got)
        want[:, :o, :, :i] = torch.from_numpy(ref).reshape(b, o, i, kh * kw).permute(0, 1, 3, 2)
        eps = modw_eps(i, kh * kw)
        assert ((got - want).abs() <= eps * want.abs() + 1e-12).all()
        assert (got[:, o:] == 0).all() and (got[..., i:] == 0).all()


FIR_FAULTS = {  # fault: (case, least fraction of elements it must put outside the bound)
    'no_round16': ('f16-9x17-alpha1.5', 0.2),
    'pad_shift': ('f16-7x15-clamp0.7', 0.5),
    'no_mirror': ('f32-9x17', 0.5),
    'noise_sample0': ('f16-9x17-alpha1.5', 0.5),
    'bias_block': ('f16-1x17-so', 0.5),
    'max_form': ('f32-alpha1.5', 0.3),
    'round_then_clamp': ('f16-7x15-clamp0.7', 0.05),
    'lo_zero': ('f32-8x16-linear-so', 0.5),
}


def _cpu_fir_result(case):
    """What a correct kernel writes, formed on the CPU: the model's values rounded in the kernel's order, in fp32 / fp16."""
    x, f, noise, bias, kw = fir_inputs(case, device='cpu', seed=1)
    kind = _kind(_case_route(case))
    xv = (x[0].float() + x[1].float()) if x.ndim == 5 else x.float()
    v = fir_exact(xv.double(), f, kw['pad0'], case['out_hw'], kw['fir_gain']).float()
    if x.dtype == torch.float16 and x.ndim == 4:
        v = v.half().float()
    if noise is not None:
        v = v + (noise[None, :, :, None] if noise.ndim == 2 else noise[..., None])
        if x.dtype == torch.float16 and x.ndim == 4:
            v = v.half().float()
    if bias is not None:
        v = v + bias
    if kw['act'] == 3:
        v = torch.where(v > 0, v, v * f32(kw['alpha']))
    v = v * f32(kw['act_gain'])
    if kw['clamp'] >= 0:
        v = v.clamp(-f32(kw['clamp']), f32(kw['clamp']))
    hi = v.half()
    y = torch.stack([hi, (v - hi.float()).half()])
    return y, (x, f, noise, bias, kw, kind)


@pytest.mark.parametrize('fault', list(FIR_FAULTS))
def test_fir_bound_rejects_planted_faults(fault):
    """A correctly rounded result passes the model; each planted fault puts at least the stated fraction of elements outside."""
    case = FIR_CASES[FIR_FAULTS[fault][0]]
    y, (x, f, noise, bias, kw, kind) = _cpu_fir_result(case)
    planes = case['planes']
    y = y[:planes]
    bad, r, _ = fir_check_all(y, x, f, noise, bias, planes, case['out_hw'], kind, **kw)
    assert bad == 0, (bad, r)
    bad, r, _ = fir_check_all(y, x, f, noise, bias, planes, case['out_hw'], kind, fault=fault, **kw)
    frac = bad / y[0].numel()
    print(f'planted fault {fault!r}: {frac:.3f} of elements outside (worst err / tol {r:.3g})')
    assert frac >= FIR_FAULTS[fault][1], frac


MODW_FAULTS = {'tap_missing': 0.9, 'cin_off8': 0.9, 'styles_b8': 0.9}


@pytest.mark.parametrize('fault', list(MODW_FAULTS))
def test_modulation_bound_rejects_planted_faults(fault):
    """fp32 emulation of the kernel's arithmetic passes; one tap missing from sum_t w^2, cin_offset off by 8 and the styles
    of sample b + 8 each put most weights outside."""
    g = torch.Generator().manual_seed(3)
    b, o, i, k, ip, off = 12, 20, 40, 3, 64, 8
    w = torch.randn(o, i, k, k, generator=g)
    st = torch.randn(b, i, generator=g) + 1
    wf = w.reshape(o, i, k * k)
    d = ((st.square() @ wf.square().sum(-1).t()) + 1e-8).rsqrt() * 128
    v = (wf[None] * (st[:, None, :] * d[:, :, None])[..., None])          # fp32, [B, O, I, kk]
    hi = v.half()
    got = torch.zeros(2, b, 32, k * k, ip, dtype=torch.float16)
    got[0, :, :o, :, off:off + i] = hi.permute(0, 1, 3, 2)
    got[1, :, :o, :, off:off + i] = (v - hi.float()).half().permute(0, 1, 3, 2)
    got = got.reshape(2, b, 32, -1)
    eps = modw_eps(i, k * k)
    assert modw_check(got, modw_model(w, st, cin_padded=ip, cin_offset=off), eps, 2)[0] == 0
    bad, r = modw_check(got, modw_model(w, st, cin_padded=ip, cin_offset=off, fault=fault), eps, 2)
    live = b * o * i * k * k
    print(f'planted fault {fault!r}: {bad / live:.3f} of the weights outside (worst err / tol {r:.3g})')
    assert bad / live >= MODW_FAULTS[fault]


def test_fir_sweep_reaches_every_instance():
    """Through the mirror of the host's routing: the sweep's cases reach all 19 FIR kernel instances."""
    routes = {name: _case_route(case) for name, case in FIR_CASES.items()}
    assert set(routes.values()) == FIR_INSTANCES, FIR_INSTANCES - set(routes.values())
    assert routes['variant1-f16'] == ('gen', 'f16') and routes['gen-f16-random-filter'] == ('gen', 'f16')
    # the rule's corners
    x = torch.zeros(1, 4, 4, 64, dtype=torch.float16)
    f = asym_filter()
    assert fir_route(x, f, 1, 3, 0.2, 256.0)[-1] and not fir_route(x, f, 1, 3, 0.2, 0.7)[-1] and fir_route(x, f, 2, 3, 0.2, 0.7)[-1]
    assert not fir_route(x, f, 1, 3, 1.5)[-1] and not fir_route(x, f, 1, 3, -0.3)[-1] and not fir_route(x, f, 1, 1, 0.2)[-1]
    assert fir_route(x, f, 1, 3, 1.0, 0.0)[-1]
    assert fir_route(x, rand_filter(), 1) == ('gen', 'f16')


MODW_CASES = {   # B, Cout, Cin, Cin_padded, k, cin_offset, demodulate, planes
    'b1-ip8': (1, 20, 8, 8, 3, 0, True, 2),
    'b8-ip16': (8, 16, 16, 16, 3, 0, True, 2),
    'b9-ip32': (9, 33, 32, 32, 3, 0, True, 1),
    'b63-ip64-torgb': (63, 3, 64, 64, 1, 0, False, 1),
    'b64-ip128-cin100': (64, 16, 100, 128, 3, 0, True, 2),
    'b65-ip256': (65, 40, 256, 256, 3, 0, True, 1),
    'b129-ip512-1x1': (129, 17, 512, 512, 1, 0, True, 2),
    'b8-ip512-3x3': (8, 16, 512, 512, 3, 0, True, 2),
    'b4-ip1024-3x3': (4, 16, 1024, 1024, 3, 0, True, 1),
    'b2-ip2048-3x3': (2, 20, 2048, 2048, 3, 0, True, 2),
    'b4-ip2048-1x1': (4, 20, 2048, 2048, 1, 0, False, 1),
    'cin-offset-32': (4, 24, 32, 64, 3, 32, True, 1),
    'cin-offset-8': (3, 16, 48, 64, 3, 8, True, 2),
    'ip36-scalar-rows': (3, 16, 30, 36, 3, 0, True, 2),
}


def test_modulation_sweep_reaches_both_paths():
    """Through the mirror of modulate_row's predicate: the sweep runs the register fast path and the general path, including
    a launch whose 64-sample chunks take both, and 3x3 layers with ktaps > 3 tstep."""
    paths = Counter()
    for name, (b, o, i, ip, k, off, _, _) in MODW_CASES.items():
        if modulate_kernel(ip, True) == 't':
            for p in modulate_paths(b, i, ip, off, k * k):
                paths[p] += 1
    assert paths['fast'] > 0 and paths['general'] > 0
    assert modulate_paths(65, 256, 256, 0, 9) == ['general', 'fast']
    assert modulate_paths(8, 512, 512, 0, 9) == ['fast'] and modulate_paths(4, 1024, 1024, 0, 9) == ['general']
    assert modulate_paths(4, 32, 64, 32, 9) == ['general'] and modulate_paths(4, 100, 128, 0, 9) == ['general']
    assert modulate_kernel(36, True) == 'plain'


# ---------------------------------------------------------------------------------------------------------------------
# GPU: sweep
# ---------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize('name', list(FIR_CASES))
def test_fir_tail_sweep(name, monkeypatch):
    from pix2pix3d_b200 import tcconv
    case = FIR_CASES[name]
    monkeypatch.setattr(tcconv, 'FIR_VARIANT', case.get('variant', 3))
    x, f, noise, bias, kw = fir_inputs(case, seed=list(FIR_CASES).index(name))
    route = fir_route(x, f, case['planes'], kw['act'], kw['alpha'], kw['clamp'], noise)
    bad, r, zw = fir_launch_check(x, f, noise, bias, case['planes'], case['out_hw'], _kind(route), **kw)
    print(f'{name}: {route}, {bad} outside, worst err/tol {r:.3g}, {zw:.4f} of the intervals of width zero')
    assert bad == 0 and r <= 1.0


@gpu
@pytest.mark.parametrize('name', list(MODW_CASES))
@pytest.mark.parametrize('fn', ['t', 'plain'])
def test_modulation_sweep(name, fn):
    from pix2pix3d_b200 import tcconv
    b, o, i, ip, k, off, demod, planes = MODW_CASES[name]
    g = torch.Generator(device='cuda').manual_seed(i + b)
    w = torch.randn(o, i, k, k, device='cuda', generator=g)
    st = torch.randn(b, i, device='cuda', generator=g) + 1
    pre = 1.0 if demod else 1 / math.sqrt(i)
    prep = tcconv.prepare_weights(w) if fn == 't' else None
    buf, out, status = modulate_launch(w, st, demod, pre, planes, ip, off, prep)
    assert status == 0
    torch.cuda.synchronize()
    assert untouched(buf, out)
    bad, r = modw_check(out, modw_model(w, st, demod, pre, ip, 128.0, off), modw_eps(i, k * k), planes)
    kern = modulate_kernel(ip, prep is not None)
    paths = modulate_paths(b, i, ip, off, k * k) if kern == 't' else ['one CTA per row']
    print(f'{name} ({fn}): kernel {kern}, paths {paths}: {bad} outside, worst err/tol {r:.3g}')
    assert bad == 0


def _weight_plan_layers(seed=0):
    """About ten mixed layers (3x3 and 1x1, fp32 split and fp16, a cin_offset) and their WeightPlan specs."""
    from pix2pix3d_b200.training.networks_stylegan2 import SynthesisLayer, ToRGBLayer
    torch.manual_seed(seed)
    mk = [SynthesisLayer(512, 512, 512, 8), SynthesisLayer(512, 256, 512, 16, up=2), ToRGBLayer(256, 96, 512),
          SynthesisLayer(256, 128, 512, 32), SynthesisLayer(128, 64, 512, 64, up=2), ToRGBLayer(64, 32, 512),
          SynthesisLayer(32, 128, 512, 64), SynthesisLayer(128, 100, 512, 128, up=2), ToRGBLayer(100, 3, 512),
          SynthesisLayer(24, 40, 512, 128)]
    layers = [(l.cuda(), k % 5) for k, l in enumerate(mk)]
    specs = []
    for k, (l, _) in enumerate(layers):
        torgb = isinstance(l, ToRGBLayer)
        cin_p, off = (64, 32) if k == 9 else (((l.in_channels + 63) // 64) * 64, 0)
        if k == 6:
            cin_p = 32
        specs.append(dict(layer=l, demodulate=not torgb, pre_scale=float(l.weight_gain) if torgb else 1.0, planes=1 + k % 2,
                          cin_padded=cin_p, cin_offset=off))
    return layers, specs


def check_weight_plan_launch(plan, b, styles_flat, out_flat, rows=None):
    """Every layer of one p3d_modulate_weights_batch launch against the model; the 64-element gaps stay NaN."""
    _, _, _, total, shapes = plan.tables(b)
    worst, bad, written = 0.0, 0, torch.zeros(total, dtype=torch.bool, device=out_flat.device)
    s_off = 0
    for k, (sp, (off, n, shape)) in enumerate(zip(plan.specs, shapes)):
        layer = sp['layer']
        o, i, kh, kw = layer.weight.shape
        st = styles_flat[s_off:s_off + b * i].view(b, i)
        s_off += b * i
        ref = modw_model(layer.weight.float(), st, sp['demodulate'], sp['pre_scale'], sp['cin_padded'], 128.0, sp['cin_offset'])
        k_bad, r = modw_check(out_flat[off:off + n].view(shape), ref, modw_eps(i, kh * kw), sp['planes'])
        bad, worst = bad + k_bad, max(worst, r)
        written[off:off + n] = True
        if rows is not None:
            path = ','.join(sorted(set(modulate_paths(b, i, sp['cin_padded'], sp['cin_offset'], kh * kw))))
            rows.append((f'modw layer {k}', f'{o}x{i}x{kh}x{kw} Ip {sp["cin_padded"]} off {sp["cin_offset"]} planes {sp["planes"]} '
                         f'{path}', k_bad, r))
    gaps = out_flat[~written]
    assert torch.isnan(gaps).all(), 'a layer wrote into the gap after it'
    return bad, worst


@gpu
@pytest.mark.parametrize('b', [1, 4, 9, 16])
def test_modulation_batch_table_and_per_layer_launches(b):
    """A WeightPlan of ten mixed layers as one batched launch: every layer against the model, the gaps between layers NaN,
    and each layer bit for bit equal to p3d_modulate_weights_t of that layer alone (both run modulate_row)."""
    from pix2pix3d_b200 import engine, tcconv
    layers, specs = _weight_plan_layers()
    plan = engine.WeightPlan(layers, specs)
    raw, bl, n_blocks, total, shapes = plan.tables(b)
    g = torch.Generator(device='cuda').manual_seed(b)
    styles = torch.randn(sum(b * l.in_channels for l, _ in layers), device='cuda', generator=g) + 1
    buf, out = nan_buffer((total,), torch.float16)
    tcconv.modulate_weights_batch(raw, bl, n_blocks, styles, out, b)
    torch.cuda.synchronize()
    assert untouched(buf, out)
    bad, worst = check_weight_plan_launch(plan, b, styles, out)
    print(f'B {b}: {len(specs)} layers, {bad} outside, worst err/tol {worst:.3g}')
    assert bad == 0
    s_off = 0
    for sp, prep, (off, n, shape) in zip(specs, plan.prepared, shapes):
        i = sp['layer'].in_channels
        st = styles[s_off:s_off + b * i].view(b, i)
        s_off += b * i
        one = tcconv.modulate_weights(sp['layer'].weight, st, demodulate=sp['demodulate'], pre_scale=sp['pre_scale'],
                                      planes=sp['planes'], cin_padded=sp['cin_padded'], cin_offset=sp['cin_offset'], prepared=prep)
        assert torch.equal(_bits(one.reshape(-1)), _bits(out[off:off + n])), sp['layer']


@gpu
@pytest.mark.parametrize('rows,w_dim,b', [(37, 512, 1), (37, 512, 16), (101, 100, 5), (8, 100, 16), (300, 512, 7)])
def test_affine_batch(rows, w_dim, b):
    """rows not a multiple of 8, w_dim 512 (float4 path) and 100 (scalar path), arbitrary ws_index, output offsets and strides."""
    from pix2pix3d_b200 import tcconv
    g = torch.Generator(device='cuda').manual_seed(rows + w_dim + b)
    num_ws = 7
    ws = torch.randn(b, num_ws, w_dim, device='cuda', generator=g)
    weight = torch.randn(rows, w_dim, device='cuda', generator=g) / math.sqrt(w_dim)
    bias = torch.randn(rows, device='cuda', generator=g)
    stride = rows + 3
    meta = torch.stack([torch.randint(0, num_ws, (rows,), device='cuda', generator=g),
                        torch.randperm(rows, device='cuda', generator=g) + 2, torch.full((rows,), stride, device='cuda'),
                        torch.zeros(rows, dtype=torch.int64, device='cuda')], 1).int().contiguous()
    n = b * stride + 5
    buf, out = nan_buffer((n,), torch.float32)
    tcconv.affine_batch(ws, weight, bias, meta, n, out=out)
    torch.cuda.synchronize()
    assert untouched(buf, out)
    exp, tol, wr = affine_model(ws, weight, bias, meta, n)
    assert torch.isnan(out[~wr]).all()
    r = float(((out[wr].double() - exp[wr]).abs() / tol[wr]).max())
    print(f'rows {rows}, w_dim {w_dim}, B {b}: worst err/tol {r:.3g}')
    assert r <= 1.0


def _sms():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


@gpu
@pytest.mark.parametrize('case', ['c3', 'c6', 'c96', 'c96-misaligned', 'hw1', 'grid-stride'])
def test_upsample2x(case):
    """C 3 and 6 (VEC 1), 96 (VEC 4), a 16-byte-misaligned input and output (VEC 1), H = W = 1, and more items than the
    grid-stride cap of SMs x 32 blocks."""
    from pix2pix3d_b200 import tcconv
    from pix2pix3d_b200.torch_utils.ops import upfirdn2d
    b, h, w, c = {'c3': (2, 7, 5, 3), 'c6': (3, 9, 16, 6), 'c96': (2, 17, 9, 96), 'c96-misaligned': (2, 17, 9, 96),
                  'hw1': (3, 1, 1, 32), 'grid-stride': (1, 256, 256, 96)}[case]
    if case == 'grid-stride':
        assert b * h * w * c // 4 > _sms() * 32 * 256
    mis = 1 if case == 'c96-misaligned' else 0
    g = torch.Generator(device='cuda').manual_seed(c + h)
    xb, x = nan_buffer((b, h, w, c), torch.float32, misalign=mis)
    x.copy_(torch.randn(b, h, w, c, device='cuda', generator=g))
    f = upfirdn2d.setup_filter([1, 3, 3, 1]).cuda()
    buf, y = nan_buffer((b, 2 * h, 2 * w, c), torch.float32, misalign=mis)
    tcconv.upsample2x_nhwc(x, f, out=y)
    torch.cuda.synchronize()
    assert untouched(buf, y)
    ref, tol = upsample_model(x, f)
    r = float(torch.nan_to_num((y.double() - ref).abs() / (tol + 1e-300), nan=math.inf).max())
    print(f'{case}: worst err/tol {r:.3g}')
    assert r <= 1.0


@gpu
@pytest.mark.parametrize('src', [torch.float32, torch.float16])
@pytest.mark.parametrize('planes', [1, 2])
def test_layout_converters_bit_exact(src, planes):
    """NCHW -> NHWC fp16 hi/lo with HW and C not multiples of 32 and channel padding; NHWC -> NCHW of a channel window."""
    from pix2pix3d_b200 import tcconv
    g = torch.Generator(device='cuda').manual_seed(planes)
    n, c, h, w, cp = 3, 45, 5, 7, 64
    x = (torch.randn(n, c, h, w, device='cuda', generator=g) * 3).to(src)
    buf, out = nan_buffer((planes, n, h, w, cp), torch.float16)
    tcconv.to_nhwc_f16(x, c_padded=cp, planes=planes, out=out)
    torch.cuda.synchronize()
    assert untouched(buf, out)
    hi = x.half()
    lo = (x.float() - hi.float()).half()
    want = torch.zeros(2, n, h, w, cp, dtype=torch.float16, device='cuda')
    want[0, ..., :c] = hi.permute(0, 2, 3, 1)
    want[1, ..., :c] = lo.permute(0, 2, 3, 1)
    assert torch.equal(_bits(out), _bits(want[:planes]))
    xs = torch.randn(n, h, w, 70, device='cuda', generator=g)
    buf, out = nan_buffer((n, 45, h, w), torch.float32)
    tcconv.nhwc_to_nchw_f32(xs, channels=45, c_offset=13, out=out)
    torch.cuda.synchronize()
    assert untouched(buf, out)
    assert torch.equal(_bits(out), _bits(xs[..., 13:58].permute(0, 3, 1, 2).contiguous()))


@gpu
def test_misaligned_outputs_are_refused():
    """16-byte (fp16 input) or 8-byte (fp32 input) FIR stores and the modulation kernels' 16-byte stores: an output two bytes
    off is refused with P3D_BAD_ARG before anything is launched."""
    from pix2pix3d_b200 import tcconv
    f = rand_filter().cuda()
    for dt in (torch.float16, torch.float32):
        x = torch.randn(1, 9, 17, 64, device='cuda').to(dt)
        buf, y = nan_buffer((1, 1, 8, 16, 64), torch.float16, misalign=1)
        with pytest.raises(RuntimeError, match='status -2'):
            tcconv.fir_act_nhwc(x, f, None, None, 1, (8, 16), out=y)
        assert torch.isnan(buf).all()
    xs = torch.randn(2, 1, 9, 17, 64, device='cuda').half()
    buf, y = nan_buffer((1, 1, 8, 16, 64), torch.float16, misalign=1)
    with pytest.raises(RuntimeError, match='status -2'):
        tcconv.fir_act_nhwc(xs, f, None, None, 1, (8, 16), out=y)
    w = torch.randn(16, 64, 3, 3, device='cuda')
    st = torch.randn(2, 64, device='cuda')
    for prep in (None, tcconv.prepare_weights(w)):
        buf, out, status = modulate_launch(w, st, prepared=prep, misalign=1)
        assert status == -2
    torch.cuda.synchronize()
    assert torch.isnan(buf).all()


# ---------------------------------------------------------------------------------------------------------------------
# GPU: bit-for-bit invariances
# ---------------------------------------------------------------------------------------------------------------------
INVARIANCE_CASES = ['f16-9x17-alpha1.5', 'f32-7x15-clamp0.7', 'gen-f32-random-filter', 'split-noise', 'f16-so-alpha1-clamp0']


@gpu
@pytest.mark.parametrize('name', INVARIANCE_CASES)
def test_fir_samples_equal_one_sample_launches(name):
    """Every sample of a B-sample launch (per-sample noise included) equals the one-sample launch of that sample."""
    from pix2pix3d_b200 import tcconv
    case = dict(FIR_CASES[name], B=5, noise='sample')
    x, f, noise, bias, kw = fir_inputs(case, seed=9)
    planes, hw = case['planes'], case['out_hw']
    full = tcconv.fir_act_nhwc(x, f, noise, bias, planes, hw, **kw)
    for b in range(5):
        xb = x[:, b:b + 1].contiguous() if x.ndim == 5 else x[b:b + 1].contiguous()
        one = tcconv.fir_act_nhwc(xb, f, noise[b:b + 1].contiguous(), bias, planes, hw, **kw)
        assert torch.equal(_bits(one[:, 0]), _bits(full[:, b])), b


@gpu
@pytest.mark.parametrize('pad', [1, 2])
@pytest.mark.parametrize('dt', ['f16', 'f32', 'gen-f16'])
def test_fir_crops_equal_windows_of_the_full_launch(dt, pad):
    """A launch over a crop of the input (pad0 shifted, output shrunk) equals the same window of the full launch bit for bit:
    no output element's arithmetic depends on its place in the 8 x 16 tile or on the halo, so tile-edge errors show exactly."""
    from pix2pix3d_b200 import tcconv
    oh, ow = 37, 53
    case = _c(dt[-3:], 2, 64, (oh, ow), 2, in_hw=(oh + 3 - 2 * pad, ow + 3 - 2 * pad), pad0=(pad, pad), noise='shared',
              clamp=0.7, scale=3.0, filt='rand' if dt.startswith('gen') else None)
    x, f, noise, bias, kw = fir_inputs(case, seed=4)
    full = tcconv.fir_act_nhwc(x, f, noise, bias, 2, (oh, ow), **kw)
    g = torch.Generator().manual_seed(pad)
    wins = [(0, 0, 8, 16), (7, 15, 9, 17), (8, 16, 8, 16), (1, 1, 29, 51), (oh - 9, ow - 17, 9, 17), (30, 40, 7, 13)]
    wins += [tuple(int(v) for v in (torch.randint(0, oh - 1, (1,), generator=g), torch.randint(0, ow - 1, (1,), generator=g))) + (1, 1)]
    for r0, c0, h, w in wins:
        h, w = min(h, oh - r0), min(w, ow - c0)
        sr, sc = max(0, r0 - pad), max(0, c0 - pad)
        xc = x[:, sr:, sc:].contiguous()
        k = dict(kw, pad0=(sc - (c0 - pad), sr - (r0 - pad)))
        part = tcconv.fir_act_nhwc(xc, f, noise[r0:r0 + h, c0:c0 + w].contiguous(), bias, 2, (h, w), **k)
        assert torch.equal(_bits(part), _bits(full[:, :, r0:r0 + h, c0:c0 + w].contiguous())), (r0, c0, h, w)


# ---------------------------------------------------------------------------------------------------------------------
# GPU: a layer's tail against the module (the reference's rounding points)
# ---------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize('fp16', [True, False])
def test_up2_layer_tail_follows_the_module(fp16, monkeypatch):
    """One up=2 SynthesisLayer through the engine: the FIR tail of the launch's own transposed-conv output must be what the
    module prescribes -- bias `layer.bias.to(x.dtype)` (fp16-rounded in an fp16 layer), gain act_gain, clamp conv_clamp."""
    from pix2pix3d_b200 import engine, tcconv
    from pix2pix3d_b200.training.networks_stylegan2 import SynthesisLayer
    torch.manual_seed(3)
    layer = SynthesisLayer(128, 128, 512, 64, up=2, conv_clamp=256).cuda()
    with torch.no_grad():
        layer.bias.copy_(torch.randn(128) * 0.5)
        layer.noise_strength.fill_(0.3)
    split = not fp16
    seen = {}
    fir = tcconv.fir_act_nhwc

    def capture(tmp, f, noise, bias, out_planes, out_hw, **kw):
        y = fir(tmp, f, noise, bias, out_planes, out_hw, **kw)
        seen.update(tmp=tmp, y=y, kw=kw, out_planes=out_planes, out_hw=out_hw, f=f)
        return y

    monkeypatch.setattr(tcconv, 'fir_act_nhwc', capture)
    with torch.no_grad():
        x = tcconv.to_nhwc_f16(torch.randn(2, 128, 32, 32, device='cuda'), planes=2 if split else 1)
        styles = layer.affine(torch.randn(2, 512, device='cuda'))
        engine.synthesis_layer(layer, x, styles, 'const', split)
    torch.cuda.synchronize()
    tmp, y = seen['tmp'], seen['y']
    dt = torch.float32 if split else torch.float16
    assert tmp.dtype == dt and seen['out_planes'] == (2 if split else 1)
    noise = (layer.noise_const * layer.noise_strength).detach().float()
    bias = layer.bias.detach().to(dt).float()
    kind = _kind(fir_route(tmp, seen['f'], seen['out_planes'], noise=noise))
    bad, r, _ = fir_check_all(y, tmp, layer.resample_filter, noise, bias, seen['out_planes'], seen['out_hw'], kind, pad0=(1, 1),
                              fir_gain=4.0, act=3, alpha=0.2, act_gain=float(layer.act_gain), clamp=float(layer.conv_clamp))
    print(f'{"fp16" if fp16 else "fp32"} up=2 layer: {bad} of {y[0].numel()} elements outside, worst err/tol {r:.3g}')
    assert bad == 0


# ---------------------------------------------------------------------------------------------------------------------
# GPU: replays of real steps
# ---------------------------------------------------------------------------------------------------------------------
CHECKED = ('p3d_fir_act_nhwc', 'p3d_fir_act_nhwc_split', 'p3d_fir_act_nhwc_sep', 'p3d_affine_batch', 'p3d_modulate_weights_batch',
           'p3d_nchw_to_nhwc_f16', 'p3d_nhwc_to_nchw_f32', 'p3d_upsample2x_nhwc')


class _Counting:
    """Proxy of the libp3d handle: counts the accepted launches of each entry point in CHECKED."""

    def __init__(self, handle):
        self._h = handle
        self.n = Counter()

    def __getattr__(self, name):
        fn = getattr(self._h, name)
        if name not in CHECKED:
            return fn

        def call(*args):
            st = fn(*args)
            if st == 0:
                self.n[name] += 1
            return st
        return call


class _Replay:
    """Wraps the tcconv entry points of these launches (the engine calls them through the module): each launch writes into
    a NaN buffer longer than it needs and is checked against the model while its inputs are alive."""

    def __init__(self, monkeypatch):
        from pix2pix3d_b200 import _lib, engine, tcconv
        self.rows, self.kinds, self.checked = [], set(), Counter()
        self.count = _Counting(_lib.lib())
        monkeypatch.setattr(_lib, '_lib', self.count)
        fir, aff, modw = tcconv.fir_act_nhwc, tcconv.affine_batch, tcconv.modulate_weights_batch
        to16, to32, up = tcconv.to_nhwc_f16, tcconv.nhwc_to_nchw_f32, tcconv.upsample2x_nhwc

        def fir_act_nhwc(x, f, noise, bias, out_planes, out_hw, out=None, **kw):
            route = fir_route(x, f, out_planes, kw.get('act', 3), kw.get('alpha', 0.2), kw.get('clamp', -1.0), noise)
            b = x.shape[1] if x.ndim == 5 else x.shape[0]
            buf, y = nan_buffer((out_planes, b, out_hw[0], out_hw[1], x.shape[-1]), torch.float16, device=x.device)
            fir(x, f, noise, bias, out_planes, out_hw, out=y, **kw)
            torch.cuda.synchronize()
            assert untouched(buf, y)
            k = {**dict(pad0=(1, 1), fir_gain=4.0, act=3, alpha=0.2, act_gain=1.0, clamp=-1.0), **kw}
            bad, r, _ = fir_check_all(y, x, f, noise, bias, out_planes, out_hw, _kind(route), **k)
            name = 'p3d_fir_act_nhwc_sep' if route[0] == 'sep' else 'p3d_fir_act_nhwc_split' if route[0] == 'split' else 'p3d_fir_act_nhwc'
            self.checked[name] += 1
            nz = 'none' if noise is None else 'shared' if noise.ndim == 2 else 'per-sample'
            self.kinds |= {route if route[0] != 'sep' else route[:2] + ('so' if route[2] else '1p',), f'noise {nz}'}
            self.row('fir', f'{route} B {b} {out_hw[0]}x{out_hw[1]}x{x.shape[-1]} noise {nz} clamp {k["clamp"]:g}', bad, r)
            return out.copy_(y) if out is not None else y

        def affine_batch(ws, weight, bias, meta, out_numel, out=None):
            buf, o = nan_buffer((out_numel,), torch.float32, device=ws.device)
            aff(ws, weight, bias, meta, out_numel, out=o)
            torch.cuda.synchronize()
            assert untouched(buf, o)
            exp, tol, wr = affine_model(ws.float(), weight, bias, meta, out_numel)
            r = float(((o[wr].double() - exp[wr]).abs() / tol[wr]).max())
            bad = int((~((o[wr].double() - exp[wr]).abs() <= tol[wr])).sum()) + int((~torch.isnan(o[~wr])).sum())
            self.checked['p3d_affine_batch'] += 1
            self.kinds.add('affine')
            self.row('affine', f'rows {weight.shape[0]} w_dim {weight.shape[1]} B {ws.shape[0]}', bad, r)
            return out.copy_(o) if out is not None else o

        def modulate_weights_batch(descs_dev, block_layer_dev, n_blocks, styles_flat, out_flat, batch):
            plan = None
            for slot in list(engine._derived.values()):
                for v in slot.values():
                    if isinstance(v, engine.WeightPlan) and batch in v._tables and v._tables[batch][0] is descs_dev:
                        plan = v
            assert plan is not None, 'the launch maps back to a WeightPlan'
            buf, o = nan_buffer((out_flat.numel(),), torch.float16, device=out_flat.device)
            modw(descs_dev, block_layer_dev, n_blocks, styles_flat, o, batch)
            torch.cuda.synchronize()
            assert untouched(buf, o)
            rows = []
            bad, r = check_weight_plan_launch(plan, batch, styles_flat, o, rows)
            for k, (tag, what, kb, kr) in enumerate(rows):
                self.kinds.add('modw ' + what.split()[-1])
            self.checked['p3d_modulate_weights_batch'] += 1
            self.row('modw', f'{len(plan.specs)} layers B {batch} paths {sorted({w.split()[-1] for _, w, _, _ in rows})}', bad, r)
            out_flat.copy_(o)

        def to_nhwc_f16(x, c_padded=None, planes=1, out=None):
            y = to16(x, c_padded=c_padded, planes=planes, out=out)
            hi = x.half()
            lo = (x.float() - hi.float()).half()
            want = torch.zeros_like(y)
            want[0, ..., :x.shape[1]] = hi.permute(0, 2, 3, 1)
            if planes == 2:
                want[1, ..., :x.shape[1]] = lo.permute(0, 2, 3, 1)
            ok = torch.equal(_bits(y), _bits(want))
            self.checked['p3d_nchw_to_nhwc_f16'] += 1
            self.kinds.add('to_nhwc')
            self.row('to_nhwc', f'{tuple(x.shape)} {x.dtype} -> Cp {y.shape[-1]} planes {planes}', 0 if ok else 1, 0.0)
            return y

        def nhwc_to_nchw_f32(x, channels=None, c_offset=0, out=None):
            y = to32(x, channels=channels, c_offset=c_offset, out=out)
            c = channels or x.shape[-1]
            ok = torch.equal(_bits(y), _bits(x[..., c_offset:c_offset + c].permute(0, 3, 1, 2).contiguous()))
            self.checked['p3d_nhwc_to_nchw_f32'] += 1
            self.kinds.add('to_nchw')
            self.row('to_nchw', f'{tuple(x.shape)} -> C {c}', 0 if ok else 1, 0.0)
            return y

        def upsample2x_nhwc(x, f, out=None):
            y = up(x, f, out=out)
            ref, tol = upsample_model(x, f)
            r = float(((y.double() - ref).abs() / (tol + 1e-300)).max())
            self.checked['p3d_upsample2x_nhwc'] += 1
            self.row('upsample', f'{tuple(x.shape)}', int(r > 1), r)
            return y

        for name, fn in (('fir_act_nhwc', fir_act_nhwc), ('affine_batch', affine_batch), ('modulate_weights_batch', modulate_weights_batch),
                         ('to_nhwc_f16', to_nhwc_f16), ('nhwc_to_nchw_f32', nhwc_to_nchw_f32), ('upsample2x_nhwc', upsample2x_nhwc)):
            monkeypatch.setattr(tcconv, name, fn)

    def row(self, kind, what, bad, r):
        self.rows.append(f'{len(self.rows):>3} {kind:<8} {what:<70} outside {bad:>3} worst err/tol {r:.3g}')
        assert bad == 0 and r <= 1.0, self.rows[-1]


REPLAY_KINDS = {('sep', 'f16', '1p'), ('sep', 'f32', 'so'), ('split',), 'noise per-sample', 'noise shared',
                'affine', 'modw fast', 'modw general', 'to_nhwc'}


@gpu
def test_replay_of_real_synthesis_steps(monkeypatch):
    """One eager G.synthesis step each of seg2cat_512 (noise_mode 'random': per-sample noise; B = 4: the fast modulation
    path), seg2face_512 (B = 16: the general path), edge2car_128 with its label encoder (hi/lo-input 16-tap FIR and fp32
    act=1 separable FIR) and seg2cat_512 under force_fp32. Every FIR, affine and modulation launch is checked."""
    from pix2pix3d_b200 import configs
    dev = torch.device('cuda')
    rp = _Replay(monkeypatch)
    worst = {}
    for name, noise_mode, fp32 in (('seg2cat_512', 'random', False), ('seg2face_512', 'const', False), ('edge2car_128', 'const', False),
                                   ('seg2cat_512', 'const', True)):
        wl = configs.WORKLOADS[name]
        mapping = name == 'edge2car_128'
        G = configs.build_generator(name, seed=0, device=dev, with_mapping=mapping)
        c = configs.camera_labels(wl['batch'], 2, wl['preset']).to(dev)
        n0 = len(rp.rows)
        k0 = sum(rp.count.n[k] for k in CHECKED[:5])
        c0 = sum(rp.checked[k] for k in CHECKED[:5])
        with torch.no_grad():
            if mapping:
                z = torch.randn(wl['batch'], 512, device=dev, generator=torch.Generator(device=dev).manual_seed(1))
                ws = G.mapping(z, c, {'mask': configs.label_map(name, wl['batch'], seed=2).to(dev), 'pose': c})
            else:
                ws = configs.synthetic_ws(wl['batch'], G.backbone.num_ws, 1).to(dev)
            torch.manual_seed(0)
            G.synthesis(ws, c, noise_mode=noise_mode, neural_rendering_resolution=wl['nrr'], force_fp32=fp32)
        torch.cuda.synchronize()
        print(f'# {name} (batch {wl["batch"]}, noise_mode {noise_mode}, force_fp32 {fp32})')
        print('\n'.join(rp.rows[n0:]))
        launches = sum(rp.count.n[k] for k in CHECKED[:5]) - k0
        assert launches == sum(rp.checked[k] for k in CHECKED[:5]) - c0 > 0, 'every FIR, affine and modulation launch is checked'
        for row in rp.rows[n0:]:
            kind = row.split()[1]
            worst[kind] = max(worst.get(kind, 0.0), float(row.split()[-1]))
        del G
    print('worst err/tol per kind: ' + ', '.join(f'{k} {v:.3g}' for k, v in sorted(worst.items())))
    missing = REPLAY_KINDS - rp.kinds
    assert not missing, (missing, rp.kinds)
