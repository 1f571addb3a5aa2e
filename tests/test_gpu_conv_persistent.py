"""The persistent conv kernel on grids where every CTA walks many work units, against a float64 model of each launch.

conv_gemm_kernel runs min(units, SMs) CTAs. CTA c takes the work units c, c + grid, ...; its two consumer warpgroups take
alternate units, the stage ring runs on across unit boundaries, and a consumer reloads its per-channel epilogue constants
(scale, bias, ToRGB weights) only when its next unit has another sample or channel tile. `reference()` models one launch in
float64 from its tcconv arguments, and `worst_ratio()` holds every output element to

    |got - ref| <= eps_out * |ref| + eps_acc * S

where S is the same model on absolute values. The sweep builds its shapes from the device's SM count, so that unit counts land
on the edges of the schedule (one unit, SMs - 1, SMs, SMs + 1, ...), and the replays check every launch of real synthesis and
training steps.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from test_gpu_tcconv import test_merged_transposed_conv_phases_equal_separate_launches as _merged_equal_separate

gpu = pytest.mark.gpu

U16 = 2.0 ** -11               # fp16 unit roundoff
U32 = 2.0 ** -24               # fp32 unit roundoff
EPS16 = 3 * U16                # fp16 outputs: one rounding plus one ulp of slack
TINY16 = 2.0 ** -24            # fp16 subnormal spacing (absolute floor of an fp16 rounding)
S_MARGIN = 1.05                # S is summed in bf16 (positive terms only): a few 2^-8 relative at most
SQRT2 = math.sqrt(2.0)


def eps_acc(n_slices):
    """Accumulation bound relative to S. Per k16 slice the tensor core adds 16 exact fp16 products into the fp32 accumulator
    and truncates; allow 2 ulps (2^-22) of the running magnitude (<= S) per slice, and 16 more for the fp32 epilogue
    (scale fma, noise, gain, residual, split-K partial sums). The sweep and the replays print the worst err / tol they see:
    on an H100 SXM (132 SMs, 400 W) it was 0.115 for fp32 outputs (an fp32 ToRGB tail of the seg2cat_512 replay), so the bound
    sits about 8x above the worst case seen, and 0.33 for fp16 outputs, where the rounding term (1 of the 3 half-ulps
    allowed) dominates. It still rejects a dropped hi*lo pass at 31x (test_bound_rejects_planted_faults)."""
    return (n_slices + 16) * 2.0 ** -22


# ---------------------------------------------------------------------------------------------------------------------
# float64 model of one launch
# ---------------------------------------------------------------------------------------------------------------------
def _gather(x, rows, cols):
    """x [n,H,W,C] -> [n,len(rows),len(cols),C] float64, zero where a row or column lies outside the image."""
    h, w = x.shape[1], x.shape[2]
    ok = ((rows >= 0) & (rows < h))[:, None] & ((cols >= 0) & (cols < w))[None, :]
    g = x[:, rows.clamp(0, h - 1)][:, :, cols.clamp(0, w - 1)].double()
    return g * ok[None, :, :, None].double()


def _mm(xg, wt):
    """xg [n,gh,gw,C] times wt [1 or n, O, C]^T -> [n,gh,gw,O] (shared or per-sample weights)."""
    n, gh, gw, c = xg.shape
    if wt.shape[0] == 1:
        return (xg.reshape(-1, c) @ wt[0].transpose(0, 1)).reshape(n, gh, gw, -1)
    return torch.bmm(xg.reshape(n, -1, c), wt.transpose(1, 2)).reshape(n, gh, gw, -1)


def _accumulate(x, w, cout, taps, grid_hw, split, stride, b0, b1, mut):
    """Accumulators [n,gh,gw,cout] of samples b0..b1 in float64, and S (the same sums over absolute values).

    A split launch executes hi*hi + hi*lo + lo*hi; in float64 that is (hi+lo)(hi+lo) - lo*lo, both exact here, with the
    lo*lo product (< 2^-22 of S) taken in bf16."""
    c = x.shape[-1]
    dev = x.device
    ys = torch.arange(grid_hw[0], device=dev) * stride
    xs = torch.arange(grid_hw[1], device=dev) * stride
    wsel = w[:, b0:b1] if w.shape[1] > 1 else w[:, :1]
    acc = s = 0
    for t, (dy, dx, kb) in enumerate(taps):
        xg = [_gather(x[p, b0:b1], ys + dy, xs + dx) for p in range(2 if split else 1)]
        wg = [wsel[p, :, :cout, kb * c:(kb + 1) * c].double() for p in range(2 if split else 1)]
        if mut.get('drop_kstep') == t:            # the tap's last 64-channel k-step never ran
            for p in range(len(xg)):
                xg[p] = xg[p].clone()
                xg[p][..., c - 64:] = 0
        if split:
            full = _mm(xg[0] + xg[1], wg[0] + wg[1])
            acc = acc + full - _mm(xg[1].bfloat16(), wg[1].bfloat16()).double()
            if mut.get('drop_hilo'):
                acc = acc - _mm(xg[0], wg[1])
            s = s + _mm((xg[0].abs() + xg[1].abs()).bfloat16(), (wg[0].abs() + wg[1].abs()).bfloat16()).double()
        else:
            acc = acc + _mm(xg[0], wg[0])
            s = s + _mm(xg[0].abs().bfloat16(), wg[0].abs().bfloat16()).double()
    return acc, s * S_MARGIN


def _upsample2d(img, f):
    """upfirdn2d.upsample2d(img, f): zero insertion, padding (2, 1), the 4x4 FIR times 4, in float64. NHWC in and out."""
    n, h, w, c = img.shape
    z = img.new_zeros(n, c, 2 * h, 2 * w, dtype=torch.float64)
    z[:, :, ::2, ::2] = img.permute(0, 3, 1, 2).double()
    z = F.pad(z, [2, 1, 2, 1])
    k = (f.double().flip([0, 1]) * 4).expand(c, 1, 4, 4)
    return F.conv2d(z, k, groups=c).permute(0, 2, 3, 1)


def _nhwc(t, nchw):
    return t.permute(0, 2, 3, 1) if nchw else t


def reference(snap, x, w, cout, taps, grid_hw, out, split=False, out_lo=None, out_mode=0, out_map=(1, 0, 1, 0), y_coff=0,
              bias=None, noise=None, dscale=None, act=1, alpha=0.2, gain=1.0, clamp=-1.0, acc_scale=1.0 / 128, split_k=True,
              up_prev=None, up_filter=None, round16=False, out_nchw=False, stride=1, residual=None, rgb=None, phases=None,
              mut=None):
    """What one launch must leave in its outputs, a chunk of samples at a time.

    Takes the arguments of tcconv.conv_gemm (or, with `phases` = [(taps, grid_hw, out_map)], of a merged launch), `snap` =
    {'out', 'out_lo', 'rgb'}: the output tensors as they were before the launch, and `out` etc. as the launch left them (the
    fused ToRGB reads the launch's own fp16 outputs where it wrote them). Yields (b0, b1, {name: (expected, tol, written)}),
    all NHWC over the whole output tensor of those samples; elements outside `written` must equal the snapshot bit for bit."""
    mut = mut or {}
    if phases is None:
        phases = [(taps, grid_hw, out_map)]
    if mut.get('phase_ox') is not None:         # one phase written one column to the right
        k = mut['phase_ox']
        t_, g_, (sy, oy, sx, ox) = phases[k]
        phases = list(phases)
        phases[k] = (t_, g_, (sy, oy, sx, ox + 1))
    b_all, c = x.shape[1], x.shape[-1]
    passes = 3 if split else 1
    px_max = max(g[0] * g[1] for _, g, _ in phases)
    step = max(1, (1 << 18) // px_max)
    for b0 in range(0, b_all, step):
        b1 = min(b_all, b0 + step)
        o_snap = _nhwc(snap['out'][b0:b1], out_nchw)
        o_got = _nhwc(out[b0:b1], out_nchw)
        exp = o_snap.double().clone()
        tol = torch.zeros_like(exp)
        wr = torch.zeros(exp.shape, dtype=torch.bool, device=exp.device)
        res = {}
        if rgb is not None:
            rout = _nhwc(snap['rgb'][b0:b1], True)
            r_exp = torch.zeros(rout.shape, dtype=torch.float64, device=rout.device)
            r_tol = torch.zeros_like(r_exp)
        for taps_p, (gh, gw), (sy, oy, sx, ox) in phases:
            acc, s_acc = _accumulate(x, w, cout, taps_p, (gh, gw), split, stride, b0, b1, mut)
            ea = eps_acc(passes * len(taps_p) * c // 16)
            ys = torch.arange(gh, device=x.device) * sy + oy
            xs = torch.arange(gw, device=x.device) * sx + ox
            sc = torch.full((1, 1, 1, cout), acc_scale, dtype=torch.float64, device=x.device)
            if dscale is not None:
                sc = sc * dscale[b0:b1, :cout].double()[:, None, None, :]
            v, s = acc * sc, s_acc * sc.abs()
            if bias is not None:
                v, s = v + bias[:cout].double(), s + bias[:cout].double().abs()
            if noise is not None:
                nz = noise.double()[None] if noise.ndim == 2 else noise[b0:b1].double()
                nz = nz[:, ys][:, :, xs][..., None]
                v, s = v + nz, s + nz.abs()
            if act == 3:
                v = torch.where(v > 0, v, v * alpha)
                s = s * max(1.0, abs(alpha))
            v, s = v * gain, s * abs(gain)
            if clamp >= 0:
                v = v.clamp(-clamp, clamp)
            if residual is not None:
                r = residual[b0:b1, :, :, :cout].double()
                v, s = v + r, s + r.abs()
            e_acc = ea * s
            idx = (slice(None), ys[:, None], xs[None, :], slice(y_coff, y_coff + cout))
            if up_prev is not None:
                up = _upsample2d(up_prev[b0:b1], up_filter)[:, ys][:, :, xs]
                s_up = _upsample2d(up_prev[b0:b1].abs(), up_filter.abs())[:, ys][:, :, xs]
                val = up + v
                t = e_acc + 8 * U32 * s_up + 2 * U32 * val.abs()
                if round16:
                    t = t + EPS16 * v.abs() + TINY16
            elif out_mode == 0:
                val, t = v, e_acc * (1 + U16) + EPS16 * v.abs() + TINY16
            elif out_mode == 1:
                val, t = v, e_acc + 2.0 ** -21 * v.abs() + TINY16
            elif out_mode == 2:
                val, t = v, e_acc + 2 * U32 * v.abs()
            else:
                val = exp[idx] + v
                t = e_acc + 2 * U32 * val.abs()
            if rgb is None or not rgb.get('skip_x', False):
                exp[idx], tol[idx], wr[idx] = val, t, True
            if rgb is not None:
                rc = snap['rgb'].shape[1]
                rw = rgb['w'][b0:b1, :rc, :cout].double()
                if rgb.get('skip_x', False):
                    # the launch kept its fp16 outputs to itself: bound a rounding flip of each by one ulp
                    yq = v.half().double()
                    dq = e_acc * (1 + U16) + 2 * U16 * v.abs() + TINY16
                else:
                    yq = o_got[idx].double()
                    dq = torch.zeros_like(yq)
                dot = torch.einsum('nhwk,nck->nhwc', yq, rw)
                s_dot = torch.einsum('nhwk,nck->nhwc', yq.abs(), rw.abs())
                d_tol = cout * U32 * s_dot + torch.einsum('nhwk,nck->nhwc', dq, rw.abs())
                r_s = rgb.get('acc_scale', 1.0 / 128)
                rb = rgb['bias'][:rc].double() if rgb.get('bias') is not None else torch.zeros(rc, dtype=torch.float64,
                                                                                                   device=x.device)
                xr = dot * r_s + rb
                xt = d_tol * abs(r_s) + 2 * U32 * ((dot * r_s).abs() + rb.abs())
                if rgb.get('clamp', -1.0) >= 0:
                    xr = xr.clamp(-rgb['clamp'], rgb['clamp'])
                xt = xt + EPS16 * xr.abs() + TINY16
                up = _upsample2d(rgb['prev'][b0:b1], rgb['filter'])[:, ys][:, :, xs]
                s_up = _upsample2d(rgb['prev'][b0:b1].abs(), rgb['filter'].abs())[:, ys][:, :, xs]
                ridx = (slice(None), ys[:, None], xs[None, :], slice(None))
                r_exp[ridx] = up + xr
                r_tol[ridx] = xt + 8 * U32 * s_up + 2 * U32 * (up + xr).abs()
        res['out'] = (exp, tol, wr)
        if rgb is not None:
            res['rgb'] = (r_exp, r_tol, torch.ones(r_exp.shape, dtype=torch.bool, device=r_exp.device))
        yield b0, b1, res


def _bits(t):
    return t.view(torch.int16 if t.element_size() == 2 else torch.int32)


def _ratio(got, snaps, exp, tol, wr):
    """max over written elements of |got - exp| / tol; inf if an element outside `written` changed (bitwise, NaN-safe)."""
    for g, sn in snaps:
        if not torch.equal(_bits(torch.where(wr, sn, g)), _bits(sn)):
            return math.inf
    err = (got.double() - exp).abs()
    r = torch.where(wr & (err != 0), err / tol, torch.zeros_like(err))
    return float(torch.nan_to_num(r, nan=math.inf).max()) if r.numel() else 0.0


def worst_ratio(snap, args, kw, phases=None, mut=None):
    """Worst err / tol of a finished launch over all its outputs."""
    x, w, cout, taps, grid_hw, out = args
    nchw, out_lo, rgb = kw.get('out_nchw', False), kw.get('out_lo'), kw.get('rgb')
    worst = 0.0
    with torch.no_grad():
        for b0, b1, res in reference(snap, *args, phases=phases, mut=mut, **kw):
            exp, tol, wr = res['out']
            got = _nhwc(out[b0:b1], nchw)
            snaps = [(got, _nhwc(snap['out'][b0:b1], nchw))]
            if kw.get('out_mode', 0) == 1:
                snaps.append((out_lo[b0:b1], snap['out_lo'][b0:b1]))
                got = got.double() + out_lo[b0:b1].double()
            worst = max(worst, _ratio(got, snaps, exp, tol, wr))
            if rgb is not None:
                exp, tol, wr = res['rgb']
                g = _nhwc(rgb['out'][b0:b1], True)
                worst = max(worst, _ratio(g, [(g, _nhwc(snap['rgb'][b0:b1], True))], exp, tol, wr))
    return worst


def snapshot(out, kw):
    return {'out': out.clone(), 'out_lo': None if kw.get('out_lo') is None else kw['out_lo'].clone(),
            'rgb': None if kw.get('rgb') is None else kw['rgb']['out'].clone()}


# ---------------------------------------------------------------------------------------------------------------------
# launching and the host rules
# ---------------------------------------------------------------------------------------------------------------------
def _sms():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def _tiling(args, kw, phases=None):
    """tools/time_conv.py's mirror of conv_launch's tiling, for the launch these arguments describe."""
    from pix2pix3d_b200 import tcconv
    from tools.time_conv import tiling
    x, w, cout, taps, grid_hw, out = args
    if phases is None:
        return tiling([tcconv._conv_args(*args, **kw)], _sms())
    return tiling([tcconv._conv_args(x, w, cout, t, g, out, out_map=m, **kw) for t, g, m in phases], _sms())


def _launch(args, kw, fn='conv_gemm'):
    """Run one conv launch, then check it against the model; returns (worst err / tol, tiling)."""
    from pix2pix3d_b200 import tcconv
    snap = snapshot(args[5], kw)
    if fn == 'conv_gemm':
        tcconv.conv_gemm(*args, **kw)
    else:
        assert tcconv.conv_gemm_try(*args, **kw), 'this launch shape qualifies for the fused ToRGB'
    torch.cuda.synchronize()
    r = worst_ratio(snap, args, kw)
    assert r <= 1.0, f'worst err / tol = {r:.3g}'
    return r, _tiling(args, kw)


def _inputs(b, c, cout, hw, k=3, split=False, per_sample=True, seed=0, in_hw=None, scale=1.0):
    """x [planes,B,H,W,C] fp16, per-sample (or shared) modulated weights, per-sample dscale and noise, bias."""
    from pix2pix3d_b200 import tcconv
    g = torch.Generator(device='cuda').manual_seed(seed)
    h, w = in_hw or hw
    planes = 2 if split else 1
    x = tcconv.to_nhwc_f16(torch.randn(b, c, h, w, device='cuda', generator=g) * scale, planes=planes)
    wt = torch.randn(cout, c, k, k, device='cuda', generator=g)
    st = torch.randn(b if per_sample else 1, c, device='cuda', generator=g) + 1
    wk = tcconv.modulate_weights(wt, st, demodulate=True, planes=planes)
    return dict(x=x, w=wk, dscale=torch.rand(b, cout, device='cuda', generator=g) + 0.5,
                noise=torch.randn(b, hw[0], hw[1], device='cuda', generator=g) * 0.5,
                bias=torch.randn(cout, device='cuda', generator=g) * 0.2)


def _grid_for(tiles):
    """A computed grid of exactly `tiles` 128-pixel tiles (16 rows x 8*tiles columns tile without padding)."""
    return (16, 8 * tiles)


def _rgb_args(b, cout, hw, skip_x, seed=0, rows=16, ci=3):
    from pix2pix3d_b200 import tcconv
    from pix2pix3d_b200.torch_utils.ops import upfirdn2d
    g = torch.Generator(device='cuda').manual_seed(seed + 100)
    wr = torch.randn(ci, cout, 1, 1, device='cuda', generator=g)
    st = torch.randn(b, cout, device='cuda', generator=g) + 1
    wk = tcconv.modulate_weights(wr, st, demodulate=False, pre_scale=1.0 / math.sqrt(cout), cin_padded=cout)   # [1,B,16,cout]
    assert wk.shape[2] == rows
    return dict(w=wk[0], bias=torch.randn(ci, device='cuda', generator=g), filter=upfirdn2d.setup_filter([1, 3, 3, 1]).cuda(),
                prev=torch.randn(b, hw[0] // 2, hw[1] // 2, ci, device='cuda', generator=g),
                out=torch.full((b, ci, hw[0], hw[1]), float('nan'), device='cuda'), clamp=256.0, skip_x=skip_x)


# ---------------------------------------------------------------------------------------------------------------------
# the model itself, against torch's convolutions (CPU)
# ---------------------------------------------------------------------------------------------------------------------
def test_model_matches_torch_convolutions():
    """The float64 model reproduces F.conv2d (padded, strided, per-sample weights), the transposed convolution as four
    phases, upfirdn2d.upsample2d, and the epilogue formula, on the CPU."""
    from pix2pix3d_b200 import tcconv
    from pix2pix3d_b200.torch_utils.ops import upfirdn2d
    torch.manual_seed(0)
    b, c, cout, h, w = 2, 64, 24, 9, 7

    def planes(t):                          # NCHW float64 -> [2,B,H,W,C] fp16 hi/lo, and the values of hi + lo and of lo
        hi = t.half()
        lo = (t - hi.double()).half()
        return torch.stack([hi, lo]).permute(0, 1, 3, 4, 2).contiguous(), hi.double() + lo.double(), lo.double()

    def conv3(fn, x, xlo, w, wlo, **kw):    # what three passes compute: (hi + lo)(hi + lo) - lo*lo
        return fn(x, w, **kw) - fn(xlo, wlo, **kw)

    x, xv, xl = planes(torch.randn(b, c, h, w, dtype=torch.float64))
    wt = torch.randn(b, cout, c, 3, 3, dtype=torch.float64) / 24
    wk, wv, wl = planes(wt.reshape(b * cout, c, 3, 3))
    wk = wk.reshape(2, b, cout, 9 * c).contiguous()          # [planes, B, O, (ky, kx, c)]: K-major, tap-major
    wv, wl = wv.reshape(b, cout, c, 3, 3), wl.reshape(b, cout, c, 3, 3)
    snap = {'out': torch.zeros(b, h, w, cout), 'out_lo': None, 'rgb': None}
    kw = dict(out_mode=2, split=True, acc_scale=1.0, act=3, alpha=-0.3, gain=-0.7, clamp=1.5,
              bias=torch.randn(cout), noise=torch.randn(b, h, w), dscale=torch.rand(b, cout) + 0.5)
    (_, _, res), = reference(snap, x, wk, cout, tcconv.TAPS_3X3, (h, w), snap['out'], **kw)
    ref = torch.cat([conv3(F.conv2d, xv[i:i + 1], xl[i:i + 1], wv[i], wl[i], padding=1) for i in range(b)])
    ref = ref * kw['dscale'].double()[:, :, None, None] + kw['bias'].double()[None, :, None, None] + kw['noise'].double()[:, None]
    ref = (torch.where(ref > 0, ref, -0.3 * ref) * -0.7).clamp(-1.5, 1.5).permute(0, 2, 3, 1)
    exp, tol, wr = res['out']
    assert wr.all() and torch.allclose(exp, ref, rtol=1e-9, atol=1e-9)
    assert 0.05 < float((ref.abs() < 1.5).double().mean()) < 0.95          # both sides of the clamp are exercised
    assert (tol > 0).all() and float(tol.max()) < 1e-3
    # strided 'valid' taps
    xs, xsv, xsl = planes(torch.randn(b, c, 2 * h + 1, 2 * w + 1, dtype=torch.float64))
    taps = [(ky, kx, ky * 3 + kx) for ky in range(3) for kx in range(3)]
    snap = {'out': torch.zeros(b, h, w, cout), 'out_lo': None, 'rgb': None}
    (_, _, res), = reference(snap, xs, wk, cout, taps, (h, w), snap['out'], out_mode=2, split=True, acc_scale=1.0, stride=2)
    ref = torch.cat([conv3(F.conv2d, xsv[i:i + 1], xsl[i:i + 1], wv[i], wl[i], stride=2) for i in range(b)]).permute(0, 2, 3, 1)
    assert torch.allclose(res['out'][0], ref, rtol=1e-9, atol=1e-9)
    # the transposed convolution as its four phases, one shared weight tensor
    w1 = wk[:, :1].contiguous()
    phases = [(tcconv.tconv_phase_taps(py, px), (h + 1 - py, w + 1 - px), (2, py, 2, px)) for py in (0, 1) for px in (0, 1)]
    snap = {'out': torch.full((b, 2 * h + 1, 2 * w + 1, 32), float('nan')), 'out_lo': None, 'rgb': None}
    (_, _, res), = reference(snap, x, w1, cout, None, None, snap['out'], out_mode=2, split=True, acc_scale=1.0, phases=phases)
    ref = conv3(F.conv_transpose2d, xv, xl, wv[0].transpose(0, 1), wl[0].transpose(0, 1), stride=2).permute(0, 2, 3, 1)
    exp, tol, wr = res['out']
    assert wr[..., :cout].all() and not wr[..., cout:].any()
    assert torch.allclose(exp[..., :cout], ref, rtol=1e-9, atol=1e-9)
    # upsample2d
    img = torch.randn(2, 5, 6, 3, dtype=torch.float64)
    f = upfirdn2d.setup_filter([1, 3, 3, 1])
    want = upfirdn2d.upsample2d(img.permute(0, 3, 1, 2).float(), f).double().permute(0, 2, 3, 1)
    assert torch.allclose(_upsample2d(img, f), want, rtol=1e-5, atol=1e-5)


# ---------------------------------------------------------------------------------------------------------------------
# the comparison is sharp enough
# ---------------------------------------------------------------------------------------------------------------------
@gpu
def test_bound_rejects_planted_faults():
    """The same comparison that passes the kernel rejects each of these faults planted in the model: the last k-step of one
    tap dropped, two samples' dscale rows swapped, noise one pixel off, two samples' ToRGB weights swapped, a split
    launch's hi*lo pass dropped, one phase of a merged launch one column off."""
    from pix2pix3d_b200 import tcconv
    sms = _sms()

    def swap01(t):
        t = t.clone()
        t[[0, 1]] = t[[1, 0]]
        return t

    def rejects(snap, args, kw, phases=None, mut=None):
        r = worst_ratio(snap, args, kw, phases=phases, mut=mut)
        return r > 1.0, r

    hw = _grid_for(4)
    d = _inputs(sms + 1, 128, 64, hw)
    out = torch.full((sms + 1, hw[0], hw[1], 64), float('nan'), device='cuda')
    kw = dict(out_mode=2, bias=d['bias'], noise=d['noise'], dscale=d['dscale'], act=3, alpha=0.2, gain=SQRT2)
    args = (d['x'], d['w'], 64, tcconv.TAPS_3X3, hw, out)
    snap = snapshot(out, kw)
    tcconv.conv_gemm(*args, **kw)
    torch.cuda.synchronize()
    assert worst_ratio(snap, args, kw) <= 1.0
    faults = {'k-step dropped': (kw, dict(drop_kstep=4)),
              'dscale rows swapped': (dict(kw, dscale=swap01(d['dscale'])), None),
              'noise one pixel off': (dict(kw, noise=d['noise'].roll(1, dims=-1)), None)}
    seen = {}
    for name, (kw_m, mut) in faults.items():
        seen[name] = rejects(snap, args, kw_m, mut=mut)
    # fused ToRGB with per-sample weights
    hw = _grid_for(2)
    d = _inputs(sms + 1, 64, 64, hw, seed=1)
    y = torch.full((sms + 1, hw[0], hw[1], 64), float('nan'), device='cuda', dtype=torch.float16)
    rgb = _rgb_args(sms + 1, 64, hw, skip_x=False)
    kw = dict(out_mode=0, bias=d['bias'], noise=d['noise'], dscale=d['dscale'], act=3, alpha=0.2, gain=SQRT2, clamp=256.0, rgb=rgb,
              split_k=False)
    args = (d['x'], d['w'], 64, tcconv.TAPS_3X3, hw, y)
    snap = snapshot(y, kw)
    assert tcconv.conv_gemm_try(*args, **kw)
    torch.cuda.synchronize()
    assert worst_ratio(snap, args, kw) <= 1.0
    seen['ToRGB weights swapped'] = rejects(snap, args, dict(kw, rgb=dict(rgb, w=swap01(rgb['w']))))
    # split (three-pass) launch
    hw = _grid_for(2)
    d = _inputs(sms + 1, 64, 64, hw, k=1, split=True, per_sample=False, seed=2)
    out = torch.full((sms + 1, hw[0], hw[1], 64), float('nan'), device='cuda')
    kw = dict(out_mode=2, split=True, bias=d['bias'], act=1, gain=1.0)
    args = (d['x'], d['w'], 64, tcconv.TAPS_1X1, hw, out)
    snap = snapshot(out, kw)
    tcconv.conv_gemm(*args, **kw)
    torch.cuda.synchronize()
    assert worst_ratio(snap, args, kw) <= 1.0
    seen['hi*lo pass dropped'] = rejects(snap, args, kw, mut=dict(drop_hilo=True))
    # merged transposed launch; phase 1 = (py 0, px 1), whose columns 2x + 1 stay inside the output one column further right
    h, w = 7, 5
    d = _inputs(4, 64, 48, (h, w), per_sample=False, seed=3)
    out = torch.full((4, 2 * h + 1, 2 * w + 1, 48), float('nan'), device='cuda', dtype=torch.float16)
    phases = [(tcconv.tconv_phase_taps(py, px), (h + 1 - py, w + 1 - px), (2, py, 2, px)) for py in (0, 1) for px in (0, 1)]
    kw = dict(out_mode=0)
    args = (d['x'], d['w'], 48, None, None, out)
    snap = snapshot(out, kw)
    tcconv.conv_transpose3x3_s2(d['x'], d['w'], 48, out)
    torch.cuda.synchronize()
    assert worst_ratio(snap, args, kw, phases=phases) <= 1.0
    seen['phase one column off'] = rejects(snap, args, kw, phases=phases, mut=dict(phase_ox=1))
    for name, (rej, r) in seen.items():
        print(f'planted fault {name!r}: worst err / tol = {r:.3g} -> {"rejected" if rej else "ACCEPTED"}')
    assert all(rej for rej, _ in seen.values()), {k: v[1] for k, v in seen.items()}


# ---------------------------------------------------------------------------------------------------------------------
# schedule edges
# ---------------------------------------------------------------------------------------------------------------------
UNIT_COUNTS = {'1': lambda s: 1, 'sms-1': lambda s: s - 1, 'sms': lambda s: s, 'sms+1': lambda s: s + 1,
               '2sms-1': lambda s: 2 * s - 1, '2sms': lambda s: 2 * s, '2sms+1': lambda s: 2 * s + 1, '3sms+2': lambda s: 3 * s + 2}


@gpu
@pytest.mark.parametrize('form', ['3x3-fp16', '1x1-fp32'])
@pytest.mark.parametrize('count', list(UNIT_COUNTS))
def test_unit_counts_around_the_sm_count(count, form):
    """One 128-pixel tile per sample, so units = B: every tail of the strided walk (the last CTA with one unit, consumer 2
    idle or not, an odd unit count per CTA). Per-sample weights, dscale and noise: each consumer's next unit has another
    sample. 3x3 at Cin 64 is 9 k-steps per unit (not a multiple of the 5/6-stage ring); 1x1 is one, so the ring spans
    several units."""
    from pix2pix3d_b200 import tcconv
    sms = _sms()
    n = UNIT_COUNTS[count](sms)
    k, dt, mode = (3, torch.float16, 0) if form == '3x3-fp16' else (1, torch.float32, 2)
    hw = _grid_for(1)
    d = _inputs(n, 64, 64, hw, k=k, seed=n)
    out = torch.full((n, hw[0], hw[1], 64), float('nan'), device='cuda', dtype=dt)
    kw = dict(out_mode=mode, bias=d['bias'], noise=d['noise'], dscale=d['dscale'], act=3, alpha=0.2, gain=SQRT2, split_k=False)
    r, t = _launch((d['x'], d['w'], 64, tcconv.TAPS_3X3 if k == 3 else tcconv.TAPS_1X1, hw, out), kw)
    assert t['units'] == n and t['splits'] == 1 and t['ksteps'] == [k * k]
    print(f'{count} ({n} units on {sms} SMs), {form}: worst err / tol {r:.3g}')


@gpu
@pytest.mark.parametrize('split_k', [False, True])
def test_long_k_loops_216_steps(split_k):
    """3x3 at Cin 512, three passes: 216 k-steps per unit, more units than SMs (or, with split-K on, what the host picks)."""
    from pix2pix3d_b200 import tcconv
    sms = _sms()
    b = sms + 1 if not split_k else 2
    hw = _grid_for(1)
    d = _inputs(b, 512, 128, hw, split=True, seed=7)
    hi = torch.full((b, hw[0], hw[1], 128), float('nan'), device='cuda', dtype=torch.float16)
    lo = torch.full_like(hi, float('nan'))
    kw = dict(out_mode=1, out_lo=lo, split=True, bias=d['bias'], noise=d['noise'], dscale=d['dscale'], act=3, alpha=0.2,
              gain=SQRT2, split_k=split_k)
    r, t = _launch((d['x'], d['w'], 128, tcconv.TAPS_3X3, hw, hi), kw)
    assert t['ksteps'] == [216]
    if split_k:
        assert t['splits'] > 1
    else:
        assert t['units'] == b and t['splits'] == 1
    print(f'216 k-steps, split-K {t["splits"]}, {t["units"]} units on {sms} SMs: worst err / tol {r:.3g}')


# (tiles_m, tiles_n, B): a consumer's consecutive units are 2 * SMs apart in the unit order
# u = (b * tiles_n + tile_n) * tiles_m + tile_m
RELOAD_CASES = {
    'same-sample-and-tile': (lambda s: 4 * s, 64, 2),      # u -> u + 2 SMs keeps b and tile_n (reload skipped), then b changes
    'sample-changes': (lambda s: 2 * s, 64, 3),            # tiles_m * tiles_n = 2 SMs: only b changes
    'channel-tile-changes': (lambda s: 2 * s, 256, 2),     # tiles_m = 2 SMs, two channel tiles: only tile_n changes, then both
}


@gpu
@pytest.mark.parametrize('case', list(RELOAD_CASES))
def test_epilogue_constants_reload(case):
    """Per-sample dscale, noise and conv weights where a consumer's next unit keeps its sample and channel tile, changes only
    the sample, or changes only the channel tile: a stale s_scale / s_bias shows as another sample's demodulation."""
    from pix2pix3d_b200 import tcconv
    sms = _sms()
    tiles_fn, cout, b = RELOAD_CASES[case]
    hw = _grid_for(tiles_fn(sms))
    d = _inputs(b, 64, cout, hw, seed=11)
    for dt, mode in ((torch.float16, 0), (torch.float32, 2)):
        out = torch.full((b, hw[0], hw[1], cout), float('nan'), device='cuda', dtype=dt)
        kw = dict(out_mode=mode, bias=d['bias'], noise=d['noise'], dscale=d['dscale'], act=3, alpha=0.2, gain=SQRT2, clamp=4.0,
                  split_k=False)
        r, t = _launch((d['x'], d['w'], cout, tcconv.TAPS_3X3, hw, out), kw)
        assert t['tiles'] == tiles_fn(sms) * (cout // 128 if cout > 128 else 1)
        assert t['units'] == t['tiles'] * b
        print(f'{case}, {dt}: {t["units"]} units on {sms} SMs: worst err / tol {r:.3g}')


@gpu
@pytest.mark.parametrize('case', ['same-sample-and-tile', 'sample-changes'])
@pytest.mark.parametrize('skip_x', [False, True])
def test_fused_torgb_weights_reload(case, skip_x):
    """The fused ToRGB keeps each sample's modulated 1x1 weights in s_rgbw, reloaded on the same rule as the scale and bias."""
    from pix2pix3d_b200 import tcconv
    sms = _sms()
    tiles_fn, _, b = RELOAD_CASES[case]
    hw = _grid_for(tiles_fn(sms))
    d = _inputs(b, 64, 64, hw, seed=12)
    y = torch.full((b, hw[0], hw[1], 64), float('nan'), device='cuda', dtype=torch.float16)
    kw = dict(out_mode=0, bias=d['bias'], noise=d['noise'], dscale=d['dscale'], act=3, alpha=0.2, gain=SQRT2, clamp=256.0,
              rgb=_rgb_args(b, 64, hw, skip_x=skip_x))
    r, t = _launch((d['x'], d['w'], 64, tcconv.TAPS_3X3, hw, y), kw, fn='try')
    assert t['units'] == tiles_fn(sms) * b
    if skip_x:
        assert torch.isnan(y).all()
    print(f'ToRGB {case}, skip_x {skip_x}: {t["units"]} units on {sms} SMs: worst err / tol {r:.3g}')


ACTS = {'linear': (1, 0.0), 'lrelu-0.2': (3, 0.2), 'lrelu-1.5': (3, 1.5), 'lrelu-neg0.3': (3, -0.3)}


@gpu
@pytest.mark.parametrize('clamp', [-1.0, 1.0])
@pytest.mark.parametrize('act', list(ACTS))
@pytest.mark.parametrize('cout', [24, 48, 96, 256])
def test_all_kernel_instances(cout, act, clamp):
    """The 18 instances: channel tile 32 / 64 / 128 (Cout 24, 48, 96 and two tiles of 256) x linear, leaky-relu in max form
    (0 <= alpha <= 1) and in select form (alpha 1.5, -0.3) x clamp on / off, with gains sqrt(2) (folded), 0 and -0.7 (applied
    after the activation), at more units than SMs."""
    from pix2pix3d_b200 import tcconv
    sms = _sms()
    a, alpha = ACTS[act]
    gain = (SQRT2, 0.0, -0.7)[(list(ACTS).index(act) + [24, 48, 96, 256].index(cout)) % 3]
    hw = _grid_for(1)
    b = sms + 1
    d = _inputs(b, 64, cout, hw, seed=cout)
    out = torch.full((b, hw[0], hw[1], cout), float('nan'), device='cuda')
    kw = dict(out_mode=2, bias=d['bias'], noise=d['noise'], dscale=d['dscale'], act=a, alpha=alpha, gain=gain, clamp=clamp,
              split_k=False)
    r, t = _launch((d['x'], d['w'], cout, tcconv.TAPS_3X3, hw, out), kw)
    assert t['BN'] == {24: 32, 48: 64, 96: 128, 256: 128}[cout] and t['units'] == b * (2 if cout == 256 else 1)
    print(f'Cout {cout}, {act}, clamp {clamp}, gain {gain:.3g}: worst err / tol {r:.3g}')


@gpu
@pytest.mark.parametrize('y_coff', [0, 8, 16])
@pytest.mark.parametrize('out_mode', [0, 1, 2, 3])
def test_output_modes_offsets_and_sentinels(out_mode, y_coff):
    """Cout 80 inside a 112-channel tensor at offset 0, 8 or 16: the third 32-channel chunk ends at channel 80 (scalar path),
    and an offset of 8 makes the fp16 chunks scalar while fp32 chunks stay vector. Outputs prefilled with NaN (random for
    the += mode) must keep every element outside [y_coff, y_coff + 80) bit for bit."""
    from pix2pix3d_b200 import tcconv
    sms = _sms()
    cout, cs = 80, 112
    hw = _grid_for(1)
    b = 2 * sms + 1
    d = _inputs(b, 64, cout, hw, seed=20 + out_mode)
    dt = torch.float16 if out_mode <= 1 else torch.float32
    if out_mode == 3:
        out = torch.randn(b, hw[0], hw[1], cs, device='cuda')
    else:
        out = torch.full((b, hw[0], hw[1], cs), float('nan'), device='cuda', dtype=dt)
    kw = dict(out_mode=out_mode, y_coff=y_coff, bias=d['bias'], noise=d['noise'], dscale=d['dscale'], act=3, alpha=0.2, gain=SQRT2,
              clamp=2.0, split_k=False)
    if out_mode == 1:
        kw['out_lo'] = torch.full_like(out, float('nan'))
    r, t = _launch((d['x'], d['w'], cout, tcconv.TAPS_3X3, hw, out), kw)
    assert t['units'] == b
    print(f'out_mode {out_mode}, y_coff {y_coff}: worst err / tol {r:.3g}')


@gpu
def test_merged_phases_split_k_between_one_and_two_waves():
    """A merged transposed convolution whose split-K puts the unit count between SMs and 2 SMs: some CTAs run two units, in
    different phases and k-ranges."""
    from pix2pix3d_b200 import tcconv
    sms = _sms()
    c, cout, h, w = 512, 512, 4, 4
    phases = [(tcconv.tconv_phase_taps(py, px), (h + 1 - py, w + 1 - px), (2, py, 2, px)) for py in (0, 1) for px in (0, 1)]
    pick = None
    for b in range(1, 17):
        xs = torch.empty(2, b, h, w, c, device='cuda', dtype=torch.float16)
        ws = torch.empty(2, 1, cout, 9 * c, device='cuda', dtype=torch.float16)
        o = torch.empty(b, 2 * h + 1, 2 * w + 1, cout, device='cuda')
        t = _tiling((xs, ws, cout, None, None, o), dict(out_mode=2, split=True), phases=phases)
        if sms < t['units'] < 2 * sms and t['splits'] > 1:
            pick = b
            break
    assert pick is not None, 'no batch puts this layer between one and two waves'
    d = _inputs(pick, c, cout, (h, w), split=True, per_sample=False, seed=30)
    out = torch.full((pick, 2 * h + 1, 2 * w + 1, cout), float('nan'), device='cuda')
    snap = snapshot(out, {})
    tcconv.conv_transpose3x3_s2(d['x'], d['w'], cout, out, split=True)
    torch.cuda.synchronize()
    r = worst_ratio(snap, (d['x'], d['w'], cout, None, None, out), dict(out_mode=2, split=True), phases=phases)
    assert r <= 1.0, r
    print(f'merged split-K, B {pick}: {t["units"]} units ({t["splits"]} splits) on {sms} SMs: worst err / tol {r:.3g}')


@gpu
@pytest.mark.parametrize('cout,cstride,out_mode', [(34, 40, 2), (38, 40, 2), (64, 64, 2), (64, 64, 1)])
def test_strided_conv_with_residual(cout, cstride, out_mode):
    """down=2 3x3 'valid' convolution plus the resnet skip, at more units than SMs. Cout 34 and 38 make the residual rows
    16-byte misaligned (Cout * 4 bytes apart): those chunks take the scalar path, Cout 64 the vector path."""
    from pix2pix3d_b200 import tcconv
    sms = _sms()
    gh, gw = 8, 16
    b = sms + 1
    d = _inputs(b, 64, cout, (gh, gw), split=True, per_sample=False, seed=40 + cout, in_hw=(2 * gh + 1, 2 * gw + 1))
    res = torch.randn(b, gh, gw, cout, device='cuda')
    dt = torch.float16 if out_mode == 1 else torch.float32
    out = torch.full((b, gh, gw, cstride), float('nan'), device='cuda', dtype=dt)
    kw = dict(out_mode=out_mode, split=True, bias=d['bias'], act=3, alpha=0.2, gain=1.0, stride=2, residual=res)
    if out_mode == 1:
        kw['out_lo'] = torch.full_like(out, float('nan'))
    taps = [(ky, kx, ky * 3 + kx) for ky in range(3) for kx in range(3)]
    r, t = _launch((d['x'], d['w'], cout, taps, (gh, gw), out), kw)
    assert t['units'] == b and t['splits'] == 1
    print(f'stride 2 + residual, Cout {cout}: worst err / tol {r:.3g}')


# ---------------------------------------------------------------------------------------------------------------------
# schedule invariance
# ---------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize('form', ['fp16', 'fp32', 'rgb'])
def test_samples_do_not_depend_on_the_schedule(form):
    """A unit's reduction order does not depend on the CTA or consumer that runs it: sample b of a B = 16 launch (per-sample
    weights, dscale and noise; more units than SMs) equals, bit for bit, the B = 1 launch of that sample's slices."""
    from pix2pix3d_b200 import tcconv
    sms = _sms()
    b = 16
    hw = _grid_for(sms // 8 + 1)
    d = _inputs(b, 64, 64, hw, seed=50)
    dt = torch.float32 if form == 'fp32' else torch.float16
    rgb = _rgb_args(b, 64, hw, skip_x=False) if form == 'rgb' else None

    def run(sl):
        n = sl.stop - sl.start
        out = torch.full((n, hw[0], hw[1], 64), float('nan'), device='cuda', dtype=dt)
        kw = dict(out_mode=2 if form == 'fp32' else 0, bias=d['bias'], noise=d['noise'][sl].contiguous(),
                  dscale=d['dscale'][sl].contiguous(), act=3, alpha=0.2, gain=SQRT2, clamp=256.0, split_k=False)
        args = (d['x'][:, sl].contiguous(), d['w'][:, sl].contiguous(), 64, tcconv.TAPS_3X3, hw, out)
        if rgb is not None:
            kw['rgb'] = dict(rgb, w=rgb['w'][sl].contiguous(), prev=rgb['prev'][sl].contiguous(),
                             out=torch.full_like(rgb['out'][sl], float('nan')))
            assert tcconv.conv_gemm_try(*args, **kw)
            return out, kw['rgb']['out'], _tiling(args, kw)
        tcconv.conv_gemm(*args, **kw)
        return out, None, _tiling(args, kw)

    big, big_rgb, t = run(slice(0, b))
    assert t['units'] > sms
    for i in range(b):
        one, one_rgb, t1 = run(slice(i, i + 1))
        assert t1['units'] < sms
        assert torch.equal(one[0], big[i]), i
        if rgb is not None:
            assert torch.equal(one_rgb[0], big_rgb[i]), i


@gpu
def test_one_cta_and_many_waves_give_the_same_tile():
    """A launch of 3 SMs + 2 one-tile units against one-unit launches (one CTA) of the same samples."""
    from pix2pix3d_b200 import tcconv
    sms = _sms()
    n = 3 * sms + 2
    hw = _grid_for(1)
    d = _inputs(n, 64, 64, hw, seed=51)
    kw = dict(out_mode=2, bias=d['bias'], act=3, alpha=0.2, gain=SQRT2, split_k=False)
    big = torch.empty(n, hw[0], hw[1], 64, device='cuda')
    tcconv.conv_gemm(d['x'], d['w'], 64, tcconv.TAPS_3X3, hw, big, noise=d['noise'], dscale=d['dscale'], **kw)
    for i in (0, 1, sms - 1, sms, 2 * sms + 1, n - 1):
        one = torch.empty(1, hw[0], hw[1], 64, device='cuda')
        args = (d['x'][:, i:i + 1].contiguous(), d['w'][:, i:i + 1].contiguous(), 64, tcconv.TAPS_3X3, hw, one)
        tcconv.conv_gemm(*args, noise=d['noise'][i:i + 1].contiguous(), dscale=d['dscale'][i:i + 1].contiguous(), **kw)
        assert _tiling(args, kw)['units'] == 1
        assert torch.equal(one[0], big[i]), i


# ---------------------------------------------------------------------------------------------------------------------
# replay of real steps: every conv launch checked against the model while its inputs are alive
# ---------------------------------------------------------------------------------------------------------------------
class _Replay:
    """Wraps tcconv.conv_gemm, conv_gemm_try and conv_transpose3x3_s2 (the engine, the encoder and native_conv call them
    through the module) and the library handle (to count the launches it accepts)."""

    def __init__(self, monkeypatch):
        from pix2pix3d_b200 import _lib, tcconv
        from tools.time_conv import _Recorder
        self.sms = _sms()
        self.rows, self.kinds = [], set()
        self.rec = _Recorder(_lib.lib())
        monkeypatch.setattr(_lib, '_lib', self.rec)
        monkeypatch.setattr(tcconv, 'MERGE_PHASES', True)
        gemm, gemm_try, tconv = tcconv.conv_gemm, tcconv.conv_gemm_try, tcconv.conv_transpose3x3_s2

        def conv_gemm(x, w, cout, taps, grid_hw, out, split=False, **kw):
            snap = snapshot(out, kw)
            gemm(x, w, cout, taps, grid_hw, out, split=split, **kw)
            self.check(snap, (x, w, cout, taps, grid_hw, out), dict(kw, split=split))
            return out

        def conv_gemm_try(x, w, cout, taps, grid_hw, out, split=False, **kw):
            snap = snapshot(out, kw)
            ok = gemm_try(x, w, cout, taps, grid_hw, out, split=split, **kw)
            if ok:
                self.check(snap, (x, w, cout, taps, grid_hw, out), dict(kw, split=split))
            return ok

        def conv_transpose3x3_s2(x, w, cout, out, split=False, acc_scale=1.0 / tcconv.WEIGHT_SCALE):
            snap = snapshot(out, {})
            tconv(x, w, cout, out, split=split, acc_scale=acc_scale)
            _, _, h, wd, _ = x.shape
            phases = [(tcconv.tconv_phase_taps(py, px), (h + 1 - py, wd + 1 - px), (2, py, 2, px)) for py in (0, 1) for px in (0, 1)]
            kw = dict(out_mode=2 if out.dtype == torch.float32 else 0, split=split, acc_scale=acc_scale)
            self.check(snap, (x, w, cout, None, None, out), kw, phases)
            return out

        monkeypatch.setattr(tcconv, 'conv_gemm', conv_gemm)
        monkeypatch.setattr(tcconv, 'conv_gemm_try', conv_gemm_try)
        monkeypatch.setattr(tcconv, 'conv_transpose3x3_s2', conv_transpose3x3_s2)

    def check(self, snap, args, kw, phases=None):
        torch.cuda.synchronize()
        r = worst_ratio(snap, args, kw, phases=phases)
        t = _tiling(args, kw, phases)
        x, w, cout, taps, grid_hw, out = args
        kinds = {k for k, on in (('split-K', t['splits'] > 1), ('merged', phases is not None), ('3-pass', kw.get('split')),
                                 ('ToRGB tail', kw.get('up_prev') is not None), ('rgb-fused', kw.get('rgb') is not None),
                                 ('residual', kw.get('residual') is not None), ('stride-2', kw.get('stride', 1) == 2),
                                 ('fp16+clamp', kw.get('out_mode', 0) == 0 and kw.get('clamp', -1.0) >= 0)) if on}
        self.kinds |= kinds
        grid = '+'.join(f'{g[0]}x{g[1]}' for _, g, _ in phases) if phases else f'{grid_hw[0]}x{grid_hw[1]}'
        taps_n = sum(len(p[0]) for p in phases) if phases else len(taps)
        self.rows.append(f'{len(self.rows):>3} B {x.shape[1]:>2} {grid:>17} Cin {x.shape[-1]:>3} Cout {cout:>3} taps {taps_n} '
                         f'mode {kw.get("out_mode", 0)} units {t["units"]:>6} = {t["units"] / self.sms:6.2f} SMs split-K '
                         f'{t["splits"]:>2} {",".join(sorted(kinds)):<32} worst err/tol {r:.3g}')
        assert r <= 1.0, self.rows[-1]

    def launches(self):
        return len(self.rec.calls)


REPLAY_KINDS = {'split-K', 'merged', '3-pass', 'ToRGB tail', 'rgb-fused', 'residual', 'fp16+clamp'}


@gpu
def test_replay_of_real_synthesis_steps(monkeypatch):
    """One eager G.synthesis step of each full-size workload (and the label encoder of edge2car_128's mapping), every conv
    launch checked against the model. Prints the launch table."""
    from pix2pix3d_b200 import configs
    dev = torch.device('cuda')
    rp = _Replay(monkeypatch)
    for name in ('seg2cat_512', 'seg2face_512', 'edge2car_128'):
        wl = configs.WORKLOADS[name]
        mapping = name == 'edge2car_128'
        G = configs.build_generator(name, seed=0, device=dev, with_mapping=mapping)
        c = configs.camera_labels(wl['batch'], 2, wl['preset']).to(dev)
        n0, k0 = len(rp.rows), rp.launches()
        with torch.no_grad():
            if mapping:
                z = torch.randn(wl['batch'], 512, device=dev, generator=torch.Generator(device=dev).manual_seed(1))
                ws = G.mapping(z, c, {'mask': configs.label_map(name, wl['batch'], seed=2).to(dev), 'pose': c})
            else:
                ws = configs.synthetic_ws(wl['batch'], G.backbone.num_ws, 1).to(dev)
            torch.manual_seed(0)
            G.synthesis(ws, c, noise_mode='const', neural_rendering_resolution=wl['nrr'])
        torch.cuda.synchronize()
        print(f'# {name} (batch {wl["batch"]}), {rp.sms} SMs')
        print('\n'.join(rp.rows[n0:]))
        assert len(rp.rows) - n0 == rp.launches() - k0 > 0, 'every conv launch goes through the checked wrappers'
        del G
    missing = REPLAY_KINDS - rp.kinds
    assert not missing, missing


@gpu
def test_replay_of_a_training_step(monkeypatch):
    """The tiny-model training step of test_gpu_synthesis: native_conv's forward (three passes), the transposed convolution
    and the stride-2 input gradient, every launch checked against the model."""
    import pix2pix3d_b200.training.triplane_cond as tc
    from make_golden import SYNTH_CASES, build_generator
    from conftest import load_golden
    from pix2pix3d_b200.training.dual_discriminator import DualDiscriminator
    from test_gpu_synthesis import _replayed
    case = SYNTH_CASES['seg_tiny']
    g = load_golden('synthesis_seg_tiny')
    dev = torch.device('cuda')
    rp = _Replay(monkeypatch)
    G = build_generator(tc, case).to(dev).train().requires_grad_(True)
    torch.manual_seed(5)
    D = DualDiscriminator(c_dim=25, img_resolution=128, img_channels=3, channel_base=1024, channel_max=16,
                          num_fp16_res=0, conv_clamp=None).to(dev).train().requires_grad_(True)
    ws = torch.from_numpy(g['ws']).to(dev).requires_grad_(True)
    c = torch.from_numpy(g['c']).to(dev)
    out = _replayed(lambda: G.synthesis(ws, c, noise_mode='const', neural_rendering_resolution=case['nrr'], force_fp32=True), g, dev)
    logits = D({'image': out['image'], 'image_raw': out['image_raw']}, c)
    loss = torch.nn.functional.softplus(-logits).mean()
    torch.autograd.grad(loss, [ws] + [p for p in G.parameters() if p.requires_grad], allow_unused=True)
    torch.cuda.synchronize()
    print(f'# training step, {rp.sms} SMs')
    print('\n'.join(rp.rows))
    assert len(rp.rows) == rp.launches() > 0
    missing = {'3-pass', 'merged', 'stride-2'} - rp.kinds
    assert not missing, missing


# ---------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize('b,c,cout,hw,split', [
    # ~2900 work units (4 phases x 2 channel tiles x 4 samples): each CTA crosses phase, channel-tile and sample boundaries
    (4, 256, 256, (96, 96), False),
])
def test_merged_phases_many_units_per_cta(b, c, cout, hw, split, monkeypatch):
    _merged_equal_separate(b, c, cout, hw, split, monkeypatch)
