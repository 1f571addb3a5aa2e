"""The fused renderer's backward (p3d_render_bwd, render_bwd_kernel in render_fused_bwd.cu) against a float64 model of each
launch, element by element.

The model restates one launch from the launch's own fp32 inputs (channels-last planes, rays, sorted depths, the effective
decoder parameters, the upstream gradients) in midpoint-radius float64 arithmetic (`MR`): every quantity the kernel forms is
carried as a float64 midpoint, the value in exact arithmetic, and a radius that bounds how far the kernel's fp32 value may lie
from it. Every fp32 operation adds its own rounding (u = 2^-24 of the result, gamma(n) u for a chain of n; the library expf /
log1pf add 2 and 1 ulp) and carries its inputs' radii through its derivative; monotone steps (exp, softplus, sigmoid) take the
image of the input interval. Exact zeros stay exact: zero-length intervals make exactly zero weights. Where an input interval
straddles one of the kernel's branch points (the softplus switch at 20 of the decoder and of the march, the depth gate, the
weight sum's zero) the radius covers both branches. The model follows the kernel's structure and rounding points:

    coordinates and taps      sample_taps / make_taps in fp32, exactly (the tap weights carry no radius)
    features                  tap_fetch4 (a product and three FMAs per plane), ((f0 + f1) + f2) * fl32(1/3)
    decoder, sweep 1          32-FMA hidden chains from b1, 64-FMA output chains from b2; sigma and G . c per sample
    march backward            warp_march_bwd: T as a product in any association, the weight sums, the depth gate, the
                              exclusive suffix sum; dL/dsigma_j = (gsm[j-1] + gsm[j]) / 2, coef_j = (w[j-1] + w[j]) / 2
    decoder, sweep 2          the output recomputed as b2 + (o_lane0 + o_lane1) (32-FMA chains), the sigmoid derivative
                              1.002 s (1 - s) at that value; dL/dh (two 16-FMA chains, their sum, one FMA), dL/dpre, dL/dx
                              (32-FMA chains, the lane pair's sum, the sum over the nets)
    plane gradients           dL/dx * fl32(1/3) times each non-zero tap weight, added by atomics in any order: gamma(n + 1)
                              of the texel's sum of |terms| for its n contributions
    parameter gradients       sequential per CTA over all the samples of its tiles, then a fixed-order sum over the CTAs:
                              the chain length comes from a mirror of the launch's grid (`bwd_grid`)

Every output element must satisfy |got - mid| <= rad + FLOOR. The model's midpoints are first shown equal to float64 autograd
of the staged chain (grid_sample -> decoder module -> the march) on CPU; planted faults show that the bound sees each one.
"""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from test_gpu_train_kernels import FLOOR, PLANE_AXES, U, F0001, F1002, F1E10, nan_buf, taps, untouched

gpu = pytest.mark.gpu

TINY = 2.0 ** -149             # the absolute error of an fp32 result in the subnormal range
THIRD = float(np.float32(1.0 / 3.0))
FP32 = dict(third=THIRD, c1002=F1002, c0001=F0001, eps=F1E10)                 # the kernel's fp32 constants
EXACT = dict(third=1.0 / 3.0, c1002=1 + 2 * 0.001, c0001=0.001, eps=1e-10)   # the float64 modules' constants
E_EXP, E_LOG1P = 4 * U, 2 * U  # expf 2 ulp, log1pf 1 ulp (an ulp is at most 2u of the value)
REL_SP = E_EXP + E_LOG1P       # log1pf(expf(x)): expf's error passes through log1p with a factor below 1
REL_SIG = E_EXP + 2 * U        # 1 / (1 + expf(-x)): expf, the add, the divide
DEC_PARAMS = 64 * 32 + 64 + 33 * 64 + 33


def _ceil(a, b):
    return -(-a // b)


def gam(n):
    """gamma(n) = n u / (1 - n u) for an int, an array or a tensor of chain lengths."""
    return n * U / (1 - n * U)


# ---------------------------------------------------------------------------------------------------------------------
# midpoint-radius float64 arithmetic
# ---------------------------------------------------------------------------------------------------------------------
class MR:
    """An fp32 quantity of the kernel: it lies in [m - r, m + r] (float64 tensors)."""
    __slots__ = ('m', 'r')

    def __init__(self, m, r=None):
        self.m = m
        self.r = torch.zeros_like(m) if r is None else r

    def mag(self):
        return self.m.abs() + self.r

    def __getitem__(self, i):
        return MR(self.m[i], self.r[i])


def _rnd(m, r, n=1):
    """n fp32 roundings of a result known to lie in [m - r, m + r]; an exact zero stays exact."""
    return MR(m, r + gam(n) * (m.abs() + r) + n * TINY * ((m != 0) | (r != 0)))


def add(a, b, n=1):
    return _rnd(a.m + b.m, a.r + b.r, n)


def sub(a, b, n=1):
    return _rnd(a.m - b.m, a.r + b.r, n)


def mul(a, b, n=1):
    return _rnd(a.m * b.m, a.m.abs() * b.r + a.r * b.m.abs() + a.r * b.r, n)


def scale(a, c, n=1):
    """a times an exact constant c (n = 0: a power of two)."""
    return _rnd(a.m * c, a.r * abs(c), n) if n else MR(a.m * c, a.r * abs(c))


def div(a, b, den_min=0.0):
    """a / b; den_min: a known lower bound of |b| (tighter than |b.m| - b.r where the interval is wide)."""
    den = torch.clamp(b.m.abs() - b.r, min=den_min)
    with np.errstate(all='ignore'):
        q = a.m / b.m
        r = torch.where(den > 0, (a.r + q.abs() * b.r) / den, torch.full_like(q, math.inf))
    return _rnd(q, r)


def clip(a, lo=-math.inf, hi=math.inf):
    """a known to lie in [lo, hi] as well: the intersection (the midpoint, the exact value, lies inside both)."""
    return MR(a.m, torch.maximum(a.m - torch.clamp(a.m - a.r, min=lo), torch.clamp(a.m + a.r, max=hi) - a.m).clamp_min(0))


def hull(sel, a, b):
    """(midpoint, radius) of a where `sel`, of b elsewhere."""
    m = torch.where(sel, a.m, b.m)
    r = torch.where(sel, a.r, b.r)
    return m, r


def either(sel, unsure, a, b):
    """Where `sel` the kernel takes branch a, elsewhere b, and where `unsure` it may take either: the midpoint follows `sel`
    (the branch exact arithmetic takes) and the radius covers both."""
    m, r = hull(sel, a, b)
    other_m, other_r = hull(sel, b, a)
    r = torch.where(unsure, torch.maximum(r, (other_m - m).abs() + other_r), r)
    return MR(m, r)


def mono(a, f, rel, exact_at_zero=False):
    """f(a) for an increasing, positive f whose fp32 evaluation carries a relative error `rel`: the image of the interval."""
    lo, hi = a.m - a.r, a.m + a.r
    mid = f(a.m)
    r = torch.maximum(mid - f(lo) * (1 - rel), f(hi) * (1 + rel) - mid) + TINY
    if exact_at_zero:                                  # expf(0) = 1 exactly
        r = torch.where((a.m == 0) & (a.r == 0), torch.zeros_like(r), r)
    return MR(mid, r)


def _sp(x):
    return torch.where(x > 20, x, torch.log1p(torch.exp(torch.clamp(x, max=20))))


def _sgm(x):
    return torch.sigmoid(x)


def switch20(a, f_lo, rel_lo, f_hi, zero_below=None):
    """x > 20 ? f_hi(x) : f_lo(x) for increasing, positive f_lo, f_hi (f_lo carries a relative error rel_lo): the
    softplus / sigmoid switch of the decoder and of the march. Where [lo, hi] straddles 20, the hull of both branches.
    zero_below: where the whole interval lies below it, the kernel's result is exactly 0 (expf underflows to 0)."""
    lo, hi = a.m - a.r, a.m + a.r
    inf = torch.full_like(lo, math.inf)
    can_lo, can_hi = lo <= 20, hi > 20
    L = torch.minimum(torch.where(can_lo, f_lo(lo) * (1 - rel_lo), inf), torch.where(can_hi, f_hi(torch.clamp(lo, min=20)), inf))
    H = torch.maximum(torch.where(can_lo, f_lo(torch.clamp(hi, max=20)) * (1 + rel_lo), -inf), torch.where(can_hi, f_hi(hi), -inf))
    mid = torch.where(a.m > 20, f_hi(a.m), f_lo(a.m))
    r = torch.maximum(mid - L, H - mid).clamp_min(0) + TINY
    if zero_below is not None:
        under = hi < zero_below
        mid, r = torch.where(under, torch.zeros_like(mid), mid), torch.where(under, torch.zeros_like(r), r)
    return MR(mid, r)


EXP_ZERO = -110.0              # expf(x) = 0 exactly below (e^-110 is far below half the smallest subnormal)


def dotw(x, w, n, bias=None):
    """sum_i x_i w_ij (+ bias_j) with exact weights w [n_in, n_out] as fp32 chains of n roundings."""
    aw = w.abs()
    m = x.m @ w
    tot = x.mag() @ aw
    if bias is not None:
        m = m + bias
        tot = tot + bias.abs()
    return MR(m, x.r @ aw + gam(n) * tot + n * TINY)


# ---------------------------------------------------------------------------------------------------------------------
# a mirror of the launch's grid (make_rb_layout / p3d_render_bwd)
# ---------------------------------------------------------------------------------------------------------------------
DEC_SMEM_FLOATS = 64 * 32 + 64 * 36 + 64 + 36        # sizeof(DecSmemW) / 4 = 4452
H100_SMEM_PER_SM, H100_SMEM_RESERVED = 228 * 1024, 1024


def rb_layout_floats(S, n_nets):
    RT = 128 // S
    return n_nets * DEC_SMEM_FLOATS + 128 * 36 + 7 * 128 + _ceil(RT * 32 * n_nets, 4) * 4 + 2 * 64 * 66 + 2 * 64 * 36


def bwd_grid(n_rays, S, n_nets, sms, smem_per_sm=H100_SMEM_PER_SM, reserved=H100_SMEM_RESERVED):
    """(rays per tile, tiles, CTAs per SM, CTAs) of p3d_render_bwd: occupancy of the layout's shared memory, at most 2."""
    RT = 128 // S
    tiles = _ceil(n_rays, RT)
    per_sm = max(1, min(2, smem_per_sm // (rb_layout_floats(S, n_nets) * 4 + reserved)))
    return dict(RT=RT, tiles=tiles, per_sm=per_sm, ctas=min(tiles, sms * per_sm))


def param_chain(n_rays, S, grid):
    """Longest fp32 chain of a parameter gradient: the samples of the busiest CTA over all its tiles (sequential FMAs across
    tiles and halves) plus the fixed-order sum over the CTAs (decoder_mlp_reduce_kernel)."""
    RT, tiles, ctas = grid['RT'], grid['tiles'], grid['ctas']
    per_tile = np.minimum(RT, n_rays - np.arange(tiles) * RT) * S
    per_cta = np.zeros(ctas, np.int64)
    np.add.at(per_cta, np.arange(tiles) % ctas, per_tile)
    return int(per_cta.max()) + ctas


def device_smem():
    p = torch.cuda.get_device_properties(0)
    return (getattr(p, 'shared_memory_per_multiprocessor', H100_SMEM_PER_SM),
            getattr(p, 'reserved_shared_memory_per_block', H100_SMEM_RESERVED))


# ---------------------------------------------------------------------------------------------------------------------
# the model
# ---------------------------------------------------------------------------------------------------------------------
FAULTS = ('drop_o11', 'no_third', 'no_1002', 'wb_no_sumG', 'no_wsum', 'no_depth', 'drop_last_ray', 'straddle_G',
          'first_image_planes', 'coef_wj')


def sample_points(o, d, ds, cs):
    """sample_taps' fp32 coordinates: cs * (o + dv * d), every operation rounded (numpy float32)."""
    f = np.float32
    return [f(cs) * (o[:, None, a] + ds * d[:, None, a]) for a in range(3)]


def _march_bwd(z, sig, dot, sumG, gd, gws, rng, white_back, c, fault):
    """warp_march_bwd for rays [N,S] -> (dL/dsigma_j, colour coef_j) per sample, as MR [N,S]."""
    N, S = z.shape
    K = _ceil(S - 1, 32)
    zero = torch.zeros_like(z)
    Z = lambda t: MR(t)                                                    # noqa: E731
    delta = sub(Z(z[:, 1:]), Z(z[:, :-1]))
    delta = MR(delta.m, torch.where(delta.m == 0, torch.zeros_like(delta.r), delta.r))   # equal depths: exactly zero
    x = sub(scale(add(sig[:, :-1], sig[:, 1:]), 0.5, 0), MR(torch.ones_like(delta.m)))
    sp = switch20(x, _sp, REL_SP, lambda v: v, EXP_ZERO)
    pd = mul(sp, delta)
    e = mono(MR(-pd.m, pd.r), torch.exp, E_EXP, exact_at_zero=True)
    one = MR(torch.ones_like(e.m))
    alpha = clip(sub(one, e), 0.0, 1.0)
    t = clip(add(sub(one, alpha), MR(torch.full_like(e.m, c['eps']))), c['eps'])                 # fl(0 + eps) = eps
    # T_i = prod_{k<i} t_k in any association (the lanes' products and the 5-level scan): at most i + 6 roundings, applied to
    # the products of the factors' interval ends (an opaque interval's t is known only to within [eps, a few u])
    excl = lambda v: torch.cat([torch.ones_like(v[:, :1]), torch.cumprod(v, 1)[:, :-1]], 1)   # noqa: E731
    idx = torch.arange(S - 1, dtype=z.dtype, device=z.device)[None]
    tm = excl(t.m)
    t_hi = excl(t.m + t.r) * (1 + gam(idx + 6))
    t_lo = excl(torch.clamp(t.m - t.r, min=c['eps'])) * (1 - gam(idx + 6))
    T = MR(tm, torch.maximum(t_hi - tm, tm - t_lo).clamp_min(0) + (idx + 6) * TINY)
    w = mul(alpha, T)
    dmid = scale(add(Z(z[:, :-1]), Z(z[:, 1:])), 0.5, 0)
    sw = MR(w.m.sum(1), w.r.sum(1) + gam(K + 5) * w.mag().sum(1))
    wd = MR(w.m * dmid.m, w.m.abs() * dmid.r + w.r * dmid.mag())
    swd = MR(wd.m.sum(1), wd.r.sum(1) + gam(K + 6) * wd.mag().sum(1))
    # dL/dw_i
    g = scale(add(dot[:, :-1], dot[:, 1:]), 0.5, 0)
    if white_back and fault != 'wb_no_sumG':
        g = sub(g, MR(sumG.m[:, None].expand_as(g.m), sumG.r[:, None].expand_as(g.m)))
    if gws is not None and fault != 'no_wsum':
        g = add(g, MR(gws[:, None].expand_as(g.m)))
    if gd is not None and fault != 'no_depth':
        draw = div(swd, sw)
        gdw = div(MR(gd), sw)
        lo, hi = float(rng[0]), float(rng[1])
        exact_zero = (sw.m == 0) & (sw.r == 0)
        with np.errstate(all='ignore'):
            ok = (gd != 0) & torch.isfinite(draw.m) & (draw.m >= lo) & (draw.m <= hi) & ~exact_zero
            sure_ok = (gd != 0) & (sw.m - sw.r > 0) & (draw.m - draw.r >= lo) & (draw.m + draw.r <= hi)
            sure_not = (gd == 0) | exact_zero | (draw.m + draw.r < lo) | (draw.m - draw.r > hi)
        unsure = ~(sure_ok | sure_not)
        dz = sub(dmid, MR(draw.m[:, None].expand_as(dmid.m), draw.r[:, None].expand_as(dmid.m)))
        gdw2 = MR(gdw.m[:, None].expand_as(dz.m), gdw.r[:, None].expand_as(dz.m))
        term = mul(gdw2, dz, 0)
        with_t = add(g, MR(torch.nan_to_num(term.m), torch.nan_to_num(term.r, nan=math.inf)))
        g = either(ok[:, None].expand_as(g.m), unsure[:, None].expand_as(g.m), with_t, g)
    gw = MR(g.m * w.m, g.m.abs() * w.r + g.r * w.mag())
    # exclusive suffix sum: up to K FMAs per lane, the 5-level scan, K more
    suf = lambda v: torch.cat([torch.flip(torch.cumsum(torch.flip(v, [1]), 1), [1])[:, 1:], torch.zeros_like(v[:, :1])], 1)  # noqa: E731
    run = MR(suf(gw.m), suf(gw.r) + gam(2 * K + 6) * suf(gw.mag()))
    g_alpha = sub(mul(g, T), div(run, t, c['eps']))
    sg = switch20(x, _sgm, REL_SIG, lambda v: torch.ones_like(v))
    gsm = mul(mul(mul(g_alpha, e), delta), sg)
    pad = lambda v: torch.cat([zero[:, :1], v, zero[:, :1]], 1)           # noqa: E731
    gsig = scale(add(MR(pad(gsm.m)[:, :-1], pad(gsm.r)[:, :-1]), MR(pad(gsm.m)[:, 1:], pad(gsm.r)[:, 1:])), 0.5, 0)
    if fault == 'coef_wj':
        coef = MR(pad(w.m)[:, 1:], pad(w.r)[:, 1:])
    else:
        coef = scale(add(MR(pad(w.m)[:, :-1], pad(w.r)[:, :-1]), MR(pad(w.m)[:, 1:], pad(w.r)[:, 1:])), 0.5, 0)
    return gsig, coef


def render_bwd_model(planes, params, sigma_net, masks, o, d, ds, g_feat, g_depth, g_wsum, depth_range, white_back, box_warp,
                     chain, fault=None, consts=FP32, device='cpu', chunk_samples=1 << 19, want_planes=True, want_params=True):
    """One p3d_render_bwd launch from its fp32 inputs (numpy or torch): planes [B,3,H,W,32], params per net (w1, b1, w2, b2)
    effective, o / d [B,R,3], ds [B,R,S], g_feat [B,R,32 n_nets], g_depth / g_wsum [B,R] or None, depth_range (lo, hi) or
    None, `chain` the parameter gradients' chain length (param_chain). Returns {'planes': (mid, rad) [B,3,H,W,32],
    'params': (mid, rad) [n_nets, 4257]} as float64 tensors on `device`."""
    npf = lambda t: None if t is None else (t.detach().cpu().numpy() if torch.is_tensor(t) else np.asarray(t)).astype(np.float32)  # noqa: E731
    dev = torch.device(device)
    f64 = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float64)).to(dev)                                           # noqa: E731
    P_ = npf(planes)
    B, _, H, W, C = P_.shape
    o_, d_, ds_ = npf(o).reshape(-1, 3), npf(d).reshape(-1, 3), npf(ds)
    R, S = ds_.shape[1], ds_.shape[2]
    ds_ = ds_.reshape(-1, S)
    N = B * R
    NN = len(params)
    RT = 128 // S
    gf = npf(g_feat).reshape(N, 32 * NN).copy()
    gdp = None if g_depth is None else npf(g_depth).reshape(N).copy()
    gws = None if g_wsum is None else npf(g_wsum).reshape(N).copy()
    if fault == 'drop_last_ray':
        gf[-1] = 0
        for v in (gdp, gws):
            if v is not None:
                v[-1] = 0
    pl = f64(P_).reshape(B * 3 * H * W, C)
    prm = [[f64(npf(t)) for t in net] for net in params]
    cs = np.float32(2.0 / float(box_warp))
    c = consts
    cnt = lambda: torch.zeros(B * 3 * H * W, C, dtype=torch.float64, device=dev)                 # noqa: E731
    gp_m, gp_r, gp_a, gp_n = cnt(), cnt(), cnt(), cnt()
    par = [dict(m=[0.0] * 4, x=[0.0] * 4, a=[0.0] * 4) for _ in range(NN)]
    G_all = 2 * f64(gf)
    rays_per = max(1, chunk_samples // S)
    for r0 in range(0, N, rays_per):
        r1 = min(N, r0 + rays_per)
        n = r1 - r0
        gi = np.arange(r0, r1)
        img = gi // R if fault != 'first_image_planes' else (gi // RT * RT) // R
        pts = sample_points(o_[r0:r1], d_[r0:r1], ds_[r0:r1], cs)
        # features: the three planes' bilinear samples (taps in fp32, weights rounded once), their mean
        offs_k, wts_k, f = [], [], []
        for k, (a0, a1) in enumerate(PLANE_AXES):
            offs, wts = taps(pts[a0].reshape(-1), pts[a1].reshape(-1), H, W)
            wts = wts.astype(np.float32).astype(np.float64)
            base = (np.repeat(img, S) * 3 + k) * H * W
            offs_k.append(f64(base[None] + offs).long())
            wts_k.append(f64(wts))
            vals = [pl[offs_k[-1][t]] * wts_k[-1][t][:, None] for t in range(4)]
            fm = vals[0] + vals[1] + vals[2] + vals[3]
            fa = vals[0].abs() + vals[1].abs() + vals[2].abs() + vals[3].abs()
            f.append(MR(fm, gam(4) * fa + 4 * TINY))
        x = scale(add(add(f[0], f[1]), f[2]), c['third'])
        P = n * S
        G = G_all[r0:r1]                                                   # [n, 32 NN]
        Gs = G.repeat_interleave(S, 0)                                     # per sample
        # sweep 1: sigma and G . c per sample
        hid, sig, dot_m, dot_r, dot_a = [], None, 0, 0, 0
        for net, (w1, b1, w2, b2) in enumerate(prm):
            a1 = dotw(x, w1.T, 32, b1)
            h = switch20(a1, _sp, REL_SP, lambda v: v, EXP_ZERO)
            dsp = switch20(a1, _sgm, REL_SIG, lambda v: torch.ones_like(v), EXP_ZERO)
            o1 = dotw(h, w2.T, 64, b2)
            o2 = dotw(h, w2.T, 34, b2)
            hid.append((h, dsp, o2))
            if net == sigma_net:
                sig = o1[:, 0]
            on = torch.tensor([(masks[net] >> k) & 1 for k in range(32)], dtype=torch.bool, device=dev)[None]
            oc = o1[:, 1:]
            s = mono(oc, _sgm, REL_SIG)
            cc = _rnd(s.m * c['c1002'] - c['c0001'], s.r * c['c1002'])
            col = MR(torch.where(on, cc.m, oc.m), torch.where(on, cc.r, oc.r))
            Gn = Gs[:, 32 * net:32 * net + 32]
            dot_m = dot_m + (Gn * col.m).sum(1)
            dot_r = dot_r + (Gn.abs() * col.r).sum(1)
            dot_a = dot_a + (Gn.abs() * col.mag()).sum(1)
        dot = MR(dot_m, dot_r + gam(32 * NN) * dot_a)
        sumG = MR(G.sum(1), gam(NN + 5) * G.abs().sum(1))
        rng = None if depth_range is None else [float(v) for v in npf(depth_range).reshape(2)]
        gsig, coef = _march_bwd(f64(ds_[r0:r1]), MR(sig.m.view(n, S), sig.r.view(n, S)), MR(dot.m.view(n, S), dot.r.view(n, S)),
                                sumG, None if gdp is None else f64(gdp[r0:r1]), None if gws is None else f64(gws[r0:r1]),
                                rng, white_back, c, fault)
        gsig, coef = MR(gsig.m.reshape(P), gsig.r.reshape(P)), MR(coef.m.reshape(P), coef.r.reshape(P))
        # sweep 2: the G row each sample reads (fault: the second half of a ray straddling sample 64 of its tile reads its
        # neighbour's)
        G2 = Gs
        if fault == 'straddle_G':
            rl = torch.from_numpy(np.repeat(gi % RT, S)).to(dev)
            sl = torch.arange(P, device=dev) % S
            p_loc = rl * S + sl
            hit = (rl >= 1) & (rl * S < 64) & ((rl + 1) * S > 64) & (p_loc >= 64)
            G2 = torch.where(hit[:, None], torch.roll(Gs, S, 0), Gs)
        gx = None
        for net, (w1, b1, w2, b2) in enumerate(prm):
            h, dsp, o2 = hid[net]
            cols = []
            on = [(masks[net] >> k) & 1 for k in range(32)]
            gsel = G2[:, 32 * net:32 * net + 32]
            d0 = mul(MR(coef.m[:, None].expand(P, 32), coef.r[:, None].expand(P, 32)), MR(gsel))
            sg2 = mono(o2[:, 1:], _sgm, REL_SIG)
            one = MR(torch.ones_like(sg2.m))
            k1002 = 1.0 if fault == 'no_1002' else c['c1002']
            der = scale(mul(sg2, sub(one, sg2)), k1002)
            dmask = mul(d0, der)
            onm = torch.tensor(on, dtype=torch.bool, device=dev)[None]
            gcol = MR(torch.where(onm, dmask.m, d0.m), torch.where(onm, dmask.r, d0.r))
            gs0 = gsig if net == sigma_net else MR(torch.zeros_like(gsig.m))
            go = MR(torch.cat([gs0.m[:, None], gcol.m], 1), torch.cat([gs0.r[:, None], gcol.r], 1))
            gh = dotw(go, w2, 18)
            ga = mul(gh, dsp)
            gxn = dotw(ga, w1, 33)
            gx = gxn if gx is None else add(gx, gxn)
            if want_params:
                for i, (A, Bv) in enumerate(((ga, x), (ga, None), (go, h), (go, None))):
                    if Bv is None:
                        m, xr, a = A.m.sum(0), A.r.sum(0), A.mag().sum(0)
                    else:
                        m = A.m.T @ Bv.m
                        a = A.mag().T @ Bv.mag()
                        xr = a - A.m.abs().T @ Bv.m.abs()
                    par[net]['m'][i] = par[net]['m'][i] + m
                    par[net]['x'][i] = par[net]['x'][i] + xr
                    par[net]['a'][i] = par[net]['a'][i] + a
        if want_planes:
            gv = gx if fault == 'no_third' else scale(gx, c['third'])
            for k in range(3):
                for t in range(4):
                    if fault == 'drop_o11' and t == 3:
                        continue
                    w = wts_k[k][t][:, None]
                    idx = offs_k[k][t]
                    gp_m.index_add_(0, idx, w * gv.m)
                    gp_r.index_add_(0, idx, torch.where(w != 0, w.abs() * gv.r, 0.0))     # skipped taps add nothing
                    gp_a.index_add_(0, idx, torch.where(w != 0, w.abs() * gv.mag(), 0.0))
                    gp_n.index_add_(0, idx, (w != 0).to(torch.float64).expand(-1, C))
    out = {}
    if want_planes:
        out['planes'] = (gp_m.view(B, 3, H, W, C), (gp_r + gam(gp_n + 1) * gp_a + gp_n * TINY).view(B, 3, H, W, C))
    if want_params:
        gc = gam(chain + 1)
        mids, rads = [], []
        for net in range(NN):
            pm, px, pa = par[net]['m'], par[net]['x'], par[net]['a']
            mids.append(torch.cat([t.reshape(-1) for t in pm]))
            rads.append(torch.cat([(px[i] + gc * pa[i]).reshape(-1) + chain * TINY for i in range(4)]))
        out['params'] = (torch.stack(mids), torch.stack(rads))
    return out


# ---------------------------------------------------------------------------------------------------------------------
# checks
# ---------------------------------------------------------------------------------------------------------------------
def out_of_bound(got, mid, rad):
    got = got.to(mid.device, torch.float64).reshape(mid.shape)
    err = torch.where(got == mid, torch.zeros_like(mid), (got - mid).abs())
    return ~(err <= rad + FLOOR)


def ratio(got, mid, rad):
    got = got.to(mid.device, torch.float64).reshape(mid.shape)
    r = torch.where(got == mid, torch.zeros_like(mid), (got - mid).abs() / (rad + FLOOR))
    r = torch.nan_to_num(r, nan=math.inf)
    return float(r.max()) if r.numel() else 0.0


WORST = {}


@pytest.fixture(scope='module', autouse=True)
def _worst_report():
    """Prints the worst err / rad seen per output by the tests of this module that ran."""
    yield
    if WORST:
        print('\nworst err / rad per output:')
        for k in sorted(WORST):
            print(f'  {k:34s} {WORST[k]:.3g}')


def check(name, got, mid, rad):
    assert bool(torch.isfinite(rad).all()), f'{name}: the model could not bound every element (a vacuous check)'
    bad = out_of_bound(got, mid, rad)
    w = ratio(got, mid, rad)
    WORST[name] = max(WORST.get(name, 0.0), w)
    assert not bool(bad.any()), f'{name}: {int(bad.sum())} of {bad.numel()} elements out of bound (worst err/rad {w:.3g})'


# ---------------------------------------------------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------------------------------------------------
def _decoder(name, gen, lr_mul=1.0):
    """A decoder module with random parameters -> (module, effective params per net, sigma_net, masks)."""
    from pix2pix3d_b200 import native
    from pix2pix3d_b200.training import triplane, triplane_cond as tc
    base = {'decoder_lr_mul': lr_mul, 'decoder_output_dim': 32}
    dec = {
        'osg': lambda: triplane.OSGDecoder(32, dict(base)),
        'semantic_sigmoid': lambda: tc.OSGDecoder_semantic(32, dict(base, sigmoid=True)),
        'semantic_raw': lambda: tc.OSGDecoder_semantic(32, dict(base, sigmoid=False)),
        'entangle_raw6': lambda: tc.OSGDecoder_semantic_entangle(32, dict(base, sigmoid=False, semantic_channels=6)),
        'entangle_raw19': lambda: tc.OSGDecoder_semantic_entangle(32, dict(base, sigmoid=False, semantic_channels=19)),
        'late_sigmoid': lambda: tc.OSGDecoder_semantic_lateSeparate(32, dict(base, sigmoid=True)),
        'late_raw': lambda: tc.OSGDecoder_semantic_lateSeparate(32, dict(base, sigmoid=False)),
    }[name]()
    with torch.no_grad():
        for p in dec.parameters():
            p.add_(0.3 * torch.randn(p.shape, generator=gen))
    nets, sigma_net, masks = native.describe_decoder(dec)
    params = [[*native._effective_fc(n[0]), *native._effective_fc(n[2])] for n in nets]
    return dec, [[t.detach().clone() for t in p] for p in params], sigma_net, masks


def make_case(B, R, S, dec_name, seed=0, H=8, W=8, box_warp=1.0, grads=('feat', 'depth', 'wsum'), white_back=False,
              narrow=False, extreme=None, quantised=False):
    """Inputs of one launch (CPU fp32 tensors). `quantised`: rays, directions and depths on coarse dyadic grids, so that every
    fp32 coordinate and grid position is exact and float64 grid_sample sees the kernel's taps. `extreme`: 'logits' (colour
    logits over [-25, 25]), 'pre20' (hidden pre-activations beyond 20), 'opaque' (densities that make T hit its 1e-10 floor),
    'zero_w' (every sample of some rays at one depth), 'contention' (all rays through one point), 'centres' (rays of zero
    direction sitting on texel centres: taps of weight 0)."""
    gen = torch.Generator().manual_seed(seed)
    torch.manual_seed(seed)                           # the modules' own initialisation
    dec, params, sigma_net, masks = _decoder(dec_name, gen)
    NN = len(params)
    if extreme == 'logits':
        for p in params:
            p[2].mul_(1e-3)
            p[3][1:] = torch.linspace(-25, 25, 32)
    elif extreme == 'pre20':
        for p in params:
            p[1].copy_(torch.linspace(18, 30, 64)[torch.randperm(64, generator=gen)])
            p[2].mul_(0.05)                         # outputs of moderate size: unsaturated colours, moderate densities
    elif extreme == 'opaque':                       # densities over +-3000: opaque samples (alpha = 1, T down to 1e-10 and
        params[sigma_net][2][0] *= 1000.0           # below) beside empty ones, and the march's softplus switch at 20
        params[sigma_net][3][0] += 500.0
    planes = 0.5 * torch.randn(B, 3, H, W, 32, generator=gen)
    o = torch.randn(B, R, 3, generator=gen)
    o = o / o.norm(dim=-1, keepdim=True) * 2.7
    d = -o + 0.3 * torch.randn(B, R, 3, generator=gen)
    d = d / d.norm(dim=-1, keepdim=True)
    ds = torch.sort(torch.linspace(2.0, 3.4, S).expand(B, R, S) + 0.05 * torch.rand(B, R, S, generator=gen), -1)[0]
    if extreme == 'contention':
        t = 2.7
        p0 = torch.tensor([0.11, -0.07, 0.05])
        d = p0 - o
        d = d / d.norm(dim=-1, keepdim=True)
        o = p0 - t * d
        ds = torch.sort(t + 0.002 * torch.randn(B, R, S, generator=gen), -1)[0]
    if extreme == 'centres':
        assert H == W and box_warp == 1.0                 # cs = 2: o = g / 2 is exact
        j = torch.randint(0, W, (B, R, 3), generator=gen).double()
        o = (((2 * j + 1) / W - 1) / 2).float()
        d[:, ::2] = 0                                     # every sample of these rays on texel centres of all three planes
    if quantised:
        o = torch.round(o * 256) / 256
        d = torch.round(d * 16) / 16
        ds = torch.sort(torch.round(ds * 32) / 32, -1)[0]
    if extreme == 'zero_w':
        ds[:, ::3] = ds[:, ::3, :1]
    g_feat = torch.randn(B, R, 32 * NN, generator=gen) if 'feat' in grads else torch.zeros(B, R, 32 * NN)
    g_depth = torch.randn(B, R, generator=gen) if 'depth' in grads else None
    if g_depth is not None:
        g_depth[:, 3::7] = 0
    g_wsum = torch.randn(B, R, generator=gen) if 'wsum' in grads else None
    rng = None
    if g_depth is not None:
        lo, hi = float(ds.min()), float(ds.max())
        if narrow:
            lo, hi = float(torch.quantile(ds.double(), 0.45)), float(torch.quantile(ds.double(), 0.5))
        rng = torch.tensor([lo, hi], dtype=torch.float32)
    return dict(dec=dec, planes=planes, params=params, sigma_net=sigma_net, masks=masks, o=o, d=d, ds=ds, g_feat=g_feat,
                g_depth=g_depth, g_wsum=g_wsum, depth_range=rng, white_back=white_back, box_warp=box_warp)


def model_of(c, chain, fault=None, consts=FP32, device='cpu', **kw):
    return render_bwd_model(c['planes'], c['params'], c['sigma_net'], c['masks'], c['o'], c['d'], c['ds'], c['g_feat'],
                            c['g_depth'], c['g_wsum'], c['depth_range'], c['white_back'], c['box_warp'], chain, fault=fault,
                            consts=consts, device=device, **kw)


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the model's midpoints against float64 autograd of the staged chain
# ---------------------------------------------------------------------------------------------------------------------
def _staged64(c):
    """Gradients of the staged chain in float64 (F.grid_sample, the decoder module, MipRayMarcher2's march with the launch's
    clamp range) at the launch's fp32 sample coordinates and sorted depths, w.r.t. the channels-last planes and the
    effective parameters."""
    import copy
    from pix2pix3d_b200.training.volumetric_rendering.renderer import generate_planes, project_onto_planes
    B, _, H, W, C = c['planes'].shape
    R, S = c['ds'].shape[1:]
    cs = np.float32(2.0 / c['box_warp'])
    pts = sample_points(c['o'].numpy().reshape(-1, 3), c['d'].numpy().reshape(-1, 3), c['ds'].numpy().reshape(-1, S), cs)
    coords = torch.from_numpy(np.stack(pts, -1).astype(np.float64)).reshape(B, R * S, 3)
    dec = copy.deepcopy(c['dec']).double()
    from pix2pix3d_b200 import native
    nets = native.describe_decoder(dec)[0]
    eff = []
    for net, prm in zip(nets, c['params']):
        for fc, w, b in ((net[0], prm[0], prm[1]), (net[2], prm[2], prm[3])):
            fc.weight.data = w.double() / fc.weight_gain
            fc.bias.data = b.double() / fc.bias_gain
            eff += [(fc.weight, fc.weight_gain), (fc.bias, fc.bias_gain)]
    planes = c['planes'].double().permute(0, 1, 4, 2, 3).contiguous().requires_grad_(True)
    grid = project_onto_planes(generate_planes().double(), coords).unsqueeze(1)
    f = F.grid_sample(planes.reshape(B * 3, C, H, W), grid, mode='bilinear', padding_mode='zeros', align_corners=False)
    feats = f.permute(0, 3, 2, 1).reshape(B, 3, R * S, C)
    out = dec(feats, None)
    colors, dens = out['rgb'].reshape(B, R, S, -1), out['sigma'].reshape(B, R, S, 1)
    z = c['ds'].double().unsqueeze(-1)
    delta = z[:, :, 1:] - z[:, :, :-1]
    c_mid = (colors[:, :, :-1] + colors[:, :, 1:]) / 2
    sigma = F.softplus((dens[:, :, :-1] + dens[:, :, 1:]) / 2 - 1)
    alpha = 1 - torch.exp(-(sigma * delta))
    trans = torch.cumprod(torch.cat([torch.ones_like(alpha[:, :, :1]), 1 - alpha + 1e-10], -2), -2)[:, :, :-1]
    w = alpha * trans
    rgb = (w * c_mid).sum(-2)
    wsum = w.sum(2)
    loss = 0
    if c['white_back']:
        rgb = rgb + 1 - wsum
    loss = loss + ((rgb * 2 - 1) * c['g_feat'].double()).sum()
    if c['g_depth'] is not None:
        # nan_to_num(0 / 0) as a where, so that the zero-weight rays' gradient is 0 rather than NaN
        pos = wsum > 0
        depth = torch.where(pos, (w * (z[:, :, :-1] + z[:, :, 1:]) / 2).sum(-2) / torch.where(pos, wsum, torch.ones_like(wsum)),
                            torch.full_like(wsum, math.inf))
        lo, hi = (float(v) for v in c['depth_range'])
        loss = loss + (torch.clamp(depth, lo, hi).reshape(B, R) * c['g_depth'].double()).sum()
    if c['g_wsum'] is not None:
        loss = loss + (wsum.reshape(B, R) * c['g_wsum'].double()).sum()
    leaves = [planes] + [p for p, _ in eff]
    gr = torch.autograd.grad(loss, leaves, allow_unused=True)
    g_planes = gr[0].permute(0, 1, 3, 4, 2)
    g_par = []
    for i in range(len(nets)):
        g4 = [(gr[1 + 4 * i + k] if gr[1 + 4 * i + k] is not None else torch.zeros_like(eff[4 * i + k][0])) / eff[4 * i + k][1]
              for k in range(4)]
        g_par.append(torch.cat([t.reshape(-1) for t in g4]))
    return g_planes, torch.stack(g_par)


def _agree(got, want, tol=1e-12):
    """Per element: |got - want| <= tol (|want| + 1e-3 max|want|) (the second term admits elements that are sums with
    cancellation: their float64 rounding is relative to the terms, not to the result)."""
    scale_ = want.abs().max().item()
    err = (got - want).abs()
    return bool((err <= tol * (want.abs() + 1e-3 * scale_)).all()), float((err / (want.abs() + 1e-3 * scale_ + 1e-300)).max())


AUTOGRAD_CASES = {
    'osg': dict(dec_name='osg'),
    'late_sigmoid white_back': dict(dec_name='late_sigmoid', white_back=True),
    'late_raw narrow': dict(dec_name='late_raw', narrow=True),
    'entangle_raw6 feat': dict(dec_name='entangle_raw6', grads=('feat',)),
    'semantic_raw feat+depth': dict(dec_name='semantic_raw', grads=('feat', 'depth')),
    'semantic_sigmoid feat+wsum': dict(dec_name='semantic_sigmoid', grads=('feat', 'wsum'), white_back=True),
    'osg depth+wsum': dict(dec_name='osg', grads=('depth', 'wsum')),
    'late_sigmoid zero_w': dict(dec_name='late_sigmoid', extreme='zero_w'),
}


@pytest.mark.parametrize('case', list(AUTOGRAD_CASES))
def test_model_midpoints_equal_float64_autograd(case):
    kw = dict(AUTOGRAD_CASES[case])
    c = make_case(2, 9, 11, seed=len(case), H=5, W=7, quantised=True, **kw)
    ref_planes, ref_params = _staged64(c)
    m = model_of(c, 100, consts=EXACT)
    ok, w = _agree(m['planes'][0], ref_planes)
    assert ok, ('planes', w)
    ok, w = _agree(m['params'][0], ref_params)
    assert ok, ('params', w)


# ---------------------------------------------------------------------------------------------------------------------
# CPU: planted faults, the grid mirror
# ---------------------------------------------------------------------------------------------------------------------
def fault_case():
    """B = 2 images of R = 7 rays, S = 43 (two rays per tile, the second straddling sample 64; tile 3 holds ray 6 of image 0
    and ray 0 of image 1; the last tile is ragged), two nets with sigmoids, every upstream gradient, white_back."""
    return make_case(2, 7, 43, 'late_sigmoid', seed=5, H=5, W=7, white_back=True)


def _fraction(bad_planes, bad_params):
    return float(bad_planes.double().mean()), float(bad_params.double().mean())


def test_bounds_reject_planted_faults():
    c = fault_case()
    grid = bwd_grid(14, 43, 2, 132)
    chain = param_chain(14, 43, grid)
    clean = model_of(c, chain)
    report = {}
    for fault in FAULTS:
        bad = model_of(c, chain, fault=fault)
        report[fault] = _fraction(out_of_bound(bad['planes'][0], *clean['planes']), out_of_bound(bad['params'][0], *clean['params']))
    print('\nfraction of elements out of bound per planted fault (planes, params):')
    for k, v in report.items():
        print(f'  {k:20s} {v[0]:.3f} {v[1]:.3f}')
    for k, v in report.items():
        assert max(v) > 0.01, (k, v)


def test_grid_mirror():
    """make_rb_layout's size and the occupancy rule: two CTAs per SM except two nets at S <= 5."""
    assert DEC_SMEM_FLOATS == 4452
    assert rb_layout_floats(96, 2) == 27528
    assert rb_layout_floats(2, 2) == 31560
    for S in range(2, 129):
        for nn in (1, 2):
            g = bwd_grid(10 ** 6, S, nn, 132)
            assert g['per_sm'] == (1 if nn == 2 and S <= 5 else 2), (S, nn)
            assert g['RT'] * S <= 128 and (g['RT'] + 1) * S > 128
    g = bwd_grid(1000, 43, 1, 132)
    assert g['tiles'] == 500 and g['ctas'] == 264
    # the chain: CTA 0 walks tiles 0, 264 (two full tiles of two rays); the reduce adds 264
    assert param_chain(1000, 43, g) == 2 * 2 * 43 + 264
    g = bwd_grid(3, 43, 1, 132)
    assert g['ctas'] == 2 and param_chain(3, 43, g) == 2 * 43 + 2


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def gpu_grid(n_rays, S, n_nets):
    smem, res = device_smem()
    return bwd_grid(n_rays, S, n_nets, _sms(), smem, res)


def run_launch(c, name, want_planes=True, want_params=True, fault=None, check_ws=True):
    """One p3d_render_bwd launch on NaN-prefilled buffers longer than it needs; checks that nothing past its own elements
    changed, that the launch wrote exactly the mirror's n_nets * ctas workspace slices, and every element against the model.
    Returns (g_planes, g_params, grid)."""
    from pix2pix3d_b200 import native
    dev = torch.device('cuda')
    B, R, S = c['ds'].shape
    NN = len(c['params'])
    H, W = c['planes'].shape[2:4]
    grid = gpu_grid(B * R, S, NN)
    n_pl, n_par = B * 3 * H * W * 32, NN * DEC_PARAMS
    ws_need = NN * grid['ctas'] * DEC_PARAMS
    bufs = dict(planes=nan_buf(n_pl), params=nan_buf(n_par), workspace=nan_buf(NN * 2 * _sms() * DEC_PARAMS))
    cu = lambda t: None if t is None else t.to(dev)                     # noqa: E731
    gp, gq = native.render_bwd(cu(c['planes']), [[cu(t) for t in p] for p in c['params']], c['sigma_net'], c['masks'], cu(c['o']),
                               cu(c['d']), cu(c['ds']), *split(S), c['box_warp'], cu(c['g_feat']), cu(c['g_depth']), cu(c['g_wsum']),
                               cu(c['depth_range']), white_back=c['white_back'], want_planes=want_planes,
                               want_params=want_params, out=bufs)
    torch.cuda.synchronize()
    ws = bufs['workspace']
    if want_params:
        if check_ws:
            written = int((~torch.isnan(ws)).sum())
            assert written == ws_need and not torch.isnan(ws[:ws_need]).any(), \
                f'{name}: the launch wrote {written / DEC_PARAMS:.2f} workspace slices, the mirror says {NN} x {grid["ctas"]}'
        assert untouched(bufs['params'], n_par), f'{name}: wrote past g_params'
    else:
        assert bool(torch.isnan(ws).all()) and bool(torch.isnan(bufs['params']).all()), f'{name}: params written without want_params'
    if want_planes:
        assert untouched(bufs['planes'], n_pl), f'{name}: wrote past g_planes'
    else:
        assert bool(torch.isnan(bufs['planes']).all())
    m = model_of(c, param_chain(B * R, S, grid), fault=fault, device='cuda', want_planes=want_planes, want_params=want_params)
    if fault is None:
        if want_planes:
            check(f'{name} planes' if name else 'planes', gp, *m['planes'])
        if want_params:
            check(f'{name} params' if name else 'params', gq, *m['params'])
    return gp, gq, grid, m


def tile_shape(T, RT):
    """(B, R): B >= 2 images of R rays whose B R rays make T tiles, the last one ragged and one crossing an image boundary
    (R % RT != 0) where RT > 1 allows it."""
    if RT == 1:
        return (1, 1) if T == 1 else min(((B, T // B) for B in range(2, T + 1) if T % B == 0))
    for n in range(T * RT - 1, (T - 1) * RT, -1):
        for B in range(2, min(n, 64) + 1):
            if n % B == 0 and (n // B) % RT != 0:
                return B, n // B
    return 1, T * RT - 1                               # one ragged tile of too few rays for two images


def split(S):
    """(Sc, Sf) of a sample count: coarse only at S = 6 (Sf = 0), 13 + 11 at S = 24, halves otherwise (each at most 64)."""
    return {6: (6, 0), 24: (13, 11)}.get(S, (S - S // 2, S // 2))


SAMPLE_COUNTS = [2, 3, 5, 6, 24, 43, 63, 64, 65, 96, 127, 128]


@gpu
@pytest.mark.parametrize('S', SAMPLE_COUNTS)
@pytest.mark.parametrize('dec_name', ['osg', 'late_sigmoid'])
def test_sample_counts(S, dec_name):
    """Every sample count class of the tile schedule (RT = floor(128 / S) rays per tile; sweep 2's halves of 64 samples, a
    ray straddling sample 64 at S = 3, 5, 24, 43; ragged second halves at 65..127), with a ragged last tile and a tile that
    crosses an image boundary; white_back on odd S."""
    RT = 128 // S
    B, R = tile_shape(5, RT)
    c = make_case(B, R, S, dec_name, seed=S, white_back=S % 2 == 1)
    run_launch(c, '')


@gpu
@pytest.mark.parametrize('which', ['1', 'ctas-1', 'ctas', 'ctas+1', '2ctas+1'])
@pytest.mark.parametrize('S,dec_name', [(5, 'late_raw'), (43, 'osg'), (96, 'late_sigmoid')])
def test_tile_counts(which, S, dec_name):
    """1, ctas - 1, ctas, ctas + 1 and 2 ctas + 1 tiles (ctas from the mirror: one CTA per SM for two nets at S = 5, two
    otherwise), each with a ragged last tile where RT > 1. The workspace check confirms the mirror's ctas."""
    NN = 2 if dec_name.startswith('late') else 1
    g = gpu_grid(10 ** 7, S, NN)
    ctas = g['ctas']
    T = {'1': 1, 'ctas-1': ctas - 1, 'ctas': ctas, 'ctas+1': ctas + 1, '2ctas+1': 2 * ctas + 1}[which]
    B, R = tile_shape(T, g['RT'])
    c = make_case(B, R, S, dec_name, seed=T, H=16, W=16, grads=('feat', 'depth'))
    _, _, grid, _ = run_launch(c, '')
    assert grid['tiles'] == T
    print(f'S={S} n_nets={NN}: {grid["per_sm"]} CTA(s)/SM, {grid["ctas"]} CTAs, {T} tiles')


@gpu
@pytest.mark.parametrize('dec_name', ['osg', 'semantic_sigmoid', 'semantic_raw', 'entangle_raw6', 'entangle_raw19', 'late_sigmoid',
                                      'late_raw'])
def test_decoders(dec_name):
    c = make_case(2, 45, 24, dec_name, seed=3, white_back=dec_name.endswith('raw'))
    run_launch(c, '')


UPSTREAM = {
    'feat': dict(grads=('feat',)),
    'feat+depth': dict(grads=('feat', 'depth')),
    'feat+depth narrow': dict(grads=('feat', 'depth'), narrow=True),
    'feat+wsum': dict(grads=('feat', 'wsum')),
    'zero feat': dict(grads=('depth', 'wsum')),
    'white_back': dict(grads=('feat', 'depth', 'wsum'), white_back=True),
}


@gpu
@pytest.mark.parametrize('case', list(UPSTREAM))
def test_upstream_gradients(case):
    c = make_case(3, 41, 43, 'late_sigmoid', seed=11, **UPSTREAM[case])
    run_launch(c, '')


@gpu
def test_want_planes_or_params_only():
    """Each output alone; g_params bit-identical with and without the plane scatter."""
    c = make_case(2, 41, 43, 'late_raw', seed=12, white_back=True)
    _, both, _, _ = run_launch(c, '')
    gp, none, _, _ = run_launch(c, 'planes only', want_params=False)
    assert none is None
    none, only, _, _ = run_launch(c, 'params only', want_planes=False)
    assert none is None and torch.equal(only, both)


PLANES = {
    '1x1': dict(H=1, W=1),
    '5x7': dict(H=5, W=7),
    '256x256 contention': dict(H=256, W=256, extreme='contention'),
    'box_warp 0.6': dict(H=12, W=10, box_warp=0.6),
    'texel centres': dict(H=6, W=6, extreme='centres'),
}


@gpu
@pytest.mark.parametrize('case', list(PLANES))
def test_planes(case):
    c = make_case(2, 61, 24, 'late_sigmoid', seed=13, **PLANES[case])
    run_launch(c, '')


@gpu
@pytest.mark.parametrize('case', ['logits', 'pre20', 'opaque', 'zero_w'])
def test_extremes(case):
    c = make_case(2, 61, 24, 'late_sigmoid' if case != 'logits' else 'osg', seed=14, extreme=case)
    run_launch(c, '')


@gpu
def test_planted_faults_against_the_kernel():
    """Each fault planted in the model puts a clear fraction of the kernel's elements outside the faulted model's bound."""
    c = fault_case()
    gp, gq, grid, _ = run_launch(c, 'fault case')
    report = {}
    for fault in FAULTS:
        B, R, S = c['ds'].shape
        m = model_of(c, param_chain(B * R, S, grid), fault=fault, device='cuda')
        report[fault] = _fraction(out_of_bound(gp, *m['planes']), out_of_bound(gq, *m['params']))
    print('\nfraction of the kernel\'s elements out of the faulted model\'s bound (planes, params):')
    for k, v in report.items():
        print(f'  {k:20s} {v[0]:.3f} {v[1]:.3f}')
    for k, v in report.items():
        assert max(v) > 0.01, (k, v)


# ---------------------------------------------------------------------------------------------------------------------
# replays
# ---------------------------------------------------------------------------------------------------------------------
@gpu
def test_config5_launch():
    """One launch at config-5 renderer shapes (tools/time_render_grad.py): 4 images, 128^2 rays, 48 + 48 samples,
    OSGDecoder_semantic_lateSeparate, 256^2 planes, every upstream gradient; the model runs on the device in float64
    chunks. Every element of g_planes and g_params is checked."""
    import time
    t0 = time.time()
    c = make_case(4, 128 * 128, 96, 'late_raw', seed=21, H=256, W=256)
    run_launch(c, 'config5')
    print(f'config-5 launch checked in {time.time() - t0:.1f} s')


REPLAY = """
import json, sys
sys.path[:0] = [{root!r}, {root!r} + '/baseline', {root!r} + '/tests', {root!r} + '/oracle']
import torch
import pix2pix3d_b200
pix2pix3d_b200.install(reference_root={ref!r})
from pix2pix3d_b200 import native, train_step as ts
import test_gpu_render_bwd_model as T
dev = torch.device('cuda')
real = native.render_bwd
stats = dict(launches=0, bad=0, elements=0, worst={{}})


def wrapped(planes_nhwc, params, sigma_net, masks, o, d, ds, Sc, Sf, box_warp, g_feat, g_depth=None, g_wsum=None,
            depth_range=None, white_back=False, want_planes=True, want_params=True, out=None):
    gp, gq = real(planes_nhwc, params, sigma_net, masks, o, d, ds, Sc, Sf, box_warp, g_feat, g_depth, g_wsum, depth_range,
                  white_back=white_back, want_planes=want_planes, want_params=want_params, out=out)
    B, R, S = ds.shape
    grid = T.gpu_grid(B * R, S, len(params))
    m = T.render_bwd_model(planes_nhwc, params, sigma_net, masks, o, d, ds, g_feat, g_depth, g_wsum, depth_range, white_back,
                           box_warp, T.param_chain(B * R, S, grid), device='cuda', want_planes=gp is not None,
                           want_params=gq is not None)
    for k, got in (('planes', gp), ('params', gq)):
        if got is None:
            continue
        bad = T.out_of_bound(got, *m[k])
        stats['bad'] += int(bad.sum())
        stats['elements'] += bad.numel()
        stats['worst'][k] = max(stats['worst'].get(k, 0.0), T.ratio(got, *m[k]))
    stats['launches'] += 1
    return gp, gq


native.render_bwd = wrapped
cfg = dict(ts.TINY_TRAIN)
st = ts.build(cfg, dev)
batch = ts.synthetic_batch(cfg, dev, 5)
torch.manual_seed(2)
st.batch_idx = 0
ts.run_iteration(st, batch)
torch.cuda.synchronize()
print('RESULT ' + json.dumps(stats))
"""


@gpu
def test_replay_training_iteration():
    """One run_iteration of the tiny training recipe (batch_idx 0: every phase); every p3d_render_bwd launch is checked
    element by element. Runs in a subprocess because install() re-maps module names."""
    import json
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    ref = os.path.join(root, 'oracle', '_ref')
    if not os.path.isdir(os.path.join(ref, 'training')):
        pytest.skip('the reference copy under oracle/_ref is made by build()')
    p = subprocess.run([sys.executable, '-c', REPLAY.format(root=root, ref=ref)], capture_output=True, text=True, timeout=900)
    line = [ln for ln in p.stdout.splitlines() if ln.startswith('RESULT ')]
    assert p.returncode == 0 and line, p.stdout[-3000:] + p.stderr[-3000:]
    r = json.loads(line[0][7:])
    print(f"\nreplay: {r['launches']} render_bwd launches, {r['elements']} elements, {r['bad']} out of bound, worst err/rad "
          f"{r['worst']}")
    for k, v in r['worst'].items():
        WORST[f'replay {k}'] = max(WORST.get(f'replay {k}', 0.0), v)
    assert r['launches'] > 0
    assert r['bad'] == 0, r
