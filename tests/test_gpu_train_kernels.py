"""The training path's stand-alone kernels against a float64 model of each launch, element by element.

These launches produce the gradients of the staged renderer chain (ImportanceSemanticRenderer, rays that require grad, density
noise, `renderer.fused_grad = False`) and of the density regulariser's `G.sample_mixed` in every Greg phase:

    p3d_sample_from_planes / _bwd      sample_planes_kernel (render.cu), sample_planes_bwd_kernel (render_bwd.cu)
    p3d_decoder_mlp_fwd / _bwd         decoder_mlp_{fwd,bwd,reduce}_kernel (decoder_train.cu)
    p3d_ray_march / _bwd               ray_march_kernel (render.cu), ray_march_bwd_kernel (render_bwd.cu)
    p3d_sample_importance              sample_importance_kernel (render.cu)

Each model restates one launch in float64 from the launch's own fp32 inputs and returns, with every result, a bound on how far
the kernel's fp32 result may lie from it. For a sum of n terms accumulated in fp32, in any order, that bound is

    gamma(n) * sum |terms|,        gamma(n) = n u / (1 - n u),  u = 2^-24,

with n the longest chain of roundings any term passes through in the kernel (the counts are derived next to each model from the
kernel's loop structure). Elementwise steps (softplus, sigmoid, the march) propagate the bounds of their inputs through the
step's derivative and add their own roundings (library expf / log1pf: 2 and 1 ulp). Every output element must satisfy
|got - ref| <= bound + FLOOR. A norm-wise check (max |a - b| / max |b|) cannot see an element far below the tensor's largest
one -- the gradient of a saturated sigmoid, of an interval behind an opaque sample, of a rarely touched texel -- so these tests
hold every element to its own bound instead.

Every launch writes into NaN-prefilled buffers longer than it needs; nothing past its own elements may change.
"""
import math

import numpy as np
import pytest
import torch

import p3d_oracle as O

gpu = pytest.mark.gpu

U = 2.0 ** -24
FLOOR = 2.0 ** -126           # fp32 subnormal results: a kernel may flush them
PAD = 1000
F1002, F0001, F1E10 = float(np.float32(1.002)), float(np.float32(0.001)), float(np.float32(1e-10))


def gam(n):
    n = np.asarray(n, np.float64)
    return n * U / (1 - n * U)


def _ceil(a, b):
    return -(-a // b)


# ---------------------------------------------------------------------------------------------------------------------
# Python mirrors of the launchers' grid rules
# ---------------------------------------------------------------------------------------------------------------------
def grid_decoder_fwd(P, sms):                 # p3d_decoder_mlp_fwd: thread per point, 128 threads, at most 8 CTAs per SM
    return min(_ceil(P, 128), 8 * sms)


def grid_decoder_bwd(P, sms):                 # p3d_decoder_mlp_bwd: 64-point tiles, 3 CTAs per SM, at most one CTA per tile
    return min(3 * sms, _ceil(P, 64))


def decoder_bwd_chain(P, sms):
    """Longest fp32 accumulation chain of a parameter gradient: the points of the busiest CTA (sequential FMAs across its
    tiles, padding rows add exact zeros) plus the fixed-order sum over the CTAs."""
    ctas = grid_decoder_bwd(P, sms)
    return _ceil(_ceil(P, 64), ctas) * 64 + ctas


def grid_sample_planes(points, sms):          # p3d_sample_from_planes: warp per point, 256 threads, at most 16 CTAs per SM
    return min(_ceil(points * 32, 256), 16 * sms)


def grid_sample_planes_bwd(points, sms):      # p3d_sample_from_planes_bwd: the same rule
    return min(_ceil(points, 8), 16 * sms)


def grid_ray_march(N, sms):                   # p3d_ray_march: warp per ray, 4 warps, at most 8 CTAs per SM
    return min(_ceil(N, 4), 8 * sms)


def grid_ray_march_bwd(N, sms):               # p3d_ray_march_bwd: warp per ray, 4 warps, at most 16 CTAs per SM
    return min(_ceil(N, 4), 16 * sms)


def importance_max_S():
    """Largest S whose per-CTA shared memory (4 warps x 4 arrays of round_up(S, 4) floats) fits the 48 KB static limit."""
    S = 4
    while 4 * 4 * _ceil(S + 1, 4) * 4 * 4 <= 48 * 1024:
        S += 1
    return S


# ---------------------------------------------------------------------------------------------------------------------
# models
# ---------------------------------------------------------------------------------------------------------------------
PLANE_AXES = ((0, 1), (0, 2), (2, 0))      # plane k samples (x, y), (x, z), (z, x) (render_common.cuh plane_values)


def taps(gx, gy, H, W, fault=None):
    """make_taps (render_common.cuh) on fp32 normalised coordinates: texel offsets [4,M] and the EXACT tap weights [4,M]
    (nw, ne, sw, se) of the fp32 positions. ix / iy and the fractions are formed with the kernel's fp32 operations (the
    fractions are exact), so the model's taps are the kernel's taps; the kernel's weight products round once."""
    f = np.float32
    with np.errstate(invalid='ignore'):
        ix = ((gx + f(1)) * f(W) - f(1)) * f(0.5)
        iy = ((gy + f(1)) * f(H) - f(1)) * f(0.5)
        inside = (ix > -1) & (ix < W) & (iy > -1) & (iy < H)
    ix, iy = np.where(inside, ix, f(0)), np.where(inside, iy, f(0))
    x0f, y0f = np.floor(ix), np.floor(iy)
    ax, bx = ((x0f + f(1)) - ix).astype(np.float64), (ix - x0f).astype(np.float64)
    ay, by = ((y0f + f(1)) - iy).astype(np.float64), (iy - y0f).astype(np.float64)
    x0, y0 = x0f.astype(np.int64), y0f.astype(np.int64)
    offs, wts = [], []
    for dy, dx, w in ((0, 0, ax * ay), (0, 1, bx * ay), (1, 0, ax * by), (1, 1, bx * by)):
        xx, yy = x0 + dx, y0 + dy
        ok = inside & (xx >= 0) & (xx < W) & (yy >= 0) & (yy < H)
        offs.append(np.where(ok, yy * W + xx, 0))
        wts.append(np.where(ok, w, 0.0))
    offs, wts = np.stack(offs), np.stack(wts)
    if fault == 'drop_tap':
        wts[3] = 0
    elif fault == 'swap_tap':
        wts[[1, 2]] = wts[[2, 1]]
    return offs, wts


def _plane_coords(coords, cs):
    return (np.float32(cs) * np.asarray(coords, np.float32))            # __fmul_rn(coord_scale, c)


def sample_planes_model(planes, coords, cs, fault=None):
    """planes [B,3,H,W,32] fp32 (channels last), coords [B,M,3], cs = coord scale -> (ref, bound) [B,3,M,32]. The kernel sums
    the four taps as one product and three FMAs after rounding each weight: 5 roundings per term."""
    B, _, H, W, C = planes.shape
    p = _plane_coords(coords, cs)
    ref = np.zeros((B, 3, p.shape[1], C))
    tab = np.zeros_like(ref)
    for b in range(B):
        for k, (a0, a1) in enumerate(PLANE_AXES):
            offs, wts = taps(p[b, :, a0], p[b, :, a1], H, W, fault)
            pl = planes[b, k].reshape(H * W, C).astype(np.float64)
            for t in range(4):
                v = pl[offs[t]] * wts[t][:, None]
                ref[b, k] += v
                tab[b, k] += np.abs(v)
    return ref, gam(5) * tab


def sample_planes_bwd_model(grad, coords, cs, H, W, fault=None):
    """grad [B,3,M,32] -> (ref, bound) [B,3,H,W,32]: the scatter of w g over the taps. Each contribution rounds twice (weight,
    product) and the fp32 atomics add a texel's n contributions in any order: gamma(n + 1) of the texel's sum of |w g|."""
    B, _, M, C = grad.shape
    p = _plane_coords(coords, cs)
    ref = np.zeros((B, 3, H * W, C))
    tab = np.zeros_like(ref)
    cnt = np.zeros((B, 3, H * W, 1))
    g = grad.astype(np.float64)
    for b in range(B):
        for k, (a0, a1) in enumerate(PLANE_AXES):
            offs, wts = taps(p[b, :, a0], p[b, :, a1], H, W, fault)
            for t in range(4):
                v = wts[t][:, None] * g[b, k]
                np.add.at(ref[b, k], offs[t], v)
                np.add.at(tab[b, k], offs[t], np.abs(v))
                np.add.at(cnt[b, k], offs[t], (wts[t] != 0).astype(np.float64)[:, None])
    return ref.reshape(B, 3, H, W, C), (gam(cnt + 1) * tab).reshape(B, 3, H, W, C)


def _softplus(a):
    z = np.exp(np.minimum(a, 20.0))
    return np.where(a > 20, a, np.log1p(z)), np.where(a > 20, 1.0, z / (z + 1.0))


def _sigmoid(x):
    return 0.5 * (1 + np.tanh(0.5 * x))


def _mean_planes(feats, fault=None):
    f = feats.astype(np.float64)
    x = (f[:, 0] + f[:, 1] + f[:, 2]).reshape(-1, f.shape[-1])
    xa = (np.abs(f[:, 0]) + np.abs(f[:, 1]) + np.abs(f[:, 2])).reshape(-1, f.shape[-1]) / 3
    return (x if fault == 'no_third' else x / 3), xa


def decoder_fwd_model(feats, w1, b1, w2, b2, mask, fault=None):
    """p3d_decoder_mlp_fwd on feats [N,3,M,32] and the EFFECTIVE parameters -> dict of (ref, bound) for rgb [P,32], sigma [P],
    pre [P,64], sig [P,32]. Roundings per term: the plane mean 4 (two adds, the rounded 1/3, the product); the hidden layer a
    32-FMA chain from b1 (+ the mean's 4 = 37); softplus is 1-Lipschitz, plus expf / log1pf (4 u of h); the output layer a
    64-FMA chain from b2 (65); sigmoid propagates its input bound through its derivative plus expf, the add and the divide
    (4 u of s); 1.002 s - 0.001 is one FMA."""
    w1, b1, w2, b2 = (np.asarray(t, np.float64) for t in (w1, b1, w2, b2))
    x, xa = _mean_planes(feats, fault)
    a1 = x @ w1.T + b1
    ea1 = gam(37) * (xa @ np.abs(w1).T + np.abs(b1))
    h, _ = _softplus(a1)
    eh = ea1 + 4 * U * h
    o = h @ w2.T + b2
    eo = gam(65) * (h @ np.abs(w2).T + np.abs(b2)) + eh @ np.abs(w2).T
    m = mask ^ (1 << 5) if fault == 'mask_bit' else mask
    on = ((m >> np.arange(32)) & 1).astype(bool)[None]
    oc, eoc = o[:, 1:], eo[:, 1:]
    s = _sigmoid(oc)
    mid = np.clip(0.0, oc - eoc, oc + eoc)               # the steepest point of the sigmoid within the input's bound
    es = _sigmoid(mid) * (1 - _sigmoid(mid)) * eoc + 4 * U * s
    y = s * F1002 - F0001
    ey = F1002 * es + U * (np.abs(y) + F1002 * es)
    return dict(rgb=(np.where(on, y, oc), np.where(on, ey, eoc)), sigma=(o[:, 0], eo[:, 0]), pre=(a1, ea1),
                sig=(np.where(on, s, 0.0), np.where(on, es, 0.0)))


def _f32_fma(a, b, c):
    return (np.asarray(a, np.float64) * b + c).astype(np.float32)


def decoder_bwd_model(feats, w1, b1, w2, b2, mask, pre, sig, g_rgb, g_sigma, chain, fault=None):
    """p3d_decoder_mlp_bwd from its own inputs (the saved fp32 pre-activations and sigmoid values are exact inputs here) ->
    dict of (ref, bound) for feats [N,3,M,32] and params [4257]. dL/do of a masked channel is autograd's g 1.002 (1 - s) s
    (1 - s rounds unless s >= 1/2; 4 roundings). dL/dh: two 16-FMA chains, their sum and one FMA (18); dL/da1 multiplies by
    sigmoid(a1) = z / (z + 1) (expf, add, divide: 4) (23); dL/dx: a 32-FMA chain per lane, the lane pair's sum, the rounded
    1/3 and its product (35). Parameter gradients: `chain` (decoder_bwd_chain) sequential roundings plus one for the product.
    fault 'deriv_from_y' forms s from the forward's output y = 1.002 s - 0.001 as (y + 0.001) / 1.002, in fp32."""
    w1, w2 = np.asarray(w1, np.float64), np.asarray(w2, np.float64)
    P = pre.shape[0]
    x, xa = _mean_planes(feats)
    ex = gam(4) * xa
    pre = np.asarray(pre, np.float64)
    h, dsp = _softplus(pre)
    eh = 4 * U * h
    go = np.zeros((P, 33))
    if g_sigma is not None:
        go[:, 0] = np.asarray(g_sigma, np.float64).reshape(P)
    on = ((mask >> np.arange(32)) & 1).astype(bool)[None]
    if g_rgb is not None:
        g = np.asarray(g_rgb, np.float64).reshape(P, 32)
        s = np.asarray(sig, np.float64).reshape(P, 32) if mask else np.zeros((P, 32))
        if fault == 'deriv_from_y':
            y = _f32_fma(s, F1002, -F0001)
            s = ((y + np.float32(0.001)) * np.float32(1.0 / np.float32(1.002))).astype(np.float64)
        go[:, 1:] = np.where(on, g * F1002 * (1 - s) * s, g)
    ego = np.zeros_like(go)
    ego[:, 1:] = np.where(on, gam(4) * np.abs(go[:, 1:]), 0.0)
    ago = np.abs(go)
    gh = go @ w2
    egh = gam(18) * (ago @ np.abs(w2)) + ego @ np.abs(w2)
    ga = gh * dsp
    aga = (ago @ np.abs(w2)) * dsp
    ega = gam(23) * aga + (ego @ np.abs(w2)) * dsp
    gx = ga @ w1 / 3
    egx = (gam(35) * (aga @ np.abs(w1)) + ega @ np.abs(w1)) / 3
    N, _, M, C = feats.shape
    gf = np.broadcast_to(gx.reshape(N, 1, M, C), (N, 3, M, C))
    egf = np.broadcast_to(egx.reshape(N, 1, M, C), (N, 3, M, C))
    gc = gam(chain + 1)
    gp = [(ga.T @ x).reshape(-1), ga.sum(0), (go.T @ h).reshape(-1), go.sum(0)]
    ep = [(gc * (aga.T @ xa) + ega.T @ xa + aga.T @ ex).reshape(-1), gc * aga.sum(0) + ega.sum(0),
          (gc * (ago.T @ h) + ego.T @ h + ago.T @ eh).reshape(-1), gc * ago.sum(0) + ego.sum(0)]
    return dict(feats=(gf, egf), params=(np.concatenate(gp), np.concatenate(ep)))


def _march_fwd_bounds(z, s):
    """Per-interval quantities of the march and their bounds, for kernels that use the accurate expf / log1pf (the backward) or
    the MUFU approximations (the forward: E_EXP covers ex2.approx / lg2.approx). z, s [N,S] fp32 depths and raw densities."""
    z, s = np.asarray(z, np.float64), np.asarray(s, np.float64)
    delta = z[:, 1:] - z[:, :-1]
    edl = U * np.abs(delta)
    x = (s[:, :-1] + s[:, 1:]) / 2 - 1
    ex = gam(2) * (np.abs(s[:, :-1]) + np.abs(s[:, 1:])) / 2 + U * np.abs(x)
    sp, sg = _softplus(x)
    esp = sg * ex + 3 * U * sp
    pd = sp * delta
    epd = esp * np.abs(delta) + sp * edl + U * np.abs(pd)
    e = np.exp(-pd)
    return dict(delta=delta, edl=edl, x=x, ex=ex, sp=sp, sg=sg, pd=pd, epd=epd, e=e)


def ray_march_bwd_model(colors, dens, depths, g_rgb, g_depth, g_w, rng, white_back, fault=None):
    """p3d_ray_march_bwd (warp_march_bwd, render_common.cuh) -> dict of (ref, bound) for colors [N,S,C] and densities [N,S].
    The transmittance T_i = prod_{k<i} a_k, a_k = 1 - alpha_k + 1e-10, is a product in any association (the lanes' scan):
    gamma(i + 6) plus the sum of the factors' relative bounds. G . c_j: 8 FMAs per lane and a 5-level warp sum (13). The
    exclusive suffix sum sum_{k>i} g_k w_k: up to K FMAs per lane, a 5-level scan and K more (2K + 6). Faults: 'no_eps' (the
    1e-10 missing from a_k), 'suffix_incl' (the suffix sum includes k = i), 'no_gate' (the depth term ignores [dlo, dhi])."""
    c = np.asarray(colors, np.float64)
    N, S, C = c.shape
    z = np.asarray(depths, np.float64)
    q = _march_fwd_bounds(depths, dens)
    e, delta = q['e'], q['delta']
    ee = e * (q['epd'] + 2 * U)
    alpha = 1 - e
    ealpha = ee + U * alpha
    eps = 0.0 if fault == 'no_eps' else F1E10
    a = 1 - alpha + eps
    ea = ealpha + 2 * U * a
    idx = np.arange(S - 1)[None]
    T = np.concatenate([np.ones((N, 1)), np.cumprod(a, 1)[:, :-1]], 1)
    rel = np.concatenate([np.zeros((N, 1)), np.cumsum(ea / a, 1)[:, :-1]], 1)
    eT = T * (gam(idx + 6) + rel)
    w = alpha * T
    ew = ealpha * T + alpha * eT + U * w
    G = 2 * np.asarray(g_rgb, np.float64)
    aG = np.abs(G)
    dot = np.einsum('nc,nsc->ns', G, c)
    adot = np.einsum('nc,nsc->ns', aG, np.abs(c))
    g = 0.5 * (dot[:, :-1] + dot[:, 1:])
    gabs = 0.5 * (adot[:, :-1] + adot[:, 1:])
    if white_back:
        g = g - G.sum(1)[:, None]
        gabs = gabs + aG.sum(1)[:, None]
    if g_w is not None:
        gwx = np.asarray(g_w, np.float64).reshape(N, S - 1)
        g, gabs = g + gwx, gabs + np.abs(gwx)
    eg = gam(17) * gabs
    if g_depth is not None:
        gd = np.asarray(g_depth, np.float64).reshape(N)
        zmid = (z[:, :-1] + z[:, 1:]) / 2
        sw = w.sum(1)
        esw = ew.sum(1) + gam(S + 5) * sw
        with np.errstate(all='ignore'):
            draw = (w * zmid).sum(1) / sw
            edraw = (((ew * np.abs(zmid - draw[:, None])).sum(1) + gam(S + 6) * (w * np.abs(zmid)).sum(1)) / sw
                     + U * np.abs(draw))
            ok = (gd != 0) & np.isfinite(draw)
            if fault != 'no_gate':
                ok &= (draw >= rng[0]) & (draw <= rng[1])
            gdw = gd / sw
            egdw = np.abs(gd) * esw / sw ** 2 + U * np.abs(gdw)
            dz = zmid - draw[:, None]
            term = gdw[:, None] * dz
            eterm = (np.abs(gdw)[:, None] * (U * np.abs(zmid) * 2 + edraw[:, None] + U * np.abs(dz)) + egdw[:, None] * np.abs(dz)
                     + U * np.abs(term))
        g = np.where(ok[:, None], g + term, g)
        eg = np.where(ok[:, None], eg + eterm + U * np.abs(g), eg)
    gw = g * w
    agw = np.abs(g) * w
    egw = eg * w + np.abs(g) * ew
    K = _ceil(S - 1, 32)
    rcum = np.cumsum(gw[:, ::-1], 1)[:, ::-1]
    acum = np.cumsum(agw[:, ::-1], 1)[:, ::-1]
    ecum = np.cumsum(egw[:, ::-1], 1)[:, ::-1]
    zero = np.zeros((N, 1))
    if fault == 'suffix_incl':
        run, arun, erun = rcum, acum, ecum
    else:
        run, arun, erun = (np.concatenate([v[:, 1:], zero], 1) for v in (rcum, acum, ecum))
    erun = gam(2 * K + 6) * arun + erun
    galpha = g * T - run / a
    egalpha = eg * T + np.abs(g) * eT + (erun + np.abs(run) * ea / a) / a + gam(3) * (np.abs(g) * T + np.abs(run) / a)
    sg = q['sg']
    esg = sg * (1 - sg) * q['ex'] + 3 * U * sg
    gsm = galpha * e * delta * sg
    egsm = (egalpha * e * np.abs(delta) * sg + np.abs(galpha) * (ee * np.abs(delta) * sg + e * q['edl'] * sg + e * np.abs(delta) * esg)
            + gam(3) * np.abs(gsm))
    pad = lambda v: np.concatenate([zero, v, zero], 1)                       # noqa: E731
    gsp, egsp = pad(gsm), pad(egsm)
    gden = 0.5 * (gsp[:, :-1] + gsp[:, 1:])
    egden = 0.5 * (egsp[:, :-1] + egsp[:, 1:]) + U * np.abs(gden)
    wp, ewp = pad(w), pad(ew)
    coef = 0.5 * (wp[:, :-1] + wp[:, 1:])
    ecoef = 0.5 * (ewp[:, :-1] + ewp[:, 1:])
    gcol = coef[..., None] * G[:, None, :]
    egcol = ecoef[..., None] * aG[:, None, :] + gam(2) * np.abs(gcol)
    return dict(colors=(gcol, egcol), densities=(gden, egden))


def ray_march_fwd_model(colors, dens, depths, white_back):
    """p3d_ray_march (warp_march: ex2.approx / lg2.approx softplus and __expf) -> dict of (ref, bound) for rgb [N,C],
    depth [N], weights [N,S-1]. The march and its bounds are test_gpu_render_model._march's (the fused SIMT renderer runs the
    same warp_march); the colour sum is a sequential FMA chain over the intervals; the launch clamps every depth to its own
    [min, max] sample depth, and a zero weight sum (NaN) comes out as the largest depth."""
    from test_gpu_render_model import _march, depth_reference
    z = torch.from_numpy(np.asarray(depths, np.float64))
    s = torch.from_numpy(np.asarray(dens, np.float64))
    c = torch.from_numpy(np.asarray(colors, np.float64))
    m = _march(z, s, torch.zeros_like(s), c, torch.zeros_like(c))
    rgb, ergb = m['rgb'], m['ergb']
    if white_back:
        rgb = rgb + 1 - m['ws'][:, None]
        ergb = ergb + m['ews'][:, None] + 2 * U * (rgb.abs() + 1)
    rgb = rgb * 2 - 1
    ergb = 2 * ergb + U * rgb.abs()
    lo, hi = float(np.min(depths)), float(np.max(depths))
    dep, edep = depth_reference(m, lo, hi)
    edep = edep + 2 * U * dep.abs()
    return dict(rgb=(rgb.numpy(), ergb.numpy()), depth=(dep.numpy(), edep.numpy()), weights=(m['w'].numpy(), m['ew'].numpy()))


def out_of_bound(got, ref, bound):
    """Boolean mask of the elements outside |got - ref| <= bound + FLOOR (NaN anywhere counts as outside; equal infinities
    pass)."""
    got = np.asarray(got, np.float64).reshape(np.shape(ref))
    with np.errstate(invalid='ignore'):
        err = np.abs(got - ref)
        err = np.where(got == ref, 0.0, err)
        return ~(err <= np.asarray(bound) + FLOOR)


def worst(got, ref, bound):
    got = np.asarray(got, np.float64).reshape(np.shape(ref))
    with np.errstate(all='ignore'):
        r = np.where(got == ref, 0.0, np.abs(got - ref) / (np.asarray(bound) + FLOOR))
    r = np.nan_to_num(r, nan=np.inf)
    return float(r.max()) if r.size else 0.0


# ---------------------------------------------------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------------------------------------------------
def decoder_params(rng, kind='random'):
    """Effective parameters (gains applied) as FullyConnectedLayer forms them, with biases that exercise the edges:
    'random'; 'logits' (small W2, so every point's 32 colour logits sit near b2, which sweeps [-25, 25]); 'pre20' (hidden
    pre-activations at and around the softplus threshold of 20)."""
    f = np.float32
    w1 = (rng.standard_normal((64, 32)) / np.sqrt(32)).astype(f)
    b1 = rng.standard_normal(64).astype(f)
    w2 = (rng.standard_normal((33, 64)) / 8).astype(f)
    b2 = rng.standard_normal(33).astype(f)
    if kind == 'logits':
        w2 = (rng.standard_normal((33, 64)) * 1e-3).astype(f)
        b2 = np.concatenate([[0.5], np.linspace(-25, 25, 32)]).astype(f)
    elif kind == 'pre20':
        w1 = (w1 * 1e-6).astype(f)
        b1 = (20 + np.repeat(np.array([-2, -1, 0, 1, 2], np.float64), 13)[:64] * 2 ** -19).astype(f)
    return w1, b1, w2, b2


def special_coords(rng, n, H, W):
    """Normalised coordinates on texel centres and edges, at +-1, just inside and outside the (-1, W) / (-1, H) test, NaN,
    plus uniform ones. The kernel's grid coordinate is ((g + 1) W - 1) / 2: centre j at g = (2 j + 1) / W - 1."""
    f = np.float32
    vals = [-1.0, 1.0, 0.0, np.nan]
    for L in {H, W}:
        vals += [(2 * j + 1) / L - 1 for j in range(min(L, 4))] + [2 * j / L - 1 for j in range(min(L, 4) + 1)]
        vals += [-1 - 1 / L, 1 + 1 / L]                          # ix = -1 and ix = W exactly: outside
    base = np.array(vals, np.float64)
    near = np.concatenate([np.nextafter(base.astype(f), f(np.inf)), np.nextafter(base.astype(f), f(-np.inf))])
    pool = np.concatenate([base.astype(f), near, rng.uniform(-1.2, 1.2, 64).astype(f)])
    return pool[rng.integers(0, pool.size, (n, 3))].astype(f)


def march_inputs(rng, N, S, Cc, special=False):
    """Depths increasing along each ray, raw densities and colours. `special`: rays with an opaque interval (alpha -> 1, so
    a = 1e-10), transmittance that underflows to 0, and all-zero weights (softplus of very negative densities)."""
    f = np.float32
    z = np.sort(rng.uniform(2.0, 3.5, (N, S)), 1).astype(f)
    s = rng.normal(0, 4, (N, S)).astype(f)
    c = rng.normal(0, 1, (N, S, Cc)).astype(f)
    if special and N >= 4:
        s[0::4, S // 2:] = 400.0                          # opaque from the middle on
        s[1::4] = 90.0                                    # transmittance underflows
        s[2::4] = -200.0                                  # zero weights
    return z, s, c


def nan_buf(n, dtype=torch.float32, device='cuda'):
    if dtype == torch.int32:
        return torch.full((n + PAD,), -123456, dtype=dtype, device=device)
    return torch.full((n + PAD,), math.nan, dtype=dtype, device=device)


def untouched(buf, n):
    t = buf[n:]
    return bool(torch.isnan(t).all()) if t.dtype.is_floating_point else bool((t == -123456).all())


# ---------------------------------------------------------------------------------------------------------------------
# CPU tests: the models reproduce the oracle, the bounds reject planted faults, the grid mirrors reach the edges
# ---------------------------------------------------------------------------------------------------------------------
def _oracle_dec(w1, b1, w2, b2):
    """Oracle decoder dict whose effective parameters equal (w1, b1, w2, b2): lr_mul 1, weight gain 1/sqrt(fan_in)."""
    return dict(kind='OSGDecoder', lr_mul=1.0, nets=[dict(w1=w1 * np.float32(np.sqrt(32)), b1=b1, w2=w2 * np.float32(8.0), b2=b2)])


def test_models_reproduce_the_oracle():
    rng = np.random.default_rng(0)
    # tri-plane lookup and its scatter
    B, M, H, W = 2, 300, 9, 13
    planes = rng.standard_normal((B, 3, H, W, 32)).astype(np.float32)
    coords = special_coords(rng, B * M, H, W).reshape(B, M, 3)
    ref, bd = sample_planes_model(planes, coords, 1.0)
    want = O.renderer.sample_from_planes(planes.transpose(0, 1, 4, 2, 3), coords, 2.0)
    assert not out_of_bound(want, ref, bd).any()
    g = rng.standard_normal((B, 3, M, 32)).astype(np.float32)
    ref, bd = sample_planes_bwd_model(g, coords, 1.0, H, W)
    want = O.renderer.sample_from_planes_backward(g, (B, 3, 32, H, W), coords, 2.0).transpose(0, 1, 3, 4, 2)
    assert np.abs(want - ref).max() <= 4 * U * np.abs(ref).max()         # the oracle rounds its float64 scatter once
    # decoder forward and backward (the oracle's backward takes dL/d(raw params); with lr_mul 1 the biases are the same)
    w1, b1, w2, b2 = decoder_params(rng)
    feats = rng.standard_normal((2, 3, 50, 32)).astype(np.float32)
    dec = _oracle_dec(w1, b1, w2, b2)
    rgb, sigma = O.renderer.decoder_forward(dec, feats)
    m = decoder_fwd_model(feats, w1, b1, w2, b2, 0xFFFFFFFF)
    assert not out_of_bound(rgb.reshape(-1, 32), *m['rgb']).any()
    assert not out_of_bound(sigma.reshape(-1), *m['sigma']).any()
    g_rgb = rng.standard_normal((2, 50, 32)).astype(np.float32)
    g_sig = rng.standard_normal((2, 50, 1)).astype(np.float32)
    gf, gp = O.renderer.decoder_backward(dec, feats, g_rgb, g_sig)
    x, _ = _mean_planes(feats)
    pre = (x @ w1.astype(np.float64).T + b1).astype(np.float32)
    h, _ = _softplus(pre.astype(np.float64))
    sig = _sigmoid(h @ w2.astype(np.float64).T[:, 1:] + b2[1:].astype(np.float64))
    mb = decoder_bwd_model(feats, w1, b1, w2, b2, 0xFFFFFFFF, pre, sig, g_rgb, g_sig, chain=100)
    # the oracle differentiates exact float64 activations, the model the fp32-rounded pre-activations: agree to ~1e-6
    assert np.abs(gf - mb['feats'][0]).max() <= 1e-5 * np.abs(gf).max()
    gw1 = gp[0]['w1'] * np.sqrt(32)                           # dL/d(raw w1) = dL/d(effective w1) / sqrt(32)
    assert np.abs(gw1.reshape(-1) - mb['params'][0][:2048]).max() <= 1e-5 * np.abs(gw1).max()
    # ray march forward and backward
    z, s, c = march_inputs(rng, 16, 20, 5, special=True)
    mf = ray_march_fwd_model(c, s, z, white_back=True)
    orgb, odep, ow = O.renderer.ray_march(c[None], s[None, ..., None], z[None, ..., None], white_back=True)
    assert not out_of_bound(ow.reshape(16, -1), *mf['weights']).any()
    assert not out_of_bound(orgb.reshape(16, -1), *mf['rgb']).any()
    assert not out_of_bound(odep.reshape(-1), *mf['depth']).any()
    grgb = rng.standard_normal((16, 5)).astype(np.float32)
    gdep = rng.standard_normal(16).astype(np.float32)
    gw = rng.standard_normal((16, 19)).astype(np.float32)
    rngz = (float(z.min()), float(z.max()))
    mb = ray_march_bwd_model(c, s, z, grgb, gdep, gw, rngz, True)
    oc, od = O.renderer.ray_march_backward(c[None], s[None, ..., None], z[None, ..., None], grgb[None], gdep[None, :, None],
                                           gw[None, ..., None], white_back=True, clamp_range=rngz)
    assert not out_of_bound(oc[0], *mb['colors']).any()
    ref, bd = mb['densities']
    assert not out_of_bound(od[0, ..., 0], ref, bd + 1e-30).any()        # the oracle clips the sigmoid's input to +-80


def _fixture_coarse_weights(case):
    """The staged chain's models on a committed reference render: the coarse samples of renderer_<case>.npz through
    sample_planes_model, the sigma net's decoder_fwd_model and the march. The features' bound is carried into sigma through
    |W2| |W1| (softplus is 1-Lipschitz) and the march propagates sigma's bound (test_gpu_render_model._march). Returns the
    fixture's coarse weights (the reference's fp32 pipeline) and the model's (weights, bound)."""
    from conftest import load_golden
    from test_gpu_render_model import EPS_OUT, _march
    from test_oracle_golden import oracle_decoder, render_opts
    g = load_golden('renderer_' + case)
    opts = render_opts(g)
    b, m = g['ray_origins'].shape[:2]
    z = O.renderer.sample_stratified(b, m, opts['ray_start'], opts['ray_end'], opts['depth_resolution'], g['jitter'])
    z = np.asarray(z, np.float32).reshape(b, m, -1)
    o, d = g['ray_origins'].astype(np.float32), g['ray_dirs'].astype(np.float32)
    coords = (o[:, :, None, :] + z[..., None] * d[:, :, None, :]).reshape(b, -1, 3)        # renderer.py:121 in fp32
    feats, efeat = sample_planes_model(g['planes'].transpose(0, 1, 3, 4, 2), coords, np.float32(2.0 / opts['box_warp']))
    net = oracle_decoder(g)['nets'][-1]                                                      # the sigma net
    w1 = (net['w1'] * np.float32(1 / np.sqrt(32))).astype(np.float32)                       # FullyConnectedLayer's gains
    w2 = (net['w2'] * np.float32(1 / 8)).astype(np.float32)
    mm = decoder_fwd_model(feats.astype(np.float32), w1, net['b1'], w2, net['b2'], 0)
    ex = ((efeat[:, 0] + efeat[:, 1] + efeat[:, 2]) / 3).reshape(-1, 32)
    es = mm['sigma'][1] + (ex @ np.abs(w1.astype(np.float64)).T) @ np.abs(w2[0].astype(np.float64)) + 2 * U * np.abs(mm['sigma'][0])
    n = b * m
    mr = _march(torch.from_numpy(z.reshape(n, -1).astype(np.float64)), torch.from_numpy(mm['sigma'][0].reshape(n, -1)),
                torch.from_numpy(es.reshape(n, -1)))
    w, ew = mr['w'].numpy(), mr['ew'].numpy()
    return g['weights_coarse'].reshape(n, -1), w, ew + EPS_OUT * np.abs(w)


@pytest.mark.parametrize('case', ['seg', 'seg48', 'car', 'rgb_only'])
def test_models_reproduce_the_reference_fixtures(case):
    """The committed reference renders (tests/golden/renderer_*.npz, fp32 torch) lie within the chained models' bounds."""
    want, w, bound = _fixture_coarse_weights(case)
    assert not out_of_bound(want, w, bound).any(), worst(want, w, bound)


def _fault_fraction(clean, faulty):
    """Fraction of elements where the faulted model leaves the clean model's bound."""
    (ref, bd), (bad, _) = clean, faulty
    return float(out_of_bound(bad, ref, bd).mean())


def test_bounds_reject_planted_faults():
    rng = np.random.default_rng(1)
    report = {}
    B, M, H, W = 1, 400, 7, 11
    planes = rng.standard_normal((B, 3, H, W, 32)).astype(np.float32)
    coords = rng.uniform(-1, 1, (B, M, 3)).astype(np.float32)
    clean = sample_planes_model(planes, coords, 1.0)
    g = rng.standard_normal((B, 3, M, 32)).astype(np.float32)
    cleanb = sample_planes_bwd_model(g, coords, 1.0, H, W)
    for fault in ('drop_tap', 'swap_tap'):
        report[f'planes {fault}'] = _fault_fraction(clean, sample_planes_model(planes, coords, 1.0, fault))
        report[f'planes_bwd {fault}'] = _fault_fraction(cleanb, sample_planes_bwd_model(g, coords, 1.0, H, W, fault))
    w1, b1, w2, b2 = decoder_params(rng)
    feats = rng.standard_normal((1, 3, 300, 32)).astype(np.float32)
    clean = decoder_fwd_model(feats, w1, b1, w2, b2, 0xFFFFFFFF)
    report['decoder 1/3 missing'] = _fault_fraction(clean['rgb'], decoder_fwd_model(feats, w1, b1, w2, b2, 0xFFFFFFFF, 'no_third')['rgb'])
    report['decoder mask bit'] = _fault_fraction(clean['rgb'], decoder_fwd_model(feats, w1, b1, w2, b2, 0xFFFFFFFF, 'mask_bit')['rgb'])
    # the sigmoid derivative from y instead of s, on saturated logits: dL/db2 of each colour channel
    w1, b1, w2, b2 = decoder_params(rng, 'logits')
    m = decoder_fwd_model(feats, w1, b1, w2, b2, 0xFFFFFFFF)
    pre = m['pre'][0].astype(np.float32)
    sig = m['sig'][0].astype(np.float32)
    g_rgb = rng.standard_normal((1, 300, 32)).astype(np.float32)
    args = (feats, w1, b1, w2, b2, 0xFFFFFFFF, pre, sig, g_rgb, None)
    cb = decoder_bwd_model(*args, chain=decoder_bwd_chain(300, 132))
    fb = decoder_bwd_model(*args, chain=decoder_bwd_chain(300, 132), fault='deriv_from_y')
    report['decoder_bwd deriv from y (db2)'] = _fault_fraction((cb['params'][0][-33:], cb['params'][1][-33:]), (fb['params'][0][-33:], None))
    # march backward
    z, s, c = march_inputs(rng, 64, 40, 4, special=True)
    grgb = rng.standard_normal((64, 4)).astype(np.float32)
    gdep = rng.standard_normal(64).astype(np.float32)
    rngz = (float(np.quantile(z, 0.3)), float(np.quantile(z, 0.7)))          # a narrow clamp range: the gate matters
    clean = ray_march_bwd_model(c, s, z, grgb, gdep, None, rngz, False)
    for fault in ('no_eps', 'suffix_incl', 'no_gate'):
        with np.errstate(all='ignore'):                     # without the 1e-10, opaque intervals divide by zero
            bad = ray_march_bwd_model(c, s, z, grgb, gdep, None, rngz, False, fault)
        report[f'march_bwd {fault}'] = _fault_fraction(clean['densities'], bad['densities'])
    print('\nfraction of elements out of bound per planted fault:')
    for k, v in report.items():
        print(f'  {k:34s} {v:.3f}')
    for k, v in report.items():
        assert v > 0, k
    # the taps, the mean and the mask each move a large share of the elements; the others only the elements they concern
    assert min(report['planes drop_tap'], report['planes swap_tap'], report['decoder 1/3 missing']) > 0.3
    assert report['decoder_bwd deriv from y (db2)'] > 0.1


def test_grid_mirrors_reach_the_sweep_edges():
    """For any SM count, the sweep's shapes hit the grid caps and the per-CTA tile counts they are meant to."""
    for sms in (132, 114, 78):
        ctas = 3 * sms
        assert grid_decoder_bwd(ctas * 64 - 65, sms) == ctas - 1     # one tile per CTA below the cap, a ragged tile at it
        assert grid_decoder_bwd(ctas * 64 - 1, sms) == ctas and grid_decoder_bwd(ctas * 64 + 1, sms) == ctas
        P = 3 * ctas * 64 + 17                          # several tiles per CTA, a ragged last tile
        assert grid_decoder_bwd(P, sms) == ctas and _ceil(P, 64) > 3 * ctas and P % 64
        cap = 8 * sms * 128
        assert grid_decoder_fwd(cap, sms) == 8 * sms and grid_decoder_fwd(cap + 1, sms) == 8 * sms
        assert grid_decoder_fwd(cap - 128, sms) < 8 * sms
        warps = 16 * sms * 8
        assert grid_sample_planes(warps, sms) == 16 * sms and grid_sample_planes(warps - 32, sms) < 16 * sms
        assert grid_sample_planes_bwd(warps + 1, sms) == 16 * sms and grid_sample_planes_bwd(warps - 8, sms) < 16 * sms
        n = 16 * sms * 4
        assert grid_ray_march_bwd(n - 1, sms) == 16 * sms and grid_ray_march_bwd(n + 1, sms) == 16 * sms
        assert grid_ray_march_bwd(n - 4, sms) < 16 * sms
        assert grid_ray_march(2 * 8 * sms * 4, sms) == 8 * sms
    # per-lane interval counts K = ceil((S - 1) / 32) of the sweep: 1, 1, 1, 2, 2, 8, 8
    assert [_ceil(S - 1, 32) for S in (2, 3, 33, 34, 65, 256, 257)] == [1, 1, 1, 2, 2, 8, 8]
    assert importance_max_S() == 768


# ---------------------------------------------------------------------------------------------------------------------
# GPU sweep
# ---------------------------------------------------------------------------------------------------------------------
def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


WORST = {}


@pytest.fixture(scope='module', autouse=True)
def _worst_report():
    """Prints the worst err / bound seen per output by the tests of this module that ran."""
    yield
    if WORST:
        print('\nworst err / bound per output:')
        for k in sorted(WORST):
            print(f'  {k:28s} {WORST[k]:.3g}')


def _check(name, got_buf, n, ref, bound):
    """got_buf: the NaN-prefilled flat buffer the launch wrote; n its own elements."""
    assert untouched(got_buf, n), f'{name}: the launch wrote past its {n} elements'
    got = got_buf[:n].cpu().numpy().astype(np.float64)
    bad = out_of_bound(got, ref, bound)
    WORST[name] = max(WORST.get(name, 0.0), worst(got, ref, bound))
    assert not bad.any(), f'{name}: {int(bad.sum())} of {bad.size} elements out of bound (worst err/bound {worst(got, ref, bound):.3g})'


def run_decoder(feats, prm, mask, g_rgb, g_sigma, check_fwd=True):
    from pix2pix3d_b200 import native
    N, _, M, _ = feats.shape
    P = N * M
    f = _t(feats)
    w = [_t(t) for t in prm]
    bufs = dict(rgb=nan_buf(P * 32), sigma=nan_buf(P), pre=nan_buf(P * 64), sig=nan_buf(P * 32))
    r = native.decoder_mlp_fwd(f, *w, mask, want_saved=True, out=bufs)
    plain = native.decoder_mlp_fwd(f, *w, mask)
    assert torch.equal(plain['rgb'], r['rgb']) and torch.equal(plain['sigma'], r['sigma']), 'rgb / sigma depend on the saved outputs'
    if check_fwd:
        m = decoder_fwd_model(feats, *prm, mask)
        _check('decoder_fwd rgb', bufs['rgb'], P * 32, *m['rgb'])
        _check('decoder_fwd sigma', bufs['sigma'], P, *m['sigma'])
        _check('decoder_fwd pre', bufs['pre'], P * 64, *m['pre'])
        if mask:
            _check('decoder_fwd sig', bufs['sig'], P * 32, *m['sig'])
    pre = r['pre'].cpu().numpy()
    sig = r['sig'].cpu().numpy() if mask else None
    gb = dict(feats=nan_buf(P * 96), params=nan_buf(4257))
    gr = None if g_rgb is None else _t(g_rgb)
    gs = None if g_sigma is None else _t(g_sigma)
    out = native.decoder_mlp_bwd(f, *w, mask, r['pre'], r.get('sig'), gr, gs, out=gb)
    again = native.decoder_mlp_bwd(f, *w, mask, r['pre'], r.get('sig'), gr, gs)
    assert torch.equal(out['feats'], again['feats']) and torch.equal(out['params'], again['params']), 'not deterministic'
    mb = decoder_bwd_model(feats, *prm, mask, pre, sig, g_rgb, g_sigma, chain=decoder_bwd_chain(P, _sms()))
    _check('decoder_bwd feats', gb['feats'], P * 96, *mb['feats'])
    _check('decoder_bwd params', gb['params'], 4257, *mb['params'])


def _dec_case(P, seed, kind='random', mask=0xFFFFFFFF, rgb=True, sigma=True, N=1):
    rng = np.random.default_rng(seed)
    M = _ceil(P, N)
    feats = (rng.standard_normal((N, 3, M, 32)) * 1.5).astype(np.float32)
    prm = decoder_params(rng, kind)
    g_rgb = rng.standard_normal((N, M, 32)).astype(np.float32) if rgb else None
    g_sig = rng.standard_normal((N, M, 1)).astype(np.float32) if sigma else None
    run_decoder(feats, prm, mask, g_rgb, g_sig)


MASK6 = (1 << 0) | (1 << 7) | (1 << 13) | (1 << 20) | (1 << 24) | (1 << 31)       # 6 of 32 channels


@gpu
@pytest.mark.parametrize('P', [1, 63, 64, 65])
def test_decoder_small_point_counts(P):
    _dec_case(P, P)


@gpu
@pytest.mark.parametrize('edge', ['ctas*64-1', 'ctas*64+1', 'tiles>ctas,ragged'])
def test_decoder_bwd_grid_edges(edge):
    ctas = 3 * _sms()
    P = {'ctas*64-1': ctas * 64 - 1, 'ctas*64+1': ctas * 64 + 1, 'tiles>ctas,ragged': 3 * ctas * 64 + 17}[edge]
    _dec_case(P, 7, N=3)


@gpu
@pytest.mark.parametrize('case', ['g_rgb=None', 'g_sigma=None', 'mask=0', 'mask=6of32'])
def test_decoder_upstream_and_masks(case):
    kw = {'g_rgb=None': dict(rgb=False), 'g_sigma=None': dict(sigma=False), 'mask=0': dict(mask=0), 'mask=6of32': dict(mask=MASK6)}[case]
    _dec_case(1000, 3, **kw)


@gpu
def test_decoder_softplus_threshold():
    _dec_case(2000, 4, kind='pre20')


@gpu
def test_decoder_saturated_sigmoid():
    """Colour logits swept over [-25, 25]: dL/do = g 1.002 (1 - s) s must be autograd's, element for element (it reaches the
    parameter gradients directly through dL/db2 and dL/dW2)."""
    _dec_case(4000, 5, kind='logits', sigma=False)


@gpu
def test_decoder_fwd_grid_cap():
    cap = 8 * _sms() * 128
    for P in (cap - 1, cap + 1):
        rng = np.random.default_rng(P)
        feats = rng.standard_normal((1, 3, P, 32)).astype(np.float32)
        prm = decoder_params(rng)
        from pix2pix3d_b200 import native
        f, w = _t(feats), [_t(t) for t in prm]
        bufs = dict(rgb=nan_buf(P * 32), sigma=nan_buf(P), pre=nan_buf(P * 64), sig=nan_buf(P * 32))
        r = native.decoder_mlp_fwd(f, *w, MASK6, want_saved=True, out=bufs)
        plain = native.decoder_mlp_fwd(f, *w, MASK6)
        assert torch.equal(plain['rgb'], r['rgb']) and torch.equal(plain['sigma'], r['sigma'])
        m = decoder_fwd_model(feats, *prm, MASK6)
        for k, n in (('rgb', P * 32), ('sigma', P), ('pre', P * 64), ('sig', P * 32)):
            _check(f'decoder_fwd {k}', bufs[k], n, *m[k])


def run_planes(planes, coords, cs):
    from pix2pix3d_b200 import native
    B, _, H, W, C = planes.shape
    M = coords.shape[1]
    n = B * 3 * M * C
    buf = nan_buf(n)
    native.sample_from_planes(_t(planes), _t(coords), 2.0 / cs, out=buf)
    _check('sample_from_planes', buf, n, *sample_planes_model(planes, coords, cs))
    g = np.random.default_rng(M).standard_normal((B, 3, M, C)).astype(np.float32)
    nb = B * 3 * H * W * C
    gbuf = nan_buf(nb)
    native.sample_from_planes_bwd(_t(g), _t(coords), 2.0 / cs, H, W, out=gbuf)
    _check('sample_from_planes_bwd', gbuf, nb, *sample_planes_bwd_model(g, coords, cs, H, W))


@gpu
@pytest.mark.parametrize('HW', [(5, 7), (1, 1), (16, 16)])
def test_sample_planes_edges(HW):
    H, W = HW
    rng = np.random.default_rng(H * 100 + W)
    planes = rng.standard_normal((2, 3, H, W, 32)).astype(np.float32)
    coords = special_coords(rng, 2 * 700, H, W).reshape(2, 700, 3)
    run_planes(planes, coords, 1.0)


@gpu
def test_sample_planes_contention():
    """256^2 planes, points clustered on a few texels: hundreds of atomics per texel."""
    rng = np.random.default_rng(9)
    planes = rng.standard_normal((1, 3, 256, 256, 32)).astype(np.float32)
    centres = rng.uniform(-0.9, 0.9, (8, 3))
    coords = (centres[rng.integers(0, 8, 6000)] + rng.uniform(-2e-3, 2e-3, (6000, 3))).astype(np.float32)[None]
    run_planes(planes, coords, 1.0)


@gpu
@pytest.mark.parametrize('d', [-32, 1, 32])
def test_sample_planes_block_cap(d):
    points = 16 * _sms() * 8 + d                      # the cap of 16 CTAs per SM, x 8 warps per CTA, +- one warp's worth
    rng = np.random.default_rng(points)
    planes = rng.standard_normal((1, 3, 12, 10, 32)).astype(np.float32)
    coords = rng.uniform(-1.1, 1.1, (1, points, 3)).astype(np.float32)
    run_planes(planes, coords, 0.9)


def run_march_bwd(z, s, c, grgb, gdep, gw, rngz, white_back):
    from pix2pix3d_b200 import native
    N, S, Cc = c.shape
    bufs = dict(colors=nan_buf(N * S * Cc), densities=nan_buf(N * S))
    native.ray_march_bwd(_t(c)[None], _t(s)[None, ..., None], _t(z)[None, ..., None], _t(grgb)[None],
                         None if gdep is None else _t(gdep)[None, :, None], None if gw is None else _t(gw)[None, ..., None],
                         None if rngz is None else torch.tensor(rngz, dtype=torch.float32, device='cuda'), white_back, out=bufs)
    m = ray_march_bwd_model(c, s, z, grgb, gdep, gw, rngz, white_back)
    _check('ray_march_bwd colors', bufs['colors'], N * S * Cc, *m['colors'])
    _check('ray_march_bwd densities', bufs['densities'], N * S, *m['densities'])


def _march_bwd_case(N, S, Cc, seed, white_back=False, depth=True, weights=True, narrow=False):
    rng = np.random.default_rng(seed)
    z, s, c = march_inputs(rng, N, S, Cc, special=True)
    grgb = rng.standard_normal((N, Cc)).astype(np.float32)
    gdep = rng.standard_normal(N).astype(np.float32) if depth else None
    if gdep is not None:
        gdep[3::7] = 0                                      # rays whose depth gradient is exactly zero skip the term
    gw = rng.standard_normal((N, S - 1)).astype(np.float32) if weights else None
    rngz = None
    if depth:
        rngz = (float(np.quantile(z, 0.3)), float(np.quantile(z, 0.7))) if narrow else (float(z.min()), float(z.max()))
    run_march_bwd(z, s, c, grgb, gdep, gw, rngz, white_back)


@gpu
@pytest.mark.parametrize('S', [2, 3, 33, 34, 65, 256, 257])
def test_ray_march_bwd_interval_counts(S):
    _march_bwd_case(40, S, 3, S, white_back=S % 2 == 1)


@gpu
@pytest.mark.parametrize('Cc', [1, 31, 32, 33, 255, 256])
def test_ray_march_bwd_channel_counts(Cc):
    _march_bwd_case(24, 34, Cc, Cc, weights=Cc % 2 == 0)


@gpu
@pytest.mark.parametrize('d', [-1, 1])
def test_ray_march_bwd_grid_cap(d):
    _march_bwd_case(16 * _sms() * 4 + d, 34, 32, 100 + d)


@gpu
@pytest.mark.parametrize('case', ['narrow_gate', 'no_depth', 'white_back'])
def test_ray_march_bwd_terms(case):
    kw = {'narrow_gate': dict(narrow=True), 'no_depth': dict(depth=False, weights=False), 'white_back': dict(white_back=True)}[case]
    _march_bwd_case(300, 48, 7, 11, **kw)


@gpu
@pytest.mark.parametrize('S', [2, 3, 33, 34, 65, 256])
def test_ray_march_fwd(S):
    """Two rays per warp slot at the grid cap, so CTAs walk several rays; the launch's largest and smallest depths sit in the
    last and the first ray (different CTAs), and zero-weight rays come out at the largest depth."""
    from pix2pix3d_b200 import native
    N = 2 * 8 * _sms() * 4 + 3 if S <= 65 else 300
    rng = np.random.default_rng(S)
    z, s, c = march_inputs(rng, N, S, 5, special=True)
    z[0, 0] = 0.5
    z[-1, -1] = 9.0
    bufs = dict(rgb=nan_buf(N * 5), depth=nan_buf(N), weights=nan_buf(N * (S - 1)))
    native.ray_march(_t(c)[None], _t(s)[None, ..., None], _t(z)[None, ..., None], white_back=S % 2 == 0, out=bufs)
    m = ray_march_fwd_model(c, s, z, S % 2 == 0)
    _check('ray_march weights', bufs['weights'], N * (S - 1), *m['weights'])
    _check('ray_march rgb', bufs['rgb'], N * 5, *m['rgb'])
    _check('ray_march depth', bufs['depth'], N, *m['depth'])
    assert float(bufs['depth'][2]) == 9.0                   # a zero-weight ray: the launch's largest depth


@gpu
@pytest.mark.parametrize('S', [4, 'max'])
def test_sample_importance_bit_exact(S):
    from pix2pix3d_b200 import _lib, native
    S = importance_max_S() if S == 'max' else S
    rng = np.random.default_rng(S)
    N, Sf = 37, 40
    z = np.sort(rng.uniform(2, 3, (N, S)), 1).astype(np.float32)
    w = rng.exponential(1, (N, S - 1)).astype(np.float32)
    w[::5] = 0
    u = rng.uniform(0, 1, (N, Sf)).astype(np.float32)
    bufs = dict(samples=nan_buf(N * Sf), inds=nan_buf(N * Sf, torch.int32))
    native.sample_importance(_t(z), _t(w), _t(u), return_inds=True, out=bufs)
    want, dbg = O.renderer.sample_importance(z, w, u, return_debug=True)
    assert untouched(bufs['samples'], N * Sf) and untouched(bufs['inds'], N * Sf)
    assert np.array_equal(bufs['samples'][:N * Sf].cpu().numpy().reshape(N, Sf), want)
    assert np.array_equal(bufs['inds'][:N * Sf].cpu().numpy().reshape(N, Sf), dbg['inds'])
    if S == importance_max_S():
        S1 = S + 1
        z1, w1 = _t(np.sort(rng.uniform(2, 3, (1, S1)), 1).astype(np.float32)), _t(np.ones((1, S1 - 1), np.float32))
        out = torch.empty(1, 4, device='cuda')
        st = _lib.lib().p3d_sample_importance(_lib.ptr(z1), _lib.ptr(w1), _lib.ptr(_t(u[:1, :4])), 1, S1, 4, _lib.ptr(out), None,
                                              _lib.stream_ptr())
        assert st == -1                                       # P3D_UNSUPPORTED


# ---------------------------------------------------------------------------------------------------------------------
# Replays from a real training iteration
# ---------------------------------------------------------------------------------------------------------------------
def _np(t):
    return None if t is None else t.detach().float().cpu().numpy()


def _score(stats, name, got, ref, bound):
    bad = out_of_bound(got, ref, bound)
    st = stats.setdefault(name, dict(bad=0, elements=0, worst=0.0))
    st['bad'] += int(bad.sum())
    st['elements'] += int(bad.size)
    st['worst'] = max(st['worst'], worst(got, ref, bound))


def install_replay_checks(native, sms):
    """Wraps the native entry points of the staged chain so that every launch is checked, element by element (so every edge
    tile and ragged tail), against its model right after it ran. Returns (launch counts per kernel, per-output stats)."""
    counts, stats = {}, {}
    real = {k: getattr(native, k) for k in ('sample_from_planes', 'sample_from_planes_bwd', 'decoder_mlp_fwd', 'decoder_mlp_bwd',
                                             'ray_march', 'ray_march_bwd', 'sample_importance')}

    def count(k):
        counts[k] = counts.get(k, 0) + 1

    def sample_from_planes(planes_nhwc, coords, box_warp, out=None):
        r = real['sample_from_planes'](planes_nhwc, coords, box_warp, out=out)
        ref, bd = sample_planes_model(_np(planes_nhwc), _np(coords), np.float32(2.0 / float(box_warp)))
        _score(stats, 'sample_from_planes', _np(r), ref, bd)
        count('sample_from_planes')
        return r

    def sample_from_planes_bwd(grad_features, coords, box_warp, H, W, out=None):
        r = real['sample_from_planes_bwd'](grad_features, coords, box_warp, H, W, out=out)
        ref, bd = sample_planes_bwd_model(_np(grad_features), _np(coords), np.float32(2.0 / float(box_warp)), H, W)
        _score(stats, 'sample_from_planes_bwd', _np(r), ref, bd)
        count('sample_from_planes_bwd')
        return r

    def decoder_mlp_fwd(feats, w1, b1, w2, b2, mask, want_saved=False, out=None):
        r = real['decoder_mlp_fwd'](feats, w1, b1, w2, b2, mask, want_saved=want_saved, out=out)
        m = decoder_fwd_model(_np(feats), *(_np(t) for t in (w1, b1, w2, b2)), int(mask))
        for k in ('rgb', 'sigma', 'pre', 'sig'):
            if k in r:
                _score(stats, f'decoder_fwd {k}', _np(r[k]).reshape(m[k][0].shape), *m[k])
        count('decoder_mlp_fwd')
        return r

    def decoder_mlp_bwd(feats, w1, b1, w2, b2, mask, pre, sig, g_rgb, g_sigma, out=None):
        r = real['decoder_mlp_bwd'](feats, w1, b1, w2, b2, mask, pre, sig, g_rgb, g_sigma, out=out)
        f = _np(feats)
        P = f.shape[0] * f.shape[2]
        m = decoder_bwd_model(f, *(_np(t) for t in (w1, b1, w2, b2)), int(mask), _np(pre), _np(sig), _np(g_rgb), _np(g_sigma),
                              chain=decoder_bwd_chain(P, sms))
        _score(stats, 'decoder_bwd feats', _np(r['feats']), *m['feats'])
        _score(stats, 'decoder_bwd params', _np(r['params']), *m['params'])
        count('decoder_mlp_bwd')
        return r

    def ray_march(colors, densities, depths, white_back=False, out=None):
        rgb, depth, weights = real['ray_march'](colors, densities, depths, white_back, out=out)
        B, R, S, C = colors.shape
        m = ray_march_fwd_model(_np(colors).reshape(-1, S, C), _np(densities).reshape(-1, S), _np(depths).reshape(-1, S), white_back)
        _score(stats, 'ray_march rgb', _np(rgb).reshape(-1, C), *m['rgb'])
        _score(stats, 'ray_march depth', _np(depth).reshape(-1), *m['depth'])
        _score(stats, 'ray_march weights', _np(weights).reshape(-1, S - 1), *m['weights'])
        count('ray_march')
        return rgb, depth, weights

    def ray_march_bwd(colors, densities, depths, g_rgb, g_depth, g_weights, depth_range, white_back=False, out=None):
        g_col, g_den = real['ray_march_bwd'](colors, densities, depths, g_rgb, g_depth, g_weights, depth_range, white_back, out=out)
        B, R, S, C = colors.shape
        N = B * R
        rng = None if depth_range is None else tuple(float(v) for v in _np(depth_range).reshape(2))
        m = ray_march_bwd_model(_np(colors).reshape(N, S, C), _np(densities).reshape(N, S), _np(depths).reshape(N, S),
                                _np(g_rgb).reshape(N, C), None if g_depth is None else _np(g_depth).reshape(N),
                                None if g_weights is None else _np(g_weights).reshape(N, S - 1), rng, white_back)
        _score(stats, 'ray_march_bwd colors', _np(g_col).reshape(N, S, C), *m['colors'])
        _score(stats, 'ray_march_bwd densities', _np(g_den).reshape(N, S), *m['densities'])
        count('ray_march_bwd')
        return g_col, g_den

    def sample_importance(z_vals, weights, u, return_inds=False, out=None):
        r = real['sample_importance'](z_vals, weights, u, return_inds=return_inds, out=out)
        samples = r[0] if return_inds else r
        want = O.renderer.sample_importance(_np(z_vals), _np(weights), _np(u))
        st = stats.setdefault('sample_importance (bit-exact)', dict(bad=0, elements=0, worst=0.0))
        st['bad'] += int((_np(samples) != want).sum())
        st['elements'] += int(want.size)
        count('sample_importance')
        return r

    for k, fn in list(locals().items()):
        if k in real:
            setattr(native, k, fn)
    return counts, stats


REPLAY = """
import json, sys
sys.path[:0] = [{root!r}, {root!r} + '/baseline', {root!r} + '/tests', {root!r} + '/oracle']
import torch
import pix2pix3d_b200
pix2pix3d_b200.install(reference_root={ref!r})
from pix2pix3d_b200 import configs, native, train_step as ts
from pix2pix3d_b200.training.volumetric_rendering import renderer as rmod
import test_gpu_train_kernels as T
dev = torch.device('cuda')
counts, stats = T.install_replay_checks(native, torch.cuda.get_device_properties(0).multi_processor_count)
cfg = dict(ts.TINY_TRAIN)
st = ts.build(cfg, dev)
batch = ts.synthetic_batch(cfg, dev, 5)
torch.manual_seed(2)
st.batch_idx = 0                       # every phase runs, Greg included
ts.run_iteration(st, batch)
torch.cuda.synchronize()
phases = dict(iteration=dict(counts))
rmod.fused_grad = False                # one Gmain phase on the staged chain
b = cfg['batch_gpu']
gen_z = torch.randn([b, st.G.z_dim], generator=torch.Generator().manual_seed(1)).to(dev)
gen_c = configs.camera_labels(b, 1000).to(dev)
st.G.requires_grad_(True)
st.loss.accumulate_gradients(phase='Gmain', batch=batch, gen_z=gen_z, gen_c=gen_c, gain=1, cur_nimg=0)
st.G.requires_grad_(False)
torch.cuda.synchronize()
phases['total'] = dict(counts)
print('RESULT ' + json.dumps(dict(phases=phases, stats=stats)))
"""


@gpu
def test_replay_training_iteration():
    """One run_iteration of the tiny training recipe with batch_idx 0 (every phase, the Greg density regulariser's
    G.sample_mixed under autograd included), then one Gmain phase with `renderer.fused_grad = False` (the staged chain's
    ray_march[_bwd], sample_importance and the sigmoid decoder path at training shapes). Every launch of the wrapped entry
    points is checked against its model. Runs in a subprocess because install() re-maps module names."""
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
    print('\nlaunches checked per kernel:', r['phases'])
    for k, v in sorted(r['stats'].items()):
        print(f"  {k:30s} {v['elements']:>10d} elements, {v['bad']} out of bound, worst err/bound {v['worst']:.3g}")
    total = r['phases']['total']
    for k in ('sample_from_planes', 'sample_from_planes_bwd', 'decoder_mlp_fwd', 'decoder_mlp_bwd', 'ray_march', 'ray_march_bwd',
              'sample_importance'):
        assert total.get(k, 0) > 0, f'{k} never ran in the replay'
    for k in ('sample_from_planes', 'sample_from_planes_bwd', 'decoder_mlp_fwd', 'decoder_mlp_bwd'):
        assert r['phases']['iteration'].get(k, 0) > 0, f'{k} did not run in the training iteration (Greg)'
    bad = {k: v['bad'] for k, v in r['stats'].items() if v['bad']}
    assert not bad, bad
