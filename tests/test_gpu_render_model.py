"""The fused renderers on launches where CTAs walk many tiles, against a float64 model of each ray.

render_fwd_tc_kernel (render_tc.cu), render_fwd_tc_pairs_kernel (render_tc2.cu) and render_fwd_kernel (render.cu) launch
min(SMs, work) CTAs (the SIMT kernel up to two per SM). Each CTA walks its tiles (ray pairs) with `tile += gridDim.x`, reusing
its shared ray buffers, partial sums and flags, and the last CTA to finish clamps every depth to the launch's [min, max] sample
depth (ray_marcher.py:49-50). `model()` restates one launch in float64 from the arguments of native.render_fwd, and every output
element is held to

    |got - ref| <= EPS_OUT * |ref| + tol

where `tol` is propagated per sample and per ray from the same model on absolute values (the constants below). Importance
sampling is discontinuous, so the model checks the kernel's choices instead of re-deriving them: the kernel's coarse weights
must lie within the bound of the model's, they must reproduce its fine depths and indices bit for bit through the fp32 oracle
(O.renderer.sample_importance), and its merge permutation must be the stable argsort of the merged depths. The model then
marches the merged samples in float64.

Sample positions and bilinear tap weights are formed with the kernels' own fp32 operations (they are the interpolation's
inputs, one rounding each, as in the reference); every product and sum after them is float64.
"""
import math

import numpy as np
import pytest
import torch

import p3d_oracle as O
from conftest import load_golden
from test_oracle_golden import RENDER_CASES, render_opts

gpu = pytest.mark.gpu

U32 = 2.0 ** -24
EPS_OUT = 8 * U32          # final fp32 roundings of an output, relative to its own magnitude
# Decoder, per sample (relative to the model on absolute values, see _decode):
#   E_GATHER  the fp32 bilinear taps (12 fused multiply-adds and two plane sums: ~8 ulps of the sum of |tap| x |texel|) and the
#             fp16 hi + lo split of the features (2^-22);
#   E_MM      one layer of the three-pass fp16 product [hi|lo] x [Whi|Whi] + hi x Wlo: the split of both operands (2 x 2^-22),
#             the dropped lo x lo term (2^-22) and the fp32 accumulation of the tensor core, which truncates (about 2^-22 of the
#             running sum per k16 slice, at most 12 slices) -- 2^-19 covers that, and the 64-term fp32 FMA chains of the SIMT
#             kernel (64 x 2^-24);
#   E_TINY    absolute floor of an fp16 lo part that falls below fp16's normal range (half its 2^-24 spacing, x 2 for the
#             log2(e) / ln 2 scaling of the packed operands), per element of either operand;
#   E_SP      softplus through ex2.approx / lg2.approx (render_tc.cuh softplus2, p3d_common.cuh softplus_f): a few 2^-22 absolute;
#   E_SIG     the mip-NeRF sigmoid through ex2.approx / rcp.approx (sigmoid_clamp_f): a few 2^-22 absolute.
E_GATHER = 2.0 ** -20
E_MM = 2.0 ** -19
E_TINY = 2.0 ** -24
E_SP = 2.0 ** -20
E_SIG = 2.0 ** -20
# March, per interval: 1 - __expf(-x) cancels to the absolute error of exp near 1 -- the subtraction's 2^-24 (6e-8) plus
# ex2.approx's 2^-22 relative; the fp32 products of the transmittance add 2^-24 relative per interval.
E_EXP = 2.0 ** -21
FTZ = 2.0 ** -126          # fp32's smallest normal: softplus below it flushes to zero in the kernels (ex2.approx.ftz)
K_FILL = -123456           # prefill of the integer debug buffers beyond the launch
PAD = 1000                 # extra elements after each output and debug buffer

# ---------------------------------------------------------------------------------------------------------------------
# Python mirrors of the host-side tiling rules
# ---------------------------------------------------------------------------------------------------------------------
K_TC_TAIL, K_TC_TAIL_FLOATS, K_NET_FLOATS, K_OUT = 65536, 324, 4260, 32


def _round_up(a, b):
    return (a + b - 1) // b * b


def _pow2_group(n):                                     # render_common.cuh pow2_group
    return min(n & -n, 32)


def _ray_floats(Sc, Sf):                                # render_common.cuh make_ray_block (every renderer layout embeds it)
    S = Sc + Sf
    return 4 * _round_up(Sc, 4) + 2 * _round_up(Sf, 4) + 3 * _round_up(S, 4)


def tc_layout(RT, Sc, Sf, n_nets):
    """render_tc.cu make_tc_layout."""
    gc, gf = _pow2_group(Sc), (_pow2_group(Sf) if Sf else 1)
    NGc, NGf = Sc // gc, (Sf // gf if Sf else 0)
    tiles_c, tiles_f = (RT * Sc + 127) // 128, (RT * Sf + 127) // 128
    total = (K_TC_TAIL + (tiles_c + tiles_f) * 16384 + K_TC_TAIL_FLOATS * 4 + RT * _ray_floats(Sc, Sf) * 4
             + RT * (NGc + NGf) * K_OUT * n_nets * 4 + (4 * RT + 4) * 4)
    return dict(RT=RT, gc=gc, gf=gf, NGc=NGc, NGf=NGf, tiles_c=tiles_c, tiles_f=tiles_f, bytes=total)


def tc_plan(Sc, Sf, n_nets, total_rays, sms, max_smem):
    """p3d_render_fwd_tc (render_tc.cu:321-329 and 349-350): RT = min(384 / max(Sc, Sf), 16), reduced while the layout does
    not fit; tiles of RT rays; grid = min(SMs, tiles)."""
    RT = min(384 // max(Sc, Sf), 16)
    L = tc_layout(RT, Sc, Sf, n_nets)
    while RT > 1 and L['bytes'] + 1024 > max_smem:
        RT -= 1
        L = tc_layout(RT, Sc, Sf, n_nets)
    tiles = -(-total_rays // RT)
    return dict(L, kind='tc', RT0=min(384 // max(Sc, Sf), 16), tiles=tiles, grid=min(sms, tiles))


def pair_plan(Sc, Sf, n_nets, total_rays, sms, max_smem):
    """render_fwd_tc_pairs (render_tc2.cu:228-240): pairs of rays, three groups per CTA, grid = min(SMs, ceil(pairs / 3))."""
    grp = _round_up(2 * 16384 + 2 * _ray_floats(Sc, Sf) * 4
                    + 2 * (Sc // _pow2_group(Sc) + (Sf // _pow2_group(Sf) if Sf else 0)) * K_OUT * n_nets * 4 + 32, 1024)
    total = K_TC_TAIL + 3 * grp + K_TC_TAIL_FLOATS * 4
    assert total + 1024 <= max_smem
    pairs = (total_rays + 1) // 2
    return dict(kind='tc_pairs', RT=2, gc=_pow2_group(Sc), gf=_pow2_group(Sf) if Sf else 1, pairs=pairs, tiles=pairs,
                grid=min(sms, (pairs + 2) // 3), bytes=total)


def simt_layout(RT, Sc, Sf, n_nets):
    """render.cu make_layout (float offsets)."""
    Scp, Sfp = _round_up(Sc, 8), (_round_up(Sf, 8) if Sf else 0)
    gc, gf = _pow2_group(Scp), (_pow2_group(Sfp) if Sf else 1)
    NGc, NGf = Scp // gc, (Sfp // gf if Sf else 0)
    o = _round_up(n_nets * K_NET_FLOATS, 32) + RT * (Sc + Sf) * 32 + RT * _ray_floats(Sc, Sf)
    o += RT * (NGc + NGf) * K_OUT * n_nets + 4 * RT + 4
    return dict(RT=RT, gc=gc, gf=gf, NGc=NGc, NGf=NGf, NT=_round_up(RT * max(Scp, Sfp), 32), bytes=4 * o)


def simt_plan(Sc, Sf, n_nets, total_rays, sms, max_smem):
    """p3d_render_fwd (render.cu:688-709): RT = min(256 / round_up(max(Sc, Sf), 8), 8), reduced while two CTAs do not fit
    in one SM; grid = min(SMs x CTAs per SM (occupancy, not mirrored: 1 or 2), tiles)."""
    RT0 = min(256 // _round_up(max(Sc, Sf), 8), 8)
    RT = RT0
    L = simt_layout(RT, Sc, Sf, n_nets)
    while RT > 1 and L['bytes'] > (max_smem - 2048) // 2:
        RT -= 1
        L = simt_layout(RT, Sc, Sf, n_nets)
    tiles = -(-total_rays // RT)
    return dict(L, kind='simt', RT0=RT0, tiles=tiles, grid=f'min({sms}x(1|2), {tiles})')


def which_kernel(impl, Sc, Sf):
    """native.render_fwd's choice of kernel (native.py: use_tc and tc_variant)."""
    from pix2pix3d_b200 import native
    impl = impl or native.render_impl
    use_tc = impl in ('auto', 'tc', 'tc_pairs') and Sc % 8 == 0 and Sf % 8 == 0 and Sc <= 128 and Sf <= 128
    if not use_tc:
        return 'simt'
    return 'tc_pairs' if (impl == 'tc_pairs' or (impl == 'auto' and Sc == 64 and Sf == 64)) else 'tc'


def plan(kind, Sc, Sf, n_nets, total_rays, sms, max_smem):
    return {'tc': tc_plan, 'tc_pairs': pair_plan, 'simt': simt_plan}[kind](Sc, Sf, n_nets, total_rays, sms, max_smem)


def _fmt(p):
    seg = f"seg {p['gc']}/{p['gf']}"
    return f"{p['kind']:<8} RT {p['RT']:>2} tiles {p['tiles']:>5} grid {p['grid']} {seg}"


def _device():
    props = torch.cuda.get_device_properties(torch.cuda.current_device())
    # sm_90's opt-in shared memory per block is 227 KB
    return props.multi_processor_count, getattr(props, 'shared_memory_per_block_optin', 227 * 1024)


# ---------------------------------------------------------------------------------------------------------------------
# the launch description and the float64 model
# ---------------------------------------------------------------------------------------------------------------------
def _f32(x):
    return torch.tensor(float(x), dtype=torch.float32)


def describe(planes, module, o, d, depths_coarse, u, box_warp, white_back=False, stratified=None, plane_index=None):
    """A launch as native.render_fwd receives it. Coarse depths are formed here with the kernels' fp32 operations
    (render_common.cuh coarse_depth) for every ray; the decoder's effective parameters are the fp32 products
    FullyConnectedLayer forms (networks_stylegan2.py:111-119)."""
    from pix2pix3d_b200 import native
    B, R = o.shape[:2]
    n = B * R
    dev = o.device
    if stratified is None:
        dc = depths_coarse.reshape(n, -1).float()
    else:
        jit = stratified['jitter'].reshape(n, -1).float()
        table = stratified['table'].reshape(-1).float()
        Sc = jit.shape[1]
        if 'ray_start' in stratified:
            rs, re_ = stratified['ray_start'].reshape(n, 1).float(), stratified['ray_end'].reshape(n, 1).float()
            span = re_ - rs
            delta = (torch.tensor(1.0, dtype=torch.float32) / torch.tensor(float(Sc - 1), dtype=torch.float32)).to(dev)
            dc = (rs + table[None] * span) + jit * (span * delta)
        else:
            dc = table[None] + jit * _f32(stratified['delta']).to(dev)
    nets, sigma_net, masks = native.describe_decoder(module)
    mnets = []
    for net, mask in zip(nets, masks):
        w1, b1 = native._effective_fc(net[0])
        w2, b2 = native._effective_fc(net[2])
        mnets.append(dict(W1=w1.detach().double().to(dev), b1=b1.detach().double().to(dev), W2=w2.detach().double().to(dev),
                          b2=b2.detach().double().to(dev),
                          mask=torch.tensor([(mask >> i) & 1 for i in range(32)], dtype=torch.bool, device=dev)))
    img = torch.arange(n, device=dev) // R
    bidx = img if plane_index is None else plane_index.to(dev).long()[img]
    return dict(planes=planes, o=o.reshape(n, 3).float(), d=d.reshape(n, 3).float(), dc=dc.contiguous(),
                u=None if u is None else u.reshape(n, -1).float(), cs=_f32(2.0 / float(box_warp)).to(dev),
                white_back=bool(white_back), bidx=bidx, nets=mnets, sigma_net=sigma_net, B=B, R=R, n=n,
                Sc=dc.shape[1], Sf=0 if u is None else int(u.shape[-1]), module=module,
                call=dict(planes=planes, o=o, d=d, dc=depths_coarse, u=u, box_warp=box_warp, white_back=white_back,
                          stratified=stratified, plane_index=plane_index))


PLANE_AXES = ((0, 1), (0, 2), (2, 0))       # plane k samples (x, y), (x, z), (z, x) (render_common.cuh plane_values)


def _gather(planes, bidx, pos, fault=None):
    """Tri-plane bilinear gather (zeros padding, align_corners=False) of planes [Bp,3,H,W,32] (any strides) at the scaled
    positions pos [N,3] (fp32) of samples whose plane set is bidx [N] -> (mean feature [N,32], the same on |tap| x |texel|)."""
    H, W = planes.shape[2], planes.shape[3]
    x = torch.zeros(pos.shape[0], 32, dtype=torch.float64, device=pos.device)
    xa = torch.zeros_like(x)
    for k, (i0, i1) in enumerate(PLANE_AXES):
        gx, gy = pos[:, i0], pos[:, i1]
        ix = ((gx + 1) * W - 1) * 0.5
        iy = ((gy + 1) * H - 1) * 0.5
        if fault == 'half_texel':
            ix = ix + 0.5
        inside = (ix > -1) & (ix < W) & (iy > -1) & (iy < H)
        x0f, y0f = torch.floor(ix), torch.floor(iy)
        ax, bx = (x0f + 1) - ix, ix - x0f
        ay, by = (y0f + 1) - iy, iy - y0f
        x0 = torch.where(inside, x0f, torch.zeros_like(x0f)).long()
        y0 = torch.where(inside, y0f, torch.zeros_like(y0f)).long()
        for dy, dx, wgt in ((0, 0, ax * ay), (0, 1, bx * ay), (1, 0, ax * by), (1, 1, bx * by)):
            xx, yy = x0 + dx, y0 + dy
            ok = inside & (xx >= 0) & (xx < W) & (yy >= 0) & (yy < H)
            v = planes[bidx, k, yy.clamp(0, H - 1), xx.clamp(0, W - 1)].double()
            wv = torch.where(ok, wgt, torch.zeros_like(wgt)).double()[:, None]
            x += wv * v
            xa += wv.abs() * v.abs()
    return x / 3, xa / 3


def _softplus(x):
    return x.clamp(min=0) + torch.log1p(torch.exp(-x.abs()))


def _decode(nets, sigma_net, x, xa, fault=None):
    """Both decoder nets on features x [N,32] -> (colours [N,32 n_nets], their bound, sigma [N], its bound).
    Per net: a = W1 x + b1, h = softplus(a), o = W2 h + b2; colour channels under the net's mask through the mip-NeRF sigmoid
    (triplane.py:133). The bound follows the error of each stage through the next one's Lipschitz constant: 1 for softplus,
    1.002 / 4 for the sigmoid, |W| for a layer."""
    cols, ecols, sig = [], [], []
    log2e3 = math.log2(math.e) / 3          # the packed layer-1 weights carry log2(e) / 3 (render_tc.cu pack_decoder_tc_kernel)
    for net in nets:
        W1, b1, W2, b2 = net['W1'], net['b1'], net['W2'], net['b2']
        W1u = (W1 * log2e3).half().double() / log2e3 if fault == 'drop_hilo' else W1
        a = x @ W1u.T + b1
        A = xa @ W1.abs().T + b1.abs()
        ea = (E_MM + E_GATHER) * A + E_TINY * (W1.abs().sum(1)[None] + xa.sum(1, keepdim=True))
        h = _softplus(a)
        eh = ea + E_SP
        o = h @ W2.T + b2
        eo = E_MM * (h @ W2.abs().T + b2.abs()) + eh @ W2.abs().T + E_TINY * (W2.abs().sum(1)[None] + h.sum(1, keepdim=True))
        c, ec = o[:, 1:33], eo[:, 1:33]
        m = net['mask']
        c = torch.where(m, torch.sigmoid(c) * 1.002 - 0.001, c)
        ec = torch.where(m, ec * (1.002 / 4) + E_SIG, ec)
        cols.append(c)
        ecols.append(ec)
        sig.append((o[:, 0], eo[:, 0]))
    s, es = sig[1 - sigma_net if fault == 'sigma_net' else sigma_net]
    return torch.cat(cols, 1), torch.cat(ecols, 1), s, es


def _march(z, s, es, c=None, ec=None, fault=None):
    """MipRayMarcher2 (ray_marcher.py:25-47) in float64 on sorted samples z [n,S] with densities s and colours c, and the
    bound of each result. alpha_i = 1 - exp(-softplus(sigma_mid - 1) delta_i); a transmittance is a product of (1 - alpha), so
    its error is at most the sum of the earlier alphas' errors, and the weight sum telescopes to 1 - T_S."""
    n, S = z.shape
    smid = (s[:, :-1] + s[:, 1:]) / 2
    esm = (es[:, :-1] + es[:, 1:]) / 2
    xm = smid - 1
    dens = _softplus(xm)
    dens = torch.where(dens < FTZ, torch.zeros_like(dens), dens)
    edens = torch.sigmoid(xm + esm) * esm + E_SP + U32 * dens
    delta = z[:, 1:] - z[:, :-1]
    xa = dens * delta
    alpha = -torch.expm1(-xa)
    ealpha = delta.abs() * edens + 2 * U32 * xa.abs() + E_EXP
    t = 1 - alpha + 1e-10
    T = torch.cat([torch.ones_like(t[:, :1]), torch.cumprod(t, 1)[:, :-1]], 1)
    w = alpha * T
    i = torch.arange(S - 1, device=z.device, dtype=torch.float64)[None]
    eT = torch.cat([torch.zeros_like(ealpha[:, :1]), torch.cumsum(ealpha, 1)[:, :-1]], 1) + i * (2 * U32 + 1e-10)
    ew = ealpha * T + alpha * eT + 2 * U32 * w
    ws = w.sum(1)
    ews = ealpha.sum(1) + 3 * S * U32 + S * 1e-10
    zmid = (z[:, :-1] + z[:, 1:]) / 2
    with np.errstate(all='ignore'):
        depth = (w * zmid).sum(1) / ws
        edepth = ((ew * (zmid - depth[:, None]).abs()).sum(1) + (S + 4) * U32 * (w * zmid.abs()).sum(1)) / ws
    r = dict(w=w, ew=ew, ws=ws, ews=ews, depth=depth, edepth=edepth)
    if c is not None:
        cm, ecm = (c[:, :-1] + c[:, 1:]) / 2, (ec[:, :-1] + ec[:, 1:]) / 2
        if fault == 'coef_wj':
            rgb = (w[..., None] * c[:, :-1]).sum(1)
        else:
            rgb = (w[..., None] * cm).sum(1)
        r['rgb'] = rgb
        r['ergb'] = (ew[..., None] * cm.abs() + w[..., None] * ecm).sum(1) + (S + 4) * U32 * (w[..., None] * cm.abs()).sum(1)
    return r


def _shade(L, rays, z, fault=None):
    """Decoder outputs of the samples at depths z [n,k] (fp32) of the given rays."""
    n, k = z.shape
    o, d = L['o'][rays], L['d'][rays]
    pos = ((o[:, None, :] + z[..., None] * d[:, None, :]) * L['cs']).reshape(-1, 3)     # render_common.cuh sample_point
    bidx = L['bidx'][rays][:, None].expand(n, k).reshape(-1)
    x, xa = _gather(L['planes'], bidx, pos, fault)
    c, ec, s, es = _decode(L['nets'], L['sigma_net'], x, xa, fault)
    return c.reshape(n, k, -1), ec.reshape(n, k, -1), s.reshape(n, k), es.reshape(n, k)


def model(L, rays, depths_fine=None, fault=None):
    """Float64 model of the given rays (global ray ids) of launch L. `depths_fine` [n, Sf]: the fine depths to march (the
    kernel's, once they are checked; None -> the fp32 oracle's sample_importance on the model's own coarse weights).
    Returns the per-ray references and bounds; the depth is not yet clamped (see clamp_depth)."""
    zc = L['dc'][rays]
    c, ec, s, es = _shade(L, rays, zc, fault)
    out = {}
    Sf = L['Sf']
    if Sf > 0:
        mc = _march(zc.double(), s, es)
        out['wc'], out['ewc'] = mc['w'], mc['ew']
        if depths_fine is None:
            depths_fine = torch.from_numpy(O.renderer.sample_importance(
                zc.cpu().numpy(), mc['w'].float().cpu().numpy(), L['u'][rays].cpu().numpy())).to(zc.device)
        zf = depths_fine.float()
        cf, ecf, sf, esf = _shade(L, rays, zf, fault)
        zall = torch.cat([zc, zf], 1)
        perm = torch.sort(zall, dim=1, stable=True)[1]
        if fault == 'swap':
            mid = perm.shape[1] // 2
            perm[:, [mid - 1, mid]] = perm[:, [mid, mid - 1]]
        if fault == 'drop_fine':
            perm = perm[perm != L['Sc']].reshape(perm.shape[0], -1)        # fine sample 0 of every ray
        g = lambda t: torch.gather(t, 1, perm if t.ndim == 2 else perm[..., None].expand(-1, -1, t.shape[-1]))
        z, s, es, c, ec = g(zall.double()), g(torch.cat([s, sf], 1)), g(torch.cat([es, esf], 1)), g(torch.cat([c, cf], 1)), \
            g(torch.cat([ec, ecf], 1))
        out['zf'], out['perm'] = zf, perm
    else:
        z = zc.double()
    m = _march(z, s, es, c, ec, fault)
    rgb, ergb = m['rgb'], m['ergb']
    if L['white_back'] and fault != 'no_white_back':
        rgb = rgb + 1 - m['ws'][:, None]
        ergb = ergb + m['ews'][:, None]
    w, ew = m['w'], m['ew']
    if w.shape[1] < L['Sc'] + Sf - 1:                                       # a dropped sample: one weight fewer
        w, ew = torch.cat([w, torch.zeros_like(w[:, :1])], 1), torch.cat([ew, ew[:, -1:]], 1)
    out.update(feat=rgb * 2 - 1, efeat=2 * ergb, ws=m['ws'], ews=m['ews'], depth=m['depth'], edepth=m['edepth'], wf=w, ewf=ew)
    return out


def clamp_range(L, depths_fine):
    """The launch's smallest and largest sample depth (coarse and fine, all rays): what the last CTA clamps to."""
    lo, hi = L['dc'].min(), L['dc'].max()
    if depths_fine is not None and depths_fine.numel():
        lo, hi = torch.minimum(lo, depths_fine.min()), torch.maximum(hi, depths_fine.max())
    return float(lo), float(hi)


def depth_reference(m, lo, hi):
    """(expected depth, bound): a zero weight sum gives NaN -> +inf -> the launch's largest depth, exactly; a sum that is not
    distinguishable from zero at the kernels' precision only has to lie in [lo, hi]; otherwise the clamped model depth."""
    exp = m['depth'].clamp(lo, hi)
    tol = m['edepth'].clone()
    zero = m['ws'] == 0
    exp = torch.where(zero, torch.full_like(exp, hi), exp)
    tol = torch.where(zero, torch.zeros_like(tol), tol)
    vague = ~zero & (m['ews'] >= 0.5 * m['ws'])
    tol = torch.where(vague, torch.full_like(tol, math.inf), tol)
    return exp, tol


def ratio(got, ref, tol):
    """max of |got - ref| / (EPS_OUT |ref| + tol) over the elements; 0 where equal, inf where NaN."""
    got = got.double().reshape(ref.shape)
    err = (got - ref).abs()
    bound = EPS_OUT * ref.abs() + tol.reshape(ref.shape)
    r = torch.where(err == 0, torch.zeros_like(err), err / bound)
    r = torch.nan_to_num(r, nan=math.inf)
    return float(r.max()) if r.numel() else 0.0


# ---------------------------------------------------------------------------------------------------------------------
# running a launch and checking it
# ---------------------------------------------------------------------------------------------------------------------
OUT_KEYS = {'feat': torch.float32, 'depth': torch.float32, 'wsum': torch.float32, 'weights_final': torch.float32,
            'perm': torch.int32, 'weights_coarse': torch.float32, 'depths_fine': torch.float32, 'inds': torch.int32}


def run(L, impl):
    """One native.render_fwd launch of L with NaN-prefilled output and debug buffers PAD elements longer than it needs;
    checks that nothing beyond the launch's elements changed. Returns the outputs as flat per-ray tensors."""
    from pix2pix3d_b200 import native
    c = L['call']
    n, Sc, Sf = L['n'], L['Sc'], L['Sf']
    dec = L.get('packed') or native.pack_decoder(L['module'])
    L['packed'] = dec
    per = {'feat': dec.out_channels, 'depth': 1, 'wsum': 1, 'weights_final': Sc + Sf - 1, 'perm': Sc + Sf,
           'weights_coarse': Sc - 1, 'depths_fine': Sf, 'inds': Sf}
    bufs = {}
    for k, dt in OUT_KEYS.items():
        if Sf == 0 and k in ('weights_coarse', 'depths_fine', 'inds'):
            continue
        fill = float('nan') if dt == torch.float32 else K_FILL
        bufs[k] = torch.full((n * per[k] + PAD,), fill, dtype=dt, device=c['o'].device)
    feat, depth, wsum, dbg = native.render_fwd(c['planes'], dec, c['o'], c['d'], c['dc'], c['u'], c['box_warp'],
                                               white_back=c['white_back'], debug=True, impl=impl, stratified=c['stratified'],
                                               plane_index=c['plane_index'], out=bufs)
    torch.cuda.synchronize()
    for k, b in bufs.items():
        tail = b[n * per[k]:]
        if b.dtype == torch.float32:
            assert torch.isnan(tail).all() and (tail.view(torch.int32) == 0x7fc00000).all(), f'{k} written beyond the launch'
        else:
            assert (tail == K_FILL).all(), f'{k} written beyond the launch'
    got = dict(feat=feat.reshape(n, -1), depth=depth.reshape(n), wsum=wsum.reshape(n))
    got.update({k: v.reshape(n, -1) for k, v in dbg.items()})
    return got


def check(L, got, rays=None, chunk=4096):
    """Every modelled ray of a finished launch: the three importance-sampling checks, then every output against the model.
    Returns the worst err / bound per output."""
    n, Sc, Sf = L['n'], L['Sc'], L['Sf']
    dev = L['o'].device
    rays = torch.arange(n, device=dev) if rays is None else rays.to(dev)
    df_all = got.get('depths_fine')
    lo, hi = clamp_range(L, df_all)
    worst = dict(wc=0.0, feat=0.0, wsum=0.0, wf=0.0, depth=0.0)
    dmin, dmax = got['depth'].min().item(), got['depth'].max().item()
    assert lo <= dmin and dmax <= hi, 'every depth lies in the launch range'
    for i in range(0, rays.numel(), chunk):
        r = rays[i:i + chunk]
        df = df_all[r] if Sf else None
        m = model(L, r, df)
        if Sf:
            worst['wc'] = max(worst['wc'], ratio(got['weights_coarse'][r], m['wc'], m['ewc']))
            dc = L['dc'][r].cpu().numpy()
            fine, od = O.renderer.sample_importance(dc, got['weights_coarse'][r].cpu().numpy(), L['u'][r].cpu().numpy(),
                                                    return_debug=True)
            assert np.array_equal(fine.view(np.uint32), df.cpu().numpy().view(np.uint32)), 'fine depths'
            assert np.array_equal(od['inds'], got['inds'][r].cpu().numpy()), 'importance indices'
            assert torch.equal(got['perm'][r].long(), m['perm']), 'merge permutation'
        else:
            assert torch.equal(got['perm'][r].long(), torch.sort(L["dc"][r], dim=1, stable=True)[1])
        worst['feat'] = max(worst['feat'], ratio(got['feat'][r], m['feat'], m['efeat']))
        worst['wsum'] = max(worst['wsum'], ratio(got['wsum'][r], m['ws'], m['ews']))
        worst['wf'] = max(worst['wf'], ratio(got['weights_final'][r], m['wf'], m['ewf']))
        exp, tol = depth_reference(m, lo, hi)
        exact = tol == 0
        assert torch.equal(got['depth'][r][exact].double(), exp[exact]), 'clamped depths'
        worst['depth'] = max(worst['depth'], ratio(got['depth'][r][~exact], exp[~exact], tol[~exact]))
    return worst


def _fmt_worst(w):
    return ' '.join(f'{k} {v:.3g}' for k, v in w.items())


def assert_within(worst, tag):
    bad = {k: v for k, v in worst.items() if not v <= 1.0}
    assert not bad, f'{tag}: worst err / bound {bad}'


# ---------------------------------------------------------------------------------------------------------------------
# synthetic launches
# ---------------------------------------------------------------------------------------------------------------------
DEC_KINDS = ['osg', 'semantic_raw', 'semantic_sigmoid', 'entangle_6', 'entangle_19', 'entangle_sigmoid', 'late_6', 'late_1',
             'late_19']


def make_decoder(kind, seed=17, device='cuda'):
    """A decoder module of every layout native.describe_decoder maps (triplane.py:112, triplane_cond.py:859,926), with
    parameters drawn N(0, 0.6)."""
    from pix2pix3d_b200.training import triplane, triplane_cond as tc
    base = {'decoder_lr_mul': 1.0, 'decoder_output_dim': 32}
    make = {
        'osg': lambda: triplane.OSGDecoder(32, dict(base)),
        'semantic_raw': lambda: tc.OSGDecoder_semantic(32, dict(base, sigmoid=False)),
        'semantic_sigmoid': lambda: tc.OSGDecoder_semantic(32, dict(base, sigmoid=True)),
        'entangle_6': lambda: tc.OSGDecoder_semantic_entangle(32, dict(base, sigmoid=False, semantic_channels=6)),
        'entangle_19': lambda: tc.OSGDecoder_semantic_entangle(32, dict(base, sigmoid=False, semantic_channels=19)),
        'entangle_sigmoid': lambda: tc.OSGDecoder_semantic_entangle(32, dict(base, sigmoid=True, semantic_channels=1)),
        'late_6': lambda: tc.OSGDecoder_semantic_lateSeparate(32, dict(base, sigmoid=False, semantic_channels=6)),
        'late_1': lambda: tc.OSGDecoder_semantic_lateSeparate(32, dict(base, sigmoid=True, semantic_channels=1)),
        'late_19': lambda: tc.OSGDecoder_semantic_lateSeparate(32, dict(base, sigmoid=False, semantic_channels=19)),
    }[kind]
    torch.manual_seed(seed)
    dec = make().requires_grad_(False)
    g = torch.Generator().manual_seed(seed)
    for p in dec.parameters():
        p.copy_(torch.randn(p.shape, generator=g) * 0.6)
    return dec.to(device)


def scene(n_rays, Sc, Sf, seed=0, kind='late_6', white_back=False, H=64, device='cuda', start=2.25, end=3.3):
    """n_rays rays (two images when the count is even) from about 2.7 units away through the [-0.5, 0.5]^3 box (box_warp 1),
    stratified coarse depths over [start, end] and uniform importance draws."""
    g = torch.Generator().manual_seed(seed)
    B = 2 if n_rays % 2 == 0 and n_rays > 1 else 1
    R = n_rays // B
    planes = torch.randn(B, 3, 32, H, H, generator=g)
    orig = torch.tensor([0.3, -0.2, 2.7]) + 0.05 * torch.randn(B, R, 3, generator=g)
    target = (torch.rand(B, R, 3, generator=g) - 0.5) * 0.9
    dirs = torch.nn.functional.normalize(target - orig, dim=-1)
    base = torch.linspace(start, end, Sc).reshape(1, 1, Sc)
    dc = base + torch.rand(B, R, Sc, generator=g) * ((end - start) / (Sc - 1))
    u = torch.rand(B * R, Sf, generator=g) if Sf else None
    dev = torch.device(device)
    pl = planes.permute(0, 1, 3, 4, 2).contiguous().to(dev)
    return describe(pl, make_decoder(kind, seed + 17, dev), orig.to(dev), dirs.to(dev), dc.to(dev),
                    None if u is None else u.to(dev), 1.0, white_back=white_back)


def _special_decoder(device):
    """A one-net decoder whose sigma is -250 at zero features (rays outside the box get a weight sum of exactly zero) and
    about 0..10 inside, where plane channel 0 carries +5: hidden unit 0 reads channel 0 and lifts sigma by about 250."""
    from pix2pix3d_b200 import native
    dec = make_decoder('osg', 5, 'cpu')
    fc1, fc2 = dec.net[0], dec.net[2]
    with torch.no_grad():
        fc1.weight[0].zero_()
        fc1.weight[0, 0] = 50.0 / fc1.weight_gain
        fc1.bias[0] = -20.0 / fc1.bias_gain
        fc2.weight[1:, 0] = 0.0                                    # the lift unit feeds sigma only
        fc2.weight[0, 0] = 1.1 / fc2.weight_gain
        w1, b1 = native._effective_fc(fc1)
        w2, b2 = native._effective_fc(fc2)
        sigma0 = float(_softplus(b1.double()) @ w2[0].double() + b2[0].double())
        fc2.bias[0] += (-250.0 - sigma0) / fc2.bias_gain
    return dec.to(device)


def clamp_scene(n_rays, Sc, Sf, special, seed=3, device='cuda'):
    """scene() with the special decoder, plane channel 0 at +5, and `special` = {ray id: kind} rays:
    'nonmono' (two coarse depths swapped), 'empty' (pointing away from the box: zero weight sum), 'max' (coarse depths out
    to 4.5: the launch's largest depth), 'min' (coarse depths from -1.0: the smallest, negative)."""
    L = scene(n_rays, Sc, Sf, seed, 'osg', device=device)
    c = L['call']
    pl = c['planes'].clone()
    pl[..., 0] = 5.0 + 0.1 * pl[..., 0]
    o, d, dc = c['o'].clone().reshape(-1, 3), c['d'].clone().reshape(-1, 3), c['dc'].clone().reshape(L['n'], Sc)
    for ray, kind in special.items():
        if kind == 'nonmono':
            dc[ray, [3, 4]] = dc[ray, [4, 3]]
        elif kind == 'empty':
            d[ray] = torch.nn.functional.normalize(torch.tensor([0.3, 0.1, 1.0], device=d.device), dim=0)
        elif kind == 'max':
            dc[ray] = torch.linspace(2.25, 4.5, Sc, device=dc.device)
        elif kind == 'min':
            dc[ray] = torch.linspace(-1.0, 3.3, Sc, device=dc.device)
    B, R = L['B'], L['R']
    return describe(pl, _special_decoder(torch.device(device)), o.reshape(B, R, 3), d.reshape(B, R, 3), dc.reshape(B, R, Sc),
                    c['u'], 1.0)


# ---------------------------------------------------------------------------------------------------------------------
# the model against the reference fixtures, and planted faults (CPU)
# ---------------------------------------------------------------------------------------------------------------------
def _fixture_launch(g):
    from test_gpu_renderer import torch_decoder
    opts = render_opts(g)
    b, m = g['ray_origins'].shape[:2]
    dc = O.renderer.sample_stratified(b, m, opts['ray_start'], opts['ray_end'], opts['depth_resolution'], g['jitter'])
    planes = torch.from_numpy(g['planes']).permute(0, 1, 3, 4, 2)
    u = torch.from_numpy(g['u']) if int(g['Sf']) > 0 else None
    return describe(planes, torch_decoder(g, 'cpu'), torch.from_numpy(g['ray_origins']), torch.from_numpy(g['ray_dirs']),
                    torch.from_numpy(dc), u, opts['box_warp'], white_back=opts['white_back'])


@pytest.mark.parametrize('case', RENDER_CASES)
def test_model_reproduces_reference_fixtures(case):
    """The model, fed each fixture's own fine depths, reproduces the reference's fp32 outputs within the bound, and the
    fixture's bookkeeping passes the checks the kernels' must: coarse weights within bound, the stable merge permutation,
    and fine depths from the fp32 oracle on its coarse weights (here to 1e-5 relative: the reference's torch.sum and cumsum
    add in an order of their own; the kernels share the oracle's order and must match it bit for bit)."""
    g = load_golden('renderer_' + case)
    L = _fixture_launch(g)
    n, Sf = L['n'], L['Sf']
    rays = torch.arange(n)
    df = torch.from_numpy(g['depths_fine']).reshape(n, Sf) if Sf else None
    m = model(L, rays, df)
    w = {}
    if Sf:
        w['wc'] = ratio(torch.from_numpy(g['weights_coarse']).reshape(n, -1), m['wc'], m['ewc'])
        fine = O.renderer.sample_importance(L['dc'].numpy(), g['weights_coarse'].reshape(n, -1), L['u'].numpy())
        assert np.abs(fine - df.numpy()).max() <= 1e-5 * np.abs(df.numpy()).max()
        assert torch.equal(torch.from_numpy(g['perm']).reshape(n, -1), m['perm'])
    w['feat'] = ratio(torch.from_numpy(g['feat']).reshape(n, -1), m['feat'], m['efeat'])
    w['wsum'] = ratio(torch.from_numpy(g['wsum']).reshape(n), m['ws'], m['ews'])
    w['wf'] = ratio(torch.from_numpy(g['weights_final']).reshape(n, -1), m['wf'], m['ewf'])
    exp, tol = depth_reference(m, *clamp_range(L, df))
    w['depth'] = ratio(torch.from_numpy(g['depth']).reshape(n), exp, tol)
    print(f'fixture {case}: worst err / bound {_fmt_worst(w)}')
    assert_within(w, case)


def _cta_rays(n, RT, grid, cta=0):
    """Rays of the tiles CTA `cta` walks (tile = cta, cta + grid, ...)."""
    return torch.tensor([r for r in range(n) if (r // RT) % grid == cta])


def _hilo_scene(n, Sc, Sf):
    """scene() with positive plane values and a raw-colour decoder whose positive layer-1 weights all sit 0.45 fp16 ulps
    above an fp16 value once packed (x log2(e) / 3): the hi x lo pass carries the same sign in every product, so dropping it
    cannot cancel (a worst case the bound has to see)."""
    L = scene(n, Sc, Sf, 2, 'semantic_raw', H=32, device='cpu')
    c = L['call']
    dec = L['module']
    fc1, fc2 = dec.net[0], dec.net[2]
    s = math.log2(math.e) / 3
    g = torch.Generator().manual_seed(4)
    with torch.no_grad():
        hi = (torch.rand(64, 32, generator=g) * 0.5 + 0.5).half().double()
        fc1.weight.copy_(((hi + 0.45 * 2.0 ** -11) / s / fc1.weight_gain).float())
        fc1.bias.fill_(-8.0)
        fc2.weight.copy_(torch.rand(33, 64, generator=g) / fc2.weight_gain * 0.05)
        fc2.weight[0] = -fc2.weight[0]
    return describe(c['planes'].abs() * 0.3, dec, c['o'], c['d'], c['dc'], c['u'], 1.0)


def test_model_rejects_planted_faults():
    """Each fault planted in the model moves some element past the bound that the exact model meets: a fine sample dropped,
    two merged samples swapped, w_j in place of (w_{j-1} + w_j) / 2, a half-texel gather shift, the layer-1 hi x lo pass
    dropped, white_back omitted, sigma from the wrong net, and the depth clamped to one CTA's range."""
    Sc = Sf = 16
    RT, grid = 16, 2                                            # tc_plan's RT at 16+16, on a two-SM device
    n = 6 * RT
    special = {0: 'empty', RT + 5: 'max', 2 * RT + 1: 'min'}     # CTA 0 owns the empty ray, CTA 1 the largest depth
    Lc = clamp_scene(n, Sc, Sf, special, device='cpu')
    Lw = scene(n, Sc, Sf, 1, 'late_6', white_back=True, H=32, device='cpu', start=2.0, end=3.6)
    rays = torch.arange(n)
    seen = {}
    for L, faults in ((Lw, ['drop_fine', 'swap', 'coef_wj', 'half_texel', 'no_white_back', 'sigma_net']),
                      (_hilo_scene(n, Sc, Sf), ['drop_hilo']), (Lc, ['cta_clamp'])):
        ref = model(L, rays)
        df = ref['zf']
        lo, hi = clamp_range(L, df)
        exp, tol = depth_reference(ref, lo, hi)
        for fault in faults:
            if fault == 'cta_clamp':
                mine = _cta_rays(n, RT, grid)
                m = dict(ref)
                lo2, hi2 = float(torch.cat([L['dc'][mine], df[mine]], 1).min()), float(torch.cat([L['dc'][mine], df[mine]], 1).max())
                got_d, _ = depth_reference(m, lo2, hi2)
                got = dict(feat=ref['feat'], ws=ref['ws'], wf=ref['wf'], depth=got_d)
            else:
                m = model(L, rays, df, fault=fault)
                got = dict(feat=m['feat'], ws=m['ws'], wf=m['wf'], depth=depth_reference(m, lo, hi)[0])
            r = max(ratio(got['feat'], ref['feat'], ref['efeat']), ratio(got['ws'], ref['ws'], ref['ews']),
                    ratio(got['wf'], ref['wf'], ref['ewf']))
            exact = tol == 0
            if not torch.equal(got['depth'][exact], exp[exact]):
                r = math.inf
            r = max(r, ratio(got['depth'][~exact], exp[~exact], tol[~exact]))
            seen[fault] = r
        # the exact model meets its own bound, and the special rays are what they claim
        assert ratio(ref['feat'], ref['feat'], ref['efeat']) == 0
    for name, r in seen.items():
        print(f'planted fault {name!r}: worst err / bound = {r:.3g} -> {"rejected" if r > 1 else "ACCEPTED"}')
    assert all(r > 1 for r in seen.values()), seen
    m = model(Lc, rays)
    assert float(m['ws'][0]) == 0 and bool((m['ws'][torch.arange(n) != 0] > 0).any())
    assert clamp_range(Lc, m['zf'])[0] < 0


def test_tiling_mirror_hits_the_layouts_the_sweep_targets():
    """The host rules restated here give the layouts the GPU sweep is built around (H100: 227 KB of shared memory per block)."""
    smem = 227 * 1024
    want_rt = {(8, 0): 16, (16, 8): 16, (24, 24): 16, (40, 40): 9, (48, 48): 8, (64, 64): 6, (72, 72): 5, (96, 32): 4,
               (32, 96): 4, (120, 120): 3, (128, 0): 3, (128, 128): 3}
    for (Sc, Sf), rt in want_rt.items():
        for nets in (1, 2):
            p = tc_plan(Sc, Sf, nets, 10 ** 6, 132, smem)
            assert p['RT'] == p['RT0'] == rt, (Sc, Sf)        # the tensor-core kernel's RT reduction never fires
    for Sc, Sf in ((40, 40), (72, 72), (120, 120)):
        p = tc_plan(Sc, Sf, 1, 1, 132, smem)
        assert p['RT'] * Sc == 360 and p['gc'] == 8 and _straddles(p['RT'], Sc)
    assert tc_plan(96, 32, 1, 1, 132, smem)['tiles_c'] == 3 and tc_plan(96, 32, 1, 1, 132, smem)['tiles_f'] == 1
    assert tc_plan(32, 96, 1, 1, 132, smem)['tiles_c'] == 1 and tc_plan(32, 96, 1, 1, 132, smem)['tiles_f'] == 3
    assert simt_plan(32, 32, 2, 1, 132, smem)['RT'] == 7 and simt_plan(32, 32, 2, 1, 132, smem)['NT'] == 224
    assert simt_plan(36, 36, 2, 1, 132, smem)['RT0'] == 6 and simt_plan(36, 36, 2, 1, 132, smem)['RT'] == 5
    assert set(SIMT_REDUCED) >= {(32, 32, 2), (36, 36, 2)}


def _straddles(RT, Sc):
    """Does some ray's run of coarse rows cross a 128-row warpgroup tile?"""
    return any((r * Sc) // 128 != ((r + 1) * Sc - 1) // 128 for r in range(RT))


SIMT_REDUCED = [(sc, sf, nets) for sc, sf in ((32, 32), (36, 36), (40, 40), (64, 64), (24, 24)) for nets in (1, 2)
                if simt_plan(sc, sf, nets, 1, 132, 227 * 1024)['RT'] < simt_plan(sc, sf, nets, 1, 132, 227 * 1024)['RT0']]


# ---------------------------------------------------------------------------------------------------------------------
# GPU: sweep at the schedule edges
# ---------------------------------------------------------------------------------------------------------------------
def _sweep(kind, Sc, Sf, n_rays, seed, tag, kind_dec='late_6', white_back=False, expect=None):
    sms, smem = _device()
    L = scene(n_rays, Sc, Sf, seed, kind_dec, white_back)
    p = plan(kind, Sc, Sf, len(L['nets']), n_rays, sms, smem)
    if expect:
        expect(p, sms)
    got = run(L, kind)
    w = check(L, got)
    print(f'{tag:<34} {Sc:>3}+{Sf:<3} rays {n_rays:>6} {_fmt(p)} | {_fmt_worst(w)}')
    assert_within(w, tag)
    return p


TC_SHAPES = [(8, 0), (16, 8), (24, 24), (40, 40), (48, 48), (64, 64), (72, 72), (96, 32), (32, 96), (120, 120), (128, 0),
             (128, 128)]
TILE_COUNTS = {'tiles=1': lambda s: 1, 'tiles=sms-1': lambda s: s - 1, 'tiles=sms': lambda s: s, 'tiles=sms+1': lambda s: s + 1,
               'tiles=3sms+2': lambda s: 3 * s + 2}


@gpu
@pytest.mark.parametrize('count', list(TILE_COUNTS) + ['rays=1', 'rays=RT-1', 'rays=RT', 'rays=RT+1'])
@pytest.mark.parametrize('shape', TC_SHAPES, ids=lambda s: f'{s[0]}+{s[1]}')
def test_tc_tile_counts(shape, count):
    """render_fwd_tc_kernel at every sample layout it accepts (segment widths 8/16/32, partial and straddled warpgroup tiles,
    groups without a fine tile, S = 256) and tile counts around the SM count, each with a ragged last tile."""
    Sc, Sf = shape
    sms, smem = _device()
    RT = tc_plan(Sc, Sf, 2, 1, sms, smem)['RT']
    if count.startswith('tiles='):
        t = TILE_COUNTS[count](sms)
        n = (t - 1) * RT + max(1, RT // 2)
    else:
        n = {'rays=1': 1, 'rays=RT-1': RT - 1, 'rays=RT': RT, 'rays=RT+1': RT + 1}[count]
        t = -(-n // RT)

    def expect(p, sms):
        assert p['tiles'] == t and p['grid'] == min(sms, t)

    _sweep('tc', Sc, Sf, n, hash(shape) % 1000 + len(count), f'tc {count}', expect=expect)


PAIR_COUNTS = [(f'rays={r}', lambda s, r=r: r) for r in range(1, 11)] + \
              [(f'pairs=3sms*{k}+{e}', lambda s, k=k, e=e: 2 * (3 * s * k + e) - (e % 2)) for k in (1, 2) for e in (0, 1, 2)]


@gpu
@pytest.mark.parametrize('count', [c for c, _ in PAIR_COUNTS])
@pytest.mark.parametrize('shape', [(48, 48), (64, 64), (8, 8)], ids=lambda s: f'{s[0]}+{s[1]}')
def test_tc_pairs_counts(shape, count):
    """render_fwd_tc_pairs_kernel with odd ray counts (the last pair without ray B), one to five pairs (groups of the only CTA
    idle), and 3 x grid x k + {0, 1, 2} pairs (the last wave with one to three groups busy)."""
    Sc, Sf = shape
    sms, _ = _device()
    n = dict(PAIR_COUNTS)[count](sms)

    def expect(p, sms):
        assert p['pairs'] == (n + 1) // 2 and p['grid'] == min(sms, (p['pairs'] + 2) // 3)

    _sweep('tc_pairs', Sc, Sf, n, 7 + n, f'tc_pairs {count}', expect=expect)


SIMT_SHAPES = [(9, 0, 'late_6'), (10, 6, 'late_6'), (13, 7, 'osg'), (255, 1, 'late_6')] + \
              [(sc, sf, 'late_6' if nets == 2 else 'osg') for sc, sf, nets in SIMT_REDUCED]


@gpu
@pytest.mark.parametrize('shape', SIMT_SHAPES, ids=lambda s: f'{s[0]}+{s[1]}-{s[2]}')
def test_simt_odd_counts_and_rt_reduction(shape):
    """render_fwd_kernel at sample counts that are not multiples of 8 (padded thread slots), S = 256, and the shapes whose
    shared memory makes the host reduce RT to keep two CTAs per SM; 3 x SMs + 2 tiles, ragged."""
    Sc, Sf, kind = shape
    sms, smem = _device()
    p = simt_plan(Sc, Sf, 2 if kind.startswith('late') else 1, 1, sms, smem)
    n = (3 * sms + 1) * p['RT'] + max(1, p['RT'] // 2)
    _sweep('simt', Sc, Sf, n, Sc + Sf, f'simt RT {p["RT0"]}->{p["RT"]}', kind_dec=kind)


@gpu
@pytest.mark.parametrize('white_back', [False, True], ids=['', 'white_back'])
@pytest.mark.parametrize('kind', DEC_KINDS)
@pytest.mark.parametrize('impl', ['tc', 'tc_pairs', 'simt'])
def test_decoder_kinds(impl, kind, white_back):
    """Every decoder layout describe_decoder maps (one or two nets, sigma from either, per-channel sigmoid masks), with and
    without white_back, on a multi-wave launch."""
    sms, _ = _device()
    n = (2 * sms + 3) * 8 + 3
    _sweep(impl, 48, 48, n, DEC_KINDS.index(kind), f'{impl} {kind} wb={int(white_back)}', kind_dec=kind, white_back=white_back)


@gpu
@pytest.mark.parametrize('impl', ['tc', 'tc_pairs', 'simt'])
def test_depth_clamp_across_ctas(impl):
    """A multi-wave launch with, in different tiles of CTA 0, a ray with non-monotone coarse depths and rays with a zero
    weight sum; the launch's largest depth sits in another CTA's tile and its smallest (negative) depth in a third. The
    zero-sum rays must come out at exactly the largest depth (NaN -> +inf -> clamp), and every clamped depth must equal the
    model's."""
    sms, smem = _device()
    Sc = Sf = 48
    p = plan(impl, Sc, Sf, 1, 10 ** 6, sms, smem)
    RT = p['RT']
    n = (3 * sms + 2) * RT
    grid = sms
    step = RT * grid                                           # rays between consecutive tiles of one CTA
    special = {0: 'nonmono', step + 1: 'empty', 2 * step + RT - 1: 'empty', 3 * step: 'nonmono',
               5 * RT + 2: 'max', 9 * RT + 1: 'min'}
    if impl == 'tc_pairs':                                     # pair p goes to CTA (p / 3) % grid
        step = 2 * 3 * grid
        n = 4 * step + 10
        special = {0: 'nonmono', step + 1: 'empty', 2 * step + 5: 'empty', 3 * step: 'nonmono', 5 * 6 + 2: 'max', 9 * 6 + 1: 'min'}
    L = clamp_scene(n, Sc, Sf, special, seed=11)
    got = run(L, impl)
    w = check(L, got)
    lo, hi = clamp_range(L, got['depths_fine'])
    empty = [r for r, k in special.items() if k == 'empty']
    assert (got['wsum'][empty] == 0).all() and (got['depth'][empty] == hi).all()
    assert lo < 0 and hi == 4.5 and (got['wsum'] > 0).sum() > n // 2
    print(f'{impl} clamp: range [{lo}, {hi}], {int((got["wsum"] == 0).sum())} zero-sum rays, {_fmt(plan(impl, Sc, Sf, 1, n, sms, smem))} '
          f'| {_fmt_worst(w)}')
    assert_within(w, 'clamp')


# ---------------------------------------------------------------------------------------------------------------------
# GPU: schedule invariance
# ---------------------------------------------------------------------------------------------------------------------
# Per-ray arithmetic does not depend on where a ray sits: a sample's features, hidden units and colours come from its own
# row of the MMA tiles, the march and the importance bookkeeping run one warp per ray on that ray's shared buffers, and a
# colour segment of g lanes starts at a sample index that is a multiple of g (g = pow2_group(S), and S and the 128-row tile
# are multiples of g), so its butterfly adds the same values in the same order wherever the ray lands. The per-ray sum of
# the segment partials runs over the same slots in the same order. The ray-pair kernel uses the same functions (gather,
# dec_hidden, dec_colours, warp_march, importance sampling, segment reduction with the same g), so it agrees with the
# row-tiled kernel bit for bit as well.
BIT_KEYS = ('feat', 'wsum', 'weights_final', 'perm', 'depths_fine', 'weights_coarse', 'inds')


def _same(a, b, keys=BIT_KEYS):
    for k in keys:
        if k in a:
            assert torch.equal(a[k].view(torch.int32) if a[k].dtype == torch.float32 else a[k],
                               b[k].view(torch.int32) if b[k].dtype == torch.float32 else b[k]), k


def _single_image(n, Sc, Sf, seed, kind='late_6'):
    L = scene(n, Sc, Sf, seed, kind)
    if L['B'] != 1:                                             # one image, so that any sub-range is a launch of its own
        L = scene(n + 1, Sc, Sf, seed, kind)
    return L


def _sub(L, lo, hi):
    """Rays lo..hi-1 of a one-image launch L as a launch of their own."""
    c = L['call']
    u = None if c['u'] is None else c['u'][lo:hi]
    return describe(c['planes'], L['module'], c['o'][:, lo:hi], c['d'][:, lo:hi], c['dc'][:, lo:hi], u, c['box_warp'],
                    c['white_back'])


@gpu
@pytest.mark.parametrize('impl,shape', [('tc', (48, 48)), ('tc', (40, 40)), ('tc', (96, 32)), ('tc_pairs', (64, 64)),
                                        ('simt', (13, 7))], ids=lambda v: v if isinstance(v, str) else f'{v[0]}+{v[1]}')
def test_shifted_launch_is_bit_identical(impl, shape):
    """Rays k..k+n-1 of one launch against rays 0..n-1 of the same draws, for every shift k in 1..RT-1 (another row, tile
    and CTA for each ray; the ray-pair kernel: the other half of a pair). The prefix repeats rays of the window, so the
    launch's depth range is the same and the depth must match as well."""
    Sc, Sf = shape
    sms, smem = _device()
    RT = plan(impl, Sc, Sf, 2, 1, sms, smem)['RT']
    n = (sms + 3) * RT + 1
    L = _single_image(n + RT, Sc, Sf, 21)
    base = _sub(L, RT, RT + n)
    ref = run(base, impl)
    for k in range(1, RT):
        c = L['call']
        idx = torch.cat([torch.arange(RT, RT + k), torch.arange(RT, RT + n)]).to(c['o'].device)    # k copies, then the window
        u = None if c['u'] is None else c['u'][idx]
        Lk = describe(c['planes'], L['module'], c['o'][:, idx], c['d'][:, idx], c['dc'][:, idx], u, 1.0)
        got = run(Lk, impl)
        tail = {key: v[k:] for key, v in got.items()}
        _same(tail, ref, BIT_KEYS + ('depth',))
    print(f'{impl} {Sc}+{Sf}: shifts 1..{RT - 1} of {n} rays bit-identical')


@gpu
@pytest.mark.parametrize('shape', [(48, 48), (40, 40), (120, 120)], ids=lambda s: f'{s[0]}+{s[1]}')
def test_one_tile_equals_its_rays_in_a_many_wave_launch(shape):
    """A one-tile launch of RT rays against the same rays inside a 3 x SMs + 2-tile launch, at tile 2 x SMs + 5 (CTA 5,
    third wave). Depths are compared where the clamp does not act."""
    Sc, Sf = shape
    sms, smem = _device()
    RT = tc_plan(Sc, Sf, 2, 1, sms, smem)['RT']
    t = 3 * sms + 2
    L = _single_image(t * RT, Sc, Sf, 5)
    at = (2 * sms + 5) * RT
    big = run(L, 'tc')
    small = run(_sub(L, at, at + RT), 'tc')
    win = {k: v[at:at + RT] for k, v in big.items()}
    _same(win, small)
    lo, hi = clamp_range(_sub(L, at, at + RT), small['depths_fine'])
    inner = (small['wsum'] > 0) & (small['depth'] > lo) & (small['depth'] < hi)
    assert inner.any() and torch.equal(win['depth'][inner], small['depth'][inner])


@gpu
@pytest.mark.parametrize('shape', [(48, 48), (64, 64), (8, 8)], ids=lambda s: f'{s[0]}+{s[1]}')
def test_tc_and_tc_pairs_agree_bit_for_bit(shape):
    """The row-tiled and the ray-pair tensor-core kernels compute every ray with the same operations in the same order."""
    Sc, Sf = shape
    sms, _ = _device()
    L = scene((3 * sms + 1) * 2 + 1, Sc, Sf, 9, 'late_1', white_back=True)
    a, b = run(L, 'tc'), run(L, 'tc_pairs')
    _same(a, b, BIT_KEYS + ('depth',))


# ---------------------------------------------------------------------------------------------------------------------
# GPU: replays of real synthesis steps
# ---------------------------------------------------------------------------------------------------------------------
def boundary_rays(kind, p, n, sample=1024, seed=0):
    """Every ray at a tile boundary (the first and last ray of each tile; the ray-pair kernel: every ray) plus a seeded
    sample of the others."""
    if kind == 'tc_pairs':
        return torch.arange(n)
    RT = p['RT']
    first = torch.arange(0, n, RT)
    last = torch.clamp(first + RT - 1, max=n - 1)
    edge = torch.unique(torch.cat([first, last]))
    rest = torch.ones(n, dtype=torch.bool)
    rest[edge] = False
    others = torch.nonzero(rest)[:, 0]
    g = torch.Generator().manual_seed(seed)
    pick = others[torch.randperm(others.numel(), generator=g)[:sample]]
    return torch.sort(torch.cat([edge, pick]))[0]


class _Replay:
    """Wraps native.pack_decoder (to keep the decoder module with its packed image) and native.render_fwd (the one call
    site behind ImportanceRenderer and the engine): every launch runs with its debug outputs and is checked against the
    model while its inputs are alive."""

    def __init__(self, monkeypatch):
        from pix2pix3d_b200 import native
        self.sms, self.smem = _device()
        self.rows, self.kinds = [], set()
        pack, render = native.pack_decoder, native.render_fwd

        def pack_decoder(decoder):
            pd = pack(decoder)
            pd.module = decoder
            return pd

        def render_fwd(planes_nhwc, dec, ray_origins, ray_dirs, depths_coarse, u, box_warp, white_back=False, debug=False, impl=None,
                       stratified=None, plane_index=None, **kw):
            res = render(planes_nhwc, dec, ray_origins, ray_dirs, depths_coarse, u, box_warp, white_back=white_back, debug=True,
                         impl=impl, stratified=stratified, plane_index=plane_index, **kw)
            self.check(res, planes_nhwc, dec, ray_origins, ray_dirs, depths_coarse, u, box_warp, white_back, impl, stratified,
                       plane_index)
            return res if debug else res[:3]

        monkeypatch.setattr(native, 'pack_decoder', pack_decoder)
        monkeypatch.setattr(native, 'render_fwd', render_fwd)

    def check(self, res, planes, dec, o, d, dc, u, box_warp, white_back, impl, stratified, plane_index):
        torch.cuda.synchronize()
        feat, depth, wsum, dbg = res
        L = describe(planes, dec.module, o, d, dc, u, box_warp, white_back, stratified, plane_index)
        n, Sc, Sf = L['n'], L['Sc'], L['Sf']
        kind = which_kernel(impl, Sc, Sf)
        p = plan(kind, Sc, Sf, len(L['nets']), n, self.sms, self.smem)
        got = dict(feat=feat.reshape(n, -1), depth=depth.reshape(n), wsum=wsum.reshape(n))
        got.update({k: v.reshape(n, -1) for k, v in dbg.items()})
        rays = boundary_rays(kind, p, n)
        w = check(L, got, rays)
        mode = 'explicit' if stratified is None else ('per-ray limits' if 'ray_start' in stratified else 'stratified')
        strided = not planes.is_contiguous()
        self.kinds |= {kind, mode} | ({'strided planes'} if strided else set()) | ({'white_back'} if white_back else set())
        self.rows.append(f'{len(self.rows):>2} B {L["B"]:>2} R {L["R"]:>6} {Sc}+{Sf} nets {len(L["nets"])} {mode:<10} '
                         f'{"strided" if strided else "dense":<7} wb {int(bool(white_back))} {_fmt(p)} checked {rays.numel():>6} '
                         f'| {_fmt_worst(w)}')
        assert_within(w, self.rows[-1])


@gpu
def test_replay_of_real_synthesis_steps(monkeypatch):
    """One eager G.synthesis step each of seg2cat_512 (48+48, tc), seg2face_512 (B = 16, 19 classes) and edge2car_128
    (64+64: the ray-pair kernel 'auto' picks, white_back), every render launch checked against the model on the planes
    read in place from the backbone's NHWC output, with in-kernel stratified depths. Prints the launch table."""
    from pix2pix3d_b200 import configs
    dev = torch.device('cuda')
    rp = _Replay(monkeypatch)
    for name in ('seg2cat_512', 'seg2face_512', 'edge2car_128'):
        wl = configs.WORKLOADS[name]
        G = configs.build_generator(name, seed=0, device=dev)
        c = configs.camera_labels(wl['batch'], 2, wl['preset']).to(dev)
        n0 = len(rp.rows)
        with torch.no_grad():
            ws = configs.synthetic_ws(wl['batch'], G.backbone.num_ws, 1).to(dev)
            torch.manual_seed(0)
            G.synthesis(ws, c, noise_mode='const', neural_rendering_resolution=wl['nrr'])
        torch.cuda.synchronize()
        print(f'# {name} (batch {wl["batch"]}), {rp.sms} SMs')
        print('\n'.join(rp.rows[n0:]))
        assert len(rp.rows) > n0, 'the step renders through native.render_fwd'
        del G
    missing = {'tc', 'tc_pairs', 'stratified', 'strided planes', 'white_back'} - rp.kinds
    assert not missing, missing
