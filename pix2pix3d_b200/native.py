"""Tensor-level wrappers over the C-ABI: allocate outputs with torch, pass raw device pointers.

These are the calls the reference-facing modules (training/..., torch_utils/ops/...) make; nothing here
has a CPU branch.
"""
import ctypes

import numpy as np
import torch

from . import _lib

PACKED_FLOATS = 2 * 4260
TC_PACKED_BYTES = 65536 + 324 * 4

# which fused renderer `render_fwd` uses: 'auto' (tensor-core decoder when the sample counts allow it), 'tc', 'simt',
# 'tc_pairs' (tensor-core decoder, ray-pair ownership: render_tc2.cu; sample counts <= 64)
render_impl = 'auto'

# when set to a list, timed_launch appends (tag, start_event, end_event, *extra) around its launch: render_fwd's
# ('render_fwd', start, end) and the convolutions' (tag, start, end, flops, tensor_flops) (bench.py)
kernel_events = None
# when set to a dict, every render_fwd call also writes the kernel's bookkeeping (importance indices, fine depths, sort
# permutation, interval weights) and leaves it there: lets tests score the bookkeeping of a whole G.synthesis call
render_debug_sink = None


def timed_launch(tag, name, *args, device, extra=(), unsupported_ok=False):
    """_lib.launch, bracketed by CUDA events when kernel_events is set; a launch the library ran is appended there as
    (tag, start, end, *extra)."""
    if kernel_events is None:
        return _lib.launch(name, *args, device=device, unsupported_ok=unsupported_ok)
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    ok = _lib.launch(name, *args, device=device, unsupported_ok=unsupported_ok)
    end.record()
    if ok:
        kernel_events.append((tag, start, end, *extra))
    return ok


def _f32c(t):
    assert t.is_cuda, 'native ops need CUDA tensors'
    if t.dtype != torch.float32:
        t = t.float()
    return t.contiguous()


def ray_sampler(cam2world, intrinsics, resolution):
    """RaySampler.forward -> (origins [B,M,3], dirs [B,M,3])."""
    c2w = _f32c(cam2world.reshape(-1, 16))
    K = _f32c(intrinsics.reshape(-1, 9))
    B = c2w.shape[0]
    M = resolution * resolution
    origins = torch.empty(B, M, 3, device=c2w.device, dtype=torch.float32)
    dirs = torch.empty_like(origins)
    _lib.launch('p3d_ray_sampler', c2w, K, B, resolution, origins, dirs, device=c2w.device)
    return origins, dirs


def planes_to_channels_last(planes):
    """[B,3,C,H,W] (or [N,C,H,W]) fp32 -> [B,3,H,W,C]."""
    p = _f32c(planes)
    shp = p.shape
    C, H, W = shp[-3], shp[-2], shp[-1]
    N = p.numel() // (C * H * W)
    out = torch.empty(*shp[:-3], H, W, C, device=p.device, dtype=torch.float32)
    _lib.launch('p3d_planes_to_channels_last', p, out, N, C, H, W, device=p.device)
    return out


class PackedDecoder:
    """Kernel-side weights of an OSG decoder plus its static description."""

    def __init__(self, packed, n_nets, sigma_net, masks, packed_tc=None):
        self.packed = packed
        self.packed_tc = packed_tc
        self.n_nets = n_nets
        self.sigma_net = sigma_net
        self.masks = masks
        self.out_channels = 32 * n_nets


def describe_decoder(decoder):
    """Map a decoder module onto (nets, sigma_net, sigmoid masks); None if the layout is not one of the
    OSG decoders the fused kernels implement (training/triplane.py:112, training/triplane_cond.py:859,926)."""
    name = type(decoder).__name__
    nets = []
    full = 0xFFFFFFFF
    if name == 'OSGDecoder':
        nets, sigma_net, masks = [decoder.net], 0, [full, 0]
    elif name == 'OSGDecoder_semantic':
        nets, sigma_net, masks = [decoder.net], 0, [full if decoder.final_sigmoid else 0, 0]
    elif name == 'OSGDecoder_semantic_lateSeparate':
        nets, sigma_net = [decoder.net, decoder.net_semantic], 1
        masks = [full, full if decoder.semantic_sigmoid else 0]
    elif name == 'OSGDecoder_semantic_entangle':
        if decoder.feature_sigmoid:
            m = full
        else:
            cs = int(decoder.semantic_channels)
            m = full & ~(((1 << cs) - 1) << 3)   # colour outputs 3..3+Cs-1 stay raw (triplane_cond.py:916-918)
        nets, sigma_net, masks = [decoder.net], 0, [m & full, 0]
    else:
        return None
    for net in nets:
        fc1, fc2 = net[0], net[2]
        if tuple(fc1.weight.shape) != (64, 32) or tuple(fc2.weight.shape) != (33, 64):
            return None
        if fc1.bias is None or fc2.bias is None:
            return None
    return nets, sigma_net, masks


def pack_decoder(decoder):
    desc = describe_decoder(decoder)
    if desc is None:
        raise NotImplementedError(f'no fused kernel for decoder type {type(decoder).__name__}')
    nets, sigma_net, masks = desc
    dev = nets[0][0].weight.device
    d = _lib.DecoderDesc()
    d.n_nets = len(nets)
    d.sigma_net = sigma_net
    keep = []
    for i, net in enumerate(nets):
        fc1, fc2 = net[0], net[2]
        w1, b1, w2, b2 = (_f32c(t.detach()) for t in (fc1.weight, fc1.bias, fc2.weight, fc2.bias))
        keep += [w1, b1, w2, b2]
        d.w1[i], d.b1[i], d.w2[i], d.b2[i] = w1.data_ptr(), b1.data_ptr(), w2.data_ptr(), b2.data_ptr()
        d.w1_gain[i], d.b1_gain[i] = float(fc1.weight_gain), float(fc1.bias_gain)
        d.w2_gain[i], d.b2_gain[i] = float(fc2.weight_gain), float(fc2.bias_gain)
        d.sigmoid_mask[i] = masks[i]
    packed = torch.empty(PACKED_FLOATS, device=dev, dtype=torch.float32)
    _lib.launch('p3d_pack_decoder', ctypes.byref(d), packed, device=dev)
    packed_tc = torch.empty(TC_PACKED_BYTES, device=dev, dtype=torch.uint8)
    _lib.launch('p3d_pack_decoder_tc', ctypes.byref(d), packed_tc, device=dev)
    del keep
    return PackedDecoder(packed, len(nets), sigma_net, masks, packed_tc)


def ray_limits_box(rays_o, rays_d, box_side_length):
    """math_utils.get_ray_limits_box on CUDA tensors: (t_near, t_far) of shape [..., 1]."""
    lead = rays_o.shape[:-1]
    o, d = _f32c(rays_o.detach().reshape(-1, 3)), _f32c(rays_d.detach().reshape(-1, 3))
    n = o.shape[0]
    tn = torch.empty(n, device=o.device, dtype=torch.float32)
    tf = torch.empty(n, device=o.device, dtype=torch.float32)
    _lib.launch('p3d_ray_limits_box', o, d, n, float(box_side_length), tn, tf, device=o.device)
    return tn.reshape(*lead, 1), tf.reshape(*lead, 1)


def _out_view(buf, shape, dtype, dev):
    """The leading elements of a caller's flat output buffer, viewed as `shape`."""
    n = int(np.prod(shape))
    assert buf.dtype == dtype and buf.device == dev and buf.is_contiguous() and buf.numel() >= n, 'out= buffer'
    return buf.reshape(-1)[:n].view(shape)


def _in_place_strides(planes_nhwc):
    """(image, plane, pixel) element strides of a non-contiguous [B,3,H,W,32] plane view that the tensor-core kernels read in
    place: channels contiguous and rows W pixels apart (e.g. the backbone's NHWC [B,H,W,96] output viewed as
    [B,3,H,W,32]). None for a contiguous tensor and for any other view, which is made dense first."""
    if planes_nhwc.is_contiguous():
        return None
    st_img, st_plane, st_row, st_pix, st_ch = planes_nhwc.stride()
    if st_ch == 1 and st_row == planes_nhwc.shape[3] * st_pix and st_pix >= 32 and st_plane > 0 and st_img > 0:
        return st_img, st_plane, st_pix
    return None


def render_fwd(planes_nhwc, dec, ray_origins, ray_dirs, depths_coarse, u, box_warp, white_back=False, debug=False, impl=None,
               stratified=None, plane_index=None, out=None):
    """Fused ImportanceRenderer.forward. Returns (feat [B,R,C], depth [B,R,1], wsum [B,R,1][, debug dict]).
    `stratified` (instead of `depths_coarse`): the ingredients of sample_stratified, combined inside the kernel --
    dict(jitter=[B,R,Sc] U[0,1) draw, table=[Sc], delta=float) for scalar ray limits or dict(jitter, table, ray_start=[B,R],
    ray_end=[B,R]) for per-ray limits (p3d_render_args_t::depth_mode 1 / 2).
    `plane_index` ([B] int32): plane set of each image; lets B views share fewer plane sets (planes batch < B).
    `out` (optional dict): contiguous buffers to write instead of fresh ones, keyed like the outputs and the debug dict
    (feat, depth, wsum, weights_final, perm, weights_coarse, depths_fine, inds); each may be longer than the launch needs,
    and the launch writes only its leading elements. `out['depths_sorted']` additionally asks for the merged depths in sorted
    order, [B,R,Sc+Sf] (what render_bwd recomputes a ray from); no other output changes when it is given."""
    Bp, _, H, W, C = planes_nhwc.shape
    B = ray_origins.shape[0]
    if plane_index is None and Bp != B:
        raise ValueError('planes batch and ray batch differ: pass plane_index')
    assert C == 32 and planes_nhwc.dtype == torch.float32
    impl = impl or render_impl
    strides = None if impl == 'simt' else _in_place_strides(planes_nhwc)
    if strides is None:
        planes_nhwc = planes_nhwc.contiguous()
    strided = strides is not None
    R = ray_origins.shape[1]
    o, d = _f32c(ray_origins), _f32c(ray_dirs)
    keep = []
    if stratified is not None:
        jit = _f32c(stratified['jitter']).reshape(B, R, -1)
        Sc = jit.shape[-1]
        table = _f32c(stratified['table']).reshape(-1)
        assert table.numel() == Sc
        dc = None
    else:
        dc = _f32c(depths_coarse).reshape(B, R, -1)
        Sc = dc.shape[-1]
    Sf = 0 if u is None else int(u.shape[-1])
    uu = None if u is None else _f32c(u)
    dev = planes_nhwc.device
    out = out or {}
    feat = _alloc(out.get('feat'), (B, R, dec.out_channels), dev)
    depth = _alloc(out.get('depth'), (B, R, 1), dev)
    wsum = _alloc(out.get('wsum'), (B, R, 1), dev)
    ws = torch.empty(4, device=dev, dtype=torch.int32)
    a = _lib.RenderArgs()
    a.planes_nhwc, a.ray_origins, a.ray_dirs = planes_nhwc.data_ptr(), o.data_ptr(), d.data_ptr()
    if dc is not None:
        a.depths_coarse = dc.data_ptr()
    else:
        a.jitter, a.depth_table = jit.data_ptr(), table.data_ptr()
        if 'ray_start' in stratified:
            rs, re_ = _f32c(stratified['ray_start']).reshape(B, R), _f32c(stratified['ray_end']).reshape(B, R)
            keep += [rs, re_]
            a.depth_mode, a.ray_start, a.ray_end = 2, rs.data_ptr(), re_.data_ptr()
            a.depth_delta = float(np.float32(1.0) / np.float32(Sc - 1))      # what `tensor / (Sc - 1)` multiplies by on CUDA
        else:
            a.depth_mode, a.depth_delta = 1, float(stratified['delta'])
    if plane_index is not None:
        pidx = plane_index.to(device=planes_nhwc.device, dtype=torch.int32).contiguous()
        assert pidx.numel() == B
        keep.append(pidx)
        a.plane_index = pidx.data_ptr()
    a.u_importance = None if uu is None else uu.data_ptr()
    a.decoder_packed = dec.packed.data_ptr()
    a.n_nets, a.sigma_net = dec.n_nets, dec.sigma_net
    a.sigmoid_mask[0], a.sigmoid_mask[1] = dec.masks[0], dec.masks[1]
    a.B, a.R, a.H, a.W, a.Sc, a.Sf = B, R, H, W, Sc, Sf         # B = images of rays; plane sets may be fewer (plane_index)
    a.coord_scale = 2.0 / float(box_warp)
    a.white_back = 1 if white_back else 0
    a.out_feat, a.out_depth, a.out_wsum = feat.data_ptr(), depth.data_ptr(), wsum.data_ptr()
    dbg = {}
    want_debug = debug or render_debug_sink is not None
    if want_debug:
        S = Sc + Sf
        dbg['weights_final'] = _alloc(out.get('weights_final'), (B, R, S - 1), dev)
        dbg['perm'] = _alloc(out.get('perm'), (B, R, S), dev, torch.int32)
        a.dbg_weights_final, a.dbg_perm = dbg['weights_final'].data_ptr(), dbg['perm'].data_ptr()
        if Sf > 0:
            dbg['weights_coarse'] = _alloc(out.get('weights_coarse'), (B, R, Sc - 1), dev)
            dbg['depths_fine'] = _alloc(out.get('depths_fine'), (B, R, Sf), dev)
            dbg['inds'] = _alloc(out.get('inds'), (B, R, Sf), dev, torch.int32)
            a.dbg_weights_coarse = dbg['weights_coarse'].data_ptr()
            a.dbg_depths_fine, a.dbg_inds = dbg['depths_fine'].data_ptr(), dbg['inds'].data_ptr()
    if 'depths_sorted' in out:
        a.out_depths_sorted = _alloc(out['depths_sorted'], (B, R, Sc + Sf), dev).data_ptr()
    a.workspace = ws.data_ptr()
    if strided:
        a.plane_strides[0], a.plane_strides[1], a.plane_strides[2] = strides
    use_tc = impl in ('auto', 'tc', 'tc_pairs') and Sc % 8 == 0 and Sf % 8 == 0 and Sc <= 128 and Sf <= 128 and dec.packed_tc is not None
    if impl in ('tc', 'tc_pairs') and not use_tc:
        raise ValueError('tensor-core renderer needs sample counts that are multiples of 8')
    # ray-pair ownership fills its 64-row halves only at 64 samples per pass; at fewer samples per ray the row-tiled kernel
    # packs its tiles densely and the pair kernel would leave rows idle
    a.tc_variant = 1 if (impl == 'tc_pairs' or (impl == 'auto' and Sc == 64 and Sf == 64)) else 0
    if use_tc:
        a.decoder_packed = dec.packed_tc.data_ptr()
    elif strided:   # the SIMT kernel reads dense planes only
        dense = planes_nhwc.contiguous()
        a.planes_nhwc = dense.data_ptr()
        a.plane_strides[0] = a.plane_strides[1] = a.plane_strides[2] = 0
    timed_launch('render_fwd', 'p3d_render_fwd_tc' if use_tc else 'p3d_render_fwd', ctypes.byref(a), device=dev)
    if render_debug_sink is not None:
        render_debug_sink.update(dbg, feat=feat, depth=depth, wsum=wsum)
    if debug:
        return feat, depth, wsum, dbg
    return feat, depth, wsum


def render_bwd(planes_nhwc, params, sigma_net, masks, ray_origins, ray_dirs, depths_sorted, Sc, Sf, box_warp, g_feat, g_depth=None,
               g_wsum=None, depth_range=None, white_back=False, want_planes=True, want_params=True, out=None):
    """First-order backward of render_fwd (p3d_render_bwd): recomputes every ray from the planes [B,3,H,W,32], its sorted
    depths [B,R,Sc+Sf] (render_fwd's out['depths_sorted']) and the decoder's EFFECTIVE parameters `params` (per net
    (w1, b1, w2, b2) with the gains applied, as _effective_fc forms them). g_feat [B,R,C]; g_depth / g_wsum [B,R(,1)] or None;
    depth_range: device [2] = (min, max) of all depths, needed with g_depth. Returns (dL/dplanes [B,3,H,W,32] or None,
    dL/dparams [n_nets,4257] = w1 | b1 | w2 | b2 per net, or None). `out`: optional dict of buffers keyed planes, params
    (see _alloc) and workspace (the per-CTA parameter partials; its whole length is passed to the launch)."""
    B, _, H, W, C = planes_nhwc.shape
    assert C == 32 and planes_nhwc.dtype == torch.float32
    p = _f32c(planes_nhwc)
    R = ray_origins.shape[1]
    o, d = _f32c(ray_origins), _f32c(ray_dirs)
    ds = _f32c(depths_sorted).reshape(B, R, Sc + Sf)
    gf = _f32c(g_feat).reshape(B, R, -1)
    n_nets = len(params)
    assert gf.shape[-1] == 32 * n_nets
    keep = [p, o, d, ds, gf]
    a = _lib.RenderBwdArgs()
    a.planes_nhwc, a.ray_origins, a.ray_dirs, a.depths_sorted = p.data_ptr(), o.data_ptr(), d.data_ptr(), ds.data_ptr()
    for i, net in enumerate(params):
        w1, b1, w2, b2 = (_f32c(t.detach()) for t in net)
        keep += [w1, b1, w2, b2]
        a.w1[i], a.b1[i], a.w2[i], a.b2[i] = w1.data_ptr(), b1.data_ptr(), w2.data_ptr(), b2.data_ptr()
        a.sigmoid_mask[i] = masks[i]
    a.n_nets, a.sigma_net = n_nets, sigma_net
    a.B, a.R, a.H, a.W, a.Sc, a.Sf = B, R, H, W, Sc, Sf
    a.coord_scale = 2.0 / float(box_warp)
    a.white_back = 1 if white_back else 0
    a.g_feat = gf.data_ptr()
    for name, t in (('g_depth', g_depth), ('g_wsum', g_wsum), ('depth_range', depth_range)):
        if t is not None:
            t = _f32c(t)
            keep.append(t)
            setattr(a, name, t.data_ptr())
    dev = p.device
    out = out or {}
    g_planes = _alloc(out.get('planes'), (B, 3, H, W, 32), dev) if want_planes else None
    g_params = None
    if want_params:
        g_params = _alloc(out.get('params'), (n_nets, DECODER_PARAM_FLOATS), dev)
        ws = out.get('workspace')
        if ws is None:
            ws = torch.empty(_lib.lib().p3d_render_bwd_workspace_floats(n_nets), device=dev, dtype=torch.float32)
        else:
            assert ws.dtype == torch.float32 and ws.device == dev and ws.is_contiguous(), 'out= buffer'
        a.g_params, a.workspace, a.workspace_floats = g_params.data_ptr(), ws.data_ptr(), ws.numel()
    if want_planes:
        a.g_planes_nhwc = g_planes.data_ptr()
    _lib.launch('p3d_render_bwd', ctypes.byref(a), device=dev, launches=1 + (n_nets if want_params else 0))
    return g_planes, g_params


def run_model(planes_nhwc, dec, coords, box_warp, impl=None, sigma_only=False):
    """Fused sample_from_planes + decoder: coords [B,M,3] -> (rgb [B,M,C], sigma [B,M,1]).

    `impl`: 'auto' / 'tc' run the tensor-core query (p3d_run_model_tc), 'simt' the CUDA-core kernel.
    `sigma_only` (tensor-core query): skip the colours and return (None, sigma) -- the mesh-extraction query."""
    B, _, H, W, C = planes_nhwc.shape
    assert C == 32 and planes_nhwc.dtype == torch.float32
    impl = impl or render_impl
    use_tc = impl in ('auto', 'tc', 'tc_pairs') and dec.packed_tc is not None
    strides = _in_place_strides(planes_nhwc) if use_tc else None
    if strides is None:
        planes_nhwc = planes_nhwc.contiguous()
    else:
        strides = (ctypes.c_int64 * 3)(*strides)
    c = _f32c(coords)
    M = c.shape[1]
    dev = planes_nhwc.device
    sigma_only = bool(sigma_only) and use_tc
    rgb = None if sigma_only else torch.empty(B, M, dec.out_channels, device=dev, dtype=torch.float32)
    sigma = torch.empty(B, M, 1, device=dev, dtype=torch.float32)
    masks = (ctypes.c_uint32 * 2)(dec.masks[0], dec.masks[1])
    if use_tc:
        _lib.launch('p3d_run_model_tc', planes_nhwc, strides, c, dec.packed_tc, dec.n_nets, dec.sigma_net, masks, B, M, H, W,
                    2.0 / float(box_warp), rgb, sigma, device=dev)
    else:
        _lib.launch('p3d_run_model', planes_nhwc, c, dec.packed, dec.n_nets, dec.sigma_net, masks, B, M, H, W,
                    2.0 / float(box_warp), rgb, sigma, device=dev)
    return rgb, sigma


def _alloc(out, shape, dev, dtype=torch.float32):
    """A fresh tensor, or the leading elements of the caller's flat buffer `out` (tests prefill longer buffers and check that a
    launch writes nothing past its own elements)."""
    return torch.empty(*shape, device=dev, dtype=dtype) if out is None else _out_view(out, shape, dtype, dev)


def sample_from_planes(planes_nhwc, coords, box_warp, out=None):
    """coords [B,M,3] -> features [B,3,M,32] (reference layout of sample_from_planes). `out`: optional buffer (see _alloc)."""
    B, _, H, W, _ = planes_nhwc.shape
    c = _f32c(coords)
    M = c.shape[1]
    out = _alloc(out, (B, 3, M, 32), planes_nhwc.device)
    _lib.launch('p3d_sample_from_planes', planes_nhwc, c, B, M, H, W, 2.0 / float(box_warp), out, device=planes_nhwc.device)
    return out


def ray_march(colors, densities, depths, white_back=False, out=None):
    """MipRayMarcher2.run_forward on [B,R,S,C] / [B,R,S,1] / [B,R,S,1] tensors. `out`: optional dict of buffers keyed rgb,
    depth, weights (see _alloc)."""
    B, R, S, Cc = colors.shape
    col, den, dep = _f32c(colors), _f32c(densities), _f32c(depths)
    dev = col.device
    out = out or {}
    rgb = _alloc(out.get('rgb'), (B, R, Cc), dev)
    depth = _alloc(out.get('depth'), (B, R, 1), dev)
    weights = _alloc(out.get('weights'), (B, R, S - 1, 1), dev)
    ws = torch.empty(4, device=dev, dtype=torch.int32)
    _lib.launch('p3d_ray_march', col, den, dep, B * R, S, Cc, 1 if white_back else 0, rgb, depth, weights, ws, device=dev)
    return rgb, depth, weights


def sample_from_planes_bwd(grad_features, coords, box_warp, H, W, out=None):
    """grad_features [B,3,M,32] -> gradient w.r.t. channels-last planes [B,3,H,W,32]. `out`: optional buffer (see _alloc)."""
    g = _f32c(grad_features)
    c = _f32c(coords)
    B, _, M, _ = g.shape
    out = _alloc(out, (B, 3, H, W, 32), g.device)
    _lib.launch('p3d_sample_from_planes_bwd', g, c, B, M, H, W, 2.0 / float(box_warp), out, device=g.device)
    return out


def ray_march_bwd(colors, densities, depths, g_rgb, g_depth, g_weights, depth_range, white_back=False, out=None):
    """Gradients of MipRayMarcher2.run_forward w.r.t. colors [B,R,S,C] and densities [B,R,S,1]. `out`: optional dict of
    buffers keyed colors, densities (see _alloc)."""
    B, R, S, Cc = colors.shape
    col, den, dep = _f32c(colors), _f32c(densities), _f32c(depths)
    grgb = _f32c(g_rgb)
    gdep = None if g_depth is None else _f32c(g_depth)
    gw = None if g_weights is None else _f32c(g_weights)
    rng = None if depth_range is None else _f32c(depth_range)
    out = out or {}
    g_col = _alloc(out.get('colors'), tuple(col.shape), col.device)
    g_den = _alloc(out.get('densities'), tuple(den.shape), col.device)
    _lib.launch('p3d_ray_march_bwd', col, den, dep, grgb, gdep, gw, rng, B * R, S, Cc, 1 if white_back else 0, g_col, g_den,
                device=col.device)
    return g_col, g_den


def sample_importance(z_vals, weights, u, return_inds=False, out=None):
    """z_vals [N,S], weights [N,S-1], u [N,Sf] -> samples [N,Sf] (and searchsorted indices). `out`: optional dict of buffers
    keyed samples, inds (see _alloc)."""
    z, w, uu = _f32c(z_vals), _f32c(weights), _f32c(u)
    N, S = z.shape
    Sf = uu.shape[1]
    bufs = out or {}
    out = _alloc(bufs.get('samples'), (N, Sf), z.device)
    inds = _alloc(bufs.get('inds'), (N, Sf), z.device, torch.int32) if return_inds else None
    _lib.launch('p3d_sample_importance', z, w, uu, N, S, Sf, out, inds, device=z.device)
    return (out, inds) if return_inds else out


# ----------------------------------------------------------------------------------------------
# OSG decoder MLP of the gradient-requiring passes (p3d_decoder_mlp_fwd / _bwd)
# ----------------------------------------------------------------------------------------------
DECODER_PARAM_FLOATS = 64 * 32 + 64 + 33 * 64 + 33


def decoder_mlp_fwd(feats, w1, b1, w2, b2, mask, want_saved=False, out=None):
    """One p3d_decoder_mlp_fwd launch: feats [N,3,M,32] and EFFECTIVE parameters -> dict(rgb [N,M,32], sigma [N,M,1]); with
    `want_saved` also pre [N*M,64] (hidden pre-activations) and, when `mask` is not 0, sig [N*M,32] (sigmoid values of the masked
    channels), which decoder_mlp_bwd consumes. `out`: optional dict of buffers under the same keys (see _alloc)."""
    f, w1c, b1c, w2c, b2c = (_f32c(t.detach()) for t in (feats, w1, b1, w2, b2))
    n, _, m, _ = f.shape
    out = out or {}
    r = dict(rgb=_alloc(out.get('rgb'), (n, m, 32), f.device), sigma=_alloc(out.get('sigma'), (n, m, 1), f.device))
    if want_saved:
        r['pre'] = _alloc(out.get('pre'), (n * m, 64), f.device)
        if mask:
            r['sig'] = _alloc(out.get('sig'), (n * m, 32), f.device)
    _lib.launch('p3d_decoder_mlp_fwd', f, n, m, w1c, b1c, w2c, b2c, int(mask), r['rgb'], r['sigma'], r.get('pre'), r.get('sig'),
                device=f.device)
    return r


def decoder_mlp_bwd(feats, w1, b1, w2, b2, mask, pre, sig, g_rgb, g_sigma, out=None):
    """One p3d_decoder_mlp_bwd launch: the forward's inputs, its saved pre / sig (decoder_mlp_fwd with want_saved) and the upstream
    gradients g_rgb [N,M,32] / g_sigma [N,M,1] (either may be None) -> dict(feats = dL/dfeats [N,3,M,32], params = dL/d(w1 | b1 |
    w2 | b2) [4257]). `out`: optional dict of buffers keyed feats, params (see _alloc)."""
    f, w1c, b1c, w2c, b2c = (_f32c(t.detach()) for t in (feats, w1, b1, w2, b2))
    n, _, m, _ = f.shape
    gr = None if g_rgb is None else _f32c(g_rgb)
    gs = None if g_sigma is None else _f32c(g_sigma)
    out = out or {}
    g_feats = _alloc(out.get('feats'), tuple(f.shape), f.device)
    g_params = _alloc(out.get('params'), (DECODER_PARAM_FLOATS,), f.device)
    nws = _lib.lib().p3d_decoder_mlp_bwd_workspace_floats()
    ws = torch.empty(nws, device=f.device, dtype=torch.float32)
    _lib.launch('p3d_decoder_mlp_bwd', f, pre, sig, n, m, w1c, b1c, w2c, b2c, int(mask), gr, gs, g_feats, g_params, ws, nws,
                device=f.device, launches=2)
    return dict(feats=g_feats, params=g_params)


class _DecoderMLP(torch.autograd.Function):
    """feats [N,3,M,32] -> (rgb [N,M,32], sigma [N,M,1]) through mean(1) -> FC(32,64) -> softplus -> FC(64,33) [-> sigmoid], forward
    and first-order backward on libp3d. w1 / b1 / w2 / b2 are the EFFECTIVE parameters (runtime gains applied by the caller under
    autograd), so their gradients flow on to the module's parameters through ordinary torch ops."""

    @staticmethod
    def forward(ctx, feats, w1, b1, w2, b2, mask):
        f, w1c, b1c, w2c, b2c = (_f32c(t.detach()) for t in (feats, w1, b1, w2, b2))
        # the hidden pre-activations (256 bytes per point) and the sigmoid values (128) for the backward pass, only when a
        # gradient can be asked for
        grad = any(ctx.needs_input_grad)
        r = decoder_mlp_fwd(f, w1c, b1c, w2c, b2c, int(mask), want_saved=grad)
        if grad:
            ctx.save_for_backward(f, w1c, b1c, w2c, b2c, r['pre'], r.get('sig'))
        ctx.mask = int(mask)
        return r['rgb'], r['sigma']

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g_rgb, g_sigma):
        f, w1, b1, w2, b2, pre, sig = ctx.saved_tensors
        g = decoder_mlp_bwd(f, w1, b1, w2, b2, ctx.mask, pre, sig, g_rgb, g_sigma)
        g_feats, g_params = g['feats'], g['params']
        gw1, gb1, gw2, gb2 = torch.split(g_params, [64 * 32, 64, 33 * 64, 33])
        return g_feats, gw1.view(64, 32), gb1, gw2.view(33, 64), gb2, None


def _effective_fc(fc):
    """weight * weight_gain, bias * bias_gain as FullyConnectedLayer.forward forms them (networks_stylegan2.py:111-119)."""
    w = fc.weight.to(torch.float32) * fc.weight_gain
    b = fc.bias.to(torch.float32)
    if fc.bias_gain != 1:
        b = b * fc.bias_gain
    return w, b


def decoder_mlp_supported(decoder, sampled_features):
    """True when `decoder(sampled_features, ...)` can run on p3d_decoder_mlp_*: a CUDA fp32 [N,3,M,32] feature tensor and one of the
    OSG decoder layouts the kernels implement."""
    f = sampled_features
    return (f.is_cuda and f.dtype == torch.float32 and f.ndim == 4 and f.shape[1] == 3 and f.shape[3] == 32 and f.numel() > 0
            and describe_decoder(decoder) is not None)


def decoder_mlp(decoder, sampled_features):
    """The OSG decoder modules' forward ({'rgb', 'sigma'}) on the fused kernels, differentiable to first order w.r.t. the features
    and the decoder parameters (training/triplane.py:122-135, triplane_cond.py:869-970)."""
    nets, sigma_net, masks = describe_decoder(decoder)
    outs = []
    for net, mask in zip(nets, masks):
        w1, b1 = _effective_fc(net[0])
        w2, b2 = _effective_fc(net[2])
        outs.append(_DecoderMLP.apply(sampled_features, w1, b1, w2, b2, mask))
    sigma = outs[sigma_net][1]
    rgb = outs[0][0] if len(outs) == 1 else torch.cat([o[0] for o in outs], dim=-1)
    return {'rgb': rgb, 'sigma': sigma}


def fc_bias_act(x, weight, bias, weight_gain, bias_gain, act, alpha, act_gain):
    """FullyConnectedLayer.forward on p3d_fc_bias_act: x [B,in] fp32 (no gradients), act = p3d_bias_act code."""
    xc, wc = _f32c(x.detach()), _f32c(weight.detach())
    bc = None if bias is None else _f32c(bias.detach())
    y = torch.empty(xc.shape[0], wc.shape[0], device=xc.device, dtype=torch.float32)
    _lib.launch('p3d_fc_bias_act', xc, wc, bc, y, xc.shape[0], xc.shape[1], wc.shape[0], float(weight_gain), float(bias_gain),
                int(act), float(alpha), float(act_gain), device=xc.device)
    return y
