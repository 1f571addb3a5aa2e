"""Two-pass (stratified + importance) tri-plane volume renderer.

Mirror of the reference's training/volumetric_rendering/renderer.py: `generate_planes` (:23),
`project_onto_planes` (:39), `sample_from_planes` (:55), `ImportanceRenderer` (:82-253) keep their signatures.
On CUDA, `ImportanceRenderer.forward` is ONE persistent kernel (`p3d_render_fwd`, pix2pix3d_b200/csrc/render.cu) fed with
the same two random tensors the reference draws (stratified jitter, importance u), in the same order, so the RNG stream is
consumed identically. When the planes or the decoder require grad, the same launch runs under `_FusedRender`, whose backward
is one recompute kernel (`p3d_render_bwd`, csrc/render_fused_bwd.cu). Anything the fused kernels do not cover (density noise,
rays that require grad, unknown decoders) takes the stage-by-stage formulation below, which is also what CPU tensors use.
"""
import torch

from ... import native
from . import math_utils
from .ray_marcher import MipRayMarcher2


def generate_planes():
    """Axes of the three feature planes, [3,3,3] (:23-37). The third plane keeps EG3D's original axis order."""
    return torch.tensor([[[1, 0, 0], [0, 1, 0], [0, 0, 1]],
                         [[1, 0, 0], [0, 0, 1], [0, 1, 0]],
                         [[0, 0, 1], [1, 0, 0], [0, 1, 0]]], dtype=torch.float32)


def project_onto_planes(planes, coordinates):
    """coordinates [N,M,3] -> [N*n_planes, M, 2] plane coordinates (:39-53)."""
    n, m, _ = coordinates.shape
    n_planes = planes.shape[0]
    inv = torch.linalg.inv(planes)                                   # [P,3,3]
    proj = torch.einsum('nmc,pcd->npmd', coordinates, inv)           # [N,P,M,3]
    return proj.reshape(n * n_planes, m, 3)[..., :2]


def sample_from_planes(plane_axes, plane_features, coordinates, mode='bilinear', padding_mode='zeros', box_warp=None):
    """plane_features [N,P,C,H,W], coordinates [N,M,3] -> [N,P,M,C] bilinear samples (:55-65)."""
    assert padding_mode == 'zeros'
    n, n_planes, c, h, w = plane_features.shape
    m = coordinates.shape[1]
    no_grad = not (torch.is_grad_enabled() and (plane_features.requires_grad or coordinates.requires_grad))
    if (plane_features.device.type == 'cuda' and mode == 'bilinear' and n_planes == 3 and c == 32
            and plane_features.dtype == torch.float32 and _is_default_axes(plane_axes)):
        if no_grad:
            return native.sample_from_planes(native.planes_to_channels_last(plane_features), coordinates, box_warp)
        if not coordinates.requires_grad:          # training: gradients reach the planes only (rays come from the camera label)
            return _SamplePlanes.apply(plane_features, coordinates, float(box_warp))
    feats = plane_features.reshape(n * n_planes, c, h, w)
    coords = (2 / box_warp) * coordinates
    grid = project_onto_planes(plane_axes, coords).unsqueeze(1)
    out = torch.nn.functional.grid_sample(feats, grid.to(feats.dtype), mode=mode, padding_mode=padding_mode, align_corners=False)
    return out.permute(0, 3, 2, 1).reshape(n, n_planes, m, c)


class _SamplePlanes(torch.autograd.Function):
    """Tri-plane lookup with its first-order backward on the kernels: p3d_sample_from_planes forward, p3d_sample_from_planes_bwd
    (scatter of the bilinear taps) backward. Coordinates are not differentiated."""

    @staticmethod
    def forward(ctx, plane_features, coordinates, box_warp):
        ctx.save_for_backward(coordinates)
        ctx.box_warp = box_warp
        ctx.plane_shape = tuple(plane_features.shape)
        return native.sample_from_planes(native.planes_to_channels_last(plane_features.detach()), coordinates, box_warp)

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_out):
        from ... import tcconv
        (coordinates,) = ctx.saved_tensors
        n, p, c, h, w = ctx.plane_shape
        g_cl = native.sample_from_planes_bwd(grad_out, coordinates, ctx.box_warp, h, w)          # [N,3,H,W,32]
        g = tcconv.nhwc_to_nchw_f32(g_cl.view(n * p, h, w, c))                                   # [N*3,32,H,W]
        return g.view(n, p, c, h, w), None, None


def sample_from_3dgrid(grid, coordinates):
    """grid [1|N,C,H,W,D], coordinates [N,M,3] -> [N,M,C] trilinear samples (:67-80)."""
    n, m, dims = coordinates.shape
    out = torch.nn.functional.grid_sample(grid.expand(n, -1, -1, -1, -1), coordinates.reshape(n, 1, 1, -1, dims),
                                          mode='bilinear', padding_mode='zeros', align_corners=False)
    nn_, c, h, w, d = out.shape
    return out.permute(0, 4, 3, 2, 1).reshape(nn_, h * w * d, c)


_DEFAULT_AXES = generate_planes()


# the gradient-requiring fused path (_FusedRender); tests switch it off to compare against the staged chain
fused_grad = True


class _FusedRender(torch.autograd.Function):
    """ImportanceRenderer.forward on the fused kernels, differentiable to first order w.r.t. the planes and the decoder's
    effective parameters (`params`: w1, b1, w2, b2 per net with the gains applied, so autograd carries the gains on to the
    module parameters as native.decoder_mlp does). Saves only the channels-last planes and the sorted sample depths; the
    backward (p3d_render_bwd) recomputes each ray from them."""

    @staticmethod
    def forward(ctx, planes, call, *params):
        planes_cl = native.planes_to_channels_last(planes.detach())
        b, r = call['ray_origins'].shape[:2]
        depths_sorted = torch.empty(b, r, call['Sc'] + call['Sf'], device=planes.device, dtype=torch.float32)
        feat, depth, wsum = native.render_fwd(planes_cl, call['dec'], call['ray_origins'], call['ray_directions'],
                                              call['depths_coarse'], call['u'], call['box_warp'], white_back=call['white_back'],
                                              out={'depths_sorted': depths_sorted}, **call['kw'])
        ctx.set_materialize_grads(False)
        ctx.save_for_backward(planes_cl, depths_sorted, call['ray_origins'], call['ray_directions'], *params)
        ctx.call = {k: call[k] for k in ('sigma_net', 'masks', 'Sc', 'Sf', 'box_warp', 'white_back')}
        ctx.n_params = len(params)
        ctx.plane_shape = tuple(planes.shape)
        return feat, depth, wsum

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g_feat, g_depth, g_wsum):
        from ... import tcconv
        planes_cl, depths_sorted, o, d, *flat = ctx.saved_tensors
        c = ctx.call
        n_nets = ctx.n_params // 4
        none = (None,) * (2 + ctx.n_params)
        if g_feat is None and g_depth is None and g_wsum is None:
            return none
        b, r = o.shape[:2]
        if g_feat is None:
            g_feat = torch.zeros(b, r, 32 * n_nets, device=o.device, dtype=torch.float32)
        rng = None
        if g_depth is not None:
            lo, hi = torch.aminmax(depths_sorted)               # the clamp range of the depth output (as _RayMarch.backward)
            rng = torch.stack([lo, hi])
        want_planes = ctx.needs_input_grad[0]
        want_params = any(ctx.needs_input_grad[2:])
        if not (want_planes or want_params):
            return none
        params = [flat[4 * i:4 * i + 4] for i in range(n_nets)]
        g_cl, g_par = native.render_bwd(planes_cl, params, c['sigma_net'], c['masks'], o, d, depths_sorted, c['Sc'], c['Sf'],
                                        c['box_warp'], g_feat, g_depth, g_wsum, rng, white_back=c['white_back'],
                                        want_planes=want_planes, want_params=want_params)
        g_planes = None
        if g_cl is not None:
            n, p, ch, h, w = ctx.plane_shape
            g_planes = tcconv.nhwc_to_nchw_f32(g_cl.view(n * p, h, w, ch)).view(n, p, ch, h, w)
        grads = [None] * ctx.n_params
        if g_par is not None:
            for i in range(n_nets):
                gw1, gb1, gw2, gb2 = torch.split(g_par[i], [64 * 32, 64, 33 * 64, 33])
                grads[4 * i:4 * i + 4] = [gw1.view(64, 32), gb1, gw2.view(33, 64), gb2]
        return (g_planes, None, *grads)


def _is_default_axes(axes):
    return tuple(axes.shape) == (3, 3, 3) and bool(torch.equal(axes.detach().cpu(), _DEFAULT_AXES))


class ImportanceRenderer(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.ray_marcher = MipRayMarcher2()
        self.plane_axes = generate_planes()

    # ------------------------------------------------------------------------------------------
    def forward(self, planes, decoder, ray_origins, ray_directions, rendering_options, planes_channels_last=None, plane_index=None):
        """planes [B,3,32,H,W]; rays [B,M,3] -> (features [B,M,C], depth [B,M,1], weight sum [B,M,1]) (:88-140).
        `planes_channels_last` ([B,3,H,W,32] fp32, optional) lets a caller that already holds the gather layout skip the
        transpose; `planes` may then be None. `plane_index` ([B] int32, with `planes_channels_last`): plane set per image,
        so that several camera views share one resident plane set."""
        self.plane_axes = self.plane_axes.to(ray_origins.device)
        opts = rendering_options

        n_importance = opts['depth_resolution_importance']
        auto = opts['ray_start'] == opts['ray_end'] == 'auto'
        if auto:
            ray_start, ray_end = math_utils.get_ray_limits_box(ray_origins, ray_directions, box_side_length=opts['box_warp'])
            is_ray_valid = ray_end > ray_start
            if torch.any(is_ray_valid).item():
                ray_start[~is_ray_valid] = ray_start[is_ray_valid].min()
                ray_end[~is_ray_valid] = ray_start[is_ray_valid].max()
        else:
            ray_start, ray_end = opts['ray_start'], opts['ray_end']

        grad_fused = planes_channels_last is None and self._fusable_grad(planes, decoder, ray_origins, ray_directions, opts)
        fused = planes_channels_last is not None or grad_fused or self._fusable(planes, decoder, ray_origins, ray_directions, opts)
        if fused:
            b, r = ray_origins.shape[:2]
            dev = ray_origins.device
            n_c = opts['depth_resolution']
            if opts['disparity_space_sampling']:
                kw = dict(depths_coarse=self.sample_stratified(ray_origins, ray_start, ray_end, n_c, True))
            else:
                # sample_stratified (:181-190) inside the kernel: the host only draws the jitter (same generator call, same
                # order as the reference's torch.rand_like) and hands over the linspace table
                jitter = torch.rand(b, r, n_c, 1, device=dev)
                if auto:
                    table = self._table(('steps', n_c, dev), lambda: torch.arange(n_c, dtype=torch.float32, device=dev) / (n_c - 1))
                    kw = dict(depths_coarse=None, stratified=dict(jitter=jitter, table=table, ray_start=ray_start, ray_end=ray_end))
                else:
                    table = self._table(('lin', float(ray_start), float(ray_end), n_c, dev),
                                        lambda: torch.linspace(ray_start, ray_end, n_c, device=dev))
                    kw = dict(depths_coarse=None, stratified=dict(jitter=jitter, table=table, delta=(ray_end - ray_start) / (n_c - 1)))
            u = torch.rand(b * r, n_importance, device=dev) if n_importance > 0 else None
            dec = native.pack_decoder(decoder)
            if grad_fused:
                nets, sigma_net, masks = native.describe_decoder(decoder)
                params = []
                for net in nets:
                    params += [*native._effective_fc(net[0]), *native._effective_fc(net[2])]
                call = dict(dec=dec, ray_origins=ray_origins, ray_directions=ray_directions, depths_coarse=kw.pop('depths_coarse'),
                            u=u, box_warp=opts['box_warp'], white_back=bool(opts.get('white_back', False)), kw=kw,
                            sigma_net=sigma_net, masks=masks, Sc=n_c, Sf=n_importance)
                return _FusedRender.apply(planes, call, *params)
            planes_cl = planes_channels_last if planes_channels_last is not None else native.planes_to_channels_last(planes)
            return native.render_fwd(planes_cl, dec, ray_origins, ray_directions, kw.pop('depths_coarse'), u, opts['box_warp'],
                                     white_back=bool(opts.get('white_back', False)), plane_index=plane_index, **kw)

        depths_coarse = self.sample_stratified(ray_origins, ray_start, ray_end, opts['depth_resolution'],
                                               opts['disparity_space_sampling'])
        return self._forward_staged(planes, decoder, ray_origins, ray_directions, depths_coarse, n_importance, opts)

    def _table(self, key, fn):
        """Small constant tensors of the stratified sampling (linspace of the ray limits), built once per configuration."""
        cache = self.__dict__.setdefault('_tables', {})
        t = cache.get(key)
        if t is None:
            t = cache[key] = fn()
        return t

    def fusable_options(self, decoder, opts):
        """True when the rendering options and decoder are covered by the fused kernel (independent of the planes)."""
        if opts.get('density_noise', 0) > 0 or opts['clamp_mode'] != 'softplus':
            return False
        if not self._axes_ok():
            return False
        s_total = opts['depth_resolution'] + opts['depth_resolution_importance']
        if opts['depth_resolution'] > 64 or opts['depth_resolution_importance'] > 64 or s_total > 256:
            return False
        if opts['depth_resolution_importance'] > 0 and opts['depth_resolution'] < 4:
            return False
        return native.describe_decoder(decoder) is not None

    def _fusable(self, planes, decoder, ray_origins, ray_directions, opts):
        if planes.device.type != 'cuda' or planes.ndim != 5 or planes.shape[1] != 3 or planes.shape[2] != 32:
            return False
        if torch.is_grad_enabled() and (planes.requires_grad or any(p.requires_grad for p in decoder.parameters())):
            return False
        if opts.get('density_noise', 0) > 0 or opts['clamp_mode'] != 'softplus':
            return False
        if not self._axes_ok():
            return False
        s_total = opts['depth_resolution'] + opts['depth_resolution_importance']
        if opts['depth_resolution'] > 64 or opts['depth_resolution_importance'] > 64 or s_total > 256:
            return False
        if opts['depth_resolution_importance'] > 0 and opts['depth_resolution'] < 4:
            return False
        return native.describe_decoder(decoder) is not None

    def _fusable_grad(self, planes, decoder, ray_origins, ray_directions, opts):
        """True when a gradient-requiring call can run on _FusedRender: gradients reach the planes or the decoder only (the
        rays carry none), CUDA fp32 [B,3,32,H,W] planes of the rays' batch, and options the fused kernels cover."""
        if not (fused_grad and torch.is_grad_enabled()):
            return False
        if not (planes.requires_grad or any(p.requires_grad for p in decoder.parameters())):
            return False
        if ray_origins.requires_grad or ray_directions.requires_grad:
            return False
        if (planes.device.type != 'cuda' or planes.dtype != torch.float32 or planes.ndim != 5 or planes.shape[1] != 3
                or planes.shape[2] != 32 or planes.shape[0] != ray_origins.shape[0]):
            return False
        return self.fusable_options(decoder, opts) and opts['depth_resolution'] + opts['depth_resolution_importance'] >= 2

    def _forward_staged(self, planes, decoder, ray_origins, ray_directions, depths_coarse, n_importance, opts):
        b, r, s, _ = depths_coarse.shape

        def shade(depths, count):
            coords = (ray_origins.unsqueeze(-2) + depths * ray_directions.unsqueeze(-2)).reshape(b, -1, 3)
            dirs = ray_directions.unsqueeze(-2).expand(-1, -1, count, -1).reshape(b, -1, 3)
            out = self.run_model(planes, decoder, coords, dirs, opts)
            colors = out['rgb']
            return colors.reshape(b, r, count, colors.shape[-1]), out['sigma'].reshape(b, r, count, 1)

        colors_coarse, dens_coarse = shade(depths_coarse, s)
        if n_importance > 0:
            _, _, weights = self.ray_marcher(colors_coarse, dens_coarse, depths_coarse, opts)
            depths_fine = self.sample_importance(depths_coarse, weights, n_importance)
            colors_fine, dens_fine = shade(depths_fine, n_importance)
            all_depths, all_colors, all_dens = self.unify_samples(depths_coarse, colors_coarse, dens_coarse,
                                                                  depths_fine, colors_fine, dens_fine)
            rgb, depth, weights = self.ray_marcher(all_colors, all_dens, all_depths, opts)
        else:
            rgb, depth, weights = self.ray_marcher(colors_coarse, dens_coarse, depths_coarse, opts)
        return rgb, depth, weights.sum(2)

    def _axes_ok(self):
        """True when `plane_axes` still holds generate_planes() (checked once per tensor object: no per-call sync)."""
        cache = getattr(self, '_axes_cache', None)
        if cache is None or cache[0] is not self.plane_axes:
            cache = (self.plane_axes, _is_default_axes(self.plane_axes))
            self._axes_cache = cache
        return cache[1]

    # ------------------------------------------------------------------------------------------
    def run_model(self, planes, decoder, sample_coordinates, sample_directions, options):
        """Tri-plane lookup + decoder at arbitrary points (:142-148); also the entry of G.sample / sample_mixed."""
        self.plane_axes = self.plane_axes.to(sample_coordinates.device)
        no_grad = not (torch.is_grad_enabled() and (planes.requires_grad or any(p.requires_grad for p in decoder.parameters())))
        if (planes.device.type == 'cuda' and no_grad and planes.ndim == 5 and planes.shape[1] == 3 and planes.shape[2] == 32
                and self._axes_ok() and native.describe_decoder(decoder) is not None):
            dec = native.pack_decoder(decoder)
            rgb, sigma = native.run_model(native.planes_to_channels_last(planes), dec, sample_coordinates, options['box_warp'])
            out = {'rgb': rgb, 'sigma': sigma}
        else:
            feats = sample_from_planes(self.plane_axes, planes, sample_coordinates, padding_mode='zeros',
                                       box_warp=options['box_warp'])
            out = decoder(feats, sample_directions)
        if options.get('density_noise', 0) > 0:
            out['sigma'] += torch.randn_like(out['sigma']) * options['density_noise']
        return out

    def sort_samples(self, all_depths, all_colors, all_densities):
        _, idx = torch.sort(all_depths, dim=-2)
        return (torch.gather(all_depths, -2, idx),
                torch.gather(all_colors, -2, idx.expand(-1, -1, -1, all_colors.shape[-1])),
                torch.gather(all_densities, -2, idx.expand(-1, -1, -1, 1)))

    def unify_samples(self, depths1, colors1, densities1, depths2, colors2, densities2):
        """Concatenate coarse and fine samples and sort them by depth (:157-167)."""
        return self.sort_samples(torch.cat([depths1, depths2], dim=-2), torch.cat([colors1, colors2], dim=-2),
                                 torch.cat([densities1, densities2], dim=-2))

    def sample_stratified(self, ray_origins, ray_start, ray_end, depth_resolution, disparity_space_sampling=False):
        """Jittered, approximately uniform depths [N,M,S,1] (:169-192)."""
        n, m, _ = ray_origins.shape
        dev = ray_origins.device
        if disparity_space_sampling:
            t = torch.linspace(0, 1, depth_resolution, device=dev).reshape(1, 1, depth_resolution, 1).repeat(n, m, 1, 1)
            t += torch.rand_like(t) * (1 / (depth_resolution - 1))
            return 1. / (1. / ray_start * (1. - t) + 1. / ray_end * t)
        if type(ray_start) == torch.Tensor:
            depths = math_utils.linspace(ray_start, ray_end, depth_resolution).permute(1, 2, 0, 3)
            delta = (ray_end - ray_start) / (depth_resolution - 1)
            depths += torch.rand_like(depths) * delta[..., None]
            return depths
        depths = torch.linspace(ray_start, ray_end, depth_resolution, device=dev).reshape(1, 1, depth_resolution, 1).repeat(n, m, 1, 1)
        depths += torch.rand_like(depths) * ((ray_end - ray_start) / (depth_resolution - 1))
        return depths

    def sample_importance(self, z_vals, weights, N_importance):
        """Depths of `N_importance` samples drawn from the smoothed coarse weights (:194-215)."""
        with torch.no_grad():
            b, r, s, _ = z_vals.shape
            z = z_vals.reshape(b * r, s)
            w = weights.reshape(b * r, -1)
            if z.device.type == 'cuda':
                u = torch.rand(b * r, N_importance, device=z.device)
                return native.sample_importance(z, w, u).reshape(b, r, N_importance, 1)
            w = torch.nn.functional.max_pool1d(w.unsqueeze(1).float(), 2, 1, padding=1)
            w = torch.nn.functional.avg_pool1d(w, 2, 1).squeeze()
            w = w + 0.01
            z_mid = 0.5 * (z[:, :-1] + z[:, 1:])
            return self.sample_pdf(z_mid, w[:, 1:-1], N_importance).detach().reshape(b, r, N_importance, 1)

    def sample_pdf(self, bins, weights, N_importance, det=False, eps=1e-5):
        """Inverse-CDF sampling of `bins` [N,K+1] with piecewise-constant pdf `weights` [N,K] (:217-253)."""
        n_rays, k = weights.shape
        weights = weights + eps
        pdf = weights / torch.sum(weights, -1, keepdim=True)
        cdf = torch.cumsum(pdf, -1)
        cdf = torch.cat([torch.zeros_like(cdf[:, :1]), cdf], -1)
        if det:
            u = torch.linspace(0, 1, N_importance, device=bins.device).expand(n_rays, N_importance)
        else:
            u = torch.rand(n_rays, N_importance, device=bins.device)
        u = u.contiguous()
        inds = torch.searchsorted(cdf, u, right=True)
        below = torch.clamp_min(inds - 1, 0)
        above = torch.clamp_max(inds, k)
        pair = torch.stack([below, above], -1).view(n_rays, 2 * N_importance)
        cdf_g = torch.gather(cdf, 1, pair).view(n_rays, N_importance, 2)
        bins_g = torch.gather(bins, 1, pair).view(n_rays, N_importance, 2)
        denom = cdf_g[..., 1] - cdf_g[..., 0]
        denom[denom < eps] = 1
        return bins_g[..., 0] + (u - cdf_g[..., 0]) / denom * (bins_g[..., 1] - bins_g[..., 0])


class ImportanceSemanticRenderer(ImportanceRenderer):
    """Two tri-plane sets and two decoders (:256-438): the semantic decoder sees the semantic planes and provides the
    density; the texture decoder sees cat(texture, semantic) features. Same two-pass sampling as ImportanceRenderer;
    features are cat(colour, semantic). Runs stage by stage (on CUDA each stage is a libp3d kernel: tri-plane gather,
    ray marcher, importance sampling; the decoders are two small GEMMs)."""

    def forward(self, planes_texture, planes_semantic, decoder_texture, decoder_semantic, ray_origins, ray_directions,
                rendering_options):
        self.plane_axes = self.plane_axes.to(ray_origins.device)
        opts = rendering_options
        if opts['ray_start'] == opts['ray_end'] == 'auto':
            ray_start, ray_end = math_utils.get_ray_limits_box(ray_origins, ray_directions, box_side_length=opts['box_warp'])
            is_ray_valid = ray_end > ray_start
            if torch.any(is_ray_valid).item():
                ray_start[~is_ray_valid] = ray_start[is_ray_valid].min()
                ray_end[~is_ray_valid] = ray_start[is_ray_valid].max()
            depths_coarse = self.sample_stratified(ray_origins, ray_start, ray_end, opts['depth_resolution'],
                                                   opts['disparity_space_sampling'])
        else:
            depths_coarse = self.sample_stratified(ray_origins, opts['ray_start'], opts['ray_end'], opts['depth_resolution'],
                                                   opts['disparity_space_sampling'])
        b, r, s, _ = depths_coarse.shape

        def shade(depths, count):
            coords = (ray_origins.unsqueeze(-2) + depths * ray_directions.unsqueeze(-2)).reshape(b, -1, 3)
            dirs = ray_directions.unsqueeze(-2).expand(-1, -1, count, -1).reshape(b, -1, 3)
            out = self.run_model(planes_texture, planes_semantic, decoder_texture, decoder_semantic, coords, dirs, opts)
            colors = out['rgb'].reshape(b, r, count, out['rgb'].shape[-1])
            sem = out['semantic'].reshape(b, r, count, out['semantic'].shape[-1])
            return colors, out['sigma'].reshape(b, r, count, 1), torch.cat([colors, sem], -1)

        colors_coarse, dens_coarse, feats_coarse = shade(depths_coarse, s)
        n_importance = opts['depth_resolution_importance']
        if n_importance > 0:
            _, _, weights = self.ray_marcher(colors_coarse, dens_coarse, depths_coarse, opts)
            depths_fine = self.sample_importance(depths_coarse, weights, n_importance)
            _, dens_fine, feats_fine = shade(depths_fine, n_importance)
            all_depths, all_feats, all_dens = self.unify_samples(depths_coarse, feats_coarse, dens_coarse,
                                                                 depths_fine, feats_fine, dens_fine)
            feat, depth, weights = self.ray_marcher(all_feats, all_dens, all_depths, opts)
        else:
            feat, depth, weights = self.ray_marcher(feats_coarse, dens_coarse, depths_coarse, opts)
        return feat, depth, weights.sum(2)

    def run_model(self, planes_texture, planes_semantic, decoder_texture, decoder_semantic, sample_coordinates,
                  sample_directions, options):
        """(:324-337) sigma and semantics from the semantic decoder, colour from the texture decoder."""
        self.plane_axes = self.plane_axes.to(sample_coordinates.device)
        f_tex = sample_from_planes(self.plane_axes, planes_texture, sample_coordinates, padding_mode='zeros',
                                   box_warp=options['box_warp'])
        f_sem = sample_from_planes(self.plane_axes, planes_semantic, sample_coordinates, padding_mode='zeros',
                                   box_warp=options['box_warp'])
        out_sem = decoder_semantic(f_sem, sample_directions)
        out_tex = decoder_texture(torch.cat([f_tex, f_sem], dim=-1), sample_directions)
        out = {'sigma': out_sem['sigma'], 'rgb': out_tex['rgb'], 'semantic': out_sem['rgb']}
        if options.get('density_noise', 0) > 0:
            out['sigma'] += torch.randn_like(out['sigma']) * options['density_noise']
        return out
