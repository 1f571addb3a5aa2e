"""Generate tests/golden/*.npz by running the REFERENCE implementation (a pix2pix3D checkout, imported read-only from
$P3D_REFERENCE_ROOT) on CPU with seeded inputs.

The tests never import the reference, which is why its outputs are committed.
    P3D_REFERENCE_ROOT=/path/to/pix2pix3D python oracle/make_golden.py     # tests/golden/{renderer,ops,synthesis}_*.npz, loss_ops.npz

The renderer's two random draws (stratified jitter, renderer.py:190; importance u, renderer.py:237) are captured
by wrapping torch.rand_like / torch.rand while the reference runs, and stored so that every implementation can be
fed the identical noise.
"""
import contextlib
import hashlib
import os
import sys

import numpy as np
import torch

REF = os.environ.get('P3D_REFERENCE_ROOT', '')
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), '..', 'tests', 'golden')


@contextlib.contextmanager
def capture_rand(store):
    o_like, o_rand, o_randn = torch.rand_like, torch.rand, torch.randn

    def rl(x, *a, **k):
        r = o_like(x, *a, **k); store.append(('rand_like', r.clone())); return r

    def rr(*a, **k):
        r = o_rand(*a, **k); store.append(('rand', r.clone())); return r

    torch.rand_like, torch.rand = rl, rr
    try:
        yield
    finally:
        torch.rand_like, torch.rand, torch.randn = o_like, o_rand, o_randn


def state_digest(module):
    h = hashlib.sha256()
    for k, v in sorted(module.state_dict().items()):
        h.update(k.encode())
        h.update(v.detach().cpu().contiguous().numpy().tobytes())
    return h.hexdigest()


def poses(n, seed, radius=2.7, pivot=(0, 0, -0.06), fov=18.837):
    import camera_utils
    g = np.random.RandomState(seed)
    c = []
    for _ in range(n):
        yaw = np.pi / 2 + g.uniform(-0.35, 0.35)
        pitch = np.pi / 2 + g.uniform(-0.25, 0.25)
        c2w = camera_utils.LookAtPoseSampler.sample(yaw, pitch, torch.tensor(pivot, dtype=torch.float32), radius=radius)
        K = camera_utils.FOV_to_intrinsics(fov)
        c.append(torch.cat([c2w.reshape(1, 16), K.reshape(1, 9)], 1))
    return torch.cat(c, 0)


# ---------------------------------------------------------------------------------------------
def golden_renderer():
    from training.volumetric_rendering.renderer import ImportanceRenderer
    from training.volumetric_rendering.ray_sampler import RaySampler
    from training.triplane import OSGDecoder
    from training.triplane_cond import OSGDecoder_semantic_lateSeparate

    cases = {
        # name: (B, plane res, nrr, Sc, Sf, decoder, options)
        'seg': (2, 32, 12, 12, 12, 'late6', dict(ray_start=2.25, ray_end=3.3, box_warp=1)),
        'seg48': (1, 40, 6, 48, 48, 'late6', dict(ray_start=2.25, ray_end=3.3, box_warp=1)),
        'car': (2, 24, 10, 16, 16, 'late1', dict(ray_start=0.1, ray_end=2.6, box_warp=1.6, white_back=True)),
        'rgb_only': (1, 32, 9, 10, 6, 'osg', dict(ray_start=2.25, ray_end=3.3, box_warp=1)),
        'coarse_only': (1, 32, 8, 9, 0, 'osg', dict(ray_start=2.25, ray_end=3.3, box_warp=1)),
        'far_outside': (1, 32, 8, 12, 12, 'late6', dict(ray_start=0.5, ray_end=6.0, box_warp=1)),
        # sample counts that are multiples of 8 (the tensor-core renderer's domain)
        'seg16': (2, 32, 9, 16, 8, 'late6', dict(ray_start=2.25, ray_end=3.3, box_warp=1)),
        'rgb24': (1, 32, 8, 24, 24, 'osg', dict(ray_start=2.25, ray_end=3.3, box_warp=1)),
        'coarse8': (1, 32, 8, 8, 0, 'osg', dict(ray_start=2.25, ray_end=3.3, box_warp=1)),
        'car64': (1, 24, 6, 64, 64, 'late1', dict(ray_start=0.1, ray_end=2.6, box_warp=1.6, white_back=True)),
    }
    only = set(sys.argv[2:]) if len(sys.argv) > 2 else None
    for name, (B, H, nrr, Sc, Sf, dkind, extra) in cases.items():
        if only is not None and name not in only:
            continue
        torch.manual_seed({'seg': 11, 'seg48': 12, 'car': 13, 'rgb_only': 14, 'coarse_only': 15, 'far_outside': 16,
                           'seg16': 17, 'rgb24': 18, 'coarse8': 19, 'car64': 20}[name])
        planes = torch.randn(B, 3, 32, H, H)
        if dkind == 'osg':
            dec = OSGDecoder(32, {'decoder_lr_mul': 1, 'decoder_output_dim': 32})
        else:
            cs = 6 if dkind == 'late6' else 1
            dec = OSGDecoder_semantic_lateSeparate(32, {'decoder_lr_mul': 1, 'decoder_output_dim': 32,
                                                        'sigmoid': cs == 1, 'semantic_channels': cs})
        with torch.no_grad():   # make biases non-trivial
            for p in dec.parameters():
                if p.ndim == 1:
                    p.copy_(torch.randn_like(p) * 0.5)
        fov = 18.837 if 'car' not in name else 45.0
        radius = 2.7 if 'car' not in name else 1.7
        c = poses(B, 3, radius=radius, pivot=(0, 0, 0) if 'car' in name else (0, 0, -0.06), fov=fov)
        c2w, K = c[:, :16].reshape(-1, 4, 4), c[:, 16:].reshape(-1, 3, 3)
        o, d = RaySampler()(c2w, K, nrr)
        opts = dict(depth_resolution=Sc, depth_resolution_importance=Sf, disparity_space_sampling=False,
                    clamp_mode='softplus', **extra)
        R = ImportanceRenderer()
        # stage tensors through hooks on the methods
        rec = {}
        orig_imp, orig_march, orig_unify = R.sample_importance, R.ray_marcher.forward, R.unify_samples
        march_calls = []

        def march(colors, dens, depths, ro):
            out = orig_march(colors, dens, depths, ro); march_calls.append(out[2].clone()); return out

        def imp(z, w, n):
            out = orig_imp(z, w, n); rec['depths_fine'] = out.clone(); return out

        def unify(d1, c1, s1, d2, c2, s2):
            alld = torch.cat([d1, d2], -2)
            rec['perm'] = torch.sort(alld, dim=-2, stable=True)[1][..., 0].clone()
            return orig_unify(d1, c1, s1, d2, c2, s2)

        R.sample_importance, R.ray_marcher.forward, R.unify_samples = imp, march, unify
        draws = []
        with torch.no_grad(), capture_rand(draws):
            feat, depth, wsum = R(planes, dec, o, d, opts)
        jitter = draws[0][1]
        u = draws[1][1] if Sf > 0 else torch.zeros(B * nrr * nrr, 0)
        save = dict(planes=planes, cam2world=c2w, intrinsics=K, ray_origins=o, ray_dirs=d, jitter=jitter, u=u,
                    feat=feat, depth=depth, wsum=wsum, weights_final=march_calls[-1][..., 0],
                    Sc=Sc, Sf=Sf, nrr=nrr, decoder=dkind, **{'opt_' + k: v for k, v in extra.items()})
        if Sf > 0:
            save.update(weights_coarse=march_calls[0][..., 0], depths_fine=rec['depths_fine'][..., 0], perm=rec['perm'])
        for k, v in dec.state_dict().items():
            save['dec.' + k] = v
        np.savez_compressed(os.path.join(OUT, f'renderer_{name}.npz'),
                            **{k: (v.detach().numpy() if isinstance(v, torch.Tensor) else np.asarray(v)) for k, v in save.items()})
        print('renderer', name, tuple(feat.shape))


# ---------------------------------------------------------------------------------------------
def golden_ops():
    from torch_utils.ops import bias_act, upfirdn2d, conv2d_resample
    from training.networks_stylegan2 import modulated_conv2d
    save = {}
    g = torch.Generator().manual_seed(5)
    # bias_act: forward + first/second order gradients of the reference's _ref path via autograd (float64 for the grads)
    x = torch.randn(3, 5, 4, 6, generator=g) * 2
    b = torch.randn(5, generator=g)
    save['ba_x'], save['ba_b'] = x, b
    for act in bias_act.activation_funcs:
        for tag, kw in (('d', {}), ('c', dict(gain=1.7, clamp=0.9, alpha=0.3))):
            xx = x.clone().double().requires_grad_(True)
            bb = b.clone().double().requires_grad_(True)
            y = bias_act.bias_act(xx, bb, act=act, impl='ref', **kw)
            gy = torch.randn(y.shape, generator=g).double()
            gx, = torch.autograd.grad(y, xx, gy, create_graph=True)
            ggx = torch.randn(gx.shape, generator=g).double()
            if gx.requires_grad:
                g2x, = torch.autograd.grad(gx, xx, ggx, allow_unused=True)
                g2x = torch.zeros_like(xx) if g2x is None else g2x
            else:
                g2x = torch.zeros_like(xx)
            save[f'ba_{act}_{tag}_y'] = bias_act.bias_act(x, b, act=act, impl='ref', **kw)
            save[f'ba_{act}_{tag}_y64'] = y.detach()
            save[f'ba_{act}_{tag}_gy'], save[f'ba_{act}_{tag}_gx'] = gy, gx.detach()
            save[f'ba_{act}_{tag}_ggx'], save[f'ba_{act}_{tag}_g2x'] = ggx, g2x.detach()
    # upfirdn2d: the shapes of SURVEY section 8(a19) at small size + odd cases
    f4 = upfirdn2d.setup_filter([1, 3, 3, 1])
    f8 = upfirdn2d.setup_filter([1, 2, 3, 4, 4, 3, 2, 1])           # separable (8 taps)
    f32_ = upfirdn2d.setup_filter(torch.randn(3, 5, generator=g), normalize=False)
    xs = torch.randn(2, 3, 9, 11, generator=g)
    save['up_x'] = xs
    save['up_f4'], save['up_f8'], save['up_f35'] = f4, f8, f32_
    cfgs = {
        'post_tconv': dict(f='f4', up=1, down=1, padding=[1, 1, 1, 1], gain=4),
        'skip_up': dict(f='f4', up=2, down=1, padding=[2, 1, 2, 1], gain=4),
        'down2': dict(f='f4', up=1, down=2, padding=[1, 1, 1, 1], gain=1),
        'pre_sconv': dict(f='f4', up=1, down=1, padding=[2, 2, 2, 2], gain=1),
        'sep8_up2': dict(f='f8', up=2, down=1, padding=[4, 3, 4, 3], gain=4),
        'odd': dict(f='f35', up=[3, 2], down=[2, 1], padding=[2, 0, -1, 3], gain=0.7, flip_filter=True),
        'crop': dict(f='f4', up=1, down=1, padding=[-1, 2, 0, -2], gain=1),
        'identity': dict(f=None, up=1, down=1, padding=0, gain=1),
    }
    fmap = dict(f4=f4, f8=f8, f35=f32_)
    for name, kw in cfgs.items():
        kw = dict(kw)
        f = fmap.get(kw.pop('f'))
        save[f'up_{name}_y'] = upfirdn2d.upfirdn2d(xs, f, impl='ref', **kw)
    # conv2d_resample + modulated_conv2d
    xc = torch.randn(2, 6, 8, 8, generator=g)
    w3 = torch.randn(5, 6, 3, 3, generator=g)
    w1 = torch.randn(5, 6, 1, 1, generator=g)
    st = torch.randn(2, 6, generator=g) + 1
    nz = torch.randn(1, 1, 16, 16, generator=g) * 0.1
    save.update(mc_x=xc, mc_w3=w3, mc_w1=w1, mc_styles=st, mc_noise16=nz)
    save['cr_up2'] = conv2d_resample.conv2d_resample(xc, w3, f=f4, up=2, padding=1, flip_weight=False)
    save['cr_down2'] = conv2d_resample.conv2d_resample(xc, w3, f=f4, down=2, padding=1)
    save['cr_1x1_down2'] = conv2d_resample.conv2d_resample(xc, w1, f=f4, down=2)
    save['cr_1x1_up2'] = conv2d_resample.conv2d_resample(xc, w1, f=f4, up=2)
    save['cr_plain'] = conv2d_resample.conv2d_resample(xc, w3, padding=1)
    for fused in (True, False):
        t = 'f' if fused else 'n'
        save[f'mc_up2_{t}'] = modulated_conv2d(xc.clone(), w3, st, noise=nz, up=2, padding=1, resample_filter=f4,
                                               flip_weight=False, fused_modconv=fused)
        save[f'mc_plain_{t}'] = modulated_conv2d(xc.clone(), w3, st, noise=nz[:, :, :8, :8], padding=1, fused_modconv=fused)
        save[f'mc_torgb_{t}'] = modulated_conv2d(xc.clone(), w1, st, demodulate=False, fused_modconv=fused)
    # filtered_lrelu (generic composition path of the reference, filtered_lrelu.py:123-155)
    from torch_utils.ops import filtered_lrelu
    xf = torch.randn(2, 4, 12, 12, generator=g)
    bf = torch.randn(4, generator=g)
    fd3 = upfirdn2d.setup_filter([1, 2, 1])
    save.update(fl_x=xf, fl_b=bf, fl_fd=fd3)
    save['fl_up2_down2'] = filtered_lrelu.filtered_lrelu(xf, f4, fd3, bf, up=2, down=2, padding=[3, 2, 3, 2], clamp=0.8, impl='ref')
    save['fl_up1'] = filtered_lrelu.filtered_lrelu(xf, None, f4, bf, up=1, down=1, padding=2, gain=1.3, slope=0.1, impl='ref')
    # DualDiscriminator forward (config-5 component), weights from the seed
    import training.dual_discriminator as dd
    torch.manual_seed(31)
    D = dd.DualDiscriminator(c_dim=25, img_resolution=64, img_channels=3, channel_base=1024, channel_max=32,
                             mapping_kwargs={}, epilogue_kwargs={'mbstd_group_size': 2}).eval().requires_grad_(False)
    img = {'image': torch.randn(2, 3, 64, 64, generator=g), 'image_raw': torch.randn(2, 3, 16, 16, generator=g)}
    cc = torch.randn(2, 25, generator=g)
    save.update(dd_image=img['image'], dd_image_raw=img['image_raw'], dd_c=cc, dd_logits=D(img, cc.clone()))
    np.savez_compressed(os.path.join(OUT, 'ops.npz'), **{k: v.detach().numpy() for k, v in save.items()})
    print('ops', len(save), 'arrays')


# ---------------------------------------------------------------------------------------------
SYNTH_CASES = {
    # config-1-like smoke models (BASELINE.json configs[0]); weights come from torch.manual_seed(seed)
    'seg_tiny': dict(seed=21, cls='TriPlaneSemanticEntangleGenerator', img_resolution=128, semantic_channels=6, nrr=16, Sc=12,
                     Sf=12, B=2, channel_base=1024, channel_max=16, ray=(2.25, 3.3, 1), mapping='mask', in_res=32),
    'car_tiny': dict(seed=22, cls='TriPlaneSemanticEntangleGenerator', img_resolution=128, semantic_channels=1, nrr=16, Sc=8,
                     Sf=8, B=1, channel_base=1024, channel_max=16, ray=(0.1, 2.6, 1.6), white_back=True, mapping='edge', in_res=32),
    # neural rendering at the super-resolution stack's native input resolution (no resize): the whole-generator fast path
    'seg_nrr64': dict(seed=24, cls='TriPlaneSemanticEntangleGenerator', img_resolution=128, semantic_channels=6, nrr=64, Sc=8,
                      Sf=8, B=1, channel_base=1024, channel_max=16, ray=(2.25, 3.3, 1), mapping='mask', in_res=32),
    # BASELINE config 3 (celeba): 19 semantic classes -> 19-channel ToRGB / raw-logit semantic branch
    'face_tiny': dict(seed=25, cls='TriPlaneSemanticEntangleGenerator', img_resolution=128, semantic_channels=19, nrr=16, Sc=8,
                      Sf=8, B=1, channel_base=1024, channel_max=16, ray=(2.25, 3.3, 1), mapping='mask', in_res=32),
    'rgb_tiny': dict(seed=23, cls='TriPlaneGenerator', img_resolution=128, semantic_channels=0, nrr=16, Sc=10, Sf=6, B=1,
                     channel_base=1024, channel_max=16, ray=(2.25, 3.3, 1), mapping='mask', in_res=32),
}


# TriPlaneSemanticGenerator (two backbones + ImportanceSemanticRenderer, triplane_cond.py:724-849; SURVEY 8 a10)
SEMGEN_CASES = {
    'semgen_tiny': dict(seed=31, cls='TriPlaneSemanticGenerator', img_resolution=128, semantic_channels=6, nrr=16, Sc=12, Sf=12,
                        B=2, channel_base=1024, channel_max=16, ray=(2.25, 3.3, 1), mapping='mask_plain', in_res=32, w_dim=512),
    'semgen_edge': dict(seed=32, cls='TriPlaneSemanticGenerator', img_resolution=128, semantic_channels=1, nrr=16, Sc=8, Sf=8,
                        B=1, channel_base=1024, channel_max=16, ray=(0.1, 2.6, 1.6), white_back=True, mapping='edge_plain',
                        in_res=32, w_dim=512),
}


# Generator / super-resolution classes no BASELINE configuration instantiates but the reference ships and train.py can select
# (train.py:389-397, triplane_cond.py:1085-1246): reference outputs only (no oracle restatement); the host-side mirror is
# checked against them on CPU and on CUDA (tests/test_extra_fixtures.py). `sub` = stored stride of the full-resolution outputs.
EXTRA_CASES = {
    'withbg_tiny': dict(seed=41, cls='TriPlaneSemanticEntangleGenerator_withBG', img_resolution=128, semantic_channels=6, nrr=16, Sc=12,
                        Sf=12, B=2, channel_base=1024, channel_max=16, ray=(2.25, 3.3, 1), mapping='mask', in_res=32, sub=1),
    'withbg_edge': dict(seed=42, cls='TriPlaneSemanticEntangleGenerator_withBG', img_resolution=128, semantic_channels=1, nrr=16, Sc=8,
                        Sf=8, B=1, channel_base=1024, channel_max=16, ray=(0.1, 2.6, 1.6), mapping='edge', in_res=32, sub=1),
    'sr8x_rgb': dict(seed=43, cls='TriPlaneGenerator', img_resolution=512, semantic_channels=0, nrr=32, Sc=10, Sf=6, B=1,
                     channel_base=1024, channel_max=16, ray=(2.25, 3.3, 1), mapping='mask', in_res=32, sub=4,
                     sr_module='training.superresolution.SuperresolutionHybrid8X'),
    'sr4x_rgb': dict(seed=44, cls='TriPlaneGenerator', img_resolution=256, semantic_channels=0, nrr=32, Sc=10, Sf=6, B=1,
                     channel_base=1024, channel_max=16, ray=(2.25, 3.3, 1), mapping='mask', in_res=32, sub=2,
                     sr_module='training.superresolution.SuperresolutionHybrid4X'),
    'sr4x_native': dict(seed=45, cls='TriPlaneGenerator', img_resolution=256, semantic_channels=0, nrr=128, Sc=4, Sf=4, B=1,
                        channel_base=1024, channel_max=16, ray=(2.25, 3.3, 1), mapping='mask', in_res=32, sub=2,
                        sr_module='training.superresolution.SuperresolutionHybrid4X'),
}


def synth_kwargs(case):
    sem = case['semantic_channels']
    rk = dict(image_resolution=case['img_resolution'], disparity_space_sampling=False, clamp_mode='softplus',
              superresolution_module=case.get('sr_module', 'training.superresolution.SuperresolutionHybrid2X'),
              superresolution_module_semantic='training.superresolution.SuperresolutionHybrid2X_semantic',
              c_gen_conditioning_zero=False, gpc_reg_prob=0.5, c_scale=1.0, superresolution_noise_mode='none',
              density_reg=0.25, density_reg_p_dist=0.004, reg_type='l1', decoder_lr_mul=1.0, sr_antialias=True,
              depth_resolution=case['Sc'], depth_resolution_importance=case['Sf'], ray_start=case['ray'][0],
              ray_end=case['ray'][1], box_warp=case['ray'][2], avg_camera_radius=2.7, avg_camera_pivot=[0, 0, -0.06])
    if case.get('white_back'):
        rk['white_back'] = True
    mclass = {'mask': 'MaskMappingNetwork_disentangle', 'edge': 'EdgeMappingNetwork_disentangle',
              'mask_plain': 'MaskMappingNetwork', 'edge_plain': 'EdgeMappingNetwork'}[case['mapping']]
    is_mask = case['mapping'].startswith('mask')
    mk = dict(class_name='training.triplane_cond.' + mclass,
              num_layers=2, in_resolution=case['in_res'], in_channels=max(sem, 1) if is_mask else 1)
    if is_mask and sem == 0:
        mk['in_channels'] = 6
    kw = dict(z_dim=32, c_dim=25, w_dim=case.get('w_dim', 512), img_resolution=case['img_resolution'], img_channels=3, mapping_kwargs=mk,
              rendering_kwargs=rk, channel_base=case['channel_base'], channel_max=case['channel_max'],
              fused_modconv_default='inference_only', num_fp16_res=0, sr_num_fp16_res=4, conv_clamp=None,
              sr_kwargs=dict(channel_base=case['channel_base'], channel_max=case['channel_max'],
                             fused_modconv_default='inference_only'))
    if sem > 0:
        kw['semantic_channels'] = sem
    return kw


def build_generator(module, case):
    """`module` is training.triplane_cond of whichever implementation is being built."""
    torch.manual_seed(case['seed'])
    G = getattr(module, case['cls'])(**synth_kwargs(case)).eval().requires_grad_(False)
    # make the noise / w_avg paths live (they initialise to zero: networks_stylegan2.py:310)
    g = torch.Generator().manual_seed(case['seed'] + 1000)
    for name, p in G.named_parameters():
        if name.endswith('noise_strength'):
            p.copy_(torch.randn([], generator=g) * 0.1)
        if name.endswith('.bias') and p.ndim == 1 and 'affine' not in name:
            p.copy_(torch.randn(p.shape, generator=g) * 0.1)
    return G


def synth_inputs(case):
    g = torch.Generator().manual_seed(case['seed'] + 2000)
    B = case['B']
    z = torch.randn(B, 32, generator=g)
    c = poses(B, case['seed'])
    if case['mapping'].startswith('mask'):
        nclass = max(case['semantic_channels'], 1) if case['semantic_channels'] else 6
        blocks = torch.randint(0, nclass, (B, 1, 4, 4), generator=g)
        mask = blocks.repeat_interleave(case['in_res'] // 4, 2).repeat_interleave(case['in_res'] // 4, 3)
    else:
        mask = (torch.rand(B, 1, case['in_res'], case['in_res'], generator=g) < 0.05).float() * 2 - 1
    return z, c, mask


def golden_synthesis():
    import training.triplane_cond as ref_tc
    only = set(sys.argv[2:]) if len(sys.argv) > 2 else None
    for name, case in SYNTH_CASES.items():
        if only is not None and name not in only:
            continue
        G = build_generator(ref_tc, case)
        z, c, mask = synth_inputs(case)
        draws = []
        with torch.no_grad():
            ws = G.mapping(z, c, {'mask': mask, 'pose': c})
            with capture_rand(draws):
                out = G.synthesis(ws, c, noise_mode='const', neural_rendering_resolution=case['nrr'])
            planes = G.backbone.synthesis(ws, noise_mode='const')
            pts = torch.rand(case['B'], 50, 3, generator=torch.Generator().manual_seed(9)) - 0.5
            smp = G.sample_mixed(pts, None, ws, noise_mode='const')
        save = dict(z=z, c=c, mask=mask, ws=ws, jitter=draws[0][1], u=draws[1][1], planes_sub=planes[:, :, 3::16, 5::16].contiguous(), pts=pts,
                    sample_rgb=smp['rgb'], sample_sigma=smp['sigma'], **{'out_' + k: v for k, v in out.items()})
        arrays = {k: v.detach().numpy() for k, v in save.items()}
        arrays['state_digest'] = np.frombuffer(state_digest(G).encode(), dtype=np.uint8)
        np.savez_compressed(os.path.join(OUT, f'synthesis_{name}.npz'), **arrays)
        print('synthesis', name, {k: tuple(v.shape) for k, v in out.items()})


def golden_extra():
    import training.triplane_cond as ref_tc
    only = set(sys.argv[2:]) if len(sys.argv) > 2 else None
    for name, case in EXTRA_CASES.items():
        if only is not None and name not in only:
            continue
        G = build_generator(ref_tc, case)
        z, c, mask = synth_inputs(case)
        draws = []
        with torch.no_grad():
            ws = G.mapping(z, c, {'mask': mask, 'pose': c})
            with capture_rand(draws):
                out = G.synthesis(ws, c, noise_mode='const', neural_rendering_resolution=case['nrr'])
        sub = case['sub']
        save = dict(z=z, c=c, mask=mask, ws=ws, jitter=draws[0][1], u=draws[1][1])
        for k, v in out.items():
            full = v.shape[-1] == case['img_resolution']
            save['out_' + k] = v[..., ::sub, ::sub].contiguous() if (full and sub > 1) else v
        arrays = {k: v.detach().numpy() for k, v in save.items()}
        arrays['state_digest'] = np.frombuffer(state_digest(G).encode(), dtype=np.uint8)
        np.savez_compressed(os.path.join(OUT, f'extra_{name}.npz'), **arrays)
        print('extra', name, {k: tuple(v.shape) for k, v in out.items()})


def golden_semgen():
    import training.triplane_cond as ref_tc
    only = set(sys.argv[2:]) if len(sys.argv) > 2 else None
    for name, case in SEMGEN_CASES.items():
        if only is not None and name not in only:
            continue
        G = build_generator(ref_tc, case)
        z, c, mask = synth_inputs(case)
        draws = []
        with torch.no_grad():
            ws = G.mapping(z, c, {'mask': mask, 'pose': c})
            with capture_rand(draws):
                out = G.synthesis(ws, c, noise_mode='const', neural_rendering_resolution=case['nrr'])
            wd = case['w_dim']
            pt = G.backbone.synthesis(ws[..., :wd], noise_mode='const')
            ps = G.backbone_semantic.synthesis(ws[..., wd:], noise_mode='const')
            pts = torch.rand(case['B'], 50, 3, generator=torch.Generator().manual_seed(9)) - 0.5
            smp = G.sample_mixed(pts, None, ws, noise_mode='const')
        save = dict(z=z, c=c, mask=mask, ws=ws, jitter=draws[0][1], u=draws[1][1],
                    planes_texture_sub=pt[:, :, 3::16, 5::16].contiguous(), planes_semantic_sub=ps[:, :, 3::16, 5::16].contiguous(),
                    pts=pts, sample_rgb=smp['rgb'], sample_sigma=smp['sigma'], sample_semantic=smp['semantic'],
                    **{'out_' + k: v for k, v in out.items()})
        arrays = {k: v.detach().numpy() for k, v in save.items()}
        arrays['state_digest'] = np.frombuffer(state_digest(G).encode(), dtype=np.uint8)
        np.savez_compressed(os.path.join(OUT, f'synthesis_{name}.npz'), **arrays)
        print('semgen', name, {k: tuple(v.shape) for k, v in out.items()})


def golden_loss_ops():
    """Loss-side image ops (SURVEY 8f-4), evaluated by the reference's own functions on CPU: `filtered_resizing`
    (training/dual_discriminator.py:86-102, all filter modes) with input gradients, and `cross_entropy2d`
    (training/loss_utils.py:4-18) with and without class weights and with the label-resolution upsample."""
    from torch_utils.ops import upfirdn2d
    from training.dual_discriminator import filtered_resizing
    from training.loss_utils import cross_entropy2d
    g = torch.Generator().manual_seed(77)
    save = {}
    f4 = upfirdn2d.setup_filter([1, 3, 3, 1])
    for tag, (src, dst) in {'up': (16, 64), 'down': (64, 16), 'odd': (24, 37)}.items():
        x = torch.randn(2, 3, src, src, generator=g).requires_grad_(True)
        gy = torch.randn(2, 3, dst, dst, generator=g)
        save[f'fr_{tag}_x'], save[f'fr_{tag}_gy'] = x.detach(), gy
        for mode in ('antialiased', 'none', 0.3) + (('classic',) if tag == 'up' else ()):
            y = filtered_resizing(x, size=dst, f=f4, filter_mode=mode)
            (gx,) = torch.autograd.grad((y * gy).sum(), x)
            save[f'fr_{tag}_{mode}_y'], save[f'fr_{tag}_{mode}_gx'] = y.detach(), gx
    for tag, (c, h, ht) in {'same': (6, 16, 16), 'lowres': (19, 8, 16)}.items():
        logits = (torch.randn(2, c, h, h, generator=g) * 3).requires_grad_(True)
        target = torch.randint(0, c, (2, ht, ht), generator=g)
        wgt = torch.rand(c, generator=g) * 4 + 0.2
        save[f'ce_{tag}_x'], save[f'ce_{tag}_t'], save[f'ce_{tag}_w'] = logits.detach(), target, wgt
        for wtag, w in (('plain', None), ('weighted', wgt)):
            loss = cross_entropy2d(logits, target, weight=w)
            (gx,) = torch.autograd.grad(loss, logits)
            save[f'ce_{tag}_{wtag}_loss'], save[f'ce_{tag}_{wtag}_gx'] = loss.detach(), gx
    np.savez_compressed(os.path.join(OUT, 'loss_ops.npz'), **{k: v.numpy() for k, v in save.items()})
    print('loss_ops', len(save), 'arrays')


# ---------------------------------------------------------------------------------------------
# Full-size cases at the BASELINE.json configurations (configs[1], [2] as released = 3b, [3]): the reference's G.synthesis on
# CPU with the constructor arguments train.py assembles (pix2pix3d_b200.configs.generator_kwargs -- a table of arguments, no
# code of this repository runs), seeded weights and seeded inputs. Stored: the seeds, a digest of the weights, SUBSAMPLED
# outputs, and for a ray subset the reference's own importance-sampling indices (torch.searchsorted, renderer.py:240), fine
# depths (:252) and the sort permutation of unify_samples (:162), so that the GPU tests can score the bookkeeping of the
# fused kernel against the reference at the metric's scale.
FULLSIZE_CASES = {
    'full_seg2cat': dict(workload='seg2cat_512', B=1, seed=0, input_seed=101),
    'full_seg2face': dict(workload='seg2face_512', B=1, seed=0, input_seed=102),
    'full_edge2car': dict(workload='edge2car_128', B=2, seed=0, input_seed=103),
}
RAY_STRIDE = 61


def fullsize_inputs(case, num_ws, nrr, Sc, Sf):
    """Inputs of a full-size case from its seeds (shared with tests/test_gpu_fullsize.py)."""
    from pix2pix3d_b200 import configs
    B, s = case['B'], case['input_seed']
    preset = configs.WORKLOADS[case['workload']]['preset']
    ws = configs.synthetic_ws(B, num_ws, s)
    c = configs.camera_labels(B, s + 1, preset)
    g = torch.Generator().manual_seed(s + 2)
    jitter = torch.rand(B, nrr * nrr, Sc, 1, generator=g)
    u = torch.rand(B * nrr * nrr, Sf, generator=g)
    return ws, c, jitter, u


def golden_fullsize():
    import training.triplane_cond as ref_tc
    repo = os.path.join(os.path.dirname(os.path.abspath(__file__)), '..')
    sys.path.append(repo)
    from pix2pix3d_b200 import configs
    only = set(sys.argv[2:]) if len(sys.argv) > 2 else None
    for name, case in FULLSIZE_CASES.items():
        if only is not None and name not in only:
            continue
        kw = configs.generator_kwargs(case['workload'])
        kw['mapping_kwargs'] = dict(class_name='training.networks_stylegan2.MappingNetwork', num_layers=2)
        torch.manual_seed(case['seed'])
        G = ref_tc.TriPlaneSemanticEntangleGenerator(**kw).eval().requires_grad_(False)
        gen = torch.Generator().manual_seed(case['seed'] + 1)
        for pname, p in G.named_parameters():
            if pname.endswith('noise_strength'):
                p.copy_(torch.randn([], generator=gen) * 0.1)
        w = configs.WORKLOADS[case['workload']]
        rk = kw['rendering_kwargs']
        nrr, Sc, Sf = w['nrr'], rk['depth_resolution'], rk['depth_resolution_importance']
        ws, c, jitter, u = fullsize_inputs(case, G.backbone.num_ws, nrr, Sc, Sf)
        rec = {}
        R = G.renderer
        o_imp, o_unify, o_march = R.sample_importance, R.unify_samples, R.ray_marcher.forward
        o_ss = torch.searchsorted
        marches, feats = [], []

        def imp(z, wgt, n):
            out = o_imp(z, wgt, n); rec['depths_fine'] = out.clone(); return out

        def unify(d1, c1, s1, d2, c2, s2):
            rec['perm'] = torch.sort(torch.cat([d1, d2], -2), dim=-2, stable=True)[1][..., 0].clone()
            return o_unify(d1, c1, s1, d2, c2, s2)

        def march(colors, dens, depths, ro):
            out = o_march(colors, dens, depths, ro); marches.append(out[2].clone()); feats.append(out[0].clone()); return out

        def ss(cdf, uu, **k):
            out = o_ss(cdf, uu, **k); rec['inds'] = out.clone(); return out

        R.sample_importance, R.unify_samples, R.ray_marcher.forward, torch.searchsorted = imp, unify, march, ss
        it = iter([jitter, u])
        o_like, o_rand = torch.rand_like, torch.rand
        torch.rand_like, torch.rand = (lambda x, *a, **k: next(it)), (lambda *a, **k: next(it))
        try:
            with torch.no_grad():
                out = G.synthesis(ws, c, noise_mode='const', neural_rendering_resolution=nrr)
        finally:
            torch.rand_like, torch.rand, torch.searchsorted = o_like, o_rand, o_ss
            R.sample_importance, R.unify_samples, R.ray_marcher.forward = o_imp, o_unify, o_march
        B, Rn = case['B'], nrr * nrr
        rays = torch.arange(0, Rn, RAY_STRIDE)
        save = dict(workload=case['workload'], B=B, seed=case['seed'], input_seed=case['input_seed'], ray_stride=RAY_STRIDE,
                    out_image_sub=out['image'][:, :, 3::8, 5::8].contiguous(), out_semantic_sub=out['semantic'][:, :, 3::8, 5::8].contiguous(),
                    out_image_raw=out['image_raw'], out_image_depth=out['image_depth'],
                    out_semantic_raw=out['semantic_raw'][:, :, ::2, ::2].contiguous(),
                    feat_rays=feats[-1].reshape(B, Rn, -1)[:, rays], weights_coarse_rays=marches[0].reshape(B, Rn, -1)[:, rays],
                    weights_final_rays=marches[-1].reshape(B, Rn, -1)[:, rays],
                    depths_fine_rays=rec['depths_fine'].reshape(B, Rn, -1)[:, rays], perm_rays=rec['perm'].reshape(B, Rn, -1)[:, rays].to(torch.int16),
                    inds_rays=rec['inds'].reshape(B, Rn, -1)[:, rays].to(torch.int16))
        arrays = {k: (v.detach().numpy() if isinstance(v, torch.Tensor) else np.asarray(v)) for k, v in save.items()}
        arrays['state_digest'] = np.frombuffer(state_digest(G).encode(), dtype=np.uint8)
        np.savez_compressed(os.path.join(OUT, f'{name}.npz'), **arrays)
        print('fullsize', name, {k: tuple(v.shape) for k, v in out.items()}, os.path.getsize(os.path.join(OUT, f'{name}.npz')) // 1024, 'KiB')


# tests/test_gpu_vs_reference.py: G.synthesis of the generator configurations behind BASELINE.json configs 1 and 3, inputs from
# seed 7, fp32 on both sides; stored on a fixed grid (every 16th pixel of the 512^2 outputs, every 4th of the neural-rendering
# outputs, odd offsets) so that the two fixtures stay small
VSREF_CASES = {'vsref_seg2cat_512': dict(workload='seg2cat_512', B=2, input_seed=7),
               'vsref_edge2car_128': dict(workload='edge2car_128', B=3, input_seed=7)}
_SUB16 = (slice(None), slice(None), slice(3, None, 16), slice(5, None, 16))
_SUB4 = (slice(None), slice(None), slice(1, None, 4), slice(2, None, 4))
VSREF_SUB = {'image': _SUB16, 'semantic': _SUB16, 'image_raw': _SUB4, 'image_depth': _SUB4, 'semantic_raw': _SUB4}


def golden_vs_reference():
    import training.triplane_cond as ref_tc
    repo = os.path.join(os.path.dirname(os.path.abspath(__file__)), '..')
    sys.path.append(repo)
    from pix2pix3d_b200 import configs
    for name, case in VSREF_CASES.items():
        kw = configs.generator_kwargs(case['workload'])
        kw['mapping_kwargs'] = dict(class_name='training.networks_stylegan2.MappingNetwork', num_layers=2)
        torch.manual_seed(0)
        G = ref_tc.TriPlaneSemanticEntangleGenerator(**kw).eval().requires_grad_(False)
        gen = torch.Generator().manual_seed(1)
        for pname, p in G.named_parameters():
            if pname.endswith('noise_strength'):
                p.copy_(torch.randn([], generator=gen) * 0.1)
        w = configs.WORKLOADS[case['workload']]
        rk = kw['rendering_kwargs']
        nrr, Sc, Sf = w['nrr'], rk['depth_resolution'], rk['depth_resolution_importance']
        ws, c, jitter, u = fullsize_inputs(case, G.backbone.num_ws, nrr, Sc, Sf)
        it = iter([jitter, u])
        o_like, o_rand = torch.rand_like, torch.rand
        torch.rand_like, torch.rand = (lambda x, *a, **k: next(it)), (lambda *a, **k: next(it))
        try:
            with torch.no_grad():
                out = G.synthesis(ws, c, noise_mode='const', neural_rendering_resolution=nrr, force_fp32=True)
        finally:
            torch.rand_like, torch.rand = o_like, o_rand
        arrays = {'out_' + k: out[k][VSREF_SUB[k]].contiguous().numpy() for k in VSREF_SUB}
        arrays['state_digest'] = np.frombuffer(state_digest(G).encode(), dtype=np.uint8)
        np.savez_compressed(os.path.join(OUT, f'{name}.npz'), **arrays)
        print('vs_reference', name, {k: tuple(v.shape) for k, v in arrays.items()}, os.path.getsize(os.path.join(OUT, f'{name}.npz')) // 1024, 'KiB')


if __name__ == '__main__':
    assert os.path.isdir(REF), 'set P3D_REFERENCE_ROOT to a checkout of the reference'
    sys.path.insert(0, REF)
    os.makedirs(OUT, exist_ok=True)
    torch.set_num_threads(os.cpu_count())
    which = sys.argv[1:] or ['renderer', 'ops', 'synthesis', 'semgen', 'loss_ops']
    if 'renderer' in which:
        golden_renderer()
    if 'ops' in which:
        golden_ops()
    if 'synthesis' in which:
        golden_synthesis()
    if 'semgen' in which:
        golden_semgen()
    if 'loss_ops' in which:
        golden_loss_ops()
    if 'fullsize' in which:
        golden_fullsize()
    if 'extra' in which:
        golden_extra()
    if 'vs_reference' in which:
        golden_vs_reference()
