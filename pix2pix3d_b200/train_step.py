"""One training iteration of pix2pix3D (BASELINE.json configs[4]: afhq_seg `train.py` step -- G forward + dual discriminator
+ R1 -- batch 32 over 8 GPUs = 4 images per GPU) as a callable, so that it can be timed and checked without datasets, logging
or snapshots.

What runs is the reference's arithmetic: its own `training.loss.Pix2Pix3DLoss.accumulate_gradients` (training/loss.py:509-1022)
drives the phases; this module restates only the inner loop of `training_loop.py` around it (:513-546): per phase
zero_grad -> accumulate gradients -> ONE flat fp32 all-reduce of all gradients of the phase's module (NCCL SUM, / num_gpus,
nan_to_num) -> Adam step, with lazy regularisation intervals (`Greg` every 4, `Dreg` / `D_semanticreg` every 16,
:363-373) and the G_ema update (:549-559).

Every network / op class is resolved through the reference's import paths (`training.*`, `torch_utils.*`, `dnnlib`):
  * product arm: `pix2pix3d_b200.install(reference_root=...)` is active, so G, D, the ops and kernels are this package's
    and only the host-side loss class comes from the reference checkout (the drop-in scenario of BASELINE.json.north_star:
    "train.py calls into it unchanged");
  * reference arm: nothing is installed and everything resolves to the unmodified reference (a verbatim copy, oracle/_ref).
`lpips` (training/loss.py:20, a VGG download) is not available offline: a stub returning zeros is injected and the
configuration sets lambda_lpips = 0, as SURVEY.md 8c prescribes; G / D / R1 arithmetic is unaffected.
"""
import copy
import sys
import types

import numpy as np


def _lpips_stub():
    if 'lpips' in sys.modules:
        return
    import torch

    class LPIPS(torch.nn.Module):
        def __init__(self, **kwargs):
            super().__init__()

        def forward(self, a, b):
            return torch.zeros([a.shape[0], 1, 1, 1], device=a.device, dtype=torch.float32)
    mod = types.ModuleType('lpips')
    mod.LPIPS = LPIPS
    sys.modules['lpips'] = mod


# train_scripts/afhq_seg.sh with --gpus=8 --batch=32 (batch_gpu 4) and --lambda_lpips=0; resume => blur off (train.py:501-503)
AFHQ_TRAIN = dict(
    img_resolution=512, semantic_channels=6, nrr=128, batch_gpu=4, mbstd_group=4, gamma=5.0, glr=0.0025, dlr=0.002,
    G_reg_interval=4, D_reg_interval=16, cbase=32768, cmax=512, d_num_fp16_res=4, sr_num_fp16_res=4,
    loss=dict(r1_gamma=5.0, random_c_prob=0.5, lambda_l1=0, lambda_lpips=0, lambda_D_semantic=0.1, seg_weight=0, edge_weight=2,
              only_raw_recons=True, silhouette_loss=False, lambda_cross_view=1e-4, blur_init_sigma=0, blur_fade_kimg=200,
              gpc_reg_prob=0.5, gpc_reg_fade_kimg=0, dual_discrimination=True, neural_rendering_resolution_initial=128,
              neural_rendering_resolution_final=None, neural_rendering_resolution_fade_kimg=1000, style_mixing_prob=0,
              filter_mode='antialiased'),
)
# a small variant of the same graph for tests. It keeps img_resolution 512: the 128 / 256 models use SynthesisBlockNoUp, whose
# in-place `img.add_(y)` on a view (superresolution.py:283) trips autograd's version check in the reference under torch 2.x
TINY_TRAIN = dict(AFHQ_TRAIN, nrr=32, batch_gpu=2, mbstd_group=2, cbase=512, cmax=8, d_num_fp16_res=0, sr_num_fp16_res=0,
                  depth_resolution=8, loss=dict(AFHQ_TRAIN['loss'], neural_rendering_resolution_initial=32))


def generator_kwargs(cfg):
    res = cfg['img_resolution']
    sr = {512: 'SuperresolutionHybrid8XDC', 256: 'SuperresolutionHybrid4X', 128: 'SuperresolutionHybrid2X'}[res]
    rk = dict(image_resolution=res, disparity_space_sampling=False, clamp_mode='softplus',
              superresolution_module='training.superresolution.' + sr,
              superresolution_module_semantic='training.superresolution.' + sr + '_semantic',
              c_gen_conditioning_zero=False, gpc_reg_prob=0.5, c_scale=1.0, superresolution_noise_mode='none', density_reg=0.25,
              density_reg_p_dist=0.004, reg_type='l1', decoder_lr_mul=1.0, sr_antialias=True, depth_resolution=48,
              depth_resolution_importance=48, ray_start=2.25, ray_end=3.3, box_warp=1, avg_camera_radius=2.7,
              avg_camera_pivot=[0, 0, -0.06])
    if 'depth_resolution' in cfg:
        rk['depth_resolution'] = rk['depth_resolution_importance'] = cfg['depth_resolution']
    mapping = dict(class_name='training.triplane_cond.MaskMappingNetwork_disentangle', num_layers=2, in_resolution=res,
                   in_channels=cfg['semantic_channels'])
    return dict(class_name='training.triplane_cond.TriPlaneSemanticEntangleGenerator', z_dim=512, w_dim=512, mapping_kwargs=mapping,
                rendering_kwargs=rk, channel_base=cfg['cbase'], channel_max=cfg['cmax'], fused_modconv_default='inference_only',
                num_fp16_res=0, conv_clamp=None, sr_num_fp16_res=cfg['sr_num_fp16_res'],
                sr_kwargs=dict(channel_base=cfg['cbase'], channel_max=cfg['cmax'], fused_modconv_default='inference_only'))


def discriminator_kwargs(cfg):
    return dict(class_name='training.dual_discriminator.DualDiscriminator', block_kwargs=dict(freeze_layers=0), mapping_kwargs={},
                epilogue_kwargs=dict(mbstd_group_size=cfg['mbstd_group']), channel_base=cfg['cbase'], channel_max=cfg['cmax'],
                num_fp16_res=cfg['d_num_fp16_res'], conv_clamp=256 if cfg['d_num_fp16_res'] > 0 else None, disc_c_noise=0)


class TrainState:
    pass


def build(cfg, device, rank=0, num_gpus=1, seed=0):
    """Networks, loss and phases as training_loop.py:296-373 builds them (random init, no resume pickle)."""
    import torch
    _lpips_stub()
    import dnnlib
    from torch_utils import misc
    from torch_utils.ops import conv2d_gradfix, grid_sample_gradfix
    torch.manual_seed(seed)                                # identical initial weights on every rank (the reference broadcasts, :349-353)
    torch.backends.cudnn.benchmark = True                  # training_loop.py:277-282
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    conv2d_gradfix.enabled = True
    grid_sample_gradfix.enabled = False
    common = dict(c_dim=25, img_resolution=cfg['img_resolution'], img_channels=3)
    st = TrainState()
    st.cfg, st.device, st.rank, st.num_gpus = cfg, device, rank, num_gpus
    st.G = dnnlib.util.construct_class_by_name(**generator_kwargs(cfg), **common, semantic_channels=cfg['semantic_channels'],
                                               data_type='seg').train().requires_grad_(False).to(device)
    st.D = dnnlib.util.construct_class_by_name(**discriminator_kwargs(cfg), **common).train().requires_grad_(False).to(device)
    dsem = dict(common, img_channels=3 + cfg['semantic_channels'])          # training_loop.py:313
    st.D_semantic = dnnlib.util.construct_class_by_name(**discriminator_kwargs(cfg), **dsem).train().requires_grad_(False).to(device)
    st.G_ema = copy.deepcopy(st.G).eval()
    st.G.neural_rendering_resolution = cfg['nrr']
    import training.loss as loss_mod
    st.loss = loss_mod.Pix2Pix3DLoss(device=device, G=st.G, D=st.D, D_semantic=st.D_semantic, augment_pipe=None, **cfg['loss'])
    st.phases = []
    for name, module, lr, interval in (('G', st.G, cfg['glr'], cfg['G_reg_interval']), ('D', st.D, cfg['dlr'], cfg['D_reg_interval']),
                                       ('D_semantic', st.D_semantic, cfg['dlr'], cfg['D_reg_interval'])):
        ratio = interval / (interval + 1)                  # lazy regularisation (:363-372)
        opt = torch.optim.Adam(module.parameters(), lr=lr * ratio, betas=[0 ** ratio, 0.99 ** ratio], eps=1e-8)
        st.phases.append(dnnlib.EasyDict(name=name + 'main', module=module, opt=opt, interval=1))
        st.phases.append(dnnlib.EasyDict(name=name + 'reg', module=module, opt=opt, interval=interval))
    st.batch_idx = 0
    st.cur_nimg = 0
    st.misc = misc
    st.flat_bytes = {}
    return st


def synthetic_batch(cfg, device, seed):
    """What `load_data` yields per GPU (training_loop.py:481-497): image [-1,1] fp32, 6-class label map, 25-float pose."""
    import torch
    from pix2pix3d_b200 import configs
    b, res, cs = cfg['batch_gpu'], cfg['img_resolution'], cfg['semantic_channels']
    g = torch.Generator().manual_seed(seed)
    blocks = torch.randint(0, cs, (b, 1, 16, 16), generator=g)
    mask = blocks.repeat_interleave(res // 16, 2).repeat_interleave(res // 16, 3).to(torch.float32)
    image = torch.nn.functional.interpolate(torch.rand(b, 3, 32, 32, generator=g), size=(res, res), mode='bilinear') * 2 - 1
    pose = configs.camera_labels(b, seed + 1)
    return {'image': image.to(device), 'mask': mask.to(device), 'pose': pose.to(device)}


def run_iteration(st, batch, timers=None):
    """training_loop.py:499-559 for one `batch_idx`. `timers`: optional {phase name: [(start_event, end_event), ...]}."""
    import torch
    cfg, dev = st.cfg, st.device
    b = cfg['batch_gpu']
    n_ph = len(st.phases)
    all_z = torch.randn([n_ph * b, st.G.z_dim], device=dev).split(b)
    from pix2pix3d_b200 import configs
    all_c = configs.camera_labels(n_ph * b, 1000 + st.batch_idx * st.num_gpus + st.rank).to(dev).split(b)
    for phase, gen_z, gen_c in zip(st.phases, all_z, all_c):
        if st.batch_idx % phase.interval != 0:
            continue
        ev = None
        if timers is not None:
            ev = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
            ev[0].record()
        phase.opt.zero_grad(set_to_none=True)
        phase.module.requires_grad_(True)
        st.loss.accumulate_gradients(phase=phase.name, batch=batch, gen_z=gen_z, gen_c=gen_c, gain=phase.interval, cur_nimg=st.cur_nimg)
        phase.module.requires_grad_(False)
        params = [p for p in phase.module.parameters() if p.numel() > 0 and p.grad is not None]
        if params:
            flat = torch.cat([p.grad.flatten() for p in params])
            st.flat_bytes[phase.name] = flat.numel() * flat.element_size()
            if st.num_gpus > 1:
                torch.distributed.all_reduce(flat)          # ONE collective per phase (training_loop.py:532-537)
                flat /= st.num_gpus
            st.misc.nan_to_num(flat, nan=0, posinf=1e5, neginf=-1e5, out=flat)
            for p, g in zip(params, flat.split([p.numel() for p in params])):
                p.grad = g.reshape(p.shape)
        phase.opt.step()
        if ev is not None:
            ev[1].record()
            timers.setdefault(phase.name, []).append(ev)
    # G_ema (:549-559), ema_kimg = batch * 10 / 32, no ramp-up on resume
    batch_size = b * st.num_gpus
    ema_beta = 0.5 ** (batch_size / max(batch_size * 10 / 32 * 1000, 1e-8))
    with torch.no_grad():
        for p_ema, p in zip(st.G_ema.parameters(), st.G.parameters()):
            p_ema.copy_(p.lerp(p_ema, ema_beta))
        for b_ema, bb in zip(st.G_ema.buffers(), st.G.buffers()):
            b_ema.copy_(bb)
    st.G_ema.neural_rendering_resolution = st.G.neural_rendering_resolution
    st.G_ema.rendering_kwargs = st.G.rendering_kwargs.copy()
    st.cur_nimg += batch_size
    st.batch_idx += 1


def grads_digest(st):
    """Sum of squares of the current parameters of every network (cheap cross-arm consistency probe)."""
    import torch
    out = {}
    for name, m in (('G', st.G), ('D', st.D), ('D_semantic', st.D_semantic)):
        out[name] = float(sum(p.detach().double().square().sum() for p in m.parameters()))
    return out
