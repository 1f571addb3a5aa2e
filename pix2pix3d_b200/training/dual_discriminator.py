"""Dual discriminator of EG3D / pix2pix3D: sees the super-resolved image concatenated with the (resized) raw render.

Mirror of the reference's training/dual_discriminator.py (`filtered_resizing` :86-102, `DualDiscriminator` :107-172,
`SingleDiscriminator` :21-80, `DummyDualDiscriminator` :179-245). Built from the same DiscriminatorBlock / Epilogue modules, whose FIR and bias_act work
runs on the sm_90a kernels; the convolutions go through `conv2d_gradfix`. Only needed by BASELINE config 5 (train step).
"""
import numpy as np
import torch

from ..torch_utils import persistence
from ..torch_utils.ops import upfirdn2d
from ..torch_utils.ops.resize import interpolate_bilinear
from .networks_stylegan2 import DiscriminatorBlock, DiscriminatorEpilogue, MappingNetwork


def filtered_resizing(image_orig_tensor, size, f, filter_mode='antialiased'):
    """Resize the raw render to the discriminator resolution (:86-102)."""
    if filter_mode == 'antialiased':
        return interpolate_bilinear(image_orig_tensor, (size, size), antialias=True)

    def interp(x, size, mode='bilinear', align_corners=False, antialias=False):
        return interpolate_bilinear(x, size, antialias=antialias)
    if filter_mode == 'classic':
        y = upfirdn2d.upsample2d(image_orig_tensor, f, up=2)
        y = interp(y, size=(size * 2 + 2, size * 2 + 2), mode='bilinear', align_corners=False)
        return upfirdn2d.downsample2d(y, f, down=2, flip_filter=True, padding=-1)
    if filter_mode == 'none':
        return interp(image_orig_tensor, size=(size, size), mode='bilinear', align_corners=False)
    assert type(filter_mode) == float and 0 < filter_mode < 1
    filtered = interp(image_orig_tensor, size=(size, size), mode='bilinear', align_corners=False, antialias=True)
    aliased = interp(image_orig_tensor, size=(size, size), mode='bilinear', align_corners=False, antialias=False)
    return (1 - filter_mode) * aliased + filter_mode * filtered


class _DiscBase(torch.nn.Module):
    def _build(self, c_dim, img_resolution, img_channels, architecture, channel_base, channel_max, num_fp16_res, conv_clamp,
               cmap_dim, block_kwargs, mapping_kwargs, epilogue_kwargs):
        self.c_dim = c_dim
        self.img_resolution = img_resolution
        self.img_resolution_log2 = int(np.log2(img_resolution))
        self.img_channels = img_channels
        self.block_resolutions = [2 ** i for i in range(self.img_resolution_log2, 2, -1)]
        channels = {res: min(channel_base // res, channel_max) for res in self.block_resolutions + [4]}
        fp16_resolution = max(2 ** (self.img_resolution_log2 + 1 - num_fp16_res), 8)
        if cmap_dim is None:
            cmap_dim = channels[4]
        if c_dim == 0:
            cmap_dim = 0
        common = dict(img_channels=img_channels, architecture=architecture, conv_clamp=conv_clamp)
        cur_layer_idx = 0
        for res in self.block_resolutions:
            block = DiscriminatorBlock(channels[res] if res < img_resolution else 0, channels[res], channels[res // 2],
                                       resolution=res, first_layer_idx=cur_layer_idx, use_fp16=(res >= fp16_resolution),
                                       **block_kwargs, **common)
            setattr(self, f'b{res}', block)
            cur_layer_idx += block.num_layers
        if c_dim > 0:
            self.mapping = MappingNetwork(z_dim=0, c_dim=c_dim, w_dim=cmap_dim, num_ws=None, w_avg_beta=None, **mapping_kwargs)
        self.b4 = DiscriminatorEpilogue(channels[4], cmap_dim=cmap_dim, resolution=4, **epilogue_kwargs, **common)

    def _trunk(self, img, c, block_kwargs, noise_c=0):
        x = None
        for res in self.block_resolutions:
            x, img = getattr(self, f'b{res}')(x, img, **block_kwargs)
        cmap = None
        if self.c_dim > 0:
            if noise_c > 0:
                c += torch.randn_like(c) * c.std(0) * noise_c
            cmap = self.mapping(None, c)
        return self.b4(x, img, cmap)

    def extra_repr(self):
        return f'c_dim={self.c_dim:d}, img_resolution={self.img_resolution:d}, img_channels={self.img_channels:d}'


@persistence.persistent_class
class SingleDiscriminator(_DiscBase):
    """Discriminator on the super-resolved image only (:21-80)."""

    def __init__(self, c_dim, img_resolution, img_channels, architecture='resnet', channel_base=32768, channel_max=512,
                 num_fp16_res=4, conv_clamp=256, cmap_dim=None, sr_upsample_factor=1, block_kwargs={}, mapping_kwargs={},
                 epilogue_kwargs={}):
        super().__init__()
        self._build(c_dim, img_resolution, img_channels, architecture, channel_base, channel_max, num_fp16_res, conv_clamp,
                    cmap_dim, block_kwargs, mapping_kwargs, epilogue_kwargs)

    def forward(self, img, c, update_emas=False, **block_kwargs):
        _ = update_emas
        return self._trunk(img['image'], c, block_kwargs)


@persistence.persistent_class
class DualDiscriminator(_DiscBase):
    """Discriminator on cat(image, resized image_raw): twice the image channels (:107-172)."""

    def __init__(self, c_dim, img_resolution, img_channels, architecture='resnet', channel_base=32768, channel_max=512,
                 num_fp16_res=4, conv_clamp=256, cmap_dim=None, disc_c_noise=0, block_kwargs={}, mapping_kwargs={},
                 epilogue_kwargs={}, **unused_kwargs):
        super().__init__()
        self._build(c_dim, img_resolution, img_channels * 2, architecture, channel_base, channel_max, num_fp16_res, conv_clamp,
                    cmap_dim, block_kwargs, mapping_kwargs, epilogue_kwargs)
        self.register_buffer('resample_filter', upfirdn2d.setup_filter([1, 3, 3, 1]))
        self.disc_c_noise = disc_c_noise

    def forward(self, img, c, update_emas=False, **block_kwargs):
        _ = update_emas
        image_raw = filtered_resizing(img['image_raw'], size=img['image'].shape[-1], f=self.resample_filter)
        return self._trunk(torch.cat([img['image'], image_raw], 1), c, block_kwargs, noise_c=self.disc_c_noise)


@persistence.persistent_class
class DummyDualDiscriminator(_DiscBase):
    """DualDiscriminator whose raw-image half fades out linearly over 500k/32 calls (:179-245; `raw_fade` starts at 1 and
    loses 32/500000 per forward, the call that reaches 0 and all later ones see a zeroed raw image)."""

    def __init__(self, c_dim, img_resolution, img_channels, architecture='resnet', channel_base=32768, channel_max=512,
                 num_fp16_res=4, conv_clamp=256, cmap_dim=None, block_kwargs={}, mapping_kwargs={}, epilogue_kwargs={}):
        super().__init__()
        self._build(c_dim, img_resolution, img_channels * 2, architecture, channel_base, channel_max, num_fp16_res, conv_clamp,
                    cmap_dim, block_kwargs, mapping_kwargs, epilogue_kwargs)
        self.register_buffer('resample_filter', upfirdn2d.setup_filter([1, 3, 3, 1]))
        self.raw_fade = 1

    def forward(self, img, c, update_emas=False, **block_kwargs):
        _ = update_emas
        self.raw_fade = max(0, self.raw_fade - 1 / (500000 / 32))
        image_raw = filtered_resizing(img['image_raw'], size=img['image'].shape[-1], f=self.resample_filter) * self.raw_fade
        return self._trunk(torch.cat([img['image'], image_raw], 1), c, block_kwargs)
