"""Oracle: AutoencoderKL encoder + the image pre-processing of img2img (test infrastructure for image keyframes).

Code behind it: diffusers==0.25.0 ``models/autoencoders/vae.py`` ``Encoder`` (double_z), ``AutoencoderKL.encode``
(``quant_conv``), ``DiagonalGaussianDistribution.mode()`` and ``VaeImageProcessor.preprocess`` (NOT vendored),
restated from the published SDXL VAE config like oracle/vae.py's decoder.
"""
import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from .sdxl_unet import ResnetBlock2D
from .vae import SDXL_VAE, VAEConfig, VAEMid

# diffusers 0.25.0 ``Encoder`` (double_z) + ``quant_conv`` + ``DiagonalGaussianDistribution.mode()``, restated: conv_in
# 3 -> C0, down blocks of layers_per_block resnets each followed (all but the last) by Downsample2D(use_conv=True,
# padding=0) -- F.pad(x, (0, 1, 0, 1)) then a 3x3 stride-2 conv --, the decoder's mid block, GroupNorm + SiLU,
# conv_out to 2 * latent moments, quant_conv (1x1); the mean is the first half of the moments.


class Downsample2DPad0(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.conv = nn.Conv2d(c, c, 3, stride=2, padding=0)

    def forward(self, x):
        return self.conv(F.pad(x, (0, 1, 0, 1), mode="constant", value=0))


class VAEDownBlock(nn.Module):
    def __init__(self, cin, cout, n, groups, add_down):
        super().__init__()
        self.resnets = nn.ModuleList(
            [ResnetBlock2D(cin if i == 0 else cout, cout, 0, groups, eps=1e-6) for i in range(n)])
        self.downsamplers = nn.ModuleList([Downsample2DPad0(cout)]) if add_down else None

    def forward(self, x):
        for r in self.resnets:
            x = r(x)
        if self.downsamplers is not None:
            x = self.downsamplers[0](x)
        return x


class VAEEncoder(nn.Module):
    """Encoder + quant_conv; ``forward(x)`` -> the posterior mean [B, latent, H/8, W/8] (unscaled)."""

    def __init__(self, cfg: VAEConfig = SDXL_VAE):
        super().__init__()
        self.cfg = cfg
        ch = list(cfg.block_out_channels)
        g = cfg.norm_num_groups
        self.conv_in = nn.Conv2d(3, ch[0], 3, padding=1)
        downs, cout = [], ch[0]
        for i, c in enumerate(ch):
            cin, cout = cout, c
            downs.append(VAEDownBlock(cin, cout, cfg.layers_per_block, g, add_down=i < len(ch) - 1))
        self.down_blocks = nn.ModuleList(downs)
        self.mid_block = VAEMid(ch[-1], g)
        self.conv_norm_out = nn.GroupNorm(g, ch[-1], eps=1e-6)
        self.conv_out = nn.Conv2d(ch[-1], 2 * cfg.latent_channels, 3, padding=1)
        self.quant_conv = nn.Conv2d(2 * cfg.latent_channels, 2 * cfg.latent_channels, 1)

    def forward(self, x):
        x = self.conv_in(x)
        for b in self.down_blocks:
            x = b(x)
        x = self.mid_block(x)
        moments = self.quant_conv(self.conv_out(F.silu(self.conv_norm_out(x))))
        return moments[:, :self.cfg.latent_channels]           # DiagonalGaussianDistribution.mode()


def preprocess_image(image_u8):
    """VaeImageProcessor.preprocess of an HxWx3 uint8 array already at the output size: fp32 u / 255, then 2x - 1,
    NCHW [1, 3, H, W]."""
    x = torch.from_numpy(np.asarray(image_u8).astype(np.float32) / np.float32(255.0))
    return (2.0 * x - 1.0).permute(2, 0, 1)[None].contiguous()


def image2latent_np(enc: VAEEncoder, image_u8):
    """scaling_factor * the posterior mean of an HxWx3 uint8 image (retrieve_latents(sample_mode="argmax")), fp32."""
    with torch.no_grad():
        return enc(preprocess_image(image_u8)) * enc.cfg.scaling_factor


def synthetic_vae_encoder_init_(enc, seed=5):
    from .sdxl_unet import synthetic_init_
    return synthetic_init_(enc, seed=seed, damp=0.3)
