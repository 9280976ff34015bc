"""Oracle: the tiny SDXL autoencoder's decoder (AutoencoderTiny / TAESDXL) + image post-processing (test
infrastructure).

Call site: latentblending/diffusers_holder.py:114-143 (``latent2image``) with ``pipe.vae`` replaced by
``AutoencoderTiny.from_pretrained('madebyollin/taesdxl')`` as both of the reference's ``__main__`` blocks do
(blending_engine.py:797,806, diffusers_holder.py:373,379): ``vae.decode(latents / scaling_factor)`` then
``image_processor.postprocess``.  Code behind it: diffusers==0.25.0 ``models/autoencoder_tiny.py`` / ``vae.py``
``DecoderTiny`` / ``unet_2d_blocks.py`` ``AutoencoderTinyBlock`` (NOT vendored; restated here, parity unpinned as
DESIGN.md section 2 says for the UNet and the KL VAE).  Built from ``nn.Sequential`` so that the parameter names
are the diffusers decoder's (``layers.{i}.conv.{0,2,4}.*``, ``layers.{i}.weight``) by construction.
"""
from dataclasses import dataclass
from typing import Tuple

import torch
import torch.nn as nn

from .vae import postprocess_to_uint8


@dataclass
class TinyVAEConfig:
    latent_channels: int = 4
    out_channels: int = 3
    decoder_block_out_channels: Tuple[int, ...] = (64, 64, 64, 64)
    num_decoder_blocks: Tuple[int, ...] = (3, 3, 3, 1)
    upsampling_scaling_factor: int = 2
    act_fn: str = "relu"
    scaling_factor: float = 1.0
    force_upcast: bool = False


TAESDXL = TinyVAEConfig()


class AutoencoderTinyBlock(nn.Module):
    """ReLU(conv3(ReLU(conv2(ReLU(conv1(x))))) + skip(x)); skip is the identity for equal channel counts."""

    def __init__(self, cin, cout):
        super().__init__()
        self.conv = nn.Sequential(nn.Conv2d(cin, cout, 3, padding=1), nn.ReLU(),
                                  nn.Conv2d(cout, cout, 3, padding=1), nn.ReLU(),
                                  nn.Conv2d(cout, cout, 3, padding=1))
        self.skip = nn.Conv2d(cin, cout, 1, bias=False) if cin != cout else nn.Identity()
        self.fuse = nn.ReLU()

    def forward(self, x):
        return self.fuse(self.conv(x) + self.skip(x))


class DecoderTiny(nn.Module):
    def __init__(self, cfg: TinyVAEConfig = TAESDXL):
        super().__init__()
        self.cfg = cfg
        ch, nb = cfg.decoder_block_out_channels, cfg.num_decoder_blocks
        layers = [nn.Conv2d(cfg.latent_channels, ch[0], 3, padding=1), nn.ReLU()]
        for i, n in enumerate(nb):
            last = i == len(nb) - 1
            for _ in range(n):
                layers.append(AutoencoderTinyBlock(ch[i], ch[i]))
            if not last:
                layers.append(nn.Upsample(scale_factor=cfg.upsampling_scaling_factor, mode="nearest"))
            layers.append(nn.Conv2d(ch[i], cfg.out_channels if last else ch[i], 3, padding=1, bias=last))
        self.layers = nn.Sequential(*layers)

    def forward(self, z):
        x = torch.tanh(z / 3) * 3
        return self.layers(x).mul(2).sub(1)


def latent2image_np(dec: DecoderTiny, latents):
    """diffusers_holder.py:129-141 with an AutoencoderTiny: decode(latents / scaling_factor) in fp32, then the
    post-processing of the KL decoder -> uint8 HxWx3 array."""
    z = latents.to(torch.float32) / dec.cfg.scaling_factor
    return postprocess_to_uint8(dec(z))[0]
