"""Oracle: SDXL ControlNet forward and its injection into the UNet, in plain PyTorch (test infrastructure).

Restates diffusers==0.25.0 ``ControlNetModel`` (models/controlnet.py: ControlNetConditioningEmbedding, the encoder
copy, the zero convs) and the non-guess-mode part of ``StableDiffusionXLControlNetPipeline.__call__`` that feeds it
(``controlnet_keep``, ``cond_scale``, ``down_block_additional_residuals`` / ``mid_block_additional_residual``) from
their published definitions.  diffusers is not installed here: this restatement was NOT checked against the package.

Parameter names mirror the diffusers state_dict keys of an SDXL ControlNet: the UNet encoder's names plus
``controlnet_cond_embedding.{conv_in, blocks.0-5, conv_out}``, ``controlnet_down_blocks.0-8`` and
``controlnet_mid_block``.
"""
import torch
import torch.nn as nn
import torch.nn.functional as F

from .sdxl_unet import DownBlock, MidBlock, SDXLUNet, TimestepEmbedding, UNetConfig, sinusoid, synthetic_init_

COND_CHANNELS = (16, 32, 96, 256)


def controlnet_keep(i, num_steps, start=0.0, end=1.0):
    """The pipeline's per-step weight: 1 - (i / N < start or (i + 1) / N > end)."""
    return 1.0 - float(i / num_steps < start or (i + 1) / num_steps > end)


class ConditioningEmbedding(nn.Module):
    def __init__(self, c0, channels=COND_CHANNELS, cin=3):
        super().__init__()
        self.conv_in = nn.Conv2d(cin, channels[0], 3, padding=1)
        blocks = []
        for i in range(len(channels) - 1):
            blocks.append(nn.Conv2d(channels[i], channels[i], 3, padding=1))
            blocks.append(nn.Conv2d(channels[i], channels[i + 1], 3, padding=1, stride=2))
        self.blocks = nn.ModuleList(blocks)
        self.conv_out = nn.Conv2d(channels[-1], c0, 3, padding=1)

    def forward(self, x):
        x = F.silu(self.conv_in(x))
        for b in self.blocks:
            x = F.silu(b(x))
        return self.conv_out(x)


class SDXLControlNet(nn.Module):
    """``cfg``: the encoder (the UNet's levels and channels, the ControlNet's own transformer depths)."""

    def __init__(self, cfg: UNetConfig, cond_channels=COND_CHANNELS):
        super().__init__()
        self.cfg = cfg
        ch = cfg.block_out_channels
        T = cfg.time_embed_dim
        self.conv_in = nn.Conv2d(cfg.in_channels, ch[0], 3, padding=1)
        self.time_embedding = TimestepEmbedding(ch[0], T)
        self.add_embedding = TimestepEmbedding(cfg.add_in_dim, T)
        self.controlnet_cond_embedding = ConditioningEmbedding(ch[0], cond_channels)
        downs, zero, cout = [], [nn.Conv2d(ch[0], ch[0], 1)], ch[0]
        for i, c in enumerate(ch):
            cin, cout = cout, c
            downs.append(DownBlock(cfg, cin, cout, cfg.transformer_layers[i], add_down=i < len(ch) - 1))
            zero += [nn.Conv2d(c, c, 1) for _ in range(cfg.layers_per_block + (i < len(ch) - 1))]
        self.down_blocks = nn.ModuleList(downs)
        self.controlnet_down_blocks = nn.ModuleList(zero)
        self.mid_block = MidBlock(cfg, ch[-1], cfg.transformer_layers[-1])
        self.controlnet_mid_block = nn.Conv2d(ch[-1], ch[-1], 1)

    def forward(self, x, t, encoder_hidden_states, text_embeds, time_ids, cond_image, conditioning_scale=1.0):
        """cond_image [B, 3, 8h, 8w] in [0, 1] -> (nine down residuals, mid residual), each times the scale."""
        B = text_embeds.shape[0]
        cfg = self.cfg
        tt = torch.as_tensor(t, dtype=torch.float32).reshape(-1).expand(B)
        emb = self.time_embedding(sinusoid(tt, cfg.block_out_channels[0]))
        tid = sinusoid(time_ids.reshape(-1), cfg.addition_time_embed_dim).reshape(B, -1)
        emb = emb + self.add_embedding(torch.cat([text_embeds.float(), tid], dim=-1))
        h = self.conv_in(x) + self.controlnet_cond_embedding(cond_image)
        res = [h]
        for blk in self.down_blocks:
            h, s = blk(h, emb, encoder_hidden_states)
            res += s
        h = self.mid_block(h, emb, encoder_hidden_states)
        down = [z(r) * conditioning_scale for z, r in zip(self.controlnet_down_blocks, res)]
        return down, self.controlnet_mid_block(h) * conditioning_scale


def unet_with_residuals(unet: SDXLUNet, x, t, encoder_hidden_states, text_embeds, time_ids, down_res=None,
                        mid_res=None):
    """SDXLUNet.forward with a ControlNet's residuals: skip i += down_res[i] after the down path, mid output +=
    mid_res (the mid block reads the un-added last down output)."""
    emb = unet.embed(t, text_embeds, time_ids)
    ctx = encoder_hidden_states
    h = unet.conv_in(x)
    skips = [h]
    for blk in unet.down_blocks:
        h, s = blk(h, emb, ctx)
        skips += s
    if down_res is not None:
        skips = [s + r for s, r in zip(skips, down_res)]
    h = unet.mid_block(h, emb, ctx)
    if mid_res is not None:
        h = h + mid_res
    for blk in unet.up_blocks:
        h = blk(h, skips, emb, ctx)
    return unet.conv_out(F.silu(unet.conv_norm_out(h)))


def image_to_cond(image_u8):
    """uint8 [H, W, 3] (already resized, RGB) -> [1, 3, H, W] float32 in [0, 1], rounded to fp16 as the pipeline's
    fp16 tensor is (VaeImageProcessor with do_normalize=False)."""
    x = torch.as_tensor(image_u8).float() / 255.0
    return x.half().float().permute(2, 0, 1)[None]


def synthetic_init_controlnet_(cn: SDXLControlNet, seed=0, damp=0.1):
    """The UNet's seeded recipe (``synthetic_init_``) with the zero convs damped like the residual branches, not
    zeroed: a zero ControlNet would leave every parity test vacuous."""
    synthetic_init_(cn, seed=seed, damp=damp)
    with torch.no_grad():
        for name, p in cn.named_parameters():
            if name.startswith(("controlnet_down_blocks.", "controlnet_mid_block.")):
                p.mul_(damp)
    return cn
