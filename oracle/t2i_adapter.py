"""Oracle: SDXL T2I-Adapter forward and its injection into the UNet's down path, in plain PyTorch (test
infrastructure).

Restates diffusers==0.25.0 ``T2IAdapter`` with ``adapter_type="full_adapter_xl"`` (models/adapter.py: FullAdapterXL,
AdapterBlock, AdapterResnetBlock), the ``down_intrablock_additional_residuals`` consumption of
``UNet2DConditionModel.forward`` / ``CrossAttnDownBlock2D.forward``, and the adapter part of
``StableDiffusionXLAdapterPipeline.__call__`` (``adapter_conditioning_scale``, ``adapter_conditioning_factor``) from
their published definitions.  diffusers is not installed here: this restatement was NOT checked against the package.
The three facts to check against it:

1. the body layout: body[0] 320 -> 320 without in_conv, body[1] a 1x1 in_conv 320 -> 640, body[2] AvgPool2d(2, 2,
   ceil_mode=True) then a 1x1 in_conv 640 -> 1280, body[3] 1280 -> 1280 without in_conv; each with num_res_blocks
   resnets relu(block1 3x3) -> block2 1x1 + x;
2. a DownBlock2D (no attention) gets ``sample += state`` AFTER its downsampler, in place, so the skip it stored last
   (the downsampler output, the same tensor) carries the add; a CrossAttnDownBlock2D adds after its last
   resnet/attention pair, before its downsampler, and stores the sum as that skip;
3. the mid block's output gets the next state only when the shapes are equal (for SDXL they always are).

The up path resizes to each skip's size as diffusers' ``forward_upsample_size`` does, so latent sides that are not
multiples of 4 (a 1280x720 image: 90x160 latents) run too.

State-dict names mirror diffusers': ``adapter.conv_in``, ``adapter.body.{i}.in_conv``,
``adapter.body.{i}.resnets.{j}.block{1,2}``.
"""
import torch
import torch.nn as nn
import torch.nn.functional as F

from .sdxl_unet import SDXLUNet

CHANNELS = (320, 640, 1280, 1280)


def adapter_factor_steps(num_steps, factor):
    """The steps i of ``num_steps`` that receive the adapter states: i < int(num_steps * factor)."""
    return int(num_steps * factor)


class AdapterResnetBlock(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.block1 = nn.Conv2d(c, c, 3, padding=1)
        self.block2 = nn.Conv2d(c, c, 1)

    def forward(self, x):
        return self.block2(F.relu(self.block1(x))) + x


class AdapterBlock(nn.Module):
    def __init__(self, cin, cout, num_res_blocks, down=False):
        super().__init__()
        self.down = down
        self.in_conv = nn.Conv2d(cin, cout, 1) if cin != cout else None
        self.resnets = nn.Sequential(*[AdapterResnetBlock(cout) for _ in range(num_res_blocks)])

    def forward(self, x):
        if self.down:
            x = F.avg_pool2d(x, 2, 2, ceil_mode=True)
        if self.in_conv is not None:
            x = self.in_conv(x)
        return self.resnets(x)


class FullAdapterXL(nn.Module):
    def __init__(self, in_channels=3, channels=CHANNELS, num_res_blocks=2, downscale_factor=16):
        super().__init__()
        self.downscale_factor = downscale_factor
        self.conv_in = nn.Conv2d(in_channels * downscale_factor ** 2, channels[0], 3, padding=1)
        body = []
        for i in range(len(channels)):
            if i == 1:
                body.append(AdapterBlock(channels[0], channels[1], num_res_blocks))
            elif i == 2:
                body.append(AdapterBlock(channels[1], channels[2], num_res_blocks, down=True))
            else:
                body.append(AdapterBlock(channels[i], channels[i], num_res_blocks))
        self.body = nn.ModuleList(body)

    def forward(self, x):
        x = self.conv_in(F.pixel_unshuffle(x, self.downscale_factor))
        feats = []
        for blk in self.body:
            x = blk(x)
            feats.append(x)
        return feats


class T2IAdapter(nn.Module):
    """The wrapper whose state dict prefixes every name with ``adapter.``."""

    def __init__(self, in_channels=3, channels=CHANNELS, num_res_blocks=2, downscale_factor=16):
        super().__init__()
        self.adapter = FullAdapterXL(in_channels, channels, num_res_blocks, downscale_factor)

    def forward(self, x):
        return self.adapter(x)


def image_to_adapter_input(image_u8):
    """uint8 [H, W] or [H, W, C] (already resized) -> [1, C, H, W] float32 u / 255, rounded to fp16 as the pipeline's
    fp16 adapter input is (``_preprocess_adapter_image`` then ``.to(adapter.dtype)``)."""
    x = torch.as_tensor(image_u8).float()
    if x.dim() == 2:
        x = x[..., None]
    return (x / 255.0).half().float().permute(2, 0, 1)[None]


def adapter_states(adapter, image, scale):
    """The pipeline's ``adapter_state``: every feature times ``adapter_conditioning_scale``."""
    return [f * scale for f in adapter(image)]


def unet_with_adapter(unet: SDXLUNet, x, t, encoder_hidden_states, text_embeds, time_ids, states=None):
    """SDXLUNet.forward with ``down_intrablock_additional_residuals = states`` (each [1, C, h, w], shared by the
    batch), consumed in order as diffusers 0.25 does (facts 2 and 3 of the module docstring)."""
    emb = unet.embed(t, text_embeds, time_ids)
    ctx = encoder_hidden_states
    rest = list(states) if states is not None else []
    h = unet.conv_in(x)
    skips = [h]
    for blk in unet.down_blocks:
        cross = blk.attentions is not None
        for i, res in enumerate(blk.resnets):
            h = res(h, emb)
            if cross:
                h = blk.attentions[i](h, ctx)
                if i == len(blk.resnets) - 1 and rest:
                    h = h + rest.pop(0)
            skips.append(h)
        if blk.downsamplers is not None:
            h = blk.downsamplers[0](h)
            skips.append(h)
        if not cross and rest:
            h = h + rest.pop(0)
            skips[-1] = h            # the in-place add: the stored skip is the same tensor
    h = unet.mid_block(h, emb, ctx)
    if rest and h.shape[1:] == rest[0].shape[1:]:
        h = h + rest.pop(0)
    # the up path with diffusers' forward_upsample_size rule: each upsampler resizes to its next skip's size (the
    # exact 2x when the latent sides are divisible by 2^(levels-1))
    for blk in unet.up_blocks:
        for i, res in enumerate(blk.resnets):
            h = res(torch.cat([h, skips.pop()], dim=1), emb)
            if blk.attentions is not None:
                h = blk.attentions[i](h, ctx)
        if blk.upsamplers is not None:
            h = blk.upsamplers[0].conv(F.interpolate(h, size=tuple(skips[-1].shape[2:]), mode="nearest"))
    return unet.conv_out(F.silu(unet.conv_norm_out(h)))


def synthetic_init_adapter_(adapter: nn.Module, seed=0, damp=0.1):
    """Default PyTorch inits under ``torch.manual_seed(seed)``, every block2 damped like the UNet's residual branches
    (not zeroed: the features must change the UNet's output for the parity tests to mean anything)."""
    torch.manual_seed(seed)
    for m in adapter.modules():
        if isinstance(m, nn.Conv2d):
            m.reset_parameters()
    with torch.no_grad():
        for name, p in adapter.named_parameters():
            if ".block2." in name:
                p.mul_(damp)
    return adapter
