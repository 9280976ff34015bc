"""diffusers' ``forward_upsample_size`` rule on top of the oracle UNet (oracle/sdxl_unet.py), for parity tests and
fixtures at latent sizes that are not divisible by 2^(levels-1), such as 90x160 (1280x720) or 135x240 (1920x1080).

UNet2DConditionModel.forward sets ``forward_upsample_size`` when a latent side is not divisible by
2**num_upsamplers; each non-final up block then passes the spatial size of the next skip as ``upsample_size``, and
Upsample2D interpolates to that size (mode "nearest") instead of by an exact 2x.  ``forward_sized`` runs the oracle's
own modules in the oracle's order and only swaps that one interpolation, so at divisible sizes it computes exactly
what ``SDXLUNet.forward`` computes.
"""
import torch
import torch.nn.functional as F


def forward_sized(net, x, t, encoder_hidden_states, text_embeds, time_ids, sized=None):
    """SDXLUNet forward with the resize-to-skip-size rule.  ``sized``: None applies diffusers' rule (on when a latent
    side is not divisible by 2^(levels-1)); True / False force it on / off."""
    emb = net.embed(t, text_embeds, time_ids)
    ctx = encoder_hidden_states
    if sized is None:
        f = 1 << (len(net.up_blocks) - 1)
        sized = any(s % f != 0 for s in x.shape[-2:])
    h = net.conv_in(x)
    skips = [h]
    for blk in net.down_blocks:
        h, s = blk(h, emb, ctx)
        skips += s
    h = net.mid_block(h, emb, ctx)
    for blk in net.up_blocks:
        for i, res in enumerate(blk.resnets):
            h = res(torch.cat([h, skips.pop()], dim=1), temb=emb)
            if blk.attentions is not None:
                h = blk.attentions[i](h, ctx)
        if blk.upsamplers is not None:
            up = blk.upsamplers[0]
            if sized:
                h = up.conv(F.interpolate(h, size=tuple(skips[-1].shape[2:]), mode="nearest"))
            else:
                h = up(h)
    return net.conv_out(F.silu(net.conv_norm_out(h)))
