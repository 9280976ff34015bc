"""CPU checks behind output sizes whose latent sides are not divisible by 2^(levels-1) (1280x720, 1920x1080 and every
other multiple of 8 px): the nearest-index rule the upsample kernel relies on, and the oracle UNet run with diffusers'
``forward_upsample_size`` rule (tests/golden/sized_unet.py)."""
import torch
import torch.nn.functional as F

from sized_unet import forward_sized


def test_nearest_resize_to_odd_size_is_2x_then_crop():
    """For every output side 1..1100 with input side ceil(out/2), F.interpolate(size=out, mode="nearest") equals
    repeat-2 then crop: output index o reads input o >> 1 (what lb_upsample_nearest computes)."""
    for out in range(1, 1101):
        n = (out + 1) // 2
        x = torch.arange(n, dtype=torch.float32).view(1, 1, n, 1)
        got = F.interpolate(x, size=(out, 1), mode="nearest").view(-1)
        want = x.view(-1).repeat_interleave(2)[:out]
        assert torch.equal(got, want), out
        # and along the width, with both sides resized at once
        y = torch.arange(n, dtype=torch.float32).view(1, 1, 1, n).expand(1, 1, 2, n)
        got = F.interpolate(y, size=(4 if out % 2 == 0 else 3, out), mode="nearest")[0, 0, 0]
        assert torch.equal(got, want), out


def _tiny_oracle():
    from oracle.sdxl_unet import SDXLUNet, synthetic_init_, tiny_config
    cfg = tiny_config()
    return synthetic_init_(SDXLUNet(cfg), seed=0).eval(), cfg


def _inputs(cfg, B, h, w, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, 4, h, w, generator=g)
    ctx = torch.randn(B, 77, cfg.cross_attention_dim, generator=g) * 0.5
    pooled = torch.randn(B, cfg.pooled_dim, generator=g)
    tids = torch.tensor([[8.0 * h, 8.0 * w, 0, 0, 8.0 * h, 8.0 * w]] * B)
    return x, ctx, pooled, tids


def test_oracle_unet_at_17x11_resizes_to_the_skip_sizes():
    """Latent 17 x 11: levels 17x11 -> 9x6 -> 5x3 (stride-2 pad-1 convs), and each upsampler conv sees the size of
    the skip its up block concatenates next (5x3 -> 9x6 -> 17x11), as with diffusers' forward_upsample_size."""
    net, cfg = _tiny_oracle()
    seen = {"down": [], "up": []}
    hooks = [net.conv_in.register_forward_hook(lambda m, i, o: seen["down"].append(tuple(o.shape[2:])))]
    for blk in net.down_blocks:
        if blk.downsamplers is not None:
            hooks.append(blk.downsamplers[0].register_forward_hook(
                lambda m, i, o: seen["down"].append(tuple(o.shape[2:]))))
    for blk in net.up_blocks:
        if blk.upsamplers is not None:
            hooks.append(blk.upsamplers[0].conv.register_forward_hook(
                lambda m, i, o: seen["up"].append(tuple(o.shape[2:]))))
    x, ctx, pooled, tids = _inputs(cfg, 2, 17, 11)
    with torch.no_grad():
        eps = forward_sized(net, x, 321.0, ctx, pooled, tids)
    for h in hooks:
        h.remove()
    assert seen["down"] == [(17, 11), (9, 6), (5, 3)]
    assert seen["up"] == [(9, 6), (17, 11)]
    assert eps.shape == (2, 4, 17, 11) and torch.isfinite(eps).all()


def test_sized_forward_is_the_oracle_forward_at_divisible_sizes():
    """At 16 x 16 (divisible by 4) the sized forward -- by diffusers' rule, and with the resize forced on -- gives the
    same bits as SDXLUNet.forward, so the oracle and the fixtures made at divisible sizes agree with it."""
    net, cfg = _tiny_oracle()
    x, ctx, pooled, tids = _inputs(cfg, 1, 16, 16, seed=1)
    with torch.no_grad():
        plain = net(x, 500.0, ctx, pooled, tids)
        auto = forward_sized(net, x, 500.0, ctx, pooled, tids)
        forced = forward_sized(net, x, 500.0, ctx, pooled, tids, sized=True)
    assert torch.equal(plain, auto) and torch.equal(plain, forced)
