"""SDXL ControlNet on liblb200: weight packing, the conditioning-image embedding and the lowering of the control
branch into the UNet's step program.

An SDXL ControlNet (diffusers 0.25 ``ControlNetModel``, e.g. diffusers/controlnet-canny-sdxl-1.0) is a trained copy
of the UNet's encoder -- conv_in, time / added-condition embeddings, down blocks, mid block -- plus a small
conditioning-image embedding and one 1x1 "zero conv" per down residual and one for the mid block.  Its forward, in
the pipeline's non-guess mode:

    h0 = conv_in(x) + cond_embedding(image)               image: uint8 / 255, not normalised
    down / mid blocks as the UNet's, with its own weights and the UNet's prompt embeddings
    r_i = zero_conv_i(down output i) * scale,  r_mid = zero_conv_mid(mid output) * scale

and the UNet adds ``r_i`` to its skip ``i`` after its down path and ``r_mid`` to its mid block output.

Here the scale is folded into the zero-conv weights and biases (repacked in place when it changes, so recorded
programs keep valid pointers), each zero conv is one GEMM with the skip as in-place residual, and the conditioning
embedding [h*w, C0] is computed once per control image and size (``ControlNetB200.embed``) and read by every step.
"""
import torch

from .lowering import pack3
from .program import Program
from .unet import PackedUNet, UNetConfig

COND_CHANNELS = (16, 32, 96, 256)      # ControlNetConditioningEmbedding's block_out_channels (the SDXL default)


def keep_scale(i, num_steps, guidance_start=0.0, guidance_end=1.0):
    """The pipeline's per-step ControlNet weight for absolute step ``i`` of ``num_steps``: 1 inside
    [guidance_start, guidance_end], else 0 (StableDiffusionXLControlNetPipeline's ``controlnet_keep``)."""
    return 1.0 - float(i / num_steps < guidance_start or (i + 1) / num_steps > guidance_end)


def cond_embedding_layers(cond_channels, c0):
    """(state-dict prefix, Cin, Cout, stride, SiLU) of the conditioning embedding's 3x3 convs, in order."""
    layers = [("controlnet_cond_embedding.conv_in", 3, cond_channels[0], 1, True)]
    for i in range(len(cond_channels) - 1):
        a, b = cond_channels[i], cond_channels[i + 1]
        layers.append((f"controlnet_cond_embedding.blocks.{2 * i}", a, a, 1, True))
        layers.append((f"controlnet_cond_embedding.blocks.{2 * i + 1}", a, b, 2, True))
    layers.append(("controlnet_cond_embedding.conv_out", cond_channels[-1], c0, 1, False))
    return layers


def num_down_residuals(cfg: UNetConfig):
    L = len(cfg.block_out_channels)
    return 1 + L * cfg.layers_per_block + (L - 1)


class PackedControlNet(PackedUNet):
    """fp16 device copies of a ControlNet's parameters: the encoder through ``PackedUNet``'s packers, plus the
    conditioning embedding and the zero convs (scaled by the conditioning scale, see ``set_scale``).  Raises
    ValueError when the state dict holds a key the packing does not use."""

    def __init__(self, cfg: UNetConfig, state_dict, device, cond_channels=COND_CHANNELS):
        if cfg.time_cond_proj_dim is not None or "time_embedding.cond_proj.weight" in state_dict:
            raise ValueError("a ControlNet with time_embedding.cond_proj is not supported")
        self._pack_encoder(cfg, state_dict, device)
        W, g = self.w, self.g
        self.cond_channels = tuple(cond_channels)
        self.cond_layers = cond_embedding_layers(self.cond_channels, cfg.block_out_channels[0])
        for name, _, _, _, _ in self.cond_layers[:-1]:
            W[name + ".w"] = g(name + ".weight").permute(2, 3, 1, 0).contiguous()     # [ky][kx][Cin][Cout]
            W[name + ".b"] = g(name + ".bias")
        name = self.cond_layers[-1][0]
        W[name + ".w"], W[name + ".b"] = pack3(g(name + ".weight")), g(name + ".bias")   # the taps = 9 GEMM's rows
        self.zero_names = [f"controlnet_down_blocks.{i}" for i in range(num_down_residuals(cfg))]
        self.zero_names.append("controlnet_mid_block")
        self.zero_master = []
        for name in self.zero_names:
            w, b = g(name + ".weight"), g(name + ".bias")
            self.zero_master.append((w.reshape(w.shape[0], -1).contiguous(), b))
            W[name + ".w"], W[name + ".b"] = torch.empty_like(self.zero_master[-1][0]), torch.empty_like(b)
        left = sorted(set(state_dict) - self.consumed)
        if left:
            raise ValueError(f"the ControlNet state dict has {len(left)} keys this lowering cannot represent, e.g. "
                             f"{left[:3]}")
        self.scale = None
        self.set_scale(1.0)

    def set_scale(self, scale):
        """Fold ``scale`` into the zero convs: W = fp16(scale * W16), b = fp16(scale * b16), written in place."""
        scale = float(scale)
        if scale == self.scale:
            return
        for name, (w, b) in zip(self.zero_names, self.zero_master):
            self.w[name + ".w"].copy_((w.float() * scale).half())
            self.w[name + ".b"].copy_((b.float() * scale).half())
        self.scale = scale


class ControlNetB200:
    """A ControlNet attached to a ``UNetB200`` (``UNetB200(..., controlnet=cn)``): its packed weights, the
    conditioning scale, and one conditioning-embedding buffer per latent size."""

    def __init__(self, cfg: UNetConfig, state_dict, device="cuda:0", cond_channels=COND_CHANNELS):
        self.cfg = cfg
        self.device = torch.device(device)
        self.dev_index = self.device.index or 0
        self.packed = PackedControlNet(cfg, state_dict, self.device, cond_channels)
        self._emb = {}

    def set_scale(self, scale):
        self.packed.set_scale(scale)

    def embedding(self, h, w):
        """The [h*w, C0] fp16 conditioning embedding the step programs at latent size (h, w) read."""
        return self._embed_plan(h, w)["out"]

    def _embed_plan(self, h, w):
        e = self._emb.get((h, w))
        if e is None:
            W, dev = self.packed.w, self.device
            img = torch.zeros((8 * h * 8 * w, 3), dtype=torch.uint8, device=dev)
            out = torch.zeros((h * w, self.cfg.block_out_channels[0]), dtype=torch.float16, device=dev)
            P = Program(self.dev_index)
            x, H, Wd = img, 8 * h, 8 * w
            for name, cin, cout, stride, silu in self.packed.cond_layers[:-1]:
                Ho, Wo = (H - 1) // stride + 1, (Wd - 1) // stride + 1
                y = torch.empty((Ho * Wo, cout), dtype=torch.float16, device=dev)
                P.cond_conv(x, 1, H, Wd, cin, W[name + ".w"], W[name + ".b"], cout, y, stride=stride, silu=silu)
                x, H, Wd = y, Ho, Wo
            if (H, Wd) != (h, w):
                raise ValueError(f"the conditioning embedding maps {8 * h}x{8 * w} to {H}x{Wd}, not {h}x{w}")
            name, cin, cout = self.packed.cond_layers[-1][:3]
            P.gemm(x, W[name + ".w"], cout, 1, h, w, out, taps=9, bias=W[name + ".b"])
            e = self._emb[(h, w)] = dict(img=img, out=out, prog=P.finalize())
        return e

    @torch.no_grad()
    def embed(self, image_u8, h, w):
        """Fill the embedding of latent size (h, w) from ``image_u8``, a uint8 [8h, 8w, 3] RGB tensor (already resized
        and channel-ordered as the ControlNet expects)."""
        if tuple(image_u8.shape) != (8 * h, 8 * w, 3) or image_u8.dtype != torch.uint8:
            raise ValueError(f"the control image must be uint8 [{8 * h}, {8 * w}, 3] (got {image_u8.dtype} "
                             f"{tuple(image_u8.shape)})")
        e = self._embed_plan(h, w)
        e["img"].copy_(image_u8.reshape(-1, 3))
        e["prog"].run()
        return e["out"]


def lower_controlnet(low, P, cn: ControlNetB200):
    """Record the ControlNet forward of the UNet lowering ``low`` into ``P``: its embeddings from the UNet's sinusoid
    features, h0 = conv_in(x) + embedding, the down path and mid block (``low.down_mid``, the UNet's shared lowering)
    into its own buffers, then each zero conv as one GEMM adding into the UNet's skip (in place) or mid output."""
    pk = cn.packed
    W, cfg = pk.w, pk.cfg
    ch = cfg.block_out_channels
    temb_all = low.embed(P, pk, low.temb_in)
    dsts = [low.persist(low.rows_at(lvl), c) for lvl, c in low.skip_meta]
    P.conv_in_add(low.x_in, W["conv_in.w"], W["conv_in.b"], ch[0], dsts[0], cn.embedding(low.H, low.W))
    mid = low.persist(low.rows_at(len(ch) - 1), ch[-1])
    low.down_mid(P, dict(W=W, packed=pk, temb_all=temb_all, depths=cfg.transformer_layers), dsts, mid)
    for (lvl, c), feat, skip, name in zip(low.skip_meta, dsts, low.skip_views, pk.zero_names):
        P.gemm(feat, W[name + ".w"], c, 1, 1, low.rows_at(lvl), skip, bias=W[name + ".b"], res=skip)
    hid = low.cats[0]["hidden"]
    P.gemm(mid, W["controlnet_mid_block.w"], ch[-1], 1, 1, low.rows_at(len(ch) - 1), hid,
           bias=W["controlnet_mid_block.b"], res=hid)
