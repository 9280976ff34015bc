"""SDXL T2I-Adapter on liblb200: weight packing, the once-per-image feature program, and the adapter's shapes and
per-step window.

An SDXL T2I-Adapter (diffusers 0.25 ``T2IAdapter`` with ``adapter_type="full_adapter_xl"``, e.g.
TencentARC/t2i-adapter-canny-sdxl-1.0) maps one control image to four feature maps, once per image and size:

    x = conv_in(PixelUnshuffle(16)(image))          image: uint8 / 255, not normalised; 3x3 conv, Cin*256 -> C0
    body[0] = AdapterBlock(C0 -> C0)                each block: optional 1x1 in_conv, then num_res_blocks resnets
    body[1] = AdapterBlock(C0 -> C1)                    h = relu(block1(x)) (3x3), x = block2(h) (1x1) + x
    body[2] = AdapterBlock(C1 -> C2, down)          AvgPool2d(2, 2, ceil_mode=True) before the in_conv
    body[3] = AdapterBlock(C2 -> C2)
    features = [output of body[i]]

StableDiffusionXLAdapterPipeline multiplies each feature by ``adapter_conditioning_scale`` once, and the UNet adds
the four states inside its down path (unet.py: ``prog_step_ad``) at the steps i < int(N * adapter_conditioning_factor).

Here the pixel unshuffle is one kernel that also converts u / 255 to fp16 and writes the channels in (i, j, c) order;
conv_in's weight columns are permuted to match.  The 3x3 convs run on the implicit-GEMM conv (taps = 9, ReLU fused
into block1's epilogue), the 1x1 convs on the GEMM (block2 with x as the residual).  The scaled states live in
persistent buffers per latent size, filled in place, so the step programs that read them stay valid.
"""
import torch

from .lowering import Scratch, pack3
from .program import Program

ADAPTER_TYPE = "full_adapter_xl"
DOWNSCALE = 16


def adapter_steps(num_steps, factor):
    """How many leading steps of ``num_steps`` receive the adapter states: int(num_steps * factor)."""
    return int(num_steps * factor)


def check_image_size(height, width, downscale=DOWNSCALE):
    """ValueError unless the output image's sides are multiples of ``downscale``: only then do the adapter's features
    have the UNet's shapes (diffusers fails on other sizes too)."""
    if height % downscale or width % downscale:
        raise ValueError(f"a T2I-Adapter needs an output width and height that are multiples of {downscale} (got "
                         f"{width}x{height}): its features are 1/{downscale} and 1/{2 * downscale} of the image")


def feature_shapes(height, width, channels, downscale=DOWNSCALE):
    """(rows, cols, channels) of the four features of a height x width image: 1/16 for body 0 and 1, then the
    ceil-mode 2x2 pool for body 2 and 3."""
    h, w = height // downscale, width // downscale
    hp, wp = (h + 1) // 2, (w + 1) // 2
    return [(h, w, channels[0]), (h, w, channels[1]), (hp, wp, channels[2]), (hp, wp, channels[3])]


def body_layout(channels):
    """(Cin, Cout, down) of the four AdapterBlocks of FullAdapterXL."""
    c = channels
    return [(c[0], c[0], False), (c[0], c[1], False), (c[1], c[2], True), (c[2], c[3], False)]


class PackedAdapter:
    """fp16 device copies of a FullAdapterXL's parameters in the layouts the kernels consume.  Raises ValueError when
    the state dict holds a key the packing does not use."""

    def __init__(self, cfg, state_dict, device):
        self.in_channels, self.channels = int(cfg["in_channels"]), tuple(cfg["channels"])
        self.num_res_blocks, r = int(cfg["num_res_blocks"]), int(cfg["downscale_factor"])
        if cfg.get("adapter_type", ADAPTER_TYPE) != ADAPTER_TYPE or r != DOWNSCALE or len(self.channels) != 4:
            raise ValueError(f"only the SDXL T2I-Adapter is supported (adapter_type {ADAPTER_TYPE!r}, downscale_factor "
                             f"{DOWNSCALE}, four channel counts); got {cfg.get('adapter_type')!r}, {r}, "
                             f"{self.channels}")
        if self.in_channels not in (1, 3):
            raise ValueError(f"a T2I-Adapter takes 1 or 3 image channels (got {self.in_channels})")
        dev = torch.device(device)
        self.consumed = set()

        def g(name):
            self.consumed.add(name)
            return state_dict[name].detach().to(device=dev, dtype=torch.float16).contiguous()

        W = self.w = {}
        w = g("adapter.conv_in.weight")
        c0, cin = w.shape[0], self.in_channels
        # torch's PixelUnshuffle channel c*r*r + i*r + j -> the kernel's (i*r + j)*Cin + c
        w = w.view(c0, cin, r * r, 3, 3).permute(0, 2, 1, 3, 4).reshape(c0, r * r * cin, 3, 3)
        W["conv_in.w"], W["conv_in.b"] = pack3(w), g("adapter.conv_in.bias")
        for i, (ci, co, _) in enumerate(body_layout(self.channels)):
            p = f"adapter.body.{i}"
            if ci != co:
                W[f"{i}.in_conv.w"] = g(p + ".in_conv.weight").reshape(co, ci).contiguous()
                W[f"{i}.in_conv.b"] = g(p + ".in_conv.bias")
            for j in range(self.num_res_blocks):
                q = f"{p}.resnets.{j}"
                W[f"{i}.{j}.block1.w"], W[f"{i}.{j}.block1.b"] = pack3(g(q + ".block1.weight")), g(q + ".block1.bias")
                W[f"{i}.{j}.block2.w"] = g(q + ".block2.weight").reshape(co, co).contiguous()
                W[f"{i}.{j}.block2.b"] = g(q + ".block2.bias")
        left = sorted(set(state_dict) - self.consumed)
        if left:
            raise ValueError(f"the T2I-Adapter state dict has {len(left)} keys this lowering cannot represent, e.g. "
                             f"{left[:3]}")


class AdapterB200:
    """A T2I-Adapter attached to a ``UNetB200`` (``UNetB200(..., adapter=ad)``): its packed weights and, per latent
    size, one recorded feature program with its uint8 image buffer, four feature buffers and the four persistent
    scaled states fp16(feature * scale) the UNet's ``prog_step_ad`` reads."""

    def __init__(self, cfg, state_dict, device="cuda:0", vae_scale_factor=8):
        self.device = torch.device(device)
        self.dev_index = self.device.index or 0
        self.packed = PackedAdapter(cfg, state_dict, self.device)
        self.in_channels, self.channels = self.packed.in_channels, self.packed.channels
        self.vae_scale_factor = vae_scale_factor
        self._plans = {}

    def supports(self, h, w):
        """Whether latents h x w (an 8h x 8w image) give features of the UNet's shapes."""
        s = self.vae_scale_factor
        return (h * s) % DOWNSCALE == 0 and (w * s) % DOWNSCALE == 0

    def states(self, h, w):
        """The four [rows, C] fp16 scaled-state buffers for latent size (h, w), filled by ``compute``."""
        return self._plan(h, w)["states"]

    def _plan(self, h, w):
        e = self._plans.get((h, w))
        if e is not None:
            return e
        s = self.vae_scale_factor
        H, Wd = h * s, w * s
        check_image_size(H, Wd)
        dev, Wt, r = self.device, self.packed.w, DOWNSCALE
        f16 = dict(dtype=torch.float16, device=dev)
        scratch = Scratch(torch.float16, dev)
        P = Program(self.dev_index)
        img = torch.zeros((H, Wd, self.in_channels), dtype=torch.uint8, device=dev)
        hh, ww = H // r, Wd // r
        xu = torch.empty((hh * ww, r * r * self.in_channels), **f16)
        P.pixel_unshuffle_u8(img, r, xu)
        x = torch.empty((hh * ww, self.channels[0]), **f16)
        P.gemm(xu, Wt["conv_in.w"], self.channels[0], 1, hh, ww, x, taps=9, bias=Wt["conv_in.b"])
        feats = []
        for i, (ci, co, down) in enumerate(body_layout(self.channels)):
            if down:
                hp, wp = (hh + 1) // 2, (ww + 1) // 2
                pooled = torch.empty((hp * wp, ci), **f16)
                P.avgpool2_ceil(x, hh, ww, ci, pooled)
                x, hh, ww = pooled, hp, wp
            M = hh * ww
            if ci != co:
                t = torch.empty((M, co), **f16)
                P.gemm(x, Wt[f"{i}.in_conv.w"], co, 1, 1, M, t, bias=Wt[f"{i}.in_conv.b"])
                x = t
            feat = torch.empty((M, co), **f16)
            for j in range(self.packed.num_res_blocks):
                xr = x if j == 0 else feat
                hb = scratch("h", M, co)
                P.gemm(xr, Wt[f"{i}.{j}.block1.w"], co, 1, hh, ww, hb, taps=9, bias=Wt[f"{i}.{j}.block1.b"], relu=True)
                P.gemm(hb, Wt[f"{i}.{j}.block2.w"], co, 1, 1, M, feat, bias=Wt[f"{i}.{j}.block2.b"], res=xr)
            feats.append(feat)
            x = feat
        states = [torch.zeros_like(f) for f in feats]
        e = self._plans[(h, w)] = dict(img=img, feats=feats, states=states, prog=P.finalize())
        return e

    @torch.no_grad()
    def compute(self, image_u8, h, w, scale):
        """Fill the features and the scaled states of latent size (h, w) from ``image_u8``, a uint8 [8h, 8w] or
        [8h, 8w, C] tensor (already resized, in the adapter's channel count).  Returns the four features."""
        e = self._plan(h, w)
        img = image_u8 if image_u8.dim() == 3 else image_u8[..., None]
        if tuple(img.shape) != tuple(e["img"].shape) or img.dtype != torch.uint8:
            raise ValueError(f"the adapter image must be uint8 {tuple(e['img'].shape)} (got {image_u8.dtype} "
                             f"{tuple(image_u8.shape)})")
        e["img"].copy_(img)
        e["prog"].run()
        for f, st in zip(e["feats"], e["states"]):
            torch.mul(f, float(scale), out=st)          # the pipeline's fp16 ``v * adapter_conditioning_scale``
        return e["feats"]
