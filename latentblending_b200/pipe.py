"""SyntheticSDXLPipe: the ``pipe`` object handed to BlendingEngine when no diffusers
checkpoint is available (there is no network here): SDXL-shaped random-init weights
generated on the device, synthetic prompt embeddings, Euler scheduler tables.

It supplies what the reference's holder reads off a StableDiffusionXLPipeline
(latentblending/diffusers_holder.py; SURVEY.md section 8b): ``_name_or_path``,
``unet`` config, ``vae_scale_factor``, ``default_sample_size``, ``scheduler``,
``encode_prompt`` and the weights.  Bench-definition recipes (SURVEY.md section 8d):
  * weights: uniform(-1/sqrt(fan_in), 1/sqrt(fan_in)); residual-branch output
    projections (resnet conv2, attention to_out, FF out, transformer proj_out)
    scaled by 0.1; norm gains ~ 1 +- 0.1;
  * prompt embeddings: 0.5*N(0,1) [1,77,ctx] and N(0,1) [1,pooled] from a CPU
    generator seeded with crc32(prompt).
"""
import math
import zlib
from collections import OrderedDict

import torch

from .schedulers import DPMTables, EulerTables, LCMTables
from .unet import UNetConfig

SDXL_BASE = UNetConfig()
SDXL_TURBO = UNetConfig(sample_size=64)
VAE_CHANNELS = (128, 256, 512, 512)
VAE_DTYPES = {"fp16": torch.float16, "bf16": torch.bfloat16}     # pipe.vae_dtype -> the VAE decoder's storage type


def vae_dtype_from_config(vcfg):
    """"bf16" when an AutoencoderKL config asks to be upcast (``force_upcast``, True unless the config says otherwise:
    the diffusers default, set for the stock SDXL VAE whose activations overflow fp16), else "fp16".  The reference
    decodes such a VAE in fp32 (diffusers_holder.py:128-139); bf16 has fp32's exponent range at the fp16 tensor rate."""
    if isinstance(vcfg, dict):          # diffusers' FrozenDict
        up = vcfg["force_upcast"] if "force_upcast" in vcfg else True
    else:
        up = getattr(vcfg, "force_upcast", True)
    return "bf16" if up else "fp16"


def unet_param_shapes(cfg: UNetConfig):
    """diffusers state_dict names -> shapes of the SDXL UNet2DConditionModel."""
    P = OrderedDict()
    ch, T, X = list(cfg.block_out_channels), cfg.time_embed_dim, cfg.cross_attention_dim

    def lin(n, i, o, bias=True):
        P[n + ".weight"] = (o, i)
        if bias:
            P[n + ".bias"] = (o,)

    def conv(n, i, o, k):
        P[n + ".weight"] = (o, i, k, k)
        P[n + ".bias"] = (o,)

    def norm(n, c):
        P[n + ".weight"] = (c,)
        P[n + ".bias"] = (c,)

    def resnet(n, i, o):
        norm(n + ".norm1", i)
        conv(n + ".conv1", i, o, 3)
        lin(n + ".time_emb_proj", T, o)
        norm(n + ".norm2", o)
        conv(n + ".conv2", o, o, 3)
        if i != o:
            conv(n + ".conv_shortcut", i, o, 1)

    def transformer(n, c, depth):
        norm(n + ".norm", c)
        lin(n + ".proj_in", c, c)
        for d in range(depth):
            t = f"{n}.transformer_blocks.{d}"
            norm(t + ".norm1", c)
            for a, kdim in (("attn1", c), ("attn2", X)):
                lin(f"{t}.{a}.to_q", c, c, False)
                lin(f"{t}.{a}.to_k", kdim, c, False)
                lin(f"{t}.{a}.to_v", kdim, c, False)
                lin(f"{t}.{a}.to_out.0", c, c)
                if a == "attn1":
                    norm(t + ".norm2", c)
            norm(t + ".norm3", c)
            lin(t + ".ff.net.0.proj", c, 8 * c)
            lin(t + ".ff.net.2", 4 * c, c)
        lin(n + ".proj_out", c, c)

    conv("conv_in", cfg.in_channels, ch[0], 3)
    lin("time_embedding.linear_1", ch[0], T)
    if cfg.time_cond_proj_dim is not None:        # LCM-SDXL's guidance-scale embedding projection (no bias)
        lin("time_embedding.cond_proj", cfg.time_cond_proj_dim, ch[0], bias=False)
    lin("time_embedding.linear_2", T, T)
    lin("add_embedding.linear_1", cfg.add_in_dim, T)
    lin("add_embedding.linear_2", T, T)
    cout = ch[0]
    for i, c in enumerate(ch):
        cin, cout = cout, c
        for j in range(cfg.layers_per_block):
            resnet(f"down_blocks.{i}.resnets.{j}", cin if j == 0 else cout, cout)
            if cfg.transformer_layers[i]:
                transformer(f"down_blocks.{i}.attentions.{j}", cout, cfg.transformer_layers[i])
        if i < len(ch) - 1:
            conv(f"down_blocks.{i}.downsamplers.0.conv", cout, cout, 3)
    resnet("mid_block.resnets.0", ch[-1], ch[-1])
    transformer("mid_block.attentions.0", ch[-1], cfg.transformer_layers[-1])
    resnet("mid_block.resnets.1", ch[-1], ch[-1])
    rev, rdepth = list(reversed(ch)), list(reversed(cfg.transformer_layers))
    cout = rev[0]
    for i, c in enumerate(rev):
        cprev, cout = cout, c
        cin = rev[min(i + 1, len(ch) - 1)]
        n = cfg.layers_per_block + 1
        for j in range(n):
            skip_c = cin if j == n - 1 else cout
            res_in = cprev if j == 0 else cout
            resnet(f"up_blocks.{i}.resnets.{j}", res_in + skip_c, cout)
            if rdepth[i]:
                transformer(f"up_blocks.{i}.attentions.{j}", cout, rdepth[i])
        if i < len(ch) - 1:
            conv(f"up_blocks.{i}.upsamplers.0.conv", cout, cout, 3)
    norm("conv_norm_out", ch[0])
    conv("conv_out", ch[0], cfg.out_channels, 3)
    return P


def controlnet_param_shapes(cfg: UNetConfig, cond_channels=None):
    """diffusers state_dict names -> shapes of an SDXL ControlNetModel whose encoder is ``cfg`` (its own transformer
    depths): the UNet's conv_in, embeddings, down and mid blocks, the conditioning embedding
    (``controlnet_cond_embedding``) and the zero convs (``controlnet_down_blocks.{i}``, ``controlnet_mid_block``)."""
    from .controlnet import COND_CHANNELS, cond_embedding_layers, num_down_residuals
    cond_channels = COND_CHANNELS if cond_channels is None else tuple(cond_channels)
    P = OrderedDict((k, v) for k, v in unet_param_shapes(cfg).items()
                    if not k.startswith(("up_blocks.", "conv_norm_out.", "conv_out.", "mid_block.")))
    for name, cin, cout, _, _ in cond_embedding_layers(cond_channels, cfg.block_out_channels[0]):
        P[name + ".weight"], P[name + ".bias"] = (cout, cin, 3, 3), (cout,)
    L, ch = len(cfg.block_out_channels), cfg.block_out_channels
    chans = [ch[0]]
    for i in range(L):
        chans += [ch[i]] * cfg.layers_per_block + ([ch[i]] if i < L - 1 else [])
    assert len(chans) == num_down_residuals(cfg)
    for i, c in enumerate(chans):
        P[f"controlnet_down_blocks.{i}.weight"], P[f"controlnet_down_blocks.{i}.bias"] = (c, c, 1, 1), (c,)
    P.update((k, v) for k, v in unet_param_shapes(cfg).items() if k.startswith("mid_block."))
    P["controlnet_mid_block.weight"], P["controlnet_mid_block.bias"] = (ch[-1], ch[-1], 1, 1), (ch[-1],)
    return P


def controlnet_config(unet_cfg: UNetConfig, variant):
    """The encoder config of SyntheticSDXLPipe's ControlNet: "full" keeps the UNet's transformer depths (as
    diffusers/controlnet-canny-sdxl-1.0 does), "small" has one transformer block, in the mid block's level only."""
    import dataclasses
    L = len(unet_cfg.block_out_channels)
    if variant == "full":
        depths = tuple(unet_cfg.transformer_layers)
    elif variant == "small":
        depths = (0,) * (L - 1) + (1,)
    else:
        raise ValueError(f"controlnet must be None, 'full' or 'small' (got {variant!r})")
    return dataclasses.replace(unet_cfg, transformer_layers=depths, time_cond_proj_dim=None)


def random_controlnet_state_dict(cfg: UNetConfig, seed, device, damp=0.1):
    """Seeded ControlNet weights with ``random_state_dict``'s recipe.  The zero convs are damped like the other
    residual branches but not zero, so the control branch changes the UNet's output."""
    sd = random_state_dict(controlnet_param_shapes(cfg), seed, device, damp=damp)
    for k in sd:
        if k.startswith(("controlnet_down_blocks.", "controlnet_mid_block.")):
            sd[k] = (sd[k].float() * damp).to(sd[k].dtype)
    return sd


def adapter_param_shapes(in_channels=3, channels=(320, 640, 1280, 1280), num_res_blocks=2, downscale_factor=16):
    """diffusers state_dict names -> shapes of an SDXL T2IAdapter (``adapter_type="full_adapter_xl"``): conv_in on
    the pixel-unshuffled image, then four AdapterBlocks (t2i_adapter.body_layout), a 1x1 in_conv where the channel
    count changes and ``num_res_blocks`` resnets of a 3x3 block1 and a 1x1 block2 each."""
    from .t2i_adapter import body_layout
    P = OrderedDict()
    P["adapter.conv_in.weight"] = (channels[0], in_channels * downscale_factor ** 2, 3, 3)
    P["adapter.conv_in.bias"] = (channels[0],)
    for i, (ci, co, _) in enumerate(body_layout(channels)):
        if ci != co:
            P[f"adapter.body.{i}.in_conv.weight"], P[f"adapter.body.{i}.in_conv.bias"] = (co, ci, 1, 1), (co,)
        for j in range(num_res_blocks):
            q = f"adapter.body.{i}.resnets.{j}"
            P[q + ".block1.weight"], P[q + ".block1.bias"] = (co, co, 3, 3), (co,)
            P[q + ".block2.weight"], P[q + ".block2.bias"] = (co, co, 1, 1), (co,)
    return P


def random_adapter_state_dict(cfg, seed, device, damp=0.1):
    """Seeded T2I-Adapter weights (``cfg``: the T2IAdapter config keys) with ``random_state_dict``'s recipe.  Every
    block2 is damped like the other residual branches, but not zeroed, so the features change the UNet's output."""
    shapes = adapter_param_shapes(cfg["in_channels"], cfg["channels"], cfg["num_res_blocks"], cfg["downscale_factor"])
    sd = random_state_dict(shapes, seed, device, damp=damp)
    for k in sd:
        if ".block2." in k:
            sd[k] = (sd[k].float() * damp).to(sd[k].dtype)
    return sd


# SyntheticSDXLPipe seeds its T2I-Adapter weights with seed + this offset: no other synthetic state dict uses it
ADAPTER_SEED_OFFSET = 5003


def adapter_config(unet_cfg: UNetConfig, in_channels):
    """The T2IAdapter config of an SDXL adapter for ``unet_cfg``: channels = block_out_channels + the last again."""
    ch = tuple(unet_cfg.block_out_channels)
    return dict(in_channels=in_channels, channels=ch + ch[-1:], num_res_blocks=2, downscale_factor=16,
                adapter_type="full_adapter_xl")


def vae_param_shapes(channels=VAE_CHANNELS, latent=4):
    P = OrderedDict()
    ch = list(reversed(channels))

    def conv(n, i, o, k):
        P[n + ".weight"] = (o, i, k, k)
        P[n + ".bias"] = (o,)

    def norm(n, c):
        P[n + ".weight"] = (c,)
        P[n + ".bias"] = (c,)

    def resnet(n, i, o):
        norm(n + ".norm1", i)
        conv(n + ".conv1", i, o, 3)
        norm(n + ".norm2", o)
        conv(n + ".conv2", o, o, 3)
        if i != o:
            conv(n + ".conv_shortcut", i, o, 1)

    conv("post_quant_conv", latent, latent, 1)
    conv("conv_in", latent, ch[0], 3)
    resnet("mid_block.resnets.0", ch[0], ch[0])
    norm("mid_block.attentions.0.group_norm", ch[0])
    for n in ("to_q", "to_k", "to_v", "to_out.0"):
        P[f"mid_block.attentions.0.{n}.weight"] = (ch[0], ch[0])
        P[f"mid_block.attentions.0.{n}.bias"] = (ch[0],)
    resnet("mid_block.resnets.1", ch[0], ch[0])
    cout = ch[0]
    for i, c in enumerate(ch):
        cin, cout = cout, c
        for j in range(3):
            resnet(f"up_blocks.{i}.resnets.{j}", cin if j == 0 else cout, cout)
        if i < len(ch) - 1:
            conv(f"up_blocks.{i}.upsamplers.0.conv", cout, cout, 3)
    norm("conv_norm_out", ch[-1])
    conv("conv_out", ch[-1], 3, 3)
    return P


def vae_encoder_param_shapes(channels=VAE_CHANNELS, latent=4, layers_per_block=2):
    """diffusers state_dict names of an AutoencoderKL's encoder (``encoder.`` stripped) and its ``quant_conv`` ->
    shapes: conv_in 3 -> C0, down blocks of ``layers_per_block`` resnets (a Downsample2D after all but the last), the
    mid block, conv_norm_out and conv_out to the 2 * latent moments."""
    P = OrderedDict()

    def conv(n, i, o, k):
        P[n + ".weight"] = (o, i, k, k)
        P[n + ".bias"] = (o,)

    def norm(n, c):
        P[n + ".weight"] = (c,)
        P[n + ".bias"] = (c,)

    def resnet(n, i, o):
        norm(n + ".norm1", i)
        conv(n + ".conv1", i, o, 3)
        norm(n + ".norm2", o)
        conv(n + ".conv2", o, o, 3)
        if i != o:
            conv(n + ".conv_shortcut", i, o, 1)

    ch = list(channels)
    conv("conv_in", 3, ch[0], 3)
    cout = ch[0]
    for i, c in enumerate(ch):
        cin, cout = cout, c
        for j in range(layers_per_block):
            resnet(f"down_blocks.{i}.resnets.{j}", cin if j == 0 else cout, cout)
        if i < len(ch) - 1:
            conv(f"down_blocks.{i}.downsamplers.0.conv", cout, cout, 3)
    resnet("mid_block.resnets.0", ch[-1], ch[-1])
    norm("mid_block.attentions.0.group_norm", ch[-1])
    for n in ("to_q", "to_k", "to_v", "to_out.0"):
        P[f"mid_block.attentions.0.{n}.weight"] = (ch[-1], ch[-1])
        P[f"mid_block.attentions.0.{n}.bias"] = (ch[-1],)
    resnet("mid_block.resnets.1", ch[-1], ch[-1])
    norm("conv_norm_out", ch[-1])
    conv("conv_out", ch[-1], 2 * latent, 3)
    conv("quant_conv", 2 * latent, 2 * latent, 1)
    return P


# SyntheticSDXLPipe seeds its VAE encoder weights with seed + this offset: no other synthetic state dict uses it
VAE_ENCODER_SEED_OFFSET = 4099


def tiny_vae_param_shapes(config=None):
    """diffusers state_dict names (``decoder.`` stripped) -> shapes of an AutoencoderTiny decoder."""
    from .taesd import decoder_layout, tiny_config
    cfg = tiny_config(config)
    ch = cfg["decoder_block_out_channels"]
    P = OrderedDict()
    for kind, idx, grp in decoder_layout(cfg):
        c = ch[grp]
        if kind == "block":
            for j in (0, 2, 4):
                P[f"layers.{idx}.conv.{j}.weight"] = (c, c, 3, 3)
                P[f"layers.{idx}.conv.{j}.bias"] = (c,)
        elif kind == "conv_in":
            P[f"layers.{idx}.weight"] = (c, cfg["latent_channels"], 3, 3)
            P[f"layers.{idx}.bias"] = (c,)
        elif kind == "up_conv":
            P[f"layers.{idx}.weight"] = (c, c, 3, 3)
        else:
            P[f"layers.{idx}.weight"] = (cfg["out_channels"], c, 3, 3)
            P[f"layers.{idx}.bias"] = (cfg["out_channels"],)
    return P


def random_tiny_vae_state_dict(seed, device, config=None, dtype=torch.float16):
    """Seeded tiny-VAE decoder weights whose frames are not degenerate.  35 convolutions and 31 ReLUs collapse a
    uniform(+-1/sqrt(fan_in)) init to a constant, so: every conv is He-uniform (+-sqrt(6/fan_in), variance 2/fan_in,
    which keeps the second moment through a ReLU); the third conv of each block is damped by 0.3 so the residual
    stream grows slowly; biases are 0.02 * uniform(+-1); the last conv is uniform(+-0.25/sqrt(fan_in)) with bias
    0.5, i.e. a mid-grey frame with a spread of a few tens of uint8 levels (decode returns layers(x) * 2 - 1)."""
    from .taesd import decoder_layout
    g = torch.Generator(device=device).manual_seed(seed)
    shapes = tiny_vae_param_shapes(config)
    last = [idx for kind, idx, _ in decoder_layout(config) if kind == "conv_out"][0]
    sd = OrderedDict()
    for name, shape in shapes.items():
        u = torch.rand(shape, generator=g, device=device) * 2 - 1
        if len(shape) >= 2:
            fan_in = shape[1] * shape[2] * shape[3]
            if name == f"layers.{last}.weight":
                t = u * (0.25 / math.sqrt(fan_in))
            else:
                t = u * math.sqrt(6.0 / fan_in)
                if name.endswith(".conv.4.weight"):
                    t = t * 0.3
        elif name == f"layers.{last}.bias":
            t = 0.5 + 0.02 * u
        else:
            t = 0.02 * u
        sd[name] = t.to(dtype)
    return sd


_DAMPED = ("conv2.weight", "conv2.bias", "to_out.0.weight", "to_out.0.bias", "ff.net.2.weight", "ff.net.2.bias",
           "proj_out.weight", "proj_out.bias")


def random_state_dict(shapes, seed, device, damp=0.1, dtype=torch.float16):
    g = torch.Generator(device=device).manual_seed(seed)
    sd = OrderedDict()
    for name, shape in shapes.items():
        if len(shape) >= 2:
            fan_in = 1
            for s in shape[1:]:
                fan_in *= s
            t = (torch.rand(shape, generator=g, device=device) * 2 - 1) * (1.0 / math.sqrt(fan_in))
        elif "norm" in name and name.endswith("weight"):
            t = 1.0 + 0.1 * (torch.rand(shape, generator=g, device=device) * 2 - 1)
        elif "norm" in name:
            t = 0.05 * (torch.rand(shape, generator=g, device=device) * 2 - 1)
        else:
            t = 0.02 * (torch.rand(shape, generator=g, device=device) * 2 - 1)
        if any(name.endswith(s) for s in _DAMPED):
            t = t * damp
        sd[name] = t.to(dtype)
    return sd


def prompt_seed(prompt: str) -> int:
    return zlib.crc32(prompt.encode("utf-8")) & 0x7FFFFFFF


# SyntheticSDXLPipe's DPM-Solver++ schedulers: DPMTables options of the common diffusers setups
DPM_SCHEDULERS = {
    "dpmpp_2m": dict(algorithm_type="dpmsolver++"),
    "dpmpp_2m_karras": dict(algorithm_type="dpmsolver++", use_karras_sigmas=True),
    "dpmpp_2m_sde": dict(algorithm_type="sde-dpmsolver++"),
    "dpmpp_2m_sde_karras": dict(algorithm_type="sde-dpmsolver++", use_karras_sigmas=True),
}


class SyntheticSDXLPipe:
    vae_scale_factor = 8
    is_synthetic = True       # seeded random weights / embeddings: BlendingEngine may fall back to seeded LPIPS weights

    def __init__(self, name="stabilityai/stable-diffusion-xl-base-1.0", device="cuda:0", unet_cfg: UNetConfig = None,
                 seed=0, unet_state_dict=None, vae_state_dict=None, vae_channels=VAE_CHANNELS,
                 lpips_state_dict=None, vae_dtype="fp16", vae="kl", scheduler=None, controlnet=None,
                 controlnet_state_dict=None, vae_encoder_state_dict=None, adapter=None, adapter_state_dict=None):
        """``scheduler``: None (Euler for SDXL base, Euler-ancestral for a name with "turbo"), "euler",
        "euler_ancestral", "lcm" (LCMScheduler tables: LCM-LoRA-style with the base UNet, LCM-SDXL-style with
        ``unet_cfg.time_cond_proj_dim`` set) or one of DPM_SCHEDULERS (DPMSolverMultistepScheduler tables for the SDXL
        config: DPM++ 2M or 2M SDE, leading or Karras sigmas).
        ``vae_dtype``: "fp16" or "bf16", the storage type of the VAE decoder DiffusersHolder builds.
        ``vae``: "kl" (the SDXL AutoencoderKL decoder) or "tiny" (the AutoencoderTiny / TAESDXL decoder with its
        default config, scaling_factor 1.0, fp16 only; ``vae_state_dict`` then holds its ``decoder.``-stripped
        weights, seeded by ``random_tiny_vae_state_dict`` when omitted).
        ``controlnet``: None, "full" or "small" (``controlnet_config``): an SDXL ControlNet with seeded weights
        (``random_controlnet_state_dict``) unless ``controlnet_state_dict`` is given.
        ``vae_encoder_state_dict``: the KL VAE's encoder + quant_conv weights (``vae_encoder_param_shapes``), seeded
        with ``seed + VAE_ENCODER_SEED_OFFSET`` when omitted; a tiny-VAE pipe has no encoder.
        ``adapter``: None, "rgb" or "gray": an SDXL T2I-Adapter taking 3 or 1 image channels (``adapter_config``) with
        weights seeded with ``seed + ADAPTER_SEED_OFFSET`` (``random_adapter_state_dict``) unless
        ``adapter_state_dict`` is given.  Not together with a ControlNet."""
        if vae_dtype not in VAE_DTYPES:
            raise ValueError(f"vae_dtype must be one of {sorted(VAE_DTYPES)} (got {vae_dtype!r})")
        if vae not in ("kl", "tiny"):
            raise ValueError(f"vae must be 'kl' or 'tiny' (got {vae!r})")
        if vae == "tiny" and vae_dtype != "fp16":
            raise ValueError("the tiny VAE decoder runs in fp16 only (vae_dtype='fp16')")
        if adapter not in (None, "rgb", "gray"):
            raise ValueError(f"adapter must be None, 'rgb' or 'gray' (got {adapter!r})")
        if adapter is not None and controlnet is not None:
            raise ValueError("a ControlNet and a T2I-Adapter together are not supported")
        if scheduler not in (None, "euler", "euler_ancestral", "lcm", *DPM_SCHEDULERS):
            raise ValueError(f"scheduler must be None, 'euler', 'euler_ancestral', 'lcm' or one of "
                             f"{sorted(DPM_SCHEDULERS)} (got {scheduler!r})")
        self._name_or_path = name
        self.device = torch.device(device)
        self._execution_device = self.device
        turbo = "turbo" in name
        self.unet_cfg = unet_cfg or (SDXL_TURBO if turbo else SDXL_BASE)
        self.default_sample_size = self.unet_cfg.sample_size
        if scheduler is None:
            scheduler = "euler_ancestral" if turbo else "euler"
        if scheduler in DPM_SCHEDULERS:
            self.scheduler = DPMTables(**DPM_SCHEDULERS[scheduler])
        else:
            self.scheduler = LCMTables() if scheduler == "lcm" else EulerTables(scheduler)
        self.unet_state_dict = unet_state_dict if unet_state_dict is not None else \
            random_state_dict(unet_param_shapes(self.unet_cfg), seed, self.device)
        self.vae_kind = vae
        if vae == "tiny":
            from .taesd import DEFAULT_CONFIG
            self.vae_config = dict(DEFAULT_CONFIG)
            self.vae_channels = tuple(DEFAULT_CONFIG["decoder_block_out_channels"])
            self.vae_state_dict = vae_state_dict if vae_state_dict is not None else \
                random_tiny_vae_state_dict(seed + 1, self.device)
            self.vae_scaling_factor = float(DEFAULT_CONFIG["scaling_factor"])
        else:
            self.vae_channels = tuple(vae_channels)
            self.vae_state_dict = vae_state_dict if vae_state_dict is not None else \
                random_state_dict(vae_param_shapes(vae_channels), seed + 1, self.device, damp=0.3)
            self.vae_scaling_factor = 0.13025
        # the KL encoder (image keyframes, DiffusersHolder.image2latent); the tiny autoencoder has none here
        self.vae_encoder_state_dict = None
        if vae == "kl":
            self.vae_encoder_state_dict = vae_encoder_state_dict if vae_encoder_state_dict is not None else \
                random_state_dict(vae_encoder_param_shapes(vae_channels), seed + VAE_ENCODER_SEED_OFFSET,
                                  self.device, damp=0.3)
        self.vae_dtype = vae_dtype
        self.lpips_state_dict = lpips_state_dict
        self.h2d_bytes = 0        # bytes of conditioning copied host->device (bench e2e)
        self.controlnet_cfg = self.controlnet_state_dict = None
        if controlnet is not None:
            self.controlnet_cfg = controlnet_config(self.unet_cfg, controlnet)
            self.controlnet_state_dict = controlnet_state_dict if controlnet_state_dict is not None else \
                random_controlnet_state_dict(self.controlnet_cfg, seed + 2, self.device)
        self.controlnet_cond_channels = None          # the default, controlnet.COND_CHANNELS
        self.controlnet_bgr = False
        self.adapter_cfg = self.adapter_state_dict = None
        if adapter is not None:
            self.adapter_cfg = adapter_config(self.unet_cfg, 3 if adapter == "rgb" else 1)
            self.adapter_state_dict = adapter_state_dict if adapter_state_dict is not None else \
                random_adapter_state_dict(self.adapter_cfg, seed + ADAPTER_SEED_OFFSET, self.device)

    def encode_prompt(self, prompt, negative_prompt=None, do_classifier_free_guidance=True, dtype=torch.float16):
        """Synthetic stand-in for StableDiffusionXLPipeline.encode_prompt (diffusers_holder.py:81-95)."""
        c = self.unet_cfg

        def emb(text):
            g = torch.Generator().manual_seed(prompt_seed(text))
            e = (torch.randn(1, 77, c.cross_attention_dim, generator=g) * 0.5).to(dtype)
            p = torch.randn(1, c.pooled_dim, generator=g).to(dtype)
            e, p = e.pin_memory(), p.pin_memory()
            self.h2d_bytes += e.numel() * e.element_size() + p.numel() * p.element_size()
            return e.to(self.device, non_blocking=True), p.to(self.device, non_blocking=True)

        pe, pp = emb(prompt)
        if not do_classifier_free_guidance:
            return pe, None, pp, None
        neg = negative_prompt[0] if isinstance(negative_prompt, (list, tuple)) else (negative_prompt or "")
        ne, npool = emb("<neg>" + neg)
        return pe, ne, pp, npool


def _sdxl_encoder_config(ucfg, what, defaults=None):
    """The UNetConfig of a diffusers SDXL UNet2DConditionModel or ControlNetModel config (``what`` names it in errors);
    keys the config lacks (a ControlNet has no out_channels or sample_size) come from ``defaults``."""

    def get(k, default=None):
        if k in ucfg:
            return ucfg[k]
        return getattr(ucfg, k, getattr(defaults, k, default) if defaults is not None else default)
    tl = get("transformer_layers_per_block", 1)
    down = list(get("down_block_types"))
    boc = tuple(get("block_out_channels"))
    if isinstance(tl, int):
        tl = [tl] * len(boc)
    tl = tuple(int(t) if "CrossAttn" in d else 0 for t, d in zip(tl, down))
    ahd = get("attention_head_dim")
    heads = ahd if isinstance(ahd, (list, tuple)) else [ahd] * len(boc)
    # SDXL's config stores the number of heads per level in attention_head_dim (5, 10, 20): head dim = C / heads
    head_dims = {c // h for c, h, t in zip(boc, heads, tl) if t}
    if head_dims != {64}:
        raise ValueError(f"this backend implements head dim 64 (SDXL); the pipeline's {what} has {sorted(head_dims)}")
    if get("addition_embed_type") != "text_time" or not get("use_linear_projection", False):
        raise ValueError(f"not an SDXL {what} (needs addition_embed_type='text_time', use_linear_projection=True)")
    pooled = int(get("projection_class_embeddings_input_dim")) - 6 * int(get("addition_time_embed_dim"))
    return UNetConfig(in_channels=get("in_channels"), out_channels=get("out_channels"),
                      block_out_channels=boc, layers_per_block=get("layers_per_block"),
                      transformer_layers=tl, head_dim=64, cross_attention_dim=get("cross_attention_dim"),
                      addition_time_embed_dim=get("addition_time_embed_dim"), pooled_dim=pooled,
                      norm_num_groups=get("norm_num_groups"), sample_size=get("sample_size"),
                      time_cond_proj_dim=get("time_cond_proj_dim"))


class DiffusersSDXLPipe:
    """Adapter: a loaded diffusers ``StableDiffusionXLPipeline`` (what the reference's constructor receives,
    latentblending/blending_engine.py:20-44 via AutoPipelineForText2Image) -> the attribute surface
    ``DiffusersHolder`` of this backend reads.  ``BlendingEngine(pipe)`` / ``DiffusersHolder(pipe)`` wrap a real
    pipeline automatically (``adapt_pipe``), so the reference's call

        pipe = AutoPipelineForText2Image.from_pretrained("stabilityai/stable-diffusion-xl-base-1.0", torch_dtype=torch.float16, variant="fp16")
        pipe.to("cuda"); be = BlendingEngine(pipe)

    keeps working.  What is taken from the pipeline: the UNet / VAE-decoder ``state_dict()`` (diffusers parameter names
    are the ones the packers use), the UNet config, the scheduler (EulerTables from its config, LCMTables for an
    LCMScheduler, DPMTables for a DPMSolverMultistepScheduler), ``encode_prompt`` (the CLIP text
    encoders stay PyTorch modules: they run once per prompt and are outside the hot path, SURVEY section 8f #4) and
    ``_execution_device`` / ``_name_or_path`` / ``default_sample_size`` / ``vae_scale_factor``.
    ``vae_dtype`` follows the VAE config: "bf16" when it sets ``force_upcast`` (the stock SDXL VAE, where the reference
    decodes in fp32), "fp16" for an fp16-safe VAE that turns it off.
    A ``pipe.vae`` of class ``AutoencoderTiny`` (``AutoencoderTiny.from_pretrained('madebyollin/taesdxl')``, as the
    reference's examples swap in) selects the tiny decoder: ``vae_kind`` "tiny", its ``decoder.`` weights and config,
    fp16.
    ``lpips_state_dict`` must be supplied (see INTEGRATION.md "LPIPS weights"): with real weights a random LPIPS
    network would silently steer the branch placement."""
    is_synthetic = False

    def __init__(self, pipe, lpips_state_dict=None):
        from .schedulers import tables_from_diffusers_scheduler
        self.inner = pipe
        self._name_or_path = getattr(pipe, "_name_or_path", None) or pipe.config.get("_name_or_path", "")
        self._execution_device = torch.device(pipe._execution_device)
        self.device = self._execution_device
        self.unet_cfg = _sdxl_encoder_config(pipe.unet.config, "UNet")
        self.default_sample_size = getattr(pipe, "default_sample_size", self.unet_cfg.sample_size)
        self.vae_scale_factor = pipe.vae_scale_factor
        self.scheduler = tables_from_diffusers_scheduler(pipe.scheduler)
        self.unet_state_dict = pipe.unet.state_dict()
        lora = [k for k in self.unet_state_dict if ".base_layer." in k or "lora_A" in k or "lora_B" in k]
        if lora:
            raise ValueError(f"the pipeline's UNet holds unfused LoRA layers ({len(lora)} keys, e.g. {lora[0]!r}): "
                             "fuse them into the weights first with pipe.fuse_lora(); pipe.unload_lora_weights()")
        self._take_controlnet(getattr(pipe, "controlnet", None))
        self._take_adapter(getattr(pipe, "adapter", None))
        vsd = pipe.vae.state_dict()
        vcfg = pipe.vae.config
        if type(pipe.vae).__name__ == "AutoencoderTiny":
            # the tiny autoencoder (e.g. madebyollin/taesdxl): its decoder only; fp16, the one precision it has here
            from .taesd import check_config, check_state_dict
            self.vae_kind = "tiny"
            self.vae_encoder_state_dict = None
            self.vae_config = check_config(vcfg)
            self.vae_state_dict = OrderedDict((k[len("decoder."):], v) for k, v in vsd.items()
                                              if k.startswith("decoder."))
            check_state_dict(self.vae_state_dict, self.vae_config)
            self.vae_channels = tuple(self.vae_config["decoder_block_out_channels"])
            self.vae_scaling_factor = float(self.vae_config["scaling_factor"])
            self.vae_dtype = "fp16"
        else:
            self.vae_kind = "kl"
            self.vae_state_dict = OrderedDict((k[len("decoder."):] if k.startswith("decoder.") else k, v)
                                              for k, v in vsd.items() if k.startswith(("decoder.", "post_quant_conv.")))
            # the encoder of image keyframes (None when the VAE was loaded without one)
            enc = OrderedDict((k[len("encoder."):] if k.startswith("encoder.") else k, v)
                              for k, v in vsd.items() if k.startswith(("encoder.", "quant_conv.")))
            self.vae_encoder_state_dict = enc if any(k.startswith("conv_in.") for k in enc) else None
            self.vae_channels = tuple(vcfg["block_out_channels"] if "block_out_channels" in vcfg
                                      else vcfg.block_out_channels)
            self.vae_scaling_factor = float(vcfg["scaling_factor"] if "scaling_factor" in vcfg else vcfg.scaling_factor)
            self.vae_dtype = vae_dtype_from_config(vcfg)
        self.lpips_state_dict = lpips_state_dict if lpips_state_dict is not None else getattr(pipe, "lpips_state_dict", None)
        self.h2d_bytes = 0

    def _take_controlnet(self, cn):
        """A StableDiffusionXLControlNetPipeline's ``controlnet`` (one ControlNetModel): its encoder config, the
        conditioning embedding's channels and channel order, and its state dict, every key of which the lowering
        must represent."""
        self.controlnet_cfg = self.controlnet_state_dict = self.controlnet_cond_channels = None
        self.controlnet_bgr = False
        if cn is None:
            return
        if type(cn).__name__ == "MultiControlNetModel" or isinstance(cn, (list, tuple)):
            raise ValueError("several ControlNets at once (MultiControlNetModel) are not supported")
        c = cn.config

        def get(k, default=None):
            return c[k] if k in c else getattr(c, k, default)
        if get("global_pool_conditions", False):
            raise ValueError("a ControlNet with global_pool_conditions=True is not supported")
        if get("conditioning_channels", 3) != 3:
            raise ValueError(f"the ControlNet takes {get('conditioning_channels')} conditioning channels; only 3 (an "
                             "RGB control image) are supported")
        if get("time_cond_proj_dim") is not None:
            raise ValueError("a ControlNet with time_embedding.cond_proj (time_cond_proj_dim) is not supported")
        order = get("controlnet_conditioning_channel_order", "rgb")
        if order not in ("rgb", "bgr"):
            raise ValueError(f"unknown controlnet_conditioning_channel_order {order!r}")
        ccfg = _sdxl_encoder_config(c, "ControlNet", defaults=self.unet_cfg)
        u = self.unet_cfg
        for f in ("in_channels", "block_out_channels", "layers_per_block", "cross_attention_dim",
                  "addition_time_embed_dim", "pooled_dim", "norm_num_groups"):
            if getattr(ccfg, f) != getattr(u, f):
                raise ValueError(f"the ControlNet's encoder does not match the UNet's: {f} {getattr(ccfg, f)} vs "
                                 f"{getattr(u, f)}")
        cond = tuple(get("conditioning_embedding_out_channels", (16, 32, 96, 256)))
        sd = cn.state_dict()
        want = controlnet_param_shapes(ccfg, cond)
        extra, missing = sorted(set(sd) - set(want)), sorted(set(want) - set(sd))
        if extra or missing:
            raise ValueError(f"the ControlNet's layout is not one this lowering represents: {len(extra)} unexpected "
                             f"keys (e.g. {extra[:3]}), {len(missing)} missing (e.g. {missing[:3]})")
        bad = [k for k, shp in want.items() if tuple(sd[k].shape) != shp]
        if bad:
            raise ValueError(f"the ControlNet's parameter shapes differ from its config's, e.g. {bad[0]!r}: "
                             f"{tuple(sd[bad[0]].shape)} vs {want[bad[0]]}")
        self.controlnet_cfg, self.controlnet_state_dict = ccfg, sd
        self.controlnet_cond_channels, self.controlnet_bgr = cond, order == "bgr"

    def _take_adapter(self, ad):
        """A StableDiffusionXLAdapterPipeline's ``adapter`` (one T2IAdapter of type "full_adapter_xl"): its config and
        its state dict, every key of which the lowering must represent."""
        self.adapter_cfg = self.adapter_state_dict = None
        if ad is None:
            return
        if type(ad).__name__ == "MultiAdapter" or isinstance(ad, (list, tuple)):
            raise ValueError("several T2I-Adapters at once (MultiAdapter) are not supported")
        if self.controlnet_state_dict is not None:
            raise ValueError("a pipeline with both a ControlNet and a T2I-Adapter is not supported")
        c = ad.config

        def get(k, default=None):
            return c[k] if k in c else getattr(c, k, default)
        kind = get("adapter_type", "full_adapter")
        if kind != "full_adapter_xl":
            raise ValueError(f"only the SDXL T2I-Adapter (adapter_type 'full_adapter_xl') is supported, not {kind!r}")
        cin = int(get("in_channels", 3))
        if cin not in (1, 3):
            raise ValueError(f"the T2I-Adapter takes {cin} image channels; only 1 or 3 are supported")
        cfg = dict(in_channels=cin, channels=tuple(get("channels")), num_res_blocks=int(get("num_res_blocks", 2)),
                   downscale_factor=int(get("downscale_factor", 16)), adapter_type=kind)
        if cfg["downscale_factor"] != 16:
            raise ValueError(f"the T2I-Adapter's downscale_factor is {cfg['downscale_factor']}; SDXL's is 16")
        ch = tuple(self.unet_cfg.block_out_channels)
        if len(ch) != 3 or cfg["channels"] != ch + ch[-1:]:
            raise ValueError(f"the T2I-Adapter's channels {cfg['channels']} do not match the UNet's "
                             f"block_out_channels {ch} followed by the last one again")
        sd = ad.state_dict()
        want = adapter_param_shapes(cin, cfg["channels"], cfg["num_res_blocks"], cfg["downscale_factor"])
        extra, missing = sorted(set(sd) - set(want)), sorted(set(want) - set(sd))
        if extra or missing:
            raise ValueError(f"the T2I-Adapter's layout is not one this lowering represents: {len(extra)} unexpected "
                             f"keys (e.g. {extra[:3]}), {len(missing)} missing (e.g. {missing[:3]})")
        bad = [k for k, shp in want.items() if tuple(sd[k].shape) != shp]
        if bad:
            raise ValueError(f"the T2I-Adapter's parameter shapes differ from its config's, e.g. {bad[0]!r}: "
                             f"{tuple(sd[bad[0]].shape)} vs {want[bad[0]]}")
        self.adapter_cfg, self.adapter_state_dict = cfg, sd

    def encode_prompt(self, prompt, negative_prompt=None, do_classifier_free_guidance=True, dtype=torch.float16):
        """diffusers_holder.py:79-96: the pipeline's own encode_prompt (both CLIP encoders), 4-tuple out."""
        pe, ne, pp, npool = self.inner.encode_prompt(
            prompt=prompt, prompt_2=prompt, device=self._execution_device, num_images_per_prompt=1,
            do_classifier_free_guidance=do_classifier_free_guidance, negative_prompt=negative_prompt,
            negative_prompt_2=negative_prompt)

        def cvt(t):
            return None if t is None else t.to(device=self._execution_device, dtype=dtype).contiguous()
        return cvt(pe), cvt(ne), cvt(pp), cvt(npool)


def adapt_pipe(pipe):
    """What DiffusersHolder is built on: our own pipe objects pass through, a diffusers pipeline is wrapped."""
    if hasattr(pipe, "unet_cfg") and hasattr(pipe, "unet_state_dict"):
        return pipe
    if hasattr(pipe, "unet") and hasattr(pipe, "vae") and hasattr(pipe, "encode_prompt"):
        return DiffusersSDXLPipe(pipe)
    raise TypeError("pipe must be a latentblending_b200 pipe (SyntheticSDXLPipe / DiffusersSDXLPipe) or a diffusers "
                    "StableDiffusionXLPipeline")


def lpips_state_dict_from_lpips(lpips_module):
    """{convs.i.weight/bias, lins.i.weight} from an ``lpips.LPIPS(net='alex')`` instance (lpips==0.1.4 layout:
    ``net.slice{1..5}`` hold AlexNet features 0,3,6,8,10; ``lin{0..4}.model[-1]`` the 1x1 weights)."""
    sd = lpips_module.state_dict()
    feats = (0, 3, 6, 8, 10)
    out = {}
    for i, f in enumerate(feats):
        wk = next(k for k in sd if k.endswith(f".{f}.weight") and k.startswith("net."))
        out[f"convs.{i}.weight"] = sd[wk]
        out[f"convs.{i}.bias"] = sd[wk[:-len("weight")] + "bias"]
        lk = next(k for k in sd if k.startswith(f"lin{i}.") and k.endswith("weight"))
        out[f"lins.{i}.weight"] = sd[lk]
    return out
