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

from .schedulers import EulerTables
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


class SyntheticSDXLPipe:
    vae_scale_factor = 8
    is_synthetic = True       # seeded random weights / embeddings: BlendingEngine may fall back to seeded LPIPS weights

    def __init__(self, name="stabilityai/stable-diffusion-xl-base-1.0", device="cuda:0", unet_cfg: UNetConfig = None,
                 seed=0, unet_state_dict=None, vae_state_dict=None, vae_channels=VAE_CHANNELS,
                 lpips_state_dict=None, vae_dtype="fp16", vae="kl"):
        """``vae_dtype``: "fp16" or "bf16", the storage type of the VAE decoder DiffusersHolder builds.
        ``vae``: "kl" (the SDXL AutoencoderKL decoder) or "tiny" (the AutoencoderTiny / TAESDXL decoder with its
        default config, scaling_factor 1.0, fp16 only; ``vae_state_dict`` then holds its ``decoder.``-stripped
        weights, seeded by ``random_tiny_vae_state_dict`` when omitted)."""
        if vae_dtype not in VAE_DTYPES:
            raise ValueError(f"vae_dtype must be one of {sorted(VAE_DTYPES)} (got {vae_dtype!r})")
        if vae not in ("kl", "tiny"):
            raise ValueError(f"vae must be 'kl' or 'tiny' (got {vae!r})")
        if vae == "tiny" and vae_dtype != "fp16":
            raise ValueError("the tiny VAE decoder runs in fp16 only (vae_dtype='fp16')")
        self._name_or_path = name
        self.device = torch.device(device)
        self._execution_device = self.device
        turbo = "turbo" in name
        self.unet_cfg = unet_cfg or (SDXL_TURBO if turbo else SDXL_BASE)
        self.default_sample_size = self.unet_cfg.sample_size
        self.scheduler = EulerTables("euler_ancestral" if turbo else "euler")
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
        self.vae_dtype = vae_dtype
        self.lpips_state_dict = lpips_state_dict
        self.h2d_bytes = 0        # bytes of conditioning copied host->device (bench e2e)

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


class DiffusersSDXLPipe:
    """Adapter: a loaded diffusers ``StableDiffusionXLPipeline`` (what the reference's constructor receives,
    latentblending/blending_engine.py:20-44 via AutoPipelineForText2Image) -> the attribute surface
    ``DiffusersHolder`` of this backend reads.  ``BlendingEngine(pipe)`` / ``DiffusersHolder(pipe)`` wrap a real
    pipeline automatically (``adapt_pipe``), so the reference's call

        pipe = AutoPipelineForText2Image.from_pretrained("stabilityai/stable-diffusion-xl-base-1.0", torch_dtype=torch.float16, variant="fp16")
        pipe.to("cuda"); be = BlendingEngine(pipe)

    keeps working.  What is taken from the pipeline: the UNet / VAE-decoder ``state_dict()`` (diffusers parameter names
    are the ones the packers use), the UNet config, the scheduler config (EulerTables), ``encode_prompt`` (the CLIP text
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
        ucfg = pipe.unet.config

        def get(k, default=None):
            return ucfg[k] if k in ucfg else getattr(ucfg, k, default)
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
            raise ValueError(f"this backend implements head dim 64 (SDXL); the pipeline's UNet has {sorted(head_dims)}")
        if get("addition_embed_type") != "text_time" or not get("use_linear_projection", False):
            raise ValueError("not an SDXL UNet (needs addition_embed_type='text_time', use_linear_projection=True)")
        pooled = int(get("projection_class_embeddings_input_dim")) - 6 * int(get("addition_time_embed_dim"))
        self.unet_cfg = UNetConfig(in_channels=get("in_channels"), out_channels=get("out_channels"),
                                   block_out_channels=boc, layers_per_block=get("layers_per_block"),
                                   transformer_layers=tl, head_dim=64, cross_attention_dim=get("cross_attention_dim"),
                                   addition_time_embed_dim=get("addition_time_embed_dim"), pooled_dim=pooled,
                                   norm_num_groups=get("norm_num_groups"), sample_size=get("sample_size"),
                                   time_cond_proj_dim=get("time_cond_proj_dim"))
        self.default_sample_size = getattr(pipe, "default_sample_size", self.unet_cfg.sample_size)
        self.vae_scale_factor = pipe.vae_scale_factor
        self.scheduler = tables_from_diffusers_scheduler(pipe.scheduler)
        self.unet_state_dict = pipe.unet.state_dict()
        vsd = pipe.vae.state_dict()
        vcfg = pipe.vae.config
        if type(pipe.vae).__name__ == "AutoencoderTiny":
            # the tiny autoencoder (e.g. madebyollin/taesdxl): its decoder only; fp16, the one precision it has here
            from .taesd import check_config, check_state_dict
            self.vae_kind = "tiny"
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
            self.vae_channels = tuple(vcfg["block_out_channels"] if "block_out_channels" in vcfg
                                      else vcfg.block_out_channels)
            self.vae_scaling_factor = float(vcfg["scaling_factor"] if "scaling_factor" in vcfg else vcfg.scaling_factor)
            self.vae_dtype = vae_dtype_from_config(vcfg)
        self.lpips_state_dict = lpips_state_dict if lpips_state_dict is not None else getattr(pipe, "lpips_state_dict", None)
        self.h2d_bytes = 0

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
