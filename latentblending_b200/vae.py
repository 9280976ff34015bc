"""AutoencoderKL decoder on liblb200 (SURVEY.md section 8f "next #1").

Replaces ``pipe.vae.decode(latents / scaling_factor)`` + ``image_processor.postprocess`` inside
``DiffusersHolder.latent2image`` (latentblending/diffusers_holder.py:114-143; diffusers 0.25.0
autoencoder_kl.py / vae.py, un-vendored).  The reference runs the stock SDXL VAE in fp32
(force_upcast); here the decoder runs in fp16 storage / fp32 accumulation on the same wgmma
implicit-GEMM conv, GroupNorm and sampler kernels as the UNet -- 10.5 TFLOP per 1024^2 frame.
``dtype=torch.bfloat16`` stores every activation in bf16 instead (fp32's exponent range, the fp16 wgmma rate): the
decoder for VAEs whose activations overflow fp16, which is what force_upcast says of the stock SDXL VAE.
The mid-block single-head attention (head dim 512, S = h*w) is three GEMMs around a row softmax:
scores = (Wq x)(Wk x)^T (1/sqrt(C) folded into Wq), P = softmax_rows(scores), out = P V with V^T
produced directly by a GEMM with swapped operands; the value bias is folded into the output bias
(softmax rows sum to one).  Weights use the diffusers state_dict names.
``VAEEncoderB200`` is the matching encoder (image keyframes, DiffusersHolder.image2latent): the same resnet and
attention lowering, a fused image-preprocessing conv_in and the asymmetric-pad stride-2 downsamples.
"""
import torch

from . import _cabi
from ._cabi import ctx
from .lowering import (Scratch, lower_conv_out, lower_resnet, lower_vae_attention, pack3, pack_resnet,
                       pack_vae_attention)
from .program import Program, pack_conv_out8


class DecoderBase:
    """What every native VAE decoder shares (this one and taesd.TinyVAEDecoderB200): one lowered program per latent
    size (``_lower(h, w)``: an object with ``z_in``, ``prog`` and ``frame``), and the count of non-finite pixels the
    post-process kernel saw (``_overflow_message(n)`` says what it means for the decoder)."""

    def __init__(self, device):
        self.device = torch.device(device)
        self.dev_index = self.device.index or 0
        self._plans = {}
        self.nonfinite = torch.zeros(1, dtype=torch.int32, device=self.device)
        self.decodes_since_check = 0

    def plan(self, h, w):
        if (h, w) not in self._plans:
            self._plans[(h, w)] = self._lower(h, w)
        return self._plans[(h, w)]

    @torch.no_grad()
    def decode_to_u8(self, latents):
        """latents [1,4,h,w] fp16 (CUDA) -> uint8 [8h,8w,3] frame on the device."""
        assert latents.is_cuda and latents.shape[0] == 1, "VAE decode: one CUDA latent at a time"
        _, _, h, w = latents.shape
        pl = self.plan(h, w)
        pl.z_in.copy_(latents)
        pl.prog.run()
        self.decodes_since_check += 1
        return pl.frame.clone()

    def overflow_count(self):
        """Non-finite pixels seen by the post-process kernel since the last call (device->host read: call it at a
        point that synchronises anyway).  The fp16 decoder stores fp16 where the reference upcasts the stock SDXL VAE to
        fp32 (diffusers_holder.py:128-133); with weights that overflow fp16 this is > 0 and the frames are invalid."""
        n = int(self.nonfinite.item())
        if n:
            self.nonfinite.zero_()
        self.decodes_since_check = 0
        return n

    def check_overflow(self):
        n = self.overflow_count()
        if n:
            raise _cabi.LB200Error(self._overflow_message(n))


class VAEDecoderB200(DecoderBase):
    def __init__(self, state_dict, channels, scaling_factor, device, groups=32, dtype=torch.float16):
        """``dtype``: torch.float16 or torch.bfloat16, the storage type of weights and activations (fp32 accumulation
        either way).  Weights are cast once from the state dict's own dtype; folded biases are formed in fp32."""
        if dtype not in (torch.float16, torch.bfloat16):
            raise ValueError(f"VAE decoder dtype must be torch.float16 or torch.bfloat16 (got {dtype})")
        super().__init__(device)
        self.channels = tuple(channels)
        self.scaling_factor = scaling_factor
        self.groups = groups
        self.dtype = dtype
        sd = state_dict
        dev = self.device

        def g(n):
            return sd[n].detach().to(device=dev, dtype=dtype).contiguous()

        def gf(n):
            return sd[n].detach().to(device=dev, dtype=torch.float32)

        W = self.w = {}
        pq = gf("post_quant_conv.weight")
        C = pq.shape[0]
        W["prep.w"] = (pq.reshape(C, C) / scaling_factor).contiguous()
        W["prep.b"] = gf("post_quant_conv.bias").contiguous()
        W["conv_in.w"] = g("conv_in.weight").permute(2, 3, 1, 0).contiguous()
        W["conv_in.b"] = g("conv_in.bias")
        self.resnets = [k[: -len(".norm1.weight")] for k in sd if k.endswith(".norm1.weight")]
        for r in self.resnets:
            pack_resnet(W, r, sd, g)
        pack_vae_attention(W, "mid_block.attentions.0", sd, g, gf, dtype)
        for k in sd:
            if k.endswith("upsamplers.0.conv.weight"):
                nm = k[: -len(".weight")]
                W[nm + ".w"], W[nm + ".b"] = pack3(g(nm + ".weight")), g(nm + ".bias")
        W["norm_out.g"], W["norm_out.b"] = g("conv_norm_out.weight"), g("conv_norm_out.bias")
        W["conv_out.w8"], W["conv_out.b8"] = pack_conv_out8(g("conv_out.weight").permute(0, 2, 3, 1),
                                                            g("conv_out.bias"))
    def _lower(self, h, w):
        return _VAELowering(self, h, w)

    def _overflow_message(self, n):
        if self.dtype == torch.float16:
            return (f"VAE decode produced {n} non-finite pixels: these VAE weights overflow fp16 (the reference upcasts "
                    "the stock SDXL VAE to fp32, diffusers_holder.py:128-133); decode in bf16 instead "
                    "(DiffusersHolder.set_vae_dtype(\"bf16\"), chosen automatically when the VAE config sets "
                    "force_upcast) or use the fp16-safe SDXL VAE weights (madebyollin/sdxl-vae-fp16-fix)")
        return f"VAE decode produced {n} non-finite pixels in bf16: the latents or the VAE weights are not finite"


class _VAELowering:
    def __init__(self, vae: VAEDecoderB200, h, w):
        Wt, dev, groups = vae.w, vae.device, vae.groups
        f16 = dict(dtype=torch.float16, device=dev)
        act = dict(dtype=vae.dtype, device=dev)       # activations and scratch: the decoder's type
        ch = list(reversed(vae.channels))            # e.g. [512, 512, 256, 128]
        B = 1
        P = self.prog = Program(vae.dev_index)
        self.z_in = torch.zeros(1, 4, h, w, **f16)
        H, W_ = 8 * h, 8 * w
        self.frame = torch.zeros(H, W_, 3, dtype=torch.uint8, device=dev)
        self.ws = torch.zeros(max(1 << 16, _cabi.load().lb_groupnorm_workspace_bytes(ctx(vae.dev_index), B, H * W_, groups)),
                              dtype=torch.uint8, device=dev)
        sc = Scratch(vae.dtype, dev)

        def resnet(rname, x, cin, cout, hh, ww, out):
            lower_resnet(P, Wt, rname, x, cin, cout, B, hh, ww, out, groups, 1e-6, self.ws, sc)

        z = torch.empty(1, 4, h, w, **act)
        P.latent_prep(self.z_in, Wt["prep.w"], Wt["prep.b"], z)
        C0 = ch[0]
        S = h * w
        x = torch.empty(S, C0, **act)
        P.conv_in(z, Wt["conv_in.w"], Wt["conv_in.b"], C0, x)
        x2 = torch.empty(S, C0, **act)
        resnet("mid_block.resnets.0", x, C0, C0, h, w, x2)
        x3 = torch.empty(S, C0, **act)
        lower_vae_attention(P, Wt, x2, S, C0, groups, self.ws, sc, x3)      # mid-block attention (single head, dim C0)
        x4 = torch.empty(S, C0, **act)
        resnet("mid_block.resnets.1", x3, C0, C0, h, w, x4)
        x, cin, hh, ww = x4, C0, h, w
        ping = {}
        for i, cout in enumerate(ch):
            for j in range(3):
                out = torch.empty(hh * ww, cout, **act) if (i, j) not in ping else ping[(i, j)]
                resnet(f"up_blocks.{i}.resnets.{j}", x, cin, cout, hh, ww, out)
                x, cin = out, cout
            nm = f"up_blocks.{i}.upsamplers.0.conv"
            if (nm + ".w") in Wt:
                up = torch.empty(4 * hh * ww, cout, **act)
                P.upsample_nearest(x, B, hh, ww, cout, up, 2 * hh, 2 * ww)
                hh, ww = 2 * hh, 2 * ww
                nx = torch.empty(hh * ww, cout, **act)
                P.gemm(up, Wt[nm + ".w"], cout, B, hh, ww, nx, taps=9, bias=Wt[nm + ".b"])
                x = nx
        no = sc("n1", hh * ww, cin)
        P.groupnorm(x, B, hh * ww, cin, groups, Wt["norm_out.g"], Wt["norm_out.b"], 1e-6, 1, no, self.ws)
        img = torch.empty(1, 3, hh, ww, **act)
        lower_conv_out(P, Wt, no, B, hh, ww, cin, 3, img, sc)
        P.postprocess_u8(img, self.frame, vae.nonfinite)
        P.finalize()


class VAEEncoderB200:
    """AutoencoderKL encoder (diffusers 0.25.0 ``Encoder`` + ``quant_conv``) on liblb200: a uint8 image in, the
    posterior mean times ``scaling_factor`` out -- ``retrieve_latents(vae.encode(x), sample_mode="argmax")`` as the
    img2img pipelines use it.  conv_in reads the image with VaeImageProcessor.preprocess fused (lb_image_conv_in);
    4 down blocks x 2 resnets; 3 Downsample2D(padding=0) as a patch matrix (lb_im2col_s2_pad01) and one GEMM each; the
    decoder's mid block (resnet, single-head attention, resnet); GroupNorm + SiLU and conv_out.  quant_conv (1x1, 8 -> 8)
    and scaling_factor are folded into conv_out's first four output rows in fp32, so the last conv is one N = 8 GEMM
    producing the scaled mean.  ``dtype``: fp16 or bf16 storage, fp32 accumulation.  One graph-replayed program per
    image size; ``state_dict``: the diffusers names with ``encoder.`` stripped, plus ``quant_conv.*``."""

    def __init__(self, state_dict, channels, scaling_factor, device, groups=32, dtype=torch.float16,
                 layers_per_block=2):
        if dtype not in (torch.float16, torch.bfloat16):
            raise ValueError(f"VAE encoder dtype must be torch.float16 or torch.bfloat16 (got {dtype})")
        self.device = torch.device(device)
        self.dev_index = self.device.index or 0
        self.channels = tuple(channels)
        self.scaling_factor = float(scaling_factor)
        self.groups, self.dtype, self.layers_per_block = groups, dtype, layers_per_block
        self._plans = {}
        self.nonfinite = torch.zeros(1, dtype=torch.int32, device=self.device)
        sd, dev = state_dict, self.device

        def g(n):
            return sd[n].detach().to(device=dev, dtype=dtype).contiguous()

        def gf(n):
            return sd[n].detach().to(device=dev, dtype=torch.float32)

        W = self.w = {}
        W["conv_in.w"] = g("conv_in.weight").permute(2, 3, 1, 0).contiguous()       # [ky][kx][Cin][Cout]
        W["conv_in.b"] = g("conv_in.bias")
        for r in [k[: -len(".norm1.weight")] for k in sd if k.endswith(".norm1.weight")]:
            pack_resnet(W, r, sd, g)
        for i in range(len(self.channels) - 1):
            nm = f"down_blocks.{i}.downsamplers.0.conv"
            W[nm + ".w"], W[nm + ".b"] = pack3(g(nm + ".weight")), g(nm + ".bias")
        pack_vae_attention(W, "mid_block.attentions.0", sd, g, gf, dtype)
        W["norm_out.g"], W["norm_out.b"] = g("conv_norm_out.weight"), g("conv_norm_out.bias")
        # scaling_factor * (quant_conv(conv_out(x)))[:4]: the mean half of the moments, folded in fp32
        wo, bo = gf("conv_out.weight"), gf("conv_out.bias")                         # [8, C, 3, 3], [8]
        q = gf("quant_conv.weight").reshape(wo.shape[0], wo.shape[0])[:4]
        qb = gf("quant_conv.bias")[:4]
        wm = (self.scaling_factor * (q @ wo.reshape(wo.shape[0], -1))).reshape(4, *wo.shape[1:])
        bm = self.scaling_factor * (q @ bo + qb)
        W["conv_out.w8"], W["conv_out.b8"] = pack_conv_out8(wm.permute(0, 2, 3, 1).to(dtype), bm.to(dtype))

    def plan(self, h, w):
        if (h, w) not in self._plans:
            self._plans[(h, w)] = _VAEEncoderLowering(self, h, w)
        return self._plans[(h, w)]

    @torch.no_grad()
    def encode(self, image_u8):
        """uint8 [H, W, 3] image on the device (H, W multiples of 8) -> [1, 4, H/8, W/8] scaled posterior mean in
        the encoder's storage type (a view of the plan's output buffer: the next encode of this size overwrites it)."""
        assert image_u8.is_cuda and image_u8.dtype == torch.uint8 and image_u8.dim() == 3, \
            "VAE encode: one uint8 HxWxC CUDA image"
        H, W_, _ = image_u8.shape
        if H % 8 or W_ % 8:
            raise ValueError(f"VAE encode: the image sides must be multiples of 8 (got {W_}x{H})")
        pl = self.plan(H // 8, W_ // 8)
        pl.img.copy_(image_u8)
        pl.prog.run()
        return pl.x0

    def check_finite(self, x0):
        """Raise when ``x0`` holds non-finite values: the count comes from lb_add_noise_rows' device counter (no rows
        written), read once per encode."""
        from . import ops
        self.nonfinite.zero_()
        ops.add_noise_rows(x0, torch.empty(x0.shape, dtype=torch.float16, device=x0.device),
                           torch.empty((0, 2), dtype=torch.float16, device=x0.device), _cabi.ADD_NOISE_SIGMA,
                           nonfinite=self.nonfinite)
        n = int(self.nonfinite.item())
        if n:
            if self.dtype == torch.float16:
                raise _cabi.LB200Error(
                    f"VAE encode produced {n} non-finite latents: these VAE weights overflow fp16 (the stock SDXL VAE "
                    "does; its config sets force_upcast); encode in bf16 instead (DiffusersHolder.set_vae_dtype(\"bf16\"), "
                    "chosen automatically when the VAE config sets force_upcast) or use the fp16-safe SDXL VAE weights "
                    "(madebyollin/sdxl-vae-fp16-fix)")
            raise _cabi.LB200Error(f"VAE encode produced {n} non-finite latents in bf16: the VAE weights are not finite")


class _VAEEncoderLowering:
    def __init__(self, enc: VAEEncoderB200, h, w):
        Wt, dev, groups = enc.w, enc.device, enc.groups
        act = dict(dtype=enc.dtype, device=dev)
        ch = list(enc.channels)                       # e.g. [128, 256, 512, 512]
        B = 1
        H, W_ = 8 * h, 8 * w
        P = self.prog = Program(enc.dev_index)
        self.img = torch.zeros(H, W_, 3, dtype=torch.uint8, device=dev)
        self.ws = torch.zeros(max(1 << 16, _cabi.load().lb_groupnorm_workspace_bytes(ctx(enc.dev_index), B, H * W_,
                                                                                      groups)),
                              dtype=torch.uint8, device=dev)
        sc = Scratch(enc.dtype, dev)

        def resnet(rname, x, cin, cout, hh, ww, out):
            lower_resnet(P, Wt, rname, x, cin, cout, B, hh, ww, out, groups, 1e-6, self.ws, sc)

        hh, ww, cin = H, W_, ch[0]
        x = torch.empty(hh * ww, cin, **act)
        P.image_conv_in(self.img.view(H * W_, 3), B, H, W_, Wt["conv_in.w"], Wt["conv_in.b"], cin, x)
        for i, cout in enumerate(ch):
            for j in range(enc.layers_per_block):
                out = torch.empty(hh * ww, cout, **act)
                resnet(f"down_blocks.{i}.resnets.{j}", x, cin, cout, hh, ww, out)
                x, cin = out, cout
            nm = f"down_blocks.{i}.downsamplers.0.conv"
            if (nm + ".w") in Wt:
                ho, wo = (hh - 2) // 2 + 1, (ww - 2) // 2 + 1
                cols = sc("im2col", ho * wo, 9 * cout)        # the largest level's patch matrix, reused by the next
                P.im2col_s2_pad01(x, B, hh, ww, cout, cols)
                nx = torch.empty(ho * wo, cout, **act)
                P.gemm(cols, Wt[nm + ".w"], cout, 1, 1, ho * wo, nx, bias=Wt[nm + ".b"])
                x, hh, ww = nx, ho, wo
        assert (hh, ww) == (h, w), f"VAE encoder: {H}x{W_} does not reduce to {h}x{w}"
        C0, S = cin, h * w
        x2 = torch.empty(S, C0, **act)
        resnet("mid_block.resnets.0", x, C0, C0, h, w, x2)
        x3 = torch.empty(S, C0, **act)
        lower_vae_attention(P, Wt, x2, S, C0, groups, self.ws, sc, x3)
        x4 = torch.empty(S, C0, **act)
        resnet("mid_block.resnets.1", x3, C0, C0, h, w, x4)
        no = sc("n1", S, C0)
        P.groupnorm(x4, B, S, C0, groups, Wt["norm_out.g"], Wt["norm_out.b"], 1e-6, 1, no, self.ws)
        self.x0 = torch.empty(1, 4, h, w, **act)
        lower_conv_out(P, Wt, no, B, h, w, C0, 4, self.x0, sc)
        P.finalize()
