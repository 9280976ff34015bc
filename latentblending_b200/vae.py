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
"""
import torch

from . import _cabi
from ._cabi import ctx
from .lowering import Scratch, lower_conv_out, lower_resnet, pack3, pack_resnet
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
        a = "mid_block.attentions.0"
        Cm = sd[a + ".to_q.weight"].shape[0]
        scale = Cm ** -0.5
        W["attn.norm.g"], W["attn.norm.b"] = g(a + ".group_norm.weight"), g(a + ".group_norm.bias")
        W["attn.qk.w"] = torch.cat([(gf(a + ".to_q.weight") * scale), gf(a + ".to_k.weight")], 0).to(dtype).contiguous()
        W["attn.qk.b"] = torch.cat([(gf(a + ".to_q.bias") * scale), gf(a + ".to_k.bias")], 0).to(dtype).contiguous()
        W["attn.v.w"] = g(a + ".to_v.weight")
        W["attn.out.w"] = g(a + ".to_out.0.weight")
        W["attn.out.b"] = (gf(a + ".to_out.0.bias") + gf(a + ".to_out.0.weight") @ gf(a + ".to_v.bias")).to(dtype).contiguous()
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
        # mid-block attention (single head, dim C0)
        # V^T and the scores take the keys as the GEMM's N, which must be a multiple of 8: hn and qk get S8 >= S rows,
        # the extra ones zero (never written), so the extra V^T and score columns are exact zeros
        S8 = -(-S // 8) * 8
        hn = torch.zeros(S8, C0, **act)
        P.groupnorm(x2, B, S, C0, groups, Wt["attn.norm.g"], Wt["attn.norm.b"], 1e-6, 0, hn, self.ws)
        qk = torch.zeros(S8, 2 * C0, **act)
        P.gemm(hn, Wt["attn.qk.w"], 2 * C0, 1, 1, S, qk, bias=Wt["attn.qk.b"])
        # P V contracts over the S keys, and the GEMM's K must be a multiple of 64: P and V^T get Sp >= S8 columns, the
        # extra ones zero, which adds exact zeros to every dot product
        Sp = -(-S // 64) * 64
        vT = torch.zeros(C0, Sp, **act)
        P.gemm(Wt["attn.v.w"], hn, S8, 1, 1, C0, vT[:, :S8], static_w=False)             # V^T = Wv hn^T
        scores = torch.zeros(S, Sp, **f16)
        # bf16: the scores are stored in fp16 (LB_GEMM_OUT_F16), whose rounding is 8x finer than bf16's -- the error of
        # a score s becomes an exp(s) error -- and whose range their modest magnitudes do not approach; the softmax
        # writes the bf16 P over them (same 2-byte slots), which P V reads as a bf16 operand
        P.gemm(qk[:, :C0], qk[:, C0:], S8, 1, 1, S, scores[:, :S8], static_w=False)      # (scaled q) k^T
        probs = scores.view(vae.dtype)
        P.softmax_rows(scores[:, :S], probs[:, :S])
        att = sc("h1", S, C0)
        P.gemm(probs, vT, C0, 1, 1, S, att, static_w=False)                               # P V
        x3 = torch.empty(S, C0, **act)
        P.gemm(att, Wt["attn.out.w"], C0, 1, 1, S, x3, bias=Wt["attn.out.b"], res=x2)
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
