"""SDXL UNet on liblb200: weight packing + lowering of one forward pass to a C-ABI program.

Host side of the executor that replaces ``pipe.unet(...)`` in the reference's
denoise loop (latentblending/diffusers_holder.py:336-344).  Parameters are taken
by their diffusers ``state_dict`` names, so ``pipe.unet.state_dict()`` of a real
StableDiffusionXLPipeline can be passed as is.

Data layout in HBM (all fp16):
  * activations NHWC, i.e. [B*H*W, C] row-major with an explicit row stride so
    that channel slices of a wider buffer are first-class tensors; the nine
    ``torch.cat([hidden, skip])`` of the up path are never materialised: every
    skip tensor is written by its producer straight into the right half of its
    future concat buffer and read from there by the down path;
  * weights [N, K] row-major (K-major for the tensor core B operand); 3x3 conv
    weights [Cout][ky][kx][Cin]; a resnet's 1x1 shortcut is appended along K of
    conv2 (one accumulator, biases pre-summed); to_q/to_k/to_v fused to one
    [3C, C] matrix, cross-attention to_k/to_v to [2C, ctx]; GEGLU rows
    interleaved per 128-row tile (64 value rows then their 64 gate rows);
    all resnet ``time_emb_proj`` stacked into one [sum Cout, T] matrix.
  * latents / eps stay NCHW [B,4,h,w] like the reference's tensors.
"""
import ctypes
import os
from dataclasses import dataclass
from typing import Tuple

import torch

from . import _cabi
from ._cabi import (GEMM_RELU, GEMM_STATIC_W, OP_ATTENTION, OP_CONV_IN, OP_CONV_OUT, OP_EMBED_INPUTS, OP_GEMM,
                    OP_GROUPNORM, OP_IM2COL, OP_IM2COL_S2, OP_LATENT_PREP, OP_LAYERNORM, OP_LINEAR_SMALL,
                    OP_LPIPS_IM2COL_U8, OP_MAXPOOL3S2, OP_NHWC_TO_NCHW, OP_POSTPROCESS_U8, OP_SOFTMAX_ROWS, OP_UPSAMPLE2X, Op, check, ctx,
                    stream_ptr)


@dataclass
class UNetConfig:
    in_channels: int = 4
    out_channels: int = 4
    block_out_channels: Tuple[int, ...] = (320, 640, 1280)
    layers_per_block: int = 2
    transformer_layers: Tuple[int, ...] = (0, 2, 10)
    head_dim: int = 64
    cross_attention_dim: int = 2048
    addition_time_embed_dim: int = 256
    pooled_dim: int = 1280
    norm_num_groups: int = 32
    sample_size: int = 128
    time_cond_proj_dim: object = None

    @property
    def time_embed_dim(self):
        return self.block_out_channels[0] * 4

    @property
    def add_in_dim(self):
        return self.pooled_dim + 6 * self.addition_time_embed_dim


def _p(t):
    return None if t is None else t.data_ptr()


class Program:
    """A recorded op list; ``finalize`` hands it to lb_program_create."""

    def __init__(self, device_index):
        self.dev = device_index
        self.ops = []
        self.keep = []          # tensors referenced by raw pointers must outlive the program
        self.handle = None

    def _new(self, kind):
        op = Op()
        op.kind = kind
        self.ops.append(op)
        return op

    def hold(self, *ts):
        self.keep.extend(t for t in ts if t is not None)

    # -- op emitters (mirror latentblending_b200.ops, but record instead of launching) --------
    def gemm(self, a0, w, N, B, H, W, out, taps=1, a0_c=None, a1=None, a1_c=None, bias=None, bias2=None, res=None,
             mode=0, static_w=True, relu=False, ln=None, stats_out=None, depth_to_space=False):
        """``static_w``: ``w`` holds model weights (not written by the preceding op), so the kernel may fetch its
        first tiles before the preceding kernel has finished (LB_GEMM_STATIC_W).  Pass False when an activation
        is used as the B operand.
        ``depth_to_space``: nearest-2x upsample + 3x3 conv as one GEMM (LB_GEMM_D2S2): ``w`` holds the four phase
        filters [4*Co, 9*C], ``out`` the [B*2H*2W, Co] upsampled map.
        ``ln``: dict(stats=[M,parts,2] fp32, csum=[N] fp32, bias=[N] fp32, eps) -- LayerNorm folded into this GEMM
        (``w`` must already hold w*gamma; see include/lb200.h).  ``stats_out``: [M,parts,2] fp32 buffer that receives
        this GEMM's per-row partial sums for a following LN-folded GEMM (parts = self.gemm_stats_parts(...)).
        Element types come from the tensors as in ``ops.gemm``: bf16 operands (LB_GEMM_BF16) write ``out``'s type."""
        from .ops import gemm_dtype_mode
        dmode = gemm_dtype_mode(a0, w, out.dtype, a1, bias, bias2, res)
        d = self._new(OP_GEMM).u.gemm
        d.a0, d.a0_ld, d.a0_c = _p(a0), a0.stride(0), (a0.shape[1] if a0_c is None else a0_c)
        if a1 is not None:
            d.a1, d.a1_ld, d.a1_c = _p(a1), a1.stride(0), (a1.shape[1] if a1_c is None else a1_c)
        d.B, d.H, d.W, d.taps = B, H, W, taps
        d.w, d.w_ld, d.N = _p(w), w.stride(0), N
        d.bias = _p(bias)
        if bias2 is not None:
            d.bias2, d.bias2_ld = _p(bias2), bias2.stride(0)
        if res is not None:
            d.res, d.res_ld = _p(res), res.stride(0)
        d.out, d.out_ld = _p(out), out.stride(0)
        d.mode = mode | (GEMM_STATIC_W if static_w else 0) | (GEMM_RELU if relu else 0) | dmode
        if depth_to_space:
            d.mode |= _cabi.GEMM_D2S2
        if ln is not None:
            st = ln["stats"]
            assert st.dtype == torch.float32 and st.dim() == 3 and st.shape[2] == 2 and st.is_contiguous()
            d.ln_stats, d.ln_parts = _p(st), st.shape[1]
            d.ln_csum, d.ln_bias, d.ln_eps = _p(ln["csum"]), _p(ln["bias"]), ln["eps"]
            self.hold(st, ln["csum"], ln["bias"])
        if stats_out is not None:
            assert stats_out.dtype == torch.float32 and stats_out.dim() == 3 and stats_out.is_contiguous()
            d.stats_out, d.stats_parts = _p(stats_out), stats_out.shape[1]
            self.hold(stats_out)
        self.hold(a0, w, a1, bias, bias2, res, out)

    def gemm_stats_parts(self, a0, w, N, B, H, W, out, **kw):
        """Number of per-row partials a GEMM with these arguments writes through ``stats_out``."""
        probe = Program(self.dev)
        probe.gemm(a0, w, N, B, H, W, out, **kw)
        n = int(_cabi.load().lb_gemm_stats_parts(ctx(self.dev), ctypes.byref(probe.ops[0].u.gemm)))
        if n < 0:
            raise _cabi.LB200Error("lb_gemm_stats_parts failed: " + _cabi.load().lb_last_error().decode())
        return n

    def lpips_im2col_u8(self, frame_u8, H, W, k, stride, pad, shift, scale, out):
        d = self._new(OP_LPIPS_IM2COL_U8).u.patch
        d.x, d.H, d.W, d.C, d.k, d.stride, d.pad = _p(frame_u8), H, W, out.shape[1], k, stride, pad
        d.out, d.ld_out = _p(out), out.stride(0)
        for i in range(3):
            d.f[i], d.f[3 + i] = shift[i], scale[i]
        self.hold(frame_u8, out)

    def im2col(self, x, H, W, C, k, stride, pad, out):
        d = self._new(OP_IM2COL).u.patch
        d.x, d.ld_x, d.H, d.W, d.C, d.k, d.stride, d.pad = _p(x), x.stride(0), H, W, C, k, stride, pad
        d.out, d.ld_out = _p(out), out.stride(0)
        self.hold(x, out)

    def maxpool3s2(self, x, H, W, C, out):
        d = self._new(OP_MAXPOOL3S2).u.patch
        d.x, d.ld_x, d.H, d.W, d.C, d.out, d.ld_out = _p(x), x.stride(0), H, W, C, _p(out), out.stride(0)
        self.hold(x, out)

    def attention(self, q, k, v, out, B, heads, Sq, Skv, q_col0=0, k_col0=0, v_col0=0, scale=0.125):
        d = self._new(OP_ATTENTION).u.attn
        d.q, d.q_ld, d.q_col0 = _p(q), q.stride(0), q_col0
        d.k, d.k_ld, d.k_col0 = _p(k), k.stride(0), k_col0
        d.v, d.v_ld, d.v_col0 = _p(v), v.stride(0), v_col0
        d.out, d.out_ld = _p(out), out.stride(0)
        d.B, d.heads, d.Sq, d.Skv, d.head_dim, d.scale = B, heads, Sq, Skv, 64, scale
        self.hold(q, k, v, out)

    # The VAE-decoder builders below take ``dtype`` (LB_DTYPE_F16 = 0 / LB_DTYPE_BF16 = 1): the lb_op.dtype of the
    # record, i.e. the element type of their 16-bit tensors (see include/lb200.h for each op's meaning).
    def _new_dt(self, kind, dtype):
        op = self._new(kind)
        op.dtype = dtype
        return op

    def groupnorm(self, x, B, HW, C, groups, gamma, beta, eps, silu, out, ws, dtype=0):
        d = self._new_dt(OP_GROUPNORM, dtype).u.norm
        d.x, d.ld_x, d.rows, d.B, d.C, d.groups, d.silu, d.eps = _p(x), x.stride(0), HW, B, C, groups, int(silu), eps
        d.gamma, d.beta, d.out, d.ld_out, d.workspace = _p(gamma), _p(beta), _p(out), out.stride(0), _p(ws)
        self.hold(x, gamma, beta, out, ws)

    def layernorm(self, x, gamma, beta, eps, out):
        d = self._new(OP_LAYERNORM).u.norm
        d.x, d.ld_x, d.rows, d.B, d.C, d.eps = _p(x), x.stride(0), x.shape[0], 1, x.shape[1], eps
        d.gamma, d.beta, d.out, d.ld_out = _p(gamma), _p(beta), _p(out), out.stride(0)
        self.hold(x, gamma, beta, out)

    def embed_inputs(self, text_embeds, time_ids, dim_t, dim_a, temb_in, add_in):
        d = self._new(OP_EMBED_INPUTS).u.embed
        d.text_embeds, d.time_ids = _p(text_embeds), _p(time_ids)
        d.B, d.dim_t, d.pooled, d.dim_a = text_embeds.shape[0], dim_t, text_embeds.shape[1], dim_a
        d.temb_in, d.add_in = _p(temb_in), _p(add_in)
        self.hold(text_embeds, time_ids, temb_in, add_in)

    def linear_small(self, x, w, out, bias=None, addend=None, act_in=0, act_out=0):
        d = self._new(OP_LINEAR_SMALL).u.lin
        d.x, d.ldx, d.M, d.K = _p(x), x.stride(0), x.shape[0], x.shape[1]
        d.w, d.ldw, d.bias = _p(w), w.stride(0), _p(bias)
        if addend is not None:
            d.addend, d.ldadd = _p(addend), addend.stride(0)
        d.act_in, d.act_out, d.out, d.ldo, d.N = act_in, act_out, _p(out), out.stride(0), w.shape[0]
        self.hold(x, w, out, bias, addend)

    def conv_in(self, x_nchw, w, bias, Cout, out, dtype=0):
        d = self._new_dt(OP_CONV_IN, dtype).u.conv
        B, Cin, H, W = x_nchw.shape
        d.x, d.B, d.Cin, d.H, d.W, d.w, d.bias, d.Cout = _p(x_nchw), B, Cin, H, W, _p(w), _p(bias), Cout
        d.out, d.ld_out = _p(out), out.stride(0)
        self.hold(x_nchw, w, bias, out)

    def conv_in_act(self, x_nchw, w, bias, Cout, out, act, in_scale=1.0, dtype=0):
        """lb_conv_in_act: ``act`` 1 is the tiny VAE decoder's input stage (tanh clamp, conv, ReLU)."""
        d = self._new_dt(_cabi.OP_CONV_IN_ACT, dtype).u.conv_act
        B, Cin, H, W = x_nchw.shape
        d.x, d.B, d.Cin, d.H, d.W, d.w, d.bias, d.Cout = _p(x_nchw), B, Cin, H, W, _p(w), _p(bias), Cout
        d.out, d.ld_out, d.act, d.in_scale = _p(out), out.stride(0), act, in_scale
        self.hold(x_nchw, w, bias, out)

    def conv_out(self, x, B, H, W, Cin, w, bias, Cout, out_nchw):
        d = self._new(OP_CONV_OUT).u.conv
        d.x, d.ld_x, d.B, d.Cin, d.H, d.W = _p(x), x.stride(0), B, Cin, H, W
        d.w, d.bias, d.Cout, d.out = _p(w), _p(bias), Cout, _p(out_nchw)
        self.hold(x, w, bias, out_nchw)

    def conv_out_gemm(self, x, B, H, W, Cin, w8, bias8, Cout, out_nchw, tmp, dtype=0):
        """The C0 -> Cout (<= 8) 3x3 output convolution on the tensor-core GEMM: N = 8 (zero-padded weight rows),
        then the Cout live columns go back to NCHW.  ``tmp``: [B*H*W, 8] scratch of the decoder's type."""
        self.gemm(x, w8, 8, B, H, W, tmp, taps=9, a0_c=Cin, bias=bias8)
        d = self._new_dt(OP_NHWC_TO_NCHW, dtype).u.aux
        d.x, d.ld_x, d.out, d.n, d.B, d.C = _p(tmp), tmp.stride(0), _p(out_nchw), H * W, B, Cout
        self.hold(tmp, out_nchw)

    def upsample2x(self, x, B, H, W, C, out, Ho=0, Wo=0, dtype=0):
        """Nearest upsample to Ho x Wo (Ho in {2H-1, 2H}, Wo in {2W-1, 2W}; 0 = exactly 2x)."""
        d = self._new_dt(OP_UPSAMPLE2X, dtype).u.resample
        d.x, d.ld_x, d.B, d.H, d.W, d.C, d.out, d.ld_out = _p(x), x.stride(0), B, H, W, C, _p(out), out.stride(0)
        d.Ho, d.Wo = Ho, Wo
        self.hold(x, out)

    def im2col_s2(self, x, B, H, W, C, out):
        d = self._new(OP_IM2COL_S2).u.resample
        d.x, d.ld_x, d.B, d.H, d.W, d.C, d.out, d.ld_out = _p(x), x.stride(0), B, H, W, C, _p(out), out.stride(0)
        self.hold(x, out)

    def latent_prep(self, x_nchw, w_f32, bias_f32, out_nchw, dtype=0):
        d = self._new_dt(OP_LATENT_PREP, dtype).u.aux
        B, C, H, W = x_nchw.shape
        d.x, d.w, d.bias, d.out, d.n, d.B, d.C = _p(x_nchw), _p(w_f32), _p(bias_f32), _p(out_nchw), H * W, B, C
        self.hold(x_nchw, w_f32, bias_f32, out_nchw)

    def softmax_rows(self, x, out, dtype=0):
        """fp16 rows in; ``dtype``: the output's type (may write over ``x``, see lb_softmax_rows_dt)."""
        d = self._new_dt(OP_SOFTMAX_ROWS, dtype).u.aux
        d.x, d.ld_x, d.out, d.ld_out, d.n, d.C = _p(x), x.stride(0), _p(out), out.stride(0), x.shape[0], x.shape[1]
        self.hold(x, out)

    def postprocess_u8(self, img_nchw, out_u8, nonfinite=None, dtype=0):
        d = self._new_dt(OP_POSTPROCESS_U8, dtype).u.aux
        B, C, H, W = img_nchw.shape
        d.x, d.out, d.n, d.B, d.C, d.w = _p(img_nchw), _p(out_u8), H * W, B, C, _p(nonfinite)
        self.hold(img_nchw, out_u8, nonfinite)

    # -- lifecycle --------------------------------------------------------------------------
    def finalize(self):
        arr = (Op * len(self.ops))(*self.ops)
        h = ctypes.c_void_p()
        check(_cabi.load().lb_program_create(ctx(self.dev), arr, len(self.ops), ctypes.byref(h)), "lb_program_create")
        self.handle = h
        self.num_launches = int(_cabi.load().lb_program_num_launches(h))
        return self

    def run(self, t=0.0):
        check(_cabi.load().lb_program_run(self.handle, float(t), stream_ptr()), "lb_program_run")
        from . import ops
        ops.LAUNCHES[0] += self.num_launches

    def run_kinds(self, kinds, t=0.0):
        """Profiling aid: replay only ops of the given kinds (e.g. [OP_GEMM])."""
        mask = 0
        for k in kinds:
            mask |= 1 << k
        check(_cabi.load().lb_program_run_kinds(self.handle, float(t), mask, stream_ptr()), "lb_program_run_kinds")
        return int(_cabi.load().lb_program_count_kinds(self.handle, mask))

    def work(self):
        """Algorithmic work of the recorded ops: {'gemm_flops', 'gemm_bytes', 'attn_flops', 'norm_bytes'}.
        gemm_bytes = fp16 bytes every GEMM must move at least once: A (M x C per input tensor -- a 3x3 conv reads its
        activation once), W (N x K), the output and the residual."""
        gemm = attn = norm = gbytes = 0
        for op in self.ops:
            if op.kind == OP_GEMM:
                d = op.u.gemm
                M, K = d.B * d.H * d.W, d.taps * d.a0_c + (d.a1_c if d.a1 else 0)
                gemm += 2 * M * d.N * K
                n_out = d.N // 2 if (d.mode & 0xff) == 1 else d.N
                gbytes += 2 * (M * (d.a0_c + (d.a1_c if d.a1 else 0)) + d.N * K + M * n_out + (M * d.N if d.res else 0))
            elif op.kind == OP_ATTENTION:
                d = op.u.attn
                attn += 4 * d.B * d.heads * d.Sq * d.Skv * d.head_dim
            elif op.kind in (OP_GROUPNORM, OP_LAYERNORM):
                d = op.u.norm
                rows = d.rows * (d.B if op.kind == OP_GROUPNORM else 1)
                norm += 4 * rows * d.C
        return dict(gemm_flops=gemm, gemm_bytes=gbytes, attn_flops=attn, norm_bytes=norm)

    def __del__(self):
        try:
            if self.handle is not None:
                _cabi.load().lb_program_destroy(self.handle)
        except Exception:
            pass


def pack_conv_out8(w_co_ky_kx_ci, bias):
    """[Cout<=8][3][3][Cin] conv_out weights -> ([8, 9*Cin] zero-padded rows, [8] bias) for the N = 8 GEMM; None when
    Cin is not a multiple of 64 (the GEMM's K blocks) -- the direct lb_conv_out kernel is used then."""
    co, cin = w_co_ky_kx_ci.shape[0], w_co_ky_kx_ci.shape[-1]
    if cin % 64 != 0 or co > 8:
        return None, None
    w8 = torch.zeros(8, 9 * cin, dtype=w_co_ky_kx_ci.dtype, device=w_co_ky_kx_ci.device)     # fp16, or bf16
    w8[:co] = w_co_ky_kx_ci.reshape(co, 9 * cin)
    b8 = torch.zeros(8, dtype=bias.dtype, device=bias.device)
    b8[:co] = bias
    return w8.contiguous(), b8.contiguous()


def _fold_layernorm(w, bias, gamma, beta):
    """(w*gamma in fp16, rowsum of THAT in fp32, w beta + bias in fp32) for the LayerNorm-folded GEMM."""
    wf = (w.float() * gamma.float()[None, :]).half().contiguous()
    csum = wf.float().sum(dim=1).contiguous()
    lnb = w.float() @ beta.float()
    if bias is not None:
        lnb = lnb + bias.float()
    return wf, csum, lnb.contiguous()


def _geglu_perm(inner, device, half=64):
    """Row order of the GEGLU projection for the kernel's N tiles: ``half`` value rows then their ``half`` gate rows."""
    idx = torch.arange(inner, device=device).view(-1, half)
    return torch.stack([idx, idx + inner], dim=1).reshape(-1)


class PackedUNet:
    """fp16 device copies of the UNet parameters in the layouts the kernels consume."""

    def __init__(self, cfg: UNetConfig, state_dict, device, fold_ln=True):
        self.cfg = cfg
        self.device = torch.device(device)
        self.fold_ln = fold_ln
        sd = state_dict
        dev = self.device

        def g(name):
            return sd[name].detach().to(device=dev, dtype=torch.float16).contiguous()

        def conv3(name):      # [Cout,Cin,3,3] -> [Cout][ky][kx][Cin]
            w = g(name + ".weight")
            return w.permute(0, 2, 3, 1).reshape(w.shape[0], -1).contiguous()

        self.g = g
        self.w = {}
        W = self.w
        W["conv_in.w"] = g("conv_in.weight").permute(2, 3, 1, 0).contiguous()      # [ky][kx][cin][Cout]
        W["conv_in.b"] = g("conv_in.bias")
        W["conv_out.w"] = g("conv_out.weight").permute(0, 2, 3, 1).contiguous()     # [co][ky][kx][Cin]
        W["conv_out.b"] = g("conv_out.bias")
        W["conv_out.w8"], W["conv_out.b8"] = pack_conv_out8(W["conv_out.w"], W["conv_out.b"])
        for nm in ("conv_norm_out",):
            W[nm + ".g"], W[nm + ".b"] = g(nm + ".weight"), g(nm + ".bias")
        for e in ("time_embedding", "add_embedding"):
            for l in ("linear_1", "linear_2"):
                W[f"{e}.{l}.w"], W[f"{e}.{l}.b"] = g(f"{e}.{l}.weight"), g(f"{e}.{l}.bias")
        # resnets (names collected in forward order so the stacked time_emb_proj offsets line up)
        self.resnet_names = [k[: -len(".norm1.weight")] for k in sd if k.endswith(".norm1.weight") and "resnets" in k]
        temb_w, temb_b, off = [], [], 0
        self.temb_off = {}
        for r in self.resnet_names:
            W[r + ".norm1.g"], W[r + ".norm1.b"] = g(r + ".norm1.weight"), g(r + ".norm1.bias")
            W[r + ".norm2.g"], W[r + ".norm2.b"] = g(r + ".norm2.weight"), g(r + ".norm2.bias")
            W[r + ".conv1.w"], W[r + ".conv1.b"] = conv3(r + ".conv1"), g(r + ".conv1.bias")
            w2, b2 = conv3(r + ".conv2"), g(r + ".conv2.bias")
            if (r + ".conv_shortcut.weight") in sd:
                ws = g(r + ".conv_shortcut.weight")
                w2 = torch.cat([w2, ws.reshape(ws.shape[0], -1)], dim=1).contiguous()
                b2 = (b2.float() + g(r + ".conv_shortcut.bias").float()).half()
                W[r + ".has_shortcut"] = True
            W[r + ".conv2.w"], W[r + ".conv2.b"] = w2, b2
            tw, tb = g(r + ".time_emb_proj.weight"), g(r + ".time_emb_proj.bias")
            self.temb_off[r] = (off, tw.shape[0])
            off += tw.shape[0]
            temb_w.append(tw)
            temb_b.append(tb)
        W["temb_all.w"], W["temb_all.b"] = torch.cat(temb_w, 0).contiguous(), torch.cat(temb_b, 0).contiguous()
        self.temb_total = off
        # transformers
        self.tf_names = [k[: -len(".proj_in.weight")] for k in sd if k.endswith(".proj_in.weight")]
        for a in self.tf_names:
            W[a + ".norm.g"], W[a + ".norm.b"] = g(a + ".norm.weight"), g(a + ".norm.bias")
            W[a + ".proj_in.w"], W[a + ".proj_in.b"] = g(a + ".proj_in.weight"), g(a + ".proj_in.bias")
            W[a + ".proj_out.w"], W[a + ".proj_out.b"] = g(a + ".proj_out.weight"), g(a + ".proj_out.bias")
            depth = 0
            while f"{a}.transformer_blocks.{depth}.norm1.weight" in sd:
                t = f"{a}.transformer_blocks.{depth}"
                for n in ("norm1", "norm2", "norm3"):
                    W[f"{t}.{n}.g"], W[f"{t}.{n}.b"] = g(f"{t}.{n}.weight"), g(f"{t}.{n}.bias")
                wqkv = torch.cat([g(t + ".attn1.to_q.weight"), g(t + ".attn1.to_k.weight"),
                                  g(t + ".attn1.to_v.weight")], 0).contiguous()
                W[t + ".attn1.out.w"], W[t + ".attn1.out.b"] = g(t + ".attn1.to_out.0.weight"), g(t + ".attn1.to_out.0.bias")
                wq = g(t + ".attn2.to_q.weight")
                W[t + ".attn2.kv.w"] = torch.cat([g(t + ".attn2.to_k.weight"), g(t + ".attn2.to_v.weight")], 0).contiguous()
                W[t + ".attn2.out.w"], W[t + ".attn2.out.b"] = g(t + ".attn2.to_out.0.weight"), g(t + ".attn2.to_out.0.bias")
                pw, pb = g(t + ".ff.net.0.proj.weight"), g(t + ".ff.net.0.proj.bias")
                perm = _geglu_perm(pw.shape[0] // 2, dev)     # per 128-column N tile of the GEGLU GEMM
                if fold_ln:
                    # LayerNorm folded into the consuming GEMM (include/lb200.h): w' = w*gamma, csum = rowsum(w'),
                    # lnb = w beta + bias
                    for key, w_, b_, nrm, pm in ((".attn1.qkv", wqkv, None, "norm1", None), (".attn2.q", wq, None, "norm2", None),
                                                 (".ff.in", pw, pb, "norm3", perm)):
                        wf, cs, lb = _fold_layernorm(w_, b_, W[f"{t}.{nrm}.g"], W[f"{t}.{nrm}.b"])
                        if pm is not None:
                            wf, cs, lb = wf[pm].contiguous(), cs[pm].contiguous(), lb[pm].contiguous()
                        W[t + key + ".w"], W[t + key + ".csum"], W[t + key + ".lnb"] = wf, cs, lb
                else:
                    W[t + ".attn1.qkv.w"], W[t + ".attn2.q.w"] = wqkv, wq
                    W[t + ".ff.in.w"], W[t + ".ff.in.b"] = pw[perm].contiguous(), pb[perm].contiguous()
                W[t + ".ff.out.w"], W[t + ".ff.out.b"] = g(t + ".ff.net.2.weight"), g(t + ".ff.net.2.bias")
                depth += 1
            W[a + ".depth"] = depth
        for k in sd:
            if k.endswith("samplers.0.conv.weight"):
                nm = k[: -len(".weight")]
                W[nm + ".w"], W[nm + ".b"] = conv3(nm), g(nm + ".bias")

    def nbytes(self):
        return sum(t.numel() * t.element_size() for t in self.w.values() if torch.is_tensor(t))


class UNetB200:
    """One lowered forward per (batch, h, w); ``forward`` replays it."""

    def __init__(self, cfg: UNetConfig, state_dict, device="cuda:0", fold_ln=None):
        import os
        self.cfg = cfg
        self.device = torch.device(device)
        self.dev_index = self.device.index or 0
        # LayerNorm folding is OFF by default: the 210 LayerNorm launches need no shared memory, so under PDL they
        # co-reside with the neighbouring GEMMs' CTAs; folding them away makes GEMM follow GEMM and adds epilogue work.
        # LB_LN_FOLD=1 or fold_ln=True enables the folded path (same numerics and tolerance).
        if fold_ln is None:
            fold_ln = os.environ.get("LB_LN_FOLD") is not None
        self.fold_ln = fold_ln
        self.packed = PackedUNet(cfg, state_dict, self.device, fold_ln=fold_ln)
        self._plans = {}

    # -- public -----------------------------------------------------------------------------
    def plan(self, B, H, W, tag=None, x_in=None):
        """The lowered program for (batch, height, width).  ``tag`` keeps several independent instances (own
        activation buffers) of the same shape apart; ``x_in`` lets the caller supply the input buffer."""
        key = (B, H, W) if tag is None else (B, H, W, tag)
        if key not in self._plans:
            self._plans[key] = _Lowering(self, B, H, W, x_in=x_in)
        return self._plans[key]

    @torch.no_grad()
    def forward(self, x, t, encoder_hidden_states, text_embeds, time_ids, ctx_changed=True):
        """x [B,4,h,w] fp16 NCHW -> eps [B,4,h,w] fp16 (a view of the plan's static output buffer)."""
        B, _, H, W = x.shape
        pl = self.plan(B, H, W)
        pl.x_in.copy_(x)
        pl.text.copy_(text_embeds)
        pl.tids.copy_(time_ids)
        if ctx_changed:
            pl.ctx.copy_(encoder_hidden_states.reshape(pl.ctx.shape))
            pl.prog_ctx.run()
        pl.prog_step.run(float(t))
        return pl.eps

    def launches_per_forward(self, B, H, W):
        pl = self.plan(B, H, W)
        return pl.prog_step.num_launches, pl.prog_ctx.num_launches


class _Lowering:
    def __init__(self, net: UNetB200, B, H, W, x_in=None):
        cfg, Wt = net.cfg, net.packed.w
        self.net, self.B, self.H, self.W = net, B, H, W
        dev = net.device
        f16 = dict(dtype=torch.float16, device=dev)
        ch = list(cfg.block_out_channels)
        L = len(ch)
        T = cfg.time_embed_dim
        groups = cfg.norm_num_groups
        if x_in is not None:
            assert tuple(x_in.shape) == (B, cfg.in_channels, H, W) and x_in.dtype == torch.float16 and x_in.is_contiguous()
        self.x_in = x_in if x_in is not None else torch.zeros(B, cfg.in_channels, H, W, **f16)
        self.eps = torch.zeros(B, cfg.out_channels, H, W, **f16)
        self.ctx = torch.zeros(B * 77, cfg.cross_attention_dim, **f16)
        self.text = torch.zeros(B, cfg.pooled_dim, **f16)
        self.tids = torch.zeros(B, 6, **f16)
        self.ws = torch.zeros(max(1 << 16, _cabi.load().lb_groupnorm_workspace_bytes(ctx(net.dev_index), B, H * W, groups)),
                              dtype=torch.uint8, device=dev)
        P = self.prog_step = Program(net.dev_index)
        PC = self.prog_ctx = Program(net.dev_index)
        self._scratch = {}

        def scratch(name, rows, cols):
            key = name
            need = rows * cols
            buf = self._scratch.get(key)
            if buf is None or buf.numel() < need:
                buf = torch.empty(need, **f16)
                self._scratch[key] = buf
            return buf[:need].view(rows, cols)

        self._persist = []

        def persist(rows, cols):
            t = torch.empty(rows, cols, **f16)
            self._persist.append(t)
            return t

        # ---- embeddings -------------------------------------------------------------------
        temb_in, add_in = persist(B, ch[0]), persist(B, cfg.add_in_dim)
        P.embed_inputs(self.text, self.tids, ch[0], cfg.addition_time_embed_dim, temb_in, add_in)
        t1, a1, temb, emb = persist(B, T), persist(B, T), persist(B, T), persist(B, T)
        P.linear_small(temb_in, Wt["time_embedding.linear_1.w"], t1, bias=Wt["time_embedding.linear_1.b"], act_out=1)
        P.linear_small(t1, Wt["time_embedding.linear_2.w"], temb, bias=Wt["time_embedding.linear_2.b"])
        P.linear_small(add_in, Wt["add_embedding.linear_1.w"], a1, bias=Wt["add_embedding.linear_1.b"], act_out=1)
        P.linear_small(a1, Wt["add_embedding.linear_2.w"], emb, bias=Wt["add_embedding.linear_2.b"], addend=temb)
        temb_all = persist(B, net.packed.temb_total)
        P.linear_small(emb, Wt["temb_all.w"], temb_all, bias=Wt["temb_all.b"], act_in=1)

        # ---- geometry + concat buffers ------------------------------------------------------
        # the stride-2 pad-1 Downsample2D conv gives ceil(s/2); the up path resizes back to each skip level's size
        res_hw = [(H, W)]
        for _ in range(L - 1):
            res_hw.append(((res_hw[-1][0] + 1) // 2, (res_hw[-1][1] + 1) // 2))

        def rows_at(level):
            return B * res_hw[level][0] * res_hw[level][1]

        # skip list: (level, channels) in production order
        skip_meta = [(0, ch[0])]
        for i in range(L):
            skip_meta += [(i, ch[i])] * cfg.layers_per_block
            if i < L - 1:
                skip_meta.append((i + 1, ch[i]))
        # up path consumption: resnet j of up block i
        rev = list(reversed(ch))
        cats = []              # in pop order
        cprev = rev[0]
        k = len(skip_meta) - 1
        for i in range(L):
            cout = rev[i]
            for j in range(cfg.layers_per_block + 1):
                hidden_c = cprev if j == 0 else cout
                lvl, sc = skip_meta[k]
                buf = persist(rows_at(lvl), hidden_c + sc)
                cats.append(dict(buf=buf, hidden=buf[:, :hidden_c], skip=buf[:, hidden_c:], level=lvl))
                k -= 1
            cprev = cout
        skip_views = [c["skip"] for c in reversed(cats)]      # index by production order

        def tslice(rname):
            off, n = net.packed.temb_off[rname]
            return temb_all[:, off:off + n]

        def resnet(rname, x, cin, cout, level, out):
            h_, w_ = res_hw[level]
            M = rows_at(level)
            n1 = scratch("n1", M, cin)
            P.groupnorm(x, B, h_ * w_, cin, groups, Wt[rname + ".norm1.g"], Wt[rname + ".norm1.b"], 1e-5, 1, n1, self.ws)
            h1 = scratch("h1", M, cout)
            P.gemm(n1, Wt[rname + ".conv1.w"], cout, B, h_, w_, h1, taps=9, bias=Wt[rname + ".conv1.b"], bias2=tslice(rname))
            n2 = scratch("n2", M, cout)
            P.groupnorm(h1, B, h_ * w_, cout, groups, Wt[rname + ".norm2.g"], Wt[rname + ".norm2.b"], 1e-5, 1, n2, self.ws)
            if Wt.get(rname + ".has_shortcut"):
                P.gemm(n2, Wt[rname + ".conv2.w"], cout, B, h_, w_, out, taps=9, a1=x, a1_c=cin, bias=Wt[rname + ".conv2.b"])
            else:
                P.gemm(n2, Wt[rname + ".conv2.w"], cout, B, h_, w_, out, taps=9, bias=Wt[rname + ".conv2.b"], res=x)

        kv_cache = {}

        fold = net.fold_ln
        geglu_mode = 1
        f32 = dict(dtype=torch.float32, device=dev)

        def transformer(aname, x, C, level, out):
            h_, w_ = res_hw[level]
            S = h_ * w_
            M = rows_at(level)
            heads = C // cfg.head_dim
            tn = scratch("tn", M, C)
            P.groupnorm(x, B, S, C, groups, Wt[aname + ".norm.g"], Wt[aname + ".norm.b"], 1e-6, 0, tn, self.ws)
            hs = scratch("hs", M, C)
            if not fold:
                P.gemm(tn, Wt[aname + ".proj_in.w"], C, 1, 1, M, hs, bias=Wt[aname + ".proj_in.b"])
                stats = None
            else:
                # every GEMM that writes the residual stream ``hs`` also writes its per-row partial sums; the three
                # LayerNorms of a block are folded into the GEMMs that consume them (no LN launches, no LN buffer)
                parts = P.gemm_stats_parts(tn, Wt[aname + ".proj_in.w"], C, 1, 1, M, hs)
                key = ("ln_stats", M, parts)
                if key not in self._scratch:
                    self._scratch[key] = torch.zeros(M, parts, 2, **f32)
                stats = self._scratch[key]
                P.gemm(tn, Wt[aname + ".proj_in.w"], C, 1, 1, M, hs, bias=Wt[aname + ".proj_in.b"], stats_out=stats)

            def ln_of(t, key):
                return dict(stats=stats, csum=Wt[t + key + ".csum"], bias=Wt[t + key + ".lnb"], eps=1e-5)

            for d in range(Wt[aname + ".depth"]):
                t = f"{aname}.transformer_blocks.{d}"
                qkv = scratch("qkv", M, 3 * C)
                att = scratch("att", M, C)
                q = scratch("q", M, C)
                gg = scratch("geglu", M, 4 * C)
                kv = persist(B * 77, 2 * C)         # depends on the conditioning only: computed by prog_ctx
                PC.gemm(self.ctx, Wt[t + ".attn2.kv.w"], 2 * C, 1, 1, B * 77, kv)
                kv_cache[t] = kv
                if fold:
                    P.gemm(hs, Wt[t + ".attn1.qkv.w"], 3 * C, 1, 1, M, qkv, ln=ln_of(t, ".attn1.qkv"))
                    P.attention(qkv, qkv, qkv, att, B, heads, S, S, 0, C, 2 * C, cfg.head_dim ** -0.5)
                    P.gemm(att, Wt[t + ".attn1.out.w"], C, 1, 1, M, hs, bias=Wt[t + ".attn1.out.b"], res=hs, stats_out=stats)
                    P.gemm(hs, Wt[t + ".attn2.q.w"], C, 1, 1, M, q, ln=ln_of(t, ".attn2.q"))
                    P.attention(q, kv, kv, att, B, heads, S, 77, 0, 0, C, cfg.head_dim ** -0.5)
                    P.gemm(att, Wt[t + ".attn2.out.w"], C, 1, 1, M, hs, bias=Wt[t + ".attn2.out.b"], res=hs, stats_out=stats)
                    P.gemm(hs, Wt[t + ".ff.in.w"], 8 * C, 1, 1, M, gg, mode=geglu_mode, ln=ln_of(t, ".ff.in"))
                    P.gemm(gg, Wt[t + ".ff.out.w"], C, 1, 1, M, hs, bias=Wt[t + ".ff.out.b"], res=hs, stats_out=stats)
                    continue
                ln = scratch("ln", M, C)
                P.layernorm(hs, Wt[t + ".norm1.g"], Wt[t + ".norm1.b"], 1e-5, ln)
                P.gemm(ln, Wt[t + ".attn1.qkv.w"], 3 * C, 1, 1, M, qkv)
                P.attention(qkv, qkv, qkv, att, B, heads, S, S, 0, C, 2 * C, cfg.head_dim ** -0.5)
                P.gemm(att, Wt[t + ".attn1.out.w"], C, 1, 1, M, hs, bias=Wt[t + ".attn1.out.b"], res=hs)
                P.layernorm(hs, Wt[t + ".norm2.g"], Wt[t + ".norm2.b"], 1e-5, ln)
                P.gemm(ln, Wt[t + ".attn2.q.w"], C, 1, 1, M, q)
                P.attention(q, kv, kv, att, B, heads, S, 77, 0, 0, C, cfg.head_dim ** -0.5)
                P.gemm(att, Wt[t + ".attn2.out.w"], C, 1, 1, M, hs, bias=Wt[t + ".attn2.out.b"], res=hs)
                P.layernorm(hs, Wt[t + ".norm3.g"], Wt[t + ".norm3.b"], 1e-5, ln)
                P.gemm(ln, Wt[t + ".ff.in.w"], 8 * C, 1, 1, M, gg, bias=Wt[t + ".ff.in.b"], mode=geglu_mode)
                P.gemm(gg, Wt[t + ".ff.out.w"], C, 1, 1, M, hs, bias=Wt[t + ".ff.out.b"], res=hs)
            P.gemm(hs, Wt[aname + ".proj_out.w"], C, 1, 1, M, out, bias=Wt[aname + ".proj_out.b"], res=x)

        # ---- down path ----------------------------------------------------------------------
        si = 0
        P.conv_in(self.x_in, Wt["conv_in.w"], Wt["conv_in.b"], ch[0], skip_views[si])
        x, cin = skip_views[si], ch[0]
        si += 1
        for i in range(L):
            cout = ch[i]
            for j in range(cfg.layers_per_block):
                rname = f"down_blocks.{i}.resnets.{j}"
                dst = skip_views[si]
                if cfg.transformer_layers[i]:
                    r_out = persist(rows_at(i), cout)
                    resnet(rname, x, cin, cout, i, r_out)
                    transformer(f"down_blocks.{i}.attentions.{j}", r_out, cout, i, dst)
                else:
                    resnet(rname, x, cin, cout, i, dst)
                x, cin = dst, cout
                si += 1
            if i < L - 1:
                nm = f"down_blocks.{i}.downsamplers.0.conv"
                h_, w_ = res_hw[i]
                cols = scratch("im2col", rows_at(i + 1), 9 * cout)
                P.im2col_s2(x, B, h_, w_, cout, cols)
                dst = skip_views[si]
                P.gemm(cols, Wt[nm + ".w"], cout, 1, 1, rows_at(i + 1), dst, bias=Wt[nm + ".b"])
                x = dst
                si += 1
        # ---- mid ----------------------------------------------------------------------------
        lv, cm = L - 1, ch[-1]
        m1 = persist(rows_at(lv), cm)
        resnet("mid_block.resnets.0", x, cm, cm, lv, m1)
        m2 = persist(rows_at(lv), cm)
        transformer("mid_block.attentions.0", m1, cm, lv, m2)
        resnet("mid_block.resnets.1", m2, cm, cm, lv, cats[0]["hidden"])
        # ---- up path ------------------------------------------------------------------------
        ci = 0
        rev_depth = list(reversed(cfg.transformer_layers))
        for i in range(L):
            cout = rev[i]
            lvl = L - 1 - i
            n_res = cfg.layers_per_block + 1
            for j in range(n_res):
                cat = cats[ci]
                cin_total = cat["buf"].shape[1]
                last_of_block = j == n_res - 1
                last_overall = last_of_block and i == L - 1
                if last_overall:
                    dst = persist(rows_at(lvl), cout)
                elif last_of_block:
                    dst = persist(rows_at(lvl), cout)          # goes through the upsampler
                else:
                    dst = cats[ci + 1]["hidden"]
                rname = f"up_blocks.{i}.resnets.{j}"
                if rev_depth[i]:
                    r_out = persist(rows_at(lvl), cout)
                    resnet(rname, cat["buf"], cin_total, cout, lvl, r_out)
                    transformer(f"up_blocks.{i}.attentions.{j}", r_out, cout, lvl, dst)
                else:
                    resnet(rname, cat["buf"], cin_total, cout, lvl, dst)
                ci += 1
                x = dst
            if i < L - 1:
                nm = f"up_blocks.{i}.upsamplers.0.conv"
                h_, w_ = res_hw[lvl]
                ho, wo = res_hw[lvl - 1]
                up = scratch("up", rows_at(lvl - 1), cout)
                P.upsample2x(x, B, h_, w_, cout, up, ho, wo)
                P.gemm(up, Wt[nm + ".w"], cout, B, ho, wo, cats[ci]["hidden"], taps=9, bias=Wt[nm + ".b"])
        # ---- out ----------------------------------------------------------------------------
        no = scratch("n1", rows_at(0), ch[0])
        P.groupnorm(x, B, H * W, ch[0], groups, Wt["conv_norm_out.g"], Wt["conv_norm_out.b"], 1e-5, 1, no, self.ws)
        if Wt.get("conv_out.w8") is not None and os.environ.get("LB_CONV_OUT_DIRECT") is None:
            P.conv_out_gemm(no, B, H, W, ch[0], Wt["conv_out.w8"], Wt["conv_out.b8"], cfg.out_channels, self.eps,
                            scratch("conv_out8", rows_at(0), 8))
        else:
            P.conv_out(no, B, H, W, ch[0], Wt["conv_out.w"], Wt["conv_out.b"], cfg.out_channels, self.eps)
        P.finalize()
        PC.finalize()
