"""The op records of liblb200's executor (``lb_op``, include/lb200.h): every op a lowering or an eager wrapper in
``ops.py`` runs is recorded here, handed to lb_program_create (which validates every record) and replayed with
lb_program_run.  Element types come from the tensors: an op with fp16 and bf16 variants records the type of the
tensor named in its emitter, and raises LB200Error on mixed types."""
import ctypes

import torch

from . import _cabi
from ._cabi import (GEMM_RELU, GEMM_STATIC_W, OP_ADD_ROWS_BCAST, OP_ATTENTION, OP_AVGPOOL2_CEIL, OP_COND_CONV, OP_CONV_IN, OP_CONV_IN_ADD,
                    OP_EMBED_INPUTS, OP_GEMM, OP_IMAGE_CONV_IN, OP_IM2COL_S2_PAD01,
                    OP_GROUPNORM, OP_IM2COL, OP_IM2COL_S2, OP_LATENT_PREP, OP_LAYERNORM, OP_LINEAR_SMALL,
                    OP_LPIPS_IM2COL_U8, OP_MAXPOOL3S2, OP_NHWC_TO_NCHW, OP_PIXEL_UNSHUFFLE_U8, OP_POSTPROCESS_U8,
                    OP_SOFTMAX_ROWS, OP_UPSAMPLE_NEAREST, Op, check, ctx, stream_ptr)

_DT16 = {torch.float16: _cabi.DTYPE_F16, torch.bfloat16: _cabi.DTYPE_BF16}   # the ops with fp16 and bf16 variants
_TILING = {"auto": 0, "box": _cabi.GEMM_TILE_BOX, "runs": _cabi.GEMM_TILE_RUNS}
LAUNCHES = [0]      # kernels of liblb200 launched through Program.run and ops.py (bench.py reports it)


def _p(t):
    return None if t is None else t.data_ptr()


def dtype16(t, what="tensor"):
    """LB_DTYPE_* of an fp16 / bf16 tensor; anything else raises."""
    if t.dtype not in _DT16:
        raise _cabi.LB200Error(f"{what} must be float16 or bfloat16 (got {t.dtype})")
    return _DT16[t.dtype]


def _same_dtype(dtype, what, *ts):
    for t in ts:
        if t is not None and t.dtype != dtype:
            raise _cabi.LB200Error(f"{what}: mixed element types ({t.dtype} with {dtype})")


def gemm_dtype_mode(a0, w, out_dtype, a1=None, bias=None, bias2=None, res=None):
    """The lb_gemm mode flags of the element types: fp16 operands (0), or bf16 operands (LB_GEMM_BF16) with a bf16 or
    (``out_dtype`` float16: LB_GEMM_OUT_F16) fp16 output.  Mixed operand types raise."""
    if a0.dtype != torch.bfloat16 and w.dtype != torch.bfloat16:
        return 0
    _same_dtype(torch.bfloat16, "gemm operands a0 / w / a1 / bias / bias2 / res", a0, w, a1, bias, bias2, res)
    if out_dtype == torch.bfloat16:
        return _cabi.GEMM_BF16
    if out_dtype == torch.float16:
        return _cabi.GEMM_BF16 | _cabi.GEMM_OUT_F16
    raise _cabi.LB200Error(f"gemm: bf16 operands give a bf16 or fp16 output (asked for {out_dtype})")


class Program:
    """A recorded op list; ``finalize`` hands it to lb_program_create."""

    def __init__(self, device_index):
        self.dev = device_index
        self.ops = []
        self.keep = []          # tensors referenced by raw pointers must outlive the program
        self.handle = None

    def _new(self, kind, dtype=_cabi.DTYPE_F16):
        op = Op()
        op.kind = kind
        op.dtype = dtype
        self.ops.append(op)
        return op

    def hold(self, *ts):
        self.keep.extend(t for t in ts if t is not None)

    # -- op emitters ---------------------------------------------------------------------------
    def gemm(self, a0, w, N, B, H, W, out, taps=1, a0_c=None, a1=None, a1_c=None, bias=None, bias2=None, res=None,
             mode=0, static_w=True, relu=False, tiling="auto", depth_to_space=False):
        """Tensor-core GEMM / implicit-GEMM conv (lb_gemm_desc).  a0: NHWC activation viewed as [B*H*W, >=a0_c]
        (row stride = a0.stride(-2)); w: [N, K] packed weights.
        ``static_w``: ``w`` holds model weights (not written by the preceding op), so the kernel may fetch its
        first tiles before the preceding kernel has finished (LB_GEMM_STATIC_W).  Pass False when an activation
        is used as the B operand.
        ``tiling``: "auto" (the M tiling with fewer tiles), "box" (pixel boxes) or "runs" (pixel runs); all give the
        same results.
        ``depth_to_space``: nearest-2x upsample + 3x3 conv as one GEMM (LB_GEMM_D2S2): ``w`` holds the four phase
        filters [4*Co, 9*C] (``taesd.pack_d2s_weights``), ``out`` the [B*2H*2W, Co] upsampled map.
        Element types come from the tensors: fp16 throughout, or bf16 a0 / w / a1 / bias / bias2 / res
        (LB_GEMM_BF16) writing ``out``'s type (bf16, or fp16: LB_GEMM_OUT_F16)."""
        if tiling not in _TILING:
            raise ValueError(f"tiling must be one of {sorted(_TILING)} (got {tiling!r})")
        dmode = gemm_dtype_mode(a0, w, out.dtype, a1, bias, bias2, res)
        d = self._new(OP_GEMM).u.gemm
        d.a0, d.a0_ld, d.a0_c = _p(a0), a0.stride(-2), (a0.shape[-1] if a0_c is None else a0_c)
        if a1 is not None:
            d.a1, d.a1_ld, d.a1_c = _p(a1), a1.stride(-2), (a1.shape[-1] if a1_c is None else a1_c)
        d.B, d.H, d.W, d.taps = B, H, W, taps
        d.w, d.w_ld, d.N = _p(w), w.stride(0), N
        d.bias = _p(bias)
        if bias2 is not None:
            d.bias2, d.bias2_ld = _p(bias2), bias2.stride(0)
        if res is not None:
            d.res, d.res_ld = _p(res), res.stride(-2)
        d.out, d.out_ld = _p(out), out.stride(-2)
        d.mode = mode | (GEMM_STATIC_W if static_w else 0) | (GEMM_RELU if relu else 0) | _TILING[tiling] | dmode
        if depth_to_space:
            d.mode |= _cabi.GEMM_D2S2
        self.hold(a0, w, a1, bias, bias2, res, out)

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
        """q/k/v: 2-D row-major fp16 buffers whose column slices hold the heads (lb_attention)."""
        d = self._new(OP_ATTENTION).u.attn
        d.q, d.q_ld, d.q_col0 = _p(q), q.stride(0), q_col0
        d.k, d.k_ld, d.k_col0 = _p(k), k.stride(0), k_col0
        d.v, d.v_ld, d.v_col0 = _p(v), v.stride(0), v_col0
        d.out, d.out_ld = _p(out), out.stride(0)
        d.B, d.heads, d.Sq, d.Skv, d.head_dim, d.scale = B, heads, Sq, Skv, 64, scale
        self.hold(q, k, v, out)

    def groupnorm(self, x, B, HW, C, groups, gamma, beta, eps, silu, out, ws):
        """fp16 or bf16 (x, gamma, beta and out of one type); ``ws``: zero-filled lb_groupnorm workspace."""
        dt = dtype16(x, "groupnorm x")
        _same_dtype(x.dtype, "groupnorm x / gamma / beta / out", gamma, beta, out)
        d = self._new(OP_GROUPNORM, dt).u.norm
        d.x, d.ld_x, d.rows, d.B, d.C, d.groups, d.silu, d.eps = _p(x), x.stride(0), HW, B, C, groups, int(silu), eps
        d.gamma, d.beta, d.out, d.ld_out, d.workspace = _p(gamma), _p(beta), _p(out), out.stride(0), _p(ws)
        self.hold(x, gamma, beta, out, ws)

    def layernorm(self, x, gamma, beta, eps, out):
        d = self._new(OP_LAYERNORM).u.norm
        d.x, d.ld_x, d.rows, d.B, d.C, d.eps = _p(x), x.stride(0), x.shape[0], 1, x.shape[1], eps
        d.gamma, d.beta, d.out, d.ld_out = _p(gamma), _p(beta), _p(out), out.stride(0)
        self.hold(x, gamma, beta, out)

    def embed_inputs(self, text_embeds, time_ids, dim_t, dim_a, temb_in, add_in):
        """The timestep is ``run``'s argument."""
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

    def conv_in(self, x_nchw, w, bias, Cout, out, act=_cabi.CONV_IN_PLAIN, in_scale=1.0):
        """fp16 or bf16 (x, weights, bias and out of one type).  ``act`` CONV_IN_TINY_VAE (fp16): the tiny VAE
        decoder's input stage, tanh(x * in_scale / 3) * 3 before the conv and ReLU after it."""
        dt = dtype16(x_nchw, "conv_in x")
        _same_dtype(x_nchw.dtype, "conv_in x / w / bias / out", w, bias, out)
        d = self._new(OP_CONV_IN, dt).u.conv
        B, Cin, H, W = x_nchw.shape
        d.x, d.B, d.Cin, d.H, d.W, d.w, d.bias, d.Cout = _p(x_nchw), B, Cin, H, W, _p(w), _p(bias), Cout
        d.out, d.ld_out, d.act, d.in_scale = _p(out), out.stride(0), int(act), float(in_scale)
        self.hold(x_nchw, w, bias, out)

    def conv_in_add(self, x_nchw, w, bias, Cout, out, addend):
        """fp16 ``conv_in`` then ``+ addend[r mod H*W]`` (lb_conv_in_add): a ControlNet's conv_in(x) plus the
        conditioning embedding [H*W, Cout] every batch row shares."""
        _same_dtype(torch.float16, "conv_in_add x / w / bias / out / addend", x_nchw, w, bias, out, addend)
        d = self._new(OP_CONV_IN_ADD).u.conv
        B, Cin, H, W = x_nchw.shape
        if addend.shape[0] != H * W:
            raise _cabi.LB200Error(f"conv_in_add: the addend has {addend.shape[0]} rows, the map {H}x{W} pixels")
        d.x, d.B, d.Cin, d.H, d.W, d.w, d.bias, d.Cout = _p(x_nchw), B, Cin, H, W, _p(w), _p(bias), Cout
        d.out, d.ld_out, d.addend, d.ld_add = _p(out), out.stride(0), _p(addend), addend.stride(0)
        self.hold(x_nchw, w, bias, out, addend)

    def cond_conv(self, x, B, H, W, Cin, w, bias, Cout, out, stride=1, silu=False):
        """Direct 3x3 pad-1 conv of NHWC ``x`` (fp16 [B*H*W, >=Cin], or a uint8 image read as u / 255) into fp16
        ``out`` [B*Ho*Wo, >=Cout] (lb_cond_conv); ``w`` packed [ky][kx][Cin][Cout]."""
        if x.dtype not in (torch.uint8, torch.float16):
            raise _cabi.LB200Error(f"cond_conv: x must be uint8 or float16 (got {x.dtype})")
        _same_dtype(torch.float16, "cond_conv w / bias / out", w, bias, out)
        d = self._new(OP_COND_CONV).u.conv
        d.x, d.ld_x, d.B, d.Cin, d.H, d.W = _p(x), x.stride(-2), B, Cin, H, W
        d.w, d.bias, d.Cout, d.out, d.ld_out = _p(w), _p(bias), Cout, _p(out), out.stride(0)
        d.act, d.stride, d.in_u8 = int(silu), stride, int(x.dtype == torch.uint8)
        self.hold(x, w, bias, out)

    def image_conv_in(self, img_u8, B, H, W, w, bias, Cout, out):
        """The VAE encoder's conv_in on a uint8 image [B*H*W, >=3] with VaeImageProcessor.preprocess fused
        (lb_image_conv_in): fp16 or bf16 ``w`` [ky][kx][Cin][Cout], ``bias`` and NHWC ``out`` [B*H*W, >=Cout]."""
        if img_u8.dtype != torch.uint8:
            raise _cabi.LB200Error(f"image_conv_in: the image must be uint8 (got {img_u8.dtype})")
        dt = dtype16(out, "image_conv_in out")
        _same_dtype(out.dtype, "image_conv_in w / bias / out", w, bias)
        d = self._new(OP_IMAGE_CONV_IN, dt).u.conv
        d.x, d.ld_x, d.B, d.Cin, d.H, d.W = _p(img_u8), img_u8.stride(-2), B, img_u8.shape[-1], H, W
        d.w, d.bias, d.Cout, d.out, d.ld_out = _p(w), _p(bias), Cout, _p(out), out.stride(0)
        self.hold(img_u8, w, bias, out)

    def conv_out_gemm(self, x, B, H, W, Cin, w8, bias8, Cout, out_nchw, tmp):
        """The C0 -> Cout (<= 8) 3x3 output convolution on the tensor-core GEMM: N = 8 (zero-padded weight rows),
        then the Cout live columns go back to NCHW.  ``tmp``: [B*H*W, 8] scratch of the output's type."""
        self.gemm(x, w8, 8, B, H, W, tmp, taps=9, a0_c=Cin, bias=bias8)
        self.nhwc_to_nchw(tmp, B, Cout, H, W, out_nchw)

    def nhwc_to_nchw(self, x, B, C, H, W, out_nchw):
        """The first C (<= 8) columns of fp16 / bf16 NHWC rows [B*H*W, ld] -> NCHW [B, C, H, W]."""
        dt = dtype16(x, "nhwc_to_nchw x")
        _same_dtype(x.dtype, "nhwc_to_nchw x / out", out_nchw)
        d = self._new(OP_NHWC_TO_NCHW, dt).u.aux
        d.x, d.ld_x, d.out, d.n, d.B, d.C = _p(x), x.stride(0), _p(out_nchw), H * W, B, C
        self.hold(x, out_nchw)

    def upsample_nearest(self, x, B, H, W, C, out, Ho, Wo):
        """F.interpolate(size=(Ho, Wo), mode="nearest") of NHWC rows [B*H*W, >=C] for Ho in {2H-1, 2H}, Wo in
        {2W-1, 2W} (lb_upsample_nearest; other sizes fail when the program runs).  fp16 or bf16."""
        dt = dtype16(x, "upsample x")
        _same_dtype(x.dtype, "upsample x / out", out)
        d = self._new(OP_UPSAMPLE_NEAREST, dt).u.resample
        d.x, d.ld_x, d.B, d.H, d.W, d.C, d.out, d.ld_out = _p(x), x.stride(0), B, H, W, C, _p(out), out.stride(0)
        d.Ho, d.Wo = Ho, Wo
        self.hold(x, out)

    def im2col_s2(self, x, B, H, W, C, out):
        d = self._new(OP_IM2COL_S2).u.resample
        d.x, d.ld_x, d.B, d.H, d.W, d.C, d.out, d.ld_out = _p(x), x.stride(0), B, H, W, C, _p(out), out.stride(0)
        self.hold(x, out)

    def im2col_s2_pad01(self, x, B, H, W, C, out):
        """Patch matrix [B*Ho*Wo, 9*C] of Downsample2D(padding=0): F.pad(x, (0, 1, 0, 1)), then 3x3 stride 2
        (lb_im2col_s2_pad01); Ho = (H - 2) // 2 + 1.  fp16 or bf16."""
        dtype16(x, "im2col_s2_pad01 x")
        _same_dtype(x.dtype, "im2col_s2_pad01 x / out", out)
        d = self._new(OP_IM2COL_S2_PAD01).u.resample
        d.x, d.ld_x, d.B, d.H, d.W, d.C, d.out, d.ld_out = _p(x), x.stride(0), B, H, W, C, _p(out), out.stride(0)
        self.hold(x, out)

    def add_rows_bcast(self, dst, src, B):
        """fp16 ``dst[b*rows + r] += src[r]`` in place for every batch row b (lb_add_rows_bcast): ``dst`` [B*rows, C]
        and ``src`` [rows, C], row-major with any row stride (a skip view inside a concat buffer, say)."""
        _same_dtype(torch.float16, "add_rows_bcast dst / src", dst, src)
        rows, C = src.shape
        if tuple(dst.shape) != (B * rows, C):
            raise _cabi.LB200Error(f"add_rows_bcast: dst {tuple(dst.shape)} is not {B} x src {tuple(src.shape)}")
        d = self._new(OP_ADD_ROWS_BCAST).u.aux
        d.out, d.ld_out, d.x, d.ld_x, d.B, d.n, d.C = _p(dst), dst.stride(0), _p(src), src.stride(0), B, rows, C
        self.hold(dst, src)

    def pixel_unshuffle_u8(self, img_u8, r, out):
        """uint8 image [H, W, Cimg] -> fp16 ``out`` [(H/r)*(W/r), r*r*Cimg], u / 255, columns in (i, j, c) order
        (lb_pixel_unshuffle_u8)."""
        if img_u8.dtype != torch.uint8 or img_u8.dim() != 3 or not img_u8.is_contiguous():
            raise _cabi.LB200Error(f"pixel_unshuffle_u8: the image must be a contiguous uint8 [H, W, C] tensor (got "
                                   f"{img_u8.dtype} {tuple(img_u8.shape)})")
        _same_dtype(torch.float16, "pixel_unshuffle_u8 out", out)
        H, W, C = img_u8.shape
        if tuple(out.shape) != ((H // r) * (W // r), r * r * C) or not out.is_contiguous():
            raise _cabi.LB200Error(f"pixel_unshuffle_u8: out must be contiguous [{(H // r) * (W // r)}, {r * r * C}]")
        d = self._new(OP_PIXEL_UNSHUFFLE_U8).u.patch
        d.x, d.H, d.W, d.C, d.k, d.out, d.ld_out = _p(img_u8), H, W, C, r, _p(out), out.stride(0)
        self.hold(img_u8, out)

    def avgpool2_ceil(self, x, H, W, C, out):
        """AvgPool2d(2, 2, ceil_mode=True) of the fp16 NHWC map ``x`` [H*W, >=C] into ``out`` [ceil(H/2)*ceil(W/2),
        >=C] (lb_avgpool2_ceil)."""
        _same_dtype(torch.float16, "avgpool2_ceil x / out", x, out)
        d = self._new(OP_AVGPOOL2_CEIL).u.patch
        d.x, d.ld_x, d.H, d.W, d.C, d.out, d.ld_out = _p(x), x.stride(0), H, W, C, _p(out), out.stride(0)
        self.hold(x, out)

    def latent_prep(self, x_nchw, w_f32, bias_f32, out_nchw):
        """post_quant_conv(latents / scaling_factor): fp16 NCHW latents in, fp16 or bf16 ``out_nchw``."""
        dt = dtype16(out_nchw, "latent_prep out")
        d = self._new(OP_LATENT_PREP, dt).u.aux
        B, C, H, W = x_nchw.shape
        d.x, d.w, d.bias, d.out, d.n, d.B, d.C = _p(x_nchw), _p(w_f32), _p(bias_f32), _p(out_nchw), H * W, B, C
        self.hold(x_nchw, w_f32, bias_f32, out_nchw)

    def softmax_rows(self, x, out):
        """Row softmax of fp16 ``x`` [rows, cols] into fp16 or bf16 ``out`` (may be ``x``'s own storage, see
        lb_softmax_rows)."""
        dt = dtype16(out, "softmax out")
        d = self._new(OP_SOFTMAX_ROWS, dt).u.aux
        d.x, d.ld_x, d.out, d.ld_out, d.n, d.C = _p(x), x.stride(0), _p(out), out.stride(0), x.shape[0], x.shape[1]
        self.hold(x, out)

    def postprocess_u8(self, img_nchw, out_u8, nonfinite=None):
        """fp16 / bf16 NCHW image -> uint8 NHWC; ``nonfinite`` (device int32[1]) accumulates the non-finite pixel
        count."""
        dt = dtype16(img_nchw, "postprocess image")
        d = self._new(OP_POSTPROCESS_U8, dt).u.aux
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
        LAUNCHES[0] += self.num_launches

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
    """[Cout<=8][3][3][Cin] conv_out weights -> ([8, 9*Cin] zero-padded rows, [8] bias) for the N = 8 GEMM.  Raises
    LB200Error when Cin is not a multiple of 64 (the GEMM's K blocks) or Cout > 8."""
    co, cin = w_co_ky_kx_ci.shape[0], w_co_ky_kx_ci.shape[-1]
    if cin % 64 != 0 or co > 8:
        raise _cabi.LB200Error(f"conv_out: the N = 8 GEMM needs Cin % 64 == 0 and Cout <= 8 (got Cin {cin}, "
                               f"Cout {co})")
    w8 = torch.zeros(8, 9 * cin, dtype=w_co_ky_kx_ci.dtype, device=w_co_ky_kx_ci.device)     # fp16, or bf16
    w8[:co] = w_co_ky_kx_ci.reshape(co, 9 * cin)
    b8 = torch.zeros(8, dtype=bias.dtype, device=bias.device)
    b8[:co] = bias
    return w8.contiguous(), b8.contiguous()
