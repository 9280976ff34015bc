"""Tensor-level wrappers over the C ABI (device memory and streams come from
PyTorch; all arithmetic happens in liblb200.so).  Every function requires CUDA
tensors and raises otherwise -- there is no CPU path."""
import numpy as np
import torch

from . import _cabi
from ._cabi import check, ctx, ptr, stream_ptr

_DT = {torch.float16: 0, torch.float32: 1}
_DT16 = {torch.float16: _cabi.DTYPE_F16, torch.bfloat16: _cabi.DTYPE_BF16}   # the ops with fp16 and bf16 variants
LAUNCHES = [0]      # kernels of liblb200 launched through this module / Program.run (bench.py reports it)


def _dev(t):
    if not t.is_cuda:
        raise _cabi.LB200Error("latentblending_b200 ops need CUDA tensors (no CPU fallback)")
    return t.device.index or 0


_ws_cache = {}


def _workspace(dev, nbytes):
    buf = _ws_cache.get(dev)
    if buf is None or buf.numel() < nbytes:
        buf = torch.empty(max(nbytes, 1 << 16), dtype=torch.uint8, device=f"cuda:{dev}")
        _ws_cache[dev] = buf
    return buf


_gn_ws_cache = {}


def _gn_workspace(dev, nbytes):
    """lb_groupnorm's workspace holds 'last block' counters that must start at zero (the kernel leaves them zeroed)."""
    buf = _gn_ws_cache.get(dev)
    if buf is None or buf.numel() < nbytes:
        buf = torch.zeros(max(nbytes, 1 << 16), dtype=torch.uint8, device=f"cuda:{dev}")
        _gn_ws_cache[dev] = buf
    return buf


def slerp_rows(p0, p1, fract, out=None, fract_rows=None):
    """rows x n whole-row slerp: p0, p1 are [rows, n] (row stride arbitrary, inner
    contiguous).  utils.py:29-71 per row."""
    assert p0.dim() == 2 and p0.shape == p1.shape and p0.dtype == p1.dtype
    assert p0.stride(1) == 1 and p1.stride(1) == 1
    dev = _dev(p0)
    rows, n = p0.shape
    if out is None:
        out = torch.empty((rows, n), dtype=p0.dtype, device=p0.device)
    assert out.shape == p0.shape and out.stride(1) == 1 and out.dtype == p0.dtype
    lib = _cabi.load()
    ws = _workspace(dev, lib.lb_slerp_workspace_bytes(rows, n))
    check(lib.lb_slerp_rows(ctx(dev), ptr(p0), ptr(p1), ptr(out), rows, n,
                            p0.stride(0) if rows > 1 else n, p1.stride(0) if rows > 1 else n,
                            out.stride(0) if rows > 1 else n, _DT[p0.dtype], float(fract),
                            ptr(fract_rows), ptr(ws), stream_ptr()), "lb_slerp_rows")
    LAUNCHES[0] += 1
    return out


def lerp(p0, p1, fract):
    assert p0.shape == p1.shape and p0.dtype == p1.dtype and p0.is_contiguous() and p1.is_contiguous()
    dev = _dev(p0)
    out = torch.empty_like(p0)
    check(_cabi.load().lb_lerp(ctx(dev), ptr(p0), ptr(p1), ptr(out), p0.numel(), _DT[p0.dtype], float(fract),
                               stream_ptr()), "lb_lerp")
    LAUNCHES[0] += 1
    return out


def scale_model_input(latents, batch, divisor, out=None):
    assert latents.dtype == torch.float16 and latents.is_contiguous()
    dev = _dev(latents)
    n = latents.numel()
    if out is None:
        out = torch.empty((batch,) + tuple(latents.shape[1:]), dtype=torch.float16, device=latents.device)
    check(_cabi.load().lb_scale_model_input(ctx(dev), ptr(latents), ptr(out), n, int(batch), float(divisor),
                                            stream_ptr()), "lb_scale_model_input")
    LAUNCHES[0] += 1
    return out


def cfg_euler_step(latents, eps, guidance, sigma, dt, sigma_up=0.0, noise=None, out=None, traj=None,
                   scaled_next=None, next_divisor=0.0, eps_text=None):
    """eps: [2,...] (uncond, text) when CFG is on else [1,...]; or eps = uncond half and eps_text = text half
    (separate buffers).  ``scaled_next`` ([batch, ...] fp16): also write the
    next step's model input fp16(x_new / next_divisor) replicated over its batch (the next scale_model_input)."""
    assert latents.dtype == torch.float16 and eps.dtype == torch.float16
    assert latents.is_contiguous() and eps.is_contiguous()
    dev = _dev(latents)
    n = latents.numel()
    use_cfg = eps.numel() == 2 * n or eps_text is not None
    assert use_cfg or eps.numel() == n
    if eps_text is not None:
        assert eps_text.dtype == torch.float16 and eps_text.is_contiguous() and eps_text.numel() == n
    if out is None:
        out = torch.empty_like(latents)
    sb = 0
    if scaled_next is not None:
        assert scaled_next.dtype == torch.float16 and scaled_next.is_contiguous() and scaled_next.numel() % n == 0
        sb = scaled_next.numel() // n
    check(_cabi.load().lb_cfg_euler_step(ctx(dev), ptr(latents), ptr(eps), ptr(eps_text), ptr(noise), ptr(out), ptr(traj), n,
                                         int(use_cfg), float(np.float32(guidance)), float(sigma), float(dt),
                                         float(sigma_up), ptr(scaled_next), sb, float(next_divisor), stream_ptr()),
          "lb_cfg_euler_step")
    LAUNCHES[0] += 1
    return out


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


_TILING = {"auto": 0, "box": _cabi.GEMM_TILE_BOX, "runs": _cabi.GEMM_TILE_RUNS}


def gemm(a0, w, N, B, H, W, taps=1, a0_c=None, a1=None, a1_c=None, bias=None, bias2=None, res=None, out=None,
         mode=0, out_cols=None, static_w=False, relu=False, ln=None, stats_out=None, tiling="auto", out_dtype=None,
         depth_to_space=False):
    """Tensor-core GEMM / implicit-GEMM conv (lb_gemm).  a0: NHWC activation viewed as
    [B*H*W, >=a0_c] (row stride = a0.stride(0)); w: [N, K] packed weights.
    ``tiling``: "auto" (the M tiling with fewer tiles), "box" (pixel boxes) or "runs" (pixel runs); all give the
    same results.
    Element types come from the tensors: fp16 throughout, or bf16 a0 / w / a1 / bias / bias2 / res (LB_GEMM_BF16)
    with a bf16 output, or an fp16 one when ``out_dtype`` (default: ``out``'s dtype, else a0's) is torch.float16.
    ``depth_to_space`` (LB_GEMM_D2S2): nearest-2x upsample + 3x3 conv of the H x W map a0, with ``w`` the [4*Co, 9*C]
    phase weights (``taesd.pack_d2s_weights``); the output is the [B*2H*2W, Co] NHWC map."""
    if tiling not in _TILING:
        raise ValueError(f"tiling must be one of {sorted(_TILING)} (got {tiling!r})")
    dev = _dev(a0)
    M = B * H * W
    a0_c = a0.shape[-1] if a0_c is None else a0_c
    n_out = (N // 2 if mode == 1 else N) if out_cols is None else out_cols
    if out_dtype is None:
        out_dtype = out.dtype if out is not None else a0.dtype
    elif out is not None and out.dtype != out_dtype:
        raise _cabi.LB200Error(f"gemm: out is {out.dtype}, out_dtype {out_dtype}")
    dmode = gemm_dtype_mode(a0, w, out_dtype, a1, bias, bias2, res)
    if depth_to_space:
        dmode |= _cabi.GEMM_D2S2
    if out is None:
        shape = (4 * M, N // 4) if depth_to_space else (M, n_out)
        out = torch.empty(shape, dtype=out_dtype, device=a0.device)
    d = _cabi.GemmDesc()
    d.a0, d.a0_ld, d.a0_c = _p(a0), a0.stride(-2), a0_c
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
    d.mode = mode | (_cabi.GEMM_STATIC_W if static_w else 0) | (_cabi.GEMM_RELU if relu else 0) | _TILING[tiling] | dmode
    if ln is not None:
        d.ln_stats, d.ln_parts = _p(ln["stats"]), ln["stats"].shape[1]
        d.ln_csum, d.ln_bias, d.ln_eps = _p(ln["csum"]), _p(ln["bias"]), ln["eps"]
    if stats_out is not None:
        d.stats_out, d.stats_parts = _p(stats_out), stats_out.shape[1]
    check(_cabi.load().lb_gemm(ctx(dev), d, stream_ptr()), "lb_gemm")
    return out


def gemm_stats_parts(a0, w, N, B, H, W, **kw):
    """Per-row partial count of lb_gemm's stats_out for this problem (4 per N tile)."""
    import ctypes
    dev = _dev(a0)
    d = _cabi.GemmDesc()
    M = B * H * W
    out = torch.empty((M, N), dtype=torch.float16, device=a0.device)
    d.a0, d.a0_ld, d.a0_c = _p(a0), a0.stride(-2), kw.get("a0_c") or a0.shape[-1]
    d.B, d.H, d.W, d.taps = B, H, W, kw.get("taps", 1)
    d.w, d.w_ld, d.N = _p(w), w.stride(0), N
    d.out, d.out_ld, d.mode = _p(out), out.stride(-2), kw.get("mode", 0)
    return int(_cabi.load().lb_gemm_stats_parts(ctx(dev), ctypes.byref(d)))


def lpips_tap(feat_a, feat_b, lin_w, out_scalar, workspace, accumulate=False):
    """One LPIPS tap reduction over [pixels, C] fp16 feature matrices (lb_lpips_tap)."""
    dev = _dev(feat_a)
    assert feat_a.shape == feat_b.shape and feat_a.stride(0) == feat_b.stride(0) and feat_a.dtype == torch.float16
    rows, C = feat_a.shape
    check(_cabi.load().lb_lpips_tap(ctx(dev), ptr(feat_a), ptr(feat_b), feat_a.stride(0), rows, C, ptr(lin_w),
                                    int(accumulate), ptr(out_scalar), ptr(workspace), stream_ptr()), "lb_lpips_tap")
    LAUNCHES[0] += 2
    return out_scalar


def frames_lerp_u8(frames, left, w0, w1, out=None):
    """frames [F, n] uint8 (contiguous); left int32 [T], w0/w1 float32 [T] on the device -> [T, n] uint8
    (lb_frames_lerp_u8: numpy-float32 blend with truncating uint8 cast)."""
    dev = _dev(frames)
    assert frames.dtype == torch.uint8 and frames.is_contiguous() and frames.dim() == 2
    T = left.numel()
    if out is None:
        out = torch.empty((T, frames.shape[1]), dtype=torch.uint8, device=frames.device)
    check(_cabi.load().lb_frames_lerp_u8(ctx(dev), ptr(frames), frames.shape[1], ptr(left), ptr(w0), ptr(w1), T,
                                         ptr(out), stream_ptr()), "lb_frames_lerp_u8")
    LAUNCHES[0] += 1
    return out


def error_flag(dev=0):
    import ctypes
    code = ctypes.c_int(0)
    check(_cabi.load().lb_ctx_error_flag(ctx(dev), ctypes.byref(code)), "lb_ctx_error_flag")
    return code.value


def attention(q, k, v, out, B, heads, Sq, Skv, q_col0=0, k_col0=0, v_col0=0, scale=0.125):
    """q/k/v: 2-D row-major fp16 buffers whose column slices hold the heads (lb_attention)."""
    dev = _dev(q)
    d = _cabi.AttnDesc()
    d.q, d.q_ld, d.q_col0 = _p(q), q.stride(0), q_col0
    d.k, d.k_ld, d.k_col0 = _p(k), k.stride(0), k_col0
    d.v, d.v_ld, d.v_col0 = _p(v), v.stride(0), v_col0
    d.out, d.out_ld = _p(out), out.stride(0)
    d.B, d.heads, d.Sq, d.Skv, d.head_dim, d.scale = B, heads, Sq, Skv, 64, scale
    check(_cabi.load().lb_attention(ctx(dev), d, stream_ptr()), "lb_attention")
    return out


def groupnorm(x, B, HW, C, groups, gamma, beta, eps, silu, out=None):
    """fp16 or bf16 (x, gamma, beta and out of one type)."""
    dev = _dev(x)
    dt = dtype16(x, "groupnorm x")
    if out is None:
        out = torch.empty((B * HW, C), dtype=x.dtype, device=x.device)
    _same_dtype(x.dtype, "groupnorm x / gamma / beta / out", gamma, beta, out)
    lib = _cabi.load()
    ws = _gn_workspace(dev, lib.lb_groupnorm_workspace_bytes(ctx(dev), B, HW, groups))
    check(lib.lb_groupnorm_dt(ctx(dev), ptr(x), x.stride(0), B, HW, C, groups, ptr(gamma), ptr(beta), float(eps),
                              int(silu), ptr(out), out.stride(0), ptr(ws), stream_ptr(), dt), "lb_groupnorm")
    return out


def layernorm(x, gamma, beta, eps=1e-5, out=None):
    dev = _dev(x)
    rows, C = x.shape
    if out is None:
        out = torch.empty((rows, C), dtype=torch.float16, device=x.device)
    check(_cabi.load().lb_layernorm(ctx(dev), ptr(x), x.stride(0), rows, C, ptr(gamma), ptr(beta), float(eps),
                                    ptr(out), out.stride(0), stream_ptr()), "lb_layernorm")
    return out


def embed_inputs(t, text_embeds, time_ids, dim_t, dim_a):
    dev = _dev(text_embeds)
    B, pooled = text_embeds.shape
    temb_in = torch.empty((B, dim_t), dtype=torch.float16, device=text_embeds.device)
    add_in = torch.empty((B, pooled + 6 * dim_a), dtype=torch.float16, device=text_embeds.device)
    check(_cabi.load().lb_embed_inputs(ctx(dev), float(t), ptr(text_embeds), ptr(time_ids), B, dim_t, pooled, dim_a,
                                       ptr(temb_in), ptr(add_in), stream_ptr()), "lb_embed_inputs")
    return temb_in, add_in


def linear_small(x, w, bias=None, addend=None, act_in=0, act_out=0, out=None):
    dev = _dev(x)
    M, K = x.shape
    N = w.shape[0]
    if out is None:
        out = torch.empty((M, N), dtype=torch.float16, device=x.device)
    check(_cabi.load().lb_linear_small(ctx(dev), ptr(x), x.stride(0), M, K, ptr(w), w.stride(0), ptr(bias),
                                       ptr(addend), 0 if addend is None else addend.stride(0), act_in, act_out,
                                       ptr(out), out.stride(0), N, stream_ptr()), "lb_linear_small")
    return out


def conv_in(x_nchw, w_packed, bias, Cout, out=None, act=0, in_scale=1.0):
    """fp16 or bf16 (x, weights, bias and out of one type).  ``act`` 1 (fp16): the tiny VAE decoder's input stage,
    tanh(x * in_scale / 3) * 3 before the conv and ReLU after it (lb_conv_in_act)."""
    dev = _dev(x_nchw)
    dt = dtype16(x_nchw, "conv_in x")
    B, Cin, H, W = x_nchw.shape
    if out is None:
        out = torch.empty((B * H * W, Cout), dtype=x_nchw.dtype, device=x_nchw.device)
    _same_dtype(x_nchw.dtype, "conv_in x / w / bias / out", w_packed, bias, out)
    if act:
        check(_cabi.load().lb_conv_in_act(ctx(dev), ptr(x_nchw), B, Cin, H, W, ptr(w_packed), ptr(bias), Cout,
                                          ptr(out), out.stride(0), int(act), float(in_scale), stream_ptr(), dt),
              "lb_conv_in_act")
        return out
    check(_cabi.load().lb_conv_in_dt(ctx(dev), ptr(x_nchw), B, Cin, H, W, ptr(w_packed), ptr(bias), Cout, ptr(out),
                                     out.stride(0), stream_ptr(), dt), "lb_conv_in")
    return out


def conv_out(x, B, H, W, Cin, w_packed, bias, Cout, out=None):
    dev = _dev(x)
    if out is None:
        out = torch.empty((B, Cout, H, W), dtype=torch.float16, device=x.device)
    check(_cabi.load().lb_conv_out(ctx(dev), ptr(x), x.stride(0), B, Cin, H, W, ptr(w_packed), ptr(bias), Cout,
                                   ptr(out), stream_ptr()), "lb_conv_out")
    return out


def upsample2x(x, B, H, W, C, out=None):
    dev = _dev(x)
    if out is None:
        out = torch.empty((B * 4 * H * W, C), dtype=torch.float16, device=x.device)
    check(_cabi.load().lb_upsample2x(ctx(dev), ptr(x), x.stride(0), B, H, W, C, ptr(out), out.stride(0),
                                     stream_ptr()), "lb_upsample2x")
    return out


def upsample_nearest(x, B, H, W, C, Ho, Wo, out=None):
    """F.interpolate(size=(Ho, Wo), mode="nearest") of NHWC rows [B*H*W, >=C] for Ho in {2H-1, 2H}, Wo in
    {2W-1, 2W} (lb_upsample_nearest; other sizes raise LB200Error)."""
    dev = _dev(x)
    dt = dtype16(x, "upsample x")
    if out is None:
        out = torch.empty((B * Ho * Wo, C), dtype=x.dtype, device=x.device)
    _same_dtype(x.dtype, "upsample x / out", out)
    check(_cabi.load().lb_upsample_nearest_dt(ctx(dev), ptr(x), x.stride(0), B, H, W, C, ptr(out), out.stride(0),
                                              Ho, Wo, stream_ptr(), dt), "lb_upsample_nearest")
    return out


def im2col_s2(x, B, H, W, C, out=None):
    dev = _dev(x)
    Ho, Wo = (H + 1) // 2, (W + 1) // 2
    if out is None:
        out = torch.empty((B * Ho * Wo, 9 * C), dtype=torch.float16, device=x.device)
    check(_cabi.load().lb_im2col_s2(ctx(dev), ptr(x), x.stride(0), B, H, W, C, ptr(out), stream_ptr()),
          "lb_im2col_s2")
    return out


# ---- VAE-decoder helpers (fp16 or bf16; the decoder itself records them into a Program) ---------------------------


def latent_prep(x_nchw, w_f32, bias_f32, out_dtype=torch.float16, out=None):
    """post_quant_conv(latents / scaling_factor): fp16 NCHW latents in, ``out_dtype`` (fp16 / bf16) NCHW out."""
    dev = _dev(x_nchw)
    assert x_nchw.dtype == torch.float16 and x_nchw.is_contiguous()
    B, C, H, W = x_nchw.shape
    if out is None:
        out = torch.empty((B, C, H, W), dtype=out_dtype, device=x_nchw.device)
    check(_cabi.load().lb_latent_prep_dt(ctx(dev), ptr(x_nchw), B, C, H * W, ptr(w_f32), ptr(bias_f32), ptr(out),
                                         stream_ptr(), dtype16(out, "latent_prep out")), "lb_latent_prep")
    return out


def softmax_rows(x, out=None, out_dtype=None):
    """Row softmax of fp16 ``x`` [rows, cols] into fp16 or bf16 ``out`` (may be x itself)."""
    dev = _dev(x)
    assert x.dtype == torch.float16
    if out is None:
        out = torch.empty(x.shape, dtype=out_dtype or x.dtype, device=x.device)
    check(_cabi.load().lb_softmax_rows_dt(ctx(dev), ptr(x), x.stride(0), x.shape[0], x.shape[1], ptr(out),
                                          out.stride(0), stream_ptr(), dtype16(out, "softmax out")), "lb_softmax_rows")
    return out


def postprocess_u8(img_nchw, out=None, nonfinite=None):
    """fp16 / bf16 NCHW image -> uint8 NHWC; ``nonfinite`` (device int32[1]) accumulates the non-finite pixel count."""
    dev = _dev(img_nchw)
    assert img_nchw.is_contiguous()
    B, C, H, W = img_nchw.shape
    if out is None:
        out = torch.empty((B, H, W, C), dtype=torch.uint8, device=img_nchw.device)
    check(_cabi.load().lb_postprocess_u8_dt(ctx(dev), ptr(img_nchw), B, C, H * W, ptr(out), ptr(nonfinite),
                                            stream_ptr(), dtype16(img_nchw, "postprocess image")), "lb_postprocess_u8")
    return out


def nhwc_to_nchw(x, B, C, H, W, out=None):
    """The first C (<= 8) columns of fp16 / bf16 NHWC rows [B*H*W, ld] -> NCHW [B, C, H, W]."""
    dev = _dev(x)
    if out is None:
        out = torch.empty((B, C, H, W), dtype=x.dtype, device=x.device)
    _same_dtype(x.dtype, "nhwc_to_nchw x / out", out)
    check(_cabi.load().lb_nhwc_to_nchw_dt(ctx(dev), ptr(x), x.stride(0), B, C, H * W, ptr(out), stream_ptr(),
                                          dtype16(x, "nhwc_to_nchw x")), "lb_nhwc_to_nchw")
    return out
