"""Tensor-level wrappers over the C ABI (device memory and streams come from
PyTorch; all arithmetic happens in liblb200.so).  Every function requires CUDA
tensors and raises otherwise -- there is no CPU path.  The wrappers of executor op kinds record one op into a fresh
``Program`` and run it, so they go through the same records and create-time validation as the lowered programs."""
import numpy as np
import torch

from . import _cabi
from ._cabi import check, ctx, ptr, stream_ptr
from .program import LAUNCHES, Program

_DT = {torch.float16: 0, torch.float32: 1}


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


def _run1(dev, emit, t=0.0):
    """Record one op with ``emit(P)`` into a fresh Program on device ``dev``, then finalize and run it."""
    P = Program(dev)
    emit(P)
    P.finalize().run(t)


def gemm(a0, w, N, B, H, W, taps=1, a0_c=None, a1=None, a1_c=None, bias=None, bias2=None, res=None, out=None,
         mode=0, out_cols=None, static_w=False, relu=False, ln=None, stats_out=None, tiling="auto", out_dtype=None,
         depth_to_space=False):
    """Tensor-core GEMM / implicit-GEMM conv (``Program.gemm``).  The output (allocated unless ``out`` is given) is
    [B*H*W, N] (N/2 with GEGLU, ``out_cols`` when given), or [B*2H*2W, N/4] with ``depth_to_space``, of type
    ``out_dtype`` (default: ``out``'s, else a0's)."""
    dev = _dev(a0)
    M = B * H * W
    n_out = (N // 2 if mode == 1 else N) if out_cols is None else out_cols
    if out_dtype is None:
        out_dtype = out.dtype if out is not None else a0.dtype
    elif out is not None and out.dtype != out_dtype:
        raise _cabi.LB200Error(f"gemm: out is {out.dtype}, out_dtype {out_dtype}")
    if out is None:
        shape = (4 * M, N // 4) if depth_to_space else (M, n_out)
        out = torch.empty(shape, dtype=out_dtype, device=a0.device)
    _run1(dev, lambda P: P.gemm(a0, w, N, B, H, W, out, taps=taps, a0_c=a0_c, a1=a1, a1_c=a1_c, bias=bias,
                                bias2=bias2, res=res, mode=mode, static_w=static_w, relu=relu, ln=ln,
                                stats_out=stats_out, tiling=tiling, depth_to_space=depth_to_space))
    return out


def gemm_stats_parts(a0, w, N, B, H, W, **kw):
    """Per-row partial count of lb_gemm's stats_out for this problem (4 per N tile)."""
    out = torch.empty((B * H * W, N), dtype=torch.float16, device=a0.device)
    return Program(_dev(a0)).gemm_stats_parts(a0, w, N, B, H, W, out, **kw)


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
    _run1(_dev(q), lambda P: P.attention(q, k, v, out, B, heads, Sq, Skv, q_col0, k_col0, v_col0, scale))
    return out


def groupnorm(x, B, HW, C, groups, gamma, beta, eps, silu, out=None):
    """fp16 or bf16 (x, gamma, beta and out of one type)."""
    dev = _dev(x)
    if out is None:
        out = torch.empty((B * HW, C), dtype=x.dtype, device=x.device)
    ws = _gn_workspace(dev, _cabi.load().lb_groupnorm_workspace_bytes(ctx(dev), B, HW, groups))
    _run1(dev, lambda P: P.groupnorm(x, B, HW, C, groups, gamma, beta, float(eps), silu, out, ws))
    return out


def layernorm(x, gamma, beta, eps=1e-5, out=None):
    dev = _dev(x)
    rows, C = x.shape
    if out is None:
        out = torch.empty((rows, C), dtype=torch.float16, device=x.device)
    _run1(dev, lambda P: P.layernorm(x, gamma, beta, float(eps), out))
    return out


def embed_inputs(t, text_embeds, time_ids, dim_t, dim_a):
    dev = _dev(text_embeds)
    B, pooled = text_embeds.shape
    temb_in = torch.empty((B, dim_t), dtype=torch.float16, device=text_embeds.device)
    add_in = torch.empty((B, pooled + 6 * dim_a), dtype=torch.float16, device=text_embeds.device)
    _run1(dev, lambda P: P.embed_inputs(text_embeds, time_ids, dim_t, dim_a, temb_in, add_in), t)
    return temb_in, add_in


def linear_small(x, w, bias=None, addend=None, act_in=0, act_out=0, out=None):
    dev = _dev(x)
    M, _ = x.shape
    if out is None:
        out = torch.empty((M, w.shape[0]), dtype=torch.float16, device=x.device)
    _run1(dev, lambda P: P.linear_small(x, w, out, bias=bias, addend=addend, act_in=act_in, act_out=act_out))
    return out


def conv_in(x_nchw, w_packed, bias, Cout, out=None, act=_cabi.CONV_IN_PLAIN, in_scale=1.0):
    """fp16 or bf16 (x, weights, bias and out of one type).  ``act`` 1 (fp16): the tiny VAE decoder's input stage,
    tanh(x * in_scale / 3) * 3 before the conv and ReLU after it."""
    dev = _dev(x_nchw)
    B, _, H, W = x_nchw.shape
    if out is None:
        out = torch.empty((B * H * W, Cout), dtype=x_nchw.dtype, device=x_nchw.device)
    _run1(dev, lambda P: P.conv_in(x_nchw, w_packed, bias, Cout, out, act, in_scale))
    return out


def conv_out(x, B, H, W, Cin, w_packed, bias, Cout, out=None):
    dev = _dev(x)
    if out is None:
        out = torch.empty((B, Cout, H, W), dtype=torch.float16, device=x.device)
    _run1(dev, lambda P: P.conv_out(x, B, H, W, Cin, w_packed, bias, Cout, out))
    return out


def upsample2x(x, B, H, W, C, out=None):
    return upsample_nearest(x, B, H, W, C, 2 * H, 2 * W, out=out)


def upsample_nearest(x, B, H, W, C, Ho, Wo, out=None):
    """F.interpolate(size=(Ho, Wo), mode="nearest") of NHWC rows [B*H*W, >=C] for Ho in {2H-1, 2H}, Wo in
    {2W-1, 2W} (lb_upsample_nearest; other sizes raise LB200Error)."""
    dev = _dev(x)
    if out is None:
        out = torch.empty((B * Ho * Wo, C), dtype=x.dtype, device=x.device)
    _run1(dev, lambda P: P.upsample_nearest(x, B, H, W, C, out, Ho, Wo))
    return out


def im2col_s2(x, B, H, W, C, out=None):
    dev = _dev(x)
    Ho, Wo = (H + 1) // 2, (W + 1) // 2
    if out is None:
        out = torch.empty((B * Ho * Wo, 9 * C), dtype=torch.float16, device=x.device)
    _run1(dev, lambda P: P.im2col_s2(x, B, H, W, C, out))
    return out


# ---- VAE-decoder helpers (fp16 or bf16) ---------------------------------------------------------------------------


def latent_prep(x_nchw, w_f32, bias_f32, out_dtype=torch.float16, out=None):
    """post_quant_conv(latents / scaling_factor): fp16 NCHW latents in, ``out_dtype`` (fp16 / bf16) NCHW out."""
    dev = _dev(x_nchw)
    assert x_nchw.dtype == torch.float16 and x_nchw.is_contiguous()
    if out is None:
        out = torch.empty(x_nchw.shape, dtype=out_dtype, device=x_nchw.device)
    _run1(dev, lambda P: P.latent_prep(x_nchw, w_f32, bias_f32, out))
    return out


def softmax_rows(x, out=None, out_dtype=None):
    """Row softmax of fp16 ``x`` [rows, cols] into fp16 or bf16 ``out`` (may be x itself)."""
    dev = _dev(x)
    assert x.dtype == torch.float16
    if out is None:
        out = torch.empty(x.shape, dtype=out_dtype or x.dtype, device=x.device)
    _run1(dev, lambda P: P.softmax_rows(x, out))
    return out


def postprocess_u8(img_nchw, out=None, nonfinite=None):
    """fp16 / bf16 NCHW image -> uint8 NHWC; ``nonfinite`` (device int32[1]) accumulates the non-finite pixel count."""
    dev = _dev(img_nchw)
    assert img_nchw.is_contiguous()
    B, C, H, W = img_nchw.shape
    if out is None:
        out = torch.empty((B, H, W, C), dtype=torch.uint8, device=img_nchw.device)
    _run1(dev, lambda P: P.postprocess_u8(img_nchw, out, nonfinite))
    return out


def nhwc_to_nchw(x, B, C, H, W, out=None):
    """The first C (<= 8) columns of fp16 / bf16 NHWC rows [B*H*W, ld] -> NCHW [B, C, H, W]."""
    dev = _dev(x)
    if out is None:
        out = torch.empty((B, C, H, W), dtype=x.dtype, device=x.device)
    _run1(dev, lambda P: P.nhwc_to_nchw(x, B, C, H, W, out))
    return out
