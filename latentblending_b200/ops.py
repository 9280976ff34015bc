"""Tensor-level wrappers over the C ABI (device memory and streams come from
PyTorch; all arithmetic happens in liblb200.so).  Every function requires CUDA
tensors and raises otherwise -- there is no CPU path.  The wrappers of executor op kinds record one op into a fresh
``Program`` and run it, so they go through the same records and create-time validation as the lowered programs."""
import numpy as np
import torch

from . import _cabi
from ._cabi import check, ctx, ptr, stream_ptr
from .program import LAUNCHES, Program, pack_conv_out8

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


def _cfg_step_args(latents, eps, eps_text, scaled_next, out):
    """Checks shared by the step wrappers -> (device, n, use_cfg, out, scaled batch)."""
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
    return dev, n, use_cfg, out, sb


def cfg_euler_step(latents, eps, guidance, sigma, dt, sigma_up=0.0, noise=None, out=None, traj=None,
                   scaled_next=None, next_divisor=0.0, eps_text=None):
    """eps: [2,...] (uncond, text) when CFG is on else [1,...]; or eps = uncond half and eps_text = text half
    (separate buffers).  ``scaled_next`` ([batch, ...] fp16): also write the
    next step's model input fp16(x_new / next_divisor) replicated over its batch (the next scale_model_input)."""
    dev, n, use_cfg, out, sb = _cfg_step_args(latents, eps, eps_text, scaled_next, out)
    check(_cabi.load().lb_cfg_euler_step(ctx(dev), ptr(latents), ptr(eps), ptr(eps_text), ptr(noise), ptr(out), ptr(traj), n,
                                         int(use_cfg), float(np.float32(guidance)), float(sigma), float(dt),
                                         float(sigma_up), ptr(scaled_next), sb, float(next_divisor), stream_ptr()),
          "lb_cfg_euler_step")
    LAUNCHES[0] += 1
    return out


def cfg_lcm_step(latents, eps, guidance, sc, noise=None, out=None, traj=None, scaled_next=None, next_divisor=0.0,
                 eps_text=None):
    """CFG combine + LCMScheduler step (lb_cfg_lcm_step).  ``sc``: one step's scalars from
    ``schedulers.LCMTables.step_scalars`` (sqrt_beta, inv_sqrt_alpha, c_skip, c_out, sqrt_alpha_prev, sqrt_beta_prev);
    ``noise``: the step's draw, None on the last step.  eps / eps_text / scaled_next as for cfg_euler_step (LCM's model
    input is the latent itself, so ``next_divisor`` is 1)."""
    dev, n, use_cfg, out, sb = _cfg_step_args(latents, eps, eps_text, scaled_next, out)
    check(_cabi.load().lb_cfg_lcm_step(ctx(dev), ptr(latents), ptr(eps), ptr(eps_text), ptr(noise), ptr(out), ptr(traj),
                                       n, int(use_cfg), float(np.float32(guidance)), float(sc["sqrt_beta"]),
                                       float(sc["inv_sqrt_alpha"]), float(sc["c_skip"]), float(sc["c_out"]),
                                       float(sc["sqrt_alpha_prev"]), float(sc["sqrt_beta_prev"]), ptr(scaled_next), sb,
                                       float(next_divisor), stream_ptr()), "lb_cfg_lcm_step")
    LAUNCHES[0] += 1
    return out


def cfg_dpm_step(latents, eps, guidance, sc, x0_out, x0_prev=None, noise=None, out=None, traj=None, scaled_next=None,
                 next_divisor=0.0, eps_text=None):
    """CFG combine + DPMSolverMultistepScheduler step (lb_cfg_dpm_step).  ``sc``: one scalar set of
    ``schedulers.DPMTables`` (sigma_s, inv_alpha_s, inv_r0, c_x, c_0, c_1, c_n); ``x0_prev``: the branch's previous x0
    for a second-order step, None for first order; ``x0_out``: receives this step's x0 (may be ``x0_prev``);
    ``noise``: the step's draw for sde-dpmsolver++, else None.  eps / eps_text / scaled_next as for cfg_euler_step
    (DPM's model input is the latent itself, so ``next_divisor`` is 1)."""
    dev, n, use_cfg, out, sb = _cfg_step_args(latents, eps, eps_text, scaled_next, out)
    for t in (x0_out, x0_prev):
        assert t is None or (t.dtype == torch.float16 and t.is_contiguous() and t.numel() == n)
    assert x0_out is not None
    check(_cabi.load().lb_cfg_dpm_step(ctx(dev), ptr(latents), ptr(eps), ptr(eps_text), ptr(noise), ptr(x0_prev),
                                       ptr(x0_out), ptr(out), ptr(traj), n, int(use_cfg), float(np.float32(guidance)),
                                       float(sc["sigma_s"]), float(sc["inv_alpha_s"]), float(sc["inv_r0"]),
                                       float(sc["c_x"]), float(sc["c_0"]), float(sc["c_1"]), float(sc["c_n"]),
                                       ptr(scaled_next), sb, float(next_divisor), stream_ptr()), "lb_cfg_dpm_step")
    LAUNCHES[0] += 1
    return out


def _run1(dev, emit, t=0.0):
    """Record one op with ``emit(P)`` into a fresh Program on device ``dev``, then finalize and run it."""
    P = Program(dev)
    emit(P)
    P.finalize().run(t)


def gemm(a0, w, N, B, H, W, taps=1, a0_c=None, a1=None, a1_c=None, bias=None, bias2=None, res=None, out=None,
         mode=0, out_cols=None, static_w=False, relu=False, tiling="auto", out_dtype=None,
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
                                bias2=bias2, res=res, mode=mode, static_w=static_w, relu=relu, tiling=tiling,
                                depth_to_space=depth_to_space))
    return out


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


def conv_in_add(x_nchw, w_packed, bias, Cout, addend, out=None):
    """fp16 ``conv_in`` plus ``addend`` [H*W, >=Cout], added to every image of the batch (lb_conv_in_add)."""
    dev = _dev(x_nchw)
    B, _, H, W = x_nchw.shape
    if out is None:
        out = torch.empty((B * H * W, Cout), dtype=torch.float16, device=x_nchw.device)
    _run1(dev, lambda P: P.conv_in_add(x_nchw, w_packed, bias, Cout, out, addend))
    return out


def cond_conv(x, B, H, W, Cin, w_packed, bias, Cout, stride=1, silu=False, out=None):
    """Direct 3x3 pad-1 conv (lb_cond_conv) of NHWC fp16 rows or a uint8 image [B*H*W, Cin] -> fp16
    [B*Ho*Wo, Cout], Ho = ceil(H / stride)."""
    dev = _dev(x)
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    if out is None:
        out = torch.empty((B * Ho * Wo, Cout), dtype=torch.float16, device=x.device)
    _run1(dev, lambda P: P.cond_conv(x, B, H, W, Cin, w_packed, bias, Cout, out, stride=stride, silu=silu))
    return out


def conv_out(x, B, H, W, Cin, w_packed, bias, Cout, out=None):
    """The Cin -> Cout 3x3 output convolution of NHWC ``x`` into NCHW, as the lowerings run it: ``w_packed``
    [Cout][3][3][Cin] through ``pack_conv_out8``, then ``Program.conv_out_gemm``."""
    dev = _dev(x)
    w8, b8 = pack_conv_out8(w_packed, bias)
    if out is None:
        out = torch.empty((B, Cout, H, W), dtype=x.dtype, device=x.device)
    tmp = torch.empty((B * H * W, 8), dtype=x.dtype, device=x.device)
    _run1(dev, lambda P: P.conv_out_gemm(x, B, H, W, Cin, w8, b8, Cout, out, tmp))
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


def im2col_s2_pad01(x, B, H, W, C, out=None):
    """Patch matrix of Downsample2D(padding=0) (F.pad(x, (0, 1, 0, 1)), 3x3 stride 2) of NHWC fp16 / bf16 rows."""
    dev = _dev(x)
    Ho, Wo = (H - 2) // 2 + 1, (W - 2) // 2 + 1
    if out is None:
        out = torch.empty((B * Ho * Wo, 9 * C), dtype=x.dtype, device=x.device)
    _run1(dev, lambda P: P.im2col_s2_pad01(x, B, H, W, C, out))
    return out


def image_conv_in(img_u8, w_packed, bias, Cout, out=None):
    """The VAE encoder's conv_in of a uint8 HxWx3 image with the preprocess fused (lb_image_conv_in): NHWC
    [H*W, Cout] of ``w_packed``'s type (fp16 / bf16)."""
    dev = _dev(img_u8)
    H, W, _ = img_u8.shape
    if out is None:
        out = torch.empty((H * W, Cout), dtype=w_packed.dtype, device=img_u8.device)
    _run1(dev, lambda P: P.image_conv_in(img_u8.reshape(H * W, -1), 1, H, W, w_packed, bias, Cout, out))
    return out


def add_rows_bcast(dst, src, B):
    """fp16 ``dst[b*rows + r] += src[r]`` in place for every batch row b (lb_add_rows_bcast); returns ``dst``."""
    _run1(_dev(dst), lambda P: P.add_rows_bcast(dst, src, B))
    return dst


def pixel_unshuffle_u8(img_u8, r, out=None):
    """uint8 [H, W, Cimg] -> fp16 [(H/r)*(W/r), r*r*Cimg] = u / 255, columns in (i, j, c) order
    (lb_pixel_unshuffle_u8)."""
    H, W, C = img_u8.shape
    if out is None:
        out = torch.empty(((H // r) * (W // r), r * r * C), dtype=torch.float16, device=img_u8.device)
    _run1(_dev(img_u8), lambda P: P.pixel_unshuffle_u8(img_u8, r, out))
    return out


def avgpool2_ceil(x, H, W, C, out=None):
    """AvgPool2d(2, 2, ceil_mode=True) of NHWC fp16 rows [H*W, >=C] -> [ceil(H/2)*ceil(W/2), C] (lb_avgpool2_ceil)."""
    if out is None:
        out = torch.empty((((H + 1) // 2) * ((W + 1) // 2), C), dtype=torch.float16, device=x.device)
    _run1(_dev(x), lambda P: P.avgpool2_ceil(x, H, W, C, out))
    return out


def add_noise_rows(x0, noise, coeffs, form, out=None, nonfinite=None):
    """out[r] = add_noise(x0, noise, coeffs[r]) (lb_add_noise_rows): ``x0`` fp16 / bf16 and ``noise`` fp16 with n
    elements each, ``coeffs`` a device fp16 [rows, 2] of (a, b), ``form`` _cabi.ADD_NOISE_SIGMA (x0 + b*noise) or
    ADD_NOISE_ALPHA_SIGMA (a*x0 + b*noise); -> fp16 [rows, n].  ``nonfinite`` (device int32[1]) counts non-finite x0
    elements."""
    dev = _dev(x0)
    assert x0.is_contiguous() and noise.is_contiguous() and noise.dtype == torch.float16
    assert x0.numel() == noise.numel() and coeffs.dtype == torch.float16 and coeffs.is_contiguous()
    n, rows = x0.numel(), coeffs.shape[0]
    if out is None:
        out = torch.empty((rows, n), dtype=torch.float16, device=x0.device)
    assert out.dtype == torch.float16 and out.is_contiguous() and out.numel() == rows * n
    from .program import dtype16
    check(_cabi.load().lb_add_noise_rows(ctx(dev), ptr(x0), ptr(noise), ptr(coeffs), int(form), n, rows, ptr(out),
                                         ptr(nonfinite), stream_ptr(), dtype16(x0, "add_noise x0")),
          "lb_add_noise_rows")
    LAUNCHES[0] += 1
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
