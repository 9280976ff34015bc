"""Per-element error bounds for the fp16 kernels of the UNet hot path (GEMM / implicit-GEMM conv, attention, GroupNorm,
LayerNorm) and the small boundary ops, each against an fp64 reference computed on the GPU from the very fp16 (bf16)
operands the kernel saw.  Every element must satisfy its own bound; a check over the whole tensor's largest value
would let a small element, a ragged tile or one head be a few percent off.

Bounds, |got - ref| <= ..., with these terms:
  ULP  = 2^-10 |ref|     one fp16 ulp of the result (the output is rounded to fp16: half an ulp, with margin)
  ACC  = 2^-16 sum|a||w| fp32 accumulation of a dot product in any order.  A rounding of 2^-24 per addition, summed
                         over K / 16 wgmma k-steps even at K = 23 040, stays far below it (test_gemm_long_k checks
                         K = 23 040 and 5 120 against it); the same constant as the bf16 GEMM tests
  TINY = 2^-24           the fp16 subnormal spacing
  * GEMM:      ULP + ACC + TINY, with |bias|, |bias2| and |res| added to sum|a||w| (they join the fp32 sum).
               ReLU is 1-Lipschitz, so it keeps the bound of its input.
  * GEGLU:     the reference rounds proj, gelu(gate) and the product to fp16; one ulp of difference is allowed at
               each of the three, propagated to first order (|gelu'| <= 1.13), plus ACC of each dot product.
  * attention: ULP + 2^-9 sum_j p_j |v_j| + TINY.  The middle term covers P rounded to fp16 before the P V product
               (2^-11 relative per term), the normaliser summing the unrounded P, and ex2.approx (2^-22 relative).
  * GroupNorm / LayerNorm: one ulp at each of the reference's rounding points (the affine output, then SiLU), plus
               SiLU's slope (<= 1.1) times the affine rounding, plus NORM = 2^-22 (rstd |gamma| (|x| + |mean|) + |beta|):
               the fp32 evaluation x * scale + shift that the kernel and torch's own GroupNorm / LayerNorm both use,
               with mean and rstd held in fp32.  NORM is what a large mean/sigma costs an exact-statistics kernel; it is
               well below the error of statistics that lose precision as mean/sigma grows.
  * postprocess_u8: equality with diffusers' chain on the same tensor.
  * linear_small / conv_in / conv_out / embed_inputs: ULP at each fp16 rounding the op makes, ACC of the dot product.

Non-vacuity: each family's bound is also applied to a deliberately wrong result, which it must reject; the rejected
error is printed as a multiple of the bound (run with -s to see it)."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

ULP = 2.0 ** -10
ACC = 2.0 ** -16
TINY = 2.0 ** -24
NORM = 2.0 ** -22
P_TERM = 2.0 ** -9
SILU_SLOPE = 1.1
GELU_SLOPE = 1.13
H = torch.float16
BF = torch.bfloat16
D = torch.float64
SENTINEL = -12344.0          # exactly representable in fp16 and bf16


def _rand(*shape, seed, s=1.0, mean=0.0, dtype=H):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(*shape, generator=g, device="cuda") * s + mean).to(dtype)


def _ops():
    from latentblending_b200 import ops
    return ops


def check(got, ref, bound, what):
    """Every element: |got - ref| <= bound (fp64).  Returns the largest err / bound; on failure reports the worst
    element, its index and err / bound, and how many elements exceed the bound."""
    got, ref = got.to(D), ref.to(D)
    bound = torch.broadcast_to(bound.to(D) if torch.is_tensor(bound) else torch.tensor(bound, dtype=D,
                                                                                      device=ref.device), ref.shape)
    err = (got - ref).abs()
    err = torch.where(torch.isnan(err), torch.full_like(err, math.inf), err)
    ratio = err / bound
    worst = int(ratio.argmax())
    r = ratio.reshape(-1)[worst].item()
    if not r <= 1.0:
        idx = tuple(int(i) for i in torch.unravel_index(torch.tensor(worst), ref.shape))
        bad = int((ratio > 1.0).sum())
        raise AssertionError(f"{what}: {bad} of {ref.numel()} elements exceed the bound; worst at {idx}: "
                             f"got {got[idx].item():.8g} ref {ref[idx].item():.8g} err {err[idx].item():.3g} "
                             f"bound {bound[idx].item():.3g} err/bound {r:.3g}")
    return r


def reject(got, ref, bound, what):
    """Non-vacuity: the bound must reject a deliberately wrong result; prints the rejected error / bound."""
    with pytest.raises(AssertionError):
        check(got, ref, bound, what)
    got, ref = got.to(D), ref.to(D)
    r = ((got - ref).abs() / torch.broadcast_to(bound.to(D), ref.shape)).max().item()
    print(f"non-vacuity {what}: rejected, worst err = {r:.3g} x bound")
    return r


def _flag_clear():
    torch.cuda.synchronize()
    assert _ops().error_flag() == 0


# ---- GEMM / implicit-GEMM conv ---------------------------------------------------------------------------------------
def _linear_ref(a, w, extra=()):
    """fp64 a w^T (+ each tensor of ``extra``, broadcast) and its magnitude term sum|a||w| (+ |extra|)."""
    ref = a.to(D) @ w.to(D).T
    mag = a.to(D).abs() @ w.to(D).abs().T
    for e in extra:
        ref = ref + e.to(D)
        mag = mag + e.to(D).abs()
    return ref, mag


def _conv3x3_ref(x, B, Hh, Ww, wp):
    """fp64 3x3 pad-1 convolution of NHWC rows x [B*H*W, C] (any row stride) with packed weights wp [N, 9*C]
    ((ky, kx, c) order): one shifted matmul per tap, one image at a time.  -> (ref, sum|a||w|), [B*H*W, N]."""
    C, N = x.shape[1], wp.shape[0]
    w = wp.to(D).view(N, 3, 3, C)
    ref = torch.zeros(B * Hh * Ww, N, dtype=D, device=x.device)
    mag = torch.zeros_like(ref)
    for b in range(B):
        rows = slice(b * Hh * Ww, (b + 1) * Hh * Ww)
        xp = F.pad(x[rows].to(D).reshape(Hh, Ww, C), (0, 0, 1, 1, 1, 1))
        for ky in range(3):
            for kx in range(3):
                xs = xp[ky:ky + Hh, kx:kx + Ww].reshape(Hh * Ww, C)
                wt = w[:, ky, kx, :]
                ref[rows] += xs @ wt.T
                mag[rows] += xs.abs() @ wt.abs().T
    return ref, mag


def _gemm_bound(ref, mag):
    return ULP * ref.abs() + ACC * mag + TINY


def _sentinel_out(rows, cols, lead=8, trail=24, dtype=H):
    """A column slice [:, lead:lead + cols] of a sentinel-filled buffer (16-byte aligned, row stride % 8 == 0)."""
    buf = torch.full((rows, lead + cols + trail), SENTINEL, dtype=dtype, device="cuda")
    return buf, buf[:, lead:lead + cols]


def _assert_sentinels(buf, lead, cols, what):
    outside = torch.cat([buf[:, :lead], buf[:, lead + cols:]], 1)
    assert bool((outside == SENTINEL).all()), f"{what}: a write outside the output columns"


@pytest.mark.parametrize("M,K,N", [(1000, 640, 8), (300, 640, 64), (777, 640, 384), (1000, 640, 200),
                                   (513, 640, 320), (1000, 1280, 1280)])
def test_gemm_every_n_tile(M, K, N):
    """N tiles 64 (N = 8, 64), 128 (N = 384, and the ragged N = 200: one full tile and 72 columns of the second) and
    160 (N = 320, 1280), ragged M, bias, the output a column slice of a sentinel-filled buffer.  Non-vacuity: the
    kernel's own output with one 16-wide k-slice of A zeroed."""
    ops = _ops()
    a, w, b = _rand(M, K, seed=1), _rand(N, K, seed=2, s=K ** -0.5), _rand(N, seed=3)
    buf, out = _sentinel_out(M, N)
    ops.gemm(a, w, N, 1, 1, M, bias=b, out=out)
    ref, mag = _linear_ref(a, w, (b,))
    bound = _gemm_bound(ref, mag)
    check(out, ref, bound, f"linear M={M} K={K} N={N}")
    _assert_sentinels(buf, 8, N, "linear")
    a_bad = a.clone()
    a_bad[:, 208:224] = 0
    reject(ops.gemm(a_bad, w, N, 1, 1, M, bias=b), ref, bound, f"GEMM N={N} with k-slice [208, 224) of A zeroed")
    _flag_clear()


def test_gemm_ragged_m_both_tilings():
    """Ragged M through the pixel box and the pixel runs, forced: a linear with M = 300 and a 3x3 conv whose second box
    holds one image of two (B = 3, 8 x 8).  Both tilings are bit-identical and within the bound."""
    ops = _ops()
    M, K, N = 300, 320, 320
    a, w, b = _rand(M, K, seed=4), _rand(N, K, seed=5, s=K ** -0.5), _rand(N, seed=6)
    outs = {t: ops.gemm(a, w, N, 1, 1, M, bias=b, tiling=t) for t in ("box", "runs")}
    assert torch.equal(outs["box"], outs["runs"])
    ref, mag = _linear_ref(a, w, (b,))
    check(outs["runs"], ref, _gemm_bound(ref, mag), "linear M=300")
    B, Hh, Ww, C, N = 3, 8, 8, 64, 320
    x, wc, bc = _rand(B * Hh * Ww, C, seed=7), _rand(N, 9 * C, seed=8, s=(9 * C) ** -0.5), _rand(N, seed=9)
    outs = {t: ops.gemm(x, wc, N, B, Hh, Ww, taps=9, bias=bc, tiling=t) for t in ("box", "runs")}
    assert torch.equal(outs["box"], outs["runs"])
    ref, mag = _conv3x3_ref(x, B, Hh, Ww, wc)
    ref, mag = ref + bc.to(D), mag + bc.to(D).abs()
    check(outs["box"], ref, _gemm_bound(ref, mag), "conv B=3 8x8")
    _flag_clear()


@pytest.mark.parametrize("B,Hh,Ww,Cin,N,tiling", [(8, 4, 4, 64, 128, "box"), (3, 9, 7, 128, 320, "runs"),
                                                  (2, 5, 27, 64, 200, "runs")])
def test_gemm_conv_epilogues(B, Hh, Ww, Cin, N, tiling):
    """3x3 conv + bias + time-embedding bias2 (a row-strided slice) + residual, separate and in place: box tiles that
    span eight images, and runs that cross image boundaries.  Then the 1x1 shortcut as a second K segment (a1) and the
    ReLU epilogue on the same shape."""
    ops = _ops()
    M = B * Hh * Ww
    x = _rand(M, Cin, seed=10)
    wc = _rand(N, 9 * Cin, seed=11, s=(9 * Cin) ** -0.5)
    b = _rand(N, seed=12)
    tbuf = _rand(B, N + 40, seed=13)
    temb = tbuf[:, 16:16 + N]
    res = _rand(M, N, seed=14)
    ref, mag = _conv3x3_ref(x, B, Hh, Ww, wc)
    rows_b = torch.arange(M, device="cuda") // (Hh * Ww)
    tb = temb.to(D)[rows_b]
    ref = ref + b.to(D) + tb + res.to(D)
    mag = mag + b.to(D).abs() + tb.abs() + res.to(D).abs()
    sep = ops.gemm(x, wc, N, B, Hh, Ww, taps=9, bias=b, bias2=temb, res=res, tiling=tiling)
    check(sep, ref, _gemm_bound(ref, mag), f"conv+bias+temb+res B={B} {Hh}x{Ww} {tiling}")
    hs = res.clone()
    ops.gemm(x, wc, N, B, Hh, Ww, taps=9, bias=b, bias2=temb, res=hs, out=hs, tiling=tiling)
    assert torch.equal(hs, sep)
    # resnet conv2 + 1x1 shortcut of the block input as a second K segment, into a sentinel-framed column slice
    xin = _rand(M, 2 * Cin, seed=15)
    ws = _rand(N, 2 * Cin, seed=16, s=(2 * Cin) ** -0.5)
    buf, out = _sentinel_out(M, N, lead=16, trail=8)
    ops.gemm(x, torch.cat([wc, ws], 1).contiguous(), N, B, Hh, Ww, taps=9, a1=xin, bias=b, out=out, tiling=tiling)
    r1, m1 = _conv3x3_ref(x, B, Hh, Ww, wc)
    r2, m2 = _linear_ref(xin, ws, (b,))
    check(out, r1 + r2, _gemm_bound(r1 + r2, m1 + m2), "conv + a1 shortcut")
    _assert_sentinels(buf, 16, N, "conv + a1 shortcut")
    relu = ops.gemm(x, wc, N, B, Hh, Ww, taps=9, bias=b, relu=True, tiling=tiling)
    r3, m3 = _conv3x3_ref(x, B, Hh, Ww, wc)
    r3 = r3 + b.to(D)
    check(relu, r3.clamp_min(0), _gemm_bound(r3, m3 + b.to(D).abs()), "conv + ReLU")
    _flag_clear()


def test_gemm_long_k():
    """The UNet's longest reductions: K = 23 040 (the 2 560-channel 3x3 conv of the up path, at 32 x 32) and K = 5 120
    (ff.out, with bias and the residual in place) -- the ACC term must hold there."""
    ops = _ops()
    B, Hh, Ww, C, N = 1, 32, 32, 2560, 1280
    x = _rand(B * Hh * Ww, C, seed=20)
    wc = _rand(N, 9 * C, seed=21, s=(9 * C) ** -0.5)
    b = _rand(N, seed=22)
    out = ops.gemm(x, wc, N, B, Hh, Ww, taps=9, bias=b, static_w=True)
    ref, mag = _conv3x3_ref(x, B, Hh, Ww, wc)
    ref, mag = ref + b.to(D), mag + b.to(D).abs()
    check(out, ref, _gemm_bound(ref, mag), "conv K=23040")
    M, K, N = 1024, 5120, 1280
    a, w, b = _rand(M, K, seed=23), _rand(N, K, seed=24, s=K ** -0.5), _rand(N, seed=25)
    hs = _rand(M, N, seed=26)
    ref, mag = _linear_ref(a, w, (b, hs))
    ops.gemm(a, w, N, 1, 1, M, bias=b, res=hs, out=hs)
    check(hs, ref, _gemm_bound(ref, mag), "linear K=5120 + residual in place")
    _flag_clear()


def test_gemm_n256_tile():
    """The 512-channel conv at 2 x 128 x 128 (K = 4 608, 512 M tiles): the cooperative 128 x 256 N tile."""
    ops = _ops()
    B, Hh, Ww, C = 2, 128, 128, 512
    x = _rand(B * Hh * Ww, C, seed=27)
    wc = _rand(C, 9 * C, seed=28, s=(9 * C) ** -0.5)
    b, res = _rand(C, seed=29), _rand(B * Hh * Ww, C, seed=30)
    out = ops.gemm(x, wc, C, B, Hh, Ww, taps=9, bias=b, res=res, static_w=True)
    ref, mag = _conv3x3_ref(x, B, Hh, Ww, wc)
    ref, mag = ref + b.to(D) + res.to(D), mag + b.to(D).abs() + res.to(D).abs()
    check(out, ref, _gemm_bound(ref, mag), "conv 512ch 2x128x128")
    _flag_clear()


def test_gemm_magnitude_edges():
    """Outputs near 3e4 (fp32 accumulators and the final rounding at the top of fp16's range) and outputs in the fp16
    subnormal range."""
    ops = _ops()
    M, K, N = 1000, 1280, 320
    a = _rand(M, K, seed=31, s=0.5, mean=2.0)
    w = _rand(N, K, seed=32, s=1.0).abs().float().mul(14.7).half()
    out = ops.gemm(a, w, N, 1, 1, M)
    ref, mag = _linear_ref(a, w)
    assert 2.5e4 < ref.max().item() < 6e4
    assert torch.isfinite(out).all()
    check(out, ref, _gemm_bound(ref, mag), "outputs near 3e4")
    a = _rand(M, K, seed=33, s=2.0 ** -4)
    w = _rand(N, K, seed=34, s=2.0 ** -12 * K ** -0.5)
    out = ops.gemm(a, w, N, 1, 1, M)
    ref, mag = _linear_ref(a, w)
    assert (ref.abs() < 2.0 ** -14).double().mean().item() > 0.5          # mostly subnormal outputs
    check(out, ref, _gemm_bound(ref, mag), "subnormal outputs")
    _flag_clear()


def _r16(t):
    return t.to(H).to(D)


@pytest.mark.parametrize("M,C", [(1000, 320), (2048, 1280)])
def test_gemm_geglu(M, C):
    """GEGLU against the reference's three fp16 rounding points emulated in fp64 (proj, gelu(gate), the product)."""
    ops = _ops()
    from latentblending_b200.unet import _geglu_perm
    inner = 4 * C
    a, w, b = _rand(M, C, seed=35), _rand(8 * C, C, seed=36, s=C ** -0.5), _rand(8 * C, seed=37)
    perm = _geglu_perm(inner, "cuda")
    out = ops.gemm(a, w[perm].contiguous(), 8 * C, 1, 1, M, bias=b[perm].contiguous(), mode=1)
    proj, mag = _linear_ref(a, w, (b,))
    v, g = proj[:, :inner], proj[:, inner:]
    mv, mg = mag[:, :inner], mag[:, inner:]
    vr, gr = _r16(v), _r16(g)
    ge = _r16(F.gelu(gr))
    ref = _r16(vr * ge)
    dv = ULP * vr.abs() + ACC * mv
    dge = ULP * ge.abs() + GELU_SLOPE * (ULP * gr.abs() + ACC * mg)
    bound = ULP * ref.abs() + ge.abs() * dv + vr.abs() * dge + dv * dge + TINY
    check(out, ref, bound, f"GEGLU M={M} C={C}")
    _flag_clear()


def _ln_ref(x, gamma, beta, eps):
    """fp64 LayerNorm rows of x -> (affine output, x_hat, mean, rstd)."""
    xd = x.to(D)
    mean = xd.mean(1, keepdim=True)
    rstd = 1.0 / torch.sqrt(((xd - mean) ** 2).mean(1, keepdim=True) + eps)
    xh = (xd - mean) * rstd
    return xh * gamma.to(D) + beta.to(D), xh, mean, rstd


def _norm_mag(x, mean, rstd, gamma, beta):
    return NORM * (rstd * gamma.to(D).abs() * (x.to(D).abs() + mean.abs()) + beta.to(D).abs())


# ---- attention -------------------------------------------------------------------------------------------------------
_Q0, _K0, _V0, _O0 = 8, 64, 24, 16          # column of head 0 in each buffer (nonzero, different)


def _attn_buffers(B, heads, Sq, Skv, scale, dist, seed):
    """q, k, v in three buffers with different row strides and column offsets, logits of the given distribution."""
    C = heads * 64
    k = _rand(B * Skv, heads, 64, seed=seed + 1).float()
    v = _rand(B * Skv, heads, 64, seed=seed + 2).float()
    if dist.startswith("std"):
        q = _rand(B * Sq, heads, 64, seed=seed, s=float(dist[3:]) / (scale * 8.0)).float()
    elif dist == "equal":
        q = torch.zeros(B * Sq, heads, 64, device="cuda")
    elif dist == "bigv":
        q = _rand(B * Sq, heads, 64, seed=seed, s=2.0 / (scale * 8.0)).float()
        v = v.clamp(-3, 3) * 1e4
    elif dist == "peaked":
        # one key per row with a +40 logit, in tile 0, a middle tile or the ragged last tile by row % 3
        nkv = (Skv + 127) // 128
        r = torch.arange(Sq, device="cuda")
        last0, mid = 128 * (nkv - 1), 128 * (nkv // 2)
        j = torch.where(r % 3 == 0, r % min(128, Skv),
                        torch.where(r % 3 == 1, mid + r % min(128, Skv - mid), last0 + r % (Skv - last0)))
        kk = k.view(B, Skv, heads, 64)[:, j]                                    # [B, Sq, heads, 64]
        c = 40.0 / (scale * (kk * kk).sum(-1, keepdim=True))
        q = _rand(B * Sq, heads, 64, seed=seed, s=1.0 / (scale * 8.0)).float() + (c * kk).reshape(B * Sq, heads, 64)
    else:
        raise ValueError(dist)
    qb = torch.zeros(B * Sq, C + 16, dtype=H, device="cuda")
    kb = torch.zeros(B * Skv, C + 128, dtype=H, device="cuda")
    vb = torch.zeros(B * Skv, C + 40, dtype=H, device="cuda")
    qb[:, _Q0:_Q0 + C] = q.reshape(B * Sq, C).half()
    kb[:, _K0:_K0 + C] = k.reshape(B * Skv, C).half()
    vb[:, _V0:_V0 + C] = v.reshape(B * Skv, C).half()
    return qb, kb, vb


def _attn_ref(qb, kb, vb, B, heads, Sq, Skv, scale):
    """fp64 softmax(q k^T scale) v per (batch, head) -> (ref, sum_j p_j |v_j|), [B*Sq, heads*64]."""
    C = heads * 64
    ref = torch.empty(B * Sq, C, dtype=D, device="cuda")
    mag = torch.empty_like(ref)
    sc = float(torch.tensor(scale, dtype=torch.float32))
    for b in range(B):
        rq, rk = slice(b * Sq, (b + 1) * Sq), slice(b * Skv, (b + 1) * Skv)
        for h in range(heads):
            q = qb[rq, _Q0 + 64 * h:_Q0 + 64 * h + 64].to(D)
            k = kb[rk, _K0 + 64 * h:_K0 + 64 * h + 64].to(D)
            v = vb[rk, _V0 + 64 * h:_V0 + 64 * h + 64].to(D)
            p = torch.softmax((q @ k.T) * sc, -1)
            ref[rq, 64 * h:64 * h + 64] = p @ v
            mag[rq, 64 * h:64 * h + 64] = p @ v.abs()
            del p
    return ref, mag


def _attn_run(qb, kb, vb, B, heads, Sq, Skv, scale):
    """Run into a column slice of a sentinel buffer with a sentinel row above and below -> (buf, out view)."""
    C = heads * 64
    buf = torch.full((B * Sq + 2, C + 40), SENTINEL, dtype=H, device="cuda")
    out = buf[1:1 + B * Sq, _O0:_O0 + C]
    _ops().attention(qb, kb, vb, out, B, heads, Sq, Skv, q_col0=_Q0, k_col0=_K0, v_col0=_V0, scale=scale)
    return buf, out


def _attn_bound(ref, mag):
    return ULP * ref.abs() + P_TERM * mag + TINY


_ATTN_CASES = [
    # B, heads, Sq, Skv, scale, logits
    (1, 1, 1, 1, 0.125, "std1"),
    (3, 5, 64, 2, 0.05, "std8"),
    (3, 10, 129, 77, 0.125, "std1"),
    (1, 20, 1000, 77, 0.125, "std8"),
    (1, 1, 64, 127, 1.0, "std30"),
    (3, 5, 129, 128, 0.125, "peaked"),
    (1, 10, 1000, 129, 0.05, "std30"),
    (3, 1, 1000, 255, 1.0, "peaked"),
    (1, 5, 129, 257, 0.125, "equal"),
    (3, 10, 64, 1024, 0.125, "peaked"),
    (1, 1, 4096, 1024, 0.125, "bigv"),
    (1, 10, 4096, 4096, 0.125, "std1"),
    (1, 5, 4096, 4096, 0.05, "peaked"),
    (1, 1, 1000, 4096, 1.0, "std8"),
    (3, 1, 129, 257, 1.0, "bigv"),
]


@pytest.mark.parametrize("B,heads,Sq,Skv,scale,dist", _ATTN_CASES)
def test_attention_bound(B, heads, Sq, Skv, scale, dist):
    """Fused attention against fp64 softmax attention of the same fp16 q / k / v: every element within its bound, and
    nothing written outside the output slice (rows above / below, columns beside).  With q = 0 the output is the mean
    of V."""
    qb, kb, vb = _attn_buffers(B, heads, Sq, Skv, scale, dist, seed=50 + Skv)
    buf, out = _attn_run(qb, kb, vb, B, heads, Sq, Skv, scale)
    ref, mag = _attn_ref(qb, kb, vb, B, heads, Sq, Skv, scale)
    if dist == "equal":
        C = heads * 64
        mean_v = vb[:, _V0:_V0 + C].to(D).view(B, Skv, C).mean(1)
        assert torch.allclose(ref.view(B, Sq, C), mean_v[:, None].expand(B, Sq, C), rtol=1e-12, atol=1e-12)
    check(out, ref, _attn_bound(ref, mag), f"attention B={B} heads={heads} Sq={Sq} Skv={Skv} scale={scale} {dist}")
    C = heads * 64
    assert bool((buf[0] == SENTINEL).all() and (buf[-1] == SENTINEL).all()), "a write outside the batch's rows"
    _assert_sentinels(buf[1:-1], _O0, C, "attention")
    _flag_clear()


@pytest.mark.parametrize("Skv", [257, 1000])
def test_attention_dropped_tile_is_rejected(Skv):
    """Non-vacuity: the kernel run with Skv cut to the previous multiple of 128 (the ragged last KV tile dropped)
    against the full reference."""
    B, heads, Sq, scale = 2, 2, 200, 0.125
    qb, kb, vb = _attn_buffers(B, heads, Sq, Skv, scale, "std1", seed=70)
    ref, mag = _attn_ref(qb, kb, vb, B, heads, Sq, Skv, scale)
    _, full = _attn_run(qb, kb, vb, B, heads, Sq, Skv, scale)
    check(full, ref, _attn_bound(ref, mag), "attention full")
    # the same buffers viewed as Skv - tail keys per batch: the first rows of each batch's keys
    short = Skv // 128 * 128
    kb2 = kb.view(B, Skv, -1)[:, :short].reshape(B * short, -1).contiguous()
    vb2 = vb.view(B, Skv, -1)[:, :short].reshape(B * short, -1).contiguous()
    _, cut = _attn_run(qb, kb2, vb2, B, heads, Sq, short, scale)
    reject(cut, ref, _attn_bound(ref, mag), f"attention Skv={Skv} without its ragged last KV tile")
    _flag_clear()


def test_attention_batch_and_head_invariance():
    """Bit for bit: a batch-1 call equals its rows of the batch-3 call, and a heads-1 call on one head's column slices
    equals that head of the heads-10 call (lockstep batching and the split CFG halves rely on this)."""
    ops = _ops()
    B, heads, Sq, Skv, scale = 3, 10, 129, 257, 0.125
    qb, kb, vb = _attn_buffers(B, heads, Sq, Skv, scale, "std8", seed=80)
    _, out3 = _attn_run(qb, kb, vb, B, heads, Sq, Skv, scale)
    for b in range(B):
        _, out1 = _attn_run(qb[b * Sq:(b + 1) * Sq], kb[b * Skv:(b + 1) * Skv], vb[b * Skv:(b + 1) * Skv], 1, heads, Sq,
                            Skv, scale)
        assert torch.equal(out1, out3[b * Sq:(b + 1) * Sq]), f"batch row block {b}"
    for h in (0, 7):
        o1 = torch.zeros(B * Sq, 64, dtype=H, device="cuda")
        ops.attention(qb, kb, vb, o1, B, 1, Sq, Skv, q_col0=_Q0 + 64 * h, k_col0=_K0 + 64 * h, v_col0=_V0 + 64 * h,
                      scale=scale)
        assert torch.equal(o1, out3[:, 64 * h:64 * h + 64]), f"head {h}"
    _flag_clear()


# ---- GroupNorm / LayerNorm -------------------------------------------------------------------------------------------
def _gn_ref(x, B, HW, C, groups, gamma, beta, eps):
    """fp64 GroupNorm of NHWC rows -> (affine output, x_hat, mean, rstd), each [B*HW, C]."""
    xd = x.to(D).reshape(B, HW, groups, C // groups)
    mean = xd.mean((1, 3), keepdim=True)
    rstd = 1.0 / torch.sqrt(((xd - mean) ** 2).mean((1, 3), keepdim=True) + eps)
    xh = (xd - mean) * rstd
    full = lambda t: t.expand(B, HW, groups, C // groups).reshape(B * HW, C)
    xh = xh.reshape(B * HW, C)
    return xh * gamma.to(D) + beta.to(D), xh, full(mean), full(rstd)


def _norm_bound(aff, mean, rstd, x, gamma, beta, silu, ulp=ULP):
    nm = _norm_mag(x, mean, rstd, gamma, beta)
    if not silu:
        return ulp * aff.abs() + nm + TINY
    return ulp * F.silu(aff).abs() + SILU_SLOPE * (ulp * aff.abs() + nm) + TINY


def _gn_run(x, B, HW, C, gamma, beta, eps, silu, dtype):
    buf, out = _sentinel_out(B * HW, C, lead=16, trail=8, dtype=dtype)
    _ops().groupnorm(x, B, HW, C, 32, gamma, beta, eps, silu, out=out)
    return buf, out


_GN_CASES = [
    # B, HW, C, mean/sigma, silu
    (1, 4096, 320, 0.0, 1),
    (2, 256, 64, 30.0, 1),
    (1, 1024, 640, 30.0, 0),
    (1, 1024, 640, 100.0, 0),
    (1, 4096, 320, 100.0, 1),
    (1, 1024, 640, 256.0, 0),
    (1, 4096, 320, 256.0, 1),
    (2, 35, 960, 256.0, 1),
    (1, 16384, 320, 30.0, 1),
    (1, 256, 2560, 100.0, 1),
    (3, 1, 1280, 30.0, 0),
    (1, 1024, 2560, 256.0, 0),
]


@pytest.mark.parametrize("B,HW,C,offset,silu", _GN_CASES)
def test_groupnorm_bound(B, HW, C, offset, silu):
    """fp16 GroupNorm(32) (+SiLU) of a row-strided input into a sentinel-framed column slice, with every group's mean
    offset by ``offset`` sigma; cpg 2 (C = 64) up to two trips of the channel loop (C = 2560), HW from 1 to 128^2."""
    ld = C + 24
    xb = _rand(B * HW, ld, seed=90 + C, mean=offset)
    x = xb[:, 8:8 + C]
    gamma, beta = _rand(C, seed=91, s=0.1, mean=1.0), _rand(C, seed=92, s=0.1)
    eps = 1e-5 if silu else 1e-6
    buf, out = _gn_run(x, B, HW, C, gamma, beta, eps, silu, H)
    aff, _, mean, rstd = _gn_ref(x, B, HW, C, 32, gamma, beta, eps)
    ref = F.silu(aff) if silu else aff
    check(out, ref, _norm_bound(aff, mean, rstd, x, gamma, beta, silu), f"GroupNorm B={B} HW={HW} C={C} "
          f"mean/sigma={offset} silu={silu}")
    _assert_sentinels(buf, 16, C, "GroupNorm")
    _flag_clear()


def test_groupnorm_rstd_error_is_rejected():
    """Non-vacuity: the fp64 reference with rstd scaled by 1 + 2^-9, rounded to fp16 like a kernel output."""
    B, HW, C, eps = 1, 1024, 640, 1e-6
    x = _rand(B * HW, C, seed=93, mean=3.0)
    gamma, beta = _rand(C, seed=94, s=0.1, mean=1.0), _rand(C, seed=95, s=0.1)
    aff, xh, mean, rstd = _gn_ref(x, B, HW, C, 32, gamma, beta, eps)
    bad = (xh * (1 + 2.0 ** -9) * gamma.to(D) + beta.to(D)).to(H)
    reject(bad, aff, _norm_bound(aff, mean, rstd, x, gamma, beta, 0), "GroupNorm with rstd * (1 + 2^-9)")


def test_groupnorm_batch_invariant():
    """B = 4 is bit-identical per image to B = 1 (the row-chunk grid depends on HW only)."""
    B, HW, C = 4, 1024, 640
    x = _rand(B * HW, C, seed=96, mean=30.0)
    gamma, beta = _rand(C, seed=97, s=0.1, mean=1.0), _rand(C, seed=98, s=0.1)
    _, o4 = _gn_run(x, B, HW, C, gamma, beta, 1e-5, 1, H)
    for b in range(B):
        _, o1 = _gn_run(x[b * HW:(b + 1) * HW], 1, HW, C, gamma, beta, 1e-5, 1, H)
        assert torch.equal(o1, o4[b * HW:(b + 1) * HW]), f"image {b}"
    _flag_clear()


@pytest.mark.parametrize("offset,silu", [(0.0, 1), (30.0, 0), (30.0, 1)])
def test_groupnorm_bf16_bound(offset, silu):
    """bf16 GroupNorm (the bf16 VAE decoder): the same bound with one bf16 ulp (2^-7) per rounding."""
    B, HW, C = 1, 4096, 512
    xb = _rand(B * HW, C + 8, seed=99, mean=offset, dtype=BF)
    x = xb[:, 8:]
    gamma, beta = _rand(C, seed=100, s=0.1, mean=1.0, dtype=BF), _rand(C, seed=101, s=0.1, dtype=BF)
    buf, out = _gn_run(x, B, HW, C, gamma, beta, 1e-6, silu, BF)
    aff, _, mean, rstd = _gn_ref(x, B, HW, C, 32, gamma, beta, 1e-6)
    ref = F.silu(aff) if silu else aff
    check(out, ref, _norm_bound(aff, mean, rstd, x, gamma, beta, silu, ulp=2.0 ** -7),
          f"bf16 GroupNorm mean/sigma={offset} silu={silu}")
    _assert_sentinels(buf, 16, C, "bf16 GroupNorm")
    _flag_clear()


@pytest.mark.parametrize("rows,C", [(77, 320), (1001, 1280), (4099, 2048)])
@pytest.mark.parametrize("offset", [0.0, 30.0, 100.0, 256.0])
def test_layernorm_bound(rows, C, offset):
    """LayerNorm (all three ln_kernel<MAXV> instantiations, row counts not a multiple of 8) of a row-strided input into
    a sentinel-framed column slice, row means offset by ``offset`` sigma.  Non-vacuity at offset 0: rstd * (1 + 2^-9)."""
    ops = _ops()
    xb = _rand(rows, C + 16, seed=110 + C, mean=offset)
    x = xb[:, 16:]
    gamma, beta = _rand(C, seed=111, s=0.1, mean=1.0), _rand(C, seed=112, s=0.1)
    buf, out = _sentinel_out(rows, C)
    ops.layernorm(x, gamma, beta, 1e-5, out=out)
    aff, xh, mean, rstd = _ln_ref(x, gamma, beta, 1e-5)
    bound = _norm_bound(aff, mean, rstd, x, gamma, beta, 0)
    check(out, aff, bound, f"LayerNorm rows={rows} C={C} mean/sigma={offset}")
    _assert_sentinels(buf, 8, C, "LayerNorm")
    if offset == 0.0:
        reject((xh * (1 + 2.0 ** -9) * gamma.to(D) + beta.to(D)).to(H), aff, bound, "LayerNorm with rstd * (1 + 2^-9)")
    _flag_clear()


# ---- boundary ops ----------------------------------------------------------------------------------------------------
def _all_values(dtype):
    """Every bit pattern of a 2-byte float type, as an NCHW image [1, 3, 256, 256]: in order in channel 0, reversed in
    channel 1, rotated in channel 2."""
    vals = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16).view(dtype)
    img = torch.stack([vals, vals.flip(0), vals.roll(12345)])
    return img.view(1, 3, 256, 256).cuda()


@pytest.mark.parametrize("dtype", [H, BF])
def test_postprocess_u8_every_value(dtype):
    """lb_postprocess_u8 on an image holding every fp16 (bf16) bit pattern.  fp16: diffusers' VaeImageProcessor chain
    run on the same fp16 tensor, (img / 2 + 0.5).clamp(0, 1) in fp16, then * 255 and round in fp32.  bf16 (an upcast
    VAE, decoded in fp32 by the reference): the fp32 chain.  Equal on every finite input; the non-finite count exact.
    Non-vacuity: one level added to one pixel is caught."""
    ops = _ops()
    img = _all_values(dtype)
    count = torch.zeros(1, dtype=torch.int32, device="cuda")
    got = ops.postprocess_u8(img, nonfinite=count)
    x = img if dtype == H else img.float()
    want = ((x / 2 + 0.5).clamp(0, 1).float() * 255).round().to(torch.uint8).permute(0, 2, 3, 1)
    finite = torch.isfinite(img).permute(0, 2, 3, 1)
    assert int(count.item()) == int((~torch.isfinite(img)).sum())
    diff = (got.int() - want.int()).abs() * finite
    n_bad = int((diff > 0).sum())
    assert n_bad == 0, (f"{dtype}: {n_bad} of {int(finite.sum())} finite values differ (max {int(diff.max())} "
                        f"levels); first at value {img.permute(0, 2, 3, 1)[diff > 0][0].item()!r}")
    bad = got.clone()
    bad.view(-1)[12345] += 1
    assert not torch.equal(bad[finite], want[finite])
    print(f"non-vacuity postprocess {dtype}: one level on one pixel rejected")
    _flag_clear()


@pytest.mark.parametrize("M", [1, 2, 3, 4, 5, 8, 9, 16])
def test_linear_small_bound(M):
    """linear_small, every MAXM instantiation and its tail: SiLU on the input (act_in), bias, SiLU on the output
    (act_out) and an addend, against the fp64 chain with one ulp per fp16 rounding the kernel makes."""
    ops = _ops()
    K, N = 1280, 203
    x = _rand(M, K, seed=120 + M)
    w, b = _rand(N, K, seed=121, s=K ** -0.5), _rand(N, seed=122)
    add = _rand(M, N + 5, seed=123)[:, :N]
    out = ops.linear_small(x, w, b, addend=add, act_in=1, act_out=1)
    xs = _r16(F.silu(x.to(D)))                    # the reference's fp16 F.silu
    r1, mag = _linear_ref(xs, w, (b,))
    r2 = F.silu(r1)
    ref = r2 + add.to(D)
    e1 = ULP * r1.abs() + ACC * mag + ULP * (xs.abs() @ w.to(D).abs().T)      # + one ulp of each SiLU input
    bound = ULP * ref.abs() + ULP * r2.abs() + SILU_SLOPE * e1 + TINY
    check(out, ref, bound, f"linear_small M={M} act_in act_out addend")
    plain = ops.linear_small(x, w)
    r0, m0 = _linear_ref(x, w)
    check(plain, r0, _gemm_bound(r0, m0), f"linear_small M={M} plain")
    _flag_clear()


@pytest.mark.parametrize("B,Hh,Ww", [(1, 1, 1), (2, 9, 7), (3, 13, 5)])
def test_conv_in_out_bound(B, Hh, Ww):
    """conv_in (4 -> 320, NCHW in) and conv_out (320 -> 4, NCHW out) at odd sizes against fp64 convolutions."""
    ops = _ops()
    C0 = 320
    x = _rand(B, 4, Hh, Ww, seed=130)
    w, b = _rand(C0, 4, 3, 3, seed=131, s=1 / 6), _rand(C0, seed=132)
    out = ops.conv_in(x, w.permute(2, 3, 1, 0).contiguous(), b, C0)
    ref = F.conv2d(x.to(D), w.to(D), b.to(D), padding=1).permute(0, 2, 3, 1).reshape(-1, C0)
    mag = F.conv2d(x.to(D).abs(), w.to(D).abs(), b.to(D).abs(), padding=1).permute(0, 2, 3, 1).reshape(-1, C0)
    check(out, ref, _gemm_bound(ref, mag), f"conv_in B={B} {Hh}x{Ww}")
    h = _rand(B * Hh * Ww, C0, seed=133)
    wo, bo = _rand(4, C0, 3, 3, seed=134, s=(9 * C0) ** -0.5), _rand(4, seed=135)
    eps = ops.conv_out(h, B, Hh, Ww, C0, wo.permute(0, 2, 3, 1).contiguous(), bo, 4)
    hn = h.to(D).view(B, Hh, Ww, C0).permute(0, 3, 1, 2)
    ref = F.conv2d(hn, wo.to(D), bo.to(D), padding=1)
    mag = F.conv2d(hn.abs(), wo.to(D).abs(), bo.to(D).abs(), padding=1)
    check(eps, ref, _gemm_bound(ref, mag), f"conv_out B={B} {Hh}x{Ww}")
    _flag_clear()


def _timestep_embedding32(t, dim):
    """diffusers get_timestep_embedding(t, dim, flip_sin_to_cos=True, downscale_freq_shift=0) in fp32, in its
    operation order."""
    half = dim // 2
    exponent = -math.log(10000) * torch.arange(0, half, dtype=torch.float32, device="cuda")
    exponent = exponent / half
    emb = torch.exp(exponent)
    emb = t[:, None].float() * emb[None, :]
    emb = torch.cat([torch.sin(emb), torch.cos(emb)], dim=-1)
    return torch.cat([emb[:, half:], emb[:, :half]], dim=-1)


@pytest.mark.parametrize("t", [0.0, 1.0, 499.5, 999.0])
def test_embed_inputs_bound(t):
    """embed_inputs: the timestep and time-id sinusoids within one fp16 ulp of the fp32 restatement (time ids up to
    4 096), the pooled text embedding copied exactly."""
    ops = _ops()
    B, dim_t, dim_a, pooled = 2, 320, 256, 1280
    text = _rand(B, pooled, seed=140)
    tids = torch.tensor([[1024., 1024, 0, 0, 1024, 1024], [4096, 3072, 37, 99, 1080, 1920]], device="cuda").half()
    temb, add = ops.embed_inputs(t, text, tids, dim_t, dim_a)
    ref_t = _timestep_embedding32(torch.full((B,), t, device="cuda"), dim_t).to(D)
    check(temb, ref_t, ULP * ref_t.abs() + TINY, f"timestep embedding t={t}")
    assert torch.equal(add[:, :pooled], text)
    ref_a = _timestep_embedding32(tids.reshape(-1), dim_a).reshape(B, -1).to(D)
    check(add[:, pooled:], ref_a, ULP * ref_a.abs() + TINY, "time-id embedding")
    _flag_clear()
