"""Weight packing and lowering pieces the UNet (unet.py) and the KL VAE decoder and encoder (vae.py) share: the 3x3
conv weight layout, the resnet block (GroupNorm + SiLU, conv1, GroupNorm + SiLU, conv2 with the shortcut or the
residual), the VAE mid-block attention, the output convolution and the scratch buffers of a lowering."""
import torch


def pack3(w):
    """[N, Ci, 3, 3] conv weights -> the GEMM's [N][ky][kx][Ci] rows."""
    return w.permute(0, 2, 3, 1).reshape(w.shape[0], -1).contiguous()


def pack_resnet(W, r, sd, g):
    """The parameters of resnet ``r`` (a diffusers ResnetBlock2D's state_dict prefix) into ``W``: norm1 / norm2,
    conv1, and conv2 with the 1x1 shortcut conv (when ``sd`` has one) appended along K and its bias added to conv2's.
    ``g(name)``: the state_dict tensor in the storage type (fp16 or bf16).  The two biases are added in fp32 and
    rounded once: in fp16 their fp16-rounded values, in bf16 the state dict's own values."""
    W[r + ".norm1.g"], W[r + ".norm1.b"] = g(r + ".norm1.weight"), g(r + ".norm1.bias")
    W[r + ".norm2.g"], W[r + ".norm2.b"] = g(r + ".norm2.weight"), g(r + ".norm2.bias")
    W[r + ".conv1.w"], W[r + ".conv1.b"] = pack3(g(r + ".conv1.weight")), g(r + ".conv1.bias")
    w2, b2 = pack3(g(r + ".conv2.weight")), g(r + ".conv2.bias")
    if (r + ".conv_shortcut.weight") in sd:
        ws = g(r + ".conv_shortcut.weight")
        w2 = torch.cat([w2, ws.reshape(ws.shape[0], -1)], 1).contiguous()
        if b2.dtype == torch.float16:
            f32 = lambda n: g(n).float()
        else:
            f32 = lambda n: sd[n].detach().to(device=b2.device, dtype=torch.float32)
        b2 = (f32(r + ".conv2.bias") + f32(r + ".conv_shortcut.bias")).to(b2.dtype)
        W[r + ".has_shortcut"] = True
    W[r + ".conv2.w"], W[r + ".conv2.b"] = w2, b2


class Scratch:
    """Named scratch buffers of one lowering: ``scratch(name, rows, cols)`` is a [rows, cols] view of the buffer
    ``name``, reallocated when a larger view is asked for (the ops recorded earlier hold the old one)."""

    def __init__(self, dtype, device):
        self.dtype, self.device = dtype, device
        self.bufs = {}

    def __call__(self, name, rows, cols):
        need = rows * cols
        buf = self.bufs.get(name)
        if buf is None or buf.numel() < need:
            buf = torch.empty(need, dtype=self.dtype, device=self.device)
            self.bufs[name] = buf
        return buf[:need].view(rows, cols)


def lower_resnet(P, W, r, x, cin, cout, B, h, w, out, groups, eps, ws, scratch, bias2=None):
    """Resnet ``r`` (packed by ``pack_resnet``) on the NHWC map ``x`` [B*h*w, cin] into ``out`` [B*h*w, cout]:
    GroupNorm(eps) + SiLU, conv1 (+ ``bias2``, the UNet's per-image time-embedding projection), GroupNorm(eps) + SiLU,
    conv2 with the shortcut conv of ``x`` as a second K segment, or with ``x`` as the residual."""
    M = B * h * w
    n1 = scratch("n1", M, cin)
    P.groupnorm(x, B, h * w, cin, groups, W[r + ".norm1.g"], W[r + ".norm1.b"], eps, 1, n1, ws)
    h1 = scratch("h1", M, cout)
    P.gemm(n1, W[r + ".conv1.w"], cout, B, h, w, h1, taps=9, bias=W[r + ".conv1.b"], bias2=bias2)
    n2 = scratch("n2", M, cout)
    P.groupnorm(h1, B, h * w, cout, groups, W[r + ".norm2.g"], W[r + ".norm2.b"], eps, 1, n2, ws)
    if W.get(r + ".has_shortcut"):
        P.gemm(n2, W[r + ".conv2.w"], cout, B, h, w, out, taps=9, a1=x, a1_c=cin, bias=W[r + ".conv2.b"])
    else:
        P.gemm(n2, W[r + ".conv2.w"], cout, B, h, w, out, taps=9, bias=W[r + ".conv2.b"], res=x)


def lower_conv_out(P, W, x, B, h, w, cin, cout, out_nchw, scratch):
    """The 3x3 output convolution cin -> cout of ``x`` into NCHW ``out_nchw``: the N = 8 GEMM
    (``W['conv_out.w8']``, ``pack_conv_out8``) then NCHW.  The GEMM's [B*h*w, 8] output reuses the "h1" scratch."""
    P.conv_out_gemm(x, B, h, w, cin, W["conv_out.w8"], W["conv_out.b8"], cout, out_nchw, scratch("h1", B * h * w, 8))


def pack_vae_attention(W, a, sd, g, gf, dtype):
    """The VAE mid-block single-head attention ``a`` (its state_dict prefix) into ``W``: 1/sqrt(C) folded into Wq, Wq
    and Wk stacked into one projection, the value bias folded into the output bias (softmax rows sum to one).
    ``g`` / ``gf``: the state_dict tensor in the storage type / in fp32."""
    Cm = sd[a + ".to_q.weight"].shape[0]
    scale = Cm ** -0.5
    W["attn.norm.g"], W["attn.norm.b"] = g(a + ".group_norm.weight"), g(a + ".group_norm.bias")
    W["attn.qk.w"] = torch.cat([(gf(a + ".to_q.weight") * scale), gf(a + ".to_k.weight")], 0).to(dtype).contiguous()
    W["attn.qk.b"] = torch.cat([(gf(a + ".to_q.bias") * scale), gf(a + ".to_k.bias")], 0).to(dtype).contiguous()
    W["attn.v.w"] = g(a + ".to_v.weight")
    W["attn.out.w"] = g(a + ".to_out.0.weight")
    W["attn.out.b"] = (gf(a + ".to_out.0.bias") + gf(a + ".to_out.0.weight") @ gf(a + ".to_v.bias")).to(dtype).contiguous()


def lower_vae_attention(P, W, x, S, C0, groups, ws, scratch, out):
    """The VAE mid-block attention (packed by ``pack_vae_attention``; single head, dim C0) of the NHWC map ``x``
    [S, C0] into ``out`` [S, C0], x added as the residual: three GEMMs around a row softmax.  Activations are of
    ``scratch``'s type (fp16 or bf16); the scores are fp16 either way."""
    B, act, dev = 1, scratch.dtype, scratch.device
    # V^T and the scores take the keys as the GEMM's N, which must be a multiple of 8: hn and qk get S8 >= S rows,
    # the extra ones zero (never written), so the extra V^T and score columns are exact zeros
    S8 = -(-S // 8) * 8
    hn = torch.zeros(S8, C0, dtype=act, device=dev)
    P.groupnorm(x, B, S, C0, groups, W["attn.norm.g"], W["attn.norm.b"], 1e-6, 0, hn, ws)
    qk = torch.zeros(S8, 2 * C0, dtype=act, device=dev)
    P.gemm(hn, W["attn.qk.w"], 2 * C0, 1, 1, S, qk, bias=W["attn.qk.b"])
    # P V contracts over the S keys, and the GEMM's K must be a multiple of 64: P and V^T get Sp >= S8 columns, the
    # extra ones zero, which adds exact zeros to every dot product
    Sp = -(-S // 64) * 64
    vT = torch.zeros(C0, Sp, dtype=act, device=dev)
    P.gemm(W["attn.v.w"], hn, S8, 1, 1, C0, vT[:, :S8], static_w=False)             # V^T = Wv hn^T
    scores = torch.zeros(S, Sp, dtype=torch.float16, device=dev)
    # bf16: the scores are stored in fp16 (LB_GEMM_OUT_F16), whose rounding is 8x finer than bf16's -- the error of
    # a score s becomes an exp(s) error -- and whose range their modest magnitudes do not approach; the softmax
    # writes the bf16 P over them (same 2-byte slots), which P V reads as a bf16 operand
    P.gemm(qk[:, :C0], qk[:, C0:], S8, 1, 1, S, scores[:, :S8], static_w=False)      # (scaled q) k^T
    probs = scores.view(act)
    P.softmax_rows(scores[:, :S], probs[:, :S])
    att = scratch("h1", S, C0)
    P.gemm(probs, vT, C0, 1, 1, S, att, static_w=False)                               # P V
    P.gemm(att, W["attn.out.w"], C0, 1, 1, S, out, bias=W["attn.out.b"], res=x)
