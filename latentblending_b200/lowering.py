"""Weight packing and lowering pieces the UNet (unet.py) and the KL VAE decoder (vae.py) share: the 3x3 conv
weight layout, the resnet block (GroupNorm + SiLU, conv1, GroupNorm + SiLU, conv2 with the shortcut or the residual),
the output convolution and the scratch buffers of a lowering."""
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
