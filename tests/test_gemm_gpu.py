"""GPU numerics: the wgmma GEMM / implicit-GEMM conv kernel (lb_gemm) against a
plain PyTorch fp32 reference of the same op on the same fp16 inputs.
Tolerance: fp16 storage of an fp32-accumulated result -> |err| <= 2e-3*|ref|_max + small abs."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _close(out, ref, rtol=2e-3):
    out, ref = out.float(), ref.float()
    scale = ref.abs().max().item() + 1e-6
    err = (out - ref).abs().max().item()
    assert err <= rtol * scale + 1e-3, f"max err {err} vs scale {scale}"


def _rand(*shape, seed=0, s=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(*shape, generator=g, device="cuda") * s).half()


@pytest.mark.parametrize("M,N,K", [(128, 128, 64), (256, 160, 128), (2048, 1280, 1280), (154, 2560, 2048),
                                   (64, 64, 64), (8192, 640, 640), (300, 320, 192), (2048, 3840, 1280),
                                   (4096, 1920, 640), (32, 8, 64), (1024, 5120, 320)])
def test_linear(M, N, K):
    from latentblending_b200 import ops
    a, w, b = _rand(M, K, seed=1), _rand(N, K, seed=2, s=K ** -0.5), _rand(N, seed=3)
    out = ops.gemm(a, w, N, 1, 1, M, bias=b)
    _close(out, a.float() @ w.float().t() + b.float())
    assert ops.error_flag() == 0


def test_linear_residual_strided_io():
    from latentblending_b200 import ops
    M, N, K = 2048, 640, 640
    big = _rand(M, 2 * K, seed=4)
    a = big[:, K:]                                  # row stride 2K: zero-copy concat slices
    w, b = _rand(N, K, seed=5, s=K ** -0.5), _rand(N, seed=6)
    res = _rand(M, N, seed=7)
    outbuf = torch.zeros(M, 3 * N, dtype=torch.float16, device="cuda")
    out = outbuf[:, N:2 * N]
    ops.gemm(a, w, N, 1, 1, M, a0_c=K, bias=b, res=res, out=out)
    _close(out, a.float() @ w.float().t() + b.float() + res.float())
    assert outbuf[:, :N].abs().max() == 0 and outbuf[:, 2 * N:].abs().max() == 0


@pytest.mark.parametrize("B,H,W,Cin,Cout", [(2, 128, 128, 64, 320), (2, 64, 64, 320, 640), (2, 32, 32, 640, 1280),
                                            (1, 16, 16, 128, 128), (2, 8, 8, 64, 64), (4, 4, 4, 64, 128),
                                            (1, 2, 2, 64, 64), (1, 64, 64, 960, 320), (2, 256, 128, 64, 64)])
def test_conv3x3(B, H, W, Cin, Cout):
    from latentblending_b200 import ops
    x = _rand(B, H, W, Cin, seed=8)                                  # NHWC
    w = _rand(Cout, Cin, 3, 3, seed=9, s=(9 * Cin) ** -0.5)
    b = _rand(Cout, seed=10)
    temb = _rand(B, Cout, seed=11)
    wp = w.permute(0, 2, 3, 1).reshape(Cout, 9 * Cin).contiguous()  # [N][ky][kx][c]
    out = ops.gemm(x.view(B * H * W, Cin), wp, Cout, B, H, W, taps=9, bias=b, bias2=temb)
    ref = F.conv2d(x.permute(0, 3, 1, 2).float(), w.float(), b.float(), padding=1) + temb.float()[:, :, None, None]
    _close(out.view(B, H, W, Cout), ref.permute(0, 2, 3, 1))
    assert ops.error_flag() == 0


def test_conv3x3_with_fused_shortcut_and_residual():
    from latentblending_b200 import ops
    B, H, W, Cin, Cout = 2, 32, 32, 128, 256
    xin = _rand(B, H, W, Cin, seed=12)        # raw resnet input (shortcut operand)
    h = _rand(B, H, W, Cout, seed=13)         # conv2 input
    w2 = _rand(Cout, Cout, 3, 3, seed=14, s=(9 * Cout) ** -0.5)
    ws = _rand(Cout, Cin, 1, 1, seed=15, s=Cin ** -0.5)
    b = _rand(Cout, seed=16)
    wp = torch.cat([w2.permute(0, 2, 3, 1).reshape(Cout, 9 * Cout), ws.reshape(Cout, Cin)], dim=1).contiguous()
    out = ops.gemm(h.view(-1, Cout), wp, Cout, B, H, W, taps=9, a1=xin.view(-1, Cin), bias=b)
    ref = F.conv2d(h.permute(0, 3, 1, 2).float(), w2.float(), b.float(), padding=1) + \
        F.conv2d(xin.permute(0, 3, 1, 2).float(), ws.float())
    _close(out.view(B, H, W, Cout), ref.permute(0, 2, 3, 1))


@pytest.mark.parametrize("M,C", [(2048, 1280), (8192, 640), (256, 128)])
def test_geglu(M, C):
    from latentblending_b200 import ops
    a = _rand(M, C, seed=17)
    w = _rand(8 * C, C, seed=18, s=C ** -0.5)
    b = _rand(8 * C, seed=19)
    inner = 4 * C
    # host-side tile interleave: per 128-row tile, 64 value rows then the matching 64 gate rows
    idx = torch.arange(inner, device="cuda").view(-1, 64)
    perm = torch.stack([idx, idx + inner], dim=1).reshape(-1)
    out = ops.gemm(a, w[perm].contiguous(), 8 * C, 1, 1, M, bias=b[perm].contiguous(), mode=1)
    proj = (a.float() @ w.float().t() + b.float()).half().float()
    ref = proj[:, :inner] * F.gelu(proj[:, inner:]).half().float()
    _close(out, ref)
