"""GPU checks of the GEMM kernel's persistent ping-pong schedule and its epilogue: in-place residuals, tile counts that
give a CTA one or an odd number of tiles, pixel-box conv tiles that span several images, GEGLU at its N tile, and
batch invariance (the rows of a small launch are bit-identical to the same rows inside a larger launch, which the
lockstep speculation and the dual-stream path rely on)."""
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


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.parametrize("M,N,K", [(2048, 1280, 1280), (4096, 1280, 5120), (300, 640, 640)])
def test_linear_residual_in_place(M, N, K):
    """out = a w^T + b + hs written over hs itself (the UNet's attn / ff output projections)."""
    from latentblending_b200 import ops
    a, w, b = _rand(M, K, seed=1), _rand(N, K, seed=2, s=K ** -0.5), _rand(N, seed=3)
    hs = _rand(M, N, seed=4)
    ref = a.float() @ w.float().t() + b.float() + hs.float()
    separate = ops.gemm(a, w, N, 1, 1, M, bias=b, res=hs.clone())
    ops.gemm(a, w, N, 1, 1, M, bias=b, res=hs, out=hs)
    _close(hs, ref)
    assert torch.equal(hs, separate)
    assert ops.error_flag() == 0


@pytest.mark.parametrize("tiles_per_cta", ["one", "odd", "one_extra", "odd_ragged"])
def test_linear_tile_counts(tiles_per_cta):
    """N = 160 * k: every tile is 128 x 160; the persistent grid is min(tiles, SMs)."""
    from latentblending_b200 import ops
    sms = _sms()
    tiles_m, tiles_n = {"one": (1, 1), "odd": (sms, 3), "one_extra": (sms + 1, 1), "odd_ragged": (2 * sms + 5, 1)}[
        tiles_per_cta]
    M, N, K = 128 * tiles_m - (37 if tiles_per_cta == "odd_ragged" else 0), 160 * tiles_n, 320
    a, w, b = _rand(M, K, seed=5), _rand(N, K, seed=6, s=K ** -0.5), _rand(N, seed=7)
    res = _rand(M, N, seed=8)
    out = ops.gemm(a, w, N, 1, 1, M, bias=b, res=res)
    _close(out, a.float() @ w.float().t() + b.float() + res.float())
    assert ops.error_flag() == 0


@pytest.mark.parametrize("B,H,W,Cin,Cout", [(4, 8, 8, 64, 128), (8, 4, 4, 128, 320), (3, 8, 8, 64, 64)])
def test_conv3x3_residual_multi_image_tiles(B, H, W, Cin, Cout):
    """H * W < 128: one 128-row tile is a box of several images (tb > 1), with time-embedding bias and residual."""
    from latentblending_b200 import ops
    x = _rand(B, H, W, Cin, seed=9)
    w = _rand(Cout, Cin, 3, 3, seed=10, s=(9 * Cin) ** -0.5)
    b, temb = _rand(Cout, seed=11), _rand(B, Cout, seed=12)
    res = _rand(B * H * W, Cout, seed=13)
    wp = w.permute(0, 2, 3, 1).reshape(Cout, 9 * Cin).contiguous()
    out = ops.gemm(x.view(B * H * W, Cin), wp, Cout, B, H, W, taps=9, bias=b, bias2=temb, res=res)
    ref = F.conv2d(x.permute(0, 3, 1, 2).float(), w.float(), b.float(), padding=1) + temb.float()[:, :, None, None]
    ref = ref.permute(0, 2, 3, 1).reshape(B * H * W, Cout) + res.float()
    _close(out, ref)
    assert ops.error_flag() == 0


@pytest.mark.parametrize("M,C", [(4096, 1280), (1024, 1280), (16384, 640)])
def test_geglu_bench_shapes(M, C):
    """GEGLU at the 32^2 / 64^2 transformer widths and batch-1 / batch-4 row counts (weights interleaved per
    128-column tile, as unet.PackedUNet packs them)."""
    from latentblending_b200 import ops
    from latentblending_b200.unet import _geglu_perm
    a = _rand(M, C, seed=14)
    w = _rand(8 * C, C, seed=15, s=C ** -0.5)
    b = _rand(8 * C, seed=16)
    inner = 4 * C
    perm = _geglu_perm(inner, "cuda")
    out = ops.gemm(a, w[perm].contiguous(), 8 * C, 1, 1, M, bias=b[perm].contiguous(), mode=1)
    proj = (a.float() @ w.float().t() + b.float()).half().float()
    ref = proj[:, :inner] * F.gelu(proj[:, inner:]).half().float()
    _close(out, ref)
    assert ops.error_flag() == 0


def test_batch_invariance():
    """The rows of a batch-1 launch are bit-identical to the same rows of a batch-4 launch, for every epilogue the
    UNet uses at 32^2 (linear + residual, GEGLU, 3x3 conv + time embedding + residual)."""
    from latentblending_b200 import ops
    from latentblending_b200.unet import _geglu_perm
    HW, C = 32, 1280
    S = HW * HW
    x4 = _rand(4 * S, C, seed=17)
    res4 = _rand(4 * S, C, seed=18)
    b = _rand(C, seed=19)
    # linear + residual (attn1.out) and ff.out-like K
    for K, seed in ((C, 20), (4 * C, 21)):
        a4 = _rand(4 * S, K, seed=seed)
        w = _rand(C, K, seed=seed + 10, s=K ** -0.5)
        o4 = ops.gemm(a4, w, C, 1, 1, 4 * S, bias=b, res=res4)
        for i in range(4):
            o1 = ops.gemm(a4[i * S:(i + 1) * S], w, C, 1, 1, S, bias=b, res=res4[i * S:(i + 1) * S])
            assert torch.equal(o1, o4[i * S:(i + 1) * S]), f"linear K={K} image {i}"
    # GEGLU
    wg = _rand(8 * C, C, seed=22, s=C ** -0.5)
    perm = _geglu_perm(4 * C, "cuda")
    wg, bg = wg[perm].contiguous(), _rand(8 * C, seed=23)[perm].contiguous()
    g4 = ops.gemm(x4, wg, 8 * C, 1, 1, 4 * S, bias=bg, mode=1)
    for i in range(4):
        g1 = ops.gemm(x4[i * S:(i + 1) * S], wg, 8 * C, 1, 1, S, bias=bg, mode=1)
        assert torch.equal(g1, g4[i * S:(i + 1) * S]), f"GEGLU image {i}"
    # 3x3 conv + time embedding + residual (resnet conv2)
    wc = _rand(C, 9 * C, seed=24, s=(9 * C) ** -0.5)
    temb = _rand(4, C, seed=25)
    c4 = ops.gemm(x4, wc, C, 4, HW, HW, taps=9, bias=b, bias2=temb, res=res4)
    for i in range(4):
        c1 = ops.gemm(x4[i * S:(i + 1) * S], wc, C, 1, HW, HW, taps=9, bias=b, bias2=temb[i:i + 1],
                      res=res4[i * S:(i + 1) * S])
        assert torch.equal(c1, c4[i * S:(i + 1) * S]), f"conv image {i}"
    assert ops.error_flag() == 0


def test_conv3x3_n256_tiles():
    """A long-K, many-tile convolution at 512 channels (the VAE decoder's shape class), which runs the 128 x 256
    tile, with residual."""
    from latentblending_b200 import ops
    B, H, W, C = 2, 128, 128, 512
    x = _rand(B, H, W, C, seed=26)
    w = _rand(C, C, 3, 3, seed=27, s=(9 * C) ** -0.5)
    b = _rand(C, seed=28)
    res = _rand(B * H * W, C, seed=29)
    wp = w.permute(0, 2, 3, 1).reshape(C, 9 * C).contiguous()
    out = ops.gemm(x.view(B * H * W, C), wp, C, B, H, W, taps=9, bias=b, res=res, static_w=True)
    ref = F.conv2d(x.permute(0, 3, 1, 2).float(), w.float(), b.float(), padding=1)
    _close(out, ref.permute(0, 2, 3, 1).reshape(B * H * W, C) + res.float())
    assert ops.error_flag() == 0
