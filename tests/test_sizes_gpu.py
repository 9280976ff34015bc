"""GPU checks of non-square and non-power-of-two output sizes: the GEMM's pixel-run M tiling (TMA im2col loads), its
agreement with the pixel-box tiling, and every layer above it (UNet, VAE, LPIPS, engine) at sizes the box cannot
tile.  Tolerances are the ones the square-size tests use, stated at each assert."""
import dataclasses
import json
import os

import numpy as np
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


def _conv_ref(x, w, b=None, temb=None, res=None, sc=None, wsc=None):
    """fp32 reference of the resnet conv2 epilogue: conv3x3(x) + b + temb[b] (+ 1x1 shortcut sc) (+ res), NHWC rows."""
    B, H, W, _ = x.shape
    ref = F.conv2d(x.permute(0, 3, 1, 2).float(), w.float(), None if b is None else b.float(), padding=1)
    if temb is not None:
        ref = ref + temb.float()[:, :, None, None]
    if sc is not None:
        ref = ref + F.conv2d(sc.permute(0, 3, 1, 2).float(), wsc.float()[:, :, None, None])
    ref = ref.permute(0, 2, 3, 1).reshape(B * H * W, -1)
    return ref if res is None else ref + res.float()


def _pack(w):
    return w.permute(0, 2, 3, 1).reshape(w.shape[0], -1).contiguous()


# ---- 1. im2col semantics ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tap", range(9))
def test_runs_tap_semantics(tap):
    """One 3x3 tap at a time on a 2 x 3 x 5 image batch (tiles span rows and images, 30 of 128 rows used): pins the
    pixel bounding box and the im2col offset of each tap against F.conv2d."""
    from latentblending_b200 import ops
    B, H, W, C, N = 2, 3, 5, 64, 64
    x = _rand(B, H, W, C, seed=1)
    w = torch.zeros(N, C, 3, 3, dtype=torch.float16, device="cuda")
    w[:, :, tap // 3, tap % 3] = _rand(N, C, seed=2, s=C ** -0.5)
    out = ops.gemm(x.view(B * H * W, C), _pack(w), N, B, H, W, taps=9, tiling="runs")
    _close(out, _conv_ref(x, w))
    assert ops.error_flag() == 0


@pytest.mark.parametrize("W", [104, 76, 52, 38, 26, 19, 5, 1, 152])
@pytest.mark.parametrize("B", [1, 2, 4])
def test_runs_conv_epilogues(W, B):
    """Pixel-run 3x3 convs at the SDXL bucket widths with bias, per-image time-embedding bias, the fused 1x1 shortcut
    (a1) and an in-place residual; several images share a tile wherever H*W is not a multiple of 128."""
    from latentblending_b200 import ops
    H = {104: 13, 76: 9, 52: 7, 38: 6, 26: 5, 19: 3, 5: 3, 1: 7, 152: 3}[W]
    Cin, Csc, N = 128, 64, 192
    x = _rand(B, H, W, Cin, seed=3)
    sc = _rand(B, H, W, Csc, seed=4)
    w = _rand(N, Cin, 3, 3, seed=5, s=(9 * Cin) ** -0.5)
    wsc = _rand(N, Csc, seed=6, s=Csc ** -0.5)
    b, temb = _rand(N, seed=7), _rand(B, N, seed=8)
    res = _rand(B * H * W, N, seed=9)
    ref = _conv_ref(x, w, b, temb, res, sc, wsc)
    wcat = torch.cat([_pack(w), wsc], 1).contiguous()
    out = ops.gemm(x.view(-1, Cin), wcat, N, B, H, W, taps=9, a1=sc.view(-1, Csc), bias=b, bias2=temb,
                   res=res, out=res, tiling="runs")
    _close(out, ref)
    # the automatic choice takes the runs wherever the box cannot tile these shapes, with the same bits
    auto = ops.gemm(x.view(-1, Cin), wcat, N, B, H, W, taps=9, a1=sc.view(-1, Csc), bias=b, bias2=temb,
                    tiling="auto")
    plain = ops.gemm(x.view(-1, Cin), wcat, N, B, H, W, taps=9, a1=sc.view(-1, Csc), bias=b, bias2=temb,
                     tiling="runs")
    assert torch.equal(auto, plain)
    assert ops.error_flag() == 0


def test_runs_1x1_conv_over_images():
    """taps = 1 with B*H > 1: a pointwise conv (proj_in / shortcut shape class) as pixel runs."""
    from latentblending_b200 import ops
    B, H, W, C, N = 3, 11, 19, 320, 640
    x = _rand(B * H * W, C, seed=10)
    w = _rand(N, C, seed=11, s=C ** -0.5)
    b, temb = _rand(N, seed=12), _rand(B, N, seed=13)
    out = ops.gemm(x, w, N, B, H, W, bias=b, bias2=temb, tiling="runs")
    ref = x.float() @ w.float().t() + b.float() + temb.float().repeat_interleave(H * W, 0)
    _close(out, ref)


def test_tiling_flags():
    from latentblending_b200 import _cabi, ops
    x = _rand(2 * 6 * 20, 64, seed=14)
    w = _rand(64, 9 * 64, seed=15)
    with pytest.raises(_cabi.LB200Error, match="cannot tile"):
        ops.gemm(x, w, 64, 2, 6, 20, taps=9, tiling="box")       # W = 20 < 128 is not a power of two
    with pytest.raises(_cabi.LB200Error, match="exclude"):
        ops.gemm(x, w, 64, 2, 6, 20, taps=9, mode=_cabi.GEMM_TILE_BOX | _cabi.GEMM_TILE_RUNS)
    with pytest.raises(ValueError):
        ops.gemm(x, w, 64, 2, 6, 20, taps=9, tiling="pixels")


# ---- 2. box and runs agree bit for bit ----------------------------------------------------------------------------
@pytest.mark.parametrize("B,H,W,C,N", [(2, 104, 152, 320, 320),      # ragged box tiles (W = 152), bucket level 0
                                       (2, 32, 32, 640, 640),        # power of two: a tie
                                       (4, 64, 128, 512, 512),       # BN = 256 cooperative tile
                                       (3, 8, 8, 64, 128)])          # several images per box tile
def test_box_and_runs_conv_bit_identical(B, H, W, C, N):
    from latentblending_b200 import ops
    x = _rand(B * H * W, C, seed=16)
    w = _rand(N, 9 * C, seed=17, s=(9 * C) ** -0.5)
    b, temb, res = _rand(N, seed=18), _rand(B, N, seed=19), _rand(B * H * W, N, seed=20)
    outs = [ops.gemm(x, w, N, B, H, W, taps=9, bias=b, bias2=temb, res=res, static_w=True, tiling=t)
            for t in ("box", "runs")]
    assert torch.equal(outs[0], outs[1])
    assert ops.error_flag() == 0


def test_box_and_runs_geglu_bit_identical():
    from latentblending_b200 import ops
    from latentblending_b200.unet import _geglu_perm
    M, C = 2 * 76 * 52, 640            # bucket level 1 rows, as a plain matrix
    a = _rand(M, C, seed=21)
    wg = _rand(8 * C, C, seed=22, s=C ** -0.5)
    perm = _geglu_perm(4 * C, "cuda")
    wg, bg = wg[perm].contiguous(), _rand(8 * C, seed=23)[perm].contiguous()
    g = [ops.gemm(a, wg, 8 * C, 1, 1, M, bias=bg, mode=1, tiling=t) for t in ("box", "runs")]
    g += [ops.gemm(a, wg, 8 * C, 2, 52, 76, bias=bg, mode=1, tiling=t) for t in ("auto", "runs")]
    assert all(torch.equal(g[0], o) for o in g[1:])
    assert ops.error_flag() == 0


# ---- 3. batch invariance under runs -------------------------------------------------------------------------------
def test_runs_batch_invariance():
    """The rows of a batch-1 launch equal the same image inside a batch-4 launch bit for bit (tiles of the batch-4
    launch start mid-image) -- what lockstep speculation and the dual-stream path rely on."""
    from latentblending_b200 import ops
    H, W, C = 38, 26, 640
    S = H * W
    x4, res4 = _rand(4 * S, C, seed=28), _rand(4 * S, C, seed=29)
    wc = _rand(C, 9 * C, seed=30, s=(9 * C) ** -0.5)
    b, temb = _rand(C, seed=31), _rand(4, C, seed=32)
    c4 = ops.gemm(x4, wc, C, 4, H, W, taps=9, bias=b, bias2=temb, res=res4)
    for i in range(4):
        c1 = ops.gemm(x4[i * S:(i + 1) * S], wc, C, 1, H, W, taps=9, bias=b, bias2=temb[i:i + 1],
                      res=res4[i * S:(i + 1) * S])
        assert torch.equal(c1, c4[i * S:(i + 1) * S]), f"conv image {i}"
    assert ops.error_flag() == 0


# ---- 4. UNet ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,h,w", [(2, 12, 20), (2, 20, 12), (1, 36, 28)])
def test_tiny_unet_non_square(B, h, w):
    from oracle.sdxl_unet import tiny_config
    from test_unet_gpu import _run_pair
    rel, eps, _, _ = _run_pair(tiny_config(), B, h, w, 611.0)
    assert torch.isfinite(eps).all() and eps.shape == (B, 4, h, w)
    assert rel <= 2e-3, f"relative L2 error {rel}"


@pytest.mark.parametrize("h,w", [(20, 12), (36, 28)])
def test_medium_unet_non_square(h, w):
    from oracle.sdxl_unet import UNetConfig
    from test_unet_gpu import _run_pair
    ocfg = UNetConfig(block_out_channels=(128, 256, 512), transformer_layers=(0, 2, 10), cross_attention_dim=256,
                      addition_time_embed_dim=64, pooled_dim=128, sample_size=32)
    rel, eps, _, _ = _run_pair(ocfg, 2, h, w, 499.0)
    assert torch.isfinite(eps).all()
    assert rel <= 2e-3, f"relative L2 error {rel}"


@pytest.mark.slow
def test_full_sdxl_unet_matches_fixture_at_portrait_bucket():
    """Full SDXL-base UNet, CFG batch 2, at the 832x1216 bucket (latent 152 x 104) vs the fp32 oracle fixture; each
    CFG half alone is bit-identical to its half of the batch-2 forward."""
    from latentblending_b200 import ops
    from make_bucket_fixtures import UNET_BUCKET_FIXTURE, UNET_BUCKET_HW, UNET_SEED, unet_inputs
    from oracle.sdxl_unet import SDXL_BASE
    from test_unet_gpu import _full_sdxl
    fx = np.load(UNET_BUCKET_FIXTURE)
    full = _full_sdxl()
    assert full["sha"] == str(fx["weights_sha1"]), "seeded weight recipe drifted from the fixture's"
    h, w = UNET_BUCKET_HW
    x, ctx, pooled, tids = unet_inputs(SDXL_BASE, 2, h, w, UNET_SEED)
    eps = full["net"].forward(x.cuda(), float(fx["t"]), ctx.cuda(), pooled.cuda(), tids.cuda()).float().cpu()
    torch.cuda.synchronize()
    assert ops.error_flag() == 0
    ref = torch.from_numpy(fx["eps"])
    assert eps.shape == ref.shape == (2, 4, h, w)
    rel = ((eps - ref).norm() / ref.norm()).item()
    print(f"full SDXL UNet @{h}x{w} B=2: rel_l2={rel:.3e}")
    assert torch.isfinite(eps).all()
    assert rel <= 2e-3, f"relative L2 error {rel}"
    for b in range(2):
        one = full["net"].forward(x[b:b + 1].cuda(), float(fx["t"]), ctx[b:b + 1].cuda(), pooled[b:b + 1].cuda(),
                                  tids[b:b + 1].cuda()).float().cpu()
        assert torch.equal(one[0], eps[b]), f"batch-1 forward of half {b} differs from the batch-2 forward"


@pytest.mark.slow
def test_full_sdxl_unet_matches_oracle_non_square():
    from latentblending_b200 import ops
    from oracle.sdxl_unet import SDXL_BASE
    from test_unet_gpu import _full_sdxl, _inputs
    full = _full_sdxl()
    x, ctx, pooled, tids = _inputs(SDXL_BASE, 2, 24, 40, 0)
    with torch.no_grad():
        ref = full["oracle"](x.float(), 701.0, ctx.float(), pooled.float(), tids.float())
    eps = full["net"].forward(x.cuda(), 701.0, ctx.cuda(), pooled.cuda(), tids.cuda()).float().cpu()
    assert ops.error_flag() == 0
    rel = ((eps - ref).norm() / ref.norm()).item()
    print(f"full SDXL UNet @24x40 B=2: rel_l2={rel:.3e}")
    assert rel <= 2e-3, f"relative L2 error {rel}"


# ---- 5. VAE -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("h,w", [(12, 20), (20, 12)])
def test_vae_non_square(h, w):
    from test_vae_gpu import test_vae_decoder_matches_oracle
    test_vae_decoder_matches_oracle(h, w)


def test_sdxl_width_vae_matches_fixture_at_bucket():
    from latentblending_b200 import ops
    from latentblending_b200.vae import VAEDecoderB200
    from make_bucket_fixtures import VAE_BUCKET_FIXTURE, VAE_BUCKET_HW, oracle_vae, vae_latent, weights_checksum
    fx = np.load(VAE_BUCKET_FIXTURE)
    ov, cfg = oracle_vae()
    assert weights_checksum(ov.state_dict()) == str(fx["weights_sha1"]), "seeded VAE recipe drifted"
    vae = VAEDecoderB200(ov.state_dict(), cfg.block_out_channels, cfg.scaling_factor, "cuda:0")
    h, w = VAE_BUCKET_HW
    got = vae.decode_to_u8(vae_latent(h, w).cuda()).cpu().numpy()
    ref = fx["frame"]
    assert got.shape == ref.shape == (8 * h, 8 * w, 3)
    d = np.abs(got.astype(np.int32) - ref.astype(np.int32))
    print(f"SDXL-width VAE @{h}x{w}: mean |d|={d.mean():.3f} max={d.max()} levels")
    assert d.mean() <= 1.0 and d.max() <= 12, (d.mean(), d.max())
    assert ops.error_flag() == 0 and vae.overflow_count() == 0


# ---- 6. LPIPS -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("H,W", [(1216, 832), (832, 1216)])
def test_native_lpips_non_square(H, W):
    from test_round2_gpu import test_native_lpips_matches_oracle
    test_native_lpips_matches_oracle(H, W)


# ---- 7. engine ----------------------------------------------------------------------------------------------------
def _engine_at(size, seed, **kw):
    from latentblending_b200 import BlendingEngine
    from test_engine_gpu import _pair
    _, pp, _ = _pair(kw.pop("turbo", False), seed=seed)
    be = BlendingEngine(pp, run_benchmark=False)
    be.set_dimensions(size)
    be.set_prompt1("photo of a lake")
    be.set_prompt2("alien planet")
    return be


@pytest.mark.parametrize("size", [(160, 96), (96, 160)])
def test_whole_transition_matches_oracle_engine_non_square(size, monkeypatch):
    """test_engine_gpu's teacher-forced whole-transition comparison, at a landscape and a portrait size."""
    import test_engine_gpu
    from latentblending_b200 import BlendingEngine
    from oracle.engine import OracleEngine
    for cls in (BlendingEngine, OracleEngine):
        orig = cls.set_dimensions
        monkeypatch.setattr(cls, "set_dimensions", lambda self, s=None, _o=orig: _o(self, size))
    test_engine_gpu.test_whole_transition_matches_oracle_engine(False)


def test_engine_paths_bit_identical_non_square():
    """At 160 x 96: batched outer pair == sequential, dual-stream == batch 2, speculation width 1 == 3, and
    get_movie_frames returns [T, H, W, 3]."""
    from latentblending_b200 import DiffusersHolder
    be = _engine_at((160, 96), seed=5)
    be.set_num_inference_steps(5)
    be.seed1, be.seed2 = 11, 12
    seq1 = [t.clone() for t in be.compute_latents1()]
    seq2 = [t.clone() for t in be.compute_latents2()]
    bat1, bat2 = be._compute_latents_pair()
    assert seq1[-1].shape[-2:] == (12, 20)
    for i in range(5):
        assert torch.equal(bat1[i], seq1[i]) and torch.equal(bat2[i], seq2[i]), i
    # dual stream
    dh = DiffusersHolder(be.dh.pipe)
    dh.guidance_scale = 3.5
    dh.set_dimensions((96, 160))
    dh.set_num_inference_steps(4)
    emb = dh.get_text_embedding("a lake")
    start = dh.get_noise(5)
    res = {}
    for dual in (False, True):
        dh.dual_stream = dual
        res[dual] = [t.clone() for t in dh.run_diffusion_sd_xl(emb, start)]
    assert all(torch.equal(a, b) for a, b in zip(res[True], res[False]))
    # lockstep speculation
    runs = []
    for width in (1, 3):
        e = _engine_at((160, 96), seed=9)
        e.set_num_inference_steps(8)
        e.set_branching(depth_strength=0.5, nmb_max_branches=7)
        e.speculative_batch = width
        e.deterministic_noise = True
        e.output_device_frames = True
        e.run_transition(fixed_seeds=[7, 8])
        runs.append((list(e.tree_fracts), [float(s) for s in e.tree_similarities],
                     torch.stack([t[-1] for t in e.tree_latents]).clone()))
    assert runs[0][0] == runs[1][0] and runs[0][1] == runs[1][1] and torch.equal(runs[0][2], runs[1][2])
    frames = e.get_movie_frames(1, fps=6)
    assert frames.ndim == 4 and frames.shape[0] >= 6 and frames.shape[1:] == (96, 160, 3) and frames.dtype == np.uint8
    from latentblending_b200 import ops
    assert ops.error_flag() == 0


def test_storyboard_with_non_square_size(tmp_path):
    from latentblending_b200.storyboard import run_storyboard
    be = _engine_at((128, 128), seed=4, turbo=True)
    fp = os.path.join(tmp_path, "story.json")
    with open(fp, "w") as f:
        json.dump([{"settings": "sdxl", "width": 96, "height": 160, "num_inference_steps": 4},
                   {"iteration": 0, "seed": 1, "prompt": "a lake"},
                   {"iteration": 1, "seed": 2, "prompt": "a forest"},
                   {"iteration": 2, "seed": 3, "prompt": "a city"}], f)
    be.set_branching(nmb_max_branches=4)
    out = run_storyboard(be, fp)
    assert len(out) == 2
    assert (be.dh.width_img, be.dh.height_img) == (96, 160)
    assert all(np.asarray(fr).shape == (160, 96, 3) for frames in out for fr in frames)
