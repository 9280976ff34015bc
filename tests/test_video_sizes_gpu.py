"""GPU checks of output sizes whose latent sides are not divisible by 2^(levels-1) -- 1280x720 (latent 90x160),
1920x1080 (135x240) and every other multiple of 8 px: the crop-aware nearest upsample (lb_upsample_nearest), and
every layer above it (UNet, VAE, LPIPS, engine) at such sizes.  Tolerances are the ones the square-size tests use,
stated at each assert."""
import dataclasses
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _rand(*shape, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(*shape, generator=g, device="cuda").half()


# ---- 1. the kernel ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,H,W,C", [(1, 1, 1, 64), (2, 5, 3, 64), (4, 23, 40, 64), (3, 12, 7, 1280), (2, 34, 60, 64)])
def test_upsample_nearest_matches_interpolate(B, H, W, C):
    """Every Ho in {2H-1, 2H} x Wo in {2W-1, 2W} against F.interpolate(size=...) bit for bit, reading a channel slice
    of a wider buffer (row stride > C) and writing into one."""
    from latentblending_b200 import ops
    src = _rand(B * H * W, C + 64, seed=B * H + W)
    x = src[:, 32:32 + C]
    ref_in = x.reshape(B, H, W, C).permute(0, 3, 1, 2)
    for Ho in (2 * H - 1, 2 * H):
        for Wo in (2 * W - 1, 2 * W):
            if Ho < 1 or Wo < 1:
                continue
            ref = F.interpolate(ref_in, size=(Ho, Wo), mode="nearest").permute(0, 2, 3, 1).reshape(-1, C)
            dst = torch.full((B * Ho * Wo, C + 16), -7.0, dtype=torch.float16, device="cuda")
            out = ops.upsample_nearest(x, B, H, W, C, Ho, Wo, out=dst[:, 8:8 + C])
            assert torch.equal(out, ref), (Ho, Wo)
            assert (dst[:, :8] == -7).all() and (dst[:, 8 + C:] == -7).all()      # nothing outside the slice
    assert ops.error_flag() == 0


def test_upsample_nearest_rejects_other_sizes():
    from latentblending_b200 import _cabi, ops
    x = _rand(2 * 5 * 3, 64)
    for Ho, Wo in ((11, 6), (8, 6), (10, 7), (10, 4)):
        with pytest.raises(_cabi.LB200Error, match="nearest 2x"):
            ops.upsample_nearest(x, 2, 5, 3, 64, Ho, Wo)
    with pytest.raises(_cabi.LB200Error, match="multiples of 8"):
        ops.upsample_nearest(_rand(30, 60)[:, :60], 2, 5, 3, 60, 10, 6)


def test_upsample2x_and_program_record_agree():
    """ops.upsample2x, ops.upsample_nearest at (2H, 2W) and a program record give the same bits; a record's Ho, Wo
    are explicit (0 is not a size)."""
    from latentblending_b200 import _cabi, ops
    from latentblending_b200.program import Program
    B, H, W, C = 2, 16, 24, 320
    x = _rand(B * H * W, C, seed=3)
    a = ops.upsample2x(x, B, H, W, C)
    b = ops.upsample_nearest(x, B, H, W, C, 2 * H, 2 * W)
    assert torch.equal(a, b)
    outs = []
    for ho, wo in ((2 * H, 2 * W), (2 * H - 1, 2 * W - 1)):
        out = torch.zeros(B * ho * wo, C, dtype=torch.float16, device="cuda")
        P = Program(0)
        P.upsample_nearest(x, B, H, W, C, out, ho, wo)
        P.finalize().run()
        outs.append(out)
    torch.cuda.synchronize()
    assert torch.equal(outs[0], a)
    assert torch.equal(outs[1], ops.upsample_nearest(x, B, H, W, C, 2 * H - 1, 2 * W - 1))
    P = Program(0)
    P.upsample_nearest(x, B, H, W, C, outs[0], 0, 0)
    with pytest.raises(_cabi.LB200Error, match="nearest 2x"):
        P.finalize().run()
    assert ops.error_flag() == 0


# ---- 2. UNet ------------------------------------------------------------------------------------------------------
def _run_pair(ocfg, B, h, w, t, seed=0):
    """test_unet_gpu._run_pair with the oracle run by diffusers' resize-to-skip-size rule (sized_unet.py)."""
    from latentblending_b200 import ops
    from latentblending_b200.unet import UNetB200, UNetConfig
    from oracle.sdxl_unet import SDXLUNet, synthetic_init_
    from sized_unet import forward_sized
    from test_unet_gpu import _inputs
    oracle = synthetic_init_(SDXLUNet(ocfg), seed=seed).eval()
    with torch.no_grad():
        for p in oracle.parameters():
            p.copy_(p.half().float())
    cfg = UNetConfig(**{f.name: getattr(ocfg, f.name) for f in dataclasses.fields(ocfg)})
    net = UNetB200(cfg, oracle.state_dict(), "cuda:0")
    x, ctx, pooled, tids = _inputs(ocfg, B, h, w, seed)
    with torch.no_grad():
        ref = forward_sized(oracle, x.float(), t, ctx.float(), pooled.float(), tids.float())
    eps = net.forward(x.cuda(), t, ctx.cuda(), pooled.cuda(), tids.cuda()).float().cpu()
    torch.cuda.synchronize()
    assert ops.error_flag() == 0
    rel = ((eps - ref).norm() / ref.norm()).item()
    print(f"unet parity: B={B} h={h} w={w} t={t} rel_l2={rel:.3e}")
    return rel, eps, ref, net


@pytest.mark.parametrize("B,h,w", [(2, 17, 11), (2, 11, 17), (2, 90, 160), (1, 135, 240)])
def test_tiny_unet_at_odd_latent_sizes(B, h, w):
    """17x11 and 11x17 crop in H and in W at both upsamplers; 90x160 (1280x720) crops at 23 -> 45 rows; 135x240
    (1920x1080) at 68 -> 135 rows.  Relative L2 of eps <= 2e-3 vs the fp32 oracle."""
    from oracle.sdxl_unet import tiny_config
    rel, eps, _, _ = _run_pair(tiny_config(), B, h, w, 611.0)
    assert torch.isfinite(eps).all() and eps.shape == (B, 4, h, w)
    assert rel <= 2e-3, f"relative L2 error {rel}"


@pytest.mark.parametrize("h,w", [(17, 11), (11, 17)])
def test_medium_unet_at_odd_latent_sizes(h, w):
    from oracle.sdxl_unet import UNetConfig
    ocfg = UNetConfig(block_out_channels=(128, 256, 512), transformer_layers=(0, 2, 10), cross_attention_dim=256,
                      addition_time_embed_dim=64, pooled_dim=128, sample_size=32)
    rel, eps, _, _ = _run_pair(ocfg, 2, h, w, 499.0)
    assert torch.isfinite(eps).all()
    assert rel <= 2e-3, f"relative L2 error {rel}"


@pytest.mark.slow
def test_full_sdxl_unet_matches_fixture_at_720p():
    """Full SDXL-base UNet, CFG batch 2, at 1280x720 (latent 90 x 160) vs the fp32 oracle fixture; each CFG half alone
    is bit-identical to its half of the batch-2 forward."""
    from latentblending_b200 import ops
    from make_video_fixtures import UNET_SEED, UNET_VIDEO_FIXTURE, UNET_VIDEO_HW, unet_inputs
    from oracle.sdxl_unet import SDXL_BASE
    from test_unet_gpu import _full_sdxl
    fx = np.load(UNET_VIDEO_FIXTURE)
    full = _full_sdxl()
    assert full["sha"] == str(fx["weights_sha1"]), "seeded weight recipe drifted from the fixture's"
    h, w = UNET_VIDEO_HW
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
    full["net"]._plans.clear()


@pytest.mark.slow
def test_full_sdxl_unet_matches_oracle_at_17x11():
    from latentblending_b200 import ops
    from oracle.sdxl_unet import SDXL_BASE
    from sized_unet import forward_sized
    from test_unet_gpu import _full_sdxl, _inputs
    full = _full_sdxl()
    x, ctx, pooled, tids = _inputs(SDXL_BASE, 2, 17, 11, 0)
    with torch.no_grad():
        ref = forward_sized(full["oracle"], x.float(), 701.0, ctx.float(), pooled.float(), tids.float())
    eps = full["net"].forward(x.cuda(), 701.0, ctx.cuda(), pooled.cuda(), tids.cuda()).float().cpu()
    assert ops.error_flag() == 0
    rel = ((eps - ref).norm() / ref.norm()).item()
    print(f"full SDXL UNet @17x11 B=2: rel_l2={rel:.3e}")
    assert rel <= 2e-3, f"relative L2 error {rel}"


@pytest.mark.slow
def test_full_sdxl_unet_runs_at_1080p():
    """One CFG-batch-2 forward at 1920x1080 (latent 135 x 240: 135 -> 68 -> 34 rows, crops at 68 -> 135)."""
    from latentblending_b200 import ops
    from oracle.sdxl_unet import SDXL_BASE
    from test_unet_gpu import _full_sdxl, _inputs
    full = _full_sdxl()
    x, ctx, pooled, tids = _inputs(SDXL_BASE, 2, 135, 240, 0)
    eps = full["net"].forward(x.cuda(), 499.0, ctx.cuda(), pooled.cuda(), tids.cuda()).float().cpu()
    torch.cuda.synchronize()
    assert ops.error_flag() == 0
    assert eps.shape == (2, 4, 135, 240) and torch.isfinite(eps).all()
    assert eps.std() > 0
    full["net"]._plans.clear()
    torch.cuda.empty_cache()


# ---- 3. VAE -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cols", [187, 5, 1, 192])
def test_softmax_rows_any_width_with_dtype(cols):
    """lb_softmax_rows over a column count that need not be a multiple of 8 (the VAE mid-block attention's h*w keys),
    in place in a wider buffer, vs torch.softmax in fp32; the columns past ``cols`` are left alone."""
    from latentblending_b200 import _cabi
    from latentblending_b200._cabi import check, ctx, ptr, stream_ptr
    rows, ld = 33, -(-cols // 64) * 64 + 64
    buf = _rand(rows, ld, seed=cols) * 4
    ref = torch.softmax(buf[:, :cols].float(), dim=-1)
    tail = buf[:, cols:].clone()
    check(_cabi.load().lb_softmax_rows(ctx(0), ptr(buf), ld, rows, cols, ptr(buf), ld, stream_ptr(), _cabi.DTYPE_F16),
          "lb_softmax_rows")
    torch.cuda.synchronize()
    assert (buf[:, :cols].float() - ref).abs().max().item() <= 2e-3          # fp16 output rounding
    assert torch.equal(buf[:, cols:], tail)


def test_vae_at_17x11():
    """h*w = 187 keys in the mid-block attention: not a multiple of 8, so its key-sized GEMM operands are padded."""
    from test_vae_gpu import test_vae_decoder_matches_oracle
    test_vae_decoder_matches_oracle(17, 11)


def test_sdxl_width_vae_at_1080p():
    from latentblending_b200 import ops
    from latentblending_b200.vae import VAEDecoderB200
    from make_fullsize_fixtures import oracle_vae, vae_latent
    ov, cfg = oracle_vae()
    vae = VAEDecoderB200(ov.state_dict(), cfg.block_out_channels, cfg.scaling_factor, "cuda:0")
    frame = vae.decode_to_u8(vae_latent(135, 240).cuda()).cpu().numpy()
    assert frame.shape == (1080, 1920, 3) and frame.dtype == np.uint8
    assert frame.std() > 5
    assert ops.error_flag() == 0 and vae.overflow_count() == 0
    vae._plans.clear()
    torch.cuda.empty_cache()


# ---- 4. LPIPS -----------------------------------------------------------------------------------------------------
def test_native_lpips_at_720p():
    from test_round2_gpu import test_native_lpips_matches_oracle
    test_native_lpips_matches_oracle(720, 1280)


# ---- 5. engine at 136 x 88 px (latent 11 x 17; 4*h*w = 748 is not a multiple of 8) --------------------------------
SIZE = (136, 88)


def _engine_at(size, seed, **kw):
    from latentblending_b200 import BlendingEngine
    from test_engine_gpu import _pair
    _, pp, _ = _pair(kw.pop("turbo", False), seed=seed)
    be = BlendingEngine(pp, run_benchmark=False)
    be.set_dimensions(size)
    be.set_prompt1("photo of a lake")
    be.set_prompt2("alien planet")
    return be


def test_whole_transition_matches_oracle_engine_at_odd_latent(monkeypatch):
    """test_engine_gpu's teacher-forced whole-transition comparison at 136 x 88 px, the oracle UNet run by diffusers'
    resize-to-skip-size rule."""
    import test_engine_gpu
    from latentblending_b200 import BlendingEngine
    from oracle.engine import OracleEngine
    from oracle.sdxl_unet import SDXLUNet
    from sized_unet import forward_sized
    monkeypatch.setattr(SDXLUNet, "forward", forward_sized)
    for cls in (BlendingEngine, OracleEngine):
        orig = cls.set_dimensions
        monkeypatch.setattr(cls, "set_dimensions", lambda self, s=None, _o=orig: _o(self, SIZE))
    test_engine_gpu.test_whole_transition_matches_oracle_engine(False)


def test_engine_paths_bit_identical_at_odd_latent():
    """At 136 x 88 px: batched outer pair == sequential, dual-stream == batch 2, speculation width 1 == 3, and
    get_movie_frames returns [T, 88, 136, 3]."""
    from latentblending_b200 import DiffusersHolder, ops
    be = _engine_at(SIZE, seed=5)
    be.set_num_inference_steps(5)
    be.seed1, be.seed2 = 11, 12
    seq1 = [t.clone() for t in be.compute_latents1()]
    seq2 = [t.clone() for t in be.compute_latents2()]
    bat1, bat2 = be._compute_latents_pair()
    assert seq1[-1].shape[-2:] == (11, 17)
    for i in range(5):
        assert torch.equal(bat1[i], seq1[i]) and torch.equal(bat2[i], seq2[i]), i
    dh = DiffusersHolder(be.dh.pipe)
    dh.guidance_scale = 3.5
    dh.set_dimensions(SIZE)
    dh.set_num_inference_steps(4)
    emb = dh.get_text_embedding("a lake")
    start = dh.get_noise(5)
    res = {}
    for dual in (False, True):
        dh.dual_stream = dual
        res[dual] = [t.clone() for t in dh.run_diffusion_sd_xl(emb, start)]
    assert all(torch.equal(a, b) for a, b in zip(res[True], res[False]))
    runs = []
    for width in (1, 3):
        e = _engine_at(SIZE, seed=9)
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
    assert frames.ndim == 4 and frames.shape[0] >= 6 and frames.shape[1:] == (88, 136, 3) and frames.dtype == np.uint8
    assert ops.error_flag() == 0


def test_storyboard_at_720p(tmp_path):
    from latentblending_b200.storyboard import run_storyboard
    be = _engine_at((128, 128), seed=4, turbo=True)
    fp = os.path.join(tmp_path, "story.json")
    with open(fp, "w") as f:
        json.dump([{"settings": "sdxl", "width": 1280, "height": 720, "num_inference_steps": 4},
                   {"iteration": 0, "seed": 1, "prompt": "a lake"},
                   {"iteration": 1, "seed": 2, "prompt": "a forest"}], f)
    be.set_branching(nmb_max_branches=4)
    out = run_storyboard(be, fp)
    assert len(out) == 1
    assert (be.dh.width_img, be.dh.height_img) == (1280, 720)
    assert all(np.asarray(fr).shape == (720, 1280, 3) for frames in out for fr in frames)
