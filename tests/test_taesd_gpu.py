"""GPU tests of the tiny VAE decoder (AutoencoderTiny / TAESDXL): the depth-to-space GEMM (LB_GEMM_D2S2) against an
fp32 upsample + conv, the tiny-VAE conv_in variant (lb_conv_in act 1), the whole decoder against the fp32 oracle
(oracle/taesd.py) and its fixtures, and the engine running a transition with it.

Tolerances (stated):
  * D2S2 GEMM: relative L2 <= 2e-3 against fp32 conv2d(interpolate(x)); max |error| <= 2^-11 * (|x| . |w|)-sum + one
    fp16 output ulp -- the pre-summed phase weights are rounded to fp16 once (half an ulp, 2^-11 relative, on every
    product) and the output once;
  * conv_in variant: within one fp16 ulp of the fp32 conv of the emulated clamp (plus fp32 summation slack);
  * frames: mean |d| <= 1.0 and max <= 12 uint8 levels, as tests/test_vae_gpu.py."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _rand(*shape, seed=0, s=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(*shape, generator=g, device="cuda") * s


def _pack3(w):
    return w.permute(0, 2, 3, 1).reshape(w.shape[0], -1).contiguous()


def _d2s_problem(B, H, W, C, Co, seed):
    from latentblending_b200.taesd import pack_d2s_weights
    x = _rand(B * H * W, C, seed=seed).half()
    w = (_rand(Co, C, 3, 3, seed=seed + 1) * (9 * C) ** -0.5).half()
    bias = (_rand(Co, seed=seed + 2) * 0.1).half()
    wp = _pack3(pack_d2s_weights(w.float())).half()
    b4 = bias.repeat(4).contiguous()
    return x, w, bias, wp, b4


def _d2s_ref(x, w, bias, B, H, W, relu=False):
    xi = x.float().view(B, H, W, -1).permute(0, 3, 1, 2)
    up = F.interpolate(xi, scale_factor=2, mode="nearest")
    ref = F.conv2d(up, w.float(), bias.float(), padding=1)
    absprod = F.conv2d(up.abs(), w.float().abs(), padding=1) + bias.float().abs()[None, :, None, None]
    if relu:
        ref = ref.clamp_min(0)
    flat = lambda t: t.permute(0, 2, 3, 1).reshape(B * 4 * H * W, -1)
    return flat(ref), flat(absprod)


D2S_SHAPES = [(1, 1, 1), (2, 1, 1), (1, 5, 7), (2, 5, 7), (1, 13, 24), (2, 13, 24), (1, 16, 16), (2, 16, 16),
              (1, 64, 64), (1, 45, 80), (1, 128, 128)]


@pytest.mark.parametrize("B,H,W", D2S_SHAPES)
@pytest.mark.parametrize("Co", [8, 64])
def test_d2s_gemm_matches_upsample_conv(B, H, W, Co):
    """N = 32 (Co 8: BN 64) and N = 256 (Co 64: BN 128); forced box and runs tilings bit-identical where the box
    applies."""
    from latentblending_b200 import ops
    C = 64
    x, w, bias, wp, b4 = _d2s_problem(B, H, W, C, Co, seed=B * 100 + H + W + Co)
    ref, absprod = _d2s_ref(x, w, bias, B, H, W, relu=True)
    outs = {}
    for t in ("auto", "box", "runs"):
        if t == "box" and W < 128 and (W & (W - 1) or (H * W < 128 and H & (H - 1))) and not (H == 1 and B == 1):
            continue
        outs[t] = ops.gemm(x, wp, 4 * Co, B, H, W, taps=9, bias=b4, relu=True, depth_to_space=True, tiling=t)
    torch.cuda.synchronize()
    for t, o in outs.items():
        assert o.shape == (4 * B * H * W, Co)
        assert torch.equal(o, outs["runs"]), t
    got = outs["auto"].float()
    rel = ((got - ref).norm() / ref.norm().clamp_min(1e-30)).item()
    assert rel <= 2e-3, rel
    bound = 2.0 ** -11 * absprod + 2.0 ** -10 * ref.abs() + 1e-6
    assert ((got - ref).abs() <= bound).all(), ((got - ref).abs() - bound).max().item()
    assert ops.error_flag() == 0


def test_d2s_gemm_large_n_tiles():
    """N = 512 over enough tiles selects the cooperative BN = 256 tile (four phases in one tile) for a long K."""
    from latentblending_b200 import ops
    B, H, W, C, Co = 1, 96, 96, 512, 128
    x, w, bias, wp, b4 = _d2s_problem(B, H, W, C, Co, seed=77)
    ref, absprod = _d2s_ref(x, w, bias, B, H, W)
    got = ops.gemm(x, wp, 4 * Co, B, H, W, taps=9, bias=b4, depth_to_space=True).float()
    rel = ((got - ref).norm() / ref.norm()).item()
    assert rel <= 2e-3, rel
    assert ((got - ref).abs() <= 2.0 ** -11 * absprod + 2.0 ** -10 * ref.abs() + 1e-6).all()
    assert ops.error_flag() == 0


def test_d2s_gemm_rejections():
    """Each combination the depth-to-space epilogue does not implement raises before any launch."""
    from latentblending_b200 import _cabi, ops
    B, H, W, C, Co = 1, 8, 8, 64, 64
    x, w, bias, wp, b4 = _d2s_problem(B, H, W, C, Co, seed=5)
    out = torch.full((4 * B * H * W, Co), 7.0, dtype=torch.float16, device="cuda")
    res = torch.zeros_like(out)
    b2 = torch.zeros(1, 4 * Co, dtype=torch.float16, device="cuda")
    bad = [dict(taps=1, w=x[:4 * Co].contiguous()),                  # not a 3x3 conv
           dict(N=4 * Co - 8, w=wp[:4 * Co - 8]),                      # N % 32 != 0
           dict(res=res), dict(bias2=b2), dict(a1=x), dict(mode=1)]
    for kw in bad:
        args = dict(taps=9, w=wp, N=4 * Co, bias=b4)
        args.update(kw)
        wk, N = args.pop("w"), args.pop("N")
        with pytest.raises(_cabi.LB200Error, match="D2S2"):
            ops.gemm(x, wk, N, B, H, W, out=out, depth_to_space=True, **args)
    with pytest.raises(_cabi.LB200Error, match="D2S2"):
        ops.gemm(x.bfloat16(), wp.bfloat16(), 4 * Co, B, H, W, taps=9, depth_to_space=True)
    stats = torch.zeros(B * H * W, 4 * 2, 2, dtype=torch.float32, device="cuda")
    with pytest.raises(_cabi.LB200Error, match="D2S2"):
        ops.gemm(x, wp, 4 * Co, B, H, W, taps=9, out=out, depth_to_space=True, stats_out=stats)
    torch.cuda.synchronize()
    assert torch.all(out == 7.0) and ops.error_flag() == 0


# ---- conv_in variant ---------------------------------------------------------------------------------------------
def _tiny_clamp_ref(v, in_scale):
    """tanh(v * in_scale / 3) * 3 with the fp16 roundings of the reference's fp16 tensor ops."""
    h = lambda t: t.half().float()
    z = h(v.float() * in_scale)
    return h(h(torch.tanh(h(z / 3))) * 3)


@pytest.mark.parametrize("h,w,in_scale", [(16, 16, 1.0), (13, 24, 1.0), (45, 80, 1 / 0.13025)])
def test_conv_in_tiny_variant(h, w, in_scale):
    from latentblending_b200 import ops
    C = 64
    lat = (_rand(1, 4, h, w, seed=h + w) * 4.0).half()           # |v| up to ~16: tanh saturates in part of the map
    wt = (_rand(C, 4, 3, 3, seed=3) * 36 ** -0.5).half()
    b = (_rand(C, seed=4) * 0.1).half()
    got = ops.conv_in(lat, wt.permute(2, 3, 1, 0).contiguous(), b, C, act=1, in_scale=in_scale).float()
    xin = _tiny_clamp_ref(lat, in_scale)
    assert (xin.abs() > 2.9).float().mean() > 0.05                # saturated region present
    ref = F.conv2d(xin, wt.float(), b.float(), padding=1).clamp_min(0).permute(0, 2, 3, 1).reshape(h * w, C)
    absprod = F.conv2d(xin.abs(), wt.float().abs(), b.float().abs(), padding=1).permute(0, 2, 3, 1).reshape(h * w, C)
    # one fp16 rounding of the output, plus one fp16 ulp on any clamped input whose tanh lands on a rounding boundary
    # (device tanhf and torch's tanh may differ in the last fp32 bit)
    assert ((got - ref).abs() <= 2.0 ** -11 * ref.abs() + 2.0 ** -10 * absprod + 1e-7).all()
    exact = (got - ref).abs() <= 2.0 ** -11 * ref.abs() + 1e-5 * absprod + 1e-7
    assert exact.float().mean() > 0.999
    assert ops.error_flag() == 0


def test_program_conv_in_plain_record_equals_eager():
    """A program conv_in record with act 0 (CONV_IN_PLAIN) is ops.conv_in's default."""
    from latentblending_b200 import _cabi, ops
    from latentblending_b200.program import Program
    lat = _rand(1, 4, 12, 20, seed=9).half()
    wt = (_rand(3, 3, 4, 64, seed=10) * 0.2).half()
    b = (_rand(64, seed=11) * 0.1).half()
    out = torch.empty(12 * 20, 64, dtype=torch.float16, device="cuda")
    P = Program(0)
    P.conv_in(lat, wt, b, 64, out, _cabi.CONV_IN_PLAIN)
    P.finalize().run()
    assert torch.equal(out, ops.conv_in(lat, wt, b, 64))


def test_conv_in_act_rejects_bf16_and_unknown_act():
    from latentblending_b200 import _cabi, ops
    lat = _rand(1, 4, 8, 8).half()
    wt = torch.zeros(3, 3, 4, 64, dtype=torch.float16, device="cuda")
    b = torch.zeros(64, dtype=torch.float16, device="cuda")
    with pytest.raises(_cabi.LB200Error, match="fp16-only"):
        ops.conv_in(lat.bfloat16(), wt.bfloat16(), b.bfloat16(), 64, act=1)
    with pytest.raises(_cabi.LB200Error, match="act"):
        ops.conv_in(lat, wt, b, 64, act=2)


# ---- the whole decoder -------------------------------------------------------------------------------------------
def _frame_diff(got, ref):
    d = np.abs(got.astype(np.int32) - ref.astype(np.int32))
    return d.mean(), d.max()


def _decoder(sd=None):
    from latentblending_b200.taesd import DEFAULT_CONFIG, TinyVAEDecoderB200
    from make_taesd_fixtures import tiny_state_dict
    return TinyVAEDecoderB200(tiny_state_dict() if sd is None else sd, DEFAULT_CONFIG, 1.0, "cuda:0")


def _check_oracle_frame(ref):
    assert ref.std() > 5, ref.std()
    assert ((ref == 0) | (ref == 255)).mean() < 0.1


@pytest.mark.parametrize("h,w", [(16, 16), (13, 24), (17, 11)])
def test_tiny_decoder_matches_oracle_small(h, w):
    from latentblending_b200 import ops
    from make_fullsize_fixtures import vae_latent
    from make_taesd_fixtures import oracle_taesd
    from oracle.taesd import latent2image_np
    lat = vae_latent(h, w)
    with torch.no_grad():
        ref = latent2image_np(oracle_taesd(), lat)
    _check_oracle_frame(ref)
    vae = _decoder()
    got = vae.decode_to_u8(lat.cuda()).cpu().numpy()
    assert got.shape == (8 * h, 8 * w, 3)
    mean, mx = _frame_diff(got, ref)
    print(f"tiny decoder {h}x{w}: mean |d| {mean:.3f} max {mx}")
    assert mean <= 1.0 and mx <= 12, (mean, mx)
    # graph replay (second and later runs) gives the same frame
    for _ in range(2):
        assert np.array_equal(vae.decode_to_u8(lat.cuda()).cpu().numpy(), got)
    assert vae.overflow_count() == 0 and ops.error_flag() == 0


@pytest.mark.parametrize("hw", [(64, 64), (90, 160)])
def test_tiny_decoder_matches_fixture(hw):
    from latentblending_b200 import ops
    from make_fullsize_fixtures import weights_checksum
    from make_taesd_fixtures import FIXTURES, frame_sample, tiny_state_dict
    fx = np.load(FIXTURES[hw])
    sd = tiny_state_dict()
    assert weights_checksum(sd) == str(fx["weights_sha1"]), "seeded tiny VAE recipe drifted"
    _check_oracle_frame(fx["frame"])
    vae = _decoder(sd)
    got = vae.decode_to_u8(torch.from_numpy(fx["latents"]).cuda()).cpu().numpy()
    assert got.shape == (8 * hw[0], 8 * hw[1], 3)
    mean, mx = _frame_diff(frame_sample(got, fx), fx["frame"])
    print(f"tiny decoder fixture {hw}: mean |d| {mean:.3f} max {mx}")
    assert mean <= 1.0 and mx <= 12, (mean, mx)
    assert vae.overflow_count() == 0 and ops.error_flag() == 0


def test_tiny_decoder_at_1080p_and_overflow_message():
    from latentblending_b200 import _cabi, ops
    from make_fullsize_fixtures import vae_latent
    vae = _decoder()
    frame = vae.decode_to_u8(vae_latent(135, 240).cuda())
    torch.cuda.synchronize()
    assert frame.shape == (1080, 1920, 3) and frame.float().std() > 5
    assert vae.overflow_count() == 0 and ops.error_flag() == 0
    # an output that overflows fp16 is counted and reported; the message must not advise bf16 (there is none here)
    from make_taesd_fixtures import tiny_state_dict
    sd = tiny_state_dict()
    sd["layers.18.bias"] = torch.full_like(sd["layers.18.bias"], 40000.0)    # 2b - 1 > 65504: Inf in fp16
    hot = _decoder(sd)
    hot.decode_to_u8(vae_latent(16, 16).cuda())
    with pytest.raises(_cabi.LB200Error, match="non-finite") as ei:
        hot.check_overflow()
    assert "bf16" not in str(ei.value)
    assert hot.overflow_count() == 0 and ops.error_flag() == 0


# ---- engine ------------------------------------------------------------------------------------------------------
def _tiny_vae_pipe(turbo=True, seed=0):
    from test_engine_gpu import _pair
    from latentblending_b200 import SyntheticSDXLPipe
    _, pp, _ = _pair(turbo, seed)
    return SyntheticSDXLPipe(pp._name_or_path, "cuda:0", unet_cfg=pp.unet_cfg, unet_state_dict=pp.unet_state_dict,
                             lpips_state_dict=pp.lpips_state_dict, seed=3, vae="tiny")


def _transition(be):
    be.deterministic_noise = True
    be.set_dimensions((128, 128))
    be.set_num_inference_steps(4)
    be.set_prompt1("photo of a lake")
    be.set_prompt2("alien planet")
    be.set_branching(nmb_max_branches=3)
    return be.run_transition(fixed_seeds=[420, 421])


def test_engine_transition_with_tiny_vae():
    from latentblending_b200 import BlendingEngine
    pp = _tiny_vae_pipe()
    be = BlendingEngine(pp, run_benchmark=False)
    assert type(be.dh.vae).__name__ == "TinyVAEDecoderB200"
    imgs = _transition(be)
    assert len(imgs) == len(be.tree_latents) >= 3
    for img, lat in zip(be.tree_final_imgs, be.tree_latents):
        frame = be.dh.vae.decode_to_u8(lat[-1].to(torch.float16)).cpu().numpy()
        assert np.array_equal(np.asarray(img), frame)
        assert frame.std() > 5
    # same seeds -> same tree and frames
    be2 = BlendingEngine(_tiny_vae_pipe(), run_benchmark=False)
    imgs2 = _transition(be2)
    assert len(imgs2) == len(imgs)
    for a, b in zip(imgs, imgs2):
        assert np.array_equal(np.asarray(a), np.asarray(b))
    for a, b in zip(be.tree_latents, be2.tree_latents):
        assert torch.equal(a[-1], b[-1])
    assert be.dh.vae.overflow_count() == 0
    with pytest.raises(ValueError, match="fp16 only"):
        be.dh.set_vae_dtype("bf16")
    be.dh.set_vae_dtype("fp16")
    assert type(be.dh.vae).__name__ == "TinyVAEDecoderB200"


def test_holder_from_mock_autoencoder_tiny_decodes_on_device():
    from latentblending_b200 import DiffusersHolder, ops
    from make_fullsize_fixtures import vae_latent
    from make_taesd_fixtures import oracle_taesd
    from oracle.taesd import latent2image_np
    from test_taesd_cpu import _mock_tiny_pipe
    from latentblending_b200.pipe import random_tiny_vae_state_dict
    sd = random_tiny_vae_state_dict(3, "cpu")
    mock = _mock_tiny_pipe(sd)
    mock._execution_device = torch.device("cuda:0")
    dh = DiffusersHolder(mock)
    assert dh.pipe.vae_kind == "tiny" and dh.vae_dtype == "fp16"
    lat = vae_latent(16, 16)
    got = dh.latent2image(lat.cuda(), output_type="np")
    with torch.no_grad():
        ref = latent2image_np(oracle_taesd(sd), lat)
    mean, mx = _frame_diff(np.round(got * 255).astype(np.uint8), ref)
    assert mean <= 1.0 and mx <= 12, (mean, mx)
    assert ops.error_flag() == 0
