"""GPU tests of the bf16 VAE decoder: the bf16 wgmma GEMM / implicit-GEMM conv (LB_GEMM_BF16, LB_GEMM_OUT_F16), the
bf16 variants of the other decoder ops, the whole decoder on weights whose activations overflow fp16
(tests/golden/make_upcast_fixtures.py) against the fp32 oracle, and the engine choosing it.

GEMM tolerance (stated): against an fp64 product of the same bf16 operands,
    |got - ref| <= 2^-8 |ref| + 2^-16 (|a| |w|^T)
-- the bf16 output rounding (half an ulp, 2^-9 relative) with margin, plus fp32 accumulation in a different order
(K <= 4608 terms: far below 2^-16 of the absolute sum).  Frame tolerance: mean <= 1.0 and max <= 12 uint8 levels, as
tests/test_vae_gpu.py."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

BF = torch.bfloat16


def _rand(*shape, seed=0, s=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(*shape, generator=g, device="cuda") * s


def _check(got, ref, absprod, what=""):
    got, ref = got.double(), ref.double()
    assert torch.isfinite(got).all(), what
    err = (got - ref).abs()
    bound = 2.0 ** -8 * ref.abs() + 2.0 ** -16 * absprod
    assert (err <= bound).all(), (what, (err - bound).max().item())


def _linear_ref(a, w, bias=None, res=None):
    ref = a.double() @ w.double().T
    absprod = a.double().abs() @ w.double().abs().T
    if bias is not None:
        ref += bias.double()
    if res is not None:
        ref += res.double()
    return ref, absprod


def _conv_ref(x_nhwc, w_oihw, B, H, W, bias=None):
    x = x_nhwc.double().view(B, H, W, -1).permute(0, 3, 1, 2)
    ref = F.conv2d(x, w_oihw.double(), padding=1)
    absprod = F.conv2d(x.abs(), w_oihw.double().abs(), padding=1)
    if bias is not None:
        ref += bias.double()[None, :, None, None]
    flat = lambda t: t.permute(0, 2, 3, 1).reshape(B * H * W, -1)
    return flat(ref), flat(absprod)


def _pack3(w_oihw):
    return w_oihw.permute(0, 2, 3, 1).reshape(w_oihw.shape[0], -1).contiguous()


# ---- GEMM ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M,K,N", [(1000, 512, 64), (777, 512, 384), (2048, 1024, 320), (300, 128, 8)])
def test_bf16_linear(M, K, N):
    """N = 64 / 384 / 320 / 8 run the 64 / 128 / 160 / 64-wide N tiles."""
    from latentblending_b200 import ops
    a = _rand(M, K, seed=1).to(BF)
    w = (_rand(N, K, seed=2) * K ** -0.5).to(BF)
    b = (_rand(N, seed=3) * 0.1).to(BF)
    out = ops.gemm(a, w, N, 1, 1, M, bias=b)
    assert out.dtype == BF
    _check(out, *_linear_ref(a, w, b), what="linear")
    _check(ops.gemm(a, w, N, 1, 1, M, bias=b, static_w=True), *_linear_ref(a, w, b), what="static_w")


def test_bf16_linear_residual_in_place_and_large_outputs():
    """+ residual, also written over the residual itself; outputs ~10^6 (past fp16's range) stay finite and exact
    to the stated bound."""
    from latentblending_b200 import ops
    M, K, N = 1500, 512, 512
    a = (_rand(M, K, seed=4) * 3e3).to(BF)
    w = (_rand(N, K, seed=5) * K ** -0.5 * 30).to(BF)
    b = (_rand(N, seed=6) * 1e4).to(BF)
    res = (_rand(M, N, seed=7) * 1e6).to(BF)
    ref, absprod = _linear_ref(a, w, b, res)
    assert ref.abs().max() > 1e6
    sep = ops.gemm(a, w, N, 1, 1, M, bias=b, res=res.clone())
    _check(sep, ref, absprod + res.double().abs(), "residual")
    hs = res.clone()
    ops.gemm(a, w, N, 1, 1, M, bias=b, res=hs, out=hs)
    assert torch.equal(hs, sep)


@pytest.mark.parametrize("B,H,W,Cin,Cout", [(1, 17, 11, 64, 128), (1, 104, 152, 128, 128), (2, 16, 16, 128, 320)])
def test_bf16_conv3x3_box_and_runs(B, H, W, Cin, Cout):
    """3x3 implicit-GEMM conv through both M tilings (bf16 TMA box and im2col loads): bit-identical to each other,
    within the bound of the fp64 convolution."""
    from latentblending_b200 import ops
    x = _rand(B * H * W, Cin, seed=8).to(BF)
    w = (_rand(Cout, Cin, 3, 3, seed=9) * (9 * Cin) ** -0.5).to(BF)
    b = (_rand(Cout, seed=10) * 0.1).to(BF)
    outs = {}
    for t in ("box", "runs", "auto"):
        if t == "box" and W < 128 and (W & (W - 1)):
            continue
        outs[t] = ops.gemm(x, _pack3(w), Cout, B, H, W, taps=9, bias=b, tiling=t)
    for t, o in outs.items():
        assert torch.equal(o, outs["runs"]), t
    _check(outs["runs"], *_conv_ref(x, w, B, H, W, b), what="conv")


def test_bf16_conv_with_shortcut_segment():
    """conv2 + the resnet's 1x1 shortcut as a second K segment (a1), the VAE's channel-changing resnets."""
    from latentblending_b200 import ops
    B, H, W, Cin, Cout = 1, 24, 20, 128, 64
    h = _rand(B * H * W, Cout, seed=11).to(BF)
    xin = _rand(B * H * W, Cin, seed=12).to(BF)
    w = (_rand(Cout, Cout, 3, 3, seed=13) * (9 * Cout) ** -0.5).to(BF)
    ws = (_rand(Cout, Cin, seed=14) * Cin ** -0.5).to(BF)
    b = (_rand(Cout, seed=15) * 0.1).to(BF)
    out = ops.gemm(h, torch.cat([_pack3(w), ws], 1).contiguous(), Cout, B, H, W, taps=9, a1=xin, bias=b)
    ref, absprod = _conv_ref(h, w, B, H, W, b)
    r2, a2 = _linear_ref(xin, ws)
    _check(out, ref + r2, absprod + a2, "shortcut")


def test_bf16_long_k_cooperative_tile():
    """512 -> 512 3x3 conv at 132x132 (K = 4608, >= 2 tiles per SM): the 256-wide cooperative N tile."""
    from latentblending_b200 import ops
    B, H, W, C = 1, 132, 132, 512
    x = _rand(B * H * W, C, seed=16).to(BF)
    w = (_rand(C, C, 3, 3, seed=17) * (9 * C) ** -0.5).to(BF)
    b = (_rand(C, seed=18) * 0.1).to(BF)
    out = ops.gemm(x, _pack3(w), C, B, H, W, taps=9, bias=b, static_w=True)
    _check(out, *_conv_ref(x, w, B, H, W, b), what="bn256")


def test_bf16_operands_fp16_output():
    """LB_GEMM_OUT_F16: the attention-score GEMM (activation as B operand), fp16 rounding of the fp32 sums."""
    from latentblending_b200 import ops
    S, C = 187, 512
    q = _rand(192, C, seed=19).to(BF)
    k = _rand(192, C, seed=20).to(BF)
    out = ops.gemm(q[:S], k, 192, 1, 1, S, out_dtype=torch.float16)
    assert out.dtype == torch.float16
    ref, absprod = _linear_ref(q[:S], k)
    err = (out.double() - ref).abs()
    assert (err <= 2.0 ** -11 * ref.abs() + 2.0 ** -16 * absprod + 2.0 ** -24).all()


def test_bf16_gemm_rejections():
    from latentblending_b200 import _cabi, ops
    a = _rand(256, 128, seed=21).to(BF)
    w = _rand(256, 128, seed=22).to(BF)
    with pytest.raises(_cabi.LB200Error, match="GEGLU"):
        ops.gemm(a, w, 256, 1, 1, 256, mode=1)
    st = torch.zeros(256, 32, 2, device="cuda")
    with pytest.raises(_cabi.LB200Error, match="stats_out"):
        ops.gemm(a, w, 256, 1, 1, 256, stats_out=st)
    ln = dict(stats=st, csum=torch.zeros(256, device="cuda"), bias=torch.zeros(256, device="cuda"), eps=1e-5)
    with pytest.raises(_cabi.LB200Error, match="LayerNorm"):
        ops.gemm(a, w, 256, 1, 1, 256, ln=ln)
    with pytest.raises(_cabi.LB200Error, match="mixed"):
        ops.gemm(a.half(), w, 256, 1, 1, 256)
    with pytest.raises(_cabi.LB200Error, match="mixed"):
        ops.gemm(a, w, 256, 1, 1, 256, bias=torch.zeros(256, device="cuda", dtype=torch.float16))
    # OUT_F16 without BF16, straight through the C ABI
    a16, w16 = a.half(), w.half()
    out = torch.empty(256, 256, dtype=torch.float16, device="cuda")
    d = _cabi.GemmDesc()
    d.a0, d.a0_ld, d.a0_c = a16.data_ptr(), 128, 128
    d.B, d.H, d.W, d.taps = 1, 1, 256, 1
    d.w, d.w_ld, d.N = w16.data_ptr(), 128, 256
    d.out, d.out_ld, d.mode = out.data_ptr(), 256, _cabi.GEMM_OUT_F16
    lib = _cabi.load()
    assert lib.lb_gemm(_cabi.ctx(0), d, _cabi.stream_ptr()) != 0
    assert b"OUT_F16" in lib.lb_last_error()
    d.mode = 0x4000                                   # unknown flags are still rejected
    assert lib.lb_gemm(_cabi.ctx(0), d, _cabi.stream_ptr()) != 0


# ---- the other decoder ops -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("silu", [0, 1])
def test_bf16_groupnorm_large_inputs(silu):
    """GroupNorm(32) +- SiLU on activations of magnitude 1e5-1e6 (fp16 would overflow) vs fp32 torch of the same bf16
    input.  Bound: the bf16 rounding of the affine result (2^-9 relative, carried through SiLU, whose slope is <= 1.1)
    and of the output, with margin: 2^-8 (1.1 |affine| + |out|) + 2^-10 absolute on the normalised scale."""
    from latentblending_b200 import ops
    HW, C = 37 * 29, 512
    x = (_rand(HW, C, seed=23) * 2e5 + 6e5).to(BF)
    g = (1 + 0.1 * _rand(C, seed=24)).to(BF)
    b = (0.1 * _rand(C, seed=25)).to(BF)
    out = ops.groupnorm(x, 1, HW, C, 32, g, b, 1e-6, silu)
    assert out.dtype == BF and torch.isfinite(out.float()).all()
    pre = F.group_norm(x.float().T[None], 32, g.float(), b.float(), 1e-6)[0].T
    ref = F.silu(pre) if silu else pre
    err = (out.float() - ref).abs()
    assert (err <= 2.0 ** -8 * (1.1 * pre.abs() + ref.abs()) + 2.0 ** -10).all(), err.max().item()


def test_bf16_softmax_fp16_scores_with_tail():
    """fp16 scores in, bf16 P out, 187 columns (23 vectors + a 3-column scalar tail), in place as the decoder runs it."""
    from latentblending_b200 import ops
    rows, cols = 190, 187
    buf = torch.zeros(rows, 192, dtype=torch.float16, device="cuda")
    buf[:, :cols] = (_rand(rows, cols, seed=26) * 6).half()
    ref = torch.softmax(buf[:, :cols].float(), dim=1)
    out = ops.softmax_rows(buf[:, :cols], out=buf.view(BF)[:, :cols])
    got = out.float()
    assert ((got - ref).abs() <= 2.0 ** -8 * ref + 1e-6).all()
    src = torch.zeros(rows, 192, dtype=torch.float16, device="cuda")
    src[:, :cols] = (_rand(rows, cols, seed=26) * 6).half()
    sep = torch.empty(rows, 192, dtype=BF, device="cuda")
    ops.softmax_rows(src[:, :cols], out=sep[:, :cols])                   # out of place: the same values
    assert torch.equal(sep[:, :cols], out)


def test_bf16_upsample_is_exact():
    from latentblending_b200 import ops
    for (H, W, Ho, Wo) in ((9, 6, 17, 11), (8, 8, 16, 16)):
        x = _rand(H * W, 128, seed=27).to(BF)
        out = ops.upsample_nearest(x, 1, H, W, 128, Ho, Wo)
        ref = F.interpolate(x.view(1, H, W, 128).permute(0, 3, 1, 2).float(), size=(Ho, Wo), mode="nearest")
        assert out.dtype == BF and torch.equal(out.float(), ref.permute(0, 2, 3, 1).reshape(Ho * Wo, 128))


def test_bf16_latent_prep_conv_in_nhwc_to_nchw():
    from latentblending_b200 import ops
    h, w = 13, 10
    lat = (_rand(1, 4, h, w, seed=28) * 0.8).half()
    wp = _rand(4, 4, seed=29) / 0.13025
    bp = _rand(4, seed=30) * 0.1
    z = ops.latent_prep(lat, wp, bp, out_dtype=BF)
    zref = torch.einsum("oc,bchw->bohw", wp, lat.float()) + bp[None, :, None, None]
    assert z.dtype == BF and ((z.float() - zref).abs() <= 2.0 ** -8 * zref.abs() + 1e-6).all()
    wc = (_rand(128, 4, 3, 3, seed=31) * 65536 / 6).to(BF)             # conv_in weights scaled like the fixture
    bc = (_rand(128, seed=32) * 1000).to(BF)
    x = ops.conv_in(z, wc.permute(2, 3, 1, 0).contiguous(), bc, 128)
    ref = F.conv2d(z.double(), wc.double(), bc.double(), padding=1)
    absprod = F.conv2d(z.double().abs(), wc.double().abs(), padding=1) + bc.double().abs()[None, :, None, None]
    flat = lambda t: t.permute(0, 2, 3, 1).reshape(h * w, -1)
    _check(x, flat(ref), flat(absprod), "conv_in")
    rows = _rand(h * w, 8, seed=33).to(BF)
    nchw = ops.nhwc_to_nchw(rows, 1, 3, h, w)
    assert nchw.dtype == BF and torch.equal(nchw, rows[:, :3].T.reshape(1, 3, h, w))


def test_bf16_postprocess_counts_nonfinite():
    from latentblending_b200 import ops
    img = (_rand(1, 3, 16, 24, seed=34) * 0.7).to(BF)
    img[0, 1, 3, 5] = float("inf")
    img[0, 2, 7, 7] = float("nan")
    img[0, 0, 0, 0] = -float("inf")
    cnt = torch.zeros(1, dtype=torch.int32, device="cuda")
    out = ops.postprocess_u8(img, nonfinite=cnt)
    assert int(cnt.item()) == 3
    fin = img.float().clone()
    fin[~torch.isfinite(fin)] = 0
    ref = ((fin / 2 + 0.5).clamp(0, 1) * 255).round().to(torch.uint8).permute(0, 2, 3, 1)
    mask = torch.isfinite(img.float()).all(1)[:, :, :, None].expand_as(ref)
    assert torch.equal(out[mask], ref[mask])


def test_program_rejects_bf16_on_fp16_only_kinds():
    from latentblending_b200 import _cabi
    from latentblending_b200.program import Program
    x = torch.zeros(64, 64, dtype=torch.float16, device="cuda")
    g = torch.ones(64, dtype=torch.float16, device="cuda")
    for build in (lambda P: P.layernorm(x, g, g, 1e-5, x),
                  lambda P: P.attention(x, x, x, x, 1, 1, 64, 64)):
        P = Program(0)
        build(P)
        P.ops[0].dtype = _cabi.DTYPE_BF16
        with pytest.raises(_cabi.LB200Error, match="dtype"):
            P.finalize()
    P = Program(0)
    P.layernorm(x, g, g, 1e-5, x)
    P.ops[0].dtype = 2                                  # not a dtype at all
    with pytest.raises(_cabi.LB200Error, match="dtype"):
        P.finalize()


# ---- the whole decoder -----------------------------------------------------------------------------------------------
def _frame_diff(got, ref):
    d = np.abs(got.astype(np.int32) - ref.astype(np.int32))
    return d.mean(), d.max()


def _tiny_upcast(scaled=True):
    from make_upcast_fixtures import upcast_
    from oracle.vae import VAEConfig, VAEDecoder, synthetic_vae_init_
    cfg = VAEConfig(block_out_channels=(64, 64, 128, 128))
    ov = synthetic_vae_init_(VAEDecoder(cfg), seed=4).eval()
    with torch.no_grad():
        for p in ov.parameters():
            p.copy_(p.half().float())
    return (upcast_(ov) if scaled else ov), cfg


@pytest.mark.parametrize("h,w", [(16, 16), (17, 11)])
def test_bf16_decoder_on_overflowing_weights_matches_oracle(h, w):
    from latentblending_b200 import _cabi, ops
    from latentblending_b200.vae import VAEDecoderB200
    from make_fullsize_fixtures import vae_latent
    from oracle.vae import latent2image_np
    ov, cfg = _tiny_upcast()
    lat = vae_latent(h, w)
    with torch.no_grad():
        ref = latent2image_np(ov, lat)
    vae = VAEDecoderB200(ov.state_dict(), cfg.block_out_channels, cfg.scaling_factor, "cuda:0", dtype=BF)
    got = vae.decode_to_u8(lat.cuda()).cpu().numpy()
    mean, mx = _frame_diff(got, ref)
    print(f"bf16 decoder, scaled weights, {h}x{w}: mean |d| {mean:.3f} max {mx}")
    assert mean <= 1.0 and mx <= 12, (mean, mx)
    assert ref.std() > 5 and vae.overflow_count() == 0 and ops.error_flag() == 0
    # the fp16 decoder on the same weights overflows and says so
    v16 = VAEDecoderB200(ov.state_dict(), cfg.block_out_channels, cfg.scaling_factor, "cuda:0")
    v16.decode_to_u8(lat.cuda())
    with pytest.raises(_cabi.LB200Error, match="overflow.*set_vae_dtype"):
        v16.check_overflow()


def test_bf16_decoder_matches_upcast_fixture():
    """SDXL-width decoder at 64x64 latents vs the fp32 oracle frame of tests/golden/vae_sdxl_64_upcast.npz."""
    from latentblending_b200 import ops
    from latentblending_b200.vae import VAEDecoderB200
    from make_fullsize_fixtures import oracle_vae, vae_latent, weights_checksum
    from make_upcast_fixtures import FP16_MAX, UPCAST_FIXTURE, upcast_
    fx = np.load(UPCAST_FIXTURE)
    ov, cfg = oracle_vae()
    upcast_(ov)
    assert weights_checksum(ov.state_dict()) == str(fx["weights_sha1"]), "seeded VAE recipe drifted"
    assert float(fx["max_abs_activation"]) > FP16_MAX
    vae = VAEDecoderB200(ov.state_dict(), cfg.block_out_channels, cfg.scaling_factor, "cuda:0", dtype=BF)
    got = vae.decode_to_u8(vae_latent(64, 64).cuda()).cpu().numpy()
    mean, mx = _frame_diff(got, fx["frame"])
    print(f"bf16 SDXL-width decoder, upcast fixture: mean |d| {mean:.3f} max {mx}")
    assert mean <= 1.0 and mx <= 12, (mean, mx)
    assert vae.overflow_count() == 0 and ops.error_flag() == 0


def test_bf16_decoder_on_fp16_safe_weights_matches_fixture():
    from latentblending_b200.vae import VAEDecoderB200
    from make_fullsize_fixtures import VAE_FIXTURE, oracle_vae, vae_latent
    fx = np.load(VAE_FIXTURE)
    ov, cfg = oracle_vae()
    vae = VAEDecoderB200(ov.state_dict(), cfg.block_out_channels, cfg.scaling_factor, "cuda:0", dtype=BF)
    got = vae.decode_to_u8(vae_latent(64, 64).cuda()).cpu().numpy()
    mean, mx = _frame_diff(got, fx["frame"])
    print(f"bf16 SDXL-width decoder, unscaled weights: mean |d| {mean:.3f} max {mx}")
    assert mean <= 1.0 and mx <= 12, (mean, mx)


def test_bf16_decoder_at_1080p():
    from latentblending_b200 import ops
    from latentblending_b200.vae import VAEDecoderB200
    from make_fullsize_fixtures import oracle_vae, vae_latent
    from make_upcast_fixtures import upcast_
    ov, cfg = oracle_vae()
    upcast_(ov)
    vae = VAEDecoderB200(ov.state_dict(), cfg.block_out_channels, cfg.scaling_factor, "cuda:0", dtype=BF)
    frame = vae.decode_to_u8(vae_latent(135, 240).cuda())
    torch.cuda.synchronize()
    assert frame.shape == (1080, 1920, 3)
    assert ops.error_flag() == 0 and vae.overflow_count() == 0
    assert frame.float().std() > 5


def test_bf16_decoder_rejects_direct_conv_out(monkeypatch):
    from latentblending_b200 import _cabi
    from latentblending_b200.vae import VAEDecoderB200
    ov, cfg = _tiny_upcast()
    vae = VAEDecoderB200(ov.state_dict(), cfg.block_out_channels, cfg.scaling_factor, "cuda:0", dtype=BF)
    monkeypatch.setenv("LB_CONV_OUT_DIRECT", "1")
    with pytest.raises(_cabi.LB200Error, match="LB_CONV_OUT_DIRECT"):
        vae.plan(8, 8)


# ---- engine ----------------------------------------------------------------------------------------------------------
def _upcast_pipe(turbo, vae_dtype):
    from latentblending_b200 import SyntheticSDXLPipe
    from make_upcast_fixtures import CONV_IN_SCALE
    from test_engine_gpu import _pair
    op, pp, _ = _pair(turbo)
    sd = {k: v.clone() for k, v in pp.vae_state_dict.items()}
    sd["conv_in.weight"] = sd["conv_in.weight"] * CONV_IN_SCALE
    sd["conv_in.bias"] = sd["conv_in.bias"] * CONV_IN_SCALE
    with torch.no_grad():
        op.vae.conv_in.weight.mul_(CONV_IN_SCALE)
        op.vae.conv_in.bias.mul_(CONV_IN_SCALE)
    p2 = SyntheticSDXLPipe(pp._name_or_path, "cuda:0", unet_cfg=pp.unet_cfg, unet_state_dict=pp.unet_state_dict,
                           vae_state_dict=sd, vae_channels=pp.vae_channels, lpips_state_dict=pp.lpips_state_dict,
                           vae_dtype=vae_dtype)
    return op, p2


def _short_transition(be, turbo):
    be.set_dimensions((128, 128))
    be.set_num_inference_steps(4 if turbo else 6)
    be.set_prompt1("photo of a lake")
    be.set_prompt2("alien planet")
    be.set_branching(nmb_max_branches=3 if turbo else 4)
    return be.run_transition(fixed_seeds=[420, 421])


@pytest.mark.parametrize("turbo", [False, True])
def test_engine_transition_with_upcast_vae(turbo):
    from latentblending_b200 import BlendingEngine, _cabi
    from oracle.vae import latent2image_np
    op, pp = _upcast_pipe(turbo, "bf16")
    be = BlendingEngine(pp, run_benchmark=False)
    assert be.dh.vae.dtype == BF
    imgs = _short_transition(be, turbo)
    assert len(imgs) == len(be.tree_latents) >= 3
    for img, lat in zip(imgs, be.tree_latents):
        with torch.no_grad():
            ref = latent2image_np(op.vae, lat[-1].cpu())
        mean, mx = _frame_diff(np.asarray(img), ref)
        assert mean <= 1.0 and mx <= 12, (mean, mx)
    _, p16 = _upcast_pipe(turbo, "fp16")
    with pytest.raises(_cabi.LB200Error, match="overflow"):
        _short_transition(BlendingEngine(p16, run_benchmark=False), turbo)


def test_holder_from_diffusers_pipe_with_force_upcast_decodes_in_bf16():
    from latentblending_b200 import DiffusersHolder
    from test_boundary_cpu import MockDiffusersPipe
    mock = MockDiffusersPipe()                         # its VAE config sets force_upcast=True
    mock._execution_device = torch.device("cuda:0")
    dh = DiffusersHolder(mock)
    assert dh.vae_dtype == "bf16" and dh.vae.dtype == BF
    dh.set_vae_dtype("fp16")
    assert dh.vae.dtype == torch.float16
    with pytest.raises(ValueError):
        dh.set_vae_dtype("fp32")
