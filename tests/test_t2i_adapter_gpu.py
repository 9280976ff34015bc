"""GPU tests of the SDXL T2I-Adapter: the three new kernels bit for bit against torch, every adapter layer against an
fp64 reference of the fp16 input it saw, the UNet + adapter step against the fp32 CPU oracle (oracle/t2i_adapter.py),
the plain step left untouched, and batch invariance of whole transitions.

Bounds are built as in tests/test_fp16_bounds_gpu.py: ULP = 2^-10 |ref| per fp16 rounding of the result, ACC =
2^-16 sum|a||w| (with |bias| and |res| added: they join the fp32 sum) for fp32 accumulation, TINY = 2^-24."""
import dataclasses
import gc
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

ULP, ACC, TINY = 2.0 ** -10, 2.0 ** -16, 2.0 ** -24
D = torch.float64
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SDXL_CHANNELS = (320, 640, 1280, 1280)


def check(got, ref, bound, what):
    got, ref = got.to(D), ref.to(D)
    err = (got - ref).abs()
    err = torch.where(torch.isnan(err), torch.full_like(err, float("inf")), err)
    ratio = err / bound
    r = float(ratio.max())
    assert r <= 1.0, f"{what}: {int((ratio > 1).sum())} of {ref.numel()} elements exceed the bound, worst {r:.3g}x"
    return r


def _image(H, W, C, seed):
    """A uint8 control image with edges and smooth regions (a canny / depth-like map is neither noise nor flat)."""
    g = torch.Generator().manual_seed(seed)
    yy, xx = torch.meshgrid(torch.arange(H), torch.arange(W), indexing="ij")
    base = ((xx * 255) // max(W - 1, 1)).to(torch.int64)
    edges = ((yy // 37 + xx // 53) % 2) * 120
    img = (base[..., None] + edges[..., None] + torch.randint(0, 40, (H, W, C), generator=g)) % 256
    return img.to(torch.uint8)


def _err_flag_clear():
    from latentblending_b200 import ops
    torch.cuda.synchronize()
    assert ops.error_flag() == 0


# ---- 1. the kernels, bit for bit ---------------------------------------------------------------------------------
@pytest.mark.parametrize("B", [1, 2, 4, 8])
def test_add_rows_bcast_matches_torch(B):
    """dst (a column slice of a wider concat buffer) += src (a strided view) broadcast over B rows: torch's fp16 +=."""
    from latentblending_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(B)
    rows, C = 45 * 80, 640
    big = (torch.randn(B * rows, 1280 + C, generator=g, device="cuda") * 3).half()
    src_big = (torch.randn(rows, C + 64, generator=g, device="cuda") * 2).half()
    dst, src = big[:, 1280:], src_big[:, 32:32 + C]
    want = (dst.reshape(B, rows, C) + src[None]).reshape(B * rows, C)
    keep = big[:, :1280].clone()
    ops.add_rows_bcast(dst, src, B)
    _err_flag_clear()
    assert torch.equal(dst, want)
    assert torch.equal(big[:, :1280], keep)


@pytest.mark.parametrize("cimg", [1, 3])
@pytest.mark.parametrize("H,W", [(1024, 1024), (720, 1280)])
def test_pixel_unshuffle_u8_matches_torch(cimg, H, W):
    from latentblending_b200 import ops
    img = _image(H, W, cimg, seed=H + cimg).cuda()
    out = ops.pixel_unshuffle_u8(img, 16)
    x = (img.float() / 255.0).half().permute(2, 0, 1)[None]
    ref = F.pixel_unshuffle(x, 16).permute(0, 2, 3, 1).reshape(-1, cimg * 256)     # columns c*256 + i*16 + j
    M = (H // 16) * (W // 16)
    got = out.view(M, 256, cimg).permute(0, 2, 1).reshape(M, cimg * 256)           # undo the (i, j, c) order
    _err_flag_clear()
    assert torch.equal(got, ref)


@pytest.mark.parametrize("H,W,C,strided", [(64, 64, 320, False), (45, 80, 640, False), (45, 80, 640, True),
                                           (23, 41, 64, True), (1, 1, 8, False)])
def test_avgpool2_ceil_matches_torch(H, W, C, strided):
    from latentblending_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(H * W)
    base = (torch.randn(H * W, C + (128 if strided else 0), generator=g, device="cuda") * 4).half()
    x = base[:, 64:64 + C] if strided else base
    out = ops.avgpool2_ceil(x, H, W, C)
    ref = F.avg_pool2d(x.reshape(1, H, W, C).permute(0, 3, 1, 2), 2, 2, ceil_mode=True)
    ref = ref.permute(0, 2, 3, 1).reshape(-1, C)
    _err_flag_clear()
    assert out.shape == ref.shape == (((H + 1) // 2) * ((W + 1) // 2), C)
    assert torch.equal(out, ref)


# ---- 2. every adapter layer against fp64 --------------------------------------------------------------------------
def _conv_ref(x_rows, h, w, cin, wt, b, k):
    """fp64 conv of the fp16 rows x [h*w, cin] with weights wt [Cout, cin, k, k]: (ref, sum|a||w| + |b|) as rows."""
    xn = x_rows.reshape(1, h, w, cin).permute(0, 3, 1, 2).to(D)
    ref = F.conv2d(xn, wt.to(D), b.to(D), padding=k // 2)
    mag = F.conv2d(xn.abs(), wt.to(D).abs(), b.to(D).abs(), padding=k // 2)
    return (t.permute(0, 2, 3, 1).reshape(h * w, -1) for t in (ref, mag))


@pytest.mark.parametrize("cin,H,W", [(3, 1024, 1024), (1, 720, 1280)])
def test_adapter_layers_bound(cin, H, W):
    """The feature program AdapterB200.compute records, replayed layer by layer with the eager ops on the same packed
    weights (which must give the program's bits), each layer within its fp64 bound."""
    from latentblending_b200 import ops
    from latentblending_b200.pipe import random_adapter_state_dict
    from latentblending_b200.t2i_adapter import AdapterB200, body_layout
    cfg = dict(in_channels=cin, channels=SDXL_CHANNELS, num_res_blocks=2, downscale_factor=16,
               adapter_type="full_adapter_xl")
    sd = random_adapter_state_dict(cfg, 7, "cuda:0")
    ad = AdapterB200(cfg, sd, "cuda:0")
    img = _image(H, W, cin, seed=W).cuda()
    feats = [f.clone() for f in ad.compute(img, H // 8, W // 8, 1.0)]
    Wt = ad.packed.w
    worst = []
    hh, ww = H // 16, W // 16
    xu = ops.pixel_unshuffle_u8(img, 16)
    c0 = SDXL_CHANNELS[0]
    x = ops.gemm(xu, Wt["conv_in.w"], c0, 1, hh, ww, taps=9, bias=Wt["conv_in.b"])
    wt = Wt["conv_in.w"].view(c0, 3, 3, 256 * cin).permute(0, 3, 1, 2)          # in the kernel's (i, j, c) order
    ref, mag = _conv_ref(xu, hh, ww, 256 * cin, wt, Wt["conv_in.b"], 3)
    worst.append(check(x, ref, ULP * ref.abs() + ACC * mag + TINY, "conv_in"))
    for i, (ci, co, down) in enumerate(body_layout(SDXL_CHANNELS)):
        if down:
            x = ops.avgpool2_ceil(x, hh, ww, ci)
            hh, ww = (hh + 1) // 2, (ww + 1) // 2
        if ci != co:
            y = ops.gemm(x, Wt[f"{i}.in_conv.w"], co, 1, 1, hh * ww, bias=Wt[f"{i}.in_conv.b"])
            ref, mag = _conv_ref(x, hh, ww, ci, Wt[f"{i}.in_conv.w"][:, :, None, None], Wt[f"{i}.in_conv.b"], 1)
            worst.append(check(y, ref, ULP * ref.abs() + ACC * mag + TINY, f"body.{i}.in_conv"))
            x = y
        for j in range(2):
            w1, b1 = Wt[f"{i}.{j}.block1.w"], Wt[f"{i}.{j}.block1.b"]
            h1 = ops.gemm(x, w1, co, 1, hh, ww, taps=9, bias=b1, relu=True)
            ref, mag = _conv_ref(x, hh, ww, co, w1.view(co, 3, 3, co).permute(0, 3, 1, 2), b1, 3)
            ref = ref.clamp(min=0)
            worst.append(check(h1, ref, ULP * ref.abs() + ACC * mag + TINY, f"body.{i}.{j}.block1+relu"))
            w2, b2 = Wt[f"{i}.{j}.block2.w"], Wt[f"{i}.{j}.block2.b"]
            y = ops.gemm(h1, w2, co, 1, 1, hh * ww, bias=b2, res=x)
            ref, mag = _conv_ref(h1, hh, ww, co, w2[:, :, None, None], b2, 1)
            ref, mag = ref + x.to(D), mag + x.to(D).abs()
            worst.append(check(y, ref, ULP * ref.abs() + ACC * mag + TINY, f"body.{i}.{j}.block2+x"))
            x = y
        assert torch.equal(x, feats[i]), f"body.{i}: the eager chain differs from the feature program"
    _err_flag_clear()
    print(f"adapter layers {cin}ch {H}x{W}: worst err/bound {[f'{r:.2f}' for r in worst]}")


# ---- 3. UNet + adapter against the oracle ------------------------------------------------------------------------
_TINY = {}


def _ucfg(ocfg):
    from latentblending_b200.unet import UNetConfig
    return UNetConfig(**{f.name: getattr(ocfg, f.name) for f in dataclasses.fields(ocfg)})


def _tiny_pair(cin=3):
    if cin not in _TINY:
        from latentblending_b200.t2i_adapter import AdapterB200
        from latentblending_b200.unet import UNetB200
        from oracle.sdxl_unet import SDXLUNet, synthetic_init_, tiny_config
        from oracle.t2i_adapter import T2IAdapter, synthetic_init_adapter_
        ocfg = tiny_config()
        ch = tuple(ocfg.block_out_channels) + (ocfg.block_out_channels[-1],)
        unet = synthetic_init_(SDXLUNet(ocfg), seed=0).eval()
        oad = synthetic_init_adapter_(T2IAdapter(cin, ch), seed=1).eval()
        with torch.no_grad():
            for m in (unet, oad):
                for p in m.parameters():
                    p.copy_(p.half().float())
        acfg = dict(in_channels=cin, channels=ch, num_res_blocks=2, downscale_factor=16, adapter_type="full_adapter_xl")
        ad = AdapterB200(acfg, oad.state_dict(), "cuda:0")
        ucfg = _ucfg(ocfg)
        _TINY[cin] = dict(unet=unet, oad=oad, ad=ad, net=UNetB200(ucfg, unet.state_dict(), "cuda:0", adapter=ad),
                          plain=UNetB200(ucfg, unet.state_dict(), "cuda:0"), cfg=ocfg)
    return _TINY[cin]


def _inputs(cfg, B, h, w, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, 4, h, w, generator=g).half()
    ctx = (torch.randn(B, 77, cfg.cross_attention_dim, generator=g) * 0.5).half()
    pooled = torch.randn(B, cfg.pooled_dim, generator=g).half()
    tids = torch.tensor([[8.0 * h, 8.0 * w, 0, 0, 8.0 * h, 8.0 * w]] * B).half()
    return x, ctx, pooled, tids


@pytest.mark.parametrize("cin,B,h,w,scale", [(3, 1, 16, 16, 1.0), (3, 2, 16, 16, 0.6), (3, 2, 18, 26, 1.0),
                                             (1, 1, 32, 16, 0.6), (1, 3, 18, 26, 0.8)])
def test_tiny_unet_adapter_matches_oracle(cin, B, h, w, scale):
    """Latents 18 x 26 give a 144 x 208 image: features 9 x 13 and, after the ceil-mode pool, 5 x 7."""
    from oracle.t2i_adapter import adapter_states, image_to_adapter_input, unet_with_adapter
    p = _tiny_pair(cin)
    x, ctx, pooled, tids = _inputs(p["cfg"], B, h, w, seed=B + h)
    img = _image(8 * h, 8 * w, cin, seed=h + w)
    t = 611.0
    with torch.no_grad():
        states = adapter_states(p["oad"], image_to_adapter_input(img), scale)
        ref = unet_with_adapter(p["unet"], x.float(), t, ctx.float(), pooled.float(), tids.float(), states)
        plain_ref = unet_with_adapter(p["unet"], x.float(), t, ctx.float(), pooled.float(), tids.float())
    p["ad"].compute(img.cuda(), h, w, scale)
    eps = p["net"].forward(x.cuda(), t, ctx.cuda(), pooled.cuda(), tids.cuda(), adapter=True).float().cpu()
    _err_flag_clear()
    rel = ((eps - ref).norm() / ref.norm()).item()
    effect = ((ref - plain_ref).norm() / ref.norm()).item()
    print(f"unet+adapter {cin}ch B={B} {h}x{w} scale={scale}: rel_l2={rel:.3e} (adapter changes eps by {effect:.3e})")
    assert effect > 5e-3                   # the comparison is not vacuous
    assert rel <= 2e-3, f"relative L2 error {rel}"


@pytest.mark.slow
def test_full_sdxl_adapter_matches_fixture():
    """The full SDXL-base UNet with an RGB SDXL T2I-Adapter, CFG batch 2 at 128x128 with a 1024x1024 image at scale
    0.8, against the committed fp32 oracle fixture (tests/golden/make_t2i_adapter_fixtures.py)."""
    from latentblending_b200.t2i_adapter import AdapterB200
    from latentblending_b200.unet import UNetB200
    from make_t2i_adapter_fixtures import FIXTURE, SCALE, T, adapter_image, inputs, oracle_adapter
    from make_fullsize_fixtures import oracle_unet, weights_checksum
    from oracle.sdxl_unet import SDXL_BASE
    fx = np.load(FIXTURE)
    unet, oad = oracle_unet(), oracle_adapter()
    assert weights_checksum(unet.state_dict()) + weights_checksum(oad.state_dict()) == str(fx["weights_sha1"])
    acfg = dict(in_channels=3, channels=SDXL_CHANNELS, num_res_blocks=2, downscale_factor=16,
                adapter_type="full_adapter_xl")
    ad = AdapterB200(acfg, oad.state_dict(), "cuda:0")
    net = UNetB200(_ucfg(SDXL_BASE), unet.state_dict(), "cuda:0", adapter=ad)
    del unet, oad
    gc.collect()
    x, ctx, pooled, tids = inputs()
    ad.compute(adapter_image().cuda(), 128, 128, SCALE)
    eps = net.forward(x.cuda(), T, ctx.cuda(), pooled.cuda(), tids.cuda(), adapter=True).float().cpu()
    _err_flag_clear()
    ref = torch.from_numpy(fx["eps"])
    rel = ((eps - ref).norm() / ref.norm()).item()
    print(f"full SDXL UNet + T2I-Adapter @128x128 B=2: rel_l2={rel:.3e} (the adapter changes eps by "
          f"{float(fx['effect']):.3e})")
    assert rel <= 2e-3


# ---- 4. nothing else changes --------------------------------------------------------------------------------------
def _signature(prog):
    return [(op.kind, op.dtype) for op in prog.ops], prog.num_launches, prog.work()


def test_plain_step_program_is_untouched():
    """With an adapter attached, the plain step program records the ops of a UNet without one and gives the same
    eps bit for bit; the adapter program is those very records with four in-place adds spliced in."""
    from latentblending_b200._cabi import OP_ADD_ROWS_BCAST
    p = _tiny_pair()
    x, ctx, pooled, tids = _inputs(p["cfg"], 2, 16, 24, seed=4)
    pl, ref = p["net"].plan(2, 16, 24), p["plain"].plan(2, 16, 24)
    assert _signature(pl.prog_step) == _signature(ref.prog_step)
    plain = p["plain"].forward(x.cuda(), 300.0, ctx.cuda(), pooled.cuda(), tids.cuda()).clone()
    with_ad = p["net"].forward(x.cuda(), 300.0, ctx.cuda(), pooled.cuda(), tids.cuda()).clone()
    assert torch.equal(plain, with_ad)
    ad_ops = pl.prog_step_ad.ops
    assert pl.prog_step_ad.num_launches == pl.prog_step.num_launches + 4
    assert len(ad_ops) == len(pl.prog_step.ops) + 4
    assert all(a is b for a, b in zip([op for op in ad_ops if op.kind != OP_ADD_ROWS_BCAST], pl.prog_step.ops))
    assert sum(op.kind == OP_ADD_ROWS_BCAST for op in ad_ops) == 4
    _err_flag_clear()


def _tiny_holder(seed=3, guidance=4.0, adapter="rgb", size=(192, 128)):
    from latentblending_b200 import DiffusersHolder, SyntheticSDXLPipe
    from oracle.sdxl_unet import tiny_config
    pp = SyntheticSDXLPipe("synthetic/sdxl-base-tiny", "cuda:0", unet_cfg=_ucfg(tiny_config()), seed=seed, vae="tiny",
                           adapter=adapter)
    dh = DiffusersHolder(pp)
    dh.guidance_scale = guidance
    dh.set_dimensions(size)
    dh.set_num_inference_steps(6)
    return dh


def test_inactive_adapter_gives_the_plain_latents():
    """Scale 0, factor 0 and set_adapter_image(None) give latents bit-identical to a holder that never had an image,
    with the same launch count; a factor of 0.5 runs the adapter program at steps 0-2 and changes every latent."""
    from latentblending_b200 import program
    dh = _tiny_holder()
    emb = dh.get_text_embedding("a lake")
    start = dh.get_noise(5)
    img = _image(256, 256, 3, seed=1).numpy()

    def run():
        l0 = program.LAUNCHES[0]
        out = dh.run_diffusion_sd_xl(emb, start)
        torch.cuda.synchronize()
        return [t.clone() for t in out], program.LAUNCHES[0] - l0

    for dual in (True, False):
        dh.dual_stream = dual
        never, n_never = run()
        for kw in (dict(conditioning_scale=0.0), dict(conditioning_factor=0.0)):
            dh.set_adapter_image(img, **kw)
            off, n_off = run()
            assert n_off == n_never and all(torch.equal(a, b) for a, b in zip(off, never)), kw
        dh.set_adapter_image(img, 0.8, conditioning_factor=0.5)                # steps 0, 1, 2 of 6
        half, n_half = run()
        assert n_half - n_never == 3 * 4 * (2 if dual else 1)
        assert all(not torch.equal(a, b) for a, b in zip(half, never))
        dh.set_adapter_image(None)
        back, n_back = run()
        assert n_back == n_never and all(torch.equal(a, b) for a, b in zip(back, never))
    _err_flag_clear()


def test_adapter_image_checks():
    from latentblending_b200 import DiffusersHolder, SyntheticSDXLPipe
    from oracle.sdxl_unet import tiny_config
    dh = DiffusersHolder(SyntheticSDXLPipe("synthetic/sdxl-base-tiny", "cuda:0", unet_cfg=_ucfg(tiny_config()),
                                           vae="tiny"))
    with pytest.raises(ValueError):
        dh.set_adapter_image(_image(64, 64, 3, 0).numpy())            # no adapter
    gray = _tiny_holder(adapter="gray", size=(200, 128))               # 200 is not a multiple of 16
    with pytest.raises(ValueError, match="multiples of 16"):
        gray.set_adapter_image(_image(64, 64, 1, 0)[..., 0].numpy())
    gray.set_dimensions((208, 128))
    gray.set_adapter_image(_image(64, 64, 3, 0).numpy())               # an RGB image is converted to "L"
    assert (gray.height_latent, gray.width_latent) in gray.adapter_cond["computed"]
    _err_flag_clear()


# ---- 5. batch invariance of whole transitions --------------------------------------------------------------------
def _fingerprint(be):
    sys.path.insert(0, ROOT)
    from bench import tree_fingerprint
    return tree_fingerprint(be)


def _transition(pp, size, steps, branches, width, dual, img, scale=0.8, factor=0.75):
    from latentblending_b200 import BlendingEngine
    be = BlendingEngine(pp, run_benchmark=False)
    be.set_dimensions(size)
    be.set_num_inference_steps(steps)
    be.set_prompt1("photo of a lake")
    be.set_prompt2("alien planet")
    be.set_branching(depth_strength=0.5, nmb_max_branches=branches)
    be.speculative_batch = width
    be.deterministic_noise = True
    be.output_device_frames = True
    be.dh.dual_stream = dual
    be.set_adapter_image(img, scale, factor)
    be.run_transition(fixed_seeds=[7, 8])
    torch.cuda.synchronize()
    fp = _fingerprint(be)
    del be
    gc.collect()                # each engine holds its own packed UNet + adapter
    torch.cuda.empty_cache()
    return fp


@pytest.mark.parametrize("turbo", [True, False])
def test_transition_fingerprint_is_batch_invariant(turbo):
    """A full-size synthetic SDXL transition with an adapter image (512^2 Turbo; 1024^2 base under CFG): the tree is
    the same with lockstep speculation width 1 and 4 (Turbo) or 2 (base, with dual-stream CFG halves on and off)."""
    from latentblending_b200 import SyntheticSDXLPipe
    name = "stabilityai/sdxl-turbo" if turbo else "stabilityai/stable-diffusion-xl-base-1.0"
    pp = SyntheticSDXLPipe(name, "cuda:0", seed=0, vae="tiny", adapter="rgb")
    size = (512, 512) if turbo else (1024, 1024)
    img = _image(size[1], size[0], 3, seed=3).numpy()
    steps, branches = (4, 6) if turbo else (5, 6)
    fps = {}
    for width in (1, 4 if turbo else 2):
        for dual in ((True,) if turbo else (True, False)):
            fps[(width, dual)] = _transition(pp, size, steps, branches, width, dual, img)
    print(f"t2i-adapter transition fingerprints {'turbo' if turbo else 'base'}: {fps}")
    assert len(set(fps.values())) == 1
    _err_flag_clear()
