"""GPU tests of the SDXL ControlNet: the conditioning-embedding kernels against fp64 references per element, the
UNet + ControlNet step against the fp32 CPU oracle (oracle/controlnet.py), the plain step left untouched, batch
invariance of whole transitions, and the engine's set_control_image.

Bounds are built as in tests/test_fp16_bounds_gpu.py: ULP = 2^-10 |ref| per fp16 rounding of the result, ACC =
2^-16 sum|a||w| for fp32 accumulation, TINY = 2^-24, and SiLU's slope (<= 1.1) times the bound of its input."""
import dataclasses
import gc
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

ULP, ACC, TINY, SILU_SLOPE = 2.0 ** -10, 2.0 ** -16, 2.0 ** -24, 1.1
D = torch.float64
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def check(got, ref, bound, what):
    got, ref = got.to(D), ref.to(D)
    err = (got - ref).abs()
    err = torch.where(torch.isnan(err), torch.full_like(err, float("inf")), err)
    ratio = err / bound
    r = float(ratio.max())
    assert r <= 1.0, f"{what}: {int((ratio > 1).sum())} of {ref.numel()} elements exceed the bound, worst {r:.3g}x"
    return r


def _image(H, W, seed):
    """A uint8 control image with edges and smooth regions (a canny/depth-like map is neither noise nor flat)."""
    g = torch.Generator().manual_seed(seed)
    yy, xx = torch.meshgrid(torch.arange(H), torch.arange(W), indexing="ij")
    base = ((xx * 255) // max(W - 1, 1)).to(torch.int64)
    edges = ((yy // 37 + xx // 53) % 2) * 120
    noise = torch.randint(0, 40, (H, W, 3), generator=g)
    img = (base[..., None] + edges[..., None] + noise) % 256
    return img.to(torch.uint8)


def _cn_cfgs(ocfg, depths=None):
    from latentblending_b200.unet import UNetConfig
    from oracle.sdxl_unet import UNetConfig as OCfg
    if depths is not None:
        ocfg = dataclasses.replace(ocfg, transformer_layers=depths)
    return ocfg, UNetConfig(**{f.name: getattr(ocfg, f.name) for f in dataclasses.fields(OCfg)})


# ---- 1. conditioning embedding -----------------------------------------------------------------------------------
@pytest.mark.parametrize("Hi,Wi", [(1024, 1024), (720, 1280), (1216, 832)])
def test_cond_embedding_bound(Hi, Wi):
    """Every layer of the conditioning embedding (uint8 image -> 16 -> 32 -> 96 -> 256 -> 320) against an fp64
    convolution of the fp16 input that layer saw; the program ControlNetB200.embed records gives the same bits."""
    from latentblending_b200 import ops
    from latentblending_b200.controlnet import ControlNetB200
    from latentblending_b200.pipe import random_controlnet_state_dict
    from oracle.sdxl_unet import SDXL_BASE
    _, cfg = _cn_cfgs(SDXL_BASE, depths=(0, 0, 1))
    cn = ControlNetB200(cfg, random_controlnet_state_dict(cfg, 5, "cuda:0"), "cuda:0")
    img = _image(Hi, Wi, seed=Hi).cuda()
    h, w = Hi // 8, Wi // 8
    emb = cn.embed(img, h, w).clone()
    W = cn.packed.w
    x, H, Wd = img.reshape(-1, 3), Hi, Wi
    xin = (img.to(torch.float32) / 255.0).half()         # the h(u / 255) every first-layer input is
    worst = []
    for name, cin, cout, stride, silu in cn.packed.cond_layers[:-1]:
        y = ops.cond_conv(x, 1, H, Wd, cin, W[name + ".w"], W[name + ".b"], cout, stride=stride, silu=silu)
        wt = W[name + ".w"].permute(3, 2, 0, 1).to(D)                   # [Cout, Cin, 3, 3]
        xn = (xin if cin == 3 else x).reshape(1, H, Wd, cin).permute(0, 3, 1, 2).to(D)
        ref = F.conv2d(xn, wt, W[name + ".b"].to(D), stride=stride, padding=1)
        mag = F.conv2d(xn.abs(), wt.abs(), W[name + ".b"].to(D).abs(), stride=stride, padding=1)
        pre = ULP * ref.abs() + ACC * mag + TINY
        if silu:
            ref, pre = F.silu(ref), ULP * F.silu(ref).abs() + SILU_SLOPE * pre + TINY
        Ho, Wo = ref.shape[2], ref.shape[3]
        ref, pre = (t.permute(0, 2, 3, 1).reshape(-1, cout) for t in (ref, pre))
        worst.append(check(y, ref, pre, f"{name} {H}x{Wd}"))
        x, H, Wd = y, Ho, Wo
    assert (H, Wd) == (h, w)
    name = cn.packed.cond_layers[-1][0]
    out = ops.gemm(x, W[name + ".w"], 320, 1, h, w, taps=9, bias=W[name + ".b"])
    wt = W[name + ".w"].view(320, 3, 3, 256).permute(0, 3, 1, 2).to(D)
    xn = x.reshape(1, h, w, 256).permute(0, 3, 1, 2).to(D)
    ref = F.conv2d(xn, wt, W[name + ".b"].to(D), padding=1).permute(0, 2, 3, 1).reshape(-1, 320)
    mag = F.conv2d(xn.abs(), wt.abs(), W[name + ".b"].to(D).abs(), padding=1).permute(0, 2, 3, 1).reshape(-1, 320)
    worst.append(check(out, ref, ULP * ref.abs() + ACC * mag + TINY, f"conv_out {h}x{w}"))
    assert torch.equal(out, emb)
    torch.cuda.synchronize()
    assert ops.error_flag() == 0
    print(f"cond embedding {Hi}x{Wi}: worst err/bound per layer {[f'{r:.2f}' for r in worst]}")


@pytest.mark.parametrize("B,Hh,Ww", [(1, 9, 7), (2, 13, 5), (3, 1, 1)])
def test_conv_in_add_bound(B, Hh, Ww):
    """conv_in + a per-pixel addend shared by the batch: h(h(conv + b) + e) at odd latent sizes."""
    from latentblending_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(B * 100 + Hh)
    x = torch.randn(B, 4, Hh, Ww, generator=g, device="cuda").half()
    w = (torch.randn(320, 4, 3, 3, generator=g, device="cuda") / 6).half()
    b = torch.randn(320, generator=g, device="cuda").half()
    e = torch.randn(Hh * Ww, 320, generator=g, device="cuda").half()
    out = ops.conv_in_add(x, w.permute(2, 3, 1, 0).contiguous(), b, 320, e)
    conv = F.conv2d(x.to(D), w.to(D), b.to(D), padding=1).permute(0, 2, 3, 1).reshape(-1, 320)
    mag = F.conv2d(x.to(D).abs(), w.to(D).abs(), b.to(D).abs(), padding=1).permute(0, 2, 3, 1).reshape(-1, 320)
    ee = e.to(D).repeat(B, 1)
    ref = conv + ee
    bound = ULP * ref.abs() + ULP * conv.abs() + ACC * mag + 2 * TINY
    check(out, ref, bound, f"conv_in_add B={B} {Hh}x{Ww}")
    plain = ops.conv_in(x, w.permute(2, 3, 1, 0).contiguous(), b, 320)
    assert torch.equal(out, (plain.float() + e.float().repeat(B, 1)).half())    # the fp16 sum of the two fp16 terms
    torch.cuda.synchronize()
    assert ops.error_flag() == 0


# ---- 2. UNet + ControlNet against the oracle -----------------------------------------------------------------------
_TINY = {}


def _tiny_pair(depths):
    if depths not in _TINY:
        from latentblending_b200.controlnet import ControlNetB200
        from latentblending_b200.unet import UNetB200
        from oracle.controlnet import SDXLControlNet, synthetic_init_controlnet_
        from oracle.sdxl_unet import SDXLUNet, synthetic_init_, tiny_config
        ocfg = tiny_config()
        ocn, ccfg = _cn_cfgs(ocfg, depths)
        unet = synthetic_init_(SDXLUNet(ocfg), seed=0).eval()
        cn = synthetic_init_controlnet_(SDXLControlNet(ocn), seed=1).eval()
        with torch.no_grad():
            for m in (unet, cn):
                for p in m.parameters():
                    p.copy_(p.half().float())
        _, ucfg = _cn_cfgs(ocfg)
        cnb = ControlNetB200(ccfg, cn.state_dict(), "cuda:0")
        _TINY[depths] = dict(unet=unet, cn=cn, cnb=cnb, net=UNetB200(ucfg, unet.state_dict(), "cuda:0", controlnet=cnb),
                             plain=UNetB200(ucfg, unet.state_dict(), "cuda:0"), cfg=ocfg)
    return _TINY[depths]


def _inputs(cfg, B, h, w, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, 4, h, w, generator=g).half()
    ctx = (torch.randn(B, 77, cfg.cross_attention_dim, generator=g) * 0.5).half()
    pooled = torch.randn(B, cfg.pooled_dim, generator=g).half()
    tids = torch.tensor([[8.0 * h, 8.0 * w, 0, 0, 8.0 * h, 8.0 * w]] * B).half()
    return x, ctx, pooled, tids


@pytest.mark.parametrize("depths", [(0, 1, 2), (0, 0, 1)])
@pytest.mark.parametrize("B,h,w,scale", [(1, 16, 16, 1.0), (2, 16, 16, 0.6), (2, 32, 16, 1.0), (1, 32, 16, 0.6)])
def test_tiny_unet_controlnet_matches_oracle(depths, B, h, w, scale):
    from latentblending_b200 import ops
    from oracle.controlnet import image_to_cond, unet_with_residuals
    p = _tiny_pair(depths)
    x, ctx, pooled, tids = _inputs(p["cfg"], B, h, w, seed=B + h)
    img = _image(8 * h, 8 * w, seed=h + w)
    t = 611.0
    with torch.no_grad():
        down, mid = p["cn"](x.float(), t, ctx.float(), pooled.float(), tids.float(),
                            image_to_cond(img).expand(B, -1, -1, -1), conditioning_scale=scale)
        ref = unet_with_residuals(p["unet"], x.float(), t, ctx.float(), pooled.float(), tids.float(), down, mid)
        plain_ref = p["unet"](x.float(), t, ctx.float(), pooled.float(), tids.float())
    p["cnb"].set_scale(scale)
    p["cnb"].embed(img.cuda(), h, w)
    eps = p["net"].forward(x.cuda(), t, ctx.cuda(), pooled.cuda(), tids.cuda(), control=True).float().cpu()
    torch.cuda.synchronize()
    assert ops.error_flag() == 0
    rel = ((eps - ref).norm() / ref.norm()).item()
    effect = ((ref - plain_ref).norm() / ref.norm()).item()
    print(f"unet+controlnet {depths} B={B} {h}x{w} scale={scale}: rel_l2={rel:.3e} (control changes eps by {effect:.3e})")
    assert effect > 1e-2                   # the comparison is not vacuous
    assert rel <= 2e-3, f"relative L2 error {rel}"


@pytest.mark.slow
def test_full_sdxl_controlnet_matches_fixture():
    """The full SDXL-base UNet with the "full" ControlNet, CFG batch 2 at 128x128, against the committed fp32 oracle
    fixture (tests/golden/make_controlnet_fixtures.py)."""
    from latentblending_b200 import ops
    from latentblending_b200.controlnet import ControlNetB200
    from latentblending_b200.unet import UNetB200
    from make_controlnet_fixtures import FIXTURE, SCALE, T, control_image, inputs, oracle_nets, weights_checksum
    from oracle.sdxl_unet import SDXL_BASE
    fx = np.load(FIXTURE)
    unet, cn = oracle_nets()
    assert weights_checksum(unet.state_dict()) + weights_checksum(cn.state_dict()) == str(fx["weights_sha1"])
    _, ucfg = _cn_cfgs(SDXL_BASE)
    cnb = ControlNetB200(ucfg, cn.state_dict(), "cuda:0")
    net = UNetB200(ucfg, unet.state_dict(), "cuda:0", controlnet=cnb)
    del unet, cn
    x, ctx, pooled, tids = inputs()
    cnb.set_scale(SCALE)
    cnb.embed(control_image().cuda(), 128, 128)
    eps = net.forward(x.cuda(), T, ctx.cuda(), pooled.cuda(), tids.cuda(), control=True).float().cpu()
    torch.cuda.synchronize()
    assert ops.error_flag() == 0
    ref = torch.from_numpy(fx["eps"])
    rel = ((eps - ref).norm() / ref.norm()).item()
    print(f"full SDXL UNet + ControlNet @128x128 B=2: rel_l2={rel:.3e}")
    assert rel <= 2e-3


# ---- 3. the plain path is untouched --------------------------------------------------------------------------------
def test_plain_step_program_is_untouched():
    """With a ControlNet attached, the plain step program has the launch count of a UNet without one and gives the
    same eps bit for bit; the control program runs only the ControlNet's records on top."""
    p = _tiny_pair((0, 1, 2))
    x, ctx, pooled, tids = _inputs(p["cfg"], 2, 16, 24, seed=4)
    assert p["net"].launches_per_forward(2, 16, 24)[0] == p["plain"].launches_per_forward(2, 16, 24)[0]
    plain = p["plain"].forward(x.cuda(), 300.0, ctx.cuda(), pooled.cuda(), tids.cuda()).clone()
    with_cn = p["net"].forward(x.cuda(), 300.0, ctx.cuda(), pooled.cuda(), tids.cuda()).clone()
    assert torch.equal(plain, with_cn)
    pl = p["net"].plan(2, 16, 24)
    assert pl.prog_step_cn.num_launches > pl.prog_step.num_launches
    n = len(pl.prog_step.ops)
    cn_ops = pl.prog_step_cn.ops
    assert len(cn_ops) > n
    # the control program is the plain program's records with the ControlNet's inserted in one contiguous run
    k = next(i for i, (a, b) in enumerate(zip(pl.prog_step.ops, cn_ops)) if a is not b)
    extra = len(cn_ops) - n
    assert all(a is b for a, b in zip(pl.prog_step.ops[k:], cn_ops[k + extra:]))


def _tiny_holder(seed=3, guidance=4.0):
    from latentblending_b200 import DiffusersHolder, SyntheticSDXLPipe
    from oracle.sdxl_unet import tiny_config
    _, cfg = _cn_cfgs(tiny_config())
    pp = SyntheticSDXLPipe("synthetic/sdxl-base-tiny", "cuda:0", unet_cfg=cfg, seed=seed, vae="tiny",
                           controlnet="full")
    dh = DiffusersHolder(pp)
    dh.guidance_scale = guidance
    dh.set_dimensions((192, 128))
    dh.set_num_inference_steps(6)
    return dh


def test_steps_outside_the_window_run_the_plain_program():
    from latentblending_b200 import program
    dh = _tiny_holder()
    emb = dh.get_text_embedding("a lake")
    start = dh.get_noise(5)
    img = _image(256, 256, seed=1).numpy()

    def run():
        l0 = program.LAUNCHES[0]
        out = dh.run_diffusion_sd_xl(emb, start)
        torch.cuda.synchronize()
        return [t.clone() for t in out], program.LAUNCHES[0] - l0

    for dual in (True, False):
        dh.dual_stream = dual
        dh.set_control_image(None)
        plain, n_plain = run()
        dh.set_control_image(img, 0.8, guidance_start=0.9, guidance_end=1.0)       # no step of 6 inside
        off, n_off = run()
        assert n_off == n_plain and all(torch.equal(a, b) for a, b in zip(off, plain))
        dh.set_control_image(img, 0.0)                                               # scale 0: plain
        zero, n_zero = run()
        assert n_zero == n_plain and all(torch.equal(a, b) for a, b in zip(zero, plain))
        dh.set_control_image(img, 0.8, guidance_start=0.0, guidance_end=0.5)         # steps 0, 1, 2
        half, n_half = run()
        assert n_half > n_plain
        assert all(not torch.equal(a, b) for a, b in zip(half, plain))
        # what runs at the window's steps is exactly the control program
        plan = dh.unet.plan(1 if dual else 2, dh.height_latent, dh.width_latent, tag="cfg_uncond") if dual else \
            dh.unet.plan(2, dh.height_latent, dh.width_latent)
        per = plan.prog_step_cn.num_launches - plan.prog_step.num_launches
        assert n_half - n_plain == 3 * per * (2 if dual else 1)
    from latentblending_b200 import ops
    assert ops.error_flag() == 0


def test_set_control_image_needs_a_controlnet():
    from latentblending_b200 import DiffusersHolder, SyntheticSDXLPipe
    from oracle.sdxl_unet import tiny_config
    _, cfg = _cn_cfgs(tiny_config())
    dh = DiffusersHolder(SyntheticSDXLPipe("synthetic/sdxl-base-tiny", "cuda:0", unet_cfg=cfg, vae="tiny"))
    with pytest.raises(ValueError):
        dh.set_control_image(_image(64, 64, 0).numpy())
    dh2 = _tiny_holder()
    with pytest.raises(ValueError):
        dh2.set_control_image(_image(64, 64, 0).numpy(), guidance_start=0.6, guidance_end=0.5)


# ---- 4. batch invariance of whole transitions --------------------------------------------------------------------
def _fingerprint(be):
    sys.path.insert(0, ROOT)
    from bench import tree_fingerprint
    return tree_fingerprint(be)


def _transition(pp, size, steps, branches, width, dual, img, scale=0.7):
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
    be.set_control_image(img, scale, guidance_start=0.0, guidance_end=0.8)
    be.run_transition(fixed_seeds=[7, 8])
    torch.cuda.synchronize()
    fp = _fingerprint(be)
    del be
    gc.collect()                # each engine holds its own packed UNet + ControlNet
    torch.cuda.empty_cache()
    return fp


@pytest.mark.parametrize("turbo", [True, False])
def test_transition_fingerprint_is_batch_invariant(turbo):
    """A full-size synthetic SDXL transition with a control image (512^2 Turbo; 1024^2 base under CFG): the tree is
    the same with lockstep speculation width 1 and 2 (4 for Turbo) and with dual-stream CFG halves on and off."""
    from latentblending_b200 import SyntheticSDXLPipe, ops
    name = "stabilityai/sdxl-turbo" if turbo else "stabilityai/stable-diffusion-xl-base-1.0"
    pp = SyntheticSDXLPipe(name, "cuda:0", seed=0, vae="tiny", controlnet="full")
    size = (512, 512) if turbo else (1024, 1024)
    img = _image(size[1], size[0], seed=3).numpy()
    steps, branches = (4, 6) if turbo else (5, 6)
    fps = {}
    for width in (1, 4 if turbo else 2):
        for dual in ((True,) if turbo else (True, False)):
            fps[(width, dual)] = _transition(pp, size, steps, branches, width, dual, img)
    print(f"controlnet transition fingerprints {'turbo' if turbo else 'base'}: {fps}")
    assert len(set(fps.values())) == 1
    assert ops.error_flag() == 0


# ---- 5. the engine end to end -------------------------------------------------------------------------------------
def test_engine_set_control_image_round_trip():
    """set_control_image -> run_transition -> set_control_image(None) -> run_transition: the second tree is the tree
    of an engine that never had an image.  set_dimensions between runs re-embeds the image at the new size."""
    from latentblending_b200 import BlendingEngine, ops
    dh = _tiny_holder()
    pp = dh.pipe
    img = _image(300, 200, seed=8).numpy()

    def engine():
        be = BlendingEngine(pp, run_benchmark=False)
        be.set_dimensions((192, 128))
        be.set_num_inference_steps(6)
        be.set_prompt1("photo of a lake")
        be.set_prompt2("alien planet")
        be.set_branching(depth_strength=0.5, nmb_max_branches=5)
        be.deterministic_noise = True
        be.output_device_frames = True
        return be

    def second_run(be):
        be.set_dimensions((128, 192))
        be.set_dimensions((192, 128))
        be.run_transition(fixed_seeds=[1, 2])
        torch.cuda.synchronize()
        assert ops.error_flag() == 0
        return _fingerprint(be)

    never = engine()
    never.run_transition(fixed_seeds=[1, 2])
    want_first = _fingerprint(never)
    want_second = second_run(never)
    be = engine()
    be.set_control_image(img, 0.9)
    be.run_transition(fixed_seeds=[1, 2])
    torch.cuda.synchronize()
    assert ops.error_flag() == 0
    assert _fingerprint(be) != want_first
    emb_a = be.dh.controlnet.embedding(be.dh.height_latent, be.dh.width_latent).clone()
    be.set_dimensions((128, 192))
    emb_b = be.dh.controlnet.embedding(be.dh.height_latent, be.dh.width_latent).clone()
    assert emb_b.shape == emb_a.shape and float(emb_b.abs().max()) > 0            # embedded at 24x16 on the spot
    assert not torch.equal(emb_a, emb_b)
    be.set_control_image(None)
    assert second_run(be) == want_second        # the same calls as ``never`` made, from here on without the image
