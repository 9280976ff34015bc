"""GPU tests of image keyframes (img2img): the three kernels (lb_image_conv_in, lb_im2col_s2_pad01, lb_add_noise_rows),
the native VAE encoder against the fp32 oracle fixtures (tests/golden/make_init_image_fixtures.py), the holder's
init trajectories and the engine's transitions with image keyframes.

Bounds.  lb_image_conv_in is held per element to tests/test_fp16_bounds_gpu.py's terms against an fp64 conv of the
same rounded input: ULP + ACC * sum|x||w| + TINY, with ULP = 2^-10 |ref| in fp16 and 2^-8 |ref| in bf16 (half an ulp
of the output rounding, with margin).  lb_im2col_s2_pad01 and lb_add_noise_rows are bit-exact (a copy; the same fp16
op chain torch runs on CUDA).  The encoder is held to relative L2 against the fp32 oracle: 3e-3 in fp16, 3e-2 in bf16.
Those are the storage types' own errors, not the kernels': on an H100 the native encoder measures 2.1e-3 (fp16) and
2.1e-2 (bf16) on both shapes, while the oracle itself run by torch on the GPU in fp16 / bf16 storage measures 2.8-2.9e-3
and 2.5e-2.  The fp16 error grows level by level as the residual stream is rounded (torch fp16 against fp32: 3e-4
after conv_in, 6e-4, 1.2e-3, 1.7e-3, 2.1e-3 after the four down blocks, 2.9e-3 at the output), and bf16 rounds 8x
coarser.  The upcast fixture's bf16 encode meets 1e-2."""
import os
import socket
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden")
if GOLD not in sys.path:
    sys.path.insert(0, GOLD)

ULP = {torch.float16: 2.0 ** -10, torch.bfloat16: 2.0 ** -8}
ACC = 2.0 ** -16
TINY = 2.0 ** -24
REL_L2 = {torch.float16: 3e-3, torch.bfloat16: 3e-2}


def _u8(H, W, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randint(0, 256, (H, W, 3), generator=g, device="cuda", dtype=torch.uint8)


# ---- kernels -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("H,W", [(1024, 1024), (720, 1280)])
def test_image_conv_in_bound(dtype, H, W):
    from latentblending_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(1)
    w = ((torch.rand(128, 3, 3, 3, generator=g, device="cuda") * 2 - 1) / 27 ** 0.5).to(dtype)
    b = ((torch.rand(128, generator=g, device="cuda") * 2 - 1) * 0.02).to(dtype)
    img = _u8(H, W, seed=2)
    out = ops.image_conv_in(img, w.permute(2, 3, 1, 0).contiguous(), b, 128)
    x = (2.0 * (img.float() / 255.0) - 1.0).to(dtype)                     # VaeImageProcessor.preprocess, one rounding
    xd = x.double().permute(2, 0, 1)[None]
    ref = F.conv2d(xd, w.double(), b.double(), padding=1)[0].permute(1, 2, 0).reshape(H * W, 128)
    mag = F.conv2d(xd.abs(), w.double().abs(), b.double().abs(), padding=1)[0].permute(1, 2, 0).reshape(H * W, 128)
    err = (out.double() - ref).abs()
    bound = ULP[dtype] * ref.abs() + ACC * mag + TINY
    assert out.dtype == dtype and torch.isfinite(out).all()
    assert (err <= bound).all(), (err / bound).max().item()
    # non-vacuity: an input read without the 2x - 1 is far outside the bound
    wrong = F.conv2d((img.float() / 255.0).double().permute(2, 0, 1)[None], w.double(), b.double(), padding=1)
    assert ((wrong[0].permute(1, 2, 0).reshape(H * W, 128) - ref).abs() > bound).float().mean() > 0.5


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("H,W,C", [(16, 24, 128), (7, 9, 64), (106, 154, 256), (2, 2, 8)])
def test_im2col_s2_pad01_matches_pad_unfold(dtype, H, W, C):
    from latentblending_b200 import ops
    x = torch.randn(H * W, C, device="cuda").to(dtype)
    got = ops.im2col_s2_pad01(x, 1, H, W, C)
    Ho, Wo = (H - 2) // 2 + 1, (W - 2) // 2 + 1
    xp = F.pad(x.view(1, H, W, C).permute(0, 3, 1, 2).float(), (0, 1, 0, 1))
    cols = F.unfold(xp, 3, stride=2)                                          # [1, C*9, Ho*Wo], (c, ky, kx)
    ref = cols.view(C, 9, Ho * Wo).permute(2, 1, 0).reshape(Ho * Wo, 9 * C).to(dtype)
    assert got.shape == ref.shape and torch.equal(got, ref)


def _table(kind, n):
    from latentblending_b200.schedulers import DPMTables, EulerTables, LCMTables
    t = {"euler": lambda: EulerTables("euler"), "euler_ancestral": lambda: EulerTables("euler_ancestral"),
         "lcm": LCMTables, "dpm": DPMTables}[kind]()
    t.set_timesteps(n)
    return t


def _torch_add_noise(t, kind, x0, eps, i):
    """diffusers 0.25.0 add_noise(x0, eps, timesteps[i:i+1]) restated op by op on fp16 CUDA tensors."""
    x0 = x0.to(torch.float16)
    ts = t.timesteps.numpy()
    hits = np.nonzero(ts == ts[i])[0]
    idx = int(hits[1] if len(hits) > 1 else hits[0])
    if kind.startswith("euler"):
        sigma = t.sigmas.to(device="cuda", dtype=torch.float16)[idx:idx + 1].view(1, 1, 1, 1)
        return x0 + eps * sigma
    if kind == "lcm":
        acp = t.alphas_cumprod.to(device="cuda", dtype=torch.float16)
        tt = int(ts[i])
        a = (acp[tt:tt + 1] ** 0.5).view(1, 1, 1, 1)
        b = ((1 - acp[tt:tt + 1]) ** 0.5).view(1, 1, 1, 1)
        return a * x0 + b * eps
    sigma = t.sigmas.to(device="cuda", dtype=torch.float16)[idx:idx + 1].view(1, 1, 1, 1)
    alpha_t = 1 / ((sigma ** 2 + 1) ** 0.5)
    sigma_t = sigma * alpha_t
    return alpha_t * x0 + sigma_t * eps


@pytest.mark.parametrize("kind,n", [("euler", 30), ("euler_ancestral", 4), ("lcm", 4), ("dpm", 20)])
@pytest.mark.parametrize("h,w", [(128, 128), (90, 160)])
@pytest.mark.parametrize("xdtype", [torch.float16, torch.bfloat16])
def test_add_noise_rows_bit_exact(kind, n, h, w, xdtype):
    from latentblending_b200 import _cabi, ops
    t = _table(kind, n)
    g = torch.Generator(device="cuda").manual_seed(3)
    x0 = (torch.randn(1, 4, h, w, generator=g, device="cuda") * 0.8).to(xdtype)
    eps = torch.randn(1, 4, h, w, generator=g, device="cuda", dtype=torch.float16)
    cf = [t.add_noise_coeffs(i) for i in range(n)]
    form = cf[0][0]
    assert all(c[0] == form for c in cf)
    coeffs = torch.tensor([[a, b] for _, a, b in cf], dtype=torch.float16, device="cuda")
    cnt = torch.zeros(1, dtype=torch.int32, device="cuda")
    rows = ops.add_noise_rows(x0, eps, coeffs, form, nonfinite=cnt)
    for i in range(n):
        ref = _torch_add_noise(t, kind, x0, eps, i)
        assert torch.equal(rows[i].view(1, 4, h, w), ref), (kind, i)
    assert int(cnt.item()) == 0
    bad = x0.clone()
    bad.view(-1)[[5, 77, 900]] = float("inf")
    bad.view(-1)[11] = float("nan")
    ops.add_noise_rows(bad, eps, coeffs[:0], form, nonfinite=cnt)            # rows = 0: count only
    assert int(cnt.item()) == 4
    assert form == (_cabi.ADD_NOISE_SIGMA if kind.startswith("euler") else _cabi.ADD_NOISE_ALPHA_SIGMA)


# ---- encoder vs fixtures ----------------------------------------------------------------------------------------------
_ENC = {}


def _encoder(dtype, upcast=False):
    key = (dtype, upcast)
    if key not in _ENC:
        from latentblending_b200.vae import VAEEncoderB200
        from make_init_image_fixtures import ENC_CHANNELS, oracle_encoder
        _ENC.clear()
        torch.cuda.empty_cache()
        sd = oracle_encoder(upcast).state_dict()
        _ENC[key] = VAEEncoderB200(sd, ENC_CHANNELS, 0.13025, "cuda:0", dtype=dtype)
    return _ENC[key]


def _fixture(name):
    from make_init_image_fixtures import SHAPES, fixture_image
    path = os.path.join(GOLD, name)
    H, W = SHAPES[path]
    return torch.from_numpy(np.load(path)["latents"]), torch.from_numpy(fixture_image(H, W)).cuda()


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("name", ["vae_encoder_sdxl_64.npz", "vae_encoder_sdxl_53x77.npz"])
def test_encoder_matches_fixture(dtype, name):
    want, img = _fixture(name)
    enc = _encoder(dtype)
    x0 = enc.encode(img).clone()
    enc.check_finite(x0)
    got = x0.float().cpu()
    rel = ((got - want).norm() / want.norm()).item()
    print(f"{name} {dtype}: rel L2 {rel:.2e}")
    assert got.shape == want.shape and rel <= REL_L2[dtype], rel


def test_encoder_upcast_fixture_fp16_raises_bf16_meets_bound():
    from latentblending_b200 import _cabi
    want, img = _fixture("vae_encoder_sdxl_64_upcast.npz")
    enc16 = _encoder(torch.float16, upcast=True)
    with pytest.raises(_cabi.LB200Error, match="bf16"):
        enc16.check_finite(enc16.encode(img).clone())
    enc = _encoder(torch.bfloat16, upcast=True)
    x0 = enc.encode(img).clone()
    enc.check_finite(x0)
    rel = ((x0.float().cpu() - want).norm() / want.norm()).item()
    print(f"upcast bf16: rel L2 {rel:.2e}")
    assert rel <= 1e-2, rel


def test_encoder_graph_replay_matches_direct_launches():
    from latentblending_b200 import _cabi
    _, img = _fixture("vae_encoder_sdxl_53x77.npz")
    enc = _encoder(torch.float16)
    pl = enc.plan(img.shape[0] // 8, img.shape[1] // 8)
    outs = [enc.encode(img).clone() for _ in range(3)]                          # direct, capture + replay, replay
    assert _cabi.load().lb_program_is_graph(pl.prog.handle) == 1
    kinds = list(range(1, 23))
    pl.x0.zero_()
    pl.prog.run_kinds(kinds)                                                    # every op, launched directly
    direct = pl.x0.clone()
    assert all(torch.equal(o, direct) for o in outs)


# ---- holder ---------------------------------------------------------------------------------------------------------
def _tiny_pipe(**kw):
    from latentblending_b200 import SyntheticSDXLPipe
    from latentblending_b200.unet import UNetConfig
    cfg = UNetConfig(block_out_channels=(64, 128, 256), transformer_layers=(0, 1, 2), cross_attention_dim=128,
                     addition_time_embed_dim=32, pooled_dim=64, sample_size=16)
    return SyntheticSDXLPipe("synthetic/sdxl-base-tiny", "cuda:0", unet_cfg=cfg, seed=5,
                             vae_channels=(64, 64, 128, 128), **kw)


def _photo(H, W, seed=9):
    from make_init_image_fixtures import fixture_image
    return fixture_image(H, W, seed=seed)


@pytest.mark.parametrize("scheduler", [None, "lcm", "dpmpp_2m"])
def test_holder_init_rows_and_denoised_rows(scheduler):
    from latentblending_b200 import DiffusersHolder, ops
    from latentblending_b200.schedulers import img2img_start
    dh = DiffusersHolder(_tiny_pipe(scheduler=scheduler))
    dh.set_dimensions((128, 96))
    N = 4 if scheduler == "lcm" else 10
    dh.set_num_inference_steps(N)
    dh.guidance_scale = 1.0 if scheduler == "lcm" else 4.0
    x0 = dh.image2latent(_photo(200, 150))
    assert x0.shape == (1, 4, 12, 16) and x0.dtype == torch.float16
    assert torch.equal(dh.image2latent(_photo(200, 150)), x0)                     # a second encode: bit-identical
    emb = dh.get_text_embedding("a harbour")
    eps = dh.init_noise(421)
    i0 = img2img_start(N, 0.5)
    out = dh.run_diffusion_sd_xl_multi([dict(text_embeddings=emb, init=(x0, eps))], idx_start=i0)[0]
    assert all(r is not None for r in out) and len(out) == N
    sched = dh.pipe.scheduler
    cf = [sched.add_noise_coeffs(i) for i in range(1, i0 + 1)]
    rows = ops.add_noise_rows(x0, eps, torch.tensor([[a, b] for _, a, b in cf], dtype=torch.float16,
                                                    device="cuda"), cf[0][0])
    for i in range(i0):
        assert torch.equal(out[i].reshape(-1), rows[i]), i
    torch.manual_seed(0)
    ref = dh.run_diffusion_sd_xl(emb, out[i0 - 1], idx_start=i0)
    torch.manual_seed(0)
    again = dh.run_diffusion_sd_xl_multi([dict(text_embeddings=emb, init=(x0, eps))], idx_start=i0)[0]
    for i in range(i0, N):
        assert torch.equal(again[i], ref[i]), i


def test_holder_strength_one_starts_from_noised_image():
    from latentblending_b200 import DiffusersHolder, ops
    dh = DiffusersHolder(_tiny_pipe())
    dh.set_dimensions((128, 128))
    dh.set_num_inference_steps(6)
    x0, eps = dh.image2latent(_photo(128, 128)), dh.init_noise(7)
    emb = dh.get_text_embedding("x")
    out = dh.run_diffusion_sd_xl_multi([dict(text_embeddings=emb, init=(x0, eps))], idx_start=0)[0]
    _, a, b = dh.pipe.scheduler.add_noise_coeffs(0)
    start = ops.add_noise_rows(x0, eps, torch.tensor([[a, b]], dtype=torch.float16, device="cuda"), 0)
    ref = dh.run_diffusion_sd_xl(emb, start.view(1, 4, 16, 16), idx_start=0)
    assert all(torch.equal(p, q) for p, q in zip(out, ref))


# ---- engine ---------------------------------------------------------------------------------------------------------
def _engine(pipe=None):
    from latentblending_b200 import BlendingEngine
    be = BlendingEngine(pipe if pipe is not None else _tiny_pipe(), run_benchmark=False)
    be.set_dimensions((128, 128))
    be.set_num_inference_steps(10)
    be.set_prompt1("a harbour at dusk")
    be.set_prompt2("a harbour at dawn, oil painting")
    be.set_branching(depth_strength=0.5, nmb_max_branches=6)
    be.output_device_frames = True
    return be


def _frames(be, seeds=(420, 421)):
    # a transition leaves the guidance at its last branch's damped value, which steers the next transition's outer
    # trajectories (the reference's behaviour): start every compared transition from the default guidance
    be.set_guidance_scale()
    return [f.clone() for f in be.run_transition(fixed_seeds=list(seeds))]


def test_engine_image_keyframe_transitions():
    be = _engine()
    img1, img2 = _photo(160, 200, seed=1), _photo(128, 128, seed=2)
    text = _frames(be)
    for a, b in ((img1, img2), (img1, None), (None, img2)):
        be.set_init_image1(a, strength=0.5)
        be.set_init_image2(b, strength=0.5)
        fr = _frames(be)
        assert len(fr) == 6 and all(f.shape == (128, 128, 3) for f in fr)
        assert (not torch.equal(fr[0], text[0])) == (a is not None)
        assert (not torch.equal(fr[-1], text[-1])) == (b is not None)
        assert all(r is not None for r in be.tree_latents[0] + be.tree_latents[-1])


def test_engine_batched_sequential_repeatable_and_none():
    be = _engine()
    img1, img2 = _photo(128, 128, seed=1), _photo(128, 128, seed=2)
    be.set_init_image1(img1, strength=0.6)
    be.set_init_image2(img2, strength=0.6)
    batched = _frames(be)
    assert torch.equal(_frames(be)[0], batched[0]) and all(torch.equal(p, q) for p, q in zip(_frames(be), batched))
    be.batch_outer_pair = False
    seq = _frames(be)
    assert all(torch.equal(p, q) for p, q in zip(seq, batched))
    be.batch_outer_pair = True
    ref = _engine()
    never = _frames(ref)
    be.set_init_image1(None)
    be.set_init_image2(None)
    assert all(torch.equal(p, q) for p, q in zip(_frames(be), never))


def test_engine_crossfeed_and_different_strengths():
    be = _engine()
    be.set_branch1_crossfeed(0.8, 0.6, 0.4)
    be.set_init_image1(_photo(128, 128, seed=1), strength=0.3)
    be.set_init_image2(_photo(128, 128, seed=2), strength=0.7)
    a = _frames(be)
    be.batch_outer_pair = False
    b = _frames(be)
    assert all(torch.equal(p, q) for p, q in zip(a, b))


def test_tiny_vae_pipe_raises():
    be = _engine(_tiny_pipe(vae="tiny"))
    with pytest.raises(ValueError, match="tiny"):
        be.set_init_image1(_photo(128, 128))


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _sharded_worker(rank, world, port, q):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device(f"cuda:{rank}"))

    def build(dev):
        from latentblending_b200 import BlendingEngine
        be = BlendingEngine(_tiny_pipe_on(dev), run_benchmark=False)
        be.set_dimensions((128, 128))
        be.set_num_inference_steps(10)
        be.set_prompt1("one")
        be.set_prompt2("two")
        be.set_branching(depth_strength=0.5, nmb_max_branches=6)
        be.set_init_image1(_photo(128, 128, seed=1), strength=0.6)
        be.output_device_frames = True
        return be

    be = build(f"cuda:{rank}")
    be.run_transition(fixed_seeds=[420, 421])
    res = [float(t[-1].float().sum()) for t in be.tree_latents]
    dist.barrier()
    dist.destroy_process_group()
    if rank == 0:
        be2 = build("cuda:0")
        be2.run_transition(fixed_seeds=[420, 421])
        q.put(("seq", [float(t[-1].float().sum()) for t in be2.tree_latents]))
    q.put((rank, res))


def _tiny_pipe_on(dev):
    from latentblending_b200 import SyntheticSDXLPipe
    from latentblending_b200.unet import UNetConfig
    cfg = UNetConfig(block_out_channels=(64, 128, 256), transformer_layers=(0, 1, 2), cross_attention_dim=128,
                     addition_time_embed_dim=32, pooled_dim=64, sample_size=16)
    return SyntheticSDXLPipe("synthetic/sdxl-base-tiny", dev, unet_cfg=cfg, seed=5, vae_channels=(64, 64, 128, 128))


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_sharded_engine_with_image_keyframe_matches_sequential():
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_sharded_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    got = [q.get(timeout=900) for _ in range(3)]
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    seq = next(g for g in got if g[0] == "seq")[1]
    for g in got:
        assert g[1] == seq, g[0]
