"""GPU tests of the round-2 additions, each against a plain fp32 PyTorch / numpy restatement or the CPU oracle:

  * ReLU epilogue;
  * lb_cfg_euler_step writing the next step's model input / taking the two CFG halves from separate buffers;
  * native LPIPS (AlexNet on lb_gemm + fused tap reduction) vs oracle/lpips_alex.py;
  * device frame fill (lb_frames_lerp_u8) vs numpy float32 arithmetic;
  * fp16-VAE overflow detection; DiffusersHolder.get_noise (SURVEY 8a10).
Tolerances are stated at each assert."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _rand(*shape, seed=0, s=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(*shape, generator=g, device="cuda") * s)


def _rel(a, b):
    return ((a.float() - b.float()).norm() / b.float().norm()).item()


def test_gemm_relu_epilogue():
    from latentblending_b200 import ops
    M, K, N = 3969, 1728, 384            # AlexNet conv3 as a patch-matrix GEMM
    a = _rand(M, K, seed=21).half()
    w = (_rand(N, K, seed=22) * K ** -0.5).half()
    b = (_rand(N, seed=23) * 0.1).half()
    out = ops.gemm(a, w, N, 1, 1, M, bias=b, relu=True)
    ref = F.relu(a.float() @ w.float().t() + b.float())
    assert (out >= 0).all()
    assert _rel(out, ref) <= 2e-3


# ---- K9: fused next-step scale, separate CFG halves -----------------------------------------------------------
def test_cfg_euler_writes_next_model_input_and_accepts_split_halves():
    from latentblending_b200 import ops
    n = 4 * 128 * 128
    x = _rand(1, 4, 128, 128, seed=31, s=3.0).half()
    eps = _rand(2, 4, 128, 128, seed=32).half()
    base = ops.cfg_euler_step(x, eps, 3.5, 7.91, -0.52)
    nxt = torch.zeros(2, 4, 128, 128, dtype=torch.float16, device="cuda")
    got = ops.cfg_euler_step(x, eps, 3.5, 7.91, -0.52, scaled_next=nxt, next_divisor=7.4586)
    assert torch.equal(got, base)
    want = ops.scale_model_input(base, 2, 7.4586)
    assert torch.equal(nxt, want)                       # bit-identical to the separate lb_scale_model_input launch
    # the two CFG halves in separate (non-adjacent) buffers, as exchanged between a GPU pair
    u, t = eps[0:1].clone(), eps[1:2].clone()
    got2 = ops.cfg_euler_step(x, u, 3.5, 7.91, -0.52, eps_text=t)
    assert torch.equal(got2, base)
    # scale_model_input: vectorised path == scalar reference arithmetic
    ref = (x.float() / np.float32(7.4586)).half()
    assert torch.equal(ops.scale_model_input(x, 1, 7.4586)[0], ref[0])


# ---- LPIPS ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("H,W", [(128, 128), (256, 192), (512, 512)])
def test_native_lpips_matches_oracle(H, W):
    """Features (five ReLU taps) and distance vs the fp32 CPU oracle (oracle/lpips_alex.py) on identical weights.
    Tolerance: taps rel-L2 <= 3e-3 (fp16 storage, fp32 accumulate), distance within 1 % (+1e-5)."""
    from latentblending_b200.lpips import LPIPSAlexB200
    from oracle.lpips_alex import LPIPSAlex, lpips_distance
    net = LPIPSAlex(seed=2).eval()
    with torch.no_grad():
        for c in net.convs:
            c.weight.copy_(c.weight.half().float())
            c.bias.copy_(torch.randn(c.bias.shape, generator=torch.Generator().manual_seed(9)) * 0.05)
            c.bias.copy_(c.bias.half().float())
    sd = {k: v for k, v in net.state_dict().items() if k.startswith(("convs.", "lins."))}
    lp = LPIPSAlexB200(sd, "cuda:0")
    g = torch.Generator().manual_seed(5)
    base = torch.rand(H, W, 3, generator=g)
    fa = (base * 255).round().to(torch.uint8)
    fb = ((base * 0.8 + 0.2 * torch.rand(H, W, 3, generator=g)) * 255).round().to(torch.uint8)
    ca, cb = fa.cuda(), fb.cuda()
    taps = lp.features(ca)
    with torch.no_grad():
        x = (2 * fa.float() / 255.0 - 1).permute(2, 0, 1).unsqueeze(0)
        ref_taps = net.features(x)
    for i, (t, r) in enumerate(zip(taps, ref_taps)):
        r2 = r[0].permute(1, 2, 0).reshape(-1, r.shape[1])
        assert t.shape == r2.shape, (i, t.shape, r2.shape)
        assert _rel(t.cpu(), r2) <= 3e-3, (i, _rel(t.cpu(), r2))
    d = lp.distance(ca, cb)
    ref = lpips_distance(net, fa.numpy(), fb.numpy())
    print(f"lpips {H}x{W}: product {d:.6f} oracle {ref:.6f}")
    assert abs(d - ref) <= 0.01 * abs(ref) + 1e-5
    assert lp.distance(ca, ca) <= 1e-6
    dl, dr = lp.distance_pair(ca, cb, ca)
    assert dl == d and dr == lp.distance(ca, ca)
    assert lp.features(ca) is taps                     # cached per frame object
    from latentblending_b200 import ops
    assert ops.error_flag() == 0


# ---- movie frame fill ----------------------------------------------------------------------------------------
def test_frames_lerp_u8_matches_numpy_float32():
    from latentblending_b200 import ops
    from latentblending_b200.utils import add_frames_linear_interp, plan_frame_fill
    g = torch.Generator().manual_seed(3)
    keys = [torch.randint(0, 256, (64, 48, 3), generator=g, dtype=torch.uint8) for _ in range(5)]
    left, w0, w1 = plan_frame_fill(len(keys), 37, seed=4)
    assert len(left) == 37
    stack = torch.stack(keys, 0).cuda().contiguous().view(5, -1)
    out = ops.frames_lerp_u8(stack, torch.from_numpy(left).cuda(), torch.from_numpy(w0).cuda(),
                             torch.from_numpy(w1).cuda()).cpu().numpy().reshape(37, 64, 48, 3)
    want = add_frames_linear_interp([k.numpy() for k in keys], nmb_frames_target=37, seed=4)
    assert len(want) == 37
    for t in range(37):
        assert np.array_equal(out[t], want[t]), t        # bit-exact: float32 products, one add, truncating cast


# ---- VAE overflow guard, get_noise --------------------------------------------------------------------------------
def _tiny_pipe(turbo=False):
    from test_engine_gpu import _pair
    return _pair(turbo)


def test_vae_overflow_is_detected():
    from latentblending_b200 import DiffusersHolder, _cabi
    _, pp, _ = _tiny_pipe()
    dh = DiffusersHolder(pp)
    dh.set_dimensions((128, 128))
    lat = dh.get_noise(1) * 0.05
    dh.decode_to_device(lat)
    dh.check_decode_overflow()                                   # finite weights: nothing to report
    # weights that overflow fp16 inside the decoder (what the stock SDXL VAE does at some activations)
    sd = {k: v.clone() for k, v in pp.vae_state_dict.items()}
    sd["conv_in.weight"] = sd["conv_in.weight"] * 6.0e4
    from latentblending_b200.vae import VAEDecoderB200
    dh.vae = VAEDecoderB200(sd, pp.vae_channels, pp.vae_scaling_factor, dh.device)
    dh.decode_to_device(dh.get_noise(1))
    with pytest.raises(_cabi.LB200Error, match="overflow"):
        dh.check_decode_overflow()


@pytest.mark.parametrize("turbo", [False, True])
def test_get_noise(turbo):
    """diffusers_holder.py:98-111: randn([1,4,h,w], fp16, CUDA generator(seed)) * init_noise_sigma."""
    from latentblending_b200 import DiffusersHolder
    _, pp, _ = _tiny_pipe(turbo)
    dh = DiffusersHolder(pp)
    dh.set_dimensions((256, 128))
    dh.set_num_inference_steps(4 if turbo else 30)
    a, b, c = dh.get_noise(420), dh.get_noise(420), dh.get_noise(421)
    assert a.shape == (1, 4, 16, 32) and a.dtype == torch.float16 and a.is_cuda
    assert torch.equal(a, b) and not torch.equal(a, c)           # deterministic per seed
    g = torch.Generator(device="cuda").manual_seed(420)
    raw = torch.randn((1, 4, 16, 32), generator=g, device="cuda", dtype=torch.float16)
    sigma0 = dh.pipe.scheduler.init_noise_sigma.to(device="cuda", dtype=torch.float16)
    assert torch.equal(a, raw * sigma0)
    # known answer, restated independently in float64 from the public scaled-linear schedule (SURVEY appendix C):
    # turbo = 'trailing' spacing -> sigma(t=999) = 14.6146; base = 'leading' + offset 1 -> sqrt(sigma(t=958)^2 + 1)
    betas = np.linspace(0.00085 ** 0.5, 0.012 ** 0.5, 1000, dtype=np.float64) ** 2
    acp = np.cumprod(1.0 - betas)
    sig = np.sqrt((1 - acp) / acp)
    want = sig[999] if turbo else (sig[958] ** 2 + 1) ** 0.5
    assert abs(sig[999] - 14.6146) < 2e-3
    assert abs(float(sigma0) - want) <= 2e-3 * want, (float(sigma0), want)
    assert abs(float(a.float().std()) / float(sigma0) - 1.0) <= 0.1
    torch.manual_seed(0)
    assert torch.equal(dh.get_noise(420), a)                     # independent of the global RNG
