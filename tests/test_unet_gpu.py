"""GPU parity of the lowered UNet program (liblb200) against the CPU oracle UNet
(oracle/sdxl_unet.py, fp32) on identical seeded weights and inputs.
Tolerance (stated): relative L2 error of eps <= 2e-3 (SURVEY section 8c) -- fp16 storage of every
activation with fp32 accumulation vs an all-fp32 oracle.  At the BENCHMARKED shape
(full SDXL-base, CFG batch 2, 128x128 latents) the comparison is against the committed
fixture tests/golden/unet_sdxl_b2_128.npz (tests/golden/make_fullsize_fixtures.py).
Measured rel-L2 values are printed (-s)."""
import dataclasses

import pytest
import torch

pytestmark = pytest.mark.gpu


def _inputs(cfg, B, h, w, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, 4, h, w, generator=g).half()
    ctx = (torch.randn(B, 77, cfg.cross_attention_dim, generator=g) * 0.5).half()
    pooled = torch.randn(B, cfg.pooled_dim, generator=g).half()
    tids = torch.tensor([[8.0 * h, 8.0 * w, 0, 0, 8.0 * h, 8.0 * w]] * B).half()
    return x, ctx, pooled, tids


def _run_pair(ocfg, B, h, w, t, seed=0):
    from latentblending_b200.unet import UNetB200, UNetConfig
    from oracle.sdxl_unet import SDXLUNet, synthetic_init_
    oracle = synthetic_init_(SDXLUNet(ocfg), seed=seed).eval()
    # the CUDA path stores weights in fp16: give the oracle the same (rounded) weights
    with torch.no_grad():
        for p in oracle.parameters():
            p.copy_(p.half().float())
    cfg = UNetConfig(**{f.name: getattr(ocfg, f.name) for f in dataclasses.fields(ocfg)})
    net = UNetB200(cfg, oracle.state_dict(), "cuda:0")
    x, ctx, pooled, tids = _inputs(ocfg, B, h, w, seed)
    with torch.no_grad():
        ref = oracle(x.float(), t, ctx.float(), pooled.float(), tids.float())
    eps = net.forward(x.cuda(), t, ctx.cuda(), pooled.cuda(), tids.cuda()).float().cpu()
    torch.cuda.synchronize()
    from latentblending_b200 import ops
    assert ops.error_flag() == 0
    rel = ((eps - ref).norm() / ref.norm()).item()
    print(f"unet parity: B={B} h={h} w={w} t={t} rel_l2={rel:.3e}")
    return rel, eps, ref, net


@pytest.mark.parametrize("B,h,w,t", [(2, 16, 16, 958.0), (1, 16, 16, 249.0), (2, 32, 16, 1.0),
                                     (2, 32, 16, 321.0)])
def test_tiny_unet_matches_oracle(B, h, w, t):
    from oracle.sdxl_unet import tiny_config
    rel, eps, ref, net = _run_pair(tiny_config(), B, h, w, t)
    assert torch.isfinite(eps).all()
    assert rel <= 2e-3, f"relative L2 error {rel}"
    # replaying the recorded program is deterministic
    x, ctx, pooled, tids = _inputs(tiny_config(), B, h, w)
    again = net.forward(x.cuda(), t, ctx.cuda(), pooled.cuda(), tids.cuda()).float().cpu()
    assert torch.equal(again, eps)


def test_medium_unet_matches_oracle():
    """SDXL topology (transformer depths 0/2/10, 10/20 heads ...) at reduced width."""
    from oracle.sdxl_unet import UNetConfig
    ocfg = UNetConfig(block_out_channels=(128, 256, 512), transformer_layers=(0, 2, 10), cross_attention_dim=256,
                      addition_time_embed_dim=64, pooled_dim=128, sample_size=32)
    rel, eps, ref, _ = _run_pair(ocfg, 2, 32, 32, 499.0)
    assert torch.isfinite(eps).all()
    assert rel <= 2e-3, f"relative L2 error {rel}"


_FULL = {}


def _full_sdxl():
    """The seeded full-size oracle UNet (2.57 B parameters, ~1 min of CPU init) and its CUDA twin, built once."""
    if not _FULL:
        from latentblending_b200.unet import UNetB200, UNetConfig
        from make_fullsize_fixtures import oracle_unet, weights_checksum
        from oracle.sdxl_unet import SDXL_BASE
        oracle = oracle_unet()
        cfg = UNetConfig(**{f.name: getattr(SDXL_BASE, f.name) for f in dataclasses.fields(SDXL_BASE)})
        _FULL.update(oracle=oracle, net=UNetB200(cfg, oracle.state_dict(), "cuda:0"),
                     sha=weights_checksum(oracle.state_dict()))
    return _FULL


@pytest.mark.slow
def test_full_sdxl_unet_matches_oracle_at_256px():
    """The real SDXL-base architecture (2.57 B parameters), 32x32 latents, CFG batch 2."""
    from latentblending_b200 import ops
    from oracle.sdxl_unet import SDXL_BASE
    full = _full_sdxl()
    x, ctx, pooled, tids = _inputs(SDXL_BASE, 2, 32, 32, 0)
    with torch.no_grad():
        ref = full["oracle"](x.float(), 925.0, ctx.float(), pooled.float(), tids.float())
    eps = full["net"].forward(x.cuda(), 925.0, ctx.cuda(), pooled.cuda(), tids.cuda()).float().cpu()
    assert ops.error_flag() == 0
    rel = ((eps - ref).norm() / ref.norm()).item()
    print(f"full SDXL UNet @32x32 B=2: rel_l2={rel:.3e}")
    assert torch.isfinite(eps).all()
    assert rel <= 2e-3, f"relative L2 error {rel}"
    assert full["net"].launches_per_forward(2, 32, 32)[0] > 600


@pytest.mark.slow
def test_full_sdxl_unet_matches_fixture_at_bench_shape():
    """Parity AT THE BENCHMARKED SHAPE: one CFG-batch-2 forward of the full SDXL-base UNet at 128x128 latents vs the
    fp32 oracle output committed as a fixture (the oracle needs ~30 s x 8 cores for this forward; the GPU box only
    rebuilds the seeded weights, whose checksum is verified first)."""
    from latentblending_b200 import ops
    from make_fullsize_fixtures import UNET_FIXTURE, UNET_SEED, UNET_T, unet_inputs
    from oracle.sdxl_unet import SDXL_BASE
    import numpy as np
    fx = np.load(UNET_FIXTURE)
    full = _full_sdxl()
    assert full["sha"] == str(fx["weights_sha1"]), "seeded weight recipe drifted from the fixture's"
    x, ctx, pooled, tids = unet_inputs(SDXL_BASE, 2, 128, 128, UNET_SEED)
    eps = full["net"].forward(x.cuda(), float(fx["t"]), ctx.cuda(), pooled.cuda(), tids.cuda()).float().cpu()
    torch.cuda.synchronize()
    assert ops.error_flag() == 0
    ref = torch.from_numpy(fx["eps"])
    assert float(fx["t"]) == UNET_T and eps.shape == ref.shape == (2, 4, 128, 128)
    rel = ((eps - ref).norm() / ref.norm()).item()
    mse = ((eps - ref) ** 2).mean().item()
    print(f"full SDXL UNet @128x128 B=2 (bench shape): rel_l2={rel:.3e} mse={mse:.3e} max={float((eps - ref).abs().max()):.3e}")
    assert torch.isfinite(eps).all()
    assert rel <= 2e-3, f"relative L2 error {rel}"
    # batch invariance at the bench shape: each CFG half alone reproduces its half of the batch-2 forward bit for bit
    # (what the multi-GPU CFG split and the lockstep batching rely on)
    for b in range(2):
        one = full["net"].forward(x[b:b + 1].cuda(), float(fx["t"]), ctx[b:b + 1].cuda(), pooled[b:b + 1].cuda(),
                                  tids[b:b + 1].cuda()).float().cpu()
        assert torch.equal(one[0], eps[b]), f"batch-1 forward of half {b} differs from the batch-2 forward"
