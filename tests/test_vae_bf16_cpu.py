"""CPU tests of the bf16 VAE decoder's host side: which precision the adapters pick (the VAE config's force_upcast,
as the reference decides when to upcast, diffusers_holder.py:128-139), and the property the upcast fixture
(tests/golden/make_upcast_fixtures.py) is built on: its activations overflow fp16 but not bf16."""
import numpy as np
import pytest
import torch


def _mock_pipe(**vae_cfg):
    from test_boundary_cpu import MockDiffusersPipe, _Cfg
    mock = MockDiffusersPipe()
    cfg = _Cfg(block_out_channels=(64, 64, 128, 128), scaling_factor=0.13025)
    cfg.update(vae_cfg)
    mock.vae.config = cfg
    return mock


@pytest.mark.parametrize("cfg,want", [(dict(force_upcast=True), "bf16"), (dict(force_upcast=False), "fp16"),
                                      (dict(), "bf16")])
def test_adapter_picks_vae_dtype_from_force_upcast(cfg, want):
    from latentblending_b200.pipe import adapt_pipe
    assert adapt_pipe(_mock_pipe(**cfg)).vae_dtype == want


def test_vae_dtype_from_attribute_config():
    from latentblending_b200.pipe import vae_dtype_from_config

    class Cfg:
        force_upcast = False
    assert vae_dtype_from_config(Cfg()) == "fp16"
    assert vae_dtype_from_config(object()) == "bf16"      # missing: the diffusers default (True)


def test_synthetic_pipe_defaults_to_fp16():
    from latentblending_b200.pipe import SyntheticSDXLPipe
    from latentblending_b200.unet import UNetConfig
    tiny = UNetConfig(block_out_channels=(64, 128, 256), transformer_layers=(0, 1, 2), cross_attention_dim=128,
                      addition_time_embed_dim=32, pooled_dim=64, sample_size=16)
    vsd = {"x": torch.zeros(1)}
    p = SyntheticSDXLPipe(device="cpu", unet_cfg=tiny, unet_state_dict={}, vae_state_dict=vsd)
    assert p.vae_dtype == "fp16"
    assert SyntheticSDXLPipe(device="cpu", unet_cfg=tiny, unet_state_dict={}, vae_state_dict=vsd,
                             vae_dtype="bf16").vae_dtype == "bf16"
    with pytest.raises(ValueError):
        SyntheticSDXLPipe(device="cpu", unet_cfg=tiny, unet_state_dict={}, vae_state_dict=vsd, vae_dtype="fp32")


def _tiny_upcast_vae():
    from make_upcast_fixtures import upcast_
    from oracle.vae import VAEConfig, VAEDecoder, synthetic_vae_init_
    cfg = VAEConfig(block_out_channels=(64, 64, 128, 128))
    ov = synthetic_vae_init_(VAEDecoder(cfg), seed=4).eval()
    with torch.no_grad():
        for p in ov.parameters():
            p.copy_(p.half().float())
    return upcast_(ov)


def test_upcast_recipe_overflows_fp16_not_bf16():
    """fp32 oracle activations exceed fp16's range; the same module cast to fp16 decodes to non-finite values, cast
    to bf16 to finite ones."""
    from make_fullsize_fixtures import vae_latent
    from make_upcast_fixtures import FP16_MAX, max_activation
    ov = _tiny_upcast_vae()
    lat = vae_latent(16, 16)
    _, peak = max_activation(ov, lat)
    assert peak > FP16_MAX
    with torch.no_grad():
        z = lat.float() / ov.cfg.scaling_factor
        out16 = ov.to(torch.float16)(z.half()).float()
        outb = ov.to(torch.bfloat16)(z.bfloat16()).float()
    assert not torch.isfinite(out16).all()
    assert torch.isfinite(outb).all()


def test_upcast_fixture_records_overflow():
    from make_upcast_fixtures import FP16_MAX, UPCAST_FIXTURE
    fx = np.load(UPCAST_FIXTURE)
    assert float(fx["max_abs_activation"]) > FP16_MAX
    assert fx["frame"].shape == (512, 512, 3) and fx["frame"].dtype == np.uint8 and fx["frame"].std() > 5
