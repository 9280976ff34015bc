"""CPU tests of the tiny VAE decoder's host side (AutoencoderTiny / TAESDXL, latentblending_b200/taesd.py): the
phase-weight packing of the depth-to-space GEMM against upsample + conv in float64, the layer layout the packer
derives from a config against the oracle's nn.Sequential, the diffusers adapter, every rejected config / key set, and
the fixtures' seeded weights."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F


def _d2s_ref_and_packed(B, H, W, Ci, Co, seed):
    from latentblending_b200.taesd import pack_d2s_weights
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, Ci, H, W, generator=g, dtype=torch.float64)
    w = torch.randn(Co, Ci, 3, 3, generator=g, dtype=torch.float64)
    ref = F.conv2d(F.interpolate(x, scale_factor=2, mode="nearest"), w, padding=1)
    low = F.conv2d(x, pack_d2s_weights(w), padding=1)                       # [B, 4*Co, H, W], channel p*Co + c
    got = torch.empty_like(ref)
    for a in range(2):
        for b in range(2):
            got[:, :, a::2, b::2] = low[:, (2 * a + b) * Co:(2 * a + b + 1) * Co]
    return got, ref


@pytest.mark.parametrize("B", [1, 2])
@pytest.mark.parametrize("H,W", [(1, 1), (5, 7), (13, 24), (16, 16)])
@pytest.mark.parametrize("Co", [8, 64])
def test_phase_weights_equal_upsample_then_conv(B, H, W, Co):
    """Every output pixel, borders included: the four phase filters over the low-resolution map equal nearest-2x
    upsample + 3x3 conv (padding 1) in float64."""
    got, ref = _d2s_ref_and_packed(B, H, W, 16, Co, seed=B * 1000 + H * 31 + W + Co)
    assert (got - ref).abs().max().item() <= 1e-12 * max(1.0, ref.abs().max().item())


def test_phase_weights_zero_unused_taps():
    """A phase reads 2 of the 3 low-resolution rows and 2 of the 3 columns: its other 5 taps are exactly zero."""
    from latentblending_b200.taesd import pack_d2s_weights
    w = torch.ones(8, 4, 3, 3, dtype=torch.float64)
    p = pack_d2s_weights(w).view(2, 2, 8, 4, 3, 3)
    assert torch.all(p[0, :, :, :, 2, :] == 0) and torch.all(p[1, :, :, :, 0, :] == 0)
    assert torch.all(p[:, 0, :, :, :, 2] == 0) and torch.all(p[:, 1, :, :, :, 0] == 0)
    assert torch.all(p.sum(dim=(-1, -2)) == 9)                                  # every original tap lands once


@pytest.mark.parametrize("nb", [(3, 3, 3, 1), (1, 1, 1, 1), (2, 1)])
def test_oracle_keys_match_packer_layout(nb):
    from latentblending_b200.pipe import tiny_vae_param_shapes
    from latentblending_b200.taesd import expected_keys
    from oracle.taesd import DecoderTiny, TinyVAEConfig
    cfg = TinyVAEConfig(num_decoder_blocks=nb, decoder_block_out_channels=(64,) * len(nb))
    dec = DecoderTiny(cfg)
    conf = dict(num_decoder_blocks=nb, decoder_block_out_channels=(64,) * len(nb))
    assert sorted(dec.state_dict()) == sorted(expected_keys(conf))
    shapes = tiny_vae_param_shapes(conf)
    assert {k: tuple(v.shape) for k, v in dec.state_dict().items()} == dict(shapes)


def test_default_layout_is_the_diffusers_one():
    from latentblending_b200.taesd import decoder_layout
    lay = decoder_layout()
    assert [i for k, i, _ in lay if k == "block"] == [2, 3, 4, 7, 8, 9, 12, 13, 14, 17]
    assert [i for k, i, _ in lay if k == "up_conv"] == [6, 11, 16]
    assert [(k, i) for k, i, _ in lay if k in ("conv_in", "conv_out")] == [("conv_in", 0), ("conv_out", 18)]


class AutoencoderTiny:                      # named like the diffusers class the adapter keys on
    def __init__(self, config, sd):
        self.config, self._sd = config, sd

    def state_dict(self):
        return self._sd


def _mock_tiny_pipe(sd=None, **cfg):
    from test_boundary_cpu import MockDiffusersPipe, _Cfg
    from latentblending_b200.pipe import random_tiny_vae_state_dict
    mock = MockDiffusersPipe()
    sd = random_tiny_vae_state_dict(3, "cpu") if sd is None else sd
    vsd = {"decoder." + k: v for k, v in sd.items()}
    vsd["encoder.layers.0.weight"] = torch.zeros(1)
    config = _Cfg(latent_channels=4, out_channels=3, decoder_block_out_channels=(64, 64, 64, 64),
                  num_decoder_blocks=(3, 3, 3, 1), upsampling_scaling_factor=2, act_fn="relu", scaling_factor=1.0,
                  force_upcast=False)
    config.update(cfg)
    mock.vae = AutoencoderTiny(config, vsd)
    return mock


def test_adapter_recognises_autoencoder_tiny():
    from latentblending_b200.pipe import adapt_pipe, random_tiny_vae_state_dict
    p = adapt_pipe(_mock_tiny_pipe())
    assert p.vae_kind == "tiny" and p.vae_dtype == "fp16" and p.vae_scaling_factor == 1.0
    assert set(p.vae_state_dict) == set(random_tiny_vae_state_dict(3, "cpu"))
    assert not any(k.startswith(("decoder.", "encoder.")) for k in p.vae_state_dict)
    assert p.vae_config["num_decoder_blocks"] == (3, 3, 3, 1)


def test_adapter_keeps_kl_for_autoencoder_kl():
    from test_boundary_cpu import MockDiffusersPipe
    from latentblending_b200.pipe import adapt_pipe
    assert adapt_pipe(MockDiffusersPipe()).vae_kind == "kl"


@pytest.mark.parametrize("cfg", [dict(decoder_block_out_channels=(64, 64, 128, 64)),
                                 dict(decoder_block_out_channels=(48, 48, 48, 48)),
                                 dict(upsampling_scaling_factor=3), dict(act_fn="silu"), dict(latent_channels=16),
                                 dict(out_channels=4)])
def test_rejected_configs(cfg):
    from latentblending_b200.pipe import adapt_pipe
    with pytest.raises(ValueError):
        adapt_pipe(_mock_tiny_pipe(**cfg))


def test_rejected_key_sets_name_the_keys():
    from latentblending_b200.pipe import adapt_pipe, random_tiny_vae_state_dict
    sd = random_tiny_vae_state_dict(3, "cpu")
    missing = dict(sd)
    del missing["layers.7.conv.2.bias"]
    with pytest.raises(ValueError, match=r"missing \['layers.7.conv.2.bias'\]"):
        adapt_pipe(_mock_tiny_pipe(missing))
    extra = dict(sd)
    extra["layers.6.bias"] = torch.zeros(64)                 # the upsampling convs have no bias
    with pytest.raises(ValueError, match=r"unexpected \['layers.6.bias'\]"):
        adapt_pipe(_mock_tiny_pipe(extra))
    with pytest.raises(ValueError, match="missing"):
        adapt_pipe(_mock_tiny_pipe(sd, num_decoder_blocks=(3, 3, 3, 2)))


def test_synthetic_pipe_tiny_option():
    from latentblending_b200.pipe import SyntheticSDXLPipe
    from latentblending_b200.taesd import expected_keys
    from latentblending_b200.unet import UNetConfig
    tiny = UNetConfig(block_out_channels=(64, 128, 256), transformer_layers=(0, 1, 2), cross_attention_dim=128,
                      addition_time_embed_dim=32, pooled_dim=64, sample_size=16)
    p = SyntheticSDXLPipe(device="cpu", unet_cfg=tiny, unet_state_dict={}, vae="tiny")
    assert p.vae_kind == "tiny" and p.vae_dtype == "fp16" and p.vae_scaling_factor == 1.0
    assert set(p.vae_state_dict) == set(expected_keys())
    assert SyntheticSDXLPipe(device="cpu", unet_cfg=tiny, unet_state_dict={}, vae_state_dict={}).vae_kind == "kl"
    with pytest.raises(ValueError):
        SyntheticSDXLPipe(device="cpu", unet_cfg=tiny, unet_state_dict={}, vae="tiny", vae_dtype="bf16")
    with pytest.raises(ValueError):
        SyntheticSDXLPipe(device="cpu", unet_cfg=tiny, unet_state_dict={}, vae="taesd")


def test_fixtures_match_seeded_recipe():
    from make_fullsize_fixtures import vae_latent, weights_checksum
    from make_taesd_fixtures import FIXTURES, SAMPLED, sample_indices, tiny_state_dict
    sha = weights_checksum(tiny_state_dict())
    for (h, w), path in FIXTURES.items():
        fx = np.load(path)
        assert str(fx["weights_sha1"]) == sha, "seeded tiny VAE recipe drifted"
        assert np.array_equal(fx["latents"], vae_latent(h, w).numpy())
        f = fx["frame"]
        if (h, w) in SAMPLED:
            rows, cols = sample_indices(8 * h), sample_indices(8 * w)
            assert np.array_equal(fx["rows"], rows) and np.array_equal(fx["cols"], cols)
            for idx, n in ((rows, 8 * h), (cols, 8 * w)):      # every phase of the three 2x levels, both borders
                assert set(np.unique(idx % 8)) == set(range(8)) and idx[0] == 0 and idx[-1] == n - 1
            assert f.shape == (len(rows), len(cols), 3) and f.dtype == np.uint8
        else:
            assert f.shape == (8 * h, 8 * w, 3) and f.dtype == np.uint8
        assert f.std() > 5 and ((f == 0) | (f == 255)).mean() < 0.1        # not degenerate


def test_oracle_reproduces_small_fixture_region():
    """The oracle on the fixture's weights reproduces the stored 512^2 frame exactly (same CPU arithmetic)."""
    from make_taesd_fixtures import FIXTURES, oracle_taesd
    from oracle.taesd import latent2image_np
    fx = np.load(FIXTURES[(64, 64)])
    with torch.no_grad():
        frame = latent2image_np(oracle_taesd(), torch.from_numpy(fx["latents"]))
    assert np.abs(frame.astype(np.int32) - fx["frame"].astype(np.int32)).max() <= 1
