"""CPU tests of the SDXL ControlNet's host side: the oracle ControlNet's state-dict layout, scale 0 giving the plain
UNet, the per-step guidance window, and the diffusers-pipeline adapter on a mock StableDiffusionXLControlNetPipeline
(what it takes from ``pipe.controlnet`` and every configuration it refuses)."""
import dataclasses

import pytest
import torch

from test_boundary_cpu import MockDiffusersPipe, _Cfg, _Module


def _tiny_cn_cfg(depths=(0, 1, 2)):
    from oracle.sdxl_unet import tiny_config
    return tiny_config(transformer_layers=depths)


def _diffusers_cn_config(**kw):
    c = _Cfg(in_channels=4, conditioning_channels=3, block_out_channels=(64, 128, 256), layers_per_block=2,
             down_block_types=["DownBlock2D", "CrossAttnDownBlock2D", "CrossAttnDownBlock2D"],
             transformer_layers_per_block=[1, 1, 2], attention_head_dim=[1, 2, 4], cross_attention_dim=128,
             addition_embed_type="text_time", addition_time_embed_dim=32,
             projection_class_embeddings_input_dim=64 + 6 * 32, use_linear_projection=True, norm_num_groups=32,
             global_pool_conditions=False, controlnet_conditioning_channel_order="rgb",
             conditioning_embedding_out_channels=(16, 32, 96, 256), time_cond_proj_dim=None)
    c.update(kw)
    return c


class ControlNetModel(_Module):          # named like the diffusers class
    pass


class MultiControlNetModel(_Module):
    pass


class MockControlNetPipe(MockDiffusersPipe):
    """Duck-typed StableDiffusionXLControlNetPipeline: the mock SDXL pipeline plus ``controlnet``."""

    def __init__(self, cls=ControlNetModel, sd=None, **cfg):
        super().__init__()
        from oracle.controlnet import SDXLControlNet
        self.controlnet = cls(_diffusers_cn_config(**cfg),
                              SDXLControlNet(_tiny_cn_cfg()).state_dict() if sd is None else sd)


def test_oracle_state_dict_matches_the_diffusers_layout():
    from latentblending_b200.pipe import controlnet_param_shapes
    from latentblending_b200.unet import UNetConfig
    from oracle.controlnet import SDXLControlNet
    from oracle.sdxl_unet import SDXL_BASE, SDXLUNet
    with torch.device("meta"):
        cn = SDXLControlNet(SDXL_BASE)
        unet = SDXLUNet(SDXL_BASE)
    keys = set(cn.state_dict())
    extra = {k for k in keys if k.startswith("controlnet_")}
    want = {f"controlnet_cond_embedding.{n}.{p}" for n in ["conv_in", "conv_out"] + [f"blocks.{i}" for i in range(6)]
            for p in ("weight", "bias")}
    want |= {f"controlnet_down_blocks.{i}.{p}" for i in range(9) for p in ("weight", "bias")}
    want |= {"controlnet_mid_block.weight", "controlnet_mid_block.bias"}
    assert extra == want
    encoder = {k for k in unet.state_dict() if not k.startswith(("up_blocks.", "conv_norm_out.", "conv_out."))}
    assert keys - extra == encoder
    shapes = {k: tuple(v.shape) for k, v in cn.state_dict().items()}
    assert shapes["controlnet_cond_embedding.conv_in.weight"] == (16, 3, 3, 3)
    assert shapes["controlnet_cond_embedding.blocks.5.weight"] == (256, 96, 3, 3)
    assert shapes["controlnet_cond_embedding.conv_out.weight"] == (320, 256, 3, 3)
    assert shapes["controlnet_down_blocks.8.weight"] == (1280, 1280, 1, 1)
    # the product's list of the keys it consumes is the same layout
    cfg = UNetConfig(**{f.name: getattr(SDXL_BASE, f.name) for f in dataclasses.fields(SDXL_BASE)})
    assert dict(controlnet_param_shapes(cfg)) == shapes


def test_scale_zero_gives_the_plain_unet():
    from oracle.controlnet import SDXLControlNet, image_to_cond, synthetic_init_controlnet_, unet_with_residuals
    from oracle.sdxl_unet import SDXLUNet, synthetic_init_, tiny_config
    cfg = tiny_config()
    unet = synthetic_init_(SDXLUNet(cfg), seed=0).eval()
    cn = synthetic_init_controlnet_(SDXLControlNet(_tiny_cn_cfg()), seed=1).eval()
    g = torch.Generator().manual_seed(3)
    x = torch.randn(2, 4, 16, 8, generator=g)
    ctx = torch.randn(2, 77, cfg.cross_attention_dim, generator=g) * 0.5
    pooled = torch.randn(2, cfg.pooled_dim, generator=g)
    tids = torch.tensor([[128.0, 64.0, 0, 0, 128.0, 64.0]] * 2)
    img = image_to_cond(torch.randint(0, 256, (128, 64, 3), generator=g, dtype=torch.uint8)).expand(2, -1, -1, -1)
    with torch.no_grad():
        plain = unet(x, 500.0, ctx, pooled, tids)
        down, mid = cn(x, 500.0, ctx, pooled, tids, img, conditioning_scale=0.0)
        assert len(down) == 9 and all(float(r.abs().max()) == 0 for r in down + [mid])
        assert torch.equal(unet_with_residuals(unet, x, 500.0, ctx, pooled, tids, down, mid), plain)
        down, mid = cn(x, 500.0, ctx, pooled, tids, img, conditioning_scale=1.0)
        ctl = unet_with_residuals(unet, x, 500.0, ctx, pooled, tids, down, mid)
    assert float((ctl - plain).norm() / plain.norm()) > 1e-3        # the seeded zero convs are not zero


@pytest.mark.parametrize("start,end,N,idx_start", [(0.0, 1.0, 30, 0), (0.0, 0.5, 30, 0), (0.2, 0.8, 30, 11),
                                                   (0.25, 1.0, 4, 2), (0.0, 0.3, 7, 0), (0.5, 0.6, 10, 3)])
def test_keep_window(start, end, N, idx_start):
    from latentblending_b200.controlnet import keep_scale
    from oracle.controlnet import controlnet_keep
    for i in range(idx_start, N):
        want = 1.0 - float(i / N < start or (i + 1) / N > end)
        assert keep_scale(i, N, start, end) == controlnet_keep(i, N, start, end) == want
    on = [i for i in range(N) if keep_scale(i, N, start, end)]
    assert all(start <= i / N and (i + 1) / N <= end for i in on)


def test_diffusers_controlnet_pipeline_is_adapted():
    from latentblending_b200.pipe import DiffusersSDXLPipe, adapt_pipe
    mock = MockControlNetPipe()
    pipe = adapt_pipe(mock)
    assert isinstance(pipe, DiffusersSDXLPipe)
    assert pipe.controlnet_cfg.transformer_layers == (0, 1, 2)
    assert pipe.controlnet_cfg.block_out_channels == pipe.unet_cfg.block_out_channels
    assert pipe.controlnet_state_dict is mock.controlnet.state_dict()
    assert pipe.controlnet_cond_channels == (16, 32, 96, 256) and not pipe.controlnet_bgr
    assert adapt_pipe(MockControlNetPipe(controlnet_conditioning_channel_order="bgr")).controlnet_bgr
    from oracle.controlnet import SDXLControlNet
    small = MockControlNetPipe(transformer_layers_per_block=[0, 0, 1],
                               sd=SDXLControlNet(_tiny_cn_cfg((0, 0, 1))).state_dict())
    assert adapt_pipe(small).controlnet_cfg.transformer_layers == (0, 0, 1)
    # a pipeline without a ControlNet
    assert adapt_pipe(MockDiffusersPipe()).controlnet_state_dict is None


@pytest.mark.parametrize("case", ["multi", "global_pool", "channels", "cond_proj", "levels", "channels_mismatch",
                                  "leftover", "missing", "shape"])
def test_refused_controlnets(case):
    from latentblending_b200.pipe import adapt_pipe
    from oracle.controlnet import SDXLControlNet
    sd = dict(SDXLControlNet(_tiny_cn_cfg()).state_dict())
    kw = {}
    if case == "multi":
        mock = MockControlNetPipe(cls=MultiControlNetModel)
    else:
        if case == "global_pool":
            kw = dict(global_pool_conditions=True)
        elif case == "channels":
            kw = dict(conditioning_channels=1)
        elif case == "cond_proj":
            kw = dict(time_cond_proj_dim=256)
        elif case == "levels":
            kw = dict(block_out_channels=(64, 128), down_block_types=["DownBlock2D", "CrossAttnDownBlock2D"],
                      transformer_layers_per_block=[1, 1], attention_head_dim=[1, 2])
        elif case == "channels_mismatch":
            kw = dict(block_out_channels=(64, 128, 320), attention_head_dim=[1, 2, 5])
        elif case == "leftover":          # e.g. a "mid"/"small" variant with a layer the lowering has no place for
            sd["controlnet_cond_embedding.blocks.6.weight"] = torch.zeros(256, 256, 3, 3)
        elif case == "missing":
            del sd["controlnet_down_blocks.3.bias"]
        elif case == "shape":
            sd["controlnet_mid_block.weight"] = torch.zeros(256, 128, 1, 1)
        mock = MockControlNetPipe(sd=sd, **kw)
    with pytest.raises(ValueError):
        adapt_pipe(mock)


def test_synthetic_pipe_controlnet_weights():
    from latentblending_b200.pipe import SyntheticSDXLPipe, controlnet_param_shapes
    from latentblending_b200.unet import UNetConfig
    with pytest.raises(ValueError):
        from latentblending_b200.pipe import controlnet_config
        controlnet_config(UNetConfig(), "medium")
    cfg = UNetConfig(block_out_channels=(64, 128, 256), transformer_layers=(0, 1, 2), cross_attention_dim=128,
                     addition_time_embed_dim=32, pooled_dim=64, sample_size=16)
    for variant, depths in (("full", (0, 1, 2)), ("small", (0, 0, 1))):
        pipe = SyntheticSDXLPipe(device="cpu", unet_cfg=cfg, controlnet=variant, vae="tiny")
        assert pipe.controlnet_cfg.transformer_layers == depths
        sd = pipe.controlnet_state_dict
        assert {k: tuple(v.shape) for k, v in sd.items()} == dict(controlnet_param_shapes(pipe.controlnet_cfg))
        for k in [k for k in sd if k.startswith(("controlnet_down_blocks.", "controlnet_mid_block."))]:
            assert float(sd[k].float().abs().max()) > 0, k
    assert SyntheticSDXLPipe(device="cpu", unet_cfg=cfg, vae="tiny").controlnet_state_dict is None
