"""CPU tests of the SDXL T2I-Adapter's host side: the parameter counts and state-dict layout, the feature shapes at
the common output sizes, the int(N * factor) step window, every adapter the backend refuses, and which step program
the denoise loop picks at each step."""
import types

import numpy as np
import pytest
import torch

from test_boundary_cpu import MockDiffusersPipe, _Cfg, _Module
from test_controlnet_cpu import MockControlNetPipe


def _count(shapes):
    return sum(int(np.prod(s)) for s in shapes.values())


@pytest.mark.parametrize("cin,want", [(3, 79_028_160), (1, 77_553_600)])
def test_parameter_counts(cin, want):
    from latentblending_b200.pipe import adapter_param_shapes
    from oracle.t2i_adapter import T2IAdapter
    with torch.device("meta"):
        ad = T2IAdapter(cin)
    assert sum(p.numel() for p in ad.parameters()) == want
    assert _count(adapter_param_shapes(cin)) == want


@pytest.mark.parametrize("cin", [1, 3])
def test_state_dict_layout(cin):
    from latentblending_b200.pipe import adapter_param_shapes
    from oracle.t2i_adapter import T2IAdapter
    with torch.device("meta"):
        ad = T2IAdapter(cin)
    shapes = {k: tuple(v.shape) for k, v in ad.state_dict().items()}
    assert shapes == dict(adapter_param_shapes(cin))
    assert "adapter.body.0.in_conv.weight" not in shapes and "adapter.body.3.in_conv.weight" not in shapes
    assert shapes["adapter.body.1.in_conv.weight"] == (640, 320, 1, 1)
    assert shapes["adapter.body.2.in_conv.weight"] == (1280, 640, 1, 1)
    assert shapes["adapter.conv_in.weight"] == (320, 256 * cin, 3, 3)


@pytest.mark.parametrize("H,W", [(1024, 1024), (720, 1280), (1216, 832)])
def test_feature_shapes(H, W):
    """The restated FullAdapterXL (narrow channels, same spatial path) gives feature_shapes', and they are the shapes
    of the UNet's injection points for H/8 x W/8 latents: the level-1 map for 0 and 1, the level-2 map for 2 and 3."""
    from latentblending_b200.t2i_adapter import feature_shapes
    from oracle.t2i_adapter import FullAdapterXL
    ch = (8, 16, 32, 32)
    ad = FullAdapterXL(3, ch)
    with torch.no_grad():
        feats = ad(torch.zeros(1, 3, H, W))
    got = feature_shapes(H, W, ch)
    assert [(f.shape[2], f.shape[3], f.shape[1]) for f in feats] == got
    h, w = H // 8, W // 8
    l1 = ((h + 1) // 2, (w + 1) // 2)
    l2 = ((l1[0] + 1) // 2, (l1[1] + 1) // 2)
    assert [g[:2] for g in got] == [l1, l1, l2, l2]
    if (H, W) == (720, 1280):
        assert got[0][:2] == (45, 80) and got[2][:2] == (23, 40)


def test_sizes_that_are_not_multiples_of_16_are_refused():
    from latentblending_b200.t2i_adapter import check_image_size
    check_image_size(720, 1280)
    for H, W in ((1080, 1920), (1024, 1000), (8, 16)):
        with pytest.raises(ValueError, match="multiples of 16"):
            check_image_size(H, W)


@pytest.mark.parametrize("N", [1, 4, 7, 30, 50])
@pytest.mark.parametrize("factor", [0.0, 0.25, 0.5, 0.8, 0.99, 1.0])
def test_factor_window(N, factor):
    from latentblending_b200.t2i_adapter import adapter_steps
    from oracle.t2i_adapter import adapter_factor_steps
    assert adapter_steps(N, factor) == adapter_factor_steps(N, factor) == int(N * factor)


def _stub_holder(scale=1.0, factor=1.0, image=True, control=None):
    """A DiffusersHolder without a device: only the per-step program choice is exercised."""
    from latentblending_b200.diffusers_holder import DiffusersHolder
    dh = object.__new__(DiffusersHolder)
    dh.control = control
    dh.adapter_cond = dict(image=None, scale=scale, factor=factor, computed=set()) if image else None
    return dh


def test_step_program_choice():
    plan = types.SimpleNamespace(prog_step="plain", prog_step_cn="controlnet", prog_step_ad="adapter")
    for N, factor in ((30, 1.0), (30, 0.5), (30, 0.0), (7, 0.8), (4, 0.3)):
        dh = _stub_holder(factor=factor)
        got = [dh.step_program(plan, i, N) for i in range(N)]
        k = int(N * factor)
        assert got == ["adapter"] * k + ["plain"] * (N - k)
    assert all(_stub_holder(scale=0.0).step_program(plan, i, 30) == "plain" for i in range(30))
    assert all(_stub_holder(image=False).step_program(plan, i, 30) == "plain" for i in range(30))
    dh = _stub_holder(factor=0.5)
    assert [dh.adapter_active(i, 30) for i in (0, 14, 15, 29)] == [True, True, False, False]


def test_engine_passes_the_adapter_image_to_the_holder():
    from fakes import FakeHolder, fake_similarity
    from latentblending_b200 import BlendingEngine

    class AdapterFakeHolder(FakeHolder):
        def __init__(self):
            super().__init__()
            self.adapter_calls = []

        def set_adapter_image(self, image, conditioning_scale=1.0, conditioning_factor=1.0):
            self.adapter_calls.append((None if image is None else image.shape, conditioning_scale,
                                       conditioning_factor))

    holder = AdapterFakeHolder()
    be = BlendingEngine(None, holder=holder, similarity_fn=fake_similarity, run_benchmark=False)
    img = np.zeros((64, 48), dtype=np.uint8)
    be.set_adapter_image(img, 0.7, 0.5)
    be.set_adapter_image(img)
    be.set_adapter_image(None)
    assert holder.adapter_calls == [((64, 48), 0.7, 0.5), ((64, 48), 1.0, 1.0), (None, 1.0, 1.0)]


# ---- the diffusers pipeline adapter ---------------------------------------------------------------------------------
class T2IAdapter(_Module):           # named like the diffusers classes
    pass


class MultiAdapter(_Module):
    pass


def _tiny_adapter_cfg(**kw):
    c = _Cfg(in_channels=3, channels=(64, 128, 256, 256), num_res_blocks=2, downscale_factor=16,
             adapter_type="full_adapter_xl")
    c.update(kw)
    return c


def _tiny_adapter_sd(cin=3, channels=(64, 128, 256, 256)):
    from oracle.t2i_adapter import T2IAdapter as OracleAdapter
    return OracleAdapter(cin, channels).state_dict()


class MockAdapterPipe(MockDiffusersPipe):
    """Duck-typed StableDiffusionXLAdapterPipeline: the mock SDXL pipeline plus ``adapter``."""

    def __init__(self, cls=T2IAdapter, sd=None, **cfg):
        super().__init__()
        c = _tiny_adapter_cfg(**cfg)
        self.adapter = cls(c, _tiny_adapter_sd(c["in_channels"]) if sd is None else sd)


def test_diffusers_adapter_pipeline_is_adapted():
    from latentblending_b200.pipe import DiffusersSDXLPipe, adapt_pipe
    mock = MockAdapterPipe()
    pipe = adapt_pipe(mock)
    assert isinstance(pipe, DiffusersSDXLPipe)
    assert pipe.adapter_cfg == dict(in_channels=3, channels=(64, 128, 256, 256), num_res_blocks=2,
                                    downscale_factor=16, adapter_type="full_adapter_xl")
    assert pipe.adapter_state_dict is mock.adapter.state_dict()
    assert adapt_pipe(MockAdapterPipe(in_channels=1)).adapter_cfg["in_channels"] == 1
    assert adapt_pipe(MockDiffusersPipe()).adapter_state_dict is None


@pytest.mark.parametrize("case", ["multi", "full_adapter", "light_adapter", "in_channels", "channels", "downscale",
                                  "leftover", "missing", "shape", "with_controlnet"])
def test_refused_adapters(case):
    from latentblending_b200.pipe import adapt_pipe
    sd = dict(_tiny_adapter_sd())
    kw = {}
    if case == "multi":
        mock = MockAdapterPipe(cls=MultiAdapter)
    elif case == "with_controlnet":
        mock = MockControlNetPipe()
        mock.adapter = T2IAdapter(_tiny_adapter_cfg(), sd)
    else:
        if case in ("full_adapter", "light_adapter"):
            kw = dict(adapter_type=case)
        elif case == "in_channels":
            kw = dict(in_channels=4)
            sd["adapter.conv_in.weight"] = torch.zeros(64, 4 * 256, 3, 3)
        elif case == "channels":
            kw = dict(channels=(64, 128, 256, 512))
        elif case == "downscale":
            kw = dict(downscale_factor=8)
        elif case == "leftover":
            sd["adapter.body.0.in_conv.weight"] = torch.zeros(64, 64, 1, 1)
        elif case == "missing":
            del sd["adapter.body.2.resnets.1.block2.bias"]
        elif case == "shape":
            sd["adapter.body.3.resnets.0.block1.weight"] = torch.zeros(256, 256, 1, 1)
        mock = MockAdapterPipe(sd=sd, **kw)
    with pytest.raises(ValueError):
        adapt_pipe(mock)


def test_packed_adapter_refuses_unconsumed_keys():
    from latentblending_b200.t2i_adapter import PackedAdapter
    sd = dict(_tiny_adapter_sd())
    cfg = dict(_tiny_adapter_cfg())
    assert set(PackedAdapter(cfg, sd, "cpu").consumed) == set(sd)
    sd["adapter.extra.weight"] = torch.zeros(1)
    with pytest.raises(ValueError):
        PackedAdapter(cfg, sd, "cpu")
    with pytest.raises(ValueError):
        PackedAdapter(dict(cfg, adapter_type="light_adapter"), _tiny_adapter_sd(), "cpu")


def test_unet_requirements():
    """UNetB200 checks the adapter against the UNet before packing anything."""
    from latentblending_b200.unet import UNetB200, UNetConfig
    cfg = UNetConfig(block_out_channels=(64, 128, 256), transformer_layers=(0, 1, 2))
    ok = types.SimpleNamespace(channels=(64, 128, 256, 256))
    for adapter, ucfg, cn in ((types.SimpleNamespace(channels=(64, 128, 256, 512)), cfg, None),
                              (types.SimpleNamespace(channels=(64, 128, 128)), UNetConfig(block_out_channels=(64, 128),
                                                                                          transformer_layers=(0, 1)),
                               None),
                              (ok, cfg, object())):
        with pytest.raises(ValueError):
            UNetB200(ucfg, {}, "cpu", controlnet=cn, adapter=adapter)


def test_synthetic_pipe_adapter_weights():
    from latentblending_b200.pipe import SyntheticSDXLPipe, adapter_param_shapes
    from latentblending_b200.unet import UNetConfig
    cfg = UNetConfig(block_out_channels=(64, 128, 256), transformer_layers=(0, 1, 2), cross_attention_dim=128,
                     addition_time_embed_dim=32, pooled_dim=64, sample_size=16)
    with pytest.raises(ValueError):
        SyntheticSDXLPipe(device="cpu", unet_cfg=cfg, adapter="depth", vae="tiny")
    with pytest.raises(ValueError):
        SyntheticSDXLPipe(device="cpu", unet_cfg=cfg, adapter="rgb", controlnet="small", vae="tiny")
    plain = SyntheticSDXLPipe(device="cpu", unet_cfg=cfg, vae="tiny")
    assert plain.adapter_state_dict is None
    for variant, cin in (("rgb", 3), ("gray", 1)):
        pipe = SyntheticSDXLPipe(device="cpu", unet_cfg=cfg, adapter=variant, vae="tiny")
        assert pipe.adapter_cfg["in_channels"] == cin and pipe.adapter_cfg["channels"] == (64, 128, 256, 256)
        sd = pipe.adapter_state_dict
        assert {k: tuple(v.shape) for k, v in sd.items()} == dict(adapter_param_shapes(cin, (64, 128, 256, 256)))
        for k in [k for k in sd if ".block2." in k]:
            assert float(sd[k].float().abs().max()) > 0, k
        # every existing synthetic weight is unchanged by the adapter's own seed
        for a, b in ((pipe.unet_state_dict, plain.unet_state_dict), (pipe.vae_state_dict, plain.vae_state_dict)):
            assert all(torch.equal(a[k], b[k]) for k in a)
