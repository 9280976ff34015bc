"""CPU tests of the boundary pieces added in round 2 (no CUDA compute): the diffusers-pipeline adapter
(reference constructor contract, blending_engine.py:20-44), the scheduler tables built from a diffusers scheduler
config, the storyboard JSON format + multi-transition driver (example_multi_trans_json.py:26-74), the frame-fill
plan of the movie writer, and the LPIPS guard."""
import json
import os

import numpy as np
import pytest
import torch


class _Cfg(dict):
    __getattr__ = dict.get


class EulerDiscreteScheduler:                     # named like the diffusers class the adapter keys on
    def __init__(self, **kw):
        self.config = _Cfg(num_train_timesteps=1000, beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear",
                           prediction_type="epsilon", timestep_spacing="leading", steps_offset=1,
                           use_karras_sigmas=False, interpolation_type="linear", **kw)


class EulerAncestralDiscreteScheduler(EulerDiscreteScheduler):
    def __init__(self):
        super().__init__()
        self.config.update(timestep_spacing="trailing", steps_offset=0)


class _Module:
    def __init__(self, config, sd):
        self.config, self._sd = config, sd

    def state_dict(self):
        return self._sd


class MockDiffusersPipe:
    """Duck-typed StableDiffusionXLPipeline: what AutoPipelineForText2Image returns, reduced to the attributes the
    reference's holder and this backend's adapter read."""

    def __init__(self, turbo=False):
        from oracle.sdxl_unet import SDXLUNet, tiny_config
        from oracle.vae import VAEConfig, VAEDecoder
        ocfg = tiny_config()
        unet = SDXLUNet(ocfg)
        self.unet = _Module(_Cfg(sample_size=16, in_channels=4, out_channels=4, block_out_channels=(64, 128, 256),
                                 layers_per_block=2, transformer_layers_per_block=[1, 1, 2],
                                 down_block_types=["DownBlock2D", "CrossAttnDownBlock2D", "CrossAttnDownBlock2D"],
                                 attention_head_dim=[1, 2, 4], cross_attention_dim=128, addition_embed_type="text_time",
                                 addition_time_embed_dim=32, projection_class_embeddings_input_dim=64 + 6 * 32,
                                 use_linear_projection=True, norm_num_groups=32, time_cond_proj_dim=None),
                            unet.state_dict())
        vae = VAEDecoder(VAEConfig(block_out_channels=(64, 64, 128, 128)))
        vsd = {("post_quant_conv." + k[len("post_quant_conv."):] if k.startswith("post_quant_conv.") else "decoder." + k): v
               for k, v in vae.state_dict().items()}
        vsd["encoder.conv_in.weight"] = torch.zeros(1)
        vsd["quant_conv.weight"] = torch.zeros(1)
        self.vae = _Module(_Cfg(block_out_channels=(64, 64, 128, 128), scaling_factor=0.13025, force_upcast=True), vsd)
        self.scheduler = EulerAncestralDiscreteScheduler() if turbo else EulerDiscreteScheduler()
        self._execution_device = torch.device("cpu")
        self._name_or_path = "stabilityai/sdxl-turbo" if turbo else "stabilityai/stable-diffusion-xl-base-1.0"
        self.vae_scale_factor = 8
        self.default_sample_size = 16
        self.calls = []

    def encode_prompt(self, **kw):
        self.calls.append(kw)
        pe, pp = torch.ones(1, 77, 128), torch.ones(1, 64)
        if kw["do_classifier_free_guidance"]:
            return pe, pe * 0, pp, pp * 0
        return pe, None, pp, None


def test_diffusers_pipeline_is_adapted():
    from latentblending_b200.pipe import DiffusersSDXLPipe, SyntheticSDXLPipe, adapt_pipe, vae_param_shapes
    from latentblending_b200.pipe import unet_param_shapes
    mock = MockDiffusersPipe()
    pipe = adapt_pipe(mock)
    assert isinstance(pipe, DiffusersSDXLPipe) and not pipe.is_synthetic
    c = pipe.unet_cfg
    assert c.block_out_channels == (64, 128, 256) and c.transformer_layers == (0, 1, 2) and c.head_dim == 64
    assert c.cross_attention_dim == 128 and c.pooled_dim == 64 and c.addition_time_embed_dim == 32 and c.sample_size == 16
    # every parameter the UNet / VAE packers ask for is present under the diffusers name, with the right shape
    for name, shape in unet_param_shapes(c).items():
        assert tuple(pipe.unet_state_dict[name].shape) == tuple(shape), name
    for name, shape in vae_param_shapes((64, 64, 128, 128)).items():
        assert tuple(pipe.vae_state_dict[name].shape) == tuple(shape), name
    assert not any(k.startswith(("encoder.", "quant_conv.")) for k in pipe.vae_state_dict)
    assert pipe.vae_channels == (64, 64, 128, 128) and abs(pipe.vae_scaling_factor - 0.13025) < 1e-12
    assert pipe.scheduler.kind == "euler" and pipe.scheduler.timestep_spacing == "leading" and pipe.scheduler.steps_offset == 1
    # encode_prompt goes through the pipeline's own text encoders with the reference's arguments (diffusers_holder.py:81-95)
    pe, ne, pp, npool = pipe.encode_prompt("a lake", negative_prompt=["blurry"], do_classifier_free_guidance=True)
    kw = mock.calls[-1]
    assert kw["prompt"] == kw["prompt_2"] == "a lake" and kw["negative_prompt"] == kw["negative_prompt_2"] == ["blurry"]
    assert kw["num_images_per_prompt"] == 1 and pe.dtype == torch.float16 and ne is not None
    assert adapt_pipe(pipe) is pipe                       # our own pipes pass through
    t = adapt_pipe(MockDiffusersPipe(turbo=True))
    assert t.scheduler.kind == "euler_ancestral" and t.scheduler.timestep_spacing == "trailing"
    with pytest.raises(TypeError):
        adapt_pipe(object())
    assert SyntheticSDXLPipe.is_synthetic


def test_scheduler_tables_from_config_match_the_oracle_schedulers():
    from latentblending_b200.schedulers import tables_from_diffusers_scheduler
    from oracle.schedulers import EulerAncestralDiscrete, EulerDiscrete
    for sched, oracle, n in ((EulerDiscreteScheduler(), EulerDiscrete(), 30), (EulerAncestralDiscreteScheduler(), EulerAncestralDiscrete(), 4)):
        tb = tables_from_diffusers_scheduler(sched)
        tb.set_timesteps(n)
        oracle.set_timesteps(n)
        np.testing.assert_array_equal(tb.sigmas.numpy(), oracle.sigmas.numpy())
        np.testing.assert_array_equal(tb.timesteps.numpy(), oracle.timesteps.numpy())
    bad = EulerDiscreteScheduler()
    bad.config["use_karras_sigmas"] = True
    with pytest.raises(ValueError):
        tables_from_diffusers_scheduler(bad)

    class DDIMScheduler(EulerDiscreteScheduler):
        pass
    with pytest.raises(ValueError):
        tables_from_diffusers_scheduler(DDIMScheduler())


class _RecordingEngine:
    def __init__(self):
        self.log = []

        class DH:
            width_img, height_img, num_inference_steps = 768, 512, 6
        self.dh = DH()

    def __getattr__(self, name):
        def f(*a, **k):
            self.log.append((name, a, tuple(sorted(k.items()))))
            return ["frame"]
        return f


def test_storyboard_roundtrip_and_call_order(tmp_path):
    from latentblending_b200.storyboard import load_storyboard, run_storyboard, write_storyboard
    be = _RecordingEngine()
    entries = [dict(prompt=f"p{i}", negative_prompt=f"n{i}", seed=100 + i) for i in range(4)]
    fp = os.path.join(tmp_path, "movie.json")
    data = write_storyboard(fp, be, entries)
    # the reference's format (gradio_ui.py:168-191): settings first, then iteration/seed/prompt/negative_prompt/preview_image
    assert data[0] == {"settings": "sdxl", "width": 768, "height": 512, "num_inference_steps": 6}
    assert set(data[1]) == {"iteration", "seed", "prompt", "negative_prompt", "preview_image"}
    settings, prompts, negs, seeds = load_storyboard(fp)
    assert prompts == ["p0", "p1", "p2", "p3"] and negs == ["n0", "n1", "n2", "n3"] and seeds == [100, 101, 102, 103]
    be.log.clear()
    out = run_storyboard(be, fp, dp_out=str(tmp_path), duration_single_trans=2, fps=5)
    names = [c[0] for c in be.log]
    # example_multi_trans_json.py:26-74, line by line
    assert names == ["set_dimensions", "set_num_inference_steps",
                     "set_prompt1", "set_negative_prompt", "set_prompt2", "run_transition", "write_movie_transition",
                     "swap_forward", "set_negative_prompt", "set_prompt2", "run_transition", "write_movie_transition",
                     "swap_forward", "set_negative_prompt", "set_prompt2", "run_transition", "write_movie_transition"]
    assert be.log[0][1] == ((768, 512),) and be.log[1][1] == (6,)
    runs = [c for c in be.log if c[0] == "run_transition"]
    assert [dict(r[2])["recycle_img1"] for r in runs] == [False, True, True]
    assert [dict(r[2])["fixed_seeds"] for r in runs] == [[100, 101], [101, 102], [102, 103]]
    negs_set = [c[1][0] for c in be.log if c[0] == "set_negative_prompt"]
    assert negs_set == ["n0", "n2", "n3"]                 # the reference indexes [i] first, [i+1] afterwards (:52,:56)
    assert [os.path.basename(p) for p in out] == ["tmp_part_000.mp4", "tmp_part_001.mp4", "tmp_part_002.mp4"]
    with open(fp, "w") as f:
        json.dump([{"width": 1}], f)
    with pytest.raises(ValueError):
        load_storyboard(fp)


def test_frame_fill_plan_matches_reference_algorithm():
    """plan_frame_fill (device path) and add_frames_linear_interp (host path) implement utils.py:105-178: exact target
    count, key frames kept, per-gap linspace weights, float32 blend with truncating cast."""
    from latentblending_b200.utils import add_frames_linear_interp, plan_frame_fill
    rng = np.random.RandomState(0)
    keys = [rng.randint(0, 256, (6, 5, 3)).astype(np.uint8) for _ in range(7)]
    for target in (7, 8, 30, 101):
        left, w0, w1 = plan_frame_fill(len(keys), target, seed=3)
        frames = add_frames_linear_interp(keys, nmb_frames_target=target, seed=3)
        assert len(left) == len(frames) == max(target, 7)
        for t in range(len(left)):
            a, b = keys[left[t]].astype(np.float32), keys[min(left[t] + 1, 6)].astype(np.float32)
            assert np.array_equal(frames[t], (w0[t] * a + w1[t] * b).astype(np.uint8))
        # key frames appear unchanged and in order
        idx = [t for t in range(len(left)) if w1[t] == 0.0 or w0[t] == 0.0]
        assert len(idx) == 7
    with pytest.raises(ValueError):
        add_frames_linear_interp(keys, fps_target=30, nmb_frames_target=10)


def test_engine_refuses_random_lpips_for_real_weights():
    """ADVICE r1: a non-synthetic pipe without lpips_state_dict must not silently get a random-weight metric."""
    from fakes import FakeHolder
    from latentblending_b200 import BlendingEngine

    class RealPipe:
        is_synthetic = False
        lpips_state_dict = None
    dh = FakeHolder()
    dh.pipe = RealPipe()
    with pytest.raises(ValueError, match="lpips_state_dict"):
        BlendingEngine(RealPipe(), holder=dh, run_benchmark=False)


def test_geglu_permutation_on_cpu():
    """Host-side GEGLU row interleave (unet._geglu_perm), checked in fp32 on the CPU against torch's LayerNorm +
    Linear + exact-erf GEGLU: the kernel reads value / gate rows per N tile."""
    import torch.nn.functional as F
    from latentblending_b200.unet import _geglu_perm
    g = torch.Generator().manual_seed(0)
    M, C, N = 37, 128, 512
    x = torch.randn(M, C, generator=g) * 2 + 0.5
    w = (torch.randn(N, C, generator=g) * C ** -0.5).half()
    b = (torch.randn(N, generator=g) * 0.1).half()
    gamma = (1 + 0.1 * torch.randn(C, generator=g)).half()
    beta = (0.05 * torch.randn(C, generator=g)).half()
    want = F.layer_norm(x, (C,), gamma.float(), beta.float(), 1e-5) @ w.float().t() + b.float()
    # GEGLU interleave: tile t of `half` value rows is followed by its `half` gate rows
    for half in (64, 128):
        perm = _geglu_perm(N // 2, "cpu", half=half)
        assert sorted(perm.tolist()) == list(range(N))
        y = want[:, perm]                                    # what the kernel's accumulator columns hold
        tiles = y.view(M, -1, 2 * half)
        out = (tiles[:, :, :half] * F.gelu(tiles[:, :, half:])).reshape(M, N // 2)
        v, gate = want.chunk(2, dim=-1)
        assert torch.allclose(out, v * F.gelu(gate), atol=1e-6)


def test_bench_helpers():
    import importlib.util
    spec = importlib.util.spec_from_file_location("bench_mod", os.path.join(os.path.dirname(os.path.dirname(__file__)), "bench.py"))
    bench = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bench)
    assert abs(bench.unet_tflop(128) - 6.761) < 1e-3                  # SURVEY 8d, exact at the bench shape
    assert abs(bench.unet_tflop(64) / 1.589 - 1) < 0.03               # pixel / pixel^2 scaling model vs the analytic 512^2 count
    assert 1 <= bench.host_cpu_budget() <= (os.cpu_count() or 1)
    for c in (2, 3, 5):
        cfg = bench.CONFIGS[c]
        assert cfg["frames"] == sum(cfg["stems"]) + 2 and cfg["metric"] and cfg["workload"]
    # forwards of the base configs: 2 outer trajectories x N + sum stems x (N - idx_injection)
    idx = [15, 18, 21, 24, 27]
    for c in (2, 3):
        cfg = bench.CONFIGS[c]
        assert cfg["unet_forwards"] == 2 * 30 + sum(s * (30 - i) for s, i in zip(cfg["stems"], idx))
    assert bench.CONFIGS[5]["unet_forwards"] == 2 * 4 + 60 * 2

    class FakeEngine:
        tree_fracts = [0.0, 0.5, 1.0]
        tree_idx_injection = [0, 2, 0]
        tree_latents = [[torch.zeros(4)], [torch.ones(4)], [torch.zeros(4)]]
    a = bench.tree_fingerprint(FakeEngine())
    FakeEngine.tree_latents[1][0][0] = 2.0
    assert a != bench.tree_fingerprint(FakeEngine()) and len(a) == 40
