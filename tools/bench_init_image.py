"""Measure image keyframes (img2img) on one GPU.

    python tools/bench_init_image.py [--rounds 2] [--branches 15] [--iters 20] [--out DIR]

1. The native VAE encoder, ms per image, fp16 and bf16, at 512^2, 1024^2, 1280x720 and 1920x1080: the graph-replayed
   program (uint8 image in, scaled posterior mean out), CUDA events around ``iters`` replays, median of 5; beside it the
   device memory its plan allocates and the encoder's GEMM FLOPs (Program.work(), computed from shapes).  The 1024^2
   decoder is timed the same way for comparison.
2. Transition frames/s on synthetic SDXL-base weights at 1024^2 (SyntheticSDXLPipe's seeded recipe), 30 Euler steps,
   guidance 4, depth_strength 0.5, ``branches`` branches, seeds [420, 421], deterministic_noise, for: text / text,
   image / image at strength 0.3 and image / image at 0.6.  Every case is warmed up once, then the cases run
   alternately, ``rounds`` transitions each; the median is reported.
The GPU's name, power limit and SM clocks (one ``nvidia-smi --query-gpu`` call) are printed beside the numbers.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PROMPTS = ("photo of a very beautiful cat, 4k, high detail, dramatic light",
           "ultra high res psychedelic skyscraper city landscape 8K unreal engine")
SIZES = ((512, 512), (1024, 1024), (1280, 720), (1920, 1080))      # (W, H)


def gpu_info():
    try:
        q = "name,power.limit,clocks.sm,clocks.max.sm"
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:       # informational only
        return f"unknown ({e})"


def photo(H, W, seed=0):
    """A seeded stand-in photograph: smooth colour fields plus per-pixel noise."""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:H, 0:W].astype(np.float64)
    img = np.zeros((H, W, 3))
    for c in range(3):
        for _ in range(4):
            fy, fx, ph = rng.uniform(0.5, 6), rng.uniform(0.5, 6), rng.uniform(0, 2 * np.pi)
            img[:, :, c] += np.sin(2 * np.pi * (fy * y / H + fx * x / W) + ph)
    return np.clip(127.5 + 127.5 * np.tanh(0.75 * img) + rng.uniform(-8, 8, (H, W, 3)), 0, 255).astype(np.uint8)


def time_ms(fn, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(3):
        fn()
    res = []
    for _ in range(5):
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        e1.synchronize()
        res.append(e0.elapsed_time(e1) / iters)
    return statistics.median(res)


def engine(pipe, branches, strength):
    from latentblending_b200 import BlendingEngine
    be = BlendingEngine(pipe, run_benchmark=False)
    be.set_dimensions((1024, 1024))
    be.set_num_inference_steps(30)
    be.set_guidance_scale(4.0)
    be.set_prompt1(PROMPTS[0])
    be.set_prompt2(PROMPTS[1])
    be.set_branching(depth_strength=0.5, nmb_max_branches=branches)
    be.deterministic_noise = True
    be.output_device_frames = True
    if strength is not None:
        be.set_init_image1(photo(1024, 1024, 1), strength)
        be.set_init_image2(photo(1024, 1024, 2), strength)
    return be


def transition_fps(be):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    be.run_transition(fixed_seeds=[420, 421])
    torch.cuda.synchronize()
    return len(be.tree_latents) / (time.perf_counter() - t0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--branches", type=int, default=15)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None, help="also write the JSON result into this directory")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_init_image needs a CUDA device")
    from latentblending_b200 import SyntheticSDXLPipe
    from latentblending_b200.vae import VAEDecoderB200, VAEEncoderB200
    info = gpu_info()
    print(f"GPU: {info}")
    pipe = SyntheticSDXLPipe("stabilityai/stable-diffusion-xl-base-1.0", "cuda:0", seed=0)
    out = dict(gpu=info, encoder={})
    for name, dt in (("fp16", torch.float16), ("bf16", torch.bfloat16)):
        enc = VAEEncoderB200(pipe.vae_encoder_state_dict, pipe.vae_channels, pipe.vae_scaling_factor, "cuda:0",
                             dtype=dt)
        for W, H in SIZES:
            torch.cuda.synchronize()
            m0 = torch.cuda.memory_allocated()
            pl = enc.plan(H // 8, W // 8)
            torch.cuda.synchronize()
            mem = torch.cuda.memory_allocated() - m0
            pl.img.copy_(torch.from_numpy(photo(H, W)).cuda())
            ms = time_ms(pl.prog.run, args.iters)
            out["encoder"][f"{name}_{W}x{H}"] = dict(ms=ms, plan_bytes=mem,
                                                      gemm_tflop=pl.prog.work()["gemm_flops"] / 1e12)
            print(name, W, H, out["encoder"][f"{name}_{W}x{H}"], flush=True)
            enc._plans.clear()
            del pl
            torch.cuda.empty_cache()
        del enc
        torch.cuda.empty_cache()
    dec = VAEDecoderB200(pipe.vae_state_dict, pipe.vae_channels, pipe.vae_scaling_factor, "cuda:0")
    pl = dec.plan(128, 128)
    pl.z_in.normal_()
    out["decoder_fp16_1024x1024"] = dict(ms=time_ms(pl.prog.run, args.iters),
                                         gemm_tflop=pl.prog.work()["gemm_flops"] / 1e12)
    del dec, pl
    torch.cuda.empty_cache()
    cases = {"text_text": None, "image_image_0.3": 0.3, "image_image_0.6": 0.6}
    engines = {k: engine(pipe, args.branches, s) for k, s in cases.items()}
    fps = {k: [] for k in engines}
    for be in engines.values():
        transition_fps(be)                                  # warm-up: plans, graphs, encodes
    for _ in range(args.rounds):
        for k, be in engines.items():
            fps[k].append(transition_fps(be))
    out.update(frames_per_s={k: statistics.median(v) for k, v in fps.items()}, frames_per_s_runs=fps,
               branches=args.branches, gpu_after=gpu_info())
    text = json.dumps(out, indent=1)
    print(text)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_init_image.json"), "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
