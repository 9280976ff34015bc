"""Measure what an SDXL ControlNet costs on one GPU.

    python tools/bench_controlnet.py [--rounds 2] [--branches 15] [--iters 20]

1. Transition frames/s on synthetic SDXL-base weights at 1024^2 (SyntheticSDXLPipe's seeded recipe), 30 Euler steps,
   guidance 4 (CFG), depth_strength 0.5, ``branches`` branches, seeds [420, 421], deterministic_noise, for: no
   ControlNet, the "full" ControlNet (transformer depths 0/2/10) and the "small" one (0/0/1), each with a control image
   over the whole schedule.  Every variant is warmed up once, then the variants run alternately, ``rounds``
   transitions each; the median is reported.
2. ms per CFG-batch-2 step program at 128x128 latents, plain and UNet + ControlNet: CUDA events around ``iters``
   replays, median of 5.
3. The ControlNet's share of the step's GEMM FLOPs (Program.work()).
4. The one-off conditioning embedding (uint8 image -> [h*w, 320]) at 1024^2 and 1920x1080: CUDA events, median of 5.
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


def gpu_info():
    try:
        q = "name,power.limit,clocks.sm,clocks.max.sm"
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:       # informational only
        return f"unknown ({e})"


def control_image(H, W, seed=0):
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:H, 0:W]
    img = (xx * 255 // max(W - 1, 1) + ((yy // 64 + xx // 64) % 2) * 120)[..., None] + rng.integers(0, 40, (H, W, 3))
    return (img % 256).astype(np.uint8)


def engine(pipe, branches, with_image):
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
    if with_image:
        be.set_control_image(control_image(1024, 1024))
    return be


def transition_fps(be):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    be.run_transition(fixed_seeds=[420, 421])
    torch.cuda.synchronize()
    return len(be.tree_latents) / (time.perf_counter() - t0)


def time_program(prog, t, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(3):
        prog.run(t)
    res = []
    for _ in range(5):
        e0.record()
        for _ in range(iters):
            prog.run(t)
        e1.record()
        e1.synchronize()
        res.append(e0.elapsed_time(e1) / iters)
    return statistics.median(res)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--branches", type=int, default=15)
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_controlnet needs a CUDA device")
    from latentblending_b200 import SyntheticSDXLPipe
    info = gpu_info()
    print(f"GPU: {info}")
    base = SyntheticSDXLPipe("stabilityai/stable-diffusion-xl-base-1.0", "cuda:0", seed=0)
    pipes = {"none": base}
    for v in ("full", "small"):
        pipes[v] = SyntheticSDXLPipe("stabilityai/stable-diffusion-xl-base-1.0", "cuda:0", seed=0, controlnet=v,
                                     unet_state_dict=base.unet_state_dict, vae_state_dict=base.vae_state_dict)
    engines = {k: engine(p, args.branches, k != "none") for k, p in pipes.items()}
    fps = {k: [] for k in engines}
    for k, be in engines.items():
        transition_fps(be)                                  # warm-up: plans, graphs, embedding
    for _ in range(args.rounds):
        for k, be in engines.items():
            fps[k].append(transition_fps(be))
    out = dict(gpu=info, frames_per_s={k: statistics.median(v) for k, v in fps.items()},
               frames_per_s_runs=fps, branches=args.branches)
    for v in ("full", "small"):
        dh = engines[v].dh
        plan = dh.unet.plan(2, 128, 128)
        plan.prog_ctx.run()
        plain_ms = time_program(plan.prog_step, 499.0, args.iters)
        cn_ms = time_program(plan.prog_step_cn, 499.0, args.iters)
        wp, wc = plan.prog_step.work(), plan.prog_step_cn.work()
        out[f"step_ms_b2_128_{v}"] = dict(plain=plain_ms, with_controlnet=cn_ms,
                                          launches=(plan.prog_step.num_launches, plan.prog_step_cn.num_launches),
                                          controlnet_gemm_flop_share=(wc["gemm_flops"] - wp["gemm_flops"]) /
                                          wc["gemm_flops"])
    cn = engines["full"].dh.controlnet
    for (H, W) in ((1024, 1024), (1080, 1920)):
        img = torch.from_numpy(control_image(H, W, 1)).cuda()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        cn.embed(img, H // 8, W // 8)
        res = []
        for _ in range(5):
            e0.record()
            cn.embed(img, H // 8, W // 8)
            e1.record()
            e1.synchronize()
            res.append(e0.elapsed_time(e1))
        out[f"embed_ms_{W}x{H}"] = statistics.median(res)
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
