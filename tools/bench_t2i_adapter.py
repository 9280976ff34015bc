"""Measure what an SDXL T2I-Adapter costs on one GPU, beside the "full" ControlNet.

    python tools/bench_t2i_adapter.py [--rounds 2] [--branches 15] [--iters 20]

1. Transition frames/s on synthetic SDXL-base weights at 1024^2 (SyntheticSDXLPipe's seeded recipe), 30 Euler steps,
   guidance 4 (CFG), depth_strength 0.5, ``branches`` branches, seeds [420, 421], deterministic_noise, for: no
   conditioning, an RGB T2I-Adapter over the whole schedule (scale 1, factor 1), and the "full" ControlNet (transformer
   depths 0/2/10) over the whole schedule.  Every variant is warmed up once, then the variants run alternately,
   ``rounds`` transitions each; the median is reported.
2. ms per CFG-batch-2 step program at 128x128 latents, plain and with the adapter's four adds: CUDA events around
   ``iters`` replays, median of 5, the two programs alternated.
3. The once-per-image feature program (uint8 image -> four scaled states) at 1024^2 and 1280x720: CUDA events, median
   of 5.
The GPU's name, power limit and SM clocks (one ``nvidia-smi --query-gpu`` call) are printed beside the numbers.
"""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(ROOT))
sys.path.insert(0, ROOT)

from bench_controlnet import control_image, engine, gpu_info, time_program, transition_fps  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--branches", type=int, default=15)
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_t2i_adapter needs a CUDA device")
    from latentblending_b200 import SyntheticSDXLPipe
    info = gpu_info()
    print(f"GPU: {info}")
    name = "stabilityai/stable-diffusion-xl-base-1.0"
    base = SyntheticSDXLPipe(name, "cuda:0", seed=0)
    shared = dict(unet_state_dict=base.unet_state_dict, vae_state_dict=base.vae_state_dict)
    pipes = {"none": base, "adapter": SyntheticSDXLPipe(name, "cuda:0", seed=0, adapter="rgb", **shared),
             "controlnet_full": SyntheticSDXLPipe(name, "cuda:0", seed=0, controlnet="full", **shared)}
    engines = {k: engine(p, args.branches, k == "controlnet_full") for k, p in pipes.items()}
    engines["adapter"].set_adapter_image(control_image(1024, 1024))
    fps = {k: [] for k in engines}
    for be in engines.values():
        transition_fps(be)                                  # warm-up: plans, graphs, features
    for _ in range(args.rounds):
        for k, be in engines.items():
            fps[k].append(transition_fps(be))
    out = dict(gpu=info, frames_per_s={k: statistics.median(v) for k, v in fps.items()},
               frames_per_s_runs=fps, branches=args.branches)
    dh = engines["adapter"].dh
    plan = dh.unet.plan(2, 128, 128)
    plan.prog_ctx.run()
    plain, with_ad = [], []
    for _ in range(3):
        plain.append(time_program(plan.prog_step, 499.0, args.iters))
        with_ad.append(time_program(plan.prog_step_ad, 499.0, args.iters))
    out["step_ms_b2_128"] = dict(plain=statistics.median(plain), with_adapter=statistics.median(with_ad),
                                 plain_runs=plain, with_adapter_runs=with_ad,
                                 launches=(plan.prog_step.num_launches, plan.prog_step_ad.num_launches))
    ad = dh.adapter
    for (H, W) in ((1024, 1024), (720, 1280)):
        img = torch.from_numpy(control_image(H, W, 1)).cuda()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ad.compute(img, H // 8, W // 8, 1.0)
        res = []
        for _ in range(5):
            e0.record()
            ad.compute(img, H // 8, W // 8, 1.0)
            e1.record()
            e1.synchronize()
            res.append(e0.elapsed_time(e1))
        out[f"features_ms_{W}x{H}"] = statistics.median(res)
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
