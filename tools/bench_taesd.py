"""Measure the tiny VAE decoder (AutoencoderTiny / TAESDXL) against the KL decoder on one GPU.

    python tools/bench_taesd.py [--iters 20] [--warmup 5] [--branches 60] [--transitions 3]

1. ms per decode (latents -> uint8 frame on the device) for the KL decoder in fp16 and in bf16 and for the tiny
   decoder, at 512^2, 1024^2, 1280x720 and 1920x1080: CUDA events around ``iters`` back-to-back decodes after
   ``warmup`` untimed ones, median (and min-max) of 5 such runs.  Seeded weights (the synthetic pipe's recipes).
2. Each upsampling level of the tiny decoder at 1024^2 (64 channels, low-resolution map 128^2, 256^2, 512^2): the
   depth-to-space GEMM (LB_GEMM_D2S2, N = 256 over the low-resolution map) against nearest-2x upsample +
   the N = 64 3x3 conv at the upsampled size, both recorded ``iters`` times into one program replayed as a CUDA
   graph (so host launch cost is not timed); median of 5.
3. SDXL-Turbo 512^2 transitions through the engine API (a config-5-like tree: 4 steps, ``branches`` branches, fixed
   seeds, deterministic_noise), frames/s with the KL fp16 decoder and with the tiny one, on the same seeded UNet.
The GPU's name, power limit and SM clocks (one ``nvidia-smi --query-gpu`` call) are printed beside the numbers.
"""
import argparse
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SIZES = [(512, 512), (1024, 1024), (1280, 720), (1920, 1080)]
PROMPTS = ("photo of a very beautiful cat, 4k, high detail, dramatic light",
           "ultra high res psychedelic skyscraper city landscape 8K unreal engine")


def gpu_info():
    try:
        q = "name,power.limit,clocks.sm,clocks.max.sm"
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:       # informational only
        return f"{torch.cuda.get_device_name()} (nvidia-smi unavailable: {e})"


def time_reps(fn, iters, reps=5):
    per = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(iters):
            fn()
        b.record()
        b.synchronize()
        per.append(a.elapsed_time(b) / iters)
    return statistics.median(per), min(per), max(per)


def fmt(r):
    return f"{r[0]:7.3f} ({r[1]:.3f}-{r[2]:.3f})"


def decode_table(args, dev):
    from latentblending_b200 import ops
    from latentblending_b200.pipe import VAE_CHANNELS, random_state_dict, random_tiny_vae_state_dict, vae_param_shapes
    from latentblending_b200.taesd import DEFAULT_CONFIG, TinyVAEDecoderB200
    from latentblending_b200.vae import VAEDecoderB200
    sd = random_state_dict(vae_param_shapes(VAE_CHANNELS), 1, dev, damp=0.3)
    vaes = {"KL fp16": VAEDecoderB200(sd, VAE_CHANNELS, 0.13025, dev),
            "KL bf16": VAEDecoderB200(sd, VAE_CHANNELS, 0.13025, dev, dtype=torch.bfloat16),
            "tiny fp16": TinyVAEDecoderB200(random_tiny_vae_state_dict(1, dev), DEFAULT_CONFIG, 1.0, dev)}
    print("\n1. ms per decode, median (min-max) of 5 x", args.iters)
    print(f"{'size':>10} | " + " | ".join(f"{n:>22}" for n in vaes) + " | KL fp16 / tiny")
    for w, h in SIZES:
        g = torch.Generator(device=dev).manual_seed(0)
        lat = (torch.randn(1, 4, h // 8, w // 8, generator=g, device=dev) * 0.8).half()
        res = {}
        for name, vae in vaes.items():
            for _ in range(args.warmup):
                vae.decode_to_u8(lat)
            torch.cuda.synchronize()
            res[name] = time_reps(lambda: vae.decode_to_u8(lat), args.iters)
            assert vae.overflow_count() == 0 and ops.error_flag() == 0
            vae._plans.clear()
        print(f"{w}x{h:>5} | " + " | ".join(f"{fmt(r):>22}" for r in res.values()) +
              f" | {res['KL fp16'][0] / res['tiny fp16'][0]:.1f}x")


def level_table(args, dev):
    from latentblending_b200 import ops
    from latentblending_b200.taesd import pack_d2s_weights
    from latentblending_b200.program import Program
    C = 64
    g = torch.Generator(device=dev).manual_seed(0)
    w = (torch.randn(C, C, 3, 3, generator=g, device=dev) * (9 * C) ** -0.5).half()
    w3 = w.permute(0, 2, 3, 1).reshape(C, -1).contiguous()
    wd = pack_d2s_weights(w.float()).permute(0, 2, 3, 1).reshape(4 * C, -1).half().contiguous()
    print("\n2. tiny decoder upsampling levels at 1024^2 (C = 64): ms per upsample + conv, median (min-max) of 5 x",
          args.iters, "graph-replayed launches")
    print(f"{'low-res':>8} -> {'out':>8} | {'D2S2 GEMM':>22} | {'upsample2x + conv':>22} | speed-up | "
          f"D2S2 TFLOP/s")
    for hh in (128, 256, 512):
        x = (torch.randn(hh * hh, C, generator=g, device=dev)).half()
        up = torch.empty(4 * hh * hh, C, dtype=torch.float16, device=dev)
        o1 = torch.empty(4 * hh * hh, C, dtype=torch.float16, device=dev)
        o2 = torch.empty_like(o1)
        pd, pu = Program(0), Program(0)
        for _ in range(args.iters):
            pd.gemm(x, wd, 4 * C, 1, hh, hh, o1, taps=9, depth_to_space=True)
            pu.upsample_nearest(x, 1, hh, hh, C, up, 2 * hh, 2 * hh)
            pu.gemm(up, w3, C, 1, 2 * hh, 2 * hh, o2, taps=9)
        pd.finalize()
        pu.finalize()
        for p in (pd, pu):
            for _ in range(3):           # the second run captures the CUDA graph
                p.run()
        torch.cuda.synchronize()
        rd = time_reps(pd.run, 1)
        ru = time_reps(pu.run, 1)
        rd = tuple(v / args.iters for v in rd)
        ru = tuple(v / args.iters for v in ru)
        rel = ((o1.float() - o2.float()).norm() / o2.float().norm()).item()
        assert rel < 2e-3 and ops.error_flag() == 0, rel
        flops = 2 * (4 * hh * hh) * C * 9 * C
        print(f"{hh:>4}^2 -> {2 * hh:>4}^2 | {fmt(rd):>22} | {fmt(ru):>22} | {ru[0] / rd[0]:7.2f}x | "
              f"{flops / rd[0] / 1e9:.0f}")


def transitions(args, dev):
    from latentblending_b200 import BlendingEngine, SyntheticSDXLPipe
    kl = SyntheticSDXLPipe("stabilityai/sdxl-turbo", dev, seed=0)
    tiny = SyntheticSDXLPipe("stabilityai/sdxl-turbo", dev, seed=0, unet_state_dict=kl.unet_state_dict, vae="tiny")
    print(f"\n3. SDXL-Turbo 512^2 transition, 4 steps, nmb_max_branches={args.branches}, seeds [420, 421], "
          f"deterministic_noise; {args.transitions} timed after 1 warm-up")
    for name, pipe in (("KL fp16", kl), ("tiny fp16", tiny)):
        be = BlendingEngine(pipe, run_benchmark=False)
        be.deterministic_noise = True
        be.set_negative_prompt("blurry, ugly, pale")
        be.set_prompt1(PROMPTS[0])
        be.set_prompt2(PROMPTS[1])
        be.set_branching(nmb_max_branches=args.branches)
        be.run_transition(fixed_seeds=[420, 421])
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        frames = 0
        for _ in range(args.transitions):
            frames += len(be.run_transition(fixed_seeds=[420, 421]))
        torch.cuda.synchronize()
        sec = time.perf_counter() - t0
        be.dh.check_decode_overflow()
        print(f"{name:>10}: {frames / sec:7.2f} frames/s ({frames} frames in {sec:.2f} s, "
              f"{frames // args.transitions} per transition)")
        del be
        torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--branches", type=int, default=60)
    ap.add_argument("--transitions", type=int, default=3)
    ap.add_argument("--skip", default="", help="comma list of sections to skip: decode, levels, transitions")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "tools/bench_taesd.py measures on a CUDA device"
    dev = "cuda:0"
    skip = set(filter(None, args.skip.split(",")))
    print(f"GPU (name, power limit, SM clock, max SM clock): {gpu_info()}")
    if "decode" not in skip:
        decode_table(args, dev)
    if "levels" not in skip:
        level_table(args, dev)
    if "transitions" not in skip:
        transitions(args, dev)


if __name__ == "__main__":
    main()
