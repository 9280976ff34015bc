"""Time one VAE decode (latents -> uint8 frame, the SDXL-width decoder) in fp16 and in bf16 storage.

    python tools/bench_vae_dtype.py [--iters 20] [--warmup 5]

Both decoders run the same program shape (wgmma implicit-GEMM convs, GroupNorm, mid-block attention, conv_out as an
N = 8 GEMM); only the element type differs.  Seeded fp16-safe weights, so the fp16 decode is valid too.  CUDA events
around ``iters`` back-to-back decodes after ``warmup`` untimed ones, per size; the median of 5 such runs is printed
with the spread.  Prints one table row per size and the GPU's name, power limit and clocks beside it.
"""
import argparse
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SIZES = [(512, 512), (1024, 1024), (1280, 720), (1920, 1080)]


def gpu_info():
    try:
        q = "name,power.limit,clocks.sm,clocks.max.sm,clocks.mem"
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:       # informational only
        return f"{torch.cuda.get_device_name()} (nvidia-smi unavailable: {e})"


def time_decode(vae, lat, iters, warmup, reps=5):
    for _ in range(warmup):
        vae.decode_to_u8(lat)
    torch.cuda.synchronize()
    per = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(iters):
            vae.decode_to_u8(lat)
        b.record()
        b.synchronize()
        per.append(a.elapsed_time(b) / iters)
    return statistics.median(per), min(per), max(per)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    from latentblending_b200 import ops
    from latentblending_b200.pipe import VAE_CHANNELS, random_state_dict, vae_param_shapes
    from latentblending_b200.vae import VAEDecoderB200
    dev = "cuda:0"
    sd = random_state_dict(vae_param_shapes(VAE_CHANNELS), 1, dev, damp=0.3)
    vaes = {name: VAEDecoderB200(sd, VAE_CHANNELS, 0.13025, dev, dtype=dt)
            for name, dt in (("fp16", torch.float16), ("bf16", torch.bfloat16))}
    print(f"GPU: {gpu_info()}")
    print(f"{'size':>10} | {'fp16 ms (min-max)':>22} | {'bf16 ms (min-max)':>22} | bf16/fp16")
    for w, h in SIZES:
        g = torch.Generator(device=dev).manual_seed(0)
        lat = (torch.randn(1, 4, h // 8, w // 8, generator=g, device=dev) * 0.8).half()
        res = {}
        for name, vae in vaes.items():
            res[name] = time_decode(vae, lat, args.iters, args.warmup)
            assert vae.overflow_count() == 0 and ops.error_flag() == 0
        f, b = res["fp16"], res["bf16"]
        print(f"{w}x{h:>5} | {f[0]:8.2f} ({f[1]:.2f}-{f[2]:.2f}) | {b[0]:8.2f} ({b[1]:.2f}-{b[2]:.2f}) | "
              f"{b[0] / f[0]:.3f}")
        for vae in vaes.values():
            vae._plans.clear()


if __name__ == "__main__":
    main()
