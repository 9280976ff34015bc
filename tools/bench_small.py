"""Micro-benchmarks / ncu targets of the memory-bound kernels at the SDXL 1024^2 shapes (CUDA-event timed):
GroupNorm(+SiLU) stats+apply, the LayerNorm, the scheduler step kernels, the embedding inputs."""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from latentblending_b200 import ops  # noqa: E402
from tools.bench_ops import time_it  # noqa: E402


def main():
    dev = "cuda"
    for B, HW, C in ((2, 128 * 128, 320), (2, 128 * 128, 640), (2, 64 * 64, 640), (2, 64 * 64, 1280), (2, 32 * 32, 1280),
                     (2, 32 * 32, 2560)):
        x = torch.randn(B * HW, C, device=dev).half()
        g, b = torch.ones(C, device=dev).half(), torch.zeros(C, device=dev).half()
        out = torch.empty_like(x)
        t = time_it(lambda: ops.groupnorm(x, B, HW, C, 32, g, b, 1e-5, 1, out=out))
        print(json.dumps(dict(op="groupnorm+silu", B=B, HW=HW, C=C, us=round(t * 1e6, 1),
                              gbs=round(4 * x.numel() / t / 1e9, 1), note="4 B/elem algorithmic")))
    for rows, C in ((2048, 1280), (8192, 640)):
        x = torch.randn(rows, C, device=dev).half()
        g, b = torch.ones(C, device=dev).half(), torch.zeros(C, device=dev).half()
        out = torch.empty_like(x)
        t = time_it(lambda: ops.layernorm(x, g, b, out=out))
        print(json.dumps(dict(op="layernorm", rows=rows, C=C, us=round(t * 1e6, 1),
                              gbs=round(4 * x.numel() / t / 1e9, 1))))
    n = 4 * 128 * 128
    x = torch.randn(1, 4, 128, 128, device=dev).half()
    eps = torch.randn(2, 4, 128, 128, device=dev).half()
    out = torch.empty_like(x)
    nxt = torch.empty(2, 4, 128, 128, device=dev, dtype=torch.float16)
    t = time_it(lambda: ops.cfg_euler_step(x, eps, 3.5, 7.9, -0.5, out=out, scaled_next=nxt, next_divisor=7.4))
    print(json.dumps(dict(op="cfg_euler_step (+next scale_model_input)", n=n, us=round(t * 1e6, 2),
                          gbs=round((3 + 1 + 2) * n * 2 / t / 1e9, 1), note="launch-bound at 128 KiB latents")))
    t = time_it(lambda: ops.scale_model_input(x, 2, 7.4, out=nxt))
    print(json.dumps(dict(op="scale_model_input", n=n, us=round(t * 1e6, 2))))
    text = torch.randn(2, 1280, device=dev).half()
    tids = torch.tensor([[1024., 1024, 0, 0, 1024, 1024]] * 2, device=dev).half()
    t = time_it(lambda: ops.embed_inputs(500.0, text, tids, 320, 256))
    print(json.dumps(dict(op="embed_inputs", us=round(t * 1e6, 2))))


if __name__ == "__main__":
    main()
