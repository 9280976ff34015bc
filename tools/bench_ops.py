"""Micro-benchmarks of the UNet kernels at the SDXL 1024^2 shapes (CUDA-event timed).  Each op is recorded once into
a one-record Program and replayed, as the lowered programs replay it."""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from latentblending_b200.program import Program  # noqa: E402


ITERS = int(os.environ.get('BENCH_ITERS', 20))
WARM = int(os.environ.get('BENCH_WARM', 5))


def time_it(fn, iters=None, warm=None):
    iters = ITERS if iters is None else iters
    warm = WARM if warm is None else warm
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters * 1e-3


def replay(emit):
    """The run() of a one-record Program holding the op ``emit(P)`` records."""
    P = Program(0)
    emit(P)
    return P.finalize().run


def main():
    which = sys.argv[1:] or ["attn", "gemm"]
    if "attn" in which:
        for B, heads, S, Skv in ((2, 10, 4096, 4096), (2, 20, 1024, 1024), (2, 10, 4096, 77), (2, 20, 1024, 77),
                                 (4, 20, 1024, 1024)):
            C = heads * 64
            qkv = torch.randn(B * S, 3 * C, device="cuda").half()
            kv = torch.randn(B * 77, 2 * C, device="cuda").half()
            out = torch.empty(B * S, C, device="cuda", dtype=torch.float16)
            if Skv == S:
                f = replay(lambda P: P.attention(qkv, qkv, qkv, out, B, heads, S, S, 0, C, 2 * C))
            else:
                f = replay(lambda P: P.attention(qkv, kv, kv, out, B, heads, S, 77, 0, 0, C))
            t = time_it(f)
            fl = 4 * B * heads * S * Skv * 64
            print(json.dumps(dict(op="attention", B=B, heads=heads, S=S, Skv=Skv, us=t * 1e6, tflops=fl / t / 1e12)))
    if "gemm" in which:
        shapes = [("to_out/q/proj", 2048, 1280, 1280, 1), ("ff_out", 2048, 1280, 5120, 1), ("qkv", 2048, 3840, 1280, 1),
                  ("ff_in_geglu", 2048, 10240, 1280, 1), ("qkv64", 8192, 1920, 640, 1), ("ff_out64", 8192, 640, 2560, 1),
                  ("conv320", 32768, 320, 320, 9), ("conv640", 8192, 640, 640, 9), ("conv1280", 2048, 1280, 1280, 9),
                  ("conv_up", 32768, 640, 640, 9), ("conv2560", 2048, 1280, 2560, 9), ("M4096", 4096, 1280, 1280, 1)]
        for name, M, N, K, taps in shapes:
            if taps == 9:
                hw = {32768: 128, 8192: 64, 2048: 32}[M]
                a = torch.randn(M, K, device="cuda").half()
                w = (torch.randn(N, 9 * K, device="cuda") * 0.02).half()
                out = torch.empty(M, N, device="cuda", dtype=torch.float16)
                f = replay(lambda P: P.gemm(a, w, N, 2, hw, hw, out, taps=9, static_w=False))
                fl = 2 * M * N * 9 * K
            else:
                a = torch.randn(M, K, device="cuda").half()
                w = (torch.randn(N, K, device="cuda") * 0.02).half()
                mode = 1 if "geglu" in name else 0
                out = torch.empty(M, N // 2 if mode else N, device="cuda", dtype=torch.float16)
                f = replay(lambda P: P.gemm(a, w, N, 1, 1, M, out, mode=mode))
                fl = 2 * M * N * K
            t = time_it(f)
            print(json.dumps(dict(op="gemm", name=name, M=M, N=N, K=K * taps, us=round(t * 1e6, 1),
                                  tflops=round(fl / t / 1e12, 1))))


def vae_shapes():
    """The big 3x3 convolutions of the SDXL VAE decoder at 1024^2 output (batch 1)."""
    for name, hw, cin, cout in (("vae_up3_128", 1024, 128, 128), ("vae_upconv_256", 1024, 256, 256),
                                ("vae_up2_256", 512, 256, 256), ("vae_upconv_512", 512, 512, 512),
                                ("vae_up1_512", 256, 512, 512), ("vae_up0_512", 128, 512, 512)):
        M = hw * hw
        a = torch.randn(M, cin, device="cuda").half()
        w = (torch.randn(cout, 9 * cin, device="cuda") * 0.02).half()
        out = torch.empty(M, cout, device="cuda", dtype=torch.float16)
        t = time_it(replay(lambda P: P.gemm(a, w, cout, 1, hw, hw, out, taps=9)), iters=5, warm=2)
        fl = 2 * M * cout * 9 * cin
        print(json.dumps(dict(op="conv3x3", name=name, M=M, N=cout, K=9 * cin, us=round(t * 1e6, 1),
                              tflops=round(fl / t / 1e12, 1))))
        del a, w, out


if __name__ == "__main__":
    if "vae" in sys.argv[1:]:
        vae_shapes()
    else:
        main()
