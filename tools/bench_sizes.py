"""Time the full-size SDXL-base path at the SDXL aspect-ratio buckets (random weights with the real shapes, as bench.py
uses), since bench.py measures 1024^2 only.

    python tools/bench_sizes.py [--sizes 1024x1024,1216x832,...] [--iters 10] [--steps 10] [--branches 6]
                                [--out FILE.jsonl]

Sizes are width x height in pixels.  Per size, one JSON line with
  * unet_ms: one CFG-batch-2 UNet forward (CUDA-graph replay of the lowered program, CUDA events, after warm-up);
  * vae_ms: one VAE decode to a uint8 frame;
  * transition_fps: frames per second of a short transition (--steps denoising steps, --branches branches,
    depth_strength 0.5), timed after one untimed transition at the same size;
and each divided by (or, for frames/s, multiplied by) the image's megapixels.  The first line records the card, its
power limit and its SM clocks (nvidia-smi, read-only).
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from gemm_shapes import card_info  # noqa: E402

SIZES = "1024x1024,1216x832,832x1216,1344x768,768x1344,1536x640"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default=SIZES)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--branches", type=int, default=6)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from latentblending_b200 import BlendingEngine, SyntheticSDXLPipe, ops
    assert torch.cuda.is_available(), "bench_sizes.py needs a CUDA device"
    sink = open(args.out, "a") if args.out else None

    def emit(d):
        line = json.dumps(d)
        print(line, flush=True)
        if sink:
            sink.write(line + "\n")

    def time_ms(fn, iters):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(iters):
            fn()
        e.record()
        torch.cuda.synchronize()
        return s.elapsed_time(e) / iters

    emit(dict(card=card_info()))
    pipe = SyntheticSDXLPipe("stabilityai/stable-diffusion-xl-base-1.0", "cuda:0", seed=0)
    be = BlendingEngine(pipe, run_benchmark=False)
    be.set_prompt1("photo of a lake at dawn")
    be.set_prompt2("an alien planet with two moons")
    unet, vae = be.dh.unet, be.dh.vae
    g = torch.Generator(device="cuda").manual_seed(0)
    for size in args.sizes.split(","):
        wpx, hpx = (int(v) for v in size.lower().split("x"))
        h, w = hpx // 8, wpx // 8
        mp = wpx * hpx / 1e6
        # UNet: one CFG-batch-2 forward
        pl = unet.plan(2, h, w)
        pl.x_in.copy_(torch.randn(pl.x_in.shape, generator=g, device="cuda").half())
        pl.ctx.copy_((torch.randn(pl.ctx.shape, generator=g, device="cuda") * 0.5).half())
        pl.text.copy_(torch.randn(pl.text.shape, generator=g, device="cuda").half())
        pl.tids.copy_(torch.tensor([[hpx, wpx, 0, 0, hpx, wpx]] * 2, dtype=torch.float16, device="cuda"))
        pl.prog_ctx.run()
        unet_ms = time_ms(lambda: pl.prog_step.run(499.0), args.iters)
        # VAE decode
        lat = (torch.randn(1, 4, h, w, generator=g, device="cuda") * 0.8).half()
        vae_ms = time_ms(lambda: vae.decode_to_u8(lat), max(3, args.iters // 2))
        # a short transition
        be.set_dimensions((wpx, hpx))
        be.set_num_inference_steps(args.steps)
        be.set_branching(depth_strength=0.5, nmb_max_branches=args.branches)
        be.output_device_frames = True
        be.run_transition(fixed_seeds=[420, 421])
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        frames = len(be.run_transition(fixed_seeds=[420, 421]))
        torch.cuda.synchronize()
        sec = time.perf_counter() - t0
        assert ops.error_flag() == 0 and vae.overflow_count() == 0
        fps = frames / sec
        emit(dict(size=f"{wpx}x{hpx}", latent=f"{h}x{w}", megapixels=round(mp, 4), unet_b2_ms=round(unet_ms, 2),
                  unet_ms_per_mp=round(unet_ms / mp, 2), vae_ms=round(vae_ms, 2), vae_ms_per_mp=round(vae_ms / mp, 2),
                  transition_frames=frames, transition_fps=round(fps, 3), transition_mp_per_s=round(fps * mp, 3),
                  steps=args.steps, branches=args.branches))
        # free this size's programs and buffers before the next one
        unet._plans.clear()
        vae._plans.clear()
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
