"""Time every distinct GEMM / implicit-GEMM conv shape of the SDXL UNet forward at 128x128 latents (1024^2 images)
for batch 1, 2 and 4, and the big 3x3 convolutions of the VAE decoder, with CUDA events.

    python tools/gemm_shapes.py [--root DIR] [--batches 1,2,4] [--out FILE.jsonl] [--latent HxW]
                                [--tiling auto|box|runs]

One JSON line per (shape, batch): us per launch, TFLOP/s, launches per forward, ms per forward.  Linear shapes also
carry the time of torch.nn.functional.linear (cuBLAS, fp16) at the same shape as a same-card reference ceiling; it
is a yardstick only, nothing in the library calls it.  The summary lines give the UNet GEMM time per forward at each
batch and the time weighted by a transition's program mix (``--mix``: forwards per transition at batch 4 and at
batch 1; the default is config 2's lockstep-speculation split, cross-check it with bench.py's `speculation` field).
``--root`` imports latentblending_b200 from another checkout (e.g. a build of an earlier commit) to compare builds.
``--latent HxW`` times the shapes of another output size (latent height x width, e.g. 152x104 for 832x1216 images);
``--tiling`` forces the GEMM's M tiling (the default lets lb_gemm choose; builds without the option need the default).
Each shape is recorded once into a one-record Program and replayed, as the lowered programs replay it.
The first line records the card, its power limit and its SM clocks (nvidia-smi, read-only).
"""
import argparse
import json
import os
import subprocess
import sys


def card_info():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30)
        vals = [v.strip() for v in r.stdout.strip().splitlines()[0].split(",")]
        return dict(zip(q.split(","), vals))
    except Exception as e:  # noqa: BLE001 -- the table is still useful without it
        return {"error": repr(e)}


def unet_shapes(h=128, w=128):
    """(name, (height, width), N, K-per-tap, taps, a1_c, res, geglu, launches per forward) of the SDXL UNet
    (block_out_channels 320/640/1280, 2 layers per block, transformer depth 0/2/10), per CFG-batch forward."""
    shapes = {}

    def add(name, hw, N, K, taps=1, a1_c=0, res=False, geglu=False, n=1):
        key = (name, hw, N, K, taps, a1_c, res, geglu)
        shapes[key] = shapes.get(key, 0) + n

    def resnet(hw, cin, cout):
        add("conv1", hw, cout, cin, taps=9)
        if cin != cout:
            add("conv2+shortcut", hw, cout, cout, taps=9, a1_c=cin)
        else:
            add("conv2+res", hw, cout, cout, taps=9, res=True)

    def transformer(hw, C, depth):
        add("proj_in", hw, C, C)
        add("proj_out+res", hw, C, C, res=True)
        add("attn1.qkv", hw, 3 * C, C, n=depth)
        add("attn1.out+res", hw, C, C, res=True, n=depth)
        add("attn2.q", hw, C, C, n=depth)
        add("attn2.out+res", hw, C, C, res=True, n=depth)
        add("ff.in(geglu)", hw, 8 * C, C, geglu=True, n=depth)
        add("ff.out+res", hw, C, 4 * C, res=True, n=depth)

    ch, depth = (320, 640, 1280), (0, 2, 10)
    hws = [(h, w)]
    for _ in range(2):      # the stride-2 pad-1 downsample conv gives ceil(s/2)
        hws.append(((hws[-1][0] + 1) // 2, (hws[-1][1] + 1) // 2))
    skips = [320]
    cin = 320
    for lvl in range(3):
        for _ in range(2):
            resnet(hws[lvl], cin, ch[lvl])
            cin = ch[lvl]
            if depth[lvl]:
                transformer(hws[lvl], cin, depth[lvl])
            skips.append(cin)
        if lvl < 2:
            add("downsample(im2col)", hws[lvl + 1], cin, 9 * cin)
            skips.append(cin)
    resnet(hws[2], 1280, 1280)
    transformer(hws[2], 1280, 10)
    resnet(hws[2], 1280, 1280)
    for lvl in (2, 1, 0):
        for _ in range(3):
            resnet(hws[lvl], cin + skips.pop(), ch[lvl])
            cin = ch[lvl]
            if depth[lvl]:
                transformer(hws[lvl], cin, depth[lvl])
        if lvl > 0:
            add("upsample", hws[lvl - 1], cin, cin, taps=9)
    return shapes


# (name, image size / latent size, cin, cout); the names give the sizes at 128x128 latents
VAE = (("vae_up3_128", 8, 128, 128), ("vae_upconv_256", 8, 256, 256), ("vae_up2_256", 4, 256, 256),
       ("vae_upconv_512", 4, 512, 512), ("vae_up1_512", 2, 512, 512), ("vae_up0_512", 1, 512, 512))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    ap.add_argument("--batches", default="1,2,4")
    ap.add_argument("--mix", default="87,48", help="programs per transition at batch 4 and at batch 1")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    ap.add_argument("--no-vae", action="store_true")
    ap.add_argument("--geglu-flags", type=lambda v: int(v, 0), default=0,
                    help="extra lb_gemm_desc.mode flags of the GEGLU launches (for builds with other GEGLU tiles)")
    ap.add_argument("--latent", default="128x128", help="latent height x width")
    ap.add_argument("--tiling", default="auto", choices=("auto", "box", "runs"))
    args = ap.parse_args()
    lh, lw = (int(v) for v in args.latent.lower().split("x"))
    tile_kw = {} if args.tiling == "auto" else dict(tiling=args.tiling)
    sys.path.insert(0, os.path.abspath(args.root))
    import torch
    import torch.nn.functional as F
    from latentblending_b200 import ops
    from latentblending_b200._cabi import LB200Error
    try:
        from latentblending_b200.program import Program
    except ImportError:             # checkouts from before program.py
        from latentblending_b200.unet import Program
    assert torch.cuda.is_available(), "gemm_shapes.py needs a CUDA device"

    sink = open(args.out, "a") if args.out else None

    def emit(d):
        line = json.dumps(d)
        print(line, flush=True)
        if sink:
            sink.write(line + "\n")

    def gemm_run(*args, **kw):
        """The run() of a one-record Program holding this GEMM."""
        P = Program(0)
        P.gemm(*args, **kw)
        return P.finalize().run

    def time_it(fn, iters):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(iters):
            fn()
        e.record()
        torch.cuda.synchronize()
        return s.elapsed_time(e) / iters * 1e3       # us

    head = dict(card=card_info(), root=os.path.abspath(args.root), lib=ops.__file__)
    if (lh, lw) != (128, 128) or tile_kw:
        head.update(latent=[lh, lw], tiling=args.tiling)
    emit(head)
    g = torch.Generator(device="cuda").manual_seed(0)

    def rnd(*shape, s=1.0):
        return (torch.randn(*shape, generator=g, device="cuda") * s).half()

    totals = {}
    for B in [int(b) for b in args.batches.split(",")]:
        total = 0.0
        for (name, (h, w), N, K, taps, a1_c, res, geglu), n in unet_shapes(lh, lw).items():
            M = B * h * w
            Ktot = taps * K + a1_c
            a = rnd(M, K)
            a1 = rnd(M, a1_c) if a1_c else None
            bias = rnd(N)
            r = rnd(M, N) if res else None
            out = torch.empty(M, N // 2 if geglu else N, device="cuda", dtype=torch.float16)
            wt = rnd(N, Ktot, s=Ktot ** -0.5)
            try:
                us = time_it(gemm_run(a, wt, N, B, h, w, out, taps=taps, a1=a1, bias=bias, res=r,
                                      mode=(1 | args.geglu_flags) if geglu else 0, **tile_kw), args.iters)
            except LB200Error as e:      # a build or tiling that cannot run this shape
                emit(dict(op="unet_gemm", name=name, B=B, hw=h if h == w else f"{h}x{w}", error=str(e)))
                continue
            assert ops.error_flag() == 0
            fl = 2.0 * M * N * Ktot
            row = dict(op="unet_gemm", name=name, B=B, hw=h if h == w else f"{h}x{w}", M=M, N=N, K=Ktot, taps=taps, us=round(us, 2),
                       tflops=round(fl / us / 1e6, 1), launches=n, ms_per_forward=round(us * n / 1e3, 3))
            if taps == 1 and not a1_c:
                us_ref = time_it(lambda: F.linear(a, wt, bias), args.iters)
                row.update(cublas_us=round(us_ref, 2), cublas_tflops=round(fl / us_ref / 1e6, 1))
            emit(row)
            total += us * n / 1e3
            del a, a1, wt, bias, r, out
        totals[B] = total
        emit(dict(op="unet_gemm_total", B=B, ms_per_forward=round(total, 3)))
    n4, n1 = (int(x) for x in args.mix.split(","))
    if 4 in totals and 1 in totals:
        emit(dict(op="unet_gemm_transition", programs_b4=n4, programs_b1=n1,
                  ms=round(n4 * totals[4] + n1 * totals[1], 1)))
    if not args.no_vae:
        for name, f, cin, cout in VAE:
            h, w = f * lh, f * lw
            M = h * w
            a = rnd(M, cin)
            wt = rnd(cout, 9 * cin, s=(9 * cin) ** -0.5)
            out = torch.empty(M, cout, device="cuda", dtype=torch.float16)
            try:
                us = time_it(gemm_run(a, wt, cout, 1, h, w, out, taps=9, **tile_kw), 5)
            except LB200Error as e:
                emit(dict(op="vae_conv3x3", name=name, h=h, w=w, error=str(e)))
                continue
            fl = 2.0 * M * cout * 9 * cin
            row = dict(op="vae_conv3x3", name=name, M=M, N=cout, K=9 * cin, us=round(us, 1),
                       tflops=round(fl / us / 1e6, 1))
            if (lh, lw) != (128, 128):
                row.update(h=h, w=w)
            emit(row)
            del a, wt, out


if __name__ == "__main__":
    main()
