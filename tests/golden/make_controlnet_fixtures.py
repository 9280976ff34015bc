"""Generate the full-size ControlNet parity fixture from the fp32 CPU oracle (minutes of CPU).

    python tests/golden/make_controlnet_fixtures.py

* controlnet_sdxl_b2_128.npz -- ONE CFG-batch-2 forward of the full SDXL-base UNet (make_fullsize_fixtures.py's
                                seeded weights) with the "full" SDXL ControlNet (oracle/controlnet.py, transformer
                                depths 0/2/10, seeded zero convs damped but non-zero), weights rounded to fp16 first,
                                at 128x128 latents with a 1024x1024 control image and conditioning scale SCALE:
                                ``eps`` [2,4,128,128] fp32 plus a checksum of both nets' seeded weights.

The inputs and the control image are rebuilt by the test from the functions below; only the oracle's output is
stored.  The oracle restates diffusers 0.25.0 ControlNetModel without having been checked against the package.
"""
import os
import sys
import time

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (ROOT, HERE):
    if p not in sys.path:
        sys.path.insert(0, p)

from make_fullsize_fixtures import oracle_unet, unet_inputs, weights_checksum  # noqa: E402

FIXTURE = os.path.join(HERE, "controlnet_sdxl_b2_128.npz")
T = 499.0
SCALE = 0.8
SEED = 0
CN_SEED = 1


def inputs():
    from oracle.sdxl_unet import SDXL_BASE
    return unet_inputs(SDXL_BASE, 2, 128, 128, SEED)


def control_image():
    """uint8 [1024, 1024, 3]: a gradient with a checkerboard of edges and some noise, like an edge or depth map."""
    g = torch.Generator().manual_seed(11)
    yy, xx = torch.meshgrid(torch.arange(1024), torch.arange(1024), indexing="ij")
    img = (xx // 4 + ((yy // 64 + xx // 64) % 2) * 120)[..., None] + torch.randint(0, 40, (1024, 1024, 3), generator=g)
    return (img % 256).to(torch.uint8)


def oracle_nets():
    from oracle.controlnet import SDXLControlNet, synthetic_init_controlnet_
    from oracle.sdxl_unet import SDXL_BASE
    unet = oracle_unet()
    cn = synthetic_init_controlnet_(SDXLControlNet(SDXL_BASE), seed=CN_SEED).eval()
    with torch.no_grad():
        for p in cn.parameters():
            p.copy_(p.half().float())
    return unet, cn


def make():
    from oracle.controlnet import image_to_cond, unet_with_residuals
    t0 = time.time()
    unet, cn = oracle_nets()
    x, ctx, pooled, tids = inputs()
    img = image_to_cond(control_image()).expand(2, -1, -1, -1)
    t1 = time.time()
    with torch.no_grad():
        down, mid = cn(x.float(), T, ctx.float(), pooled.float(), tids.float(), img, conditioning_scale=SCALE)
        eps = unet_with_residuals(unet, x.float(), T, ctx.float(), pooled.float(), tids.float(), down, mid)
    t2 = time.time()
    sha = weights_checksum(unet.state_dict()) + weights_checksum(cn.state_dict())
    np.savez_compressed(FIXTURE, eps=eps.numpy().astype(np.float32), t=np.float32(T), scale=np.float32(SCALE),
                        weights_sha1=np.array(sha), seconds=np.float32(t2 - t1))
    print(f"controlnet fixture: init {t1 - t0:.0f}s forward {t2 - t1:.0f}s |eps|={eps.norm():.4f} "
          f"finite={bool(torch.isfinite(eps).all())} -> {FIXTURE}")


if __name__ == "__main__":
    make()
