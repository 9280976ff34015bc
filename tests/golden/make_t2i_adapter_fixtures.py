"""Generate the full-size T2I-Adapter parity fixture from the fp32 CPU oracle (a few minutes of CPU).

    python tests/golden/make_t2i_adapter_fixtures.py

* t2i_adapter_sdxl_b2_128.npz -- ONE CFG-batch-2 forward of the full SDXL-base UNet (make_fullsize_fixtures.py's
                                 seeded weights) with an RGB SDXL T2I-Adapter (oracle/t2i_adapter.py, FullAdapterXL,
                                 seeded, block2 damped but non-zero), weights rounded to fp16 first, at 128x128 latents
                                 with a 1024x1024 image and adapter_conditioning_scale SCALE: ``eps`` [2,4,128,128]
                                 fp32 plus a checksum of both nets' seeded weights.

The inputs and the image are rebuilt by the test from the functions below; only the oracle's output is stored.  The
oracle restates diffusers 0.25.0 T2IAdapter without having been checked against the package.
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

from make_controlnet_fixtures import control_image  # noqa: E402
from make_fullsize_fixtures import oracle_unet, unet_inputs, weights_checksum  # noqa: E402

FIXTURE = os.path.join(HERE, "t2i_adapter_sdxl_b2_128.npz")
T = 499.0
SCALE = 0.8
SEED = 0
ADAPTER_SEED = 2


def inputs():
    from oracle.sdxl_unet import SDXL_BASE
    return unet_inputs(SDXL_BASE, 2, 128, 128, SEED)


def adapter_image():
    """uint8 [1024, 1024, 3]: the ControlNet fixture's edge / gradient map."""
    return control_image()


def oracle_adapter():
    from oracle.t2i_adapter import T2IAdapter, synthetic_init_adapter_
    ad = synthetic_init_adapter_(T2IAdapter(3), seed=ADAPTER_SEED).eval()
    with torch.no_grad():
        for p in ad.parameters():
            p.copy_(p.half().float())
    return ad


def make():
    from oracle.t2i_adapter import adapter_states, image_to_adapter_input, unet_with_adapter
    t0 = time.time()
    unet, ad = oracle_unet(), oracle_adapter()
    x, ctx, pooled, tids = inputs()
    t1 = time.time()
    with torch.no_grad():
        states = adapter_states(ad, image_to_adapter_input(adapter_image()), SCALE)
        eps = unet_with_adapter(unet, x.float(), T, ctx.float(), pooled.float(), tids.float(), states)
        plain = unet_with_adapter(unet, x.float(), T, ctx.float(), pooled.float(), tids.float())
    t2 = time.time()
    sha = weights_checksum(unet.state_dict()) + weights_checksum(ad.state_dict())
    effect = float((eps - plain).norm() / eps.norm())
    np.savez_compressed(FIXTURE, eps=eps.numpy().astype(np.float32), t=np.float32(T), scale=np.float32(SCALE),
                        effect=np.float32(effect), weights_sha1=np.array(sha), seconds=np.float32(t2 - t1))
    print(f"t2i-adapter fixture: init {t1 - t0:.0f}s forward {t2 - t1:.0f}s |eps|={eps.norm():.4f} "
          f"adapter changes eps by {effect:.3e} finite={bool(torch.isfinite(eps).all())} -> {FIXTURE}")


if __name__ == "__main__":
    make()
