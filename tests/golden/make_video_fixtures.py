"""Generate the parity fixture at a video output size from the fp32 CPU oracle (minutes of CPU).

    python tests/golden/make_video_fixtures.py

* unet_sdxl_b2_90x160.npz -- ONE CFG-batch-2 forward of the full SDXL-base UNet at 1280x720 (latent h=90, w=160).
                             90 is not divisible by 4: the levels are 90x160 -> 45x80 -> 23x40, and the level-2 ->
                             level-1 upsampler resizes 23 -> 45 rows (nearest 2x, then the last row dropped).
                             ``eps`` [2,4,90,160] fp32 plus the seeded weights' checksum.

Same seeded weights, inputs and storage as make_fullsize_fixtures.py (whose recipe this reuses); only the shape
differs.  The oracle forward applies diffusers' resize-to-skip-size rule (sized_unet.py).
"""
import os
import sys
import time

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)
from make_fullsize_fixtures import UNET_SEED, UNET_T, oracle_unet, unet_inputs, weights_checksum  # noqa: E402
from sized_unet import forward_sized  # noqa: E402

UNET_VIDEO_FIXTURE = os.path.join(HERE, "unet_sdxl_b2_90x160.npz")
UNET_VIDEO_HW = (90, 160)


def make_unet():
    from oracle.sdxl_unet import SDXL_BASE
    t0 = time.time()
    net = oracle_unet()
    x, ctx, pooled, tids = unet_inputs(SDXL_BASE, 2, *UNET_VIDEO_HW, UNET_SEED)
    t1 = time.time()
    with torch.no_grad():
        eps = forward_sized(net, x.float(), UNET_T, ctx.float(), pooled.float(), tids.float())
    t2 = time.time()
    np.savez_compressed(UNET_VIDEO_FIXTURE, eps=eps.numpy().astype(np.float32), t=np.float32(UNET_T),
                        weights_sha1=np.array(weights_checksum(net.state_dict())),
                        threads=np.int32(torch.get_num_threads()), seconds=np.float32(t2 - t1))
    print(f"unet video fixture: init {t1 - t0:.0f}s forward {t2 - t1:.0f}s  |eps|={eps.norm():.4f} "
          f"finite={bool(torch.isfinite(eps).all())} threads={torch.get_num_threads()} -> {UNET_VIDEO_FIXTURE}")


if __name__ == "__main__":
    make_unet()
