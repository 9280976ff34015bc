"""Generate the parity fixtures at an SDXL aspect-ratio bucket from the fp32 CPU oracle (about a minute of CPU).

    python tests/golden/make_bucket_fixtures.py [unet] [vae]

* unet_sdxl_b2_152x104.npz -- ONE CFG-batch-2 forward of the full SDXL-base UNet at the 832x1216 (portrait) bucket,
                              latent h=152, w=104: every level width (104, 52, 26) is one the pixel-box GEMM tiling
                              cannot tile.  ``eps`` [2,4,152,104] fp32 plus the seeded weights' checksum.
* vae_sdxl_52x76.npz       -- one decode of the SDXL-width VAE decoder at 52x76 latents -> uint8 frame [416,608,3].

Same seeded weights, inputs and storage as make_fullsize_fixtures.py (whose recipe this reuses); only the shape
differs.
"""
import os
import sys
import time

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)
from make_fullsize_fixtures import (UNET_SEED, UNET_T, oracle_unet, oracle_vae, unet_inputs,  # noqa: E402
                                    vae_latent, weights_checksum)

UNET_BUCKET_FIXTURE = os.path.join(HERE, "unet_sdxl_b2_152x104.npz")
UNET_BUCKET_HW = (152, 104)
VAE_BUCKET_FIXTURE = os.path.join(HERE, "vae_sdxl_52x76.npz")
VAE_BUCKET_HW = (52, 76)


def make_unet():
    from oracle.sdxl_unet import SDXL_BASE
    t0 = time.time()
    net = oracle_unet()
    x, ctx, pooled, tids = unet_inputs(SDXL_BASE, 2, *UNET_BUCKET_HW, UNET_SEED)
    t1 = time.time()
    with torch.no_grad():
        eps = net(x.float(), UNET_T, ctx.float(), pooled.float(), tids.float())
    t2 = time.time()
    np.savez_compressed(UNET_BUCKET_FIXTURE, eps=eps.numpy().astype(np.float32), t=np.float32(UNET_T),
                        weights_sha1=np.array(weights_checksum(net.state_dict())),
                        threads=np.int32(torch.get_num_threads()), seconds=np.float32(t2 - t1))
    print(f"unet bucket fixture: init {t1 - t0:.0f}s forward {t2 - t1:.0f}s  |eps|={eps.norm():.4f} "
          f"finite={bool(torch.isfinite(eps).all())} -> {UNET_BUCKET_FIXTURE}")


def make_vae():
    from oracle.vae import latent2image_np
    ov, cfg = oracle_vae()
    lat = vae_latent(*VAE_BUCKET_HW)
    t0 = time.time()
    with torch.no_grad():
        frame = latent2image_np(ov, lat)
    np.savez_compressed(VAE_BUCKET_FIXTURE, frame=frame, weights_sha1=np.array(weights_checksum(ov.state_dict())),
                        seconds=np.float32(time.time() - t0))
    print(f"vae bucket fixture: {time.time() - t0:.0f}s frame {frame.shape} std {frame.std():.1f} -> {VAE_BUCKET_FIXTURE}")


if __name__ == "__main__":
    what = sys.argv[1:] or ["vae", "unet"]
    if "vae" in what:
        make_vae()
    if "unet" in what:
        make_unet()
