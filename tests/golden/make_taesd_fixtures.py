"""Generate the tiny-VAE (AutoencoderTiny / TAESDXL) decoder fixtures from the fp32 CPU oracle (seconds of CPU).

    python tests/golden/make_taesd_fixtures.py

Weights: ``random_tiny_vae_state_dict(TAESD_SEED, "cpu")`` (the synthetic pipe's seeded recipe, fp16), default config
(64 channels, blocks (3, 3, 3, 1)), loaded into oracle/taesd.py's DecoderTiny in fp32.  Latents: ``vae_latent`` of
make_fullsize_fixtures.py (seeded N(0, 0.8^2), fp16).

* taesd_sdxl_64.npz     -- 64x64 latents -> the whole 512x512 frame (SDXL-Turbo's size)
* taesd_sdxl_90x160.npz -- 90x160 latents -> a pixel sample of the 720x1280 frame
each holding ``latents`` [1,4,h,w] fp16, the oracle's uint8 ``frame`` and ``weights_sha1`` (so a drift of the init
recipe is caught before the comparison).  The whole 720p frame is noise-like and does not compress (2.4 MB), so that
fixture keeps ``frame`` = frame[rows][:, cols] with ``rows`` / ``cols`` every third index (3 is odd, so every
upsampling phase of all three 2x levels is sampled) plus the 8 pixels next to each border, where the zero padding of
every level shows; ``frame_sample`` applies the same selection to a decoded frame.
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

from make_fullsize_fixtures import vae_latent, weights_checksum  # noqa: E402

TAESD_SEED = 11
FIXTURES = {(64, 64): os.path.join(HERE, "taesd_sdxl_64.npz"), (90, 160): os.path.join(HERE, "taesd_sdxl_90x160.npz")}
SAMPLED = {(90, 160)}       # fixtures that store a pixel sample of the frame (see the module docstring)
BORDER = 8


def sample_indices(n):
    """Every third index of a side of n pixels plus the BORDER pixels next to each end."""
    return np.array(sorted(set(range(0, n, 3)) | set(range(BORDER)) | set(range(n - BORDER, n))), dtype=np.int64)


def frame_sample(frame, fx):
    """``frame`` reduced to what fixture ``fx`` stores: itself, or its rows[fx["rows"]] x cols[fx["cols"]] sample."""
    if "rows" not in fx:
        return frame
    return frame[np.ix_(fx["rows"], fx["cols"])]


def tiny_state_dict():
    from latentblending_b200.pipe import random_tiny_vae_state_dict
    return random_tiny_vae_state_dict(TAESD_SEED, "cpu")


def oracle_taesd(state_dict=None, config=None):
    """fp32 DecoderTiny holding ``state_dict`` (default: the fixtures' seeded fp16 weights)."""
    from oracle.taesd import DecoderTiny, TinyVAEConfig
    dec = DecoderTiny(config or TinyVAEConfig()).eval()
    sd = tiny_state_dict() if state_dict is None else state_dict
    dec.load_state_dict({k: v.float() for k, v in sd.items()}, strict=True)
    return dec


def make(h, w):
    from oracle.taesd import latent2image_np
    sd = tiny_state_dict()
    dec = oracle_taesd(sd)
    lat = vae_latent(h, w)
    t0 = time.time()
    with torch.no_grad():
        frame = latent2image_np(dec, lat)
    path = FIXTURES[(h, w)]
    extra = {}
    if (h, w) in SAMPLED:
        extra = dict(rows=sample_indices(frame.shape[0]), cols=sample_indices(frame.shape[1]))
        frame = frame_sample(frame, extra)
    np.savez_compressed(path, latents=lat.numpy(), frame=frame, weights_sha1=np.array(weights_checksum(sd)), **extra)
    clipped = float(((frame == 0) | (frame == 255)).mean())
    print(f"taesd fixture {h}x{w}: {time.time() - t0:.1f}s frame {frame.shape} std {frame.std():.1f} "
          f"clipped {clipped:.4f} -> {path}")


if __name__ == "__main__":
    for (h, w) in FIXTURES:
        make(h, w)
