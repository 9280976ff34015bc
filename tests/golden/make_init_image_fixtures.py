"""Generate the VAE-encoder fixtures of image keyframes (fp32 CPU oracle; a few minutes of CPU).

    python tests/golden/make_init_image_fixtures.py

The encoder is oracle/vae_encoder.py's VAEEncoder (diffusers 0.25.0 Encoder + quant_conv + the posterior's mode) at the SDXL
widths (128, 256, 512, 512), seeded with ENC_SEED and its weights rounded to fp16 (``oracle_encoder``).  The images
come from ``fixture_image(H, W)``: smooth seeded colour fields with a little per-pixel noise, so every down level sees
structure.  Stored per fixture: the fp32 latents ``scaling_factor * mean``, the weights checksum and the largest
|activation| of the oracle's modules.

* vae_encoder_sdxl_64.npz        -- a 512x512 image, 64x64 latents.
* vae_encoder_sdxl_53x77.npz     -- a 424x616 image (H x W), 53x77 latents: odd latent sides, so the GEMMs of the
                                    lowest levels take the pixel-run tiling.
* vae_encoder_sdxl_64_upcast.npz -- the 512x512 image through the encoder with conv_in's weight and bias times 2^16:
                                    the residual stream overflows fp16 (asserted: the peak exceeds 65504) while
                                    conv_norm_out brings the output back to ordinary magnitudes.
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

from make_fullsize_fixtures import weights_checksum  # noqa: E402
from make_upcast_fixtures import CONV_IN_SCALE, FP16_MAX  # noqa: E402

ENC_SEED = 5
ENC_CHANNELS = (128, 256, 512, 512)
SQUARE_FIXTURE = os.path.join(HERE, "vae_encoder_sdxl_64.npz")
ODD_FIXTURE = os.path.join(HERE, "vae_encoder_sdxl_53x77.npz")
UPCAST_FIXTURE = os.path.join(HERE, "vae_encoder_sdxl_64_upcast.npz")
SHAPES = {SQUARE_FIXTURE: (512, 512), ODD_FIXTURE: (424, 616), UPCAST_FIXTURE: (512, 512)}


def oracle_encoder(upcast=False):
    from oracle.vae import VAEConfig
    from oracle.vae_encoder import VAEEncoder, synthetic_vae_encoder_init_
    enc = synthetic_vae_encoder_init_(VAEEncoder(VAEConfig(block_out_channels=ENC_CHANNELS)), seed=ENC_SEED).eval()
    with torch.no_grad():
        for p in enc.parameters():
            p.copy_(p.half().float())
        if upcast:
            enc.conv_in.weight.mul_(CONV_IN_SCALE)
            enc.conv_in.bias.mul_(CONV_IN_SCALE)
    return enc


def fixture_image(H, W, seed=7):
    """uint8 [H, W, 3]: a sum of seeded low-frequency sinusoids per channel through tanh (saturated, high-contrast
    colour fields like a photograph's) plus +-8 levels of per-pixel noise."""
    g = np.random.default_rng(seed)
    y, x = np.mgrid[0:H, 0:W].astype(np.float64)
    img = np.zeros((H, W, 3))
    for c in range(3):
        for _ in range(4):
            fy, fx, ph = g.uniform(0.5, 6.0), g.uniform(0.5, 6.0), g.uniform(0, 2 * np.pi)
            img[:, :, c] += np.sin(2 * np.pi * (fy * y / H + fx * x / W) + ph)
    img = 127.5 + 127.5 * np.tanh(0.75 * img) + g.uniform(-8, 8, size=(H, W, 3))
    return np.clip(np.round(img), 0, 255).astype(np.uint8)


def encode_with_peak(enc, image):
    from oracle.vae_encoder import image2latent_np
    peak = [0.0]

    def hook(_m, _i, out):
        if torch.is_tensor(out) and out.is_floating_point():
            peak[0] = max(peak[0], out.detach().abs().max().item())
    hs = [m.register_forward_hook(hook) for m in enc.modules()]
    try:
        lat = image2latent_np(enc, image)
    finally:
        for h in hs:
            h.remove()
    return lat, peak[0]


def make(path, upcast=False):
    H, W = SHAPES[path]
    enc = oracle_encoder(upcast)
    t0 = time.time()
    lat, peak = encode_with_peak(enc, fixture_image(H, W))
    if upcast:
        assert peak > FP16_MAX, f"the recipe must overflow fp16 (max |activation| {peak})"
    np.savez_compressed(path, latents=lat.numpy().astype(np.float32),
                        weights_sha1=np.array(weights_checksum(enc.state_dict())),
                        max_abs_activation=np.float32(peak), seconds=np.float32(time.time() - t0))
    print(f"{os.path.basename(path)}: {time.time() - t0:.0f}s latents {tuple(lat.shape)} std {lat.std():.3f} "
          f"max |act| {peak:.3g}")


if __name__ == "__main__":
    make(SQUARE_FIXTURE)
    make(ODD_FIXTURE)
    make(UPCAST_FIXTURE, upcast=True)
