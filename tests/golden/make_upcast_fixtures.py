"""Generate the fixture of a VAE decoder whose activations overflow fp16 (fp32 CPU oracle; about a minute of CPU).

    python tests/golden/make_upcast_fixtures.py

* vae_sdxl_64_upcast.npz -- one decode of the SDXL-width VAE decoder (128,256,512,512; oracle/vae.py, fp32; seed 4,
                            weights rounded to fp16 as in make_fullsize_fixtures.py) at 64x64 latents, with conv_in's
                            weight and bias multiplied by 2^16 (``upcast_state_dict``).  GroupNorm undoes the scale
                            inside every resnet branch, but the residual stream carries it: activations reach ~10^6,
                            far past fp16's 65504, as the stock SDXL VAE's do (its config sets force_upcast).  The
                            factor is a power of two, so the scaled weights are exact and still fp16-representable,
                            like real checkpoint weights.  Stored: the uint8 frame [512,512,3], the weights checksum
                            and the largest |activation| the oracle produced.
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

from make_fullsize_fixtures import oracle_vae, vae_latent, weights_checksum  # noqa: E402

UPCAST_FIXTURE = os.path.join(HERE, "vae_sdxl_64_upcast.npz")
CONV_IN_SCALE = 2.0 ** 16
FP16_MAX = 65504.0


def upcast_(ov):
    """Scale conv_in of an oracle decoder (whose weights are already fp16-rounded) by 2^16, in place."""
    with torch.no_grad():
        ov.conv_in.weight.mul_(CONV_IN_SCALE)
        ov.conv_in.bias.mul_(CONV_IN_SCALE)
    wmax = max(ov.conv_in.weight.abs().max().item(), ov.conv_in.bias.abs().max().item())
    assert wmax < FP16_MAX, f"scaled conv_in weights ({wmax}) must stay fp16-representable"
    for t in (ov.conv_in.weight, ov.conv_in.bias):
        assert torch.equal(t.half().float(), t), "scaled conv_in weights must be exact in fp16"
    return ov


def max_activation(ov, lat):
    """(frame, largest |output| of any oracle module) for one decode."""
    from oracle.vae import latent2image_np
    peak = [0.0]

    def hook(_m, _i, out):
        if torch.is_tensor(out) and out.is_floating_point():
            peak[0] = max(peak[0], out.detach().abs().max().item())
    hs = [m.register_forward_hook(hook) for m in ov.modules()]
    try:
        with torch.no_grad():
            frame = latent2image_np(ov, lat)
    finally:
        for h in hs:
            h.remove()
    return frame, peak[0]


def make_upcast():
    ov, cfg = oracle_vae()
    upcast_(ov)
    lat = vae_latent(64, 64)
    t0 = time.time()
    frame, peak = max_activation(ov, lat)
    assert peak > FP16_MAX, f"the recipe must overflow fp16 (max |activation| {peak})"
    np.savez_compressed(UPCAST_FIXTURE, frame=frame, weights_sha1=np.array(weights_checksum(ov.state_dict())),
                        max_abs_activation=np.float32(peak), seconds=np.float32(time.time() - t0))
    print(f"upcast vae fixture: {time.time() - t0:.0f}s frame {frame.shape} std {frame.std():.1f} "
          f"max |act| {peak:.3g} -> {UPCAST_FIXTURE}")


if __name__ == "__main__":
    make_upcast()
