"""Seeded inputs of the slerp / lerp golden vectors (slerp.npz stores only the reference's outputs for them)."""
import torch

SIZES = ((64, torch.float16), (4 * 16 * 16, torch.float16), (4 * 64 * 64, torch.float16),
         (4 * 128 * 128, torch.float16), (777, torch.float32))
FRACTS = (0.0, 0.25, 0.5, 0.3141, 1.0)


def slerp_inputs():
    """[(p0, p1, fract)] for case k = 0, 1, ... and the generator, positioned for lerp_inputs()."""
    g = torch.Generator().manual_seed(1234)
    cases = []
    for k, (n, dt, f) in enumerate((n, dt, f) for n, dt in SIZES for f in FRACTS):
        p0 = (torch.randn(n, generator=g) * (1 + k % 3)).to(dt)
        p1 = (torch.randn(n, generator=g) * 2).to(dt)
        if k % 7 == 3:
            p1 = (p0.float() * 1.5).to(dt)          # parallel vectors -> exercises the 1e-7 clamp
        cases.append((p0, p1, f))
    return cases, g
