"""LPIPS (AlexNet, v0.1) branch-placement metric on liblb200 (SURVEY.md section 8f "next #2").

Replaces ``lpips.LPIPS(net='alex')`` + ``get_lpips_similarity`` of the reference
(latentblending/blending_engine.py:74-76, :744-758; lpips==0.1.4, un-vendored): the reference converts both PIL images
to numpy, copies them to the GPU, scales them to [-1, 1] and runs AlexNet twice per comparison.  Here
  * frames never leave the device (the VAE kernel writes uint8 HWC frames);
  * the five AlexNet convolutions run on the wgmma GEMM (lb_gemm, ReLU epilogue) over patch matrices; conv1's patch
    matrix is built straight from the uint8 frame with the [-1,1] + ScalingLayer arithmetic fused (lb_lpips_im2col_u8);
  * the feature stack of a frame is computed ONCE and cached -- every frame of the tree is compared twice or more;
  * a comparison is five fused tap reductions (unit-normalise, squared difference, 1x1 lin, spatial mean).
fp16 feature storage, fp32 accumulation and tap arithmetic; there is no CPU path.

Weights use the lpips state_dict layout reduced to what the metric needs:
``convs.{i}.weight/bias`` (AlexNet features 0,3,6,8,10) and ``lins.{i}.weight`` ([1,C,1,1]).
"""
from collections import OrderedDict

import torch

from . import _cabi, ops
from ._cabi import ctx
from .program import Program

_LP_SHIFT = (-0.030, -0.088, -0.188)
_LP_SCALE = (0.458, 0.448, 0.450)
# (cin, cout, kernel, stride, pad) of the five AlexNet convolutions; max-pool 3/2 after the first two taps
_SPEC = ((3, 64, 11, 4, 2), (64, 192, 5, 1, 2), (192, 384, 3, 1, 1), (384, 256, 3, 1, 1), (256, 256, 3, 1, 1))


def lpips_random_state_dict(seed, device):
    """Seeded stand-in weights (no pretrained lpips weights offline): only ranks gaps of a SYNTHETIC pipe."""
    g = torch.Generator(device=device).manual_seed(seed)
    sd = {}
    for i, (ci, co, k, _, _) in enumerate(_SPEC):
        fan_in = ci * k * k
        sd[f"convs.{i}.weight"] = torch.randn(co, ci, k, k, generator=g, device=device) * (2.0 / fan_in) ** 0.5
        sd[f"convs.{i}.bias"] = torch.zeros(co, device=device)
        sd[f"lins.{i}.weight"] = torch.rand(1, co, 1, 1, generator=g, device=device) / co
    return sd


def _conv_out(n, k, s, p):
    return (n + 2 * p - k) // s + 1


class LPIPSAlexB200:
    def __init__(self, state_dict, device, cache_frames=128):
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise _cabi.LB200Error("LPIPSAlexB200 needs a CUDA device (no CPU fallback)")
        self.dev_index = self.device.index or 0
        self.w, self.b, self.lin, self.kp = [], [], [], []
        for i, (ci, co, k, _, _) in enumerate(_SPEC):
            w = state_dict[f"convs.{i}.weight"].detach().to(self.device, torch.float32)
            w = w.permute(0, 2, 3, 1).reshape(co, k * k * ci)              # [co][ky][kx][ci]
            kp = (w.shape[1] + 63) // 64 * 64                               # K padded to the GEMM's 64-column blocks
            wp = torch.zeros(co, kp, dtype=torch.float16, device=self.device)
            wp[:, :w.shape[1]] = w.half()
            self.w.append(wp)
            self.kp.append(kp)
            self.b.append(state_dict[f"convs.{i}.bias"].detach().to(self.device, torch.float16).contiguous())
            self.lin.append(state_dict[f"lins.{i}.weight"].detach().to(self.device, torch.float32).reshape(co).contiguous())
        self._plans = {}
        self._cache = OrderedDict()            # id(frame) -> (frame, taps); the strong ref keeps the id unique
        self._cache_frames = cache_frames
        self._ws = torch.zeros(max(1 << 12, _cabi.load().lb_lpips_tap_workspace_bytes(ctx(self.dev_index))),
                               dtype=torch.uint8, device=self.device)

    # ---- features -------------------------------------------------------------------------------------
    def _plan(self, H, W):
        if (H, W) not in self._plans:
            self._plans[(H, W)] = _LPIPSLowering(self, H, W)
        return self._plans[(H, W)]

    @torch.no_grad()
    def features(self, frame_u8):
        """uint8 [H,W,3] device frame -> list of five [pixels, C] fp16 ReLU taps (cached per frame object)."""
        if not (torch.is_tensor(frame_u8) and frame_u8.is_cuda and frame_u8.dtype == torch.uint8 and frame_u8.dim() == 3):
            raise _cabi.LB200Error("LPIPS needs uint8 [H,W,3] CUDA frames (no CPU fallback)")
        key = id(frame_u8)
        hit = self._cache.get(key)
        if hit is not None and hit[0] is frame_u8:
            self._cache.move_to_end(key)
            return hit[1]
        H, W, _ = frame_u8.shape
        pl = self._plan(H, W)
        pl.frame.copy_(frame_u8)
        pl.prog.run()
        taps = [t.clone() for t in pl.taps]
        self._cache[key] = (frame_u8, taps)
        while len(self._cache) > self._cache_frames:
            self._cache.popitem(last=False)
        return taps

    # ---- distance -------------------------------------------------------------------------------------
    @torch.no_grad()
    def distance_dev(self, frame_a_u8, frame_b_u8, out=None):
        """-> float32 device tensor [1] (no host sync)."""
        fa, fb = self.features(frame_a_u8), self.features(frame_b_u8)
        if out is None:
            out = torch.empty(1, dtype=torch.float32, device=self.device)
        for i in range(5):
            ops.lpips_tap(fa[i], fb[i], self.lin[i], out, self._ws, accumulate=i > 0)
        return out

    def distance(self, frame_a_u8, frame_b_u8):
        """uint8 HxWx3 device frames -> python float (blending_engine.py:750-758)."""
        return float(self.distance_dev(frame_a_u8, frame_b_u8))

    def distance_pair(self, frame, left, right):
        """(d(frame,left), d(frame,right)) with ONE device->host read (the two comparisons of an insertion, :577-579)."""
        both = torch.empty(2, dtype=torch.float32, device=self.device)
        self.distance_dev(frame, left, both[0:1])
        self.distance_dev(frame, right, both[1:2])
        v = both.cpu()
        return float(v[0]), float(v[1])


class _LPIPSLowering:
    """One AlexNet feature pass for a fixed frame size as a C-ABI program: 5 patch-matrix + 5 GEMM + 2 max-pool ops."""

    def __init__(self, net: LPIPSAlexB200, H, W):
        dev = net.device
        f16 = dict(dtype=torch.float16, device=dev)
        P = self.prog = Program(net.dev_index)
        self.frame = torch.zeros(H, W, 3, dtype=torch.uint8, device=dev)
        self.taps = []
        keep = []
        x, h, w = self.frame, H, W
        for i, (ci, co, k, s, p) in enumerate(_SPEC):
            ho, wo = _conv_out(h, k, s, p), _conv_out(w, k, s, p)
            assert ho >= 1 and wo >= 1, "frame too small for the AlexNet feature stack"
            cols = torch.empty(ho * wo, net.kp[i], **f16)
            if i == 0:
                P.lpips_im2col_u8(x, H, W, k, s, p, _LP_SHIFT, _LP_SCALE, cols)
            else:
                P.im2col(x, h, w, ci, k, s, p, cols)
            tap = torch.empty(ho * wo, co, **f16)
            P.gemm(cols, net.w[i], co, 1, 1, ho * wo, tap, bias=net.b[i], relu=True)
            self.taps.append(tap)
            keep.append(cols)
            x, h, w = tap, ho, wo
            if i in (0, 1):
                hp, wp = (h - 3) // 2 + 1, (w - 3) // 2 + 1
                pooled = torch.empty(hp * wp, co, **f16)
                P.maxpool3s2(x, h, w, co, pooled)
                keep.append(pooled)
                x, h, w = pooled, hp, wp
        self._keep = keep
        P.finalize()
