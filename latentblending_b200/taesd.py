"""Tiny SDXL autoencoder decoder (AutoencoderTiny / TAESDXL) on liblb200.

What the reference decodes when ``pipe.vae`` is ``AutoencoderTiny.from_pretrained('madebyollin/taesdxl')``
(blending_engine.py:797,806, diffusers_holder.py:373,379): ``latent2image`` calls ``vae.decode(latents /
scaling_factor)``, which for diffusers 0.25.0 ``DecoderTiny`` is

    x = tanh(z / 3) * 3
    Conv2d(4, C, 3) ReLU, then per group i: num_decoder_blocks[i] x Block(C, C), nearest-2x Upsample (not after the
    last group), Conv2d(C, C or 3, 3) (bias only on the last)
    Block(x) = ReLU(conv3(ReLU(conv2(ReLU(conv1(x))))) + x)
    return layers(x) * 2 - 1

About 0.56 TFLOP per 1024^2 frame against the KL decoder's 10.5.  Lowering (fp16 storage, fp32 accumulation):
  * the clamp, conv_in and its ReLU: one lb_conv_in (act 1) launch;
  * every block conv: an implicit-GEMM 3x3 conv with LB_GEMM_RELU; the third also adds the block input as the
    GEMM residual (bias, then residual, then ReLU: the reference's order), written over that input in place;
  * upsample + conv: ONE GEMM over the low-resolution map (LB_GEMM_D2S2) with four phase filters, whose epilogue
    stores each phase's outputs at their upsampled pixels -- the upsampled map is never written or read;
  * the final C -> 3 conv with ``* 2 - 1`` folded into its weights and bias (in fp32): the N = 8 conv_out GEMM, then
    NCHW and the uint8 post-processing, which counts non-finite pixels.
Activations ping-pong between three [pixels, C] buffers sized for the output resolution.  Weights use the diffusers
``decoder.`` state_dict names with that prefix stripped.
"""
import torch

from . import _cabi
from .lowering import pack3
from .program import Program, pack_conv_out8
from .vae import DecoderBase

DEFAULT_CONFIG = dict(latent_channels=4, out_channels=3, decoder_block_out_channels=(64, 64, 64, 64),
                      num_decoder_blocks=(3, 3, 3, 1), upsampling_scaling_factor=2, act_fn="relu",
                      scaling_factor=1.0, force_upcast=False)


def tiny_config(config=None):
    """The decoder fields of an AutoencoderTiny config (dict, diffusers FrozenDict or attribute object), with the
    diffusers defaults for missing keys."""
    out = {}
    for k, default in DEFAULT_CONFIG.items():
        if config is None:
            v = default
        elif isinstance(config, dict):
            v = config[k] if k in config else default
        else:
            v = getattr(config, k, default)
        out[k] = tuple(v) if isinstance(v, (list, tuple)) else v
    return out


def decoder_layout(config=None):
    """[(kind, layer index, group)] of ``decoder.layers`` for this config: kind "conv_in", "block", "up_conv" (the
    conv after a group's Upsample) or "conv_out".  ReLU / Upsample indices carry no parameters and are skipped."""
    cfg = tiny_config(config)
    nb = cfg["num_decoder_blocks"]
    layout = [("conv_in", 0, 0)]
    idx = 2                                   # 1: the ReLU after conv_in
    for i, n in enumerate(nb):
        last = i == len(nb) - 1
        for _ in range(n):
            layout.append(("block", idx, i))
            idx += 1
        if not last:
            idx += 1                          # Upsample
        layout.append(("conv_out" if last else "up_conv", idx, i))
        idx += 1
    return layout


def expected_keys(config=None):
    """The decoder state_dict keys (``decoder.`` stripped) an AutoencoderTiny with this config has."""
    keys = []
    for kind, idx, _ in decoder_layout(config):
        if kind == "block":
            for j in (0, 2, 4):
                keys += [f"layers.{idx}.conv.{j}.weight", f"layers.{idx}.conv.{j}.bias"]
        else:
            keys.append(f"layers.{idx}.weight")
            if kind != "up_conv":
                keys.append(f"layers.{idx}.bias")
    return keys


def check_config(config=None):
    """ValueError unless this is a decoder the native path implements; returns the normalised config."""
    cfg = tiny_config(config)
    ch, nb = cfg["decoder_block_out_channels"], cfg["num_decoder_blocks"]
    if len(ch) != len(nb) or len(ch) < 1:
        raise ValueError(f"tiny VAE: decoder_block_out_channels {ch} and num_decoder_blocks {nb} differ in length")
    if len(set(ch)) != 1 or ch[0] % 64 != 0:
        raise ValueError(f"tiny VAE: the native decoder needs equal decoder_block_out_channels that are a multiple of "
                         f"64 (got {ch})")
    if cfg["upsampling_scaling_factor"] != 2:
        raise ValueError(f"tiny VAE: upsampling_scaling_factor must be 2 (got {cfg['upsampling_scaling_factor']})")
    if cfg["act_fn"] != "relu":
        raise ValueError(f"tiny VAE: act_fn must be 'relu' (got {cfg['act_fn']!r})")
    if cfg["latent_channels"] != 4:
        raise ValueError(f"tiny VAE: latent_channels must be 4 (got {cfg['latent_channels']})")
    if cfg["out_channels"] != 3:
        raise ValueError(f"tiny VAE: out_channels must be 3 (got {cfg['out_channels']})")
    return cfg


def check_state_dict(state_dict, config=None):
    """ValueError listing the missing and unexpected keys unless the decoder state_dict matches the config exactly."""
    want, have = set(expected_keys(config)), set(state_dict)
    if want != have:
        raise ValueError(f"tiny VAE decoder state_dict does not match its config: missing {sorted(want - have)}, "
                         f"unexpected {sorted(have - want)}")


def pack_d2s_weights(w):
    """Phase filters of nearest-2x upsample + 3x3 conv (padding 1): ``w`` [Co, Ci, 3, 3] -> [4*Co, Ci, 3, 3], row
    p*Co + c with p = 2a + b the phase of output pixel (2y + a, 2x + b), each a 3x3 filter over LOW-resolution taps.
    Upsampled row offset dy reads low-resolution row y + (a + dy) // 2: for a = 0, dy = -1 -> -1 and dy in {0, 1} ->
    0; for a = 1, dy in {-1, 0} -> 0 and dy = 1 -> +1 (columns alike with b).  The original taps that land on the
    same low-resolution tap are summed in ``w``'s dtype (at least fp32); taps a phase never reads stay zero.  Zero
    padding agrees at every border: upsampled rows -1 and 2H are low-resolution rows -1 and H."""
    acc_dtype = torch.float64 if w.dtype == torch.float64 else torch.float32
    Co, Ci = w.shape[0], w.shape[1]
    wf = w.to(acc_dtype)
    out = torch.zeros(2, 2, Co, Ci, 3, 3, dtype=acc_dtype, device=w.device)
    for a in range(2):
        for ky in range(3):
            ly = (a + ky - 1) // 2 + 1
            for b in range(2):
                for kx in range(3):
                    lx = (b + kx - 1) // 2 + 1
                    out[a, b, :, :, ly, lx] += wf[:, :, ky, kx]
    return out.reshape(4 * Co, Ci, 3, 3)


class TinyVAEDecoderB200(DecoderBase):
    """The AutoencoderTiny decoder, fp16 storage / fp32 accumulation (the only precision it has here)."""
    dtype = torch.float16

    def __init__(self, state_dict, config, scaling_factor, device):
        cfg = check_config(config)
        check_state_dict(state_dict, cfg)
        super().__init__(device)
        self.config = cfg
        self.scaling_factor = float(scaling_factor)
        self.channels = cfg["decoder_block_out_channels"][0]
        self.layout = decoder_layout(cfg)
        dev = self.device
        sd = state_dict

        def f32(n):
            return sd[n].detach().to(device=dev, dtype=torch.float32)

        def f16(t):
            return t.to(torch.float16).contiguous()

        W = self.w = {}
        for kind, idx, _ in self.layout:
            if kind == "conv_in":
                W["in.w"] = f16(f32(f"layers.{idx}.weight").permute(2, 3, 1, 0))      # [ky][kx][cin][Cout]
                W["in.b"] = f16(f32(f"layers.{idx}.bias"))
            elif kind == "block":
                for j in (0, 2, 4):
                    W[f"{idx}.{j}.w"] = f16(pack3(f32(f"layers.{idx}.conv.{j}.weight")))
                    W[f"{idx}.{j}.b"] = f16(f32(f"layers.{idx}.conv.{j}.bias"))
            elif kind == "up_conv":
                W[f"{idx}.w"] = f16(pack3(pack_d2s_weights(f32(f"layers.{idx}.weight"))))
            else:
                # decode() returns layers(x) * 2 - 1: folded into the last conv in fp32
                w = f32(f"layers.{idx}.weight") * 2.0
                b = f32(f"layers.{idx}.bias") * 2.0 - 1.0
                W["out.w8"], W["out.b8"] = pack_conv_out8(f16(w.permute(0, 2, 3, 1)), f16(b))

    def _lower(self, h, w):
        return _TinyLowering(self, h, w)

    def _overflow_message(self, n):
        return (f"tiny VAE decode produced {n} non-finite pixels: the latents or the tiny VAE weights are not finite, "
                "or its fp16 activations overflow (the tiny decoder runs in fp16 only)")


class _TinyLowering:
    def __init__(self, vae: TinyVAEDecoderB200, h, w):
        Wt, dev, C = vae.w, vae.device, vae.channels
        f16 = dict(dtype=torch.float16, device=dev)
        P = self.prog = Program(vae.dev_index)
        ups = sum(1 for kind, _, _ in vae.layout if kind == "up_conv")
        Ho, Wo = h << ups, w << ups
        self.z_in = torch.zeros(1, 4, h, w, **f16)
        self.frame = torch.zeros(Ho, Wo, 3, dtype=torch.uint8, device=dev)
        bufs = [torch.empty(Ho * Wo, C, **f16) for _ in range(3)]
        xi, hh, ww = 0, h, w
        P.conv_in(self.z_in, Wt["in.w"], Wt["in.b"], C, bufs[xi][: h * w], _cabi.CONV_IN_TINY_VAE,
                  1.0 / vae.scaling_factor)
        for kind, idx, _ in vae.layout[1:]:
            M = hh * ww
            x = bufs[xi][:M]
            t1, t2 = (bufs[j][:M] for j in range(3) if j != xi)
            if kind == "block":
                P.gemm(x, Wt[f"{idx}.0.w"], C, 1, hh, ww, t1, taps=9, bias=Wt[f"{idx}.0.b"], relu=True)
                P.gemm(t1, Wt[f"{idx}.2.w"], C, 1, hh, ww, t2, taps=9, bias=Wt[f"{idx}.2.b"], relu=True)
                P.gemm(t2, Wt[f"{idx}.4.w"], C, 1, hh, ww, x, taps=9, bias=Wt[f"{idx}.4.b"], res=x, relu=True)
            elif kind == "up_conv":
                nx = (xi + 1) % 3
                P.gemm(x, Wt[f"{idx}.w"], 4 * C, 1, hh, ww, bufs[nx][: 4 * M], taps=9, depth_to_space=True)
                xi, hh, ww = nx, 2 * hh, 2 * ww
            else:
                img = torch.empty(1, 3, hh, ww, **f16)
                tmp = torch.empty(M, 8, **f16)
                P.conv_out_gemm(x, 1, hh, ww, C, Wt["out.w8"], Wt["out.b8"], 3, img, tmp)
                P.postprocess_u8(img, self.frame, vae.nonfinite)
        self._keep = bufs
        P.finalize()
