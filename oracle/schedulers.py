"""Oracle: Euler / Euler-ancestral schedulers (test infrastructure).

The reference calls ``pipe.scheduler.set_timesteps / scale_model_input / step``
(latentblending/diffusers_holder.py:42,53,247,330,356) and, via
``pipe.prepare_latents``, ``init_noise_sigma`` (diffusers_holder.py:100-109).
The code behind those calls is diffusers==0.25.0 (requirements.txt:3),
``schedulers/scheduling_euler_discrete.py`` and
``scheduling_euler_ancestral_discrete.py`` -- NOT vendored in /root/reference.
This file restates their published algorithm (k-diffusion Euler, eps-prediction,
scaled-linear betas 0.00085 -> 0.012 over 1000 train steps).

Pinned by the known-answer vectors in SURVEY.md appendix C
(tests/test_oracle_schedulers.py): sigma_max 14.6146 / sigma_min 0.0292.

All tensor arithmetic is written as individual torch ops on purpose: with fp16
latents every op rounds to fp16 exactly like the reference stack does, which is
what the fused CUDA step kernel has to reproduce bit for bit.

Scalar semantics (probed by tools/probe_scalar_semantics.py): on the
reference's real stack the sigmas live on the CUDA device, and PyTorch's CUDA
binary kernels cast an fp32 0-dim *CUDA tensor* operand to the fp16 common
dtype before the fp32 op-math (Python scalars such as guidance_scale stay fp32).
PyTorch's CPU kernels do this only for some operand orders, so the oracle makes
the cast explicit (``_s``) to be device-independent and faithful to CUDA.
"""
import numpy as np
import torch


def _s(scalar, like):
    """0-dim fp32 scheduler scalar as the CUDA stack sees it next to ``like``."""
    return scalar.to(like.dtype)


def _train_sigmas(num_train_timesteps=1000, beta_start=0.00085, beta_end=0.012):
    betas = torch.linspace(beta_start ** 0.5, beta_end ** 0.5, num_train_timesteps, dtype=torch.float32) ** 2
    alphas_cumprod = torch.cumprod(1.0 - betas, dim=0)
    return (((1 - alphas_cumprod) / alphas_cumprod) ** 0.5).numpy()


class EulerDiscrete:
    """SDXL-base scheduler: timestep_spacing='leading', steps_offset=1."""
    order = 1
    ancestral = False

    def __init__(self, timestep_spacing="leading", steps_offset=1, num_train_timesteps=1000):
        self.timestep_spacing = timestep_spacing
        self.steps_offset = steps_offset
        self.num_train_timesteps = num_train_timesteps
        self._sig_train = _train_sigmas(num_train_timesteps)
        self.sigmas = torch.from_numpy(np.concatenate([self._sig_train[::-1], [0.0]]).astype(np.float32))
        self.timesteps = None

    def set_timesteps(self, num_inference_steps, device=None):
        n, T = num_inference_steps, self.num_train_timesteps
        if self.timestep_spacing == "leading":
            ts = (np.arange(0, n) * (T // n)).round()[::-1].copy().astype(np.float32) + self.steps_offset
        elif self.timestep_spacing == "trailing":
            ts = (np.arange(T, 0, -T / n)).round().astype(np.float32) - 1
        elif self.timestep_spacing == "linspace":
            ts = np.linspace(0, T - 1, n, dtype=np.float32)[::-1].copy()
        else:
            raise ValueError(self.timestep_spacing)
        sig = np.interp(ts, np.arange(0, T), self._sig_train)
        self.sigmas = torch.from_numpy(np.concatenate([sig, [0.0]]).astype(np.float32))
        self.timesteps = torch.from_numpy(ts.astype(np.float32))
        self.num_inference_steps = n

    @property
    def init_noise_sigma(self):
        smax = self.sigmas.max()
        if self.timestep_spacing in ("linspace", "trailing"):
            return smax
        return (smax ** 2 + 1) ** 0.5

    def scale_model_input(self, sample, i):
        sigma = self.sigmas[i]
        return sample / _s((sigma ** 2 + 1) ** 0.5, sample)

    def step(self, model_output, i, sample, noise=None):
        sigma = self.sigmas[i]
        pred_original = sample - _s(sigma, sample) * model_output
        derivative = (sample - pred_original) / _s(sigma, sample)
        dt = self.sigmas[i + 1] - sigma
        return sample + derivative * _s(dt, sample)


class EulerAncestralDiscrete(EulerDiscrete):
    """SDXL-Turbo scheduler: timestep_spacing='trailing'; adds randn * sigma_up."""
    ancestral = True

    def __init__(self, timestep_spacing="trailing", steps_offset=0, num_train_timesteps=1000):
        super().__init__(timestep_spacing, steps_offset, num_train_timesteps)

    def set_timesteps(self, num_inference_steps, device=None):
        n, T = num_inference_steps, self.num_train_timesteps
        if self.timestep_spacing == "trailing":
            ts = np.round(np.arange(T, 0, -T / n)).astype(np.int64) - 1
        elif self.timestep_spacing == "leading":
            ts = (np.arange(0, n) * (T // n)).round()[::-1].copy().astype(np.int64) + self.steps_offset
        else:
            ts = np.linspace(0, T - 1, n, dtype=np.float32)[::-1].copy()
        sig = np.interp(ts, np.arange(0, T), self._sig_train)
        self.sigmas = torch.from_numpy(np.concatenate([sig, [0.0]]).astype(np.float32))
        self.timesteps = torch.from_numpy(np.asarray(ts, dtype=np.float32))
        self.num_inference_steps = n

    def sigma_up_down(self, i):
        s_from, s_to = self.sigmas[i], self.sigmas[i + 1]
        s_up = (s_to ** 2 * (s_from ** 2 - s_to ** 2) / s_from ** 2) ** 0.5
        s_down = (s_to ** 2 - s_up ** 2) ** 0.5
        return s_up, s_down

    def step(self, model_output, i, sample, noise=None):
        """``noise`` must be injected (the reference draws it from the global
        generator because generator=None, diffusers_holder.py:192,255,356)."""
        sigma = self.sigmas[i]
        pred_original = sample - _s(sigma, sample) * model_output
        s_up, s_down = self.sigma_up_down(i)
        derivative = (sample - pred_original) / _s(sigma, sample)
        dt = s_down - sigma
        prev = sample + derivative * _s(dt, sample)
        if noise is None:
            noise = torch.zeros_like(model_output)
        return prev + noise * _s(s_up, sample)
