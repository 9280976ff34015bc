"""Host-side scheduler tables for the fused step kernel (lb_cfg_euler_step).

The reference calls ``pipe.scheduler.set_timesteps / scale_model_input / step``
(latentblending/diffusers_holder.py:42,53,247,330,356): diffusers 0.25.0
EulerDiscreteScheduler (SDXL base: 'leading' spacing, steps_offset 1) and
EulerAncestralDiscreteScheduler (SDXL-Turbo: 'trailing').  Here only the scalar
tables live on the host; the tensor arithmetic is in csrc/step.cu.

Scalars are produced with the same fp32 torch expressions the scheduler uses and
then rounded to fp16 where the reference's CUDA stack rounds them (a 0-dim fp32
CUDA tensor next to an fp16 tensor is cast to fp16 by PyTorch's binary kernels;
probed by tools/probe_scalar_semantics.py).
"""
import numpy as np
import torch


def _train_sigmas(num_train_timesteps=1000, beta_start=0.00085, beta_end=0.012):
    betas = torch.linspace(beta_start ** 0.5, beta_end ** 0.5, num_train_timesteps, dtype=torch.float32) ** 2
    acp = torch.cumprod(1.0 - betas, dim=0)
    return (((1 - acp) / acp) ** 0.5).numpy()


def _h(x):
    """fp32 0-dim tensor -> python float of its fp16 rounding."""
    return float(x.to(torch.float16))


class EulerTables:
    """kind: 'euler' (SDXL base) or 'euler_ancestral' (SDXL-Turbo)."""

    def __init__(self, kind="euler", timestep_spacing=None, steps_offset=None, num_train_timesteps=1000,
                 beta_start=0.00085, beta_end=0.012):
        assert kind in ("euler", "euler_ancestral")
        self.kind = kind
        self.ancestral = kind == "euler_ancestral"
        self.timestep_spacing = timestep_spacing or ("trailing" if self.ancestral else "leading")
        self.steps_offset = (0 if self.ancestral else 1) if steps_offset is None else steps_offset
        self.T = num_train_timesteps
        self.order = 1
        self._train = _train_sigmas(num_train_timesteps, beta_start, beta_end)
        self.num_inference_steps = None

    def set_timesteps(self, n, device=None):
        T = self.T
        if self.timestep_spacing == "leading":
            ts = (np.arange(0, n) * (T // n)).round()[::-1].copy().astype(np.float32) + self.steps_offset
        elif self.timestep_spacing == "trailing":
            ts = np.round(np.arange(T, 0, -T / n)).astype(np.float32) - 1
        elif self.timestep_spacing == "linspace":
            ts = np.linspace(0, T - 1, n, dtype=np.float32)[::-1].copy()
        else:
            raise ValueError(self.timestep_spacing)
        sig = np.interp(ts, np.arange(0, T), self._train)
        self.sigmas = torch.from_numpy(np.concatenate([sig, [0.0]]).astype(np.float32))
        self.timesteps = torch.from_numpy(ts.astype(np.float32))
        self.num_inference_steps = n
        # per-step scalars for the kernels
        self.step_scalars = []
        for i in range(n):
            s, s_next = self.sigmas[i], self.sigmas[i + 1]
            div = (s ** 2 + 1) ** 0.5
            if self.ancestral:
                s_up = (s_next ** 2 * (s ** 2 - s_next ** 2) / s ** 2) ** 0.5
                s_down = (s_next ** 2 - s_up ** 2) ** 0.5
                dt = s_down - s
            else:
                s_up = torch.tensor(0.0)
                dt = s_next - s
            self.step_scalars.append(dict(t=float(self.timesteps[i]), divisor=_h(div), sigma=_h(s), dt=_h(dt),
                                          sigma_up=_h(s_up)))

    @property
    def init_noise_sigma(self):
        smax = self.sigmas.max()
        if self.timestep_spacing in ("linspace", "trailing"):
            return smax
        return (smax ** 2 + 1) ** 0.5


def tables_from_diffusers_scheduler(scheduler):
    """EulerTables for a diffusers EulerDiscreteScheduler / EulerAncestralDiscreteScheduler instance (what
    AutoPipelineForText2Image loads for SDXL base / SDXL-Turbo), from its ``config``.  Other scheduler classes,
    beta schedules or prediction types are outside the reference's path (diffusers_holder.py:42,330,356) and raise."""
    cfg = scheduler.config
    name = type(scheduler).__name__
    kinds = {"EulerDiscreteScheduler": "euler", "EulerAncestralDiscreteScheduler": "euler_ancestral"}
    if name not in kinds:
        raise ValueError(f"unsupported scheduler {name}: the latentblending path uses the Euler / Euler-ancestral "
                         "schedulers SDXL base / SDXL-Turbo ship with")

    def get(k, default=None):
        return cfg[k] if k in cfg else getattr(cfg, k, default)
    if get("beta_schedule", "scaled_linear") != "scaled_linear" or get("prediction_type", "epsilon") != "epsilon":
        raise ValueError("only beta_schedule='scaled_linear' with prediction_type='epsilon' is implemented")
    if get("use_karras_sigmas", False) or get("interpolation_type", "linear") != "linear":
        raise ValueError("karras sigmas / log-linear interpolation are not implemented")
    return EulerTables(kinds[name], timestep_spacing=get("timestep_spacing"), steps_offset=get("steps_offset", 0),
                       num_train_timesteps=get("num_train_timesteps", 1000), beta_start=get("beta_start", 0.00085),
                       beta_end=get("beta_end", 0.012))
