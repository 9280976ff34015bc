"""DiffusersHolder: the denoise operator behind BlendingEngine, on liblb200.

Same attributes and methods the reference engine touches on ``self.dh``
(latentblending/diffusers_holder.py:20-366; the 14-item seam in SURVEY.md
section 8b): device, pipe, get_text_embedding, get_noise, run_diffusion_sd_xl,
latent2image, is_sdxl_turbo, set_dimensions, guidance_scale, set_negative_prompt,
set_num_inference_steps, height_img / width_img.

H100-first differences (results are the same, layout and launch structure are not):
  * a trajectory is ONE contiguous [N,4,h,w] fp16 slab in HBM; the returned
    ``list_latents_out`` holds views into it (None for i < idx_start), so the
    parental mix of a whole branch is a single batched lb_slerp_rows launch;
  * per step: (optional crossfeed slerp) -> lb_scale_model_input straight into the
    UNet program's input buffer -> lb_program_run (~930 pre-planned launches) ->
    lb_cfg_euler_step (CFG + Euler + trajectory store) -- no torch arithmetic;
  * the cross-attention K/V projections depend only on the conditioning and are
    computed once per branch, not once per step.
There is no CPU path: everything raises without CUDA + liblb200.so.
"""
import os

import numpy as np
import torch

from . import ops
from .taesd import TinyVAEDecoderB200
from .vae import VAEDecoderB200
from .unet import UNetB200


class DiffusersHolder:
    def __init__(self, pipe):
        self.negative_prompt = ""                 # reference defaults, diffusers_holder.py:23-25
        self.guidance_scale = 5.0
        self.num_inference_steps = 30
        from .pipe import adapt_pipe
        pipe = adapt_pipe(pipe)               # a diffusers StableDiffusionXLPipeline is wrapped (reference contract)
        self.pipe = pipe
        self.device = str(pipe._execution_device)
        if not torch.cuda.is_available() or not self.device.startswith("cuda"):
            raise RuntimeError("latentblending_b200 needs a CUDA device (no CPU fallback)")
        self.dtype = torch.float16
        self.is_sdxl_turbo = "turbo" in pipe._name_or_path
        self.pipe.scheduler.set_timesteps(self.num_inference_steps, device=self.device)
        s = pipe.unet_cfg.sample_size
        self.width_latent = self.height_latent = s
        self.width_img = self.height_img = s * pipe.vae_scale_factor
        self.unet = UNetB200(pipe.unet_cfg, pipe.unet_state_dict, self.device)
        self.vae = None
        self.set_vae_dtype(getattr(pipe, "vae_dtype", "fp16"))
        self.noise_fn = None          # tests: inject the ancestral-step noise, noise_fn(i, shape)
        self.noise_fn_multi = None    # same for run_diffusion_sd_xl_multi with k > 1: noise_fn_multi(job, i, shape)
        self._cond_key = None
        self.n_unet_calls = 0
        # multi-GPU CFG split (latentblending_b200/sharding.py): dict(group=<2-rank process group>, half=0|1) makes this
        # rank compute only the unconditional (0) or the text (1) half of every CFG batch; the halves' eps are
        # exchanged once per step (one all-gather of k x 128 KB over NVLink), then both ranks take the identical step.
        self.cfg_split = None
        self._eps_pair = {}
        # Two CUDA streams for the two CFG halves of a single branch (k = 1): the unconditional and the text half run
        # as two independent batch-1 programs that space-share the SMs, so one half's kernel ramp / drain overlaps the
        # other's main loop (every kernel is batch-invariant: identical eps).
        self.dual_stream = os.environ.get("LB_DUAL_STREAM", "1") != "0"
        self._dual = {}

    # ---- configuration --------------------------------------------------------------------
    def set_vae_dtype(self, vae_dtype):
        """Rebuild the VAE decoder with "fp16" or "bf16" storage (fp32 accumulation either way).  bf16 decodes VAEs
        whose activations overflow fp16, such as the stock SDXL VAE; a diffusers pipeline picks it from the VAE
        config's force_upcast.  The tiny autoencoder (``pipe.vae_kind == "tiny"``, AutoencoderTiny) is fp16 only."""
        from .pipe import VAE_DTYPES
        if vae_dtype not in VAE_DTYPES:
            raise ValueError(f"vae_dtype must be one of {sorted(VAE_DTYPES)} (got {vae_dtype!r})")
        p = self.pipe
        if getattr(p, "vae_kind", "kl") == "tiny":
            if vae_dtype != "fp16":
                raise ValueError(f"the tiny VAE decoder (AutoencoderTiny) runs in fp16 only (got {vae_dtype!r}): its "
                                 "activations stay within fp16's range, and there is no bf16 build of it")
            self.vae = TinyVAEDecoderB200(p.vae_state_dict, p.vae_config, p.vae_scaling_factor, self.device)
        else:
            self.vae = VAEDecoderB200(p.vae_state_dict, p.vae_channels, p.vae_scaling_factor, self.device,
                                      dtype=VAE_DTYPES[vae_dtype])
        self.vae_dtype = vae_dtype

    def set_num_inference_steps(self, num_inference_steps):
        self.num_inference_steps = num_inference_steps
        self.pipe.scheduler.set_timesteps(num_inference_steps, device=self.device)

    def set_dimensions(self, size_output):
        s = self.pipe.vae_scale_factor
        if size_output is None:
            width = height = self.pipe.unet_cfg.sample_size
        else:
            width, height = size_output
        self.width_img = int(round(width / s) * s)
        self.width_latent = int(self.width_img / s)
        self.height_img = int(round(height / s) * s)
        self.height_latent = int(self.height_img / s)

    def set_negative_prompt(self, negative_prompt):
        self.negative_prompt = [negative_prompt] if isinstance(negative_prompt, str) else negative_prompt
        if len(self.negative_prompt) > 1:
            self.negative_prompt = [self.negative_prompt[0]]

    # ---- inputs -----------------------------------------------------------------------------
    def get_text_embedding(self, prompt):
        do_cfg = self.guidance_scale > 1 and self.pipe.unet_cfg.time_cond_proj_dim is None
        return self.pipe.encode_prompt(prompt, negative_prompt=self.negative_prompt,
                                       do_classifier_free_guidance=do_cfg)

    def get_noise(self, seed=420):
        """randn([1,4,h,w], fp16, CUDA generator(seed)) * init_noise_sigma -- as pipe.prepare_latents does."""
        g = torch.Generator(device=self.device).manual_seed(int(seed))
        lat = torch.randn((1, self.pipe.unet_cfg.in_channels, self.height_latent, self.width_latent), generator=g,
                          device=self.device, dtype=torch.float16)
        return lat * self.pipe.scheduler.init_noise_sigma.to(device=self.device, dtype=torch.float16)

    @torch.no_grad()
    def decode_to_device(self, latents):
        """latents [1,4,h,w] -> uint8 [H,W,3] frame on the device."""
        return self.vae.decode_to_u8(latents.to(torch.float16))

    def check_decode_overflow(self):
        if self.vae.decodes_since_check:
            self.vae.check_overflow()

    @torch.no_grad()
    def latent2image(self, latents, output_type="pil"):
        assert output_type in ["pil", "np"]
        arr = self.decode_to_device(latents).cpu().numpy()
        if output_type == "np":
            return arr.astype(np.float32) / 255.0
        from PIL import Image
        return Image.fromarray(arr)

    # ---- the loop -----------------------------------------------------------------------------
    def prepare_mixing(self, mixing_coeffs, list_latents_mixing):
        N = self.num_inference_steps
        if type(mixing_coeffs) == float:
            list_mixing_coeffs = (1 + N) * [mixing_coeffs]
        elif type(mixing_coeffs) == list:
            assert len(mixing_coeffs) == N, f"len(mixing_coeffs) {len(mixing_coeffs)} != self.num_inference_steps {N}"
            list_mixing_coeffs = mixing_coeffs
        else:
            raise ValueError("mixing_coeffs should be float or list with len=num_inference_steps")
        if np.sum(list_mixing_coeffs) > 0:
            assert len(list_latents_mixing) == N, \
                f"len(list_latents_mixing) {len(list_latents_mixing)} != self.num_inference_steps {N}"
        return list_mixing_coeffs

    def run_diffusion(self, text_embeddings, latents_start, idx_start=0, list_latents_mixing=None, mixing_coeffs=0.0,
                      return_image=False):
        return self.run_diffusion_sd_xl(text_embeddings, latents_start, idx_start, list_latents_mixing, mixing_coeffs,
                                        return_image)

    @torch.no_grad()
    def run_diffusion_sd_xl(self, text_embeddings, latents_start, idx_start=0, list_latents_mixing=None,
                            mixing_coeffs=0.0, return_image=False):
        """latentblending/diffusers_holder.py:172-366 for ONE branch (the reference's signature)."""
        out = self.run_diffusion_sd_xl_multi([dict(text_embeddings=text_embeddings, latents_start=latents_start,
                                                   list_latents_mixing=list_latents_mixing,
                                                   mixing_coeffs=mixing_coeffs)], idx_start)[0]
        if return_image:
            return self.latent2image(out[-1])
        return out

    @torch.no_grad()
    def run_diffusion_sd_xl_multi(self, jobs, idx_start=0):
        """The denoise loop for k independent branches that share ``idx_start``, advanced in lockstep through ONE
        UNet forward of batch 2k per step (the 1280-channel levels of a batch-2 SDXL forward are launch- /
        latency-bound, so doubling M costs less than two forwards; tools/time_unet_batch.py measures it).  Per branch the arithmetic
        is exactly run_diffusion_sd_xl's: every kernel on the path is batch-invariant (tests/test_engine_gpu.py).

        jobs: dicts with text_embeddings (4-tuple), latents_start, list_latents_mixing, mixing_coeffs and optionally
        guidance_scale (default: self.guidance_scale) and noise_fn(step, shape) (ancestral noise source of this job).  ``list_latents_mixing`` may be ``("job", j)``: mix against
        the trajectory job j is producing in this very call (branch-1 crossfeed reads step i-1, which job j has
        already written).  Returns one len-N list per job (None for i < idx_start, else [1,4,h,w] fp16 views of that
        job's trajectory slab)."""
        sched = self.pipe.scheduler
        N = self.num_inference_steps
        sched.set_timesteps(N, device=self.device)
        cfg_on = self.guidance_scale > 1                       # pipe.do_classifier_free_guidance
        hw = self.pipe.default_sample_size * self.pipe.vae_scale_factor   # original/target size, :216-220
        tid = torch.tensor([[hw, hw, 0, 0, hw, hw]], dtype=torch.float16, device=self.device)
        split = self.cfg_split if cfg_on else None           # without CFG there is nothing to split
        Bj = 1 if (split is not None or not cfg_on) else 2      # UNet batch rows per job ON THIS RANK
        k = len(jobs)
        _, C, h, w = jobs[0]["latents_start"].shape
        ctxs, texts = [], []
        for job in jobs:
            pe, ne, pp, npool = job["text_embeddings"]
            if split is not None:
                ctxs.append(pe if split["half"] else ne)
                texts.append(pp if split["half"] else npool)
            elif cfg_on:
                ctxs += [ne, pe]
                texts += [npool, pp]
            else:
                ctxs.append(pe)
                texts.append(pp)
        dual = None
        if self.dual_stream and cfg_on and split is None and k == 1:
            dual = self._dual.get((h, w))
            if dual is None:
                xin = torch.zeros((2, C, h, w), dtype=torch.float16, device=self.device)
                dual = self._dual[(h, w)] = dict(
                    xin=xin, plans=(self.unet.plan(1, h, w, tag="cfg_uncond", x_in=xin[0:1]),
                                    self.unet.plan(1, h, w, tag="cfg_text", x_in=xin[1:2])),
                    streams=(torch.cuda.Stream(device=self.device), torch.cuda.Stream(device=self.device)),
                    fork=torch.cuda.Event(), done=(torch.cuda.Event(), torch.cuda.Event()))
            for pl, c_, t_ in zip(dual["plans"], ctxs, texts):        # ctxs / texts = [uncond, text] of the one job
                pl.ctx.copy_(c_.reshape(pl.ctx.shape))
                pl.text.copy_(t_)
                pl.tids.copy_(tid)
                pl.prog_ctx.run()
        plan = dual["plans"][0] if dual is not None else self.unet.plan(Bj * k, h, w)
        if dual is None:
            plan.ctx.copy_(torch.cat(ctxs, dim=0).reshape(plan.ctx.shape))
            plan.text.copy_(torch.cat(texts, dim=0))
            plan.tids.copy_(tid.expand(Bj * k, -1))
        x_in = dual["xin"] if dual is not None else plan.x_in
        eps_pair = None
        if split is not None:
            key = (k, C, h, w)
            if key not in self._eps_pair:
                self._eps_pair[key] = torch.empty((2, k, C, h, w), dtype=torch.float16, device=self.device)
            eps_pair = self._eps_pair[key]
        if dual is None:
            plan.prog_ctx.run()                                # cross-attention K/V: once per conditioning
        n = C * h * w
        outs = [[None] * N for _ in jobs]
        trajs = [torch.empty((N, C, h, w), dtype=torch.float16, device=self.device) for _ in jobs]
        coeffs, mixing, guidance, latents = [], [], [], []
        for job in jobs:
            m = job.get("list_latents_mixing")
            if isinstance(m, tuple) and m[0] == "job":
                m = outs[m[1]]
            coeffs.append(self.prepare_mixing(job.get("mixing_coeffs", 0.0), m))
            mixing.append(m)
            guidance.append(job.get("guidance_scale", self.guidance_scale))
            latents.append(None)
        # Ancestral schedulers draw one noise tensor per step from the global RNG.  The reference (and the sequential
        # path) runs trajectory 1 to the end before trajectory 2, so under torch.manual_seed the draws are ordered
        # job-major; the lockstep loop consumes them step-major.  Pre-draw them in the reference's order.
        drawn = None
        if (sched.ancestral and k > 1 and self.noise_fn_multi is None and self.noise_fn is None
                and all(job.get("noise_fn") is None for job in jobs)):
            drawn = [[torch.randn((1, C, h, w), device=self.device, dtype=torch.float16) for _ in range(idx_start, N)]
                     for _ in jobs]
        scaled = [False] * k          # the previous step's lb_cfg_euler_step already wrote this job's model input
        for i in range(N):
            if i < idx_start:
                continue
            sc = sched.step_scalars[i]
            for j, job in enumerate(jobs):
                if i == idx_start:
                    latents[j] = job["latents_start"].clone().contiguous()
                if i > 0 and coeffs[j][i] > 0:
                    latents[j] = ops.slerp_rows(latents[j].view(1, n), mixing[j][i - 1].reshape(1, n),
                                                float(coeffs[j][i])).view(1, C, h, w)
                    scaled[j] = False
                if not scaled[j]:
                    ops.scale_model_input(latents[j], Bj, sc["divisor"], out=x_in[j * Bj:(j + 1) * Bj])
            if dual is None:
                plan.prog_step.run(sc["t"])
            else:
                main = torch.cuda.current_stream()
                dual["fork"].record(main)
                for pl, st, ev in zip(dual["plans"], dual["streams"], dual["done"]):
                    st.wait_event(dual["fork"])
                    with torch.cuda.stream(st):
                        pl.prog_step.run(sc["t"])
                        ev.record(st)
                for ev in dual["done"]:
                    main.wait_event(ev)
            self.n_unet_calls += 1
            if eps_pair is not None:
                import torch.distributed as dist
                dist.all_gather_into_tensor(eps_pair, plan.eps, group=split["group"])   # [uncond | text] x k jobs
            for j in range(k):
                noise = None
                if sched.ancestral:
                    if jobs[j].get("noise_fn") is not None:        # per-job source (BlendingEngine.deterministic_noise)
                        noise = jobs[j]["noise_fn"](i, latents[j].shape).to(device=self.device,
                                                                            dtype=torch.float16).contiguous()
                    elif k > 1 and self.noise_fn_multi is not None:
                        noise = self.noise_fn_multi(j, i, latents[j].shape).to(device=self.device,
                                                                               dtype=torch.float16).contiguous()
                    elif self.noise_fn is not None:
                        noise = self.noise_fn(i, latents[j].shape).to(device=self.device,
                                                                      dtype=torch.float16).contiguous()
                    elif drawn is not None:
                        noise = drawn[j][i - idx_start]
                    else:
                        noise = torch.randn(latents[j].shape, device=self.device, dtype=torch.float16)
                new = trajs[j][i:i + 1]
                # fold the NEXT step's scale_model_input (+ CFG duplicate) into this launch unless a crossfeed mix
                # sits in between (diffusers_holder.py:322-330 order: mix, then scale)
                fuse = i + 1 < N and not (coeffs[j][i + 1] > 0)
                if dual is not None:
                    e_u, e_t = dual["plans"][0].eps, dual["plans"][1].eps
                elif eps_pair is not None:
                    e_u, e_t = eps_pair[0, j], eps_pair[1, j]
                else:
                    e_u, e_t = plan.eps[j * Bj:(j + 1) * Bj], None
                ops.cfg_euler_step(latents[j], e_u, guidance[j], sc["sigma"], sc["dt"], sc["sigma_up"], noise=noise,
                                   out=new, eps_text=e_t,
                                   scaled_next=x_in[j * Bj:(j + 1) * Bj] if fuse else None,
                                   next_divisor=sched.step_scalars[i + 1]["divisor"] if fuse else 0.0)
                scaled[j] = fuse
                latents[j] = new
                outs[j][i] = new
        return outs
