"""BlendingEngine: drop-in for latentblending.BlendingEngine on the H100 backend.

Public surface, defaults and quirks follow latentblending/blending_engine.py
(:20-96 constructor, :120-293 setters, :295-365 run_transition, :370-465
compute_latents1/2/_mix, :467-529 get_time_based_branching, :531-588 tree
placement, :643-654 mixed conditioning, :669-742 writers / swap_forward).

What is different underneath (H100-first, same results):
  * the parental mix of a branch (30 per-step slerps in the reference, :442-450)
    is one batched lb_slerp_rows launch over the parents' contiguous trajectory
    slabs (rows where either parent has no latent are simply not computed);
  * decoded frames stay on the device for the LPIPS placement metric (the
    reference round-trips every frame through PIL and back, :575-579, :750-755);
    PIL images are produced once per frame for the API;
  * timing estimates use CUDA events (the reference's time.time() pairs are not
    synchronised, :110-117).
"""
import os
import time
import warnings
from typing import List, Optional

import numpy as np
import torch
from PIL import Image

from . import ops
from .diffusers_holder import DiffusersHolder
from .lpips import LPIPSAlexB200, lpips_random_state_dict
from .utils import add_frames_linear_interp, interpolate_linear

warnings.filterwarnings('ignore')
torch.set_grad_enabled(False)


class BlendingEngine():
    def __init__(self, pipe, do_compile: bool = False, guidance_scale_mid_damper: float = 0.5,
                 mid_compression_scaler: float = 1.2, *, holder=None, similarity_fn=None, run_benchmark=True):
        assert guidance_scale_mid_damper > 0 and guidance_scale_mid_damper <= 1.0, \
            f"guidance_scale_mid_damper neees to be in interval (0,1], you provided {guidance_scale_mid_damper}"
        if do_compile:
            raise ValueError("do_compile selects the reference's stable-fast/Triton path; this backend is already "
                             "compiled CUDA (sm_90a) and has no such option")
        self.dh = holder if holder is not None else DiffusersHolder(pipe)
        self.device = self.dh.device
        self.set_dimensions()
        self.guidance_scale_mid_damper = guidance_scale_mid_damper
        self.mid_compression_scaler = mid_compression_scaler
        self.seed1 = 0
        self.seed2 = 0
        self.prompt1 = ""
        self.prompt2 = ""
        self.tree_latents = [None, None]
        self.tree_fracts = None
        self.idx_injection = []
        self.tree_status = None
        self.tree_final_imgs = []
        self.text_embedding1 = None
        self.text_embedding2 = None
        self.image1_lowres = None
        self.image2_lowres = None
        self.negative_prompt = None
        self.set_guidance_scale()
        self.multi_transition_img_first = None
        self.multi_transition_img_last = None
        self.dt_unet_step = 0
        self.dt_vae = 0
        self._similarity_fn = similarity_fn
        self.output_device_frames = False     # True: run_transition returns uint8 device frames, no D2H / PIL
        self.batch_outer_pair = True          # the two outer trajectories share batch-4 UNet forwards (same results)
        # single-GPU speculation width: candidate branches of a level advanced in lockstep through ONE batched UNet
        # forward (sharding.run_level_local).  None = by model: SDXL-Turbo 512^2 (weight-bandwidth / launch bound, a
        # batch-4 forward costs about one batch-1 forward) -> 4; SDXL base 1024^2 -> 2 while >= 78 % of the second
        # candidates end up in the tree -- the running hit rate is tracked and the width drops to 1 below that.
        self.speculative_batch = None
        self._spec_hits = [0, 0]            # second-or-later candidates: [used, computed], over the engine's lifetime
        # ancestral-scheduler noise per (seeds, branch position, step) from its own generator instead of the global
        # RNG: results then do not depend on the order branches are computed in (speculation, multi-GPU sharding)
        self.deterministic_noise = False
        self.d2h_bytes = 0                    # bytes copied device->host for returned frames (bench e2e)
        self.lpips = None
        self._pending_timing = None
        if similarity_fn is None:
            pipe = getattr(self.dh, "pipe", pipe)       # the adapted pipe (a diffusers pipeline is wrapped by the holder)
            sd = getattr(pipe, "lpips_state_dict", None)
            if sd is None:
                # Random AlexNet weights only RANK gaps of a synthetic pipe; with real UNet / VAE weights they would
                # silently steer branch placement away from the reference's LPIPS (blending_engine.py:74-76).
                if not getattr(pipe, "is_synthetic", False):
                    raise ValueError(
                        "pipe has no lpips_state_dict: export the lpips==0.1.4 AlexNet weights (see INTEGRATION.md, "
                        "'LPIPS weights') and pass them as pipe.lpips_state_dict, or supply similarity_fn=...")
                sd = lpips_random_state_dict(2, self.device)
            self.lpips = LPIPSAlexB200(sd, self.device)
        self.set_prompt1("")
        self.set_prompt2("")
        self.set_branch1_crossfeed()
        self.set_parental_crossfeed()
        self.set_num_inference_steps()
        if run_benchmark:
            self.benchmark_speed()
        else:
            self.dt_unet_step, self.dt_vae = 0.05, 0.1
        self.set_branching()

    # ---- timing -------------------------------------------------------------------------------
    def benchmark_speed(self):
        """dt_unet_step / dt_vae for the time-based branching planner (blending_engine.py:100-118),
        measured with a device synchronisation on both sides."""
        text_embeddings = self.dh.get_text_embedding("test")
        latents_start = self.dh.get_noise(np.random.randint(111111))
        N = self.num_inference_steps
        self.dh.run_diffusion_sd_xl(text_embeddings, latents_start, idx_start=N - 1)      # warm-up
        torch.cuda.synchronize()
        t0 = time.time()
        list_latents = self.dh.run_diffusion_sd_xl(text_embeddings, latents_start, idx_start=N - 1)
        torch.cuda.synchronize()
        self.dt_unet_step = time.time() - t0
        self._decode_frame(list_latents[-1])
        torch.cuda.synchronize()
        t0 = time.time()
        self._decode_frame(list_latents[-1])
        torch.cuda.synchronize()
        self.dt_vae = time.time() - t0

    # ---- setters (defaults keyed on the model like the reference) ------------------------------
    def set_dimensions(self, size_output=None):
        if size_output is None:
            size_output = (512, 512) if self.dh.is_sdxl_turbo else (1024, 1024)
        self.dh.set_dimensions(size_output)

    def set_guidance_scale(self, guidance_scale=None):
        if guidance_scale is None:
            guidance_scale = 0.0 if self.dh.is_sdxl_turbo else 4.0
        self.guidance_scale_base = guidance_scale
        self.guidance_scale = guidance_scale
        self.dh.guidance_scale = guidance_scale

    def set_negative_prompt(self, negative_prompt):
        self.negative_prompt = negative_prompt
        self.dh.set_negative_prompt(negative_prompt)

    def set_guidance_mid_dampening(self, fract_mixing):
        mid_factor = 1 - np.abs(fract_mixing - 0.5) / 0.5
        max_guidance_reduction = self.guidance_scale_base * (1 - self.guidance_scale_mid_damper) - 1
        guidance_scale_effective = self.guidance_scale_base - max_guidance_reduction * mid_factor
        self.guidance_scale = guidance_scale_effective
        self.dh.guidance_scale = guidance_scale_effective

    def set_branch1_crossfeed(self, crossfeed_power=0, crossfeed_range=0, crossfeed_decay=0):
        self.branch1_crossfeed_power = np.clip(crossfeed_power, 0, 1)
        self.branch1_crossfeed_range = np.clip(crossfeed_range, 0, 1)
        self.branch1_crossfeed_decay = np.clip(crossfeed_decay, 0, 1)

    def set_parental_crossfeed(self, crossfeed_power=None, crossfeed_range=None, crossfeed_decay=None):
        if self.dh.is_sdxl_turbo:
            crossfeed_power = 1.0 if crossfeed_power is None else crossfeed_power
            crossfeed_range = 1.0 if crossfeed_range is None else crossfeed_range
            crossfeed_decay = 1.0 if crossfeed_decay is None else crossfeed_decay
        else:
            # the reference overrides whatever the caller passed for the base model (blending_engine.py:200-203)
            crossfeed_power, crossfeed_range, crossfeed_decay = 0.3, 0.6, 0.9
        self.parental_crossfeed_power = np.clip(crossfeed_power, 0, 1)
        self.parental_crossfeed_range = np.clip(crossfeed_range, 0, 1)
        self.parental_crossfeed_decay = np.clip(crossfeed_decay, 0, 1)

    def set_prompt1(self, prompt: str):
        prompt = prompt.replace("_", " ")
        self.prompt1 = prompt
        self.text_embedding1 = self.get_text_embeddings(self.prompt1)

    def set_prompt2(self, prompt: str):
        prompt = prompt.replace("_", " ")
        self.prompt2 = prompt
        self.text_embedding2 = self.get_text_embeddings(self.prompt2)

    def set_image1(self, image):
        self.image1_lowres = image

    def set_image2(self, image):
        self.image2_lowres = image

    def set_num_inference_steps(self, num_inference_steps=None):
        if num_inference_steps is None:
            num_inference_steps = 4 if self.dh.is_sdxl_turbo else 30
        self.num_inference_steps = num_inference_steps
        self.dh.set_num_inference_steps(num_inference_steps)

    def set_branching(self, depth_strength=None, t_compute_max_allowed=None, nmb_max_branches=None):
        self._resolve_timing()
        if self.dh.is_sdxl_turbo:
            assert t_compute_max_allowed is None, "time-based branching not supported for SDXL Turbo"
            idx_inject = int(round(self.num_inference_steps * depth_strength)) if depth_strength is not None else 2
            if nmb_max_branches is None:
                nmb_max_branches = 10
            self.list_idx_injection = [idx_inject]
            self.list_nmb_stems = [nmb_max_branches]
        else:
            if depth_strength is None:
                depth_strength = 0.5
            if t_compute_max_allowed is None and nmb_max_branches is None:
                t_compute_max_allowed = 20
            elif t_compute_max_allowed is not None and nmb_max_branches is not None:
                raise ValueError("Either specify t_compute_max_allowed or nmb_max_branches")
            self.list_idx_injection, self.list_nmb_stems = self.get_time_based_branching(
                depth_strength, t_compute_max_allowed, nmb_max_branches)

    # ---- the transition ---------------------------------------------------------------------------
    def run_transition(self, recycle_img1: Optional[bool] = False, recycle_img2: Optional[bool] = False,
                       fixed_seeds: Optional[List[int]] = None):
        assert self.text_embedding1 is not None, 'Set the first text embedding with .set_prompt1(...) before'
        assert self.text_embedding2 is not None, 'Set the second text embedding with .set_prompt2(...) before'
        if fixed_seeds is not None:
            if isinstance(fixed_seeds, str) and fixed_seeds == 'randomize':
                fixed_seeds = list(np.random.randint(0, 1000000, 2).astype(np.int32))
            else:
                assert len(fixed_seeds) == 2, "Supply a list with len = 2"
            self.seed1 = fixed_seeds[0]
            self.seed2 = fixed_seeds[1]
        N = self.num_inference_steps
        have1 = self.tree_latents[0] is not None and len(self.tree_latents[0]) == N
        have2 = self.tree_latents[-1] is not None and len(self.tree_latents[-1]) == N
        rank, world = self._dist()
        if world > 1:
            return self._run_transition_sharded(recycle_img1 and have1, recycle_img2 and have2, rank, world)
        if (self.batch_outer_pair and hasattr(self.dh, "run_diffusion_sd_xl_multi")
                and not (recycle_img1 and have1) and not (recycle_img2 and have2)):
            list_latents1, list_latents2 = self._compute_latents_pair()
        else:
            list_latents1 = self.tree_latents[0] if (recycle_img1 and have1) else self.compute_latents1()
            list_latents2 = self.tree_latents[-1] if (recycle_img2 and have2) else self.compute_latents2()

        self.tree_latents = [list_latents1, list_latents2]
        self.tree_fracts = [0.0, 1.0]
        self._tree_frames = [self._decode_frame(list_latents1[-1]), self._decode_frame(list_latents2[-1])]
        self.tree_idx_injection = [0, 0]
        # the reference seeds this list with a bound method (blending_engine.py:349); only its length
        # matters for the first argmax, so a placeholder keeps the same behaviour
        self.tree_similarities = [None]

        self.spec_stats = dict(rounds=0, computed=0, used=0)
        for s_idx in range(len(self.list_idx_injection)):
            nmb_stems = int(self.list_nmb_stems[s_idx])
            idx_injection = int(self.list_idx_injection[s_idx])
            width = self._speculation_width()
            if width > 1 and nmb_stems > 1:
                from .sharding import run_level_local
                before = dict(self.spec_stats)
                # the half-gap similarity estimate (split_ratio) keeps adapting across levels and transitions, like the
                # sharder's: it orders the speculative candidates
                self._split_ratio = run_level_local(
                    self, idx_injection, nmb_stems, self._compute_candidates, self.get_lpips_similarity, width,
                    on_insert=self.set_guidance_mid_dampening, stats=self.spec_stats,
                    split_ratio=getattr(self, "_split_ratio", 0.6))
                rounds = self.spec_stats["rounds"] - before["rounds"]
                # every round's first candidate is the reference's own next pick; the others are the speculation
                self._spec_hits[0] += (self.spec_stats["used"] - before["used"]) - rounds
                self._spec_hits[1] += (self.spec_stats["computed"] - before["computed"]) - rounds
                continue
            for _ in range(nmb_stems):
                fract_mixing, b_parent1, b_parent2 = self.get_mixing_parameters(idx_injection)
                self.set_guidance_mid_dampening(fract_mixing)
                list_latents = self.compute_latents_mix(fract_mixing, b_parent1, b_parent2, idx_injection)
                self.insert_into_tree(fract_mixing, idx_injection, list_latents)
        return self._finish_transition()

    def _speculation_width(self):
        if self._similarity_fn is not None or not hasattr(self.dh, "run_diffusion_sd_xl_multi"):
            return 1
        if self.speculative_batch is not None:
            return max(1, int(self.speculative_batch))
        if self.dh.is_sdxl_turbo:
            return 4
        used, computed = self._spec_hits
        return 2 if (computed < 4 or used >= 0.78 * computed) else 1

    def _guidance_for(self, fract_mixing):
        """set_guidance_mid_dampening's value without touching the engine / holder state."""
        mid_factor = 1 - np.abs(fract_mixing - 0.5) / 0.5
        return self.guidance_scale_base - (self.guidance_scale_base * (1 - self.guidance_scale_mid_damper) - 1) * mid_factor

    def _parental_coeffs(self, idx_injection):
        """blending_engine.py:452-457."""
        N = self.num_inference_steps
        idx_mixing_stop = int(round(N * self.parental_crossfeed_range))
        mixing_coeffs = idx_injection * [self.parental_crossfeed_power]
        nmb_mixing = idx_mixing_stop - idx_injection
        if nmb_mixing > 0:
            mixing_coeffs.extend(list(np.linspace(self.parental_crossfeed_power,
                                                  self.parental_crossfeed_power * self.parental_crossfeed_decay,
                                                  nmb_mixing)))
        mixing_coeffs.extend((N - len(mixing_coeffs)) * [0])
        return mixing_coeffs

    def _compute_candidates(self, cands, idx_injection):
        """compute_latents_mix for several candidate branches of one level in ONE lockstep batch."""
        self.dh.set_num_inference_steps(self.num_inference_steps)
        jobs = []
        for fract, p1, p2 in cands:
            f_par = (fract - self.tree_fracts[p1]) / (self.tree_fracts[p2] - self.tree_fracts[p1])
            mix = self._parental_mix(self.tree_latents[p1], self.tree_latents[p2], f_par)
            jobs.append(dict(text_embeddings=self.get_mixed_conditioning(fract)[0], latents_start=mix[idx_injection - 1],
                             list_latents_mixing=mix, mixing_coeffs=self._parental_coeffs(idx_injection),
                             guidance_scale=self._guidance_for(fract), noise_fn=self._noise_source(fract)))
        trajs = self.dh.run_diffusion_sd_xl_multi(jobs, idx_start=idx_injection)
        return [(t, self._decode_frame(t[-1])) for t in trajs]

    def _noise_source(self, key):
        """noise_fn(step, shape) of the branch at position ``key`` (None: the scheduler's default global-RNG draws)."""
        if not self.deterministic_noise:
            return None
        sched = getattr(getattr(self.dh, "pipe", None), "scheduler", None)
        if not getattr(sched, "ancestral", False):
            return None
        return lambda step, shape: self._noise_for(key, step, shape)

    def _noise_for(self, key, step, shape):
        """Ancestral noise of (branch position ``key``, step) from a generator seeded by (seed1, seed2, key, step)."""
        import struct
        import zlib
        seed = zlib.crc32(struct.pack("<qqdq", int(self.seed1), int(self.seed2), float(key), int(step))) & 0x7FFFFFFF
        g = torch.Generator(device=self.device).manual_seed(seed)
        return torch.randn(shape, generator=g, device=self.device, dtype=torch.float16)

    def _finish_transition(self):
        if hasattr(self.dh, "check_decode_overflow"):
            self.dh.check_decode_overflow()       # fp16 VAE: raise instead of returning black / garbage frames
        if self.output_device_frames:
            self.tree_final_imgs = list(self._tree_frames)
        else:
            self.tree_final_imgs = [self._frame_to_pil(f) for f in self._tree_frames]
        return self.tree_final_imgs

    # ---- multi-GPU: branches of a level sharded over the ranks (latentblending_b200/sharding.py) -----------
    @staticmethod
    def _dist():
        import torch.distributed as dist
        if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
            return dist.get_rank(), dist.get_world_size()
        return 0, 1

    @property
    def frames(self):
        return self._tree_frames

    def _bcast_trajectory(self, traj, src):
        """Make a full trajectory (list of N latents) computed on rank ``src`` available on every rank."""
        import torch.distributed as dist
        N = self.num_inference_steps
        lat_shape = (1, 4, self.dh.height_latent, self.dh.width_latent)
        n = int(np.prod(lat_shape))
        if traj is not None:
            slab = torch.stack([t.reshape(n) for t in traj], 0).contiguous()
        else:
            slab = torch.empty((N, n), dtype=torch.float16, device=self.device)
        dist.broadcast(slab, src=src)
        return [slab[i].view(lat_shape) for i in range(N)]

    def _run_transition_sharded(self, reuse1, reuse2, rank, world):
        import torch.distributed as dist
        from .sharding import LevelSharder
        N = self.num_inference_steps
        seeds = [int(self.seed1), int(self.seed2)]
        dist.broadcast_object_list(seeds, src=0)            # 'randomize' draws must agree across ranks
        self.seed1, self.seed2 = seeds
        crossfed = self.branch1_crossfeed_power > 0.0
        cfg_on = self.dh.guidance_scale > 1
        sharder = getattr(self, "_sharder", None)
        if sharder is None or sharder.world != world:
            sharder = self._sharder = LevelSharder(rank, world, device=self.device, cfg_pairs=cfg_on)
        sharder.cfg_pairs = cfg_on and world >= 2
        sharder.stats = dict(rounds=0, computed=0, used=0, paired_rounds=0)
        # ---- outer trajectories.  Owners: trajectory 1 -> rank 0, trajectory 2 -> rank 1 (both on rank 0 in one
        # lockstep batch when branch-1 crossfeed couples them).  From 4 ranks up (CFG on) each owner becomes a PAIR:
        # ranks (0,1) / (2,3) split the CFG halves of their trajectory (batch-1 forwards + one eps exchange per step).
        # On 2-3 ranks a pair is used when only one trajectory has to be computed (the other is recycled) or when
        # crossfeed forces both onto the same ranks anyway.
        n_outer = int(not reuse1) + int(not reuse2)
        paired = cfg_on and (world >= 4 or (world >= 2 and n_outer >= 1 and (n_outer == 1 or crossfed)))
        split = dict(group=sharder.pair_group(), half=rank % 2) if paired else None
        t1 = self.tree_latents[0] if reuse1 else None
        t2 = self.tree_latents[-1] if reuse2 else None
        own1 = (0, 1) if paired else (0,)
        # crossfeed: trajectory 2 reads trajectory 1, so it runs where trajectory 1 lives
        own2 = own1 if (crossfed or (paired and world < 4)) else ((2, 3) if paired else (1,))
        mine1 = mine2 = None
        self.dh.cfg_split = split
        try:
            if crossfed and not reuse1 and not reuse2:
                if rank in own1:
                    mine1, mine2 = self._compute_latents_pair()          # lockstep: step i of 2 reads step i-1 of 1
            else:
                if not reuse1 and rank in own1:
                    mine1 = self.compute_latents1()
                if not reuse2 and rank in own2:
                    mine2 = self.compute_latents2()                       # crossfed here implies reuse1: every rank has t1
        finally:
            self.dh.cfg_split = None
        if not reuse1:
            t1 = self._bcast_trajectory(mine1, own1[0])
        if not reuse2:
            t2 = self._bcast_trajectory(mine2, own2[0])
        self.tree_latents = [t1, t2]
        self.tree_fracts = [0.0, 1.0]
        self._tree_frames = [self._decode_frame(t1[-1]), self._decode_frame(t2[-1])]
        self.tree_idx_injection = [0, 0]
        self.tree_similarities = [None]

        def compute(fract, p1, p2, idx_injection, cfg_split=None):
            self.set_guidance_mid_dampening(fract)
            self.dh.cfg_split = cfg_split
            try:
                traj = self.compute_latents_mix(fract, p1, p2, idx_injection)
            finally:
                self.dh.cfg_split = None
            return traj, self._decode_frame(traj[-1])

        for s_idx in range(len(self.list_idx_injection)):
            # every rank evaluates the (deterministic) similarities on the replicated frames and replays
            # set_guidance_mid_dampening for every INSERTED branch in insertion order, so all ranks leave the
            # transition with the sequential path's tree AND guidance state (the latter steers the next transition's
            # outer trajectories and the do_cfg decision of set_prompt, blending_engine.py:147,164)
            sharder.run_level(self, int(self.list_idx_injection[s_idx]), int(self.list_nmb_stems[s_idx]), compute,
                              self.get_lpips_similarity, N, on_insert=self.set_guidance_mid_dampening)
        self.shard_stats = dict(sharder.stats)
        return self._finish_transition()

    def compute_latents1(self, return_image=False):
        list_conditionings = self.get_mixed_conditioning(0)
        ev0, ev1 = self._events()
        latents_start = self.get_noise(self.seed1)
        list_latents1 = self.run_diffusion(list_conditionings, latents_start=latents_start, idx_start=0, noise_key=0.0)
        self._finish_timing(ev0, ev1)
        self.tree_latents[0] = list_latents1
        if return_image:
            return self.dh.latent2image(list_latents1[-1])
        return list_latents1

    def _branch1_crossfeed_coeffs(self):
        """blending_engine.py:403-408: linspace(power, power*decay, round(N*range)) ++ zeros."""
        N = self.num_inference_steps
        idx_mixing_stop = int(round(N * self.branch1_crossfeed_range))
        mixing_coeffs = list(np.linspace(self.branch1_crossfeed_power,
                                         self.branch1_crossfeed_power * self.branch1_crossfeed_decay,
                                         idx_mixing_stop))
        mixing_coeffs.extend((N - idx_mixing_stop) * [0])
        return mixing_coeffs

    def _compute_latents_pair(self):
        """compute_latents1 + compute_latents2 advanced in lockstep through batch-4 UNet forwards (same results:
        the two trajectories are independent, or -- with branch-1 crossfeed -- trajectory 2 reads step i-1 of
        trajectory 1, which the lockstep loop has already produced)."""
        self.dh.set_num_inference_steps(self.num_inference_steps)
        job1 = dict(text_embeddings=self.get_mixed_conditioning(0)[0], latents_start=self.get_noise(self.seed1),
                    noise_fn=self._noise_source(0.0))
        job2 = dict(text_embeddings=self.get_mixed_conditioning(1)[0], latents_start=self.get_noise(self.seed2),
                    noise_fn=self._noise_source(1.0))
        if self.branch1_crossfeed_power > 0.0:
            job2.update(list_latents_mixing=("job", 0), mixing_coeffs=self._branch1_crossfeed_coeffs())
        ev0, ev1 = self._events()
        list_latents1, list_latents2 = self.dh.run_diffusion_sd_xl_multi([job1, job2], idx_start=0)
        self._finish_timing(ev0, ev1, branches=2)
        self.tree_latents[0] = list_latents1
        self.tree_latents[-1] = list_latents2
        return list_latents1, list_latents2

    def compute_latents2(self, return_image=False):
        list_conditionings = self.get_mixed_conditioning(1)
        latents_start = self.get_noise(self.seed2)
        if self.branch1_crossfeed_power > 0.0:
            mixing_coeffs = self._branch1_crossfeed_coeffs()
            list_latents2 = self.run_diffusion(list_conditionings, latents_start=latents_start, idx_start=0,
                                               list_latents_mixing=self.tree_latents[0], mixing_coeffs=mixing_coeffs,
                                               noise_key=1.0)
        else:
            list_latents2 = self.run_diffusion(list_conditionings, latents_start, noise_key=1.0)
        self.tree_latents[-1] = list_latents2
        if return_image:
            return self.dh.latent2image(list_latents2[-1])
        return list_latents2

    def _parental_mix(self, traj1, traj2, fract):
        """One batched slerp over the steps where both parents have latents (blending_engine.py:442-450)."""
        N = self.num_inference_steps
        first = 0
        while first < N and (traj1[first] is None or traj2[first] is None):
            first += 1
        out = [None] * N
        if first == N:
            return out
        rows = N - first
        ref = traj1[first]
        n = ref.numel()

        def slab(traj):
            # trajectories produced by the holder are contiguous slabs: rows are `n` elements apart
            base = traj[first]
            store = base.untyped_storage().data_ptr()
            ok = all(traj[first + r].untyped_storage().data_ptr() == store and
                     traj[first + r].data_ptr() == base.data_ptr() + r * n * base.element_size()
                     for r in range(rows))
            if ok:
                return torch.as_strided(base, (rows, n), (n, 1))
            return torch.stack([t.reshape(n) for t in traj[first:]], 0)

        if not (torch.is_tensor(ref) and ref.is_cuda):
            raise RuntimeError("parental mix needs CUDA latents (no CPU fallback)")
        mixed = ops.slerp_rows(slab(traj1), slab(traj2), float(fract))
        for r in range(rows):
            out[first + r] = mixed[r].view(ref.shape)
        return out

    def compute_latents_mix(self, fract_mixing, b_parent1, b_parent2, idx_injection):
        list_conditionings = self.get_mixed_conditioning(fract_mixing)
        fract_mixing_parental = (fract_mixing - self.tree_fracts[b_parent1]) / \
            (self.tree_fracts[b_parent2] - self.tree_fracts[b_parent1])
        list_latents_parental_mix = self._parental_mix(self.tree_latents[b_parent1], self.tree_latents[b_parent2],
                                                       fract_mixing_parental)
        N = self.num_inference_steps
        idx_mixing_stop = int(round(N * self.parental_crossfeed_range))
        mixing_coeffs = idx_injection * [self.parental_crossfeed_power]
        nmb_mixing = idx_mixing_stop - idx_injection
        if nmb_mixing > 0:
            mixing_coeffs.extend(list(np.linspace(self.parental_crossfeed_power,
                                                  self.parental_crossfeed_power * self.parental_crossfeed_decay,
                                                  nmb_mixing)))
        mixing_coeffs.extend((N - len(mixing_coeffs)) * [0])
        latents_start = list_latents_parental_mix[idx_injection - 1]
        return self.run_diffusion(list_conditionings, latents_start=latents_start, idx_start=idx_injection,
                                  list_latents_mixing=list_latents_parental_mix, mixing_coeffs=mixing_coeffs,
                                  noise_key=fract_mixing)

    def get_time_based_branching(self, depth_strength, t_compute_max_allowed=None, nmb_max_branches=None):
        self._resolve_timing()
        N = self.num_inference_steps
        idx_injection_base = int(np.floor(N * depth_strength))
        steps = int(np.ceil(N / 10))
        list_idx_injection = np.arange(idx_injection_base, N, steps)
        list_nmb_stems = np.ones(len(list_idx_injection), dtype=np.int32)
        if nmb_max_branches is None:
            assert t_compute_max_allowed is not None, "Either specify t_compute_max_allowed or nmb_max_branches"
            stop_criterion = "t_compute_max_allowed"
        elif t_compute_max_allowed is None:
            stop_criterion = "nmb_max_branches"
            nmb_max_branches -= 2  # the two outer frames
        else:
            raise ValueError("Either specify t_compute_max_allowed or nmb_max_branches")
        stop, first_iteration = False, True
        while not stop:
            list_compute_steps = (N - list_idx_injection) * list_nmb_stems
            t_compute = np.sum(list_compute_steps) * self.dt_unet_step + self.dt_vae * np.sum(list_nmb_stems)
            t_compute += 2 * (N * self.dt_unet_step + self.dt_vae)
            increased = False
            for s_idx in range(len(list_nmb_stems) - 1):
                if list_nmb_stems[s_idx + 1] / list_nmb_stems[s_idx] >= 1:
                    list_nmb_stems[s_idx] += 1
                    increased = True
                    break
            if not increased:
                list_nmb_stems[-1] += 1
            if stop_criterion == "t_compute_max_allowed" and t_compute > t_compute_max_allowed:
                stop = True
            elif stop_criterion == "nmb_max_branches" and np.sum(list_nmb_stems) >= nmb_max_branches:
                stop = True
                if first_iteration:
                    list_idx_injection = np.linspace(list_idx_injection[0], list_idx_injection[-1],
                                                     nmb_max_branches).astype(np.int32)
                    list_nmb_stems = np.ones(len(list_idx_injection), dtype=np.int32)
            else:
                first_iteration = False
        return list_idx_injection, list_nmb_stems

    def get_mixing_parameters(self, idx_injection):
        similarities = self.tree_similarities
        b_closest1 = 0 if len(similarities) == 1 else int(np.argmax(similarities))
        b_closest2 = b_closest1 + 1
        fract_mixing = (self.tree_fracts[b_closest1] + self.tree_fracts[b_closest2]) / 2
        b_parent1 = b_closest1
        while self.tree_idx_injection[b_parent1] >= idx_injection:
            b_parent1 -= 1
        b_parent2 = b_closest2
        while self.tree_idx_injection[b_parent2] >= idx_injection:
            b_parent2 += 1
        return fract_mixing, b_parent1, b_parent2

    def insert_into_tree(self, fract_mixing, idx_injection, list_latents):
        frame = self._decode_frame(list_latents[-1])
        b_parent1, b_parent2 = self.get_closest_idx(fract_mixing)
        left_sim = self.get_lpips_similarity(frame, self._tree_frames[b_parent1])
        right_sim = self.get_lpips_similarity(frame, self._tree_frames[b_parent2])
        idx_insert = b_parent1 + 1
        self.tree_latents.insert(idx_insert, list_latents)
        self._tree_frames.insert(idx_insert, frame)
        self.tree_fracts.insert(idx_insert, fract_mixing)
        self.tree_idx_injection.insert(idx_insert, idx_injection)
        self.tree_similarities[b_parent1] = left_sim
        self.tree_similarities.insert(idx_insert, right_sim)

    def get_noise(self, seed):
        return self.dh.get_noise(seed)

    @torch.no_grad()
    def run_diffusion(self, list_conditionings, latents_start=None, idx_start=0, list_latents_mixing=None,
                      mixing_coeffs=0.0, return_image=False, noise_key=None):
        self.dh.set_num_inference_steps(self.num_inference_steps)
        assert type(list_conditionings) is list, "list_conditionings need to be a list"
        src = self._noise_source(noise_key) if (noise_key is not None and hasattr(self.dh, "pipe")
                                                and self.dh.pipe is not None) else None
        if src is not None:
            out = self.dh.run_diffusion_sd_xl_multi([dict(text_embeddings=list_conditionings[0], latents_start=latents_start,
                                                          list_latents_mixing=list_latents_mixing,
                                                          mixing_coeffs=mixing_coeffs, noise_fn=src)], idx_start)[0]
            return self.dh.latent2image(out[-1]) if return_image else out
        return self.dh.run_diffusion_sd_xl(text_embeddings=list_conditionings[0], latents_start=latents_start,
                                           idx_start=idx_start, list_latents_mixing=list_latents_mixing,
                                           mixing_coeffs=mixing_coeffs, return_image=return_image)

    @torch.no_grad()
    def get_mixed_conditioning(self, fract_mixing):
        mix = [None if a is None else interpolate_linear(a, b, fract_mixing)
               for a, b in zip(self.text_embedding1, self.text_embedding2)]
        return [mix]

    @torch.no_grad()
    def get_text_embeddings(self, prompt: str):
        return self.dh.get_text_embedding(prompt)

    # ---- outputs ------------------------------------------------------------------------------------
    def write_imgs_transition(self, dp_img):
        os.makedirs(dp_img, exist_ok=True)
        for i, img in enumerate(self.tree_final_imgs):
            img.save(os.path.join(dp_img, f"lowres_img_{str(i).zfill(4)}.jpg"))

    def write_movie_transition(self, fp_movie, duration_transition, fps=30):
        """Fill up to duration*fps frames by linear interpolation and encode with OpenCV
        (the reference uses lunar_tools.MovieSaver/ffmpeg, blending_engine.py:684-706)."""
        import cv2
        frames = self.get_movie_frames(duration_transition, fps)
        if os.path.isfile(fp_movie):
            os.remove(fp_movie)
        h, w = self.dh.height_img, self.dh.width_img
        vw = cv2.VideoWriter(fp_movie, cv2.VideoWriter_fourcc(*"mp4v"), fps, (w, h))
        for f in frames:
            f = np.asarray(f)
            if f.shape[0] != h or f.shape[1] != w:
                f = cv2.resize(f, (w, h))
            vw.write(cv2.cvtColor(f, cv2.COLOR_RGB2BGR))
        vw.release()

    def get_movie_frames(self, duration_transition, fps=30, seed=None):
        """The duration*fps frames of the transition movie as one uint8 array [T,H,W,3]: the tree frames plus the
        linear fill of utils.py:105-178 (add_frames_linear_interp), blended ON THE DEVICE by lb_frames_lerp_u8 from
        the device-resident key frames -- one launch, one device->host copy (the reference blends T float32 images
        on the CPU).  With a foreign holder whose frames are host images the same plan runs through the numpy
        version (utils.add_frames_linear_interp), which is the reference's own algorithm."""
        from .utils import plan_frame_fill
        keys = getattr(self, "_tree_frames", None)
        if not keys or not all(torch.is_tensor(f) and f.is_cuda for f in keys):
            return np.stack([np.asarray(f) for f in add_frames_linear_interp(
                [np.asarray(im) for im in self.tree_final_imgs], fps_target=fps, duration_target=duration_transition,
                seed=seed)], 0)
        left, w0, w1 = plan_frame_fill(len(keys), fps * duration_transition, seed=seed)
        stack = torch.stack(keys, 0).contiguous()
        F_, H, W, C = stack.shape
        dev = stack.device
        out = ops.frames_lerp_u8(stack.view(F_, H * W * C), torch.from_numpy(left).to(dev),
                                 torch.from_numpy(w0).to(dev), torch.from_numpy(w1).to(dev))
        return out.view(-1, H, W, C).cpu().numpy()

    def get_state_dict(self):
        state_dict = {}
        for v in ['prompt1', 'prompt2', 'seed1', 'seed2', 'num_inference_steps', 'guidance_scale',
                  'guidance_scale_mid_damper', 'mid_compression_scaler', 'negative_prompt',
                  'branch1_crossfeed_power', 'branch1_crossfeed_range', 'branch1_crossfeed_decay',
                  'parental_crossfeed_power', 'parental_crossfeed_range', 'parental_crossfeed_decay']:
            if hasattr(self, v):
                val = getattr(self, v)
                if v in ('seed1', 'seed2'):
                    val = int(val)
                elif v == 'guidance_scale' or isinstance(val, (np.floating,)):
                    val = float(val)
                state_dict[v] = val
        return state_dict

    def swap_forward(self):
        self.tree_latents[0] = self.tree_latents[-1]
        self.prompt1 = self.prompt2
        self.text_embedding1 = self.text_embedding2
        self.tree_final_imgs = []

    # ---- similarity / helpers ---------------------------------------------------------------------------
    def get_lpips_similarity(self, imgA, imgB):
        """High values = dissimilar.  Accepts device uint8 frames (internal) or PIL/numpy images (API parity)."""
        if self._similarity_fn is not None:
            return self._similarity_fn(self._to_numpy(imgA), self._to_numpy(imgB))
        return self.lpips.distance(self._to_device_frame(imgA), self._to_device_frame(imgB))

    def get_tree_similarities(self):
        return [self.get_lpips_similarity(self._tree_frames[i], self._tree_frames[i + 1])
                for i in range(len(self._tree_frames) - 1)]

    def get_closest_idx(self, fract_mixing: float):
        pdist = fract_mixing - np.asarray(self.tree_fracts)
        pdist_pos = pdist.copy()
        pdist_pos[pdist_pos < 0] = np.inf
        b_parent1 = int(np.argmin(pdist_pos))
        pdist_neg = -pdist.copy()
        pdist_neg[pdist_neg <= 0] = np.inf
        b_parent2 = int(np.argmin(pdist_neg))
        if b_parent1 > b_parent2:
            b_parent1, b_parent2 = b_parent2, b_parent1
        return b_parent1, b_parent2

    def _decode_frame(self, latents):
        if hasattr(self.dh, "decode_to_device"):
            return self.dh.decode_to_device(latents)
        return self.dh.latent2image(latents)          # foreign holder (tests): whatever it returns

    def _frame_to_pil(self, frame):
        if torch.is_tensor(frame):
            self.d2h_bytes += frame.numel() * frame.element_size()
            return Image.fromarray(frame.cpu().numpy())
        return frame

    def _to_numpy(self, img):
        return img.cpu().numpy() if torch.is_tensor(img) else np.asarray(img)

    def _to_device_frame(self, img):
        if torch.is_tensor(img):
            return img
        return torch.from_numpy(np.asarray(img)).to(self.device)

    def _events(self):
        if torch.cuda.is_available():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            return e0, e1
        return time.time(), None

    def _finish_timing(self, e0, e1, branches=1):
        if e1 is None:
            self.dt_unet_step = (time.time() - e0) / (self.num_inference_steps * branches)
            return
        e1.record()
        # resolved lazily by set_branching / get_time_based_branching: no host sync inside the transition
        self._pending_timing = (e0, e1, branches, self.num_inference_steps)

    def _resolve_timing(self):
        """dt_unet_step tracks the last outer trajectory like blending_engine.py:379-386 (time per UNet step of ONE
        branch), from CUDA events recorded around it."""
        pend = getattr(self, "_pending_timing", None)
        if pend is None:
            return
        self._pending_timing = None
        e0, e1, branches, n = pend
        e1.synchronize()
        self.dt_unet_step = e0.elapsed_time(e1) / 1e3 / (n * branches)
