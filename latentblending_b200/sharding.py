"""Branch-level sharding of one transition across the GPUs of a node (one process per GPU).

The reference builds the tree strictly sequentially (latentblending/blending_engine.py:354-362):
each insertion takes the arg-max LPIPS gap, computes the branch at its midpoint and updates the
two neighbouring similarities, which the NEXT insertion of the same level reads (:541-547 /
:586-588).  What makes sharding possible is that a branch's latents depend only on its
``fract_mixing``, the level's ``idx_injection`` and strictly OLDER parents (:549-561, :439-458) --
never on branches of its own level.  So within a level:

  1. plan:    every rank derives the same list of up to ``world`` candidate midpoints from the
              replicated tree -- a best-first subdivision of the current gaps (a gap's halves are
              estimated at half its similarity), skipping midpoints already computed;
  2. compute: rank r runs candidate r (parental mix + denoise + decode) on its GPU;
  3. gather:  ONE all-gather per round collects the finished trajectory slabs and decoded frames
              (``torch.distributed``: NCCL over NVLink on GPUs, gloo in the CPU tests);
  4. replay:  every rank replays the reference's greedy loop on the replicated tree, consuming
              cached candidates for as long as the arg-max gap's midpoint has been computed; the
              first miss starts the next round.  Mis-speculated branches stay cached for later
              rounds of the level and are dropped at its end.

The tree that results is exactly the sequential one (same ``tree_fracts`` order, same parents).
Every rank evaluates the similarity pair of every insertion itself on the replicated (all-gathered)
frames: the metric kernels are deterministic, so all replicas take identical decisions without any
further collective (a one-word agreement check per level guards that assumption).

CFG split (SURVEY.md section 8e, "GPU pair per branch splitting the CFG halves"): with classifier-free
guidance every UNet forward is a batch of two (unconditional, text).  When there are more ranks than
useful candidates the ranks pair up into TEAMS of two: each team computes ONE candidate, each member one
CFG half (a batch-1 forward, ~0.6x the time of the batch-2 one), and the two 128 KB eps halves are
exchanged once per step inside the team (DiffusersHolder.cfg_split).  The per-round all-gather then takes
each team's slab from its first member.  Pairs shorten the dependent chain but halve the candidates per round, so
they are used for the outer trajectories (from 4 ranks) and for the last stems of a level (``team_size``).

This module is pure host logic + collectives; the arithmetic is injected (``compute``,
``similarity``), which is how the world_size-2 gloo test drives it on CPU.
"""
import heapq

import numpy as np
import torch


def older_parents(tree_fracts, tree_idx_injection, fract, idx_injection):
    """Indices of the nearest tree nodes left/right of ``fract`` whose idx_injection is older
    (blending_engine.py:549-561 applied to an arbitrary midpoint)."""
    fr = np.asarray(tree_fracts)
    left = int(np.max(np.nonzero(fr <= fract)[0])) if np.any(fr <= fract) else 0
    # nodes exactly at `fract` cannot exist (midpoints are new); left < right always
    right = left + 1
    while tree_idx_injection[left] >= idx_injection:
        left -= 1
    while tree_idx_injection[right] >= idx_injection:
        right += 1
    return left, right


def plan_candidates(tree_fracts, tree_similarities, budget, cached, split_ratio=0.5):
    """Best-first subdivision of the current gaps -> up to ``budget`` (mid, lo, hi) midpoints not in ``cached``.
    The first returned candidate is always the reference's next choice (arg-max gap) unless it is cached;
    the halves of a split gap are estimated at ``split_ratio`` x its similarity."""
    sims = list(tree_similarities)
    if len(sims) == 1 and not isinstance(sims[0], (int, float, np.floating)):
        sims = [1.0]                                  # blending_engine.py:349: first arg-max is over a 1-list
    heap = []
    for i, s in enumerate(sims):
        # ties resolve like np.argmax: lowest index first
        heapq.heappush(heap, (-float(s), i, 0, float(tree_fracts[i]), float(tree_fracts[i + 1])))
    out, guard = [], 0
    while heap and len(out) < budget and guard < 64 * max(1, budget):
        guard += 1
        neg, order, depth, lo, hi = heapq.heappop(heap)
        mid = (lo + hi) / 2
        if mid not in cached and all(mid != c[0] for c in out):
            out.append((mid, lo, hi))
        if depth < 6:
            heapq.heappush(heap, (neg * split_ratio, order, depth + 1, lo, mid))
            heapq.heappush(heap, (neg * split_ratio, order, depth + 1, mid, hi))
    return out


class LevelSharder:
    """Runs the stems of one tree level over ``world`` ranks.

    tree: object with lists tree_fracts, tree_idx_injection, tree_similarities, tree_latents, frames
          (``frames`` = decoded frames used by ``similarity``) -- replicated on every rank.
    compute(fract, b_parent1, b_parent2, idx_injection) -> (list_latents, frame)
    similarity(frame_a, frame_b) -> float
    """

    def __init__(self, rank, world, group=None, device=None, cfg_pairs=False):
        self.rank, self.world, self.group = rank, world, group
        self.device = device
        self.stats = dict(rounds=0, computed=0, used=0, paired_rounds=0)
        self.split_ratio = 0.6        # running estimate of (similarity of a half) / (similarity of the split gap)
        self.cfg_pairs = bool(cfg_pairs) and world >= 2     # CFG is on: ranks may pair up (one CFG half each)
        self._pair_groups = None

    # -- teams ---------------------------------------------------------------------------------
    def team_size(self, remaining):
        """Ranks per candidate this round.  A pair (one CFG half per rank) shortens the dependent chain -- a batch-1
        forward costs less than a batch-2 one -- but halves the number of speculative
        candidates per round, and a missed pick costs a whole extra round.  So pairs are used when the pair-teams still
        cover every remaining stem of the level (world // 2 >= remaining: all levels of the 15-branch tree on 8 ranks,
        the 2- and 1-stem levels on 4 ranks) and for the last stem of a level."""
        if not self.cfg_pairs:
            return 1
        return 2 if (remaining <= 1 or self.world // 2 >= remaining) else 1

    def pair_group(self):
        """The 2-rank process group of this rank's team; all groups are created collectively on first use."""
        import torch.distributed as dist
        if self._pair_groups is None:
            self._pair_groups = [dist.new_group(ranks=[2 * t, 2 * t + 1]) for t in range(self.world // 2)]
        t = self.rank // 2
        return self._pair_groups[t] if t < len(self._pair_groups) else None

    # -- collectives -------------------------------------------------------------------------
    def _all_gather(self, t):
        import torch.distributed as dist
        outs = [torch.empty_like(t) for _ in range(self.world)]
        dist.all_gather(outs, t.contiguous(), group=self.group)
        return outs

    def _check_agreement(self, tree):
        """All replicas must hold the same tree (they decide independently on replicated data)."""
        import torch.distributed as dist
        v = float(np.sum(np.asarray(tree.tree_fracts, dtype=np.float64) * np.arange(1, len(tree.tree_fracts) + 1)))
        t = torch.tensor([v, -v], dtype=torch.float64, device=self.device if self.device is not None else "cpu")
        dist.all_reduce(t, op=dist.ReduceOp.MAX, group=self.group)
        if float(t[0]) != -float(t[1]):
            raise RuntimeError("sharded transition: the ranks' trees diverged (non-deterministic similarity?)")

    # -- one level ---------------------------------------------------------------------------------
    def run_level(self, tree, idx_injection, n_stems, compute, similarity, num_steps, on_insert=None):
        """``on_insert(mid)`` runs on EVERY rank for every inserted branch, in insertion order (state the sequential
        engine updates per branch -- the guidance dampening -- must end up identical on all ranks)."""
        cache = {}                # mid -> (list_latents, frame)
        remaining = int(n_stems)
        while remaining > 0:
            team = self.team_size(remaining)
            n_teams = self.world // team
            cands = plan_candidates(tree.tree_fracts, tree.tree_similarities, n_teams, cache, self.split_ratio)
            self.stats["rounds"] += 1
            self.stats["paired_rounds"] += int(team == 2)
            my_team = self.rank // team
            mine = cands[my_team] if my_team < len(cands) and self.rank < n_teams * team else None
            slab = frame = None
            if team == 2:
                self.pair_group()              # collective creation on first use: every rank must get here
            if mine is not None:
                p1, p2 = older_parents(tree.tree_fracts, tree.tree_idx_injection, mine[0], idx_injection)
                if team == 2:
                    traj, frame = compute(mine[0], p1, p2, idx_injection,
                                          cfg_split=dict(group=self.pair_group(), half=self.rank % 2))
                else:
                    traj, frame = compute(mine[0], p1, p2, idx_injection)
                slab = torch.stack([t.reshape(-1) for t in traj[idx_injection:]], 0)
            # shapes are identical on every rank that has work; idle ranks send zeros of the same shape
            ref_shape = self._agree_shapes(slab, frame, tree, idx_injection, num_steps)
            if slab is None:
                slab = torch.zeros(ref_shape[0], dtype=ref_shape[2], device=ref_shape[4])
                frame = torch.zeros(ref_shape[1], dtype=ref_shape[3], device=ref_shape[4])
            slabs = self._all_gather(slab)
            frames = self._all_gather(frame)
            lat_shape = tree.tree_latents[0][-1].shape
            for c, (mid, lo, hi) in enumerate(cands):
                r = c * team                   # a team's slab is taken from its first member (both hold the same data)
                traj = [None] * idx_injection + [slabs[r][i].view(lat_shape) for i in range(num_steps - idx_injection)]
                cache[mid] = (traj, frames[r])
                self.stats["computed"] += 1
            # replay the reference's greedy loop on the replicated tree
            while remaining > 0:
                sims = tree.tree_similarities
                c1 = 0 if len(sims) == 1 else int(np.argmax(sims))
                mid = (tree.tree_fracts[c1] + tree.tree_fracts[c1 + 1]) / 2
                if mid not in cache:
                    break
                traj, frm = cache.pop(mid)
                left = similarity(frm, tree.frames[c1])
                right = similarity(frm, tree.frames[c1 + 1])
                parent_sim = sims[c1]
                if isinstance(parent_sim, (int, float, np.floating)) and parent_sim > 0:
                    obs = min(1.0, max(left, right) / float(parent_sim))
                    self.split_ratio = 0.7 * self.split_ratio + 0.3 * obs     # identical on every rank
                if on_insert is not None:
                    on_insert(mid)
                k = c1 + 1
                tree.tree_latents.insert(k, traj)
                tree.frames.insert(k, frm)
                tree.tree_fracts.insert(k, mid)
                tree.tree_idx_injection.insert(k, idx_injection)
                tree.tree_similarities[c1] = left
                tree.tree_similarities.insert(k, right)
                remaining -= 1
                self.stats["used"] += 1
        self._check_agreement(tree)

    def _agree_shapes(self, slab, frame, tree, idx_injection, num_steps):
        lat = tree.tree_latents[0][-1]
        f0 = tree.frames[0]
        n = lat.numel()
        return ((num_steps - idx_injection, n), tuple(f0.shape), lat.dtype, f0.dtype, lat.device)


def run_level_local(tree, idx_injection, n_stems, compute_many, similarity, width, on_insert=None, stats=None,
                    split_ratio=0.6):
    """Single-GPU speculation: the stems of one level with up to ``width`` candidate branches advanced in LOCKSTEP
    through one batched UNet forward per step (DiffusersHolder.run_diffusion_sd_xl_multi).  Same planning and replay as
    LevelSharder.run_level with the ranks replaced by batch slots: candidates = best-first subdivision of the current
    gaps, replay = the reference's greedy loop consuming cached candidates; mis-speculated candidates stay cached
    until the level ends.  Every kernel is batch-invariant, so the tree equals the sequential one.  Pays when a
    batch-k forward costs much less than k batch-1 forwards: SDXL-Turbo at 512^2 (weight-bandwidth / launch bound);
    not SDXL-base at 1024^2 on one GPU (batch 4 costs 1.76x batch 2).

    compute_many([(mid, p1, p2), ...], idx_injection) -> [(list_latents, frame), ...]"""
    cache = {}
    remaining = int(n_stems)
    ratio = split_ratio
    while remaining > 0:
        cands = plan_candidates(tree.tree_fracts, tree.tree_similarities, min(width, remaining), cache, ratio)
        todo = []
        for mid, lo, hi in cands:
            p1, p2 = older_parents(tree.tree_fracts, tree.tree_idx_injection, mid, idx_injection)
            todo.append((mid, p1, p2))
        for (mid, _, _), res in zip(todo, compute_many(todo, idx_injection)):
            cache[mid] = res
        if stats is not None:
            stats["rounds"] += 1
            stats["computed"] += len(todo)
        while remaining > 0:
            sims = tree.tree_similarities
            c1 = 0 if len(sims) == 1 else int(np.argmax(sims))
            mid = (tree.tree_fracts[c1] + tree.tree_fracts[c1 + 1]) / 2
            if mid not in cache:
                break
            traj, frm = cache.pop(mid)
            left = similarity(frm, tree.frames[c1])
            right = similarity(frm, tree.frames[c1 + 1])
            parent_sim = sims[c1]
            if isinstance(parent_sim, (int, float, np.floating)) and parent_sim > 0:
                ratio = 0.7 * ratio + 0.3 * min(1.0, max(left, right) / float(parent_sim))
            if on_insert is not None:
                on_insert(mid)
            k = c1 + 1
            tree.tree_latents.insert(k, traj)
            tree.frames.insert(k, frm)
            tree.tree_fracts.insert(k, mid)
            tree.tree_idx_injection.insert(k, idx_injection)
            tree.tree_similarities[c1] = left
            tree.tree_similarities.insert(k, right)
            remaining -= 1
            if stats is not None:
                stats["used"] += 1
    return ratio
