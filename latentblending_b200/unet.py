"""SDXL UNet on liblb200: weight packing + lowering of one forward pass to a C-ABI program.

Host side of the executor that replaces ``pipe.unet(...)`` in the reference's
denoise loop (latentblending/diffusers_holder.py:336-344).  Parameters are taken
by their diffusers ``state_dict`` names, so ``pipe.unet.state_dict()`` of a real
StableDiffusionXLPipeline can be passed as is.

Data layout in HBM (all fp16):
  * activations NHWC, i.e. [B*H*W, C] row-major with an explicit row stride so
    that channel slices of a wider buffer are first-class tensors; the nine
    ``torch.cat([hidden, skip])`` of the up path are never materialised: every
    skip tensor is written by its producer straight into the right half of its
    future concat buffer and read from there by the down path;
  * weights [N, K] row-major (K-major for the tensor core B operand); 3x3 conv
    weights [Cout][ky][kx][Cin]; a resnet's 1x1 shortcut is appended along K of
    conv2 (one accumulator, biases pre-summed); to_q/to_k/to_v fused to one
    [3C, C] matrix, cross-attention to_k/to_v to [2C, ctx]; GEGLU rows
    interleaved per 128-row tile (64 value rows then their 64 gate rows);
    all resnet ``time_emb_proj`` stacked into one [sum Cout, T] matrix.
  * latents / eps stay NCHW [B,4,h,w] like the reference's tensors.
"""
from dataclasses import dataclass
from typing import Tuple

import torch

from . import _cabi
from ._cabi import ctx
from .lowering import Scratch, lower_conv_out, lower_resnet, pack3, pack_resnet
from .program import Program, pack_conv_out8


@dataclass
class UNetConfig:
    in_channels: int = 4
    out_channels: int = 4
    block_out_channels: Tuple[int, ...] = (320, 640, 1280)
    layers_per_block: int = 2
    transformer_layers: Tuple[int, ...] = (0, 2, 10)
    head_dim: int = 64
    cross_attention_dim: int = 2048
    addition_time_embed_dim: int = 256
    pooled_dim: int = 1280
    norm_num_groups: int = 32
    sample_size: int = 128
    time_cond_proj_dim: object = None

    @property
    def time_embed_dim(self):
        return self.block_out_channels[0] * 4

    @property
    def add_in_dim(self):
        return self.pooled_dim + 6 * self.addition_time_embed_dim


def _fold_layernorm(w, bias, gamma, beta):
    """(w*gamma in fp16, rowsum of THAT in fp32, w beta + bias in fp32) for the LayerNorm-folded GEMM."""
    wf = (w.float() * gamma.float()[None, :]).half().contiguous()
    csum = wf.float().sum(dim=1).contiguous()
    lnb = w.float() @ beta.float()
    if bias is not None:
        lnb = lnb + bias.float()
    return wf, csum, lnb.contiguous()


def _geglu_perm(inner, device, half=64):
    """Row order of the GEGLU projection for the kernel's N tiles: ``half`` value rows then their ``half`` gate rows."""
    idx = torch.arange(inner, device=device).view(-1, half)
    return torch.stack([idx, idx + inner], dim=1).reshape(-1)


class PackedUNet:
    """fp16 device copies of the UNet parameters in the layouts the kernels consume."""

    def __init__(self, cfg: UNetConfig, state_dict, device, fold_ln=True):
        self.cfg = cfg
        self.device = torch.device(device)
        self.fold_ln = fold_ln
        sd = state_dict
        dev = self.device

        def g(name):
            return sd[name].detach().to(device=dev, dtype=torch.float16).contiguous()

        self.g = g
        self.w = {}
        W = self.w
        W["conv_in.w"] = g("conv_in.weight").permute(2, 3, 1, 0).contiguous()      # [ky][kx][cin][Cout]
        W["conv_in.b"] = g("conv_in.bias")
        W["conv_out.w"] = g("conv_out.weight").permute(0, 2, 3, 1).contiguous()     # [co][ky][kx][Cin]
        W["conv_out.b"] = g("conv_out.bias")
        W["conv_out.w8"], W["conv_out.b8"] = pack_conv_out8(W["conv_out.w"], W["conv_out.b"])
        for nm in ("conv_norm_out",):
            W[nm + ".g"], W[nm + ".b"] = g(nm + ".weight"), g(nm + ".bias")
        for e in ("time_embedding", "add_embedding"):
            for l in ("linear_1", "linear_2"):
                W[f"{e}.{l}.w"], W[f"{e}.{l}.b"] = g(f"{e}.{l}.weight"), g(f"{e}.{l}.bias")
        # resnets (names collected in forward order so the stacked time_emb_proj offsets line up)
        self.resnet_names = [k[: -len(".norm1.weight")] for k in sd if k.endswith(".norm1.weight") and "resnets" in k]
        temb_w, temb_b, off = [], [], 0
        self.temb_off = {}
        for r in self.resnet_names:
            pack_resnet(W, r, sd, g)
            tw, tb = g(r + ".time_emb_proj.weight"), g(r + ".time_emb_proj.bias")
            self.temb_off[r] = (off, tw.shape[0])
            off += tw.shape[0]
            temb_w.append(tw)
            temb_b.append(tb)
        W["temb_all.w"], W["temb_all.b"] = torch.cat(temb_w, 0).contiguous(), torch.cat(temb_b, 0).contiguous()
        self.temb_total = off
        # transformers
        self.tf_names = [k[: -len(".proj_in.weight")] for k in sd if k.endswith(".proj_in.weight")]
        for a in self.tf_names:
            W[a + ".norm.g"], W[a + ".norm.b"] = g(a + ".norm.weight"), g(a + ".norm.bias")
            W[a + ".proj_in.w"], W[a + ".proj_in.b"] = g(a + ".proj_in.weight"), g(a + ".proj_in.bias")
            W[a + ".proj_out.w"], W[a + ".proj_out.b"] = g(a + ".proj_out.weight"), g(a + ".proj_out.bias")
            depth = 0
            while f"{a}.transformer_blocks.{depth}.norm1.weight" in sd:
                t = f"{a}.transformer_blocks.{depth}"
                for n in ("norm1", "norm2", "norm3"):
                    W[f"{t}.{n}.g"], W[f"{t}.{n}.b"] = g(f"{t}.{n}.weight"), g(f"{t}.{n}.bias")
                wqkv = torch.cat([g(t + ".attn1.to_q.weight"), g(t + ".attn1.to_k.weight"),
                                  g(t + ".attn1.to_v.weight")], 0).contiguous()
                W[t + ".attn1.out.w"], W[t + ".attn1.out.b"] = g(t + ".attn1.to_out.0.weight"), g(t + ".attn1.to_out.0.bias")
                wq = g(t + ".attn2.to_q.weight")
                W[t + ".attn2.kv.w"] = torch.cat([g(t + ".attn2.to_k.weight"), g(t + ".attn2.to_v.weight")], 0).contiguous()
                W[t + ".attn2.out.w"], W[t + ".attn2.out.b"] = g(t + ".attn2.to_out.0.weight"), g(t + ".attn2.to_out.0.bias")
                pw, pb = g(t + ".ff.net.0.proj.weight"), g(t + ".ff.net.0.proj.bias")
                perm = _geglu_perm(pw.shape[0] // 2, dev)     # per 128-column N tile of the GEGLU GEMM
                if fold_ln:
                    # LayerNorm folded into the consuming GEMM (include/lb200.h): w' = w*gamma, csum = rowsum(w'),
                    # lnb = w beta + bias
                    for key, w_, b_, nrm, pm in ((".attn1.qkv", wqkv, None, "norm1", None), (".attn2.q", wq, None, "norm2", None),
                                                 (".ff.in", pw, pb, "norm3", perm)):
                        wf, cs, lb = _fold_layernorm(w_, b_, W[f"{t}.{nrm}.g"], W[f"{t}.{nrm}.b"])
                        if pm is not None:
                            wf, cs, lb = wf[pm].contiguous(), cs[pm].contiguous(), lb[pm].contiguous()
                        W[t + key + ".w"], W[t + key + ".csum"], W[t + key + ".lnb"] = wf, cs, lb
                else:
                    W[t + ".attn1.qkv.w"], W[t + ".attn2.q.w"] = wqkv, wq
                    W[t + ".ff.in.w"], W[t + ".ff.in.b"] = pw[perm].contiguous(), pb[perm].contiguous()
                W[t + ".ff.out.w"], W[t + ".ff.out.b"] = g(t + ".ff.net.2.weight"), g(t + ".ff.net.2.bias")
                depth += 1
            W[a + ".depth"] = depth
        for k in sd:
            if k.endswith("samplers.0.conv.weight"):
                nm = k[: -len(".weight")]
                W[nm + ".w"], W[nm + ".b"] = pack3(g(nm + ".weight")), g(nm + ".bias")

    def nbytes(self):
        return sum(t.numel() * t.element_size() for t in self.w.values() if torch.is_tensor(t))


class UNetB200:
    """One lowered forward per (batch, h, w); ``forward`` replays it."""

    def __init__(self, cfg: UNetConfig, state_dict, device="cuda:0", fold_ln=None):
        import os
        self.cfg = cfg
        self.device = torch.device(device)
        self.dev_index = self.device.index or 0
        # LayerNorm folding is OFF by default: the 210 LayerNorm launches need no shared memory, so under PDL they
        # co-reside with the neighbouring GEMMs' CTAs; folding them away makes GEMM follow GEMM and adds epilogue work.
        # LB_LN_FOLD=1 or fold_ln=True enables the folded path (same numerics and tolerance).
        if fold_ln is None:
            fold_ln = os.environ.get("LB_LN_FOLD") is not None
        self.fold_ln = fold_ln
        self.packed = PackedUNet(cfg, state_dict, self.device, fold_ln=fold_ln)
        self._plans = {}

    # -- public -----------------------------------------------------------------------------
    def plan(self, B, H, W, tag=None, x_in=None):
        """The lowered program for (batch, height, width).  ``tag`` keeps several independent instances (own
        activation buffers) of the same shape apart; ``x_in`` lets the caller supply the input buffer."""
        key = (B, H, W) if tag is None else (B, H, W, tag)
        if key not in self._plans:
            self._plans[key] = _Lowering(self, B, H, W, x_in=x_in)
        return self._plans[key]

    @torch.no_grad()
    def forward(self, x, t, encoder_hidden_states, text_embeds, time_ids, ctx_changed=True):
        """x [B,4,h,w] fp16 NCHW -> eps [B,4,h,w] fp16 (a view of the plan's static output buffer)."""
        B, _, H, W = x.shape
        pl = self.plan(B, H, W)
        pl.x_in.copy_(x)
        pl.text.copy_(text_embeds)
        pl.tids.copy_(time_ids)
        if ctx_changed:
            pl.ctx.copy_(encoder_hidden_states.reshape(pl.ctx.shape))
            pl.prog_ctx.run()
        pl.prog_step.run(float(t))
        return pl.eps

    def launches_per_forward(self, B, H, W):
        pl = self.plan(B, H, W)
        return pl.prog_step.num_launches, pl.prog_ctx.num_launches


class _Lowering:
    def __init__(self, net: UNetB200, B, H, W, x_in=None):
        cfg, Wt = net.cfg, net.packed.w
        self.net, self.B, self.H, self.W = net, B, H, W
        dev = net.device
        f16 = dict(dtype=torch.float16, device=dev)
        ch = list(cfg.block_out_channels)
        L = len(ch)
        T = cfg.time_embed_dim
        groups = cfg.norm_num_groups
        if x_in is not None:
            assert tuple(x_in.shape) == (B, cfg.in_channels, H, W) and x_in.dtype == torch.float16 and x_in.is_contiguous()
        self.x_in = x_in if x_in is not None else torch.zeros(B, cfg.in_channels, H, W, **f16)
        self.eps = torch.zeros(B, cfg.out_channels, H, W, **f16)
        self.ctx = torch.zeros(B * 77, cfg.cross_attention_dim, **f16)
        self.text = torch.zeros(B, cfg.pooled_dim, **f16)
        self.tids = torch.zeros(B, 6, **f16)
        self.ws = torch.zeros(max(1 << 16, _cabi.load().lb_groupnorm_workspace_bytes(ctx(net.dev_index), B, H * W, groups)),
                              dtype=torch.uint8, device=dev)
        P = self.prog_step = Program(net.dev_index)
        PC = self.prog_ctx = Program(net.dev_index)
        scratch = Scratch(torch.float16, dev)
        ln_stats = {}

        self._persist = []

        def persist(rows, cols):
            t = torch.empty(rows, cols, **f16)
            self._persist.append(t)
            return t

        # ---- embeddings -------------------------------------------------------------------
        temb_in, add_in = persist(B, ch[0]), persist(B, cfg.add_in_dim)
        P.embed_inputs(self.text, self.tids, ch[0], cfg.addition_time_embed_dim, temb_in, add_in)
        t1, a1, temb, emb = persist(B, T), persist(B, T), persist(B, T), persist(B, T)
        P.linear_small(temb_in, Wt["time_embedding.linear_1.w"], t1, bias=Wt["time_embedding.linear_1.b"], act_out=1)
        P.linear_small(t1, Wt["time_embedding.linear_2.w"], temb, bias=Wt["time_embedding.linear_2.b"])
        P.linear_small(add_in, Wt["add_embedding.linear_1.w"], a1, bias=Wt["add_embedding.linear_1.b"], act_out=1)
        P.linear_small(a1, Wt["add_embedding.linear_2.w"], emb, bias=Wt["add_embedding.linear_2.b"], addend=temb)
        temb_all = persist(B, net.packed.temb_total)
        P.linear_small(emb, Wt["temb_all.w"], temb_all, bias=Wt["temb_all.b"], act_in=1)

        # ---- geometry + concat buffers ------------------------------------------------------
        # the stride-2 pad-1 Downsample2D conv gives ceil(s/2); the up path resizes back to each skip level's size
        res_hw = [(H, W)]
        for _ in range(L - 1):
            res_hw.append(((res_hw[-1][0] + 1) // 2, (res_hw[-1][1] + 1) // 2))

        def rows_at(level):
            return B * res_hw[level][0] * res_hw[level][1]

        # skip list: (level, channels) in production order
        skip_meta = [(0, ch[0])]
        for i in range(L):
            skip_meta += [(i, ch[i])] * cfg.layers_per_block
            if i < L - 1:
                skip_meta.append((i + 1, ch[i]))
        # up path consumption: resnet j of up block i
        rev = list(reversed(ch))
        cats = []              # in pop order
        cprev = rev[0]
        k = len(skip_meta) - 1
        for i in range(L):
            cout = rev[i]
            for j in range(cfg.layers_per_block + 1):
                hidden_c = cprev if j == 0 else cout
                lvl, sc = skip_meta[k]
                buf = persist(rows_at(lvl), hidden_c + sc)
                cats.append(dict(buf=buf, hidden=buf[:, :hidden_c], skip=buf[:, hidden_c:], level=lvl))
                k -= 1
            cprev = cout
        skip_views = [c["skip"] for c in reversed(cats)]      # index by production order

        def tslice(rname):
            off, n = net.packed.temb_off[rname]
            return temb_all[:, off:off + n]

        def resnet(rname, x, cin, cout, level, out):
            h_, w_ = res_hw[level]
            lower_resnet(P, Wt, rname, x, cin, cout, B, h_, w_, out, groups, 1e-5, self.ws, scratch, bias2=tslice(rname))

        kv_cache = {}

        fold = net.fold_ln
        geglu_mode = 1
        f32 = dict(dtype=torch.float32, device=dev)

        def transformer(aname, x, C, level, out):
            h_, w_ = res_hw[level]
            S = h_ * w_
            M = rows_at(level)
            heads = C // cfg.head_dim
            tn = scratch("tn", M, C)
            P.groupnorm(x, B, S, C, groups, Wt[aname + ".norm.g"], Wt[aname + ".norm.b"], 1e-6, 0, tn, self.ws)
            hs = scratch("hs", M, C)
            if not fold:
                P.gemm(tn, Wt[aname + ".proj_in.w"], C, 1, 1, M, hs, bias=Wt[aname + ".proj_in.b"])
                stats = None
            else:
                # every GEMM that writes the residual stream ``hs`` also writes its per-row partial sums; the three
                # LayerNorms of a block are folded into the GEMMs that consume them (no LN launches, no LN buffer)
                parts = P.gemm_stats_parts(tn, Wt[aname + ".proj_in.w"], C, 1, 1, M, hs)
                if (M, parts) not in ln_stats:
                    ln_stats[(M, parts)] = torch.zeros(M, parts, 2, **f32)
                stats = ln_stats[(M, parts)]
                P.gemm(tn, Wt[aname + ".proj_in.w"], C, 1, 1, M, hs, bias=Wt[aname + ".proj_in.b"], stats_out=stats)

            def ln_of(t, key):
                return dict(stats=stats, csum=Wt[t + key + ".csum"], bias=Wt[t + key + ".lnb"], eps=1e-5)

            for d in range(Wt[aname + ".depth"]):
                t = f"{aname}.transformer_blocks.{d}"
                qkv = scratch("qkv", M, 3 * C)
                att = scratch("att", M, C)
                q = scratch("q", M, C)
                gg = scratch("geglu", M, 4 * C)
                kv = persist(B * 77, 2 * C)         # depends on the conditioning only: computed by prog_ctx
                PC.gemm(self.ctx, Wt[t + ".attn2.kv.w"], 2 * C, 1, 1, B * 77, kv)
                kv_cache[t] = kv
                if fold:
                    P.gemm(hs, Wt[t + ".attn1.qkv.w"], 3 * C, 1, 1, M, qkv, ln=ln_of(t, ".attn1.qkv"))
                    P.attention(qkv, qkv, qkv, att, B, heads, S, S, 0, C, 2 * C, cfg.head_dim ** -0.5)
                    P.gemm(att, Wt[t + ".attn1.out.w"], C, 1, 1, M, hs, bias=Wt[t + ".attn1.out.b"], res=hs, stats_out=stats)
                    P.gemm(hs, Wt[t + ".attn2.q.w"], C, 1, 1, M, q, ln=ln_of(t, ".attn2.q"))
                    P.attention(q, kv, kv, att, B, heads, S, 77, 0, 0, C, cfg.head_dim ** -0.5)
                    P.gemm(att, Wt[t + ".attn2.out.w"], C, 1, 1, M, hs, bias=Wt[t + ".attn2.out.b"], res=hs, stats_out=stats)
                    P.gemm(hs, Wt[t + ".ff.in.w"], 8 * C, 1, 1, M, gg, mode=geglu_mode, ln=ln_of(t, ".ff.in"))
                    P.gemm(gg, Wt[t + ".ff.out.w"], C, 1, 1, M, hs, bias=Wt[t + ".ff.out.b"], res=hs, stats_out=stats)
                    continue
                ln = scratch("ln", M, C)
                P.layernorm(hs, Wt[t + ".norm1.g"], Wt[t + ".norm1.b"], 1e-5, ln)
                P.gemm(ln, Wt[t + ".attn1.qkv.w"], 3 * C, 1, 1, M, qkv)
                P.attention(qkv, qkv, qkv, att, B, heads, S, S, 0, C, 2 * C, cfg.head_dim ** -0.5)
                P.gemm(att, Wt[t + ".attn1.out.w"], C, 1, 1, M, hs, bias=Wt[t + ".attn1.out.b"], res=hs)
                P.layernorm(hs, Wt[t + ".norm2.g"], Wt[t + ".norm2.b"], 1e-5, ln)
                P.gemm(ln, Wt[t + ".attn2.q.w"], C, 1, 1, M, q)
                P.attention(q, kv, kv, att, B, heads, S, 77, 0, 0, C, cfg.head_dim ** -0.5)
                P.gemm(att, Wt[t + ".attn2.out.w"], C, 1, 1, M, hs, bias=Wt[t + ".attn2.out.b"], res=hs)
                P.layernorm(hs, Wt[t + ".norm3.g"], Wt[t + ".norm3.b"], 1e-5, ln)
                P.gemm(ln, Wt[t + ".ff.in.w"], 8 * C, 1, 1, M, gg, bias=Wt[t + ".ff.in.b"], mode=geglu_mode)
                P.gemm(gg, Wt[t + ".ff.out.w"], C, 1, 1, M, hs, bias=Wt[t + ".ff.out.b"], res=hs)
            P.gemm(hs, Wt[aname + ".proj_out.w"], C, 1, 1, M, out, bias=Wt[aname + ".proj_out.b"], res=x)

        # ---- down path ----------------------------------------------------------------------
        si = 0
        P.conv_in(self.x_in, Wt["conv_in.w"], Wt["conv_in.b"], ch[0], skip_views[si])
        x, cin = skip_views[si], ch[0]
        si += 1
        for i in range(L):
            cout = ch[i]
            for j in range(cfg.layers_per_block):
                rname = f"down_blocks.{i}.resnets.{j}"
                dst = skip_views[si]
                if cfg.transformer_layers[i]:
                    r_out = persist(rows_at(i), cout)
                    resnet(rname, x, cin, cout, i, r_out)
                    transformer(f"down_blocks.{i}.attentions.{j}", r_out, cout, i, dst)
                else:
                    resnet(rname, x, cin, cout, i, dst)
                x, cin = dst, cout
                si += 1
            if i < L - 1:
                nm = f"down_blocks.{i}.downsamplers.0.conv"
                h_, w_ = res_hw[i]
                cols = scratch("im2col", rows_at(i + 1), 9 * cout)
                P.im2col_s2(x, B, h_, w_, cout, cols)
                dst = skip_views[si]
                P.gemm(cols, Wt[nm + ".w"], cout, 1, 1, rows_at(i + 1), dst, bias=Wt[nm + ".b"])
                x = dst
                si += 1
        # ---- mid ----------------------------------------------------------------------------
        lv, cm = L - 1, ch[-1]
        m1 = persist(rows_at(lv), cm)
        resnet("mid_block.resnets.0", x, cm, cm, lv, m1)
        m2 = persist(rows_at(lv), cm)
        transformer("mid_block.attentions.0", m1, cm, lv, m2)
        resnet("mid_block.resnets.1", m2, cm, cm, lv, cats[0]["hidden"])
        # ---- up path ------------------------------------------------------------------------
        ci = 0
        rev_depth = list(reversed(cfg.transformer_layers))
        for i in range(L):
            cout = rev[i]
            lvl = L - 1 - i
            n_res = cfg.layers_per_block + 1
            for j in range(n_res):
                cat = cats[ci]
                cin_total = cat["buf"].shape[1]
                last_of_block = j == n_res - 1
                last_overall = last_of_block and i == L - 1
                if last_overall:
                    dst = persist(rows_at(lvl), cout)
                elif last_of_block:
                    dst = persist(rows_at(lvl), cout)          # goes through the upsampler
                else:
                    dst = cats[ci + 1]["hidden"]
                rname = f"up_blocks.{i}.resnets.{j}"
                if rev_depth[i]:
                    r_out = persist(rows_at(lvl), cout)
                    resnet(rname, cat["buf"], cin_total, cout, lvl, r_out)
                    transformer(f"up_blocks.{i}.attentions.{j}", r_out, cout, lvl, dst)
                else:
                    resnet(rname, cat["buf"], cin_total, cout, lvl, dst)
                ci += 1
                x = dst
            if i < L - 1:
                nm = f"up_blocks.{i}.upsamplers.0.conv"
                h_, w_ = res_hw[lvl]
                ho, wo = res_hw[lvl - 1]
                up = scratch("up", rows_at(lvl - 1), cout)
                P.upsample_nearest(x, B, h_, w_, cout, up, ho, wo)
                P.gemm(up, Wt[nm + ".w"], cout, B, ho, wo, cats[ci]["hidden"], taps=9, bias=Wt[nm + ".b"])
        # ---- out ----------------------------------------------------------------------------
        no = scratch("n1", rows_at(0), ch[0])
        P.groupnorm(x, B, H * W, ch[0], groups, Wt["conv_norm_out.g"], Wt["conv_norm_out.b"], 1e-5, 1, no, self.ws)
        lower_conv_out(P, Wt, no, B, H, W, ch[0], cfg.out_channels, self.eps, scratch)
        P.finalize()
        PC.finalize()
