"""Stock-PyTorch-on-the-same-GPU context arm: the same encode path written the way a PyTorch user would run it
on the GPU today — bf16 modules, cuBLAS `F.linear`, `F.scaled_dot_product_attention` (flash / cuDNN kernels), `F.layer_norm`,
batched over all pages — with none of this repo's kernels. It answers "how far are the hand-written sm_90a kernels ahead
of cuBLAS + library attention", which the CPU arm cannot. Same algorithm as the reference modules it restates
(`timm/models/vision_transformer.py:86-107,682-692`, `resampler.py:146-168`, `modeling_minicpm.py:824-1004`,
`dense_retrieval_model.py:170-225`); stronger than the reference's own loop, which runs the ViT page by page
(`modeling_minicpmv.py:95-122`). Restricted to the bench workload: every page is ONE slice of the same h x w and every
sequence has the same length (so batches need no padding mask).

`TorchPageEncoder(sd, cfg).encode(pixels_u8 [P,h,w,3] cuda, token_src [P*L] int32, L)` -> [P, H] fp32 embeddings.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

from visrag_b200.weights import sincos_2d


class TorchPageEncoder:
    def __init__(self, sd, cfg, dtype=torch.bfloat16):
        self.cfg, self.dt = cfg, dtype
        self.sd = {k: v.to(dtype) for k, v in sd.items()}
        self.dev = next(iter(self.sd.values())).device
        hd = cfg.head_dim
        inv = 1.0 / (cfg.rope_theta ** (torch.arange(0, hd, 2, device=self.dev).float() / hd))
        fr = torch.outer(torch.arange(cfg.max_pos, device=self.dev).float(), inv)
        emb = torch.cat([fr, fr], dim=-1)
        self.cos, self.sin = emb.cos().to(dtype), emb.sin().to(dtype)
        self._pos = {}

    def _vit_pos(self, gh, gw):
        key = (gh, gw)
        if key not in self._pos:
            pos = self.sd["vpm.pos_embed"].float()
            S = int(math.sqrt(pos.shape[1]))
            if not (gh == S and gw == S):
                p = pos.reshape(1, S, S, -1).permute(0, 3, 1, 2)
                p = F.interpolate(p, size=(gh, gw), mode="bicubic", antialias=True)
                pos = p.permute(0, 2, 3, 1).reshape(1, gh * gw, -1)
            rs = torch.from_numpy(sincos_2d(self.cfg.hidden, gh, gw)).to(self.dev, self.dt)
            self._pos[key] = (pos.to(self.dt), rs)
        return self._pos[key]

    @torch.no_grad()
    def vision(self, pixels_u8):
        sd, cfg, dt = self.sd, self.cfg, self.dt
        P, h, w, _ = pixels_u8.shape
        D, nh = cfg.vit_dim, cfg.vit_heads
        x = ((pixels_u8.permute(0, 3, 1, 2).float() / 255.0 - 0.5) / 0.5).to(dt)
        x = F.conv2d(x, sd["vpm.patch_embed.proj.weight"], sd["vpm.patch_embed.proj.bias"], stride=cfg.patch_size)
        gh, gw = x.shape[2], x.shape[3]
        N = gh * gw
        pos, rs_pos = self._vit_pos(gh, gw)
        x = x.flatten(2).transpose(1, 2) + pos
        for i in range(cfg.vit_depth):
            p = f"vpm.blocks.{i}."
            y = F.layer_norm(x, (D,), sd[p + "norm1.weight"], sd[p + "norm1.bias"], cfg.ln_eps)
            qkv = F.linear(y, sd[p + "attn.qkv.weight"], sd[p + "attn.qkv.bias"]).reshape(P, N, 3, nh, D // nh).permute(2, 0, 3, 1, 4)
            o = F.scaled_dot_product_attention(qkv[0], qkv[1], qkv[2]).transpose(1, 2).reshape(P, N, D)
            x = x + F.linear(o, sd[p + "attn.proj.weight"], sd[p + "attn.proj.bias"])
            y = F.layer_norm(x, (D,), sd[p + "norm2.weight"], sd[p + "norm2.bias"], cfg.ln_eps)
            y = F.gelu(F.linear(y, sd[p + "mlp.fc1.weight"], sd[p + "mlp.fc1.bias"]))
            x = x + F.linear(y, sd[p + "mlp.fc2.weight"], sd[p + "mlp.fc2.bias"])
        x = F.layer_norm(x, (D,), sd["vpm.norm.weight"], sd["vpm.norm.bias"], cfg.ln_eps)
        # resampler (nn.MultiheadAttention math, 64 learned queries shared by all pages)
        E = cfg.hidden
        rh = E // 128
        kv = F.layer_norm(F.linear(x, sd["resampler.kv_proj.weight"]), (E,), sd["resampler.ln_kv.weight"], sd["resampler.ln_kv.bias"], 1e-6)
        q_in = F.layer_norm(sd["resampler.query"], (E,), sd["resampler.ln_q.weight"], sd["resampler.ln_q.bias"], 1e-6) + sd["resampler.pos_embed"]
        W, b = sd["resampler.attn.in_proj_weight"], sd["resampler.attn.in_proj_bias"]
        q = F.linear(q_in, W[:E], b[:E]).reshape(1, -1, rh, 128).transpose(1, 2).expand(P, -1, -1, -1)
        k = F.linear(kv + rs_pos, W[E:2 * E], b[E:2 * E]).reshape(P, N, rh, 128).transpose(1, 2)
        v = F.linear(kv, W[2 * E:], b[2 * E:]).reshape(P, N, rh, 128).transpose(1, 2)
        o = F.scaled_dot_product_attention(q, k, v).transpose(1, 2).reshape(P, -1, E)
        o = F.linear(o, sd["resampler.attn.out_proj.weight"], sd["resampler.attn.out_proj.bias"])
        o = F.layer_norm(o, (E,), sd["resampler.ln_post.weight"], sd["resampler.ln_post.bias"], 1e-6)
        return o @ sd["resampler.proj"]  # [P, 64, E]

    @staticmethod
    def _rms(x, w, eps):
        var = x.float().pow(2).mean(-1, keepdim=True)
        return (x.float() * torch.rsqrt(var + eps)).to(x.dtype) * w  # MiniCPMRMSNorm: fp32 statistics, weight in model dtype

    @torch.no_grad()
    def lm(self, h):
        sd, cfg = self.sd, self.cfg
        P, L, H = h.shape
        nh, hd = cfg.heads, cfg.head_dim
        cos, sin = self.cos[:L], self.sin[:L]
        s = cfg.depth_scale

        def rot(x):
            return torch.cat([-x[..., hd // 2:], x[..., : hd // 2]], dim=-1)

        for i in range(cfg.layers):
            p = f"llm.model.layers.{i}."
            a = self._rms(h, sd[p + "input_layernorm.weight"], cfg.rms_eps)
            q = F.linear(a, sd[p + "self_attn.q_proj.weight"]).reshape(P, L, nh, hd).transpose(1, 2)
            k = F.linear(a, sd[p + "self_attn.k_proj.weight"]).reshape(P, L, nh, hd).transpose(1, 2)
            v = F.linear(a, sd[p + "self_attn.v_proj.weight"]).reshape(P, L, nh, hd).transpose(1, 2)
            q = q * cos + rot(q) * sin
            k = k * cos + rot(k) * sin
            o = F.scaled_dot_product_attention(q, k, v, is_causal=True).transpose(1, 2).reshape(P, L, H)
            h = h + F.linear(o, sd[p + "self_attn.o_proj.weight"]) * s
            m = self._rms(h, sd[p + "post_attention_layernorm.weight"], cfg.rms_eps)
            m = F.linear(F.silu(F.linear(m, sd[p + "mlp.gate_proj.weight"])) * F.linear(m, sd[p + "mlp.up_proj.weight"]),
                         sd[p + "mlp.down_proj.weight"])
            h = h + m * s
        return self._rms(h, sd["llm.model.norm.weight"], cfg.rms_eps)

    @torch.no_grad()
    def encode(self, pixels_u8, token_src, L):
        """token_src: the engine's packed source map (>= 0: vision row, < 0: -(token id + 1)), P sequences of length L."""
        cfg = self.cfg
        P = pixels_u8.shape[0]
        vis = self.vision(pixels_u8).reshape(P * cfg.query_num, cfg.hidden)
        src = token_src.to(torch.int64)
        is_vis = src >= 0
        tok = torch.where(is_vis, torch.zeros_like(src), -(src + 1))
        h = self.sd["llm.model.embed_tokens.weight"][tok] * cfg.scale_emb
        h[is_vis] = vis[src[is_vis]]
        hid = self.lm(h.reshape(P, L, cfg.hidden)).float()
        w = torch.arange(1, L + 1, device=hid.device, dtype=torch.float32)
        reps = (hid * w[None, :, None]).sum(1) / w.sum()
        return F.normalize(reps, dim=1)
