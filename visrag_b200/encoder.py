"""H100 engine for the VisRAG-Ret encode path: uint8 slices + packed tokens -> pooled fp32 embeddings.

Replaces the GPU work of `VisRAG_Ret.forward` (`modeling_visrag_ret.py:86-126`), `get_vllm_embedding`
(`modeling_minicpmv.py:124-171`), the timm ViT, the Resampler and `MiniCPMModel.forward`, plus the pooling of
`DRModel.encode` (`dense_retrieval_model.py:170-223`). Differences in *schedule* (never in math):
  * the ViT runs over ALL slices of a batch that share a geometry at once (the reference loops page by page
    with batch 1, `modeling_minicpmv.py:130-135`);
  * LM sequences are packed (cu_seqlens) instead of right-padded;
  * the residual streams stay fp32 in HBM; every GEMM reads 16-bit operands and accumulates in fp32 (registers).
    The 16-bit type is the engine's `dtype`: bf16 (the default) or fp16, the type of the reference's evaluation
    (`--dtype float16`). It applies to the weights and to every activation stored in 16 bits; the residual streams, biases,
    norm and softmax statistics, RoPE tables, pooling and the embeddings stay fp32 in both.
Every kernel is a C-ABI call (visrag_b200/ops.py); torch only owns the buffers.
"""
from __future__ import annotations

import functools
import os
from collections import OrderedDict
from typing import Dict, Optional, Sequence, Tuple

import numpy as np
import torch
import torch.nn.functional as F

from . import _lib as L
from . import ops
from .config import VisRAGConfig
from .host import PreparedBatch, prepare_batch, select_prefix, suffix_batch
from .weights import sincos_2d

VIT_HEAD_STRIDE = 80  # 72 padded to a multiple of 16 (the MMA K step); pad rows of Wqkv are zero
# The ViT MLP width is padded to a multiple of 64 (4304 -> 4352, the tiny config's 1008 -> 1024) with zero rows of fc1_w,
# zero fc1_b and zero columns of fc2_w: the fc1 output rows and fc2's operand rows then start on 128-byte lines (8608 B
# rows straddle them), and fc2's last k-block is full. The pad columns of the fc1 output are exactly +0 (0 + 0, GELU(0) =
# +0), so fc2 adds the same zeros TMA used to fill in past column 4304: the embeddings do not change by a bit.
VIT_MLP_ALIGN = 64

# CUDA-graph path (small batches): eligibility and cache bounds
GRAPH_MAX_VIT_TOKENS = 32 * 1024   # up to 32 slices of 448x448: beyond that the kernels are long enough to hide launches
GRAPH_MAX_LM_TOKENS = 4096
GRAPH_TEXT_BUCKET = 16             # text-only batches: total tokens and longest sequence are padded to multiples of this
GRAPH_CACHE = 12                   # captured graphs kept (LRU); each owns its activation buffers

PREFIX_CACHE = 4                   # prefix-cache entries kept (LRU); ~378 KB per prefix token at full size


class _GraphEntry:
    __slots__ = ("graph", "groups", "src", "pos", "cu", "reps", "launches")


class _PrefixEntry:
    """One cached token prefix: its ids, P = len(ids), the K|V columns of every layer's RoPE'd qkv rows kv [layers, P, 2H]
    (engine dtype) and the fp32 residual rows before the final norm h [P, H]. `serial` names it in graph signatures."""
    __slots__ = ("ids", "P", "kv", "h", "serial")


def _half(t: torch.Tensor, dev, dtype: torch.dtype) -> torch.Tensor:
    return t.to(device=dev, dtype=dtype).contiguous()


def _f32(t: torch.Tensor, dev) -> torch.Tensor:
    return t.to(device=dev, dtype=torch.float32).contiguous()


def _on_own_device(fn):
    """Run a VisRAGEngine method with the engine's device current (kernels launch on the current device's stream)."""

    @functools.wraps(fn)
    def wrapper(self, *args, **kwargs):
        with L.on_device(self.device):
            return fn(self, *args, **kwargs)

    return wrapper


class VisRAGEngine:
    """Holds device weights in kernel-ready layouts and runs the encode pipeline. Every public method makes the engine's
    own device current for its launches, so an engine on cuda:1 works while cuda:0 is the process's current device.
    `dtype` (torch.bfloat16 or torch.float16) is the type of the weights and of every 16-bit activation."""

    def __init__(self, cfg: VisRAGConfig, state_dict: Dict[str, torch.Tensor], device: str = "cuda:0",
                 max_vit_tokens: int = 131072, device_frontend: bool = True, cuda_graphs: Optional[bool] = None,
                 dtype: torch.dtype = torch.bfloat16, prefix_cache: bool = True):
        cfg.validate()
        if dtype not in ops.HALF_DTYPES:
            raise ValueError(f"VisRAGEngine: dtype must be torch.bfloat16 or torch.float16, got {dtype}")
        L.lib()  # fail loudly if the CUDA library is missing
        self.cfg = cfg
        self.dtype = dtype
        # True: pages travel as raw RGB and are resampled / cut into slices on the GPU (bit-identical to PIL,
        # frontend.py); False: PIL renders the slices on the host as the reference does
        self.device_frontend = device_frontend
        self.device = L.norm_device(device)
        self.max_vit_tokens = max_vit_tokens
        # Small batches are launch bound (one query = ~290 ctypes launches of a few microseconds each): their whole
        # device step is captured into a CUDA graph per shape signature and replayed (see _encode_graphed)
        self.cuda_graphs = (os.environ.get("VR_CUDA_GRAPHS", "1") != "0") if cuda_graphs is None else bool(cuda_graphs)
        self._graphs: "OrderedDict[tuple, _GraphEntry]" = OrderedDict()
        self._graph_seen: Dict[tuple, int] = {}
        self.graph_stats = {"captured": 0, "replayed": 0, "eager": 0}
        # Text-only batches whose items share a token prefix (every query starts with the same instruction) run only the
        # suffixes through the LM and read the prefix rows from this cache; the embeddings keep their bits (DESIGN §5).
        # tokens_skipped counts the LM tokens the full path would have computed and the cached path did not.
        self.prefix_cache = bool(prefix_cache)
        self._prefixes: "OrderedDict[tuple, _PrefixEntry]" = OrderedDict()
        self._prefix_serial = 0
        self.prefix_stats = {"created": 0, "hits": 0, "tokens_skipped": 0}
        with L.on_device(self.device):
            self._load(cfg, state_dict)

    def _load(self, cfg: VisRAGConfig, state_dict: Dict[str, torch.Tensor]) -> None:
        sd, dev, dt = state_dict, self.device, self.dtype
        D, E, H, I = cfg.vit_dim, cfg.hidden, cfg.hidden, cfg.inter
        nh, hd, hs = cfg.vit_heads, cfg.vit_head_dim, VIT_HEAD_STRIDE
        with torch.no_grad():
            # ---- ViT
            P2 = 3 * cfg.patch_size ** 2
            self.patch_k = ((P2 + 63) // 64) * 64  # 588 -> 640: TMA rows must be 16-byte multiples
            pw = sd["vpm.patch_embed.proj.weight"].float().reshape(D, P2)
            w = torch.zeros((D, self.patch_k), dtype=torch.float32, device=pw.device)
            w[:, :P2] = pw
            self.patch_w = _half(w, dev, dt)
            self.patch_b = _f32(sd["vpm.patch_embed.proj.bias"], dev)
            self.pos_embed = sd["vpm.pos_embed"].float().cpu()
            self._pos_cache: Dict[Tuple[int, int], torch.Tensor] = {}
            self._sincos_cache: Dict[Tuple[int, int], torch.Tensor] = {}
            self.blocks = []
            mlp = cfg.vit_mlp
            mlp_pad = -(-mlp // VIT_MLP_ALIGN) * VIT_MLP_ALIGN - mlp
            for i in range(cfg.vit_depth):
                p = f"vpm.blocks.{i}."
                wq = sd[p + "attn.qkv.weight"].float().reshape(3, nh, hd, D)
                bq = sd[p + "attn.qkv.bias"].float().reshape(3, nh, hd)
                wpad = torch.zeros((3, nh, hs, D), device=wq.device)
                bpad = torch.zeros((3, nh, hs), device=wq.device)
                wpad[:, :, :hd] = wq
                bpad[:, :, :hd] = bq
                self.blocks.append(dict(
                    n1w=_f32(sd[p + "norm1.weight"], dev), n1b=_f32(sd[p + "norm1.bias"], dev),
                    qkv_w=_half(wpad.reshape(3 * nh * hs, D), dev, dt), qkv_b=_f32(bpad.reshape(-1), dev),
                    proj_w=_half(sd[p + "attn.proj.weight"], dev, dt), proj_b=_f32(sd[p + "attn.proj.bias"], dev),
                    n2w=_f32(sd[p + "norm2.weight"], dev), n2b=_f32(sd[p + "norm2.bias"], dev),
                    fc1_w=_half(F.pad(sd[p + "mlp.fc1.weight"], (0, 0, 0, mlp_pad)), dev, dt),
                    fc1_b=_f32(F.pad(sd[p + "mlp.fc1.bias"], (0, mlp_pad)), dev),
                    fc2_w=_half(F.pad(sd[p + "mlp.fc2.weight"], (0, mlp_pad)), dev, dt), fc2_b=_f32(sd[p + "mlp.fc2.bias"], dev),
                ))
            self.vnorm_w, self.vnorm_b = _f32(sd["vpm.norm.weight"], dev), _f32(sd["vpm.norm.bias"], dev)
            # ---- Resampler
            self.rs_kv_w = _half(sd["resampler.kv_proj.weight"], dev, dt)
            self.rs_lnkv = (_f32(sd["resampler.ln_kv.weight"], dev), _f32(sd["resampler.ln_kv.bias"], dev))
            self.rs_lnpost = (_f32(sd["resampler.ln_post.weight"], dev), _f32(sd["resampler.ln_post.bias"], dev))
            Win, bin_ = sd["resampler.attn.in_proj_weight"].float(), sd["resampler.attn.in_proj_bias"].float()
            self.rs_wk, self.rs_bk = _half(Win[E:2 * E], dev, dt), _f32(bin_[E:2 * E], dev)
            self.rs_wv, self.rs_bv = _half(Win[2 * E:], dev, dt), _f32(bin_[2 * E:], dev)
            self.rs_wo, self.rs_bo = _half(sd["resampler.attn.out_proj.weight"], dev, dt), _f32(sd["resampler.attn.out_proj.bias"], dev)
            self.rs_projT = _half(sd["resampler.proj"].float().t(), dev, dt)  # y = x @ proj  ->  B operand = proj^T
            # the query side is input independent (`resampler.py:158-160`): Q = Wq (LN_q(query) + pos_8x8) + bq, once
            q_in = ops.layernorm(_f32(sd["resampler.query"], dev), _f32(sd["resampler.ln_q.weight"], dev),
                                 _f32(sd["resampler.ln_q.bias"], dev), 1e-6, add=_f32(sd["resampler.pos_embed"], dev), dtype=dt)[1]
            self.rs_q = torch.zeros((128, E), dtype=dt, device=dev)  # padded to one 128-row query tile
            ops.gemm(q_in, _half(Win[:E], dev, dt), bias=_f32(bin_[:E], dev), out=self.rs_q[: cfg.query_num])
            # ---- MiniCPM
            self.embed = _half(sd["llm.model.embed_tokens.weight"], dev, dt)
            self.layers = []
            for i in range(cfg.layers):
                p = f"llm.model.layers.{i}."
                wqkv = torch.cat([sd[p + f"self_attn.{n}_proj.weight"].float() for n in ("q", "k", "v")], dim=0)
                wg, wu = sd[p + "mlp.gate_proj.weight"].float(), sd[p + "mlp.up_proj.weight"].float()
                # rows interleaved in blocks of 32 so that gate_j and up_j land in the same epilogue thread
                wgu = torch.stack([wg.reshape(I // 32, 32, H), wu.reshape(I // 32, 32, H)], dim=1).reshape(2 * I, H)
                self.layers.append(dict(
                    in_w=_f32(sd[p + "input_layernorm.weight"], dev), post_w=_f32(sd[p + "post_attention_layernorm.weight"], dev),
                    qkv_w=_half(wqkv, dev, dt), o_w=_half(sd[p + "self_attn.o_proj.weight"], dev, dt),
                    gu_w=_half(wgu, dev, dt), down_w=_half(sd[p + "mlp.down_proj.weight"], dev, dt),
                ))
            self.final_w = _f32(sd["llm.model.norm.weight"], dev)
            inv = 1.0 / (cfg.rope_theta ** (torch.arange(0, cfg.head_dim, 2).float() / cfg.head_dim))
            fr = torch.outer(torch.arange(cfg.max_pos).float(), inv)  # `modeling_minicpm.py:142-182`
            self.rope_cos, self.rope_sin = _f32(fr.cos(), dev), _f32(fr.sin(), dev)
            torch.cuda.synchronize(dev)

    # ------------------------------------------------------------------------------------------ tables
    def _pos_table(self, gh: int, gw: int) -> torch.Tensor:
        """ViT position embedding resampled to (gh, gw): bicubic + antialias in fp32, once per distinct grid
        (`timm/layers/pos_embed.py:17-57`; the reference redoes it every forward)."""
        key = (gh, gw)
        if key not in self._pos_cache:
            S, D = self.cfg.vit_pos_grid, self.cfg.vit_dim
            if gh == S and gw == S:
                t = self.pos_embed[0]
            else:
                p = self.pos_embed.reshape(1, S, S, D).permute(0, 3, 1, 2)
                p = torch.nn.functional.interpolate(p, size=(gh, gw), mode="bicubic", antialias=True)
                t = p.permute(0, 2, 3, 1).reshape(gh * gw, D)
            self._pos_cache[key] = _f32(t, self.device)
        return self._pos_cache[key]

    def _sincos_table(self, gh: int, gw: int) -> torch.Tensor:
        key = (gh, gw)
        if key not in self._sincos_cache:
            self._sincos_cache[key] = _f32(torch.from_numpy(sincos_2d(self.cfg.hidden, gh, gw)), self.device)
        return self._sincos_cache[key]

    # ------------------------------------------------------------------------------------------ vision
    @_on_own_device
    def vit_tokens(self, pixels: torch.Tensor) -> torch.Tensor:
        """uint8 [S,h,w,3] (device) -> final-LayerNorm ViT tokens [S*N, D] in the engine's dtype."""
        cfg, dt = self.cfg, self.dtype
        S, h, w, _ = pixels.shape
        gh, gw = h // cfg.patch_size, w // cfg.patch_size
        N, D, nh = gh * gw, cfg.vit_dim, cfg.vit_heads
        M = S * N
        a = ops.im2col_norm(pixels, cfg.patch_size, self.patch_k, dt)
        x = ops.gemm(a, self.patch_w, bias=self.patch_b, rowadd=self._pos_table(gh, gw), out_dtype=torch.float32)
        cu = torch.arange(0, (S + 1) * N, N, dtype=torch.int32, device=self.device)
        qkv = torch.empty((M, 3 * nh * VIT_HEAD_STRIDE), dtype=dt, device=self.device)
        att = torch.empty((M, D), dtype=dt, device=self.device)
        scale = cfg.vit_head_dim ** -0.5
        for blk in self.blocks:
            y = ops.layernorm(x, blk["n1w"], blk["n1b"], cfg.ln_eps, dtype=dt)
            ops.gemm(y, blk["qkv_w"], bias=blk["qkv_b"], out=qkv)
            ops.attention(qkv, qkv, qkv, q_col0=0, k_col0=nh * VIT_HEAD_STRIDE, v_col0=2 * nh * VIT_HEAD_STRIDE,
                          head_stride=VIT_HEAD_STRIDE, head_dim=cfg.vit_head_dim, heads=nh, batch=S, cu_k=cu, max_k=N,
                          cu_q=cu, max_q=N, causal=False, scale=scale, out=att)
            ops.gemm(att, blk["proj_w"], bias=blk["proj_b"], resid=x, out=x, out_dtype=torch.float32)
            y = ops.layernorm(x, blk["n2w"], blk["n2b"], cfg.ln_eps, dtype=dt)
            y = ops.gemm(y, blk["fc1_w"], bias=blk["fc1_b"], gelu=True)
            ops.gemm(y, blk["fc2_w"], bias=blk["fc2_b"], resid=x, out=x, out_dtype=torch.float32)
        return ops.layernorm(x, self.vnorm_w, self.vnorm_b, cfg.ln_eps, dtype=dt)

    @_on_own_device
    def resample(self, tokens: torch.Tensor, S: int, gh: int, gw: int, out: torch.Tensor) -> None:
        """ViT tokens [S*N, D] (engine dtype) -> 64 query tokens per slice, written to fp32 `out` [S*64, E]."""
        cfg, dt = self.cfg, self.dtype
        E, N, nh = cfg.hidden, gh * gw, cfg.rs_heads
        kv = ops.gemm(tokens, self.rs_kv_w, out_dtype=torch.float32)
        v_in, k_in = ops.layernorm(kv, self.rs_lnkv[0], self.rs_lnkv[1], 1e-6, add=self._sincos_table(gh, gw), dtype=dt)
        k = ops.gemm(k_in, self.rs_wk, bias=self.rs_bk)
        v = ops.gemm(v_in, self.rs_wv, bias=self.rs_bv)
        cu = torch.arange(0, (S + 1) * N, N, dtype=torch.int32, device=self.device)
        att = torch.empty((S * cfg.query_num, E), dtype=dt, device=self.device)
        ops.attention(self.rs_q, k, v, q_col0=0, k_col0=0, v_col0=0, head_stride=128, head_dim=128, heads=nh, batch=S,
                      cu_k=cu, max_k=N, cu_q=None, max_q=cfg.query_num, causal=False, scale=128 ** -0.5, out=att)
        o = ops.gemm(att, self.rs_wo, bias=self.rs_bo, out_dtype=torch.float32)
        o = ops.layernorm(o, self.rs_lnpost[0], self.rs_lnpost[1], 1e-6, dtype=dt)
        ops.gemm(o, self.rs_projT, out=out, out_dtype=torch.float32)

    @_on_own_device
    def encode_vision(self, groups: Dict[Tuple[int, int], torch.Tensor], group_row0: Dict[Tuple[int, int], int],
                      n_slices: int) -> Optional[torch.Tensor]:
        """All slices of a batch -> fp32 [n_slices*64, E] (slice i occupies rows 64i..64i+63)."""
        if n_slices == 0:
            return None
        cfg = self.cfg
        out = torch.empty((n_slices * cfg.query_num, cfg.hidden), dtype=torch.float32, device=self.device)
        for (h, w), px in groups.items():
            gh, gw = h // cfg.patch_size, w // cfg.patch_size
            per = max(1, self.max_vit_tokens // (gh * gw))
            for s0 in range(0, px.shape[0], per):
                chunk = px[s0:s0 + per]
                S = chunk.shape[0]
                r0 = (group_row0[(h, w)] + s0) * cfg.query_num
                self.resample(self.vit_tokens(chunk), S, gh, gw, out[r0:r0 + S * cfg.query_num])
        return out

    # ------------------------------------------------------------------------------------------ LM
    @_on_own_device
    def lm_hidden(self, token_src: torch.Tensor, positions: torch.Tensor, cu: torch.Tensor, max_len: int,
                  vision: Optional[torch.Tensor], prefix: Optional[_PrefixEntry] = None,
                  cu_full: Optional[torch.Tensor] = None, kv_out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Packed decoder: returns the fp32 residual stream BEFORE the final RMSNorm, [T, H].
        With `prefix`, the rows are the suffixes of sequences that start with the prefix's P tokens (positions stay
        absolute, cu / max_len count suffix tokens); every layer attends over [prefix K|V ; own K|V] laid out as the full
        sequences cu_full, and the result is the full sequences' residual stream [T + B*P, H]. `kv_out` [layers, T, 2H]
        receives every layer's K|V columns (how a prefix entry is built)."""
        cfg, dt = self.cfg, self.dtype
        H, nh = cfg.hidden, cfg.heads
        B = cu.shape[0] - 1
        h = ops.build_lm_input(token_src, self.embed, cfg.scale_emb, vision)
        T = h.shape[0]
        qkv = torch.empty((T, 3 * H), dtype=dt, device=self.device)
        att = torch.empty((T, H), dtype=dt, device=self.device)
        if prefix is not None:
            kv = torch.empty((T + B * prefix.P, 2 * H), dtype=dt, device=self.device)
        s = cfg.depth_scale
        for i, lyr in enumerate(self.layers):
            a = ops.rmsnorm(h, lyr["in_w"], cfg.rms_eps, dt)
            ops.gemm(a, lyr["qkv_w"], mode=L.VR_EPI_ROPE, positions=positions, rope_cos=self.rope_cos,
                     rope_sin=self.rope_sin, rope_cols=2 * H, out=qkv)
            if kv_out is not None:
                kv_out[i].copy_(qkv[:, H:])
            if prefix is None:
                ops.attention(qkv, qkv, qkv, q_col0=0, k_col0=H, v_col0=2 * H, head_stride=64, head_dim=64, heads=nh,
                              batch=B, cu_k=cu, max_k=max_len, cu_q=cu, max_q=max_len, causal=True,
                              scale=cfg.head_dim ** -0.5, out=att)
            else:
                ops.prefix_rows(prefix.kv[i], qkv[:, H:], kv, cu, cu_full)
                ops.attention(qkv, kv, kv, q_col0=0, k_col0=0, v_col0=H, head_stride=64, head_dim=64, heads=nh, batch=B,
                              cu_k=cu_full, max_k=max_len + prefix.P, cu_q=cu, max_q=max_len, causal=True,
                              scale=cfg.head_dim ** -0.5, out=att)
            ops.gemm(att, lyr["o_w"], resid=h, out=h, scale=s, out_dtype=torch.float32)
            a = ops.rmsnorm(h, lyr["post_w"], cfg.rms_eps, dt)
            a = ops.gemm(a, lyr["gu_w"], mode=L.VR_EPI_SWIGLU)
            ops.gemm(a, lyr["down_w"], resid=h, out=h, scale=s, out_dtype=torch.float32)
        if prefix is None:
            return h
        return ops.prefix_rows(prefix.h, h, torch.empty((kv.shape[0], H), dtype=torch.float32, device=self.device), cu, cu_full)

    # ------------------------------------------------------------------------------------------ end to end
    def _pinned_buf(self, key, n: int, dtype) -> torch.Tensor:
        """Persistent (grow-only) pinned staging buffer identified by `key`."""
        buf = self._pinned.get(key)
        if buf is None or buf.numel() < n or buf.dtype != dtype:
            buf = torch.empty(max(n, 1), dtype=dtype).pin_memory()
            self._pinned[key] = buf
        return buf[:n]

    def _stage(self, a: np.ndarray, key) -> torch.Tensor:
        """numpy -> device through pinned staging; the copy is enqueued on the CURRENT stream (the caller selects it)."""
        t = torch.from_numpy(np.ascontiguousarray(a))
        stage = self._pinned_buf(key, t.numel(), t.dtype).view(t.shape)
        stage.copy_(t)
        return stage.to(self.device, non_blocking=True)

    def _stage_slices(self, slices, key) -> torch.Tensor:
        """List of S uint8 [h,w,3] arrays -> device [S,h,w,3], copied slice by slice into the pinned staging buffer."""
        h, w, c = slices[0].shape
        stage = self._pinned_buf(key, len(slices) * h * w * c, torch.uint8).view(len(slices), h, w, c)
        dst = stage.numpy()
        for j, a in enumerate(slices):
            dst[j] = a
        return stage.to(self.device, non_blocking=True)

    def _upload_group(self, key, slices, s: int) -> torch.Tensor:
        """One geometry group -> device [S,h,w,3]; entries rendered by the device front-end (None) are left to it."""
        host = [i for i, a in enumerate(slices) if a is not None]
        if len(host) == len(slices):
            return self._stage_slices(slices, (s, "px", key))
        dev = torch.empty((len(slices), key[0], key[1], 3), dtype=torch.uint8, device=self.device)
        if host:
            dev[torch.tensor(host, device=self.device)] = self._stage_slices([slices[i] for i in host], (s, "px", key))
        return dev

    def _render_jobs(self, jobs, groups, s: int) -> None:
        """Device front-end: raw pages (stacked per page size) -> thumbnails and grid cells, written into `groups`."""
        from .frontend import DeviceFrontEnd

        if not hasattr(self, "_frontend"):
            self._frontend = DeviceFrontEnd(self.device)
        by_size = {}
        for j in jobs:
            by_size.setdefault(j.pixels.shape, []).append(j)  # (H, W, 3 | 4): RGB and RGBX pages are stacked apart
        for (H, W, ps), lst in by_size.items():
            pages = self._stage_slices([j.pixels for j in lst], (s, "page", (H, W, ps)))
            plan = lst[0].plan  # a function of (W, H) only
            tkey = lst[0].thumb[0]
            first = self._stage(np.asarray([j.thumb[1] for j in lst], dtype=np.int32), (s, "first_t", (H, W, ps)))
            self._frontend.resize_into(pages, plan.source_size[0], plan.source_size[1], groups[tkey], first,
                                       plan.source_size[0], plan.source_size[1])
            if plan.grid is not None:
                ckey = lst[0].cells[0]
                first = self._stage(np.asarray([j.cells[1] for j in lst], dtype=np.int32), (s, "first_c", (H, W, ps)))
                self._frontend.resize_into(pages, plan.refine_size[0], plan.refine_size[1], groups[ckey], first,
                                           plan.cell_size[0], plan.cell_size[1])
            pages.record_stream(torch.cuda.current_stream(self.device))

    @_on_own_device
    def upload(self, pb: PreparedBatch):
        """Host -> device copies of one prepared batch. Pinned staging is double buffered and the copies run on a
        dedicated copy stream, so batch i+1 travels over PCIe while batch i's kernels run; the compute stream only
        waits on the copy's event. A staging set is reused every second upload, after its previous copy completed."""
        if not hasattr(self, "_pinned"):
            self._pinned, self._upload_done, self._flip = {}, [None, None], 0
            self._copy_stream = torch.cuda.Stream(device=self.device)
        s = self._flip
        self._flip ^= 1
        if self._upload_done[s] is not None:
            self._upload_done[s].synchronize()
        compute = torch.cuda.current_stream(self.device)
        with torch.cuda.stream(self._copy_stream):
            groups = {k: self._upload_group(k, v, s) for k, v in pb.groups.items()}
            if pb.jobs:
                self._render_jobs(pb.jobs, groups, s)
            out = (groups, self._stage(pb.token_src, (s, "src")), self._stage(pb.positions, (s, "pos")),
                   self._stage(pb.cu_seqlens, (s, "cu")))
            ev = torch.cuda.Event()
            ev.record()
        self._upload_done[s] = ev
        compute.wait_event(ev)
        for t in (*groups.values(), *out[1:]):
            t.record_stream(compute)  # allocated on the copy stream, consumed (and later freed) under the compute stream
        return out

    @_on_own_device
    def encode_device(self, groups, group_row0, n_slices: int, src, pos, cu, max_len: int, pooling: str = "wmean",
                      normalize: bool = True, return_hidden: bool = False, prefix: Optional[_PrefixEntry] = None):
        """Inputs already in HBM -> pooled embeddings [B, hidden] fp32 (the device-resident hot path).
        With `prefix` (text only) src / pos / max_len describe the suffixes, and cu is [cu_suffix ; cu_full], 2 (B+1)
        offsets (one upload); the hidden rows returned are the full sequences'."""
        vision = self.encode_vision(groups, group_row0, n_slices)
        cu_full = None
        if prefix is not None:
            n = cu.shape[0] // 2
            cu, cu_full = cu[:n], cu[n:]
        h = self.lm_hidden(src, pos, cu, max_len, vision, prefix, cu_full)
        reps = ops.pool_norm(h, self.final_w, self.cfg.rms_eps, cu if prefix is None else cu_full, pooling, normalize)
        return (reps, h) if return_hidden else reps

    # ------------------------------------------------------------------------------------------ CUDA graphs
    def _graph_plan(self, pb: PreparedBatch, prefix_len: int = 0):
        """Decide whether this batch takes the graph path; text-only batches are padded into shape buckets with ONE extra
        dummy sequence (token 0, dropped after pooling) so that different queries share a captured graph.
        With prefix_len, pb holds the suffixes of a cached-prefix batch and the dummy is prefix + pad tokens (positions
        from prefix_len on). Returns (token_src, positions, cu_seqlens, max_len, n_out) or None."""
        if not self.cuda_graphs or pb.n_items == 0:
            return None
        T = int(pb.cu_seqlens[-1])
        max_len = int(pb.seq_lens.max())
        vit_tokens = sum(len(v) * (k[0] // self.cfg.patch_size) * (k[1] // self.cfg.patch_size) for k, v in pb.groups.items())
        if vit_tokens > GRAPH_MAX_VIT_TOKENS or T > GRAPH_MAX_LM_TOKENS:
            return None
        if pb.n_slices > 0:
            return pb.token_src, pb.positions, pb.cu_seqlens, max_len, pb.n_items
        b = GRAPH_TEXT_BUCKET
        Tb = -(-(T + 1) // b) * b          # at least one pad token: the dummy sequence is never empty
        pad = Tb - T
        Lb = min(-(-max(max_len, pad) // b) * b, self.cfg.max_pos)
        if prefix_len + pad > self.cfg.max_pos:
            return None
        src = np.concatenate([pb.token_src, np.full(pad, -1, dtype=np.int32)])        # -(0 + 1): token id 0
        pos = np.concatenate([pb.positions, np.arange(prefix_len, prefix_len + pad, dtype=np.int32)])
        cu = np.concatenate([pb.cu_seqlens, np.asarray([Tb], dtype=np.int32)])
        return src, pos, cu, Lb, pb.n_items

    def _encode_graphed(self, sig, groups, group_row0, n_slices, src, pos, cu, max_len, pooling, normalize, prefix=None):
        """Replay (or, on the second sighting of a signature, capture) the device step for this shape. The first sighting
        runs eagerly: it also warms every per-shape table and one-time kernel attribute the capture must not touch."""
        ent = self._graphs.get(sig)
        if ent is None:
            seen = self._graph_seen.get(sig, 0)
            if len(self._graph_seen) > 4096:  # a stream of never-repeating shapes must not grow this without bound
                self._graph_seen.clear()
            self._graph_seen[sig] = seen + 1
            if seen == 0:
                self.graph_stats["eager"] += 1
                return self.encode_device(groups, group_row0, n_slices, src, pos, cu, max_len, pooling, normalize, prefix=prefix)
            if seen < 0:  # an earlier capture of this shape failed: stay on eager launches
                self.graph_stats["eager"] += 1
                return self.encode_device(groups, group_row0, n_slices, src, pos, cu, max_len, pooling, normalize, prefix=prefix)
            ent = _GraphEntry()
            ent.groups = {k: v.clone() for k, v in groups.items()}
            ent.src, ent.pos, ent.cu = src.clone(), pos.clone(), cu.clone()
            launches0 = L.LAUNCHES
            torch.cuda.synchronize(self.device)
            ent.graph = torch.cuda.CUDAGraph()
            try:
                with torch.cuda.graph(ent.graph):
                    ent.reps = self.encode_device(ent.groups, group_row0, n_slices, ent.src, ent.pos, ent.cu, max_len, pooling, normalize,
                                                   prefix=prefix)
            except Exception as exc:  # the capture is an optimisation of the launch path only: same kernels, eager launches
                import warnings

                warnings.warn(f"visrag_b200: CUDA-graph capture failed for this batch shape ({exc!r}); using eager launches")
                self._graph_seen[sig] = -(1 << 30)
                self.graph_stats["eager"] += 1
                return self.encode_device(groups, group_row0, n_slices, src, pos, cu, max_len, pooling, normalize, prefix=prefix)
            ent.launches = L.LAUNCHES - launches0
            self._graphs[sig] = ent
            self.graph_stats["captured"] += 1
            while len(self._graphs) > GRAPH_CACHE:
                self._graphs.popitem(last=False)
        else:
            self._graphs.move_to_end(sig)
            for k, v in groups.items():
                ent.groups[k].copy_(v, non_blocking=True)
            ent.src.copy_(src, non_blocking=True)
            ent.pos.copy_(pos, non_blocking=True)
            ent.cu.copy_(cu, non_blocking=True)
        ent.graph.replay()
        L.LAUNCHES += ent.launches  # the kernels of the captured step launch again (the counter is the bench's claim)
        self.graph_stats["replayed"] += 1
        return ent.reps.clone()

    @_on_own_device
    def encode_prepared(self, pb: PreparedBatch, pooling: str = "wmean", normalize: bool = True,
                        return_hidden: bool = False):
        if pb.n_items == 0:
            return torch.zeros((0, self.cfg.hidden), dtype=torch.float32, device=self.device)
        if int(pb.seq_lens.max()) > self.cfg.max_pos:
            raise ValueError(f"sequence longer than max_pos={self.cfg.max_pos}")
        ent = self._prefix_for(pb) if self.prefix_cache else None
        if ent is not None:
            return self._encode_suffixes(pb, ent, pooling, normalize, return_hidden)
        plan = None if return_hidden or ops.profiling() else self._graph_plan(pb)
        if plan is not None:
            src_h, pos_h, cu_h, max_len, n_out = plan
            shaped = PreparedBatch(pb.n_items, pb.seq_lens, cu_h, pos_h, src_h, pb.groups, pb.group_row0, pb.n_slices, pb.jobs)
            groups, src, pos, cu = self.upload(shaped)
            sig = (tuple(sorted((k, v.shape[0]) for k, v in groups.items())), tuple(sorted(pb.group_row0.items())), pb.n_slices,
                   int(src.shape[0]), int(cu.shape[0]), max_len, pooling, bool(normalize))
            reps = self._encode_graphed(sig, groups, pb.group_row0, pb.n_slices, src, pos, cu, max_len, pooling, normalize)
            return reps[:n_out]
        groups, src, pos, cu = self.upload(pb)
        return self.encode_device(groups, pb.group_row0, pb.n_slices, src, pos, cu, int(pb.seq_lens.max()), pooling,
                                  normalize, return_hidden)

    # ------------------------------------------------------------------------------------------ prefix cache
    def _prefix_for(self, pb: PreparedBatch) -> Optional[_PrefixEntry]:
        """The cache entry this batch runs from (host.select_prefix), created now if the batch calls for a new one;
        None -> the full path. Runs on the caller's thread: the cache is not shared with prepare()'s workers."""
        sel = select_prefix(pb, list(self._prefixes))
        if sel is None:
            return None
        ids, new = sel
        if new:
            ent = self._make_prefix(ids)
            self._prefixes[ids] = ent
            self.prefix_stats["created"] += 1
            self.prefix_stats["tokens_skipped"] += ent.P * (pb.n_items - 1)  # the prefix itself ran once
            while len(self._prefixes) > PREFIX_CACHE:
                _, old = self._prefixes.popitem(last=False)
                for sig in [s for s in self._graphs if s[-1] == ("prefix", old.serial)]:  # they bake its buffers
                    del self._graphs[sig]
        else:
            ent = self._prefixes[ids]
            self._prefixes.move_to_end(ids)
            self.prefix_stats["hits"] += 1
            self.prefix_stats["tokens_skipped"] += ent.P * pb.n_items
        return ent

    def _make_prefix(self, ids: Tuple[int, ...]) -> _PrefixEntry:
        """Run the prefix's tokens as one sequence through the same kernels (eagerly, never captured) and keep every
        layer's K|V rows and the residual rows before the final norm."""
        cfg, dev = self.cfg, self.device
        ent = _PrefixEntry()
        ent.ids, ent.P = ids, len(ids)
        self._prefix_serial += 1
        ent.serial = self._prefix_serial
        src = torch.tensor([-(i + 1) for i in ids], dtype=torch.int32, device=dev)
        pos = torch.arange(ent.P, dtype=torch.int32, device=dev)
        cu = torch.tensor([0, ent.P], dtype=torch.int32, device=dev)
        ent.kv = torch.empty((cfg.layers, ent.P, 2 * cfg.hidden), dtype=self.dtype, device=dev)
        ent.h = self.lm_hidden(src, pos, cu, ent.P, None, kv_out=ent.kv)
        return ent

    def _encode_suffixes(self, pb: PreparedBatch, ent: _PrefixEntry, pooling: str, normalize: bool, return_hidden: bool):
        """The cached-prefix path: only the suffix tokens run through the LM; the prefix rows come from `ent`. Small
        batches replay CUDA graphs bucketed on the suffixes as _graph_plan does, one graph per shape and entry."""
        sb = suffix_batch(pb, ent.P)
        plan = None if return_hidden or ops.profiling() else self._graph_plan(sb, ent.P)
        if plan is None:
            src_h, pos_h, cu_h, max_len, n_out = sb.token_src, sb.positions, sb.cu_seqlens, int(sb.seq_lens.max()), pb.n_items
        else:
            src_h, pos_h, cu_h, max_len, n_out = plan
        cu_full = cu_h + ent.P * np.arange(len(cu_h), dtype=np.int32)
        _, src, pos, cu = self.upload(PreparedBatch(pb.n_items, sb.seq_lens, np.concatenate([cu_h, cu_full]), pos_h, src_h))
        if plan is None:
            return self.encode_device({}, {}, 0, src, pos, cu, max_len, pooling, normalize, return_hidden, prefix=ent)
        sig = ((), (), 0, int(src.shape[0]), int(cu.shape[0]), max_len, pooling, bool(normalize), ("prefix", ent.serial))
        return self._encode_graphed(sig, {}, {}, 0, src, pos, cu, max_len, pooling, normalize, prefix=ent)[:n_out]

    @_on_own_device
    def encode(self, texts: Sequence[str], images: Sequence, tokenizer, max_inp_length: Optional[int] = 2048,
               pooling: str = "wmean", normalize: bool = True) -> torch.Tensor:
        """(texts, PIL images | None) -> fp32 device tensor [B, hidden], L2-normalised."""
        pb = prepare_batch(texts, images, tokenizer, self.cfg, max_inp_length, self.device_frontend)
        return self.encode_prepared(pb, pooling, normalize)
