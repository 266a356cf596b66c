"""Drop-in classes with the reference's call signatures (SURVEY.md §8b), backed by the H100 engine.

  B1  `VisRAGRetB200.forward(text, image, tokenizer, vision_hidden_states=None, max_inp_length=2048, **kw)`
      == `VisRAG_Ret.forward` (`modeling_visrag_ret/modeling_visrag_ret.py:86-126`): returns an object with
      `.last_hidden_state [B, Lmax, H]` (right padded) and `.attention_mask [B, Lmax]`.
  B2  `DRModelForInference.forward(query=None, passage=None, **kw) -> DROutput(q_reps, p_reps)`,
      `encode_passage / encode_query -> (None, reps [B, H] fp32, L2-normalised)`, `encode(items, model, head, ...)`
      == `dense_retrieval_model.py:142-231,387-408`. When `lm_q` is a `VisRAGRetB200` the pooling + normalise
      run fused on the device (no padded hidden states are ever built).
Extra kwargs the reference passes down and the backbone ignores (`is_query`, `id`, `instruction`) are accepted.
"""
from __future__ import annotations

import json
import os
from dataclasses import dataclass
from typing import Dict, List, Optional

import torch

from . import ops
from .config import VisRAGConfig
from .encoder import VisRAGEngine
from .host import prepare_batch


@dataclass
class BaseModelOutputWithAttentionMask:
    last_hidden_state: torch.Tensor = None
    attention_mask: Optional[torch.Tensor] = None

    def __contains__(self, key):  # the reference probes `"attention_mask" in items_out`
        return getattr(self, key, None) is not None


@dataclass
class DROutput:
    q_reps: torch.Tensor = None
    p_reps: torch.Tensor = None
    loss: torch.Tensor = None
    scores: torch.Tensor = None
    accuracy: torch.Tensor = None


_VISION_ENCODERS = {  # timm model name -> (dim, blocks defined, heads, mlp); `vision_transformer.py:2612-2619`
    "vit_so400m_patch14_siglip_384": (1152, 27, 16, 4304),
}


def config_from_hf(d: dict) -> VisRAGConfig:
    """MiniCPM-V `config.json` -> VisRAGConfig (field names `configuration_minicpm.py:109-160,197-222`). The vision tower is
    named by `vision_encoder` (+ `drop_vision_last_layer`, `modeling_minicpmv.py:57-73`) in real checkpoints; synthetic ones
    written by `weights.save_checkpoint` carry explicit `vit_*` fields (reduced towers have no timm name)."""
    base = VisRAGConfig()
    if not d.get("slice_mode", True):
        # `prepare_context` emits ONE un-sliced image and a single placeholder when slice_mode is off
        # (`modeling_visrag_ret.py:57-84`); the packing code here always slices, so refuse rather than embed other tokens
        raise NotImplementedError("config.json has slice_mode=false: the un-sliced path of VisRAG_Ret.prepare_context is not implemented")
    if "vit_dim" not in d and d.get("vision_encoder") is not None:
        enc = d["vision_encoder"]
        if enc not in _VISION_ENCODERS:
            raise NotImplementedError(f"vision_encoder {enc!r}: only {sorted(_VISION_ENCODERS)} is supported")
        dim, depth, heads, mlp = _VISION_ENCODERS[enc]
        d = dict(d, vit_dim=dim, vit_depth=depth - (1 if d.get("drop_vision_last_layer", True) else 0), vit_heads=heads, vit_mlp=mlp)
    return VisRAGConfig(
        patch_size=d.get("patch_size", base.patch_size), query_num=d.get("query_num", base.query_num),
        hidden=d.get("hidden_size", base.hidden), layers=d.get("num_hidden_layers", base.layers),
        heads=d.get("num_attention_heads", base.heads), inter=d.get("intermediate_size", base.inter),
        vocab=d.get("vocab_size", base.vocab), scale_emb=float(d.get("scale_emb", base.scale_emb)),
        scale_depth=float(d.get("scale_depth", base.scale_depth)), rms_eps=float(d.get("rms_norm_eps", base.rms_eps)),
        rope_theta=float(d.get("rope_theta", base.rope_theta)), max_pos=d.get("max_position_embeddings", base.max_pos),
        scale_resolution=d.get("scale_resolution", base.scale_resolution), max_slice_nums=d.get("max_slice_nums", base.max_slice_nums),
        slice_mode=d.get("slice_mode", base.slice_mode),
        vit_dim=d.get("vit_dim", base.vit_dim), vit_depth=d.get("vit_depth", base.vit_depth),
        vit_heads=d.get("vit_heads", base.vit_heads), vit_mlp=d.get("vit_mlp", base.vit_mlp),
    )


def load_checkpoint(path: str) -> Dict[str, torch.Tensor]:
    """state_dict from a HF-style directory (*.safetensors or pytorch_model*.bin); names per SURVEY.md A.7."""
    sd: Dict[str, torch.Tensor] = {}
    st = sorted(f for f in os.listdir(path) if f.endswith(".safetensors"))
    if st:
        from safetensors.torch import load_file

        for f in st:
            sd.update(load_file(os.path.join(path, f)))
    else:
        bins = sorted(f for f in os.listdir(path) if f.startswith("pytorch_model") and f.endswith(".bin"))
        if not bins:
            raise FileNotFoundError(f"no *.safetensors / pytorch_model*.bin under {path}")
        for f in bins:
            sd.update(torch.load(os.path.join(path, f), map_location="cpu", weights_only=True))
    return sd


def is_float16(dtype) -> bool:
    """True for the reference's fp16 setting: torch.float16 (`torch_dtype=`) or "float16" (`--dtype float16`, what
    `DRModel.build` maps to torch.float16, `dense_retrieval_model.py:301-309`)."""
    return dtype is torch.float16 or dtype in ("float16", "fp16", "half", "torch.float16")


class VisRAGRetB200:
    """B1 boundary: the backbone (`lm_q`). `dtype` is the engine's 16-bit type: torch.bfloat16 (default) or torch.float16."""

    def __init__(self, cfg: VisRAGConfig, state_dict: Dict[str, torch.Tensor], device: str = "cuda:0",
                 dtype: torch.dtype = torch.bfloat16):
        self.config = cfg
        self.engine = VisRAGEngine(cfg, state_dict, device, dtype=dtype)
        self.device = self.engine.device
        self.dtype = self.engine.dtype
        self.training = False

    @classmethod
    def from_pretrained(cls, path: str, config=None, torch_dtype=None, attn_implementation=None, device: str = "cuda:0", **_):
        """torch_dtype=torch.float16 builds an fp16 engine (weights and 16-bit activations in fp16). Anything else -
        None, torch.bfloat16, torch.float32 - builds the bf16 engine: there is no fp32 encode path, so float32 runs bf16."""
        with open(os.path.join(path, "config.json")) as f:
            cfg = config_from_hf(json.load(f))
        if is_float16(torch_dtype):
            return cls(cfg, load_checkpoint(path), device, dtype=torch.float16)
        return cls(cfg, load_checkpoint(path), device)

    def eval(self):
        return self

    def to(self, *_a, **_k):
        return self

    def forward(self, text: List[str], image: List, tokenizer, vision_hidden_states=None, max_inp_length: int = 2048,
                **kwargs) -> BaseModelOutputWithAttentionMask:
        if vision_hidden_states is not None:
            raise NotImplementedError("precomputed vision_hidden_states are not forwarded by the reference either "
                                      "(`modeling_visrag_ret.py:106-111`)")
        eng = self.engine
        pb = prepare_batch(text, image, tokenizer, self.config, max_inp_length, eng.device_frontend)
        if pb.n_items and int(pb.seq_lens.max()) > self.config.max_pos:
            raise ValueError(f"sequence of {int(pb.seq_lens.max())} tokens exceeds max_position_embeddings={self.config.max_pos} "
                             "(the RoPE tables end there); lower max_inp_length")
        groups, src, pos, cu = eng.upload(pb)
        vision = eng.encode_vision(groups, pb.group_row0, pb.n_slices)
        h = eng.lm_hidden(src, pos, cu, int(pb.seq_lens.max()), vision)
        hn = ops.rmsnorm(h, eng.final_w, self.config.rms_eps, eng.dtype)  # final norm (`modeling_minicpm.py:1280`)
        B, Lmax = pb.n_items, int(pb.seq_lens.max())
        out = torch.zeros((B, Lmax, self.config.hidden), dtype=hn.dtype, device=self.device)
        mask = torch.zeros((B, Lmax), dtype=torch.int8, device=self.device)
        lens = torch.from_numpy(pb.seq_lens).to(self.device)
        valid = torch.arange(Lmax, device=self.device)[None, :] < lens[:, None]
        out[valid] = hn  # packed rows are in (batch, position) order
        mask[valid] = 1
        return BaseModelOutputWithAttentionMask(last_hidden_state=out, attention_mask=mask)

    __call__ = forward


class DRModelForInference:
    """B2 boundary (`dense_retrieval_model.py:46-231,387-408`), inference only."""

    def __init__(self, lm_q, feature: str = "last_hidden_state", pooling: str = "lasttoken", attention: str = "causal",
                 head_q=None, head_p=None, normalize: bool = False, model_args=None, data_args=None, train_args=None,
                 base_model_arch: str = "Llama"):
        self.lm_q = lm_q
        self.head_q, self.head_p = head_q, head_p
        self.feature, self.pooling, self.normalize, self.attention = feature, pooling, normalize, attention
        self.model_args, self.data_args, self.train_args = model_args, data_args, train_args
        self.base_model_arch = base_model_arch

    @classmethod
    def build(cls, model_args, cache_dir=None, device: str = "cuda:0", **_):
        """`DRModel.build` (`dense_retrieval_model.py:233-366`) for a VisRAG-Ret checkpoint directory. `model_args.dtype`
        "float16" (the reference evaluation's `--dtype float16`) builds an fp16 engine; "bfloat16", "float32" or no dtype
        build the bf16 one (float32 runs bf16: there is no fp32 encode path)."""
        if is_float16(getattr(model_args, "dtype", None)):
            lm = VisRAGRetB200.from_pretrained(model_args.model_name_or_path, torch_dtype=torch.float16, device=device)
        else:
            lm = VisRAGRetB200.from_pretrained(model_args.model_name_or_path, device=device)
        return cls(lm_q=lm, feature=getattr(model_args, "feature", "last_hidden_state"), pooling=model_args.pooling,
                   attention=getattr(model_args, "attention", "causal"), normalize=model_args.normalize, model_args=model_args)

    def eval(self):
        return self

    def to(self, *_a, **_k):
        return self

    @torch.no_grad()
    def encode(self, items, model, head, is_query: bool = False, **kwargs):
        if items is None:
            return None, None
        assert self.normalize is True, "Normalize must be true"  # same assertion as `dense_retrieval_model.py:222`
        if self.pooling not in ops.POOLING:
            raise ValueError("Unknown pooling type: {}".format(self.pooling))
        if isinstance(model, VisRAGRetB200):
            return None, self.encode_prepared(self.prepare(items, **kwargs))
        raise TypeError("DRModelForInference (visrag_b200) only drives a VisRAGRetB200 backbone: there is no "
                        "PyTorch/CPU fallback path in this package")

    # The two halves of encode(): host preparation (CPU only, thread safe) and the device part (asynchronous launches).
    # `inference.encode_stream` runs prepare() for batch i+1 on a worker thread while batch i is on the GPU.
    def prepare(self, items, **kwargs):
        return prepare_batch(items["text"], items["image"], kwargs["tokenizer"], self.lm_q.config,
                             kwargs.get("max_inp_length", 2048), self.lm_q.engine.device_frontend)

    @torch.no_grad()
    def encode_prepared(self, pb):
        assert self.normalize is True, "Normalize must be true"
        return self.lm_q.engine.encode_prepared(pb, self.pooling, True)

    def encode_passage(self, psg, **kwargs):
        return self.encode(psg, self.lm_q, self.head_p, is_query=False, **kwargs)

    def encode_query(self, qry, **kwargs):
        return self.encode(qry, self.lm_q, self.head_q, is_query=True, **kwargs)

    def forward(self, query=None, passage=None, **kwargs) -> DROutput:
        _, q_reps = self.encode_query(query, **kwargs)
        _, p_reps = self.encode_passage(passage, **kwargs)
        return DROutput(q_reps=q_reps, p_reps=p_reps)

    __call__ = forward
