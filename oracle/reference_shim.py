"""TEST INFRASTRUCTURE (oracle/) — never imported by the product path.

Runs the UNMODIFIED reference implementation (a checkout of OpenBMB/VisRAG, ``VISRAG_REFERENCE``: timm_modified + src/openmatch) on CPU so
that (1) the restatement in ``oracle/restated.py`` can be validated against it and (2) golden vectors can be
generated (``oracle/gen_golden.py``). Only usable where a checkout of the reference exists (``VISRAG_REFERENCE``), so nothing under
tests/ -m gpu, smoke() or bench.py touches this module.

Shims (SURVEY.md §8c; the reference pins transformers 4.40, this image has 5.x):
  1. ``transformers.utils.import_utils.is_torch_fx_available`` is gone -> provide ``lambda: False``
     (`modeling_minicpm.py:57`).
  2. ``MiniCPMVConfig(use_cache=False)`` + ``cfg.rope_scaling = None`` (`modeling_minicpm.py:408,1196-1200`).
  3. A reduced-size timm ViT variant is *registered* (not patched) so tiny goldens are possible; the full
     model uses the reference's own ``vit_so400m_patch14_siglip_384``.
"""
from __future__ import annotations

import os
import sys
from typing import Dict, List

REF_ROOT = os.environ.get("VISRAG_REFERENCE", "/root/reference")


def available() -> bool:
    return os.path.isdir(os.path.join(REF_ROOT, "src", "openmatch"))


_loaded = {}


def _import_reference():
    if _loaded:
        return _loaded
    if not available():
        raise RuntimeError(f"reference not found under {REF_ROOT}")
    sys.dont_write_bytecode = True
    for p in (os.path.join(REF_ROOT, "timm_modified"), os.path.join(REF_ROOT, "src")):
        if p not in sys.path:
            sys.path.append(p)  # at the END: the reference trees carry their own `tests` package, which must not shadow ours
    import transformers.utils.import_utils as iu

    if not hasattr(iu, "is_torch_fx_available"):
        iu.is_torch_fx_available = lambda: False
    import timm  # noqa: F401  (reference's vendored timm 0.9.16)
    from timm.models import register_model
    from timm.models.vision_transformer import _create_vision_transformer

    def _make_variant(name, dim, depth, heads, mlp_hidden):
        def fn(pretrained: bool = False, **kwargs):
            args = dict(patch_size=14, embed_dim=dim, depth=depth, num_heads=heads, mlp_ratio=mlp_hidden / dim,
                        class_token=False, global_pool="map", img_size=384)
            return _create_vision_transformer("vit_so400m_patch14_siglip_384", pretrained=False, **dict(args, **kwargs))

        fn.__name__ = name
        fn.__module__ = "timm.models.vision_transformer"
        return register_model(fn)

    _loaded["make_variant"] = _make_variant
    from openmatch.modeling.modeling_visrag_ret.modeling_visrag_ret import VisRAG_Ret
    from openmatch.modeling.modeling_minicpmv.configuration_minicpm import MiniCPMVConfig
    from openmatch.modeling.dense_retrieval_model import DRModelForInference
    from openmatch.arguments import ModelArguments
    from openmatch.inference.inference import naive_collator

    _loaded.update(VisRAG_Ret=VisRAG_Ret, MiniCPMVConfig=MiniCPMVConfig, DRModelForInference=DRModelForInference,
                   ModelArguments=ModelArguments, naive_collator=naive_collator)
    return _loaded


_variants = {}


def build_reference_model(cfg, state_dict: Dict[str, "torch.Tensor"], attn_implementation: str = "sdpa",
                          pooling: str = "wmean"):
    """Instantiate the reference ``DRModelForInference(lm_q=VisRAG_Ret(...))`` with the given weights (fp32, CPU)."""
    import torch

    R = _import_reference()
    if cfg.vit_dim == 1152 and cfg.vit_depth == 26 and cfg.vit_mlp == 4304:
        enc_name = "vit_so400m_patch14_siglip_384"
    else:
        enc_name = f"vit_test{cfg.vit_dim}x{cfg.vit_depth}_patch14_siglip_384"
        if enc_name not in _variants:
            R["make_variant"](enc_name, cfg.vit_dim, cfg.vit_depth + 1, cfg.vit_heads, cfg.vit_mlp)
            _variants[enc_name] = True
    mcfg = R["MiniCPMVConfig"](
        vision_encoder=enc_name, query_num=cfg.query_num, drop_vision_last_layer=True, slice_mode=cfg.slice_mode,
        patch_size=cfg.patch_size, max_slice_nums=cfg.max_slice_nums, scale_resolution=cfg.scale_resolution,
        vocab_size=cfg.vocab, hidden_size=cfg.hidden, intermediate_size=cfg.inter, num_hidden_layers=cfg.layers,
        num_attention_heads=cfg.heads, num_key_value_heads=cfg.heads, max_position_embeddings=cfg.max_pos,
        rms_norm_eps=cfg.rms_eps, rope_theta=cfg.rope_theta, scale_emb=cfg.scale_emb, scale_depth=cfg.scale_depth,
        dim_model_base=256, use_cache=False, attn_implementation=attn_implementation, tie_word_embeddings=False,
    )
    mcfg.rope_scaling = None
    mcfg._attn_implementation = attn_implementation
    torch.manual_seed(0)
    lm = R["VisRAG_Ret"](mcfg).float().eval()
    own = lm.state_dict()
    missing = [k for k in own if k not in state_dict and not k.startswith("llm.lm_head") and "rotary_emb" not in k
               and not k.startswith("vpm.blocks.%d." % cfg.vit_depth)]
    unexpected = [k for k in state_dict if k not in own]
    if missing or unexpected:
        raise RuntimeError(f"state_dict mismatch: missing={missing[:8]} unexpected={unexpected[:8]}")
    lm.load_state_dict({k: v.float() for k, v in state_dict.items()}, strict=False)
    margs = R["ModelArguments"](model_name_or_path="synthetic", pooling=pooling, normalize=True)
    model = R["DRModelForInference"](lm_q=lm, feature="last_hidden_state", pooling=pooling, normalize=True,
                                     model_args=margs)
    return model


def encode(model, tokenizer, items: List[dict], is_query: bool, max_inp_length: int = 2048):
    """``items`` = [{id,text,image}]; returns fp32 numpy [n, hidden] through the reference B2 boundary."""
    R = _import_reference()
    batch = R["naive_collator"](items)
    if is_query:
        out = model(query=batch, tokenizer=tokenizer, max_inp_length=max_inp_length)
        return out.q_reps.cpu().numpy()
    out = model(passage=batch, tokenizer=tokenizer, max_inp_length=max_inp_length)
    return out.p_reps.cpu().numpy()


def hidden_states(model, tokenizer, texts: List[str], images: list, max_inp_length: int = 2048):
    """B1 boundary: reference ``VisRAG_Ret.forward`` -> (last_hidden_state, attention_mask) as numpy."""
    import torch

    with torch.no_grad():
        o = model.lm_q(text=texts, image=images, tokenizer=tokenizer, max_inp_length=max_inp_length)
    return o.last_hidden_state.float().numpy(), o.attention_mask.numpy()
