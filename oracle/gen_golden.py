"""TEST INFRASTRUCTURE. Generates tests/golden/*.npz by running the REAL reference (through
oracle/reference_shim.py) where a checkout of it is available (VISRAG_REFERENCE):   python -m oracle.gen_golden [--full]

The .npz files hold everything needed to replay the case without the reference: the config, the weight seed
(weights are re-drawn by visrag_b200.weights.random_state_dict), the page sizes + pixel seed (pages are
re-drawn by synth_pages), the query strings, and the reference outputs (fp32 embeddings, score top-k,
slice geometry).
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import warnings

import numpy as np
from PIL import Image

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
warnings.filterwarnings("ignore")

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")

from visrag_b200.synth import QUERY_PREFIX, synth_pages, synth_queries  # noqa: E402,F401


def geometry_cases():
    sizes = [(224, 224), (448, 448), (336, 336), (1344, 1344), (564, 3040), (1114, 1670), (700, 900), (1200, 500),
             (500, 1200), (640, 480), (2000, 300), (300, 2000), (449, 449), (1000, 1000), (896, 448), (447, 448)]
    rs = np.random.RandomState(11)
    for _ in range(150):
        sizes.append((int(rs.randint(100, 1500)), int(rs.randint(100, 1500))))
    return sizes


def geometry_v2_cases():
    """Tall and wide pages: long screenshots, infographics, banners and thin strips, aspect ratios up to about 1:3000 and
    sides up to 40000 (area at most 6e7 pixels, so that the blank test images stay small)."""
    sizes = [(1280, 10000), (1280, 40000), (600, 8000), (8000, 600), (3000, 100), (100, 3000), (33964, 287), (287, 33964),
             (30000, 30), (30, 30000), (3000, 14), (14, 3000), (3000, 1), (1, 3000), (40000, 14), (14, 40000), (40000, 1000),
             (1000, 40000), (13000, 400), (12288, 500), (12289, 500), (4858, 42), (1, 1), (2, 40000), (40000, 2)]
    rs = np.random.RandomState(12)
    while len(sizes) < 200:
        long_side = int(np.exp(rs.uniform(np.log(100), np.log(40000))))
        short = max(1, int(round(long_side / np.exp(rs.uniform(0, np.log(3000))))))
        if long_side * short <= 60_000_000:
            sizes.append((long_side, short) if rs.randint(2) else (short, long_side))
    return sizes


def gen_geometry(cases=geometry_cases, name="geometry_v1"):
    """Slice geometry from the reference's own slice_image (modeling_minicpmv.py:482-537)."""
    from oracle import reference_shim as RS

    RS._import_reference()
    from openmatch.modeling.modeling_minicpmv.modeling_minicpmv import slice_image

    rows = []
    for (w, h) in cases():
        src, patches, grid = slice_image(Image.new("RGB", (w, h)), 9, 448, 14)
        g = grid if grid is not None else [0, 0]
        pw, ph = (patches[0][0].size if patches else (0, 0))
        rows.append([w, h, src.size[0], src.size[1], g[0], g[1], pw, ph, sum(len(r) for r in patches)])
    np.savez(os.path.join(GOLDEN_DIR, f"{name}.npz"), cases=np.asarray(rows, dtype=np.int64),
             columns=np.asarray(["W", "H", "src_w", "src_h", "grid_x", "grid_y", "patch_w", "patch_h", "n_patches"]))
    print(f"{name}:", len(rows), "cases")


def gen_model_case(name, cfg, weight_seed, page_sizes, page_seed, n_queries, query_seed, topk):
    import torch
    from oracle import reference_shim as RS
    from visrag_b200.tokenizer_stub import StubTokenizer
    from visrag_b200.weights import random_state_dict

    sd = random_state_dict(cfg, weight_seed)
    model = RS.build_reference_model(cfg, sd, attn_implementation="sdpa")
    tok = StubTokenizer(cfg.vocab)
    pages = synth_pages(page_sizes, page_seed)
    queries = synth_queries(n_queries, query_seed)
    p_items = [{"id": f"d{i}", "text": "", "image": im} for i, im in enumerate(pages)]
    q_items = [{"id": f"q{i}", "text": t, "image": None} for i, t in enumerate(queries)]
    # the reference encodes in batches; padding must not matter -> encode pages in two uneven batches
    half = max(1, len(p_items) // 2)
    p = np.concatenate([RS.encode(model, tok, p_items[:half], False), RS.encode(model, tok, p_items[half:], False)])
    q = RS.encode(model, tok, q_items, True)
    # reference scoring: torch.matmul + torch.topk (dense_retriever.py:25-30)
    S = torch.matmul(torch.from_numpy(q), torch.from_numpy(p).T)
    ts, ti = torch.topk(S, min(topk, p.shape[0]), dim=1)
    np.savez(os.path.join(GOLDEN_DIR, f"{name}.npz"), config=json.dumps(cfg.to_dict()), weight_seed=weight_seed,
             page_sizes=np.asarray(page_sizes, dtype=np.int64), page_seed=page_seed, queries=np.asarray(queries),
             query_seed=query_seed, page_reps=p.astype(np.float32), query_reps=q.astype(np.float32),
             topk_scores=ts.numpy(), topk_indices=ti.numpy())
    print(name, "pages", p.shape, "queries", q.shape)


REAL_PAGES = [os.path.join(GOLDEN_DIR, n) for n in ("real_pages_parquet.npz", "real_pages_demo.npz")]  # each below 1 MB


def gen_real_pages():
    """The reference's own example inputs, kept as the ENCODED bytes the reference ships (data, not code): the two
    (query, page) rows of examples/training_data/0.parquet and the demo's cat/dog photos
    (visrag_scripts/demo/retriever/test_image, README.md:315-319). Decoded with PIL at test time."""
    import pyarrow.parquet as pq
    from oracle.reference_shim import REF_ROOT

    t = pq.read_table(os.path.join(REF_ROOT, "examples", "training_data", "0.parquet"))
    out, demo, queries = {}, {}, []
    for i in range(t.num_rows):
        out[f"parquet{i}"] = np.frombuffer(t.column("image")[i].as_py()["bytes"], dtype=np.uint8)
        queries.append(t.column("query")[i].as_py())
    for n in ("cat.jpeg", "dog.jpg"):
        with open(os.path.join(REF_ROOT, "visrag_scripts", "demo", "retriever", "test_image", n), "rb") as f:
            demo[n.split(".")[0]] = np.frombuffer(f.read(), dtype=np.uint8)
    np.savez(REAL_PAGES[0], queries=np.asarray(queries), **out)
    np.savez(REAL_PAGES[1], **demo)
    print("real pages:", {k: v.size for k, v in dict(out, **demo).items()})


def full_v2_spec():
    """>= 32 pages (>= 8 multi-slice + the reference's 4 real example images) and >= 8 queries: a corpus on which the
    top-5 ranking is a real statement."""
    single = [(448, 448), (400, 500), (300, 600), (224, 224), (336, 336), (420, 420), (500, 390), (448, 448), (360, 540),
              (640, 300), (448, 448), (280, 280), (512, 384), (384, 512), (448, 448), (330, 600), (600, 330), (448, 440),
              (224, 224), (436, 452)]
    multi = [(700, 900), (640, 480), (1000, 700), (900, 450), (1344, 336), (600, 600), (800, 1000), (448, 900)]
    spec = [{"kind": "doc", "size": list(s), "seed": 5000 + i} for i, s in enumerate(single + multi)]
    spec += [{"kind": "noise", "size": list(s), "seed": 6000 + i} for i, s in enumerate([(448, 448), (448, 448), (224, 224), (640, 480)])]
    spec += [{"kind": "real", "name": n} for n in ("parquet0", "parquet1", "cat", "dog")]
    return spec


def gen_spec_case(name, cfg, weight_seed, spec, n_queries, query_seed, topk, batch=6):
    """Like gen_model_case, for a page list described by a spec (see tests/helpers.pages_from_spec)."""
    import time

    import torch
    from oracle import reference_shim as RS
    from tests.helpers import pages_from_spec, real_queries
    from visrag_b200.tokenizer_stub import StubTokenizer
    from visrag_b200.weights import random_state_dict

    sd = random_state_dict(cfg, weight_seed)
    model = RS.build_reference_model(cfg, sd, attn_implementation="sdpa")
    tok = StubTokenizer(cfg.vocab)
    pages = pages_from_spec(spec)
    queries = synth_queries(n_queries, query_seed) + [QUERY_PREFIX + q for q in real_queries()]
    p_items = [{"id": f"d{i}", "text": "", "image": im} for i, im in enumerate(pages)]
    q_items = [{"id": f"q{i}", "text": t, "image": None} for i, t in enumerate(queries)]
    t0 = time.time()
    parts = []
    for s in range(0, len(p_items), batch):  # the reference's own batch loop, right-padded batches of mixed pages
        parts.append(RS.encode(model, tok, p_items[s:s + batch], False))
        print(f"  pages {s + len(parts[-1])}/{len(p_items)}  {time.time() - t0:.0f}s", flush=True)
    p = np.concatenate(parts)
    q = RS.encode(model, tok, q_items, True)
    S = torch.matmul(torch.from_numpy(q), torch.from_numpy(p).T)      # dense_retriever.py:25-30
    ts, ti = torch.topk(S, topk, dim=1)
    full = np.sort(S.numpy(), axis=1)[:, ::-1]
    gaps = full[:, :topk] - full[:, 1:topk + 1]
    np.savez(os.path.join(GOLDEN_DIR, f"{name}.npz"), config=json.dumps(cfg.to_dict()), weight_seed=weight_seed,
             page_spec=json.dumps(spec), queries=np.asarray(queries), query_seed=query_seed,
             page_reps=p.astype(np.float32), query_reps=q.astype(np.float32), topk_scores=ts.numpy(),
             topk_indices=ti.numpy(), min_gap=np.float32(gaps.min()))
    print(name, "pages", p.shape, "queries", q.shape, "min score gap inside top-(k+1):", gaps.min(), "median", np.median(gaps))


def gen_reference_pins():
    """What tests/test_oracle_vs_reference.py compares the oracle with: outputs of the reference on the test's own seeded
    inputs (embeddings, hidden states, the other poolings on a ragged batch, `_retrieve_one_shard`, run files, MRR)."""
    import pickle
    import tempfile

    import torch
    from oracle import reference_shim as RS
    from visrag_b200 import retriever as R
    from visrag_b200.config import VisRAGConfig
    from visrag_b200.tokenizer_stub import StubTokenizer
    from visrag_b200.weights import random_state_dict

    out = {}
    cfg = VisRAGConfig.tiny()
    tok = StubTokenizer(cfg.vocab)
    sd = random_state_dict(cfg, 777)
    model = RS.build_reference_model(cfg, sd, attn_implementation="sdpa")
    pages = synth_pages([(300, 300), (1000, 600), (448, 448)], 21)
    items = [{"id": str(i), "text": "doc text" if i == 1 else "", "image": im} for i, im in enumerate(pages)]
    out["fresh_pages"] = RS.encode(model, tok, items, False)
    qs = [QUERY_PREFIX + "what is shown", QUERY_PREFIX + "x"]
    out["fresh_queries"] = RS.encode(model, tok, [{"id": f"q{i}", "text": t, "image": None} for i, t in enumerate(qs)], True)
    hs, mask = RS.hidden_states(model, tok, [it["text"] for it in items], pages)
    out["fresh_hidden"], out["fresh_mask"] = hs.astype(np.float32), mask.astype(np.int64)
    sd = random_state_dict(cfg, 778)
    page = synth_pages([(448, 448)], 5)[0]
    texts = [QUERY_PREFIX + "a", QUERY_PREFIX + "a much longer query about the page content", ""]
    items = [{"id": str(i), "text": t, "image": im} for i, (t, im) in enumerate(zip(texts, [None, None, page]))]
    for pooling in ("lasttoken", "mean", "cls"):
        model = RS.build_reference_model(cfg, sd, attn_implementation="sdpa", pooling=pooling)
        out[f"pooling_{pooling}"] = RS.encode(model, tok, items, False)
    # scoring side: the reference's shard reader + top-k, run-file writer / reader and MRR on the test's vectors
    from openmatch import utils as ref_utils
    from openmatch.retriever.dense_retriever import _retrieve_one_shard as ref_retrieve

    rs = np.random.RandomState(12)
    D = rs.randn(500, 64).astype(np.float32)
    D /= np.linalg.norm(D, axis=1, keepdims=True)
    Q = rs.randn(7, 64).astype(np.float32)
    Q /= np.linalg.norm(Q, axis=1, keepdims=True)
    lookup = [f"doc{i}" for i in range(len(D))]
    with tempfile.TemporaryDirectory() as tmp:
        shard = os.path.join(tmp, "embeddings.corpus.rank.0")
        R.save_shard(shard, D, lookup)
        s_ref, i_ref, look_ref = ref_retrieve(shard, torch.from_numpy(Q), 10, "cpu")
        assert look_ref == lookup and pickle.load(open(shard, "rb"))[1] == lookup
        s, i = s_ref.numpy(), i_ref.numpy()
        run = {f"q{q}": {lookup[j]: float(s[q, r]) for r, j in enumerate(i[q])} for q in range(len(Q))}
        qrel = {f"q{q}": {lookup[int(i[q, q % 10])]: 1} for q in range(len(Q))}
        trec = os.path.join(tmp, "ref.trec")
        ref_utils.save_as_trec(run, trec)
        out["trec_text"] = np.asarray(open(trec).read())
        from visrag_b200 import inference as I

        ours = os.path.join(tmp, "ours.trec")
        I.save_as_trec(run, ours)   # the reference's reader on OUR writer's file
        assert ref_utils.load_from_trec(ours) == ref_utils.load_from_trec(trec)
        out["trec_loaded"] = np.asarray(json.dumps(ref_utils.load_from_trec(trec), sort_keys=True))
        out["mrr"] = np.asarray(json.dumps([ref_utils.eval_mrr(qrel, run, 10), ref_utils.eval_mrr(qrel, run, 3)], sort_keys=True))
    out["topk_scores"], out["topk_indices"] = s, i
    np.savez_compressed(os.path.join(GOLDEN_DIR, "reference_pins.npz"), **out)
    print("reference pins:", {k: getattr(v, "shape", None) for k, v in out.items()})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pins", action="store_true", help="only generate reference_pins.npz (tests/test_oracle_vs_reference.py)")
    ap.add_argument("--full", action="store_true", help="also generate the full-size (3.1 B parameter) case")
    ap.add_argument("--full-v2", action="store_true", help="only generate full_v2 (36 pages, 10 queries, top-5; ~15 min of CPU)")
    ap.add_argument("--tiny-v2", action="store_true", help="only generate tiny_v2 (same corpus as full_v2, tiny model)")
    ap.add_argument("--geometry-v2", action="store_true", help="only generate geometry_v2 (tall and wide pages; ~1 min of CPU)")
    a = ap.parse_args()
    from visrag_b200.config import VisRAGConfig as _C

    if a.pins:
        gen_reference_pins()
        return
    if a.geometry_v2:
        gen_geometry(geometry_v2_cases, "geometry_v2")
        return
    if a.full_v2 or a.tiny_v2:
        if not all(os.path.exists(p) for p in REAL_PAGES):
            gen_real_pages()
        if a.tiny_v2:
            gen_spec_case("tiny_v2", _C.tiny(), 1234, full_v2_spec(), 8, 25, 5)
        if a.full_v2:
            gen_spec_case("full_v2", _C.full(), 4321, full_v2_spec(), 8, 25, 5)
        return
    os.makedirs(GOLDEN_DIR, exist_ok=True)
    from visrag_b200.config import VisRAGConfig

    gen_geometry()
    gen_geometry(geometry_v2_cases, "geometry_v2")
    sizes =[(224, 224), (448, 448), (224, 224), (700, 900), (760, 141), (1200, 500), (320, 240), (448, 448)]
    gen_model_case("tiny_v1", VisRAGConfig.tiny(), 1234, sizes, 7, 4, 5, 5)
    if a.full:
        gen_model_case("full_v1", VisRAGConfig.full(), 4321, [(448, 448), (224, 224), (640, 480)], 17, 3, 15, 3)


if __name__ == "__main__":
    main()
