"""Encode-path parity on the H100: CUDA engine (through the C ABI and the reference-signature classes) against
  (1) golden embeddings produced by the REAL reference (tests/golden/*.npz), tiny and full-size model,
  (2) the oracle restatement on freshly seeded inputs, at the B1 (hidden states) and B2 (embeddings) boundaries.
Stated tolerance (north_star: "within a stated fp tolerance"): cosine(embedding, fp32 reference) >= 0.9999 per vector
and max |diff| <= 1e-3 on unit vectors; ORDERED top-k ids identical to the reference's torch.topk on the golden
(query, corpus) sets (k < n), Recall@1/5 equal with zero slack. The engine computes
in bf16 operands / fp32 accumulate with fp32 residual streams; the reference run is fp32."""
import numpy as np
import pytest
import torch

from tests.helpers import QUERY_PREFIX, cosine_rows, load_case, synth_pages

pytestmark = pytest.mark.gpu

COS_MIN, ABS_MAX = 0.9999, 1e-3


def _engine_model(cfg, sd, pooling="wmean"):
    from visrag_b200.modeling import DRModelForInference, VisRAGRetB200

    return DRModelForInference(lm_q=VisRAGRetB200(cfg, sd, "cuda:0"), pooling=pooling, normalize=True)


def _items(texts, images, prefix):
    return {"id": [f"{prefix}{i}" for i in range(len(texts))], "text": list(texts), "image": list(images)}


def _check_case(name):
    from visrag_b200.tokenizer_stub import StubTokenizer
    from visrag_b200.weights import random_state_dict

    cfg, wseed, pages, queries, z = load_case(name)
    sd = random_state_dict(cfg, wseed)
    model = _engine_model(cfg, sd)
    del sd
    tok = StubTokenizer(cfg.vocab)
    out = model(query=_items(queries, [None] * len(queries), "q"), passage=_items([""] * len(pages), pages, "d"),
                tokenizer=tok, max_inp_length=2048)
    assert out.p_reps.dtype == torch.float32 and out.p_reps.is_cuda
    p, q = out.p_reps.cpu().numpy(), out.q_reps.cpu().numpy()
    cp, cq = cosine_rows(p, z["page_reps"]), cosine_rows(q, z["query_reps"])
    assert cp.min() >= COS_MIN and cq.min() >= COS_MIN, (cp, cq)
    assert np.abs(p - z["page_reps"]).max() <= ABS_MAX and np.abs(q - z["query_reps"]).max() <= ABS_MAX
    assert np.allclose(np.linalg.norm(p, axis=1), 1.0, atol=1e-5)
    k = z["topk_indices"].shape[1]
    ref_top = z["topk_indices"]
    if k >= len(pages):  # v1 goldens (k == n): only the id sets can be compared
        top = np.argsort(-(q @ p.T), axis=1)[:, :k]
        assert np.array_equal(np.sort(top, 1), np.sort(ref_top, 1))
        return cp.min(), cq.min()
    # ranking parity through the engine's own scorer (tensor-core filter + exact fp32 rescoring), k < n:
    # the ORDERED top-k ids must equal the reference's torch.matmul + torch.topk (dense_retriever.py:25-30)
    from visrag_b200 import retriever as R

    s_run, i_run = R.score_topk(out.q_reps, R.build_index(out.p_reps), k)
    i_run, s_run = i_run.cpu().numpy(), s_run.cpu().numpy()
    print(f"{name}: cos pages >= {cp.min():.7f}, queries >= {cq.min():.7f}, max |score diff| "
          f"{np.abs(s_run - z['topk_scores']).max():.2e}, golden min gap "
          f"{float(z['min_gap']) if 'min_gap' in z.files else float('nan'):.2e}")
    assert np.array_equal(i_run, ref_top), (i_run, ref_top)
    assert np.abs(s_run - z["topk_scores"]).max() <= 2 * ABS_MAX
    # Recall@1/5 with zero slack: relevance = the reference's own best page per query, and for the two real
    # (query, page) rows of the reference's parquet example the page that belongs to the query
    from oracle import restated as O

    relevant = [{int(ref_top[qi, 0])} for qi in range(len(queries))]
    if "page_spec" in z.files:
        spec = [e.get("name") for e in __import__("json").loads(str(z["page_spec"]))]
        for r, nm in enumerate(("parquet0", "parquet1")):
            relevant[len(queries) - 2 + r].add(spec.index(nm))
    for kk in (1, 5):
        assert O.recall_at_k(i_run, relevant, kk) == O.recall_at_k(ref_top, relevant, kk)
    return cp.min(), cq.min()


def test_tiny_model_matches_reference_golden():
    _check_case("tiny_v1")


def test_tiny_model_ranking_matches_reference_golden():
    """36 pages (28 structured synthetic documents incl. 8 multi-slice, 4 noise pages, the reference's 4 real example
    images) x 10 queries (8 synthetic + the 2 real parquet queries), top-5 of 36."""
    _check_case("tiny_v2")


def test_full_size_model_matches_reference_golden():
    """SigLIP-so400m (26 blocks) + Resampler + MiniCPM-2B (40 layers), 3.1 B parameters, vs the real reference's fp32 run."""
    _check_case("full_v1")


def test_full_size_model_ranking_matches_reference_golden():
    """The 3.1 B-parameter engine on a corpus where ranking can differ: the full_v2 golden (36 pages incl. 8 synthetic
    multi-slice documents and the reference's own parquet pages + cat/dog photos, 10 queries, top-5 with k < n) was produced
    by the REAL reference in fp32 (oracle/gen_golden.py --full-v2). Ordered ids identical, Recall@1/5 equal, cos >= 0.9999."""
    _check_case("full_v2")


def test_boundaries_against_oracle_on_fresh_inputs():
    from oracle import restated as O
    from visrag_b200.config import VisRAGConfig
    from visrag_b200.tokenizer_stub import StubTokenizer
    from visrag_b200.weights import random_state_dict

    cfg = VisRAGConfig.tiny()
    sd = random_state_dict(cfg, 31337)
    tok = StubTokenizer(cfg.vocab)
    pages = synth_pages([(224, 224), (564 // 2, 3040 // 2), (1344, 1344), (336, 340)], 77)  # 1, 1+8, 1+9, 1 slices
    texts = ["", "a caption", "", "x"]
    model = _engine_model(cfg, sd)
    # B2: pooled embeddings, all pooling modes the kernel implements
    for pooling in ("wmean", "mean", "lasttoken", "cls"):
        model.pooling = pooling
        _, got = model.encode_passage(_items(texts, pages, "d"), tokenizer=tok, max_inp_length=2048)
        want = O.encode(sd, cfg, tok, texts, pages, pooling=pooling)
        c = cosine_rows(got.cpu().numpy(), want)
        assert c.min() >= COS_MIN, (pooling, c)
    # B1: right-padded final-norm hidden states + mask
    out = model.lm_q(text=texts, image=pages, tokenizer=tok, max_inp_length=2048)
    _, hid = O.encode(sd, cfg, tok, texts, pages, return_hidden=True)
    assert out.last_hidden_state.shape[:2] == out.attention_mask.shape
    for b, h in enumerate(hid):
        n = int(out.attention_mask[b].sum())
        assert n == h.shape[0]
        got = out.last_hidden_state[b, :n].float().cpu().numpy()
        assert np.abs(got - h).max() <= 0.05 * np.abs(h).max()
        assert (out.last_hidden_state[b, n:] == 0).all()
    # text-only queries incl. a 1-token-ish and a long one; empty batch
    qs = [QUERY_PREFIX + "a", QUERY_PREFIX + " ".join(["word"] * 150)]
    model.pooling = "wmean"
    _, gq = model.encode_query(_items(qs, [None, None], "q"), tokenizer=tok, max_inp_length=2048)
    assert cosine_rows(gq.cpu().numpy(), O.encode(sd, cfg, tok, qs, [None, None])).min() >= COS_MIN
    assert model(query=None, passage=None).q_reps is None
    # truncation at max_inp_length behaves like the reference (ids[:max])
    _, gt = model.encode_query(_items(qs[1:], [None], "q"), tokenizer=tok, max_inp_length=40)
    assert cosine_rows(gt.cpu().numpy(), O.encode(sd, cfg, tok, qs[1:], [None], max_inp_length=40)).min() >= COS_MIN


def test_vision_tower_and_resampler_against_oracle():
    """One boundary further in than B1: ViT tokens (after the final LayerNorm) and the resampler's 64 x hidden output for
    single slices of two geometries, against the oracle's fp32 towers on the same pixels. Tolerance 3e-2 relative to the
    largest reference value (26 bf16 transformer blocks)."""
    from PIL import Image

    from oracle import restated as O
    from visrag_b200 import host
    from visrag_b200.encoder import VisRAGEngine
    from visrag_b200.weights import random_state_dict

    cfg, wseed, pages, _, _ = load_case("tiny_v1")
    sd = random_state_dict(cfg, wseed)
    eng = VisRAGEngine(cfg, sd)

    def close(got, want, tol):
        want = torch.as_tensor(want).float()
        err = (got.float().cpu() - want).abs().max().item()
        return err <= tol * max(want.abs().max().item(), 1.0) and bool(torch.isfinite(got.float()).all())

    for img in (pages[0], pages[3]):
        slices = host.render_slices(img, host.plan_slices(*img.size, cfg))
        for s in slices[:2]:
            tok = eng.vit_tokens(torch.from_numpy(s)[None].cuda())
            want = O.vit_forward(sd, cfg, O.pixel_values(Image.fromarray(s)))
            assert close(tok, want, 3e-2), s.shape
            gh, gw = s.shape[0] // 14, s.shape[1] // 14
            out = torch.empty(cfg.query_num, cfg.hidden, device="cuda")
            eng.resample(tok, 1, gh, gw, out)
            assert close(out, O.resampler_forward(sd, cfg, want, gh, gw), 3e-2), s.shape


def _short_queries(n):
    words = ["cat", "tax", "map", "2020", "dog", "sofa", "chart", "x"]
    return [" ".join(words[(i + j) % len(words)] for j in range(1 + i % 5)) for i in range(n)]


def test_batch_composition_does_not_change_results():
    """Same item alone vs inside a mixed batch: bit-identical (no padding, no cross-sequence leakage). The batch decides
    which attention kernel runs (longest sequence <= 64 or not), the cluster size of the final pooling (more than
    5 x #SMs / 8 sequences or not) and whether a CUDA graph replays; none of that may change an embedding."""
    from visrag_b200.config import VisRAGConfig
    from visrag_b200.encoder import VisRAGEngine
    from visrag_b200.tokenizer_stub import StubTokenizer
    from visrag_b200.weights import random_state_dict

    cfg = VisRAGConfig.tiny()
    sd = random_state_dict(cfg, 5)
    eng = VisRAGEngine(cfg, sd)
    eager = VisRAGEngine(cfg, sd, cuda_graphs=False)
    tok = StubTokenizer(cfg.vocab)
    pages = synth_pages([(448, 448), (700, 900), (448, 448)], 9)
    alone = eng.encode([""], [pages[1]], tok)
    mixed = eng.encode(["", "", "query text", ""], [pages[0], pages[1], None, pages[2]], tok)
    assert torch.equal(alone[0], mixed[1])
    assert eng.encode([], [], tok).shape == (0, cfg.hidden)
    # short text queries (<= 64 LM tokens, prefix included): alone, next to a longer query, next to pages
    short = ["cat", QUERY_PREFIX + "tax", "revenue table 2020", QUERY_PREFIX + "2020"]
    assert all(len(tok.encode(q)) < 64 for q in short)
    long_q = QUERY_PREFIX + " ".join(["word"] * 30)
    assert len(tok.encode(long_q)) > 64
    for e in (eng, eager):
        for qi, q in enumerate(short):
            alone = e.encode([q], [None], tok)[0]
            with_long = e.encode([long_q, q], [None, None], tok)[1]
            with_pages = e.encode(["", q, ""], [pages[0], None, pages[2]], tok)[1]
            assert torch.equal(alone, with_long) and torch.equal(alone, with_pages), (q, e.cuda_graphs)
    # 128 pages in one batch (eager: more LM tokens than a graph takes) and in batches of 16
    many = synth_pages([(224, 224)] * 128, 10)
    whole = eng.encode([""] * 128, many, tok)
    parts = torch.cat([eng.encode([""] * 16, many[i:i + 16], tok) for i in range(0, 128, 16)])
    assert torch.equal(whole, parts), (whole - parts).abs().max().item()
    # 128 short queries in one batch (small enough for a CUDA graph) and in batches of 16, graphs on and off
    qs = _short_queries(128)
    for e in (eng, eager):
        whole = e.encode(qs, [None] * 128, tok)
        parts = torch.cat([e.encode(qs[i:i + 16], [None] * 16, tok) for i in range(0, 128, 16)])
        assert torch.equal(whole, parts), (e.cuda_graphs, (whole - parts).abs().max().item())
    assert eng.graph_stats["captured"] + eng.graph_stats["replayed"] > 0


def test_encode_stream_equals_blocking_calls():
    """The pipelined loop (prep of batch i+1 on a worker thread, async D2H) returns exactly what one blocking
    model(passage=...) call per batch returns, in order, including a ragged last batch and an empty dataset."""
    from visrag_b200 import inference as I
    from visrag_b200.config import VisRAGConfig
    from visrag_b200.tokenizer_stub import StubTokenizer
    from visrag_b200.weights import random_state_dict

    cfg = VisRAGConfig.tiny()
    model = _engine_model(cfg, random_state_dict(cfg, 3))
    tok = StubTokenizer(cfg.vocab)
    pages = synth_pages([(448, 448), (300, 500), (700, 900), (224, 224), (448, 448), (640, 320), (500, 500)], 21)
    data = [{"id": f"p{i}", "text": "", "image": im} for i, im in enumerate(pages)]
    kw = {"tokenizer": tok, "max_inp_length": 2048}
    got_ids, got = [], []
    for ids, arr in I.encode_stream(I._batches(data, 3), model, kw):
        got_ids += ids
        got.append(arr)
    assert got_ids == [d["id"] for d in data] and [len(g) for g in got] == [3, 3, 1]
    for b, batch in enumerate(I._batches(data, 3)):
        want = model(passage=batch, **kw).p_reps.cpu().numpy()
        assert np.array_equal(got[b], want)
    assert list(I.encode_stream([], model, kw)) == []
    # a ramped first batch (cut into 4 pieces, re-joined before it is yielded)
    big = [{"id": f"r{i}", "text": "", "image": pages[i % len(pages)]} for i in range(19)]
    out = list(I.encode_stream(I._batches(big, 17), model, kw, ramp_parts=4))
    assert [len(ids) for ids, _ in out] == [17, 2] and out[0][0] == [d["id"] for d in big[:17]]
    want = model(passage=I.naive_collator(big[:17]), **kw).p_reps.cpu().numpy()
    assert np.array_equal(out[0][1], want)
    # queries, first batch of 100 (above the 5 x #SMs / 8 sequences where pooling changes cluster size) cut in 4 pieces
    qs = [{"id": f"q{i}", "text": t, "image": None} for i, t in enumerate(_short_queries(130))]
    out = list(I.encode_stream(I._batches(qs, 100), model, kw, ramp_parts=4))
    assert [len(ids) for ids, _ in out] == [100, 30]
    for (ids, got), batch in zip(out, I._batches(qs, 100)):
        assert np.array_equal(got, model(query=batch, **kw).q_reps.cpu().numpy())


def test_config1_pipeline_encode_shards_retrieve_trec_metrics(tmp_path):
    """BASELINE configs[0]: 4 queries x 32 synthetic 224x224 pages through the reference-signature pipeline
    (encode loop -> pickle shards -> retrieve -> TREC run -> metrics) vs the oracle's embeddings + numpy cosine top-5."""
    from types import SimpleNamespace

    from oracle import restated as O
    from visrag_b200 import inference as I
    from visrag_b200 import retriever as R
    from visrag_b200.config import VisRAGConfig
    from visrag_b200.synth import synth_queries
    from visrag_b200.tokenizer_stub import StubTokenizer
    from visrag_b200.weights import random_state_dict

    cfg = VisRAGConfig.tiny()
    sd = random_state_dict(cfg, 2025)
    tok = StubTokenizer(cfg.vocab)
    pages = synth_pages([(224, 224)] * 32, 1235)
    queries = synth_queries(4, 1235)
    model = _engine_model(cfg, sd)
    args = SimpleNamespace(output_dir=str(tmp_path), per_device_eval_batch_size=5, max_inmem_docs=12, world_size=1,
                           process_index=0, device="cuda:0")
    corpus = [{"id": f"d{i}", "text": "", "image": im} for i, im in enumerate(pages)]
    qset = [{"id": f"q{i}", "text": t, "image": None} for i, t in enumerate(queries)]
    kw = {"tokenizer": tok, "max_inp_length": 2048}
    I.distributed_parallel_embedding_inference(corpus, model, args, "corpus", True, kw)
    I.distributed_parallel_embedding_inference(qset, model, args, "query", False, kw)
    import glob
    import os

    shards = sorted(glob.glob(os.path.join(str(tmp_path), "embeddings.corpus.rank.0.*")))
    assert [os.path.basename(s).split(".")[-1] for s in shards] == ["0-15", "15-30", "30-32"]  # flush rule of inference.py:112
    emb, ids = R.load_shard(shards[0])
    assert emb.dtype == np.float32 and emb.shape == (15, cfg.hidden) and ids[0] == "d0"
    run = R.distributed_parallel_retrieve(args, 5)
    I.save_as_trec(run, os.path.join(str(tmp_path), "test.0.trec"))
    run2 = I.load_from_trec(os.path.join(str(tmp_path), "test.0.trec"))
    p_ref = O.encode(sd, cfg, tok, [""] * 32, pages)
    q_ref = O.encode(sd, cfg, tok, queries, [None] * 4)
    s_ref, top_ref = O.score_topk(q_ref, p_ref, 5)
    full_ref = q_ref @ p_ref.T
    qrels = {}
    for qi in range(4):
        ranked = sorted(run2[f"q{qi}"].items(), key=lambda kv: -kv[1])[:5]
        got = [int(d[1:]) for d, _ in ranked]
        # same top-5 up to near-ties: noise pages of one size embed close together, so allow the bf16 score noise (5e-3)
        assert (full_ref[qi, got] >= s_ref[qi, -1] - 5e-3).all() and len(set(got)) == 5
        assert abs(ranked[0][1] - s_ref[qi, 0]) <= 5e-3
        qrels[f"q{qi}"] = {ranked[0][0]: 1}
    m = I.save_results(str(tmp_path), qrels, run2)
    assert m["recall_10"] == 1.0 and m["mrr_10"] == 1.0 and m["ndcg_cut_10"] == 1.0


def test_mixed_resolution_corpus_recall_parity():
    """BASELINE configs[4] in miniature: pages with sides in [336, 1344] (1..10 slices, many distinct grids), dynamic
    grouping by geometry, Recall@1/5/10 of the engine's run vs the oracle's run on the same (query, corpus) set."""
    from oracle import restated as O
    from visrag_b200 import retriever as R
    from visrag_b200.config import VisRAGConfig
    from visrag_b200.synth import synth_queries
    from visrag_b200.tokenizer_stub import StubTokenizer
    from visrag_b200.weights import random_state_dict

    cfg = VisRAGConfig.tiny()
    sd = random_state_dict(cfg, 606)
    tok = StubTokenizer(cfg.vocab)
    rs = np.random.RandomState(44)
    sizes = [(int(rs.randint(336, 1345)), int(rs.randint(336, 1345))) for _ in range(14)] + [(1344, 1344), (336, 336), (448, 1344)]
    pages = synth_pages(sizes, 45)
    queries = synth_queries(6, 46)
    model = _engine_model(cfg, sd)
    _, p = model.encode_passage(_items([""] * len(pages), pages, "d"), tokenizer=tok, max_inp_length=2048)
    _, q = model.encode_query(_items(queries, [None] * len(queries), "q"), tokenizer=tok, max_inp_length=2048)
    p_ref = O.encode(sd, cfg, tok, [""] * len(pages), pages)
    q_ref = O.encode(sd, cfg, tok, queries, [None] * len(queries))
    assert cosine_rows(p.cpu().numpy(), p_ref).min() >= COS_MIN and cosine_rows(q.cpu().numpy(), q_ref).min() >= COS_MIN
    s_ref, i_ref = O.score_topk(q_ref, p_ref, 10)
    _, i_run = R.score_topk(q, R.build_index(p), 10)
    i_run = i_run.cpu().numpy()
    relevant = [{int(i_ref[qi, 0])} for qi in range(len(queries))]          # planted relevance = the oracle's best page
    for k in (1, 5, 10):
        assert O.recall_at_k(i_run, relevant, k) == O.recall_at_k(i_ref, relevant, k) == 1.0
    # identical top-10 up to bf16 near-ties (score gap below 2e-3)
    full = q_ref @ p_ref.T
    for qi in range(len(queries)):
        assert (full[qi, i_run[qi]] >= s_ref[qi, -1] - 2e-3).all()


def test_build_from_checkpoint_directory(tmp_path):
    """`DRModelForInference.build(model_args)` - what the reference driver's `setup_model` calls (`driver/eval.py:118-134`) - on
    a synthetic HF checkpoint directory in the public checkpoint's layout (config.json + sharded *.safetensors, bf16): the
    loaded model gives bit-identical embeddings to an engine built from the same state dict in memory and matches the
    oracle; `.to()` / `.eval()` return the model; the pickle shards it writes load with the reference's format reader.
    (The reference-side half - the unmodified driver driving these classes - is tests/test_dropin_reference_driver.py.)"""
    from types import SimpleNamespace

    from oracle import restated as O
    from visrag_b200 import inference as I
    from visrag_b200.config import VisRAGConfig
    from visrag_b200.modeling import DRModelForInference
    from visrag_b200.synth import synth_doc_pages
    from visrag_b200.tokenizer_stub import StubTokenizer
    from visrag_b200.weights import random_state_dict, save_checkpoint

    cfg = VisRAGConfig.tiny()
    sd = random_state_dict(cfg, 77)
    ckpt = str(tmp_path / "VisRAG-Ret-synthetic")
    save_checkpoint(ckpt, cfg, sd)
    margs = SimpleNamespace(model_name_or_path=ckpt, pooling="wmean", normalize=True, cache_dir=None)
    model = DRModelForInference.build(model_args=margs, cache_dir=None)
    assert model.to("cuda:0") is model and model.eval() is model and model.pooling == "wmean" and model.lm_q.config == cfg
    tok = StubTokenizer(cfg.vocab)
    pages = synth_doc_pages([(448, 448), (700, 900), (640, 300)], 31)
    batch = _items([""] * 3, pages, "d")
    got = model(passage=batch, tokenizer=tok, max_inp_length=2048).p_reps
    direct = _engine_model(cfg, sd)(passage=batch, tokenizer=tok, max_inp_length=2048).p_reps
    assert torch.equal(got, direct)
    assert cosine_rows(got.cpu().numpy(), O.encode(sd, cfg, tok, [""] * 3, pages)).min() >= COS_MIN
    args = SimpleNamespace(output_dir=str(tmp_path / "out"), per_device_eval_batch_size=2, max_inmem_docs=100, world_size=1,
                           process_index=0, device="cuda:0")
    I.distributed_parallel_embedding_inference([{"id": f"d{i}", "text": "", "image": im} for i, im in enumerate(pages)], model, args,
                                               "corpus", True, {"tokenizer": tok, "max_inp_length": 2048})
    import pickle

    with open(str(tmp_path / "out" / "embeddings.corpus.rank.0.0-3"), "rb") as f:
        emb, ids = pickle.load(f)                      # `dense_retriever.py:19-23`
    assert ids == ["d0", "d1", "d2"] and emb.dtype == np.float32 and np.array_equal(emb, got.cpu().numpy())
    # a config the packing code does not implement must be refused, not silently mis-tokenised
    import json

    bad = json.load(open(ckpt + "/config.json"))
    bad["slice_mode"] = False
    from visrag_b200.modeling import config_from_hf

    with pytest.raises(NotImplementedError):
        config_from_hf(bad)


def test_cuda_graph_path_is_bit_identical_to_eager_launches():
    """Small batches replay a captured CUDA graph of the same C-ABI launches (second sighting of a shape signature
    captures, later ones replay). Pages: new pixel content through the same graph; queries: different texts share a
    graph through the padded token buckets (one dummy sequence). Everything must equal the eager engine bit for bit."""
    from visrag_b200.config import VisRAGConfig
    from visrag_b200.encoder import VisRAGEngine
    from visrag_b200.tokenizer_stub import StubTokenizer
    from visrag_b200.weights import random_state_dict

    cfg = VisRAGConfig.tiny()
    sd = random_state_dict(cfg, 5)
    eager = VisRAGEngine(cfg, sd, cuda_graphs=False)
    graphed = VisRAGEngine(cfg, sd, cuda_graphs=True)
    tok = StubTokenizer(cfg.vocab)
    sizes = [(448, 448), (700, 900), (448, 448)]
    for seed in (1, 2, 3, 4):                       # same shapes, fresh pixels: eager, capture, replay, replay
        pages = synth_pages(sizes, seed)
        assert torch.equal(graphed.encode([""] * 3, pages, tok), eager.encode([""] * 3, pages, tok)), seed
    assert graphed.graph_stats == {"captured": 1, "replayed": 3, "eager": 1}
    queries = ["revenue table 2020", "a much longer question about the climate chart on page seven of the report",
               "cat", "dog on a sofa", "what is the total", "x"]
    for rep in range(2):
        for n in (1, 2, 3):                          # batches of different composition, several token buckets
            for i in range(0, len(queries) - n + 1):
                q = queries[i:i + n]
                for pooling in ("wmean", "lasttoken"):
                    a = graphed.encode(q, [None] * n, tok, pooling=pooling)
                    b = eager.encode(q, [None] * n, tok, pooling=pooling)
                    assert a.shape == (n, cfg.hidden) and torch.equal(a, b), (q, pooling)
    assert graphed.graph_stats["replayed"] > graphed.graph_stats["captured"] > 1
    assert eager.graph_stats == {"captured": 0, "replayed": 0, "eager": 0}
