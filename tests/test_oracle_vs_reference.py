"""Pins the oracle against outputs of the REAL reference on this file's own seeded inputs. The reference outputs are stored
in tests/golden/reference_pins.npz (written by `python -m oracle.gen_golden --pins` where a checkout of the reference is
available), so the comparison runs everywhere. Two cross-reads are checked only when the pins are generated, not here: the
reference's shard reader unpickling a shard written by `retriever.save_shard`, and the reference's `load_from_trec` reading a
run file written by OUR writer (the generator asserts both; this file reads the reference's run file with OUR reader)."""
import json
import os

import numpy as np
import pytest

from tests.conftest import GOLDEN


@pytest.fixture(scope="module")
def pins():
    return np.load(os.path.join(GOLDEN, "reference_pins.npz"))


def test_restatement_equals_reference_on_fresh_inputs(pins):
    from oracle import restated as O
    from tests.helpers import QUERY_PREFIX, synth_pages
    from visrag_b200.config import VisRAGConfig
    from visrag_b200.tokenizer_stub import StubTokenizer
    from visrag_b200.weights import random_state_dict

    cfg = VisRAGConfig.tiny()
    sd = random_state_dict(cfg, 777)
    tok = StubTokenizer(cfg.vocab)
    pages = synth_pages([(300, 300), (1000, 600), (448, 448)], 21)
    items = [{"id": str(i), "text": "doc text" if i == 1 else "", "image": im} for i, im in enumerate(pages)]
    p_ref = pins["fresh_pages"]
    p = O.encode(sd, cfg, tok, [it["text"] for it in items], pages)
    assert np.abs(p - p_ref).max() < 2e-6
    qs = [QUERY_PREFIX + "what is shown", QUERY_PREFIX + "x"]
    q_ref = pins["fresh_queries"]
    assert np.abs(O.encode(sd, cfg, tok, qs, [None, None]) - q_ref).max() < 2e-6
    # B1 boundary: hidden states of the valid positions
    hs, mask = pins["fresh_hidden"], pins["fresh_mask"]
    _, hid = O.encode(sd, cfg, tok, [it["text"] for it in items], pages, return_hidden=True)
    for b, h in enumerate(hid):
        n = int(mask[b].sum())
        assert n == h.shape[0] and np.abs(hs[b, :n] - h).max() < 5e-5


@pytest.mark.parametrize("pooling", ["lasttoken", "mean", "cls"])
def test_other_poolings_equal_reference_on_a_ragged_batch(pooling, pins):
    """SURVEY.md §8f.4: the pooling variants of `dense_retrieval_model.py:170-218` on a right-padded batch of unequal
    lengths (the oracle and the engine pool unpadded sequences; this pins that they mean the same thing)."""
    from oracle import restated as O
    from tests.helpers import QUERY_PREFIX, synth_pages
    from visrag_b200.config import VisRAGConfig
    from visrag_b200.tokenizer_stub import StubTokenizer
    from visrag_b200.weights import random_state_dict

    cfg = VisRAGConfig.tiny()
    sd = random_state_dict(cfg, 778)
    tok = StubTokenizer(cfg.vocab)
    page = synth_pages([(448, 448)], 5)[0]
    texts = [QUERY_PREFIX + "a", QUERY_PREFIX + "a much longer query about the page content", ""]
    images = [None, None, page]
    ref = pins[f"pooling_{pooling}"]
    got = O.encode(sd, cfg, tok, texts, images, pooling=pooling)
    assert np.abs(got - ref).max() < 2e-6, pooling


def test_score_topk_and_run_files_equal_reference(tmp_path, pins):
    """The scoring side of the path against the REAL reference functions' stored results: `_retrieve_one_shard`
    (`retriever/dense_retriever.py:13-34`) on a pickle shard written by our writer, `save_as_trec` / `load_from_trec` /
    `eval_mrr` (`utils.py:125-175,285-308`). Random unit vectors: no score ties, so torch.topk's unspecified tie order cannot differ."""
    import pickle

    from oracle import restated as O
    from visrag_b200 import inference as I
    from visrag_b200 import retriever as R

    rs = np.random.RandomState(12)
    D = rs.randn(500, 64).astype(np.float32)
    D /= np.linalg.norm(D, axis=1, keepdims=True)
    Q = rs.randn(7, 64).astype(np.float32)
    Q /= np.linalg.norm(Q, axis=1, keepdims=True)
    lookup = [f"doc{i}" for i in range(len(D))]
    shard = str(tmp_path / "embeddings.corpus.rank.0")
    R.save_shard(shard, D, lookup)                      # our writer, in the layout the reference's reader unpickles
    assert pickle.load(open(shard, "rb"))[1] == lookup
    s_ref, i_ref = pins["topk_scores"], pins["topk_indices"]
    s, i = O.score_topk(Q, D, 10)
    assert np.array_equal(i, i_ref) and np.abs(s - s_ref).max() < 1e-6
    # run files and MRR: our functions write and read what the reference's wrote and read, and agree on the measures
    run = {f"q{q}": {lookup[j]: float(s_ref[q, r]) for r, j in enumerate(i_ref[q])} for q in range(len(Q))}
    qrel = {f"q{q}": {lookup[int(i_ref[q, q % 10])]: 1} for q in range(len(Q))}
    ours, theirs = str(tmp_path / "ours.trec"), str(tmp_path / "theirs.trec")
    I.save_as_trec(run, ours)
    open(theirs, "w").write(str(pins["trec_text"]))
    assert open(ours).read() == open(theirs).read()
    assert json.loads(str(pins["trec_loaded"])) == json.loads(json.dumps(I.load_from_trec(theirs), sort_keys=True))
    assert json.loads(str(pins["mrr"])) == json.loads(json.dumps([I.eval_mrr(qrel, run, 10), I.eval_mrr(qrel, run, 3)], sort_keys=True))
