"""Similarity + top-k on the H100 against the oracle's fp32 scan: ids bit-identical (tie rule: score desc, id asc),
scores within fp32 summation-order noise (2e-6 on unit vectors)."""
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from oracle import restated as O

pytestmark = pytest.mark.gpu


def _unit(rs, n, d):
    x = rs.randn(n, d).astype(np.float32)
    return x / np.linalg.norm(x, axis=1, keepdims=True)


def _run(Q, D, k, **kw):
    from visrag_b200 import retriever as R

    idx = R.build_index(D)
    stats = {}
    s, i = R.score_topk(torch.from_numpy(Q).cuda(), idx, k, stats=stats, **kw)
    return s.cpu().numpy(), i.cpu().numpy(), stats


@pytest.mark.parametrize("nq,nd,d,k", [(300, 5000, 256, 10), (1000, 10000, 2304, 10), (129, 4097, 2304, 5), (4, 32, 256, 5),
                                       (2049, 20000, 64, 16), (1, 100000, 128, 10), (3, 300000, 64, 12)])
def test_topk_equals_fp32_scan(nq, nd, d, k):
    rs = np.random.RandomState(nq + nd)
    Q, D = _unit(rs, nq, d), _unit(rs, nd, d)
    s, i, stats = _run(Q, D, k)
    s_ref, i_ref = O.score_topk(Q, D, k)
    assert np.array_equal(i, i_ref), stats
    assert np.abs(s - s_ref).max() <= 2e-6
    if nq * nd > (1 << 22) and nd >= 256:
        assert stats["path"] == "filter+rescore"


def test_ties_duplicates_and_short_corpus():
    rs = np.random.RandomState(3)
    base = _unit(rs, 3000, 128)
    D = np.concatenate([base, base[:500]])          # 500 exact duplicates -> exact score ties
    Q = _unit(rs, 2000, 128)
    s, i, stats = _run(Q, D, 10)
    s_ref, i_ref = O.score_topk(Q, D, 10)
    assert np.array_equal(i, i_ref) and stats["path"] == "filter+rescore"
    # k > nd: tail is (-inf, -1)
    s, i, _ = _run(Q[:3], D[:4], 6)
    assert (i[:, 4:] == -1).all() and np.isinf(s[:, 4:]).all() and np.array_equal(i[:, :4], O.score_topk(Q[:3], D[:4], 4)[1])


def test_clustered_corpus_takes_the_exact_fallback_and_stays_correct():
    """More than 16 near-identical relevant docs inside one doc range defeat the per-range top-16 filter; the proof
    step must notice (flag) and the fp32 fallback must still return the exact answer. The planted docs score within
    ~1e-7 of each other, i.e. inside fp32 summation-order noise, so ids are compared through their oracle scores:
    every returned doc must score (by the oracle) at least the oracle's k-th score minus 2e-6."""
    rs = np.random.RandomState(4)
    d = 128
    D = _unit(rs, 40000, d)
    Q = _unit(rs, 1500, d)
    for qi in range(5):                               # 40 docs within ~1e-3 of query qi, all inside one doc tile
        pert = Q[qi] + rs.randn(40, d).astype(np.float32) * 1e-4
        D[5000 + 300 * qi: 5040 + 300 * qi] = pert / np.linalg.norm(pert, axis=1, keepdims=True)
    s, i, stats = _run(Q, D, 10)
    s_ref, i_ref = O.score_topk(Q, D, 10)
    assert stats["flagged"] >= 5
    assert np.abs(s - s_ref).max() <= 2e-6 and (np.diff(s, axis=1) <= 0).all()
    full = Q @ D.T
    got_scores = np.take_along_axis(full, i, axis=1)
    assert (got_scores >= s_ref[:, -1:] - 2e-6).all()
    assert np.array_equal(i[5:], i_ref[5:])           # unperturbed queries: no near-ties, ids identical
    assert all(len(set(r)) == 10 for r in i)
    s2, i2, st2 = _run(Q[5:55], D, 10, force_exact=True)
    assert st2["path"] == "exact" and np.array_equal(i2, i_ref[5:55])


def test_large_problem_sets_match_torch_fp32():
    """BASELINE config-3 scale (1 k x 10 k x 2304) and a 200 k corpus: compare with torch fp32 matmul + topk on the GPU."""
    from visrag_b200 import retriever as R

    g = torch.Generator(device="cuda").manual_seed(0)
    for nq, nd in ((1000, 10000), (512, 200000)):
        Dm = torch.nn.functional.normalize(torch.randn(nd, 2304, device="cuda", generator=g), dim=1)
        Qm = torch.nn.functional.normalize(torch.randn(nq, 2304, device="cuda", generator=g), dim=1)
        idx = R.build_index(Dm)
        s, i = R.score_topk(Qm, idx, 10)
        prev = torch.backends.cuda.matmul.allow_tf32
        torch.backends.cuda.matmul.allow_tf32 = False
        ts, ti = torch.topk(Qm @ Dm.T, 10, dim=1)
        torch.backends.cuda.matmul.allow_tf32 = prev
        assert torch.equal(torch.sort(i, 1).values, torch.sort(ti, 1).values)
        assert (s - ts).abs().max().item() <= 5e-6


def test_reference_signature_drop_ins(tmp_path):
    from visrag_b200 import retriever as R

    rs = np.random.RandomState(8)
    D, Q = _unit(rs, 700, 256), _unit(rs, 9, 256)
    out = str(tmp_path)
    R.save_shard(os.path.join(out, "embeddings.corpus.rank.0.0-400"), D[:400], [f"d{i}" for i in range(400)])
    R.save_shard(os.path.join(out, "embeddings.corpus.rank.1.0-300"), D[400:], [f"d{i}" for i in range(400, 700)])
    R.save_shard(os.path.join(out, "embeddings.query.rank.0"), Q, [f"q{i}" for i in range(9)])
    s, i, lookup = R._retrieve_one_shard(os.path.join(out, "embeddings.corpus.rank.0.0-400"), torch.from_numpy(Q).cuda(), 5, "cuda:0")
    assert s.shape == (9, 5) and i.dtype == torch.int64 and lookup[3] == "d3"
    assert np.array_equal(i.cpu().numpy(), O.score_topk(Q, D[:400], 5)[1])
    res = R.distributed_parallel_retrieve(SimpleNamespace(output_dir=out, process_index=0, device="cuda:0"), 5)
    assert set(res) == {f"q{i}" for i in range(9)}
    _, gi = O.score_topk(Q, D, 5)
    for qn in range(9):
        run = sorted(res[f"q{qn}"].items(), key=lambda kv: (-kv[1], kv[0]))
        assert len(run) == 10                                    # union of two shards' top-5, like the reference
        assert {int(x[0][1:]) for x in run[:5]} == set(gi[qn].tolist())


def test_merge_topk_kernel():
    from visrag_b200 import retriever as R

    rs = np.random.RandomState(2)
    s = rs.randn(50, 24).astype(np.float32)
    i = np.stack([rs.permutation(1000)[:24] for _ in range(50)]).astype(np.int64)
    i[:, 20:] = -1
    ms, mi = R.merge_topk(torch.from_numpy(s).cuda(), torch.from_numpy(i).cuda(), 7)
    ws, wi = O.merge_topk([(s[:, :20], i[:, :20])], 7)
    assert np.array_equal(mi.cpu().numpy(), wi) and np.allclose(ms.cpu().numpy(), ws)


def test_knowledge_base_single_query_retrieval(tmp_path):
    """Demo layout (reps.npy + index2img_filename.txt): resident index, one query -> top-k page paths; equals the
    fp32 scan the reference's answer.py does (torch.matmul + topk), ties by lower page index."""
    from visrag_b200 import knowledge_base as KB

    rs = np.random.RandomState(8)
    D = _unit(rs, 50000, 256)
    D[123] = D[77]                                  # an exact duplicate page -> a score tie
    names = [f"doc.pdf_{i}.png" for i in range(len(D))]
    KB.save_knowledge_base(str(tmp_path), D, names)
    kb = KB.KnowledgeBase(str(tmp_path))
    assert len(kb) == 50000
    q = D[77:78] + 0.01 * _unit(rs, 1, 256)
    q /= np.linalg.norm(q)
    paths = kb.retrieve(q, 5)
    s_ref, i_ref = O.score_topk(q.astype(np.float32), D, 5)
    assert paths == [os.path.join(str(tmp_path), names[i]) for i in i_ref[0]]
    assert i_ref[0][0] == 77 and i_ref[0][1] == 123
    s, i = kb.search(q, 5)
    assert np.abs(s.cpu().numpy() - s_ref).max() <= 2e-6
    # several queries at once and k larger than the index
    s, i = kb.search(D[:4], 3)
    assert np.array_equal(i.cpu().numpy()[:, 0], np.arange(4))
    small = KB.KnowledgeBase.__new__(KB.KnowledgeBase)
    KB.save_knowledge_base(str(tmp_path / "s"), D[:3], names[:3])
    small.__init__(str(tmp_path / "s"))
    assert len(small.retrieve(D[:1], 10)) == 3


from visrag_b200 import retriever as R  # noqa: E402  (importing does not load the CUDA library)


def _nccl_worker(rank, world, port, out_q):
    import os

    import torch.distributed as dist

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device(f"cuda:{rank}"))
    try:
        dev = f"cuda:{rank}"
        g = torch.Generator(device=dev).manual_seed(1234)           # same stream on every rank: the FULL corpus / query set
        D = torch.nn.functional.normalize(torch.randn(12000, 256, device=dev, generator=g), dim=1)  # 6000 per shard: filter path
        Q = torch.nn.functional.normalize(torch.randn(1000, 256, device=dev, generator=g), dim=1)
        lo, hi = R.shard_range(D.shape[0], rank, world)
        index = R.build_index(D[lo:hi].contiguous())
        # queries sharded for "encoding" (here: each rank simply owns a slice), gathered, then the partial-top-k exchange
        qlo, qhi = R.shard_range(Q.shape[0], rank, world)
        q_all = R.gather_queries(Q[qlo:qhi].contiguous(), Q.shape[0])
        ok = bool(torch.equal(q_all, Q))
        stats = {}
        s, i = R.sharded_topk(q_all, index, 10, lo, stats=stats)
        ref = torch.topk(Q @ D.T, 10, dim=1)                         # brute-force fp32 scan of the whole corpus
        ok = ok and bool(torch.equal(i, ref.indices)) and float((s - ref.values).abs().max()) <= 2e-6
        out_q.put((rank, ok, stats.get("path")))
    finally:
        dist.destroy_process_group()


def test_sharded_topk_under_nccl_equals_the_brute_force_scan():
    """World-size-2 NCCL run on two real GPUs (skipped on a one-GPU machine): query all-gather + partial-top-k all-gather +
    merge kernel give exactly the ids of a brute-force fp32 scan of the unsharded corpus, on every rank."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    import os

    import torch.multiprocessing as mp

    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29700 + os.getpid() % 1000
    procs = [ctx.Process(target=_nccl_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=300) for _ in procs]
    for p in procs:
        p.join(60)
    assert sorted(r[0] for r in res) == [0, 1] and all(r[1] for r in res), res
    assert all(r[2] == "filter+rescore" for r in res)


def test_engine_and_index_on_a_non_current_device():
    """Kernels must launch on the device that owns the buffers, not on the process's current device."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    from tests.helpers import cosine_rows, synth_pages
    from visrag_b200.config import VisRAGConfig
    from visrag_b200.encoder import VisRAGEngine
    from visrag_b200.tokenizer_stub import StubTokenizer
    from visrag_b200.weights import random_state_dict

    torch.cuda.set_device(0)
    cfg = VisRAGConfig.tiny()
    sd = random_state_dict(cfg, 11)
    tok = StubTokenizer(cfg.vocab)
    pages = synth_pages([(448, 448), (700, 900)], 4)
    e0, e1 = VisRAGEngine(cfg, sd, "cuda:0"), VisRAGEngine(cfg, sd, "cuda:1")
    a = e0.encode(["", ""], pages, tok)
    b = e1.encode(["", ""], pages, tok)          # cuda:0 is still the current device
    assert b.device.index == 1 and torch.cuda.current_device() == 0
    assert torch.equal(a.cpu(), b.cpu())
    rs = np.random.RandomState(0)
    D = rs.randn(9000, 256).astype(np.float32)
    Q = rs.randn(600, 256).astype(np.float32)
    i0 = R.score_topk(torch.from_numpy(Q).to("cuda:0"), R.build_index(D, device="cuda:0"), 10)[1]
    i1 = R.score_topk(torch.from_numpy(Q).to("cuda:1"), R.build_index(D, device="cuda:1"), 10)[1]
    assert torch.equal(i0.cpu(), i1.cpu())


def test_non_finite_and_out_of_fp16_range_inputs_fall_back_to_the_fp32_scan():
    """|x| > 65504 or NaN would become inf/NaN in the fp16 copies; the rescoring kernel flags those queries (or
    every query when the corpus is affected) and the fp32 scan answers them."""
    rs = np.random.RandomState(3)
    D = rs.randn(8000, 256).astype(np.float32)
    Q = rs.randn(700, 256).astype(np.float32)
    Q[5] *= 1e6                                  # fp16 overflow in one query
    Dbig = D.copy()
    Dbig[17] *= 1e6                              # fp16 overflow in one document: the whole index is affected
    for dd in (D, Dbig):
        stats = {}
        s, i = R.score_topk(torch.from_numpy(Q).cuda(), R.build_index(dd), 10, stats=stats)
        ref = torch.topk(torch.from_numpy(Q).cuda().double() @ torch.from_numpy(dd).cuda().double().T, 10, dim=1)
        assert torch.equal(i, ref.indices), stats
        assert stats["flagged"] >= 1


@pytest.mark.parametrize("nq,nd,d", [(700, 33333, 256), (257, 70001, 128), (2600, 9000, 64), (100, 50000, 2304)])
def test_filter_candidate_lists_cover_every_query_block_piece(nq, nd, d):
    """The filter's work split (query block x doc range items dealt round-robin to the CTA pairs) must leave every list
    slot of every query written: a real sorted list or an empty one. Buffers are poisoned first; then the union of a query's lists has
    to contain the fp16-approximate top-16 of the whole corpus (every list keeps the best 16 of its span)."""
    from visrag_b200 import _lib as L
    from visrag_b200 import retriever as R

    rs = np.random.RandomState(nq)
    Q, D = _unit(rs, nq, d), _unit(rs, nd, d)
    q = torch.from_numpy(Q).cuda()
    idx = R.build_index(D)
    lib = L.lib()
    ranges = lib.vr_score_ranges(nq, nd)
    kt = lib.vr_score_list_len()
    lists = ranges * 2
    cand_s = torch.full((nq, lists * kt), float("nan"), device="cuda")
    cand_i = torch.full((nq, lists * kt), 0x7F7F7F7F, dtype=torch.int32, device="cuda")
    q16 = R.to_f16_rows(q)
    L.check(lib.vr_score_filter(q16.data_ptr(), nq, idx.emb_f16.data_ptr(), nd, d, ranges, cand_s.data_ptr(), cand_i.data_ptr(),
                                L.stream_ptr()))
    torch.cuda.synchronize()
    ci, cs = cand_i.cpu().numpy().reshape(nq, lists, kt), cand_s.cpu().numpy().reshape(nq, lists, kt)
    assert not np.isnan(cs).any() and ((ci == -1) | ((ci >= 0) & (ci < nd))).all()
    assert (cs[:, :, 1:] <= cs[:, :, :-1]).all()                  # every list sorted descending (empties are -inf)
    assert (np.isinf(cs) == (ci == -1))[:, :-1].all()             # (the last slot's first score is the query's threshold)
    assert (ci[:, -1] == -1).all()
    approx = (q16.float() @ idx.emb_f16.float().T).cpu().numpy()  # fp16 operands, fp32 accumulate like the filter
    for r in rs.choice(nq, 40, replace=False):
        have = set(ci[r][ci[r] >= 0].tolist())
        assert len(have) == (ci[r] >= 0).sum()                    # no doc in two lists
        kth = np.sort(approx[r])[-kt]
        must = set(np.nonzero(approx[r] > kth + 1e-4)[0].tolist())  # clear members of the approximate top-16
        assert must <= have


# ------------------------------------------------------------------------------------------------------------------------
# The top-k does not depend on the path that answers it (tensor-core filter + exact rescoring, or the plain fp32 scan), on
# the other queries of the batch, or on how the corpus is sharded: the same scores and ids, bit for bit. The rescoring
# kernel and the fp32 scan sum a dot product in the same lane-strided FMA order and the same butterfly.


def _topk(Q, idx, k, **kw):
    return R.score_topk(torch.from_numpy(Q).cuda() if isinstance(Q, np.ndarray) else Q, idx, k, **kw)


def _assert_same(a, b, what):
    (sa, ia), (sb, ib) = a, b
    assert torch.equal(ia, ib), (what, int((ia != ib).sum()))
    assert torch.equal(sa, sb), (what, float((sa - sb).abs().max()))


def _corpora():
    rs = np.random.RandomState(31)
    yield "random", _unit(rs, 1000, 2304), _unit(rs, 10000, 2304), [10]
    base = _unit(rs, 3000, 128)
    yield "exact duplicates", _unit(rs, 2000, 128), np.concatenate([base, base[:500]]), [10]
    D = _unit(rs, 40000, 128)
    Q = _unit(rs, 1500, 128)
    for qi in range(5):                               # the clustered corpus: the filter flags these, the fp32 scan answers
        pert = Q[qi] + rs.randn(40, 128).astype(np.float32) * 1e-4
        D[5000 + 300 * qi: 5040 + 300 * qi] = pert / np.linalg.norm(pert, axis=1, keepdims=True)
    yield "clustered", Q, D, [10]
    yield "k 17 to 300", _unit(rs, 500, 256), _unit(rs, 20000, 256), [17, 64, 300]
    D = rs.randn(8000, 256).astype(np.float32)
    Q = rs.randn(700, 256).astype(np.float32)
    Q[5] *= 1e6
    yield "fp16-overflow query", Q, D, [10]
    Dbig = D.copy()
    Dbig[17] *= 1e6
    yield "fp16-overflow document", Q, Dbig, [10]


def test_filter_path_equals_the_exact_scan_bit_for_bit():
    for name, Q, D, ks in _corpora():
        idx = R.build_index(D)
        for k in ks:
            stats = {}
            got = _topk(Q, idx, k, stats=stats)
            assert stats["path"] == "filter+rescore", (name, stats)
            _assert_same(got, _topk(Q, idx, k, force_exact=True), f"{name} k={k}")


def test_one_query_alone_equals_the_same_query_in_a_batch():
    """Alone, one query over 20000 docs takes the fp32 scan with the chunked top-k; in a batch of 2000 it takes the filter."""
    rs = np.random.RandomState(12)
    Q, D = _unit(rs, 2000, 256), _unit(rs, 20000, 256)
    idx = R.build_index(D)
    batch = _topk(Q, idx, 10)
    for r in (0, 777, 1999):
        _assert_same(_topk(Q[r:r + 1], idx, 10), (batch[0][r:r + 1], batch[1][r:r + 1]), f"query {r}")


def test_three_shards_merged_equal_the_unsharded_index():
    """sharded_topk on one GPU: each shard's top-k with its global id offset, then merge_topk."""
    rs = np.random.RandomState(13)
    Q, D = _unit(rs, 500, 256), _unit(rs, 30001, 256)
    D[20000] = D[3]                                   # a tie across shards: the lower global id wins
    q = torch.from_numpy(Q).cuda()
    want = _topk(q, R.build_index(D), 10)
    parts = []
    for r in range(3):
        lo, hi = R.shard_range(len(D), r, 3)
        parts.append(_topk(q, R.build_index(D[lo:hi]), 10, id_offset=lo))
    got = R.merge_topk(torch.cat([p[0] for p in parts], 1), torch.cat([p[1] for p in parts], 1), 10)
    _assert_same(got, want, "3 shards")


def test_knowledge_base_one_query_equals_a_batch_of_100(tmp_path):
    from visrag_b200 import knowledge_base as KBase

    rs = np.random.RandomState(14)
    D = _unit(rs, 50000, 256)
    KBase.save_knowledge_base(str(tmp_path), D, [f"p{i}.png" for i in range(len(D))])
    kb = KBase.KnowledgeBase(str(tmp_path))
    Q = _unit(rs, 100, 256)
    s, i = kb.search(Q, 7)
    for r in (0, 42, 99):
        _assert_same(kb.search(Q[r:r + 1], 7), (s[r:r + 1], i[r:r + 1]), f"query {r}")


def test_exact_scan_takes_more_than_65535_query_blocks():
    """8 x 65535 + 9 queries: more query blocks of the fp32 scan than one launch's grid.y holds. The index needs a
    dimension divisible by 8; with 3 docs this is 17 MB of queries."""
    nq = 8 * 65535 + 9
    g = torch.Generator(device="cuda").manual_seed(15)
    q = torch.randn(nq, 8, device="cuda", generator=g)
    idx = R.build_index(torch.randn(3, 8, device="cuda", generator=g))
    stats = {}
    whole = _topk(q, idx, 2, stats=stats)
    assert stats["path"] == "exact"
    h = nq // 2
    a, b = _topk(q[:h].contiguous(), idx, 2), _topk(q[h:].contiguous(), idx, 2)
    _assert_same(whole, (torch.cat([a[0], b[0]]), torch.cat([a[1], b[1]])), "two halves")
