"""Filtered retrieval on the H100: with a doc mask, score_topk returns exactly (torch.equal on scores and ids) the fp32
scan over the eligible docs alone, on the tensor-core filter path and on the plain scan, independent of batching; the
knowledge base's `within`, `remove`, `add` and `save` equal a fresh knowledge base of the same pages."""
import os

import numpy as np
import pytest
import torch

from visrag_b200 import _lib as L
from visrag_b200 import retriever as R

pytestmark = pytest.mark.gpu


def _unit(rs, n, d):
    x = rs.randn(n, d).astype(np.float32)
    return x / np.linalg.norm(x, axis=1, keepdims=True)


def _exact_scores(q: torch.Tensor, idx: R.CorpusIndex) -> torch.Tensor:
    """[nq, nd] fp32 scores from vr_score_exact: the bits both retrieval paths return."""
    out = torch.empty((q.shape[0], idx.nd), dtype=torch.float32, device=q.device)
    L.check(L.lib().vr_score_exact(q.data_ptr(), q.shape[0], idx.emb.data_ptr(), idx.nd, q.shape[1], out.data_ptr(),
                                   L.stream_ptr()))
    return out


def _reference(q, idx, k, mask: np.ndarray):
    """vr_score_exact scores, ineligible columns removed, sorted by (score desc, id asc), padded with (-inf, -1)."""
    full = _exact_scores(q, idx).cpu().numpy()
    cols = np.nonzero(mask)[0]
    s = full[:, cols]
    order = np.lexsort((np.broadcast_to(cols, s.shape), -s), axis=1)[:, :k]
    out_s = np.full((len(q), k), -np.inf, np.float32)
    out_i = np.full((len(q), k), -1, np.int64)
    out_s[:, :order.shape[1]] = np.take_along_axis(s, order, 1)
    out_i[:, :order.shape[1]] = cols[order]
    return torch.from_numpy(out_s).cuda(), torch.from_numpy(out_i).cuda()


def _masked(q, idx, k, mask, **kw):
    m = mask if isinstance(mask, torch.Tensor) else torch.from_numpy(mask).cuda()
    return R.score_topk(q, idx, k, doc_mask=m, **kw)


def _assert_same(a, b, what):
    (sa, ia), (sb, ib) = a, b
    assert torch.equal(ia, ib), (what, int((ia != ib).sum()))
    assert torch.equal(sa, sb), (what, float((sa - sb).abs().nan_to_num().max()))


def test_all_ones_mask_equals_no_mask():
    rs = np.random.RandomState(40)
    Q, D = _unit(rs, 1000, 256), _unit(rs, 20001, 256)
    q, idx = torch.from_numpy(Q).cuda(), R.build_index(D)
    ones = torch.ones(len(D), dtype=torch.bool, device="cuda")
    for kw in ({}, {"force_exact": True}):
        stats = {}
        got = R.score_topk(q, idx, 10, doc_mask=ones, stats=stats, **kw)
        assert stats["path"] == ("exact" if kw else "filter+rescore")
        _assert_same(got, R.score_topk(q, idx, 10, **kw), str(kw))
    _assert_same(R.score_topk(q[:2], idx, 10, doc_mask=ones), R.score_topk(q[:2], idx, 10), "two queries (chunked top-k)")


def _masks(rs, Q, D, idx):
    nd = len(D)
    single = np.zeros(nd, bool)
    single[4321] = True
    block = np.zeros(nd, bool)
    block[3000:3700] = True
    top16 = R.score_topk(torch.from_numpy(Q).cuda(), idx, 16, force_exact=True)[1].cpu().numpy()
    no_top = np.ones(nd, bool)
    no_top[np.unique(top16)] = False
    return {"random 50 %": rs.rand(nd) < 0.5, "random 1 %": rs.rand(nd) < 0.01, "single doc": single,
            "none": np.zeros(nd, bool), "contiguous block": block, "without every query's top-16": no_top}


def test_masked_topk_equals_the_masked_fp32_scan():
    """nd = 9999 (not a multiple of 32 or 256): the filter path (700 queries), the fp32 scan (force_exact) and the chunked
    top-k of few queries over the long index all equal the reference."""
    rs = np.random.RandomState(41)
    Q, D = _unit(rs, 700, 256), _unit(rs, 9999, 256)
    q, idx = torch.from_numpy(Q).cuda(), R.build_index(D)
    for name, m in _masks(rs, Q, D, idx).items():
        want = _reference(q, idx, 10, m)
        stats = {}
        _assert_same(_masked(q, idx, 10, m, stats=stats), want, name)
        assert stats["path"] == "filter+rescore"
        if name == "without every query's top-16":
            assert stats["flagged"] < len(Q) // 2, stats       # the filter answers, not the fallback
        _assert_same(_masked(q, idx, 10, m, force_exact=True), want, f"{name}, exact")
        _assert_same(_masked(q[:3], idx, 10, m), (want[0][:3], want[1][:3]), f"{name}, 3 queries")


def test_fewer_eligible_docs_than_k():
    rs = np.random.RandomState(42)
    Q, D = _unit(rs, 600, 128), _unit(rs, 12000, 128)
    q, idx = torch.from_numpy(Q).cuda(), R.build_index(D)
    m = np.zeros(len(D), bool)
    m[[5, 700, 701, 9000, 11999]] = True
    for kw in ({}, {"force_exact": True}):
        s, i = _masked(q, idx, 10, m, **kw)
        assert set(i[:, :5].flatten().tolist()) == {5, 700, 701, 9000, 11999}
        assert (i[:, 5:] == -1).all() and torch.isinf(s[:, 5:]).all() and (s[:, 5:] < 0).all()
        _assert_same((s, i), _reference(q, idx, 10, m), str(kw))


def _plan(nq, nd):
    out = np.zeros(6, np.int32)
    L.check(L.lib().vr_score_plan(nq, nd, out.ctypes.data))
    return dict(zip(("T", "R", "QB", "items", "pairs", "lists"), (int(v) for v in out)))


@pytest.mark.parametrize("nq,nd,d", [(17001, 20000, 64), (5001, 60000, 128)])
def test_filter_equals_exact_under_a_mask_over_several_waves(nq, nd, d):
    p = _plan(nq, nd)
    assert p["items"] > p["pairs"] and p["R"] > 1, p
    g = torch.Generator(device="cuda").manual_seed(nq)
    q = torch.nn.functional.normalize(torch.randn(nq, d, device="cuda", generator=g), dim=1)
    idx = R.build_index(torch.nn.functional.normalize(torch.randn(nd, d, device="cuda", generator=g), dim=1))
    for frac in (0.3, 0.02):
        m = torch.rand(nd, device="cuda", generator=g) < frac
        stats = {}
        got = _masked(q, idx, 10, m, stats=stats)
        assert stats["path"] == "filter+rescore"
        _assert_same(got, _masked(q, idx, 10, m, force_exact=True), f"{nq}x{nd} {frac}")


def test_clustered_corpus_under_a_mask_is_flagged_and_exact():
    rs = np.random.RandomState(43)
    d = 128
    D, Q = _unit(rs, 40000, d), _unit(rs, 1500, d)
    for qi in range(5):                               # 40 near-identical docs per query in one tile: lists overflow
        pert = Q[qi] + rs.randn(40, d).astype(np.float32) * 1e-4
        D[5000 + 300 * qi: 5040 + 300 * qi] = pert / np.linalg.norm(pert, axis=1, keepdims=True)
    m = rs.rand(len(D)) < 0.5
    for qi in range(5):
        m[5000 + 300 * qi: 5040 + 300 * qi] = True
    q, idx = torch.from_numpy(Q).cuda(), R.build_index(D)
    stats = {}
    got = _masked(q, idx, 10, m, stats=stats)
    assert stats["flagged"] > 0, stats
    _assert_same(got, _reference(q, idx, 10, m), "clustered")


def test_masked_query_alone_equals_its_row_in_a_batch_of_100():
    rs = np.random.RandomState(44)
    Q, D = _unit(rs, 100, 256), _unit(rs, 50000, 256)
    q, idx = torch.from_numpy(Q).cuda(), R.build_index(D)
    m = torch.from_numpy(rs.rand(len(D)) < 0.1).cuda()
    stats = {}
    s, i = _masked(q, idx, 7, m, stats=stats)
    assert stats["path"] == "filter+rescore"
    for r in (0, 42, 99):
        _assert_same(_masked(q[r:r + 1], idx, 7, m), (s[r:r + 1], i[r:r + 1]), f"query {r}")


@pytest.mark.parametrize("nq,nd,d", [(700, 33333, 256), (2600, 9000, 64), (300, 70001, 128)])
def test_masked_filter_lists_hold_eligible_docs_and_cover_the_eligible_top16(nq, nd, d):
    rs = np.random.RandomState(nq)
    Q, D = _unit(rs, nq, d), _unit(rs, nd, d)
    q, idx = torch.from_numpy(Q).cuda(), R.build_index(D)
    m = rs.rand(nd) < 0.25
    lib = L.lib()
    ranges, kt = lib.vr_score_ranges(nq, nd), lib.vr_score_list_len()
    lists = ranges * 2
    cand_s = torch.full((nq, lists * kt), float("nan"), device="cuda")
    cand_i = torch.full((nq, lists * kt), 0x7F7F7F7F, dtype=torch.int32, device="cuda")
    words = R.pack_doc_mask(torch.from_numpy(m).cuda())
    q16 = R.to_f16_rows(q)
    L.check(lib.vr_score_filter_masked(q16.data_ptr(), nq, idx.emb_f16.data_ptr(), nd, d, ranges, cand_s.data_ptr(),
                                       cand_i.data_ptr(), words.data_ptr(), L.stream_ptr()))
    torch.cuda.synchronize()
    ci, cs = cand_i.cpu().numpy().reshape(nq, lists, kt), cand_s.cpu().numpy().reshape(nq, lists, kt)
    assert not np.isnan(cs).any() and ((ci == -1) | ((ci >= 0) & (ci < nd))).all()
    assert m[ci[ci >= 0]].all()                                       # no ineligible doc in any list
    assert (cs[:, :, 1:] <= cs[:, :, :-1]).all()
    assert (np.isinf(cs) == (ci == -1))[:, :-1].all()
    approx = (q16.float() @ idx.emb_f16.float().T).cpu().numpy()
    approx[:, ~m] = -np.inf
    for r in rs.choice(nq, 40, replace=False):
        have = set(ci[r][ci[r] >= 0].tolist())
        kth = np.sort(approx[r])[-kt]
        must = set(np.nonzero(approx[r] > kth + 1e-4)[0].tolist())  # clear members of the eligible approximate top-16
        assert must <= have


def test_mask_of_the_wrong_shape_dtype_or_device_is_refused():
    rs = np.random.RandomState(45)
    idx = R.build_index(_unit(rs, 1000, 64))
    q = torch.from_numpy(_unit(rs, 3, 64)).cuda()
    for bad in (torch.ones(999, dtype=torch.bool, device="cuda"), torch.ones(1000, dtype=torch.uint8, device="cuda"),
                torch.ones(1000, dtype=torch.bool), torch.ones(1, 1000, dtype=torch.bool, device="cuda")):
        with pytest.raises(ValueError):
            R.score_topk(q, idx, 5, doc_mask=bad)


# ---------------------------------------------------------------------------------------------------- knowledge base


def _kb(path, D, names):
    from visrag_b200 import knowledge_base as KB

    KB.save_knowledge_base(str(path), D, names)
    return KB.KnowledgeBase(str(path))


def _by_name(kb, Q, k, **kw):
    s, i = kb.search(Q, k, **kw)
    return s.cpu(), [[kb.filenames[j] for j in row] for row in i.tolist()]


def test_knowledge_base_within_remove_add_and_save(tmp_path):
    """Each operation equals a fresh knowledge base of the pages it leaves searchable: same filenames, same score bits.
    1 query takes the fp32 scan, 300 queries the tensor-core filter."""
    from visrag_b200 import knowledge_base as KB

    rs = np.random.RandomState(46)
    D = _unit(rs, 30000, 256)
    names = [f"doc{i // 100}.pdf_{i % 100}.png" for i in range(len(D))]
    kb = _kb(tmp_path / "kb", D, names)
    Q = _unit(rs, 300, 256)
    # within: one PDF, and a scattered subset
    for sel in ([i for i in range(len(D)) if names[i].startswith("doc7.pdf_")], sorted(rs.choice(len(D), 9000, replace=False))):
        fresh = _kb(tmp_path / f"w{len(sel)}", D[sel], [names[i] for i in sel])
        for nq in (1, 300):
            s, n = _by_name(kb, Q[:nq], 10, within=[names[i] for i in sel])
            s2, n2 = _by_name(fresh, Q[:nq], 10)
            assert n == n2 and torch.equal(s, s2), (len(sel), nq)
    assert kb.retrieve(Q[:1], 3, within=["doc7.pdf_3.png"]) == [os.path.join(str(tmp_path / "kb"), "doc7.pdf_3.png")]
    with pytest.raises(KeyError):
        kb.search(Q, 5, within=["no such page.png"])
    # remove + add
    gone = sorted(rs.choice(len(D), 5000, replace=False))
    live = [i for i in range(len(D)) if i not in set(gone)]
    kb.remove([names[i] for i in gone])
    assert len(kb) == len(D) - 5000
    with pytest.raises(KeyError):
        kb.search(Q, 5, within=[names[gone[0]]])
    with pytest.raises(KeyError):
        kb.remove([names[gone[0]]])
    new = _unit(rs, 2000, 256) * 1.5                 # a larger norm: the filter's bound must grow with it
    new_names = [f"new.pdf_{i}.png" for i in range(2000)]
    with pytest.raises(ValueError):
        kb.add(new[:2], [names[live[0]], "x.png"])    # a live page's name
    kb.add(new[:1000], new_names[:1000])
    kb.add(new[1000:], new_names[1000:])
    assert len(kb) == len(D) - 5000 + 2000
    all_D, all_names = np.concatenate([D[live], new]), [names[i] for i in live] + new_names
    fresh = _kb(tmp_path / "fresh", all_D, all_names)
    assert torch.equal(kb.index.max_norm, fresh.index.max_norm)
    for nq in (1, 300):
        s, n = _by_name(kb, Q[:nq], 10)
        s2, n2 = _by_name(fresh, Q[:nq], 10)
        assert n == n2 and torch.equal(s, s2), nq
    # save, reload
    kb.save(str(tmp_path / "saved"))
    again = KB.KnowledgeBase(str(tmp_path / "saved"))
    assert again.filenames == all_names
    for nq in (1, 300):
        s, n = _by_name(kb, Q[:nq], 10)
        s2, n2 = _by_name(again, Q[:nq], 10)
        assert n == n2 and torch.equal(s, s2), nq


def _nccl_worker(rank, world, port, out_q):
    import torch.distributed as dist

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device(f"cuda:{rank}"))
    try:
        dev = f"cuda:{rank}"
        g = torch.Generator(device=dev).manual_seed(4321)           # same stream on every rank: the full corpus and mask
        D = torch.nn.functional.normalize(torch.randn(12000, 256, device=dev, generator=g), dim=1)
        Q = torch.nn.functional.normalize(torch.randn(1000, 256, device=dev, generator=g), dim=1)
        mask = torch.rand(12000, device=dev, generator=g) < 0.3
        lo, hi = R.shard_range(D.shape[0], rank, world)
        index = R.build_index(D[lo:hi].contiguous())
        stats = {}
        s, i = R.sharded_topk(Q, index, 10, lo, stats=stats, doc_mask=mask[lo:hi].contiguous())
        cols = torch.nonzero(mask).flatten()
        ref = torch.topk(Q @ D[cols].T, 10, dim=1)                  # brute-force fp32 scan of the eligible docs
        ok = bool(torch.equal(i, cols[ref.indices])) and float((s - ref.values).abs().max()) <= 2e-6
        out_q.put((rank, ok, stats.get("path")))
    finally:
        dist.destroy_process_group()


def test_sharded_topk_with_per_rank_masks_under_nccl():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    import torch.multiprocessing as mp

    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29700 + (os.getpid() + 500) % 1000
    procs = [ctx.Process(target=_nccl_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=300) for _ in procs]
    for p in procs:
        p.join(60)
    assert sorted(r[0] for r in res) == [0, 1] and all(r[1] for r in res), res
