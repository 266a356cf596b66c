"""Hybrid retrieval on the H100: score_topk_hybrid and score_topk_groups_hybrid return exactly (torch.equal on ids and
score bits) a brute-force reference - vr_score_exact over every page, the torch fp32 add dense + w * v on the full
matrix, and a stable (score desc, id asc) order - on every route of score_topk (scan, filter and rescore, masks,
per-query masks, lists, deep k), for RRF windows of 10, 100 and 1000, for documents of 1, 8 and 64 pages, batch by
batch and query by query, with hit lists longer than any shared-memory table, and through the knowledge base."""

import numpy as np
import pytest
import torch

from tests.test_hybrid_host import order, rrf_full
from visrag_b200 import _lib as L
from visrag_b200 import retriever as R
from visrag_b200.knowledge_base import KnowledgeBase, save_knowledge_base

pytestmark = pytest.mark.gpu


def _unit(rs, n, d):
    x = rs.randn(n, d).astype(np.float32)
    return x / np.linalg.norm(x, axis=1, keepdims=True)


def _exact(q, idx):
    out = torch.empty((q.shape[0], idx.nd), dtype=torch.float32, device=q.device)
    L.check(L.lib().vr_score_exact(q.data_ptr(), q.shape[0], idx.emb.data_ptr(), idx.nd, q.shape[1], out.data_ptr(),
                                   L.stream_ptr()))
    return out


def _hits(rs, S, n_max, lift=2.0, long_row=None):
    """Per query: some random pages (values up to `lift`, enough to lift a page from anywhere into the top-k), some of
    its dense top-20 (pages in both sets) and value-0 pages; long_row: (row, length) of one very long list."""
    nq, nd = S.shape
    top = torch.topk(S, 20, dim=1).indices.cpu().numpy()
    offsets, ids, vals = [0], [], []
    for r in range(nq):
        n = long_row[1] if long_row and long_row[0] == r else int(rs.randint(0, n_max + 1))
        pages = set(rs.choice(nd, size=min(n, nd), replace=False).tolist())
        pages |= set(top[r, rs.randint(0, 20, 3)].tolist()) if n else set()
        pages = sorted(pages)
        rs.shuffle(pages)
        v = (rs.rand(len(pages)) * lift).astype(np.float32)
        v[rs.rand(len(pages)) < 0.1] = 0.0
        v[rs.rand(len(pages)) < 0.1] = np.float32(0.5)  # ties in the external ranks
        v[rs.rand(len(pages)) < 0.05] = np.float32(-0.0)  # a zero score with the sign bit set
        ids += pages
        vals += v.tolist()
        offsets.append(len(ids))
    dev = S.device
    return (torch.tensor(offsets, dtype=torch.int64, device=dev), torch.tensor(ids, dtype=torch.int32, device=dev),
            torch.tensor(vals, dtype=torch.float32, device=dev))


def _dense_matrix(hits, nq, nd):
    off, ids, vals = hits
    V = torch.zeros((nq, nd), dtype=torch.float32, device=ids.device)
    row = torch.repeat_interleave(torch.arange(nq, device=ids.device), off[1:] - off[:-1])
    V[row, ids.long()] = vals
    return V


def _elig_rows(elig, nq, nd):
    if elig is None:
        return [None] * nq
    e = elig.cpu().numpy()
    return [e] * nq if e.ndim == 1 else list(e)


def _ref_sum(q, idx, hits, w, k, elig=None, id_offset=0):
    nq, nd = q.shape[0], idx.nd
    F = (_exact(q, idx) + w * _dense_matrix(hits, nq, nd)).cpu().numpy()  # torch fp32: fl(w v), then fl(s + .)
    s, i = np.full((nq, k), -np.inf, np.float32), np.full((nq, k), -1, np.int64)
    for r, e in enumerate(_elig_rows(elig, nq, nd)):
        o = order(F[r], e)[:k]
        s[r, :len(o)], i[r, :len(o)] = F[r, o], o + id_offset
    return torch.from_numpy(s).cuda(), torch.from_numpy(i).cuda()


def _ref_groups(q, idx, hits, w, k, groups, elig=None):
    nq, nd = q.shape[0], idx.nd
    F = (_exact(q, idx) + w * _dense_matrix(hits, nq, nd)).cpu().numpy()
    g_np = groups.cpu().numpy()
    out = (np.full((nq, k), -np.inf, np.float32), np.full((nq, k), -1, np.int64), np.full((nq, k), -1, np.int64))
    for r, e in enumerate(_elig_rows(elig, nq, nd)):
        o = order(F[r], e)
        _, first = np.unique(g_np[o], return_index=True)  # scatter-max: each document's first page in that order
        best = o[np.sort(first)][:k]
        out[0][r, :len(best)], out[1][r, :len(best)], out[2][r, :len(best)] = F[r, best], best, g_np[best]
    return tuple(torch.from_numpy(x).cuda() for x in out)


def _hits_rows(hits, nq):
    off, ids, vals = (t.cpu().numpy() for t in hits)
    return [dict(zip(ids[off[r]:off[r + 1]].tolist(), vals[off[r]:off[r + 1]].tolist())) for r in range(nq)]


def _ref_rrf(q, idx, hits, k, window, c=60, elig=None):
    nq = q.shape[0]
    S = _exact(q, idx).cpu().numpy()
    s, i = np.full((nq, k), -np.inf, np.float32), np.full((nq, k), -1, np.int64)
    for r, (h, e) in enumerate(zip(_hits_rows(hits, nq), _elig_rows(elig, nq, idx.nd))):
        rs_, ri_ = rrf_full(S[r], h, k, window, c, e)
        s[r, :len(ri_)], i[r, :len(ri_)] = rs_, ri_
    return torch.from_numpy(s).cuda(), torch.from_numpy(i).cuda()


def _same(got, want, what):
    for j, (a, b) in enumerate(zip(got, want)):
        assert a.shape == b.shape, (what, j, a.shape, b.shape)
        x = a.view(torch.int32) if a.dtype == torch.float32 else a
        y = b.view(torch.int32) if b.dtype == torch.float32 else b
        assert torch.equal(x, y), (what, j, int((x != y).sum()))


def _scope_hits(hits, elig):
    """The hits inside each row's scope (what the library keeps), for the references."""
    if elig is None:
        return hits
    off, ids, vals = hits
    nq = off.shape[0] - 1
    row = torch.repeat_interleave(torch.arange(nq, device=ids.device), off[1:] - off[:-1])
    keep = elig[ids.long()] if elig.dim() == 1 else elig[row, ids.long()]
    counts = torch.bincount(row[keep], minlength=nq)
    new_off = torch.zeros(nq + 1, dtype=torch.int64, device=ids.device)
    new_off[1:] = torch.cumsum(counts, 0)
    return new_off, ids[keep], vals[keep]


@pytest.fixture(scope="module")
def corpus():
    rs = np.random.RandomState(0)
    nd, d = 70_000, 256
    D = _unit(rs, nd, d)
    Q = _unit(rs, 64, d)
    return R.build_index(D), torch.from_numpy(Q).cuda(), rs


ROUTES = ["scan", "filter", "mask", "per_query_mask", "lists", "deep"]


def _route(route, idx, q, rs):
    """(queries, k, scope kwargs, eligibility bool [nd] / [nq, nd] or None, expected stats path)."""
    nd, nq = idx.nd, q.shape[0]
    if route == "scan":
        return q[:1], 10, {}, None, "exact"
    if route == "filter":
        return q, 10, {}, None, "filter+rescore"
    if route == "mask":
        m = torch.from_numpy(rs.rand(nd) < 0.6).cuda()
        return q, 10, dict(doc_mask=m), m, "filter+rescore"
    if route == "per_query_mask":
        m = torch.from_numpy(rs.rand(nq, nd) < 0.5).cuda()
        return q, 10, dict(doc_mask=m), m, "filter+rescore"
    if route == "lists":
        lens = rs.randint(5, 3000, nq)
        ids = np.concatenate([rs.choice(nd, n, replace=False) for n in lens])
        off = torch.tensor(np.concatenate([[0], np.cumsum(lens)]), dtype=torch.int64).cuda()
        ids_t = torch.from_numpy(ids).cuda()
        m = torch.zeros((nq, nd), dtype=torch.bool, device="cuda")
        m[torch.repeat_interleave(torch.arange(nq, device="cuda"), off[1:] - off[:-1]), ids_t] = True
        return q, 10, dict(doc_lists=(off, ids_t)), m, "lists"
    return q, 400, {}, None, "deep"


@pytest.mark.parametrize("route", ROUTES)
def test_weighted_sum_equals_the_full_matrix_on_every_route(corpus, route):
    idx, q0, rs = corpus
    q, k, scope, elig, path = _route(route, idx, q0, rs)
    hits = _hits(rs, _exact(q, idx), 60)
    for w, id_offset in ((1.0, 0), (0.25, 1000)):
        stats = {}
        got = R.score_topk_hybrid(q, idx, k, hits, weight=w, id_offset=id_offset, stats=stats, **scope)
        want = _ref_sum(q, idx, _scope_hits(hits, elig), w, k, elig, id_offset)
        _same(got, want, (route, w))
        assert stats["path"] == path and stats["candidates"].shape == (q.shape[0],)
    # weight 0 and no hits: score_topk, bit for bit
    empty = (torch.zeros(q.shape[0] + 1, dtype=torch.int64, device="cuda"), torch.zeros(0, dtype=torch.int32, device="cuda"),
             torch.zeros(0, dtype=torch.float32, device="cuda"))
    dense = R.score_topk(q, idx, k, **scope)
    _same(R.score_topk_hybrid(q, idx, k, hits, weight=0.0, **scope), dense, (route, "w=0"))
    _same(R.score_topk_hybrid(q, idx, k, empty, **scope), dense, (route, "empty"))


@pytest.mark.parametrize("window", [10, 100, 1000])
def test_rrf_equals_the_full_matrix(corpus, window):
    idx, q, rs = corpus
    hits = _hits(rs, _exact(q, idx), 80)
    got = R.score_topk_hybrid(q, idx, 10, hits, fusion="rrf", window=window)
    _same(got, _ref_rrf(q, idx, hits, 10, window), ("rrf", window))
    m = torch.from_numpy(rs.rand(q.shape[0], idx.nd) < 0.5).cuda()
    got = R.score_topk_hybrid(q, idx, 10, hits, fusion="rrf", window=window, rrf_c=1, doc_mask=m)
    _same(got, _ref_rrf(q, idx, _scope_hits(hits, m), 10, window, 1, m), ("rrf masked", window))


@pytest.mark.parametrize("pages", [1, 8, 64])
def test_documents_equal_a_scatter_max_of_the_full_matrix(corpus, pages):
    idx, q, rs = corpus
    nd = idx.nd
    groups = torch.from_numpy(rs.permutation(nd) // pages).to(torch.int32).cuda()  # documents of scattered pages
    hits = _hits(rs, _exact(q, idx), 60)
    for w in (1.0, 0.3):
        got = R.score_topk_groups_hybrid(q, idx, 10, groups, hits, weight=w)
        _same(got, _ref_groups(q, idx, hits, w, 10, groups), ("documents", pages, w))
    m = torch.from_numpy(rs.rand(q.shape[0], nd) < 0.5).cuda()
    got = R.score_topk_groups_hybrid(q, idx, 10, groups, hits, doc_mask=m)
    _same(got, _ref_groups(q, idx, _scope_hits(hits, m), 1.0, 10, groups, m), ("documents masked", pages))
    dense = R.score_topk_groups(q, idx, 10, groups)
    _same(R.score_topk_groups_hybrid(q, idx, 10, groups, hits, weight=0.0), dense, ("documents w=0", pages))


def test_documents_longer_than_a_piece(corpus):
    idx, q, rs = corpus
    groups = torch.from_numpy(np.minimum(np.arange(idx.nd) // 1000, 40)).to(torch.int32).cuda()  # up to 30 000 pages
    hits = _hits(rs, _exact(q[:8], idx), 40)
    got = R.score_topk_groups_hybrid(q[:8], idx, 5, groups, hits, weight=0.5)
    _same(got, _ref_groups(q[:8], idx, hits, 0.5, 5, groups), "long documents")


def test_rows_equal_each_query_alone(corpus):
    idx, q, rs = corpus
    q = q[:12]
    hits = _hits(rs, _exact(q, idx), 50)
    groups = torch.from_numpy(np.arange(idx.nd) // 8).to(torch.int32).cuda()
    batch = (R.score_topk_hybrid(q, idx, 10, hits), R.score_topk_hybrid(q, idx, 10, hits, fusion="rrf", window=50),
             R.score_topk_groups_hybrid(q, idx, 10, groups, hits))
    off, ids, vals = hits
    for r in range(q.shape[0]):
        a, b = int(off[r]), int(off[r + 1])
        one = (torch.tensor([0, b - a], dtype=torch.int64, device="cuda"), ids[a:b], vals[a:b])
        alone = (R.score_topk_hybrid(q[r:r + 1], idx, 10, one),
                 R.score_topk_hybrid(q[r:r + 1], idx, 10, one, fusion="rrf", window=50),
                 R.score_topk_groups_hybrid(q[r:r + 1], idx, 10, groups, one))
        for x, y in zip(batch, alone):
            _same([t[r:r + 1] for t in x], y, ("row", r))


def test_hit_lists_longer_than_any_shared_memory_table(corpus):
    idx, q, rs = corpus
    q = q[:6]
    hits = _hits(rs, _exact(q, idx), 30, long_row=(2, 20_000))
    assert int((hits[0][1:] - hits[0][:-1]).max()) >= 20_000
    _same(R.score_topk_hybrid(q, idx, 10, hits, weight=0.5), _ref_sum(q, idx, hits, 0.5, 10), "long sum")
    _same(R.score_topk_hybrid(q, idx, 10, hits, fusion="rrf", window=100), _ref_rrf(q, idx, hits, 10, 100), "long rrf")
    groups = torch.from_numpy(np.arange(idx.nd) // 8).to(torch.int32).cuda()
    _same(R.score_topk_groups_hybrid(q, idx, 10, groups, hits, weight=0.5), _ref_groups(q, idx, hits, 0.5, 10, groups),
          "long documents")


def test_stages_are_reported(corpus):
    idx, q, rs = corpus
    hits = _hits(rs, _exact(q, idx), 20)
    stats = {"stages": {}}
    R.score_topk_hybrid(q, idx, 10, hits, stats=stats)
    torch.cuda.synchronize()
    st = R.resolve_stages(stats)
    assert {"dense", "lists", "fuse", "select"} <= set(st)
    lens = (hits[0][1:] - hits[0][:-1]).cpu()
    assert (stats["candidates"].cpu() <= 10 + lens).all() and (stats["candidates"].cpu() >= lens).all()


def test_entry_points_refuse_operands_before_launch():
    lib = L.lib()
    t = {n: torch.zeros(64, dtype=torch.int64, device="cuda") for n in ("ds", "di", "off", "ids", "vals", "hd", "os", "oi", "st")}
    p = {n: v.data_ptr() for n, v in t.items()}

    def fuse(**kw):
        a = dict(ds=p["ds"], di=p["di"], rows=2, kd=4, off=p["off"], ids=p["ids"], vals=p["vals"], hd=p["hd"], pitch=4, mode=0,
                 w=1.0, c=60, width=8, os=p["os"], oi=p["oi"], st=p["st"])
        a.update(kw)
        return lib.vr_fuse_rows(*a.values(), None), lib.vr_last_error().decode()

    for kw, word in ((dict(kd=0), "kd"), (dict(mode=3), "mode"), (dict(w=-1.0), "weight"), (dict(w=float("nan")), "weight"),
                     (dict(width=3), "width"), (dict(di=p["di"] + 4), "dense_ids"), (dict(oi=p["oi"] + 4), "out_ids"),
                     (dict(hd=None), "hit_dense"), (dict(mode=1, c=-1), "rrf_c")):
        rc, msg = fuse(**kw)
        assert rc == 2 and word in msg, (kw, rc, msg)
    rc, msg = lib.vr_group_pages_fused(p["ds"], 1, p["hd"], 4, 8, p["di"], 1, p["off"], p["ids"], 1, None, p["off"] + 4,
                                       p["ids"], p["vals"], 1.0, 4, 1, 0, p["os"], p["oi"], None), lib.vr_last_error().decode()
    assert rc == 2 and "hit_offsets" in msg, msg
    rc, msg = lib.vr_group_pages_fused(p["ds"], 1, p["hd"], 4, 8, p["di"], 1, p["off"], p["ids"], 1, None, p["off"],
                                       p["ids"], p["vals"], -2.0, 4, 1, 0, p["os"], p["oi"], None), lib.vr_last_error().decode()
    assert rc == 2 and "weight" in msg, msg
    torch.cuda.synchronize()


def test_knowledge_base_forms_equal_the_index_forms(tmp_path):
    rs = np.random.RandomState(5)
    n, d = 3000, 128
    names = [f"doc{i // 6}.pdf_{i % 6}.png" for i in range(n)]
    save_knowledge_base(str(tmp_path), _unit(rs, n, d), names)
    kb = KnowledgeBase(str(tmp_path))
    kb.remove(names[10:400])
    extra = [f"new{i // 4}.pdf_{i % 4}.png" for i in range(200)]
    kb.add(_unit(rs, 200, d), extra)
    q = torch.from_numpy(_unit(rs, 5, d)).cuda()
    live = [f for f in names + extra if f in kb._row]
    hits = [{f: float(v) for f, v in zip(rs.choice(names + extra, 40, replace=False), rs.rand(40) * 2)} for _ in range(5)]
    hits[0]["no such page.png"] = 1.0
    # the index forms with the same hits, live pages only
    off, ids, vals = [0], [], []
    for h in hits:
        for f, v in h.items():
            if f in kb._row:
                ids.append(kb._row[f])
                vals.append(v)
        off.append(len(ids))
    ih = (torch.tensor(off, dtype=torch.int64, device="cuda"), torch.tensor(ids, dtype=torch.int32, device="cuda"),
          torch.tensor(vals, dtype=torch.float32, device="cuda"))
    _same(kb.search_hybrid(q, 10, hits, weight=0.5),
          R.score_topk_hybrid(q, kb.index, 10, ih, weight=0.5, doc_mask=kb._live), "kb sum")
    _same(kb.search_hybrid(q, 10, hits, fusion="rrf", window=30),
          R.score_topk_hybrid(q, kb.index, 10, ih, fusion="rrf", window=30, doc_mask=kb._live), "kb rrf")
    s, p, names_out = kb.search_documents_hybrid(q, 10, hits, weight=0.5)
    ws, wp, wg = R.score_topk_groups_hybrid(q, kb.index, 10, kb._doc_groups, ih, weight=0.5, doc_mask=kb._live)
    _same((s, p), (ws, wp), "kb documents")
    assert names_out == [[kb.documents[g] for g in row if g >= 0] for row in wg.tolist()]
    # a scope: the hits outside it are dropped, as on an index of only the scope's pages
    within = live[:300]
    scope = torch.zeros(kb.index.nd, dtype=torch.bool, device="cuda")
    scope[torch.tensor([kb._row[f] for f in within], device="cuda")] = True
    _same(kb.search_hybrid(q, 10, hits, within=within),
          _ref_sum(q, kb.index, _scope_hits(ih, scope), 1.0, 10, scope), "kb within")
    each = [within, None, within[:50], None, live[100:900]]
    elig = kb._live[None, :].repeat(5, 1)
    for r, sc in enumerate(each):
        if sc is not None:
            elig[r] = False
            elig[r, torch.tensor([kb._row[f] for f in sc], device="cuda")] = True
    _same(kb.search_hybrid(q, 10, hits, within_each=each), _ref_sum(q, kb.index, _scope_hits(ih, elig), 1.0, 10, elig),
          "kb within_each")
    _same(kb.search_hybrid(q, 10, hits, fusion="rrf", window=20, within_each=each),
          _ref_rrf(q, kb.index, _scope_hits(ih, elig), 10, 20, 60, elig), "kb within_each rrf")
    groups = kb._doc_groups
    _same(kb.search_documents_hybrid(q, 10, hits, within_each=each)[:2],
          _ref_groups(q, kb.index, _scope_hits(ih, elig), 1.0, 10, groups, elig)[:2], "kb documents within_each")


def test_chunked_passes_and_document_lists(corpus, monkeypatch):
    """Query rows in several passes (small FUSE_BUDGET / GROUP_STAGE_BUDGET), and documents scoped by candidate lists."""
    idx, q, rs = corpus
    q = q[:20]
    hits = _hits(rs, _exact(q, idx), 60)
    groups = torch.from_numpy(np.arange(idx.nd) // 8).to(torch.int32).cuda()
    whole = (R.score_topk_hybrid(q, idx, 10, hits, weight=0.5), R.score_topk_hybrid(q, idx, 10, hits, fusion="rrf"),
             R.score_topk_groups_hybrid(q, idx, 10, groups, hits, weight=0.5))
    monkeypatch.setattr(R, "FUSE_BUDGET", 300)        # a few rows per pass
    monkeypatch.setattr(R, "GROUP_STAGE_BUDGET", 200)
    parts = (R.score_topk_hybrid(q, idx, 10, hits, weight=0.5), R.score_topk_hybrid(q, idx, 10, hits, fusion="rrf"),
             R.score_topk_groups_hybrid(q, idx, 10, groups, hits, weight=0.5))
    for a, b in zip(parts, whole):
        _same(a, b, "chunked")
    _same(whole[0], _ref_sum(q, idx, hits, 0.5, 10), "chunked sum")
    _same(whole[2], _ref_groups(q, idx, hits, 0.5, 10, groups), "chunked documents")
    monkeypatch.undo()
    lens = rs.randint(50, 3000, q.shape[0])
    lids = np.concatenate([rs.choice(idx.nd, n, replace=False) for n in lens])
    off = torch.tensor(np.concatenate([[0], np.cumsum(lens)]), dtype=torch.int64).cuda()
    lids_t = torch.from_numpy(lids).cuda()
    m = torch.zeros((q.shape[0], idx.nd), dtype=torch.bool, device="cuda")
    m[torch.repeat_interleave(torch.arange(q.shape[0], device="cuda"), off[1:] - off[:-1]), lids_t] = True
    got = R.score_topk_groups_hybrid(q, idx, 10, groups, hits, weight=0.5, doc_lists=(off, lids_t))
    _same(got, _ref_groups(q, idx, _scope_hits(hits, m), 0.5, 10, groups, m), "documents over lists")
