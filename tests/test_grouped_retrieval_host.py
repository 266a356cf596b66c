"""Document-level retrieval without a GPU: the C ABI's refusals of bad group tables (before any CUDA call), a numpy
emulation of the group-distinct filter lists + grouped rescoring + proof, two mutants of the proof that return a wrong
answer, the knowledge base's filename-to-document rule, and a model of the per-rank merge.

The grouped proof: every page a list dropped is <= that list's tail or <= its own group's entry in that list. The
rescoring fully rescores the distinct groups of the kept candidates (within a page budget) and certifies the top-k groups
when B + eps < k-th group score, B = max(list tails, pruned heads, approximate entries of kept groups not rescored)."""
import functools
import os

import numpy as np
import pytest

import __graft_entry__ as G
from tests import score_fixtures as SF
from visrag_b200 import _lib as L
from visrag_b200.knowledge_base import document_of

@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(L.LIB_PATH):
        G.build()
    return L.lib()


def test_grouped_entry_points_refuse_bad_arguments_before_any_cuda_call(lib):
    """Pointers here are never dereferenced: every call must be refused by argument checks on the host."""
    fake = 1 << 20
    r = lib.vr_score_ranges(300, 5000)
    rc = lib.vr_score_filter_groups(fake, 300, fake, 5000, 256, r, fake, fake, None, None, None)
    assert rc != 0 and b"doc_groups" in lib.vr_last_error()
    rc = lib.vr_score_filter_groups(fake, 300, fake, 5000, 256, r, fake, fake, fake + 2, None, None)
    assert rc != 0 and b"aligned" in lib.vr_last_error()
    rc = lib.vr_score_filter_groups(fake, 300, fake, 5000, 256, r, fake, fake, fake, fake + 1, None)
    assert rc != 0 and b"doc_mask" in lib.vr_last_error()
    rc = lib.vr_score_filter_groups(fake, 300, fake, 1 << 31, 256, r, fake, fake, fake, None, None)
    assert rc != 0 and b"int32" in lib.vr_last_error()

    def rescore(groups=fake, offsets=fake, pages=fake, G=100, nd=5000, mask=None):
        return lib.vr_score_rescore_groups(fake, 300, fake, nd, 256, r, fake, fake, groups, offsets, pages, G, mask, fake, 10,
                                           0, fake, fake, fake, fake, None)

    for kw, msg in (({"groups": None}, b"doc_groups"), ({"offsets": None}, b"group_offsets"),
                    ({"pages": fake + 2}, b"aligned"), ({"G": 0}, b"G=0"), ({"nd": 1 << 31}, b"int32"),
                    ({"mask": fake + 3}, b"doc_mask")):
        assert rescore(**kw) != 0 and msg in lib.vr_last_error(), kw

    need = lib.vr_group_topk_ws_bytes(4, 1000, 10, 0)
    assert need >= 4 * 1000 * 12
    assert lib.vr_group_topk_ws_bytes(1, 1000000, 10, 100) >= 1000000 * 12 + 100 * 10 * 12

    def topk(ws_bytes=need, groups=fake, G=1000, nd=5000, ws=fake):
        return lib.vr_group_topk_rows(fake, 4, nd, groups, G, None, 10, 0, 0, ws, ws_bytes, fake, fake, fake, None)

    for kw, msg in (({"ws_bytes": need - 1}, b"workspace"), ({"ws": fake + 8}, b"workspace"),
                    ({"groups": None}, b"doc_groups"), ({"G": -1}, b"G=-1"), ({"nd": 1 << 31}, b"int32")):
        assert topk(**kw) != 0 and msg in lib.vr_last_error(), kw
    rc = lib.vr_merge_group_topk(fake, fake, fake, 10, 513, 10, fake, fake, fake, None)
    assert rc != 0 and b"cols" in lib.vr_last_error()


def test_group_table_cache_lets_go_of_freed_tensors():
    """The CSR cache holds its own copy of the groups: an entry leaves with the caller's tensor (int32, int64 or a slice
    of a longer tensor), is reused while the tensor lives, and is rebuilt after an in-place change."""
    import gc

    import torch

    from visrag_b200 import retriever as R

    nd = 1000
    idx = R.CorpusIndex(torch.zeros(nd, 8), torch.zeros(nd, 8, dtype=torch.float16), torch.ones(1))
    base = len(R._GROUP_TABLES)
    longer = torch.arange(3 * nd, dtype=torch.int32) // 7
    for make in (lambda: torch.arange(nd, dtype=torch.int32) // 3, lambda: torch.arange(nd) // 3,
                 lambda: longer[nd:2 * nd], lambda: longer.to(torch.int64)[:nd]):
        tables = []
        for _ in range(5):
            t = make()
            tables.append(R._group_table(t, idx))
            assert R._group_table(t, idx) is tables[-1]                   # reused while the tensor lives
            assert tables[-1].groups.data_ptr() != t.data_ptr()          # its own copy
            del t
        gc.collect()
        assert len(R._GROUP_TABLES) == base, make
    t = torch.arange(nd) // 3
    a = R._group_table(t, idx)
    t[0] = 400
    b = R._group_table(t, idx)
    assert b is not a and b.G == 401 and int(b.groups[0]) == 400
    del t, a, b
    gc.collect()
    assert len(R._GROUP_TABLES) == base


def test_filename_to_document_rule():
    assert document_of("a_b.pdf_12.png") == "a_b.pdf"
    assert document_of("report.pdf_0.png") == "report.pdf"
    assert document_of("cat.jpeg") == "cat.jpeg"
    for own in ("x_.png", "x_1a.png", "x_1.jpg", "nounderscore.png", "a_b_c"):
        assert document_of(own) == own


# ------------------------------------------------------------------------------------------------------ emulation


def _same(a, b):
    return all(np.array_equal(x, y) for x, y in zip(a, b))


@functools.lru_cache(maxsize=None)
def _fixtures():
    return tuple(SF.fixtures())


@pytest.mark.parametrize("name", SF.FIXTURES)
def test_grouped_emulation_returns_the_grouped_fp32_answer_on_the_proof_fixtures(name):
    fx = {f.name: f for f in _fixtures()}[name]
    nd = fx.D.shape[0]
    Q = fx.Q[:1]
    p = SF.plan(fx.Q.shape[0], nd)
    exact, approx = SF.exact_scores(Q, fx.D), SF.approx_scores(Q, fx.D)
    for what, groups in {"one page each": np.arange(nd), "contiguous 8": np.arange(nd) // 8,
                         "true doc with its decoys": SF._true_with_decoys(fx)}.items():
        cs, ci = SF.grouped_filter_lists(approx, groups, p)
        for r in range(p["lists"] - 1):
            g = groups[ci[0, r][ci[0, r] >= 0]]
            assert len(g) == len(set(g.tolist())), (what, r)
        out = SF.grouped_rescore(cs, ci, exact, groups, SF.row_norms(Q), SF.row_norms(fx.D).max(), fx.k, Q.shape[1])
        ref = SF.grouped_reference(exact, groups, fx.k)
        if out[3][0]:
            out = ref
        assert _same(out[:3], ref), what


def test_group_score_from_the_kept_entry_returns_a_wrong_answer():
    """The true document's exact score is the highest, but fp16 rounding puts its approximate score below its group's
    decoys: the group-distinct list keeps a decoy as the group's entry and drops the true document. Full rescoring of the
    group finds it; taking the group's score from its kept entry does not."""
    fx = {f.name: f for f in _fixtures()}["fp16 rounds down 0.49 ulp"]
    Q, D = fx.Q[:1], fx.D
    groups = SF._true_with_decoys(fx)
    p = SF.plan(fx.Q.shape[0], D.shape[0])
    exact, approx = SF.exact_scores(Q, D), SF.approx_scores(Q, D)
    cs, ci = SF.grouped_filter_lists(approx, groups, p)
    assert fx.true_doc not in ci[0]                                   # dropped: <= its group's entry
    ref = SF.grouped_reference(exact, groups, 1)
    assert ref[1][0, 0] == fx.true_doc
    args = (cs, ci, exact, groups, SF.row_norms(Q), SF.row_norms(D).max(), 1, Q.shape[1])
    good = SF.grouped_rescore(*args)
    assert not good[3][0] and _same(good[:3], ref)
    bad = SF.grouped_rescore(*args, mut="entry score")
    assert not bad[3][0] and bad[1][0, 0] != fx.true_doc and bad[0][0, 0] < ref[0][0, 0]


def test_bound_without_the_unrescored_groups_returns_a_wrong_answer():
    Q, D, groups, T, Y = SF._budget_fixture()
    exact, approx = SF.exact_scores(Q, D)[0], SF.approx_scores(Q, D)[0]
    assert exact[T] > exact[Y] and approx[Y] > approx[T] and np.argsort(-approx)[:2].tolist() == [Y, T]
    assert (groups == groups[T]).sum() > SF.BUDGET
    got, flags, info = SF.emulate_grouped(Q, D, groups, 1)
    assert flags.all() and _same(got, info["ref"]) and got[1][0, 0] == T     # T's group is not rescored: flagged
    bad, flags, info = SF.emulate_grouped(Q, D, groups, 1, mut="B without unrescored groups")
    assert not flags.any() and bad[1][0, 0] == Y and not _same(bad, info["ref"])


def _clustered_multi_wave():
    """600 queries over 4096 pages at 5 CTA pairs (8 doc ranges, 5 waves): documents of 8 contiguous pages, each a centre
    plus small noise; queries near document centres."""
    rs = np.random.RandomState(22)
    n_docs, pages, dim, nq = 512, 8, 8, 600
    c = rs.randn(n_docs, dim).astype(np.float32)
    c /= np.linalg.norm(c, axis=1, keepdims=True)
    D = (np.repeat(c, pages, axis=0) + 0.01 * rs.randn(n_docs * pages, dim)).astype(np.float32)
    Q = (c[rs.randint(0, n_docs, nq)] + 0.2 * rs.randn(nq, dim)).astype(np.float32)
    return Q, D, np.arange(n_docs * pages) // pages, 5


def test_grouped_emulation_on_a_clustered_multi_wave_fixture():
    Q, D, groups, pairs = _clustered_multi_wave()
    p = SF.plan(Q.shape[0], D.shape[0], pairs)
    assert p["items"] > p["pairs"] and p["R"] > 1, p
    for k in (1, 10):
        got, flags_g, info = SF.emulate_grouped(Q, D, groups, k, pairs)
        assert _same(got, info["ref"]), k
        got, flags_p, info = SF.emulate_grouped(Q, D, groups, k, pairs, page_lists=True)
        assert _same(got, info["ref"]), k
        if k == 10:   # page lists hold a few documents each: their tails sit above the 10th document
            assert flags_g.sum() == 0 and flags_p.sum() > len(Q) // 2, (flags_g.sum(), flags_p.sum())


# ------------------------------------------------------------------------------------------------------ sharding


def merge_groups(parts, k):
    """vr_merge_group_topk: the first k distinct groups of the concatenated lists in (score desc, page asc) order."""
    s = np.concatenate([x[0] for x in parts], 1)
    p = np.concatenate([x[1] for x in parts], 1)
    g = np.concatenate([x[2] for x in parts], 1)
    out = [np.full((len(s), k), v, t) for v, t in ((-np.inf, np.float32), (-1, np.int64), (-1, np.int64))]
    for r in range(len(s)):
        live = np.nonzero(p[r] >= 0)[0]
        order = live[np.lexsort((p[r, live], -s[r, live]))]
        seen, n = set(), 0
        for c in order:
            if g[r, c] in seen or n == k:
                continue
            seen.add(g[r, c])
            out[0][r, n], out[1][r, n], out[2][r, n] = s[r, c], p[r, c], g[r, c]
            n += 1
    return tuple(out)


def test_per_rank_group_lists_merge_to_the_global_answer():
    """Documents of 7 pages over 3 ranks of 1000 pages: documents straddle the rank boundaries. Scores are rounded
    to a coarse grid, so equal scores (ties on the page id) are frequent."""
    rs = np.random.RandomState(23)
    nq, nd, world = 50, 3000, 3
    exact = (np.round(rs.randn(nq, nd) * 8) / 8).astype(np.float32)
    groups = np.arange(nd) // 7
    for k in (1, 5, 20):
        parts = []
        for rank in range(world):
            lo, hi = rank * nd // world, (rank + 1) * nd // world
            s, p, g = SF.grouped_reference(exact[:, lo:hi], groups[lo:hi], k)
            parts.append((s, np.where(p >= 0, p + lo, -1), g))
        assert _same(merge_groups(parts, k), SF.grouped_reference(exact, groups, k)), k
