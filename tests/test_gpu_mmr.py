"""Diverse retrieval on the GPU: vr_mmr_select against the numpy model of tests/test_mmr_host.py, bit for bit. The model is
fed with the GPU's own candidates (score_topk with force_exact) and the Gram of the candidate rows from vr_score_exact,
so every score and similarity it compares has the kernel's bits; the picks and the output rows must then be identical."""
import numpy as np
import pytest
import torch

from tests.test_mmr_host import mmr_model, rows_of
from visrag_b200 import _lib as L
from visrag_b200 import knowledge_base as KB
from visrag_b200 import retriever as R

pytestmark = pytest.mark.gpu


def _unit(n, dim, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn((n, dim), generator=g)
    return x / x.norm(dim=1, keepdim=True)


def _queries(nq, dim, seed, docs=None):
    q = _unit(nq, dim, seed)
    if docs is not None:  # near some docs, so that their neighbours (and duplicates) are candidates
        g = torch.Generator().manual_seed(seed + 1)
        q = docs[torch.randint(0, docs.shape[0], (nq,), generator=g)].cpu() + 0.3 * q
        q /= q.norm(dim=1, keepdim=True)
    return q.cuda()


def _clusters(n_clusters, per, dim, seed, noise=0.01):
    """Planted near-duplicate clusters: `per` noisy copies of each of n_clusters random unit centers."""
    c = _unit(n_clusters, dim, seed)
    g = torch.Generator().manual_seed(seed + 7)
    d = c.repeat_interleave(per, 0) + noise * torch.randn((n_clusters * per, dim), generator=g) / dim ** 0.5
    d /= d.norm(dim=1, keepdim=True)
    return c, d, torch.arange(n_clusters).repeat_interleave(per)


def gram(index, ids):
    """vr_score_exact of the candidate rows against each other: sim(c_a, c_b) with the kernel's bits."""
    rows = index.emb.index_select(0, ids).contiguous()
    n = rows.shape[0]
    g = torch.empty((n, n), dtype=torch.float32, device=rows.device)
    L.check(L.lib().vr_score_exact(rows.data_ptr(), n, rows.data_ptr(), n, rows.shape[1], g.data_ptr(), L.stream_ptr()))
    return g.cpu().numpy()


def model(index, s, i, k, lam, id_offset=0):
    """The model's output rows for candidates (s, i) [nq, F] and lam (float or [nq])."""
    s_np, i_np = s.cpu().numpy(), i.cpu().numpy()
    lam = np.broadcast_to(np.asarray(lam.cpu().numpy() if isinstance(lam, torch.Tensor) else lam, np.float32), (len(s_np),))
    out_s = np.empty((len(s_np), k), np.float32)
    out_i = np.empty((len(s_np), k), np.int64)
    for r in range(len(s_np)):
        bad = np.nonzero(i_np[r] < 0)[0]
        n = int(bad[0]) if bad.size else i_np.shape[1]
        g = gram(index, i[r, :n]) if n else np.zeros((0, 0), np.float32)
        picks = mmr_model(s_np[r], i_np[r], g, lam[r], k)
        out_s[r], out_i[r] = rows_of(picks, s_np[r], i_np[r], k, id_offset)
    return out_s, out_i


def assert_bits(got, want):
    gs, gi = (t.cpu().numpy() for t in got)
    ws, wi = want
    assert np.array_equal(gi, wi), np.argwhere(gi != wi)[:5]
    assert np.array_equal(gs.view(np.uint32), ws.view(np.uint32))


_INDEX = {}


def _index(nd, dim, seed):
    key = (nd, dim, seed)
    if key not in _INDEX:
        d = _unit(nd, dim, seed)
        d[7::97] = d[3]  # exact duplicate rows: equal scores and equal similarities, decided by position
        _INDEX[key] = R.build_index(d.cuda())
    return _INDEX[key]


# ------------------------------------------------------------------------------------------------ the kernel's bits
@pytest.mark.parametrize("dim", [2304, 64])
@pytest.mark.parametrize("fetch", [8, 20, 40, 128])
def test_rows_match_the_model(dim, fetch):
    """Every cluster size (F = 8, 20, 40, 128 at dim 2304 take 1, 2, 4, 8 CTAs), every lambda and a per-query lambda."""
    index = _index(20_000, dim, 1)
    q = _queries(24, dim, 2, index.emb[:100])
    s, i = R.score_topk(q, index, fetch, force_exact=True)
    k = min(10, fetch)
    lam_q = torch.linspace(0, 1, 24, device="cuda")
    for lam in (0.0, 0.3, 0.5, 1.0, lam_q):
        got = R.mmr_select(index, s, i, k, lam, id_offset=1000)
        assert_bits(got, model(index, s, i, k, lam, id_offset=1000))
        if not isinstance(lam, torch.Tensor) and lam == 1.0:
            assert torch.equal(got[0], s[:, :k]) and torch.equal(got[1], i[:, :k] + 1000)
    # every candidate picked: k = F
    got = R.mmr_select(index, s[:4], i[:4], fetch, 0.5)
    assert_bits(got, model(index, s[:4], i[:4], fetch, 0.5))
    assert torch.equal(torch.sort(got[1], 1).values, torch.sort(i[:4], 1).values)


def test_score_mmr_is_score_topk_then_mmr_select():
    index = _index(20_000, 2304, 1)
    q = _queries(40, 2304, 3, index.emb[:200])
    stats = {"stages": {}}
    got = R.score_mmr(q, index, 5, 0.5, fetch_k=40, id_offset=7, stats=stats)
    torch.cuda.synchronize()
    stages = R.resolve_stages(stats)
    assert {"candidates", "select"} <= set(stages) and stats["fetch_k"] == 40 and stats["path"] == "exact"
    s, i = R.score_topk(q, index, 40, force_exact=True)
    assert_bits(got, model(index, s, i, 5, 0.5, id_offset=7))
    st = {}
    R.score_mmr(q, index, 10, stats=st)
    assert st["fetch_k"] == 40


def test_many_waves_and_batch_invariance():
    index = _index(20_000, 2304, 1)
    q = _queries(2000, 2304, 4, index.emb[:3000])
    s, i = R.score_topk(q, index, 40, force_exact=True)
    lam = torch.rand(2000, generator=torch.Generator().manual_seed(5)).cuda()
    got = R.mmr_select(index, s, i, 10, lam)
    sel = torch.arange(0, 2000, 7)
    assert_bits(tuple(t[sel] for t in got), model(index, s[sel], i[sel], 10, lam[sel]))
    for r in (0, 1, 999, 1999):
        alone = R.mmr_select(index, s[r:r + 1], i[r:r + 1], 10, lam[r:r + 1])
        assert torch.equal(alone[0], got[0][r:r + 1]) and torch.equal(alone[1], got[1][r:r + 1])
    for r in (0, 5):  # alone through score_mmr: the whole pipeline is batch invariant
        a = R.score_mmr(q[r:r + 1], index, 10, lam[r:r + 1], fetch_k=40)
        b = R.score_mmr(q, index, 10, lam, fetch_k=40)
        assert torch.equal(a[0], b[0][r:r + 1]) and torch.equal(a[1], b[1][r:r + 1])


def test_exact_duplicates_tie_to_the_earlier_candidate():
    index = _index(20_000, 2304, 1)
    q = _queries(8, 2304, 6, index.emb[3:4].repeat(8, 1))  # near row 3, whose copies sit at 7, 104, 201, ...
    s, i = R.score_topk(q, index, 20, force_exact=True)
    assert (i == 7).any(1).all() and (i == 104).any(1).all()
    for lam in (0.0, 0.5, 1.0):
        assert_bits(R.mmr_select(index, s, i, 8, lam), model(index, s, i, 8, lam))


def test_scopes_masks_and_lists():
    index = _index(20_000, 2304, 1)
    nd = index.nd
    q = _queries(12, 2304, 8, index.emb[:500])
    m1 = torch.zeros(nd, dtype=torch.bool, device="cuda")
    m1[::3] = True
    ar = torch.arange(nd, device="cuda")
    m2 = torch.stack([(ar % 12 == r) if r % 4 else (ar < 3 + r) for r in range(12)])  # rows 0, 4, 8: 3-11 pages
    for kw in (dict(doc_mask=m1), dict(doc_mask=m2)):
        s, i = R.score_topk(q, index, 40, force_exact=True, **kw)
        got = R.score_mmr(q, index, 10, 0.3, fetch_k=40, **kw)
        assert_bits(got, model(index, s, i, 10, 0.3))
    # rows of fewer than k pages end in (-inf, -1)
    got = R.score_mmr(q, index, 10, 0.3, fetch_k=40, doc_mask=m2)
    assert (got[1][0, 3:] == -1).all() and (got[1][0, :3] >= 0).all()
    offsets = torch.tensor([0, 5, 5 + 300, 5 + 300 + 2], device="cuda")
    ids = torch.cat([torch.arange(100, 105), torch.arange(1000, 1300), torch.tensor([9, 4])]).cuda()
    list_of = torch.tensor([0, 1, 2] * 4, device="cuda")
    s, i = R.score_topk(q, index, 20, doc_lists=(offsets, ids), list_of=list_of)
    got = R.score_mmr(q, index, 8, 0.5, fetch_k=20, doc_lists=(offsets, ids), list_of=list_of)
    assert_bits(got, model(index, s, i, 8, 0.5))
    assert (got[1][2, 2:] == -1).all()


def test_nan_and_inf_rows():
    """Candidates from any source: a row with a NaN component and one with an inf component among them give NaN and
    inf relevance scores and similarities; the selection follows the definition through every one."""
    d = _unit(5000, 64, 9)
    d[10, 5] = float("nan")
    d[20, 7] = float("inf")
    index = R.build_index(d.cuda())
    q = _queries(6, 64, 10, index.emb[30:40])
    s, i = R.score_topk(q, index, 19, force_exact=True)
    i = torch.cat([i, torch.full((6, 2), 10, device="cuda")], 1)
    i[:, -1] = 20
    i[3, 5], i[4, 0] = 10, 20  # in the middle and first as well
    ex = torch.empty((6, index.nd), device="cuda")
    L.check(L.lib().vr_score_exact(q.data_ptr(), 6, index.emb.data_ptr(), index.nd, 64, ex.data_ptr(), L.stream_ptr()))
    s = torch.gather(ex, 1, i).contiguous()
    assert torch.isnan(s[:, -2]).all() and torch.isinf(s[:, -1]).all()
    for lam in (0.0, 0.5, 1.0):
        assert_bits(R.mmr_select(index, s, i, 12, lam), model(index, s, i, 12, lam))
    assert_bits(R.mmr_select(index, s, i, 21, 0.3), model(index, s, i, 21, 0.3))


def test_planted_clusters_are_covered_once_each():
    """Plain top-k returns several copies of one page; MMR at lambda 0.5 returns at most one page per cluster."""
    dim = 2304
    centers, d, cl = _clusters(3000, 6, dim, 11)
    index = R.build_index(d.cuda())
    w = torch.tensor([1.0, 0.95, 0.9, 0.85, 0.8, 0.75, 0.7, 0.65])
    g = torch.Generator().manual_seed(12)
    picks = torch.stack([torch.randperm(3000, generator=g)[:8] for _ in range(16)])
    q = (w[None, :, None] * centers[picks]).sum(1)
    q = (q / q.norm(dim=1, keepdim=True)).cuda()
    top = R.score_topk(q, index, 5)[1].cpu()
    assert all(len(set(cl[r].tolist())) < 5 for r in top)
    s, i = R.score_topk(q, index, 40, force_exact=True)
    for lam in (0.0, 0.3, 0.5, 1.0):
        got = R.score_mmr(q, index, 5, lam, fetch_k=40)
        assert_bits(got, model(index, s, i, 5, lam))
        if lam == 0.5:
            assert all(len(set(cl[r].tolist())) == 5 for r in got[1].cpu())


# ------------------------------------------------------------------------------------------------ knowledge base
def test_search_diverse_equals_mmr_select_on_search(tmp_path):
    dim = 256
    docs = _unit(12_000, dim, 13)
    docs[50:60] = docs[40]  # repeated pages
    names = [f"doc{j // 10}.pdf_{j % 10}.png" for j in range(12_000)]
    KB.save_knowledge_base(str(tmp_path), docs.numpy(), names)
    kb = KB.KnowledgeBase(str(tmp_path))
    q = _queries(30, dim, 14, docs[:100].cuda())
    kb.remove(names[:20] + names[45:52])
    lam = torch.linspace(0, 1, 30, device="cuda")

    def check(got, searched, k, lam):
        s, i = searched
        want = R.mmr_select(kb.index, s, i, k, lam)
        assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])
        assert_bits(got, model(kb.index, s, i, k, lam))

    check(kb.search_diverse(q, 5, 0.5), kb.search(q, 20), 5, 0.5)
    check(kb.search_diverse(q, 6, lam, fetch_k=30), kb.search(q, 30), 6, lam)
    within = [n for n in names[30:200] if n in kb._row]
    check(kb.search_diverse(q, 5, 0.5, within=within), kb.search(q, 20, within=within), 5, 0.5)
    # the live pages of 4-page scopes (some partly or wholly removed), and every live page for a third of the queries
    each = [[n for n in names[j * 10:j * 10 + 4] if n in kb._row] if j % 3 else None for j in range(30)]
    got = kb.search_diverse(q, 5, 0.3, within_each=each)
    check(got, kb.search(q, 20, within_each=each), 5, 0.3)
    assert not ((got[1] >= 0) & (got[1] < 20)).any() and not ((got[1] >= 45) & (got[1] < 52)).any()
    paths = kb.retrieve_diverse(q[0], 4, 0.5)
    assert paths == [str(tmp_path / names[j]) for j in kb.search_diverse(q[0:1], 4, 0.5)[1][0].tolist()]
    tiny = kb.search_diverse(q[:2], 5, 0.5, within=names[100:103])
    assert tiny[1].shape == (2, 3)
