"""Every retrieval operation against the independent reference of tests/dot_reference.py, bit for bit (torch.equal on
ids and score bits, CSR offsets and MMR pick order). No result of this library enters the reference: the scores are
`dot32` (the documented FMA order, emulated on the host), screened by torch float64 products.

a. Kernel level: every element of vr_score_exact (inside finite poison that must keep its bits) for each NQ
   instantiation with partial query blocks, nd around the EX_DW = 4 clamp, dims that leave lanes without a float4, and
   the largest dim the NQ = 8 instantiation fits; vr_score_lists and vr_group_pages_topm for every listed pair.
b. Operation level: a covering set (`plan()`, CASES) in which every operation meets every class of every other dimension - scope,
   k, path, data, dim, id_offset - at least once; a combination the API refuses asserts its documented error."""
import itertools
import zlib

import numpy as np
import pytest
import torch

from tests import dot_reference as X
from tests.test_mmr_host import mmr_model, rows_of
from visrag_b200 import _lib as L
from visrag_b200 import retriever as R

pytestmark = pytest.mark.gpu
f32 = np.float32


def _bits_equal(got, want):
    got = got.detach().cpu().numpy() if isinstance(got, torch.Tensor) else np.asarray(got)
    want = np.asarray(want)
    if got.dtype == f32:
        return got.shape == want.shape and np.array_equal(got.view(np.int32), want.astype(f32).view(np.int32))
    return got.shape == want.shape and np.array_equal(got, want)


def _same(got, want, what):
    assert len(got) == len(want), (what, len(got), len(want))
    for j, (g, w) in enumerate(zip(got, want)):
        assert _bits_equal(g, w), (what, j, g, w)


# ------------------------------------------------------------------------------------------------ a. kernel level
def _kernel_data(rs, n, dim):
    """Mixed-norm rows with cancelling pairs of elements, so that the FMA order shows in the bits."""
    x = rs.randn(n, dim) * 10.0 ** rs.uniform(-2, 2, (n, 1)) * 10.0 ** rs.uniform(-1, 1, (n, dim))
    h = dim // 2
    x[::3, h:2 * h] = -x[::3, :h] * (1 + 1e-3 * rs.randn((n + 2) // 3, h))
    return x.astype(f32)


NQS = [1, 2, 3, 4, 5, 7, 8, 9, 17]
NDS = [1, 2, 3, 4, 5, 31, 33, 4097]
DIMS = [4, 8, 12, 124, 128, 132, 2304, 6400]  # 6400: 8 query rows of 6400 floats fill the 200 KiB of shared memory


@pytest.mark.parametrize("dim", DIMS)
def test_score_exact_every_element(dim):
    """nd = 4097 meets NQ = 1, 4 and 8 (NQ = 1 and 2 at the large dims, <= 1e8 host FMAs); at dims up to 132 one nd
    larger than 32 pages x 3 blocks per SM makes each warp stride over several groups of EX_DW pages."""
    rs = np.random.RandomState(dim)
    big = dim > 1024
    nqs = NQS if not big else [1, 2, 3, 5, 8, 9]
    wide = {2304: [1, 4], 6400: [1, 2]}.get(dim, [1, 3, 4, 9, 17])  # query counts of the nd = 4097 cases
    nds = list(NDS)
    long_nd = 2 * 32 * 3 * torch.cuda.get_device_properties(0).multi_processor_count + 7
    if dim <= 132:
        nds.append(long_nd)
    Q, D = _kernel_data(rs, max(nqs), dim), _kernel_data(rs, max(nds), dim)
    ref33 = X.dot32(np.repeat(Q, 33, 0), np.tile(D[:33], (len(Q), 1))).reshape(len(Q), 33)
    ref_wide = X.dot32(np.repeat(Q[:max(wide)], max(nds), 0), np.tile(D, (max(wide), 1))).reshape(max(wide), max(nds))
    Qg, Dg = torch.from_numpy(Q).cuda(), torch.from_numpy(D).cuda()
    poison = f32(-1234.5)
    for nq, nd in itertools.product(nqs, nds):
        if nd > 33 and nq not in wide:
            continue
        pad = 37
        buf = torch.full((nq * nd + 2 * pad,), float(poison), device="cuda")
        L.check(L.lib().vr_score_exact(Qg.data_ptr(), nq, Dg.data_ptr(), nd, dim, buf[pad:].data_ptr(), L.stream_ptr()))
        out = buf.cpu().numpy()
        want = (ref_wide if nd > 33 else ref33)[:nq, :nd]
        assert _bits_equal(out[pad:pad + nq * nd].reshape(nq, nd), want), (nq, nd, dim)
        assert (out[:pad].view(np.int32) == poison.view(np.int32)).all() and \
            (out[pad + nq * nd:].view(np.int32) == poison.view(np.int32)).all(), ("poison", nq, nd, dim)


@pytest.mark.parametrize("dim", [8, 72, 136, 2304])
def test_score_lists_and_group_pages_every_pair(dim):
    rs = np.random.RandomState(dim + 1)
    nq, nd = 11, 3001
    Q, D = _kernel_data(rs, nq, dim), _kernel_data(rs, nd, dim)
    idx = R.build_index(D)
    q = torch.from_numpy(Q).cuda()
    # lists: lengths 0 .. 700 with repeated pages, shared by rows through list_of
    lens = [0, 1, 5, 33, 700]
    ids = np.concatenate([rs.randint(0, nd, n) for n in lens])
    off = np.r_[0, np.cumsum(lens)]
    of = rs.randint(0, len(lens), nq)
    ls = R._check_doc_lists((torch.from_numpy(off).cuda(), torch.from_numpy(ids).cuda()), idx, nq,
                            torch.from_numpy(of).cuda())
    W = ls.width
    sc = torch.empty((nq, W), device="cuda")
    si = torch.empty((nq, W), dtype=torch.int64, device="cuda")
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    L.check(L.lib().vr_score_lists(q.data_ptr(), nq, idx.emb.data_ptr(), nd, dim, ls.arg(ls.of_query), W, None,
                                   sc.data_ptr(), si.data_ptr(), None, status.data_ptr(), L.stream_ptr()))
    assert int(status.item()) == 0
    s, i = sc.cpu().numpy(), si.cpu().numpy()
    for r in range(nq):
        listed = np.sort(ids[off[of[r]]:off[of[r] + 1]])  # a repeated page keeps its entries (the select counts it once)
        live = i[r] >= 0
        assert np.array_equal(np.sort(i[r][live]), listed), r
        assert _bits_equal(s[r][live], X.dot32(np.repeat(Q[r:r + 1], live.sum(), 0), D[i[r][live]])), r
    # group pages: documents of 1 .. 9 pages and one of 600 (three pieces), m = 7
    groups = np.minimum(np.repeat(np.arange(nd), rs.randint(1, 10, nd))[:nd], 400)
    groups[2000:2600] = 401
    dg = torch.from_numpy(groups).cuda()
    ask = np.stack([rs.choice(402, 6, replace=False) for _ in range(nq)])
    ask[:, 0] = 401
    ps, pp = R.group_pages_topm(q, idx, torch.from_numpy(ask).cuda(), dg, 7, id_offset=3)
    ex = X.Exact(Q, D)
    ex.fill(np.stack([np.isin(groups, a) for a in ask]))
    for r in range(nq):
        for j, g in enumerate(ask[r]):
            cols = np.nonzero(groups == g)[0]
            o = X.order(ex.F[r, cols], cols)[:7]
            want_s = np.full(7, -np.inf, f32)
            want_p = np.full(7, -1, np.int64)
            want_s[:o.size], want_p[:o.size] = ex.F[r, cols[o]], cols[o] + 3
            assert _bits_equal(ps[r, j], want_s) and _bits_equal(pp[r, j], want_p), (r, g)


# ------------------------------------------------------------------------------------------------ b. operation level
OPS = ["topk", "groups", "capped", "groups_pages", "range", "range_groups", "hybrid_sum", "hybrid_rrf", "hybrid_groups",
       "mmr"]
SCOPES = ["none", "mask", "masks", "lists"]
KS = [1, 16, 17, 32, 33, 300, 301, 1024, 4096]
PATHS = ["scan", "filter", "fallback", "deep", "force_exact"]
DATA = ["unit", "mixed", "dup0", "nonfinite", "big"]
CASE_DIMS = [8, 72, 136, 2304]
OFFSETS = [0, 1 << 33]
AXES = dict(scope=SCOPES, k=KS, path=PATHS, data=DATA, dim=CASE_DIMS, off=OFFSETS)
RANGE_OPS = ("range", "range_groups")
# no deep route: range search has a threshold, not a k, and MMR's dense call fetches at most MMR_MAX_FETCH = 128 pages
NO_DEEP = RANGE_OPS + ("mmr",)
ZERO_PAGES = np.arange(6, 14)  # the dup0 class's zero-score pages: eligible in every scope, never a hit


def refusal(op, c):
    """The documented error of a combination the API refuses (None: allowed)."""
    return _refused(op, c)[0]


def _refused(op, c):
    """(error, the axis whose class the API refuses) or (None, None)."""
    if op in RANGE_OPS and c["scope"] == "lists":
        return TypeError, "scope"  # score_range(_groups) take no doc_lists
    if op in ("hybrid_sum", "hybrid_rrf", "hybrid_groups", "mmr") and c["path"] == "force_exact":
        return TypeError, "path"  # no force_exact argument: the dense call picks its route
    if op == "mmr" and c["k"] > R.MMR_MAX_FETCH:
        return ValueError, "k"  # k <= fetch_k <= mmr_fetch_max(dim)
    return None, None


def valid(op, c):
    """Whether a combination is a meaningful case (refused ones are)."""
    if refusal(op, c):
        return True
    if c["path"] == "deep":  # the route of 300 < k <= 1024 (the dense call's k), with no lists
        if op in NO_DEEP or c["scope"] == "lists" or not 300 < c["k"] <= 1024:
            return False
    elif c["k"] in (301, 1024) and c["path"] in ("filter", "fallback") and op not in RANGE_OPS + ("mmr",):
        return False  # those k take the deep route on a large problem
    if c["data"] == "nonfinite" and c["dim"] > 136:
        return False  # a non-finite query row is scored against every page on the host
    if c["dim"] == 2304 and (c["k"] > 33 or c["path"] == "fallback"):
        return False  # host budget
    if c["data"] == "dup0" and (c["dim"] < 128 or (c["k"] < 16 and op not in RANGE_OPS)):
        return False  # -0 needs every lane to hold a float4; k >= 16 takes all eight zero-score pages of a row
    return True


def plan():
    """Greedy covering set: walk the combinations in a fixed pseudo-random order and keep each valid one that covers a
    new (operation, axis, class) cell."""
    rs = np.random.RandomState(2024)
    need = {(op, a, v) for op in OPS for a, vals in AXES.items() for v in vals}
    cases = []
    combos = [dict(zip(AXES, t)) for t in itertools.product(*AXES.values())]
    order = rs.permutation(len(combos))
    for op in OPS:
        for i in order:
            c = combos[i]
            if not valid(op, c):
                continue
            err, axis = _refused(op, c)
            cells = {(op, axis, c[axis])} if err else {(op, a, c[a]) for a in AXES}  # a refusal covers its own cell
            if cells & need:
                need -= cells
                cases.append((op, c))
        # cells no valid combination can reach stay in need
    # -0 against +0 on the large routes: per-query masks on the filter path and, where it exists, the deep route
    for op in OPS:
        cases.append((op, dict(scope="masks", k=33, path="filter", data="dup0", dim=136, off=0)))
        if op not in NO_DEEP:
            cases.append((op, dict(scope="masks", k=301, path="deep", data="dup0", dim=136, off=1 << 33)))
    return cases, need


CASES, UNREACHED = plan()


def test_covering_set():
    """Every (operation, axis, class) cell is met, except the ones no valid combination has (printed)."""
    table = {}
    for op, c in CASES:
        err, axis = _refused(op, c)
        for a in [axis] if err else AXES:
            table.setdefault((op, a, c[a]), "refused" if err else "run")
    lines = []
    for a, vals in AXES.items():
        lines.append(f"{a:>6} | " + " ".join(f"{str(v):>11}" for v in vals))
        for op in OPS:
            lines.append(f"{op:>14} " + " ".join(f"{table.get((op, a, v), '-'):>11}" for v in vals))
    print("\n".join(lines))
    allowed = {(op, "path", "deep") for op in NO_DEEP}
    assert UNREACHED <= allowed, sorted(UNREACHED - allowed)


def _unit(rs, n, dim):
    x = rs.randn(n, dim)
    return x / np.linalg.norm(x, axis=1, keepdims=True)


def make_problem(c, seed):
    """(Q, D, doc_groups) for one case: a small problem for the scan, nq * nd > 2^22 otherwise; clustered pages for the
    fallback path; then the data class."""
    rs = np.random.RandomState(seed)
    dim = c["dim"]
    if c["path"] == "scan":
        nq, nd = 6, 2003
    else:
        nq = 48 if dim == 2304 else 16
        nd = (1 << 22) // nq + 101
    if c["path"] == "fallback":  # 64 centres, each with thousands of pages a relative 1e-6 apart
        cen = _unit(rs, 64, dim)
        D = cen[rs.randint(0, 64, nd)] * (1 + 1e-6 * rs.randn(nd, 1)) + 1e-6 * rs.randn(nd, dim) / np.sqrt(dim)
        Q = cen[rs.randint(0, 64, nq)] + 1e-3 * rs.randn(nq, dim) / np.sqrt(dim)
    else:
        D, Q = _unit(rs, nd, dim), _unit(rs, nq, dim)
    if c["data"] == "mixed":
        D = D * 10.0 ** rs.uniform(-3, 3, (nd, 1))
        Q = Q * 10.0 ** rs.uniform(-3, 3, (nq, 1))
    Q, D = Q.astype(f32), D.astype(f32)
    if c["data"] == "dup0":
        # queries 0 .. 2 point away from every page (scores near -0.9), so the zero-score pages 6 .. 13 head their rows
        away = _unit(rs, 1, dim)[0]
        D = D + f32(2) * away.astype(f32)
        D /= np.linalg.norm(D, axis=1, keepdims=True)
        Q[:3] = -away + 0.01 * rs.randn(3, dim) / np.sqrt(dim)
        D[1::5] = D[0:-1:5][: len(D[1::5])]  # exact duplicates
        D[6] = D[13] = 0  # +0 for every query
        for r in range(3):  # every product of query r rounds to -0: exactly (-0 q_i) or by underflow (2^-149 |q_i| < 2^-150)
            D[7 + r] = -np.sign(Q[r]) * np.where(np.abs(Q[r]) < 0.5, f32(2.0 ** -149), f32(0))
            D[10 + r] = D[7 + r]
    elif c["data"] == "nonfinite":
        D[3, 0], D[4, 0], D[5, 0] = np.nan, np.inf, -np.inf
        Q[1, 0] = np.nan
    elif c["data"] == "big":
        Q[0] *= f32(1e6)  # the fp16 copy overflows: the row cannot be proved on the tensor cores
    sizes = rs.randint(1, 10, nd)
    groups = np.repeat(np.arange(nd), sizes)[:nd]
    groups[100:400] = groups[100]  # one document of 300 pages (two pieces of the page stage)
    groups[ZERO_PAGES] = nd + np.arange(ZERO_PAGES.size)  # each zero-score page is a document of its own
    return Q, D, np.unique(groups, return_inverse=True)[1].astype(np.int64)


def make_scope(c, rs, nq, nd):
    """(kwargs of the call, eligibility [nq, nd] of the reference)."""
    dev = "cuda"
    if c["scope"] == "none":
        return {}, np.ones((nq, nd), bool)
    if c["scope"] == "mask":
        m = rs.rand(nd) < 0.7
        m[ZERO_PAGES] = True
        return dict(doc_mask=torch.from_numpy(m).to(dev)), np.repeat(m[None], nq, 0)
    if c["scope"] == "masks":
        M = rs.rand(3, nd) < np.asarray([[0.9], [0.5], [0.02]])
        M[:, ZERO_PAGES] = True
        of = rs.randint(0, 3, nq)
        return dict(doc_mask=torch.from_numpy(M).to(dev), mask_of=torch.from_numpy(of).to(dev)), M[of]
    lens = [min(nd, 5000), 40, 700]
    ids = np.concatenate([np.r_[ZERO_PAGES, rs.randint(0, nd, n)] for n in lens])
    off = np.r_[0, np.cumsum(np.asarray(lens) + ZERO_PAGES.size)]
    of = rs.randint(0, 3, nq)
    elig = np.zeros((nq, nd), bool)
    for r in range(nq):
        elig[r, ids[off[of[r]]:off[of[r] + 1]]] = True
    return dict(doc_lists=(torch.from_numpy(off).to(dev), torch.from_numpy(ids).to(dev)),
                list_of=torch.from_numpy(of).to(dev)), elig


def make_hits(rs, ex, elig, k):
    """Per query: 60 random pages and a few of its eligible top pages (pages 16 and up: the zero-score pages keep their
    dense bits), values up to the spread of its scores, some 0 and -0."""
    nq, nd = elig.shape
    top = X.topk(ex, min(k, 50) + ZERO_PAGES.size, elig)[1]
    off, ids, vals = [0], [], []
    for r in range(nq):
        pages = set(rs.choice(np.arange(16, nd), 60, replace=False).tolist()) | set([int(p) for p in top[r] if p >= 16][:5])
        pages = np.asarray(sorted(pages))
        v = rs.rand(pages.size).astype(f32)
        v[rs.rand(pages.size) < 0.1] = 0.0
        v[rs.rand(pages.size) < 0.1] = -0.0
        ids.append(pages)
        vals.append(v)
        off.append(off[-1] + pages.size)
    return np.asarray(off), np.concatenate(ids), np.concatenate(vals)


def _to_dev(hits):
    off, ids, vals = hits
    return (torch.from_numpy(off).cuda(), torch.from_numpy(ids).cuda(), torch.from_numpy(vals).cuda())


def _screen(Q, D):
    q64, d64 = torch.from_numpy(Q).cuda().double(), torch.from_numpy(D).cuda().double()
    S64, A64 = (q64 @ d64.T).cpu().numpy(), (q64.abs() @ d64.abs().T).cpu().numpy()
    return X.Exact(Q, D, S64, A64)


def _path_ok(op, c, stats):
    """stats say that the intended route ran."""
    p = stats.get("path")
    pages = op in ("topk", "hybrid_sum", "hybrid_rrf", "mmr")
    if c["scope"] == "lists" and (pages or c["k"] <= R.LIST_GROUPS_MAX_K):  # documents past 256 take the masked path
        return p == "lists"
    if c["path"] in ("scan", "force_exact"):
        return p == "exact"
    if c["path"] == "deep":
        return p == "deep"
    if c["path"] == "fallback":
        if op in RANGE_OPS:
            return p == "filter+rescore" and stats["fallback"] > 0
        return p == "filter+rescore" and stats["flagged"] > 0
    return p == "filter+rescore"


@pytest.mark.parametrize("op,c", CASES, ids=[f"{op}-" + "-".join(str(v) for v in c.values()) for op, c in CASES])
def test_operation_against_the_reference(op, c):
    seed = zlib.crc32(repr((op, c)).encode())
    rs = np.random.RandomState(seed)
    Q, D, groups = make_problem(c, seed)
    nq, nd = Q.shape[0], D.shape[0]
    idx = R.build_index(D)
    q = torch.from_numpy(Q).cuda()
    dg = torch.from_numpy(groups).cuda()
    kw, elig = make_scope(c, rs, nq, nd)
    k, off = c["k"], c["off"]
    force = dict(force_exact=True) if c["path"] == "force_exact" else {}
    err = refusal(op, c)
    stats = {}
    if err is not None:
        with pytest.raises(err):
            if op in RANGE_OPS:
                R.score_range(q, idx, 0.0, **kw, **force) if op == "range" else R.score_range_groups(q, idx, 0.0, dg, **kw)
            elif op == "mmr":
                R.score_mmr(q, idx, k, 0.5, fetch_k=min(max(k, 20), R.MMR_MAX_FETCH), **kw, **force)
            else:
                hits = _to_dev((np.zeros(nq + 1, np.int64), np.zeros(0, np.int64), np.zeros(0, f32)))
                fn = {"hybrid_sum": R.score_topk_hybrid, "hybrid_rrf": R.score_topk_hybrid,
                      "hybrid_groups": R.score_topk_groups_hybrid}[op]
                fn(q, idx, k, *((dg,) if op == "hybrid_groups" else ()), hits, **kw, **force)
        return
    ex = _screen(Q, D)
    if op == "topk":
        got = R.score_topk(q, idx, k, off, stats=stats, **kw, **force)
        want = X.topk(ex, k, elig, off)
    elif op == "groups":
        got = R.score_topk_groups(q, idx, k, dg, off, stats=stats, **kw, **force)
        want = X.topk_groups(ex, k, groups, elig, off)
    elif op == "capped":
        m = 1 + seed % 3
        got = R.score_topk_capped(q, idx, k, dg, m, off, stats=stats, **kw, **force)
        want = X.topk_capped(ex, k, groups, m, elig, off)
    elif op == "groups_pages":
        m = 1 + seed % 4
        got = R.score_topk_groups_pages(q, idx, k, dg, m, off, stats=stats, **kw, **force)
        want = X.topk_groups_pages(ex, k, groups, m, elig, off)
    elif op in RANGE_OPS:
        # thresholds per query: each row's k-th best score (finite), -inf for a row without one
        kth = X.topk(ex, k, elig)[0][:, -1]
        t = np.where(np.isfinite(kth), kth, -np.inf).astype(f32)
        if c["path"] == "scan" and c["dim"] <= 72:
            t[0] = -np.inf  # every eligible page, -inf scores included
        cap = dict(cap=1) if c["path"] == "fallback" else {}
        tt = torch.from_numpy(t).cuda()
        if op == "range":
            got = R.score_range(q, idx, tt, off, stats=stats, **kw, **force, **cap)
            want = X.range_pages(ex, t, elig, off)
        else:
            got = R.score_range_groups(q, idx, tt, dg, off, stats=stats, **kw, **force, **cap)
            want = X.range_groups(ex, t, groups, elig, off)
    elif op in ("hybrid_sum", "hybrid_groups"):
        hits = make_hits(rs, ex, elig, k)
        w = 0.05 * float(np.nanmedian(np.abs(D[np.isfinite(D).all(1)])) * np.sqrt(c["dim"]))
        if op == "hybrid_sum":
            got = R.score_topk_hybrid(q, idx, k, _to_dev(hits), w, id_offset=off, stats=stats, **kw)
            want = X.hybrid_sum(ex, k, hits, w, elig, off)
        else:
            got = R.score_topk_groups_hybrid(q, idx, k, dg, _to_dev(hits), w, id_offset=off, stats=stats, **kw)
            want = X.hybrid_groups(ex, k, groups, hits, w, elig, off)
    elif op == "hybrid_rrf":
        hits = make_hits(rs, ex, elig, k)
        window = min(4096, max(k, 10 if k < 300 else k))
        got = R.score_topk_hybrid(q, idx, k, _to_dev(hits), fusion="rrf", window=window, rrf_c=60, id_offset=off,
                                  stats=stats, **kw)
        want = X.hybrid_rrf(ex, k, hits, window, 60, elig, off)
    else:  # mmr
        fetch = min(R.mmr_fetch_max(c["dim"]), max(k, 40))
        lam = 0.5 if seed % 2 else 0.25
        got = R.score_mmr(q, idx, k, lam, fetch_k=fetch, id_offset=off, stats=stats, **kw)
        cs, ci = X.topk(ex, fetch, elig)
        rows = [rows_of(mmr_model(cs[r], ci[r], X.gram32(D, ci[r]), lam, k), cs[r], ci[r], k, off) for r in range(nq)]
        want = (np.stack([r[0] for r in rows]), np.stack([r[1] for r in rows]))
    if c["data"] == "dup0" and op not in ("hybrid_rrf", "mmr"):  # the fixture must keep producing both zeros
        z = np.asarray(want[1] if op in RANGE_OPS else want[0]).ravel()
        z = z[z == 0]
        assert np.signbit(z).any() and (~np.signbit(z)).any(), (op, c, "the reference holds no -0 or no +0 score")
    _same(got, want, (op, c))
    assert _path_ok(op, c, stats), (op, c, {a: b for a, b in stats.items() if a != "candidates"})


def test_range_every_page_and_minus_inf_scores():
    """t = -inf: every eligible page, a -inf score included; t = +inf: only +inf scores."""
    rs = np.random.RandomState(5)
    Q, D = _unit(rs, 3, 136).astype(f32), _unit(rs, 900, 136).astype(f32)
    D[10, 0], D[11, 0], D[12, 0] = -np.inf, np.inf, np.nan
    Q[:, 0] = np.abs(Q[:, 0]) + f32(0.01)
    idx = R.build_index(D)
    ex = X.Exact(Q, D)
    for t in (-np.inf, np.inf):
        tt = np.full(3, t, f32)
        got = R.score_range(torch.from_numpy(Q).cuda(), idx, float(t), id_offset=1 << 33)
        _same(got, X.range_pages(ex, tt, None, 1 << 33), t)
    off, s, i = X.range_pages(ex, np.full(3, -np.inf, f32), None)
    assert off[1] - off[0] == 899 and s[off[1] - 1] == -np.inf  # NaN left out, -inf kept last
