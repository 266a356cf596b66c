"""An independent, bit-exact host reference of the retrieval operations (numpy only; nothing of visrag_b200).

Every path that scores a (query, page) pair computes the fp32 dot product in one documented order (DESIGN §4): lane l
of a warp takes the float4s l, l + 32, ... of the row, and within each float4 runs fma(d.x, q.x, acc), then y, z and w;
then the warp adds its lanes by the butterfly v += shfl_xor(v, o) for o = 16, 8, 4, 2, 1, and lane 0 holds the score.
`dot32` restates that order with a correctly rounded fp32 FMA emulated in float64 (`fma32`), so its bits are the bits a
kernel must produce, whatever kernel of this library computes them.

Scoring every pair of a real problem that way is too slow on a CPU, so the reference screens with float64:

* `dot_bound(A)` bounds |dot32 - q.d| for a pair with A = sum |q_i d_i|, and `width` adds the error of a float64
  product (any summation order) to it. With S64 and A64 the float64 products, lo = S64 - width and hi = S64 + width
  bracket the fp32 score: lo <= dot32 <= hi.
* Top-k: let L_k be the k-th largest lo of a row. A page with hi < L_k has fp32 <= hi < L_k, while the k pages with the
  largest lo have fp32 >= lo >= L_k; so at least k pages rank strictly before it, and it cannot be among the first k.
  Only pages with hi >= L_k (the candidates) are scored by `dot32`, and the answer is decided from those bits alone.
* Range: a page with hi < t has fp32 < t. Documents: the same rules on each document's best page (max lo, max hi).
* Capped top-k: L is the k-th largest lo among at most m pages of each document (each document's m largest lo).
  When the walk reaches a page with hi < L, every one of those k pages comes before it and was picked, or skipped
  because its document already had m picks, each of which also comes before it: k picks precede it.

Pairs whose operands are not finite, or whose sum could overflow fp32, bypass the screen (lo = -inf, hi = +inf): they
are always candidates and are scored by `dot32` directly.

The operations follow their DESIGN §4 definitions: rows ordered by (score desc, id asc), +0 and -0 tie, NaN is never
selected, a top-k row ends in (-inf, -1), ids carry id_offset.
"""
import numpy as np

f32, f64 = np.float32, np.float64
U32 = 2.0 ** -24           # unit roundoff of fp32
U64 = 2.0 ** -53           # unit roundoff of float64
TINY32 = 2.0 ** -149       # the smallest fp32 subnormal: an underflowing operation errs by at most half of it


def gamma(n, u=U32):
    return n * u / (1 - n * u)


# ------------------------------------------------------------------------------------------------ the arithmetic
def fma32(a, b, c):
    """fl32(a * b + c) rounded once, elementwise, for fp32 arrays a, b, c. a * b is exact in float64 (24 + 24 bits);
    TwoSum gives p + c = s + e exactly; s is rounded to odd (an even last bit steps one ulp toward e when e != 0),
    which keeps the sticky information, and the cast to fp32 then rounds correctly (53 >= 24 + 2 bits). When p or c is
    not finite, fl32(p + c) is already the IEEE result."""
    a, b, c = (np.asarray(x, f32).astype(f64) for x in (a, b, c))
    with np.errstate(invalid="ignore", over="ignore"):
        p = a * b
        s = p + c
        bb = s - p
        e = (p - (s - bb)) + (c - bb)
        finite = np.isfinite(p) & np.isfinite(c)
        bits = s.view(np.int64)
        fix = finite & (e != 0) & ((bits & 1) == 0)
        bits = np.where(fix, bits + np.where((e > 0) == (s > 0), 1, -1), bits)
        return bits.view(f64).astype(f32)


def lane_sums(q, d, fma=fma32):
    """[P, 32] fp32: each lane's FMA chain for the paired rows q[p], d[p] ([P, dim] fp32, dim % 4 == 0)."""
    P, dim = q.shape
    nv = dim // 4
    acc = np.zeros((P, 32), f32)
    q4, d4 = q.reshape(P, nv, 4), d.reshape(P, nv, 4)
    for i0 in range(0, nv, 32):
        n = min(32, nv - i0)
        for c in range(4):
            acc[:, :n] = fma(d4[:, i0:i0 + n, c], q4[:, i0:i0 + n, c], acc[:, :n])
    return acc


def butterfly(acc):
    """Lane 0 of the xor butterfly v += shfl_xor(v, o), o = 16, 8, 4, 2, 1 (each add rounded to fp32)."""
    lanes = np.arange(32)
    with np.errstate(invalid="ignore", over="ignore"):
        for o in (16, 8, 4, 2, 1):
            acc = acc + acc[:, lanes ^ o]
    return acc[:, 0]


def dot32(q, d, chunk=4096):
    """The fp32 score of each pair of rows (q[p], d[p]) in the kernels' order: [P] fp32."""
    q, d = np.asarray(q, f32), np.asarray(d, f32)
    out = np.empty(q.shape[0], f32)
    for p0 in range(0, q.shape[0], chunk):
        out[p0:p0 + chunk] = butterfly(lane_sums(q[p0:p0 + chunk], d[p0:p0 + chunk]))
    return out


def chain_len(dim):
    """m: the FMAs of the longest lane chain."""
    return 4 * -(-dim // 128)


def dot_bound(A, dim):
    """|dot32 - q.d| <= gamma_{m+5} A + (dim + 31) 2^-149 for A = sum |q_i d_i|: a product reaches lane 0 through at most
    m FMAs and 5 butterfly adds, and each of the dim + 31 operations adds at most half a subnormal ulp when it underflows
    (finite operands and no fp32 overflow)."""
    return gamma(chain_len(dim) + 5) * A + (dim + 31) * TINY32


def width(A64, dim):
    """Half-width of [lo, hi] around a float64 score S64 computed in any order, A64 the float64 sum |q_i d_i| computed
    likewise: S64 and A64 each err by at most gamma64_dim times the exact A."""
    g = gamma(dim, U64)
    A = A64 / (1 - g) * (1 + 2.0 ** -40)
    return dot_bound(A, dim) + g * A


# ------------------------------------------------------------------------------------------------ orderings
def order(scores, ids):
    """Positions of the entries in (score desc, id asc) order, NaN dropped, +0 == -0."""
    scores, ids = np.asarray(scores, f32), np.asarray(ids, np.int64)
    at = np.nonzero(~np.isnan(scores))[0]
    key = -scores[at].astype(f64) + 0.0  # -(-0) = +0 and -(+0) + 0 = +0: the zeros tie
    return at[np.lexsort((ids[at], key))]


def first_per_group(pos, groups):
    """The first position of each group, in the given order."""
    _, first = np.unique(groups[pos], return_index=True)
    return pos[np.sort(first)]


def kth_largest(v, k):
    """Row-wise k-th largest of v [n, c] (-inf where a row has fewer than k entries)."""
    if k > v.shape[1]:
        return np.full(v.shape[0], -np.inf)
    return -np.partition(-v, k - 1, axis=1)[:, k - 1]


def _pad(rows, k, dtypes):
    out = [np.full((len(rows), k), -np.inf if dt == f32 else -1, dt) for dt in dtypes]
    for r, row in enumerate(rows):
        for o, v in zip(out, row):
            o[r, :len(v)] = v[:k]
    return out


# ------------------------------------------------------------------------------------------------ the screen
class Exact:
    """fp32 scores of Q [nq, dim] x D [nd, dim] on demand. S64 / A64: float64 Q @ D.T and |Q| @ |D|.T (computed here
    when not given). screen=False makes every pair a candidate (the full dot32 answer). `F[r, c]` holds dot32 for every
    pair `fill` has been asked for."""

    def __init__(self, Q, D, S64=None, A64=None, screen=True):
        self.Q, self.D = np.ascontiguousarray(Q, f32), np.ascontiguousarray(D, f32)
        nq, dim = self.Q.shape
        nd = self.D.shape[0]
        with np.errstate(invalid="ignore", over="ignore"):
            if S64 is None:
                S64 = self.Q.astype(f64) @ self.D.T.astype(f64)
            if A64 is None:
                A64 = np.abs(self.Q.astype(f64)) @ np.abs(self.D.T.astype(f64))
            w = width(np.asarray(A64, f64), dim)
            risky = ~(np.isfinite(self.Q).all(1)[:, None] & np.isfinite(self.D).all(1)[None, :]) | ~(A64 < 2.0 ** 126)
            if not screen:
                risky = np.ones((nq, nd), bool)
            self.lo = np.where(risky, -np.inf, S64 - w)
            self.hi = np.where(risky, np.inf, S64 + w)
        self.F = np.full((nq, nd), np.nan, f32)
        self.known = np.zeros((nq, nd), bool)
        self.scored = 0

    def fill(self, want):
        r, c = np.nonzero(want & ~self.known)
        if r.size:
            for p0 in range(0, r.size, 1 << 16):
                rr, cc = r[p0:p0 + (1 << 16)], c[p0:p0 + (1 << 16)]
                self.F[rr, cc] = dot32(self.Q[rr], self.D[cc])
            self.known[r, c] = True
            self.scored += r.size

    def scores(self, r, cols):
        assert self.known[r, cols].all()
        return self.F[r, cols]


def _elig(ex, elig):
    return np.ones(ex.F.shape, bool) if elig is None else np.asarray(elig, bool)


def screen_topk(lo, hi, elig, k):
    """Candidates of a top-k: eligible pages with hi >= the k-th largest eligible lo."""
    Lk = kth_largest(np.where(elig, lo, -np.inf), k)
    return elig & (hi >= Lk[:, None])


def _doc_max(v, groups, G):
    """Row-wise max of v [n, nd] over each group's pages: [n, G] (-inf for a group without pages)."""
    by = np.argsort(groups, kind="stable")
    g = groups[by]
    start = np.r_[0, np.nonzero(g[1:] != g[:-1])[0] + 1]
    out = np.full((v.shape[0], G), -np.inf)
    out[:, g[start]] = np.maximum.reduceat(v[:, by], start, axis=1)
    return out


def screen_groups(lo, hi, elig, groups, k):
    """Candidate pages of a top-k over documents scored by their best page: the pages of documents whose best hi
    reaches the k-th largest best lo, and of those only pages whose hi reaches their document's best lo."""
    G = int(groups.max()) + 1
    dlo = _doc_max(np.where(elig, lo, -np.inf), groups, G)
    dhi = _doc_max(np.where(elig, hi, -np.inf), groups, G)
    has = _doc_max(np.where(elig, 0.0, -np.inf), groups, G) == 0
    Lk = kth_largest(dlo, k)
    keep_doc = has & (dhi >= Lk[:, None])
    return elig & keep_doc[:, groups] & (hi >= dlo[:, groups])


# ------------------------------------------------------------------------------------------------ the operations
def topk(ex, k, elig=None, id_offset=0):
    """score_topk: (scores [nq, k] f32, ids [nq, k] i64)."""
    elig = _elig(ex, elig)
    cand = screen_topk(ex.lo, ex.hi, elig, k)
    ex.fill(cand)
    rows = []
    for r in range(cand.shape[0]):
        cols = np.nonzero(cand[r])[0]
        s = ex.scores(r, cols)
        o = order(s, cols)[:k]
        rows.append((s[o], cols[o] + id_offset))
    return _pad(rows, k, (f32, np.int64))


def _group_rows(ex, cand, groups):
    """Per row: (scores, pages) of each document's best candidate page, documents in (score desc, best page asc)."""
    ex.fill(cand)
    for r in range(cand.shape[0]):
        cols = np.nonzero(cand[r])[0]
        s = ex.scores(r, cols)
        o = first_per_group(order(s, cols), groups[cols])
        yield s[o], cols[o]


def topk_groups(ex, k, groups, elig=None, id_offset=0):
    """score_topk_groups: (scores, best pages, groups) [nq, k]."""
    elig = _elig(ex, elig)
    rows = [(s, p + id_offset, groups[p]) for s, p in _group_rows(ex, screen_groups(ex.lo, ex.hi, elig, groups, k), groups)]
    rows = [tuple(v[:k] for v in row) for row in rows]
    return _pad(rows, k, (f32, np.int64, np.int64))


def topk_groups_pages(ex, k, groups, m, elig=None, id_offset=0):
    """score_topk_groups_pages: the top-k documents, each with its m best eligible pages ([nq, k, m], (-inf, -1) tail)."""
    elig = _elig(ex, elig)
    s, p, g = topk_groups(ex, k, groups, elig, id_offset)
    ps = np.full((s.shape[0], k, m), -np.inf, f32)
    pp = np.full((s.shape[0], k, m), -1, np.int64)
    want = np.zeros(elig.shape, bool)
    for r in range(s.shape[0]):
        want[r] = elig[r] & np.isin(groups, g[r][g[r] >= 0])
    ex.fill(want)
    for r in range(s.shape[0]):
        for j, doc in enumerate(g[r]):
            if doc < 0:
                continue
            cols = np.nonzero(want[r] & (groups == doc))[0]
            sc = ex.scores(r, cols)
            o = order(sc, cols)[:m]
            ps[r, j, :o.size], pp[r, j, :o.size] = sc[o], cols[o] + id_offset
    return s, p, g, ps, pp


def topk_capped(ex, k, groups, m, elig=None, id_offset=0):
    """score_topk_capped: walk the pages in (score desc, id asc) order and pick each whose document has fewer than m
    picks, until k picks: (scores, pages, groups) [nq, k]."""
    elig = _elig(ex, elig)
    nq, nd = elig.shape
    L = np.full(nq, -np.inf)
    for r in range(nq):  # the k-th largest lo among each document's m largest lo
        at = np.nonzero(elig[r] & np.isfinite(ex.lo[r]))[0]
        o = at[np.lexsort((-ex.lo[r, at], groups[at]))]
        g = groups[o]
        start = np.r_[0, np.nonzero(g[1:] != g[:-1])[0] + 1]
        rank = np.arange(o.size) - np.repeat(start, np.diff(np.r_[start, o.size]))
        top = np.sort(ex.lo[r, o[rank < m]])[::-1]
        if top.size >= k:
            L[r] = top[k - 1]
    cand = elig & (ex.hi >= L[:, None])
    ex.fill(cand)
    rows = []
    for r in range(nq):
        cols = np.nonzero(cand[r])[0]
        s = ex.scores(r, cols)
        picks, count = [], {}
        for i in order(s, cols):
            g = int(groups[cols[i]])
            if count.get(g, 0) < m:
                count[g] = count.get(g, 0) + 1
                picks.append(i)
                if len(picks) == k:
                    break
        picks = np.asarray(picks, np.int64)
        rows.append((s[picks], cols[picks] + id_offset, groups[cols[picks]]))
    return _pad(rows, k, (f32, np.int64, np.int64))


def _csr(rows, with_groups=False):
    counts = [len(r[0]) for r in rows]
    offsets = np.zeros(len(rows) + 1, np.int64)
    offsets[1:] = np.cumsum(counts)
    cat = [np.concatenate([r[j] for r in rows]) if rows else np.zeros(0) for j in range(3 if with_groups else 2)]
    return (offsets, cat[0].astype(f32), *[c.astype(np.int64) for c in cat[1:]])


def range_pages(ex, t, elig=None, id_offset=0):
    """score_range: CSR (offsets, scores, ids) of every eligible page with fp32 score >= t[r]."""
    elig = _elig(ex, elig)
    t = np.asarray(t, f32)
    cand = elig & (ex.hi >= t[:, None])
    ex.fill(cand)
    rows = []
    for r in range(cand.shape[0]):
        cols = np.nonzero(cand[r])[0]
        s = ex.scores(r, cols)
        o = order(s, cols)
        o = o[s[o] >= t[r]]
        rows.append((s[o], cols[o] + id_offset))
    return _csr(rows)


def range_groups(ex, t, groups, elig=None, id_offset=0):
    """score_range_groups: CSR (offsets, scores, best pages, groups) of every document whose best eligible page scores
    >= t[r]; that page has fp32 >= t, so hi >= t, and the page screen keeps it."""
    elig = _elig(ex, elig)
    t = np.asarray(t, f32)
    cand = elig & (ex.hi >= t[:, None])
    rows = []
    for r, (s, p) in enumerate(_group_rows(ex, cand, groups)):
        keep = s >= t[r]
        rows.append((s[keep], p[keep] + id_offset, groups[p[keep]]))
    return _csr(rows, with_groups=True)


def hit_matrix(hits, nq, nd, elig=None):
    """Dense (values f32 [nq, nd] with -0 as +0, listed bool [nq, nd]) of a CSR hit list (offsets, ids, values); hits
    outside a query's scope are dropped."""
    off, ids, vals = (np.asarray(h) for h in hits)
    V = np.zeros((nq, nd), f32)
    listed = np.zeros((nq, nd), bool)
    row = np.repeat(np.arange(nq), np.diff(off))
    V[row, ids] = vals.astype(f32) + f32(0)
    listed[row, ids] = True
    if elig is not None:
        listed &= elig
        V = np.where(listed, V, f32(0))
    return V, listed


def _fused_bounds(ex, wv, listed):
    """[lo, hi] of fl(dense + wv) on listed pages (fl is monotone, and errs by at most 2^-24 |x| + 2^-150)."""
    with np.errstate(invalid="ignore"):
        lo, hi = ex.lo + wv, ex.hi + wv
        lo = np.where(listed, lo - 2.0 ** -23 * np.abs(lo) - TINY32, ex.lo)
        hi = np.where(listed, hi + 2.0 ** -23 * np.abs(hi) + TINY32, ex.hi)
    return lo, hi


def _fused(ex, r, cols, wv, listed):
    s = ex.scores(r, cols)
    with np.errstate(invalid="ignore", over="ignore"):
        return np.where(listed[r, cols], s + wv[r, cols], s).astype(f32)


def hybrid_sum(ex, k, hits, w, elig=None, id_offset=0):
    """score_topk_hybrid(fusion="sum"): a listed page scores fl(dense + fl(w v)), an unlisted one its dense score."""
    elig = _elig(ex, elig)
    V, listed = hit_matrix(hits, *elig.shape, elig)
    wv = (f32(w) * V).astype(f32)
    lo, hi = _fused_bounds(ex, wv, listed)
    cand = screen_topk(lo, hi, elig, k)
    ex.fill(cand)
    rows = []
    for r in range(cand.shape[0]):
        cols = np.nonzero(cand[r])[0]
        s = _fused(ex, r, cols, wv, listed)
        o = order(s, cols)[:k]
        rows.append((s[o], cols[o] + id_offset))
    return _pad(rows, k, (f32, np.int64))


def hybrid_groups(ex, k, groups, hits, w, elig=None, id_offset=0):
    """score_topk_groups_hybrid: a document scores the max fused score of its eligible pages."""
    elig = _elig(ex, elig)
    V, listed = hit_matrix(hits, *elig.shape, elig)
    wv = (f32(w) * V).astype(f32)
    lo, hi = _fused_bounds(ex, wv, listed)
    cand = screen_groups(lo, hi, elig, groups, k)
    ex.fill(cand)
    rows = []
    for r in range(cand.shape[0]):
        cols = np.nonzero(cand[r])[0]
        s = _fused(ex, r, cols, wv, listed)
        o = first_per_group(order(s, cols), groups[cols])[:k]
        rows.append((s[o], cols[o] + id_offset, groups[cols[o]]))
    return _pad(rows, k, (f32, np.int64, np.int64))


def rrf_term(c, rank):
    return (f32(1) / f32(c + rank)).astype(f32)


def hybrid_rrf(ex, k, hits, window, c, elig=None, id_offset=0):
    """score_topk_hybrid(fusion="rrf"): over the union of the dense top-window and the query's hits,
    fl(1/fl(c + rank_dense) + 1/fl(c + rank_ext)), ranks from 1, the external rank by (value desc, id asc), a missing
    rank adding 0."""
    elig = _elig(ex, elig)
    nq, nd = elig.shape
    _, dense = topk(ex, window, elig)
    off, ids, vals = (np.asarray(h) for h in hits)
    rows = []
    for r in range(nq):
        score = {}
        for j, p in enumerate(dense[r]):
            if p >= 0:
                score[int(p)] = [rrf_term(c, j + 1), f32(0)]
        hi_ids, hi_v = ids[off[r]:off[r + 1]].astype(np.int64), vals[off[r]:off[r + 1]].astype(f32) + f32(0)
        keep = elig[r, hi_ids]
        hi_ids, hi_v = hi_ids[keep], hi_v[keep]
        for j, i in enumerate(np.lexsort((hi_ids, -hi_v.astype(f64)))):
            score.setdefault(int(hi_ids[i]), [f32(0), f32(0)])[1] = rrf_term(c, j + 1)
        cols = np.asarray(sorted(score), np.int64)
        s = np.asarray([f32(score[p][0] + score[p][1]) for p in cols], f32)
        o = order(s, cols)[:k]
        rows.append((s[o], cols[o] + id_offset))
    return _pad(rows, k, (f32, np.int64))


def gram32(D, ids):
    """sim(c_a, c_b) = dot32(D[c_a], D[c_b]) for the candidate ids (the first id < 0 ends them): [F', F'] fp32."""
    ids = np.asarray(ids, np.int64)
    bad = np.nonzero(ids < 0)[0]
    n = int(bad[0]) if bad.size else ids.size
    a, b = np.meshgrid(ids[:n], ids[:n], indexing="ij")
    return dot32(D[a.ravel()], D[b.ravel()]).reshape(n, n)
