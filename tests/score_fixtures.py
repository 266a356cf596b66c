"""Retrieval proof fixtures and a numpy emulation of the tensor-core filter + exact rescoring of csrc/score.cu.

The filter keeps, per (query, doc range), the 16 best APPROXIMATE scores (fp16 operands, fp32 accumulation); items of
later waves drop everything at or below the query's published threshold tau. The rescoring kernel keeps the best
`keep` candidates by approximate score, rescored in fp32, and certifies the top-k when

    max(list tails, best pruned head) + eps < k-th exact score,
    eps = (2^-10 + dim 2^-23) |q| max|d| + sqrt(dim) 2^-24 (|q| + max|d|) + 1e-6,

otherwise the query is flagged and answered by the fp32 scan. `emulate` follows that arithmetic; its `mut` argument
names one mutant (a plausible weakening of the proof) from MUTANTS.

The fixtures put the proof near its edge with CORRELATED fp16 rounding: every component of the query and of one
"true" document rounds the same way, so the true document's approximate score is low by almost the whole operand
term of eps. Decoys with exactly representable components (their approximate scores are exact) then push the true
document out of its list, and an exactly representable anchor in another doc range scores between the decoy list's
tail + a weakened eps and the true document's exact score. Accumulation is exact for all of them: every product is a
multiple of a power of two the fp32 partial sums still hold.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional

import numpy as np

KT = 16                 # candidates per list (SC_KT)
SC_BN = 256             # docs per tile
MAX_RANGES = 64
PAIRS = 66              # CTA pairs of a 132-SM H100 (the CPU emulation's default)

MUTANTS = ["eps halved", "operand term 2^-11", "round-toward-zero fp16", "no subnormal term",
           "bound from the last list only", "bound without the pruned heads"]


def plan(nq: int, nd: int, pairs: int = PAIRS) -> dict:
    """score_plan of csrc/score.cu."""
    QB = (nq + 255) // 256
    T = (nd + SC_BN - 1) // SC_BN
    best, R = 1e30, 1
    for r in range(1, min(MAX_RANGES, T) + 1):
        waves = (QB * r + pairs - 1) // pairs
        cost = waves * ((T + r - 1) // r + 0.5)
        if cost < best * 0.98:
            best, R = cost, r
    items = QB * R
    return dict(T=T, R=R, QB=QB, items=items, pairs=min(items, pairs), lists=2 * ((R + 2) // 2))


def range_docs(p: dict, nd: int, r: int):
    """Doc span [lo, hi) of doc range r."""
    return SC_BN * (p["T"] * r // p["R"]), min(nd, SC_BN * (p["T"] * (r + 1) // p["R"]))


def wave(p: dict, r: int, b: int) -> int:
    """Wave in which query block b sweeps doc range r (item r*QB + b runs on pair item % pairs)."""
    return (r * p["QB"] + b) // p["pairs"]


def to_f16(x: np.ndarray, rtz: bool = False) -> np.ndarray:
    """fp32 -> fp16, round to nearest even (numpy's conversion), or toward zero."""
    h = np.asarray(x, dtype=np.float32).astype(np.float16)
    if rtz:
        over = np.abs(h.astype(np.float64)) > np.abs(x.astype(np.float64))
        h = np.where(over, np.nextafter(h, np.float16(0)), h)
    return h


def eps_of(qn, dn, dim, mut: Optional[str] = None):
    """The rescoring kernel's eps, in fp32 (or a mutant's)."""
    f = np.float32
    op = f(2.0 ** -11) if mut == "operand term 2^-11" else f(9.765625e-4)
    e = (op + f(dim) * f(1.1920929e-7)) * f(qn) * f(dn)
    if mut != "no subnormal term":
        e = e + np.sqrt(f(dim)) * f(5.9604645e-8) * (f(qn) + f(dn))
    e = e + f(1e-6)
    return e * f(0.5) if mut == "eps halved" else e


def row_norms(x: np.ndarray) -> np.ndarray:
    return np.sqrt((x.astype(np.float64) ** 2).sum(1)).astype(np.float32)


def _scores(Q, D, cast):
    """cast(Q) @ cast(D).T in float64, over the distinct query rows only."""
    if (Q == Q[:1]).all():
        u, inv = Q[:1], np.zeros(len(Q), np.int64)
    else:
        u, inv = np.unique(Q, axis=0, return_inverse=True)
    s = cast(u).astype(np.float64) @ cast(D).astype(np.float64).T
    return s[inv.reshape(-1)]


def exact_scores(Q, D):
    """The fp32 dot products (rounded from float64: the fp32 scan's values up to summation order)."""
    return _scores(Q, D, lambda x: x).astype(np.float32)


def approx_scores(Q, D, rtz=False):
    """The filter's scores: fp16 operands, products summed exactly and rounded to fp32."""
    return _scores(Q, D, lambda x: to_f16(x, rtz)).astype(np.float32)


def topk_rows(s: np.ndarray, k: int):
    """(score desc, id asc) top-k of each row."""
    if k < s.shape[1] // 4:        # only the entries at or above the k-th largest can be in it
        kth = -np.partition(-s, k - 1, axis=1)[:, k - 1:k]
        cand = np.where(s >= kth, s, -np.inf)
        order = np.argsort(-cand, axis=1, kind="stable")[:, :k]
        return np.take_along_axis(s, order, 1), order.astype(np.int64)
    order = np.argsort(-s, axis=1, kind="stable")[:, :k]
    return np.take_along_axis(s, order, 1), order.astype(np.int64)


def filter_lists(approx: np.ndarray, p: dict):
    """Candidate lists [nq, lists, 16] (scores, ids) with the per-query threshold of the later waves: an item starts
    from the tails its query's items of EARLIER waves published (items of one wave do not see each other: the least
    a pair can rely on). The last slot's first score holds the final tau."""
    nq, nd = approx.shape
    L = p["lists"]
    cs = np.full((nq, L, KT), -np.inf, np.float32)
    ci = np.full((nq, L, KT), -1, np.int64)
    tau = np.full(nq, -np.inf, np.float32)
    for b in range(p["QB"]):
        rows = slice(256 * b, min(nq, 256 * b + 256))
        by_wave = {}
        for r in range(p["R"]):
            by_wave.setdefault(wave(p, r, b), []).append(r)
        for w in sorted(by_wave):
            start = tau[rows].copy()
            for r in by_wave[w]:
                lo, hi = range_docs(p, nd, r)
                s = approx[rows, lo:hi]
                s = np.where(s > start[:, None], s, -np.inf).astype(np.float32)
                o = np.argsort(-s, axis=1, kind="stable")[:, :KT]
                v = np.take_along_axis(s, o, 1)
                n = v.shape[1]
                cs[rows, r, :n] = v
                ci[rows, r, :n] = np.where(np.isinf(v), -1, o + lo)
                tail = cs[rows, r, KT - 1]
                tau[rows] = np.maximum(tau[rows], tail)
    cs[:, L - 1, 0] = tau
    return cs, ci


def rescore(cs, ci, exact, qn, dn, k, dim, p, mut=None):
    """rescore_topk_kernel: (scores [nq,k], ids [nq,k], flags [nq], bound [nq], eps [nq]). `exact` is [nq, nd]."""
    nq, L, _ = cs.shape
    keep = min(max(2 * k, 32), L * KT, 256)
    lane, j = np.arange(L) % 32, np.arange(L) // 32
    out_s = np.full((nq, k), -np.inf, np.float32)
    out_i = np.full((nq, k), -1, np.int64)
    flags = np.zeros(nq, np.int32)
    bounds = np.zeros(nq, np.float32)
    epss = np.zeros(nq, np.float32)
    for q in range(nq):
        l, pos = np.nonzero(ci[q] >= 0)
        sc = cs[q][l, pos]
        # head merge = global order by (approx desc, lane, slot, position)
        order = np.lexsort((pos, j[l], lane[l], -sc))
        kept = ci[q][l, pos][order[:keep]]
        rem = sc[order[keep:]].max() if len(order) > keep else -np.inf
        if mut == "bound from the last list only":
            tail = cs[q, p["R"] - 1, KT - 1]
        else:
            tail = cs[q, :, KT - 1].max()
        bound = np.float32(tail if mut == "bound without the pruned heads" else max(tail, rem))
        ex = exact[q, kept]
        o = np.lexsort((kept, -ex))[:k]
        n = len(o)
        out_s[q, :n], out_i[q, :n] = ex[o], kept[o]
        kth = out_s[q, k - 1]
        e = eps_of(qn[q], dn, dim, mut)
        flag = bound > -np.inf and not (bound + e < kth)
        flag = flag or not (qn[q] < 65504) or not (dn < 65504)
        flags[q], bounds[q], epss[q] = flag, bound, e
    return out_s, out_i, flags, bounds, epss


def emulate(Q, D, k, mut=None, pairs=PAIRS):
    """The whole filter path on the CPU: (scores, ids, flags, info). Flagged queries take the fp32 scan's answer."""
    nq, dim = Q.shape
    p = plan(nq, D.shape[0], pairs)
    exact = exact_scores(Q, D)
    approx = approx_scores(Q, D, rtz=mut == "round-toward-zero fp16")
    cs, ci = filter_lists(approx, p)
    s, i, flags, bound, eps = rescore(cs, ci, exact, row_norms(Q), row_norms(D).max(), k, dim, p, mut)
    ref_s, ref_i = topk_rows(exact, k)
    bad = flags.astype(bool)
    s[bad], i[bad] = ref_s[bad], ref_i[bad]
    return s, i, flags, dict(plan=p, cs=cs, ci=ci, bound=bound, eps=eps, exact=exact, approx=approx, ref=(ref_s, ref_i))


# ------------------------------------------------------------------------------------------------------------ fixtures


@dataclass
class Fixture:
    name: str
    Q: np.ndarray        # [nq, dim] fp32, every row the same query
    D: np.ndarray        # [nd, dim] fp32
    k: int
    true_doc: int        # the exact top-1
    dropped: bool        # the true document falls out of its list (round to nearest)
    note: str            # what the fixture is built to catch


def _up(v):
    """The next fp16 value above v, as float64."""
    return float(np.nextafter(np.float16(v), np.float16(np.inf)))


def _rep(base, n_up, dim, rs):
    """A doc row of exactly representable components: `base` everywhere, one fp16 step above it at n_up places."""
    x = np.full(dim, base, np.float64)
    x[rs.choice(dim, n_up, replace=False)] = _up(base)
    return x


def _eps64(qn, dn, dim):
    return (2.0 ** -10 + dim * 2.0 ** -23) * qn * dn + np.sqrt(dim) * 2.0 ** -24 * (qn + dn) + 1e-6


def correlated(name, q_c, t_c, *, anchor_frac=None, rtz_tail=False, spread=False, nq=600, nd=8192, dim=2304, k=1,
               seed=0, note=""):
    """Query of constant components q_c, true document of constant components t_c at doc 1797 (tile 7); decoys of
    exactly representable components whose approximate scores beat the true document's.
    spread=False: 20 decoys in the true document's tile, so its list holds 16 decoys and drops it.
    spread=True: 33 decoys, 3 in each of 11 other doc ranges, so the true document stays in its list but is pruned
    by the head merge (keep = 32): only the best pruned head bounds it.
    anchor_frac: an anchor doc in tile 20 whose exact score is the decoy list's tail + anchor_frac * eps (tail taken
    with round-toward-zero copies if rtz_tail)."""
    rs = np.random.RandomState(seed)
    t16 = float(to_f16(np.float32(t_c), rtz_tail))
    q16 = float(to_f16(np.float32(q_c), rtz_tail))
    step = _up(t16) - t16
    D = t16 * np.where(rs.rand(nd, dim) < 0.5, -1.0, 1.0)    # filler: components +-t16, scores near 0
    true_doc = 7 * SC_BN + 5
    D[true_doc] = t_c
    n_true = dim * (np.float32(t_c) - t16) / step     # the true doc's exact sum, in steps above dim * t16
    if spread:
        p = plan(nq, nd)
        assert p["R"] >= 13, p
        decoys = []
        for r in range(1, 12):
            lo, hi = range_docs(p, nd, r + (r >= 3))  # skip the true document's range (range 3 at R = 16)
            decoys += [lo + 9, lo + 60, lo + 200]
    else:
        decoys = list(range(true_doc + 1, true_doc + 21))
    for n, d in enumerate(decoys, 1):
        D[d] = _rep(t16, n, dim, rs)
    assert len(decoys) < n_true
    qn, dn = np.sqrt(dim) * q_c, np.sqrt(dim) * t_c
    if anchor_frac is not None:
        tail = q16 * (dim * t16 + (len(decoys) - KT + 1) * step)    # approximate score of the list's 16th decoy
        target = tail + anchor_frac * _eps64(qn, dn, dim)
        n_a = int(np.ceil((target / np.float32(q_c) - dim * t16) / step))
        assert len(decoys) < n_a < n_true and n_a <= dim, (n_a, n_true)
        D[20 * SC_BN + 11] = _rep(t16, n_a, dim, rs)
    Q = np.full((nq, dim), q_c, np.float32)
    D = D.astype(np.float32)
    return Fixture(name, Q, D, k, true_doc, not spread and not rtz_tail, note)


FIXTURES = ["fp16 rounds down 0.49 ulp", "pruned head", "fp16 subnormal query",
            "rounds up 0.01 ulp (toward zero: down 0.99)"]


def fixtures():
    """The proof fixtures (dim 2304, 600 identical queries over 8192 docs: the filter path, R = 16 doc ranges)."""
    h = 2.0 ** -16
    yield correlated("fp16 rounds down 0.49 ulp", 2.0 ** -6 + 0.49 * h, 2.0 ** -6 + 0.49 * h, anchor_frac=0.70, seed=1,
                     note="eps halved, operand term 2^-11, bound from the last list only")
    yield correlated("pruned head", 2.0 ** -6 + 0.49 * h, 2.0 ** -6 + 0.49 * h, spread=True, seed=2,
                     note="bound without the pruned heads")
    yield correlated("fp16 subnormal query", 2.0 ** -18 + 0.49 * 2.0 ** -24, 1364 * 2.0 ** -12 + 0.49 * 2.0 ** -12,
                     seed=3, note="no subnormal term")
    yield correlated("rounds up 0.01 ulp (toward zero: down 0.99)", 2.0 ** -6 + 0.99 * h, 2.0 ** -6 + 0.99 * h,
                     anchor_frac=1.25, rtz_tail=True, seed=4, note="round-toward-zero fp16")


def closeness(fx: Fixture):
    """(true doc's exact - approximate score) / eps, and (exact - its list's tail) / eps, for the printouts."""
    q = fx.Q[:1]
    ex = exact_scores(q, fx.D[[fx.true_doc]])[0, 0]
    ap = approx_scores(q, fx.D[[fx.true_doc]])[0, 0]
    eps = eps_of(row_norms(q)[0], row_norms(fx.D).max(), fx.Q.shape[1])
    return float((ex - ap) / eps), float(eps)


# ---------------------------------------------------------------------------------------------------- masked filters


def masked_filter_lists(approx, mask, p, tau_from_unmasked=False):
    """filter_lists with the kernel's masking: ineligible scores are -inf before the threshold test and the insertion,
    so lists and tau see eligible docs only. tau_from_unmasked: the mutant that publishes tau from the unmasked lists."""
    nq, nd = approx.shape
    masked = np.where(mask[None, :], approx, -np.inf).astype(np.float32)
    cs = np.full((nq, p["lists"], KT), -np.inf, np.float32)
    ci = np.full((nq, p["lists"], KT), -1, np.int64)
    tau = np.full(nq, -np.inf, np.float32)
    for b in range(p["QB"]):
        rows = slice(256 * b, min(nq, 256 * b + 256))
        by_wave = {}
        for r in range(p["R"]):
            by_wave.setdefault(wave(p, r, b), []).append(r)
        for w in sorted(by_wave):
            start = tau[rows].copy()
            for r in by_wave[w]:
                lo, hi = range_docs(p, nd, r)
                tails = []
                for src in (masked, approx) if tau_from_unmasked else (masked,):
                    s = np.where(src[rows, lo:hi] > start[:, None], src[rows, lo:hi], -np.inf).astype(np.float32)
                    o = np.argsort(-s, axis=1, kind="stable")[:, :KT]
                    v = np.take_along_axis(s, o, 1)
                    if src is masked:
                        cs[rows, r, :v.shape[1]] = v
                        ci[rows, r, :v.shape[1]] = np.where(np.isinf(v), -1, o + lo)
                    tails.append(v[:, KT - 1] if v.shape[1] == KT else np.full(v.shape[0], -np.inf, np.float32))
                tau[rows] = np.maximum(tau[rows], tails[-1])
    cs[:, -1, 0] = tau
    return cs, ci


def filter_lists_per_query(approx, elig, p, leak=False):
    """filter_lists with a mask per query row (elig [nq, nd]): ineligible scores are -inf before the threshold test and
    the insertion. leak: the mutant that publishes the tail of the thread's other accumulator row (row ^ 8 of the block)
    as this row's tau."""
    nq, nd = approx.shape
    masked = np.where(elig, approx, -np.inf).astype(np.float32)
    cs = np.full((nq, p["lists"], KT), -np.inf, np.float32)
    ci = np.full((nq, p["lists"], KT), -1, np.int64)
    tau = np.full(nq, -np.inf, np.float32)
    for b in range(p["QB"]):
        rows = slice(256 * b, min(nq, 256 * b + 256))
        n = rows.stop - rows.start
        by_wave = {}
        for r in range(p["R"]):
            by_wave.setdefault(wave(p, r, b), []).append(r)
        for w in sorted(by_wave):
            start = tau[rows].copy()
            for r in by_wave[w]:
                lo, hi = range_docs(p, nd, r)
                s = np.where(masked[rows, lo:hi] > start[:, None], masked[rows, lo:hi], -np.inf).astype(np.float32)
                o = np.argsort(-s, axis=1, kind="stable")[:, :KT]
                v = np.take_along_axis(s, o, 1)
                cs[rows, r, :v.shape[1]] = v
                ci[rows, r, :v.shape[1]] = np.where(np.isinf(v), -1, o + lo)
                tail = v[:, KT - 1] if v.shape[1] == KT else np.full(n, -np.inf, np.float32)
                if leak:
                    tail = tail[np.minimum(np.arange(n) ^ 8, n - 1)]
                tau[rows] = np.maximum(tau[rows], tail)
    cs[:, -1, 0] = tau
    return cs, ci


def reference_per_query(exact, elig, k):
    """Each query's fp32 scan over its own eligible docs: (score desc, id asc), then (-inf, -1)."""
    s = np.where(elig, exact, -np.inf).astype(np.float32)
    order = np.lexsort((np.broadcast_to(np.arange(s.shape[1]), s.shape), -s), axis=1)[:, :k]
    out_s = np.take_along_axis(s, order, 1)
    out_i = np.where(np.isinf(out_s) & (out_s < 0), -1, order)
    return out_s, out_i.astype(np.int64)


# ---------------------------------------------------------------------------------------------------- documents


BUDGET = 4096  # RG_PAGE_BUDGET of csrc/score.cu


def grouped_reference(exact, groups, k, mask=None):
    """The contract: walk the eligible pages in (score desc, page asc) order, keep the first page of each group."""
    nq, nd = exact.shape
    cols = np.arange(nd) if mask is None else np.nonzero(mask)[0]
    out_s = np.full((nq, k), -np.inf, np.float32)
    out_p = np.full((nq, k), -1, np.int64)
    out_g = np.full((nq, k), -1, np.int64)
    for r in range(nq):
        order = cols[np.lexsort((cols, -exact[r, cols]))]
        _, first = np.unique(groups[order], return_index=True)
        pick = order[np.sort(first)][:k]
        out_s[r, :len(pick)], out_p[r, :len(pick)], out_g[r, :len(pick)] = exact[r, pick], pick, groups[pick]
    return out_s, out_p, out_g


def grouped_filter_lists(approx, groups, p, elig=None):
    """filter_lists with group-distinct lists: each (query, doc range) list holds the 16 best groups of the range by
    their best approximate page above the starting threshold, one entry (that page) per group. elig [nq, nd] (optional):
    only the eligible pages of each query enter its lists."""
    nq, nd = approx.shape
    L_ = p["lists"]
    cs = np.full((nq, L_, KT), -np.inf, np.float32)
    ci = np.full((nq, L_, KT), -1, np.int64)
    tau = np.full(nq, -np.inf, np.float32)
    for b in range(p["QB"]):
        rows = range(256 * b, min(nq, 256 * b + 256))
        by_wave = {}
        for r in range(p["R"]):
            by_wave.setdefault(wave(p, r, b), []).append(r)
        for w in sorted(by_wave):
            start = tau.copy()
            for r in by_wave[w]:
                lo, hi = range_docs(p, nd, r)
                for q in rows:
                    s = approx[q, lo:hi]
                    above = s > start[q]
                    if elig is not None:
                        above &= elig[q, lo:hi]
                    cand = np.nonzero(above)[0]
                    order = cand[np.lexsort((cand, -s[cand]))]
                    _, first = np.unique(groups[lo + order], return_index=True)
                    pick = order[np.sort(first)][:KT]
                    cs[q, r, :len(pick)] = s[pick]
                    ci[q, r, :len(pick)] = pick + lo
                    tau[q] = max(tau[q], cs[q, r, KT - 1])
    cs[:, L_ - 1, 0] = tau
    return cs, ci


def grouped_rescore(cs, ci, exact, groups, qn, dn, k, dim, budget=BUDGET, mut=None, elig=None):
    """rescore_groups_kernel: (scores, pages, groups, flags). mut: 'entry score' takes a group's score from its kept
    entries without full rescoring; 'B without unrescored groups' leaves their approximate entries out of the bound.
    elig [nq, nd] (optional): a rescored group's ineligible pages are not scored (they still count against the budget),
    and a group without an eligible page is no result."""
    nq, L_, _ = cs.shape
    keep = min(max(2 * k, 32), L_ * KT, 256)
    lane, j = np.arange(L_) % 32, np.arange(L_) // 32
    sizes = np.bincount(groups)
    out_s = np.full((nq, k), -np.inf, np.float32)
    out_p = np.full((nq, k), -1, np.int64)
    out_g = np.full((nq, k), -1, np.int64)
    flags = np.zeros(nq, np.int32)
    for q in range(nq):
        l, pos = np.nonzero(ci[q] >= 0)
        sc = cs[q][l, pos]
        order = np.lexsort((pos, j[l], lane[l], -sc))
        kept, kept_s = ci[q][l, pos][order[:keep]], sc[order[:keep]]
        rem = sc[order[keep:]].max() if len(order) > keep else -np.inf
        bound = max(cs[q, :, KT - 1].max(), rem)
        done, seen, total, full = [], set(), 0, False
        for c in range(len(kept)):                    # distinct groups of the kept candidates, in approximate order
            g = groups[kept[c]]
            if g in seen:
                continue
            seen.add(g)
            if not full and sizes[g] <= budget - total:
                done.append(g)
                total += sizes[g]
            else:                                     # the first group that does not fit ends the walk
                full = True
                if mut != "B without unrescored groups":
                    bound = max(bound, kept_s[c])
        res = []
        for g in done:
            pages = kept[groups[kept] == g] if mut == "entry score" else np.nonzero(groups == g)[0]
            if elig is not None:
                pages = pages[elig[q, pages]]
                if len(pages) == 0:
                    continue
            s = exact[q, pages]
            b = pages[np.lexsort((pages, -s))][0]
            res.append((exact[q, b], b, g))
        res.sort(key=lambda x: (-x[0], x[1]))
        res = res[:k]
        for i, (s, b, g) in enumerate(res):
            out_s[q, i], out_p[q, i], out_g[q, i] = s, b, g
        kth = out_s[q, k - 1]
        e = eps_of(qn[q], dn, dim)
        flags[q] = (bound > -np.inf and not (bound + e < kth)) or not (qn[q] < 65504) or not (dn < 65504)
    return out_s, out_p, out_g, flags


def emulate_grouped(Q, D, groups, k, pairs=PAIRS, page_lists=False, budget=BUDGET, mut=None):
    nq, dim = Q.shape
    p = plan(nq, D.shape[0], pairs)
    exact, approx = exact_scores(Q, D), approx_scores(Q, D)
    cs, ci = filter_lists(approx, p) if page_lists else grouped_filter_lists(approx, groups, p)
    s, pg, g, flags = grouped_rescore(cs, ci, exact, groups, row_norms(Q), row_norms(D).max(), k, dim, budget, mut)
    ref = grouped_reference(exact, groups, k)
    bad = flags.astype(bool)
    s[bad], pg[bad], g[bad] = ref[0][bad], ref[1][bad], ref[2][bad]
    return (s, pg, g), flags, dict(plan=p, cs=cs, ci=ci, ref=ref)


def _true_with_decoys(fx):
    """The true document and the 20 decoys next to it form one group; every other page is its own group."""
    groups = np.arange(fx.D.shape[0])
    groups[fx.true_doc:fx.true_doc + 21] = fx.true_doc
    _, groups = np.unique(groups, return_inverse=True)
    return groups


def _budget_fixture():
    """One query over 8192 pages at dim 2304 with correlated fp16 rounding (as correlated): the true page T
    has the highest exact score, but a decoy Y of exactly representable components beats it in approximate score by
    less than eps. Y is a group of its own; T shares its group with 4097 low pages, more than the page budget. The walk
    rescores Y's group and stops at T's: only T's approximate entry in the bound keeps the proof from certifying Y."""
    rs = np.random.RandomState(31)
    nd, dim = 8192, 2304
    c = 2.0 ** -6 + 0.49 * 2.0 ** -16
    t16 = float(to_f16(np.float32(c)))
    D = t16 * np.where(rs.rand(nd, dim) < 0.5, -1.0, 1.0)
    T, Y = 7 * SC_BN + 5, 20 * SC_BN + 11
    D[T] = c
    D[Y] = _rep(t16, 2, dim, rs)
    groups = np.arange(nd) + 1
    groups[T] = 0
    groups[np.setdiff1d(np.arange(nd), [T, Y])[:BUDGET + 1]] = 0
    _, groups = np.unique(groups, return_inverse=True)
    return np.full((1, dim), c, np.float32), D.astype(np.float32), groups, T, Y


# ---------------------------------------------------------------------------------------------------- range


def fsub_rd(a, b):
    """a - b in fp32, rounded toward -inf (__fsub_rd)."""
    a, b = np.float32(a), np.float32(b)
    exact = float(a) - float(b)                    # exact in float64 for these magnitudes
    r = np.float32(exact)
    return np.nextafter(r, np.float32(-np.inf)) if float(r) > exact else r


def range_model(approx, exact, t, eps, sub=fsub_rd):
    """The threshold filter and the rescoring on one query row: candidates are the docs with approximate score >= the
    drop threshold, results the candidates with exact score >= t."""
    thr = sub(t, eps)
    cand = np.nonzero(approx >= thr)[0]
    return set(cand[exact[cand] >= t].tolist())
