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
