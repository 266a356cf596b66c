"""The retrieval reference of tests/dot_reference.py, proved on the CPU: its FMA against exact rational rounding, its dot
product against the documented order run in exact arithmetic and against the error bound its screen relies on, the
screen against the unscreened answer on near-ties, and a mutant for each plausible mistake, each rejected on a fixture of
its own (the mutants stand for kernels with that fault: the GPU comparison would reject them the same way)."""
from fractions import Fraction

import numpy as np
import pytest

from tests import dot_reference as X

f32, f64 = np.float32, np.float64


# ------------------------------------------------------------------------------------------------ exact arithmetic
def round32(v: Fraction) -> f32:
    """v correctly rounded to fp32 (ties to even); |v| stays below the overflow threshold here."""
    f = f32(float(v))  # float(Fraction) rounds correctly to float64; the fp32 answer is f or a neighbour of it
    cands = [np.nextafter(f, f32(-np.inf)), f, np.nextafter(f, f32(np.inf))]
    best = min(cands, key=lambda x: (abs(Fraction(float(x)) - v), int(np.array(x).view(np.int32)) & 1))
    if best == 0 and v < 0:
        return f32(-0.0)
    return best


def fma_exact(a, b, c):
    if a * b == 0 and c == 0:  # the signed-zero rules of IEEE 754 for an exact zero result
        return f32(np.float32(a) * np.float32(b) + np.float32(c))
    return round32(Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c)))


def add_exact(a, b):
    if a == 0 and b == 0:
        return f32(a) + f32(b)
    return round32(Fraction(float(a)) + Fraction(float(b)))


def dot_exact_order(q, d):
    """The documented order with every operation rounded exactly: lanes, x y z w FMAs, the xor butterfly, lane 0."""
    nv = q.size // 4
    acc = [f32(0)] * 32
    for i in range(nv):
        for c in range(4):
            acc[i % 32] = fma_exact(d[4 * i + c], q[4 * i + c], acc[i % 32])
    for o in (16, 8, 4, 2, 1):
        acc = [add_exact(acc[l], acc[l ^ o]) for l in range(32)]
    return acc[0]


def dot_real(q, d):
    return sum(Fraction(float(x)) * Fraction(float(y)) for x, y in zip(q, d))


# ------------------------------------------------------------------------------------------------ fixtures
def midpoint_triples(rs, n):
    """(a, b, c) with a b + c = (an fp32 midpoint) - 2^-2u, scaled by powers of two: c = (2^24 + 2j) 2^e with j odd (odd
    last bit), a b = (1 + 2^-u)(1 - 2^-u) 2^e. The exact result lies just below the midpoint between c and the next
    fp32 up, so it rounds to c; float64 rounds it to the midpoint itself (2^-2u is below its half ulp), and the second
    rounding goes to the even neighbour, c + 2^(e+1)."""
    a, b, c = [], [], []
    for _ in range(n):
        u = rs.randint(15, 24)
        j = 2 * rs.randint(0, 1 << 21) + 1
        e, ea = rs.randint(-60, 40), rs.randint(-20, 20)
        s = rs.choice([-1.0, 1.0])
        a.append(s * (1 + 2.0 ** -u) * 2.0 ** ea)
        b.append((1 - 2.0 ** -u) * 2.0 ** (e - ea))
        c.append(s * (2.0 ** 24 + 2 * j) * 2.0 ** e)
    return (np.asarray(v, f32) for v in (a, b, c))


def adversarial_pairs(rs, dim, kind, n=4):
    """n pairs of fp32 rows of one kind: cancel (q.d = 0 exactly against a large sum |q_i d_i|, and near it), mixed
    (elements over 1e-3 .. 1e3), subnormal (every product below the fp32 normal range), plain (Gaussian)."""
    q = rs.randn(n, dim)
    d = rs.randn(n, dim)
    if kind == "cancel":
        h = dim // 2 // 4 * 4
        q[:, h:2 * h], d[:, h:2 * h] = -q[:, :h], d[:, :h]
        q[:, 2 * h:] = 0
        q[1:, 0] += 1e-3 * rs.randn(n - 1)  # near cancellation
        q *= 1e3
    elif kind == "mixed":
        q *= 10.0 ** rs.uniform(-3, 3, q.shape)
        d *= 10.0 ** rs.uniform(-3, 3, d.shape)
    elif kind == "subnormal":
        q *= 1e-21
        d *= 1e-22
    return q.astype(f32), d.astype(f32)


# ------------------------------------------------------------------------------------------------ fma32
def test_fma32_rounds_once_on_random_triples():
    rs = np.random.RandomState(0)
    n = 3000
    a = (rs.randn(n) * 10.0 ** rs.uniform(-5, 5, n)).astype(f32)
    b = (rs.randn(n) * 10.0 ** rs.uniform(-5, 5, n)).astype(f32)
    c = np.concatenate([(rs.randn(n // 2) * 10.0 ** rs.uniform(-5, 5, n // 2)).astype(f32),
                        -(a[n // 2:].astype(f64) * b[n // 2:]).astype(f32)])  # near-cancelling half
    got = X.fma32(a, b, c)
    want = np.asarray([fma_exact(*t) for t in zip(a, b, c)], f32)
    assert np.array_equal(got.view(np.int32), want.view(np.int32))


def test_fma32_on_midpoints_where_double_rounding_fails():
    a, b, c = midpoint_triples(np.random.RandomState(1), 500)
    want = np.asarray([fma_exact(*t) for t in zip(a, b, c)], f32)
    assert np.array_equal(want, c)  # the fixture: the exact result rounds back to c
    assert np.array_equal(X.fma32(a, b, c).view(np.int32), want.view(np.int32))
    naive = (a.astype(f64) * b + c).astype(f32)
    assert (naive != want).all()


def test_fma32_signed_zeros_subnormals_and_non_finite():
    a = np.asarray([-1e-30, 1e-30, 0.0, np.inf, np.inf, np.nan, 3e38, 1e-20, -0.0], f32)
    b = np.asarray([1e-30, 1e-30, -1.0, 0.0, 1.0, 1.0, 10.0, 1e-25, 1.0], f32)
    c = np.asarray([0.0, -0.0, 0.0, 1.0, -np.inf, 0.0, 0.0, 1e-44, -0.0], f32)
    got = X.fma32(a, b, c)
    want = np.asarray([-0.0, 0.0, 0.0, np.nan, np.nan, np.nan, np.inf, f32(1e-44) + f32(1e-45), -0.0], f32)
    num = ~np.isnan(want)
    assert np.array_equal(got, want, equal_nan=True) and np.array_equal(np.signbit(got[num]), np.signbit(want[num]))


# ------------------------------------------------------------------------------------------------ dot32
@pytest.mark.parametrize("dim", [4, 12, 124, 132])
def test_dot32_is_the_documented_order_rounded_exactly(dim):
    rs = np.random.RandomState(dim)
    for kind in ("plain", "cancel", "mixed", "subnormal"):
        q, d = adversarial_pairs(rs, dim, kind, n=3)
        got = X.dot32(q, d)
        want = np.asarray([dot_exact_order(a, b) for a, b in zip(q, d)], f32)
        assert np.array_equal(got.view(np.int32), want.view(np.int32)), kind


@pytest.mark.parametrize("dim", [4, 12, 124, 132, 2308])
@pytest.mark.parametrize("kind", ["plain", "cancel", "mixed", "subnormal"])
def test_dot32_within_its_bound(dim, kind):
    rs = np.random.RandomState(dim + len(kind))
    q, d = adversarial_pairs(rs, dim, kind)
    got = X.dot32(q, d)
    for p in range(q.shape[0]):
        exact = dot_real(q[p], d[p])
        A = sum(abs(Fraction(float(x)) * Fraction(float(y))) for x, y in zip(q[p], d[p]))
        err = abs(Fraction(float(got[p])) - exact)
        assert err <= Fraction(X.dot_bound(float(A), dim)), (kind, p, float(err))
        assert err <= Fraction(X.width(float(A), dim))


def test_dot32_gives_minus_zero_only_when_every_lane_does():
    q = np.full((2, 128), 1e-30, f32)
    d = np.full((2, 128), -1e-30, f32)
    d[1, :4] = 1e-30  # lane 0 underflows positive: +0, and +0 + -0 = +0
    got = X.dot32(q, d)
    assert got[0] == 0 and np.signbit(got[0]) and got[1] == 0 and not np.signbit(got[1])
    assert not np.signbit(X.dot32(q[:, :124], d[:, :124])[0])  # a lane without a float4 holds +0


# ------------------------------------------------------------------------------------------------ the dot mutants
def _mutant_dot(name, q, d):
    if name == "np.dot in fp32":
        return np.asarray([np.dot(a, b) for a, b in zip(q, d)], f32)
    if name == "one sequential accumulator":
        out = []
        for a, b in zip(q, d):
            acc = np.zeros(1, f32)
            for x, y in zip(b, a):
                acc = X.fma32(np.asarray([x]), np.asarray([y]), acc)
            out.append(acc[0])
        return np.asarray(out, f32)
    if name == "lanes summed 0..31 in sequence":
        acc = X.lane_sums(q, d)
        s = acc[:, 0].copy()
        for l in range(1, 32):
            s = s + acc[:, l]
        return s
    if name == "mul + add":
        return X.butterfly(X.lane_sums(q, d, fma=lambda a, b, c: (np.asarray(a, f32) * np.asarray(b, f32)) + c))
    if name == "double-rounded fma":
        return X.butterfly(X.lane_sums(q, d, fma=lambda a, b, c: (np.asarray(a, f64) * b + c).astype(f32)))
    raise KeyError(name)


def _midpoint_rows(rs, n):
    """dim-4 rows whose second FMA is a midpoint triple: q = (c, a, 0, 0), d = (1, b, 0, 0)."""
    a, b, c = midpoint_triples(rs, n)
    q = np.zeros((n, 4), f32)
    d = np.zeros((n, 4), f32)
    q[:, 0], q[:, 1], d[:, 0], d[:, 1] = c, a, 1, b
    return q, d


DOT_MUTANTS = {
    "np.dot in fp32": lambda rs: adversarial_pairs(rs, 2308, "mixed", n=6),
    "one sequential accumulator": lambda rs: adversarial_pairs(rs, 132, "plain", n=6),
    "lanes summed 0..31 in sequence": lambda rs: adversarial_pairs(rs, 128, "mixed", n=6),
    "mul + add": lambda rs: adversarial_pairs(rs, 12, "mixed", n=6),
    "double-rounded fma": lambda rs: _midpoint_rows(rs, 6),
}


@pytest.mark.parametrize("name", sorted(DOT_MUTANTS))
def test_dot_mutant_is_rejected(name):
    q, d = DOT_MUTANTS[name](np.random.RandomState(7))
    want = np.asarray([dot_exact_order(a, b) for a, b in zip(q, d)], f32)
    assert np.array_equal(X.dot32(q, d).view(np.int32), want.view(np.int32))
    bad = _mutant_dot(name, q, d)
    assert not np.array_equal(bad.view(np.int32), want.view(np.int32)), f"mutant {name!r} survived its fixture"


# ------------------------------------------------------------------------------------------------ ordering mutants
def _order_ties_high(s, ids):
    at = np.nonzero(~np.isnan(s))[0]
    return at[np.lexsort((-np.asarray(ids)[at], -s[at].astype(f64) + 0.0))]


def _order_minus_zero_low(s, ids):
    at = np.nonzero(~np.isnan(s))[0]
    return at[np.lexsort((np.asarray(ids)[at], np.signbit(s[at]), -s[at].astype(f64) + 0.0))]


def _order_nan_first(s, ids):
    key = np.where(np.isnan(s), -np.inf, -s.astype(f64) + 0.0)
    return np.lexsort((np.asarray(ids), key))


ORDER_MUTANTS = {
    # name: (mutant, scores, ids, the reference order)
    "ties to the higher id": (_order_ties_high, [0.5, 0.25, 0.5], [7, 1, 3], [2, 0, 1]),
    "-0 ranked below +0": (_order_minus_zero_low, [-0.0, 0.0, -1.0], [2, 5, 0], [0, 1, 2]),
    "NaN selected first": (_order_nan_first, [1.0, np.nan, -np.inf], [0, 1, 2], [0, 2]),
}


@pytest.mark.parametrize("name", sorted(ORDER_MUTANTS))
def test_order_mutant_is_rejected(name):
    fn, s, ids, want = ORDER_MUTANTS[name]
    s = np.asarray(s, f32)
    assert X.order(s, ids).tolist() == want
    assert fn(s, ids).tolist() != want, f"mutant {name!r} survived its fixture"


def test_topk_ties_minus_zero_and_nan_end_to_end():
    """The same rules through Exact and topk: dim 128, so that every lane of the -0 rows underflows negative."""
    Q = np.full((1, 128), 1e-30, f32)
    D = np.zeros((6, 128), f32)
    D[0] = -1e-30                  # -0
    D[1] = 0.0                     # +0
    D[2] = 1e-30                   # +0 (underflow, positive)
    D[3, 0] = np.nan               # NaN
    D[4] = -1.0                    # negative
    D[5, 0] = np.inf               # +inf
    s, i = X.topk(X.Exact(Q, D), 6, id_offset=10)
    assert i.tolist() == [[15, 10, 11, 12, 14, -1]]
    assert np.signbit(s[0, 1]) and not np.signbit(s[0, 2]) and s[0, 5] == -np.inf


# ------------------------------------------------------------------------------------------------ the screen
def test_screen_mutant_testing_lo_is_rejected():
    """Page 1's fp32 score (2.0) exceeds its float64 score (1.5) by a rounding that its wide bracket allows; page 0
    scores 1.75 exactly with a narrow bracket. The top-1 is page 1: only a screen on hi keeps it."""
    Q = np.asarray([[1.0, 1.0, 1.0, 0.0]], f32)
    D = np.asarray([[1.75, 0, 0, 0], [2.0 ** 24, 1.5, -(2.0 ** 24), 0]], f32)
    ex = X.Exact(Q, D)
    s, i = X.topk(ex, 1)
    assert i.tolist() == [[1]] and s[0, 0] == 2.0
    Lk = X.kth_largest(ex.lo, 1)
    assert (ex.lo >= Lk[:, None]).tolist() == [[True, False]]  # the mutant's candidates miss page 1
    assert X.screen_topk(ex.lo, ex.hi, np.ones((1, 2), bool), 1).tolist() == [[True, True]]


def near_tie_problem(seed, nq=5, nd=600, dim=132, dup=True):
    """Rows with many exact duplicates and one-ulp nudges of one another, mixed norms, and documents of 1 .. 9 pages."""
    rs = np.random.RandomState(seed)
    base = rs.randn(nd // 6, dim).astype(f32)
    D = base[rs.randint(0, base.shape[0], nd)]
    nudge = rs.rand(nd) < 0.5
    col = rs.randint(0, dim, nd)
    D[nudge, col[nudge]] = np.nextafter(D[nudge, col[nudge]], f32(np.inf))
    D *= np.where(rs.rand(nd) < 0.2, f32(1e3), f32(1))[:, None]
    Q = base[rs.randint(0, base.shape[0], nq)].copy()
    Q[0] *= f32(1e-3)
    groups = np.repeat(np.arange(nd), rs.randint(1, 10, nd))[:nd]
    return Q, D, groups


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_screened_answers_equal_full_dot32(seed):
    Q, D, groups = near_tie_problem(seed)
    nq, nd = Q.shape[0], D.shape[0]
    rs = np.random.RandomState(seed + 10)
    elig = rs.rand(nq, nd) < 0.8
    off = np.r_[0, np.cumsum(rs.randint(0, 30, nq))]
    ids = np.concatenate([rs.choice(nd, off[r + 1] - off[r], replace=False) for r in range(nq)])
    vals = (rs.rand(ids.size) * 50).astype(f32)
    hits = (off, ids, vals)
    t = np.asarray([X.topk(X.Exact(Q, D), 40)[0][r, 39] for r in range(nq)], f32)
    ex, full = X.Exact(Q, D), X.Exact(Q, D, screen=False)
    cases = [
        (X.topk, (1,)), (X.topk, (33,)), (X.topk, (300,)),
        (X.topk_groups, (17, groups)), (X.topk_capped, (20, groups, 2)), (X.topk_groups_pages, (9, groups, 3)),
        (X.range_pages, (t,)), (X.range_groups, (t, groups)),
        (X.hybrid_sum, (16, hits, 0.01)), (X.hybrid_groups, (16, groups, hits, 0.01)), (X.hybrid_rrf, (16, hits, 50, 60)),
    ]
    for fn, args in cases:
        for e in (None, elig):
            a, b = fn(ex, *args, elig=e), fn(full, *args, elig=e)
            for x, y in zip(a, b):
                assert np.array_equal(x, y) and (x.dtype != f32 or np.array_equal(x.view(np.int32), y.view(np.int32))), fn.__name__
    assert ex.scored < full.scored  # the screen did screen


def test_capped_walk_and_documents_by_hand():
    """Scores 5 4 3 2 1 on pages 0..4 of documents 0 0 0 1 1 (dim 4, exact)."""
    Q = np.asarray([[1, 0, 0, 0]], f32)
    D = np.zeros((5, 4), f32)
    D[:, 0] = [5, 4, 3, 2, 1]
    groups = np.asarray([0, 0, 0, 1, 1])
    ex = X.Exact(Q, D)
    assert X.topk_capped(ex, 4, groups, 2)[1].tolist() == [[0, 1, 3, 4]]
    assert X.topk_groups(ex, 3, groups)[1].tolist() == [[0, 3, -1]]
    off, s, p, g = X.range_groups(ex, np.asarray([1.5], f32), groups)
    assert off.tolist() == [0, 2] and p.tolist() == [0, 3] and g.tolist() == [0, 1]
    hits = (np.asarray([0, 1]), np.asarray([4]), np.asarray([10.0], f32))
    assert X.hybrid_sum(ex, 2, hits, 1.0)[1].tolist() == [[4, 0]]
    s, i = X.hybrid_rrf(ex, 3, hits, 2, 0)
    assert s.tolist() == [[1.0, 1.0, 0.5]] and i.tolist() == [[0, 4, 1]]
