"""Deep top-k on the CPU (DESIGN §4, "Deep top-k"): a numpy model of the radix select of vr_select_rows against a full
sort, and a model of score_topk's deep route (sampled threshold, range answer when kept >= k, scan otherwise) with the
mutants it must reject."""
import numpy as np
import pytest

SPECIAL = np.array([0.0, -0.0, np.nan, np.inf, -np.inf, 1e-45, -1e-45, 1e-40, -1e-40, 1.0, -1.0], np.float32)


def score_order(s):
    """The 32-bit key of select_rows_kernel: increasing in the score, -0 as +0."""
    b = np.asarray(s, np.float32).view(np.uint32).copy()
    b[b == 0x80000000] = 0
    return np.where(b & 0x80000000, ~b, b | 0x80000000).astype(np.uint32)


def reference(scores, ids, k):
    """vr_topk_rows of one row: valid entries (id >= 0, not NaN), distinct (score, id) pairs (+0 = -0), sorted by
    (score desc, id asc); the first k, then (-inf, -1)."""
    seen, rows = set(), []
    for s, i in zip(scores, ids):
        if i < 0 or np.isnan(s) or (float(s), int(i)) in seen:
            continue
        seen.add((float(s), int(i)))
        rows.append((-float(s), int(i), s))
    rows.sort(key=lambda r: (r[0], r[1]))
    out_s = np.full(k, -np.inf, np.float32)
    out_i = np.full(k, -1, np.int64)
    for j, (_, i, s) in enumerate(rows[:k]):
        out_s[j], out_i[j] = s, i
    return out_s, out_i


def _bin(hist, need, desc):
    """select_bin: (bin, entries before it, entries in it) of the need-th entry, bins walked down (desc) or up."""
    past = 0
    for b in (range(255, -1, -1) if desc else range(256)):
        if past + hist[b] >= need:
            return b, past, hist[b]
        past += hist[b]
    raise AssertionError("fewer entries than need")


def select_model(scores, ids, k, low_ids=True):
    """The digit passes of select_rows_kernel. low_ids=False is a mutant: boundary ties go to the higher ids."""
    scores = np.asarray(scores, np.float32)
    ids = np.asarray(ids, np.int64)
    valid = (ids >= 0) & ~np.isnan(scores)
    key = score_order(scores)
    thr, pmask, id_hi, split = 0, 0, None, True
    need = k
    for shift in (24, 16, 8, 0):
        m = valid & ((key & np.uint32(pmask)) == thr)
        hist = np.bincount((key[m] >> shift) & 255, minlength=256)
        if shift == 24 and m.sum() <= k:
            split = False
            break
        b, past, cnt = _bin(hist, need, True)
        need -= past
        thr |= b << shift
        pmask |= 255 << shift
        if cnt == need:
            split = False
            break
    if split:
        tied = valid & (key == thr)
        if not low_ids:  # the mutant: the highest ids of the boundary key
            order = np.sort(ids[tied])[::-1][:need]
            win = valid & (key > thr) | (tied & np.isin(ids, order))
        else:
            top = int(ids[tied].max())
            shift = (top.bit_length() - 1) // 8 * 8 if top else 0
            ip, imask = 0, 0
            while True:
                m = tied & ((ids & imask) == ip)
                hist = np.bincount((ids[m] >> shift) & 255, minlength=256)
                b, past, cnt = _bin(hist, need, False)
                need -= past
                ip |= b << shift
                imask |= 255 << shift
                if shift == 0 or cnt == need:
                    break
                shift -= 8
            id_hi = ip | ((1 << shift) - 1)
            win = valid & ((key > thr) | ((key == thr) & (ids <= id_hi)))
    elif thr == 0 and pmask == 0:
        win = valid
    else:
        win = valid & (key >= thr)
    sel = np.nonzero(win)[0]
    if len(sel) > k or len(set(zip(key[sel].tolist(), ids[sel].tolist()))) < len(sel):
        return reference(scores, ids, k)  # a repeated pair among the winners: the k-pass rerun
    order = sel[np.lexsort((ids[sel], ~key[sel]))]
    out_s = np.full(k, -np.inf, np.float32)
    out_i = np.full(k, -1, np.int64)
    out_s[:len(order)], out_i[:len(order)] = scores[order], ids[order]
    return out_s, out_i


def _same(a, b):
    return np.array_equal(a[1], b[1]) and np.array_equal(a[0].view(np.uint32), b[0].view(np.uint32))


def _rows(rs, cols):
    yield "random", rs.randn(cols).astype(np.float32), np.arange(cols)
    yield "all equal", np.full(cols, 0.5, np.float32), np.arange(cols)
    yield "few values", (rs.randint(0, 3, cols) / 3).astype(np.float32), rs.permutation(cols) * 1000 + 7
    yield "special values", SPECIAL[rs.randint(0, len(SPECIAL), cols)], np.arange(cols)
    yield "signed zeros", np.where(rs.rand(cols) < 0.5, np.float32(0.0), np.float32(-0.0)), np.arange(cols)
    yield "negative ids", rs.randn(cols).astype(np.float32), np.where(rs.rand(cols) < 0.4, -1, np.arange(cols))
    yield "mostly NaN", np.where(rs.rand(cols) < 0.9, np.float32(np.nan), rs.randn(cols).astype(np.float32)), np.arange(cols)
    yield "repeated pairs", (rs.randint(0, 5, cols) / 5).astype(np.float32), rs.randint(0, cols // 3 + 1, cols)


@pytest.mark.parametrize("cols", [1, 5, 64, 700, 3000])
def test_select_model_equals_a_full_sort(cols):
    rs = np.random.RandomState(cols)
    for name, s, i in _rows(rs, cols):
        for k in sorted({1, 3, 17, 100, cols, cols + 5}):
            assert _same(select_model(s, i, k), reference(s, i, k)), (name, k)


def test_tie_mutant_is_rejected():
    s = np.full(100, 0.5, np.float32)
    i = np.arange(100)
    assert _same(select_model(s, i, 10), reference(s, i, 10))
    assert not _same(select_model(s, i, 10, low_ids=False), reference(s, i, 10))


# ------------------------------------------------------------------------------------------------------------ deep route
def deep_model(S, k, elig=None, check_kept=True):
    """score_topk's deep route over exact scores S [nq, nd] (the scan's bits): t = the 16th score of the eligible pages
    0, s, 2s, ... (s = k // 8); A = eligible pages with S >= t; rows with |A| >= k answer from A, the rest from the scan.
    check_kept=False is a mutant: every row answers from A. Returns ((scores, ids), fallback rows)."""
    nq, nd = S.shape
    elig = np.ones_like(S, bool) if elig is None else elig
    stride = max(1, k // 8)
    out_s = np.full((nq, k), -np.inf, np.float32)
    out_i = np.full((nq, k), -1, np.int64)
    fallback = []
    for r in range(nq):
        ids = np.arange(nd)
        samp = reference(np.where(elig[r, ::stride], S[r, ::stride], np.nan), ids[::stride], 16)
        full = np.where(elig[r], S[r], np.nan)
        if samp[1][15] < 0:
            fallback.append(r)
            out_s[r], out_i[r] = reference(full, ids, k)
            continue
        a = full >= samp[0][15]
        if a.sum() < k and check_kept:
            fallback.append(r)
            out_s[r], out_i[r] = reference(full, ids, k)
        else:
            out_s[r], out_i[r] = reference(np.where(a, full, np.nan), ids, k)
    return (out_s, out_i), fallback


def _scan(S, k, elig=None):
    elig = np.ones_like(S, bool) if elig is None else elig
    rows = [reference(np.where(elig[r], S[r], np.nan), np.arange(S.shape[1]), k) for r in range(S.shape[0])]
    return np.stack([r[0] for r in rows]), np.stack([r[1] for r in rows])


def test_deep_model_equals_the_scan():
    rs = np.random.RandomState(1)
    S = rs.randn(20, 4000).astype(np.float32)
    S[3] = (rs.randint(0, 20, 4000) / 20).astype(np.float32)     # many exact ties
    elig = rs.rand(20, 4000) < 0.8
    for k in [40, 301, 1000]:
        for e in [None, elig]:
            got, _ = deep_model(S, k, e)
            assert _same(got, _scan(S, k, e)), k


def test_misleading_sample_needs_the_fallback():
    """Only the sampled pages score high: A holds them alone (fewer than k), so the row must rerun through the scan.
    The mutant that answers from A without the kept >= k check returns a short row."""
    k, nd = 400, 8000
    stride = k // 8
    S = np.random.RandomState(2).rand(1, nd).astype(np.float32) * 0.5
    S[0, ::stride] = 0.9 + np.arange(len(S[0, ::stride]), dtype=np.float32) * 1e-4
    got, fb = deep_model(S, k)
    assert fb == [0] and _same(got, _scan(S, k))
    bad, _ = deep_model(S, k, check_kept=False)
    assert not _same(bad, _scan(S, k)) and int((bad[1][0] >= 0).sum()) < k


def test_short_sample_falls_back():
    """Fewer than 16 eligible sampled pages: no threshold, the scan answers."""
    k, nd = 800, 5000
    S = np.random.RandomState(3).randn(1, nd).astype(np.float32)
    elig = np.zeros((1, nd), bool)
    elig[0, 1::2] = True                                       # no sampled page (stride 100) is eligible
    got, fb = deep_model(S, k, elig)
    assert fb == [0] and _same(got, _scan(S, k, elig))
