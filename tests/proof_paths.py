"""What the filter kernels did, step by step, against the models of tests/score_fixtures.py: the candidate lists, the
rescoring kernels' per-row flags and outputs, and the range filter's candidate sets.

The drivers call the C entry points directly, so a filter kernel runs whatever path the Python routing would have
chosen, and each writes into NaN / 0x7F7F7F7F-poisoned buffers: a slot or counter a kernel forgot to write shows up.
They return numpy arrays; the rescoring drivers take numpy lists, so the GPU's own lists can be fed back. Importing
this module touches no CUDA (torch and the library load inside the drivers).

The checkers take the kernel's output and the model's, and compare what does not depend on the kernel's tie order:
many filler docs of the fixtures have equal approximate scores, so which of two equal docs a list keeps is free, but
the multiset of scores, the eligibility and span of every id, and the tail published as tau are not. The host tests
feed known mutants through the same checkers to show that each check can fail."""
import ctypes as C

import numpy as np

from tests import score_fixtures as SF

KT = SF.KT
POISON = 0x7F7F7F7F


def _bits(x):
    return np.ascontiguousarray(x, np.float32).view(np.uint32)


# ------------------------------------------------------------------------------------------------------------ drivers


def _lib():
    from visrag_b200 import _lib as L

    return L, L.lib()


def gpu_plan(nq, nd):
    """vr_score_plan: the work decomposition the library launches on this GPU (its pairs follow the SM count)."""
    L, lib = _lib()
    out = np.zeros(6, np.int32)
    L.check(lib.vr_score_plan(nq, nd, out.ctypes.data))
    return dict(zip(("T", "R", "QB", "items", "pairs", "lists"), (int(v) for v in out)))


def _poisoned(nq, nd):
    import torch

    L, lib = _lib()
    ranges = lib.vr_score_ranges(nq, nd)
    return ranges, (torch.full((nq, 2 * ranges, KT), float("nan"), device="cuda"),
                    torch.full((nq, 2 * ranges, KT), POISON, dtype=torch.int32, device="cuda"))


def _np(*ts):
    return tuple(t.cpu().numpy() for t in ts)


def mask_set(masks, of_query=None):
    """bool [M, nd] masks and int [nq] of_query (None: mask 0 for every row) -> (vr_doc_masks, tensors to keep alive)."""
    import torch

    from visrag_b200 import _lib as L
    from visrag_b200.retriever import pack_doc_mask

    words = pack_doc_mask(masks.reshape(-1, masks.shape[-1]).cuda())
    of = None if of_query is None else torch.as_tensor(np.asarray(of_query), dtype=torch.int32).cuda().contiguous()
    m = L.DocMasks()
    m.words, m.pitch, m.count = words.data_ptr(), words.shape[1], words.shape[0]
    m.of_query = None if of is None else of.data_ptr()
    return m, (words, of)


def _filter(fn, q, idx, *extra):
    from visrag_b200 import retriever as R

    L, lib = _lib()
    nq, d = q.shape
    ranges, (cs, ci) = _poisoned(nq, idx.nd)
    q16 = R.to_f16_rows(q)
    L.check(getattr(lib, fn)(q16.data_ptr(), nq, idx.emb_f16.data_ptr(), idx.nd, d, ranges, cs.data_ptr(), ci.data_ptr(),
                             *extra, L.stream_ptr()))
    return _np(cs, ci)


def vr_score_filter(q, idx):
    """The unmasked page filter: (cand_scores, cand_ids) [nq, lists, 16]."""
    return _filter("vr_score_filter", q, idx)


def vr_score_filter_masked(q, idx, mask):
    """The page filter with one bool [nd] doc mask."""
    from visrag_b200.retriever import pack_doc_mask

    words = pack_doc_mask(mask.cuda())
    return _filter("vr_score_filter_masked", q, idx, words.data_ptr())


def vr_score_filter_masks(q, idx, masks, of_query):
    """The page filter with a mask per query row: row r searches masks[of_query[r]]."""
    m, keep = mask_set(masks, of_query)
    return _filter("vr_score_filter_masks", q, idx, C.byref(m))


def vr_score_filter_groups(q, idx, gt, mask=None):
    """The group-distinct filter (gt: the retriever's group table), optionally with one bool [nd] doc mask."""
    from visrag_b200.retriever import pack_doc_mask

    words = None if mask is None else pack_doc_mask(mask.cuda())
    return _filter("vr_score_filter_groups", q, idx, gt.groups.data_ptr(), None if words is None else words.data_ptr())


def vr_score_filter_groups_masks(q, idx, gt, masks, of_query):
    m, keep = mask_set(masks, of_query)
    return _filter("vr_score_filter_groups_masks", q, idx, gt.groups.data_ptr(), C.byref(m))


def _lists_to_device(cs, ci):
    import torch

    return (torch.from_numpy(np.ascontiguousarray(cs, np.float32)).cuda(),
            torch.from_numpy(np.ascontiguousarray(ci).astype(np.int32)).cuda())


def vr_score_rescore(q, idx, cs, ci, k):
    """rescore_topk_kernel on the lists (cs, ci) [nq, lists, 16]: (scores [nq, k], ids [nq, k], flags [nq])."""
    import torch

    L, lib = _lib()
    nq, d = q.shape
    dcs, dci = _lists_to_device(cs, ci)
    s = torch.full((nq, k), float("nan"), device="cuda")
    i = torch.full((nq, k), POISON, dtype=torch.int64, device="cuda")
    flags = torch.full((nq,), POISON, dtype=torch.int32, device="cuda")
    L.check(lib.vr_score_rescore(q.data_ptr(), nq, idx.emb.data_ptr(), idx.nd, d, cs.shape[1] // 2, dcs.data_ptr(),
                                 dci.data_ptr(), idx.max_norm.data_ptr(), k, 0, s.data_ptr(), i.data_ptr(), flags.data_ptr(),
                                 L.stream_ptr()))
    return _np(s, i, flags)


def _rescore_groups(fn, q, idx, cs, ci, gt, k, mask_arg):
    import torch

    L, lib = _lib()
    nq, d = q.shape
    dcs, dci = _lists_to_device(cs, ci)
    s = torch.full((nq, k), float("nan"), device="cuda")
    p = torch.full((nq, k), POISON, dtype=torch.int64, device="cuda")
    g = torch.full((nq, k), POISON, dtype=torch.int64, device="cuda")
    flags = torch.full((nq,), POISON, dtype=torch.int32, device="cuda")
    L.check(getattr(lib, fn)(q.data_ptr(), nq, idx.emb.data_ptr(), idx.nd, d, cs.shape[1] // 2, dcs.data_ptr(), dci.data_ptr(),
                             gt.groups.data_ptr(), gt.offsets.data_ptr(), gt.pages.data_ptr(), gt.G, mask_arg,
                             idx.max_norm.data_ptr(), k, 0, s.data_ptr(), p.data_ptr(), g.data_ptr(), flags.data_ptr(),
                             L.stream_ptr()))
    return _np(s, p, g, flags)


def vr_score_rescore_groups(q, idx, cs, ci, gt, k, mask=None):
    """rescore_groups_kernel: (scores, best pages, groups) [nq, k] and flags [nq]."""
    from visrag_b200.retriever import pack_doc_mask

    words = None if mask is None else pack_doc_mask(mask.cuda())
    return _rescore_groups("vr_score_rescore_groups", q, idx, cs, ci, gt, k, None if words is None else words.data_ptr())


def vr_score_rescore_groups_masks(q, idx, cs, ci, gt, k, masks, of_query):
    m, keep = mask_set(masks, of_query)
    return _rescore_groups("vr_score_rescore_groups_masks", q, idx, cs, ci, gt, k, C.byref(m))


def vr_score_filter_range(q, idx, t, cap, masks=None, of_query=None):
    """The range filter with thresholds t [nq]: (counts [nq], cand_ids [nq, cap]); counts > cap marks an overflow."""
    import torch

    L, lib = _lib()
    nq, d = q.shape
    q16 = torch.empty((nq, d), dtype=torch.float16, device="cuda")
    qn = torch.empty(nq, device="cuda")
    L.check(lib.vr_f32_to_f16_rows(q.data_ptr(), nq, d, q16.data_ptr(), qn.data_ptr(), None, L.stream_ptr()))
    tt = torch.as_tensor(np.asarray(t, np.float32)).cuda()
    counts = torch.full((nq,), POISON, dtype=torch.int32, device="cuda")
    cand = torch.full((nq, cap), POISON, dtype=torch.int32, device="cuda")
    m, keep = mask_set(masks, of_query) if masks is not None else (None, None)
    L.check(lib.vr_score_filter_range(q16.data_ptr(), nq, idx.emb_f16.data_ptr(), idx.nd, d, tt.data_ptr(), qn.data_ptr(),
                                      idx.max_norm.data_ptr(), None if m is None else C.byref(m), cap, counts.data_ptr(),
                                      cand.data_ptr(), L.stream_ptr()))
    return _np(counts, cand)


def vr_score_rescore_range(q, idx, t, counts, cand):
    """range_rescore_kernel on the filter's candidates: (scores [nq, cap], ids [nq, cap], kept [nq])."""
    import torch

    L, lib = _lib()
    nq, d = q.shape
    cap = cand.shape[1]
    tt = torch.as_tensor(np.asarray(t, np.float32)).cuda()
    dc = torch.from_numpy(np.ascontiguousarray(counts, np.int32)).cuda()
    di = torch.from_numpy(np.ascontiguousarray(cand, np.int32)).cuda()
    s = torch.full((nq, cap), float("nan"), device="cuda")
    i = torch.full((nq, cap), POISON, dtype=torch.int32, device="cuda")
    kept = torch.full((nq,), POISON, dtype=torch.int32, device="cuda")
    L.check(lib.vr_score_rescore_range(q.data_ptr(), nq, idx.emb.data_ptr(), idx.nd, d, tt.data_ptr(), cap, dc.data_ptr(),
                                       di.data_ptr(), s.data_ptr(), i.data_ptr(), kept.data_ptr(), L.stream_ptr()))
    return _np(s, i, kept)


def vr_score_exact(q, idx):
    """The fp32 scan's scores [nq, nd] (the bits every rescoring kernel gives a pair)."""
    import torch

    L, lib = _lib()
    s = torch.full((q.shape[0], idx.nd), float("nan"), device="cuda")
    L.check(lib.vr_score_exact(q.data_ptr(), q.shape[0], idx.emb.data_ptr(), idx.nd, q.shape[1], s.data_ptr(),
                               L.stream_ptr()))
    return s.cpu().numpy()


# ----------------------------------------------------------------------------------------------------------- checkers


def sums_exactly(q, D):
    """Whether every dot product of q's fp16 copy with a row of D's fp16 copy is exact in fp32 whatever the summation
    order: every product is a multiple of 2^-(kq + kd) (kq, kd: the finest bit of the fp16 vectors) and the sum of the
    products' magnitudes stays below 2^(24 - kq - kd). Then the filter's approximate scores are SF.approx_scores' bits;
    otherwise the tensor cores round partial sums (within the accumulation term of eps) and the bits may differ."""
    def finest(x):                    # smallest k with x * 2^k integral, per row (fp16 values are multiples of 2^-24)
        xi = np.abs(SF.to_f16(x).astype(np.float64) * 2.0 ** 24).astype(np.int64)
        low = np.where(xi > 0, xi & -xi, 1 << 40)
        return 24 - np.log2(low.min(axis=-1)).astype(np.int64)
    q16, d16 = SF.to_f16(q).astype(np.float64), SF.to_f16(D).astype(np.float64)
    mag = np.abs(d16) @ np.abs(q16)
    return bool((mag * 2.0 ** (finest(q[None])[0] + finest(D)) < 2.0 ** 24).all())



def check_lists(gpu_cs, gpu_ci, model_cs, model_ci, approx, plan, elig=None, groups=None):
    """The kernel's candidate lists [nq, lists, 16] against the model's, independent of tie order. approx [nq, nd]: the
    approximate scores (fp16 operands, exact sums); elig [nq, nd]: each row's eligible docs (None: all); groups [nd]:
    the lists are group-distinct. What a list may hold is checked first (span, eligibility, no doc twice, the
    approximate score, one entry per group and that its group's best), then the score multisets and tau."""
    nq, L_, kt = gpu_cs.shape
    nd = approx.shape[1]
    R = plan["R"]
    assert (L_, kt) == (plan["lists"], KT) and model_cs.shape == gpu_cs.shape, (gpu_cs.shape, plan)
    assert not np.isnan(gpu_cs).any(), "a list slot was not written"
    assert ((gpu_ci == -1) | ((gpu_ci >= 0) & (gpu_ci < nd))).all(), "an id outside [-1, nd)"
    s, i = gpu_cs[:, :R], gpu_ci[:, :R]
    live = i >= 0
    assert np.array_equal(live, ~np.isneginf(s)), "empty slots and -inf scores differ"
    # every id in its list's doc range, eligible for its row, not twice in a row, with its approximate score
    lo, hi = np.array([SF.range_docs(plan, nd, r) for r in range(R)]).T
    out = live & ((i < lo[None, :, None]) | (i >= hi[None, :, None]))
    assert not out.any(), f"ids outside their doc range at {np.argwhere(out)[:5].tolist()}"
    rows = np.broadcast_to(np.arange(nq)[:, None, None], i.shape)[live]
    ids = i[live]
    if elig is not None:
        ok = elig[rows, ids]
        assert ok.all(), f"ineligible (row, id) in the lists: {list(zip(rows[~ok][:5], ids[~ok][:5]))}"
    srt = np.sort(gpu_ci.reshape(nq, -1), axis=1)
    twice = ((srt[:, 1:] == srt[:, :-1]) & (srt[:, 1:] >= 0)).any(1)
    assert not twice.any(), f"a doc twice in rows {np.nonzero(twice)[0][:5].tolist()}"
    same = _bits(approx[rows, ids]) == _bits(s[live])
    assert same.all(), f"list scores are not the approximate scores at (row, id) {list(zip(rows[~same][:5], ids[~same][:5]))}"
    if groups is not None:
        for r in range(R):
            gr = np.where(i[:, r] >= 0, groups[np.maximum(i[:, r], 0)], -1 - np.arange(KT)[None, :])
            gs = np.sort(gr, axis=1)
            rep = ((gs[:, 1:] == gs[:, :-1]) & (gs[:, 1:] >= 0)).any(1)
            assert not rep.any(), f"list {r} repeats a group in rows {np.nonzero(rep)[0][:5].tolist()}"
            # each entry is its group's best eligible approximate score in the span
            span = groups[lo[r]:hi[r]]
            order = np.argsort(span, kind="stable")
            ug, start = np.unique(span[order], return_index=True)
            a = approx[:, lo[r]:hi[r]]
            if elig is not None:
                a = np.where(elig[:, lo[r]:hi[r]], a, -np.inf)
            best = np.maximum.reduceat(a[:, order], start, axis=1)
            v = i[:, r] >= 0
            want = np.take_along_axis(best, np.searchsorted(ug, groups[np.where(v, i[:, r], lo[r])]), 1)
            wrong = v & (_bits(want) != _bits(s[:, r]))
            assert not wrong.any(), f"list {r}: an entry is not its group's best at {np.argwhere(wrong)[:5].tolist()}"
    # against the model: the multiset of score bits of every list
    bad = (np.sort(_bits(s), axis=2) != np.sort(_bits(model_cs[:, :R]), axis=2)).any(2)
    assert not bad.any(), f"list scores differ from the model's at (row, list) {np.argwhere(bad)[:5].tolist()}"
    # the unused lists are empty; the last one carries tau in its first score and nothing else
    assert (gpu_ci[:, R:] == -1).all() and np.isneginf(gpu_cs[:, R:L_ - 1]).all(), "an unused list was written"
    assert np.isneginf(gpu_cs[:, -1, 1:]).all(), "the tau slot holds more than tau"
    tau = _bits(gpu_cs[:, -1, 0]) != _bits(model_cs[:, -1, 0])
    assert not tau.any(), f"tau differs from the model's in rows {np.nonzero(tau)[0][:5].tolist()}"


def _distinct_rows(*arrays):
    """Row indices of the distinct rows of the arrays taken together, and each row's index among them."""
    keys = [b"".join(np.ascontiguousarray(a[r]).tobytes() for a in arrays if a is not None) for r in range(len(arrays[0]))]
    first, inv = {}, np.empty(len(keys), np.int64)
    for r, kb in enumerate(keys):
        inv[r] = first.setdefault(kb, len(first))
    reps = np.empty(len(first), np.int64)
    reps[inv[::-1]] = np.arange(len(keys))[::-1]
    return reps, inv


def check_rescore(gpu_cs, gpu_ci, gpu_out, exact, qn, dn, k, dim, plan, groups=None, elig=None):
    """Feeds the kernel's lists to the model's rescoring (SF.rescore for pages, SF.grouped_rescore with groups) and
    requires the kernel's flags, row by row, and its outputs, bit for bit. gpu_out: (scores, ids, flags) for pages,
    (scores, pages, groups, flags) for documents. exact [nq, nd]: the fp32 scan's scores; qn [nq]: the query norms.
    The model runs once per distinct row. Returns the model's flags."""
    qn = np.asarray(qn, np.float32)
    reps, inv = _distinct_rows(gpu_cs, gpu_ci, exact, qn[:, None], elig)
    args = (gpu_cs[reps], gpu_ci[reps], exact[reps])
    if groups is None:
        model = SF.rescore(*args, qn[reps], dn, k, dim, plan)[:3]
    else:
        model = SF.grouped_rescore(*args, groups, qn[reps], dn, k, dim, elig=None if elig is None else elig[reps])
    flags = model[-1][inv]
    diff = np.asarray(gpu_out[-1]) != flags
    assert not diff.any(), f"flags differ from the model's in rows {np.nonzero(diff)[0][:5].tolist()}"
    for name, g, m in zip(("scores", "ids", "groups"), gpu_out[:-1], model[:-1]):
        m = m[inv]
        diff = (_bits(g) != _bits(m)).any(1) if name == "scores" else (np.asarray(g) != m).any(1)
        assert not diff.any(), f"rescored {name} differ from the model's in rows {np.nonzero(diff)[0][:5].tolist()}"
    return flags


def check_range(cands, counts, approx, t, eps, elig=None):
    """The range filter's candidates [nq, cap] (first counts[r] of row r): no row overflowed, no doc twice, and
        {eligible, approx >= t - eps (1 - 2^-20)}  <=  candidates  <=  {eligible, approx >= t - eps (1 + 2^-20)}
    in float64, with eps = SF.eps_of per row. The slack covers an FMA-contracted eps in the kernel, whose last bits
    need not be eps_of's. Returns the candidate membership [nq, nd]."""
    nq, cap = cands.shape
    nd = approx.shape[1]
    counts = np.asarray(counts)
    over = (counts < 0) | (counts > cap)
    assert not over.any(), f"rows overflowed (or counts not written): {np.nonzero(over)[0][:5].tolist()}"
    live = np.arange(cap)[None, :] < counts[:, None]
    ids = cands[live].astype(np.int64)
    assert ((ids >= 0) & (ids < nd)).all(), "a candidate id outside [0, nd)"
    rows = np.nonzero(live)[0]
    n = np.bincount(rows * nd + ids, minlength=nq * nd).reshape(nq, nd)
    assert n.max(initial=0) <= 1, f"a doc twice in rows {np.nonzero(n.max(1) > 1)[0][:5].tolist()}"
    member = n > 0
    t64 = np.broadcast_to(np.asarray(t, np.float64), (nq,))[:, None]
    e64 = np.broadcast_to(np.asarray(eps, np.float64), (nq,))[:, None]
    a64 = approx.astype(np.float64)
    ok = np.ones((nq, nd), bool) if elig is None else elig
    must = ok & (a64 >= t64 - e64 * (1 - 2.0 ** -20))
    may = ok & (a64 >= t64 - e64 * (1 + 2.0 ** -20))
    lost = must & ~member
    assert not lost.any(), f"docs above t - eps are not candidates: (row, id) {np.argwhere(lost)[:5].tolist()}"
    extra = member & ~may
    assert not extra.any(), f"candidates below t - eps: (row, id) {np.argwhere(extra)[:5].tolist()}"
    return member
