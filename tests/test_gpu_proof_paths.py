"""The proof fixtures of tests/score_fixtures.py through every filter-epilogue and rescoring path on the H100: the
unmasked, single-mask and per-query-mask page filters, the group-distinct filter and the grouped rescoring (with and
without masks), and the range filter. At each step the kernel's output is compared with the model's by the checkers
of tests/proof_paths.py (lists, flags and outputs, candidate sets), and the Python entry points' answers with the
fp32 scan's, bit for bit. The fixtures bring the true doc within a few per cent of eps of every decision, so a kernel
that scored a group from its kept entry, left unrescored groups out of its bound or used eps / 2 as the range margin
fails here; random data never comes near enough."""
import functools

import numpy as np
import pytest
import torch

from tests import proof_paths as PP
from tests import score_fixtures as SF

pytestmark = pytest.mark.gpu


class Env:
    """One fixture on the device: the index, the queries, the GPU's plan, and the one query's approximate scores
    (float64 sums of the fp16 operands, rounded once) and fp32-scan scores."""

    def __init__(self, fx):
        from visrag_b200 import retriever as R

        self.fx = fx
        self.nq, self.dim = fx.Q.shape
        self.nd = fx.D.shape[0]
        self.q = torch.from_numpy(fx.Q).cuda()
        self.idx = R.build_index(fx.D)
        self.p = PP.gpu_plan(self.nq, self.nd)
        assert self.p["R"] == 16, self.p                       # the doc ranges the fixtures' layout assumes
        assert self.p["items"] <= self.p["pairs"], self.p      # one wave: every item starts from tau = -inf, as the models
        ex = PP.vr_score_exact(self.q, self.idx)
        assert (ex == ex[:1]).all()                           # identical queries, identical rows
        self.ex = ex[0]
        self.ap = SF.approx_scores(fx.Q[:1], fx.D)[0]
        self.qn = SF.row_norms(fx.Q)
        self.dn = np.float32(self.idx.max_norm.item())
        self.eps = SF.eps_of(self.qn[0], self.dn, self.dim)
        # rows that are not filler (every component of a filler row is +-t16): the true doc, the decoys and the anchor
        self.planted = np.nonzero((fx.D >= 0).all(1))[0]
        # the toward-zero fixture's fp16 query is 2^-6 (1 + 2^-10): its sums need more than 24 bits, so the tensor cores
        # round partial sums and its list scores need not be the model's bits; its lists are not compared, its flags are
        self.exact_sums = PP.sums_exactly(fx.Q[0], fx.D)

    def check_lists(self, *args, **kw):
        if self.exact_sums:
            PP.check_lists(*args, **kw)

    def rows(self, x):
        return np.broadcast_to(x, (self.nq,) + np.shape(x)[1:])

    def masks(self):
        """The per-query mask set of the emulation test plus "true doc + filler"; of_query puts rows r and r + 8 of the
        first warp on different masks."""
        nd, fx = self.nd, self.fx
        rs = np.random.RandomState(11)
        without_true = np.ones(nd, bool)
        without_true[fx.true_doc] = False
        true_and_filler = np.ones(nd, bool)
        true_and_filler[self.planted] = False
        true_and_filler[fx.true_doc] = True
        masks = np.stack([np.ones(nd, bool), rs.rand(nd) < 0.5, without_true, (np.arange(nd) // SF.SC_BN) == 7,
                          np.zeros(nd, bool), np.arange(nd) < 3, true_and_filler])
        of = rs.randint(0, len(masks), self.nq)
        of[:16] = np.arange(16) % len(masks)
        return masks, of


@functools.lru_cache(maxsize=None)
def _fixtures():
    return {f.name: f for f in SF.fixtures()}


@functools.lru_cache(maxsize=None)
def _env(name):
    return Env(_fixtures()[name])


@pytest.fixture(scope="module", autouse=True)
def _release():
    yield
    _env.cache_clear()


def _report(name, path, flags, model_flags, ci, e):
    listed = (ci == e.fx.true_doc).any(axis=(1, 2))
    ratio, _ = SF.closeness(e.fx)
    print(f"\n{name} | {path}: flagged {int(flags.sum())}/{len(flags)} on the GPU, {int(model_flags.sum())} in the model; "
          f"true doc in the lists of {int(listed.sum())} rows; closeness {ratio:.3f} eps")
    return listed


def _same(a, b, what):
    for x, y in zip(a, b):
        x, y = np.asarray(x), np.asarray(y)
        assert np.array_equal(x.view(np.uint32) if x.dtype == np.float32 else x,
                              y.view(np.uint32) if y.dtype == np.float32 else y), what


# ------------------------------------------------------------------------------------------------------------ pages


@pytest.mark.parametrize("name", SF.FIXTURES)
def test_premise_true_doc_listed_with_the_models_approximate_score(name):
    """Under "true doc + filler" the true doc heads its list: its GPU score is SF.approx_scores' bits, and its distance
    below the fp32 scan's score is the closeness the CPU computes."""
    e = _env(name)
    masks, _ = e.masks()
    cs, ci = PP.vr_score_filter_masked(e.q, e.idx, torch.from_numpy(masks[-1]))
    model = SF.masked_filter_lists(e.ap[None], masks[-1], e.p)
    e.check_lists(cs, ci, *(e.rows(m) for m in model), e.rows(e.ap[None]), e.p, elig=e.rows(masks[-1][None]))
    at = ci == e.fx.true_doc
    assert (at.sum(axis=(1, 2)) == 1).all()
    got = cs[at]
    if not e.exact_sums:     # within the accumulation term of eps, dim 2^-23 sum|q16 d16|
        mag = np.abs(SF.to_f16(e.fx.Q[0]).astype(np.float64)) @ np.abs(SF.to_f16(e.fx.D[e.fx.true_doc]).astype(np.float64))
        err = np.abs(got.astype(np.float64) - float(e.ap[e.fx.true_doc]))
        print(f"\n{name}: sums not exact in fp32: GPU approx {got[0]!r}, model {e.ap[e.fx.true_doc]!r}, "
              f"|diff| / (dim 2^-23 sum|q16 d16|) = {err.max() / (e.dim * 2.0 ** -23 * mag):.3e}")
        assert (err <= e.dim * 2.0 ** -23 * mag).all()
        return
    assert (got.view(np.uint32) == e.ap[e.fx.true_doc:e.fx.true_doc + 1].view(np.uint32)).all()
    ratio = float((e.ex[e.fx.true_doc] - got[0]) / e.eps)
    want, _ = SF.closeness(e.fx)
    print(f"\n{name}: premise: GPU approx {got[0]!r} = model's; (exact - approx) / eps = {ratio:.4f} (CPU {want:.4f})")
    assert abs(ratio - want) <= 1e-3 * abs(want)


@pytest.mark.parametrize("name", SF.FIXTURES)
def test_unmasked_page_lists_and_flags(name):
    e = _env(name)
    cs, ci = PP.vr_score_filter(e.q, e.idx)
    model = SF.filter_lists(e.ap[None], e.p)
    e.check_lists(cs, ci, *(e.rows(m) for m in model), e.rows(e.ap[None]), e.p)
    out = PP.vr_score_rescore(e.q, e.idx, cs, ci, e.fx.k)
    mf = PP.check_rescore(cs, ci, out, e.rows(e.ex[None]), e.qn, e.dn, e.fx.k, e.dim, e.p)
    listed = _report(name, "pages", out[2], mf, ci, e)
    assert (~listed).all() == e.fx.dropped and (~listed).any() == e.fx.dropped and out[2].all()


@pytest.mark.parametrize("name", SF.FIXTURES)
def test_single_mask_page_lists_and_flags(name):
    e = _env(name)
    masks, _ = e.masks()
    flagged = []
    for m in masks:
        cs, ci = PP.vr_score_filter_masked(e.q, e.idx, torch.from_numpy(m))
        model = SF.masked_filter_lists(e.ap[None], m, e.p)
        e.check_lists(cs, ci, *(e.rows(x) for x in model), e.rows(e.ap[None]), e.p, elig=e.rows(m[None]))
        out = PP.vr_score_rescore(e.q, e.idx, cs, ci, e.fx.k)
        PP.check_rescore(cs, ci, out, e.rows(e.ex[None]), e.qn, e.dn, e.fx.k, e.dim, e.p)
        flagged.append(int(out[2].sum()))
    print(f"\n{name} | single mask: flagged per mask (GPU = model) {flagged}")


@pytest.mark.parametrize("name", SF.FIXTURES)
def test_per_query_mask_lists_flags_and_score_topk(name):
    from visrag_b200 import retriever as R

    e = _env(name)
    masks, of = e.masks()
    elig = masks[of]
    cs, ci = PP.vr_score_filter_masks(e.q, e.idx, torch.from_numpy(masks), of)
    ccs, cci = SF.filter_lists_per_query(np.repeat(e.ap[None], len(masks), 0), masks, e.p)
    e.check_lists(cs, ci, ccs[of], cci[of], e.rows(e.ap[None]), e.p, elig=elig)
    out = PP.vr_score_rescore(e.q, e.idx, cs, ci, e.fx.k)
    mf = PP.check_rescore(cs, ci, out, e.rows(e.ex[None]), e.qn, e.dn, e.fx.k, e.dim, e.p, elig=elig)
    stats = {}
    s, i = R.score_topk(e.q, e.idx, e.fx.k, doc_mask=torch.from_numpy(masks).cuda(), mask_of=torch.from_numpy(of).cuda(),
                        stats=stats)
    ref = SF.reference_per_query(np.repeat(e.ex[None], len(masks), 0), masks, e.fx.k)
    assert stats["path"] == "filter+rescore", stats
    _same((s.cpu().numpy(), i.cpu().numpy()), (ref[0][of], ref[1][of]), "score_topk with per-query masks")
    assert stats["flagged"] == int(mf.sum()), (stats, int(mf.sum()))
    _report(name, "per-query masks", out[2], mf, ci, e)


# -------------------------------------------------------------------------------------------------------- documents


def _groupings(e):
    return {"one page each": np.arange(e.nd), "contiguous 8": np.arange(e.nd) // 8,
            "true doc with its decoys": SF._true_with_decoys(e.fx)}


@pytest.mark.parametrize("masked", [False, True], ids=["no mask", "per-query masks"])
@pytest.mark.parametrize("name", SF.FIXTURES)
def test_document_lists_flags_and_score_topk_groups(name, masked):
    from visrag_b200 import retriever as R

    e = _env(name)
    masks, of = e.masks() if masked else (np.ones((1, e.nd), bool), np.zeros(e.nq, np.int64))
    elig = masks[of] if masked else None
    for what, groups in _groupings(e).items():
        gt_t = torch.from_numpy(groups.astype(np.int32)).cuda()
        gt = R._group_table(gt_t, e.idx)
        if masked:
            cs, ci = PP.vr_score_filter_groups_masks(e.q, e.idx, gt, torch.from_numpy(masks), of)
        else:
            cs, ci = PP.vr_score_filter_groups(e.q, e.idx, gt)
        ccs, cci = SF.grouped_filter_lists(np.repeat(e.ap[None], len(masks), 0), groups, e.p,
                                           elig=masks if masked else None)
        e.check_lists(cs, ci, ccs[of], cci[of], e.rows(e.ap[None]), e.p, elig=elig, groups=groups)
        if masked:
            out = PP.vr_score_rescore_groups_masks(e.q, e.idx, cs, ci, gt, e.fx.k, torch.from_numpy(masks), of)
        else:
            out = PP.vr_score_rescore_groups(e.q, e.idx, cs, ci, gt, e.fx.k)
        mf = PP.check_rescore(cs, ci, out, e.rows(e.ex[None]), e.qn, e.dn, e.fx.k, e.dim, e.p, groups=groups, elig=elig)
        kw = dict(doc_mask=torch.from_numpy(masks).cuda(), mask_of=torch.from_numpy(of).cuda()) if masked else {}
        stats = {}
        got = R.score_topk_groups(e.q, e.idx, e.fx.k, gt_t, stats=stats, **kw)
        assert stats["path"] == "filter+rescore", stats
        ref = [SF.grouped_reference(e.ex[None], groups, e.fx.k, mask=m if masked else None) for m in masks]
        ref = tuple(np.concatenate([r[j] for r in ref])[of] for j in range(3))
        _same(tuple(t.cpu().numpy() for t in got), ref, (what, masked))
        assert stats["flagged"] == int(mf.sum())
        listed = _report(name, f"documents, {what}, {'masks' if masked else 'no mask'}", out[3], mf, ci, e)
        if what == "true doc with its decoys" and name == "fp16 rounds down 0.49 ulp" and not masked:
            # the group's entry is a decoy; full rescoring of the group finds the true doc, and the proof holds
            assert not listed.any() and not out[3].any() and (got[1].cpu().numpy()[:, 0] == e.fx.true_doc).all()


def test_budget_fixture_flags_every_row_and_answers_the_true_page():
    """T's group holds more pages than the rescoring budget: only T's approximate entry in the bound keeps the proof from
    certifying the decoy Y, so every row is flagged and the scan answers T."""
    from visrag_b200 import retriever as R

    Q1, D, groups, T, Y = SF._budget_fixture()
    Q = np.repeat(Q1, 600, axis=0)
    q, idx = torch.from_numpy(Q).cuda(), R.build_index(D)
    p = PP.gpu_plan(*Q.shape[:1], D.shape[0])
    assert p["R"] == 16 and p["items"] <= p["pairs"], p
    gt_t = torch.from_numpy(groups.astype(np.int32)).cuda()
    gt = R._group_table(gt_t, idx)
    cs, ci = PP.vr_score_filter_groups(q, idx, gt)
    ap = SF.approx_scores(Q1, D)
    model = SF.grouped_filter_lists(ap, groups, p)
    assert PP.sums_exactly(Q1[0], D)
    PP.check_lists(cs, ci, *(np.broadcast_to(m, cs.shape) for m in model), np.broadcast_to(ap, (600, D.shape[0])), p,
                   groups=groups)
    ex = PP.vr_score_exact(q[:1], idx)
    out = PP.vr_score_rescore_groups(q, idx, cs, ci, gt, 1)
    mf = PP.check_rescore(cs, ci, out, np.broadcast_to(ex, (600, D.shape[0])), SF.row_norms(Q), np.float32(idx.max_norm.item()),
                          1, Q.shape[1], p, groups=groups)
    stats = {}
    s, pg, g = R.score_topk_groups(q, idx, 1, gt_t, stats=stats)
    print(f"\nbudget fixture | documents: flagged {int(out[3].sum())}/600 on the GPU, {int(mf.sum())} in the model; "
          f"rescored answer before the scan {sorted(set(out[1][:, 0].tolist()))}")
    assert out[3].all() and stats["flagged"] == 600 and (pg.cpu().numpy()[:, 0] == T).all()


# ------------------------------------------------------------------------------------------------------------ range


@pytest.mark.parametrize("masked", [False, True], ids=["no mask", "per-query masks"])
@pytest.mark.parametrize("name", SF.FIXTURES)
def test_range_candidates_rescoring_and_score_range(name, masked):
    from tests.test_gpu_range_search import reference
    from visrag_b200 import retriever as R

    e = _env(name)
    td = e.fx.true_doc
    s_star = e.ex[td]
    decoys = np.setdiff1d(e.planted, [td, 20 * SF.SC_BN + 11])
    ts = {"s*": s_star, "s* - 1 ulp": np.nextafter(s_star, np.float32(-1)), "s* + 1 ulp": np.nextafter(s_star, np.float32(2)),
          "fl(s* - eps)": np.float32(s_star - e.eps), "0": np.float32(0.0), "best decoy": e.ex[decoys].max()}
    masks, of = e.masks()
    elig = masks[of] if masked else None
    mk = dict(masks=torch.from_numpy(masks), of_query=of) if masked else {}
    for what, t in ts.items():
        tt = np.full(e.nq, t, np.float32)
        counts, cand = PP.vr_score_filter_range(e.q, e.idx, tt, e.nd, **mk)
        member = PP.check_range(cand, counts, e.rows(e.ap[None]), tt, e.eps, elig)
        rs, ri, kept = PP.vr_score_rescore_range(e.q, e.idx, tt, counts, cand)
        want = member & (e.ex[None] >= t)
        assert (kept == want.sum(1)).all(), what
        for r in np.unique(of if masked else [0]):
            row = int(np.nonzero(of == r)[0][0]) if masked else 0
            ids = ri[row, :kept[row]]
            assert set(ids.tolist()) == set(np.nonzero(want[row])[0].tolist()), (what, row)
            assert (rs[row, :kept[row]].view(np.uint32) == e.ex[ids].view(np.uint32)).all(), (what, row)
        if what == "s*":
            # no margin or eps / 2 would lose the true doc: its approximate score lies most of eps below s*
            if SF.closeness(e.fx)[0] > 0:   # the fixtures whose fp16 copies round the true doc down
                assert e.ap[td] < s_star
            ok = elig[:, td] if masked else np.ones(e.nq, bool)
            assert member[ok, td].all()
            print(f"\n{name} | range, {'masks' if masked else 'no mask'}: true doc a candidate in {int(member[:, td].sum())}"
                  f"/{e.nq} rows at t = s*; closeness {SF.closeness(e.fx)[0]:.3f} eps; candidates per row at t = s*: "
                  f"{sorted(set(counts.tolist()))}")
        stats = {}
        kw = dict(doc_mask=torch.from_numpy(masks).cuda(), mask_of=torch.from_numpy(of).cuda()) if masked else {}
        got = R.score_range(e.q, e.idx, float(t), stats=stats, **kw)
        assert stats["path"] == "filter+rescore" and stats["fallback"] == 0, (what, stats)
        ref = reference(e.q, e.idx, float(t), mask=torch.from_numpy(elig).cuda() if masked else None)
        for x, y in zip(got, ref):
            assert x.dtype == y.dtype and torch.equal(x, y), what
