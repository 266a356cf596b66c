"""The checkers of tests/proof_paths.py are not vacuous: each passes the models' own output on the proof fixtures and
rejects a plausible wrong kernel, modelled as a mutant of the filter or the rescoring, on at least one fixture:

    masked tau taken from the unmasked scores   -> check_lists (tau)
    row r searched with the mask of row r ^ 8   -> check_lists (an ineligible id)
    page lists where group-distinct lists go    -> check_lists (a group twice)
    a group scored by its kept entry            -> check_rescore, and the answer is not the true doc
    B without the groups left unrescored        -> check_rescore (flags)
    range margin 0, eps / 2 and 2 eps           -> check_range (lower / upper inclusion)

The plan is the CPU default (66 CTA pairs: one wave for 600 queries, as on the H100)."""
import functools

import numpy as np
import pytest

from tests import proof_paths as PP
from tests import score_fixtures as SF


@functools.lru_cache(maxsize=None)
def _fixtures():
    return {f.name: f for f in SF.fixtures()}


@functools.lru_cache(maxsize=None)
def _fixture(name):
    """(fixture, approximate scores [nd], exact scores [nd], plan) of the fixture's one query."""
    fx = _fixtures()[name]
    q = fx.Q[:1]
    return fx, SF.approx_scores(q, fx.D)[0], SF.exact_scores(q, fx.D)[0], SF.plan(fx.Q.shape[0], fx.D.shape[0])


def _rows(x, nq):
    return np.broadcast_to(x, (nq,) + x.shape[1:])


def _norms(fx):
    return SF.row_norms(fx.Q[:1]), SF.row_norms(fx.D).max()


def _mask_set(fx, seed=11):
    """The per-query mask set of the emulation test, with rows r and r + 8 of the first warp on different masks."""
    nd, nq = fx.D.shape[0], fx.Q.shape[0]
    rs = np.random.RandomState(seed)
    without_true = np.ones(nd, bool)
    without_true[fx.true_doc] = False
    masks = np.stack([np.ones(nd, bool), rs.rand(nd) < 0.5, without_true, (np.arange(nd) // SF.SC_BN) == 7,
                      np.zeros(nd, bool), np.arange(nd) < 3])
    of_query = rs.randint(0, len(masks), nq)
    of_query[:16] = np.arange(16) % len(masks)
    return masks, of_query


@pytest.mark.parametrize("name", SF.FIXTURES)
def test_checkers_pass_the_models_on_every_fixture(name):
    fx, ap, ex, p = _fixture(name)
    masks, of = _mask_set(fx)
    M = len(masks)
    cs, ci = SF.filter_lists_per_query(_rows(ap[None], M), masks, p)
    PP.check_lists(cs, ci, cs, ci, _rows(ap[None], M), p, elig=masks)
    qn, dn = _norms(fx)
    out = SF.rescore(cs, ci, _rows(ex[None], M), np.repeat(qn, M), dn, fx.k, fx.Q.shape[1], p)[:3]
    PP.check_rescore(cs, ci, out, _rows(ex[None], M), np.repeat(qn, M), dn, fx.k, fx.Q.shape[1], p)
    groups = np.arange(fx.D.shape[0]) // 8
    gcs, gci = SF.grouped_filter_lists(_rows(ap[None], M), groups, p, elig=masks)
    PP.check_lists(gcs, gci, gcs, gci, _rows(ap[None], M), p, elig=masks, groups=groups)
    eps = SF.eps_of(qn[0], dn, fx.Q.shape[1])
    for t in (ex[fx.true_doc], np.float32(0.0)):
        cand = masks & (ap[None] >= SF.fsub_rd(t, eps))
        counts = cand.sum(1)
        ids = np.full((M, fx.D.shape[0]), -1, np.int32)
        for r in range(M):
            ids[r, :counts[r]] = np.nonzero(cand[r])[0]
        PP.check_range(ids, counts, _rows(ap[None], M), t, eps, masks)


def test_grouped_model_without_a_mask_is_the_unmasked_model():
    fx, ap, ex, p = _fixture("fp16 rounds down 0.49 ulp")
    groups = SF._true_with_decoys(fx)
    a = SF.grouped_filter_lists(ap[None], groups, p)
    b = SF.grouped_filter_lists(ap[None], groups, p, elig=np.ones((1, fx.D.shape[0]), bool))
    assert all(np.array_equal(x, y) for x, y in zip(a, b))
    qn, dn = _norms(fx)
    args = (*a, ex[None], groups, qn, dn, 1, fx.Q.shape[1])
    ra, rb = SF.grouped_rescore(*args), SF.grouped_rescore(*args, elig=np.ones((1, fx.D.shape[0]), bool))
    assert all(np.array_equal(x, y) for x, y in zip(ra, rb))
    # a mask without the true doc: the group is scored by its other (eligible) pages
    m = np.ones((1, fx.D.shape[0]), bool)
    m[0, fx.true_doc] = False
    rm = SF.grouped_rescore(*SF.grouped_filter_lists(ap[None], groups, p, elig=m), ex[None], groups, qn, dn, 1,
                            fx.Q.shape[1], elig=m)
    ref = SF.grouped_reference(ex[None], groups, 1, mask=m[0])
    assert rm[1][0, 0] != fx.true_doc and (rm[3][0] or all(np.array_equal(x, y) for x, y in zip(rm[:3], ref)))


def test_tau_from_unmasked_scores_fails_check_lists():
    fx, ap, ex, p = _fixture("fp16 rounds down 0.49 ulp")
    mask = np.random.RandomState(7).rand(fx.D.shape[0]) < 0.5
    good = SF.masked_filter_lists(ap[None], mask, p)
    bad = SF.masked_filter_lists(ap[None], mask, p, tau_from_unmasked=True)
    PP.check_lists(*good, *good, ap[None], p, elig=mask[None])
    with pytest.raises(AssertionError, match="tau differs"):
        PP.check_lists(*bad, *good, ap[None], p, elig=mask[None])


def test_the_mask_of_row_r_xor_8_fails_check_lists():
    fx, ap, ex, p = _fixture("fp16 rounds down 0.49 ulp")
    masks, of = _mask_set(fx)
    nq = len(of)
    cs, ci = SF.filter_lists_per_query(_rows(ap[None], len(masks)), masks, p)
    other = of[np.minimum(np.arange(nq) ^ 8, nq - 1)]
    approx, elig = _rows(ap[None], nq), masks[of]
    PP.check_lists(cs[of], ci[of], cs[of], ci[of], approx, p, elig=elig)
    with pytest.raises(AssertionError, match="ineligible"):
        PP.check_lists(cs[other], ci[other], cs[of], ci[of], approx, p, elig=elig)


@pytest.mark.parametrize("name", SF.FIXTURES)
def test_page_lists_where_group_distinct_lists_go_fail_check_lists(name):
    fx, ap, ex, p = _fixture(name)
    groups = np.arange(fx.D.shape[0]) // 8
    good = SF.grouped_filter_lists(ap[None], groups, p)
    bad = SF.filter_lists(ap[None], p)
    with pytest.raises(AssertionError, match="repeats a group"):
        PP.check_lists(*bad, *good, ap[None], p, groups=groups)


def test_group_score_from_the_kept_entry_fails_check_rescore_and_answers_wrong():
    fx, ap, ex, p = _fixture("fp16 rounds down 0.49 ulp")
    groups = SF._true_with_decoys(fx)
    cs, ci = SF.grouped_filter_lists(ap[None], groups, p)
    assert fx.true_doc not in ci
    qn, dn = _norms(fx)
    args = (cs, ci, ex[None], groups, qn, dn, 1, fx.Q.shape[1])
    ref = SF.grouped_reference(ex[None], groups, 1)
    good, bad = SF.grouped_rescore(*args), SF.grouped_rescore(*args, mut="entry score")
    PP.check_rescore(cs, ci, good, ex[None], qn, dn, 1, fx.Q.shape[1], p, groups=groups)
    assert not good[3][0] and good[1][0, 0] == ref[1][0, 0] == fx.true_doc
    assert not bad[3][0] and bad[1][0, 0] != fx.true_doc                 # unflagged: this is the final answer
    with pytest.raises(AssertionError, match="rescored scores differ"):
        PP.check_rescore(cs, ci, bad, ex[None], qn, dn, 1, fx.Q.shape[1], p, groups=groups)


def test_bound_without_the_unrescored_groups_fails_check_rescore():
    Q, D, groups, T, Y = SF._budget_fixture()
    p = SF.plan(600, D.shape[0])
    ap, ex = SF.approx_scores(Q, D), SF.exact_scores(Q, D)
    cs, ci = SF.grouped_filter_lists(ap, groups, p)
    qn, dn = SF.row_norms(Q), SF.row_norms(D).max()
    args = (cs, ci, ex, groups, qn, dn, 1, Q.shape[1])
    good, bad = SF.grouped_rescore(*args), SF.grouped_rescore(*args, mut="B without unrescored groups")
    assert good[3][0] and not bad[3][0] and bad[1][0, 0] == Y
    PP.check_rescore(cs, ci, good, ex, qn, dn, 1, Q.shape[1], p, groups=groups)
    with pytest.raises(AssertionError, match="flags differ"):
        PP.check_rescore(cs, ci, bad, ex, qn, dn, 1, Q.shape[1], p, groups=groups)


def _range_cands(ap, t, margin):
    cand = np.nonzero(ap >= SF.fsub_rd(t, margin))[0].astype(np.int32)
    return cand[None], np.array([len(cand)])


@pytest.mark.parametrize("mut,t_at,match", [(0.0, "true doc", "not candidates"), (0.5, "true doc", "not candidates"),
                                            (2.0, "zero", "below t - eps")])
def test_range_margin_mutants_fail_check_range(mut, t_at, match):
    fx, ap, ex, p = _fixture("fp16 rounds down 0.49 ulp")
    qn, dn = _norms(fx)
    eps = SF.eps_of(qn[0], dn, fx.Q.shape[1])
    t = ex[fx.true_doc] if t_at == "true doc" else np.float32(0.0)
    PP.check_range(*_range_cands(ap, t, eps), ap[None], t, eps)
    with pytest.raises(AssertionError, match=match):
        PP.check_range(*_range_cands(ap, t, np.float32(mut * eps)), ap[None], t, eps)


def test_sums_are_exact_in_fp32_where_the_fp16_query_is_a_power_of_two():
    """The list checks compare bits only where no summation order can round: the toward-zero fixture's fp16 query is
    2^-6 (1 + 2^-10), and its true doc's and decoys' sums need more than 24 bits."""
    exact = {name: PP.sums_exactly(fx.Q[0], fx.D) for name, fx in _fixtures().items()}
    assert exact == {n: n != "rounds up 0.01 ulp (toward zero: down 0.99)" for n in SF.FIXTURES}
    Q, D, _, _, _ = SF._budget_fixture()
    assert PP.sums_exactly(Q[0], D)
