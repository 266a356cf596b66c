"""Filtered retrieval without a GPU: the doc-mask packing, the C ABI's refusals of a bad mask (before any CUDA call), and
a numpy emulation of the masked filter + proof. The filter replaces an ineligible doc's score by -inf before the fast
path and the insertion, so it never enters a list and never reaches a published threshold tau; the proof then bounds
only eligible docs. The emulation returns the masked fp32 top-k on the proof fixtures, and a mutant that publishes tau
from the UNMASKED list tails returns a wrong one on a multi-wave fixture whose mask removes every query's best docs."""
import functools
import os

import numpy as np
import pytest
import torch

import __graft_entry__ as G
from tests import score_fixtures as SF
from visrag_b200 import _lib as L
from visrag_b200.retriever import pack_doc_mask


@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(L.LIB_PATH):
        G.build()
    return L.lib()


@pytest.mark.parametrize("nd", [1, 31, 32, 33, 100, 4097, 125_001])
def test_pack_doc_mask_equals_numpy_packbits(nd):
    rs = np.random.RandomState(nd)
    for frac in (0.5, 0.01, 1.0):
        m = rs.rand(nd) < frac
        w = pack_doc_mask(torch.from_numpy(m))
        ref = np.packbits(np.concatenate([m, np.zeros(-nd % 32, bool)]), bitorder="little").view(np.uint32)
        assert w.dtype == torch.uint32 and w.shape == ((nd + 31) // 32,)
        assert np.array_equal(w.view(torch.int32).numpy().view(np.uint32), ref)


def test_masked_entry_points_refuse_a_bad_mask_before_any_cuda_call(lib):
    """Pointers here are never dereferenced: every call must be refused by argument checks on the host."""
    fake = 1 << 20
    rc = lib.vr_score_filter_masked(fake, 300, fake, 5000, 256, lib.vr_score_ranges(300, 5000), fake, fake, None, None)
    assert rc != 0 and b"doc_mask" in lib.vr_last_error()
    rc = lib.vr_score_filter_masked(fake, 300, fake, 5000, 256, lib.vr_score_ranges(300, 5000), fake, fake, fake + 2, None)
    assert rc != 0 and b"aligned" in lib.vr_last_error()
    rc = lib.vr_topk_rows_masked(fake, None, 4, 1000, 10, 0, fake, fake, None, None)
    assert rc != 0 and b"doc_mask" in lib.vr_last_error()
    rc = lib.vr_topk_rows_masked(fake, fake, 4, 1000, 10, 0, fake, fake, fake, None)
    assert rc != 0 and b"ids must be NULL" in lib.vr_last_error()
    rc = lib.vr_topk_rows_chunked_masked(fake, 1, 100000, 10, 0, 16, fake, fake, fake, fake, None, None)
    assert rc != 0 and b"doc_mask" in lib.vr_last_error()
    rc = lib.vr_topk_rows_chunked_masked(fake, 1, 100000, 10, 0, 16, fake, fake, fake, fake, fake + 1, None)
    assert rc != 0 and b"aligned" in lib.vr_last_error()


# ------------------------------------------------------------------------------------------------------ emulation


def masked_reference(exact, mask, k):
    """The fp32 scan over the eligible docs: (score desc, id asc), then (-inf, -1)."""
    s = np.where(mask[None, :], exact, -np.inf).astype(np.float32)
    order = np.lexsort((np.broadcast_to(np.arange(s.shape[1]), s.shape), -s), axis=1)[:, :k]
    out_s = np.take_along_axis(s, order, 1)
    out_i = np.where(np.isinf(out_s) & (out_s < 0), -1, order)
    return out_s, out_i.astype(np.int64)


def emulate_masked(Q, D, k, mask, pairs=SF.PAIRS, tau_from_unmasked=False):
    nq, dim = Q.shape
    p = SF.plan(nq, D.shape[0], pairs)
    exact, approx = SF.exact_scores(Q, D), SF.approx_scores(Q, D)
    cs, ci = SF.masked_filter_lists(approx, mask, p, tau_from_unmasked)
    # the index's max row norm covers every doc, eligible or not: still an upper bound over the eligible ones
    s, i, flags, _, _ = SF.rescore(cs, ci, exact, SF.row_norms(Q), SF.row_norms(D).max(), k, dim, p)
    ref_s, ref_i = masked_reference(exact, mask, k)
    bad = flags.astype(bool)
    s[bad], i[bad] = ref_s[bad], ref_i[bad]          # flagged: the masked fp32 scan answers
    return s, i, flags, dict(plan=p, ci=ci, ref=(ref_s, ref_i))


@functools.lru_cache(maxsize=None)
def _fixtures():
    return tuple(SF.fixtures())


@pytest.mark.parametrize("name", SF.FIXTURES)
def test_masked_emulation_returns_the_masked_fp32_topk_on_the_proof_fixtures(name):
    fx = {f.name: f for f in _fixtures()}[name]
    nd = fx.D.shape[0]
    rs = np.random.RandomState(7)
    without_true = np.ones(nd, bool)
    without_true[fx.true_doc] = False
    masks = {"all": np.ones(nd, bool), "random 50 %": rs.rand(nd) < 0.5, "without the true doc": without_true,
             "one tile": (np.arange(nd) // SF.SC_BN) == 7}
    for what, m in masks.items():
        s, i, flags, info = emulate_masked(fx.Q, fx.D, fx.k, m)
        ref_s, ref_i = info["ref"]
        assert np.array_equal(i, ref_i) and np.array_equal(s, ref_s), what
        assert m[info["ci"][info["ci"] >= 0]].all(), what                  # no ineligible doc in any list
    # the all-ones mask reproduces the unmasked emulation's lists exactly
    _, _, _, plain = SF.emulate(fx.Q, fx.D, fx.k)
    _, _, _, info = emulate_masked(fx.Q, fx.D, fx.k, np.ones(nd, bool))
    assert np.array_equal(info["ci"], plain["ci"])


def _multi_wave_fixture():
    """600 copies of one query over 4096 docs at 5 CTA pairs (8 doc ranges, 5 waves); the mask removes the 400 best docs
    (every query's best), so every unmasked list tail lies above every eligible doc."""
    rs = np.random.RandomState(21)
    nq, nd, dim, pairs = 600, 4096, 8, 5
    D = rs.randn(nd, dim).astype(np.float32)
    Q = np.repeat(rs.randn(1, dim).astype(np.float32), nq, axis=0)
    best = np.argsort(-SF.exact_scores(Q[:1], D)[0], kind="stable")[:400]
    mask = np.ones(nd, bool)
    mask[best] = False
    return Q, D, mask, pairs


def test_tau_from_unmasked_tails_returns_a_wrong_topk():
    Q, D, mask, pairs = _multi_wave_fixture()
    p = SF.plan(Q.shape[0], D.shape[0], pairs)
    assert p["items"] > p["pairs"] and p["R"] > 1, p                       # several waves and doc ranges
    for k in (1, 10):
        s, i, flags, info = emulate_masked(Q, D, k, mask, pairs)
        assert np.array_equal(i, info["ref"][1]) and np.array_equal(s, info["ref"][0]), k
    wrong = 0
    for k in (1, 10):
        _, i, _, info = emulate_masked(Q, D, k, mask, pairs, tau_from_unmasked=True)
        wrong += int((i != info["ref"][1]).any(1).sum())
    assert wrong > 0
