"""Per-query masks without a GPU: 2-D mask packing, the refusals of the mask-set entry points (C ABI, before any CUDA call)
and of the Python arguments, and a numpy emulation of the filter with a mask per query. Each query row reads its own mask,
so its lists, its lane thresholds and its published tau are over its own eligible docs; the emulation returns every
query's masked fp32 top-k, and a mutant that publishes one query's tau to another query of the same block (the thread's
other accumulator row) returns a wrong one on a multi-wave fixture where queries with the same vector have different
masks."""
import ctypes as C
import functools
import os
import re

import numpy as np
import pytest
import torch

import __graft_entry__ as G
from tests import score_fixtures as SF
from visrag_b200 import _lib as L
from visrag_b200.retriever import CorpusIndex, _check_doc_mask, pack_doc_mask


@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(L.LIB_PATH):
        G.build()
    return L.lib()


def _packbits(m):
    nd = m.shape[-1]
    pad = np.zeros(m.shape[:-1] + (-nd % 32,), bool)
    return np.packbits(np.concatenate([m, pad], -1), axis=-1, bitorder="little").view(np.uint32)


@pytest.mark.parametrize("M,nd", [(1, 1), (3, 31), (5, 32), (2, 33), (7, 100), (4, 4097), (3, 125_001)])
def test_pack_doc_mask_2d_equals_numpy_packbits_row_by_row(M, nd):
    rs = np.random.RandomState(M * 1000 + nd)
    m = rs.rand(M, nd) < rs.rand(M, 1)
    m[0] = True
    w = pack_doc_mask(torch.from_numpy(m))
    assert w.dtype == torch.uint32 and w.shape == (M, (nd + 31) // 32)
    got = w.view(torch.int32).numpy().view(np.uint32)
    assert np.array_equal(got, _packbits(m))
    for r in range(M):  # each row is the 1-D packing of that row
        assert np.array_equal(pack_doc_mask(torch.from_numpy(m[r])).view(torch.int32).numpy().view(np.uint32), got[r])


def test_pack_doc_mask_2d_without_rows():
    w = pack_doc_mask(torch.zeros((0, 70), dtype=torch.bool))
    assert w.shape == (0, 3) and w.dtype == torch.uint32


# ------------------------------------------------------------------------------------------------ Python refusals
def _cpu_index(nd=100, d=8):
    return CorpusIndex(torch.zeros((nd, d)), torch.zeros((nd, d), dtype=torch.float16), torch.zeros(1))


@pytest.mark.parametrize("doc_mask,mask_of,nq,match", [
    (torch.ones((3, 99), dtype=torch.bool), None, 3, "doc_mask must have shape"),
    (torch.ones((2, 3, 100), dtype=torch.bool), None, 3, "doc_mask must have shape"),
    (torch.ones((3, 100), dtype=torch.uint8), None, 3, "doc_mask must be a torch.bool"),
    (torch.ones((2, 100), dtype=torch.bool), None, 3, "2 rows for 3 queries"),
    (torch.ones((2, 100), dtype=torch.bool), torch.tensor([0, 1]), 3, r"mask_of must have shape \[3\]"),
    (torch.ones((2, 100), dtype=torch.bool), torch.tensor([[0, 1, 1]]), 3, r"mask_of must have shape \[3\]"),
    (torch.ones((2, 100), dtype=torch.bool), torch.tensor([0., 1., 1.]), 3, "mask_of must be an int32 or int64"),
    (torch.ones((2, 100), dtype=torch.bool), [0, 1, 1], 3, "mask_of must be an int32 or int64"),
    (torch.ones((2, 100), dtype=torch.bool), torch.tensor([0, 2, 1]), 3, r"mask_of must lie in \[0, 2\)"),
    (torch.ones((2, 100), dtype=torch.bool), torch.tensor([0, -1, 1]), 3, r"mask_of must lie in \[0, 2\)"),
    (torch.ones(100, dtype=torch.bool), torch.tensor([0, 0, 0]), 3, "this doc_mask is 1-D"),
])
def test_python_refuses_bad_mask_sets(doc_mask, mask_of, nq, match):
    with pytest.raises(ValueError, match=match):
        _check_doc_mask(doc_mask, _cpu_index(), nq, mask_of)


def test_python_mask_set_defaults_to_one_row_per_query():
    m = torch.from_numpy(np.random.RandomState(0).rand(4, 100) < 0.5)
    ms = _check_doc_mask(m, _cpu_index(), 4)
    assert ms.of_query.tolist() == [0, 1, 2, 3] and ms.of_query.dtype == torch.int32
    assert torch.equal(ms.words, pack_doc_mask(m))
    one = _check_doc_mask(m[0], _cpu_index(), 4)       # a 1-D mask: the set of one, no of_query
    assert one.of_query is None and one.words.shape == (1, 4)
    sel = _check_doc_mask(m, _cpu_index(), 3, torch.tensor([3, 3, 1]))
    assert sel.of_query.tolist() == [3, 3, 1] and sel.rows(torch.tensor([2, 0])).of_query.tolist() == [1, 3]


# ------------------------------------------------------------------------------------------------ C ABI refusals
FAKE = 0x7F0000000000  # never dereferenced: every call below must stop in argument validation


def _set(words=FAKE + 0x1000, pitch=None, of_query=FAKE + 0x2000, count=3, nd=5000):
    m = L.DocMasks()
    m.words, m.pitch, m.of_query, m.count = words, (nd + 31) // 32 if pitch is None else pitch, of_query, count
    return m


def _calls(lib):
    """Each _masks entry point with valid fake arguments, nd = cols = 5000."""
    nq, nd, dim = 300, 5000, 256
    ranges = lib.vr_score_ranges(nq, nd)
    p = lambda i: FAKE + 0x100000 * i  # noqa: E731
    return {
        "vr_score_filter_masks": lambda m: lib.vr_score_filter_masks(p(1), nq, p(2), nd, dim, ranges, p(3), p(4), m, None),
        "vr_score_filter_groups_masks": lambda m: lib.vr_score_filter_groups_masks(p(1), nq, p(2), nd, dim, ranges, p(3),
                                                                                   p(4), p(5), m, None),
        "vr_score_rescore_groups_masks": lambda m: lib.vr_score_rescore_groups_masks(
            p(1), nq, p(2), nd, dim, ranges, p(3), p(4), p(5), p(6), p(7), 50, m, p(8), 10, 0, p(9), p(10), p(11), p(12), None),
        "vr_topk_rows_masks": lambda m: lib.vr_topk_rows_masks(p(1), None, 4, nd, 10, 0, p(2), p(3), m, None),
        "vr_topk_rows_chunked_masks": lambda m: lib.vr_topk_rows_chunked_masks(p(1), 1, nd, 10, 0, 16, p(2), p(3), p(4), p(5),
                                                                               m, None),
        "vr_group_topk_rows_masks": lambda m: lib.vr_group_topk_rows_masks(
            p(1), 4, nd, p(2), 50, m, 10, 0, 0, p(3), lib.vr_group_topk_ws_bytes(4, 50, 10, 0), p(4), p(5), p(6), None),
    }


ENTRIES = ["vr_score_filter_masks", "vr_score_filter_groups_masks", "vr_score_rescore_groups_masks", "vr_topk_rows_masks",
           "vr_topk_rows_chunked_masks", "vr_group_topk_rows_masks"]
BAD = {
    "masks NULL": (None, r"\bmasks\b"),
    "words NULL": (_set(words=None), r"masks->words"),
    "words misaligned": (_set(words=FAKE + 0x1002), r"masks->words must be 4-byte aligned"),
    "count 0": (_set(count=0), r"masks->count=0"),
    "count -1": (_set(count=-1), r"masks->count=-1"),
    "pitch short": (_set(pitch=156), r"masks->pitch=156"),
    "of_query NULL with count 2": (_set(of_query=None, count=2), r"masks->of_query is NULL"),
    "of_query misaligned": (_set(of_query=FAKE + 0x2002), r"masks->of_query must be 4-byte aligned"),
}
no_device = pytest.mark.skipif(torch.cuda.is_available(), reason="fake pointers: run only where no CUDA device is visible")


@no_device
@pytest.mark.parametrize("entry", ENTRIES)
@pytest.mark.parametrize("bad", sorted(BAD))
def test_masks_entry_points_refuse_a_bad_mask_set_before_any_cuda_call(lib, entry, bad):
    m, pattern = BAD[bad]
    rc = _calls(lib)[entry](None if m is None else C.byref(m))
    msg = lib.vr_last_error().decode()
    assert rc == 2, (rc, msg)
    assert entry in msg and re.search(pattern, msg), msg


@no_device
@pytest.mark.parametrize("entry", ENTRIES)
def test_masks_entry_points_accept_valid_mask_sets(lib, entry):
    """A set of one without of_query, and a set of three with it (pitch above the minimum), get past validation; without a
    device they then stop at their first CUDA call (status 1)."""
    for m in (_set(of_query=None, count=1), _set(pitch=200)):
        rc = _calls(lib)[entry](C.byref(m))
        assert rc != 2, lib.vr_last_error().decode()


@no_device
def test_masks_entry_points_keep_the_other_pointer_checks(lib):
    m = _set()
    nq, nd = 300, 5000
    rc = lib.vr_score_filter_masks(FAKE + 4, nq, FAKE, nd, 256, lib.vr_score_ranges(nq, nd), FAKE, FAKE, C.byref(m), None)
    assert rc == 2 and b"q_f16" in lib.vr_last_error()
    rc = lib.vr_topk_rows_masks(FAKE, FAKE, 4, nd, 10, 0, FAKE, FAKE, C.byref(m), None)
    assert rc == 2 and b"ids must be NULL" in lib.vr_last_error()
    rc = lib.vr_score_filter_groups_masks(FAKE, nq, FAKE, nd, 256, lib.vr_score_ranges(nq, nd), FAKE, FAKE, FAKE + 2,
                                          C.byref(m), None)
    assert rc == 2 and b"doc_groups" in lib.vr_last_error()


# ------------------------------------------------------------------------------------------------ emulation
def emulate_per_query(Q, D, k, masks, of_query, pairs=SF.PAIRS, leak=False):
    nq, dim = Q.shape
    p = SF.plan(nq, D.shape[0], pairs)
    elig = masks[of_query]
    exact, approx = SF.exact_scores(Q, D), SF.approx_scores(Q, D)
    cs, ci = SF.filter_lists_per_query(approx, elig, p, leak)
    s, i, flags, _, _ = SF.rescore(cs, ci, exact, SF.row_norms(Q), SF.row_norms(D).max(), k, dim, p)
    ref_s, ref_i = SF.reference_per_query(exact, elig, k)
    bad = flags.astype(bool)
    s[bad], i[bad] = ref_s[bad], ref_i[bad]          # flagged: each query's own masked fp32 scan answers
    return s, i, flags, dict(plan=p, ci=ci, elig=elig, ref=(ref_s, ref_i))


@functools.lru_cache(maxsize=None)
def _fixtures():
    return tuple(SF.fixtures())


@pytest.mark.parametrize("name", SF.FIXTURES)
def test_per_query_emulation_returns_each_querys_masked_fp32_topk_on_the_proof_fixtures(name):
    fx = {f.name: f for f in _fixtures()}[name]
    nq, nd = fx.Q.shape[0], fx.D.shape[0]
    rs = np.random.RandomState(11)
    without_true = np.ones(nd, bool)
    without_true[fx.true_doc] = False
    masks = np.stack([np.ones(nd, bool), rs.rand(nd) < 0.5, without_true, (np.arange(nd) // SF.SC_BN) == 7,
                      np.zeros(nd, bool), np.arange(nd) < 3])
    of_query = rs.randint(0, len(masks), nq)
    of_query[:16] = np.arange(16) % len(masks)    # rows r and r + 8 of the first warp: different masks
    s, i, flags, info = emulate_per_query(fx.Q, fx.D, fx.k, masks, of_query)
    ref_s, ref_i = info["ref"]
    assert np.array_equal(i, ref_i) and np.array_equal(s, ref_s)
    listed = info["ci"] >= 0
    rows = np.nonzero(listed)[0]
    assert info["elig"][rows, info["ci"][listed]].all()  # every list holds its own query's eligible docs only
    # a mask set of one with of_query all zeros gives the lists of the single-mask emulation
    _, _, _, one = emulate_per_query(fx.Q, fx.D, fx.k, masks[1:2], np.zeros(nq, np.int64))
    _, ci = SF.masked_filter_lists(SF.approx_scores(fx.Q, fx.D), masks[1], one["plan"])
    assert np.array_equal(one["ci"], ci)


def _multi_wave_fixture():
    """600 copies of one query over 4096 docs at 5 CTA pairs (8 doc ranges, 5 waves). Mask 0 keeps every doc; mask 1 removes
    the 400 best. Rows alternate in runs of 8, so rows r and r + 8 of every warp search different masks with the same
    vector: the unmasked row's tails lie above every doc the masked row may return."""
    rs = np.random.RandomState(21)
    nq, nd, dim, pairs = 600, 4096, 8, 5
    D = rs.randn(nd, dim).astype(np.float32)
    Q = np.repeat(rs.randn(1, dim).astype(np.float32), nq, axis=0)
    best = np.argsort(-SF.exact_scores(Q[:1], D)[0], kind="stable")[:400]
    masks = np.ones((2, nd), bool)
    masks[1, best] = False
    of_query = (np.arange(nq) // 8) % 2
    return Q, D, masks, of_query, pairs


def test_tau_published_to_another_query_returns_a_wrong_topk():
    Q, D, masks, of_query, pairs = _multi_wave_fixture()
    p = SF.plan(Q.shape[0], D.shape[0], pairs)
    assert p["items"] > p["pairs"] and p["R"] > 1, p                       # several waves and doc ranges
    for k in (1, 10):
        s, i, flags, info = emulate_per_query(Q, D, k, masks, of_query, pairs)
        assert np.array_equal(i, info["ref"][1]) and np.array_equal(s, info["ref"][0]), k
        assert not np.array_equal(info["ref"][1][0], info["ref"][1][8])  # the two masks do give different answers
    wrong = 0
    for k in (1, 10):
        _, i, _, info = emulate_per_query(Q, D, k, masks, of_query, pairs, leak=True)
        wrong += int((i != info["ref"][1]).any(1).sum())
    assert wrong > 0
