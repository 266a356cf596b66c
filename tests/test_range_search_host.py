"""Range search without a GPU: the margin of the threshold filter on the correlated fp16-rounding fixtures (a numpy model
against the fp32 scan's set, and three mutants that lose a page), the sort key of the ordering step (a numpy model of
range_key against the before() order), the routing of overflowed and unboundable rows to the scan (with a fake library),
the refusals of every new entry point (C ABI, before any CUDA call, fake pointers) and the Python argument checks (with a
library stub that fails if reached)."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

import __graft_entry__ as G
from tests import score_fixtures as F
from visrag_b200 import _lib as L
from visrag_b200 import retriever as R

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "visrag_b200.h")


# ------------------------------------------------------------------------------------------------ the margin
def fsub_rn(a, b):
    return np.float32(np.float32(a) - np.float32(b))


def _fixture_scores(fx):
    q = fx.Q[:1]
    ex = F.exact_scores(q, fx.D)[0]
    ap = F.approx_scores(q, fx.D)[0]
    eps = F.eps_of(F.row_norms(q)[0], F.row_norms(fx.D).max(), fx.Q.shape[1])
    return ex, ap, eps


@pytest.mark.parametrize("name", F.FIXTURES)
def test_threshold_filter_returns_the_scan_set_on_every_fixture(name):
    """t at the true page's exact score (its approximate score is low by most of the operand term of eps) and at the
    scores around it: the model's set is the fp32 scan's."""
    fx = next(f for f in F.fixtures() if f.name == name)
    ex, ap, eps = _fixture_scores(fx)
    s = ex[fx.true_doc]
    for t in (s, np.nextafter(s, np.float32(-1)), np.nextafter(s, np.float32(2)), np.float32(s - eps), np.float32(0.0)):
        assert F.range_model(ap, ex, t, eps) == set(np.nonzero(ex >= t)[0].tolist())


def test_the_fixture_puts_the_true_page_most_of_eps_low():
    fx = next(F.fixtures())
    ex, ap, eps = _fixture_scores(fx)
    gap = float(ex[fx.true_doc]) - float(ap[fx.true_doc])
    assert 0.5 * eps < gap < eps


def test_threshold_without_margin_loses_the_page():
    fx = next(F.fixtures())
    ex, ap, eps = _fixture_scores(fx)
    t = ex[fx.true_doc]
    assert fx.true_doc not in F.range_model(ap, ex, t, np.float32(0.0))


def test_eps_halved_loses_the_page():
    fx = next(F.fixtures())
    ex, ap, eps = _fixture_scores(fx)
    t = ex[fx.true_doc]
    assert fx.true_doc in F.range_model(ap, ex, t, eps)
    assert fx.true_doc not in F.range_model(ap, ex, t, np.float32(eps * 0.5))


def test_rounding_t_minus_eps_to_nearest_loses_the_page_where_it_rounds_up():
    """Rounding t - eps toward -inf leaves the filter one ulp of slack for eps's own fp32 evaluation: with an eps that
    falls short of the true page's gap by 3/4 of an ulp of its score, the rounded-down threshold still lands on the
    approximate score, while rounding to nearest goes up past it and loses the page."""
    fx = next(F.fixtures())
    ex, ap, _ = _fixture_scores(fx)
    t, a = ex[fx.true_doc], ap[fx.true_doc]
    ulp = float(np.nextafter(a, np.float32(1))) - float(a)
    short = np.float32(float(t) - float(a) - 0.75 * ulp)  # t - short lies 3/4 ulp above a
    assert float(t) - float(short) > float(a) + 0.5 * ulp
    assert fx.true_doc in F.range_model(ap, ex, t, short, F.fsub_rd)
    assert fx.true_doc not in F.range_model(ap, ex, t, short, fsub_rn)


# ------------------------------------------------------------------------------------------------ the sort key
def range_key(s, ids):
    """range_key of score.cu on numpy arrays: uint64 keys, ascending = (score desc, id asc)."""
    b = np.asarray(s, np.float32).view(np.uint32).copy()
    negzero = (b == 0x80000000).astype(np.uint64)
    b[b == 0x80000000] = 0
    o = np.where(b & 0x80000000, ~b, b | 0x80000000).astype(np.uint32)
    return ((~o).astype(np.uint64) << np.uint64(32)) | (np.asarray(ids, np.uint64) << np.uint64(1)) | negzero


def range_unkey(k):
    o = (~(k >> np.uint64(32))).astype(np.uint32)
    lo = (k & np.uint64(0xFFFFFFFF)).astype(np.uint32)
    b = np.where(o & 0x80000000, o & 0x7FFFFFFF, ~o).astype(np.uint32)
    b = np.where(lo & 1, np.uint32(0x80000000), b).astype(np.uint32)
    return b.view(np.float32), (lo >> 1).astype(np.int64)


def test_sort_key_orders_by_score_desc_then_id_asc_and_keeps_the_bits():
    rs = np.random.RandomState(0)
    s = np.concatenate([rs.randn(500).astype(np.float32), np.float32([0.0, -0.0, 0.0, -0.0, np.inf, -np.inf, 1e-45, -1e-45,
                                                                        3.0, 3.0])])
    ids = rs.permutation(len(s)) * 3 + 1
    order = np.argsort(range_key(s, ids), kind="stable")
    want = sorted(range(len(s)), key=lambda i: (-float(s[i]), ids[i]))  # before(): -0 == +0, so the id decides
    assert order.tolist() == want
    back_s, back_i = range_unkey(range_key(s, ids))
    assert np.array_equal(back_s.view(np.uint32), s.view(np.uint32)) and np.array_equal(back_i, ids)
    assert range_key(np.float32([np.inf]), [(1 << 31) - 1])[0] < np.uint64(0xFFFFFFFFFFFFFFFF)  # below the padding


# ------------------------------------------------------------------------------------------------ routing
class _FakeLib:
    """The filter path's library calls on CPU memory: counts and kept are what the test sets; nothing else is read."""

    def __init__(self, counts, kept):
        self.counts, self.kept = counts, kept

    @staticmethod
    def _write(ptr, values):
        (C.c_int32 * len(values)).from_address(ptr)[:] = list(values)

    def vr_f32_to_f16_rows(self, src, n, d, dst, norms, mx, stream):
        return 0

    def vr_score_filter_range(self, q16, n, d16, nd, d, t, qn, mx, masks, cap, counts, cand, stream):
        self._write(counts, self.counts)
        return 0

    def vr_score_rescore_range(self, q, n, emb, nd, d, t, cap, counts, cand, rs, ri, kept, stream):
        self._write(kept, self.kept)
        return 0


def test_overflowed_and_unboundable_rows_go_to_the_scan(monkeypatch):
    cap = 16
    # row 1 overflowed (more candidates than slots); row 2 has no bound (the kernel marks it cap + 1); rows 0, 3 fit
    monkeypatch.setattr(L, "_lib", _FakeLib([5, cap + 9, cap + 1, 0], [3, 0, 0, 0]))
    monkeypatch.setattr(L, "stream_ptr", lambda: 0)
    sorted_rows, scanned = [], []

    def fake_sort(rs, ri, pitch, counts, counts_host, sel, rows, id_offset):
        sorted_rows.extend(rows[sel].tolist())
        return rows[sel], counts_host[sel].long(), torch.zeros(0), torch.zeros(0, dtype=torch.int64)

    def fake_scan(q, index, t, masks, rows, id_offset):
        scanned.extend(rows.tolist())
        return [(rows, torch.zeros(rows.numel(), dtype=torch.int64), torch.zeros(0), torch.zeros(0, dtype=torch.int64))]

    monkeypatch.setattr(R, "_range_sort", fake_sort)
    monkeypatch.setattr(R, "_range_scan", fake_scan)
    index = _cpu_index(nd=1000, d=8)
    info = dict(candidates=0, fallback=0)
    R._range_filter(torch.zeros((4, 8)), index, torch.zeros(4), None, 0, torch.arange(10, 14), cap, 0, info)
    assert sorted_rows == [10, 13] and scanned == [11, 12]
    assert info["fallback"] == 2 and info["candidates"] == 5


def test_small_problems_and_force_exact_take_the_scan(monkeypatch):
    scanned = []

    def fake_scan(q, index, t, masks, rows, id_offset):
        scanned.append(rows.tolist())
        return [(rows, torch.zeros(rows.numel(), dtype=torch.int64), torch.zeros(0), torch.zeros(0, dtype=torch.int64))]

    monkeypatch.setattr(R, "_range_scan", fake_scan)
    monkeypatch.setattr(R, "_range_filter", lambda *a: pytest.fail("the filter ran"))
    big = _cpu_index(nd=100_000, d=8)
    for q, index, force in ((torch.zeros((3, 8)), _cpu_index(nd=1000, d=8), False), (torch.zeros((100, 8)), big, True)):
        stats = {}
        off, s, i = R._score_range(q, index, torch.zeros(q.shape[0]), 0, None, force, stats, 64)
        assert stats["path"] == "exact" and off.tolist() == [0] * (q.shape[0] + 1)
    assert scanned == [[0, 1, 2], list(range(100))]


def test_assembly_puts_pieces_back_in_row_order():
    pieces = [(torch.tensor([2, 0]), torch.tensor([1, 2]), torch.tensor([5., 1., 0.5]), torch.tensor([50, 10, 11])),
              (torch.tensor([1, 3]), torch.tensor([0, 2]), torch.tensor([7., 6.]), torch.tensor([30, 31]))]
    off, s, i = R._range_assemble(4, pieces, torch.device("cpu"))
    assert off.tolist() == [0, 2, 2, 3, 5] and s.tolist() == [1., 0.5, 5., 7., 6.] and i.tolist() == [10, 11, 50, 30, 31]


# ------------------------------------------------------------------------------------------------ C ABI refusals
no_device = pytest.mark.skipif(torch.cuda.is_available(), reason="fake pointers: run only where no CUDA device is visible")
FAKE = 0x7F0000000000

TABLES = {
    "vr_score_filter_range": {"q_f16": 16, "d_f16": 16, "thresholds": 4, "q_norms": 4, "max_doc_norm": 4, "counts": 4,
                              "cand_ids": 4},
    "vr_score_rescore_range": {"q_f32": 4, "d_f32": 16, "thresholds": 4, "counts": 4, "cand_ids": 4, "out_scores": 4,
                               "out_ids": 4, "kept": 4},
    "vr_range_rows": {"scores": 4, "thresholds": 4, "out_scores": 4, "out_ids": 4, "counts": 4},
    "vr_range_sort": {"scores": 4, "ids": 4, "counts": 4, "row_of": 4, "out_offsets": 8, "out_scores": 4, "out_ids": 8,
                      "ws": 8},
}


def _header_alignments(entry):
    text = open(HEADER).read()
    m = re.search(rf"Alignment \(bytes\) of the {entry} arguments: (.*?)(?:\n \* Alignment|\*/)", text, re.S)
    assert m, entry
    return {name: int(n) for name, n in re.findall(r"(\w+) (\d+)", m.group(1))}


@pytest.mark.parametrize("entry", sorted(TABLES))
def test_alignment_tables_match_header(entry):
    assert _header_alignments(entry) == TABLES[entry]


@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(L.LIB_PATH):
        G.build()
    return L.lib()


def _masks(words=FAKE + 0x1000, pitch=100, of_query=FAKE + 0x2000, count=3):
    m = L.DocMasks()
    m.words, m.pitch, m.of_query, m.count = words, pitch, of_query, count
    return m


def _call(lib, entry, masks="none", **over):
    p = {name: FAKE + 0x100000 * (i + 1) for i, name in enumerate(TABLES[entry])}
    a = dict(nq=40, nd=3000, dim=256, cap=64, rows=40, pitch=3000, max_count=5000, ws_bytes=1 << 30)
    for k, v in over.items():
        (p if k in p else a)[k] = v
    m = None if masks == "none" else C.byref(masks)
    if entry == "vr_score_filter_range":
        return lib.vr_score_filter_range(p["q_f16"], a["nq"], p["d_f16"], a["nd"], a["dim"], p["thresholds"], p["q_norms"],
                                         p["max_doc_norm"], m, a["cap"], p["counts"], p["cand_ids"], None)
    if entry == "vr_score_rescore_range":
        return lib.vr_score_rescore_range(p["q_f32"], a["nq"], p["d_f32"], a["nd"], a["dim"], p["thresholds"], a["cap"],
                                          p["counts"], p["cand_ids"], p["out_scores"], p["out_ids"], p["kept"], None)
    if entry == "vr_range_rows":
        return lib.vr_range_rows(p["scores"], a["rows"], a["nd"], p["thresholds"], m, a["pitch"], p["out_scores"],
                                 p["out_ids"], p["counts"], None)
    return lib.vr_range_sort(p["scores"], p["ids"], a["pitch"] if "pitch" in over else 8192, p["counts"], a["rows"],
                             p["row_of"], p["out_offsets"], a["max_count"], 0, p["ws"], a["ws_bytes"], p["out_scores"],
                             p["out_ids"], None)


BAD = [
    ("vr_score_filter_range", dict(nq=0), r"nq=0"),
    ("vr_score_filter_range", dict(nd=0), r"nd=0"),
    ("vr_score_filter_range", dict(nd=1 << 31), r"nd=2147483648"),
    ("vr_score_filter_range", dict(dim=12), r"dim=12"),
    ("vr_score_filter_range", dict(cap=0), r"cap=0"),
    ("vr_score_filter_range", dict(cap=-5), r"cap=-5"),
    ("vr_score_filter_range", dict(masks=_masks(count=0)), r"masks->count=0"),
    ("vr_score_filter_range", dict(masks=_masks(pitch=10)), r"masks->pitch=10"),
    ("vr_score_filter_range", dict(masks=_masks(words=FAKE + 0x1002)), r"masks->words must be 4-byte aligned"),
    ("vr_score_filter_range", dict(masks=_masks(of_query=None)), r"masks->of_query is NULL"),
    ("vr_score_rescore_range", dict(nq=0), r"nq=0"),
    ("vr_score_rescore_range", dict(dim=6), r"dim=6"),
    ("vr_score_rescore_range", dict(cap=0), r"cap=0"),
    ("vr_score_rescore_range", dict(nd=-1), r"nd=-1"),
    ("vr_range_rows", dict(rows=0), r"rows=0"),
    ("vr_range_rows", dict(rows=65536), r"rows=65536"),
    ("vr_range_rows", dict(pitch=2999), r"pitch=2999"),
    ("vr_range_rows", dict(masks=_masks(pitch=1)), r"masks->pitch=1"),
    ("vr_range_sort", dict(rows=0), r"rows=0"),
    ("vr_range_sort", dict(max_count=-1), r"max_count=-1"),
    ("vr_range_sort", dict(max_count=9000), r"max_count=9000"),
    ("vr_range_sort", dict(ws_bytes=1000), r"ws of 1000 bytes"),
    ("vr_range_sort", dict(ws=None), r"ws of"),
]


@no_device
@pytest.mark.parametrize("entry,kw,pattern", BAD, ids=[f"{e}-{sorted(k)[0]}-{i}" for i, (e, k, _) in enumerate(BAD)])
def test_refuses_bad_arguments_before_any_cuda_call(lib, entry, kw, pattern):
    rc = _call(lib, entry, **kw)
    msg = lib.vr_last_error().decode()
    assert rc == 2 and entry in msg and re.search(pattern, msg), (rc, msg)


@no_device
@pytest.mark.parametrize("entry,name", [(e, n) for e in sorted(TABLES) for n in TABLES[e]])
def test_refuses_each_null_and_misaligned_pointer(lib, entry, name):
    n = TABLES[entry][name]
    base = FAKE + 0x100000 * (list(TABLES[entry]).index(name) + 1)
    rc = _call(lib, entry, **{name: base + (4 if n >= 8 else 2)})
    msg = lib.vr_last_error().decode()
    assert rc == 2 and re.search(rf"\b{name}\b must be {n}-byte aligned", msg), (rc, msg)
    if name == "row_of":  # optional
        return
    rc = _call(lib, entry, **{name: None})
    msg = lib.vr_last_error().decode()
    assert rc == 2 and re.search(rf"\b{name}\b", msg), (rc, msg)


@no_device
@pytest.mark.parametrize("entry", sorted(TABLES))
def test_accepts_valid_arguments(lib, entry):
    """Past validation a call without a device stops at its first CUDA call (status 1), with or without masks."""
    for kw in (dict(), dict(masks=_masks()), dict(masks=_masks(count=1, of_query=None))):
        if entry in ("vr_score_rescore_range", "vr_range_sort") and kw:
            continue
        rc = _call(lib, entry, **kw)
        assert rc != 2, lib.vr_last_error().decode()
    if entry == "vr_range_sort":
        assert _call(lib, entry, max_count=100, ws=None, ws_bytes=0, row_of=None) != 2  # shared memory: no workspace
    assert lib.vr_range_sort_ws_bytes(3, 4096) == 0 and lib.vr_range_sort_ws_bytes(3, 4097) == 3 * 8192 * 8


# ------------------------------------------------------------------------------------------------ Python refusals
def _cpu_index(nd=100, d=8):
    return R.CorpusIndex(torch.zeros((nd, d)), torch.zeros((nd, d), dtype=torch.float16), torch.zeros(1))


class _NoLib:
    def __getattr__(self, name):
        raise AssertionError(f"the library was reached ({name}) although the arguments are invalid")


@pytest.fixture
def stub(monkeypatch):
    monkeypatch.setattr(L, "_lib", _NoLib())


@pytest.mark.parametrize("min_score,match", [
    (float("nan"), "must not be NaN"),
    (np.float32("nan"), "must not be NaN"),
    (torch.tensor([0.1, float("nan"), 0.2]), "must not be NaN"),
    (torch.tensor([0.1, 0.2]), r"shape \[3\]"),
    (torch.zeros((3, 1)), r"shape \[3\]"),
    (torch.zeros(3, dtype=torch.float64), "torch.float32"),
    ("0.5", "must be a float"),
    (None, "must be a float"),
    (True, "must be a float"),
])
def test_python_refuses_bad_thresholds(stub, min_score, match):
    with pytest.raises(ValueError, match=match):
        R._check_min_score(min_score, 3, torch.device("cpu"))


def test_python_threshold_forms(stub):
    t = R._check_min_score(0.25, 3, torch.device("cpu"))
    assert t.dtype == torch.float32 and t.tolist() == [0.25] * 3
    assert R._check_min_score(float("-inf"), 2, torch.device("cpu")).tolist() == [float("-inf")] * 2
    assert R._check_min_score(torch.tensor([0.5, 1.0]), 2, torch.device("cpu")).tolist() == [0.5, 1.0]
    for bad in (0, -1, 2.5, True, 1 << 31):
        with pytest.raises(ValueError, match="cap"):
            R._check_cap(bad)
    assert R._check_cap(None) == R.RANGE_CAP and R._check_cap(7) == 7


def test_python_refuses_bad_queries_and_masks(stub):
    idx = _cpu_index()
    with pytest.raises(ValueError, match="CUDA tensor"):
        R.score_range(torch.zeros((2, 8)), idx, 0.5)
    with pytest.raises(ValueError, match="doc_mask must be a torch.bool"):
        R._check_doc_mask(torch.ones(100), idx, 2)
