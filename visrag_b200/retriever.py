"""Dense retrieval on the H100: drop-in for `src/openmatch/retriever/dense_retriever.py`.

Same call signatures and on-disk formats as the reference:
  * `_retrieve_one_shard(corpus_shard_path, encoded_queries_tensor, topk, device)` -> (scores, indices, lookup)
    (`dense_retriever.py:13-34`), shard file = `pickle((float32[n, d], List[str]))` (`inference/inference.py:126`);
  * `distributed_parallel_retrieve(args, topk)` -> {qid: {docid: score}} (`dense_retriever.py:37-97`).
Underneath, `torch.matmul` + `torch.topk` are replaced by the fused wgmma filter + exact fp32 rescoring kernels
(csrc/score.cu): the returned scores are fp32 dot products and the top-k equals the fp32 scan's
(order: score descending, then doc index ascending — `torch.topk` leaves tie order unspecified).

For a corpus that lives in HBM (index build + many query batches) use `CorpusIndex` / `score_topk` directly; the
multi-GPU form (`sharded_topk`) shards the corpus by page across ranks, takes the local top-k with global ids and
merges after ONE all-gather of [nq, k] (score, id) pairs. Both take an optional `doc_mask` (bool [nd], local to the
shard): only the docs it marks are searched, and the result equals the fp32 scan over those docs alone. A 2-D doc_mask
(bool [M, nd]) with `mask_of` (int [nq] in [0, M), default row i for query i) gives every query its own subset, in the
same one pass over the index: each query's row equals its call alone with its own mask.
Candidate lists (`doc_lists=(offsets, ids)`, CSR, with `list_of`): each query scores only the pages of its list and reads
no others; the result equals the masked call with a mask of exactly the listed pages, bit for bit.

Document-level retrieval (`score_topk_groups`, `sharded_topk_groups`): `doc_groups` (int [nd]) gives every doc (page) its
group (document); the top-k groups by their best page's exact fp32 score, ranked by (score desc, best page asc). For
300 < k <= 1024 they take the deep route over a sample of documents. `score_range_groups`: every document whose best
page scores at least a threshold, in the same order (DESIGN §4).

Per-document caps (`score_topk_capped`, `score_topk_groups_pages`, `group_pages_topm` and the sharded forms): k pages with
at most m from any document, or the top-k documents each with its m best pages, with the bits of the fp32 scan (DESIGN §4).

Diverse retrieval (`score_mmr`, `mmr_select`): maximal marginal relevance over each query's top fetch_k pages, picked
on the GPU (vr_mmr_select) with the bits fixed by the definition in DESIGN §4.

Hybrid retrieval (`score_topk_hybrid`, `score_topk_groups_hybrid`): the dense score fused with an external score per
page (e.g. BM25 over OCR text), by weighted sum or reciprocal rank fusion, exactly over the whole index (DESIGN §4).

Sharded forms of range search, document range search, hybrid retrieval and MMR (`sharded_range`,
`sharded_range_groups`, `sharded_topk_hybrid`, `sharded_topk_groups_hybrid`, `sharded_mmr`): the bits of the plain call
over the shards concatenated in rank order, from each rank's local call, a few collectives and a merge (DESIGN §4).
"""
from __future__ import annotations

import ctypes as C
import glob
import os
import pickle
import weakref
from dataclasses import dataclass
from typing import Dict, List, Optional, Tuple

import numpy as np
import torch

from . import _lib as L

SMALL_PROBLEM = 1 << 22  # nq*nd below this: plain fp32 scan (the GEMM pipeline would not even fill)
SELECT_K_MIN = 32        # k above this (up to SELECT_K_MAX): the radix select vr_select_rows instead of the k-pass vr_topk_rows
SELECT_K_MAX = 4096
DEEP_K_MIN = 300         # k above this (up to DEEP_K_MAX): score_topk's deep route (DESIGN §4, "Deep top-k")
DEEP_K_MAX = 1024
DEEP_SAMPLE_RANK = 16    # the threshold is the sample's 16th exact score; a sample of every (k // 8)-th page puts it near
                         # rank 2k of the whole index


@dataclass
class CorpusIndex:
    """One corpus shard resident in HBM: fp32 embeddings (exact rescoring), fp16 copy (tensor-core filter)."""
    emb: torch.Tensor          # [nd, d] fp32
    emb_f16: torch.Tensor      # [nd, d] fp16
    max_norm: torch.Tensor     # [1] fp32: max row L2 norm (error bound of the filter)
    lookup: Optional[List[str]] = None

    @property
    def nd(self) -> int:
        return self.emb.shape[0]


def _check_f32(t: torch.Tensor, name: str) -> torch.Tensor:
    if not t.is_cuda:
        raise ValueError(f"{name} must be a CUDA tensor (visrag_b200 has no CPU path)")
    if t.dtype != torch.float32:
        t = t.float()
    return t.contiguous()


def to_f16_rows(x: torch.Tensor, want_max_norm: bool = False):
    """fp32 [n,d] -> fp16 copy (+ max row norm) with the library kernel."""
    n, d = x.shape
    out = torch.empty((n, d), dtype=torch.float16, device=x.device)
    mx = torch.zeros(1, dtype=torch.float32, device=x.device) if want_max_norm else None
    L.check(L.lib().vr_f32_to_f16_rows(x.data_ptr(), n, d, out.data_ptr(), None, L.ptr(mx), L.stream_ptr()))
    return (out, mx) if want_max_norm else out


def build_index(emb, lookup: Optional[List[str]] = None, device: str = "cuda") -> CorpusIndex:
    """numpy / torch fp32 [nd, d] -> device-resident index (a tensor stays on the device it lives on).
    The tensor-core filter's exactness proof needs finite fp16 copies of Q and D (|x| < 65504). The L2-normalised
    embeddings of the encoder always are; for anything else the rescoring kernel sees a query or max document row norm
    that is not < 65504 (inf / NaN included), flags the query, and `score_topk` reruns it through the plain fp32 scan."""
    if isinstance(emb, np.ndarray):
        emb = torch.from_numpy(np.ascontiguousarray(emb, dtype=np.float32)).to(L.norm_device(device))
    emb = _check_f32(emb, "emb")
    if emb.shape[1] % 8 != 0:
        raise ValueError("embedding dim must be a multiple of 8")
    with L.on_device(emb.device):
        f16, mx = to_f16_rows(emb, want_max_norm=True)
    return CorpusIndex(emb, f16, mx, lookup)


def pack_doc_mask(mask: torch.Tensor) -> torch.Tensor:
    """bool [nd] -> uint32 [ceil(nd / 32)] words on the same device: doc i is bit (i & 31) of word (i >> 5), the layout the
    _masked kernels read. Bits past nd are 0. bool [M, nd] -> uint32 [M, ceil(nd / 32)], row by row (a mask set)."""
    nd = mask.shape[-1]
    rows = mask.reshape(-1, nd)
    w = (nd + 31) // 32
    out = torch.empty((rows.shape[0], w * 4), dtype=torch.uint8, device=mask.device)
    weights = torch.ones(8, dtype=torch.uint8, device=mask.device) << torch.arange(8, dtype=torch.uint8, device=mask.device)
    step = max(1, (1 << 26) // (w * 32))  # rows per pass: <= 64 MiB of byte-per-bit scratch
    for r0 in range(0, rows.shape[0], step):
        part = rows[r0:r0 + step]
        bits = torch.zeros((part.shape[0], w * 32), dtype=torch.uint8, device=mask.device)
        bits[:, :nd] = part
        out[r0:r0 + step] = (bits.view(part.shape[0], w * 4, 8) * weights).sum(-1, dtype=torch.uint8)
    # little-endian bytes: byte j of a word holds docs 8j .. 8j + 7 of it
    return out.view(torch.int32).view(torch.uint32).reshape(*mask.shape[:-1], w)


@dataclass
class _MaskSet:
    """A packed mask set on the index's device: words uint32 [M, pitch], of_query int32 [nq] (None: mask 0 for every row)."""
    words: torch.Tensor
    of_query: Optional[torch.Tensor]

    def rows(self, sel: torch.Tensor) -> "_MaskSet":
        """The set of the query rows `sel` (an index tensor), each keeping its own mask."""
        return self if self.of_query is None else _MaskSet(self.words, self.of_query.index_select(0, sel))

    def arg(self, r0: int = 0):
        """The vr_doc_masks of the query rows from r0 on (a call over rows [r0, r0 + n) of the batch)."""
        m = L.DocMasks()
        m.words, m.pitch, m.count = self.words.data_ptr(), self.words.shape[1], self.words.shape[0]
        m.of_query = None if self.of_query is None else self.of_query[r0:].data_ptr()
        return C.byref(m)


def _check_doc_mask(doc_mask: torch.Tensor, index: CorpusIndex, nq: int, mask_of: Optional[torch.Tensor] = None) -> _MaskSet:
    """Validate a bool [nd] doc mask, or a bool [M, nd] mask set with its mask_of ([nq] ints in [0, M); None: query i
    uses row i, so M == nq), on the index's device, and pack it."""
    if not isinstance(doc_mask, torch.Tensor) or doc_mask.dtype != torch.bool:
        raise ValueError("doc_mask must be a torch.bool tensor")
    if doc_mask.dim() not in (1, 2) or doc_mask.shape[-1] != index.nd:
        raise ValueError(f"doc_mask must have shape [{index.nd}] or [M, {index.nd}] (one entry per doc of the index), "
                         f"got {list(doc_mask.shape)}")
    if doc_mask.device != index.emb.device:
        raise ValueError(f"doc_mask lives on {doc_mask.device}, the index on {index.emb.device}")
    if doc_mask.dim() == 1:
        if mask_of is not None:
            raise ValueError("mask_of picks rows of a 2-D doc_mask [M, nd]; this doc_mask is 1-D")
        return _MaskSet(pack_doc_mask(doc_mask).view(1, -1), None)
    M = doc_mask.shape[0]
    if mask_of is None:
        if M != nq:
            raise ValueError(f"doc_mask has {M} rows for {nq} queries: pass mask_of, or one mask row per query")
        of_query = torch.arange(nq, dtype=torch.int32, device=doc_mask.device)
    else:
        if not isinstance(mask_of, torch.Tensor) or mask_of.dtype not in (torch.int32, torch.int64):
            raise ValueError("mask_of must be an int32 or int64 torch tensor")
        if mask_of.dim() != 1 or mask_of.shape[0] != nq:
            raise ValueError(f"mask_of must have shape [{nq}] (one mask row per query), got {list(mask_of.shape)}")
        if mask_of.device != doc_mask.device:
            raise ValueError(f"mask_of lives on {mask_of.device}, doc_mask on {doc_mask.device}")
        if nq > 0:
            lo, hi = (int(v) for v in torch.aminmax(mask_of))
            if lo < 0 or hi >= M:
                raise ValueError(f"mask_of must lie in [0, {M}) (rows of doc_mask), got [{lo}, {hi}]")
        of_query = mask_of.to(torch.int32).contiguous()
    return _MaskSet(pack_doc_mask(doc_mask), of_query)


def _rows_fn(k: int, form: str = ""):
    """The row selection of k for the entry point form ("", "_masks", "_chunked", "_chunked_masks"): vr_select_rows for
    SELECT_K_MIN < k <= SELECT_K_MAX, else vr_topk_rows. Both take the same arguments and give the same bits."""
    name = "vr_select_rows" if SELECT_K_MIN < k <= SELECT_K_MAX else "vr_topk_rows"
    return getattr(L.lib(), name + form)


def _exact_topk(q: torch.Tensor, index: CorpusIndex, k: int, id_offset: int, masks: Optional[_MaskSet]):
    """The plain fp32 scan: (scores, ids)."""
    nq, d = q.shape
    nd = index.nd
    out_s = torch.empty((nq, k), dtype=torch.float32, device=q.device)
    out_i = torch.empty((nq, k), dtype=torch.int64, device=q.device)
    rows_per = max(1, min(nq, (1 << 28) // max(nd, 1)))  # <= 1 GiB of fp32 scratch
    scratch = torch.empty((rows_per, nd), dtype=torch.float32, device=q.device)
    lib = L.lib()
    for r0 in range(0, nq, rows_per):
        n = min(rows_per, nq - r0)
        mw = () if masks is None else (masks.arg(r0),)  # rows r0.. of the batch keep their own masks
        L.check(lib.vr_score_exact(q[r0:].data_ptr(), n, index.emb.data_ptr(), nd, d, scratch.data_ptr(), L.stream_ptr()))
        chunks = min(1024, nd // 4096) if n <= 64 else 0  # few queries over a long index: spread each row over many SMs
        if chunks >= 2:
            ws_s = torch.empty((n, chunks, k), dtype=torch.float32, device=q.device)
            ws_i = torch.empty((n, chunks, k), dtype=torch.int64, device=q.device)
            fn = _rows_fn(k, "_chunked_masks" if mw else "_chunked")
            args = (scratch.data_ptr(), n, nd, k, id_offset, chunks, ws_s.data_ptr(), ws_i.data_ptr())
        else:
            fn = _rows_fn(k, "_masks" if mw else "")
            args = (scratch.data_ptr(), None, n, nd, k, id_offset)
        L.check(fn(*args, out_s[r0:].data_ptr(), out_i[r0:].data_ptr(), *mw, L.stream_ptr()))
    return out_s, out_i


def score_topk(queries: torch.Tensor, index: CorpusIndex, k: int, id_offset: int = 0, force_exact: bool = False,
               stats: Optional[dict] = None, doc_mask: Optional[torch.Tensor] = None, mask_of: Optional[torch.Tensor] = None,
               doc_lists: Optional[Tuple[torch.Tensor, torch.Tensor]] = None, list_of: Optional[torch.Tensor] = None
               ) -> Tuple[torch.Tensor, torch.Tensor]:
    """Exact fp32 top-k of `queries @ index.emb.T`: (scores [nq,k] f32, ids [nq,k] i64 = local index + id_offset).
    Rows are sorted by (score desc, id asc); if k > nd the tail is (-inf, -1).
    doc_mask: optional bool [nd] on the index's device; only docs marked True are searched (the same bits as the fp32 scan
    over those docs alone). With fewer than k of them the tail is (-inf, -1).
    Per-query masks: doc_mask bool [M, nd] and mask_of int [nq] in [0, M) (default: row i for query i, M == nq); query i
    searches the docs of row mask_of[i], and its row equals its call alone with that row as a 1-D doc_mask.
    Candidate lists: doc_lists = (offsets int [M+1] from 0, non-decreasing; ids int32/int64 local doc ids) holds M lists in
    CSR form, list m = ids[offsets[m]:offsets[m+1]] (any order, repeats count once), and list_of int [nq] in [0, M) picks
    each query's list (default: list i for query i when M == nq, or the one list for every query when M == 1). Only the
    listed docs are read; each row equals this call with a doc_mask of exactly its list's docs. stats["path"] is "lists".
    doc_lists cannot be combined with doc_mask or mask_of.
    For DEEP_K_MIN < k <= DEEP_K_MAX (without lists) the rows go the deep route (_deep_topk): stats path "deep",
    sample_stride, candidates (rescored by the range filter) and fallback (rows rerun through the scan)."""
    if doc_lists is not None or list_of is not None:
        q, ls = _queries_and_lists(queries, index, doc_mask, mask_of, doc_lists, list_of)
        with L.on_device(q.device):
            return _lists_topk(q, index, k, id_offset, ls, None, stats)
    q, masks = _queries_and_mask(queries, index, doc_mask, mask_of)
    with L.on_device(q.device):
        return _score_topk(q, index, k, id_offset, force_exact, stats, masks)


def _queries_and_mask(queries: torch.Tensor, index: CorpusIndex, doc_mask: Optional[torch.Tensor],
                      mask_of: Optional[torch.Tensor] = None):
    """The queries as contiguous fp32 on the index's device, and the packed mask set (None: every doc)."""
    q = _check_f32(queries, "queries")
    if q.device != index.emb.device:
        raise ValueError(f"queries live on {q.device}, the index on {index.emb.device}")
    if doc_mask is None:
        if mask_of is not None:
            raise ValueError("mask_of needs a 2-D doc_mask [M, nd] to pick rows from")
        return q, None
    return q, _check_doc_mask(doc_mask, index, q.shape[0], mask_of)


@dataclass
class _ListSet:
    """A validated list set on the index's device: offsets int64 [M + 1], ids int32, of_query int32 [nq] (None: list 0 for
    every row), width = the longest list a query uses, sort = the rows must be grouped by list first (list_of given)."""
    offsets: torch.Tensor
    ids: torch.Tensor
    of_query: Optional[torch.Tensor]
    width: int
    sort: bool

    def arg(self, of_query: Optional[torch.Tensor], r0: int = 0):
        """The vr_doc_lists of the query rows from r0 on, of_query being this call's (possibly sorted) list of each row."""
        ls = L.DocLists()
        ls.offsets, ls.ids, ls.count = self.offsets.data_ptr(), self.ids.data_ptr(), self.offsets.shape[0] - 1
        ls.of_query = None if of_query is None else of_query[r0:].data_ptr()
        return C.byref(ls)

    def masks(self, nd: int) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
        """The equivalent (doc_mask, mask_of) of the masked calls: bool [nd] for one shared list, else bool [M, nd]."""
        M = self.offsets.shape[0] - 1
        lens = self.offsets[1:] - self.offsets[:-1]
        m = torch.zeros((M, nd), dtype=torch.bool, device=self.ids.device)
        m[torch.repeat_interleave(torch.arange(M, device=self.ids.device), lens), self.ids.long()] = True
        return (m[0], None) if self.of_query is None else (m, self.of_query)


def _int_tensor(t, name: str, shape: Optional[int], device) -> None:
    if not isinstance(t, torch.Tensor) or t.dtype not in (torch.int32, torch.int64):
        raise ValueError(f"{name} must be an int32 or int64 torch tensor")
    if t.dim() != 1 or (shape is not None and t.shape[0] != shape):
        want = f"[{shape}]" if shape is not None else "1-D"
        raise ValueError(f"{name} must have shape {want}, got {list(t.shape)}")
    if t.device != device:
        raise ValueError(f"{name} lives on {t.device}, the index on {device}")


def _check_doc_lists(doc_lists, index: CorpusIndex, nq: int, list_of: Optional[torch.Tensor] = None) -> _ListSet:
    """Validate doc_lists = (offsets, ids) and list_of on the index's device (one host read for all the value checks)."""
    if not isinstance(doc_lists, (tuple, list)) or len(doc_lists) != 2:
        raise ValueError("doc_lists must be a pair (offsets, ids) of int tensors")
    offsets, ids = doc_lists
    dev = index.emb.device
    _int_tensor(offsets, "doc_lists offsets", None, dev)
    _int_tensor(ids, "doc_lists ids", None, dev)
    M = offsets.shape[0] - 1
    if M < 1:
        raise ValueError("doc_lists offsets must have M + 1 >= 2 entries (M lists)")
    if list_of is None:
        if M not in (1, nq):
            raise ValueError(f"doc_lists has {M} lists for {nq} queries: pass list_of, one list per query, or one list")
        of_query = torch.arange(nq, dtype=torch.int32, device=dev) if M > 1 else None
    else:
        _int_tensor(list_of, "list_of", nq, dev)
        of_query = list_of.to(torch.int32).contiguous()
    offsets = offsets.to(torch.int64).contiguous()
    lens = offsets[1:] - offsets[:-1]
    used = lens if of_query is None else lens.index_select(0, of_query.clamp(0, M - 1).long())
    z = offsets.new_zeros(())
    vals = torch.stack([offsets[0], offsets[-1], lens.min(), used.max() if used.numel() else z,
                        ids.min().long() if ids.numel() else z, ids.max().long() if ids.numel() else z,
                        of_query.min().long() if nq and of_query is not None else z,
                        of_query.max().long() if nq and of_query is not None else z]).tolist()
    first, last, min_len, width, lo, hi, lq, hq = vals
    if first != 0:
        raise ValueError(f"doc_lists offsets must start at 0, got {first}")
    if min_len < 0:
        raise ValueError("doc_lists offsets must be non-decreasing")
    if last != ids.shape[0]:
        raise ValueError(f"doc_lists offsets must end at len(ids) = {ids.shape[0]}, got {last}")
    if ids.numel() and (lo < 0 or hi >= index.nd):
        raise ValueError(f"doc_lists ids must lie in [0, {index.nd}) (local docs of the index), got [{lo}, {hi}]")
    if list_of is not None and nq and (lq < 0 or hq >= M):
        raise ValueError(f"list_of must lie in [0, {M}) (lists of doc_lists), got [{lq}, {hq}]")
    ids = ids.to(torch.int32).contiguous() if ids.numel() else torch.zeros(1, dtype=torch.int32, device=dev)  # never read
    return _ListSet(offsets, ids, of_query, max(1, width), list_of is not None)


def _queries_and_lists(queries, index: CorpusIndex, doc_mask, mask_of, doc_lists, list_of):
    """The queries (as _queries_and_mask) and the validated list set."""
    if doc_mask is not None or mask_of is not None:
        raise ValueError("doc_lists cannot be combined with doc_mask or mask_of")
    if doc_lists is None:
        raise ValueError("list_of needs doc_lists to pick lists from")
    q, _ = _queries_and_mask(queries, index, None)
    return q, _check_doc_lists(doc_lists, index, q.shape[0], list_of)


LIST_CHUNK = 4096  # list positions per first-level row of the page selection (the chunked scan's 4096 columns a block)


def _lists_topk(q: torch.Tensor, index: CorpusIndex, k: int, id_offset: int, ls: _ListSet, gt: Optional["_GroupTable"],
                stats: Optional[dict]):
    """Top-k over candidate lists: vr_score_lists writes each row's listed (score, id[, group]) entries into a padded
    [n, W] block, and the selection kernels of the masked path pick from it. Pages: vr_topk_rows, in two levels when W
    > LIST_CHUNK ([n * C, LIST_CHUNK] rows with id_offset 0, then their [n, C * k] lists). Documents (k <= 256):
    vr_merge_group_topk over [n * C, 512] rows, repeated over the [n, C * k] results until a row fits 512 entries."""
    nq, d = q.shape
    grouped = gt is not None
    dtypes = (torch.float32, torch.int64) if not grouped else (torch.float32, torch.int64, torch.int64)
    out = tuple(torch.empty((nq, k), dtype=t, device=q.device) for t in dtypes)
    if stats is not None:
        stats.update(path="lists", flagged=0)
    if nq == 0:
        return out
    if d != index.emb.shape[1]:
        raise ValueError("query / corpus dim mismatch")
    lib, sp = L.lib(), L.stream_ptr()
    of, order = ls.of_query, None
    if ls.sort:  # rows of one list next to each other, so that a tile of queries reads each listed row once
        order = torch.sort(of, stable=True).indices
        q, of = q.index_select(0, order), of.index_select(0, order)
    step = MERGE_GROUPS_MAX if grouped else LIST_CHUNK
    W = ls.width if ls.width <= step else -(-ls.width // step) * step
    rows_per = max(1, min(nq, (1 << 30) // (W * (20 if grouped else 12))))  # <= 1 GiB of [n, W] entries
    sc = torch.empty((rows_per, W), dtype=torch.float32, device=q.device)
    si = torch.empty((rows_per, W), dtype=torch.int64, device=q.device)
    sg = torch.empty((rows_per, W), dtype=torch.int64, device=q.device) if grouped else None
    status = torch.zeros(1, dtype=torch.int32, device=q.device)
    for r0 in range(0, nq, rows_per):
        n = min(rows_per, nq - r0)
        L.check(lib.vr_score_lists(q[r0:].data_ptr(), n, index.emb.data_ptr(), index.nd, d, ls.arg(of, r0), W,
                                   gt.groups.data_ptr() if grouped else None, sc.data_ptr(), si.data_ptr(), L.ptr(sg),
                                   status.data_ptr(), sp))
        if grouped:
            _merge_group_levels(sc[:n], si[:n], sg[:n], k, [t[r0:r0 + n] for t in out])
        elif W <= LIST_CHUNK:
            L.check(_rows_fn(k)(sc.data_ptr(), si.data_ptr(), n, W, k, id_offset, out[0][r0:].data_ptr(),
                                out[1][r0:].data_ptr(), sp))
        else:
            c = W // LIST_CHUNK
            ws_s = torch.empty((n * c, k), dtype=torch.float32, device=q.device)
            ws_i = torch.empty((n * c, k), dtype=torch.int64, device=q.device)
            L.check(_rows_fn(k)(sc.data_ptr(), si.data_ptr(), n * c, LIST_CHUNK, k, 0, ws_s.data_ptr(), ws_i.data_ptr(), sp))
            L.check(_rows_fn(k)(ws_s.data_ptr(), ws_i.data_ptr(), n, c * k, k, id_offset, out[0][r0:].data_ptr(),
                                out[1][r0:].data_ptr(), sp))
    bad = int(status.item())  # host sync: the caller reads the result next anyway
    if bad:
        raise RuntimeError(f"vr_score_lists reported status {bad} (a list longer than its width, or a list index out of range)")
    if grouped and id_offset:
        out[1].add_(torch.where(out[1] >= 0, id_offset, 0))
    if order is None:
        return out
    res = tuple(torch.empty_like(t) for t in out)
    for r, t in zip(res, out):
        r.index_copy_(0, order, t)
    return res


def _merge_group_levels(s: torch.Tensor, p: torch.Tensor, g: torch.Tensor, k: int, out) -> None:
    """[n, W] (score, page, group) entries -> the first k distinct groups of each row in (score desc, page asc) order.
    A group of the row's top-k has fewer than k groups ahead of it in the chunk that holds its best page, so it is among
    that chunk's first k distinct groups: merging the chunks' lists again is exact, and each level shrinks a row by
    512 / k (k <= 256)."""
    lib, sp = L.lib(), L.stream_ptr()
    n = s.shape[0]
    while s.shape[1] > MERGE_GROUPS_MAX:
        c = s.shape[1] // MERGE_GROUPS_MAX  # the width is a multiple of 512 here
        nxt = (torch.empty((n * c, k), dtype=torch.float32, device=s.device),
               torch.empty((n * c, k), dtype=torch.int64, device=s.device),
               torch.empty((n * c, k), dtype=torch.int64, device=s.device))
        L.check(lib.vr_merge_group_topk(s.data_ptr(), p.data_ptr(), g.data_ptr(), n * c, MERGE_GROUPS_MAX, k,
                                        *[t.data_ptr() for t in nxt], sp))
        s, p, g = (t.view(n, c * k) for t in nxt)
        pad = -s.shape[1] % MERGE_GROUPS_MAX if s.shape[1] > MERGE_GROUPS_MAX else 0
        if pad:
            s = torch.nn.functional.pad(s, (0, pad), value=float("-inf"))
            p, g = (torch.nn.functional.pad(t, (0, pad), value=-1) for t in (p, g))
    s, p, g = s.contiguous(), p.contiguous(), g.contiguous()
    L.check(lib.vr_merge_group_topk(s.data_ptr(), p.data_ptr(), g.data_ptr(), n, s.shape[1], k,
                                    *[t.data_ptr() for t in out], sp))


class _Stages:
    """Optional per-stage CUDA-event timing: pass stats={"stages": {}} and read stats["stages"] (ms) after a synchronize."""

    def __init__(self, stats: Optional[dict]):
        self.on = stats is not None and "stages" in stats
        self.stats = stats
        if self.on:
            self.last = torch.cuda.Event(enable_timing=True)
            self.last.record()
            stats.setdefault("_events", [])

    def mark(self, name: str) -> None:
        if self.on:
            e = torch.cuda.Event(enable_timing=True)
            e.record()
            self.stats["_events"].append((name, self.last, e))
            self.last = e


def resolve_stages(stats: dict) -> dict:
    """After torch.cuda.synchronize(): turn the recorded event pairs into stats["stages"][name] += ms."""
    for name, e0, e1 in stats.pop("_events", []):
        stats["stages"][name] = stats["stages"].get(name, 0.0) + e0.elapsed_time(e1)
    return stats["stages"]


def _score_topk(q: torch.Tensor, index: CorpusIndex, k: int, id_offset: int, force_exact: bool, stats: Optional[dict],
                masks: Optional[_MaskSet], gt: Optional[_GroupTable] = None, page_lists: bool = False):
    """The filter + rescoring pipeline. Pages (gt None): (scores, ids); groups (gt, the group table): (scores, best pages,
    groups). masks: the packed mask set (None: every doc). page_lists: feed the page filter's lists to the grouped
    rescoring (tests and measurements of the proof)."""
    nq, d = q.shape
    nd = index.nd

    def exact(rows: torch.Tensor, m: Optional[_MaskSet]):
        if gt is None:
            return _exact_topk(rows, index, k, id_offset, m)
        return _exact_topk_groups(rows, index, k, id_offset, m, gt)

    def outputs(n: int):
        dtypes = (torch.float32, torch.int64) if gt is None else (torch.float32, torch.int64, torch.int64)
        return tuple([torch.empty((n, k), dtype=t, device=q.device) for t in dtypes])

    if nq == 0:
        return outputs(0)
    if d != index.emb.shape[1]:
        raise ValueError("query / corpus dim mismatch")
    if force_exact or nq * nd <= SMALL_PROBLEM or nd < 256:
        if stats is not None:
            stats.update(path="exact", flagged=0)
        return exact(q, masks)
    if not page_lists and DEEP_K_MIN < k <= DEEP_K_MAX:
        return _deep_topk(q, index, k, id_offset, stats, masks, gt)
    lib = L.lib()
    ranges = lib.vr_score_ranges(nq, nd)
    lists = ranges * 2 * lib.vr_score_list_len()
    q16 = to_f16_rows(q)
    cand_s = torch.empty((nq, lists), dtype=torch.float32, device=q.device)
    cand_i = torch.empty((nq, lists), dtype=torch.int32, device=q.device)
    out = outputs(nq)
    flags = torch.empty((nq,), dtype=torch.int32, device=q.device)
    sp = L.stream_ptr()
    ev = _Stages(stats)
    ev.mark("q_to_f16")
    filt = (q16.data_ptr(), nq, index.emb_f16.data_ptr(), nd, d, ranges, cand_s.data_ptr(), cand_i.data_ptr())
    if gt is not None and not page_lists:
        if masks is None:
            L.check(lib.vr_score_filter_groups(*filt, gt.groups.data_ptr(), None, sp))
        else:
            L.check(lib.vr_score_filter_groups_masks(*filt, gt.groups.data_ptr(), masks.arg(), sp))
    elif masks is None:
        L.check(lib.vr_score_filter(*filt, sp))
    else:
        L.check(lib.vr_score_filter_masks(*filt, masks.arg(), sp))
    ev.mark("filter")
    cand = (q.data_ptr(), nq, index.emb.data_ptr(), nd, d, ranges, cand_s.data_ptr(), cand_i.data_ptr())
    tail = (index.max_norm.data_ptr(), k, id_offset, *[t.data_ptr() for t in out], flags.data_ptr(), sp)
    if gt is None:
        L.check(lib.vr_score_rescore(*cand, *tail))  # a masked filter's lists hold each query's eligible docs only
    else:
        csr = (gt.groups.data_ptr(), gt.offsets.data_ptr(), gt.pages.data_ptr(), gt.G)
        if masks is None:
            L.check(lib.vr_score_rescore_groups(*cand, *csr, None, *tail))
        else:
            L.check(lib.vr_score_rescore_groups_masks(*cand, *csr, masks.arg(), *tail))
    ev.mark("rescore")
    bad = torch.nonzero(flags).flatten()  # host sync: the caller reads the result next anyway
    if stats is not None:
        stats.update(path="filter+rescore", flagged=int(bad.numel()), ranges=ranges)
    if bad.numel() > 0:
        # each flagged row reruns with its own mask; many rows at a deep k take the deep route, which is exact as well
        rows, m = q.index_select(0, bad), None if masks is None else masks.rows(bad)
        deep = not page_lists and SELECT_K_MIN < k <= DEEP_K_MAX and bad.numel() * nd > SMALL_PROBLEM
        for t, fix in zip(out, _deep_topk(rows, index, k, id_offset, None, m, gt) if deep else exact(rows, m)):
            t.index_copy_(0, bad, fix)
    return out


# ------------------------------------------------------------------------------------------------------
# Document-level top-k: groups of pages, each scored by its best page
# ------------------------------------------------------------------------------------------------------
@dataclass
class _GroupTable:
    groups: torch.Tensor    # [nd] int32: the group of each page
    offsets: torch.Tensor   # [G+1] int32: group g owns pages[offsets[g]:offsets[g+1]]
    pages: torch.Tensor     # [nd] int32: pages by group, ascending within a group
    G: int
    max_pages: int          # pages of the largest group (the pieces of vr_group_pages_topm)


MERGE_GROUPS_MAX = 512  # entries per row vr_merge_group_topk takes: world * k of sharded_topk_groups
LIST_GROUPS_MAX_K = MERGE_GROUPS_MAX // 2  # the list path's group merge shrinks a row by 512 / k per level
_GROUP_TABLES: Dict[int, Tuple["weakref.ref", int, _GroupTable]] = {}


def _group_table(doc_groups: torch.Tensor, index: CorpusIndex) -> _GroupTable:
    """Validate doc_groups and build its CSR on the device (a stable sort keeps pages ascending within a group). Cached per
    tensor object until it is freed or modified in place: keep one tensor for repeated searches (a new slice or view per
    call is a new object and builds the CSR again). The table holds its own copy of the groups, never the key itself,
    so the entry goes when the caller's tensor does."""
    if not isinstance(doc_groups, torch.Tensor) or doc_groups.dtype not in (torch.int32, torch.int64):
        raise ValueError("doc_groups must be an int32 or int64 torch tensor")
    if doc_groups.dim() != 1 or doc_groups.shape[0] != index.nd:
        raise ValueError(f"doc_groups must have shape [{index.nd}] (one group per doc of the index), got {list(doc_groups.shape)}")
    if doc_groups.device != index.emb.device:
        raise ValueError(f"doc_groups lives on {doc_groups.device}, the index on {index.emb.device}")
    hit = _GROUP_TABLES.get(id(doc_groups))
    if hit is not None and hit[0]() is doc_groups and hit[1] == doc_groups._version:
        return hit[2]
    lo, hi = (int(v) for v in torch.aminmax(doc_groups))
    if lo < 0 or hi >= 1 << 31:
        raise ValueError(f"doc_groups must lie in [0, 2^31), got [{lo}, {hi}]")
    G = hi + 1
    order = torch.sort(doc_groups, stable=True).indices
    counts = torch.bincount(doc_groups, minlength=G)
    offsets = torch.zeros(G + 1, dtype=torch.int64, device=doc_groups.device)
    offsets[1:] = torch.cumsum(counts, 0)
    table = _GroupTable(doc_groups.to(torch.int32, copy=True).contiguous(), offsets.to(torch.int32), order.to(torch.int32), G,
                        int(counts.max()))
    key = id(doc_groups)
    _GROUP_TABLES[key] = (weakref.ref(doc_groups, lambda _r, key=key: _GROUP_TABLES.pop(key, None)), doc_groups._version, table)
    return table


def _exact_topk_groups(q: torch.Tensor, index: CorpusIndex, k: int, id_offset: int, masks: Optional[_MaskSet],
                       gt: _GroupTable):
    """The plain fp32 scan, reduced per group: (scores, best pages, groups)."""
    nq, d = q.shape
    nd = index.nd
    out_s = torch.empty((nq, k), dtype=torch.float32, device=q.device)
    out_p = torch.empty((nq, k), dtype=torch.int64, device=q.device)
    out_g = torch.empty((nq, k), dtype=torch.int64, device=q.device)
    # <= 512 MiB of fp32 scores + 1.5 GiB of per-group workspace (G may exceed nd: global group ids on one shard)
    rows_per = max(1, min(nq, (1 << 27) // max(nd, gt.G, 1)))
    scratch = torch.empty((rows_per, nd), dtype=torch.float32, device=q.device)
    lib = L.lib()
    for r0 in range(0, nq, rows_per):
        n = min(rows_per, nq - r0)
        L.check(lib.vr_score_exact(q[r0:].data_ptr(), n, index.emb.data_ptr(), nd, d, scratch.data_ptr(), L.stream_ptr()))
        chunks = min(1024, gt.G // 4096) if n <= 64 else 0  # few queries over many groups: spread each row over many SMs
        ws_bytes = lib.vr_group_topk_ws_bytes(n, gt.G, k, chunks)
        ws = torch.empty((ws_bytes + 15) // 16 * 2, dtype=torch.float64, device=q.device)  # 16-byte aligned
        fn, mw = (lib.vr_group_topk_rows, None) if masks is None else (lib.vr_group_topk_rows_masks, masks.arg(r0))
        L.check(fn(scratch.data_ptr(), n, nd, gt.groups.data_ptr(), gt.G, mw, k, id_offset, chunks, ws.data_ptr(), ws_bytes,
                   out_s[r0:].data_ptr(), out_p[r0:].data_ptr(), out_g[r0:].data_ptr(), L.stream_ptr()))
    return out_s, out_p, out_g


def score_topk_groups(queries: torch.Tensor, index: CorpusIndex, k: int, doc_groups: torch.Tensor, id_offset: int = 0,
                      force_exact: bool = False, stats: Optional[dict] = None, doc_mask: Optional[torch.Tensor] = None,
                      mask_of: Optional[torch.Tensor] = None, doc_lists: Optional[Tuple[torch.Tensor, torch.Tensor]] = None,
                      list_of: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """Exact top-k GROUPS (documents) of pages: doc_groups (int32/int64 [nd] on the index's device) gives each page its
    group in [0, G). A group's score is the maximum exact fp32 page score over its eligible pages, its best page the lowest
    page with that maximum; groups rank by (score desc, best page asc). Returns (scores [nq,k] f32, best pages [nq,k] i64
    = local index + id_offset, groups [nq,k] i64); fewer than k groups with an eligible page leave (-inf, -1, -1).
    With doc_groups = arange(nd) the result equals score_topk's, with groups == pages. doc_mask and mask_of as in score_topk
    (per-query masks: each query's documents are scored by its own eligible pages). doc_lists and list_of as in
    score_topk: each query's documents are scored by the pages of its list; k > 256 takes the masked path with the
    equivalent masks (the same result)."""
    if doc_lists is not None or list_of is not None:
        q, ls = _queries_and_lists(queries, index, doc_mask, mask_of, doc_lists, list_of)
        with L.on_device(q.device):
            gt = _group_table(doc_groups, index)
            if k <= LIST_GROUPS_MAX_K:
                return _lists_topk(q, index, k, id_offset, ls, gt, stats)
            doc_mask, mask_of = ls.masks(index.nd)
            return _score_topk_groups(q, index, k, id_offset, force_exact, stats, gt,
                                      _check_doc_mask(doc_mask, index, q.shape[0], mask_of))
    q, masks = _queries_and_mask(queries, index, doc_mask, mask_of)
    with L.on_device(q.device):
        gt = _group_table(doc_groups, index)
        return _score_topk_groups(q, index, k, id_offset, force_exact, stats, gt, masks)


def _score_topk_groups(q, index, k, id_offset, force_exact, stats, gt: _GroupTable, masks, page_lists: bool = False):
    """_score_topk for groups. page_lists=True is the entry of the tests and measurements of the proof on page lists."""
    return _score_topk(q, index, k, id_offset, force_exact, stats, masks, gt, page_lists)


def merge_topk_groups(scores: torch.Tensor, pages: torch.Tensor, groups: torch.Tensor, k: int):
    """[nq, m] partial group lists (score, page, group; page < 0 = empty) -> the first k distinct groups in
    (score desc, page asc) order. m <= MERGE_GROUPS_MAX (the merge keeps a row in one warp's registers)."""
    if scores.shape[1] > MERGE_GROUPS_MAX:
        raise ValueError(f"merge_topk_groups merges at most {MERGE_GROUPS_MAX} entries per row (world * k), got {scores.shape[1]}")
    scores = scores.contiguous().float()
    pages = pages.contiguous().to(torch.int64)
    groups = groups.contiguous().to(torch.int64)
    nq, m = scores.shape
    out_s = torch.empty((nq, k), dtype=torch.float32, device=scores.device)
    out_p = torch.empty((nq, k), dtype=torch.int64, device=scores.device)
    out_g = torch.empty((nq, k), dtype=torch.int64, device=scores.device)
    with L.on_device(scores.device):
        L.check(L.lib().vr_merge_group_topk(scores.data_ptr(), pages.data_ptr(), groups.data_ptr(), nq, m, k, out_s.data_ptr(),
                                            out_p.data_ptr(), out_g.data_ptr(), L.stream_ptr()))
    return out_s, out_p, out_g


def merge_topk(scores: torch.Tensor, ids: torch.Tensor, k: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """[nq, m] candidate (score, id) pairs (id < 0 = empty) -> top-k by (score desc, id asc)."""
    scores = scores.contiguous().float()
    ids = ids.contiguous().to(torch.int64)
    nq, m = scores.shape
    out_s = torch.empty((nq, k), dtype=torch.float32, device=scores.device)
    out_i = torch.empty((nq, k), dtype=torch.int64, device=scores.device)
    with L.on_device(scores.device):
        L.check(_rows_fn(k)(scores.data_ptr(), ids.data_ptr(), nq, m, k, 0, out_s.data_ptr(), out_i.data_ptr(),
                            L.stream_ptr()))
    return out_s, out_i


# ------------------------------------------------------------------------------------------------------
# Per-document caps: capped page top-k and inner hits (DESIGN §4)
# ------------------------------------------------------------------------------------------------------
GROUP_PAGES_MAX = 256   # m (pages per document) vr_group_pages_topm keeps
GROUP_PIECE = 256       # pages of one document a block of vr_group_pages_topm scores
GROUP_STAGE_BUDGET = 1 << 26  # [rows, kg, pieces, m] entries of the stage per pass: query rows go in chunks


def _check_per_group(v, name: str) -> int:
    v = _check_count(v, name)
    if v < 1:
        raise ValueError(f"{name}={v} must be at least 1")
    return v


def _check_pages(m) -> int:
    m = _check_per_group(m, "pages")
    if m > GROUP_PAGES_MAX:
        raise ValueError(f"pages={m} must lie in [1, {GROUP_PAGES_MAX}]")
    return m


def _group_pages_topm(q: torch.Tensor, index: CorpusIndex, groups: torch.Tensor, gt: _GroupTable, m: int, id_offset: int,
                      masks: Optional[_MaskSet]) -> Tuple[torch.Tensor, torch.Tensor]:
    """vr_group_pages_topm over every (row, slot) of groups [nq, kg] (int64), with the pieces of long documents reduced
    to each document's m best by vr_topk_rows: (scores [nq, kg, m], pages [nq, kg, m] = page + id_offset)."""
    nq, kg = groups.shape
    dev = q.device
    out_s = torch.empty((nq, kg, m), dtype=torch.float32, device=dev)
    out_p = torch.empty((nq, kg, m), dtype=torch.int64, device=dev)
    if nq == 0:
        return out_s, out_p
    if q.shape[1] != index.emb.shape[1]:
        raise ValueError("query / corpus dim mismatch")
    piece = max(1, min(GROUP_PIECE, gt.max_pages))
    pieces = max(1, -(-gt.max_pages // piece))
    lib, sp = L.lib(), L.stream_ptr()
    rows_per = max(1, min(nq, GROUP_STAGE_BUDGET // (kg * pieces * m)))
    ws_s = torch.empty((rows_per, kg, pieces, m), dtype=torch.float32, device=dev) if pieces > 1 else None
    ws_p = torch.empty((rows_per, kg, pieces, m), dtype=torch.int64, device=dev) if pieces > 1 else None
    for r0 in range(0, nq, rows_per):
        n = min(rows_per, nq - r0)
        s, p = (out_s[r0:], out_p[r0:]) if pieces == 1 else (ws_s, ws_p)
        L.check(lib.vr_group_pages_topm(q[r0:].data_ptr(), n, index.emb.data_ptr(), index.nd, q.shape[1],
                                        groups[r0:].data_ptr(), kg, gt.offsets.data_ptr(), gt.pages.data_ptr(), gt.G,
                                        None if masks is None else masks.arg(r0), m, piece, pieces, id_offset, s.data_ptr(),
                                        p.data_ptr(), sp))
        if pieces > 1:
            L.check(lib.vr_topk_rows(ws_s.data_ptr(), ws_p.data_ptr(), n * kg, pieces * m, m, 0, out_s[r0:].data_ptr(),
                                     out_p[r0:].data_ptr(), sp))
    return out_s, out_p


def group_pages_topm(queries: torch.Tensor, index: CorpusIndex, groups: torch.Tensor, doc_groups: torch.Tensor, m: int,
                     id_offset: int = 0, doc_mask: Optional[torch.Tensor] = None, mask_of: Optional[torch.Tensor] = None
                     ) -> Tuple[torch.Tensor, torch.Tensor]:
    """The m best eligible pages of given documents: groups int [nq, kg] on the index's device (e.g. the groups of
    score_topk_groups; a value outside [0, G) is an empty document) -> (scores [nq, kg, m] f32, pages [nq, kg, m] i64 =
    local page + id_offset), each (row, slot) the document's pages in (exact fp32 score desc, page asc) order, ending in
    (-inf, -1). Scores have the bits of the fp32 scan; NaN is never selected. doc_mask / mask_of as in score_topk."""
    m = _check_pages(m)
    q, masks = _queries_and_mask(queries, index, doc_mask, mask_of)
    if not isinstance(groups, torch.Tensor) or groups.dtype not in (torch.int32, torch.int64) or groups.dim() != 2:
        raise ValueError("groups must be an int32 or int64 torch tensor [nq, kg]")
    if groups.shape[0] != q.shape[0] or groups.shape[1] < 1:
        raise ValueError(f"groups must have shape [{q.shape[0]}, kg >= 1] (one row per query), got {list(groups.shape)}")
    if groups.device != index.emb.device:
        raise ValueError(f"groups live on {groups.device}, the index on {index.emb.device}")
    with L.on_device(q.device):
        gt = _group_table(doc_groups, index)
        return _group_pages_topm(q, index, groups.to(torch.int64).contiguous(), gt, m, id_offset, masks)


def _stage_masks(q: torch.Tensor, index: CorpusIndex, doc_mask, mask_of, doc_lists, list_of) -> Optional[_MaskSet]:
    """The mask set of the stage for a search's scope: the masks themselves, or the masks equivalent to doc_lists."""
    if doc_lists is not None or list_of is not None:
        _, ls = _queries_and_lists(q, index, doc_mask, mask_of, doc_lists, list_of)
        doc_mask, mask_of = ls.masks(index.nd)
    return _queries_and_mask(q, index, doc_mask, mask_of)[1]


def score_topk_groups_pages(queries: torch.Tensor, index: CorpusIndex, k: int, doc_groups: torch.Tensor, pages: int,
                            id_offset: int = 0, force_exact: bool = False, stats: Optional[dict] = None,
                            doc_mask: Optional[torch.Tensor] = None, mask_of: Optional[torch.Tensor] = None,
                            doc_lists: Optional[Tuple[torch.Tensor, torch.Tensor]] = None,
                            list_of: Optional[torch.Tensor] = None):
    """Inner hits: the top-k documents of score_topk_groups (same arguments, same result), each with its `pages` best
    eligible pages. Returns (scores [nq,k] f32, best pages [nq,k] i64, groups [nq,k] i64, page scores [nq,k,pages] f32,
    pages [nq,k,pages] i64 = local page + id_offset); column 0 is the best page and its score, a document with fewer
    pages and a missing document end in (-inf, -1). stats: score_topk_groups', and with stats={"stages": {}} the
    CUDA-event times of "documents" and "pages"."""
    m = _check_pages(pages)
    q = _check_f32(queries, "queries")
    ev = _Stages(stats)
    s, p, g = score_topk_groups(q, index, k, doc_groups, id_offset, force_exact, stats, doc_mask, mask_of, doc_lists, list_of)
    ev.mark("documents")
    with L.on_device(q.device):
        masks = _stage_masks(q, index, doc_mask, mask_of, doc_lists, list_of)
        ps, pp = _group_pages_topm(q, index, g, _group_table(doc_groups, index), m, id_offset, masks)
    ev.mark("pages")
    return s, p, g, ps, pp


def _capped_merge(scores: torch.Tensor, pages: torch.Tensor, groups: torch.Tensor, k: int):
    """[nq, n] distinct candidate pages (score, page, group; page < 0 = empty) -> the top-k pages by (score desc,
    page asc) with their groups: (scores, pages, groups) [nq, k]."""
    nq = scores.shape[0]
    if nq == 0 or scores.shape[1] == 0:
        e = torch.full((nq, k), -1, dtype=torch.int64, device=scores.device)
        return torch.full((nq, k), float("-inf"), device=scores.device), e, e.clone()
    s, p = merge_topk(scores, pages, k)
    key, order = torch.sort(pages.to(torch.int64), dim=1)  # each page appears once: find each pick's candidate
    at = torch.searchsorted(key, p).clamp(max=key.shape[1] - 1)
    g = torch.gather(groups.to(torch.int64), 1, torch.gather(order, 1, at))
    return s, p, torch.where(p >= 0, g, -1)


def score_topk_capped(queries: torch.Tensor, index: CorpusIndex, k: int, doc_groups: torch.Tensor, per_group: int,
                      id_offset: int = 0, force_exact: bool = False, stats: Optional[dict] = None,
                      doc_mask: Optional[torch.Tensor] = None, mask_of: Optional[torch.Tensor] = None,
                      doc_lists: Optional[Tuple[torch.Tensor, torch.Tensor]] = None, list_of: Optional[torch.Tensor] = None
                      ) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """Capped page top-k: walk the eligible pages in (exact fp32 score desc, page asc) order and pick each page whose
    document has fewer than per_group picks, until k picks. Returns (scores [nq,k] f32, pages [nq,k] i64 = local page +
    id_offset, groups [nq,k] i64) in pick order, ending in (-inf, -1, -1) when the caps leave fewer than k pages. Scope
    arguments as in score_topk_groups. per_group = 1 gives score_topk_groups' result; per_group >= k can not bind and is
    answered by score_topk. Otherwise (DESIGN §4): the top-k documents, the per_group best pages of each
    (vr_group_pages_topm), and the top-k of those k * per_group pages. stats: the searches', and with
    stats={"stages": {}} the CUDA-event times of "documents", "pages" and "merge"."""
    m = _check_per_group(per_group, "per_group")
    k = _check_count(k, "k")
    if m >= k:
        q = _check_f32(queries, "queries")
        s, p = score_topk(q, index, k, id_offset, force_exact, stats, doc_mask, mask_of, doc_lists, list_of)
        with L.on_device(q.device):
            gt = _group_table(doc_groups, index)
            return s, p, torch.where(p >= 0, gt.groups[(p - id_offset).clamp(min=0)].long(), -1)
    if m > GROUP_PAGES_MAX:
        raise ValueError(f"per_group={m} must be >= k or lie in [1, {GROUP_PAGES_MAX}]")
    _, _, g, ps, pp = score_topk_groups_pages(queries, index, k, doc_groups, m, id_offset, force_exact, stats, doc_mask,
                                              mask_of, doc_lists, list_of)
    ev = _Stages(stats)
    with L.on_device(ps.device):
        nq = ps.shape[0]
        out = _capped_merge(ps.view(nq, k * m), pp.view(nq, k * m), g[:, :, None].expand(nq, k, m).reshape(nq, k * m), k)
    ev.mark("merge")
    return out


# ------------------------------------------------------------------------------------------------------
# Range search: every page scoring at least a threshold
# ------------------------------------------------------------------------------------------------------
RANGE_CAP = 16384          # candidate slots per query row of the filter path; a row with more reruns through the scan
RANGE_SORT_SMEM = 4096     # rows of up to this many entries are ordered in shared memory (vr_range_sort)
RANGE_BUDGET = 1 << 26     # entries of scratch per pass: query rows are processed in chunks of this many (row x slot)


def _check_min_score(min_score, nq: int, device) -> torch.Tensor:
    """min_score as an f32 [nq] tensor on the index's device: a float for every query, or an f32 tensor [nq]."""
    if isinstance(min_score, torch.Tensor):
        if min_score.dtype != torch.float32:
            raise ValueError(f"min_score must be a float or a torch.float32 tensor, got {min_score.dtype}")
        if min_score.dim() != 1 or min_score.shape[0] != nq:
            raise ValueError(f"min_score must have shape [{nq}] (one threshold per query), got {list(min_score.shape)}")
        if min_score.device != device:
            raise ValueError(f"min_score lives on {min_score.device}, the index on {device}")
        t = min_score.contiguous()
        if nq and bool(torch.isnan(t).any()):
            raise ValueError("min_score must not be NaN")
        return t
    if isinstance(min_score, bool) or not isinstance(min_score, (int, float, np.floating, np.integer)):
        raise ValueError(f"min_score must be a float or a torch.float32 tensor, got {type(min_score).__name__}")
    if np.isnan(min_score):
        raise ValueError("min_score must not be NaN")
    return torch.full((nq,), float(min_score), dtype=torch.float32, device=device)


def _check_cap(cap: Optional[int]) -> int:
    if cap is None:
        return RANGE_CAP
    if isinstance(cap, bool) or not isinstance(cap, (int, np.integer)) or cap < 1 or cap >= 1 << 31:
        raise ValueError(f"cap must be an int in [1, 2^31), got {cap!r}")
    return int(cap)


def score_range(queries: torch.Tensor, index: CorpusIndex, min_score, id_offset: int = 0,
                doc_mask: Optional[torch.Tensor] = None, mask_of: Optional[torch.Tensor] = None, force_exact: bool = False,
                stats: Optional[dict] = None, cap: Optional[int] = None
                ) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """Range search: for query i, every eligible doc j with exact fp32 score s_ij >= t_i, where t = min_score (a float
    for every query, or an f32 tensor [nq] on the index's device; NaN is refused). Returns CSR on the index's device:
    (offsets int64 [nq + 1], scores f32 [R], ids int64 [R] = local index + id_offset); row i is
    [offsets[i], offsets[i + 1]), ordered by (score desc, id asc). Scores have the bits of the fp32 scan; NaN scores never
    qualify, t = -inf returns every eligible doc and t = +inf only +inf scores. doc_mask / mask_of as in score_topk.
    The tensor-core filter keeps every doc whose approximate score is >= t - eps (eps: the filter's error bound, DESIGN
    §4), so its candidates hold every result; they are rescored exactly. A query with more than `cap` candidates
    (default RANGE_CAP), or whose norms allow no bound, reruns through the fp32 scan, as do small problems and
    force_exact. stats: path ("exact" or "filter+rescore"), candidates (rescored: the filter's candidates of the rows
    that did not overflow), fallback (rows rerun through the scan), cap."""
    q, masks = _queries_and_mask(queries, index, doc_mask, mask_of)
    t = _check_min_score(min_score, q.shape[0], index.emb.device)
    cap = _check_cap(cap)
    with L.on_device(q.device):
        return _score_range(q, index, t, id_offset, masks, force_exact, stats, cap)


def score_range_groups(queries: torch.Tensor, index: CorpusIndex, min_score, doc_groups: torch.Tensor, id_offset: int = 0,
                       doc_mask: Optional[torch.Tensor] = None, mask_of: Optional[torch.Tensor] = None,
                       force_exact: bool = False, stats: Optional[dict] = None, cap: Optional[int] = None
                       ) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor]:
    """Document range search: for query i, every document (doc_groups as in score_topk_groups) with at least one eligible
    page whose exact fp32 score is >= t_i. A document's score is the maximum over all its eligible pages, with that
    page's bits; its best page the lowest page with it. Returns CSR on the index's device: (offsets int64 [nq + 1],
    scores f32 [R], best pages int64 [R] = local page + id_offset, groups int64 [R]); row i is [offsets[i],
    offsets[i + 1]), ordered by (score desc, best page asc) as in score_topk_groups. min_score, doc_mask / mask_of, cap,
    force_exact and stats as in score_range (its pages s >= t, reduced to each document's first page in that order, are
    exactly the documents scoring >= t: DESIGN §4); stats["documents"] = R."""
    q, masks = _queries_and_mask(queries, index, doc_mask, mask_of)
    t = _check_min_score(min_score, q.shape[0], index.emb.device)
    cap = _check_cap(cap)
    with L.on_device(q.device):
        gt = _group_table(doc_groups, index)
        offsets, s, p = _score_range(q, index, t, id_offset, masks, force_exact, stats, cap, gt)
        g = gt.groups.index_select(0, p - id_offset).long()
    if stats is not None:
        stats["documents"] = p.numel()
    return offsets, s, p, g


def _score_range(q: torch.Tensor, index: CorpusIndex, t: torch.Tensor, id_offset: int, masks: Optional[_MaskSet],
                 force_exact: bool, stats: Optional[dict], cap: int, gt: Optional[_GroupTable] = None):
    """score_range, and with the group table gt the documents of score_range_groups (the same paths, each region reduced
    to the best page of every document before it is ordered)."""
    nq, d = q.shape
    nd = index.nd
    if d != index.emb.shape[1]:
        raise ValueError("query / corpus dim mismatch")
    rows = torch.arange(nq, dtype=torch.int64)
    info = dict(path="exact", candidates=0, fallback=0, cap=cap)
    grouping = () if gt is None else (gt,)
    if nq == 0:
        pieces = []
    elif force_exact or nq * nd <= SMALL_PROBLEM or nd < 256:
        pieces = _range_scan(q, index, t, masks, rows, id_offset, *grouping)
    else:
        info["path"] = "filter+rescore"
        pieces = []
        step = max(1, min(nq, RANGE_BUDGET // cap))
        for r0 in range(0, nq, step):
            n = min(step, nq - r0)
            pieces += _range_filter(q[r0:r0 + n], index, t[r0:r0 + n], masks, r0, rows[r0:r0 + n], cap, id_offset, info,
                                    *grouping)
    if stats is not None:
        stats.update(info)
    return _range_assemble(nq, pieces, q.device)


def _range_filter(q: torch.Tensor, index: CorpusIndex, t: torch.Tensor, masks: Optional[_MaskSet], r0: int,
                  rows: torch.Tensor, cap: int, id_offset: int, info: dict, gt: Optional[_GroupTable] = None):
    """Query rows r0 .. r0 + n of the batch through the range filter and the candidate rescoring (then, with gt, the
    reduction to documents); rows that overflowed (or have no bound) rerun through the scan. Returns the CSR pieces of
    these rows."""
    n, d = q.shape
    dev = q.device
    counts, kept, rs, ri = _range_candidates(q, index, t, masks, r0, cap)
    host = torch.stack([counts, kept]).cpu()  # host sync: the CSR sizes are needed to allocate the output
    over = host[0] > cap
    info["candidates"] += int(host[0][~over].sum())
    ok = torch.nonzero(~over).flatten()
    pieces = []
    if ok.numel():
        kept_host = host[1]
        if gt is not None:  # overflowed rows kept nothing, so every row of the region can be reduced
            rs, ri, kept = _range_groups(rs, ri, kept, n, int(kept_host.max()), gt.groups, gt.G)
            kept_host = kept.cpu()
        pieces.append(_range_sort(rs, ri, cap, kept, kept_host, ok, rows, id_offset))
    bad = torch.nonzero(over).flatten()
    if bad.numel():
        info["fallback"] += int(bad.numel())
        sel = bad.to(dev)
        m = None if masks is None else _MaskSet(masks.words, None if masks.of_query is None else masks.of_query[r0:r0 + n]).rows(sel)
        grouping = () if gt is None else (gt,)
        pieces += _range_scan(q.index_select(0, sel), index, t.index_select(0, sel), m, rows[bad], id_offset, *grouping)
    return pieces


def _range_groups(rs: torch.Tensor, ri: torch.Tensor, counts: torch.Tensor, n: int, most: int, groups: torch.Tensor, G: int):
    """Rows [0, n) of the region (rs, ri [*, pitch], counts) reduced by vr_range_groups to the first entry of each
    document in (score desc, page asc) order, with its own bits: (scores, ids, counts) of a region of the same pitch.
    groups (int32, indexed by the region's ids) and G as vr_range_groups takes them. most >= every counts[r]; rows
    longer than the shared-memory table go in chunks that bound the workspace."""
    pitch, dev = rs.shape[1], rs.device
    lib, sp = L.lib(), L.stream_ptr()
    gs = torch.empty((n, pitch), dtype=torch.float32, device=dev)
    gi = torch.empty((n, pitch), dtype=torch.int32, device=dev)
    gc = torch.empty(n, dtype=torch.int32, device=dev)
    row_ws = lib.vr_range_groups_ws_bytes(1, most)
    per = 65535 if row_ws == 0 else max(1, min(65535, RANGE_BUDGET // (row_ws // 8)))
    ws_bytes = lib.vr_range_groups_ws_bytes(min(per, n), most) if n else 0
    ws = torch.empty(ws_bytes // 8, dtype=torch.int64, device=dev) if ws_bytes else None
    for r0 in range(0, n, per):
        m = min(per, n - r0)
        L.check(lib.vr_range_groups(rs[r0:].data_ptr(), ri[r0:].data_ptr(), pitch, counts[r0:].data_ptr(), m, most,
                                    groups.data_ptr(), groups.shape[0], G, L.ptr(ws), ws_bytes, gs[r0:].data_ptr(),
                                    gi[r0:].data_ptr(), gc[r0:].data_ptr(), sp))
    return gs, gi, gc


def _range_candidates(q: torch.Tensor, index: CorpusIndex, t: torch.Tensor, masks: Optional[_MaskSet], r0: int, cap: int):
    """The range filter and the candidate rescoring of query rows r0 .. r0 + n of the batch: (counts [n] (> cap: the row
    overflowed), kept [n], the region scores / ids [n, cap] (row r's first kept[r] entries, in no order))."""
    n, d = q.shape
    nd, dev = index.nd, q.device
    lib, sp = L.lib(), L.stream_ptr()
    q16 = torch.empty((n, d), dtype=torch.float16, device=dev)
    qn = torch.empty(n, dtype=torch.float32, device=dev)
    L.check(lib.vr_f32_to_f16_rows(q.data_ptr(), n, d, q16.data_ptr(), qn.data_ptr(), None, sp))
    counts = torch.empty(n, dtype=torch.int32, device=dev)
    cand = torch.empty((n, cap), dtype=torch.int32, device=dev)
    L.check(lib.vr_score_filter_range(q16.data_ptr(), n, index.emb_f16.data_ptr(), nd, d, t.data_ptr(), qn.data_ptr(),
                                      index.max_norm.data_ptr(), None if masks is None else masks.arg(r0), cap,
                                      counts.data_ptr(), cand.data_ptr(), sp))
    del q16
    rs = torch.empty((n, cap), dtype=torch.float32, device=dev)
    ri = torch.empty((n, cap), dtype=torch.int32, device=dev)
    kept = torch.empty(n, dtype=torch.int32, device=dev)
    L.check(lib.vr_score_rescore_range(q.data_ptr(), n, index.emb.data_ptr(), nd, d, t.data_ptr(), cap, counts.data_ptr(),
                                       cand.data_ptr(), rs.data_ptr(), ri.data_ptr(), kept.data_ptr(), sp))
    return counts, kept, rs, ri


def _range_scan(q: torch.Tensor, index: CorpusIndex, t: torch.Tensor, masks: Optional[_MaskSet], rows: torch.Tensor,
                id_offset: int, gt: Optional[_GroupTable] = None):
    """The fp32 scan path over query rows q (global row ids `rows`): vr_score_exact, then vr_range_rows keeps the eligible
    columns with s >= t (with gt: reduced to documents), in chunks of rows that bound the [rows, nd] scratch. Returns the
    CSR pieces."""
    n, d = q.shape
    nd, dev = index.nd, q.device
    lib, sp = L.lib(), L.stream_ptr()
    step = max(1, min(n, RANGE_BUDGET // nd, 65535))
    scratch = torch.empty((step, nd), dtype=torch.float32, device=dev)
    rs = torch.empty((step, nd), dtype=torch.float32, device=dev)
    ri = torch.empty((step, nd), dtype=torch.int32, device=dev)
    counts = torch.empty(step, dtype=torch.int32, device=dev)
    pieces = []
    for r0 in range(0, n, step):
        m = min(step, n - r0)
        L.check(lib.vr_score_exact(q[r0:].data_ptr(), m, index.emb.data_ptr(), nd, d, scratch.data_ptr(), sp))
        L.check(lib.vr_range_rows(scratch.data_ptr(), m, nd, t[r0:].data_ptr(), None if masks is None else masks.arg(r0), nd,
                                  rs.data_ptr(), ri.data_ptr(), counts.data_ptr(), sp))
        region = (rs, ri, counts, counts[:m].cpu())
        if gt is not None:
            gs, gi, gc = _range_groups(rs, ri, counts, m, int(region[3].max()), gt.groups, gt.G)
            region = (gs, gi, gc, gc.cpu())
        pieces.append(_range_sort(*region[:2], nd, *region[2:], torch.arange(m), rows[r0:r0 + m], id_offset))
    return pieces


def _range_sort(rs: torch.Tensor, ri: torch.Tensor, pitch: int, counts: torch.Tensor, counts_host: torch.Tensor,
                sel: torch.Tensor, rows: torch.Tensor, id_offset: int):
    """Order the region rows `sel` (host int64) of (rs, ri, pitch, counts) into one CSR piece: (global rows, counts,
    scores, ids), the entries of rows[sel] one after the other in that order."""
    dev = rs.device
    lib, sp = L.lib(), L.stream_ptr()
    c = counts_host.to(torch.int64)
    off = torch.zeros(c.shape[0], dtype=torch.int64)
    cs = c[sel]
    off[sel] = torch.cumsum(cs, 0) - cs           # each selected region row's place in the piece
    total = int(cs.sum())
    out_s = torch.empty(total, dtype=torch.float32, device=dev)
    out_i = torch.empty(total, dtype=torch.int64, device=dev)
    if total:
        off_d = off.to(dev)
        short, long_ = sel[(cs > 0) & (cs <= RANGE_SORT_SMEM)], sel[cs > RANGE_SORT_SMEM]
        for r0 in range(0, short.numel(), 65535):
            part = short[r0:r0 + 65535]
            L.check(lib.vr_range_sort(rs.data_ptr(), ri.data_ptr(), pitch, counts.data_ptr(), part.numel(),
                                      part.to(torch.int32).to(dev).data_ptr(), off_d.data_ptr(), int(c[part].max()), id_offset,
                                      None, 0, out_s.data_ptr(), out_i.data_ptr(), sp))
        if long_.numel():
            most = int(c[long_].max())
            per = max(1, min(65535, RANGE_BUDGET // (lib.vr_range_sort_ws_bytes(1, most) // 8)))
            ws = torch.empty(lib.vr_range_sort_ws_bytes(min(per, long_.numel()), most) // 8, dtype=torch.int64, device=dev)
            for r0 in range(0, long_.numel(), per):
                part = long_[r0:r0 + per]
                L.check(lib.vr_range_sort(rs.data_ptr(), ri.data_ptr(), pitch, counts.data_ptr(), part.numel(),
                                          part.to(torch.int32).to(dev).data_ptr(), off_d.data_ptr(), most, id_offset,
                                          ws.data_ptr(), ws.numel() * 8, out_s.data_ptr(), out_i.data_ptr(), sp))
    return rows[sel], cs, out_s, out_i


def _range_assemble(nq: int, pieces, device) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """CSR (offsets, scores, ids) of all rows from pieces (rows, counts, scores, ids) that cover each row once."""
    counts = torch.zeros(nq, dtype=torch.int64)
    for rows, c, _, _ in pieces:
        counts[rows] = c
    offsets = torch.zeros(nq + 1, dtype=torch.int64)
    offsets[1:] = torch.cumsum(counts, 0)
    if pieces and torch.equal(torch.cat([p[0] for p in pieces]), torch.arange(nq)):  # the pieces are in row order
        if len(pieces) == 1:
            return offsets.to(device), pieces[0][2], pieces[0][3]
        return offsets.to(device), torch.cat([p[2] for p in pieces]), torch.cat([p[3] for p in pieces])
    total = int(offsets[-1])
    out_s = torch.empty(total, dtype=torch.float32, device=device)
    out_i = torch.empty(total, dtype=torch.int64, device=device)
    for rows, c, s, i in pieces:
        if s.numel() == 0:
            continue
        # entry e of the piece's row k goes to offsets[rows[k]] + (e - the piece's start of row k)
        shift = offsets[rows] - (torch.cumsum(c, 0) - c)
        dst = torch.arange(s.numel(), device=device) + torch.repeat_interleave(shift.to(device), c.to(device))
        out_s[dst] = s
        out_i[dst] = i
    return offsets.to(device), out_s, out_i


# ------------------------------------------------------------------------------------------------------
# Deep top-k: a sampled threshold on the range filter (DESIGN §4, "Deep top-k")
# ------------------------------------------------------------------------------------------------------
def _sample_masks(masks: Optional[_MaskSet], cols: torch.Tensor) -> Optional[_MaskSet]:
    """The mask set over the pages `cols` (int64, on the device), in that order (each mask keeps its rows)."""
    if masks is None:
        return None
    w = masks.words.view(torch.int32).index_select(1, cols >> 5)
    bits = ((w >> (cols & 31).to(torch.int32)) & 1).bool()
    return _MaskSet(pack_doc_mask(bits), masks.of_query)


def _sample_documents(gt: _GroupTable, stride: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """Every stride-th document by group id with all its pages, through the group CSR: (pages int64, their groups
    renumbered as g // stride, int32)."""
    g = torch.arange(0, gt.G, stride, device=gt.offsets.device)
    starts = gt.offsets.index_select(0, g).long()
    lens = gt.offsets.index_select(0, g + 1).long() - starts
    shift = torch.repeat_interleave(starts - (torch.cumsum(lens, 0) - lens), lens)
    cols = gt.pages.index_select(0, torch.arange(shift.numel(), device=g.device) + shift).long()
    return cols, torch.div(gt.groups.index_select(0, cols), stride, rounding_mode="floor")


def _deep_topk(q: torch.Tensor, index: CorpusIndex, k: int, id_offset: int, stats: Optional[dict],
               masks: Optional[_MaskSet], gt: Optional[_GroupTable] = None):
    """score_topk for DEEP_K_MIN < k <= DEEP_K_MAX. Every (k // 8)-th page forms a sample; t_q = the 16th best exact score
    of query q over its eligible sampled pages. The range filter and rescoring give A = {eligible pages with exact s >=
    t_q} with the scan's bits. When |A| >= k the top-k of q is the top-k of A (its k-th score is >= t_q, and every page
    ranked above it has s >= t_q). Rows with |A| < k, rows that overflowed RANGE_CAP and rows
    whose sample holds fewer than 16 eligible pages rerun through the fp32 scan. A poor threshold costs time, never bits.
    The first k of A come from vr_select_rows over the rescored region.
    Documents (gt, the group table): the sample is every (k // 8)-th document by group id with all its pages, t_q the
    16th document score of that sample, and A is reduced to the best page of each document (vr_range_groups) before the
    select; a row is answered when A holds at least k distinct documents (DESIGN §4)."""
    nq, d = q.shape
    nd, dev = index.nd, q.device
    ev = _Stages(stats)
    stride = max(1, k // 8)
    if gt is None:
        cols, sample_groups = torch.arange(0, nd, stride, device=dev), None
    else:
        cols, sample_groups = _sample_documents(gt, stride)
    if cols.numel():
        sample = CorpusIndex(index.emb.index_select(0, cols), index.emb_f16.index_select(0, cols), index.max_norm)
        sample_gt = None if gt is None else _group_table(sample_groups, sample)
        res = _score_topk(q, sample, DEEP_SAMPLE_RANK, 0, False, None, _sample_masks(masks, cols), sample_gt)
        t = res[0][:, DEEP_SAMPLE_RANK - 1].contiguous()
        short = res[1][:, DEEP_SAMPLE_RANK - 1] < 0
        del sample, sample_gt, res
    else:  # no sampled document has a page: every row reruns through the scan
        t = torch.full((nq,), float("inf"), dtype=torch.float32, device=dev)
        short = torch.ones(nq, dtype=torch.bool, device=dev)
    ev.mark("sample")
    dtypes = (torch.float32, torch.int64) if gt is None else (torch.float32, torch.int64, torch.int64)
    out = tuple(torch.empty((nq, k), dtype=dt, device=dev) for dt in dtypes)
    info = dict(path="deep", flagged=0, sample_stride=stride, candidates=0, fallback=0)
    bad = [torch.nonzero(short).flatten().cpu()]
    step = max(1, min(nq, RANGE_BUDGET // RANGE_CAP))
    for r0 in range(0, nq, step):
        n = min(step, nq - r0)
        counts, kept, rs, ri = _range_candidates(q[r0:r0 + n], index, t[r0:r0 + n], masks, r0, RANGE_CAP)
        if gt is not None:  # A reduced to documents (overflowed rows kept nothing)
            rs, ri, kept = _range_groups(rs, ri, kept, n, int(kept.max()), gt.groups, gt.G)
        host = torch.stack([counts, kept, short[r0:r0 + n].to(torch.int32)]).cpu()
        ev.mark("range")
        over = host[0] > RANGE_CAP
        info["candidates"] += int(host[0][~over].sum())
        ok = (~over) & (host[1] >= k) & (host[2] == 0)
        bad.append(torch.nonzero(~ok & (host[2] == 0)).flatten() + r0)
        sel = torch.nonzero(ok).flatten().to(dev)
        if sel.numel():  # the top-k of each row's kept region: vr_select_rows with explicit ids (-1 past kept)
            m = sel.numel()
            ids = torch.where(torch.arange(RANGE_CAP, device=dev) < kept.index_select(0, sel)[:, None],
                              ri.index_select(0, sel), -1).long()
            sc = rs.index_select(0, sel)
            ps = torch.empty((m, k), dtype=torch.float32, device=dev)
            pi = torch.empty((m, k), dtype=torch.int64, device=dev)
            L.check(L.lib().vr_select_rows(sc.data_ptr(), ids.data_ptr(), m, RANGE_CAP, k, id_offset, ps.data_ptr(),
                                           pi.data_ptr(), L.stream_ptr()))
            out[0][sel + r0], out[1][sel + r0] = ps, pi
            if gt is not None:
                out[2][sel + r0] = torch.where(pi >= 0, gt.groups.index_select(0, (pi - id_offset).clamp(min=0).flatten())
                                               .view(m, k).long(), -1)
        ev.mark("pick")
    bad = torch.cat(bad)
    if bad.numel():
        info["fallback"] = int(bad.numel())
        sel = bad.to(dev)
        rows, m = q.index_select(0, sel), None if masks is None else masks.rows(sel)
        fix = _exact_topk(rows, index, k, id_offset, m) if gt is None else _exact_topk_groups(rows, index, k, id_offset, m, gt)
        for o, f in zip(out, fix):
            o[sel] = f
        ev.mark("fallback")
    if stats is not None:
        stats.update(info)
    return out


# ------------------------------------------------------------------------------------------------------
# Diverse retrieval: maximal marginal relevance over the top candidates
# ------------------------------------------------------------------------------------------------------
MMR_MAX_FETCH = 128               # candidates per query row (vr_mmr_select)
MMR_MAX_ELEMS = 128 * 2304        # fetch * dim: the candidate rows one cluster holds
MMR_CTA_FLOATS = 144 * 1024 // 4  # ceil(fetch / C) rows of dim: one CTA's share in a cluster of C <= 8
MMR_SMEM_FLOATS = 200 * 1024 // 4  # that share and a copy of the pick's row


def _mmr_fits(fetch: int, dim: int) -> bool:
    """vr_mmr_select's caps (mmr_cluster in score.cu): the smallest cluster whose share fits also fits the pick's row."""
    if fetch > MMR_MAX_FETCH or fetch * dim > MMR_MAX_ELEMS:
        return False
    for c in (1, 2, 4, 8):
        rows = -(-fetch // c)
        if rows * dim <= MMR_CTA_FLOATS:
            return (rows + 1) * dim <= MMR_SMEM_FLOATS
    return False


def mmr_fetch_max(dim: int) -> int:
    """The largest fetch_k vr_mmr_select takes at this embedding dim (0: none)."""
    return next((f for f in range(MMR_MAX_FETCH, 0, -1) if _mmr_fits(f, dim)), 0)


def _check_count(v, name: str) -> int:
    if isinstance(v, bool) or not isinstance(v, (int, np.integer)):
        raise ValueError(f"{name} must be an int, got {v!r}")
    return int(v)


def _check_fetch(k, fetch_k, dim: int) -> Tuple[int, int]:
    """(k, fetch): 1 <= k <= fetch <= mmr_fetch_max(dim); fetch_k None: the largest allowed value <= max(20, 4 k)."""
    k = _check_count(k, "k")
    top = mmr_fetch_max(dim)
    if top == 0:
        raise ValueError(f"dim={dim} is too large for the selection: two candidate rows must fit {MMR_SMEM_FLOATS} floats")
    fetch =min(max(20, 4 * k), top) if fetch_k is None else _check_count(fetch_k, "fetch_k")
    if fetch < 1 or not _mmr_fits(fetch, dim):
        raise ValueError(f"fetch_k={fetch} must lie in [1, {top}] at dim {dim} (at most {MMR_MAX_FETCH} candidates and "
                         f"{MMR_MAX_ELEMS} floats of candidate rows)")
    if k < 1 or k > fetch:
        raise ValueError(f"k={k} must lie in [1, fetch_k={fetch}]")
    return k, fetch


def _check_lambda(lambda_mult, nq: int, device) -> torch.Tensor:
    """lambda_mult as an f32 [nq] tensor on the index's device: a float for every query, or an f32 tensor [nq]; every
    value in [0, 1]."""
    if isinstance(lambda_mult, torch.Tensor):
        if lambda_mult.dtype != torch.float32:
            raise ValueError(f"lambda_mult must be a float or a torch.float32 tensor, got {lambda_mult.dtype}")
        if lambda_mult.dim() != 1 or lambda_mult.shape[0] != nq:
            raise ValueError(f"lambda_mult must have shape [{nq}] (one lambda per query), got {list(lambda_mult.shape)}")
        if lambda_mult.device != device:
            raise ValueError(f"lambda_mult lives on {lambda_mult.device}, the index on {device}")
        t = lambda_mult.contiguous()
        if nq:
            nan, lo, hi = torch.stack([t.isnan().any().float(), t.min(), t.max()]).tolist()
            if nan or lo < 0 or hi > 1:
                raise ValueError(f"lambda_mult must lie in [0, 1] and not be NaN, got values in [{lo}, {hi}]")
        return t
    if isinstance(lambda_mult, bool) or not isinstance(lambda_mult, (int, float, np.floating, np.integer)):
        raise ValueError(f"lambda_mult must be a float or a torch.float32 tensor, got {type(lambda_mult).__name__}")
    if not 0 <= lambda_mult <= 1:  # NaN fails too
        raise ValueError(f"lambda_mult must lie in [0, 1] and not be NaN, got {lambda_mult}")
    return torch.full((nq,), float(lambda_mult), dtype=torch.float32, device=device)


def mmr_select(index: CorpusIndex, scores: torch.Tensor, ids: torch.Tensor, k: int, lambda_mult=0.5, id_offset: int = 0
               ) -> Tuple[torch.Tensor, torch.Tensor]:
    """Maximal marginal relevance over given candidates (DESIGN §4). scores f32 / ids int [nq, F] on the index's device are
    each query's candidates in (score desc, id asc) order with a (-inf, -1) tail, as score_topk returns them (local ids:
    id_offset 0). Pick 1 is the first candidate; each later pick is the unpicked candidate j with the largest
    fl(fl(lambda s_j) - fl((1 - lambda) r_j)), r_j = the largest exact fp32 similarity emb[c_j] . emb[e] over the picks e
    so far (NaN ignored); NaN values rank last and ties go to the earlier candidate. lambda_mult: a float in [0, 1]
    (1: relevance only, as score_topk; 0: diversity only), or an f32 tensor [nq] of them on the index's device.
    Returns (scores [nq, k] f32, ids [nq, k] i64 = local id + id_offset) in pick order, each pick with its relevance
    score; a row with fewer than k candidates ends in (-inf, -1). Caps: 1 <= k <= F <= mmr_fetch_max(dim)."""
    dev = index.emb.device
    if not isinstance(scores, torch.Tensor) or scores.dtype != torch.float32 or scores.dim() != 2:
        raise ValueError("scores must be a torch.float32 tensor [nq, F]")
    if not isinstance(ids, torch.Tensor) or ids.dtype not in (torch.int32, torch.int64) or ids.shape != scores.shape:
        raise ValueError(f"ids must be an int32 or int64 torch tensor of the shape of scores {list(scores.shape)}")
    if scores.device != dev or ids.device != dev:
        raise ValueError(f"scores live on {scores.device} and ids on {ids.device}, the index on {dev}")
    nq, F = scores.shape
    k, _ = _check_fetch(k, F, index.emb.shape[1])
    lam = _check_lambda(lambda_mult, nq, dev)
    ids = ids.to(torch.int64).contiguous()
    if ids.numel():
        lo, hi = torch.aminmax(ids)
        lo, hi = int(lo), int(hi)
        if lo < -1 or hi >= index.nd:
            raise ValueError(f"ids must lie in [0, {index.nd}) (local docs of the index; -1 ends a row), got [{lo}, {hi}]")
    with L.on_device(dev):
        return _mmr_select(index, scores.contiguous(), ids, k, lam, id_offset)


def _mmr_select(index: CorpusIndex, scores: torch.Tensor, ids: torch.Tensor, k: int, lam: torch.Tensor, id_offset: int):
    nq, F = scores.shape
    out_s = torch.empty((nq, k), dtype=torch.float32, device=scores.device)
    out_i = torch.empty((nq, k), dtype=torch.int64, device=scores.device)
    if nq:
        L.check(L.lib().vr_mmr_select(index.emb.data_ptr(), index.nd, index.emb.shape[1], scores.data_ptr(), ids.data_ptr(),
                                      nq, F, lam.data_ptr(), k, id_offset, out_s.data_ptr(), out_i.data_ptr(),
                                      L.stream_ptr()))
    return out_s, out_i


def score_mmr(queries: torch.Tensor, index: CorpusIndex, k: int, lambda_mult=0.5, fetch_k: Optional[int] = None,
              id_offset: int = 0, doc_mask: Optional[torch.Tensor] = None, mask_of: Optional[torch.Tensor] = None,
              doc_lists: Optional[Tuple[torch.Tensor, torch.Tensor]] = None, list_of: Optional[torch.Tensor] = None,
              stats: Optional[dict] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """Diverse top-k: score_topk(queries, index, fetch_k, doc_mask=..., mask_of=..., doc_lists=..., list_of=...) gives each
    query's fetch_k best pages, and mmr_select picks k of them (see there). fetch_k None: the largest allowed value <=
    max(20, 4 k). stats: score_topk's (path, ...), fetch_k, and with stats={"stages": {}} the CUDA-event times of the
    stages "candidates" and "select" (ms, after a synchronize and resolve_stages)."""
    k, fetch = _check_fetch(k, fetch_k, index.emb.shape[1])
    nq = queries.shape[0] if isinstance(queries, torch.Tensor) else 0
    lam = _check_lambda(lambda_mult, nq, index.emb.device)
    with L.on_device(index.emb.device):
        ev = _Stages(stats)
        s, i = score_topk(queries, index, fetch, 0, False, stats, doc_mask, mask_of, doc_lists, list_of)
        ev.mark("candidates")
        out = _mmr_select(index, s, i, k, lam, id_offset)
        ev.mark("select")
    if stats is not None:
        stats["fetch_k"] = fetch
    return out


# ------------------------------------------------------------------------------------------------------
# Hybrid retrieval: the dense score fused with an external score (DESIGN §4, "Hybrid retrieval")
# ------------------------------------------------------------------------------------------------------
FUSIONS = {"sum": L.VR_FUSE_SUM, "rrf": L.VR_FUSE_RRF}
FUSE_K_MAX = 4096          # dense entries per row vr_fuse_rows takes (k of the sum, the window of RRF)
FUSE_BUDGET = 1 << 27      # fused candidate entries per pass: query rows go in chunks


@dataclass
class _Hits:
    """A validated hit list on the index's device, CSR over query rows: offsets int64 [nq + 1], ids int32 (local pages),
    values f32, width = the longest row, n = offsets[-1] (ids / values may hold unused entries after it). Each row is in
    (id asc) order, or (value desc, id asc) for RRF."""
    offsets: torch.Tensor
    ids: torch.Tensor
    values: torch.Tensor
    width: int
    n: int


def _check_weight(weight) -> float:
    if isinstance(weight, bool) or not isinstance(weight, (int, float, np.floating, np.integer)):
        raise ValueError(f"weight must be a float, got {type(weight).__name__}")
    w = float(np.float32(weight))
    if not np.isfinite(w) or w < 0:
        raise ValueError(f"weight must be finite and >= 0 (in fp32), got {weight}")
    return w


def _check_fusion(fusion, k, window, rrf_c) -> Tuple[int, int, int]:
    """(k, dense entries per row, rrf_c) of a hybrid page search."""
    if fusion not in FUSIONS:
        raise ValueError(f"fusion must be one of {sorted(FUSIONS)}, got {fusion!r}")
    k = _check_count(k, "k")
    if not 1 <= k <= FUSE_K_MAX:
        raise ValueError(f"k={k} must lie in [1, {FUSE_K_MAX}]")
    if fusion == "sum":
        if window is not None:
            raise ValueError('window is the dense window of fusion="rrf"; the weighted sum needs none')
        return k, k, 0
    window = k if window is None else _check_count(window, "window")
    if not 1 <= window <= FUSE_K_MAX:
        raise ValueError(f"window={window} must lie in [1, {FUSE_K_MAX}]")
    rrf_c = _check_count(rrf_c, "rrf_c")
    if not 0 <= rrf_c < 1 << 24:
        raise ValueError(f"rrf_c={rrf_c} must lie in [0, 2^24)")
    return k, window, rrf_c


def _hits_in_scope(row: torch.Tensor, ids: torch.Tensor, nd: int, masks: Optional[_MaskSet], ls: Optional[_ListSet]):
    """bool [N]: hit (row, id) lies in the scope of its query row (masks, or lists; neither: every page). ids must lie in
    [0, nd). No host read."""
    if masks is not None:
        m = row.new_zeros(row.shape) if masks.of_query is None else masks.of_query.long().index_select(0, row)
        w = masks.words.view(torch.int32)[m, ids >> 5]
        return ((w >> (ids & 31).to(torch.int32)) & 1).bool()
    if ls is not None:
        # every (list, page) of the list set as a sorted key; the placeholder id of an empty set gets list M (no query's)
        pos = torch.arange(ls.ids.shape[0], device=ids.device)
        listed = torch.searchsorted(ls.offsets[1:], pos, right=True) * nd + ls.ids.long()
        listed = torch.sort(listed).values
        m = row.new_zeros(row.shape) if ls.of_query is None else ls.of_query.long().index_select(0, row)
        key = m * nd + ids
        at = torch.searchsorted(listed, key).clamp(max=listed.numel() - 1)
        return listed[at] == key
    return torch.ones_like(ids, dtype=torch.bool)


def _hit_rows(offsets: torch.Tensor, n: int, nq: int) -> torch.Tensor:
    """The query row of each of the n hit entries, by search (no host read; any offsets give rows in [0, nq))."""
    return torch.searchsorted(offsets[1:], torch.arange(n, device=offsets.device), right=True).clamp(max=max(nq - 1, 0))


def _hit_tensors(hits, nq: int, device) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """The shape, dtype and device checks of a hit list: (offsets int64, ids int64, values f32)."""
    if not isinstance(hits, (tuple, list)) or len(hits) != 3:
        raise ValueError("hits must be a triple (offsets, ids, values) of tensors")
    offsets, ids, values = hits
    _int_tensor(offsets, "hits offsets", nq + 1, device)
    _int_tensor(ids, "hits ids", None, device)
    if not isinstance(values, torch.Tensor) or values.dtype != torch.float32 or values.dim() != 1:
        raise ValueError("hits values must be a 1-D torch.float32 tensor")
    if values.shape[0] != ids.shape[0]:
        raise ValueError(f"hits values has {values.shape[0]} entries for {ids.shape[0]} ids")
    if values.device != device:
        raise ValueError(f"hits values live on {values.device}, the index on {device}")
    return offsets.to(torch.int64), ids.to(torch.int64), values


def _check_hits(hits, nq: int, nd: int, device, masks: Optional[_MaskSet] = None, ls: Optional[_ListSet] = None,
                rank_order: bool = False, keep: Optional[torch.Tensor] = None) -> _Hits:
    """Validate hits = (offsets int [nq + 1], ids int (local pages), values f32) on `device`, drop the hits outside each
    query's scope, and order each row by id (rank_order: by (value desc, id asc), the external ranks of RRF). One host
    read serves every value check (offsets from 0 to len(ids) and non-decreasing, ids in [0, nd), values finite and
    >= 0, no page twice in a row) and the sizes of the result; nothing before it can index out of bounds. A value of -0.0
    is a zero score and becomes +0.0. keep (bool [len(ids)], optional) replaces the scope test: the hits to keep."""
    offsets, ids, values = _hit_tensors(hits, nq, device)
    values = values + 0.0  # -0.0 -> +0.0: the sign bit would break the rank key below
    n = ids.shape[0]
    z = offsets.new_zeros(())
    # the row of each entry (any offsets give rows in [0, nq); they are checked below)
    row = _hit_rows(offsets, n, nq)
    safe = ids.clamp(0, nd - 1)
    key = row * nd + safe                       # (row, id): distinct keys unless a page repeats in a row
    order = torch.argsort(key)
    srt = key.index_select(0, order)
    if keep is None:
        keep = _hits_in_scope(row, safe, nd, masks, ls)
    counts = offsets.new_zeros(max(nq, 1)).scatter_add_(0, row, keep.long())[:nq]
    checks = torch.stack([offsets[0], offsets[-1], (offsets[1:] - offsets[:-1]).min() if nq else z,
                          ids.min() if n else z, ids.max() if n else z,
                          (~torch.isfinite(values)).sum() if n else z, (values < 0).sum() if n else z,
                          (srt[1:] == srt[:-1]).sum() if n > 1 else z, counts.max() if nq else z, counts.sum()]).tolist()
    first, last, min_len, lo, hi, bad_values, negative, repeats, width, kept = checks
    if first != 0:
        raise ValueError(f"hits offsets must start at 0, got {first}")
    if min_len < 0:
        raise ValueError("hits offsets must be non-decreasing")
    if last != n:
        raise ValueError(f"hits offsets must end at len(ids) = {n}, got {last}")
    if n and (lo < 0 or hi >= nd):
        raise ValueError(f"hits ids must lie in [0, {nd}) (local pages of the index), got [{lo}, {hi}]")
    if bad_values:
        raise ValueError(f"hits values must be finite: {bad_values} are NaN or infinite")
    if negative:
        raise ValueError(f"hits values must be >= 0 (a negative external score needs a deeper dense top-k): {negative} are not")
    if repeats:
        raise ValueError(f"a page appears more than once in one query's hits ({repeats} repeats)")
    out_off = torch.zeros(nq + 1, dtype=torch.int64, device=device)
    out_off[1:] = torch.cumsum(counts, 0)
    if not n:
        return _Hits(out_off, torch.zeros(1, dtype=torch.int32, device=device),
                     torch.zeros(1, dtype=torch.float32, device=device), 0, 0)
    # kept entries first, by (row, id) or (row, value desc, id asc); a stable sort keeps id order within equal keys
    outside = (~keep).long().index_select(0, order)
    if rank_order:  # values >= 0 here: their bits order like the values
        vkey = (outside << 62) | (row.index_select(0, order) << 31) | (0x7FFFFFFF - values.index_select(0, order).view(torch.int32).long())
    else:
        vkey = outside
    order = order.index_select(0, torch.sort(vkey, stable=True).indices)
    return _Hits(out_off, ids.index_select(0, order).to(torch.int32), values.index_select(0, order).contiguous(), width,
                 kept)


def score_topk_hybrid(queries: torch.Tensor, index: CorpusIndex, k: int, hits, weight=1.0, fusion: str = "sum",
                      window: Optional[int] = None, rrf_c: int = 60, id_offset: int = 0,
                      doc_mask: Optional[torch.Tensor] = None, mask_of: Optional[torch.Tensor] = None,
                      doc_lists: Optional[Tuple[torch.Tensor, torch.Tensor]] = None, list_of: Optional[torch.Tensor] = None,
                      stats: Optional[dict] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """Exact hybrid top-k pages: (fused scores [nq, k] f32, ids [nq, k] i64 = local page + id_offset) in (fused score
    desc, id asc) order, ending in (-inf, -1) when fewer pages have a score. hits = (offsets int [nq + 1], ids int local
    pages, values f32 >= 0) on the index's device: query i's external scores are values[offsets[i]:offsets[i + 1]]
    (CSR), an unlisted page having v = 0. A page may appear once per query; negative, NaN or infinite values are refused.
    fusion="sum": fl(dense + fl(weight * v)), dense the exact fp32 score (the bits of the fp32 scan). The answer lies in
    score_topk(k) plus the query's hits (DESIGN §4), whose dense scores come from vr_score_lists.
    fusion="rrf": reciprocal rank fusion in fp32, fl(1/(rrf_c + rank_dense) + 1/(rrf_c + rank_ext)), ranks from 1: the
    dense rank within score_topk(window) (default window = k, at most 4096), the external rank within the query's hits
    by (value desc, id asc); a missing rank contributes 0 and weight is not used.
    Scopes (doc_mask / mask_of, doc_lists / list_of, as in score_topk) apply to both sides: a hit outside its query's
    scope is dropped. stats: score_topk's, candidates (int64 [nq]: fused candidates of each row), and with
    stats={"stages": {}} the CUDA-event times of "dense", "lists", "fuse" and "select"."""
    k, kd, rrf_c = _check_fusion(fusion, k, window, rrf_c)
    w = _check_weight(weight)
    q = _check_f32(queries, "queries")
    nq = q.shape[0]
    ls = masks = None
    if doc_lists is not None or list_of is not None:
        q, ls = _queries_and_lists(q, index, doc_mask, mask_of, doc_lists, list_of)
    else:
        q, masks = _queries_and_mask(q, index, doc_mask, mask_of)
    rrf = fusion == "rrf"
    with L.on_device(q.device):
        h = _check_hits(hits, nq, index.nd, q.device, masks, ls, rank_order=rrf)
        ev = _Stages(stats)
        ds, di = score_topk(q, index, kd, 0, False, stats, doc_mask, mask_of, doc_lists, list_of)
        ev.mark("dense")
        return _fuse_select(q, index, ds, di, h, k, fusion, w, rrf_c, id_offset, stats, ev)


def _fuse_select(q: torch.Tensor, index: CorpusIndex, ds: torch.Tensor, di: torch.Tensor, h: _Hits, k: int, fusion: str,
                 w: float, rrf_c: int, id_offset: int, stats: Optional[dict], ev: _Stages):
    """The stages of score_topk_hybrid after the dense top-kd (ds, di [nq, kd], ids in the hits' id space): the hits'
    dense scores (sum), vr_fuse_rows and the select of k, ids + id_offset. RRF reads no index rows."""
    nq, kd = ds.shape
    rrf = fusion == "rrf"
    out_s = torch.empty((nq, k), dtype=torch.float32, device=q.device)
    out_i = torch.empty((nq, k), dtype=torch.int64, device=q.device)
    cands = torch.zeros(nq, dtype=torch.int64, device=q.device) if stats is not None else None
    if nq == 0:
        if stats is not None:
            stats["candidates"] = cands
        return out_s, out_i
    lib, sp = L.lib(), L.stream_ptr()
    hw = max(1, h.width)
    W = kd + h.width
    rows_per = max(1, min(nq, FUSE_BUDGET // (W + hw)))
    hs = torch.empty((rows_per, hw), dtype=torch.float32, device=q.device) if not rrf else None
    hi = torch.empty((rows_per, hw), dtype=torch.int64, device=q.device) if not rrf else None
    fs = torch.empty((rows_per, W), dtype=torch.float32, device=q.device)
    fi = torch.empty((rows_per, W), dtype=torch.int64, device=q.device)
    status = torch.zeros(1, dtype=torch.int32, device=q.device)
    of = torch.arange(nq, dtype=torch.int32, device=q.device)
    lists = _ListSet(h.offsets, h.ids, of if nq > 1 else None, hw, False)
    for r0 in range(0, nq, rows_per):
        n = min(rows_per, nq - r0)
        if hs is not None and h.width:  # the exact dense scores of the hits, hit j of a row at column j
            L.check(lib.vr_score_lists(q[r0:].data_ptr(), n, index.emb.data_ptr(), index.nd, q.shape[1],
                                       lists.arg(lists.of_query, r0), hw, None, hs.data_ptr(), hi.data_ptr(), None,
                                       status.data_ptr(), sp))
        ev.mark("lists")
        L.check(lib.vr_fuse_rows(ds[r0:].data_ptr(), di[r0:].data_ptr(), n, kd, h.offsets[r0:].data_ptr(),
                                 h.ids.data_ptr(), h.values.data_ptr(), L.ptr(hs), hw, FUSIONS[fusion], w, rrf_c, W,
                                 fs.data_ptr(), fi.data_ptr(), status.data_ptr(), sp))
        ev.mark("fuse")
        L.check(_rows_fn(k)(fs.data_ptr(), fi.data_ptr(), n, W, k, id_offset, out_s[r0:].data_ptr(),
                            out_i[r0:].data_ptr(), sp))
        ev.mark("select")
        if cands is not None:
            cands[r0:r0 + n] = (fi[:n] >= 0).sum(1)
    # status is not read: the width is the longest row, so neither call can truncate a list
    if stats is not None:
        stats["candidates"] = cands
    return out_s, out_i


def _group_pages_fused(q: torch.Tensor, index: CorpusIndex, groups: torch.Tensor, gt: _GroupTable, h: _Hits, w: float,
                       masks: Optional[_MaskSet]) -> Tuple[torch.Tensor, torch.Tensor]:
    """vr_group_pages_fused over every (row, slot) of groups [nq, kg] (int64), the pieces of long documents reduced by
    vr_topk_rows: (fused scores [nq, kg], best pages [nq, kg], local)."""
    nq, kg = groups.shape
    dev = q.device
    out_s = torch.empty((nq, kg), dtype=torch.float32, device=dev)
    out_p = torch.empty((nq, kg), dtype=torch.int64, device=dev)
    piece = max(1, min(GROUP_PIECE, gt.max_pages))
    pieces = max(1, -(-gt.max_pages // piece))
    lib, sp = L.lib(), L.stream_ptr()
    rows_per = max(1, min(nq, GROUP_STAGE_BUDGET // (kg * pieces)))
    ws_s = torch.empty((rows_per, kg, pieces), dtype=torch.float32, device=dev) if pieces > 1 else None
    ws_p = torch.empty((rows_per, kg, pieces), dtype=torch.int64, device=dev) if pieces > 1 else None
    for r0 in range(0, nq, rows_per):
        n = min(rows_per, nq - r0)
        s, p = (out_s[r0:], out_p[r0:]) if pieces == 1 else (ws_s, ws_p)
        L.check(lib.vr_group_pages_fused(q[r0:].data_ptr(), n, index.emb.data_ptr(), index.nd, q.shape[1],
                                         groups[r0:].data_ptr(), kg, gt.offsets.data_ptr(), gt.pages.data_ptr(), gt.G,
                                         None if masks is None else masks.arg(r0), h.offsets[r0:].data_ptr(),
                                         h.ids.data_ptr(), h.values.data_ptr(), w, piece, pieces, 0, s.data_ptr(),
                                         p.data_ptr(), sp))
        if pieces > 1:
            L.check(lib.vr_topk_rows(ws_s.data_ptr(), ws_p.data_ptr(), n * kg, pieces, 1, 0, out_s[r0:].data_ptr(),
                                     out_p[r0:].data_ptr(), sp))
    return out_s, out_p


def _check_group_fusion(fusion, name: str) -> None:
    if fusion != "sum":
        raise ValueError(f'{name} fuses by weighted sum only (fusion="sum"), got {fusion!r}: reciprocal '
                         "rank fusion of documents needs the external retriever's document ranks, not page hits")


def score_topk_groups_hybrid(queries: torch.Tensor, index: CorpusIndex, k: int, doc_groups: torch.Tensor, hits,
                             weight=1.0, fusion: str = "sum", id_offset: int = 0, doc_mask: Optional[torch.Tensor] = None,
                             mask_of: Optional[torch.Tensor] = None,
                             doc_lists: Optional[Tuple[torch.Tensor, torch.Tensor]] = None,
                             list_of: Optional[torch.Tensor] = None, stats: Optional[dict] = None
                             ) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """Exact hybrid top-k documents (doc_groups as in score_topk_groups): a document's fused score is the maximum over
    its eligible pages of fl(dense + fl(weight * v)) (hits and v as in score_topk_hybrid), its best page the lowest page
    with it; documents rank by (score desc, best page asc). Returns (scores [nq, k] f32, best pages [nq, k] i64 = local
    page + id_offset, groups [nq, k] i64), ending in (-inf, -1, -1). The candidates are the dense top-k documents
    (score_topk_groups) and the documents of the query's hits; every page of each is scored exactly
    (vr_group_pages_fused), since a document's best page need not be a hit. Only fusion="sum": RRF over documents needs
    the external retriever's document ranks, which page hits do not give. Scopes and stats as in score_topk_hybrid
    (stages "dense", "lists" (the candidate documents), "fuse" and "select"; candidates: documents scored per row)."""
    _check_group_fusion(fusion, "score_topk_groups_hybrid")
    k = _check_count(k, "k")
    if not 1 <= k <= FUSE_K_MAX:
        raise ValueError(f"k={k} must lie in [1, {FUSE_K_MAX}]")
    w = _check_weight(weight)
    q = _check_f32(queries, "queries")
    nq = q.shape[0]
    ls = masks = None
    if doc_lists is not None or list_of is not None:
        q, ls = _queries_and_lists(q, index, doc_mask, mask_of, doc_lists, list_of)
    else:
        q, masks = _queries_and_mask(q, index, doc_mask, mask_of)
    with L.on_device(q.device):
        gt = _group_table(doc_groups, index)
        h = _check_hits(hits, nq, index.nd, q.device, masks, ls)
        ev = _Stages(stats)
        _, _, dg = score_topk_groups(q, index, k, doc_groups, 0, False, stats, doc_mask, mask_of, doc_lists, list_of)
        ev.mark("dense")
        out = tuple(torch.empty((nq, k), dtype=t, device=q.device) for t in (torch.float32, torch.int64, torch.int64))
        if nq == 0:
            return out
        # candidate documents: the dense top-k and the documents of the hits, each once per row (-1: empty)
        hg = torch.full((nq, max(1, h.width)), -1, dtype=torch.int64, device=q.device)
        if h.n:
            pos = torch.arange(h.n, device=q.device)
            row = torch.searchsorted(h.offsets[1:], pos, right=True)
            hg[row, pos - h.offsets[row]] = gt.groups.index_select(0, h.ids[:h.n].long()).long()
        cand = torch.sort(torch.cat([dg, hg], 1), dim=1).values
        cand[:, 1:].masked_fill_(cand[:, 1:] == cand[:, :-1], -1)
        masks = _stage_masks(q, index, doc_mask, mask_of, doc_lists, list_of) if ls is not None else masks
        ev.mark("lists")
        fs, fp = _group_pages_fused(q, index, cand.contiguous(), gt, h, w, masks)
        ev.mark("fuse")
        L.check(_rows_fn(k)(fs.data_ptr(), fp.data_ptr(), nq, fs.shape[1], k, id_offset, out[0].data_ptr(),
                            out[1].data_ptr(), L.stream_ptr()))
        out[2].copy_(torch.where(out[1] >= 0, gt.groups.index_select(0, (out[1] - id_offset).clamp(min=0).flatten())
                                 .view(nq, k).long(), -1))
        ev.mark("select")
        if stats is not None:
            stats["candidates"] = (cand >= 0).sum(1)
    return out


def shard_range(n_items: int, rank: int, world: int) -> Tuple[int, int]:
    """Contiguous page range [lo, hi) owned by `rank` (SURVEY.md §8e: corpus sharded by page)."""
    base, rem = divmod(n_items, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def _world(group) -> int:
    """The size of the process group, or 1 outside torch.distributed."""
    import torch.distributed as dist

    return dist.get_world_size(group) if dist.is_available() and dist.is_initialized() else 1


def _all_gather_rows(packed: torch.Tensor, group) -> torch.Tensor:
    """[nq, k, c] int64 on every rank -> [nq, world*k, c]: rank r's entries of a row at [r*k, (r+1)*k). Callers pack score
    bits inside int64 so that ONE all_gather moves every array (the message is latency bound either way)."""
    import torch.distributed as dist

    world = dist.get_world_size(group)
    nq, k, c = packed.shape
    flat = torch.empty((world * nq, k, c), dtype=torch.int64, device=packed.device)  # rank-major concatenation
    dist.all_gather_into_tensor(flat, packed.contiguous(), group=group)
    return flat.view(world, nq, k, c).permute(1, 0, 2, 3).reshape(nq, world * k, c)


def gather_partials(scores: torch.Tensor, ids: torch.Tensor, group=None) -> Tuple[torch.Tensor, torch.Tensor]:
    """The ONE collective of the retrieval path: all-gather every rank's [nq, k] (score, global id) pairs.
    Returns ([nq, world*k] scores, [nq, world*k] ids) on every rank."""
    g = _all_gather_rows(torch.stack([scores.contiguous().view(torch.int32).to(torch.int64), ids.to(torch.int64)], dim=-1), group)
    return g[..., 0].to(torch.int32).view(torch.float32).contiguous(), g[..., 1].contiguous()


def sharded_topk(queries: torch.Tensor, index: CorpusIndex, k: int, id_offset: int, group=None, stats: Optional[dict] = None,
                 doc_mask: Optional[torch.Tensor] = None, mask_of: Optional[torch.Tensor] = None,
                 doc_lists: Optional[Tuple[torch.Tensor, torch.Tensor]] = None, list_of: Optional[torch.Tensor] = None):
    """Corpus sharded by page across ranks (every rank holds the same queries): local exact top-k with GLOBAL ids,
    one all-gather of [nq, k] (score, id) pairs over NCCL/NVLink, k-way merge on every rank (SURVEY.md §8e).
    doc_mask: this rank's bool [nd] mask of its own shard, or bool [M, nd] (this shard's columns of M masks) with mask_of
    (see score_topk). doc_lists / list_of: this rank's lists of its own shard, in local ids (see score_topk)."""
    s, i = score_topk(queries, index, k, id_offset, stats=stats, doc_mask=doc_mask, mask_of=mask_of, doc_lists=doc_lists,
                      list_of=list_of)
    if _world(group) == 1:
        return s, i
    ev = _Stages(stats)
    gs, gi = gather_partials(s, i, group)
    ev.mark("all_gather_partials")
    out = merge_topk(gs, gi, k)
    ev.mark("merge")
    return out


def sharded_topk_groups(queries: torch.Tensor, index: CorpusIndex, k: int, doc_groups: torch.Tensor, id_offset: int,
                        group=None, stats: Optional[dict] = None, doc_mask: Optional[torch.Tensor] = None,
                        mask_of: Optional[torch.Tensor] = None, doc_lists: Optional[Tuple[torch.Tensor, torch.Tensor]] = None,
                        list_of: Optional[torch.Tensor] = None):
    """Document-level sharded_topk: doc_groups holds this shard's pages' GLOBAL group ids (a document may span ranks).
    Local group top-k with global page ids, one all-gather of [nq, k, 3] int64 (score bits, page, group), then the merge
    keeps the first k distinct groups. A group's best page lies on one rank, and that rank's local top-k holds it whenever
    the group is in the global top-k, so the result equals score_topk_groups over the whole corpus.
    world * k must be <= MERGE_GROUPS_MAX (512), checked before any work. Pass the same doc_groups tensor on every call:
    the CSR is cached per tensor object. doc_mask / mask_of and doc_lists / list_of as in sharded_topk."""
    import torch.distributed as dist

    if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) * k > MERGE_GROUPS_MAX:
        raise ValueError(f"sharded_topk_groups: world * k = {dist.get_world_size(group) * k} > {MERGE_GROUPS_MAX}")

    s, p, g = score_topk_groups(queries, index, k, doc_groups, id_offset, stats=stats, doc_mask=doc_mask, mask_of=mask_of,
                                doc_lists=doc_lists, list_of=list_of)
    if _world(group) == 1:
        return s, p, g
    ev = _Stages(stats)
    gathered = _all_gather_rows(torch.stack([s.contiguous().view(torch.int32).to(torch.int64), p, g], dim=-1), group)
    ev.mark("all_gather_partials")
    out = merge_topk_groups(gathered[..., 0].to(torch.int32).view(torch.float32), gathered[..., 1], gathered[..., 2], k)
    ev.mark("merge")
    return out


def _score_bits(s: torch.Tensor) -> torch.Tensor:
    return s.contiguous().view(torch.int32).to(torch.int64)


def _bits_score(b: torch.Tensor) -> torch.Tensor:
    return b.to(torch.int32).view(torch.float32)


def sharded_topk_groups_pages(queries: torch.Tensor, index: CorpusIndex, k: int, doc_groups: torch.Tensor, pages: int,
                              id_offset: int, group=None, stats: Optional[dict] = None, doc_mask: Optional[torch.Tensor] = None,
                              mask_of: Optional[torch.Tensor] = None,
                              doc_lists: Optional[Tuple[torch.Tensor, torch.Tensor]] = None,
                              list_of: Optional[torch.Tensor] = None):
    """Inner hits over a corpus sharded by page (score_topk_groups_pages of the whole corpus): sharded_topk_groups gives
    the global top-k documents on every rank; each rank takes the `pages` best of its own pages of each (global group
    ids, as in sharded_topk_groups: a document this rank does not hold is empty); ONE all-gather of [nq, k, pages]
    (score bits, page); and per (row, slot) the top-`pages` of the world * pages entries. That last step is exact because
    a document's global top-m pages lie in the union of its ranks' local top-m lists (a page with m better pages on its
    own rank has m better pages globally), and it may not be skipped: the capped top-k over the gathered lists directly
    could take more than m pages of one document. Returns as score_topk_groups_pages."""
    m = _check_pages(pages)
    s, p, g = sharded_topk_groups(queries, index, k, doc_groups, id_offset, group, stats, doc_mask, mask_of, doc_lists,
                                  list_of)
    q = _check_f32(queries, "queries")
    ev = _Stages(stats)
    with L.on_device(q.device):
        masks = _stage_masks(q, index, doc_mask, mask_of, doc_lists, list_of)
        ps, pp = _group_pages_topm(q, index, g, _group_table(doc_groups, index), m, id_offset, masks)
        ev.mark("pages")
        world = _world(group)
        if world == 1:
            return s, p, g, ps, pp
        nq = q.shape[0]
        got = _all_gather_rows(torch.stack([_score_bits(ps), pp], dim=-1).view(nq, k * m, 2), group)  # [nq, world*k*m, 2]
        ev.mark("all_gather_pages")
        got = got.view(nq, world, k, m, 2).permute(0, 2, 1, 3, 4).reshape(nq * k, world * m, 2)
        ms, mp = merge_topk(_bits_score(got[..., 0]), got[..., 1], m)
        ev.mark("merge_pages")
    return s, p, g, ms.view(nq, k, m), mp.view(nq, k, m)


def sharded_topk_capped(queries: torch.Tensor, index: CorpusIndex, k: int, doc_groups: torch.Tensor, per_group: int,
                        id_offset: int, group=None, stats: Optional[dict] = None, doc_mask: Optional[torch.Tensor] = None,
                        mask_of: Optional[torch.Tensor] = None, doc_lists: Optional[Tuple[torch.Tensor, torch.Tensor]] = None,
                        list_of: Optional[torch.Tensor] = None):
    """score_topk_capped over a corpus sharded by page: the top-k of the k * per_group pages of sharded_topk_groups_pages
    (per_group >= k: sharded_topk's pages, with their groups gathered alongside)."""
    m = _check_per_group(per_group, "per_group")
    k = _check_count(k, "k")
    if m < k:
        if m > GROUP_PAGES_MAX:
            raise ValueError(f"per_group={m} must be >= k or lie in [1, {GROUP_PAGES_MAX}]")
        _, _, g, ps, pp = sharded_topk_groups_pages(queries, index, k, doc_groups, m, id_offset, group, stats, doc_mask,
                                                    mask_of, doc_lists, list_of)
        nq = ps.shape[0]
        ev = _Stages(stats)
        with L.on_device(ps.device):
            out = _capped_merge(ps.view(nq, k * m), pp.view(nq, k * m), g[:, :, None].expand(nq, k, m).reshape(nq, k * m), k)
        ev.mark("merge")
        return out
    s, p, g = score_topk_capped(queries, index, k, doc_groups, m, id_offset, False, stats, doc_mask, mask_of, doc_lists,
                                list_of)
    if _world(group) == 1:
        return s, p, g
    ev = _Stages(stats)
    got = _all_gather_rows(torch.stack([_score_bits(s), p, g], dim=-1), group)
    ev.mark("all_gather_partials")
    with L.on_device(s.device):
        out = _capped_merge(_bits_score(got[..., 0]), got[..., 1], got[..., 2], k)
    ev.mark("merge")
    return out


def gather_queries(local: torch.Tensor, n_total: int, group=None) -> torch.Tensor:
    """Queries sharded by rank for ENCODING (the reference's partition, `dense_retriever.py:48-50`): rank r encoded
    queries shard_range(n_total, r, world); one all-gather of the [ceil(n/world), d] fp32 blocks gives every rank all
    n_total embeddings in query order (10 k x 2304 fp32 = 92 MB: sub-millisecond over NVLink)."""
    import torch.distributed as dist

    world = _world(group)
    if world == 1:
        return local
    per = (n_total + world - 1) // world
    d = local.shape[1]
    block = torch.zeros((per, d), dtype=local.dtype, device=local.device)
    block[: local.shape[0]] = local
    flat = torch.empty((world * per, d), dtype=local.dtype, device=local.device)
    dist.all_gather_into_tensor(flat, block, group=group)
    parts = []
    for r in range(world):
        lo, hi = shard_range(n_total, r, world)
        parts.append(flat[r * per: r * per + (hi - lo)])
    return torch.cat(parts)


# ------------------------------------------------------------------------------------------------------
# Sharded range search, document range search, hybrid retrieval and MMR (DESIGN §4, "Sharded retrieval")
# ------------------------------------------------------------------------------------------------------
# Each sharded_* function below is three stages: the rank's local stage, an exchange (collectives only) and a merge that
# every rank runs on identical inputs. The local stages and merges are the functions named here, so that a test on one
# process can run every rank's local stage, replace the exchange by concatenation in rank order, and run the merge.
def _check_spans(spans: torch.Tensor) -> torch.Tensor:
    """spans int64 [world, 2] on the host: every rank's (id_offset, nd). The ranks' page ranges must follow each other
    in rank order from page 0 (rank r starts where rank r - 1 ends), so that the shards in rank order are one index and
    every page has one owner; overlapping, out-of-order and gapped ranges are refused. Returns the range ends [world]."""
    lo, nd = spans[:, 0], spans[:, 1]
    hi = lo + nd
    if bool((nd < 0).any()) or int(lo[0]) != 0 or bool((lo[1:] != hi[:-1]).any()):
        raise ValueError("sharded retrieval needs the ranks' page ranges [id_offset, id_offset + nd) to follow each other "
                         f"in rank order from page 0 (one contiguous range per rank), got {spans.tolist()}")
    if int(hi[-1]) >= 1 << 31:
        raise ValueError(f"sharded retrieval takes fewer than 2^31 pages in all, got {int(hi[-1])}")
    return hi


def _gather_spans(id_offset: int, nd: int, device, group) -> torch.Tensor:
    """One all-gather of every rank's (id_offset, nd): int64 [world, 2] on the host, checked by _check_spans."""
    import torch.distributed as dist

    mine = torch.tensor([id_offset, nd], dtype=torch.int64, device=device)
    got = torch.empty(dist.get_world_size(group) * 2, dtype=torch.int64, device=device)  # rank-major concatenation
    dist.all_gather_into_tensor(got, mine, group=group)
    spans = got.view(-1, 2).cpu()
    _check_spans(spans)
    return spans


def concat_csr(parts) -> Tuple[torch.Tensor, torch.Tensor]:
    """CSR arrays over the same nq rows -> one CSR array whose row r is the parts' rows r one after the other, in part
    order. parts: (offsets int64 [nq + 1] from 0, entries [n, c]) on one device (entries past offsets[-1] are ignored).
    The merge step of gather_csr, and on one process the exchange itself. Returns (offsets int64 [nq + 1], entries)."""
    offs = [o.to(torch.int64) for o, _ in parts]
    counts = torch.stack([o[1:] - o[:-1] for o in offs])           # [parts, nq]
    nq, dev = counts.shape[1], counts.device
    offsets = torch.zeros(nq + 1, dtype=torch.int64, device=dev)
    offsets[1:] = torch.cumsum(counts.sum(0), 0)
    base = offsets[:-1] + torch.cumsum(counts, 0) - counts         # where part p's row r starts
    sizes = torch.cat([offsets[-1:], counts.sum(1)]).tolist()      # host read: the sizes of the output and of each part
    first = parts[0][1]
    out = torch.empty((sizes[0],) + tuple(first.shape[1:]), dtype=first.dtype, device=dev)
    rows = torch.arange(nq, device=dev)
    for p, ((_, e), o, n) in enumerate(zip(parts, offs, sizes[1:])):
        if n:
            row = torch.repeat_interleave(rows, counts[p], output_size=n)
            out[base[p].index_select(0, row) + torch.arange(n, device=dev) - o.index_select(0, row)] = e[:n]
    return offsets, out


def gather_csr(offsets: torch.Tensor, entries: torch.Tensor, group=None, head: Optional[torch.Tensor] = None):
    """Variable-length rows across ranks: every rank holds a CSR array over the same nq rows (offsets int64 [nq + 1] from
    0, entries int64 [n, c]); every rank gets concat_csr of all ranks' arrays in rank order. Two all-gathers: the per-row
    counts [nq] (after `head`, an optional int64 [h] of per-rank values such as (id_offset, nd)), then the entries
    padded to the largest rank's n. Returns (offsets, entries, heads int64 [world, h] on the host)."""
    import torch.distributed as dist

    world = dist.get_world_size(group)
    dev, nq, c = entries.device, offsets.shape[0] - 1, entries.shape[1]
    offsets = offsets.to(torch.int64)
    head = torch.zeros(0, dtype=torch.int64, device=dev) if head is None else head.to(device=dev, dtype=torch.int64)
    h = head.shape[0]
    got = torch.empty(world * (h + nq), dtype=torch.int64, device=dev)  # rank-major concatenation
    dist.all_gather_into_tensor(got, torch.cat([head, offsets[1:] - offsets[:-1]]), group=group)
    got = got.view(world, h + nq)
    info = torch.cat([got[:, :h], got[:, h:].sum(1, keepdim=True)], 1).cpu()  # host read: heads and each rank's n
    pad = max(1, int(info[:, h].max()))
    mine = torch.zeros((pad, c), dtype=torch.int64, device=dev)
    n = int(offsets[-1])
    mine[:n] = entries[:n]
    flat = torch.empty((world * pad, c), dtype=torch.int64, device=dev)
    dist.all_gather_into_tensor(flat, mine, group=group)
    parts = []
    for r in range(world):
        o = torch.zeros(nq + 1, dtype=torch.int64, device=dev)
        o[1:] = torch.cumsum(got[r, h:], 0)
        parts.append((o, flat[r * pad:(r + 1) * pad]))
    return (*concat_csr(parts), info[:, :h])


def _range_entries(offsets: torch.Tensor, s: torch.Tensor, p: torch.Tensor, g: Optional[torch.Tensor] = None):
    """A rank's range CSR as (offsets, entries int64 [R, 2 or 3] = (score bits, page[, group]))."""
    cols = [_score_bits(s), p] + ([] if g is None else [g])
    return offsets, torch.stack(cols, 1)


def _merge_range(offsets: torch.Tensor, entries: torch.Tensor, groups: bool = False):
    """The merge of sharded_range (groups False) and sharded_range_groups: the ranks' local results, each row the ranks'
    rows in rank order (concat_csr's layout; entries from _range_entries, global pages) -> score_range's CSR (offsets,
    scores, pages), or score_range_groups' (offsets, scores, best pages, groups).
    Pages: each row's region is ordered by vr_range_sort with the global pages as ids. Documents: the region's ids are
    the entries' positions and its groups the entries' groups; vr_range_groups keeps each document's first entry in
    (score desc, position asc) order, and vr_range_sort orders the kept ones the same way. Within a rank's row, equal
    scores are in page order, and the ranks hold increasing page ranges: position order is page order (DESIGN §4)."""
    dev, nq = entries.device, offsets.shape[0] - 1
    off_h = offsets.cpu()
    tot = off_h[1:] - off_h[:-1]
    total = int(off_h[-1])
    rows = torch.arange(nq, dtype=torch.int64)
    scores = _bits_score(entries[:, 0]).contiguous()
    if total == 0:
        pieces = [(rows, tot, scores, entries[:, 1].contiguous())]
    else:
        if groups:
            if total >= 1 << 31:
                raise ValueError(f"the document merge takes fewer than 2^31 entries, got {total}")
            ids = torch.arange(total, dtype=torch.int32, device=dev)
            grp = entries[:, 2].to(torch.int32).contiguous()
            G = int(grp.max()) + 1
        else:
            ids = entries[:, 1].to(torch.int32)
        step = max(1, min(nq, RANGE_BUDGET // int(tot.max())))
        pieces = []
        for r0 in range(0, nq, step):
            n = min(step, nq - r0)
            c_h = tot[r0:r0 + n]
            pitch = max(1, int(c_h.max()))
            a, b = int(off_h[r0]), int(off_h[r0 + n])
            rs = torch.empty((n, pitch), dtype=torch.float32, device=dev)
            ri = torch.empty((n, pitch), dtype=torch.int32, device=dev)
            counts = c_h.to(torch.int32).to(dev)
            if b > a:  # row r0 + j of the merged CSR -> region row j, its entries from column 0
                row = torch.repeat_interleave(torch.arange(n, device=dev), counts, output_size=b - a)
                at = row * pitch + torch.arange(a, b, device=dev) - offsets[r0:r0 + n].index_select(0, row)
                rs.view(-1)[at] = scores[a:b]
                ri.view(-1)[at] = ids[a:b]
                if groups:
                    rs, ri, counts = _range_groups(rs, ri, counts, n, int(c_h.max()), grp, G)
                    c_h = counts.cpu()
            pieces.append(_range_sort(rs, ri, pitch, counts, c_h, torch.arange(n), rows[r0:r0 + n], 0))
    offsets, s, i = _range_assemble(nq, pieces, dev)
    if not groups:
        return offsets, s, i
    return offsets, s, entries[:, 1].index_select(0, i), entries[:, 2].index_select(0, i)


def sharded_range(queries: torch.Tensor, index: CorpusIndex, min_score, id_offset: int, group=None,
                  doc_mask: Optional[torch.Tensor] = None, mask_of: Optional[torch.Tensor] = None, force_exact: bool = False,
                  stats: Optional[dict] = None, cap: Optional[int] = None):
    """score_range over a corpus sharded by page (every rank holds the same queries; rank r's shard holds pages
    [id_offset, id_offset + nd), the ranks' ranges following each other in rank order from page 0). Each rank runs
    score_range on its shard with global ids; gather_csr moves the rows (an all-gather of the per-row counts, then one
    of the (score bits, page) int64 entries padded to the largest rank's total: 16 bytes an entry from every rank to
    every rank); vr_range_sort orders each row. A page lives on one rank and its score bits depend only on its query and
    page rows, so the union of the ranks' rows is the whole-index answer: the result equals score_range over the shards
    concatenated in rank order, bit for bit. min_score must be the same on every rank (it is not checked: that would
    take another collective). doc_mask / mask_of: this rank's part of its own shard, as in sharded_topk. stats: the local
    call's, and with stats={"stages": {}} the times of "local", "exchange" and "merge"."""
    ev = _Stages(stats)
    offsets, s, i = score_range(queries, index, min_score, id_offset, doc_mask, mask_of, force_exact, stats, cap)
    if _world(group) == 1:
        return offsets, s, i
    ev.mark("local")
    head = torch.tensor([id_offset, index.nd], dtype=torch.int64)
    offsets, entries, spans = gather_csr(*_range_entries(offsets, s, i), group, head)
    _check_spans(spans)
    ev.mark("exchange")
    with L.on_device(entries.device):
        out = _merge_range(offsets, entries)
    ev.mark("merge")
    return out


def sharded_range_groups(queries: torch.Tensor, index: CorpusIndex, min_score, doc_groups: torch.Tensor, id_offset: int,
                         group=None, doc_mask: Optional[torch.Tensor] = None, mask_of: Optional[torch.Tensor] = None,
                         force_exact: bool = False, stats: Optional[dict] = None, cap: Optional[int] = None):
    """score_range_groups over a corpus sharded by page: doc_groups holds this shard's pages' GLOBAL group ids (a
    document may span ranks). Each rank runs score_range_groups on its shard (each document's best page on that rank);
    gather_csr moves the rows as in sharded_range, with the groups (24 bytes an entry); then each (row, document) keeps
    the first of the ranks' entries in (score desc, page asc) order, and the rows are ordered (_merge_range). A
    document's best page is the best of its ranks' best pages, so the result equals score_range_groups over the shards
    concatenated in rank order, bit for bit. Arguments, stats and the page ranges as in sharded_range."""
    ev = _Stages(stats)
    offsets, s, p, g = score_range_groups(queries, index, min_score, doc_groups, id_offset, doc_mask, mask_of, force_exact,
                                          stats, cap)
    if _world(group) == 1:
        return offsets, s, p, g
    ev.mark("local")
    head = torch.tensor([id_offset, index.nd], dtype=torch.int64)
    offsets, entries, spans = gather_csr(*_range_entries(offsets, s, p, g), group, head)
    _check_spans(spans)
    ev.mark("exchange")
    with L.on_device(entries.device):
        out = _merge_range(offsets, entries, groups=True)
    ev.mark("merge")
    if stats is not None:
        stats["documents"] = out[1].numel()
    return out


def _scope(queries, index: CorpusIndex, doc_mask, mask_of, doc_lists, list_of):
    """(queries, mask set, list set) of a search's scope, validated as the plain calls do (at most one set is given)."""
    q = _check_f32(queries, "queries")
    if doc_lists is not None or list_of is not None:
        q, ls = _queries_and_lists(q, index, doc_mask, mask_of, doc_lists, list_of)
        return q, None, ls
    q, masks = _queries_and_mask(q, index, doc_mask, mask_of)
    return q, masks, None


def _hit_marks(hits, nq: int, id_offset: int, index: CorpusIndex, masks: Optional[_MaskSet], ls: Optional[_ListSet]
               ) -> torch.Tensor:
    """int32 [len(ids)]: 1 for each hit (a global page) that this rank holds (id_offset <= id < id_offset + nd) and that
    lies in its query's scope on this rank, else 0. Only the owner can apply the scope. No host read."""
    offsets, ids, _ = _hit_tensors(hits, nq, index.emb.device)
    local = ids - id_offset
    if index.nd == 0 or ids.numel() == 0:
        return torch.zeros(ids.shape[0], dtype=torch.int32, device=ids.device)
    inside = _hits_in_scope(_hit_rows(offsets, ids.shape[0], nq), local.clamp(0, index.nd - 1), index.nd, masks, ls)
    return ((local >= 0) & (local < index.nd) & inside).to(torch.int32)


def _combine_marks(marks: torch.Tensor, group) -> torch.Tensor:
    """The exchange of the sharded RRF: every rank's _hit_marks summed by one int32 all-reduce (a hit has one owner, so
    the sum is 0 or 1 and exact) -> bool, the same on every rank."""
    import torch.distributed as dist

    marks = marks.clone()
    dist.all_reduce(marks, group=group)
    return marks > 0


def _local_hits(hits, nq: int, spans: torch.Tensor, rank: int, index: CorpusIndex, masks: Optional[_MaskSet],
                ls: Optional[_ListSet]):
    """The local stage's hits of the sharded weighted sum: hits in global pages, checked against the whole corpus as the
    plain call checks them (every rank refuses the same lists), reduced to the ones rank `rank` holds and keeps, in local
    ids: an (offsets, ids, values) triple for score_topk_hybrid on the rank's shard."""
    total = int(_check_spans(spans)[-1])
    lo = int(spans[rank, 0])
    keep = _hit_marks(hits, nq, lo, index, masks, ls) > 0
    h = _check_hits(hits, nq, total, index.emb.device, keep=keep)
    return h.offsets, (h.ids[:h.n] - lo).to(torch.int32), h.values[:h.n]


def _rrf_merge(q: torch.Tensor, ds: torch.Tensor, di: torch.Tensor, hits, keep: torch.Tensor, k: int, rrf_c: int,
               total: int, stats: Optional[dict]):
    """The merge of the sharded RRF, the same on every rank: the global dense top-window (ds, di: global pages) and the
    kept hits (global pages) fused by vr_fuse_rows and selected, as score_topk_hybrid does on one index."""
    h = _check_hits(hits, q.shape[0], total, q.device, rank_order=True, keep=keep)
    return _fuse_select(q, None, ds, di, h, k, "rrf", 0.0, rrf_c, 0, stats, _Stages(None))


def _shift_hits(hits, id_offset: int):
    """hits in global pages -> in this index's local pages (world 1: the plain call's argument)."""
    if id_offset == 0 or not isinstance(hits, (tuple, list)) or len(hits) != 3 or not isinstance(hits[1], torch.Tensor):
        return hits
    return hits[0], hits[1] - id_offset, hits[2]


def sharded_topk_hybrid(queries: torch.Tensor, index: CorpusIndex, k: int, hits, id_offset: int, group=None, weight=1.0,
                        fusion: str = "sum", window: Optional[int] = None, rrf_c: int = 60,
                        doc_mask: Optional[torch.Tensor] = None, mask_of: Optional[torch.Tensor] = None,
                        doc_lists: Optional[Tuple[torch.Tensor, torch.Tensor]] = None, list_of: Optional[torch.Tensor] = None,
                        stats: Optional[dict] = None):
    """score_topk_hybrid over a corpus sharded by page (page ranges as in sharded_range). hits are in GLOBAL pages and
    the same on every rank; they are checked against the whole corpus on every rank, with the plain call's refusals.
    Scopes (doc_mask / mask_of, doc_lists / list_of) are this rank's part of its own shard, in local ids; only a hit's
    owner applies its query's scope. One all-gather of (id_offset, nd) first.
    fusion="sum": each rank runs score_topk_hybrid on its shard with the hits it holds (local ids) and global ids out;
    then gather_partials ([nq, k] pairs) and merge_topk. A page's fused score does not depend on the shard, so the
    global top-k lies in the union of the local top-k's.
    fusion="rrf": the dense ranks must be global. sharded_topk(window) gives every rank the global dense top-window;
    each rank marks the hits it holds and keeps, and one int32 all-reduce over the hits combines the marks; every rank
    then fuses and selects on identical inputs (RRF reads no index rows). The result equals score_topk_hybrid over the
    shards concatenated in rank order, bit for bit. stats: with stats={"stages": {}} the times of "local" ("dense" for
    RRF: the whole sharded_topk), "exchange" and "merge"; sum also gives the local call's stats."""
    k, kd, rrf_c = _check_fusion(fusion, k, window, rrf_c)
    w = _check_weight(weight)
    if _world(group) == 1:
        return score_topk_hybrid(queries, index, k, _shift_hits(hits, id_offset), w, fusion, window, rrf_c, id_offset,
                                 doc_mask, mask_of, doc_lists, list_of, stats)
    import torch.distributed as dist

    q, masks, ls = _scope(queries, index, doc_mask, mask_of, doc_lists, list_of)
    nq = q.shape[0]
    _hit_tensors(hits, nq, q.device)  # a malformed triple is refused before any collective
    with L.on_device(q.device):
        ev = _Stages(stats)
        spans = _gather_spans(id_offset, index.nd, q.device, group)
        if fusion == "sum":
            local = _local_hits(hits, nq, spans, dist.get_rank(group), index, masks, ls)
            s, i = score_topk_hybrid(q, index, k, local, w, "sum", None, rrf_c, id_offset, doc_mask, mask_of, doc_lists,
                                     list_of, stats)
            ev.mark("local")
            gs, gi = gather_partials(s, i, group)
            ev.mark("exchange")
            out = merge_topk(gs, gi, k)
            ev.mark("merge")
            return out
        ds, di = sharded_topk(q, index, kd, id_offset, group, None, doc_mask, mask_of, doc_lists, list_of)
        marks = _hit_marks(hits, nq, id_offset, index, masks, ls)
        ev.mark("dense")
        keep = _combine_marks(marks, group)
        ev.mark("exchange")
        out = _rrf_merge(q, ds, di, hits, keep, k, rrf_c, int(_check_spans(spans)[-1]), stats)
        ev.mark("merge")
        return out


def sharded_topk_groups_hybrid(queries: torch.Tensor, index: CorpusIndex, k: int, doc_groups: torch.Tensor, hits,
                               id_offset: int, group=None, weight=1.0, fusion: str = "sum",
                               doc_mask: Optional[torch.Tensor] = None, mask_of: Optional[torch.Tensor] = None,
                               doc_lists: Optional[Tuple[torch.Tensor, torch.Tensor]] = None,
                               list_of: Optional[torch.Tensor] = None, stats: Optional[dict] = None):
    """score_topk_groups_hybrid over a corpus sharded by page: doc_groups holds this shard's pages' GLOBAL group ids,
    hits and scopes as in sharded_topk_hybrid. Each rank runs score_topk_groups_hybrid on its shard with the hits it
    holds, then one all-gather of [nq, k, 3] int64 (score bits, page, group) and merge_topk_groups. A document's fused
    score is the best of its ranks' local fused scores, and the rank holding its best page ranks it in its local top-k
    whenever it is in the global top-k (the argument of sharded_topk_groups), so the result equals the plain call over
    the shards concatenated in rank order. Only fusion="sum"; with world > 1, world * k must be <= MERGE_GROUPS_MAX
    (512). Both are checked before any work. stats: the local call's, and with stats={"stages": {}} the times of "local", "exchange", "merge"."""
    _check_group_fusion(fusion, "sharded_topk_groups_hybrid")
    k = _check_count(k, "k")
    world = _world(group)
    if world > 1 and world * k > MERGE_GROUPS_MAX:
        raise ValueError(f"sharded_topk_groups_hybrid: world * k = {world * k} > {MERGE_GROUPS_MAX}")
    w = _check_weight(weight)
    if world == 1:
        return score_topk_groups_hybrid(queries, index, k, doc_groups, _shift_hits(hits, id_offset), w, "sum", id_offset,
                                        doc_mask, mask_of, doc_lists, list_of, stats)
    import torch.distributed as dist

    q, masks, ls = _scope(queries, index, doc_mask, mask_of, doc_lists, list_of)
    nq = q.shape[0]
    _hit_tensors(hits, nq, q.device)  # a malformed triple is refused before any collective
    with L.on_device(q.device):
        ev = _Stages(stats)
        spans = _gather_spans(id_offset, index.nd, q.device, group)
        local = _local_hits(hits, nq, spans, dist.get_rank(group), index, masks, ls)
        s, p, g = score_topk_groups_hybrid(q, index, k, doc_groups, local, w, "sum", id_offset, doc_mask, mask_of,
                                           doc_lists, list_of, stats)
        ev.mark("local")
        got = _all_gather_rows(torch.stack([_score_bits(s), p, g], dim=-1), group)
        ev.mark("exchange")
        out = merge_topk_groups(_bits_score(got[..., 0]), got[..., 1], got[..., 2], k)
        ev.mark("merge")
    return out


def _mmr_routes(ids: torch.Tensor, spans: torch.Tensor, world: int) -> torch.Tensor:
    """int64 [world, world] on the host: entry (r, s) counts the candidates (global ids [nq, fetch], -1 = none) of rank
    r's queries (shard_range(nq, r, world)) that rank s holds; the sizes of sharded_mmr's all-to-all, computed alike on
    every rank."""
    nq, fetch = ids.shape
    dev = ids.device
    q_ends = torch.tensor([shard_range(nq, r, world)[1] for r in range(world)], dtype=torch.int64, device=dev)
    receiver = torch.searchsorted(q_ends, torch.arange(nq, device=dev), right=True)[:, None].expand(nq, fetch)
    owner = torch.searchsorted(_check_spans(spans).to(dev), ids, right=True)
    owner = torch.where(ids >= 0, owner, world)
    n = torch.bincount((receiver * (world + 1) + owner).flatten(), minlength=world * (world + 1))
    return n.view(world, world + 1)[:, :world].cpu()


def _mmr_send(index: CorpusIndex, ids: torch.Tensor, spans: torch.Tensor, rank: int) -> torch.Tensor:
    """The rows rank `rank` sends in sharded_mmr's all-to-all: the fp32 rows of the candidates it holds, in (query, slot)
    order over all queries, which is receiver order (_mmr_routes' column `rank` gives each receiver's share)."""
    lo = int(spans[rank, 0])
    flat = ids.flatten()
    local = flat[(flat >= lo) & (flat < lo + index.nd)] - lo
    return index.emb.index_select(0, local)


def _all_to_all_rows(send: torch.Tensor, send_sizes: List[int], recv_sizes: List[int], group) -> torch.Tensor:
    """The exchange of sharded_mmr: one all_to_all_single of rows [n, dim]; rank r receives every rank's share for it,
    in rank order."""
    import torch.distributed as dist

    recv = torch.empty((sum(recv_sizes),) + tuple(send.shape[1:]), dtype=send.dtype, device=send.device)
    dist.all_to_all_single(recv, send.contiguous(), recv_sizes, send_sizes, group=group)
    return recv


def _mmr_place(ids: torch.Tensor, recv: torch.Tensor, spans: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """A rank's query block: ids [n, fetch] (global candidates, -1 = none) and recv, the candidates' rows in owner order,
    each owner's in (query, slot) order -> (buf [n * fetch, dim] with candidate (i, j)'s row at i * fetch + j, the ids
    remapped to those rows [n, fetch], -1 kept). Rows of missing candidates are not written."""
    n, fetch = ids.shape
    flat = ids.flatten()
    owner = torch.searchsorted(_check_spans(spans).to(ids.device), flat, right=True)
    owner = torch.where(flat >= 0, owner, spans.shape[0])
    order = torch.sort(owner, stable=True).indices[:recv.shape[0]]
    buf = torch.empty((n * fetch, recv.shape[1]), dtype=torch.float32, device=ids.device)
    buf[order] = recv
    return buf, torch.where(flat >= 0, torch.arange(n * fetch, device=ids.device), -1).view(n, fetch)


def _mmr_block(scores: torch.Tensor, ids: torch.Tensor, recv: torch.Tensor, spans: torch.Tensor, k: int,
               lam: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """The selection of a rank's query block: scores / ids [n, fetch] (global candidates) and recv (as _mmr_place
    takes it) -> (scores, global ids) [n, k] of vr_mmr_select over the placed rows. The picks depend only on the
    candidates' scores, rows and order, so they are the picks over the whole index."""
    buf, pos = _mmr_place(ids, recv, spans)
    s, p = _mmr_select(CorpusIndex(buf, None, None), scores.contiguous(), pos, k, lam.contiguous(), 0)
    flat = ids.flatten()
    return s, torch.where(p >= 0, flat.index_select(0, p.clamp(min=0).flatten()).view(p.shape), -1)


def sharded_mmr(queries: torch.Tensor, index: CorpusIndex, k: int, lambda_mult=0.5, fetch_k: Optional[int] = None,
                id_offset: int = 0, group=None, doc_mask: Optional[torch.Tensor] = None,
                mask_of: Optional[torch.Tensor] = None, doc_lists: Optional[Tuple[torch.Tensor, torch.Tensor]] = None,
                list_of: Optional[torch.Tensor] = None, stats: Optional[dict] = None):
    """score_mmr over a corpus sharded by page (page ranges as in sharded_range; scopes as in sharded_topk).
    sharded_topk(fetch_k) gives every rank the global candidates (bit-identical to score_topk over the whole index).
    Rank r runs the selection for its queries shard_range(nq, r, world) and needs the candidates' rows that other ranks
    hold: one all_to_all_single routes them, rank s sending the rows of the candidates it holds among rank r's queries
    in (query, slot) order; every rank computes the split sizes from the candidate ids and the all-gathered
    (id_offset, nd) of each rank. The selection (vr_mmr_select) runs on a buffer of those rows. One all-gather of the
    [ceil(nq / world), k] picks gives every rank every row. The picks depend only on the candidates' scores, rows and
    order (and the cluster size on fetch_k and dim), so the result equals score_mmr over the shards concatenated in rank
    order, bit for bit. Each rank receives about nq / world * fetch_k * dim * 4 bytes: 0.46 GB at 10 k queries, 8
    ranks, fetch_k = 40 and dim 2304. stats: fetch_k, and with stats={"stages": {}} the times of "candidates",
    "exchange", "select" and "gather"."""
    k, fetch = _check_fetch(k, fetch_k, index.emb.shape[1])
    world = _world(group)
    if world == 1:
        return score_mmr(queries, index, k, lambda_mult, fetch, id_offset, doc_mask, mask_of, doc_lists, list_of, stats)
    import torch.distributed as dist

    q = _check_f32(queries, "queries")
    nq, dev = q.shape[0], q.device
    lam = _check_lambda(lambda_mult, nq, index.emb.device)
    rank = dist.get_rank(group)
    with L.on_device(dev):
        ev = _Stages(stats)
        spans = _gather_spans(id_offset, index.nd, dev, group)
        s, i = sharded_topk(q, index, fetch, id_offset, group, None, doc_mask, mask_of, doc_lists, list_of)
        routes = _mmr_routes(i, spans, world)
        ev.mark("candidates")
        recv = _all_to_all_rows(_mmr_send(index, i, spans, rank), routes[:, rank].tolist(), routes[rank].tolist(), group)
        ev.mark("exchange")
        lo, hi = shard_range(nq, rank, world)
        ps, pi = _mmr_block(s[lo:hi], i[lo:hi], recv, spans, k, lam[lo:hi])
        ev.mark("select")
        got = gather_queries(torch.stack([_score_bits(ps), pi], -1).view(hi - lo, 2 * k), nq, group).view(nq, k, 2)
        ev.mark("gather")
    if stats is not None:
        stats["fetch_k"] = fetch
    return _bits_score(got[..., 0]).contiguous(), got[..., 1].contiguous()


# ------------------------------------------------------------------------------------------------------
# Reference-signature drop-ins
# ------------------------------------------------------------------------------------------------------
def load_shard(path: str):
    """`pickle((float32[n,d], List[str]))` written by `inference.py:114-126`."""
    with open(path, "rb") as f:
        data = pickle.load(f)
    return np.asarray(data[0], dtype=np.float32), list(data[1])


def save_shard(path: str, emb: np.ndarray, lookup: List[str]) -> None:
    with open(path, "wb") as f:
        pickle.dump((np.asarray(emb, dtype=np.float32), list(lookup)), f, protocol=4)


def _retrieve_one_shard(corpus_shard_path: str, encoded_queries_tensor: torch.Tensor, topk: int, device: str):
    """Same contract as `dense_retriever.py:13-34`: indices index INTO the shard; lookup maps them to doc ids."""
    emb, lookup = load_shard(corpus_shard_path)
    index = build_index(emb, lookup, device=device)
    k = min(topk, index.nd)  # torch.topk would raise for k > n; a short shard simply yields fewer candidates
    scores, idx = score_topk(encoded_queries_tensor.to(device), index, k)
    return scores, idx, lookup


def distributed_parallel_retrieve(args, topk: int) -> Dict[str, Dict[str, float]]:
    """`dense_retriever.py:37-97`: this rank's query shards x ALL corpus shards -> {qid: {docid: score}}.
    The per-shard results are unioned exactly like the reference (<= k * n_shards docs per query); the element-wise
    `.item()` loop (`:88-92`) is replaced by one device->host copy per shard."""
    with torch.no_grad():
        q_parts = sorted(glob.glob(os.path.join(args.output_dir, f"embeddings.query.rank.{args.process_index}*")))
        encoded, query_lookup = [], []
        for part in q_parts:
            emb, ids = load_shard(part)
            if len(ids) == 0:
                continue
            encoded.append(emb)
            query_lookup.extend(ids)
        c_parts = sorted(glob.glob(os.path.join(args.output_dir, "embeddings.corpus.rank.*")))
        if len(c_parts) == 0:
            raise ValueError("No pre-computed document embeddings found")
        result: Dict[str, Dict[str, float]] = {qid: {} for qid in query_lookup}
        if not encoded:
            return result
        q = torch.from_numpy(np.concatenate(encoded)).to(args.device)
        for part in c_parts:
            scores, idx, lookup = _retrieve_one_shard(part, q, topk, args.device)
            s_host, i_host = scores.cpu().numpy(), idx.cpu().numpy()
            for r, qid in enumerate(query_lookup):
                row = result[qid]
                for j in range(s_host.shape[1]):
                    if i_host[r, j] >= 0:
                        row[lookup[int(i_host[r, j])]] = float(s_host[r, j])
        return result
