"""Demo knowledge-base layout and single-query retrieval (SURVEY.md §8f.3).

Drop-in for the reference's demo pipeline:
  * `visrag_scripts/demo/visrag_pipeline/build_index.py:52-58` writes `reps.npy` (float32 [n, d], the L2-normalised page
    embeddings) and `index2img_filename.txt` ('\\n'-joined image basenames) into the knowledge-base directory;
  * `answer.py:26-35` (`retrieve`) reloads both files and re-uploads the embeddings for EVERY query, then
    `torch.matmul(query_rep, doc_reps.T)` + `torch.topk`.
Here the index is loaded once and stays resident in HBM (`KnowledgeBase`); a query is one fp32 scan of the index
(`vr_score_exact`, HBM bound: n*d*4 bytes) plus a two-level top-k spread over many SMs (`vr_topk_rows_chunked`).
Scores are the same fp32 dot products; ties are ordered by lower page index (torch.topk leaves tie order unspecified).

Beyond the reference: a search can be restricted to some pages (`within`, e.g. the pages of one PDF), pages can be
removed (a tombstone bit, so the other pages keep their indices) and added, and `save` writes the live pages back in the
demo's layout. A scope runs as a doc mask inside the same kernels, or, when it is small, as a candidate list of its pages
that reads only those pages (`list_path_wins`), with the same exact fp32 results either way. A batch of queries
can give each query its own scope (`within_each`, e.g. each question about its own PDF, or each user's own collections):
one pass over the index serves them all, and each query's row equals its search alone.

Documents: `build_index.py` stores page i of `report.pdf` as `report.pdf_i.png`, so a page's document is its filename up to
the last `_` when the rest is `<digits>.png` (any other filename is its own document). `search_documents` returns the
top-k documents by their best page (`retriever.score_topk_groups`), so one long document cannot fill every slot.
`search(…, per_document=m)` caps the pages of any one document at m, and `search_document_pages` returns the top-k
documents each with its m best pages. `search_hybrid` / `search_documents_hybrid` fuse the dense score with another
retriever's score of each page (e.g. BM25 over OCR text). `search_diverse` / `retrieve_diverse` pick pages by maximal marginal relevance (`retriever.mmr_select`), so near-copies
of one page, in one document or several, do not fill every slot either.
"""
from __future__ import annotations

import os
import re
from typing import Iterable, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib as L
from . import retriever

REPS_FILE = "reps.npy"
NAMES_FILE = "index2img_filename.txt"
# the demo's instruction (`answer.py:33`; singular "document", unlike the eval scripts' "documents")
DEMO_QUERY_PREFIX = "Represent this query for retrieving relevant document: "


_PAGE_SUFFIX = re.compile(r"_[0-9]+\.png")


def document_of(filename: str) -> str:
    """The document a page belongs to: `report.pdf_12.png` -> `report.pdf` (`build_index.py`'s naming); any other
    filename is its own document."""
    cut = filename.rfind("_")
    return filename[:cut] if cut >= 0 and _PAGE_SUFFIX.fullmatch(filename[cut:]) else filename


def save_knowledge_base(path: str, reps, filenames: Sequence[str]) -> None:
    """Write the two files exactly as `build_index.py:52-58` does."""
    reps = np.asarray(reps.detach().cpu().numpy() if isinstance(reps, torch.Tensor) else reps, dtype=np.float32)
    if reps.ndim != 2 or reps.shape[0] != len(filenames):
        raise ValueError("reps must be [n, d] with one filename per row")
    if any("\n" in f for f in filenames):
        raise ValueError("filenames must not contain newlines")
    os.makedirs(path, exist_ok=True)
    np.save(os.path.join(path, REPS_FILE), reps)
    with open(os.path.join(path, NAMES_FILE), "w") as f:
        f.write("\n".join(filenames))


LIST_TILE = 8              # queries that share a list and read each of its rows once (vr_score_lists' query tile)
LIST_ROUTE = 1.0           # index rows per 256-query block the masked path costs, per listed row of the list path
LIST_FIXED_ROWS = 80_000   # the list path's fixed cost (checks, launches, two host reads), in index rows of one query


def list_path_wins(list_rows: int, nq: int, nd: int, k: int, documents: bool) -> bool:
    """The routing rule of scoped searches. list_rows is the listed page rows summed over the distinct scopes, each scope
    counted once per tile of LIST_TILE queries that search it (a None scope, every live page, counts nd rows): what the
    list path reads, at 4 * dim bytes a row. The masked path passes over all nd rows once per 256-query block. Lists win
    when list_rows + LIST_FIXED_ROWS < LIST_ROUTE * nd * ceil(nq / 256). The constants come from the measurements in the
    README (H100, dim 2304): a listed row and an index row per 256-query block cost about the same (3-6 ns), and the list
    path's fixed cost is about that of scanning 65-80 k rows for one query. Documents with k above
    retriever.LIST_GROUPS_MAX_K take the masks."""
    if documents and k > retriever.LIST_GROUPS_MAX_K:
        return False
    return list_rows + LIST_FIXED_ROWS < LIST_ROUTE * nd * -(-nq // 256)


class KnowledgeBase:
    """A knowledge base resident on one GPU. Pages keep their index (row) for the life of the object: `remove` only marks
    a page dead, and `add` appends."""

    def __init__(self, path: str, device: str = "cuda"):
        self.path = path
        with open(os.path.join(path, NAMES_FILE), "r") as f:
            self.filenames: List[str] = f.read().split("\n")
        reps = np.load(os.path.join(path, REPS_FILE))
        if reps.ndim != 2 or reps.shape[0] != len(self.filenames):
            raise ValueError(f"{path}: reps.npy has {reps.shape} rows/dims but {len(self.filenames)} filenames")
        self.index = retriever.build_index(np.ascontiguousarray(reps, dtype=np.float32), self.filenames, device)
        self._row = {name: i for i, name in enumerate(self.filenames)}   # filename -> row, live pages only
        self._live = torch.ones(len(self.filenames), dtype=torch.bool, device=self.index.emb.device)
        self._n_live = len(self.filenames)
        self.documents: List[str] = []                # document id -> name; ids are dense and never reused
        self._doc_id = {}
        self._doc_groups = torch.empty(0, dtype=torch.int32, device=self.index.emb.device)
        self._add_documents(self.filenames)

    def _add_documents(self, filenames: Sequence[str]) -> None:
        """Give every new page its document id: a page of a known document name joins it, a new name takes the next id."""
        ids = []
        for f in filenames:
            doc = document_of(f)
            if doc not in self._doc_id:
                self._doc_id[doc] = len(self.documents)
                self.documents.append(doc)
            ids.append(self._doc_id[doc])
        new = torch.tensor(ids, dtype=torch.int32).to(self._doc_groups.device)
        self._doc_groups = torch.cat([self._doc_groups, new])

    def __len__(self) -> int:
        return self._n_live

    def _rows(self, filenames: Iterable[str]) -> List[int]:
        if isinstance(filenames, str):
            filenames = [filenames]
        try:
            return sorted({self._row[name] for name in filenames})
        except KeyError as e:
            raise KeyError(f"no live page named {e.args[0]!r} in the knowledge base") from None

    def _queries(self, query_reps) -> torch.Tensor:
        """queries [nq, d] fp32 on the index's device."""
        q = query_reps if isinstance(query_reps, torch.Tensor) else torch.from_numpy(np.asarray(query_reps, dtype=np.float32))
        return q.to(self.index.emb.device, torch.float32).reshape(-1, self.index.emb.shape[1]).contiguous()

    def _query_and_mask(self, query_reps, within: Optional[Iterable[str]]):
        """(queries [nq, d] fp32 on the index's device, bool [nd] mask of the pages searched or None for every page, number
        of pages searched)."""
        q = self._queries(query_reps)
        if within is None:
            return q, None if len(self) == self.index.nd else self._live, len(self)  # None: the unmasked kernels
        rows = self._rows(within)
        return q, self._scope_masks([rows]).view(-1), len(rows)

    def _scope_masks(self, scopes: Sequence[Optional[Sequence[int]]]) -> torch.Tensor:
        """bool [M, nd]: row m marks the page rows of scope m (None: every live page)."""
        dev = self.index.emb.device
        masks = torch.zeros((len(scopes), self.index.nd), dtype=torch.bool, device=dev)
        every = [m for m, rows in enumerate(scopes) if rows is None]
        pairs = [(m, r) for m, rows in enumerate(scopes) if rows is not None for r in rows]
        if every:
            masks[torch.tensor(every, dtype=torch.int64, device=dev)] = self._live
        if pairs:
            idx = torch.tensor(pairs, dtype=torch.int64, device=dev)
            masks[idx[:, 0], idx[:, 1]] = True
        return masks

    def _query_and_scopes(self, query_reps, within, within_each):
        """Per-query scopes: (queries, the distinct scopes (sorted page rows, or None for every live page), list_of [nq]
        int32 (the scope of each query), the live page rows of each distinct scope). Identical scopes are one scope."""
        if within is not None:
            raise ValueError("within and within_each cannot be combined: give every query its scope in within_each")
        q = self._queries(query_reps)
        scopes = list(within_each)
        if len(scopes) != q.shape[0]:
            raise ValueError(f"within_each has {len(scopes)} entries for {q.shape[0]} queries (one scope per query)")
        slot, keys, scope_of = {}, [], []
        for scope in scopes:
            key = None if scope is None else tuple(self._rows(scope))
            if key not in slot:
                slot[key] = len(keys)
                keys.append(key)
            scope_of.append(slot[key])
        live = torch.nonzero(self._live).flatten().tolist() if None in slot else []
        rows_of = [live if rows is None else list(rows) for rows in keys]
        return q, keys, torch.tensor(scope_of, dtype=torch.int32, device=q.device), rows_of

    def _lists(self, rows_of: Sequence[Sequence[int]]) -> Tuple[torch.Tensor, torch.Tensor]:
        """The candidate lists (offsets, ids) of the scopes' page rows."""
        dev = self.index.emb.device
        offsets = torch.tensor(np.cumsum([0] + [len(r) for r in rows_of]), dtype=torch.int64, device=dev)
        ids = torch.tensor([r for rows in rows_of for r in rows], dtype=torch.int32, device=dev)
        return offsets, ids

    def _use_lists(self, keys, rows_of, scope_of: Optional[torch.Tensor], nq: int, k: int, documents: bool) -> bool:
        """Whether these scopes go through candidate lists (see list_path_wins); a None scope counts as nd pages."""
        per_scope = torch.bincount(scope_of.long(), minlength=len(keys)).tolist() if scope_of is not None else [nq]
        rows = sum((self.index.nd if key is None else len(r)) * -(-n // LIST_TILE)
                   for key, r, n in zip(keys, rows_of, per_scope))
        return list_path_wins(rows, nq, self.index.nd, k, documents)

    def _scopes(self, query_reps, within, within_each):
        """(queries, the distinct scopes (sorted page rows; keys None: every live page, in one scope), list_of [nq] int32
        (the scope of each query, None: one scope for every query), the live page rows of each distinct scope)."""
        if within_each is not None:
            return self._query_and_scopes(query_reps, within, within_each)
        if within is not None:
            key = tuple(self._rows(within))
            return self._queries(query_reps), [key], None, [list(key)]
        return self._queries(query_reps), None, None, None

    def _scope_args(self, q, keys, rows_of, scope_of, k: int, documents: bool) -> dict:
        """The scope arguments of a retriever call: every live page through the mask of the live pages (none when no page
        was removed), else candidate lists of the scopes' pages when they win (list_path_wins), else their masks."""
        if keys is None:
            return dict(doc_mask=None if len(self) == self.index.nd else self._live)
        if self._use_lists(keys, rows_of, scope_of, q.shape[0], k, documents):
            return dict(doc_lists=self._lists(rows_of), list_of=scope_of)
        masks = self._scope_masks(keys)
        return dict(doc_mask=masks if scope_of is not None else masks[0], mask_of=scope_of)

    def _n_documents(self, q, keys, rows_of) -> int:
        """The documents of the largest scope."""
        if keys is None:
            searched = self._doc_groups if len(self) == self.index.nd else self._doc_groups[self._live]
            return int(torch.unique(searched).numel())
        if len(keys) == 1:
            idx = torch.tensor(rows_of[0], dtype=torch.int64, device=q.device)
            return int(torch.unique(self._doc_groups[idx]).numel())   # documents searched, counted on the device
        groups = self._doc_groups.tolist()
        return max(len({groups[r] for r in rows}) for rows in rows_of)

    def search(self, query_reps, topk: int, within: Optional[Iterable[str]] = None,
               within_each: Optional[Sequence[Optional[Iterable[str]]]] = None,
               per_document: Optional[int] = None) -> Tuple[torch.Tensor, torch.Tensor]:
        """query_reps [nq, d] (tensor or ndarray, fp32) -> (scores [nq,k] f32, page indices [nq,k] i64) on the device.
        within: page filenames to search (default: every live page); k = min(topk, pages searched).
        within_each: one scope per query instead (a list of page filenames, or None for every live page), all searched in
        one pass; k = min(topk, pages of the largest scope), and a query whose scope is shorter ends in (-inf, -1).
        Small scopes are scored from candidate lists of their pages (list_path_wins), the others through masks of the
        whole index: the results are the same bits either way.
        per_document: at most this many pages of any one document (retriever.score_topk_capped): the pages are walked
        best first and a page is skipped once its document has per_document pages. When the caps leave fewer than k
        pages, the row ends in (-inf, -1)."""
        if per_document is not None:
            retriever._check_per_group(per_document, "per_document")
        q, keys, scope_of, rows_of = self._scopes(query_reps, within, within_each)
        if keys is None:
            k = min(topk, len(self))
        else:
            k = min(topk, max(len(rows) for rows in rows_of)) if rows_of else 0
        if k == 0:
            return (torch.empty((q.shape[0], 0), dtype=torch.float32, device=q.device),
                    torch.empty((q.shape[0], 0), dtype=torch.int64, device=q.device))
        if per_document is None:
            return retriever.score_topk(q, self.index, k, **self._scope_args(q, keys, rows_of, scope_of, k, False))
        s, p, _ = retriever.score_topk_capped(q, self.index, k, self._doc_groups, per_document,
                                              **self._scope_args(q, keys, rows_of, scope_of, k, True))
        return s, p

    def search_documents(self, query_reps, topk: int, within: Optional[Iterable[str]] = None,
                         within_each: Optional[Sequence[Optional[Iterable[str]]]] = None
                         ) -> Tuple[torch.Tensor, torch.Tensor, List[List[str]]]:
        """The top-k DOCUMENTS, each scored by its best page: (scores [nq,k] f32, best page indices [nq,k] i64 on the
        device, document names [nq][k]). within: page filenames to search (default: every live page); k = min(topk,
        documents searched). Ties rank the document with the lower best page index first.
        within_each: one scope per query, as in search; k = min(topk, documents of the largest scope), a shorter row ends
        in (-inf, -1), and each query's names list holds only the documents it found. Scopes are routed as in search."""
        q, keys, scope_of, rows_of = self._scopes(query_reps, within, within_each)
        k = min(topk, self._n_documents(q, keys, rows_of)) if rows_of != [] else 0
        if k == 0:
            return (torch.empty((q.shape[0], 0), dtype=torch.float32, device=q.device),
                    torch.empty((q.shape[0], 0), dtype=torch.int64, device=q.device), [[] for _ in range(q.shape[0])])
        s, p, g = retriever.score_topk_groups(q, self.index, k, self._doc_groups,
                                              **self._scope_args(q, keys, rows_of, scope_of, k, True))
        return s, p, self._names(g)

    def _names(self, groups: torch.Tensor) -> List[List[str]]:
        return [[self.documents[j] for j in row if j >= 0] for row in groups.tolist()]

    def search_document_pages(self, query_reps, topk: int, pages: int, within: Optional[Iterable[str]] = None,
                              within_each: Optional[Sequence[Optional[Iterable[str]]]] = None
                              ) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor, List[List[str]]]:
        """The top-k documents of search_documents, each with its `pages` best pages (inner hits,
        retriever.score_topk_groups_pages): (document scores [nq,k] f32, page scores [nq,k,pages] f32, page indices
        [nq,k,pages] i64 on the device, document names [nq][k]). A document's pages are in (score desc, page asc) order,
        column 0 its best page; fewer pages end in (-inf, -1). within / within_each and k as in search_documents."""
        pages = retriever._check_pages(pages)
        q, keys, scope_of, rows_of = self._scopes(query_reps, within, within_each)
        k = min(topk, self._n_documents(q, keys, rows_of)) if rows_of != [] else 0
        if k == 0:
            return (torch.empty((q.shape[0], 0), dtype=torch.float32, device=q.device),
                    torch.empty((q.shape[0], 0, pages), dtype=torch.float32, device=q.device),
                    torch.empty((q.shape[0], 0, pages), dtype=torch.int64, device=q.device), [[] for _ in range(q.shape[0])])
        s, _, g, ps, pp = retriever.score_topk_groups_pages(q, self.index, k, self._doc_groups, pages,
                                                            **self._scope_args(q, keys, rows_of, scope_of, k, True))
        return s, ps, pp, self._names(g)

    def search_above(self, query_reps, min_score, within: Optional[Iterable[str]] = None,
                     within_each: Optional[Sequence[Optional[Iterable[str]]]] = None
                     ) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """Every page scoring at least min_score (a float, or an f32 tensor [nq] on the device: one threshold per query),
        as CSR on the device: (offsets int64 [nq + 1], scores f32 [R], page indices int64 [R]); query i's pages are
        [offsets[i], offsets[i + 1]), by (score desc, page asc), with the exact fp32 scores (retriever.score_range).
        within / within_each: the pages searched, as in search (default: every live page); removed pages never appear."""
        q, scope = self._range_scope(query_reps, within, within_each)
        return retriever.score_range(q, self.index, min_score, **scope)

    def search_documents_above(self, query_reps, min_score, within: Optional[Iterable[str]] = None,
                               within_each: Optional[Sequence[Optional[Iterable[str]]]] = None
                               ) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor, List[List[str]]]:
        """Every document with a page scoring at least min_score (a float, or an f32 tensor [nq] on the device), each
        scored by its best page: (offsets int64 [nq + 1], scores f32 [R], best page indices int64 [R] on the device,
        document names [nq][*]); query i's documents are [offsets[i], offsets[i + 1]), by (score desc, best page asc) as
        in search_documents (retriever.score_range_groups). within / within_each as in search_above: a document is
        scored by its searched live pages only, and one whose searched pages all score below min_score is left out."""
        q, scope = self._range_scope(query_reps, within, within_each)
        offsets, s, p, g = retriever.score_range_groups(q, self.index, min_score, self._doc_groups, **scope)
        groups, ends = g.tolist(), offsets.tolist()
        names = [[self.documents[j] for j in groups[a:b]] for a, b in zip(ends[:-1], ends[1:])]
        return offsets, s, p, names

    def _range_scope(self, query_reps, within, within_each):
        """(queries, the mask arguments of a range search over the scopes' live pages)."""
        if within_each is not None:
            q, keys, scope_of, _ = self._query_and_scopes(query_reps, within, within_each)
            if q.shape[0] == 0:
                return q, {}
            return q, dict(doc_mask=self._scope_masks(keys), mask_of=scope_of)
        q, mask, _ = self._query_and_mask(query_reps, within)
        return q, dict(doc_mask=mask)

    NEAR_DUPLICATE_ROWS = 8192  # pages scored as queries per pass of near_duplicates

    def near_duplicates(self, min_score: float, within: Optional[Iterable[str]] = None
                        ) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """Every pair of live pages (of `within`, default every live page) with a < b and exact fp32 score
        reps[a] . reps[b] >= min_score: (a int64 [P], b int64 [P], scores f32 [P]) on the device, by a ascending, then
        (score desc, b asc). Each page's row of score_range over the same pages, without the entries b <= a: the score
        of (a, b) has the same bits as that of (b, a) (the fp32 FMA chain multiplies the same pairs in the same order),
        so each pair is reported once, from its lower page. Pages are scored as queries in chunks."""
        dev = self.index.emb.device
        if within is None:
            rows = torch.nonzero(self._live).flatten()
            mask = None if len(self) == self.index.nd else self._live
        else:
            rows = torch.tensor(self._rows(within), dtype=torch.int64, device=dev)
            mask = self._scope_masks([rows.tolist()]).view(-1)
        a_parts, b_parts, s_parts = [], [], []
        for r0 in range(0, rows.numel(), self.NEAR_DUPLICATE_ROWS):
            sel = rows[r0:r0 + self.NEAR_DUPLICATE_ROWS]
            off, s, b = retriever.score_range(self.index.emb.index_select(0, sel), self.index, min_score, doc_mask=mask)
            a = torch.repeat_interleave(sel, off[1:] - off[:-1])
            keep = b > a
            a_parts.append(a[keep])
            b_parts.append(b[keep])
            s_parts.append(s[keep])
        if not a_parts:
            e = torch.empty(0, dtype=torch.int64, device=dev)
            return e, e.clone(), torch.empty(0, dtype=torch.float32, device=dev)
        return torch.cat(a_parts), torch.cat(b_parts), torch.cat(s_parts)

    def search_diverse(self, query_reps, topk: int, lambda_mult=0.5, fetch_k: Optional[int] = None,
                       within: Optional[Iterable[str]] = None,
                       within_each: Optional[Sequence[Optional[Iterable[str]]]] = None) -> Tuple[torch.Tensor, torch.Tensor]:
        """Diverse top-k pages by maximal marginal relevance: (relevance scores [nq,k] f32, page indices [nq,k] i64) on the
        device, in pick order. The candidates are search(query_reps, fetch_k, within, within_each), so scopes and removed
        pages behave exactly as there, and retriever.mmr_select picks k = min(topk, candidates) of them. lambda_mult: a
        float in [0, 1] or an f32 tensor [nq] on the device (1: the order of search; lower values trade relevance for
        pages unlike those already picked). fetch_k None: the largest allowed value <= max(20, 4 topk)."""
        _, fetch = retriever._check_fetch(topk, fetch_k, self.index.emb.shape[1])
        q = self._queries(query_reps)
        lam = retriever._check_lambda(lambda_mult, q.shape[0], self.index.emb.device)
        s, ids = self.search(q, fetch, within, within_each)
        k = min(topk, s.shape[1])
        if k == 0 or s.shape[0] == 0:
            return s[:, :k], ids[:, :k]
        with L.on_device(s.device):
            return retriever._mmr_select(self.index, s, ids, k, lam, 0)

    def retrieve_diverse(self, query_rep, topk: int, lambda_mult=0.5, fetch_k: Optional[int] = None,
                         within: Optional[Iterable[str]] = None) -> List[str]:
        """Paths of k diverse page images (search_diverse), in pick order: for a generator with a small image budget."""
        _, ids = self.search_diverse(query_rep, topk, lambda_mult, fetch_k, within)
        return [os.path.join(self.path, self.filenames[i]) for i in ids[0].tolist() if i >= 0]

    def retrieve_diverse_text(self, model, tokenizer, query: str, topk: int, lambda_mult=0.5,
                              fetch_k: Optional[int] = None, within: Optional[Iterable[str]] = None) -> List[str]:
        """retrieve_text with diverse pages: instruction + query -> embedding -> retrieve_diverse."""
        out = model(query={"text": [DEMO_QUERY_PREFIX + query], "image": [None]}, tokenizer=tokenizer)
        return self.retrieve_diverse(out.q_reps, topk, lambda_mult, fetch_k, within)

    def retrieve_document_pages(self, query_rep, topk: int, pages: int,
                                within: Optional[Iterable[str]] = None) -> List[Tuple[str, List[str]]]:
        """[(document name, paths of its best page images, best first)] of the top-k documents, best first: for a list
        of documents with page thumbnails."""
        _, _, idx, names = self.search_document_pages(query_rep, topk, pages, within)
        return [(n, [os.path.join(self.path, self.filenames[i]) for i in row if i >= 0])
                for n, row in zip(names[0], idx[0].tolist())]

    def retrieve_documents(self, query_rep, topk: int, within: Optional[Iterable[str]] = None) -> List[Tuple[str, str]]:
        """[(document name, path of its best page image)] of the top-k documents, best first."""
        _, pages, names = self.search_documents(query_rep, topk, within)
        return [(n, os.path.join(self.path, self.filenames[i])) for n, i in zip(names[0], pages[0].tolist())]

    def retrieve_documents_text(self, model, tokenizer, query: str, topk: int,
                                within: Optional[Iterable[str]] = None) -> List[Tuple[str, str]]:
        """retrieve_text at the document level: instruction + query -> embedding -> top-k documents."""
        out = model(query={"text": [DEMO_QUERY_PREFIX + query], "image": [None]}, tokenizer=tokenizer)
        return self.retrieve_documents(out.q_reps, topk, within)

    def retrieve(self, query_rep, topk: int, within: Optional[Iterable[str]] = None,
                 per_document: Optional[int] = None) -> List[str]:
        """`answer.py: retrieve` after the query is encoded: paths of the top-k page images, best first. per_document: at
        most this many pages of any one document (see search); the list is shorter when the caps leave fewer pages."""
        _, ids = self.search(query_rep, topk, within, per_document=per_document)
        return [os.path.join(self.path, self.filenames[i]) for i in ids[0].tolist() if i >= 0]

    def retrieve_text(self, model, tokenizer, query: str, topk: int, within: Optional[Iterable[str]] = None,
                      per_document: Optional[int] = None) -> List[str]:
        """Full `retrieve(knowledge_base_path, query, topk)`: instruction + query -> embedding (B2 wrapper) -> top-k."""
        out = model(query={"text": [DEMO_QUERY_PREFIX + query], "image": [None]}, tokenizer=tokenizer)
        return self.retrieve(out.q_reps, topk, within, per_document)

    def _hits(self, hits: Sequence[dict], nq: int) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """One {filename: external score} mapping per query -> the retriever's hit CSR (offsets, page rows, values) on
        the device. Unknown and removed filenames are dropped."""
        hits = list(hits)
        if len(hits) != nq:
            raise ValueError(f"hits has {len(hits)} entries for {nq} queries (one {{filename: score}} mapping per query)")
        rows, vals, offsets = [], [], [0]
        for h in hits:
            live = [(self._row[f], v) for f, v in h.items() if f in self._row]
            rows.extend(r for r, _ in live)
            vals.extend(v for _, v in live)
            offsets.append(len(rows))
        dev = self.index.emb.device
        return (torch.tensor(offsets, dtype=torch.int64, device=dev), torch.tensor(rows, dtype=torch.int32, device=dev),
                torch.tensor(vals, dtype=torch.float32, device=dev))

    def search_hybrid(self, query_reps, topk: int, hits: Sequence[dict], weight=1.0, fusion: str = "sum",
                      window: Optional[int] = None, within: Optional[Iterable[str]] = None,
                      within_each: Optional[Sequence[Optional[Iterable[str]]]] = None) -> Tuple[torch.Tensor, torch.Tensor]:
        """Hybrid top-k pages (retriever.score_topk_hybrid): the dense score fused with an external score of each page,
        e.g. BM25 over its OCR text. hits: one {filename: score >= 0} mapping per query (unknown or removed filenames
        are dropped; an unlisted page scores 0). fusion="sum": dense + weight * score; fusion="rrf": reciprocal rank
        fusion of the dense top-`window` (default k) and the hits ranked by score. Returns (fused scores [nq,k] f32, page
        indices [nq,k] i64) on the device. within / within_each and k as in search; hits outside a query's scope are
        dropped."""
        q, keys, scope_of, rows_of = self._scopes(query_reps, within, within_each)
        h = self._hits(hits, q.shape[0])
        if keys is None:
            k = min(topk, len(self))
        else:
            k = min(topk, max(len(rows) for rows in rows_of)) if rows_of else 0
        if k == 0:
            return (torch.empty((q.shape[0], 0), dtype=torch.float32, device=q.device),
                    torch.empty((q.shape[0], 0), dtype=torch.int64, device=q.device))
        return retriever.score_topk_hybrid(q, self.index, k, h, weight, fusion, window,
                                           **self._scope_args(q, keys, rows_of, scope_of, k, False))

    def search_documents_hybrid(self, query_reps, topk: int, hits: Sequence[dict], weight=1.0, fusion: str = "sum",
                                within: Optional[Iterable[str]] = None,
                                within_each: Optional[Sequence[Optional[Iterable[str]]]] = None
                                ) -> Tuple[torch.Tensor, torch.Tensor, List[List[str]]]:
        """Hybrid top-k documents (retriever.score_topk_groups_hybrid): each document scored by its best page under
        dense + weight * score, hits as in search_hybrid (weighted sum only). Returns (scores [nq,k] f32, best page
        indices [nq,k] i64 on the device, document names [nq][k]); within / within_each and k as in search_documents."""
        q, keys, scope_of, rows_of = self._scopes(query_reps, within, within_each)
        h = self._hits(hits, q.shape[0])
        k = min(topk, self._n_documents(q, keys, rows_of)) if rows_of != [] else 0
        if k == 0:
            return (torch.empty((q.shape[0], 0), dtype=torch.float32, device=q.device),
                    torch.empty((q.shape[0], 0), dtype=torch.int64, device=q.device), [[] for _ in range(q.shape[0])])
        s, p, g = retriever.score_topk_groups_hybrid(q, self.index, k, self._doc_groups, h, weight, fusion,
                                                     **self._scope_args(q, keys, rows_of, scope_of, k, True))
        return s, p, self._names(g)

    def retrieve_hybrid_text(self, model, tokenizer, query: str, topk: int, hits: dict, weight=1.0, fusion: str = "sum",
                             window: Optional[int] = None, within: Optional[Iterable[str]] = None) -> List[str]:
        """retrieve_text with hybrid ranking: instruction + query -> embedding -> search_hybrid with the query's
        {filename: score} hits -> paths of the top-k page images, best first."""
        out = model(query={"text": [DEMO_QUERY_PREFIX + query], "image": [None]}, tokenizer=tokenizer)
        _, ids = self.search_hybrid(out.q_reps, topk, [hits], weight, fusion, window, within)
        return [os.path.join(self.path, self.filenames[i]) for i in ids[0].tolist() if i >= 0]

    def remove(self, filenames: Iterable[str]) -> None:
        """Mark pages dead: no search returns them again. The other pages keep their indices, and the index's max row norm
        (the filter's error bound) stays as it is: an upper bound over a superset of the live pages is still one."""
        rows = self._rows(filenames)
        for r in rows:
            del self._row[self.filenames[r]]
        self._n_live -= len(rows)
        if rows:
            self._live[torch.tensor(rows, dtype=torch.int64, device=self._live.device)] = False

    def add(self, reps, filenames: Sequence[str]) -> None:
        """Append pages (fp32 [n, d] embeddings, one filename each) after the existing ones. A name may not be a live page
        already; the name of a removed page may come back, as a new page."""
        filenames = list(filenames)
        dev = self.index.emb.device
        x = reps if isinstance(reps, torch.Tensor) else torch.from_numpy(np.asarray(reps, dtype=np.float32))
        x = x.to(dev, torch.float32).contiguous()
        if x.dim() != 2 or x.shape[0] != len(filenames) or x.shape[1] != self.index.emb.shape[1]:
            raise ValueError(f"reps must be [n, {self.index.emb.shape[1]}] with one filename per row")
        if any("\n" in f for f in filenames):
            raise ValueError("filenames must not contain newlines")
        dup = sorted({f for f in filenames if f in self._row} | {f for f in filenames if filenames.count(f) > 1})
        if dup:
            raise ValueError(f"duplicate page filenames: {dup[:5]}")
        if not filenames:
            return
        n0, n, d = self.index.nd, x.shape[0], x.shape[1]
        f16 = torch.empty((n, d), dtype=torch.float16, device=dev)
        with L.on_device(dev):
            # the kernel's atomicMax raises the index's max row norm to cover the new rows
            L.check(L.lib().vr_f32_to_f16_rows(x.data_ptr(), n, d, f16.data_ptr(), None, self.index.max_norm.data_ptr(),
                                               L.stream_ptr()))
        self.index.emb = torch.cat([self.index.emb, x])
        self.index.emb_f16 = torch.cat([self.index.emb_f16, f16])
        self._live = torch.cat([self._live, torch.ones(n, dtype=torch.bool, device=dev)])
        self._add_documents(filenames)
        self.filenames.extend(filenames)
        self._row.update((f, n0 + i) for i, f in enumerate(filenames))
        self._n_live += n

    def save(self, path: Optional[str] = None) -> None:
        """Write the live pages, in index order, as the demo's two files (to `path`, default the directory loaded from).
        A knowledge base loaded from them returns the same pages and score bits for any query."""
        rows = torch.nonzero(self._live).flatten().tolist()
        keep = torch.tensor(rows, dtype=torch.int64, device=self.index.emb.device)
        save_knowledge_base(self.path if path is None else path, self.index.emb.index_select(0, keep),
                            [self.filenames[r] for r in rows])
