"""Encode loop, run files and metrics around the hot path — drop-ins for the reference's callers (SURVEY.md §8f.1):

  * `distributed_parallel_embedding_inference(dataset, model, args, dataset_type, split_save, model_additional_args)`
    == `src/openmatch/inference/inference.py:53-172`: batches of `{id,text,image}` -> `model(passage=|query=...)` ->
    pickle shards `embeddings.{corpus|query}.rank.{r}[.{a}-{b}]` = `pickle((float32[n,d], List[str]))`, barrier.
    Built on `encode_stream`: host preparation of batch i+1, kernels of batch i and the device->host copy of batch i-1
    overlap (the reference blocks on `.cpu()` every batch, `:98`).
  * `save_as_trec` / `load_from_trec` == `src/openmatch/utils.py:125-175` (same 6-column tab format).
  * `eval_mrr` == `utils.py:285-308`; `recall_at_k`, `ndcg_at_k` reproduce pytrec_eval's `recall.k` / `ndcg_cut.k`
    (`driver/eval.py:281-283`; pytrec_eval is not installed here): ranking by score descending, ties by doc id descending
    (trec_eval's rule), nDCG with gain = relevance and log2(rank+1) discount, ideal DCG over the judged docs.
"""
from __future__ import annotations

import math
import os
import pathlib
import pickle
import sys
import time
from typing import Any, Dict, Iterable, List, Optional

import numpy as np
import torch


def naive_collator(batch: List[dict]) -> dict:
    """`inference.py:40-50`: list of dicts -> dict of lists."""
    keys = batch[0].keys()
    return {k: [b[k] for b in batch] for k in keys}


def _batches(dataset: Iterable[dict], batch_size: int):
    cur = []
    for item in dataset:
        cur.append(item)
        if len(cur) == batch_size:
            yield naive_collator(cur)
            cur = []
    if cur:
        yield naive_collator(cur)


def _dump(output_dir: str, name: str, encoded: List[np.ndarray], lookup: List[str]) -> None:
    with open(os.path.join(output_dir, name), "wb") as f:
        pickle.dump((np.concatenate(encoded) if encoded else np.zeros((0, 0), np.float32), lookup), f, protocol=4)


def _split_batch(batch: dict, parts: int) -> List[dict]:
    n = len(batch["id"])
    parts = max(1, min(parts, n))
    bounds = [n * i // parts for i in range(parts + 1)]
    return [{k: v[a:b] for k, v in batch.items()} for a, b in zip(bounds, bounds[1:]) if b > a]


@torch.no_grad()
def encode_stream(batches: Iterable[dict], model, model_additional_args: Optional[dict] = None, ramp_parts: int = 1):
    """Pipelined encode: yields (ids, float32 ndarray [n, d]) per batch, in order.

    Three things overlap: the host preparation of batch i+1 (PIL resampling, tokenisation; worker thread), the kernels
    of batch i (asynchronous launches on the current stream) and the device->host copy of batch i-1 (pinned buffer +
    event instead of the reference's blocking `.cpu()`, `inference.py:98`). `ramp_parts` > 1 cuts the FIRST batch into
    pieces (re-joined before it is yielded) so that the GPU starts after a fraction of a batch has been prepared. That
    pays off only when host preparation is slow (PIL resampling on the host); with the zero-copy RGBX page path it is a small
    fraction of a step, and differently sized pieces make the caching allocator re-carve its blocks (a synchronising
    cudaFree/cudaMalloc on the first full-size batch), so the default is no ramp."""
    from collections import deque
    from concurrent.futures import ThreadPoolExecutor

    kw = model_additional_args or {}

    def work_items():  # (batch, is_last_piece_of_its_batch)
        first = True
        for b in batches:
            pieces = _split_batch(b, ramp_parts) if first and len(b["id"]) >= 4 * ramp_parts else [b]
            first = False
            for i, piece in enumerate(pieces):
                yield piece, i == len(pieces) - 1

    it = work_items()
    cur = next(it, None)
    if cur is None:
        return
    pending = deque()
    joined_ids: List[str] = []
    joined: List[np.ndarray] = []

    def collect():
        ids, host, ev, last = pending.popleft()
        ev.synchronize()
        mark(f"collected {len(ids)} items")
        joined_ids.extend(ids)
        joined.append(host.numpy().copy())
        if not last:
            return None
        out = (list(joined_ids), joined[0] if len(joined) == 1 else np.concatenate(joined))
        joined_ids.clear()
        joined.clear()
        return out

    trace = os.environ.get("VR_TRACE_STREAM")
    t_start = time.perf_counter()

    def mark(what):
        if trace:
            print(f"[encode_stream +{(time.perf_counter() - t_start) * 1e3:7.1f} ms] {what}", file=sys.stderr, flush=True)

    with ThreadPoolExecutor(max_workers=1) as pool:
        fut = pool.submit(model.prepare, cur[0], **kw)
        while cur is not None:
            pb = fut.result()
            mark(f"prepared {pb.n_items} items")
            nxt = next(it, None)
            if nxt is not None:
                fut = pool.submit(model.prepare, nxt[0], **kw)
            reps = model.encode_prepared(pb)
            mark("launched")
            host = torch.empty(reps.shape, dtype=torch.float32).pin_memory()
            host.copy_(reps, non_blocking=True)
            ev = torch.cuda.Event()
            ev.record()
            pending.append((cur[0]["id"], host, ev, cur[1]))
            if len(pending) > 1:
                out = collect()
                if out is not None:
                    yield out
            cur = nxt
    while pending:
        out = collect()
        if out is not None:
            yield out


@torch.no_grad()
def distributed_parallel_embedding_inference(dataset, model, args, dataset_type: str = "corpus", split_save: bool = True,
                                             model_additional_args: Optional[dict] = None) -> None:
    if dataset is None:
        raise ValueError("No dataset provided")
    if dataset_type not in ("corpus", "query"):
        raise ValueError(f"dataset_type: {dataset_type} is not valid.")
    os.makedirs(args.output_dir, exist_ok=True)
    world = max(1, getattr(args, "world_size", 1))
    encoded: List[np.ndarray] = []
    lookup: List[str] = []
    idx = prev_idx = 0
    first = True
    for ids, arr in encode_stream(_batches(dataset, args.per_device_eval_batch_size), model, model_additional_args):
        if first:
            assert not np.isnan(arr).any(), "vital error, model output has nan, please check."  # `inference.py:105-108`
            first = False
        encoded.append(arr)
        lookup.extend(ids)
        idx += len(ids)
        if split_save and len(lookup) >= args.max_inmem_docs // world:
            _dump(args.output_dir, f"embeddings.{dataset_type}.rank.{args.process_index}.{prev_idx}-{idx}", encoded, lookup)
            encoded, lookup, prev_idx = [], [], idx
    if split_save:
        if lookup:
            _dump(args.output_dir, f"embeddings.{dataset_type}.rank.{args.process_index}.{prev_idx}-{idx}", encoded, lookup)
    else:
        _dump(args.output_dir, f"embeddings.{dataset_type}.rank.{args.process_index}", encoded, lookup)
    if world > 1 and torch.distributed.is_available() and torch.distributed.is_initialized():
        torch.distributed.barrier()


# ----------------------------------------------------------------------------------------------- run files
def save_as_trec(rank_result: Dict[str, Dict[str, Any]], output_path: str, run_id: str = "OpenMatch") -> None:
    """`<query_id>\\tQ0\\t<doc_id>\\t<rank>\\t<score>\\t<run_id>`, docs sorted by score descending (`utils.py:125-140`)."""
    pathlib.Path(output_path).parent.mkdir(parents=True, exist_ok=True)
    with open(output_path, "w") as f:
        for qid in rank_result:
            ranked = sorted(rank_result[qid].items(), key=lambda x: x[1], reverse=True)
            for i, (doc_id, score) in enumerate(ranked):
                f.write("{}\tQ0\t{}\t{}\t{}\t{}\n".format(qid, doc_id, i + 1, score, run_id))


def load_from_trec(input_path: str, as_list: bool = False, max_len_per_q: Optional[int] = None):
    """6-column or 3-column tab separated run file (`utils.py:143-175`)."""
    rank_result: Dict[str, Any] = {}
    cnt = 0
    with open(input_path, "r") as f:
        for line in f:
            content = line.strip().split("\t")
            if len(content) == 6:
                qid, _, doc_id, _, score, _ = content
            elif len(content) == 3:
                qid, doc_id, score = content
            else:
                raise ValueError("Invalid run format")
            if qid not in rank_result:
                rank_result[qid] = [] if as_list else {}
                cnt = 0
            if max_len_per_q is None or cnt < max_len_per_q:
                if as_list:
                    rank_result[qid].append((doc_id, float(score)))
                else:
                    rank_result[qid][doc_id] = float(score)
            cnt += 1
    return rank_result


# ----------------------------------------------------------------------------------------------- metrics
def eval_mrr(qrel: Dict[str, Dict[str, int]], run: Dict[str, Dict[str, float]], cutoff: Optional[int] = None) -> Dict[str, float]:
    """MRR@cutoff exactly as `utils.py:285-308` (python sort: stable, score descending)."""
    mrr, n = 0.0, 0
    results: Dict[str, float] = {}
    for qid in qrel:
        if qid not in run:
            continue
        n += 1
        ranked = sorted(run[qid].items(), key=lambda x: x[1], reverse=True)
        rr = 0.0
        for i, (docid, _) in enumerate(ranked):
            if cutoff is None or i < cutoff:
                if docid in qrel[qid] and qrel[qid][docid] > 0:
                    rr = 1.0 / (i + 1)
                    break
        results[qid] = rr
        mrr += rr
    results["all"] = mrr / n if n else 0.0
    return results


def _trec_ranking(docs: Dict[str, float]) -> List[str]:
    """trec_eval order: score descending, ties broken by doc id descending."""
    return [d for d, _ in sorted(docs.items(), key=lambda kv: (kv[1], kv[0]), reverse=True)]


def recall_at_k(qrel, run, k: int) -> Dict[str, float]:
    """pytrec_eval `recall.k`: |relevant in top-k| / |relevant| per judged query that appears in the run."""
    res: Dict[str, float] = {}
    for qid, judged in qrel.items():
        if qid not in run:
            continue
        rel = {d for d, r in judged.items() if r > 0}
        if not rel:
            res[qid] = 0.0
            continue
        res[qid] = len(rel & set(_trec_ranking(run[qid])[:k])) / len(rel)
    res["all"] = float(np.mean([v for q, v in res.items()])) if res else 0.0
    return res


def ndcg_at_k(qrel, run, k: int) -> Dict[str, float]:
    """pytrec_eval `ndcg_cut.k`: gain = relevance grade, discount log2(rank + 1), ideal over the judged docs."""
    res: Dict[str, float] = {}
    for qid, judged in qrel.items():
        if qid not in run:
            continue
        ranking = _trec_ranking(run[qid])[:k]
        dcg = sum(max(judged.get(d, 0), 0) / math.log2(i + 2) for i, d in enumerate(ranking))
        ideal = sorted((r for r in judged.values() if r > 0), reverse=True)[:k]
        idcg = sum(r / math.log2(i + 2) for i, r in enumerate(ideal))
        res[qid] = dcg / idcg if idcg > 0 else 0.0
    res["all"] = float(np.mean([v for q, v in res.items()])) if res else 0.0
    return res


def save_results(output_dir: str, qrels, run) -> Dict[str, float]:
    """`driver/eval.py:272-304` without its bug of rewriting the log per measure: all three measures are kept."""
    out = {"ndcg_cut_10": ndcg_at_k(qrels, run, 10)["all"], "recall_10": recall_at_k(qrels, run, 10)["all"],
           "mrr_10": eval_mrr(qrels, run, 10)["all"]}
    with open(os.path.join(output_dir, "test_result.log"), "w", encoding="utf-8") as fw:
        for measure, value in out.items():
            fw.write("{:25s}{:8s}{:.4f}\n".format(measure, "all", value))
    return out
