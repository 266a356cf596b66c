"""Roofline of the non-GEMM kernels at the bench step's shapes (BASELINE configs[2] at 128 pages/step, configs[3] shard):
achieved algorithmic GB/s (HBM-bound kernels) or TFLOP/s (score filter) per kernel, CUDA events on the launching stream,
L2 flushed between timed launches (a 256 MB buffer is rewritten), one JSON line per kernel.
  python tools/bench_kernels.py [--reps 10] [--only name,name] [--ncu]   (--ncu: 1 warm-up + 1 launch each, no flush)
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from visrag_b200 import _lib as L  # noqa: E402
from visrag_b200 import ops  # noqa: E402
from visrag_b200 import retriever as R  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PEAKS = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json"))) if os.path.exists(os.path.join(ROOT, "MEASURED_PEAKS.json")) else {}
# without measured peaks: the H100 SXM data sheet (3.35 TB/s HBM3, 989 TFLOP/s dense bf16, card allowed up to 700 W)
HBM = PEAKS.get("hbm_gbs_burst") or PEAKS.get("hbm_gbs") or 3350.0
TF = PEAKS.get("bf16_tflops_burst") or PEAKS.get("bf16_tflops") or 989.0


def run(name, fn, bytes_alg, flops, a, flush):
    if a.only and name not in a.only:
        return
    fn()
    torch.cuda.synchronize()
    if a.ncu:
        fn()
        torch.cuda.synchronize()
        return
    tot = 0.0
    for _ in range(a.reps):
        flush.add_(1.0)  # rewrites 256 MB: evicts the previous launch's lines from the 50 MB L2
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        tot += e0.elapsed_time(e1)
    ms = tot / a.reps
    rec = {"kernel": name, "us": round(ms * 1e3, 1)}
    if flops:
        rec.update(tflops=round(flops / ms / 1e9, 1), frac_of_tensor_peak=round(flops / ms / 1e9 / TF, 3), peak_tflops=TF)
    if bytes_alg:
        rec.update(algorithmic_MB=round(bytes_alg / 1e6, 1), GBps=round(bytes_alg / ms / 1e6, 1),
                   frac_of_hbm_peak=round(bytes_alg / ms / 1e6 / HBM, 3), peak_GBps=HBM)
    print(json.dumps(rec), flush=True)


def unit(n, d, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    out = torch.empty((n, d), dtype=torch.float32, device="cuda")
    for r0 in range(0, n, 65536):
        x = torch.randn((min(65536, n - r0), d), device="cuda", generator=g)
        out[r0:r0 + x.shape[0]] = torch.nn.functional.normalize(x, dim=1)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--pages", type=int, default=128)
    ap.add_argument("--corpus", type=int, default=125000)
    ap.add_argument("--queries", type=int, default=10000)
    ap.add_argument("--only", type=lambda s: set(s.split(",")), default=None)
    ap.add_argument("--ncu", action="store_true")
    a = ap.parse_args()
    dev = "cuda"
    torch.manual_seed(0)
    flush = torch.zeros(64 << 20, device=dev)
    S = a.pages
    M = S * 1024

    px = torch.randint(0, 256, (S, 448, 448, 3), dtype=torch.uint8, device=dev)
    run("im2col_norm", lambda: ops.im2col_norm(px, 14, 640), px.numel() + M * 640 * 2, 0, a, flush)
    del px

    x = torch.randn(M, 1152, device=dev)
    g1, b1 = torch.randn(1152, device=dev), torch.randn(1152, device=dev)
    run("layernorm_1152", lambda: ops.layernorm(x, g1, b1, 1e-6), M * 1152 * 6, 0, a, flush)
    del x

    T = S * 68
    h = torch.randn(T, 2304, device=dev)
    g2 = torch.randn(2304, device=dev)
    run("rmsnorm_2304", lambda: ops.rmsnorm(h, g2, 1e-5), T * 2304 * 6, 0, a, flush)
    cu = torch.arange(0, T + 1, 68, dtype=torch.int32, device=dev)
    run("pool_norm_wmean", lambda: ops.pool_norm(h, g2, 1e-5, cu, "wmean", True), T * 2304 * 4 + S * 2304 * 4, 0, a, flush)
    emb = torch.randn(4096, 2304, device=dev).bfloat16()
    vis = torch.randn(S * 64, 2304, device=dev)
    src = torch.full((T,), -1, dtype=torch.int32, device=dev).view(S, 68)
    src[:, 2:66] = torch.arange(S * 64, dtype=torch.int32, device=dev).view(S, 64)
    src = src.reshape(-1).contiguous()
    run("build_lm_input", lambda: ops.build_lm_input(src, emb, 12.0, vis), S * 64 * 2304 * 8 + S * 4 * 2304 * 6, 0, a, flush)
    del h, vis

    nd, nq, d, k = a.corpus, a.queries, 2304, 10
    D = unit(nd, d, 1)
    Q = unit(nq, d, 2)
    run("f32_to_f16_rows", lambda: R.to_f16_rows(D, want_max_norm=True), nd * d * 6, 0, a, flush)
    index = R.build_index(D)
    lib = L.lib()
    ranges = lib.vr_score_ranges(nq, nd)
    lists = ranges * 2
    kt = lib.vr_score_list_len()
    q16 = R.to_f16_rows(Q)
    cs = torch.empty((nq, lists * kt), dtype=torch.float32, device=dev)
    ci = torch.empty((nq, lists * kt), dtype=torch.int32, device=dev)
    out_s = torch.empty((nq, k), dtype=torch.float32, device=dev)
    out_i = torch.empty((nq, k), dtype=torch.int64, device=dev)
    flags = torch.empty((nq,), dtype=torch.int32, device=dev)

    def filt():
        L.check(lib.vr_score_filter(q16.data_ptr(), nq, index.emb_f16.data_ptr(), nd, d, ranges, cs.data_ptr(), ci.data_ptr(),
                                    L.stream_ptr()))

    def resc():
        L.check(lib.vr_score_rescore(Q.data_ptr(), nq, D.data_ptr(), nd, d, ranges, cs.data_ptr(), ci.data_ptr(),
                                     index.max_norm.data_ptr(), k, 0, out_s.data_ptr(), out_i.data_ptr(), flags.data_ptr(),
                                     L.stream_ptr()))

    run("score_filter", filt, 0, 2.0 * nq * nd * d, a, flush)
    filt()
    torch.cuda.synchronize()
    n_cand = int((ci >= 0).sum().item())
    if not a.ncu:
        print(json.dumps({"note": "filter plan", "lists_per_query": lists, "real_candidates_per_query": round(n_cand / nq, 1)}), flush=True)
    keep = min(32, lists * kt)  # vr_score_rescore rescoring budget for k = 10: the 32 best candidates by approximate score
    n_resc = int(torch.clamp((ci >= 0).sum(dim=1), max=keep).sum().item())
    run("rescore_topk", resc, n_resc * d * 4 + nq * d * 4 + nq * lists * kt * 8, 0, a, flush)
    if not a.ncu and (not a.only or "rescore_topk" in a.only):
        print(json.dumps({"note": "rescore result", "flagged": int(flags.sum().item())}), flush=True)

    # fp32 scan + chunked top-k: 8 queries over the shard (the demo / small-batch retrieval path)
    Q8 = Q[:8].contiguous()
    scratch = torch.empty((8, nd), dtype=torch.float32, device=dev)
    run("exact_scores_8q", lambda: L.check(lib.vr_score_exact(Q8.data_ptr(), 8, D.data_ptr(), nd, d, scratch.data_ptr(), L.stream_ptr())),
        nd * d * 4, 0, a, flush)
    chunks = min(1024, nd // 4096)
    ws_s = torch.empty((8, chunks, k), dtype=torch.float32, device=dev)
    ws_i = torch.empty((8, chunks, k), dtype=torch.int64, device=dev)
    run("topk_rows_chunked_8q", lambda: L.check(lib.vr_topk_rows_chunked(scratch.data_ptr(), 8, nd, k, 0, chunks, ws_s.data_ptr(),
                                                                          ws_i.data_ptr(), out_s.data_ptr(), out_i.data_ptr(), L.stream_ptr())),
        8 * nd * 4, 0, a, flush)
    # merge of 8 ranks' partial top-10 lists (the step after the all-gather)
    ms_s = torch.randn(nq, 80, device=dev)
    ms_i = torch.randint(0, 1 << 20, (nq, 80), device=dev)
    run("topk_rows_merge_8x10", lambda: R.merge_topk(ms_s, ms_i, 10), nq * 80 * 12, 0, a, flush)


if __name__ == "__main__":
    main()
