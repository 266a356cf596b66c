"""BASELINE configs[1]: SigLIP-so400m tower only (26 blocks + final LayerNorm, no head), batch 1 -> 512, 384x384 inputs.
Through the VisRAG `vpm` (dynamic_img_pad) a 384 px image pads to 392 -> 28x28 = 784 tokens (SURVEY.md 8d); here the
synthetic input is generated at 392x392 directly. Prints images/s and model TFLOP/s per batch size.
  python tools/bench_vit_sweep.py [--max-batch 512]"""
import argparse
import os
import tempfile
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from visrag_b200.config import VisRAGConfig  # noqa: E402
from visrag_b200.encoder import VisRAGEngine  # noqa: E402
from visrag_b200.weights import random_state_dict_device  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--max-batch", type=int, default=512)
    ap.add_argument("--px", type=int, nargs="+", default=[378, 392],
                    help="378 -> 27x27 = 729 tokens (stock timm at 384, the CSV row in the reference), 392 -> 784 tokens (VisRAG vpm)")
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "vit_sweep.json"))
    a = ap.parse_args()
    import json

    cfg = VisRAGConfig.full()
    eng = VisRAGEngine(cfg, random_state_dict_device(cfg, 2024, "cuda:0"))
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    peaks = json.load(open(os.path.join(root, "MEASURED_PEAKS.json"))) if os.path.exists(os.path.join(root, "MEASURED_PEAKS.json")) else {}
    peak = peaks.get("bf16_tflops_sustained") or 1429.0
    rows = []
    for px_side in a.px:
        rows += sweep(eng, cfg, px_side, a.max_batch, peak)
    os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
    json.dump({"what": "BASELINE configs[1]: SigLIP-so400m tower only (26 blocks + final LN), bf16, one H100", "peak_tflops_sustained": peak,
               "rows": rows}, open(a.out, "w"), indent=1)


def sweep(eng, cfg, px_side, max_batch, peak):
    n = (px_side // cfg.patch_size) ** 2
    flop_per_image = 793_046_016 * n + 119_808 * n * n  # SURVEY.md appendix B: F_vit(N)
    g = torch.Generator(device="cuda").manual_seed(0)
    bs = 1
    rows = []
    a = argparse.Namespace(px=px_side, max_batch=max_batch)
    while bs <= a.max_batch:
        px = torch.randint(0, 256, (bs, a.px, a.px, 3), dtype=torch.uint8, device="cuda", generator=g)
        for _ in range(3):
            eng.vit_tokens(px)
        torch.cuda.synchronize()
        reps = max(3, min(50, 2048 // bs))
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            eng.vit_tokens(px)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / reps
        tf = flop_per_image * bs / ms / 1e9
        print(f"batch {bs:4d} x {n} tokens: {ms:8.3f} ms  {bs / ms * 1e3:9.1f} images/s  {tf:7.1f} TFLOP/s  {tf / peak:.3f} of sustained peak",
              flush=True)
        rows.append({"px": px_side, "tokens": n, "batch": bs, "ms": round(ms, 4), "images_per_s": round(bs / ms * 1e3, 1),
                     "tflops": round(tf, 1), "frac_of_tensor_peak": round(tf / peak, 3)})
        bs *= 2
    return rows


if __name__ == "__main__":
    main()
