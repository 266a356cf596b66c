"""Device-resident step time of the full model for different batch shapes: pages per step x ViT sub-batch (tokens).
Answers two layout questions with measurements: does a ViT sub-batch whose fp32 residual stream fits the 50 MB L2
beat the wave-quantisation loss of smaller GEMMs, and how much does a larger step amortise the LM tail.
  python tools/sweep_step.py [--pages 128,256] [--vit-tokens 16384,32768,65536,131072]"""
import argparse
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from visrag_b200.config import VisRAGConfig  # noqa: E402
from visrag_b200.encoder import VisRAGEngine  # noqa: E402
from visrag_b200.host import prepare_batch  # noqa: E402
from visrag_b200.tokenizer_stub import StubTokenizer  # noqa: E402
from visrag_b200.weights import random_state_dict_device  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pages", default="112,120,128,144,150,256")
    ap.add_argument("--vit-tokens", default="65536,131072,163840")
    ap.add_argument("--steps", type=int, default=4)
    a = ap.parse_args()
    from PIL import Image

    cfg = VisRAGConfig.full()
    tok = StubTokenizer(cfg.vocab)
    eng = VisRAGEngine(cfg, random_state_dict_device(cfg, 2024, "cuda:0"))
    rs = np.random.RandomState(1)
    for P in [int(x) for x in a.pages.split(",")]:
        pages = [Image.fromarray(x) for x in rs.randint(0, 256, (P, 448, 448, 3), dtype=np.uint8)]
        pb = prepare_batch([""] * P, pages, tok, cfg, 2048)
        groups, src, pos, cu = eng.upload(pb)
        max_len = int(pb.seq_lens.max())
        for vt in [int(x) for x in a.vit_tokens.split(",")]:
            if vt > P * 1024:
                continue
            eng.max_vit_tokens = vt
            for _ in range(2):
                eng.encode_device(groups, pb.group_row0, pb.n_slices, src, pos, cu, max_len)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.steps):
                eng.encode_device(groups, pb.group_row0, pb.n_slices, src, pos, cu, max_len)
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / a.steps
            print(f"pages {P:4d}  vit sub-batch {vt:7d} tokens  {ms:8.2f} ms/step  {P / ms * 1e3:7.1f} pages/s", flush=True)


if __name__ == "__main__":
    main()
