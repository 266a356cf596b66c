"""Shared test helpers: synthetic pages/queries (same generators the golden script used) and golden loading."""
import json
import os

import numpy as np
from PIL import Image

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
from visrag_b200.synth import QUERY_PREFIX, synth_doc_pages, synth_pages  # noqa: E402,F401


def load_case(name):
    from visrag_b200.config import VisRAGConfig

    z = np.load(os.path.join(GOLDEN, f"{name}.npz"), allow_pickle=False)
    cfg = VisRAGConfig(**json.loads(str(z["config"])))
    if "page_spec" in z.files:
        pages = pages_from_spec(json.loads(str(z["page_spec"])))
    else:
        pages = synth_pages(z["page_sizes"], int(z["page_seed"]))
    queries = [str(q) for q in z["queries"]]
    return cfg, int(z["weight_seed"]), pages, queries, z


def _real():
    """The reference's example inputs (encoded bytes), in two files so that each stays below 1 MB."""
    out = {}
    for name in ("real_pages_parquet.npz", "real_pages_demo.npz"):
        z = np.load(os.path.join(GOLDEN, name), allow_pickle=False)
        out.update({k: z[k] for k in z.files})
    return out


def real_queries():
    """The two queries of the reference's examples/training_data/0.parquet (query i belongs to page parquet{i})."""
    return [str(q) for q in _real()["queries"]]


def pages_from_spec(spec):
    """[{kind: doc|noise, size, seed} | {kind: real, name}] -> PIL RGB pages (real ones decoded from the shipped bytes)."""
    import io

    out = []
    for e in spec:
        if e["kind"] == "doc":
            out.append(synth_doc_pages([tuple(e["size"])], e["seed"])[0])
        elif e["kind"] == "noise":
            out.append(synth_pages([tuple(e["size"])], e["seed"])[0])
        else:
            out.append(Image.open(io.BytesIO(_real()[e["name"]].tobytes())).convert("RGB"))
    return out


def cosine_rows(a, b):
    a = np.asarray(a, dtype=np.float64)
    b = np.asarray(b, dtype=np.float64)
    return (a * b).sum(1) / (np.linalg.norm(a, axis=1) * np.linalg.norm(b, axis=1))
