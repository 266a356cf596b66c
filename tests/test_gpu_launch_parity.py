"""Every kernel launch of real encodes, checked on its own against the float64 operation of the reference model at that
point (tests/launch_parity.py), with the per-element bounds of tests/kernel_bounds.py.

The end-to-end tests compare embeddings after 26 + 40 layers of accumulated 16-bit rounding, so their tolerances
(cos >= 0.9999, max |d| <= 1e-3) cannot see a wiring mistake that moves the embeddings by less: a position table
resampled with the wrong filter, RoPE tables from the wrong theta, an eps, a swapped grid. Here the `visrag_b200.ops`
entry points are wrapped (eager launches, cuda_graphs=False); each launch is identified by the weight or gain tensor it
reads (attention by the GEMM output it reads) and mapped to its state-dict key; its output is checked right away
against a reference built from the state dict in its original layout, the reference's constants and the oracle's
token plan (ids, image bounds, positions, sequence lengths), applied to the launch's actual input. Nothing of the
reference comes from the arguments the engine passed. A launch the checker cannot place fails, and the number of
launches of each kind is asserted.

Not covered: CUDA-graph replay (bit-identical to eager launches, test_gpu_encode.py) and the prefix cache's bit
equality with the full path (test_gpu_prefix_cache.py)."""
import dataclasses
import hashlib
from collections import Counter

import numpy as np
import pytest
import torch

from tests import launch_parity as LP
from tests.helpers import QUERY_PREFIX, cosine_rows, synth_pages

pytestmark = pytest.mark.gpu

DEV = "cuda"
DTYPES = [torch.bfloat16, torch.float16]
DT_IDS = ["bf16", "f16"]
MAX_INP = 2048


def _digest(a):
    return hashlib.sha1(np.ascontiguousarray(a).tobytes()).hexdigest()


class Plan:
    """The oracle's token plan for one encode call: per item ids, image bounds and the digests of its slices in LM order
    (oracle.restated.prepare_context / convert_to_tensors)."""

    def __init__(self, cfg, tok, texts, images):
        from oracle import restated as O

        self.ids, self.bounds, self.slices, self.geoms = [], [], [], set()
        for text, image in zip(texts, images):
            content, slices = O.prepare_context(text, image, tok, cfg.query_num, cfg.max_slice_nums, cfg.scale_resolution,
                                                cfg.patch_size)
            ids, bound = O.convert_to_tensors(tok, content, MAX_INP)
            arrs = [np.asarray(s.convert("RGB")) for s in slices][: len(bound)]
            self.ids.append(ids)
            self.bounds.append(bound)
            self.slices.append([_digest(a) for a in arrs])
            self.geoms |= {a.shape[:2] for a in arrs}


class Recorder:
    """Checks every launch of the engines it is bound to. `cfg` is the reference configuration (constants: eps, scales,
    theta, head counts), `sd` the checkpoint on the device."""

    def __init__(self, cfg, sd, dtype):
        self.cfg, self.sd, self.dt = cfg, sd, dtype
        self.roles = {}
        self.eng = None
        self.stats = {}                 # kind -> [count, worst fraction of the bound]
        self.failures = []              # (kind, message)
        self.runs = []                  # expected LM runs, in launch order
        self.run = None
        self.pooling = None
        self.vision = {}                # slice digest -> its 64 resampler rows (fp32)
        self.prefixes = {}              # prefix ids -> {"kv": [per layer K|V rows], "h": residual rows}
        self.chunk = None
        self.last = {}
        self.layer = None

    # ------------------------------------------------------------------------------------------------ bookkeeping
    def bind(self, eng):
        """data_ptr of every weight / gain the engine holds -> (kind, state-dict key prefix)."""
        self.eng = eng
        r = {eng.patch_w.data_ptr(): ("patch", "vpm.patch_embed.proj"), eng.vnorm_w.data_ptr(): ("vit.ln", "vpm.norm"),
             eng.rs_kv_w.data_ptr(): ("rs.kv", "resampler.kv_proj"), eng.rs_wk.data_ptr(): ("rs.k", "resampler.attn.k"),
             eng.rs_wv.data_ptr(): ("rs.v", "resampler.attn.v"), eng.rs_wo.data_ptr(): ("rs.out", "resampler.attn.out_proj"),
             eng.rs_projT.data_ptr(): ("rs.proj", "resampler.proj"), eng.rs_lnkv[0].data_ptr(): ("rs.ln_kv", "resampler.ln_kv"),
             eng.rs_lnpost[0].data_ptr(): ("rs.ln_post", "resampler.ln_post"), eng.final_w.data_ptr(): ("lm.final", "llm.model.norm"),
             eng.embed.data_ptr(): ("lm.input", "llm.model.embed_tokens")}
        for i, b in enumerate(eng.blocks):
            p = f"vpm.blocks.{i}."
            r.update({b["n1w"].data_ptr(): ("vit.ln", p + "norm1"), b["qkv_w"].data_ptr(): ("vit.qkv", p + "attn.qkv"),
                      b["proj_w"].data_ptr(): ("vit.proj", p + "attn.proj"), b["n2w"].data_ptr(): ("vit.ln", p + "norm2"),
                      b["fc1_w"].data_ptr(): ("vit.fc1", p + "mlp.fc1"), b["fc2_w"].data_ptr(): ("vit.fc2", p + "mlp.fc2")})
        for i, l in enumerate(eng.layers):
            p = f"llm.model.layers.{i}."
            r.update({l["in_w"].data_ptr(): ("lm.rms", p + "input_layernorm"), l["qkv_w"].data_ptr(): ("lm.qkv", p),
                      l["o_w"].data_ptr(): ("lm.o", p + "self_attn.o_proj"), l["post_w"].data_ptr(): ("lm.rms", p + "post_attention_layernorm"),
                      l["gu_w"].data_ptr(): ("lm.gu", p + "mlp"), l["down_w"].data_ptr(): ("lm.down", p + "mlp.down_proj")})
        assert len(r) == 11 + 6 * len(eng.blocks) + 6 * len(eng.layers), "two engine weights share storage"
        self.roles = r

    def _note(self, kind, fn):
        st = self.stats.setdefault(kind, [0, 0.0])
        st[0] += 1
        try:
            st[1] = max(st[1], fn()["frac"])
        except AssertionError as exc:
            self.failures.append((kind, str(exc)[:400]))

    def unplaced(self, what):
        self.failures.append(("unplaced", what))

    def expect(self, plan, pooling="wmean", prefix=None, pooled=True):
        """Queue the LM runs one encode call makes. prefix: None (full sequences), ("create", P) or ("hit", P)."""
        lens = [len(i) for i in plan.ids]
        if prefix is not None:
            mode, P = prefix
            key = tuple(int(t) for t in plan.ids[0][:P])
            assert all(tuple(int(t) for t in ids[:P]) == key for ids in plan.ids)
            if mode == "create":
                self.runs.append(dict(ids=[plan.ids[0][:P]], bounds=[np.zeros((0, 2))], slices=[[]], p0=0, build=key))
            self.runs.append(dict(ids=[i[P:] for i in plan.ids], bounds=[np.zeros((0, 2))] * len(lens),
                                  slices=[[]] * len(lens), p0=P, key=key, full=lens))
        else:
            self.runs.append(dict(ids=plan.ids, bounds=plan.bounds, slices=plan.slices, p0=0, full=lens))
        self.pooling = pooling if pooled else None

    # ------------------------------------------------------------------------------------------------ wrappers
    def im2col_norm(self, real, pixels, patch, ld_out, dtype=torch.bfloat16):
        out = real(pixels, patch, ld_out, dtype)
        px16 = LP.normalized_pixels(pixels, self.dt)
        S, h, w, _ = pixels.shape
        host = pixels.cpu().numpy()
        self.chunk = dict(px16=px16, S=S, gh=h // self.cfg.patch_size, gw=w // self.cfg.patch_size,
                          digests=[_digest(host[s]) for s in range(S)])
        self._note("im2col", lambda: LP.check_im2col("im2col", out, px16, 3 * self.cfg.patch_size ** 2))
        return out

    def layernorm(self, real, x, gamma, beta, eps, *, add=None, dtype=torch.bfloat16):
        out = real(x, gamma, beta, eps, add=add, dtype=dtype)
        sd, cfg = self.sd, self.cfg
        if self.eng is None:                                     # construction: the resampler's fixed queries
            kind, key, ref_eps, table = "rs_q.ln", "resampler.ln_q", 1e-6, sd["resampler.pos_embed"].double()
            if not torch.equal(x, sd["resampler.query"].float()):
                self.unplaced("construction layernorm of another input")
                return out
        else:
            role = self.roles.get(gamma.data_ptr())
            if role is None or role[0] not in ("vit.ln", "rs.ln_kv", "rs.ln_post"):
                self.unplaced(f"layernorm with gain {role}")
                return out
            kind, key = role
            ref_eps = cfg.ln_eps if kind == "vit.ln" else 1e-6
            table = LP.sincos64(cfg.hidden, self.chunk["gh"], self.chunk["gw"], DEV) if kind == "rs.ln_kv" else None
        if (table is None) != (add is None):
            self.failures.append((kind, f"add table passed: {add is not None}, expected: {table is not None}"))
            return out
        got, got2 = (out, None) if table is None else out
        self._note(kind, lambda: LP.check_layernorm(key, got, x, sd[key + ".weight"], sd[key + ".bias"], ref_eps, add=table,
                                                    got_add=got2))
        return out

    def rmsnorm(self, real, x, gamma, eps, dtype=torch.bfloat16):
        out = real(x, gamma, eps, dtype)
        role = self.roles.get(gamma.data_ptr())
        if role is None or role[0] not in ("lm.rms", "lm.final"):
            self.unplaced(f"rmsnorm with gain {role}")
            return out
        self._note(role[0], lambda: LP.check_rmsnorm(role[1], out, x, self.sd[role[1] + ".weight"], self.cfg.rms_eps))
        return out

    def gemm(self, real, a, w, **kw):
        resid = kw.get("resid")
        resid0 = None if resid is None else resid.clone()
        out = real(a, w, **kw)
        sd, cfg, E = self.sd, self.cfg, self.cfg.hidden
        if self.eng is None:
            Win, b = sd["resampler.attn.in_proj_weight"], sd["resampler.attn.in_proj_bias"]
            self._note("rs_q.gemm", lambda: LP.check_linear("rs_q", out, a, Win[:E], b[:E]))
            self.rs_q = out
            return out
        role = self.roles.get(w.data_ptr())
        if role is None:
            self.unplaced(f"gemm with weight {tuple(w.shape)}")
            return out
        kind, key = role
        s = cfg.scale_depth / cfg.layers ** 0.5
        if kind == "patch":
            ch = self.chunk
            fn = lambda: LP.check_patch(key, out, ch["px16"], sd[key + ".weight"], sd[key + ".bias"], sd["vpm.pos_embed"])  # noqa: E731
        elif kind == "vit.qkv":
            self.last["vit.qkv"] = (out.data_ptr(), LP.vit_qkv_canonical(out, cfg.vit_heads, cfg.vit_head_dim)[0])
            fn = lambda: LP.check_vit_qkv(key, out, a, sd[key + ".weight"], sd[key + ".bias"], cfg.vit_heads,  # noqa: E731
                                          cfg.vit_head_dim)
        elif kind == "vit.proj":
            fn = lambda: LP.check_linear(key, out, a, sd[key + ".weight"], sd[key + ".bias"], resid=resid0)  # noqa: E731
        elif kind == "vit.fc1":
            fn = lambda: LP.check_fc1(key, out, a, sd[key + ".weight"], sd[key + ".bias"])  # noqa: E731
        elif kind == "vit.fc2":
            fn = lambda: LP.check_fc2(key, out, a, sd[key + ".weight"], sd[key + ".bias"], resid0)  # noqa: E731
        elif kind == "rs.kv":
            fn = lambda: LP.check_linear(key, out, a, sd[key + ".weight"])  # noqa: E731
        elif kind in ("rs.k", "rs.v"):
            j = 1 if kind == "rs.k" else 2
            Win, b = sd["resampler.attn.in_proj_weight"], sd["resampler.attn.in_proj_bias"]
            self.last[kind] = out
            fn = lambda: LP.check_linear(key, out, a, Win[j * E:(j + 1) * E], b[j * E:(j + 1) * E])  # noqa: E731
        elif kind == "rs.out":
            fn = lambda: LP.check_linear(key, out, a, sd[key + ".weight"], sd[key + ".bias"])  # noqa: E731
        elif kind == "rs.proj":
            for i, d in enumerate(self.chunk["digests"]):
                self.vision[d] = out[i * cfg.query_num:(i + 1) * cfg.query_num].clone()
            fn = lambda: LP.check_linear(key, out, a, sd["resampler.proj"].t())  # noqa: E731
        elif kind == "lm.qkv":
            self.layer = int(key.split(".")[3])
            self.last["lm.qkv"] = out
            run = self.run
            if "build" in run:
                run.setdefault("kv", []).append(out[:, E:].clone())
            pos = torch.cat([torch.arange(run["p0"], run["p0"] + len(i)) for i in run["ids"]]).to(DEV)
            cos, sin = LP.rope_tables(cfg.head_dim, cfg.rope_theta, int(pos.max()) + 1, DEV)
            fn = lambda: LP.check_rope_qkv(key + "qkv", out, a, *(sd[key + f"self_attn.{n}_proj.weight"] for n in "qkv"),  # noqa: E731
                                           pos, cos, sin)
        elif kind == "lm.o":
            fn = lambda: LP.check_linear(key, out, a, sd[key + ".weight"], scale=s, resid=resid0)  # noqa: E731
        elif kind == "lm.gu":
            fn = lambda: LP.check_swiglu(key, out, a, sd[key + ".gate_proj.weight"], sd[key + ".up_proj.weight"])  # noqa: E731
        else:   # lm.down
            self.last["lm.down"] = out
            if "build" in self.run and self.layer == cfg.layers - 1:
                self.prefixes[self.run["build"]] = dict(kv=self.run["kv"], h=out.clone())
            fn = lambda: LP.check_linear(key, out, a, sd[key + ".weight"], scale=s, resid=resid0)  # noqa: E731
        self._note(kind, fn)
        return out

    def attention(self, real, q, k, v, **kw):
        out = real(q, k, v, **kw)
        cfg = self.cfg
        qp = q.data_ptr()
        if "vit.qkv" in self.last and qp == self.last["vit.qkv"][0]:
            kind, ch = "vit.attn", self.chunk
            nh, hd = cfg.vit_heads, cfg.vit_head_dim
            canon = self.last["vit.qkv"][1]
            N = ch["gh"] * ch["gw"]
            cu = torch.arange(0, (ch["S"] + 1) * N, N, dtype=torch.int32)
            qq, kk, vv = (canon[:, i * nh * hd:(i + 1) * nh * hd] for i in range(3))
            fn = lambda: LP.check_attention("vit attention", out, qq, kk, vv, heads=nh, head_dim=hd, cu_k=cu, cu_q=cu,  # noqa: E731
                                            max_q=N, causal=False, scale=hd ** -0.5)
        elif self.eng is not None and qp == self.eng.rs_q.data_ptr():
            kind, ch = "rs.attn", self.chunk
            N = ch["gh"] * ch["gw"]
            cu = torch.arange(0, (ch["S"] + 1) * N, N, dtype=torch.int32)
            qq, kk, vv = self.rs_q, self.last["rs.k"], self.last["rs.v"]
            fn = lambda: LP.check_attention("resampler attention", out, qq, kk, vv, heads=cfg.hidden // 128, head_dim=128,  # noqa: E731
                                            cu_k=cu, cu_q=None, max_q=cfg.query_num, causal=False, scale=128 ** -0.5)
        elif "lm.qkv" in self.last and qp == self.last["lm.qkv"].data_ptr():
            kind, run, H = "lm.attn", self.run, cfg.hidden
            qkv = self.last["lm.qkv"]
            lens = [len(i) for i in run["ids"]]
            cu_q = torch.tensor([0] + list(np.cumsum(lens)), dtype=torch.int32)
            if "key" in run:        # suffix rows attend over [cached prefix K|V of this layer ; own K|V]
                pkv = self.prefixes[run["key"]]["kv"][self.layer]
                kv = torch.cat([torch.cat([pkv, qkv[int(cu_q[b]):int(cu_q[b + 1]), H:]]) for b in range(len(lens))])
                kk, vv = kv[:, :H], kv[:, H:]
                cu_k = torch.tensor([0] + list(np.cumsum(run["full"])), dtype=torch.int32)
            else:
                kk, vv, cu_k = qkv[:, H:2 * H], qkv[:, 2 * H:], cu_q
            fn = lambda: LP.check_attention("lm attention", out, qkv[:, :H], kk, vv, heads=cfg.heads, head_dim=cfg.head_dim,  # noqa: E731
                                            cu_k=cu_k, cu_q=cu_q, max_q=max(lens), causal=True, scale=cfg.head_dim ** -0.5)
        else:
            self.unplaced("attention reading no recorded q")
            return out
        self._note(kind, fn)
        return out

    def build_lm_input(self, real, src, embed, scale_emb, vision):
        out = real(src, embed, scale_emb, vision)
        if not self.runs or self.roles.get(embed.data_ptr(), ("",))[0] != "lm.input":
            self.unplaced("build_lm_input with no LM run expected")
            return out
        self.run = run = self.runs.pop(0)

        def fn():
            missing = [d for sl in run["slices"] for d in sl if d not in self.vision]
            assert not missing, f"{len(missing)} slices of the oracle's plan went through no resampler launch"
            rows = [[self.vision[d] for d in sl] for sl in run["slices"]]
            return LP.check_lm_input("lm input", out, self.sd["llm.model.embed_tokens.weight"], self.cfg.scale_emb,
                                     run["ids"], run["bounds"], rows, self.dt)
        self._note("lm.input", fn)
        return out

    def prefix_rows(self, real, prefix, rows, out, cu_rows, cu_out):
        res = real(prefix, rows, out, cu_rows, cu_out)
        run, H = self.run, self.cfg.hidden
        ent = self.prefixes.get(run.get("key"))
        if ent is None:
            self.unplaced("prefix_rows outside a cached-prefix run")
            return res
        if out.dtype == torch.float32:
            pre, own = ent["h"], self.last["lm.down"]
        else:
            pre, own = ent["kv"][self.layer], self.last["lm.qkv"][:, H:]
        cu = np.cumsum([0] + [len(i) for i in run["ids"]])
        want = torch.cat([torch.cat([pre, own[cu[b]:cu[b + 1]]]) for b in range(len(cu) - 1)])

        def fn():
            assert torch.equal(out, want), "prefix_rows: rows differ from [cached prefix ; own rows]"
            return {"frac": 0.0}
        self._note("lm.prefix_rows", fn)
        return res

    def pool_norm(self, real, h, gamma, eps, cu, pooling, normalize):
        out = real(h, gamma, eps, cu, pooling, normalize)
        if self.roles.get(gamma.data_ptr(), ("",))[0] != "lm.final" or self.pooling is None:
            self.unplaced("pool_norm")
            return out
        self._note("pool", lambda: LP.check_pool("pool_norm", out, h, self.sd["llm.model.norm.weight"], self.cfg.rms_eps,
                                                 self.run["full"], self.pooling, normalize))
        return out

    def report(self, title):
        print(f"\n{title}: kind, launches, worst fraction of the bound")
        for k in sorted(self.stats):
            print(f"  {k:15s} {self.stats[k][0]:5d}  {self.stats[k][1]:.3f}")
        for kind, msg in self.failures[:8]:
            print(f"  FAILED {kind}: {msg}")


OPS = ("gemm", "attention", "layernorm", "rmsnorm", "im2col_norm", "build_lm_input", "prefix_rows", "pool_norm")


@pytest.fixture
def parity(monkeypatch):
    """Wraps the ops entry points; `make(cfg, sd, dtype)` starts a Recorder the wrappers report to."""
    from visrag_b200 import ops

    state = {}
    for name in OPS:
        real = getattr(ops, name)
        monkeypatch.setattr(ops, name, lambda *a, _n=name, _r=real, **k: getattr(state["rec"], _n)(_r, *a, **k)
                            if "rec" in state else _r(*a, **k))

    def make(cfg, sd, dtype):
        state["rec"] = Recorder(cfg, sd, dtype)
        return state["rec"]

    return make


def _engine(rec, cfg, sd_host, **kw):
    from visrag_b200.encoder import VisRAGEngine

    eng = VisRAGEngine(cfg, sd_host, cuda_graphs=False, dtype=rec.dt, **kw)
    rec.bind(eng)
    return eng


def expected_counts(cfg, calls):
    """Launches per kind for a list of (plan, prefix mode or None, pooled) encode calls and the engines built (rs_q)."""
    n = Counter()
    for plan, prefix, pooled in calls:
        groups = len(plan.geoms)
        n.update({"im2col": groups, "patch": groups, "vit.ln": groups * (2 * cfg.vit_depth + 1)})
        n.update({k: groups * cfg.vit_depth for k in ("vit.qkv", "vit.attn", "vit.proj", "vit.fc1", "vit.fc2")})
        n.update({k: groups for k in ("rs.kv", "rs.ln_kv", "rs.k", "rs.v", "rs.attn", "rs.out", "rs.ln_post", "rs.proj")})
        runs = 1 + (prefix is not None and prefix[0] == "create")
        n.update({"lm.input": runs, "lm.rms": 2 * cfg.layers * runs})
        n.update({k: cfg.layers * runs for k in ("lm.qkv", "lm.attn", "lm.o", "lm.gu", "lm.down")})
        if prefix is not None:
            n["lm.prefix_rows"] += cfg.layers + 1
        n["pool" if pooled else "lm.final"] += 1
    return +n


def _lcp(plan):
    ids = plan.ids
    n = min(len(i) for i in ids) - 1
    for t in range(n):
        if any(i[t] != ids[0][t] for i in ids):
            return t
    return n


def _queries(words):
    return [QUERY_PREFIX + w for w in words]


def _encode(rec, eng, tok, texts, images, pooling="wmean", prefix=None, calls=None):
    plan = Plan(rec.cfg, tok, texts, images)
    if prefix == "create":
        prefix = ("create", _lcp(plan))
    elif prefix == "hit":
        prefix = ("hit", max((len(k) for k in rec.prefixes if all(tuple(int(t) for t in i[:len(k)]) == k for i in plan.ids)),
                             default=0))
    rec.expect(plan, pooling, prefix)
    got = eng.encode(texts, images, tok, max_inp_length=MAX_INP, pooling=pooling)
    if calls is not None:
        calls.append((plan, prefix, True))
    assert not rec.runs, "an expected LM run did not happen"
    return got


def _check_all(rec, cfg, calls, engines, title):
    rec.report(title)
    assert not rec.failures, rec.failures[:5]
    want = expected_counts(cfg, calls) + Counter({"rs_q.ln": engines, "rs_q.gemm": engines})
    assert Counter({k: v[0] for k, v in rec.stats.items()}) == want


# ------------------------------------------------------------------------------------------------------- tiny model


@pytest.fixture(scope="module")
def tiny():
    from visrag_b200.config import VisRAGConfig
    from visrag_b200.tokenizer_stub import StubTokenizer
    from visrag_b200.weights import random_state_dict

    cfg = VisRAGConfig.tiny()
    sd = random_state_dict(cfg, 31337)
    return cfg, sd, {k: v.to(DEV) for k, v in sd.items()}, StubTokenizer(cfg.vocab)


# pages: square single slice, tall 1 + 8 slices, square 1 + 9, near-square single, wide 1 + 2, very tall and very wide
TINY_PAGES = [(224, 224), (282, 1520), (1344, 1344), (336, 340), (1280, 400), (600, 8000), (3000, 100)]


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_every_launch_of_tiny_encodes(parity, tiny, dtype):
    """Pages of several geometry groups (tall, wide, multi-slice) with and without text, every pooling, text items next to
    pages, a query batch that creates a prefix-cache entry and one that hits it, and the B1 boundary (VisRAGRetB200)."""
    from visrag_b200.modeling import VisRAGRetB200

    cfg, sd_host, sd, tok = tiny
    rec = parity(cfg, sd, dtype)
    eng = _engine(rec, cfg, sd_host)
    pages = synth_pages(TINY_PAGES, 77)
    texts = ["", "a caption", "", "x", "", "", "tall and wide"]
    calls = []
    for pooling in ("wmean", "mean", "lasttoken", "cls"):
        _encode(rec, eng, tok, texts, pages, pooling, calls=calls)
    _encode(rec, eng, tok, ["", "revenue table", ""], [pages[1], None, pages[4]], calls=calls)
    _encode(rec, eng, tok, _queries(["a", "chart of the energy policy", "x y"]), [None] * 3, prefix="create", calls=calls)
    _encode(rec, eng, tok, _queries(["growth", "network model summary"]), [None] * 2, prefix="hit", calls=calls)
    assert eng.prefix_stats["created"] == 1 and eng.prefix_stats["hits"] == 1
    rec.eng = None                                      # its construction launches (the resampler's queries)
    b1 = VisRAGRetB200(cfg, sd_host, dtype=dtype)
    rec.bind(b1.engine)
    plan = Plan(cfg, tok, texts[:3], pages[:3])
    rec.expect(plan, pooled=False)
    b1(text=texts[:3], image=pages[:3], tokenizer=tok, max_inp_length=MAX_INP)
    calls.append((plan, None, False))
    _check_all(rec, cfg, calls, 2, f"tiny {dtype}")


# ------------------------------------------------------------------------------------------------------- full model


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_every_launch_of_full_size_encodes(parity, dtype):
    """SigLIP-so400m + Resampler + MiniCPM-2B: one wide page cut into 1 + 2 slices of two geometries, and two queries that
    create a prefix-cache entry."""
    from visrag_b200.config import VisRAGConfig
    from visrag_b200.tokenizer_stub import StubTokenizer
    from visrag_b200.weights import random_state_dict_device

    cfg = VisRAGConfig.full()
    sd = random_state_dict_device(cfg, 2024, DEV)
    tok = StubTokenizer(cfg.vocab)
    rec = parity(cfg, sd, dtype)
    eng = _engine(rec, cfg, sd)
    calls = []
    _encode(rec, eng, tok, [""], synth_pages([(700, 300)], 5), calls=calls)
    _encode(rec, eng, tok, _queries(["climate chart", "total revenue in 2020"]), [None, None], prefix="create", calls=calls)
    assert len(calls[0][0].geoms) == 2 and len(calls[0][0].slices[0]) == 3
    _check_all(rec, cfg, calls, 1, f"full {dtype}")


# ----------------------------------------------------------------------------------------------------- engine mutants


def _mutant_sincos_transposed(monkeypatch, eng):
    from visrag_b200.encoder import VisRAGEngine

    orig = VisRAGEngine._sincos_table
    monkeypatch.setattr(VisRAGEngine, "_sincos_table", lambda self, gh, gw: orig(self, gw, gh))


def _mutant_pos_bilinear(monkeypatch, eng):
    from visrag_b200.encoder import VisRAGEngine

    def table(self, gh, gw):
        S, D = self.cfg.vit_pos_grid, self.cfg.vit_dim
        p = self.pos_embed.reshape(1, S, S, D).permute(0, 3, 1, 2)
        p = torch.nn.functional.interpolate(p, size=(gh, gw), mode="bilinear", antialias=True)
        return p.permute(0, 2, 3, 1).reshape(gh * gw, D).contiguous().to(self.device)
    monkeypatch.setattr(VisRAGEngine, "_pos_table", table)


def _mutant_rope_theta(monkeypatch, eng):
    cfg = eng.cfg
    inv = 1.0 / ((1.5 * cfg.rope_theta) ** (torch.arange(0, cfg.head_dim, 2).float() / cfg.head_dim))
    fr = torch.outer(torch.arange(cfg.max_pos).float(), inv)
    eng.rope_cos, eng.rope_sin = fr.cos().to(eng.device), fr.sin().to(eng.device)


def _mutant_pool_mean(monkeypatch, eng):
    from visrag_b200 import ops

    checked = ops.pool_norm
    monkeypatch.setattr(ops, "pool_norm", lambda h, g, eps, cu, pooling, normalize:
                        checked(h, g, eps, cu, "mean" if pooling == "wmean" else pooling, normalize))


def _mutant_resampler_kv_swapped(monkeypatch, eng):
    from visrag_b200 import ops

    checked = ops.attention

    def attention(q, k, v, **kw):
        if q.data_ptr() == eng.rs_q.data_ptr():
            k, v = v, k
        return checked(q, k, v, **kw)
    monkeypatch.setattr(ops, "attention", attention)


def _mutant_suffix_positions(monkeypatch, eng):
    from visrag_b200 import encoder

    orig = encoder.suffix_batch

    def suffix_batch(pb, prefix_len):
        sb = orig(pb, prefix_len)
        sb.positions = sb.positions - prefix_len
        return sb
    monkeypatch.setattr(encoder, "suffix_batch", suffix_batch)


# name -> (engine-side mutation or None, engine config change, the launch kind that must reject it)
MUTANTS = {
    "sincos table gh, gw swapped": (_mutant_sincos_transposed, {}, "rs.ln_kv"),
    "ViT position table bilinear": (_mutant_pos_bilinear, {}, "patch"),
    "RoPE tables from theta x 1.5": (_mutant_rope_theta, {}, "lm.qkv"),
    "ViT LayerNorm eps 1e-5": (None, {"ln_eps": 1e-5}, "vit.ln"),
    "pool_norm mean for wmean": (_mutant_pool_mean, {}, "pool"),
    "resampler k and v swapped": (_mutant_resampler_kv_swapped, {}, "rs.attn"),
    "suffix positions not offset by P": (_mutant_suffix_positions, {}, "lm.qkv"),
}


@pytest.fixture(scope="module")
def mutant_case(tiny):
    from oracle import restated as O

    cfg, sd_host, _, tok = tiny
    pages = synth_pages([(282, 1520), (1280, 400)], 77)
    texts = ["", "a caption"]
    queries = _queries(["energy chart", "policy summary of the network"])
    return pages, texts, queries, O.encode(sd_host, cfg, tok, texts, pages), O.encode(sd_host, cfg, tok, queries, [None] * 2)


@pytest.mark.parametrize("name", list(MUTANTS))
def test_engine_mutant_is_rejected_at_its_launch(parity, tiny, mutant_case, monkeypatch, name):
    """Each mutant changes one piece of the engine's wiring; its embeddings stay close to the oracle's (printed), but the
    launch it touches fails its check, and no other launch does."""
    cfg, sd_host, sd, tok = tiny
    mutate, change, kind = MUTANTS[name]
    pages, texts, queries, want_p, want_q = mutant_case
    rec = parity(cfg, sd, torch.bfloat16)
    from visrag_b200.encoder import VisRAGEngine

    eng = VisRAGEngine(dataclasses.replace(cfg, **change), sd_host, cuda_graphs=False, dtype=torch.bfloat16)
    rec.bind(eng)
    if mutate is not None:
        mutate(monkeypatch, eng)
    p = _encode(rec, eng, tok, texts, pages)
    q = _encode(rec, eng, tok, queries, [None] * 2, prefix="create")
    cos = min(cosine_rows(p.cpu().numpy(), want_p).min(), cosine_rows(q.cpu().numpy(), want_q).min())
    failed = Counter(k for k, _ in rec.failures)
    print(f"\nmutant '{name}': end-to-end cos min {cos:.7f}; rejected at {dict(failed)}; first: "
          f"{rec.failures[0][1] if rec.failures else None}")
    assert set(failed) == {kind}, (name, dict(failed))
