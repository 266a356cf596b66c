"""The prefix cache must not change a bit. A text-only batch whose items share a cached token prefix runs only the
suffixes through the LM; that rests on three kernel facts checked here, then on the engine end to end:
  * attention with fewer query rows than key rows (the queries are the last rows of each causal sequence) gives the
    same bits as the matching rows of the full causal run, and stays within the float64 bound of tests/kernel_bounds.py;
  * vr_prefix_rows writes exactly the [prefix ; own rows] layout, every target row and nothing else;
  * the engine with the cache equals the engine without it, for every pooling, both dtypes, graphs on and off."""
import ctypes as C

import numpy as np
import pytest
import torch

from tests import kernel_bounds as KB
from tests import kernel_bounds_f16 as KF

pytestmark = pytest.mark.gpu

DEV = "cuda"
DTYPES = [torch.bfloat16, torch.float16]
DT_IDS = ["bf16", "fp16"]


def _cu(lens):
    return torch.tensor([0] + list(np.cumsum(lens)), dtype=torch.int32, device=DEV)


@pytest.fixture(params=[0, 1], ids=["auto", "single_tile"])
def attn_variant(request):
    from visrag_b200 import _lib as L

    L.lib().vr_attention_force_v1(request.param)
    yield request.param
    L.lib().vr_attention_force_v1(0)


# ----------------------------------------------------------------------------------------------------------- attention

PREFIXES = [1, 9, 57, 127, 128, 129, 300]
SUFFIXES = [1, 17, 64, 65, 200]


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("S", SUFFIXES)
def test_attention_suffix_queries_equal_full_causal_rows(dtype, S, attn_variant):
    """Seven sequences per launch, one per prefix length P, each with S query rows: the suffix launch (cu_q = suffixes,
    cu_k = full sequences) against the full causal launch over the same qkv rows."""
    from visrag_b200 import ops

    nh, hd = 4, 64
    H = nh * hd
    full = [P + S for P in PREFIXES]
    cu_full = _cu(full)
    cu_s = _cu([S] * len(PREFIXES))
    gen = torch.Generator(device=DEV).manual_seed(S * 7 + (dtype == torch.float16))
    qkv = (torch.randn(sum(full), 3 * H, device=DEV, generator=gen) * 1.5).to(dtype)
    rows = torch.cat([torch.arange(int(cu_full[b]) + P, int(cu_full[b + 1]), device=DEV) for b, P in enumerate(PREFIXES)])
    kw = dict(k_col0=H, v_col0=2 * H, head_stride=64, head_dim=hd, heads=nh, batch=len(full), causal=True, scale=hd ** -0.5)
    want = torch.full((sum(full), H), float("nan"), dtype=dtype, device=DEV)
    ops.attention(qkv, qkv, qkv, q_col0=0, cu_k=cu_full, max_k=max(full), cu_q=cu_full, max_q=max(full), out=want, **kw)
    q = qkv[rows].contiguous()
    got = torch.full((rows.numel(), H), float("nan"), dtype=dtype, device=DEV)
    ops.attention(q, qkv, qkv, q_col0=0, cu_k=cu_full, max_k=max(full), cu_q=cu_s, max_q=S, out=got, **kw)
    assert torch.equal(got, want[rows]), (got.float() - want[rows].float()).abs().max()
    ref_fn, check = (KB.attention_ref, KB.check) if dtype == torch.bfloat16 else (KF.attention_ref_f16, KF.check)
    ref, e = ref_fn(q, qkv, qkv, q_col0=0, k_col0=H, v_col0=2 * H, head_stride=64, head_dim=hd, heads=nh, cu_k=cu_full,
                    cu_q=cu_s, max_q=S, causal=True, scale=hd ** -0.5)
    check(f"suffix attention S={S} {dtype}", got, ref, e)


# ------------------------------------------------------------------------------------------------------ vr_prefix_rows


def _gather_ref(prefix, rows, lens):
    """[prefix ; rows of sequence b] for every b, by torch indexing."""
    parts, r0 = [], 0
    for n in lens:
        parts += [prefix, rows[r0:r0 + n]]
        r0 += n
    return torch.cat(parts)


@pytest.mark.parametrize("kind", ["kv16", "h32"])
@pytest.mark.parametrize("P,lens", [(1, [1]), (1, [1, 1, 1]), (57, [1]), (57, [1, 17, 200, 3]), (5, [1] * 100),
                                    (130, [64, 65, 0, 128])])
def test_prefix_rows_equals_a_gather(kind, P, lens):
    """Into a NaN-poisoned buffer with a margin of rows and columns around the target: the target equals the gather and
    the margin is untouched. kv16: the K|V column block of a wider qkv row (as the engine passes it); h32: fp32 rows."""
    from visrag_b200 import ops

    H = 256
    T = sum(lens)
    gen = torch.Generator(device=DEV).manual_seed(P * 1000 + T)
    if kind == "kv16":
        qkv = torch.randn(T, 3 * H, device=DEV, generator=gen).bfloat16()
        rows = qkv[:, H:]
        store = torch.randn(3, P, 2 * H, device=DEV, generator=gen).bfloat16()   # a layer of a [layers, P, 2H] entry
        prefix = store[1]
    else:
        rows = torch.randn(T, H, device=DEV, generator=gen)
        prefix = torch.randn(P, H, device=DEV, generator=gen)
    cols = rows.shape[1]
    n_out = T + P * len(lens)
    buf = torch.full((n_out + 3, cols + 16), float("nan"), dtype=rows.dtype, device=DEV)
    out = buf[1:1 + n_out, 8:8 + cols]
    ops.prefix_rows(prefix, rows, out, _cu(lens), _cu([P + n for n in lens]))
    assert torch.equal(out, _gather_ref(prefix, rows, lens))
    margin = torch.ones_like(buf, dtype=torch.bool)
    margin[1:1 + n_out, 8:8 + cols] = False
    assert torch.isnan(buf[margin].float()).all()


def test_prefix_rows_refuses_bad_shapes():
    """Misaligned columns, leading dimensions or pointers and bad element sizes return an error before any launch."""
    from visrag_b200 import _lib as L

    lib = L.lib()
    buf = torch.zeros(64, 64, dtype=torch.bfloat16, device=DEV)
    cu = _cu([2])
    cu_out = _cu([3])
    p = buf.data_ptr()

    def call(prefix=p, ldp=64, rows=p, ldr=64, out=p, ldo=64, P=1, out_rows=3, cols=64, elem=2):
        return lib.vr_prefix_rows(prefix, ldp, rows, ldr, out, ldo, cu.data_ptr(), cu_out.data_ptr(), 1, P, out_rows, cols,
                                  elem, C.c_void_p(torch.cuda.current_stream().cuda_stream))

    assert call() == 0
    torch.cuda.synchronize()
    for bad in (dict(cols=4), dict(cols=12), dict(ldo=60), dict(ldp=63), dict(rows=p + 2), dict(out=p + 8), dict(elem=3),
                dict(elem=1), dict(ldr=32), dict(P=-1), dict(out_rows=0), dict(prefix=None)):
        assert call(**bad) != 0, bad
        assert lib.vr_last_error()


# -------------------------------------------------------------------------------------------------------------- engine

POOLINGS = ["wmean", "mean", "lasttoken", "cls"]


def _words(rs, n_chars):
    return "".join(rs.choice(list("abcdefghijklmnopqrstuvwxyz "), n_chars))


def _queries(prefix, suffix_chars, seed):
    """prefix + n characters each; consecutive suffixes start with different letters, so that the common prefix of a
    batch is `prefix` itself."""
    rs = np.random.RandomState(seed)
    return [prefix + "abcdefghijklmnopqrstuvwxyz"[i % 26] + _words(rs, n - 1) for i, n in enumerate(suffix_chars)]


def _pair(dtype, graphs, seed=5):
    from visrag_b200.config import VisRAGConfig
    from visrag_b200.encoder import VisRAGEngine
    from visrag_b200.weights import random_state_dict

    cfg = VisRAGConfig.tiny()
    sd = random_state_dict(cfg, seed)
    return (cfg, VisRAGEngine(cfg, sd, cuda_graphs=graphs, dtype=dtype, prefix_cache=True),
            VisRAGEngine(cfg, sd, cuda_graphs=graphs, dtype=dtype, prefix_cache=False))


@pytest.mark.parametrize("graphs", [False, True], ids=["eager", "graphs"])
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_engine_cache_on_equals_off(dtype, graphs):
    from visrag_b200.encoder import GRAPH_MAX_LM_TOKENS
    from visrag_b200.synth import QUERY_PREFIX
    from visrag_b200.tokenizer_stub import StubTokenizer

    cfg, on, off = _pair(dtype, graphs)
    tok = StubTokenizer(cfg.vocab)
    long_prefix = "Given the following long instruction, " * 4        # 152 characters: a prefix longer than 128 tokens
    cases = [
        _queries(QUERY_PREFIX, [5, 40], 1),                                   # creates the 57-token entry
        _queries(QUERY_PREFIX, [3], 2),                                       # a single query on the entry
        [QUERY_PREFIX + "z"],                                                 # the prefix plus one token
        _queries(QUERY_PREFIX, [63, 64, 65, 127, 128, 129, 200, 1] * 2, 3),  # 16: suffixes crossing 64 and 128
        _queries(QUERY_PREFIX, list(np.random.RandomState(4).randint(1, 60, 128)), 4),   # 128
        _queries(long_prefix, [10, 70], 5),
        _queries(long_prefix, [1, 130, 64], 6),
        _queries(QUERY_PREFIX, [120] * 40, 7),                               # above GRAPH_MAX_LM_TOKENS: eager even with graphs
    ]
    assert sum(len(tok.encode(q)) for q in cases[-1]) > GRAPH_MAX_LM_TOKENS
    for rep in range(2):                                                      # graphs: eager, capture, then replay
        for qs in cases:
            for pooling in POOLINGS:
                a = on.encode(qs, [None] * len(qs), tok, pooling=pooling)
                b = off.encode(qs, [None] * len(qs), tok, pooling=pooling)
                assert a.shape == (len(qs), cfg.hidden) and torch.equal(a, b), (len(qs), pooling, rep)
    st = on.prefix_stats
    assert st["created"] == 2 and st["hits"] > 0, st
    assert off.prefix_stats == {"created": 0, "hits": 0, "tokens_skipped": 0}
    if graphs:
        assert on.graph_stats["replayed"] > 0


def test_engine_stats_hidden_rows_eviction_and_pages():
    from visrag_b200.encoder import PREFIX_CACHE
    from visrag_b200.host import prepare_batch
    from visrag_b200.synth import QUERY_PREFIX, synth_pages
    from visrag_b200.tokenizer_stub import StubTokenizer

    cfg, on, off = _pair(torch.bfloat16, True, seed=11)
    tok = StubTokenizer(cfg.vocab)
    P = len(tok.encode(QUERY_PREFIX))
    # pages only, and pages next to queries: the full path, stats stay at zero
    pages = synth_pages([(448, 448), (300, 500)], 2)
    mixed_q = _queries(QUERY_PREFIX, [10, 20], 1)
    assert torch.equal(on.encode(["", ""], pages, tok), off.encode(["", ""], pages, tok))
    texts, imgs = ["", mixed_q[0], "", mixed_q[1]], [pages[0], None, pages[1], None]
    assert torch.equal(on.encode(texts, imgs, tok), off.encode(texts, imgs, tok))
    assert on.prefix_stats == {"created": 0, "hits": 0, "tokens_skipped": 0}
    # creation counts the items after the first, a hit counts every item
    qs = _queries(QUERY_PREFIX, [7, 30, 90], 2)
    created = on.encode(qs, [None] * 3, tok)
    assert on.prefix_stats == {"created": 1, "hits": 0, "tokens_skipped": 2 * P}
    # a hit in a batch of another composition: the same bits as the batch that created the entry
    other = on.encode([qs[2], _queries(QUERY_PREFIX, [200], 3)[0], qs[0]], [None] * 3, tok)
    assert torch.equal(other[0], created[2]) and torch.equal(other[2], created[0])
    assert on.prefix_stats == {"created": 1, "hits": 1, "tokens_skipped": 5 * P}
    # return_hidden: the full sequences' residual rows, equal to the full path's
    pb = prepare_batch(qs, [None] * 3, tok, cfg, 2048)
    r_on, h_on = on.encode_prepared(pb, return_hidden=True)
    r_off, h_off = off.encode_prepared(pb, return_hidden=True)
    assert torch.equal(r_on, r_off) and torch.equal(h_on, h_off) and h_on.shape == (int(pb.cu_seqlens[-1]), cfg.hidden)
    # eviction: PREFIX_CACHE other prefixes push the first out; re-creating it gives the same bits
    for i in range(PREFIX_CACHE):
        pfx = f"Instruction number {i} for this engine: "
        q2 = _queries(pfx, [5, 9], 10 + i)
        assert torch.equal(on.encode(q2, [None] * 2, tok), off.encode(q2, [None] * 2, tok))
    assert on.prefix_stats["created"] == 1 + PREFIX_CACHE
    again = on.encode(qs, [None] * 3, tok)
    assert on.prefix_stats["created"] == 2 + PREFIX_CACHE and torch.equal(again, created)
    assert all(s[-1] != ("prefix", 1) for s in on._graphs)                   # graphs of the evicted entry are gone


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_full_size_cache_on_equals_off(dtype, golden_dir):
    """The full model: the golden queries plus synthetic ones. The suffix GEMMs run M <= 128 rows (the 128 x 64 tile
    kernel) where the full path's M is above 128 (the ping-pong kernel): the rows must still agree bit for bit."""
    import os

    from visrag_b200.config import VisRAGConfig
    from visrag_b200.encoder import VisRAGEngine
    from visrag_b200.synth import synth_queries
    from visrag_b200.tokenizer_stub import StubTokenizer
    from visrag_b200.weights import random_state_dict_device

    z = np.load(os.path.join(golden_dir, "full_v2.npz"), allow_pickle=False)
    golden_q = [str(q) for q in z["queries"]]
    cfg = VisRAGConfig.full()
    sd = random_state_dict_device(cfg, int(z["weight_seed"]), "cuda:0")   # exactness needs no golden weights
    on = VisRAGEngine(cfg, sd, dtype=dtype, prefix_cache=True)
    off = VisRAGEngine(cfg, sd, dtype=dtype, prefix_cache=False)
    del sd
    tok = StubTokenizer(cfg.vocab)
    qs = synth_queries(40, 7)
    for batch in (qs[:2] + golden_q, qs[2:4], qs[4:5], qs[5:40]):
        a, b = on.encode(batch, [None] * len(batch), tok), off.encode(batch, [None] * len(batch), tok)
        assert torch.equal(a, b), (len(batch), (a - b).abs().max().item())
    assert on.prefix_stats["created"] >= 1 and on.prefix_stats["hits"] >= 2, on.prefix_stats
