"""Host side of the prefix cache (host.select_prefix, host.suffix_batch): which cached token prefix a batch runs from,
when a batch creates one, and the suffix layout the cached LM path consumes. Pure numpy, no GPU."""
import numpy as np

from visrag_b200.config import VisRAGConfig
from visrag_b200.host import PREFIX_MIN_TOKENS, PreparedBatch, prepare_batch, select_prefix, suffix_batch
from visrag_b200.synth import QUERY_PREFIX, synth_pages, synth_queries
from visrag_b200.tokenizer_stub import StubTokenizer

CFG = VisRAGConfig.tiny()
TOK = StubTokenizer(CFG.vocab)


def _batch(id_lists):
    """A text-only PreparedBatch from explicit token ids."""
    lens = np.asarray([len(x) for x in id_lists], dtype=np.int32)
    cu = np.zeros(len(lens) + 1, dtype=np.int32)
    np.cumsum(lens, out=cu[1:])
    src = np.concatenate([-(np.asarray(x, dtype=np.int64) + 1) for x in id_lists]).astype(np.int32)
    pos = np.concatenate([np.arange(n, dtype=np.int32) for n in lens])
    return PreparedBatch(len(lens), lens, cu, pos, src)


def _texts(texts):
    return prepare_batch(texts, [None] * len(texts), TOK, CFG, 2048)


def test_new_entry_is_the_longest_common_id_prefix():
    pb = _batch([list(range(1, 21)) + [50, 51], list(range(1, 21)) + [60], list(range(1, 21)) + [70, 71, 72]])
    assert select_prefix(pb, []) == (tuple(range(1, 21)), True)
    pb = _texts(synth_queries(64, 7))
    ids, new = select_prefix(pb, [])
    assert new and len(ids) >= len(TOK.encode(QUERY_PREFIX))
    for b in range(pb.n_items):
        assert tuple(-(pb.token_src[pb.cu_seqlens[b]:pb.cu_seqlens[b] + len(ids)] + 1)) == ids


def test_longest_applicable_entry_wins():
    pb = _batch([list(range(1, 31)) + [90], list(range(1, 31)) + [91, 92]])
    cached = [tuple(range(1, 11)), tuple(range(1, 26)), tuple(range(1, 21)), tuple(range(1, 26)) + (99,)]
    assert select_prefix(pb, cached) == (tuple(range(1, 26)), False)
    # an entry that does not start every item is skipped, even when it is the longest
    pb2 = _batch([list(range(1, 31)) + [90], [7] + list(range(2, 31))])
    assert select_prefix(pb2, cached) is None


def test_p_max_cap_keeps_one_token_per_item():
    base = list(range(1, 41))
    pb = _batch([base, base + [5, 6], base + [7]])          # the shortest item is all prefix
    ids, new = select_prefix(pb, [])
    assert new and ids == tuple(base[:39])                   # P_max = 40 - 1
    assert select_prefix(pb, [tuple(base)]) == (tuple(base[:39]), True)   # the 40-token entry is too long for it
    assert select_prefix(pb, [tuple(base[:30]), tuple(base)]) == (tuple(base[:30]), False)
    same = _batch([base, base])                              # identical items: capped at P_max as well
    assert select_prefix(same, []) == (tuple(base[:39]), True)


def test_item_equal_to_a_cached_prefix_plus_one_token():
    base = tuple(range(3, 3 + 12))
    pb = _batch([list(base) + [1]])
    assert select_prefix(pb, [base]) == (base, False)
    assert select_prefix(_batch([list(base)]), [base]) is None    # nothing of its own would be left


def test_threshold():
    n = PREFIX_MIN_TOKENS
    short = _batch([list(range(1, n)) + [100, 101], list(range(1, n)) + [200]])        # n - 1 shared tokens
    assert select_prefix(short, []) is None
    exact = _batch([list(range(1, n + 1)) + [100], list(range(1, n + 1)) + [200]])     # n shared tokens
    assert select_prefix(exact, []) == (tuple(range(1, n + 1)), True)
    assert select_prefix(exact, [], min_tokens=n + 1) is None
    # an existing entry below the threshold still applies (it was created under another setting or by another batch)
    assert select_prefix(short, [tuple(range(1, 5))]) == (tuple(range(1, 5)), False)


def test_single_item_only_uses_an_existing_entry():
    one = _batch([list(range(1, 40))])
    assert select_prefix(one, []) is None
    assert select_prefix(one, [tuple(range(1, 21))]) == (tuple(range(1, 21)), False)


def test_batches_with_slices_never_qualify():
    pages = synth_pages([(448, 448), (448, 448)], 1)
    pb = prepare_batch(["", ""], pages, TOK, CFG, 2048)
    assert pb.n_slices > 0 and select_prefix(pb, []) is None
    mixed = prepare_batch([QUERY_PREFIX + "a b", QUERY_PREFIX + "c d", ""], [None, None, pages[0]], TOK, CFG, 2048)
    assert select_prefix(mixed, []) is None
    ids = tuple(TOK.encode(QUERY_PREFIX))[:8]
    assert select_prefix(mixed, [ids]) is None


def test_selection_is_deterministic():
    qs = synth_queries(32, 3)
    pb = _texts(qs)
    first = select_prefix(pb, [])
    cached = [first[0][:9], first[0], first[0][:20]]
    for _ in range(3):
        assert select_prefix(_texts(qs), []) == first
        assert select_prefix(pb, cached) == (first[0], False)
        assert select_prefix(pb, list(reversed(cached))) == (first[0], False)


def test_suffix_batch_layout():
    base = list(range(1, 11))
    pb = _batch([base + [50], base + [60, 61, 62], base + [70, 71]])
    sb = suffix_batch(pb, 10)
    assert sb.n_items == 3 and list(sb.seq_lens) == [1, 3, 2] and list(sb.cu_seqlens) == [0, 1, 4, 6]
    assert list(sb.positions) == [10, 10, 11, 12, 10, 11]                     # absolute positions
    assert list(-(sb.token_src + 1)) == [50, 60, 61, 62, 70, 71]
