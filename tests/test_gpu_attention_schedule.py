"""The two-warpgroup attention kernel (pipelined, ping-pong between warpgroups) on the tile layouts its schedule has to get
right, against the float64 reference and error bound of tests/kernel_bounds.py: many more tiles than SMs with ragged
and zero-length sequences, tile counts around the SM count, and causal batches where whole q-tiles and whole
warpgroups lie past the end of a sequence (those warpgroups still take their turns)."""
import numpy as np
import pytest
import torch

from tests import kernel_bounds as KB

pytestmark = pytest.mark.gpu

DEV = "cuda"


def _cu(lens):
    return torch.tensor([0] + list(np.cumsum(lens)), dtype=torch.int32, device=DEV)


def _qkv(lens, nh, hd, hs, seed):
    T = sum(lens)
    g = torch.Generator(device=DEV).manual_seed(seed)
    qkv = torch.zeros(max(T, 1), 3, nh, hs, device=DEV)
    qkv[:T, ..., :hd] = torch.randn(T, 3, nh, hd, device=DEV, generator=g)
    return qkv.reshape(max(T, 1), 3 * nh * hs).bfloat16()


def _attend(name, lens, nh, hd, hs, causal, seed):
    from visrag_b200 import ops

    assert max(lens) > 64, "the two-warpgroup kernel serves sequences longer than 64 queries"
    qkv = _qkv(lens, nh, hd, hs, seed)
    cu = _cu(lens)
    out = torch.zeros(qkv.shape[0], nh * hd, dtype=torch.bfloat16, device=DEV)
    kw = dict(q_col0=0, k_col0=nh * hs, v_col0=2 * nh * hs, head_stride=hs, head_dim=hd, heads=nh, causal=causal,
              scale=hd ** -0.5)
    ops.attention(qkv, qkv, qkv, batch=len(lens), cu_k=cu, max_k=max(lens), cu_q=cu, max_q=max(lens), out=out, **kw)
    ref, e = KB.attention_ref(qkv, qkv, qkv, cu_k=cu, cu_q=cu, max_q=max(lens), **kw)
    T = sum(lens)
    return KB.check(name, out[:T], ref[:T], e[:T])


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.parametrize("causal", [False, True], ids=["vit", "causal"])
def test_many_tiles_ragged_and_empty_sequences(causal):
    """Zero-length sequences between ragged ones; with max_q 1036 every sequence spans 9 q-tiles, most of them empty."""
    lens = [1024, 0, 300, 0, 0, 129, 1, 784, 0, 128, 1036, 65, 0, 200, 513]
    _attend(f"ragged causal={causal}", lens, 8, 72, 80, causal, 11 + causal)
    _attend(f"ragged d64 causal={causal}", lens, 6, 64, 64, causal, 13 + causal)


@pytest.mark.parametrize("causal", [False, True], ids=["noncausal", "causal"])
def test_head_stride_128_two_warpgroups(causal):
    """Head stride 128 with more than 64 queries: two warpgroups per CTA, each taking each key tile in turn."""
    _attend(f"d128 causal={causal}", [300, 129, 0, 65, 1036], 3, 128, 128, causal, 21 + causal)


@pytest.mark.parametrize("delta", [-1, 0, 1])
def test_tile_count_around_sm_count(delta):
    """One 128-query tile per sequence and head: #SMs - 1, #SMs and #SMs + 1 tiles in one launch. With one CTA per SM,
    that is one wave one CTA short, one full wave, and one full wave plus a second wave of a single CTA."""
    n = _sms() + delta
    rs = np.random.RandomState(n)
    lens = [int(x) for x in rs.randint(65, 129, size=n)]
    _attend(f"{n} tiles non-causal", lens, 1, 72, 80, False, n)
    _attend(f"{n} tiles causal", lens, 1, 64, 64, True, n + 1)


def test_causal_rows_past_sequence_end():
    """LM-like: 68 tokens leave warpgroup 1 with 4 live rows, 64 and 2 tokens leave it with none, and with max_q 300
    the short sequences' second and third q-tiles are skipped whole."""
    lens = [68, 2, 300, 129, 64, 65, 127, 1, 256]
    _attend("causal past len_q", lens, 36, 64, 64, True, 7)
    _attend("non-causal past len_q", lens, 16, 72, 80, False, 8)
