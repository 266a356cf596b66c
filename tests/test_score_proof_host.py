"""The retrieval proof has power: on the CPU, a numpy emulation of the filter, its candidate lists, the per-query
threshold tau, the head merge, the exact rescoring and the proof (tests/score_fixtures.py) returns the fp32 top-k on
fixtures whose fp16 rounding error comes within a few per cent of eps, and each mutant of a catalogue of plausible
weakenings of the proof returns a wrong top-k on at least one of them."""
import functools

import numpy as np
import pytest

from tests import score_fixtures as SF


@functools.lru_cache(maxsize=None)
def _fixtures():
    return tuple(SF.fixtures())


def _by_name():
    return {f.name: f for f in _fixtures()}


def _wrong(fx, mut):
    s, i, _, info = SF.emulate(fx.Q, fx.D, fx.k, mut=mut)
    ref_s, ref_i = info["ref"]
    return int((i != ref_i).any(1).sum())


@pytest.mark.parametrize("name", SF.FIXTURES)
def test_faithful_emulation_returns_the_fp32_topk(name):
    fx = _by_name()[name]
    s, i, flags, info = SF.emulate(fx.Q, fx.D, fx.k)
    ref_s, ref_i = info["ref"]
    assert np.array_equal(i, ref_i) and np.array_equal(s, ref_s)
    assert (ref_i[:, 0] == fx.true_doc).all()
    in_lists = (info["ci"] == fx.true_doc).any(axis=(1, 2))
    assert (in_lists != fx.dropped).all()                  # the fixture does what it is built for
    assert flags.all()                                     # and the proof notices
    ratio, eps = SF.closeness(fx)
    print(f"\n{name}: true doc's fp16 error = {ratio:.3f} eps (eps {eps:.3e}); "
          f"bound - exact top-1 = {float((info['bound'][0] - ref_s[0, 0]) / info['eps'][0]):+.3f} eps; "
          f"flagged {int(flags.sum())}/{len(flags)}; catches: {fx.note}")


@pytest.mark.parametrize("mut", SF.MUTANTS)
def test_mutant_returns_a_wrong_topk(mut):
    wrong = {f.name: _wrong(f, mut) for f in _fixtures()}
    print(f"\n{mut}: wrong top-1 on {wrong}")
    assert max(wrong.values()) > 0, wrong


def test_fixtures_reach_within_a_third_of_eps():
    """The operand rounding of the two correlated fixtures is 0.78 eps and 0.46 eps (the subnormal one), against about
    0.02 eps for random unit vectors at dim 2304."""
    f = _by_name()
    assert SF.closeness(f["fp16 rounds down 0.49 ulp"])[0] > 0.75
    assert SF.closeness(f["fp16 subnormal query"])[0] > 0.4
    rs = np.random.RandomState(0)
    Q, D = rs.randn(4, 2304).astype(np.float32), rs.randn(2000, 2304).astype(np.float32)
    Q /= np.linalg.norm(Q, axis=1, keepdims=True)
    D /= np.linalg.norm(D, axis=1, keepdims=True)
    err = np.abs(SF.exact_scores(Q, D).astype(np.float64) - SF.approx_scores(Q, D)).max()
    assert err < 0.05 * SF.eps_of(1.0, 1.0, 2304)


def test_plan_replica_waves():
    """At 66 CTA pairs, every filter shape of the older GPU tests runs one wave; 17000 x 20000 runs nine (R = 8)."""
    for nq, nd in ((2600, 9000), (700, 33333), (512, 200000), (300, 20000), (1000, 10000)):
        p = SF.plan(nq, nd)
        assert p["items"] <= p["pairs"], (nq, nd, p)
    p = SF.plan(17000, 20000)
    assert (p["items"], p["R"], -(-p["items"] // p["pairs"])) == (536, 8, 9)


def test_emulated_tau_prunes_later_waves_and_stays_exact():
    """Multi-wave emulation on random data with all-negative, zero and scaled queries: later-wave lists are shorter
    than 16 (tau pruned them), and the proof still yields the fp32 top-k."""
    rs = np.random.RandomState(5)
    nq, nd, dim, pairs = 1000, 4096, 8, 3         # 3 CTA pairs: 4 query blocks x R ranges run in several waves
    D = np.abs(rs.randn(nd, dim)).astype(np.float32)
    Q = rs.randn(nq, dim).astype(np.float32)
    Q[1] = -D.mean(0)
    Q[2] = 0
    Q[3] *= 1e3
    Q[4] *= 1e-3
    p = SF.plan(nq, nd, pairs)
    assert p["items"] > p["pairs"] and p["R"] > 1, p
    s, i, flags, info = SF.emulate(Q, D, 10, pairs=pairs)
    ref_s, ref_i = SF.topk_rows(info["exact"], 10)
    assert np.array_equal(i, ref_i) and np.array_equal(s, ref_s)
    assert (info["cs"][1, :p["R"], 0] < 0).all() and info["cs"][1, -1, 0] < 0    # negative tails, negative tau
    assert (info["ci"][:, :p["R"], SF.KT - 1] < 0).sum() > 0                     # lists that tau cut short
    assert flags[2] == 1                                                          # all scores 0: never certified
