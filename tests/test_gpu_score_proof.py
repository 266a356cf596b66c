"""The retrieval filter and its exactness proof on the H100, where the older tests do not reach them: the persistent
filter in several waves (items > CTA pairs, so items read the per-query threshold tau that earlier items published),
heterogeneous queries in one 256-query block, a stale threshold in reused buffers, dimensions that are not a multiple
of 64, the proof fixtures of tests/score_fixtures.py that bring fp16 rounding within a few per cent of eps, and the
two things the proof assumes of the hardware: the fp16 copies round to nearest even, and wgmma's fp32 accumulation
errs by at most dim 2^-23 sum|q16 d16|."""
import numpy as np
import pytest
import torch

from tests import score_fixtures as SF

pytestmark = pytest.mark.gpu

KT = SF.KT


def _lib():
    from visrag_b200 import _lib as L

    return L, L.lib()


def _plan(nq, nd):
    L, lib = _lib()
    out = np.zeros(6, np.int32)
    L.check(lib.vr_score_plan(nq, nd, out.ctypes.data))
    return dict(zip(("T", "R", "QB", "items", "pairs", "lists"), (int(v) for v in out)))


def _unit(n, d, g, positive=False):
    x = torch.randn(n, d, device="cuda", generator=g)
    return torch.nn.functional.normalize(x.abs() if positive else x, dim=1)


def _filter(q, idx, cand=None):
    """The raw filter into fresh, poisoned buffers (or into `cand`): (cand_s, cand_i) [nq, lists, 16] on the device."""
    from visrag_b200 import retriever as R

    L, lib = _lib()
    nq, d = q.shape
    ranges = lib.vr_score_ranges(nq, idx.nd)
    if cand is None:
        cand = (torch.full((nq, 2 * ranges, KT), float("nan"), device="cuda"),
                torch.full((nq, 2 * ranges, KT), 0x7F7F7F7F, dtype=torch.int32, device="cuda"))
    q16 = R.to_f16_rows(q)
    L.check(lib.vr_score_filter(q16.data_ptr(), nq, idx.emb_f16.data_ptr(), idx.nd, d, ranges, cand[0].data_ptr(),
                                cand[1].data_ptr(), L.stream_ptr()))
    return cand


def _rescore(q, idx, cand, k):
    L, lib = _lib()
    nq, d = q.shape
    s = torch.empty((nq, k), device="cuda")
    i = torch.empty((nq, k), dtype=torch.int64, device="cuda")
    flags = torch.empty(nq, dtype=torch.int32, device="cuda")
    L.check(lib.vr_score_rescore(q.data_ptr(), nq, idx.emb.data_ptr(), idx.nd, d, cand[0].shape[1] // 2, cand[0].data_ptr(),
                                 cand[1].data_ptr(), idx.max_norm.data_ptr(), k, 0, s.data_ptr(), i.data_ptr(),
                                 flags.data_ptr(), L.stream_ptr()))
    return s, i, flags


def _check_lists(q, idx, cand, R, sample=40, seed=0, rows=()):
    """Every slot written, lists sorted, no doc twice, the last slot's first score = tau = the largest tail of a full
    list, and the clear members of the fp16-approximate top-16 of the whole corpus in the lists."""
    from visrag_b200 import retriever as R_

    cs, ci = cand[0].cpu().numpy(), cand[1].cpu().numpy()
    nq, nd = q.shape[0], idx.nd
    assert not np.isnan(cs).any() and ((ci == -1) | ((ci >= 0) & (ci < nd))).all()
    assert (cs[:, :, 1:] <= cs[:, :, :-1]).all()
    assert (np.isinf(cs) == (ci == -1))[:, :-1].all() and (ci[:, -1] == -1).all()
    assert (ci[:, R:-1] == -1).all() and (cs[:, -1, 1:] == -np.inf).all()
    tau, tails = cs[:, -1, 0], cs[:, :R, KT - 1].max(1)
    assert np.array_equal(tau, tails), np.nonzero(tau != tails)[0][:10]
    srt = np.sort(ci.reshape(nq, -1), axis=1)
    assert not ((srt[:, 1:] == srt[:, :-1]) & (srt[:, 1:] >= 0)).any()          # no doc in two lists
    rows = np.concatenate([np.random.RandomState(seed).choice(nq, min(sample, nq), replace=False), rows]).astype(np.int64)
    q16 = R_.to_f16_rows(q)
    approx = (q16[torch.from_numpy(rows).cuda()].double() @ idx.emb_f16.double().T).cpu().numpy()
    for j, r in enumerate(rows):
        kth = np.sort(approx[j])[-KT]
        must = set(np.nonzero(approx[j] > kth + 1e-4 * max(1.0, abs(kth)))[0].tolist())
        assert must <= set(ci[r][ci[r] >= 0].tolist()), r
    return cs, ci


def _check_exact(q, idx, k):
    """score_topk is bit-identical to the fp32 scan (force_exact), and that scan's top-k is the float64 top-k up to
    the fp32 dot product's error dim 2^-24 |q| max|d|."""
    from visrag_b200 import retriever as R

    stats = {}
    s, i = R.score_topk(q, idx, k, stats=stats)
    s2, i2 = R.score_topk(q, idx, k, force_exact=True)
    assert stats["path"] == "filter+rescore", stats
    assert torch.equal(i, i2) and torch.equal(s, s2), int((i != i2).any(1).sum())
    D64 = idx.emb.double()
    tol_row = q.shape[1] * 2.0 ** -24 * q.double().norm(dim=1) * float(idx.max_norm) + 1e-30
    for r0 in range(0, q.shape[0], 2048):
        S = q[r0:r0 + 2048].double() @ D64.T
        tol = tol_row[r0:r0 + 2048, None]
        got = S.gather(1, i[r0:r0 + 2048])
        assert ((got - s[r0:r0 + 2048].double()).abs() <= tol).all()
        best = torch.topk(S, k, dim=1).values
        assert ((best - got.sort(dim=1, descending=True).values).abs() <= 2 * tol).all()
    return s, i, stats


# --------------------------------------------------------------------------------------------------- multi-wave filter


MULTI_WAVE = [(17000, 20000, 64), (18000, 50000, 128), (20000, 100000, 256)]


@pytest.mark.parametrize("nq,nd,d", MULTI_WAVE)
def test_multi_wave_filter_lists_and_exact_topk(nq, nd, d):
    p = _plan(nq, nd)
    assert p["items"] > p["pairs"] and p["R"] > 1, p          # several waves, several doc ranges
    from visrag_b200 import retriever as R

    g = torch.Generator(device="cuda").manual_seed(nq + d)
    q, D = _unit(nq, d, g), _unit(nd, d, g)
    idx = R.build_index(D)
    cand = _filter(q, idx)
    _check_lists(q, idx, cand, p["R"])
    _, _, stats = _check_exact(q, idx, 10)
    print(f"\n{nq}x{nd}x{d}: {p}, waves {-(-p['items'] // p['pairs'])}, flagged {stats['flagged']}")


def test_heterogeneous_queries_in_one_block():
    """One 256-query block holds: all-negative scores (q = -mean of a positive corpus, and -q of a planted query), a
    zero and a -0.0 query (every score +-0: ties by id, and a -0.0 tail published as tau), queries scaled by 1e3 and
    1e-3 (fp16 subnormals), and a query whose top-1 lies in a doc range of a LATER wave than a range holding 20 docs
    just below it (a high tail, so the later item starts from a high tau)."""
    from visrag_b200 import retriever as R

    nq, nd, d = 17000, 40000, 128
    p = _plan(nq, nd)
    assert p["items"] > p["pairs"] and p["R"] > 1, p
    g = torch.Generator(device="cuda").manual_seed(7)
    D = _unit(nd, d, g, positive=True)
    q = _unit(nq, d, g)
    b = 1                                                  # the block under test: rows 256..511
    r0 = 256 * b
    u = _unit(1, d, g, positive=True)[0]
    early, late = SF.range_docs(p, nd, 0), SF.range_docs(p, nd, p["R"] - 1)
    assert SF.wave(p, p["R"] - 1, b) > SF.wave(p, 0, b), p
    D[early[0]:early[0] + 20] = torch.nn.functional.normalize(u + 0.3 * _unit(20, d, g, positive=True), dim=1)
    D[late[0] + 7] = torch.nn.functional.normalize(u + 0.05 * _unit(1, d, g, positive=True)[0], dim=0)
    q[r0 + 0] = -D.mean(0) / D.mean(0).norm()
    q[r0 + 1] = 0.0
    q[r0 + 2] = -0.0
    q[r0 + 3] *= 1e3
    q[r0 + 4] *= 1e-3
    q[r0 + 5] = u
    q[r0 + 6] = -u
    q[r0 + 7] = -D.mean(0) / D.mean(0).norm() * 1e-3
    idx = R.build_index(D)
    cs, ci = _check_lists(q, idx, _filter(q, idx), p["R"], rows=np.arange(r0, r0 + 8))
    s, i, stats = _check_exact(q, idx, 10)
    S = (q[r0:r0 + 8].double() @ D.double().T).cpu().numpy()
    assert (S[[0, 6, 7]] < 0).all() and (cs[[r0, r0 + 6, r0 + 7], :p["R"], 0] < 0).all()
    assert (cs[[r0, r0 + 6, r0 + 7], -1, 0] < 0).all()                        # negative tau
    assert int(i[r0 + 5, 0]) == late[0] + 7
    assert torch.equal(i[r0 + 1].cpu(), torch.arange(10)) and torch.equal(i[r0 + 2].cpu(), torch.arange(10))
    zero_tails = cs[[r0 + 1, r0 + 2], :p["R"], KT - 1]
    print(f"\nflagged {stats['flagged']}; zero-query tails negative-zero: {np.signbit(zero_tails).sum(1).tolist()} of "
          f"{p['R']}; late list of the planted query: {int((ci[r0 + 5, p['R'] - 1] >= 0).sum())} entries")


def test_stale_threshold_is_reset():
    """The filter run twice on the same buffers, first with the queries scaled by 4 (a threshold no unscaled score
    reaches), gives the lists of a run on fresh buffers: score_init_lists_kernel resets tau. Entries above the final
    tau, and tau itself, do not depend on how the waves interleave."""
    from visrag_b200 import retriever as R

    nq, nd, d = 17000, 20000, 64
    p = _plan(nq, nd)
    assert p["items"] > p["pairs"], p
    g = torch.Generator(device="cuda").manual_seed(9)
    q, D = _unit(nq, d, g), _unit(nd, d, g)
    idx = R.build_index(D)
    reused = _filter(q * 4, idx)
    hi_tau = reused[0][:, -1, 0].clone()
    _filter(q, idx, reused)
    fresh = _filter(q, idx)
    assert (hi_tau > reused[0][:, -1, 0]).all()

    def above_tau(c):
        cs, ci = c[0].cpu().numpy(), c[1].cpu().numpy()
        tau = cs[:, -1:, :1]
        return cs[:, -1, 0], np.sort(np.where(cs > tau, ci, -1), axis=2)

    (ta, la), (tb, lb) = above_tau(reused), above_tau(fresh)
    assert np.array_equal(ta, tb) and np.array_equal(la, lb)
    _check_lists(q, idx, reused, p["R"])
    a, b = _rescore(q, idx, reused, 10), _rescore(q, idx, fresh, 10)
    ok = (a[2] == 0) & (b[2] == 0)
    assert torch.equal(a[1][ok], b[1][ok])


# ------------------------------------------------------------------------------------------- dims not a multiple of 64


@pytest.mark.parametrize("nq,nd,d", [(2000, 3000, 8), (1500, 3000, 72), (1100, 4000, 200), (600, 8000, 1000)])
def test_filter_dims_not_a_multiple_of_64(nq, nd, d):
    """The last k block of the TMA loads is zero-filled past d."""
    from visrag_b200 import retriever as R

    assert nq * nd > 1 << 22 and nd >= 256
    g = torch.Generator(device="cuda").manual_seed(d)
    q, D = _unit(nq, d, g), _unit(nd, d, g)
    idx = R.build_index(D)
    _check_lists(q, idx, _filter(q, idx), _plan(nq, nd)["R"])
    _check_exact(q, idx, 10)


# ----------------------------------------------------------------------------------------------------- proof fixtures


@pytest.mark.parametrize("name", SF.FIXTURES)
def test_proof_fixture(name):
    """Every query of a fixture must be flagged and answered by the fp32 scan; where the filter's lists miss the true
    top-1 (the decoy fixtures) that is the proof's doing. The toward-zero fixture keeps its true document in the lists
    only because the fp16 copies round to nearest."""
    from visrag_b200 import retriever as R

    fx = next(f for f in SF.fixtures() if f.name == name)
    nq = fx.Q.shape[0]
    p = _plan(nq, fx.D.shape[0])
    assert p["R"] == 16, p                                 # the doc ranges the fixture's layout assumes
    q = torch.from_numpy(fx.Q).cuda()
    idx = R.build_index(fx.D)
    s, i, stats = _check_exact(q, idx, fx.k)
    assert (i[:, 0] == fx.true_doc).all()
    cand = _filter(q, idx)
    cs, ci = _check_lists(q, idx, cand, p["R"], sample=4)
    _, _, flags = _rescore(q, idx, cand, fx.k)
    flags = flags.cpu().numpy()
    missing = ~(ci == fx.true_doc).any(axis=(1, 2))
    assert flags[missing].all()
    assert missing.all() == fx.dropped and missing.any() == fx.dropped
    assert flags.all() and stats["flagged"] == nq
    ratio, eps = SF.closeness(fx)
    print(f"\n{name}: fp16 error of the true doc {ratio:.3f} eps; lists miss it for {int(missing.sum())}/{nq} "
          f"queries; flagged {int(flags.sum())}/{nq}")


# ------------------------------------------------------------------------------------ what the bound assumes, measured


def test_f16_rows_round_like_torch_and_norms_within_bound():
    """vr_f32_to_f16_rows: bit-identical to torch's .half() (ties to even, subnormals and their ties, the largest
    finite value, >= 65520 -> inf, -0.0); row norms within (dim/2 + 1) 2^-24 of float64 (fp32 squares and sums, one
    sqrt), max_norm the largest of them."""
    from visrag_b200 import _lib as L

    lib = L.lib()
    specials = [1 + 2 ** -11, 1 + 3 * 2 ** -11, 1 + 2 ** -11 + 2 ** -20, -(1 + 2 ** -11), 2 ** -25, 3 * 2 ** -25,
                5 * 2 ** -25, 2 ** -25 + 2 ** -40, 2 ** -14 - 2 ** -25, 2 ** -14 - 2 ** -26, 1e-30, -1e-30, 0.0, -0.0,
                65504.0, 65519.0, 65519.99, 65520.0, -65520.0, 1e6, -1e6, 2 ** -24, -(2 ** -24)]
    g = torch.Generator(device="cuda").manual_seed(17)
    for dim in (72, 1000, 2304):
        rows = 1500
        x = torch.randn(rows, dim, device="cuda", generator=g) * 2.0 ** torch.randint(-30, 17, (rows, dim), device="cuda",
                                                                                    generator=g)
        sp = torch.tensor(specials, device="cuda")
        pos = torch.randperm(rows * dim, device="cuda", generator=g)[: 40 * len(specials)]
        x.view(-1)[pos] = sp.repeat(40)
        x[3] = -0.0
        out = torch.empty(rows, dim, dtype=torch.float16, device="cuda")
        norms = torch.empty(rows, device="cuda")
        mx = torch.zeros(1, device="cuda")
        L.check(lib.vr_f32_to_f16_rows(x.data_ptr(), rows, dim, out.data_ptr(), norms.data_ptr(), mx.data_ptr(),
                                       L.stream_ptr()))
        assert torch.equal(out.view(torch.int16), x.half().view(torch.int16)), dim
        n64 = x.double().norm(dim=1)
        fin = torch.isfinite(n64) & torch.isfinite(norms)
        assert ((norms.double() - n64).abs()[fin] <= (dim / 2 + 1) * 2.0 ** -24 * n64[fin]).all()
        assert torch.equal(torch.isinf(norms), torch.isinf(n64.float()))
        assert float(mx) == float(norms.max()) and (mx >= norms).all()


def _stress(n, dim, g, cancel):
    """fp16-exact rows with a wide dynamic range within a k block (element exponents +-4 around a block exponent) and
    across k blocks (block exponents -8..8). Rows with `cancel` repeat (queries) or negate (docs) the first half of
    k block 0, scaled by 2^8: the block's products cancel exactly, after the accumulator has held their large sum."""
    kb = (dim + 63) // 64
    e = torch.randint(-8, 9, (n, kb), device="cuda", generator=g).repeat_interleave(64, 1)[:, :dim]
    e = e + torch.randint(-4, 5, (n, dim), device="cuda", generator=g)
    x = torch.randn(n, dim, device="cuda", generator=g) * 2.0 ** e.float()
    if cancel:
        x[:, :32] = torch.randn(n, 32, device="cuda", generator=g) * 256
        x[:, 32:64] = x[:, :32] * cancel
    return x.clamp(-60000, 60000).half().float()


@pytest.mark.parametrize("dim", [256, 2304])
def test_wgmma_accumulation_error_within_the_assumed_bound(dim):
    """The filter's approximate scores, read from its lists, against float64 dot products of the same fp16 operands:
    |err| <= dim 2^-23 sum|q16 d16| (the accumulation term of eps). Prints the largest ratio seen."""
    from visrag_b200 import retriever as R

    g = torch.Generator(device="cuda").manual_seed(dim)
    nq, nd = 1024, 4096
    q = torch.cat([_stress(nq // 2, dim, g, 0), _stress(nq // 2, dim, g, 1)])
    D = torch.cat([_stress(nd // 2, dim, g, 0), _stress(nd // 2, dim, g, -1)])
    idx = R.build_index(D)
    cs, ci = _filter(q, idx)
    ok = ci >= 0
    qi = torch.arange(nq, device="cuda")[:, None, None].expand_as(ci)[ok]
    di = ci[ok].long()
    got = cs[ok].double()
    q64, d64 = q.double(), D.double()
    exact = torch.empty_like(got)
    mag = torch.empty_like(got)
    step = (1 << 24) // dim
    for a in range(0, len(got), step):
        prod = q64[qi[a:a + step]] * d64[di[a:a + step]]
        exact[a:a + step] = prod.sum(1)
        mag[a:a + step] = prod.abs().sum(1)
    err = (got - exact).abs()
    ratio = err / (dim * 2.0 ** -23 * mag + 1e-300)
    worst = int(ratio.argmax())
    print(f"\ndim {dim}: {len(got)} scores; max |err| / (dim 2^-23 sum|q16 d16|) = {float(ratio.max()):.3e}; "
          f"max |err| / (2^-24 sum|q16 d16|) = {float((err / (2.0 ** -24 * mag)).max()):.3f}; "
          f"worst pair: err {float(err[worst]):.3e}, score {float(exact[worst]):.3e}, sum|q d| {float(mag[worst]):.3e}")
    assert (ratio <= 1).all()
