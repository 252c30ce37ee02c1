"""Coding-theory layer + oracles (CPU, fp64)."""
import itertools

import numpy as np
import pytest
import torch

from draco_b200.codes import adversary, cyclic, oracle
from draco_b200.codes.repetition import group_assign


@pytest.mark.parametrize("n,s", [(3, 1), (5, 1), (5, 2), (7, 1), (7, 2), (7, 3), (8, 2), (9, 4)])
def test_search_w_invariants(n, s):
    c = cyclic.search_w(n, s)
    assert c.W.shape == (n, n) and c.W_perp.shape == (2 * s, n) and c.C1.shape == (n, n - 2 * s)
    # support: worker i touches exactly batches i..i+2s (mod n)
    assert np.all((np.abs(c.W) > 1e-12) <= (c.support > 0))
    assert np.all(c.support.sum(1) == 2 * s + 1) and np.all(c.support.sum(0) == 2 * s + 1)
    assert np.abs(c.W_perp @ c.W).max() < 1e-9          # honest codewords have zero syndrome
    assert np.abs(c.S @ c.W - 1.0).max() < 1e-9          # S W = 1^T
    assert np.allclose(c.S, np.ones((1, n)) / np.sqrt(n))


@pytest.mark.parametrize("n,s", [(5, 1), (7, 2), (7, 3), (8, 2)])
def test_cyclic_decode_recovers_sum_for_every_adversary_subset(n, s):
    rng = np.random.RandomState(0)
    c = cyclic.search_w(n, s)
    G = rng.randn(n, 40)
    f = rng.randn(40) + 1.0
    R0 = np.stack([cyclic.encode(c, i, G) for i in range(n)])
    for k in range(0, s + 1):
        for liars in itertools.combinations(range(n), k):
            R = R0.copy()
            for l in liars:
                R[l] += rng.choice([-100.0, 37.0]) * (1 + rng.rand(40)) * (1 if rng.rand() < 0.5 else 1j)
            dec, healthy = cyclic.decode(c, R, f)
            assert not set(healthy) & set(liars)
            assert np.abs(dec - G.sum(0)).max() < 1e-6 * max(1.0, np.abs(G.sum(0)).max())


@pytest.mark.parametrize("n,s,liars", [(7, 2, (1, 4)), (7, 3, (0, 2, 6)), (7, 2, ()), (5, 1, (3,)), (9, 2, (8,)), (7, 2, (5,))])
def test_ifft_decoder_agrees_and_exposes_the_error(n, s, liars):
    """The alternative 'estimate eps and subtract' decoder (reference's dead `_obtain_E` path / orphan decoding.o)."""
    rng = np.random.RandomState(5)
    c = cyclic.search_w(n, s)
    G = rng.randn(n, 24)
    f = rng.randn(24) + 1.0
    R = np.stack([cyclic.encode(c, i, G) for i in range(n)])
    for l in liars:
        R[l] += -100.0 * (1 + rng.rand(24))
    d1, _ = cyclic.decode(c, R, f)
    d2 = cyclic.decode_ifft(c, R, f)
    assert np.abs(d1 - G.sum(0)).max() < 1e-8 and np.abs(d2 - G.sum(0)).max() < 1e-8


def test_cyclic_decode_fails_beyond_tolerance():
    rng = np.random.RandomState(1)
    c = cyclic.search_w(7, 1)
    G = rng.randn(7, 30)
    R = np.stack([cyclic.encode(c, i, G) for i in range(7)])
    R[0] += 100.0
    R[3] -= 55.0          # two liars, s = 1
    dec, _ = cyclic.decode(c, R, rng.randn(30) + 1.0)
    assert np.abs(dec - G.sum(0)).max() > 1e-3


def test_group_assign_matches_reference_layout():
    plan = group_assign(7, 3)
    assert plan.groups == [[1, 2, 3], [4, 5, 6, 7]]      # remainder joins the last group (src/util.py:69-75)
    assert plan.group_of(0) == -1 and plan.group_of(5) == 1 and plan.member_index(6) == 2
    # seeds: RandomState(428).randint(0, 20000) per group, identical on every rank
    rs = np.random.RandomState(428)
    assert plan.seeds == [int(rs.randint(0, 20000)) for _ in plan.groups]
    assert group_assign(8, 4).groups == [[1, 2, 3, 4], [5, 6, 7, 8]]
    tab = plan.as_table()
    assert tab.shape == (2, 4) and tab[0].tolist() == [0, 1, 2, -1] and tab[1].tolist() == [3, 4, 5, 6]
    assert plan.tolerance(0) == 1 and plan.tolerance(1) == 1


def test_adversary_schedule_is_the_reference_stream():
    s = adversary.generate_schedule(7, 2, 20)
    np.random.seed(428)                                   # reference: src/util.py:100-103
    ref = [np.random.choice(np.arange(1, 8), size=2, replace=False) for _ in range(21)]
    for a, b in zip(s.ranks, ref):
        assert sorted(a.tolist()) == sorted(b.tolist())
    bm = s.bitmaps()
    for t in range(21):
        for w in range(1, 8):
            assert bool((bm[t] >> (w - 1)) & 1) == s.is_adversary(w, t)


def test_err_simulation_modes():
    g = np.arange(6, dtype=np.float64) - 2
    assert np.array_equal(adversary.err_simulation(g, "rev_grad"), -100 * g)
    assert np.array_equal(adversary.err_simulation(g, "rev_grad", cyclic=True), g - 100 * g)
    assert np.array_equal(adversary.err_simulation(g, "constant"), np.full(6, -100.0))
    assert np.array_equal(adversary.err_simulation(g, "constant", cyclic=True), g - 100)
    r1 = adversary.err_simulation(g, "random", step=3, worker=2)
    r2 = adversary.err_simulation(g, "random", step=3, worker=2)
    assert np.array_equal(r1, r2) and not np.array_equal(r1, g) and np.abs(r1).max() > 1
    om = adversary.err_simulation(g, "omniscient", honest_mean=np.ones(6))
    assert np.array_equal(om, -100 * np.ones(6))


def test_majority_vote_semantics():
    rng = np.random.RandomState(0)
    good = rng.randn(10)
    bad = -100 * good
    groups = [[1, 2, 3], [4, 5, 6, 7]]
    slots = np.stack([good, bad, good, good + 1, good + 1, bad, good + 1])
    agg, winners = oracle.majority_vote(slots, groups)
    assert winners == [2, 0]          # streaming Boyer-Moore: [good, bad, good] re-elects member 2 (same tensor as member 0)
    assert np.allclose(agg, (good + good + 1) / 2)
    # no strict majority: Boyer-Moore keeps the last surviving candidate (reference behaviour)
    slots2 = np.stack([good, bad, good * 2])
    assert oracle.boyer_moore_winner(list(slots2)) == 2
    # NaN never equals itself (np.array_equal semantics)
    n = good.copy(); n[0] = np.nan
    assert oracle.boyer_moore_winner([n, n, good]) == 2


def test_krum_and_geomedian_oracles_vs_host_library():
    from draco_b200 import _native as N
    rng = np.random.RandomState(2)
    X = rng.randn(7, 200).astype(np.float32)
    X[2] = -100 * X[2]
    X[5] = 50.0
    k = oracle.krum_index(X, 2)
    assert k not in (2, 5)
    kh = N.host().drc_host_krum(X.ctypes.data, 7, 200, 200, 2)
    assert kh == k
    gm = oracle.geometric_median(X.astype(np.float64), eps=1e-10, max_iter=500)
    out = np.zeros(200, dtype=np.float32)
    N.host().drc_host_geomedian(X.ctypes.data, 7, 200, 200, 1e-10, 500, out.ctypes.data)
    assert np.abs(out - gm).max() < 1e-3
    honest = np.delete(X, [2, 5], axis=0)
    assert np.linalg.norm(gm - honest.mean(0)) < np.linalg.norm(X.mean(0) - honest.mean(0))
    rows = np.array([0, 1, 3], dtype=np.int32)
    Y = np.stack([X[0], X[0], X[1]]).copy()
    assert N.host().drc_host_vote(Y.ctypes.data, 200, 200, np.array([0, 1, 2], dtype=np.int32).ctypes.data, 3) == 0


@pytest.mark.parametrize("nesterov,wd,damp", [(False, 0.0, 0.0), (True, 1e-3, 0.0), (False, 5e-4, 0.1)])
def test_sgd_modified_matches_torch_sgd(nesterov, wd, damp):
    from draco_b200.optim import SGDModified
    torch.manual_seed(0)
    p_ref = [torch.randn(5, 3, requires_grad=True), torch.randn(7, requires_grad=True)]
    p_new = [p.detach().clone() for p in p_ref]
    ref = torch.optim.SGD(p_ref, lr=0.05, momentum=0.9, nesterov=nesterov, weight_decay=wd, dampening=damp)
    new = SGDModified(p_new, lr=0.05, momentum=0.9, nesterov=nesterov, weight_decay=wd, dampening=damp)
    for _ in range(4):
        grads = [torch.randn_like(p) for p in p_ref]
        for p, g in zip(p_ref, grads):
            p.grad = g.clone()
        ref.step()
        new.step(grads=[g.numpy() for g in grads], mode="normal")
    for a, b in zip(p_ref, p_new):
        assert torch.allclose(a.detach(), b, atol=1e-6)
    # oracle helper agrees too
    p, buf = np.ones(4), np.zeros(4)
    p1, buf1 = oracle.sgd_momentum_step(p, buf, np.full(4, 2.0), lr=0.1, momentum=0.9, first_step=True)
    assert np.allclose(p1, 1 - 0.2) and np.allclose(buf1, 2.0)


def test_adam_modified_matches_torch_adam():
    from draco_b200.optim import AdamModified
    torch.manual_seed(0)
    p_ref = [torch.randn(4, 4, requires_grad=True)]
    p_new = [p_ref[0].detach().clone()]
    ref = torch.optim.Adam(p_ref, lr=1e-2)
    new = AdamModified(p_new, lr=1e-2)
    for _ in range(5):
        g = torch.randn(4, 4)
        p_ref[0].grad = g.clone()
        ref.step()
        new.step(grads=[g], mode="normal")
    assert torch.allclose(p_ref[0].detach(), p_new[0], atol=1e-6)


def test_geometric_median_in_weight_space_matches_weiszfeld():
    """Host model of the one-pass device algorithm: Weiszfeld on convex weights from pairwise distances."""
    rng = np.random.RandomState(5)
    for n in (3, 40, 1500):
        h = rng.randn(n) * 0.1
        X = h[None] + 0.02 * rng.randn(7, n)
        X[0] *= -100
        X[3] = -100
        w = oracle.geometric_median_weights(X)
        assert abs(w.sum() - 1) < 1e-12 and w.min() >= 0
        ref = oracle.geometric_median(X, eps=1e-12, max_iter=5000)
        assert np.abs(w @ X - ref).max() < 1e-8
    same = np.tile(rng.randn(1, 10), (5, 1))
    assert np.allclose(oracle.geometric_median_weights(same), 0.2)
    # the median sits on one of the inputs (3 identical points out of 5): the weights collapse onto them without NaN
    X = rng.randn(5, 20)
    X[1] = X[2] = X[0]
    w = oracle.geometric_median_weights(X)
    assert np.isfinite(w).all() and np.abs(w @ X - X[0]).max() < 1e-6

