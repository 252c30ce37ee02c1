"""DETOX on the GPU: the vote's winner_slot table feeding aggregate_update mode 3 (coordinate-wise rules), pair_dist + krum_select
(multi-Krum) and the weight-space geometric median; against the fp64 oracles, bucketing and grid-size determinism, the argument
checks, and whole jobs on the fused engine, including the attack the plain vote average does not survive."""
import ctypes as C

import numpy as np
import pytest
import torch

from draco_b200 import JobConfig
from draco_b200 import _native as N
from draco_b200.codes import oracle
from draco_b200.codes.adversary import generate_schedule
from draco_b200.codes.repetition import group_assign
from draco_b200.models import build_model
from draco_b200.parallel.arena import ArenaLayout
from draco_b200.parallel.ps import hyperparams_tensor
from draco_b200.parallel.trainer import Trainer

pytestmark = pytest.mark.gpu
INF, NAN = float("inf"), float("nan")


@pytest.fixture(scope="module")
def K():
    from draco_b200.ops import kernels
    return kernels


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda", 0)


def lenet_layout():
    return ArenaLayout.from_model(build_model("LeNet"), bf16=False, channels_last=True)


def grouped_slab(L, P, r, dev, seed, captured=(0,), nan_liar=True):
    """[P, D] fp32: every member of a group holds the group's N(0, 1) gradient.  In each ``captured`` group all members but one
    send the same poisoned row (+-Inf / +-1e30 per coordinate), which wins the vote; with ``nan_liar`` one member of the next
    group sends NaN, which never wins (NaN != NaN)."""
    g = torch.Generator().manual_seed(seed)
    groups = group_assign(P, r).groups
    mask = torch.from_numpy(L.valid_mask())
    H = torch.randn(len(groups), L.total, generator=g)
    X = torch.empty(P, L.total)
    for gi, grp in enumerate(groups):
        X[[w - 1 for w in grp]] = H[gi]
    pool = torch.tensor([1e30, -1e30, INF, -INF])
    for gi in captured:
        bad = pool[torch.randint(0, 4, (L.total,), generator=g)]
        for w in groups[gi][:-1]:
            X[w - 1] = bad
    nxt = (max(captured) + 1) if captured else 0
    if nan_liar and nxt < len(groups) and len(groups[nxt]) >= 3:
        X[groups[nxt][1] - 1] = NAN
    X[:, ~mask] = 0
    return X.to(dev).contiguous(), groups


def run_vote(K, L, slots, groups, dev):
    table = -np.ones((len(groups), max(len(g) for g in groups)), dtype=np.int32)
    for gi, grp in enumerate(groups):
        table[gi, :len(grp)] = np.asarray(grp) - 1
    table = torch.from_numpy(table).to(dev)
    G, T = len(groups), L.ntensors
    neq = torch.zeros(G, T, dtype=torch.int32, device=dev)
    win = torch.full((G, T), -1, dtype=torch.int32, device=dev)
    K.vote(L, slots, L.total, table, neq, win)
    torch.cuda.synchronize()
    return win


def winner_rows(L, slots, win):
    """[G, D]: tensor t's range of row g taken from worker slot win[g, t]."""
    W = torch.zeros(win.shape[0], L.total, device=slots.device)
    for t, spec in enumerate(L.specs):
        W[:, spec.offset:spec.offset + spec.numel] = slots[win[:, t].long(), spec.offset:spec.offset + spec.numel]
    return W


def ascending_sum(X, b):
    P = X.shape[0]
    S = X.sort(0).values
    acc = S[b].clone()
    for k in range(b + 1, P - b):
        acc += S[k]
    return acc * (1.0 / (P - 2 * b))


def update_kw(dev, L, lr=0.1):
    hp = hyperparams_tensor(JobConfig(lr=lr, momentum=0.9), dev)
    return dict(params=torch.zeros(L.total, device=dev), momentum=torch.zeros(L.total, device=dev), hp=hp,
                step_ptr=torch.ones(1, dtype=torch.int64, device=dev), done_counter=torch.zeros(4, dtype=torch.int32, device=dev)[0:1])


# ------------------------------------------------------------------------------------------------ mode 3 with the winner table
@pytest.mark.parametrize("P,r", [(9, 3), (15, 3), (12, 4), (16, 2), (32, 2)])
def test_vote_then_trimmed_mean_over_the_winners_matches_oracle(K, dev, P, r):
    L = lenet_layout()
    slots, groups = grouped_slab(L, P, r, dev, seed=P * 7 + r)
    G = len(groups)
    win = run_vote(K, L, slots, groups, dev)
    sl = slots.cpu().double().numpy()
    for t, spec in enumerate(L.specs):
        assert win[:, t].tolist() == oracle.detox_winner_slots(sl[:, spec.offset:spec.offset + spec.numel], groups), t
    assert (win[0] == groups[0][0] - 1).all()                                          # group 0 is captured
    W = winner_rows(L, slots, win)
    for b in sorted({1, (G - 1) // 2}):
        gout = torch.full((L.total,), 7.0, device=dev)
        K.aggregate_update(L, slots, L.total, K=G, scale=1.0 / (G - 2 * b), trim=b, select=win, grad_out=gout, **update_kw(dev, L))
        torch.cuda.synchronize()
        assert torch.equal(gout, ascending_sum(W, b)), (G, b)                              # same fp32 additions, same order
        assert torch.isfinite(gout).all()
        for spec in L.specs:
            ref = oracle.trimmed_mean(W[:, spec.offset:spec.offset + spec.numel].cpu().double().numpy(), b)
            np.testing.assert_allclose(gout[spec.offset:spec.offset + spec.numel].cpu().double().numpy(), ref, rtol=1e-6, atol=1e-6)


def test_detox_trimmed_mean_is_independent_of_buckets_and_grid(K, dev):
    L = ArenaLayout.from_model(build_model("ResNet18"), bf16=True, channels_last=True)
    slots, groups = grouped_slab(L, 9, 3, dev, seed=3)
    G, b = 3, 1
    win = run_vote(K, L, slots, groups, dev)
    nt = L.ntiles
    bounds = [0, nt // 5, nt // 5 + 1, (2 * nt) // 3, nt]
    results = []
    for how in ("one", "buckets", "grid1", "grid37"):
        kw = update_kw(dev, L)
        kw.update(K=G, scale=1.0 / (G - 2 * b), trim=b, select=win)
        if how == "buckets":
            for i in range(len(bounds) - 1):
                K.aggregate_update(L, slots, L.total, tile_range=(bounds[i], bounds[i + 1]), **kw)
        else:
            K.aggregate_update(L, slots, L.total, grid={"one": None, "grid1": 1, "grid37": 37}[how], **kw)
        torch.cuda.synchronize()
        results.append(kw["params"])
    for p in results[1:]:
        assert torch.equal(p, results[0])
    assert torch.isfinite(results[0]).all()


# ------------------------------------------------------------------------------------------------ multi-Krum / geometric median
def test_krum_select_over_the_winners_returns_worker_slots(K, dev):
    L = lenet_layout()
    T = L.ntensors
    slots, groups = grouped_slab(L, 15, 3, dev, seed=11, captured=(), nan_liar=False)
    slots[[0, 1]] = -100 * slots[0]                            # group 0 captured by a sign flip
    win = run_vote(K, L, slots, groups, dev)
    G, b = 5, 1
    m = G - b
    pair = torch.zeros(T, G * (G - 1) // 2, dtype=torch.float64, device=dev)
    sel = torch.full((m, T), -1, dtype=torch.int32, device=dev)
    K.krum_select(L, slots, L.total, G, b, pair, sel, m=m, rows=win)
    torch.cuda.synchronize()
    assert float(pair.abs().sum()) == 0
    sl = slots.cpu().double().numpy()
    for t, spec in enumerate(L.specs):
        ws = oracle.detox_winner_slots(sl[:, spec.offset:spec.offset + spec.numel], groups)
        rows = oracle.multi_krum_indices(sl[ws, spec.offset:spec.offset + spec.numel], b, m)
        assert sel[:, t].tolist() == [ws[i] for i in rows], t                  # worker slots, not winner rows
        assert 0 not in sel[:, t].tolist()
    kw = update_kw(dev, L, lr=1.0)
    gout = torch.zeros(L.total, device=dev)
    K.aggregate_update(L, slots, L.total, K=m, scale=1.0 / m, select=sel, grad_out=gout, **kw)
    torch.cuda.synchronize()
    for spec in L.specs:
        ref = oracle.detox(sl[:, spec.offset:spec.offset + spec.numel], groups, "multi_krum", b)
        np.testing.assert_allclose(gout[spec.offset:spec.offset + spec.numel].cpu().double().numpy(), ref, rtol=1e-5, atol=1e-6)


def test_geometric_median_weights_over_the_winners(K, dev):
    L = lenet_layout()
    T = L.ntensors
    slots, groups = grouped_slab(L, 15, 3, dev, seed=12, captured=(), nan_liar=False)
    slots[[3, 4]] = 30.0 * slots[3]                            # group 1 captured
    win = run_vote(K, L, slots, groups, dev)
    G = 5
    pair = torch.zeros(T, G * (G - 1) // 2, dtype=torch.float64, device=dev)
    w = torch.zeros(T, G, dtype=torch.float32, device=dev)
    K.geometric_median_weights(L, slots, L.total, G, pair, w, rows=win)
    torch.cuda.synchronize()
    assert float(pair.abs().sum()) == 0
    W = winner_rows(L, slots, win).cpu().double().numpy()
    for t, spec in enumerate(L.specs):
        ref = oracle.geometric_median_weights(W[:, spec.offset:spec.offset + spec.numel])
        np.testing.assert_allclose(w[t].cpu().double().numpy(), ref, rtol=1e-4, atol=1e-6)
    gout = torch.zeros(L.total, device=dev)
    K.aggregate_update(L, slots, L.total, K=G, scale=1.0, weights=w, select=win, grad_out=gout, **update_kw(dev, L))
    torch.cuda.synchronize()
    for t, spec in enumerate(L.specs):
        ref = w[t].cpu().double().numpy() @ W[:, spec.offset:spec.offset + spec.numel]
        np.testing.assert_allclose(gout[spec.offset:spec.offset + spec.numel].cpu().double().numpy(), ref, rtol=1e-5, atol=1e-6)


def test_row_tables_are_checked(K, dev):
    L = lenet_layout()
    T = L.ntensors
    slots = torch.zeros(17, L.total, device=dev)
    kw = update_kw(dev, L)
    good = torch.zeros(5, T, dtype=torch.int32, device=dev)
    for table in (torch.zeros(4, T, dtype=torch.int32, device=dev), good.long(), good.cpu(), good.t().contiguous().t()):
        with pytest.raises(ValueError):
            K.aggregate_update(L, slots, L.total, K=5, scale=1.0 / 3, trim=1, select=table, **kw)
    with pytest.raises(ValueError):                            # a table with more than 16 rows
        K.aggregate_update(L, slots, L.total, K=17, scale=1.0 / 15, trim=1,
                           select=torch.zeros(17, T, dtype=torch.int32, device=dev), **kw)
    with pytest.raises(ValueError):
        K.aggregate_update(L, slots, L.total, K=5, scale=1.0, weights=torch.zeros(T, 5, device=dev),
                           select=torch.zeros(4, T, dtype=torch.int32, device=dev), **kw)
    pair = torch.zeros(T, 10, dtype=torch.float64, device=dev)
    with pytest.raises(ValueError):
        K.krum_select(L, slots, L.total, 5, 1, pair, torch.zeros(4, T, dtype=torch.int32, device=dev), m=4,
                      rows=torch.zeros(4, T, dtype=torch.int32, device=dev))
    with pytest.raises(ValueError):
        K.geometric_median_weights(L, slots, L.total, 5, pair, torch.zeros(T, 5, device=dev),
                                   rows=torch.zeros(5, T + 1, dtype=torch.int32, device=dev))
    # the C entry points refuse tables on their own, without launching anything
    a = N.UpdateArgs()
    a.mode, a.K, a.select, a.scale = 2, 17, good.data_ptr(), 1.0
    assert N.cuda().drc_aggregate_update(C.byref(a), 1, K._stream()) == 1
    a.mode, a.K = 1, 5
    assert N.cuda().drc_aggregate_update(C.byref(a), 1, K._stream()) == 1
    a.mode, a.K, a.trim = 3, 17, 1
    assert N.cuda().drc_aggregate_update(C.byref(a), 1, K._stream()) == 1
    pa = N.PairDistArgs(slots.data_ptr(), L.total, 17, L.tile_view(dev), pair.data_ptr(), good.data_ptr())
    assert N.cuda().drc_pair_dist(C.byref(pa), 1, K._stream()) == 1
    ka = N.KrumSelectArgs(pair.data_ptr(), T, 17, 1, 4, good.data_ptr(), good.data_ptr())
    assert N.cuda().drc_krum_select(C.byref(ka), K._stream()) == 1
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------ engine
def _cfg(**kw):
    base = dict(network="LeNet", dataset="MNIST", batch_size=16, max_steps=12, num_workers=9, transport="nvl", lr=0.02,
                momentum=0.9, synthetic_size=512, eval_freq=10 ** 6, compress_grad="None", dtype="fp32", cuda_graphs=False,
                approach="detox", group_size=3, worker_fail=2)
    base.update(kw)
    return JobConfig(**base)


def _run(cfg, steps):
    t = Trainer(cfg, rank=0, world=1, device=torch.device("cuda", 0), quiet=True)
    losses = [t.train_step()["loss"] for _ in range(steps)]
    t.synchronize()
    return t, losses


def _workers(mode):
    return 15 if mode == "multi_krum" else 9                   # multi-Krum needs G > 2 b_G + 2


@pytest.mark.parametrize("mode", ["coordinate_median", "trimmed_mean", "multi_krum", "geometric_median"])
def test_fused_detox_matches_library_op_engine(monkeypatch, mode):
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    kw = dict(mode=mode, num_workers=_workers(mode), err_mode="rev_grad")
    a, _ = _run(_cfg(**kw), 4)
    b, _ = _run(_cfg(transport="nccl", **kw), 4)
    assert a.engine.pipeline_ps == (mode in ("coordinate_median", "trimmed_mean"))
    pa, pb = a.engine.master_params(), b.engine.master_params()
    assert torch.isfinite(pa).all()
    assert torch.allclose(pa, pb, atol=2e-5), float((pa - pb).abs().max())


def test_detox_graph_replay_equals_eager():
    kw = dict(mode="trimmed_mean", num_workers=6, group_size=2, worker_fail=1, err_mode="rev_grad", network="ResNet18",
              dataset="Cifar10", batch_size=8, dtype="bf16", synthetic_size=256)
    e, le = _run(_cfg(cuda_graphs=False, **kw), 6)
    g, lg = _run(_cfg(cuda_graphs=True, **kw), 6)
    assert e.engine.pipeline_ps and g.engine.pipeline_ps and g.engine.graph is not None
    assert torch.equal(e.engine.master_params(), g.engine.master_params())
    assert le == lg


@pytest.mark.parametrize("modes,P,f", [(("coordinate_median", "trimmed_mean", "geometric_median"), 9, 2), (("multi_krum",), 15, 3)])
def test_detox_trains_under_attack_where_the_vote_average_does_not(modes, P, f):
    """Same workers, batches and adversary schedule in every run; only the attack and the rule change.  The schedule captures a
    group in some of the first 10 steps: the vote average then leaves its attack-free trajectory, DETOX stays close to its own."""
    steps = 10
    sched, groups = generate_schedule(P, f, steps), group_assign(P, 3).groups
    captured = [t for t in range(1, steps + 1) if any(len(set(sched.ranks[t].tolist()) & set(g)) >= 2 for g in groups)]
    assert captured, "the schedule never captures a group in the first steps"

    def dist(a, b):
        d = (a - b).abs().max()
        return float(d) if torch.isfinite(d) else float("inf")
    kw = dict(num_workers=P, worker_fail=f, lr=0.05)
    clean, _ = _run(_cfg(approach="maj_vote", mode="maj_vote", err_mode="none", **kw), steps)
    vote, _ = _run(_cfg(approach="maj_vote", mode="maj_vote", err_mode="rev_grad", **kw), steps)
    d_vote = dist(vote.engine.master_params(), clean.engine.master_params())
    assert d_vote > 1e-1, d_vote
    for mode in modes:
        ref, _ = _run(_cfg(mode=mode, err_mode="none", **kw), steps)
        t, losses = _run(_cfg(mode=mode, err_mode="rev_grad", **kw), steps)
        assert losses[-1] < losses[0], (mode, losses)
        p = t.engine.master_params()
        assert torch.isfinite(p).all(), mode
        assert dist(p, ref.engine.master_params()) < 0.1 * d_vote, (mode, dist(p, ref.engine.master_params()), d_vote)
