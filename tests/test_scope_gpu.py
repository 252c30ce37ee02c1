"""Whole-model scope on the GPU: the pair-table scope fold (csrc/cuda/robust.cu), centered clipping's model weights
(csrc/cuda/clip.cu) and min-max's model solve (csrc/cuda/attack.cu) against the oracle and an exact restatement, grid and
bucket invariance, the argument checks, and whole jobs: fused against the library-op engine, graph replay against eager, the
flag's effect, and training under attack."""
import ctypes as C

import numpy as np
import pytest
import torch

from draco_b200 import JobConfig
from draco_b200 import _native as N
from draco_b200.codes import adversary as A
from draco_b200.codes import oracle
from draco_b200.models import build_model
from draco_b200.parallel.arena import ArenaLayout
from draco_b200.parallel.trainer import Trainer

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def K():
    from draco_b200.ops import kernels
    return kernels


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda", 0)


def lenet_layout():
    return ArenaLayout.from_model(build_model("LeNet"), bf16=False, channels_last=True)


def resnet_layout():
    return ArenaLayout.from_model(build_model("ResNet18"), bf16=True, channels_last=True)


def int_slots(L, rows, dev, seed, lo=-3, hi=4):
    """Small-integer fp32 rows (padding 0): every fp64 sum the kernels form is exact, whatever the order of their atomics."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randint(lo, hi, (rows, L.total), generator=g).float()
    x[:, ~torch.from_numpy(L.valid_mask())] = 0
    return x.contiguous().to(dev)


def tensor_d2(L, X):
    """Per-tensor [T, P, P] fp64 distance tables of the rows ``X`` (numpy)."""
    return [oracle._raw_d2(X[:, s.offset: s.offset + s.numel]) for s in L.specs]


def pair_vec(D):
    P = D.shape[0]
    return np.array([D[i, j] for j in range(1, P) for i in range(j)])


def model_table(K, L, X, P, dev, rows=None):
    pair = torch.zeros(L.ntensors, P * (P - 1) // 2, dtype=torch.float64, device=dev)
    K.pair_dist(L, X, L.total, P, pair, rows=rows)
    K.pair_scope_fold(L, P, pair)
    return pair


# ------------------------------------------------------------------------------------------------ kernels
def test_scope_fold_is_the_in_order_sum_written_to_every_tensor(K, dev):
    L = resnet_layout()
    for P in (2, 7, 15, 16):
        g = torch.Generator().manual_seed(P)
        t = (torch.randn(L.ntensors, P * (P - 1) // 2, generator=g, dtype=torch.float64) *
             10.0 ** torch.randint(-6, 6, (L.ntensors, 1), generator=g)).abs()
        t[3, 0] = float("nan") if P == 7 else t[3, 0]
        want = oracle.model_d2(t.numpy())
        d = t.to(dev)
        K.pair_scope_fold(L, P, d)
        got = d.cpu().numpy()
        assert np.array_equal(got, np.broadcast_to(want, got.shape), equal_nan=True), P


@pytest.mark.parametrize("P,f", [(7, 1), (15, 3), (16, 3)])
def test_selection_tables_are_the_model_oracle_in_every_tensor(K, dev, P, f):
    L = resnet_layout()
    X = int_slots(L, P, dev, seed=P)
    X[0] *= 3                                              # a far worker, and a tie-free model table
    D = oracle.model_d2(tensor_d2(L, X.cpu().numpy()))
    pair = model_table(K, L, X, P, dev)
    assert np.array_equal(pair.cpu().numpy(), np.broadcast_to(pair_vec(D), pair.shape))
    T = L.ntensors
    m = P - f
    sel = torch.zeros(m, T, dtype=torch.int32, device=dev)
    K.krum_select(L, X, L.total, P, f, pair, sel, m=m, filled=True)
    want = np.argsort(oracle._krum_scores_d2(D, f), kind="stable")[:m]
    assert (sel.cpu().numpy() == want[:, None]).all() and float(pair.abs().sum()) == 0.0
    if P >= 4 * f + 3:
        pair = model_table(K, L, X, P, dev)
        bsel = torch.zeros(P - 2 * f, T, dtype=torch.int32, device=dev)
        K.bulyan_select(L, X, L.total, P, f, pair, bsel, filled=True)
        assert (bsel.cpu().numpy() == np.array(oracle._bulyan_rounds(D, f))[:, None]).all()
    pair = model_table(K, L, X, P, dev)
    w = torch.zeros(T, P, dtype=torch.float32, device=dev)
    K.geometric_median_weights(L, X, L.total, P, pair, w, filled=True)
    ww = w.cpu().numpy()
    assert (ww == ww[:1]).all()
    assert np.allclose(ww[0], oracle._weiszfeld_weights(D, 1e-10, 256), rtol=0, atol=1e-6)
    pair = model_table(K, L, X, P, dev)
    mix = torch.zeros(P, T, dtype=torch.int32, device=dev)
    K.nnm_mix_table(L, P, f, pair, mix, mixed_out=True)
    Am = oracle.nnm_neighbours_d2(D, f)
    masks = np.array([sum(1 << j for j in np.flatnonzero(a)) for a in Am])
    assert (mix.cpu().numpy().astype(np.int64) == masks[:, None]).all()
    got = pair.cpu().numpy()
    want_mixed = pair_vec(oracle.nnm_pair_d2(D, Am, f))
    assert (got == got[:1]).all() and np.allclose(got[0], want_mixed, rtol=1e-12, atol=0)


def test_detox_rows_use_the_vote_winners_table(K, dev):
    L = lenet_layout()
    P, G = 9, 5
    X = int_slots(L, P, dev, seed=3)
    g = torch.Generator().manual_seed(4)
    rows = torch.stack([torch.randperm(P, generator=g)[:G] for _ in range(L.ntensors)], 1).to(torch.int32).contiguous().to(dev)
    Xn, rn = X.cpu().numpy(), rows.cpu().numpy()
    D = oracle.model_d2([oracle._raw_d2(Xn[rn[:, t], s.offset: s.offset + s.numel]) for t, s in enumerate(L.specs)])
    pair = model_table(K, L, X, G, dev, rows=rows)
    assert np.array_equal(pair.cpu().numpy()[0], pair_vec(D))
    sel = torch.zeros(3, L.ntensors, dtype=torch.int32, device=dev)
    K.krum_select(L, X, L.total, G, 1, pair, sel, m=3, rows=rows, filled=True)
    best = np.argsort(oracle._krum_scores_d2(D, 1), kind="stable")[:3]
    assert (sel.cpu().numpy() == rn[best]).all()           # worker slots, a different one per tensor, of the same rows


def _cc_model(K, L, X, v, n, tau, dev, grid=None, buckets=None):
    partials = torch.zeros(L.ntiles, n, dtype=torch.float64, device=dev)
    dist = torch.zeros(L.ntensors, n, dtype=torch.float64, device=dev)
    w = torch.zeros(L.ntensors, n, dtype=torch.float32, device=dev)
    for tr in buckets or [None]:
        K.centered_clip_dist(L, X, L.total, n, v, partials, tile_range=tr, grid=grid)
    K.centered_clip_model_weights(L, n, tau, partials, dist, w)
    return w, dist


@pytest.mark.parametrize("n", [1, 5, 15, 16])
def test_cc_model_weights_are_the_exact_composition(K, dev, n):
    L = resnet_layout()
    X = int_slots(L, n, dev, seed=n)
    v = int_slots(L, 1, dev, seed=100 + n, lo=-1, hi=2)[0].contiguous()
    if n > 2:
        X[2, L.specs[5].offset + 1] = float("nan")
    Xn, vn = X.cpu().numpy().astype(np.float64), v.cpu().numpy().astype(np.float64)
    with np.errstate(invalid="ignore"):
        per = [((Xn[:, s.offset: s.offset + s.numel] - vn[s.offset: s.offset + s.numel]) ** 2).sum(1) for s in L.specs]
    d = oracle.model_d2(per)
    for tau in (0.5, 50.0, 1e6):
        w, dist = _cc_model(K, L, X, v, n, tau, dev)
        want = np.array([oracle.centered_clip_weight(float(x), tau, n) for x in d], dtype=np.float32)
        assert np.array_equal(w.cpu().numpy(), np.broadcast_to(want, w.shape)), tau
        assert np.array_equal(dist.cpu().numpy(), np.array(per), equal_nan=True)
    if n > 2:
        assert (w[:, 2] == 0).all()                          # NaN in one tensor: weight 0 in every tensor


def test_cc_model_weights_do_not_depend_on_grid_or_buckets(K, dev):
    L = resnet_layout()
    g = torch.Generator().manual_seed(9)
    X = (torch.randn(15, L.total, generator=g) * torch.rand(15, 1, generator=g)).to(dev)
    v = (torch.randn(L.total, generator=g) * 0.1).to(dev)
    ref, _ = _cc_model(K, L, X, v, 15, 3.0, dev)
    t = L.ntiles
    for grid, buckets in ((1, None), (7, None), (None, [(0, t // 3), (t // 3, t)]), (3, [(0, 1), (1, t - 5), (t - 5, t)])):
        w, _ = _cc_model(K, L, X, v, 15, 3.0, dev, grid=grid, buckets=buckets)
        assert torch.equal(w, ref), (grid, buckets)


def _minmax(K, L, X, P, liars, dev, grid=None, model=True):
    slab = X.clone()
    ws = K.AttackWorkspace(L, P, dev)
    fold = K.attack_fold_buffer(L, P, dev)
    bitmap = torch.tensor([sum(1 << w for w in liars)], dtype=torch.int32, device=dev)
    step = torch.zeros(1, dtype=torch.int64, device=dev)
    if model:
        n = K.ps_attack_model(L, slab, L.total, P, adv_bitmap=bitmap, adv_len=1, step_ptr=step, ws=ws, fold=fold, grid=grid)
        assert n == 4
    else:
        K.ps_attack(L, slab, L.total, P, 6, adv_bitmap=bitmap, adv_len=1, step_ptr=step, ws=ws, grid=grid)
    return slab, ws, fold


@pytest.mark.parametrize("P,liars", [(7, [1]), (15, [0, 4, 9]), (16, [15])])
def test_minmax_model_gamma_is_the_exact_composition(K, dev, P, liars):
    L = resnet_layout()
    g = torch.Generator().manual_seed(P)
    X = (torch.randn(P, L.total, generator=g) * torch.rand(P, 1, generator=g)).to(dev)
    X[:, ~torch.from_numpy(L.valid_mask()).to(dev)] = 0
    slab, ws, fold = _minmax(K, L, X, P, liars, dev)
    gamma = ws.gamma.cpu().numpy()
    assert (gamma == gamma[0]).all() and gamma[0] > 0
    # restated from the device's own per-tile partials: per tensor in tile order, over the tensors in order, the closed form
    Q = 2 * P + 1 + P * (P - 1) // 2
    parts = ws.partials.cpu().numpy()
    per = []
    for s in L.specs:
        t0 = s.offset // 1024
        acc = np.zeros(Q)
        for t in range(t0, t0 + (s.numel + 1023) // 1024):
            acc = acc + parts[t]
        per.append(acc)
    assert np.array_equal(fold.cpu().numpy(), np.array(per))
    honest = [i for i in range(P) if i not in liars]
    keep = honest + [P + i for i in honest] + [2 * P] + [2 * P + 1 + j * (j - 1) // 2 + i for j in range(1, P) for i in range(j)
                                                          if i in honest and j in honest]
    want = A.minmax_solve(oracle.model_d2(per)[keep])
    assert gamma[0] == pytest.approx(want, rel=1e-13)
    Xn = X.cpu().numpy()
    spans = [(s.offset, s.numel) for s in L.specs]
    oracle_gamma = A.minmax_gamma_model([Xn[honest, o:o + n].astype(np.float64) for o, n in spans])
    assert gamma[0] == pytest.approx(oracle_gamma, rel=1e-9)
    want_slab = A.ps_attack(Xn, liars, "minmax", spans, scope="model")
    assert np.allclose(slab.cpu().numpy(), want_slab, rtol=1e-6, atol=1e-7)
    for grid in (1, 5):
        assert torch.equal(_minmax(K, L, X, P, liars, dev, grid=grid)[0], slab)
    per_tensor, ws_t, _ = _minmax(K, L, X, P, liars, dev, model=False)
    assert not torch.equal(per_tensor, slab) and not (ws_t.gamma == ws_t.gamma[0]).all()


def test_argument_checks(K, dev):
    L = lenet_layout()
    T = L.ntensors
    lib = N.cuda()
    pair = torch.zeros(T, 21, dtype=torch.float64, device=dev)
    for P in (1, 17):
        with pytest.raises(ValueError):
            K.pair_scope_fold(L, P, pair)
    with pytest.raises(ValueError):
        K.pair_scope_fold(L, 6, pair)                       # 15 pairs, not 21
    with pytest.raises(ValueError):
        K.pair_scope_fold(L, 7, pair.float())
    with pytest.raises(ValueError):
        K.pair_dist(L, torch.zeros(7, L.total, device=dev), L.total, 7, pair[:, :20])
    with pytest.raises(ValueError):
        K.nnm_mix_table(L, 7, 7, pair, torch.zeros(7, T, dtype=torch.int32, device=dev), True)
    st = K._stream()
    assert lib.drc_pair_scope_fold(None, T, 7, st) == 1
    assert lib.drc_pair_scope_fold(pair.data_ptr(), 0, 7, st) == 1
    assert lib.drc_pair_scope_fold(pair.data_ptr(), T, 17, st) == 1
    partials = torch.zeros(L.ntiles, 5, dtype=torch.float64, device=dev)
    dist = torch.zeros(T, 5, dtype=torch.float64, device=dev)
    w = torch.zeros(T, 5, dtype=torch.float32, device=dev)
    for n, tau in ((0, 1.0), (17, 1.0), (5, 0.0), (5, float("inf")), (5, float("nan"))):
        with pytest.raises(ValueError):
            K.centered_clip_model_weights(L, n, tau, partials, dist, w)
    with pytest.raises(ValueError):
        K.centered_clip_model_weights(L, 5, 1.0, partials, dist[:, :4], w)
    a = N.CcArgs()
    a.n, a.tau, a.tv, a.partials, a.weights = 5, 1.0, L.tile_view(dev), partials.data_ptr(), w.data_ptr()
    assert lib.drc_cc_model_weights(C.byref(a), st) == 1      # no dist
    a.dist, a.tau = dist.data_ptr(), -1.0
    assert lib.drc_cc_model_weights(C.byref(a), st) == 1
    ws = K.AttackWorkspace(L, 7, dev)
    bitmap = torch.ones(1, dtype=torch.int32, device=dev)
    step = torch.zeros(1, dtype=torch.int64, device=dev)
    with pytest.raises(ValueError):
        K.ps_attack_model(L, torch.zeros(7, L.total, device=dev), L.total, 7, adv_bitmap=bitmap, adv_len=1, step_ptr=step, ws=ws,
                          fold=K.attack_fold_buffer(L, 6, dev))
    with pytest.raises(ValueError):
        K.ps_attack_model(L, torch.zeros(7, L.total, device=dev), L.total, 7, adv_bitmap=bitmap, adv_len=1, step_ptr=step, ws=None,
                          fold=K.attack_fold_buffer(L, 7, dev))
    aa = N.AttackArgs()
    aa.P, aa.mode, aa.tv = 7, 6, L.tile_view(dev)
    aa.stats, aa.partials, aa.gamma = ws.stats.data_ptr(), ws.partials.data_ptr(), ws.gamma.data_ptr()
    assert lib.drc_attack_solve_model(C.byref(aa), st) == 1   # no fold
    aa.mode = 5
    aa.fold = K.attack_fold_buffer(L, 7, dev).data_ptr()
    assert lib.drc_attack_solve_model(C.byref(aa), st) == 1   # ALIE has no solve
    torch.cuda.synchronize()


def test_the_flag_changes_the_fused_choice(K, dev):
    """Worker 0 far off in the first tensor only, worker 1 in the last: per tensor, multi-Krum drops a different worker in those
    two tensors; at model scope it drops one worker everywhere.  Both choices match the oracle of their scope."""
    L = lenet_layout()
    P, f, m = 7, 1, 6
    X = int_slots(L, P, dev, seed=11, lo=-1, hi=2)
    first, last = L.specs[0], L.specs[-1]
    X[0, first.offset: first.offset + first.numel] += 40
    X[1, last.offset: last.offset + last.numel] += 40
    Xn = X.cpu().numpy()
    T = L.ntensors
    pair = torch.zeros(T, P * (P - 1) // 2, dtype=torch.float64, device=dev)
    sel_t = torch.zeros(m, T, dtype=torch.int32, device=dev)
    K.krum_select(L, X, L.total, P, f, pair, sel_t, m=m)
    for t, s in enumerate(L.specs):
        assert sorted(sel_t[:, t].tolist()) == sorted(oracle.multi_krum_indices(Xn[:, s.offset: s.offset + s.numel], f, m))
    assert 0 not in sel_t[:, 0].tolist() and 1 not in sel_t[:, T - 1].tolist()
    pair = model_table(K, L, X, P, dev)
    sel_m = torch.zeros(m, T, dtype=torch.int32, device=dev)
    K.krum_select(L, X, L.total, P, f, pair, sel_m, m=m, filled=True)
    want = oracle.multi_krum_indices(oracle.model_rows(Xn, [(s.offset, s.numel) for s in L.specs]), f, m)
    assert (sel_m.cpu().numpy() == np.array(want)[:, None]).all() and len({0, 1} & set(want)) == 1
    assert not torch.equal(sel_m, sel_t)


# ------------------------------------------------------------------------------------------------ engine
def _cfg(**kw):
    base = dict(network="LeNet", dataset="MNIST", batch_size=16, max_steps=12, num_workers=7, transport="nvl", lr=0.02,
                momentum=0.9, synthetic_size=512, eval_freq=10 ** 6, compress_grad="None", dtype="fp32", cuda_graphs=False,
                approach="baseline", mode="multi_krum", worker_fail=1, err_mode="rev_grad", rule_scope="model")
    base.update(kw)
    if base["mode"] == "centered_clip":
        base.setdefault("clip_tau", 0.05)
    return JobConfig(**base)


def _run(cfg, steps):
    t = Trainer(cfg, rank=0, world=1, device=torch.device("cuda", 0), quiet=True)
    losses = [t.train_step()["loss"] for _ in range(steps)]
    t.synchronize()
    return t, losses


ENGINE_RULES = [dict(mode="krum"), dict(mode="multi_krum"), dict(mode="geometric_median"), dict(mode="bulyan"),
                dict(mode="centered_clip"), dict(mode="multi_krum", err_mode="minmax", attack_scope="model", worker_fail=2),
                dict(approach="detox", mode="multi_krum", num_workers=15, group_size=3, worker_fail=3),
                dict(approach="detox", mode="centered_clip", num_workers=9, group_size=3),
                dict(approach="nnm", mode="krum"), dict(approach="nnm", mode="coordinate_median"),
                dict(approach="nnm", mode="bulyan"), dict(approach="nnm", mode="geometric_median")]


@pytest.mark.parametrize("rule", ENGINE_RULES, ids=lambda r: "-".join(str(v) for v in r.values()))
def test_fused_matches_library_op_engine(monkeypatch, rule):
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    a, _ = _run(_cfg(**rule), 4)
    b, _ = _run(_cfg(transport="nccl", **rule), 4)
    assert not a.engine.pipeline_ps and a.engine.ps.plan.scope == "model"
    pa, pb = a.engine.master_params(), b.engine.master_params()
    assert torch.isfinite(pa).all()
    tol = 2e-4 if "geometric_median" in rule.values() else 2e-5
    assert torch.allclose(pa, pb, atol=tol), float((pa - pb).abs().max())


_RESNET = dict(network="ResNet18", dataset="Cifar10", batch_size=8, dtype="bf16", synthetic_size=256, num_workers=7)


@pytest.mark.parametrize("kw", [dict(mode="multi_krum", err_mode="minmax", attack_scope="model"), dict(mode="centered_clip"),
                                dict(approach="nnm", mode="coordinate_median", err_mode="alie"),
                                dict(mode="coordinate_median", rule_scope="tensor", err_mode="minmax", attack_scope="model")])
def test_graph_replay_equals_eager(kw):
    e, le = _run(_cfg(cuda_graphs=False, **dict(_RESNET, **kw)), 4)
    g, lg = _run(_cfg(cuda_graphs=True, **dict(_RESNET, **kw)), 4)
    assert g.engine.graph is not None and not g.engine.pipeline_ps
    assert torch.equal(e.engine.master_params(), g.engine.master_params())
    assert le == lg and all(np.isfinite(lg))


@pytest.mark.parametrize("err", ["alie", "minmax"])
def test_training_under_attack_stays_finite(err):
    for kw in (dict(mode="multi_krum"), dict(mode="centered_clip", clip_tau=0.5, worker_momentum=0.9, momentum=0.0, lr=0.1),
               dict(approach="nnm", mode="multi_krum")):
        extra = dict(attack_scope="model") if err == "minmax" else {}
        t, losses = _run(_cfg(num_workers=15, worker_fail=3, err_mode=err, lr=kw.pop("lr", 0.05), **kw, **extra), 8)
        assert all(np.isfinite(losses)) and torch.isfinite(t.engine.master_params()).all(), (err, kw)
