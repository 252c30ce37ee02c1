"""Bulyan on the GPU: ``bulyan_select`` (csrc/cuda/robust.cu) against the fp64 oracle's recursive Krum selection, the mode-4
nearest-to-median average (csrc/cuda/aggregate_update.cu) bit for bit against an fp32 torch restatement and against the oracle,
bucketing and grid-size determinism, the argument checks, and whole jobs on the fused engine."""
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


def fill_valid(L, rows, dev, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(rows, L.total, generator=g) * scale
    x[:, ~torch.from_numpy(L.valid_mask())] = 0
    return x.to(dev)


def grid_valid(L, rows, dev, seed=0):
    """Multiples of 1/64 in [-2, 2]: every fp32 sum, difference and median of them is exact, so fp32 and fp64 meet the same
    distance ties (and there are many)."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randint(-128, 129, (rows, L.total), generator=g).float() / 64
    x[:, ~torch.from_numpy(L.valid_mask())] = 0
    return x.to(dev)


def poison(L, X, b, seed):
    """Replace up to ``b`` rows of every valid coordinate of ``X`` [P, D] with +-1e30, +-Inf or NaN."""
    if b == 0:
        return X
    P = X.shape[0]
    g = torch.Generator().manual_seed(seed)
    rank = torch.rand(P, L.total, generator=g).argsort(0)
    nbad = torch.randint(0, b + 1, (L.total,), generator=g)
    pool = torch.tensor([1e30, -1e30, INF, -INF, NAN])
    vals = pool[torch.randint(0, 5, (P, L.total), generator=g)]
    bad = (rank < nbad) & torch.from_numpy(L.valid_mask())
    return torch.where(bad.to(X.device), vals.to(X.device), X)


def near_median_sum(X, f):
    """fp32 restatement of mode 4 on X [theta, d]: sort, fp32 median, window walk, ascending sum, times 1 / beta."""
    S = X.sort(0).values
    theta = S.shape[0]
    beta = theta - 2 * f
    lo, hi = S[(theta - 1) // 2], S[theta // 2]
    m = lo if theta % 2 else 0.5 * lo + 0.5 * hi
    s = torch.zeros(S.shape[1], dtype=torch.int64, device=S.device)
    moving = torch.ones(S.shape[1], dtype=torch.bool, device=S.device)
    for j in range(2 * f):
        vin, vout = S[j + beta], S[j]
        din, dout = (vin - m).abs(), (vout - m).abs()
        moving &= (din < dout) | (dout.isnan() & ~din.isnan()) | (vin == vout) | (vin.isnan() & vout.isnan())
        s += moving
    acc = S.gather(0, s[None])[0].clone()
    for k in range(1, beta):
        acc += S.gather(0, (s + k)[None])[0]
    return acc * (1.0 / beta)


def ctrl(dev):
    return (torch.ones(1, dtype=torch.int64, device=dev), torch.zeros(4, dtype=torch.int32, device=dev),
            torch.zeros(8, dtype=torch.int64, device=dev))


def slot_table(L, rows, slots, dev, seed):
    """int32 [rows, T]: for every tensor a random choice of ``rows`` distinct slots out of ``slots``."""
    g = torch.Generator().manual_seed(seed)
    cols = [torch.randperm(slots, generator=g)[:rows] for _ in range(L.ntensors)]
    return torch.stack(cols, 1).to(torch.int32).contiguous().to(dev)


# ------------------------------------------------------------------------------------------------ selection
@pytest.mark.parametrize("with_rows", [False, True])
@pytest.mark.parametrize("P", [3, 7, 11, 15, 16])
def test_bulyan_select_matches_oracle(K, dev, P, with_rows):
    L = lenet_layout()
    T = L.ntensors
    S = P + 3 if with_rows else P                                        # slots in the slab
    mask = torch.from_numpy(L.valid_mask()).to(dev)
    for f in sorted({0, (P - 3) // 4}):
        honest = fill_valid(L, 1, dev, seed=6, scale=0.1)[0]
        slab = honest[None] + 0.01 * fill_valid(L, S, dev, seed=7 + P + f)
        slab[S - 1] = fill_valid(L, 1, dev, seed=8, scale=30.0)[0]
        slab[2] = -100 * slab[2]
        slab[0, mask] = NAN                                              # slot 0: NaN, the first index a plain scan keeps
        slab = slab.contiguous()
        rows = slot_table(L, P, S, dev, seed=P + f) if with_rows else None
        pair = torch.zeros(T, P * (P - 1) // 2, dtype=torch.float64, device=dev)
        theta = P - 2 * f
        sel = torch.full((theta, T), -1, dtype=torch.int32, device=dev)
        K.bulyan_select(L, slab, L.total, P, f, pair, sel, rows=rows)
        torch.cuda.synchronize()
        assert float(pair.abs().sum()) == 0
        sl = slab.cpu().double().numpy()
        for t, spec in enumerate(L.specs):
            slots = rows[:, t].tolist() if with_rows else list(range(P))
            X = sl[slots, spec.offset:spec.offset + spec.numel]
            want = [slots[i] for i in oracle.bulyan_indices(X, f)]
            assert sel[:, t].tolist() == want, (f, t, sel[:, t].tolist(), want)


def test_bulyan_select_rejects_bad_arguments(K, dev):
    L = lenet_layout()
    T = L.ntensors
    slab = fill_valid(L, 8, dev)
    pair = torch.zeros(T, 28, dtype=torch.float64, device=dev)
    for P, f in ((6, 1), (17, 0), (7, -1)):
        with pytest.raises(ValueError):
            K.bulyan_select(L, slab, L.total, P, f, pair, torch.zeros(max(P - 2 * f, 1), T, dtype=torch.int32, device=dev))
    with pytest.raises(ValueError):                                      # select must have theta = P - 2f rows
        K.bulyan_select(L, slab, L.total, 7, 1, pair, torch.zeros(6, T, dtype=torch.int32, device=dev))
    for P, f in ((6, 1), (17, 0)):                                       # the C entry point refuses them itself
        a = N.BulyanSelectArgs(None, T, P, f, 1, None)
        assert N.cuda().drc_bulyan_select(C.byref(a), K._stream()) == 1


# ------------------------------------------------------------------------------------------------ mode 4
def _grid():
    return [(theta, f) for theta in (3, 4, 5, 8, 9, 13, 16) for f in range((theta + 1) // 2) if 2 * f < theta]


@pytest.mark.parametrize("theta,f", _grid())
def test_near_median_kernel_matches_torch_and_oracle(K, dev, theta, f):
    L = lenet_layout()
    S = theta + 2
    sel = slot_table(L, theta, S, dev, seed=theta * 17 + f)
    hp = hyperparams_tensor(JobConfig(lr=0.1, momentum=0.9, weight_decay=1e-3), dev)
    for kind in ("normal", "grid"):
        base = fill_valid(L, S, dev, seed=theta * 31 + f) if kind == "normal" else grid_valid(L, S, dev, seed=theta + f)
        slab = poison(L, base, f, seed=theta + 7 * f).contiguous()
        params = fill_valid(L, 1, dev, seed=5)[0]
        p0 = params.clone()
        mom = torch.zeros_like(params)
        gout = torch.full((L.total,), 7.0, device=dev)
        step, cnt, flags = ctrl(dev)
        K.aggregate_update(L, slab, L.total, params=params, momentum=mom, hp=hp, step_ptr=step, done_counter=cnt[0:1], K=theta,
                           scale=1.0 / (theta - 2 * f), near_median=f, select=sel, grad_out=gout, flags=[flags[0:1]])
        torch.cuda.synchronize()
        sl = slab.cpu().double().numpy()
        for t, spec in enumerate(L.specs):
            cols = slice(spec.offset, spec.offset + spec.numel)
            X = slab[sel[:, t].long(), cols]
            got = gout[cols]
            assert torch.equal(got, near_median_sum(X, f)), (kind, t)  # the same fp32 operations in the same order
            assert torch.isfinite(got).all()
            if kind == "grid":
                ref = oracle.nearest_to_median_mean(sl[sel[:, t].cpu().numpy(), cols], f)
                np.testing.assert_allclose(got.cpu().double().numpy(), ref, rtol=1e-6, atol=1e-6)
        mask = torch.from_numpy(L.valid_mask()).to(dev)
        assert float(gout[~mask].abs().sum()) == 0
        p_ref = p0.double() - 0.1 * (gout.double() + 1e-3 * p0.double())       # first SGD step: momentum buffer = d_p
        assert torch.allclose(params.double(), p_ref, atol=1e-5)
        assert flags[0].item() == 2 and cnt[0].item() == 0


def test_near_median_is_independent_of_buckets_and_grid(K, dev):
    L = ArenaLayout.from_model(build_model("ResNet18"), bf16=True, channels_last=True)
    theta, f = 9, 2
    slab = poison(L, fill_valid(L, 11, dev, seed=3, scale=0.01), f, seed=4).contiguous()
    sel = slot_table(L, theta, 11, dev, seed=5)
    hp = hyperparams_tensor(JobConfig(lr=0.1, momentum=0.9), dev)
    p0 = fill_valid(L, 1, dev, seed=5)[0]
    nt = L.ntiles
    bounds = [0, nt // 5, nt // 5 + 1, (2 * nt) // 3, nt]
    results = []
    for how in ("one", "buckets", "grid1", "grid37"):
        params, mom = p0.clone(), torch.zeros_like(p0)
        step, cnt, flags = ctrl(dev)
        for it in (1, 2):
            step.fill_(it)
            kw = dict(params=params, momentum=mom, hp=hp, step_ptr=step, done_counter=cnt[0:1], K=theta,
                      scale=1.0 / (theta - 2 * f), near_median=f, select=sel)
            if how == "buckets":
                for i in range(len(bounds) - 1):
                    K.aggregate_update(L, slab, L.total, tile_range=(bounds[i], bounds[i + 1]),
                                       flags=[flags[0:1]] if i == len(bounds) - 2 else [], **kw)
            else:
                K.aggregate_update(L, slab, L.total, grid={"one": None, "grid1": 1, "grid37": 37}[how], flags=[flags[0:1]], **kw)
        torch.cuda.synchronize()
        assert flags[0].item() == 3
        results.append(params)
    for r in results[1:]:
        assert torch.equal(r, results[0])
    assert torch.isfinite(results[0]).all()


def test_near_median_rejects_bad_arguments(K, dev):
    L = lenet_layout()
    T = L.ntensors
    slab = fill_valid(L, 17, dev)
    hp = hyperparams_tensor(JobConfig(), dev)
    params, mom = torch.zeros(L.total, device=dev), torch.zeros(L.total, device=dev)
    step, cnt, _ = ctrl(dev)
    kw = dict(params=params, momentum=mom, hp=hp, step_ptr=step, done_counter=cnt[0:1])
    for theta, f, scale in ((17, 1, 1.0 / 15), (5, 3, 1.0), (7, 2, 1.0 / 7)):      # too many rows, nothing kept, wrong scale
        sel = torch.zeros(theta, T, dtype=torch.int32, device=dev)
        with pytest.raises(ValueError):
            K.aggregate_update(L, slab, L.total, K=theta, scale=scale, near_median=f, select=sel, **kw)
    with pytest.raises(ValueError):                                                 # no select table
        K.aggregate_update(L, slab, L.total, K=5, scale=1.0 / 3, near_median=1, **kw)
    sel = torch.zeros(16, T, dtype=torch.int32, device=dev)
    for theta, f, table in ((17, 1, sel), (5, 3, sel), (5, 1, None)):             # the C entry point refuses them itself
        a = N.UpdateArgs()
        a.mode, a.K, a.trim, a.scale, a.select = 4, theta, f, 1.0, None if table is None else table.data_ptr()
        assert N.cuda().drc_aggregate_update(C.byref(a), 1, K._stream()) == 1


# ------------------------------------------------------------------------------------------------ engine
def _cfg(**kw):
    base = dict(network="LeNet", dataset="MNIST", batch_size=16, max_steps=12, num_workers=7, transport="nvl", lr=0.02,
                momentum=0.9, synthetic_size=512, eval_freq=10 ** 6, compress_grad="None", dtype="fp32", cuda_graphs=False,
                approach="baseline", mode="bulyan", worker_fail=1)
    base.update(kw)
    return JobConfig(**base)


def _run(cfg, steps):
    t = Trainer(cfg, rank=0, world=1, device=torch.device("cuda", 0), quiet=True)
    losses = [t.train_step()["loss"] for _ in range(steps)]
    t.synchronize()
    return t, losses


@pytest.mark.parametrize("rule", [dict(), dict(approach="detox", num_workers=14, group_size=2)])
def test_fused_bulyan_matches_library_op_engine(monkeypatch, rule):
    """pair_dist + bulyan_select + mode 4 against the torch-op PS, in true fp32."""
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    kw = dict(err_mode="constant", **rule)
    a, _ = _run(_cfg(**kw), 4)
    b, _ = _run(_cfg(transport="nccl", **kw), 4)
    assert not a.engine.pipeline_ps and a.engine.ps.rule == ("detox_bulyan" if rule else "bulyan")
    pa, pb = a.engine.master_params(), b.engine.master_params()
    assert torch.isfinite(pa).all()
    assert torch.allclose(pa, pb, atol=2e-5), float((pa - pb).abs().max())


_RESNET = dict(network="ResNet18", dataset="Cifar10", batch_size=8, dtype="bf16", synthetic_size=256, err_mode="rev_grad")


def test_bulyan_graph_replay_equals_eager():
    e, le = _run(_cfg(cuda_graphs=False, **_RESNET), 6)
    g, lg = _run(_cfg(cuda_graphs=True, **_RESNET), 6)
    assert g.engine.graph is not None and not g.engine.pipeline_ps
    assert torch.equal(e.engine.master_params(), g.engine.master_params())
    assert le == lg


def test_bulyan_trains_under_attack_where_the_mean_does_not():
    """Same workers, batches and adversary schedule (worker_fail = 1 of 7); only the attack and the rule change.  Under the
    sign-flip attack the mean leaves the attack-free trajectory, Bulyan stays close to it."""
    def dist(a, b):
        d = (a - b).abs().max()
        return float(d) if torch.isfinite(d) else float("inf")
    kw = dict(lr=0.05)
    clean, _ = _run(_cfg(mode="normal", err_mode="none", **kw), 10)
    ref = clean.engine.master_params()
    mean, _ = _run(_cfg(mode="normal", err_mode="rev_grad", **kw), 10)
    d_mean = dist(mean.engine.master_params(), ref)
    assert d_mean > 1e-1, d_mean
    t, losses = _run(_cfg(err_mode="rev_grad", **kw), 10)
    assert losses[-1] < losses[0], losses
    p = t.engine.master_params()
    assert torch.isfinite(p).all()
    assert dist(p, ref) < 0.1 * d_mean, (dist(p, ref), d_mean)


@pytest.mark.parametrize("mode", ["alie", "minmax"])
def test_bulyan_under_ps_attacks_in_the_captured_step(mode):
    kw = dict(_RESNET, err_mode=mode)
    e, le = _run(_cfg(cuda_graphs=False, **kw), 5)
    g, lg = _run(_cfg(cuda_graphs=True, **kw), 5)
    eng = g.engine
    assert eng.graph is not None and eng.ps.attack == A.attack_code(mode) and eng.ps.rule == "bulyan"
    assert torch.equal(e.engine.master_params(), eng.master_params())
    assert le == lg and all(np.isfinite(lg))
