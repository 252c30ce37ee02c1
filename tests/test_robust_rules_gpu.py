"""Coordinate-wise median / trimmed mean (aggregate_update mode 3) and multi-Krum (krum_select with m rows) on the GPU: the kernels
against the fp64 oracles and torch, bucketing and grid-size determinism, and whole jobs on the fused engine."""
import numpy as np
import pytest
import torch

from draco_b200 import JobConfig
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


@pytest.fixture
def fill_valid():
    def fill(L, rows, dev, seed=0, scale=1.0):
        g = torch.Generator().manual_seed(seed)
        mask = torch.from_numpy(L.valid_mask())
        x = torch.randn(rows, L.total, generator=g) * scale
        x[:, ~mask] = 0
        return x.to(dev)
    return fill


@pytest.fixture
def ctrl():
    def make(dev, step=1):
        return (torch.full((1,), step, dtype=torch.int64, device=dev), torch.zeros(4, dtype=torch.int32, device=dev),
                torch.zeros(8, dtype=torch.int64, device=dev))
    return make


def lenet_layout():
    """LeNet: 8 tensors, most of which end inside a tile."""
    return ArenaLayout.from_model(build_model("LeNet"), bf16=False, channels_last=True)


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


def ascending_sum(X, b):
    """fp32 trimmed mean summed in ascending order, as the kernel does it."""
    P = X.shape[0]
    S = X.sort(0).values
    acc = S[b].clone()
    for k in range(b + 1, P - b):
        acc += S[k]
    return acc * (1.0 / (P - 2 * b))


# ------------------------------------------------------------------------------------------------ mode 3
def _grid():
    out = []
    for P in (3, 4, 7, 8, 13, 16):
        for b in sorted({0, 1, (P - 1) // 2}):
            out.append((P, b))
    return out


@pytest.mark.parametrize("P,b", _grid())
def test_trimmed_mean_kernel_matches_oracle(K, dev, fill_valid, ctrl, P, b):
    L = lenet_layout()
    mask = torch.from_numpy(L.valid_mask()).to(dev)
    slots = poison(L, fill_valid(L, P, dev, seed=P * 31 + b), b, seed=P + 7 * b).contiguous()
    cfg = JobConfig(lr=0.1, momentum=0.9, weight_decay=1e-3)
    hp = hyperparams_tensor(cfg, dev)
    params = fill_valid(L, 1, dev, seed=5)[0]
    p0 = params.clone()
    mom = torch.zeros_like(params)
    gout = torch.full((L.total,), 7.0, device=dev)
    peer = torch.zeros(L.total, device=dev)
    step, cnt, flags = ctrl(dev, 1)
    K.aggregate_update(L, slots, L.total, params=params, momentum=mom, hp=hp, step_ptr=step, done_counter=cnt[0:1], K=P,
                       scale=1.0 / (P - 2 * b), trim=b, grad_out=gout, dst=[peer], flags=[flags[0:1]])
    torch.cuda.synchronize()
    assert torch.equal(gout, ascending_sum(slots, b))                 # same fp32 additions in the same order
    if P % 2 == 1 and b == (P - 1) // 2:
        assert torch.equal(gout, slots.sort(0).values[P // 2])        # odd-P median: the middle value, bit for bit
    sl = slots.cpu().double().numpy()
    for spec in L.specs:
        ref = oracle.trimmed_mean(sl[:, spec.offset:spec.offset + spec.numel], b)
        got = gout[spec.offset:spec.offset + spec.numel].cpu().double().numpy()
        # 1e-6 of the data's unit scale: an fp32 sum that cancels to near zero keeps only its absolute accuracy
        np.testing.assert_allclose(got, ref, rtol=1e-6, atol=1e-6)
    assert torch.isfinite(params).all() and torch.isfinite(mom).all()
    assert float(gout[~mask].abs().sum()) == 0 and float(params[~mask].abs().sum()) == 0
    p_ref = p0.double() - 0.1 * (gout.double() + 1e-3 * p0.double())          # first SGD step: momentum buffer = d_p
    assert torch.allclose(params.double(), p_ref, atol=1e-5)
    assert torch.equal(peer, params) and flags[0].item() == 2 and cnt[0].item() == 0


@pytest.mark.parametrize("optimizer", ["sgd", "adam"])
def test_trimmed_mean_update_matches_library_optimizers_over_steps(K, dev, fill_valid, ctrl, optimizer):
    L = lenet_layout()
    P, b = 7, 2
    if optimizer == "sgd":
        cfg = JobConfig(lr=0.05, momentum=0.8, weight_decay=5e-4, nesterov=True)
    else:
        cfg = JobConfig(optimizer="adam", lr=1e-3, weight_decay=1e-4)
    hp = hyperparams_tensor(cfg, dev)
    params = fill_valid(L, 1, dev, seed=2)[0]
    ref_p = params.clone().requires_grad_(True)
    if optimizer == "sgd":
        opt = torch.optim.SGD([ref_p], lr=0.05, momentum=0.8, weight_decay=5e-4, nesterov=True)
    else:
        # the fused Adam folds the bias corrections into the step size like AdamModified (the reference's formula): eps is not
        # scaled by sqrt(1 - beta2^t) as in torch.optim.Adam, which matters where the aggregate is close to zero
        from draco_b200.optim import AdamModified
        opt = AdamModified([ref_p], lr=1e-3, weight_decay=1e-4)
    mom = torch.zeros_like(params)
    v = torch.zeros_like(params) if optimizer == "adam" else None
    gout = torch.zeros_like(params)
    step, cnt, _ = ctrl(dev, 1)
    for it in range(1, 5):
        slots = poison(L, fill_valid(L, P, dev, seed=10 + it, scale=0.3), b, seed=it).contiguous()
        step.fill_(it)
        K.aggregate_update(L, slots, L.total, params=params, momentum=mom, exp_avg_sq=v, hp=hp, step_ptr=step,
                           done_counter=cnt[0:1], K=P, scale=1.0 / (P - 2 * b), trim=b, first_step=1, grad_out=gout)
        torch.cuda.synchronize()
        assert torch.isfinite(gout).all()
        if optimizer == "sgd":
            ref_p.grad = gout.clone()
            opt.step()
        else:
            opt.step(grads=[gout.clone()], mode="trimmed_mean")
    torch.cuda.synchronize()
    assert torch.allclose(params, ref_p.detach(), atol=2e-6 if optimizer == "sgd" else 1e-5), \
        float((params - ref_p.detach()).abs().max())


def test_trimmed_mean_is_independent_of_buckets_and_grid(K, dev, fill_valid, ctrl):
    """The sum order is fixed by the sort: one launch, several tile-range buckets and other grid sizes give the same bits."""
    L = ArenaLayout.from_model(build_model("ResNet18"), bf16=True, channels_last=True)
    P, b = 7, 2
    slots = poison(L, fill_valid(L, P, dev, seed=3, scale=0.01), b, seed=4).contiguous()
    cfg = JobConfig(lr=0.1, momentum=0.9)
    hp = hyperparams_tensor(cfg, dev)
    p0 = fill_valid(L, 1, dev, seed=5)[0]
    nt = L.ntiles
    bounds = [0, nt // 5, nt // 5 + 1, (2 * nt) // 3, nt]
    results = []
    for how in ("one", "buckets", "grid1", "grid37"):
        params, mom = p0.clone(), torch.zeros_like(p0)
        step, cnt, flags = ctrl(dev, 1)
        for it in (1, 2):
            step.fill_(it)
            kw = dict(params=params, momentum=mom, hp=hp, step_ptr=step, done_counter=cnt[0:1], K=P, scale=1.0 / (P - 2 * b), trim=b)
            if how == "buckets":
                for i in range(len(bounds) - 1):
                    K.aggregate_update(L, slots, L.total, tile_range=(bounds[i], bounds[i + 1]),
                                       flags=[flags[0:1]] if i == len(bounds) - 2 else [], **kw)
            else:
                K.aggregate_update(L, slots, L.total, grid={"one": None, "grid1": 1, "grid37": 37}[how], flags=[flags[0:1]], **kw)
        torch.cuda.synchronize()
        assert flags[0].item() == 3
        results.append(params)
    for r in results[1:]:
        assert torch.equal(r, results[0])
    assert torch.isfinite(results[0]).all()


def test_trimmed_mean_rejects_bad_arguments(K, dev, fill_valid, ctrl):
    import ctypes as C

    from draco_b200 import _native as N
    L = lenet_layout()
    slots = fill_valid(L, 17, dev)
    hp = hyperparams_tensor(JobConfig(), dev)
    params, mom = torch.zeros(L.total, device=dev), torch.zeros(L.total, device=dev)
    step, cnt, _ = ctrl(dev, 1)
    kw = dict(params=params, momentum=mom, hp=hp, step_ptr=step, done_counter=cnt[0:1])
    for P, b, scale in ((17, 1, 1.0 / 15), (5, 3, 1.0), (7, 2, 1.0 / 7)):        # too many rows, nothing kept, wrong scale
        with pytest.raises(ValueError):
            K.aggregate_update(L, slots, L.total, K=P, scale=scale, trim=b, **kw)
    # the C entry point refuses the same shapes itself (cudaErrorInvalidValue) without launching anything
    for P, b in ((17, 1), (5, 3)):
        a = N.UpdateArgs()
        a.mode, a.K, a.trim, a.scale = 3, P, b, 1.0
        assert N.cuda().drc_aggregate_update(C.byref(a), 1, K._stream()) == 1


# ------------------------------------------------------------------------------------------------ multi-Krum
@pytest.mark.parametrize("P,s", [(7, 2), (16, 3), (5, 1)])
def test_multi_krum_select_matches_oracle(K, dev, fill_valid, ctrl, P, s):
    L = lenet_layout()
    T = L.ntensors
    honest = fill_valid(L, 1, dev, seed=6, scale=0.1)[0]
    slots = honest[None] + 0.01 * fill_valid(L, P, dev, seed=7 + P)
    slots[2] = -100 * slots[2]
    slots[P - 1] = fill_valid(L, 1, dev, seed=8, scale=30.0)[0]
    slots = slots.contiguous()
    pair = torch.zeros(T, P * (P - 1) // 2, dtype=torch.float64, device=dev)
    sl = slots.cpu().double().numpy()
    one = torch.full((T,), -1, dtype=torch.int32, device=dev)
    K.krum_select(L, slots, L.total, P, s, pair, one)                 # the Krum call as it has always been made
    torch.cuda.synchronize()
    assert float(pair.abs().sum()) == 0
    for t, spec in enumerate(L.specs):
        assert int(one[t]) == oracle.krum_index(sl[:, spec.offset:spec.offset + spec.numel], s), t
    for m in (1, 3, P - s):
        sel = torch.full((m, T), -1, dtype=torch.int32, device=dev)
        K.krum_select(L, slots, L.total, P, s, pair, sel, m=m)
        torch.cuda.synchronize()
        assert float(pair.abs().sum()) == 0
        assert torch.equal(sel[0], one)
        for t, spec in enumerate(L.specs):
            assert sel[:, t].tolist() == oracle.multi_krum_indices(sl[:, spec.offset:spec.offset + spec.numel], s, m), (m, t)
    # the multi-Krum aggregate: mode 0 averages the m selected rows
    m = P - s
    hp = hyperparams_tensor(JobConfig(lr=1.0, momentum=0.0), dev)
    params, mom, gout = (torch.zeros(L.total, device=dev) for _ in range(3))
    step, cnt, _ = ctrl(dev, 1)
    K.aggregate_update(L, slots, L.total, params=params, momentum=mom, hp=hp, step_ptr=step, done_counter=cnt[0:1], K=m,
                       scale=1.0 / m, select=sel, grad_out=gout)
    torch.cuda.synchronize()
    for spec in L.specs:
        ref = oracle.multi_krum(sl[:, spec.offset:spec.offset + spec.numel], s, m)
        np.testing.assert_allclose(gout[spec.offset:spec.offset + spec.numel].cpu().double().numpy(), ref, rtol=1e-5, atol=1e-6)


def test_multi_krum_ranks_a_nan_row_last(K, dev, fill_valid, ctrl):
    """A row that sends NaN has NaN distances: they sort last in every honest row's neighbour list, and its own NaN score
    ranks last, so neither Krum nor multi-Krum picks it -- as on the library path (torch.sort / argsort put NaN last)."""
    L = lenet_layout()
    T, P, s = L.ntensors, 7, 2
    honest = fill_valid(L, 1, dev, seed=16, scale=0.1)[0]
    slots = honest[None] + 0.01 * fill_valid(L, P, dev, seed=17)
    mask = torch.from_numpy(L.valid_mask()).to(dev)
    slots[0, mask] = NAN                                   # slot 0: the first index, which a plain `<` scan would keep
    slots[4] = -100 * slots[4]
    slots = slots.contiguous()
    pair = torch.zeros(T, P * (P - 1) // 2, dtype=torch.float64, device=dev)
    sel = torch.full((P - s, T), -1, dtype=torch.int32, device=dev)
    K.krum_select(L, slots, L.total, P, s, pair, sel, m=P - s)
    torch.cuda.synchronize()
    sl = slots.cpu().double().numpy()
    for t, spec in enumerate(L.specs):
        want = oracle.multi_krum_indices(sl[:, spec.offset:spec.offset + spec.numel], s, P - s)
        assert 0 not in want and sel[:, t].tolist() == want, (t, sel[:, t].tolist(), want)


# ------------------------------------------------------------------------------------------------ engine
def _cfg(**kw):
    base = dict(network="LeNet", dataset="MNIST", batch_size=16, max_steps=12, num_workers=7, transport="nvl", lr=0.02,
                momentum=0.9, synthetic_size=512, eval_freq=10 ** 6, compress_grad="None", dtype="fp32", cuda_graphs=False)
    base.update(kw)
    return JobConfig(**base)


def _run(cfg, steps):
    t = Trainer(cfg, rank=0, world=1, device=torch.device("cuda", 0), quiet=True)
    losses = [t.train_step()["loss"] for _ in range(steps)]
    t.synchronize()
    return t, losses


@pytest.mark.parametrize("mode", ["coordinate_median", "trimmed_mean", "multi_krum"])
def test_fused_robust_rules_match_library_op_engine(monkeypatch, mode):
    """The kernels path (pipelined buckets for the coordinate-wise rules) against the torch-op PS, in true fp32."""
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    kw = dict(approach="baseline", mode=mode, worker_fail=2, err_mode="constant")
    a, _ = _run(_cfg(**kw), 4)
    b, _ = _run(_cfg(transport="nccl", **kw), 4)
    assert a.engine.pipeline_ps == (mode != "multi_krum")
    pa, pb = a.engine.master_params(), b.engine.master_params()
    assert torch.allclose(pa, pb, atol=2e-5), float((pa - pb).abs().max())


def test_fused_robust_rules_train_under_attack_where_the_mean_does_not():
    """Every run has the same workers, batches and adversary schedule (worker_fail = 2); only the attack and the rule change.
    Under the sign-flip attack the mean leaves the attack-free trajectory, the robust rules stay close to it."""
    def dist(a, b):
        d = (a - b).abs().max()
        return float(d) if torch.isfinite(d) else float("inf")
    kw = dict(approach="baseline", worker_fail=2, lr=0.05)
    clean, _ = _run(_cfg(mode="normal", err_mode="none", **kw), 10)
    ref = clean.engine.master_params()
    mean, _ = _run(_cfg(mode="normal", err_mode="rev_grad", **kw), 10)
    d_mean = dist(mean.engine.master_params(), ref)
    assert d_mean > 1e-1, d_mean                               # the attack is real
    for mode in ("coordinate_median", "trimmed_mean", "multi_krum"):
        t, losses = _run(_cfg(mode=mode, err_mode="rev_grad", **kw), 10)
        assert losses[-1] < losses[0], (mode, losses)
        p = t.engine.master_params()
        assert torch.isfinite(p).all(), mode
        assert dist(p, ref) < 0.1 * d_mean, (mode, dist(p, ref), d_mean)


def test_coordinate_median_graph_replay_equals_eager():
    kw = dict(approach="baseline", mode="coordinate_median", worker_fail=1, err_mode="rev_grad", network="ResNet18", dataset="Cifar10",
              batch_size=8, num_workers=3, dtype="bf16", synthetic_size=256)
    e, le = _run(_cfg(cuda_graphs=False, **kw), 6)
    g, lg = _run(_cfg(cuda_graphs=True, **kw), 6)
    assert e.engine.pipeline_ps and g.engine.pipeline_ps and g.engine.graph is not None
    assert torch.equal(e.engine.master_params(), g.engine.master_params())
    assert le == lg
