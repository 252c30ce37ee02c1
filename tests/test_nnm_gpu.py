"""Nearest-neighbour mixing on the GPU: ``nnm_mix`` (csrc/cuda/robust.cu) masks and mixed distance table against the fp64
oracle, ``nnm_fold`` against A^T w / n_mix, the mixing variants of update modes 3 and 4 (csrc/cuda/aggregate_update.cu) bit for
bit against an fp32 torch restatement and against the oracle, bucketing and grid-size determinism, the argument checks, and
whole jobs on the fused engine for every base rule."""
import ctypes as C

import numpy as np
import pytest
import torch

from draco_b200 import JobConfig
from draco_b200 import _native as N
from draco_b200.codes import adversary as A
from draco_b200.codes import oracle
from draco_b200.config import NNM_MODES
from draco_b200.models import build_model
from draco_b200.parallel.arena import ArenaLayout
from draco_b200.parallel.ps import hyperparams_tensor
from draco_b200.parallel.trainer import Trainer

pytestmark = pytest.mark.gpu
NAN = float("nan")


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
    x = torch.randn(rows, L.total, generator=g) * scale * torch.rand(rows, 1, generator=g).add(0.2)
    x[:, ~torch.from_numpy(L.valid_mask())] = 0
    return x.to(dev)


def ctrl(dev):
    return (torch.ones(1, dtype=torch.int64, device=dev), torch.zeros(4, dtype=torch.int32, device=dev),
            torch.zeros(8, dtype=torch.int64, device=dev))


def pair_dist(K, L, slab, P, pair):
    pa = N.PairDistArgs(slab.data_ptr(), L.total, P, L.tile_view(slab.device), pair.data_ptr(), None)
    N.check(N.cuda().drc_pair_dist(C.byref(pa), K.stream_grid(L, 4), K._stream()), "pair_dist")


def square(row, P):
    """[P(P-1)/2] pair table (pair i < j at j(j-1)/2 + i) -> symmetric [P, P] with a zero diagonal."""
    D = np.zeros((P, P))
    for j in range(1, P):
        for i in range(j):
            D[i, j] = D[j, i] = row[j * (j - 1) // 2 + i]
    return D


def masks_to_A(col, P):
    return np.array([[(int(col[i]) >> j) & 1 for j in range(P)] for i in range(P)])


def mix_rows(X, masks, P, f):
    """fp32 restatement of the kernel's mixing: from +0, add the raw rows of the mask in ascending order, one multiply."""
    scale = torch.tensor(1.0 / (P - f), dtype=torch.float32, device=X.device)
    out = []
    for m in masks:
        y = torch.zeros_like(X[0])
        for j in range(P):
            if (int(m) >> j) & 1:
                y = y + X[j]
        out.append(y * scale)
    return torch.stack(out)


def trimmed_sum(Y, trim):
    S = Y.sort(0).values
    acc = torch.zeros_like(S[0])
    for k in range(trim, S.shape[0] - trim):
        acc = acc + S[k]
    return acc * (1.0 / (S.shape[0] - 2 * trim))


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


# ------------------------------------------------------------------------------------------------ nnm_mix
@pytest.mark.parametrize("P", list(range(3, 17)))
def test_nnm_mix_matches_oracle(K, dev, P):
    L = lenet_layout()
    T = L.ntensors
    mask = torch.from_numpy(L.valid_mask()).to(dev)
    for f in range(P):
        slab = fill_valid(L, P, dev, seed=P * 31 + f)
        slab[P - 1] = 40 * slab[P - 1]
        if f % 3 == 1:
            slab[1, mask] = NAN                                      # a NaN row
        slab = slab.contiguous()
        pair = torch.zeros(T, P * (P - 1) // 2, dtype=torch.float64, device=dev)
        pair_dist(K, L, slab, P, pair)
        raw = pair.clone()
        mix = torch.full((P, T), -1, dtype=torch.int32, device=dev)
        na = N.NnmMixArgs(pair.data_ptr(), T, P, f, mix.data_ptr(), 1)
        N.check(N.cuda().drc_nnm_mix(C.byref(na), K._stream()), "nnm_mix")
        torch.cuda.synchronize()
        sl = slab.cpu().double().numpy()
        for t, spec in enumerate(L.specs):
            D = square(raw[t].cpu().numpy(), P)
            A_ref = oracle.nnm_neighbours_d2(D, f)
            A_k = masks_to_A(mix[:, t].cpu().numpy().astype(np.uint32), P)
            assert A_k.tolist() == A_ref.tolist(), (P, f, t)
            if f % 3 != 1:                                           # no near ties in random data: the same as from the rows
                assert A_k.tolist() == oracle.nnm_neighbours(sl[:, spec.offset:spec.offset + spec.numel], f).tolist()
            got = square(pair[t].cpu().numpy(), P)
            want = oracle.nnm_pair_d2(D, A_ref, f)
            iu = np.triu_indices(P, 1)
            g, w = got[iu], want[iu]
            assert (np.isnan(g) == np.isnan(w)).all(), (P, f, t)
            ok = ~np.isnan(w)
            np.testing.assert_allclose(g[ok], w[ok], rtol=1e-9, atol=1e-11 * max(D[np.isfinite(D)].max(), 1e-30))
        # without mixed_out the table is left zeroed and the masks are the same
        pair2 = raw.clone()
        mix2 = torch.zeros_like(mix)
        K.nnm_mix(L, slab, L.total, P, f, torch.zeros_like(pair), mix2, mixed_out=False)
        torch.cuda.synchronize()
        assert torch.equal(mix2, mix)
        na = N.NnmMixArgs(pair2.data_ptr(), T, P, f, mix2.data_ptr(), 0)
        N.check(N.cuda().drc_nnm_mix(C.byref(na), K._stream()), "nnm_mix")
        torch.cuda.synchronize()
        assert float(pair2.abs().sum()) == 0


def test_nnm_mix_with_f_zero_is_the_mean_everywhere(K, dev):
    L = lenet_layout()
    P, T = 9, L.ntensors
    slab = fill_valid(L, P, dev, seed=1)
    pair = torch.zeros(T, P * (P - 1) // 2, dtype=torch.float64, device=dev)
    mix = torch.zeros(P, T, dtype=torch.int32, device=dev)
    K.nnm_mix(L, slab, L.total, P, 0, pair, mix, mixed_out=True)
    torch.cuda.synchronize()
    assert (mix == (1 << P) - 1).all()
    assert float(pair.abs().max()) < 1e-9 * float(slab.double().pow(2).sum())


# ------------------------------------------------------------------------------------------------ nnm_fold
@pytest.mark.parametrize("P,f", [(3, 1), (7, 1), (11, 4), (16, 3), (16, 0)])
def test_nnm_fold_matches_the_transpose(K, dev, P, f):
    L = lenet_layout()
    T = L.ntensors
    slab = fill_valid(L, P, dev, seed=P + f)
    pair = torch.zeros(T, P * (P - 1) // 2, dtype=torch.float64, device=dev)
    mix = torch.zeros(P, T, dtype=torch.int32, device=dev)
    K.nnm_mix(L, slab, L.total, P, f, pair, mix, mixed_out=False)
    g = torch.Generator().manual_seed(P)
    w_mix = torch.rand(T, P, generator=g).to(dev)
    w_mix /= w_mix.sum(1, keepdim=True)
    m = P - f
    sel = torch.stack([torch.randperm(P, generator=g)[:m] for _ in range(T)], 1).to(torch.int32).contiguous().to(dev)
    w1, w2 = torch.full((T, P), 7.0, device=dev), torch.full((T, P), 7.0, device=dev)
    K.nnm_fold(L, P, f, mix, w1, w_mix=w_mix)
    K.nnm_fold(L, P, f, mix, w2, select=sel, m=m)
    torch.cuda.synchronize()
    for t in range(T):
        Am = masks_to_A(mix[:, t].cpu().numpy().astype(np.uint32), P).astype(np.float64)
        ref1 = Am.T @ w_mix[t].cpu().double().numpy() / (P - f)
        u = np.zeros(P)
        u[sel[:, t].cpu().numpy()] = 1.0 / m
        ref2 = Am.T @ u / (P - f)
        np.testing.assert_allclose(w1[t].cpu().double().numpy(), ref1, rtol=1e-7, atol=1e-9)
        np.testing.assert_allclose(w2[t].cpu().double().numpy(), ref2, rtol=1e-7, atol=1e-9)
        assert abs(float(w1[t].double().sum()) - 1.0) < 1e-6 and abs(float(w2[t].double().sum()) - 1.0) < 1e-6


# ------------------------------------------------------------------------------------------------ modes 3 and 4 with mixing
def _cases():
    out = []
    for P in (3, 4, 5, 7, 8, 9, 11, 15, 16):
        for f in sorted({0, 1, (P - 1) // 2, P // 3}):
            if 2 * f < P:
                out.append(("median", P, f))
                out.append(("trimmed", P, f))
            if P >= 4 * f + 3:
                out.append(("bulyan", P, f))
    return out


@pytest.mark.parametrize("rule,P,f", _cases())
def test_mixed_modes_match_torch_and_oracle(K, dev, rule, P, f):
    L = lenet_layout()
    T = L.ntensors
    hp = hyperparams_tensor(JobConfig(lr=0.1, momentum=0.9, weight_decay=1e-3), dev)
    slab = fill_valid(L, P, dev, seed=P * 13 + f)
    slab[0] = -30 * slab[0]
    slab = slab.contiguous()
    pair = torch.zeros(T, P * (P - 1) // 2, dtype=torch.float64, device=dev)
    mix = torch.zeros(P, T, dtype=torch.int32, device=dev)
    K.nnm_mix(L, slab, L.total, P, f, pair, mix, mixed_out=rule == "bulyan")
    params = fill_valid(L, 1, dev, seed=5)[0]
    p0 = params.clone()
    mom = torch.zeros_like(params)
    gout = torch.full((L.total,), 7.0, device=dev)
    step, cnt, flags = ctrl(dev)
    kw = dict(params=params, momentum=mom, hp=hp, step_ptr=step, done_counter=cnt[0:1], grad_out=gout, flags=[flags[0:1]],
              mix=mix, mix_f=f)
    if rule == "bulyan":
        theta = P - 2 * f
        sel = torch.zeros(theta, T, dtype=torch.int32, device=dev)
        K.bulyan_select(L, slab, L.total, P, f, pair, sel, filled=True)
        K.aggregate_update(L, slab, L.total, K=theta, scale=1.0 / (theta - 2 * f), near_median=f, select=sel, **kw)
    else:
        trim = (P - 1) // 2 if rule == "median" else f
        K.aggregate_update(L, slab, L.total, K=P, scale=1.0 / (P - 2 * trim), trim=trim, **kw)
    torch.cuda.synchronize()
    assert float(pair.abs().sum()) == 0
    sl = slab.cpu().double().numpy()
    for t, spec in enumerate(L.specs):
        cols = slice(spec.offset, spec.offset + spec.numel)
        Y = mix_rows(slab[:, cols], mix[:, t].tolist(), P, f)
        got = gout[cols]
        if rule == "bulyan":
            want = near_median_sum(Y[sel[:, t].long()], f)
            ref = oracle.nnm(sl[:, cols], f, "bulyan")
        else:
            want = trimmed_sum(Y, trim)
            ref = oracle.nnm(sl[:, cols], f, "coordinate_median" if rule == "median" else "trimmed_mean")
        assert torch.equal(got, want), (rule, P, f, t)                 # the same fp32 operations in the same order
        np.testing.assert_allclose(got.cpu().double().numpy(), ref, rtol=1e-5, atol=1e-5)
    valid = torch.from_numpy(L.valid_mask()).to(dev)
    assert float(gout[~valid].abs().sum()) == 0
    p_ref = p0.double() - 0.1 * (gout.double() + 1e-3 * p0.double())
    assert torch.allclose(params.double(), p_ref, atol=1e-5)
    assert flags[0].item() == 2 and cnt[0].item() == 0


@pytest.mark.parametrize("rule", ["trimmed", "bulyan"])
def test_mixed_modes_are_independent_of_buckets_and_grid(K, dev, rule):
    L = ArenaLayout.from_model(build_model("ResNet18"), bf16=True, channels_last=True)
    T, P, f = L.ntensors, 11, 2
    slab = fill_valid(L, P, dev, seed=3, scale=0.01).contiguous()
    pair = torch.zeros(T, P * (P - 1) // 2, dtype=torch.float64, device=dev)
    mix = torch.zeros(P, T, dtype=torch.int32, device=dev)
    K.nnm_mix(L, slab, L.total, P, f, pair, mix, mixed_out=rule == "bulyan")
    if rule == "bulyan":
        theta = P - 2 * f
        sel = torch.zeros(theta, T, dtype=torch.int32, device=dev)
        K.bulyan_select(L, slab, L.total, P, f, pair, sel, filled=True)
        rk = dict(K=theta, scale=1.0 / (theta - 2 * f), near_median=f, select=sel)
    else:
        rk = dict(K=P, scale=1.0 / (P - 2 * f), trim=f)
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
            kw = dict(params=params, momentum=mom, hp=hp, step_ptr=step, done_counter=cnt[0:1], mix=mix, mix_f=f, **rk)
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


def test_nnm_launchers_reject_bad_arguments(K, dev):
    L = lenet_layout()
    T = L.ntensors
    slab = fill_valid(L, 17, dev)
    pair = torch.zeros(T, 136, dtype=torch.float64, device=dev)
    lib = N.cuda()
    for P, f in ((7, 7), (7, -1), (17, 0)):
        with pytest.raises(ValueError):
            K.nnm_mix(L, slab, L.total, P, f, pair, torch.zeros(min(P, 16), T, dtype=torch.int32, device=dev), mixed_out=True)
        a = N.NnmMixArgs(pair.data_ptr(), T, P, f, 1, 1)                  # the C entry point refuses them itself
        assert lib.drc_nnm_mix(C.byref(a), K._stream()) == 1
    assert lib.drc_nnm_mix(C.byref(N.NnmMixArgs(pair.data_ptr(), T, 7, 1, None, 1)), K._stream()) == 1     # no masks
    mix = torch.zeros(7, T, dtype=torch.int32, device=dev)
    w = torch.zeros(T, 7, device=dev)
    sel = torch.zeros(6, T, dtype=torch.int32, device=dev)
    with pytest.raises(ValueError):
        K.nnm_fold(L, 7, 1, mix, w, select=sel, m=6, w_mix=w)             # both choices
    with pytest.raises(ValueError):
        K.nnm_fold(L, 7, 1, mix, w)                                       # neither
    with pytest.raises(ValueError):
        K.nnm_fold(L, 7, 1, mix, w, select=sel, m=5)                      # table of the wrong height
    for fa in (N.NnmFoldArgs(mix.data_ptr(), T, 7, 7, sel.data_ptr(), 1, None, w.data_ptr()),
               N.NnmFoldArgs(mix.data_ptr(), T, 7, 1, sel.data_ptr(), 0, None, w.data_ptr()),
               N.NnmFoldArgs(mix.data_ptr(), T, 7, 1, None, 1, None, w.data_ptr()),
               N.NnmFoldArgs(None, T, 7, 1, sel.data_ptr(), 1, None, w.data_ptr())):
        assert lib.drc_nnm_fold(C.byref(fa), K._stream()) == 1
    hp = hyperparams_tensor(JobConfig(), dev)
    params, moms = torch.zeros(L.total, device=dev), torch.zeros(L.total, device=dev)
    step, cnt, _ = ctrl(dev)
    kw = dict(params=params, momentum=moms, hp=hp, step_ptr=step, done_counter=cnt[0:1])
    with pytest.raises(ValueError):                                       # mixing needs a robust coordinate rule
        K.aggregate_update(L, slab, L.total, K=7, scale=1.0 / 7, mix=mix, mix_f=1, **kw)
    with pytest.raises(ValueError):                                       # f out of range
        K.aggregate_update(L, slab, L.total, K=7, scale=1.0 / 5, trim=1, mix=mix, mix_f=7, **kw)
    with pytest.raises(ValueError):                                       # mode 3 runs on all P mixed rows
        K.aggregate_update(L, slab, L.total, K=5, scale=1.0 / 3, trim=1, mix=mix, mix_f=1, **kw)
    with pytest.raises(ValueError):                                       # ... and takes no select table
        K.aggregate_update(L, slab, L.total, K=7, scale=1.0 / 5, trim=1, select=torch.zeros(7, T, dtype=torch.int32,
                                                                                                  device=dev), mix=mix, mix_f=1, **kw)
    with pytest.raises(ValueError):                                       # masks of 17 rows
        K.aggregate_update(L, slab, L.total, K=17, scale=1.0 / 15, trim=1, mix=torch.zeros(17, T, dtype=torch.int32, device=dev),
                           mix_f=1, **kw)
    table = torch.zeros(16, T, dtype=torch.int32, device=dev)
    for mode, Kr, mixP, scale, select in ((3, 17, 17, 0.1, None), (3, 7, 7, 0.0, None), (3, 5, 7, 0.2, None),
                                         (3, 7, 7, 0.2, table), (4, 5, 7, 0.2, None), (4, 9, 7, 0.2, table)):
        a = N.UpdateArgs()
        a.mode, a.K, a.trim, a.scale, a.select = mode, Kr, 1, 1.0, None if select is None else select.data_ptr()
        a.mix, a.mixP, a.mix_scale = mix.data_ptr(), mixP, scale
        assert lib.drc_aggregate_update(C.byref(a), 1, K._stream()) == 1, (mode, Kr, mixP, scale)


# ------------------------------------------------------------------------------------------------ engine
def _cfg(**kw):
    base = dict(network="LeNet", dataset="MNIST", batch_size=16, max_steps=12, num_workers=7, transport="nvl", lr=0.02,
                momentum=0.9, synthetic_size=512, eval_freq=10 ** 6, compress_grad="None", dtype="fp32", cuda_graphs=False,
                approach="nnm", mode="multi_krum", worker_fail=1)
    base.update(kw)
    return JobConfig(**base)


def _run(cfg, steps):
    t = Trainer(cfg, rank=0, world=1, device=torch.device("cuda", 0), quiet=True)
    losses = [t.train_step()["loss"] for _ in range(steps)]
    t.synchronize()
    return t, losses


@pytest.mark.parametrize("mode", NNM_MODES)
def test_fused_nnm_matches_library_op_engine(monkeypatch, mode):
    """pair_dist + nnm_mix + (select) + (fold) + update against the torch-op PS, in true fp32."""
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    kw = dict(mode=mode, err_mode="constant")
    a, _ = _run(_cfg(**kw), 4)
    b, _ = _run(_cfg(transport="nccl", **kw), 4)
    assert not a.engine.pipeline_ps and a.engine.ps.rule.startswith("nnm_")
    pa, pb = a.engine.master_params(), b.engine.master_params()
    assert torch.isfinite(pa).all()
    assert torch.allclose(pa, pb, atol=2e-5), float((pa - pb).abs().max())


_RESNET = dict(network="ResNet18", dataset="Cifar10", batch_size=8, dtype="bf16", synthetic_size=256, err_mode="rev_grad")


@pytest.mark.parametrize("mode", ["multi_krum", "bulyan"])
def test_nnm_graph_replay_equals_eager(mode):
    e, le = _run(_cfg(cuda_graphs=False, mode=mode, **_RESNET), 6)
    g, lg = _run(_cfg(cuda_graphs=True, mode=mode, **_RESNET), 6)
    assert g.engine.graph is not None and not g.engine.pipeline_ps
    assert torch.equal(e.engine.master_params(), g.engine.master_params())
    assert le == lg


@pytest.mark.parametrize("mode,rule", [("alie", "coordinate_median"), ("minmax", "geometric_median")])
def test_nnm_under_ps_attacks_in_the_captured_step(mode, rule):
    kw = dict(_RESNET, err_mode=mode, mode=rule)
    e, le = _run(_cfg(cuda_graphs=False, **kw), 5)
    g, lg = _run(_cfg(cuda_graphs=True, **kw), 5)
    eng = g.engine
    assert eng.graph is not None and eng.ps.attack == A.attack_code(mode) and eng.ps.rule.startswith("nnm_")
    assert torch.equal(e.engine.master_params(), eng.master_params())
    assert le == lg and all(np.isfinite(lg))
