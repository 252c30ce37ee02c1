"""Centered clipping on the GPU: ``centered_clip_dist`` + ``centered_clip_weights`` (csrc/cuda/clip.cu) against the oracle, the
mode-5 update (csrc/cuda/aggregate_update.cu) bit for bit against an fp32 torch restatement, grid and bucket invariance, the
argument checks, and whole jobs on the fused engine."""
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
from draco_b200.parallel.ps import _fma_f32, hyperparams_tensor
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


def resnet_layout():
    return ArenaLayout.from_model(build_model("ResNet18"), bf16=True, channels_last=True)


def fill_valid(L, rows, dev, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(rows, L.total, generator=g) * scale
    x[:, ~torch.from_numpy(L.valid_mask())] = 0
    return x.to(dev)


def slot_table(L, rows, slots, dev, seed):
    g = torch.Generator().manual_seed(seed)
    cols = [torch.randperm(slots, generator=g)[:rows] for _ in range(L.ntensors)]
    return torch.stack(cols, 1).to(torch.int32).contiguous().to(dev)


def ctrl(dev):
    return (torch.ones(1, dtype=torch.int64, device=dev), torch.zeros(4, dtype=torch.int32, device=dev),
            torch.zeros(8, dtype=torch.int64, device=dev))


def slab_with_outliers(L, S, dev, seed, center):
    """S slots around ``center`` at spreads that straddle tau, with slot 1 = the centre, and (for S >= 5) slot 2 holding a NaN,
    slot 3 a +Inf / -Inf and slot 4 a 1e30 in every tensor."""
    g = torch.Generator().manual_seed(seed)
    scale = 10.0 ** (torch.rand(S, 1, generator=g) * 4 - 3)
    x = center[None].cpu() + torch.randn(S, L.total, generator=g) * scale
    x[:, ~torch.from_numpy(L.valid_mask())] = 0
    if S > 1:
        x[1] = center.cpu()
    for s, val in ((2, NAN), (3, INF if seed % 2 else -INF), (4, 1e30)):
        if s < S:
            for spec in L.specs:
                x[s, spec.offset + (seed + s) % spec.numel] = val
    return x.contiguous().to(dev)


def ulp_diff(a, b):
    ai, bi = a.view(torch.int32).long(), b.view(torch.int32).long()
    return (ai - bi).abs()


def run_dist_weights(K, L, slab, n, center, tau, rows=None, grid=None):
    partials = torch.full((L.ntiles, n), NAN, dtype=torch.float64, device=slab.device)
    weights = torch.full((L.ntensors, n), NAN, dtype=torch.float32, device=slab.device)
    K.centered_clip_dist(L, slab, L.total, n, center, partials, rows=rows, grid=grid)
    K.centered_clip_weights(L, n, tau, partials, weights)
    torch.cuda.synchronize()
    return weights


def weights_ref(L, slab, n, center, tau, rows=None):
    """The oracle's weights per tensor, from fp64 distances formed on the device."""
    out = torch.zeros(L.ntensors, n, dtype=torch.float32)
    for t, spec in enumerate(L.specs):
        cols = slice(spec.offset, spec.offset + spec.numel)
        sel = rows[:, t].long() if rows is not None else torch.arange(n, device=slab.device)
        d = (slab[sel, cols].double() - center[cols].double()).pow(2).sum(1).tolist()
        out[t] = torch.tensor([oracle.centered_clip_weight(di, tau, n) for di in d])
    return out


# ------------------------------------------------------------------------------------------------ dist + weights
@pytest.mark.parametrize("with_rows", [False, True])
def test_weights_match_the_oracle_for_every_row_count(K, dev, with_rows):
    L = lenet_layout()
    center = fill_valid(L, 1, dev, seed=1, scale=0.1)[0]
    for n in range(1, 17):
        S = n + 3 if with_rows else n
        slab = slab_with_outliers(L, S, dev, seed=n, center=center)
        rows = slot_table(L, n, S, dev, seed=n) if with_rows else None
        for tau in (1e-3, 0.5, 1e6):
            got = run_dist_weights(K, L, slab, n, center, tau, rows)
            sl, c = slab.cpu().numpy(), center.cpu().numpy()
            want = torch.zeros_like(got.cpu())
            for t, spec in enumerate(L.specs):
                cols = slice(spec.offset, spec.offset + spec.numel)
                sel = rows[:, t].cpu().numpy() if with_rows else np.arange(n)
                want[t] = torch.from_numpy(oracle.centered_clip_weights(sl[sel, cols], c[cols], tau))
            assert int(ulp_diff(got.cpu(), want).max()) <= 1, (n, tau)
            assert torch.equal(got.cpu() == 0, want == 0), (n, tau)


@pytest.mark.parametrize("n", [1, 7, 15, 16])
def test_weights_on_the_resnet18_arena(K, dev, n):
    """Single-tile tensors (the BatchNorm vectors) and multi-thousand-tile ones (the 512-channel convolutions)."""
    L = resnet_layout()
    tiles = [(s.numel + 1023) // 1024 for s in L.specs]
    assert min(tiles) == 1 and max(tiles) >= 2000
    center = fill_valid(L, 1, dev, seed=2, scale=1e-3)[0]
    slab = slab_with_outliers(L, n + 2, dev, seed=n, center=center)
    rows = slot_table(L, n, n + 2, dev, seed=n)
    for r in (None, rows):
        got = run_dist_weights(K, L, slab, n, center, 0.05, r)
        want = weights_ref(L, slab, n, center, 0.05, r)
        assert int(ulp_diff(got.cpu(), want).max()) <= 1
        assert torch.equal(got.cpu() == 0, want == 0)


# ------------------------------------------------------------------------------------------------ mode 5
def cc_restatement(X, v, w):
    """fp32 torch restatement of mode 5 on one tensor: X [K, d], v [d], w [K] (the kernel's weights)."""
    acc = torch.zeros_like(v)
    for k in range(X.shape[0]):
        if float(w[k]) != 0.0:
            acc = _fma_f32(float(w[k]), X[k] - v, acc)
    return v + acc


@pytest.mark.parametrize("with_rows", [False, True])
@pytest.mark.parametrize("n", [1, 5, 16])
def test_update_matches_the_torch_restatement_bit_for_bit(K, dev, n, with_rows):
    L = lenet_layout()
    hp = hyperparams_tensor(JobConfig(lr=0.1, momentum=0.9, weight_decay=1e-3), dev)
    v0 = fill_valid(L, 1, dev, seed=3, scale=0.1)[0]
    S = n + 2 if with_rows else n
    slab = slab_with_outliers(L, S, dev, seed=10 + n, center=v0)
    rows = slot_table(L, n, S, dev, seed=n) if with_rows else None
    center = v0.clone()
    w = run_dist_weights(K, L, slab, n, center, 0.3, rows)
    params = fill_valid(L, 1, dev, seed=5)[0]
    p0 = params.clone()
    mom = torch.zeros_like(params)
    gout = torch.full((L.total,), 7.0, device=dev)
    step, cnt, flags = ctrl(dev)
    K.centered_clip_update(L, slab, L.total, center=center, weights=w, K=n, select=rows, params=params, momentum=mom, hp=hp,
                           step_ptr=step, done_counter=cnt[0:1], grad_out=gout, flags=[flags[0:1]])
    torch.cuda.synchronize()
    for t, spec in enumerate(L.specs):
        cols = slice(spec.offset, spec.offset + spec.numel)
        sel = rows[:, t].long() if with_rows else torch.arange(n, device=dev)
        want = cc_restatement(slab[sel, cols], v0[cols], w[t])
        assert torch.equal(gout[cols], want), t
        assert torch.isfinite(want).all()
        np_want = oracle.centered_clip(slab[sel, cols].cpu().numpy(), v0[cols].cpu().numpy(), 0.3, weights=w[t].cpu().numpy())
        assert np.array_equal(want.cpu().numpy().view(np.int32), np_want.view(np.int32))
    mask = torch.from_numpy(L.valid_mask()).to(dev)
    assert torch.equal(center[mask], gout[mask])
    p_ref = p0.double() - 0.1 * (gout.double() + 1e-3 * p0.double())
    assert torch.allclose(params.double(), p_ref, atol=1e-5)
    assert flags[0].item() == 2 and cnt[0].item() == 0


def test_weights_centre_and_params_do_not_depend_on_grid_or_buckets(K, dev):
    L = resnet_layout()
    n = 9
    slab = slab_with_outliers(L, 11, dev, seed=4, center=torch.zeros(L.total, device=dev))
    rows = slot_table(L, n, 11, dev, seed=5)
    hp = hyperparams_tensor(JobConfig(lr=0.1, momentum=0.9), dev)
    p0 = fill_valid(L, 1, dev, seed=5)[0]
    nt = L.ntiles
    starts = [s.offset // 1024 for s in L.specs]
    cut = [0, 3, L.ntensors // 2, L.ntensors - 1, L.ntensors]        # buckets of whole tensors
    buckets = [((starts[a], starts[b] if b < L.ntensors else nt), (a, b)) for a, b in zip(cut, cut[1:])]
    results = []
    for how in ("one", "buckets", "grid1", "grid37"):
        params, mom, center = p0.clone(), torch.zeros_like(p0), torch.zeros_like(p0)
        partials = torch.zeros(nt, n, dtype=torch.float64, device=dev)
        weights = torch.zeros(L.ntensors, n, dtype=torch.float32, device=dev)
        step, cnt, flags = ctrl(dev)
        for it in (1, 2):
            step.fill_(it)
            kw = dict(center=center, weights=weights, K=n, select=rows, params=params, momentum=mom, hp=hp, step_ptr=step,
                      done_counter=cnt[0:1])
            if how == "buckets":
                for i, (tiles, tensors) in enumerate(buckets):
                    K.centered_clip_dist(L, slab, L.total, n, center, partials, rows=rows, tile_range=tiles)
                    K.centered_clip_weights(L, n, 0.01, partials, weights, tensor_range=tensors)
                    K.centered_clip_update(L, slab, L.total, tile_range=tiles,
                                           flags=[flags[0:1]] if i == len(buckets) - 1 else [], **kw)
            else:
                grid = {"one": None, "grid1": 1, "grid37": 37}[how]
                K.centered_clip_dist(L, slab, L.total, n, center, partials, rows=rows, grid=grid)
                K.centered_clip_weights(L, n, 0.01, partials, weights)
                K.centered_clip_update(L, slab, L.total, grid=grid, flags=[flags[0:1]], **kw)
        torch.cuda.synchronize()
        assert flags[0].item() == 3
        results.append((weights, center, params))
    for r in results[1:]:
        for a, b in zip(r, results[0]):
            assert torch.equal(a, b)
    assert torch.isfinite(results[0][2]).all() and float(results[0][1].abs().sum()) > 0


def test_launchers_and_c_entries_reject_bad_arguments(K, dev):
    L = lenet_layout()
    T, nt = L.ntensors, L.ntiles
    slab = fill_valid(L, 17, dev)
    center = torch.zeros(L.total, device=dev)
    part = lambda n: torch.zeros(nt, n, dtype=torch.float64, device=dev)       # noqa: E731
    wts = lambda n: torch.zeros(T, n, dtype=torch.float32, device=dev)         # noqa: E731
    for n in (0, 17):
        with pytest.raises(ValueError):
            K.centered_clip_dist(L, slab, L.total, n, center, part(max(n, 1)))
        with pytest.raises(ValueError):
            K.centered_clip_weights(L, n, 1.0, part(max(n, 1)), wts(max(n, 1)))
    with pytest.raises(ValueError):
        K.centered_clip_dist(L, slab, L.total, 4, center, part(5))                          # partials shape
    with pytest.raises(ValueError):
        K.centered_clip_dist(L, slab, L.total, 4, center[:-4], part(4))                     # centre size
    with pytest.raises(ValueError):
        K.centered_clip_dist(L, slab, L.total, 4, center, part(4).float())                  # partials dtype
    with pytest.raises(ValueError):
        K.centered_clip_dist(L, slab, L.total, 4, center, part(4), rows=torch.zeros(3, T, dtype=torch.int32, device=dev))
    for tau in (0.0, -1.0, INF, NAN):
        with pytest.raises(ValueError):
            K.centered_clip_weights(L, 4, tau, part(4), wts(4))
    with pytest.raises(ValueError):
        K.centered_clip_weights(L, 4, 1.0, part(4), wts(5))
    hp = hyperparams_tensor(JobConfig(), dev)
    params, mom = torch.zeros(L.total, device=dev), torch.zeros(L.total, device=dev)
    step, cnt, _ = ctrl(dev)
    kw = dict(params=params, momentum=mom, hp=hp, step_ptr=step, done_counter=cnt[0:1])
    for n, w, c in ((17, wts(16), center), (4, wts(5), center), (4, wts(4), center[:-4])):
        with pytest.raises(ValueError):
            K.centered_clip_update(L, slab, L.total, center=c, weights=w, K=n, **kw)
    with pytest.raises(ValueError):
        K.centered_clip_update(L, slab, L.total, center=center, weights=wts(4), K=4,
                               select=torch.zeros(4, T + 1, dtype=torch.int32, device=dev), **kw)
    # the C entry points refuse them themselves
    lib = N.cuda()
    for n, has_center, has_w, has_part in ((0, 1, 1, 1), (17, 1, 1, 1), (4, 0, 1, 1), (4, 1, 1, 0)):
        a = N.CcArgs()
        a.n, a.tau, a.tv = n, 1.0, L.tile_view(dev)
        a.center = center.data_ptr() if has_center else None
        a.partials = part(4).data_ptr() if has_part else None
        a.weights = wts(4).data_ptr() if has_w else None
        assert lib.drc_cc_dist(C.byref(a), 1, K._stream()) == 1
    keep = (part(4), wts(4))
    for n, tau, t0, t1 in ((4, 0.0, 0, 0), (4, INF, 0, 0), (4, NAN, 0, 0), (17, 1.0, 0, 0), (4, 1.0, 3, 2), (4, 1.0, 0, T + 1)):
        a = N.CcArgs()
        a.n, a.tau, a.tv, a.t_begin, a.t_end = n, tau, L.tile_view(dev), t0, t1
        a.partials, a.weights = keep[0].data_ptr(), keep[1].data_ptr()
        assert lib.drc_cc_weights(C.byref(a), K._stream()) == 1, (n, tau, t0, t1)
    for n, has_w, has_c in ((0, 1, 1), (17, 1, 1), (4, 0, 1), (4, 1, 0)):
        a = N.UpdateArgs()
        a.mode, a.K = 5, n
        a.recomb = keep[1].data_ptr() if has_w else None
        a.center = center.data_ptr() if has_c else None
        assert lib.drc_aggregate_update(C.byref(a), 1, K._stream()) == 1
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------ engine
def _cfg(**kw):
    base = dict(network="LeNet", dataset="MNIST", batch_size=16, max_steps=12, num_workers=7, transport="nvl", lr=0.02,
                momentum=0.9, synthetic_size=512, eval_freq=10 ** 6, compress_grad="None", dtype="fp32", cuda_graphs=False,
                approach="baseline", mode="centered_clip", clip_tau=0.05, worker_fail=2, err_mode="rev_grad")
    base.update(kw)
    return JobConfig(**base)


def _run(cfg, steps):
    t = Trainer(cfg, rank=0, world=1, device=torch.device("cuda", 0), quiet=True)
    losses = [t.train_step()["loss"] for _ in range(steps)]
    t.synchronize()
    return t, losses


@pytest.mark.parametrize("rule", [dict(), dict(approach="detox", num_workers=9, group_size=3),
                                  dict(worker_momentum=0.9, momentum=0.0, lr=0.1), dict(optimizer="adam", lr=1e-3)])
def test_fused_matches_library_op_engine(monkeypatch, rule):
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    a, _ = _run(_cfg(**rule), 4)
    b, _ = _run(_cfg(transport="nccl", **rule), 4)
    assert a.engine.pipeline_ps and a.engine.ps.rule == ("detox_centered_clip" if "approach" in rule else "centered_clip")
    pa, pb = a.engine.master_params(), b.engine.master_params()
    assert torch.isfinite(pa).all()
    assert torch.allclose(pa, pb, atol=2e-5), float((pa - pb).abs().max())
    ca, cb = a.engine.ps.cc_center, b.engine.ps.cc_center
    assert float(ca.abs().sum()) > 0 and torch.allclose(ca, cb, atol=1e-4), float((ca - cb).abs().max())


_RESNET = dict(network="ResNet18", dataset="Cifar10", batch_size=8, dtype="bf16", synthetic_size=256, num_workers=7)


@pytest.mark.parametrize("kw", [dict(err_mode="rev_grad"), dict(err_mode="alie"), dict(err_mode="minmax"),
                                dict(approach="detox", group_size=3, err_mode="rev_grad", num_workers=9),
                                dict(err_mode="alie", worker_momentum=0.9, momentum=0.0)])
def test_graph_replay_equals_eager(kw):
    e, le = _run(_cfg(cuda_graphs=False, **dict(_RESNET, **kw)), 5)
    g, lg = _run(_cfg(cuda_graphs=True, **dict(_RESNET, **kw)), 5)
    eng = g.engine
    assert eng.graph is not None and eng.pipeline_ps
    if kw["err_mode"] != "rev_grad":
        assert eng.ps.attack == A.attack_code(kw["err_mode"])
    assert torch.equal(e.engine.master_params(), eng.master_params())
    assert torch.equal(e.engine.ps.cc_center, eng.ps.cc_center)
    assert le == lg and all(np.isfinite(lg))


def test_debug_checksum_and_compression_compose():
    a, la = _run(_cfg(debug_checksum=True), 3)
    b, lb = _run(_cfg(compress_grad="compress"), 3)
    c, lc = _run(_cfg(), 3)
    assert not b.engine.pipeline_ps and c.engine.pipeline_ps
    assert torch.equal(a.engine.master_params(), c.engine.master_params())
    assert torch.equal(b.engine.master_params(), c.engine.master_params())
    assert la == lb == lc


def test_resume_is_bit_for_bit(tmp_path):
    d = str(tmp_path) + "/"
    kw = dict(train_dir=d, max_steps=6)
    t = Trainer(_cfg(eval_freq=3, **kw), rank=0, world=1, device=torch.device("cuda", 0), quiet=True)
    t.fit(6)
    t.synchronize()
    final, center = t.engine.master_params().clone(), t.engine.ps.cc_center.clone()
    t.close()
    t2 = Trainer(_cfg(eval_freq=10 ** 6, checkpoint_step=3, **kw), rank=0, world=1, device=torch.device("cuda", 0), quiet=True)
    for _ in range(3):
        t2.train_step()
    t2.synchronize()
    assert torch.equal(t2.engine.master_params(), final)
    assert torch.equal(t2.engine.ps.cc_center, center)


def test_centered_clip_trains_under_attack_where_the_mean_does_not():
    def dist(a, b):
        d = (a - b).abs().max()
        return float(d) if torch.isfinite(d) else float("inf")
    kw = dict(lr=0.05)
    clean, _ = _run(_cfg(mode="normal", clip_tau=None, err_mode="none", **kw), 10)
    ref = clean.engine.master_params()
    mean, _ = _run(_cfg(mode="normal", clip_tau=None, err_mode="rev_grad", **kw), 10)
    d_mean = dist(mean.engine.master_params(), ref)
    assert d_mean > 1e-1, d_mean
    t, losses = _run(_cfg(err_mode="rev_grad", **kw), 10)
    assert losses[-1] < losses[0], losses
    p = t.engine.master_params()
    assert torch.isfinite(p).all()
    assert dist(p, ref) < 0.1 * d_mean, (dist(p, ref), d_mean)
