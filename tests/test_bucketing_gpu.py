"""Worker buckets (``--bucketing s``) on the GPU: ``wbucket_plan_kernel`` (csrc/cuda/bucketing.cu) against the host buckets,
update mode 7 (csrc/cuda/aggregate_update.cu) bit for bit against the fp32 library-op PS with NaN / +-Inf rows, s = 1 against
plain mode 3, gradient-bucket and grid independence, graph replay against eager, nvl against nccl, and a heterogeneous job."""
import numpy as np
import pytest
import torch

from draco_b200 import JobConfig
from draco_b200.codes.bucketing import bucket_schedule, wbucket_masks
from draco_b200.models import build_model
from draco_b200.parallel.arena import ArenaLayout
from draco_b200.parallel.ps import TorchPS, hyperparams_tensor
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


def fill_valid(L, rows, dev, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(rows, L.total, generator=g) * torch.rand(rows, 1, generator=g).add(0.2)
    x[:, ~torch.from_numpy(L.valid_mask())] = 0
    return x.to(dev)


def _plan(K, dev, P, s):
    sched = torch.from_numpy(bucket_schedule(P, 9, 4)).to(dev)
    nb = -(-P // s)
    masks = torch.zeros(nb, dtype=torch.int32, device=dev)
    scales = torch.zeros(nb, dtype=torch.float32, device=dev)
    return sched, masks, scales


def _cases():
    out = []
    for P in range(3, 17):
        for s in range(1, P + 1):
            nb = -(-P // s)
            for f in (0, 1, 2):
                if nb > 2 * f:
                    out.append((P, s, f))
    return out


@pytest.mark.parametrize("P", range(3, 17))
def test_plan_kernel_writes_the_host_buckets(K, dev, P):
    for s in range(1, P + 1):
        sched, masks, scales = _plan(K, dev, P, s)
        for step in (1, 2, 9, 10, 23):
            st = torch.tensor([step], dtype=torch.int64, device=dev)
            K.wbucket_plan(sched, s, step_ptr=st, masks=masks, scales=scales)
            want = wbucket_masks(sched[step % sched.shape[0]].tolist(), s)
            assert masks.cpu().numpy().view(np.uint32).tolist() == want.tolist()
            cnt = [bin(int(m)).count("1") for m in want]
            assert scales.cpu().tolist() == [float(np.float32(1.0 / c)) for c in cnt]


def _same_bits(a, b):
    """Equal bit for bit, except that any NaN equals any NaN (the payload is not part of the result)."""
    na, nb = a.isnan(), b.isnan()
    return torch.equal(na, nb) and torch.equal(a[~na].view(torch.int32), b[~nb].view(torch.int32))


def _update(K, dev, L, slab, masks, scales, trim, tile_ranges=None, grid=None):
    hp = hyperparams_tensor(JobConfig(lr=0.1, momentum=0.9, weight_decay=1e-3), dev)
    params = fill_valid(L, 1, dev, seed=5)[0]
    mom = torch.zeros_like(params)
    gout = torch.full((L.total,), 7.0, device=dev)
    step = torch.ones(1, dtype=torch.int64, device=dev)
    cnt = torch.zeros(4, dtype=torch.int32, device=dev)
    for tr in tile_ranges or [None]:
        K.wbucket_update(L, slab, L.total, masks=masks, scales=scales, trim=trim, params=params, momentum=mom, hp=hp, step_ptr=step,
                         done_counter=cnt[0:1], grad_out=gout, tile_range=tr, grid=grid)
    torch.cuda.synchronize()
    return gout, params


@pytest.mark.parametrize("P,s,f", _cases())
def test_mode7_equals_the_library_op_ps_bit_for_bit(K, dev, P, s, f):
    """Median and trimmed mean of the bucket rows, with a liar, a NaN row and a +-Inf row."""
    L = lenet_layout()
    slab = fill_valid(L, P, dev, seed=P * 31 + s)
    slab[0] = -30 * slab[0]
    slab[P - 1, ::3] = NAN
    slab[P // 2, ::5] = INF
    slab[P // 2, 1::5] = -INF
    slab = slab.contiguous()
    for mode in ("coordinate_median", "trimmed_mean"):
        cfg = JobConfig(approach="baseline", mode=mode, num_workers=P, worker_fail=f, bucketing=s, transport="nccl", max_steps=9,
                        seed=4).resolve(1)
        ps = TorchPS(cfg, L, dev, L.new_arena(dev), None, None)
        sched, masks, scales = _plan(K, dev, P, s)
        K.wbucket_plan(sched, s, step_ptr=torch.tensor([5], dtype=torch.int64, device=dev), masks=masks, scales=scales)
        want = ps.aggregate(slab, step=5)
        gout, _ = _update(K, dev, L, slab, masks, scales, ps.plan.trim)
        for t, spec in enumerate(L.specs):
            got = gout[spec.offset: spec.offset + spec.numel]
            assert _same_bits(got, want[t]), (mode, t)


@pytest.mark.parametrize("P,f", [(5, 1), (9, 2), (16, 3)])
def test_s_equal_one_is_plain_mode3(K, dev, P, f):
    L = lenet_layout()
    slab = fill_valid(L, P, dev, seed=P)
    slab[1, ::7] = NAN
    for trim in ((P - 1) // 2, f):
        sched, masks, scales = _plan(K, dev, P, 1)
        K.wbucket_plan(sched, 1, step_ptr=torch.tensor([3], dtype=torch.int64, device=dev), masks=masks, scales=scales)
        a, pa = _update(K, dev, L, slab, masks, scales, trim)
        hp = hyperparams_tensor(JobConfig(lr=0.1, momentum=0.9, weight_decay=1e-3), dev)
        params = fill_valid(L, 1, dev, seed=5)[0]
        b = torch.full((L.total,), 7.0, device=dev)
        K.aggregate_update(L, slab, L.total, K=P, scale=1.0 / (P - 2 * trim), trim=trim, params=params, momentum=torch.zeros_like(params),
                           hp=hp, step_ptr=torch.ones(1, dtype=torch.int64, device=dev),
                           done_counter=torch.zeros(4, dtype=torch.int32, device=dev)[0:1], grad_out=b)
        torch.cuda.synchronize()
        assert torch.equal(a, b) and torch.equal(pa, params)


def test_result_does_not_depend_on_gradient_buckets_or_grid(K, dev):
    L = lenet_layout()
    P, s = 13, 3
    slab = fill_valid(L, P, dev, seed=1)
    sched, masks, scales = _plan(K, dev, P, s)
    K.wbucket_plan(sched, s, step_ptr=torch.tensor([2], dtype=torch.int64, device=dev), masks=masks, scales=scales)
    ref, pref = _update(K, dev, L, slab, masks, scales, 1)
    nt = L.ntiles
    bounds = [0, nt // 5, nt // 5 + 1, (2 * nt) // 3, nt]
    for tr, grid in (([(bounds[i], bounds[i + 1]) for i in range(4)], None), (None, 1), (None, 3), (None, 1000)):
        g, p = _update(K, dev, L, slab, masks, scales, 1, tile_ranges=tr, grid=grid)
        assert torch.equal(g, ref) and torch.equal(p, pref)


def test_argument_checks(K, dev):
    L = lenet_layout()
    sched = torch.from_numpy(bucket_schedule(17, 3, 1)).to(dev)
    m, sc = torch.zeros(9, dtype=torch.int32, device=dev), torch.zeros(9, device=dev)
    with pytest.raises(ValueError):
        K.wbucket_plan(sched, 2, step_ptr=torch.ones(1, dtype=torch.int64, device=dev), masks=m, scales=sc)
    with pytest.raises(ValueError):
        _update(K, dev, L, fill_valid(L, 4, dev), torch.zeros(4, dtype=torch.int32, device=dev), torch.zeros(4, device=dev), 2)


# ------------------------------------------------------------------------------------------------ engine
def _cfg(**kw):
    base = dict(network="LeNet", dataset="MNIST", batch_size=16, max_steps=12, num_workers=7, transport="nvl", lr=0.02,
                momentum=0.9, synthetic_size=512, eval_freq=10 ** 6, compress_grad="None", dtype="fp32", cuda_graphs=False,
                approach="baseline", mode="coordinate_median", worker_fail=1, bucketing=2, err_mode="constant")
    base.update(kw)
    return JobConfig(**base)


def _run(cfg, steps):
    t = Trainer(cfg, rank=0, world=1, device=torch.device("cuda", 0), quiet=True)
    losses = [t.train_step()["loss"] for _ in range(steps)]
    t.synchronize()
    return t, losses


@pytest.mark.parametrize("mode", ["coordinate_median", "trimmed_mean", "krum", "multi_krum", "geometric_median",
                                  "centered_clip"])
def test_fused_bucketing_matches_the_library_op_engine(monkeypatch, mode):
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    kw = dict(mode=mode, num_workers=9, clip_tau=0.5 if mode == "centered_clip" else None)
    a, _ = _run(_cfg(**kw), 4)
    b, _ = _run(_cfg(transport="nccl", **kw), 4)
    assert a.engine.ps.rule.startswith("wbucket_")
    pa, pb = a.engine.master_params(), b.engine.master_params()
    assert torch.isfinite(pa).all()
    assert torch.allclose(pa, pb, atol=2e-5), float((pa - pb).abs().max())


_RESNET = dict(network="ResNet18", dataset="Cifar10", batch_size=8, dtype="bf16", synthetic_size=256, err_mode="rev_grad")


@pytest.mark.parametrize("err", ["rev_grad", "alie"])
def test_graph_replay_equals_eager_and_follows_each_permutation(err):
    kw = dict(_RESNET, err_mode=err, num_workers=9, bucketing=3, worker_fail=1)
    e, le = _run(_cfg(cuda_graphs=False, **kw), 6)
    g, lg = _run(_cfg(cuda_graphs=True, **kw), 6)
    assert g.engine.graph is not None and g.engine.pipeline_ps
    assert torch.equal(e.engine.master_params(), g.engine.master_params())
    assert le == lg and all(np.isfinite(lg))
    # the replayed graph planned the last step's buckets
    want = wbucket_masks(g.engine.ps.wb_schedule[6 % g.engine.ps.wb_schedule.shape[0]].tolist(), 3)
    assert g.engine.ps.wb_mask.cpu().numpy().view(np.uint32).tolist() == want.tolist()


def test_resnet_nvl_equals_nccl(monkeypatch):
    """The two transports run different convolution kernels (the project's against cuDNN), so the parameters agree to the
    forward / backward pass's rounding, not bit for bit; the bucket rule itself is compared exactly above."""
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    kw = dict(_RESNET, dtype="fp32", num_workers=7, bucketing=2, worker_fail=1)
    a, la = _run(_cfg(**kw), 3)
    b, lb = _run(_cfg(transport="nccl", **kw), 3)
    pa, pb = a.engine.master_params(), b.engine.master_params()
    assert torch.isfinite(pa).all() and np.allclose(la, lb, rtol=1e-2)
    assert torch.allclose(pa, pb, atol=5e-3, rtol=1e-2), float((pa - pb).abs().max())


def test_dirichlet_job_trains_on_the_fused_path():
    t, losses = _run(_cfg(dirichlet_alpha=0.1, num_workers=5, bucketing=2, max_steps=8, synthetic_size=2048, batch_size=16), 6)
    assert t.engine.worker.plan.shards is not None and all(np.isfinite(losses))


# ------------------------------------------------------------------------------------------------ centered clipping over buckets
def _bad_slab(L, P, dev, seed):
    slab = fill_valid(L, P, dev, seed=seed)
    slab[0] = -30 * slab[0]
    slab[P - 1, ::3] = NAN
    slab[P // 2, ::5] = INF
    return slab.contiguous()


def _cc_cases():
    return [(P, s, f) for P, s, f in _cases() if P in (3, 5, 8, 11, 16) and f <= 1]


@pytest.mark.parametrize("P,s,f", _cc_cases())
@pytest.mark.parametrize("scope", ["tensor", "model"])
def test_bucket_centered_clip_equals_the_fp32_definition(K, dev, P, s, f, scope):
    """Bucket cc_dist + the unchanged weights + mode 8 against oracle.centered_clip on oracle.wbucket_rows: the weights to
    fp64 rounding of the distance sums, the aggregate and the new centre bit for bit given the weights."""
    from draco_b200.codes import oracle
    from draco_b200.codes.bucketing import wbuckets
    L = lenet_layout()
    T, tau = L.ntensors, 0.3
    slab = _bad_slab(L, P, dev, P * 7 + s)
    sched, masks, scales = _plan(K, dev, P, s)
    K.wbucket_plan(sched, s, step_ptr=torch.tensor([4], dtype=torch.int64, device=dev), masks=masks, scales=scales)
    nb = masks.shape[0]
    center = fill_valid(L, 1, dev, seed=9)[0] * 0.1
    c0 = center.clone()
    partials = torch.zeros(L.ntiles, nb, dtype=torch.float64, device=dev)
    w = torch.zeros(T, nb, dtype=torch.float32, device=dev)
    K.wbucket_cc_dist(L, slab, L.total, masks=masks, scales=scales, center=center, partials=partials)
    if scope == "model":
        K.centered_clip_model_weights(L, nb, tau, partials, torch.zeros(T, nb, dtype=torch.float64, device=dev), w)
    else:
        K.centered_clip_weights(L, nb, tau, partials, w)
    hp = hyperparams_tensor(JobConfig(lr=0.1, momentum=0.9), dev)
    params = fill_valid(L, 1, dev, seed=5)[0]
    gout = torch.zeros(L.total, device=dev)
    K.wbucket_cc_update(L, slab, L.total, masks=masks, scales=scales, center=center, weights=w, params=params,
                        momentum=torch.zeros_like(params), hp=hp, step_ptr=torch.ones(1, dtype=torch.int64, device=dev),
                        done_counter=torch.zeros(4, dtype=torch.int32, device=dev)[0:1], grad_out=gout)
    torch.cuda.synchronize()
    B = wbuckets(sched[4].tolist(), s)
    S, V, W = slab.cpu().numpy(), c0.cpu().numpy(), w.cpu().numpy()
    ds = []
    for t, spec in enumerate(L.specs):
        cols = slice(spec.offset, spec.offset + spec.numel)
        Y = oracle.wbucket_rows(S[:, cols], B)
        with np.errstate(invalid="ignore", over="ignore"):
            ds.append(((Y.astype(np.float64) - V[cols].astype(np.float64)) ** 2).sum(1))
        want = oracle.centered_clip(Y, V[cols], tau, weights=W[t])
        assert _same_bits(gout[cols].cpu(), torch.from_numpy(want)), t
        assert _same_bits(center[cols].cpu(), torch.from_numpy(want)), t
    D = [oracle.model_d2(ds)] * T if scope == "model" else ds
    for t in range(T):
        wt = [oracle.centered_clip_weight(float(d), tau, nb) for d in D[t]]
        np.testing.assert_allclose(W[t], wt, rtol=1e-6, atol=0)


@pytest.mark.parametrize("P", [4, 9, 16])
def test_s_equal_one_centered_clip_is_the_baseline_build(K, dev, P):
    L = lenet_layout()
    T, tau = L.ntensors, 0.5
    slab = fill_valid(L, P, dev, seed=P)
    slab[0] = -30 * slab[0]
    sched, masks, scales = _plan(K, dev, P, 1)
    K.wbucket_plan(sched, 1, step_ptr=torch.tensor([2], dtype=torch.int64, device=dev), masks=masks, scales=scales)
    outs = []
    for wb in (True, False):
        center = fill_valid(L, 1, dev, seed=9)[0] * 0.1
        partials = torch.zeros(L.ntiles, P, dtype=torch.float64, device=dev)
        w = torch.zeros(T, P, dtype=torch.float32, device=dev)
        if wb:
            K.wbucket_cc_dist(L, slab, L.total, masks=masks, scales=scales, center=center, partials=partials)
        else:
            K.centered_clip_dist(L, slab, L.total, P, center, partials)
        K.centered_clip_weights(L, P, tau, partials, w)
        hp = hyperparams_tensor(JobConfig(lr=0.1, momentum=0.9), dev)
        params = fill_valid(L, 1, dev, seed=5)[0]
        kw = dict(center=center, weights=w, params=params, momentum=torch.zeros_like(params), hp=hp,
                  step_ptr=torch.ones(1, dtype=torch.int64, device=dev), done_counter=torch.zeros(4, dtype=torch.int32, device=dev)[0:1])
        if wb:
            K.wbucket_cc_update(L, slab, L.total, masks=masks, scales=scales, **kw)
        else:
            K.centered_clip_update(L, slab, L.total, K=P, **kw)
        torch.cuda.synchronize()
        outs.append((w, center, params))
    for a, b in zip(*outs):
        assert torch.equal(a, b)


# ------------------------------------------------------------------------------------------------ Krum / multi-Krum / geomedian
def _choice(K, dev, L, slab, P, s, rule, f, step=6):
    T = L.ntensors
    sched, masks, scales = _plan(K, dev, P, s)
    K.wbucket_plan(sched, s, step_ptr=torch.tensor([step], dtype=torch.int64, device=dev), masks=masks, scales=scales)
    nb = masks.shape[0]
    raw = torch.zeros(T, P * (P - 1) // 2, dtype=torch.float64, device=dev)
    tab = torch.zeros(T, nb * (nb - 1) // 2, dtype=torch.float64, device=dev)
    K.pair_dist(L, slab, L.total, P, raw)
    K.wbucket_table(L, P, masks=masks, raw_d2=raw, wb_d2=tab)
    tab_copy = tab.clone()
    if rule == "geomedian":
        gw = torch.zeros(T, nb, dtype=torch.float32, device=dev)
        K.geometric_median_weights(L, slab, L.total, nb, tab, gw, filled=True)
        w = torch.zeros(T, P, dtype=torch.float32, device=dev)
        K.wbucket_fold(L, P, masks=masks, weights=w, w_rows=gw)
        sel, wsel = gw, None
    else:
        m = 1 if rule == "krum" else nb - f
        sel = torch.zeros(m, T, dtype=torch.int32, device=dev)
        K.krum_select(L, slab, L.total, nb, f, tab, sel, m=m, filled=True)
        kc = min(m * s, P)
        wsel = torch.zeros(kc, T, dtype=torch.int32, device=dev)
        w = torch.zeros(T, kc, dtype=torch.float32, device=dev)
        K.wbucket_fold(L, P, masks=masks, weights=w, select=sel, m=m, wsel=wsel)
    torch.cuda.synchronize()
    assert float(raw.abs().sum()) == 0 and float(tab.abs().sum()) == 0       # both tables left zeroed for the next step
    return sched[step].tolist(), masks, tab_copy, sel, wsel, w


def _choice_cases():
    out = []
    for P in (5, 8, 11, 16):
        for s in (1, 2, 3):
            nb = -(-P // s)
            for rule, f in (("krum", 1), ("multi_krum", 1), ("geomedian", 1), ("geomedian", 0)):
                if (nb > 2 * f + 2) if rule != "geomedian" else nb >= 2:
                    out.append((P, s, rule, f))
    return out


@pytest.mark.parametrize("P,s,rule,f", _choice_cases())
def test_bucket_table_selection_and_weights_match_the_oracle(K, dev, P, s, rule, f):
    from draco_b200.codes import oracle
    from draco_b200.codes.bucketing import wbuckets
    L = lenet_layout()
    slab = fill_valid(L, P, dev, seed=P * 5 + s)
    slab[0] = -30 * slab[0]
    perm, masks, tab, sel, wsel, w = _choice(K, dev, L, slab, P, s, rule, f)
    B = wbuckets(perm, s)
    nb = len(B)
    S = slab.cpu().numpy()
    for t, spec in enumerate(L.specs):
        # the table against the fp64 definition (pair_dist forms each difference in fp32, so to about 1e-7), then the choice
        # and the weights against the oracle run on the kernel's own table
        Db = oracle.wbucket_pair_d2(oracle._raw_d2(S[:, spec.offset: spec.offset + spec.numel]), B, P)
        iu = [(b, k) for k in range(nb) for b in range(k)]
        got = tab[t].cpu().numpy()
        np.testing.assert_allclose(got, [Db[b, k] for b, k in iu], rtol=1e-6, atol=1e-9)
        Db = np.zeros((nb, nb))
        for q, (b, k) in enumerate(iu):
            Db[b, k] = Db[k, b] = got[q]
        if rule == "geomedian":
            wb = oracle._weiszfeld_weights(Db, 1e-10, 256)
            want = np.zeros(P)
            for b, g in enumerate(B):
                want[g] = wb[b] / len(g)
            np.testing.assert_allclose(w[t].cpu().numpy(), want, rtol=1e-4, atol=1e-6)
        else:
            m = sel.shape[0]
            best = np.argsort(oracle._krum_scores_d2(Db, f), kind="stable")[:m].tolist()
            assert sel[:, t].tolist() == best
            slots = [j for b in best for j in B[b]]
            ws = [np.float32(1.0 / m / len(B[b])) for b in best for _ in B[b]]
            kc = wsel.shape[0]
            assert wsel[:len(slots), t].tolist() == slots[:kc]
            assert w[t, :len(slots)].cpu().tolist() == [float(x) for x in ws[:kc]]
            assert all(float(x) == 0.0 for x in w[t, len(slots):].cpu()) and set(wsel[len(slots):, t].tolist()) <= {slots[0]}


def test_a_nan_row_in_an_unchosen_bucket_leaves_krum_finite(K, dev):
    L = lenet_layout()
    P, s, f = 11, 2, 1
    slab = fill_valid(L, P, dev, seed=3)
    slab[4] = NAN
    perm, masks, tab, sel, wsel, w = _choice(K, dev, L, slab, P, s, "krum", f)
    hp = hyperparams_tensor(JobConfig(lr=0.1, momentum=0.0), dev)
    params = fill_valid(L, 1, dev, seed=5)[0]
    gout = torch.zeros(L.total, device=dev)
    K.aggregate_update(L, slab, L.total, K=wsel.shape[0], scale=1.0, weights=w, select=wsel, params=params,
                       momentum=torch.zeros_like(params), hp=hp, step_ptr=torch.ones(1, dtype=torch.int64, device=dev),
                       done_counter=torch.zeros(4, dtype=torch.int32, device=dev)[0:1], grad_out=gout)
    torch.cuda.synchronize()
    assert 4 not in wsel.flatten().tolist()
    assert torch.isfinite(gout).all() and torch.isfinite(params).all()


@pytest.mark.parametrize("P", [5, 9, 16])
def test_s_equal_one_geometric_median_is_the_baseline_weights(K, dev, P):
    L = lenet_layout()
    T = L.ntensors
    slab = fill_valid(L, P, dev, seed=P + 1)
    slab[0] = -30 * slab[0]
    _, masks, tab, gw, _, w = _choice(K, dev, L, slab, P, 1, "geomedian", 0)
    raw = torch.zeros(T, P * (P - 1) // 2, dtype=torch.float64, device=dev)
    base = torch.zeros(T, P, dtype=torch.float32, device=dev)
    K.geometric_median_weights(L, slab, L.total, P, raw, base)
    torch.cuda.synchronize()
    assert torch.equal(w, base)
