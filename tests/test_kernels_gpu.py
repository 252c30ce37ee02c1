"""sm_90a kernel numerics against plain PyTorch fp32 / numpy fp64 references ("loopback ranks": every peer buffer is a
distinct buffer on the same device, so push / decode+update / broadcast semantics are checked without NVSwitch)."""
import numpy as np
import pytest
import torch

from draco_b200.codes import cyclic, oracle
from draco_b200.codes.repetition import group_assign
from draco_b200.models import build_model
from draco_b200.parallel.arena import ArenaLayout
from draco_b200.parallel.ps import hyperparams_tensor
from draco_b200 import JobConfig

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def K():
    from draco_b200.ops import kernels
    return kernels


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda", 0)


def small_layout(bf16_some=True):
    """LeNet layout (8 tensors, includes tensors that are not multiples of the tile)."""
    m = build_model("LeNet")
    return ArenaLayout.from_model(m, bf16=bf16_some, channels_last=True)


def fill_valid(L, rows, dev, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    mask = torch.from_numpy(L.valid_mask())
    x = torch.randn(rows, L.total, generator=g) * scale
    x[:, ~mask] = 0
    return x.to(dev)


def ctrl(dev, step=1):
    return (torch.full((1,), step, dtype=torch.int64, device=dev), torch.zeros(4, dtype=torch.int32, device=dev),
            torch.zeros(8, dtype=torch.int64, device=dev))


# ------------------------------------------------------------------------------------------------ push / encode
def test_push_identity_mixed_dtypes_and_flag(K, dev):
    L = small_layout()
    g32 = fill_valid(L, 1, dev)[0]
    g16 = g32.to(torch.bfloat16)
    dst = torch.full((L.total,), 7.0, device=dev)
    step, cnt, flags = ctrl(dev, 5)
    K.push_encode(L, [g32], [g16], dst, step_ptr=step, worker=2, done_counter=cnt[0:1], flag=flags[3:4])
    torch.cuda.synchronize()
    expect = g32.clone()
    for s in L.specs:
        if s.is_bf16:
            expect[s.offset:s.offset + s.numel] = g16[s.offset:s.offset + s.numel].float()
    assert torch.equal(dst, expect)
    assert flags[3].item() == 5 and cnt[0].item() == 0


@pytest.mark.parametrize("attack,name", [(1, "rev_grad"), (2, "constant"), (3, "random")])
def test_push_adversary_hook(K, dev, attack, name):
    L = ArenaLayout.from_model(build_model("LeNet"), bf16=False, channels_last=True)
    g32 = fill_valid(L, 1, dev)[0]
    dst = torch.zeros(L.total, device=dev)
    step, cnt, flags = ctrl(dev, 2)
    bitmap = torch.tensor([0, 0, 0b100, 0], dtype=torch.int32, device=dev)      # worker slot 2 lies at step 2
    mask = torch.from_numpy(L.valid_mask()).to(dev)
    for worker, lies in ((2, True), (1, False)):
        dst.zero_()
        K.push_encode(L, [g32], [None], dst, step_ptr=step, worker=worker, done_counter=cnt[0:1], adv_bitmap=bitmap,
                      adv_len=4, attack=attack, magnitude=-100.0)
        torch.cuda.synchronize()
        if not lies:
            assert torch.equal(dst, g32)
        elif name == "rev_grad":
            assert torch.equal(dst, -100.0 * g32)
        elif name == "constant":
            assert torch.equal(dst[mask], torch.full_like(dst[mask], -100.0)) and float(dst[~mask].abs().sum()) == 0
        else:
            v = dst[mask]
            assert float(dst[~mask].abs().sum()) == 0
            assert abs(float(v.mean())) < 1.5 and 85 < float(v.std()) < 115        # ~ 100 * N(0,1)


def test_push_cyclic_encode_matches_oracle(K, dev):
    n, s = 7, 2
    code = cyclic.search_w(n, s)
    L = ArenaLayout.from_model(build_model("LeNet"), bf16=False, channels_last=True)
    G = fill_valid(L, n, dev, seed=3)                      # gradient of every batch
    step, cnt, flags = ctrl(dev, 1)
    for w in (0, 4, 6):
        batches = code.batches_of(w)
        dst = torch.zeros(2 * L.total, device=dev)
        K.push_encode(L, [G[b] for b in batches], [None] * len(batches), dst, step_ptr=step, worker=w,
                      done_counter=cnt[0:1], coef=list(code.coeffs_of(w)))
        torch.cuda.synchronize()
        got = torch.view_as_complex(dst.view(-1, 2)).cpu().numpy()
        ref = cyclic.encode(code, w, G.cpu().double().numpy())
        assert np.abs(got - ref).max() < 1e-5 * max(1.0, np.abs(ref).max())


# ------------------------------------------------------------------------------------------------ vote + update
def _sgd_ref(p, m, g, lr, mu, wd=0.0, first=True):
    d = g + wd * p
    m2 = d.clone() if first else mu * m + d
    return p - lr * m2, m2


def test_vote_and_fused_update_match_oracle(K, dev):
    L = small_layout()
    P = 7
    plan = group_assign(P, 3)
    base = fill_valid(L, plan.num_groups, dev, seed=1, scale=0.1)       # honest gradient of each group
    slots = torch.stack([base[plan.group_of(w)] for w in range(1, P + 1)]).contiguous()
    # liars: worker 2 (group 0) everywhere; worker 5 only in tensor 3; worker 7 NaN in tensor 0
    slots[1] = -100 * slots[1]
    s3, s0 = L.specs[3], L.specs[0]
    slots[4, s3.offset + 5] += 1.0
    slots[6, s0.offset] = float("nan")
    table = torch.from_numpy(plan.as_table()).to(dev)
    G, T = table.shape[0], L.ntensors
    neq = torch.zeros(G, T, dtype=torch.int32, device=dev)
    win_slot = torch.zeros(G, T, dtype=torch.int32, device=dev)
    win_mem = torch.zeros(G, T, dtype=torch.int32, device=dev)
    K.vote(L, slots, L.total, table, neq, win_slot, win_mem)
    torch.cuda.synchronize()
    assert int(neq.abs().sum()) == 0                                    # scratch left clean for the next step
    sl = slots.cpu().double().numpy()
    for t, spec in enumerate(L.specs):
        X = sl[:, spec.offset:spec.offset + spec.numel]
        _, winners = oracle.majority_vote(X, plan.groups)
        assert win_mem[:, t].tolist() == winners, (t, win_mem[:, t].tolist(), winners)

    # fused select-sum + SGD-momentum + broadcast to 3 "peers" + flags
    cfg = JobConfig(lr=0.1, momentum=0.9, weight_decay=1e-3)
    hp = hyperparams_tensor(cfg, dev)
    params = fill_valid(L, 1, dev, seed=9)[0]
    p0 = params.clone()
    mom = torch.zeros_like(params)
    peers = [torch.zeros(L.total, device=dev) for _ in range(3)]
    grad_out = torch.zeros(L.total, device=dev)
    step, cnt, flags = ctrl(dev, 1)
    K.aggregate_update(L, slots, L.total, params=params, momentum=mom, hp=hp, step_ptr=step, done_counter=cnt[0:1],
                       K=G, scale=1.0 / G, select=win_slot, first_step=1, grad_out=grad_out, dst=peers,
                       flags=[flags[0:1], flags[2:3]])
    torch.cuda.synchronize()
    agg = torch.zeros(L.total, dtype=torch.float64)
    for t, spec in enumerate(L.specs):
        X = sl[:, spec.offset:spec.offset + spec.numel]
        a, _ = oracle.majority_vote(X, plan.groups)
        agg[spec.offset:spec.offset + spec.numel] = torch.from_numpy(a)
    ok = ~torch.isnan(agg)
    assert torch.allclose(grad_out.cpu().double()[ok], agg[ok], atol=1e-6)
    p_ref, m_ref = _sgd_ref(p0.cpu().double(), 0, agg, 0.1, 0.9, 1e-3, first=True)
    assert torch.allclose(params.cpu().double()[ok], p_ref[ok], atol=1e-5)
    assert torch.allclose(mom.cpu().double()[ok], m_ref[ok], atol=1e-5)
    for q in peers:
        assert torch.equal(q, params)                                   # broadcast is bit-exact
    assert flags[0].item() == 2 and flags[2].item() == 2 and flags[1].item() == 0

    # second step exercises the momentum recurrence (first_step != step)
    step.fill_(2)
    p1, m1 = params.clone(), mom.clone()
    K.aggregate_update(L, slots, L.total, params=params, momentum=mom, hp=hp, step_ptr=step, done_counter=cnt[0:1],
                       K=G, scale=1.0 / G, select=win_slot, first_step=1, dst=peers, flags=[flags[0:1]])
    torch.cuda.synchronize()
    p_ref2, m_ref2 = _sgd_ref(p1.cpu().double(), m1.cpu().double(), agg, 0.1, 0.9, 1e-3, first=False)
    assert torch.allclose(params.cpu().double()[ok], p_ref2[ok], atol=1e-5)
    assert flags[0].item() == 3


def test_update_matches_torch_sgd_over_steps(K, dev):
    """Mean aggregation + fused SGD vs torch.optim.SGD with nesterov + weight decay."""
    L = ArenaLayout.from_model(build_model("FC"), bf16=False)
    P = 4
    cfg = JobConfig(lr=0.05, momentum=0.8, weight_decay=5e-4, nesterov=True)
    hp = hyperparams_tensor(cfg, dev)
    params = fill_valid(L, 1, dev, seed=2)[0]
    ref_p = params.clone().requires_grad_(True)
    opt = torch.optim.SGD([ref_p], lr=0.05, momentum=0.8, weight_decay=5e-4, nesterov=True)
    mom = torch.zeros_like(params)
    step, cnt, flags = ctrl(dev, 1)
    for it in range(1, 5):
        slots = fill_valid(L, P, dev, seed=10 + it, scale=0.3)
        step.fill_(it)
        K.aggregate_update(L, slots, L.total, params=params, momentum=mom, hp=hp, step_ptr=step, done_counter=cnt[0:1],
                           K=P, scale=1.0 / P, first_step=1)
        ref_p.grad = slots.mean(0)
        opt.step()
    torch.cuda.synchronize()
    assert torch.allclose(params, ref_p.detach(), atol=2e-6)


# ------------------------------------------------------------------------------------------------ cyclic decode
@pytest.mark.parametrize("n,s,liars", [(7, 2, (1, 4)), (7, 2, ()), (7, 3, (0, 2, 6)), (7, 1, (3,)), (5, 2, (4,))])
def test_cyclic_decode_kernels(K, dev, n, s, liars):
    code = cyclic.search_w(n, s)
    L = ArenaLayout.from_model(build_model("LeNet"), bf16=False, channels_last=True)     # fp32 gradient streams only
    Gm = fill_valid(L, n, dev, seed=4, scale=0.05)
    step, cnt, flags = ctrl(dev, 1)
    R = torch.zeros(n, 2 * L.total, device=dev)
    bitmap = torch.tensor([sum(1 << l for l in liars)], dtype=torch.int32, device=dev)
    for w in range(n):
        b = code.batches_of(w)
        K.push_encode(L, [Gm[j] for j in b], [None] * len(b), R[w], step_ptr=step, worker=w, done_counter=cnt[0:1],
                      coef=list(code.coeffs_of(w)), adv_bitmap=bitmap, adv_len=1, attack=2 if w % 2 else 1, magnitude=-100.0)
    T = L.ntensors
    E = torch.zeros(T, n, 2, dtype=torch.float64, device=dev)
    recomb = torch.zeros(T, n, 2, dtype=torch.float32, device=dev)
    healthy = torch.zeros(T, dtype=torch.int32, device=dev)
    flagged = torch.zeros(T, dtype=torch.int32, device=dev)
    g = torch.Generator().manual_seed(5)
    f = ((torch.randn(L.total, generator=g) + 1.0) * torch.from_numpy(L.valid_mask()).float()).to(dev)
    K.cyclic_project(L, R, L.total, n, f, E)
    torch.cuda.synchronize()
    Rc = torch.view_as_complex(R.view(n, L.total, 2)).cpu().numpy().astype(np.complex128)
    fc = f.cpu().double().numpy()
    Eh = torch.view_as_complex(E).cpu().numpy()
    for t, spec in enumerate(L.specs):
        ref = Rc[:, spec.offset:spec.offset + spec.numel] @ fc[spec.offset:spec.offset + spec.numel]
        assert np.abs(Eh[t] - ref).max() <= 1e-9 * max(1.0, np.abs(ref).max())
    K.cyclic_locate(E, n, s, recomb, healthy, flagged)
    torch.cuda.synchronize()
    assert float(E.abs().sum()) == 0                                     # accumulator handed back zeroed
    assert flagged.tolist() == [len(liars)] * T
    for t in range(T):
        for l in liars:
            assert not (int(healthy[t]) >> l) & 1
    cfg = JobConfig(lr=1.0, momentum=0.0)
    hp = hyperparams_tensor(cfg, dev)
    params = torch.zeros(L.total, device=dev)
    mom = torch.zeros(L.total, device=dev)
    gout = torch.zeros(L.total, device=dev)
    K.aggregate_update(L, R, L.total, params=params, momentum=mom, hp=hp, step_ptr=step, done_counter=cnt[0:1], K=n,
                       scale=1.0 / n, recomb=recomb, grad_out=gout)
    torch.cuda.synchronize()
    want = Gm.double().mean(0)
    assert torch.allclose(gout.double(), want, atol=5e-5), float((gout.double() - want).abs().max())
    assert torch.allclose(params.double(), -want, atol=5e-5)


# ------------------------------------------------------------------------------------------------ robust baselines
def test_krum_kernel(K, dev):
    L = small_layout()
    P, s = 7, 2
    honest = fill_valid(L, 1, dev, seed=6, scale=0.1)[0]
    slots = honest[None] + 0.01 * fill_valid(L, P, dev, seed=7)
    slots[2] = -100 * slots[2]
    slots[5] = fill_valid(L, 1, dev, seed=8, scale=30.0)[0]
    T = L.ntensors
    pair = torch.zeros(T, P * (P - 1) // 2, dtype=torch.float64, device=dev)
    sel = torch.zeros(T, dtype=torch.int32, device=dev)
    K.krum_select(L, slots, L.total, P, s, pair, sel)
    torch.cuda.synchronize()
    assert float(pair.abs().sum()) == 0
    sl = slots.cpu().double().numpy()
    for t, spec in enumerate(L.specs):
        assert int(sel[t]) == oracle.krum_index(sl[:, spec.offset:spec.offset + spec.numel], s), t


def test_geometric_median_kernel(K, dev):
    L = small_layout()
    P = 7
    honest = fill_valid(L, 1, dev, seed=11, scale=0.1)[0]
    slots = honest[None] + 0.02 * fill_valid(L, P, dev, seed=12)
    slots[0] = -100 * slots[0]
    slots[3] = -100 * torch.from_numpy(L.valid_mask()).float().to(dev)
    ws = K.GeoMedianWorkspace(L, P, dev)
    med = K.geometric_median(L, slots, L.total, P, ws, iters=80, eps=1e-7)
    torch.cuda.synchronize()
    sl = slots.cpu().double().numpy()
    for t, spec in enumerate(L.specs):
        X = sl[:, spec.offset:spec.offset + spec.numel]
        ref = oracle.geometric_median(X, eps=1e-9, max_iter=400)
        got = med[spec.offset:spec.offset + spec.numel].cpu().double().numpy()
        assert np.abs(got - ref).max() < 2e-3 * max(1.0, np.abs(ref).max()), (t, np.abs(got - ref).max())
    assert float(med[~torch.from_numpy(L.valid_mask()).to(dev)].abs().sum()) == 0


def test_geometric_median_weight_space_kernel(K, dev):
    """pairwise distances + Weiszfeld on the weights (one pass over the slab) against the fp64 oracle."""
    L = small_layout()
    P = 7
    T = L.ntensors
    honest = fill_valid(L, 1, dev, seed=21, scale=0.1)[0]
    slots = honest[None] + 0.02 * fill_valid(L, P, dev, seed=22)
    slots[1] = -100 * slots[1]
    slots[4] = -100 * torch.from_numpy(L.valid_mask()).float().to(dev)
    slots[6] = slots[6] + 3.0 * torch.from_numpy(L.valid_mask()).float().to(dev)
    pair = torch.zeros(T, P * (P - 1) // 2, dtype=torch.float64, device=dev)
    w = torch.zeros(T, P, dtype=torch.float32, device=dev)
    its = torch.zeros(T, dtype=torch.int32, device=dev)
    K.geometric_median_weights(L, slots, L.total, P, pair, w, iters_out=its)
    torch.cuda.synchronize()
    assert float(pair.abs().sum()) == 0                                   # scratch handed back zeroed
    assert torch.allclose(w.sum(1), torch.ones(T, device=dev), atol=1e-5) and float(w.min()) >= 0
    assert int(its.max()) < 256, its                                       # converged, not cut off
    sl = slots.cpu().double().numpy()
    wn = w.cpu().double().numpy()
    for t, spec in enumerate(L.specs):
        X = sl[:, spec.offset:spec.offset + spec.numel]
        ref = oracle.geometric_median(X, eps=1e-12, max_iter=2000)
        got = wn[t] @ X
        assert np.abs(got - ref).max() < 1e-3 * max(1.0, np.abs(ref).max()), (t, np.abs(got - ref).max())
    # all inputs identical -> uniform weights, no NaN
    same = honest[None].repeat(P, 1).contiguous()
    K.geometric_median_weights(L, same, L.total, P, pair, w)
    torch.cuda.synchronize()
    assert torch.allclose(w, torch.full_like(w, 1.0 / P))


# ------------------------------------------------------------------------------------------------ cast / flags
def test_cast_and_flag_kernels(K, dev):
    L = small_layout()
    src = fill_valid(L, 1, dev, seed=13)[0]
    dst = torch.zeros(L.total, dtype=torch.bfloat16, device=dev)
    K.cast_params(L, src, dst)
    step, cnt, flags = ctrl(dev, 3)
    err = torch.zeros(1, dtype=torch.int32, device=dev)
    K.set_flags([flags[0:1], flags[1:2]], step, 1)
    K.wait_flags([flags[0:1], flags[1:2]], step, 1, err, timeout_s=5.0)          # already satisfied
    K.step_add(step, 2)
    torch.cuda.synchronize()
    for s in L.specs:
        sl = slice(s.offset, s.offset + s.numel)
        if s.is_bf16:
            assert torch.equal(dst[sl], src[sl].to(torch.bfloat16))
        else:
            assert float(dst[sl].float().abs().sum()) == 0
    assert flags[:2].tolist() == [4, 4] and step.item() == 5 and err.item() == 0
    # watchdog: a flag nobody raises -> error code, not a hang
    K.wait_flags([flags[5:6]], step, 0, err, timeout_s=0.2)
    torch.cuda.synchronize()
    assert err.item() == 1


def test_cross_stream_flag_handshake(K, dev):
    """Producer and consumer on different streams synchronise only through the flag word."""
    L = small_layout(bf16_some=False)
    g32 = fill_valid(L, 1, dev, seed=14)[0]
    dst = torch.zeros(L.total, device=dev)
    out = torch.zeros(L.total, device=dev)
    step, cnt, flags = ctrl(dev, 9)
    err = torch.zeros(1, dtype=torch.int32, device=dev)
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    # CUDA loads kernels lazily and the first launch of a kernel synchronises with running work: launch every kernel
    # involved once (tables uploaded, modules loaded) before anything spins -- exactly what the engine's two eager
    # warm-up steps do before the step graph is captured.
    K.set_flags([flags[7:8]], step, 0)
    K.wait_flags([flags[7:8]], step, 0, err, timeout_s=5.0)
    K.push_encode(L, [g32], [None], out, step_ptr=step, worker=0, done_counter=cnt[0:1], flag=flags[6:7])
    with torch.cuda.stream(s1):
        torch.cuda._sleep(1000)
    out.zero_()
    torch.cuda.synchronize()
    with torch.cuda.stream(s2):                      # consumer first: spins until the producer's release
        K.wait_flags([flags[0:1]], step, 0, err, timeout_s=20.0)
        out.copy_(dst)
    with torch.cuda.stream(s1):
        torch.cuda._sleep(20_000_000)
        K.push_encode(L, [g32], [None], dst, step_ptr=step, worker=0, done_counter=cnt[0:1], flag=flags[0:1])
    torch.cuda.synchronize()
    assert err.item() == 0 and torch.equal(out, g32)


@pytest.mark.timeout(120)
def test_fused_cross_entropy_kernel(monkeypatch):
    """One-launch softmax-CE + gradient + Prec@k (csrc/cuda/loss_fused.cu) vs the PyTorch ops it replaces."""
    import torch.nn.functional as F

    from draco_b200.ops.loss import accuracy, cross_entropy_with_metrics
    dev = torch.device("cuda", 0)
    for (B, Cn, dt) in [(128, 10, torch.bfloat16), (37, 10, torch.float32), (64, 1000, torch.bfloat16), (5, 3, torch.float32)]:
        torch.manual_seed(B + Cn)
        logits = (torch.randn(B, Cn, device=dev) * 3).to(dt)
        # spread the values so that no two logits of a row tie after rounding (topk's tie order is unspecified)
        logits = (logits.float() + torch.arange(Cn, device=dev).float().view(1, -1) * 1e-2 * (1 if dt == torch.float32 else 8)).to(dt)
        labels = torch.randint(0, Cn, (B,), device=dev)
        met_ref = torch.zeros(3, device=dev)
        monkeypatch.setenv("DRACO_FUSED_LOSS", "0")
        l0 = logits.clone().requires_grad_(True)
        loss0 = cross_entropy_with_metrics(l0, labels, met_ref, 0.5)
        (loss0 * 2.0).backward()
        monkeypatch.setenv("DRACO_FUSED_LOSS", "1")
        met = torch.zeros(3, device=dev)
        l1 = logits.clone().requires_grad_(True)
        loss1 = cross_entropy_with_metrics(l1, labels, met, 0.5)
        (loss1 * 2.0).backward()
        assert abs(float(loss1) - float(loss0)) < 2e-3 * max(1.0, abs(float(loss0)))
        tol = 2e-2 if dt == torch.bfloat16 else 1e-4
        assert float((l1.grad.float() - l0.grad.float()).abs().max()) <= tol * float(l0.grad.float().abs().max())
        assert torch.allclose(met, met_ref, rtol=2e-3, atol=1e-3), (met, met_ref)
        # deterministic
        met2 = torch.zeros(3, device=dev)
        l2 = logits.clone().requires_grad_(True)
        cross_entropy_with_metrics(l2, labels, met2, 0.5).backward()
        l3 = logits.clone().requires_grad_(True)
        cross_entropy_with_metrics(l3, labels, torch.zeros(3, device=dev), 0.5).backward()
        assert torch.equal(l2.grad, l3.grad)


@pytest.mark.timeout(120)
def test_fused_input_prep_kernel(monkeypatch):
    from draco_b200 import JobConfig
    from draco_b200.data import synthetic_dataset
    from draco_b200.parallel.fused_engine import make_plan
    from draco_b200.parallel.ps import build_codes
    from draco_b200.parallel.worker import WorkerCompute
    dev = torch.device("cuda", 0)
    for net, dsn in (("ResNet18", "Cifar10"), ("LeNet", "MNIST")):
        cfg = JobConfig(network=net, dataset=dsn, approach="baseline", mode="normal", num_workers=1, batch_size=32, worker_fail=0,
                        err_mode="none", transport="nvl", dtype="bf16", synthetic_size=64)
        ds = synthetic_dataset(dsn, 64)
        wc = WorkerCompute(cfg, dev, [1], make_plan(cfg, ds, build_codes(cfg)[0]), ds)
        x = ds.images[:32].to(dev)
        monkeypatch.setenv("DRACO_FUSED_PREP", "0")
        ref = wc._prep_input(x)
        monkeypatch.setenv("DRACO_FUSED_PREP", "1")
        got = wc._prep_input(x)
        assert got.shape == ref.shape and got.dtype == ref.dtype
        assert got.is_contiguous(memory_format=torch.channels_last) and ref.is_contiguous(memory_format=torch.channels_last)
        assert float((got.float() - ref.float()).abs().max()) <= 2e-2          # at most one bf16 ulp of a value ~2.6


@pytest.mark.timeout(120)
def test_replica_dropout_is_keyed_by_device_step_and_graph_safe():
    """ops.dropout.ReplicaDropout: the mask depends only on (seed, step in DEVICE memory, batch id, layer) -- identical for two
    "holders", different across steps / batches / layers, backward uses the forward mask, and a replayed CUDA graph follows the
    device step without re-capture (ADVICE r1: nn.Dropout under graph replay gave every worker a different mask)."""
    from draco_b200.ops import dropout as D
    dev = torch.device("cuda", 0)
    step = torch.ones(1, dtype=torch.int64, device=dev)
    l1, l2 = D.ReplicaDropout(0.5, salt=1).to(dev), D.ReplicaDropout(0.5, salt=2).to(dev)
    x = torch.randn(128, 512, device=dev).to(torch.bfloat16)

    def run(layer, batch):
        D.set_context(step, 428, batch)
        xi = x.clone().requires_grad_(True)
        y = layer(xi)
        y.backward(torch.ones_like(y))
        D.clear_context()
        return y.detach(), xi.grad

    ya, ga = run(l1, 3)
    yb, gb = run(l1, 3)                                     # second holder of batch 3
    assert torch.equal(ya, yb) and torch.equal(ga, gb)
    keep = ya != 0
    assert 0.4 < keep.float().mean() < 0.6
    assert torch.equal(ga != 0, keep | (x == 0)) or torch.equal((ga != 0) & (x != 0), keep & (x != 0))   # same mask in backward
    assert torch.allclose(ya[keep].float(), x[keep].float() * 2, rtol=1e-2)
    assert not torch.equal(run(l1, 4)[0], ya) and not torch.equal(run(l2, 3)[0], ya)
    # graph replay follows the device step
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    D.set_context(step, 428, 3)
    out = torch.empty_like(x)
    with torch.cuda.stream(side):
        l1(x)
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out.copy_(l1(x))
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, ya)
    step.fill_(2)
    g.replay()
    torch.cuda.synchronize()
    y2 = out.clone()
    assert not torch.equal(y2, ya)
    D.clear_context()
    step.fill_(2)
    assert torch.equal(run(l1, 3)[0], y2)


@pytest.mark.parametrize("n,c,hw", [(128, 512, 4), (6, 2048, 7), (3, 64, 1), (17, 256, 5)])
def test_global_avg_pool_kernels(n, c, hw):
    """Global average pool forward / backward on channels-last bf16 (csrc/cuda/pool_head.cu) vs fp32 torch."""
    from draco_b200.ops.pool import backend_counters, global_avg_pool
    dev = torch.device("cuda", 0)
    torch.manual_seed(n + c)
    x = torch.randn(n, c, hw, hw, device=dev).to(torch.bfloat16).contiguous(memory_format=torch.channels_last).requires_grad_(True)
    before = backend_counters["native"]
    y = global_avg_pool(x)
    assert backend_counters["native"] == before + 1 and y.shape == (n, c)
    ref = x.detach().float().mean((2, 3))
    assert (y.float() - ref).abs().max() <= 1e-2 * ref.abs().max() + 1e-3
    gy = torch.randn(n, c, device=dev).to(torch.bfloat16)
    y.backward(gy)
    gref = (gy.float() / (hw * hw))[:, :, None, None].expand(n, c, hw, hw)
    assert x.grad.shape == x.shape and x.grad.is_contiguous(memory_format=torch.channels_last)
    assert (x.grad.float() - gref).abs().max() <= 1e-2 * gref.abs().max() + 1e-6
    # fp32 / non-channels-last inputs take the library path with the same result
    assert torch.allclose(global_avg_pool(x.detach().float()), ref, atol=1e-5)


def test_narrow_head_backward_prep_kernel():
    """dy zero-padded to a 16-byte row + bias gradient in one launch (the 10-class Linear backward)."""
    from draco_b200.ops.pool import head_prep
    dev = torch.device("cuda", 0)
    torch.manual_seed(3)
    dy = torch.randn(128, 10, device=dev).to(torch.bfloat16)
    dyp, db = head_prep(dy, 16, True)
    assert torch.equal(dyp[:, :10], dy) and torch.count_nonzero(dyp[:, 10:]) == 0
    assert (db.float() - dy.float().sum(0)).abs().max() < 0.1
    assert torch.equal(head_prep(dy, 16, True)[1], db)
    assert head_prep(dy, 16, False)[1] is None
