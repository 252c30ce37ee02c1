"""signSGD with majority vote (``--mode sign_vote``) on the CPU: the configuration, the oracle (bit order, edge values, ties,
padding, the honest majority), the library transports' byte packing against the oracle on a ResNet-18 arena, Gloo jobs replayed
step by step through the oracle with and without worker momentum, a multi-process Gloo job against the single-process one with
its wire volume, and the fused PS's launch sequence."""
import multiprocessing as mp
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist

from draco_b200 import JobConfig
from draco_b200.codes import oracle
from draco_b200.config import MODES
from draco_b200.models import build_model
from draco_b200.ops import kernels as K
from draco_b200.parallel.arena import ArenaLayout
from draco_b200.parallel.collective_engine import sign_bytes
from draco_b200.parallel.ps import PIPELINED_RULES, FusedPS, TorchPS, build_codes, rule_plan
from draco_b200.parallel.trainer import Trainer

CPU = torch.device("cpu")


def _cfg(**kw):
    base = dict(network="LeNet", dataset="MNIST", batch_size=16, max_steps=12, transport="gloo", lr=0.002, momentum=0.0,
                synthetic_size=512, eval_freq=10 ** 6, compress_grad="None", approach="baseline", mode="sign_vote", num_workers=5,
                worker_fail=2, err_mode="rev_grad")
    base.update(kw)
    return JobConfig(**base)


# ------------------------------------------------------------------------------------------------ configuration
def test_configuration_accepts_the_mode_and_rejects_every_misuse():
    assert "sign_vote" in MODES
    for kw in (dict(), dict(transport="nvl"), dict(transport="nccl"), dict(worker_momentum=0.9), dict(optimizer="adam"),
               dict(optimizer="adam", amsgrad=True, worker_momentum=0.9), dict(err_mode="constant"), dict(err_mode="random"),
               dict(err_mode="none", worker_fail=0), dict(transport="nvl", num_workers=32, worker_fail=15),
               dict(transport="nccl", num_workers=40, worker_fail=3), dict(num_workers=1, worker_fail=0)):
        cfg = _cfg(**kw).resolve(1)
        plan = rule_plan(cfg)
        assert (plan.rule, plan.base, plan.source, plan.rows, plan.opt_mode) == ("sign_vote", "sign_vote", "raw",
                                                                                  cfg.num_workers, "sign_vote")
        assert plan.pipelined and "sign_vote" in PIPELINED_RULES

    def bad(match, **kw):
        with pytest.raises(ValueError, match=match):
            _cfg(**kw).resolve(1)
    for approach in ("maj_vote", "cyclic", "detox", "nnm"):
        bad("use --approach baseline", approach=approach, num_workers=9, group_size=3, worker_fail=1)
    for err in ("omniscient", "alie", "minmax"):
        bad(f"--err-mode {err} builds a real-valued row", err_mode=err)
    bad("pass --compress-grad None", compress_grad="compress")
    bad("use --transport nccl for --mode sign_vote", transport="nccl_flat")
    bad("strict majority", num_workers=4, worker_fail=2)
    bad("strict majority", num_workers=5, worker_fail=3)
    bad("at most 32 workers", transport="nvl", num_workers=33, worker_fail=1)
    bad("coordinate-wise, so the scope would change nothing", rule_scope="model")
    # the default --compress-grad is the codec: a sign_vote job at the defaults does not resolve
    with pytest.raises(ValueError):
        JobConfig(approach="baseline", mode="sign_vote").resolve(1)


# ------------------------------------------------------------------------------------------------ oracle
def test_pack_unpack_round_trip_and_bit_order():
    rng = np.random.default_rng(0)
    x = rng.normal(size=(3, 2048)).astype(np.float32)
    w = oracle.sign_pack(x)
    assert w.dtype == np.uint32 and w.shape == (3, 64)
    assert np.array_equal(oracle.sign_unpack(w), (x < 0).astype(np.uint8))
    e = np.zeros(64, dtype=np.float32)
    e[[0, 5, 31, 32, 63]] = -1.0
    assert oracle.sign_pack(e).tolist() == [(1 << 0) | (1 << 5) | (1 << 31), (1 << 0) | (1 << 31)]
    # the library transports' bytes: byte i, bit b = element 8 i + b
    b = oracle.sign_pack(e).view(np.uint8)
    assert b.tolist() == [0b00100001, 0, 0, 0x80, 0x01, 0, 0, 0x80]
    with pytest.raises(ValueError, match="multiple of 32"):
        oracle.sign_pack(np.zeros(33, dtype=np.float32))


def test_edge_values_send_plus_except_strictly_negative_ones():
    tiny = np.float32(1e-45)                                    # the smallest subnormal
    vals = np.array([0.0, -0.0, np.nan, -np.nan, np.inf, -np.inf, tiny, -tiny, 1e-40, -1e-40, 3.4e38, -3.4e38,
                     np.float32(-1.0) * np.float32(0.0), 1.0, -1.0, -np.finfo(np.float32).tiny], dtype=np.float32)
    vals = np.concatenate([vals, np.full(16, 2.0, dtype=np.float32)])
    bits = oracle.sign_unpack(oracle.sign_pack(vals))[:16]
    assert bits.tolist() == [0, 0, 0, 0, 0, 1, 0, 1, 0, 1, 0, 1, 0, 0, 1, 1]


def test_padding_bits_are_zero_and_padding_votes_zero():
    x = -np.ones((3, 64), dtype=np.float32)
    valid = np.zeros(64, dtype=bool)
    valid[:40] = True
    w = oracle.sign_pack(x, valid)
    assert w[:, 0].tolist() == [0xFFFFFFFF] * 3 and w[:, 1].tolist() == [0xFF] * 3
    # whatever the bits say, a padding coordinate votes +0
    g = oracle.sign_vote(np.ones((3, 64), dtype=np.uint8), 3, valid)
    assert g[:40].tolist() == [-1.0] * 40 and g[40:].tolist() == [0.0] * 24
    assert not np.signbit(g[40:]).any()


@pytest.mark.parametrize("P", [1, 2, 3, 4, 7, 8, 16, 31, 32])
def test_vote_counts_every_split_including_ties(P):
    # column j: the first j rows say "-" (bit 1)
    bits = (np.arange(P)[:, None] < np.arange(P + 1)[None, :]).astype(np.uint8)
    g = oracle.sign_vote(bits, P, np.ones(P + 1, dtype=bool))
    want = [1.0 if P - j > j else -1.0 if j > P - j else 0.0 for j in range(P + 1)]
    assert g.dtype == np.float32 and g.tolist() == want
    if P % 2 == 0:
        assert g[P // 2] == 0.0 and not np.signbit(g[P // 2])    # a tie is +0
    with pytest.raises(ValueError, match="expected"):
        oracle.sign_vote(bits, P + 1, np.ones(P + 1, dtype=bool))


@pytest.mark.parametrize("P,f", [(3, 1), (5, 2), (7, 3), (15, 7), (32, 15), (9, 0)])
def test_honest_majority_returns_the_honest_signs_under_rev_grad(P, f):
    rng = np.random.default_rng(P)
    n = 4096
    valid = np.ones(n, dtype=bool)
    valid[-77:] = False
    honest = rng.normal(size=n).astype(np.float32)
    honest[::13] = 0.0                                          # a zero sends "+" and rev_grad cannot flip it
    rows = np.stack([honest] * P)
    rows[:f] = rows[:f] * np.float32(-100.0)                     # the liars
    g = oracle.sign_vote(oracle.sign_unpack(oracle.sign_pack(rows, valid)), P, valid)
    want = np.where(valid, np.where(honest < 0, -1.0, 1.0), 0.0).astype(np.float32)
    assert np.array_equal(g, want)


def test_signum_is_the_worker_momentum_oracle_then_the_pack():
    rng = np.random.default_rng(3)
    m = np.zeros(1024, dtype=np.float32)
    for _ in range(4):
        g = rng.normal(size=1024).astype(np.float32)
        m = oracle.worker_momentum(m, g, 0.9)
    assert np.array_equal(oracle.sign_unpack(oracle.sign_pack(m)), (m < 0).astype(np.uint8))


# ------------------------------------------------------------------------------------------------ library packing
def test_library_packing_equals_the_oracle_on_a_resnet18_arena():
    L = ArenaLayout.from_model(build_model("ResNet18"), bf16=True, channels_last=True)
    g = torch.Generator().manual_seed(0)
    x = torch.randn(L.total, generator=g)
    x[:12] = torch.tensor([0.0, -0.0, float("nan"), -float("nan"), float("inf"), -float("inf"), 1e-45, -1e-45, 1e-40, -1e-40,
                           -1.0, 1.0])
    x[x.abs() < 0.01] = -0.0
    valid = L.valid_mask()
    x[torch.from_numpy(~valid)] = -5.0                           # padding that is not zero must still send 0 bits
    b = sign_bytes(x, torch.from_numpy(valid))
    assert b.dtype == torch.uint8 and b.shape == (L.total // 8,)
    assert np.array_equal(b.numpy(), oracle.sign_pack(x.numpy(), valid).view(np.uint8))


# ------------------------------------------------------------------------------------------------ Gloo jobs
def _replay(cfg, steps):
    """Run the job and replay it through the oracle: each worker's flat gradient (through worker momentum), the attack, the
    pack, the vote, then p <- p - fp32(lr) g in fp32 (SGD without momentum: g is +-1 or 0, so every path rounds the same)."""
    t = Trainer(cfg, rank=0, world=1, device=CPU, quiet=True)
    eng, wc = t.engine, t.engine.worker
    L = eng.layout
    valid = L.valid_mask()
    grads = {}
    real_fb = wc.forward_backward

    def fb(w, step_host=None, **kw):
        real_fb(w, step_host, **kw)
        grads[w] = wc.flat_gradient(0).numpy().copy()
    wc.forward_backward = fb
    p = eng.master_params().numpy().copy()
    m = {w: np.zeros(L.total, dtype=np.float32) for w in range(1, cfg.num_workers + 1)}
    liars = 0
    for step in range(1, steps + 1):
        t.train_step()
        rows = []
        for w in range(1, cfg.num_workers + 1):
            x = grads[w]
            if cfg.worker_momentum:
                m[w] = oracle.worker_momentum(m[w], x, cfg.worker_momentum)
                x = m[w]
            if cfg.worker_fail and eng.schedule.is_adversary(w, step):
                liars += 1
                x = np.where(valid, x * np.float32(cfg.attack_magnitude) if cfg.err_mode == "rev_grad"
                             else np.float32(cfg.attack_magnitude), x).astype(np.float32)
            rows.append(oracle.sign_pack(x, valid))
            assert np.array_equal(eng.slots[w - 1].numpy(), rows[-1].view(np.uint8)), (step, w)
        g = oracle.sign_vote(oracle.sign_unpack(np.stack(rows)), cfg.num_workers, valid)
        p = np.subtract(p, np.multiply(np.float32(cfg.lr), g, dtype=np.float32), dtype=np.float32)
        assert np.array_equal(eng.master_params().numpy().view(np.int32), p.view(np.int32)), step
    return t, liars


@pytest.mark.parametrize("kw", [dict(), dict(worker_momentum=0.9), dict(num_workers=3, worker_fail=1, err_mode="constant"),
                                dict(num_workers=4, worker_fail=1, worker_momentum=0.5)])
def test_gloo_job_equals_the_oracle_replay(kw):
    cfg = _cfg(**kw)
    t, liars = _replay(cfg, 5)
    assert liars > 0
    assert torch.isfinite(t.engine.master_params()).all()


def test_a_tie_leaves_the_coordinate_alone_with_two_workers():
    cfg = _cfg(num_workers=2, worker_fail=0, err_mode="none")
    _replay(cfg, 3)


def test_sign_vote_trains_and_composes_with_adam():
    t = Trainer(_cfg(worker_momentum=0.9, lr=0.002), rank=0, world=1, device=CPU, quiet=True)
    losses = [t.train_step()["loss"] for _ in range(12)]
    assert losses[-1] < losses[0], losses
    a = Trainer(_cfg(optimizer="adam", lr=1e-3), rank=0, world=1, device=CPU, quiet=True)
    la = [a.train_step()["loss"] for _ in range(4)]
    assert np.isfinite(la).all() and torch.isfinite(a.engine.master_params()).all()


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _gloo_proc(rank, world, port, kw, steps, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    t = Trainer(_cfg(**kw), rank=rank, world=world, device=CPU, quiet=True)
    for _ in range(steps):
        t.train_step()
    t.engine._broadcast_params()
    q.put((rank, t.engine.master_params().numpy().copy(), t.engine.bytes_up, list(t.engine.local_workers)))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("kw", [dict(num_workers=3, worker_fail=1), dict(num_workers=2, worker_fail=0, err_mode="none",
                                                                         worker_momentum=0.9)])
def test_multi_process_gloo_job_equals_the_single_process_job_and_sends_bits(kw):
    steps, world = 3, 3
    port = _free_port()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_gloo_proc, args=(r, world, port, kw, steps, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = sorted((q.get(timeout=300) for _ in range(world)), key=lambda r: r[0])
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    single = Trainer(_cfg(**kw), rank=0, world=1, device=CPU, quiet=True)
    for _ in range(steps):
        single.train_step()
    want = single.engine.master_params().numpy()
    L = single.engine.layout
    per_step = sum((s.numel + 7) // 8 for s in L.specs)
    assert per_step < L.total // 8 + 1 and per_step * 32 < L.total * 4
    for rank, params, up, workers in res:
        assert np.array_equal(params.view(np.int32), want.view(np.int32)), rank
        remote = [w for w in workers if rank != 0]
        assert up == steps * per_step * len(remote), (rank, up, workers)
    assert sum(len(r[3]) for r in res) == kw["num_workers"] and any(r[2] > 0 for r in res)


# ------------------------------------------------------------------------------------------------ fused PS launch sequence
@pytest.mark.parametrize("bucketed", [False, True])
def test_fused_ps_launches_one_sign_vote_update_per_bucket_like_the_mean(monkeypatch, bucketed):
    L = ArenaLayout.from_model(build_model("LeNet"), bf16=False, channels_last=True)
    buckets = [(0, 3, [0, 1]), (3, 7, [2, 3, 4]), (7, L.ntiles, list(range(5, L.ntensors)))] if bucketed else None

    def launches(mode):
        calls = []
        for name in ("aggregate_update", "sign_vote_update", "vote", "ps_attack"):
            monkeypatch.setattr(K, name, lambda *a, _n=name, **kw: calls.append((_n, a[2], kw.get("P"), kw.get("K"),
                                                                                  kw.get("tile_range"), kw.get("flags"))))
        cfg = _cfg(mode=mode, transport="nvl", num_workers=20, worker_fail=3).resolve(1)
        P = cfg.num_workers
        words = P * L.total // 32 if mode == "sign_vote" else P * L.total
        ps = FusedPS(cfg, L, CPU, L.new_arena(CPU), torch.zeros(words), *build_codes(cfg),
                     adv_bitmap=torch.zeros(8, dtype=torch.int32), adv_len=8)
        kw = dict(buckets=buckets, wait_bucket=lambda b: calls.append(("wait", b)) or 1) if buckets else {}
        n = ps.enqueue_step(torch.ones(1, dtype=torch.int64), mc_params=None, dst=[4096], flags=[16, 32], **kw)
        return ps, calls, n
    ps, calls, n = launches("sign_vote")
    _, mean_calls, n_mean = launches("normal")
    assert ps.slot_stride == L.total // 32 and n == n_mean
    ranges = [(t0, t1) for t0, t1, _ in buckets] if bucketed else [None]
    want = []
    for bi, tiles in enumerate(ranges):
        if bucketed:
            want.append(("wait", bi))
        want.append(("sign_vote_update", L.total // 32, 20, None, tiles, [16, 32] if bi == len(ranges) - 1 else []))
    assert calls == want
    assert [c[0] for c in mean_calls] == [c[0].replace("sign_vote_update", "aggregate_update") for c in calls]


def test_torch_ps_passes_the_optimizer_mode_and_votes_per_tensor():
    cfg = _cfg(num_workers=3, worker_fail=1).resolve(1)
    L = ArenaLayout.from_model(build_model("LeNet"), bf16=False, channels_last=False)
    params = L.new_arena(CPU)
    ps = TorchPS(cfg, L, CPU, params, *build_codes(cfg))
    rng = np.random.default_rng(7)
    valid = L.valid_mask()
    rows = rng.normal(size=(3, L.total)).astype(np.float32)
    slots = torch.from_numpy(oracle.sign_pack(rows, valid).view(np.uint8).copy())
    grads = ps.aggregate(slots)
    want = oracle.sign_vote(oracle.sign_unpack(oracle.sign_pack(rows, valid)), 3, valid)
    for s, g in zip(L.specs, grads):
        assert g.dtype == torch.float32 and np.array_equal(g.numpy(), want[s.offset: s.offset + s.numel])
    seen = []
    real_step = ps.optimizer.step
    ps.optimizer.step = lambda grads, mode: seen.append(mode) or real_step(grads=grads, mode=mode)
    ps.apply(grads)
    assert seen == ["sign_vote"]
