"""The ALIE and min-max attacks on the CPU: the fp64 oracle on hand-worked cases and random rows, the configuration checks and
the flag surface, and whole jobs on the library-op PS over Gloo (exact recovery by the vote, damage to the median and trimmed
mean, DETOX over every liar subset, a multi-process job equal to the single-process one)."""
import argparse
import hashlib
import itertools
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from draco_b200 import JobConfig
from draco_b200.codes import adversary as A
from draco_b200.codes import oracle
from draco_b200.codes.repetition import group_assign
from draco_b200.config import add_fit_args, config_from_args
from draco_b200.models import build_model
from draco_b200.parallel.arena import ArenaLayout
from draco_b200.parallel.collective_engine import attack_row
from draco_b200.parallel.ps import TorchPS, build_codes
from draco_b200.parallel.trainer import Trainer


# ------------------------------------------------------------------------------------------------ oracle
def test_alie_z_max_values():
    assert A.alie_z_max(7, 3) == pytest.approx(1.0676, abs=1e-4)
    assert A.alie_z_max(15, 3) == pytest.approx(0.4307, abs=1e-4)
    assert A.alie_z_max(7, 1) == pytest.approx(0.1800, abs=1e-4)
    assert (A.alie_s(7, 3), A.alie_s(15, 3), A.alie_s(7, 1)) == (1, 5, 3)
    with pytest.raises(ValueError, match="undefined"):
        A.alie_z_max(7, 4)                                             # s = 0


def test_alie_hand_worked():
    H = np.array([[1.0, 0.0], [3.0, 0.0]])                              # mu = [2, 0], sigma = [1, 0]
    assert A.alie_row(H, 1.5).tolist() == [0.5, 0.0]


def test_minmax_with_equal_honest_rows_sends_them():
    H = np.array([[1.0, -2.0, 3.0]] * 4)                                 # sigma = 0, c = 0: gamma = 0
    assert A.minmax_gamma(H) == 0.0
    assert A.minmax_row(H).tolist() == [1.0, -2.0, 3.0]


def test_minmax_with_one_honest_row_sends_it():
    H = np.array([[0.5, -7.0]])
    assert A.minmax_gamma(H) == 0.0 and A.minmax_row(H).tolist() == [0.5, -7.0]
    assert A.alie_row(H, 1.0).tolist() == [0.5, -7.0]


def test_minmax_hand_worked():
    """Two honest rows g_1 = [0, 0], g_2 = [2, 0]: mu = [1, 0], sigma = [1, 0], Dmax = 2, row = [1 - gamma, 0].  The farthest
    honest row is g_2 at distance 1 + gamma, so gamma = 1 and the row is g_1 itself."""
    H = np.array([[0.0, 0.0], [2.0, 0.0]])
    assert A.minmax_gamma(H) == 1.0
    assert A.minmax_row(H).tolist() == [0.0, 0.0]


def test_duplicate_honest_rows_each_count():
    """Under maj_vote every copy of a group's gradient is an honest slot: duplicates weigh in the mean and the spread."""
    H = np.array([[0.0], [0.0], [4.0]])                                 # mu = 4/3, sigma = sqrt(32/9)
    mu, sd = A.honest_stats(H)
    assert mu[0] == pytest.approx(4 / 3) and sd[0] == pytest.approx(np.sqrt(32 / 9))
    assert A.alie_row(H, 1.0)[0] == pytest.approx(4 / 3 - np.sqrt(32 / 9))
    X = np.array([[0.0], [0.0], [4.0], [9.0]])
    out = A.ps_attack(X, [3], "alie", [(0, 1)], z=1.0)
    assert out[3, 0] == pytest.approx(4 / 3 - np.sqrt(32 / 9)) and out[:3].tolist() == X[:3].tolist()


@pytest.mark.parametrize("n,d", [(2, 5), (4, 300), (12, 1000), (15, 64)])
def test_minmax_row_meets_the_distance_bound_and_gamma_is_the_largest(n, d):
    rng = np.random.default_rng(n * d)
    for trial in range(20):
        H = rng.normal(size=(n, d)) * rng.uniform(0.01, 10, size=d)
        if trial % 2:
            H += rng.normal(size=d) * 5                                  # a common offset
        D2 = max(((H[i] - H[j]) ** 2).sum() for j in range(n) for i in range(j))
        mu, sd = A.honest_stats(H)
        g = A.minmax_gamma(H)
        assert g > 0
        far = max(((mu - g * sd - h) ** 2).sum() for h in H)
        assert far <= D2 * (1 + 1e-12)
        assert far >= D2 * (1 - 1e-9)                                    # binding: equality up to rounding
        assert max(((mu - 1.01 * g * sd - h) ** 2).sum() for h in H) > D2
        # the library PS's torch version gives the same row
        np.testing.assert_allclose(attack_row(torch.from_numpy(H), "minmax").numpy(), A.minmax_row(H), rtol=1e-12, atol=1e-12)


def test_nan_in_the_honest_rows_poisons_the_row():
    H = np.array([[1.0, np.nan], [2.0, 0.0], [4.0, 1.0]])
    assert np.isnan(A.minmax_gamma(H)) and np.isnan(A.minmax_row(H)).all()
    r = A.alie_row(H, 1.0)
    assert np.isfinite(r[0]) and np.isnan(r[1])                          # ALIE is per coordinate


def test_existing_attack_codes_are_unchanged():
    assert [A.attack_code(m) for m in ("none", "rev_grad", "constant", "random", "omniscient", "alie", "minmax")] == list(range(7))


# ------------------------------------------------------------------------------------------------ configuration
def _c(**kw):
    return JobConfig(**dict(dict(num_workers=7, worker_fail=3, approach="baseline", mode="coordinate_median", err_mode="alie"), **kw))


def test_config_accepts_and_rejects_attack_jobs():
    assert _c().resolve(1).alie_z == pytest.approx(1.0676, abs=1e-4)
    assert _c(attack_z=2.5).resolve(1).alie_z == 2.5
    _c(err_mode="minmax").resolve(1)
    _c(approach="maj_vote", mode="maj_vote", group_size=3).resolve(1)
    with pytest.raises(ValueError, match="--attack-z sets ALIE's z"):
        _c(err_mode="minmax", attack_z=1.0).resolve(1)
    with pytest.raises(ValueError, match="--attack-z sets ALIE's z"):
        _c(err_mode="rev_grad", attack_z=1.0).resolve(1)
    for m in ("alie", "minmax"):
        with pytest.raises(ValueError, match="cyclic code's slots hold complex"):
            _c(err_mode=m, approach="cyclic", worker_fail=1).resolve(1)
        with pytest.raises(ValueError, match="nccl_flat implements the rev_grad and constant attacks only"):
            _c(err_mode=m, transport="nccl_flat", compress_grad="None").resolve(1)
        with pytest.raises(ValueError, match="worker_fail < num_workers"):
            _c(err_mode=m, approach="maj_vote", mode="maj_vote", worker_fail=7, attack_z=1.0 if m == "alie" else None).resolve(1)
        with pytest.raises(ValueError, match="at most 16 workers"):
            _c(err_mode=m, num_workers=17, approach="maj_vote", mode="normal", group_size=1).resolve(1)
        _c(err_mode=m, num_workers=17, approach="maj_vote", mode="normal", group_size=1, transport="nccl").resolve(1)
    with pytest.raises(ValueError, match="undefined.*pass --attack-z"):
        _c(approach="maj_vote", mode="maj_vote", worker_fail=4).resolve(1)           # s = 0
    _c(approach="maj_vote", mode="maj_vote", worker_fail=4, attack_z=1.0).resolve(1)
    # the other attacks are unchanged: omniscient still goes everywhere it went
    JobConfig(err_mode="omniscient", num_workers=7, worker_fail=7, compress_grad="None").resolve(1)


def test_flag_surface():
    p = add_fit_args(argparse.ArgumentParser())
    c = config_from_args(p.parse_args(["--err-mode", "alie", "--attack-z", "0.75"]))
    assert (c.err_mode, c.attack_z) == ("alie", 0.75)
    c = config_from_args(p.parse_args(["--err-mode", "minmax"]))
    assert (c.err_mode, c.attack_z) == ("minmax", None)
    h = p.format_help()
    assert "alie" in h and "minmax" in h and "--attack-z" in h


# ------------------------------------------------------------------------------------------------ library-op PS
def _layout():
    return ArenaLayout.from_model(build_model("LeNet"), bf16=False, channels_last=True)


def _cfg(**kw):
    base = dict(network="LeNet", dataset="MNIST", batch_size=16, max_steps=8, num_workers=7, transport="gloo", lr=0.05,
                momentum=0.9, synthetic_size=512, eval_freq=10 ** 6, compress_grad="None")
    base.update(kw)
    return JobConfig(**base)


def _run(cfg, steps):
    t = Trainer(cfg, rank=0, world=1, device=torch.device("cpu"), quiet=True)
    losses = [t.train_step()["loss"] for _ in range(steps)]
    return t, losses


@pytest.mark.parametrize("mode", ["alie", "minmax"])
def test_vote_is_bitwise_clean_while_no_group_is_captured(mode):
    kw = dict(approach="maj_vote", mode="maj_vote", num_workers=6, group_size=3, worker_fail=1)
    clean, lc = _run(_cfg(err_mode="none", **kw), 5)
    att, la = _run(_cfg(err_mode=mode, **kw), 5)
    assert torch.equal(clean.engine.master_params(), att.engine.master_params())
    assert lc == la


def test_engine_overwrites_the_liar_slots_with_the_oracle_row():
    """The library PS's step: liar slots = the fp64 oracle's row rounded to fp32, honest slots untouched."""
    t = Trainer(_cfg(approach="baseline", mode="coordinate_median", worker_fail=2, err_mode="minmax"), rank=0, world=1,
                device=torch.device("cpu"), quiet=True)
    eng = t.engine
    g = torch.Generator().manual_seed(3)
    eng.slots.copy_(torch.randn(eng.slots.shape, generator=g))
    eng.slots[:, ~torch.from_numpy(eng.layout.valid_mask())] = 0
    before = eng.slots.numpy().copy()
    eng._ps_attack(5)
    liars = [int(w) - 1 for w in eng.schedule.ranks[5]]
    spans = [(s.offset, s.numel) for s in eng.layout.specs]
    ref = A.ps_attack(before, liars, "minmax", spans)
    got = eng.slots.numpy()
    honest = [w for w in range(7) if w not in liars]
    assert np.array_equal(got[honest], before[honest])
    np.testing.assert_allclose(got[liars], ref[liars], rtol=1e-6, atol=1e-7)


@pytest.mark.parametrize("mode", ["coordinate_median", "trimmed_mean"])
def test_alie_moves_the_coordinate_rules_off_the_honest_aggregate(mode):
    """P = 7, f = 2: the ALIE row sits inside every coordinate's honest spread, yet it shifts the median and the trimmed mean
    away from the rule applied to the honest rows alone -- the attack bites."""
    L = _layout()
    cfg = _cfg(approach="baseline", mode=mode, worker_fail=2, err_mode="alie").resolve(1)
    ps = TorchPS(cfg, L, torch.device("cpu"), L.new_arena(torch.device("cpu")), None, None)
    g = torch.Generator().manual_seed(1)
    X = torch.randn(7, L.total, generator=g) + 0.5
    X[:, ~torch.from_numpy(L.valid_mask())] = 0
    liars, honest = [1, 4], [0, 2, 3, 5, 6]
    Xa = torch.from_numpy(A.ps_attack(X.numpy(), liars, "alie", [(s.offset, s.numel) for s in L.specs], z=cfg.alie_z))
    out = ps.aggregate(Xa)
    moved = 0.0
    for s, o in zip(L.specs, out):
        H = X[honest, s.offset:s.offset + s.numel].double().numpy()
        ref = oracle.coordinate_median(H) if mode == "coordinate_median" else oracle.trimmed_mean(H, 1)
        moved += float(np.abs(o.double().numpy() - ref).mean()) * s.numel
        lo, hi = H.min(0), H.max(0)
        assert np.all((o.double().numpy() >= lo - 1e-6) & (o.double().numpy() <= hi + 1e-6))
    assert moved / L.num_params > 0.05, moved / L.num_params


@pytest.mark.parametrize("attack", ["alie", "minmax"])
def test_detox_median_stays_within_the_honest_groups_for_every_liar_subset(attack):
    """P = 9, r = 3, f = 3 (G = 3, b_G = 1), all 84 liar subsets: at most one group is captured and every coordinate of the DETOX
    median lies within the range of the honest groups' gradients."""
    L = _layout()
    groups = group_assign(9, 3).groups
    cfg = _cfg(approach="detox", mode="coordinate_median", num_workers=9, group_size=3, worker_fail=3, err_mode=attack,
               attack_z=1.0).resolve(1) if attack == "alie" else \
        _cfg(approach="detox", mode="coordinate_median", num_workers=9, group_size=3, worker_fail=3, err_mode=attack).resolve(1)
    gr, _ = build_codes(cfg)
    ps = TorchPS(cfg, L, torch.device("cpu"), L.new_arena(torch.device("cpu")), gr, None)
    spans = [(s.offset, s.numel) for s in L.specs]
    g = torch.Generator().manual_seed(0)
    H = torch.randn(3, L.total, generator=g)
    H[:, ~torch.from_numpy(L.valid_mask())] = 0
    X = torch.empty(9, L.total)
    for gi, grp in enumerate(groups):
        X[[w - 1 for w in grp]] = H[gi]
    n = 0
    for liars in itertools.combinations(range(9), 3):
        Xa = torch.from_numpy(A.ps_attack(X.numpy(), liars, attack, spans, z=cfg.alie_z if attack == "alie" else None))
        captured = [gi for gi, grp in enumerate(groups) if len(set(liars) & {w - 1 for w in grp}) >= 2]
        assert len(captured) <= 1
        honest = [gi for gi in range(3) if gi not in captured]
        lo, hi = H[honest].min(0).values, H[honest].max(0).values
        for s, o in zip(L.specs, ps.aggregate(Xa)):
            assert bool(((o >= lo[s.offset:s.offset + s.numel]) & (o <= hi[s.offset:s.offset + s.numel])).all()), liars
        n += 1
    assert n == 84


# ------------------------------------------------------------------------------------------------ multi-process
def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _job(err_mode):
    return _cfg(approach="baseline", mode="trimmed_mean", num_workers=5, worker_fail=1, err_mode=err_mode, batch_size=8,
                synthetic_size=128, max_steps=6)


def _gloo_proc(rank, world, port, err_mode, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    torch.set_num_threads(2)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    t = Trainer(_job(err_mode), rank=rank, world=world, device=torch.device("cpu"), quiet=True)
    for _ in range(4):
        t.train_step()
    q.put((rank, hashlib.sha256(t.engine.master_params().numpy().tobytes()).hexdigest()))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("err_mode", ["alie", "minmax"])
def test_multi_process_job_equals_the_single_process_job(err_mode):
    """1 PS + 5 workers on 2 Gloo processes: the PS's parameters after 4 steps are bit-identical to the same job in one process."""
    world, port = 2, _free_port()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_gloo_proc, args=(r, world, port, err_mode, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = dict(q.get(timeout=300) for _ in range(world))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    threads = torch.get_num_threads()
    torch.set_num_threads(2)                     # the CPU convolutions' reduction order depends on the thread count
    try:
        single, _ = _run(_job(err_mode), 4)
    finally:
        torch.set_num_threads(threads)
    assert res[0] == hashlib.sha256(single.engine.master_params().numpy().tobytes()).hexdigest()
