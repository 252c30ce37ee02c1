"""The mimic and IPM attacks on the CPU: the configuration checks and the flag surface, the fp64 oracle on hand-worked cases and
its power iteration on rows with one dominant direction, the library-op PS against the oracle across the warm-up, the fused
PS's plan, a multi-process Gloo job against the single-process one, and checkpoint / resume inside the warm-up."""
import argparse
import hashlib
import math
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from draco_b200 import JobConfig
from draco_b200.codes import adversary as A
from draco_b200.config import MODES, add_fit_args, config_from_args
from draco_b200.models import build_model
from draco_b200.parallel.arena import ArenaLayout
from draco_b200.parallel.ps import TorchPS, rule_plan
from draco_b200.parallel.trainer import Trainer
from draco_b200.utils.checkpoint import load_checkpoint

CPU = torch.device("cpu")
NAN = float("nan")


def _bits(x):
    return np.asarray(x, dtype=np.float32).view(np.int32)


# ------------------------------------------------------------------------------------------------ configuration
def _c(**kw):
    return JobConfig(**dict(dict(num_workers=7, worker_fail=3, approach="baseline", mode="coordinate_median", err_mode="ipm"), **kw))


def test_codes_and_defaults():
    assert (A.attack_code("ipm"), A.attack_code("mimic")) == (A.ATTACK_IPM, A.ATTACK_MIMIC) == (7, 8)
    assert A.PS_ATTACKS == ("alie", "minmax", "ipm", "mimic")
    assert _c().resolve(1).ipm_eps == 0.1 and _c(attack_eps=0.5).resolve(1).ipm_eps == 0.5
    assert _c(err_mode="mimic").resolve(1).mimic_w == A.MIMIC_WARMUP
    assert _c(err_mode="mimic", mimic_warmup=0).resolve(1).mimic_w == 0


@pytest.mark.parametrize("m", ["ipm", "mimic"])
def test_every_misuse_is_rejected_with_its_reason(m):
    with pytest.raises(ValueError, match="cyclic code's slots hold complex"):
        _c(err_mode=m, approach="cyclic", worker_fail=1).resolve(1)
    with pytest.raises(ValueError, match=f"--err-mode {m} builds a real-valued row.*sign wire"):
        _c(err_mode=m, mode="sign_vote", compress_grad="None", worker_fail=1).resolve(1)
    with pytest.raises(ValueError, match="nccl_flat implements the rev_grad and constant attacks only"):
        _c(err_mode=m, transport="nccl_flat", compress_grad="None").resolve(1)
    with pytest.raises(ValueError, match="worker_fail < num_workers"):
        _c(err_mode=m, approach="maj_vote", mode="maj_vote", worker_fail=7).resolve(1)
    with pytest.raises(ValueError, match="at most 16 workers"):
        _c(err_mode=m, num_workers=17, approach="maj_vote", mode="normal", group_size=1).resolve(1)
    _c(err_mode=m, num_workers=17, approach="maj_vote", mode="normal", group_size=1, transport="nccl").resolve(1)
    with pytest.raises(ValueError, match="--attack-scope model sets one gamma"):
        _c(err_mode=m, attack_scope="model").resolve(1)
    for ok in (dict(approach="maj_vote", mode="maj_vote", group_size=3), dict(approach="detox", group_size=3, worker_fail=1),
               dict(approach="nnm", worker_fail=2), dict(bucketing=2, worker_fail=1), dict(worker_momentum=0.9)):
        _c(err_mode=m, **ok).resolve(1)


def test_flag_misuse_is_rejected():
    with pytest.raises(ValueError, match="--attack-eps sets IPM's eps: it needs --err-mode ipm"):
        _c(err_mode="alie", attack_eps=0.1).resolve(1)
    for bad in (0.0, -0.1, NAN, math.inf):
        with pytest.raises(ValueError, match="--attack-eps must be a finite eps > 0"):
            _c(attack_eps=bad).resolve(1)
    with pytest.raises(ValueError, match="--mimic-warmup sets how many steps.*needs --err-mode mimic"):
        _c(err_mode="ipm", mimic_warmup=3).resolve(1)
    with pytest.raises(ValueError, match="--mimic-warmup must be >= 0"):
        _c(err_mode="mimic", mimic_warmup=-1).resolve(1)


def test_flag_surface():
    p = add_fit_args(argparse.ArgumentParser())
    c = config_from_args(p.parse_args(["--err-mode", "ipm", "--attack-eps", "0.25"]))
    assert (c.err_mode, c.attack_eps, c.mimic_warmup) == ("ipm", 0.25, None)
    c = config_from_args(p.parse_args(["--err-mode", "mimic", "--mimic-warmup", "7"]))
    assert (c.err_mode, c.mimic_warmup, c.attack_eps) == ("mimic", 7, None)
    h = p.format_help()
    assert "ipm" in h and "mimic" in h and "--attack-eps" in h and "--mimic-warmup" in h


# ------------------------------------------------------------------------------------------------ oracle
def _state(m, z):
    return A.MimicState(np.asarray(m, dtype=np.float32), np.asarray(z, dtype=np.float32))


def test_ipm_row_hand_worked():
    H = np.array([[1.0, -2.0, 0.0], [3.0, 2.0, -0.0]])             # mu = [2, 0, 0]
    r = A.ipm_row(H, 0.5)
    assert r.tolist() == [-1.0, 0.0, 0.0] and _bits(r.astype(np.float32))[2] == _bits(np.float32(-0.0))
    out = A.ps_attack(np.array([[1.0, -2.0], [9.0, 9.0], [3.0, 2.0]], dtype=np.float32), [1], "ipm", [(0, 2)], z=0.1)
    assert out[1].tolist() == [np.float32(-0.2), np.float32(0.0)] and out[0].tolist() == [1.0, -2.0]


def test_target_is_the_largest_projection_ties_to_the_lower_slot_and_nan_wins():
    z = [1.0, 0.0, 0.0, 0.0]
    X = np.array([[1, 5, 0, 0], [3, 0, 0, 0], [9, 9, 9, 9], [3, 1, 0, 0]], dtype=np.float32)
    out, k, _ = A.mimic_step(X, [2], [(0, 4)], _state(np.zeros(4), z), t=0, W=0)
    assert k == 1                                                   # s = 1, 3, -, 3: the tie goes to slot 1
    assert _bits(out[2]).tolist() == _bits(X[1]).tolist() and np.array_equal(out[[0, 1, 3]], X[[0, 1, 3]])
    Xn = X.copy()
    Xn[3, 0] = NAN
    _, k, _ = A.mimic_step(Xn, [2], [(0, 4)], _state(np.zeros(4), z), t=0, W=0)
    assert k == 3                                                   # a NaN projection counts as the largest (np.argmax)
    Xn[0, 0] = NAN
    _, k, _ = A.mimic_step(Xn, [2], [(0, 4)], _state(np.zeros(4), z), t=0, W=0)
    assert k == 0                                                   # the first NaN


def test_padding_is_never_read_or_written():
    X = np.array([[1, NAN, 2], [0, 7, 5], [4, NAN, 3]], dtype=np.float32)    # column 1 is padding
    spans = [(0, 1), (2, 1)]
    out, k, st = A.mimic_step(X, [1], spans, _state(np.zeros(3), [0.6, 0.0, 0.8]), t=0, W=1)
    assert k == 2 and out[1, 0] == 4 and out[1, 2] == 3 and out[1, 1] == 7
    assert st.m[1] == 0 and st.z[1] == 0 and np.isfinite(st.z).all()


def test_one_warm_up_update_hand_worked():
    """x_0 = [1, 2], x_1 = [3, 0], z = [0.6, 0.8], m = 0, t = 0 (slot 2 lies): s = [2.2, 1.8] so k = 0; c = m' = [2, 1];
    <m', z> = 2, w = [0.2, -0.2]; u = 0.2 [-1, 1] - 0.2 [1, -1] = [-0.4, 0.4]; z' = [-1, 1] / sqrt 2."""
    X = np.array([[1, 2], [3, 0], [-50, 80]], dtype=np.float32)
    out, k, st = A.mimic_step(X, [2], [(0, 2)], _state([0, 0], [0.6, 0.8]), t=0, W=1)
    assert k == 0 and out[2].tolist() == [1.0, 2.0]
    assert st.m.tolist() == [2.0, 1.0]
    np.testing.assert_allclose(st.z, [-2 ** -0.5, 2 ** -0.5], rtol=1e-6)
    # t = 1: m = fp32((1 * m + c) / 2) with the new honest mean; past W nothing moves
    X2 = np.array([[0, 0], [-2, 4], [5, 5]], dtype=np.float32)    # slot 0 lies: c = [1.5, 4.5]
    _, k2, st2 = A.mimic_step(X2, [0], [(0, 2)], st, t=1, W=2)
    assert st2.m.tolist() == [1.75, 2.75] and k2 == 1              # z ~ [-1, 1] / sqrt 2 prefers [-2, 4]
    _, _, st3 = A.mimic_step(X2, [0], [(0, 2)], st2, t=2, W=2)
    assert _bits(st3.m).tolist() == _bits(st2.m).tolist() and _bits(st3.z).tolist() == _bits(st2.z).tolist()


def test_z0_is_a_unit_vector_on_the_valid_coordinates_and_fixed_by_the_seed():
    spans = [(0, 5), (8, 3)]
    z = A.mimic_z0(spans, 12)
    assert z.dtype == np.float32 and z[5:8].tolist() == [0, 0, 0] and z[11] == 0
    assert abs(float(np.linalg.norm(z.astype(np.float64))) - 1.0) < 1e-6
    assert np.array_equal(z, A.mimic_z0(spans, 12)) and not np.array_equal(z, A.mimic_z0(spans, 12, seed=1))


def test_warm_up_learns_the_dominant_direction_of_the_honest_rows():
    """Stationary honest rows mean + a_i v + 0.01 noise (D = 200, 10 honest of 12): after 50 warm-up steps z lies along the
    top eigenvector of the honest covariance, and from then on the liars copy the honest row with the largest projection."""
    rng = np.random.default_rng(0)
    D, P, liars, W = 200, 12, [3, 8], 50
    honest = [w for w in range(P) if w not in liars]
    v = rng.standard_normal(D)
    v /= np.linalg.norm(v)
    mean = rng.standard_normal(D)
    st = _state(np.zeros(D), A.mimic_z0([(0, D)], D))
    rows = []
    for t in range(W + 5):
        X = (mean + rng.standard_normal((P, 1)) * v + 0.01 * rng.standard_normal((P, D))).astype(np.float32)
        out, k, st = A.mimic_step(X, liars, [(0, D)], st, t=t, W=W)
        rows.append(X[honest].astype(np.float64))
        if t >= W:
            assert k == honest[int(np.argmax(X[honest].astype(np.float64) @ st.z.astype(np.float64)))]
            assert all(np.array_equal(out[w], X[k]) for w in liars)
    Hs = np.concatenate(rows)
    _, vecs = np.linalg.eigh(np.cov(Hs.T))
    assert abs(float(vecs[:, -1] @ st.z.astype(np.float64))) > 0.99


# ------------------------------------------------------------------------------------------------ fused plan
def test_mimic_leaves_the_pipeline_and_every_other_plan_is_unchanged():
    """``RulePlan.pipelined`` per --mode under baseline at the default scopes, the same for every pre-existing --err-mode (the
    table is the parent's behaviour), and False for every mode under mimic.  IPM keeps the table."""
    table = {"normal": True, "geometric_median": False, "krum": False, "maj_vote": True, "coordinate_median": True,
             "trimmed_mean": True, "multi_krum": False, "bulyan": False, "centered_clip": True, "sign_vote": True}
    assert set(table) == set(MODES)
    for err in ("rev_grad", "constant", "random", "omniscient", "alie", "minmax", "none", "ipm"):
        for mode, pipelined in table.items():
            for approach in ("baseline", "maj_vote", "nnm") if mode in ("coordinate_median", "krum") else ("baseline",):
                cfg = JobConfig(approach=approach, mode=mode, err_mode=err, num_workers=7, worker_fail=2, group_size=3)
                ref = rule_plan(JobConfig(approach=approach, mode=mode, err_mode="none", num_workers=7, worker_fail=2,
                                          group_size=3))
                assert rule_plan(cfg) == ref
                if approach == "baseline":
                    assert rule_plan(cfg).pipelined is pipelined, (err, mode)
    for mode in table:
        assert rule_plan(JobConfig(approach="baseline", mode=mode, err_mode="mimic", num_workers=7, worker_fail=2)).pipelined is False
    assert rule_plan(JobConfig(approach="maj_vote", mode="maj_vote", err_mode="mimic", num_workers=6, group_size=3)).pipelined is False


def test_fused_ps_reads_alies_z_only_under_alie():
    """3 workers, 2 liars: ALIE's z_max is undefined (s < 1), so the fused PS of every other attack must not form it.  The
    PS's attack parameter is IPM's eps under ipm and unused otherwise.  (The PS's state is built on the CPU here; it launches
    nothing until a step.)"""
    from draco_b200.parallel.ps import FusedPS
    L = ArenaLayout.from_model(build_model("LeNet"), bf16=False, channels_last=True)
    for err, code, z in (("rev_grad", 0, 0.0), ("ipm", A.ATTACK_IPM, 0.1)):
        cfg = JobConfig(num_workers=3, worker_fail=2, approach="maj_vote", mode="normal", group_size=1, err_mode=err,
                        network="LeNet").resolve(1)
        with pytest.raises(ValueError, match="undefined"):
            cfg.alie_z
        ps = FusedPS(cfg, L, CPU, L.new_arena(CPU), torch.zeros(3, L.total), None, None,
                     adv_bitmap=torch.zeros(4, dtype=torch.int32), adv_len=4)
        assert (ps.attack, ps.attack_z) == (code, z)


# ------------------------------------------------------------------------------------------------ library-op PS
def _layout():
    return ArenaLayout.from_model(build_model("LeNet"), bf16=False, channels_last=True)


def _cfg(**kw):
    base = dict(network="LeNet", dataset="MNIST", batch_size=16, max_steps=12, num_workers=7, worker_fail=2, transport="gloo",
                lr=0.05, momentum=0.9, synthetic_size=512, eval_freq=10 ** 6, compress_grad="None", approach="baseline",
                mode="coordinate_median", err_mode="mimic", mimic_warmup=3)
    base.update(kw)
    return JobConfig(**base)


def _trainer(cfg):
    return Trainer(cfg, rank=0, world=1, device=CPU, quiet=True)


def test_torch_ps_matches_the_oracle_across_the_warm_up():
    """Six steps with W = 3 on the LeNet arena, the same random slots into both.  The targets and the liar slots agree bit for
    bit; m too (its sums are sequential on both sides).  z goes through whole-model sums that torch and numpy order differently,
    each within ~1e-16 relative over 4e4 terms, so ||z_torch - z_oracle|| <= 1e-9 per step, allowed 1e-7 in total."""
    L = _layout()
    cfg = _cfg().resolve(1)
    ps = TorchPS(cfg, L, CPU, L.new_arena(CPU), None, None)
    spans = [(s.offset, s.numel) for s in L.specs]
    st = _state(ps.mimic_m.numpy(), ps.mimic_z.numpy())
    assert np.array_equal(st.z, A.mimic_z0(spans, L.total))
    rng = np.random.default_rng(5)
    valid = L.valid_mask()
    targets = []
    for t in range(6):
        X = (rng.standard_normal((7, L.total)) + 0.3 * rng.standard_normal((1, L.total))).astype(np.float32)
        X[:, ~valid] = 0
        liars = sorted(rng.choice(7, size=2, replace=False).tolist())
        ref, k, st = A.mimic_step(X, liars, spans, st, t=t, W=3)
        slots = torch.from_numpy(X.copy())
        ps.mimic_attack(slots, liars, t)
        assert ps.mimic_target == k
        targets.append(k)
        assert np.array_equal(_bits(slots.numpy()), _bits(ref))
        assert np.array_equal(_bits(ps.mimic_m.numpy()), _bits(st.m))
        assert float(np.linalg.norm(ps.mimic_z.numpy().astype(np.float64) - st.z.astype(np.float64))) <= 1e-7
    assert len(set(targets)) > 1


def test_library_job_overwrites_the_liars_and_keeps_finite():
    t = _trainer(_cfg(max_steps=6))
    losses = [t.train_step()["loss"] for _ in range(6)]
    assert all(math.isfinite(x) for x in losses)
    assert not torch.equal(t.engine.ps.mimic_z, torch.from_numpy(A.mimic_z0([(s.offset, s.numel) for s in t.engine.layout.specs],
                                                                             t.engine.layout.total)))
    ti = _trainer(_cfg(err_mode="ipm", mimic_warmup=None, attack_eps=0.5, max_steps=4))
    assert all(math.isfinite(ti.train_step()["loss"]) for _ in range(4))


def test_ipm_library_rows_equal_the_oracle():
    t = _trainer(_cfg(err_mode="ipm", mimic_warmup=None, attack_eps=0.3, mode="trimmed_mean"))
    eng = t.engine
    g = torch.Generator().manual_seed(3)
    eng.slots.copy_(torch.randn(eng.slots.shape, generator=g))
    eng.slots[:, ~torch.from_numpy(eng.layout.valid_mask())] = 0
    before = eng.slots.numpy().copy()
    eng._ps_attack(5)
    liars = [int(w) - 1 for w in eng.schedule.ranks[5]]
    ref = A.ps_attack(before, liars, "ipm", [(s.offset, s.numel) for s in eng.layout.specs], z=0.3)
    assert np.array_equal(_bits(eng.slots.numpy()), _bits(ref))


# ------------------------------------------------------------------------------------------------ checkpoint / resume
@pytest.mark.parametrize("kw", [dict(), dict(approach="maj_vote", mode="maj_vote", num_workers=6, group_size=3, worker_fail=1)])
def test_checkpoint_in_the_warm_up_resumes_bit_for_bit(tmp_path, kw):
    d = str(tmp_path) + "/"
    kw = dict(kw, train_dir=d, max_steps=8, mimic_warmup=5)
    t = _trainer(_cfg(eval_freq=2, **kw))
    t.fit(8)
    final, m, z = t.engine.master_params().clone(), t.engine.ps.mimic_m.clone(), t.engine.ps.mimic_z.clone()
    saved = load_checkpoint(d + "model_step_2")["opt_state"]
    assert {"mimic_m", "mimic_z"} <= set(saved)
    t2 = _trainer(_cfg(eval_freq=10 ** 6, checkpoint_step=2, **kw))
    assert t2.step == 3
    for _ in range(6):
        t2.train_step()
    assert torch.equal(t2.engine.master_params(), final)
    assert torch.equal(t2.engine.ps.mimic_m, m) and torch.equal(t2.engine.ps.mimic_z, z)


def test_other_checkpoints_have_no_mimic_state_and_mismatched_resumes_are_rejected(tmp_path):
    d0, d1 = str(tmp_path / "alie") + "/", str(tmp_path / "mimic") + "/"
    _trainer(_cfg(err_mode="ipm", mimic_warmup=None, train_dir=d0, eval_freq=2, max_steps=2)).fit(2)
    _trainer(_cfg(train_dir=d1, eval_freq=2, max_steps=2)).fit(2)
    assert load_checkpoint(d0 + "model_step_2")["opt_state"] == {}
    with pytest.raises(ValueError, match="holds no mimic state"):
        _trainer(_cfg(train_dir=d0, checkpoint_step=2))
    with pytest.raises(ValueError, match="holds the mimic attack's state"):
        _trainer(_cfg(err_mode="ipm", mimic_warmup=None, train_dir=d1, checkpoint_step=2))


# ------------------------------------------------------------------------------------------------ multi-process
def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _job(err_mode):
    extra = dict(mimic_warmup=2) if err_mode == "mimic" else dict(mimic_warmup=None)
    return _cfg(mode="trimmed_mean", num_workers=5, worker_fail=1, err_mode=err_mode, batch_size=8, synthetic_size=128,
                max_steps=6, **extra)


def _gloo_proc(rank, world, port, err_mode, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    torch.set_num_threads(2)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    t = Trainer(_job(err_mode), rank=rank, world=world, device=CPU, quiet=True)
    for _ in range(4):
        t.train_step()
    q.put((rank, hashlib.sha256(t.engine.master_params().numpy().tobytes()).hexdigest()))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("err_mode", ["ipm", "mimic"])
def test_multi_process_job_equals_the_single_process_job(err_mode):
    """1 PS + 5 workers on 2 Gloo processes: the PS's parameters after 4 steps (mimic: across its 2 warm-up steps) are
    bit-identical to the same job in one process."""
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
        single = _trainer(_job(err_mode))
        for _ in range(4):
            single.train_step()
    finally:
        torch.set_num_threads(threads)
    assert res[0] == hashlib.sha256(single.engine.master_params().numpy().tobytes()).hexdigest()
