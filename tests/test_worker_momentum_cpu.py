"""Worker-side momentum (``--worker-momentum``) on the CPU: the fp32 oracle against a torch restatement and an fp64 recursion,
the configuration, the library-op engine over Gloo step by step against the oracle, the majority vote staying exact, checkpoint
/ resume, and a multi-process Gloo job against the single-process one."""
import argparse
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from draco_b200 import JobConfig
from draco_b200.codes import oracle
from draco_b200.config import add_fit_args, config_from_args
from draco_b200.parallel.trainer import Trainer
from draco_b200.utils.checkpoint import load_checkpoint

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _cfg(**kw):
    base = dict(network="LeNet", dataset="MNIST", batch_size=16, max_steps=12, transport="gloo", lr=0.05, momentum=0.0,
                synthetic_size=512, eval_freq=10 ** 6, compress_grad="None", approach="baseline", mode="normal", num_workers=5,
                worker_fail=0, err_mode="none", worker_momentum=0.9)
    base.update(kw)
    return JobConfig(**base)


def _trainer(cfg):
    return Trainer(cfg, rank=0, world=1, device=torch.device("cpu"), quiet=True)


# ------------------------------------------------------------------------------------------------ oracle
def _torch_step(m, g, beta):
    b, c = oracle.worker_momentum_coefficients(beta)
    m = m.clone()
    m.mul_(b)
    m.add_(g * c)
    return m


@pytest.mark.parametrize("beta", [0.0, 0.5, 0.9, 0.99, 0.1])
def test_oracle_is_bit_equal_to_the_fp32_torch_restatement(beta):
    rng = np.random.default_rng(int(beta * 100))
    m = np.zeros(4096, dtype=np.float32)
    mt = torch.zeros(4096)
    for step in range(20):
        g = (rng.normal(size=4096) * 10.0 ** rng.integers(-6, 4, size=4096)).astype(np.float32)
        g[:7] = [0.0, -0.0, 1e-45, -1e-45, 3.4e38, -3.4e38, 1.0]
        m = oracle.worker_momentum(m, g, beta)
        mt = _torch_step(mt, torch.from_numpy(g), beta)
        assert m.dtype == np.float32
        assert np.array_equal(m.view(np.int32), mt.numpy().view(np.int32)), step


def test_oracle_widens_bf16_exactly_and_rounds_each_op():
    g16 = torch.randn(1000).to(torch.bfloat16)
    g = g16.float().numpy()                                     # bf16 -> fp32 is exact
    m = np.random.default_rng(0).normal(size=1000).astype(np.float32)
    b, c = oracle.worker_momentum_coefficients(0.9)
    assert b == float(np.float32(0.9)) and c == float(np.float32(1.0 - 0.9)) and c != float(np.float32(1.0) - np.float32(0.9))
    want = np.float32(b) * m
    want = want + np.float32(c) * g
    assert np.array_equal(oracle.worker_momentum(m, g, 0.9), want)
    # no fused multiply-add: the sum of the rounded products, not the rounded exact sum
    fma = (np.float64(b) * m.astype(np.float64) + np.float64(c) * g.astype(np.float64)).astype(np.float32)
    assert not np.array_equal(fma, want)


def test_oracle_tracks_the_fp64_recursion_over_50_steps():
    rng = np.random.default_rng(1)
    beta = 0.9
    m32 = np.zeros(2048, dtype=np.float32)
    m64 = np.zeros(2048)
    gmax = 0.0
    for _ in range(50):
        g = rng.normal(size=2048).astype(np.float32)
        gmax = max(gmax, float(np.abs(g).max()))
        m32 = oracle.worker_momentum(m32, g, beta)
        m64 = beta * m64 + (1.0 - beta) * g.astype(np.float64)
    assert np.abs(m32 - m64).max() <= 1e-5 * gmax


# ------------------------------------------------------------------------------------------------ configuration
def test_configuration_default_flag_and_rejections():
    assert JobConfig().worker_momentum == 0.0
    ap = add_fit_args(argparse.ArgumentParser())
    assert ap.parse_args([]).worker_momentum == 0.0
    cfg = config_from_args(ap.parse_args(["--worker-momentum", "0.9", "--momentum", "0", "--approach", "baseline", "--mode",
                                          "coordinate_median", "--worker-fail", "1", "--num-workers", "5"])).resolve(1)
    assert cfg.worker_momentum == 0.9 and cfg.momentum == 0.0

    def bad(match, **kw):
        with pytest.raises(ValueError, match=match):
            _cfg(**kw).resolve(1)
    for beta in (1.0, -0.1, 1.5, float("nan")):
        bad(r"--worker-momentum must lie in \[0, 1\)", worker_momentum=beta)
    bad("under --approach cyclic: its decode recovers the exact sum", approach="cyclic", worker_fail=1)
    bad("--transport nccl_flat pushes the raw gradient", transport="nccl_flat")
    bad("--err-mode omniscient replaces the liars' push", approach="maj_vote", mode="maj_vote", group_size=5, worker_fail=1,
        err_mode="omniscient")
    # beta = 0 is off: every combination above is accepted as before
    _cfg(worker_momentum=0.0, approach="cyclic", worker_fail=1).resolve(1)
    _cfg(worker_momentum=0.0, transport="nccl_flat").resolve(1)
    for approach, mode in (("baseline", "bulyan"), ("maj_vote", "maj_vote"), ("detox", "coordinate_median"),
                           ("nnm", "coordinate_median")):
        for err in ("rev_grad", "alie", "minmax", "constant", "random"):
            _cfg(approach=approach, mode=mode, num_workers=15, worker_fail=3, group_size=3, err_mode=err,
                 transport="nvl").resolve(1)


# ------------------------------------------------------------------------------------------------ library-op engine
@pytest.mark.parametrize("err", ["rev_grad", "constant"])
def test_gloo_slots_hold_the_state_or_the_attack_on_it(err):
    t = _trainer(_cfg(worker_fail=2, err_mode=err, mode="coordinate_median"))
    eng = t.engine
    assert set(eng.worker_momentum) == {1, 2, 3, 4, 5}
    valid = torch.from_numpy(eng.layout.valid_mask())           # the attack rewrites the tensors, not the padding between them
    liars_seen = 0
    for step in range(1, 7):
        t.train_step()
        for w, m in eng.worker_momentum.items():
            slot = eng.slots[w - 1]
            if eng.schedule.is_adversary(w, step):
                liars_seen += 1
                sent = m * -100.0 if err == "rev_grad" else torch.full_like(m, -100.0)
                assert torch.equal(slot[valid], sent[valid]) and torch.equal(slot[~valid], m[~valid]), (step, w)
            else:
                assert torch.equal(slot, m), (step, w)
    assert liars_seen > 0


def test_gloo_states_equal_the_oracle_on_each_workers_own_gradient():
    """Every worker's state after every step is oracle(previous state, that worker's flat gradient), bit for bit."""
    t = _trainer(_cfg(worker_fail=1, err_mode="rev_grad"))
    eng, wc = t.engine, t.engine.worker
    grads = {}
    real_fb = wc.forward_backward

    def fb(w, step_host=None, **kw):
        real_fb(w, step_host, **kw)
        grads[w] = wc.flat_gradient(0).numpy().copy()
    wc.forward_backward = fb
    prev = {w: np.zeros(eng.layout.total, dtype=np.float32) for w in eng.worker_momentum}
    for step in range(1, 6):
        t.train_step()
        for w, m in eng.worker_momentum.items():
            want = oracle.worker_momentum(prev[w], grads[w], 0.9)
            assert np.array_equal(m.numpy().view(np.int32), want.view(np.int32)), (step, w)
            prev[w] = want


def test_worker_momentum_trains():
    t = _trainer(_cfg(lr=0.1))                                  # baseline mean, beta = 0.9, no PS momentum
    losses = [t.train_step()["loss"] for _ in range(12)]
    assert losses[-1] < losses[0], losses
    assert torch.isfinite(t.engine.master_params()).all()


def test_beta_zero_keeps_no_state_and_runs_the_plain_job():
    a = _trainer(_cfg(worker_momentum=0.0, worker_fail=1, err_mode="rev_grad", mode="coordinate_median"))
    assert a.engine.worker_momentum == {}
    for _ in range(3):
        a.train_step()
    b = _trainer(_cfg(worker_momentum=0.5, worker_fail=1, err_mode="rev_grad", mode="coordinate_median"))
    for _ in range(3):
        b.train_step()
    assert not torch.equal(a.engine.master_params(), b.engine.master_params())


def test_vote_stays_exact_with_worker_momentum():
    """One sign-flip liar in a group of 3: the vote must return the honest holders' pushed momentum every step.  If a liar's
    state absorbed its attack, its later honest pushes would differ from the other holders' and the group would lose its
    majority."""
    kw = dict(approach="maj_vote", mode="maj_vote", group_size=3, num_workers=7, momentum=0.5)
    clean = _trainer(_cfg(worker_fail=0, err_mode="none", **kw))
    dirty = _trainer(_cfg(worker_fail=1, err_mode="rev_grad", **kw))
    for _ in range(8):
        clean.train_step()
        dirty.train_step()
    assert torch.equal(clean.engine.master_params(), dirty.engine.master_params())
    for w in range(1, 8):
        assert torch.equal(clean.engine.worker_momentum[w], dirty.engine.worker_momentum[w])
    mean = _trainer(_cfg(worker_fail=1, err_mode="rev_grad", **dict(kw, mode="normal")))
    for _ in range(8):
        mean.train_step()
    assert not torch.allclose(clean.engine.master_params(), mean.engine.master_params(), atol=1e-3)


# ------------------------------------------------------------------------------------------------ checkpoint / resume
def test_checkpoint_resume_is_bit_for_bit(tmp_path):
    d = str(tmp_path) + "/"
    kw = dict(mode="coordinate_median", worker_fail=1, err_mode="rev_grad", momentum=0.9, train_dir=d, max_steps=6)
    t = _trainer(_cfg(eval_freq=3, **kw))
    t.fit(6)
    final = t.engine.master_params().clone()
    states = {w: m.clone() for w, m in t.engine.worker_momentum.items()}
    blob = load_checkpoint(d + "model_step_3")
    L = t.engine.layout
    assert sorted(blob["worker_momentum"]) == [1, 2, 3, 4, 5]
    for w, per in blob["worker_momentum"].items():
        assert set(per) == {s.name for s in L.specs}
        assert all(v.dtype == torch.float32 for v in per.values())
        assert any(float(v.abs().sum()) > 0 for v in per.values())
    t2 = _trainer(_cfg(eval_freq=10 ** 6, checkpoint_step=3, **kw))
    assert t2.step == 4
    for _ in range(3):
        t2.train_step()
    assert torch.equal(t2.engine.master_params(), final)
    for w, m in states.items():
        assert torch.equal(t2.engine.worker_momentum[w], m)


def test_checkpoints_without_worker_momentum_have_no_key_and_mismatched_resumes_are_rejected(tmp_path):
    d0, d1 = str(tmp_path / "plain") + "/", str(tmp_path / "wm") + "/"
    _trainer(_cfg(worker_momentum=0.0, train_dir=d0, eval_freq=2, max_steps=2)).fit(2)
    _trainer(_cfg(worker_momentum=0.9, train_dir=d1, eval_freq=2, max_steps=2)).fit(2)
    assert "worker_momentum" not in load_checkpoint(d0 + "model_step_2")
    assert "worker_momentum" in load_checkpoint(d1 + "model_step_2")
    with pytest.raises(ValueError, match="holds no worker momentum"):
        _trainer(_cfg(worker_momentum=0.9, train_dir=d0, checkpoint_step=2))
    with pytest.raises(ValueError, match="holds worker momentum"):
        _trainer(_cfg(worker_momentum=0.0, train_dir=d1, checkpoint_step=2))


# ------------------------------------------------------------------------------------------------ multi-process
def test_multi_process_job_equals_the_single_process_job(tmp_path):
    """1 PS + 2 worker processes over Gloo against one process hosting everything: the same checkpoint at step 3, the
    gathered worker momenta included."""
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""), OMP_NUM_THREADS="1")
    common = ["-m", "draco_b200.cli.distributed_nn", "--no-cuda", "--network", "LeNet", "--dataset", "MNIST", "--num-workers", "5",
              "--batch-size", "8", "--max-steps", "3", "--eval-freq", "3", "--synthetic-size", "128", "--log-interval", "1",
              "--compress-grad", "None", "--approach", "baseline", "--mode", "coordinate_median", "--worker-fail", "1",
              "--err-mode", "rev_grad", "--worker-momentum", "0.9", "--momentum", "0"]
    blobs = []
    for name, extra in (("multi", ["--launch", "3", "--master-port", "29761"]), ("single", [])):
        d = str(tmp_path / name) + "/"
        r = subprocess.run([sys.executable, *common, "--train-dir", d, *extra], capture_output=True, text=True, timeout=420,
                           env=env, cwd=ROOT)
        assert r.returncode == 0, (r.stdout[-2000:], r.stderr[-3000:])
        blobs.append(load_checkpoint(d + "model_step_3"))
    multi, single = blobs
    assert sorted(multi["worker_momentum"]) == sorted(single["worker_momentum"]) == [1, 2, 3, 4, 5]
    for k, v in single["state_dict"].items():
        assert torch.equal(multi["state_dict"][k], v), k
    for w, per in single["worker_momentum"].items():
        for k, v in per.items():
            assert torch.equal(multi["worker_momentum"][w][k], v), (w, k)
