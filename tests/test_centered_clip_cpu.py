"""Centered clipping (``--mode centered_clip --clip-tau``) on the CPU: the oracle on hand-worked cases and against the paper's
formula in fp64, the configuration, the library-op PS against the oracle over several steps (baseline and DETOX), Gloo jobs
(single- against multi-process), checkpoint / resume, and the fused PS's launch sequence per bucket."""
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
from draco_b200.models import build_model
from draco_b200.ops import kernels as K
from draco_b200.parallel.arena import ArenaLayout
from draco_b200.parallel.ps import FusedPS, TorchPS, build_codes, rule_plan
from draco_b200.parallel.trainer import Trainer
from draco_b200.utils.checkpoint import load_checkpoint

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CPU = torch.device("cpu")


def _bits(x):
    return np.asarray(x, dtype=np.float32).view(np.int32)


def _cfg(**kw):
    base = dict(network="LeNet", dataset="MNIST", batch_size=16, max_steps=12, transport="gloo", lr=0.05, momentum=0.0,
                synthetic_size=512, eval_freq=10 ** 6, compress_grad="None", approach="baseline", mode="centered_clip",
                clip_tau=0.5, num_workers=5, worker_fail=1, err_mode="rev_grad")
    base.update(kw)
    return JobConfig(**base)


def _trainer(cfg):
    return Trainer(cfg, rank=0, world=1, device=CPU, quiet=True)


# ------------------------------------------------------------------------------------------------ oracle
def test_tau_above_every_distance_gives_the_plain_mean_around_the_centre():
    rng = np.random.default_rng(0)
    X = rng.normal(size=(5, 300)).astype(np.float32)
    v = rng.normal(size=300).astype(np.float32) * 0.1
    w = oracle.centered_clip_weights(X, v, 1e6)
    assert np.array_equal(w, np.full(5, np.float32(0.2)))
    g = oracle.centered_clip(X, v, 1e6)
    want = v.astype(np.float64) + (X.astype(np.float64) - v).mean(0)
    assert np.abs(g - want).max() <= 1e-6 * np.abs(want).max()


def test_a_row_equal_to_the_centre_has_weight_one_over_n_and_adds_nothing():
    v = np.array([1.0, -2.0, 3.0], dtype=np.float32)
    X = np.stack([v, v + 100.0]).astype(np.float32)
    w = oracle.centered_clip_weights(X, v, 1.0)
    assert w[0] == np.float32(0.5)
    d = np.sqrt(3 * 100.0 ** 2)
    assert w[1] == np.float32(1.0 / d / 2)
    g = oracle.centered_clip(X, v, 1.0)
    assert np.allclose(g, v + 100.0 * w[1], rtol=1e-6)


@pytest.mark.parametrize("bad", [np.nan, np.inf, -np.inf])
def test_a_nan_or_inf_row_gets_weight_zero_and_never_reaches_the_result(bad):
    rng = np.random.default_rng(1)
    X = rng.normal(size=(4, 64)).astype(np.float32)
    v = np.zeros(64, dtype=np.float32)
    X[2, 7] = bad
    w = oracle.centered_clip_weights(X, v, 2.0)
    assert w[2] == 0 and (w[[0, 1, 3]] > 0).all()
    g = oracle.centered_clip(X, v, 2.0)
    assert np.isfinite(g).all()
    assert np.array_equal(_bits(g), _bits(oracle.centered_clip(X[[0, 1, 3]], v, 2.0, weights=w[[0, 1, 3]])))


def test_an_overflowing_distance_gets_weight_zero():
    X = np.array([[3e38, -3e38], [1.0, 1.0]], dtype=np.float32)
    v = np.array([-3e38, 3e38], dtype=np.float32)
    w = oracle.centered_clip_weights(X, v, 1.0)             # (6e38)^2 is finite in fp64: only a real +Inf / NaN is dropped
    assert w[0] > 0 and w[1] > 0
    X[0, 0] = np.inf
    assert oracle.centered_clip_weights(X, v, 1.0)[0] == 0


def test_a_single_row_is_clipped_to_tau():
    x = np.array([[3.0, 4.0]], dtype=np.float32)
    v = np.zeros(2, dtype=np.float32)
    assert np.allclose(oracle.centered_clip(x, v, 1.0), [0.6, 0.8], rtol=1e-7)
    assert np.array_equal(oracle.centered_clip(x, v, 10.0), x[0])


def test_a_far_row_moves_the_result_by_at_most_tau_over_n():
    rng = np.random.default_rng(2)
    X = rng.normal(size=(7, 500)).astype(np.float32)
    v = rng.normal(size=500).astype(np.float32)
    tau = 0.7
    g0 = oracle.centered_clip(X, v, tau)
    for scale in (1e3, 1e10, 1e30):
        Y = X.copy()
        Y[3] = scale * rng.normal(size=500).astype(np.float32)
        g = oracle.centered_clip(Y, v, tau)
        contrib = lambda Z, g_: g_.astype(np.float64) - v            # noqa: E731
        # the far row's own term is bounded by tau / n in norm; the other rows' terms are unchanged
        diff = np.linalg.norm(contrib(Y, g) - contrib(X, g0))
        assert diff <= 2 * tau / 7 * (1 + 1e-5)


def test_oracle_matches_the_papers_formula_in_fp64():
    rng = np.random.default_rng(3)
    for n in (1, 2, 5, 16):
        for _ in range(5):
            X = (rng.normal(size=(n, 1000)) * 10.0 ** rng.integers(-3, 3, size=(n, 1))).astype(np.float32)
            v = rng.normal(size=1000).astype(np.float32)
            tau = float(10.0 ** rng.uniform(-2, 2))
            X64, v64 = X.astype(np.float64), v.astype(np.float64)
            want = v64 + sum((x - v64) * min(1.0, tau / np.linalg.norm(x - v64)) for x in X64) / n
            g = oracle.centered_clip(X, v, tau)
            assert np.abs(g - want).max() <= 1e-5 * max(np.abs(want).max(), 1e-30), (n, tau)


def test_fma_f32_rounds_once():
    # 1 + 2^-24 needs 25 bits: fma keeps the low part the separate product would lose
    a, b, c = np.float32(1 + 2 ** -12), np.float32(1 + 2 ** -12), np.float32(-1.0)
    assert oracle.fma_f32(a, b, c) == np.float32(2 ** -11 + 2 ** -24)
    assert np.float32(a * b) + c != np.float32(2 ** -11 + 2 ** -24)
    rng = np.random.default_rng(4)
    a, b, c = (rng.normal(size=(3, 10000)) * 10.0 ** rng.integers(-8, 8, size=(3, 10000))).astype(np.float32)
    got = oracle.fma_f32(a, b, c)
    exact = a.astype(np.longdouble) * b + c                  # 64-bit significand where the platform has it: a loose check
    assert np.allclose(got, exact.astype(np.float32), rtol=1.5e-7, atol=0)


# ------------------------------------------------------------------------------------------------ configuration
def test_configuration_accepts_the_flag_and_rejects_every_misuse():
    ap = add_fit_args(argparse.ArgumentParser())
    assert ap.parse_args([]).clip_tau is None
    cfg = config_from_args(ap.parse_args(["--approach", "baseline", "--mode", "centered_clip", "--clip-tau", "0.25",
                                          "--num-workers", "5", "--worker-fail", "2", "--transport", "gloo"])).resolve(1)
    assert cfg.clip_tau == 0.25 and rule_plan(cfg).rule == "centered_clip" and rule_plan(cfg).pipelined
    plan = rule_plan(_cfg(approach="detox", group_size=3, num_workers=15, worker_fail=3).resolve(1))
    assert (plan.rule, plan.source, plan.base, plan.rows, plan.opt_mode) == ("detox_centered_clip", "detox", "centered_clip", 5,
                                                                              "centered_clip")

    def bad(match, **kw):
        with pytest.raises(ValueError, match=match):
            _cfg(**kw).resolve(1)
    for approach in ("baseline", "detox"):
        bad("needs --clip-tau", approach=approach, clip_tau=None, group_size=1)
    for tau in (0.0, -1.0, float("inf"), float("nan")):
        bad("needs --clip-tau, a finite radius > 0", clip_tau=tau)
    bad("--clip-tau sets centered clipping's radius", mode="coordinate_median")
    bad("--clip-tau sets centered clipping's radius", approach="maj_vote", mode="maj_vote", group_size=5)
    bad("--clip-tau sets centered clipping's radius", approach="maj_vote", mode="normal", group_size=5)
    bad("--clip-tau sets centered clipping's radius", approach="cyclic", mode="normal")
    bad("runs under --approach baseline", approach="cyclic", clip_tau=None)
    bad("runs under --approach baseline", approach="maj_vote", group_size=5, clip_tau=None)
    bad("--approach nnm takes --mode", approach="nnm")
    bad("num_workers > 2\\*worker_fail", num_workers=4, worker_fail=2)
    bad("groups > 2\\*b_G", approach="detox", num_workers=6, group_size=3, worker_fail=2)   # G = 2, b_G = 1
    bad("handles at most 16 rows", num_workers=17, transport="nvl")
    bad("handles at most 16 groups", approach="detox", num_workers=17, group_size=1, transport="nvl")
    bad("--transport nccl_flat runs the plain mean", transport="nccl_flat", err_mode="none")
    # what the issue's composition list allows
    for err in ("rev_grad", "alie", "minmax", "constant", "random", "omniscient", "none"):
        _cfg(num_workers=15, worker_fail=3, err_mode=err, transport="nvl").resolve(1)
    _cfg(approach="detox", num_workers=15, group_size=3, worker_fail=3, transport="nvl", worker_momentum=0.9).resolve(1)
    _cfg(approach="detox", num_workers=5, group_size=1, worker_fail=1).resolve(1)
    _cfg(optimizer="adam", amsgrad=True, compress_grad="compress").resolve(1)


# ------------------------------------------------------------------------------------------------ library-op PS
def _layout():
    return ArenaLayout.from_model(build_model("LeNet"), bf16=False, channels_last=True)


def _slots(g, cfg, L, groups):
    S = torch.randn(cfg.num_workers, L.total, generator=g)
    S *= torch.rand(cfg.num_workers, 1, generator=g) * 4
    if groups is not None:                                   # replicas agree, then the first worker_fail workers lie
        for grp in groups.groups:
            for w in grp[1:]:
                S[w - 1] = S[grp[0] - 1]
    S[: cfg.worker_fail] = torch.randn(cfg.worker_fail, L.total, generator=g) * 50
    return S


@pytest.mark.parametrize("approach,P,f,r", [("baseline", 5, 1, 1), ("baseline", 16, 7, 1), ("detox", 15, 3, 3),
                                             ("detox", 5, 1, 1)])
def test_torch_ps_equals_the_oracle_over_several_steps(approach, P, f, r):
    """The carried centre included: every step's result, and the centre it leaves, bit for bit."""
    cfg = _cfg(approach=approach, num_workers=P, worker_fail=f, group_size=r, clip_tau=3.0).resolve(1)
    L = _layout()
    groups, code = build_codes(cfg)
    ps = TorchPS(cfg, L, CPU, L.new_arena(CPU), groups, code)
    g = torch.Generator().manual_seed(P * 10 + f)
    centers = [np.zeros(s.numel, dtype=np.float32) for s in L.specs]
    for step in range(4):
        S = _slots(g, cfg, L, groups)
        if step == 2:
            S[f, 3] = float("nan")                           # an honest row turns NaN in the first tensor
        out = ps.aggregate(S)
        for i, spec in enumerate(L.specs):
            X = S[:, spec.offset: spec.offset + spec.numel].numpy()
            if approach == "detox":
                X = X[oracle.detox_winner_slots(X, groups.groups)]
            want = oracle.centered_clip(X, centers[i], cfg.clip_tau)
            assert np.array_equal(_bits(out[i].numpy()), _bits(want)), (step, spec.name)
            assert np.array_equal(_bits(ps.cc_center[spec.offset: spec.offset + spec.numel].numpy()), _bits(want))
            centers[i] = want
        assert np.isfinite(np.concatenate(centers)).all()


def test_torch_ps_passes_the_optimizer_mode():
    cfg = _cfg().resolve(1)
    L = _layout()
    ps = TorchPS(cfg, L, CPU, L.new_arena(CPU), None, None)
    seen = {}

    class _Opt:
        def step(self, grads, mode):
            seen["mode"] = mode
    ps.optimizer = _Opt()
    ps.step(torch.randn(5, L.total))
    assert seen["mode"] == "centered_clip"


# ------------------------------------------------------------------------------------------------ Gloo jobs
def test_centered_clip_holds_against_rev_grad_where_the_mean_does_not():
    kw = dict(num_workers=7, worker_fail=2, lr=0.05, clip_tau=1.0)
    clean = _trainer(_cfg(err_mode="none", **kw))
    cc = _trainer(_cfg(err_mode="rev_grad", **kw))
    mean = _trainer(_cfg(err_mode="rev_grad", mode="normal", **dict(kw, clip_tau=None)))
    runs = {"clean": clean, "cc": cc, "mean": mean}
    loss = {k: [t.train_step()["loss"] for _ in range(12)][-1] for k, t in runs.items()}
    assert np.isfinite(loss["cc"]) and loss["cc"] < loss["clean"] * 1.5, loss
    dist = {k: float((t.engine.master_params() - clean.engine.master_params()).norm()) for k, t in runs.items()}
    assert not dist["mean"] < 10 * dist["cc"], dist           # the mean leaves the clean trajectory (or diverges to NaN)


def test_worker_momentum_and_adam_compose():
    for kw in (dict(worker_momentum=0.9), dict(optimizer="adam", lr=1e-3), dict(optimizer="adam", amsgrad=True, lr=1e-3),
               dict(compress_grad="compress")):
        t = _trainer(_cfg(**kw))
        for _ in range(3):
            m = t.train_step()
        assert np.isfinite(m["loss"]) and torch.isfinite(t.engine.master_params()).all(), kw
        assert float(t.engine.ps.cc_center.abs().sum()) > 0


# ------------------------------------------------------------------------------------------------ checkpoint / resume
@pytest.mark.parametrize("kw", [dict(), dict(momentum=0.9, worker_momentum=0.9), dict(optimizer="adam", lr=1e-3),
                                dict(approach="detox", group_size=3, num_workers=6, worker_fail=1)])
def test_checkpoint_resume_is_bit_for_bit(tmp_path, kw):
    d = str(tmp_path) + "/"
    kw = dict(kw, train_dir=d, max_steps=6)
    t = _trainer(_cfg(eval_freq=3, **kw))
    t.fit(6)
    final, center = t.engine.master_params().clone(), t.engine.ps.cc_center.clone()
    blob = load_checkpoint(d + "model_step_3")
    saved = blob["opt_state"]["cc_center"]
    assert set(saved) == {s.name for s in t.engine.layout.specs} and any(float(v.abs().sum()) > 0 for v in saved.values())
    t2 = _trainer(_cfg(eval_freq=10 ** 6, checkpoint_step=3, **kw))
    assert t2.step == 4
    for _ in range(3):
        t2.train_step()
    assert torch.equal(t2.engine.master_params(), final)
    assert torch.equal(t2.engine.ps.cc_center, center)


def test_other_checkpoints_have_no_centre_and_mismatched_resumes_are_rejected(tmp_path):
    d0, d1 = str(tmp_path / "plain") + "/", str(tmp_path / "cc") + "/"
    _trainer(_cfg(mode="coordinate_median", clip_tau=None, train_dir=d0, eval_freq=2, max_steps=2)).fit(2)
    _trainer(_cfg(train_dir=d1, eval_freq=2, max_steps=2)).fit(2)
    assert load_checkpoint(d0 + "model_step_2")["opt_state"] == {}
    assert "cc_center" in load_checkpoint(d1 + "model_step_2")["opt_state"]
    with pytest.raises(ValueError, match="holds no centre"):
        _trainer(_cfg(train_dir=d0, checkpoint_step=2))
    with pytest.raises(ValueError, match="holds centered clipping's centre"):
        _trainer(_cfg(mode="coordinate_median", clip_tau=None, train_dir=d1, checkpoint_step=2))


# ------------------------------------------------------------------------------------------------ multi-process
@pytest.mark.parametrize("err,port", [("rev_grad", 29771), ("alie", 29772)])
def test_multi_process_job_equals_the_single_process_job(tmp_path, err, port):
    """1 PS + 2 worker processes over Gloo against one process hosting everything, with worker momentum: the same parameters
    and the same centre at step 3."""
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""), OMP_NUM_THREADS="1")
    common = ["-m", "draco_b200.cli.distributed_nn", "--no-cuda", "--network", "LeNet", "--dataset", "MNIST", "--num-workers", "5",
              "--batch-size", "8", "--max-steps", "3", "--eval-freq", "3", "--synthetic-size", "128", "--log-interval", "1",
              "--compress-grad", "None", "--approach", "baseline", "--mode", "centered_clip", "--clip-tau", "0.1",
              "--worker-fail", "1", "--err-mode", err, "--worker-momentum", "0.9", "--momentum", "0"]
    blobs = []
    for name, extra in (("multi", ["--launch", "3", "--master-port", str(port)]), ("single", [])):
        d = str(tmp_path / name) + "/"
        r = subprocess.run([sys.executable, *common, "--train-dir", d, *extra], capture_output=True, text=True, timeout=420,
                           env=env, cwd=ROOT)
        assert r.returncode == 0, (r.stdout[-2000:], r.stderr[-3000:])
        blobs.append(load_checkpoint(d + "model_step_3"))
    multi, single = blobs
    for key in ("state_dict",):
        for k, v in single[key].items():
            assert torch.equal(multi[key][k], v), k
    for k, v in single["opt_state"]["cc_center"].items():
        assert torch.equal(multi["opt_state"]["cc_center"][k], v), k
        assert float(v.abs().sum()) > 0


# ------------------------------------------------------------------------------------------------ fused PS launch sequence
KEYS = ("tile_range", "tensor_range", "rows", "select", "center", "weights", "K", "flags")


def _record_launches(cfg, monkeypatch, buckets):
    """FusedPS.enqueue_step with every launcher replaced by a recorder: (launcher, its row count, the keywords of KEYS) per call,
    the PS's own tensors named."""
    L = _layout()
    calls, named = [], {}

    def rec(name, ret=None):
        def f(*args, **kw):
            vals = {k: named.get(id(v), v) if isinstance(v, torch.Tensor) else v for k, v in kw.items() if k in KEYS}
            n = args[3] if name == "centered_clip_dist" else args[1] if name == "centered_clip_weights" else None
            calls.append((name, n, vals))
            return ret
        return f
    for name in ("vote", "aggregate_update", "krum_select", "bulyan_select", "geometric_median_weights", "nnm_mix", "nnm_fold",
                 "centered_clip_dist", "centered_clip_weights", "centered_clip_update"):
        monkeypatch.setattr(K, name, rec(name))
    monkeypatch.setattr(K, "ps_attack", rec("ps_attack", 1))
    groups, code = build_codes(cfg)
    P = cfg.num_workers
    ps = FusedPS(cfg, L, CPU, L.new_arena(CPU), torch.zeros(P, L.total), groups, code, adv_bitmap=torch.zeros(8, dtype=torch.int32),
                 adv_len=8)
    named.update({id(ps.cc_center): "center", id(ps.cc_weights): "weights"})
    if cfg.approach == "detox":
        named[id(ps.winner_slot)] = "winner_slot"
    kw = dict(buckets=buckets, wait_bucket=lambda b: calls.append(("wait", b)) or 1) if buckets else {}
    n = ps.enqueue_step(torch.ones(1, dtype=torch.int64), mc_params=None, dst=[4096], flags=[16, 32],
                        before_update=lambda: calls.append(("before_update",)) or 1, **kw)
    return ps, calls, n


@pytest.mark.parametrize("approach", ["baseline", "detox"])
@pytest.mark.parametrize("bucketed", [False, True])
def test_fused_ps_launches_dist_weights_update_per_bucket(monkeypatch, approach, bucketed):
    cfg = _cfg(approach=approach, num_workers=15, worker_fail=3, group_size=3, transport="nvl", err_mode="alie").resolve(1)
    L = _layout()
    buckets = [(0, 3, [0, 1]), (3, 7, [2, 3, 4]), (7, 12, list(range(5, L.ntensors)))] if bucketed else None
    ps, calls, n = _record_launches(cfg, monkeypatch, buckets)
    assert ps.plan.pipelined and ps.cc_center.shape == (L.total,) and "cc_center" in ps.opt_state
    assert ps.cc_partials.shape == (L.ntiles, ps.plan.rows) and ps.cc_weights.shape == (L.ntensors, ps.plan.rows)
    rows = "winner_slot" if approach == "detox" else None
    ranges = [((t0, t1), (min(i), max(i) + 1)) for t0, t1, i in buckets] if bucketed else [(None, None)]
    want = []
    for bi, (tiles, tensors) in enumerate(ranges):
        last = bi == len(ranges) - 1
        if bucketed:
            want.append(("wait", bi))
        want.append(("ps_attack", None, {"tile_range": tiles, "tensor_range": tensors}))
        if approach == "detox":
            want.append(("vote", None, {"tile_range": tiles, "tensor_range": tensors}))
        want.append(("centered_clip_dist", ps.plan.rows, {"rows": rows, "tile_range": tiles}))
        want.append(("centered_clip_weights", ps.plan.rows, {"tensor_range": tensors}))
        if last:
            want.append(("before_update",))
        want.append(("centered_clip_update", None, {"center": "center", "weights": "weights", "K": ps.plan.rows, "select": rows,
                                                     "tile_range": tiles, "flags": [16, 32] if last else []}))
    assert calls == want
    assert n == len(ranges) * (int(bucketed) + 1 + (2 if approach == "detox" else 0) + 3) + 1
