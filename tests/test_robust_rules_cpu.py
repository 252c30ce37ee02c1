"""Coordinate-wise median, coordinate-wise trimmed mean and multi-Krum on the CPU: the fp64 oracles on hand-worked cases, the
library-op PS against the oracles, the configuration checks, and whole jobs over Gloo."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from draco_b200 import JobConfig
from draco_b200.codes import oracle
from draco_b200.models import build_model
from draco_b200.parallel.arena import ArenaLayout
from draco_b200.parallel.ps import TorchPS
from draco_b200.parallel.trainer import Trainer

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_MODES = ("coordinate_median", "trimmed_mean", "multi_krum")
INF, NAN = math.inf, math.nan


# ------------------------------------------------------------------------------------------------ oracles
def test_trimmed_mean_and_median_hand_worked():
    odd = np.array([[3.0, 1.0], [-1.0, 1.0], [7.0, 5.0], [2.0, 1.0], [100.0, -4.0]])       # P = 5
    # column 0 sorted: -1 2 3 7 100 ; column 1 sorted: -4 1 1 1 5
    assert oracle.coordinate_median(odd).tolist() == [3.0, 1.0]
    assert oracle.trimmed_mean(odd, 1).tolist() == [4.0, 1.0]
    assert oracle.trimmed_mean(odd, 0).tolist() == [22.2, 0.8]
    even = np.array([[4.0], [1.0], [3.0], [2.0]])                                              # P = 4: mean of the middle two
    assert oracle.coordinate_median(even).tolist() == [2.5]
    assert oracle.trimmed_mean(even, 1).tolist() == [2.5]
    assert np.median(even, axis=0).tolist() == [2.5]
    with pytest.raises(ValueError):
        oracle.trimmed_mean(even, 2)


def test_trimmed_mean_orders_non_finite_values():
    """-Inf < finite < +Inf < NaN: at most b non-finite values per coordinate are trimmed away."""
    X = np.array([[NAN, INF, -INF, 1.0],
                  [1.0, 1.0, 5.0, NAN],
                  [2.0, -INF, 6.0, -INF],
                  [3.0, 3.0, 7.0, 2.0],
                  [-INF, 2.0, NAN, 3.0]])
    assert oracle.trimmed_mean(X, 1).tolist() == [2.0, 2.0, 6.0, 2.0]
    assert oracle.coordinate_median(X).tolist() == [2.0, 2.0, 6.0, 2.0]
    # NaN sorts above +Inf: with one NaN and one +Inf, b = 1 keeps the +Inf
    Y = np.array([[NAN], [INF], [1.0]])
    assert oracle.trimmed_mean(Y, 1).tolist() == [INF]
    # more than b poisoned values reach the result
    assert math.isnan(oracle.trimmed_mean(np.array([[NAN], [NAN], [1.0]]), 1)[0])


def test_multi_krum_hand_worked():
    X = np.array([[0.0], [1.0], [2.0], [10.0], [100.0]])       # P = 5, s = 1: keep the 2 nearest
    np.testing.assert_array_equal(oracle.krum_scores(X, 1), [5.0, 2.0, 5.0, 145.0, 8100.0 + 9604.0])
    assert oracle.multi_krum_indices(X, 1, 4) == [1, 0, 2, 3]   # tie 0 / 2 at score 5 -> lower index first
    assert oracle.multi_krum(X, 1, 4).tolist() == [13.0 / 4]
    assert oracle.multi_krum_indices(X, 1, 1) == [oracle.krum_index(X, 1)] == [1]


@pytest.mark.parametrize("P,s", [(5, 1), (7, 2), (9, 3), (16, 2)])
def test_multi_krum_with_one_row_is_krum(P, s):
    rng = np.random.default_rng(P * 10 + s)
    for _ in range(20):
        X = rng.normal(size=(P, 13))
        X[rng.integers(P)] *= 50
        assert oracle.multi_krum_indices(X, s, 1) == [oracle.krum_index(X, s)]
        full = oracle.multi_krum_indices(X, s, P)
        assert sorted(full) == list(range(P)) and full[0] == oracle.krum_index(X, s)


def test_krum_ranks_nan_rows_last():
    X = np.array([[NAN, 0.0], [0.0, 0.0], [0.1, 0.0], [0.2, 0.1], [9.0, 9.0], [0.1, 0.1]])     # row 0 sent NaN
    scores = oracle.krum_scores(X, 1)
    assert math.isnan(scores[0]) and np.isfinite(scores[1:]).all()                             # NaN distances sort last
    assert oracle.krum_index(X, 1) != 0 and oracle.multi_krum_indices(X, 1, 6)[-1] == 0 and 0 not in oracle.multi_krum_indices(X, 1, 5)


# ------------------------------------------------------------------------------------------------ library-op PS
def _layout():
    return ArenaLayout.from_model(build_model("LeNet"), bf16=False, channels_last=True)


def poisoned_slab(L, P, b, seed):
    """[P, D] fp32: N(0, 1) rows, and in every coordinate up to ``b`` rows replaced by +-1e30, +-Inf or NaN."""
    g = torch.Generator().manual_seed(seed)
    X = torch.randn(P, L.total, generator=g)
    if b > 0:
        rank = torch.rand(P, L.total, generator=g).argsort(0)                 # random row order per coordinate
        nbad = torch.randint(0, b + 1, (L.total,), generator=g)
        pool = torch.tensor([1e30, -1e30, INF, -INF, NAN])
        bad = torch.where(rank < nbad, pool[torch.randint(0, 5, (P, L.total), generator=g)], X)
        X = bad
    X[:, ~torch.from_numpy(L.valid_mask())] = 0
    return X


@pytest.mark.parametrize("mode,P,f", [("coordinate_median", 7, 2), ("coordinate_median", 8, 2), ("trimmed_mean", 7, 2),
                                      ("trimmed_mean", 16, 3), ("trimmed_mean", 5, 0)])
def test_torch_ps_coordinate_rules_match_oracle(mode, P, f):
    L = _layout()
    cfg = JobConfig(approach="baseline", mode=mode, num_workers=P, worker_fail=f, transport="gloo").resolve(1)
    ps = TorchPS(cfg, L, torch.device("cpu"), L.new_arena(torch.device("cpu")), None, None)
    b = (P - 1) // 2 if mode == "coordinate_median" else f
    X = poisoned_slab(L, P, b, seed=P + f)
    out = ps.aggregate(X)
    Xn = X.double().numpy()
    for spec, g in zip(L.specs, out):
        ref = oracle.trimmed_mean(Xn[:, spec.offset:spec.offset + spec.numel], b)
        assert np.isfinite(ref).all() and torch.isfinite(g).all()
        np.testing.assert_allclose(g.double().numpy(), ref, rtol=1e-6, atol=1e-6)
        if mode == "coordinate_median" and P % 2 == 1:
            assert torch.equal(g, X[:, spec.offset:spec.offset + spec.numel].sort(0).values[P // 2])


@pytest.mark.parametrize("P,f", [(7, 2), (9, 1)])
def test_torch_ps_multi_krum_matches_oracle(P, f):
    L = _layout()
    cfg = JobConfig(approach="baseline", mode="multi_krum", num_workers=P, worker_fail=f, transport="gloo").resolve(1)
    ps = TorchPS(cfg, L, torch.device("cpu"), L.new_arena(torch.device("cpu")), None, None)
    g = torch.Generator().manual_seed(P)
    X = 0.1 * torch.randn(1, L.total, generator=g) + 0.01 * torch.randn(P, L.total, generator=g)
    X[1] *= -100
    X[P - 1] = 30 * torch.randn(L.total, generator=g)
    X[0, torch.from_numpy(L.valid_mask())] = NAN                      # a NaN row ranks last and stays out of the average
    out = ps.aggregate(X)
    Xn = X.double().numpy()
    for spec, agg in zip(L.specs, out):
        ref = oracle.multi_krum(Xn[:, spec.offset:spec.offset + spec.numel], f, P - f)
        assert torch.isfinite(agg).all()
        np.testing.assert_allclose(agg.double().numpy(), ref, rtol=1e-5, atol=1e-6)


# ------------------------------------------------------------------------------------------------ configuration
def test_config_rejects_impossible_robust_rules():
    def cfg(**kw):
        return JobConfig(**dict(dict(approach="baseline", transport="nccl"), **kw))
    for mode in ("trimmed_mean", "coordinate_median"):
        with pytest.raises(ValueError, match="2\\*worker_fail"):
            cfg(mode=mode, num_workers=4, worker_fail=2).resolve(1)
        cfg(mode=mode, num_workers=5, worker_fail=2).resolve(1)
    with pytest.raises(ValueError, match="Krum's condition"):
        cfg(mode="multi_krum", num_workers=6, worker_fail=2).resolve(1)
    cfg(mode="multi_krum", num_workers=7, worker_fail=2).resolve(1)
    for mode in NEW_MODES:
        with pytest.raises(ValueError, match="at most 16 workers"):
            cfg(mode=mode, num_workers=17, worker_fail=1, transport="nvl").resolve(1)
        cfg(mode=mode, num_workers=17, worker_fail=1).resolve(1)                 # library path: no limit
        cfg(mode=mode, num_workers=16, worker_fail=1, transport="nvl").resolve(1)
    # the existing modes are validated as before
    cfg(mode="krum", num_workers=4, worker_fail=2).resolve(1)
    cfg(mode="normal", num_workers=32, worker_fail=20, transport="nvl").resolve(1)


# ------------------------------------------------------------------------------------------------ jobs
@pytest.mark.parametrize("mode", NEW_MODES)
def test_robust_rules_train_under_attack_over_gloo(mode):
    cfg = JobConfig(network="LeNet", dataset="MNIST", batch_size=16, max_steps=12, num_workers=7, transport="gloo", lr=0.05,
                    momentum=0.9, synthetic_size=512, eval_freq=10 ** 6, compress_grad="None", approach="baseline", mode=mode,
                    worker_fail=2, err_mode="rev_grad")
    t = Trainer(cfg, rank=0, world=1, device=torch.device("cpu"), quiet=True)
    losses = [t.train_step()["loss"] for _ in range(12)]
    assert losses[-1] < losses[0], losses
    assert torch.isfinite(t.engine.master_params()).all()


@pytest.mark.parametrize("mode", NEW_MODES)
def test_robust_rules_as_a_multi_process_job(tmp_path, mode):
    """1 PS + 5 workers packed onto 2 Gloo processes, 3 steps."""
    port = 29710 + NEW_MODES.index(mode)
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""), OMP_NUM_THREADS="2")
    r = subprocess.run([sys.executable, "-m", "draco_b200.cli.distributed_nn", "--launch", "2", "--master-port", str(port), "--no-cuda",
                        "--network", "LeNet", "--dataset", "MNIST", "--num-workers", "5", "--batch-size", "8", "--max-steps", "3",
                        "--eval-freq", "1000", "--train-dir", str(tmp_path) + "/", "--synthetic-size", "128", "--log-interval", "1",
                        "--compress-grad", "None", "--approach", "baseline", "--mode", mode, "--worker-fail", "1", "--err-mode",
                        "rev_grad"], capture_output=True, text=True, timeout=420, env=env, cwd=ROOT)
    out = r.stdout + r.stderr
    assert r.returncode == 0, out[-3000:]
    assert out.count("done at step 3") == 2, out[-2500:]
