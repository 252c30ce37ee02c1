"""Nearest-neighbour mixing (NNM; Allouah et al., AISTATS 2023) on the CPU: the fp64 oracle on hand-worked cases and against a
brute-force restatement of the paper's definition, the mixed distance table against direct distances of the mixed rows,
robustness to far-away bad rows, the library-op PS against the oracle for every base rule, the configuration checks, and whole
jobs over Gloo."""
import itertools
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from draco_b200 import JobConfig
from draco_b200.codes import oracle
from draco_b200.config import NNM_MODES
from draco_b200.models import build_model
from draco_b200.parallel.arena import ArenaLayout
from draco_b200.parallel.ps import TorchPS, select_rule
from draco_b200.parallel.trainer import Trainer

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAN = float("nan")


def _mode_ok(P, f, mode):
    return {"coordinate_median": 2 * f < P, "trimmed_mean": 2 * f < P, "krum": True, "multi_krum": P > 2 * f + 2,
            "geometric_median": True, "bulyan": P >= 4 * f + 3}[mode]


# ------------------------------------------------------------------------------------------------ oracle, hand-worked
def test_neighbours_hand_worked_with_ties():
    # rows on a line at 0, 1, 2, 4; f = 1, n_mix = 3: each row plus its 2 nearest others
    X = np.array([[0.0], [1.0], [2.0], [4.0]])
    A = oracle.nnm_neighbours(X, 1)
    # row 1: 0 and 2 are both at distance 1 -> both; row 2: 1 (1) and then 0 and 4 tie at 4 -> the lower row, 0
    assert A.tolist() == [[1, 1, 1, 0], [1, 1, 1, 0], [1, 1, 1, 0], [0, 1, 1, 1]]
    np.testing.assert_allclose(oracle.nnm_mix(X, 1)[:, 0], [1.0, 1.0, 1.0, 7.0 / 3], rtol=0, atol=1e-15)


def test_a_duplicated_row_does_not_displace_row_i_itself():
    X = np.array([[5.0], [0.0], [0.0], [3.0]])                  # rows 1 and 2 are equal
    A = oracle.nnm_neighbours(X, 2)                             # n_mix = 2: row i and its single nearest other row
    assert A[2].tolist() == [0, 1, 1, 0]                        # row 2 keeps itself and takes its duplicate, row 1
    assert A[1].tolist() == [0, 1, 1, 0]
    assert A[0].tolist() == [1, 0, 0, 1]
    assert oracle.nnm_neighbours(X, 3).tolist() == np.eye(4, dtype=int).tolist()     # n_mix = 1: no mixing


def test_a_nan_row_sorts_last_and_poisons_only_the_rows_that_take_it():
    X = np.array([[0.0, 0.0], [1.0, 0.0], [NAN, 0.0], [0.0, 2.0], [9.0, 9.0]])
    A = oracle.nnm_neighbours(X, 1)                             # n_mix = 4: the NaN row is nobody's choice but its own
    assert all(A[i, 2] == 0 for i in (0, 1, 3, 4))
    assert A[2].tolist() == [1, 1, 1, 1, 0]                     # NaN row: every distance NaN, ties to the lower rows
    Y = oracle.nnm_mix(X, 1)
    assert np.isnan(Y[2, 0]) and np.isfinite(np.delete(Y, 2, axis=0)).all()
    Dm = oracle.nnm_pair_d2(oracle._raw_d2(X), A, 1)
    assert np.isnan(Dm[2]).sum() == 4 and np.isnan(Dm[:, 2]).sum() == 4              # NaN stays NaN through the clamp
    assert np.isfinite(np.delete(np.delete(Dm, 2, 0), 2, 1)).all()


@pytest.mark.parametrize("mode", NNM_MODES)
def test_f_zero_mixes_every_row_into_the_mean(mode):
    rng = np.random.default_rng(3)
    X = rng.normal(size=(7, 13))
    Y = oracle.nnm_mix(X, 0)
    np.testing.assert_allclose(Y, np.broadcast_to(X.mean(0), Y.shape), rtol=0, atol=1e-14)
    np.testing.assert_allclose(oracle.nnm(X, 0, mode), X.mean(0), rtol=0, atol=1e-12)


# ------------------------------------------------------------------------------------------------ oracle, brute force
def _brute_force_neighbours(X, f):
    """Straight from the paper: N_i is a set of n_mix rows containing i minimising the sum of squared distances to x_i; among
    those, the one whose sorted (distance, row) list is smallest (NaN largest, ties to the lower row)."""
    P = X.shape[0]
    n = P - f
    d = [[float(((X[i] - X[j]) ** 2).sum()) for j in range(P)] for i in range(P)]
    key = lambda i, j: (np.isnan(d[i][j]), 0.0 if np.isnan(d[i][j]) else d[i][j], j)     # noqa: E731
    A = np.zeros((P, P), dtype=np.int64)
    for i in range(P):
        others = [j for j in range(P) if j != i]
        best = min(itertools.combinations(others, n - 1), key=lambda c: sorted(key(i, j) for j in c))
        A[i, [i, *best]] = 1
    return A


@pytest.mark.parametrize("P,f", [(3, 1), (5, 1), (6, 2), (7, 3), (8, 1)])
def test_neighbours_match_brute_force(P, f):
    rng = np.random.default_rng(P * 10 + f)
    for trial in range(4):
        X = rng.integers(-3, 4, size=(P, 2)).astype(np.float64)     # small integers: many distance ties
        if trial == 3:
            X[P - 1] = NAN
        assert oracle.nnm_neighbours(X, f).tolist() == _brute_force_neighbours(X, f).tolist(), (trial, X)


@pytest.mark.parametrize("P,f", [(3, 1), (7, 2), (11, 3), (16, 5), (16, 0)])
def test_mixed_pair_table_matches_direct_distances(P, f):
    rng = np.random.default_rng(P + f)
    X = rng.normal(size=(P, 50)) * rng.uniform(0.1, 10, size=(P, 1))
    A = oracle.nnm_neighbours(X, f)
    Dm = oracle.nnm_pair_d2(oracle._raw_d2(X), A, f)
    Y = A @ X / (P - f)
    direct = ((Y[:, None, :] - Y[None, :, :]) ** 2).sum(axis=2)
    np.testing.assert_allclose(Dm, direct, rtol=1e-9, atol=1e-9 * direct.max())
    assert (Dm >= 0).all()


@pytest.mark.parametrize("P,f", [(7, 1), (11, 2), (15, 3), (16, 3)])
def test_far_bad_rows_never_mix_into_honest_rows(P, f):
    """Up to f rows far away (1e6 in random directions): no honest row takes one as a neighbour, so every rule's result stays
    in the honest rows' per-coordinate range."""
    rng = np.random.default_rng(P + 7 * f)
    for trial in range(4):
        X = rng.normal(size=(P, 30))
        bad = rng.choice(P, size=trial % (f + 1), replace=False)
        X[bad] = rng.normal(size=(len(bad), 30)) * 1e6
        A = oracle.nnm_neighbours(X, f)
        honest = [i for i in range(P) if i not in bad]
        assert not A[np.ix_(honest, bad)].any()
        lo, hi = X[honest].min(0), X[honest].max(0)
        for mode in NNM_MODES:
            if _mode_ok(P, f, mode):
                out = oracle.nnm(X, f, mode)
                assert ((out >= lo - 1e-9) & (out <= hi + 1e-9)).all(), (mode, trial)


# ------------------------------------------------------------------------------------------------ library-op PS
def _layout():
    return ArenaLayout.from_model(build_model("LeNet"), bf16=False, channels_last=True)


@pytest.mark.parametrize("mode", NNM_MODES)
@pytest.mark.parametrize("P,f", [(7, 1), (15, 3)])
def test_torch_ps_matches_oracle(mode, P, f):
    L = _layout()
    cfg = JobConfig(approach="nnm", mode=mode, num_workers=P, worker_fail=f, transport="gloo").resolve(1)
    assert select_rule(cfg).startswith("nnm_")
    ps = TorchPS(cfg, L, torch.device("cpu"), L.new_arena(torch.device("cpu")), None, None)
    g = torch.Generator().manual_seed(P * 7 + f)
    X = torch.randn(P, L.total, generator=g) * torch.rand(P, 1, generator=g)
    X[P - 1] = -50 * X[P - 1]                                       # one far row
    X[:, ~torch.from_numpy(L.valid_mask())] = 0
    out = ps.aggregate(X)
    Xn = X.double().numpy()
    for spec, gt in zip(L.specs, out):
        cols = slice(spec.offset, spec.offset + spec.numel)
        ref = oracle.nnm(Xn[:, cols], f, mode)
        atol = 1e-4 if mode == "geometric_median" else 1e-6                # TorchPS runs its own Weiszfeld on the mixed rows
        np.testing.assert_allclose(gt.double().numpy(), ref, rtol=1e-5, atol=atol)


def test_torch_ps_mixes_in_the_kernels_fp32_order():
    X = torch.tensor([[1e8, 0.0], [1.0, 0.0], [-1e8, 0.0], [3.0, 0.0]])
    cfg = JobConfig(approach="nnm", mode="coordinate_median", num_workers=4, worker_fail=1, transport="gloo").resolve(1)
    ps = TorchPS(cfg, _layout(), torch.device("cpu"), torch.zeros(1), None, None)
    Y = ps._nnm_mix_tensor(X, 1)
    A = oracle.nnm_neighbours(X.double().numpy(), 1)
    for i in range(4):
        y = torch.zeros(2)
        for j in np.flatnonzero(A[i]):                               # ascending rows from +0, then one multiply
            y = y + X[j]
        assert torch.equal(Y[i], y * torch.tensor(1.0 / 3, dtype=torch.float32))


# ------------------------------------------------------------------------------------------------ configuration
def test_config_bounds_for_nnm():
    def cfg(**kw):
        return JobConfig(**dict(dict(approach="nnm", transport="nvl", num_workers=15, worker_fail=3), **kw))
    for mode in NNM_MODES:
        c = cfg(mode=mode).resolve(1)
        assert select_rule(c) == "nnm_" + {"coordinate_median": "median", "geometric_median": "geomedian"}.get(mode, mode)
    for bad in ("normal", "maj_vote", "bogus"):
        with pytest.raises(ValueError, match="--approach nnm takes --mode"):
            cfg(mode=bad).resolve(1)
    with pytest.raises(ValueError, match="0 <= worker_fail < num_workers"):
        cfg(mode="krum", num_workers=4, worker_fail=4).resolve(1)
    # the base rule's own conditions, with messages naming the approach
    with pytest.raises(ValueError, match="--approach nnm --mode trimmed_mean trims"):
        cfg(mode="trimmed_mean", num_workers=6, worker_fail=3).resolve(1)
    with pytest.raises(ValueError, match="--approach nnm --mode multi_krum needs num_workers > 2\\*worker_fail \\+ 2"):
        cfg(mode="multi_krum", num_workers=8, worker_fail=3).resolve(1)
    with pytest.raises(ValueError, match="--approach nnm --mode bulyan needs num_workers >= 4\\*worker_fail \\+ 3"):
        cfg(mode="bulyan", num_workers=14, worker_fail=3).resolve(1)
    cfg(mode="krum", num_workers=5, worker_fail=4).resolve(1)                # Krum and the geometric median: f < P only
    cfg(mode="geometric_median", num_workers=5, worker_fail=4).resolve(1)
    with pytest.raises(ValueError, match="at most 16 workers"):
        cfg(mode="krum", num_workers=17).resolve(1)
    cfg(mode="krum", num_workers=17, transport="nccl").resolve(1)
    with pytest.raises(ValueError, match="nccl_flat"):
        cfg(mode="krum", transport="nccl_flat", compress_grad="None").resolve(1)
    # the baseline's messages are unchanged
    with pytest.raises(ValueError, match="^--mode bulyan needs num_workers >= 4\\*worker_fail \\+ 3"):
        cfg(approach="baseline", mode="bulyan", num_workers=14).resolve(1)


def test_nnm_workers_draw_distinct_batches_like_the_baseline():
    from draco_b200.data import BatchPlan
    a, b = BatchPlan("nnm", 1000, 8, 5), BatchPlan("baseline", 1000, 8, 5)
    for step, rank in ((1, 1), (3, 2), (200, 5)):
        assert a.indices(step, rank)[0].tolist() == b.indices(step, rank)[0].tolist()
        assert a.batch_ids(step, rank) == b.batch_ids(step, rank) == [rank]
    assert a.indices(1, 1)[0].tolist() != a.indices(1, 2)[0].tolist()


# ------------------------------------------------------------------------------------------------ jobs
def _job(**kw):
    base = dict(network="LeNet", dataset="MNIST", batch_size=16, max_steps=12, transport="gloo", lr=0.05, momentum=0.9,
                synthetic_size=512, eval_freq=10 ** 6, compress_grad="None", approach="nnm", num_workers=7, worker_fail=1)
    base.update(kw)
    t = Trainer(JobConfig(**base), rank=0, world=1, device=torch.device("cpu"), quiet=True)
    losses = [t.train_step()["loss"] for _ in range(12)]
    assert losses[-1] < losses[0], losses
    assert torch.isfinite(t.engine.master_params()).all()


@pytest.mark.parametrize("mode,err", [("multi_krum", "rev_grad"), ("coordinate_median", "alie"), ("bulyan", "minmax")])
def test_nnm_trains_under_attack_over_gloo(mode, err):
    _job(mode=mode, err_mode=err)


def test_nnm_as_a_multi_process_job(tmp_path):
    """1 PS + 7 workers packed onto 2 Gloo processes, 3 steps."""
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""), OMP_NUM_THREADS="2")
    r = subprocess.run([sys.executable, "-m", "draco_b200.cli.distributed_nn", "--launch", "2", "--master-port", "29734", "--no-cuda",
                        "--network", "LeNet", "--dataset", "MNIST", "--num-workers", "7", "--batch-size", "8", "--max-steps", "3",
                        "--eval-freq", "1000", "--train-dir", str(tmp_path) + "/", "--synthetic-size", "128", "--log-interval", "1",
                        "--compress-grad", "None", "--approach", "nnm", "--mode", "multi_krum", "--worker-fail", "1", "--err-mode",
                        "rev_grad"], capture_output=True, text=True, timeout=420, env=env, cwd=ROOT)
    out = r.stdout + r.stderr
    assert r.returncode == 0, out[-3000:]
    assert out.count("done at step 3") == 2, out[-2500:]
