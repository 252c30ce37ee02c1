"""Bulyan (El Mhamdi, Guerraoui and Rouault, ICML 2018) on the CPU: the fp64 oracle on hand-worked cases and against a
brute-force restatement of the paper's definition, its robustness to bad rows, the library-op PS against the oracle, the
configuration checks, and whole jobs over Gloo."""
import itertools
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from draco_b200 import JobConfig
from draco_b200.codes import oracle
from draco_b200.codes.repetition import group_assign
from draco_b200.models import build_model
from draco_b200.parallel.arena import ArenaLayout
from draco_b200.parallel.ps import TorchPS
from draco_b200.parallel.trainer import Trainer

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INF, NAN = math.inf, math.nan
BAD = (1e30, -1e30, INF, -INF, NAN)


# ------------------------------------------------------------------------------------------------ oracle, hand-worked
def test_nearest_to_median_mean_odd_and_even():
    # theta = 5, f = 1, beta = 3; column 0 sorted 0 1 2 3 10, m = 2: 3 enters for 0, 10 does not enter for 1 -> {1, 2, 3}
    # column 1 sorted -9 4 5 6 7, m = 5: 6 enters for -9, 7 (distance 2) does not enter for 4 (distance 1) -> {4, 5, 6}
    odd = np.array([[10.0, 5.0], [1.0, -9.0], [3.0, 7.0], [0.0, 4.0], [2.0, 6.0]])
    assert oracle.nearest_to_median_mean(odd, 1).tolist() == [2.0, 5.0]
    # not the 1-trimmed mean, which keeps the middle window {8, 9, 30} / {1, 9, 10} whatever the distances:
    X = np.array([[0.0], [8.0], [9.0], [30.0], [40.0]])               # m = 9: 30 (21 away) does not enter for 0 (9 away)
    assert oracle.nearest_to_median_mean(X, 1).tolist() == [17.0 / 3]
    Y = np.array([[0.0], [1.0], [9.0], [10.0], [11.0]])               # m = 9: 10 enters for 0, 11 (2) enters for 1 (8)
    assert oracle.nearest_to_median_mean(Y, 1).tolist() == [10.0]
    assert oracle.trimmed_mean(X, 1).tolist() == [47.0 / 3] and oracle.trimmed_mean(Y, 1).tolist() == [20.0 / 3]
    # theta = 4, f = 1, beta = 2: m = 0.5 * 1 + 0.5 * 3 = 2; 3 enters for 0, 7 does not enter for 1 -> {1, 3}
    even = np.array([[7.0], [0.0], [3.0], [1.0]])
    assert oracle.nearest_to_median_mean(even, 1).tolist() == [2.0]
    # theta = 6, f = 2, beta = 2: m = 2.5; 2 enters for -4, 3 enters for 0, 9 does not enter for 2 -> {2, 3}
    assert oracle.nearest_to_median_mean(np.array([[-4.0], [0.0], [2.0], [3.0], [9.0], [12.0]]), 2).tolist() == [2.5]
    with pytest.raises(ValueError):
        oracle.nearest_to_median_mean(even, 2)


def test_a_distance_tie_keeps_the_smaller_value():
    # theta = 5, f = 1, beta = 3, m = 5: 6 enters for 0; then 3 (below) and 7 (above) are both 2 away: 7 does not enter
    X = np.array([[0.0], [3.0], [5.0], [6.0], [7.0]])
    assert oracle.nearest_to_median_mean(X, 1).tolist() == [(3.0 + 5.0 + 6.0) / 3]
    # the tie at the first step: 3 and 7 are both 2 away from m = 5, the window stays at {3, 4, 5}
    X = np.array([[3.0], [4.0], [5.0], [7.0], [100.0]])
    assert oracle.nearest_to_median_mean(X, 1).tolist() == [4.0]
    # beta = 1 (theta = 3, f = 1): the median itself
    assert oracle.nearest_to_median_mean(np.array([[1.0], [2.0], [3.0]]), 1).tolist() == [2.0]
    # even theta = 8, f = 2, beta = 4, m = 0.5 * 3 + 0.5 * 5 = 4: 5 enters for -100; 1 and 7 are both 3 away: 7 does not enter
    X = np.array([[-100.0], [1.0], [2.0], [3.0], [5.0], [7.0], [8.0], [100.0]])
    assert oracle.nearest_to_median_mean(X, 2).tolist() == [(1.0 + 2.0 + 3.0 + 5.0) / 4]


def test_nearest_to_median_mean_orders_non_finite_values():
    """A NaN distance is the farthest, so up to f NaN / +-Inf / +-1e30 values never enter the window."""
    X = np.array([[NAN, INF, -INF, 1.0, 1e30],
                  [1.0, 1.0, 5.0, NAN, 2.0],
                  [2.0, -INF, 6.0, -INF, 3.0],
                  [3.0, 3.0, 7.0, 2.0, -1e30],
                  [2.5, 2.0, 5.5, 3.0, 2.5]])
    assert oracle.nearest_to_median_mean(X, 1).tolist() == [2.5, 2.0, 5.5, 2.0, 2.5]
    # more than f NaN: the median is NaN, every distance NaN, the window stays at the smallest values and takes a NaN in
    assert math.isnan(oracle.nearest_to_median_mean(np.array([[NAN], [NAN], [NAN], [1.0], [2.0]]), 1)[0])


def _dist2(X):
    return ((X[:, None, :] - X[None, :, :]) ** 2).sum(axis=2)


def test_bulyan_selection_hand_worked():
    # P = 7, f = 1, theta = 5 (one dimension): rows 0..5 at 0, 1, 2, 3, 4, 5 and row 6 at 100
    X = np.array([[0.0], [1.0], [2.0], [3.0], [4.0], [5.0], [100.0]])
    # round 1, keep = 7 - 1 - 2 = 4: row 2 scores 1 + 1 + 4 + 4 = 10, row 3 the same -> the lower row, 2
    # round 2, R = {0, 1, 3, 4, 5, 6}, keep = 3: row 3 scores 1 + 4 + 4 = 9, row 1: 1 + 4 + 9 = 14, row 4: 1 + 1 + 9 = 11 -> 3
    # round 3, R = {0, 1, 4, 5, 6}, keep = 2: row 0: 1 + 16, row 1: 1 + 9, row 4: 1 + 9, row 5: 1 + 16 -> 1 (tie with 4)
    # round 4, R = {0, 4, 5, 6}, keep = 1: row 4: 1, row 5: 1 -> 4; round 5, R = {0, 5, 6}, keep = 0: all 0 -> row 0
    assert oracle.bulyan_indices(X, 1) == [2, 3, 1, 4, 0]
    # the keep = 0 last round takes the lowest remaining row: the far row 6 stays out only because it is not the lowest.
    # The chosen values sorted are 0 1 2 3 4, m = 2: 3 enters for 0, 4 does not enter for 1 -> {1, 2, 3}
    assert oracle.bulyan(X, 1).tolist() == [2.0]


def test_keep_zero_last_round_picks_the_lowest_remaining_row():
    """f = 1, P = 7: the fifth round scores |R| - f - 2 = 0 distances, so every score is 0 and the lowest row left wins, even
    a row that sent NaN (it scored last in every earlier round).  The coordinate stage keeps it out of the result."""
    rng = np.random.default_rng(3)
    X = rng.normal(size=(7, 9))
    X[0] = NAN
    sel = oracle.bulyan_indices(X, 1)
    assert sel[-1] == 0 and 0 not in sel[:-1]
    out = oracle.bulyan(X, 1)
    assert np.isfinite(out).all()
    H = X[1:]
    assert ((out >= H.min(0)) & (out <= H.max(0))).all()


def test_f_zero_is_the_mean_of_all_rows():
    rng = np.random.default_rng(4)
    for P in (3, 4, 8):
        X = rng.normal(size=(P, 11))
        assert sorted(oracle.bulyan_indices(X, 0)) == list(range(P))
        np.testing.assert_allclose(oracle.bulyan(X, 0), X.mean(0), rtol=1e-12, atol=1e-12)


def _brute_force_bulyan_indices(X, f):
    """The paper's recursion restated literally: A(R) = Krum over R with n = |R|, i.e. argmin_i sum of the n - f - 2 smallest
    ||x_i - x_j||^2 over j in R, j != i, found by enumerating every subset of that size (ties to the lower row)."""
    d2 = _dist2(X)
    R, S = list(range(X.shape[0])), []
    for _ in range(X.shape[0] - 2 * f):
        keep = max(len(R) - f - 2, 0)
        best = None
        for i in R:
            others = [j for j in R if j != i]
            score = min((sum(d2[i, j] for j in sub) for sub in itertools.combinations(others, keep)), default=0.0)
            if best is None or score < best[0]:
                best = (score, i)
        S.append(best[1])
        R.remove(best[1])
    return S


@pytest.mark.parametrize("P,f", [(3, 0), (7, 1), (8, 1), (11, 2)])
def test_bulyan_selection_matches_brute_force(P, f):
    rng = np.random.default_rng(P * 7 + f)
    for _ in range(4):
        X = rng.normal(size=(P, 6))
        X[rng.integers(P)] *= 30
        assert oracle.bulyan_indices(X, f) == _brute_force_bulyan_indices(X, f)


@pytest.mark.parametrize("P,f", [(7, 1), (11, 2), (15, 3), (16, 3)])
def test_bad_rows_are_never_selected_and_the_result_stays_in_the_honest_range(P, f):
    """Up to f whole rows replaced by distinct bad values (+-1e30, +-Inf, NaN).  For f >= 2 no bad row is ever selected; for
    f = 1 the keep = 0 last round may take one in a low slot.  Every output coordinate lies within the honest rows' range."""
    rng = np.random.default_rng(P + 100 * f)
    for trial in range(6):
        X = rng.normal(size=(P, 40))
        nbad = trial % (f + 1)
        bad = rng.choice(P, size=nbad, replace=False)
        for b, v in zip(bad, rng.choice(len(BAD), size=nbad, replace=False)):
            X[b] = BAD[v]
        sel = oracle.bulyan_indices(X, f)
        if f >= 2:
            assert not set(sel) & set(bad.tolist()), (sel, bad)
        else:
            assert not set(sel[:-1]) & set(bad.tolist())
        honest = np.delete(X, bad, axis=0)
        out = oracle.bulyan(X, f)
        assert np.isfinite(out).all() and ((out >= honest.min(0)) & (out <= honest.max(0))).all()


def test_detox_with_group_size_one_is_bulyan():
    rng = np.random.default_rng(5)
    X = rng.normal(size=(11, 17))
    X[4] *= -100
    groups = group_assign(11, 1).groups
    np.testing.assert_allclose(oracle.detox(X, groups, "bulyan", 2), oracle.bulyan(X, 2), rtol=0, atol=0)


# ------------------------------------------------------------------------------------------------ library-op PS
def _layout():
    return ArenaLayout.from_model(build_model("LeNet"), bf16=False, channels_last=True)


def bad_row_slab(L, P, f, seed):
    """[P, D] fp32: honest rows on a grid of multiples of 1/64 (every fp32 sum, difference and median of them is exact, so
    the fp32 library path and the fp64 oracle meet the same distance ties), and up to f rows of distinct bad values."""
    g = torch.Generator().manual_seed(seed)
    X = torch.randint(-128, 129, (P, L.total), generator=g).float() / 64
    rows = torch.randperm(P, generator=g)[:f]
    for r, v in zip(rows.tolist(), torch.randperm(len(BAD), generator=g).tolist()):
        X[r] = BAD[v]
    X[:, ~torch.from_numpy(L.valid_mask())] = 0
    return X, rows.tolist()


@pytest.mark.parametrize("P,f", [(7, 1), (11, 2), (15, 3)])
def test_torch_ps_bulyan_matches_oracle(P, f):
    L = _layout()
    cfg = JobConfig(approach="baseline", mode="bulyan", num_workers=P, worker_fail=f, transport="gloo").resolve(1)
    ps = TorchPS(cfg, L, torch.device("cpu"), L.new_arena(torch.device("cpu")), None, None)
    X, bad = bad_row_slab(L, P, f, seed=P)
    out = ps.aggregate(X)
    Xn = X.double().numpy()
    honest = np.delete(Xn, bad, axis=0)
    for spec, g in zip(L.specs, out):
        cols = slice(spec.offset, spec.offset + spec.numel)
        ref = oracle.bulyan(Xn[:, cols], f)
        assert np.isfinite(ref).all() and torch.isfinite(g).all()
        np.testing.assert_allclose(g.double().numpy(), ref, rtol=1e-6, atol=1e-6)
        assert ((ref >= honest[:, cols].min(0)) & (ref <= honest[:, cols].max(0))).all()


@pytest.mark.parametrize("P,r,f", [(14, 2, 1), (21, 3, 3)])
def test_torch_ps_detox_bulyan_matches_oracle(P, r, f):
    L = _layout()
    cfg = JobConfig(approach="detox", mode="bulyan", num_workers=P, group_size=r, worker_fail=f, transport="gloo").resolve(1)
    assert (cfg.num_groups, cfg.captured_group_bound) == (7, 1)
    ps = TorchPS(cfg, L, torch.device("cpu"), L.new_arena(torch.device("cpu")), *_groups(cfg))
    G = cfg.num_groups
    H, _ = bad_row_slab(L, G, 1, seed=P)                   # one group row is bad: the group the liars captured
    groups = group_assign(P, r).groups
    X = torch.stack([H[gi] for gi, grp in enumerate(groups) for _ in grp])
    out = ps.aggregate(X)
    Xn = X.double().numpy()
    for spec, g in zip(L.specs, out):
        cols = slice(spec.offset, spec.offset + spec.numel)
        ref = oracle.detox(Xn[:, cols], groups, "bulyan", cfg.captured_group_bound)
        np.testing.assert_allclose(g.double().numpy(), ref, rtol=1e-6, atol=1e-6)
        np.testing.assert_allclose(ref, oracle.bulyan(H.double().numpy()[:, cols], 1), rtol=0, atol=0)


def _groups(cfg):
    from draco_b200.parallel.ps import build_codes
    return build_codes(cfg)


# ------------------------------------------------------------------------------------------------ configuration
def test_config_bounds_for_bulyan():
    def cfg(**kw):
        return JobConfig(**dict(dict(approach="baseline", mode="bulyan", transport="nvl"), **kw))
    for P, f in ((3, 0), (7, 1), (11, 2), (15, 3), (16, 3)):
        cfg(num_workers=P, worker_fail=f).resolve(1)
    for P, f in ((2, 0), (6, 1), (10, 2), (14, 3)):
        with pytest.raises(ValueError, match="4\\*worker_fail \\+ 3"):
            cfg(num_workers=P, worker_fail=f).resolve(1)
    with pytest.raises(ValueError, match="at most 16 workers"):
        cfg(num_workers=19, worker_fail=4).resolve(1)
    cfg(num_workers=19, worker_fail=4, transport="nccl").resolve(1)           # library path: no limit
    # DETOX: G >= 4 b_G + 3 over the group winners
    det = dict(approach="detox")
    c = cfg(num_workers=14, group_size=2, worker_fail=1, **det).resolve(1)
    assert (c.num_groups, c.captured_group_bound) == (7, 1)
    cfg(num_workers=21, group_size=3, worker_fail=3, **det).resolve(1)         # G = 7, b_G = 1
    cfg(num_workers=9, group_size=3, worker_fail=1, **det).resolve(1)          # G = 3, b_G = 0
    with pytest.raises(ValueError, match="groups >= 4\\*b_G \\+ 3"):
        cfg(num_workers=15, group_size=3, worker_fail=3, **det).resolve(1)     # G = 5, b_G = 1
    with pytest.raises(ValueError, match="at most 16 groups"):
        cfg(num_workers=17, group_size=1, worker_fail=0, **det).resolve(1)
    # nccl_flat implements only the vote and the mean
    from draco_b200.parallel.flat_engine import FlatNcclEngine
    c = cfg(num_workers=7, worker_fail=1, transport="nccl_flat", compress_grad="None").resolve(1)
    with pytest.raises(ValueError, match="nccl_flat implements the repetition-code vote and the plain mean.*mode=bulyan"):
        FlatNcclEngine(c, 0, 1, torch.device("cpu"), None)


# ------------------------------------------------------------------------------------------------ jobs
def _job(**kw):
    base = dict(network="LeNet", dataset="MNIST", batch_size=16, max_steps=12, transport="gloo", lr=0.05, momentum=0.9,
                synthetic_size=512, eval_freq=10 ** 6, compress_grad="None", mode="bulyan", err_mode="rev_grad")
    base.update(kw)
    t = Trainer(JobConfig(**base), rank=0, world=1, device=torch.device("cpu"), quiet=True)
    losses = [t.train_step()["loss"] for _ in range(12)]
    assert losses[-1] < losses[0], losses
    assert torch.isfinite(t.engine.master_params()).all()


def test_bulyan_trains_under_attack_over_gloo():
    _job(approach="baseline", num_workers=7, worker_fail=1)


def test_detox_bulyan_trains_under_attack_over_gloo():
    _job(approach="detox", num_workers=14, group_size=2, worker_fail=1)


def test_bulyan_as_a_multi_process_job(tmp_path):
    """1 PS + 7 workers packed onto 2 Gloo processes, 3 steps."""
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""), OMP_NUM_THREADS="2")
    r = subprocess.run([sys.executable, "-m", "draco_b200.cli.distributed_nn", "--launch", "2", "--master-port", "29730", "--no-cuda",
                        "--network", "LeNet", "--dataset", "MNIST", "--num-workers", "7", "--batch-size", "8", "--max-steps", "3",
                        "--eval-freq", "1000", "--train-dir", str(tmp_path) + "/", "--synthetic-size", "128", "--log-interval", "1",
                        "--compress-grad", "None", "--approach", "baseline", "--mode", "bulyan", "--worker-fail", "1", "--err-mode",
                        "rev_grad"], capture_output=True, text=True, timeout=420, env=env, cwd=ROOT)
    out = r.stdout + r.stderr
    assert r.returncode == 0, out[-3000:]
    assert out.count("done at step 3") == 2, out[-2500:]
