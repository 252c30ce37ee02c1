"""DETOX on the CPU (majority vote inside every repetition group, then a robust rule across the group winners): the fp64 oracle on
hand-worked cases, the identity with the baseline rules at group size 1, the library-op PS against the oracle, an exhaustive
tolerance check over every liar subset, the configuration checks, the batch plan, and whole jobs over Gloo."""
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
from draco_b200.codes.adversary import err_simulation
from draco_b200.codes.repetition import group_assign
from draco_b200.models import build_model
from draco_b200.parallel.arena import ArenaLayout
from draco_b200.parallel.fused_engine import make_plan
from draco_b200.parallel.ps import TorchPS, build_codes
from draco_b200.parallel.trainer import Trainer

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DETOX_MODES = ("coordinate_median", "trimmed_mean", "multi_krum", "geometric_median")
NAN = math.nan
G3 = [[1, 2, 3], [4, 5, 6], [7, 8, 9]]


# ------------------------------------------------------------------------------------------------ oracle
def test_captured_group_bound():
    assert oracle.captured_group_bound(2, 3) == 1 and oracle.captured_group_bound(3, 3) == 1
    assert oracle.captured_group_bound(4, 3) == 2 and oracle.captured_group_bound(1, 3) == 0
    assert oracle.captured_group_bound(2, 4) == 1 and oracle.captured_group_bound(3, 1) == 3      # even r: r / 2 liars can tie
    assert JobConfig(approach="detox", num_workers=15, group_size=3, worker_fail=3).captured_group_bound == 1
    # an even group with r / 2 identical liars can be captured: L L H H leaves the liars' candidate standing
    assert oracle.boyer_moore_winner([np.array([-1.0]), np.array([-1.0]), np.array([1.0]), np.array([1.0])]) == 0


def test_detox_hand_worked_with_one_captured_group():
    """Groups of 3; group 2 is captured by two liars that send [-100, 1e30]."""
    X = np.array([[1.0, 10.0], [1.0, 10.0], [1.0, 10.0],
                  [2.0, 20.0], [2.0, 20.0], [2.0, 20.0],
                  [-100.0, 1e30], [-100.0, 1e30], [3.0, 30.0]])
    assert oracle.detox_winner_slots(X, G3) == [0, 3, 6]
    b = oracle.captured_group_bound(2, 3)
    # winners [1, 10], [2, 20], [-100, 1e30]: the middle value of each coordinate
    assert oracle.detox(X, G3, "coordinate_median", b).tolist() == [1.0, 20.0]
    assert oracle.detox(X, G3, "trimmed_mean", b).tolist() == [1.0, 20.0]
    vote, _ = oracle.majority_vote(X, G3)
    assert vote.tolist() == [-97.0 / 3, (30.0 + 1e30) / 3]                          # the vote average takes the liars' row
    # two liars that send NaN never agree (NaN != NaN, as np.array_equal has it): the honest member wins their group
    X[6:8] = NAN
    assert oracle.detox_winner_slots(X, G3) == [0, 3, 8]
    assert oracle.detox(X, G3, "coordinate_median", b).tolist() == [2.0, 20.0]


def test_detox_hand_worked_with_a_nan_liar_that_captures_nothing():
    """One NaN-sending liar per group is out-voted; the rule then sees honest winners only."""
    X = np.array([[1.0], [NAN], [1.0], [2.0], [2.0], [NAN], [NAN], [5.0], [5.0]])
    assert oracle.detox_winner_slots(X, G3) == [2, 3, 8]
    for mode in ("coordinate_median", "trimmed_mean"):
        assert oracle.detox(X, G3, mode, oracle.captured_group_bound(3, 3)).tolist() == [2.0]
    assert oracle.detox(X, G3, "geometric_median", 1)[0] == pytest.approx(2.0, abs=1e-6)


@pytest.mark.parametrize("mode", DETOX_MODES)
def test_group_size_one_is_the_baseline_rule(mode):
    """With group size 1 every worker is its own group, b_G = f, and DETOX is the baseline rule on the same rows."""
    rng = np.random.default_rng(7)
    P, f = 7, 2
    X = rng.normal(size=(P, 11))
    X[3] *= -100
    X[5] = 50.0
    groups = [[w] for w in range(1, P + 1)]
    got = oracle.detox(X, groups, mode, oracle.captured_group_bound(f, 1))
    want = {"coordinate_median": lambda: oracle.coordinate_median(X), "trimmed_mean": lambda: oracle.trimmed_mean(X, f),
            "multi_krum": lambda: oracle.multi_krum(X, f, P - f), "geometric_median": lambda: oracle.geometric_median(X)}[mode]()
    np.testing.assert_array_equal(got, want)
    # the library PS too: the detox job with group size 1 applies exactly what the baseline job applies
    L = _layout()
    S = poisoned(L, P, seed=3)
    base = _torch_ps(JobConfig(approach="baseline", mode=mode, num_workers=P, worker_fail=f, transport="gloo"), L).aggregate(S)
    det = _torch_ps(JobConfig(approach="detox", mode=mode, num_workers=P, group_size=1, worker_fail=f, transport="gloo"), L).aggregate(S)
    for a, b in zip(base, det):
        assert torch.equal(a, b)


# ------------------------------------------------------------------------------------------------ library-op PS
def _layout():
    return ArenaLayout.from_model(build_model("LeNet"), bf16=False, channels_last=True)


def _torch_ps(cfg, L):
    cfg.resolve(1)
    groups, _ = build_codes(cfg)
    return TorchPS(cfg, L, torch.device("cpu"), L.new_arena(torch.device("cpu")), groups, None)


def poisoned(L, P, seed):
    """[P, D] fp32 N(0, 1) rows with a -100x row and a 1e30 row (no group structure: every worker its own group)."""
    g = torch.Generator().manual_seed(seed)
    X = torch.randn(P, L.total, generator=g)
    X[1] *= -100
    X[P - 1] = 1e30
    X[:, ~torch.from_numpy(L.valid_mask())] = 0
    return X


def grouped_slab(L, groups, liars, attack, seed):
    """Every member of a group holds the group's N(0, 1) gradient; the workers in ``liars`` send err_simulation of it."""
    g = torch.Generator().manual_seed(seed)
    H = torch.randn(len(groups), L.total, generator=g)
    H[:, ~torch.from_numpy(L.valid_mask())] = 0
    P = sum(len(grp) for grp in groups)
    X = torch.empty(P, L.total)
    for gi, grp in enumerate(groups):
        for w in grp:
            row = H[gi].numpy()
            X[w - 1] = torch.from_numpy(err_simulation(row, attack) if w in liars else row.copy())
    return X, H


def _check_against_oracle(cfg, L, X):
    ps = _torch_ps(cfg, L)
    groups = group_assign(cfg.num_workers, cfg.group_size).groups
    out = ps.aggregate(X)
    Xn = X.double().numpy()
    # the library PS stops Weiszfeld at a relative step of 1e-6 (the oracle at 1e-8): a looser bound for the geometric median
    tol = 1e-4 if cfg.mode == "geometric_median" else 1e-6
    for spec, g in zip(L.specs, out):
        ref = oracle.detox(Xn[:, spec.offset:spec.offset + spec.numel], groups, cfg.mode, cfg.captured_group_bound)
        assert torch.isfinite(g).all() and np.isfinite(ref).all()
        np.testing.assert_allclose(g.double().numpy(), ref, rtol=10 * tol, atol=tol)


@pytest.mark.parametrize("mode", DETOX_MODES)
@pytest.mark.parametrize("P,r,f", [(9, 3, 2), (15, 3, 3), (12, 4, 2), (16, 2, 3), (11, 2, 1)])
def test_torch_ps_detox_matches_oracle(mode, P, r, f):
    cfg = JobConfig(approach="detox", mode=mode, num_workers=P, group_size=r, worker_fail=f, transport="gloo")
    try:
        cfg.resolve(1)
    except ValueError:
        assert mode == "multi_krum"                        # G <= 2 b_G + 2 at these sizes
        return
    groups = group_assign(P, r).groups
    # the first f workers lie: with r = 3 and f >= 2 that captures group 0
    X, _ = grouped_slab(_layout(), groups, set(range(1, f + 1)), "rev_grad", seed=P * 10 + f)
    _check_against_oracle(cfg, _layout(), X)


def _liar_subsets():
    for f in (2, 3):
        for liars in itertools.combinations(range(1, 10), f):
            yield f, set(liars)


@pytest.mark.parametrize("attack", ["rev_grad", "constant"])
def test_detox_coordinate_rules_stay_within_the_honest_groups_for_every_liar_subset(attack):
    """P = 9, r = 3, every liar subset of size 2 and 3 (36 + 84): at most b_G = 1 group is ever captured, and every coordinate of
    the DETOX median / trimmed mean lies within the range of the honest groups' gradients.  The vote average leaves it."""
    L = _layout()
    groups = group_assign(9, 3).groups
    ps = {(mode, f): _torch_ps(JobConfig(approach="detox", mode=mode, num_workers=9, group_size=3, worker_fail=f,
                                         transport="gloo"), L)
          for mode in ("coordinate_median", "trimmed_mean") for f in (2, 3)}
    vote_ps = _torch_ps(JobConfig(approach="maj_vote", mode="maj_vote", num_workers=9, group_size=3, worker_fail=2,
                                  transport="gloo"), L)
    def inside(out, lo, hi):
        return all(bool(((g >= lo[sp.offset:sp.offset + sp.numel]) & (g <= hi[sp.offset:sp.offset + sp.numel])).all())
                   for sp, g in zip(L.specs, out))
    n, vote_left = 0, 0
    for f, liars in _liar_subsets():
        captured = [gi for gi, grp in enumerate(groups) if len(liars & set(grp)) >= 2]
        assert len(captured) <= oracle.captured_group_bound(f, 3)
        X, H = grouped_slab(L, groups, liars, attack, seed=n % 7)
        honest = [gi for gi in range(3) if gi not in captured]
        lo, hi = H[honest].min(0).values, H[honest].max(0).values
        for mode in ("coordinate_median", "trimmed_mean"):
            assert inside(ps[(mode, f)].aggregate(X), lo, hi), (mode, f, sorted(liars))
        vote_left += int(not inside(vote_ps.aggregate(X), lo, hi))
        n += 1
    assert n == 36 + 84
    assert vote_left > 0


# ------------------------------------------------------------------------------------------------ configuration
def test_config_accepts_and_rejects_detox_jobs():
    def cfg(**kw):
        return JobConfig(**dict(dict(approach="detox", transport="nvl", num_workers=15, group_size=3, worker_fail=3), **kw))
    for mode in DETOX_MODES:                                  # G = 5, b_G = 1: every rule
        c = cfg(mode=mode).resolve(1)
        assert (c.num_groups, c.captured_group_bound, c.redundancy) == (5, 1, 3)
    for mode in ("normal", "maj_vote", "krum", "bogus"):
        with pytest.raises(ValueError, match="--approach detox takes --mode"):
            cfg(mode=mode).resolve(1)
    for mode in ("coordinate_median", "trimmed_mean", "geometric_median"):   # G = 2, b_G = 1
        with pytest.raises(ValueError, match="groups > 2\\*b_G"):
            cfg(mode=mode, num_workers=6, worker_fail=2).resolve(1)
        cfg(mode=mode, num_workers=9, worker_fail=2).resolve(1)               # G = 3, b_G = 1
    with pytest.raises(ValueError, match="Krum's condition"):
        cfg(mode="multi_krum", num_workers=12, worker_fail=2).resolve(1)      # G = 4 <= 2 b_G + 2
    cfg(mode="multi_krum", num_workers=15, worker_fail=2).resolve(1)
    with pytest.raises(ValueError, match="at most 16 groups"):
        cfg(mode="trimmed_mean", num_workers=17, group_size=1, worker_fail=1).resolve(1)
    cfg(mode="trimmed_mean", num_workers=17, group_size=1, worker_fail=1, transport="nccl").resolve(1)
    cfg(mode="trimmed_mean", num_workers=32, group_size=2, worker_fail=3).resolve(1)            # G = 16
    with pytest.raises(ValueError, match="at most 8"):                       # the vote kernel's group-size limit
        cfg(mode="trimmed_mean", num_workers=14, group_size=5, worker_fail=1, transport="nccl").resolve(1)
    with pytest.raises(ValueError, match="group_size <= num_workers"):
        cfg(mode="trimmed_mean", num_workers=4, group_size=5, worker_fail=0).resolve(1)
    # nccl_flat keeps implementing only the vote and the mean
    from draco_b200.parallel.flat_engine import FlatNcclEngine
    c = cfg(mode="coordinate_median", transport="nccl_flat", compress_grad="None").resolve(1)
    with pytest.raises(ValueError, match="nccl_flat implements the repetition-code vote and the plain mean.*approach=detox"):
        FlatNcclEngine(c, 0, 1, torch.device("cpu"), None)


def test_existing_configurations_resolve_as_before():
    c = JobConfig().resolve(8)
    assert (c.approach, c.mode, c.num_workers, c.redundancy, c.transport) == ("maj_vote", "normal", 7, 5, "nvl")
    c = JobConfig(approach="maj_vote", mode="maj_vote", group_size=3, num_workers=7, worker_fail=3).resolve(1)
    assert c.redundancy == 3 and c.num_groups == 2
    assert JobConfig(approach="baseline", mode="multi_krum", num_workers=7, worker_fail=2).resolve(1).redundancy == 1
    assert JobConfig(approach="cyclic", num_workers=7, worker_fail=2).resolve(1).redundancy == 5
    with pytest.raises(ValueError, match="at most 8"):
        JobConfig(approach="maj_vote", num_workers=14, group_size=5).resolve(1)
    with pytest.raises(ValueError, match="--approach must be one of"):
        JobConfig(approach="nope").resolve(1)


def test_batch_plan_gives_group_members_identical_batches():
    cfg = JobConfig(approach="detox", mode="trimmed_mean", num_workers=11, group_size=3, worker_fail=2, synthetic_size=4096,
                    transport="gloo").resolve(1)
    groups, _ = build_codes(cfg)
    plan = make_plan(cfg, None, groups)
    vote_plan = make_plan(JobConfig(approach="maj_vote", mode="maj_vote", num_workers=11, group_size=3, synthetic_size=4096), None,
                          groups)
    for step in (1, 2, 50):
        for grp in groups.groups:
            first = plan.indices(step, grp[0])[0]
            for w in grp:
                assert np.array_equal(plan.indices(step, w)[0], first)
                assert plan.batch_ids(step, w) == plan.batch_ids(step, grp[0])
                assert np.array_equal(vote_plan.indices(step, w)[0], first)        # the batches of maj_vote
        assert not np.array_equal(plan.indices(step, 1)[0], plan.indices(step, 4)[0])
    assert len(groups.groups[-1]) == 5                                              # the remainder joins the last group


# ------------------------------------------------------------------------------------------------ jobs
@pytest.mark.parametrize("mode", DETOX_MODES)
def test_detox_trains_under_attack_over_gloo(mode):
    P = 15 if mode == "multi_krum" else 9                    # multi-Krum needs G > 2 b_G + 2
    cfg = JobConfig(network="LeNet", dataset="MNIST", batch_size=16, max_steps=12, num_workers=P, transport="gloo", lr=0.05,
                    momentum=0.9, synthetic_size=512, eval_freq=10 ** 6, compress_grad="None", approach="detox", mode=mode,
                    group_size=3, worker_fail=2, err_mode="rev_grad")
    t = Trainer(cfg, rank=0, world=1, device=torch.device("cpu"), quiet=True)
    losses = [t.train_step()["loss"] for _ in range(12)]
    assert losses[-1] < losses[0], losses
    assert torch.isfinite(t.engine.master_params()).all()


def test_detox_as_a_multi_process_job(tmp_path):
    """1 PS + 6 workers (3 groups of 2) packed onto 2 Gloo processes, 3 steps."""
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""), OMP_NUM_THREADS="2")
    r = subprocess.run([sys.executable, "-m", "draco_b200.cli.distributed_nn", "--launch", "2", "--master-port", "29720", "--no-cuda",
                        "--network", "LeNet", "--dataset", "MNIST", "--num-workers", "6", "--batch-size", "8", "--max-steps", "3",
                        "--eval-freq", "1000", "--train-dir", str(tmp_path) + "/", "--synthetic-size", "128", "--log-interval", "1",
                        "--compress-grad", "None", "--approach", "detox", "--mode", "coordinate_median", "--group-size", "2",
                        "--worker-fail", "1", "--err-mode", "rev_grad"], capture_output=True, text=True, timeout=420, env=env, cwd=ROOT)
    out = r.stdout + r.stderr
    assert r.returncode == 0, out[-3000:]
    assert out.count("done at step 3") == 2, out[-2500:]
