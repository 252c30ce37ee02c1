"""Heterogeneous worker data (``--dirichlet-alpha``) on the CPU: the Dirichlet split, the holders' batches, and the IID plan
left as it was when the flag is unset."""
import json

import numpy as np
import pytest
import torch

from draco_b200 import JobConfig
from draco_b200.codes.repetition import group_assign
from draco_b200.data import BatchPlan, class_histograms, dirichlet_shards, synthetic_dataset
from draco_b200.parallel.fused_engine import make_plan
from draco_b200.parallel.trainer import Trainer


def _labels(n=8192, k=10, seed=0):
    return np.random.RandomState(seed).randint(0, k, n)


@pytest.mark.parametrize("H,alpha", [(15, 0.1), (15, 0.3), (7, 1.0), (3, 100.0)])
def test_shards_are_disjoint_cover_the_dataset_and_hold_a_batch(H, alpha):
    y = _labels()
    shards = dirichlet_shards(y, H, alpha, 128, seed=1)
    assert len(shards) == H and min(len(s) for s in shards) >= 128
    allidx = np.concatenate(shards)
    assert len(allidx) == len(y) and np.array_equal(np.sort(allidx), np.arange(len(y)))
    assert all(np.array_equal(a, b) for a, b in zip(shards, dirichlet_shards(y, H, alpha, 128, seed=1)))
    assert not all(np.array_equal(a, b) for a, b in zip(shards, dirichlet_shards(y, H, alpha, 128, seed=2)))


def test_large_alpha_is_near_uniform_and_small_alpha_is_skewed():
    y = _labels()
    def skew(alpha):
        h = np.array(class_histograms(y, dirichlet_shards(y, 8, alpha, 64, seed=3)), dtype=np.float64)
        p = h / h.sum(1, keepdims=True)
        return np.abs(p - 0.1).sum(1).mean()                # mean total-variation-like distance from uniform classes
    assert skew(1000.0) < 0.1
    assert skew(0.1) > 0.8


def test_an_impossible_split_names_its_sizes():
    with pytest.raises(ValueError, match=r"alpha 0.01.*512 samples over 15 holders.*B = 128"):
        dirichlet_shards(_labels(512), 15, 0.01, 128, seed=1)


def _plan(approach, alpha, P=6, r=3):
    cfg = JobConfig(approach=approach, mode="maj_vote" if approach == "maj_vote" else "coordinate_median", num_workers=P,
                    group_size=r, worker_fail=1, batch_size=16, dirichlet_alpha=alpha, network="LeNet", dataset="MNIST",
                    transport="gloo")
    groups = group_assign(P, r) if approach in ("maj_vote", "detox") else None
    return make_plan(cfg, synthetic_dataset("MNIST", 1024, seed=5), groups)


@pytest.mark.parametrize("approach", ["maj_vote", "detox"])
def test_group_members_share_their_holders_batches(approach):
    plan = _plan(approach, 0.5)
    assert len(plan.shards) == 2
    for step in (1, 2, 17, 40):
        for grp in ([1, 2, 3], [4, 5, 6]):
            b = [plan.indices(step, w)[0] for w in grp]
            assert all(np.array_equal(b[0], x) for x in b[1:]) and len(b[0]) == 16
        g0 = set(plan.shards[0].tolist())
        assert set(plan.indices(step, 1)[0].tolist()) <= g0


def test_each_worker_draws_from_its_own_shard_and_runs_epochs_over_it():
    plan = _plan("baseline", 0.5)
    assert len(plan.shards) == 6
    for w in range(1, 7):
        shard = plan.shards[w - 1]
        spe = len(shard) // 16
        epoch = np.concatenate([plan.indices(s, w)[0] for s in range(1, spe + 1)])
        assert len(np.unique(epoch)) == len(epoch) == spe * 16 and set(epoch.tolist()) <= set(shard.tolist())


def test_flag_unset_keeps_the_iid_plan():
    ds = synthetic_dataset("MNIST", 1024, seed=5)
    for approach, mode in (("baseline", "normal"), ("nnm", "coordinate_median"), ("maj_vote", "maj_vote"),
                           ("detox", "coordinate_median"), ("cyclic", "normal")):
        cfg = JobConfig(approach=approach, mode=mode, num_workers=6, group_size=3, worker_fail=1, batch_size=16)
        groups = group_assign(6, 3) if approach in ("maj_vote", "detox") else None
        plan = make_plan(cfg, ds, groups)
        ref = BatchPlan(approach, 1024, 16, 6, group_of=groups.rank_to_group if groups else None,
                        group_seeds=groups.seeds if groups else None, seed=428,
                        redundancy=cfg.redundancy if approach == "cyclic" else 1)
        assert plan.shards is None
        for step in (1, 5, 70):
            for w in range(1, 7):
                assert all(np.array_equal(a, b) for a, b in zip(plan.indices(step, w), ref.indices(step, w)))


def test_configuration_rejects_cyclic_and_bad_alpha():
    for a in (0.0, -1.0, float("inf"), float("nan")):
        with pytest.raises(ValueError, match="finite concentration > 0"):
            JobConfig(approach="baseline", num_workers=4, dirichlet_alpha=a).resolve(1)
    with pytest.raises(ValueError, match="cyclic"):
        JobConfig(approach="cyclic", num_workers=5, worker_fail=1, dirichlet_alpha=0.5).resolve(1)


def test_a_heterogeneous_job_trains_and_logs_the_histograms_once(tmp_path):
    path = str(tmp_path / "m.jsonl")
    cfg = JobConfig(network="LeNet", dataset="MNIST", batch_size=16, max_steps=4, transport="gloo", synthetic_size=512,
                    eval_freq=10 ** 6, compress_grad="None", approach="baseline", mode="coordinate_median", num_workers=5,
                    worker_fail=1, bucketing=2, dirichlet_alpha=0.3, metrics_file=path)
    t = Trainer(cfg, rank=0, world=1, device=torch.device("cpu"), quiet=True)
    for _ in range(3):
        m = t.train_step()
    t.close()
    recs = [json.loads(line) for line in open(path)]
    data = [r for r in recs if r["role"] == "data"]
    assert len(data) == 1 and len(data[0]["class_hist"]) == 5 and sum(map(sum, data[0]["class_hist"])) == 512
    assert m is None or np.isfinite(m["loss"])
