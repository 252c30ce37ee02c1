"""Worker buckets (``--bucketing s``) on the CPU: the configuration rules, the permutation schedule, the oracle against
``TorchPS`` on every accepted mode, s = 1 against the baseline, the fused PS's launch plan, and a multi-process Gloo job with
checkpoint / resume."""
import os
import socket
import subprocess
import sys

import numpy as np
import pytest
import torch

from draco_b200 import JobConfig
from draco_b200.codes import oracle
from draco_b200.codes.bucketing import bucket_schedule, wbucket_masks, wbuckets
from draco_b200.models import build_model
from draco_b200.ops import kernels as K
from draco_b200.parallel.arena import ArenaLayout
from draco_b200.parallel.ps import FusedPS, TorchPS, rule_plan
from draco_b200.parallel.trainer import Trainer
from draco_b200.utils.checkpoint import load_checkpoint

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CPU = torch.device("cpu")


def _cfg(**kw):
    base = dict(network="LeNet", dataset="MNIST", batch_size=16, max_steps=12, transport="gloo", lr=0.05, momentum=0.0,
                synthetic_size=512, eval_freq=10 ** 6, compress_grad="None", approach="baseline", mode="coordinate_median",
                num_workers=7, worker_fail=1, err_mode="rev_grad", bucketing=2)
    base.update(kw)
    if base["mode"] == "centered_clip":
        base.setdefault("clip_tau", 0.5)
    return JobConfig(**base)


def _layout():
    return ArenaLayout.from_model(build_model("LeNet"), bf16=False, channels_last=True)


# ------------------------------------------------------------------------------------------------ configuration
def test_configuration_accepts_the_rules_and_bounds_over_nb():
    # P = 15, f = 3, s = 2: nb = 8 admits the coordinate rules, the geometric median and centered clipping, not Krum
    for mode in ("coordinate_median", "trimmed_mean", "geometric_median", "centered_clip"):
        cfg = _cfg(mode=mode, num_workers=15, worker_fail=3).resolve(1)
        assert rule_plan(cfg).rows == 8 and rule_plan(cfg).source == "wbucket"
    for mode in ("krum", "multi_krum"):
        with pytest.raises(ValueError, match=r"needs nb > 2\*worker_fail \+ 2"):
            _cfg(mode=mode, num_workers=15, worker_fail=3).resolve(1)
        assert rule_plan(_cfg(mode=mode, num_workers=15, worker_fail=2).resolve(1)).rows == 8
    with pytest.raises(ValueError, match=r"needs nb > 2\*worker_fail \(the honest"):
        _cfg(num_workers=15, worker_fail=3, bucketing=3).resolve(1)          # nb = 5
    plan = rule_plan(_cfg(num_workers=15, worker_fail=3).resolve(1))
    assert (plan.trim, plan.f, plan.pipelined) == (3, 3, True)
    assert rule_plan(_cfg(mode="multi_krum", num_workers=15, worker_fail=2).resolve(1)).m == 6
    # the library path takes more than 16 workers, the nvl PS does not
    _cfg(num_workers=20, worker_fail=2, bucketing=2).resolve(1)
    with pytest.raises(ValueError, match="at most 16 workers"):
        _cfg(num_workers=20, worker_fail=2, bucketing=2, transport="nvl").resolve(1)


@pytest.mark.parametrize("kw,msg", [
    (dict(mode="normal"), "--bucketing takes --mode"),
    (dict(mode="bulyan", num_workers=15), "--bucketing takes --mode"),
    (dict(mode="sign_vote"), "--bucketing takes --mode"),
    (dict(approach="nnm"), "use --approach baseline"),
    (dict(approach="detox", group_size=3), "use --approach baseline"),
    (dict(approach="maj_vote", mode="maj_vote", group_size=3), "use --approach baseline"),
    (dict(transport="nccl_flat"), "nccl_flat"),
    (dict(bucketing=-1), "1 <= s <= num_workers"),
    (dict(bucketing=8), "1 <= s <= num_workers"),
    (dict(transport="nvl", mode="krum"), r"needs nb > 2\*worker_fail \+ 2"),
])
def test_configuration_rejects_every_misuse(kw, msg):
    with pytest.raises(ValueError, match=msg):
        _cfg(**kw).resolve(1)


def test_flag_unset_changes_no_plan():
    for mode in ("coordinate_median", "krum", "centered_clip"):
        a = rule_plan(_cfg(mode=mode, bucketing=0).resolve(1))
        assert a.source == "raw" and a.rows == 7 and not a.rule.startswith("wbucket")


# ------------------------------------------------------------------------------------------------ schedule
def test_schedule_is_a_permutation_per_step_and_deterministic_in_the_seed():
    S = bucket_schedule(9, 20, 1)
    assert S.shape == (21, 9) and S.dtype == np.int32
    assert all(sorted(r) == list(range(9)) for r in S)
    assert np.array_equal(S, bucket_schedule(9, 20, 1)) and not np.array_equal(S, bucket_schedule(9, 20, 2))
    assert len({tuple(r) for r in S}) > 10


def test_buckets_are_ordered_by_their_lowest_member():
    perm = [5, 2, 0, 6, 1, 4, 3]
    assert wbuckets(perm, 2) == [[0, 6], [1, 4], [2, 5], [3]]
    assert wbuckets(perm, 1) == [[j] for j in range(7)]
    assert wbuckets(perm, 3) == [[0, 2, 5], [1, 4, 6], [3]]
    assert wbucket_masks(perm, 3).tolist() == [0b0100101, 0b1010010, 0b0001000]
    assert wbuckets(perm, 7) == [list(range(7))]


def test_one_member_row_is_its_member_bit_for_bit_and_others_round_in_fp32():
    X = np.array([[np.nan, -0.0, 1e-45], [1.0, 2.0, 3.0], [1e38, 3e38, -0.0]], dtype=np.float32)
    Y = oracle.wbucket_rows(X, [[0], [1, 2]])
    assert np.array_equal(Y[0].view(np.int32), X[0].view(np.int32))
    want = np.multiply(np.add(X[1], X[2], dtype=np.float32), np.float32(0.5), dtype=np.float32)
    assert np.array_equal(Y[1].view(np.int32), want.view(np.int32))


def test_bucket_table_from_the_raw_table_matches_the_rows():
    rng = np.random.default_rng(0)
    X = rng.standard_normal((7, 40)).astype(np.float32)
    B = wbuckets(rng.permutation(7), 3)
    Y = oracle.wbucket_rows(X, B).astype(np.float64)
    Db = oracle.wbucket_pair_d2(oracle._raw_d2(X), B, 7)
    want = ((Y[:, None] - Y[None]) ** 2).sum(2)
    np.testing.assert_allclose(Db, want, rtol=1e-5, atol=1e-5)


# ------------------------------------------------------------------------------------------------ oracle vs TorchPS
def _slots(P, d, seed, liars=()):
    g = torch.Generator().manual_seed(seed)
    S = torch.randn(P, d, generator=g)
    for w in liars:
        S[w] = -100.0 * S[w]
    return S


@pytest.mark.parametrize("mode", ["coordinate_median", "trimmed_mean", "krum", "multi_krum", "geometric_median",
                                  "centered_clip"])
@pytest.mark.parametrize("P,f,s", [(9, 1, 2), (12, 1, 2), (16, 1, 3)])
def test_torch_ps_equals_the_oracle(mode, P, f, s):
    cfg = _cfg(mode=mode, num_workers=P, worker_fail=f, bucketing=s).resolve(1)
    L = _layout()
    ps = TorchPS(cfg, L, CPU, L.new_arena(CPU), None, None)
    for step in (1, 2, 5):
        S = _slots(P, L.total, 100 * step + P, liars=(0,))
        centers = [ps.cc_center[sp.offset: sp.offset + sp.numel].clone() for sp in L.specs] if ps.cc_center is not None else None
        out = ps.aggregate(S, step=step)
        perm = ps.wb_schedule[step % len(ps.wb_schedule)]
        for i, sp in enumerate(L.specs):
            X = S[:, sp.offset: sp.offset + sp.numel].numpy()
            kw = dict(center=centers[i].numpy(), tau=cfg.clip_tau) if mode == "centered_clip" else {}
            want = oracle.bucketing(X, perm, s, f, mode, **kw)
            got = out[i].numpy()
            if mode == "centered_clip" or (mode == "coordinate_median" and rule_plan(cfg).rows % 2):
                assert np.array_equal(got.view(np.int32), np.asarray(want, dtype=np.float32).view(np.int32))
            else:
                np.testing.assert_allclose(got, want, rtol=2e-5, atol=2e-5)


def test_torch_ps_needs_the_step():
    cfg = _cfg().resolve(1)
    L = _layout()
    with pytest.raises(ValueError, match="needs the step"):
        TorchPS(cfg, L, CPU, L.new_arena(CPU), None, None).aggregate(torch.zeros(7, L.total))


@pytest.mark.parametrize("mode", ["coordinate_median", "trimmed_mean", "centered_clip"])
def test_s_equal_one_is_the_baseline_rule(mode):
    L = _layout()
    S = _slots(7, L.total, 3, liars=(2,))
    got = TorchPS(_cfg(mode=mode, bucketing=1).resolve(1), L, CPU, L.new_arena(CPU), None, None).aggregate(S, step=4)
    want = TorchPS(_cfg(mode=mode, bucketing=0).resolve(1), L, CPU, L.new_arena(CPU), None, None).aggregate(S)
    for a, b in zip(got, want):
        assert torch.equal(a, b)


@pytest.mark.parametrize("mode", ["krum", "multi_krum", "geometric_median", "centered_clip"])
def test_model_scope_equals_the_oracle_on_the_whole_model(mode):
    cfg = _cfg(mode=mode, rule_scope="model", num_workers=9, worker_fail=1, bucketing=2).resolve(1)
    L = _layout()
    ps = TorchPS(cfg, L, CPU, L.new_arena(CPU), None, None)
    S = _slots(9, L.total, 11, liars=(4,))
    out = ps.aggregate(S, step=3)
    perm = ps.wb_schedule[3]
    spans = [(sp.offset, sp.offset + sp.numel) for sp in L.specs]
    X = np.concatenate([S[:, a:b].numpy() for a, b in spans], axis=1)
    if mode == "centered_clip":
        want = oracle.bucketing(X, perm, 2, 1, mode, center=np.zeros(X.shape[1], np.float32), tau=cfg.clip_tau)
    else:
        D = oracle.model_d2([oracle._raw_d2(S[:, a:b].numpy()) for a, b in spans])
        want = oracle.bucketing(X, perm, 2, 1, mode, D=D)
    got = np.concatenate([o.numpy() for o in out])
    np.testing.assert_allclose(got, want, rtol=2e-5, atol=2e-5)


# ------------------------------------------------------------------------------------------------ fused PS launch plan
def _record(cfg, monkeypatch, buckets):
    L = _layout()
    calls = []

    def rec(name):
        def f(*args, **kw):
            calls.append((name, {k: v for k, v in kw.items() if k in ("tile_range", "trim", "flags", "tensor_range", "K", "m")}))
            return 1 if name == "ps_attack" else None
        return f
    for name in ("ps_attack", "wbucket_plan", "wbucket_update", "aggregate_update", "pair_dist", "pair_scope_fold", "krum_select",
                 "geometric_median_weights", "wbucket_table", "wbucket_fold", "wbucket_cc_dist", "centered_clip_weights",
                 "centered_clip_model_weights", "wbucket_cc_update", "centered_clip_dist", "centered_clip_update"):
        monkeypatch.setattr(K, name, rec(name))
    P = cfg.num_workers
    ps = FusedPS(cfg, L, CPU, L.new_arena(CPU), torch.zeros(P, L.total), None, None, adv_bitmap=torch.zeros(8, dtype=torch.int32),
                 adv_len=8)
    kw = dict(buckets=buckets, wait_bucket=lambda b: calls.append(("wait", b)) or 1) if buckets else {}
    n = ps.enqueue_step(torch.ones(1, dtype=torch.int64), mc_params=None, dst=[4096], flags=[16, 32],
                        before_update=lambda: calls.append(("before_update",)) or 1, **kw)
    return ps, calls, n


@pytest.mark.parametrize("mode", ["coordinate_median", "trimmed_mean"])
@pytest.mark.parametrize("err", ["rev_grad", "alie"])
@pytest.mark.parametrize("bucketed", [False, True])
def test_fused_ps_plans_once_then_updates_per_gradient_bucket(monkeypatch, mode, err, bucketed):
    cfg = _cfg(mode=mode, num_workers=15, worker_fail=3, transport="nvl", err_mode=err).resolve(1)
    L = _layout()
    buckets = [(0, 3, [0, 1]), (3, 7, [2, 3, 4]), (7, 12, list(range(5, L.ntensors)))] if bucketed else None
    ps, calls, n = _record(cfg, monkeypatch, buckets)
    assert ps.plan.pipelined and ps.wb_schedule.shape == (cfg.max_steps + 1, 15) and ps.wb_mask.shape == (8,)
    ranges = [((t0, t1), (min(i), max(i) + 1)) for t0, t1, i in buckets] if bucketed else [(None, None)]
    want = [("wbucket_plan", {})]
    for bi, (tiles, tensors) in enumerate(ranges):
        last = bi == len(ranges) - 1
        if bucketed:
            want.append(("wait", bi))
        if err == "alie":
            want.append(("ps_attack", {"tile_range": tiles, "tensor_range": tensors}))
        if last:
            want.append(("before_update",))
        want.append(("wbucket_update", {"tile_range": tiles, "trim": ps.plan.trim, "flags": [16, 32] if last else []}))
    assert calls == want
    assert n == 1 + len(ranges) * (1 + int(bucketed) + int(err == "alie")) + 1


# ------------------------------------------------------------------------------------------------ jobs
def test_training_is_deterministic_and_resume_is_bit_for_bit(tmp_path):
    d = str(tmp_path) + "/"
    kw = dict(train_dir=d, max_steps=6, mode="trimmed_mean")
    t = Trainer(_cfg(eval_freq=3, **kw), rank=0, world=1, device=CPU, quiet=True)
    t.fit(6)
    final = t.engine.master_params().clone()
    assert load_checkpoint(d + "model_step_3")["opt_state"] == {}            # no new PS state
    t2 = Trainer(_cfg(eval_freq=10 ** 6, checkpoint_step=3, **kw), rank=0, world=1, device=CPU, quiet=True)
    for _ in range(3):
        t2.train_step()
    assert torch.equal(t2.engine.master_params(), final)


def _free_port() -> int:
    with socket.socket() as sk:
        sk.bind(("127.0.0.1", 0))
        return sk.getsockname()[1]


def test_multi_process_gloo_job_equals_the_single_process_job_and_resumes(tmp_path):
    """1 PS + 2 worker processes over Gloo against one process hosting everything, then a resume from step 2 of the
    multi-process run: the same parameters at step 3."""
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""), OMP_NUM_THREADS="1")
    common = ["-m", "draco_b200.cli.distributed_nn", "--no-cuda", "--network", "LeNet", "--dataset", "MNIST", "--num-workers", "5",
              "--batch-size", "8", "--max-steps", "3", "--synthetic-size", "128", "--log-interval", "1",
              "--compress-grad", "None", "--approach", "baseline", "--mode", "centered_clip", "--clip-tau", "0.1",
              "--worker-fail", "1", "--err-mode", "alie", "--bucketing", "2", "--momentum", "0"]
    blobs = []
    for name, extra in (("multi", ["--eval-freq", "1", "--launch", "3", "--master-port", str(_free_port())]),
                        ("single", ["--eval-freq", "3"]),
                        ("multi", ["--eval-freq", "1", "--checkpoint-step", "2", "--launch", "3", "--master-port", str(_free_port())])):
        d = str(tmp_path / name) + "/"
        r = subprocess.run([sys.executable, *common, "--train-dir", d, *extra], capture_output=True, text=True, timeout=420,
                           env=env, cwd=ROOT)
        assert r.returncode == 0, (r.stdout[-2000:], r.stderr[-3000:])
        blobs.append(load_checkpoint(d + "model_step_3"))
    multi, single, resumed = blobs
    for k, v in single["state_dict"].items():
        assert torch.equal(multi["state_dict"][k], v), k
        assert torch.equal(resumed["state_dict"][k], v), k


@pytest.mark.parametrize("scope", ["tensor", "model"])
@pytest.mark.parametrize("bucketed", [False, True])
def test_fused_ps_centered_clip_over_buckets(monkeypatch, scope, bucketed):
    """Tensor scope: per gradient bucket, the bucket cc_dist + unchanged weights + mode 8.  Model scope: once, after the last
    gradient bucket, the bucket cc_dist over the arena + unchanged model weights + mode 8."""
    cfg = _cfg(mode="centered_clip", num_workers=15, worker_fail=3, transport="nvl", rule_scope=scope).resolve(1)
    L = _layout()
    buckets = [(0, 3, [0, 1]), (3, 7, [2, 3, 4]), (7, 12, list(range(5, L.ntensors)))] if bucketed else None
    ps, calls, n = _record(cfg, monkeypatch, buckets)
    assert ps.plan.pipelined == (scope == "tensor") and ps.cc_weights.shape == (L.ntensors, 8)
    names = [c[0] for c in calls]
    assert "centered_clip_dist" not in names and "centered_clip_update" not in names
    if scope == "model" or not bucketed:
        assert names == ["wbucket_plan", "wbucket_cc_dist", "centered_clip_model_weights" if scope == "model"
                                                           else "centered_clip_weights", "before_update", "wbucket_cc_update"]
    else:
        assert names == ["wbucket_plan"] + ["wait", "wbucket_cc_dist", "centered_clip_weights", "wbucket_cc_update"] * 2 + [
            "wait", "wbucket_cc_dist", "centered_clip_weights", "before_update", "wbucket_cc_update"]


@pytest.mark.parametrize("mode,scope", [("krum", "tensor"), ("multi_krum", "tensor"), ("geometric_median", "tensor"),
                                        ("multi_krum", "model"), ("geometric_median", "model")])
def test_fused_ps_distance_rules_over_buckets(monkeypatch, mode, scope):
    """After the last gradient bucket: the raw pair table (folded at model scope), the bucket table, the unchanged selection
    with filled=True, the fold into raw-slot weights, then the weighted-sum update."""
    cfg = _cfg(mode=mode, num_workers=15, worker_fail=2, transport="nvl", rule_scope=scope).resolve(1)
    L = _layout()
    buckets = [(0, 3, [0, 1]), (3, 7, [2, 3, 4]), (7, 12, list(range(5, L.ntensors)))]
    ps, calls, n = _record(cfg, monkeypatch, buckets)
    assert not ps.plan.pipelined and ps.pair_d2.shape == (L.ntensors, 28) and ps.wb_raw_d2.shape == (L.ntensors, 105)
    names = [c[0] for c in calls]
    choose = "geometric_median_weights" if mode == "geometric_median" else "krum_select"
    want = ["wbucket_plan", "pair_dist"] + (["pair_scope_fold"] if scope == "model" else []) + [
        "wbucket_table", choose, "wbucket_fold", "before_update", "aggregate_update"]
    assert names == want and n == len(want)
    upd = calls[-1][1]
    if mode == "geometric_median":
        assert upd["K"] == 15 and ps.w_raw.shape == (L.ntensors, 15)
    else:
        m = ps.plan.m
        assert upd["K"] == min(m * 2, 15) == ps.wb_wsel.shape[0] and calls[names.index("wbucket_fold")][1]["m"] == m


def test_vectorised_bucket_table_matches_the_oracle():
    from draco_b200.parallel.ps import _wbucket_table
    rng = np.random.default_rng(3)
    X = rng.standard_normal((11, 50)).astype(np.float32)
    B = wbuckets(rng.permutation(11), 3)
    D = oracle._raw_d2(X)
    np.testing.assert_allclose(_wbucket_table(D, B, 11), oracle.wbucket_pair_d2(D, B, 11), rtol=1e-12, atol=1e-12)
    D[2, 5] = D[5, 2] = np.nan                             # non-finite: the per-pair form keeps the NaN to the pairs it touches
    got = _wbucket_table(D, B, 11)
    assert np.array_equal(np.isnan(got), np.isnan(oracle.wbucket_pair_d2(D, B, 11))) and not np.isnan(got).all()
