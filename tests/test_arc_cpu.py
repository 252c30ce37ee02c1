"""Adaptive robust clipping (``--arc tensor | model``) on the CPU: the configuration, k, the oracle on hand-worked cases, the
library-op PS against the oracle for every rule at both scopes, a Gloo multi-process job, and the fused PS's launch plan."""
import argparse
import os
import subprocess
import sys
from fractions import Fraction

import numpy as np
import pytest
import torch

from draco_b200 import JobConfig
from draco_b200.codes import oracle
from draco_b200.config import APPROACHES, MODES, add_fit_args, config_from_args
from draco_b200.models import build_model
from draco_b200.ops import kernels as K
from draco_b200.parallel.arena import ArenaLayout
from draco_b200.parallel.ps import FusedPS, TorchPS, build_codes, rule_plan
from draco_b200.utils.checkpoint import load_checkpoint

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CPU = torch.device("cpu")


def _bits(x):
    return np.asarray(x, dtype=np.float32).view(np.int32)


def _cfg(**kw):
    base = dict(network="LeNet", dataset="MNIST", transport="gloo", compress_grad="None", approach="baseline", mode="normal",
                num_workers=7, worker_fail=1, arc="tensor")
    base.update(kw)
    return JobConfig(**base)


# ------------------------------------------------------------------------------------------------ configuration
def test_configuration_accepts_the_flag_and_rejects_every_misuse():
    ap = add_fit_args(argparse.ArgumentParser())
    assert ap.parse_args([]).arc is None and JobConfig().arc is None
    for scope in ("tensor", "model"):
        cfg = config_from_args(ap.parse_args(["--arc", scope, "--approach", "baseline", "--mode", "coordinate_median",
                                              "--num-workers", "15", "--worker-fail", "3", "--transport", "nvl"])).resolve(1)
        assert cfg.arc == scope and rule_plan(cfg).pipelined == (scope == "tensor")
    with pytest.raises(SystemExit):
        ap.parse_args(["--arc", "layer"])
    # every approach but cyclic, every transport but nccl_flat
    for approach, mode, r in (("baseline", "normal", 1), ("maj_vote", "maj_vote", 3), ("maj_vote", "normal", 3),
                              ("detox", "coordinate_median", 3), ("nnm", "multi_krum", 1)):
        for transport in ("nvl", "nccl", "gloo"):
            _cfg(approach=approach, mode=mode, group_size=r, num_workers=15, worker_fail=3, transport=transport).resolve(1)
    _cfg(mode="centered_clip", clip_tau=1.0, arc="model").resolve(1)
    _cfg(mode="krum", bucketing=2, num_workers=15, worker_fail=2).resolve(1)
    _cfg(err_mode="mimic", mode="coordinate_median", transport="nvl").resolve(1)
    _cfg(num_workers=40, worker_fail=5, transport="nccl").resolve(1)
    _cfg(worker_fail=0).resolve(1)                                       # k = 0: accepted, and a no-op

    def bad(match, **kw):
        with pytest.raises(ValueError, match=match):
            _cfg(**kw).resolve(1)
    bad("--arc must be one of", arc="layer")
    bad("--arc scales real gradient rows; the cyclic code's slots hold complex codewords", approach="cyclic")
    bad("--arc multiplies a row by a positive factor.*--mode sign_vote.*drop --arc", mode="sign_vote")
    bad("use --transport nvl or nccl for --arc", transport="nccl_flat", err_mode="none")
    bad("--arc on the nvl transport handles at most 16 workers.*use --transport nccl", num_workers=17, transport="nvl")
    bad("--arc clips .* needs 0 <= worker_fail <= num_workers", worker_fail=8)
    bad("--arc clips .* needs 0 <= worker_fail <= num_workers", worker_fail=-1)


def test_model_arc_takes_the_job_off_the_pipelined_ps_and_tensor_arc_does_not():
    for mode, kw in (("normal", {}), ("coordinate_median", {}), ("centered_clip", dict(clip_tau=1.0))):
        plans = {arc: rule_plan(_cfg(mode=mode, arc=arc, **kw).resolve(1)) for arc in (None, "tensor", "model")}
        assert plans[None].pipelined and plans["tensor"] == plans[None]
        assert not plans["model"].pipelined
        assert plans["model"] == plans[None].__class__(**dict(vars(plans[None]), pipelined=False))


# ------------------------------------------------------------------------------------------------ k
def test_k_over_every_worker_count_and_f():
    table = {P: [oracle.arc_k(P, f) for f in range(P + 1)] for P in range(1, 17)}
    for P, ks in table.items():
        for f, k in enumerate(ks):
            assert k == int(Fraction(2 * f * (P - f), P)), (P, f)       # floor, as an exact rational
            assert 0 <= k < P or P == 1
            if 2 * f <= P:
                assert k >= f, (P, f)
    assert table[15][3] == 4 and table[7][1] == 1 and table[16][3] == 4
    assert all(ks[0] == 0 and ks[-1] == 0 for ks in table.values())
    assert table[4] == [0, 1, 2, 1, 0] and table[16][8] == 8


# ------------------------------------------------------------------------------------------------ oracle
def test_the_k_largest_rows_are_clipped_to_the_next_norm():
    d = np.array([1.0, 25.0, 4.0, 9.0, 16.0])
    a = oracle.arc_row_factors(d, 2)                                   # d_tau = 9: rows of 25 and 16 go to norm 3
    assert a.tolist() == [1.0, np.float32(3 / 5), 1.0, 1.0, np.float32(3 / 4)]
    assert oracle.arc_row_factors(d, 0)[1] == 1.0                       # k = 0: d_tau is the largest, nothing above it


def test_ties_at_d_tau_are_not_clipped():
    d = np.array([4.0, 9.0, 9.0, 9.0, 1.0])
    assert oracle.arc_row_factors(d, 1).tolist() == [1.0] * 5           # d_tau = 9: no row is strictly above it
    assert oracle.arc_row_factors(d, 3).tolist() == [1.0, np.float32(2 / 3), np.float32(2 / 3), np.float32(2 / 3), 1.0]
    d = np.array([16.0, 16.0, 4.0])
    assert oracle.arc_row_factors(d, 1).tolist() == [1.0, 1.0, 1.0]


def test_nan_and_inf_rows():
    X = np.array([[3.0, 4.0], [np.nan, 0.0], [1.0, 0.0], [np.inf, 1.0], [0.0, 2.0], [0.5, 0.5]], dtype=np.float32)
    spans = [(0, 2)]
    assert oracle.arc_factors(X, spans, f=2)[0].tolist() == [1.0, 1.0, 1.0, 0.0, 1.0, 1.0]   # k = 2: NaN, Inf, then d_tau = 25
    a = oracle.arc_factors(X, spans, f=3)                               # k = 3: d_tau = 4, the norm-2 row
    assert oracle.arc_k(6, 2) == 2 and oracle.arc_k(6, 3) == 3
    assert a[0].tolist() == [np.float32(2 / 5), 1.0, 1.0, 0.0, 1.0, 1.0]
    Y = oracle.arc(X, spans, f=3)
    assert np.isnan(Y[1, 0]) and Y[1, 1] == 0                           # a NaN row stays NaN (factor 1)
    assert np.isnan(Y[3, 0]) and Y[3, 1] == 0                           # Inf * 0 = NaN, the finite elements become 0
    assert np.array_equal(_bits(Y[0]), _bits(X[0] * np.float32(0.4)))
    assert np.array_equal(_bits(Y[[2, 4, 5]]), _bits(X[[2, 4, 5]]))


def test_more_than_k_non_finite_rows_clip_nothing():
    X = np.array([[np.nan, 0.0], [np.inf, 1.0], [-np.inf, 1.0], [30.0, 40.0], [1.0, 0.0]], dtype=np.float32)
    assert oracle.arc_k(5, 1) == 1
    for f in (1, 2):                                                    # k = 1 or 2 <= 3 non-finite rows: d_tau is NaN or Inf
        assert oracle.arc_factors(X, [(0, 2)], f=f).tolist() == [[1.0] * 5]
        assert np.array_equal(_bits(oracle.arc(X, [(0, 2)], f=f)), _bits(X))


def test_k_zero_changes_nothing_and_padding_is_never_touched():
    rng = np.random.default_rng(0)
    X = rng.normal(size=(6, 40)).astype(np.float32) * np.arange(1, 7, dtype=np.float32)[:, None]
    spans = [(0, 10), (16, 20)]                                         # elements 10..15 and 36..39 are padding
    X[:, 10:16] = 7.0
    X[:, 36:] = -7.0
    assert np.array_equal(_bits(oracle.arc(X, spans, f=0)), _bits(X))
    for scope in ("tensor", "model"):
        Y = oracle.arc(X, spans, f=2, scope=scope)
        assert (Y[:, 10:16] == 7.0).all() and (Y[:, 36:] == -7.0).all()
        a = oracle.arc_factors(X, spans, f=2, scope=scope)
        assert (a < 1).sum(1).tolist() == [oracle.arc_k(6, 2)] * 2         # the largest rows here are distinct
        if scope == "model":
            assert np.array_equal(a[0], a[1])
        norms = [np.linalg.norm(Y[:, o:o + n].astype(np.float64), axis=1) for o, n in spans]
        if scope == "tensor":                                          # clipped rows land on the (k+1)-th norm
            for t, nrm in enumerate(norms):
                d_tau = np.sort(np.linalg.norm(X[:, spans[t][0]:sum(spans[t])].astype(np.float64), axis=1))[::-1][2]
                assert np.allclose(np.sort(nrm)[::-1][:3], d_tau, rtol=1e-6)


def test_model_scope_is_the_whole_model_norm():
    rng = np.random.default_rng(1)
    X = rng.normal(size=(9, 50)).astype(np.float32) * rng.uniform(0.1, 5, size=(9, 1)).astype(np.float32)
    spans = [(0, 13), (13, 37)]
    a = oracle.arc_factors(X, spans, f=2, scope="model")
    d = (X[:, :50].astype(np.float64) ** 2).sum(1)
    k = oracle.arc_k(9, 2)
    tau = np.sort(d)[::-1][k]
    want = np.where(d > tau, np.sqrt(tau) / np.sqrt(d), 1.0).astype(np.float32)
    assert np.allclose(a[0], want, rtol=2e-7, atol=0) and np.array_equal(a[0], a[1])


# ------------------------------------------------------------------------------------------------ library-op PS
def _layout():
    return ArenaLayout.from_model(build_model("LeNet"), bf16=False, channels_last=True)


SHAPES = ((15, 3, 3), (16, 1, 2))            # (16, 1, 2), for DETOX only: its Bulyan (8 groups, b_G = 1)


def _rule_configs(**kw):
    """Every (approach, mode) that resolves with --arc at every shape, bucketing and centered clipping included."""
    out = {}
    for P, f, r in SHAPES:
        for approach in APPROACHES if P == 15 else ("detox",):
            modes = {"cyclic": ("normal",), "maj_vote": ("normal", "maj_vote")}.get(approach, MODES)
            for mode in modes:
                for extra in ({}, dict(bucketing=2)) if approach == "baseline" else ({},):
                    tau = dict(clip_tau=2.0) if mode == "centered_clip" else {}
                    cfg = _cfg(approach=approach, mode=mode, num_workers=P, worker_fail=f, group_size=r, **extra, **tau, **kw)
                    try:
                        cfg.resolve(1)
                    except ValueError:
                        continue
                    out[f"{approach}/{mode}/P{P}f{f}r{r}{'/b2' if extra else ''}"] = cfg
    return out


def _slots(cfg, L, groups):
    g = torch.Generator().manual_seed(100 * cfg.num_workers + cfg.worker_fail)
    P = cfg.num_workers
    S = torch.randn(P, L.total, generator=g) * torch.rand(P, 1, generator=g) * 4
    S *= torch.from_numpy(L.valid_mask()).float()
    if groups is not None:                                              # replicas agree, then the first worker_fail workers lie
        for grp in groups.groups:
            for w in grp[1:]:
                S[w - 1] = S[grp[0] - 1]
    S[: cfg.worker_fail] = torch.randn(cfg.worker_fail, L.total, generator=g) * 50
    return S


def test_the_rule_configs_cover_every_approach_but_cyclic():
    cfgs = _rule_configs()
    assert {c.approach for c in cfgs.values()} == set(APPROACHES) - {"cyclic"}
    assert len({(c.approach, c.mode) for c in cfgs.values()}) >= 1 + 2 + 6 + 6 + 8


@pytest.mark.parametrize("scope", ["tensor", "model"])
def test_torch_ps_with_arc_equals_torch_ps_without_it_on_the_oracles_clip(scope):
    L = _layout()
    spans = [(s.offset, s.numel) for s in L.specs]
    for name, cfg in _rule_configs(arc=scope).items():
        groups, code = build_codes(cfg)
        S = _slots(cfg, L, groups)
        on = TorchPS(cfg, L, CPU, L.new_arena(CPU), groups, code)
        off_cfg = _cfg(**dict(vars(cfg), arc=None)).resolve(1)
        off = TorchPS(off_cfg, L, CPU, L.new_arena(CPU), groups, code)
        clipped = torch.from_numpy(oracle.arc(S.numpy(), spans, cfg.worker_fail, scope))
        assert not torch.equal(clipped, S), name                           # the liars' rows are the largest: k >= 1 of them clip
        slots = S.clone()
        got = on.aggregate(slots, step=1)
        want = off.aggregate(clipped.clone(), step=1)
        assert torch.equal(slots.view(torch.int32), clipped.view(torch.int32)), name   # clipped in place
        assert len(got) == len(want)
        for t, (a, b) in enumerate(zip(got, want)):
            assert torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32)), (name, t)


def test_torch_ps_at_f_zero_leaves_the_slots_alone():
    L = _layout()
    cfg = _cfg(mode="coordinate_median", worker_fail=0).resolve(1)
    ps = TorchPS(cfg, L, CPU, L.new_arena(CPU), None, None)
    S = torch.randn(7, L.total)
    S[0] *= 100
    slots = S.clone()
    ps.aggregate(slots)
    assert torch.equal(slots, S) and "arc_factors" not in ps.last_info


# ------------------------------------------------------------------------------------------------ multi-process
def test_multi_process_job_equals_the_single_process_job(tmp_path):
    """1 PS + 2 worker processes over Gloo against one process hosting everything, with --arc tensor under ALIE: the same
    parameters at step 3."""
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""), OMP_NUM_THREADS="1")
    common = ["-m", "draco_b200.cli.distributed_nn", "--no-cuda", "--network", "LeNet", "--dataset", "MNIST", "--num-workers", "5",
              "--batch-size", "8", "--max-steps", "3", "--eval-freq", "3", "--synthetic-size", "128", "--log-interval", "1",
              "--compress-grad", "None", "--approach", "baseline", "--mode", "coordinate_median", "--arc", "tensor",
              "--worker-fail", "1", "--err-mode", "alie"]
    blobs = []
    for name, extra in (("multi", ["--launch", "3", "--master-port", "29781"]), ("single", [])):
        d = str(tmp_path / name) + "/"
        r = subprocess.run([sys.executable, *common, "--train-dir", d, *extra], capture_output=True, text=True, timeout=420,
                           env=env, cwd=ROOT)
        assert r.returncode == 0, (r.stdout[-2000:], r.stderr[-3000:])
        blobs.append(load_checkpoint(d + "model_step_3"))
    multi, single = blobs
    assert single["config"]["arc"] == "tensor"
    for k, v in single["state_dict"].items():
        assert torch.equal(multi["state_dict"][k], v), k


# ------------------------------------------------------------------------------------------------ fused PS launch plan
RECORDED = ("vote", "aggregate_update", "krum_select", "bulyan_select", "geometric_median_weights", "geometric_median", "nnm_mix",
            "nnm_mix_table", "nnm_fold", "pair_dist", "pair_scope_fold", "ps_attack", "ps_attack_model", "mimic_step",
            "centered_clip_dist", "centered_clip_weights", "centered_clip_model_weights", "centered_clip_update", "wbucket_plan",
            "wbucket_update", "wbucket_cc_dist", "wbucket_cc_update", "wbucket_table", "wbucket_fold", "arc_clip")
# what the launchers that report their own count return
COUNTS = {"ps_attack": lambda args: 1, "ps_attack_model": lambda args: 4, "mimic_step": lambda args: 6,
          "arc_clip": lambda args: 4 if args[5].dist is not None else 3}


def _record(cfg, monkeypatch, bucketed):
    """FusedPS.enqueue_step with every launcher replaced by a recorder: (launcher, tile_range, tensor_range) per call."""
    L = _layout()
    calls = []

    def rec(name):
        def f(*args, **kw):
            calls.append((name, kw.get("tile_range"), kw.get("tensor_range")))
            if name == "arc_clip":
                assert args[3:5] == (cfg.num_workers, oracle.arc_k(cfg.num_workers, cfg.worker_fail))
            return COUNTS[name](args) if name in COUNTS else None
        return f
    for name in RECORDED:
        monkeypatch.setattr(K, name, rec(name))
    groups, code = build_codes(cfg)
    P = cfg.num_workers
    ps = FusedPS(cfg, L, CPU, L.new_arena(CPU), torch.zeros(P, L.total), groups, code,
                 adv_bitmap=torch.zeros(8, dtype=torch.int32), adv_len=8)
    buckets = [(0, 3, [0, 1]), (3, 7, [2, 3, 4]), (7, 12, list(range(5, L.ntensors)))]
    kw = dict(buckets=buckets, wait_bucket=lambda b: calls.append(("wait", b, None)) or 1) if bucketed else {}
    n = ps.enqueue_step(torch.ones(1, dtype=torch.int64), mc_params=None, dst=[4096], flags=[16, 32],
                        before_update=lambda: calls.append(("before_update", None, None)) or 1, **kw)
    return ps, calls, n


PLAN_CASES = [dict(mode="normal"), dict(mode="coordinate_median", err_mode="alie"), dict(mode="multi_krum"),
              dict(mode="centered_clip", clip_tau=1.0, err_mode="minmax"), dict(mode="bulyan", num_workers=16, worker_fail=3),
              dict(approach="detox", mode="coordinate_median", group_size=3), dict(approach="maj_vote", mode="maj_vote", group_size=3),
              dict(approach="nnm", mode="coordinate_median"), dict(mode="coordinate_median", bucketing=2),
              dict(mode="centered_clip", clip_tau=1.0, bucketing=2), dict(mode="krum", rule_scope="model")]


def _plan_cfg(**kw):
    base = dict(num_workers=15, worker_fail=3, transport="nvl")
    base.update(kw)
    return _cfg(**base).resolve(1)


@pytest.mark.parametrize("bucketed", [False, True])
@pytest.mark.parametrize("case", PLAN_CASES, ids=lambda c: "-".join(f"{v}" for v in c.values()))
def test_tensor_arc_adds_three_launches_per_bucket_right_after_the_attack(monkeypatch, case, bucketed):
    ps0, off, n0 = _record(_plan_cfg(arc=None, **case), monkeypatch, bucketed)
    ps, on, n = _record(_plan_cfg(arc="tensor", **case), monkeypatch, bucketed)
    assert ps.plan == ps0.plan and ps.arc_k == 4 and ps.arc_ws.dist is None
    assert ps.arc_ws.partials.shape == (_layout().ntiles, ps.P) and ps.arc_ws.factors.shape == (_layout().ntensors, ps.P)
    arcs = [i for i, c in enumerate(on) if c[0] == "arc_clip"]
    assert [c for c in on if c[0] != "arc_clip"] == off
    pipelined = bucketed and ps.plan.pipelined
    buckets = [((0, 3), (0, 2)), ((3, 7), (2, 5)), ((7, 12), (5, _layout().ntensors))] if pipelined else [(None, None)]
    assert [on[i][1:] for i in arcs] == buckets
    for i in arcs:                                # after the bucket's wait and attack, before its row source and rule
        j = i - 1
        if on[j][0] in ("ps_attack", "ps_attack_model", "mimic_step"):
            j -= 1
        assert j < 0 or on[j][0] in ("wait", "wbucket_plan", "aggregate_update", "centered_clip_update", "wbucket_update",
                                     "wbucket_cc_update"), on[j]
    assert n == n0 + 3 * len(buckets)


@pytest.mark.parametrize("bucketed", [False, True])
@pytest.mark.parametrize("case", PLAN_CASES, ids=lambda c: "-".join(f"{v}" for v in c.values()))
def test_model_arc_adds_four_launches_once_and_no_pipelining(monkeypatch, case, bucketed):
    _, off, n0 = _record(_plan_cfg(arc=None, **case), monkeypatch, False)     # the whole-arena plan of the same rule
    ps, on, n = _record(_plan_cfg(arc="model", **case), monkeypatch, bucketed)
    assert not ps.plan.pipelined and ps.arc_ws.dist.shape == (_layout().ntensors, ps.P)
    assert [c for c in on if c[0] != "arc_clip"] == off
    assert [c for c in on if c[0] == "arc_clip"] == [("arc_clip", None, None)]
    assert n == n0 + 4


@pytest.mark.parametrize("scope", ["tensor", "model"])
@pytest.mark.parametrize("case", PLAN_CASES[:4], ids=lambda c: "-".join(f"{v}" for v in c.values()))
def test_f_zero_launches_nothing_and_allocates_nothing(monkeypatch, case, scope):
    case = dict(case, worker_fail=0)
    if case.get("err_mode") in ("minmax",):
        case.pop("err_mode")
    ps0, off, n0 = _record(_plan_cfg(arc=None, **case), monkeypatch, True)
    ps, on, n = _record(_plan_cfg(arc=scope, **case), monkeypatch, True)
    assert ps.arc_k == 0 and ps.arc_ws is None
    assert on == off and n == n0 and ps.plan.pipelined == ps0.plan.pipelined


def test_arc_clip_takes_no_bucket_at_model_scope():
    L = _layout()
    ws = K.ArcWorkspace(L, 5, CPU, model=True)
    with pytest.raises(ValueError, match="takes no bucket"):
        K.arc_clip(L, torch.zeros(5, L.total), L.total, 5, 1, ws, tile_range=(0, 3))
    with pytest.raises(ValueError, match="takes 1..16 rows"):
        K.ArcWorkspace(L, 17, CPU, model=False)
