"""Whole-model scope (``--rule-scope model``, ``--attack-scope model``) on the CPU: the oracles (one tensor, the concatenation,
a hand-built case where the scopes disagree, NaN), the configuration, the library-op PS against the oracle over several steps
for every rule under baseline, DETOX and NNM, min-max's one gamma, Gloo jobs (single- against multi-process), checkpoint /
resume, and the fused PS's launch sequence and pipelining decision."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from draco_b200 import JobConfig
from draco_b200.codes import adversary as A
from draco_b200.codes import oracle
from draco_b200.config import APPROACHES, MODES
from draco_b200.models import build_model
from draco_b200.ops import kernels as K
from draco_b200.parallel.arena import ArenaLayout
from draco_b200.parallel.collective_engine import minmax_gamma_model
from draco_b200.parallel.fused_engine import pipelines_ps
from draco_b200.parallel.ps import PIPELINED_RULES, FusedPS, TorchPS, build_codes, rule_plan
from draco_b200.parallel.trainer import Trainer
from draco_b200.utils.checkpoint import load_checkpoint

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CPU = torch.device("cpu")
DISTANCE = ("krum", "multi_krum", "geometric_median", "bulyan", "centered_clip")


def _cfg(**kw):
    base = dict(network="LeNet", dataset="MNIST", batch_size=16, max_steps=12, transport="gloo", lr=0.05, momentum=0.0,
                synthetic_size=512, eval_freq=10 ** 6, compress_grad="None", approach="baseline", mode="multi_krum",
                num_workers=7, worker_fail=1, err_mode="rev_grad", rule_scope="model")
    base.update(kw)
    if base["mode"] == "centered_clip":
        base.setdefault("clip_tau", 2.0)
    return JobConfig(**base)


def _layout():
    return ArenaLayout.from_model(build_model("LeNet"), bf16=False, channels_last=True)


def _spans(L):
    return [(s.offset, s.numel) for s in L.specs]


def _rule(mode, P, f):
    """The per-tensor oracle of ``mode`` over P rows tolerating f, as a function of the rows."""
    return {"krum": lambda X: oracle.krum(X, f), "multi_krum": lambda X: oracle.multi_krum(X, f, P - f),
            "geometric_median": lambda X: oracle.geometric_median_weights(X) @ np.asarray(X, dtype=np.float64),
            "bulyan": lambda X: oracle.bulyan(X, f), "coordinate_median": oracle.coordinate_median,
            "trimmed_mean": lambda X: oracle.trimmed_mean(X, f)}[mode]


# ------------------------------------------------------------------------------------------------ oracles
def test_model_scope_on_a_one_tensor_layout_is_the_per_tensor_rule():
    rng = np.random.default_rng(0)
    X = rng.normal(size=(7, 50)).astype(np.float32)
    spans = [(0, 50)]
    for mode in ("krum", "multi_krum", "geometric_median", "bulyan"):
        assert np.array_equal(oracle.model_scope(_rule(mode, 7, 1), X, spans)[0], _rule(mode, 7, 1)(X)), mode
    for mode in oracle.NNM_MODES:
        assert np.array_equal(oracle.model_scope(oracle.nnm, X, spans, 1, mode)[0], oracle.nnm(X, 1, mode)), mode
    v = rng.normal(size=50).astype(np.float32)
    assert np.array_equal(oracle.model_scope(oracle.centered_clip, X, spans, v, 0.5)[0], oracle.centered_clip(X, v, 0.5))
    assert A.minmax_gamma_model([X[1:].astype(np.float64)]) == A.minmax_gamma(X[1:])


def test_model_distances_are_the_in_order_sum_of_the_tensor_distances():
    """model_d2 against the distances of the concatenated rows, for the pair table, the distances to a centre and min-max's
    terms; the selections made from either agree."""
    rng = np.random.default_rng(1)
    L = _layout()
    S = rng.normal(size=(7, L.total)).astype(np.float32) * rng.uniform(0.1, 3, size=(7, 1)).astype(np.float32)
    spans = _spans(L)
    M = oracle.model_rows(S, spans)
    assert M.shape == (7, sum(n for _, n in spans))
    D = oracle.model_d2([oracle._raw_d2(S[:, o:o + n]) for o, n in spans])
    assert np.allclose(D, oracle._raw_d2(M), rtol=1e-12, atol=0)
    assert oracle.multi_krum_indices(M, 1, 6) == [int(i) for i in np.argsort(oracle._krum_scores_d2(D, 1), kind="stable")[:6]]
    assert oracle.bulyan_indices(M, 1) == oracle._bulyan_rounds(D, 1)
    assert np.array_equal(oracle.nnm_neighbours(M, 2), oracle.nnm_neighbours_d2(D, 2))
    parts = [M[1:, o:o + n].astype(np.float64) for o, n in ((0, 100), (100, 1000), (1100, M.shape[1] - 1100))]
    assert A.minmax_gamma_model(parts) == pytest.approx(A.minmax_gamma(M[1:]), rel=1e-12)
    terms = oracle.model_d2([A.minmax_terms(H) for H in parts])
    assert np.allclose(terms, A.minmax_terms(M[1:]), rtol=1e-12, atol=1e-12)


def _disagreeing_slots():
    """Two tensors, P = 7, f = 1: worker 0 is far off in the small first tensor only, worker 1 farther off (in total) in the
    large second tensor only, so each tensor alone drops a different worker and the whole model drops worker 1."""
    rng = np.random.default_rng(2)
    S = rng.normal(size=(7, 40)).astype(np.float32) * 0.1
    S[0, :8] += 6.0
    S[1, 8:] += 4.0
    return S, [(0, 8), (8, 32)]


def test_the_scopes_choose_differently_on_a_hand_built_case():
    S, spans = _disagreeing_slots()
    T = [S[:, o:o + n] for o, n in spans]
    per_tensor = [oracle.multi_krum_indices(X, 1, 6) for X in T]
    assert 0 not in per_tensor[0] and 1 in per_tensor[0] and 1 not in per_tensor[1] and 0 in per_tensor[1]
    D = oracle.model_d2([oracle._raw_d2(X) for X in T])
    model = [int(i) for i in np.argsort(oracle._krum_scores_d2(D, 1), kind="stable")[:6]]
    assert 1 not in model and 0 in model
    # Bulyan's last round keeps f - 1 = 0 distances, so it takes the lowest remaining row whatever its distance
    assert oracle.bulyan_indices(T[0], 1) != oracle.bulyan_indices(T[1], 1) != oracle._bulyan_rounds(D, 1)
    A_t = [oracle.nnm_neighbours(X, 2) for X in T]
    A_m = oracle.nnm_neighbours_d2(D, 2)
    assert not np.array_equal(A_t[0], A_t[1]) and not np.array_equal(A_m, A_t[0])
    got = oracle.model_scope(lambda X: oracle.multi_krum(X, 1, 6), S, spans)
    assert np.allclose(np.concatenate(got), S[model].astype(np.float64).mean(0))


def test_nan_in_one_tensor_puts_that_row_last_in_every_tensor():
    S, spans = _disagreeing_slots()
    S[4, 20] = np.nan                                        # second tensor only
    D = oracle.model_d2([oracle._raw_d2(S[:, o:o + n]) for o, n in spans])
    assert np.isnan(D[4, [0, 1, 2, 3, 5, 6]]).all()
    order = np.argsort(oracle._krum_scores_d2(D, 1), kind="stable")
    assert order[-1] == 4
    assert 4 not in oracle._bulyan_rounds(D, 1)
    assert not oracle.nnm_neighbours_d2(D, 1)[[0, 1, 2, 3, 5, 6], 4].any()
    cfg = _cfg(num_workers=7, worker_fail=1).resolve(1)
    L = _layout()
    slots = torch.randn(7, L.total, generator=torch.Generator().manual_seed(3))
    slots[4, L.specs[-1].offset] = float("nan")
    out = TorchPS(cfg, L, CPU, L.new_arena(CPU), None, None).aggregate(slots)
    assert all(torch.isfinite(g).all() for g in out)


# ------------------------------------------------------------------------------------------------ configuration
def test_configuration_accepts_the_distance_rules_and_rejects_every_misuse():
    assert JobConfig().rule_scope == "tensor" and JobConfig().attack_scope == "tensor"
    ok, rejected = [], []
    for approach in APPROACHES:
        for mode in MODES:
            kw = dict(approach=approach, mode=mode, num_workers=15, worker_fail=3, group_size=3, transport="nvl")
            if mode == "centered_clip":
                kw["clip_tau"] = 1.0
            try:
                JobConfig(**kw).resolve(1)
            except ValueError:
                continue                                     # not a valid job at the default scope either (DETOX's Bulyan: 5 groups)
            try:
                JobConfig(rule_scope="model", **kw).resolve(1)
                ok.append((approach, mode))
            except ValueError as e:
                assert "coordinate-wise, so the scope would change nothing" in str(e), (approach, mode, e)
                rejected.append((approach, mode))
    assert sorted(ok) == sorted([("baseline", m) for m in DISTANCE] + [("detox", m) for m in DISTANCE if m not in ("krum", "bulyan")]
                                + [("nnm", m) for m in oracle.NNM_MODES])
    assert ("baseline", "coordinate_median") in rejected and ("detox", "trimmed_mean") in rejected
    assert ("maj_vote", "maj_vote") in rejected and ("cyclic", "normal") in rejected and ("baseline", "normal") in rejected

    def bad(match, **kw):
        with pytest.raises(ValueError, match=match):
            _cfg(**kw).resolve(1)
    bad("--rule-scope must be one of", rule_scope="layer")
    bad("--attack-scope must be one of", attack_scope="global", err_mode="minmax")
    for err in ("alie", "rev_grad", "none"):
        bad("--attack-scope model sets one gamma", attack_scope="model", err_mode=err, rule_scope="tensor")
    bad("--transport nccl_flat runs the plain mean", transport="nccl_flat", err_mode="none")
    bad("--transport nccl_flat", transport="nccl_flat", err_mode="minmax", attack_scope="model", rule_scope="tensor",
        mode="normal")
    bad("streams over the slab per tensor", mode="geometric_median", num_workers=20, worker_fail=2, transport="nvl")
    # the rule's own bounds apply unchanged
    bad("Bulyan's condition", mode="bulyan", num_workers=6, worker_fail=1)
    # accepted: the streaming sizes on the library path, the attack scope with any rule, and both together
    _cfg(mode="geometric_median", num_workers=20, worker_fail=2, transport="nccl").resolve(1)
    _cfg(mode="coordinate_median", rule_scope="tensor", attack_scope="model", err_mode="minmax", transport="nvl").resolve(1)
    _cfg(approach="detox", group_size=3, num_workers=15, worker_fail=3, attack_scope="model", err_mode="minmax",
         transport="nvl").resolve(1)


# ------------------------------------------------------------------------------------------------ library-op PS
def _slots(g, cfg, L, groups):
    S = torch.randn(cfg.num_workers, L.total, generator=g)
    S *= torch.rand(cfg.num_workers, 1, generator=g) * 4
    if groups is not None:                                   # replicas agree, then the first worker_fail workers lie
        for grp in groups.groups:
            for w in grp[1:]:
                S[w - 1] = S[grp[0] - 1]
    S[: cfg.worker_fail] = torch.randn(cfg.worker_fail, L.total, generator=g) * 5
    return S


def _model_oracle(cfg, S, L, groups, center=None):
    """The oracle's whole-model result, split per tensor, from the rows of the row source."""
    X = S.numpy()
    spans = _spans(L)
    plan = rule_plan(cfg)
    if cfg.approach == "detox":                              # row k: group k's per-tensor vote winners, concatenated
        W = np.zeros((plan.rows, L.total), dtype=np.float32)
        for o, n in spans:
            W[:, o:o + n] = X[oracle.detox_winner_slots(X[:, o:o + n], groups.groups), o:o + n]
        X = W
    if cfg.approach == "nnm":
        return oracle.model_scope(oracle.nnm, X, spans, plan.f, cfg.mode)
    if cfg.mode == "centered_clip":
        return oracle.model_scope(oracle.centered_clip, X, spans, oracle.model_rows(center, spans), cfg.clip_tau)
    return oracle.model_scope(_rule(cfg.mode, plan.rows, plan.f), X, spans)


def _torch_cases():
    cases = [("baseline", m, 7, 1, 1) for m in DISTANCE]
    cases += [("detox", m, 15, 3, 3) for m in ("multi_krum", "geometric_median", "centered_clip")]
    cases += [("detox", "bulyan", 16, 1, 2)]
    cases += [("nnm", m, 7, 1, 1) for m in oracle.NNM_MODES]
    return cases


@pytest.mark.parametrize("approach,mode,P,f,r", _torch_cases())
def test_torch_ps_equals_the_model_oracle_over_several_steps(approach, mode, P, f, r):
    """Every step's result against the oracle on the concatenated rows; centered clipping carries its centre across steps."""
    cfg = _cfg(approach=approach, mode=mode, num_workers=P, worker_fail=f, group_size=r).resolve(1)
    L = _layout()
    groups, code = build_codes(cfg)
    ps = TorchPS(cfg, L, CPU, L.new_arena(CPU), groups, code)
    g = torch.Generator().manual_seed(P * 10 + f)
    center = np.zeros(L.total, dtype=np.float32)
    for step in range(3):
        S = _slots(g, cfg, L, groups)
        out = ps.aggregate(S)
        want = _model_oracle(cfg, S, L, groups, center)
        tol = 1e-4 if mode == "geometric_median" else 1e-5
        for spec, got, w in zip(L.specs, out, want):
            assert np.allclose(got.numpy(), w, rtol=tol, atol=tol * np.abs(w).max()), (step, spec.name)
        if mode == "centered_clip":
            for spec, w in zip(L.specs, want):
                center[spec.offset: spec.offset + spec.numel] = w
            assert np.allclose(ps.cc_center.numpy(), center, rtol=1e-5, atol=1e-6)
            center = ps.cc_center.numpy().copy()


def test_torch_ps_model_scope_keeps_one_row_set_for_every_tensor():
    """Multi-Krum's result in each tensor is the mean of the same rows: those the whole-model distances select."""
    cfg = _cfg(num_workers=7, worker_fail=1).resolve(1)
    L = _layout()
    g = torch.Generator().manual_seed(5)
    S = torch.randn(7, L.total, generator=g)
    S[0, : L.specs[0].numel] += 50.0                         # far off in the first tensor only
    out = TorchPS(cfg, L, CPU, L.new_arena(CPU), None, None).aggregate(S)
    D = oracle.model_d2([oracle._raw_d2(S[:, s.offset: s.offset + s.numel].numpy()) for s in L.specs])
    rows = np.argsort(oracle._krum_scores_d2(D, 1), kind="stable")[:6].tolist()
    assert 0 not in rows
    for spec, got in zip(L.specs, out):
        assert torch.equal(got, S[rows, spec.offset: spec.offset + spec.numel].sum(0) / 6)


def test_minmax_model_gamma_equals_the_oracle():
    L = _layout()
    g = torch.Generator().manual_seed(6)
    S = torch.randn(7, L.total, generator=g) * torch.rand(7, 1, generator=g)
    Hs = [S[2:, s.offset: s.offset + s.numel].double() for s in L.specs]
    want = A.minmax_gamma_model([H.numpy() for H in Hs])
    assert minmax_gamma_model(Hs) == pytest.approx(want, rel=1e-12)
    assert want != pytest.approx(A.minmax_gamma(Hs[0].numpy()), rel=1e-3)      # not the first tensor's own gamma


def test_gloo_minmax_model_scope_rows_equal_the_oracle():
    cfg = _cfg(mode="multi_krum", err_mode="minmax", attack_scope="model", num_workers=7, worker_fail=2, max_steps=4)
    t = Trainer(cfg, rank=0, world=1, device=CPU, quiet=True)
    eng = t.engine
    step = next(s for s in range(1, 5) if any(eng.schedule.is_adversary(w, s) for w in range(1, 8)))
    g = torch.Generator().manual_seed(7)
    eng.slots.copy_(torch.randn(7, eng.layout.total, generator=g))
    before = eng.slots.numpy().copy()
    eng._ps_attack(step)
    liars = [w - 1 for w in range(1, 8) if eng.schedule.is_adversary(w, step)]
    want = A.ps_attack(before, liars, "minmax", _spans(eng.layout), scope="model")
    assert np.allclose(eng.slots.numpy(), want, rtol=1e-6, atol=1e-7)
    per_tensor = A.ps_attack(before, liars, "minmax", _spans(eng.layout))
    assert not np.allclose(want, per_tensor)
    for _ in range(3):
        m = t.train_step()
    assert np.isfinite(m["loss"])


# ------------------------------------------------------------------------------------------------ Gloo jobs
@pytest.mark.parametrize("mode,extra,port", [("multi_krum", [], 29781), ("centered_clip", ["--clip-tau", "0.1"], 29782)])
def test_multi_process_job_equals_the_single_process_job(tmp_path, mode, extra, port):
    """1 PS + 2 worker processes over Gloo against one process hosting everything, at model scope under min-max's model
    scope: the same parameters (and centre) at step 3."""
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""), OMP_NUM_THREADS="1")
    common = ["-m", "draco_b200.cli.distributed_nn", "--no-cuda", "--network", "LeNet", "--dataset", "MNIST", "--num-workers", "7",
              "--batch-size", "8", "--max-steps", "3", "--eval-freq", "3", "--synthetic-size", "128", "--log-interval", "1",
              "--compress-grad", "None", "--approach", "baseline", "--mode", mode, *extra, "--worker-fail", "1",
              "--err-mode", "minmax", "--rule-scope", "model", "--attack-scope", "model"]
    blobs = []
    for name, launch in (("multi", ["--launch", "3", "--master-port", str(port)]), ("single", [])):
        d = str(tmp_path / name) + "/"
        r = subprocess.run([sys.executable, *common, "--train-dir", d, *launch], capture_output=True, text=True, timeout=420,
                           env=env, cwd=ROOT)
        assert r.returncode == 0, (r.stdout[-2000:], r.stderr[-3000:])
        blobs.append(load_checkpoint(d + "model_step_3"))
    multi, single = blobs
    for k, v in single["state_dict"].items():
        assert torch.equal(multi["state_dict"][k], v), k
    for k, v in single["opt_state"].get("cc_center", {}).items():
        assert torch.equal(multi["opt_state"]["cc_center"][k], v), k


def test_checkpoint_resume_of_a_model_scope_centered_clip_job_is_bit_for_bit(tmp_path):
    d = str(tmp_path) + "/"
    kw = dict(mode="centered_clip", clip_tau=0.5, train_dir=d, max_steps=6, num_workers=5)
    t = Trainer(_cfg(eval_freq=3, **kw), rank=0, world=1, device=CPU, quiet=True)
    t.fit(6)
    final, center = t.engine.master_params().clone(), t.engine.ps.cc_center.clone()
    assert set(load_checkpoint(d + "model_step_3")["opt_state"]) == {"cc_center"}
    t2 = Trainer(_cfg(eval_freq=10 ** 6, checkpoint_step=3, **kw), rank=0, world=1, device=CPU, quiet=True)
    for _ in range(3):
        t2.train_step()
    assert torch.equal(t2.engine.master_params(), final) and torch.equal(t2.engine.ps.cc_center, center)
    # the scope is no state: a resume may change it
    t3 = Trainer(_cfg(eval_freq=10 ** 6, checkpoint_step=3, **dict(kw, rule_scope="tensor")), rank=0, world=1, device=CPU,
                 quiet=True)
    assert t3.step == 4 and torch.isfinite(t3.train_step()["loss"] * torch.ones(1)).all()


# ------------------------------------------------------------------------------------------------ fused PS launch sequence
RECORDED = ("vote", "aggregate_update", "krum_select", "bulyan_select", "geometric_median_weights", "nnm_mix", "nnm_fold",
            "centered_clip_dist", "centered_clip_weights", "centered_clip_update", "pair_dist", "pair_scope_fold",
            "nnm_mix_table", "centered_clip_model_weights", "ps_attack", "ps_attack_model")


def _buckets(T):
    return [(0, 3, [0, 1]), (3, 7, [2, 3, 4]), (7, 12, list(range(5, T)))]


def _record(cfg, monkeypatch, bucketed):
    """FusedPS.enqueue_step with the launchers replaced by recorders: (launcher, filled=) per call, the waits, the count."""
    L = _layout()
    calls = []

    def rec(name):
        def f(*args, **kw):
            calls.append((name, kw["filled"]) if "filled" in kw else (name,))
            return {"ps_attack": 3, "ps_attack_model": 4}.get(name)
        return f
    for name in RECORDED:
        monkeypatch.setattr(K, name, rec(name))
    groups, code = build_codes(cfg)
    ps = FusedPS(cfg, L, CPU, L.new_arena(CPU), torch.zeros(cfg.num_workers, L.total), groups, code,
                 adv_bitmap=torch.zeros(8, dtype=torch.int32), adv_len=8)
    kw = dict(buckets=_buckets(L.ntensors), wait_bucket=lambda b: calls.append(("wait", b)) or 1) if bucketed else {}
    n = ps.enqueue_step(torch.ones(1, dtype=torch.int64), mc_params=None, dst=[4096], flags=[16],
                        before_update=lambda: calls.append(("before_update",)) or 1, **kw)
    return ps, calls, n


PAIR = [("pair_dist",), ("pair_scope_fold",)]
LAUNCH_SEQUENCES = {
    ("baseline", "krum"): PAIR + [("krum_select", True)],
    ("baseline", "multi_krum"): PAIR + [("krum_select", True)],
    ("baseline", "geometric_median"): PAIR + [("geometric_median_weights", True)],
    ("baseline", "bulyan"): PAIR + [("bulyan_select", True)],
    ("baseline", "centered_clip"): [("centered_clip_dist",), ("centered_clip_model_weights",)],
    ("detox", "multi_krum"): [("vote",)] + PAIR + [("krum_select", True)],
    ("detox", "geometric_median"): [("vote",)] + PAIR + [("geometric_median_weights", True)],
    ("detox", "centered_clip"): [("vote",), ("centered_clip_dist",), ("centered_clip_model_weights",)],
    ("nnm", "coordinate_median"): PAIR + [("nnm_mix_table",)],
    ("nnm", "trimmed_mean"): PAIR + [("nnm_mix_table",)],
    ("nnm", "krum"): PAIR + [("nnm_mix_table",), ("krum_select", True), ("nnm_fold",)],
    ("nnm", "multi_krum"): PAIR + [("nnm_mix_table",), ("krum_select", True), ("nnm_fold",)],
    ("nnm", "geometric_median"): PAIR + [("nnm_mix_table",), ("geometric_median_weights", True), ("nnm_fold",)],
    ("nnm", "bulyan"): PAIR + [("nnm_mix_table",), ("bulyan_select", True)],
}


@pytest.mark.parametrize("approach,mode", sorted(LAUNCH_SEQUENCES))
@pytest.mark.parametrize("attack", ["tensor", "model"])
def test_fused_ps_model_scope_launch_sequence(monkeypatch, approach, mode, attack):
    """Whole-arena: (the attack), the row source, the pair pass and its scope fold (or CC's model weights), the selection on the
    filled table, the update -- even when the engine hands the PS its buckets."""
    cfg = _cfg(approach=approach, mode=mode, num_workers=15, worker_fail=3, group_size=3, transport="nvl", err_mode="minmax",
               attack_scope=attack).resolve(1)
    for bucketed in (False, True):
        ps, calls, n = _record(cfg, monkeypatch, bucketed)
        assert not ps.plan.pipelined
        attack_call = ("ps_attack_model",) if attack == "model" else ("ps_attack",)
        update = ("centered_clip_update",) if mode == "centered_clip" else ("aggregate_update",)
        assert calls == [attack_call] + LAUNCH_SEQUENCES[(approach, mode)] + [("before_update",), update]
        kernels = {"vote": 2, "pair_dist": 1, "pair_scope_fold": 1, "centered_clip_dist": 1, "centered_clip_model_weights": 2,
                   "nnm_mix_table": 1, "krum_select": 1, "bulyan_select": 1, "geometric_median_weights": 1, "nnm_fold": 1}
        want = (4 if attack == "model" else 3) + sum(kernels[c[0]] for c in LAUNCH_SEQUENCES[(approach, mode)]) + 1 + 1
        assert n == want
    if attack == "model":
        assert ps.attack_fold.shape == (ps.layout.ntensors, 2 * 15 + 1 + 15 * 14 // 2)
    if mode == "centered_clip":
        assert ps.cc_dist.shape == (ps.layout.ntensors, ps.plan.rows)


def test_attack_scope_model_takes_a_pipelined_rule_off_the_pipeline(monkeypatch):
    cfg = _cfg(mode="coordinate_median", rule_scope="tensor", num_workers=15, worker_fail=3, transport="nvl", err_mode="minmax",
               attack_scope="model").resolve(1)
    ps, calls, n = _record(cfg, monkeypatch, True)
    assert calls == [("ps_attack_model",), ("before_update",), ("aggregate_update",)] and n == 6


@pytest.mark.parametrize("rule_scope", ["tensor", "model"])
@pytest.mark.parametrize("attack_scope", ["tensor", "model"])
def test_engine_and_ps_agree_on_pipelining_for_every_scope(monkeypatch, rule_scope, attack_scope):
    """For every rule the scopes allow: the engine pipelines exactly when the PS does, and a pipelined PS waits for every bucket."""
    seen = 0
    for approach in ("baseline", "detox", "nnm", "maj_vote"):
        for mode in MODES:
            try:
                cfg = _cfg(approach=approach, mode=mode, num_workers=15, worker_fail=3, group_size=3, transport="nvl",
                           err_mode="minmax", rule_scope=rule_scope, attack_scope=attack_scope,
                           clip_tau=1.0 if mode == "centered_clip" else None).resolve(1)
            except ValueError:
                continue
            plan = rule_plan(cfg)
            assert pipelines_ps(cfg, True) == plan.pipelined == (
                plan.rule in PIPELINED_RULES and rule_scope == "tensor" and attack_scope == "tensor"), plan.rule
            assert not pipelines_ps(cfg, False)
            ps, calls, _ = _record(cfg, monkeypatch, True)
            waits = [c for c in calls if c[0] == "wait"]
            assert len(waits) == (3 if pipelines_ps(cfg, True) else 0), plan.rule
            seen += 1
    assert seen >= 8
