"""Every PS aggregation rule pinned to goldens, on the CPU.

* ``FusedPS.enqueue_step``: the launchers of ``draco_b200.ops.kernels`` are replaced by recorders, so the test sees the launch
  plan of a step -- every call in order, its bound arguments (numbers exactly; tensors as (ordinal of first appearance, shape,
  dtype), which captures the data flow from one call to the next) and the launch count the step returns.  The golden keeps
  the rule, the launch count and a digest of the calls.
* ``TorchPS``: the sha256 of every tensor ``aggregate`` returns on seeded slots, and the mode string ``apply`` passes to the
  optimizer.  The golden keeps the rule, the mode and a digest of the hashes.

Regenerate the goldens with ``python tests/test_ps_plan_cpu.py --write`` only when a rule is meant to change."""
import functools
import hashlib
import inspect
import json
import os
import sys

import pytest
import torch

from draco_b200 import JobConfig
from draco_b200.config import APPROACHES, MODES
from draco_b200.models import build_model
from draco_b200.ops import kernels as K
from draco_b200.parallel.arena import ArenaLayout
from draco_b200.parallel.ps import FusedPS, TorchPS, build_codes

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
GOLDEN_FILE = os.path.join(GOLDEN, "ps_rules.json")

LAUNCHERS = ("vote", "aggregate_update", "krum_select", "bulyan_select", "geometric_median_weights", "geometric_median",
             "nnm_mix", "nnm_fold", "cyclic_project", "cyclic_locate", "ps_attack")
SIGNATURES = {name: inspect.signature(getattr(K, name)) for name in LAUNCHERS}
# (num_workers, worker_fail, group_size): P = 20 takes the streaming geometric median, (16, 1, 2) DETOX's Bulyan (8 groups, b_G = 1)
SHAPES = ((15, 3, 3), (7, 1, 3), (9, 2, 2), (16, 1, 2), (20, 2, 4))
CPU = torch.device("cpu")


def _digest(obj) -> str:
    return hashlib.sha256(json.dumps(obj, sort_keys=True, separators=(",", ":")).encode()).hexdigest()[:32]


def _golden(kind):
    with open(GOLDEN_FILE) as fh:
        return json.load(fh)[kind]


@functools.lru_cache(maxsize=None)
def _layout():
    return ArenaLayout.from_model(build_model("LeNet"), bf16=False, channels_last=True)


def _modes(approach):
    """--mode values that select a distinct rule: cyclic ignores it, maj_vote reads only maj_vote (vote) against the rest (mean)."""
    return {"cyclic": ("normal",), "maj_vote": ("normal", "maj_vote")}.get(approach, [m for m in MODES if m != "maj_vote"])


def _configs(transport, **kw):
    """Every (approach, mode) that resolves at every shape, keyed by a readable name."""
    out = {}
    for P, f, r in SHAPES:
        for approach in APPROACHES:
            for mode in _modes(approach):
                cfg = JobConfig(approach=approach, mode=mode, num_workers=P, worker_fail=f, group_size=r, transport=transport, **kw)
                try:
                    cfg.resolve(1)
                except ValueError:
                    continue
                out[f"{approach}/{mode}/P{P}f{f}r{r}"] = cfg
    return out


# ------------------------------------------------------------------------------------------------ FusedPS launch plan
class _Trace:
    def __init__(self):
        self.calls, self.ids = [], {}

    def value(self, v):
        if isinstance(v, torch.Tensor):
            key = (v.data_ptr(), tuple(v.shape), tuple(v.stride()), v.dtype)
            return ["tensor", self.ids.setdefault(key, len(self.ids)), list(v.shape), str(v.dtype)]
        if isinstance(v, ArenaLayout):
            return "layout"
        if isinstance(v, (list, tuple)):
            return [self.value(x) for x in v]
        if isinstance(v, (K.AttackWorkspace, K.GeoMedianWorkspace)):
            return {type(v).__name__: {k: self.value(x) for k, x in sorted(vars(v).items())}}
        if v is None or isinstance(v, (bool, int, float, str)):
            return v
        raise TypeError(f"unrecorded argument type {type(v)}")

    def recorder(self, name):
        sig = SIGNATURES[name]

        def record(*args, **kwargs):
            bound = sig.bind(*args, **kwargs)
            bound.apply_defaults()
            self.calls.append([name, {k: self.value(v) for k, v in bound.arguments.items()}])
            if name == "ps_attack":                     # what the real launcher returns: its launch count
                return 1 if bound.arguments["mode"] == 5 else 3
            return None
        return record


def _buckets(T):
    """Three push buckets: (first tile, end tile, tensor indices)."""
    return [(0, 3, [0, 1]), (3, 7, [2, 3, 4]), (7, 12, list(range(5, T)))]


def _launch_cases():
    cases = {}
    for name, cfg in _configs("nvl").items():
        for bucketed in (False, True):
            cases[f"{name}/{'buckets' if bucketed else 'whole'}"] = (cfg, bucketed)
    for err in ("alie", "minmax"):
        for name, cfg in _configs("nvl", err_mode=err).items():
            if name.endswith("P15f3r3"):
                cases[f"{name}/{err}/buckets"] = (cfg, True)
                cases[f"{name}/{err}/whole"] = (cfg, False)
    for opt, ams in (("adam", False), ("adam", True)):
        for name, cfg in _configs("nvl", optimizer=opt, amsgrad=ams).items():
            if name.endswith("P15f3r3") and name.split("/")[0] in ("baseline", "maj_vote"):
                cases[f"{name}/{'amsgrad' if ams else opt}/buckets"] = (cfg, True)
    return cases


def _launch_plan(cfg, bucketed, monkeypatch):
    L = _layout()
    trace = _Trace()
    for name in LAUNCHERS:
        monkeypatch.setattr(K, name, trace.recorder(name))
    groups, code = build_codes(cfg)
    P = cfg.num_workers
    params = L.new_arena(CPU)
    grad_in = torch.zeros(P, L.total, dtype=torch.float32)
    adv = torch.zeros(8, dtype=torch.int32)
    ps = FusedPS(cfg, L, CPU, params, grad_in, groups, code, adv_bitmap=adv, adv_len=8)
    step = torch.ones(1, dtype=torch.int64)

    def wait_bucket(b):
        trace.calls.append(["wait_bucket", b])
        return 1

    def before_update():
        trace.calls.append(["before_update"])
        return 1
    kw = dict(buckets=_buckets(L.ntensors), wait_bucket=wait_bucket) if bucketed else {}
    n = ps.enqueue_step(step, mc_params=None, dst=[4096, 8192], flags=[16, 32, 48], before_update=before_update, **kw)
    return f"{ps.rule} n={n} {_digest(trace.calls)}"


def _all_launch_plans(monkeypatch):
    return {name: _launch_plan(cfg, bucketed, monkeypatch) for name, (cfg, bucketed) in _launch_cases().items()}


def test_fused_ps_launch_plan_matches_golden(monkeypatch):
    golden = _golden("launch")
    got = _all_launch_plans(monkeypatch)
    assert sorted(got) == sorted(golden)
    assert {name: got[name] for name in golden if got[name] != golden[name]} == {}


def test_launch_cases_cover_every_rule_and_the_streaming_geometric_median():
    cfgs = [c for c, _ in _launch_cases().values()]
    assert len({(c.approach, c.mode) for c in cfgs if c.approach in ("baseline", "detox", "nnm")}) == 7 + 5 + 6
    assert any(c.num_workers > K.GEOMED_FAST_MAXP and c.approach == "baseline" and c.mode == "geometric_median" for c in cfgs)


# ------------------------------------------------------------------------------------------------ TorchPS outputs
def _slots(cfg, L, groups):
    g = torch.Generator().manual_seed(1000 * cfg.num_workers + 10 * cfg.worker_fail + cfg.group_size)
    P = cfg.num_workers
    if cfg.approach == "cyclic":
        return torch.complex(torch.randn(P, L.total, generator=g), torch.randn(P, L.total, generator=g))
    S = torch.randn(P, L.total, generator=g)
    if groups is not None:                                 # replicas agree, then the first worker_fail workers lie
        for grp in groups.groups:
            for w in grp[1:]:
                S[w - 1] = S[grp[0] - 1]
        S[: cfg.worker_fail] = torch.randn(cfg.worker_fail, L.total, generator=g) * 10
    return S


def _torch_result(cfg):
    L = _layout()
    groups, code = build_codes(cfg)
    ps = TorchPS(cfg, L, CPU, L.new_arena(CPU), groups, code)
    out = ps.aggregate(_slots(cfg, L, groups))
    seen = {}

    class _Opt:
        def step(self, grads, mode):
            seen["mode"] = mode
    ps.optimizer = _Opt()
    ps.apply(out)
    return f"{ps.rule} mode={seen['mode']} {_digest([hashlib.sha256(t.contiguous().numpy().tobytes()).hexdigest() for t in out])}"


def _all_torch_results():
    return {name: _torch_result(cfg) for name, cfg in _configs("gloo").items()}


def test_torch_ps_outputs_match_golden():
    golden = _golden("torch")
    got = _all_torch_results()
    assert sorted(got) == sorted(golden)
    assert {name: got[name] for name in golden if got[name] != golden[name]} == {}


if __name__ == "__main__" and "--write" in sys.argv:
    mp = pytest.MonkeyPatch()
    try:
        plans = _all_launch_plans(mp)
    finally:
        mp.undo()
    os.makedirs(GOLDEN, exist_ok=True)
    with open(GOLDEN_FILE, "w") as fh:
        json.dump({"launch": plans, "torch": _all_torch_results()}, fh, sort_keys=True, indent=1)
        fh.write("\n")
