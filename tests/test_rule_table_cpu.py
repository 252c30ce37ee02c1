"""What ``JobConfig.resolve`` accepts, and the rule plan of every accepted job, pinned to a golden over a grid of jobs.

Every case of the grid goes through ``JobConfig(...).resolve(1)`` and ``rule_plan``.  An accepted case records every
``RulePlan`` field; a rejected one records only that it was rejected (the ``match=`` tests of the rule modules pin the
messages).  The cases are grouped by (approach, mode, transport), and the golden keeps per group the number of cases, the
number accepted and a digest of the outcomes in grid order, so a diff names exactly the groups that changed.

The rule dimensions (approach, mode, num_workers, worker_fail, group_size, bucketing, rule scope, transport) are crossed
fully, except that group_size takes two values outside maj_vote / detox and bucketing two values outside baseline; the attack,
compression and clipping-radius dimensions are crossed with the dimensions they interact with.

Regenerate the golden with ``python tests/test_rule_table_cpu.py --write`` only when what a job may be is meant to change."""
import hashlib
import json
import os
import sys

import pytest

from draco_b200 import JobConfig
from draco_b200.config import APPROACHES, MODES, TRANSPORTS
from draco_b200.rules import rule_plan

GOLDEN_FILE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "rule_table.json")

WORKERS = tuple(range(1, 21)) + (32, 33)
FAILS = tuple(range(6))
# --err-mode, with min-max at both attack scopes
ATTACKS = (("none", "tensor"), ("rev_grad", "tensor"), ("omniscient", "tensor"), ("alie", "tensor"), ("minmax", "tensor"),
           ("minmax", "model"), ("ipm", "tensor"), ("mimic", "tensor"))


def _cases():
    """(group key, case) in grid order; a case is the JobConfig keywords as a tuple of items."""
    for approach in APPROACHES:
        groups = (1, 2, 3, 4, 5) if approach in ("maj_vote", "detox") else (1, 3)
        buckets = (0, 1, 2, 3, 5) if approach == "baseline" else (0, 2)
        for mode in MODES:
            tau = 1.0 if mode == "centered_clip" else None
            for transport in TRANSPORTS:
                key = f"{approach}/{mode}/{transport}"
                base = dict(approach=approach, mode=mode, transport=transport)
                for P in WORKERS:
                    for f in FAILS:
                        # the rule dimensions
                        for r in groups:
                            for s in buckets:
                                for scope in ("tensor", "model"):
                                    yield key, dict(base, num_workers=P, worker_fail=f, group_size=r, bucketing=s,
                                                    rule_scope=scope, err_mode="none", compress_grad="None", clip_tau=tau)
                        # the attacks and the codec
                        for err, attack_scope in ATTACKS:
                            for compress in ("compress", "None"):
                                yield key, dict(base, num_workers=P, worker_fail=f, group_size=3, err_mode=err,
                                                attack_scope=attack_scope, compress_grad=compress, clip_tau=tau)
                        # the clipping radius, set and unset, with any rule
                        for clip in (None, 0.5):
                            yield key, dict(base, num_workers=P, worker_fail=f, group_size=3, err_mode="none",
                                            compress_grad="None", clip_tau=clip)


def _outcomes():
    """{group: {"cases": n, "accepted": k, "digest": sha256 of the outcomes}}."""
    hashes, out = {}, {}
    for key, kw in _cases():
        try:
            cfg = JobConfig(**kw).resolve(1)
        except ValueError:
            outcome = None
        else:
            outcome = tuple(vars(rule_plan(cfg)).values())
        h = hashes.get(key)
        if h is None:
            h = hashes[key] = hashlib.sha256()
            out[key] = {"cases": 0, "accepted": 0}
        h.update(repr((tuple(sorted(kw.items())), outcome)).encode())
        out[key]["cases"] += 1
        out[key]["accepted"] += outcome is not None
    for key, h in hashes.items():
        out[key]["digest"] = h.hexdigest()[:32]
    return out


def test_accepted_jobs_and_their_plans_match_golden():
    with open(GOLDEN_FILE) as fh:
        golden = json.load(fh)
    got = _outcomes()
    assert sorted(got) == sorted(golden)
    assert {key: (golden[key], got[key]) for key in golden if got[key] != golden[key]} == {}


def test_krum_over_more_than_16_worker_slots_is_rejected_on_nvl():
    """Krum's pair table holds 16 rows (KRUM_MAXP): the job fails when it is configured, not at its first step."""
    for scope in ("tensor", "model"):
        with pytest.raises(ValueError, match="at most 16 workers .*use --transport nccl"):
            JobConfig(approach="baseline", mode="krum", num_workers=17, worker_fail=1, rule_scope=scope, transport="nvl").resolve(1)
        JobConfig(approach="baseline", mode="krum", num_workers=16, worker_fail=1, rule_scope=scope, transport="nvl").resolve(1)
        JobConfig(approach="baseline", mode="krum", num_workers=17, worker_fail=1, rule_scope=scope, transport="nccl").resolve(1)


if __name__ == "__main__" and "--write" in sys.argv:
    with open(GOLDEN_FILE, "w") as fh:
        json.dump(_outcomes(), fh, sort_keys=True, indent=1)
        fh.write("\n")
