"""The PS aggregation rules as one table: a row source, which gives the rows and how many of them may be bad, and a base rule
that runs on those rows.

For every row source the table states its rows and f, the base rules it takes and its limit on the nvl transport; for every
base rule its ``--mode`` string, its condition on the rows and f and the rows its fused kernels take.  ``PIPELINED_RULES``
names the rules the fused PS may apply bucket by bucket.  ``check`` rejects the jobs the table rules out and ``rule_plan``
works out the plan both parameter servers build from.  Torch-free: ``config.py`` checks every job with it."""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional, Tuple

ROBUST_MAXP = 16        # rows of the fused sort, pair-table and register kernels (TRIM_MAXP, KRUM_MAXP, the row table)
SIGN_VOTE_MAXP = 32     # rows of the fused sign vote: the adversary bitmaps are 32-bit (DRC_MAX_WORKERS)

# row conditions on n rows of which f may be bad: (holds, the condition, words between the label and "needs", the reason).
# Their messages read "<label><lead> needs <condition> (<reason>; got ...)" with the source's names of n and f
CONDITIONS = {
    "trim": (lambda n, f: 2 * f < n, "{n} > 2*{f}", " trims {f} values at each end of every coordinate, so it",
             "the honest values must be a strict majority of every coordinate"),
    "majority": (lambda n, f: 2 * f < n, "{n} > 2*{f}", "", "the honest rows must be a strict majority"),
    "krum": (lambda n, f: n > 2 * f + 2, "{n} > 2*{f} + 2", "", "Krum's condition"),
    "bulyan": (lambda n, f: n >= 4 * f + 3, "{n} >= 4*{f} + 3", "", "Bulyan's condition"),
}


@dataclass(frozen=True)
class Base:
    mode: str                   # its --mode string, which is also the optimizer's mode string
    condition: Optional[str]    # its row condition: a key of CONDITIONS, or None
    nvl_max: Optional[int]      # rows its fused kernels take (None: any) ...
    nvl_why: str                # ... and why
    nccl_flat: bool             # resolve() passes it on --transport nccl_flat


# nccl_flat runs the mean and the vote.  The robust rules older than centered clipping pass resolve() there as well, and
# FlatNcclEngine rejects them when it is built
BASES = {
    "mean": Base("normal", None, None, "", True),
    "vote": Base("maj_vote", None, None, "", True),
    "cyclic": Base("cyclic", None, None, "", True),
    "median": Base("coordinate_median", "trim", ROBUST_MAXP, "a sorting network", True),
    "trimmed_mean": Base("trimmed_mean", "trim", ROBUST_MAXP, "a sorting network", True),
    "krum": Base("krum", "krum", ROBUST_MAXP, "the pair table", True),
    "multi_krum": Base("multi_krum", "krum", ROBUST_MAXP, "the pair table", True),
    # over the worker slots at --rule-scope tensor, more rows take the streaming geometric median (check)
    "geomedian": Base("geometric_median", "majority", ROBUST_MAXP,
                      "the pair table; beyond it the median streams over the slab per tensor, at --rule-scope tensor", True),
    "bulyan": Base("bulyan", "bulyan", ROBUST_MAXP, "the pair table", True),
    "centered_clip": Base("centered_clip", "majority", ROBUST_MAXP, "the rows live in registers", False),
    "sign_vote": Base("sign_vote", "majority", SIGN_VOTE_MAXP, "the adversary bitmaps are 32-bit", False),
}
BASE_OF_MODE = {b.mode: name for name, b in BASES.items()}


@dataclass(frozen=True)
class Source:
    label: str                  # the flag that selects it, in messages
    what: str                   # what its base rule is applied to, in messages
    rows: str                   # the names of its rows and of f, in messages
    f: str
    bases: Tuple[str, ...]      # the base rules --mode may choose on it
    unbounded: Tuple[str, ...]  # those of them that carry no row condition here
    nvl_max: Optional[int]      # its own limit on the nvl transport, on its groups or on the workers (None: none)
    nvl_unit: str               # "groups" | "workers"
    nccl_flat: bool             # resolve() passes it on --transport nccl_flat


SOURCES = {
    "raw": Source(label="", what="the worker slots", rows="num_workers", f="worker_fail",
                  bases=("mean", "median", "trimmed_mean", "krum", "multi_krum", "geomedian", "bulyan", "centered_clip",
                         "sign_vote"),
                  unbounded=("krum", "geomedian"), nvl_max=None, nvl_unit="workers", nccl_flat=True),
    "detox": Source(label="--approach detox", what="the rule applied across the group winners", rows="groups", f="b_G",
                    bases=("median", "trimmed_mean", "multi_krum", "geomedian", "bulyan", "centered_clip"),
                    unbounded=(), nvl_max=ROBUST_MAXP, nvl_unit="groups", nccl_flat=True),
    "nnm": Source(label="--approach nnm", what="the rule applied to the mixed rows", rows="num_workers", f="worker_fail",
                  bases=("median", "trimmed_mean", "krum", "multi_krum", "geomedian", "bulyan"),
                  unbounded=("krum", "geomedian"), nvl_max=ROBUST_MAXP, nvl_unit="workers", nccl_flat=False),
    "wbucket": Source(label="--bucketing", what="the rule applied to the bucket means", rows="nb", f="worker_fail",
                      bases=("median", "trimmed_mean", "krum", "multi_krum", "geomedian", "centered_clip"),
                      unbounded=(), nvl_max=ROBUST_MAXP, nvl_unit="workers", nccl_flat=False),
}


def route(cfg) -> Tuple[str, str]:
    """(row source, base rule) of a job.  Mirrors the reference's dispatch: cyclic approach -> Fourier decode
    (cyclic_master.py:24); maj_vote approach -> vote only when ``--mode maj_vote``, plain mean otherwise
    (rep_master.py:118-129); baseline approach -> ``--mode`` on the worker slots, the mean for a --mode they do not take
    (baseline_master.py:118-129).  Beyond the reference: ``--bucketing`` runs the baseline's rule on the worker-bucket means,
    and the detox and nnm approaches run ``--mode`` across the group winners of the vote / on the mixed rows."""
    if cfg.approach == "cyclic":
        return "raw", "cyclic"
    if cfg.approach == "maj_vote":
        return ("detox", "vote") if cfg.mode == "maj_vote" else ("raw", "mean")
    base = BASE_OF_MODE.get(cfg.mode)
    if cfg.approach == "baseline":
        return "wbucket" if cfg.bucketing else "raw", base if base in SOURCES["raw"].bases else "mean"
    return cfg.approach, base


# rules the fused PS applies bucket by bucket while the workers still push (buckets hold whole tensors, and centered clipping's
# centre is known before the step starts); with the worker buckets too.  Not NNM, whose neighbourhoods need whole-tensor
# distances, and only at the default scopes and without the mimic attack or a clipping --arc model, which need whole-model sums
# (RulePlan.pipelined)
PIPELINED_RULES = ("mean", "vote", "median", "trimmed_mean", "detox_median", "detox_trimmed_mean", "centered_clip",
                   "detox_centered_clip", "sign_vote")


def arc_k(P: int, f: int) -> int:
    """Rows adaptive robust clipping (--arc) clips among the P worker slots: k = floor(2 f (P - f) / P) in integer arithmetic
    (k >= f when f <= P / 2; k = 0 when f = 0, and --arc is then a no-op)."""
    return (2 * f * (P - f)) // P


def select_rule(cfg) -> str:
    """A job's rule name: its base rule, prefixed with its row source (detox_ | nnm_ | wbucket_) off the slots and the vote."""
    source, base = route(cfg)
    return base if source == "raw" or base == "vote" else f"{source}_{base}"


def _rows(source: str, cfg) -> Tuple[int, int, str]:
    """(rows, f, both in words) of a row source: P and worker_fail, G and b_G, or nb = ceil(P / s) and worker_fail."""
    P, f = cfg.num_workers, cfg.worker_fail
    if source == "detox":
        G, b = cfg.num_groups, cfg.captured_group_bound
        return G, b, f"{G} groups, b_G = worker_fail // ceil(group_size / 2) = {b}"
    if source == "wbucket":
        nb = -(-P // cfg.bucketing)
        return nb, f, f"{P} workers in buckets of {cfg.bucketing} give nb = {nb} bucket rows, worker_fail {f}"
    return P, f, f"{P} workers, worker_fail {f}"


def _check_source(source: str, cfg) -> None:
    """The parameter a row source forms its rows with."""
    P, f, r, s = cfg.num_workers, cfg.worker_fail, cfg.group_size, cfg.bucketing
    if source == "detox" and not 1 <= r <= P:
        raise ValueError(f"--approach detox needs 1 <= group_size <= num_workers (got group_size {r}, {P} workers)")
    if source == "nnm" and not 0 <= f < P:
        raise ValueError(f"--approach nnm mixes num_workers - worker_fail rows: it needs 0 <= worker_fail < num_workers "
                         f"(got worker_fail {f}, {P} workers)")
    if source == "wbucket" and not 1 <= s <= P:
        raise ValueError(f"--bucketing s needs 1 <= s <= num_workers (got {s} with {P} workers; 0 turns it off)")


def check(cfg) -> None:
    """Raise ValueError when the table rules the job's aggregation out: a base rule its row source does not take, a source
    parameter out of range, a row condition that fails, more rows than the nvl transport's kernels take, or a rule that
    --transport nccl_flat does not run."""
    source, base = route(cfg)
    src, rule = SOURCES[source], BASES.get(base)
    label = f"{src.label} --mode {cfg.mode}".lstrip()
    if cfg.approach in ("maj_vote", "cyclic"):            # the approach fixes the rule: the mean, the vote over any number
        label = f"--approach {cfg.approach}"              # of groups, or the cyclic decode
    else:
        if base not in src.bases:
            raise ValueError(f"{src.label} takes --mode {' | '.join(BASES[b].mode for b in src.bases)} ({src.what}), got "
                             f"--mode {cfg.mode}")
        _check_source(source, cfg)
        n, f, got = _rows(source, cfg)
        if rule.condition and base not in src.unbounded:
            holds, cond, lead, reason = CONDITIONS[rule.condition]
            if not holds(n, f):
                raise ValueError(f"{label}{lead.format(f=src.f)} needs {cond.format(n=src.rows, f=src.f)} ({reason}; got {got})")
        held = n if src.nvl_unit == "groups" else cfg.num_workers
        if cfg.transport == "nvl" and src.nvl_max is not None and held > src.nvl_max:
            raise ValueError(f"{src.label} on the nvl transport handles at most {src.nvl_max} {src.nvl_unit} (got {held}); use "
                             f"--transport nccl for more")
        streams = base == "geomedian" and source == "raw" and cfg.rule_scope == "tensor"
        if cfg.transport == "nvl" and rule.nvl_max is not None and not streams and n > rule.nvl_max:
            raise ValueError(f"{label} on the nvl transport handles at most {rule.nvl_max} rows ({rule.nvl_why}), that is at "
                             f"most {rule.nvl_max} {src.nvl_unit} (got {n}); use --transport nccl for more")
    model = [f"{flag} model" for flag, v in (("--rule-scope", cfg.rule_scope), ("--attack-scope", cfg.attack_scope))
             if v == "model"]
    if cfg.transport == "nccl_flat" and (model or not (src.nccl_flat and rule.nccl_flat)):
        raise ValueError(f"--transport nccl_flat runs the plain mean and the vote only; use --transport nccl for "
                         f"{' '.join([label] + model)}")


@dataclass(frozen=True)
class RulePlan:
    """A job's aggregation rule as a row source and a base rule, with every parameter worked out once."""
    rule: str           # select_rule's name
    source: str         # raw: the P worker slots | detox: the G group winners of the vote | nnm: the P mixed rows |
                        # wbucket: the nb = ceil(P / s) worker-bucket means of --bucketing s
    base: str           # mean | vote | cyclic | median | trimmed_mean | krum | multi_krum | geomedian | bulyan | centered_clip |
                        # sign_vote
    rows: int           # rows the base rule runs on: P, G over the group winners, or nb over the worker buckets
    f: int              # rows it tolerates: worker_fail, or b_G over the group winners
    trim: int           # median / trimmed mean: values dropped at each end of a coordinate
    m: int              # Krum / multi-Krum: rows averaged
    theta: int          # Bulyan: rows selected
    opt_mode: str       # the optimizer's mode string
    pipelined: bool     # the fused PS may apply it bucket by bucket: PIPELINED_RULES, both scopes "tensor", no mimic, no
                        # --arc model that clips (k > 0)
    scope: str          # --rule-scope: tensor | model (one choice over the whole model for every tensor)
    attack_scope: str   # --attack-scope: tensor | model (min-max: one gamma over the whole model)


def rule_plan(cfg) -> RulePlan:
    """The plan of a job that passed ``check``: the vote is the mean of the group winners, ``detox_*`` runs the rule across
    them (f = b_G), ``nnm_*`` on the mixed rows and ``wbucket_*`` on the worker-bucket means."""
    source, base = route(cfg)
    rule = select_rule(cfg)
    rows, f, _ = _rows(source, cfg)
    trim = {"median": (rows - 1) // 2, "trimmed_mean": f}.get(base, 0)
    m = {"krum": 1, "multi_krum": rows - f}.get(base, 0)
    scope, attack_scope = cfg.rule_scope, cfg.attack_scope
    pipelined = (rule.removeprefix("wbucket_") in PIPELINED_RULES and scope == "tensor" and attack_scope == "tensor"
                 and cfg.err_mode != "mimic" and not (cfg.arc == "model" and arc_k(cfg.num_workers, cfg.worker_fail) > 0))
    return RulePlan(rule, source, base, rows, f, trim, m, rows - 2 * f if base == "bulyan" else 0, BASES[base].mode, pipelined,
                    scope, attack_scope)
