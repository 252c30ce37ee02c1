"""Parameter-server side: aggregation rules + optimizer.

Two implementations of the same semantics (reference: ``SyncReplicasMaster_NN`` / ``CodedMaster`` / ``CyclicMaster`` in
src/master/*.py):

* ``FusedPS``  -- the product path.  Decode + SGD + parameter broadcast are sm_90a kernels working on the flat
  ``grad_in`` slab that workers filled through peer stores (ops/kernels.py); nothing returns to the host.
* ``TorchPS``  -- reference-faithful structure: per-tensor decode with library ops, a separate optimizer step, used by
  the NCCL baseline transport and the CPU/Gloo transport (where the small dense solves go through the C++ host
  library instead of Eigen/scipy).
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Sequence

import numpy as np
import torch

from .. import _native as N
from ..codes.adversary import ATTACK_ALIE, ATTACK_IPM, ATTACK_MIMIC, ATTACK_MINMAX, PS_ATTACKS, attack_code, mimic_z0
from ..codes.bucketing import bucket_schedule, wbuckets
from ..codes.cyclic import CyclicCode, search_w
from ..codes.oracle import (_bulyan_rounds, _krum_scores_d2, _weiszfeld_weights, arc_factors, arc_k, centered_clip_weight,
                            model_d2, nnm_neighbours_d2, nnm_pair_d2, wbucket_pair_d2)
from ..codes.repetition import GroupPlan
from ..config import JobConfig
from ..rules import PIPELINED_RULES, rule_plan, select_rule  # noqa: F401  (the rule names, importable here as before)
from .arena import ArenaLayout


def hyperparams_tensor(cfg: JobConfig, device) -> torch.Tensor:
    opt = {"sgd": 0, "adam": 2 if getattr(cfg, "amsgrad", False) else 1}[cfg.optimizer]
    # fp32(1 - dampening) with 1 - dampening formed in fp64; the kernel forms fp32(1 - beta) the same way from the fp64 betas
    # (DESIGN.md section 7)
    hp = N.HyperParams(lr=cfg.lr, momentum=cfg.momentum, weight_decay=cfg.weight_decay,
                       one_minus_dampening=1.0 - float(cfg.dampening), nesterov=int(cfg.nesterov), optimizer=opt,
                       beta1=float(cfg.adam_beta1), eps=float(cfg.adam_eps), beta2=float(cfg.adam_beta2))
    raw = np.frombuffer(bytes(hp), dtype=np.uint8).copy()
    return torch.from_numpy(raw).to(device)


class FusedPS:
    """Kernel-driven PS state for one job (lives on the PS GPU)."""

    def __init__(self, cfg: JobConfig, layout: ArenaLayout, device: torch.device, params: torch.Tensor,
                 grad_in: torch.Tensor, groups: Optional[GroupPlan], code: Optional[CyclicCode],
                 adv_bitmap: Optional[torch.Tensor] = None, adv_len: int = 0):
        from ..ops import kernels as K
        self.K = K
        self.cfg, self.layout, self.device = cfg, layout, device
        self.P = cfg.num_workers
        self.params = params                       # fp32 [D] master copy (inside the exported region)
        self.grad_in = grad_in                     # fp32 [P, D], complex64-as-fp32 [P, 2D], or sign words [P, D / 32]
        self.momentum = layout.new_arena(device)             # SGD momentum buffer / Adam first moment
        # Adam / AMSGrad state lives in arenas too (checkpointed with the momentum: utils/checkpoint.py)
        self.exp_avg_sq = layout.new_arena(device) if cfg.optimizer == "adam" else None
        self.max_exp_avg_sq = layout.new_arena(device) if (cfg.optimizer == "adam" and getattr(cfg, "amsgrad", False)) else None
        self.hp = hyperparams_tensor(cfg, device)
        self.counters = torch.zeros(16, dtype=torch.int32, device=device)
        T = layout.ntensors
        self.cyclic = cfg.approach == "cyclic"
        self.plan = plan = rule_plan(cfg)
        # the sign wire packs 32 coordinates into one uint32 word (push_encode(sign=True)); the stride is then in words
        self.slot_stride = layout.total // 32 if plan.base == "sign_vote" else layout.total
        self.rule = plan.rule
        # --err-mode alie | minmax | ipm: the liar slots of each bucket are overwritten after its flags and before its decode;
        # mimic: once, after the last bucket
        self.attack = attack_code(cfg.err_mode) if cfg.err_mode in PS_ATTACKS and adv_bitmap is not None else 0
        self.adv_bitmap, self.adv_len = adv_bitmap, adv_len
        # ALIE's z (z_max is only defined, and only read, under alie) or IPM's eps
        self.attack_z = cfg.alie_z if self.attack == ATTACK_ALIE else cfg.ipm_eps if self.attack == ATTACK_IPM else 0.0
        # mimic's state (checkpointed as opt_state["mimic_m"] / ["mimic_z"]) exists in every --err-mode mimic job
        self.mimic = None
        if cfg.err_mode == "mimic":
            z0 = mimic_z0([(sp.offset, sp.numel) for sp in layout.specs], layout.total)
            self.mimic = K.MimicState(layout, self.P, device, torch.from_numpy(z0))
        self.attack_ws = K.AttackWorkspace(layout, self.P, device) if self.attack == ATTACK_MINMAX else None
        # --arc: the worker slots clipped in place after the attack, per bucket (tensor) or after the last one (model); k = 0
        # (worker_fail 0) clips nothing, so nothing is allocated or launched
        self.arc_k = arc_k(self.P, cfg.worker_fail) if cfg.arc else 0
        self.arc_ws = K.ArcWorkspace(layout, self.P, device, model=cfg.arc == "model") if self.arc_k > 0 else None
        # --attack-scope model: min-max's per-tensor sums, folded, then one solve over the whole arena
        self.attack_fold = (K.attack_fold_buffer(layout, self.P, device)
                            if self.attack == ATTACK_MINMAX and plan.attack_scope == "model" else None)
        # row source.  DETOX: the rule runs on the G rows the vote's winner_slot table names, inside the kernels that read the
        # slab anyway.  NNM: the mixing masks; the rule then runs on the mixed rows.
        if plan.source == "detox":
            self.group_table = torch.from_numpy(groups.as_table()).to(device)
            G = self.group_table.shape[0]
            self.neq_mask = torch.zeros(G, T, dtype=torch.int32, device=device)
            self.winner_slot = torch.zeros(G, T, dtype=torch.int32, device=device)
            self.winner_member = torch.zeros(G, T, dtype=torch.int32, device=device)
        elif plan.source == "nnm":
            self.mix = torch.zeros(self.P, T, dtype=torch.int32, device=device)
        elif plan.source == "wbucket":                    # the permutation table, and the step's bucket rows (wbucket_plan)
            self.wb_schedule = torch.from_numpy(bucket_schedule(self.P, cfg.max_steps, cfg.seed)).to(device)
            self.wb_mask = torch.zeros(plan.rows, dtype=torch.int32, device=device)
            self.wb_scale = torch.zeros(plan.rows, dtype=torch.float32, device=device)
        # base rule.  The geometric median of more than GEOMED_FAST_MAXP rows streams over the slab once per Weiszfeld iteration;
        # every other choice starts from the table of pairwise distances between the rows
        rows = plan.rows
        self.gm = K.GeoMedianWorkspace(layout, rows, device) if plan.base == "geomedian" and rows > K.GEOMED_FAST_MAXP else None
        if self.gm is None and (plan.base in ("krum", "multi_krum", "geomedian", "bulyan") or plan.source == "nnm"):
            self.pair_d2 = torch.zeros(T, rows * (rows - 1) // 2, dtype=torch.float64, device=device)
        if plan.base in ("krum", "multi_krum", "bulyan"):    # the rows each tensor keeps (worker slots, or mixed rows under NNM)
            kept = plan.theta if plan.base == "bulyan" else plan.m
            self.select = torch.zeros((T,) if plan.source == "raw" and plan.base == "krum" else (kept, T), dtype=torch.int32,
                                      device=device)
        if self.gm is None and plan.base == "geomedian":
            self.gm_weights = torch.zeros(T, rows, dtype=torch.float32, device=device)
        if plan.base == "centered_clip":                  # the centre v (last step's aggregate, +0 at the start) is PS state
            self.cc_center = layout.new_arena(device)
            self.cc_partials = torch.zeros(layout.ntiles, rows, dtype=torch.float64, device=device)
            self.cc_weights = torch.zeros(T, rows, dtype=torch.float32, device=device)
            if plan.scope == "model":                     # the per-tensor d_i the whole-model norm is summed from
                self.cc_dist = torch.zeros(T, rows, dtype=torch.float64, device=device)
        if plan.source in ("nnm", "wbucket") and plan.base in ("krum", "multi_krum", "geomedian"):
            self.w_raw = torch.zeros(T, self.P, dtype=torch.float32, device=device)   # the choice, folded into raw-slot weights
        if plan.source == "wbucket" and plan.base in ("krum", "multi_krum", "geomedian"):
            # the raw slots' pair table, turned into the bucket rows' table (pair_d2) by wbucket_table
            self.wb_raw_d2 = torch.zeros(T, self.P * (self.P - 1) // 2, dtype=torch.float64, device=device)
            if plan.base == "geomedian" and rows == 1:    # one bucket holds every slot: its Weiszfeld weight is 1
                self.gm_weights.fill_(1.0)
            if plan.base != "geomedian":                  # Krum / multi-Krum: the compact table of the chosen buckets' slots
                kc = min(plan.m * cfg.bucketing, self.P)
                self.wb_wsel = torch.zeros(kc, T, dtype=torch.int32, device=device)
                self.w_raw = torch.zeros(T, kc, dtype=torch.float32, device=device)
        if plan.base == "cyclic":
            self.code = code
            self.E = torch.zeros(T, self.P, 2, dtype=torch.float64, device=device)
            self.recomb = torch.zeros(T, self.P, 2, dtype=torch.float32, device=device)
            self.healthy = torch.zeros(T, dtype=torch.int32, device=device)
            self.flagged = torch.zeros(T, dtype=torch.int32, device=device)
            # per-tensor random projection f ~ N(1,1), fixed at build time (reference: cyclic_master.py:58-61)
            g = torch.Generator().manual_seed(cfg.seed + 4242)
            f = (torch.randn(layout.total, generator=g) + 1.0) * torch.from_numpy(layout.valid_mask()).float()
            self.f = f.to(device)

    @property
    def opt_state(self) -> Dict[str, Optional[torch.Tensor]]:
        """Optimizer arenas beyond ``momentum`` (Adam second moment, AMSGrad maximum) for checkpoints, and centered clipping's
        centre (``cc_center``, only under that rule)."""
        state = {"exp_avg_sq": self.exp_avg_sq, "max_exp_avg_sq": self.max_exp_avg_sq}
        if self.plan.base == "centered_clip":
            state["cc_center"] = self.cc_center
        if self.mimic is not None:
            state["mimic_m"], state["mimic_z"] = self.mimic.m, self.mimic.z
        return state

    def enqueue_step(self, step_ptr: torch.Tensor, *, mc_params: Optional[int], dst: Sequence[int], flags: Sequence[int],
                     grad_out: Optional[torch.Tensor] = None, buckets=None, wait_bucket=None, before_update=None) -> int:
        """Decode + update + broadcast for the step in ``*step_ptr``.  Returns the number of kernels launched.

        With ``buckets`` (the workers' push buckets, in arrival order) and ``wait_bucket(b)`` the PS is pipelined: bucket
        ``b`` is voted on, applied and broadcast as soon as every worker has pushed it, while the workers are still
        back-propagating / pushing the later buckets; only the last bucket is on the critical path."""
        K, L, plan = self.K, self.layout, self.plan
        before_update = before_update or (lambda: 0)      # called right before the (last) fused update + broadcast kernel
        common = dict(params=self.params, momentum=self.momentum, exp_avg_sq=self.exp_avg_sq, max_exp_avg_sq=self.max_exp_avg_sq,
                      hp=self.hp, step_ptr=step_ptr,
                      done_counter=self.counters[0:1], first_step=1, grad_out=grad_out, mc_params=mc_params, dst=dst)
        pipelined = buckets is not None and plan.pipelined
        # (tile range, tensor range) of every bucket; None: the whole arena
        ranges = [((t0, t1), (min(idxs), max(idxs) + 1)) for t0, t1, idxs in buckets] if pipelined else [(None, None)]
        nnm = plan.source == "nnm"
        model = plan.scope == "model"                     # one choice for every tensor, from the whole-model distances
        n = 0
        if plan.source == "wbucket":                      # the step's worker buckets, before the first gradient bucket arrives
            K.wbucket_plan(self.wb_schedule, self.cfg.bucketing, step_ptr=step_ptr, masks=self.wb_mask, scales=self.wb_scale)
            n += 1
        for bi, (tiles, tensors) in enumerate(ranges):
            last = bi == len(ranges) - 1
            if pipelined:
                n += wait_bucket(bi)
            if self.attack == ATTACK_MIMIC:
                n += K.mimic_step(L, self.grad_in, self.slot_stride, self.P, adv_bitmap=self.adv_bitmap, adv_len=self.adv_len,
                                  step_ptr=step_ptr, warmup=self.cfg.mimic_w, st=self.mimic)
            elif self.attack_fold is not None:
                n += K.ps_attack_model(L, self.grad_in, self.slot_stride, self.P, adv_bitmap=self.adv_bitmap, adv_len=self.adv_len,
                                       step_ptr=step_ptr, ws=self.attack_ws, fold=self.attack_fold)
            elif self.attack:
                n += K.ps_attack(L, self.grad_in, self.slot_stride, self.P, self.attack, adv_bitmap=self.adv_bitmap,
                                 adv_len=self.adv_len, step_ptr=step_ptr, z=self.attack_z, ws=self.attack_ws,
                                 tile_range=tiles, tensor_range=tensors)
            if self.arc_ws is not None:                    # --arc model is never pipelined: one pass over the arena
                n += K.arc_clip(L, self.grad_in, self.slot_stride, self.P, self.arc_k, self.arc_ws, tile_range=tiles,
                                tensor_range=tensors)
            # row source: `rows` is the table of the worker slots the base rule reads (None: slot i is row i)
            rows = None
            if plan.source == "detox":
                K.vote(L, self.grad_in, self.slot_stride, self.group_table, self.neq_mask, self.winner_slot, self.winner_member,
                       tile_range=tiles, tensor_range=tensors); n += 2
                rows = self.winner_slot
            elif nnm and model:                            # one neighbourhood per worker over the whole model
                K.pair_dist(L, self.grad_in, self.slot_stride, self.P, self.pair_d2)
                K.pair_scope_fold(L, self.P, self.pair_d2)
                K.nnm_mix_table(L, self.P, plan.f, self.pair_d2, self.mix, mixed_out=plan.base not in ("median", "trimmed_mean"))
                n += 3
            elif nnm:                                      # the choices below read the mixed rows' distances (filled=True)
                K.nnm_mix(L, self.grad_in, self.slot_stride, self.P, plan.f, self.pair_d2, self.mix,
                          mixed_out=plan.base not in ("median", "trimmed_mean")); n += 2
            # model scope: the pair table summed over the tensors and written back into each, then filled=True below
            filled = nnm
            wb_choice = plan.source == "wbucket" and plan.base in ("krum", "multi_krum", "geomedian")
            if wb_choice and plan.rows > 1:                # the raw table, folded at model scope, then the bucket rows' table
                K.pair_dist(L, self.grad_in, self.slot_stride, self.P, self.wb_raw_d2)
                n += 1
                if model:
                    K.pair_scope_fold(L, self.P, self.wb_raw_d2); n += 1
                K.wbucket_table(L, self.P, masks=self.wb_mask, raw_d2=self.wb_raw_d2, wb_d2=self.pair_d2); n += 1
            filled = filled or wb_choice
            if model and not nnm and not wb_choice and plan.base in ("krum", "multi_krum", "geomedian", "bulyan"):
                K.pair_dist(L, self.grad_in, self.slot_stride, plan.rows, self.pair_d2, rows=rows)
                K.pair_scope_fold(L, plan.rows, self.pair_d2); n += 2
                filled = True
            # selection, then the arguments of the one fused update
            src, agg = self.grad_in, dict(K=plan.rows, select=rows)
            if plan.base in ("mean", "vote"):
                agg.update(scale=1.0 / plan.rows)
            elif plan.base == "sign_vote":                 # nothing to choose: the update kernel counts the signs
                pass
            elif plan.base == "cyclic":
                K.cyclic_project(L, self.grad_in, self.slot_stride, self.P, self.f, self.E); n += 1
                K.cyclic_locate(self.E, self.P, self.cfg.worker_fail, self.recomb, self.healthy, self.flagged); n += 1
                agg.update(scale=1.0 / self.P, recomb=self.recomb)
            elif plan.base in ("median", "trimmed_mean"):   # coordinate-wise: element by element, nothing per tensor
                agg.update(scale=1.0 / (plan.rows - 2 * plan.trim), trim=plan.trim)
            elif plan.base == "centered_clip" and model:   # one norm over the whole model, after the last bucket
                if plan.source == "wbucket":
                    self._wbucket_cc_dist(None)
                else:
                    K.centered_clip_dist(L, self.grad_in, self.slot_stride, plan.rows, self.cc_center, self.cc_partials, rows=rows)
                K.centered_clip_model_weights(L, plan.rows, self.cfg.clip_tau, self.cc_partials, self.cc_dist, self.cc_weights)
                n += 3
            elif plan.base == "centered_clip":             # per tensor, from the n distances to the centre: bucket by bucket
                if plan.source == "wbucket":
                    self._wbucket_cc_dist(tiles)
                else:
                    K.centered_clip_dist(L, self.grad_in, self.slot_stride, plan.rows, self.cc_center, self.cc_partials, rows=rows,
                                         tile_range=tiles)
                K.centered_clip_weights(L, plan.rows, self.cfg.clip_tau, self.cc_partials, self.cc_weights,
                                        tensor_range=tensors); n += 2
            elif plan.base == "bulyan":                    # select holds the rows Bulyan keeps
                K.bulyan_select(L, self.grad_in, self.slot_stride, plan.rows, plan.f, self.pair_d2, self.select, rows=rows,
                                filled=filled); n += 1 if filled else 2
                agg.update(K=plan.theta, scale=1.0 / (plan.theta - 2 * plan.f), near_median=plan.f, select=self.select)
            elif self.gm is not None:
                iters = 48
                K.geometric_median(L, self.grad_in, self.slot_stride, plan.rows, self.gm, iters=iters); n += 2 * iters + 1
                src = self.gm.median
                agg.update(K=1, scale=1.0)
            else:                                          # geometric median weights, or the m best Krum rows
                if plan.base == "geomedian" and plan.rows == 1:
                    n -= 1                                 # one bucket: its weight is 1, nothing to choose
                elif plan.base == "geomedian":
                    K.geometric_median_weights(L, self.grad_in, self.slot_stride, plan.rows, self.pair_d2, self.gm_weights,
                                               rows=rows, filled=filled)
                    choice = dict(w_mix=self.gm_weights)
                    agg.update(scale=1.0, weights=self.gm_weights)
                else:
                    K.krum_select(L, self.grad_in, self.slot_stride, plan.rows, plan.f, self.pair_d2, self.select, m=plan.m,
                                  rows=rows, filled=filled)
                    choice = dict(select=self.select, m=plan.m)
                    agg.update(K=plan.m, scale=1.0 / plan.m, select=self.select)
                n += 1 if filled else 2
                if nnm:                                    # a choice over the mixed rows, as weights over the raw slots
                    K.nnm_fold(L, self.P, plan.f, self.mix, self.w_raw, **choice); n += 1
                    agg = dict(K=self.P, scale=1.0, weights=self.w_raw)
                elif wb_choice and plan.base == "geomedian":   # the bucket rows' weights over every raw slot
                    K.wbucket_fold(L, self.P, masks=self.wb_mask, weights=self.w_raw, w_rows=self.gm_weights); n += 1
                    agg = dict(K=self.P, scale=1.0, weights=self.w_raw)
                elif wb_choice:                            # the chosen buckets' slots only, so no other slot is read
                    K.wbucket_fold(L, self.P, masks=self.wb_mask, weights=self.w_raw, select=self.select, m=plan.m,
                                   wsel=self.wb_wsel); n += 1
                    agg = dict(K=self.wb_wsel.shape[0], scale=1.0, weights=self.w_raw, select=self.wb_wsel)
            if nnm and plan.base in ("median", "trimmed_mean", "bulyan"):
                agg.update(mix=self.mix, mix_f=plan.f)
            if last:
                n += before_update()
            if plan.base == "sign_vote":                   # the vote over the P sign rows is the update's gradient source
                K.sign_vote_update(L, self.grad_in, self.slot_stride, P=plan.rows, tile_range=tiles, flags=flags if last else [],
                                   **common)
            elif plan.base == "centered_clip" and plan.source == "wbucket":
                K.wbucket_cc_update(L, src, self.slot_stride, masks=self.wb_mask, scales=self.wb_scale, center=self.cc_center,
                                    weights=self.cc_weights, tile_range=tiles, flags=flags if last else [], **common)
            elif plan.base == "centered_clip":             # the update reads and replaces the centre
                K.centered_clip_update(L, src, self.slot_stride, center=self.cc_center, weights=self.cc_weights, K=plan.rows,
                                       select=rows, tile_range=tiles, flags=flags if last else [], **common)
            elif plan.source == "wbucket" and plan.base in ("median", "trimmed_mean"):   # bucket rows formed in the kernel
                K.wbucket_update(L, self.grad_in, self.slot_stride, masks=self.wb_mask, scales=self.wb_scale, trim=plan.trim,
                                 tile_range=tiles, flags=flags if last else [], **common)
            else:
                K.aggregate_update(L, src, self.slot_stride, tile_range=tiles, flags=flags if last else [], **agg, **common)
            n += 1
        return n

    def _wbucket_cc_dist(self, tiles) -> None:
        """Centered clipping's row-to-centre partials of the bucket rows over ``tiles`` (None: the arena)."""
        self.K.wbucket_cc_dist(self.layout, self.grad_in, self.slot_stride, masks=self.wb_mask, scales=self.wb_scale,
                               center=self.cc_center, partials=self.cc_partials, tile_range=tiles)


# =====================================================================================================
# Library-op PS (NCCL baseline + CPU/Gloo)
# =====================================================================================================
class TorchPS:
    """Per-tensor decode with torch / host-C++ ops + a separate optimizer step (reference-faithful structure)."""

    def __init__(self, cfg: JobConfig, layout: ArenaLayout, device: torch.device, params: torch.Tensor,
                 groups: Optional[GroupPlan], code: Optional[CyclicCode]):
        from ..optim import SGDModified, AdamModified
        self.cfg, self.layout, self.device, self.params = cfg, layout, device, params
        self.P = cfg.num_workers
        self.groups, self.code = groups, code
        self.plan = rule_plan(cfg)
        self.rule = self.plan.rule
        # flat per-tensor views in arena element order (the optimizer is element-wise, so order is irrelevant)
        views = [params[s.offset: s.offset + s.numel] for s in layout.specs]
        self._views = views
        if cfg.optimizer == "adam":
            self.optimizer = AdamModified(views, lr=cfg.lr, betas=(cfg.adam_beta1, cfg.adam_beta2), eps=cfg.adam_eps,
                                          weight_decay=cfg.weight_decay, amsgrad=cfg.amsgrad)
        else:
            self.optimizer = SGDModified(views, lr=cfg.lr, momentum=cfg.momentum, weight_decay=cfg.weight_decay,
                                         dampening=cfg.dampening, nesterov=cfg.nesterov)
        # centered clipping's centre: last step's aggregate, +0 at the start (PS state, checkpointed as opt_state["cc_center"])
        self.cc_center = layout.new_arena(device) if self.plan.base == "centered_clip" else None
        # --err-mode mimic: the running mean and the direction (opt_state["mimic_m"] / ["mimic_z"]), see ``mimic_attack``
        self.mimic_m = self.mimic_z = None
        if cfg.err_mode == "mimic":
            self.mimic_m = layout.new_arena(device)
            self.mimic_z = torch.from_numpy(mimic_z0([(sp.offset, sp.numel) for sp in layout.specs], layout.total)).to(device)
        self.mimic_target = -1
        self.arc_k = arc_k(self.P, cfg.worker_fail) if cfg.arc else 0
        # --bucketing: the permutation of every step (row step % len, as the fused PS reads it)
        self.wb_schedule = bucket_schedule(self.P, cfg.max_steps, cfg.seed) if self.plan.source == "wbucket" else None
        if self.plan.base == "cyclic":
            g = torch.Generator().manual_seed(cfg.seed + 4242)
            f = (torch.randn(layout.total, generator=g) + 1.0) * torch.from_numpy(layout.valid_mask()).float()
            self.f = f.to(device)
        self.last_info: Dict[str, object] = {}

    # --- optimizer state for checkpoints (the reference saves none: src/master/baseline_master.py:237-243) ----------
    @property
    def momentum(self) -> Optional[torch.Tensor]:
        """SGD momentum buffers gathered into a flat arena (a copy), or None when there is nothing to save yet."""
        from ..optim import SGDModified
        if not isinstance(self.optimizer, SGDModified):
            return self._gather("exp_avg")                  # Adam: the first moment plays the momentum's role in checkpoints
        if self.cfg.momentum == 0:
            return None
        arena, found = self.layout.new_arena(self.device), False
        for v, spec in zip(self._views, self.layout.specs):
            buf = self.optimizer.state.get(v, {}).get("momentum_buffer")
            if buf is not None:
                arena[spec.offset: spec.offset + spec.numel].copy_(buf)
                found = True
        return arena if found else None

    def load_momentum(self, arena: torch.Tensor) -> None:
        key = "momentum_buffer" if self.cfg.optimizer != "adam" else "exp_avg"
        for v, spec in zip(self._views, self.layout.specs):
            self.optimizer.state[v][key] = arena[spec.offset: spec.offset + spec.numel].clone()

    def _gather(self, key: str) -> Optional[torch.Tensor]:
        arena, found = self.layout.new_arena(self.device), False
        for v, spec in zip(self._views, self.layout.specs):
            buf = self.optimizer.state.get(v, {}).get(key)
            if buf is not None:
                arena[spec.offset: spec.offset + spec.numel].copy_(buf)
                found = True
        return arena if found else None

    @property
    def opt_state(self) -> Dict[str, Optional[torch.Tensor]]:
        state = {} if self.cfg.optimizer != "adam" else {"exp_avg_sq": self._gather("exp_avg_sq"),
                                                          "max_exp_avg_sq": self._gather("max_exp_avg_sq")}
        if self.cc_center is not None:
            state["cc_center"] = self.cc_center.clone()
        if self.mimic_m is not None:
            state["mimic_m"], state["mimic_z"] = self.mimic_m.clone(), self.mimic_z.clone()
        return state

    def load_opt_state(self, arenas: Dict[str, torch.Tensor], step: int) -> None:
        """Adam: second moment (+ AMSGrad maximum) and the per-tensor step count (= updates applied so far).  Centered
        clipping: the centre."""
        arenas = dict(arenas)
        center = arenas.pop("cc_center", None)
        if self.cc_center is not None and center is not None:
            self.cc_center.copy_(center)
        for key, dst in (("mimic_m", self.mimic_m), ("mimic_z", self.mimic_z)):
            saved = arenas.pop(key, None)
            if dst is not None and saved is not None:
                dst.copy_(saved)
        if self.cfg.optimizer != "adam":
            return
        for v, spec in zip(self._views, self.layout.specs):
            st = self.optimizer.state[v]
            st["step"] = int(step)
            st.setdefault("exp_avg", torch.zeros_like(v))
            for key, arena in arenas.items():
                if arena is not None:
                    st[key] = arena[spec.offset: spec.offset + spec.numel].clone()
            st.setdefault("exp_avg_sq", torch.zeros_like(v))

    # --- the mimic attack -----------------------------------------------------------------------
    def mimic_attack(self, slots: torch.Tensor, liars: List[int], t: int) -> None:
        """``--err-mode mimic`` on the PS's slots [P, D] (``codes.adversary.mimic_step``, in fp64 torch ops on the slots'
        device): every liar slot (0-based) becomes a copy of the honest slot with the largest <x_i, z>, and while t < W (t =
        step - 1) the running mean and the direction advance.  Whole-model sums are the per-tensor fp64 sums added in
        ascending tensor order."""
        honest = [w for w in range(self.P) if w not in liars]
        if not honest:
            return
        specs = self.layout.specs
        z = self.mimic_z

        def model_dot(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:       # [..., D] x [D] -> [...]
            acc = None
            for sp in specs:
                d = (a[..., sp.offset: sp.offset + sp.numel].double() * b[sp.offset: sp.offset + sp.numel].double()).sum(-1)
                acc = d if acc is None else acc + d
            return acc

        X = slots[honest]
        s = model_dot(X, z).cpu().numpy()
        k = honest[int(np.argmax(s))]
        self.mimic_target = k
        for sp in specs:
            slots[liars, sp.offset: sp.offset + sp.numel] = slots[k, sp.offset: sp.offset + sp.numel]
        if t >= self.cfg.mimic_w:
            return
        n = len(honest)
        u = torch.zeros(self.layout.total, dtype=torch.float64, device=slots.device)
        for sp in specs:
            sl = slice(sp.offset, sp.offset + sp.numel)
            c = torch.zeros(sp.numel, dtype=torch.float64, device=slots.device)
            for i in range(n):
                c = c + X[i, sl].double()
            self.mimic_m[sl] = ((t * self.mimic_m[sl].double() + c / n) / (t + 1)).float()
        mz = float(model_dot(self.mimic_m, z))
        w = [float(si) - mz for si in s]
        for sp in specs:
            sl = slice(sp.offset, sp.offset + sp.numel)
            acc = t * z[sl].double()
            m64 = self.mimic_m[sl].double()
            for i in range(n):
                acc = acc + w[i] * (X[i, sl].double() - m64)
            u[sl] = acc
        nrm = math.sqrt(float(model_dot(u, u)))
        if nrm != 0.0:
            for sp in specs:
                sl = slice(sp.offset, sp.offset + sp.numel)
                z[sl] = (u[sl] / nrm).float()

    # --- adaptive robust clipping ----------------------------------------------------------------
    def arc_clip(self, slots: torch.Tensor) -> torch.Tensor:
        """``--arc``: every tensor of every worker slot with factor a_i < 1 (``oracle.arc_factors`` over the slots) multiplied by
        a_i in place, one fp32 multiply per element, as the fused PS clips its slab.  Returns the factors [T, P]."""
        specs = self.layout.specs
        a = arc_factors(slots.detach().cpu().numpy(), [(sp.offset, sp.numel) for sp in specs], self.cfg.worker_fail,
                        self.cfg.arc)
        for t, sp in enumerate(specs):
            for i in np.flatnonzero(a[t] < 1).tolist():
                slots[i, sp.offset: sp.offset + sp.numel] *= torch.tensor(a[t, i], dtype=torch.float32, device=slots.device)
        self.last_info["arc_factors"] = a
        return torch.from_numpy(a)

    # --- per-tensor rules -----------------------------------------------------------------------
    def _vote_tensor(self, rows: List[torch.Tensor]) -> int:
        cand, count = 0, 0
        for k, r in enumerate(rows):
            if count == 0:
                cand, count = k, 1
            elif torch.equal(r, rows[cand]):
                count += 1
            else:
                count -= 1
        return cand

    def _geomedian_tensor(self, X: torch.Tensor, iters: int = 100, eps: float = 1e-6) -> torch.Tensor:
        if X.device.type == "cpu":
            out = torch.empty(X.shape[1], dtype=torch.float32)
            Xc = X.contiguous()
            N.host().drc_host_geomedian(Xc.data_ptr(), Xc.shape[0], Xc.shape[1], Xc.stride(0), eps, iters, out.data_ptr())
            return out
        m = X.mean(0)
        for _ in range(iters):
            d = (X - m).norm(dim=1).clamp_min(1e-30)
            w = 1.0 / d
            m_new = (w[:, None] * X).sum(0) / w.sum()
            done = (m_new - m).norm() <= eps * max(1.0, float(m.norm()))
            m = m_new
            if done:
                break
        return m

    def _krum_scores(self, X: torch.Tensor, s: int) -> torch.Tensor:
        d2 = torch.cdist(X.double(), X.double()).pow(2)
        P = X.shape[0]
        keep = max(P - s - 2, 0)
        d2 = d2 + torch.diag(torch.full((P,), float("inf"), dtype=d2.dtype, device=d2.device))
        return d2.sort(dim=1).values[:, :keep].sum(1)

    def _krum_tensor(self, X: torch.Tensor) -> int:
        return int(torch.argsort(self._krum_scores(X, self.plan.f), stable=True)[0])      # NaN scores last, like the kernel

    def _multi_krum_tensor(self, X: torch.Tensor, s: int, m: int) -> torch.Tensor:
        best = torch.argsort(self._krum_scores(X, s), stable=True)[:m]
        return X[best].sum(0) / m

    def _trimmed_mean_tensor(self, X: torch.Tensor) -> torch.Tensor:
        """Sort every coordinate (NaN sorts last), drop ``trim`` values at each end, sum the rest in ascending order."""
        P, b = X.shape[0], self.plan.trim
        S = X.sort(0).values
        acc = S[b].clone()
        for k in range(b + 1, P - b):
            acc += S[k]
        return acc * (1.0 / (P - 2 * b))

    def _bulyan_tensor(self, X: torch.Tensor, f: int) -> torch.Tensor:
        """Bulyan (``oracle.bulyan``): theta = P - 2f rounds of Krum over the rows not chosen yet (squared distances in fp64, NaN
        last, ties to the lower row), then per coordinate the mean of the beta = theta - 2f chosen values nearest their median,
        in fp32 with the fused kernel's window walk and ascending sum."""
        P = X.shape[0]
        d2 = torch.cdist(X.double(), X.double()).pow(2)
        R, chosen = list(range(P)), []
        for _ in range(P - 2 * f):
            keep = max(len(R) - f - 2, 0)
            sub = d2[R][:, R].clone()
            sub.fill_diagonal_(float("nan"))               # sorts last; keep <= |R| - 2 never reaches it unless a real NaN does
            scores = sub.sort(1).values[:, :keep].sum(1)
            chosen.append(R.pop(int(torch.argsort(scores, stable=True)[0])))
        return self._nearest_to_median_mean(X[chosen], f)

    def _nearest_to_median_mean(self, X: torch.Tensor, f: int) -> torch.Tensor:
        """Bulyan's coordinate stage over the theta chosen rows ``X`` (``oracle.nearest_to_median_mean``, fp32)."""
        S = X.sort(0).values
        theta = S.shape[0]
        beta = theta - 2 * f
        lo, hi = S[(theta - 1) // 2], S[theta // 2]
        m = lo if theta % 2 else 0.5 * lo + 0.5 * hi
        s = torch.zeros(S.shape[1], dtype=torch.int64, device=S.device)
        moving = torch.ones(S.shape[1], dtype=torch.bool, device=S.device)
        for j in range(2 * f):                             # slide the window right while the entering value is nearer
            vin, vout = S[j + beta], S[j]
            din, dout = (vin - m).abs(), (vout - m).abs()
            nearer = (din < dout) | (dout.isnan() & ~din.isnan())
            moving &= nearer | (vin == vout) | (vin.isnan() & vout.isnan())
            s += moving
        acc = S.gather(0, s[None]).squeeze(0).clone()
        for k in range(1, beta):
            acc += S.gather(0, (s + k)[None]).squeeze(0)
        return acc * (1.0 / beta)

    def _nnm_mix_tensor(self, X: torch.Tensor, f: int) -> torch.Tensor:
        """Nearest-neighbour mixing (``oracle.nnm_mix``): row i becomes the mean of itself and its P - f - 1 nearest rows
        (squared distances in fp64, NaN last, ties to the lower row), formed in fp32 as the fused kernel does: from +0, add the
        neighbours in ascending row order, then multiply once by fp32(1 / (P - f))."""
        P = X.shape[0]
        d2 = torch.cdist(X.double(), X.double()).pow(2)
        d2.fill_diagonal_(-1.0)                            # row i is its own first neighbour
        return self._mix_rows(X, d2.argsort(dim=1, stable=True)[:, :P - f].sort(dim=1).values.tolist(), f)

    def _mix_rows(self, X: torch.Tensor, nbrs: List[List[int]], f: int) -> torch.Tensor:
        """Mixed row i: the fp32 sum of the rows ``nbrs[i]`` (ascending) from +0, times fp32(1 / (P - f))."""
        P = X.shape[0]
        scale = torch.tensor(1.0 / (P - f), dtype=torch.float32, device=X.device)
        Y = torch.empty_like(X)
        for i in range(P):
            y = torch.zeros_like(X[0])
            for j in nbrs[i]:
                y = y + X[j]
            Y[i] = y * scale
        return Y

    def _centered_clip_tensor(self, X: torch.Tensor, v: torch.Tensor, weights: Optional[List[float]] = None) -> torch.Tensor:
        """Centered clipping (``oracle.centered_clip``) around the centre ``v``, which it replaces: fp64 distances, fp32 weights
        from ``centered_clip_weight`` (or ``weights``, the whole-model ones), then per coordinate acc = fma_rn(w_i, rn(x_i - v),
        acc) over the rows with w_i != 0 in ascending order, and g = rn(v + acc) -- the fused kernel's fp32 order."""
        n = X.shape[0]
        if weights is None:
            weights = [centered_clip_weight(di, self.cfg.clip_tau, n) for di in (X.double() - v.double()).pow(2).sum(1).tolist()]
        acc = torch.zeros_like(v)
        for i, w in enumerate(weights):
            if w != 0.0:
                acc = _fma_f32(w, X[i] - v, acc)
        g = v + acc
        v.copy_(g)
        return g

    def _cyclic_tensor(self, R: torch.Tensor, f: torch.Tensor) -> torch.Tensor:
        """R: [n, d] complex64 -> Re(v^T R) / n with v from the C++ locator (N1 replacement)."""
        n, s = self.P, self.cfg.worker_fail
        E = (R.to(torch.complex128) @ f.to(torch.complex128))
        Eh = torch.view_as_real(E).contiguous().cpu().double().numpy()
        v = np.zeros((n, 2)); mask = np.zeros(1, dtype=np.uint32); fl = np.zeros(1, dtype=np.int32)
        N.check(N.host().drc_host_locate(Eh.ctypes.data, 1, n, s, 1e-4, v.ctypes.data, mask.ctypes.data, fl.ctypes.data), "locate")
        vt = torch.from_numpy(v[:, 0] + 1j * v[:, 1]).to(R.device).to(torch.complex64)
        self.last_info.setdefault("flagged", []).append(int(fl[0]))
        return (vt @ R).real / n

    # --- step -----------------------------------------------------------------------------------
    def _sign_vote(self, slots: torch.Tensor) -> List[torch.Tensor]:
        """``--mode sign_vote``: ``slots`` holds the P workers' sign bytes [P, D / 8] (byte i, bit b = element 8 i + b is < 0).
        Per tensor, the majority sign of every coordinate (``oracle.sign_vote``): +1, -1, or +0 on a tie."""
        P = self.P
        shifts = torch.arange(8, dtype=torch.uint8, device=slots.device)
        one = torch.ones((), dtype=torch.float32, device=slots.device)
        out = []
        for s in self.layout.specs:
            b = slots[:, s.offset // 8: s.offset // 8 + (s.numel + 7) // 8]
            bits = ((b[:, :, None] >> shifts) & 1).reshape(P, -1)[:, :s.numel]
            n_neg = bits.sum(0, dtype=torch.int32)
            n_pos = P - n_neg
            out.append(torch.where(n_pos > n_neg, one, torch.where(n_neg > n_pos, -one, torch.zeros_like(one))))
        return out

    def _wbuckets(self, step: Optional[int]) -> List[List[int]]:
        """The worker buckets of ``step`` (``codes.bucketing.wbuckets`` of the schedule's row step % len)."""
        if step is None:
            raise ValueError("--bucketing: aggregate() needs the step, which picks the permutation")
        return wbuckets(self.wb_schedule[step % len(self.wb_schedule)], self.cfg.bucketing)

    @staticmethod
    def _wbucket_rows(X: torch.Tensor, buckets: List[List[int]]) -> torch.Tensor:
        """The fp32 bucket rows (``oracle.wbucket_rows``): the lowest member, plus the others in ascending slot order, each add
        rounded, then one rounded multiply by fp32(1 / |b|); a one-member bucket's row is its member, bit for bit."""
        Y = torch.empty((len(buckets),) + tuple(X.shape[1:]), dtype=X.dtype, device=X.device)
        for b, members in enumerate(buckets):
            y = X[members[0]].clone()
            for j in members[1:]:
                y = y + X[j]
            Y[b] = y if len(members) == 1 else y * torch.tensor(1.0 / len(members), dtype=torch.float32, device=X.device)
        return Y

    def _wbucket_choice(self, Y: torch.Tensor, Db: np.ndarray) -> torch.Tensor:
        """Krum / multi-Krum / the geometric median on the bucket rows ``Y`` from their fp64 table ``Db``."""
        plan = self.plan
        if plan.base in ("krum", "multi_krum"):
            best = np.argsort(_krum_scores_d2(Db, plan.f), kind="stable")[:plan.m].tolist()
            return Y[best[0]] if plan.base == "krum" else Y[best].sum(0) / plan.m
        w = torch.from_numpy(_weiszfeld_weights(Db, 1e-10, 256)).float().to(Y.device)
        return (w[:, None] * Y).sum(0)

    def aggregate(self, slots: torch.Tensor, step: Optional[int] = None) -> List[torch.Tensor]:
        """``slots``: [P, D] fp32 (or [P, D] complex64 for cyclic, or [P, D / 8] sign bytes for sign_vote).  Returns the
        per-tensor aggregated gradients: per tensor the rows of the row source (the worker slots, the group winners of the vote,
        the mixed rows, or the worker-bucket means of ``step``'s permutation), then the base rule's helper on them."""
        plan = self.plan
        self.last_info = {}
        if self.arc_k > 0:
            self.arc_clip(slots)
        if plan.base == "sign_vote":
            return self._sign_vote(slots)
        if plan.scope == "model":
            return self._aggregate_model(slots, step)
        buckets = self._wbuckets(step) if plan.source == "wbucket" else None
        out = []
        for spec in self.layout.specs:
            X = slots[:, spec.offset: spec.offset + spec.numel]
            if plan.source == "detox":                   # the vote inside every group
                X = self._detox_rows(X)
            elif plan.source == "nnm":
                X = self._nnm_mix_tensor(X, plan.f)
            elif buckets is not None:
                Y = self._wbucket_rows(X, buckets)
                if plan.base in ("krum", "multi_krum", "geomedian"):   # distances from the raw table (oracle.wbucket_pair_d2)
                    out.append(self._wbucket_choice(Y, _wbucket_table(_pair_d2(X), buckets, self.P)))
                    continue
                X = Y
            if plan.base == "mean":
                g = X.sum(0) / plan.rows
            elif plan.base == "vote":                    # the winners summed in group order, then divided by G
                g = torch.zeros_like(X[0])
                for w in X:
                    g += w
                g = g / float(plan.rows)
            elif plan.base == "krum":
                g = X[self._krum_tensor(X)]
            elif plan.base == "multi_krum":
                g = self._multi_krum_tensor(X, plan.f, plan.m)
            elif plan.base in ("median", "trimmed_mean"):
                g = self._trimmed_mean_tensor(X)
            elif plan.base == "geomedian":
                g = self._geomedian_tensor(X)
            elif plan.base == "bulyan":
                g = self._bulyan_tensor(X, plan.f)
            elif plan.base == "centered_clip":
                g = self._centered_clip_tensor(X, self.cc_center[spec.offset: spec.offset + spec.numel])
            else:
                g = self._cyclic_tensor(X, self.f[spec.offset: spec.offset + spec.numel])
            out.append(g)
        return out

    def _detox_rows(self, X: torch.Tensor) -> torch.Tensor:
        """The G group winners of one tensor's vote, in group order."""
        winners = []
        for grp in self.groups.groups:
            rows = [X[w - 1] for w in grp]
            winners.append(rows[self._vote_tensor(rows)])
        return torch.stack(winners)

    def _aggregate_model(self, slots: torch.Tensor, step: Optional[int] = None) -> List[torch.Tensor]:
        """``--rule-scope model``: the rows of every tensor (worker slots, the per-tensor vote winners, or the worker-bucket
        means), one choice from the whole-model distances -- the per-tensor fp64 distances summed in ascending tensor order
        (``oracle.model_d2``) -- and that choice applied to every tensor: Krum / multi-Krum rows, Bulyan's theta rows (then its
        per-tensor coordinate stage), NNM neighbourhoods (then the rule on the mixed rows), the Weiszfeld weights, centered
        clipping's weights.  Worker buckets take their table from the whole-model raw table (``oracle.wbucket_pair_d2``)."""
        plan, specs = self.plan, self.layout.specs
        Xs = [slots[:, s.offset: s.offset + s.numel] for s in specs]
        if plan.source == "detox":
            Xs = [self._detox_rows(X) for X in Xs]
        if plan.source == "wbucket":
            buckets = self._wbuckets(step)
            Ys = [self._wbucket_rows(X, buckets) for X in Xs]
            if plan.base != "centered_clip":
                Db = _wbucket_table(model_d2([_pair_d2(X) for X in Xs]), buckets, self.P)
                if plan.base in ("krum", "multi_krum"):
                    best = np.argsort(_krum_scores_d2(Db, plan.f), kind="stable")[:plan.m].tolist()
                    return [Y[best[0]] if plan.base == "krum" else Y[best].sum(0) / plan.m for Y in Ys]
                w = torch.from_numpy(_weiszfeld_weights(Db, 1e-10, 256)).float().to(slots.device)
                return [(w[:, None] * Y).sum(0) for Y in Ys]
            Xs = Ys
        if plan.base == "centered_clip":
            vs = [self.cc_center[s.offset: s.offset + s.numel] for s in specs]
            d = model_d2([(X.double() - v.double()).pow(2).sum(1).cpu().numpy() for X, v in zip(Xs, vs)])
            w = [centered_clip_weight(float(di), self.cfg.clip_tau, plan.rows) for di in d]
            return [self._centered_clip_tensor(X, v, w) for X, v in zip(Xs, vs)]
        D = model_d2([_pair_d2(X) for X in Xs])
        if plan.source == "nnm":
            A = nnm_neighbours_d2(D, plan.f)
            nbrs = [[int(j) for j in np.flatnonzero(a)] for a in A]
            Xs = [self._mix_rows(X, nbrs, plan.f) for X in Xs]
            if plan.base in ("median", "trimmed_mean"):
                return [self._trimmed_mean_tensor(X) for X in Xs]
            D = nnm_pair_d2(D, A, plan.f)
        if plan.base in ("krum", "multi_krum"):
            best = np.argsort(_krum_scores_d2(D, plan.f), kind="stable")[:plan.m].tolist()
            return [X[best[0]] if plan.base == "krum" else X[best].sum(0) / plan.m for X in Xs]
        if plan.base == "bulyan":
            chosen = _bulyan_rounds(D, plan.f)
            return [self._nearest_to_median_mean(X[chosen], plan.f) for X in Xs]
        # geometric median: the Weiszfeld weights of the concatenated rows, fp32 as the fused update applies them
        w = torch.from_numpy(_weiszfeld_weights(D, 1e-10, 256)).float().to(slots.device)
        return [(w[:, None] * X).sum(0) for X in Xs]

    def step(self, slots: torch.Tensor, step: Optional[int] = None) -> None:
        self.apply(self.aggregate(slots, step=step))

    def apply(self, grads: List[torch.Tensor]) -> None:
        self.optimizer.step(grads=grads, mode=self.plan.opt_mode)


def _pair_d2(X: torch.Tensor) -> np.ndarray:
    """[P, P] fp64 squared distances between the rows of one tensor, from the fp32 values (diagonal 0)."""
    X64 = X.double()
    D = torch.stack([((X64 - X64[i]) ** 2).sum(1) for i in range(X.shape[0])]).cpu().numpy()
    np.fill_diagonal(D, 0.0)                           # a row holding NaN or Inf is NaN off the diagonal only
    return D


def _wbucket_table(D: np.ndarray, buckets: List[List[int]], P: int) -> np.ndarray:
    """[nb, nb] fp64 squared distances between the bucket rows from the raw table ``D`` [P, P]: with M = A D A^T (row b of A
    is 1 / |b| on b's members), ||y_b - y_k||^2 = M_bk - (M_bb + M_kk) / 2, clamped at 0.  A non-finite entry anywhere in D
    would reach every entry of the products, so such a table takes the per-pair form of ``oracle.wbucket_pair_d2``, which
    only reads the members of b and k."""
    if not np.isfinite(D).all():
        return wbucket_pair_d2(D, buckets, P)
    A = np.zeros((len(buckets), P))
    for b, members in enumerate(buckets):
        A[b, members] = 1.0 / len(members)
    M = A @ D @ A.T
    d = np.diag(M)
    Db = np.maximum(M - 0.5 * (d[:, None] + d[None, :]), 0.0)
    np.fill_diagonal(Db, 0.0)
    return Db


def _fma_f32(w: float, b: torch.Tensor, c: torch.Tensor) -> torch.Tensor:
    """fp32 rn(w * b + c) with one rounding, element-wise (``oracle.fma_f32``): the fp64 product is exact, the sum is rounded to
    odd in fp64 (TwoSum), then once to fp32."""
    p = b.double() * float(w)
    c64 = c.double()
    s = p + c64
    bb = s - p
    err = (p - (s - bb)) + (c64 - bb)
    odd = torch.isfinite(s) & (err != 0) & ((s.view(torch.int64) & 1) == 0)
    s = torch.where(odd, torch.nextafter(s, torch.where(err > 0, torch.full_like(s, math.inf), torch.full_like(s, -math.inf))), s)
    return s.float()


def build_codes(cfg: JobConfig):
    """(GroupPlan | None, CyclicCode | None) for a job -- the coding part of the reference's ``prepare``."""
    from ..codes.repetition import group_assign
    groups = group_assign(cfg.num_workers, cfg.group_size) if cfg.approach in ("maj_vote", "detox") else None
    code = search_w(cfg.num_workers, cfg.worker_fail) if cfg.approach == "cyclic" else None
    return groups, code
