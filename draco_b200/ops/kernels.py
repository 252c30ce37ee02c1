"""Python launchers for the sm_90a step-path kernels (thin: build the argument struct, launch on the current stream).

Every function takes either torch CUDA tensors or raw device addresses (``int``) -- peer-mapped and multicast pointers
coming from the symmetric-memory runtime are plain integers.  Nothing here falls back to PyTorch ops: if the CUDA
library is missing the call raises (see ``_native.cuda``).
"""
from __future__ import annotations

import ctypes as C
import math
import os
from typing import Optional, Sequence, Union

import torch

from .. import _native as N
from ..parallel.arena import ArenaLayout

Addr = Union[int, torch.Tensor, None]

_sm_count = {}


def addr(x: Addr) -> Optional[int]:
    if x is None:
        return None
    if isinstance(x, torch.Tensor):
        return x.data_ptr()
    return int(x)


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def sm_count(device=None) -> int:
    dev = torch.cuda.current_device() if device is None else torch.device(device).index
    if dev not in _sm_count:
        _sm_count[dev] = torch.cuda.get_device_properties(dev).multi_processor_count
    return _sm_count[dev]


def stream_grid(layout: ArenaLayout, ctas_per_sm: int = 8) -> int:
    return max(1, min(layout.ntiles, sm_count() * ctas_per_sm))


def _flag_list(flags: Sequence[Addr]) -> N.FlagList:
    fl = N.FlagList()
    assert len(flags) <= N.MAX_DST
    for i, f in enumerate(flags):
        fl.ptr[i] = addr(f)
    fl.n = len(flags)
    return fl


# ------------------------------------------------------------------------------------------------ push (K1/K2/K11)
def push_encode(layout: ArenaLayout, g32: Sequence[Addr], g16: Sequence[Addr], dst: Addr, *, step_ptr: Addr,
                worker: int, done_counter: Addr, flag: Addr = None, coef: Optional[Sequence[complex]] = None,
                adv_bitmap: Addr = None, adv_len: int = 0, attack: int = 0, magnitude: float = -100.0, seed: int = 428,
                local_copy: Addr = None, grid: Optional[int] = None, tile_range: Optional[tuple] = None,
                src_table: Addr = None, wmom: Addr = None, wm_beta: float = 0.0, sign: bool = False) -> None:
    """Fused encode + adversary + store into ``dst`` (a peer pointer) + release flag.  ``coef`` given => cyclic encode
    of ``len(coef)`` gradient streams into an interleaved complex64 slot.  ``tile_range=(t0, t1)`` pushes one bucket.
    ``wmom``: this worker's fp32 momentum arena; the push then advances it, m <- fp32(wm_beta) m + fp32(1 - wm_beta) g
    (codes/oracle.py ``worker_momentum``), and sends m (through the adversary hook) instead of g.
    ``sign``: the signSGD wire (codes/oracle.py ``sign_pack``).  ``dst`` and ``local_copy`` are then ``layout.total / 32``
    uint32 words: bit b of word w is 1 iff element 32w + b of what the plain push would store is < 0; padding bits are 0."""
    if sign and coef is not None:
        raise ValueError("the sign wire is not defined for the cyclic encode (coef)")
    if wmom is not None:
        if coef is not None:
            raise ValueError("worker momentum is not defined for the cyclic encode (coef)")
        if not 0.0 <= wm_beta < 1.0:
            raise ValueError(f"worker momentum beta must lie in [0, 1), got {wm_beta}")
    a = N.PushArgs()
    if src_table is not None:
        # zero-copy mode: `src_table` is a device int64 [R, ntensors] table of per-tensor gradient pointers
        R = len(coef) if coef is not None else 1
        a.src_table = addr(src_table)
    else:
        R = len(g32)
        needs_bf16 = any(sp.is_bf16 for sp in layout.specs)
        for k in range(R):
            a.g32[k] = addr(g32[k])
            a.g16[k] = addr(g16[k]) if g16 and g16[k] is not None else None
            if needs_bf16 and not a.g16[k]:
                raise ValueError("layout has bf16 tensors: push_encode needs the bf16 gradient arena of every stream")
    assert 1 <= R <= N.MAX_R
    a.R = R
    a.cyclic = 1 if coef is not None else 0
    if coef is not None:
        assert len(coef) == R
        for k, c in enumerate(coef):
            a.coef_re[k] = float(complex(c).real)
            a.coef_im[k] = float(complex(c).imag)
    a.dst = addr(dst)
    dev = torch.device("cuda", torch.cuda.current_device())
    a.tv = layout.tile_view(dev)
    a.adv_bitmap = addr(adv_bitmap)
    a.adv_len = adv_len if adv_bitmap is not None else 0
    a.step_ptr = addr(step_ptr)
    a.worker = worker
    a.attack = attack
    a.magnitude = magnitude
    a.seed = seed
    a.done_counter = addr(done_counter)
    a.flag = addr(flag)
    a.local_copy = addr(local_copy)
    if wmom is not None:
        from ..codes.oracle import worker_momentum_coefficients
        a.wmom = addr(wmom)
        a.wm_beta, a.wm_scale = worker_momentum_coefficients(wm_beta)
    a.sign = 1 if sign else 0
    ntiles = layout.ntiles
    if tile_range is not None:
        a.tile_begin, a.tile_end = int(tile_range[0]), int(tile_range[1])
        ntiles = a.tile_end - a.tile_begin
    N.check(N.cuda().drc_push_encode(C.byref(a), grid or max(1, min(ntiles, sm_count() * 8)), _stream()), "push_encode")


def omniscient(grad_in: Addr, slot_stride: int, honest_mask: int, worker: int, magnitude: float, total: int, *,
               step_ptr: Addr, done_counter: Addr, flag: Addr = None) -> None:
    a = N.OmniArgs(addr(grad_in), slot_stride, honest_mask, worker, magnitude, total, addr(done_counter), addr(flag),
                   addr(step_ptr))
    grid = max(1, min(sm_count() * 8, total // (N.THREADS * 4)))
    N.check(N.cuda().drc_omniscient(C.byref(a), grid, _stream()), "omniscient")


# ------------------------------------------------------------------------------------------------ PS-side attacks (C12)
ATTACK_MAXP = 16


class AttackWorkspace:
    """Scratch of the min-max attack: fp32 [2, D] mu / sigma, fp64 [ntiles, Q] per-tile partials, fp64 [T] gamma.  ALIE needs
    none (one pass writes the liars' row)."""

    def __init__(self, layout: ArenaLayout, P: int, device):
        Q = 2 * P + 1 + P * (P - 1) // 2
        self.stats = torch.zeros(2, layout.total, dtype=torch.float32, device=device)
        self.partials = torch.zeros(layout.ntiles, Q, dtype=torch.float64, device=device)
        self.gamma = torch.zeros(layout.ntensors, dtype=torch.float64, device=device)


def ps_attack(layout: ArenaLayout, grad_in: Addr, slot_stride: int, P: int, mode: int, *, adv_bitmap: Addr, adv_len: int,
              step_ptr: Addr, z: float = 0.0, ws: Optional[AttackWorkspace] = None, tile_range: Optional[tuple] = None,
              tensor_range: Optional[tuple] = None, grid: Optional[int] = None) -> int:
    """Overwrite the liar slots of the step (``adv_bitmap[*step_ptr % adv_len]``) of ``grad_in`` [P, slot_stride] with the ALIE
    (``mode`` 5, ``z``), min-max (``mode`` 6, workspace ``ws``) or IPM (``mode`` 7, ``z`` = eps) row of every tensor, built from
    the honest slots (csrc/cuda/attack.cu).  ``tile_range`` / ``tensor_range``: one bucket (whole tensors).  Returns the
    kernels launched."""
    a, g = _attack_args(layout, grad_in, slot_stride, P, mode, adv_bitmap, adv_len, step_ptr, z, ws, tile_range, grid)
    if tensor_range is not None:
        a.t_begin, a.t_end = int(tensor_range[0]), int(tensor_range[1])
    lib = N.cuda()
    if mode == 7:
        N.check(lib.drc_attack_ipm(C.byref(a), g, _stream()), "attack_ipm")
        return 1
    N.check(lib.drc_attack_stats(C.byref(a), g, _stream()), "attack_stats")
    if mode == 5:
        return 1
    N.check(lib.drc_attack_solve(C.byref(a), _stream()), "attack_solve")
    N.check(lib.drc_attack_write(C.byref(a), g, _stream()), "attack_write")
    return 3


def _attack_args(layout, grad_in, slot_stride, P, mode, adv_bitmap, adv_len, step_ptr, z, ws, tile_range, grid):
    """The ``AttackArgs`` both attack launchers share, and the grid of the tile kernels."""
    if not 1 <= P <= ATTACK_MAXP:
        raise ValueError(f"the PS-side attacks take 1..{ATTACK_MAXP} worker slots, got {P}")
    if mode not in (5, 6, 7):
        raise ValueError(f"attack mode must be 5 (alie), 6 (minmax) or 7 (ipm), got {mode}")
    if mode == 6 and ws is None:
        raise ValueError("the min-max attack needs an AttackWorkspace")
    dev = torch.device("cuda", torch.cuda.current_device())
    a = N.AttackArgs()
    a.grad_in, a.slot_stride, a.P, a.mode = addr(grad_in), slot_stride, P, mode
    a.tv = layout.tile_view(dev)
    a.adv_bitmap, a.adv_len, a.step_ptr, a.z = addr(adv_bitmap), int(adv_len) if adv_bitmap is not None else 0, addr(step_ptr), float(z)
    if ws is not None:
        a.stats, a.partials, a.gamma = ws.stats.data_ptr(), ws.partials.data_ptr(), ws.gamma.data_ptr()
    ntiles = layout.ntiles
    if tile_range is not None:
        a.tile_begin, a.tile_end = int(tile_range[0]), int(tile_range[1])
        ntiles = a.tile_end - a.tile_begin
    return a, grid or max(1, min(ntiles, sm_count() * 8))


def attack_fold_buffer(layout: ArenaLayout, P: int, device) -> torch.Tensor:
    """The fp64 [T, Q] scratch of ``ps_attack_model``: each tensor's min-max partials folded in tile order."""
    return torch.zeros(layout.ntensors, 2 * P + 1 + P * (P - 1) // 2, dtype=torch.float64, device=device)


def ps_attack_model(layout: ArenaLayout, grad_in: Addr, slot_stride: int, P: int, *, adv_bitmap: Addr, adv_len: int,
                    step_ptr: Addr, ws: AttackWorkspace, fold: torch.Tensor, grid: Optional[int] = None) -> int:
    """The min-max attack with one gamma and one Dmax over the whole model (``--attack-scope model``; codes/adversary.py
    ``minmax_gamma_model``): the stats pass over the arena, the per-tensor fold of its partials into ``fold``
    (``attack_fold_buffer``), one solve over their sum in ascending tensor order, which writes gamma into every tensor, then
    the write pass.  Returns the kernels launched."""
    Q = 2 * P + 1 + P * (P - 1) // 2
    _check_buffer("ps_attack_model: fold", fold, torch.float64, (layout.ntensors, Q))
    a, g = _attack_args(layout, grad_in, slot_stride, P, 6, adv_bitmap, adv_len, step_ptr, 0.0, ws, None, grid)
    a.fold = fold.data_ptr()
    lib = N.cuda()
    N.check(lib.drc_attack_stats(C.byref(a), g, _stream()), "attack_stats")
    N.check(lib.drc_attack_solve_model(C.byref(a), _stream()), "attack_solve_model")
    N.check(lib.drc_attack_write(C.byref(a), g, _stream()), "attack_write")
    return 4


class MimicState:
    """The mimic attack's PS state and scratch (csrc/cuda/mimic.cu): the fp32 arenas ``m`` (running mean of the honest means,
    +0 at the start) and ``z`` (the unit direction, ``z0`` at the start), the fp64 arena ``u``, the per-tile and per-tensor
    fp64 partials, the w_i and the step's target slot."""

    def __init__(self, layout: ArenaLayout, P: int, device, z0: torch.Tensor):
        if not 1 <= P <= ATTACK_MAXP:
            raise ValueError(f"the mimic attack takes 1..{ATTACK_MAXP} worker slots, got {P}")
        self.m = layout.new_arena(device)
        self.z = z0.to(device=device, dtype=torch.float32).clone()
        _check_buffer("MimicState: z0", self.z, torch.float32, (layout.total,))
        self.u = torch.zeros(layout.total, dtype=torch.float64, device=device)
        self.partials = torch.zeros(layout.ntiles, P + 1, dtype=torch.float64, device=device)
        self.fold = torch.zeros(layout.ntensors, P + 1, dtype=torch.float64, device=device)
        self.upart = torch.zeros(layout.ntiles, dtype=torch.float64, device=device)
        self.ufold = torch.zeros(layout.ntensors, dtype=torch.float64, device=device)
        self.w = torch.zeros(P, dtype=torch.float64, device=device)
        self.target = torch.zeros(1, dtype=torch.int32, device=device)


def mimic_step(layout: ArenaLayout, grad_in: Addr, slot_stride: int, P: int, *, adv_bitmap: Addr, adv_len: int, step_ptr: Addr,
               warmup: int, st: MimicState, grid: Optional[int] = None) -> int:
    """One step of the mimic attack over the whole arena (codes/adversary.py ``mimic_step``): every liar slot of the step becomes
    a copy of the honest slot with the largest <x_i, z>, and while ``*step_ptr - 1 < warmup`` the state ``st`` advances.  Six
    kernels, the last two warm-up only (they return on the device after it).  Returns the kernels launched."""
    if warmup < 0:
        raise ValueError(f"mimic warm-up must be >= 0, got {warmup}")
    dev = torch.device("cuda", torch.cuda.current_device())
    a = N.MimicArgs()
    a.grad_in, a.slot_stride, a.P, a.warmup = addr(grad_in), slot_stride, P, int(warmup)
    a.tv = layout.tile_view(dev)
    a.adv_bitmap, a.adv_len, a.step_ptr = addr(adv_bitmap), int(adv_len) if adv_bitmap is not None else 0, addr(step_ptr)
    a.m, a.z, a.u = st.m.data_ptr(), st.z.data_ptr(), st.u.data_ptr()
    a.partials, a.fold, a.upart, a.ufold = st.partials.data_ptr(), st.fold.data_ptr(), st.upart.data_ptr(), st.ufold.data_ptr()
    a.w, a.target = st.w.data_ptr(), st.target.data_ptr()
    N.check(N.cuda().drc_mimic_step(C.byref(a), grid or stream_grid(layout), _stream()), "mimic_step")
    return 6


# ------------------------------------------------------------------------------------------------ vote (K3)
def vote(layout: ArenaLayout, grad_in: Addr, slot_stride: int, group_table: torch.Tensor, neq_mask: torch.Tensor,
         winner_slot: torch.Tensor, winner_member: Optional[torch.Tensor] = None, tile_range: Optional[tuple] = None,
         tensor_range: Optional[tuple] = None) -> None:
    """Exact-equality majority vote.  ``group_table``: int32 [G, max_r] worker slots (-1 padded); ``neq_mask``: zeroed
    uint32/int32 [G, T] scratch (left zeroed again on return); ``winner_slot``: int32 [G, T] out."""
    G, max_r = group_table.shape
    dev = group_table.device
    t0, t1 = tile_range if tile_range is not None else (0, 0)
    va = N.VoteArgs(addr(grad_in), slot_stride, group_table.data_ptr(), G, max_r, layout.tile_view(dev), neq_mask.data_ptr(),
                    int(t0), int(t1))
    ntiles = (t1 - t0) if tile_range is not None else layout.ntiles
    N.check(N.cuda().drc_vote_compare(C.byref(va), max(1, min(ntiles, sm_count() * 8)), _stream()), "vote_compare")
    q0, q1 = tensor_range if tensor_range is not None else (0, 0)
    ra = N.ResolveArgs(neq_mask.data_ptr(), group_table.data_ptr(), G, max_r, layout.ntensors, winner_slot.data_ptr(),
                       addr(winner_member), neq_mask.data_ptr(), int(q0), int(q1))
    N.check(N.cuda().drc_vote_resolve(C.byref(ra), _stream()), "vote_resolve")


# ------------------------------------------------------------------------------------------------ update (K7/K8/K9)
ROW_TABLE_MAXROWS = 16


def _check_row_table(layout: ArenaLayout, table, rows: int) -> None:
    """A row table of the trimmed mean, the weighted sum, pair distances or Krum: a contiguous int32 CUDA tensor [rows, T] with
    1 <= rows <= 16 (the kernels read entry (k, t) at k * T + t)."""
    T = layout.ntensors
    if not isinstance(table, torch.Tensor) or table.dtype != torch.int32 or not table.is_cuda or not table.is_contiguous():
        raise ValueError("row table: expected a contiguous int32 CUDA tensor")
    if tuple(table.shape) != (rows, T) or not 1 <= rows <= ROW_TABLE_MAXROWS:
        raise ValueError(f"row table: expected shape ({rows}, {T}) with at most {ROW_TABLE_MAXROWS} rows, got {tuple(table.shape)}")


def aggregate_update(layout: ArenaLayout, grad_in: Addr, slot_stride: int, *, params: Addr, momentum: Addr, hp: Addr,
                     step_ptr: Addr, done_counter: Addr, K: int, scale: float, select: Addr = None,
                     recomb: Addr = None, first_step: int = 1, grad_out: Addr = None, mc_params: Addr = None,
                     dst: Sequence[Addr] = (), flags: Sequence[Addr] = (), grid: Optional[int] = None,
                     tile_range: Optional[tuple] = None, weights: Addr = None, exp_avg_sq: Addr = None,
                     max_exp_avg_sq: Addr = None, trim: Optional[int] = None, near_median: Optional[int] = None,
                     mix: Optional[torch.Tensor] = None, mix_f: Optional[int] = None) -> None:
    """Fused aggregate (select-sum, cyclic recombination, real per-tensor ``weights`` [T, K], -- with ``trim`` -- the
    coordinate-wise trimmed mean of K <= 16 rows that drops ``trim`` values at each end, or -- with ``near_median = f`` --
    Bulyan's coordinate stage: the mean of the K - 2f values nearest the coordinate median of the K <= 16 rows ``select``
    names, csrc/cuda/aggregate_update.cu mode 4) + optimizer step (SGD-momentum, or
    Adam / AMSGrad when the hyper-parameter block says so: ``momentum`` = first moment, ``exp_avg_sq`` / ``max_exp_avg_sq`` = second
    moment / its running maximum) + parameter broadcast + flags.

    ``select``: int32 [K, T] table of the worker slot that row k of tensor t is read from (rows 0..K-1 when None).  It applies to
    the select-sum, to the ``weights`` sum and to the trimmed mean; DETOX passes the vote's ``winner_slot`` so that the rule runs
    on the group winners.

    ``mix`` (with ``trim`` or ``near_median``): the int32 [P, T] neighbour masks of ``nnm_mix`` and ``mix_f`` = f.  The trimmed
    mean / median then runs on the K = P mixed rows (no ``select``), Bulyan's coordinate stage on the K = theta mixed rows that
    ``select`` names (mixed-row indices from ``bulyan_select``); mixed row i is the fp32 mean of the raw slots in N_i, formed in
    the kernel (csrc/cuda/aggregate_update.cu, mixed_robust_f4)."""
    a = N.UpdateArgs()
    a.mode = 1 if recomb is not None else (2 if weights is not None else 0)
    if weights is not None:
        assert recomb is None
        if select is not None:
            _check_row_table(layout, select, K)
        recomb = weights
    if trim is not None or near_median is not None:       # modes 3 and 4 sort K <= 16 rows and drop 2 * trim of them
        assert recomb is None and (trim is None or near_median is None)
        name, var, t = ("trimmed mean", "trim", trim) if trim is not None else ("nearest-to-median mean", "f", near_median)
        if near_median is not None and select is None:
            raise ValueError("nearest-to-median mean: needs the select table of the rows bulyan_select chose")
        if select is not None:
            _check_row_table(layout, select, K)
        if not (1 <= K <= 16 and 0 <= 2 * t < K):
            raise ValueError(f"{name}: K = {K} rows (at most 16) must exceed 2 * {var} = {2 * t}")
        if abs(scale * (K - 2 * t) - 1.0) > 1e-6:
            raise ValueError(f"{name}: scale must be 1 / (K - 2 * {var}) = {1.0 / (K - 2 * t)}, got {scale}")
        a.mode, a.trim = 3 if trim is not None else 4, int(t)
    if mix is not None:
        if trim is None and near_median is None:
            raise ValueError("mixing: only the trimmed mean / median (trim=) and Bulyan's stage (near_median=) take mix=")
        P = mix.shape[0] if mix.dim() == 2 else 0
        _check_row_table(layout, mix, P)
        if mix_f is None or not 0 <= mix_f < P:
            raise ValueError(f"mixing: needs 0 <= mix_f < P = {P} (got {mix_f})")
        if trim is not None and (K != P or select is not None):
            raise ValueError(f"mixing: the trimmed mean runs on all P = {P} mixed rows (K = {K}) and takes no select table")
        if near_median is not None and K > P:
            raise ValueError(f"mixing: Bulyan's stage takes at most P = {P} mixed rows (K = {K})")
        a.mix, a.mixP, a.mix_scale = mix.data_ptr(), P, 1.0 / (P - mix_f)
    _launch_update(a, layout, grad_in, slot_stride, select=select, K=K, scale=scale, recomb=recomb, params=params,
                   momentum=momentum, exp_avg_sq=exp_avg_sq, max_exp_avg_sq=max_exp_avg_sq, hp=hp, step_ptr=step_ptr,
                   first_step=first_step, grad_out=grad_out, mc_params=mc_params, dst=dst, done_counter=done_counter, flags=flags,
                   tile_range=tile_range, grid=grid)


def _launch_update(a: N.UpdateArgs, layout: ArenaLayout, grad_in: Addr, slot_stride: int, *, select, K, scale, recomb, params,
                   momentum, exp_avg_sq, max_exp_avg_sq, hp, step_ptr, first_step, grad_out, mc_params, dst, done_counter, flags,
                   tile_range, grid) -> None:
    """Fill the fields every mode of ``UpdateArgs`` shares and launch the fused update (``a`` holds the mode's own fields)."""
    a.grad_in = addr(grad_in)
    a.slot_stride = slot_stride
    a.select = addr(select)
    a.K = K
    a.scale = scale
    a.recomb = addr(recomb)
    dev = torch.device("cuda", torch.cuda.current_device())
    a.tv = layout.tile_view(dev)
    a.params = addr(params)
    a.momentum = addr(momentum)
    a.exp_avg_sq = addr(exp_avg_sq)
    a.max_exp_avg_sq = addr(max_exp_avg_sq)
    a.hp = addr(hp)
    a.step_ptr = addr(step_ptr)
    a.first_step = first_step
    a.grad_out = addr(grad_out)
    a.mc_params = addr(mc_params)
    assert len(dst) <= N.MAX_DST
    for i, d in enumerate(dst):
        a.dst[i] = addr(d)
    a.ndst = len(dst)
    a.done_counter = addr(done_counter)
    a.flags = _flag_list(flags)
    ntiles = layout.ntiles
    if tile_range is not None:
        a.tile_begin, a.tile_end = int(tile_range[0]), int(tile_range[1])
        ntiles = a.tile_end - a.tile_begin
    N.check(N.cuda().drc_aggregate_update(C.byref(a), grid or max(1, min(ntiles, sm_count() * 8)), _stream()), "aggregate_update")


WBUCKET_MAXP = 16      # raw slots the fused bucket rules take (the sorting networks' TRIM_MAXP)


def wbucket_plan(schedule: torch.Tensor, s: int, *, step_ptr: Addr, masks: torch.Tensor, scales: torch.Tensor) -> None:
    """--bucketing s: from row ``*step_ptr % len`` of the int32 [len, P] permutation ``schedule`` (codes.bucketing.
    bucket_schedule), write the step's nb = ceil(P / s) bucket rows into ``masks`` (int32 [nb], bit j = slot j; codes.bucketing.
    wbucket_masks) and ``scales`` (fp32 [nb], fp32(1 / |b|)), rows ordered by their lowest member.  One single-thread kernel."""
    if schedule.dim() != 2 or schedule.dtype != torch.int32 or not schedule.is_cuda or not schedule.is_contiguous():
        raise ValueError("wbucket plan: schedule must be a contiguous int32 CUDA tensor [len, P]")
    L, P = schedule.shape
    if not (1 <= P <= WBUCKET_MAXP and 1 <= s <= P and L >= 1):
        raise ValueError(f"wbucket plan: needs 1 <= s <= P <= {WBUCKET_MAXP} (got P = {P}, s = {s})")
    nb = -(-P // s)
    _check_buffer("wbucket plan: masks", masks, torch.int32, (nb,))
    _check_buffer("wbucket plan: scales", scales, torch.float32, (nb,))
    a = N.WbucketPlanArgs(schedule.data_ptr(), L, P, s, addr(step_ptr), masks.data_ptr(), scales.data_ptr())
    N.check(N.cuda().drc_wbucket_plan(C.byref(a), _stream()), "wbucket_plan")


def wbucket_update(layout: ArenaLayout, grad_in: Addr, slot_stride: int, *, masks: torch.Tensor, scales: torch.Tensor, trim: int,
                   params: Addr, momentum: Addr, hp: Addr, step_ptr: Addr, done_counter: Addr, first_step: int = 1,
                   grad_out: Addr = None, mc_params: Addr = None, dst: Sequence[Addr] = (), flags: Sequence[Addr] = (),
                   grid: Optional[int] = None, tile_range: Optional[tuple] = None, exp_avg_sq: Addr = None,
                   max_exp_avg_sq: Addr = None) -> None:
    """The coordinate-wise trimmed mean / median over the K = nb worker-bucket rows of ``masks`` / ``scales`` (``wbucket_plan``;
    update-kernel mode 7: each bucket row formed in fp32 from its raw slots, codes/oracle.py ``wbucket_rows``), dropping ``trim``
    values at each end, scaled by 1 / (nb - 2 trim), + the unchanged optimizer step, broadcast and flags."""
    nb = masks.shape[0] if masks.dim() == 1 else 0
    if not (1 <= nb <= WBUCKET_MAXP and 0 <= 2 * trim < nb):
        raise ValueError(f"wbucket trimmed mean: nb = {nb} rows (at most {WBUCKET_MAXP}) must exceed 2 * trim = {2 * trim}")
    _check_buffer("wbucket update: masks", masks, torch.int32, (nb,))
    _check_buffer("wbucket update: scales", scales, torch.float32, (nb,))
    a = N.UpdateArgs()
    a.mode, a.trim, a.wb_mask, a.wb_scale = 7, int(trim), masks.data_ptr(), scales.data_ptr()
    _launch_update(a, layout, grad_in, slot_stride, select=None, K=nb, scale=1.0 / (nb - 2 * trim), recomb=None, params=params,
                   momentum=momentum, exp_avg_sq=exp_avg_sq, max_exp_avg_sq=max_exp_avg_sq, hp=hp, step_ptr=step_ptr,
                   first_step=first_step, grad_out=grad_out, mc_params=mc_params, dst=dst, done_counter=done_counter, flags=flags,
                   tile_range=tile_range, grid=grid)


def wbucket_cc_dist(layout: ArenaLayout, grad_in: Addr, slot_stride: int, *, masks: torch.Tensor, scales: torch.Tensor,
                    center: torch.Tensor, partials: torch.Tensor, tile_range: Optional[tuple] = None,
                    grid: Optional[int] = None) -> None:
    """``centered_clip_dist`` over the n = nb worker-bucket rows of ``masks`` / ``scales`` (each row formed in fp32 from its raw
    slots, codes/oracle.py ``wbucket_rows``; csrc/cuda/clip.cu ``cc_dist_wbucket_kernel``).  ``centered_clip_weights`` /
    ``centered_clip_model_weights`` then run unchanged with n = nb."""
    nb = masks.shape[0] if masks.dim() == 1 else 0
    _check_cc_rows("wbucket_cc_dist", nb)
    _check_buffer("wbucket_cc_dist: masks", masks, torch.int32, (nb,))
    _check_buffer("wbucket_cc_dist: scales", scales, torch.float32, (nb,))
    _check_buffer("wbucket_cc_dist: center", center, torch.float32, (layout.total,))
    _check_buffer("wbucket_cc_dist: partials", partials, torch.float64, (layout.ntiles, nb))
    a = N.CcArgs()
    a.grad_in, a.slot_stride, a.n = addr(grad_in), slot_stride, nb
    a.tv = layout.tile_view(center.device)
    a.center, a.partials, a.wb_mask, a.wb_scale = center.data_ptr(), partials.data_ptr(), masks.data_ptr(), scales.data_ptr()
    ntiles = layout.ntiles
    if tile_range is not None:
        a.tile_begin, a.tile_end = int(tile_range[0]), int(tile_range[1])
        ntiles = a.tile_end - a.tile_begin
    N.check(N.cuda().drc_cc_dist(C.byref(a), grid or max(1, min(ntiles, sm_count() * 8)), _stream()), "cc_dist")


def wbucket_cc_update(layout: ArenaLayout, grad_in: Addr, slot_stride: int, *, masks: torch.Tensor, scales: torch.Tensor,
                      center: torch.Tensor, weights: torch.Tensor, params: Addr, momentum: Addr, hp: Addr, step_ptr: Addr,
                      done_counter: Addr, first_step: int = 1, grad_out: Addr = None, mc_params: Addr = None,
                      dst: Sequence[Addr] = (), flags: Sequence[Addr] = (), grid: Optional[int] = None,
                      tile_range: Optional[tuple] = None, exp_avg_sq: Addr = None, max_exp_avg_sq: Addr = None) -> None:
    """``centered_clip_update`` over the K = nb worker-bucket rows (update-kernel mode 8): a bucket of weight 0 is never read,
    the others are formed in fp32 from their raw slots as in ``wbucket_update``."""
    nb = masks.shape[0] if masks.dim() == 1 else 0
    _check_cc_rows("wbucket_cc_update", nb)
    _check_buffer("wbucket_cc_update: masks", masks, torch.int32, (nb,))
    _check_buffer("wbucket_cc_update: scales", scales, torch.float32, (nb,))
    _check_buffer("wbucket_cc_update: center", center, torch.float32, (layout.total,))
    _check_buffer("wbucket_cc_update: weights", weights, torch.float32, (layout.ntensors, nb))
    a = N.UpdateArgs()
    a.mode, a.center, a.wb_mask, a.wb_scale = 8, center.data_ptr(), masks.data_ptr(), scales.data_ptr()
    _launch_update(a, layout, grad_in, slot_stride, select=None, K=nb, scale=1.0, recomb=weights, params=params,
                   momentum=momentum, exp_avg_sq=exp_avg_sq, max_exp_avg_sq=max_exp_avg_sq, hp=hp, step_ptr=step_ptr,
                   first_step=first_step, grad_out=grad_out, mc_params=mc_params, dst=dst, done_counter=done_counter, flags=flags,
                   tile_range=tile_range, grid=grid)


def wbucket_table(layout: ArenaLayout, P: int, *, masks: torch.Tensor, raw_d2: torch.Tensor, wb_d2: torch.Tensor) -> None:
    """The nb bucket rows' pair table ``wb_d2`` [T, nb(nb-1)/2] fp64 from the raw slots' table ``raw_d2`` [T, P(P-1)/2]
    (``pair_dist``, then ``pair_scope_fold`` at model scope), which it zeroes: -1/2 c^T D c clamped at 0 (codes/oracle.py
    ``wbucket_pair_d2``; csrc/cuda/bucketing.cu).  ``krum_select`` / ``geometric_median_weights`` then read ``wb_d2`` with
    ``filled=True``."""
    nb = masks.shape[0] if masks.dim() == 1 else 0
    if not 2 <= nb <= P <= WBUCKET_MAXP:
        raise ValueError(f"wbucket_table: needs 2 <= nb <= P <= {WBUCKET_MAXP} (got nb = {nb}, P = {P})")
    _check_buffer("wbucket_table: masks", masks, torch.int32, (nb,))
    _check_pair_table("wbucket_table: raw", layout, P, raw_d2)
    _check_pair_table("wbucket_table: bucket", layout, nb, wb_d2)
    a = N.WbucketArgs(masks.data_ptr(), nb, P, layout.ntensors, raw_d2.data_ptr(), wb_d2.data_ptr())
    N.check(N.cuda().drc_wbucket_table(C.byref(a), _stream()), "wbucket_table")


def wbucket_fold(layout: ArenaLayout, P: int, *, masks: torch.Tensor, weights: torch.Tensor, select: Optional[torch.Tensor] = None,
                 m: int = 0, wsel: Optional[torch.Tensor] = None, w_rows: Optional[torch.Tensor] = None) -> None:
    """A choice over the bucket rows as weights over the raw slots (w_b / |b|, formed in fp64, rounded to fp32 once;
    csrc/cuda/bucketing.cu).  Krum / multi-Krum (``select``: int32 [m, T] bucket rows): the compact ``wsel`` int32 [K, T] slots
    and ``weights`` fp32 [T, K], K = min(m s, P), padded with weight 0 on a chosen slot, for ``aggregate_update(K=K,
    weights=weights, select=wsel)``.  Geometric median (``w_rows``: fp32 [T, nb]): ``weights`` fp32 [T, P] over every slot."""
    nb, T = (masks.shape[0] if masks.dim() == 1 else 0), layout.ntensors
    if not 1 <= nb <= P <= WBUCKET_MAXP:
        raise ValueError(f"wbucket_fold: needs 1 <= nb <= P <= {WBUCKET_MAXP} (got nb = {nb}, P = {P})")
    _check_buffer("wbucket_fold: masks", masks, torch.int32, (nb,))
    a = N.WbucketArgs()
    a.masks, a.nb, a.P, a.T = masks.data_ptr(), nb, P, T
    if (select is None) == (w_rows is None):
        raise ValueError("wbucket_fold: pass either select (Krum / multi-Krum) or w_rows (geometric median)")
    if select is not None:
        if not 1 <= m <= nb:
            raise ValueError(f"wbucket_fold: needs 1 <= m <= nb = {nb}, got {m}")
        _check_buffer("wbucket_fold: select", select, torch.int32, (m, T))
        K = wsel.shape[0] if isinstance(wsel, torch.Tensor) and wsel.dim() == 2 else 0
        if not 1 <= K <= P:
            raise ValueError(f"wbucket_fold: wsel must be int32 [K, T] with 1 <= K <= P = {P}")
        _check_buffer("wbucket_fold: wsel", wsel, torch.int32, (K, T))
        _check_buffer("wbucket_fold: weights", weights, torch.float32, (T, K))
        a.select, a.m, a.wsel, a.wts, a.K = select.data_ptr(), m, wsel.data_ptr(), weights.data_ptr(), K
    else:
        _check_buffer("wbucket_fold: w_rows", w_rows, torch.float32, (T, nb))
        _check_buffer("wbucket_fold: weights", weights, torch.float32, (T, P))
        a.w_rows, a.wts = w_rows.data_ptr(), weights.data_ptr()
    N.check(N.cuda().drc_wbucket_fold(C.byref(a), _stream()), "wbucket_fold")


SIGN_VOTE_MAXP = N.MAX_WORKERS


def sign_vote_update(layout: ArenaLayout, grad_in: Addr, slot_stride: int, *, P: int, params: Addr, momentum: Addr, hp: Addr,
                     step_ptr: Addr, done_counter: Addr, first_step: int = 1, grad_out: Addr = None, mc_params: Addr = None,
                     dst: Sequence[Addr] = (), flags: Sequence[Addr] = (), grid: Optional[int] = None,
                     tile_range: Optional[tuple] = None, exp_avg_sq: Addr = None, max_exp_avg_sq: Addr = None) -> None:
    """signSGD with majority vote (update-kernel mode 6, codes/oracle.py ``sign_vote``) + the unchanged optimizer step,
    broadcast and flags.  ``grad_in``: the P <= 32 sign rows of ``push_encode(sign=True)`` in slots 0..P-1, ``slot_stride``
    uint32 words apart (at least ``layout.total / 32``).  Per coordinate g = +1 if more rows say "+" than "-", -1 if more say
    "-", +0 on a tie and on padding; g enters the optimizer with scale 1."""
    if not 1 <= P <= SIGN_VOTE_MAXP:
        raise ValueError(f"sign vote: takes 1..{SIGN_VOTE_MAXP} rows (the adversary bitmaps' width), got {P}")
    if slot_stride < layout.total // 32:
        raise ValueError(f"sign vote: slot_stride is in uint32 words and must hold a slot of {layout.total // 32}, got {slot_stride}")
    a = N.UpdateArgs()
    a.mode = 6
    _launch_update(a, layout, grad_in, slot_stride, select=None, K=P, scale=1.0, recomb=None, params=params,
                   momentum=momentum, exp_avg_sq=exp_avg_sq, max_exp_avg_sq=max_exp_avg_sq, hp=hp, step_ptr=step_ptr,
                   first_step=first_step, grad_out=grad_out, mc_params=mc_params, dst=dst, done_counter=done_counter, flags=flags,
                   tile_range=tile_range, grid=grid)


# ------------------------------------------------------------------------------------------------ centered clipping (C13)
CC_MAXROWS = 16


def _check_buffer(what: str, t, dtype: torch.dtype, shape: tuple) -> None:
    if (not isinstance(t, torch.Tensor) or t.dtype != dtype or not t.is_cuda or not t.is_contiguous()
            or tuple(t.shape) != tuple(shape)):
        got = (tuple(t.shape), t.dtype) if isinstance(t, torch.Tensor) else type(t).__name__
        raise ValueError(f"{what}: expected a contiguous {dtype} CUDA tensor of shape {tuple(shape)}, got {got}")


def _check_cc_rows(what: str, n: int) -> None:
    if not 1 <= n <= CC_MAXROWS:
        raise ValueError(f"{what}: takes 1..{CC_MAXROWS} rows, got {n}")


def centered_clip_dist(layout: ArenaLayout, grad_in: Addr, slot_stride: int, n: int, center: torch.Tensor,
                       partials: torch.Tensor, *, rows: Optional[torch.Tensor] = None, tile_range: Optional[tuple] = None,
                       grid: Optional[int] = None) -> None:
    """Centered clipping's distances (csrc/cuda/clip.cu): for every tile of ``tile_range`` (one bucket; None: the arena) and
    each of the ``n`` rows, the fp64 sum of ((double)x - (double)v)^2 over the tile's real elements into ``partials``
    [ntiles, n] fp64.  ``center``: the fp32 arena v.  ``rows``: optional int32 [n, T] table, row i of tensor t is worker slot
    ``rows[i, t]`` (DETOX: the vote's winner_slot); slot i without one."""
    _check_cc_rows("centered_clip_dist", n)
    if rows is not None:
        _check_row_table(layout, rows, n)
    _check_buffer("centered_clip_dist: center", center, torch.float32, (layout.total,))
    _check_buffer("centered_clip_dist: partials", partials, torch.float64, (layout.ntiles, n))
    a = N.CcArgs()
    a.grad_in, a.slot_stride, a.n, a.rows = addr(grad_in), slot_stride, n, addr(rows)
    a.tv = layout.tile_view(center.device)
    a.center, a.partials = center.data_ptr(), partials.data_ptr()
    ntiles = layout.ntiles
    if tile_range is not None:
        a.tile_begin, a.tile_end = int(tile_range[0]), int(tile_range[1])
        ntiles = a.tile_end - a.tile_begin
    N.check(N.cuda().drc_cc_dist(C.byref(a), grid or max(1, min(ntiles, sm_count() * 8)), _stream()), "cc_dist")


def centered_clip_weights(layout: ArenaLayout, n: int, tau: float, partials: torch.Tensor, weights: torch.Tensor, *,
                          tensor_range: Optional[tuple] = None) -> None:
    """Fold ``centered_clip_dist``'s partials per tensor in tile order into d_i and write ``weights`` [T, n] fp32:
    fp32(min(1, tau / sqrt(d_i)) / n), fp32(1 / n) for d_i = 0 and 0 for a NaN or +Inf d_i (codes/oracle.py
    ``centered_clip_weights``).  ``tensor_range``: the tensors of one bucket (None: every tensor)."""
    _check_cc_rows("centered_clip_weights", n)
    if not (math.isfinite(tau) and tau > 0):
        raise ValueError(f"centered_clip_weights: tau must be finite and > 0, got {tau}")
    _check_buffer("centered_clip_weights: partials", partials, torch.float64, (layout.ntiles, n))
    _check_buffer("centered_clip_weights: weights", weights, torch.float32, (layout.ntensors, n))
    a = N.CcArgs()
    a.n, a.tv = n, layout.tile_view(weights.device)
    a.partials, a.weights, a.tau = partials.data_ptr(), weights.data_ptr(), float(tau)
    if tensor_range is not None:
        a.t_begin, a.t_end = int(tensor_range[0]), int(tensor_range[1])
    N.check(N.cuda().drc_cc_weights(C.byref(a), _stream()), "cc_weights")


def centered_clip_model_weights(layout: ArenaLayout, n: int, tau: float, partials: torch.Tensor, dist: torch.Tensor,
                                weights: torch.Tensor) -> None:
    """Model scope (``--rule-scope model``): fold ``centered_clip_dist``'s partials per tensor in tile order into ``dist``
    [T, n] fp64, sum them over the tensors in ascending order into the whole-model d_i, and write the one set of weights
    w_i = ``centered_clip_weight(d_i, tau, n)`` into every row of ``weights`` [T, n] (two kernels, csrc/cuda/clip.cu)."""
    _check_cc_rows("centered_clip_model_weights", n)
    if not (math.isfinite(tau) and tau > 0):
        raise ValueError(f"centered_clip_model_weights: tau must be finite and > 0, got {tau}")
    _check_buffer("centered_clip_model_weights: partials", partials, torch.float64, (layout.ntiles, n))
    _check_buffer("centered_clip_model_weights: dist", dist, torch.float64, (layout.ntensors, n))
    _check_buffer("centered_clip_model_weights: weights", weights, torch.float32, (layout.ntensors, n))
    a = N.CcArgs()
    a.n, a.tv = n, layout.tile_view(weights.device)
    a.partials, a.dist, a.weights, a.tau = partials.data_ptr(), dist.data_ptr(), weights.data_ptr(), float(tau)
    N.check(N.cuda().drc_cc_model_weights(C.byref(a), _stream()), "cc_model_weights")


def centered_clip_update(layout: ArenaLayout, grad_in: Addr, slot_stride: int, *, center: torch.Tensor, weights: torch.Tensor,
                         K: int, params: Addr, momentum: Addr, hp: Addr, step_ptr: Addr, done_counter: Addr,
                         select: Optional[torch.Tensor] = None, first_step: int = 1, grad_out: Addr = None,
                         mc_params: Addr = None, dst: Sequence[Addr] = (), flags: Sequence[Addr] = (), grid: Optional[int] = None,
                         tile_range: Optional[tuple] = None, exp_avg_sq: Addr = None, max_exp_avg_sq: Addr = None) -> None:
    """The fused update in mode 5 (csrc/cuda/aggregate_update.cu): g = v + sum_k w[t, k] (x_k - v) in fp32 over the K rows with
    a non-zero weight, stored back into ``center`` as the next step's v, then the optimizer step, broadcast and flags of
    ``aggregate_update``.  ``weights``: centered_clip_weights's fp32 [T, K]; ``select``: optional int32 [K, T] row table."""
    _check_cc_rows("centered_clip_update", K)
    if select is not None:
        _check_row_table(layout, select, K)
    _check_buffer("centered_clip_update: center", center, torch.float32, (layout.total,))
    _check_buffer("centered_clip_update: weights", weights, torch.float32, (layout.ntensors, K))
    a = N.UpdateArgs()
    a.mode, a.center = 5, center.data_ptr()
    _launch_update(a, layout, grad_in, slot_stride, select=select, K=K, scale=1.0, recomb=weights, params=params,
                   momentum=momentum, exp_avg_sq=exp_avg_sq, max_exp_avg_sq=max_exp_avg_sq, hp=hp, step_ptr=step_ptr,
                   first_step=first_step, grad_out=grad_out, mc_params=mc_params, dst=dst, done_counter=done_counter, flags=flags,
                   tile_range=tile_range, grid=grid)


# ------------------------------------------------------------------------------------------------ adaptive robust clipping
class ArcWorkspace:
    """ARC's scratch (csrc/cuda/arc.cu): the per-tile fp64 partials [ntiles, P], the fp32 factors [T, P] of the last clip and,
    with ``model``, the per-tensor fp64 d_i [T, P] the whole-model norm is summed from."""

    def __init__(self, layout: ArenaLayout, P: int, device, model: bool):
        _check_cc_rows("ArcWorkspace", P)
        self.partials = torch.zeros(layout.ntiles, P, dtype=torch.float64, device=device)
        self.factors = torch.ones(layout.ntensors, P, dtype=torch.float32, device=device)
        self.dist = torch.zeros(layout.ntensors, P, dtype=torch.float64, device=device) if model else None


def _arc_args(layout: ArenaLayout, P: int, k: int, ws: ArcWorkspace, grad_in: Addr = None) -> N.ArcArgs:
    _check_cc_rows("arc", P)
    if not 0 <= k < P:
        raise ValueError(f"arc: clips k in 0..P-1 of the P = {P} rows, got k = {k}")
    _check_buffer("arc: partials", ws.partials, torch.float64, (layout.ntiles, P))
    _check_buffer("arc: factors", ws.factors, torch.float32, (layout.ntensors, P))
    a = N.ArcArgs()
    a.grad_in, a.P, a.k, a.tv = addr(grad_in), P, k, layout.tile_view(ws.factors.device)
    a.partials, a.factors = ws.partials.data_ptr(), ws.factors.data_ptr()
    return a


def _tile_grid(layout: ArenaLayout, a: N.ArcArgs, tile_range: Optional[tuple], grid: Optional[int]) -> int:
    ntiles = layout.ntiles
    if tile_range is not None:
        a.tile_begin, a.tile_end = int(tile_range[0]), int(tile_range[1])
        ntiles = a.tile_end - a.tile_begin
    return grid or max(1, min(ntiles, sm_count() * 8))


def arc_norm(layout: ArenaLayout, grad_in: Addr, slot_stride: int, P: int, ws: ArcWorkspace, *,
             tile_range: Optional[tuple] = None, grid: Optional[int] = None) -> None:
    """ARC's squared norms: for every tile of ``tile_range`` (one bucket; None: the arena) and each of the P worker slots, the
    fp64 sum of (double)x^2 over the tile's real elements into ``ws.partials``."""
    a = _arc_args(layout, P, 0, ws, grad_in)
    a.slot_stride = slot_stride
    N.check(N.cuda().drc_arc_norm(C.byref(a), _tile_grid(layout, a, tile_range, grid), _stream()), "arc_norm")


def arc_factors(layout: ArenaLayout, P: int, k: int, ws: ArcWorkspace, *, tensor_range: Optional[tuple] = None) -> None:
    """Fold ``arc_norm``'s partials per tensor in tile order into d_i and write the factors of ``tensor_range`` (None: every
    tensor) into ``ws.factors`` (codes/oracle.py ``arc_row_factors``)."""
    a = _arc_args(layout, P, k, ws)
    if tensor_range is not None:
        a.t_begin, a.t_end = int(tensor_range[0]), int(tensor_range[1])
    N.check(N.cuda().drc_arc_factors(C.byref(a), _stream()), "arc_factors")


def arc_model_factors(layout: ArenaLayout, P: int, k: int, ws: ArcWorkspace) -> None:
    """``--arc model``: fold ``arc_norm``'s partials per tensor into ``ws.dist`` (clip.cu's cc_fold_kernel), sum them over the
    tensors in ascending order and write the one factor row into every row of ``ws.factors``.  Two kernels."""
    a = _arc_args(layout, P, k, ws)
    _check_buffer("arc: dist", ws.dist, torch.float64, (layout.ntensors, P))
    a.dist = ws.dist.data_ptr()
    f = N.CcArgs()
    f.n, f.tv, f.partials, f.dist = P, a.tv, ws.partials.data_ptr(), ws.dist.data_ptr()
    N.check(N.cuda().drc_cc_fold(C.byref(f), _stream()), "cc_fold")
    N.check(N.cuda().drc_arc_model_factors(C.byref(a), _stream()), "arc_model_factors")


def arc_scale(layout: ArenaLayout, grad_in: Addr, slot_stride: int, P: int, ws: ArcWorkspace, *,
              tile_range: Optional[tuple] = None, grid: Optional[int] = None) -> None:
    """Multiply in place, over the tiles of ``tile_range``, every slot row whose factor for the tile's tensor is below 1 (one
    fp32 multiply per real element; padding and the other rows are not touched)."""
    a = _arc_args(layout, P, 0, ws, grad_in)
    a.slot_stride = slot_stride
    N.check(N.cuda().drc_arc_scale(C.byref(a), _tile_grid(layout, a, tile_range, grid), _stream()), "arc_scale")


def arc_clip(layout: ArenaLayout, grad_in: Addr, slot_stride: int, P: int, k: int, ws: ArcWorkspace, *,
             tile_range: Optional[tuple] = None, tensor_range: Optional[tuple] = None, grid: Optional[int] = None) -> int:
    """Adaptive robust clipping of the P worker slots in place (codes/oracle.py ``arc``): the norms, the factors, the scale.
    Per tensor over one bucket (``tile_range`` / ``tensor_range``; None: the arena), or, when ``ws`` holds ``dist``, once over
    the whole model (no ranges).  The factors stay in ``ws.factors``.  Returns the kernels launched."""
    if ws.dist is not None and (tile_range is not None or tensor_range is not None):
        raise ValueError("arc_clip: the whole-model norm needs every tile, so it takes no bucket")
    arc_norm(layout, grad_in, slot_stride, P, ws, tile_range=tile_range, grid=grid)
    if ws.dist is not None:
        arc_model_factors(layout, P, k, ws)
    else:
        arc_factors(layout, P, k, ws, tensor_range=tensor_range)
    arc_scale(layout, grad_in, slot_stride, P, ws, tile_range=tile_range, grid=grid)
    return 4 if ws.dist is not None else 3


def stream_push(src: Addr, dst: Addr, nbytes: Addr, nbytes_out: Addr = None, *, step_ptr: Addr, done_counter: Addr, flag: Addr = None,
                grid: int = 16) -> None:
    """Store ``*nbytes`` bytes (device scalar) of a packed stream into a peer buffer and raise the step-stamped flag
    (compressed push of the fused transport, csrc/cuda/codec.cu)."""
    a = N.StreamPushArgs(addr(src), addr(dst), addr(nbytes), addr(nbytes_out), addr(step_ptr), addr(done_counter), addr(flag))
    lib = N.cuda()
    if not getattr(lib, "_stream_push_ready", False):
        lib.drc_stream_push.argtypes = [C.c_void_p, C.c_int, N.ptr]
        lib.drc_stream_push.restype = C.c_int
        lib._stream_push_ready = True
    N.check(lib.drc_stream_push(C.byref(a), int(grid), _stream()), "stream_push")


def cast_params(layout: ArenaLayout, src: Addr, dst: Addr) -> None:
    dev = torch.device("cuda", torch.cuda.current_device())
    a = N.CastArgs(addr(src), addr(dst), layout.tile_view(dev))
    N.check(N.cuda().drc_cast_params(C.byref(a), stream_grid(layout), _stream()), "cast_params")


# ------------------------------------------------------------------------------------------------ flags
def wait_flags(flags: Sequence[Addr], step_ptr: Addr, addend: int, error: Addr, timeout_s: float = 30.0,
               stamps: Addr = None) -> None:
    a = N.WaitArgs()
    a.stamps = addr(stamps)
    assert len(flags) <= N.MAX_WORKERS
    for i, f in enumerate(flags):
        a.flags[i] = addr(f)
    a.n = len(flags)
    a.step_ptr = addr(step_ptr)
    a.addend = addend
    a.timeout_ns = int(timeout_s * 1e9)
    a.error = addr(error)
    N.check(N.cuda().drc_wait_flags(C.byref(a), _stream()), "wait_flags")


def set_flags(flags: Sequence[Addr], step_ptr: Addr, addend: int) -> None:
    a = N.SetFlagArgs(_flag_list(flags), addr(step_ptr), addend)
    N.check(N.cuda().drc_set_flags(C.byref(a), _stream()), "set_flags")


def stamp(ring: Addr, step_ptr: Addr, col: int) -> None:
    """ring[(step & 63)][col] = %globaltimer (ring: int64 [64, 8])."""
    lib = N.cuda()
    if not getattr(lib, "_stamp_ready", False):
        lib.drc_stamp.argtypes = [N.ptr, N.ptr, C.c_int, N.ptr]
        lib.drc_stamp.restype = C.c_int
        lib._stamp_ready = True
    N.check(lib.drc_stamp(addr(ring), addr(step_ptr), int(col), _stream()), "stamp")


def step_add(step_ptr: Addr, delta: int = 1) -> None:
    N.check(N.cuda().drc_step_add(addr(step_ptr), delta, _stream()), "step_add")


# ------------------------------------------------------------------------------------------------ cyclic decode (K4)
_epart_cache = {}


def cyclic_project(layout: ArenaLayout, R: Addr, slot_stride: int, n: int, f: Addr, E: torch.Tensor) -> None:
    """E[T, n, 2] (fp64) = R_i . f per tensor: per-tile partials, then a fixed-order fold per tensor (deterministic)."""
    key = (E.device, layout.ntiles, n)
    if key not in _epart_cache:
        _epart_cache[key] = torch.empty(layout.ntiles, n, 2, dtype=torch.float64, device=E.device)
    a = N.ProjectArgs(addr(R), slot_stride, n, addr(f), layout.tile_view(E.device), E.data_ptr(), _epart_cache[key].data_ptr())
    N.check(N.cuda().drc_cyclic_project(C.byref(a), stream_grid(layout), _stream()), "cyclic_project")


def cyclic_locate(E: torch.Tensor, n: int, s: int, recomb: torch.Tensor, healthy: Optional[torch.Tensor] = None,
                  flagged: Optional[torch.Tensor] = None, rel_tol: float = 1e-4) -> None:
    a = N.LocateArgs(E.data_ptr(), E.shape[0], n, s, rel_tol, recomb.data_ptr(), addr(healthy), addr(flagged))
    N.check(N.cuda().drc_cyclic_locate(C.byref(a), _stream()), "cyclic_locate")


# ------------------------------------------------------------------------------------------------ robust baselines (K5/K6)
class GeoMedianWorkspace:
    def __init__(self, layout: ArenaLayout, P: int, device):
        T = layout.ntensors
        self.median = layout.new_arena(device)
        self.weights = torch.zeros(T, P, dtype=torch.float32, device=device)
        self.done = torch.zeros(T, dtype=torch.int32, device=device)
        self.dist2 = torch.zeros(T, P, dtype=torch.float64, device=device)
        self.move2 = torch.zeros(T, 2, dtype=torch.float64, device=device)


def geometric_median(layout: ArenaLayout, grad_in: Addr, slot_stride: int, P: int, ws: GeoMedianWorkspace,
                     iters: int = 64, eps: float = 1e-6) -> torch.Tensor:
    """Per-tensor Weiszfeld geometric median of the P slots; result in ``ws.median`` (fp32 arena)."""
    lib = N.cuda()
    T = layout.ntensors
    dev = ws.median.device
    tv = layout.tile_view(dev)
    grid = stream_grid(layout)
    for it in range(iters + 1):
        pa = N.GeoMedPrepArgs(T, P, ws.dist2.data_ptr(), ws.move2.data_ptr(), ws.weights.data_ptr(), ws.done.data_ptr(), it, eps)
        N.check(lib.drc_geomed_prep(C.byref(pa), _stream()), "geomed_prep")
        if it == iters:
            break
        ga = N.GeoMedArgs(addr(grad_in), slot_stride, P, tv, ws.median.data_ptr(), ws.weights.data_ptr(), ws.done.data_ptr(),
                          ws.dist2.data_ptr(), ws.move2.data_ptr())
        N.check(lib.drc_geomed_iter(C.byref(ga), grid, _stream()), "geomed_iter")
    return ws.median


GEOMED_FAST_MAXP = 16


def _pair_dist(layout: ArenaLayout, grad_in: Addr, slot_stride: int, P: int, pair_d2: torch.Tensor,
               rows: Optional[torch.Tensor]) -> None:
    """One pass over the slab: the squared distances between the P rows of every tensor, added into the zeroed fp64
    ``pair_d2`` [T, P(P-1)/2] (row i of tensor t is worker slot ``rows[i, t]``, or slot i without a table)."""
    pa = N.PairDistArgs(addr(grad_in), slot_stride, P, layout.tile_view(pair_d2.device), pair_d2.data_ptr(), addr(rows))
    N.check(N.cuda().drc_pair_dist(C.byref(pa), stream_grid(layout, 4), _stream()), "pair_dist")


def _check_pair_table(what: str, layout: ArenaLayout, P: int, pair_d2) -> None:
    if not 2 <= P <= GEOMED_FAST_MAXP:
        raise ValueError(f"{what}: takes 2..{GEOMED_FAST_MAXP} rows, got {P}")
    _check_buffer(f"{what}: pair_d2", pair_d2, torch.float64, (layout.ntensors, P * (P - 1) // 2))


def pair_dist(layout: ArenaLayout, grad_in: Addr, slot_stride: int, P: int, pair_d2: torch.Tensor,
              rows: Optional[torch.Tensor] = None) -> None:
    """The pair-distance pass alone (the one ``krum_select`` / ``bulyan_select`` / ``geometric_median_weights`` / ``nnm_mix``
    launch unless ``filled``): the squared distances between the P rows of every tensor, added into the zeroed fp64 ``pair_d2``
    [T, P(P-1)/2].  ``rows``: optional int32 [P, T] table, row i of tensor t is worker slot ``rows[i, t]``."""
    _check_pair_table("pair_dist", layout, P, pair_d2)
    if rows is not None:
        _check_row_table(layout, rows, P)
    _pair_dist(layout, grad_in, slot_stride, P, pair_d2, rows)


def pair_scope_fold(layout: ArenaLayout, P: int, pair_d2: torch.Tensor) -> None:
    """Model scope (``--rule-scope model``): replace every tensor's pair table by the model-level one, each pair's entries summed
    over the tensors in ascending order in fp64 (codes/oracle.py ``model_d2``; csrc/cuda/robust.cu).  The selection kernels
    then run with ``filled=True`` and make the same choice in every tensor; they zero the table as usual."""
    _check_pair_table("pair_scope_fold", layout, P, pair_d2)
    N.check(N.cuda().drc_pair_scope_fold(pair_d2.data_ptr(), layout.ntensors, P, _stream()), "pair_scope_fold")


def geometric_median_weights(layout: ArenaLayout, grad_in: Addr, slot_stride: int, P: int, pair_d2: torch.Tensor,
                             weights: torch.Tensor, max_iter: int = 256, eps: float = 1e-10,
                             iters_out: Optional[torch.Tensor] = None, rows: Optional[torch.Tensor] = None,
                             filled: bool = False) -> torch.Tensor:
    """Per-tensor geometric median as convex weights: ``median_t = sum_i weights[t, i] * slot_i`` (Weiszfeld run in weight
    space from the pairwise distances -- one pass over the slab; see csrc/cuda/robust.cu).  ``pair_d2``: zeroed fp64
    [T, P(P-1)/2] scratch (left zeroed); ``weights``: fp32 [T, P] out.  ``rows``: optional int32 [P, T] table, row i of tensor t
    is worker slot ``rows[i, t]`` (the weights stay in row space: pass the same table to ``aggregate_update(select=)``).
    ``filled``: ``pair_d2`` already holds the distances (``nnm_mix(mixed_out=True)``), so no pair-distance pass is launched."""
    assert P <= GEOMED_FAST_MAXP
    if rows is not None:
        _check_row_table(layout, rows, P)
    if not filled:
        _pair_dist(layout, grad_in, slot_stride, P, pair_d2, rows)
    wa = N.GeoMedWeightsArgs(pair_d2.data_ptr(), layout.ntensors, P, max_iter, eps, weights.data_ptr(),
                             iters_out.data_ptr() if iters_out is not None else None)
    N.check(N.cuda().drc_geomed_weights(C.byref(wa), _stream()), "geomed_weights")
    return weights


def krum_select(layout: ArenaLayout, grad_in: Addr, slot_stride: int, P: int, s: int, pair_d2: torch.Tensor,
                select: torch.Tensor, m: int = 1, rows: Optional[torch.Tensor] = None, filled: bool = False) -> None:
    """``pair_d2``: zeroed fp64 [T, P*(P-1)/2] scratch (left zeroed); ``select``: int32 [m, T] out, the ``m`` lowest Krum scores
    per tensor ordered by (score, slot) -- ``m = 1``: the Krum winner, ``m = P - s``: multi-Krum (int32 [T] is fine for m = 1).
    ``rows``: optional int32 [P, T] table, row i of tensor t is worker slot ``rows[i, t]``; ``select`` then holds worker slots.
    ``filled``: ``pair_d2`` already holds the distances (``nnm_mix(mixed_out=True)``), so no pair-distance pass is launched."""
    assert 1 <= m <= P and select.numel() >= m * layout.ntensors
    if rows is not None:
        _check_row_table(layout, rows, P)
    if not filled:
        _pair_dist(layout, grad_in, slot_stride, P, pair_d2, rows)
    ka = N.KrumSelectArgs(pair_d2.data_ptr(), layout.ntensors, P, s, m, select.data_ptr(), addr(rows))
    N.check(N.cuda().drc_krum_select(C.byref(ka), _stream()), "krum_select")


def bulyan_select(layout: ArenaLayout, grad_in: Addr, slot_stride: int, P: int, f: int, pair_d2: torch.Tensor,
                  select: torch.Tensor, rows: Optional[torch.Tensor] = None, filled: bool = False) -> None:
    """Bulyan's selection stage per tensor (``oracle.bulyan_indices``): theta = P - 2f rounds of Krum over the rows not chosen
    yet, for P >= 4f + 3 rows.  ``pair_d2``: zeroed fp64 [T, P*(P-1)/2] scratch (left zeroed); ``select``: int32 [theta, T] out,
    the worker slot chosen in round k at ``select[k, t]`` -- pass it to ``aggregate_update(K=theta, near_median=f, select=)``.
    ``rows``: optional int32 [P, T] table, row i of tensor t is worker slot ``rows[i, t]`` (DETOX: the vote's winner_slot).
    ``filled``: ``pair_d2`` already holds the distances (``nnm_mix(mixed_out=True)``), so no pair-distance pass is launched."""
    if not (f >= 0 and 4 * f + 3 <= P <= ROW_TABLE_MAXROWS):
        raise ValueError(f"bulyan_select: needs 4 * f + 3 <= P <= {ROW_TABLE_MAXROWS} (got P = {P}, f = {f})")
    _check_row_table(layout, select, P - 2 * f)
    if rows is not None:
        _check_row_table(layout, rows, P)
    if not filled:
        _pair_dist(layout, grad_in, slot_stride, P, pair_d2, rows)
    ba = N.BulyanSelectArgs(pair_d2.data_ptr(), layout.ntensors, P, f, select.data_ptr(), addr(rows))
    N.check(N.cuda().drc_bulyan_select(C.byref(ba), _stream()), "bulyan_select")


def nnm_mix(layout: ArenaLayout, grad_in: Addr, slot_stride: int, P: int, f: int, pair_d2: torch.Tensor, mix: torch.Tensor,
            mixed_out: bool) -> None:
    """Nearest-neighbour mixing per tensor (``oracle.nnm_neighbours`` / ``oracle.nnm_pair_d2``): the pair-distance pass over the
    P raw slots, then ``nnm_mix_kernel`` (csrc/cuda/robust.cu).  ``mix``: int32 [P, T] out, bit j of ``mix[i, t]`` = slot j is
    one of the n_mix = P - f rows row i is mixed from.  ``pair_d2``: zeroed fp64 [T, P*(P-1)/2] scratch.  ``mixed_out``: leave
    the mixed rows' distances in it for ``krum_select`` / ``bulyan_select`` / ``geometric_median_weights`` with ``filled=True``
    (which zero it); otherwise it is left zeroed."""
    if not (0 <= f < P <= ROW_TABLE_MAXROWS):
        raise ValueError(f"nnm_mix: needs 0 <= f < P <= {ROW_TABLE_MAXROWS} (got P = {P}, f = {f})")
    _check_row_table(layout, mix, P)
    _pair_dist(layout, grad_in, slot_stride, P, pair_d2, None)
    _nnm_mix_kernel(layout, P, f, pair_d2, mix, mixed_out)


def nnm_mix_table(layout: ArenaLayout, P: int, f: int, pair_d2: torch.Tensor, mix: torch.Tensor, mixed_out: bool) -> None:
    """``nnm_mix`` without its pair-distance pass: ``pair_d2`` already holds the raw rows' distances (``pair_dist``, then
    ``pair_scope_fold`` for one neighbourhood per worker over the whole model)."""
    if not (0 <= f < P <= ROW_TABLE_MAXROWS):
        raise ValueError(f"nnm_mix_table: needs 0 <= f < P <= {ROW_TABLE_MAXROWS} (got P = {P}, f = {f})")
    _check_row_table(layout, mix, P)
    _check_pair_table("nnm_mix_table", layout, P, pair_d2)
    _nnm_mix_kernel(layout, P, f, pair_d2, mix, mixed_out)


def _nnm_mix_kernel(layout, P, f, pair_d2, mix, mixed_out) -> None:
    na = N.NnmMixArgs(pair_d2.data_ptr(), layout.ntensors, P, f, mix.data_ptr(), int(bool(mixed_out)))
    N.check(N.cuda().drc_nnm_mix(C.byref(na), _stream()), "nnm_mix")


def nnm_fold(layout: ArenaLayout, P: int, f: int, mix: torch.Tensor, w_raw: torch.Tensor, *, select: Optional[torch.Tensor] = None,
             m: int = 1, w_mix: Optional[torch.Tensor] = None) -> None:
    """A choice over the mixed rows as fp32 weights over the raw slots: ``w_raw[t] = A_t^T w_mix[t] / (P - f)`` (fp64 sums),
    with w_mix = 1/m on the m mixed rows ``select[:m, t]`` names (Krum, multi-Krum) or the fp32 [T, P] ``w_mix`` (geometric
    median).  Pass ``w_raw`` to ``aggregate_update(K=P, scale=1, weights=w_raw)``."""
    T = layout.ntensors
    if not (0 <= f < P <= ROW_TABLE_MAXROWS):
        raise ValueError(f"nnm_fold: needs 0 <= f < P <= {ROW_TABLE_MAXROWS} (got P = {P}, f = {f})")
    _check_row_table(layout, mix, P)
    if (select is None) == (w_mix is None):
        raise ValueError("nnm_fold: pass exactly one of select= and w_mix=")
    if select is not None:
        if not 1 <= m <= P:
            raise ValueError(f"nnm_fold: needs 1 <= m <= P = {P} (got m = {m})")
        _check_row_table(layout, select, m)
    for name, w in (("w_mix", w_mix), ("w_raw", w_raw)):
        if w is not None and (w.dtype != torch.float32 or not w.is_cuda or not w.is_contiguous() or tuple(w.shape) != (T, P)):
            raise ValueError(f"nnm_fold: {name} must be a contiguous fp32 CUDA tensor of shape ({T}, {P})")
    fa = N.NnmFoldArgs(mix.data_ptr(), T, P, f, addr(select), m, addr(w_mix), w_raw.data_ptr())
    N.check(N.cuda().drc_nnm_fold(C.byref(fa), _stream()), "nnm_fold")


# ------------------------------------------------------------------------------------------------ GEMM (K10)
def gemm_bf16(A: torch.Tensor, B: torch.Tensor, *, a_mn: bool = False, b_mn: bool = False, out: Optional[torch.Tensor] = None,
              out_dtype: torch.dtype = torch.bfloat16, bias: Optional[torch.Tensor] = None, relu: bool = False,
              accumulate: bool = False, block_n: int = 0) -> torch.Tensor:
    """``C[M, N] = op(A) op(B)^T`` on the wgmma tensor cores (csrc/cuda/gemm_wgmma.cu).

    K-major operands (default) are ``A[M, K]`` / ``B[N, K]``; with ``a_mn`` / ``b_mn`` the tensor passed is the
    transposed storage ``A[K, M]`` / ``B[K, N]`` (MN contiguous), so no transpose copy is ever needed.
    ``block_n``: tile width, 0 = chosen by size, else 32 / 64 / 128.  256 is accepted and runs 128-wide tiles: one warpgroup's
    registers hold at most a 128 x 128 fp32 accumulator, so results are those of ``block_n=128``.
    """
    assert A.dtype == torch.bfloat16 and B.dtype == torch.bfloat16 and A.is_cuda and B.is_cuda
    assert A.dim() == 2 and B.dim() == 2 and A.stride(1) == 1 and B.stride(1) == 1
    M, K = (A.shape[1], A.shape[0]) if a_mn else (A.shape[0], A.shape[1])
    Nn, Kb = (B.shape[1], B.shape[0]) if b_mn else (B.shape[0], B.shape[1])
    assert K == Kb, f"K mismatch {K} vs {Kb}"
    if out is None:
        out = torch.empty(M, Nn, dtype=out_dtype, device=A.device)
    assert out.shape == (M, Nn) and out.stride(1) == 1
    bias_f32 = bias.data_ptr() if bias is not None and bias.dtype == torch.float32 else None
    bias_b16 = bias.data_ptr() if bias is not None and bias.dtype == torch.bfloat16 else None
    code = N.cuda().drc_gemm_bf16(A.data_ptr(), A.stride(0), int(a_mn), B.data_ptr(), B.stride(0), int(b_mn), out.data_ptr(),
                                  out.stride(0), int(out.dtype == torch.float32), M, Nn, K, bias_f32, bias_b16, int(relu),
                                  int(accumulate), block_n, sm_count(A.device), A.device.index, _stream())
    N.check(code, "gemm_bf16")
    return out


def gemm_supported(A: torch.Tensor, B: torch.Tensor) -> bool:
    """Shape/alignment gate of the TMA descriptors (16-byte rows and bases)."""
    return (A.is_cuda and A.dtype == torch.bfloat16 and B.dtype == torch.bfloat16 and A.stride(-1) == 1 and B.stride(-1) == 1
            and A.stride(0) % 8 == 0 and B.stride(0) % 8 == 0 and A.data_ptr() % 16 == 0 and B.data_ptr() % 16 == 0)
