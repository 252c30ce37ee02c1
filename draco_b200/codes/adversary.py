"""Simulated Byzantine workers: per-step schedule and attack models.

Schedule parity: the reference draws, with numpy's global RNG seeded to 428, ``max_steps+1``
samples of ``worker_fail`` distinct worker ranks out of ``1..P`` (src/util.py:100-103) and a
worker lies at step ``t`` iff ``rank in schedule[t]`` (src/worker/rep_worker.py:162).  We draw the
same stream from a private ``RandomState(428)`` so the *same ranks lie at the same steps*.

Attack parity (src/model_ops/utils.py:3-23), ``mag = -100``:
  rev_grad : replace  g -> mag*g           (cyclic: add, i.e. g + mag*g)
  constant : replace  g -> mag             (cyclic: g + mag)
  random   : reference is a no-op (TODO there).  Here it is a real attack: g -> sigma*N(0,1)
             (cyclic: g + sigma*N(0,1)) from a counter-based generator keyed by (seed, step, worker)
  omniscient (north-star extension): g -> -k * mean(honest gradients); needs a view of the honest
             gradients so it is applied by the engine, not by the per-worker hook.
  alie     : "A Little Is Enough" (Baruch, Baruch and Goldberg, NeurIPS 2019): mu - z * sigma
  minmax   : min-max (Shejwalkar and Houmansadr, NDSS 2021): mu - gamma * sigma with the largest gamma that keeps the row
             within the largest honest pairwise distance of every honest row
             (both per tensor, over the honest workers' pushed slots; applied by the PS, see ``alie_row`` / ``minmax_row``;
             ``--attack-scope model`` gives min-max one gamma and one Dmax over the whole model, ``minmax_gamma_model``)
  ipm      : inner-product manipulation (Xie, Koyejo and Gupta, UAI 2019): -eps * mu per coordinate (``ipm_row``)
  mimic    : (Karimireddy, He and Jaggi, ICLR 2022) every liar copies the honest slot that lies furthest along a direction z
             the PS learns during the first W steps (``mimic_z0`` / ``mimic_step``; whole model, stateful)

The device implementation of the same hook lives in csrc/cuda/push_encode.cu; the integer codes
below are shared with it.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from statistics import NormalDist
from typing import List, Optional, Tuple

import numpy as np

SEED = 428
ADVERSARY_MAG = -100.0     # reference: ADVERSARY_ / CONST_ in src/model_ops/utils.py:3-4

ATTACK_NONE = 0
ATTACK_REV_GRAD = 1
ATTACK_CONSTANT = 2
ATTACK_RANDOM = 3
ATTACK_OMNISCIENT = 4
ATTACK_ALIE = 5
ATTACK_MINMAX = 6
ATTACK_IPM = 7
ATTACK_MIMIC = 8
# built by the PS from the honest slots; the liars push their true gradient
PS_ATTACKS = ("alie", "minmax", "ipm", "mimic")
IPM_EPS = 0.1             # --attack-eps default: this repository's choice (the paper evaluates several eps)
MIMIC_WARMUP = 20         # --mimic-warmup default: this repository's choice (steps of the online power iteration)

_ATTACK_CODES = {
    "none": ATTACK_NONE,
    "rev_grad": ATTACK_REV_GRAD,
    "constant": ATTACK_CONSTANT,
    "random": ATTACK_RANDOM,
    "omniscient": ATTACK_OMNISCIENT,
    "alie": ATTACK_ALIE,
    "minmax": ATTACK_MINMAX,
    "ipm": ATTACK_IPM,
    "mimic": ATTACK_MIMIC,
}


def attack_code(name: str) -> int:
    try:
        return _ATTACK_CODES[name]
    except KeyError:
        raise ValueError(f"unknown --err-mode {name!r}; choose from {sorted(_ATTACK_CODES)}") from None


@dataclass(frozen=True)
class AdversarySchedule:
    """``ranks[t]`` = sorted worker ranks (1-based) that lie at step ``t`` (t = 0..max_steps)."""

    num_workers: int
    worker_fail: int
    ranks: List[np.ndarray]

    def is_adversary(self, rank: int, step: int) -> bool:
        return bool(np.any(self.ranks[step % len(self.ranks)] == rank))

    def bitmaps(self) -> np.ndarray:
        """uint32 bitmap per step: bit ``w-1`` set iff worker ``w`` lies (consumed on device)."""
        out = np.zeros(len(self.ranks), dtype=np.uint32)
        for t, r in enumerate(self.ranks):
            for w in r:
                out[t] |= np.uint32(1) << np.uint32(int(w) - 1)
        return out


def generate_schedule(num_workers: int, worker_fail: int, max_steps: int, seed: int = SEED) -> AdversarySchedule:
    if worker_fail > num_workers:
        raise ValueError("more adversaries than workers")
    if num_workers > 32:
        raise ValueError("adversary bitmaps are 32-bit: at most 32 workers")
    rng = np.random.RandomState(seed)
    pool = np.arange(1, num_workers + 1)
    ranks = [np.sort(rng.choice(pool, size=worker_fail, replace=False)) for _ in range(max_steps + 1)]
    return AdversarySchedule(num_workers, worker_fail, ranks)


def _philox_like_normal(shape, seed: int, step: int, worker: int) -> np.ndarray:
    rng = np.random.Generator(np.random.Philox(key=[(seed << 32) ^ (step & 0xFFFFFFFF), worker]))
    return rng.standard_normal(shape)


def err_simulation(grad: np.ndarray, mode: str, cyclic: bool = False, *, magnitude: float = ADVERSARY_MAG,
                   seed: int = SEED, step: int = 0, worker: int = 0,
                   honest_mean: Optional[np.ndarray] = None) -> np.ndarray:
    """Host oracle of the adversary hook (same name as the reference's function)."""
    g = np.asarray(grad)
    if mode in ("none", None):
        return g
    if mode == "rev_grad":
        adv = magnitude * g
    elif mode == "constant":
        adv = np.full(g.shape, magnitude, dtype=g.dtype if np.iscomplexobj(g) else np.float64)
    elif mode == "random":
        adv = abs(magnitude) * _philox_like_normal(g.shape, seed, step, worker)
    elif mode == "omniscient":
        if honest_mean is None:
            raise ValueError("omniscient attack needs the honest mean")
        adv = magnitude * np.asarray(honest_mean)
    else:
        raise ValueError(f"unknown err mode {mode!r}")
    if cyclic:
        return g + adv
    return adv if np.iscomplexobj(g) else adv.astype(g.dtype, copy=False)


# ------------------------------------------------------------------------------------------------ PS-side attacks (fp64 oracle)
def alie_s(num_workers: int, worker_fail: int) -> int:
    """Baruch et al.'s s = floor(P/2 + 1) - f: honest workers the liars need on their side for a majority."""
    return num_workers // 2 + 1 - worker_fail


def alie_z_max(num_workers: int, worker_fail: int) -> float:
    """z_max = Phi^-1((P - s) / P); undefined (ValueError) when s < 1."""
    s = alie_s(num_workers, worker_fail)
    if s < 1:
        raise ValueError(f"ALIE's z_max is undefined for {num_workers} workers and {worker_fail} liars (s = {s} < 1)")
    return NormalDist().inv_cdf((num_workers - s) / num_workers)


def honest_stats(H: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
    """Per-coordinate mean and population standard deviation (ddof 0) of the honest rows ``H`` [n_h, d], in fp64."""
    H = np.asarray(H, dtype=np.float64)
    with np.errstate(invalid="ignore", over="ignore"):            # +-Inf rows: NaN sigma, as on the device
        mu = H.sum(0) / H.shape[0]
        return mu, np.sqrt(((H - mu) ** 2).sum(0) / H.shape[0])


def alie_row(H: np.ndarray, z: float) -> np.ndarray:
    """The row every ALIE liar sends for one tensor: mu - z * sigma (fp64)."""
    mu, sd = honest_stats(H)
    with np.errstate(invalid="ignore"):
        return mu - z * sd


def minmax_gamma(H: np.ndarray) -> float:
    """Largest gamma with max_i ||mu + gamma p - g_i|| <= Dmax = max_{i<j} ||g_i - g_j|| over the honest rows, p = -sigma.

    Each constraint is c g^2 + 2 b_i g + (a_i - Dmax^2) <= 0 with a_i = ||mu - g_i||^2, b_i = <mu - g_i, p>, c = ||p||^2; its
    largest root is (-b_i + sqrt(b_i^2 - c (a_i - Dmax^2))) / c, written as (Dmax^2 - a_i) / (b_i + sqrt(.)) when b_i > 0
    (the same number without cancellation).  a_i <= Dmax^2 because mu lies in the honest hull, so every root is real and
    >= 0; the clamps only absorb rounding.  c == 0 (all honest rows equal): gamma = 0.  NaN in, NaN out."""
    return minmax_solve(minmax_terms(H))


def minmax_terms(H: np.ndarray) -> np.ndarray:
    """The fp64 sums gamma depends on, in the device's order: a_i (i < n), b_i, c, then the squared distance of every honest
    pair (i < j) at 2n + 1 + j(j-1)/2 + i.  Over the whole model each is the sum of the per-tensor ones (``minmax_gamma_model``)."""
    H = np.asarray(H, dtype=np.float64)
    n = H.shape[0]
    mu, sd = honest_stats(H)
    with np.errstate(invalid="ignore", over="ignore"):
        p = -sd
        E = mu[None, :] - H
        a = (E * E).sum(1)
        b = (E * p[None, :]).sum(1)
        c = float((p * p).sum())
        d2 = [float(((H[i] - H[j]) ** 2).sum()) for j in range(1, n) for i in range(j)]
    return np.concatenate([a, b, [c], d2])


def minmax_solve(terms: np.ndarray) -> float:
    """gamma from ``minmax_terms`` (see ``minmax_gamma``)."""
    terms = np.asarray(terms, dtype=np.float64)
    n = int(round((-3 + math.sqrt(9 + 8 * (len(terms) - 1))) / 2))        # len = 2n + 1 + n(n-1)/2
    a, b, c, d2 = terms[:n], terms[n:2 * n], float(terms[2 * n]), [float(x) for x in terms[2 * n + 1:]]
    with np.errstate(invalid="ignore", over="ignore"):
        D2 = max(d2, key=lambda x: (math.isnan(x), x)) if d2 else 0.0
        if c == 0.0:
            return 0.0
        roots = []
        for ai, bi in zip(a, b):
            disc = bi * bi + c * (D2 - ai)
            disc = 0.0 if disc < 0.0 else disc
            r = math.sqrt(disc) if not math.isnan(disc) else math.nan
            g = (r - bi) / c if bi <= 0.0 else (D2 - ai) / (bi + r)
            roots.append(0.0 if g < 0.0 else g)
    return math.nan if any(math.isnan(g) for g in roots) else min(roots)


def minmax_gamma_model(parts) -> float:
    """Min-max over the whole model (``--attack-scope model``, as in Shejwalkar and Houmansadr's paper): one gamma and one Dmax
    for the concatenation of the honest rows' tensors ``parts`` (a list of [n_h, numel_t]).  Every term of ``minmax_terms`` is
    the fp64 sum, in ascending tensor order, of the per-tensor terms (``oracle.model_d2``), as the fused solve forms it; up to
    rounding this is ``minmax_gamma`` of the concatenated rows."""
    from .oracle import model_d2
    return minmax_solve(model_d2([minmax_terms(H) for H in parts]))


def minmax_row(H: np.ndarray) -> np.ndarray:
    """The row every min-max liar sends for one tensor: mu + gamma * p = mu - gamma * sigma (fp64)."""
    mu, sd = honest_stats(H)
    with np.errstate(invalid="ignore"):
        return mu - minmax_gamma(H) * sd


def ipm_row(H: np.ndarray, eps: float) -> np.ndarray:
    """The row every IPM liar sends for one tensor: -eps * mu, mu the fp64 honest mean summed in slot order and divided once
    (ALIE's mu), in fp64; the slot gets it rounded to fp32 once."""
    H = np.asarray(H, dtype=np.float64)
    acc = np.zeros(H.shape[1:], dtype=np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        for h in H:
            acc = acc + h
        return -eps * (acc / H.shape[0])


def mimic_z0(spans, total: int, seed: int = SEED) -> np.ndarray:
    """Mimic's starting direction, fp32 [total]: standard normals on the valid coordinates (one Philox stream keyed by the
    adversary seed, laid out over the spans in ascending order, 0 on padding), divided by their norm -- per-tensor fp64 sums
    of squares added in ascending tensor order (``oracle.model_d2``), one sqrt -- and rounded to fp32 once."""
    from .oracle import model_d2
    n = sum(int(numel) for _, numel in spans)
    g = np.random.Generator(np.random.Philox(key=seed)).standard_normal(n)
    x = np.zeros(total, dtype=np.float64)
    at = 0
    for off, numel in spans:
        x[off:off + numel] = g[at:at + numel]
        at += numel
    nrm = math.sqrt(float(model_d2([[float((x[o:o + k] ** 2).sum())] for o, k in spans])[0]))
    return (x / nrm).astype(np.float32)


@dataclass
class MimicState:
    """Mimic's PS state: ``m`` the running mean of the honest means (+0 at the start) and ``z`` the unit direction, both fp32
    [D] and 0 on padding."""
    m: np.ndarray
    z: np.ndarray


def _model_dot(a: np.ndarray, b: np.ndarray, spans) -> float:
    """<a, b> over the spans: each tensor's fp64 sum, added in ascending tensor order (``oracle.model_d2``)."""
    from .oracle import model_d2
    with np.errstate(invalid="ignore", over="ignore"):
        per = [[float((a[o:o + k].astype(np.float64) * b[o:o + k].astype(np.float64)).sum())] for o, k in spans]
    return float(model_d2(per)[0])


def mimic_step(slots: np.ndarray, liars, spans, state: MimicState, t: int, W: int):
    """One PS step of the mimic attack (the definition the fused kernels and the library path share).

    With H the honest slots in ascending order, n = |H|, and every whole-model sum the per-tensor fp64 sums added in ascending
    tensor order:

    1. s_i = <x_i, z> for i in H;
    2. k = the first i in H with the largest s_i (``np.argmax``: a NaN counts as the largest, ties go to the lower slot);
    3. every liar slot becomes a bit copy of x_k on the spans (padding is never written);
    4. only while t < W (t = step - 1, the warm-up index): c = (sum_{i in H} x_i) / n in fp64; m = fp32((t m + c) / (t + 1));
       w_i = s_i - <m, z> (the new m; equal to <x_i - m, z> up to rounding, the form the kernels use);
       u = t z + sum_{i in H} w_i (x_i - m) in fp64 without contraction; z = fp32(u / ||u||), unchanged when ||u|| = 0.
       Steps 1-3 use the z from before the update.

    Returns (the new slots, k, the new ``MimicState``).  ``slots`` [P, D] fp32; ``liars`` 0-based."""
    out = np.array(slots, copy=True)
    liars = sorted(set(int(w) for w in liars))
    honest = [w for w in range(out.shape[0]) if w not in liars]
    m, z = state.m.copy(), state.z.copy()
    if not honest:
        return out, -1, MimicState(m, z)
    s = np.array([_model_dot(slots[i], z, spans) for i in honest])
    k = honest[int(np.argmax(s))]
    for off, numel in spans:
        out[liars, off:off + numel] = slots[k, off:off + numel]
    if t < W:
        n = len(honest)
        with np.errstate(invalid="ignore", over="ignore"):
            for off, numel in spans:
                sl = slice(off, off + numel)
                c = np.zeros(numel, dtype=np.float64)
                for i in honest:
                    c = c + slots[i, sl].astype(np.float64)
                m[sl] = ((t * m[sl].astype(np.float64) + c / n) / (t + 1)).astype(np.float32)
            mz = _model_dot(m, z, spans)
            w = [float(si) - mz for si in s]
            u = np.zeros(out.shape[1], dtype=np.float64)
            for off, numel in spans:
                sl = slice(off, off + numel)
                acc = t * z[sl].astype(np.float64)
                for wi, i in zip(w, honest):
                    acc = acc + wi * (slots[i, sl].astype(np.float64) - m[sl].astype(np.float64))
                u[sl] = acc
            nrm = math.sqrt(_model_dot(u, u, spans))
            if nrm != 0.0:
                for off, numel in spans:
                    z[off:off + numel] = (u[off:off + numel] / nrm).astype(np.float32)
    return out, k, MimicState(m, z)


def ps_attack(slots: np.ndarray, liars, mode: str, spans, z: Optional[float] = None, scope: str = "tensor") -> np.ndarray:
    """Oracle of the whole PS-side step: ``slots`` [P, D] with the liar slots (0-based) replaced, per tensor span
    ``(offset, numel)``, by the attack row built from the honest slots (fp64, rounded to the slots' dtype).  Padding outside
    the spans is left alone.  ``scope="model"`` (min-max only): one gamma over every span (``minmax_gamma_model``).  ``z`` is
    ALIE's z or IPM's eps; mimic has state and its own ``mimic_step``."""
    out = np.array(slots, copy=True)
    liars = sorted(set(int(w) for w in liars))
    honest = [w for w in range(out.shape[0]) if w not in liars]
    if not liars or not honest:
        return out
    parts = [np.asarray(slots[honest, off:off + numel], dtype=np.float64) for off, numel in spans]
    gamma = minmax_gamma_model(parts) if scope == "model" and mode == "minmax" else None
    for (off, numel), H in zip(spans, parts):
        if gamma is not None:
            mu, sd = honest_stats(H)
            with np.errstate(invalid="ignore"):
                row = mu - gamma * sd
        elif mode == "ipm":
            row = ipm_row(H, z)
        else:
            row = alie_row(H, z) if mode == "alie" else minmax_row(H)
        with np.errstate(over="ignore", invalid="ignore"):
            out[liars, off:off + numel] = row.astype(out.dtype)
    return out
