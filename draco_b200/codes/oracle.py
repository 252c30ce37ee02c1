"""fp64 numpy oracles for every PS-side aggregation rule.

They define the semantics the CUDA kernels (csrc/cuda/*.cu) and the C++ host twins
(csrc/host/*.cpp) are tested against, tensor by tensor -- the reference applies every rule
*per parameter tensor*, never on the concatenated model (src/master/rep_master.py:154-168,
src/master/baseline_master.py:271-296).

Every rule that measures distances also has a model scope (``--rule-scope model``, ``model_scope``): the same oracle on the
rows formed by concatenating every tensor, as the papers define it.  ``model_d2`` restates how the kernels form those
distances.

``worker_momentum`` is the one worker-side rule here, and it is fp32 on purpose: every path must produce its exact bits.
``centered_clip`` is fp64 where it measures (the distances, the weights) and fp32 where it combines rows, for the same reason.
``sign_pack`` / ``sign_vote`` (signSGD with majority vote) are exact integer arithmetic on the signs of fp32 values.
``arc`` (adaptive robust clipping, a pre-aggregation step on the raw worker slots) measures in fp64 and scales with one fp32
multiply per element.
"""
from __future__ import annotations

import math
from typing import List, Sequence, Tuple

import numpy as np

from ..rules import arc_k  # noqa: F401  (ARC's k, with its semantics below)


def boyer_moore_winner(members: Sequence[np.ndarray]) -> int:
    """Index of the Boyer-Moore candidate using whole-tensor equality (``np.array_equal``).

    Mirrors the reference's streaming vote (rep_master.py:157-165) including its behaviour when no
    strict majority exists (the last surviving candidate wins).
    """
    cand, count = 0, 0
    for i, m in enumerate(members):
        if count == 0:
            cand, count = i, 1
        elif np.array_equal(m, members[cand]):
            count += 1
        else:
            count -= 1
    return cand


def majority_vote(slots: np.ndarray, groups: Sequence[Sequence[int]]) -> Tuple[np.ndarray, List[int]]:
    """``slots``: [P, d] one tensor from every worker (row w-1 = worker w).  Returns (mean of group
    winners, winner member index per group)."""
    acc = np.zeros(slots.shape[1], dtype=np.float64)
    winners = []
    for g in groups:
        members = [slots[w - 1] for w in g]
        k = boyer_moore_winner(members)
        winners.append(k)
        acc += members[k]
    return acc / float(len(groups)), winners


def mean(slots: np.ndarray) -> np.ndarray:
    return np.asarray(slots, dtype=np.float64).mean(axis=0)


def geometric_median(slots: np.ndarray, eps: float = 1e-8, max_iter: int = 200) -> np.ndarray:
    """Weiszfeld iteration started at the mean (what hdmedians.geomedian does; baseline_master.py:274)."""
    X = np.asarray(slots, dtype=np.float64)
    m = X.mean(axis=0)
    for _ in range(max_iter):
        d = np.linalg.norm(X - m, axis=1)
        nz = d > 1e-300
        if not nz.any():
            return m
        w = np.zeros_like(d)
        w[nz] = 1.0 / d[nz]
        m_new = (w[:, None] * X).sum(axis=0) / w.sum()
        if np.linalg.norm(m_new - m) <= eps * max(1.0, np.linalg.norm(m)):
            return m_new
        m = m_new
    return m


def geometric_median_weights(slots: np.ndarray, eps: float = 1e-10, max_iter: int = 256) -> np.ndarray:
    """The same Weiszfeld iteration carried out on the convex weights only (host model of ``geomed_weights_kernel``,
    csrc/cuda/robust.cu).  Every iterate is ``m = w @ X`` with ``sum(w) = 1``, for which
    ``||x_i - m||^2 = (D w)_i - w^T D w / 2`` with ``D_ij = ||x_i - x_j||^2`` -- the data is touched once (for D)."""
    X = np.asarray(slots, dtype=np.float64)
    return _weiszfeld_weights(((X[:, None, :] - X[None, :, :]) ** 2).sum(axis=2), eps, max_iter)


def _weiszfeld_weights(D: np.ndarray, eps: float, max_iter: int) -> np.ndarray:
    P = D.shape[0]
    w = np.full(P, 1.0 / P)
    if D.max() <= 0:
        return w
    floor_d = 1e-12 * np.sqrt(D.max()) + 1e-300
    for _ in range(max_iter):
        s = D @ w
        d = np.maximum(np.sqrt(np.maximum(s - 0.5 * (w @ s), 0.0)), floor_d)
        wn = (1.0 / d) / (1.0 / d).sum()
        delta = np.abs(wn - w).max()
        w = wn
        if delta <= eps:
            break
    return w


def krum_index(slots: np.ndarray, s: int) -> int:
    """Krum (arXiv:1703.02757) as the reference implements it (baseline_master.py:278-296):
    score_i = sum of the (P - s - 2) smallest squared distances to the others; argmin wins (the lowest index on ties, and
    NaN scores -- a row that sent NaN -- rank last, like every sort here)."""
    return int(np.argsort(krum_scores(slots, s), kind="stable")[0])


def krum(slots: np.ndarray, s: int) -> np.ndarray:
    return np.asarray(slots, dtype=np.float64)[krum_index(slots, s)]


def krum_scores(slots: np.ndarray, s: int) -> np.ndarray:
    """score_i of ``krum_index``: the sum of the (P - s - 2) smallest squared distances from row i to the others (NaN
    distances sort last)."""
    X = np.asarray(slots, dtype=np.float64)
    return _krum_scores_d2(((X[:, None, :] - X[None, :, :]) ** 2).sum(axis=2), s)


def _krum_scores_d2(d2: np.ndarray, s: int) -> np.ndarray:
    P = d2.shape[0]
    keep = max(P - s - 2, 0)
    return np.array([np.sort(np.delete(d2[i], i))[:keep].sum() for i in range(P)])


def multi_krum_indices(slots: np.ndarray, s: int, m: int) -> List[int]:
    """Multi-Krum (Blanchard et al., NeurIPS 2017): the ``m`` rows with the lowest Krum scores, ordered by (score, index).
    ``m = 1`` is ``[krum_index(slots, s)]``; the trainer averages ``m = P - s`` rows."""
    return [int(i) for i in np.argsort(krum_scores(slots, s), kind="stable")[:m]]


def multi_krum(slots: np.ndarray, s: int, m: int) -> np.ndarray:
    return np.asarray(slots, dtype=np.float64)[multi_krum_indices(slots, s, m)].mean(axis=0)


def trimmed_mean(slots: np.ndarray, b: int) -> np.ndarray:
    """Coordinate-wise b-trimmed mean (Yin et al., ICML 2018): per coordinate, sort the P values ascending, drop ``b`` at each
    end and average the remaining P - 2b.  The order is -Inf < finite < +Inf < NaN (``np.sort``), so at most ``b`` non-finite
    values in a coordinate are always dropped."""
    X = np.asarray(slots, dtype=np.float64)
    P = X.shape[0]
    if not 0 <= 2 * b < P:
        raise ValueError(f"trim {b} leaves nothing of {P} rows")
    return np.sort(X, axis=0)[b:P - b].mean(axis=0)


def coordinate_median(slots: np.ndarray) -> np.ndarray:
    """Coordinate-wise median: the trimmed mean with b = (P - 1) // 2 -- the middle value for odd P, the mean of the two
    middle values for even P (``np.median``; not ``torch.median``, which returns the lower one)."""
    return trimmed_mean(slots, (np.asarray(slots).shape[0] - 1) // 2)


def bulyan_indices(slots: np.ndarray, f: int) -> List[int]:
    """Bulyan's selection stage (El Mhamdi, Guerraoui and Rouault, *The Hidden Vulnerability of Distributed Learning in
    Byzantium*, ICML 2018) with A = Krum, for n = P >= 4f + 3 rows: S = {A(R_1), ..., A(R_theta)}, theta = n - 2f, where R_1
    is all rows and R_{k+1} = R_k minus the row A(R_k) picked.  Each round scores every row i of R as Krum does over R
    (``krum_scores``: the sum of the keep = max(|R| - f - 2, 0) smallest squared distances from i to the other rows of R, NaN
    distances last, a sum of zero terms is 0) and moves the lowest-scoring row out of R into S (NaN scores last, ties to the
    lower row index).  Returns the row chosen in each round, in round order.

    keep = |R| - f - 2 is the paper's recursion as written: R shrinks by one per round, so keep falls by one per round too.  In
    the last round |R| = 2f + 1 and keep = f - 1, which is 0 for f <= 1: every score is then 0 and the lowest remaining row
    index wins.  That is kept as written rather than patched."""
    X = np.asarray(slots, dtype=np.float64)
    P = X.shape[0]
    if not (f >= 0 and P >= 4 * f + 3):
        raise ValueError(f"Bulyan needs P >= 4f + 3 rows (got P = {P}, f = {f})")
    with np.errstate(invalid="ignore", over="ignore"):                # Inf - Inf: a NaN distance, which sorts last
        d2 = ((X[:, None, :] - X[None, :, :]) ** 2).sum(axis=2)
    return _bulyan_rounds(d2, f)


def _bulyan_rounds(d2: np.ndarray, f: int) -> List[int]:
    P = d2.shape[0]
    R, chosen = list(range(P)), []
    for _ in range(P - 2 * f):
        keep = max(len(R) - f - 2, 0)
        scores = np.array([np.sort(d2[i, [j for j in R if j != i]])[:keep].sum() for i in R])
        chosen.append(R.pop(int(np.argsort(scores, kind="stable")[0])))
    return chosen


def nearest_to_median_mean(slots: np.ndarray, b: int) -> np.ndarray:
    """Bulyan's coordinate stage (El Mhamdi et al., ICML 2018): with beta = theta - 2f, coordinate i of the result is
    (1 / beta) sum_{x in M_i} x, M_i = argmin_{|M| = beta} sum_{x in M} |x - median_i| over the theta selected values -- the beta
    values closest to the coordinate median.  Here over the theta rows of ``slots``, with b = f.  Per coordinate:

    * sort the theta values, -Inf < finite < +Inf < NaN (``np.sort``);
    * m = the median: the middle value for odd theta, 0.5 a + 0.5 b of the two middle values for even theta;
    * keep beta = theta - 2b values nearest to m (distance |v - m|, a NaN distance the farthest; a tie in distance keeps the
      smaller value).  They form a window [s, s + beta) of the sorted order with 0 <= s <= 2b: starting from s = 0 the window
      moves right while the value entering it is strictly nearer to m than the value leaving it, or equal to it;
    * average the kept values.

    This is not the b-trimmed mean, which keeps the middle window s = b whatever the distances."""
    S = np.sort(np.asarray(slots, dtype=np.float64), axis=0)
    theta = S.shape[0]
    if not 0 <= 2 * b < theta:
        raise ValueError(f"f = {b} leaves nothing of {theta} rows")
    beta = theta - 2 * b
    lo, hi = S[(theta - 1) // 2], S[theta // 2]
    m = lo if theta % 2 else 0.5 * lo + 0.5 * hi
    s = np.zeros(S.shape[1:], dtype=np.int64)
    moving = np.ones(S.shape[1:], dtype=bool)
    with np.errstate(invalid="ignore"):
        for j in range(2 * b):
            vin, vout = S[j + beta], S[j]
            din, dout = np.abs(vin - m), np.abs(vout - m)
            nearer = (din < dout) | (np.isnan(dout) & ~np.isnan(din))
            same = (vin == vout) | (np.isnan(vin) & np.isnan(vout))
            moving &= nearer | same
            s += moving
    win = np.arange(theta).reshape((theta,) + (1,) * (S.ndim - 1))
    keep = (win >= s) & (win < s + beta)
    return np.where(keep, S, 0.0).sum(axis=0) / beta


def bulyan(slots: np.ndarray, f: int) -> np.ndarray:
    """Bulyan with Krum (El Mhamdi, Guerraoui and Rouault, ICML 2018) on one tensor of P >= 4f + 3 rows:
    ``nearest_to_median_mean`` over the theta = P - 2f rows ``bulyan_indices`` selects.  With f = 0 it is the mean of all rows."""
    X = np.asarray(slots, dtype=np.float64)
    return nearest_to_median_mean(X[bulyan_indices(X, f)], f)


NNM_MODES = ("coordinate_median", "trimmed_mean", "krum", "multi_krum", "geometric_median", "bulyan")


def _raw_d2(slots: np.ndarray) -> np.ndarray:
    """Squared distances between the rows, in fp64 from the (fp32) inputs; the diagonal is 0."""
    X = np.asarray(slots, dtype=np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        D = ((X[:, None, :] - X[None, :, :]) ** 2).sum(axis=2)
    np.fill_diagonal(D, 0.0)
    return D


def nnm_neighbours_d2(D: np.ndarray, f: int) -> np.ndarray:
    """``nnm_neighbours`` from a table of squared distances ``D`` [P, P] (only its off-diagonal entries are read)."""
    D = np.asarray(D, dtype=np.float64)
    P = D.shape[0]
    if not 0 <= f < P:
        raise ValueError(f"nearest-neighbour mixing needs 0 <= f < P (got P = {P}, f = {f})")
    A = np.zeros((P, P), dtype=np.int64)
    for i in range(P):
        others = np.array([j for j in range(P) if j != i], dtype=np.int64)
        order = others[np.argsort(D[i, others], kind="stable")]      # ascending, NaN last, ties to the lower row
        A[i, i] = 1
        A[i, order[:P - f - 1]] = 1
    return A


def nnm_neighbours(slots: np.ndarray, f: int) -> np.ndarray:
    """Nearest-neighbour mixing (NNM; Allouah, Farhadkhani, Guerraoui, Gupta, Pinot and Stephan, *Fixing by Mixing: A Recipe
    for Optimal Byzantine ML under Heterogeneity*, AISTATS 2023), the neighbourhoods: with n_mix = P - f, N_i is row i itself
    plus the n_mix - 1 rows nearest to it among the others, by squared distance in fp64 from the inputs, ascending, NaN last,
    ties to the lower row index.  Row i is its own first neighbour even when another row duplicates it.  Returns the P x P 0/1
    matrix A with A[i, j] = 1 iff j is in N_i."""
    return nnm_neighbours_d2(_raw_d2(slots), f)


def nnm_mix(slots: np.ndarray, f: int) -> np.ndarray:
    """The mixed rows y_i = (1 / n_mix) sum over j in N_i of x_j (``nnm_neighbours``), in fp64."""
    X = np.asarray(slots, dtype=np.float64)
    return _mix_rows(X, nnm_neighbours(X, f), f)


def _mix_rows(X: np.ndarray, A: np.ndarray, f: int) -> np.ndarray:
    """Row i: the sum of the rows in N_i over n_mix (not ``A @ X``, where 0 * NaN would reach the rows that do not take it)."""
    return np.stack([X[np.flatnonzero(a)].sum(axis=0) for a in A]) / (X.shape[0] - f)


def nnm_pair_d2(D: np.ndarray, A: np.ndarray, f: int) -> np.ndarray:
    """Squared distances between the mixed rows from the raw table ``D`` alone, with no pass over the data: with
    c = (A[i] - A[k]) / n_mix (which sums to 0), ||y_i - y_k||^2 = -1/2 c^T D c, in fp64 and clamped at 0.  The sum runs over
    the rows of N_i and N_k and D's diagonal counts as 0, so a NaN distance between any two of those rows makes the result NaN
    (as it would be for the mixed rows themselves), and the clamp keeps a NaN a NaN."""
    D = np.array(D, dtype=np.float64)
    np.fill_diagonal(D, 0.0)
    A = np.asarray(A, dtype=np.float64)
    P, n = A.shape[0], A.shape[0] - f
    out = np.zeros((P, P))
    for i in range(P):
        for k in range(P):
            if i == k:
                continue
            u = np.flatnonzero(A[i] + A[k])
            c = (A[i, u] - A[k, u]) / n
            v = -0.5 * (c @ D[np.ix_(u, u)] @ c)
            out[i, k] = v if not v < 0.0 else 0.0
    return out


def nnm(slots: np.ndarray, f: int, mode: str) -> np.ndarray:
    """NNM, then the robust rule ``mode`` on the mixed rows (``nnm_mix``), per tensor.  The rules that use distances (Krum,
    multi-Krum, Bulyan's selection, the geometric median's Weiszfeld in weight space) take them from ``nnm_pair_d2``:

    * ``coordinate_median``; * ``trimmed_mean``: trim f;  * ``krum``: s = f;  * ``multi_krum``: s = f, averaging P - f rows;
    * ``geometric_median``: ``geometric_median_weights`` over the mixed table, applied to the mixed rows;
    * ``bulyan``: f, for P >= 4f + 3.

    With f = 0 every mixed row is the mean of all rows, and so is the result."""
    X = np.asarray(slots, dtype=np.float64)
    P = X.shape[0]
    D = _raw_d2(X)
    A = nnm_neighbours_d2(D, f)
    Y = _mix_rows(X, A, f)
    if mode == "coordinate_median":
        return coordinate_median(Y)
    if mode == "trimmed_mean":
        return trimmed_mean(Y, f)
    Dm = nnm_pair_d2(D, A, f)
    if mode == "krum":
        return Y[int(np.argsort(_krum_scores_d2(Dm, f), kind="stable")[0])]
    if mode == "multi_krum":
        return Y[np.argsort(_krum_scores_d2(Dm, f), kind="stable")[:P - f]].mean(axis=0)
    if mode == "geometric_median":
        return _weiszfeld_weights(Dm, 1e-10, 256) @ Y
    if mode == "bulyan":
        if P < 4 * f + 3:
            raise ValueError(f"Bulyan needs P >= 4f + 3 rows (got P = {P}, f = {f})")
        return nearest_to_median_mean(Y[_bulyan_rounds(Dm, f)], f)
    raise ValueError(f"NNM has no rule {mode!r}")


BUCKETING_MODES = ("coordinate_median", "trimmed_mean", "krum", "multi_krum", "geometric_median", "centered_clip")


def wbucket_rows(slots: np.ndarray, buckets: Sequence[Sequence[int]]) -> np.ndarray:
    """The fp32 worker-bucket rows (``--bucketing``; Karimireddy, He and Jaggi, ICLR 2022), one per bucket of
    ``codes.bucketing.wbuckets`` (members ascending, buckets ordered by their lowest member).  A one-member bucket's row is
    that member's value, bit for bit; otherwise y = x_lowest, then y = rn(y + x_j) for the other members in ascending slot
    order, then one rounded multiply by fp32(1 / |b|), with no contraction.  fp32 on purpose: every path forms these bits."""
    X = np.asarray(slots, dtype=np.float32)
    out = np.empty((len(buckets),) + X.shape[1:], dtype=np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        for b, members in enumerate(buckets):
            y = X[members[0]].copy()
            for j in members[1:]:
                y = np.add(y, X[j], dtype=np.float32)
            out[b] = y if len(members) == 1 else np.multiply(y, np.float32(1.0 / len(members)), dtype=np.float32)
    return out


def wbucket_pair_d2(D: np.ndarray, buckets: Sequence[Sequence[int]], P: int) -> np.ndarray:
    """Squared distances between the bucket rows from the raw table ``D`` [P, P] alone (``nnm_pair_d2``'s identity): with
    c = a_b / |b| - a_k / |k| (a_b the 0/1 membership of bucket b), ||y_b - y_k||^2 = -1/2 c^T D c in fp64, clamped at 0 (a NaN
    stays a NaN).  Buckets are disjoint, so c touches the members of b and k only."""
    A = np.zeros((len(buckets), P))
    for b, members in enumerate(buckets):
        A[b, list(members)] = 1.0 / len(members)
    D = np.array(D, dtype=np.float64)
    np.fill_diagonal(D, 0.0)
    nb = len(buckets)
    out = np.zeros((nb, nb))
    with np.errstate(invalid="ignore", over="ignore"):
        for b in range(nb):
            for k in range(nb):
                if b == k:
                    continue
                u = np.array(sorted(list(buckets[b]) + list(buckets[k])))
                c = A[b, u] - A[k, u]
                v = -0.5 * (c @ D[np.ix_(u, u)] @ c)
                out[b, k] = v if not v < 0.0 else 0.0
    return out


def bucketing(slots: np.ndarray, perm, s: int, f: int, mode: str, center=None, tau=None, D=None):
    """Bucketing, then the robust rule ``mode`` on the nb = ceil(P / s) bucket rows (``wbucket_rows``) of the permutation
    ``perm``, per tensor, with f = ``--worker-fail`` (each liar spoils at most one bucket):

    * ``coordinate_median``: trim (nb - 1) // 2;  * ``trimmed_mean``: trim f;  * ``krum``: s = f;  * ``multi_krum``: s = f,
      averaging nb - f rows;  * ``geometric_median``: Weiszfeld weights over the bucket table, applied to the bucket rows;
    * ``centered_clip``: around ``center`` with n = nb and radius ``tau`` (returns the aggregate, which is the next centre).

    The distance rules take their table from ``wbucket_pair_d2`` over the raw table ``D`` (``_raw_d2(slots)`` unless given:
    ``--rule-scope model`` passes the whole-model table).  With s = 1 this is the baseline rule on the raw slots."""
    from .bucketing import wbuckets
    X = np.asarray(slots, dtype=np.float32)
    P = X.shape[0]
    B = wbuckets(perm, s)
    nb = len(B)
    Y = wbucket_rows(X, B)
    if mode == "coordinate_median":
        return coordinate_median(Y)
    if mode == "trimmed_mean":
        return trimmed_mean(Y, f)
    if mode == "centered_clip":
        return centered_clip(Y, center, tau)
    Db = wbucket_pair_d2(_raw_d2(X) if D is None else D, B, P)
    if mode == "krum":
        return Y[int(np.argsort(_krum_scores_d2(Db, f), kind="stable")[0])].astype(np.float64)
    if mode == "multi_krum":
        return Y[np.argsort(_krum_scores_d2(Db, f), kind="stable")[:nb - f]].astype(np.float64).mean(axis=0)
    if mode == "geometric_median":
        return _weiszfeld_weights(Db, 1e-10, 256) @ Y.astype(np.float64)
    raise ValueError(f"bucketing has no rule {mode!r}")


def captured_group_bound(worker_fail: int, group_size: int) -> int:
    """DETOX's b_G: a group of r >= ``group_size`` members returns a liar's row only when at least (r + 1) // 2 of them lie
    (fewer leave the honest rows a strict majority, which Boyer-Moore always returns; for even r, r / 2 liars can tie and win),
    so ``worker_fail`` liars capture at most ``worker_fail // ((group_size + 1) // 2)`` groups."""
    return worker_fail // ((group_size + 1) // 2)


def detox_winner_slots(slots: np.ndarray, groups: Sequence[Sequence[int]]) -> List[int]:
    """Stage 1 of DETOX: the 0-based worker slot of each group's Boyer-Moore winner (``majority_vote``'s winners)."""
    _, members = majority_vote(np.asarray(slots), groups)
    return [int(g[k]) - 1 for g, k in zip(groups, members)]


def detox(slots: np.ndarray, groups: Sequence[Sequence[int]], mode: str, b: int) -> np.ndarray:
    """DETOX (Rajput, Wang, Charles and Papailiopoulos, NeurIPS 2019) on one tensor: majority vote inside every group, then
    ``mode`` across the G winner rows, with the tolerance b = b_G (``captured_group_bound``) in place of the worker count f:

    * ``coordinate_median``: trim (G - 1) // 2;   * ``trimmed_mean``: trim b;
    * ``multi_krum``: s = b, averaging G - b rows; * ``geometric_median``: Weiszfeld over the G rows;
    * ``bulyan``: f = b, for G >= 4b + 3 rows.

    With group size 1 every worker is its own group and this is the baseline rule on the same rows."""
    X = np.asarray(slots, dtype=np.float64)
    W = X[detox_winner_slots(slots, groups)]
    G = W.shape[0]
    if mode == "coordinate_median":
        return coordinate_median(W)
    if mode == "trimmed_mean":
        return trimmed_mean(W, b)
    if mode == "multi_krum":
        return multi_krum(W, b, G - b)
    if mode == "geometric_median":
        return geometric_median(W)
    if mode == "bulyan":
        return bulyan(W, b)
    raise ValueError(f"DETOX has no rule {mode!r}")


def model_rows(slots: np.ndarray, spans: Sequence[Tuple[int, int]]) -> np.ndarray:
    """The whole-model rows of an arena-laid ``slots`` [..., D]: every tensor's real elements ``(offset, numel)`` in tensor
    order, padding excluded, concatenated along the last axis."""
    X = np.asarray(slots)
    return np.concatenate([X[..., off:off + n] for off, n in spans], axis=-1)


def split_model(vec: np.ndarray, spans: Sequence[Tuple[int, int]]) -> List[np.ndarray]:
    """``model_rows`` undone for one result vector: its per-tensor pieces, in tensor order."""
    out, k = [], 0
    for _, n in spans:
        out.append(np.asarray(vec)[..., k:k + n])
        k += n
    return out


def model_scope(rule, slots: np.ndarray, spans: Sequence[Tuple[int, int]], *args) -> List[np.ndarray]:
    """Model scope of a per-tensor oracle: ``rule`` applied to ``model_rows(slots, spans)`` (with ``args``), its result split
    back per tensor.  Under DETOX the rows are the concatenations of each group's per-tensor vote winners (the vote itself
    stays per tensor); pass those as ``slots``."""
    return split_model(rule(model_rows(slots, spans), *args), spans)


def model_d2(per_tensor) -> np.ndarray:
    """A model-level distance as the fused kernels form it: the fp64 sum, in ascending tensor id, of the per-tensor fp64
    distances ``per_tensor`` [T, ...] (pair tables, centered clipping's d_i, or min-max's a_i, b_i, c and pair sums).  A NaN or
    Inf in any tensor reaches the sum, and the NaN-last and lower-row tie rules of every selection then apply unchanged."""
    D = np.asarray(per_tensor, dtype=np.float64)
    acc = np.zeros(D.shape[1:], dtype=np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        for d in D:
            acc = acc + d
    return acc


def sgd_momentum_step(p: np.ndarray, buf: np.ndarray, g: np.ndarray, lr: float, momentum: float,
                      weight_decay: float = 0.0, dampening: float = 0.0, nesterov: bool = False,
                      first_step: bool = False) -> Tuple[np.ndarray, np.ndarray]:
    """One SGD step with torch.optim.SGD semantics (reference: src/optim/sgd_modified.py:53-88)."""
    d_p = g + weight_decay * p if weight_decay != 0 else g
    if momentum != 0:
        buf = d_p.copy() if first_step else momentum * buf + (1.0 - dampening) * d_p
        d_p = d_p + momentum * buf if nesterov else buf
    return p - lr * d_p, buf


def worker_momentum_coefficients(beta: float) -> Tuple[float, float]:
    """(b, c) of worker momentum as fp32 values: b = fp32(beta), c = fp32(1 - beta) with 1 - beta formed in fp64 and rounded
    once.  Every path (push kernel, library-op PS, this oracle) multiplies by exactly these two numbers."""
    return float(np.float32(beta)), float(np.float32(1.0 - float(beta)))


def worker_momentum(m: np.ndarray, g: np.ndarray, beta: float) -> np.ndarray:
    """One step of worker-side momentum, dampened form (Karimireddy, He and Jaggi, ICML 2021; Allouah et al., AISTATS 2023):
    m' = b m + c g in fp32, each product rounded, then the sum rounded (no fused multiply-add).  The state starts at zero and
    there is no first-step copy.  bf16 gradients widen to fp32 exactly before the update."""
    b, c = worker_momentum_coefficients(beta)
    m32 = np.asarray(m, dtype=np.float32)
    g32 = np.asarray(g, dtype=np.float32)
    bm = np.multiply(np.float32(b), m32, dtype=np.float32)
    cg = np.multiply(np.float32(c), g32, dtype=np.float32)
    return np.add(bm, cg, dtype=np.float32)


def fma_f32(a, b, c) -> np.ndarray:
    """fp32 fused multiply-add, rn(a * b + c) with one rounding, element-wise.  The product of two fp32 values is exact in fp64;
    the sum is formed exactly as s + err (TwoSum), rounded to odd in fp64, then rounded once to fp32 (53 >= 24 + 2 bits makes
    the second rounding exact).  Non-finite sums are rounded as they are."""
    a64 = np.asarray(a, dtype=np.float32).astype(np.float64)
    b64 = np.asarray(b, dtype=np.float32).astype(np.float64)
    c64 = np.asarray(c, dtype=np.float32).astype(np.float64)
    p = a64 * b64
    with np.errstate(invalid="ignore", over="ignore"):
        s = p + c64
        bb = s - p
        err = (p - (s - bb)) + (c64 - bb)
    s, err = np.broadcast_to(s, np.broadcast(s, err).shape).copy(), np.broadcast_to(err, s.shape)
    odd = np.isfinite(s) & (err != 0) & ((s.view(np.int64) & 1) == 0)
    s[odd] = np.nextafter(s[odd], np.where(err[odd] > 0, np.inf, -np.inf))
    return s.astype(np.float32)


def centered_clip_weights(rows: np.ndarray, center: np.ndarray, tau: float) -> np.ndarray:
    """The fp32 weights of one centered-clipping step over one tensor: d_i = sum_e ((double)x_ie - (double)v_e)^2 in fp64,
    w_i = fp32(min(1, tau / sqrt(d_i)) / n) formed in fp64 and rounded once; d_i = 0 gives fp32(1 / n), and a NaN or +Inf d_i
    gives 0 (the row is then never read)."""
    X = np.asarray(rows, dtype=np.float32).astype(np.float64)
    v = np.asarray(center, dtype=np.float32).astype(np.float64)
    n = X.shape[0]
    with np.errstate(invalid="ignore", over="ignore"):
        d = ((X - v[None, :]) ** 2).sum(axis=1)
    return np.array([centered_clip_weight(float(di), tau, n) for di in d], dtype=np.float32)


def centered_clip_weight(d: float, tau: float, n: int) -> float:
    """One row's fp32 weight from its fp64 squared distance ``d`` to the centre (see ``centered_clip_weights``)."""
    if not d < math.inf:
        return 0.0
    return float(np.float32(1.0 / n)) if d == 0.0 else float(np.float32(min(1.0, tau / math.sqrt(d)) / n))


def centered_clip(rows: np.ndarray, center: np.ndarray, tau: float, weights=None) -> np.ndarray:
    """Centered clipping (Karimireddy, He and Jaggi, ICML 2021), one iteration on one tensor:
    g = v + (1/n) sum_i (x_i - v) min(1, tau / ||x_i - v||), with the n fp32 rows x_i and the fp32 centre v (the previous
    aggregate of this tensor, +0 at the start).  The weights come from ``centered_clip_weights`` (or ``weights``); then per
    coordinate acc = +0, acc = fma_rn(w_i, rn(x_i - v), acc) for i ascending with w_i != 0, and g = rn(v + acc), all fp32 with
    no other contraction.  g is both the aggregated gradient and the next centre.  The norm and tau are those of the rows given:
    per tensor by default, the paper's whole-model vector under ``model_scope`` (``--rule-scope model``)."""
    X = np.asarray(rows, dtype=np.float32)
    v = np.asarray(center, dtype=np.float32)
    w = centered_clip_weights(X, v, tau) if weights is None else np.asarray(weights, dtype=np.float32)
    acc = np.zeros_like(v)
    with np.errstate(invalid="ignore", over="ignore"):
        for i in range(X.shape[0]):
            if w[i] != 0:
                acc = fma_f32(w[i], np.subtract(X[i], v, dtype=np.float32), acc)
        return np.add(v, acc, dtype=np.float32)


def sign_pack(x: np.ndarray, valid=None) -> np.ndarray:
    """The signSGD wire of fp32 values ``x`` [..., n] (n a multiple of 32, in the slot's element layout): uint32 words
    [..., n / 32] with bit b (LSB = 0) of word w equal to 1 iff x[32 w + b] < 0.  So +0, -0, NaN and +Inf send 0 ("+").
    ``valid`` (bool [n], the arena's valid mask): padding bits are 0 whatever ``x`` holds there.  Signum is this applied to
    ``worker_momentum``'s output.  The library transports send the little-endian bytes of these words
    (``sign_pack(x).view(np.uint8)``): byte i, bit b is element 8 i + b."""
    x = np.asarray(x, dtype=np.float32)
    if x.shape[-1] % 32:
        raise ValueError(f"sign_pack: the last axis must be a multiple of 32, got {x.shape[-1]}")
    with np.errstate(invalid="ignore"):
        neg = x < 0
    if valid is not None:
        neg = neg & np.asarray(valid, dtype=bool)
    bits = neg.reshape(*x.shape[:-1], x.shape[-1] // 32, 32).astype(np.uint64)
    return (bits << np.arange(32, dtype=np.uint64)).sum(axis=-1).astype(np.uint32)


def sign_unpack(words: np.ndarray) -> np.ndarray:
    """uint32 sign words [..., m] -> uint8 bits [..., 32 m] (``sign_pack``'s layout; 1 = "-")."""
    w = np.asarray(words, dtype=np.uint32)
    bits = (w[..., None] >> np.arange(32, dtype=np.uint32)) & np.uint32(1)
    return bits.reshape(*w.shape[:-1], w.shape[-1] * 32).astype(np.uint8)


def sign_vote(bits: np.ndarray, P: int, valid) -> np.ndarray:
    """signSGD with majority vote (Bernstein, Zhao, Azizzadenesheli and Anandkumar, ICLR 2019) over the sign bits [P, n] of
    the P workers: per coordinate n_neg = rows with bit 1 and n_pos = P - n_neg; g = +1 if n_pos > n_neg, -1 if n_neg > n_pos,
    +0 on a tie, and +0 on every padding coordinate (``valid`` False) whatever its bits say.  fp32 [n]."""
    b = np.asarray(bits, dtype=np.int64)
    if b.ndim != 2 or b.shape[0] != P:
        raise ValueError(f"sign_vote: expected [{P}, n] bits, got {b.shape}")
    n_neg = b.sum(axis=0)
    n_pos = P - n_neg
    g = np.where(n_pos > n_neg, 1.0, np.where(n_neg > n_pos, -1.0, 0.0)).astype(np.float32)
    return np.where(np.asarray(valid, dtype=bool), g, np.float32(0.0)).astype(np.float32)


def arc_row_factors(d, k: int) -> np.ndarray:
    """ARC's fp32 factors from the fp64 squared norms ``d`` [P]: d_tau is the (k+1)-th largest d_i, a NaN ranking above every
    number (ties do not matter: only the value is used).  a_i = 1 when !(d_i > d_tau), else fp32(sqrt(d_tau) / sqrt(d_i))
    formed in fp64.  So a NaN row keeps factor 1, a row holding an Inf gets 0, and with more than k non-finite rows d_tau is
    non-finite and no row is clipped."""
    d = [float(x) for x in d]
    tau = sorted(d, key=lambda x: (not math.isnan(x), -x if not math.isnan(x) else 0.0))[k]
    return np.array([np.float32(math.sqrt(tau) / math.sqrt(x)) if x > tau else np.float32(1.0) for x in d], dtype=np.float32)


def _arc_d2(X: np.ndarray) -> np.ndarray:
    """fp64 squared norm of every row of one tensor's [P, n] fp32 values (each square exact in fp64)."""
    X64 = np.asarray(X, dtype=np.float32).astype(np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        return (X64 * X64).sum(axis=1)


def arc_factors(slots: np.ndarray, spans: Sequence[Tuple[int, int]], f: int, scope: str = "tensor") -> np.ndarray:
    """Adaptive robust clipping's factors [T, P] fp32 (Allouah et al., arXiv 2405.14432) over the P arena-laid worker slots
    ``slots`` [P, D] with the tensors ``spans`` (offset, numel): per tensor from its d_i (``scope="tensor"``), or one row from
    the whole-model d_i -- the per-tensor d_i summed in ascending tensor order, ``model_d2`` -- in every tensor
    (``scope="model"``).  k = ``arc_k(P, f)``; see ``arc_row_factors``."""
    X = np.asarray(slots, dtype=np.float32)
    k = arc_k(X.shape[0], f)
    d = [_arc_d2(X[:, off:off + n]) for off, n in spans]
    if scope == "model":
        return np.tile(arc_row_factors(model_d2(d), k), (len(spans), 1))
    return np.stack([arc_row_factors(di, k) for di in d])


def arc(slots: np.ndarray, spans: Sequence[Tuple[int, int]], f: int, scope: str = "tensor", factors=None) -> np.ndarray:
    """Adaptive robust clipping: a copy of ``slots`` in which every tensor of every row with factor a_i < 1 (``arc_factors``, or
    ``factors``) is multiplied by a_i, one fp32 multiply per element.  Padding and the other rows are left as they are, and
    with k = 0 nothing changes."""
    X = np.array(slots, dtype=np.float32, copy=True)
    if arc_k(X.shape[0], f) == 0:
        return X
    a = arc_factors(X, spans, f, scope) if factors is None else np.asarray(factors, dtype=np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        for t, (off, n) in enumerate(spans):
            for i in np.flatnonzero(a[t] < 1):
                X[i, off:off + n] = np.multiply(X[i, off:off + n], a[t, i], dtype=np.float32)
    return X
