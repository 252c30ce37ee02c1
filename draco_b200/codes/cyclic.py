"""Cyclic (Fourier / Reed-Solomon-over-C) gradient code.

What the reference computes (src/coding.py:4-68, src/master/cyclic_master.py:152-197,
src/c_coding.cpp:15-84) re-derived here from the algebra rather than transliterated:

* ``n`` workers, ``s`` adversaries, redundancy ``r = 2s+1``.  Worker ``i`` computes
  the gradients of batches ``i .. i+2s (mod n)`` (support mask ``B``).
* ``C`` is the unitary ``n x n`` DFT.  ``C1`` = its first ``n-2s`` columns, ``C2`` = the
  last ``2s``.  The encoding matrix is ``W = C1 Q`` with ``Q[0, :] = 1`` and the other
  rows chosen so that ``W`` vanishes off the support.  Hence ``C2^H W = 0`` (every honest
  codeword has a zero "syndrome") and ``e1^T C1^H W = 1^T / ... `` recovers the plain sum.
* Worker ``i`` ships ``R[i, :] = sum_j W[i, j] g_j`` (+ an arbitrary error if Byzantine).
* PS: syndrome ``C2^H R f`` (``f`` a fixed random projection) are ``2s`` consecutive DFT
  coefficients of an ``<= s``-sparse error vector -> Prony: an ``s x s`` Hankel solve
  yields the error-locator polynomial, whose roots among the ``n``-th roots of unity are
  the Byzantine rows.  Any ``n-2s`` healthy rows ``h`` then give ``v`` with
  ``C1[h]^T v = e1`` and ``v^T R[h] = sum_j g_j``.

Everything here is float64/complex128 numpy: it is the *oracle* the CUDA decode
(csrc/cuda/fourier.cu) and the C++ locator (csrc/host/locator.cpp) are tested against.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional, Sequence, Tuple

import numpy as np


@dataclass(frozen=True)
class CyclicCode:
    n: int
    s: int
    W: np.ndarray          # [n, n] complex128 encoding matrix (row = worker, col = batch)
    support: np.ndarray    # [n, n] {0,1}: support[i, j] = 1 iff worker i computes batch j
    W_perp: np.ndarray     # [2s, n] = C2^H   (syndrome map)
    S: np.ndarray          # [1, n]  = e1^T C1^H
    C1: np.ndarray         # [n, n-2s]

    @property
    def r(self) -> int:
        return 2 * self.s + 1

    def batches_of(self, worker: int) -> np.ndarray:
        """Batch ids (0-based) worker ``worker`` (0-based) must compute, in ring order."""
        return (worker + np.arange(self.r)) % self.n

    def coeffs_of(self, worker: int) -> np.ndarray:
        """Complex encode coefficients aligned with :meth:`batches_of`."""
        return self.W[worker, self.batches_of(worker)]


def dft_matrix(n: int) -> np.ndarray:
    k = np.arange(n)
    return np.exp(-2j * np.pi * np.outer(k, k) / n) / np.sqrt(n)


def support_mask(n: int, s: int) -> np.ndarray:
    m = np.zeros((n, n), dtype=np.float64)
    for i in range(n):
        m[i, (i + np.arange(2 * s + 1)) % n] = 1.0
    return m


def search_w(n: int, s: int) -> CyclicCode:
    """Construct the code (same outputs as the reference's ``search_w``: W, mask, W_perp, S, C1)."""
    if n < 2 * s + 1:
        raise ValueError(f"cyclic code needs n >= 2s+1 (n={n}, s={s})")
    C = dft_matrix(n)
    k = n - 2 * s
    C1, C2 = C[:, :k], C[:, k:]
    mask = support_mask(n, s)
    Q = np.ones((k, n), dtype=np.complex128)
    for j in range(n):
        zero_rows = np.flatnonzero(mask[:, j] == 0)          # workers that must not touch batch j
        if k > 1:
            A = C1[zero_rows, 1:]
            b = -C1[zero_rows, 0]
            Q[1:, j] = np.linalg.lstsq(A, b, rcond=None)[0]
    W = C1 @ Q
    W = np.where(mask > 0, W, 0.0)                            # kill the 1e-16 leakage off-support
    S = np.zeros((1, k), dtype=np.complex128)
    S[0, 0] = 1.0
    return CyclicCode(n, s, W, mask, C2.conj().T, S @ C1.conj().T, C1)


# ---------------------------------------------------------------------------------------------
# numpy decode oracle
# ---------------------------------------------------------------------------------------------

def hankel_system(syndrome: np.ndarray, s: int) -> Tuple[np.ndarray, np.ndarray]:
    """Hankel system of the reference (src/c_coding.cpp:75-79): A[i,:]=E[s-i-1:2s-i-1], b[i]=E[2s-i-1]."""
    A = np.zeros((s, s), dtype=np.complex128)
    b = np.zeros(s, dtype=np.complex128)
    for i in range(s):
        A[i, :] = syndrome[s - i - 1: 2 * s - i - 1]
        b[i] = syndrome[2 * s - i - 1]
    return A, b


def locator_values(alpha: np.ndarray, n: int) -> np.ndarray:
    """Evaluate p(z) = z^s - sum_j alpha_j z^j at the n-th roots of unity z_t = exp(+2 pi i t / n)."""
    s = alpha.shape[0]
    z = np.exp(2j * np.pi * np.arange(n) / n)
    p = z ** s
    for j in range(s):
        p = p - alpha[j] * z ** j
    return p


def pick_healthy(pvals: np.ndarray, n: int, s: int, rel_tol: float = 1e-6) -> np.ndarray:
    """Rows whose locator value is *not* ~0, first ``n-2s`` in index order.

    The reference uses an absolute 1e-9 threshold in complex128 (cyclic_master.py:162); our payload is
    complex64 so the threshold is relative to the largest locator magnitude, with a top-k fallback.
    """
    mag = np.abs(pvals)
    need = n - 2 * s
    healthy = np.flatnonzero(mag > rel_tol * max(mag.max(), 1e-300))
    if healthy.size < need:
        healthy = np.sort(np.argsort(-mag, kind="stable")[:need])
    return healthy[:need]


def recombination_vector(code: CyclicCode, healthy: Sequence[int]) -> np.ndarray:
    """v (length n, zero off ``healthy``) with C1[healthy]^T v_h = e1."""
    n, s = code.n, code.s
    k = n - 2 * s
    h = np.asarray(healthy[:k])
    M = code.C1[h, :].T                        # [k, k]
    e1 = np.zeros(k, dtype=np.complex128)
    e1[0] = 1.0
    vh = np.linalg.solve(M, e1)
    v = np.zeros(n, dtype=np.complex128)
    v[h] = vh
    return v


def decode(code: CyclicCode, R: np.ndarray, f: Optional[np.ndarray] = None,
           rel_tol: float = 1e-6) -> Tuple[np.ndarray, np.ndarray]:
    """Oracle decode of one tensor.  ``R``: [n, d] complex.  Returns (sum_j g_j as real [d], healthy rows)."""
    n, s = code.n, code.s
    R = np.asarray(R, dtype=np.complex128)
    if f is None:
        f = np.ones(R.shape[1])
    if s == 0:
        healthy = np.arange(n)
    else:
        E = R @ f
        synd = code.W_perp @ E
        A, b = hankel_system(synd, s)
        scale = np.abs(E).max()
        if np.abs(synd).max() <= 1e-7 * max(scale, 1e-300):
            alpha = np.zeros(s, dtype=np.complex128)          # no adversary: p(z) = z^s
        else:
            alpha = np.linalg.lstsq(A, b, rcond=1e-10)[0]     # min-norm, like the reference's JacobiSVD
        healthy = pick_healthy(locator_values(alpha, n), n, s, rel_tol)
    v = recombination_vector(code, healthy)
    return np.real(v @ R), healthy


def encode(code: CyclicCode, worker: int, grads_by_batch: np.ndarray) -> np.ndarray:
    """Oracle encode: ``grads_by_batch`` is [n, d] (all batches); returns worker's complex row [d]."""
    return code.W[worker, :] @ np.asarray(grads_by_batch, dtype=np.complex128)


def decode_ifft(code: CyclicCode, R: np.ndarray, f: Optional[np.ndarray] = None) -> np.ndarray:
    """Alternative decoder: estimate the error matrix and subtract it (the reference's earlier, now dead, decoder --
    ``_obtain_E`` / ``_obtain_epsilon`` in src/master/cyclic_master.py:175-188 and the orphan Cython ``decoding`` module).

    The syndrome ``C2^H R`` holds the last 2s DFT coefficients of every error column.  The locator polynomial (from the
    projected syndrome, as in :func:`decode`) gives a linear recurrence that extends them cyclically to all n
    coefficients; an inverse DFT then yields the error matrix ``eps`` itself, and ``S (R - eps) = sum_j g_j``.
    Cost: O(n d) like the recombination decoder, but it also *returns what every liar added*."""
    n, s = code.n, code.s
    R = np.asarray(R, dtype=np.complex128)
    d = R.shape[1]
    if f is None:
        f = np.ones(d)
    if s == 0:
        return np.real((code.S @ R)[0])
    k = n - 2 * s
    synd_full = code.W_perp @ R                                   # [2s, d] : spectrum indices k .. n-1
    proj = synd_full @ f
    A, b = hankel_system(proj, s)
    if np.abs(proj).max() <= 1e-7 * max(np.abs(R @ f).max(), 1e-300):
        eps = np.zeros_like(R)
    else:
        alpha = np.linalg.lstsq(A, b, rcond=1e-10)[0]
        spec = np.zeros((n + k, d), dtype=np.complex128)          # spectrum laid out k .. n-1, then n .. n+k-1 (== 0 .. k-1)
        spec[: 2 * s] = synd_full
        for t in range(2 * s, 2 * s + k):                         # E[t] = sum_j alpha_j E[t - s + j]
            spec[t] = sum(alpha[j] * spec[t - s + j] for j in range(s))
        full = np.zeros((n, d), dtype=np.complex128)
        full[k:] = spec[: 2 * s]
        full[:k] = spec[2 * s: 2 * s + k]
        C = dft_matrix(n)
        eps = C @ full                                            # eps = C * (C^H eps)
    clean = R - eps
    return np.real((code.S @ clean)[0])
