"""Worker buckets (``--bucketing s``; Karimireddy, He and Jaggi, *Byzantine-Robust Learning on Heterogeneous Datasets via
Bucketing*, ICLR 2022): each step the PS permutes the P worker slots at random, averages them in buckets of s and runs the
robust rule on the ceil(P / s) bucket means.

The permutations are a table fixed by ``--seed``, one row per step like the adversary schedule, so every PS implementation, a
graph replay (which reads row ``step % len`` on the device) and a resumed job see the same buckets.  These worker buckets are
not the gradient buckets the workers push in.
"""
from __future__ import annotations

from typing import List

import numpy as np


def bucket_schedule(P: int, steps: int, seed: int) -> np.ndarray:
    """int32 [steps + 1, P]: row t is the permutation of the slots 0..P-1 at step t (the adversary schedule's length)."""
    rng = np.random.RandomState((seed * 1000003 + 0x5B0C) & 0x7FFFFFFF)
    return np.stack([rng.permutation(P) for _ in range(steps + 1)]).astype(np.int32)


def wbuckets(perm, s: int) -> List[List[int]]:
    """The worker buckets of one permutation: bucket b holds perm[b s : min((b + 1) s, P)], its members in ascending slot
    order, and the buckets ordered by their lowest member (so s = 1 gives the slots in slot order)."""
    perm = [int(x) for x in perm]
    groups = [sorted(perm[b: b + s]) for b in range(0, len(perm), s)]
    return sorted(groups, key=lambda g: g[0])


def wbucket_masks(perm, s: int) -> np.ndarray:
    """uint32 [nb]: bit j of entry b is set iff slot j is in bucket row b (``wbuckets`` order) -- what the plan kernel writes."""
    return np.array([sum(1 << j for j in g) for g in wbuckets(perm, s)], dtype=np.uint32)
