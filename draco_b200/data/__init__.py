"""Datasets and identical-batch plans.

Reference behaviour being reproduced (src/util.py:23-66, src/worker/rep_worker.py:89, src/worker/cyclic_worker.py:88-95,
src/datasets/utils.py:7-29):

* MNIST is normalised with (0.1307, 0.3081); CIFAR-10 with per-channel mean/std and, for training, reflect-pad-4 +
  random-crop-32 + horizontal flip.
* baseline workers shuffle independently; members of a repetition group share a seed (re-seeded per epoch with
  ``group_seed + epoch``) so they see *the same batches*; under the cyclic code every worker derives the same global
  batch of ``n*B`` consecutive samples (seed ``428 + 23*epoch``) and computes its ``2s+1`` sub-batches of it.

There is no network here, so ``load_dataset`` returns a deterministic synthetic dataset of the right shape (class
templates + noise, learnable) unless the real files already exist under ``root``.  Instead of the reference's
per-process DataLoaders (every cyclic worker materialised the whole global batch), a ``BatchPlan`` maps
``(step, worker)`` to sample indices, and augmentation is a seeded tensor op so replicas stay bit-identical.
"""
from __future__ import annotations

import os
from dataclasses import dataclass
from typing import List, Optional, Sequence, Tuple

import numpy as np
import torch

MNIST_MEAN, MNIST_STD = (0.1307,), (0.3081,)
CIFAR_MEAN = tuple(x / 255.0 for x in (125.3, 123.0, 113.9))
CIFAR_STD = tuple(x / 255.0 for x in (63.0, 62.1, 66.7))

SHAPES = {"MNIST": (1, 28, 28), "Cifar10": (3, 32, 32), "ImageNet": (3, 224, 224)}
NUM_CLASSES = {"MNIST": 10, "Cifar10": 10, "ImageNet": 1000}


class TensorDataset:
    """uint8 images [N, C, H, W] + int64 labels, with the dataset's normalisation constants."""

    def __init__(self, name: str, images: torch.Tensor, labels: torch.Tensor, synthetic: bool):
        self.name, self.images, self.labels, self.synthetic = name, images, labels, synthetic
        mean, std = (MNIST_MEAN, MNIST_STD) if name == "MNIST" else (CIFAR_MEAN, CIFAR_STD)
        c = images.shape[1]
        self.mean = torch.tensor((mean * c)[:c], dtype=torch.float32).view(1, c, 1, 1)
        self.std = torch.tensor((std * c)[:c], dtype=torch.float32).view(1, c, 1, 1)

    def __len__(self) -> int:
        return self.images.shape[0]

    def pin(self) -> "TensorDataset":
        if torch.cuda.is_available():
            self.images, self.labels = self.images.pin_memory(), self.labels.pin_memory()
        return self

    def get_batch(self, indices: Sequence[int]) -> Tuple[torch.Tensor, torch.Tensor]:
        """Raw (uint8 images, labels) for ``indices`` -- the reference's ``get_batch(dataset, indices)``."""
        idx = torch.as_tensor(np.asarray(indices), dtype=torch.long)
        return self.images[idx], self.labels[idx]

    def next_batch(self, batch_size: int, shuffle: bool = True) -> Tuple[torch.Tensor, torch.Tensor]:
        """Sequential mini-batches with an epoch counter -- the reference's legacy ``MNISTDataset.next_batch`` /
        ``DataLoader.next_batch`` API (src/datasets/__init__.py:5-51, src/data_loader_ops/my_data_loader.py:254-319)."""
        st = self.__dict__.setdefault("_nb_state", {"pos": 0, "perm": None, "epochs_completed": 0})
        n = len(self)
        if st["perm"] is None or st["pos"] + batch_size > n:
            if st["perm"] is not None:
                st["epochs_completed"] += 1
            st["perm"] = torch.randperm(n) if shuffle else torch.arange(n)
            st["pos"] = 0
        idx = st["perm"][st["pos"]: st["pos"] + batch_size]
        st["pos"] += batch_size
        return self.normalize(self.images[idx]), self.labels[idx]

    @property
    def epochs_completed(self) -> int:
        return self.__dict__.get("_nb_state", {}).get("epochs_completed", 0)

    def normalize(self, x_u8: torch.Tensor, dtype=torch.float32) -> torch.Tensor:
        x = x_u8.to(torch.float32) / 255.0
        return ((x - self.mean.to(x.device)) / self.std.to(x.device)).to(dtype)


def synthetic_dataset(name: str, size: int = 8192, seed: int = 428) -> TensorDataset:
    c, h, w = SHAPES[name]
    k = NUM_CLASSES[name]
    g = torch.Generator().manual_seed(seed)
    low = torch.rand(k, c, max(h // 4, 1), max(w // 4, 1), generator=g)
    templates = torch.nn.functional.interpolate(low, size=(h, w), mode="nearest")
    labels = torch.randint(0, k, (size,), generator=g)
    noise = torch.rand(size, c, h, w, generator=g)
    imgs = (0.65 * templates[labels] + 0.35 * noise).clamp_(0, 1)
    return TensorDataset(name, (imgs * 255).to(torch.uint8), labels, synthetic=True)


def load_dataset(name: str, root: str = "./data", train: bool = True, synthetic_size: int = 8192,
                 seed: int = 428) -> TensorDataset:
    """Real torchvision data when already on disk (never downloads), else the synthetic stand-in."""
    if name not in SHAPES:
        raise ValueError(f"unknown --dataset {name!r}; choose from {sorted(SHAPES)}")
    try:
        if name == "MNIST" and os.path.isdir(os.path.join(root, "mnist_data")):
            from torchvision import datasets
            ds = datasets.MNIST(os.path.join(root, "mnist_data"), train=train, download=False)
            return TensorDataset(name, ds.data.unsqueeze(1).contiguous(), ds.targets.long(), synthetic=False)
        if name == "Cifar10" and os.path.isdir(os.path.join(root, "cifar10_data")):
            from torchvision import datasets
            ds = datasets.CIFAR10(os.path.join(root, "cifar10_data"), train=train, download=False)
            imgs = torch.from_numpy(ds.data).permute(0, 3, 1, 2).contiguous()
            return TensorDataset(name, imgs, torch.tensor(ds.targets, dtype=torch.long), synthetic=False)
    except Exception:
        pass
    return synthetic_dataset(name, synthetic_size if train else max(synthetic_size // 8, 256), seed + (0 if train else 1))


def augment_cifar(x_u8: torch.Tensor, seed: int) -> torch.Tensor:
    """Reflect-pad-4 + random-crop-32 + horizontal flip, deterministic in ``seed`` (so replicas agree)."""
    n, c, h, w = x_u8.shape
    g = torch.Generator().manual_seed(int(seed) & 0x7FFFFFFF)
    dx = torch.randint(0, 9, (n,), generator=g)
    dy = torch.randint(0, 9, (n,), generator=g)
    flip = torch.rand(n, generator=g) < 0.5
    xp = torch.nn.functional.pad(x_u8.float(), (4, 4, 4, 4), mode="reflect")
    ar = torch.arange(w)
    cols = (dx.view(n, 1) + ar.view(1, w))
    cols = torch.where(flip.view(n, 1), cols.flip(1), cols)
    rows = dy.view(n, 1) + torch.arange(h).view(1, h)
    idx_n = torch.arange(n).view(n, 1, 1, 1)
    idx_c = torch.arange(c).view(1, c, 1, 1)
    out = xp[idx_n, idx_c, rows.view(n, 1, h, 1), cols.view(n, 1, 1, w)]
    return out.to(torch.uint8)


DIRICHLET_MAX_DRAWS = 100


def dirichlet_shards(labels, holders: int, alpha: float, batch_size: int, seed: int) -> List[np.ndarray]:
    """Heterogeneous split of a dataset over ``holders`` (Hsu, Qi and Brown, 2019): for each class c in ascending order, its
    indices ascending are cut by shares p ~ Dir(alpha 1_H) at ``(cumsum(p)[:-1] * n_c).astype(int)``, and holder h takes chunk
    h.  When a shard holds fewer than ``batch_size`` samples, every class is drawn again from the same generator, up to
    ``DIRICHLET_MAX_DRAWS`` draws.  Returns each holder's indices, ascending."""
    y = np.asarray(labels).reshape(-1)
    rng = np.random.RandomState((seed * 1000003 + 0xD1C1) & 0x7FFFFFFF)
    by_class = [np.flatnonzero(y == c) for c in np.unique(y)]
    for _ in range(DIRICHLET_MAX_DRAWS):
        parts: List[List[np.ndarray]] = [[] for _ in range(holders)]
        for idx in by_class:
            p = rng.dirichlet(np.full(holders, float(alpha)))
            for h, chunk in enumerate(np.split(idx, (np.cumsum(p)[:-1] * len(idx)).astype(int))):
                parts[h].append(chunk)
        shards = [np.sort(np.concatenate(c)) for c in parts]
        if min(len(s) for s in shards) >= batch_size:
            return shards
    raise ValueError(f"--dirichlet-alpha {alpha}: no split of {len(y)} samples over {holders} holders gave every shard at least "
                     f"B = {batch_size} samples in {DIRICHLET_MAX_DRAWS} draws; raise alpha or the dataset size, or lower the "
                     f"batch size")


def class_histograms(labels, shards: Sequence[np.ndarray]) -> List[List[int]]:
    """Samples of each class in every shard."""
    y = np.asarray(labels).reshape(-1)
    k = int(y.max()) + 1 if len(y) else 0
    return [np.bincount(y[s], minlength=k).tolist() for s in shards]


@dataclass
class BatchPlan:
    """Maps (step, worker rank) to dataset indices for one approach."""

    approach: str                 # baseline | maj_vote | cyclic | detox | nnm
    dataset_size: int
    batch_size: int
    num_workers: int
    group_of: Optional[dict] = None          # rank -> group id (maj_vote, detox)
    group_seeds: Optional[List[int]] = None
    seed: int = 428
    redundancy: int = 1                       # cyclic: 2s+1
    shards: Optional[List[np.ndarray]] = None  # --dirichlet-alpha: the dataset indices of every data holder (dirichlet_shards)

    def _perm(self, seed: int) -> np.ndarray:
        cache = self.__dict__.setdefault("_perm_cache", {})
        key = seed & 0x7FFFFFFF
        if key not in cache:
            if len(cache) > 64:
                cache.clear()
            cache[key] = np.random.RandomState(key).permutation(self.dataset_size)
        return cache[key]

    def _slice(self, perm: np.ndarray, pos: int, width: int) -> np.ndarray:
        start = (pos * width) % max(self.dataset_size - width + 1, 1)
        return perm[start: start + width]

    def steps_per_epoch(self) -> int:
        width = self.batch_size * (self.num_workers if self.approach == "cyclic" else 1)
        return max(self.dataset_size // width, 1)

    def _holder(self, rank: int) -> int:
        """The data holder of a worker: itself (baseline, nnm), or its repetition group (maj_vote, detox)."""
        return self.group_of[rank] if self.approach in ("maj_vote", "detox") else rank - 1

    def _shard_indices(self, step: int, rank: int) -> List[np.ndarray]:
        """Heterogeneous data: the holder's own epochs over its shard, a permutation per epoch seeded as the IID batches are."""
        shard, B = self.shards[self._holder(rank)], self.batch_size
        epoch, pos = divmod(max(step - 1, 0), len(shard) // B)
        seed = (self.group_seeds[self.group_of[rank]] + epoch if self.approach in ("maj_vote", "detox")
                else self.seed * 1000003 + rank * 7919 + epoch)
        perm = np.random.RandomState(seed & 0x7FFFFFFF).permutation(len(shard))
        return [shard[perm[pos * B: (pos + 1) * B]]]

    def indices(self, step: int, rank: int) -> List[np.ndarray]:
        """List of index arrays (one per sub-batch this worker computes at ``step``; length 1 unless cyclic)."""
        if self.shards is not None:
            return self._shard_indices(step, rank)
        spe = self.steps_per_epoch()
        epoch, pos = divmod(max(step - 1, 0), spe)
        B = self.batch_size
        if self.approach in ("baseline", "nnm"):                  # every worker draws its own batch
            return [self._slice(self._perm(self.seed * 1000003 + rank * 7919 + epoch), pos, B)]
        if self.approach in ("maj_vote", "detox"):
            gseed = self.group_seeds[self.group_of[rank]]
            return [self._slice(self._perm(gseed + epoch), pos, B)]
        if self.approach == "cyclic":
            n = self.num_workers
            glob = self._slice(self._perm(self.seed + 23 * epoch), pos, n * B)
            return [glob[j * B:(j + 1) * B] for j in (rank - 1 + np.arange(self.redundancy)) % n]
        raise ValueError(self.approach)

    def batch_ids(self, step: int, rank: int) -> List[int]:
        """Identity of each sub-batch (used to seed dropout / augmentation identically across holders)."""
        if self.approach == "cyclic":
            return [int(j) for j in (rank - 1 + np.arange(self.redundancy)) % self.num_workers]
        if self.approach in ("maj_vote", "detox"):
            return [int(self.group_of[rank])]
        return [int(rank)]
