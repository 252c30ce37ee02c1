"""Job configuration: the reference's flag surface (src/distributed_nn.py:23-77) as a dataclass + parser.

Every reference flag keeps its name and default.  Flags the reference parses but ignores are honoured here where that
is meaningful (``--seed`` seeds model init, ``--adversarial`` scales the attack magnitude, ``--log-interval`` throttles
logging, ``--no-cuda`` forces the CPU/Gloo path) -- see DESIGN.md "flag semantics".  New flags are additive.
"""
from __future__ import annotations

import argparse
import math
from dataclasses import asdict, dataclass
from typing import Optional

from . import rules

APPROACHES = ("baseline", "maj_vote", "cyclic", "detox", "nnm")
MODES = ("normal", "geometric_median", "krum", "maj_vote", "coordinate_median", "trimmed_mean", "multi_krum", "bulyan",
         "centered_clip", "sign_vote")
ERR_MODES = ("rev_grad", "constant", "random", "omniscient", "alie", "minmax", "ipm", "mimic", "none")
TRANSPORTS = ("nvl", "nccl", "nccl_flat", "gloo")
SCOPES = ("tensor", "model")        # --rule-scope / --attack-scope: distances per parameter tensor, or over the whole model
# the --mode values whose rule measures distances between rows (every --approach nnm mode does, through its neighbourhoods)
DISTANCE_MODES = ("krum", "multi_krum", "geometric_median", "bulyan", "centered_clip")
# the --approach nnm modes: the base rules of the mixed rows
NNM_MODES = tuple(rules.BASES[b].mode for b in rules.SOURCES["nnm"].bases)


@dataclass
class JobConfig:
    # ---- reference flags ------------------------------------------------------------------
    batch_size: int = 128
    test_batch_size: int = 100
    max_steps: int = 10000
    epochs: int = 100
    lr: float = 0.01
    momentum: float = 0.5
    no_cuda: bool = False
    seed: int = 1
    log_interval: int = 10
    network: str = "LeNet"
    mode: str = "normal"
    dataset: str = "MNIST"
    comm_type: str = "Bcast"
    err_mode: str = "rev_grad"
    approach: str = "maj_vote"
    num_aggregate: int = 5
    eval_freq: int = 50
    train_dir: str = "output/models/"
    adversarial: int = 1
    worker_fail: int = 2
    group_size: int = 5
    compress_grad: str = "compress"  # lossless DRC2 codec on the wire (reference default: blosc on every gradient message)
    checkpoint_step: int = 0
    # ---- additions --------------------------------------------------------------------------
    num_workers: int = 0            # logical workers P (0: world_size - 1, like `mpirun -n P+1`)
    transport: str = "nvl"          # nvl: fused sm_90a kernels over peer memory | nccl: baseline | gloo: CPU
    dtype: str = "bf16"             # compute dtype on workers (bf16 | fp32)
    cuda_graphs: bool = True
    weight_decay: float = 0.0
    nesterov: bool = False
    dampening: float = 0.0
    optimizer: str = "sgd"          # sgd | adam (reference: src/optim/{sgd,adam}_modified.py); every transport
    amsgrad: bool = False
    adam_beta1: float = 0.9
    adam_beta2: float = 0.999
    adam_eps: float = 1e-8
    data_root: str = "./data"
    synthetic_size: int = 8192
    augment: bool = False
    data_on_device: bool = False    # keep the dataset in HBM and gather batches on the device
    metrics_file: Optional[str] = None
    debug_checksum: bool = False    # verify every pushed gradient: loopback re-encode vs what landed in the PS slot (eager mode)
    profile_phases: bool = False    # CUDA-event timers per phase (fetch/comp/encode/comm/decode/update); disables CUDA graphs
    multicast: str = "auto"         # auto | on | off  (NVLS multimem.st broadcast)
    wgrad_stream: str = "auto"      # weight-gradient kernels on a low-priority side stream: auto (= on with zero-copy gradients) | on | off
    spin_timeout_s: float = 60.0
    ps_stream: bool = False         # PS co-located with workers consumes gradient buckets on its own stream (captured graph only).
                                    # Off by default: its spin-wait kernels then depend on kernels of OTHER graph branches making
                                    # progress, which holds only while every branch gets its own hardware queue
                                    # (CUDA_DEVICE_MAX_CONNECTIONS >= number of concurrent streams)
    num_classes: int = 10
    deterministic: bool = True
    overlap_push: bool = True       # ship gradient buckets while the remaining layers are still back-propagating
    pipeline_ps: bool = True        # PS votes / applies / broadcasts a bucket as soon as every worker pushed it
    push_ctas: int = 16             # CTAs of an overlapped bucket push (NVLink-bound: a handful of SMs saturates the link)
    worker_streams: int = 4         # >1: logical workers sharing a GPU run on (up to) this many concurrent CUDA streams
    zero_copy_grads: bool = True    # push reads gradients where autograd left them (pointer table), no flat gather
    attack_z: Optional[float] = None  # --err-mode alie: z of mu - z * sigma (None: Baruch et al.'s z_max for P and f)
    worker_momentum: float = 0.0    # beta of worker-side momentum: every worker pushes m <- beta m + (1 - beta) g (0: off)
    clip_tau: Optional[float] = None  # --mode centered_clip: the clipping radius tau in the gradient's units (per rule_scope)
    rule_scope: str = "tensor"      # distance-based rules: one choice per parameter tensor, or one over the whole model
    attack_scope: str = "tensor"    # --err-mode minmax: one gamma per parameter tensor, or one over the whole model
    bucketing: int = 0              # worker buckets of s: the robust rule runs on the means of ceil(P / s) random buckets (0: off)
    dirichlet_alpha: Optional[float] = None  # heterogeneous data: each holder's shard has Dirichlet(alpha) class shares (None: IID)
    attack_eps: Optional[float] = None  # --err-mode ipm: the liars send -eps * mu (None: codes.adversary.IPM_EPS)
    mimic_warmup: Optional[int] = None  # --err-mode mimic: steps that learn the direction (None: codes.adversary.MIMIC_WARMUP)
    arc: Optional[str] = None       # adaptive robust clipping of the worker slots before the rule: tensor | model (None: off)

    # ---- derived --------------------------------------------------------------------------
    def resolve(self, world_size: int) -> "JobConfig":
        if self.num_workers <= 0:
            self.num_workers = max(world_size - 1, 1)
        if self.approach not in APPROACHES:
            raise ValueError(f"--approach must be one of {APPROACHES}")
        if self.err_mode not in ERR_MODES:
            raise ValueError(f"--err-mode must be one of {ERR_MODES}")
        if self.compress_grad not in ("compress", "None", "none"):
            # the reference deadlocks on anything but the two magic strings (baseline_master.py:92-96)
            raise ValueError("--compress-grad must be 'compress' or 'None'")
        if self.approach == "cyclic" and self.num_workers < 2 * self.worker_fail + 1:
            raise ValueError("cyclic code needs num_workers >= 2*worker_fail + 1")
        if self.approach == "cyclic" and 2 * self.worker_fail + 1 > 8:
            raise ValueError("cyclic code: redundancy 2*worker_fail + 1 is limited to 8 (DRC_MAX_R)")
        if self.approach in ("maj_vote", "detox") and self.num_workers >= self.group_size > 0:
            # all remainder workers join the last group (codes/repetition.py): it can hold up to 2r-1 members, the vote kernel 8
            largest = self.group_size + self.num_workers % self.group_size
            if largest > 8:
                raise ValueError(f"repetition code: the last group would have {largest} members (num_workers % group_size "
                                 f"remainder joins it); the vote kernel handles at most 8 (DRC_MAX_R) -- pick a group size that "
                                 f"divides num_workers more evenly")
        if self.no_cuda:
            self.transport = "gloo"
        self._check_sign_vote()
        rules.check(self)
        if self.compress and self.transport == "nvl" and self.err_mode == "omniscient":
            raise ValueError("--err-mode omniscient reads the honest slots in PS memory while they arrive; with --compress-grad "
                             "compress they only exist after the PS unpacked them -- pass --compress-grad None")
        if self.compress and self.transport == "nccl_flat":
            raise ValueError("--transport nccl_flat is the uncompressed library comparator: pass --compress-grad None")
        self._check_ps_attack()
        self._check_worker_momentum()
        self._check_centered_clip()
        self._check_scope()
        self._check_bucketing()
        self._check_dirichlet()
        self._check_arc()
        if self.transport == "gloo":
            self.dtype = "fp32"
            self.cuda_graphs = False
        return self

    def _check_ps_attack(self) -> None:
        """--err-mode alie | minmax | ipm | mimic: the PS replaces the liars' slots with a row built from the honest slots."""
        from .codes.adversary import PS_ATTACKS, alie_s
        if self.attack_z is not None and self.err_mode != "alie":
            raise ValueError(f"--attack-z sets ALIE's z: it needs --err-mode alie (got --err-mode {self.err_mode})")
        if self.attack_eps is not None and self.err_mode != "ipm":
            raise ValueError(f"--attack-eps sets IPM's eps: it needs --err-mode ipm (got --err-mode {self.err_mode})")
        if self.attack_eps is not None and not (math.isfinite(self.attack_eps) and self.attack_eps > 0):
            raise ValueError(f"--attack-eps must be a finite eps > 0 (got {self.attack_eps}): the liars send -eps times the "
                             f"honest mean")
        if self.mimic_warmup is not None and self.err_mode != "mimic":
            raise ValueError(f"--mimic-warmup sets how many steps mimic learns its direction: it needs --err-mode mimic (got "
                             f"--err-mode {self.err_mode})")
        if self.mimic_warmup is not None and self.mimic_warmup < 0:
            raise ValueError(f"--mimic-warmup must be >= 0 steps (got {self.mimic_warmup}; 0 mimics along the random starting "
                             f"direction)")
        if self.err_mode not in PS_ATTACKS:
            return
        m = self.err_mode
        if self.approach == "cyclic":
            raise ValueError(f"--err-mode {m} builds a real gradient row from the honest ones; the cyclic code's slots hold complex "
                             f"codewords, so it has no meaning there -- use another --approach or --err-mode")
        if self.transport == "nccl_flat":
            raise ValueError(f"--transport nccl_flat implements the rev_grad and constant attacks only (got --err-mode {m})")
        if self.worker_fail >= self.num_workers:
            raise ValueError(f"--err-mode {m} builds the liars' row from the honest workers: it needs worker_fail < num_workers "
                             f"(got {self.worker_fail} of {self.num_workers})")
        if self.transport == "nvl" and self.num_workers > rules.ROBUST_MAXP:
            raise ValueError(f"--err-mode {m} on the nvl transport handles at most {rules.ROBUST_MAXP} workers (got "
                             f"{self.num_workers}); use --transport nccl for more")
        if m == "alie" and self.attack_z is None and alie_s(self.num_workers, self.worker_fail) < 1:
            raise ValueError(f"--err-mode alie: z_max = Phi^-1((P - s) / P) with s = floor(P/2 + 1) - f is undefined for "
                             f"{self.num_workers} workers and worker_fail {self.worker_fail} (s < 1); pass --attack-z")

    def _check_worker_momentum(self) -> None:
        """--worker-momentum beta: every worker keeps its own momentum and pushes it in place of its gradient."""
        beta = self.worker_momentum
        if not 0.0 <= beta < 1.0:
            raise ValueError(f"--worker-momentum must lie in [0, 1) (0 = off; got {beta}): at 1 the gradient would never enter "
                             f"the state")
        if beta == 0.0:
            return
        if self.approach == "cyclic":
            raise ValueError("--worker-momentum has no meaning under --approach cyclic: its decode recovers the exact sum of the "
                             "gradients, so worker momentum would only re-derive the PS momentum (--momentum), and the codeword "
                             "would need complex state")
        if self.transport == "nccl_flat":
            raise ValueError("--transport nccl_flat pushes the raw gradient buckets and keeps no worker state: use "
                             "--transport nvl or nccl for --worker-momentum")
        if self.err_mode == "omniscient":
            raise ValueError("--err-mode omniscient replaces the liars' push with a row read from the PS, so their momentum "
                             "could never advance: pick another --err-mode for --worker-momentum")

    def _check_centered_clip(self) -> None:
        """--mode centered_clip --clip-tau tau: the PS clips every row's distance to last step's aggregate at tau, per tensor."""
        cc = self.mode == "centered_clip"
        if self.clip_tau is not None and not (cc and self.approach in ("baseline", "detox")):
            raise ValueError(f"--clip-tau sets centered clipping's radius: it needs --approach baseline | detox with --mode "
                             f"centered_clip (got --approach {self.approach} --mode {self.mode})")
        if not cc:
            return
        if self.approach not in ("baseline", "detox"):
            raise ValueError(f"--mode centered_clip runs under --approach baseline (over the workers) or detox (over the group "
                             f"winners), got --approach {self.approach}")
        if self.clip_tau is None or not (math.isfinite(self.clip_tau) and self.clip_tau > 0):
            raise ValueError(f"--mode centered_clip needs --clip-tau, a finite radius > 0 (got {self.clip_tau}): tau is in the "
                             f"gradient's own units, per tensor, so no default would mean anything")

    def _check_sign_vote(self) -> None:
        """--mode sign_vote: every worker sends one bit per coordinate (its sign) and the PS takes the coordinate-wise majority."""
        if self.mode != "sign_vote":
            return
        if self.approach != "baseline":
            raise ValueError(f"--mode sign_vote votes over the signs of the P workers' rows: use --approach baseline (got "
                             f"--approach {self.approach})")
        if self.err_mode in ("omniscient", "alie", "minmax", "ipm", "mimic"):
            raise ValueError(f"--err-mode {self.err_mode} builds a real-valued row from the honest workers' fp32 slots, and the sign "
                             f"wire has none: use --err-mode rev_grad | constant | random | none with --mode sign_vote")
        if self.compress:
            raise ValueError("--mode sign_vote sends 1-bit words of signs, which the lossless codec cannot shrink: pass "
                             "--compress-grad None")

    def _check_scope(self) -> None:
        """--rule-scope / --attack-scope model: the rule's distances, or min-max's gamma and Dmax, over the whole model."""
        for flag, v in (("--rule-scope", self.rule_scope), ("--attack-scope", self.attack_scope)):
            if v not in SCOPES:
                raise ValueError(f"{flag} must be one of {SCOPES}, got {v!r}")
        if self.attack_scope == "model" and self.err_mode != "minmax":
            raise ValueError(f"--attack-scope model sets one gamma for the whole model: it needs --err-mode minmax (got --err-mode "
                             f"{self.err_mode}; alie is coordinate-wise, so the scope would change nothing)")
        if self.rule_scope == "tensor":
            return
        if not (self.approach == "nnm" or (self.approach in ("baseline", "detox") and self.mode in DISTANCE_MODES)):
            raise ValueError(f"--rule-scope model applies to the rules that measure distances between rows (--mode "
                             f"{' | '.join(DISTANCE_MODES)} under baseline or detox, and every --approach nnm mode); --approach "
                             f"{self.approach} --mode {self.mode} is coordinate-wise, so the scope would change nothing")

    def _check_bucketing(self) -> None:
        """--bucketing s: each step the PS permutes the P worker slots at random, averages them in worker buckets of s and runs
        ``--mode`` on the nb = ceil(P / s) bucket means, with the rule's bound over nb rows (one liar spoils one bucket)."""
        if self.bucketing != 0 and self.approach != "baseline":
            raise ValueError(f"--bucketing averages the raw worker rows before the rule: use --approach baseline (got --approach "
                             f"{self.approach})")

    def _check_dirichlet(self) -> None:
        """--dirichlet-alpha a: each data holder (a worker, or a repetition group) draws from its own shard, whose class shares
        follow Dirichlet(a)."""
        a = self.dirichlet_alpha
        if a is None:
            return
        if not (math.isfinite(a) and a > 0):
            raise ValueError(f"--dirichlet-alpha must be a finite concentration > 0 (got {a}); leave it unset for IID data")
        if self.approach == "cyclic":
            raise ValueError("--dirichlet-alpha gives every data holder its own shard; under --approach cyclic the workers split "
                             "one global batch, so there is no holder to give it to")

    def _check_arc(self) -> None:
        """--arc tensor | model: before the row source and the rule, the PS clips the k = floor(2 f (P - f) / P) worker slots
        of largest norm to the norm of the next largest (per tensor, or over the whole model)."""
        if self.arc is None:
            return
        if self.arc not in SCOPES:
            raise ValueError(f"--arc must be one of {SCOPES} (or unset for no clipping), got {self.arc!r}")
        if self.approach == "cyclic":
            raise ValueError("--arc scales real gradient rows; the cyclic code's slots hold complex codewords, so it has no "
                             "meaning there -- use another --approach or drop --arc")
        if self.mode == "sign_vote":
            raise ValueError("--arc multiplies a row by a positive factor, which changes none of its signs: --mode sign_vote "
                             "would vote exactly as without it -- drop --arc")
        if self.transport == "nccl_flat":
            raise ValueError("--transport nccl_flat runs the plain mean and the vote on the raw buckets only; use --transport "
                             "nvl or nccl for --arc")
        if not 0 <= self.worker_fail <= self.num_workers:
            raise ValueError(f"--arc clips floor(2 f (P - f) / P) rows with f = --worker-fail: it needs 0 <= worker_fail <= "
                             f"num_workers (got {self.worker_fail} of {self.num_workers})")
        if self.transport == "nvl" and self.num_workers > rules.ROBUST_MAXP:
            raise ValueError(f"--arc on the nvl transport handles at most {rules.ROBUST_MAXP} workers (its norm pass holds the "
                             f"rows in registers; got {self.num_workers}); use --transport nccl for more")

    @property
    def ipm_eps(self) -> float:
        """eps of the IPM attack: --attack-eps, else the repository's default (codes.adversary.IPM_EPS)."""
        from .codes.adversary import IPM_EPS
        return float(self.attack_eps) if self.attack_eps is not None else IPM_EPS

    @property
    def mimic_w(self) -> int:
        """Mimic's warm-up steps W: --mimic-warmup, else the repository's default (codes.adversary.MIMIC_WARMUP)."""
        from .codes.adversary import MIMIC_WARMUP
        return int(self.mimic_warmup) if self.mimic_warmup is not None else MIMIC_WARMUP

    @property
    def alie_z(self) -> float:
        """z of the ALIE attack: --attack-z, else z_max(num_workers, worker_fail)."""
        from .codes.adversary import alie_z_max
        return float(self.attack_z) if self.attack_z is not None else alie_z_max(self.num_workers, self.worker_fail)

    @property
    def compress(self) -> bool:
        return self.compress_grad == "compress"

    @property
    def redundancy(self) -> int:
        if self.approach == "cyclic":
            return 2 * self.worker_fail + 1
        if self.approach in ("maj_vote", "detox"):
            return self.group_size
        return 1

    @property
    def num_groups(self) -> int:
        """Repetition groups G of ``maj_vote`` / ``detox``: num_workers // group_size (the remainder joins the last group)."""
        return self.num_workers // min(self.group_size, self.num_workers)

    @property
    def captured_group_bound(self) -> int:
        """DETOX's b_G = worker_fail // ceil(group_size / 2): a group of r >= group_size members returns a liar's row only when
        at least (r + 1) // 2 of them lie, so the liars capture at most b_G groups."""
        return self.worker_fail // ((self.group_size + 1) // 2)

    @property
    def attack_magnitude(self) -> float:
        return -100.0 * float(self.adversarial)

    def to_dict(self) -> dict:
        return asdict(self)


def add_fit_args(parser: argparse.ArgumentParser) -> argparse.ArgumentParser:
    """Same flag names/defaults as the reference's ``add_fit_args`` plus the additive ones."""
    d = JobConfig()
    a = parser.add_argument
    a("--batch-size", type=int, default=d.batch_size, help="per-worker batch size")
    a("--test-batch-size", type=int, default=d.test_batch_size)
    a("--max-steps", type=int, default=d.max_steps)
    a("--epochs", type=int, default=d.epochs)
    a("--lr", type=float, default=d.lr)
    a("--momentum", type=float, default=d.momentum)
    a("--no-cuda", action="store_true", default=False, help="run on CPU over the Gloo transport")
    a("--seed", type=int, default=d.seed)
    a("--log-interval", type=int, default=d.log_interval)
    a("--worker-streams", type=int, default=d.worker_streams,
      help="logical workers that share one GPU are issued round-robin on this many CUDA streams (small layers of "
           "different workers overlap); 1 = serial")
    a("--debug-checksum", action="store_true", default=d.debug_checksum,
      help="transport self-check: each worker re-encodes its gradient into a local buffer and the PS compares 64-bit "
           "checksums with what arrived in its slots, every step (eager mode, nvl transport)")
    a("--profile-phases", action="store_true", default=d.profile_phases,
      help="time the reference's phases (Comm / Comp / Encode / Method / Update) with CUDA events each step; eager mode")
    a("--network", type=str, default=d.network)
    a("--mode", type=str, default=d.mode,
      help="normal | geometric_median | krum | coordinate_median | trimmed_mean | multi_krum | bulyan (baseline); normal | "
           "maj_vote (maj_vote); coordinate_median | trimmed_mean | multi_krum | geometric_median | bulyan (detox: the rule "
           "across the group winners).  trimmed_mean drops --worker-fail values at each end of every coordinate (detox: b_G = "
           "worker_fail // ceil(group_size / 2)); multi_krum averages the num_workers - worker_fail workers (detox: G - b_G group "
           "winners) with the lowest Krum scores; bulyan picks num_workers - 2 worker_fail workers by repeated Krum, then "
           "averages, per coordinate, the num_workers - 4 worker_fail picked values nearest their median (needs num_workers >= "
           "4 worker_fail + 3; detox: G and b_G); coordinate_median | trimmed_mean | krum | multi_krum | geometric_median | "
           "bulyan (nnm: the rule applied to the mixed rows, with --worker-fail as f).  centered_clip (baseline, detox; needs "
           "--clip-tau): one step of centered clipping around last step's aggregate v, g = v + (1/n) sum_i (x_i - v) min(1, "
           "tau / ||x_i - v||) per tensor, and g becomes the next v.  sign_vote (baseline; needs --compress-grad None): signSGD "
           "with majority vote, every worker sends one bit per coordinate (its sign) and the PS applies the coordinate-wise "
           "majority sign (+1 / -1, 0 on a tie) through the optimizer, so --lr is the sign step; with --worker-momentum 0.9 "
           "--momentum 0 it is Signum")
    a("--dataset", type=str, default=d.dataset)
    a("--comm-type", type=str, default=d.comm_type)
    a("--err-mode", type=str, default=d.err_mode,
      help="rev_grad | constant | random | omniscient | alie | minmax | ipm | mimic | none.  alie (A Little Is Enough) and minmax "
           "(min-max, inverse-std direction) are applied by the PS per tensor from the honest workers' mean and standard "
           "deviation; ipm (inner-product manipulation): the liars send -eps times the honest mean; mimic: every liar sends a "
           "copy of the honest worker furthest along a direction the PS learns over the first --mimic-warmup steps")
    a("--attack-z", type=float, default=None,
      help="--err-mode alie: the liars send mu - z * sigma (default: z_max = Phi^-1((P - s) / P), s = floor(P/2 + 1) - f)")
    a("--attack-eps", type=float, default=None,
      help="--err-mode ipm: the liars send -eps * mu, mu the honest mean (default 0.1, this repository's choice)")
    a("--mimic-warmup", type=int, default=None,
      help="--err-mode mimic: the first W steps learn the top principal direction of the honest gradients by an online power "
           "iteration (default 20, this repository's choice; 0: a fixed random direction)")
    a("--worker-momentum", type=float, default=d.worker_momentum,
      help="beta of worker-side momentum (0 = off): every worker keeps m <- beta m + (1 - beta) g and pushes m instead of its "
           "gradient, which shrinks the honest workers' spread before the robust rule sees it (Karimireddy et al. 2021, El "
           "Mhamdi et al. 2021).  --momentum still applies at the PS on top; the papers' recipe is --worker-momentum 0.9 "
           "--momentum 0")
    a("--clip-tau", type=float, default=None,
      help="--mode centered_clip: the clipping radius tau, per tensor (--rule-scope model: of the whole model's norm), in the "
           "gradient's own units (required; the papers' recipe pairs it with --worker-momentum 0.9 --momentum 0)")
    a("--rule-scope", type=str, default=d.rule_scope, choices=SCOPES,
      help="tensor (default): the distance-based rules (krum, multi_krum, geometric_median, bulyan's selection, centered_clip's "
           "norm, every --approach nnm neighbourhood) measure distances per parameter tensor and may choose differently in each; "
           "model: over the flattened model, one choice for every tensor, as in the papers")
    a("--attack-scope", type=str, default=d.attack_scope, choices=SCOPES,
      help="--err-mode minmax: tensor (default) solves gamma and Dmax per parameter tensor; model: one gamma and one Dmax over "
           "the flattened model, as in the NDSS paper")
    a("--bucketing", type=int, default=d.bucketing,
      help="s (0 = off; --approach baseline): every step the PS permutes the workers at random, averages them in worker buckets "
           "of s and runs --mode (coordinate_median | trimmed_mean | krum | multi_krum | geometric_median | centered_clip) on "
           "the ceil(P / s) bucket means, with --worker-fail as f (Karimireddy, He and Jaggi, ICLR 2022)")
    a("--dirichlet-alpha", type=float, default=None,
      help="heterogeneous data: every data holder (a worker; a group under maj_vote / detox) samples from its own shard, whose "
           "class shares are drawn from Dirichlet(alpha) (small alpha: few classes per holder).  Unset: every worker samples "
           "the whole dataset")
    a("--arc", type=str, default=None, choices=SCOPES,
      help="adaptive robust clipping (Allouah et al. 2024; every approach but cyclic, not with --mode sign_vote): before the "
           "row source and the rule, the PS clips the k = floor(2 f (P - f) / P) worker rows of largest norm (f = --worker-fail) "
           "to the norm of the next largest.  tensor: one norm per parameter tensor; model: one norm per worker over the whole "
           "model, as in the paper.  No parameter of its own; with f = 0 it does nothing")
    a("--approach", type=str, default=d.approach,
      help="baseline | maj_vote | cyclic | detox (majority vote inside each repetition group, then --mode across the G group "
           "winners) | nnm (nearest-neighbour mixing: every worker's row is replaced, per tensor, by the mean of its "
           "num_workers - worker_fail nearest rows, itself included, then --mode runs on the mixed rows)")
    a("--num-aggregate", type=int, default=d.num_aggregate)
    a("--eval-freq", type=int, default=d.eval_freq)
    a("--train-dir", type=str, default=d.train_dir)
    a("--adversarial", type=int, default=d.adversarial, help="attack magnitude multiplier (x -100)")
    a("--worker-fail", type=int, default=d.worker_fail)
    a("--group-size", type=int, default=d.group_size)
    a("--compress-grad", type=str, default=d.compress_grad)
    a("--checkpoint-step", type=int, default=d.checkpoint_step)
    a("--num-workers", type=int, default=0, help="logical workers P (default world_size-1)")
    a("--transport", type=str, default=d.transport, choices=TRANSPORTS)
    a("--dtype", type=str, default=d.dtype, choices=("bf16", "fp32"))
    a("--no-cuda-graphs", dest="cuda_graphs", action="store_false", default=True)
    a("--weight-decay", type=float, default=0.0)
    a("--nesterov", action="store_true", default=False)
    a("--dampening", type=float, default=0.0)
    a("--optimizer", type=str, default="sgd", choices=("sgd", "adam"))
    a("--amsgrad", action="store_true", default=False, help="AMSGrad variant of --optimizer adam (reference: adam_modified.py:16)")
    a("--data-root", type=str, default=d.data_root)
    a("--synthetic-size", type=int, default=d.synthetic_size)
    a("--augment", action="store_true", default=False)
    a("--data-on-device", action="store_true", default=False)
    a("--metrics-file", type=str, default=None)
    a("--multicast", type=str, default="auto", choices=("auto", "on", "off"))
    a("--wgrad-stream", type=str, default=d.wgrad_stream, choices=("auto", "on", "off"))
    a("--spin-timeout-s", type=float, default=d.spin_timeout_s)
    a("--ps-stream", action="store_true", default=d.ps_stream,
      help="co-located PS on its own stream inside the captured graph (set CUDA_DEVICE_MAX_CONNECTIONS=32)")
    a("--num-classes", type=int, default=10)
    a("--no-overlap-push", dest="overlap_push", action="store_false", default=True)
    return parser


def config_from_args(args: argparse.Namespace) -> JobConfig:
    fields = JobConfig.__dataclass_fields__
    return JobConfig(**{k: v for k, v in vars(args).items() if k in fields})
