"""Time the fused PS update kernel alone (csrc/cuda/aggregate_update.cu): mode 0, the mean of P gradient rows, against mode 3,
the coordinate-wise trimmed mean and median, on the ResNet-18 (CIFAR) parameter arena.  With a G-row winner table (DETOX: the
majority vote's winner slot per group and tensor, here drawn at random from groups of 3) it times mode 0, the average of the G
winners that ``--approach maj_vote`` applies, against mode 3 over the same G rows: the median and the b_G-trimmed mean.

Each call reads the P x D fp32 gradient slab once and reads + writes the fp32 parameters and momentum (SGD-momentum, no
broadcast destinations).  Timed with CUDA events over --iters back-to-back launches; the rules alternate over --rounds and the
median round is reported.  Bandwidth is the slab bytes (P * D * 4) per microsecond, also as a share of the H100 SXM data-sheet
HBM3 bandwidth of 3.35 TB/s (3.35e6 bytes/us); ``total_bytes_per_us`` adds the 16 * D bytes of parameter / momentum traffic.

With --attack-workers it also times the PS-side attacks alone (csrc/cuda/attack.cu) on the same arena with --attack-fail liar
slots: ALIE (one pass: reads the honest rows, writes the liar rows) and min-max (stats pass + per-tensor solve + write pass).
``bytes`` counts the HBM traffic the algorithm needs: ALIE (n_h + f) * D * 4; min-max n_h * D * 4 read, 2 * D * 4 of mu / sigma
written and read again, the fp64 per-tile partials twice, and f * D * 4 written.

With --bulyan-workers it times Bulyan against multi-Krum on the same arena, f = (P - 3) // 4 (P = 7: f = 1, P = 15: f = 3),
each launch on its own and as the chain the PS runs after the last bucket: the pair-distance pass (shared), ``bulyan_select``
(theta = P - 2f rounds of Krum, csrc/cuda/robust.cu) against ``krum_select`` with m = P - f, and the update kernel's mode 4
(the beta = theta - 2f values nearest the coordinate median of theta rows) against mode 0 over the P - f multi-Krum rows and
mode 3 over the same theta rows (the f-trimmed mean: the same sort, without the median and the window walk).

With --nnm-workers it times nearest-neighbour mixing (NNM) on the same arena, f = (P - 3) // 4 (P = 7: f = 1, P = 15: f = 3):
``nnm_mix`` (neighbour masks plus the mixed rows' distance table, csrc/cuda/robust.cu) and ``nnm_fold`` (a multi-Krum choice over
the mixed rows as raw-slot weights) alone; the update kernel's mode 3 (coordinate-wise median) and mode 4 (Bulyan's coordinate
stage) with mixing against the same modes without it, over the same rows; and the whole chains the PS runs after the last
bucket -- NNM + multi-Krum and NNM + Bulyan against plain multi-Krum and plain Bulyan.

With --cc-workers it times centered clipping over P rows on the same arena: ``centered_clip_dist`` (the fp64 per-tile partials
of the P row-to-centre distances, csrc/cuda/clip.cu), ``centered_clip_weights`` (the per-tensor fold and the weights), the update
kernel's mode 5 and the whole chain, against mode 0 (the mean) over the same rows.  ``bytes`` counts the HBM traffic the algorithm
needs: the distances read the P rows and the centre, (P + 1) * D * 4, and write the partials, ntiles * P * 8; the weights read the
partials and write T * P * 4; mode 5 reads the rows and the centre and writes the centre, (P + 2) * D * 4, and mode 0 reads the
rows, P * D * 4, both plus the 16 * D bytes of parameter / momentum traffic.

    python tools/bench_aggregate.py [--workers 7 16] [--groups 3 5 8] [--attack-workers 7 15] [--bulyan-workers 7 15]
                                    [--nnm-workers 7 15] [--cc-workers 7 15] [--iters 200] [--rounds 3] [--out FILE]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_US = 3.35e6


def gpu_info() -> dict:
    import torch
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        info["power_limit_and_max_sm_clock"] = q.stdout.strip()
    except Exception as e:          # the measurement still stands; the card's limits are then unknown
        info["power_limit_and_max_sm_clock"] = f"unavailable: {e}"
    return info


def attack_arm(K, L, P, f, iters, rounds, dev) -> list:
    import torch
    from draco_b200.codes.adversary import alie_z_max
    D, nh = L.total, P - f
    slab = torch.randn(P, D, device=dev) * 1e-3
    bm = torch.tensor([(1 << f) - 1], dtype=torch.int32, device=dev)          # slots 0..f-1 lie
    step = torch.ones(1, dtype=torch.int64, device=dev)
    ws = K.AttackWorkspace(L, P, dev)
    Q = ws.partials.shape[1]
    arms = {"alie": (5, (nh + f) * D * 4), "minmax": (6, (nh + 4 + f) * D * 4 + 2 * L.ntiles * Q * 8)}

    def launch(mode):
        K.ps_attack(L, slab, D, P, mode, adv_bitmap=bm, adv_len=1, step_ptr=step, z=alie_z_max(P, f), ws=ws)

    for mode, _ in arms.values():
        for _ in range(20):
            launch(mode)
    torch.cuda.synchronize()
    times = {name: [] for name in arms}
    for _ in range(rounds):
        for name, (mode, _) in arms.items():
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            for _ in range(iters):
                launch(mode)
            e.record()
            e.synchronize()
            times[name].append(s.elapsed_time(e) * 1e3 / iters)
    out = []
    for name, ts in times.items():
        us, nbytes = sorted(ts)[len(ts) // 2], arms[name][1]
        out.append({"P": P, "liars": f, "attack": name, "us_per_call": round(us, 2), "us_rounds": [round(t, 2) for t in ts],
                    "bytes": nbytes, "bytes_per_us": round(nbytes / us), "share_of_3.35TBps": round(nbytes / us / HBM_BYTES_PER_US, 3)})
    return out


def bulyan_arm(K, L, P, iters, rounds, dev, update) -> list:
    """Bulyan's three launches against multi-Krum's, timed alone and chained (see the module docstring)."""
    import ctypes as C

    import torch
    from draco_b200 import _native as N
    f = (P - 3) // 4
    theta, m, T, D = P - 2 * f, P - f, L.ntensors, L.total
    slab = torch.randn(P, D, device=dev) * 1e-3
    pair = torch.zeros(T, P * (P - 1) // 2, dtype=torch.float64, device=dev)
    sel_b = torch.zeros(theta, T, dtype=torch.int32, device=dev)
    sel_k = torch.zeros(m, T, dtype=torch.int32, device=dev)
    K.bulyan_select(L, slab, D, P, f, pair, sel_b)
    K.krum_select(L, slab, D, P, f, pair, sel_k, m=m)
    lib, tv = N.cuda(), L.tile_view(dev)
    pa = N.PairDistArgs(slab.data_ptr(), D, P, tv, pair.data_ptr(), None)
    ba = N.BulyanSelectArgs(pair.data_ptr(), T, P, f, sel_b.data_ptr(), None)
    ka = N.KrumSelectArgs(pair.data_ptr(), T, P, f, m, sel_k.data_ptr(), None)
    grid = K.stream_grid(L, 4)
    arms = {
        "pair_dist": lambda: lib.drc_pair_dist(C.byref(pa), grid, K._stream()),
        "bulyan_select": lambda: lib.drc_bulyan_select(C.byref(ba), K._stream()),
        "krum_select_m": lambda: lib.drc_krum_select(C.byref(ka), K._stream()),
        "mode4_near_median": lambda: update(slab, dict(K=theta, scale=1.0 / (theta - 2 * f), near_median=f, select=sel_b)),
        "mode3_trimmed_theta": lambda: update(slab, dict(K=theta, scale=1.0 / (theta - 2 * f), trim=f, select=sel_b)),
        "mode0_multi_krum": lambda: update(slab, dict(K=m, scale=1.0 / m, select=sel_k)),
        "bulyan_chain": lambda: (K.bulyan_select(L, slab, D, P, f, pair, sel_b),
                                 update(slab, dict(K=theta, scale=1.0 / (theta - 2 * f), near_median=f, select=sel_b))),
        "multi_krum_chain": lambda: (K.krum_select(L, slab, D, P, f, pair, sel_k, m=m),
                                     update(slab, dict(K=m, scale=1.0 / m, select=sel_k))),
    }
    for fn in arms.values():
        for _ in range(20):
            fn()
    torch.cuda.synchronize()
    times = {name: [] for name in arms}
    for _ in range(rounds):
        for name, fn in arms.items():
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            for _ in range(iters):
                fn()
            e.record()
            e.synchronize()
            times[name].append(s.elapsed_time(e) * 1e3 / iters)
    pair.zero_()
    return [{"P": P, "f": f, "theta": theta, "arm": name, "us_per_call": round(sorted(ts)[len(ts) // 2], 2),
             "us_rounds": [round(t, 2) for t in ts]} for name, ts in times.items()]


def nnm_arm(K, L, P, iters, rounds, dev, update) -> list:
    """NNM's launches alone and chained, against the unmixed rules (see the module docstring)."""
    import ctypes as C

    import torch
    from draco_b200 import _native as N
    f = (P - 3) // 4
    theta, m, T, D = P - 2 * f, P - f, L.ntensors, L.total
    med = (P - 1) // 2
    slab = torch.randn(P, D, device=dev) * 1e-3
    pair = torch.zeros(T, P * (P - 1) // 2, dtype=torch.float64, device=dev)
    mix = torch.zeros(P, T, dtype=torch.int32, device=dev)
    sel_b = torch.zeros(theta, T, dtype=torch.int32, device=dev)
    sel_k = torch.zeros(m, T, dtype=torch.int32, device=dev)
    w_raw = torch.zeros(T, P, device=dev)
    K.nnm_mix(L, slab, D, P, f, pair, mix, mixed_out=True)
    K.bulyan_select(L, slab, D, P, f, pair, sel_b, filled=True)
    lib = N.cuda()
    na = N.NnmMixArgs(pair.data_ptr(), T, P, f, mix.data_ptr(), 0)     # alone: zeroes the (already zero) table after the masks
    na_out = N.NnmMixArgs(pair.data_ptr(), T, P, f, mix.data_ptr(), 1)
    fa = N.NnmFoldArgs(mix.data_ptr(), T, P, f, sel_k.data_ptr(), m, None, w_raw.data_ptr())

    def mix_then_zero():                                                # the mixed table, then zeroed as a select kernel would
        lib.drc_nnm_mix(C.byref(na_out), K._stream())
        pair.zero_()
    arms = {
        "nnm_mix_masks": lambda: lib.drc_nnm_mix(C.byref(na), K._stream()),
        "nnm_mix_table_plus_zero": mix_then_zero,
        "table_zero_alone": pair.zero_,
        "nnm_fold_select": lambda: lib.drc_nnm_fold(C.byref(fa), K._stream()),
        "mode3_median_mixed": lambda: update(slab, dict(K=P, scale=1.0 / (P - 2 * med), trim=med, mix=mix, mix_f=f)),
        "mode3_median": lambda: update(slab, dict(K=P, scale=1.0 / (P - 2 * med), trim=med)),
        "mode4_near_median_mixed": lambda: update(slab, dict(K=theta, scale=1.0 / (theta - 2 * f), near_median=f, select=sel_b,
                                                             mix=mix, mix_f=f)),
        "mode4_near_median": lambda: update(slab, dict(K=theta, scale=1.0 / (theta - 2 * f), near_median=f, select=sel_b)),
        "nnm_multi_krum_chain": lambda: (K.nnm_mix(L, slab, D, P, f, pair, mix, mixed_out=True),
                                         K.krum_select(L, slab, D, P, f, pair, sel_k, m=m, filled=True),
                                         K.nnm_fold(L, P, f, mix, w_raw, select=sel_k, m=m),
                                         update(slab, dict(K=P, scale=1.0, weights=w_raw))),
        "multi_krum_chain": lambda: (K.krum_select(L, slab, D, P, f, pair, sel_k, m=m),
                                     update(slab, dict(K=m, scale=1.0 / m, select=sel_k))),
        "nnm_median_chain": lambda: (K.nnm_mix(L, slab, D, P, f, pair, mix, mixed_out=False),
                                     update(slab, dict(K=P, scale=1.0 / (P - 2 * med), trim=med, mix=mix, mix_f=f))),
        "nnm_bulyan_chain": lambda: (K.nnm_mix(L, slab, D, P, f, pair, mix, mixed_out=True),
                                     K.bulyan_select(L, slab, D, P, f, pair, sel_b, filled=True),
                                     update(slab, dict(K=theta, scale=1.0 / (theta - 2 * f), near_median=f, select=sel_b, mix=mix,
                                                       mix_f=f))),
        "bulyan_chain": lambda: (K.bulyan_select(L, slab, D, P, f, pair, sel_b),
                                 update(slab, dict(K=theta, scale=1.0 / (theta - 2 * f), near_median=f, select=sel_b))),
    }
    for fn in arms.values():
        for _ in range(20):
            fn()
    torch.cuda.synchronize()
    times = {name: [] for name in arms}
    for _ in range(rounds):
        for name, fn in arms.items():
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            for _ in range(iters):
                fn()
            e.record()
            e.synchronize()
            times[name].append(s.elapsed_time(e) * 1e3 / iters)
    return [{"P": P, "f": f, "theta": theta, "arm": name, "us_per_call": round(sorted(ts)[len(ts) // 2], 2),
             "us_rounds": [round(t, 2) for t in ts]} for name, ts in times.items()]


def cc_arm(K, L, P, iters, rounds, dev, update) -> list:
    """Centered clipping's launches alone and chained, against mode 0 over the same rows (see the module docstring)."""
    import torch
    T, D, nt = L.ntensors, L.total, L.ntiles
    slab = torch.randn(P, D, device=dev) * 1e-3
    center = torch.zeros(D, device=dev)
    partials = torch.zeros(nt, P, dtype=torch.float64, device=dev)
    weights = torch.zeros(T, P, dtype=torch.float32, device=dev)
    tau = 1e-2                                                          # every row is read: no weight is zero
    K.centered_clip_dist(L, slab, D, P, center, partials)
    K.centered_clip_weights(L, P, tau, partials, weights)

    def mode5():
        update(slab, dict(K=P, center=center, weights=weights), cc=True)
    arms = {
        "cc_dist": (lambda: K.centered_clip_dist(L, slab, D, P, center, partials), (P + 1) * D * 4 + nt * P * 8),
        "cc_weights": (lambda: K.centered_clip_weights(L, P, tau, partials, weights), nt * P * 8 + T * P * 4),
        "mode5_centered_clip": (mode5, (P + 2) * D * 4 + 16 * D),
        "cc_chain": (lambda: (K.centered_clip_dist(L, slab, D, P, center, partials),
                              K.centered_clip_weights(L, P, tau, partials, weights), mode5()),
                     (2 * P + 3) * D * 4 + 2 * nt * P * 8 + T * P * 4 + 16 * D),
        "mode0_mean": (lambda: update(slab, dict(K=P, scale=1.0 / P)), P * D * 4 + 16 * D),
    }
    for fn, _ in arms.values():
        for _ in range(20):
            fn()
    torch.cuda.synchronize()
    times = {name: [] for name in arms}
    for _ in range(rounds):
        for name, (fn, _) in arms.items():
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            for _ in range(iters):
                fn()
            e.record()
            e.synchronize()
            times[name].append(s.elapsed_time(e) * 1e3 / iters)
    out = []
    for name, ts in times.items():
        us, nbytes = sorted(ts)[len(ts) // 2], arms[name][1]
        out.append({"P": P, "arm": name, "us_per_call": round(us, 2), "us_rounds": [round(t, 2) for t in ts], "bytes": nbytes,
                    "bytes_per_us": round(nbytes / us), "share_of_3.35TBps": round(nbytes / us / HBM_BYTES_PER_US, 3)})
    return out


def main() -> int:
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--workers", type=int, nargs="*", default=[7, 16])
    ap.add_argument("--trim", type=int, default=2, help="values dropped at each end by the trimmed mean (= --worker-fail)")
    ap.add_argument("--groups", type=int, nargs="*", default=[3, 5, 8], help="G of the winner-table rows (groups of 3 workers)")
    ap.add_argument("--group-trim", type=int, default=1, help="b_G of the DETOX trimmed mean (worker_fail 3, group size 3: 1)")
    ap.add_argument("--attack-workers", type=int, nargs="*", default=[], help="P of the ALIE / min-max kernel arm (none: skipped)")
    ap.add_argument("--attack-fail", type=int, default=3, help="liar slots of the attack arm")
    ap.add_argument("--bulyan-workers", type=int, nargs="*", default=[], help="P of the Bulyan / multi-Krum arm (none: skipped)")
    ap.add_argument("--nnm-workers", type=int, nargs="*", default=[], help="P of the NNM arm (none: skipped)")
    ap.add_argument("--cc-workers", type=int, nargs="*", default=[], help="P of the centered-clipping arm (none: skipped)")
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", type=str, default=None, help="also append the JSON lines to this file")
    a = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        print(json.dumps({"error": "no CUDA device visible"}))
        return 1
    from draco_b200 import JobConfig
    from draco_b200.models import build_model
    from draco_b200.ops import kernels as K
    from draco_b200.parallel.arena import ArenaLayout
    from draco_b200.parallel.ps import hyperparams_tensor

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    L = ArenaLayout.from_model(build_model("ResNet18"), bf16=True, channels_last=True)
    D = L.total
    hp = hyperparams_tensor(JobConfig(lr=0.01, momentum=0.9), dev)
    params = torch.zeros(D, device=dev)
    mom = torch.zeros(D, device=dev)
    step = torch.full((1,), 2, dtype=torch.int64, device=dev)
    cnt = torch.zeros(4, dtype=torch.int32, device=dev)
    lines = [dict(gpu_info(), arena="ResNet18/Cifar10", D=D, iters=a.iters, rounds=a.rounds)]
    cases = []
    for P in a.workers:
        cases.append((dict(P=P), P, {"mean": dict(K=P, scale=1.0 / P),
                                     f"trimmed_mean_b{a.trim}": dict(K=P, scale=1.0 / (P - 2 * a.trim), trim=a.trim),
                                     "median": dict(K=P, scale=1.0 / (P - 2 * ((P - 1) // 2)), trim=(P - 1) // 2)}))
    T = L.ntensors
    for G in a.groups:
        win = (torch.arange(G, device=dev)[:, None] * 3 + torch.randint(0, 3, (G, T), device=dev)).to(torch.int32).contiguous()
        b = a.group_trim
        cases.append((dict(G=G, P=3 * G), 3 * G, {"vote_mean": dict(K=G, scale=1.0 / G, select=win),
                                                  f"detox_trimmed_mean_b{b}": dict(K=G, scale=1.0 / (G - 2 * b), trim=b, select=win),
                                                  "detox_median": dict(K=G, scale=1.0 / (G - 2 * ((G - 1) // 2)), trim=(G - 1) // 2,
                                                                       select=win)}))
    for key, P, rules in cases:
        slab = torch.randn(P, D, device=dev) * 1e-3

        def launch(kw):
            K.aggregate_update(L, slab, D, params=params, momentum=mom, hp=hp, step_ptr=step, done_counter=cnt[0:1], **kw)

        for kw in rules.values():                                  # load the module, settle the clocks
            for _ in range(20):
                launch(kw)
        torch.cuda.synchronize()
        times = {name: [] for name in rules}
        for _ in range(a.rounds):
            for name, kw in rules.items():
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record()
                for _ in range(a.iters):
                    launch(kw)
                e.record()
                e.synchronize()
                times[name].append(s.elapsed_time(e) * 1e3 / a.iters)
        for name, ts in times.items():
            rows = rules[name]["K"]                                # rows read per coordinate: P, or the G winners
            slab_bytes = rows * D * 4
            us = sorted(ts)[len(ts) // 2]
            lines.append({**key, "rule": name, "mode": 3 if "trim" in rules[name] else 0, "us_per_call": round(us, 2),
                          "us_rounds": [round(t, 2) for t in ts], "slab_bytes": slab_bytes,
                          "slab_bytes_per_us": round(slab_bytes / us), "slab_share_of_3.35TBps": round(slab_bytes / us / HBM_BYTES_PER_US, 3),
                          "total_bytes_per_us": round((slab_bytes + 16 * D) / us)})
        del slab
    for P in a.attack_workers:
        lines += attack_arm(K, L, P, a.attack_fail, a.iters, a.rounds, dev)

    def update(slab, kw, cc=False):
        launcher = K.centered_clip_update if cc else K.aggregate_update
        launcher(L, slab, D, params=params, momentum=mom, hp=hp, step_ptr=step, done_counter=cnt[0:1], **kw)
    for P in a.bulyan_workers:
        lines += bulyan_arm(K, L, P, a.iters, a.rounds, dev, update)
    for P in a.nnm_workers:
        lines += nnm_arm(K, L, P, a.iters, a.rounds, dev, update)
    for P in a.cc_workers:
        lines += cc_arm(K, L, P, a.iters, a.rounds, dev, update)
    for ln in lines:
        print(json.dumps(ln), flush=True)
    if a.out:
        with open(a.out, "a") as fh:
            for ln in lines:
                fh.write(json.dumps(ln) + "\n")
    return 0


if __name__ == "__main__":
    sys.exit(main())
