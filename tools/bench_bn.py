"""BatchNorm kernels (csrc/cuda/bn_fused.cu) at every BatchNorm shape of ResNet-18 / CIFAR-10 at B = 128: the forward apply and the
backward reduce + apply, timed separately with CUDA events, for

* a single BatchNorm + ReLU layer with the ReLU mask read from the saved output y (``mask y``) and from the forward's bits
  (``mask bits``);
* a downsampling block's pair relu(bn2(c2) + bn_sc(s)) as two layers (``pair 2x``: y mask, shortcut output and masked gradient
  through memory) and as one pass each way (``pair 1x``).

Bytes are the minimum traffic of each variant, counted from the shapes below; bandwidth is reported as a share of the H100 SXM
data-sheet HBM3 bandwidth (3.35 TB/s).  Needs a GPU; there is no fallback.

    python tools/bench_bn.py [--iters 200] [--json out.json]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from draco_b200 import _native as N  # noqa: E402
from draco_b200.ops import norm  # noqa: E402

HBM_BPS = 3.35e12
B = 128
# (C, H = W, BatchNorm + ReLU layers of this shape outside the pairs, downsampling pairs of this shape): 14 + 3 pairs = 20 layers
SHAPES = [(64, 32, 5, 0), (128, 16, 3, 1), (256, 8, 3, 1), (512, 4, 3, 1)]
# bytes per element of each variant (bf16 tensors 2 B, ReLU bits 1/8 B)
BYTES = {
    "fwd mask y": 2 + 2,                        # x -> y
    "fwd mask bits": 2 + 2 + 1 / 8,             # x -> y, bits
    "bwd mask y": (2 + 2 + 2) + (2 + 2 + 2 + 2),             # reduce dy, x, y; apply dy, x, y -> dx
    "bwd mask bits": (2 + 2 + 1 / 8) + (2 + 2 + 1 / 8 + 2),  # reduce dy, x, bits; apply dy, x, bits -> dx
    "fwd pair 2x": (2 + 2) + (2 + 2 + 2),       # s -> y_sc; c2, y_sc -> y
    "fwd pair 1x": 2 + 2 + 2 + 1 / 8,           # c2, s -> y, bits
    "bwd pair 2x": (2 + 2 + 2) + (2 + 2 + 2 + 2 + 2) + (2 + 2) + (2 + 2 + 2),  # bn2 reduce, apply (dx, dres); bn_sc reduce, apply
    "bwd pair 1x": (2 + 2 + 2 + 1 / 8) + (2 + 2 + 2 + 1 / 8 + 2 + 2),          # reduce dy, c2, s, bits; apply -> dx, dxs
}


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def timed(fn, iters):
    for _ in range(10):
        fn()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) * 1e3 / iters            # us per call


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--json", type=str, default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_bn.py needs a GPU")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    lib, sms = norm._lib(), norm._sms(dev)
    st = torch.cuda.current_stream().cuda_stream
    cnt = norm._counter(dev)
    rows = []
    print(f"# BatchNorm kernels, ResNet-18 / CIFAR-10 shapes at B = {B} ({gpu_info()}), {a.iters} launches per number\n")
    print("| C x H x W | elements | variant | us | GB/s | share of 3.35 TB/s |\n|---|---:|---|---:|---:|---:|")
    for c, hw, n_layers, n_pairs in SHAPES:
        M = B * hw * hw
        g = torch.Generator(device=dev).manual_seed(c)

        def t():
            return torch.randn(B, c, hw, hw, device=dev, generator=g).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)

        x, s, dy = t(), t(), t()
        y, ysc, dx, dxs, dres = (torch.empty_like(x) for _ in range(5))
        mask = torch.empty(M * c // 8, dtype=torch.uint8, device=dev)
        p = [torch.rand(c, device=dev) + 0.5 for _ in range(8)]      # gamma, beta, mean, invstd (two layers)
        gam, bet, mea, ist, gam_s, bet_s, mea_s, ist_s = p
        out = [torch.empty(c, device=dev) for _ in range(4)]
        sums = torch.empty(4 * c, device=dev)
        ws = torch.empty(int(lib.drc_bn_workspace(M, c, sms)) // 2 * 3, device=dev)

        def fwd(xx, res, yy, mk, relu, gm, bt, mn, iv):
            N.check(lib.drc_bn_fwd(xx.data_ptr(), res, yy.data_ptr(), mk, gm.data_ptr(), bt.data_ptr(), None, None, mn.data_ptr(),
                                   iv.data_ptr(), None, None, M, c, 1e-5, 0.1, relu, sms, 1, st), "bn_fwd")

        def bwd(ddy, yy, mk, xx, ddx, dr, mode, gm, mn, iv):
            N.check(lib.drc_bn_bwd(ddy.data_ptr(), yy, mk, xx.data_ptr(), gm.data_ptr(), None, mn.data_ptr(), iv.data_ptr(),
                                   ddx.data_ptr(), dr, out[0].data_ptr(), out[1].data_ptr(), ws.data_ptr(), sums.data_ptr(),
                                   cnt[8:].data_ptr(), M, c, mode, sms, st), "bn_bwd")

        variants = {
            "fwd mask y": lambda: fwd(x, None, y, None, 1, gam, bet, mea, ist),
            "fwd mask bits": lambda: fwd(x, None, y, mask.data_ptr(), 1, gam, bet, mea, ist),
            "bwd mask y": lambda: bwd(dy, y.data_ptr(), None, x, dx, None, norm.MASK_Y, gam, mea, ist),
            "bwd mask bits": lambda: bwd(dy, None, mask.data_ptr(), x, dx, None, norm.MASK_BITS, gam, mea, ist),
        }
        if n_pairs:
            def fwd_pair_2x():
                fwd(s, None, ysc, None, 0, gam_s, bet_s, mea_s, ist_s)
                fwd(x, ysc.data_ptr(), y, None, 1, gam, bet, mea, ist)

            def fwd_pair_1x():
                N.check(lib.drc_bn_fwd_dual(x.data_ptr(), s.data_ptr(), y.data_ptr(), mask.data_ptr(), gam.data_ptr(), bet.data_ptr(),
                                            mea.data_ptr(), ist.data_ptr(), gam_s.data_ptr(), bet_s.data_ptr(), mea_s.data_ptr(),
                                            ist_s.data_ptr(), M, c, sms, st), "bn_fwd_dual")

            def bwd_pair_2x():
                bwd(dy, y.data_ptr(), None, x, dx, dres.data_ptr(), norm.MASK_Y, gam, mea, ist)
                bwd(dres, None, None, s, dxs, None, norm.MASK_NONE, gam_s, mea_s, ist_s)

            def bwd_pair_1x():
                N.check(lib.drc_bn_bwd_dual(dy.data_ptr(), mask.data_ptr(), x.data_ptr(), s.data_ptr(), gam.data_ptr(), mea.data_ptr(),
                                            ist.data_ptr(), gam_s.data_ptr(), mea_s.data_ptr(), ist_s.data_ptr(), dx.data_ptr(),
                                            dxs.data_ptr(), out[0].data_ptr(), out[1].data_ptr(), out[2].data_ptr(),
                                            out[3].data_ptr(), ws.data_ptr(), sums.data_ptr(), sums[2 * c:].data_ptr(),
                                            cnt[8:].data_ptr(), M, c, sms, st), "bn_bwd_dual")
            variants.update({"fwd pair 2x": fwd_pair_2x, "fwd pair 1x": fwd_pair_1x,
                             "bwd pair 2x": bwd_pair_2x, "bwd pair 1x": bwd_pair_1x})
        # the mask variants read what the forward wrote
        fwd(x, None, y, mask.data_ptr(), 1, gam, bet, mea, ist)
        for name, fn in variants.items():
            us = timed(fn, a.iters)
            nbytes = BYTES[name] * M * c
            gbs = nbytes / us * 1e-3
            share = gbs * 1e9 / HBM_BPS
            rows.append({"C": c, "HW": hw, "elements": M * c, "variant": name, "us": us, "GBps": gbs, "hbm_share": share,
                         "layers": n_pairs if "pair" in name else n_layers})
            print(f"| {c} x {hw} x {hw} | {M * c} | {name} | {us:.1f} | {gbs:.0f} | {100 * share:.0f} % |")
    # per worker step: the y-mask single layers + two-layer pairs vs bits + one-pass pairs (ResNet-18 layer counts above)
    tot = {}
    for r in rows:
        tot[r["variant"]] = tot.get(r["variant"], 0.0) + r["us"] * r["layers"]
    before = tot["fwd mask y"] + tot["bwd mask y"] + tot["fwd pair 2x"] + tot["bwd pair 2x"]
    after = tot["fwd mask bits"] + tot["bwd mask bits"] + tot["fwd pair 1x"] + tot["bwd pair 1x"]
    print(f"\nper worker step (14 single layers timed without their residual input, 3 pairs): {before:.0f} us -> {after:.0f} us "
          "(isolated kernels, back to back on one stream)")
    if a.json:
        with open(a.json, "w") as fh:
            json.dump({"gpu": gpu_info(), "rows": rows, "per_worker_us": {"before": before, "after": after}}, fh, indent=1)


if __name__ == "__main__":
    main()
