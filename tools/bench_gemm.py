"""wgmma GEMM (csrc/cuda/gemm_wgmma.cu) throughput vs cuBLAS (torch.matmul), CUDA-event timed, L2 flushed between iterations.
    python tools/bench_gemm.py [--json gpurun_out/gemm_bench.json]
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from draco_b200.ops import kernels as K  # noqa: E402

SHAPES = [(8192, 8192, 8192), (4096, 4096, 4096), (16384, 512, 4608), (131072, 64, 576), (32768, 128, 1152), (8192, 256, 2304),
          (2048, 512, 4608), (128, 800, 784), (896, 512, 512)]


def timeit(fn, flush, iters=10, warm=3):
    for _ in range(warm):
        fn()
    ts = []
    for _ in range(iters):
        flush.zero_()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record(); fn(); e.record()
        torch.cuda.synchronize()
        ts.append(s.elapsed_time(e))
    ts.sort()
    return ts[len(ts) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--json", default=None)
    ap.add_argument("--quick", action="store_true")
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)
    rows = []
    for (M, N, Kd) in (SHAPES[1:4] if a.quick else SHAPES):
        A = torch.randn(M, Kd, device=dev).to(torch.bfloat16)
        B = torch.randn(N, Kd, device=dev).to(torch.bfloat16)
        out = torch.empty(M, N, dtype=torch.bfloat16, device=dev)
        t_ours = timeit(lambda: K.gemm_bf16(A, B, out=out), flush)
        t_64 = timeit(lambda: K.gemm_bf16(A, B, out=out, block_n=64), flush) if N >= 64 else None
        t_128 = timeit(lambda: K.gemm_bf16(A, B, out=out, block_n=128), flush) if N >= 128 else None
        t_cublas = timeit(lambda: torch.matmul(A, B.t(), out=out), flush)
        fl = 2.0 * M * N * Kd
        rows.append({"M": M, "N": N, "K": Kd, "ours_ms": t_ours, "cublas_ms": t_cublas, "ours_tflops": fl / t_ours / 1e9,
                     "cublas_tflops": fl / t_cublas / 1e9, "ratio": t_cublas / t_ours,
                     "bn64_tflops": fl / t_64 / 1e9 if t_64 else None, "bn128_tflops": fl / t_128 / 1e9 if t_128 else None})
        print(rows[-1], flush=True)
    if a.json:
        with open(a.json, "w") as fh:
            json.dump(rows, fh, indent=1)


if __name__ == "__main__":
    main()
