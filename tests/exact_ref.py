"""Exact and component-wise references for the tensor-core GEMM / convolution kernels and the BatchNorm kernels.

Integer operands.  Operands drawn from {-1, 0, +1} make every bf16 x bf16 product exact and every partial sum an integer; as
long as no partial sum exceeds 2^24 in magnitude, every fp32 sum of them is exact in ANY order, on any tile, split-K or cluster
plan.  A bf16 output must then equal ``bf16_rn(exact)`` bit for bit, and one reference checks every kernel variant with
``torch.equal``.  The magnitude of a sum of K terms is at most K (< 2^24 for every layer here); ``int_operand`` additionally
draws the nonzeros with a density p such that the expected number of nonzero products K * p^2 stays near ``target`` (2^11 by
default), far below 2^24, as a margin against reduced-precision adders inside the tensor core.

Component-wise bound.  For real-valued data a kernel that accumulates K exact products in fp32 (round-to-nearest, or
round-toward-zero adders: relative error <= 2^-23 per addition) and rounds the result once to bf16 (relative error <= 2^-9)
satisfies, element by element,

    |y - ref64| <= 2^-8 * |ref64| + gamma * (|x| (*) |w|),   gamma = (K + 1) * 2^-23,

where (*) is the same operation applied to the absolute values in fp64 (the standard dot-product bound with a factor 2 of slack
in each term; the +1 covers a bias or residual added before rounding).  ``check_bound`` reports the worst element with its index.

References are computed in fp64 (exact for integer data), by the tap decomposition the kernels use: a k x k convolution is the
sum over its taps of one [pixels, Cin] x [Cin, Cout] product each; dgrad is the adjoint (scatter of the same slices), wgrad the
product of dy^T with the same slices.
"""
from __future__ import annotations

import math

import numpy as np
import torch

from draco_b200.codes.oracle import fma_f32

FP32_EXACT = 2 ** 24          # every integer of magnitude <= 2^24 is an fp32


# ---------------------------------------------------------------------------------------------------------------------
# operands
# ---------------------------------------------------------------------------------------------------------------------
def density_for(K: int, target: int = 2 ** 11) -> float:
    """Nonzero density p of both operands of a K-term dot product: K * p^2 nonzero products expected, at most ``target``."""
    return min(1.0, math.sqrt(target / K))


def int_operand(shape, K: int, gen: torch.Generator, target: int = 2 ** 11, device="cpu") -> torch.Tensor:
    """fp32 tensor of {-1, 0, +1}: nonzero with probability ``density_for(K, target)``, sign uniform."""
    p = density_for(K, target)
    nz = torch.rand(shape, generator=gen) < p
    sign = torch.randint(0, 2, shape, generator=gen) * 2 - 1
    return (nz * sign).to(torch.float32).to(device)


def cl(t: torch.Tensor) -> torch.Tensor:
    """bf16 channels-last copy (exact for integer data)."""
    return t.to(torch.bfloat16).contiguous(memory_format=torch.channels_last)


def wt(w: torch.Tensor) -> torch.Tensor:
    """Weights [Cout, Cin, k, k] as bf16 in the arena storage order [Cout, k, k, Cin]."""
    return w.to(torch.bfloat16).permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2)


# ---------------------------------------------------------------------------------------------------------------------
# rounding
# ---------------------------------------------------------------------------------------------------------------------
def bf16_rn(x: torch.Tensor) -> torch.Tensor:
    """Round an fp64 tensor to bf16 once, to nearest, ties to even (no intermediate fp32 rounding).  Normal range only."""
    x = x.double()
    m, e = torch.frexp(x)                                   # x = m * 2^e, 0.5 <= |m| < 1
    r = torch.ldexp(torch.round(m * 256.0), (e - 8).double())   # 8 significant bits; torch.round is half-to-even
    r = torch.where(x == 0, x, r)
    return r.float().to(torch.bfloat16)                     # exact: r has 8 significant bits


def bf16_rz(x: torch.Tensor) -> torch.Tensor:
    """Round an fp64 tensor to bf16 toward zero (the truncating store a kernel must not use)."""
    x = x.double()
    m, e = torch.frexp(x)
    r = torch.ldexp(torch.trunc(m * 256.0), (e - 8).double())
    return torch.where(x == 0, x, r).float().to(torch.bfloat16)


def ulp_bf16(x: torch.Tensor) -> torch.Tensor:
    """Spacing of bf16 values at |x| (normal range)."""
    _, e = torch.frexp(x.double().abs().clamp_min(2.0 ** -126))
    return torch.ldexp(torch.ones_like(x, dtype=torch.float64), (e - 8).double())


def ulp_f32(x: torch.Tensor) -> torch.Tensor:
    _, e = torch.frexp(x.double().abs().clamp_min(2.0 ** -126))
    return torch.ldexp(torch.ones_like(x, dtype=torch.float64), (e - 24).double())


# ---------------------------------------------------------------------------------------------------------------------
# fp64 convolution references (NCHW logical tensors, any memory format)
# ---------------------------------------------------------------------------------------------------------------------
def _taps(ks, stride, oh, ow):
    for r in range(ks):
        for s in range(ks):
            yield r, s, slice(r, r + stride * (oh - 1) + 1, stride), slice(s, s + stride * (ow - 1) + 1, stride)


def conv_ref(x: torch.Tensor, w: torch.Tensor, stride: int, bias=None) -> torch.Tensor:
    """fp64 y[N, Cout, H/s, W/s] of a k x k convolution with padding k // 2."""
    ks = w.shape[2]
    pad = ks // 2
    n, _, h, wd = x.shape
    oh, ow = h // stride, wd // stride
    xp = torch.nn.functional.pad(x.double().permute(0, 2, 3, 1), (0, 0, pad, pad, pad, pad))     # [N, H+2p, W+2p, Cin]
    wd64 = w.double()
    y = torch.zeros(n, oh, ow, w.shape[0], dtype=torch.float64, device=x.device)
    for r, s, hs, ws in _taps(ks, stride, oh, ow):
        y += xp[:, hs, ws, :] @ wd64[:, :, r, s].t()
    if bias is not None:
        y += bias.double()
    return y.permute(0, 3, 1, 2)


def dgrad_ref(dy: torch.Tensor, w: torch.Tensor, in_hw, stride: int) -> torch.Tensor:
    """fp64 dx[N, Cin, H, W] = adjoint of ``conv_ref`` applied to dy."""
    ks = w.shape[2]
    pad = ks // 2
    h, wd = in_hw
    n, _, oh, ow = dy.shape
    d = dy.double().permute(0, 2, 3, 1)
    wd64 = w.double()
    dxp = torch.zeros(n, h + 2 * pad, wd + 2 * pad, w.shape[1], dtype=torch.float64, device=dy.device)
    for r, s, hs, ws in _taps(ks, stride, oh, ow):
        dxp[:, hs, ws, :] += d @ wd64[:, :, r, s]
    return dxp[:, pad:pad + h, pad:pad + wd, :].permute(0, 3, 1, 2)


def wgrad_ref(dy: torch.Tensor, x: torch.Tensor, ks: int, stride: int) -> torch.Tensor:
    """fp64 dw[Cout, Cin, k, k] = sum over pixels of dy (outer) the tap slice of x."""
    pad = ks // 2
    n, cout, oh, ow = dy.shape
    xp = torch.nn.functional.pad(x.double().permute(0, 2, 3, 1), (0, 0, pad, pad, pad, pad))
    d = dy.double().permute(0, 2, 3, 1).reshape(-1, cout)
    dw = torch.zeros(cout, x.shape[1], ks, ks, dtype=torch.float64, device=dy.device)
    for r, s, hs, ws in _taps(ks, stride, oh, ow):
        dw[:, :, r, s] = d.t() @ xp[:, hs, ws, :].reshape(-1, x.shape[1])
    return dw


def assert_exact_domain(*refs: torch.Tensor, limit: int = FP32_EXACT) -> None:
    """The integer-operand argument needs every partial sum below 2^24: the sums of absolute values bound them all."""
    for r in refs:
        assert float(r.abs().max()) <= limit, f"reference magnitude {float(r.abs().max())} leaves the exact fp32 range"


# ---------------------------------------------------------------------------------------------------------------------
# checkers
# ---------------------------------------------------------------------------------------------------------------------
def _where(idx, shape, tile_rows: int):
    """Index tuple, plus (pixel row, 128-row tile) for 4-D NCHW activations whose GEMM rows are NHWC pixels."""
    pos = [int(v) for v in torch.unravel_index(torch.tensor(idx), shape)]
    if len(shape) == 4:
        n, c, h, w = pos
        row = (n * shape[2] + h) * shape[3] + w
        return f"(n={n}, c={c}, h={h}, w={w}), pixel row {row}, tile {row // tile_rows}"
    return f"index {tuple(pos)}"


def mismatch(out: torch.Tensor, ref: torch.Tensor, tile_rows: int = 128) -> str:
    """'' if ``out`` equals ``ref`` bit for bit (same dtype), else a description of the first differing element and the count."""
    assert out.shape == ref.shape, (out.shape, ref.shape)
    a, b = out.float().cpu(), ref.float().cpu()
    bad = (a != b) & ~(a.isnan() & b.isnan())
    if not bool(bad.any()):
        return ""
    idx = int(bad.flatten().nonzero()[0])
    return (f"{int(bad.sum())} of {bad.numel()} elements differ; first at {_where(idx, out.shape, tile_rows)}: "
            f"got {float(a.flatten()[idx])}, expected {float(b.flatten()[idx])}")


def assert_equal(out: torch.Tensor, ref: torch.Tensor, what: str = "", tile_rows: int = 128) -> None:
    msg = mismatch(out, ref, tile_rows)
    assert not msg, f"{what}: {msg}"


def bound_violation(out: torch.Tensor, ref64: torch.Tensor, absref64: torch.Tensor, K: int, rel: float = 2.0 ** -8,
                    tile_rows: int = 128) -> str:
    """'' if |out - ref64| <= rel * |ref64| + (K + 1) * 2^-23 * absref64 everywhere, else the worst element (largest ratio of
    error to bound) with its index, pixel row and tile."""
    assert out.shape == ref64.shape == absref64.shape, (out.shape, ref64.shape, absref64.shape)
    err = (out.double() - ref64).abs()
    bound = rel * ref64.abs() + (K + 1) * 2.0 ** -23 * absref64
    ratio = err / bound.clamp_min(1e-300)
    ratio = torch.where(err == 0, torch.zeros_like(ratio), ratio)
    worst = int(ratio.flatten().argmax())
    if float(ratio.flatten()[worst]) <= 1.0 and bool(torch.isfinite(out).all()):
        return ""
    if not bool(torch.isfinite(out).all()):
        worst = int((~torch.isfinite(out)).flatten().nonzero()[0])
    return (f"{int((ratio > 1).sum())} elements outside the bound; worst at {_where(worst, out.shape, tile_rows)}: "
            f"got {float(out.flatten()[worst])}, ref {float(ref64.flatten()[worst])}, |err| {float(err.flatten()[worst]):.3e} "
            f"> bound {float(bound.flatten()[worst]):.3e}")


def assert_bound(out, ref64, absref64, K: int, what: str = "", rel: float = 2.0 ** -8) -> None:
    msg = bound_violation(out, ref64, absref64, K, rel)
    assert not msg, f"{what}: {msg}"


def rel_err(a: torch.Tensor, b: torch.Tensor) -> float:
    """The global metric the older tests use: max |a - b| / max |b|."""
    return float((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-6))


# ---------------------------------------------------------------------------------------------------------------------
# BatchNorm statistics
# ---------------------------------------------------------------------------------------------------------------------
def _f32(x: torch.Tensor) -> torch.Tensor:
    return x.double().float().double()


def bn_stats_ref(y: torch.Tensor, eps: float, momentum: float, running_mean=None, running_var=None):
    """The kernels' fp32 finalisation applied to the EXACT per-channel sums of the bf16 tensor ``y`` [N, C, H, W]:

        m = S * (1/M);  var = max(fma(-m, m, Q * (1/M)), 0);  invstd = rsqrt(var + eps)
        running_mean += momentum * (m - running_mean);  running_var += momentum * (var * (M / (M - 1)) - running_var)

    every operation rounded to fp32 (fma once).  The sums are exact in fp32 when S and Q stay below 2^24 (asserted here).
    Returns fp64 tensors holding fp32 values (mean, var, invstd_ref64, rm, rv); ``invstd_ref64`` is the fp64 rsqrt of the fp32
    ``var + eps`` (the kernels' rsqrtf is within 2 ulp of it)."""
    yd = y.double()
    M = yd.numel() // yd.shape[1]
    S = yd.sum((0, 2, 3))
    Q = (yd * yd).sum((0, 2, 3))
    assert_exact_domain(yd.abs().sum((0, 2, 3)), Q)
    inv_m = _f32(torch.tensor(1.0 / float(torch.tensor(float(M), dtype=torch.float32)), dtype=torch.float64))
    m = _f32(S * inv_m)
    var = _f32(-m * m + _f32(Q * inv_m))              # fma: one rounding (the fp64 sum is exact or within 2^-53)
    var = var.clamp_min(0.0)
    v = _f32(var + _f32(torch.tensor(eps, dtype=torch.float64)))
    invstd = 1.0 / v.sqrt()
    rm = rv = None
    if running_mean is not None:
        r = _f32(torch.tensor(float(torch.tensor(float(M), dtype=torch.float32)) / float(torch.tensor(float(M - 1),
                                                                                                        dtype=torch.float32)),
                              dtype=torch.float64))
        unb = _f32(var * r)
        mom = _f32(torch.tensor(momentum, dtype=torch.float64))
        rm0, rv0 = running_mean.double().to(m.device), running_var.double().to(m.device)
        rm = _f32(mom * _f32(m - rm0) + rm0)
        rv = _f32(mom * _f32(unb - rv0) + rv0)
    return m, var, invstd, rm, rv


def ulps_f32(got: torch.Tensor, ref: torch.Tensor) -> float:
    """max |got - ref| in units of the fp32 spacing at ref."""
    g, r = got.double().to(ref.device), ref.double()
    return float(((g - r).abs() / ulp_f32(r)).max())


# ---------------------------------------------------------------------------------------------------------------------
# BatchNorm apply and backward (csrc/cuda/bn_fused.cu), restated operation by operation in fp32
# ---------------------------------------------------------------------------------------------------------------------
# Activations are [M, C] (one NHWC pixel row per row), per-channel vectors [C]; any float dtype is read as its fp32 value.
# rn32(a op b) is the fp64 result rounded once to fp32: a product of two fp32 values is exact in fp64, and a sum rounded
# first to fp64 then to fp32 equals the fp32 sum (53 >= 2 * 24 + 2).  fma is codes.oracle.fma_f32 (one rounding), bf16 is
# torch's fp32 -> bf16 conversion (round to nearest even, NaN stays NaN), as __float2bfloat16_rn.
def _np32(t) -> np.ndarray:
    return t.detach().cpu().float().numpy() if isinstance(t, torch.Tensor) else np.asarray(t, dtype=np.float32)


def _mul32(a, b) -> np.ndarray:
    with np.errstate(all="ignore"):
        return (np.asarray(a, np.float32).astype(np.float64) * np.asarray(b, np.float32).astype(np.float64)).astype(np.float32)


def _add32(a, b) -> np.ndarray:
    with np.errstate(all="ignore"):
        return (np.asarray(a, np.float32).astype(np.float64) + np.asarray(b, np.float32).astype(np.float64)).astype(np.float32)


def _fma32(a, b, c) -> np.ndarray:
    with np.errstate(all="ignore"):
        return fma_f32(a, b, c)


def _bf16(f: np.ndarray) -> torch.Tensor:
    return torch.from_numpy(np.ascontiguousarray(f, dtype=np.float32)).to(torch.bfloat16)


def _scale_shift(gamma, beta, mean, invstd):
    """The forward's per-channel coefficients: sc = rn32(gamma * invstd), sh = fma(-mean, sc, beta)."""
    sc = _mul32(_np32(gamma), _np32(invstd))
    return sc, _fma32(-_np32(mean), sc, _np32(beta))


def bn_apply_ref(x, res, gamma, beta, mean, invstd, relu: bool, pair=None):
    """bn_apply_kernel: y = bf16(relu?(fma(x, sc, sh) [+ r])) and the ReLU bits keep = (y > 0), per element of [M, C]:

        sc = rn32(gamma * invstd);  sh = fma(-mean, sc, beta);  f = fma(x, sc, sh)
        r  = res, or with ``pair = (xs, gamma_s, beta_s, mean_s, invstd_s)`` the shortcut layer's bf16(fma(xs, sc_s, sh_s))
        f  = rn32(f + r);  relu: f = fmaxf(f, 0) (a NaN becomes 0);  y = bf16(f)

    Returns (y bf16 [M, C], keep bool [M, C])."""
    sc, sh = _scale_shift(gamma, beta, mean, invstd)
    f = _fma32(_np32(x), sc, sh)
    if pair is not None:
        xs, gamma_s, beta_s, mean_s, invstd_s = pair
        sc_s, sh_s = _scale_shift(gamma_s, beta_s, mean_s, invstd_s)
        f = _add32(f, _np32(_bf16(_fma32(_np32(xs), sc_s, sh_s))))
    elif res is not None:
        f = _add32(f, _np32(res))
    if relu:
        f = np.fmax(f, np.float32(0.0))
    y = _bf16(f)
    return y, y.float() > 0


def bn_bwd_coeffs_ref(gamma, invstd, mean, sums):
    """bn_bwd_apply_kernel's per-channel coefficients from sums = [m1 = mean(dz), m2 = mean(dz * xhat)] ([2C] or [2, C]):

        cA = gs = rn32(gamma * invstd);  cB = -rn32(rn32(gs * m2) * invstd);  cC = rn32(gs * fma(rn32(m2 * invstd), mean, -m1))

    so that dx = cA dz + cB x + cC = gs (dz - m1 - xhat m2).  Returns fp32 tensors (cA, cB, cC)."""
    s = _np32(sums).reshape(2, -1)
    m1, m2, istd = s[0], s[1], _np32(invstd)
    gs = _mul32(_np32(gamma), istd)
    cB = -_mul32(_mul32(gs, m2), istd)
    cC = _mul32(gs, _fma32(_mul32(m2, istd), _np32(mean), -m1))
    return tuple(torch.from_numpy(v) for v in (gs, cB, cC))


def bn_bwd_apply_ref(dy, keep, x, coeffs):
    """bn_bwd_apply_kernel / bn_bwd_apply_dual_kernel / drc_bn_bwd_apply, per element of [M, C]:

        dz = keep ? dy : 0;  dx = bf16(fma(cA, dz, fma(cB, x, cC)));  dres = bf16(dz) (exact)

    ``keep`` None keeps every element (mask mode 0).  Returns (dx bf16, dres bf16)."""
    dz = _np32(dy)
    if keep is not None:
        dz = np.where(keep.cpu().numpy(), dz, np.float32(0.0))
    cA, cB, cC = (_np32(c) for c in coeffs)
    return _bf16(_fma32(cA, dz, _fma32(cB, _np32(x), cC))), _bf16(dz)


def bn_bwd_sums_ref(dz, x, mean, invstd):
    """bn_bwd_reduce_kernel's sums over the rows of [M, C], for the masked gradient dz:

        xhat = rn32(rn32(x - mean) * invstd);  dbeta = sum dz;  dgamma = sum dz * xhat;
        sums = [rn32(dbeta * rn32(1/M)), rn32(dgamma * rn32(1/M))]

    dbeta and dgamma are returned EXACT (fp64 sums of fp32 terms).  The kernel's fp32 sums equal them in any order when every
    partial sum is an fp32 value: integer dz with xhat on a grid of 2^-k (an integer mean and invstd = 2^-k) whose absolute
    sums stay below 2^(24 - k).  ``assert_exact_domain`` checks the absolute sums against 2^24; the caller keeps k small.
    For the dual reduce call it again with the shortcut input xs, mean_s, invstd_s (its dbeta is the same).
    Returns (dbeta fp64 [C], dgamma fp64 [C], sums fp32 [2C])."""
    d = _np32(dz).astype(np.float64)
    xhat = _mul32(_add32(_np32(x), -_np32(mean)), _np32(invstd)).astype(np.float64)
    assert_exact_domain(torch.from_numpy(np.abs(d).sum(0)), torch.from_numpy(np.abs(d * xhat).sum(0)))
    dbeta, dgamma = d.sum(0), (d * xhat).sum(0)
    M = d.shape[0]
    inv_m = np.float64(np.float32(1.0) / np.float32(M))
    sums = np.concatenate([dbeta * inv_m, dgamma * inv_m]).astype(np.float32)
    return torch.from_numpy(dbeta), torch.from_numpy(dgamma), torch.from_numpy(sums)


def unpack_relu_bits(mask: torch.Tensor, shape) -> torch.Tensor:
    """The forward's ReLU bits (bit i of byte (row, cv) is channel 8 cv + i of that row) as a bool tensor: [M, C] for
    shape (M, C), NCHW for shape (n, c, h, w)."""
    c = shape[1]
    m = mask.reshape(-1, c // 8).long()
    bits = torch.stack([(m >> i) & 1 for i in range(8)], dim=-1).reshape(-1, c).bool()
    if len(shape) == 2:
        return bits
    n, _, h, w = shape
    return bits.reshape(n, h, w, c).permute(0, 3, 1, 2)


# ---------------------------------------------------------------------------------------------------------------------
# PS update (csrc/cuda/aggregate_update.cu: the gradient sources of modes 0 / 1 / 2 and the SGD / Adam / AMSGrad tail),
# the bf16 parameter cast and the cyclic projection (csrc/cuda/fourier.cu), restated operation by operation
# ---------------------------------------------------------------------------------------------------------------------
# Every function takes numpy arrays (or anything np.asarray reads) and returns fp32 numpy arrays.  rn32 is one rounding to
# fp32 of the exact result: +, -, *, / and sqrt are formed in fp64 and rounded once more to fp32, which is innocuous
# (53 >= 2 * 24 + 2), subnormals included; fma is codes.oracle.fma_f32.  Nothing here flushes subnormals, like the kernels
# (built without --use_fast_math).
def _a32(x) -> np.ndarray:
    return np.asarray(x, dtype=np.float32)


def _div32(a, b) -> np.ndarray:
    with np.errstate(all="ignore"):
        return (_a32(a).astype(np.float64) / _a32(b).astype(np.float64)).astype(np.float32)


def _sqrt32(a) -> np.ndarray:
    with np.errstate(all="ignore"):
        return np.sqrt(_a32(a).astype(np.float64)).astype(np.float32)


def one_minus_f32(x: float) -> np.float32:
    """fp32(1 - x) with 1 - x formed in fp64 and rounded once: the coefficient the update kernel reads from HyperParams."""
    return np.float32(1.0 - float(x))


def update_source_ref(mode: int, rows, scale: float, weights=None, recomb=None) -> np.ndarray:
    """The aggregated gradient g (``grad_out``) of one tensor.  ``rows``: the K rows that contribute, [K, n] fp32 for modes 0
    and 2 (row k is worker slot select[k][tensor], or slot k), complex [K, n] (or a pair (re, im)) for mode 1.  Starting from
    acc = +0 in every mode, for k = 0, 1, ..., K - 1 in ascending order:

        mode 0 (select-sum):   acc = rn32(acc + x_k)
        mode 2 (weights):      acc = fma(w_k, x_k, acc)                         w = ``weights`` [K] fp32
        mode 1 (cyclic):       acc = rn32(acc + fma(v.re, c.re, -rn32(v.im * c.im)))   v = ``recomb`` [K] complex64, c = x_k;
                               a row with v.re == 0 and v.im == 0 is skipped (it is never read)

    then g = rn32(acc * scale): one rounded multiply by the fp32 ``scale`` (1/K, 1/n, 1), not a divide."""
    sc = np.float32(scale)
    if mode == 1:
        re, im = (rows if isinstance(rows, tuple) else (np.real(rows), np.imag(rows)))
        re, im = _a32(re), _a32(im)
        v = np.asarray(recomb)
        vr, vi = _a32(np.real(v)), _a32(np.imag(v))
        acc = np.zeros(re.shape[1:], np.float32)
        for k in range(re.shape[0]):
            if vr[k] == 0 and vi[k] == 0:
                continue
            acc = _add32(acc, _fma32(vr[k], re[k], -_mul32(vi[k], im[k])))
        return _mul32(acc, sc)
    x = _a32(rows)
    acc = np.zeros(x.shape[1:], np.float32)
    for k in range(x.shape[0]):
        acc = _add32(acc, x[k]) if mode == 0 else _fma32(_a32(weights)[k], x[k], acc)
    return _mul32(acc, sc)


def sgd_tail_ref(g, p, m, *, lr: float, momentum: float, dampening: float, weight_decay: float, nesterov: bool, first: bool):
    """SGD-momentum (torch.optim.SGD semantics) per element, on fp32 values lr, mu, wd and c = one_minus_f32(dampening):

        d = g;  wd != 0: d = fma(wd, p, d)
        mu != 0:  b = d on the first step (no dampening), else fma(mu, m, rn32(c * d));  m = b;
                  d = nesterov ? fma(mu, b, d) : b
        p = fma(-lr, d, p)

    Returns (p, m); m is returned unchanged when mu == 0."""
    lr32, mu, wd, c = np.float32(lr), np.float32(momentum), np.float32(weight_decay), one_minus_f32(dampening)
    d, p, m = _a32(g), _a32(p), _a32(m)
    if wd != 0:
        d = _fma32(wd, p, d)
    if mu != 0:
        b = d.copy() if first else _fma32(mu, m, _mul32(c, d))
        m = b
        d = _fma32(mu, b, d) if nesterov else b
    return _fma32(-lr32, d, p), m


def adam_step_size_ref(lr: float, beta1: float, beta2: float, step: int, first_step: int = 1) -> np.float32:
    """The folded Adam step size fp32(lr32 * sqrt(1 - beta2^t) / (1 - beta1^t)) formed in fp64 from the fp32 lr and the fp64
    betas, with t = step - first_step + 1 (the updates so far, plus one).  The kernel's fp64 pow may differ from the host's
    in the last fp64 bit; one rounding to fp32 absorbs that unless the value sits within a few fp64 ulp of an fp32 midpoint."""
    t = float(step - first_step + 1)
    bc1, bc2 = 1.0 - float(beta1) ** t, 1.0 - float(beta2) ** t
    return np.float32(float(np.float32(lr)) * math.sqrt(bc2) / bc1)


def adam_tail_ref(g, p, m, v, vmax, *, step_size, beta1: float, beta2: float, eps: float, weight_decay: float,
                  amsgrad: bool, c1=None, c2=None):
    """Adam / AMSGrad per element, on fp32 b1, b2, eps, wd, c1 = one_minus_f32(beta1), c2 = one_minus_f32(beta2) and the
    fp32 ``step_size`` of ``adam_step_size_ref``:

        d = g;  wd != 0: d = fma(wd, p, d)
        m = fma(b1, m, rn32(c1 * d));  v = fma(b2, v, rn32(rn32(c2 * d) * d))
        amsgrad: vmax = fmaxf(vmax, v) (a NaN loses to a number), s = vmax;  else s = v
        p = fma(-step_size, rn32(m / rn32(sqrt(s) + eps)), p)       (IEEE sqrt and divide)

    Returns (p, m, v, vmax) (vmax unchanged without amsgrad)."""
    b1, b2, e, wd = np.float32(beta1), np.float32(beta2), np.float32(eps), np.float32(weight_decay)
    c1 = one_minus_f32(beta1) if c1 is None else np.float32(c1)
    c2 = one_minus_f32(beta2) if c2 is None else np.float32(c2)
    d, p, m, v = _a32(g), _a32(p), _a32(m), _a32(v)
    if wd != 0:
        d = _fma32(wd, p, d)
    m = _fma32(b1, m, _mul32(c1, d))
    v = _fma32(b2, v, _mul32(_mul32(c2, d), d))
    s = v
    if amsgrad:
        vmax = np.fmax(_a32(vmax), v)
        s = vmax
    u = _div32(m, _add32(_sqrt32(s), e))
    return _fma32(-np.float32(step_size), u, p), m, v, (vmax if amsgrad else _a32(vmax))


def cast_bf16_ref(x) -> np.ndarray:
    """cast_params_kernel (__floats2bfloat162_rn): fp32 -> bf16 to nearest, ties to even, on the bit pattern; overflow rounds
    to +-Inf, subnormals round like normals, +-0 keep their sign, a NaN stays a NaN (its payload is not specified).
    Returns the bf16 bit patterns as uint16."""
    u = _a32(x).view(np.uint32).astype(np.uint64)
    r = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16).astype(np.uint16)
    nan = np.isnan(_a32(x))
    return np.where(nan, (u >> 16).astype(np.uint16) | np.uint16(0x0040), r)


def cyclic_project_ref(R_re, R_im, f, tile_tensor, valid) -> tuple:
    """cyclic_project_kernel + cyclic_fold_kernel: E[t][i] = sum over tensor t of R_i[d] f[d] in fp64, in the kernels' order.
    ``R_re`` / ``R_im``: [n, D] fp32 (D a multiple of 1024), ``f``: [D] fp32, ``tile_tensor``: [ntiles] tensor of each tile,
    ``valid``: [ntiles] real elements of each tile.  Per tile (1024 elements, 256 threads of 4, 8 warps):

        thread j (active iff 4 j < valid): x_j = ((R[4j] f[4j] + R[4j+1] f[4j+1]) + R[4j+2] f[4j+2]) + R[4j+3] f[4j+3] in fp64
                 (every fp32 x fp32 product is exact in fp64, so contraction into DFMA cannot change a bit); inactive: 0
        warp w:  lane values y_l = x_{32w+l}; for o = 16, 8, 4, 2, 1: y_l = y_l + y_{l xor o}; the warp's value is y_0
        tile:    t = 0;  for w = 0..7: t = t + warp_w                                      (Epart[tile])
    Per tensor (one warp over its tiles q = 0 .. ntile - 1):
        lane l:  s_l = 0;  for q = l, l + 32, ...: s_l = s_l + Epart[tile0 + q];  then the same xor butterfly; E = s_0
    The worker chunks of 8 (DRC_MAX_R) only split the work: every (worker, re / im) has its own sum.
    Returns (E_re, E_im) fp64 [T, n]."""
    tile_tensor = np.asarray(tile_tensor)
    ntiles = tile_tensor.shape[0]
    f64 = _a32(f).astype(np.float64).reshape(ntiles, 256, 4)
    active = (np.arange(256)[None, :] * 4) < np.asarray(valid)[:, None]                  # [ntiles, 256]

    def butterfly(y):                                                                    # y [..., 32] -> lane 0's value
        for o in (16, 8, 4, 2, 1):
            y = y + y[..., np.arange(32) ^ o]
        return y[..., 0]

    out = []
    for Rc in (R_re, R_im):
        Rd = _a32(Rc).astype(np.float64).reshape(-1, ntiles, 256, 4)
        pr = Rd * f64[None]
        x = ((pr[..., 0] + pr[..., 1]) + pr[..., 2]) + pr[..., 3]
        x = np.where(active[None], x, 0.0)                                              # [n, ntiles, 256]
        warps = butterfly(x.reshape(x.shape[0], ntiles, 8, 32))                         # [n, ntiles, 8]
        ep = np.zeros(warps.shape[:2])
        for w in range(8):
            ep = ep + warps[..., w]                                                      # [n, ntiles]
        T = int(tile_tensor.max()) + 1
        E = np.zeros((T, ep.shape[0]))
        for t in range(T):
            tiles = np.nonzero(tile_tensor == t)[0]
            part = ep[:, tiles]                                                          # [n, ntile]
            s = np.zeros((ep.shape[0], 32))
            for q0 in range(0, part.shape[1], 32):
                blk = part[:, q0:q0 + 32]
                s[:, :blk.shape[1]] = s[:, :blk.shape[1]] + blk
            E[t] = butterfly(s)
        out.append(E)
    return out[0], out[1]
