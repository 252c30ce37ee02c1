"""Exact tests of the fragment-native convolution epilogues across tile counts per CTA.

The halo kernels (csrc/cuda/conv_halo_wgmma.cu) and the tap kernel (csrc/cuda/conv_tap_wgmma.cu, including the strided stride-2
dgrad tiles) stage every tile straight from the wgmma accumulator fragments, and the persistent CTAs carry the BatchNorm
statistics in registers from tile to tile.  Forcing a small SM count makes the CTAs take 1, 2, an odd and an even number of
tiles; every output, the BatchNorm statistics and the BatchNorm-backward sums must then equal the default-grid launch and the
fp64 reference bit for bit (integer operands, see tests/exact_ref.py).
"""
import pytest
import torch

import exact_ref as X

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)

# SM counts forced on the launchers; None = the device's own.  With the 24 tiles of the halo case: 24, 8 (even), 5 and 4 or 3 and
# 4, 1 and 2 (23) tiles per CTA; with the 18 tiles of the tap case: 18, 9 (odd), 6, 4 and 3, 3 and 2, 1 and 2 (17).
SMS = [1, 3, 5, 7, 23, 17]


def _gen(seed):
    g = torch.Generator()
    g.manual_seed(seed)
    return g


def _force_sms(monkeypatch, sms):
    from draco_b200.ops import kernels as K
    if sms is not None:
        monkeypatch.setattr(K, "sm_count", lambda device=None: sms)


def _bias(c):
    k = torch.arange(c, device=DEV)
    return ((1000 + (k * 7) % 61) * (1 - 2 * (k % 2))).float()


def _small_bias(c):
    """small integer channel means: the statistics' sums of squares stay exact in fp32"""
    return ((torch.arange(c, device=DEV) % 7) - 3).float()


def _stats_equal(req, ref_req, ref_y, what):
    m, _, invstd, rm, rv = X.bn_stats_ref(ref_y, req.eps, req.momentum, ref_req.rm0, ref_req.rv0)
    X.assert_equal(req.mean, m.float(), f"{what}: mean vs fp64")
    assert X.ulps_f32(req.invstd, invstd) <= 2, f"{what}: invstd {X.ulps_f32(req.invstd, invstd)} ulp"
    for name in ("mean", "invstd", "running_mean", "running_var"):
        X.assert_equal(getattr(req, name), getattr(ref_req, name), f"{what}: {name} vs default grid")


def _stat_request(rm0, rv0):
    from draco_b200.ops.conv import BnStatRequest
    req = BnStatRequest(1e-5, 0.1, rm0.clone(), rv0.clone())
    req.rm0, req.rv0 = rm0, rv0
    return req


def _bwd_case(g, n, c, cout, h, w):
    wt = X.int_operand((cout, c, 3, 3), 9 * cout, g, 64, DEV)
    dy = X.int_operand((n, cout, h, w), 9 * cout, g, 64, DEV)
    xbn = torch.randint(-8, 9, (n, c, h, w), generator=g).float().to(DEV)
    ybn = torch.randint(-2, 3, (n, c, h, w), generator=g).float().to(DEV)
    mean = torch.randint(-3, 4, (c,), generator=g).float().to(DEV)
    res = torch.randint(-20, 21, (n, c, h, w), generator=g).float().to(DEV)
    return wt, dy, xbn, ybn, mean, res


def _bwd_run(kind, wt, dy, xbn, ybn, mean, res, with_res, h, w):
    from draco_b200.ops.conv import BnBwdLink, conv3x3_halo, convg_tcgen05
    c = xbn.shape[1]
    link = BnBwdLink(X.cl(xbn), mean, torch.full((c,), 0.25, device=DEV), True)
    rb = X.cl(res) if with_res else None
    if kind == "halo":
        dz = conv3x3_halo(X.cl(dy), X.wt(wt), True, None, None, rb, (link, X.cl(ybn)))
    else:
        dz = convg_tcgen05(X.cl(dy), X.wt(wt), (h, w), 1, True, None, None, rb, (link, X.cl(ybn)))
    return dz, link


def _bwd_check(dz, link, ref, wt, dy, xbn, ybn, mean, res, with_res, h, w, what):
    dx64 = X.dgrad_ref(dy, wt, (h, w), 1) + (res.double() if with_res else 0)
    ref_dz = X.bf16_rn(dx64 * (ybn > 0))
    X.assert_equal(dz, ref_dz, f"{what}: dz vs fp64")
    dzd = ref_dz.double()
    xhat = (xbn.double() - mean.double().view(1, -1, 1, 1)) * 0.25
    X.assert_equal(link.dbeta, dzd.sum((0, 2, 3)).float(), f"{what}: dbeta vs fp64")
    X.assert_equal(link.dgamma, (dzd * xhat).sum((0, 2, 3)).float(), f"{what}: dgamma vs fp64")
    if ref is not None:
        X.assert_equal(dz, ref[0], f"{what}: dz vs default grid")
        for name in ("dbeta", "dgamma", "sums"):
            X.assert_equal(getattr(link, name), getattr(ref[1], name), f"{what}: {name} vs default grid")


@pytest.mark.timeout(300)
@pytest.mark.parametrize("sms", SMS)
def test_halo_fragment_epilogue_every_tile_count(sms, monkeypatch):
    from draco_b200.ops.conv import conv3x3_halo, conv3x3_halo_wgrad
    n, h, w = 3, 16, 64                                                   # 24 tiles of 8 x 16 pixels
    g = _gen(41)
    x, wt = X.int_operand((n, 64, h, w), 576, g, 16, DEV), X.int_operand((64, 64, 3, 3), 576, g, 16, DEV)
    dy = X.int_operand((n, 64, h, w), 576, g, device=DEV)
    res = (torch.randint(-150, 151, (n, 64, h, w), generator=g) * 2).float().to(DEV)
    bias = _bias(64)
    rm0 = torch.randint(-4, 5, (64,), generator=g).float().to(DEV) * 0.25
    rv0 = torch.rand(64, generator=g).to(DEV) + 0.5
    bwd = _bwd_case(g, n, 64, 64, h, w)

    def run():
        req = _stat_request(rm0, rv0)
        out = {"y_stats": conv3x3_halo(X.cl(x), X.wt(wt), False, _small_bias(64), bn_stats=req), "req": req,
               "y": conv3x3_halo(X.cl(x), X.wt(wt), False, bias),
               "dx_res": conv3x3_halo(X.cl(dy), X.wt(wt), True, None, None, X.cl(res)),
               "dx": conv3x3_halo(X.cl(dy), X.wt(wt), True),
               "dw": conv3x3_halo_wgrad(X.cl(dy), X.cl(x))}
        for with_res in (False, True):
            out[f"bwd{with_res}"] = _bwd_run("halo", *bwd, with_res, h, w)
        return out

    base = run()
    _force_sms(monkeypatch, sms)
    got = run()
    ref_y = X.bf16_rn(X.conv_ref(x, wt, 1, _small_bias(64)))
    for key, ref in (("y_stats", ref_y), ("y", X.bf16_rn(X.conv_ref(x, wt, 1, bias))), ("dx_res", X.bf16_rn(X.dgrad_ref(dy, wt, (h, w), 1) + res.double())),
                     ("dx", X.bf16_rn(X.dgrad_ref(dy, wt, (h, w), 1))), ("dw", X.bf16_rn(X.wgrad_ref(dy, x, 3, 1)))):
        X.assert_equal(got[key], ref, f"halo {key} [sms={sms}] vs fp64")
        X.assert_equal(got[key], base[key], f"halo {key} [sms={sms}] vs default grid")
    _stats_equal(got["req"], base["req"], ref_y, f"halo statistics [sms={sms}]")
    for with_res in (False, True):
        _bwd_check(*got[f"bwd{with_res}"], base[f"bwd{with_res}"], *bwd, with_res, h, w, f"halo bwd res={with_res} [sms={sms}]")


@pytest.mark.timeout(300)
@pytest.mark.parametrize("sms", SMS)
def test_tap_fragment_epilogue_every_tile_count(sms, monkeypatch):
    from draco_b200.ops.conv import convg_tcgen05, convg_wgrad_tcgen05
    n, h, w, cin, cout = 9, 16, 16, 64, 128                              # 18 pixel tiles (16 x 8 x 1) per stride-1 launch
    g = _gen(43)
    x, wt = X.int_operand((n, cin, h, w), 9 * cin, g, 16, DEV), X.int_operand((cout, cin, 3, 3), 9 * cin, g, 16, DEV)
    dy1 = X.int_operand((n, cout, h, w), 9 * cout, g, device=DEV)
    dy2 = X.int_operand((n, cout, h // 2, w // 2), 9 * cout, g, device=DEV)
    res = (torch.randint(-150, 151, (n, cin, h, w), generator=g) * 2).float().to(DEV)
    bias = _bias(cout)
    rm0 = torch.randint(-4, 5, (cout,), generator=g).float().to(DEV) * 0.25
    rv0 = torch.rand(cout, generator=g).to(DEV) + 0.5
    bwd = _bwd_case(g, n, cin, cout, h, w)

    def run():
        req = _stat_request(rm0, rv0)
        out = {"y_stats": convg_tcgen05(X.cl(x), X.wt(wt), (h, w), 1, False, _small_bias(cout), bn_stats=req), "req": req,
               "y": convg_tcgen05(X.cl(x), X.wt(wt), (h, w), 1, False, bias),
               "dx_res": convg_tcgen05(X.cl(dy1), X.wt(wt), (h, w), 1, True, None, None, X.cl(res)),
               "dx_s2_res": convg_tcgen05(X.cl(dy2), X.wt(wt), (h, w), 2, True, None, None, X.cl(res)),
               "dx_s2": convg_tcgen05(X.cl(dy2), X.wt(wt), (h, w), 2, True),
               "dw": convg_wgrad_tcgen05(X.cl(dy1), X.cl(x), 3, 1)}
        for with_res in (False, True):
            out[f"bwd{with_res}"] = _bwd_run("tap", *bwd, with_res, h, w)
        return out

    base = run()
    _force_sms(monkeypatch, sms)
    got = run()
    ref_y = X.bf16_rn(X.conv_ref(x, wt, 1, _small_bias(cout)))
    refs = (("y_stats", ref_y), ("y", X.bf16_rn(X.conv_ref(x, wt, 1, bias))), ("dx_res", X.bf16_rn(X.dgrad_ref(dy1, wt, (h, w), 1) + res.double())),
            ("dx_s2_res", X.bf16_rn(X.dgrad_ref(dy2, wt, (h, w), 2) + res.double())),
            ("dx_s2", X.bf16_rn(X.dgrad_ref(dy2, wt, (h, w), 2))), ("dw", X.bf16_rn(X.wgrad_ref(dy1, x, 3, 1))))
    for key, ref in refs:
        X.assert_equal(got[key], ref, f"tap {key} [sms={sms}] vs fp64")
        X.assert_equal(got[key], base[key], f"tap {key} [sms={sms}] vs default grid")
    _stats_equal(got["req"], base["req"], ref_y, f"tap statistics [sms={sms}]")
    for with_res in (False, True):
        _bwd_check(*got[f"bwd{with_res}"], base[f"bwd{with_res}"], *bwd, with_res, h, w, f"tap bwd res={with_res} [sms={sms}]")
