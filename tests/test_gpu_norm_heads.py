"""BatchNorm, ReLU and row L2-normalisation (norm.cu) and the loss and graph heads (heads.cu, losses.cu) against plain fp64
restatements of the same operations.

The kernels are driven through the C ABI (_cabi.lib), which exposes what ops.* hides: row strides, both BatchNorm sweep widths
(the 16-byte sweeps are taken for C % 4 == 0 with 16-byte aligned rows, the scalar ones otherwise: an odd C, an odd row stride or
a view shifted by one float forces them), null optional outputs, and the two sweeps only the whole encoder reaches
(pgnn_debug_bn_apply_fold / pgnn_debug_bn_bwd_colsum).  Every input is a view inside a NaN-filled allocation and every output
one inside a sentinel-filled allocation (device_buffers), so an over-read shows up as NaN and an over-write as a broken
sentinel.  References are computed in fp64 from the exact fp32 inputs.

Bounds (u = 2^-24, the fp32 unit roundoff; e = 2^-53, fp64's).  Each is the sum, over the roundings the kernel performs, of u
times the magnitude of the quantity rounded:
  * BatchNorm forward y = fmaf(x, sc, sh), sc = gamma*invstd, sh = fmaf(-mean, sc, beta) with mean / invstd rounded to fp32:
      |y - y64| <= u (|y| + |beta| + 6 (|x| + |mean|) |sc|) + |gamma xhat| rho / 2
    (mean: 1 rounding, invstd: <= 3 (the fold's fp32 1/sqrtf(var + eps)), sc: 1, sh: 1, the fma: 1), where
    rho = (M / 64 + 32) e E[x^2] / (var + eps) is the relative error of the variance from fp64 sums of M squares (8-row lanes,
    an 8-way fold, one atomic per 64- or 128-row block).  save_invstd: 3 u + rho / 2 relative; save_mean: u |mean| + e sum|x| / M.
  * running_var = (1-m) rv + m (float)(var M/(M-1)): u (3 |new| + m |var_unbiased|) + m var_unbiased rho.
  * BatchNorm backward gx = gamma invstd (d - k1 - xhat k2), k1 = mean(d), k2 = mean(d xhat), xhat = (x - mean) invstd in fp32:
      |gx - gx64| <= 8 u |gamma invstd| (|d| + |k1| + |xhat| (|k2| + mean|d xhat|))
    gbeta / ggamma (fp64 sums rounded once): u |ref| + 2 u sum|d xhat| for ggamma (xhat's two roundings), u |ref| + e M sum|d|.
  * heads: fp32 sums of n terms in a fixed order are within (depth) u sum|terms|; fp64 losses within (terms folded) e sum|terms|
    plus the one fp32 rounding of d loss / d logits (u |ref|).
Each *_bound_rejects_wrong_variants test restates a plausible wrong kernel on the same inputs and shows the bound rejects it.
"""
import ctypes
import importlib
import math
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from device_buffers import DEV, NAN, SENT, Region, filled
import dropout_oracle as DO

cabi = importlib.import_module("pretrain-gnns_b200._cabi")
ops = importlib.import_module("pretrain-gnns_b200.ops")
gpu = pytest.mark.gpu
OK, EINVAL = 0, -1
U = 2.0 ** -24
E64 = 2.0 ** -53
EPS = 1e-5
DEVERR_LABEL, DEVERR_GATHER = 8, 16
KVEC, KSTAT, MAX_GRID_Y = 64, 128, 65535
KBCE_MAX_BLOCKS = 132 * 4


def _st():
    return torch.cuda.current_stream().cuda_stream


def _ptr(t):
    return t.data_ptr() if t is not None else None


def _dev_flags():
    return cabi.lib.pgnn_device_error_flags(1)


def _ulps(a, b):
    """|a - b| in units in the last place of fp32 (elementwise, finite values)."""
    ia = a.float().contiguous().view(torch.int32).to(torch.int64)
    ib = b.float().contiguous().view(torch.int32).to(torch.int64)
    ia = torch.where(ia < 0, -(ia & 0x7FFFFFFF), ia)
    ib = torch.where(ib < 0, -(ib & 0x7FFFFFFF), ib)
    return (ia - ib).abs()


def _excess(out, ref, bound):
    """max |out - ref| / bound (NaN in out where ref is finite counts as infinite excess)."""
    out, ref, bound = out.double(), ref.double(), bound.double()
    err = (out - ref).abs()
    err = torch.where(torch.isnan(err) & ~torch.isnan(ref), torch.full_like(err, math.inf), err)
    return float((err / bound.clamp_min(1e-300)).nan_to_num(nan=0.0, posinf=math.inf).max()) if err.numel() else 0.0


# ---------------------------------------------------------------------------------------------------------------------------
# BatchNorm: data, fp64 reference, bounds, device runs
# ---------------------------------------------------------------------------------------------------------------------------
def bn_data(M, C, regime="plain", seed=0):
    g = torch.Generator().manual_seed(seed * 7919 + M * 31 + C)
    if regime == "plain":
        x = torch.randn(M, C, generator=g) * 2 + 3
    elif regime == "offset":      # mean >> std: 1e3 +- 1e-2
        x = 1e3 + torch.randn(M, C, generator=g) * 1e-2
    elif regime == "mixed":       # constant, negative-mean, tiny and huge columns side by side
        x = torch.randn(M, C, generator=g)
        x[:, 0::4] = 0.1                                   # var = 0: invstd = 1/sqrt(eps)
        x[:, 1::4] = -50 + x[:, 1::4] * 0.5
        x[:, 2::4] = x[:, 2::4] * 1e-3
        x[:, 3::4] = x[:, 3::4] * 1e3
    else:
        raise ValueError(regime)
    gamma = 0.5 + torch.rand(C, generator=g)
    beta = torch.rand(C, generator=g) - 0.5
    return x.float(), gamma.float(), beta.float()


def bn_stats64(x):
    xd = x.double()
    M = xd.shape[0]
    mean = xd.mean(0)
    var = ((xd * xd).sum(0) / M - mean * mean).clamp_min(0.0)
    rho = (M / 64 + 32) * E64 * (xd * xd).mean(0) / (var + EPS)
    return mean, var, rho


def bn_fwd_ref(x, gamma, beta, relu):
    mean, var, rho = bn_stats64(x)
    inv = 1.0 / torch.sqrt(var + EPS)
    xhat = (x.double() - mean) * inv
    pre = xhat * gamma.double() + beta.double()
    sc = gamma.double() * inv
    bound = U * (pre.abs() + beta.double().abs() + 6 * (x.double().abs() + mean.abs()) * sc.abs()) \
        + (gamma.double() * xhat).abs() * rho / 2
    y = pre.clamp_min(0.0) if relu else pre
    return dict(mean=mean, var=var, inv=inv, rho=rho, y=y, bound=bound)


class BnFwd:
    """pgnn_bn_fwd_train on a poisoned copy of x (row stride ldx, `shift` floats in front of the view)."""

    def __init__(self, x, gamma, beta, relu=0, ldx=None, ldy=None, shift=0, with_y=True, with_affine=True, momentum=0.1,
                 rm0=None, rv0=None, nbt0=3):
        M, C = x.shape
        self.X = filled(x, ld=ldx or C, shift=shift)
        self.G, self.B = filled(gamma[None]), filled(beta[None])
        self.Y = Region(M, C, ldy or C, SENT) if with_y else None
        self.MEAN, self.INV = Region(1, C, C, SENT), Region(1, C, C, SENT)
        self.SC = Region(1, C, C, SENT) if with_affine else None
        self.SH = Region(1, C, C, SENT) if with_affine else None
        self.RM = filled((rm0 if rm0 is not None else torch.rand(C))[None].float(), fill=SENT)
        self.RV = filled((rv0 if rv0 is not None else 0.5 + torch.rand(C))[None].float(), fill=SENT)
        self.rm0, self.rv0 = self.RM.view.cpu()[0].clone(), self.RV.view.cpu()[0].clone()
        self.NBT = torch.tensor([nbt0], dtype=torch.int64, device=DEV)
        wsb = cabi.lib.pgnn_bn_workspace_bytes(M, C)
        self.WS = torch.full((wsb // 4 + 16,), NAN, device=DEV)
        self.rc = cabi.lib.pgnn_bn_fwd_train(self.X.ptr(), self.X.ld, M, C, self.G.ptr(), self.B.ptr(), self.RM.ptr(), self.RV.ptr(),
                                             self.NBT.data_ptr(), momentum, EPS, relu, self.Y.ptr() if self.Y else None,
                                             self.Y.ld if self.Y else 0, self.MEAN.ptr(), self.INV.ptr(),
                                             self.SC.ptr() if self.SC else None, self.SH.ptr() if self.SH else None,
                                             self.WS.data_ptr(), wsb, _st())

    def regions(self):
        return [r for r in (self.Y, self.MEAN, self.INV, self.SC, self.SH, self.RM, self.RV) if r is not None]


def check_bn_fwd(x, gamma, beta, relu, run, momentum=0.1):
    assert run.rc == OK, run.rc
    torch.cuda.synchronize()
    M, C = x.shape
    r = bn_fwd_ref(x, gamma, beta, relu)
    mean = run.MEAN.view.cpu()[0]
    inv = run.INV.view.cpu()[0]
    assert _excess(mean, r["mean"], U * r["mean"].abs() + E64 * x.double().abs().sum(0) + 1e-300) <= 1, "save_mean"
    assert _excess(inv, r["inv"], (3 * U + r["rho"] / 2) * r["inv"]) <= 1, "save_invstd"
    if run.Y is not None:
        y = run.Y.view.cpu()
        assert _excess(y, r["y"], r["bound"]) <= 1, ("y", _excess(y, r["y"], r["bound"]))
    if run.SC is not None:
        sc, sh = run.SC.view.cpu()[0], run.SH.view.cpu()[0]
        # scale / shift are the fp32 products of the saved statistics, bit for bit (the gathers apply exactly these)
        assert torch.equal(sc, gamma * inv)
        assert torch.equal(sh, ops.fma32(-mean, sc, beta))
    unb = r["var"] * M / max(M - 1, 1)
    m = float(np.float32(momentum))
    rm_ref = (1 - m) * run.rm0.double() + m * r["mean"]
    rv_ref = (1 - m) * run.rv0.double() + m * unb
    # (1 - m), two products, the sum, and the mean's / variance's own rounding to fp32: 3 u of each term's magnitude
    rm_bound = 3 * U * ((1 - m) * run.rm0.double().abs() + m * r["mean"].abs()) + 1e-30
    assert _excess(run.RM.view.cpu()[0], rm_ref, rm_bound) <= 1, "running_mean"
    rv_bound = 3 * U * ((1 - m) * run.rv0.double().abs() + m * unb) + m * unb * r["rho"] + 1e-30
    assert _excess(run.RV.view.cpu()[0], rv_ref, rv_bound) <= 1, "running_var"
    assert int(run.NBT.item()) == 4  # num_batches_tracked went up by exactly one
    assert all(g.outside_intact() for g in run.regions())
    return r


M_EDGES = [1, 2, 7, 8, 9, 63, 64, 65, 127, 128, 129, 8 * 64 + 1, 5888, 100003]
C_TILES = [4, 32, 124, 128, 132, 300, 600]


@gpu
@pytest.mark.parametrize("M", M_EDGES)
@pytest.mark.parametrize("layout", ["v4", "odd_ld", "shifted"])
def test_bn_fwd_train_row_edges(M, layout):
    """Both sweep widths across the row tiles (8 row-lanes, kVecRows = 64, kStatRows = 128) at C = 132 (a column tail past 128)."""
    C = 132
    x, gamma, beta = bn_data(M, C, seed=1)
    kw = dict(v4={}, odd_ld=dict(ldx=C + 1), shifted=dict(shift=1))[layout]
    check_bn_fwd(x, gamma, beta, 1, BnFwd(x, gamma, beta, relu=1, ldy=C + 4, **kw))


@gpu
@pytest.mark.parametrize("C", C_TILES + [1, 3, 33, 301])
@pytest.mark.parametrize("relu", [0, 1])
def test_bn_fwd_train_column_tiles(C, relu):
    """Column tiles of 32 (scalar) and 128 (16-byte) columns, with row strides past C; C in {1, 3, 33, 301} forces the scalar
    sweeps on an otherwise aligned layout."""
    M = 777
    x, gamma, beta = bn_data(M, C, seed=2)
    check_bn_fwd(x, gamma, beta, relu, BnFwd(x, gamma, beta, relu=relu, ldx=C + 8 if C % 4 == 0 else C + 3, ldy=C + 4))


@gpu
@pytest.mark.parametrize("regime", ["offset", "mixed"])
@pytest.mark.parametrize("layout", ["v4", "scalar"])
def test_bn_fwd_train_data_regimes(regime, layout):
    """mean >> std, constant columns (var = 0), negative means, tiny and huge magnitudes; momentum 0.3."""
    M, C = 4099, 128
    x, gamma, beta = bn_data(M, C, regime, seed=3)
    run = BnFwd(x, gamma, beta, relu=0, shift=1 if layout == "scalar" else 0, momentum=0.3)
    r = check_bn_fwd(x, gamma, beta, 0, run, momentum=0.3)
    if regime == "mixed":   # a constant column: invstd = 1/sqrt(eps) exactly as fp32 rounds it, and y == beta
        inv = run.INV.view.cpu()[0]
        assert torch.equal(inv[0::4], torch.full_like(inv[0::4], float(np.float32(1 / np.sqrt(np.float64(np.float32(EPS)))))))


@gpu
def test_bn_fwd_train_optional_outputs_and_momenta():
    """y = NULL (statistics only) and no scale / shift; several momenta; num_batches_tracked is bumped once per call."""
    M, C = 300, 300
    x, gamma, beta = bn_data(M, C, seed=4)
    for mom in (0.0, 0.1, 0.5, 1.0):
        check_bn_fwd(x, gamma, beta, 0, BnFwd(x, gamma, beta, with_y=False, with_affine=False, momentum=mom), momentum=mom)


@gpu
def test_bn_fwd_train_single_row():
    """M = 1: mean = x, biased var = 0, invstd = 1/sqrt(eps), y = beta up to the rounding of the shift, and the unbiased running
    variance uses M / max(M - 1, 1) = 1: it becomes (1 - m) running_var, one fp32 product."""
    x, gamma, beta = bn_data(1, 132, seed=5)
    run = BnFwd(x, gamma, beta)
    check_bn_fwd(x, gamma, beta, 0, run)
    assert torch.equal(run.MEAN.view.cpu()[0], x[0])
    one_minus_m = torch.tensor(1.0, dtype=torch.float32) - torch.tensor(0.1, dtype=torch.float32)
    assert torch.equal(run.RV.view.cpu()[0], one_minus_m * run.rv0)


@gpu
def test_bn_fwd_train_nan_stays_in_its_column():
    M, C = 513, 132
    x, gamma, beta = bn_data(M, C, seed=6)
    x[100, 7] = float("nan")
    for shift in (0, 1):
        run = BnFwd(x, gamma, beta, relu=1, shift=shift)
        assert run.rc == OK
        y, mean = run.Y.view.cpu(), run.MEAN.view.cpu()[0]
        assert torch.isnan(mean[7]) and torch.isnan(y[:, 7]).all()
        others = torch.ones(C, dtype=torch.bool)
        others[7] = False
        assert torch.isfinite(y[:, others]).all() and torch.isfinite(mean[others]).all()


@gpu
def test_bn_v4_and_scalar_sweeps_agree():
    """The same data through both widths: the statistics differ only in the order of fp64 additions, so save_mean / save_invstd
    and y agree to one ulp."""
    M, C = 5888, 300
    x, gamma, beta = bn_data(M, C, seed=7)
    a = BnFwd(x, gamma, beta, relu=1)
    b = BnFwd(x, gamma, beta, relu=1, shift=1)
    assert a.rc == OK and b.rc == OK
    for ra, rb in ((a.MEAN, b.MEAN), (a.INV, b.INV), (a.Y, b.Y)):
        assert int(_ulps(ra.view.cpu(), rb.view.cpu()).max()) <= 1


@gpu
def test_bn_eval_against_fp64():
    for C, ld, relu in ((300, 304, 0), (33, 35, 1), (4, 4, 1)):
        M = 1000
        x, gamma, beta = bn_data(M, C, seed=8)
        rm, rv = torch.randn(C), 0.2 + torch.rand(C)
        X, G, B, RM, RV = filled(x, ld=ld), filled(gamma[None]), filled(beta[None]), filled(rm[None]), filled(rv[None])
        Y = Region(M, C, ld + 1, SENT)
        assert cabi.lib.pgnn_bn_fwd_eval(X.ptr(), ld, M, C, G.ptr(), B.ptr(), RM.ptr(), RV.ptr(), EPS, relu, Y.ptr(), Y.ld, _st()) == OK
        inv = 1 / torch.sqrt(rv.double() + EPS)
        xhat = (x.double() - rm.double()) * inv
        ref = xhat * gamma.double() + beta.double()
        ref = ref.clamp_min(0) if relu else ref
        # fp32: rv + eps, sqrt, reciprocal (3 roundings on invstd), x - rm, * invstd, the fma
        bound = U * (ref.abs() + 6 * (xhat * gamma.double()).abs() + 2 * (x.double().abs() + rm.double().abs()) * (inv * gamma.double()).abs())
        assert _excess(Y.view.cpu(), ref, bound) <= 1 and Y.outside_intact()


# ---- backward -------------------------------------------------------------------------------------------------------------
def bn_saved(x):
    """save_mean / save_invstd as the forward leaves them (fp64 statistics rounded to fp32)."""
    mean, var, _ = bn_stats64(x)
    return mean.float(), (1.0 / torch.sqrt(var + EPS)).float()


def preact_keep(x, mean, inv, gamma, beta):
    """The forward's ReLU decision, bit for bit: fmaf(x, sc, sh) > 0 with sc = gamma*invstd, sh = fmaf(-mean, sc, beta)."""
    sc = gamma * inv
    sh = ops.fma32(-mean, sc, beta)
    return x.double() * sc.double() + sh.double() > 0


def bn_bwd_ref(gy, x, gamma, beta, mean, inv, relu, mask=None, variant=None):
    """fp64 BatchNorm backward from the exact fp32 inputs (save_mean / save_invstd given).  mask: dropout factors [M, C] or None."""
    M = x.shape[0]
    d = gy.double() * (mask if mask is not None else 1.0)
    if relu:
        d = torch.where(preact_keep(x, mean, inv, gamma, beta), d, torch.zeros_like(d))
    xhat = (x.double() - mean.double()) * inv.double()
    k1, k2 = d.mean(0), (d * xhat).mean(0)
    gi = gamma.double() * inv.double()
    if variant == "dropped xhat*k2":
        gx = gi * (d - k1)
    else:
        gx = gi * (d - k1 - xhat * k2)
    bound = 8 * U * gi.abs() * (d.abs() + k1.abs() + xhat.abs() * (k2.abs() + (d * xhat).abs().mean(0)))
    gb, gg = d.sum(0), (d * xhat).sum(0)
    return dict(gx=gx, bound=bound, gb=gb, gg=gg, gb_bound=U * gb.abs() + E64 * M * d.abs().sum(0) + 1e-300,
                gg_bound=U * gg.abs() + 2 * U * (d * xhat).abs().sum(0) + 1e-300)


def bn_bwd_data(M, C, seed):
    x, gamma, beta = bn_data(M, C, seed=seed)
    g = torch.Generator().manual_seed(seed + 11)
    # a gradient correlated with x: sum(dy * xhat) (the k2 term) is then not small
    gy = (torch.randn(M, C, generator=g) + 0.7 * (x - x.mean(0)) / x.std(0).clamp_min(1e-3)).float()
    mean, inv = bn_saved(x)
    return x, gamma, beta, gy, mean, inv


def run_bn_bwd(gy, x, gamma, beta, mean, inv, relu, ldgy=None, ldx=None, ldgx=None, shift=0, with_grads=True, colsum=False,
               drop=(0.0, 0, 0)):
    M, C = x.shape
    GY, X = filled(gy, ld=ldgy or C, shift=shift), filled(x, ld=ldx or C, shift=shift)
    G, B, MU, IS = filled(gamma[None]), filled(beta[None]), filled(mean[None]), filled(inv[None])
    GX = Region(M, C, ldgx or C, SENT, shift=shift)
    GG, GB = (Region(1, C, C, SENT), Region(1, C, C, SENT)) if with_grads else (None, None)
    CS = Region(1, C, C, SENT) if colsum else None
    wsb = cabi.lib.pgnn_bn_workspace_bytes(M, C)
    WS = torch.full((wsb // 4 + 16,), NAN, device=DEV)
    if colsum:
        rc = cabi.lib.pgnn_debug_bn_bwd_colsum(GY.ptr(), GY.ld, X.ptr(), X.ld, M, C, G.ptr(), B.ptr(), MU.ptr(), IS.ptr(), relu, GX.ptr(),
                                               GX.ld, GG.ptr() if GG else None, GB.ptr() if GB else None, CS.ptr(), drop[0], drop[1],
                                               drop[2], WS.data_ptr(), wsb, _st())
    else:
        rc = cabi.lib.pgnn_bn_bwd(GY.ptr(), GY.ld, X.ptr(), X.ld, M, C, G.ptr(), B.ptr(), MU.ptr(), IS.ptr(), relu, GX.ptr(), GX.ld,
                                  GG.ptr() if GG else None, GB.ptr() if GB else None, WS.data_ptr(), wsb, _st())
    assert rc == OK, rc
    torch.cuda.synchronize()
    out = dict(gx=GX.view.cpu(), regions=[r for r in (GX, GG, GB, CS) if r is not None])
    if GG is not None:
        out["gg"], out["gb"] = GG.view.cpu()[0], GB.view.cpu()[0]
    if CS is not None:
        out["colsum"] = CS.view.cpu()[0]
    return out


def check_bn_bwd(out, ref):
    assert _excess(out["gx"], ref["gx"], ref["bound"]) <= 1, ("gx", _excess(out["gx"], ref["gx"], ref["bound"]))
    if "gb" in out:
        assert _excess(out["gb"], ref["gb"], ref["gb_bound"]) <= 1, "gbeta"
        assert _excess(out["gg"], ref["gg"], ref["gg_bound"]) <= 1, "ggamma"
    assert all(r.outside_intact() for r in out["regions"])


@gpu
@pytest.mark.parametrize("M", M_EDGES + [3])
@pytest.mark.parametrize("layout", ["v4", "odd_ld", "shifted"])
@pytest.mark.parametrize("relu", [0, 1])
def test_bn_bwd_row_edges(M, layout, relu):
    """Both sweep widths across the row tiles; M = 2, 3: gx is a difference of large terms."""
    C = 132
    x, gamma, beta, gy, mean, inv = bn_bwd_data(M, C, seed=20)
    kw = dict(v4=dict(ldgx=C + 4), odd_ld=dict(ldgy=C + 1, ldx=C + 3), shifted=dict(shift=1))[layout]
    check_bn_bwd(run_bn_bwd(gy, x, gamma, beta, mean, inv, relu, **kw), bn_bwd_ref(gy, x, gamma, beta, mean, inv, relu))


@gpu
@pytest.mark.parametrize("C", C_TILES + [1, 3, 33, 301])
@pytest.mark.parametrize("with_grads", [True, False])
def test_bn_bwd_column_tiles(C, with_grads):
    M = 777
    x, gamma, beta, gy, mean, inv = bn_bwd_data(M, C, seed=21)
    out = run_bn_bwd(gy, x, gamma, beta, mean, inv, 1, ldgy=C + 4, ldx=C + 8, ldgx=C + 4, with_grads=with_grads)
    check_bn_bwd(out, bn_bwd_ref(gy, x, gamma, beta, mean, inv, 1))


# ---- the fused variants (whole-encoder only) --------------------------------------------------------------------------------
def run_fold(x, gamma, beta, relu, drop=(0.0, 0, 0), momentum=0.1, ldx=None, ldy=None):
    M, C = x.shape
    xd = x.double()
    sums = torch.stack([xd.sum(0), (xd * xd).sum(0)]).to(DEV)
    X, G, B = filled(x, ld=ldx or C), filled(gamma[None]), filled(beta[None])
    RM, RV = filled(torch.zeros(1, C), fill=SENT), filled(torch.ones(1, C), fill=SENT)
    NBT = torch.tensor([5], dtype=torch.int64, device=DEV)
    MU, IS, Y = Region(1, C, C, SENT), Region(1, C, C, SENT), Region(M, C, ldy or C, SENT)
    rc = cabi.lib.pgnn_debug_bn_apply_fold(X.ptr(), X.ld, M, C, sums.data_ptr(), G.ptr(), B.ptr(), RM.ptr(), RV.ptr(), NBT.data_ptr(),
                                           momentum, EPS, MU.ptr(), IS.ptr(), relu, Y.ptr(), Y.ld, drop[0], drop[1], drop[2], _st())
    assert rc == OK, rc
    torch.cuda.synchronize()
    assert all(r.outside_intact() for r in (MU, IS, Y, RM, RV))
    return dict(y=Y.view.cpu(), mean=MU.view.cpu()[0], inv=IS.view.cpu()[0], rm=RM.view.cpu()[0], rv=RV.view.cpu()[0],
                nbt=int(NBT.item()))


def drop_factors(M, C, p, seed, layer):
    if p == 0:
        return None
    return torch.from_numpy(DO.keep_mask(seed, layer, M, C, p)).double() * DO.scale(p)


@gpu
@pytest.mark.parametrize("M", [1, 65, 5888, 40000])
@pytest.mark.parametrize("p", [0.0, 0.5])
def test_bn_apply_fold_against_fp64(M, p):
    """The fold derives the statistics in every CTA; CTA 0 alone performs the module-state side effects, exactly once whatever
    the grid (M = 1: one CTA; 40000 x 300: the capped grid of 2112 CTAs).  save_invstd agrees with k_bn_finalize's within 4 ulps
    (fold: (float)var, + eps, sqrtf, 1/x = 3 u relative; finalize: one rounding of the fp64 value)."""
    C, seed, layer = 300, 77, 3
    x, gamma, beta = bn_data(M, C, seed=30)
    f = run_fold(x, gamma, beta, 1, drop=(p, seed, layer), momentum=0.25, ldx=C + 4)
    r = bn_fwd_ref(x, gamma, beta, 1)
    ref = r["y"]
    mask = drop_factors(M, C, p, seed, layer)
    bound = r["bound"]
    if mask is not None:
        ref, bound = ref * mask, bound * mask + U * (ref * mask).abs()
    assert _excess(f["y"], ref, bound) <= 1
    fin = BnFwd(x, gamma, beta, with_y=False)
    assert fin.rc == OK
    assert int(_ulps(f["inv"], fin.INV.view.cpu()[0]).max()) <= 4
    assert int(_ulps(f["mean"], fin.MEAN.view.cpu()[0]).max()) <= 1
    unb = r["var"] * M / max(M - 1, 1)
    assert _excess(f["rm"], 0.25 * r["mean"], 3 * U * 0.25 * r["mean"].abs() + 1e-30) <= 1
    assert _excess(f["rv"], 0.75 + 0.25 * unb, 3 * U * (0.75 + 0.25 * unb) + 0.25 * unb * r["rho"]) <= 1
    assert f["nbt"] == 6


@gpu
@pytest.mark.parametrize("C,layout", [(300, "v4"), (300, "scalar"), (33, "scalar"), (128, "v4")])
@pytest.mark.parametrize("p", [0.0, 0.5])
@pytest.mark.parametrize("M", [3, 129, 5888])
def test_bn_bwd_colsum_against_fp64(C, layout, p, M):
    """pgnn_internal_bn_bwd with colsum (through pgnn_debug_bn_bwd_colsum): gx, ggamma, gbeta against fp64 with the dropout mask
    applied to gy before the ReLU mask, and colsum equal to the column sums of gx (fp32 sums over <= 8-row lanes and 8 + M / 64
    atomics: (M / 8 + 8 + M / 64) u sum|gx|)."""
    seed, layer = 5, 2
    x, gamma, beta, gy, mean, inv = bn_bwd_data(M, C, seed=22)
    kw = dict(shift=1) if layout == "scalar" else {}
    out = run_bn_bwd(gy, x, gamma, beta, mean, inv, 1, colsum=True, drop=(p, seed, layer), **kw)
    ref = bn_bwd_ref(gy, x, gamma, beta, mean, inv, 1, mask=drop_factors(M, C, p, seed, layer))
    check_bn_bwd(out, ref)
    gx = out["gx"].double()
    cs_bound = (M / 8 + 8 + M / 64) * U * gx.abs().sum(0) + 1e-30
    assert _excess(out["colsum"], gx.sum(0), cs_bound) <= 1


@gpu
def test_bn_bound_rejects_wrong_variants():
    """On the tests' own inputs: (a) a biased running_var, (b) fp32 statistic sums on a mean >> std column, (c) a dropped
    xhat*k2 term in the backward -- each is rejected by its bound by 10x or more, while the kernel passes it."""
    # (a) biased instead of unbiased running_var
    M, C = 65, 128
    x, gamma, beta = bn_data(M, C, seed=40)
    run = BnFwd(x, gamma, beta)
    r = check_bn_fwd(x, gamma, beta, 0, run)
    unb = r["var"] * M / (M - 1)
    rv_ref = 0.9 * run.rv0.double() + 0.1 * unb
    bound = 3 * U * (0.9 * run.rv0.double().abs() + 0.1 * unb) + 0.1 * unb * r["rho"]
    assert _excess(0.9 * run.rv0.double() + 0.1 * r["var"], rv_ref, bound) >= 10
    # (b) fp32 accumulation of sum and sum of squares, sequentially per column
    M = 4099
    x, gamma, beta = bn_data(M, C, "offset", seed=41)
    check_bn_fwd(x, gamma, beta, 0, BnFwd(x, gamma, beta))
    xn = x.numpy()
    s = np.cumsum(xn, 0, dtype=np.float32)[-1]
    ss = np.cumsum(xn * xn, 0, dtype=np.float32)[-1]
    m32 = s / np.float32(M)
    var32 = np.maximum(ss / np.float32(M) - m32 * m32, np.float32(0))
    inv32 = torch.from_numpy(1 / np.sqrt(var32 + np.float32(EPS))).double()
    y_bad = (x.double() - torch.from_numpy(m32).double()) * inv32 * gamma.double() + beta.double()
    r = bn_fwd_ref(x, gamma, beta, 0)
    assert _excess(y_bad, r["y"], r["bound"]) >= 10
    # (c) the backward without the xhat * k2 term
    x, gamma, beta, gy, mean, inv = bn_bwd_data(777, C, seed=42)
    ref = bn_bwd_ref(gy, x, gamma, beta, mean, inv, 1)
    bad = bn_bwd_ref(gy, x, gamma, beta, mean, inv, 1, variant="dropped xhat*k2")
    assert _excess(bad["gx"], ref["gx"], ref["bound"]) >= 10


# ---- one ReLU decision ----------------------------------------------------------------------------------------------------------
def boundary_data(M, C, seed=50, spread=8):
    """Rows of x on and within `spread` ulps of each column's ReLU root (and ordinary rows around them).  The root depends on the
    batch statistics, which depend on those rows: a fixed-point iteration in fp64 places them (the device's statistics may
    differ in the last bit, which only moves the root by a fraction of the spread)."""
    g = torch.Generator().manual_seed(seed)
    base = (torch.randn(M // 2, C, generator=g) * 1.5 + 2).float()
    gamma = (0.5 + torch.rand(C, generator=g)).float()
    beta = (torch.rand(C, generator=g) - 0.5).float()
    k = torch.arange(M - M // 2) % (2 * spread + 1) - spread
    root = base.mean(0)
    for _ in range(60):
        near = _step_ulps(root.expand(len(k), C).clone(), k[:, None].expand(len(k), C))
        x = torch.cat([base, near])
        mean, inv = bn_saved(x)
        sc = gamma * inv
        sh = ops.fma32(-mean, sc, beta)
        new = (-sh.double() / sc.double()).float()
        if torch.equal(new, root):
            break
        root = new
    return x, gamma, beta


def _step_ulps(v, k):
    """v moved by k ulps (int tensor of the same shape)."""
    out = v.clone()
    for s in range(1, int(k.abs().max()) + 1):
        up, dn = k >= s, k <= -s
        out = torch.where(up, torch.nextafter(out, torch.full_like(out, math.inf)), out)
        out = torch.where(dn, torch.nextafter(out, torch.full_like(out, -math.inf)), out)
    return out


def old_decision(x, mean, inv, gamma, beta):
    """The backward's test before the BatchNorm pre-activation was defined once: fmaf((x - mean) * invstd, gamma, beta) > 0."""
    t = (x - mean) * inv
    return t.double() * gamma.double() + beta.double() > 0


@gpu
@pytest.mark.parametrize("C", [132, 33])
def test_relu_decision_fused_gather_matches_backward(C):
    """As the fused GIN forward runs it: statistics (pgnn_bn_fwd_train, y = NULL) then pgnn_aggregate_fwd with in_scale / in_shift /
    in_relu on a graph of self-loops only; then pgnn_bn_bwd with relu and gy = 1.  gbeta[c] counts the rows whose gradient the
    backward let through: it must equal the number of rows the forward kept, exactly (counts < 2^24 are exact in fp32)."""
    M = 4096
    x, gamma, beta = boundary_data(M, C)
    C4 = (C + 3) // 4 * 4
    xp = torch.zeros(M, C4)
    xp[:, :C] = x
    gp, bp = torch.ones(C4), torch.zeros(C4)
    gp[:C], bp[:C] = gamma, beta
    # the aggregation takes C % 4 == 0: padded columns (gamma 1, beta 0, x 0) are ignored below
    st = BnFwd(xp, gp, bp, with_y=False)
    assert st.rc == OK
    rowptr = torch.zeros(M + 1, dtype=torch.int32, device=DEV)
    nbr = torch.zeros(1, dtype=torch.int32, device=DEV)
    OUT = Region(M, C4, C4, SENT)
    assert cabi.lib.pgnn_aggregate_fwd(st.X.ptr(), C4, st.SC.ptr(), st.SH.ptr(), 1, M, C4, rowptr.data_ptr(), nbr.data_ptr(), 0, None,
                                       None, 0, None, 0, OUT.ptr(), C4, _st()) == OK
    kept = (OUT.view.cpu()[:, :C] > 0).sum(0)
    ones = torch.ones(M, C4)
    out = run_bn_bwd(ones, xp, gp, bp, st.MEAN.view.cpu()[0], st.INV.view.cpu()[0], 1)
    gb = out["gb"][:C]
    mean, inv = st.MEAN.view.cpu()[0][:C], st.INV.view.cpu()[0][:C]
    differ = old_decision(x, mean, inv, gamma, beta) != preact_keep(x, mean, inv, gamma, beta)
    assert int(differ.sum()) > 0, "the data must put elements where the two expressions disagree"
    wrong = (gb != kept.float()).nonzero().flatten().tolist()
    assert not wrong, dict(columns=wrong[:10], off_by=[int(gb[c] - kept[c]) for c in wrong[:10]], disagreeing_elements=int(differ.sum()))


@gpu
@pytest.mark.parametrize("path", ["layerwise", "fold"])
def test_relu_decision_apply_matches_backward(path):
    """The same count for the layer-by-layer pair (pgnn_bn_fwd_train with relu, then pgnn_bn_bwd) and for the fold apply
    (pgnn_debug_bn_apply_fold with relu, then the colsum backward on the fold's own save_mean / save_invstd)."""
    M, C = 4096, 132
    x, gamma, beta = boundary_data(M, C, seed=51)
    if path == "layerwise":
        st = BnFwd(x, gamma, beta, relu=1)
        assert st.rc == OK
        y, mean, inv = st.Y.view.cpu(), st.MEAN.view.cpu()[0], st.INV.view.cpu()[0]
        out = run_bn_bwd(torch.ones(M, C), x, gamma, beta, mean, inv, 1)
    else:
        f = run_fold(x, gamma, beta, 1)
        y, mean, inv = f["y"], f["mean"], f["inv"]
        out = run_bn_bwd(torch.ones(M, C), x, gamma, beta, mean, inv, 1, colsum=True)
    kept = (y > 0).sum(0).float()
    wrong = (out["gb"] != kept).nonzero().flatten().tolist()
    assert not wrong, dict(columns=wrong[:10], off_by=[int(out["gb"][c] - kept[c]) for c in wrong[:10]])


@gpu
@pytest.mark.parametrize("precision", ["fp32", "tf32x3"])
def test_gin_encoder_relu_decisions_forward_equals_backward(precision):
    """A whole-encoder GIN training step (chem.GNN(3, 300), forward and backward) on both precisions: tf32x3 takes the
    stats-fused GEMM and the gather that derives scale / shift itself (bn_fold_column), fp32 the statistics pass and
    k_bn_finalize.  On a graph without edges and with zero edge tables, layer l + 1's gathered input aggr[l + 1] is exactly
    relu(bn_preact(z2[l])): the decisions the forward took, read from the workspace.  Boundary-heavy: in half of the columns
    mlp.2 is scaled by 1e-7 and beta is 0, so z2 is the bias +- an ulp or two and every element sits on or next to its column's
    root (the mean).  Per inner layer, the forward's kept set must equal ops.chem_gin_relu_masks bit for bit, and the encoder's
    BatchNorm backward sweep on the workspace's own z2 / mean / invstd with gy = 1 must count exactly those rows in gbeta."""
    chem = importlib.import_module("pretrain-gnns_b200.chem.model")
    N, L, D, H = 4096, 3, 300, 150
    torch.manual_seed(140)
    model = chem.GNN(L, D).to(DEV).train()
    with torch.no_grad():
        for layer, bn in zip(model.gnns, model.batch_norms):
            layer.edge_embedding1.weight.zero_()
            layer.edge_embedding2.weight.zero_()
            layer.mlp[2].weight[:H] *= 1e-7
            layer.mlp[2].bias[:H] = 1 + torch.rand(H, device=DEV)
            bn.bias[:H] = 0
    g = torch.Generator().manual_seed(141)
    x = torch.stack([torch.randint(0, 119, (N,), generator=g), torch.randint(0, 3, (N,), generator=g)], 1).to(DEV)
    ei, ea = torch.zeros(2, 0, dtype=torch.int64, device=DEV), torch.zeros(0, 2, dtype=torch.int64, device=DEV)
    plan = model._fused_plan()
    assert plan is not None
    old = ops.get_precision()
    ops.set_precision(precision)
    plan.keep_workspace = True
    try:
        out = model(x, ei, ea)
        torch.cuda.synchronize()
        ws, (n, E, L_, D_) = plan.last_ws
        aggr_off = cabi.lib.pgnn_chem_gin_debug_aggr_offset(N, 0, L, D)
        off = (ctypes.c_int64 * 4)()
        assert cabi.lib.pgnn_chem_gin_debug_layout(N, 0, L, D, off) == OK and aggr_off > 0
        f = lambda o, k: ws[o:o + 4 * k].view(torch.float32).clone().cpu()
        aggr = f(aggr_off, L * N * D).view(L, N, D)
        z2 = f(off[1], L * N * D).view(L, N, D)
        mean, inv = f(off[2], L * D).view(L, D), f(off[3], L * D).view(L, D)
        masks = [m.cpu() for m in ops.chem_gin_relu_masks(plan, model)]
        out.backward(torch.randn(N, D, generator=g).to(DEV))   # the rest of the training step
        torch.cuda.synchronize()
    finally:
        ops.set_precision(old)
        plan.keep_workspace, plan.last_ws = False, None
    disagree = 0
    for l in range(L - 1):
        kept = aggr[l + 1] > 0
        assert torch.equal(kept, masks[2 * l + 1]), (l, int((kept != masks[2 * l + 1]).sum()))
        gamma = model.batch_norms[l].weight.detach().cpu()
        beta = model.batch_norms[l].bias.detach().cpu()
        res = run_bn_bwd(torch.ones(N, D), z2[l], gamma, beta, mean[l], inv[l], 1, colsum=True)
        wrong = (res["gb"] != kept.sum(0).float()).nonzero().flatten().tolist()
        assert not wrong, dict(layer=l, columns=wrong[:10], off_by=[int(res["gb"][c] - kept[:, c].sum()) for c in wrong[:10]])
        disagree += int((old_decision(z2[l], mean[l], inv[l], gamma, beta) != kept).sum())
    assert disagree > 0, "the inputs must put elements where the backward's former test disagrees with the forward"


# ---- M past the gridDim.y limit -----------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("width", ["v4", "scalar"])
def test_bn_large_m_past_grid_limit(width):
    """M just past 65535 row blocks (v4: 64 rows per block, C = 4; scalar: 128 rows per block, C = 1): computed, not refused."""
    if width == "v4":
        M, C = MAX_GRID_Y * KVEC + 1, 4
    else:
        M, C = MAX_GRID_Y * KSTAT + 1, 1
    g = torch.Generator().manual_seed(60)
    x = (torch.randn(M, C, generator=g) + 1).float()
    gamma, beta = torch.full((C,), 1.25), torch.full((C,), 0.5)
    run = BnFwd(x, gamma, beta, relu=1)
    check_bn_fwd(x, gamma, beta, 1, run)
    mean, inv = run.MEAN.view.cpu()[0], run.INV.view.cpu()[0]
    gy = torch.randn(M, C, generator=g).float()
    out = run_bn_bwd(gy, x, gamma, beta, mean, inv, 1)
    check_bn_bwd(out, bn_bwd_ref(gy, x, gamma, beta, mean, inv, 1))


# ---------------------------------------------------------------------------------------------------------------------------
# ReLU and L2 normalisation
# ---------------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("C,ld,shift", [(128, 132, 0), (33, 35, 0), (128, 128, 1)])
def test_relu_fwd_bwd_exact(C, ld, shift):
    """y = x < 0 ? 0 : x (NaN and -0.0 pass through unchanged), gx = y > 0 ? gy : 0, bit for bit, on both widths."""
    M = 1000
    g = torch.Generator().manual_seed(70)
    x = torch.randn(M, C, generator=g)
    x[0, :4] = torch.tensor([float("nan"), -0.0, 0.0, float("inf")])
    x[1, :2] = torch.tensor([-float("inf"), 1e-45])
    gy = torch.randn(M, C, generator=g)
    X, GY = filled(x, ld=ld, shift=shift), filled(gy, ld=ld, shift=shift)
    Y, GX = Region(M, C, ld, SENT, shift=shift), Region(M, C, ld, SENT, shift=shift)
    assert cabi.lib.pgnn_relu_fwd(X.ptr(), ld, M, C, Y.ptr(), ld, _st()) == OK
    assert cabi.lib.pgnn_relu_bwd(GY.ptr(), ld, Y.ptr(), ld, M, C, GX.ptr(), ld, _st()) == OK
    y = Y.view.cpu()
    ref = torch.where(x < 0, torch.zeros_like(x), x)
    assert torch.equal(y.view(torch.int32), ref.view(torch.int32))
    assert torch.equal(GX.view.cpu(), torch.where(ref > 0, gy, torch.zeros_like(gy)))
    assert Y.outside_intact() and GX.outside_intact()


L2_MAG = [1e-20, 1e-13, 1e-6, 1.0, 1e6, 1e18]


def l2_bwd_ref(gy, y, nrm, variant=None):
    """fp64 gx of y = x / max(||x||, eps) from the kernel's own y and norm, and its bound: the fp32 dot is within (C/32 + 5) u of
    sum|g y|; g - y dot and the division add three roundings.  variant "no clamp branch": (g - y <g, y>) / n on clamped rows too."""
    C = y.shape[1]
    yd, gd, nd = y.double(), gy.double(), nrm.double()[:, None]
    dot = (gd * yd).sum(1, keepdim=True)
    clamped = nd <= float(np.float32(1e-12))
    if variant == "no clamp branch":
        clamped = torch.zeros_like(clamped)
    ref = torch.where(clamped, gd / nd, (gd - yd * dot) / nd)
    k = C / 32 + 5
    bound = U * (k * (gd * yd).abs().sum(1, keepdim=True) * yd.abs() + 3 * gd.abs() + 3 * (yd * dot).abs()) / nd + 1e-300
    return ref, bound


@gpu
@pytest.mark.parametrize("C,ld", [(33, 37), (300, 300), (1, 3)])
def test_l2norm_fwd_bwd_against_fp64(C, ld):
    """Rows of magnitudes 1e-20 .. 1e18 (row norms below the 1e-12 clamp take x / eps and g / eps), zero rows, C not a
    multiple of 32.  Forward: the fp32 sum of squares is within (C/32 + 5) u of sum x^2 (per-lane fmas, a 5-step butterfly), so
    |y - y64| <= ((C/32 + 5)/2 + 2) u |y64|.  Backward on the kernel's own y and norm: gx = (g - y <g, y>) / n with the same dot
    bound."""
    if C >= 300:
        mags = L2_MAG[:-1]   # 300 squares of 1e18 overflow fp32's sum of squares, as torch's fp32 norm does
    else:
        mags = L2_MAG
    g = torch.Generator().manual_seed(71)
    rows = []
    for m in mags:
        rows.append(torch.randn(5, C, generator=g) * m)
    rows.append(torch.zeros(3, C))
    x = torch.cat(rows).float()
    M = x.shape[0]
    X, Y, NRM = filled(x, ld=ld), Region(M, C, ld + 1, SENT), Region(1, M, M, SENT)
    assert cabi.lib.pgnn_l2norm_fwd(X.ptr(), ld, M, C, Y.ptr(), Y.ld, NRM.ptr(), _st()) == OK
    torch.cuda.synchronize()
    eps32 = float(np.float32(1e-12))
    n64 = x.double().norm(dim=1).clamp_min(eps32)
    y64 = x.double() / n64[:, None]
    k = (C / 32 + 5)
    assert _excess(Y.view.cpu(), y64, (k / 2 + 2) * U * y64.abs() + 1e-300) <= 1
    assert _excess(NRM.view.cpu()[0], n64, (k / 2 + 1) * U * n64) <= 1
    gy = torch.randn(M, C, generator=g).float()
    y, nrm = Y.view.cpu(), NRM.view.cpu()[0]
    GY, YY, NN = filled(gy, ld=ld), filled(y, ld=ld + 2), filled(nrm[None])
    GX = Region(M, C, ld, SENT)
    assert cabi.lib.pgnn_l2norm_bwd(GY.ptr(), ld, YY.ptr(), YY.ld, NN.ptr(), M, C, GX.ptr(), ld, _st()) == OK
    ref, bound = l2_bwd_ref(gy, y, nrm)
    assert _excess(GX.view.cpu(), ref, bound) <= 1
    assert all(r.outside_intact() for r in (Y, NRM, GX))


# ---------------------------------------------------------------------------------------------------------------------------
# loss heads
# ---------------------------------------------------------------------------------------------------------------------------
def run_ce(logits, labels, ld, lddl):
    M, V = logits.shape
    # padding columns of the logits hold zeros, as the library's 16-byte-aligned rows do; NaN past the padded rows
    Lb = Region(M, ld, ld, NAN)
    Lb.view.zero_()
    Lb.view[:, :V] = logits.to(DEV)
    LAB = filled(labels[:, None], fill=-99)
    DL = Region(M, lddl, lddl, SENT)
    loss = torch.full((1,), NAN, dtype=torch.float64, device=DEV)
    _dev_flags()
    assert cabi.lib.pgnn_softmax_ce_fwd(Lb.ptr(), ld, M, V, LAB.ptr(), loss.data_ptr(), DL.ptr(), lddl, _st()) == OK
    flags = _dev_flags()
    dl = DL.view.cpu()
    assert DL.outside_intact()
    assert (dl[:, V:] == 0).all(), "padding columns of dlogits are zeroed"
    return float(loss.item()), dl[:, :V], flags


def ce_ref(logits, labels):
    x = logits.double()
    M, V = x.shape
    lse = torch.logsumexp(x, 1)
    valid = (labels >= 0) & (labels < V)
    lab = labels.clamp(0, V - 1)
    picked = torch.where(valid, x.gather(1, lab[:, None])[:, 0], torch.zeros_like(lse))
    terms = lse - picked
    mag = lse.abs() + picked.abs()
    p = torch.softmax(x, 1)
    onehot = torch.zeros_like(p)
    onehot[valid.nonzero()[:, 0], lab[valid]] = 1.0
    dl = (p - onehot) / M
    return float(terms.mean()), dl, mag


@gpu
@pytest.mark.parametrize("V", [1, 2, 31, 32, 33, 119, 1000])
@pytest.mark.parametrize("M", [1, 33, 4097])
def test_softmax_ce_against_fp64(V, M):
    """Loss (fp64 atomics over M rows of lse - logit[label], each within a few e of |lse| + |logit|: (M + 64) e mean(|lse| +
    |logit|)) and dlogits (exp in fp64 is within ~200 e of p for |logit - lse| <= 160, then one fp32 rounding:
    u |ref| + (256 + 8 V) e / M) against fp64; labels 0 and V-1 included; ld, lddl > V with zeroed padding columns."""
    g = torch.Generator().manual_seed(80 + V)
    logits = (torch.randn(M, V, generator=g) * 3).float()
    labels = torch.randint(0, V, (M,), generator=g)
    labels[0] = 0
    labels[-1] = V - 1
    ld, lddl = (V + 3) // 4 * 4 + 4, (V + 3) // 4 * 4 + 8
    loss, dl, flags = run_ce(logits, labels, ld, lddl)
    ref, dref, terms = ce_ref(logits, labels)
    assert flags & DEVERR_LABEL == 0
    assert abs(loss - ref) <= (M + 64) * E64 * float(terms.abs().mean()) + 1e-300
    assert _excess(dl, dref, U * dref.abs() + (256 + 8 * V) * E64 / M) <= 1


@gpu
def test_softmax_ce_large_m_and_special_rows():
    """~100 k rows at V = 119, with rows at +-80, an all-equal row, -inf entries, bad labels (-1, V: flagged, contributing their
    log-sum-exp only), then a NaN (the loss and that row's gradient are NaN, as F.cross_entropy's are)."""
    M, V = 100003, 119
    g = torch.Generator().manual_seed(81)
    logits = (torch.randn(M, V, generator=g) * 2).float()
    labels = torch.randint(0, V, (M,), generator=g)
    logits[0] = 80.0 * torch.sign(torch.randn(V, generator=g))
    logits[1] = 0.25
    logits[2, :50] = -float("inf")
    labels[2] = 60
    labels[3], labels[4] = -1, V
    ld = lddl = 120
    loss, dl, flags = run_ce(logits, labels, ld, lddl)
    ref, dref, terms = ce_ref(logits, labels)
    assert flags & DEVERR_LABEL
    assert abs(loss - ref) <= (M + 64) * E64 * float(terms.abs().mean())
    assert _excess(dl, dref, U * dref.abs() + (256 + 8 * V) * E64 / M) <= 1
    ok = labels[5:].clone()
    good = F.cross_entropy(logits[5:].double(), ok)
    assert math.isfinite(good.item())
    logits[7, 3] = float("nan")
    loss, dl, _ = run_ce(logits, labels, ld, lddl)
    assert math.isnan(loss) and torch.isnan(dl[7]).all() and torch.isfinite(dl[8]).all()
    assert math.isnan(float(F.cross_entropy(logits[5:].double(), ok)))


def run_bce(x, kind, target=None, tconst=0.0, ld=None, ldt=None, lddl=None, ws=None):
    M, N = x.shape
    X = filled(x, ld=ld or N)
    T = filled(target, ld=ldt or N, fill=7) if target is not None else None
    DL = Region(M, N, lddl or N, SENT)
    loss = torch.full((1,), NAN, dtype=torch.float64, device=DEV)
    wsb = cabi.lib.pgnn_bce_logits_workspace_bytes()
    ws = ws if ws is not None else torch.full((wsb // 4 + 4,), NAN, device=DEV)
    assert cabi.lib.pgnn_bce_logits_fwd(X.ptr(), X.ld, M, N, T.ptr() if T else None, T.ld if T else 0, kind, tconst, loss.data_ptr(),
                                        DL.ptr(), DL.ld, ws.data_ptr(), wsb, _st()) == OK
    torch.cuda.synchronize()
    assert DL.outside_intact()
    return float(loss.item()), DL.view.cpu(), ws


def bce_ref(x, kind, target=None, tconst=0.0, denominator="valid"):
    xd = x.double()
    if kind == 0:
        t, valid = torch.full_like(xd, tconst), torch.ones_like(xd, dtype=torch.bool)
    elif kind == 1:
        t, valid = target.double(), torch.ones_like(xd, dtype=torch.bool)
    else:
        t, valid = (target.double() + 1) / 2, target != 0
    terms = torch.where(valid, F.binary_cross_entropy_with_logits(xd, t, reduction="none"), torch.zeros_like(xd))
    count = float(valid.sum()) if denominator == "valid" else float(xd.numel())
    inv = 1.0 / count if count > 0 else 0.0
    loss = float(terms.sum()) * inv
    dl = torch.where(valid, (torch.sigmoid(xd) - t) * inv, torch.zeros_like(xd))
    return loss, dl, terms, inv


def bce_bounds(M, N, terms, inv, dref):
    """The fp64 fold: <= ceil(M N / (256 blocks)) sequential terms per thread, a 5-step butterfly, 8 warps, `blocks` partials,
    each term within 4 e of itself (exp / log1p); dlogits: one fp32 rounding."""
    total = M * N
    blocks = min(max(-(-total // 1024), 1), KBCE_MAX_BLOCKS)
    depth = -(-total // (256 * blocks)) + 5 + 8 + blocks + 4
    return depth * E64 * float(terms.abs().sum()) * inv + 1e-300, U * dref.abs() + 4 * E64 * inv


BCE_SIZES = [(1, 1), (4, 256), (1, 1025), (541, 1000), (3, 200003)]


@gpu
@pytest.mark.parametrize("M,N", BCE_SIZES)
@pytest.mark.parametrize("kind", ["const0", "const1", "bin", "masked"])
def test_bce_logits_against_fp64(M, N, kind):
    """Kinds 0 (targets 0 / 1), 1 and 2 from one element through exactly 256*4, to past kBceMaxBlocks*256*4 (the grid-stride loop
    and the ticket fold), with ld, ldt, lddl strides and |x| up to 1e4."""
    g = torch.Generator().manual_seed(90 + M)
    x = (torch.randn(M, N, generator=g) * 3).float()
    x.view(-1)[:: 97] *= 3000
    ld, ldt, lddl = N + 3, N + 5, N + 1
    if kind.startswith("const"):
        tc = float(kind[-1])
        loss, dl, _ = run_bce(x, 0, tconst=tc, ld=ld, lddl=lddl)
        ref, dref, terms, inv = bce_ref(x, 0, tconst=tc)
    else:
        target = torch.randint(0, 2, (M, N), generator=g) if kind == "bin" else torch.randint(-1, 2, (M, N), generator=g)
        k = 1 if kind == "bin" else 2
        loss, dl, _ = run_bce(x, k, target, ld=ld, ldt=ldt, lddl=lddl)
        ref, dref, terms, inv = bce_ref(x, k, target)
    lb, db = bce_bounds(M, N, terms, inv, dref)
    assert abs(loss - ref) <= lb, (loss, ref, lb)
    assert _excess(dl, dref, db) <= 1


@gpu
def test_bce_logits_all_missing_repeat_and_workspace_reuse():
    """Kind 2 with every target 0: loss 0 and a zero gradient (the defined value where the reference's sum / #valid is 0/0).  The
    loss repeats bit for bit, and back-to-back calls with different inputs on one workspace stay correct."""
    g = torch.Generator().manual_seed(91)
    x = torch.randn(64, 300, generator=g).float()
    loss, dl, ws = run_bce(x, 2, torch.zeros(64, 300, dtype=torch.int64))
    assert loss == 0.0 and (dl == 0).all()
    big = (torch.randn(700, 1000, generator=g) * 2).float()
    tgt = torch.randint(-1, 2, (700, 1000), generator=g)
    l1, d1, ws = run_bce(big, 2, tgt, ws=ws)
    l2, d2, ws = run_bce(big, 2, tgt, ws=ws)
    assert l1 == l2 and torch.equal(d1, d2)
    l3, _, ws = run_bce(x, 0, tconst=1.0, ws=ws)
    r3 = bce_ref(x, 0, tconst=1.0)
    assert abs(l3 - r3[0]) <= bce_bounds(64, 300, r3[2], r3[3], r3[1])[0]
    ref = bce_ref(big, 2, tgt)
    assert abs(l1 - ref[0]) <= bce_bounds(700, 1000, ref[2], ref[3], ref[1])[0]


@gpu
def test_loss_bounds_reject_wrong_variants():
    """BCE kind 2 normalised by M*N instead of the number of valid entries, and a cross-entropy gradient without its 1/M, are
    rejected by their bounds on these inputs by far more than 10x."""
    g = torch.Generator().manual_seed(92)
    x = torch.randn(50, 12, generator=g).float()
    tgt = torch.randint(-1, 2, (50, 12), generator=g)
    loss, dl, _ = run_bce(x, 2, tgt)
    ref, dref, terms, inv = bce_ref(x, 2, tgt)
    bad, dbad, _, _ = bce_ref(x, 2, tgt, denominator="all")
    lb, db = bce_bounds(50, 12, terms, inv, dref)
    assert abs(loss - ref) <= lb and abs(bad - ref) >= 10 * lb and _excess(dbad, dref, db) >= 10
    logits = torch.randn(40, 119, generator=g).float()
    labels = torch.randint(0, 119, (40,), generator=g)
    _, dl, _ = run_ce(logits, labels, 120, 120)
    _, dref, _ = ce_ref(logits, labels)
    assert _excess(dl, dref, U * dref.abs() + (256 + 8 * 119) * E64 / 40) <= 1
    assert _excess(dref * 40, dref, U * dref.abs() + (256 + 8 * 119) * E64 / 40) >= 10


# ---------------------------------------------------------------------------------------------------------------------------
# segment mean, row gather, shifted row-dot
# ---------------------------------------------------------------------------------------------------------------------------
SEG_SIZES = [0, 1, 7, 8, 24, 25, 31, 32, 33, 1000]


def segments(sizes, seed):
    n = sum(sizes)
    order = torch.from_numpy(np.random.default_rng(seed).permutation(n)).to(torch.int32)
    ptr = torch.zeros(len(sizes) + 1, dtype=torch.int32)
    ptr[1:] = torch.cumsum(torch.tensor(sizes), 0).to(torch.int32)
    seg = torch.empty(n, dtype=torch.int64)
    for b in range(len(sizes)):
        seg[order[ptr[b]:ptr[b + 1]].long()] = b
    return n, order, ptr, seg


def seg_mean_ref(x, order, ptr, variant=None):
    B = len(ptr) - 1
    out = torch.zeros(B, x.shape[1], dtype=torch.float64)
    bound = torch.zeros_like(out)
    for b in range(B):
        rows = order[ptr[b]:ptr[b + 1]].long()
        cnt = len(rows)
        s, a = x[rows].double().sum(0), x[rows].double().abs().sum(0)
        div = cnt if variant == "no clamp" else max(cnt, 1)
        out[b] = s / div if div else torch.full_like(s, float("nan"))
        # 8 row-lanes of <= cnt/8 sequential adds, an 8-way fold, the division
        bound[b] = (cnt / 8 + 10) * U * a / max(cnt, 1) + U * out[b].abs().nan_to_num(0)
    return out, bound


@gpu
@pytest.mark.parametrize("C", [4, 128, 132, 300, 516])
def test_segment_mean_fwd_bwd(C):
    """Segment sizes around the four-deep unroll (k + 24 < hi) and its tail, including empty segments (count.clamp(min=1): 0);
    column chunks of 32 float4; strides; a permuted seg_order."""
    sizes = SEG_SIZES + [3, 0, 64]
    n, order, ptr, seg = segments(sizes, seed=C)
    g = torch.Generator().manual_seed(100 + C)
    x = torch.randn(n, C, generator=g).float()
    X, OUT = filled(x, ld=C + 4), Region(len(sizes), C, C + 8, SENT)
    O_, P_ = order.to(DEV), ptr.to(DEV)
    assert cabi.lib.pgnn_segment_mean_fwd(X.ptr(), X.ld, P_.data_ptr(), O_.data_ptr(), len(sizes), C, OUT.ptr(), OUT.ld, _st()) == OK
    ref, bound = seg_mean_ref(x, order, ptr)
    out = OUT.view.cpu()
    assert _excess(out, ref, bound + 1e-300) <= 1 and OUT.outside_intact()
    gy = torch.randn(len(sizes), C, generator=g).float()
    GY, GX, SEG = filled(gy, ld=C + 4), Region(n, C, C + 4, SENT), seg.to(DEV)
    assert cabi.lib.pgnn_segment_mean_bwd(GY.ptr(), GY.ld, SEG.data_ptr(), P_.data_ptr(), n, C, GX.ptr(), GX.ld, _st()) == OK
    cnt = (ptr[1:] - ptr[:-1]).clamp_min(1).double()
    gref = gy.double()[seg] / cnt[seg][:, None]
    assert _excess(GX.view.cpu(), gref, U * gref.abs() + 1e-300) <= 1 and GX.outside_intact()
    bad, _ = seg_mean_ref(x, order, ptr, variant="no clamp")
    assert _excess(bad, ref, bound + 1e-300) == math.inf   # a missing clamp (0/0 for an empty segment) is rejected


@gpu
@pytest.mark.parametrize("pair", [False, True])
def test_row_gather_fwd_bwd(pair):
    """Gather with and without idx2, one row gathered 1000 times (float4 atomics in the backward), strides, an out-of-range
    index flagged and read as zero."""
    rows, C, m = 300, 132, 2500
    g = torch.Generator().manual_seed(110)
    x = torch.randn(rows, C, generator=g).float()
    i1 = torch.randint(0, rows, (m,), generator=g)
    i1[:1000] = 17
    i2 = torch.randint(0, rows, (m,), generator=g) if pair else None
    i1[1500] = rows   # out of range
    X, OUT = filled(x, ld=C + 4), Region(m, C, C + 8, SENT)
    I1, I2 = i1.to(DEV), (i2.to(DEV) if pair else None)
    _dev_flags()
    assert cabi.lib.pgnn_row_gather_fwd(X.ptr(), X.ld, rows, I1.data_ptr(), _ptr(I2), m, C, OUT.ptr(), OUT.ld, _st()) == OK
    assert _dev_flags() & DEVERR_GATHER
    ok = i1 < rows
    a = torch.where(ok[:, None], x[i1.clamp(max=rows - 1)], torch.zeros(1))
    ref = a + x[i2] if pair else a
    assert torch.equal(OUT.view.cpu(), ref) and OUT.outside_intact()
    gy = torch.randn(m, C, generator=g).float()
    gx0 = torch.randn(rows, C, generator=g).float()
    GY, GX = filled(gy, ld=C + 4), filled(gx0, ld=C + 8, fill=SENT)
    assert cabi.lib.pgnn_row_gather_bwd(GY.ptr(), GY.ld, I1.data_ptr(), _ptr(I2), m, C, GX.ptr(), GX.ld, rows, _st()) == OK
    gref, bound = gather_bwd_ref(gx0, i1, i2, gy)
    assert _excess(GX.view.cpu(), gref, bound) <= 1 and GX.outside_intact()


def gather_bwd_ref(gx0, i1, i2, gy, variant=None):
    """gx0 + the rows of gy added at i1 (in range) and i2, in fp64, and the bound: atomics in any order, so a sum of cnt + 1 terms
    is within cnt u of the sum of their magnitudes.  Variants: "overwrites gx" (gx0 not accumulated onto), "duplicates collapse"
    (index_put without accumulate: the last of a row's duplicates wins)."""
    rows, m = gx0.shape[0], gy.shape[0]
    ok = i1 < rows
    base = torch.zeros_like(gx0.double()) if variant == "overwrites gx" else gx0.double()
    if variant == "duplicates collapse":
        gref = base.clone()
        gref[i1[ok]] = gy.double()[ok]
        if i2 is not None:
            gref[i2] = gy.double()
    else:
        gref = base.index_add(0, i1[ok], gy.double()[ok])
        if i2 is not None:
            gref = gref.index_add(0, i2, gy.double())
    mag = gx0.double().abs().index_add(0, i1[ok], gy.double().abs()[ok])
    cnt = torch.zeros(rows, dtype=torch.float64).index_add(0, i1[ok], torch.ones(int(ok.sum()), dtype=torch.float64))
    if i2 is not None:
        mag = mag.index_add(0, i2, gy.double().abs())
        cnt = cnt.index_add(0, i2, torch.ones(m, dtype=torch.float64))
    return gref, (cnt[:, None] + 1) * U * mag + 1e-300


@gpu
@pytest.mark.parametrize("C", [1, 31, 33, 300])
@pytest.mark.parametrize("shift_kind", ["0", "1", "B-1", "B", "3B+1"])
def test_shifted_rowdot_fwd_bwd(C, shift_kind):
    """out[r] = <a[r], b[(r + shift) mod B]> (per-lane fmas over C/32 columns and a 5-step butterfly: (C/32 + 5) u sum|a b|);
    the backward's products are single roundings, and accumulate = 1 adds them onto non-zero ga / gb (one more rounding)."""
    B = 97
    shift = dict(zip(["0", "1", "B-1", "B", "3B+1"], [0, 1, B - 1, B, 3 * B + 1]))[shift_kind]
    g = torch.Generator().manual_seed(120 + C)
    a, b = torch.randn(B, C, generator=g).float(), torch.randn(B, C, generator=g).float()
    A, Bb, OUT = filled(a, ld=C + 3), filled(b, ld=C + 5), Region(1, B, B, SENT)
    assert cabi.lib.pgnn_shifted_rowdot_fwd(A.ptr(), A.ld, Bb.ptr(), Bb.ld, B, C, shift, OUT.ptr(), _st()) == OK
    perm = (torch.arange(B) + shift) % B
    prod = a.double() * b.double()[perm]
    ref = prod.sum(1)
    assert _excess(OUT.view.cpu()[0], ref, (C / 32 + 5) * U * prod.abs().sum(1) + 1e-300) <= 1 and OUT.outside_intact()
    gv = torch.randn(B, generator=g).float()
    G = filled(gv[None])
    for acc in (0, 1):
        ga0, gb0 = torch.randn(B, C, generator=g).float(), torch.randn(B, C, generator=g).float()
        GA, GB = filled(ga0, ld=C + 2, fill=SENT), filled(gb0, ld=C + 4, fill=SENT)
        assert cabi.lib.pgnn_shifted_rowdot_bwd(G.ptr(), A.ptr(), A.ld, Bb.ptr(), Bb.ld, B, C, shift, acc, GA.ptr(), GA.ld, GB.ptr(),
                                                GB.ld, _st()) == OK
        (ra, ba), (rb, bb) = rowdot_bwd_ref(gv, a, b, shift, acc, ga0, gb0)
        assert _excess(GA.view.cpu(), ra, ba) <= 1 and _excess(GB.view.cpu(), rb, bb) <= 1
        assert GA.outside_intact() and GB.outside_intact()


def rowdot_bwd_ref(gv, a, b, shift, acc, ga0, gb0, variant=None):
    """fp64 ga = g[r] b[(r + shift) % B] and gb = g[(r - shift) % B] a[(r - shift) % B], added onto ga0 / gb0 under accumulate,
    with bounds of the product's rounding (plus a possible fma contraction) and the accumulation's.  Variant "accumulate ignored"
    overwrites."""
    B = a.shape[0]
    perm = (torch.arange(B) + shift) % B
    inv = torch.empty(B, dtype=torch.long)
    inv[perm] = torch.arange(B)
    va = gv.double()[:, None] * b.double()[perm]
    vb = gv.double()[inv][:, None] * a.double()[inv]
    add = acc and variant != "accumulate ignored"
    ra, rb = (ga0.double() + va, gb0.double() + vb) if add else (va, vb)
    ba = U * (2 * va.abs() + (ga0.double().abs() if acc else 0)) + 1e-300
    bb = U * (2 * vb.abs() + (gb0.double().abs() if acc else 0)) + 1e-300
    return (ra, ba), (rb, bb)


@gpu
def test_head_bounds_reject_wrong_variants():
    """On inputs of the tests above: an L2 backward that skips the clamped g / n branch, a shifted row-dot backward that ignores
    accumulate, and a row-gather backward that overwrites gx or collapses duplicate indices -- each is rejected by its bound by
    10x or more, while the kernel passes it."""
    g = torch.Generator().manual_seed(150)
    # L2: rows below the clamp (norm 1e-13 * sqrt(C)) next to ordinary ones
    C, M = 33, 12
    x = torch.cat([torch.randn(6, C, generator=g) * 1e-13, torch.randn(6, C, generator=g)]).float()
    X, Y, NRM = filled(x), Region(M, C, C, SENT), Region(1, M, M, SENT)
    assert cabi.lib.pgnn_l2norm_fwd(X.ptr(), C, M, C, Y.ptr(), C, NRM.ptr(), _st()) == OK
    y, nrm = Y.view.cpu(), NRM.view.cpu()[0]
    gy = torch.randn(M, C, generator=g).float()
    GY, GX = filled(gy), Region(M, C, C, SENT)
    assert cabi.lib.pgnn_l2norm_bwd(GY.ptr(), C, Y.ptr(), C, NRM.ptr(), M, C, GX.ptr(), C, _st()) == OK
    ref, bound = l2_bwd_ref(gy, y, nrm)
    bad, _ = l2_bwd_ref(gy, y, nrm, variant="no clamp branch")
    assert _excess(GX.view.cpu(), ref, bound) <= 1 and _excess(bad, ref, bound) >= 10
    # shifted row-dot with accumulate = 1
    B, C, shift = 97, 33, 3 * 97 + 1
    a, b, gv = torch.randn(B, C, generator=g), torch.randn(B, C, generator=g), torch.randn(B, generator=g)
    ga0, gb0 = torch.randn(B, C, generator=g), torch.randn(B, C, generator=g)
    A, Bb, G, GA, GB = filled(a), filled(b), filled(gv[None]), filled(ga0, fill=SENT), filled(gb0, fill=SENT)
    assert cabi.lib.pgnn_shifted_rowdot_bwd(G.ptr(), A.ptr(), C, Bb.ptr(), C, B, C, shift, 1, GA.ptr(), C, GB.ptr(), C, _st()) == OK
    (ra, ba), (rb, bb) = rowdot_bwd_ref(gv, a, b, shift, 1, ga0, gb0)
    (xa, _), (xb, _) = rowdot_bwd_ref(gv, a, b, shift, 1, ga0, gb0, variant="accumulate ignored")
    assert _excess(GA.view.cpu(), ra, ba) <= 1 and _excess(GB.view.cpu(), rb, bb) <= 1
    assert _excess(xa, ra, ba) >= 10 and _excess(xb, rb, bb) >= 10
    # row gather backward: row 17 gathered 1000 times, onto a non-zero gx
    rows, C, m = 300, 132, 2500
    i1 = torch.randint(0, rows, (m,), generator=g)
    i1[:1000] = 17
    i2 = torch.randint(0, rows, (m,), generator=g)
    gy, gx0 = torch.randn(m, C, generator=g), torch.randn(rows, C, generator=g)
    GY, GX, I1, I2 = filled(gy), filled(gx0, fill=SENT), i1.to(DEV), i2.to(DEV)
    assert cabi.lib.pgnn_row_gather_bwd(GY.ptr(), C, I1.data_ptr(), I2.data_ptr(), m, C, GX.ptr(), C, rows, _st()) == OK
    gref, bound = gather_bwd_ref(gx0, i1, i2, gy)
    assert _excess(GX.view.cpu(), gref, bound) <= 1
    for variant in ("overwrites gx", "duplicates collapse"):
        assert _excess(gather_bwd_ref(gx0, i1, i2, gy, variant)[0], gref, bound) >= 10, variant


def test_fma32_is_fp32_fma():
    """ops.fma32 (the host restatement of the BatchNorm pre-activation these tests and ops.chem_gin_relu_masks use) rounds once:
    checked against exact rational arithmetic on random triples, on c = -(a*b rounded) (the exact rounding error of the product),
    and on constructed ties: a*b = 2^-24 (1 - 2^-46) s (a = 2^-24 (1 + 2^-23) s, b = 1 - 2^-23) added to c = +-(1 + 2^-23) s. The
    fp64 sum then lies exactly halfway between two floats, 2^-70 s short of / past the true value, so plain fp64 -> fp32
    rounding (ties to even) is wrong on both -- once rounding down, once up in magnitude -- and only the TwoSum branch is right."""
    from fractions import Fraction
    g = torch.Generator().manual_seed(130)
    a, b = torch.randn(3000, generator=g), torch.randn(3000, generator=g)
    c = torch.cat([torch.randn(1500, generator=g) * 3, (-(a[1500:].double() * b[1500:].double())).float()])
    r = ops.fma32(a, b, c)
    scales = torch.tensor([1.0, 2.0 ** -20, 2.0 ** 30, 2.0 ** -3]).repeat_interleave(2)  # powers of two keep the construction exact
    ta = (2.0 ** -24 * (1 + 2.0 ** -23)) * scales
    tb = torch.full_like(ta, 1 - 2.0 ** -23)
    tc = (1 + 2.0 ** -23) * scales * torch.tensor([1.0, -1.0]).repeat(4)
    tr = ops.fma32(ta.float(), tb.float(), tc.float())
    naive = (ta.double() * tb.double() + tc.double()).float()
    assert bool((tr != naive).all()), "every constructed triple lands on an fp32 tie that ties-to-even gets wrong"
    a, b, c, r = torch.cat([a, ta.float()]), torch.cat([b, tb.float()]), torch.cat([c, tc.float()]), torch.cat([r, tr])
    for i in list(range(0, 3000, 7)) + list(range(3000, 3000 + len(ta))):
        v = Fraction(float(a[i])) * Fraction(float(b[i])) + Fraction(float(c[i]))
        f = np.float32(float(v))
        cands = [np.nextafter(f, np.float32(-np.inf)), f, np.nextafter(f, np.float32(np.inf))]
        best = min(cands, key=lambda q: (abs(Fraction(float(q)) - v), int(np.float32(q).view(np.int32)) & 1))
        assert np.float32(r[i].item()) == best, i


NVCC = "/usr/local/cuda/bin/nvcc"


@pytest.mark.skipif(not (os.path.exists(NVCC) or shutil.which("nvcc")), reason="nvcc not available")
@pytest.mark.parametrize("unit", ["norm", "aggregate"])
def test_ptxas_no_spills(unit, tmp_path):
    """Every kernel of norm.cu and aggregate.cu compiles for sm_90a without spills, and k_bn_bwd_apply_colsum<4, false> (the
    encoder's BatchNorm backward sweep) fits three 256-thread CTAs per SM (<= 80 registers)."""
    nvcc = NVCC if os.path.exists(NVCC) else shutil.which("nvcc")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = os.path.join(root, "pretrain-gnns_b200", "csrc", unit + ".cu")
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--expt-relaxed-constexpr",
           "-I" + os.path.join(root, "include"), "-Xptxas", "-v", "-c", src, "-o", str(tmp_path / (unit + ".o"))]
    out = subprocess.run(cmd, capture_output=True, text=True)
    assert out.returncode == 0, out.stderr[-4000:]
    kernels, cur = {}, None
    for line in (out.stdout + out.stderr).splitlines():
        m = re.search(r"Compiling entry function '(\w+)'", line)
        if m:
            cur = m.group(1)
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if cur and m:
            kernels[cur] = [int(m.group(1)) + int(m.group(2))]
        m = re.search(r"Used (\d+) registers", line)
        if cur and m and cur in kernels:
            kernels[cur].append(int(m.group(1)))
            cur = None
    assert len(kernels) == (24 if unit == "norm" else 11), sorted(kernels)
    assert all(v[0] == 0 for v in kernels.values()), kernels
    if unit == "norm":
        (regs,) = [v[1] for k, v in kernels.items() if re.search(r"k_bn_bwd_apply_colsumILi4ELb0EE", k)]
        assert regs <= 80, regs
