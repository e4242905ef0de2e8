"""The 3xTF32 wgmma GEMM (dense_tc.cu, precision 1) and the FFMA GEMM (dense.cu, precision 0) against a plain fp64 matmul of the
same fp32 inputs, followed by the same epilogue written out in fp64.

The tensor-core kernel is driven through its test entry points (include/pgnn_b200.h, pgnn_debug_*), which choose the operand
majors, the tile width and the epilogue; the production entry points pgnn_linear_* are checked at the shapes of the masking
step on both precisions.  Families:
  * bit-exact: integer A, B = n (1 + 2^-12) (the lo part in one operand only).  Every hi*hi product sum is an integer S and the
    cross terms sum to S 2^-12, so the exact result S (1 + 2^-12) is an fp32 number: any misplaced element, swizzle slip, dropped
    tail or dropped cross term changes bits.  Compared with torch.equal.
  * random: per element |C - C64| / sum_k |a_mk| |b_nk| <= TAU.  The CPU tests at the bottom emulate the scheme and show that TAU
    accepts 3xTF32 and an fp32 GEMM and rejects plain TF32 and each single-cross-term variant.
Every operand is a view inside a NaN-filled allocation (row stride past the extent, rows and slack past the end), so an
over-read shows up as NaN in the result; every output sits in a sentinel-filled allocation whose sentinels must survive.
"""
import ctypes
import importlib
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest
import torch

from device_buffers import DEV, NAN, SENT, Region, ceil4 as _ceil4, card as _card, operand, zeroed
from golden_util import write_report

cabi = importlib.import_module("pretrain-gnns_b200._cabi")
gpu = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OK, EINVAL, EUNSUPPORTED = 0, -1, -4
LAYOUTS = ((1, 1), (1, 0), (0, 1), (0, 0))  # (A reduction-contiguous, B reduction-contiguous)
COMBOS = [(ak, bk, bn) for ak, bk in LAYOUTS for bn in (64, 128)]
# Bound on the normalized error of both GEMMs.  CPU emulation (test_tau_separates_the_scheme_from_its_bugs): 3xTF32 <= 2e-7, an
# fp32 GEMM <= 2e-7, one cross term dropped >= 1.1e-4, plain TF32 >= 2e-4.  Measured on an H100 80GB HBM3 at 700 W: <= 6.2e-7 for
# K <= 600, 1.24e-6 for the 5986-long reduction, in every layout and tile width (DESIGN.md §4).
TAU = 5e-6


def _stream():
    return torch.cuda.current_stream().cuda_stream


def tc_gemm(a, b, a_kc, b_kc, bn, bias=None, relu=False, mask=None, ldm_pad=4, mask_shift=0, colsum=False, stats=False, S=None,
            q_split=0, ldc_pad=4, pads=(4, 8), keep_operands=False):
    """pgnn_debug_tc_gemm on a [M,K], b [N,K]; returns the outputs on the CPU and whether every sentinel survived.  Row strides
    of C and the mask: the extent rounded up to 4, plus ldc_pad / ldm_pad."""
    M, K = a.shape
    N = b.shape[0]
    A, B = operand(a, a_kc, pads[0]), operand(b, b_kc, pads[1])
    C = Region(M, N, _ceil4(N) + ldc_pad, SENT)
    outs = {"C": C}
    bias_d = None if bias is None else bias.to(DEV)
    mk = None
    if mask is not None:
        mk = Region(M, N, _ceil4(N) + ldm_pad, NAN, shift=mask_shift)
        mk.view.copy_(mask)
    if colsum:
        outs["colsum"] = zeroed(1, N, N + 4)
    if stats:
        outs["stats"] = zeroed(2, N, N, torch.float64)
    Q, ldt, S_d = 0, N + 4, None
    if S is not None:
        Q = S.shape[1]
        S_d = S.contiguous().to(DEV)
        if q_split > 0:
            outs["gT"] = zeroed(q_split, N, ldt)
        if q_split < Q:
            outs["gT2"] = zeroed(Q - q_split, N, ldt)
    p = lambda k: outs[k].ptr() if k in outs else None
    rc = cabi.lib.pgnn_debug_tc_gemm(a_kc, b_kc, bn, A.ptr(), A.ld, B.ptr(), B.ld, C.ptr(), C.ld, M, N, K,
                                     None if bias_d is None else bias_d.data_ptr(), int(relu), None if mk is None else mk.ptr(),
                                     0 if mk is None else mk.ld, p("colsum"), p("stats"), None if S_d is None else S_d.data_ptr(),
                                     Q, p("gT"), p("gT2"), q_split, ldt, _stream())
    assert rc == OK, rc
    torch.cuda.synchronize()
    res = {k: r.view.cpu() for k, r in outs.items()}
    res["intact"] = all(r.outside_intact() for r in outs.values())
    if keep_operands:
        res["A"], res["B"] = A.view.cpu(), B.view.cpu()
    return res


def reference(a, b, bias=None, relu=False, mask=None):
    c = a.double() @ b.double().t()
    if bias is not None:
        c = c + bias.double()
    if relu:
        c = torch.where(c < 0, torch.zeros_like(c), c)  # keeps NaN, as torch.relu
    if mask is not None:
        c = torch.where(mask > 0, c, torch.zeros_like(c))
    return c


def scale_of(a, b, bias=None):
    d = a.double().abs() @ b.double().abs().t()
    return d if bias is None else d + bias.double().abs()


def norm_err(c, ref, den):
    """max over the output of |c - ref| / sum_k |a_mk| |b_nk| (exact agreement required where that sum is 0; NaN propagates)."""
    e = (c.double() - ref).abs()
    e = torch.where(den > 0, e / den.clamp_min(1e-300), torch.where(e == 0, 0.0, float("inf")))
    return float(e.max()) if e.numel() else 0.0


def exact_pair(M, N, K, seed, lo_in="b"):
    """Bit-exact family: integers in [-2, 2] for one operand, n (1 + 2^-12) for the other (trunc_tf32 = n, lo = n 2^-12)."""
    g = torch.Generator().manual_seed(seed)
    ints = lambda r: torch.randint(-2, 3, (r, K), generator=g).float()
    a, b = ints(M), ints(N)
    if lo_in == "b":
        b = b * (1 + 2 ** -12)
    else:
        a = a * (1 + 2 ** -12)
    return a, b


def exact_ref(a, b, **ep):
    ref = reference(a, b, **ep)
    r32 = ref.float()
    assert torch.equal(r32.double(), ref), "bit-exact family: the exact result must be an fp32 number (|S| < 4096)"
    return r32


def rnd(*shape, seed=0):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed))


# ---------------------------------------------------------------------------------------------------------------------------
# a. bit-exact family: layouts x tile widths, both placements of the lo part
# ---------------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("lo_in", ["a", "b"])
@pytest.mark.parametrize("M,N,K", [(200, 190, 300), (129, 65, 36)])
def test_bit_exact_every_layout_and_tile(M, N, K, lo_in):
    a, b = exact_pair(M, N, K, seed=M + N + K, lo_in=lo_in)
    ref = exact_ref(a, b)
    for ak, bk, bn in COMBOS:
        r = tc_gemm(a, b, ak, bk, bn)
        assert r["intact"], (ak, bk, bn)
        assert torch.equal(r["C"], ref), (ak, bk, bn, int((r["C"] != ref).sum()))


# ---------------------------------------------------------------------------------------------------------------------------
# c. shape edges, one extent at a time (bit-exact family), and the production shapes (random family)
# ---------------------------------------------------------------------------------------------------------------------------
EDGE_SHAPES = ([(m, 123, 300) for m in (1, 63, 64, 65, 127, 128, 129, 5986)]
               + [(129, n, 300) for n in (1, 3, 4, 63, 64, 65, 119, 123, 127, 128, 129, 300, 600)]
               + [(129, 123, k) for k in (1, 3, 4, 8, 31, 32, 33, 36, 300, 600, 1028)])


@gpu
@pytest.mark.parametrize("M,N,K", EDGE_SHAPES)
def test_shape_edges_bit_exact(M, N, K):
    for i, (ak, bk, bn) in enumerate(COMBOS):
        a, b = exact_pair(M, N, K, seed=7 * M + N + K, lo_in="ab"[i % 2])
        ref = exact_ref(a, b)
        r = tc_gemm(a, b, ak, bk, bn)
        assert r["intact"], (ak, bk, bn)
        assert torch.equal(r["C"], ref), (ak, bk, bn, int((r["C"] != ref).sum()))


# b. random family: the error level of the scheme, per layout and tile width (reported)
RANDOM_SHAPES = [(300, 200, 32), (300, 200, 300), (300, 200, 600),
                 (5986, 600, 300), (5986, 300, 600),  # GIN layer GEMM1 / GEMM2 and the two dgrads, B = 256
                 (1020, 119, 300), (1020, 300, 119),  # masking head: logits, dgrad over the 119 classes
                 (123, 300, 5986)]                    # one-hot embedding wgrad as one unsplit reduction


@gpu
@pytest.mark.parametrize("M,N,K", RANDOM_SHAPES)
def test_random_error_level(M, N, K):
    a, b = rnd(M, K, seed=1), rnd(N, K, seed=2)
    ref, den = reference(a, b), scale_of(a, b)
    rows, worst = [], 0.0
    for ak, bk, bn in COMBOS:
        r = tc_gemm(a, b, ak, bk, bn)
        e = norm_err(r["C"], ref, den)
        rows.append(dict(kind="A%s B%s bn%d" % ("K" if ak else "MN", "K" if bk else "MN", bn), name="%dx%dx%d" % (M, N, K),
                         err=e, err_ref32=0.0, intact=r["intact"]))
        worst = max(worst, e)
        assert r["intact"], (ak, bk, bn)
    write_report("gemm_random_%dx%dx%d" % (M, N, K), rows, dict(tau=TAU, **_card()))
    assert worst <= TAU, rows


# ---------------------------------------------------------------------------------------------------------------------------
# production entry points (pgnn_linear_*) at the masking step's shapes, both precisions
# ---------------------------------------------------------------------------------------------------------------------------
def _lin_fwd(prec, x, w, bias, relu, ldy):
    M, K = x.shape
    N = w.shape[0]
    X, W = Region(M, K, K, NAN), Region(N, K, K, NAN)
    X.view.copy_(x)
    W.view.copy_(w)
    Y = Region(M, N, ldy, SENT)
    bd = None if bias is None else bias.to(DEV)
    cabi.check(cabi.lib.pgnn_linear_fwd(X.ptr(), K, W.ptr(), None if bd is None else bd.data_ptr(), M, N, K, int(relu), Y.ptr(), ldy,
                                        prec, _stream()), "linear_fwd")
    torch.cuda.synchronize()
    return Y.view.cpu(), Y.outside_intact()


def _lin_bwd_x(prec, gy, ldgy, w, relu_src):
    M, N = gy.shape
    K = w.shape[1]
    G, W = Region(M, N, ldgy, NAN), Region(N, K, K, NAN)
    G.view.copy_(gy)
    W.view.copy_(w)
    R = None
    if relu_src is not None:
        R = Region(M, K, K, NAN)
        R.view.copy_(relu_src)
    GX = Region(M, K, K, SENT)
    cabi.check(cabi.lib.pgnn_linear_bwd_x(G.ptr(), ldgy, W.ptr(), M, N, K, None if R is None else R.ptr(), K, GX.ptr(), K, prec,
                                          _stream()), "linear_bwd_x")
    torch.cuda.synchronize()
    return GX.view.cpu(), GX.outside_intact()


def _lin_bwd_w(prec, gy, ldgy, x):
    M, N = gy.shape
    K = x.shape[1]
    G, X = Region(M, N, ldgy, NAN), Region(M, K, K, NAN)
    G.view.copy_(gy)
    X.view.copy_(x)
    GW, GB = Region(N, K, K, SENT), Region(1, N, N, SENT)
    cabi.check(cabi.lib.pgnn_linear_bwd_w(G.ptr(), ldgy, X.ptr(), K, M, N, K, GW.ptr(), GB.ptr(), prec, _stream()), "linear_bwd_w")
    torch.cuda.synchronize()
    return GW.view.cpu(), GB.view.cpu()[0], GW.outside_intact() and GB.outside_intact()


def _colsum_ok(got, rows):
    """fp32 column sums (sequential per CTA, atomics across CTAs) against fp64, bounded on the sum of magnitudes."""
    ref = rows.double().sum(0)
    return bool(((got.double() - ref).abs() <= 2e-5 * rows.double().abs().sum(0) + 1e-30).all())


PRODUCTION = {  # name: (M, N, K, ld of the N-wide operand)
    "gin_gemm1": (5986, 600, 300, 600), "gin_gemm2": (5986, 300, 600, 300),
    "head": (1020, 119, 300, 120), "onehot": (5986, 123, 300, 124),
}


@gpu
@pytest.mark.parametrize("prec", [0, 1])
@pytest.mark.parametrize("name", ["gin_gemm1", "gin_gemm2", "head"])
def test_production_fwd_and_dgrad(name, prec):
    M, N, K, ldn = PRODUCTION[name]
    x, w, bias = rnd(M, K, seed=1), rnd(N, K, seed=2) * 0.06, rnd(N, seed=3)
    relu = name == "gin_gemm1"
    y, intact = _lin_fwd(prec, x, w, bias, relu, ldn)
    assert intact
    assert norm_err(y, reference(x, w, bias=bias, relu=relu), scale_of(x, w, bias)) <= TAU
    # dgrad of the same layer: gx[M,K] = gy[M,N] . w[N,K], masked by the layer input's ReLU where it has one
    gy = torch.zeros(M, ldn)
    gy[:, :N] = rnd(M, N, seed=4)
    relu_src = rnd(M, K, seed=5) if name == "gin_gemm2" else None
    gx, intact = _lin_bwd_x(prec, gy[:, :N], ldn, w, relu_src)
    assert intact
    assert norm_err(gx, reference(gy[:, :N], w.t(), mask=relu_src), scale_of(gy[:, :N], w.t())) <= TAU


@gpu
@pytest.mark.parametrize("prec", [0, 1])
@pytest.mark.parametrize("name", ["gin_gemm1", "gin_gemm2", "head", "onehot"])
def test_production_wgrad(name, prec):
    M, N, K, ldn = PRODUCTION[name]
    if name == "onehot":  # onehot[m, code] = 1 for the atom code (rows 0..119) and the chirality code (rows 120..122)
        gy = torch.zeros(M, N)
        g = torch.Generator().manual_seed(6)
        gy[torch.arange(M), torch.randint(0, 120, (M,), generator=g)] = 1.0
        gy[torch.arange(M), 120 + torch.randint(0, 3, (M,), generator=g)] = 1.0
    else:
        gy = rnd(M, N, seed=6)
    x = rnd(M, K, seed=7)
    gw, gb, intact = _lin_bwd_w(prec, gy, ldn, x)
    assert intact
    assert norm_err(gw, reference(gy.t(), x.t()), scale_of(gy.t(), x.t())) <= TAU
    assert _colsum_ok(gb, gy)


# ---------------------------------------------------------------------------------------------------------------------------
# d + e. strides, alignment, sentinels and the fused epilogues (bit-exact family: every output compared exactly)
# ---------------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("ldc_pad,ldm_pad,mask_shift", [(4, 4, 0), (3, 1, 1)])  # aligned; ldc, ldm % 4 != 0, mask + 1 float
def test_bias_relu_mask_epilogues(ldc_pad, ldm_pad, mask_shift):
    M, N, K = 200, 123, 300
    a, b = exact_pair(M, N, K, seed=3, lo_in="b")
    bias = torch.randint(-8, 9, (N,), generator=torch.Generator().manual_seed(4)).float()
    mask = torch.tensor([-1.0, -0.0, 0.0, NAN, 1.0])[torch.randint(0, 5, (M, N), generator=torch.Generator().manual_seed(5))]
    for ak, bk, bn in COMBOS:
        for ep in (dict(bias=bias), dict(bias=bias, relu=True), dict(mask=mask), dict(bias=bias, relu=True, mask=mask)):
            ref = exact_ref(a, b, **ep)
            r = tc_gemm(a, b, ak, bk, bn, ldc_pad=ldc_pad, ldm_pad=ldm_pad, mask_shift=mask_shift, **ep)
            assert r["intact"], (ak, bk, bn, list(ep))
            assert torch.equal(r["C"], ref), (ak, bk, bn, list(ep), int((r["C"] != ref).sum()))


@gpu
@pytest.mark.parametrize("Q,q_split", [(1, 0), (1, 1), (9, 0), (9, 6), (9, 9), (16, 0), (16, 6), (16, 16)])
def test_fused_column_reductions(Q, q_split):
    M, N, K = 333, 190, 300
    a, b = exact_pair(M, N, K, seed=Q + q_split, lo_in="a")
    bias = torch.randint(-4, 5, (N,), generator=torch.Generator().manual_seed(9)).float()
    S = rnd(M, Q, seed=10)
    ref = exact_ref(a, b, bias=bias, relu=True)
    for ak, bk, bn in COMBOS:
        r = tc_gemm(a, b, ak, bk, bn, bias=bias, relu=True, colsum=True, stats=True, S=S, q_split=q_split)
        assert r["intact"], (ak, bk, bn)
        C = r["C"]
        assert torch.equal(C, ref), (ak, bk, bn)
        c64 = C.double()
        assert _colsum_ok(r["colsum"][0], C), (ak, bk, bn)
        st = r["stats"]
        assert bool(((st[0] - c64.sum(0)).abs() <= 1e-12 * c64.abs().sum(0)).all()), (ak, bk, bn)
        assert bool(((st[1] - (c64 * c64).sum(0)).abs() <= 1e-12 * (c64 * c64).sum(0)).all()), (ak, bk, bn)
        gt_ref, gt_den = S.double().t() @ c64, S.double().abs().t() @ c64.abs()
        got = torch.cat([r[k] for k in ("gT", "gT2") if k in r]).double()
        assert bool(((got - gt_ref).abs() <= 2e-5 * gt_den + 1e-30).all()), (ak, bk, bn, float((got - gt_ref).abs().max()))


# ---------------------------------------------------------------------------------------------------------------------------
# f. weight gradient: split-K plan boundaries, the ordered fold (bit-reproducible) and the atomic path
# ---------------------------------------------------------------------------------------------------------------------------
def _plan(M, N, K):
    out = (ctypes.c_int64 * 4)()
    assert cabi.lib.pgnn_debug_tc_wgrad_plan(M, N, K, out) == OK
    return dict(bn=out[0], tiles=out[1], splits=out[2], per=out[3])


def _tc_wgrad(G, X, M, N, K, partials, partial_floats):
    GW, GB = Region(N, K, K, SENT), Region(1, N, N, SENT)
    rc = cabi.lib.pgnn_debug_tc_wgrad(G.ptr(), G.ld, X.ptr(), X.ld, M, N, K, GW.ptr(), GB.ptr(), partials, partial_floats, _stream())
    assert rc == OK, rc
    torch.cuda.synchronize()
    assert GW.outside_intact() and GB.outside_intact()
    return GW.view.cpu(), GB.view.cpu()[0]


@gpu
@pytest.mark.parametrize("M", [40, 1023, 1024, 1025, 16383, 16384, 16385, 32000])
def test_wgrad_split_k(M):
    N, K = 300, 600
    gy, x = rnd(M, N, seed=M), rnd(M, K, seed=M + 1)
    G, X = Region(M, N, N + 4, NAN), Region(M, K, K + 8, NAN)
    G.view.copy_(gy)
    X.view.copy_(x)
    plan = _plan(M, N, K)
    need = plan["splits"] * N * K
    ref, den = reference(gy.t(), x.t()), scale_of(gy.t(), x.t())
    part = torch.full((need + 64,), SENT, device=DEV)
    gw1, gb1 = _tc_wgrad(G, X, M, N, K, part.data_ptr(), need)
    gw2, gb2 = _tc_wgrad(G, X, M, N, K, part.data_ptr(), need)
    assert torch.equal(gw1, gw2), "the ordered split-K fold must repeat bit for bit"
    assert bool((part[need:] == SENT).all()), "partial tiles past splits * N * K"
    assert (plan["splits"] > 1) == bool((part[:need] != SENT).any()), plan
    rows = [dict(kind="partials", name=str(M), err=norm_err(gw1, ref, den), err_ref32=0.0, **plan)]
    for label, floats in (("atomics", 0), ("too few partials", need - 1)):
        part.fill_(SENT)
        gw, gb = _tc_wgrad(G, X, M, N, K, part.data_ptr() if floats else None, floats)
        assert bool((part == SENT).all()), label + ": the workspace must not be touched"
        rows.append(dict(kind=label, name=str(M), err=norm_err(gw, ref, den), err_ref32=0.0, **plan))
        assert _colsum_ok(gb, gy), label
    write_report("gemm_wgrad_%d" % M, rows, dict(tau=TAU, **_card()))
    assert _colsum_ok(gb1, gy) and torch.equal(gb1.isnan(), torch.zeros(N, dtype=torch.bool))
    assert max(r["err"] for r in rows) <= TAU, rows


# ---------------------------------------------------------------------------------------------------------------------------
# g. shapes and pointers the tensor path refuses: the FFMA kernels answer, with the same bound
# ---------------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("case", ["K % 4", "base + 1 float", "ld % 4"])
def test_fallback_to_ffma(case):
    M, N, K = 300, 190, 299 if case == "K % 4" else 300
    ld = K + 1 if case == "ld % 4" else K
    shift = 1 if case == "base + 1 float" else 0
    x, w, gy = rnd(M, K, seed=1), rnd(N, K, seed=2), rnd(M, N, seed=3)
    X = Region(M, K, ld, NAN, shift=shift)
    X.view.copy_(x)
    W = Region(N, K, K, NAN)
    W.view.copy_(w)
    G = Region(M, N, N, NAN)
    G.view.copy_(gy)
    if case != "K % 4":  # the tensor-core entry itself refuses the operand
        C = Region(M, N, N, SENT)
        assert cabi.lib.pgnn_debug_tc_gemm(1, 1, 128, X.ptr(), ld, W.ptr(), K, C.ptr(), N, M, N, K, None, 0, None, 0, None, None,
                                           None, 0, None, None, 0, 0, _stream()) == EUNSUPPORTED
    Y = Region(M, N, N, SENT)
    cabi.check(cabi.lib.pgnn_linear_fwd(X.ptr(), ld, W.ptr(), None, M, N, K, 0, Y.ptr(), N, 1, _stream()))
    GX = Region(M, K, ld, SENT, shift=shift)
    cabi.check(cabi.lib.pgnn_linear_bwd_x(G.ptr(), N, W.ptr(), M, N, K, None, 0, GX.ptr(), ld, 1, _stream()))
    GW = Region(N, K, K, SENT)
    cabi.check(cabi.lib.pgnn_linear_bwd_w(G.ptr(), N, X.ptr(), ld, M, N, K, GW.ptr(), None, 1, _stream()))
    torch.cuda.synchronize()
    assert Y.outside_intact() and GX.outside_intact() and GW.outside_intact()
    assert norm_err(Y.view.cpu(), reference(x, w), scale_of(x, w)) <= TAU
    assert norm_err(GX.view.cpu(), reference(gy, w.t()), scale_of(gy, w.t())) <= TAU
    assert norm_err(GW.view.cpu(), reference(gy.t(), x.t()), scale_of(gy.t(), x.t())) <= TAU


# ---------------------------------------------------------------------------------------------------------------------------
# h. non-finite values propagate as in fp32
# ---------------------------------------------------------------------------------------------------------------------------
LOW_NAN_BITS = 0x7F800001


def _nonfinite_pair(where):
    M, N, K = 70, 67, 40
    g = torch.Generator().manual_seed(12)
    a = torch.randn(M, K, generator=g)
    choices = torch.tensor([0.0, 0.5, -0.5, 1.5, -0.0])
    b = torch.where(torch.rand(N, K, generator=g) < 0.6, choices[torch.randint(0, 5, (N, K), generator=g)], torch.randn(N, K, generator=g))
    for (m, k), v in {(3, 5): float("inf"), (10, 7): float("-inf"), (20, 11): NAN, (40, 2): float("inf"), (40, 30): float("-inf")}.items():
        a[m, k] = v
    a.view(torch.int32)[33, 13] = LOW_NAN_BITS  # a NaN whose payload lies only in the 13 bits trunc_tf32 drops
    return (a, b) if where == "a" else (b, a)


def _classes(c):
    return c.isnan(), c == float("inf"), c == float("-inf")


def _fp32_semantics(a, b, relu):
    # elementwise IEEE products, summed in fp64: where fp32 gives NaN / +Inf / -Inf
    c = (a.double()[:, None, :] * b.double()[None, :, :]).sum(-1)
    return torch.where(c < 0, torch.zeros_like(c), c) if relu else c


@gpu
@pytest.mark.parametrize("where", ["a", "b"])
@pytest.mark.parametrize("relu", [False, True])
def test_non_finite_values(where, relu):
    a, b = _nonfinite_pair(where)
    ref = _fp32_semantics(a, b, relu)
    want = _classes(ref)
    assert want[0].any() and want[1].any() and (relu or want[2].any())
    fin = torch.isfinite(ref)
    den = scale_of(torch.nan_to_num(a, 0.0, 0.0, 0.0), torch.nan_to_num(b, 0.0, 0.0, 0.0))
    results = []
    for ak, bk, bn in COMBOS:
        r = tc_gemm(a, b, ak, bk, bn, relu=relu, keep_operands=True)
        for got, t, kc in ((r["A"], a, ak), (r["B"], b, bk)):  # the planted bits reached the device (stored layout)
            assert torch.equal(got.view(torch.int32), (t if kc else t.t()).contiguous().view(torch.int32))
        results.append(("tc", ak, bk, bn, r["C"]))
    for prec in (0, 1):
        results.append(("linear", prec, 1, 0, _lin_fwd(prec, a, b, None, relu, b.shape[0])[0]))
    for tag in results:
        got = _classes(tag[-1])
        for g, w, what in zip(got, want, ("NaN", "+Inf", "-Inf")):
            assert torch.equal(g, w), (tag[:4], what, int((g != w).sum()))
        assert norm_err(tag[-1][fin], ref[fin], den[fin]) <= TAU, tag[:4]


# ---------------------------------------------------------------------------------------------------------------------------
# i. the weight-transpose batch of the encoder backward
# ---------------------------------------------------------------------------------------------------------------------------
def _transpose(shapes):
    ins, outs = [], []
    for i, (r, c) in enumerate(shapes):
        t = rnd(r, c, seed=i)
        ins.append(t.to(DEV))
        o = torch.full((r * c + 9,), SENT, device=DEV)
        outs.append(o)
    n = len(shapes)
    rc = cabi.lib.pgnn_debug_transpose_batch(n, (ctypes.c_void_p * n)(*[t.data_ptr() for t in ins]),
                                             (ctypes.c_void_p * n)(*[o.data_ptr() for o in outs]),
                                             (ctypes.c_int32 * n)(*[s[0] for s in shapes]), (ctypes.c_int32 * n)(*[s[1] for s in shapes]),
                                             _stream())
    torch.cuda.synchronize()
    return rc, ins, outs


@gpu
def test_transpose_batch_bit_exact():
    shapes = [(600, 300), (300, 600), (37, 45), (1, 70), (65, 1), (33, 31), (1, 1), (96, 64)]
    shapes = (shapes * 4)[:32]
    rc, ins, outs = _transpose(shapes)
    assert rc == OK
    for (r, c), t, o in zip(shapes, ins, outs):
        assert torch.equal(o[:r * c].view(c, r), t.t()), (r, c)
        assert bool((o[r * c:] == SENT).all()), (r, c)
    rc, _, outs = _transpose(shapes + [(8, 8)])
    assert rc == EUNSUPPORTED and all(bool((o == SENT).all()) for o in outs)


# ---------------------------------------------------------------------------------------------------------------------------
# j. two devices in one process: the shared-memory opt-in is per device
# ---------------------------------------------------------------------------------------------------------------------------
_TWO_DEVICES = textwrap.dedent("""
    import sys
    sys.path.insert(0, sys.argv[1]); sys.path.insert(0, sys.argv[1] + "/tests")
    import torch
    import device_buffers as B
    import test_gpu_gemm as T
    a, b = T.rnd(300, 600, seed=1), T.rnd(190, 600, seed=2)
    ref, den = T.reference(a, b), T.scale_of(a, b)
    for d in (0, 1):
        torch.cuda.set_device(d)
        B.DEV = T.DEV = "cuda:%d" % d
        for ak, bk, bn in T.COMBOS:
            e = T.norm_err(T.tc_gemm(a, b, ak, bk, bn)["C"], ref, den)
            assert e <= T.TAU, (d, ak, bk, bn, e)
    print("two devices ok")
""")


@gpu
def test_two_devices_in_one_process():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two visible GPUs")
    r = subprocess.run([sys.executable, "-c", _TWO_DEVICES, ROOT], capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0 and "two devices ok" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]


# ---------------------------------------------------------------------------------------------------------------------------
# CPU: the bound can see the bugs it is meant to catch; the split-K plan; argument checks that return before any launch
# ---------------------------------------------------------------------------------------------------------------------------
def _split_np(x):
    hi = (x.view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)
    return hi, (x - hi).astype(np.float32)


def emulate(a, b, variant):
    """C = a . b^T (fp32 numpy) as `variant` computes it; tensor-core accumulation modelled as fp64 sums rounded to fp32."""
    if variant == "fp32":
        return (a @ b.T).astype(np.float32)
    (ah, al), (bh, bl) = _split_np(a), _split_np(b)
    d = np.float64
    main = (ah.astype(d) @ bh.astype(d).T).astype(np.float32)
    if variant == "tf32":
        return main
    lo_hi, hi_lo = al.astype(d) @ bh.astype(d).T, ah.astype(d) @ bl.astype(d).T
    cross = {"3xtf32": lo_hi + hi_lo, "no lo*hi": hi_lo, "no hi*lo": lo_hi}[variant].astype(np.float32)
    return main + cross


def test_tau_separates_the_scheme_from_its_bugs():
    rng = np.random.default_rng(0)
    for K in (32, 300, 600):
        a, b = rng.standard_normal((96, K)).astype(np.float32), rng.standard_normal((80, K)).astype(np.float32)
        ref = torch.from_numpy(a.astype(np.float64) @ b.astype(np.float64).T)
        den = torch.from_numpy(np.abs(a).astype(np.float64) @ np.abs(b).astype(np.float64).T)
        err = {v: norm_err(torch.from_numpy(emulate(a, b, v)), ref, den) for v in ("3xtf32", "fp32", "tf32", "no lo*hi", "no hi*lo")}
        assert err["3xtf32"] <= TAU and err["fp32"] <= TAU, (K, err)
        for v in ("tf32", "no lo*hi", "no hi*lo"):
            assert err[v] >= 5 * TAU, (K, v, err)


def test_exact_family_premise():
    for n in range(-8, 9):
        b = np.array([n * (1 + 2 ** -12)], dtype=np.float32)
        hi, lo = _split_np(b)
        assert hi[0] == n and lo[0] == n * 2.0 ** -12


def test_wgrad_plan_invariants():
    for M in (1, 31, 32, 33, 63, 64, 65, 1000, 1023, 1024, 1025, 2047, 5986, 16383, 16384, 16385, 32000, 100000, 1 << 20):
        for N, K in ((300, 600), (600, 300), (119, 300), (123, 300), (1, 4), (2048, 2048)):
            p = _plan(M, N, K)
            assert p["bn"] in (64, 128)
            assert p["tiles"] == -(-N // 128) * -(-K // p["bn"])
            assert p["per"] % 32 == 0 and p["per"] <= 1024, (M, N, K, p)
            assert (p["splits"] - 1) * p["per"] < M <= p["splits"] * p["per"], (M, N, K, p)


def test_debug_entry_argument_checks():
    L = cabi.lib
    fake = 1 << 20  # 16-byte aligned, never dereferenced: every call below returns before any launch
    args = lambda **kw: [kw.get(k, v) for k, v in (
        ("a_kc", 1), ("b_kc", 1), ("bn", 128), ("A", fake), ("lda", 8), ("B", fake), ("ldb", 8), ("C", fake), ("ldc", 8), ("M", 8),
        ("N", 8), ("K", 8), ("bias", None), ("relu", 0), ("mask", None), ("ldm", 0), ("colsum", None), ("stats", None),
        ("S", None), ("Q", 0), ("gT", None), ("gT2", None), ("q_split", 0), ("ldt", 0), ("stream", None))]
    g = lambda **kw: L.pgnn_debug_tc_gemm(*args(**kw))
    for bn in (0, 32, 96, 256):
        assert g(bn=bn) == EINVAL
    assert g(M=0) == EINVAL and g(N=0) == EINVAL and g(K=0) == EINVAL and g(A=None) == EINVAL and g(C=None) == EINVAL
    assert g(ldc=7) == EINVAL and g(lda=7) == EINVAL and g(a_kc=0, lda=4, M=8) == EINVAL and g(mask=fake, ldm=4) == EINVAL
    assert g(S=fake, Q=17, gT=fake, q_split=17, ldt=8) == EINVAL, "Q > 16 must be refused"
    assert g(S=fake, Q=0, ldt=8) == EINVAL and g(S=fake, Q=9, q_split=10, gT=fake, ldt=8) == EINVAL
    assert g(S=fake, Q=9, q_split=6, gT=fake, ldt=8) == EINVAL, "gT2 missing"
    assert g(S=fake, Q=9, q_split=6, gT2=fake, ldt=8) == EINVAL, "gT missing"
    assert g(lda=10) == EUNSUPPORTED and g(A=fake + 4) == EUNSUPPORTED
    assert g(B=fake + 8) == EUNSUPPORTED and g(b_kc=0, ldb=10) == EUNSUPPORTED
    w = lambda M=8, N=8, K=8, gy=fake, x=fake, gw=fake, ldgy=8, ldx=8, pf=0: L.pgnn_debug_tc_wgrad(
        gy, ldgy, x, ldx, M, N, K, gw, None, None, pf, None)
    assert w(M=0) == EINVAL and w(N=0) == EINVAL and w(gy=None) == EINVAL and w(gw=None) == EINVAL and w(ldx=4) == EINVAL
    assert w(pf=-1) == EINVAL and w(K=6, ldx=8) == EUNSUPPORTED
    out = (ctypes.c_int64 * 4)()
    assert L.pgnn_debug_tc_wgrad_plan(0, 8, 8, out) == EINVAL and L.pgnn_debug_tc_wgrad_plan(8, 8, 8, None) == EINVAL
    ptrs = (ctypes.c_void_p * 33)(*([fake] * 33))
    dims = (ctypes.c_int32 * 33)(*([4] * 33))
    assert L.pgnn_debug_transpose_batch(33, ptrs, ptrs, dims, dims, None) == EUNSUPPORTED
    assert L.pgnn_debug_transpose_batch(-1, ptrs, ptrs, dims, dims, None) == EINVAL
    assert L.pgnn_debug_transpose_batch(0, None, None, None, None, None) == OK
    zero = (ctypes.c_int32 * 1)(0)
    assert L.pgnn_debug_transpose_batch(1, ptrs, ptrs, zero, dims, None) == EINVAL
