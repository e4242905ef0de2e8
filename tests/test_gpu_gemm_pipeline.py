"""The mainloop of the 3xTF32 wgmma GEMM (dense_tc.cu): A fragments in registers with the reduction index permuted inside each
32-wide block (kperm), B in three shared-memory stages, commit groups kept in flight across k-steps and blocks.

Through pgnn_debug_tc_gemm, every layout x tile width, with the NaN-filled operand / sentinel-filled output regions of
test_gpu_gemm.py:
  * pipeline fill and drain: 1-5 k-blocks, and reduction tails of 1-31 past a block boundary;
  * row tails that end inside a warp's 16-row fragment slice;
  * the permutation: a one-hot A picks exactly one reduction index of B, so an A / B permutation mismatch reads the wrong one;
  * NaN / +-Inf in A at positions held by each of the four fragment registers;
  * a bit-for-bit repeat;
and through pgnn_debug_tc_wgrad the split-K weight gradient (MN-major A and B), whose splits start at k != 0 and hold 1-4
blocks each.
The CPU test compiles dense_tc.cu for sm_90a and checks every instantiation for spills and serialized wgmma."""
import os
import re
import shutil
import subprocess

import pytest
import torch

from device_buffers import DEV, NAN, SENT, Region
from test_gpu_gemm import (COMBOS, TAU, _classes, _fp32_semantics, _plan, _tc_wgrad, exact_pair, exact_ref, norm_err, rnd, scale_of,
                           tc_gemm)

gpu = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")


def _all_combos_bit_exact(M, N, K, seed):
    for i, (ak, bk, bn) in enumerate(COMBOS):
        a, b = exact_pair(M, N, K, seed=seed + i, lo_in="ab"[i % 2])
        ref = exact_ref(a, b)
        r = tc_gemm(a, b, ak, bk, bn)
        assert r["intact"], (M, N, K, ak, bk, bn)
        assert torch.equal(r["C"], ref), (M, N, K, ak, bk, bn, int((r["C"] != ref).sum()))


@gpu
@pytest.mark.parametrize("blocks", [1, 2, 3, 4, 5])
@pytest.mark.parametrize("tail", [1, 5, 16, 31, 32])
def test_pipeline_fill_and_drain(blocks, tail):
    # blocks k-blocks, the last one holding `tail` of its 32 reduction elements
    _all_combos_bit_exact(129, 72, 32 * (blocks - 1) + tail, seed=31 * blocks + tail)


@gpu
@pytest.mark.parametrize("r", [1, 8, 9, 63, 64, 65, 127])
def test_row_tails_inside_a_fragment(r):
    _all_combos_bit_exact(128 + r, 136, 100, seed=r)


@gpu
@pytest.mark.parametrize("K", [32, 77, 300])
def test_permutation_pairs_each_k_with_itself(K):
    # C[m, n] = b[n, m mod K]: any A slot paired with a B slot of another reduction index changes that output
    M, N = 2 * K + 3, 136
    a = torch.zeros(M, K)
    a[torch.arange(M), torch.arange(M) % K] = 1.0
    b = ((torch.arange(N)[:, None] * 7 + torch.arange(K)[None, :] * 3) % 2001 - 1000).float()
    for lo_a in (False, True):  # the lo part (n 2^-12) in one operand
        aa, bb = (a * (1 + 2 ** -12), b) if lo_a else (a, b * (1 + 2 ** -12))
        want = exact_ref(aa, bb)
        assert torch.equal(want, (b * (1 + 2 ** -12)).t()[torch.arange(M) % K])
        for ak, bk, bn in COMBOS:
            r = tc_gemm(aa, bb, ak, bk, bn)
            assert r["intact"], (ak, bk, bn)
            assert torch.equal(r["C"], want), (lo_a, ak, bk, bn, int((r["C"] != want).sum()))


@gpu
@pytest.mark.parametrize("relu", [False, True])
def test_non_finite_in_every_fragment_register(relu):
    # fragment register q of a k-step holds row 16w + l/4 + 8 (q % 2) and the reduction index with k % 2 == q // 2 (kperm)
    M, N, K = 80, 70, 72
    g = torch.Generator().manual_seed(5)
    a = torch.randn(M, K, generator=g)
    choices = torch.tensor([0.0, 0.5, -0.5, 1.5, -0.0])
    b = torch.where(torch.rand(N, K, generator=g) < 0.6, choices[torch.randint(0, 5, (N, K), generator=g)],
                    torch.randn(N, K, generator=g))
    planted = {}
    for q in range(4):
        for i, v in enumerate((float("inf"), float("-inf"), float("nan"))):
            m = 16 * (q + i) + 8 * (q % 2) + (3 * q + i) % 8
            k = 32 * (i % 2) + 2 * (5 * q + 3 * i) % 32 + q // 2
            planted[(m % M, k)] = v
    for (m, k), v in planted.items():
        a[m, k] = v
    ref = _fp32_semantics(a, b, relu)
    want = _classes(ref)
    assert want[0].any() and want[1].any() and (relu or want[2].any())
    fin = torch.isfinite(ref)
    den = scale_of(torch.nan_to_num(a, 0.0, 0.0, 0.0), torch.nan_to_num(b, 0.0, 0.0, 0.0))
    for ak, bk, bn in COMBOS:
        r = tc_gemm(a, b, ak, bk, bn, relu=relu)
        assert r["intact"], (ak, bk, bn)
        for got, w, what in zip(_classes(r["C"]), want, ("NaN", "+Inf", "-Inf")):
            assert torch.equal(got, w), (ak, bk, bn, what, int((got != w).sum()))
        assert norm_err(r["C"][fin], ref[fin], den[fin]) <= TAU, (ak, bk, bn)


@gpu
def test_bit_for_bit_repeat():
    a, b = rnd(777, 600, seed=3), rnd(300, 600, seed=4)
    for ak, bk, bn in COMBOS:
        r1, r2 = tc_gemm(a, b, ak, bk, bn), tc_gemm(a, b, ak, bk, bn)
        assert r1["intact"] and r2["intact"]
        assert torch.equal(r1["C"].view(torch.int32), r2["C"].view(torch.int32)), (ak, bk, bn)


@gpu
@pytest.mark.parametrize("N,K", [(600, 300), (300, 600)])
@pytest.mark.parametrize("M", [200, 640, 650, 960, 999])
def test_wgrad_splits_bit_exact(M, N, K):
    # gw = gy^T x over M node rows, split-K with the partial tiles folded in split order; integer family, |S| < 4096: exact
    g = torch.Generator().manual_seed(M + N)
    gy = torch.randint(-2, 3, (M, N), generator=g).float()
    x = torch.randint(-2, 3, (M, K), generator=g).float() * (1 + 2 ** -12)
    ref = exact_ref(gy.t(), x.t())
    plan = _plan(M, N, K)
    assert plan["splits"] > 1 and plan["per"] <= 4 * 32, plan
    G, X = Region(M, N, N + 4, NAN), Region(M, K, K + 8, NAN)
    G.view.copy_(gy)
    X.view.copy_(x)
    need = plan["splits"] * N * K
    part = torch.full((need + 64,), SENT, device=DEV)
    gw, _ = _tc_wgrad(G, X, M, N, K, part.data_ptr(), need)
    assert bool((part[need:] == SENT).all())
    assert torch.equal(gw, ref), (plan, int((gw != ref).sum()))


@pytest.mark.skipif(not (os.path.exists(NVCC) or shutil.which("nvcc")), reason="nvcc not available")
def test_ptxas_no_spills_and_no_serialized_wgmma(tmp_path):
    nvcc = NVCC if os.path.exists(NVCC) else shutil.which("nvcc")
    src = os.path.join(ROOT, "pretrain-gnns_b200", "csrc", "dense_tc.cu")
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--expt-relaxed-constexpr",
           "-I" + os.path.join(ROOT, "include"), "-Xptxas", "-v", "-c", src, "-o", str(tmp_path / "dense_tc.o")]
    out = subprocess.run(cmd, capture_output=True, text=True)
    assert out.returncode == 0, out.stderr[-4000:]
    log = out.stdout + out.stderr
    assert not re.search(r"wgmma.*serializ", log, re.I), log
    kernels, cur = {}, None
    for line in log.splitlines():
        m = re.search(r"Compiling entry function '(\w+)'", line)
        if m:
            k = re.search(r"k_gemm_3xtf32ILb(\d)ELb(\d)ELi(\d+)E", m.group(1))
            cur = k.groups() if k else None
            continue
        if cur is None:
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m:
            kernels[cur] = (int(m.group(1)), int(m.group(2)))
    assert len(kernels) == 8, kernels
    assert all(v == (0, 0) for v in kernels.values()), kernels
