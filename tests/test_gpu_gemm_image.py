"""The weight-image path of the 3xTF32 wgmma GEMM (dense_tc.cu, B_IMG): a weight used as a reduction-contiguous B operand is split
into tf32 hi / lo once per pass, into two planes laid out like the GEMM's shared-memory stage, and the mainloop copies B from there
with cp.async.  The values that reach the tensor cores are the same bits in the same order as on the raw path, so:
  * CPU: a numpy restatement of the image format; its planes sum back to the input bit for bit wherever the input is finite;
    every GEMM instantiation (raw and image) compiles for sm_90a without spills, the BN = 64 ones within 128 registers;
  * GPU: the pack kernel's image equals the restatement and stays inside its padded size; pgnn_debug_tc_gemm_img is bit for bit
    pgnn_debug_tc_gemm with a_kc = b_kc = 1 over every epilogue, row and reduction tails, N past the tile and NaN / +-Inf in
    either operand (the operand / output regions of test_gpu_gemm.py: NaN-poisoned inputs, sentinel-guarded outputs);
  * GPU: a chem GIN forward + backward (D = 300, L = 5, B = 256) on the image path and with PGNN_WEIGHT_IMAGES=0 (raw weights):
    node_rep, the running statistics and the weight / embedding gradients identical, the atomically reduced bias, BatchNorm and
    bond-table gradients within the run-to-run bound (3e-4 of scale, test_gpu_parity_full.py)."""
import ctypes
import importlib
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from device_buffers import DEV, NAN, SENT, Region, ceil4 as _ceil4, operand, zeroed
from test_gpu_gemm import OK, tc_gemm

cabi = importlib.import_module("pretrain-gnns_b200._cabi")
gpu = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
CANON_NAN = np.uint32(0x7FFFFFFF)  # the GPU's NaN result of an fp32 add


# ---------------------------------------------------------------------------------------------------------------------------
# numpy restatement of the image format
# ---------------------------------------------------------------------------------------------------------------------------
def kperm(k):
    return (k & 16) | ((k & 3) << 2) | ((k >> 2) & 3)


SLOT_TO_K = np.array([kperm(s) for s in range(32)])


def split_tf32(x):
    """hi = trunc_tf32(x + 0), lo = x - hi, NaN results as the GPU gives them (canonical)."""
    x = np.asarray(x, np.float32)
    with np.errstate(invalid="ignore"):
        y = (x + np.float32(0)).view(np.uint32).copy()
        y[np.isnan(x)] = CANON_NAN
        hi = (y & np.uint32(0xFFFFE000)).view(np.float32)
        lo = (x - hi).view(np.uint32).copy()
    lo[np.isnan(lo.view(np.float32))] = CANON_NAN
    return hi, lo.view(np.float32)


def pad_dims(rows, k):
    return -(-rows // 128) * 128, -(-k // 32) * 32


def image_np(b):
    """b [rows, K] (the K-major B operand) -> (hi, lo) planes [rows_pad, K_pad], slot s of each 32-block holding k = kperm(s)."""
    rows, K = b.shape
    R, Kp = pad_dims(rows, K)
    full = np.zeros((R, Kp), np.float32)
    full[:rows, :K] = b
    perm = (np.arange(Kp) // 32) * 32 + SLOT_TO_K[np.arange(Kp) % 32]
    return split_tf32(full[:, perm])


def unpack_np(hi, lo, rows, K):
    Kp = hi.shape[1]
    inv = np.empty(Kp, np.int64)
    inv[(np.arange(Kp) // 32) * 32 + SLOT_TO_K[np.arange(Kp) % 32]] = np.arange(Kp)  # kperm is an involution; written out anyway
    return hi[:rows, inv][:, :K], lo[:rows, inv][:, :K]


def weight(rows, cols, seed, specials=True):
    rng = np.random.default_rng(seed)
    w = rng.standard_normal((rows, cols)).astype(np.float32)
    w[rng.random((rows, cols)) < 0.1] = 0.0
    w[rng.random((rows, cols)) < 0.05] = -0.0
    if specials:
        for v in (np.nan, np.inf, -np.inf):
            w[rng.integers(0, rows, 3), rng.integers(0, cols, 3)] = v
    return w


@pytest.mark.parametrize("rows,K", [(1, 1), (7, 31), (64, 32), (130, 33), (300, 600), (600, 300), (129, 95)])
def test_image_restatement_sums_back(rows, K):
    w = weight(rows, K, seed=rows * 1000 + K)
    hi, lo = image_np(w)
    R, Kp = pad_dims(rows, K)
    assert hi.shape == lo.shape == (R, Kp)
    h, l = unpack_np(hi, lo, rows, K)
    fin = np.isfinite(w)
    assert np.array_equal((h + l)[fin].view(np.uint32), (w + np.float32(0))[fin].view(np.uint32))
    assert np.array_equal(h.view(np.uint32) & np.uint32(0x1FFF), np.zeros_like(h.view(np.uint32)))  # hi is a tf32 number
    assert np.isnan(h[np.isnan(w)]).all() and np.array_equal(h[np.isinf(w)], w[np.isinf(w)])
    # padding: zero in both planes
    pad = np.ones((R, Kp), bool)
    pad[:rows, :] = False
    for b0 in range(0, Kp, 32):
        for s in range(32):
            if b0 + SLOT_TO_K[s] >= K:
                pad[:, b0 + s] = True
    assert not hi[pad].any() and not lo[pad].any()


@pytest.mark.skipif(not (os.path.exists(NVCC) or shutil.which("nvcc")), reason="nvcc not available")
def test_all_gemm_instantiations_compile_without_spills(tmp_path):
    """8 raw instantiations (A_KC, B_KC, BN) and the 2 image ones (K-major A and B, BN 64 / 128): 0 spills, no serialized wgmma,
    and the BN = 64 tiles within the 128 registers that keep two CTAs per SM."""
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
            k = re.search(r"k_gemm_3xtf32ILb(\d)ELb(\d)ELi(\d+)ELb(\d)E", m.group(1))
            cur = k.groups() if k else None
            if cur:
                kernels[cur] = {}
            continue
        if cur is None:
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m:
            kernels[cur]["spills"] = (int(m.group(1)), int(m.group(2)))
        m = re.search(r"Used (\d+) registers", line)
        if m:
            kernels[cur]["regs"] = int(m.group(1))
    raw = {k for k in kernels if k[3] == "0"}
    img = {k for k in kernels if k[3] == "1"}
    assert len(raw) == 8 and img == {("1", "1", "64", "1"), ("1", "1", "128", "1")}, sorted(kernels)
    assert all(v["spills"] == (0, 0) for v in kernels.values()), kernels
    assert all(v["regs"] <= 128 for k, v in kernels.items() if k[2] == "64"), kernels


# ---------------------------------------------------------------------------------------------------------------------------
# GPU: the pack kernel and the image GEMM
# ---------------------------------------------------------------------------------------------------------------------------
def _image_floats(rows, K):
    R, Kp = pad_dims(rows, K)
    return 2 * R * Kp


def _bits_equal_nan_aware(got, want):
    g, w = got.view(np.uint32), want.view(np.uint32)
    both_nan = np.isnan(got) & np.isnan(want)
    return bool(((g == w) | both_nan).all())


@gpu
def test_pack_matches_restatement_and_stays_inside():
    """One launch, jobs of both orientations with row / reduction tails of 1-31 and a row stride past the extent; every image in a
    sentinel-filled allocation with slack behind it."""
    shapes = [(1, 1, 0), (7, 31, 1), (33, 64, 0), (130, 33, 1), (300, 600, 0), (600, 300, 1), (129, 95, 0), (96, 129, 1)]
    ws, lds, srcs, imgs, wants = [], [], [], [], []
    for i, (r, c, tr) in enumerate(shapes):
        w = weight(r, c, seed=i)
        reg = Region(r, c, _ceil4(c) + 4 * (i % 3), NAN)
        reg.view.copy_(torch.from_numpy(w))
        b = w.T if tr else w
        n = _image_floats(*b.shape)
        buf = torch.full((n + 257,), SENT, device=DEV)
        ws.append(w)
        lds.append(reg.ld)
        srcs.append(reg)
        imgs.append(buf)
        wants.append(image_np(np.ascontiguousarray(b)))
    k = len(shapes)
    rc = cabi.lib.pgnn_debug_pack_weight_images(k, (ctypes.c_void_p * k)(*[s.ptr() for s in srcs]), (ctypes.c_int64 * k)(*lds),
                                                (ctypes.c_int32 * k)(*[s[0] for s in shapes]), (ctypes.c_int32 * k)(*[s[1] for s in shapes]),
                                                (ctypes.c_int32 * k)(*[s[2] for s in shapes]),
                                                (ctypes.c_void_p * k)(*[b.data_ptr() for b in imgs]), torch.cuda.current_stream().cuda_stream)
    assert rc == OK, rc
    torch.cuda.synchronize()
    for (r, c, tr), buf, (hi, lo) in zip(shapes, imgs, wants):
        got = buf.cpu().numpy()
        n = hi.size
        assert _bits_equal_nan_aware(got[:n].reshape(hi.shape), hi), (r, c, tr, "hi")
        assert _bits_equal_nan_aware(got[n:2 * n].reshape(lo.shape), lo), (r, c, tr, "lo")
        assert bool((got[2 * n:] == SENT).all()), (r, c, tr, "write past the image")


def img_gemm(a, b, bn, bias=None, relu=False, mask=None, colsum=False, stats=False, S=None, q_split=0):
    """pgnn_debug_tc_gemm_img on the same regions as test_gpu_gemm.tc_gemm with a_kc = b_kc = 1; the image in a sentinel-guarded
    allocation."""
    M, K = a.shape
    N = b.shape[0]
    A, B = operand(a, 1, 4), operand(b, 1, 8)
    C = Region(M, N, _ceil4(N) + 4, SENT)
    n_img = _image_floats(N, K)
    img = torch.full((n_img + 64,), SENT, device=DEV)
    outs = {"C": C}
    bias_d = None if bias is None else bias.to(DEV)
    mk = None
    if mask is not None:
        mk = Region(M, N, _ceil4(N) + 4, NAN)
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
    rc = cabi.lib.pgnn_debug_tc_gemm_img(bn, A.ptr(), A.ld, B.ptr(), B.ld, img.data_ptr(), C.ptr(), C.ld, M, N, K,
                                         None if bias_d is None else bias_d.data_ptr(), int(relu), None if mk is None else mk.ptr(),
                                         0 if mk is None else mk.ld, p("colsum"), p("stats"), None if S_d is None else S_d.data_ptr(),
                                         Q, p("gT"), p("gT2"), q_split, ldt, torch.cuda.current_stream().cuda_stream)
    assert rc == OK, rc
    torch.cuda.synchronize()
    res = {k: r.view.cpu() for k, r in outs.items()}
    res["intact"] = all(r.outside_intact() for r in outs.values()) and bool((img[n_img:] == SENT).all())
    return res


def _same(x, y):
    """bit for bit, NaN payloads included"""
    if x.dtype == torch.float64:
        return torch.equal(x.view(torch.int64), y.view(torch.int64))
    return torch.equal(x.contiguous().view(torch.int32), y.contiguous().view(torch.int32))


def _check(a, b, bn, **ep):
    raw = tc_gemm(a, b, 1, 1, bn, **ep)
    img = img_gemm(a, b, bn, **ep)
    assert raw["intact"] and img["intact"], (bn, ep.keys())
    for k in img:
        if k != "intact":
            assert _same(img[k], raw[k]), (k, bn, a.shape, b.shape, int((img[k] != raw[k]).sum()))


def _rnd(*shape, seed):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed))


BNS = (64, 128)


@gpu
@pytest.mark.parametrize("bn", BNS)
@pytest.mark.parametrize("blocks", [1, 2, 3, 4, 5])
@pytest.mark.parametrize("tail", [1, 5, 16, 31, 32])
def test_reduction_blocks_and_tails(bn, blocks, tail):
    K = 32 * (blocks - 1) + tail
    _check(_rnd(200, K, seed=blocks), _rnd(136, K, seed=tail), bn)


@gpu
@pytest.mark.parametrize("bn", BNS)
@pytest.mark.parametrize("r", [1, 8, 9, 63, 64, 65, 127])
def test_row_tails(bn, r):
    _check(_rnd(128 + r, 100, seed=r), _rnd(72, 100, seed=r + 1), bn)


@gpu
@pytest.mark.parametrize("bn", BNS)
@pytest.mark.parametrize("N", [1, 63, 65, 129, 300, 600])
def test_output_columns_past_the_tile(bn, N):
    _check(_rnd(257, 300, seed=N), _rnd(N, 300, seed=N + 7), bn)


@gpu
@pytest.mark.parametrize("bn", BNS)
def test_every_epilogue(bn):
    # one row tile (M <= 128) for the fused column reductions: one atomic per column onto zero, so those are bit-exact too
    M, N, K = 117, 150, 77
    a, b = _rnd(M, K, seed=1), _rnd(N, K, seed=2)
    g = torch.Generator().manual_seed(3)
    bias = torch.randn(N, generator=g)
    mask = torch.where(torch.rand(M, N, generator=g) < 0.3, torch.tensor(float("nan")), torch.randn(M, N, generator=g))
    _check(a, b, bn, bias=bias)
    _check(a, b, bn, bias=bias, relu=True)
    _check(a, b, bn, mask=mask)
    _check(a, b, bn, colsum=True)
    _check(a, b, bn, bias=bias, stats=True)
    for Q, q_split in ((1, 0), (1, 1), (9, 6), (16, 10)):
        _check(a, b, bn, S=torch.randn(M, Q, generator=g), q_split=q_split)
    _check(a, b, bn, bias=bias, relu=True, mask=mask, colsum=True, stats=True, S=torch.randn(M, 9, generator=g), q_split=6)


@gpu
@pytest.mark.parametrize("bn", BNS)
def test_non_finite_in_either_operand(bn):
    M, N, K = 150, 130, 72
    a, b = _rnd(M, K, seed=5), _rnd(N, K, seed=6)
    for i, v in enumerate((float("inf"), float("-inf"), float("nan"))):
        a[17 * i + 3, 11 * i + 1] = v
        b[23 * i + 5, 13 * i + 2] = v
    b[40, :] = 0.0
    _check(a, b, bn)
    _check(a, b, bn, relu=True)


# ---------------------------------------------------------------------------------------------------------------------------
# GPU: the chem GIN encoder on both paths
# ---------------------------------------------------------------------------------------------------------------------------
@gpu
def test_gin_encoder_image_path_matches_raw_weights():
    import test_gpu_encoder as TE
    from golden_util import probe
    from oracle import gnn_oracle as O
    syn = importlib.import_module("pretrain-gnns_b200.synthetic")
    L, D = 5, 300
    b = syn.zinc_batch(256, 4)
    P = O.make_params("chem", "gin", L, D, seed=3, randomize_bn=True)
    g = probe((b["x"].shape[0], D), 11)
    runs = []
    old = os.environ.get("PGNN_WEIGHT_IMAGES")
    try:
        for flag in ("1", "0"):
            os.environ["PGNN_WEIGHT_IMAGES"] = flag
            enc = TE.Encoder("gin", L, D, b, P)
            assert enc.forward(True, 0.0, 0, TE.TF32X3) == OK
            rc, flat = enc.backward(g, 0.0, 0, TE.TF32X3)
            assert rc == OK
            torch.cuda.synchronize()
            assert enc.guards_intact()
            runs.append((enc.out.view.cpu(), enc.stats(), dict(enc.grads(flat))))
    finally:
        if old is None:
            os.environ.pop("PGNN_WEIGHT_IMAGES", None)
        else:
            os.environ["PGNN_WEIGHT_IMAGES"] = old
    (rep0, st0, g0), (rep1, st1, g1) = runs
    assert torch.equal(rep0, rep1), float((rep0 - rep1).abs().max())
    for k in st0:
        assert torch.equal(st0[k], st1[k]), k
    gmax = max(float(v.abs().max()) for v in g0.values())
    for k in g0:
        if k.endswith(("mlp.0.weight", "mlp.2.weight")) or k.startswith("x_embedding"):
            assert torch.equal(g0[k], g1[k]), (k, float((g0[k] - g1[k]).abs().max()))
        else:  # biases, BatchNorm affine, bond tables: fp32 / fp64 atomics whose order varies from run to run
            tmax = float(g0[k].abs().max())
            scale = max(gmax if tmax < 1e-3 * gmax else tmax, 1e-30)
            assert float((g0[k] - g1[k]).abs().max()) / scale <= 3e-4, k
