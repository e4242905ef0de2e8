"""Per-shape timing of the 3xTF32 wgmma GEMM (k_gemm_3xtf32): the six GEMMs of one GIN-300 layer as csrc/encoder.cu issues them
on the masking step, at that batch's node count N, each through the library's test entry points with the same tile width,
epilogue hooks and split-K workspace the encoder gets.  The four with a weight as B (fwd1, fwd2, dgrad2, dgrad1) run twice: from
the raw weight, and from the weight image the encoder packs once per pass ("img" lines: GEMM only, the pack is not timed).  Prints one JSON line per (library, GEMM): us per call, TFLOP/s
(2 N K_in K_out over the time) and the fraction of 165 TFLOP/s, the 3xTF32 ceiling of a 495 TFLOP/s dense-TF32 H100 SXM.

    python tools/bench_gemm.py [--rows 5930] [--reps 200] [--rounds 1] [--lib PATH ...]

Each --lib (default: this tree's libpgnn_b200.so) is timed in a process of its own; with several, the rounds alternate
between them (e.g. --lib pretrain-gnns_b200/libpgnn_b200.so --lib /tmp/parent/libpgnn_b200.so).  The forward and dgrad GEMMs run
at the tile width pick_bn below restates (it must follow dense_tc.cu's pick_bn, TileCfg::MIN_BLOCKS and kNumSMs); each line
reports the width it used, the wgrad lines the library's own plan.  Needs a GPU."""
import argparse
import ctypes
import json
import os
import subprocess
import sys

ROOT = os.path.abspath(os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
D = 300
NUM_SMS = 132


def pick_bn(M, N):
    """dense_tc.cu's pick_bn for one split: the tile width with the least per-SM work over the grid."""
    cdiv = lambda a, b: -(-a // b)
    mt = cdiv(M, 128)
    cost = lambda bn, per_sm: cdiv(mt * cdiv(N, bn), NUM_SMS * per_sm) * bn * per_sm
    return 64 if cost(64, 2) < cost(128, 1) else 128


def child(rows, reps, label):
    import torch
    sys.path.insert(0, ROOT)
    import importlib
    lib = importlib.import_module("pretrain-gnns_b200._cabi").lib
    dev = torch.device("cuda:0")
    g = torch.Generator(device="cpu").manual_seed(0)
    r = lambda *s: torch.randn(*s, generator=g).to(dev)
    N = rows
    aggr, z1, gz2 = r(N, D), r(N, 2 * D), r(N, D)
    gz1 = r(N, 2 * D)
    w1, w2 = r(2 * D, D) * 0.05, r(D, 2 * D) * 0.05
    w1T, w2T = w1.t().contiguous(), w2.t().contiguous()
    b1, b2 = r(2 * D), r(D)
    S = r(N, 9)
    y1, y2, gx1, gx0 = (torch.empty(N, 2 * D, device=dev), torch.empty(N, D, device=dev), torch.empty(N, 2 * D, device=dev),
                        torch.empty(N, D, device=dev))
    stats = torch.zeros(2, D, dtype=torch.float64, device=dev)
    colsum = torch.zeros(2 * D, device=dev)
    gT, gT2 = torch.zeros(6, D, device=dev), torch.zeros(3, D, device=dev)
    gw2, gw1 = torch.empty(D, 2 * D, device=dev), torch.empty(2 * D, D, device=dev)
    st = torch.cuda.current_stream().cuda_stream

    def plan(M, Nn, K):
        out = (ctypes.c_int64 * 4)()
        assert lib.pgnn_debug_tc_wgrad_plan(M, Nn, K, out) == 0
        return list(out)

    img = torch.empty(2 * 640 * 320 + 2 * 384 * 608, device=dev)  # room for either image shape of the layer

    part2, part1 = (torch.empty(plan(N, n, k)[2] * n * k, device=dev) for n, k in ((D, 2 * D), (2 * D, D)))
    p = lambda t: t.data_ptr()

    def gemm(A, B, C, K, Nout, bias=None, relu=0, mask=None, colsum=None, stats=None, S=None, image=False):
        # image: pgnn_debug_tc_gemm_img, which packs B into the image and runs the GEMM from it (the "pack" lines time the pack alone)
        head = (pick_bn(N, Nout), p(A), A.shape[1], p(B), B.shape[1], p(img)) if image else (1, 1, pick_bn(N, Nout), p(A), A.shape[1],
                                                                                          p(B), B.shape[1])
        rc = (lib.pgnn_debug_tc_gemm_img if image else lib.pgnn_debug_tc_gemm)(*head, p(C), C.shape[1], N, Nout, K,
                                    p(bias) if bias is not None else None, relu, p(mask) if mask is not None else None,
                                    mask.shape[1] if mask is not None else 0, p(colsum) if colsum is not None else None,
                                    p(stats) if stats is not None else None, p(S) if S is not None else None, 9 if S is not None else 0,
                                    p(gT) if S is not None else None, p(gT2) if S is not None else None, 6 if S is not None else 0,
                                    D, st)
        assert rc == 0, rc

    def wgrad(G, X, GW, part):
        rc = lib.pgnn_debug_tc_wgrad(p(G), G.shape[1], p(X), X.shape[1], N, G.shape[1], X.shape[1], p(GW), None, p(part),
                                     part.numel(), st)
        assert rc == 0, rc

    def pack(B):
        one = lambda t, c: (c * 1)(t)
        rc = lib.pgnn_debug_pack_weight_images(1, one(p(B), ctypes.c_void_p), one(B.shape[1], ctypes.c_int64),
                                               one(B.shape[0], ctypes.c_int32), one(B.shape[1], ctypes.c_int32), one(0, ctypes.c_int32),
                                               one(p(img), ctypes.c_void_p), st)
        assert rc == 0, rc

    cases = [  # (name, output columns, reduction, tile width, splits, call)
        ("fwd1 300->600 +bias ReLU", 2 * D, D, pick_bn(N, 2 * D), 1, lambda: gemm(aggr, w1, y1, D, 2 * D, bias=b1, relu=1)),
        ("fwd2 600->300 +bias stats", D, 2 * D, pick_bn(N, D), 1, lambda: gemm(z1, w2, y2, 2 * D, D, bias=b2, stats=stats)),
        ("dgrad2 300->600 mask colsum", 2 * D, D, pick_bn(N, 2 * D), 1,
         lambda: gemm(gz2, w2T, gx1, D, 2 * D, mask=z1, colsum=colsum)),
        ("dgrad1 600->300 S-hook", D, 2 * D, pick_bn(N, D), 1, lambda: gemm(gz1, w1T, gx0, 2 * D, D, S=S)),
        ("wgrad2 [300,600] split-K", D, 2 * D, *plan(N, D, 2 * D)[0:3:2], lambda: wgrad(gz2, z1, gw2, part2)),
        ("wgrad1 [600,300] split-K", 2 * D, D, *plan(N, 2 * D, D)[0:3:2], lambda: wgrad(gz1, aggr, gw1, part1)),
    ]
    cases += [
        ("fwd1 img (+pack)", 2 * D, D, pick_bn(N, 2 * D), 1, lambda: gemm(aggr, w1, y1, D, 2 * D, bias=b1, relu=1, image=True)),
        ("fwd2 img (+pack)", D, 2 * D, pick_bn(N, D), 1, lambda: gemm(z1, w2, y2, 2 * D, D, bias=b2, stats=stats, image=True)),
        ("dgrad2 img (+pack)", 2 * D, D, pick_bn(N, 2 * D), 1, lambda: gemm(gz2, w2T, gx1, D, 2 * D, mask=z1, colsum=colsum, image=True)),
        ("dgrad1 img (+pack)", D, 2 * D, pick_bn(N, D), 1, lambda: gemm(gz1, w1T, gx0, 2 * D, D, S=S, image=True)),
        ("pack [600,300]", 0, 0, 0, 1, lambda: pack(w1)),
        ("pack [300,600]", 0, 0, 0, 1, lambda: pack(w2)),
    ]
    name = torch.cuda.get_device_name(0)
    for title, n_out, k, bn, splits, fn in cases:
        for _ in range(10):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        us = e0.elapsed_time(e1) / reps * 1e3
        tf = 2.0 * N * n_out * k / us / 1e6
        print(json.dumps(dict(label=label, gemm=title, rows=N, bn=bn, splits=splits, us=round(us, 2), tflops=round(tf, 1),
                              of_165=round(tf / 165, 3), card=name)), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=5930, help="node rows N (a B = 256 masking batch has about 5930)")
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=1)
    ap.add_argument("--lib", action="append", default=[])
    ap.add_argument("--child", default=None)
    a = ap.parse_args()
    if a.child is not None:
        child(a.rows, a.reps, a.child)
        return
    libs = a.lib or [os.path.join(ROOT, "pretrain-gnns_b200", "libpgnn_b200.so")]
    for rnd in range(a.rounds):
        for lib in libs:
            env = dict(os.environ, PGNN_LIB=os.path.abspath(lib))
            subprocess.run([sys.executable, os.path.abspath(__file__), "--rows", str(a.rows), "--reps", str(a.reps),
                            "--child", "%s#%d" % (lib, rnd)], env=env, check=True)


if __name__ == "__main__":
    main()
