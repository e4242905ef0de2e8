"""GPU dev check for the 3xTF32 wgmma GEMMs: accuracy against an fp64 reference, and timing of both
precisions (CUDA events, L2 flushed between launches).  Run on an H100:  python tools/check_tc.py"""
import importlib
import os
import sys

import torch

sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), "..")))
ops = importlib.import_module("pretrain-gnns_b200.ops")
dev = "cuda:0"
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)


COLD = True


def timeit(fn, reps=10):
    fn(); torch.cuda.synchronize()
    tot = 0.0
    for _ in range(reps):
        if COLD:
            flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record(); b.synchronize()
        tot += a.elapsed_time(b)
    return tot / reps * 1e3  # us


def relerr(a, ref):
    return ((a.double() - ref).abs().max() / ref.abs().max()).item()


def run(M, N, K, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    x = torch.randn(M, K, generator=g).to(dev)
    w = (torch.randn(N, K, generator=g) * 0.1).to(dev)
    b = torch.randn(N, generator=g).to(dev)
    gy = torch.randn(M, N, generator=g).to(dev)
    mask = torch.randn(M, K, generator=g).to(dev)
    ref_y = torch.relu(x.double() @ w.double().t() + b.double())
    ref_gx = (gy.double() @ w.double()) * (mask > 0)
    ref_gw = gy.double().t() @ x.double()
    ref_gb = gy.double().sum(0)
    out = {}
    for name in ("fp32", "tf32x3"):
        ops.set_precision(name)
        y = ops._linear_fwd(x, w, b, True)
        gx = ops._linear_bwd_x(gy, w, mask)
        gw, gb = ops._linear_bwd_w(gy, x)
        torch.cuda.synchronize()
        e = (relerr(y, ref_y), relerr(gx, ref_gx), relerr(gw, ref_gw), relerr(gb, ref_gb))
        t = (timeit(lambda: ops._linear_fwd(x, w, b, True)), timeit(lambda: ops._linear_bwd_x(gy, w, mask)),
             timeit(lambda: ops._linear_bwd_w(gy, x)))
        out[name] = (e, t)
    gf = 2.0 * M * N * K / 1e6  # MFLOP
    for name, (e, t) in out.items():
        print("M=%5d N=%4d K=%4d %-7s err fwd %.1e dgrad %.1e wgrad %.1e gb %.1e | us fwd %7.1f dgrad %7.1f wgrad %7.1f | TF/s %6.1f %6.1f %6.1f"
              % (M, N, K, name, *e, *t, gf / t[0], gf / t[1], gf / t[2]), flush=True)


if __name__ == "__main__":
    if len(sys.argv) > 1 and sys.argv[1] == "warm":
        COLD = False
        print("warm L2 (no flush between launches)")
    shapes = [(5986, 600, 300), (5986, 300, 600), (130, 600, 300), (1, 8, 4), (1024, 119, 300), (32000, 600, 600), (777, 300, 300)]
    if 'quick' in sys.argv:
        shapes = shapes[:2]
    for shape in shapes:
        M, N, K = shape
        run(*shape)
