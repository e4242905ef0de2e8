"""Oracle runs and bounds of the chem whole encoder (tests/test_gpu_encoder.py, tests/test_encoder_host.py).

One case runs tests/dropout_oracle.chem_gnn (oracle.gnn_oracle.chem_gnn when there are no masks) on the CPU twice, in fp64 and
in fp32, from the same fp32 parameters, with gradients by autograd against one upstream g.  The fp32 run measures how far an
honest fp32 computation of the same thing lands from fp64, and every bound is stated against that:
  node_rep             golden_util.output_check: 1e-4 abs + rel against the fp32 run, and max(OUT_REL, SLACK x the fp32 run's
                       error) against fp64, relative to the largest |fp64|;
  gradients            golden_util.gradient_check for every tensor of the flat buffer: max(GRAD_REL, SLACK x the fp32 run's
                       error), relative to the tensor's largest |fp64|; the ReLU-boundary allowance only when the fp64 run has
                       near-zero pre-activations, or a match with the fp64 run in which one of those units' ReLU decision is
                       inverted (check_grads), and every use of either is reported;
  running mean / var   max(STATS_FLOOR, STATS_SLACK x the fp32 run's error) against fp64, relative to the buffer's largest |fp64|;
  num_batches_tracked  exact.
"""
import torch

import dropout_oracle as DO
from golden_util import OUT_REL, SLACK, gradient_check, output_check
from oracle import gnn_oracle as O

STATS_FLOOR, STATS_SLACK = 1e-6, 3.0
NEAR_ZERO = 4e-6  # oracle.gnn_oracle.near_zero_preactivations' rounding distance of the ReLU kink
F32, F64 = torch.float32, torch.float64


def _flipped_relu(unit):
    """O._relu with the decision of one unit (call index, row, column) inverted."""
    calls = [0]

    def relu(x):
        keep = x > 0
        if calls[0] == unit[0]:
            keep = keep.clone()
            keep[unit[1], unit[2]] = ~keep[unit[1], unit[2]]
        calls[0] += 1
        return torch.where(keep, x, torch.zeros_like(x))
    return relu


def run(P, b, t, L, training, dt, g=None, masks=None, p=0.0, steps=1, fn=DO.chem_gnn, flip=None):
    """One oracle run in dtype dt.  `steps` training forwards in a row, each starting from the running statistics the one before
    left; the gradients (against g) are those of the last.  `flip`: invert that ReLU unit's decision.
    -> (out, grads, new running statistics, the ReLU inputs in call order)."""
    lp = O.leaf_params(P, dt)
    trace, relu = [], O._relu
    O.RELU_TRACE = trace
    if flip is not None:
        O._relu = _flipped_relu(flip)
    try:
        for _ in range(steps):
            stats = {}
            out = fn(lp, b["x"], b["edge_index"], b["edge_attr"], L, t, training, stats, masks=masks, p=p)
            lp.update(stats)
    finally:
        O.RELU_TRACE, O._relu = None, relu
    grads = {}
    if training and g is not None:
        (out * g.to(dt)).sum().backward()
        grads = {k: v.grad for k, v in lp.items() if v.requires_grad}
    return out.detach(), grads, stats, trace


class Ref:
    """Both oracle runs of one case: out / grads / stats keyed by dtype; near_zero counts the fp64 run's ReLU inputs within
    rounding distance of the kink, near_units lists them as (ReLU call, row, column)."""

    def __init__(self, P, b, t, L, training, g=None, masks=None, p=0.0, steps=1):
        self.args = (P, b, t, L, training)
        self.kw = dict(g=g, masks=masks, p=p, steps=steps)
        self.out, self.grads, self.stats = {}, {}, {}
        for dt in (F64, F32):
            self.out[dt], self.grads[dt], self.stats[dt], trace = run(P, b, t, L, training, dt, **self.kw)
            if dt == F64:
                self.near_zero = O.near_zero_preactivations(trace)
                self.near_units = [(i, r, c) for i, x in enumerate(trace)
                                   for r, c in (x.abs() <= NEAR_ZERO * x.abs().max()).nonzero().tolist()]


def check_output(name, mine, ref, rows, north_star=True):
    """output_check; north_star=False keeps only its scale-relative half (deep stacks, where the element-wise 1e-4 bound is
    below what the compounded rounding of any fp32 GEMM order can promise)."""
    ok = output_check(name, mine, ref.out[F32], ref.out[F64], rows)
    if not north_star:
        r = rows[-1]
        r["ok"] = ok = r["err"] <= max(OUT_REL, SLACK * r["err_ref32"])
        r["north_star"] = "not applied (%s)" % r["north_star"]
    return ok


def check_grads(named_mine, ref, rows, noise_floor=0.0):
    """gradient_check over the flat buffer's tensors.
    * every fp64 gradient exactly zero (every unit dropped): the kernel's must be exactly zero too;
    * a miss with near-zero ReLU inputs in the fp64 run: accepted when the kernel passes the same bounds against the fp64 oracle
      with one of those units' decisions inverted (the fp32 run shifted by the same amount, so the bounds do not widen);
    * noise_floor: the bound of an ill-conditioned case is at least this (two-row BatchNorm)."""
    named_mine = list(named_mine)
    g32, g64 = ref.grads[F32], ref.grads[F64]
    if max(float(v.abs().max()) for v in g64.values()) == 0:
        ok_all = True
        for k, mine in named_mine:
            e = float(mine.detach().abs().max())
            rows.append(dict(kind="grad", name=k, err=e, err_ref32=0.0, tol=0.0, ok=e == 0, via="exact zero", structurally_zero=True))
            ok_all &= e == 0
        return ok_all
    mine_rows = []
    ok = gradient_check(named_mine, g32, g64, ref.near_zero, mine_rows)
    for unit in ([] if ok else ref.near_units):
        g64f = run(*ref.args, F64, flip=unit, **ref.kw)[1]
        alt = []
        if gradient_check(named_mine, {k: g32[k] + (g64f[k] - g64[k]) for k in g64}, g64f, 0, alt):
            for r in alt:
                r["via"] = "fp64 oracle with the decision of near-zero ReLU unit %s inverted" % (unit,)
            mine_rows, ok = alt, True
            break
    if not ok and noise_floor:
        ok = True
        for r in mine_rows:
            if not r["ok"] and r["err"] <= noise_floor:
                r["ok"], r["via"] = True, "ill-conditioned case: noise floor %g" % noise_floor
            ok &= r["ok"]
    rows += mine_rows
    return ok


def check_stats(name, mine, s32, s64, rows):
    mine, s32, s64 = (torch.as_tensor(t).detach().cpu().double() for t in (mine, s32, s64))
    scale = max(float(s64.abs().max()), 1e-30)
    e = float((mine - s64).abs().max()) / scale
    eref = float((s32 - s64).abs().max()) / scale
    tol = max(STATS_FLOOR, STATS_SLACK * eref)
    rows.append(dict(kind="stats", name=name, err=e, err_ref32=eref, tol=tol, ok=e <= tol))
    return e <= tol


def check_all_stats(mine, ref, L, rows):
    """mine: {'batch_norms.l.running_mean' / '.running_var': tensor} of the L layers."""
    ok = True
    for l in range(L):
        for s in ("running_mean", "running_var"):
            k = f"batch_norms.{l}.{s}"
            ok &= check_stats(k, mine[k], ref.stats[F32][k], ref.stats[F64][k], rows)
    return ok


def margin(rows):
    """The largest error / bound ratio of a set of check rows (> 1: some check failed by that factor)."""
    m = 0.0
    for r in rows:
        tol = r.get("tol")
        if tol is None:  # output rows: output_check's fp64 bound
            tol = max(OUT_REL, SLACK * r["err_ref32"])
        if tol > 0:
            m = max(m, r["err"] / tol)
        elif r["err"] > 0:
            m = float("inf")
    return m
