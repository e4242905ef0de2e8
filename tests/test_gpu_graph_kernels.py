"""The graph kernels against plain fp64 restatements of the same operations: GAT attention forward and backward (gat.cu), the
neighbour aggregation, its transpose and the edge-table gradients (aggregate.cu), the edge summaries and the GCN normalisation
(graph_prep.cu), and ReLU on non-finite values (aggregate.cu, norm.cu).

The kernels are driven through the C ABI (_cabi.lib), which exposes what ops.* hides: row strides, the head count and the raw
GAT outputs alpha / pq.  Every input is a view inside a NaN-filled allocation and every output one inside a sentinel-filled
allocation (device_buffers), so an over-read shows up as NaN and an over-write as a broken sentinel.  Graphs are bucketed on
the CPU by oracle/graph_prep_oracle.py, and their edge columns are shuffled so that an edge id is not its bucket position.

Bounds:
  * GAT, per output tensor: max |mine - ref64| over the tensor's largest |ref64| <= max(floor, SLACK x the same error of the fp32
    restatement), with golden_util's OUT_REL / GRAD_REL floors and SLACK.  test_gat_bound_rejects_wrong_variants shows on the
    test's own inputs that this rejects six plausible mistakes by 10x or more.
  * aggregation, summaries and edge tables: |mine - ref64| <= TAU x the same sum taken over magnitudes (sum |w| |x|).
  * SUM / MEAN aggregation of plain rows and the SUM transpose gather: bit-exact against a sequential CPU index_add_ in edge
    order, self-loop last (the kernels add in that order by construction).
"""
import importlib
import math
import os
import subprocess
import sys
import textwrap
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from device_buffers import DEV, NAN, SENT, Region, card, ceil4, filled
from golden_util import GRAD_REL, OUT_REL, SLACK, write_report
from oracle import gnn_oracle as O
from oracle import graph_prep_oracle as GP

cabi = importlib.import_module("pretrain-gnns_b200._cabi")
syn = importlib.import_module("pretrain-gnns_b200.synthetic")
gpu = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OK, EINVAL, EWORKSPACE, EUNSUPPORTED = 0, -1, -3, -4
SUM, MEAN, GCN = 0, 1, 2
MODES = {"sum": SUM, "mean": MEAN, "gcn": GCN}
# |mine - ref64| <= TAU x sum of |terms|: fp32 sums of up to ~1000 terms in a fixed order stay near 1e-7 of that; one term
# dropped or doubled in a 1000-term sum moves the result by ~1e-3 of it
TAU = 1e-5
FLOOR = dict(out=OUT_REL, alpha=OUT_REL, pq=OUT_REL, gxl=GRAD_REL, gatt=GRAD_REL, gT=GRAD_REL, gbias=GRAD_REL)


def _stream():
    return torch.cuda.current_stream().cuda_stream


# ---------------------------------------------------------------------------------------------------------------------------
# graphs
# ---------------------------------------------------------------------------------------------------------------------------
class Graph:
    """edge_index [2, E] (row 0 = target) on the CPU and its two bucketings; the device copies are made on first use."""

    def __init__(self, ei, n):
        self.ei, self.n, self.E = ei.to(torch.int64), n, int(ei.shape[1])
        (rt, nt, et), (rs, ns, es) = GP.graph_prep(self.ei.numpy(), n)
        self.host = dict(rowptr_t=rt, nbr_t=nt, eid_t=et, rowptr_s=rs, nbr_s=ns, eid_s=es)
        self.in_deg = torch.from_numpy(np.diff(rt).astype(np.int64))
        self._dev = None

    def ptr(self, key):
        if self._dev is None:
            self._dev = {k: torch.from_numpy(np.ascontiguousarray(v, dtype=np.int32)).to(DEV) for k, v in self.host.items()}
        t = self._dev[key]
        return t.data_ptr() if t.numel() else None

    def looped(self):
        """edge_index with the self-loops appended after the real edges (chem/model.py:39)"""
        return O.with_self_loops(self.ei, self.n)

    def bucket_perm(self):
        """position p of the target-bucket order (self-loop of node i at E + i) -> edge id in edge_index order"""
        return torch.cat([torch.from_numpy(self.host["eid_t"].astype(np.int64)), self.E + torch.arange(self.n)])


def _shuffle(ei, seed):
    return ei[:, torch.from_numpy(np.random.default_rng(seed).permutation(ei.shape[1]))]


def molecules(graphs=6, seed=3, one_direction=False):
    b = syn.zinc_batch(graphs, seed)
    if one_direction:
        b = syn.one_direction_only(b, seed)
    return Graph(_shuffle(b["edge_index"], seed), b["x"].shape[0])


IN_DEGREES = list(range(10)) + [30, 31, 32, 33, 1000]


def shaped_graph(seed=7, fan_out=1000, isolated=6):
    """Nodes 0..14 with in-degrees 0..9 (every tail of the four-way unrolled gather), 30..33 (31..34 messages with the self-loop:
    one, two warp trips) and a hub of 1000; one node that is the source of `fan_out` edges; `isolated` nodes touched by no edge."""
    rng = np.random.default_rng(seed)
    k = len(IN_DEGREES)
    body = k + fan_out + 8
    tgt = np.repeat(np.arange(k), IN_DEGREES)
    src = rng.integers(0, body, size=len(tgt))
    tgt = np.concatenate([tgt, k + rng.permutation(body - k)[:fan_out]])  # the fan-out hub feeds nodes past the degree classes
    src = np.concatenate([src, np.full(fan_out, body)])
    return Graph(_shuffle(torch.from_numpy(np.stack([tgt, src])), seed), body + 1 + isolated)


def empty_graph(n=40):
    return Graph(torch.zeros(2, 0, dtype=torch.int64), n)


# ---------------------------------------------------------------------------------------------------------------------------
# GAT: case, fp64 / fp32 restatement, device run
# ---------------------------------------------------------------------------------------------------------------------------
class GatCase:
    """Inputs of one GAT layer.  Regimes of the activated logits (set through att[:, 0], which multiplies a 0/1 column 0 of xl):
    ordinary |raw| ~ 1; large ~ +60; negative: every logit of every node below -40; mixed: that for a seeded half of the nodes."""

    def __init__(self, graph, H, D, domain, seed=0, regime="ordinary", slope=0.2, fractional=False):
        self.graph, self.n, self.E, self.H, self.D, self.domain, self.slope = graph, graph.n, graph.E, H, D, domain, slope
        self.regime = regime
        self.Q = 9 if domain == "chem" else 10
        g = torch.Generator().manual_seed(1000 * H + D + seed)
        self.xl = torch.randn(graph.n, H, D, generator=g)
        self.att = torch.randn(H, 2 * D, generator=g) / math.sqrt(2 * D)
        self.T = torch.randn(self.Q, H * D, generator=g) * 0.5
        self.bias = torch.randn(D, generator=g) * 0.1
        self.R = torch.randn(graph.n, D, generator=g)
        E = graph.E
        if domain == "chem":
            self.feat = torch.stack([torch.randint(0, 6, (E,), generator=g), torch.randint(0, 3, (E,), generator=g)], 1)
        elif fractional:
            self.feat = torch.rand(E, 9, generator=g)
        else:
            self.feat = (torch.rand(E, 9, generator=g) < 0.3).float()
        if regime != "ordinary":
            on = torch.ones(graph.n) if regime in ("large", "negative") else (torch.rand(graph.n, generator=g) < 0.5).float()
            self.xl[:, :, 0] = on[:, None]
            self.att[:, 0] = 60.0 if regime == "large" else -45.0 / slope


def edge_features(c, dtype, wrong_loop=False):
    """[E + n, Q] feature weights f_k (self-loops last): chem one-hot bond type, one-hot direction, self-loop [4, 0]; bio the 9
    attributes with the self-loop one-hot at column 7, then a constant 1 for the encoder bias."""
    n, E = c.n, c.E
    if c.domain == "chem":
        loops = torch.zeros(n, 2, dtype=torch.int64)
        loops[:, 0] = 0 if wrong_loop else O.SELF_LOOP_BOND
        codes = torch.cat([c.feat, loops])
        f = torch.zeros(E + n, 9, dtype=dtype)
        r = torch.arange(E + n)
        f[r, codes[:, 0]] = 1
        f[r, 6 + codes[:, 1]] = 1
        return f
    loops = torch.zeros(n, 9)
    loops[:, 0 if wrong_loop else O.BIO_SELF_LOOP_COL] = 1
    return torch.cat([torch.cat([c.feat, loops]), torch.ones(E + n, 1)], 1).to(dtype)


VARIANTS = ("plain segment max", "no 1e-16", "wrong self-loop feature", "slope ignored in backward", "p and q swapped",
            "heads summed")


def _softmax(act, tgt, n, variant):
    if variant not in ("plain segment max", "no 1e-16"):
        return O.segment_softmax(act, tgt, n)
    idx = tgt.view(-1, 1).expand_as(act)
    mx = torch.zeros(n, act.shape[1], dtype=act.dtype).scatter_reduce(0, idx, act.detach(), reduce="amax",
                                                                       include_self=variant != "plain segment max")
    ex = (act - mx[tgt]).exp()
    den = torch.zeros(n, act.shape[1], dtype=act.dtype).index_add_(0, tgt, ex)
    return ex / (den[tgt] + (0.0 if variant == "no 1e-16" else O.SOFTMAX_EPS))


def gat_reference(c, dtype=torch.float64, variant=None):
    """The GAT layer for general H in `dtype`:  x'_k = xl[src] + f_k T;  raw = <att[h,:D], xl[tgt]> + <att[h,D:], x'_k>;
    leaky_relu(slope); segment softmax over targets (the oracle's: shift max(0, segment max), +1e-16); mean over heads + bias.
    Gradients by autograd of sum(out * R).  `variant` restates one of VARIANTS instead."""
    n, H, D = c.n, c.H, c.D
    xl, att, T, bias = (t.to(dtype, copy=True).requires_grad_(True) for t in (c.xl, c.att, c.T, c.bias))
    ei = c.graph.looped()
    tgt, src = ei[0], ei[1]
    f = edge_features(c, dtype, wrong_loop=variant == "wrong self-loop feature")
    xj = xl[src] + (f @ T).view(-1, H, D)
    ap, aq = (att[:, D:], att[:, :D]) if variant == "p and q swapped" else (att[:, :D], att[:, D:])
    raw = (xl[tgt] * ap).sum(-1) + (xj * aq).sum(-1)
    act = F.leaky_relu(raw, c.slope)
    if variant == "slope ignored in backward":
        act = raw + (act - raw).detach()
    alpha = _softmax(act, tgt, n, variant)
    msg = O.reduce_onto_target(xj * alpha.unsqueeze(-1), tgt, n)
    out = (msg.sum(1) if variant == "heads summed" else msg.mean(1)) + bias
    with torch.no_grad():
        pq = torch.stack([(xl * ap).sum(-1), (xl * aq).sum(-1)], -1)
    (out * c.R.to(dtype)).sum().backward()
    return dict(out=out.detach(), alpha=alpha.detach(), pq=pq, gxl=xl.grad.reshape(n, H * D), gatt=att.grad, gT=T.grad,
                gbias=bias.grad)


def run_gat(c, ldo=None, ldg=None, ws_bytes=None):
    """pgnn_gat_fwd + pgnn_gat_bwd on the device; alpha is returned in edge_index order (self-loops last).  The backward's
    workspace is NaN-filled: every slot must be written before it is read."""
    L, gr = cabi.lib, c.graph
    n, H, D, E, Q = c.n, c.H, c.D, c.E, c.Q
    ldo = ldo or D + 3
    ldg = ldg or ceil4(D) + 4
    XL, ATT, TT, BIAS = filled(c.xl.reshape(n, H * D)), filled(c.att), filled(c.T), filled(c.bias[None])
    FEAT = filled(c.feat, fill=-1) if c.domain == "chem" else filled(c.feat)
    feat = FEAT.ptr() if E else None
    bio = int(c.domain == "bio")
    OUT, ALPHA, PQ = Region(n, D, ldo, SENT), Region(E + n, H, H, SENT), Region(n, 2 * H, 2 * H, SENT)
    rc = L.pgnn_gat_fwd(XL.ptr(), n, H, D, ATT.ptr(), TT.ptr(), bio, feat, gr.ptr("rowptr_t"), gr.ptr("nbr_t"), gr.ptr("eid_t"), E,
                        BIAS.ptr(), c.slope, ALPHA.ptr(), PQ.ptr(), OUT.ptr(), ldo, _stream())
    assert rc == OK, rc
    G = filled(c.R, ld=ldg)
    GXL, GATT, GT, GB = Region(n, H * D, H * D, SENT), Region(H, 2 * D, 2 * D, SENT), Region(Q, H * D, H * D, SENT), Region(1, D, D, SENT)
    need = L.pgnn_gat_bwd_workspace_bytes(n, E, H, D)
    assert need > 0
    WS = torch.full((need // 4 + 64,), NAN, device=DEV)
    rc = L.pgnn_gat_bwd(G.ptr(), ldg, XL.ptr(), n, H, D, ATT.ptr(), TT.ptr(), bio, feat, gr.ptr("rowptr_t"), gr.ptr("nbr_t"),
                        gr.ptr("eid_t"), gr.ptr("rowptr_s"), gr.ptr("nbr_s"), gr.ptr("eid_s"), E, c.slope, ALPHA.ptr(), PQ.ptr(),
                        GXL.ptr(), GATT.ptr(), GT.ptr(), GB.ptr(), WS.data_ptr(), need if ws_bytes is None else ws_bytes, _stream())
    torch.cuda.synchronize()
    res = dict(rc=rc, intact=all(r.outside_intact() for r in (OUT, ALPHA, PQ, GXL, GATT, GT, GB)),
               ws_tail_untouched=bool(WS[need // 4:].isnan().all()), ws_untouched=bool(WS.isnan().all()))
    alpha = torch.empty(E + n, H)
    alpha[gr.bucket_perm()] = ALPHA.view.cpu()
    res.update(out=OUT.view.cpu(), alpha=alpha, pq=PQ.view.cpu().view(n, H, 2), gxl=GXL.view.cpu(), gatt=GATT.view.cpu(),
               gT=GT.view.cpu(), gbias=GB.view.cpu()[0])
    return res


def bound_rows(mine, r32, r64, label):
    """Outputs on their own scale; a gradient on its own scale floored at 1e-3 of the largest gradient, and on that largest
    gradient where it is structurally ~0 (gatt when every node has only its self-loop), as golden_util.gradient_check does."""
    rows = []
    gmax = max(float(r64[k].abs().max()) for k, floor in FLOOR.items() if floor == GRAD_REL)
    for k, floor in FLOOR.items():
        ref = r64[k].double()
        scale = max(float(ref.abs().max()), 1e-30)
        if floor == GRAD_REL:
            scale = gmax if scale < 1e-9 * gmax else max(scale, 1e-3 * gmax)
        e = float((mine[k].double() - ref).abs().max()) / scale
        eref = float((r32[k].double() - ref).abs().max()) / scale
        tol = max(floor, SLACK * eref)
        rows.append(dict(kind=k, name=label, err=e, err_ref32=eref, tol=tol, ok=bool(e <= tol)))
    return rows


def check_gat(c, label, report, **kw):
    r64, r32 = gat_reference(c), gat_reference(c, torch.float32)
    mine = run_gat(c, **kw)
    assert mine["rc"] == OK, mine["rc"]
    rows = bound_rows(mine, r32, r64, label)
    write_report(report, rows, dict(H=c.H, D=c.D, domain=c.domain, regime=c.regime, slope=c.slope, n=c.n, E=c.E, **card()))
    assert mine["intact"], label + ": a sentinel around an output was overwritten"
    assert mine["ws_tail_untouched"], label + ": workspace written past its size"
    bad = [r for r in rows if not r["ok"]]
    assert not bad, bad
    return mine


# ---------------------------------------------------------------------------------------------------------------------------
# 1. GAT forward and backward
# ---------------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("domain", ["chem", "bio"])
@pytest.mark.parametrize("D", [1, 4, 33, 300, 301, 320])
@pytest.mark.parametrize("H", [1, 2, 3, 4])
def test_gat_heads_and_widths(H, D, domain):
    # H <= 2 with D % 4 == 0 reduces the tables in one batched float4 launch; H >= 3 or D % 4 != 0 per head on the scalar kernel
    check_gat(GatCase(molecules(), H, D, domain), "H%d D%d %s" % (H, D, domain), "graph_gat_H%d_D%d_%s" % (H, D, domain))


GRAPH_SHAPES = {
    "one direction only": lambda: molecules(8, 5, one_direction=True),
    "degrees 0-9 30-33 hubs isolated": lambda: shaped_graph(),
    "no edges": lambda: empty_graph(),
}


@gpu
@pytest.mark.parametrize("domain,fractional", [("chem", False), ("bio", False), ("bio", True)])
@pytest.mark.parametrize("shape", list(GRAPH_SHAPES))
def test_gat_graph_shapes(shape, domain, fractional):
    c = GatCase(GRAPH_SHAPES[shape](), 2, 300, domain, seed=1, fractional=fractional)
    label = "%s %s%s" % (shape, domain, " fractional" if fractional else "")
    check_gat(c, label, "graph_gat_shape_" + label.replace(" ", "_"))


@gpu
@pytest.mark.parametrize("domain", ["chem", "bio"])
@pytest.mark.parametrize("slope", [0.2, 0.01])
@pytest.mark.parametrize("regime", ["ordinary", "large", "negative", "mixed"])
def test_gat_logit_regimes(regime, slope, domain):
    c = GatCase(molecules(), 2, 300, domain, seed=2, regime=regime, slope=slope)
    label = "%s slope %g %s" % (regime, slope, domain)
    check_gat(c, label, "graph_gat_regime_" + label.replace(" ", "_"))


@gpu
@pytest.mark.parametrize("ldo,ldg", [(301, 304), (600, 900), (307, 301)])  # aligned; wide; ldg % 4 != 0 (per-head tables)
def test_gat_strides(ldo, ldg):
    check_gat(GatCase(molecules(), 2, 300, "chem", seed=3), "ldo %d ldg %d" % (ldo, ldg), "graph_gat_ld_%d_%d" % (ldo, ldg),
              ldo=ldo, ldg=ldg)


@gpu
def test_gat_forward_and_gxl_repeat_bit_for_bit():
    c = GatCase(shaped_graph(), 2, 300, "chem", seed=4)
    a, b = run_gat(c), run_gat(c)
    for k in ("out", "alpha", "pq", "gxl"):
        assert torch.equal(a[k], b[k]), k


@gpu
def test_gat_backward_refuses_a_short_workspace():
    c = GatCase(molecules(), 2, 300, "chem", seed=5)
    need = cabi.lib.pgnn_gat_bwd_workspace_bytes(c.n, c.E, c.H, c.D)
    r = run_gat(c, ws_bytes=need - 1)
    assert r["rc"] == EWORKSPACE and r["ws_untouched"]
    assert bool((r["gxl"] == SENT).all()), "gxl must not be written when the workspace is refused"


_TABLE_ENV = textwrap.dedent("""
    import sys
    sys.path.insert(0, sys.argv[1]); sys.path.insert(0, sys.argv[1] + "/tests")
    import test_gpu_graph_kernels as T
    for job in sys.argv[2:]:
        getattr(T, job)()
    print("jobs ok")
""")


def _run_with_env(env_value, *jobs):
    env = dict(os.environ, PGNN_TABLE_V4=env_value)
    r = subprocess.run([sys.executable, "-c", _TABLE_ENV, ROOT, *jobs], capture_output=True, text=True, timeout=1200, cwd=ROOT, env=env)
    assert r.returncode == 0 and "jobs ok" in r.stdout, r.stdout[-3000:] + r.stderr[-6000:]


def gat_scalar_tables_job():
    for domain in ("chem", "bio"):
        c = GatCase(molecules(), 2, 300, domain, seed=6)
        check_gat(c, "PGNN_TABLE_V4=0 " + domain, "graph_gat_table_v4_off_" + domain)


@gpu
def test_gat_with_the_batched_table_kernel_off():
    # PGNN_TABLE_V4=0 (read once per process): H = 2, D = 300 goes through the per-head scalar table reductions
    _run_with_env("0", "gat_scalar_tables_job")


# ---------------------------------------------------------------------------------------------------------------------------
# 2. aggregation, summaries, edge tables
# ---------------------------------------------------------------------------------------------------------------------------
def agg_weights(gr, mode, dinv64):
    """per message of graph.looped(): w_k (fp64)"""
    ei = gr.looped()
    if mode == SUM:
        return torch.ones(ei.shape[1], dtype=torch.float64)
    if mode == MEAN:
        return 1.0 / (gr.in_deg.double() + 1.0)[ei[0]]
    return dinv64[ei[0]] * dinv64[ei[1]]


def dinv_of(gr):
    d64 = (gr.in_deg.double() + 1.0).pow(-0.5)
    return d64, d64.float()


def agg_reference(gr, x, mode, dinv64, scale=None, shift=None, relu=False, S=None, T=None):
    """(sum_k w_k x_eff[src_k] onto targets, same over magnitudes, S.T, |S|.|T|) in fp64; x_eff = act(x * scale + shift)"""
    ei = gr.looped()
    xe, mag = x.double(), x.double().abs()
    if scale is not None:
        xe = xe * scale.double() + shift.double()
        mag = mag * scale.double().abs() + shift.double().abs()
    if relu:
        xe = torch.relu(xe)
    w = agg_weights(gr, mode, dinv64)[:, None]
    z = torch.zeros(gr.n, x.shape[1], dtype=torch.float64)
    ref = z.clone().index_add_(0, ei[0], w * xe[ei[1]])
    den = z.clone().index_add_(0, ei[0], w.abs() * mag[ei[1]])
    if S is None:
        return ref, den, None, None
    return ref, den, S.double() @ T.double(), S.double().abs() @ T.double().abs()


def run_aggregate(gr, x, mode, dinv32, scale=None, shift=None, relu=False, S=None, T=None, edge_off=0, ldx=None, ldo=None):
    n, C = x.shape
    X = filled(x, ld=ldx or C + 4)
    width = edge_off + C if edge_off else C
    OUT = Region(n, width, ldo or ceil4(width) + 8, SENT)
    keep = [filled(t) if t is not None else None for t in (scale, shift, S, T)]
    SC, SH, SS, TT = keep
    DI = filled(dinv32[None]) if mode == GCN else None
    p = lambda r: r.ptr() if r is not None else None
    rc = cabi.lib.pgnn_aggregate_fwd(X.ptr(), X.ld, p(SC), p(SH), int(relu), n, C, gr.ptr("rowptr_t"), gr.ptr("nbr_t"), mode, p(DI),
                                     p(SS), 0 if S is None else S.shape[1], p(TT), edge_off, OUT.ptr(), OUT.ld, _stream())
    assert rc == OK, rc
    torch.cuda.synchronize()
    out = OUT.view.cpu()
    intact = OUT.outside_intact() and (not edge_off or bool((out[:, C:edge_off] == SENT).all()))
    return out, intact


def _within(got, ref, den, tau=TAU):
    """worst |got - ref| / den (exact agreement required where den == 0)"""
    e = (got.double() - ref).abs()
    e = torch.where(den > 0, e / den.clamp_min(1e-300), torch.where(e == 0, 0.0, float("inf")))
    return float(e.max()) if e.numel() else 0.0


AGG_GRAPHS = {"degrees": lambda: shaped_graph(seed=11), "molecules": lambda: molecules(16, 9)}


@gpu
@pytest.mark.parametrize("graph", list(AGG_GRAPHS))
@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("C", [4, 8, 300, 600])
def test_aggregate_fwd(C, mode, graph):
    gr, m = AGG_GRAPHS[graph](), MODES[mode]
    g = torch.Generator().manual_seed(C + m)
    x = torch.randn(gr.n, C, generator=g)
    Q = 10
    S = torch.rand(gr.n, Q, generator=g) * (torch.rand(gr.n, Q, generator=g) < 0.5)
    T = torch.randn(Q, C, generator=g)
    scale, shift = torch.randn(C, generator=g), torch.randn(C, generator=g) * 0.5
    d64, d32 = dinv_of(gr)
    rows = []
    for with_S, concat in ((False, False), (True, False), (True, True)):
        for aff, relu in ((False, False), (False, True), (True, False), (True, True)):
            kw = dict(scale=scale, shift=shift) if aff else {}
            ref, den, e_ref, e_den = agg_reference(gr, x, m, d64, relu=relu, S=S if with_S else None, T=T, **kw)
            out, intact = run_aggregate(gr, x, m, d32, relu=relu, S=S if with_S else None, T=T if with_S else None,
                                        edge_off=C + 4 if concat else 0, **kw)
            label = "S%d concat%d affine%d relu%d" % (with_S, concat, aff, relu)
            assert intact, label
            if concat:
                err = max(_within(out[:, :C], ref, den), _within(out[:, C + 4:], e_ref, e_den))
            elif with_S:
                err = _within(out, ref + e_ref, den + e_den)
            else:
                err = _within(out, ref, den)
            rows.append(dict(kind="aggregate_fwd", name="%s C%d %s %s" % (mode, C, graph, label), err=err, err_ref32=0.0))
            assert err <= TAU, (label, err)
    write_report("graph_aggregate_fwd_%s_C%d_%s" % (mode, C, graph), rows, dict(tau=TAU, **card()))


@gpu
@pytest.mark.parametrize("graph", list(AGG_GRAPHS))
@pytest.mark.parametrize("mode", ["sum", "mean"])
@pytest.mark.parametrize("C", [4, 8, 300, 600])
def test_aggregate_fwd_bit_exact(C, mode, graph):
    gr = AGG_GRAPHS[graph]()
    x = torch.randn(gr.n, C, generator=torch.Generator().manual_seed(C))
    ei = gr.looped()
    ref = O.reduce_onto_target(x[ei[1]], ei[0], gr.n, mean=mode == "mean")
    out, intact = run_aggregate(gr, x, MODES[mode], None, ldx=C + 8, ldo=C + 12)
    assert intact
    assert torch.equal(out, ref), int((out != ref).sum())


def run_aggregate_bwd(gr, gy, mode, dinv32):
    n, C = gy.shape
    G, GX = filled(gy, ld=C + 4), Region(n, C, C + 8, SENT)
    DI = filled(dinv32[None]) if mode == GCN else None
    rc = cabi.lib.pgnn_aggregate_bwd(G.ptr(), G.ld, n, C, gr.ptr("rowptr_s"), gr.ptr("nbr_s"), mode, DI.ptr() if DI else None,
                                     gr.ptr("rowptr_t"), GX.ptr(), GX.ld, _stream())
    assert rc == OK, rc
    torch.cuda.synchronize()
    return GX.view.cpu(), GX.outside_intact()


@gpu
@pytest.mark.parametrize("graph", list(AGG_GRAPHS))
@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("C", [4, 300, 600])
def test_aggregate_bwd(C, mode, graph):
    gr, m = AGG_GRAPHS[graph](), MODES[mode]
    gy = torch.randn(gr.n, C, generator=torch.Generator().manual_seed(C + 7))
    d64, d32 = dinv_of(gr)
    got, intact = run_aggregate_bwd(gr, gy, m, d32)
    assert intact
    ei = gr.looped()
    if m == SUM:  # transpose gather: source-bucket order (edge order), self-loop last -- the order of index_add_ onto sources
        ref = O.reduce_onto_target(gy[ei[0]], ei[1], gr.n)
        assert torch.equal(got, ref), int((got != ref).sum())
        return
    w = agg_weights(gr, m, d64)[:, None]
    ref = torch.zeros(gr.n, C, dtype=torch.float64).index_add_(0, ei[1], w * gy.double()[ei[0]])
    den = torch.zeros(gr.n, C, dtype=torch.float64).index_add_(0, ei[1], w.abs() * gy.double().abs()[ei[0]])
    err = _within(got, ref, den)
    write_report("graph_aggregate_bwd_%s_C%d_%s" % (mode, C, graph),
                 [dict(kind="aggregate_bwd", name="%s C%d %s" % (mode, C, graph), err=err, err_ref32=0.0)], dict(tau=TAU, **card()))
    assert err <= TAU, err


def summary_reference(gr, domain, feat, mode, dinv64):
    f = edge_features(types.SimpleNamespace(domain=domain, feat=feat, n=gr.n, E=gr.E), torch.float64)
    w = agg_weights(gr, mode, dinv64)[:, None]
    ei = gr.looped()
    return torch.zeros(gr.n, f.shape[1], dtype=torch.float64).index_add_(0, ei[0], w * f)


@gpu
@pytest.mark.parametrize("graph", list(AGG_GRAPHS) + ["no edges"])
@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("domain,fractional", [("chem", False), ("bio", False), ("bio", True)])
def test_edge_summaries(domain, fractional, mode, graph):
    gr, m = (empty_graph() if graph == "no edges" else AGG_GRAPHS[graph]()), MODES[mode]
    g = torch.Generator().manual_seed(m + 3 * fractional)
    if domain == "chem":
        feat = torch.stack([torch.randint(0, 6, (gr.E,), generator=g), torch.randint(0, 3, (gr.E,), generator=g)], 1)
        FEAT, Q = filled(feat, fill=-1), 9
    else:
        feat = torch.rand(gr.E, 9, generator=g) if fractional else (torch.rand(gr.E, 9, generator=g) < 0.3).float()
        FEAT, Q = filled(feat), 10
    d64, d32 = dinv_of(gr)
    DI = filled(d32[None])
    S = Region(gr.n, Q, Q, SENT)
    fn = cabi.lib.pgnn_chem_edge_summary if domain == "chem" else cabi.lib.pgnn_bio_edge_summary
    rc = fn(FEAT.ptr() if gr.E else None, gr.ptr("rowptr_t"), gr.ptr("nbr_t"), gr.ptr("eid_t"), gr.n, m, DI.ptr(), S.ptr(), _stream())
    assert rc == OK, rc
    torch.cuda.synchronize()
    got = S.view.cpu()
    assert S.outside_intact()
    ref = summary_reference(gr, domain, feat, m, d64)
    if domain == "chem" and m == SUM:
        assert torch.equal(got, ref.float()), "chem SUM summaries are integer counts"
        return
    # every weight and feature is >= 0, so the rounding errors of the sequential fp32 sum do not cancel: a row of in-degree d
    # is held to (d + 2) u of its value (d + 1 additions, one rounded weight), and at least TAU
    tau = ((gr.in_deg.double() + 2) * 2.0 ** -24).clamp_min(TAU)[:, None]
    ok = bool(((got.double() - ref).abs() <= tau * ref).all())
    err = _within(got, ref, ref)  # relative error, reported
    write_report("graph_edge_summary_%s%s_%s_%s" % (domain, "_fractional" if fractional else "", mode, graph.replace(" ", "_")),
                 [dict(kind="edge_summary", name="%s %s %s" % (domain, mode, graph), err=err, err_ref32=0.0)], card())
    assert ok, err


@gpu
def test_gcn_dinv_within_one_ulp():
    deg = np.concatenate([np.arange(0, 4100), [8191, 8192, 65535, 65536, 1 << 20, (1 << 24) - 2, (1 << 24) + 7]]).astype(np.int64)
    rowptr = np.zeros(len(deg) + 1, dtype=np.int64)
    np.cumsum(deg, out=rowptr[1:])
    rp = torch.from_numpy(rowptr.astype(np.int32)).to(DEV)
    out = Region(1, len(deg), len(deg), SENT)
    assert cabi.lib.pgnn_gcn_dinv(rp.data_ptr(), len(deg), out.ptr(), _stream()) == OK
    torch.cuda.synchronize()
    got = out.view.cpu()[0].double().numpy()
    ref = (deg.astype(np.float64) + 1.0) ** -0.5
    ulp = np.spacing(ref.astype(np.float32)).astype(np.float64)
    assert out.outside_intact()
    worst = np.abs(got - ref) / ulp
    assert float(worst.max()) <= 1.0, (deg[np.argmax(worst)], float(worst.max()))


TABLE_ROWS = [1, 63, 64, 65, 16383, 16384, 16385]  # the 64-row blocks, the switch to 256-row blocks at n = 16384


def check_edge_tables(n):
    rows = []
    for C in (300, 45):  # 45: not a multiple of 32 (nor of 4: the float4 kernel declines it)
        for Q in (1, 2, 9, 10, 16):
            for g_off in (0, C):
                g = torch.Generator().manual_seed(n + 17 * Q + C + g_off)
                S = torch.rand(n, Q, generator=g) * (torch.rand(n, Q, generator=g) < 0.6)
                gy = torch.randn(n, C, generator=g)
                SS = filled(S)
                G = Region(n, g_off + C, ceil4(g_off + C) + 4, NAN)  # the g_off columns before the view stay NaN
                G.view[:, g_off:] = gy.to(DEV)
                GT = Region(Q, C, C, SENT)
                rc = cabi.lib.pgnn_edge_table_bwd(SS.ptr(), Q, G.ptr(), G.ld, g_off, n, C, GT.ptr(), _stream())
                assert rc == OK, rc
                torch.cuda.synchronize()
                assert GT.outside_intact(), (n, C, Q, g_off)
                ref, den = S.double().t() @ gy.double(), S.double().t().abs() @ gy.double().abs()
                err = _within(GT.view.cpu(), ref, den)
                rows.append(dict(kind="edge_table_bwd", name="n%d C%d Q%d off%d" % (n, C, Q, g_off), err=err, err_ref32=0.0))
                assert err <= TAU, rows[-1]
    write_report("graph_edge_table_n%d_v4%s" % (n, os.environ.get("PGNN_TABLE_V4", "")), rows, dict(tau=TAU, **card()))


def edge_table_all_job():
    for n in TABLE_ROWS:
        check_edge_tables(n)


@gpu
@pytest.mark.parametrize("n", TABLE_ROWS)
def test_edge_table_bwd(n):
    check_edge_tables(n)


@gpu
def test_edge_table_bwd_float4_kernel():
    # PGNN_TABLE_V4=1 (read once per process) sends single reductions with C % 4 == 0 to the float4 kernel
    _run_with_env("1", "edge_table_all_job")


# ---------------------------------------------------------------------------------------------------------------------------
# 3. ReLU keeps NaN: on the aggregation's load, in BatchNorm and in the inter-layer ReLU
# ---------------------------------------------------------------------------------------------------------------------------
def _classes(t):
    return t.isnan(), t == float("inf"), t == float("-inf")


def _plant(x):
    x = x.clone()
    for (r, c), v in {(3, 5): NAN, (10, 7): float("inf"), (20, 11): float("-inf"), (40, 2): float("inf"), (41, 2): NAN}.items():
        x[r, c] = v
    return x


@gpu
@pytest.mark.parametrize("affine", [False, True])
@pytest.mark.parametrize("mode", list(MODES))
def test_aggregate_relu_on_load_keeps_nan(mode, affine):
    gr, m = molecules(8, 4), MODES[mode]
    C = 300
    g = torch.Generator().manual_seed(31)
    x = _plant(torch.randn(gr.n, C, generator=g))
    scale, shift = None, None
    if affine:  # mixed signs: the -Inf planted in column 11 comes out as +Inf, the +Inf of column 7 stays +Inf
        scale, shift = torch.randn(C, generator=g), torch.randn(C, generator=g) * 0.5
        scale[[2, 7]], scale[11] = scale[[2, 7]].abs(), -scale[11].abs()
    d64, d32 = dinv_of(gr)
    ref = agg_reference(gr, x, m, d64, scale, shift, relu=True)[0]
    den = agg_reference(gr, torch.nan_to_num(x, 0.0, 0.0, 0.0), m, d64, scale, shift, relu=True)[1]
    got, intact = run_aggregate(gr, x, m, d32, scale, shift, relu=True)
    assert intact
    want = _classes(ref)
    assert want[0].any() and want[1].any()
    for a, b, what in zip(_classes(got), want, ("NaN", "+Inf", "-Inf")):
        assert torch.equal(a, b), (what, int((a != b).sum()))
    fin = torch.isfinite(ref)
    assert _within(got[fin], ref[fin], den[fin]) <= TAU


def _bn_inputs(C, seed):
    g = torch.Generator().manual_seed(seed)
    x = _plant(torch.randn(97, C, generator=g) * 2 + 1)
    gamma, beta = torch.randn(C, generator=g), torch.randn(C, generator=g) * 0.3
    rm, rv = torch.randn(C, generator=g) * 0.1, 0.5 + torch.rand(C, generator=g)
    return x, gamma, beta, rm, rv


def _same_nonfinite(got, ref):
    for a, b, what in zip(_classes(got), _classes(ref), ("NaN", "+Inf", "-Inf")):
        assert torch.equal(a, b), (what, int((a != b).sum()))
    fin = torch.isfinite(ref)
    assert bool(((got[fin].double() - ref[fin]).abs() <= 1e-4 + 1e-4 * ref[fin].abs()).all())


# scalar kernels: C odd; float4 kernels: C and every row stride a multiple of 4
BN_PATHS = {"scalar": (301, 305), "float4": (300, 304)}


@gpu
@pytest.mark.parametrize("path", list(BN_PATHS))
def test_batch_norm_and_relu_keep_nan(path):
    C, ld = BN_PATHS[path]
    x, gamma, beta, rm, rv = _bn_inputs(C, 5)
    M = x.shape[0]
    L = cabi.lib
    X = filled(x, ld=ld)
    GA, BE, RM, RV = (filled(t[None]) for t in (gamma, beta, rm, rv))
    # train: a non-finite value makes its whole column's statistics NaN, and so the column
    Y = Region(M, C, ld, SENT)
    SM, SI = Region(1, C, C, SENT), Region(1, C, C, SENT)
    wsb = L.pgnn_bn_workspace_bytes(M, C)
    ws = torch.empty(wsb // 4 + 16, device=DEV)
    assert L.pgnn_bn_fwd_train(X.ptr(), ld, M, C, GA.ptr(), BE.ptr(), None, None, None, 0.1, 1e-5, 1, Y.ptr(), ld, SM.ptr(), SI.ptr(),
                               None, None, ws.data_ptr(), wsb, _stream()) == OK
    torch.cuda.synchronize()
    ref = torch.relu(F.batch_norm(x.double(), None, None, gamma.double(), beta.double(), True, 0.1, 1e-5))
    assert Y.outside_intact()
    assert ref.isnan().any()
    _same_nonfinite(Y.view.cpu(), ref)
    # eval: element by element
    Y = Region(M, C, ld, SENT)
    assert L.pgnn_bn_fwd_eval(X.ptr(), ld, M, C, GA.ptr(), BE.ptr(), RM.ptr(), RV.ptr(), 1e-5, 1, Y.ptr(), ld, _stream()) == OK
    torch.cuda.synchronize()
    ref = torch.relu(F.batch_norm(x.double(), rm.double(), rv.double(), gamma.double(), beta.double(), False, 0.1, 1e-5))
    assert Y.outside_intact()
    _same_nonfinite(Y.view.cpu(), ref)
    # the inter-layer ReLU
    Y = Region(M, C, ld, SENT)
    assert L.pgnn_relu_fwd(X.ptr(), ld, M, C, Y.ptr(), ld, _stream()) == OK
    torch.cuda.synchronize()
    assert Y.outside_intact()
    got, ref = Y.view.cpu(), torch.relu(x)
    _same_nonfinite(got, ref.double())
    assert torch.equal(got.isnan(), x.isnan())


# ---------------------------------------------------------------------------------------------------------------------------
# CPU: the GAT bound can see the mistakes it is meant to catch; argument checks that return before any device work
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("domain", ["chem", "bio"])
def test_gat_bound_rejects_wrong_variants(domain):
    """On the mixed-regime inputs of test_gat_logit_regimes (some nodes with every logit below -40, where the max(0, .) shift and
    the 1e-16 decide the result), the fp32 restatement passes the bound and each variant misses it by 10x or more."""
    c = GatCase(molecules(), 2, 300, domain, seed=2, regime="mixed", slope=0.2)
    r64, r32 = gat_reference(c), gat_reference(c, torch.float32)
    assert all(r["ok"] for r in bound_rows(r32, r32, r64, "fp32"))
    misses = {}
    for v in VARIANTS:
        rows = bound_rows(gat_reference(c, torch.float32, v), r32, r64, v)
        misses[v] = max(r["err"] / r["tol"] for r in rows)
    assert min(misses.values()) >= 10, misses


def test_gat_mixed_regime_is_what_it_claims():
    c = GatCase(molecules(), 2, 300, "chem", seed=2, regime="mixed", slope=0.2)
    ei = c.graph.looped()
    with torch.no_grad():
        f = edge_features(c, torch.float64)
        xl, att = c.xl.double(), c.att.double()
        xj = xl[ei[1]] + (f @ c.T.double()).view(-1, 2, 300)
        act = F.leaky_relu((xl[ei[0]] * att[:, :300]).sum(-1) + (xj * att[:, 300:]).sum(-1), 0.2)
    node_max = torch.full((c.n, 2), -float("inf"), dtype=torch.float64).scatter_reduce(0, ei[0].view(-1, 1).expand_as(act), act, "amax")
    low = (node_max < -40).all(1)
    assert 0.3 * c.n < int(low.sum()) < 0.7 * c.n
    assert float(node_max[~low].abs().max()) < 10


def test_argument_checks():
    L = cabi.lib
    fake = 1 << 20  # 16-byte aligned, never dereferenced: every call below returns before any device work
    def fwd(H=2, D=300):
        return L.pgnn_gat_fwd(fake, 10, H, D, fake, fake, 0, fake, fake, fake, fake, 20, fake, 0.2, fake, fake, fake, D, None)

    def bwd(H=2, D=300):
        return L.pgnn_gat_bwd(fake, D, fake, 10, H, D, fake, fake, 0, fake, fake, fake, fake, fake, fake, fake, 20, 0.2, fake, fake,
                              fake, fake, fake, fake, fake, 1 << 30, None)
    for f in (fwd, bwd):
        assert f(H=0) == EINVAL and f(D=0) == EINVAL
        assert f(H=5) == EUNSUPPORTED and f(D=321) == EUNSUPPORTED
    assert L.pgnn_gat_bwd_workspace_bytes(10, 20, 0, 300) == EINVAL

    def agg(Q=9, edge_off=0, S=fake):
        return L.pgnn_aggregate_fwd(fake, 300, None, None, 0, 10, 300, fake, fake, SUM, None, S, Q, fake, edge_off, fake, 904, None)
    assert agg(Q=17) == EINVAL and agg(Q=0) == EINVAL and agg(edge_off=302) == EINVAL and agg(edge_off=300, S=None) == EINVAL
    assert L.pgnn_aggregate_fwd(fake, 300, fake, None, 1, 10, 300, fake, fake, SUM, None, None, 0, None, 0, fake, 300, None) == EINVAL
    assert L.pgnn_aggregate_fwd(fake, 300, None, None, 0, 10, 300, fake, fake, GCN, None, None, 0, None, 0, fake, 300, None) == EINVAL
    for Q in (0, 17):
        assert L.pgnn_edge_table_bwd(fake, Q, fake, 300, 0, 10, 300, fake, None) == EINVAL
