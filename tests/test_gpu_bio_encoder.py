"""GPU: the bio whole-encoder entry points (pgnn_bio_encoder_forward / _backward, csrc/encoder.cu) directly against fp64, and
bio.GNN's fused path against its layer-by-layer composition.

Every direct case calls the two entry points through ctypes on poisoned buffers (tests/device_buffers.py), as
tests/test_gpu_encoder.py does for chem: each parameter in its own NaN-padded allocation, the workspace NaN-filled before the
forward, g_node_rep NaN-padded with row stride ldg, node_rep a sentinel region with row stride ld_out, the flat gradient buffer
sentinel-filled with slack past `total`, GIN's running statistics in sentinel-guarded regions.  The reference is
tests/encoder_oracle.run with the masked bio encoder in fp64 and fp32, checked with output_check / gradient_check, a running-statistics
bound and an exact num_batches_tracked.

Sweeps: width (one not a multiple of the GEMM tile) x depth (L = 1, 2, 3 and a deep stack), batch shapes (no edges, an in-degree
hub with isolated nodes, one-direction edges, N past one 128-row tile, a PPI-sized batch), modes (eval, dropout p in {0, 0.3, 1},
strides, num_batches_tracked NULL, the side stream off), both precisions, state across calls, a workspace one byte short and
refused shapes.  Module level: fused vs layer-by-layer with dropout under one torch.manual_seed, a refused second backward, one
enqueuing library call per pass, and the two-rank flat-buffer all-reduce."""
import ctypes
import importlib
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import dropout_oracle as DO
import encoder_oracle as EO
from device_buffers import DEV, SENT, Region, card, filled
from golden_util import probe, write_report
from oracle import gnn_oracle as O

pytestmark = pytest.mark.gpu
ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
syn = importlib.import_module("pretrain-gnns_b200.synthetic")
bio = importlib.import_module("pretrain-gnns_b200.bio.model")
ops = importlib.import_module("pretrain-gnns_b200.ops")
cabi = importlib.import_module("pretrain-gnns_b200._cabi")
lib = cabi.lib
TYPES = ("gin", "gcn", "graphsage", "gat")
CODE = {"gin": 0, "gcn": 1, "graphsage": 2, "gat": 3}
OK, EWORKSPACE = 0, -3
FP32, TF32X3 = 0, 1
ISENT = -7777
NBT0 = 7
SLACK_FLOATS = 61
MOMENTUM, EPS = 0.1, 1e-5
DEEP = 12            # from this depth on only output_check's scale-relative half applies (as tests/test_gpu_encoder.py's DEEP)
TWO_ROW_NOISE = 1e-3
# GIN's running statistics against fp64 on the 3xTF32 path (relative to the buffer's largest value): measured on an H100 80GB HBM3
# at 700 W up to 2.0e-6 at D = 300, L = 3 (the fp32 oracle: 1.2e-7), growing with depth; encoder_oracle's floor is 1e-6
TC_STATS_FLOOR = 1e-5
F32, F64 = torch.float32, torch.float64


def bio_gnn(P, x, edge_index, edge_attr, num_layer, gnn_type="gin", training=False, new_stats=None, pre="", masks=None, p=0.0):
    """dropout_oracle.bio_gnn with its inter-layer ReLUs traced (O._relu) like the oracle's own, so that encoder_oracle's ReLU-boundary
    allowance sees every ReLU of the encoder."""
    n = x.shape[0]
    ei = O.with_self_loops(edge_index, n)
    edge_attr = edge_attr.to(P[pre + "gnns.0.input_node_embeddings.weight"].dtype)  # the fp64 run's edge rows in fp64
    h = x
    for l in range(num_layer):
        lp = f"{pre}gnns.{l}."
        rows = O.bio_edge_rows(P, lp, edge_attr, n)
        if l == 0:
            h = F.embedding(h.to(torch.int64).view(-1), P[lp + "input_node_embeddings.weight"])
        if gnn_type == "gin":
            h = O.gin_conv_bio(P, lp, h, ei, rows, training, new_stats)
        else:
            h = {"gcn": O.gcn_conv, "graphsage": O.sage_conv, "gat": O.gat_conv}[gnn_type](P, lp, h, ei, rows)
        if l != num_layer - 1:
            h = O._relu(h)
        h = DO._drop(h, masks, l, p)
    return h


class Ref(EO.Ref):
    """encoder_oracle.Ref on the bio encoder."""

    def __init__(self, P, b, t, L, training, g=None, masks=None, p=0.0, steps=1):
        self.args = (P, b, t, L, training)
        self.kw = dict(g=g, masks=masks, p=p, steps=steps, fn=bio_gnn)
        self.out, self.grads, self.stats = {}, {}, {}
        for dt in (F64, F32):
            self.out[dt], self.grads[dt], self.stats[dt], trace = EO.run(P, b, t, L, training, dt, **self.kw)
            if dt == F64:
                self.near_zero = O.near_zero_preactivations(trace)
                self.near_units = [(i, r, c) for i, x in enumerate(trace)
                                   for r, c in (x.abs() <= EO.NEAR_ZERO * x.abs().max()).nonzero().tolist()]


# ---------------------------------------------------------------------------------------------------------------------------
# batches: x the dummy label (0 / 1, float [N, 1]), edge_attr 9 float bits per edge
# ---------------------------------------------------------------------------------------------------------------------------
def _batch(n, src, dst, seed):
    rng = np.random.default_rng(seed)
    E = len(src)
    ea = (rng.random((E, 9)) < 0.3).astype(np.float32)
    ea[:, 7] = 0  # column 7 is the self-loop bit
    return dict(x=torch.as_tensor(rng.integers(0, 2, size=(n, 1)), dtype=torch.float32),
                edge_index=torch.as_tensor(np.stack([dst, src]).reshape(2, E), dtype=torch.int64), edge_attr=torch.as_tensor(ea).reshape(E, 9))


def random_graph(n, seed, deg=4):
    rng = np.random.default_rng(seed)
    m = deg * n // 2
    u, v = rng.integers(0, n, size=m), rng.integers(0, n, size=m)
    keep = u != v
    return _batch(n, np.concatenate([u[keep], v[keep]]), np.concatenate([v[keep], u[keep]]), seed)


def star(n, fan_in, seed):
    src = np.arange(1, fan_in + 1)
    return _batch(n, src, np.zeros_like(src), seed)


def small_ppi(num_graphs, seed):
    b = syn.ppi_batch(num_graphs, seed, n_lo=40, n_hi=60, num_tasks=8)
    return {k: b[k] for k in ("x", "edge_index", "edge_attr")}


BATCHES = {
    "ppi": lambda: small_ppi(3, 5),
    "no edges": lambda: _batch(150, np.zeros(0, dtype=np.int64), np.zeros(0, dtype=np.int64), 6),
    "hub 300 in-degree + isolated": lambda: star(340, 300, 7),
    "one direction only": lambda: syn.one_direction_only(small_ppi(3, 8), 8),
    "N=2": lambda: _batch(2, np.array([0, 1]), np.array([1, 0]), 9),
    "N=129": lambda: random_graph(129, 10),
    "PPI-sized (8 graphs, 400-600 nodes)": lambda: {k: v for k, v in syn.ppi_batch(8, 11, num_tasks=8).items()
                                                     if k in ("x", "edge_index", "edge_attr")},
}


# ---------------------------------------------------------------------------------------------------------------------------
# the harness
# ---------------------------------------------------------------------------------------------------------------------------
def layout(t, L, D, P):
    """(parameter names in pointer-table order, flat-buffer offsets) from ops.BioEncoderPlan on a bio.GNN holding P (L >= 2); for
    L = 1 (refused by the module, accepted by the C ABI) layer 0 of the two-layer table with pgnn_bio_encoder_grad_offsets."""
    m = bio.GNN(max(L, 2), D, gnn_type=t)
    if L >= 2:
        m.load_state_dict({k: v for k, v in P.items()})
    plan = ops.BioEncoderPlan(m, t)
    key = {id(p): k for k, p in m.named_parameters()}
    names = [key[id(p)] for p in plan.params]
    if L >= 2:
        return names, plan.offsets
    names = [k for k in names if not k.startswith("gnns.1.")]
    off = (ctypes.c_int64 * (len(names) + 1))()
    assert lib.pgnn_bio_encoder_num_params(CODE[t], 1) == len(names)
    assert lib.pgnn_bio_encoder_grad_offsets(CODE[t], 1, D, off) == OK
    off = list(off)
    assert [off[i + 1] - off[i] for i in range(len(names))] == [P[k].numel() for k in names]
    return names, off


def bn_key(l, s):
    return f"gnns.{l}.mlp.1.{s}"


class Encoder:
    """Poisoned device buffers for a (type, L, D, batch) case and the two C calls on them."""

    def __init__(self, t, L, D, b, P, nbt=True, ld_out=None, ldg=None, ws_short=0):
        self.t, self.L, self.D, self.P = t, L, D, P
        self.names, self.off = layout(t, L, D, P)
        self.total = self.off[-1]
        self.params = [filled(P[k].reshape(P[k].shape[0], -1)) for k in self.names]
        self.x = b["x"].reshape(-1).contiguous().to(DEV)
        self.ei, self.ea = b["edge_index"].contiguous().to(DEV), b["edge_attr"].contiguous().to(DEV)
        self.N, self.E = self.x.shape[0], self.ei.shape[1]
        self.gin = t == "gin"
        C = 2 * D
        self.rm = [filled(P[bn_key(l, "running_mean")].view(1, C), fill=SENT) for l in range(L)] if self.gin else []
        self.rv = [filled(P[bn_key(l, "running_var")].view(1, C), fill=SENT) for l in range(L)] if self.gin else []
        self.nbt = [filled(torch.full((1, 1), NBT0, dtype=torch.int64), fill=ISENT) for _ in range(L)] if self.gin and nbt else []
        self.ld_out = D if ld_out is None else ld_out
        self.ldg = D if ldg is None else ldg
        self.wsb = lib.pgnn_bio_encoder_workspace_bytes(CODE[t], self.N, self.E, L, D)
        assert self.wsb > 0
        self.ws = torch.full((self.wsb,), 255, dtype=torch.uint8, device=DEV)
        self.wsb -= ws_short
        self.out = Region(self.N, D, self.ld_out, SENT)
        self.ptrs = (ctypes.c_void_p * len(self.params))(*[r.ptr() for r in self.params])
        arr = ctypes.c_void_p * L
        self.rm_p = arr(*[r.ptr() for r in self.rm]) if self.gin else None   # the conv types have no BatchNorm: NULL tables
        self.rv_p = arr(*[r.ptr() for r in self.rv]) if self.gin else None
        self.nbt_p = arr(*[r.ptr() for r in self.nbt]) if self.nbt else None

    def forward(self, training, p=0.0, seed=0, precision=TF32X3):
        P = ops._p
        return lib.pgnn_bio_encoder_forward(CODE[self.t], self.ptrs, self.rm_p, self.rv_p, self.nbt_p, P(self.x), P(self.ei), P(self.ea),
                                            self.N, self.E, self.L, self.D, int(training), MOMENTUM, EPS, p, seed, precision,
                                            self.out.ptr(), self.ld_out, P(self.ws), self.wsb, ctypes.c_void_p(ops._st()))

    def backward(self, g, p=0.0, seed=0, precision=TF32X3):
        self.g = filled(g, ld=self.ldg)
        flat = torch.full((self.total + SLACK_FLOATS,), SENT, device=DEV)
        rc = lib.pgnn_bio_encoder_backward(CODE[self.t], self.ptrs, self.g.ptr(), self.ldg, ops._p(self.x), ops._p(self.ea), self.N,
                                           self.E, self.L, self.D, p, seed, precision, flat.data_ptr(), ops._p(self.ws), self.wsb,
                                           ctypes.c_void_p(ops._st()))
        return rc, flat

    def grads(self, flat):
        f = flat.cpu()
        return [(k, f[self.off[i]:self.off[i + 1]].view(self.P[k].shape)) for i, k in enumerate(self.names)]

    def stats(self):
        s = {}
        for l in range(self.L if self.gin else 0):
            s[bn_key(l, "running_mean")] = self.rm[l].view.cpu().view(-1)
            s[bn_key(l, "running_var")] = self.rv[l].view.cpu().view(-1)
        return s

    def guards_intact(self):
        return all(r.outside_intact() for r in self.rm + self.rv + self.nbt + [self.out])


def check_stats(mine, ref, rows, precision=TF32X3):
    """encoder_oracle.check_stats on GIN's inner BatchNorms.  On the tensor-core path the floor is TC_STATS_FLOOR: the batch mean of
    Linear(2D, 2D) over summed neighbour rows cancels most of its elements' magnitude, so the 3xTF32 GEMM's per-element rounding,
    which the fp32 oracle's does not share, shows in it undiluted (the layer-by-layer path computes the same statistics from the
    same GEMM)."""
    ok = True
    for k, v in mine.items():
        r = []
        good = EO.check_stats(k, v, ref.stats[F32][k], ref.stats[F64][k], r)
        if not good and precision == TF32X3 and r[-1]["err"] <= TC_STATS_FLOOR:
            r[-1].update(ok=True, tol=TC_STATS_FLOOR, via="3xTF32 statistics floor %g" % TC_STATS_FLOOR)
            good = True
        rows += r
        ok &= good
    return ok


def run_case(t, L, D, b, rows, *, training=True, p=0.0, precision=TF32X3, ld_out=None, ldg=None, nbt=True, side=True, param_seed=3,
             label=""):
    N = b["x"].shape[0]
    P = O.make_params("bio", t, L, D, seed=param_seed, randomize_bn=True)
    seed = 0x5EED0000 + L * 1000 + D
    masks = DO.layer_masks(seed, L, N, D, p) if training and p > 0 else None
    g = probe((N, D), 11)
    ref = Ref(P, b, t, L, training, g if training else None, masks, p)
    enc = Encoder(t, L, D, b, P, nbt=nbt, ld_out=ld_out, ldg=ldg)
    case = dict(type=t, L=L, D=D, N=N, E=enc.E, training=training, p=p, precision=precision, ld_out=enc.ld_out, ldg=enc.ldg,
                nbt=nbt, side_stream=side, case=label)
    mine = []
    if not side:
        assert lib.pgnn_profile_enable(1) == OK  # per-kernel timing mode: the backward runs without its side stream
    try:
        assert enc.forward(training, p, seed, precision) == OK, case
        if training:
            rc, flat = enc.backward(g, p, seed, precision)
            assert rc == OK, case
        torch.cuda.synchronize()
    finally:
        if not side:
            buf = ctypes.create_string_buffer(1 << 16)
            lib.pgnn_profile_read(buf, len(buf))
            lib.pgnn_profile_enable(0)
    ok = EO.check_output("node_rep", enc.out.view.cpu(), ref, mine, north_star=L < DEEP)
    assert enc.guards_intact(), case
    if training:
        f = flat.cpu()
        assert not bool((f[:enc.total] == SENT).any()), ("gradient element not written", case)
        assert bool((f[enc.total:] == SENT).all()), ("write past the flat buffer", case)
        ok &= EO.check_grads(enc.grads(flat), ref, mine, noise_floor=TWO_ROW_NOISE if N == 2 else 0.0)
        ok &= check_stats(enc.stats(), ref, mine, precision)
        assert all(int(r.view.item()) == NBT0 + 1 for r in enc.nbt), case
    else:
        for k, v in enc.stats().items():
            assert torch.equal(v, P[k]), (k, case)
        assert all(int(r.view.item()) == NBT0 for r in enc.nbt), case
    for r in mine:
        r.update(case)
    rows += mine
    return ok


def report(name, rows, **extra):
    write_report("bio_encoder_" + name, rows, extra=dict(card(), **extra))
    bad = [r for r in rows if not r["ok"]]
    allowance = [r for r in rows if r.get("via", "max") not in ("max", "exact zero")]
    if allowance:
        print("ReLU-boundary allowance used:", [(r["case"], r["type"], r["L"], r["D"], r["name"], r["via"]) for r in allowance])
    assert not bad, bad[:8]


# ---------------------------------------------------------------------------------------------------------------------------
# width x depth (training, p = 0, tf32x3)
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("t", TYPES)
def test_width_and_depth(t):
    """D = 100 is not a multiple of the GEMM tile (64 / 128 columns)."""
    b = small_ppi(2, 21)
    rows, ok = [], True
    cases = [(D, L) for D in (4, 36, 100, 300) for L in (1, 2, 3)] + [(36, DEEP)]
    for D, L in cases:
        ok &= run_case(t, L, D, b, rows, label=f"D={D} L={L}")
    report("width_depth_" + t, rows, cases=len(cases))
    assert ok


@pytest.mark.parametrize("t", TYPES)
def test_batch_shapes(t):
    rows, ok = [], True
    for name, make in BATCHES.items():
        b = make()
        for precision in (FP32, TF32X3):
            ok &= run_case(t, 3, 36, b, rows, precision=precision, label=name)
    report("batch_shapes_" + t, rows)
    assert ok


def _modes(D):
    return [dict(label="train p=0, ld_out=D+4, ldg=D+3", ld_out=D + 4, ldg=D + 3),
            dict(label="train p=0.3, ld_out=D+1, ldg=D+4, num_batches_tracked NULL", p=0.3, ld_out=D + 1, ldg=D + 4, nbt=False),
            dict(label="train p=1", p=1.0),
            dict(label="train p=0.3, side stream off", p=0.3, side=False),
            dict(label="train p=0, side stream off, ld_out=D+1, ldg=D+3", side=False, ld_out=D + 1, ldg=D + 3),
            dict(label="eval, ld_out=D+1", training=False, ld_out=D + 1),
            dict(label="eval, num_batches_tracked NULL", training=False, nbt=False)]


@pytest.mark.parametrize("D,L", [(300, 5), (36, 2)])
@pytest.mark.parametrize("t", TYPES)
def test_modes(t, D, L):
    b = small_ppi(3, 22)
    rows, ok = [], True
    for m in _modes(D):
        m = dict(m)
        label = m.pop("label")
        for precision in (FP32, TF32X3):
            ok &= run_case(t, L, D, b, rows, precision=precision, label=label, **m)
    report(f"modes_{t}_D{D}_L{L}", rows)
    assert ok


@pytest.mark.parametrize("precision", [FP32, TF32X3])
@pytest.mark.parametrize("t", TYPES)
def test_state_across_calls(t, precision):
    """Two training steps on one workspace (running statistics after both, num_batches_tracked + 2), then two backwards from the
    second forward's workspace, both within the bound."""
    L, D = 3, 36
    b = small_ppi(3, 23)
    N = b["x"].shape[0]
    P = O.make_params("bio", t, L, D, seed=5, randomize_bn=True)
    g = probe((N, D), 12)
    ref = Ref(P, b, t, L, True, g, steps=2)
    enc = Encoder(t, L, D, b, P)
    rows = []
    for _ in range(2):
        assert enc.forward(True, precision=precision) == OK
        rc, flat = enc.backward(g, precision=precision)
        assert rc == OK
    rc, flat2 = enc.backward(g, precision=precision)
    assert rc == OK
    torch.cuda.synchronize()
    ok = check_stats(enc.stats(), ref, rows, precision)
    assert all(int(r.view.item()) == NBT0 + 2 for r in enc.nbt)
    ok &= EO.check_output("node_rep", enc.out.view.cpu(), ref, rows)
    for f in (flat, flat2):
        assert not bool((f[:enc.total] == SENT).any()) and bool((f[enc.total:] == SENT).all())
        ok &= EO.check_grads(enc.grads(f), ref, rows)
    assert enc.guards_intact()
    for r in rows:
        r.update(dict(type=t, L=L, D=D, precision=precision, case="two steps, two backwards"))
    report(f"state_{t}_p{precision}", rows)
    assert ok


@pytest.mark.parametrize("t", TYPES)
def test_empty_batch(t):
    L, D = 3, 36
    b = _batch(0, np.zeros(0, dtype=np.int64), np.zeros(0, dtype=np.int64), 1)
    P = O.make_params("bio", t, L, D, seed=6, randomize_bn=True)
    enc = Encoder(t, L, D, b, P)
    assert enc.forward(True) == OK
    rc, flat = enc.backward(torch.zeros(0, D))
    assert rc == OK
    torch.cuda.synchronize()
    assert enc.guards_intact() and bool((enc.out.buf == SENT).all())
    for k, v in enc.stats().items():
        assert torch.equal(v, P[k]), k
    assert all(int(r.view.item()) == NBT0 for r in enc.nbt)
    f = flat.cpu()
    assert bool((f[:enc.total] == 0).all()) and bool((f[enc.total:] == SENT).all())


@pytest.mark.parametrize("t", TYPES)
def test_workspace_one_byte_short(t):
    L, D = 2, 36
    b = small_ppi(1, 24)
    P = O.make_params("bio", t, L, D, seed=7, randomize_bn=True)
    enc = Encoder(t, L, D, b, P, ws_short=1)
    assert enc.forward(True) == EWORKSPACE
    rc, flat = enc.backward(probe((enc.N, D), 1))
    assert rc == EWORKSPACE
    torch.cuda.synchronize()
    assert bool((enc.out.buf == SENT).all()) and bool((flat == SENT).all())
    for k, v in enc.stats().items():
        assert torch.equal(v, P[k]), k


@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("t,D", [("gin", 30), ("gcn", 30), ("graphsage", 30), ("gat", 30), ("gat", 324)])
def test_refused_shapes(t, D, fused):
    """emb_dim not a multiple of 4, and GAT wider than the attention kernels' 320: refused on both paths, BatchNorm state kept."""
    P = O.make_params("bio", t, 2, D, seed=10, randomize_bn=True)
    m = bio.GNN(2, D, JK="last", gnn_type=t)
    m.load_state_dict(P)
    m.fused = fused
    m.to(DEV).train()
    assert (m._fused_plan() is not None) == fused
    before = {k: v.clone() for k, v in m.state_dict().items() if "mlp.1." in k}
    b = small_ppi(1, 27)
    with pytest.raises(cabi.PgnnError):
        m(b["x"].to(DEV), b["edge_index"].to(DEV), b["edge_attr"].to(DEV))
    torch.cuda.synchronize()
    after = m.state_dict()
    for k, v in before.items():
        assert torch.equal(v, after[k]), k


# ---------------------------------------------------------------------------------------------------------------------------
# module level
# ---------------------------------------------------------------------------------------------------------------------------
def _module(t, P, fused, drop_ratio=0.0, L=5, D=300):
    m = bio.GNN(L, D, JK="last", drop_ratio=drop_ratio, gnn_type=t)
    m.load_state_dict(P)
    m.fused = fused
    return m.to(DEV).train()


@pytest.mark.parametrize("t", TYPES)
def test_fused_and_layerwise_paths_agree(t):
    """bio.GNN's whole-encoder path against its layer-by-layer composition (fused = False), in training with dropout 0.3 under one
    torch.manual_seed: the same kernels and the same masks, so outputs, gradients and BatchNorm state agree to rounding.  Then a
    second backward through the fused graph is refused, and eval mode agrees too."""
    b = {k: v.to(DEV) for k, v in syn.one_direction_only(small_ppi(6, 100), 5).items()}
    P = O.make_params("bio", t, 5, 300, seed=21)
    R = probe((b["x"].shape[0], 300), 5).to(DEV)
    res = []
    for fused in (True, False):
        m = _module(t, P, fused, drop_ratio=0.3)
        assert (m._fused_plan() is not None) == fused
        torch.manual_seed(1234)
        out = m(b["x"], b["edge_index"], b["edge_attr"])
        loss = (out * R).sum()
        loss.backward(retain_graph=fused)
        res.append((out.detach(), {k: p.grad for k, p in m.named_parameters()}, m.state_dict()))
        if fused:
            with pytest.raises(ops.PgnnError):
                loss.backward()
    assert float((res[0][0] == 0).float().mean()) > 0.2  # dropout is live
    assert torch.allclose(res[0][0], res[1][0], atol=2e-5, rtol=1e-5)
    gmax = max(float(g.abs().max()) for g in res[1][1].values())
    for k, g in res[1][1].items():
        scale = max(float(g.abs().max()), 1e-3 * gmax)
        assert float((res[0][1][k] - g).abs().max()) <= 2e-4 * scale + 3e-6 * gmax, k
    for k in res[0][2]:
        assert torch.allclose(res[0][2][k].float(), res[1][2][k].float(), atol=1e-5, rtol=1e-5), k
    with torch.no_grad():
        e = [_module(t, P, fused).eval()(b["x"], b["edge_index"], b["edge_attr"]) for fused in (True, False)]
    assert torch.allclose(e[0], e[1], atol=2e-5, rtol=1e-5)


class _CountingLib:
    """ops.lib stand-in that records the name of every library function looked up through it."""

    def __init__(self, real):
        self.real, self.calls = real, []

    def __getattr__(self, name):
        self.calls.append(name)
        return getattr(self.real, name)


@pytest.mark.parametrize("t", TYPES)
def test_one_library_call_per_pass(t):
    """The fused forward and backward each make exactly one enqueuing library call; only size queries come on top."""
    b = {k: v.to(DEV) for k, v in small_ppi(3, 31).items()}
    m = _module(t, O.make_params("bio", t, 5, 300, seed=22), True, drop_ratio=0.1)
    assert m._fused_plan() is not None
    out = m(b["x"], b["edge_index"], b["edge_attr"])  # the plan and its workspace size exist
    out.sum().backward()
    for p in m.parameters():
        p.grad = None
    real = ops.lib
    counting = _CountingLib(real)
    ops.lib = counting
    try:
        out = m(b["x"], b["edge_index"], b["edge_attr"])
        fwd, counting.calls = counting.calls, []
        out.sum().backward()
        bwd = counting.calls
    finally:
        ops.lib = real
    torch.cuda.synchronize()
    enq = lambda calls: [c for c in calls if not c.endswith("_workspace_bytes")]
    assert enq(fwd) == ["pgnn_bio_encoder_forward"], fwd
    assert enq(bwd) == ["pgnn_bio_encoder_backward"], bwd
    assert all(p.grad is not None for p in m.parameters())


# ---------------------------------------------------------------------------------------------------------------------------
# data parallel: the encoder's flat gradient buffer under GradAllReducer's peer-memory exchange
# ---------------------------------------------------------------------------------------------------------------------------
def _dist_worker(rank, world, port, out, t):
    sys.path.insert(0, ROOT)
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    syn_ = importlib.import_module("pretrain-gnns_b200.synthetic")
    bio_ = importlib.import_module("pretrain-gnns_b200.bio.model")
    pdist = importlib.import_module("pretrain-gnns_b200.dist")
    dev = torch.device("cuda", rank)
    torch.manual_seed(0)
    gnn = bio_.GNN(3, 300, gnn_type=t).to(dev).train()
    head = torch.nn.Linear(300, 7).to(dev)
    params = list(gnn.parameters()) + list(head.parameters())
    red = pdist.GradAllReducer(params, flat_sources=[pdist.encoder_flat_source(gnn)], backend="p2p")
    res = {"steps": []}
    for step in range(3):
        b = syn_.ppi_batch(2, 100 * step + rank, n_lo=60, n_hi=90, num_tasks=8)
        for p in params:
            p.grad = None
        head(gnn(*(b[k].to(dev) for k in ("x", "edge_index", "edge_attr")))).square().mean().backward()
        want = [p.grad.clone() for p in params]
        for g in want:
            dist.all_reduce(g)
            g.div_(world)
        flat = gnn._fused_plan().last_flat_grad
        red.all_reduce_mean()
        torch.cuda.synchronize()
        res["steps"].append({"want": [g.cpu() for g in want], "got": [p.grad.detach().cpu().clone() for p in params],
                             "encoder_wrote_region": flat.data_ptr() in [r.data_ptr() for r in red.regions]})
    red.close()
    torch.save(res, os.path.join(out, f"r{rank}.pt"))
    dist.destroy_process_group()


@pytest.mark.parametrize("t", ["gin", "gat"])
def test_p2p_allreduce_bio_flat_buffer(tmp_path, t):
    """Two ranks: the bio encoder's backward writes into the all-reduce's peer-memory region (no packing copy), and the reduced
    gradients are NCCL's mean of the two ranks' local gradients, identical on both ranks."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    world, port = 2, 29400 + os.getpid() % 2000 + (t == "gat")
    mp.spawn(_dist_worker, args=(world, port, str(tmp_path), t), nprocs=world, join=True)
    r = [torch.load(os.path.join(tmp_path, f"r{k}.pt")) for k in range(world)]
    for s0, s1 in zip(r[0]["steps"], r[1]["steps"]):
        assert s0["encoder_wrote_region"] and s1["encoder_wrote_region"]
        for w, g0, g1 in zip(s0["want"], s0["got"], s1["got"]):
            assert torch.equal(g0, g1)
            assert torch.allclose(g0, w, rtol=1e-6, atol=1e-9)
