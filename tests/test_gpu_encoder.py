"""GPU: the chem whole-encoder entry points (pgnn_chem_encoder_forward / _backward, csrc/encoder.cu) directly against fp64.

Every case calls the two entry points through ctypes on poisoned buffers (tests/device_buffers.py):
  * each parameter in its own NaN-padded allocation, the workspace filled with NaN bytes before the forward and untouched between
    forward and backward, g_node_rep a NaN-padded region with row stride ldg: an over-read or a read of something the forward
    did not write shows up as NaN;
  * node_rep a sentinel region with row stride ld_out, the flat gradient buffer sentinel-filled with slack past `total` (no
    sentinel may survive inside [0, total), every one after it must), the running statistics in sentinel-guarded regions;
and compares with tests/encoder_oracle.py's fp64 / fp32 oracle runs at its bounds (output_check, gradient_check, running
statistics, num_batches_tracked exact).  tests/test_encoder_host.py shows the bounds reject plausible encoder bugs.

Sweeps: width x depth (L = 1 is a single layer that is also the last; L = 2 has one layer of each side-stream parity; L = 17 takes
GIN's dgrad without the transposed weights), batch shapes (no edges, an in-degree hub with isolated atoms, one-direction edges,
N past a 128-row tile and a 1024-row split-K chain), modes (eval, dropout p in {0, 0.3, 1}, strides, num_batches_tracked NULL,
the side stream off), state across calls, and refused shapes.  Each case group's measured errors are written
by golden_util.write_report (one report per group, named encoder_*)."""
import ctypes
import importlib

import numpy as np
import pytest
import torch

import dropout_oracle as DO
import encoder_oracle as EO
from device_buffers import DEV, SENT, Region, card, filled
from golden_util import probe, write_report
from oracle import gnn_oracle as O

pytestmark = pytest.mark.gpu
syn = importlib.import_module("pretrain-gnns_b200.synthetic")
chem = importlib.import_module("pretrain-gnns_b200.chem.model")
ops = importlib.import_module("pretrain-gnns_b200.ops")
cabi = importlib.import_module("pretrain-gnns_b200._cabi")
lib = cabi.lib
TYPES = ("gin", "gcn", "graphsage", "gat")
CODE = {"gin": 0, "gcn": 1, "graphsage": 2, "gat": 3}
OK, EWORKSPACE = 0, -3
FP32, TF32X3 = 0, 1
ISENT = -7777          # int64 sentinel of num_batches_tracked's region
NBT0 = 7               # num_batches_tracked before a call
SLACK_FLOATS = 61      # sentinel floats past the flat gradient buffer's `total`
MOMENTUM, EPS = 0.1, 1e-5
# From this depth on only output_check's scale-relative half applies to node_rep: 3xTF32's rounding, compounded through 17
# BatchNorm layers, reaches 2.2e-5 of the output's scale (2x the fp32 oracle's 1.0e-5), over the element-wise 1e-4 on its
# largest elements; at 65 layers the fp32 oracle itself is 1.9e-2 of scale from fp64.
DEEP = 17
# With two rows a training BatchNorm column's invstd is 2 / |x0 - x1|: a column whose two rows nearly coincide amplifies every
# rounding error before it.  GIN at N = 2 measures 3.7e-5 of scale for the fp32 oracle and 1.1e-4 for 3xTF32 (3.1x, over SLACK);
# the gradients of the N = 2 case are held to at least this floor.
TWO_ROW_NOISE = 1e-3


# ---------------------------------------------------------------------------------------------------------------------------
# batches
# ---------------------------------------------------------------------------------------------------------------------------
def _batch(x, src, dst, seed):
    """x [N, 2] codes, directed edges src -> dst (edge_index row 0 = the aggregation target dst), random bond codes."""
    rng = np.random.default_rng(seed)
    E = len(src)
    ea = np.stack([rng.integers(0, 4, size=E), rng.integers(0, 3, size=E)], axis=1) if E else np.zeros((0, 2))
    return dict(x=torch.as_tensor(x, dtype=torch.int64), edge_index=torch.as_tensor(np.stack([dst, src]).reshape(2, E), dtype=torch.int64),
                edge_attr=torch.as_tensor(ea, dtype=torch.int64).reshape(E, 2))


def _codes(n, seed):
    """Atom codes over the whole vocabulary (0..119, 119 the mask token) and every chirality tag."""
    rng = np.random.default_rng(seed + 1)
    return np.stack([rng.integers(0, 120, size=n), rng.integers(0, 3, size=n)], axis=1)


def random_graph(n, seed, deg=2):
    """n atoms, ~deg * n / 2 random bonds, both directions."""
    rng = np.random.default_rng(seed)
    m = deg * n // 2
    u, v = rng.integers(0, n, size=m), rng.integers(0, n, size=m)
    keep = u != v
    u, v = u[keep], v[keep]
    return _batch(_codes(n, seed), np.concatenate([u, v]), np.concatenate([v, u]), seed)


def star(n, fan_in, seed):
    """Atom 0 receives an edge from each of atoms 1..fan_in; atoms past fan_in are isolated."""
    src = np.arange(1, fan_in + 1)
    return _batch(_codes(n, seed), src, np.zeros_like(src), seed)


def no_edges(n, seed):
    return _batch(_codes(n, seed), np.zeros(0, dtype=np.int64), np.zeros(0, dtype=np.int64), seed)


BATCHES = {
    "zinc": lambda: syn.zinc_batch(8, 5),
    "no edges": lambda: no_edges(150, 6),
    "hub 300 in-degree + isolated": lambda: star(340, 300, 7),
    "one direction only": lambda: syn.one_direction_only(syn.zinc_batch(8, 8), 8),
    "N=2": lambda: _batch(_codes(2, 9), np.array([0, 1]), np.array([1, 0]), 9),
    "N=129": lambda: random_graph(129, 10),
    "N=1025": lambda: random_graph(1025, 11),
    "hub N=4100": lambda: star(4100, 4099, 12),
}


# ---------------------------------------------------------------------------------------------------------------------------
# the harness
# ---------------------------------------------------------------------------------------------------------------------------
def layout(t, L, D, P):
    """(parameter names in pointer-table order, flat-buffer offsets): ops.ChemEncoderPlan on a chem.GNN holding P for L >= 2.
    The module refuses L = 1, which the C ABI accepts: its table is layer 0 of the L = 2 plan's, its offsets those of
    pgnn_chem_*_grad_offsets."""
    m = chem.GNN(max(L, 2), D, gnn_type=t)
    if L >= 2:
        m.load_state_dict(P)
    plan = ops.ChemEncoderPlan(m, t)
    key = {id(p): k for k, p in m.named_parameters()}
    names = [key[id(p)] for p in plan.params]
    if L >= 2:
        return names, plan.offsets
    names = [k for k in names if not k.startswith(("gnns.1.", "batch_norms.1."))]
    off = (ctypes.c_int64 * (len(names) + 1))()
    if CODE[t]:
        assert lib.pgnn_chem_conv_num_params(CODE[t], 1) == len(names)
        assert lib.pgnn_chem_conv_grad_offsets(CODE[t], 1, D, off) == OK
    else:
        assert lib.pgnn_chem_gin_num_params(1) == len(names)
        assert lib.pgnn_chem_gin_grad_offsets(1, D, off) == OK
    off = list(off)
    assert [off[i + 1] - off[i] for i in range(len(names))] == [P[k].numel() for k in names]
    return names, off


def workspace_bytes(t, N, E, L, D):
    if CODE[t]:
        return lib.pgnn_chem_conv_workspace_bytes(CODE[t], N, E, L, D)
    return lib.pgnn_chem_gin_workspace_bytes(N, E, L, D)


class Encoder:
    """One set of poisoned device buffers for a (type, L, D, batch) case, and the two C calls on them."""

    def __init__(self, t, L, D, b, P, nbt=True, ld_out=None, ldg=None, ws_short=0):
        self.t, self.L, self.D, self.P = t, L, D, P
        self.names, self.off = layout(t, L, D, P)
        self.total = self.off[-1]
        self.params = [filled(P[k].reshape(P[k].shape[0], -1)) for k in self.names]
        self.x, self.ei, self.ea = (b[k].contiguous().to(DEV) for k in ("x", "edge_index", "edge_attr"))
        self.N, self.E = b["x"].shape[0], b["edge_index"].shape[1]
        self.rm = [filled(P[f"batch_norms.{l}.running_mean"].view(1, D), fill=SENT) for l in range(L)]
        self.rv = [filled(P[f"batch_norms.{l}.running_var"].view(1, D), fill=SENT) for l in range(L)]
        self.nbt = [filled(torch.full((1, 1), NBT0, dtype=torch.int64), fill=ISENT) for _ in range(L)] if nbt else None
        self.ld_out = D if ld_out is None else ld_out
        self.ldg = D if ldg is None else ldg
        self.wsb = workspace_bytes(t, self.N, self.E, L, D)
        assert self.wsb > 0
        self.ws = torch.full((self.wsb,), 255, dtype=torch.uint8, device=DEV)  # 0xFFFFFFFF: NaN
        self.wsb -= ws_short
        self.out = Region(self.N, D, self.ld_out, SENT)
        self.ptrs = (ctypes.c_void_p * len(self.params))(*[r.ptr() for r in self.params])
        arr = ctypes.c_void_p * L
        self.rm_p, self.rv_p = arr(*[r.ptr() for r in self.rm]), arr(*[r.ptr() for r in self.rv])
        self.nbt_p = arr(*[r.ptr() for r in self.nbt]) if nbt else None

    def forward(self, training, p=0.0, seed=0, precision=TF32X3):
        P = ops._p
        return lib.pgnn_chem_encoder_forward(CODE[self.t], self.ptrs, self.rm_p, self.rv_p, self.nbt_p, P(self.x), P(self.ei), P(self.ea),
                                             self.N, self.E, self.L, self.D, int(training), MOMENTUM, EPS, p, seed, precision,
                                             self.out.ptr(), self.ld_out, P(self.ws), self.wsb, ctypes.c_void_p(ops._st()))

    def backward(self, g, p=0.0, seed=0, precision=TF32X3):
        """-> (return code, flat sentinel-filled gradient buffer with slack)"""
        self.g = filled(g, ld=self.ldg)
        flat = torch.full((self.total + SLACK_FLOATS,), SENT, device=DEV)
        rc = lib.pgnn_chem_encoder_backward(CODE[self.t], self.ptrs, self.g.ptr(), self.ldg, ops._p(self.x), ops._p(self.ea), self.N,
                                            self.E, self.L, self.D, p, seed, precision, flat.data_ptr(), ops._p(self.ws), self.wsb,
                                            ctypes.c_void_p(ops._st()))
        return rc, flat

    def grads(self, flat):
        f = flat.cpu()
        return [(k, f[self.off[i]:self.off[i + 1]].view(self.P[k].shape)) for i, k in enumerate(self.names)]

    def stats(self):
        s = {}
        for l in range(self.L):
            s[f"batch_norms.{l}.running_mean"] = self.rm[l].view.cpu().view(-1)
            s[f"batch_norms.{l}.running_var"] = self.rv[l].view.cpu().view(-1)
        return s

    def guards_intact(self):
        regions = self.rm + self.rv + (self.nbt or []) + [self.out]
        return all(r.outside_intact() for r in regions)


def run_case(t, L, D, b, rows, *, training=True, p=0.0, precision=TF32X3, ld_out=None, ldg=None, nbt=True, side=True, param_seed=3,
             label=""):
    """One forward (+ backward in training mode) against the oracle; appends the check rows, returns whether all passed."""
    N = b["x"].shape[0]
    P = O.make_params("chem", t, L, D, seed=param_seed, randomize_bn=True)
    seed = 0x5EED0000 + L * 1000 + D
    masks = DO.layer_masks(seed, L, N, D, p) if training and p > 0 else None
    g = probe((N, D), 11)
    ref = EO.Ref(P, b, t, L, training, g if training else None, masks, p)
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
        ok &= EO.check_all_stats(enc.stats(), ref, L, mine)
        if nbt:
            assert all(int(r.view.item()) == NBT0 + 1 for r in enc.nbt), case
    else:
        for k, v in enc.stats().items():
            assert torch.equal(v, P[k]), (k, case)
        if nbt:
            assert all(int(r.view.item()) == NBT0 for r in enc.nbt), case
    for r in mine:
        r.update(case)
    rows += mine
    return ok


def report(name, rows, **extra):
    write_report("encoder_" + name, rows, extra=dict(card(), **extra))
    bad = [r for r in rows if not r["ok"]]
    allowance = [r for r in rows if r.get("via", "max") not in ("max", "exact zero")]
    if allowance:
        print("ReLU-boundary allowance used:", [(r["case"], r["type"], r["L"], r["D"], r["name"], r["via"]) for r in allowance])
    assert not bad, bad[:8]


# ---------------------------------------------------------------------------------------------------------------------------
# width x depth (training, p = 0, tf32x3)
# ---------------------------------------------------------------------------------------------------------------------------
WIDTHS = {"gin": (4, 36, 128, 300, 512), "gcn": (4, 36, 128, 300, 512), "graphsage": (4, 36, 128, 300, 512),
          "gat": (4, 36, 128, 300, 320)}


@pytest.mark.parametrize("t", TYPES)
def test_width_and_depth(t):
    b = syn.zinc_batch(4, 21)
    rows, ok = [], True
    cases = [(D, L) for D in WIDTHS[t] for L in (1, 2, 3)] + [(36, 17)]
    for D, L in cases:
        ok &= run_case(t, L, D, b, rows, label=f"D={D} L={L}")
    report("width_depth_" + t, rows, cases=len(cases))
    assert ok


# ---------------------------------------------------------------------------------------------------------------------------
# batch shapes (D = 36, L = 3, both precisions)
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("t", TYPES)
def test_batch_shapes(t):
    rows, ok = [], True
    for name, make in BATCHES.items():
        b = make()
        for precision in (FP32, TF32X3):
            ok &= run_case(t, 3, 36, b, rows, precision=precision, label=name)
    report("batch_shapes_" + t, rows)
    assert ok


# ---------------------------------------------------------------------------------------------------------------------------
# modes (D = 300, L = 5 and D = 36, L = 2; both precisions)
# ---------------------------------------------------------------------------------------------------------------------------
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
    b = syn.zinc_batch(8, 22)
    rows, ok = [], True
    for m in _modes(D):
        m = dict(m)
        label = m.pop("label")
        for precision in (FP32, TF32X3):
            ok &= run_case(t, L, D, b, rows, precision=precision, label=label, **m)
    report(f"modes_{t}_D{D}_L{L}", rows)
    assert ok


# ---------------------------------------------------------------------------------------------------------------------------
# state across calls
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", [FP32, TF32X3])
@pytest.mark.parametrize("t", TYPES)
def test_state_across_calls(t, precision):
    """Two training steps on one workspace: the running statistics after both, num_batches_tracked + 2; then two backwards
    from the second forward's workspace, both within the bound (the backward leaves what the forward saved intact)."""
    L, D = 3, 36
    b = syn.zinc_batch(8, 23)
    N = b["x"].shape[0]
    P = O.make_params("chem", t, L, D, seed=5, randomize_bn=True)
    g = probe((N, D), 12)
    ref = EO.Ref(P, b, t, L, True, g, steps=2)
    enc = Encoder(t, L, D, b, P)
    rows = []
    for _ in range(2):
        assert enc.forward(True, precision=precision) == OK
        rc, flat = enc.backward(g, precision=precision)
        assert rc == OK
    rc, flat2 = enc.backward(g, precision=precision)
    assert rc == OK
    torch.cuda.synchronize()
    ok = EO.check_all_stats(enc.stats(), ref, L, rows)
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
    """N = 0: the forward returns OK and writes nothing (running statistics, num_batches_tracked, node_rep's region); the
    backward zeroes exactly `total` floats."""
    L, D = 3, 36
    b = no_edges(0, 1)
    P = O.make_params("chem", t, L, D, seed=6, randomize_bn=True)
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
    b = syn.zinc_batch(2, 24)
    P = O.make_params("chem", t, L, D, seed=7, randomize_bn=True)
    enc = Encoder(t, L, D, b, P, ws_short=1)
    assert enc.forward(True) == EWORKSPACE
    rc, flat = enc.backward(probe((enc.N, D), 1))
    assert rc == EWORKSPACE
    torch.cuda.synchronize()
    assert bool((enc.out.buf == SENT).all()) and bool((flat == SENT).all())
    for k, v in enc.stats().items():
        assert torch.equal(v, P[k]), k


# ---------------------------------------------------------------------------------------------------------------------------
# defects at the module level
# ---------------------------------------------------------------------------------------------------------------------------
def _module(t, L, D, P):
    m = chem.GNN(L, D, JK="last", gnn_type=t)
    m.load_state_dict(P)
    m.fused = True
    return m.to(DEV).train()


@pytest.mark.parametrize("order", ["fp32 forward, tf32x3 backward", "tf32x3 forward, fp32 backward"])
@pytest.mark.parametrize("t", TYPES)
def test_backward_uses_the_forward_precision(t, order):
    """The backward reads what the forward saved, and what the forward saves depends on its precision (the tensor path's one-hot
    atom-code rows).  A precision switch between the two must not change the gradients: the op keeps the forward's.  The
    workspace block is NaN-filled just before the forward, so a read of rows the forward did not write gives NaN."""
    L, D = 3, 36
    b = syn.zinc_batch(8, 25)
    N, E = b["x"].shape[0], b["edge_index"].shape[1]
    P = O.make_params("chem", t, L, D, seed=8, randomize_bn=True)
    g = probe((N, D), 13)
    ref = EO.Ref(P, b, t, L, True, g)
    m = _module(t, L, D, P)
    d = {k: b[k].to(DEV) for k in ("x", "edge_index", "edge_attr")}
    first, second = ("fp32", "tf32x3") if order.startswith("fp32") else ("tf32x3", "fp32")
    before = ops.get_precision()
    try:
        ops.set_precision(first)
        plan = m._fused_plan()
        assert plan is not None
        torch.cuda.synchronize()
        stale = torch.full((plan.workspace_bytes(N, E),), 255, dtype=torch.uint8, device=DEV)
        del stale
        out = m(d["x"], d["edge_index"], d["edge_attr"])
        ops.set_precision(second)
        (out * g.to(DEV)).sum().backward()
        torch.cuda.synchronize()
    finally:
        ops.set_precision(before)
    rows = []
    ok = EO.check_output("node_rep", out.detach().cpu(), ref, rows)
    ok &= EO.check_grads([(k, p.grad) for k, p in m.named_parameters()], ref, rows)
    ok_emb = all(r["ok"] for r in rows if r["name"].startswith("x_embedding"))
    for r in rows:
        r.update(dict(type=t, L=L, D=D, case=order))
    report(f"precision_switch_{t}_{first}", rows)
    assert ok_emb and ok


@pytest.mark.parametrize("precision", ["fp32", "tf32x3"])
@pytest.mark.parametrize("t", TYPES)
def test_65_layer_training_step(t, precision):
    """A depth the forward accepts trains through the backward too.  On the FFMA path the gradients pass gradient_check.  A
    65-layer stack is chaotic in fp32 (GIN's fp32 oracle is up to 0.2 of scale from fp64 on some gradients) and the 3xTF32 GEMMs
    round differently from the oracle's, so on that path the step must complete with finite gradients and node_rep within the
    scale-relative bound."""
    L, D = 65, 8
    b = syn.zinc_batch(4, 26)
    N = b["x"].shape[0]
    P = O.make_params("chem", t, L, D, seed=9, randomize_bn=True)
    g = probe((N, D), 14)
    ref = EO.Ref(P, b, t, L, True, g)
    d = {k: b[k].to(DEV) for k in ("x", "edge_index", "edge_attr")}
    before = ops.get_precision()
    try:
        ops.set_precision(precision)
        m = _module(t, L, D, P)
        out = m(d["x"], d["edge_index"], d["edge_attr"])
        (out * g.to(DEV)).sum().backward()
        torch.cuda.synchronize()
    finally:
        ops.set_precision(before)
    rows = []
    ok = EO.check_output("node_rep", out.detach().cpu(), ref, rows, north_star=False)
    grads = [(k, p.grad.cpu()) for k, p in m.named_parameters()]
    assert all(bool(torch.isfinite(v).all()) for _, v in grads)
    if precision == "fp32":
        ok &= EO.check_grads(grads, ref, rows)
    for r in rows:
        r.update(dict(type=t, L=L, D=D, precision=precision, case="65 layers through the module"))
    report(f"depth65_{t}_{precision}", rows)
    assert ok


# ---------------------------------------------------------------------------------------------------------------------------
# refused shapes
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("t,D", [("gin", 30), ("gcn", 30), ("graphsage", 30), ("gat", 30), ("gat", 324)])
def test_refused_shapes(t, D, fused):
    """emb_dim not a multiple of 4, and GAT wider than the attention kernels' 320: refused, with the BatchNorm buffers as they
    were, on the whole-encoder and on the layer-by-layer path."""
    P = O.make_params("chem", t, 2, D, seed=10, randomize_bn=True)
    m = chem.GNN(2, D, JK="last", gnn_type=t)
    m.load_state_dict(P)
    m.fused = fused
    m.to(DEV).train()
    assert (m._fused_plan() is not None) == fused
    before = {k: v.clone() for k, v in m.state_dict().items() if k.startswith("batch_norms")}
    b = syn.zinc_batch(2, 27)
    with pytest.raises(cabi.PgnnError):
        m(b["x"].to(DEV), b["edge_index"].to(DEV), b["edge_attr"].to(DEV))
    torch.cuda.synchronize()
    after = m.state_dict()
    for k, v in before.items():
        assert torch.equal(v, after[k]), k
