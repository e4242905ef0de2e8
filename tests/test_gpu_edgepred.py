"""GPU: edge-prediction pre-training on the device.

* pgnn_negative_edges against the oracle bit for bit: chem B = 256 and bio B = 64 / 256 batches, the corner graphs of
  tests/test_edgepred_host.py collated into one batch, and graphs too large for the shared-memory bitmap (n = 3 000).  Outputs sit
  inside sentinel-filled allocations that must stay intact; a second call repeats bit for bit; an endpoint outside its graph is
  ignored and flagged.
* ops.edge_pair_bce (forward and backward kernels) against an fp64 restatement, P and Q from 0 (a NaN loss) to the ~1.3 M pairs of
  a bio B = 256 step, with a strided pos_index, u = v pairs and node rows inside NaN-filled allocations; loss and d node_rep repeat
  bit for bit.
* EdgePredStep / BioEdgePredStep (four gnn_types, B = 64; GIN at B = 256) against the oracle bodies of tests/edgepred_oracle.py at
  the bars of tests/golden_util.py, and the pipeline collate -> data.negative_edges -> step on both stores."""
import importlib

import numpy as np
import pytest
import torch

import edgepred_oracle as EO
from device_buffers import DEV, SENT, filled
from golden_util import OUT_REL, SLACK, gradient_check, output_check, write_report
from oracle import gnn_oracle as O
from oracle import steps_oracle as S
from test_edgepred_host import _corner_batch
from test_gpu_bio_objectives import _dev

pytestmark = pytest.mark.gpu
syn = importlib.import_module("pretrain-gnns_b200.synthetic")
ts = importlib.import_module("pretrain-gnns_b200.train_steps")
ops = importlib.import_module("pretrain-gnns_b200.ops")
data = importlib.import_module("pretrain-gnns_b200.data")
cabi = importlib.import_module("pretrain-gnns_b200._cabi")
GATHER_ERR = ops.DEVICE_ERROR_BITS[16]
PAD = 8


# ---------------------------------------------------------------------------------------------------------------------
# the transform
# ---------------------------------------------------------------------------------------------------------------------
def call_negative_edges(edge_index, node_off, edge_off, seed):
    """One pgnn_negative_edges call with both outputs inside sentinel-filled allocations.
    -> (negative_edge_index [2, M] numpy, negative_edge_off numpy, sentinels intact, flagged)"""
    import ctypes
    lib = cabi.lib
    eoff = np.ascontiguousarray(edge_off, dtype=np.int64)
    B = len(eoff) - 1
    cap = int(lib.pgnn_negative_edges_capacity(eoff.ctypes.data_as(ctypes.c_void_p), B))
    E = int(edge_index.shape[1])
    ei = torch.as_tensor(np.ascontiguousarray(edge_index, dtype=np.int64)).to(DEV)
    no, eo = torch.as_tensor(np.asarray(node_off, np.int64)).to(DEV), torch.from_numpy(eoff).to(DEV)
    wsb = int(lib.pgnn_negative_edges_workspace_bytes(B, E, cap))
    ws = torch.full((wsb // 8 + 1,), -1, dtype=torch.int64, device=DEV)
    out = torch.full((2 * cap + 2 * PAD,), int(SENT), dtype=torch.int64, device=DEV)
    off = torch.full((B + 1 + 2 * PAD,), int(SENT), dtype=torch.int64, device=DEV)
    ops.device_errors(clear=True)
    cabi.check(lib.pgnn_negative_edges(ei.data_ptr(), E, no.data_ptr(), eo.data_ptr(), B, int(seed) & ((1 << 63) - 1), cap, ws.data_ptr(), wsb,
                                       out[PAD:].data_ptr(), off[PAD:].data_ptr(), torch.cuda.current_stream().cuda_stream), "negative_edges")
    flagged = GATHER_ERR in ops.device_errors(clear=True)
    o = off.cpu().numpy()
    M = int(o[PAD + B])
    res = out.cpu().numpy()
    intact = (o[:PAD] == int(SENT)).all() and (o[PAD + B + 1:] == int(SENT)).all() and (res[:PAD] == int(SENT)).all() \
        and (res[PAD + 2 * M:] == int(SENT)).all()
    return res[PAD:PAD + 2 * M].reshape(2, M), o[PAD:PAD + B + 1], bool(intact), flagged


def _check_transform(ei, node_off, edge_off, seed, ref=None):
    if ref is None:
        ref, ref_off = EO.negative_edges_batch(ei, node_off, edge_off, seed)
    else:
        ref_off = None
    neg, off, intact, flagged = call_negative_edges(ei, node_off, edge_off, seed)
    assert intact, "a sentinel around the outputs was overwritten"
    assert not flagged
    assert neg.shape == ref.shape and np.array_equal(neg, ref)
    if ref_off is not None:
        assert np.array_equal(off, ref_off)
    neg2, off2, _, _ = call_negative_edges(ei, node_off, edge_off, seed)
    assert np.array_equal(neg2, neg) and np.array_equal(off2, off), "not bit-for-bit repeatable"
    return neg


@pytest.mark.parametrize("seed", [0, 5, 2 ** 62 + 1])
def test_negative_edges_corner_graphs(seed):
    """One node, no edges, a complete graph, duplicate bonds, an odd one-direction graph, repeats before the quota."""
    ei, node_off, edge_off = _corner_batch()
    _check_transform(ei, node_off, edge_off, seed)


def test_negative_edges_chem_b256():
    b = syn.zinc_batch(256, 31)
    eoff = syn.edge_offsets(b)
    neg = _check_transform(b["edge_index"].numpy(), b["ptr"].numpy(), eoff, 31)
    assert neg.shape[1] == b["edge_index"].shape[1] // 2


def test_negative_edges_chem_one_direction():
    b = syn.one_direction_only(syn.zinc_batch(64, 32), 32)
    _check_transform(b["edge_index"].numpy(), b["ptr"].numpy(), syn.edge_offsets(b), 32)


@pytest.mark.parametrize("B", [64, 256])
def test_negative_edges_bio(B):
    b = syn.ppi_batch(B, 33 + B)
    ei, no, eoff = b["edge_index"].numpy(), b["ptr"].numpy(), syn.edge_offsets(b)
    # B = 64: the oracle's literal loop; B = 256: its vectorised restatement (pinned to the loop by tests/test_edgepred_host.py)
    ref = None if B == 64 else syn.negative_edge_index(ei, no, eoff, 7)
    _check_transform(ei, no, eoff, 7, ref)


def test_negative_edges_large_graphs():
    """n = 3 000 (past the shared-memory bitmap: the global-hash path), an odd one-direction large graph (no early stop), beside
    small graphs in the same batch."""
    big = syn.ppi_batch(2, 35, n_lo=3000, n_hi=3000, pairs_per_node=2)
    odd = syn.one_direction_only(syn.ppi_batch(1, 36, n_lo=2500, n_hi=2600, pairs_per_node=1), 36)
    small = syn.zinc_batch(3, 37)
    items = []
    for bb in (big, odd, small):
        for n, ei, _ in (syn.ppi_graphs(bb)[0] if bb["x"].shape[1] == 1 else [(x.shape[0], ei, ea) for x, ei, ea in syn.split_graphs(bb)]):
            items.append(dict(x=np.zeros((n, 1)), edge_index=np.asarray(ei, np.int64)))
    if items[2]["edge_index"].shape[1] % 2 == 0:
        items[2]["edge_index"] = items[2]["edge_index"][:, 1:]
    col = EO.batch_ae(items)
    node_off = np.concatenate([[0], np.cumsum([d["x"].shape[0] for d in items])]).astype(np.int64)
    edge_off = np.concatenate([[0], np.cumsum([d["edge_index"].shape[1] for d in items])]).astype(np.int64)
    neg = _check_transform(col["edge_index"], node_off, edge_off, 11)
    e2 = int(edge_off[3] - edge_off[2])
    assert e2 % 2 == 1 and int(((neg[0] >= node_off[2]) & (neg[0] < node_off[3])).sum()) > e2 // 2


def test_negative_edges_flags_out_of_range_endpoints():
    """A column whose endpoint lies outside its graph is left out of the graph's edge set (it cannot match a candidate) and flagged."""
    b = syn.zinc_batch(8, 38)
    ei, no, eoff = b["edge_index"].numpy().copy(), b["ptr"].numpy(), syn.edge_offsets(b)
    ei[1, int(eoff[2]) + 3] = int(no[-1]) + 50
    ei[0, int(eoff[5])] = int(no[1])       # a node of graph 1 inside graph 5's columns
    ref, _ = EO.negative_edges_batch(ei, no, eoff, 4)
    neg, _, intact, flagged = call_negative_edges(ei, no, eoff, 4)
    assert flagged and intact and np.array_equal(neg, ref)


# ---------------------------------------------------------------------------------------------------------------------
# the head
# ---------------------------------------------------------------------------------------------------------------------
def head_reference(x, pos_index, neg_index, pos_dev, neg_dev):
    """fp64 on the device: scores, the loss on the kernel's own scores, and d node_rep from those scores.
    -> (pos64, neg64, loss_on_device_scores, gx64, gx_abs (sum of |g x|, for the rounding bound), degree)"""
    x64 = x.to(DEV).double()
    N = x64.shape[0]

    def dots(idx):
        idx = idx.to(DEV)
        return torch.cat([(x64[idx[0, i:i + 200000]] * x64[idx[1, i:i + 200000]]).sum(1) for i in range(0, idx.shape[1], 200000)]) \
            if idx.shape[1] else torch.zeros(0, dtype=torch.float64, device=DEV)

    p64, q64 = dots(pos_index), dots(neg_index)
    loss = EO.edgepred_head(pos_dev.double(), neg_dev.double())
    P, Q = pos_dev.shape[0], neg_dev.shape[0]
    gp = (torch.sigmoid(pos_dev.double()) - 1.0) / max(P, 1)
    gq = torch.sigmoid(neg_dev.double()) / max(Q, 1)
    gx, ga = torch.zeros_like(x64), torch.zeros_like(x64)
    deg = torch.zeros(N, dtype=torch.float64, device=DEV)
    for g, idx in ((gp, pos_index.to(DEV)), (gq, neg_index.to(DEV))):
        for i in range(0, idx.shape[1], 200000):
            u, v, gg = idx[0, i:i + 200000], idx[1, i:i + 200000], g[i:i + 200000, None]
            gx.index_add_(0, u, gg * x64[v]).index_add_(0, v, gg * x64[u])
            ga.index_add_(0, u, (gg * x64[v]).abs()).index_add_(0, v, (gg * x64[u]).abs())
            deg.index_add_(0, u, torch.ones_like(gg[:, 0])).index_add_(0, v, torch.ones_like(gg[:, 0]))
    return p64, q64, float(loss), gx, ga, deg


def call_head(x, pos_index, neg_index, ld):
    xr = filled(x, ld)
    xv = xr.view.requires_grad_(True)
    ops.device_errors(clear=True)
    loss, pos, neg = ops.edge_pair_bce(xv, pos_index.to(DEV), neg_index.to(DEV))
    loss.backward()
    gx = xv.grad.clone()
    xv.grad = None
    return float(loss), pos, neg, gx


def _pairs(N, m, g, self_pairs=0):
    idx = torch.randint(0, max(N, 1), (2, m), generator=g)
    if self_pairs and m:
        k = torch.randint(0, m, (self_pairs,), generator=g)
        idx[1, k] = idx[0, k]
    return idx


@pytest.mark.parametrize("N,P,Q", [(16, 0, 0), (16, 0, 5), (16, 7, 0), (16, 1, 1), (64, 33, 65), (300, 1000, 3000), (5000, 40000, 41000),
                                   (128000, 640000, 640000)])
def test_edge_pair_bce_vs_fp64(N, P, Q):
    g = torch.Generator().manual_seed(N + 7 * P + Q)
    x = torch.randn(N, 300, generator=g) * 0.3
    full = _pairs(N, 2 * P, g, self_pairs=P // 10 + (1 if P else 0))
    pos_index = full.to(DEV)[:, ::2]              # strided view: column stride 2, read in place
    neg_index = _pairs(N, Q, g, self_pairs=Q // 10 + (1 if Q else 0))
    loss, pos, neg, gx = call_head(x, pos_index, neg_index, 304)
    p64, q64, lref, gref, gabs, deg = head_reference(x, pos_index, neg_index, pos, neg)
    eps = 2.0 ** -24
    for mine, ref, idx in ((pos, p64, pos_index), (neg, q64, neg_index)):
        if ref.numel():
            x64 = x.to(DEV).double()
            bound = 300 * eps * torch.cat([(x64[idx[0, i:i + 200000]] * x64[idx[1, i:i + 200000]]).abs().sum(1)
                                           for i in range(0, idx.shape[1], 200000)])
            assert bool(((mine.double() - ref).abs() <= bound + 1e-30).all())
    if P == 0 or Q == 0:
        assert np.isnan(loss)
    else:
        assert abs(loss - lref) <= 1e-12 * abs(lref), (loss, lref)
    bound = (deg[:, None] + 4) * 2 * eps * gabs + 1e-30
    assert bool(((gx.double() - gref).abs() <= bound).all()), float(((gx.double() - gref).abs() - bound).max())
    assert not ops.device_errors()
    loss2, pos2, neg2, gx2 = call_head(x, pos_index, neg_index, 304)
    assert (loss2 == loss or (np.isnan(loss) and np.isnan(loss2))) and torch.equal(gx2, gx) and torch.equal(pos2, pos) and torch.equal(neg2, neg)


def test_edge_pair_bce_flags_out_of_range_pairs():
    g = torch.Generator().manual_seed(1)
    x = torch.randn(20, 300, generator=g)
    pos, neg = _pairs(20, 10, g), _pairs(20, 10, g)
    neg[1, 3] = 20
    xd = x.to(DEV)
    ops.device_errors(clear=True)
    _, _, q = ops.edge_pair_bce(xd, pos.to(DEV), neg.to(DEV))
    errs = ops.device_errors(clear=True)
    assert GATHER_ERR in errs and float(q[3]) == 0.0
    with pytest.raises(cabi.PgnnError):
        ops.edge_pair_bce(xd, pos.to(DEV).int(), neg.to(DEV))


# ---------------------------------------------------------------------------------------------------------------------
# the steps against the oracle
# ---------------------------------------------------------------------------------------------------------------------
def _aux(step, d):
    rep = step.model(d["x"], d["edge_index"], d["edge_attr"])
    _, pos, neg = ops.edge_pair_bce(rep, d["edge_index"][:, ::2], d["negative_edge_index"])
    return dict(rep=rep, pos=pos, neg=neg)


def _head(a):
    return EO.edgepred_head(a["pos"], a["neg"])


def score_check(name, mine, ref32, ref64, rows):
    """The scores are dot products of 300-wide unnormalised encoder rows.  Where such a product cancels, its error is set by the
    rows' magnitude, not by its own, and no fp32 summation order meets an element-wise relative bound there (the oracle's own fp32
    scores miss its fp64 ones by as much as the device's do).  So they are held to output_check's scale-relative bound: the largest
    error against fp64 over the tensor's largest magnitude <= max(OUT_REL, SLACK x the oracle's own fp32 error).  The encoder
    output `rep` they are made of keeps output_check's element-wise bound as well."""
    mine, ref32, ref64 = (torch.as_tensor(t).detach().cpu().double() for t in (mine, ref32, ref64))
    scale = max(float(ref64.abs().max()), 1e-30)
    e64, eref = float((mine - ref64).abs().max()) / scale, float((ref32 - ref64).abs().max()) / scale
    rows.append(dict(kind="out", name=name, err=e64, err_ref32=eref, bound="scale-relative", ok=e64 <= max(OUT_REL, SLACK * eref)))
    return rows[-1]["ok"]


def compare_step(name, step, loss_fn, P, b):
    """tests/test_gpu_bio_objectives._compare for these steps: `rep` by output_check, the scores by score_check, the loss within
    max(2e-6, 3 x the oracle's own fp32 error) of fp64 or -- DESIGN.md section 4's rule -- equal to the oracle's fp64 head on the
    step's own scores to 1e-9 when those scores pass their bound, every gradient by gradient_check."""
    torch.set_num_threads(min(16, torch.get_num_threads()))
    l32, a32, g32, l64, a64, g64, near = S.grads_fp32_fp64(loss_fn, P, b)
    step.load_state(P)
    d = _dev(b)
    loss = step(d)
    grads = [(k, p.grad) for k, p in step.named_parameters()]
    assert all(g is not None for _, g in grads)
    with torch.no_grad():
        aux = _aux(step, d)
    rows = []
    ok = output_check("rep", aux["rep"], a32["rep"], a64["rep"], rows)
    for k in ("pos", "neg"):
        ok &= score_check(k, aux[k], a32[k], a64[k], rows)
    lerr = abs(float(loss) - float(l64)) / max(abs(float(l64)), 1e-30)
    lref = abs(float(l32) - float(l64)) / max(abs(float(l64)), 1e-30)
    lhead = float(_head({k: v.detach().cpu().double() for k, v in aux.items()}))
    lok, via = lerr <= max(2e-6, 3 * lref), "oracle"
    if not lok and ok and abs(float(loss) - lhead) <= 1e-9 * abs(lhead):
        lok, via = True, "the oracle head on the step's scores (err %.2e)" % (abs(float(loss) - lhead) / abs(lhead))
    rows.append(dict(kind="loss", name="loss", err=lerr, err_ref32=lref, ok=lok, via=via))
    ok &= lok
    ok &= gradient_check(grads, g32, g64, near, rows)
    write_report(name, rows, dict(near_zero_preactivations=near, loss=float(loss), loss_oracle64=float(l64), loss_head_on_scores=lhead))
    assert not ops.device_errors(), "index range flags raised on a valid batch"
    assert ok, [r for r in rows if not r["ok"]][:8]


@pytest.mark.parametrize("domain", ["chem", "bio"])
@pytest.mark.parametrize("t", ["gin", "gcn", "graphsage", "gat"])
def test_edgepred_step_b64_vs_oracle(domain, t):
    step = (ts.EdgePredStep if domain == "chem" else ts.BioEdgePredStep)(DEV, t, batch_size=64)
    b = step.make_batches(0, 1)[0]
    compare_step("edgepred_%s_b64_%s" % (domain, t), step, lambda L, bb: EO.edgepred_loss(L, bb, domain, t), EO.make_params(domain, 15, t), b)


@pytest.mark.parametrize("domain", ["chem", "bio"])
def test_edgepred_gin_step_b256(domain):
    """The scripts' default batch (B = 256): loss and every gradient finite, the loss within the bar of the fp64 oracle, or equal to
    the oracle's fp64 head on the step's own scores when those pass score_check (compare_step's rule; the oracle's forward only)."""
    step = (ts.EdgePredStep if domain == "chem" else ts.BioEdgePredStep)(DEV)
    b = step.make_batches(0, 1)[0]
    P = EO.make_params(domain, 16)
    step.load_state(P)
    d = _dev(b)
    loss = float(step(d))
    for k, p in step.named_parameters():
        assert p.grad is not None and bool(torch.isfinite(p.grad).all()), k
    assert not ops.device_errors()
    with torch.no_grad():
        a = _aux(step, d)
        lhead = float(_head({k: v.cpu().double() for k, v in a.items()}))
        torch.set_num_threads(min(16, torch.get_num_threads()))
        (l32, a32), (l64, a64) = (EO.edgepred_loss(O.leaf_params(P, dt), b, domain) for dt in (torch.float32, torch.float64))
        l32, l64 = float(l32), float(l64)
    rows = []
    scores_ok = all([score_check(k, a[k], a32[k], a64[k], rows) for k in ("pos", "neg")])
    lerr, lref = abs(loss - l64) / abs(l64), abs(l32 - l64) / abs(l64)
    ok = lerr <= max(2e-6, 3 * lref) or (scores_ok and abs(loss - lhead) <= 1e-9 * abs(lhead))
    write_report("edgepred_%s_b256_gin" % domain, rows + [dict(kind="loss", name="loss", err=lerr, err_ref32=lref, ok=ok)],
                 dict(pairs=int(b["edge_index"].shape[1] // 2 + b["negative_edge_index"].shape[1]), loss=loss, loss_oracle64=l64, loss_head=lhead))
    assert np.isfinite(loss) and ok, (loss, l64, l32, lhead)


# ---------------------------------------------------------------------------------------------------------------------
# the device pipeline
# ---------------------------------------------------------------------------------------------------------------------
def test_device_pipeline_chem():
    """MoleculeStore.collate -> data.negative_edges -> EdgePredStep gives exactly the batch and the loss of edgepred_batch."""
    B, seed = 48, 8123
    ref = syn.edgepred_batch(B, seed)
    graphs = syn.split_graphs(ref)
    store = data.MoleculeStore(np.cumsum([0] + [g[0].shape[0] for g in graphs]), np.cumsum([0] + [g[1].shape[1] for g in graphs]),
                               np.concatenate([g[0] for g in graphs]), np.concatenate([g[1] for g in graphs], 1),
                               np.concatenate([g[2] for g in graphs]), device=DEV)
    ids = np.arange(B)
    o = store.collate(ids)
    data.negative_edges(o, o.edge_off.cpu().numpy(), seed)
    for k in ts.EdgePredStep.KEYS:
        assert torch.equal(getattr(o, k).cpu(), ref[k]), k
    assert int(o.negative_edge_off[-1]) == ref["negative_edge_index"].shape[1]
    step = ts.EdgePredStep(DEV, batch_size=B)
    step.load_state(EO.make_params("chem", 17))
    l_dev = float(step({k: getattr(o, k) for k in ts.EdgePredStep.KEYS}))
    l_syn = float(step(_dev({k: ref[k] for k in ts.EdgePredStep.KEYS})))
    assert l_dev == l_syn and np.isfinite(l_dev)
    assert not ops.device_errors()


def test_device_pipeline_bio():
    """BioGraphStore.collate -> data.negative_edges -> BioEdgePredStep gives exactly the batch and the loss of bio_edgepred_batch."""
    B, seed = 12, 9077
    kw = dict(n_lo=60, n_hi=90, pairs_per_node=3, num_tasks=4)
    ref = syn.bio_edgepred_batch(B, seed, **kw)
    graphs, _ = syn.ppi_graphs(ref)
    store = data.BioGraphStore([g[0] for g in graphs], [g[1] for g in graphs], [g[2] for g in graphs], [0] * B, device=DEV)
    o = store.collate(np.arange(B))
    data.negative_edges(o, o.edge_off.cpu().numpy(), seed)
    for k in ts.BioEdgePredStep.KEYS:
        assert torch.equal(getattr(o, k).cpu(), ref[k]), k
    step = ts.BioEdgePredStep(DEV, batch_size=B)
    step.load_state(EO.make_params("bio", 18))
    l_dev = float(step({k: getattr(o, k) for k in ts.BioEdgePredStep.KEYS}))
    l_syn = float(step(_dev({k: ref[k] for k in ts.BioEdgePredStep.KEYS})))
    assert l_dev == l_syn and np.isfinite(l_dev)
    assert not ops.device_errors()
