"""GPU: each C-ABI operator against the oracle / plain torch on the same seeded inputs.

Integer work (bucketing) must be bit-exact; fp32 work is held to the north_star tolerance of 1e-4
(abs + rel), and the SUM aggregation additionally to bit-exactness against a sequential CPU
index_add_ in edge order (same summation order by construction)."""
import importlib

import numpy as np
import pytest
import torch

from oracle import gnn_oracle as O
from oracle import graph_prep_oracle as GP

pytestmark = pytest.mark.gpu
ops = importlib.import_module("pretrain-gnns_b200.ops")
syn = importlib.import_module("pretrain-gnns_b200.synthetic")
DEV = "cuda:0"
ATOL = RTOL = 1e-4


def close(a, b, atol=ATOL, rtol=RTOL):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    assert a.shape == b.shape, (a.shape, b.shape)
    err = (a - b).abs()
    assert bool((err <= atol + rtol * b.abs()).all()), "max err %.3e (ref max %.3e)" % (err.max().item(), b.abs().max().item())


def rnd(*shape, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(*shape, generator=g) * scale


@pytest.mark.parametrize("graphs,seed", [(1, 0), (32, 1), (256, 2)])
def test_graph_prep_bit_exact(graphs, seed):
    b = syn.zinc_batch(graphs, seed)
    n = b["x"].shape[0]
    # shuffle the edge order so stability is actually exercised
    perm = torch.from_numpy(np.random.default_rng(seed).permutation(b["edge_index"].shape[1]))
    ei = b["edge_index"][:, perm].contiguous()
    g = ops.Graph(ei.to(DEV), n)
    (rt, nt, et), (rs, ns, es) = GP.graph_prep(ei.numpy(), n)
    for mine, ref in ((g.rowptr_t, rt), (g.nbr_t, nt), (g.eid_t, et), (g.rowptr_s, rs), (g.nbr_s, ns), (g.eid_s, es)):
        assert np.array_equal(mine.cpu().numpy(), ref)


def test_graph_prep_edge_cases():
    # no edges at all; isolated nodes; one giant bucket
    g = ops.Graph(torch.zeros(2, 0, dtype=torch.int64, device=DEV), 5)
    assert g.rowptr_t.cpu().tolist() == [0] * 6
    ei = torch.stack([torch.zeros(3000, dtype=torch.int64), torch.arange(3000) % 7])
    g = ops.Graph(ei.to(DEV), 7)
    (rt, nt, et), (rs, ns, es) = GP.graph_prep(ei.numpy(), 7)
    assert np.array_equal(g.nbr_t.cpu().numpy(), nt) and np.array_equal(g.eid_s.cpu().numpy(), es)
    assert np.array_equal(g.rowptr_s.cpu().numpy(), rs)


def test_segments_bucket_large_scan():
    # > 1024 buckets exercises the multi-tile scan carry
    seg = torch.from_numpy(np.sort(np.random.default_rng(3).integers(0, 5000, size=20000)))
    s = ops.Segments(seg.to(DEV), 5000)
    rp, _, order = GP.segments(seg.numpy(), 5000)
    assert np.array_equal(s.ptr.cpu().numpy(), rp) and np.array_equal(s.order.cpu().numpy()[:20000], order)


@pytest.mark.parametrize("mode", [ops.AGG_SUM, ops.AGG_MEAN, ops.AGG_GCN])
def test_chem_aggregate_fwd_bwd(mode):
    b = syn.zinc_batch(16, 5)
    n, C = b["x"].shape[0], 300
    x = rnd(n, C, seed=1).requires_grad_(True)
    T1, T2 = rnd(6, C, seed=2).requires_grad_(True), rnd(3, C, seed=3).requires_grad_(True)
    ei = O.with_self_loops(b["edge_index"], n)
    rows = O.chem_edge_rows({"edge_embedding1.weight": T1, "edge_embedding2.weight": T2}, "", b["edge_attr"], n)
    msg = x[ei[1]] + rows
    if mode == ops.AGG_GCN:
        msg = O.gcn_norm(ei, n, torch.float32).view(-1, 1) * msg
    ref = O.reduce_onto_target(msg, ei[0], n, mean=(mode == ops.AGG_MEAN))
    R = rnd(n, C, seed=4)
    (ref * R).sum().backward()

    xd = x.detach().to(DEV).requires_grad_(True)
    T1d, T2d = T1.detach().to(DEV).requires_grad_(True), T2.detach().to(DEV).requires_grad_(True)
    g = ops.Graph(b["edge_index"].to(DEV), n)
    S = g.summary("chem", mode, b["edge_attr"].to(DEV))
    out = ops.aggregate(xd, torch.cat([T1d, T2d]), g, S, mode)
    (out * R.to(DEV)).sum().backward()
    close(out, ref, 1e-5, 1e-5)
    close(xd.grad, x.grad, 1e-5, 1e-5)
    close(T1d.grad, T1.grad, 1e-3, 1e-4)  # sums over ~1000 rows
    close(T2d.grad, T2.grad, 1e-3, 1e-4)


def test_sum_aggregate_of_rows_is_bit_exact():
    """Same summation order as CPU index_add_ (edge order, self-loop last) => identical bits for the x part."""
    b = syn.zinc_batch(64, 9)
    n, C = b["x"].shape[0], 300
    x = rnd(n, C, seed=1)
    ei = O.with_self_loops(b["edge_index"], n)
    ref = O.reduce_onto_target(x[ei[1]], ei[0], n)
    g = ops.Graph(b["edge_index"].to(DEV), n)
    zero_T = torch.zeros(9, C, device=DEV)
    S = g.summary("chem", ops.AGG_SUM, b["edge_attr"].to(DEV))
    out = ops.aggregate(x.to(DEV), zero_T, g, S, ops.AGG_SUM)
    assert torch.equal(out.cpu(), ref)


def test_bio_aggregate_concat():
    b = syn.ppi_batch(2, 3, n_lo=50, n_hi=80, num_tasks=4)
    n, C = b["x"].shape[0], 300
    x = rnd(n, C, seed=1).requires_grad_(True)
    W, bias = rnd(C, 9, seed=2, scale=0.3).requires_grad_(True), rnd(C, seed=3, scale=0.3).requires_grad_(True)
    ei = O.with_self_loops(b["edge_index"], n)
    rows = O.bio_edge_rows({"edge_encoder.weight": W, "edge_encoder.bias": bias}, "", b["edge_attr"], n)
    ref = O.reduce_onto_target(torch.cat([x[ei[1]], rows], 1), ei[0], n)
    R = rnd(n, 2 * C, seed=4)
    (ref * R).sum().backward()
    xd, Wd, bd = (t.detach().to(DEV).requires_grad_(True) for t in (x, W, bias))
    g = ops.Graph(b["edge_index"].to(DEV), n)
    S = g.summary("bio", ops.AGG_SUM, b["edge_attr"].to(DEV))
    out = ops.aggregate(xd, torch.cat([Wd.t(), bd[None]]), g, S, ops.AGG_SUM, concat=True)
    (out * R.to(DEV)).sum().backward()
    close(out, ref, 1e-4, 1e-5)
    close(xd.grad, x.grad, 1e-5, 1e-5)
    close(Wd.grad, W.grad, 2e-3, 1e-4)
    close(bd.grad, bias.grad, 2e-3, 1e-4)


@pytest.mark.parametrize("M,N,K", [(1, 7, 5), (130, 600, 300), (777, 300, 600), (64, 119, 300), (1000, 1, 300)])
def test_linear_fwd_bwd(M, N, K):
    x, w, b = rnd(M, K, seed=1).requires_grad_(True), rnd(N, K, seed=2, scale=0.1).requires_grad_(True), rnd(N, seed=3).requires_grad_(True)
    ref = torch.nn.functional.linear(x, w, b)
    R = rnd(M, N, seed=4)
    (ref * R).sum().backward()
    xd, wd, bd = (t.detach().to(DEV).requires_grad_(True) for t in (x, w, b))
    out = ops.linear(xd, wd, bd)
    (out * R.to(DEV)).sum().backward()
    close(out, ref, 1e-4, 1e-5)
    close(xd.grad, x.grad, 1e-4, 1e-5)
    close(wd.grad, w.grad, 2e-4 * max(1.0, M ** 0.5 / 8), 1e-4)
    close(bd.grad, b.grad, 2e-4 * max(1.0, M ** 0.5 / 8), 1e-4)


def test_mlp2_matches_torch():
    M, D = 500, 300
    a = rnd(M, D, seed=1).requires_grad_(True)
    w1, b1 = rnd(2 * D, D, seed=2, scale=0.06).requires_grad_(True), rnd(2 * D, seed=3, scale=0.1).requires_grad_(True)
    w2, b2 = rnd(D, 2 * D, seed=4, scale=0.04).requires_grad_(True), rnd(D, seed=5, scale=0.1).requires_grad_(True)
    F = torch.nn.functional
    ref = F.linear(F.relu(F.linear(a, w1, b1)), w2, b2)
    R = rnd(M, D, seed=6)
    (ref * R).sum().backward()
    d = [t.detach().to(DEV).requires_grad_(True) for t in (a, w1, b1, w2, b2)]
    out = ops.mlp2(*d)
    (out * R.to(DEV)).sum().backward()
    close(out, ref, 1e-4, 1e-5)
    for mine, r in zip(d, (a, w1, b1, w2, b2)):
        close(mine.grad, r.grad, 5e-4, 1e-4)


@pytest.mark.parametrize("relu", [False, True])
@pytest.mark.parametrize("M,C", [(3, 300), (5888, 300), (1000, 600)])
def test_batch_norm_train(M, C, relu):
    bn = torch.nn.BatchNorm1d(C)
    with torch.no_grad():
        bn.weight.copy_(0.5 + torch.rand(C)); bn.bias.copy_(torch.rand(C) - 0.5)
        bn.running_mean.copy_(torch.rand(C)); bn.running_var.copy_(0.5 + torch.rand(C))
    import copy
    bd = copy.deepcopy(bn).to(DEV)
    x = (rnd(M, C, seed=1) * 2 + 3).requires_grad_(True)  # mean >> 0 stresses the variance computation
    pre = bn(x)
    y = torch.relu(pre) if relu else pre
    R = rnd(M, C, seed=2)
    (y * R).sum().backward()
    xd = x.detach().to(DEV).requires_grad_(True)
    yd = ops.batch_norm(xd, bd, relu)
    (yd * R.to(DEV)).sum().backward()
    close(yd, y, 1e-4, 1e-4)
    if relu:
        # an element whose pre-activation is within rounding of zero may take the other ReLU branch on the GPU (the batch statistics
        # are accumulated in a different order): its own gradient then differs by R, not by rounding.  Compare everything else.
        edge = pre.detach().abs() <= 2e-6
        assert int(edge.sum()) <= 8
        g_dev = torch.where(edge, x.grad, xd.grad.cpu())
        close(g_dev, x.grad, 1e-4 + 4e-4 * int(edge.any()), 1e-3)
        # the parameter gradients sum R (times xhat) over the kept elements: count those edge elements as the GPU's forward took
        # them (its y > 0, which its backward's mask equals), at the same tolerances
        kept_dev, kept_cpu = yd.detach().cpu() > 0, pre.detach() > 0
        dR = torch.where(edge, R * (kept_dev.float() - kept_cpu.float()), torch.zeros_like(R))
        xhat = (x.detach() - x.detach().mean(0)) / torch.sqrt(x.detach().var(0, unbiased=False) + bn.eps)
        gw_ref, gb_ref = bn.weight.grad + (dR * xhat).sum(0), bn.bias.grad + dR.sum(0)
    else:
        close(xd.grad, x.grad, 1e-4, 1e-3)
        gw_ref, gb_ref = bn.weight.grad, bn.bias.grad
    close(bd.weight.grad, gw_ref, 1e-4 * M ** 0.5, 1e-4)
    close(bd.bias.grad, gb_ref, 1e-4 * M ** 0.5, 1e-4)
    close(bd.running_mean, bn.running_mean, 1e-5, 1e-5)
    close(bd.running_var, bn.running_var, 1e-5, 1e-5)
    assert int(bd.num_batches_tracked) == int(bn.num_batches_tracked) == 1


def test_batch_norm_eval():
    bn = torch.nn.BatchNorm1d(300).eval()
    with torch.no_grad():
        bn.running_mean.copy_(torch.rand(300)); bn.running_var.copy_(0.5 + torch.rand(300))
    import copy
    bd = copy.deepcopy(bn).to(DEV)
    x = rnd(100, 300, seed=1)
    close(ops.batch_norm(x.to(DEV), bd, True), torch.relu(bn(x)), 1e-5, 1e-5)


def test_relu_l2norm():
    x = rnd(333, 300, seed=1).requires_grad_(True)
    R = rnd(333, 300, seed=2)
    y = torch.nn.functional.normalize(torch.relu(x), p=2, dim=-1)
    (y * R).sum().backward()
    xd = x.detach().to(DEV).requires_grad_(True)
    yd = ops.l2_normalize(ops.relu(xd))
    (yd * R.to(DEV)).sum().backward()
    close(yd, y, 1e-6, 1e-5)
    close(xd.grad, x.grad, 1e-6, 1e-4)


def test_embeddings():
    b = syn.zinc_batch(32, 1)
    t1, t2 = rnd(120, 300, seed=1).requires_grad_(True), rnd(3, 300, seed=2).requires_grad_(True)
    ref = t1[b["x"][:, 0]] + t2[b["x"][:, 1]]
    R = rnd(*ref.shape, seed=3)
    (ref * R).sum().backward()
    d1, d2 = t1.detach().to(DEV).requires_grad_(True), t2.detach().to(DEV).requires_grad_(True)
    out = ops.chem_embed(b["x"].to(DEV), d1, d2)
    (out * R.to(DEV)).sum().backward()
    assert torch.equal(out.cpu(), ref.detach())
    close(d1.grad, t1.grad, 1e-4, 1e-5)
    close(d2.grad, t2.grad, 1e-3, 1e-4)
    tab = rnd(2, 300, seed=4).requires_grad_(True)
    xb = torch.ones(50, 1)
    xb[::3] = 0
    refb = tab[xb.long().view(-1)]
    (refb * R[:50]).sum().backward()
    td = tab.detach().to(DEV).requires_grad_(True)
    ob = ops.bio_embed(xb.to(DEV), td)
    (ob * R[:50].to(DEV)).sum().backward()
    assert torch.equal(ob.cpu(), refb.detach())
    close(td.grad, tab.grad, 1e-4, 1e-5)


def test_segment_mean_and_empty_segment():
    b = syn.zinc_batch(32, 1)
    n = b["x"].shape[0]
    x = rnd(n, 300, seed=1).requires_grad_(True)
    ref = O.segment_mean(x, b["batch"], 34)  # two trailing empty graphs -> zeros (count.clamp(min=1))
    R = rnd(34, 300, seed=2)
    (ref * R).sum().backward()
    xd = x.detach().to(DEV).requires_grad_(True)
    out = ops.global_mean_pool(xd, b["batch"].to(DEV), 34)
    (out * R.to(DEV)).sum().backward()
    close(out, ref, 1e-6, 1e-5)
    close(xd.grad, x.grad, 1e-6, 1e-5)
    assert float(out[32:].detach().abs().max()) == 0.0
    # size inferred like PyG does
    assert ops.global_mean_pool(xd, b["batch"].to(DEV)).shape[0] == 32


def test_row_gather_with_duplicates():
    x = rnd(100, 300, seed=1).requires_grad_(True)
    i1 = torch.tensor([5, 5, 7, 99, 0, 5]); i2 = torch.tensor([7, 5, 5, 0, 0, 1])
    ref = x[i1] + x[i2]
    R = rnd(6, 300, seed=2)
    (ref * R).sum().backward()
    xd = x.detach().to(DEV).requires_grad_(True)
    out = ops.row_gather(xd, i1.to(DEV), i2.to(DEV))
    (out * R.to(DEV)).sum().backward()
    close(out, ref, 1e-6, 1e-6)
    close(xd.grad, x.grad, 1e-5, 1e-5)
    assert ops.row_gather(xd, torch.zeros(0, dtype=torch.int64, device=DEV)).shape == (0, 300)


@pytest.mark.parametrize("B,shift", [(128, 0), (128, 1), (7, 3), (1, 1)])
def test_shifted_rowdot(B, shift):
    a, b = rnd(B, 300, seed=1).requires_grad_(True), rnd(B, 300, seed=2).requires_grad_(True)
    ref = (a * b[O.cycle_rows(B, shift)]).sum(1)
    R = rnd(B, seed=3)
    (ref * R).sum().backward()
    ad, bd = a.detach().to(DEV).requires_grad_(True), b.detach().to(DEV).requires_grad_(True)
    out = ops.shifted_rowdot(ad, bd, shift)
    (out * R.to(DEV)).sum().backward()
    close(out, ref, 1e-4, 1e-5)
    close(ad.grad, a.grad, 1e-5, 1e-5)
    close(bd.grad, b.grad, 1e-5, 1e-5)


def test_host_tensor_is_rejected():
    cabi = importlib.import_module("pretrain-gnns_b200._cabi")
    with pytest.raises(cabi.PgnnError):
        ops.linear(torch.zeros(2, 3), torch.zeros(4, 3), None)


def test_out_of_range_indices_are_flagged_not_dereferenced():
    """ADVICE r1: an out-of-range node id / atom code / bond code / label / gather index must not become a silent
    out-of-bounds access.  The kernels drop or clamp the element and raise a PGNN_DEVERR_* bit (include/pgnn_b200.h)."""
    ops.device_errors(clear=True)
    b = syn.zinc_batch(4, 3)
    n = b["x"].shape[0]
    assert ops.device_errors() == []
    ei = b["edge_index"].clone()
    ei[0, 5] = n + 1000           # target far outside the node range
    ei[1, 9] = -3
    g = ops.Graph(ei.to(DEV), n)
    errs = ops.device_errors()
    assert len(errs) == 1 and "node" in errs[0]
    assert int(g.rowptr_t[-1]) == ei.shape[1] - 2 and int(g.rowptr_s[-1]) == ei.shape[1] - 2   # both bad edges dropped from both bucketings
    kept = ei.shape[1] - 2   # entries past rowptr[-1] are never written (nor read: every consumer walks rowptr)
    assert int(g.nbr_t[:kept].max()) < n and int(g.nbr_s[:kept].max()) < n and int(g.nbr_t[:kept].min()) >= 0
    x = b["x"].clone()
    x[3, 0] = 500
    t1, t2 = torch.randn(120, 300, device=DEV), torch.randn(3, 300, device=DEV)
    out = ops.chem_embed(x.to(DEV), t1, t2)
    assert torch.isfinite(out).all() and any("atom" in e for e in ops.device_errors())
    ea = b["edge_attr"].clone()
    ea[2, 0] = 77
    g2 = ops.Graph(b["edge_index"].to(DEV), n)
    g2.summary("chem", ops.AGG_SUM, ea.to(DEV))
    assert any("bond" in e for e in ops.device_errors())
    rep = torch.randn(n, 300, device=DEV)
    rows = ops.row_gather(rep, torch.tensor([0, n + 5, 2], device=DEV))
    assert any("gather" in e for e in ops.device_errors()) and float(rows[1].abs().max()) == 0.0
    W, bias = torch.randn(119, 300, device=DEV) * 0.05, torch.zeros(119, device=DEV)
    loss, _ = ops.masked_atom_loss(rep, torch.tensor([0, 1], device=DEV), torch.tensor([5, 4000], device=DEV), W, bias)
    assert torch.isfinite(loss) and any("label" in e for e in ops.device_errors())
    with pytest.raises(ops.PgnnError):
        ops.Graph(ei.to(DEV), n)
        ops.raise_on_device_errors()
    assert ops.device_errors() == []
