"""GPU: Deep Graph Infomax pre-training on the device.

* ops.infomax_bce (summary, scores + BCE, per-graph reduction, node pass and the three GEMMs) against an fp64 torch composition of
  the script's lines: loss, pos, neg, d node_emb and d weight, at G = 1, 2 and 256 at chem size (N ~ 6 k) and G = 256 at bio size
  (N ~ 128 k); a one-node graph and an empty graph in the middle of the batch; a permuted batch vector; node rows read in place
  through a row stride inside a NaN-filled allocation, and a column-strided view (copied); an upstream gradient != 1; both
  ops.set_precision settings.  Forward and backward repeat bit for bit.  The C entry points write into NaN-filled output buffers
  (device_buffers) and must fill them exactly, leaving the surroundings intact.
* InfomaxStep / BioInfomaxStep (four gnn_types, B = 64; GIN at B = 256) against the oracle bodies of tests/infomax_oracle.py at the
  bars of tests/golden_util.py, and the store pipeline MoleculeStore / BioGraphStore.collate -> step."""
import importlib
import math

import numpy as np
import pytest
import torch

import infomax_oracle as IO
from device_buffers import DEV, NAN, Region, filled
from golden_util import gradient_check, output_check, write_report
from oracle import gnn_oracle as O
from oracle import steps_oracle as S
from test_gpu_bio_objectives import _dev
from test_gpu_edgepred import score_check

pytestmark = pytest.mark.gpu
syn = importlib.import_module("pretrain-gnns_b200.synthetic")
ts = importlib.import_module("pretrain-gnns_b200.train_steps")
ops = importlib.import_module("pretrain-gnns_b200.ops")
data = importlib.import_module("pretrain-gnns_b200.data")
cabi = importlib.import_module("pretrain-gnns_b200._cabi")
D = 300


# ---------------------------------------------------------------------------------------------------------------------
# the head
# ---------------------------------------------------------------------------------------------------------------------
def make_case(G, per_graph, seed, one_node=False, empty=False, permute=False):
    """-> (x [N, 300] CPU, batch [N] CPU int64, W [300, 300] CPU).  Rows scaled like encoder outputs (|score| up to ~10)."""
    g = torch.Generator().manual_seed(seed)
    counts = torch.randint(max(1, per_graph // 2), per_graph * 3 // 2 + 1, (G,), generator=g)
    if one_node:
        counts[min(1, G - 1)] = 1
    if empty:
        counts[G // 2] = 0
    batch = torch.repeat_interleave(torch.arange(G), counts)
    if permute:
        batch = batch[torch.randperm(batch.numel(), generator=g)]
    x = torch.randn(batch.numel(), D, generator=g) * 0.5 + 0.2
    W = (torch.rand(D, D, generator=g) * 2 - 1) / math.sqrt(D)
    return x, batch, W


def torch_head(x, batch, W, G, gscale, dtype):
    """The script's lines 62-73 on the device in `dtype` (global_mean_pool as scatter_mean with count.clamp(min=1)).
    -> (loss, pos, neg, d x, d W) for the upstream gradient gscale."""
    xx = x.to(DEV, dtype).requires_grad_(True)
    WW = W.to(DEV, dtype).requires_grad_(True)
    b = batch.to(DEV)
    tot = torch.zeros(G, D, dtype=dtype, device=DEV).index_add_(0, b, xx)
    cnt = torch.zeros(G, dtype=dtype, device=DEV).index_add_(0, b, torch.ones(b.numel(), dtype=dtype, device=DEV))
    summary = torch.sigmoid(tot / cnt.clamp(min=1)[:, None])
    h = summary @ WW
    pos = (xx * h[b]).sum(1)
    neg = (xx * h[IO.cycle_index(G, 1).to(DEV)][b]).sum(1)
    loss = IO.bce_pair(pos, neg)
    (loss * gscale).backward()
    return float(loss), pos.detach(), neg.detach(), xx.grad, WW.grad


def call_head(x, batch, W, G, gscale=1.0, ld=None, colstride=False, pass_g=True):
    if colstride:   # a column-strided view: the op copies it
        big = torch.zeros(x.shape[0], 2 * D)
        big[:, ::2] = x
        xv = big.to(DEV).requires_grad_(True)
        rows = xv[:, ::2]
    else:
        xr = filled(x, ld)
        xv = xr.view.requires_grad_(True)
        rows = xv
    Wd = W.to(DEV).requires_grad_(True)
    ops.device_errors(clear=True)
    loss, pos, neg = ops.infomax_bce(rows, batch.to(DEV), Wd, G if pass_g else None)
    assert not pos.requires_grad and not neg.requires_grad
    (loss * gscale).backward()
    gx = xv.grad[:, ::2].clone() if colstride else xv.grad.clone()
    return float(loss), pos, neg, gx, Wd.grad.clone()


def check_head(name, x, batch, W, G, gscale=1.0, **kw):
    loss, pos, neg, gx, gW = call_head(x, batch, W, G, gscale, **kw)
    l64, p64, n64, gx64, gW64 = torch_head(x, batch, W, G, gscale, torch.float64)
    l32, p32, n32, gx32, gW32 = torch_head(x, batch, W, G, gscale, torch.float32)
    rows = []
    ok = score_check("pos", pos, p32, p64, rows) & score_check("neg", neg, n32, n64, rows)
    lhead = float(IO.bce_pair(pos.double(), neg.double()))
    lerr, lref = abs(loss - l64) / abs(l64), abs(l32 - l64) / abs(l64)
    lok = abs(loss - lhead) <= 1e-12 * abs(lhead) and lerr <= max(2e-6, 3 * lref)
    rows.append(dict(kind="loss", name="loss", err=lerr, err_ref32=lref, ok=lok))
    ok &= lok
    ok &= gradient_check([("x", gx), ("W", gW)], {"x": gx32.cpu(), "W": gW32.cpu()}, {"x": gx64.cpu(), "W": gW64.cpu()}, 0, rows)
    write_report("infomax_head_" + name, rows, dict(N=int(x.shape[0]), G=G, gscale=gscale, precision=ops.get_precision()))
    assert not ops.device_errors()
    assert ok, [r for r in rows if not r["ok"]]
    again = call_head(x, batch, W, G, gscale, **kw)
    assert again[0] == loss and all(torch.equal(a, b) for a, b in zip(again[1:], (pos, neg, gx, gW))), "not bit-for-bit repeatable"


@pytest.fixture
def precision(request):
    old = ops.get_precision()
    ops.set_precision(request.param)
    yield request.param
    ops.set_precision(old)


@pytest.mark.parametrize("G,precision", [(1, "tf32x3"), (2, "tf32x3"), (256, "tf32x3"), (256, "fp32")], indirect=["precision"])
def test_infomax_bce_chem_size(G, precision):
    """Chem size, N ~ 6 k: ~23 nodes per graph at G = 256; at G = 1 and 2 the same rows in one or two graphs (G = 1 scores each
    node against its own graph on both sides).  Both ops.set_precision settings at G = 256."""
    x, batch, W = make_case(G, 23 if G == 256 else 6000 // G, 100 + G)   # N ~ 6 k: molecules, or one / two long segments
    kw = dict(ld=304) if G == 256 else {}
    if precision == "fp32":   # the FFMA weight-gradient GEMM folds its split-K partials with atomics: no bitwise repeat of dW
        loss, pos, neg, gx, gW = call_head(x, batch, W, G, **kw)
        l64, p64, n64, gx64, gW64 = torch_head(x, batch, W, G, 1.0, torch.float64)
        l32, p32, n32, gx32, gW32 = torch_head(x, batch, W, G, 1.0, torch.float32)
        rows = []
        ok = score_check("pos", pos, p32, p64, rows) & score_check("neg", neg, n32, n64, rows)
        ok &= gradient_check([("x", gx), ("W", gW)], {"x": gx32.cpu(), "W": gW32.cpu()}, {"x": gx64.cpu(), "W": gW64.cpu()}, 0, rows)
        write_report("infomax_head_chem_fp32", rows)
        assert ok and abs(loss - l64) <= 2e-6 * abs(l64), rows
        return
    check_head("chem_G%d" % G, x, batch, W, G, **kw)


def test_infomax_bce_bio_size():
    """Bio size: B = 256 ego graphs of ~500 nodes, N ~ 128 k, rows read through a 304-float stride."""
    x, batch, W = make_case(256, 500, 7)
    x = x * 0.3
    check_head("bio_G256", x, batch, W, 256, ld=304)


def test_infomax_bce_one_node_and_empty_graphs():
    """A one-node graph and an empty graph in the middle of the batch (its summary is sigmoid(0) = 0.5 and it still serves as
    the negative of the graph before it); G passed explicitly, and read back from the batch vector."""
    x, batch, W = make_case(40, 20, 11, one_node=True, empty=True)
    assert int((batch == 1).sum()) == 1 and int((batch == 20).sum()) == 0
    check_head("one_node_empty", x, batch, W, 40)
    check_head("one_node_empty_readback", x, batch, W, 40, pass_g=False)


def test_infomax_bce_permuted_batch_and_strided_rows():
    """An unsorted batch vector, and node rows given as a column-strided view."""
    x, batch, W = make_case(64, 23, 12, permute=True)
    assert not bool((batch[1:] >= batch[:-1]).all())
    check_head("permuted", x, batch, W, 64)
    check_head("colstride", x, batch, W, 64, colstride=True)


def test_infomax_bce_upstream_gradient():
    x, batch, W = make_case(32, 23, 13)
    check_head("gscale", x, batch, W, 32, gscale=-2.75)


def test_infomax_bce_rejects_bad_widths():
    x = torch.randn(10, 302, device=DEV)
    with pytest.raises(cabi.PgnnError):
        ops.infomax_bce(x, torch.zeros(10, dtype=torch.int64, device=DEV), torch.randn(302, 302, device=DEV), 1)
    with pytest.raises(cabi.PgnnError):
        ops.infomax_bce(torch.randn(10, 300, device=DEV), torch.zeros(10, dtype=torch.int64, device=DEV), torch.randn(300, 296, device=DEV), 1)


def test_infomax_bce_empty_batch_is_nan():
    loss, pos, neg = ops.infomax_bce(torch.zeros(0, D, device=DEV), torch.zeros(0, dtype=torch.int64, device=DEV), torch.randn(D, D, device=DEV))
    assert math.isnan(float(loss)) and pos.numel() == 0 and neg.numel() == 0


def _nan_outside(r):
    """Region.outside_intact for a NaN fill (NaN != NaN)."""
    c = r.buf.clone()
    r._view(c).fill_(float("nan"))
    return bool(torch.isnan(c).all())


def test_infomax_entry_points_fill_nan_poisoned_outputs():
    """The C entry points on outputs inside NaN-filled allocations (rows strided past the extent): every output element is
    written (finite, and equal to ops.infomax_bce's results bit for bit) and nothing outside the views is touched."""
    lib = cabi.lib
    G = 48
    x, batch, W = make_case(G, 23, 14)
    N = x.shape[0]
    ref_loss, ref_pos, ref_neg, ref_gx, ref_gW = call_head(x, batch, W, G, gscale=1.5)
    xd, bd, Wd = x.to(DEV), batch.to(DEV), W.to(DEV)
    segs = ops.Segments(bd, G)
    st = torch.cuda.current_stream().cuda_stream
    prec = 1 if ops.get_precision() == "tf32x3" else 0
    Sr, Hr = Region(G, D, D, NAN), Region(G, D, D, NAN)
    cabi.check(lib.pgnn_infomax_summary_fwd(xd.data_ptr(), D, segs.ptr.data_ptr(), segs.order.data_ptr(), G, D, Sr.ptr(), D, st))
    cabi.check(lib.pgnn_linear_bwd_x(Sr.ptr(), D, Wd.data_ptr(), G, D, D, None, 0, Hr.ptr(), D, prec, st))
    loss = filled(torch.full((1, 1), float("nan"), dtype=torch.float64))
    pos, neg, dscore = (filled(torch.full((1, n), float("nan"))) for n in (N, N, 2 * N))
    wsb = int(lib.pgnn_infomax_bce_workspace_bytes())
    ws = torch.full((wsb // 4 + 1,), float("nan"), device=DEV)
    cabi.check(lib.pgnn_infomax_bce_fwd(xd.data_ptr(), D, N, D, bd.data_ptr(), Hr.ptr(), G, loss.ptr(), pos.ptr(), neg.ptr(), dscore.ptr(),
                                        ws.data_ptr(), wsb, st))
    gscale = torch.tensor(1.5, dtype=torch.float64, device=DEV)
    gx, gW = Region(N, D, 304, NAN), Region(D, D, D, NAN)
    bwsb = int(lib.pgnn_infomax_bce_bwd_workspace_bytes(G, D))
    bws = torch.full((bwsb // 4 + 1,), float("nan"), device=DEV)
    cabi.check(lib.pgnn_infomax_bce_bwd(xd.data_ptr(), D, N, D, bd.data_ptr(), segs.ptr.data_ptr(), segs.order.data_ptr(), G, Sr.ptr(), Hr.ptr(),
                                        Wd.data_ptr(), dscore.ptr(), gscale.data_ptr(), gx.ptr(), 304, gW.ptr(), prec, bws.data_ptr(), bwsb, st))
    torch.cuda.synchronize()
    for r in (Sr, Hr, loss, pos, neg, dscore, gx, gW):
        assert _nan_outside(r) and bool(torch.isfinite(r.view).all())
    assert float(loss.view[0, 0]) == ref_loss
    assert torch.equal(pos.view[0], ref_pos) and torch.equal(neg.view[0], ref_neg)
    assert torch.equal(gx.view, ref_gx) and torch.equal(gW.view, ref_gW)


# ---------------------------------------------------------------------------------------------------------------------
# the steps against the oracle
# ---------------------------------------------------------------------------------------------------------------------
def _aux(step, d):
    rep = step.gnn(d["x"], d["edge_index"], d["edge_attr"])
    _, pos, neg = ops.infomax_bce(rep, d["batch"], step.discriminator.weight, d.get("num_graphs"))
    return dict(rep=rep, pos=pos, neg=neg)


def compare_step(name, step, loss_fn, P, b):
    """test_gpu_edgepred.compare_step's rule: `rep` by output_check, the scores by score_check, the loss within max(2e-6, 3 x the
    oracle's own fp32 error) of fp64 or equal to the oracle's fp64 head on the step's own scores to 1e-9 when those scores pass
    their bound, every gradient (encoder and discriminator) by gradient_check."""
    torch.set_num_threads(min(16, torch.get_num_threads()))
    l32, a32, g32, l64, a64, g64, near = S.grads_fp32_fp64(loss_fn, P, b)
    step.load_state(P)
    d = _dev(b)
    loss = step(d)
    grads = [(k, p.grad) for k, p in step.named_parameters()]
    assert all(g is not None for _, g in grads) and any(k == "discriminator.weight" for k, _ in grads)
    with torch.no_grad():
        aux = _aux(step, d)
    rows = []
    ok = output_check("rep", aux["rep"], a32["rep"], a64["rep"], rows)
    for k in ("pos", "neg"):
        ok &= score_check(k, aux[k], a32[k], a64[k], rows)
    lerr = abs(float(loss) - float(l64)) / max(abs(float(l64)), 1e-30)
    lref = abs(float(l32) - float(l64)) / max(abs(float(l64)), 1e-30)
    lhead = float(IO.bce_pair(aux["pos"].cpu().double(), aux["neg"].cpu().double()))
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
def test_infomax_step_b64_vs_oracle(domain, t):
    step = (ts.InfomaxStep if domain == "chem" else ts.BioInfomaxStep)(DEV, t, batch_size=64)
    b = step.make_batches(0, 1)[0]
    compare_step("infomax_%s_b64_%s" % (domain, t), step, lambda L, bb: IO.infomax_loss(L, bb, domain, t), IO.make_params(domain, 15, t), b)


@pytest.mark.parametrize("domain", ["chem", "bio"])
def test_infomax_gin_step_b256(domain):
    """The scripts' default batch (B = 256): loss and every gradient finite, the loss within the bar of the fp64 oracle or equal to
    the oracle's fp64 head on the step's own scores when those pass score_check (the oracle's forward only)."""
    step = (ts.InfomaxStep if domain == "chem" else ts.BioInfomaxStep)(DEV)
    b = step.make_batches(0, 1)[0]
    P = IO.make_params(domain, 16)
    step.load_state(P)
    d = _dev(b)
    loss = float(step(d))
    for k, p in step.named_parameters():
        assert p.grad is not None and bool(torch.isfinite(p.grad).all()), k
    assert not ops.device_errors()
    with torch.no_grad():
        a = _aux(step, d)
        lhead = float(IO.bce_pair(a["pos"].cpu().double(), a["neg"].cpu().double()))
        torch.set_num_threads(min(16, torch.get_num_threads()))
        (l32, a32), (l64, a64) = (IO.infomax_loss(O.leaf_params(P, dt), b, domain) for dt in (torch.float32, torch.float64))
        l32, l64 = float(l32), float(l64)
    rows = []
    scores_ok = all([score_check(k, a[k], a32[k], a64[k], rows) for k in ("pos", "neg")])
    lerr, lref = abs(loss - l64) / abs(l64), abs(l32 - l64) / abs(l64)
    ok = lerr <= max(2e-6, 3 * lref) or (scores_ok and abs(loss - lhead) <= 1e-9 * abs(lhead))
    write_report("infomax_%s_b256_gin" % domain, rows + [dict(kind="loss", name="loss", err=lerr, err_ref32=lref, ok=ok)],
                 dict(nodes=int(b["x"].shape[0]), loss=loss, loss_oracle64=l64, loss_head=lhead))
    assert np.isfinite(loss) and ok, (loss, l64, l32, lhead)


# ---------------------------------------------------------------------------------------------------------------------
# the store pipeline
# ---------------------------------------------------------------------------------------------------------------------
def test_store_pipeline_chem():
    """MoleculeStore.collate -> InfomaxStep gives exactly the batch and the loss of zinc_batch."""
    B, seed = 48, 10123
    ref = syn.zinc_batch(B, seed)
    graphs = syn.split_graphs(ref)
    store = data.MoleculeStore(np.cumsum([0] + [g[0].shape[0] for g in graphs]), np.cumsum([0] + [g[1].shape[1] for g in graphs]),
                               np.concatenate([g[0] for g in graphs]), np.concatenate([g[1] for g in graphs], 1),
                               np.concatenate([g[2] for g in graphs]), device=DEV)
    o = store.collate(np.arange(B))
    for k in ts.InfomaxStep.KEYS:
        assert torch.equal(getattr(o, k).cpu(), ref[k]), k
    step = ts.InfomaxStep(DEV, batch_size=B)
    step.load_state(IO.make_params("chem", 17))
    l_dev = float(step({k: getattr(o, k) for k in ts.InfomaxStep.KEYS + ("num_graphs",)}))
    l_syn = float(step(_dev({k: ref[k] for k in ts.InfomaxStep.KEYS + ("num_graphs",)})))
    assert l_dev == l_syn and np.isfinite(l_dev)
    assert not ops.device_errors()


def test_store_pipeline_bio():
    """BioGraphStore.collate -> BioInfomaxStep gives exactly the batch and the loss of ppi_batch."""
    B, seed = 12, 11077
    ref = syn.ppi_batch(B, seed, n_lo=60, n_hi=90, pairs_per_node=3, num_tasks=4)
    graphs, _ = syn.ppi_graphs(ref)
    store = data.BioGraphStore([g[0] for g in graphs], [g[1] for g in graphs], [g[2] for g in graphs], [0] * B, device=DEV)
    o = store.collate(np.arange(B))
    for k in ts.BioInfomaxStep.KEYS:
        assert torch.equal(getattr(o, k).cpu(), ref[k]), k
    step = ts.BioInfomaxStep(DEV, batch_size=B)
    step.load_state(IO.make_params("bio", 18))
    l_dev = float(step({k: getattr(o, k) for k in ts.BioInfomaxStep.KEYS + ("num_graphs",)}))
    l_syn = float(step(_dev({k: ref[k] for k in ts.BioInfomaxStep.KEYS + ("num_graphs",)})))
    assert l_dev == l_syn and np.isfinite(l_dev)
    assert not ops.device_errors()
