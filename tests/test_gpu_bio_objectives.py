"""GPU: bio masking and bio context prediction on the device.

* pgnn_softmax_ce_rows_fwd against an fp64 restatement: every row-group width (V = 1, 7, 9, 33), both label widths (Q = 7, 9),
  row counts around the group, warp and CTA boundaries up to the ~96 k rows of a B = 256 bio-masking step; multi-hot label rows
  with ties, all-zero rows, labels past V and non-finite label rows.  Inputs are views inside NaN-filled allocations, outputs
  inside sentinel-filled ones (device_buffers); the loss must repeat bit for bit.
* BioMaskingStep (four gnn_types) and BioContextPredStep against the oracle bodies of tests/bio_objectives_oracle.py at B = 64
  with the bars of tests/golden_util.py, and one bio-masking GIN step at the script's B = 256.
* The device pipeline: BioGraphStore.collate -> data.mask_edges_bio -> BioMaskingStep, and extract_context(center=False, seed)
  bit for bit against the oracle's extraction from the same roots."""
import importlib

import numpy as np
import pytest
import torch

import bio_objectives_oracle as BO
from device_buffers import DEV, NAN, SENT, Region, ceil4, filled
from golden_util import gradient_check, output_check, write_report
from oracle import gnn_oracle as O
from oracle import step_io_oracle as SO
from oracle import steps_oracle as S

pytestmark = pytest.mark.gpu
syn = importlib.import_module("pretrain-gnns_b200.synthetic")
ts = importlib.import_module("pretrain-gnns_b200.train_steps")
ops = importlib.import_module("pretrain-gnns_b200.ops")
data = importlib.import_module("pretrain-gnns_b200.data")
cabi = importlib.import_module("pretrain-gnns_b200._cabi")
LABEL_ERR = ops.DEVICE_ERROR_BITS[8]


# ---------------------------------------------------------------------------------------------------------------------
# the kernel
# ---------------------------------------------------------------------------------------------------------------------
def ce_rows_reference(logits, lab, V):
    """fp64: label = the first index of the row maximum; a row with a NaN, a non-finite maximum or a label >= V is bad and
    contributes its log-sum-exp only.  -> (mean loss, d loss / d logits [M, V], bad [M])"""
    x, t = logits.double(), lab.double()
    M, Q = t.shape
    if M == 0:
        return 0.0, torch.zeros(0, V, dtype=torch.float64), torch.zeros(0, dtype=torch.bool)
    mx = torch.where(t.isnan(), float("-inf"), t).max(1).values
    first = torch.where(t == mx[:, None], torch.arange(Q), Q).min(1).values
    bad = t.isnan().any(1) | ~torch.isfinite(mx) | (first >= V)
    y = torch.where(bad, 0, first)
    lse = torch.logsumexp(x, 1)
    loss = (lse - torch.where(bad, 0.0, x.gather(1, y[:, None])[:, 0])).sum() / M
    onehot = torch.zeros_like(x)
    onehot[torch.arange(M)[~bad], y[~bad]] = 1.0
    return float(loss), (torch.exp(x - lse[:, None]) - onehot) / M, bad


def label_rows(M, Q, seed):
    """Bio-shaped label rows: the 7 evidence channels multi-hot at 0.3 (ties and all-zero rows are common), the self-loop / mask
    columns mostly zero, a few rows with their maximum there, a few with fractional and negative values."""
    g = torch.Generator().manual_seed(seed)
    t = torch.zeros(M, Q)
    t[:, :7] = (torch.rand(M, 7, generator=g) < 0.3).float()
    if M:
        r = torch.randint(0, M, (max(M // 50, 1),), generator=g)
        t[r, Q - 1] = 2.0
        r = torch.randint(0, M, (max(M // 40, 1),), generator=g)
        t[r] = torch.randn(len(r), Q, generator=g).round(decimals=1)
    return t


def call_ce_rows(logits, lab, V, ld_pad=4, label_pad=3):
    """One pgnn_softmax_ce_rows_fwd call on poisoned buffers -> (loss, dlogits view, regions intact, flagged)."""
    M, Q = lab.shape
    L = filled(logits, ceil4(V) + ld_pad)
    T = filled(lab, Q + label_pad)
    ldd = ceil4(V)
    D = Region(M, ldd, ldd, SENT)
    loss = torch.full((3,), SENT, dtype=torch.float64, device=DEV)
    wsb = int(cabi.lib.pgnn_softmax_ce_rows_workspace_bytes())
    ws = torch.full((wsb // 4 + 1,), NAN, device=DEV)
    ops.device_errors(clear=True)
    cabi.check(cabi.lib.pgnn_softmax_ce_rows_fwd(L.ptr(), L.ld, M, V, T.ptr(), T.ld, Q, loss[1:].data_ptr(), D.ptr(), ldd, ws.data_ptr(), wsb,
                                                 torch.cuda.current_stream().cuda_stream), "softmax_ce_rows_fwd")
    flagged = LABEL_ERR in ops.device_errors(clear=True)
    intact = D.outside_intact() and float(loss[0]) == SENT and float(loss[2]) == SENT
    return float(loss[1]), D.view.cpu(), intact, flagged


@pytest.mark.parametrize("Q", [7, 9])
@pytest.mark.parametrize("V", [1, 7, 9, 33])
@pytest.mark.parametrize("M", [0, 1, 31, 32, 33, 4097, 96001])
def test_softmax_ce_rows_vs_fp64(M, V, Q):
    g = torch.Generator().manual_seed(M * 131 + V * 7 + Q)
    logits = torch.randn(M, V, generator=g) * 3
    lab = label_rows(M, Q, M + V + Q)
    loss, dl, intact, flagged = call_ce_rows(logits, lab, V)
    ref, dref, bad = ce_rows_reference(logits, lab, V)
    assert intact, "a sentinel around dlogits or the loss was overwritten"
    assert flagged == bool(bad.any()), (flagged, int(bad.sum()))
    assert abs(loss - ref) <= 1e-12 * max(abs(ref), 1.0), (loss, ref)
    assert torch.equal(dl[:, V:], torch.zeros(M, ceil4(V) - V)), "padding columns not zeroed"
    assert torch.allclose(dl[:, :V].double(), dref, rtol=1e-6, atol=1e-12 / max(M, 1))
    loss2, dl2, _, _ = call_ce_rows(logits, lab, V)
    assert loss2 == loss and torch.equal(dl2, dl), "not bit-for-bit repeatable"


def test_softmax_ce_rows_non_finite_label_rows():
    """A NaN anywhere in a label row, a +Inf maximum or a row of -Inf: flagged, the row contributes its log-sum-exp only; a -Inf
    beside a finite maximum is an ordinary row.  A row whose maximum is in column 7 or 8 is flagged at V = 7."""
    M, V, Q = 40, 7, 9
    g = torch.Generator().manual_seed(3)
    logits = torch.randn(M, V, generator=g)
    lab = label_rows(M, Q, 4)
    lab[:, 7:] = 0.0
    lab[(lab[:, :7].max(1).values > 1.5) | (lab.min(1).values < 0), :] = 0.0
    lab[3, 2] = NAN
    lab[5, 0] = float("inf")
    lab[6] = float("-inf")
    lab[7, 1], lab[7, 4] = float("-inf"), 1.0
    ok_rows = torch.ones(M, dtype=torch.bool)
    ok_rows[[3, 5, 6]] = False
    loss, dl, intact, flagged = call_ce_rows(logits, lab, V)
    ref, dref, bad = ce_rows_reference(logits, lab, V)
    assert torch.equal(bad, ~ok_rows) and flagged and intact
    assert abs(loss - ref) <= 1e-12 * abs(ref) and torch.allclose(dl.double()[:, :V], dref, rtol=1e-6, atol=1e-12)
    lab2 = lab.clone()
    lab2[[3, 5, 6]] = 0.0
    assert not call_ce_rows(logits, lab2, V)[3]
    lab2[9, 8] = 5.0
    assert call_ce_rows(logits, lab2, V)[3]


def test_masked_edge_type_loss_vs_torch_fp64():
    """ops.masked_edge_type_loss (gather, wgmma Linear, the new CE, backward) against torch's fp64 loss on argmax labels."""
    F = torch.nn.functional
    b = syn.bio_masking_batch(8, 21, n_lo=60, n_hi=90, num_tasks=4)
    g = torch.Generator().manual_seed(2)
    rep = torch.randn(b["x"].shape[0], 300, generator=g)
    W, bias = torch.randn(7, 300, generator=g) * 0.05, torch.randn(7, generator=g) * 0.05
    rr = [t.clone().double().requires_grad_(True) for t in (rep, W, bias)]
    me = b["edge_index"][:, b["masked_edge_idx"]]
    logits_ref = F.linear(rr[0][me[0]] + rr[0][me[1]], rr[1], rr[2])
    lref = F.cross_entropy(logits_ref, torch.argmax(b["mask_edge_label"], dim=1))
    lref.backward()
    dd = [t.clone().to(DEV).requires_grad_(True) for t in (rep, W, bias)]
    l, logits = ops.masked_edge_type_loss(dd[0], b["edge_index"].to(DEV), b["masked_edge_idx"].to(DEV), b["mask_edge_label"].to(DEV), dd[1], dd[2])
    l.backward()
    assert l.dtype == torch.float64 and logits.shape == (len(b["masked_edge_idx"]), 7)
    assert abs(float(l) - float(lref)) < 1e-6 and torch.allclose(logits.cpu().double(), logits_ref.detach(), atol=1e-4, rtol=1e-4)
    for mine, ref in zip(dd, rr):
        assert float((mine.grad.cpu().double() - ref.grad).abs().max()) <= 2e-5 * float(ref.grad.abs().max())
    assert not ops.device_errors()
    for lab in (b["mask_edge_label"].double(), b["mask_edge_label"][:-1]):   # fp64 rows; one row short
        with pytest.raises(cabi.PgnnError):
            ops.masked_edge_type_loss(dd[0], b["edge_index"].to(DEV), b["masked_edge_idx"].to(DEV), lab.to(DEV), dd[1], dd[2])


# ---------------------------------------------------------------------------------------------------------------------
# the steps against the oracle
# ---------------------------------------------------------------------------------------------------------------------
def _dev(b):
    return {k: (v.to(DEV) if torch.is_tensor(v) else v) for k, v in b.items()}


def _compare(name, step, loss_fn, P, b, aux_fn, head=None):
    """tests/test_gpu_parity_full.py's yardstick: loss within max(2e-6, 3 x the oracle's own fp32 error) relative to fp64, the
    forward outputs by output_check, every parameter gradient by gradient_check; the measured errors go to golden_util.write_report.
    head(aux) -> the loss the oracle's fp64 head gives on the step's own forward outputs.  With it, a loss outside that bar is
    still accepted when it equals head(aux) to 1e-9 and those outputs pass output_check: the difference from the oracle then
    comes from the outputs alone, which are held to their own bound (bio context prediction: the dot products of unnormalised
    300-wide bio GIN outputs carry the 3xTF32 error of the encoders into the loss at about 2e-6)."""
    torch.set_num_threads(min(16, torch.get_num_threads()))
    l32, a32, g32, l64, a64, g64, near = S.grads_fp32_fp64(loss_fn, P, b)
    step.load_state(P)
    d = _dev(b)
    loss = step(d)
    grads = [(k, p.grad) for k, p in step.named_parameters()]
    assert all(g is not None for _, g in grads)
    with torch.no_grad():
        aux = aux_fn(step, d)
    rows, ok = [], True
    for k, v in aux.items():
        ok &= output_check(k, v, a32[k], a64[k], rows)
    lerr = abs(float(loss) - float(l64)) / max(abs(float(l64)), 1e-30)
    lref = abs(float(l32) - float(l64)) / max(abs(float(l64)), 1e-30)
    outputs_ok = ok
    lhead = None if head is None else float(head({k: v.detach().cpu().double() for k, v in aux.items()}))
    via = "oracle"
    lok = lerr <= max(2e-6, 3 * lref)
    if not lok and lhead is not None and outputs_ok and abs(float(loss) - lhead) <= 1e-9 * abs(lhead):
        lok, via = True, "the oracle head on the step's outputs (err %.2e)" % (abs(float(loss) - lhead) / abs(lhead))
    rows.append(dict(kind="loss", name="loss", err=lerr, err_ref32=lref, ok=lok, via=via))
    ok &= rows[-1]["ok"]
    ok &= gradient_check(grads, g32, g64, near, rows)
    write_report(name, rows, dict(near_zero_preactivations=near, loss=float(loss), loss_oracle64=float(l64), loss_head_on_outputs=lhead))
    assert not ops.device_errors(), "index range flags raised on a valid batch"
    bad = [r for r in rows if not r["ok"]]
    assert ok, bad[:8]


def _masking_aux(step, d):
    rep = step.model(d["x"], d["edge_index"], d["edge_attr"])
    _, logits = ops.masked_edge_type_loss(rep, d["edge_index"], d["masked_edge_idx"], d["mask_edge_label"], step.head.weight, step.head.bias)
    return dict(rep=rep, logits=logits)


@pytest.mark.parametrize("t", ["gin", "gcn", "graphsage", "gat"])
def test_bio_masking_step_b64_vs_oracle(t):
    step = ts.BioMaskingStep(DEV, t, batch_size=64)
    b = step.make_batches(0, 1)[0]
    _compare("bio_masking_b64_" + t, step, lambda L, bb: BO.bio_masking_loss(L, bb, t), BO.make_params("bio_masking", 11, t), b, _masking_aux)


def test_bio_contextpred_step_b64_vs_oracle():
    step = ts.BioContextPredStep(DEV, batch_size=64)
    b = step.make_batches(0, 1)[0]

    def aux(step, d):
        pos, neg = step.scores(d)
        return dict(pos=pos, neg=neg)

    _compare("bio_contextpred_b64", step, BO.bio_contextpred_loss, BO.make_params("bio_contextpred", 12), b, aux,
             head=lambda a: O.contextpred_loss(a["pos"], a["neg"], 1))


def test_bio_masking_gin_step_b256():
    """The script's default batch (B = 256, ~96 k masked edges): loss and every gradient finite, the loss within the bar of the
    fp64 oracle (the oracle's forward only, fp32 and fp64)."""
    step = ts.BioMaskingStep(DEV)
    b = step.make_batches(0, 1)[0]
    P = BO.make_params("bio_masking", 13)
    step.load_state(P)
    loss = float(step(_dev(b)))
    for k, p in step.named_parameters():
        assert p.grad is not None and bool(torch.isfinite(p.grad).all()), k
    assert not ops.device_errors()
    torch.set_num_threads(min(16, torch.get_num_threads()))
    with torch.no_grad():
        l32, l64 = (float(BO.bio_masking_loss(O.leaf_params(P, dt), b)[0]) for dt in (torch.float32, torch.float64))
    lerr, lref = abs(loss - l64) / abs(l64), abs(l32 - l64) / abs(l64)
    write_report("bio_masking_b256_gin", [dict(kind="loss", name="loss", err=lerr, err_ref32=lref, ok=lerr <= max(2e-6, 3 * lref))],
                 dict(masked_edges=int(len(b["masked_edge_idx"])), loss=loss, loss_oracle64=l64))
    assert np.isfinite(loss) and lerr <= max(2e-6, 3 * lref), (loss, l64, l32)


# ---------------------------------------------------------------------------------------------------------------------
# the device pipeline
# ---------------------------------------------------------------------------------------------------------------------
def _store(num, seed):
    pb = syn.ppi_batch(num, seed, n_lo=60, n_hi=90, pairs_per_node=3, num_tasks=4)
    graphs, _ = syn.ppi_graphs(pb)
    centers = [int(s) % g[0] for s, g in zip(np.random.default_rng(seed).integers(0, 1 << 20, size=num), graphs)]
    return data.BioGraphStore([g[0] for g in graphs], [g[1] for g in graphs], [g[2] for g in graphs], centers, device=DEV), graphs, centers


def test_device_masking_pipeline_gives_the_oracle_loss():
    """BioGraphStore.collate -> data.mask_edges_bio -> BioMaskingStep equals the oracle body on the oracle-masked batch."""
    bs, graphs, _ = _store(24, 41)
    ids = np.array([3, 0, 17, 17, 9, 22, 5, 11, 1, 20, 8, 14])
    o = bs.collate(ids)
    eoff = o.edge_off.cpu().numpy()
    data.mask_edges_bio(o, eoff, 0.15, seed=77)
    ref = SO.collate_bio(graphs, ids)
    ea, idx, lab, _ = SO.mask_edges_bio(ref["edge_attr"], ref["edge_off"], 0.15, seed=77)
    hb = dict(x=torch.from_numpy(ref["x"]), edge_index=torch.from_numpy(ref["edge_index"]), edge_attr=torch.from_numpy(ea),
              masked_edge_idx=torch.from_numpy(idx), mask_edge_label=torch.from_numpy(lab))
    for k, v in hb.items():
        assert torch.equal(getattr(o, k).cpu(), v), k
    step = ts.BioMaskingStep(DEV, batch_size=len(ids))
    P = BO.make_params("bio_masking", 14)
    step.load_state(P)
    loss = float(step({k: getattr(o, k) for k in ts.BioMaskingStep.KEYS}))
    with torch.no_grad():
        l32, l64 = (float(BO.bio_masking_loss(O.leaf_params(P, dt), hb)[0]) for dt in (torch.float32, torch.float64))
    assert abs(loss - l64) <= max(2e-6, 3 * abs(l32 - l64)) * abs(l64), (loss, l64, l32)
    assert not ops.device_errors()


_CONTEXT_KEYS = ("x_context", "edge_index_context", "edge_attr_context", "overlap_context_substruct_idx", "batch_overlapped_context",
                 "overlapped_context_size")


def test_extract_context_random_root_bit_exact():
    """extract_context(center=False, seed): the roots are splitmix64(seed, slot) mod n; the context side equals the oracle's
    extraction from those roots bit for bit, the substructure side is the plain collation with the ego centres."""
    bs, graphs, centers = _store(20, 43)
    ids = np.array([4, 4, 0, 19, 7, 12, 3, 15, 15, 9])
    ograph = [(np.ones((g[0], 1), np.float32), g[1], g[2]) for g in graphs]
    for seed in (0, 5, 1234567):
        o = bs.extract_context(ids, 1, center=False, seed=seed)
        roots = SO.draw_roots([graphs[g][0] for g in ids], seed)
        ref = SO.extract_pairs_batch(ograph, ids, roots, 0, 1, 0, whole_graph=True)
        assert o.kept == len(ids)
        for key in _CONTEXT_KEYS:
            mine = getattr(o, key).cpu().numpy()
            assert mine.shape == ref[key].shape and np.array_equal(mine, ref[key]), (key, seed)
        full = SO.collate_bio(graphs, ids)
        assert np.array_equal(o.edge_index_substruct.cpu().numpy(), full["edge_index"])
        cen, _, _, _ = SO.collate_lists(np.arange(len(graphs) + 1), np.array(centers), ids, add=full["node_off"])
        assert np.array_equal(o.center_substruct_idx.cpu().numpy(), cen)
    # a different seed draws different roots (and so, on these graphs, a different context)
    a, b = bs.extract_context(ids, 1, center=False, seed=1), bs.extract_context(ids, 1, center=False, seed=2)
    assert not np.array_equal(SO.draw_roots([graphs[g][0] for g in ids], 1), SO.draw_roots([graphs[g][0] for g in ids], 2))
    assert a.x_context.shape != b.x_context.shape or not torch.equal(a.overlap_context_substruct_idx, b.overlap_context_substruct_idx) \
        or not torch.equal(a.edge_index_context, b.edge_index_context)


def test_extract_context_default_is_the_centre():
    """The default call is center=True: the roots are the ego centres, `seed` plays no part."""
    bs, graphs, centers = _store(12, 47)
    ids = np.array([2, 0, 11, 5, 5, 8])
    ograph = [(np.ones((g[0], 1), np.float32), g[1], g[2]) for g in graphs]
    ref = SO.extract_pairs_batch(ograph, ids, [centers[g] for g in ids], 0, 2, 0, whole_graph=True)
    d0, d1 = bs.extract_context(ids, 2), bs.extract_context(ids, 2, center=True, seed=99)
    for key in _CONTEXT_KEYS + ("x_substruct", "edge_index_substruct", "edge_attr_substruct", "center_substruct_idx"):
        assert torch.equal(getattr(d0, key), getattr(d1, key)), key
        if key in _CONTEXT_KEYS:
            assert np.array_equal(getattr(d0, key).cpu().numpy(), ref[key]), key
