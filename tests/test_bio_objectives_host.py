"""CPU: the bio masking and bio context-prediction train() bodies of tests/bio_objectives_oracle.py on the oracle port against
the same bodies on the reference's OWN bio/model.py (loss and every gradient), the edge-type label's tie rule against
torch.argmax, the synthetic bio batches against the fields the train steps read, and the argument checks and ptxas report of
pgnn_softmax_ce_rows_fwd (no device touched)."""
import ctypes
import importlib
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

import bio_objectives_oracle as BO
from oracle import gnn_oracle as O
from oracle import reference_runner as R

syn = importlib.import_module("pretrain-gnns_b200.synthetic")
ts = importlib.import_module("pretrain-gnns_b200.train_steps")
cabi = importlib.import_module("pretrain-gnns_b200._cabi")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
needs_reference = pytest.mark.skipif(not R.available(), reason="the reference sources are not staged under oracle/_ref")


def _masking_batch(directed, seed=5):
    b = syn.bio_masking_batch(3, seed, one_direction=directed, n_lo=30, n_hi=50, num_tasks=4)
    return {k: b[k] for k in ts.BioMaskingStep.KEYS}


def _context_batch(directed, seed=5):
    b = syn.bio_context_batch(4, seed, n_lo=30, n_hi=50, pairs_per_node=3, num_tasks=4)
    if directed:
        b = syn.one_direction_only(b, seed, keys=("edge_index_substruct", "edge_attr_substruct"))
        b = syn.one_direction_only(b, seed + 1, keys=("edge_index_context", "edge_attr_context"))
    return {k: b[k] for k in ts.BioContextPredStep.KEYS}


def _compare_with_reference(ref, loss_fn, P, b):
    """oracle/steps_oracle's yardstick (test_train_bodies_port_equals_reference): loss within 1e-6, every gradient within 2e-4
    of its scale (the model's largest gradient for a structurally zero one)."""
    ref.load(P)
    loss_ref = ref(b)
    L = O.leaf_params(P)
    loss, _ = loss_fn(L, b)
    loss.backward()
    assert abs(float(loss) - float(loss_ref)) <= 1e-6 * max(1.0, abs(float(loss_ref))), (float(loss), float(loss_ref))
    named = {name + "." + k: p for name, m in ref.named.items() for k, p in m.named_parameters()}
    gmax = max(float(p.grad.abs().max()) for p in named.values())
    L64 = O.leaf_params(P, torch.float64)
    loss_fn(L64, b)[0].backward()
    for k, p in named.items():
        zero = float(L64[k].grad.abs().max()) < 1e-9 * gmax
        scale = gmax if zero else max(float(p.grad.abs().max()), 1e-3 * gmax)
        assert float((L[k].grad - p.grad).abs().max()) <= 2e-4 * scale, (k, float((L[k].grad - p.grad).abs().max()) / scale)


@needs_reference
@pytest.mark.parametrize("directed", [False, True])
@pytest.mark.parametrize("t", ["gin", "gcn", "graphsage", "gat"])
def test_bio_masking_port_equals_reference(t, directed):
    """bio/pretrain_masking.py:43-55 on the reference's bio GNN with torch.argmax + nn.CrossEntropyLoss, against the port."""
    torch.set_num_threads(1)
    b = _masking_batch(directed)
    lab = b["mask_edge_label"]
    assert (lab.sum(1) == 0).any() and (lab.sum(1) >= 2).any()   # all-zero rows and multi-hot ties are in the batch
    _compare_with_reference(BO.ReferenceBioMaskingStep(t), lambda L, bb: BO.bio_masking_loss(L, bb, t), BO.make_params("bio_masking", 3, t), b)


@needs_reference
@pytest.mark.parametrize("directed", [False, True])
@pytest.mark.parametrize("neg_samples", [1, 2])
def test_bio_contextpred_port_equals_reference(neg_samples, directed):
    """bio/pretrain_contextpred.py:53-97 (cbow, mean pooling, center = 0) on the reference's bio GNNs, against the port."""
    torch.set_num_threads(1)
    b = _context_batch(directed)
    _compare_with_reference(BO.ReferenceBioContextPredStep(neg_samples), lambda L, bb: BO.bio_contextpred_loss(L, bb, neg_samples),
                            BO.make_params("bio_contextpred", 4), b)


def test_edge_type_label_is_the_first_maximum():
    """The oracle's label equals torch.argmax (torch >= 1.7: the first maximal index) on multi-hot rows with ties, all-zero rows,
    rows whose maximum sits in the self-loop / mask columns, and negative and fractional values."""
    rows = [[0, 0, 0, 0, 0, 0, 0, 0, 0], [1, 1, 1, 1, 1, 1, 1, 0, 0], [0, 1, 0, 1, 0, 0, 1, 0, 0], [0, 0, 0, 0, 0, 0, 0, 0, 1],
            [0, 0, 0, 0, 0, 0, 0, 1, 1], [-1, -2, -1, -3, -5, -1, -4, -2, -1], [0.5, 0.25, 0.5, 0, 0, 0, 0.5, 0, 0]]
    lab = torch.cat([torch.tensor(rows, dtype=torch.float32), syn.bio_masking_batch(4, 9, n_lo=40, n_hi=60, num_tasks=4)["mask_edge_label"]])
    ties = int(((lab == lab.max(1, keepdim=True).values).sum(1) > 1).sum())
    assert ties > lab.shape[0] // 4 and (lab.sum(1) == 0).sum() > 0
    assert torch.equal(BO.edge_type_label(lab), torch.argmax(lab, dim=1))
    assert BO.edge_type_label(lab)[:7].tolist() == [0, 0, 1, 8, 7, 0, 0]
    assert BO.edge_type_label(torch.zeros(0, 9)).shape == (0,)


def test_synthetic_bio_batches_hold_the_step_fields():
    """bio_masking_batch: MaskEdge'd columns carry [0,...,0,1] in both directions, labels are the pre-mask attribute rows, one pair
    per int(e/2 * 0.15 + 1) per graph (bio/util.py:78-80).  bio_context_batch: the whole ego graph and its centre on the
    substructure side, the context from the defined root draw; both carry every field their step reads."""
    b = syn.bio_masking_batch(3, 7, n_lo=30, n_hi=50, num_tasks=4)
    clean = syn.ppi_batch(3, 7, n_lo=30, n_hi=50, num_tasks=4)
    assert set(ts.BioMaskingStep.KEYS) <= set(b)
    idx, ea = b["masked_edge_idx"], b["edge_attr"]
    mask = torch.tensor([0, 0, 0, 0, 0, 0, 0, 0, 1], dtype=torch.float32)
    assert (ea[idx] == mask).all() and (ea[idx + 1] == mask).all()
    assert torch.equal(b["mask_edge_label"], clean["edge_attr"][idx])
    _, eoff = syn.ppi_graphs(clean)
    assert len(idx) == sum(int((eoff[g + 1] - eoff[g]) // 2 * 0.15 + 1) for g in range(3))
    assert b["masked_edge_idx"].dtype == torch.int64 and b["mask_edge_label"].dtype == torch.float32
    c = syn.bio_context_batch(3, 7, n_lo=30, n_hi=50, num_tasks=4)
    assert set(ts.BioContextPredStep.KEYS) <= set(c)
    assert torch.equal(c["edge_index_substruct"], clean["edge_index"]) and torch.equal(c["center_substruct_idx"], clean["center_node_idx"])
    assert c["x_context"].dtype == torch.float32 and c["edge_attr_context"].shape[1] == 9
    assert torch.equal(c["overlapped_context_size"], torch.bincount(c["batch_overlapped_context"], minlength=3))


@pytest.mark.parametrize("directed", [False, True])
def test_synthetic_bio_batches_equal_the_oracle_transforms(directed):
    """The package's generators restate the device draws without importing oracle/: bio_masking_batch equals the oracle's MaskEdge
    (step_io_oracle.mask_edges_bio, pinned to the reference's MaskEdge) and bio_context_batch equals the oracle's extraction
    (extract_pairs_batch, pinned to the reference's ExtractSubstructureContextPair) from the roots draw_roots gives, bit for bit."""
    from oracle import step_io_oracle as SO
    kw = dict(n_lo=30, n_hi=60, pairs_per_node=2, num_tasks=4)
    clean = syn.ppi_batch(5, 13, **kw)
    if directed:
        clean = syn.one_direction_only(clean, 13)
    _, eoff = syn.ppi_graphs(clean)
    b = syn.bio_masking_batch(5, 13, 0.15, one_direction=directed, **kw)
    ea, idx, lab, _ = SO.mask_edges_bio(clean["edge_attr"].numpy(), eoff, 0.15, 13)
    assert np.array_equal(b["edge_attr"].numpy(), ea) and np.array_equal(b["masked_edge_idx"].numpy(), idx)
    assert np.array_equal(b["mask_edge_label"].numpy(), lab) and len(idx) > 0
    if directed:
        return
    graphs, _ = syn.ppi_graphs(clean)
    for l1 in (1, 2):
        c = syn.bio_context_batch(5, 13, l1, **kw)
        roots = SO.draw_roots([g[0] for g in graphs], 13)
        ref = SO.extract_pairs_batch([(np.ones((g[0], 1), np.float32), g[1], g[2]) for g in graphs], np.arange(5), roots, 0, l1, 0, whole_graph=True)
        assert len(ref["kept"]) == 5
        for key in ("x_context", "edge_index_context", "edge_attr_context", "overlap_context_substruct_idx", "batch_overlapped_context",
                    "overlapped_context_size"):
            assert c[key].shape == ref[key].shape and np.array_equal(c[key].numpy(), ref[key]), (key, l1)


def test_softmax_ce_rows_argument_validation_without_gpu():
    dll = cabi.lib.load()
    wsb = dll.pgnn_softmax_ce_rows_workspace_bytes()
    assert wsb >= 8 * 132
    ws = ctypes.create_string_buffer(wsb)   # a host address: no argument check below reaches the device
    w = ctypes.addressof(ws)
    f = dll.pgnn_softmax_ce_rows_fwd
    one = ctypes.addressof(ctypes.create_string_buffer(8))
    # (logits, ld, M, V, label_rows, ld_label, Q, loss_mean, dlogits, lddl, workspace, workspace_bytes, stream)
    assert f(None, 8, -1, 7, None, 9, 9, one, None, 8, w, wsb, None) == -1    # M < 0
    assert f(None, 8, 4, 0, None, 9, 9, one, None, 8, w, wsb, None) == -1     # V == 0
    assert f(None, 8, 4, 7, None, 9, 0, one, None, 8, w, wsb, None) == -1     # Q == 0
    assert f(None, 8, 4, 7, None, 8, 9, one, None, 8, w, wsb, None) == -1     # ld_label < Q
    assert f(None, 6, 4, 7, None, 9, 9, one, None, 8, w, wsb, None) == -1     # ld < V
    assert f(None, 8, 4, 7, None, 9, 9, one, None, 6, w, wsb, None) == -1     # lddl < V
    assert f(None, 8, 4, 7, None, 9, 9, None, None, 8, w, wsb, None) == -1    # no loss
    assert f(None, 8, 4, 7, None, 9, 9, one, None, 8, None, wsb, None) == -1  # no workspace
    assert f(None, 8, 4, 7, None, 9, 9, one, None, 8, w, wsb - 1, None) == -3  # workspace too small
    assert f(None, 8, 4, 7, one, 9, 9, one, one, 8, w, wsb, None) == -1       # M > 0 without logits
    assert f(one, 8, 4, 7, None, 9, 9, one, one, 8, w, wsb, None) == -1       # ... without label rows
    assert f(one, 8, 4, 7, one, 9, 9, one, None, 8, w, wsb, None) == -1       # ... without dlogits


@pytest.mark.skipif(not (os.path.exists(NVCC) or shutil.which("nvcc")), reason="nvcc not available")
def test_heads_ptxas_no_spills(tmp_path):
    """Every instantiation of k_softmax_ce_rows (and the int64-label k_softmax_ce beside it) compiles for sm_90a without spills."""
    nvcc = NVCC if os.path.exists(NVCC) else shutil.which("nvcc")
    src = os.path.join(ROOT, "pretrain-gnns_b200", "csrc", "heads.cu")
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--expt-relaxed-constexpr",
           "-I" + os.path.join(ROOT, "include"), "-Xptxas", "-v", "-c", src, "-o", str(tmp_path / "heads.o")]
    out = subprocess.run(cmd, capture_output=True, text=True)
    assert out.returncode == 0, out.stderr[-4000:]
    kernels, cur = {}, None
    for line in (out.stdout + out.stderr).splitlines():
        m = re.search(r"Compiling entry function '(\w+)'", line)
        if m:
            cur = m.group(1) if "softmax_ce" in m.group(1) else None
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if cur and m:
            kernels[cur] = (int(m.group(1)), int(m.group(2)))
    assert len(kernels) == 7, kernels   # k_softmax_ce + k_softmax_ce_rows<1, 2, 4, 8, 16, 32>
    assert all(v == (0, 0) for v in kernels.values()), kernels
