"""CPU: edge-prediction pre-training.  The oracle's NegativeEdge loop against the reference's own NegativeEdge.__call__ (chem and bio
util.py, torch.randint replaced by the defined candidates) on ordinary and corner-case graphs; the oracle's BatchAE against the
reference's; synthetic.negative_edge_index / edgepred_batch / bio_edgepred_batch against the oracle bit for bit; the train() body on
the oracle port against the same body on the reference's own model.py; the C argument checks and the ptxas report of the new kernels
(no device touched)."""
import ctypes
import importlib
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

import edgepred_oracle as EO
from oracle import reference_runner as R
from test_bio_objectives_host import _compare_with_reference

syn = importlib.import_module("pretrain-gnns_b200.synthetic")
ts = importlib.import_module("pretrain-gnns_b200.train_steps")
cabi = importlib.import_module("pretrain-gnns_b200._cabi")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
needs_reference = pytest.mark.skipif(not R.available(), reason="the reference sources are not staged under oracle/_ref")


def _complete(n):
    a, b = np.meshgrid(np.arange(n), np.arange(n), indexing="ij")
    keep = a != b
    return np.stack([a[keep], b[keep]])


def corner_graphs():
    """(name, n, graph-local edge_index [2, e]) of every case the transform must get right."""
    mol = syn.split_graphs(syn.zinc_batch(2, 3))
    ppi, _ = syn.ppi_graphs(syn.ppi_batch(1, 4, n_lo=40, n_hi=60, num_tasks=4))
    one_dir = syn.split_graphs(syn.one_direction_only(syn.zinc_batch(1, 5), 5))[0]
    one_dir_odd = one_dir[1][:, :one_dir[1].shape[1] - (1 - one_dir[1].shape[1] % 2)]
    dup = np.array([[0, 1, 0, 1, 2, 3, 2, 3], [1, 0, 1, 0, 3, 2, 3, 2]])
    return [("molecule", mol[0][0].shape[0], mol[0][1]), ("molecule2", mol[1][0].shape[0], mol[1][1]),
            ("ppi", ppi[0][0], ppi[0][1]),
            ("one_node", 1, np.zeros((2, 2), np.int64)),
            ("no_edges", 5, np.zeros((2, 0), np.int64)),
            ("complete", 4, _complete(4)),
            ("duplicate_bonds", 5, dup),
            ("one_direction_odd", one_dir[0].shape[0], one_dir_odd),
            ("repeats", 3, np.array([[0, 1, 1, 2], [1, 0, 2, 1]]))]


def _reference_negative_edge(mod, Data, n, ei, cand, monkeypatch):
    class DataWithEdges(Data):
        @property
        def num_edges(self):   # PyG 1.0.3's Data.num_edges: the size of edge_index along its cat dimension
            return self.edge_index.size(self.cat_dim("edge_index", self.edge_index))

    calls = []

    def randint(lo, hi, size):
        calls.append((lo, hi, tuple(size)))
        assert (lo, hi, tuple(size)) == (0, n, tuple(cand.shape))
        return torch.from_numpy(cand.copy())

    monkeypatch.setattr(torch, "randint", randint)
    d = DataWithEdges(x=torch.zeros(n, 2, dtype=torch.int64), edge_index=torch.from_numpy(np.ascontiguousarray(ei, dtype=np.int64)))
    out = mod.NegativeEdge()(d).negative_edge_index
    monkeypatch.undo()
    assert len(calls) == 1
    return out.numpy()


@needs_reference
@pytest.mark.parametrize("domain", ["chem", "bio"])
def test_negative_edge_equals_reference(domain, monkeypatch):
    mod = R.load(domain, "util")
    from torch_geometric.data import Data
    for name, n, ei in corner_graphs():
        e = ei.shape[1]
        for seed, e0 in ((0, 0), (7, 123), (2 ** 40 + 3, 5)):
            cand = EO.negative_edge_candidates(n, e, e0, seed)
            ref = _reference_negative_edge(mod, Data, n, ei, cand, monkeypatch)
            mine = EO.negative_edge(ei, n, cand)
            assert mine.shape == ref.shape and np.array_equal(mine, ref), (domain, name, seed)
            if name in ("one_node", "complete", "no_edges"):
                assert mine.shape == (2, 0), name
            if name == "one_direction_odd":
                assert e % 2 == 1 and mine.shape[1] > e // 2, "an odd e must not stop at e / 2"
            if name == "repeats" and seed == 0:
                valid = [(a, b) for a, b in cand.T if a != b and (a, b) not in set(map(tuple, ei.T))]
                assert len(valid) > len(set(valid)) and mine.shape[1] == 2, "no candidate repeated before the quota"
            if name in ("molecule", "ppi") and e % 2 == 0:
                assert mine.shape[1] == e // 2


@needs_reference
@pytest.mark.parametrize("domain", ["chem", "bio"])
def test_batch_ae_equals_reference(domain):
    mod = R.load(domain, "batch")
    from torch_geometric.data import Data
    graphs = syn.split_graphs(syn.zinc_batch(4, 9))
    items = []
    for i, (x, ei, ea) in enumerate(graphs):
        neg = EO.negative_edge(ei, x.shape[0], EO.negative_edge_candidates(x.shape[0], ei.shape[1], 10 * i, 11))
        items.append(dict(x=np.asarray(x, np.int64), edge_index=np.asarray(ei, np.int64), edge_attr=np.asarray(ea, np.int64), negative_edge_index=neg))
    ref = mod.BatchAE.from_data_list([Data(**{k: torch.from_numpy(v) for k, v in d.items()}) for d in items])
    mine = EO.batch_ae(items)
    for k in ("x", "edge_index", "edge_attr", "negative_edge_index", "batch"):
        assert np.array_equal(ref[k].numpy(), mine[k]), k


def _corner_batch():
    """The corner graphs as one collated batch: (edge_index, node_off, edge_off)."""
    items = [dict(x=np.zeros((n, 2), np.int64), edge_index=np.asarray(ei, np.int64)) for _, n, ei in corner_graphs()]
    b = EO.batch_ae(items)
    node_off = np.concatenate([[0], np.cumsum([d["x"].shape[0] for d in items])]).astype(np.int64)
    edge_off = np.concatenate([[0], np.cumsum([d["edge_index"].shape[1] for d in items])]).astype(np.int64)
    return b["edge_index"], node_off, edge_off


def test_synthetic_restatement_equals_the_oracle():
    """synthetic.negative_edge_index (vectorised over the batch) equals the oracle's per-graph loop bit for bit: on the corner
    graphs collated, on chem and bio edgepred batches, and on a one-direction batch."""
    for seed in (0, 3, 2 ** 62 + 17):
        ei, node_off, edge_off = _corner_batch()
        ref, _ = EO.negative_edges_batch(ei, node_off, edge_off, seed)
        assert np.array_equal(syn.negative_edge_index(ei, node_off, edge_off, seed), ref)
    b = syn.edgepred_batch(6, 21)
    ref, _ = EO.negative_edges_batch(b["edge_index"].numpy(), b["ptr"].numpy(), b["edge_off"].numpy(), 21)
    assert np.array_equal(b["negative_edge_index"].numpy(), ref) and ref.shape[1] == b["edge_index"].shape[1] // 2
    bb = syn.bio_edgepred_batch(2, 22, n_lo=60, n_hi=90, num_tasks=4)
    ref, _ = EO.negative_edges_batch(bb["edge_index"].numpy(), bb["ptr"].numpy(), bb["edge_off"].numpy(), 22)
    assert np.array_equal(bb["negative_edge_index"].numpy(), ref)
    od = syn.one_direction_only(syn.zinc_batch(5, 23), 23)
    eoff = syn.edge_offsets(od)
    ref, off = EO.negative_edges_batch(od["edge_index"].numpy(), od["ptr"].numpy(), eoff, 23)
    assert np.array_equal(syn.negative_edge_index(od["edge_index"].numpy(), od["ptr"].numpy(), eoff, 23), ref)
    assert set(ts.EdgePredStep.KEYS) <= set(b) and set(ts.BioEdgePredStep.KEYS) <= set(bb)


@needs_reference
@pytest.mark.parametrize("domain", ["chem", "bio"])
@pytest.mark.parametrize("t", ["gin", "gcn", "graphsage", "gat"])
def test_edgepred_port_equals_reference(domain, t):
    """chem/pretrain_edgepred.py:33-39 (and bio's) on the reference's own GNN with nn.BCEWithLogitsLoss on fp32 scores, against the
    port's body with the BCE on fp64 scores."""
    torch.set_num_threads(1)
    if domain == "chem":
        b = syn.edgepred_batch(3, 5)
        ref = EO.ReferenceEdgePredStep(t)
    else:
        b = syn.bio_edgepred_batch(2, 5, n_lo=30, n_hi=50, num_tasks=4)
        ref = EO.ReferenceBioEdgePredStep(t)
    b = {k: b[k] for k in ts.EdgePredStep.KEYS}
    _compare_with_reference(ref, lambda L, bb: EO.edgepred_loss(L, bb, domain, t), EO.make_params(domain, 3, t), b)


def test_negative_edges_argument_validation_without_gpu():
    dll = cabi.lib.load()
    off = np.array([0, 4, 7, 7, 12], dtype=np.int64)
    assert dll.pgnn_negative_edges_capacity(off.ctypes.data_as(ctypes.c_void_p), 4) == 2 + 15 + 0 + 25
    assert dll.pgnn_negative_edges_capacity(None, 4) == -1
    assert dll.pgnn_negative_edges_capacity(off.ctypes.data_as(ctypes.c_void_p), -1) == -1
    assert dll.pgnn_negative_edges_workspace_bytes(-1, 0, 0) == -1 and dll.pgnn_negative_edges_workspace_bytes(4, -1, 0) == -1
    assert dll.pgnn_negative_edges_workspace_bytes(4, 0, -1) == -1
    wsb = dll.pgnn_negative_edges_workspace_bytes(4, 12, 42)
    assert wsb >= 8 * 12 * 8 + 42 * 8
    ws = ctypes.create_string_buffer(wsb)
    w, one = ctypes.addressof(ws), ctypes.addressof(ctypes.create_string_buffer(64))
    f = dll.pgnn_negative_edges
    # (edge_index, E, node_off, edge_off, B, seed, capacity, workspace, workspace_bytes, out, out_off, stream)
    assert f(one, 12, one, one, -1, 0, 42, w, wsb, one, one, None) == -1      # B < 0
    assert f(one, -1, one, one, 4, 0, 42, w, wsb, one, one, None) == -1       # E < 0
    assert f(one, 12, one, one, 4, 0, -1, w, wsb, one, one, None) == -1       # capacity < 0
    assert f(None, 12, one, one, 4, 0, 42, w, wsb, one, one, None) == -1      # E > 0 without edge_index
    assert f(one, 12, None, one, 4, 0, 42, w, wsb, one, one, None) == -1      # no node_off
    assert f(one, 12, one, None, 4, 0, 42, w, wsb, one, one, None) == -1      # no edge_off
    assert f(one, 12, one, one, 4, 0, 42, w, wsb, None, one, None) == -1      # capacity > 0 without output
    assert f(one, 12, one, one, 4, 0, 42, w, wsb, one, None, None) == -1      # no output offsets
    assert f(one, 12, one, one, 4, 0, 42, None, wsb, one, one, None) == -1    # no workspace
    assert f(one, 12, one, one, 4, 0, 42, w, wsb - 1, one, one, None) == -3   # workspace too small


def test_edge_pair_bce_argument_validation_without_gpu():
    dll = cabi.lib.load()
    wsb = dll.pgnn_edge_pair_bce_workspace_bytes()
    assert wsb >= 2 * 8 * 132
    ws = ctypes.create_string_buffer(wsb + 16)
    w = (ctypes.addressof(ws) + 15) // 16 * 16
    one = (ctypes.addressof(ctypes.create_string_buffer(64)) + 15) // 16 * 16
    f = dll.pgnn_edge_pair_bce_fwd
    # (x, ldx, N, C, pos_u, pos_v, pos_stride, P, neg_u, neg_v, neg_stride, Q, loss, pos, neg, dscore, pairs, ws, wsb, stream)
    assert f(one, 300, -1, 300, one, one, 2, 4, one, one, 1, 4, one, one, one, one, one, w, wsb, None) == -1   # N < 0
    assert f(one, 300, 8, 0, one, one, 2, 4, one, one, 1, 4, one, one, one, one, one, w, wsb, None) == -1     # C == 0
    assert f(one, 296, 8, 300, one, one, 2, 4, one, one, 1, 4, one, one, one, one, one, w, wsb, None) == -1   # ldx < C
    assert f(one, 300, 8, 300, one, one, 2, -1, one, one, 1, 4, one, one, one, one, one, w, wsb, None) == -1  # P < 0
    assert f(one, 300, 8, 300, None, one, 2, 4, one, one, 1, 4, one, one, one, one, one, w, wsb, None) == -1  # P > 0 without pos_u
    assert f(one, 300, 8, 300, one, one, 2, 4, one, None, 1, 4, one, one, one, one, one, w, wsb, None) == -1  # Q > 0 without neg_v
    assert f(one, 300, 8, 300, one, one, 2, 4, one, one, 1, 4, None, one, one, one, one, w, wsb, None) == -1  # no loss
    assert f(one, 300, 8, 300, one, one, 2, 4, one, one, 1, 4, one, one, one, None, one, w, wsb, None) == -1  # no dscore
    assert f(one, 300, 8, 300, one, one, 2, 4, one, one, 1, 4, one, one, one, one, None, w, wsb, None) == -1  # no pairs
    assert f(one, 300, 8, 300, one, one, 2, 4, one, one, 1, 4, one, one, one, one, one, None, wsb, None) == -1  # no workspace
    assert f(one, 300, 8, 300, one, one, 2, 4, one, one, 1, 4, one, one, one, one, one, w, wsb - 1, None) == -3  # too small
    assert f(one, 302, 8, 302, one, one, 2, 4, one, one, 1, 4, one, one, one, one, one, w, wsb, None) == -4  # C % 4
    assert f(one + 4, 300, 8, 300, one, one, 2, 4, one, one, 1, 4, one, one, one, one, one, w, wsb, None) == -4  # misaligned x
    b = dll.pgnn_edge_pair_bce_bwd
    # (x, ldx, N, C, dscore, gscale, rowptr_t, nbr_t, eid_t, rowptr_s, nbr_s, eid_s, gx, ldgx, stream)
    assert b(one, 300, -1, 300, one, one, one, one, one, one, one, one, one, 300, None) == -1
    assert b(one, 300, 8, 300, one, None, one, one, one, one, one, one, one, 300, None) == -1                  # no gscale
    assert b(one, 300, 8, 300, one, one, None, one, one, one, one, one, one, 300, None) == -1                  # no rowptr_t
    assert b(one, 300, 8, 300, one, one, one, one, one, one, one, one, one, 296, None) == -1                   # ldgx < C
    assert b(one, 300, 0, 300, None, None, None, None, None, None, None, None, None, 300, None) == 0         # N == 0: nothing


def _ptxas(src_name, tmp_path):
    nvcc = NVCC if os.path.exists(NVCC) else shutil.which("nvcc")
    src = os.path.join(ROOT, "pretrain-gnns_b200", "csrc", src_name)
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--expt-relaxed-constexpr",
           "-I" + os.path.join(ROOT, "include"), "-Xptxas", "-v", "-c", src, "-o", str(tmp_path / (src_name + ".o"))]
    out = subprocess.run(cmd, capture_output=True, text=True)
    assert out.returncode == 0, out.stderr[-4000:]
    kernels, cur = {}, None
    for line in (out.stdout + out.stderr).splitlines():
        m = re.search(r"Compiling entry function '(\w+)'", line)
        if m:
            cur = m.group(1) if ("negative" in m.group(1) or "edge_pair" in m.group(1)) else None
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if cur and m:
            kernels[cur] = (int(m.group(1)), int(m.group(2)))
    return kernels


@pytest.mark.skipif(not (os.path.exists(NVCC) or shutil.which("nvcc")), reason="nvcc not available")
def test_edgepred_kernels_ptxas_no_spills(tmp_path):
    """The four kernels of the transform and the two of the head compile for sm_90a without spills."""
    k = _ptxas("negative_edges.cu", tmp_path)
    assert len(k) == 4 and all(v == (0, 0) for v in k.values()), k
    k = _ptxas("heads.cu", tmp_path)
    assert len(k) == 2 and all(v == (0, 0) for v in k.values()), k
