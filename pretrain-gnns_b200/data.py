"""Device-resident molecule store and on-device batch collation (SURVEY.md section 8(f), row f1), and the staging of
host-collated batches (one pinned buffer, one asynchronous copy per batch) for callers that keep the reference's DataLoader.

The reference collates on the host, one Python loop of `torch.cat`s per batch (chem/batch.py:17-52 BatchMasking,
:141-210 BatchSubstructContext) inside DataLoader workers, then copies the batch to the GPU.  An H100 has 80 GB of
HBM: the whole pre-training set (ZINC15, 2M molecules x ~23 atoms: < 1 GB in the compact form below) stays resident and a
batch is one `pgnn_collate_chem` call on a list of graph ids -- no host work, no H2D copy per step.
"""
from __future__ import annotations

from types import SimpleNamespace

import numpy as np
import torch

from ._cabi import check, lib


def _pair_first(edge_ptr_host, edge_index):
    """[Et/2] uint8: 1 where the bond pair (columns 2p, 2p+1) is the first of its graph with those endpoints.  The reference's
    transforms go through networkx, which keeps one edge per unordered pair (chem/loader.py:173 `if not G.has_edge(...)`)."""
    ep = np.asarray(edge_ptr_host, dtype=np.int64)
    if (ep % 2).any():
        raise ValueError("every graph must hold its bonds as adjacent (u,v),(v,u) column pairs (chem/loader.py:83-86)")
    P = int(ep[-1]) // 2
    if P == 0:
        return np.zeros(0, np.uint8)
    u, v = np.asarray(edge_index[0][0::2], dtype=np.int64), np.asarray(edge_index[1][0::2], dtype=np.int64)
    lo, hi = np.minimum(u, v), np.maximum(u, v)
    g = np.searchsorted(ep // 2, np.arange(P), side="right") - 1
    M = int(hi.max()) + 1
    key = (g * M + lo) * M + hi
    _, first = np.unique(key, return_index=True)
    out = np.zeros(P, np.uint8)
    out[first] = 1
    return out


def _extract(store, ids, roots, seed, k, l1, l2, whole_graph):
    """BFS + scans (pgnn_extract_pairs) -> (ids_dev, workspace, offsets [6,B+1] device, N_full, E_full)."""
    ids = np.ascontiguousarray(ids, dtype=np.int64)
    if ids.size and (ids.min() < 0 or ids.max() >= store.num_graphs):
        raise IndexError("graph id out of range")
    dev, B = store.device, len(ids)
    N = int((store.node_ptr_host[ids + 1] - store.node_ptr_host[ids]).sum())
    E = int((store.edge_ptr_host[ids + 1] - store.edge_ptr_host[ids]).sum())
    if store.pair_first is None:
        store.pair_first = torch.from_numpy(_pair_first(store.edge_ptr_host, store.edge_index.cpu().numpy())).to(dev)
    ids_dev = torch.from_numpy(ids).to(dev, non_blocking=True)
    ws = torch.empty(int(check(lib.pgnn_extract_pairs_workspace_bytes(B, N), "pgnn_extract_pairs_workspace_bytes")), dtype=torch.uint8, device=dev)
    offsets = torch.empty((6, B + 1), dtype=torch.int64, device=dev)
    if roots is not None and not torch.is_tensor(roots):
        roots = torch.from_numpy(np.ascontiguousarray(roots, dtype=np.int32)).to(dev, non_blocking=True)
    if roots is not None:
        roots = roots.to(torch.int32).contiguous()
        if roots.numel() != B:
            raise ValueError("one root per selected graph")
    check(lib.pgnn_extract_pairs(store.node_ptr.data_ptr(), store.edge_ptr.data_ptr(), store.edge_index.data_ptr(), store.num_edges,
                                 store.pair_first.data_ptr(), ids_dev.data_ptr(), B, N, None if roots is None else roots.data_ptr(),
                                 int(seed) & ((1 << 63) - 1), int(k), int(l1), int(l2), int(whole_graph), ws.data_ptr(), ws.numel(),
                                 offsets.data_ptr(), torch.cuda.current_stream(dev).cuda_stream), "pgnn_extract_pairs")
    return ids_dev, ws, offsets, N, E


class MoleculeStore:
    """Compact CSR-of-graphs for chem molecules (value ranges: chem/loader.py:22-51; all fit a byte).

    node_ptr / edge_ptr [G+1] int64; x [Nt,2] uint8; edge_index [2,Et] int32 graph-local; edge_attr [Et,2] uint8."""

    def __init__(self, node_ptr, edge_ptr, x, edge_index, edge_attr, device="cuda"):
        self.node_ptr_host = np.ascontiguousarray(node_ptr, dtype=np.int64)
        self.edge_ptr_host = np.ascontiguousarray(edge_ptr, dtype=np.int64)
        G = len(self.node_ptr_host) - 1
        if G < 0 or len(self.edge_ptr_host) != G + 1:
            raise ValueError("node_ptr and edge_ptr must both have num_graphs + 1 entries")
        Nt, Et = int(self.node_ptr_host[-1]), int(self.edge_ptr_host[-1])
        x, edge_index, edge_attr = np.asarray(x), np.asarray(edge_index), np.asarray(edge_attr)
        if x.shape != (Nt, 2) or edge_index.shape != (2, Et) or edge_attr.shape != (Et, 2):
            raise ValueError("store arrays do not match the prefix sums")
        if Nt and (x.min() < 0 or x.max() > 255) or Et and (edge_attr.min() < 0 or edge_attr.max() > 255):
            raise ValueError("atom / bond features must fit a byte")
        self.num_graphs, self.num_nodes, self.num_edges = G, Nt, Et
        self.device = torch.device(device)
        dev = self.device
        self.node_ptr = torch.from_numpy(self.node_ptr_host).to(dev)
        self.edge_ptr = torch.from_numpy(self.edge_ptr_host).to(dev)
        self.x = torch.from_numpy(np.ascontiguousarray(x, dtype=np.uint8)).to(dev)
        self.edge_index = torch.from_numpy(np.ascontiguousarray(edge_index, dtype=np.int32)).to(dev)
        self.edge_attr = torch.from_numpy(np.ascontiguousarray(edge_attr, dtype=np.uint8)).to(dev)
        self.pair_first = None    # built on first use by extract_pairs

    @classmethod
    def from_data_list(cls, data_list, device="cuda"):
        """data_list: objects with .x [n,2], .edge_index [2,e] (graph-local), .edge_attr [e,2] (the reference's Data)."""
        n = np.array([0] + [int(d.x.shape[0]) for d in data_list], dtype=np.int64)
        e = np.array([0] + [int(d.edge_index.shape[1]) for d in data_list], dtype=np.int64)
        cat = lambda xs, ax, shape: np.concatenate([np.asarray(a) for a in xs], axis=ax) if xs else np.zeros(shape, np.int64)
        return cls(np.cumsum(n), np.cumsum(e), cat([d.x for d in data_list], 0, (0, 2)),
                   cat([d.edge_index for d in data_list], 1, (2, 0)), cat([d.edge_attr for d in data_list], 0, (0, 2)), device)

    def batch_sizes(self, graph_ids_host):
        """(N, E) of the batch, from the host copy of the prefix sums (no device sync)."""
        ids = np.asarray(graph_ids_host, dtype=np.int64)
        if ids.size and (ids.min() < 0 or ids.max() >= self.num_graphs):
            raise IndexError("graph id out of range")
        return (int((self.node_ptr_host[ids + 1] - self.node_ptr_host[ids]).sum()),
                int((self.edge_ptr_host[ids + 1] - self.edge_ptr_host[ids]).sum()))

    def node_offsets_host(self, graph_ids_host):
        """Host copy of the collated batch's node_off [B+1] (what mask_atoms needs to size its outputs without a sync)."""
        ids = np.asarray(graph_ids_host, dtype=np.int64)
        return np.concatenate([[0], np.cumsum(self.node_ptr_host[ids + 1] - self.node_ptr_host[ids])]).astype(np.int64)

    def collate(self, graph_ids_host, graph_ids_dev=None):
        """-> namespace(x [N,2], edge_index [2,E], edge_attr [E,2], batch [N], node_off [B+1], edge_off [B+1], num_graphs),
        int64 CUDA tensors exactly as BatchMasking.from_data_list([dataset[i] for i in ids]) would hold them."""
        ids = np.ascontiguousarray(graph_ids_host, dtype=np.int64)
        N, E = self.batch_sizes(ids)
        B, dev = len(ids), self.device
        if graph_ids_dev is None:
            graph_ids_dev = torch.from_numpy(ids).to(dev, non_blocking=True)
        i64 = dict(dtype=torch.int64, device=dev)
        out = SimpleNamespace(x=torch.empty((N, 2), **i64), edge_index=torch.empty((2, E), **i64), edge_attr=torch.empty((E, 2), **i64),
                              batch=torch.empty((N,), **i64), node_off=torch.empty((B + 1,), **i64),
                              edge_off=torch.empty((B + 1,), **i64), num_graphs=B)
        check(lib.pgnn_collate_chem(self.node_ptr.data_ptr(), self.edge_ptr.data_ptr(), self.x.data_ptr(), self.edge_index.data_ptr(),
                                    self.num_edges, self.edge_attr.data_ptr(), graph_ids_dev.data_ptr(), B, out.node_off.data_ptr(),
                                    out.edge_off.data_ptr(), out.x.data_ptr(), out.edge_index.data_ptr(), out.edge_attr.data_ptr(),
                                    out.batch.data_ptr(), torch.cuda.current_stream(dev).cuda_stream), "pgnn_collate_chem")
        return out


def extract_substruct_context_pairs(store, graph_ids_host, k, l1, l2, roots=None, seed=0):
    """ExtractSubstructureContextPair(k, l1, l2) (chem/util.py:55-151; the script's defaults are k = num_layer, l1 = k - 1,
    l2 = l1 + csize: chem/pretrain_contextpred.py:145-150) applied to the molecules `graph_ids_host` of a MoleculeStore and
    collated as BatchSubstructContext.from_data_list does (chem/batch.py:141-210) -- on the device, three kernels, no
    networkx.  `roots`: graph-local root atoms (host array or device tensor, one per graph); None draws them from `seed`
    (a fresh value per step).  Returns the namespace SubstructContextStore.collate returns, plus `kept` = how many of the
    selected molecules have a context (the reference silently drops the others, chem/batch.py:168).  One 48-byte read-back
    sizes the views (the sizes are data dependent)."""
    ids_dev, ws, offsets, N, E = _extract(store, graph_ids_host, roots, seed, k, l1, l2, 0)
    B, dev = len(ids_dev), store.device
    i64 = dict(dtype=torch.int64, device=dev)
    xs, es, as_, cen = torch.empty((N, 2), **i64), torch.empty((2 * E,), **i64), torch.empty((E, 2), **i64), torch.empty((B,), **i64)
    xc, ec, ac = torch.empty((N, 2), **i64), torch.empty((2 * E,), **i64), torch.empty((E, 2), **i64)
    ov, seg, sizes = torch.empty((N,), **i64), torch.empty((N,), **i64), torch.empty((B,), **i64)
    check(lib.pgnn_extract_fill_chem(store.node_ptr.data_ptr(), store.edge_ptr.data_ptr(), store.x.data_ptr(), store.edge_index.data_ptr(),
                                     store.num_edges, store.edge_attr.data_ptr(), store.pair_first.data_ptr(), ids_dev.data_ptr(), B, N,
                                     ws.data_ptr(), offsets.data_ptr(), xs.data_ptr(), es.data_ptr(), as_.data_ptr(), cen.data_ptr(), xc.data_ptr(),
                                     ec.data_ptr(), ac.data_ptr(), ov.data_ptr(), seg.data_ptr(), sizes.data_ptr(),
                                     torch.cuda.current_stream(dev).cuda_stream), "pgnn_extract_fill_chem")
    ns, e_s, nc, e_c, ko, kept = (int(v) for v in offsets[:, B].tolist())      # the one host read-back
    return SimpleNamespace(x_substruct=xs[:ns], edge_index_substruct=es[:2 * e_s].view(2, e_s), edge_attr_substruct=as_[:e_s],
                           center_substruct_idx=cen[:kept], x_context=xc[:nc], edge_index_context=ec[:2 * e_c].view(2, e_c),
                           edge_attr_context=ac[:e_c], overlap_context_substruct_idx=ov[:ko], batch_overlapped_context=seg[:ko],
                           overlapped_context_size=sizes[:kept], num_graphs=kept, kept=kept)


def mask_edges_bio(batch, edge_off_host, mask_rate=0.15, seed=0):
    """MaskEdge (bio/util.py:46-104) on a batch collated by BioGraphStore.collate, on the device: adds `masked_edge_idx` [M],
    `mask_edge_label` [M,9], `mask_edge_off` [B+1] and overwrites both directions of the chosen bond pairs in `batch.edge_attr`
    with the mask vector.  `edge_off_host`: host copy of batch.edge_off (np.int64 [B+1])."""
    import ctypes
    off = np.ascontiguousarray(edge_off_host, dtype=np.int64)
    B = len(off) - 1
    M = int(check(lib.pgnn_mask_edges_bio_count(off.ctypes.data_as(ctypes.c_void_p), B, float(mask_rate)), "pgnn_mask_edges_bio_count"))
    dev = batch.edge_attr.device
    batch.masked_edge_idx = torch.empty((M,), dtype=torch.int64, device=dev)
    batch.mask_edge_label = torch.empty((M, 9), dtype=torch.float32, device=dev)
    batch.mask_edge_off = torch.empty((B + 1,), dtype=torch.int64, device=dev)
    check(lib.pgnn_mask_edges_bio(batch.edge_attr.data_ptr(), batch.edge_off.data_ptr(), B, float(mask_rate), int(seed) & ((1 << 63) - 1),
                                  batch.mask_edge_off.data_ptr(), batch.masked_edge_idx.data_ptr(), batch.mask_edge_label.data_ptr(),
                                  torch.cuda.current_stream(dev).cuda_stream), "pgnn_mask_edges_bio")
    return batch


def negative_edges(batch, edge_off_host, seed=0):
    """NegativeEdge (chem/util.py:22-52, bio/util.py:16-44) + BatchAE's offset (chem/batch.py:69-121, bio/batch.py:123-175) on a batch
    collated by MoleculeStore.collate or BioGraphStore.collate, on the device: adds `negative_edge_index` [2, M] (batch-global ids)
    and `negative_edge_off` [B+1].  Per graph of e columns, the first e/2 distinct valid pairs (all of them when e is odd) among
    5e candidates drawn as pgnn_negative_edges defines.  `edge_off_host`: host copy of batch.edge_off (np.int64 [B+1]) to size
    the output; M is data dependent, so one 8-byte read-back narrows the view.  `seed`: a fresh value per step."""
    import ctypes
    off = np.ascontiguousarray(edge_off_host, dtype=np.int64)
    B = len(off) - 1
    cap = int(check(lib.pgnn_negative_edges_capacity(off.ctypes.data_as(ctypes.c_void_p), B), "pgnn_negative_edges_capacity"))
    ei = batch.edge_index.contiguous()
    E, dev = int(ei.shape[1]), ei.device
    wsb = int(check(lib.pgnn_negative_edges_workspace_bytes(B, E, cap), "pgnn_negative_edges_workspace_bytes"))
    ws = torch.empty(wsb, dtype=torch.uint8, device=dev)
    out = torch.empty((2 * max(cap, 1),), dtype=torch.int64, device=dev)
    neg_off = torch.empty((B + 1,), dtype=torch.int64, device=dev)
    check(lib.pgnn_negative_edges(ei.data_ptr(), E, batch.node_off.data_ptr(), batch.edge_off.data_ptr(), B, int(seed) & ((1 << 63) - 1), cap,
                                  ws.data_ptr(), wsb, out.data_ptr(), neg_off.data_ptr(), torch.cuda.current_stream(dev).cuda_stream),
          "pgnn_negative_edges")
    M = int(neg_off[B])
    batch.negative_edge_index, batch.negative_edge_off = out[:2 * M].view(2, M), neg_off
    return batch


def mask_edges_chem(batch, num_edge_type=5):
    """The mask_edge=True half of MaskAtom (chem/util.py:243-272) on a batch that mask_atoms has processed: adds
    `connected_edge_indices` [Mc], `mask_edge_label` [Mc,2] and overwrites the attribute rows of every bond touching a masked
    atom with [num_edge_type, 0].  The list length is data dependent: one 8-byte read-back narrows the views."""
    dev = batch.x.device
    N, E, B = int(batch.x.shape[0]), int(batch.edge_index.shape[1]), int(batch.node_off.shape[0]) - 1
    M = int(batch.masked_atom_indices.shape[0])
    ws = torch.empty(int(check(lib.pgnn_mask_edges_chem_workspace_bytes(N, B), "pgnn_mask_edges_chem_workspace_bytes")), dtype=torch.uint8, device=dev)
    cap = E // 2 + B
    conn, labels = torch.empty((cap,), dtype=torch.int64, device=dev), torch.empty((cap, 2), dtype=torch.int64, device=dev)
    conn_off = torch.empty((B + 1,), dtype=torch.int64, device=dev)
    check(lib.pgnn_mask_edges_chem(batch.edge_index.data_ptr(), batch.edge_attr.data_ptr(), batch.edge_off.data_ptr(), B, N, E,
                                   batch.masked_atom_indices.data_ptr(), M, int(num_edge_type), ws.data_ptr(), ws.numel(), conn_off.data_ptr(),
                                   conn.data_ptr(), labels.data_ptr(), torch.cuda.current_stream(dev).cuda_stream), "pgnn_mask_edges_chem")
    total = int(conn_off[B])
    batch.connected_edge_indices, batch.mask_edge_label, batch.connected_edge_off = conn[:total], labels[:total], conn_off
    return batch


def mask_atoms(batch, node_off_host, mask_rate=0.15, seed=0, num_atom_type=119):
    """MaskAtom (chem/util.py:189-241, mask_edge=False) on a batch collated by MoleculeStore.collate, on the device: adds
    `masked_atom_indices` [M], `mask_node_label` [M,2], `mask_off` [B+1] to `batch` and overwrites the masked rows of
    `batch.x` with [num_atom_type, 0].  `node_off_host`: host copy of batch.node_off (np.int64 [B+1]; from
    MoleculeStore.node_offsets_host(ids), no device sync).  `seed`: a fresh value per step (the draw is a pure function of it)."""
    import ctypes
    off = np.ascontiguousarray(node_off_host, dtype=np.int64)
    B = len(off) - 1
    M = int(check(lib.pgnn_mask_atoms_count(off.ctypes.data_as(ctypes.c_void_p), B, float(mask_rate)), "pgnn_mask_atoms_count"))
    dev = batch.x.device
    i64 = dict(dtype=torch.int64, device=dev)
    batch.masked_atom_indices, batch.mask_node_label = torch.empty((M,), **i64), torch.empty((M, 2), **i64)
    batch.mask_off = torch.empty((B + 1,), **i64)
    check(lib.pgnn_mask_atoms(batch.x.data_ptr(), batch.node_off.data_ptr(), B, float(mask_rate), int(num_atom_type), int(seed) & ((1 << 63) - 1),
                              batch.mask_off.data_ptr(), batch.masked_atom_indices.data_ptr(), batch.mask_node_label.data_ptr(),
                              torch.cuda.current_stream(dev).cuda_stream), "pgnn_mask_atoms")
    return batch


class IndexLists:
    """Per-graph lists of graph-local node ids held in HBM (list_ptr [G+1] int64, values int32): the centre node of a
    substructure, the overlap nodes of a context graph, a PPI ego graph's centre node."""

    def __init__(self, lists, device="cuda"):
        lens = np.array([0] + [len(l) for l in lists], dtype=np.int64)
        self.ptr_host = np.cumsum(lens)
        vals = np.concatenate([np.asarray(l, dtype=np.int32) for l in lists]) if len(lists) and self.ptr_host[-1] else np.zeros(0, np.int32)
        self.device = torch.device(device)
        self.ptr = torch.from_numpy(self.ptr_host).to(self.device)
        self.values = torch.from_numpy(np.ascontiguousarray(vals, dtype=np.int32)).to(self.device)

    def collate(self, ids_host, ids_dev, add=None, want_seg=False, want_sizes=False):
        """-> (out [K], seg [K] | None, sizes [B] | None): entries offset by add[i] (a device int64 [>= B] tensor, e.g. node_off)."""
        ids = np.asarray(ids_host, dtype=np.int64)
        B, K = len(ids), int((self.ptr_host[ids + 1] - self.ptr_host[ids]).sum())
        i64 = dict(dtype=torch.int64, device=self.device)
        out, off = torch.empty((K,), **i64), torch.empty((B + 1,), **i64)
        seg = torch.empty((K,), **i64) if want_seg else None
        sizes = torch.empty((B,), **i64) if want_sizes else None
        p = lambda t: None if t is None else t.data_ptr()
        check(lib.pgnn_collate_lists(self.ptr.data_ptr(), self.values.data_ptr(), ids_dev.data_ptr(), B, p(add), off.data_ptr(), out.data_ptr(),
                                     p(seg), p(sizes), torch.cuda.current_stream(self.device).cuda_stream), "pgnn_collate_lists")
        return out, seg, sizes


class SubstructContextStore:
    """Pre-extracted (substructure, context) graph pairs in HBM and BatchSubstructContext.from_data_list on the device
    (chem/batch.py:141-210): two molecule stores plus the centre / overlap index lists of every pair."""

    def __init__(self, substruct: "MoleculeStore", context: "MoleculeStore", center_idx, overlap_idx):
        self.substruct, self.context = substruct, context
        dev = substruct.device
        self.center = IndexLists([[int(c)] for c in center_idx], dev)
        self.overlap = IndexLists(overlap_idx, dev)

    def collate(self, graph_ids_host):
        ids = np.ascontiguousarray(graph_ids_host, dtype=np.int64)
        ids_dev = torch.from_numpy(ids).to(self.substruct.device, non_blocking=True)
        s = self.substruct.collate(ids, ids_dev)
        c = self.context.collate(ids, ids_dev)
        center, _, _ = self.center.collate(ids, ids_dev, add=s.node_off)
        overlap, seg, sizes = self.overlap.collate(ids, ids_dev, add=c.node_off, want_seg=True, want_sizes=True)
        return SimpleNamespace(x_substruct=s.x, edge_index_substruct=s.edge_index, edge_attr_substruct=s.edge_attr, center_substruct_idx=center,
                               x_context=c.x, edge_index_context=c.edge_index, edge_attr_context=c.edge_attr,
                               overlap_context_substruct_idx=overlap, batch_overlapped_context=seg, overlapped_context_size=sizes,
                               num_graphs=len(ids))


class BioGraphStore:
    """PPI ego graphs in HBM (node counts, int32 graph-local edge_index, the 9 binary edge attributes packed into a uint16)
    and bio/batch.py:17-50 on the device: x [N,1] float ones, edge_index + node offset, edge_attr [E,9] float, batch,
    center_node_idx + node offset."""

    def __init__(self, num_nodes, edge_index_list, edge_attr_list, center_idx, device="cuda"):
        n = np.array([0] + [int(v) for v in num_nodes], dtype=np.int64)
        e = np.array([0] + [int(ei.shape[1]) for ei in edge_index_list], dtype=np.int64)
        self.node_ptr_host, self.edge_ptr_host = np.cumsum(n), np.cumsum(e)
        self.num_graphs, self.num_edges = len(num_nodes), int(self.edge_ptr_host[-1])
        self.device = torch.device(device)
        ei = np.concatenate([np.asarray(a, dtype=np.int32) for a in edge_index_list], axis=1) if self.num_edges else np.zeros((2, 0), np.int32)
        ea = np.concatenate([np.asarray(a) for a in edge_attr_list], axis=0) if self.num_edges else np.zeros((0, 9))
        if ea.size and not np.isin(ea, (0, 1)).all():
            raise ValueError("bio edge attributes must be 0/1 (bio/loader.py:57-75)")
        bits = (ea.astype(np.uint16) << np.arange(9, dtype=np.uint16)).sum(axis=1).astype(np.uint16)
        dev = self.device
        self.node_ptr, self.edge_ptr = torch.from_numpy(self.node_ptr_host).to(dev), torch.from_numpy(self.edge_ptr_host).to(dev)
        self.edge_index = torch.from_numpy(np.ascontiguousarray(ei)).to(dev)
        self.edge_bits = torch.from_numpy(bits.view(np.int16).copy()).to(dev)   # same 16 bits; torch has no uint16 arithmetic we need
        self.center = IndexLists([[int(c)] for c in center_idx], dev)
        self.pair_first = None

    def extract_context(self, graph_ids_host, l1, center=True, seed=0):
        """bio ExtractSubstructureContextPair(l1, center) + BatchSubstructContext.from_data_list (bio/util.py:123-205,
        bio/batch.py:196-265) on the device: the substructure side is the ordinary collation of the whole ego graphs, the
        context side holds the nodes further than l1 hops from the root node, every one of them an overlap node.  The root is
        the centre node with center=True; with center=False (bio/pretrain_contextpred.py's default) it is a uniform draw per
        graph, pgnn_extract_pairs' splitmix64(seed, batch slot) mod n (bio/util.py:159-164 uses random.sample; `seed`: a fresh
        value per step).  center_substruct_idx is the ego centre either way (bio/util.py:172).  Graphs without a context are
        dropped by the reference; here that is reported (`kept`) and raised if it happens, because the substructure side would
        have to be re-collated without them."""
        ids = np.ascontiguousarray(graph_ids_host, dtype=np.int64)
        out = self.collate(ids)
        # one centre per graph: list_ptr = arange
        roots = self.center.values[torch.from_numpy(ids).to(self.device)] if center else None
        ids_dev, ws, offsets, N, E = _extract(self, ids, roots, seed if not center else 0, 0, l1, 0, 1)
        B, dev = len(ids), self.device
        i64, f32 = dict(dtype=torch.int64, device=dev), dict(dtype=torch.float32, device=dev)
        xc, ec, ac = torch.empty((N, 1), **f32), torch.empty((2 * E,), **i64), torch.empty((E, 9), **f32)
        ov, seg, sizes = torch.empty((N,), **i64), torch.empty((N,), **i64), torch.empty((B,), **i64)
        check(lib.pgnn_extract_fill_bio(self.node_ptr.data_ptr(), self.edge_ptr.data_ptr(), self.edge_index.data_ptr(), self.num_edges,
                                        self.edge_bits.data_ptr(), self.pair_first.data_ptr(), ids_dev.data_ptr(), B, N, ws.data_ptr(),
                                        offsets.data_ptr(), xc.data_ptr(), ec.data_ptr(), ac.data_ptr(), ov.data_ptr(), seg.data_ptr(),
                                        sizes.data_ptr(), torch.cuda.current_stream(dev).cuda_stream), "pgnn_extract_fill_bio")
        _, _, nc, e_c, ko, kept = (int(v) for v in offsets[:, B].tolist())
        if kept != B:
            raise ValueError("%d of %d ego graphs have no node further than l1 = %d hops from their root" % (B - kept, B, l1))
        return SimpleNamespace(x_substruct=out.x, edge_index_substruct=out.edge_index, edge_attr_substruct=out.edge_attr,
                               center_substruct_idx=out.center_node_idx, x_context=xc[:nc], edge_index_context=ec[:2 * e_c].view(2, e_c),
                               edge_attr_context=ac[:e_c], overlap_context_substruct_idx=ov[:ko], batch_overlapped_context=seg[:ko],
                               overlapped_context_size=sizes[:kept], num_graphs=kept, kept=kept)

    def collate(self, graph_ids_host):
        ids = np.ascontiguousarray(graph_ids_host, dtype=np.int64)
        if ids.size and (ids.min() < 0 or ids.max() >= self.num_graphs):
            raise IndexError("graph id out of range")
        N = int((self.node_ptr_host[ids + 1] - self.node_ptr_host[ids]).sum())
        E = int((self.edge_ptr_host[ids + 1] - self.edge_ptr_host[ids]).sum())
        B, dev = len(ids), self.device
        ids_dev = torch.from_numpy(ids).to(dev, non_blocking=True)
        i64, f32 = dict(dtype=torch.int64, device=dev), dict(dtype=torch.float32, device=dev)
        out = SimpleNamespace(x=torch.empty((N, 1), **f32), edge_index=torch.empty((2, E), **i64), edge_attr=torch.empty((E, 9), **f32),
                              batch=torch.empty((N,), **i64), node_off=torch.empty((B + 1,), **i64), edge_off=torch.empty((B + 1,), **i64),
                              num_graphs=B)
        check(lib.pgnn_collate_bio(self.node_ptr.data_ptr(), self.edge_ptr.data_ptr(), self.edge_index.data_ptr(), self.num_edges,
                                   self.edge_bits.data_ptr(), ids_dev.data_ptr(), B, out.node_off.data_ptr(), out.edge_off.data_ptr(),
                                   out.x.data_ptr(), out.edge_index.data_ptr(), out.edge_attr.data_ptr(), out.batch.data_ptr(),
                                   torch.cuda.current_stream(dev).cuda_stream), "pgnn_collate_bio")
        out.center_node_idx, _, _ = self.center.collate(ids, ids_dev, add=out.node_off)
        return out


class PackedHostBatch:
    """A batch dict packed into ONE pinned host buffer (fields 16-byte aligned), built once per batch by BatchStager.pack."""

    def __init__(self, buf, fields):
        self.buf, self.fields = buf, fields  # fields: name -> (byte offset, byte length, dtype, shape)
        self.nbytes = int(buf.numel())


class BatchStager:
    """Host -> device staging of batches with the copy off the critical path.

    The reference moves a batch with one `.to(device)` per tensor right before the step (chem/pretrain_masking.py:47,
    `batch = batch.to(device)`), i.e. five small synchronous-looking copies in front of the first kernel.  Here a batch is ONE
    pinned buffer and ONE `cudaMemcpyAsync` on a side stream into one of `slots` device buffers, so the copy of batch i+1 runs
    under the kernels of batch i:

        t = stager.submit(packed[0])
        for i in range(steps):
            b = stager.take(t)                       # dict of device views; the compute stream waits for the copy
            loss = train_step(b)                      # enqueue the step
            t = stager.submit(packed[i + 1])         # prefetch under the step just enqueued
            log(loss.item())

    A slot is overwritten only after the work enqueued on the batch that last occupied it (everything up to the following
    `take`) has finished: the side stream waits on an event of the compute stream, so no host synchronisation is assumed."""

    def __init__(self, device, slots=2):
        self.device = torch.device(device)
        self.cuda = self.device.type == "cuda"
        self.slots = int(slots)
        self.dev = [None] * self.slots          # device buffers, grown on demand
        self.ready = [None] * self.slots        # copy finished (side stream)
        self.release = [None] * self.slots      # consumers enqueued (compute stream)
        self.stream = torch.cuda.Stream(self.device) if self.cuda else None
        self._next, self._last_taken = 0, None

    def pack(self, batch):
        fields, off = {}, 0
        for k, v in batch.items():
            if not torch.is_tensor(v):
                continue
            v = v.contiguous()
            nb = v.numel() * v.element_size()
            fields[k] = (off, nb, v.dtype, tuple(v.shape), v)
            off = (off + nb + 15) // 16 * 16
        buf = torch.empty(max(off, 16), dtype=torch.uint8)
        if self.cuda:
            buf = buf.pin_memory()
        out = {}
        for k, (o, nb, dt, shape, v) in fields.items():
            if nb:
                buf[o:o + nb].copy_(v.view(-1).view(torch.uint8))
            out[k] = (o, nb, dt, shape)
        return PackedHostBatch(buf, out)

    def submit(self, packed):
        """Start copying `packed` into the next slot; returns a ticket for take()."""
        s = self._next
        self._next = (s + 1) % self.slots
        if self.dev[s] is None or self.dev[s].numel() < packed.nbytes:
            self.dev[s] = torch.empty(max(packed.nbytes, 1 << 20), dtype=torch.uint8, device=self.device)
            if self.cuda:  # the allocator may hand back a block whose previous user is still running on the compute stream
                self.stream.wait_stream(torch.cuda.current_stream(self.device))
        if self.cuda:
            if s == self._last_taken:  # the slot's batch is still the one in use: everything enqueued so far must finish first
                self.release[s] = torch.cuda.Event()
                self.release[s].record(torch.cuda.current_stream(self.device))
                self._last_taken = None
            if self.release[s] is not None:
                self.stream.wait_event(self.release[s])
            with torch.cuda.stream(self.stream):
                self.dev[s][:packed.nbytes].copy_(packed.buf, non_blocking=True)
                self.ready[s] = torch.cuda.Event()
                self.ready[s].record(self.stream)
        else:
            self.dev[s][:packed.nbytes].copy_(packed.buf)
        return (s, packed)

    def take(self, ticket):
        """-> dict of device tensors (views of the slot).  Everything enqueued on the previous batch is now 'released'."""
        s, packed = ticket
        if self.cuda:
            cur = torch.cuda.current_stream(self.device)
            if self._last_taken is not None and self._last_taken != s:
                self.release[self._last_taken] = torch.cuda.Event()
                self.release[self._last_taken].record(cur)
            cur.wait_event(self.ready[s])
        self._last_taken = s
        d = self.dev[s]
        return {k: (d[o:o + nb].view(dt).view(shape) if nb else torch.empty(shape, dtype=dt, device=self.device))
                for k, (o, nb, dt, shape) in packed.fields.items()}
