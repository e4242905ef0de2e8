"""Seeded synthetic batches shaped like the reference's inputs (SURVEY.md §8(d)).

No dataset or rdkit is available, so every test / bench input comes from here.
The layouts follow the reference's collation code exactly:

* chem molecules: ``x [N,2] int64`` (atom type, chirality), ``edge_index [2,E] int64`` with both
  directions of a bond adjacent and carrying the same ``edge_attr [E,2] int64``
  (/root/reference/chem/loader.py:53-100), node ids offset per graph and a sorted ``batch`` vector
  (/root/reference/chem/batch.py:17-52).
* MaskAtom: per graph ``int(n*rate + 1)`` distinct atoms, labels saved, ``x`` row overwritten with
  ``[119, 0]`` (/root/reference/chem/util.py:229-241); optional bond masking with type 5
  (/root/reference/chem/util.py:243-272).
* substructure/context pairs (/root/reference/chem/batch.py:141-210).
* bio PPI ego graphs: ``x [N,1] float32`` ones, ``edge_attr [E,9] float32`` 0/1 with cols 7,8 zero
  (/root/reference/bio/loader.py:47-75), ``center_node_idx`` offset per graph
  (/root/reference/bio/batch.py:17-50).

numpy's PCG64 is used (not torch's generator) so the same seed gives the same tensors on every
machine and torch build.
"""
from __future__ import annotations

import numpy as np
import torch

NUM_ATOM_TYPE_MASK = 119   # chem/pretrain_masking.py:122
NUM_BOND_TYPE_MASK = 5     # chem/pretrain_masking.py:122 (num_edge_type=5)


def _t(a, dtype=torch.int64):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dtype)


def _molecule(rng, n, extra, tree_only=False):
    """One molecule's undirected bond list as (u, v) with u != v. Spanning tree + `extra` chords."""
    parent = (rng.random(n - 1) * np.arange(1, n)).astype(np.int64)  # node k attaches to a node < k
    u = np.arange(1, n, dtype=np.int64)
    v = parent
    if not tree_only and extra > 0:
        a = rng.integers(0, n, size=extra)
        b = (a + 1 + rng.integers(0, n - 1, size=extra)) % n  # never a self pair
        u = np.concatenate([u, a])
        v = np.concatenate([v, b])
    return u, v


def _directed(u, v, attr):
    """Both directions adjacent, identical attributes (chem/loader.py:83-86)."""
    m = len(u)
    ei = np.empty((2, 2 * m), dtype=np.int64)
    ei[0, 0::2], ei[1, 0::2] = u, v
    ei[0, 1::2], ei[1, 1::2] = v, u
    ea = np.repeat(attr, 2, axis=0)
    return ei, ea


def zinc_batch(num_graphs: int, seed: int, n_lo: int = 18, n_hi: int = 28, extra: int = 3,
               tree_only: bool = False):
    """ZINC-shaped batch. Returns dict of CPU tensors: x, edge_index, edge_attr, batch, ptr."""
    rng = np.random.default_rng(seed)
    xs, eis, eas, bs = [], [], [], []
    ptr = [0]
    off = 0
    for g in range(num_graphs):
        n = int(rng.integers(n_lo, n_hi + 1))
        u, v = _molecule(rng, n, extra, tree_only)
        attr = np.stack([rng.integers(0, 4, size=len(u)), rng.integers(0, 3, size=len(u))], axis=1)
        ei, ea = _directed(u, v, attr)
        xs.append(np.stack([rng.integers(0, 119, size=n), rng.integers(0, 3, size=n)], axis=1))
        eis.append(ei + off)
        eas.append(ea)
        bs.append(np.full(n, g, dtype=np.int64))
        off += n
        ptr.append(off)
    if num_graphs == 0:
        return dict(x=torch.zeros(0, 2, dtype=torch.int64), edge_index=torch.zeros(2, 0, dtype=torch.int64),
                    edge_attr=torch.zeros(0, 2, dtype=torch.int64), batch=torch.zeros(0, dtype=torch.int64),
                    ptr=torch.zeros(1, dtype=torch.int64), num_graphs=0)
    return dict(x=_t(np.concatenate(xs)), edge_index=_t(np.concatenate(eis, axis=1)),
                edge_attr=_t(np.concatenate(eas)), batch=_t(np.concatenate(bs)), ptr=_t(np.array(ptr)),
                num_graphs=num_graphs)


def mask_atoms(batch: dict, seed: int, rate: float = 0.15, mask_edge: bool = False) -> dict:
    """Apply MaskAtom semantics per graph, in place on a copy; adds the BatchMasking keys."""
    rng = np.random.default_rng(seed + 7919)
    out = {k: (v.clone() if torch.is_tensor(v) else v) for k, v in batch.items()}
    ptr = batch["ptr"].numpy()
    idx = []
    for g in range(len(ptr) - 1):
        n = int(ptr[g + 1] - ptr[g])
        k = int(n * rate + 1)
        idx.append(ptr[g] + rng.choice(n, size=k, replace=False))
    idx = np.concatenate(idx) if idx else np.zeros(0, dtype=np.int64)
    out["masked_atom_indices"] = _t(idx)
    out["mask_node_label"] = out["x"][out["masked_atom_indices"]].clone()
    out["x"][out["masked_atom_indices"]] = torch.tensor([NUM_ATOM_TYPE_MASK, 0])
    if mask_edge:
        ei = out["edge_index"].numpy()
        hit = np.isin(ei[0], idx) | np.isin(ei[1], idx)
        conn = np.nonzero(hit)[0]
        conn_pairs = conn[conn % 2 == 0]  # one id per undirected bond (first of the adjacent pair)
        out["connected_edge_indices"] = _t(conn_pairs)
        out["mask_edge_label"] = out["edge_attr"][out["connected_edge_indices"]].clone()
        both = np.concatenate([conn_pairs, conn_pairs + 1])
        out["edge_attr"][_t(both)] = torch.tensor([NUM_BOND_TYPE_MASK, 0])
    return out


def finetune_batch(num_graphs: int, seed: int, num_tasks: int = 12, missing_rate: float = 0.2) -> dict:
    """chem/finetune.py's input: a zinc_batch plus `y [B, T] int64` in {-1, 0, +1} (chem/loader.py's MoleculeNet labels: +-1 a
    label, 0 a missing one, about `missing_rate` of them)."""
    out = zinc_batch(num_graphs, seed)
    rng = np.random.default_rng(seed + 2750159)
    y = np.where(rng.random((num_graphs, num_tasks)) < 0.5, 1, -1)
    y[rng.random((num_graphs, num_tasks)) < missing_rate] = 0
    out["y"] = _t(y)
    return out


def substruct_context_batch(num_graphs: int, seed: int) -> dict:
    """Config 3 (chem/pretrain_contextpred.py): substructure graphs + context graphs + overlap ids."""
    sub = zinc_batch(num_graphs, seed * 2 + 1, n_lo=12, n_hi=22)
    ctx = zinc_batch(num_graphs, seed * 2 + 2, n_lo=4, n_hi=14, tree_only=True)
    rng = np.random.default_rng(seed + 104729)
    sp, cp = sub["ptr"].numpy(), ctx["ptr"].numpy()
    center = sp[:-1] + np.array([rng.integers(0, sp[g + 1] - sp[g]) for g in range(num_graphs)], dtype=np.int64)
    ov, ovb = [], []
    for g in range(num_graphs):
        nc = int(cp[g + 1] - cp[g])
        k = int(rng.integers(1, min(4, nc) + 1))
        ov.append(cp[g] + rng.choice(nc, size=k, replace=False))
        ovb.append(np.full(k, g, dtype=np.int64))
    return dict(x_substruct=sub["x"], edge_index_substruct=sub["edge_index"], edge_attr_substruct=sub["edge_attr"],
                center_substruct_idx=_t(center),
                x_context=ctx["x"], edge_index_context=ctx["edge_index"], edge_attr_context=ctx["edge_attr"],
                overlap_context_substruct_idx=_t(np.concatenate(ov)),
                batch_overlapped_context=_t(np.concatenate(ovb)),
                overlapped_context_size=_t(np.array([len(o) for o in ov])), num_graphs=num_graphs)


def ppi_batch(num_graphs: int, seed: int, n_lo: int = 400, n_hi: int = 600, pairs_per_node: int = 5,
              num_tasks: int = 5000, target_rate: float = 0.05) -> dict:
    """Config 4 (bio/pretrain_supervised.py): PPI-ego-shaped graphs."""
    rng = np.random.default_rng(seed)
    eis, eas, bs, ns = [], [], [], []
    off = 0
    ptr = [0]
    for g in range(num_graphs):
        n = int(rng.integers(n_lo, n_hi + 1))
        m = pairs_per_node * n
        a = rng.integers(0, n, size=m)
        b = (a + 1 + rng.integers(0, n - 1, size=m)) % n
        attr = np.zeros((m, 9), dtype=np.float32)
        attr[:, :7] = (rng.random((m, 7)) < 0.3)
        ei, ea = _directed(a, b, attr)
        eis.append(ei + off)
        eas.append(ea)
        bs.append(np.full(n, g, dtype=np.int64))
        ns.append(n)
        off += n
        ptr.append(off)
    ptr = np.array(ptr)
    y = (rng.random((num_graphs, num_tasks)) < target_rate).astype(np.int64)
    return dict(x=torch.ones(off, 1, dtype=torch.float32), edge_index=_t(np.concatenate(eis, axis=1)),
                edge_attr=_t(np.concatenate(eas), torch.float32), batch=_t(np.concatenate(bs)),
                center_node_idx=_t(ptr[:-1]), ptr=_t(ptr), go_target_pretrain=_t(y.reshape(-1)),
                num_graphs=num_graphs)


def ppi_graphs(batch: dict):
    """Per-graph (num_nodes, edge_index [2,e] graph-LOCAL, edge_attr [e,9]) numpy arrays of a ppi_batch, and its edge offsets
    [B+1] (np.int64): the form a BioDataset holds before collation."""
    ptr = batch["ptr"].numpy()
    ei, ea = batch["edge_index"].numpy(), batch["edge_attr"].numpy()
    owner = np.searchsorted(ptr, ei[0], side="right") - 1  # edges are emitted graph by graph
    eptr = np.searchsorted(owner, np.arange(len(ptr))).astype(np.int64)
    graphs = [(int(ptr[g + 1] - ptr[g]), ei[:, eptr[g]:eptr[g + 1]] - ptr[g], ea[eptr[g]:eptr[g + 1]]) for g in range(len(ptr) - 1)]
    return graphs, eptr


def splitmix64(seed: int, idx) -> np.ndarray:
    """The library's defined draw (csrc/common.cuh): the 64-bit key of each index in `idx` under `seed`, as np.uint64."""
    with np.errstate(over="ignore"):
        z = np.uint64(int(seed) & 0xFFFFFFFFFFFFFFFF) + (np.asarray(idx).astype(np.uint64) + np.uint64(1)) * np.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return z ^ (z >> np.uint64(31))


def bio_masking_batch(num_graphs: int, seed: int, mask_rate: float = 0.15, one_direction: bool = False, **ppi_kw) -> dict:
    """bio/pretrain_masking.py's input: a ppi_batch after MaskEdge (bio/util.py:46-104) and bio BatchMasking (bio/batch.py:95-96):
    `masked_edge_idx` [M] (offset by the running edge count), `mask_edge_label` [M,9] (the edge's attribute row: multi-hot,
    ties and all-zero rows included) and `edge_attr` with both columns of every masked pair set to [0,...,0,1].  The choice is
    the one data.mask_edges_bio makes on the device under the same seed: per graph the int(e/2 * rate + 1) column pairs with the
    smallest splitmix64(seed, first column) keys, ties by index.  one_direction: keep one of the two directed columns of every
    bond first (one_direction_only); MaskEdge then masks column pairs that are two different bonds."""
    b = ppi_batch(num_graphs, seed, **ppi_kw)
    if one_direction:
        b = one_direction_only(b, seed)
    _, eoff = ppi_graphs(b)
    idx = []
    for g in range(num_graphs):
        e0, m = int(eoff[g]), int(eoff[g + 1] - eoff[g]) // 2
        k = min(int(m * mask_rate + 1), m) if m > 0 else 0      # bio/util.py:78-80
        cols = e0 + 2 * np.arange(m, dtype=np.int64)
        idx.append(np.sort(cols[np.lexsort((cols, splitmix64(seed, cols)))[:k]]))
    idx = _t(np.concatenate(idx) if idx else np.zeros(0, np.int64))
    ea = b["edge_attr"].clone()
    b["masked_edge_idx"], b["mask_edge_label"] = idx, ea[idx].clone()
    mask = torch.zeros(9)
    mask[8] = 1.0                                               # bio/util.py:98-102
    ea[idx], ea[idx + 1] = mask, mask
    b["edge_attr"] = ea
    return b


def bio_context_batch(num_graphs: int, seed: int, l1: int = 1, **ppi_kw) -> dict:
    """bio/pretrain_contextpred.py's input with the script's defaults (l1 = 1, center = 0): ExtractSubstructureContextPair
    (bio/util.py:123-205) per ppi_batch graph and BatchSubstructContext (bio/batch.py:196-265).  The substructure side is the
    whole ego graph and center_substruct_idx its centre node.  The context holds the nodes further than l1 hops from a root drawn
    per graph as BioGraphStore.extract_context(center=False, seed) draws it on the device (splitmix64(seed, slot) mod n), in
    the library's defined order: nodes ascending, the first pair of every bond (networkx keeps one edge per node pair) in
    source order with both directions adjacent, the self-loop / mask columns zeroed (bio/loader.py:60-62), every node an
    overlap node."""
    from scipy.sparse import csr_matrix
    from scipy.sparse.csgraph import shortest_path
    b = ppi_batch(num_graphs, seed, **ppi_kw)
    graphs, _ = ppi_graphs(b)
    xs, eis, eas, ovs, segs, sizes, cc = [], [], [], [], [], [], 0
    for g, (n, ei, ea) in enumerate(graphs):
        root = int(splitmix64(seed, g) % np.uint64(n))
        u, v = ei[0, 0::2], ei[1, 0::2]
        first = np.zeros(len(u), bool)
        first[np.unique(np.minimum(u, v) * n + np.maximum(u, v), return_index=True)[1]] = True
        adj = csr_matrix((np.ones(int(first.sum())), (u[first], v[first])), shape=(n, n))
        ctx = shortest_path(adj, directed=False, unweighted=True, indices=root) > max(int(l1), 0)
        nc = int(ctx.sum())
        if nc == 0:
            raise ValueError("an ego graph has no node further than l1 = %d hops from its root" % l1)
        new = np.cumsum(ctx) - 1
        p = np.nonzero(first & ctx[u] & ctx[v])[0]
        pe = np.empty((2, 2 * len(p)), np.int64)
        pe[0, 0::2], pe[1, 0::2] = new[u[p]], new[v[p]]
        pe[0, 1::2], pe[1, 1::2] = new[v[p]], new[u[p]]
        pa = np.repeat(ea[2 * p], 2, axis=0)
        pa[:, 7:] = 0
        xs.append(np.ones((nc, 1), np.float32))
        eis.append(pe + cc)
        eas.append(pa)
        ovs.append(cc + np.arange(nc, dtype=np.int64))
        segs.append(np.full(nc, g, np.int64))
        sizes.append(nc)
        cc += nc
    cat = lambda a, axis=0: np.concatenate(a, axis=axis)
    return dict(x_substruct=b["x"], edge_index_substruct=b["edge_index"], edge_attr_substruct=b["edge_attr"],
                center_substruct_idx=b["center_node_idx"], x_context=_t(cat(xs), torch.float32), edge_index_context=_t(cat(eis, 1)),
                edge_attr_context=_t(cat(eas), torch.float32), overlap_context_substruct_idx=_t(cat(ovs)), batch_overlapped_context=_t(cat(segs)),
                overlapped_context_size=_t(np.array(sizes)), num_graphs=num_graphs)


def split_graphs(batch: dict):
    """Per-graph (x [n,2], edge_index [2,e] graph-LOCAL, edge_attr [e,2]) numpy arrays of a zinc_batch: the form a dataset
    holds before collation (chem/loader.py:53-100 builds one such Data per molecule)."""
    ptr = batch["ptr"].numpy()
    x, ei, ea = batch["x"].numpy(), batch["edge_index"].numpy(), batch["edge_attr"].numpy()
    owner = np.searchsorted(ptr, ei[0], side="right") - 1  # edges are emitted graph by graph
    eptr = np.searchsorted(owner, np.arange(len(ptr)))
    return [(x[ptr[g]:ptr[g + 1]], ei[:, eptr[g]:eptr[g + 1]] - ptr[g], ea[eptr[g]:eptr[g + 1]]) for g in range(len(ptr) - 1)]


def one_direction_only(batch: dict, seed: int, keys=("edge_index", "edge_attr")) -> dict:
    """Asymmetric variant of a batch: of every bond's two adjacent directed edges (u,v),(v,u) keep exactly one, chosen at
    random.  The reference never feeds such a graph (chem/loader.py:83-86 always emits both directions), but only on it
    does a swapped target/source — aggregation onto edge_index[1] instead of edge_index[0] — change GIN/GCN/GraphSAGE
    results (SURVEY.md 8(c)); the parity tests use it to pin the direction convention of every kernel."""
    rng = np.random.default_rng(seed + 15485863)
    out = dict(batch)
    ei = batch[keys[0]]
    m = ei.shape[1] // 2
    keep = _t(2 * np.arange(m) + rng.integers(0, 2, size=m))
    out[keys[0]] = ei[:, keep].contiguous()
    out[keys[1]] = batch[keys[1]][keep].contiguous()
    return out


def edge_offsets(batch: dict) -> np.ndarray:
    """[B+1] np.int64 edge offsets of a zinc_batch / ppi_batch (edges are emitted graph by graph)."""
    ptr, ei = batch["ptr"].numpy(), batch["edge_index"].numpy()
    owner = np.searchsorted(ptr, ei[0], side="right") - 1
    return np.searchsorted(owner, np.arange(len(ptr))).astype(np.int64)


def negative_edge_index(edge_index, node_off, edge_off, seed: int) -> np.ndarray:
    """NegativeEdge (chem/util.py:22-52) per graph + BatchAE's node offset, with the draw data.negative_edges makes on the device:
    candidate j of graph g is (splitmix64(seed, 2 (5 e0 + j)) mod n, splitmix64(seed, 2 (5 e0 + j) + 1) mod n), e0 = edge_off[g],
    j < 5e.  The reference's loop keeps, in candidate order, the first occurrence of every valid pair (endpoints differ, not a
    directed column of the graph) and stops at e/2 of them when e is even; restated over the whole batch at once: np.unique's first
    occurrences, then a per-graph cumulative count.  -> [2, M] int64 (batch-global ids)."""
    ei = np.asarray(edge_index, dtype=np.int64)
    node_off, edge_off = np.asarray(node_off, dtype=np.int64), np.asarray(edge_off, dtype=np.int64)
    n, e = np.diff(node_off), np.diff(edge_off)
    B = len(n)
    K = np.where((n > 0) & (e > 0), 5 * e, 0)
    if K.sum() == 0:
        return np.zeros((2, 0), np.int64)
    g = np.repeat(np.arange(B), K)
    j = np.arange(int(K.sum()), dtype=np.int64) - np.repeat(np.cumsum(K) - K, K)
    c = 2 * (5 * edge_off[g] + j)
    ng = n[g].astype(np.uint64)
    a = (splitmix64(seed, c) % ng).astype(np.int64)
    b = (splitmix64(seed, c + 1) % ng).astype(np.int64)
    W = int(n.max()) + 1
    key = (g * W + a) * W + b
    eg = np.repeat(np.arange(B), e)
    u, v = ei[0] - node_off[eg], ei[1] - node_off[eg]
    inside = (u >= 0) & (u < n[eg]) & (v >= 0) & (v < n[eg])
    ekey = (eg[inside] * W + u[inside]) * W + v[inside]
    cand = np.nonzero((a != b) & ~np.isin(key, ekey))[0]
    _, first = np.unique(key[cand], return_index=True)
    keep = np.sort(cand[first])
    kg = g[keep]
    rank = np.arange(len(keep)) - np.searchsorted(kg, kg)          # position among the graph's accepted pairs
    keep = keep[(e[kg] % 2 == 1) | (rank < e[kg] // 2)]
    return np.stack([node_off[g[keep]] + a[keep], node_off[g[keep]] + b[keep]])


def edgepred_batch(num_graphs: int, seed: int, **zinc_kw) -> dict:
    """chem/pretrain_edgepred.py's input: a zinc_batch after NegativeEdge and BatchAE (chem/batch.py:69-121), the negatives drawn
    as data.negative_edges draws them under `seed`."""
    b = zinc_batch(num_graphs, seed, **zinc_kw)
    b["edge_off"] = _t(edge_offsets(b))
    b["negative_edge_index"] = _t(negative_edge_index(b["edge_index"].numpy(), b["ptr"].numpy(), b["edge_off"].numpy(), seed))
    return b


def bio_edgepred_batch(num_graphs: int, seed: int, **ppi_kw) -> dict:
    """bio/pretrain_edgepred.py's input: a ppi_batch after NegativeEdge and BatchAE (bio/batch.py:123-175), drawn as
    edgepred_batch draws them."""
    b = ppi_batch(num_graphs, seed, **ppi_kw)
    b["edge_off"] = _t(edge_offsets(b))
    b["negative_edge_index"] = _t(negative_edge_index(b["edge_index"].numpy(), b["ptr"].numpy(), b["edge_off"].numpy(), seed))
    return b
