"""TEST INFRASTRUCTURE ONLY — edge-prediction pre-training (chem/pretrain_edgepred.py, bio/pretrain_edgepred.py) restated for the
tests:
  * the transform: `negative_edge_candidates` (the draw pgnn_negative_edges defines), `negative_edge` (NegativeEdge.__call__ of
    chem/util.py:22-52 and bio/util.py:16-44, its loop restated literally over given candidates), `batch_ae`
    (BatchAE.from_data_list, chem/batch.py:69-121 and bio/batch.py:123-175) and `negative_edges_batch`, the three composed on a
    collated batch;
  * `edgepred_loss`   the train() body on the oracle port (oracle/gnn_oracle.py) over flat leaf dictionaries;
  * `ReferenceEdgePredStep` / `ReferenceBioEdgePredStep`   the same body on the reference's OWN chem / bio model.py
    (oracle/reference_runner.py) with nn.BCEWithLogitsLoss on the fp32 scores, exactly as the scripts call it.
Parameters come from `make_params`, keyed `model.<state_dict key>` like train_steps.EdgePredStep names them."""
import numpy as np
import torch
import torch.nn.functional as F

from oracle import gnn_oracle as O
from oracle.step_io_oracle import _M64, splitmix64
from oracle.steps_oracle import _RefStep, sub


# ---------------------------------------------------------------------------------------------------------------------
# the transform
# ---------------------------------------------------------------------------------------------------------------------
def negative_edge_candidates(n, e, e0, seed):
    """The 2 x 5e candidates of a graph of n nodes and e columns whose columns start at e0 in the batch: column j is
    (splitmix64(seed, 2 (5 e0 + j)) mod n, splitmix64(seed, 2 (5 e0 + j) + 1) mod n) (torch.randint(0, n, (2, 5e)) in the
    reference; a graph with n = 0 draws nothing)."""
    K = 5 * e if n > 0 else 0
    out = np.zeros((2, K), dtype=np.int64)
    for j in range(K):
        c = 2 * (5 * e0 + j)
        out[0, j] = splitmix64(seed & _M64, c) % n
        out[1, j] = splitmix64(seed & _M64, c + 1) % n
    return out


def negative_edge(ei_local, n, candidates):
    """NegativeEdge.__call__ (chem/util.py:29-52) with `redandunt_sample` = candidates: string keys of the DIRECTED columns, candidates
    in order, accept when new, not a column and not a self pair, stop once the count == num_edges / 2 (a float comparison)."""
    ei = np.asarray(ei_local)
    num_edges = ei.shape[1]
    edge_set = set([str(int(ei[0, i])) + "," + str(int(ei[1, i])) for i in range(num_edges)])
    sampled_ind = []
    sampled_edge_set = set([])
    for i in range(5 * num_edges if n > 0 else 0):
        node1, node2 = int(candidates[0, i]), int(candidates[1, i])
        edge_str = str(node1) + "," + str(node2)
        if not edge_str in edge_set and not edge_str in sampled_edge_set and not node1 == node2:
            sampled_edge_set.add(edge_str)
            sampled_ind.append(i)
        if len(sampled_ind) == num_edges / 2:
            break
    return np.asarray(candidates, dtype=np.int64).reshape(2, -1)[:, sampled_ind]


def batch_ae(data_list):
    """BatchAE.from_data_list: per graph i, `batch` gets full((n_i,), i), edge_index and negative_edge_index get the running node
    count; edge_index / negative_edge_index are concatenated along the last dimension, every other key along dim 0.
    data_list: dicts of numpy arrays with 'x' and any of 'edge_index', 'negative_edge_index', 'edge_attr'."""
    keys = sorted(set().union(*[set(d) for d in data_list]))
    acc = {k: [] for k in keys}
    bvec, cumsum_node = [], 0
    for i, d in enumerate(data_list):
        n = d["x"].shape[0]
        bvec.append(np.full((n,), i, dtype=np.int64))
        for k in d:
            acc[k].append(d[k] + cumsum_node if k in ("edge_index", "negative_edge_index") else d[k])
        cumsum_node += n
    out = {k: np.concatenate(v, axis=-1 if k in ("edge_index", "negative_edge_index") else 0) for k, v in acc.items()}
    out["batch"] = np.concatenate(bvec)
    return out


def negative_edges_batch(edge_index, node_off, edge_off, seed):
    """The transform on a collated batch: per graph the candidates and the reference's loop on graph-local ids, then BatchAE's
    offset.  An endpoint outside its graph is left out of the graph's edge set (it can never equal a candidate).
    -> (negative_edge_index [2, M], negative_edge_off [B+1])"""
    ei = np.asarray(edge_index, dtype=np.int64)
    cols, off = [], [0]
    for g in range(len(node_off) - 1):
        n0, n = int(node_off[g]), int(node_off[g + 1] - node_off[g])
        e0, e = int(edge_off[g]), int(edge_off[g + 1] - edge_off[g])
        local = ei[:, e0:e0 + e] - n0
        neg = negative_edge(local, n, negative_edge_candidates(n, e, e0, seed))
        cols.append(neg + n0)
        off.append(off[-1] + neg.shape[1])
    return (np.concatenate(cols, axis=1) if cols else np.zeros((2, 0), np.int64)), np.array(off, dtype=np.int64)


# ---------------------------------------------------------------------------------------------------------------------
# the train() body
# ---------------------------------------------------------------------------------------------------------------------
def edgepred_loss(L, b, domain="chem", gnn_type="gin"):
    """chem/pretrain_edgepred.py:33-39 (bio alike).  L: 'model.*' encoder.  The BCE is taken on fp64 scores."""
    dt = next(v.dtype for v in L.values() if v.is_floating_point())
    ei, neg_ei = b["edge_index"], b["negative_edge_index"]
    if domain == "chem":
        rep = O.chem_gnn(sub(L, "model."), b["x"], ei, b["edge_attr"], 5, gnn_type, True)
    else:
        rep = O.bio_gnn(sub(L, "model."), b["x"].to(dt), ei, b["edge_attr"].to(dt), 5, gnn_type, True)
    pos = torch.sum(rep[ei[0, ::2]] * rep[ei[1, ::2]], dim=1)
    neg = torch.sum(rep[neg_ei[0]] * rep[neg_ei[1]], dim=1)
    return edgepred_head(pos, neg), dict(rep=rep, pos=pos, neg=neg)


def edgepred_head(pos, neg):
    """BCEWithLogits(pos, 1) + BCEWithLogits(neg, 0) on fp64 scores, each a mean over its own side."""
    pos, neg = pos.double(), neg.double()
    return F.binary_cross_entropy_with_logits(pos, torch.ones_like(pos)) + F.binary_cross_entropy_with_logits(neg, torch.zeros_like(neg))


def make_params(domain, seed, gnn_type="gin"):
    return {"model." + k: v for k, v in O.make_params(domain, gnn_type, 5, 300, seed).items()}


class ReferenceEdgePredStep(_RefStep):
    domain = "chem"

    def __init__(self, gnn_type="gin"):
        from oracle import reference_runner as R
        mod = R.load(self.domain)
        self.model = mod.GNN(5, 300, JK="last", drop_ratio=0, gnn_type=gnn_type).train()
        self.criterion = torch.nn.BCEWithLogitsLoss()
        self.named = {"model": self.model}
        self.modules = [self.model]

    def __call__(self, b):
        self.zero_grad()
        node_emb = self.model(b["x"], b["edge_index"], b["edge_attr"])
        positive_score = torch.sum(node_emb[b["edge_index"][0, ::2]] * node_emb[b["edge_index"][1, ::2]], dim=1)
        negative_score = torch.sum(node_emb[b["negative_edge_index"][0]] * node_emb[b["negative_edge_index"][1]], dim=1)
        loss = self.criterion(positive_score, torch.ones_like(positive_score)) + self.criterion(negative_score, torch.zeros_like(negative_score))
        loss.backward()
        return loss


class ReferenceBioEdgePredStep(ReferenceEdgePredStep):
    domain = "bio"
