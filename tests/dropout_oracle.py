"""Host restatement of the library's dropout draw and the masked oracle encoders (tests/test_dropout_host.py,
tests/test_gpu_dropout.py).

The draw (include/pgnn_b200.h, pgnn_dropout_fwd): element (row i, column c) of layer l's [N, C] activation is kept iff
    r = splitmix64(seed, (l << 40) | (i * C + c)) >> 32,   r >= thr,   thr = floor(p * 2^32) (p < 1),  2^32 (p == 1)
with p the fp32 value the library receives, and a kept element is multiplied by scale = fp32(1 / (1 - p)), a dropped one by 0.

The masked encoders are the oracle's (oracle/gnn_oracle.py) with `h = h * m_l * scale` where the reference calls F.dropout
(chem/model.py:271-275, bio/model.py:278-281): after every inner layer's ReLU, and on the last layer's output without one.
"""
import numpy as np
import torch
import torch.nn.functional as F

from oracle import gnn_oracle as O
from oracle import steps_oracle as S

_C1, _C2, _C3 = np.uint64(0x9E3779B97F4A7C15), np.uint64(0xBF58476D1CE4E5B9), np.uint64(0x94D049BB133111EB)


def splitmix64(seed, idx):
    """Vectorised splitmix64 (csrc/common.cuh; oracle/step_io_oracle.splitmix64 is the scalar form) on uint64 arrays."""
    with np.errstate(over="ignore"):
        z = np.uint64(int(seed) & ((1 << 64) - 1)) + (np.asarray(idx, dtype=np.uint64) + np.uint64(1)) * _C1
        z = (z ^ (z >> np.uint64(30))) * _C2
        z = (z ^ (z >> np.uint64(27))) * _C3
        return z ^ (z >> np.uint64(31))


def threshold(p):
    p32 = np.float32(p)
    return 1 << 32 if p32 == 1 else int(np.floor(np.float64(p32) * 2.0 ** 32))


def scale(p):
    p32 = np.float64(np.float32(p))
    return 0.0 if p32 == 1 else float(np.float32(1.0 / (1.0 - p32)))


def draws(seed, layer, rows, C):
    """The 32-bit draws r of a [rows, C] activation of `layer` (uint64 array holding values < 2^32)."""
    idx = (np.uint64(layer) << np.uint64(40)) | np.arange(rows * C, dtype=np.uint64)
    return (splitmix64(seed, idx) >> np.uint64(32)).reshape(rows, C)


def keep_mask(seed, layer, rows, C, p):
    """bool [rows, C]: which elements of layer `layer`'s activation the library keeps."""
    return draws(seed, layer, rows, C) >= np.uint64(threshold(p)) if threshold(p) < (1 << 32) else np.zeros((rows, C), dtype=bool)


def layer_masks(seed, num_layer, rows, C, p, dtype=torch.float64):
    """0/1 masks of every layer of one forward (one seed per forward, layer l = the mask index)."""
    return [torch.from_numpy(keep_mask(seed, l, rows, C, p)).to(dtype) for l in range(num_layer)]


def _drop(h, masks, l, p):
    """The library's factor: the fp32 scale(p), which is 0 at p = 1 (every element dropped) rather than 0 * inf."""
    return h if masks is None else h * masks[l].to(h.dtype) * scale(p)


def chem_gnn(P, x, edge_index, edge_attr, num_layer, gnn_type="gin", training=False, new_stats=None, pre="", masks=None, p=0.0):
    """O.chem_gnn with dropout: layer l's output (after BatchNorm and the ReLU of an inner layer) times masks[l] / (1 - p)."""
    n = x.shape[0]
    h = F.embedding(x[:, 0], P[pre + "x_embedding1.weight"]) + F.embedding(x[:, 1], P[pre + "x_embedding2.weight"])
    ei = O.with_self_loops(edge_index, n)
    conv = {"gin": O.gin_conv_chem, "gcn": O.gcn_conv, "graphsage": O.sage_conv, "gat": O.gat_conv}[gnn_type]
    for l in range(num_layer):
        lp = f"{pre}gnns.{l}."
        h = conv(P, lp, h, ei, O.chem_edge_rows(P, lp, edge_attr, n))
        h = O.batch_norm(P, f"{pre}batch_norms.{l}.", h, training, new_stats)
        if l != num_layer - 1:
            h = O._relu(h)  # traced (O.RELU_TRACE) like the oracle's own ReLUs
        h = _drop(h, masks, l, p)
    return h


def bio_gnn(P, x, edge_index, edge_attr, num_layer, gnn_type="gin", training=False, new_stats=None, pre="", masks=None, p=0.0):
    """O.bio_gnn with dropout: layer l's conv output (after the ReLU of an inner layer) times masks[l] / (1 - p); never inside
    GIN's MLP BatchNorm."""
    n = x.shape[0]
    ei = O.with_self_loops(edge_index, n)
    h = x
    for l in range(num_layer):
        lp = f"{pre}gnns.{l}."
        rows = O.bio_edge_rows(P, lp, edge_attr, n)
        if l == 0:
            h = F.embedding(h.to(torch.int64).view(-1), P[lp + "input_node_embeddings.weight"])
        if gnn_type == "gin":
            h = O.gin_conv_bio(P, lp, h, ei, rows, training, new_stats)
        else:
            h = {"gcn": O.gcn_conv, "graphsage": O.sage_conv, "gat": O.gat_conv}[gnn_type](P, lp, h, ei, rows)
        if l != num_layer - 1:
            h = torch.relu(h)
        h = _drop(h, masks, l, p)
    return h


def chem_graphpred(P, x, edge_index, edge_attr, batch, num_graphs, num_layer, gnn_type="gin", training=False, masks=None, p=0.0):
    """chem/model.py:358-369 (mean pooling) on the masked encoder; the head has no dropout."""
    h = chem_gnn(P, x, edge_index, edge_attr, num_layer, gnn_type, training, pre="gnn.", masks=masks, p=p)
    return F.linear(O.segment_mean(h, batch, num_graphs), P["graph_pred_linear.weight"], P["graph_pred_linear.bias"])


def bio_graphpred(P, x, edge_index, edge_attr, batch, center_node_idx, num_graphs, num_layer, gnn_type="gin", training=False,
                  masks=None, p=0.0):
    """bio/model.py:338-347 on the masked encoder."""
    h = bio_gnn(P, x, edge_index, edge_attr, num_layer, gnn_type, training, pre="gnn.", masks=masks, p=p)
    rep = torch.cat([O.segment_mean(h, batch, num_graphs), h[center_node_idx]], dim=1)
    return F.linear(rep, P["graph_pred_linear.weight"], P["graph_pred_linear.bias"])


def finetune_loss(L, b, masks, p, gnn_type="gin", num_layer=5):
    """chem/finetune.py:27-46.  L: 'model.gnn.*', 'model.graph_pred_linear.*' (FinetuneStep's names); masks: one per layer."""
    P = S.sub(L, "model.")
    B = b["y"].shape[0]
    pred = chem_graphpred(P, b["x"], b["edge_index"], b["edge_attr"], b["batch"], B, num_layer, gnn_type, True, masks, p)
    y = b["y"].view(pred.shape).to(torch.float64)
    is_valid = y ** 2 > 0
    loss_mat = F.binary_cross_entropy_with_logits(pred.double(), (y + 1) / 2, reduction="none")
    loss_mat = torch.where(is_valid, loss_mat, torch.zeros_like(loss_mat))
    return torch.sum(loss_mat) / torch.sum(is_valid), dict(pred=pred)


def finetune_params(gnn_type, seed, num_tasks=12, num_layer=5, emb_dim=300):
    """Seeded parameters of FinetuneStep's model, keyed as FinetuneStep.load_state takes them."""
    g = torch.Generator().manual_seed(seed + 977)
    P = {"model.gnn." + k: v for k, v in O.make_params("chem", gnn_type, num_layer, emb_dim, seed).items()}
    P["model.graph_pred_linear.weight"] = torch.randn(num_tasks, emb_dim, generator=g) * 0.05
    P["model.graph_pred_linear.bias"] = torch.randn(num_tasks, generator=g) * 0.05
    return P
