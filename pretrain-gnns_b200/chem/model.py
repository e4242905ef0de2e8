"""chem message-passing stack on libpgnn_b200 — host-side mirror of /root/reference/chem/model.py.

Same public surface as the reference so `pretrain_masking.py`, `pretrain_contextpred.py` and `finetune.py`
can `from model import GNN, GNN_graphpred` unchanged (SURVEY.md section 8(b)):

    GINConv(emb_dim, aggr="add").forward(x, edge_index, edge_attr)                    chem/model.py:26,37
    GNN(num_layer, emb_dim, JK="last", drop_ratio=0, gnn_type="gin").forward(x, ei, ea) | forward(data)   :222,255
    GNN_graphpred(num_layer, emb_dim, num_tasks, JK, drop_ratio, graph_pooling, gnn_type)
        .forward(x, ei, ea, batch) | forward(data), .from_pretrained(file)            :309,354,358

and the same parameter / buffer names, so every shipped `.pth` loads with all keys matched.  What differs
is underneath: no torch_geometric, no per-edge tensors.  Each batch is bucketed once (ops.Graph), the bond
embedding sum is folded into a per-node 9-bin summary, and every op is a CUDA kernel behind the C ABI.
"""
import torch
from torch import nn

from .. import ops

num_atom_type = 120      # incl. the mask token (chem/model.py:9)
num_chirality_tag = 3
num_bond_type = 6        # incl. aromatic, self-loop (4) and mask (5) (chem/model.py:12)
num_bond_direction = 3

_AGGR_MODE = {"add": ops.AGG_SUM, "mean": ops.AGG_MEAN}


def global_mean_pool(x, batch, size=None):
    return ops.global_mean_pool(x, batch, size)


class _BondTables(nn.Module):
    """Shared by the four convs: the two bond-feature tables (chem/model.py:30-34) of width `width`."""

    def _make_tables(self, width):
        self.edge_embedding1 = nn.Embedding(num_bond_type, width)
        self.edge_embedding2 = nn.Embedding(num_bond_direction, width)
        nn.init.xavier_uniform_(self.edge_embedding1.weight.data)
        nn.init.xavier_uniform_(self.edge_embedding2.weight.data)

    def _table(self):
        # rows 0..5 bond type, rows 6..8 direction: the layout pgnn_chem_edge_summary's 9 bins index
        return torch.cat([self.edge_embedding1.weight, self.edge_embedding2.weight], dim=0)

    def _mode(self):
        try:
            return _AGGR_MODE[self.aggr]
        except KeyError:
            raise ValueError("aggr=%r is not supported by this path (add / mean only)" % (self.aggr,))


class GINConv(_BondTables):
    """aggr_i = sum_{j in N(i) + i} (x_j + e_ij);  out = W2 relu(W1 aggr + b1) + b2   (chem/model.py:37-55)."""

    def __init__(self, emb_dim, aggr="add"):
        super().__init__()
        self.mlp = nn.Sequential(nn.Linear(emb_dim, 2 * emb_dim), nn.ReLU(), nn.Linear(2 * emb_dim, emb_dim))
        self._make_tables(emb_dim)
        self.aggr = aggr

    def forward(self, x, edge_index, edge_attr, graph=None):
        g = graph if graph is not None else ops.graph_for(edge_index, x.size(0))
        mode = self._mode()
        a = ops.aggregate(x, self._table(), g, g.summary("chem", mode, edge_attr), mode)
        return ops.mlp2(a, self.mlp[0].weight, self.mlp[0].bias, self.mlp[2].weight, self.mlp[2].bias)


class GCNConv(_BondTables):
    """x <- Linear(x);  out_i = sum_j d_i^-1/2 d_j^-1/2 (x_j + e_ij), degrees incl. self-loop (chem/model.py:73-104)."""

    def __init__(self, emb_dim, aggr="add"):
        super().__init__()
        self.emb_dim = emb_dim
        self.linear = nn.Linear(emb_dim, emb_dim)
        self._make_tables(emb_dim)
        self.aggr = aggr

    def forward(self, x, edge_index, edge_attr, graph=None):
        g = graph if graph is not None else ops.graph_for(edge_index, x.size(0))
        h = ops.linear(x, self.linear.weight, self.linear.bias)
        return ops.aggregate(h, self._table(), g, g.summary("chem", ops.AGG_GCN, edge_attr), ops.AGG_GCN)


class GraphSAGEConv(_BondTables):
    """x <- Linear(x);  out_i = normalize(mean_j (x_j + e_ij))   (chem/model.py:182-202)."""

    def __init__(self, emb_dim, aggr="mean"):
        super().__init__()
        self.emb_dim = emb_dim
        self.linear = nn.Linear(emb_dim, emb_dim)
        self._make_tables(emb_dim)
        self.aggr = aggr

    def forward(self, x, edge_index, edge_attr, graph=None):
        g = graph if graph is not None else ops.graph_for(edge_index, x.size(0))
        mode = self._mode()
        h = ops.linear(x, self.linear.weight, self.linear.bias)
        return ops.l2_normalize(ops.aggregate(h, self._table(), g, g.summary("chem", mode, edge_attr), mode))


class GATConv(_BondTables):
    """Two-head additive attention over (x_i, x_j + e_ij), softmax per target, head mean + bias (chem/model.py:107-165)."""

    def __init__(self, emb_dim, heads=2, negative_slope=0.2, aggr="add"):
        super().__init__()
        self.aggr = aggr
        self.emb_dim = emb_dim
        self.heads = heads
        self.negative_slope = negative_slope
        self.weight_linear = nn.Linear(emb_dim, heads * emb_dim)
        self.att = nn.Parameter(torch.empty(1, heads, 2 * emb_dim))
        self.bias = nn.Parameter(torch.empty(emb_dim))
        self._make_tables(heads * emb_dim)
        self.reset_parameters()

    def reset_parameters(self):
        bound = (6.0 / (self.att.size(-2) + self.att.size(-1))) ** 0.5  # torch_geometric.nn.inits.glorot
        self.att.data.uniform_(-bound, bound)
        self.bias.data.zero_()

    def forward(self, x, edge_index, edge_attr, graph=None):
        g = graph if graph is not None else ops.graph_for(edge_index, x.size(0))
        xl = ops.linear(x, self.weight_linear.weight, self.weight_linear.bias)
        return ops.gat(xl, self.att, self._table(), edge_attr, g, self.bias, self.heads, self.negative_slope, False)


_CONVS = {"gin": lambda d: GINConv(d, aggr="add"), "gcn": GCNConv, "gat": GATConv, "graphsage": GraphSAGEConv}


class GNN(nn.Module):
    """Node encoder: atom embedding, `num_layer` x (conv -> BatchNorm1d -> ReLU except last -> dropout), JK readout
    (chem/model.py:206-290).  Output: node representations [N, emb_dim] (JK='last')."""

    def __init__(self, num_layer, emb_dim, JK="last", drop_ratio=0, gnn_type="gin"):
        super().__init__()
        if num_layer < 2:
            raise ValueError("Number of GNN layers must be greater than 1.")
        self.num_layer, self.drop_ratio, self.JK = num_layer, drop_ratio, JK
        self.x_embedding1 = nn.Embedding(num_atom_type, emb_dim)
        self.x_embedding2 = nn.Embedding(num_chirality_tag, emb_dim)
        nn.init.xavier_uniform_(self.x_embedding1.weight.data)
        nn.init.xavier_uniform_(self.x_embedding2.weight.data)
        # an unknown gnn_type leaves `gnns` empty in the reference (chem/model.py:239-247); fail early instead
        if gnn_type not in _CONVS:
            raise ValueError("unknown gnn_type %r" % (gnn_type,))
        self.gnns = nn.ModuleList([_CONVS[gnn_type](emb_dim) for _ in range(num_layer)])
        self.batch_norms = nn.ModuleList([nn.BatchNorm1d(emb_dim) for _ in range(num_layer)])
        self._gnn_type = gnn_type
        self._plan = None          # lazily built bookkeeping of the whole-encoder path (ops.ChemEncoderPlan)
        self.fused = True          # set False to force the layer-by-layer composition (used by the tests)

    _DEFAULT_AGGR = {"gin": "add", "gcn": "add", "gat": "add", "graphsage": "mean"}

    def _fused_plan(self):
        """The whole-encoder kernels (pgnn_chem_encoder_*) cover every gnn_type with JK='last', the conv's default aggregation
        (and GAT's 2 heads / slope 0.2), with or without dropout."""
        if not (self.fused and self.JK == "last"):
            return None
        if any(conv.aggr != self._DEFAULT_AGGR[self._gnn_type] for conv in self.gnns) or any(bn.training != self.training for bn in self.batch_norms):
            return None
        if self._gnn_type == "gat" and any(conv.heads != 2 or conv.negative_slope != 0.2 for conv in self.gnns):
            return None
        if self._plan is None:
            self._plan = ops.ChemEncoderPlan(self, self._gnn_type)
        return self._plan

    def forward(self, *argv):
        if len(argv) == 3:
            x, edge_index, edge_attr = argv
        elif len(argv) == 1:
            x, edge_index, edge_attr = argv[0].x, argv[0].edge_index, argv[0].edge_attr
        else:
            raise ValueError("unmatched number of arguments.")
        # one dropout seed per forward, drawn on the host only when dropout is live (the RNG stream is untouched otherwise); both
        # paths below derive layer l's mask from (seed, l), so under the same torch.manual_seed they drop the same units
        drop = self.training and self.drop_ratio > 0
        seed = ops.draw_seed() if drop else 0
        plan = self._fused_plan()
        if plan is not None:
            return ops.chem_encoder(plan, x, edge_index, edge_attr, self.training, self.drop_ratio if drop else 0.0, seed)
        graph = ops.graph_for(edge_index, x.size(0))
        h = ops.chem_embed(x, self.x_embedding1.weight, self.x_embedding2.weight)
        hs = [h]
        last = self.num_layer - 1
        for l, (conv, bn) in enumerate(zip(self.gnns, self.batch_norms)):
            h = conv(h, edge_index, edge_attr, graph=graph)
            h = ops.batch_norm(h, bn, relu=(l != last))        # BN + ReLU fused (chem/model.py:269-275)
            if drop:
                h = ops.dropout(h, self.drop_ratio, seed, l)
            hs.append(h)
        if self.JK == "last":
            return hs[-1]
        if self.JK == "concat":
            return torch.cat(hs, dim=1)
        if self.JK == "max":
            return torch.stack(hs, dim=0).max(dim=0)[0]
        if self.JK == "sum":  # reproduces the reference's `[0]` after the sum (chem/model.py:288): one row
            return torch.stack(hs, dim=0).sum(dim=0)[0]
        raise ValueError("unknown JK %r" % (self.JK,))


class GNN_graphpred(nn.Module):
    """Encoder + global pooling + Linear head (chem/model.py:293-369).  graph_pooling='mean' is the in-scope
    pooling (SURVEY.md section 2 row 3); the others raise."""

    def __init__(self, num_layer, emb_dim, num_tasks, JK="last", drop_ratio=0, graph_pooling="mean", gnn_type="gin"):
        super().__init__()
        if num_layer < 2:
            raise ValueError("Number of GNN layers must be greater than 1.")
        self.num_layer, self.drop_ratio, self.JK = num_layer, drop_ratio, JK
        self.emb_dim, self.num_tasks = emb_dim, num_tasks
        self.gnn = GNN(num_layer, emb_dim, JK, drop_ratio, gnn_type=gnn_type)
        if graph_pooling == "mean":
            self.pool = global_mean_pool
        elif graph_pooling in ("sum", "max", "attention") or graph_pooling[:-1] == "set2set":
            raise NotImplementedError("graph_pooling=%r is outside this hot path (mean only)" % (graph_pooling,))
        else:
            raise ValueError("Invalid graph pooling type.")
        self.mult = 1
        width = (num_layer + 1) * emb_dim if JK == "concat" else emb_dim
        self.graph_pred_linear = nn.Linear(self.mult * width, num_tasks)

    def from_pretrained(self, model_file):
        dev = next(self.gnn.parameters()).device
        self.gnn.load_state_dict(torch.load(model_file, map_location=dev))

    def forward(self, *argv):
        if len(argv) == 4:
            x, edge_index, edge_attr, batch = argv
        elif len(argv) == 1:
            d = argv[0]
            x, edge_index, edge_attr, batch = d.x, d.edge_index, d.edge_attr, d.batch
        else:
            raise ValueError("unmatched number of arguments.")
        rep = self.gnn(x, edge_index, edge_attr)
        return ops.linear(self.pool(rep, batch), self.graph_pred_linear.weight, self.graph_pred_linear.bias)
