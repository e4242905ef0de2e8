"""bio (PPI) message-passing stack on libpgnn_b200 — host-side mirror of /root/reference/bio/model.py.

Differences from chem that the reference encodes and this file keeps (SURVEY.md section 8(a) a12-a14):
edge features are 9 floats through `edge_encoder = Linear(9, .)` with the self-loop row one-hot at
column 7; layer 0 embeds the dummy node label with `input_node_embeddings`; GIN concatenates
[x_j, e_ij] (2*emb wide) and its MLP carries an inner BatchNorm1d; the encoder has NO outer BatchNorm;
the graph head is Linear(2*emb, T) on [mean_pool, centre-node row].

Because the message is linear in e_ij, `Linear(9, .)` is applied once per NODE to the summed edge bits
(ops.Graph.summary('bio', ...), Q = 10: nine attribute sums + the weight sum that multiplies the bias),
not once per edge: the reference's [E+N, 600] message tensor (845 MB at B=64) never exists.
"""
import torch
from torch import nn

from .. import ops

_AGGR_MODE = {"add": ops.AGG_SUM, "mean": ops.AGG_MEAN}


def global_mean_pool(x, batch, size=None):
    return ops.global_mean_pool(x, batch, size)


class _EdgeEncoder(nn.Module):
    def _make_encoder(self, emb_dim, width, input_layer):
        self.edge_encoder = nn.Linear(9, width)
        self.input_layer = input_layer
        if input_layer:
            self.input_node_embeddings = nn.Embedding(2, emb_dim)
            nn.init.xavier_uniform_(self.input_node_embeddings.weight.data)

    def _table(self):
        # [10, width]: rows 0..8 = W^T, row 9 = bias (multiplied by the per-node weight sum)
        return torch.cat([self.edge_encoder.weight.t(), self.edge_encoder.bias.unsqueeze(0)], dim=0)

    def _input(self, x):
        return ops.bio_embed(x, self.input_node_embeddings.weight) if self.input_layer else x  # bio/model.py:49-50

    def _mode(self):
        try:
            return _AGGR_MODE[self.aggr]
        except KeyError:
            raise ValueError("aggr=%r is not supported by this path (add / mean only)" % (self.aggr,))


class GINConv(_EdgeEncoder):
    """aggr_i = sum_j [x_j || e_ij];  out = W2 relu(BN(W1 aggr + b1)) + b2   (bio/model.py:37-58)."""

    def __init__(self, emb_dim, aggr="add", input_layer=False):
        super().__init__()
        self.mlp = nn.Sequential(nn.Linear(2 * emb_dim, 2 * emb_dim), nn.BatchNorm1d(2 * emb_dim), nn.ReLU(),
                                 nn.Linear(2 * emb_dim, emb_dim))
        self._make_encoder(emb_dim, emb_dim, input_layer)
        self.aggr = aggr

    def forward(self, x, edge_index, edge_attr, graph=None):
        g = graph if graph is not None else ops.graph_for(edge_index, x.size(0))
        mode = self._mode()
        a = ops.aggregate(self._input(x), self._table(), g, g.summary("bio", mode, edge_attr), mode, concat=True)
        z = ops.linear(a, self.mlp[0].weight, self.mlp[0].bias)
        z = ops.batch_norm(z, self.mlp[1], relu=True)
        return ops.linear(z, self.mlp[3].weight, self.mlp[3].bias)


class GCNConv(_EdgeEncoder):
    def __init__(self, emb_dim, aggr="add", input_layer=False):
        super().__init__()
        self.emb_dim = emb_dim
        self.linear = nn.Linear(emb_dim, emb_dim)
        self._make_encoder(emb_dim, emb_dim, input_layer)
        self.aggr = aggr

    def forward(self, x, edge_index, edge_attr, graph=None):
        g = graph if graph is not None else ops.graph_for(edge_index, x.size(0))
        h = ops.linear(self._input(x), self.linear.weight, self.linear.bias)
        return ops.aggregate(h, self._table(), g, g.summary("bio", ops.AGG_GCN, edge_attr), ops.AGG_GCN)


class GraphSAGEConv(_EdgeEncoder):
    def __init__(self, emb_dim, aggr="mean", input_layer=False):
        super().__init__()
        self.emb_dim = emb_dim
        self.linear = nn.Linear(emb_dim, emb_dim)
        self._make_encoder(emb_dim, emb_dim, input_layer)
        self.aggr = aggr

    def forward(self, x, edge_index, edge_attr, graph=None):
        g = graph if graph is not None else ops.graph_for(edge_index, x.size(0))
        mode = self._mode()
        h = ops.linear(self._input(x), self.linear.weight, self.linear.bias)
        return ops.l2_normalize(ops.aggregate(h, self._table(), g, g.summary("bio", mode, edge_attr), mode))


class GATConv(_EdgeEncoder):
    def __init__(self, emb_dim, heads=2, negative_slope=0.2, aggr="add", input_layer=False):
        super().__init__()
        self.aggr = aggr
        self.emb_dim = emb_dim
        self.heads = heads
        self.negative_slope = negative_slope
        self.weight_linear = nn.Linear(emb_dim, heads * emb_dim)
        self.att = nn.Parameter(torch.empty(1, heads, 2 * emb_dim))
        self.bias = nn.Parameter(torch.empty(emb_dim))
        self._make_encoder(emb_dim, heads * emb_dim, input_layer)
        self.reset_parameters()

    def reset_parameters(self):
        bound = (6.0 / (self.att.size(-2) + self.att.size(-1))) ** 0.5
        self.att.data.uniform_(-bound, bound)
        self.bias.data.zero_()

    def forward(self, x, edge_index, edge_attr, graph=None):
        g = graph if graph is not None else ops.graph_for(edge_index, x.size(0))
        xl = ops.linear(self._input(x), self.weight_linear.weight, self.weight_linear.bias)
        return ops.gat(xl, self.att, self._table(), edge_attr, g, self.bias, self.heads, self.negative_slope, True)


_CONVS = {"gin": lambda d, il: GINConv(d, aggr="add", input_layer=il), "gcn": lambda d, il: GCNConv(d, input_layer=il),
          "gat": lambda d, il: GATConv(d, input_layer=il), "graphsage": lambda d, il: GraphSAGEConv(d, input_layer=il)}


class GNN(nn.Module):
    """`num_layer` convs with ReLU (+dropout) between them, no outer BatchNorm (bio/model.py:227-290)."""

    def __init__(self, num_layer, emb_dim, JK="last", drop_ratio=0, gnn_type="gin"):
        super().__init__()
        if num_layer < 2:
            raise ValueError("Number of GNN layers must be greater than 1.")
        if gnn_type not in _CONVS:
            raise ValueError("unknown gnn_type %r" % (gnn_type,))
        self.num_layer, self.drop_ratio, self.JK = num_layer, drop_ratio, JK
        self.gnns = nn.ModuleList([_CONVS[gnn_type](emb_dim, l == 0) for l in range(num_layer)])
        self._gnn_type = gnn_type
        self._plan = None          # lazily built bookkeeping of the whole-encoder path (ops.BioEncoderPlan)
        self.fused = True          # set False to force the layer-by-layer composition (used by the tests)

    _DEFAULT_AGGR = {"gin": "add", "gcn": "add", "gat": "add", "graphsage": "mean"}

    def _fused_plan(self):
        """The whole-encoder kernels (pgnn_bio_encoder_*) cover every gnn_type with JK='last', the conv's default aggregation
        (and GAT's 2 heads / slope 0.2), with or without dropout."""
        if not (self.fused and self.JK == "last"):
            return None
        if any(conv.aggr != self._DEFAULT_AGGR[self._gnn_type] for conv in self.gnns):
            return None
        if self._gnn_type == "gin" and any(conv.mlp[1].training != self.training for conv in self.gnns):
            return None
        if self._gnn_type == "gat" and any(conv.heads != 2 or conv.negative_slope != 0.2 for conv in self.gnns):
            return None
        if self._plan is None:
            self._plan = ops.BioEncoderPlan(self, self._gnn_type)
        return self._plan

    def forward(self, x, edge_index, edge_attr):
        drop = self.training and self.drop_ratio > 0
        plan = self._fused_plan()
        if plan is not None:
            seed = ops.draw_seed() if drop else 0  # the same draw as below: both paths drop the same units
            return ops.bio_encoder(plan, x, edge_index, edge_attr, self.training, self.drop_ratio if drop else 0.0, seed)
        graph = ops.graph_for(edge_index, x.size(0))
        seed = ops.draw_seed() if drop else 0  # one per forward; layer l's mask is ops.dropout's of (seed, l)
        h = x
        hs = []
        for l, conv in enumerate(self.gnns):
            h = conv(h, edge_index, edge_attr, graph=graph)
            if l != self.num_layer - 1:
                h = ops.relu(h)
            if drop:
                h = ops.dropout(h, self.drop_ratio, seed, l)
            hs.append(h)
        if self.JK == "last":
            return hs[-1]
        if self.JK == "sum":  # the reference's `[0]` after the sum (bio/model.py:288): one row
            return torch.stack(hs, dim=0).sum(dim=0)[0]
        raise ValueError("unknown JK %r" % (self.JK,))


class GNN_graphpred(nn.Module):
    """Linear(2*emb, T) on [mean_pool(node_rep), node_rep[center_node_idx]]   (bio/model.py:293-347)."""

    def __init__(self, num_layer, emb_dim, num_tasks, JK="last", drop_ratio=0, graph_pooling="mean", gnn_type="gin"):
        super().__init__()
        if num_layer < 2:
            raise ValueError("Number of GNN layers must be greater than 1.")
        self.num_layer, self.drop_ratio, self.JK = num_layer, drop_ratio, JK
        self.emb_dim, self.num_tasks = emb_dim, num_tasks
        self.gnn = GNN(num_layer, emb_dim, JK, drop_ratio, gnn_type=gnn_type)
        if graph_pooling == "mean":
            self.pool = global_mean_pool
        elif graph_pooling in ("sum", "max", "attention"):
            raise NotImplementedError("graph_pooling=%r is outside this hot path (mean only)" % (graph_pooling,))
        else:
            raise ValueError("Invalid graph pooling type.")
        self.graph_pred_linear = nn.Linear(2 * emb_dim, num_tasks)

    def from_pretrained(self, model_file):
        self.gnn.load_state_dict(torch.load(model_file, map_location=lambda storage, loc: storage))

    def forward(self, data):
        rep = self.gnn(data.x, data.edge_index, data.edge_attr)
        # one centre node per graph (bio/batch.py:39-40): the segment count is known without reading batch.max() back
        pooled = self.pool(rep, data.batch, int(data.center_node_idx.shape[0]))
        center = ops.row_gather(rep, data.center_node_idx)
        return ops.linear(torch.cat([pooled, center], dim=1), self.graph_pred_linear.weight, self.graph_pred_linear.bias)
