"""TEST INFRASTRUCTURE ONLY — Deep Graph Infomax pre-training (chem/pretrain_deepgraphinfomax.py, bio/pretrain_deepgraphinfomax.py)
restated for the tests:
  * `cycle_index`, `uniform`, `Discriminator` and `Infomax`   the script's own definitions (and PyG 1.0.3's inits.uniform, which
    the script imports), restated literally with their line citations: the script itself cannot be imported (it pulls in loader,
    sklearn and tensorboardX);
  * `infomax_loss`   the train() body on the oracle port (oracle/gnn_oracle.py) over flat leaf dictionaries;
  * `ReferenceInfomaxStep` / `ReferenceBioInfomaxStep`   the same body on the reference's OWN chem / bio model.py
    (oracle/reference_runner.py) inside the restated Infomax, with nn.BCEWithLogitsLoss on the fp32 scores as the script calls it.
Parameters come from `make_params`, keyed `gnn.<state_dict key>` and `discriminator.weight`, as Infomax.state_dict() names them."""
import math

import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle import gnn_oracle as O
from oracle.steps_oracle import _RefStep, sub


# ---------------------------------------------------------------------------------------------------------------------
# the script's definitions
# ---------------------------------------------------------------------------------------------------------------------
def cycle_index(num, shift):
    """chem/pretrain_deepgraphinfomax.py:25-28."""
    arr = torch.arange(num) + shift
    arr[-shift:] = torch.arange(shift)
    return arr


def uniform(size, tensor):
    """torch_geometric 1.0.3 nn/inits.py `uniform` (imported by chem/pretrain_deepgraphinfomax.py:5)."""
    bound = 1.0 / math.sqrt(size)
    if tensor is not None:
        tensor.data.uniform_(-bound, bound)


class Discriminator(nn.Module):
    """chem/pretrain_deepgraphinfomax.py:30-42."""
    def __init__(self, hidden_dim):
        super(Discriminator, self).__init__()
        self.weight = nn.Parameter(torch.Tensor(hidden_dim, hidden_dim))
        self.reset_parameters()

    def reset_parameters(self):
        size = self.weight.size(0)
        uniform(size, self.weight)

    def forward(self, x, summary):
        h = torch.matmul(summary, self.weight)
        return torch.sum(x * h, dim=1)


class Infomax(nn.Module):
    """chem/pretrain_deepgraphinfomax.py:44-50; `pool` is the global_mean_pool the reference's model module imports."""
    def __init__(self, gnn, discriminator, pool):
        super(Infomax, self).__init__()
        self.gnn = gnn
        self.discriminator = discriminator
        self.loss = nn.BCEWithLogitsLoss()
        self.pool = pool


# ---------------------------------------------------------------------------------------------------------------------
# the train() body
# ---------------------------------------------------------------------------------------------------------------------
def num_graphs_of(b):
    return int(b["num_graphs"]) if "num_graphs" in b else int(b["batch"].max()) + 1


def infomax_head(node_emb, batch, W, G):
    """Lines 62-70 on given node rows: -> (pos, neg, summary)."""
    summary = torch.sigmoid(O.segment_mean(node_emb, batch, G))
    h = torch.matmul(summary, W)
    pos = torch.sum(node_emb * h[batch], dim=1)
    neg = torch.sum(node_emb * h[cycle_index(G, 1).to(batch.device)][batch], dim=1)
    return pos, neg, summary


def bce_pair(pos, neg):
    """Line 73: BCEWithLogits(pos, 1) + BCEWithLogits(neg, 0) on fp64 scores, each a mean over the N nodes."""
    pos, neg = pos.double(), neg.double()
    return F.binary_cross_entropy_with_logits(pos, torch.ones_like(pos)) + F.binary_cross_entropy_with_logits(neg, torch.zeros_like(neg))


def infomax_loss(L, b, domain="chem", gnn_type="gin"):
    """chem/pretrain_deepgraphinfomax.py:61-73 (bio alike).  L: 'gnn.*' encoder, 'discriminator.weight'.  The BCE is taken on
    fp64 scores."""
    dt = L["discriminator.weight"].dtype
    if domain == "chem":
        rep = O.chem_gnn(sub(L, "gnn."), b["x"], b["edge_index"], b["edge_attr"], 5, gnn_type, True)
    else:
        rep = O.bio_gnn(sub(L, "gnn."), b["x"].to(dt), b["edge_index"], b["edge_attr"].to(dt), 5, gnn_type, True)
    pos, neg, summary = infomax_head(rep, b["batch"], L["discriminator.weight"], num_graphs_of(b))
    return bce_pair(pos, neg), dict(rep=rep, summary=summary, pos=pos, neg=neg)


def make_params(domain, seed, gnn_type="gin"):
    P = {"gnn." + k: v for k, v in O.make_params(domain, gnn_type, 5, 300, seed).items()}
    g = torch.Generator().manual_seed(seed + 977)
    P["discriminator.weight"] = (torch.rand(300, 300, generator=g) * 2.0 - 1.0) / math.sqrt(300)
    return P


class ReferenceInfomaxStep(_RefStep):
    domain = "chem"

    def __init__(self, gnn_type="gin"):
        from oracle import reference_runner as R
        mod = R.load(self.domain)
        gnn = mod.GNN(5, 300, JK="last", drop_ratio=0, gnn_type=gnn_type)
        self.model = Infomax(gnn, Discriminator(300), mod.global_mean_pool).train()
        self.named = {"gnn": self.model.gnn, "discriminator": self.model.discriminator}
        self.modules = [self.model]

    def __call__(self, b):
        """chem/pretrain_deepgraphinfomax.py:61-74 as written."""
        model, batch = self.model, b
        self.zero_grad()
        node_emb = model.gnn(batch["x"], batch["edge_index"], batch["edge_attr"])
        summary_emb = torch.sigmoid(model.pool(node_emb, batch["batch"]))

        positive_expanded_summary_emb = summary_emb[batch["batch"]]

        shifted_summary_emb = summary_emb[cycle_index(len(summary_emb), 1)]
        negative_expanded_summary_emb = shifted_summary_emb[batch["batch"]]

        positive_score = model.discriminator(node_emb, positive_expanded_summary_emb)
        negative_score = model.discriminator(node_emb, negative_expanded_summary_emb)

        loss = model.loss(positive_score, torch.ones_like(positive_score)) + model.loss(negative_score, torch.zeros_like(negative_score))
        loss.backward()
        return loss


class ReferenceBioInfomaxStep(ReferenceInfomaxStep):
    domain = "bio"
