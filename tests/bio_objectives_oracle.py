"""TEST INFRASTRUCTURE ONLY — the bio masking and bio context-prediction train() bodies, in the two flavours of
oracle/steps_oracle.py:
  * `bio_masking_loss` / `bio_contextpred_loss`   on the oracle port (oracle/gnn_oracle.py) over flat leaf dictionaries;
  * `ReferenceBioMaskingStep` / `ReferenceBioContextPredStep`   on the reference's OWN bio/model.py (oracle/reference_runner.py),
    with torch.argmax and nn.CrossEntropyLoss / nn.BCEWithLogitsLoss exactly as bio/pretrain_masking.py and
    bio/pretrain_contextpred.py call them.
Parameters come from `make_params`, keyed `<module attribute>.<state_dict key>` like train_steps.BioMaskingStep and
BioContextPredStep name them."""
import torch
import torch.nn.functional as F

from oracle import gnn_oracle as O
from oracle.steps_oracle import _RefStep, sub

NUM_EDGE_TYPES = 7   # bio/pretrain_masking.py:121  linear_pred_edges = torch.nn.Linear(args.emb_dim, 7)


def edge_type_label(mask_edge_label):
    """The class of each masked edge: the FIRST index of the maximum of its label row (torch >= 1.7 documents this rule for
    torch.argmax; torch 1.0.1's CUDA tie rule is not documented).  Restated without argmax: the smallest column index holding
    the row maximum; an all-zero row gives 0."""
    lab = torch.as_tensor(mask_edge_label)
    if lab.shape[0] == 0:
        return torch.zeros(0, dtype=torch.int64)
    cols = torch.arange(lab.shape[1]).expand(lab.shape)
    return torch.where(lab == lab.max(dim=1, keepdim=True).values, cols, lab.shape[1]).min(dim=1).values


def _float(t, dt):
    return t.to(dt) if t.is_floating_point() else t


def bio_masking_loss(L, b, gnn_type="gin"):
    """bio/pretrain_masking.py:43-55.  L: 'model.*' bio encoder, 'head.weight', 'head.bias'.  The loss is taken on fp64 logits."""
    dt = L["head.bias"].dtype
    rep = O.bio_gnn(sub(L, "model."), _float(b["x"], dt), b["edge_index"], _float(b["edge_attr"], dt), 5, gnn_type, True)
    me = b["edge_index"][:, b["masked_edge_idx"]]
    logits = F.linear(rep[me[0]] + rep[me[1]], L["head.weight"], L["head.bias"])
    return F.cross_entropy(logits.double(), edge_type_label(b["mask_edge_label"])), dict(rep=rep, logits=logits)


def bio_contextpred_loss(L, b, neg_samples=1):
    """bio/pretrain_contextpred.py:53-97 (cbow, mean).  L: 'model_substruct.*' (5 layers), 'model_context.*' (3 layers), GIN."""
    dt = L["model_substruct.gnns.0.edge_encoder.bias"].dtype
    B = b["center_substruct_idx"].shape[0]
    s = O.bio_gnn(sub(L, "model_substruct."), _float(b["x_substruct"], dt), b["edge_index_substruct"], _float(b["edge_attr_substruct"], dt),
                  5, "gin", True)
    c = O.bio_gnn(sub(L, "model_context."), _float(b["x_context"], dt), b["edge_index_context"], _float(b["edge_attr_context"], dt),
                  3, "gin", True)
    pos, neg = O.contextpred_scores(s[b["center_substruct_idx"]], c[b["overlap_context_substruct_idx"]], b["batch_overlapped_context"], B,
                                    neg_samples)
    return O.contextpred_loss(pos, neg, neg_samples), dict(pos=pos, neg=neg)


def make_params(config, seed, gnn_type="gin"):
    """config: 'bio_masking' (encoder of `gnn_type` + the edge-type head) or 'bio_contextpred' (two GIN encoders)."""
    g = torch.Generator().manual_seed(seed + 977)
    P = {}
    if config == "bio_masking":
        P.update({"model." + k: v for k, v in O.make_params("bio", gnn_type, 5, 300, seed).items()})
        P["head.weight"] = torch.randn(NUM_EDGE_TYPES, 300, generator=g) * 0.05
        P["head.bias"] = torch.randn(NUM_EDGE_TYPES, generator=g) * 0.05
    elif config == "bio_contextpred":
        P.update({"model_substruct." + k: v for k, v in O.make_params("bio", "gin", 5, 300, seed).items()})
        P.update({"model_context." + k: v for k, v in O.make_params("bio", "gin", 3, 300, seed + 1).items()})
    else:
        raise ValueError(config)
    return P


class ReferenceBioMaskingStep(_RefStep):
    def __init__(self, gnn_type="gin"):
        from oracle import reference_runner as R
        mod = R.load("bio")
        self.model = mod.GNN(5, 300, JK="last", drop_ratio=0, gnn_type=gnn_type).train()
        self.head = torch.nn.Linear(300, NUM_EDGE_TYPES)
        self.criterion = torch.nn.CrossEntropyLoss()
        self.named = {"model": self.model, "head": self.head}
        self.modules = list(self.named.values())

    def __call__(self, b):
        self.zero_grad()
        node_rep = self.model(b["x"], b["edge_index"], b["edge_attr"])
        masked_edge_index = b["edge_index"][:, b["masked_edge_idx"]]
        edge_rep = node_rep[masked_edge_index[0]] + node_rep[masked_edge_index[1]]
        pred_edge = self.head(edge_rep)
        edge_label = torch.argmax(b["mask_edge_label"], dim=1)
        loss = self.criterion(pred_edge, edge_label)
        loss.backward()
        return loss


def _cycle_index(num, shift):
    """bio/pretrain_contextpred.py:32-35."""
    arr = torch.arange(num) + shift
    arr[-shift:] = torch.arange(shift)
    return arr


class ReferenceBioContextPredStep(_RefStep):
    def __init__(self, neg_samples=1):
        from oracle import reference_runner as R
        mod = R.load("bio")
        self.neg_samples = neg_samples
        self.model_substruct = mod.GNN(5, 300, JK="last", drop_ratio=0, gnn_type="gin").train()
        self.model_context = mod.GNN(3, 300, JK="last", drop_ratio=0, gnn_type="gin").train()
        self.pool = mod.global_mean_pool
        self.criterion = torch.nn.BCEWithLogitsLoss()
        self.named = {"model_substruct": self.model_substruct, "model_context": self.model_context}
        self.modules = list(self.named.values())

    def __call__(self, b):
        self.zero_grad()
        substruct_rep = self.model_substruct(b["x_substruct"], b["edge_index_substruct"], b["edge_attr_substruct"])[b["center_substruct_idx"]]
        overlapped_node_rep = self.model_context(b["x_context"], b["edge_index_context"], b["edge_attr_context"])[b["overlap_context_substruct_idx"]]
        context_rep = self.pool(overlapped_node_rep, b["batch_overlapped_context"])
        neg_context_rep = torch.cat([context_rep[_cycle_index(len(context_rep), i + 1)] for i in range(self.neg_samples)], dim=0)
        pred_pos = torch.sum(substruct_rep * context_rep, dim=1)
        pred_neg = torch.sum(substruct_rep.repeat((self.neg_samples, 1)) * neg_context_rep, dim=1)
        loss_pos = self.criterion(pred_pos.double(), torch.ones(len(pred_pos)).double())
        loss_neg = self.criterion(pred_neg.double(), torch.zeros(len(pred_neg)).double())
        loss = loss_pos + self.neg_samples * loss_neg
        loss.backward()
        return loss
