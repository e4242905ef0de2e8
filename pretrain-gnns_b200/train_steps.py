"""The `train()` bodies of the reference's pre-training scripts on the library's modules — one callable per BASELINE config.

Each class owns the modules the script builds, draws the synthetic batches of its config (SURVEY.md 8(d)) and, called
on one device-resident batch, runs exactly what the script runs between `batch.to(device)` and `optimizer.step()`:
zero the gradients, forward, the script's own loss head, `loss.backward()`.  The optimizer step is outside (SURVEY.md
8(d) defines the metric without it).  bench.py times these; the parity tests compare them with the oracle's
restatement of the same bodies (oracle/steps_oracle.py) and with the reference's own modules.

    MaskingStep        chem/pretrain_masking.py:46-70     GNN(5,300,gnn_type) + Linear(300,119), CE on fp64 logits
    ContextPredStep    chem/pretrain_contextpred.py:50-97 GNN(5,300) + GNN(3,300), cbow / mean pooling, BCE on fp64 scores
    BioSupervisedStep  bio/pretrain_supervised.py:25-42   bio GNN_graphpred(5,300,T=5000), BCE on fp64 logits
    FinetuneStep       chem/finetune.py:27-46             chem GNN_graphpred(5,300,T=12) with dropout 0.5, masked BCE on fp64
                                                          logits (not a bench.py config: it is not in CONFIGS)
    BioMaskingStep     bio/pretrain_masking.py:39-55      bio GNN(5,300,gnn_type) + Linear(300,7), CE against the argmax of the
                                                          masked edges' label rows (not in CONFIGS)
    BioContextPredStep bio/pretrain_contextpred.py:43-97  bio GNN(5,300) + GNN(3,300), cbow / mean pooling, BCE on fp64 scores
                                                          (not in CONFIGS)
    EdgePredStep       chem/pretrain_edgepred.py:31-41    GNN(5,300,gnn_type), BCE of the dot products of the bonds and of the
                                                          NegativeEdge pairs, on fp64 (not in CONFIGS)
    BioEdgePredStep    bio/pretrain_edgepred.py           the same on bio GNN(5,300,gnn_type) (not in CONFIGS)
    InfomaxStep        chem/pretrain_deepgraphinfomax.py:59-74
                                                          GNN(5,300,gnn_type) + Discriminator(300), BCE of each node's score
                                                          against its graph's sigmoid mean-pool summary and the next graph's,
                                                          on fp64 (not in CONFIGS)
    BioInfomaxStep     bio/pretrain_deepgraphinfomax.py   the same on bio GNN(5,300,gnn_type) (not in CONFIGS)
"""
from __future__ import annotations

import math
import types

import torch

from . import ops, synthetic as syn
from .bio import model as bio
from .chem import model as chem

NUM_LAYER, EMB = 5, 300


def _fields(b, keys):
    return {k: b[k] for k in keys}


CONFIG_ID = {"masking": 2, "contextpred": 3, "bio_supervised": 4, "gcn": 2, "gat": 2, "graphsage": 2}
DEFAULT_BATCH = {"masking": 256, "contextpred": 128, "bio_supervised": 64, "gcn": 256, "gat": 256, "graphsage": 256}
MASKING_KEYS = ("x", "edge_index", "edge_attr", "masked_atom_indices")
CONTEXT_KEYS = ("x_substruct", "edge_index_substruct", "edge_attr_substruct", "center_substruct_idx", "x_context", "edge_index_context",
                "edge_attr_context", "overlap_context_substruct_idx", "batch_overlapped_context")
BIO_KEYS = ("x", "edge_index", "edge_attr", "batch", "center_node_idx", "go_target_pretrain")
FINETUNE_KEYS = ("x", "edge_index", "edge_attr", "batch", "y")
FINETUNE_SEED = 5  # seed = 5 * 1000 + 1000 * rank + batch index, in the scheme of make_batches
BIO_MASKING_KEYS = ("x", "edge_index", "edge_attr", "masked_edge_idx", "mask_edge_label")
BIO_MASKING_SEED, BIO_CONTEXT_SEED = 6, 7
EDGEPRED_KEYS = ("x", "edge_index", "edge_attr", "negative_edge_index")
EDGEPRED_SEED, BIO_EDGEPRED_SEED = 8, 9
INFOMAX_KEYS = ("x", "edge_index", "edge_attr", "batch")
INFOMAX_SEED, BIO_INFOMAX_SEED = 10, 11


def make_batches(config, rank, count, batch_size=None, num_tasks=5000):
    """Host (CPU tensor) batches of one config: seed = config-id * 1000 + 1000 * rank + batch index (SURVEY.md 8(d))."""
    B = batch_size or DEFAULT_BATCH[config]
    out = []
    for i in range(count):
        seed = CONFIG_ID[config] * 1000 + 1000 * rank + i
        if config == "contextpred":
            out.append(_fields(syn.substruct_context_batch(B, seed), CONTEXT_KEYS))
        elif config == "bio_supervised":
            out.append(_fields(syn.ppi_batch(B, seed, num_tasks=num_tasks), BIO_KEYS))
        else:
            b = syn.mask_atoms(syn.zinc_batch(B, seed), seed)
            out.append(_fields(b, MASKING_KEYS) | {"labels": b["mask_node_label"][:, 0].contiguous()})
    return out


class _Step:
    modules: list

    def parameters(self):
        # the module set of a step is fixed: walk it once (nn.Module.parameters() re-traverses every submodule on each call,
        # ~200 us of host time per training step when zero_grad does it)
        ps = getattr(self, "_params", None)
        if ps is None:
            ps = self._params = [p for m in self.modules for p in m.parameters()]
        return ps

    def zero_grad(self):
        for p in self.parameters():
            p.grad = None

    def flat_sources(self):
        """(module, ...) whose fused backward leaves one flat gradient buffer (dist.encoder_flat_source)."""
        return []

    def named_modules(self):
        return {}

    def load_state(self, P):
        """P: one flat dict keyed `<attribute>.<state_dict key>` ('model.gnns.0...', 'head.weight', ...)."""
        for name, m in self.named_modules().items():
            dev = next(m.parameters()).device
            m.load_state_dict({k[len(name) + 1:]: v for k, v in P.items() if k.startswith(name + ".")})
            m.to(dev)

    def named_parameters(self):
        return [(name + "." + k, p) for name, m in self.named_modules().items() for k, p in m.named_parameters()]


class MaskingStep(_Step):
    """chem/pretrain_masking.py:46-70 (mask_edge off, the script's default): node_rep = model(x, ei, ea);
    pred = linear_pred_atoms(node_rep[masked_atom_indices]); loss = CE(pred.double(), mask_node_label[:,0])."""
    def __init__(self, device, gnn_type="gin", batch_size=256):
        self.graphs_per_batch = batch_size
        self.config = "masking" if gnn_type == "gin" else gnn_type
        self.model = chem.GNN(NUM_LAYER, EMB, JK="last", drop_ratio=0, gnn_type=gnn_type).to(device).train()
        self.head = torch.nn.Linear(EMB, 119).to(device)
        self.modules = [self.model, self.head]
        self.workload = ("chem pretrain_masking 5-layer %s emb_dim=300 batch_size=%d (BASELINE configs[%d])"
                         % (gnn_type.upper() if gnn_type != "graphsage" else "GraphSAGE", batch_size, 1 if gnn_type == "gin" else 4))

    def make_batches(self, rank, count):
        return make_batches(self.config, rank, count, self.graphs_per_batch)

    def flat_sources(self):
        return [self.model]

    def named_modules(self):
        return {"model": self.model, "head": self.head}

    def __call__(self, b):
        self.zero_grad()
        rep = self.model(b["x"], b["edge_index"], b["edge_attr"])
        loss, _ = ops.masked_atom_loss(rep, b["masked_atom_indices"], b["labels"], self.head.weight, self.head.bias)
        loss.backward()
        return loss


class ContextPredStep(_Step):
    """chem/pretrain_contextpred.py:50-97 with the script's defaults: num_layer 5, csize 3 -> context encoder of
    l2 - l1 = 7 - 4 = 3 layers (:145-146,156-157), mode cbow, context_pooling mean, neg_samples 1.
    `encoder`: the GNN class of both encoders, `source(B, seed)`: the host batch of one step, drawn with seed
    seed_base * 1000 + 1000 * rank + batch index (BioContextPredStep passes the bio ones)."""
    def __init__(self, device, batch_size=128, neg_samples=1, encoder=chem.GNN, source=syn.substruct_context_batch,
                 seed_base=CONFIG_ID["contextpred"]):
        self.graphs_per_batch, self.neg_samples = batch_size, neg_samples
        self.source, self.seed_base = source, seed_base
        self.model_substruct = encoder(NUM_LAYER, EMB, JK="last", drop_ratio=0, gnn_type="gin").to(device).train()
        self.model_context = encoder(3, EMB, JK="last", drop_ratio=0, gnn_type="gin").to(device).train()
        self.modules = [self.model_substruct, self.model_context]
        self.concurrent, self._side = True, None   # context encoder on a second CUDA stream (see scores)
        self.workload = "chem pretrain_contextpred 5-layer GIN emb_dim=300 batch_size=%d, substruct + 3-layer context encoder (BASELINE configs[2])" % batch_size

    KEYS = CONTEXT_KEYS

    def make_batches(self, rank, count):
        return [_fields(self.source(self.graphs_per_batch, self.seed_base * 1000 + 1000 * rank + i), CONTEXT_KEYS) for i in range(count)]

    def flat_sources(self):
        return [self.model_substruct, self.model_context]

    def named_modules(self):
        return {"model_substruct": self.model_substruct, "model_context": self.model_context}

    def scores(self, b):
        B = b["center_substruct_idx"].shape[0]
        # The two encoders are independent until the dot products (the script runs them back to back, :54-57), and at
        # B = 128 neither fills the chip (17 and 10 row tiles of 128 nodes): the context encoder runs on a second stream,
        # forward and — autograd replays a node's backward on its forward stream — backward alike.
        main = torch.cuda.current_stream() if b["x_context"].is_cuda else None
        if main is not None and self.concurrent:
            if self._side is None:
                self._side = torch.cuda.Stream(b["x_context"].device)
            self._side.wait_stream(main)
            with torch.cuda.stream(self._side):
                ov = ops.row_gather(self.model_context(b["x_context"], b["edge_index_context"], b["edge_attr_context"]),
                                    b["overlap_context_substruct_idx"])
            ov.record_stream(main)
        else:
            ov = ops.row_gather(self.model_context(b["x_context"], b["edge_index_context"], b["edge_attr_context"]),
                                b["overlap_context_substruct_idx"])
        sub = ops.row_gather(self.model_substruct(b["x_substruct"], b["edge_index_substruct"], b["edge_attr_substruct"]),
                             b["center_substruct_idx"])
        if main is not None and self.concurrent:
            main.wait_stream(self._side)
        ctx = ops.global_mean_pool(ov, b["batch_overlapped_context"], B)   # one segment per graph of the batch
        pos = ops.shifted_rowdot(sub, ctx, 0)
        neg = torch.cat([ops.shifted_rowdot(sub, ctx, i + 1) for i in range(self.neg_samples)], dim=0)
        return pos, neg

    def __call__(self, b):
        self.zero_grad()
        pos, neg = self.scores(b)
        loss = ops.bce_with_logits_const(pos, 1.0) + self.neg_samples * ops.bce_with_logits_const(neg, 0.0)
        loss.backward()
        return loss


class BioSupervisedStep(_Step):
    """bio/pretrain_supervised.py:25-42: pred = model(batch); loss = BCEWithLogits(pred.double(), y.double()).
    drop_ratio = 0 (the script's default is 0.2; dropout has no RNG parity, SURVEY.md 8(d) config 4)."""
    def __init__(self, device, gnn_type="gin", batch_size=64, num_tasks=5000):
        self.graphs_per_batch, self.num_tasks = batch_size, num_tasks
        self.model = bio.GNN_graphpred(NUM_LAYER, EMB, num_tasks, JK="last", drop_ratio=0, graph_pooling="mean", gnn_type=gnn_type).to(device).train()
        self.modules = [self.model]
        self.workload = "bio pretrain_supervised 5-layer GIN emb_dim=300 PPI-ego-shaped graphs batch_size=%d T=%d (BASELINE configs[3])" % (batch_size, num_tasks)

    KEYS = BIO_KEYS

    def make_batches(self, rank, count):
        return make_batches("bio_supervised", rank, count, self.graphs_per_batch, self.num_tasks)

    def flat_sources(self):
        return [self.model.gnn]

    def named_modules(self):
        return {"model": self.model}

    def __call__(self, b):
        self.zero_grad()
        pred = self.model(types.SimpleNamespace(**b))
        loss = ops.bce_with_logits(pred, b["go_target_pretrain"].view(pred.shape))
        loss.backward()
        return loss


class BioMaskingStep(_Step):
    """bio/pretrain_masking.py:39-55 with the script's defaults (num_layer 5, emb_dim 300, dropout 0, mask_rate 0.15, batch_size 256,
    any gnn_type): node_rep = model(x, ei, ea) on the MaskEdge'd batch; pred = linear_pred_edges(node_rep[u] + node_rep[v]) over
    edge_index[:, masked_edge_idx]; loss = CE(pred, argmax(mask_edge_label, 1)), evaluated in fp64 (the script: fp32)."""
    def __init__(self, device, gnn_type="gin", batch_size=256, mask_rate=0.15):
        self.graphs_per_batch, self.mask_rate = batch_size, mask_rate
        self.model = bio.GNN(NUM_LAYER, EMB, JK="last", drop_ratio=0, gnn_type=gnn_type).to(device).train()
        self.head = torch.nn.Linear(EMB, 7).to(device)
        self.modules = [self.model, self.head]
        self.workload = ("bio pretrain_masking 5-layer %s emb_dim=300 PPI-ego-shaped graphs batch_size=%d mask_rate=%g"
                         % (gnn_type.upper() if gnn_type != "graphsage" else "GraphSAGE", batch_size, mask_rate))

    KEYS = BIO_MASKING_KEYS

    def make_batches(self, rank, count):
        return [_fields(syn.bio_masking_batch(self.graphs_per_batch, BIO_MASKING_SEED * 1000 + 1000 * rank + i, self.mask_rate), BIO_MASKING_KEYS)
                for i in range(count)]

    def flat_sources(self):
        return [self.model]

    def named_modules(self):
        return {"model": self.model, "head": self.head}

    def __call__(self, b):
        self.zero_grad()
        rep = self.model(b["x"], b["edge_index"], b["edge_attr"])
        loss, _ = ops.masked_edge_type_loss(rep, b["edge_index"], b["masked_edge_idx"], b["mask_edge_label"], self.head.weight, self.head.bias)
        loss.backward()
        return loss


class BioContextPredStep(ContextPredStep):
    """bio/pretrain_contextpred.py:43-97 with the script's defaults (num_layer 5, emb_dim 300, batch_size 256, l1 1, center 0, mode
    cbow, context_pooling mean, neg_samples 1): bio GNN(5, 300) over the whole ego graphs read at their centre nodes, bio
    GNN(3, 300) over the context (the nodes further than l1 hops from a random root), then ContextPredStep's head."""
    def __init__(self, device, batch_size=256, neg_samples=1, l1=1):
        super().__init__(device, batch_size, neg_samples, encoder=bio.GNN, source=lambda B, seed: syn.bio_context_batch(B, seed, l1),
                         seed_base=BIO_CONTEXT_SEED)
        self.l1 = l1
        self.workload = ("bio pretrain_contextpred 5-layer GIN emb_dim=300 PPI-ego-shaped graphs batch_size=%d l1=%d, substruct + 3-layer "
                         "context encoder" % (batch_size, l1))


class EdgePredStep(_Step):
    """chem/pretrain_edgepred.py:31-41 with the script's defaults (num_layer 5, emb_dim 300, JK last, dropout 0, batch_size 256, any
    gnn_type): node_emb = model(x, ei, ea); pos = sum(node_emb[ei[0, ::2]] * node_emb[ei[1, ::2]], 1), neg likewise over
    negative_edge_index; loss = BCEWithLogits(pos, 1) + BCEWithLogits(neg, 0), evaluated in fp64 (the script: fp32)."""
    encoder, source, seed_base, domain = chem.GNN, staticmethod(syn.edgepred_batch), EDGEPRED_SEED, "chem"

    def __init__(self, device, gnn_type="gin", batch_size=256):
        self.graphs_per_batch = batch_size
        self.model = self.encoder(NUM_LAYER, EMB, JK="last", drop_ratio=0, gnn_type=gnn_type).to(device).train()
        self.modules = [self.model]
        self.workload = ("%s pretrain_edgepred 5-layer %s emb_dim=300 batch_size=%d"
                         % (self.domain, gnn_type.upper() if gnn_type != "graphsage" else "GraphSAGE", batch_size))

    KEYS = EDGEPRED_KEYS

    def make_batches(self, rank, count):
        return [_fields(self.source(self.graphs_per_batch, self.seed_base * 1000 + 1000 * rank + i), EDGEPRED_KEYS) for i in range(count)]

    def flat_sources(self):
        return [self.model]

    def named_modules(self):
        return {"model": self.model}

    def scores(self, b):
        """-> (loss, pos, neg): the loss and the two score vectors (the script's train_acc reads them)."""
        rep = self.model(b["x"], b["edge_index"], b["edge_attr"])
        return ops.edge_pair_bce(rep, b["edge_index"][:, ::2], b["negative_edge_index"])

    def __call__(self, b):
        self.zero_grad()
        loss, _, _ = self.scores(b)
        loss.backward()
        return loss


class BioEdgePredStep(EdgePredStep):
    """bio/pretrain_edgepred.py: EdgePredStep's body on bio GNN(5, 300) over PPI ego graphs."""
    encoder, source, seed_base, domain = bio.GNN, staticmethod(syn.bio_edgepred_batch), BIO_EDGEPRED_SEED, "bio"


class Discriminator(torch.nn.Module):
    """The Discriminator of chem/pretrain_deepgraphinfomax.py:30-42 (bio alike): weight [D, D] drawn by
    torch_geometric.nn.inits.uniform(D, weight), i.e. U(-1/sqrt(D), 1/sqrt(D)), so the same torch.manual_seed draws the same
    values.  forward(x, summary) = sum(x * (summary @ weight), 1), as the script's; InfomaxStep calls ops.infomax_bce instead."""
    def __init__(self, hidden_dim):
        super().__init__()
        self.weight = torch.nn.Parameter(torch.empty(hidden_dim, hidden_dim))
        self.reset_parameters()

    def reset_parameters(self):
        bound = 1.0 / math.sqrt(self.weight.size(0))
        self.weight.data.uniform_(-bound, bound)

    def forward(self, x, summary):
        return torch.sum(x * torch.matmul(summary, self.weight), dim=1)


class InfomaxStep(_Step):
    """chem/pretrain_deepgraphinfomax.py:59-74 with the script's defaults (num_layer 5, emb_dim 300, JK last, dropout 0, batch_size
    256, any gnn_type): node_emb = gnn(x, ei, ea); summary = sigmoid(global_mean_pool(node_emb, batch)); pos / neg = the
    Discriminator's scores against each node's own summary and against the next graph's (cycle_index(G, 1)); loss =
    BCEWithLogits(pos, 1) + BCEWithLogits(neg, 0), evaluated in fp64 (the script: fp32).  The modules are named as Infomax names
    them ('gnn', 'discriminator'), so load_state takes Infomax.state_dict()'s keys as they are."""
    encoder, source, seed_base, domain = chem.GNN, staticmethod(syn.zinc_batch), INFOMAX_SEED, "chem"

    def __init__(self, device, gnn_type="gin", batch_size=256):
        self.graphs_per_batch = batch_size
        self.gnn = self.encoder(NUM_LAYER, EMB, JK="last", drop_ratio=0, gnn_type=gnn_type).to(device).train()
        self.discriminator = Discriminator(EMB).to(device)
        self.modules = [self.gnn, self.discriminator]
        self.workload = ("%s pretrain_deepgraphinfomax 5-layer %s emb_dim=300 batch_size=%d"
                         % (self.domain, gnn_type.upper() if gnn_type != "graphsage" else "GraphSAGE", batch_size))

    KEYS = INFOMAX_KEYS

    def make_batches(self, rank, count):
        """Host batches (INFOMAX_KEYS + 'num_graphs', an int: the graph count is known on the host, so the step reads nothing back)."""
        out = []
        for i in range(count):
            b = self.source(self.graphs_per_batch, self.seed_base * 1000 + 1000 * rank + i)
            out.append(_fields(b, INFOMAX_KEYS) | {"num_graphs": b["num_graphs"]})
        return out

    def flat_sources(self):
        return [self.gnn]

    def named_modules(self):
        return {"gnn": self.gnn, "discriminator": self.discriminator}

    def scores(self, b):
        """-> (loss, pos, neg): the loss and the two score vectors (the script's train_acc reads them).  b["num_graphs"], when
        present, is G; otherwise G = batch.max() + 1 is read back, as global_mean_pool does."""
        node_emb = self.gnn(b["x"], b["edge_index"], b["edge_attr"])
        return ops.infomax_bce(node_emb, b["batch"], self.discriminator.weight, b.get("num_graphs"))

    def __call__(self, b):
        self.zero_grad()
        loss, _, _ = self.scores(b)
        loss.backward()
        return loss


class BioInfomaxStep(InfomaxStep):
    """bio/pretrain_deepgraphinfomax.py: InfomaxStep's body on bio GNN(5, 300) over PPI ego graphs."""
    encoder, source, seed_base, domain = bio.GNN, staticmethod(syn.ppi_batch), BIO_INFOMAX_SEED, "bio"


class FinetuneStep(_Step):
    """chem/finetune.py:27-46 with the script's defaults (num_layer 5, emb_dim 300, JK last, dropout_ratio 0.5, graph_pooling
    mean, batch_size 32; T = 12 tasks is tox21): pred = model(x, edge_index, edge_attr, batch); loss = BCEWithLogits(pred.double(),
    (y+1)/2) over the entries with y != 0, divided by their number.  The dropout masks come from the library's draw, one seed per
    forward from torch's default generator (torch.manual_seed makes a run reproducible)."""
    def __init__(self, device, gnn_type="gin", batch_size=32, num_tasks=12, drop_ratio=0.5):
        self.graphs_per_batch, self.num_tasks = batch_size, num_tasks
        self.model = chem.GNN_graphpred(NUM_LAYER, EMB, num_tasks, JK="last", drop_ratio=drop_ratio, graph_pooling="mean",
                                        gnn_type=gnn_type).to(device).train()
        self.modules = [self.model]
        self.workload = ("chem finetune 5-layer %s emb_dim=300 dropout=%g batch_size=%d T=%d"
                         % (gnn_type.upper() if gnn_type != "graphsage" else "GraphSAGE", drop_ratio, batch_size, num_tasks))

    KEYS = FINETUNE_KEYS

    def make_batches(self, rank, count):
        return [_fields(syn.finetune_batch(self.graphs_per_batch, FINETUNE_SEED * 1000 + 1000 * rank + i, self.num_tasks), FINETUNE_KEYS)
                for i in range(count)]

    def flat_sources(self):
        return [self.model.gnn]

    def named_modules(self):
        return {"model": self.model}

    def __call__(self, b):
        self.zero_grad()
        pred = self.model(b["x"], b["edge_index"], b["edge_attr"], b["batch"])
        loss = ops.masked_bce_with_logits(pred, b["y"].view(pred.shape))
        loss.backward()
        return loss


CONFIGS = {
    "masking": lambda dev: MaskingStep(dev, "gin"),
    "contextpred": lambda dev: ContextPredStep(dev),
    "bio_supervised": lambda dev: BioSupervisedStep(dev),
    "gcn": lambda dev: MaskingStep(dev, "gcn"),
    "gat": lambda dev: MaskingStep(dev, "gat"),
    "graphsage": lambda dev: MaskingStep(dev, "graphsage"),
}
