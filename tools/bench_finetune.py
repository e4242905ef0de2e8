"""Graphs/s of the chem fine-tuning step (chem/finetune.py:27-46: GNN_graphpred(5, 300, T) with dropout, masked BCE; the optimizer
step excluded), device-resident batches, for every gnn_type at B = 32 and 256, plus the CUDA kernels one step launches.  Prints
one JSON line per (type, B).

    python tools/bench_finetune.py [--root TREE] [--types gin,gcn] [--batch 32,256] [--drop 0.5] [--steps 50] [--warmup 10]

--root imports the package from another checkout (e.g. an older one, to compare): a tree without train_steps.FinetuneStep is
measured on the same body built from its GNN_graphpred, i.e. whatever that tree does for dropout.  Needs a GPU."""
import argparse
import importlib
import json
import os
import sys

import numpy as np
import torch

ap = argparse.ArgumentParser()
ap.add_argument("--root", default=os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
ap.add_argument("--types", default="gin,gcn,graphsage,gat")
ap.add_argument("--batch", default="32,256")
ap.add_argument("--drop", type=float, default=0.5)
ap.add_argument("--tasks", type=int, default=12)
ap.add_argument("--steps", type=int, default=50)
ap.add_argument("--warmup", type=int, default=10)
ap.add_argument("--label", default="")
a = ap.parse_args()
if not torch.cuda.is_available():
    sys.exit("bench_finetune.py needs a GPU")
sys.path.insert(0, os.path.abspath(a.root))
ts = importlib.import_module("pretrain-gnns_b200.train_steps")
syn = importlib.import_module("pretrain-gnns_b200.synthetic")
ops = importlib.import_module("pretrain-gnns_b200.ops")
chem = importlib.import_module("pretrain-gnns_b200.chem.model")
dev = torch.device("cuda:0")


def batch(B, seed, T):
    if hasattr(syn, "finetune_batch"):
        return syn.finetune_batch(B, seed, T)
    out = syn.zinc_batch(B, seed)  # the same labels synthetic.finetune_batch draws
    rng = np.random.default_rng(seed + 2750159)
    y = np.where(rng.random((B, T)) < 0.5, 1, -1)
    y[rng.random((B, T)) < 0.2] = 0
    out["y"] = torch.from_numpy(y).to(torch.int64)
    return out


class _Body:
    """FinetuneStep's body on a tree that lacks the class."""

    def __init__(self, t, T, p):
        self.model = chem.GNN_graphpred(5, 300, T, JK="last", drop_ratio=p, graph_pooling="mean", gnn_type=t).to(dev).train()

    def __call__(self, b):
        for q in self.model.parameters():
            q.grad = None
        pred = self.model(b["x"], b["edge_index"], b["edge_attr"], b["batch"])
        loss = ops.masked_bce_with_logits(pred, b["y"].view(pred.shape))
        loss.backward()
        return loss


def kernels_per_step(step, b):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step(b)
        torch.cuda.synchronize()
    return sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and not e.name.startswith("Memcpy")
               and not e.name.startswith("Memset"))


name = torch.cuda.get_device_name(0)
for t in a.types.split(","):
    for B in (int(x) for x in a.batch.split(",")):
        torch.manual_seed(0)
        step = (ts.FinetuneStep(dev, t, batch_size=B, num_tasks=a.tasks, drop_ratio=a.drop) if hasattr(ts, "FinetuneStep")
                else _Body(t, a.tasks, a.drop))
        batches = [{k: v.to(dev) for k, v in batch(B, 5000 + i, a.tasks).items() if torch.is_tensor(v)} for i in range(8)]
        for i in range(a.warmup):
            step(batches[i % 8])
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(a.steps):
            loss = step(batches[i % 8])
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / a.steps
        print(json.dumps(dict(label=a.label, gnn_type=t, B=B, drop=a.drop, ms_per_step=round(ms, 4),
                              graphs_per_s=round(B / ms * 1e3, 1), kernels_per_step=kernels_per_step(step, batches[0]),
                              loss=loss.item(), card=name)), flush=True)
