"""Edge-prediction pre-training on the device (chem/pretrain_edgepred.py, bio/pretrain_edgepred.py), the optimizer step excluded:
  * graphs/s of train_steps.EdgePredStep for every gnn_type and of BioEdgePredStep (GIN by default) on device-resident batches;
  * the NegativeEdge transform at B graphs: data.negative_edges on the collated batch (device), synthetic.negative_edge_index (the
    vectorised numpy restatement) and the oracle's literal per-graph loop of tests/edgepred_oracle.py (the reference's algorithm,
    timed on the first --loop-graphs graphs and reported per graph);
  * the head at bio size: ops.edge_pair_bce forward and forward + backward against the torch composition (index_select, multiply,
    sum, fp64 BCE, autograd).
Device times are CUDA events after warm-up, host times perf_counter; the card's name and power limit are read in the same run.
Prints one JSON line per measurement.

    python tools/bench_edgepred.py [--types gin,gcn,graphsage,gat] [--bio-types gin] [--batch 256] [--steps 20] [--warmup 5]

Needs a GPU."""
import argparse
import importlib
import json
import os
import subprocess
import sys
import time
from types import SimpleNamespace

import torch
import torch.nn.functional as F

ap = argparse.ArgumentParser()
ap.add_argument("--types", default="gin,gcn,graphsage,gat")
ap.add_argument("--bio-types", default="gin")
ap.add_argument("--batch", type=int, default=256)
ap.add_argument("--steps", type=int, default=20)
ap.add_argument("--warmup", type=int, default=5)
ap.add_argument("--batches", type=int, default=2, help="distinct device-resident batches cycled through")
ap.add_argument("--loop-graphs", type=int, default=16, help="graphs the oracle's literal loop is timed on")
a = ap.parse_args()
if not torch.cuda.is_available():
    sys.exit("bench_edgepred.py needs a GPU")
ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
ts = importlib.import_module("pretrain-gnns_b200.train_steps")
syn = importlib.import_module("pretrain-gnns_b200.synthetic")
ops = importlib.import_module("pretrain-gnns_b200.ops")
data = importlib.import_module("pretrain-gnns_b200.data")
import edgepred_oracle as EO  # noqa: E402

dev = torch.device("cuda:0")


def card():
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "unknown"
    return dict(card=torch.cuda.get_device_name(0), power_limit_and_max_sm_clock=q)


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def emit(d):
    print(json.dumps(d | info), flush=True)


def run_step(step, host_batches, name):
    batches = [{k: v.to(dev) for k, v in b.items() if torch.is_tensor(v)} for b in host_batches]
    i = [0]

    def one():
        step(batches[i[0] % len(batches)])
        i[0] += 1

    ms = timed(one, a.steps, a.warmup)
    loss = float(step(batches[0]))
    emit(dict(step=name, B=a.batch, ms_per_step=round(ms, 3), graphs_per_s=round(a.batch / ms * 1e3, 1), loss=loss, steps=a.steps,
              pairs=int(batches[0]["edge_index"].shape[1] // 2 + batches[0]["negative_edge_index"].shape[1])))


info = card()
emit(dict(what="card"))
chem_host = bio_host = None
for t in a.types.split(","):
    step = ts.EdgePredStep(dev, t, batch_size=a.batch)
    chem_host = chem_host or step.make_batches(0, a.batches)
    run_step(step, chem_host, "edgepred_chem_" + t)
    del step
for t in a.bio_types.split(","):
    step = ts.BioEdgePredStep(dev, t, batch_size=a.batch)
    bio_host = bio_host or step.make_batches(0, a.batches)
    run_step(step, bio_host, "edgepred_bio_" + t)
    del step


# the transform alone
def transform(domain, b, seed=123):
    node_off, edge_off = b["ptr"], torch.from_numpy(syn.edge_offsets(b))
    nb = SimpleNamespace(edge_index=b["edge_index"].to(dev), node_off=node_off.to(dev), edge_off=edge_off.to(dev))
    eoff_host = edge_off.numpy()
    ms = timed(lambda: data.negative_edges(nb, eoff_host, seed), 20, 3)
    ei, no = b["edge_index"].numpy(), node_off.numpy()
    t0 = time.perf_counter()
    host = syn.negative_edge_index(ei, no, eoff_host, seed)
    t_host = time.perf_counter() - t0
    G = min(a.loop_graphs, len(no) - 1)
    t0 = time.perf_counter()
    EO.negative_edges_batch(ei[:, :eoff_host[G]], no[:G + 1], eoff_host[:G + 1], seed)
    t_loop = (time.perf_counter() - t0) / G
    same = bool(torch.equal(nb.negative_edge_index.cpu(), torch.from_numpy(host)))
    emit(dict(what="negative_edges", domain=domain, B=len(no) - 1, E=int(ei.shape[1]), M=int(host.shape[1]), device_ms=round(ms, 4),
              host_vectorised_ms=round(t_host * 1e3, 2), oracle_loop_ms_per_graph=round(t_loop * 1e3, 2), oracle_loop_graphs=G,
              device_equals_host=same))


transform("chem", syn.zinc_batch(a.batch, 8000))
transform("bio", syn.ppi_batch(a.batch, 9000))

# the head alone, at bio size
bb = syn.bio_edgepred_batch(a.batch, 9001) if bio_host is None else None
ei = (bio_host[0] if bio_host else bb)["edge_index"].to(dev)
neg = (bio_host[0] if bio_host else bb)["negative_edge_index"].to(dev)
N = int(ei.max()) + 1
g = torch.Generator(device=dev).manual_seed(0)
x = (torch.randn(N, 300, device=dev, generator=g) * 0.05).requires_grad_(True)
pos = ei[:, ::2]


def lib_fwd():
    with torch.no_grad():
        ops.edge_pair_bce(x, pos, neg)


def lib_fwd_bwd():
    x.grad = None
    ops.edge_pair_bce(x, pos, neg)[0].backward()


def torch_fwd():
    with torch.no_grad():
        torch_loss()


def torch_loss():
    p = (x.index_select(0, pos[0]) * x.index_select(0, pos[1])).sum(1).double()
    q = (x.index_select(0, neg[0]) * x.index_select(0, neg[1])).sum(1).double()
    return F.binary_cross_entropy_with_logits(p, torch.ones_like(p)) + F.binary_cross_entropy_with_logits(q, torch.zeros_like(q))


def torch_fwd_bwd():
    x.grad = None
    torch_loss().backward()


res = {}
for _ in range(3):   # alternate, three rounds
    for name, fn in (("edge_pair_bce_fwd", lib_fwd), ("torch_fwd", torch_fwd), ("edge_pair_bce_fwd_bwd", lib_fwd_bwd),
                     ("torch_fwd_bwd", torch_fwd_bwd)):
        res.setdefault(name, []).append(round(timed(fn, 20, 3) * 1e3, 1))
l_lib = float(ops.edge_pair_bce(x, pos, neg)[0])
l_torch = float(torch_loss())
emit(dict(what="edge_pair_bce", N=N, P=int(pos.shape[1]), Q=int(neg.shape[1]), us_per_call=res, loss=l_lib, loss_torch=l_torch))
