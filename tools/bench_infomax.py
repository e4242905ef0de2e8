"""Deep Graph Infomax pre-training on the device (chem/pretrain_deepgraphinfomax.py, bio/pretrain_deepgraphinfomax.py), the
optimizer step excluded:
  * graphs/s of train_steps.InfomaxStep for every gnn_type and of BioInfomaxStep (GIN by default) on device-resident batches;
  * the head alone at chem size (N ~ 6 k rows, G = 256) and bio size (N ~ 128 k, G = 256): ops.infomax_bce forward and
    forward + backward against the script's own torch composition (global_mean_pool as scatter_mean, sigmoid, summary @ W, the two
    index_select expansions, x * h sums, fp32 BCEWithLogits, autograd) on the same GPU, with the bytes each pass of the head must
    move (computed from the shapes) and the bandwidth that implies.
Device times are CUDA events after warm-up, alternating the contenders over three rounds; the card's name and power limit are read
in the same run.  Prints one JSON line per measurement.

    python tools/bench_infomax.py [--types gin,gcn,graphsage,gat] [--bio-types gin] [--batch 256] [--steps 20] [--warmup 5]

Needs a GPU."""
import argparse
import importlib
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

ap = argparse.ArgumentParser()
ap.add_argument("--types", default="gin,gcn,graphsage,gat")
ap.add_argument("--bio-types", default="gin")
ap.add_argument("--batch", type=int, default=256)
ap.add_argument("--steps", type=int, default=20)
ap.add_argument("--warmup", type=int, default=5)
ap.add_argument("--batches", type=int, default=2, help="distinct device-resident batches cycled through")
a = ap.parse_args()
if not torch.cuda.is_available():
    sys.exit("bench_infomax.py needs a GPU")
ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
ts = importlib.import_module("pretrain-gnns_b200.train_steps")
syn = importlib.import_module("pretrain-gnns_b200.synthetic")
ops = importlib.import_module("pretrain-gnns_b200.ops")

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


def to_dev(b):
    return {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in b.items()}


def run_step(step, host_batches, name):
    batches = [to_dev(b) for b in host_batches]
    i = [0]

    def one():
        step(batches[i[0] % len(batches)])
        i[0] += 1

    ms = timed(one, a.steps, a.warmup)
    loss = float(step(batches[0]))
    emit(dict(step=name, B=a.batch, ms_per_step=round(ms, 3), graphs_per_s=round(a.batch / ms * 1e3, 1), loss=loss, steps=a.steps,
              nodes=int(batches[0]["x"].shape[0])))


info = card()
emit(dict(what="card"))
chem_host = bio_host = None
for t in a.types.split(","):
    step = ts.InfomaxStep(dev, t, batch_size=a.batch)
    chem_host = chem_host or step.make_batches(0, a.batches)
    run_step(step, chem_host, "infomax_chem_" + t)
    del step
for t in a.bio_types.split(","):
    step = ts.BioInfomaxStep(dev, t, batch_size=a.batch)
    bio_host = bio_host or step.make_batches(0, a.batches)
    run_step(step, bio_host, "infomax_bio_" + t)
    del step


# the head alone
def cycle_index(num, shift):   # chem/pretrain_deepgraphinfomax.py:25-28
    arr = torch.arange(num) + shift
    arr[-shift:] = torch.arange(shift)
    return arr


def head(domain, batch, G):
    N, D = int(batch.shape[0]), 300
    g = torch.Generator(device=dev).manual_seed(0)
    x = (torch.randn(N, D, device=dev, generator=g) * 0.3).requires_grad_(True)
    W = ((torch.rand(D, D, device=dev, generator=g) * 2 - 1) / D ** 0.5).requires_grad_(True)
    shift = cycle_index(G, 1).to(dev)

    def torch_loss():
        tot = torch.zeros(G, D, device=dev).index_add_(0, batch, x)
        cnt = torch.zeros(G, device=dev).index_add_(0, batch, torch.ones(N, device=dev)).clamp(min=1)
        summary_emb = torch.sigmoid(tot / cnt[:, None])
        pos = torch.sum(x * torch.matmul(summary_emb[batch], W), dim=1)
        neg = torch.sum(x * torch.matmul(summary_emb[shift][batch], W), dim=1)
        return F.binary_cross_entropy_with_logits(pos, torch.ones_like(pos)) + F.binary_cross_entropy_with_logits(neg, torch.zeros_like(neg))

    def lib_fwd():
        with torch.no_grad():
            ops.infomax_bce(x, batch, W, G)

    def lib_fwd_bwd():
        x.grad = W.grad = None
        ops.infomax_bce(x, batch, W, G)[0].backward()

    def torch_fwd():
        with torch.no_grad():
            torch_loss()

    def torch_fwd_bwd():
        x.grad = W.grad = None
        torch_loss().backward()

    res = {}
    for _ in range(3):   # alternate, three rounds
        for name, fn in (("infomax_bce_fwd", lib_fwd), ("torch_fwd", torch_fwd), ("infomax_bce_fwd_bwd", lib_fwd_bwd),
                         ("torch_fwd_bwd", torch_fwd_bwd)):
            res.setdefault(name, []).append(round(timed(fn, 20, 3) * 1e3, 1))
    # bytes the head must move, from the shapes: the forward reads x twice (the segment mean, then the scores) and the batch ids,
    # and writes pos, neg and the two d loss / d score columns; the backward reads x (the per-graph reduction), the ids and the
    # d loss / d score columns twice and writes d x.  The G x D tables (S, H, dH, dS, W) stay in L2 and are left out.
    row = 4 * D
    fwd = 2 * N * row + 2 * N * 8 + 4 * N * 4 + N * 4
    bwd = N * row + 2 * N * 8 + 4 * N * 4 + N * row
    best = {k: min(v) for k, v in res.items()}
    emit(dict(what="infomax_bce", domain=domain, N=N, G=G, us_per_call=res, hbm_bytes_fwd=fwd, hbm_bytes_fwd_bwd=fwd + bwd,
              implied_gb_per_s_fwd=round(fwd / best["infomax_bce_fwd"] / 1e3, 1),
              implied_gb_per_s_fwd_bwd=round((fwd + bwd) / best["infomax_bce_fwd_bwd"] / 1e3, 1),
              speedup_fwd=round(best["torch_fwd"] / best["infomax_bce_fwd"], 2),
              speedup_fwd_bwd=round(best["torch_fwd_bwd"] / best["infomax_bce_fwd_bwd"], 2),
              loss=float(ops.infomax_bce(x, batch, W, G)[0]), loss_torch=float(torch_loss())))


head("chem", (chem_host[0] if chem_host else syn.zinc_batch(a.batch, 10000))["batch"].to(dev), a.batch)
head("bio", (bio_host[0] if bio_host else syn.ppi_batch(a.batch, 11000))["batch"].to(dev), a.batch)
