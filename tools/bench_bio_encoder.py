"""Graphs/s of the bio training steps with the whole-encoder path (bio.GNN.fused = True, pgnn_bio_encoder_*) against the
layer-by-layer composition (fused = False), timed alternately on the same card in one run: bio supervised pre-training at
bench.py's per-GPU batch (train_steps.BioSupervisedStep, B = 64), bio masking for every gnn_type and bio context prediction at the
scripts' batch size (B = 256).  Device-resident batches, the optimizer step excluded, CUDA events after warm-up; the card's name
and power limit are read in the same run.  Prints one JSON line per workload.

    python tools/bench_bio_encoder.py [--types gin,gcn,graphsage,gat] [--steps 20] [--warmup 5] [--rounds 3] [--batches 3]

Needs a GPU."""
import argparse
import importlib
import json
import os
import subprocess
import sys

import torch

ap = argparse.ArgumentParser()
ap.add_argument("--types", default="gin,gcn,graphsage,gat")
ap.add_argument("--steps", type=int, default=20)
ap.add_argument("--warmup", type=int, default=5)
ap.add_argument("--rounds", type=int, default=3, help="alternations of the two paths")
ap.add_argument("--batches", type=int, default=3, help="distinct device-resident batches cycled through")
a = ap.parse_args()
if not torch.cuda.is_available():
    sys.exit("bench_bio_encoder.py needs a GPU")
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
ts = importlib.import_module("pretrain-gnns_b200.train_steps")
bio = importlib.import_module("pretrain-gnns_b200.bio.model")
dev = torch.device("cuda:0")


def card():
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "unknown"
    return dict(card=torch.cuda.get_device_name(0), power_limit=q)


def set_fused(step, flag):
    n = 0
    for mod in step.modules:
        for m in mod.modules():
            if isinstance(m, bio.GNN):
                m.fused = flag
                n += 1
    assert n > 0


def timed(fn):
    for _ in range(a.warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(a.steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / a.steps


def run(name, step, B, host):
    batches = [{k: v.to(dev) for k, v in b.items() if torch.is_tensor(v)} | {k: v for k, v in b.items() if not torch.is_tensor(v)}
               for b in host]
    i = [0]

    def one():
        step(batches[i[0] % len(batches)])
        i[0] += 1

    res = {"fused": [], "layerwise": []}
    for _ in range(a.rounds):
        for label, flag in (("fused", True), ("layerwise", False)):
            set_fused(step, flag)
            res[label].append(round(B / timed(one) * 1e3, 1))
    set_fused(step, True)
    best = {k: max(v) for k, v in res.items()}
    print(json.dumps(dict(step=name, B=B, graphs_per_s=res, best=best, speedup=round(best["fused"] / best["layerwise"], 3),
                          steps=a.steps, rounds=a.rounds) | info), flush=True)


info = card()
print(json.dumps(dict(what="card") | info), flush=True)
step = ts.CONFIGS["bio_supervised"](dev)
run("bio_supervised_gin", step, 64, step.make_batches(0, a.batches))
del step
mask_host = None
for t in a.types.split(","):
    step = ts.BioMaskingStep(dev, t, batch_size=256)
    if mask_host is None:
        mask_host = step.make_batches(0, a.batches)
    run("bio_masking_" + t, step, 256, mask_host)
    del step
step = ts.BioContextPredStep(dev, batch_size=256)
run("bio_contextpred_gin", step, 256, step.make_batches(0, a.batches))
