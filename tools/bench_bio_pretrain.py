"""Graphs/s of the bio pre-training steps on device-resident batches (the optimizer step excluded), at the scripts' batch size:
bio masking (bio/pretrain_masking.py:39-55, train_steps.BioMaskingStep) for every gnn_type and bio context prediction
(bio/pretrain_contextpred.py:43-97, train_steps.BioContextPredStep).  Also times the edge-type loss of one masking batch (~96 k
rows, V = 7): pgnn_softmax_ce_rows_fwd against torch.argmax over the label rows followed by pgnn_softmax_ce_fwd (k_softmax_ce).
Steps are timed with CUDA events after warm-up; the card's name and power limit are read in the same run.  Prints one JSON line
per measurement.

    python tools/bench_bio_pretrain.py [--types gin,gcn,graphsage,gat] [--batch 256] [--steps 30] [--warmup 5] [--batches 3]

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
ap.add_argument("--batch", type=int, default=256)
ap.add_argument("--steps", type=int, default=30)
ap.add_argument("--warmup", type=int, default=5)
ap.add_argument("--batches", type=int, default=3, help="distinct device-resident batches cycled through")
ap.add_argument("--ce-iters", type=int, default=200)
ap.add_argument("--no-contextpred", action="store_true")
a = ap.parse_args()
if not torch.cuda.is_available():
    sys.exit("bench_bio_pretrain.py needs a GPU")
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
ts = importlib.import_module("pretrain-gnns_b200.train_steps")
cabi = importlib.import_module("pretrain-gnns_b200._cabi")
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


def run_step(step, host_batches, name):
    batches = [{k: v.to(dev) for k, v in b.items() if torch.is_tensor(v)} for b in host_batches]
    i = [0]

    def one():
        step(batches[i[0] % len(batches)])
        i[0] += 1

    ms = timed(one, a.steps, a.warmup)
    loss = float(step(batches[0]))
    print(json.dumps(dict(step=name, B=a.batch, ms_per_step=round(ms, 3), graphs_per_s=round(a.batch / ms * 1e3, 1), loss=loss,
                          steps=a.steps, batches=len(batches)) | info), flush=True)


info = card()
print(json.dumps(dict(what="card") | info), flush=True)
mask_host = None
for t in a.types.split(","):
    step = ts.BioMaskingStep(dev, t, batch_size=a.batch)
    if mask_host is None:   # the batches do not depend on gnn_type: draw them once
        mask_host = step.make_batches(0, a.batches)
    run_step(step, mask_host, "bio_masking_" + t)
    del step

if not a.no_contextpred:
    step = ts.BioContextPredStep(dev, batch_size=a.batch)
    run_step(step, step.make_batches(0, a.batches), "bio_contextpred_gin")
    del step

# the edge-type loss alone, on the first masking batch's label rows
lab = mask_host[0]["mask_edge_label"].to(dev)
M, V, ldv = lab.shape[0], 7, 8
g = torch.Generator(device=dev).manual_seed(0)
logits = torch.randn(M, ldv, device=dev, generator=g)
dl = torch.empty(M, ldv, device=dev)
loss = torch.empty((), dtype=torch.float64, device=dev)
wsb = int(cabi.lib.pgnn_softmax_ce_rows_workspace_bytes())
ws = torch.empty(wsb, dtype=torch.uint8, device=dev)
st = torch.cuda.current_stream().cuda_stream


def ce_rows():
    cabi.check(cabi.lib.pgnn_softmax_ce_rows_fwd(logits.data_ptr(), ldv, M, V, lab.data_ptr(), lab.stride(0), lab.shape[1], loss.data_ptr(),
                                                 dl.data_ptr(), ldv, ws.data_ptr(), wsb, st), "softmax_ce_rows_fwd")


def argmax_then_ce():
    y = torch.argmax(lab, dim=1)
    cabi.check(cabi.lib.pgnn_softmax_ce_fwd(logits.data_ptr(), ldv, M, V, y.data_ptr(), loss.data_ptr(), dl.data_ptr(), ldv, st), "softmax_ce_fwd")


res = {}
for rep in range(3):   # alternate the two, three rounds
    for name, fn in (("softmax_ce_rows", ce_rows), ("argmax+softmax_ce", argmax_then_ce)):
        res.setdefault(name, []).append(round(timed(fn, a.ce_iters, 20) * 1e3, 2))
ce_rows()
l_new = float(loss)
argmax_then_ce()
l_old = float(loss)
print(json.dumps(dict(what="edge_type_loss", M=M, V=V, Q=int(lab.shape[1]), us_per_call=res, loss_rows=l_new, loss_argmax=l_old) | info),
      flush=True)
