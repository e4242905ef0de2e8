"""Golden vectors from the reference's own model.py loaded with the reference's SHIPPED checkpoints (SURVEY.md section 8(d)
config 1: B = 32, eval-mode forward, weights = chem/model_gin/masking.pth; plus the GCN checkpoint whose activations reach
|x| ~ 190, the GAT / GraphSAGE checkpoints and the bio GIN one).

Run in the build container only (needs /root/reference):

    python tests/golden/make_golden_pretrained.py

Stored per case: the reference's eval-mode node representations `[N, 300]` fp32 and fp64 (a train-mode forward would overwrite nothing
here, but the checkpoints' BatchNorm running statistics are what eval mode exercises), an input checksum, and a SHA-256 of the
checkpoint file so the test can tell a wrong staged file from a wrong kernel.  The weights themselves are never committed:
`oracle/reference_runner.stage()` copies the checkpoint files next to the staged model.py (git-ignored `oracle/_ref/weights/`),
which is where the GPU box reads them.
"""
import hashlib
import importlib
import os
import sys

import numpy as np
import torch

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), "..", ".."))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from golden_util import PRETRAINED, input_checksum, pretrained_batch, pretrained_rows  # noqa: E402
from oracle import reference_runner  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
REF = "/root/reference"


def main():
    torch.manual_seed(0)
    torch.set_num_threads(1)
    out = {}
    for name, c in PRETRAINED.items():
        assert reference_runner.root() == REF, "goldens are generated from /root/reference itself, not from a staged copy"
        ref = reference_runner.load(c["domain"])
        path = os.path.join(REF, c["file"])
        model = ref.GNN(5, 300, JK="last", drop_ratio=0, gnn_type=c["type"])
        sd = torch.load(path, map_location="cpu", weights_only=True)
        assert str(model.load_state_dict(sd)) == "<All keys matched successfully>"
        model.eval()
        b = pretrained_batch(name)
        with torch.no_grad():
            y = model(b["x"], b["edge_index"], b["edge_attr"])
        rows = pretrained_rows(y.shape[0])
        # the same forward in float64: the yardstick for how well conditioned the checkpoint is (the trained GIN's pre-BatchNorm
        # activations reach 1e5, and eval-mode BatchNorm turns a uniform absolute error of the Linear output into per-column errors)
        m64 = ref.GNN(5, 300, JK="last", drop_ratio=0, gnn_type=c["type"])
        m64.load_state_dict(sd)
        m64.double().eval()
        with torch.no_grad():
            y64 = m64(b["x"].double() if b["x"].is_floating_point() else b["x"], b["edge_index"],
                      b["edge_attr"].double() if b["edge_attr"].is_floating_point() else b["edge_attr"])
        # a seeded sample of the rows is stored; the full tensor's scale goes with it so that errors keep their meaning
        out[name + ":rows"] = rows.numpy()
        out[name + ":n"] = np.int64(y.shape[0])
        out[name + ":scale"] = np.float64(y64.abs().max())
        out[name + ":out_eval"] = y[rows].numpy()
        out[name + ":d64"] = (y64 - y.double())[rows].float().numpy()     # ref64 = out_eval + d64 (the difference is tiny: stored in fp32)
        out[name + ":input_checksum"] = input_checksum(b)
        out[name + ":sha256"] = np.frombuffer(hashlib.sha256(open(path, "rb").read()).digest(), dtype=np.uint8)
        print("%-14s N = %5d  max|out| = %8.3f  %s" % (name, y.shape[0], float(y.abs().max()), c["file"]))
    p = os.path.join(HERE, "pretrained.npz")
    np.savez_compressed(p, **out)
    print(p, os.path.getsize(p) // 1024, "KiB")


if __name__ == "__main__":
    main()
