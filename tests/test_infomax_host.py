"""CPU: Deep Graph Infomax pre-training.  The train() body on the oracle port against the same body on the reference's own chem / bio
model.py inside the script's restated Infomax (four gnn_types, G = 1 included); train_steps.Discriminator's draw against the
script's under the same seed; InfomaxStep.load_state with Infomax.state_dict()'s keys; the C argument checks and the ptxas report
of csrc/infomax.cu (no device touched)."""
import ctypes
import importlib
import os
import re
import shutil
import subprocess

import pytest
import torch

import infomax_oracle as IO
from oracle import reference_runner as R
from test_bio_objectives_host import _compare_with_reference

syn = importlib.import_module("pretrain-gnns_b200.synthetic")
ts = importlib.import_module("pretrain-gnns_b200.train_steps")
cabi = importlib.import_module("pretrain-gnns_b200._cabi")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
needs_reference = pytest.mark.skipif(not R.available(), reason="the reference sources are not staged under oracle/_ref")


def test_cycle_index_is_a_shift_by_one():
    for G in (1, 2, 5, 256):
        assert torch.equal(IO.cycle_index(G, 1), (torch.arange(G) + 1) % G), G


@needs_reference
@pytest.mark.parametrize("G", [1, 3])
@pytest.mark.parametrize("domain", ["chem", "bio"])
@pytest.mark.parametrize("t", ["gin", "gcn", "graphsage", "gat"])
def test_infomax_port_equals_reference(domain, t, G):
    """chem/pretrain_deepgraphinfomax.py:61-74 (and bio's) on the reference's own GNN with the stand-in's global_mean_pool and
    nn.BCEWithLogitsLoss on fp32 scores, against the port's body with the BCE on fp64 scores.  G = 1 pairs a graph with itself."""
    torch.set_num_threads(1)
    if domain == "chem":
        b = syn.zinc_batch(G, 5 + G)
        ref = IO.ReferenceInfomaxStep(t)
    else:
        b = syn.ppi_batch(G, 5 + G, n_lo=30, n_hi=50, num_tasks=4)
        ref = IO.ReferenceBioInfomaxStep(t)
    b = {k: b[k] for k in ts.InfomaxStep.KEYS}
    _compare_with_reference(ref, lambda L, bb: IO.infomax_loss(L, bb, domain, t), IO.make_params(domain, 3, t), b)


def test_discriminator_draw_equals_the_script():
    """train_steps.Discriminator draws U(-1/sqrt(D), 1/sqrt(D)) exactly as the script's Discriminator under the same seed."""
    for seed, D in ((0, 300), (7, 300), (3, 16)):
        torch.manual_seed(seed)
        mine = ts.Discriminator(D).weight.detach().clone()
        torch.manual_seed(seed)
        ref = IO.Discriminator(D).weight.detach().clone()
        assert mine.shape == (D, D) and torch.equal(mine, ref), (seed, D)
        assert float(mine.abs().max()) <= 1.0 / D ** 0.5
    x, s = torch.randn(5, 16), torch.rand(5, 16)
    d = ts.Discriminator(16)
    r = IO.Discriminator(16)
    r.weight.data.copy_(d.weight.data)
    assert torch.equal(d(x, s), r(x, s))


@needs_reference
@pytest.mark.parametrize("step_cls,domain", [(ts.InfomaxStep, "chem"), (ts.BioInfomaxStep, "bio")])
def test_load_state_takes_infomax_state_dict(step_cls, domain):
    """The script's model is Infomax(gnn, discriminator): its state_dict ('gnn.*', 'discriminator.weight') loads as it is."""
    ref = (IO.ReferenceInfomaxStep if domain == "chem" else IO.ReferenceBioInfomaxStep)("gin")
    torch.manual_seed(1)
    ref.model.discriminator.reset_parameters()
    sd = ref.model.state_dict()
    assert "discriminator.weight" in sd and any(k.startswith("gnn.gnns.0.") for k in sd)
    step = step_cls("cpu", "gin", batch_size=4)
    step.load_state(sd)
    mine = {k: p for k, p in step.named_parameters()}
    trainable = {k for k, _ in ref.model.named_parameters()}
    assert set(mine) == trainable
    for k in trainable:
        assert torch.equal(mine[k].detach(), sd[k]), k
    buffers = {name + "." + k: v for name, m in step.named_modules().items() for k, v in m.state_dict().items()}
    assert set(buffers) == set(sd) and all(torch.equal(buffers[k], sd[k]) for k in sd)


def test_infomax_batches_carry_the_graph_count():
    for step_cls in (ts.InfomaxStep, ts.BioInfomaxStep):
        step = step_cls("cpu", "gin", batch_size=3)
        b = step.make_batches(0, 1)[0]
        assert set(step_cls.KEYS) <= set(b) and b["num_graphs"] == 3 == int(b["batch"].max()) + 1
    assert (ts.INFOMAX_SEED, ts.BIO_INFOMAX_SEED) == (10, 11)


def _buf(n=64):
    return (ctypes.addressof(ctypes.create_string_buffer(n + 16)) + 15) // 16 * 16


def test_infomax_argument_validation_without_gpu():
    dll = cabi.lib.load()
    wsb = dll.pgnn_infomax_bce_workspace_bytes()
    assert wsb >= 2 * 8 * 132
    w, one = _buf(wsb), _buf()
    s = dll.pgnn_infomax_summary_fwd
    # (x, ldx, seg_ptr, seg_order, G, C, S, lds, stream)
    assert s(one, 300, one, one, -1, 300, one, 300, None) == -1     # G < 0
    assert s(one, 300, one, one, 4, 0, one, 300, None) == -1        # C == 0
    assert s(one, 296, one, one, 4, 300, one, 300, None) == -1      # ldx < C
    assert s(one, 300, None, one, 4, 300, one, 300, None) == -1     # no seg_ptr
    assert s(one, 300, one, one, 4, 300, None, 300, None) == -1     # no output
    assert s(one, 302, one, one, 4, 302, one, 302, None) == -4      # C % 4
    assert s(one + 4, 300, one, one, 4, 300, one, 300, None) == -4  # misaligned x
    assert s(None, 300, None, None, 0, 300, None, 300, None) == 0   # G == 0: nothing
    f = dll.pgnn_infomax_bce_fwd
    # (x, ldx, N, C, batch, H, G, loss, pos, neg, dscore, ws, wsb, stream)
    assert f(one, 300, -1, 300, one, one, 4, one, one, one, one, w, wsb, None) == -1      # N < 0
    assert f(one, 300, 8, 0, one, one, 4, one, one, one, one, w, wsb, None) == -1        # C == 0
    assert f(one, 296, 8, 300, one, one, 4, one, one, one, one, w, wsb, None) == -1      # ldx < C
    assert f(one, 300, 8, 300, one, one, 0, one, one, one, one, w, wsb, None) == -1      # N > 0 without a graph
    assert f(one, 300, 8, 300, None, one, 4, one, one, one, one, w, wsb, None) == -1     # no batch
    assert f(one, 300, 8, 300, one, None, 4, one, one, one, one, w, wsb, None) == -1     # no H
    assert f(one, 300, 8, 300, one, one, 4, None, one, one, one, w, wsb, None) == -1     # no loss
    assert f(one, 300, 8, 300, one, one, 4, one, one, one, None, w, wsb, None) == -1     # no dscore
    assert f(one, 300, 8, 300, one, one, 4, one, one, one, one, None, wsb, None) == -1   # no workspace
    assert f(one, 300, 8, 300, one, one, 4, one, one, one, one, w, wsb - 1, None) == -3  # workspace too small
    assert f(one, 302, 8, 302, one, one, 4, one, one, one, one, w, wsb, None) == -4      # C % 4
    assert f(one, 302, 8, 300, one, one, 4, one, one, one, one, w, wsb, None) == -4      # ldx % 4
    assert f(one + 4, 300, 8, 300, one, one, 4, one, one, one, one, w, wsb, None) == -4  # misaligned x
    assert dll.pgnn_infomax_bce_bwd_workspace_bytes(-1, 300) == -1 and dll.pgnn_infomax_bce_bwd_workspace_bytes(4, 0) == -1
    bwsb = dll.pgnn_infomax_bce_bwd_workspace_bytes(4, 300)
    assert bwsb >= 2 * 4 * 300 * 4
    bw = _buf(bwsb)
    b = dll.pgnn_infomax_bce_bwd
    # (x, ldx, N, C, batch, seg_ptr, seg_order, G, S, H, W, dscore, gscale, gx, ldgx, gW, precision, ws, wsb, stream)
    assert b(one, 300, -1, 300, one, one, one, 4, one, one, one, one, one, one, 300, one, 1, bw, bwsb, None) == -1   # N < 0
    assert b(one, 300, 8, 300, one, one, one, 0, one, one, one, one, one, one, 300, one, 1, bw, bwsb, None) == -1    # N > 0, G = 0
    assert b(one, 300, 8, 300, one, one, one, 4, one, one, one, one, None, one, 300, one, 1, bw, bwsb, None) == -1   # no gscale
    assert b(one, 300, 8, 300, one, None, one, 4, one, one, one, one, one, one, 300, one, 1, bw, bwsb, None) == -1   # no seg_ptr
    assert b(one, 300, 8, 300, one, one, one, 4, one, one, None, one, one, one, 300, one, 1, bw, bwsb, None) == -1   # no W
    assert b(one, 300, 8, 300, one, one, one, 4, one, one, one, None, one, one, 300, one, 1, bw, bwsb, None) == -1   # no dscore
    assert b(one, 300, 8, 300, one, one, one, 4, one, one, one, one, one, one, 296, one, 1, bw, bwsb, None) == -1   # ldgx < C
    assert b(one, 300, 8, 300, one, one, one, 4, one, one, one, one, one, one, 300, one, 1, bw, bwsb - 1, None) == -3  # too small
    big = dll.pgnn_infomax_bce_bwd_workspace_bytes(4, 302)
    assert b(one, 302, 8, 302, one, one, one, 4, one, one, one, one, one, one, 302, one, 1, _buf(big), big, None) == -4   # C % 4
    assert b(one + 4, 300, 8, 300, one, one, one, 4, one, one, one, one, one, one, 300, one, 1, bw, bwsb, None) == -4  # misaligned x


def _ptxas(src_name, tmp_path):
    nvcc = NVCC if os.path.exists(NVCC) else shutil.which("nvcc")
    src = os.path.join(ROOT, "pretrain-gnns_b200", "csrc", src_name)
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--expt-relaxed-constexpr",
           "-I" + os.path.join(ROOT, "include"), "-Xptxas", "-v", "-c", src, "-o", str(tmp_path / (src_name + ".o"))]
    out = subprocess.run(cmd, capture_output=True, text=True)
    assert out.returncode == 0, out.stderr[-4000:]
    kernels, cur = {}, None
    for line in (out.stdout + out.stderr).splitlines():
        m = re.search(r"Compiling entry function '(\w+)'", line)
        if m:
            cur = m.group(1)
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if cur and m:
            kernels[cur] = (int(m.group(1)), int(m.group(2)))
    return kernels


@pytest.mark.skipif(not (os.path.exists(NVCC) or shutil.which("nvcc")), reason="nvcc not available")
def test_infomax_kernels_ptxas_no_spills(tmp_path):
    """The four kernels of csrc/infomax.cu (summary, scores + BCE, per-graph reduction, node pass) compile for sm_90a without
    spills."""
    k = _ptxas("infomax.cu", tmp_path)
    assert len(k) == 4 and all(v == (0, 0) for v in k.values()), k
