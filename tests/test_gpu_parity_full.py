"""GPU: CUDA path vs the CPU oracle AT BASELINE SIZES (configs[1..4]) and on one-direction-only graphs.

Each test runs one train() body of pretrain-gnns_b200/train_steps.py on cuda:0 and the oracle's restatement of the same
body (oracle/steps_oracle.py) on the host in fp32 and fp64, on the same seeded batch and parameters, and compares the
loss, the forward outputs and EVERY parameter gradient with the bounds of tests/golden_util.py (stated there against
the measured errors).  The measured errors of every tensor are written to gpurun_out/parity/*.json."""
import importlib

import pytest
import torch

from oracle import gnn_oracle as O
from oracle import steps_oracle as S
from golden_util import gradient_check, output_check, write_report

pytestmark = pytest.mark.gpu
syn = importlib.import_module("pretrain-gnns_b200.synthetic")
ts = importlib.import_module("pretrain-gnns_b200.train_steps")
DEV = "cuda:0"


def _dev(b):
    return {k: (v.to(DEV) if torch.is_tensor(v) else v) for k, v in b.items()}


def _compare(name, step, config, b, P, aux_fn, loss_fn=None):
    """aux_fn(step, device batch) -> dict of forward tensors named as the oracle's aux dict."""
    loss_fn = loss_fn or S.LOSSES[config]
    torch.set_num_threads(min(16, torch.get_num_threads()))
    l32, a32, g32, l64, a64, g64, near = S.grads_fp32_fp64(loss_fn, P, b)
    trace64 = S.LAST_RELU_TRACE
    step.load_state(P)
    d = _dev(b)
    plan = getattr(getattr(step, "model", None), "_fused_plan", lambda: None)()
    track = plan is not None and plan.gnn_type == "gin" and config == "masking"
    if track:
        plan.keep_workspace = True
    loss = step(d)
    flips = None
    if track:
        # ReLU decisions the fused GIN encoder actually took vs the fp64 oracle's: the allowance below needs a REAL flip
        ops = importlib.import_module("pretrain-gnns_b200.ops")
        mine = ops.chem_gin_relu_masks(plan, step.model)
        assert len(mine) == len(trace64)
        flips = int(sum(int((m.cpu() != (t > 0)).sum()) for m, t in zip(mine, trace64)))
        plan.keep_workspace, plan.last_ws = False, None
        near = min(near, flips)   # no flip, no allowance
    grads = [(k, p.grad) for k, p in step.named_parameters()]
    assert all(g is not None for _, g in grads)
    with torch.no_grad():
        aux = aux_fn(step, d)
    rows = []
    ok = True
    for k, v in aux.items():
        ok &= output_check(k, v, a32[k], a64[k], rows)
    lerr = abs(float(loss) - float(l64)) / max(abs(float(l64)), 1e-30)
    lref = abs(float(l32) - float(l64)) / max(abs(float(l64)), 1e-30)
    rows.append(dict(kind="loss", name="loss", err=lerr, err_ref32=lref, ok=lerr <= max(2e-6, 3 * lref)))
    ok &= rows[-1]["ok"]
    ok &= gradient_check(grads, g32, g64, near, rows)
    write_report(name, rows, dict(near_zero_preactivations=near, relu_flips_detected=flips, loss=float(loss), loss_oracle64=float(l64)))
    bad = [r for r in rows if not r["ok"]]
    assert ok, bad[:8]


def _masking_aux(step, d):
    rep = step.model(d["x"], d["edge_index"], d["edge_attr"])
    ops = importlib.import_module("pretrain-gnns_b200.ops")
    _, logits = ops.masked_atom_loss(rep, d["masked_atom_indices"], d["labels"], step.head.weight, step.head.bias)
    return dict(rep=rep, logits=logits)


def _frozen_bn(step):
    """aux forwards run a second train-mode pass: keep them from touching the module state the comparison already used."""
    return step


@pytest.mark.parametrize("config", ["masking", "gcn", "graphsage", "gat"])
def test_masking_step_b256_vs_oracle(config):
    """BASELINE configs[1] (GIN) and configs[4] (GCN / GraphSAGE / GAT): B = 256, the script's own masking head."""
    step = ts.CONFIGS[config](DEV)
    b = step.make_batches(0, 1)[0]
    _compare("masking_b256_" + config, step, config, b, S.make_params(config, 11), _masking_aux)


def test_contextpred_step_b128_vs_oracle():
    """BASELINE configs[2]: B = 128 substructure/context pairs, 5-layer + 3-layer encoders, cbow/mean, one negative."""
    step = ts.ContextPredStep(DEV)
    b = step.make_batches(0, 1)[0]

    def aux(step, d):
        pos, neg = step.scores(d)
        return dict(pos=pos, neg=neg)

    _compare("contextpred_b128", step, "contextpred", b, S.make_params("contextpred", 12), aux)


def test_bio_supervised_step_b64_t5000_vs_oracle():
    """BASELINE configs[3] per GPU: 64 PPI-ego-shaped graphs (~32k nodes, ~320k edges), GNN_graphpred with T = 5000."""
    import types
    step = ts.BioSupervisedStep(DEV)
    b = step.make_batches(0, 1)[0]

    def aux(step, d):
        return dict(pred=step.model(types.SimpleNamespace(**d)))

    _compare("bio_supervised_b64", step, "bio_supervised", b, S.make_params("bio_supervised", 13), aux)


@pytest.mark.parametrize("config", ["masking", "gcn", "graphsage", "gat"])
@pytest.mark.parametrize("fused", [True, False])
def test_one_direction_graphs_chem(config, fused):
    """Every bond keeps only ONE of its two directed edges: a swapped target/source anywhere in the forward, the
    transpose-graph backward, the edge summaries or the degree normalisation changes the result (SURVEY.md 8(c))."""
    step = ts.MaskingStep(DEV, "gin" if config == "masking" else config, batch_size=48)
    step.model.fused = fused
    mb = syn.mask_atoms(syn.one_direction_only(syn.zinc_batch(48, 71), 71), 71)
    b = {k: mb[k] for k in ("x", "edge_index", "edge_attr", "masked_atom_indices")} | {"labels": mb["mask_node_label"][:, 0].contiguous()}
    _compare("one_direction_%s_%s" % (config, "fused" if fused else "layerwise"), step, config, b, S.make_params(config, 14), _masking_aux)


@pytest.mark.parametrize("t", ["gin", "gcn", "graphsage", "gat"])
def test_one_direction_graphs_bio(t):
    import types
    step = ts.BioSupervisedStep(DEV, gnn_type=t, batch_size=3, num_tasks=40)
    pb = syn.one_direction_only(syn.ppi_batch(3, 72, n_lo=60, n_hi=90, num_tasks=40), 72)
    b = {k: pb[k] for k in ts.BioSupervisedStep.KEYS}
    P = {"model.gnn." + k: v for k, v in O.make_params("bio", t, 5, 300, seed=15).items()}
    g = torch.Generator().manual_seed(3)
    P["model.graph_pred_linear.weight"] = torch.randn(40, 600, generator=g) * 0.03
    P["model.graph_pred_linear.bias"] = torch.randn(40, generator=g) * 0.03

    def aux(step, d):
        return dict(pred=step.model(types.SimpleNamespace(**d)))

    _compare("one_direction_bio_" + t, step, "bio_supervised", b, P, aux, loss_fn=lambda L, bb: S.bio_supervised_loss(L, bb, t))


def test_loss_heads_vs_torch_fp64():
    """ops.bce_with_logits / bce_with_logits_const / masked_bce_with_logits / masked_bond_loss against torch's fp64 losses."""
    ops = importlib.import_module("pretrain-gnns_b200.ops")
    F = torch.nn.functional
    g = torch.Generator().manual_seed(9)
    x = (torch.randn(64, 5000, generator=g) * 3).to(DEV).requires_grad_(True)
    y = (torch.rand(64, 5000, generator=g) < 0.05).to(torch.int64).to(DEV)
    loss = ops.bce_with_logits(x, y)
    loss.backward()
    xr = x.detach().double().requires_grad_(True)
    ref = F.binary_cross_entropy_with_logits(xr, y.double())
    ref.backward()
    assert loss.dtype == torch.float64 and abs(float(loss) - float(ref)) <= 1e-13 * abs(float(ref)) + 1e-15
    assert torch.allclose(x.grad.double(), xr.grad, rtol=1e-6, atol=1e-12)
    l2 = ops.bce_with_logits(x.detach(), y)
    assert float(l2) == float(loss)  # deterministic reduction
    s = (torch.randn(128, generator=g) * 2).to(DEV).requires_grad_(True)
    for tv in (1.0, 0.0):
        s.grad = None
        l = ops.bce_with_logits_const(s, tv)
        l.backward()
        sr = s.detach().double().requires_grad_(True)
        r = F.binary_cross_entropy_with_logits(sr, torch.full_like(sr, tv))
        r.backward()
        assert abs(float(l) - float(r)) <= 1e-13 and torch.allclose(s.grad.double(), sr.grad, rtol=1e-6, atol=1e-12)
    # chem/finetune.py:33-43
    z = (torch.randn(32, 12, generator=g)).to(DEV).requires_grad_(True)
    yy = torch.randint(-1, 2, (32, 12), generator=g).to(DEV)
    l = ops.masked_bce_with_logits(z, yy)
    l.backward()
    zr = z.detach().double().requires_grad_(True)
    valid = yy ** 2 > 0
    lm = F.binary_cross_entropy_with_logits(zr, (yy.double() + 1) / 2, reduction="none")
    r = torch.where(valid, lm, torch.zeros_like(lm)).sum() / valid.sum()
    r.backward()
    assert abs(float(l) - float(r)) <= 1e-13 and torch.allclose(z.grad.double(), zr.grad, rtol=1e-6, atol=1e-12)
    # bond head, chem/pretrain_masking.py:57-61
    mb = syn.mask_atoms(syn.zinc_batch(32, 5), 5, mask_edge=True)
    rep = torch.randn(mb["x"].shape[0], 300, generator=g)
    W, bias = torch.randn(4, 300, generator=g) * 0.05, torch.randn(4, generator=g) * 0.05
    rr = [t.clone().requires_grad_(True) for t in (rep, W, bias)]
    lref, logits_ref = O.masking_edge_loss(rr[0], mb["edge_index"], mb["connected_edge_indices"], mb["mask_edge_label"][:, 0], rr[1], rr[2])
    lref.backward()
    dd = [t.clone().to(DEV).requires_grad_(True) for t in (rep, W, bias)]
    l, logits = ops.masked_bond_loss(dd[0], mb["edge_index"].to(DEV), mb["connected_edge_indices"].to(DEV), mb["mask_edge_label"][:, 0].to(DEV), dd[1], dd[2])
    l.backward()
    assert abs(float(l) - float(lref)) < 1e-6 and torch.allclose(logits.cpu(), logits_ref.detach(), atol=1e-4, rtol=1e-4)
    for mine, ref in zip(dd, rr):
        assert float((mine.grad.cpu() - ref.grad).abs().max()) <= 2e-5 * float(ref.grad.abs().max())


@pytest.mark.parametrize("config", ["masking", "gcn", "gat"])
def test_training_step_run_to_run_reproducibility(config):
    """Two training steps on the same batch and parameters.  The loss (ordered fp64 fold) must repeat to 1e-9; every gradient must
    repeat to 3e-4 of its scale (the tensor's own largest magnitude; the model's largest gradient for the structurally zero biases).
    What is ordered by construction --
    weight and embedding-table gradients from split-K partial tiles folded in split order -- is expected BIT-identical, the
    bias / BatchNorm / bond-table gradients and the GAT scalar folds go through fp32 / fp64 atomics whose order varies: the number
    of bit-identical tensors and the worst difference are MEASURED and reported (write_report), not asserted -- training is reproducible to rounding, not bitwise (DESIGN.md section 4)."""
    step = ts.CONFIGS[config](DEV)
    b = step.make_batches(0, 1)[0]
    P = S.make_params(config, 17)
    d = _dev(b)
    runs = []
    for _ in range(2):
        step.load_state(P)
        step.zero_grad()
        loss = step(d)
        torch.cuda.synchronize()
        runs.append((float(loss), {k: p.grad.detach().clone() for k, p in step.named_parameters()}))
    (l0, g0), (l1, g1) = runs
    rows, bitwise, worst = [], 0, 0.0
    gmax = max(float(v.abs().max()) for v in g0.values())
    for k in g0:
        tmax = float(g0[k].abs().max())
        # run-to-run noise comes from the ORDER of fp32 / fp64 atomic additions, so it scales with the summands, not with the sum: the
        # biases in front of train-mode BatchNorm (mlp.2.bias, GAT's bias) have an exactly zero gradient in exact arithmetic -- what is
        # computed is cancellation noise below 1e-3 of the model's largest gradient -- and are judged on the model's scale
        scale = max(gmax if tmax < 1e-3 * gmax else tmax, 1e-30)
        diff = float((g0[k] - g1[k]).abs().max()) / scale
        same = bool(torch.equal(g0[k], g1[k]))
        bitwise += same
        worst = max(worst, diff)
        rows.append(dict(kind="grad", name=k, err=diff, err_ref32=0.0, ok=diff <= 3e-4, bitwise=same))
    write_report("reproducibility_" + config, rows, dict(loss_run0=l0, loss_run1=l1, tensors=len(g0), bitwise_identical=bitwise, worst=worst))
    assert abs(l0 - l1) <= 1e-9 * max(abs(l0), 1.0), (l0, l1)
    bad = [(r["name"], r["err"]) for r in rows if not r["ok"]]
    assert not bad, bad[:6]
