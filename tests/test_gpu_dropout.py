"""GPU: live dropout.  The operator's kept / dropped pattern against the host restatement of the draw (tests/dropout_oracle.py), the
whole-encoder path against the layer-by-layer composition and the masked oracle, the fine-tuning step, the dropout-free identity
of the new entry points, and the seed behaviour of the modules."""
import ctypes
import importlib
import types

import numpy as np
import pytest
import torch

import dropout_oracle as DO
from device_buffers import DEV, SENT, Region, filled
from golden_util import grad_close, probe
from oracle import gnn_oracle as O

pytestmark = pytest.mark.gpu
syn = importlib.import_module("pretrain-gnns_b200.synthetic")
chem = importlib.import_module("pretrain-gnns_b200.chem.model")
bio = importlib.import_module("pretrain-gnns_b200.bio.model")
ops = importlib.import_module("pretrain-gnns_b200.ops")
ts = importlib.import_module("pretrain-gnns_b200.train_steps")
lib = importlib.import_module("pretrain-gnns_b200._cabi").lib
TYPES = ("gin", "gcn", "graphsage", "gat")


def _dev(b):
    return {k: (v.to(DEV) if torch.is_tensor(v) else v) for k, v in b.items()}


def _same_bits(a, b):
    """Equal as fp32 bit patterns after mapping every NaN to one pattern."""
    a, b = a.float().cpu().clone(), b.float().cpu().clone()
    na, nb = torch.isnan(a), torch.isnan(b)
    if not torch.equal(na, nb):
        return False
    a[na], b[nb] = 0, 0
    return torch.equal(a.view(torch.int32), b.view(torch.int32))


def _factor(seed, layer, rows, C, p):
    return torch.from_numpy(DO.keep_mask(seed, layer, rows, C, p).astype(np.float32)) * np.float32(DO.scale(p))


# ---------------------------------------------------------------------------------------------------------------------
# 1. the operator
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("p", [0.0, 0.2, 0.5, 0.9, 1.0])
@pytest.mark.parametrize("C", [4, 7, 300])
def test_dropout_op_bits_equal_host_restatement(p, C):
    M, seed, layer = 517, (1 << 61) + 12345, 3
    g = torch.Generator().manual_seed(C)
    x = torch.randn(M, C, generator=g)
    # non-finite values in both kept and dropped slots (a dropped NaN / Inf must come out NaN)
    keep = DO.keep_mask(seed, layer, M, C, p)
    for r in range(0, M, 37):
        x[r, r % C] = float("nan")
        x[r + 1 if r + 1 < M else r, (r + 3) % C] = float("inf")
        x[r + 2 if r + 2 < M else r, (r + 5) % C] = float("-inf")
    f = _factor(seed, layer, M, C, p)
    want = x * f
    if 0 < p < 1:
        assert keep.any() and (~keep).any()
        assert torch.isnan(want[torch.from_numpy(~keep) & torch.isinf(x)]).all()
    for ld_in, ld_out in ((C, C), (C + 5, C + 3)):
        xin = filled(x, ld=ld_in)                   # NaN-filled allocation around the rows
        out = Region(M, C, ld_out, SENT)           # sentinel-filled
        assert lib.pgnn_dropout_fwd(ctypes.c_void_p(xin.ptr()), ld_in, M, C, p, seed, layer, ctypes.c_void_p(out.ptr()), ld_out,
                                    ctypes.c_void_p(ops._st())) == 0
        gout = Region(M, C, ld_out, SENT)
        assert lib.pgnn_dropout_bwd(ctypes.c_void_p(xin.ptr()), ld_in, M, C, p, seed, layer, ctypes.c_void_p(gout.ptr()), ld_out,
                                    ctypes.c_void_p(ops._st())) == 0
        torch.cuda.synchronize()
        assert _same_bits(out.view, want) and out.outside_intact(), (ld_in, ld_out)
        assert _same_bits(gout.view, want) and gout.outside_intact(), (ld_in, ld_out)
    # the autograd op: forward pattern and backward = g * mask * scale exactly
    xd = torch.randn(M, C, generator=g).to(DEV).requires_grad_(True)
    y = ops.dropout(xd, p, seed, layer)
    gy = torch.randn(M, C, generator=g)
    y.backward(gy.to(DEV))
    assert _same_bits(y.detach(), xd.detach().cpu() * f)
    assert _same_bits(xd.grad, gy * f)


# ---------------------------------------------------------------------------------------------------------------------
# 2. / 3. the whole-encoder path with dropout
# ---------------------------------------------------------------------------------------------------------------------
def _chem_model(t, P, fused, drop):
    m = chem.GNN(5, 300, JK="last", drop_ratio=drop, gnn_type=t)
    m.fused = fused
    m.load_state_dict(P)
    return m.to(DEV).train()


@pytest.mark.parametrize("t", TYPES)
def test_fused_and_layerwise_agree_with_dropout(t):
    """drop_ratio 0.5, training, the same torch.manual_seed: the two paths draw the same seed and so drop the same units; the rest
    agrees within the bounds of test_fused_and_layerwise_paths_agree."""
    b = syn.one_direction_only(syn.zinc_batch(32, 100), 5)
    P = O.make_params("chem", t, 5, 300, seed=21)
    R = probe((b["x"].shape[0], 300), 5).to(DEV)
    d = _dev(b)
    res = []
    for fused in (True, False):
        model = _chem_model(t, P, fused, 0.5)
        assert (model._fused_plan() is not None) == fused
        torch.manual_seed(1234)
        out = model(d["x"], d["edge_index"], d["edge_attr"])
        (out * R).sum().backward()
        res.append((out.detach(), {k: p.grad for k, p in model.named_parameters()}, model.state_dict()))
    assert torch.equal(res[0][0] == 0, res[1][0] == 0)
    assert float((res[1][0] == 0).float().mean()) > 0.4  # the last layer has no ReLU: its zeros are the dropped units
    assert torch.allclose(res[0][0], res[1][0], atol=2e-5, rtol=1e-5)
    gmax = max(float(g.abs().max()) for g in res[1][1].values())
    for k, g in res[1][1].items():
        scale = max(float(g.abs().max()), 1e-3 * gmax)
        assert float((res[0][1][k] - g).abs().max()) <= 2e-4 * scale + 3e-6 * gmax, k
    for k in res[0][2]:
        assert torch.allclose(res[0][2][k].float(), res[1][2][k].float(), atol=1e-5, rtol=1e-5), k


def _oracle_grads(fn, P):
    res = []
    for dt in (torch.float32, torch.float64):
        L = O.leaf_params(P, dt)
        fn(L).backward()
        res.append({k: v.grad for k, v in L.items() if v.requires_grad})
    mags = sorted(float(v.abs().max()) for v in res[1].values())
    return res[0], res[1], max(mags[len(mags) // 2], 1e-3)


def _check_grads(named_params, g32, g64, floor, prefix=""):
    bad = []
    for k, p in named_params:
        ok, e, tol = grad_close(p.grad.cpu(), g32[prefix + k], g64[prefix + k], floor)
        if not ok:
            bad.append((k, e, tol))
    assert not bad, bad


def _seed_after(s):
    torch.manual_seed(s)
    return ops.draw_seed()


@pytest.mark.parametrize("t", TYPES)
def test_fused_encoder_with_dropout_vs_masked_oracle(t):
    b = syn.zinc_batch(32, 100)
    P = O.make_params("chem", t, 5, 300, seed=21)
    n, p = b["x"].shape[0], 0.5
    masks = DO.layer_masks(_seed_after(77), 5, n, 300, p, torch.float32)
    R = probe((n, 300), 5)
    ref = DO.chem_gnn(P, b["x"], b["edge_index"], b["edge_attr"], 5, t, True, masks=masks, p=p)
    g32, g64, floor = _oracle_grads(lambda L: (DO.chem_gnn(L, b["x"], b["edge_index"], b["edge_attr"], 5, t, True, masks=masks, p=p)
                                               * R.to(L["x_embedding1.weight"].dtype)).sum(), P)
    model = _chem_model(t, P, True, p)
    d = _dev(b)
    torch.manual_seed(77)
    out = model(d["x"], d["edge_index"], d["edge_attr"])
    (out * R.to(DEV)).sum().backward()
    err = (out.detach().cpu() - ref.detach()).abs()
    assert bool((err <= 1e-4 + 1e-4 * ref.detach().abs()).all()), err.max()
    _check_grads(model.named_parameters(), g32, g64, floor)


def test_bio_graphpred_with_dropout_vs_masked_oracle():
    b = syn.ppi_batch(3, 8, n_lo=60, n_hi=90, num_tasks=40)
    P = O.make_params("bio", "gin", 5, 300, seed=4)
    g = torch.Generator().manual_seed(2)
    full = {"gnn." + k: v for k, v in P.items()}
    full["graph_pred_linear.weight"] = torch.randn(40, 600, generator=g) * 0.03
    full["graph_pred_linear.bias"] = torch.randn(40, generator=g) * 0.03
    y = b["go_target_pretrain"].view(3, 40).double()
    p, n = 0.2, b["x"].shape[0]
    masks = DO.layer_masks(_seed_after(5), 5, n, 300, p, torch.float32)

    def logits(L):
        dt = L["graph_pred_linear.bias"].dtype
        return DO.bio_graphpred(L, b["x"].to(dt), b["edge_index"], b["edge_attr"].to(dt), b["batch"], b["center_node_idx"], 3, 5, "gin",
                                True, masks=masks, p=p)

    with torch.no_grad():
        ref = logits(full)
    g32, g64, floor = _oracle_grads(lambda L: torch.nn.functional.binary_cross_entropy_with_logits(logits(L).double(), y), full)
    model = bio.GNN_graphpred(5, 300, 40, drop_ratio=p)
    model.load_state_dict(full)
    model.to(DEV).train()
    torch.manual_seed(5)
    out = model(types.SimpleNamespace(**_dev(b)))
    torch.nn.functional.binary_cross_entropy_with_logits(out.double(), y.to(DEV)).backward()
    assert torch.allclose(out.detach().cpu(), ref.detach(), atol=1e-4, rtol=1e-4)
    _check_grads(model.named_parameters(), g32, g64, floor)


# ---------------------------------------------------------------------------------------------------------------------
# 4. the fine-tuning step
# ---------------------------------------------------------------------------------------------------------------------
def test_finetune_step_vs_oracle():
    T, p = 12, 0.5
    step = ts.FinetuneStep(DEV, "gin", batch_size=32, num_tasks=T, drop_ratio=p)
    P = DO.finetune_params("gin", 3, T)
    step.load_state(P)
    b = step.make_batches(0, 1)[0]
    n = b["x"].shape[0]
    masks = DO.layer_masks(_seed_after(11), 5, n, 300, p, torch.float32)
    L64 = O.leaf_params(P, torch.float64)
    loss64, _ = DO.finetune_loss(L64, b, masks, p)
    loss64.backward()
    L32 = O.leaf_params(P, torch.float32)
    loss32, _ = DO.finetune_loss(L32, b, masks, p)
    loss32.backward()
    torch.manual_seed(11)
    loss = step(_dev(b))
    assert abs(loss.item() - loss64.item()) <= 2e-6 * abs(loss64.item()), (loss.item(), loss64.item())
    g32 = {k: v.grad for k, v in L32.items() if v.requires_grad}
    g64 = {k: v.grad for k, v in L64.items() if v.requires_grad}
    mags = sorted(float(v.abs().max()) for v in g64.values())
    _check_grads(step.named_parameters(), g32, g64, max(mags[len(mags) // 2], 1e-3))


# ---------------------------------------------------------------------------------------------------------------------
# 5. p = 0 through the new entry points is the old entry points, bit for bit
# ---------------------------------------------------------------------------------------------------------------------
def _run_entry(model, plan, d, g, new):
    ptrs = plan.PtrArr(*[p.data_ptr() for p in plan.params])
    rm = plan.BnArr(*[bn.running_mean.data_ptr() for bn in plan.bns])
    rv = plan.BnArr(*[bn.running_var.data_ptr() for bn in plan.bns])
    nbt = plan.BnArr(*[bn.num_batches_tracked.data_ptr() for bn in plan.bns])
    x, ei, ea = d["x"], d["edge_index"], d["edge_attr"]
    N, E, L, D = x.shape[0], ei.shape[1], plan.L, plan.D
    wsb = plan.workspace_bytes(N, E)
    ws = torch.empty(wsb, dtype=torch.uint8, device=DEV)
    out = torch.empty(N, D, device=DEV)
    flat = torch.full((plan.total,), SENT, device=DEV)
    st = ctypes.c_void_p(ops._st())
    P = ops._p
    head = (ptrs, rm, rv, nbt, P(x), P(ei), P(ea), N, E, L, D, 1, 0.1, 1e-5)
    tail = (1, P(out), D, P(ws), wsb, st)
    torch.cuda.synchronize()
    n0 = lib.pgnn_kernel_launch_count()
    if new:
        assert lib.pgnn_chem_encoder_forward(plan.conv, *head, 0.0, 987654321, *tail) == 0
        assert lib.pgnn_chem_encoder_backward(plan.conv, ptrs, P(g), D, P(x), P(ea), N, E, L, D, 0.0, 987654321, 1, P(flat), P(ws), wsb,
                                              st) == 0
    elif plan.conv:
        assert lib.pgnn_chem_conv_forward(plan.conv, *head, *tail) == 0
        assert lib.pgnn_chem_conv_backward(plan.conv, ptrs, P(g), D, P(x), P(ea), N, E, L, D, 1, P(flat), P(ws), wsb, st) == 0
    else:
        assert lib.pgnn_chem_gin_forward(*head, *tail) == 0
        assert lib.pgnn_chem_gin_backward(ptrs, P(g), D, P(x), N, E, L, D, 1, P(flat), P(ws), wsb, st) == 0
    torch.cuda.synchronize()
    launches = lib.pgnn_kernel_launch_count() - n0
    grads = [v.cpu() for v in flat.split(plan.sizes)]
    return out.cpu(), grads, {k: v.cpu().clone() for k, v in model.state_dict().items()}, launches


@pytest.mark.parametrize("t", TYPES)
def test_new_entry_points_at_p0_equal_old_ones(t):
    """drop_p = 0 through pgnn_chem_encoder_* against pgnn_chem_gin_* / pgnn_chem_conv_* on a masking batch (B = 256): the same
    kernels (launch count), bit-identical outputs, and every gradient tensor and BatchNorm buffer bit-identical wherever the old
    entry points repeat themselves bit for bit.  (Bias, BatchNorm and bond-table gradients are folded with fp32 / fp64 atomics
    whose order varies from run to run: where two runs of the old entry points differ, the new one must lie within that
    run-to-run difference, as test_training_step_run_to_run_reproducibility measures it.)"""
    b = _dev(ts.make_batches("masking", 0, 1)[0])
    P = O.make_params("chem", t, 5, 300, seed=13)
    g = probe((b["x"].shape[0], 300), 8).to(DEV)
    res = []
    for new in (False, False, True):
        model = _chem_model(t, P, True, 0.0)
        res.append(_run_entry(model, model._fused_plan(), b, g, new))
    (o0, g0, s0, n0), (o1, g1, s1, n1), (o2, g2, s2, n2) = res
    assert n0 == n1 == n2
    assert torch.equal(o0, o1) and torch.equal(o0, o2)
    gmax = max(float(v.abs().max()) for v in g0)
    for i, (a, a1, c) in enumerate(zip(g0, g1, g2)):
        if torch.equal(a, a1):
            assert torch.equal(a, c), (t, i, "bit-reproducible on the old path, different on the new one")
        else:
            noise = float((a - a1).abs().max())
            scale = max(float(a.abs().max()), 1e-3 * gmax)
            assert float((a - c).abs().max()) <= max(4 * noise, 3e-4 * scale), (t, i)
    for k in s0:
        if torch.equal(s0[k], s1[k]):
            assert torch.equal(s0[k], s2[k]), k
        else:
            assert torch.allclose(s0[k].double(), s2[k].double(), atol=1e-6, rtol=1e-6), k


# ---------------------------------------------------------------------------------------------------------------------
# 6. seeds
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fused", [True, False])
def test_seed_behaviour(fused):
    b = _dev(syn.zinc_batch(16, 3))
    P = O.make_params("chem", "gin", 5, 300, seed=2)
    model = _chem_model("gin", P, fused, 0.5)
    with torch.no_grad():
        torch.manual_seed(42)
        a = model(b["x"], b["edge_index"], b["edge_attr"])
        a2 = model(b["x"], b["edge_index"], b["edge_attr"])
        torch.manual_seed(42)
        c = model(b["x"], b["edge_index"], b["edge_attr"])
        assert torch.equal(a == 0, c == 0)                   # same manual_seed, same masks
        assert not torch.equal(a == 0, a2 == 0)              # consecutive forwards, different masks
        model.eval()
        state = torch.get_rng_state()
        e = model(b["x"], b["edge_index"], b["edge_attr"])
        assert torch.equal(torch.get_rng_state(), state)     # eval draws nothing
        assert float((e == 0).float().mean()) < 0.05         # and drops nothing
        model.train()
        model.drop_ratio = 0
        state = torch.get_rng_state()
        model(b["x"], b["edge_index"], b["edge_attr"])
        assert torch.equal(torch.get_rng_state(), state)     # p = 0 draws nothing either
