"""CPU: the dropout draw's definition (tests/dropout_oracle.py restates it), where dropout sits in the reference's own chem / bio
models (through oracle/reference_runner.py, skipped when the reference sources are absent), and the argument checks of the
dropout entry points."""
import ctypes
import importlib

import numpy as np
import pytest
import torch
from scipy import stats

import dropout_oracle as DO
from oracle import gnn_oracle as O
from oracle import reference_runner as R
from oracle import step_io_oracle as SO

syn = importlib.import_module("pretrain-gnns_b200.synthetic")
TYPES = ("gin", "gcn", "graphsage", "gat")


# ---------------------------------------------------------------------------------------------------------------------
# the draw
# ---------------------------------------------------------------------------------------------------------------------
def test_vectorised_hash_is_the_scalar_one():
    idx = np.array([0, 1, 2, 12345, (7 << 40) | 99, (1 << 63) + 5], dtype=np.uint64)
    for seed in (0, 1, (1 << 62) - 1, 0x123456789ABCDEF):
        assert [int(v) for v in DO.splitmix64(seed, idx)] == [SO.splitmix64(seed, int(i)) for i in idx]


def test_threshold_and_scale_definition():
    assert DO.threshold(0.0) == 0 and DO.threshold(1.0) == 1 << 32
    assert DO.threshold(0.5) == 1 << 31
    assert DO.threshold(0.1) == int(np.floor(float(np.float32(0.1)) * 2 ** 32))  # the fp32 p the library receives
    assert DO.scale(0.5) == 2.0 and DO.scale(1.0) == 0.0
    assert not DO.keep_mask(3, 0, 4, 5, 1.0).any() and DO.keep_mask(3, 0, 4, 5, 0.0).all()


@pytest.mark.parametrize("p", [0.1, 0.2, 0.5, 0.9])
def test_keep_rate_within_5_sigma(p):
    rows, C = 40000, 300  # 1.2e7 draws over 8 layers x a few seeds
    kept = n = 0
    for seed, layer in ((1, 0), (2, 3), ((1 << 62) - 7, 4), (12345, 1)):
        m = DO.keep_mask(seed, layer, rows // 4, C, p)
        kept += int(m.sum())
        n += m.size
    q = 1.0 - DO.threshold(p) / 2.0 ** 32
    sigma = (q * (1 - q) / n) ** 0.5
    assert abs(kept / n - q) <= 5 * sigma, (kept / n, q, sigma)


def _chi2_independent(a, b):
    table = np.array([[np.sum(a & b), np.sum(a & ~b)], [np.sum(~a & b), np.sum(~a & ~b)]])
    return stats.chi2_contingency(table, correction=False).pvalue


@pytest.mark.parametrize("p", [0.2, 0.5, 0.9])
def test_pairs_show_no_dependence(p):
    """Keep decisions of adjacent columns, of the same element in adjacent layers and under consecutive seeds are independent
    by a 2x2 chi-square test (each over ~3.6e6 pairs)."""
    rows, C, seed = 12000, 301, 77
    m0 = DO.keep_mask(seed, 2, rows, C, p)
    pv = [_chi2_independent(m0[:, :-1].ravel(), m0[:, 1:].ravel()),                       # adjacent columns
          _chi2_independent(m0.ravel(), DO.keep_mask(seed, 3, rows, C, p).ravel()),        # adjacent layers
          _chi2_independent(m0.ravel(), DO.keep_mask(seed + 1, 2, rows, C, p).ravel())]    # consecutive seeds
    assert min(pv) > 1e-4, pv


# ---------------------------------------------------------------------------------------------------------------------
# where dropout sits: the reference's own models with F.dropout replaced by the given masks, against the masked oracle (fp64)
# ---------------------------------------------------------------------------------------------------------------------
class _MaskedF:
    """Stands in for the `F` (torch.nn.functional) a reference model module imported: F.dropout applies the next mask in call
    order (training mode) and counts its calls; everything else is torch's."""

    def __init__(self, masks):
        self.masks, self.calls = masks, 0

    def __getattr__(self, name):
        return getattr(torch.nn.functional, name)

    def dropout(self, x, p=0.5, training=True, inplace=False):
        if not training:
            return x
        m = self.masks[self.calls]
        self.calls += 1
        assert m.shape == x.shape, (m.shape, x.shape)
        return x * m.to(x.dtype) * (1.0 / (1.0 - p))


def _grads_close(ref_params, L, what):
    gmax = max(float(p.grad.abs().max()) for p in ref_params.values() if p.grad is not None)
    for k, p in ref_params.items():
        if p.grad is None:
            continue
        g = L[k].grad
        assert g is not None, (what, k)
        err = float((g - p.grad).abs().max())
        assert err <= 1e-9 * max(float(p.grad.abs().max()), 1e-4 * gmax), (what, k, err)


needs_ref = pytest.mark.skipif(not R.available(), reason="reference sources not available (no /root/reference, no oracle/_ref)")


@needs_ref
@pytest.mark.parametrize("domain", ["chem", "bio"])
@pytest.mark.parametrize("t", TYPES)
def test_reference_dropout_placement_equals_masked_oracle(domain, t, monkeypatch):
    torch.set_num_threads(1)
    mod = R.load(domain)
    p = 0.5 if domain == "chem" else 0.2
    b = syn.zinc_batch(6, 31) if domain == "chem" else syn.ppi_batch(2, 31, n_lo=30, n_hi=50, num_tasks=8)
    P = O.make_params(domain, t, 5, 300, seed=8)
    n = b["x"].shape[0]
    masks = DO.layer_masks(1234, 5, n, 300, p)
    fake = _MaskedF(masks)
    monkeypatch.setattr(mod, "F", fake)
    model = mod.GNN(5, 300, JK="last", drop_ratio=p, gnn_type=t)
    assert str(model.load_state_dict(P)) == "<All keys matched successfully>"
    model.double().train()
    x = b["x"].double() if b["x"].is_floating_point() else b["x"]
    ea = b["edge_attr"].double() if b["edge_attr"].is_floating_point() else b["edge_attr"]
    y = model(x, b["edge_index"], ea)
    assert fake.calls == 5  # one dropout per layer: never on h0, never inside bio GIN's MLP
    Rm = torch.randn(y.shape, generator=torch.Generator().manual_seed(3), dtype=torch.float64)
    (y * Rm).sum().backward()
    L = O.leaf_params(P, torch.float64)
    fwd = DO.chem_gnn if domain == "chem" else DO.bio_gnn
    y2 = fwd(L, x, b["edge_index"], ea, 5, t, True, masks=masks, p=p)
    (y2 * Rm).sum().backward()
    assert torch.allclose(y2, y, atol=1e-10, rtol=1e-9), (y2 - y).abs().max()
    _grads_close(dict(model.named_parameters()), L, (domain, t))


@needs_ref
def test_reference_finetune_step_equals_masked_oracle(monkeypatch):
    """GNN_graphpred + chem/finetune.py:31-44's loss on the reference's own module: dropout only inside the encoder, never in
    the graph head."""
    torch.set_num_threads(1)
    mod = R.load("chem")
    p, T = 0.5, 12
    b = syn.finetune_batch(6, 44, T)
    P = DO.finetune_params("gin", 5, T)
    n = b["x"].shape[0]
    masks = DO.layer_masks(99, 5, n, 300, p)
    fake = _MaskedF(masks)
    monkeypatch.setattr(mod, "F", fake)
    model = mod.GNN_graphpred(5, 300, T, JK="last", drop_ratio=p, graph_pooling="mean", gnn_type="gin")
    assert str(model.load_state_dict({k[len("model."):]: v for k, v in P.items()})) == "<All keys matched successfully>"
    model.double().train()
    pred = model(b["x"], b["edge_index"], b["edge_attr"], b["batch"])
    assert fake.calls == 5
    y = b["y"].view(pred.shape).to(torch.float64)
    is_valid = y ** 2 > 0
    loss_mat = torch.nn.BCEWithLogitsLoss(reduction="none")(pred.double(), (y + 1) / 2)
    loss_mat = torch.where(is_valid, loss_mat, torch.zeros(loss_mat.shape).to(loss_mat.dtype))
    loss = torch.sum(loss_mat) / torch.sum(is_valid)
    loss.backward()
    L = O.leaf_params(P, torch.float64)
    loss2, _ = DO.finetune_loss(L, b, masks, p)
    loss2.backward()
    assert abs(loss2.item() - loss.item()) <= 1e-12 * abs(loss.item())
    _grads_close({"model." + k: v for k, v in model.named_parameters()}, L, "finetune")


# ---------------------------------------------------------------------------------------------------------------------
# argument checks (need the library, not a GPU: every check runs before anything is enqueued)
# ---------------------------------------------------------------------------------------------------------------------
def _lib():
    cabi = importlib.import_module("pretrain-gnns_b200._cabi")
    try:
        return cabi.lib.load()
    except cabi.PgnnError:
        pytest.skip("libpgnn_b200.so is not built")


def test_dropout_argument_validation_without_gpu():
    lib = _lib()
    EINVAL, EWS = -1, -3
    fake = ctypes.c_void_p(0x1000)
    for p in (-0.1, 1.5, float("nan")):
        assert lib.pgnn_dropout_fwd(fake, 4, 2, 4, p, 1, 0, fake, 4, None) == EINVAL
        assert lib.pgnn_dropout_bwd(fake, 4, 2, 4, p, 1, 0, fake, 4, None) == EINVAL
    assert lib.pgnn_dropout_fwd(fake, 4, 2, 4, 0.5, 1, -1, fake, 4, None) == EINVAL      # negative layer
    assert lib.pgnn_dropout_fwd(fake, 4, 2, 4, 0.5, 1, 1 << 24, fake, 4, None) == EINVAL  # layer past its 24 bits
    assert lib.pgnn_dropout_fwd(fake, 2, 2, 4, 0.5, 1, 0, fake, 4, None) == EINVAL       # ldx < C
    assert lib.pgnn_dropout_fwd(None, 4, 0, 4, 0.5, 1, 0, None, 4, None) == 0            # M == 0: nothing to do

    L, D, N, E = 5, 300, 10, 20
    arr = (ctypes.c_void_p * 64)(*([0x1000] * 64))
    for t, ws_of in ((0, lambda: lib.pgnn_chem_gin_workspace_bytes(N, E, L, D)),
                     (1, lambda: lib.pgnn_chem_conv_workspace_bytes(1, N, E, L, D)),
                     (2, lambda: lib.pgnn_chem_conv_workspace_bytes(2, N, E, L, D)),
                     (3, lambda: lib.pgnn_chem_conv_workspace_bytes(3, N, E, L, D))):
        wsb = ws_of()
        assert wsb > 0

        def fwd(p, ws=wsb, gnn_type=t):
            return lib.pgnn_chem_encoder_forward(gnn_type, arr, arr, arr, arr, fake, fake, fake, N, E, L, D, 1, 0.1, 1e-5, p, 7, 1, fake,
                                                 D, fake, ws, None)

        def bwd(p, ws=wsb, gnn_type=t):
            return lib.pgnn_chem_encoder_backward(gnn_type, arr, fake, D, fake, fake, N, E, L, D, p, 7, 1, fake, fake, ws, None)

        for p in (-0.1, 1.0000001, float("nan")):
            assert fwd(p) == EINVAL and bwd(p) == EINVAL, (t, p)
        assert fwd(0.5, wsb - 1) == EWS and bwd(0.5, wsb - 1) == EWS, t
    for bad in (-1, 4, 5):
        assert lib.pgnn_chem_encoder_forward(bad, arr, arr, arr, arr, fake, fake, fake, N, E, L, D, 1, 0.1, 1e-5, 0.5, 7, 1, fake, D, fake,
                                             1 << 40, None) == EINVAL
        assert lib.pgnn_chem_encoder_backward(bad, arr, fake, D, fake, fake, N, E, L, D, 0.5, 7, 1, fake, fake, 1 << 40, None) == EINVAL
    # the dropout-free entry points still refuse the types they never served
    for bad in (0, 4):
        assert lib.pgnn_chem_conv_forward(bad, arr, arr, arr, arr, fake, fake, fake, N, E, L, D, 1, 0.1, 1e-5, 1, fake, D, fake, 1 << 40,
                                          None) == EINVAL
        assert lib.pgnn_chem_conv_backward(bad, arr, fake, D, fake, fake, N, E, L, D, 1, fake, fake, 1 << 40, None) == EINVAL


def test_seed_draw_is_a_host_op_of_the_default_generator():
    ops = importlib.import_module("pretrain-gnns_b200.ops")
    torch.manual_seed(5)
    a = [ops.draw_seed() for _ in range(3)]
    torch.manual_seed(5)
    assert [ops.draw_seed() for _ in range(3)] == a
    assert len(set(a)) == 3 and all(0 <= s < 1 << 62 for s in a)
