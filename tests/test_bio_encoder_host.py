"""CPU: the bio whole-encoder's host-side contract (pgnn_bio_encoder_*, include/pgnn_b200.h), from the built library alone.

  * num_params and grad_offsets describe bio.GNN's parameters exactly, in ops.BioEncoderPlan's order, for every type, depth and
    width;
  * workspace sizes are positive and grow with N and with E;
  * bad types, depths, drop probabilities and sizes are refused with PGNN_EINVAL before anything touches a device pointer."""
import ctypes
import importlib

import pytest

bio = importlib.import_module("pretrain-gnns_b200.bio.model")
ops = importlib.import_module("pretrain-gnns_b200.ops")
lib = importlib.import_module("pretrain-gnns_b200._cabi").lib

TYPES = ("gin", "gcn", "graphsage", "gat")
CODE = {"gin": 0, "gcn": 1, "graphsage": 2, "gat": 3}
OK, EINVAL = 0, -1
PER_LAYER = {"gin": 8, "gcn": 4, "graphsage": 4, "gat": 6}


@pytest.mark.parametrize("t", TYPES)
@pytest.mark.parametrize("L", [2, 3, 7])
@pytest.mark.parametrize("D", [4, 36, 300])
def test_layout_matches_module(t, L, D):
    m = bio.GNN(L, D, gnn_type=t)
    plan = ops.BioEncoderPlan(m, t)
    names = {id(p): k for k, p in m.named_parameters()}
    order = [names[id(p)] for p in plan.params]
    assert sorted(order) == sorted(names.values())  # every parameter once
    assert order[0] == "gnns.0.input_node_embeddings.weight"
    assert order[-2:] == [f"gnns.{L - 1}.edge_encoder.weight", f"gnns.{L - 1}.edge_encoder.bias"]
    assert lib.pgnn_bio_encoder_num_params(CODE[t], L) == len(order) == 1 + PER_LAYER[t] * L
    off = (ctypes.c_int64 * (len(order) + 1))()
    assert lib.pgnn_bio_encoder_grad_offsets(CODE[t], L, D, off) == OK
    off = list(off)
    assert off[0] == 0
    assert [off[i + 1] - off[i] for i in range(len(order))] == [p.numel() for p in plan.params]
    assert off[-1] == sum(p.numel() for p in m.parameters())


@pytest.mark.parametrize("t", TYPES)
def test_single_layer_layout(t):
    """L = 1 (the C ABI accepts it; the module does not): layer 0 of the two-layer layout."""
    off1 = (ctypes.c_int64 * (2 + PER_LAYER[t]))()
    off2 = (ctypes.c_int64 * (2 + 2 * PER_LAYER[t]))()
    assert lib.pgnn_bio_encoder_grad_offsets(CODE[t], 1, 36, off1) == OK
    assert lib.pgnn_bio_encoder_grad_offsets(CODE[t], 2, 36, off2) == OK
    assert list(off1) == list(off2)[:2 + PER_LAYER[t]]


@pytest.mark.parametrize("t", TYPES)
def test_workspace_positive_and_monotone(t):
    c = CODE[t]
    for L, D in ((1, 4), (5, 300)):
        prev = first = None
        for N in (0, 1, 129, 4100, 40000):
            row = [lib.pgnn_bio_encoder_workspace_bytes(c, N, E, L, D) for E in (0, 1, 10 * N + 7)]
            assert all(b > 0 for b in row)
            assert row == sorted(row)
            if prev is not None:
                assert all(b >= a for a, b in zip(prev, row))
            prev, first = row, first or row
        assert prev[0] > first[0] and prev[2] > prev[0]


@pytest.mark.parametrize("t", TYPES)
def test_refused(t):
    c = CODE[t]
    assert lib.pgnn_bio_encoder_num_params(c, 0) == EINVAL
    assert lib.pgnn_bio_encoder_workspace_bytes(c, 10, 10, 0, 36) == EINVAL
    assert lib.pgnn_bio_encoder_workspace_bytes(c, -1, 10, 2, 36) == EINVAL
    assert lib.pgnn_bio_encoder_workspace_bytes(c, 10, -1, 2, 36) == EINVAL
    assert lib.pgnn_bio_encoder_workspace_bytes(c, 10, 10, 2, 0) == EINVAL
    off = (ctypes.c_int64 * 64)()
    assert lib.pgnn_bio_encoder_grad_offsets(c, 0, 36, off) == EINVAL
    assert lib.pgnn_bio_encoder_grad_offsets(c, 2, 36, None) == EINVAL
    # the entry points check their arguments before any device pointer is read: null pointers are safe here
    fwd = lambda t_, L, D, p, **kw: lib.pgnn_bio_encoder_forward(t_, None, None, None, None, None, None, None, 4, 0, L, D, 1, 0.1, 1e-5,
                                                                 p, 0, 1, None, D, None, 1 << 30, None)
    bwd = lambda t_, L, D, p: lib.pgnn_bio_encoder_backward(t_, None, None, D, None, None, 4, 0, L, D, p, 0, 1, None, None, 1 << 30, None)
    for call in (fwd, bwd):
        assert call(c, 2, 36, -0.1) == EINVAL
        assert call(c, 2, 36, 1.5) == EINVAL
        assert call(c, 2, 36, float("nan")) == EINVAL
        assert call(c, 0, 36, 0.0) == EINVAL     # L < 1
        assert call(c, 2, 30, 0.0) == EINVAL     # D not a multiple of 4
        assert call(c, 2, 36, 0.0) == EINVAL     # null parameter table / workspace
    for bad in (-1, 4, 7):
        assert lib.pgnn_bio_encoder_num_params(bad, 2) == EINVAL
        assert lib.pgnn_bio_encoder_workspace_bytes(bad, 10, 10, 2, 36) == EINVAL
        assert lib.pgnn_bio_encoder_grad_offsets(bad, 2, 36, off) == EINVAL
        assert fwd(bad, 2, 36, 0.0) == EINVAL and bwd(bad, 2, 36, 0.0) == EINVAL
