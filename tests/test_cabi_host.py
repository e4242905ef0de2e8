"""CPU: the C-ABI library loads, exports every symbol include/pgnn_b200.h declares, validates arguments
without touching a device, and the host-side modules keep the reference's state_dict contract."""
import ctypes
import importlib
import os

import pytest
import torch

from oracle import gnn_oracle as O

cabi = importlib.import_module("pretrain-gnns_b200._cabi")


def test_library_built_and_exports_header_symbols():
    assert os.path.exists(cabi.LIB_PATH), "run `python pretrain-gnns_b200/build.py`"
    protos = cabi.parse_header()
    assert len(protos) >= 38
    dll = cabi.lib.load()
    for name in protos:
        assert hasattr(dll, name), name
    assert dll.pgnn_version() >= 100
    assert dll.pgnn_error_string(-3) == b"workspace too small"


def test_argument_validation_without_gpu():
    dll = cabi.lib.load()
    assert dll.pgnn_bucket_workspace_bytes(-1, 3) == -1
    assert dll.pgnn_bucket_workspace_bytes(100, 10) > 0
    assert dll.pgnn_linear_fwd(None, 0, None, None, 4, 0, 3, 0, None, 0, 0, None) == -1   # N == 0
    assert dll.pgnn_linear_fwd(None, 0, None, None, 0, 4, 3, 0, None, 0, 0, None) == 0    # M == 0: nothing to do
    assert dll.pgnn_aggregate_fwd(None, 0, None, None, 0, 0, 300, None, None, 0, None, None, 0, None, 0, None, 0, None) == 0
    assert dll.pgnn_aggregate_fwd(None, 0, None, None, 0, 5, 300, None, None, 7, None, None, 0, None, 0, None, 0, None) == -1
    off = (ctypes.c_int64 * 64)()
    for conv_type in (0, 4):   # 1..3 are GCN / GraphSAGE / GAT; GIN has entry points of its own
        assert dll.pgnn_chem_conv_num_params(conv_type, 5) == -1
        assert dll.pgnn_chem_conv_grad_offsets(conv_type, 5, 300, off) == -1
        assert dll.pgnn_chem_conv_workspace_bytes(conv_type, 100, 200, 5, 300) == -1
    with pytest.raises(cabi.PgnnError):
        cabi.check(-4, "x")


def test_debug_bn_entries_validate_arguments_without_gpu():
    """pgnn_debug_bn_apply_fold / pgnn_debug_bn_bwd_colsum reject bad sizes and row strides, missing pointers, a dropout p outside
    [0, 1] and a short workspace before anything is enqueued (the fake addresses below are never dereferenced)."""
    dll = cabi.lib.load()
    P = 256  # a non-null address

    def fold(M=8, C=4, x=P, sums=P, y=P, ldx=4, ldy=4, p=0.0):
        return dll.pgnn_debug_bn_apply_fold(x, ldx, M, C, sums, P, P, None, None, None, 0.1, 1e-5, None, None, 1, y, ldy, p, 0, 0, None)

    assert fold(M=0) == -1 and fold(C=0) == -1 and fold(M=1 << 31) == -1
    assert fold(C=6145, ldx=6148, ldy=6148) == -1   # scale / shift of more columns than 48 KiB of shared memory holds
    assert fold(x=None) == -1 and fold(sums=None) == -1 and fold(y=None) == -1
    assert fold(ldx=3) == -1 and fold(ldy=3) == -1
    assert fold(p=1.5) == -1 and fold(p=-0.1) == -1 and fold(p=float("nan")) == -1
    wsb = dll.pgnn_bn_workspace_bytes(8, 4)
    assert wsb > 0

    def bwd(M=8, C=4, gy=P, colsum=P, ws=P, wsb=wsb, p=0.0, ldgy=4, ldx=4, ldgx=4):
        return dll.pgnn_debug_bn_bwd_colsum(gy, ldgy, P, ldx, M, C, P, P, P, P, 1, P, ldgx, None, None, colsum, p, 0, 0, ws, wsb, None)

    assert bwd(M=0) == -1 and bwd(C=0) == -1 and bwd(M=1 << 31) == -1
    assert bwd(gy=None) == -1 and bwd(colsum=None) == -1 and bwd(ws=None) == -1
    assert bwd(p=2.0) == -1
    assert bwd(wsb=wsb - 1) == -3
    assert bwd(ldgy=3) == -1 and bwd(ldx=3) == -1 and bwd(ldgx=3) == -1
    # the whole-encoder gather's view of the workspace (GIN debug layout): additive to pgnn_chem_gin_debug_layout
    off4 = (ctypes.c_int64 * 4)()
    assert dll.pgnn_chem_gin_debug_layout(100, 200, 3, 300, off4) == 0
    aggr = dll.pgnn_chem_gin_debug_aggr_offset(100, 200, 3, 300)
    assert aggr > 0 and all(aggr + 3 * 100 * 300 * 4 <= o or o + 4 <= aggr for o in off4)
    assert dll.pgnn_chem_gin_debug_aggr_offset(-1, 0, 3, 300) == -1 and dll.pgnn_chem_gin_debug_aggr_offset(10, 0, 0, 300) == -1


@pytest.mark.parametrize("domain", ["chem", "bio"])
@pytest.mark.parametrize("t", ["gin", "gcn", "graphsage", "gat"])
def test_state_dict_contract(domain, t):
    mod = importlib.import_module(f"pretrain-gnns_b200.{domain}.model")
    model = mod.GNN(5, 300, gnn_type=t)
    P = O.make_params(domain, t, 5, 300, seed=1)
    assert set(model.state_dict().keys()) == set(P.keys())
    for k, v in model.state_dict().items():
        assert tuple(v.shape) == tuple(P[k].shape), k
    total = {
        ("chem", "gin"): 1857900, ("chem", "gcn"): 504900, ("chem", "graphsage"): 504900, ("chem", "gat"): 977400,
        ("bio", "gin"): 2726100, ("bio", "gcn"): 467100, ("bio", "graphsage"): 467100, ("bio", "gat"): 941100}[(domain, t)]
    assert sum(p.numel() for p in model.parameters()) == total
    if domain == "chem":
        # the whole-encoder plan (host calls only): its flat gradient layout tiles [0, total) in parameter order
        plan = model._fused_plan()
        assert plan is not None and plan.gnn_type == t
        assert sorted(map(id, plan.params)) == sorted(map(id, model.parameters()))
        assert len(plan.offsets) == len(plan.params) + 1 and plan.offsets[0] == 0 and plan.offsets[-1] == plan.total == total
        for i, p in enumerate(plan.params):
            assert plan.offsets[i + 1] - plan.offsets[i] == p.numel(), i


def test_shipped_checkpoints_load():
    """The reference's shipped checkpoints (model_gin/*.pth, model_architecture/{gcn,gat,graphsage}_*.pth) load into the drop-in
    modules key for key: their state_dict key names, dtypes and shapes are recorded in tests/golden/checkpoint_keys.json."""
    import json
    chem = importlib.import_module("pretrain-gnns_b200.chem.model")
    bio = importlib.import_module("pretrain-gnns_b200.bio.model")
    with open(os.path.join(os.path.dirname(__file__), "golden", "checkpoint_keys.json")) as fh:
        rec = json.load(fh)   # {"files": {path: schema index}, "schemas": [{key: [dtype, shape]}]}
    n = 0
    for f, i in sorted(rec["files"].items()):
        keys = rec["schemas"][i]
        mod = chem if f.startswith("chem/") else bio
        t = "gin" if "/model_gin/" in f else "gcn" if "gcn" in f else "gat" if "gat" in f else "graphsage"
        sd = {k: torch.zeros(shape, dtype=getattr(torch, dt)) for k, (dt, shape) in keys.items()}
        assert str(mod.GNN(5, 300, gnn_type=t).load_state_dict(sd)) == "<All keys matched successfully>", f
        n += 1
    assert n >= 18


def test_cpu_forward_fails_loudly():
    chem = importlib.import_module("pretrain-gnns_b200.chem.model")
    g = chem.GNN(5, 300)
    with pytest.raises(cabi.PgnnError):
        g(torch.zeros(3, 2, dtype=torch.long), torch.zeros(2, 0, dtype=torch.long), torch.zeros(0, 2, dtype=torch.long))


def test_constructor_errors():
    chem = importlib.import_module("pretrain-gnns_b200.chem.model")
    bio = importlib.import_module("pretrain-gnns_b200.bio.model")
    for mod in (chem, bio):
        with pytest.raises(ValueError):
            mod.GNN(1, 300)
        with pytest.raises(ValueError):
            mod.GNN_graphpred(1, 300, 3)
        with pytest.raises(ValueError):
            mod.GNN_graphpred(5, 300, 3, graph_pooling="nope")
