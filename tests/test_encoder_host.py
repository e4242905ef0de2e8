"""The whole-encoder bounds of tests/test_gpu_encoder.py reject plausible encoder bugs (CPU only).

Each variant restates one mistake an encoder kernel could make, in fp64 on the same inputs, parameters, dropout masks and upstream
gradient as the GPU test's oracle, and the same checks (tests/encoder_oracle.py: output_check, gradient_check with its
ReLU-boundary allowance, the running-statistics bound) must reject it at the bounds the fp32 oracle's own error sets, while the
unperturbed restatement passes them.  The margin of each variant (largest error / bound) is printed."""
import importlib

import pytest
import torch
import torch.nn.functional as F

import dropout_oracle as DO
import encoder_oracle as EO
from golden_util import probe
from oracle import gnn_oracle as O

syn = importlib.import_module("pretrain-gnns_b200.synthetic")
TYPES = ("gin", "gcn", "graphsage", "gat")
P_DROP, SEED = 0.3, 4242
FORWARD_VARIANTS = ("previous layer's dropout mask", "ReLU after the last layer", "self-loop bond row missing",
                    "self-loop bond type 0 instead of 4", "bond tables swapped", "BatchNorm normalised with the unbiased variance",
                    "running variance updated with the biased variance")
GRAD_VARIANTS = ("chirality rows written into the atom table's last rows", "one layer's weight gradient left at zero")


def _edge_rows(P, lp, edge_attr, n, v):
    loops = torch.zeros(n, 2, dtype=edge_attr.dtype)
    loops[:, 0] = 0 if v == "self-loop bond type 0 instead of 4" else O.SELF_LOOP_BOND
    t1, t2 = P[lp + "edge_embedding1.weight"], P[lp + "edge_embedding2.weight"]
    ea = torch.cat([edge_attr, loops])
    if v == "bond tables swapped":  # the [9, C] block the kernels index, with the direction table in front
        T = torch.cat([t2, t1])
        return T[ea[:, 0]] + T[6 + ea[:, 1]]
    rows = F.embedding(ea[:, 0], t1) + F.embedding(ea[:, 1], t2)
    if v == "self-loop bond row missing":
        rows = torch.cat([rows[:-n], torch.zeros_like(rows[-n:])])
    return rows


def _batch_norm(P, pre, h, new_stats, v):
    if v not in ("BatchNorm normalised with the unbiased variance", "running variance updated with the biased variance"):
        return O.batch_norm(P, pre, h, True, new_stats)
    mean, vb, vu = h.mean(0), h.var(0, unbiased=False), h.var(0, unbiased=True)
    vn = vu if v == "BatchNorm normalised with the unbiased variance" else vb
    vr = vb if v == "running variance updated with the biased variance" else vu
    new_stats[pre + "running_mean"] = (1 - O.BN_MOMENTUM) * P[pre + "running_mean"] + O.BN_MOMENTUM * mean.detach()
    new_stats[pre + "running_var"] = (1 - O.BN_MOMENTUM) * P[pre + "running_var"] + O.BN_MOMENTUM * vr.detach()
    return (h - mean) / torch.sqrt(vn + O.BN_EPS) * P[pre + "weight"] + P[pre + "bias"]


def variant_gnn(v):
    """DO.chem_gnn (training mode) with the mistake `v` (None: none)."""
    def fn(P, x, edge_index, edge_attr, L, t, training, new_stats, masks=None, p=0.0):
        assert training
        n = x.shape[0]
        h = F.embedding(x[:, 0], P["x_embedding1.weight"]) + F.embedding(x[:, 1], P["x_embedding2.weight"])
        ei = O.with_self_loops(edge_index, n)
        conv = {"gin": O.gin_conv_chem, "gcn": O.gcn_conv, "graphsage": O.sage_conv, "gat": O.gat_conv}[t]
        for l in range(L):
            lp = f"gnns.{l}."
            h = conv(P, lp, h, ei, _edge_rows(P, lp, edge_attr, n, v))
            h = _batch_norm(P, f"batch_norms.{l}.", h, new_stats, v)
            if l != L - 1 or v == "ReLU after the last layer":
                h = torch.relu(h)
            h = DO._drop(h, masks, l - 1 if v == "previous layer's dropout mask" and l > 0 else l, p)
        return h
    return fn


def _grad_variant(g64, v, t, L):
    g = {k: x.clone() for k, x in g64.items()}
    if v == "chirality rows written into the atom table's last rows":
        g["x_embedding1.weight"][-3:] = g["x_embedding2.weight"]
    else:
        w = "mlp.0.weight" if t == "gin" else "weight_linear.weight" if t == "gat" else "linear.weight"
        g[f"gnns.{L // 2}.{w}"].zero_()
    return g


def _checks(ref, out, grads, stats, L):
    rows = []
    ok = EO.check_output("node_rep", out, ref, rows)
    ok &= EO.check_grads(sorted(grads.items()), ref, rows)
    ok &= EO.check_all_stats(stats, ref, L, rows)
    return ok, rows


@pytest.mark.parametrize("D,L", [(36, 3), (300, 5)])
@pytest.mark.parametrize("t", TYPES)
def test_encoder_bounds_reject_wrong_variants(t, D, L):
    torch.set_num_threads(min(torch.get_num_threads(), 8))
    b = syn.zinc_batch(8, 31)
    n = b["x"].shape[0]
    P = O.make_params("chem", t, L, D, seed=17, randomize_bn=True)
    masks = DO.layer_masks(SEED, L, n, D, P_DROP)
    g = probe((n, D), 3)
    ref = EO.Ref(P, b, t, L, True, g, masks, P_DROP)
    # the bounds admit the fp32 oracle and the unperturbed restatement
    ok, rows = _checks(ref, ref.out[EO.F32], ref.grads[EO.F32], ref.stats[EO.F32], L)
    assert ok, [r for r in rows if not r["ok"]]
    out, grads, stats, _ = EO.run(P, b, t, L, True, EO.F64, g, masks, P_DROP, fn=variant_gnn(None))
    ok, rows = _checks(ref, out, grads, stats, L)
    assert ok, [r for r in rows if not r["ok"]]
    margins = {}
    for v in FORWARD_VARIANTS + GRAD_VARIANTS:
        if v in GRAD_VARIANTS:
            out, grads, stats = ref.out[EO.F64], _grad_variant(ref.grads[EO.F64], v, t, L), ref.stats[EO.F64]
        else:
            out, grads, stats, _ = EO.run(P, b, t, L, True, EO.F64, g, masks, P_DROP, fn=variant_gnn(v))
        ok, rows = _checks(ref, out, grads, stats, L)
        margins[v] = EO.margin(rows)
        assert not ok, (v, margins[v])
    print("\n%s D=%d L=%d: bound margins of the wrong variants (error / bound):" % (t, D, L))
    for v, m in margins.items():
        print("  %-58s %10.3g" % (v, m))
    assert min(margins.values()) > 1, margins
