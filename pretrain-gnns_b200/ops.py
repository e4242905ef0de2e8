"""Host-side operators: torch tensors in, C-ABI calls out (device pointers + the current CUDA stream).

Every function here is a thin `torch.autograd.Function` (or plain call) around one or two entry points
of `include/pgnn_b200.h`.  torch is used for device memory, the stream and autograd bookkeeping only;
all arithmetic on the path happens in libpgnn_b200.so.  Host tensors are rejected: there is no CPU
fallback.
"""
from __future__ import annotations

import os

import torch
from torch.autograd import Function

from ._cabi import PgnnError, check, lib

AGG_SUM, AGG_MEAN, AGG_GCN = 0, 1, 2
_PRECISION = {"fp32": 0, "tf32x3": 1}
# default: the tensor-core path (measured fp32-class accuracy, tools/check_tc.py); PGNN_PRECISION=fp32 forces FFMA
_precision = _PRECISION.get(os.environ.get("PGNN_PRECISION", "tf32x3"), 1)


def set_precision(name: str):
    """'fp32' = FFMA SIMT GEMMs (exact fp32); 'tf32x3' = error-compensated 3xTF32 wgmma GEMMs."""
    global _precision
    _precision = _PRECISION[name]


def get_precision() -> str:
    return "tf32x3" if _precision == 1 else "fp32"


def _p(t):
    return None if t is None else t.data_ptr()


DEVICE_ERROR_BITS = {1: "node / segment id out of range (edge_index, batch)", 2: "atom code out of range (x)",
                     4: "bond code out of range (edge_attr)", 8: "class label out of range", 16: "gather index out of range"}


def device_errors(clear=True):
    """Names of the index-range violations the kernels of the current device have flagged so far (synchronises the device;
    include/pgnn_b200.h, PGNN_DEVERR_*).  The offending elements were dropped or clamped, never dereferenced."""
    bits = check(lib.pgnn_device_error_flags(int(clear)), "device_error_flags")
    return [name for bit, name in DEVICE_ERROR_BITS.items() if bits & bit]


def raise_on_device_errors():
    """The reference's torch index ops raise a device-side assert on an out-of-range index; call this wherever the host
    synchronises anyway (after reading the loss) to get the same diagnosis.  PGNN_VALIDATE=1 calls it after every graph
    preparation / embedding / loss op (one device synchronisation each: debugging only)."""
    errs = device_errors(clear=True)
    if errs:
        raise PgnnError("out-of-range indices reached the kernels: " + "; ".join(errs))


_VALIDATE = os.environ.get("PGNN_VALIDATE", "") == "1"


_raw_stream = getattr(torch._C, "_cuda_getCurrentRawStream", None)
_cur_device = getattr(torch._C, "_cuda_getDevice", None)


def _st():
    """cudaStream_t of torch's current stream on the current device.  The raw accessor (the one triton's launcher uses) costs ~0.3 us
    against ~4 us for building a torch.cuda.Stream object: every op calls this, eight to thirty times per training step."""
    if _raw_stream is not None and _cur_device is not None:
        return _raw_stream(_cur_device())
    return torch.cuda.current_stream().cuda_stream


def _dev(*tensors):
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise PgnnError("pretrain-gnns_b200 runs on CUDA tensors only: no CPU fallback exists for this path "
                            "(got a %s tensor)" % t.device)


def _f32(t):
    if t.dtype != torch.float32:
        raise PgnnError("fp32 tensors expected, got %s" % t.dtype)
    return t if t.stride(-1) == 1 and (t.dim() < 2 or t.stride(0) >= t.shape[1]) else t.contiguous()


# ------------------------------------------------------------------------------------------------
# graph preparation
# ------------------------------------------------------------------------------------------------
class Graph:
    """Target- and source-bucketed CSR of one batch (pgnn_graph_prep), shared by all layers/passes."""

    def __init__(self, edge_index: torch.Tensor, num_nodes: int):
        _dev(edge_index)
        if edge_index.dtype != torch.int64 or edge_index.dim() != 2 or edge_index.shape[0] != 2:
            raise PgnnError("edge_index must be int64 [2, E]")
        ei = edge_index.contiguous()
        n, e = int(num_nodes), int(ei.shape[1])
        dev = ei.device
        self.n, self.e, self.device = n, e, dev
        self._edge_index = ei  # keeps the storage alive while this object is cached
        i32 = dict(dtype=torch.int32, device=dev)
        buf = torch.empty(2 * (n + 1) + 4 * max(e, 1), **i32)
        o = 0
        self.rowptr_t = buf[o:o + n + 1]; o += n + 1
        self.rowptr_s = buf[o:o + n + 1]; o += n + 1
        self.nbr_t = buf[o:o + e]; o += max(e, 1)
        self.eid_t = buf[o:o + e]; o += max(e, 1)
        self.nbr_s = buf[o:o + e]; o += max(e, 1)
        self.eid_s = buf[o:o + e]
        wsb = lib.pgnn_graph_prep_workspace_bytes(n, e)
        ws = torch.empty(wsb, dtype=torch.uint8, device=dev)
        check(lib.pgnn_graph_prep(_p(ei), e, n, _p(self.rowptr_t), _p(self.nbr_t), _p(self.eid_t), _p(self.rowptr_s),
                                  _p(self.nbr_s), _p(self.eid_s), _p(ws), wsb, _st()), "graph_prep")
        if _VALIDATE:
            raise_on_device_errors()
        self._dinv = None
        self._summaries = {}

    @property
    def dinv(self):
        if self._dinv is None:
            self._dinv = torch.empty(self.n, dtype=torch.float32, device=self.device)
            check(lib.pgnn_gcn_dinv(_p(self.rowptr_t), self.n, _p(self._dinv), _st()), "gcn_dinv")
        return self._dinv

    def summary(self, domain: str, mode: int, edge_attr: torch.Tensor) -> torch.Tensor:
        """S [N,9] (chem) / [N,10] (bio) edge-feature summary for this aggregation mode (cached per batch)."""
        key = (domain, mode)
        hit = self._summaries.get(key)
        if hit is not None and hit[0] is edge_attr and hit[1] == edge_attr._version:
            return hit[2]
        _dev(edge_attr)
        ea = edge_attr.contiguous()
        dinv = self.dinv if mode == AGG_GCN else None
        if domain == "chem":
            if ea.dtype != torch.int64 or ea.shape != (self.e, 2):
                raise PgnnError("chem edge_attr must be int64 [E, 2]")
            S = torch.empty(self.n, 9, dtype=torch.float32, device=self.device)
            check(lib.pgnn_chem_edge_summary(_p(ea), _p(self.rowptr_t), _p(self.nbr_t), _p(self.eid_t), self.n, mode,
                                             _p(dinv), _p(S), _st()), "chem_edge_summary")
        else:
            if ea.dtype != torch.float32 or ea.shape != (self.e, 9):
                raise PgnnError("bio edge_attr must be float32 [E, 9]")
            S = torch.empty(self.n, 10, dtype=torch.float32, device=self.device)
            check(lib.pgnn_bio_edge_summary(_p(ea), _p(self.rowptr_t), _p(self.nbr_t), _p(self.eid_t), self.n, mode,
                                            _p(dinv), _p(S), _st()), "bio_edge_summary")
        self._summaries[key] = (edge_attr, edge_attr._version, S)
        if _VALIDATE:
            raise_on_device_errors()
        return S


_graph_cache = [None]


def graph_for(edge_index: torch.Tensor, num_nodes: int) -> Graph:
    """One-entry cache so that convs called layer by layer on the same batch bucket it once.  The entry
    holds the edge_index tensor itself, so an address match can only be the same live storage; in-place
    edits bump `_version` and invalidate it."""
    hit = _graph_cache[0]
    if hit is not None and hit[0] is edge_index and hit[1] == edge_index._version and hit[2].n == num_nodes:
        return hit[2]
    g = Graph(edge_index, num_nodes)
    _graph_cache[0] = (edge_index, edge_index._version, g)
    return g


def clear_graph_cache():
    _graph_cache[0] = None


class Segments:
    """`batch`-style assignment vector bucketed by segment id (pgnn_bucket): rowptr + stable order."""

    def __init__(self, seg: torch.Tensor, num_seg: int):
        _dev(seg)
        if seg.dtype != torch.int64 or seg.dim() != 1:
            raise PgnnError("segment ids must be int64 [N]")
        self.seg = seg.contiguous()
        n = int(seg.shape[0])
        self.n, self.num_seg = n, int(num_seg)
        self.ptr = torch.empty(self.num_seg + 1, dtype=torch.int32, device=seg.device)
        self.order = torch.empty(max(n, 1), dtype=torch.int32, device=seg.device)
        wsb = lib.pgnn_bucket_workspace_bytes(n, self.num_seg)
        ws = torch.empty(wsb, dtype=torch.uint8, device=seg.device)
        check(lib.pgnn_bucket(_p(self.seg), 1, n, self.num_seg, None, 0, _p(self.ptr), _p(self.order), None, _p(ws),
                              wsb, _st()), "bucket")


# ------------------------------------------------------------------------------------------------
# autograd functions
# ------------------------------------------------------------------------------------------------
class _Aggregate(Function):
    @staticmethod
    def forward(ctx, x, T, graph, S, mode, concat):
        _dev(x, T)
        x, T = _f32(x), _f32(T).contiguous()
        n, C = x.shape
        Q = T.shape[0]
        out = torch.empty(n, 2 * C if concat else C, dtype=torch.float32, device=x.device)
        dinv = graph.dinv if mode == AGG_GCN else None
        check(lib.pgnn_aggregate_fwd(_p(x), x.stride(0), None, None, 0, n, C, _p(graph.rowptr_t), _p(graph.nbr_t), mode,
                                     _p(dinv), _p(S), Q, _p(T), C if concat else 0, _p(out), out.stride(0), _st()),
              "aggregate_fwd")
        ctx.graph, ctx.S, ctx.mode, ctx.concat, ctx.C, ctx.Q = graph, S, mode, concat, C, Q
        return out

    @staticmethod
    def backward(ctx, g):
        g = _f32(g)
        graph, n, C, Q = ctx.graph, ctx.graph.n, ctx.C, ctx.Q
        gx = gT = None
        dinv = graph.dinv if ctx.mode == AGG_GCN else None
        if ctx.needs_input_grad[0]:
            gx = torch.empty(n, C, dtype=torch.float32, device=g.device)
            check(lib.pgnn_aggregate_bwd(_p(g), g.stride(0), n, C, _p(graph.rowptr_s), _p(graph.nbr_s), ctx.mode, _p(dinv),
                                         _p(graph.rowptr_t), _p(gx), C, _st()), "aggregate_bwd")
        if ctx.needs_input_grad[1]:
            gT = torch.empty(Q, C, dtype=torch.float32, device=g.device)
            check(lib.pgnn_edge_table_bwd(_p(ctx.S), Q, _p(g), g.stride(0), C if ctx.concat else 0, n, C, _p(gT), _st()),
                  "edge_table_bwd")
        return gx, gT, None, None, None, None


def aggregate(x, T, graph, S, mode=AGG_SUM, concat=False):
    return _Aggregate.apply(x, T, graph, S, mode, concat)


def _linear_fwd(x, w, b, relu):
    M, K = x.shape
    N = w.shape[0]
    y = torch.empty(M, N, dtype=torch.float32, device=x.device)
    check(lib.pgnn_linear_fwd(_p(x), x.stride(0), _p(w), _p(b), M, N, K, int(relu), _p(y), N, _precision, _st()), "linear_fwd")
    return y


def _linear_bwd_x(gy, w, mask=None):
    M, N = gy.shape
    K = w.shape[1]
    gx = torch.empty(M, K, dtype=torch.float32, device=gy.device)
    check(lib.pgnn_linear_bwd_x(_p(gy), gy.stride(0), _p(w), M, N, K, _p(mask), 0 if mask is None else mask.stride(0),
                                _p(gx), K, _precision, _st()), "linear_bwd_x")
    return gx


def _linear_bwd_w(gy, x, want_bias=True):
    M, N = gy.shape
    K = x.shape[1]
    gw = torch.empty(N, K, dtype=torch.float32, device=gy.device)
    gb = torch.empty(N, dtype=torch.float32, device=gy.device) if want_bias else None
    check(lib.pgnn_linear_bwd_w(_p(gy), gy.stride(0), _p(x), x.stride(0), M, N, K, _p(gw), _p(gb), _precision, _st()),
          "linear_bwd_w")
    return gw, gb


class _Linear(Function):
    @staticmethod
    def forward(ctx, x, w, b):
        _dev(x, w, b)
        x, w = _f32(x), _f32(w).contiguous()
        ctx.save_for_backward(x, w)
        ctx.has_bias = b is not None
        return _linear_fwd(x, w, b, False)

    @staticmethod
    def backward(ctx, g):
        x, w = ctx.saved_tensors
        g = _f32(g)
        gx = _linear_bwd_x(g, w) if ctx.needs_input_grad[0] else None
        gw = gb = None
        if ctx.needs_input_grad[1] or (ctx.has_bias and ctx.needs_input_grad[2]):
            gw, gb = _linear_bwd_w(g, x, ctx.has_bias)
        return gx, gw, gb


def linear(x, w, b=None):
    return _Linear.apply(x, w, b)


class _Mlp2(Function):
    """Linear -> ReLU -> Linear (GINConv.mlp, chem/model.py:29): the hidden activation doubles as the ReLU mask."""

    @staticmethod
    def forward(ctx, a, w1, b1, w2, b2):
        _dev(a, w1, b1, w2, b2)
        a, w1, w2 = _f32(a), _f32(w1).contiguous(), _f32(w2).contiguous()
        z1 = _linear_fwd(a, w1, b1, True)
        z2 = _linear_fwd(z1, w2, b2, False)
        ctx.save_for_backward(a, w1, w2, z1)
        return z2

    @staticmethod
    def backward(ctx, g):
        a, w1, w2, z1 = ctx.saved_tensors
        g = _f32(g)
        gw2, gb2 = _linear_bwd_w(g, z1)
        gz1 = _linear_bwd_x(g, w2, mask=z1)
        gw1, gb1 = _linear_bwd_w(gz1, a)
        ga = _linear_bwd_x(gz1, w1) if ctx.needs_input_grad[0] else None
        return ga, gw1, gb1, gw2, gb2


def mlp2(a, w1, b1, w2, b2):
    return _Mlp2.apply(a, w1, b1, w2, b2)


class _BatchNorm(Function):
    @staticmethod
    def forward(ctx, x, gamma, beta, running_mean, running_var, nbt, training, relu, momentum, eps):
        _dev(x, gamma, beta)
        x = _f32(x)
        M, C = x.shape
        y = torch.empty(M, C, dtype=torch.float32, device=x.device)
        if training:
            if M == 0:
                raise PgnnError("BatchNorm in training mode needs at least one row")
            mean = torch.empty(C, dtype=torch.float32, device=x.device)
            invstd = torch.empty(C, dtype=torch.float32, device=x.device)
            wsb = lib.pgnn_bn_workspace_bytes(M, C)
            ws = torch.empty(wsb, dtype=torch.uint8, device=x.device)
            check(lib.pgnn_bn_fwd_train(_p(x), x.stride(0), M, C, _p(gamma), _p(beta), _p(running_mean), _p(running_var),
                                        _p(nbt), float(momentum), float(eps), int(relu), _p(y), C, _p(mean), _p(invstd),
                                        None, None, _p(ws), wsb, _st()), "bn_fwd_train")
            ctx.save_for_backward(x, gamma, beta, mean, invstd)
        else:
            check(lib.pgnn_bn_fwd_eval(_p(x), x.stride(0), M, C, _p(gamma), _p(beta), _p(running_mean), _p(running_var),
                                       float(eps), int(relu), _p(y), C, _st()), "bn_fwd_eval")
        ctx.training, ctx.relu = training, relu
        return y

    @staticmethod
    def backward(ctx, g):
        if not ctx.training:
            raise PgnnError("backward through eval-mode BatchNorm is not implemented (no in-scope caller trains with "
                            "model.eval(); SURVEY.md section 3.3)")
        x, gamma, beta, mean, invstd = ctx.saved_tensors
        g = _f32(g)
        M, C = x.shape
        gx = torch.empty(M, C, dtype=torch.float32, device=g.device)
        gg = torch.empty(C, dtype=torch.float32, device=g.device)
        gb = torch.empty(C, dtype=torch.float32, device=g.device)
        wsb = lib.pgnn_bn_workspace_bytes(M, C)
        ws = torch.empty(wsb, dtype=torch.uint8, device=g.device)
        check(lib.pgnn_bn_bwd(_p(g), g.stride(0), _p(x), x.stride(0), M, C, _p(gamma), _p(beta), _p(mean), _p(invstd),
                              int(ctx.relu), _p(gx), C, _p(gg), _p(gb), _p(ws), wsb, _st()), "bn_bwd")
        return gx, gg, gb, None, None, None, None, None, None, None


def batch_norm(x, bn: torch.nn.BatchNorm1d, relu: bool):
    """Apply a torch.nn.BatchNorm1d module's parameters/buffers with the library kernels (+ fused ReLU)."""
    training = bn.training or bn.running_mean is None
    return _BatchNorm.apply(x, bn.weight, bn.bias, bn.running_mean, bn.running_var,
                            bn.num_batches_tracked if training else None, training, relu,
                            0.1 if bn.momentum is None else bn.momentum, bn.eps)


class _Relu(Function):
    @staticmethod
    def forward(ctx, x):
        _dev(x)
        x = _f32(x)
        y = torch.empty_like(x, memory_format=torch.contiguous_format)
        check(lib.pgnn_relu_fwd(_p(x), x.stride(0), x.shape[0], x.shape[1], _p(y), y.stride(0), _st()), "relu_fwd")
        ctx.save_for_backward(y)
        return y

    @staticmethod
    def backward(ctx, g):
        (y,) = ctx.saved_tensors
        g = _f32(g)
        gx = torch.empty_like(y)
        check(lib.pgnn_relu_bwd(_p(g), g.stride(0), _p(y), y.stride(0), y.shape[0], y.shape[1], _p(gx), gx.stride(0), _st()),
              "relu_bwd")
        return gx


def relu(x):
    return _Relu.apply(x)


class _Dropout(Function):
    @staticmethod
    def forward(ctx, x, p, seed, layer):
        _dev(x)
        x = _f32(x)
        if x.dim() != 2:
            raise PgnnError("dropout takes [N, C] activations")
        M, C = x.shape
        y = torch.empty(M, C, dtype=torch.float32, device=x.device)
        check(lib.pgnn_dropout_fwd(_p(x), x.stride(0), M, C, float(p), int(seed), int(layer), _p(y), C, _st()), "dropout_fwd")
        ctx.args = (float(p), int(seed), int(layer))
        return y

    @staticmethod
    def backward(ctx, g):
        g = _f32(g)
        M, C = g.shape
        gx = torch.empty(M, C, dtype=torch.float32, device=g.device)
        check(lib.pgnn_dropout_bwd(_p(g), g.stride(0), M, C, *ctx.args, _p(gx), C, _st()), "dropout_bwd")
        return gx, None, None, None


def dropout(x, p, seed, layer):
    """F.dropout(x, p, training=True) (chem/model.py:271-275, bio/model.py:283-286) with the library's defined draw: element (i, c)
    of `layer`'s [N, C] activation is kept iff splitmix64(seed, (layer << 40) | (i * C + c)) >> 32 >= floor(p * 2^32), and scaled by
    1 / (1 - p) (include/pgnn_b200.h, pgnn_dropout_fwd).  The backward regenerates the mask from (seed, layer)."""
    return _Dropout.apply(x, p, seed, layer)


def draw_seed():
    """One 62-bit dropout seed from torch's default CPU generator: a host operation (no device synchronisation), so
    torch.manual_seed(...) makes a training run's masks reproducible."""
    return int(torch.randint(0, 1 << 62, (), dtype=torch.int64))


class _L2Norm(Function):
    @staticmethod
    def forward(ctx, x):
        _dev(x)
        x = _f32(x)
        y = torch.empty_like(x, memory_format=torch.contiguous_format)
        nrm = torch.empty(x.shape[0], dtype=torch.float32, device=x.device)
        check(lib.pgnn_l2norm_fwd(_p(x), x.stride(0), x.shape[0], x.shape[1], _p(y), y.stride(0), _p(nrm), _st()), "l2norm_fwd")
        ctx.save_for_backward(y, nrm)
        return y

    @staticmethod
    def backward(ctx, g):
        y, nrm = ctx.saved_tensors
        g = _f32(g)
        gx = torch.empty_like(y)
        check(lib.pgnn_l2norm_bwd(_p(g), g.stride(0), _p(y), y.stride(0), _p(nrm), y.shape[0], y.shape[1], _p(gx),
                                  gx.stride(0), _st()), "l2norm_bwd")
        return gx


def l2_normalize(x):
    return _L2Norm.apply(x)


class _ChemEmbed(Function):
    @staticmethod
    def forward(ctx, x, t1, t2):
        _dev(x, t1, t2)
        if x.dtype != torch.int64 or x.dim() != 2 or x.shape[1] != 2:
            raise PgnnError("chem node features must be int64 [N, 2]")
        x, t1, t2 = x.contiguous(), _f32(t1).contiguous(), _f32(t2).contiguous()
        n, C = x.shape[0], t1.shape[1]
        out = torch.empty(n, C, dtype=torch.float32, device=x.device)
        check(lib.pgnn_chem_embed_fwd(_p(x), _p(t1), t1.shape[0], _p(t2), t2.shape[0], n, C, _p(out), C, _st()), "chem_embed_fwd")
        ctx.x, ctx.shapes = x, (t1.shape[0], t2.shape[0], C)
        if _VALIDATE:
            raise_on_device_errors()
        return out

    @staticmethod
    def backward(ctx, g):
        g = _f32(g)
        r1, r2, C = ctx.shapes
        g1 = torch.empty(r1, C, dtype=torch.float32, device=g.device)
        g2 = torch.empty(r2, C, dtype=torch.float32, device=g.device)
        check(lib.pgnn_chem_embed_bwd(_p(ctx.x), _p(g), g.stride(0), ctx.x.shape[0], C, _p(g1), r1, _p(g2), r2, _st()),
              "chem_embed_bwd")
        return None, g1, g2


def chem_embed(x, t1, t2):
    return _ChemEmbed.apply(x, t1, t2)


class _BioEmbed(Function):
    @staticmethod
    def forward(ctx, x, tab):
        _dev(x, tab)
        xv = x.reshape(-1)
        if xv.dtype != torch.float32:
            xv = xv.to(torch.float32)
        xv, tab = xv.contiguous(), _f32(tab).contiguous()
        n, C = xv.shape[0], tab.shape[1]
        out = torch.empty(n, C, dtype=torch.float32, device=tab.device)
        check(lib.pgnn_bio_embed_fwd(_p(xv), _p(tab), n, C, _p(out), C, _st()), "bio_embed_fwd")
        ctx.xv, ctx.C = xv, C
        return out

    @staticmethod
    def backward(ctx, g):
        g = _f32(g)
        gt = torch.empty(2, ctx.C, dtype=torch.float32, device=g.device)
        check(lib.pgnn_bio_embed_bwd(_p(ctx.xv), _p(g), g.stride(0), ctx.xv.shape[0], ctx.C, _p(gt), _st()), "bio_embed_bwd")
        return None, gt


def bio_embed(x, tab):
    return _BioEmbed.apply(x, tab)


class _SegmentMean(Function):
    @staticmethod
    def forward(ctx, x, segs):
        _dev(x)
        x = _f32(x)
        C = x.shape[1]
        out = torch.empty(segs.num_seg, C, dtype=torch.float32, device=x.device)
        check(lib.pgnn_segment_mean_fwd(_p(x), x.stride(0), _p(segs.ptr), _p(segs.order), segs.num_seg, C, _p(out), C, _st()),
              "segment_mean_fwd")
        ctx.segs, ctx.C = segs, C
        return out

    @staticmethod
    def backward(ctx, g):
        g = _f32(g)
        s = ctx.segs
        gx = torch.empty(s.n, ctx.C, dtype=torch.float32, device=g.device)
        check(lib.pgnn_segment_mean_bwd(_p(g), g.stride(0), _p(s.seg), _p(s.ptr), s.n, ctx.C, _p(gx), ctx.C, _st()),
              "segment_mean_bwd")
        return gx, None


def global_mean_pool(x, batch, size=None):
    """torch_geometric.nn.global_mean_pool replacement (chem/model.py:326): scatter_mean over `batch`."""
    if size is None:
        size = int(batch.max().item()) + 1 if batch.numel() else 0  # same D2H sync PyG 1.0.3 performs
    return _SegmentMean.apply(x, Segments(batch, size))


def segment_mean(x, segs: Segments):
    return _SegmentMean.apply(x, segs)


class _RowGather(Function):
    @staticmethod
    def forward(ctx, x, idx, idx2):
        _dev(x, idx, idx2)
        x = _f32(x)
        idx = idx.contiguous()
        idx2 = None if idx2 is None else idx2.contiguous()
        if idx.dtype != torch.int64 or (idx2 is not None and idx2.dtype != torch.int64):
            raise PgnnError("gather indices must be int64")
        m, C = idx.shape[0], x.shape[1]
        out = torch.empty(m, C, dtype=torch.float32, device=x.device)
        check(lib.pgnn_row_gather_fwd(_p(x), x.stride(0), x.shape[0], _p(idx), _p(idx2), m, C, _p(out), C, _st()), "row_gather_fwd")
        ctx.idx, ctx.idx2, ctx.shape = idx, idx2, tuple(x.shape)
        if _VALIDATE:
            raise_on_device_errors()
        return out

    @staticmethod
    def backward(ctx, g):
        g = _f32(g)
        n, C = ctx.shape
        gx = torch.zeros(n, C, dtype=torch.float32, device=g.device)
        check(lib.pgnn_row_gather_bwd(_p(g), g.stride(0), _p(ctx.idx), _p(ctx.idx2), ctx.idx.shape[0], C, _p(gx), C, n, _st()),
              "row_gather_bwd")
        return gx, None, None


def row_gather(x, idx, idx2=None):
    """x[idx] (+ x[idx2]): node_rep[masked_atom_indices], rep[u]+rep[v], node_rep[center_node_idx]."""
    return _RowGather.apply(x, idx, idx2)


class _ShiftedRowDot(Function):
    @staticmethod
    def forward(ctx, a, b, shift):
        _dev(a, b)
        a, b = _f32(a), _f32(b)
        B, C = a.shape
        out = torch.empty(B, dtype=torch.float32, device=a.device)
        check(lib.pgnn_shifted_rowdot_fwd(_p(a), a.stride(0), _p(b), b.stride(0), B, C, shift, _p(out), _st()),
              "shifted_rowdot_fwd")
        ctx.save_for_backward(a, b)
        ctx.shift = shift
        return out

    @staticmethod
    def backward(ctx, g):
        a, b = ctx.saved_tensors
        g = g.contiguous()
        B, C = a.shape
        ga, gb = torch.empty(B, C, dtype=torch.float32, device=g.device), torch.empty(B, C, dtype=torch.float32, device=g.device)
        check(lib.pgnn_shifted_rowdot_bwd(_p(g), _p(a), a.stride(0), _p(b), b.stride(0), B, C, ctx.shift, 0, _p(ga), C,
                                          _p(gb), C, _st()), "shifted_rowdot_bwd")
        return ga, gb, None


def shifted_rowdot(a, b, shift=0):
    """sum(a * b[cycle_index(B, shift)], dim=1) (chem/pretrain_contextpred.py:36-39,66-67); shift 0 = positives."""
    return _ShiftedRowDot.apply(a, b, int(shift))


class _BceLogits(Function):
    @staticmethod
    def forward(ctx, logits, target, kind, const):
        _dev(logits, target)
        x = _f32(logits)
        x2 = x.reshape(1, -1) if x.dim() == 1 else x
        if x2.stride(-1) != 1:
            x2 = x2.contiguous()
        M, N = x2.shape
        t = None
        if kind != 0:
            t = target.reshape(M, N).contiguous()
            if t.dtype != torch.int64:
                raise PgnnError("BCE targets must be int64 ({0,1}, or {-1,0,+1} for the masked form)")
        dev = x.device
        loss = torch.empty((), dtype=torch.float64, device=dev)
        dl = torch.empty(M, N, dtype=torch.float32, device=dev)
        wsb = lib.pgnn_bce_logits_workspace_bytes()
        ws = torch.empty(wsb, dtype=torch.uint8, device=dev)
        check(lib.pgnn_bce_logits_fwd(_p(x2), x2.stride(0) if M > 1 else max(N, 1), M, N, _p(t), N, int(kind), float(const), _p(loss),
                                      _p(dl), max(N, 1), _p(ws), wsb, _st()), "bce_logits_fwd")
        ctx.save_for_backward(dl)
        ctx.shape = tuple(logits.shape)
        return loss

    @staticmethod
    def backward(ctx, g):
        (dl,) = ctx.saved_tensors
        return (dl * g.to(torch.float32)).view(ctx.shape), None, None, None


def bce_with_logits(logits, target):
    """`nn.BCEWithLogitsLoss()(logits.double(), target.double())` (bio/pretrain_supervised.py:33-36): mean over all entries,
    evaluated in fp64; target int64 in {0,1}, same shape as logits.  Returns an fp64 scalar."""
    return _BceLogits.apply(logits, target, 1, 0.0)


def bce_with_logits_const(logits, target_value):
    """Same against a constant target (chem/pretrain_contextpred.py:86-87: ones for the positive, zeros for the negative scores)."""
    return _BceLogits.apply(logits, None, 0, float(target_value))


def masked_bce_with_logits(logits, y):
    """chem/finetune.py:33-43: y in {-1,0,+1}, entries with y == 0 carry no label; BCE on (y+1)/2 summed over the valid entries
    and divided by their number."""
    return _BceLogits.apply(logits, y, 2, 0.0)


class _Gat(Function):
    @staticmethod
    def forward(ctx, xl, att, T, bias, edge_attr, graph, heads, slope, is_bio):
        _dev(xl, att, T, bias, edge_attr)
        xl, att, T, bias = _f32(xl).contiguous(), _f32(att).contiguous(), _f32(T).contiguous(), _f32(bias).contiguous()
        ea = edge_attr.contiguous()
        want = torch.float32 if is_bio else torch.int64
        if ea.dtype != want or ea.shape != (graph.e, 9 if is_bio else 2):
            raise PgnnError("edge_attr has the wrong dtype/shape for %s GAT" % ("bio" if is_bio else "chem"))
        n, H = graph.n, int(heads)
        D = xl.shape[1] // H
        alpha = torch.empty(graph.e + n, H, dtype=torch.float32, device=xl.device)
        pq = torch.empty(n, H, 2, dtype=torch.float32, device=xl.device)
        out = torch.empty(n, D, dtype=torch.float32, device=xl.device)
        check(lib.pgnn_gat_fwd(_p(xl), n, H, D, _p(att), _p(T), int(is_bio), _p(ea), _p(graph.rowptr_t), _p(graph.nbr_t),
                               _p(graph.eid_t), graph.e, _p(bias), float(slope), _p(alpha), _p(pq), _p(out), D, _st()), "gat_fwd")
        ctx.save_for_backward(xl, att, T, alpha, pq, ea)
        ctx.graph, ctx.H, ctx.D, ctx.slope, ctx.is_bio, ctx.att_shape = graph, H, D, float(slope), bool(is_bio), att.shape
        return out

    @staticmethod
    def backward(ctx, g):
        xl, att, T, alpha, pq, ea = ctx.saved_tensors
        g = _f32(g)
        gr, n, H, D = ctx.graph, ctx.graph.n, ctx.H, ctx.D
        dev = g.device
        gxl = torch.empty(n, H * D, dtype=torch.float32, device=dev)
        gatt = torch.empty(H, 2 * D, dtype=torch.float32, device=dev)
        gT = torch.empty(T.shape[0], H * D, dtype=torch.float32, device=dev)
        gbias = torch.empty(D, dtype=torch.float32, device=dev)
        wsb = lib.pgnn_gat_bwd_workspace_bytes(n, gr.e, H, D)
        ws = torch.empty(wsb, dtype=torch.uint8, device=dev)
        check(lib.pgnn_gat_bwd(_p(g), g.stride(0), _p(xl), n, H, D, _p(att), _p(T), int(ctx.is_bio), _p(ea), _p(gr.rowptr_t),
                               _p(gr.nbr_t), _p(gr.eid_t), _p(gr.rowptr_s), _p(gr.nbr_s), _p(gr.eid_s), gr.e, ctx.slope, _p(alpha),
                               _p(pq), _p(gxl), _p(gatt), _p(gT), _p(gbias), _p(ws), wsb, _st()), "gat_bwd")
        return gxl, gatt.view(ctx.att_shape), gT, gbias, None, None, None, None, None


def gat(xl, att, T, edge_attr, graph, bias, heads=2, slope=0.2, is_bio=False):
    """GATConv.propagate + update (chem/model.py:148-165): xl = weight_linear(x) [N, heads*D]; att [1, heads, 2D]."""
    return _Gat.apply(xl, att, T, bias, edge_attr, graph, heads, slope, is_bio)


# ------------------------------------------------------------------------------------------------
# whole-encoder fast path: chem and bio GIN / GCN / GraphSAGE / GAT with dropout (pgnn_chem_encoder_*, pgnn_bio_encoder_*)
# ------------------------------------------------------------------------------------------------
import ctypes as _ct

CONV_TYPE = {"gcn": 1, "graphsage": 2, "gat": 3}


def _layer_params(gnn_type, conv):
    """One chem conv's parameters in the order of include/pgnn_b200.h (also the flat gradient order)."""
    if gnn_type == "gin":
        ps = [conv.mlp[0].weight, conv.mlp[0].bias, conv.mlp[2].weight, conv.mlp[2].bias]
    elif gnn_type == "gat":
        ps = [conv.weight_linear.weight, conv.weight_linear.bias, conv.att, conv.bias]
    else:
        ps = [conv.linear.weight, conv.linear.bias]
    return ps + [conv.edge_embedding1.weight, conv.edge_embedding2.weight]


def _bio_layer_params(gnn_type, conv):
    """One bio conv's parameters in the order of include/pgnn_b200.h (pgnn_bio_encoder_*)."""
    if gnn_type == "gin":
        ps = [conv.mlp[0].weight, conv.mlp[0].bias, conv.mlp[1].weight, conv.mlp[1].bias, conv.mlp[3].weight, conv.mlp[3].bias]
    elif gnn_type == "gat":
        ps = [conv.weight_linear.weight, conv.weight_linear.bias, conv.att, conv.bias]
    else:
        ps = [conv.linear.weight, conv.linear.bias]
    return ps + [conv.edge_encoder.weight, conv.edge_encoder.bias]


class _EncoderPlan:
    """Per-module bookkeeping of a whole-encoder GNN: parameter order, gradient layout, pointer tables, and the C calls.  The
    domain's subclass collects the parameters and BatchNorm modules, checks the inputs and makes the C calls; everything else is
    shared."""
    domain = None

    def _setup(self, gnn_type, L, D, params, bns, offsets):
        self.gnn_type = gnn_type
        self.conv = 0 if gnn_type == "gin" else CONV_TYPE[gnn_type]
        self.L, self.D = L, D
        self.params = params
        n = len(params)
        self.offsets = list(offsets)
        self.sizes = [self.offsets[i + 1] - self.offsets[i] for i in range(n)]
        self.shapes = [tuple(p.shape) for p in params]
        for p, s in zip(params, self.sizes):
            if p.numel() != s:
                raise PgnnError("parameter shape does not match the %s %s layout (emb_dim / heads / vocabulary sizes)" % (self.domain, gnn_type))
        self.total = self.offsets[-1]
        self.PtrArr = _ct.c_void_p * n
        self.BnArr = _ct.c_void_p * L
        self.bns = bns              # the BatchNorm1d modules whose state the encoder updates: one per layer, or none
        self._ws_alloc = 0          # workspace bytes requested from the allocator so far (see workspace_bytes)
        self.last_flat_grad = None  # the flat gradient buffer of the most recent backward (all-reduce target)
        # optional caller-owned destination ([total] fp32, e.g. a slice of NVLink-symmetric memory): used instead of a fresh
        # buffer whenever no parameter still holds a gradient (autograd would otherwise add a view of the buffer to itself)
        self.grad_buffer = None
        # forwards of this module that still await their backward.  The shared grad_buffer is handed out only when exactly
        # one is live: with two forwards in one autograd graph both backward nodes would see `p.grad is None` and the second
        # would overwrite the buffer whose views the engine still holds as the first node's gradients.  (A forward whose
        # graph is dropped without a backward leaves the count raised: the fresh-buffer path is then taken, which is safe.)
        self.live_forwards = 0
        self.direct_grads = True    # False: every gradient goes back through autograd (see _deliver_flat_grads)
        self._own_flat = None       # the plan's own flat gradient buffer when no grad_buffer is bound
        self._views = None          # (data_ptr, per-parameter views) of the last fast-path flat buffer
        self.keep_workspace = False  # GIN tests: keep the last training forward's workspace (chem_gin_relu_masks)
        self.last_ws = None

    def workspace_bytes(self, N, E):
        """Workspace size actually requested from the allocator: the largest need seen so far plus headroom, rounded to 16 MiB.
        Batches differ by a few percent in N and E; asking for exactly the need makes every new maximum a cudaMalloc
        (milliseconds, and a device synchronisation) in the middle of training, whereas one size per plan is served from the
        caching allocator's free list."""
        need = self._need(N, E)
        if need < 0:
            return need
        if need > self._ws_alloc:
            self._ws_alloc = ((need + need // 16) + (16 << 20) - 1) // (16 << 20) * (16 << 20)
        return self._ws_alloc

    def bn_pointers(self):
        """(running_mean, running_var, num_batches_tracked) host pointer tables of the L BatchNorms, or Nones without any."""
        if not self.bns:
            return None, None, None
        return tuple(self.BnArr(*[getattr(b, k).data_ptr() for b in self.bns]) for k in ("running_mean", "running_var", "num_batches_tracked"))

    def bn_constants(self):
        """(momentum, eps) the BatchNorms run with (torch's defaults for an encoder without BatchNorm)."""
        if not self.bns:
            return 0.1, 1e-5
        b = self.bns[0]
        return (b.momentum if b.momentum is not None else 0.1), b.eps


class ChemEncoderPlan(_EncoderPlan):
    """The chem GNN on pgnn_chem_encoder_* (type code 0 = GIN, else PGNN_CONV_*); GIN's layout queries are pgnn_chem_gin_*, the
    conv types' pgnn_chem_conv_*."""
    domain = "chem"

    def __init__(self, gnn, gnn_type):
        L, D = len(gnn.gnns), gnn.x_embedding1.weight.shape[1]
        ps = [gnn.x_embedding1.weight, gnn.x_embedding2.weight]
        for conv, bn in zip(gnn.gnns, gnn.batch_norms):
            ps += _layer_params(gnn_type, conv) + [bn.weight, bn.bias]
        n = len(ps)
        off = (_ct.c_int64 * (n + 1))()
        if gnn_type != "gin":
            assert n == lib.pgnn_chem_conv_num_params(CONV_TYPE[gnn_type], L)
            check(lib.pgnn_chem_conv_grad_offsets(CONV_TYPE[gnn_type], L, D, off), "chem_conv_grad_offsets")
        else:
            assert n == lib.pgnn_chem_gin_num_params(L)
            check(lib.pgnn_chem_gin_grad_offsets(L, D, off), "chem_gin_grad_offsets")
        self._setup(gnn_type, L, D, ps, list(gnn.batch_norms), off)

    def _need(self, N, E):
        if self.conv:
            return lib.pgnn_chem_conv_workspace_bytes(self.conv, N, E, self.L, self.D)
        return lib.pgnn_chem_gin_workspace_bytes(N, E, self.L, self.D)

    @staticmethod
    def inputs(x, edge_index, edge_attr):
        if x.dtype != torch.int64 or x.dim() != 2 or x.shape[1] != 2:
            raise PgnnError("chem node features must be int64 [N, 2]")
        if edge_index.dtype != torch.int64 or edge_index.dim() != 2 or edge_index.shape[0] != 2:
            raise PgnnError("edge_index must be int64 [2, E]")
        x, ei, ea = x.contiguous(), edge_index.contiguous(), edge_attr.contiguous()
        if ea.dtype != torch.int64 or tuple(ea.shape) != (ei.shape[1], 2):
            raise PgnnError("chem edge_attr must be int64 [E, 2]")
        return x, ei, ea

    def forward(self, ptrs, rm, rv, nbt, x, ei, ea, N, E, training, momentum, eps, drop_p, drop_seed, precision, out, ws, wsb):
        check(lib.pgnn_chem_encoder_forward(self.conv, ptrs, rm, rv, nbt, _p(x), _p(ei), _p(ea), N, E, self.L, self.D, int(training),
                                            float(momentum), float(eps), float(drop_p), int(drop_seed), precision, _p(out), self.D,
                                            _p(ws), wsb, _st()), "chem_encoder_forward")

    def backward(self, ptrs, g, x, ea, N, E, drop_p, drop_seed, precision, flat, ws, wsb):
        """`precision` must be the one the forward ran with: the backward reads what that forward saved in `ws` (the tensor path
        also the one-hot atom-code rows, which only a tf32x3 training forward writes)."""
        check(lib.pgnn_chem_encoder_backward(self.conv, ptrs, _p(g), g.stride(0), _p(x), _p(ea), N, E, self.L, self.D, float(drop_p),
                                             int(drop_seed), precision, _p(flat), _p(ws), wsb, _st()), "chem_encoder_backward")


class BioEncoderPlan(_EncoderPlan):
    """The bio GNN on pgnn_bio_encoder_* (type code 0 = GIN, else PGNN_CONV_*).  Only GIN has BatchNorm state: the inner
    BatchNorm1d(2D) of each layer's MLP."""
    domain = "bio"

    def __init__(self, gnn, gnn_type):
        L, D = len(gnn.gnns), gnn.gnns[0].input_node_embeddings.weight.shape[1]
        ps = [gnn.gnns[0].input_node_embeddings.weight]
        for conv in gnn.gnns:
            ps += _bio_layer_params(gnn_type, conv)
        code = 0 if gnn_type == "gin" else CONV_TYPE[gnn_type]
        n = len(ps)
        assert n == lib.pgnn_bio_encoder_num_params(code, L)
        off = (_ct.c_int64 * (n + 1))()
        check(lib.pgnn_bio_encoder_grad_offsets(code, L, D, off), "bio_encoder_grad_offsets")
        self._setup(gnn_type, L, D, ps, [conv.mlp[1] for conv in gnn.gnns] if gnn_type == "gin" else [], off)

    def _need(self, N, E):
        return lib.pgnn_bio_encoder_workspace_bytes(self.conv, N, E, self.L, self.D)

    @staticmethod
    def inputs(x, edge_index, edge_attr):
        """x: the dummy node label, [N] or [N, 1] (any dtype, taken as float32 as the layer-by-layer embedding does)."""
        if x.dim() not in (1, 2) or (x.dim() == 2 and x.shape[1] != 1):
            raise PgnnError("bio node labels must be [N] or [N, 1]")
        if edge_index.dtype != torch.int64 or edge_index.dim() != 2 or edge_index.shape[0] != 2:
            raise PgnnError("edge_index must be int64 [2, E]")
        x, ei, ea = x.reshape(-1).to(torch.float32).contiguous(), edge_index.contiguous(), edge_attr.contiguous()
        if ea.dtype != torch.float32 or tuple(ea.shape) != (ei.shape[1], 9):
            raise PgnnError("bio edge_attr must be float32 [E, 9]")
        return x, ei, ea

    def forward(self, ptrs, rm, rv, nbt, x, ei, ea, N, E, training, momentum, eps, drop_p, drop_seed, precision, out, ws, wsb):
        check(lib.pgnn_bio_encoder_forward(self.conv, ptrs, rm, rv, nbt, _p(x), _p(ei), _p(ea), N, E, self.L, self.D, int(training),
                                           float(momentum), float(eps), float(drop_p), int(drop_seed), precision, _p(out), self.D,
                                           _p(ws), wsb, _st()), "bio_encoder_forward")

    def backward(self, ptrs, g, x, ea, N, E, drop_p, drop_seed, precision, flat, ws, wsb):
        check(lib.pgnn_bio_encoder_backward(self.conv, ptrs, _p(g), g.stride(0), _p(x), _p(ea), N, E, self.L, self.D, float(drop_p),
                                            int(drop_seed), precision, _p(flat), _p(ws), wsb, _st()), "bio_encoder_backward")


def _deliver_flat_grads(plan, ctx, run):
    """Tail of the whole-encoder backward: pick the flat gradient buffer, run the C backward into it (`run(flat)`), and hand
    the per-parameter views to autograd.

    Fast path (the normal training step: one live forward, no parameter holds a gradient yet, every parameter is a leaf that
    wants one): the gradients land in a buffer that persists across steps (the caller's `plan.grad_buffer`, e.g. NVLink-symmetric
    memory, else one the plan owns) and each `p.grad` is set to its cached view directly; autograd gets None for the
    parameters.  That skips 40-odd AccumulateGrad nodes and as many split/view calls per step (~250 us of host time, more than
    the C side spends enqueueing the whole backward).  Hooks on the parameters / DDP are not supported on this path: set
    `plan.direct_grads = False` to have every gradient returned through autograd instead."""
    params = plan.params
    sole = plan.live_forwards == 1
    plan.live_forwards = max(plan.live_forwards - 1, 0)
    needs = ctx.needs_input_grad[_ENC_ARGS:]
    clean = sole and all(p.grad is None for p in params)
    if clean and plan.direct_grads and all(needs) and all(p.is_leaf for p in params):
        flat = plan.grad_buffer
        if flat is None:
            flat = plan._own_flat
            if flat is None or flat.device != ctx.x.device:
                flat = plan._own_flat = torch.empty(plan.total, dtype=torch.float32, device=ctx.x.device)
        cache = plan._views
        if cache is None or cache[0] != flat.data_ptr():
            cache = plan._views = (flat.data_ptr(), [v.view(s) for v, s in zip(flat.split(plan.sizes), plan.shapes)])
        run(flat)
        plan.last_flat_grad = flat
        for p, v in zip(params, cache[1]):
            p.grad = v
        return (None,) * (_ENC_ARGS + len(params))
    if plan.grad_buffer is not None and clean:
        flat = plan.grad_buffer
    else:
        flat = torch.empty(plan.total, dtype=torch.float32, device=ctx.x.device)
    run(flat)
    plan.last_flat_grad = flat
    grads = [v.view(s) for v, s in zip(flat.split(plan.sizes), plan.shapes)]
    return (None,) * _ENC_ARGS + tuple(gr if need else None for gr, need in zip(grads, needs))


def _release_ctx(ctx):
    """Drop the encoder node's references to its ~200 MB workspace and inputs once the backward has been enqueued.  They are plain
    ctx attributes (not save_for_backward tensors), so autograd does not free them with the graph's buffers: as long as the caller
    keeps the loss tensor (e.g. to log it after the NEXT step has started), loss.grad_fn keeps this node and the node kept the
    workspace, the next forward then needed a second one, and that cudaMalloc (40 ms, device-synchronising) was the stall seen at
    step 1 of every end-to-end loop.  A second backward through the same graph is not supported by this op anyway."""
    ctx.ws = ctx.keep = ctx.ptrs = ctx.x = ctx.ea = None
    ctx.released = True


_ENC_ARGS = 7  # _Encoder.forward's arguments in front of the parameters


class _Encoder(Function):
    """The whole encoder of either domain as one autograd node; the plan (ChemEncoderPlan / BioEncoderPlan) checks the inputs and
    makes the two C calls."""

    @staticmethod
    def forward(ctx, plan, x, edge_index, edge_attr, training, drop_p, drop_seed, *params):
        _dev(x, edge_index, edge_attr, *params)
        x, ei, ea = plan.inputs(x, edge_index, edge_attr)
        N, E, D = x.shape[0], ei.shape[1], plan.D
        for p in params:
            if p.dtype != torch.float32 or not p.is_contiguous():
                raise PgnnError("the fused encoder needs contiguous fp32 parameters")
        if training and N == 0 and plan.bns:
            raise PgnnError("BatchNorm in training mode needs at least one node")
        dev = x.device
        ptrs = plan.PtrArr(*[p.data_ptr() for p in params])
        rm, rv, nbt = plan.bn_pointers()
        wsb = plan.workspace_bytes(N, E)
        ws = torch.empty(wsb, dtype=torch.uint8, device=dev)
        out = torch.empty(N, D, dtype=torch.float32, device=dev)
        mom, eps = plan.bn_constants()
        precision = _precision
        plan.forward(ptrs, rm, rv, nbt, x, ei, ea, N, E, training, mom, eps, drop_p, drop_seed, precision, out, ws, wsb)
        ctx.plan, ctx.ws, ctx.wsb, ctx.ptrs, ctx.x, ctx.ea, ctx.dims, ctx.training = plan, ws, wsb, ptrs, x, ea, (N, E), training
        ctx.drop = (drop_p, drop_seed)  # the backward regenerates the masks from these
        ctx.precision = precision       # and reads the workspace this precision's forward wrote, whatever set_precision says by then
        ctx.keep = params  # the pointer table refers to these storages
        if training and plan.keep_workspace:
            plan.last_ws = (ws, (N, E, plan.L, D))
        if training and any(ctx.needs_input_grad[_ENC_ARGS:]):
            plan.live_forwards += 1
        if _VALIDATE:
            raise_on_device_errors()
        return out

    @staticmethod
    def backward(ctx, g):
        if not ctx.training:
            raise PgnnError("backward through the eval-mode encoder is not implemented (SURVEY.md section 3.3)")
        if getattr(ctx, "released", False):
            raise PgnnError("the whole-encoder op released its workspace after its first backward: a second backward through the same "
                            "graph (retain_graph) is not supported; set model.fused = False for that")
        plan = ctx.plan
        N, E = ctx.dims
        g = _f32(g)
        out = _deliver_flat_grads(plan, ctx, lambda flat: plan.backward(ctx.ptrs, g, ctx.x, ctx.ea, N, E, *ctx.drop, ctx.precision, flat,
                                                                          ctx.ws, ctx.wsb))
        _release_ctx(ctx)
        return out


def chem_encoder(plan: ChemEncoderPlan, x, edge_index, edge_attr, training: bool, drop_p: float = 0.0, drop_seed: int = 0):
    """The whole chem encoder in one call per pass.  With training and drop_p > 0, layer l's output carries the ops.dropout mask
    of (drop_p, drop_seed, l): the same mask the layer-by-layer composition applies under the same seed."""
    return _Encoder.apply(plan, x, edge_index, edge_attr, training, float(drop_p), int(drop_seed), *plan.params)


def bio_encoder(plan: BioEncoderPlan, x, edge_index, edge_attr, training: bool, drop_p: float = 0.0, drop_seed: int = 0):
    """The whole bio encoder in one call per pass, with the dropout masks of chem_encoder."""
    return _Encoder.apply(plan, x, edge_index, edge_attr, training, float(drop_p), int(drop_seed), *plan.params)


def chem_gin_relu_masks(plan: ChemEncoderPlan, gnn):
    """The ReLU decisions of the last training forward of the fused GIN encoder (plan.keep_workspace = True), in the order the
    reference takes them: per layer the MLP's hidden units [N, 2D], then (all but the last layer) the post-BatchNorm units [N, D]."""
    if plan.gnn_type != "gin" or plan.domain != "chem":
        raise PgnnError("chem_gin_relu_masks reads the GIN workspace layout (pgnn_chem_gin_debug_layout)")
    ws, (N, E, L, D) = plan.last_ws
    off = (_ct.c_int64 * 4)()
    check(lib.pgnn_chem_gin_debug_layout(N, E, L, D, off), "chem_gin_debug_layout")
    f = lambda o, n: ws[o:o + 4 * n].view(torch.float32)
    z1 = f(off[0], L * N * 2 * D).view(L, N, 2 * D)
    z2 = f(off[1], L * N * D).view(L, N, D)
    mean, invstd = f(off[2], L * D).view(L, D), f(off[3], L * D).view(L, D)
    masks = []
    for l in range(L):
        masks.append(z1[l] > 0)
        if l != L - 1:
            bn = gnn.batch_norms[l]
            # the one BatchNorm pre-activation the forward's gather applied and the backward recomputes (common.cuh bn_preact):
            # fmaf(z2, scale, shift) with scale = gamma * invstd, shift = fmaf(-mean, scale, beta).  Its sign is that of the exact
            # z2 * scale + shift, which fp64 gives exactly (the product of two floats is exact there).
            scale = bn.weight.detach() * invstd[l]
            shift = fma32(-mean[l], scale, bn.bias.detach())
            masks.append(z2[l].double() * scale.double() + shift.double() > 0)
    return masks


def fma32(a, b, c):
    """fp32 fmaf(a, b, c) of fp32 tensors, bit for bit (one rounding of the exact a * b + c).  The product is exact in fp64; the
    fp64 sum s is rounded once more to fp32, which is the correctly rounded result unless s lands exactly halfway between two
    floats, where the sign of the fp64 sum's own rounding error (TwoSum) decides."""
    p, cd = a.double() * b.double(), c.double()
    s = p + cd
    bb = s - p
    err = (p - (s - bb)) + (cd - bb)
    f = s.float()
    toward = torch.where(s > f.double(), torch.full_like(f, float("inf")), torch.full_like(f, float("-inf")))
    nb = torch.nextafter(f, toward)
    tie = (s != f.double()) & ((s - f.double()) * 2 == nb.double() - f.double())
    past = tie & (err != 0) & ((err > 0) == (s > f.double()))
    return torch.where(past, nb, f)


# ------------------------------------------------------------------------------------------------
# masking head: node_rep[idx] -> Linear -> mean cross-entropy in fp64 (chem/pretrain_masking.py:51-52) as one op
# ------------------------------------------------------------------------------------------------
def _pad4(n):
    return (n + 3) // 4 * 4


class _MaskedCE(Function):
    @staticmethod
    def forward(ctx, node_rep, idx, labels, weight, bias, idx2=None):
        _dev(node_rep, idx, labels, weight, bias, idx2)
        rep, w = _f32(node_rep), _f32(weight).contiguous()
        idx, labels = idx.contiguous(), labels.contiguous()
        idx2 = None if idx2 is None else idx2.contiguous()
        label_rows = labels.dim() == 2   # [M, Q] floats whose argmax is the class (bio masking), else int64 [M] classes
        if label_rows and (labels.dtype != torch.float32 or labels.shape[0] != idx.shape[0]):
            raise PgnnError("label rows must be fp32 [M, Q] with one row per gathered row")
        if idx.dtype != torch.int64 or not (label_rows or labels.dtype == torch.int64) or (idx2 is not None and idx2.dtype != torch.int64):
            raise PgnnError("indices and labels must be int64")
        M, D, V = idx.shape[0], rep.shape[1], w.shape[0]
        ldv = _pad4(V)  # 16-byte aligned logit rows (the tensor path's vector loads); the GEMM loaders never read past column V
        dev = rep.device
        rows = torch.empty(M, D, dtype=torch.float32, device=dev)
        check(lib.pgnn_row_gather_fwd(_p(rep), rep.stride(0), rep.shape[0], _p(idx), _p(idx2), M, D, _p(rows), D, _st()), "row_gather_fwd")
        logits = torch.empty(M, ldv, dtype=torch.float32, device=dev)
        check(lib.pgnn_linear_fwd(_p(rows), D, _p(w), _p(bias), M, V, D, 0, _p(logits), ldv, _precision, _st()), "linear_fwd")
        loss = torch.empty((), dtype=torch.float64, device=dev)
        dlogits = torch.empty(M, ldv, dtype=torch.float32, device=dev)
        if label_rows:
            wsb = int(lib.pgnn_softmax_ce_rows_workspace_bytes())
            ws = torch.empty(wsb, dtype=torch.uint8, device=dev)
            check(lib.pgnn_softmax_ce_rows_fwd(_p(logits), ldv, M, V, _p(labels), labels.stride(0), labels.shape[1], _p(loss), _p(dlogits), ldv,
                                               _p(ws), wsb, _st()), "softmax_ce_rows_fwd")
        else:
            check(lib.pgnn_softmax_ce_fwd(_p(logits), ldv, M, V, _p(labels), _p(loss), _p(dlogits), ldv, _st()), "softmax_ce_fwd")
        ctx.save_for_backward(rows, dlogits, w, idx)
        ctx.idx2 = idx2
        ctx.dims = (tuple(rep.shape), M, D, V, ldv, bias is not None)
        ctx.logits = logits[:, :V]
        ctx.mark_non_differentiable(ctx.logits)
        if _VALIDATE:
            raise_on_device_errors()
        return loss, ctx.logits

    @staticmethod
    def backward(ctx, g, _g_logits):
        rows, dlogits, w, idx = ctx.saved_tensors
        (n, D_), M, D, V, ldv, has_bias = ctx.dims
        dev = rows.device
        dl = dlogits * g.to(torch.float32)  # d loss / d logits scaled by the incoming gradient (a scalar, normally 1)
        gw = torch.empty(V, D, dtype=torch.float32, device=dev)
        gb = torch.empty(V, dtype=torch.float32, device=dev) if has_bias else None
        check(lib.pgnn_linear_bwd_w(_p(dl), ldv, _p(rows), D, M, V, D, _p(gw), _p(gb), _precision, _st()), "linear_bwd_w")
        grep = None
        if ctx.needs_input_grad[0]:
            drows = torch.empty(M, D, dtype=torch.float32, device=dev)
            check(lib.pgnn_linear_bwd_x(_p(dl), ldv, _p(w), M, V, D, None, 0, _p(drows), D, _precision, _st()), "linear_bwd_x")
            grep = torch.zeros(n, D, dtype=torch.float32, device=dev)
            check(lib.pgnn_row_gather_bwd(_p(drows), D, _p(idx), _p(ctx.idx2), M, D, _p(grep), D, n, _st()), "row_gather_bwd")
        return grep, None, None, gw, gb, None


def masked_atom_loss(node_rep, masked_atom_indices, labels, weight, bias=None):
    """`criterion(linear(node_rep[masked_atom_indices]).double(), labels)` of chem/pretrain_masking.py:51-52 with
    nn.CrossEntropyLoss (mean): gather, Linear(emb_dim, V), softmax cross-entropy evaluated in fp64.
    Returns (loss: fp64 scalar tensor, logits: [M, V] fp32, non-differentiable — e.g. for compute_accuracy)."""
    return _MaskedCE.apply(node_rep, masked_atom_indices, labels, weight, bias)


def masked_bond_loss(node_rep, edge_index, connected_edge_indices, labels, weight, bias=None):
    """chem/pretrain_masking.py:57-61: `edge_rep = node_rep[u] + node_rep[v]` for the masked bonds
    `edge_index[:, connected_edge_indices]`, `Linear(emb_dim, 4)`, mean CE on fp64 logits.  -> (loss fp64, logits [M, 4])."""
    me = edge_index.index_select(1, connected_edge_indices)
    return _MaskedCE.apply(node_rep, me[0], labels, weight, bias, me[1])


def masked_edge_type_loss(node_rep, edge_index, masked_edge_idx, mask_edge_label, weight, bias=None):
    """bio/pretrain_masking.py:47-55: `edge_rep = node_rep[u] + node_rep[v]` for the masked edges `edge_index[:, masked_edge_idx]`,
    `Linear(emb_dim, 7)`, and CrossEntropyLoss (mean) against `torch.argmax(mask_edge_label, dim=1)`: the label of a row is the
    first index of the maximum of its 9 label floats.  The script evaluates the loss in fp32; it is evaluated in fp64 here.
    A label past the V classes (the maximum in column 7 or 8) raises PGNN_DEVERR_LABEL.  -> (loss fp64, logits [M, V])."""
    me = edge_index.index_select(1, masked_edge_idx)
    return _MaskedCE.apply(node_rep, me[0], mask_edge_label, weight, bias, me[1])


# ------------------------------------------------------------------------------------------------
# edge-prediction head: pair dot products + BCE of both sides (chem/pretrain_edgepred.py:31-41) as one op
# ------------------------------------------------------------------------------------------------
def _pair_rows(index, name):
    if index.dtype != torch.int64 or index.dim() != 2 or index.shape[0] != 2:
        raise PgnnError("%s must be int64 [2, n]" % name)
    m = int(index.shape[1])
    if m == 0:
        return None, None, 1, 0
    return index[0].data_ptr(), index[1].data_ptr(), index.stride(1), m


class _EdgePairBce(Function):
    @staticmethod
    def forward(ctx, node_rep, pos_index, neg_index):
        _dev(node_rep, pos_index, neg_index)
        x = _f32(node_rep)
        if x.data_ptr() % 16 or x.stride(0) % 4:
            x = x.contiguous()
        N, C = x.shape
        pu, pv, ps, P = _pair_rows(pos_index, "pos_index")
        qu, qv, qs, Q = _pair_rows(neg_index, "neg_index")
        dev = x.device
        loss = torch.empty((), dtype=torch.float64, device=dev)
        pos = torch.empty(P, dtype=torch.float32, device=dev)
        neg = torch.empty(Q, dtype=torch.float32, device=dev)
        dscore = torch.empty(P + Q, dtype=torch.float32, device=dev)
        pairs = torch.empty(2, P + Q, dtype=torch.int64, device=dev)
        wsb = int(lib.pgnn_edge_pair_bce_workspace_bytes())
        ws = torch.empty(wsb, dtype=torch.uint8, device=dev)
        check(lib.pgnn_edge_pair_bce_fwd(_p(x), x.stride(0), N, C, pu, pv, ps, P, qu, qv, qs, Q, _p(loss), _p(pos), _p(neg), _p(dscore),
                                         _p(pairs), _p(ws), wsb, _st()), "edge_pair_bce_fwd")
        ctx.graph = Graph(pairs, N) if ctx.needs_input_grad[0] else None   # both bucketings of the P + Q pairs, for the backward
        ctx.save_for_backward(x, dscore)
        ctx.mark_non_differentiable(pos, neg)
        if _VALIDATE:
            raise_on_device_errors()
        return loss, pos, neg

    @staticmethod
    def backward(ctx, g, _g_pos, _g_neg):
        x, dscore = ctx.saved_tensors
        graph = ctx.graph
        N, C = x.shape
        g = g.to(torch.float64).contiguous()
        gx = torch.empty(N, C, dtype=torch.float32, device=x.device)
        check(lib.pgnn_edge_pair_bce_bwd(_p(x), x.stride(0), N, C, _p(dscore), _p(g), _p(graph.rowptr_t), _p(graph.nbr_t), _p(graph.eid_t),
                                         _p(graph.rowptr_s), _p(graph.nbr_s), _p(graph.eid_s), _p(gx), C, _st()), "edge_pair_bce_bwd")
        return gx, None, None


def edge_pair_bce(node_rep, pos_index, neg_index):
    """chem/pretrain_edgepred.py:35-39 (bio/pretrain_edgepred.py alike): pos = sum(node_rep[pos_index[0]] * node_rep[pos_index[1]], 1),
    neg likewise over neg_index, loss = BCEWithLogits(pos, 1) + BCEWithLogits(neg, 0), each a mean over its own scores and
    evaluated in fp64 (the script: fp32).  pos_index may be the strided view edge_index[:, ::2] (read in place).  An empty side
    makes the loss NaN, as torch's mean over nothing does.  -> (loss fp64, pos [P] fp32, neg [Q] fp32; the scores are
    non-differentiable, e.g. for the script's train_acc)."""
    return _EdgePairBce.apply(node_rep, pos_index, neg_index)


# ------------------------------------------------------------------------------------------------
# Deep Graph Infomax head: summary, discriminator scores and both BCE terms (chem/pretrain_deepgraphinfomax.py:61-73) as one op
# ------------------------------------------------------------------------------------------------
class _InfomaxBce(Function):
    @staticmethod
    def forward(ctx, node_emb, weight, segs):
        _dev(node_emb, weight)
        x = _f32(node_emb)
        if x.data_ptr() % 16 or x.stride(0) % 4:
            x = x.contiguous()
        w = _f32(weight).contiguous()
        N, C = x.shape
        G = segs.num_seg
        if tuple(w.shape) != (C, C):
            raise PgnnError("weight must be [%d, %d], got %s" % (C, C, tuple(w.shape)))
        if segs.n != N:
            raise PgnnError("batch has %d entries for %d node rows" % (segs.n, N))
        dev = x.device
        S = torch.empty(G, C, dtype=torch.float32, device=dev)
        check(lib.pgnn_infomax_summary_fwd(_p(x), x.stride(0), _p(segs.ptr), _p(segs.order), G, C, _p(S), C, _st()), "infomax_summary_fwd")
        H = torch.empty(G, C, dtype=torch.float32, device=dev)
        check(lib.pgnn_linear_bwd_x(_p(S), C, _p(w), G, C, C, None, 0, _p(H), C, _precision, _st()), "linear_bwd_x")   # H = S . W
        loss = torch.empty((), dtype=torch.float64, device=dev)
        pos = torch.empty(N, dtype=torch.float32, device=dev)
        neg = torch.empty(N, dtype=torch.float32, device=dev)
        dscore = torch.empty(2 * N, dtype=torch.float32, device=dev)
        wsb = int(lib.pgnn_infomax_bce_workspace_bytes())
        ws = torch.empty(wsb, dtype=torch.uint8, device=dev)
        check(lib.pgnn_infomax_bce_fwd(_p(x), x.stride(0), N, C, _p(segs.seg), _p(H), G, _p(loss), _p(pos), _p(neg), _p(dscore), _p(ws), wsb,
                                       _st()), "infomax_bce_fwd")
        ctx.segs = segs
        ctx.save_for_backward(x, w, S, H, dscore)
        ctx.mark_non_differentiable(pos, neg)
        if _VALIDATE:
            raise_on_device_errors()
        return loss, pos, neg

    @staticmethod
    def backward(ctx, g, _g_pos, _g_neg):
        x, w, S, H, dscore = ctx.saved_tensors
        segs = ctx.segs
        N, C = x.shape
        G = segs.num_seg
        g = g.to(torch.float64).contiguous()
        gx = torch.empty(N, C, dtype=torch.float32, device=x.device) if ctx.needs_input_grad[0] else None
        gw = torch.empty(C, C, dtype=torch.float32, device=x.device) if ctx.needs_input_grad[1] else None
        wsb = int(lib.pgnn_infomax_bce_bwd_workspace_bytes(G, C))
        ws = torch.empty(wsb, dtype=torch.uint8, device=x.device)
        check(lib.pgnn_infomax_bce_bwd(_p(x), x.stride(0), N, C, _p(segs.seg), _p(segs.ptr), _p(segs.order), G, _p(S), _p(H), _p(w), _p(dscore),
                                       _p(g), _p(gx), C, _p(gw), _precision, _p(ws), wsb, _st()), "infomax_bce_bwd")
        return gx, gw, None


def infomax_bce(node_emb, batch, weight, num_graphs=None):
    """chem/pretrain_deepgraphinfomax.py:61-73 (bio/pretrain_deepgraphinfomax.py alike) after the encoder:
    summary = sigmoid(global_mean_pool(node_emb, batch)); pos_i = <node_emb_i, (summary @ weight)[batch_i]>, neg_i likewise against
    the next graph's summary (cycle_index(G, 1)); loss = BCEWithLogits(pos, 1) + BCEWithLogits(neg, 0), each a mean over the N
    nodes, evaluated in fp64 (the script: fp32).  `batch` is any vector global_mean_pool accepts (sorted or not); num_graphs=None
    means batch.max() + 1, read back to the host as PyG 1.0.3 does.  Differentiable in node_emb and weight [D, D].  N = 0 makes
    the loss NaN, as torch's mean over nothing does.  -> (loss fp64, pos [N] fp32, neg [N] fp32; the scores are
    non-differentiable, e.g. for the script's train_acc)."""
    if num_graphs is None:
        num_graphs = int(batch.max().item()) + 1 if batch.numel() else 0  # same D2H sync PyG 1.0.3 performs
    return _InfomaxBce.apply(node_emb, weight, Segments(batch, num_graphs))
