"""Data-parallel plumbing: shard graphs across ranks, one all-reduce of a flat fp32 gradient buffer per step.

The reference has no parallelism at all (SURVEY.md section 2.2); graphs in a batch are independent, so the
path shards by graph with no activation exchange and the only collective is the gradient all-reduce
(section 8(e)).  Each rank's BatchNorm statistics are local (like DDP without SyncBN).

Two transports for that all-reduce:
  * "p2p"  -- this library's own kernels over NVLink peer memory (csrc/collective.cu): the gradients are written by the
              backward pass straight into a symmetric allocation, reduce-scattered with peer loads and all-gathered with
              peer stores, three flag barriers, bit-identical on every rank.  torch.distributed's symmetric-memory
              allocator is used for what it is: allocation and the exchange of peer addresses.
  * "nccl" -- torch.distributed.all_reduce (NCCL on GPUs, gloo in the CPU tests), with the head's small buffer launched
              from a gradient hook so that it overlaps the encoder's backward.
"""
from __future__ import annotations

import sys

import torch
import torch.distributed as dist


def shard_graphs(num_graphs: int, rank: int, world: int):
    """Contiguous slice [lo, hi) of a global batch's graphs owned by `rank` (sizes differ by at most one)."""
    base, rem = divmod(num_graphs, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def _flat_is_live(flat, params):
    """True when every parameter's .grad is the contiguous view of `flat` at its running offset, i.e. all-reducing `flat`
    in place all-reduces the gradients.  False e.g. after autograd ACCUMULATED a new backward into older gradient tensors."""
    if flat is None:
        return False
    at = flat.data_ptr()
    for p in params:
        g = p.grad
        if g is None or g.data_ptr() != at or not g.is_contiguous():
            return False
        at += 4 * p.numel()
    return True


def _pack(views, params):
    torch._foreach_copy_(views, [p.grad if p.grad is not None else torch.zeros_like(p) for p in params])


def _unpack(views, params):
    for p, v in zip(params, views):
        if p.grad is None:
            p.grad = v.clone()
    torch._foreach_copy_([p.grad for p in params], views)


class P2PAllReduce:
    """Symmetric fp32 buffers of `numel` elements plus the flag words of the library's NVLink all-reduces.

    mode (argument, else PGNN_ALLREDUCE, else "p2p"; measured at 2 GPUs on the masking step, 50 steps, max over ranks: p2p 415 k graphs/s,
    fused 357 k, nvls 346 k -- the one-kernel variants have the better median step (1.183 / 1.192 vs 1.196 ms on rank 0) but one rank
    carries ~12 ms more inside its timed steps, not yet explained; bench.py now reports every rank's figures):
      "fused"   one kernel, out of place (`pgnn_allreduce_fused`): gradients are written into `buf`, the mean lands in `out`
      "nvls"    the same kernel with the NVSwitch doing the sum (multimem.ld_reduce / multimem.st on the multicast mappings);
                falls back to "fused" when the allocation has no multicast mapping
      "p2p"     round 1's five-launch two-shot exchange, in place (`pgnn_allreduce_p2p`): `out` is `buf`
    `run()` returns the buffer that holds the result."""

    FLAG_FLOATS = 128  # 512 bytes in front of the data (keeps it 16-byte aligned): words [0,32) p2p, [32,64) old nvls, [64,128) fused

    def __init__(self, numel, device, group=None, mode=None):
        import os
        import torch.distributed._symmetric_memory as symm
        from ._cabi import lib
        group = group if group is not None else dist.group.WORLD
        self.rank, self.world, self.numel = dist.get_rank(group), dist.get_world_size(group), int(numel)
        mode = mode or os.environ.get("PGNN_ALLREDUCE", "") or "p2p"
        if mode not in ("fused", "nvls", "p2p"):
            raise ValueError("PGNN_ALLREDUCE must be fused, nvls or p2p")
        quantum = 4 * self.world
        self.padded = (self.numel + quantum - 1) // quantum * quantum  # whole float4s per rank (the multimem path needs them)
        two = mode != "p2p"
        self.sym = symm.empty(self.FLAG_FLOATS + (2 if two else 1) * self.padded, dtype=torch.float32, device=device)
        self.sym.zero_()
        hdl = symm.rendezvous(self.sym, group)
        ptrs = [int(p) for p in hdl.buffer_ptrs]
        self._hdl = hdl
        F = self.FLAG_FLOATS
        self.buf = self.sym[F:F + self.numel]
        self.out = self.sym[F + self.padded:F + self.padded + self.numel] if two else self.buf
        self.flag_ptrs = torch.tensor(ptrs, dtype=torch.int64, device=device)
        self.buf_ptrs = torch.tensor([p + 4 * F for p in ptrs], dtype=torch.int64, device=device)
        self.out_ptrs = torch.tensor([p + 4 * (F + self.padded) for p in ptrs], dtype=torch.int64, device=device)
        nscratch = lib.pgnn_allreduce_p2p_scratch_floats(self.numel, self.world)
        self.scratch = torch.empty(max(int(nscratch), 4), dtype=torch.float32, device=device)
        self.counter = torch.zeros(4, dtype=torch.int32, device=device)
        self.epoch = 0
        self.mc_in = self.mc_out = 0
        if mode == "nvls":
            mc = 0
            try:
                mc = int(getattr(hdl, "multicast_ptr", 0) or 0)
            except Exception:
                mc = 0
            if mc and self.world <= 32:
                self.mc_in, self.mc_out = mc + 4 * F, mc + 4 * (F + self.padded)
            else:
                mode = "fused"
        self.transport = mode
        torch.cuda.synchronize(device)
        dist.barrier(group)  # every rank's zeroed flag words are in place before anyone signals

    def run(self, scale=1.0):
        from ._cabi import check, lib
        st = torch.cuda.current_stream(self.sym.device).cuda_stream
        if self.transport == "p2p":
            check(lib.pgnn_allreduce_p2p(self.buf_ptrs.data_ptr(), self.flag_ptrs.data_ptr(), self.rank, self.world, self.numel,
                                         float(scale), self.scratch.data_ptr(), self.scratch.numel(), self.epoch, st),
                  "pgnn_allreduce_p2p")
        else:
            n = self.padded if self.mc_in else self.numel
            check(lib.pgnn_allreduce_fused(self.buf_ptrs.data_ptr(), self.out_ptrs.data_ptr(), self.flag_ptrs.data_ptr(),
                                           self.mc_in or None, self.mc_out or None, self.counter.data_ptr(), self.rank, self.world, n,
                                           float(scale), self.epoch, st), "pgnn_allreduce_fused")
        self.epoch += 1
        return self.out


class GradAllReducer:
    """One all-reduce of every gradient per step.

    `flat_sources`: callables returning (flat_tensor, [params it covers]) for modules whose backward already leaves its
    gradients in ONE flat fp32 buffer (the fused encoder: every `p.grad` is a view of it).  The remaining parameters
    (heads) are packed into a small buffer.

    backend "p2p": one symmetric buffer holds [flat sources | packed rest]; flat sources that can be bound
    (`src.bind(buffer)`) write their gradients straight into it, so the step is: backward -> copy the head's two tensors in
    -> `pgnn_allreduce_p2p` -> copy them out.  backend "nccl": the flat buffers are all-reduced in place by
    torch.distributed; with `overlap=True` the packed buffer's all-reduce is launched from a gradient hook as soon as the
    last of its parameters has a gradient, i.e. under the encoder's backward (one backward per all_reduce_mean call).
    backend "auto": p2p on CUDA when the symmetric-memory rendezvous works, else nccl (reported on stderr).

    `scale=False` leaves the SUM in place (pass `grad_scale=1/world` to `optim.Adam` instead)."""

    def __init__(self, params, flat_sources=(), group=None, overlap=True, scale=True, backend="auto"):
        self.group, self.scale = group, scale
        self.flat_sources = list(flat_sources)
        covered = set()
        for src in self.flat_sources:
            covered.update(id(p) for p in src()[1])
        self.params = [p for p in params if p.requires_grad and id(p) not in covered]
        self.sizes = [p.numel() for p in self.params]
        self.flat, self._pending, self._seen, self._hooks, self.p2p = None, None, 0, [], None
        all_params = self.params + [p for src in self.flat_sources for p in src()[1]]
        on_cuda = bool(all_params) and all(p.is_cuda for p in all_params)
        if backend not in ("auto", "p2p", "nccl"):
            raise ValueError("backend must be 'auto', 'p2p' or 'nccl'")
        if backend == "p2p" and not on_cuda:
            raise ValueError("the p2p all-reduce needs CUDA parameters")
        self.backend = "nccl"
        if backend != "nccl" and on_cuda and dist.get_world_size(group) > 1:
            try:
                self._setup_p2p(all_params[0].device)
                self.backend = self.p2p.transport  # "p2p" (default), "fused" or "nvls"
            except Exception as e:  # no peer access / symmetric memory unavailable on this box
                if backend == "p2p":
                    raise
                print("[pretrain_gnns_b200.dist] p2p all-reduce unavailable (%s: %s); using torch.distributed" % (type(e).__name__, e),
                      file=sys.stderr, flush=True)
                self.p2p = None
        if self.backend == "nccl" and self.params:
            self.flat = torch.zeros(sum(self.sizes), dtype=torch.float32, device=self.params[0].device)
            self.views = [v.view_as(p) for v, p in zip(self.flat.split(self.sizes), self.params)]
            if overlap:
                for p in self.params:
                    self._hooks.append(p.register_post_accumulate_grad_hook(self._on_grad))

    # ---- p2p transport ----------------------------------------------------------------------------------------------
    def _setup_p2p(self, device):
        src_sizes = [sum(p.numel() for p in src()[1]) for src in self.flat_sources]
        pad4 = lambda n: (n + 3) // 4 * 4  # every region starts 16-byte aligned
        offs, tot = [], 0
        for n in src_sizes + [sum(self.sizes)]:
            offs.append(tot)
            tot += pad4(n)
        self.p2p = P2PAllReduce(tot, device, self.group)
        inb, outb = self.p2p.buf, self.p2p.out
        self.in_place = outb.data_ptr() == inb.data_ptr()
        split = lambda buf, src: [v.view_as(p) for v, p in zip(buf.split([p.numel() for p in src()[1]]), src()[1])]
        self.regions = [inb[o:o + n] for o, n in zip(offs[:-1], src_sizes)]            # where the backward writes
        self.out_regions = [outb[o:o + n] for o, n in zip(offs[:-1], src_sizes)]       # where the mean lands
        self.region_views = [split(r, src) for src, r in zip(self.flat_sources, self.regions)]
        self.out_views = [split(r, src) for src, r in zip(self.flat_sources, self.out_regions)]
        for src, region in zip(self.flat_sources, self.regions):
            if hasattr(src, "bind"):
                src.bind(region)
        self.flat = inb[offs[-1]:offs[-1] + sum(self.sizes)] if self.params else None
        self.flat_out = outb[offs[-1]:offs[-1] + sum(self.sizes)] if self.params else None
        if self.params:
            self.views = [v.view_as(p) for v, p in zip(self.flat.split(self.sizes), self.params)]
            self.views_out = [v.view_as(p) for v, p in zip(self.flat_out.split(self.sizes), self.params)]

    def _all_reduce_p2p(self, inv):
        """Gradients -> the symmetric input buffer (the bound encoders' backward already wrote them there) -> one exchange ->
        every p.grad refers to / is refreshed from the buffer that holds the mean.  Out of place (the default one-kernel
        exchange) the encoders' `p.grad` are RE-POINTED to the views of the output buffer: no copy in either direction."""
        after = []
        for src, region, views, oregion, oviews in zip(self.flat_sources, self.regions, self.region_views, self.out_regions, self.out_views):
            flat, ps = src()
            if _flat_is_live(flat, ps):
                if flat.data_ptr() != region.data_ptr():  # live, but somewhere else: one bulk copy each way
                    region.copy_(flat)
                    after.append(lambda flat=flat, oregion=oregion: flat.copy_(oregion))
                elif not self.in_place:
                    def repoint(src=src, ps=ps, oviews=oviews, oregion=oregion):
                        for p, v in zip(ps, oviews):
                            p.grad = v
                        if hasattr(src, "set_flat"):
                            src.set_flat(oregion)
                    after.append(repoint)
            else:  # e.g. gradients accumulated over several backward passes: the parameters' .grad are the truth
                _pack(views, ps)
                after.append(lambda oviews=oviews, ps=ps: _unpack(oviews, ps))
        if self.params:
            _pack(self.views, self.params)
        self.p2p.run(inv if self.scale else 1.0)
        for src in self.flat_sources:
            if hasattr(src, "step_done"):
                src.step_done()   # every backward of this step has run: no forward is awaiting one any more
        for fn in after:
            fn()
        if self.params:
            _unpack(self.views_out, self.params)
        return self.flat_out

    # ---- torch.distributed transport --------------------------------------------------------------------------------
    def _on_grad(self, _param):
        self._seen += 1
        if self._seen == len(self.params) and self._pending is None:
            self._launch_packed()

    def _launch_packed(self):
        _pack(self.views, self.params)
        self._pending = dist.all_reduce(self.flat, op=dist.ReduceOp.SUM, group=self.group, async_op=True)

    def all_reduce_mean(self):
        """Call after loss.backward().  Returns the packed buffer of the non-flat parameters (or None)."""
        world = dist.get_world_size(self.group)
        inv = 1.0 / world
        if self.p2p is not None:
            return self._all_reduce_p2p(inv)
        works = []
        for src in self.flat_sources:
            flat, ps = src()
            unpack = None
            if not _flat_is_live(flat, ps):  # fall back to packing this module's gradients
                if not ps:
                    continue
                flat = torch.empty(sum(p.numel() for p in ps), dtype=torch.float32, device=ps[0].device)
                views = [v.view_as(p) for v, p in zip(flat.split([p.numel() for p in ps]), ps)]
                _pack(views, ps)
                unpack = (views, ps)
            works.append((dist.all_reduce(flat, op=dist.ReduceOp.SUM, group=self.group, async_op=True), flat, unpack))
        if self.flat is not None:
            if self._pending is None:  # no hooks, or a parameter got no gradient this step
                self._launch_packed()
            self._pending.wait()
            self._pending, self._seen = None, 0
            if self.scale:
                self.flat.mul_(inv)
            _unpack(self.views, self.params)
        for work, flat, unpack in works:
            work.wait()
            if self.scale:
                flat.mul_(inv)
            if unpack is not None:
                _unpack(*unpack)
        return self.flat

    def close(self):
        for h in self._hooks:
            h.remove()
        self._hooks = []
        for src in self.flat_sources:
            if self.p2p is not None and hasattr(src, "bind"):
                src.bind(None)


def encoder_flat_source(gnn):
    """flat_sources entry for a chem or bio GNN running the fused path: (last flat gradient buffer, its parameters).
    `bind(buffer)` makes the encoder's backward write its gradients into `buffer` (see ops._EncoderPlan.grad_buffer)."""
    def src():
        plan = gnn._fused_plan()
        if plan is None:
            return None, []
        return plan.last_flat_grad, plan.params

    def bind(buffer):
        plan = gnn._fused_plan()
        if plan is not None:
            if buffer is not None and buffer.numel() != plan.total:
                raise ValueError("bound gradient buffer does not match the encoder's flat layout")
            plan.grad_buffer = buffer
    def step_done():
        plan = gnn._fused_plan()
        if plan is not None:
            plan.live_forwards = 0
    def set_flat(buffer):
        plan = gnn._fused_plan()
        if plan is not None:
            plan.last_flat_grad = buffer
    src.bind = bind
    src.step_done = step_done
    src.set_flat = set_flat
    return src
