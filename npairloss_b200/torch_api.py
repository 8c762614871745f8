"""PyTorch autograd surface over the C ABI (SURVEY.md 8f item 3: "so the layer is usable outside Caffe").

    loss_fn = NPairLoss(margin_diff=-0.05, an_method=synth.HARD, ...)      # NPairLossParameter fields, caffe.proto:2-23
    loss, tops = loss_fn(embeddings, labels)                                # CUDA fp32 tensors [Q, D], [Q]
    loss.backward()                                                         # through npair_backward

torch is plumbing only (device memory, streams, the autograd graph); forward and backward are the library's kernels.  There
is no CPU path: CPU tensors raise.  `tops` = [loss, top1, top5, top10, feature_asum] as in the reference (.cu:388-401).

WHAT THE BACKWARD RETURNS.  npair_backward reproduces the reference's Backward_gpu (.cu:420-499), which is NOT the analytic
gradient of the loss it reports: at world = 1 it is exactly HALF of it (the 1/2 - 1/2 blend of .cu:492-497, SURVEY Q8), and at
world > 1 the transposed term is additionally divided by the world size (.cu:474).  `true_gradient=True` (world = 1 only) multiplies
by 2 so that torch.autograd.gradcheck-style expectations hold; the default keeps the reference's values, which is what a net
trained with the reference layer sees.

The library context is stateful (S and the row records of the last forward): a second forward through the same module before the
backward of the first would silently change what that backward computes.  Every forward therefore stamps a generation number and
the backward refuses to run against a newer forward.

CROSS-BATCH MEMORY.  NPairLoss(memory_rows=M) (world = 1) keeps the last M embeddings and labels it has seen in a device FIFO ring and
passes them to every forward as extra database rows (npair_forward_memory, DESIGN 4.3; Wang et al., CVPR 2020): they take part in the
mining and in the softmax of the current anchors but receive no gradient.  reset_memory() empties the ring, so when the memory starts
(XBM warms up for some iterations first) is the caller's choice.

ASYNCHRONOUS STEP.  NPairLoss(blocking=False) (world = 1) makes no host synchronisation: the forward writes the tops into a 5-float CUDA
tensor (npair_forward_async) and the loss is its element 0 on the device; the backward reads grad_loss on the device
(npair_backward_device_weight) instead of calling .item().  Same values, bit for bit, as blocking=True.  A whole training step through it
can be captured with torch.cuda.graph (DESIGN 4.4); a device error (the cases the blocking forward raises for) gives NaN tops and is
reported by async_status().  With memory_rows > 0 it runs eagerly only: the ring's head is Python state that a graph would freeze.

LIBRARY MEMORY.  NPairLoss(memory_rows=M, library_memory=True) keeps the ring in the library context instead (npair_forward_ring,
DESIGN 4.3.1): the same results bit for bit, the ring advanced on the device, and only the ring rows pushed since the last step
re-split.  With blocking=False a whole step can then be captured with torch.cuda.graph once the ring is full (M rows pushed).

ANCHOR WEIGHTS.  loss_fn(x, labels, anchor_weight=w) weights anchor i's term by w_i in [0, 1] (npair_set_anchor_io, DESIGN 4.5): the loss
is -(1/Z) sum_i w_i log(A_i / T_i), Z = Q (Q * world under global_scope), not renormalised, and the backward is its gradient.  A row with
w_i = 0 still serves the other anchors as a positive or negative, and still gets gradient through their terms.  row_losses=True adds a
third output, the unweighted per-anchor losses -log(A_i / T_i) (not differentiable).  When w requires grad, its gradient is
grad_loss * row_loss_i / Z (the analytic one, whatever true_gradient says).  Works with blocking=False and graph capture (w is then a
static input like the embeddings), memory_rows, normalize_input and world > 1.  A weight outside [0, 1] or NaN makes the blocking
forward raise capi.NpairError (E_ARG) and the asynchronous one give NaN tops, reported by async_status().

EXTRA ROWS.  loss_fn(x, labels, extra_rows=y, extra_labels=l) adds the m rows of y (CUDA fp32 [m, D], used as given: normalise them
first) to the database as non-anchor columns (npair_forward_memory, DESIGN 4.3): every anchor is mined and scored against them too.
When y requires grad, autograd receives its gradient (npair_backward_memory, DESIGN 4.6), so learnable class proxies (Proxy-NCA style:
one row per class, labels arange(C)) or a second encoder's rows train through the layer; true_gradient=True doubles it as it does the
embeddings' gradient.  Works with blocking=False and graph capture (y is a static input like the embeddings, m fixed per graph),
anchor_weight / row_losses and normalize_input (which normalises x only).  Not with memory_rows > 0 (both would fill the memory
columns), at world > 1, with global_scope, row-block mode or the SIMT backend (ValueError), nor, when y requires grad, with
FLAG_NO_FUSED_GRAD.  The context is then a memory context whose capacity grows to the largest m seen; later calls without extra rows
run on it as plain forwards.
"""
from __future__ import annotations

import math

import torch

from . import capi


def _fp32_labels(label):
    """Labels as the library compares them: fp32.  Any numeric dtype is accepted whose values fp32 holds exactly; a value it does not
    (an int64 id above 2^24 that would round onto its neighbour, a float64 fraction) raises ValueError instead of silently merging two
    classes.  fp32 labels pass unchanged, NaN included."""
    lab = label.to(torch.float32)
    if label.dtype != torch.float32:
        exact = lab.to(label.dtype) == label
        if label.is_floating_point():
            exact |= torch.isnan(label)
        if not bool(exact.all()):
            bad = label[~exact].reshape(-1)[0].item()
            raise ValueError(f"labels of dtype {label.dtype} that fp32 cannot hold exactly (e.g. {bad!r}); the library compares labels in "
                             "fp32, so such labels would merge classes: renumber them as integers below 2^24")
    return lab


class _NPairFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, feat, label, weight, extra, extra_label, owner, want_rows):
        m = 0 if extra is None else extra.shape[0]
        layer = owner._context(feat, m)
        rl = None
        if want_rows or ctx.needs_input_grad[2]:              # the weights' gradient is made of the per-anchor losses
            rl = torch.empty(feat.shape[0], dtype=torch.float32, device=feat.device)
        io = weight is not None or rl is not None
        if io:
            layer.set_anchor_io(weight, rl)
        try:
            if owner._library_memory:
                if owner._blocking:
                    t = torch.tensor(layer.forward_ring(feat, label), dtype=torch.float32, device=feat.device)
                else:
                    t = layer.forward_ring_async(feat, label, torch.empty(5, dtype=torch.float32, device=feat.device))
                owner._mem_count += feat.shape[0]
            elif owner._blocking:
                if owner._mem_cap:
                    tops = owner._forward_memory(layer, feat, label)
                elif extra is not None:
                    tops = layer.forward_memory(feat, label, extra, extra_label, m)
                else:
                    tops = layer.forward(feat, label)         # blocks until the five scalars are on the host (as the reference)
                t = torch.tensor(tops, dtype=torch.float32, device=feat.device)
            else:
                t = torch.empty(5, dtype=torch.float32, device=feat.device)   # under capture: from the graph's pool
                if owner._mem_cap:
                    owner._forward_memory(layer, feat, label, t)
                elif extra is not None:
                    layer.forward_memory_async(feat, label, extra, extra_label, m, t)
                else:
                    layer.forward_async(feat, label, t)
        finally:
            if io:                                            # the forward is enqueued: the next one through this context is unweighted
                layer.set_anchor_io(None, None)
        owner._generation += 1
        ctx.owner, ctx.layer, ctx.generation = owner, layer, owner._generation
        ctx.save_for_backward(feat, label)                    # the C ABI wants both unchanged until the backward is enqueued
        ctx.row_loss = rl
        ctx.extra_shape = None if extra is None else tuple(extra.shape)
        ctx.norm = feat.shape[0] * (owner._world if owner._config.get("global_scope") else 1)   # Z: Q, or N in world scope
        if want_rows:
            ctx.mark_non_differentiable(t, rl)
            return t[0].clone(), t, rl
        ctx.mark_non_differentiable(t)
        return t[0].clone(), t

    @staticmethod
    def backward(ctx, grad_loss, _grad_tops, *_grad_rows):
        if ctx.generation != ctx.owner._generation or ctx.layer is not ctx.owner._ctx:
            raise RuntimeError("NPairLoss: another forward ran through this module after the one being differentiated; the library "
                               "context holds the newer batch.  Use one NPairLoss module per outstanding graph.")
        feat, _label = ctx.saved_tensors
        diff = torch.empty_like(feat)
        mem_diff = None
        if ctx.needs_input_grad[3]:                           # the extra rows' gradient: npair_backward_memory
            mem_diff = torch.empty(ctx.extra_shape, dtype=torch.float32, device=feat.device)
        with_mem = mem_diff is not None and mem_diff.numel() > 0
        if ctx.owner._blocking:
            # the reference scales by top[0]->cpu_diff()[0] (.cu:435): a host scalar, hence the .item()
            if with_mem:
                ctx.layer.backward_memory(float(grad_loss.item()), diff, mem_diff)
            else:
                ctx.layer.backward(float(grad_loss.item()), diff)
        else:
            lw = grad_loss.detach().to(torch.float32).contiguous().reshape(1)
            if with_mem:
                ctx.layer.backward_memory_device_weight(lw, diff, mem_diff)
            else:
                ctx.layer.backward_device_weight(lw, diff)
        if ctx.owner._true_gradient:
            diff.mul_(2.0)
            if with_mem:
                mem_diff.mul_(2.0)
        grad_w = None
        if ctx.needs_input_grad[2]:                           # d loss / d w_i = row_loss_i / Z
            grad_w = grad_loss.to(torch.float32) * ctx.row_loss / ctx.norm
        return diff, None, grad_w, mem_diff, None, None, None


class NPairLoss(torch.nn.Module):
    """Module form; the library context is created on first use for the (rows, dims, device) it sees and re-created when
    they change.  Keyword arguments are the fields of capi.make_config (mining regions/methods, margins, SN, precision,
    normalize_input, ...).

    memory_rows=M > 0 (world = 1 only): a cross-batch memory of the last M rows this module has seen.  Each forward passes the ring's
    m = min(rows enqueued, M) valid rows, slots 0 .. m-1 in slot order, and then enqueues the batch's own rows, detached (under
    normalize_input the normalised rows the layer used), so a batch is never in the memory during its own step.  The ring survives the
    context being re-created for a new batch size; it is emptied when the dimension or device changes and by reset_memory().

    library_memory=True (with memory_rows > 0): the ring lives in the library context (LIBRARY MEMORY in the module docstring), with the
    same slots, results and rules; memory() returns copies, and the ring is carried into a context re-created for a new batch size.

    blocking=False (world = 1 only): the asynchronous step of the module docstring.  The loss and the tops are computed on the device and
    nothing waits for them; async_status() reports a device error of the forwards since the last call."""

    def __init__(self, world: int = 1, rank: int = 0, nccl_id: bytes | None = None, true_gradient: bool = False, _context_factory=None,
                 memory_rows: int = 0, blocking: bool = True, library_memory: bool = False, **config):
        super().__init__()
        if not blocking and world != 1:
            raise ValueError("blocking=False is defined for world = 1 (the multi-rank exchanges keep host state per step)")
        if true_gradient and world != 1:
            raise ValueError("true_gradient is defined for world = 1 (the reference's multi-rank blend is not a gradient of one loss)")
        if int(memory_rows) < 0:
            raise ValueError("memory_rows must be >= 0")
        if int(memory_rows) and world != 1:
            raise ValueError("a cross-batch memory (memory_rows > 0) is defined for world = 1")
        self._config, self._world, self._rank, self._nccl_id = dict(config), world, rank, nccl_id
        self._mem_cap = int(memory_rows)
        self._library_memory = bool(library_memory)
        if self._library_memory and not self._mem_cap:
            raise ValueError("library_memory=True needs memory_rows > 0")
        if _context_factory is not None:
            self._factory = _context_factory
        elif self._library_memory:
            self._factory = lambda cfg, nid: capi.Context(cfg, nid, memory_rows=self._mem_cap, ring=True)
        elif self._mem_cap:
            self._factory = lambda cfg, nid: capi.Context(cfg, nid, memory_rows=self._mem_cap)
        else:   # extra_rows: a memory context of the largest m seen
            self._factory = lambda cfg, nid: capi.Context(cfg, nid, memory_rows=self._extra_cap)
        self._extra_cap = 0
        self._ctx, self._key = None, None
        self._generation = 0
        self._true_gradient = bool(true_gradient)
        self._blocking = bool(blocking)
        self._mem_x = self._mem_l = None      # the ring: [M, D] rows and [M] fp32 labels, allocated at the first forward
        self._ring_device = None              # library_memory: the device of the context's ring
        # rows enqueued since the last reset (the valid slots are 0 .. min(count, M) - 1); library_memory: as this module enqueued them,
        # which a replayed graph does not add to (only whether the ring is full matters then)
        self._mem_count = 0

    def reset_memory(self):
        """Empties the cross-batch memory: the next forward sees no memory rows."""
        self._mem_count = 0
        if self._library_memory and self._ctx is not None:
            self._ctx.ring_load(None, None, 0)

    def memory(self):
        """(rows [m, D], labels [m]) the next forward passes as its memory, in slot order: views of the ring's valid slots, or with
        library_memory copies read from the context."""
        if self._library_memory:
            if self._ctx is None:
                return None, None
            x, lab, count = self._read_ring(self._ctx)
            m = min(count, self._mem_cap)
            return x[:m], lab[:m]
        m = min(self._mem_count, self._mem_cap)
        if self._mem_x is None:
            return None, None
        return self._mem_x[:m], self._mem_l[:m]

    def _read_ring(self, layer):
        """(rows [M, D], labels [M], push count) of a library_memory context's ring."""
        dev = self._ring_device
        x = torch.empty(self._mem_cap, layer.cfg.D, dtype=torch.float32, device=dev)
        lab = torch.empty(self._mem_cap, dtype=torch.float32, device=dev)
        count = torch.zeros(1, dtype=torch.int64, device=dev)
        layer.ring_read(x, lab, count)
        return x, lab, int(count.item())

    def async_status(self):
        """blocking=False: waits for the module's last library call and raises capi.NpairError if a forward since the previous call met a
        device error (its tops are NaN); nothing to report before the first forward."""
        if self._ctx is not None:
            self._ctx.async_status()

    def _forward_memory(self, layer, feat, label, tops_out=None):
        d = feat.shape[1]
        if self._mem_x is None or self._mem_x.shape[1] != d or self._mem_x.device != feat.device:
            self._mem_x = torch.empty(self._mem_cap, d, dtype=torch.float32, device=feat.device)
            self._mem_l = torch.empty(self._mem_cap, dtype=torch.float32, device=feat.device)
            self._mem_count = 0
        m = min(self._mem_count, self._mem_cap)
        if tops_out is None:
            tops = layer.forward_memory(feat, label, self._mem_x, self._mem_l, m)
        else:
            tops = layer.forward_memory_async(feat, label, self._mem_x, self._mem_l, m, tops_out)
        # the forward has read the memory: this batch's rows go in behind it, in stream order
        rows = feat.detach()
        if self._config.get("normalize_input"):
            rows = capi.l2normalize_forward(rows)[0]
        q = rows.shape[0]
        if q > self._mem_cap:                 # a batch larger than the memory leaves its last M rows
            rows, label, self._mem_count = rows[q - self._mem_cap:], label[q - self._mem_cap:], self._mem_count + q - self._mem_cap
            q = self._mem_cap
        head = self._mem_count % self._mem_cap
        first = min(q, self._mem_cap - head)
        self._mem_x[head:head + first].copy_(rows[:first])
        self._mem_l[head:head + first].copy_(label[:first])
        if first < q:
            self._mem_x[:q - first].copy_(rows[first:])
            self._mem_l[:q - first].copy_(label[first:])
        self._mem_count += q
        return tops

    def _capture_refusal(self, feat):
        """Why a library_memory step on feat cannot be captured now, or None: every replay must find the ring full."""
        if self._blocking:
            return "NPairLoss(blocking=True) waits for its tops on the host and cannot be captured: use blocking=False"
        q = feat.shape[0]
        if (q, feat[0].numel(), feat.device.index) != self._key:
            return ("NPairLoss(library_memory=True): run an eager step with this batch shape before capturing one (it creates the "
                    "library context and carries the memory ring into it)")
        if self._mem_count < self._mem_cap:
            left = self._mem_cap - self._mem_count
            return (f"NPairLoss(library_memory=True) can be captured once its memory ring is full: {left} of its {self._mem_cap} rows "
                    f"are missing; run {-(-left // q)} more eager step(s) of {q} rows first")
        return None

    def _context(self, feat, extra_m=0):
        q, d = feat.shape[0], feat[0].numel()
        key = (q, d, feat.device.index)
        grow = extra_m > self._extra_cap
        self._extra_cap = max(self._extra_cap, extra_m)
        if key != self._key or grow:
            old, old_key = self._ctx, self._key
            cfg = capi.make_config(q, d, world=self._world, rank=self._rank, device=feat.device.index or 0, **self._config)
            # the new context is created BEFORE the old one is closed: contexts made with the same NCCL id share one
            # communicator inside the library, which must stay referenced (a unique id can be consumed only once)
            self._ctx, self._key = self._factory(cfg, self._nccl_id), key
            if self._library_memory:
                # the ring survives a new batch size as the module's own ring does (slots do not depend on Q); a new dimension or
                # device starts it empty
                self._ring_device = feat.device
                if old is not None and old_key[1:] == key[1:]:
                    x, lab, self._mem_count = self._read_ring(old)
                    self._ctx.ring_load(x, lab, self._mem_count)
                else:
                    self._mem_count = 0
            if old is not None and hasattr(old, "close"):
                old.close()
        return self._ctx

    def forward(self, feat, label, anchor_weight=None, row_losses=False, extra_rows=None, extra_labels=None):
        """(loss, tops), or (loss, tops, row_loss) with row_losses=True; anchor_weight: None or Q fp32 weights in [0, 1] on feat's
        device (ANCHOR WEIGHTS in the module docstring); extra_rows / extra_labels: None or [m, D] fp32 rows and their m labels on feat's
        device (EXTRA ROWS in the module docstring)."""
        if feat.dtype != torch.float32:
            raise TypeError("NPairLoss computes in fp32 like the reference (Dtype=float); cast the embeddings")
        extra_rows, extra_labels = self._extra(feat, extra_rows, extra_labels)
        if anchor_weight is not None:
            if not isinstance(anchor_weight, torch.Tensor) or anchor_weight.dtype != torch.float32:
                raise TypeError("anchor_weight must be a float32 tensor (weights in [0, 1], one per row of the batch)")
            if anchor_weight.dim() != 1 or anchor_weight.shape[0] != feat.shape[0]:
                raise ValueError(f"anchor_weight must have shape [{feat.shape[0]}] (one weight per row), got {list(anchor_weight.shape)}")
            if anchor_weight.device != feat.device:
                raise ValueError("anchor_weight must be on the embeddings' device")
            anchor_weight = anchor_weight.contiguous()
        if self._library_memory and feat.is_cuda and torch.cuda.is_current_stream_capturing():
            refusal = self._capture_refusal(feat)
            if refusal:
                raise RuntimeError(refusal)
        elif not self._blocking and self._mem_cap and feat.is_cuda and torch.cuda.is_current_stream_capturing():
            raise RuntimeError("NPairLoss(memory_rows > 0, blocking=False) cannot be captured into a CUDA graph: the memory ring's head "
                               "and count are Python state that the graph would freeze")
        feat2 = feat.reshape(feat.shape[0], -1).contiguous()
        label = _fp32_labels(label).contiguous()               # labels are stored as Dtype in the reference (bottom[1])
        return _NPairFunction.apply(feat2, label, anchor_weight, extra_rows, extra_labels, self, bool(row_losses))

    def _extra(self, feat, rows, labels):
        """The extra rows and their fp32 labels as the library takes them, after the checks of EXTRA ROWS (module docstring)."""
        if rows is None and labels is None:
            return None, None
        if rows is None or labels is None:
            raise ValueError("extra_rows and extra_labels go together")
        if self._mem_cap:
            raise ValueError("extra_rows cannot be combined with memory_rows > 0: both would be the step's memory columns")
        if self._world != 1:
            raise ValueError("extra_rows are defined for world = 1 (a cross-batch memory step is a world-1 step)")
        cfg = self._config
        flags = int(cfg.get("flags", 0))
        if cfg.get("global_scope") or cfg.get("sim_block_rows") or (flags >> capi.SIM_BLOCK_SHIFT) & capi.SIM_BLOCK_MAX_UNITS \
                or cfg.get("gemm_backend", capi.GEMM_TCGEN05) != capi.GEMM_TCGEN05:
            raise ValueError("extra_rows run a cross-batch memory step, which needs the tensor-core backend and supports neither "
                             "global_scope nor row-block similarity mode (sim_block_rows)")
        if flags & capi.FLAG_NO_FUSED_GRAD and isinstance(rows, torch.Tensor) and rows.requires_grad:
            raise ValueError("the gradient of extra_rows runs on the fused gradient kernel: drop FLAG_NO_FUSED_GRAD from flags")
        if not isinstance(rows, torch.Tensor) or rows.dtype != torch.float32:
            raise TypeError("extra_rows must be a float32 tensor [m, D]")
        d = feat[0].numel() if feat.dim() else 0
        if rows.dim() != 2 or rows.shape[1] != d:
            raise ValueError(f"extra_rows must have shape [m, {d}] (the embeddings' dimension), got {list(rows.shape)}")
        if not isinstance(labels, torch.Tensor) or labels.dim() != 1 or labels.shape[0] != rows.shape[0]:
            raise ValueError(f"extra_labels must be a tensor of shape [{rows.shape[0]}] (one label per extra row)")
        if rows.device != feat.device or labels.device != feat.device:
            raise ValueError("extra_rows and extra_labels must be on the embeddings' device")
        return rows.contiguous(), _fp32_labels(labels).contiguous()


def recall_at_k(query, qlabel, gallery=None, glabel=None, ks=(1, 2, 4, 8), precision=capi.PREC_FP32_FP16X2, self_offset=None):
    """Recall@K of a whole embedding set (DESIGN 8; not part of the reference layer): query i is a hit at K when its best positive --
    the most similar gallery row of its label, itself excluded -- is among its K nearest gallery rows, ties counting against it.

    gallery=None: self-retrieval, every query against all the others.  Otherwise query/gallery with disjoint sets, or, with
    `self_offset` = k, queries that are gallery rows k, k+1, ...  Takes CUDA fp32 embeddings as given (L2-normalise them first for
    cosine similarity); labels of any numeric dtype whose values fp32 holds exactly (ValueError otherwise).  Returns ({K: recall},
    rank) with rank the int32 CUDA tensor of the best positive's rank per query (0: the query has no positive)."""
    q, ql, g, gl, off = _retrieval_sets("recall_at_k", query, qlabel, gallery, glabel, self_offset)
    ev = capi.Evaluator(q.shape[0], g.shape[0], q.shape[1], precision, q.device.index or 0)
    try:
        rank = ev.rank(q, ql, g, gl, off)
        hits = {int(k): ((rank >= 1) & (rank <= int(k))).sum() for k in ks}
        nq = q.shape[0]
        return {k: int(v) / nq for k, v in hits.items()}, rank
    finally:
        ev.close()


def retrieval_metrics(query, qlabel, gallery=None, glabel=None, ks=(1, 2, 4, 8), precision=capi.PREC_FP32_FP16X2, self_offset=None):
    """MAP@R, R-Precision and Recall@K of a whole embedding set in one evaluator call (DESIGN 8; not part of the reference layer).

    Sets, labels and ties as in recall_at_k.  Query i has R_i positives (gallery rows of its label, itself excluded); MAP@R_i and
    R-Precision_i look at where each of them lands among its R_i nearest gallery rows, a negative that ties a positive placed before it.
    Returns ({"map@r": mean MAP@R, "r_precision": mean R-Precision, "recall@K": Recall@K for each K in ks, "no_positive": n},
    per_query) with per_query the CUDA tensors "map_r" and "r_precision" (fp64, NaN where R_i = 0), "R" and "rank" (int32, rank as in
    recall_at_k).

    The MAP@R and R-Precision means are taken over the queries with R_i >= 1 only, and "no_positive" is the number of queries left out
    (NaN means when every query is).  recall_at_k and "recall@K" instead count a query without a positive as a miss, over all nq."""
    q, ql, g, gl, off = _retrieval_sets("retrieval_metrics", query, qlabel, gallery, glabel, self_offset)
    ev = capi.Evaluator(q.shape[0], g.shape[0], q.shape[1], precision, q.device.index or 0)
    try:
        per_query = ev.map_at_r(q, ql, g, gl, off)
    finally:
        ev.close()
    nq, R, rank = q.shape[0], per_query["R"], per_query["rank"]
    has = R > 0
    n_has = int(has.sum())
    nan = float("nan")
    out = {"map@r": float(per_query["map_r"][has].mean()) if n_has else nan,
           "r_precision": float(per_query["r_precision"][has].mean()) if n_has else nan}
    for k in ks:
        out[f"recall@{int(k)}"] = int(((rank >= 1) & (rank <= int(k))).sum()) / nq
    out["no_positive"] = nq - n_has
    return out, per_query


def clustering_metrics(emb, labels, k=None, seed=0, max_iter=100, precision=capi.PREC_FP32_FP16X2, init="random", n_init=1,
                       local_trials=0):
    """NMI and F1 of a k-means clustering of a whole embedding set, the clustering half of the metric-learning protocol (Sohn 2016;
    Song et al. 2016), with Lloyd's k-means on the tensor cores (Evaluator.kmeans, DESIGN 8.2; not part of the reference layer).

    Takes CUDA fp32 embeddings as given (L2-normalise them first for cosine geometry) and labels of any numeric dtype that fp32 holds
    exactly (ValueError otherwise), compared as floats.  k=None: the number of distinct labels.  n_init runs, r = 0 .. n_init - 1, each
    seeded with seed + r and started from k rows of the points:
      init="random":     centroid c starts as row init[c] of init = torch.randperm(n, generator=torch.Generator().manual_seed(seed + r))[:k]
      init="k-means++":  the rows of Evaluator.kmeans_seed(x, k, seed + r, local_trials) (exact, GPU; local_trials 0: 2 + floor(ln k))
    The run with the least inertia (fp64, fixed order) is kept, ties to the lowest r, so the same arguments give the same result; the
    defaults are one run from a random permutation.  Returns ({"nmi", "f1", "inertia", "iterations", "converged", "empty_clusters",
    "restart", "inertias"}, assign, centroids) with the scores of clustering_scores, "converged" whether the last sweep changed no
    assignment, "restart" the r kept, "inertias" every run's inertia, and assign / centroids CUDA tensors of the run kept."""
    if init not in ("random", "k-means++"):
        raise ValueError(f'clustering_metrics: init = {init!r} is not "random" or "k-means++"')
    if int(n_init) < 1:
        raise ValueError(f"clustering_metrics needs n_init >= 1 (got {n_init})")
    x, lab, _, _, _ = _retrieval_sets("clustering_metrics", emb, labels, None, None, None)
    n, D = x.shape
    if k is None:
        k = int(torch.unique(lab).numel())
    k = int(k)
    if not 1 <= k <= n:
        raise ValueError(f"clustering_metrics needs 1 <= k <= n (n = {n}, k = {k})")
    ev = capi.Evaluator(n, k, D, precision, x.device.index or 0)
    best, best_r, inertias = None, 0, []
    try:
        for r in range(int(n_init)):
            s = int(seed) + r
            if init == "random":
                rows = torch.randperm(n, generator=torch.Generator().manual_seed(s))[:k].tolist()
            else:
                rows = ev.kmeans_seed(x, k, s, local_trials)[0]
            res = ev.kmeans(x, k, rows, max_iter)
            inertias.append(float(res["inertia"]))
            if best is None or inertias[-1] < inertias[best_r]:
                best, best_r = res, r
    finally:
        ev.close()
    nmi, f1 = clustering_scores(lab, best["assign"])
    out = {"nmi": nmi, "f1": f1, "inertia": inertias[best_r], "iterations": best["iterations"], "converged": best["changed"] == 0,
           "empty_clusters": best["empty"], "restart": best_r, "inertias": inertias}
    return out, best["assign"], best["centroids"]


def clustering_scores(labels, assign):
    """(NMI, F1) of the clustering `assign` against `labels` (compared as fp32 floats; ValueError for labels fp32 cannot hold
    exactly), by fp64 / int64 bookkeeping over the non-zero cells of the contingency table, on the tensors' device.
      NMI = 2 I(Y;C) / (H(Y) + H(C)), natural log, over the non-empty clusters; 1.0 when both entropies are 0.
      F1  = pairwise: TP = sum over cells of C(n_lc, 2), precision = TP / sum_c C(n_c, 2), recall = TP / sum_l C(n_l, 2); a 0/0 term
            counts as 0, and F1 = 0 when precision + recall = 0.
    Each entropy and the mutual information sum their terms in ascending order, so a perfect clustering gives exactly 1.0."""
    lab = _fp32_labels(labels.reshape(-1))
    a = assign.reshape(-1).to(device=lab.device, dtype=torch.int64)
    if lab.numel() != a.numel():
        raise ValueError("labels and assign differ in length")
    n = lab.numel()
    _, y = torch.unique(lab, return_inverse=True)
    _, c = torch.unique(a, return_inverse=True)                   # the non-empty clusters, renumbered
    n_c_ids = int(c.max()) + 1
    cells, n_lc = torch.unique(y * n_c_ids + c, return_counts=True)
    n_l, n_c = torch.bincount(y), torch.bincount(c)

    def plogn(counts, denom):                                     # sum of (m / n) log(n / denom) over the terms, ascending
        p = counts.double() / n
        return float(torch.sort(p * torch.log(n / denom.double())).values.sum())

    i_yc = plogn(n_lc, n_l[cells // n_c_ids] * n_c[cells % n_c_ids] / n_lc.double())
    h_y, h_c = plogn(n_l, n_l), plogn(n_c, n_c)
    nmi = 1.0 if h_y + h_c == 0 else 2.0 * i_yc / (h_y + h_c)

    def pairs(m):
        return int((m * (m - 1) // 2).sum())

    tp, pc, pl = pairs(n_lc), pairs(n_c), pairs(n_l)
    prec = tp / pc if pc else 0.0
    rec = tp / pl if pl else 0.0
    f1 = 2.0 * prec * rec / (prec + rec) if prec + rec > 0 else 0.0
    return nmi, f1


def _retrieval_sets(who, query, qlabel, gallery, glabel, self_offset):
    """(query, query labels, gallery, gallery labels, self_offset) as the evaluator takes them: contiguous 2-D CUDA fp32 rows, fp32
    labels; gallery=None is self-retrieval."""
    q = _embeddings(who, query)
    ql = _fp32_labels(qlabel.to(q.device)).contiguous()
    if gallery is None:
        if glabel is not None:
            raise ValueError("glabel without gallery")
        g, gl, off = q, ql, 0 if self_offset is None else self_offset
    else:
        if glabel is None:
            raise ValueError("gallery without glabel")
        g = _embeddings(who, gallery)
        gl = _fp32_labels(glabel.to(q.device)).contiguous()
        off = -1 if self_offset is None else self_offset
    if g.shape[1] != q.shape[1]:
        raise ValueError("query and gallery dimensions differ")
    return q, ql, g, gl, off


def _embeddings(who, x):
    """x as the evaluator takes embeddings: contiguous 2-D CUDA fp32 rows."""
    if not x.is_cuda or x.dtype != torch.float32:
        raise TypeError(f"{who} takes CUDA float32 embeddings (there is no CPU path)")
    return x.reshape(x.shape[0], -1).contiguous()


def knn(query, gallery=None, *, k, precision=capi.PREC_FP32_FP16X2, self_offset=None, block_rows=None):
    """Exact k nearest neighbours of every query among the gallery rows (Evaluator.knn, DESIGN 8.3; not part of the reference layer),
    by the library's similarity: the same values recall_at_k ranks by.

    Sets as in recall_at_k, without labels: gallery=None is self-retrieval, every row against all the others; otherwise disjoint
    query / gallery sets, or, with `self_offset` = o, queries that are gallery rows o, o+1, ...  Row i lists the k gallery rows that
    come first by similarity descending, then gallery index ascending; a NaN similarity ranks below every number.  block_rows: queries
    per block of the similarity matrix the call holds (a multiple of 128; None: 1024), which changes memory, never the result.
    Returns (sim [nq, k] fp32, index [nq, k] int64) CUDA tensors."""
    q = _embeddings("knn", query)
    if gallery is None:
        g, off = q, 0 if self_offset is None else self_offset
    else:
        g, off = _embeddings("knn", gallery), -1 if self_offset is None else self_offset
    if g.shape[1] != q.shape[1]:
        raise ValueError("query and gallery dimensions differ")
    ev = capi.Evaluator(q.shape[0], g.shape[0], q.shape[1], precision, q.device.index or 0)
    try:
        sim, index = ev.knn(q, g, int(k), off, block_rows=int(block_rows or 0))
    finally:
        ev.close()
    return sim, index.long()


def knn_merge(sims, indices, k):
    """Merges the k-NN lists of the same queries over several gallery shards (each from Evaluator.knn with the shard's gallery_row0 and
    a shared absmax) into the first k by knn's order: similarity descending with NaN last, then index ascending.  Takes sequences of
    [nq, k_s] tensors on one device; stable sorts, so ties are decided by the index alone.  Returns (sim [nq, k], index [nq, k] int64)."""
    s = torch.cat([t.to(torch.float32) for t in sims], dim=1)
    ix = torch.cat([t.to(torch.int64) for t in indices], dim=1)
    if not 1 <= int(k) <= s.shape[1]:
        raise ValueError(f"knn_merge: k = {k} outside [1, {s.shape[1]}]")
    order = torch.argsort(ix, dim=1, stable=True)
    nan = torch.isnan(s)
    key = torch.where(nan, torch.full_like(s, float("-inf")), s)
    order = order.gather(1, torch.argsort(key.gather(1, order), dim=1, descending=True, stable=True))
    order = order.gather(1, torch.argsort(nan.gather(1, order).to(torch.uint8), dim=1, stable=True))
    order = order[:, :int(k)]
    return s.gather(1, order), ix.gather(1, order)


def hard_class_batches(class_emb, classes_per_batch, num_batches, pool_size=None, seed=0, precision=capi.PREC_FP32_FP16X2):
    """Hard negative class mining (Sohn 2016; Evaluator.class_batches, DESIGN 8.4; not part of the reference layer): the classes of
    num_batches N-pair batches, each chosen greedily from a random pool by the library's similarity of the class embeddings.

    class_emb: CUDA fp32 [C, D], one row per class (class_embeddings makes them from example embeddings).  Pool t is
    torch.randperm(C, generator=g)[:pool_size] for t = 0, 1, ... in order, g = torch.Generator().manual_seed(seed); pool_size=None is
    min(C, capi.CLASS_POOL_MAX).  Batch t seeds with pool t's first class, then adds, classes_per_batch - 1 times, the pool class whose
    largest similarity to the classes already in the batch is the largest (a NaN similarity ranks last; ties go to the earlier pool
    position, a random tie-break since pools are random).  Returns (batches [num_batches, classes_per_batch] int64 class indices in the
    order picked, scores [num_batches, classes_per_batch] fp32: the similarity each class was picked at, NaN for the seed), CUDA tensors."""
    x = _embeddings("hard_class_batches", class_emb)
    C, D = x.shape
    P = min(C, capi.CLASS_POOL_MAX) if pool_size is None else int(pool_size)
    g = torch.Generator().manual_seed(int(seed))
    pools = torch.stack([torch.randperm(C, generator=g)[:P] for _ in range(int(num_batches))]) if int(num_batches) > 0 \
        else torch.empty(0, P, dtype=torch.int64)
    ev = capi.Evaluator(C, C, D, precision, x.device.index or 0)
    try:
        batches, scores = ev.class_batches(x, pools, int(classes_per_batch))
    finally:
        ev.close()
    return batches.long(), scores


def class_embeddings(emb, labels, normalize=True):
    """One embedding per class: the mean of its examples' rows, for hard_class_batches.  Returns (class_labels fp32 [C] ascending,
    class_emb fp32 [C, D]), row c the class class_labels[c].

    The mean is the fixed-point rule of the k-means update (DESIGN 8.2): with sigma the pre-scale of max|x| over emb (a power of two
    with max|x * sigma| in [0.5, 1), up to its exponent clamp at the ends of the fp32 range), int64 sums of rint(x * sigma * 2^32), exact and independent of order, then
    (float)(ldexp(sum / count, -32) / sigma); so the result has the same bits on every run and device.  Labels of any numeric dtype
    that fp32 holds exactly; NaN labels raise ValueError.  normalize=True then L2-normalises each row (npair_l2normalize_forward, CUDA
    only); normalize=False also takes CPU tensors."""
    if emb.dtype != torch.float32:
        raise TypeError("class_embeddings takes float32 embeddings")
    x = emb.reshape(emb.shape[0], -1).contiguous()
    if normalize and not x.is_cuda:
        raise TypeError("class_embeddings(normalize=True) takes CUDA embeddings (the normalisation has no CPU path)")
    lab = _fp32_labels(labels.reshape(-1).to(x.device))
    if lab.numel() != x.shape[0]:
        raise ValueError("emb and labels differ in length")
    if bool(torch.isnan(lab).any()):
        raise ValueError("class_embeddings: a NaN label belongs to no class")
    amax = float(x.abs().max()) if x.numel() else 0.0
    if not math.isfinite(amax):
        raise ValueError("class_embeddings takes finite embeddings")
    e = min(max(math.frexp(amax)[1], -126), 127) if amax > 0 else 0      # pre_scale's exponent: 2^-e and 2^e finite in fp32
    class_labels, cls = torch.unique(lab, sorted=True, return_inverse=True)
    q = torch.round((x * (2.0 ** -e)).double() * 2.0 ** 32).long()          # x * sigma and the scaling by 2^32 are exact
    sums = torch.zeros(class_labels.numel(), x.shape[1], dtype=torch.int64, device=x.device).index_add_(0, cls, q)
    count = torch.bincount(cls, minlength=class_labels.numel()).double()
    mean = ((sums.double() / count[:, None]) * 2.0 ** -32 * 2.0 ** e).float()
    if normalize:
        mean = capi.l2normalize_forward(mean)[0]
    return class_labels, mean
