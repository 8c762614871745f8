"""ctypes binding of libnpair_b200.so (include/npair_b200.h).  Plumbing only: torch supplies device memory and
streams; every computation happens inside the CUDA library.  There is NO CPU fallback: if the library or an H100
is missing, calls fail loudly."""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("NPAIR_LIB") or os.path.join(_HERE, "lib", "libnpair_b200.so")   # NPAIR_LIB: tuning builds only

GLOBAL, LOCAL = 0, 1
HARD, EASY, RAND, RELATIVE_HARD, RELATIVE_EASY = 0, 1, 2, 3, 4
PREC_FP32_BF16X3, PREC_BF16, PREC_FP32_FP16X2 = 0, 1, 2
GEMM_TCGEN05, GEMM_SIMT_CHECK = 0, 1

ERRORS = {0: "OK", -1: "E_ARG", -2: "E_CUDA", -3: "E_NCCL", -4: "E_EMPTY_LIST", -5: "E_POS_RANGE", -6: "E_STATE"}


class NpairConfig(C.Structure):
    _fields_ = [("Q", C.c_int32), ("D", C.c_int32), ("world", C.c_int32), ("rank", C.c_int32), ("num_tops", C.c_int32),
                ("margin_ident", C.c_float), ("margin_diff", C.c_float), ("identsn", C.c_float), ("diffsn", C.c_float),
                ("ap_region", C.c_int32), ("ap_method", C.c_int32), ("an_region", C.c_int32), ("an_method", C.c_int32),
                ("sim_precision", C.c_int32), ("gemm_backend", C.c_int32), ("device", C.c_int32), ("bwd_exchange", C.c_int32),
                # ABI 2 extensions (0 = reference behaviour)
                ("global_scope", C.c_int32), ("normalize_input", C.c_int32), ("grad_chunk_cols", C.c_int32), ("flags", C.c_int32)]


FLAG_NO_FUSED_GRAD, FLAG_SIM_1CTA, FLAG_GRAD_1CTA, FLAG_NCCL_RECORDS, FLAG_NCCL_FEATURES, FLAG_LSEL_WARP, FLAG_GRAD_GENERAL = 1, 2, 4, 8, 16, 32, 64
# row-block similarity mode: flags bits 16-27 = block height in units of 128 rows (NPAIR_SIM_BLOCK_ROWS)
SIM_BLOCK_SHIFT, SIM_BLOCK_MAX_UNITS = 16, 0xFFF


def sim_block_flags(rows: int) -> int:
    """flags bits of a row-block height of `rows` (rounded up to a multiple of 128); 0 = S materialised whole."""
    units = (int(rows) + 127) // 128
    if rows < 0 or units > SIM_BLOCK_MAX_UNITS:
        raise ValueError(f"sim_block_rows must be in [0, {128 * SIM_BLOCK_MAX_UNITS}]")
    return units << SIM_BLOCK_SHIFT


EXPORTS = ["npair_config_default", "npair_workspace_bytes", "npair_nccl_unique_id", "npair_create", "npair_create_with_comm",
           "npair_destroy", "npair_forward", "npair_backward", "npair_forward_backward", "npair_forward_gathered", "npair_backward_partial", "npair_bwd_exchange_mode", "npair_row_scalars", "npair_backward_gathered", "npair_profile_enable", "npair_profile_read", "npair_kernel_launches", "npair_util_f64_to_f32", "npair_util_f32_to_f64", "npair_last_error", "npair_version", "npair_debug_read",
           "npair_debug_gemm", "npair_debug_mma_symmetric", "npair_l2normalize_forward", "npair_l2normalize_backward",
           # cross-batch memory (not part of the reference layer)
           "npair_create_memory", "npair_memory_workspace_bytes", "npair_forward_memory",
           "npair_create_memory_ring", "npair_memory_ring_workspace_bytes", "npair_forward_ring", "npair_forward_ring_async",
           "npair_memory_ring_read", "npair_memory_ring_load",
           # asynchronous step and graph capture (not part of the reference layer)
           "npair_forward_async", "npair_forward_memory_async", "npair_backward_device_weight", "npair_async_status",
           # the memory rows' gradient (not part of the reference layer)
           "npair_backward_memory", "npair_backward_memory_device_weight",
           # per-anchor loss weights and losses (not part of the reference layer)
           "npair_set_anchor_io",
           # retrieval evaluation (not part of the reference layer)
           "npair_eval_workspace_bytes", "npair_eval_create", "npair_eval_destroy", "npair_eval_last_error", "npair_eval_rank",
           "npair_eval_best_positive", "npair_eval_count", "npair_eval_map_at_r", "npair_eval_map_at_r_bytes",
           "npair_eval_kmeans", "npair_eval_kmeans_bytes", "npair_eval_kmeans_seed", "npair_eval_kmeans_seed_bytes", "npair_eval_knn", "npair_eval_knn_bytes",
           "npair_eval_class_batches", "npair_eval_class_batches_bytes"]

_LIB = None


def kernel_launches() -> int:
    """Cumulative number of CUDA kernels libnpair_b200 has launched in this process (include/npair_b200.h)."""
    return int(lib().npair_kernel_launches())


class NpairError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"libnpair_b200: {ERRORS.get(code, code)}: {msg}")
        self.code = code


def lib():
    global _LIB
    if _LIB is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                              "(there is no CPU fallback)")
        L = C.CDLL(LIB_PATH)
        vp, fp = C.c_void_p, C.POINTER(C.c_float)
        L.npair_config_default.argtypes = [C.POINTER(NpairConfig), C.c_int32, C.c_int32]
        L.npair_config_default.restype = None
        L.npair_workspace_bytes.argtypes = [C.POINTER(NpairConfig)]
        L.npair_workspace_bytes.restype = C.c_size_t
        L.npair_nccl_unique_id.argtypes = [vp]
        L.npair_create.argtypes = [C.POINTER(NpairConfig), vp, C.POINTER(vp)]
        L.npair_create_with_comm.argtypes = [C.POINTER(NpairConfig), vp, C.POINTER(vp)]
        L.npair_destroy.argtypes = [vp]
        L.npair_destroy.restype = None
        L.npair_forward.argtypes = [vp, vp, vp, fp, vp]
        L.npair_create_memory.argtypes = [C.POINTER(NpairConfig), C.c_int32, C.POINTER(vp)]
        L.npair_memory_workspace_bytes.argtypes = [C.POINTER(NpairConfig), C.c_int32]
        L.npair_memory_workspace_bytes.restype = C.c_size_t
        L.npair_forward_memory.argtypes = [vp, vp, vp, vp, vp, C.c_int32, fp, vp]
        L.npair_create_memory_ring.argtypes = [C.POINTER(NpairConfig), C.c_int32, C.POINTER(vp)]
        L.npair_memory_ring_workspace_bytes.argtypes = [C.POINTER(NpairConfig), C.c_int32]
        L.npair_memory_ring_workspace_bytes.restype = C.c_size_t
        L.npair_forward_ring.argtypes = [vp, vp, vp, fp, vp]
        L.npair_forward_ring_async.argtypes = [vp, vp, vp, vp, vp]
        L.npair_memory_ring_read.argtypes = [vp, vp, vp, vp, vp]
        L.npair_memory_ring_load.argtypes = [vp, vp, vp, C.c_int64, vp]
        L.npair_backward.argtypes = [vp, C.c_float, vp, vp]
        L.npair_forward_backward.argtypes = [vp, vp, vp, C.c_float, vp, fp, vp]
        L.npair_set_anchor_io.argtypes = [vp, vp, vp]
        L.npair_kernel_launches.restype = C.c_ulonglong
        L.npair_forward_async.argtypes = [vp, vp, vp, vp, vp]
        L.npair_forward_memory_async.argtypes = [vp, vp, vp, vp, vp, C.c_int32, vp, vp]
        L.npair_backward_device_weight.argtypes = [vp, vp, vp, vp]
        L.npair_backward_memory.argtypes = [vp, C.c_float, vp, vp, vp]
        L.npair_backward_memory_device_weight.argtypes = [vp, vp, vp, vp, vp]
        L.npair_async_status.argtypes = [vp]
        L.npair_forward_gathered.argtypes = [vp, vp, vp, fp, vp]
        L.npair_backward_partial.argtypes = [vp, C.c_float, vp, vp, vp]
        L.npair_bwd_exchange_mode.argtypes = [vp]
        L.npair_row_scalars.argtypes = [vp, vp, vp]
        L.npair_backward_gathered.argtypes = [vp, C.c_float, vp, vp, vp]
        L.npair_profile_enable.argtypes = [vp, C.c_int]
        L.npair_profile_read.argtypes = [vp, fp]
        L.npair_last_error.argtypes = [vp]
        L.npair_last_error.restype = C.c_char_p
        L.npair_version.restype = C.c_char_p
        L.npair_debug_read.argtypes = [vp, C.c_int, fp, C.c_size_t]
        L.npair_debug_gemm.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, vp, vp, vp, vp]
        L.npair_l2normalize_forward.argtypes = [vp, C.c_int, C.c_int, vp, vp, vp]
        L.npair_l2normalize_backward.argtypes = [vp, vp, vp, C.c_int, C.c_int, vp, vp]
        i32 = C.c_int32
        L.npair_eval_workspace_bytes.argtypes = [i32, i32, i32, i32]
        L.npair_eval_workspace_bytes.restype = C.c_size_t
        L.npair_eval_create.argtypes = [i32, i32, i32, i32, i32, C.POINTER(vp)]
        L.npair_eval_destroy.argtypes = [vp]
        L.npair_eval_destroy.restype = None
        L.npair_eval_last_error.argtypes = [vp]
        L.npair_eval_last_error.restype = C.c_char_p
        L.npair_eval_rank.argtypes = [vp, vp, vp, i32, vp, vp, i32, i32, vp, vp]
        L.npair_eval_best_positive.argtypes = [vp, vp, vp, i32, vp, vp, i32, i32, i32, C.c_float, vp, vp]
        L.npair_eval_count.argtypes = [vp, vp, i32, vp, i32, i32, i32, C.c_float, vp, vp, vp]
        L.npair_eval_map_at_r.argtypes = [vp, vp, vp, i32, vp, vp, i32, i32, vp, vp, vp, vp, vp]
        L.npair_eval_map_at_r_bytes.argtypes = [i32, C.c_int64]
        L.npair_eval_map_at_r_bytes.restype = C.c_size_t
        L.npair_eval_kmeans.argtypes = [vp, vp, i32, i32, vp, i32, vp, vp, vp, vp, vp]
        L.npair_eval_kmeans_bytes.argtypes = [i32, i32, i32]
        L.npair_eval_kmeans_bytes.restype = C.c_size_t
        L.npair_eval_kmeans_seed.argtypes = [vp, vp, i32, i32, C.c_uint64, i32, vp, C.POINTER(C.c_uint64), vp]
        L.npair_eval_kmeans_seed_bytes.argtypes = [i32, i32, i32]
        L.npair_eval_kmeans_seed_bytes.restype = C.c_size_t
        L.npair_eval_knn.argtypes = [vp, vp, i32, vp, i32, i32, i32, C.c_float, i32, i32, vp, vp, vp]
        L.npair_eval_knn_bytes.argtypes = [i32, i32, i32]
        L.npair_eval_knn_bytes.restype = C.c_size_t
        L.npair_eval_class_batches.argtypes = [vp, vp, i32, vp, i32, i32, i32, vp, vp, vp]
        L.npair_eval_class_batches_bytes.argtypes = [i32, i32, i32]
        L.npair_eval_class_batches_bytes.restype = C.c_size_t
        _LIB = L
    return _LIB


def _ptr(t, what, numel=0, dim=None, row=None):
    """data_ptr() of a tensor the library reads or writes, which must be a contiguous CUDA float32 tensor of `dim` dimensions (when
    given) and at least `numel` elements; row: a 2-D tensor whose rows hold at least `row` floats.  Raises TypeError for any other kind
    of tensor and ValueError for one too small, before anything reaches the library: it would take a host pointer for a device one, or
    read a view as if it were contiguous."""
    import torch
    if not (isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == torch.float32 and t.is_contiguous()):
        raise TypeError(f"{what} must be a contiguous CUDA float32 tensor")
    dim = 2 if row is not None else dim
    if dim is not None and t.dim() != dim:
        raise TypeError(f"{what} must have {dim} dimension(s), got {t.dim()}")
    if row is not None:
        numel = t.shape[0] * row
    if t.numel() < numel:
        raise ValueError(f"{what} holds {t.numel()} floats, the call needs {numel}")
    return t.data_ptr()


def _stream():
    import torch
    return torch.cuda.current_stream().cuda_stream


def make_config(Q, D, world=1, rank=0, num_tops=5, margin_ident=0.0, margin_diff=0.0, identsn=-1.0, diffsn=-1.0,
                ap_region=LOCAL, ap_method=RAND, an_region=LOCAL, an_method=RAND, sim_precision=PREC_FP32_FP16X2,
                gemm_backend=GEMM_TCGEN05, device=-1, bwd_exchange=0, global_scope=0, normalize_input=0, grad_chunk_cols=0,
                flags=0, sim_block_rows=0) -> NpairConfig:
    """sim_block_rows > 0: row-block similarity mode with blocks of that many rows (rounded up to a multiple of 128), folded into
    flags; the library keeps one block of the Q x N similarity matrix instead of all of it (include/npair_b200.h)."""
    return NpairConfig(Q, D, world, rank, num_tops, margin_ident, margin_diff, identsn, diffsn, ap_region, ap_method,
                       an_region, an_method, sim_precision, gemm_backend, device, bwd_exchange, global_scope, normalize_input,
                       grad_chunk_cols, flags | sim_block_flags(sim_block_rows))


def nccl_unique_id() -> bytes:
    buf = C.create_string_buffer(128)
    rc = lib().npair_nccl_unique_id(buf)
    if rc:
        raise NpairError(rc, lib().npair_last_error(None).decode())
    return buf.raw


def memory_workspace_bytes(cfg: NpairConfig, memory_rows: int, ring: bool = False) -> int:
    """Device bytes a Context(cfg, memory_rows=memory_rows, ring=ring) allocates (npair_memory_workspace_bytes /
    npair_memory_ring_workspace_bytes; 0 for a refused configuration)."""
    f = lib().npair_memory_ring_workspace_bytes if ring else lib().npair_memory_workspace_bytes
    return int(f(C.byref(cfg), int(memory_rows)))


class Context:
    """One per rank.  forward()/backward() take torch CUDA tensors (device pointers) and return host scalars.
    memory_rows > 0: a cross-batch memory context (npair_create_memory, DESIGN 4.3) whose forward_memory takes up to that many rows.
    ring=True: a context that keeps its memory ring of memory_rows slots itself (npair_create_memory_ring, DESIGN 4.3.1): forward_ring,
    forward_ring_async, ring_read and ring_load."""

    def __init__(self, cfg: NpairConfig, nccl_id: bytes | None = None, memory_rows: int = 0, ring: bool = False):
        L = lib()
        self.cfg = cfg
        self.memory_rows = int(memory_rows)
        self.ring = bool(ring)
        self.last_m = 0                       # memory rows of the last forward (backward_memory's m x D output)
        self._h = C.c_void_p()
        idbuf = C.create_string_buffer(nccl_id, 128) if nccl_id is not None else None
        if self.ring:
            if nccl_id is not None:
                raise ValueError("a cross-batch memory context is a world-1 context: it takes no NCCL id")
            rc = L.npair_create_memory_ring(C.byref(cfg), self.memory_rows, C.byref(self._h))
        elif self.memory_rows > 0:
            if nccl_id is not None:
                raise ValueError("a cross-batch memory context is a world-1 context: it takes no NCCL id")
            rc = L.npair_create_memory(C.byref(cfg), self.memory_rows, C.byref(self._h))
        else:
            rc = L.npair_create(C.byref(cfg), idbuf, C.byref(self._h))
        if rc:
            raise NpairError(rc, L.npair_last_error(None).decode())

    def close(self):
        if self._h:
            lib().npair_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc):
        if rc:
            raise NpairError(rc, lib().npair_last_error(self._h).decode())

    def forward_ptr(self, feat_ptr: int, label_ptr: int, stream: int = 0):
        tops = (C.c_float * 5)()
        self._check(lib().npair_forward(self._h, feat_ptr, label_ptr, tops, stream))
        self.last_m = 0
        return [tops[i] for i in range(5)]

    def _rows(self, feat, label, rows=None):
        """Pointers of `rows` (default Q) rows of features and their labels."""
        rows = self.cfg.Q if rows is None else rows
        return _ptr(feat, "feat", rows * self.cfg.D), _ptr(label, "label", rows)

    def _grad(self, diff, what="diff"):
        return _ptr(diff, what, self.cfg.Q * self.cfg.D)

    def forward_backward(self, feat, label, loss_weight, diff):
        """npair_forward_backward: both passes, one host synchronisation."""
        tops = (C.c_float * 5)()
        self._check(lib().npair_forward_backward(self._h, *self._rows(feat, label), C.c_float(loss_weight), self._grad(diff), tops,
                                                 _stream()))
        self.last_m = 0
        return [tops[i] for i in range(5)]

    def forward(self, feat, label):
        return self.forward_ptr(*self._rows(feat, label), _stream())

    def forward_memory_ptr(self, feat_ptr: int, label_ptr: int, mem_feat_ptr, mem_label_ptr, m: int, stream: int = 0):
        tops = (C.c_float * 5)()
        self._check(lib().npair_forward_memory(self._h, feat_ptr, label_ptr, mem_feat_ptr, mem_label_ptr, int(m), tops, stream))
        self.last_m = int(m)
        return [tops[i] for i in range(5)]

    def _memory(self, mem_feat, mem_label, m):
        """Pointers of m memory rows and their labels; None for mem_feat None (the library refuses that for m > 0)."""
        if mem_feat is None:
            return None, None
        return _ptr(mem_feat, "mem_feat", int(m) * self.cfg.D), _ptr(mem_label, "mem_label", int(m))

    def forward_memory(self, feat, label, mem_feat, mem_label, m=None):
        """npair_forward_memory: the forward over [feat; mem_feat[:m]] with anchors feat only (m = None: all rows of mem_feat).
        mem_feat / mem_label may be None for m = 0; the library reads them during this call only."""
        if m is None:
            m = 0 if mem_feat is None else mem_feat.shape[0]
        return self.forward_memory_ptr(*self._rows(feat, label), *self._memory(mem_feat, mem_label, m), m, _stream())

    def backward(self, loss_weight, diff):
        self._check(lib().npair_backward(self._h, C.c_float(loss_weight), self._grad(diff), _stream()))

    # ---- asynchronous step (DESIGN 4.4): world 1, nothing read back on the host, capturable into a CUDA graph ----
    def forward_async(self, feat, label, tops_out):
        """npair_forward_async: enqueues the forward and returns at once; tops_out (5 fp32 on the device) receives the tops in stream
        order, all NaN on a device error (see async_status)."""
        self._check(lib().npair_forward_async(self._h, *self._rows(feat, label), _ptr(tops_out, "tops_out", 5), _stream()))
        self.last_m = 0
        return tops_out

    def forward_memory_async(self, feat, label, mem_feat, mem_label, m, tops_out):
        """npair_forward_memory_async: forward_memory with the tops written to tops_out as in forward_async."""
        self._check(lib().npair_forward_memory_async(self._h, *self._rows(feat, label), *self._memory(mem_feat, mem_label, m), int(m),
                                                     _ptr(tops_out, "tops_out", 5), _stream()))
        self.last_m = int(m)
        return tops_out

    # ---- the memory rows' gradient (DESIGN 4.6) ----
    def backward_memory(self, loss_weight, diff, mem_diff):
        """npair_backward_memory: after forward_memory(_async) with m rows, diff [Q, D] receives backward's bits and mem_diff (at least
        m x D floats) the memory rows' gradient (1/2)(lw/Q) G[:, Q:]^T . x; m = 0 leaves mem_diff untouched."""
        self._check(lib().npair_backward_memory(self._h, C.c_float(loss_weight), self._grad(diff),
                                                _ptr(mem_diff, "mem_diff", self.last_m * self.cfg.D), _stream()))

    def backward_memory_device_weight(self, loss_weight, diff, mem_diff):
        """npair_backward_memory_device_weight: backward_memory with the loss weight read on the device from loss_weight (a one-element
        CUDA fp32 tensor), as backward_device_weight; capturable after forward_memory_async."""
        lw = _ptr(loss_weight, "loss_weight", 1)
        if loss_weight.numel() != 1:
            raise ValueError("loss_weight is one element")
        self._check(lib().npair_backward_memory_device_weight(self._h, lw, self._grad(diff),
                                                              _ptr(mem_diff, "mem_diff", self.last_m * self.cfg.D), _stream()))

    # ---- the context's own memory ring (ring=True, DESIGN 4.3.1) ----
    def forward_ring(self, feat, label):
        """npair_forward_ring: forward_memory over the ring's min(count, M) slots, then the batch's rows go into the ring."""
        tops = (C.c_float * 5)()
        self._check(lib().npair_forward_ring(self._h, *self._rows(feat, label), tops, _stream()))
        self.last_m = 0
        return [tops[i] for i in range(5)]

    def forward_ring_async(self, feat, label, tops_out):
        """npair_forward_ring_async: forward_ring with the tops written to tops_out as in forward_async; capturable once the ring is
        full."""
        self._check(lib().npair_forward_ring_async(self._h, *self._rows(feat, label), _ptr(tops_out, "tops_out", 5), _stream()))
        self.last_m = 0
        return tops_out

    def ring_read(self, rows, labels, count):
        """npair_memory_ring_read: the valid slots into rows [M, D] and labels [M] (the first min(count, M) of each), and the push count
        into count, a one-element CUDA int64 tensor; all in stream order."""
        import torch
        if not (isinstance(count, torch.Tensor) and count.is_cuda and count.dtype == torch.int64 and count.numel() >= 1):
            raise TypeError("count must be a CUDA int64 tensor of one element")
        M, D = self.memory_rows, self.cfg.D
        self._check(lib().npair_memory_ring_read(self._h, _ptr(rows, "rows", M * D), _ptr(labels, "labels", M), count.data_ptr(),
                                                 _stream()))

    def ring_load(self, rows, labels, count):
        """npair_memory_ring_load: restores min(count, M) rows and labels in slot order and the push count (a host int); count = 0
        (rows and labels may be None) empties the ring."""
        count = int(count)
        m = min(max(count, 0), self.memory_rows)
        ptrs = (None, None) if rows is None else (_ptr(rows, "rows", m * self.cfg.D), _ptr(labels, "labels", m))
        self._check(lib().npair_memory_ring_load(self._h, *ptrs, count, _stream()))

    def backward_device_weight(self, loss_weight, diff):
        """npair_backward_device_weight: backward with the loss weight read on the device from loss_weight (a one-element CUDA fp32
        tensor), with the gradient bits of backward(float(loss_weight))."""
        lw = _ptr(loss_weight, "loss_weight", 1)
        if loss_weight.numel() != 1:
            raise ValueError("loss_weight is one element")
        self._check(lib().npair_backward_device_weight(self._h, lw, self._grad(diff), _stream()))

    def async_status(self):
        """npair_async_status: waits for the context's last call and raises NpairError (E_EMPTY_LIST, E_POS_RANGE, or E_ARG for an
        anchor weight outside [0, 1]) if an asynchronous forward since the previous status call met a device error; clears it."""
        self._check(lib().npair_async_status(self._h))

    def set_anchor_io(self, weight=None, row_loss=None):
        """npair_set_anchor_io (DESIGN 4.5): the next forwards read the Q anchor weights in [0, 1] from `weight` and write the Q
        unweighted per-anchor losses -log(A_i / T_i) to `row_loss`, in stream order; each a contiguous CUDA float32 tensor of Q elements,
        or None (unweighted / not written).  The library keeps the pointers until the next call: keep the tensors alive until then."""
        ptrs = []
        for t, what in ((weight, "weight"), (row_loss, "row_loss")):
            ptrs.append(None if t is None else _ptr(t, what, self.cfg.Q))
            if t is not None and t.numel() != self.cfg.Q:
                raise ValueError(f"{what} holds Q = {self.cfg.Q} floats, got {t.numel()}")
        self._check(lib().npair_set_anchor_io(self._h, *ptrs))

    def forward_gathered(self, feat_total, label_total):
        """npair_forward_gathered: the world's N = Q * world rows and labels, gathered by the caller."""
        tops = (C.c_float * 5)()
        self._check(lib().npair_forward_gathered(self._h, *self._rows(feat_total, label_total, self.cfg.Q * self.cfg.world), tops,
                                                 _stream()))
        self.last_m = 0
        return [tops[i] for i in range(5)]

    def backward_partial(self, loss_weight, local_half, total_half=None):
        """npair_backward_partial: local_half [Q, D], and at world > 1 total_half [N, D], this rank's addend of the all-reduce."""
        total = None if total_half is None else _ptr(total_half, "total_half", self.cfg.Q * self.cfg.world * self.cfg.D)
        self._check(lib().npair_backward_partial(self._h, C.c_float(loss_weight), self._grad(local_half, "local_half"), total, _stream()))

    def bwd_exchange_mode(self):
        return lib().npair_bwd_exchange_mode(self._h)

    def row_scalars(self, out):
        """npair_row_scalars: the rank's Q row records, 8 floats each, into out."""
        self._check(lib().npair_row_scalars(self._h, _ptr(out, "out", 8 * self.cfg.Q), _stream()))

    def backward_gathered(self, loss_weight, rs_total, diff):
        """npair_backward_gathered: the backward from the world's row records rs_total (8 floats for each of the N rows)."""
        rs = _ptr(rs_total, "rs_total", 8 * self.cfg.Q * self.cfg.world)
        self._check(lib().npair_backward_gathered(self._h, C.c_float(loss_weight), rs, self._grad(diff), _stream()))

    def profile_enable(self, on=True):
        self._check(lib().npair_profile_enable(self._h, 1 if on else 0))

    def profile_read(self):
        ms = (C.c_float * 9)()
        self._check(lib().npair_profile_read(self._h, ms))
        return [ms[i] for i in range(9)]

    def debug_read(self, which: int, n: int):
        """npair_debug_read: n floats of introspection array `which` (0 = S, Q x N; 12 = the hit flags, 3 x Q; 10 = one float; 13 = the
        count k of ring tiles the last ring forward re-split, then the k tiles; else Q)."""
        import numpy as np
        out = np.zeros(n, dtype=np.float32)
        self._check(lib().npair_debug_read(self._h, which, out.ctypes.data_as(C.POINTER(C.c_float)), n))
        return out


def eval_workspace_bytes(max_queries: int, max_gallery: int, D: int, precision: int = PREC_FP32_FP16X2) -> int:
    """Device bytes an Evaluator of this capacity allocates (0 for invalid arguments)."""
    return int(lib().npair_eval_workspace_bytes(max_queries, max_gallery, D, precision))


def eval_map_at_r_bytes(nq: int, sum_r: int) -> int:
    """Device bytes Evaluator.map_at_r adds on top of the workspace for nq queries with sum_r positive pairs in all (0 if invalid)."""
    return int(lib().npair_eval_map_at_r_bytes(nq, sum_r))


def eval_kmeans_bytes(n: int, k: int, D: int) -> int:
    """Device bytes Evaluator.kmeans adds on top of the workspace for n points of dimension D in k clusters (0 if invalid)."""
    return int(lib().npair_eval_kmeans_bytes(n, k, D))


def eval_kmeans_seed_bytes(n: int, D: int, local_trials: int = 0) -> int:
    """Device bytes Evaluator.kmeans_seed adds on top of the workspace for n points of dimension D (local_trials 0: the default
    trials of k = n, an upper bound; 0 if invalid)."""
    return int(lib().npair_eval_kmeans_seed_bytes(n, D, local_trials))


def eval_knn_bytes(ng: int, k: int, block_rows: int = 0) -> int:
    """Device bytes Evaluator.knn adds on top of the workspace for a gallery of ng rows (block_rows 0: the default; 0 if invalid)."""
    return int(lib().npair_eval_knn_bytes(ng, k, block_rows))


def eval_class_batches_bytes(n_classes: int, pool_size: int, n_batches: int) -> int:
    """Device bytes Evaluator.class_batches adds on top of the workspace: the class set's whole S and the pools (0 if invalid)."""
    return int(lib().npair_eval_class_batches_bytes(n_classes, pool_size, n_batches))


CLASS_POOL_MAX = 16384   # NPAIR_EVAL_CLASS_POOL_MAX


class Evaluator:
    """Retrieval evaluation (include/npair_b200.h, DESIGN 8): the rank of every query's best positive among the gallery, computed on
    the tensor cores without storing the similarity matrix.  Takes contiguous CUDA fp32 tensors; results are int32 / fp32 CUDA
    tensors, produced asynchronously on the current stream."""

    def __init__(self, max_queries: int, max_gallery: int, D: int, precision: int = PREC_FP32_FP16X2, device: int = -1):
        L = lib()
        self.max_queries, self.max_gallery, self.D, self.precision = max_queries, max_gallery, D, precision
        self._h = C.c_void_p()
        rc = L.npair_eval_create(max_queries, max_gallery, D, precision, device, C.byref(self._h))
        if rc:
            raise NpairError(rc, L.npair_eval_last_error(None).decode())

    def close(self):
        if self._h:
            lib().npair_eval_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc):
        if rc:
            raise NpairError(rc, lib().npair_eval_last_error(self._h).decode())

    def _rows(self, x, what):
        """The pointer of x, a 2-D tensor of rows of D floats."""
        return _ptr(x, what, row=self.D)

    def rank(self, query, qlabel, gallery, glabel, self_offset=-1):
        """int32 rank[nq] (npair_eval_rank)."""
        import torch
        q, g = self._rows(query, "query"), self._rows(gallery, "gallery")
        nq, ng = query.shape[0], gallery.shape[0]
        ql, gl = _ptr(qlabel, "qlabel", nq, 1), _ptr(glabel, "glabel", ng, 1)
        rank = torch.empty(nq, dtype=torch.int32, device=query.device)
        self._check(lib().npair_eval_rank(self._h, q, ql, nq, g, gl, ng, self_offset, rank.data_ptr(), _stream()))
        return rank

    def best_positive(self, query, qlabel, gallery, glabel, absmax, self_offset=-1, gallery_row0=0):
        """Phase 1 on one gallery shard: fp32 best[nq], -inf where the shard holds no positive."""
        import torch
        q, g = self._rows(query, "query"), self._rows(gallery, "gallery")
        nq, ng = query.shape[0], gallery.shape[0]
        ql, gl = _ptr(qlabel, "qlabel", nq, 1), _ptr(glabel, "glabel", ng, 1)
        best = torch.empty(nq, dtype=torch.float32, device=query.device)
        self._check(lib().npair_eval_best_positive(self._h, q, ql, nq, g, gl, ng, self_offset, gallery_row0, C.c_float(absmax),
                                                   best.data_ptr(), _stream()))
        return best

    def count(self, query, gallery, cut, absmax, self_offset=-1, gallery_row0=0):
        """Phase 2 on one gallery shard: int32 count[nq] of the shard's columns >= cut (0 where cut is -inf)."""
        import torch
        q, g = self._rows(query, "query"), self._rows(gallery, "gallery")
        nq = query.shape[0]
        ct = _ptr(cut, "cut", nq, 1)
        count = torch.empty(nq, dtype=torch.int32, device=query.device)
        self._check(lib().npair_eval_count(self._h, q, nq, g, gallery.shape[0], self_offset, gallery_row0, C.c_float(absmax), ct,
                                           count.data_ptr(), _stream()))
        return count

    def knn(self, query, gallery, k, self_offset=-1, gallery_row0=0, absmax=-1.0, block_rows=0):
        """npair_eval_knn: each query's k nearest gallery rows, s descending, then global gallery index ascending (NaN last).  Returns
        (fp32 sim[nq, k], int32 index[nq, k]) with index = gallery_row0 + the row in `gallery`; absmax >= 0 for a gallery shard."""
        import torch
        q, g = self._rows(query, "query"), self._rows(gallery, "gallery")
        nq, dev = query.shape[0], query.device
        sim = torch.empty(nq, int(k), dtype=torch.float32, device=dev)
        index = torch.empty(nq, int(k), dtype=torch.int32, device=dev)
        self._check(lib().npair_eval_knn(self._h, q, nq, g, gallery.shape[0], self_offset, gallery_row0, C.c_float(absmax), int(k),
                                         block_rows, sim.data_ptr(), index.data_ptr(), _stream()))
        return sim, index

    def class_batches(self, class_emb, pools, n, scores=True):
        """npair_eval_class_batches (DESIGN 8.4): hard negative class mining over the rows of class_emb [C, D], one row per class.
        pools: host int array [b, P] of distinct class ids per row (numpy, a CPU tensor or nested lists); batch t seeds with pools[t][0]
        and adds, n - 1 times, the pool class whose largest similarity to the classes already picked is the largest (NaN last, ties to
        the lower pool position).  Returns (int32 batches[b, n], fp32 scores[b, n] with NaN for the seed, or None when scores=False)."""
        import numpy as np
        import torch
        p = np.asarray(pools.cpu() if isinstance(pools, torch.Tensor) else pools)
        if p.ndim != 2 or p.dtype.kind not in "iu":
            raise ValueError("pools must be a 2-D integer array [n_batches, pool_size]")
        if p.dtype != np.int32:
            if p.size and (p.min() < 0 or p.max() >= 2 ** 31):
                raise ValueError("pool entries must be class ids")   # the library checks them against n_classes
            p = p.astype(np.int32)
        p = np.ascontiguousarray(p)
        emb = self._rows(class_emb, "class_emb")
        nb, dev = p.shape[0], class_emb.device
        batches = torch.empty(nb, int(n), dtype=torch.int32, device=dev)
        sc = torch.empty(nb, int(n), dtype=torch.float32, device=dev) if scores else None
        self._check(lib().npair_eval_class_batches(self._h, emb, class_emb.shape[0], p.ctypes.data, p.shape[1], nb, int(n),
                                                   batches.data_ptr(), sc.data_ptr() if scores else None, _stream()))
        return batches, sc

    def map_at_r(self, query, qlabel, gallery, glabel, self_offset=-1):
        """npair_eval_map_at_r: fp64 map_r[nq] and r_precision[nq] (NaN where a query has no positive), int32 R[nq] and rank[nq]
        (rank as Evaluator.rank).  Synchronises with the host once, to size its positive-pair buffer."""
        import torch
        q, g = self._rows(query, "query"), self._rows(gallery, "gallery")
        nq, ng, dev = query.shape[0], gallery.shape[0], query.device
        ql, gl = _ptr(qlabel, "qlabel", nq, 1), _ptr(glabel, "glabel", ng, 1)
        map_r = torch.empty(nq, dtype=torch.float64, device=dev)
        r_prec = torch.empty(nq, dtype=torch.float64, device=dev)
        R = torch.empty(nq, dtype=torch.int32, device=dev)
        rank = torch.empty(nq, dtype=torch.int32, device=dev)
        self._check(lib().npair_eval_map_at_r(self._h, q, ql, nq, g, gl, ng, self_offset, map_r.data_ptr(), r_prec.data_ptr(),
                                              R.data_ptr(), rank.data_ptr(), _stream()))
        return {"map_r": map_r, "r_precision": r_prec, "R": R, "rank": rank}

    def kmeans(self, x, k, init_rows, max_iter):
        """npair_eval_kmeans (DESIGN 8.2): Lloyd's k-means of the rows of x into k clusters, centroid c starting as row init_rows[c].
        Returns {"assign": int32[n], "centroids": fp32[k, D] (those assign was computed against), "inertia": fp64 scalar tensor,
        "iterations": sweeps run, "changed": assignments the last sweep changed, "empty": empty clusters}.  Synchronises with the host
        once per iteration."""
        import torch
        xp = self._rows(x, "x")
        n, dev = x.shape[0], x.device
        init_rows = [int(r) for r in init_rows]
        if len(init_rows) != int(k):
            raise ValueError("init_rows must hold k row indices")
        rows = (C.c_int32 * int(k))(*init_rows)
        centroids = torch.empty(int(k), self.D, dtype=torch.float32, device=dev)
        assign = torch.empty(n, dtype=torch.int32, device=dev)
        inertia = torch.empty((), dtype=torch.float64, device=dev)
        stats = (C.c_int32 * 3)()
        self._check(lib().npair_eval_kmeans(self._h, xp, n, int(k), rows, int(max_iter), centroids.data_ptr(), assign.data_ptr(),
                                            inertia.data_ptr(), stats, _stream()))
        return {"assign": assign, "centroids": centroids, "inertia": inertia, "iterations": stats[0], "changed": stats[1],
                "empty": stats[2]}

    def kmeans_seed(self, x, k, seed, local_trials=0):
        """npair_eval_kmeans_seed (DESIGN 8.2): k-means++ seeding of the rows of x, local_trials trials per step (0: 2 + floor(ln k)),
        random numbers from SplitMix64 seeded with seed modulo 2^64.  Returns (rows, potential): the k row indices, a list that
        Evaluator.kmeans takes as init_rows, and the final potential phi (a Python int, in the fixed-point units of the header).
        Synchronises with the host once, at the end."""
        xp = self._rows(x, "x")
        rows = (C.c_int32 * max(int(k), 1))()
        phi = C.c_uint64(0)
        self._check(lib().npair_eval_kmeans_seed(self._h, xp, x.shape[0], int(k), C.c_uint64(int(seed) % 2 ** 64), int(local_trials),
                                                 rows, C.byref(phi), _stream()))
        return [rows[i] for i in range(int(k))], int(phi.value)


def debug_gemm(precision, backend, A, B):
    """C = A @ B.T through the split-operand GEMM (unit test hook)."""
    import torch
    a = _ptr(A, "A", dim=2)
    M, K = A.shape
    b = _ptr(B, "B", row=K)
    Nn = B.shape[0]
    Cout = torch.empty((M, Nn), dtype=torch.float32, device=A.device)
    rc = lib().npair_debug_gemm(precision, backend, M, Nn, K, a, b, Cout.data_ptr(), _stream())
    if rc:
        raise NpairError(rc, lib().npair_last_error(None).decode())
    return Cout


def l2normalize_forward(x):
    """y = x / ||x||_2 per row (npair_l2normalize_forward); returns (y, inv_norm) as CUDA tensors."""
    import torch
    xp = _ptr(x, "x", dim=2)
    y = torch.empty_like(x)
    inv = torch.empty(x.shape[0], dtype=torch.float32, device=x.device)
    rc = lib().npair_l2normalize_forward(xp, x.shape[0], x.shape[1], y.data_ptr(), inv.data_ptr(), _stream())
    if rc:
        raise NpairError(rc, lib().npair_last_error(None).decode())
    return y, inv


def l2normalize_backward(y, inv, dy):
    """dx of the rows of y (2-D) from their inv_norm and dy (npair_l2normalize_backward); dx has the shape of dy."""
    import torch
    yp = _ptr(y, "y", dim=2)
    rows, dim = y.shape
    ip, dyp = _ptr(inv, "inv", rows), _ptr(dy, "dy", rows * dim)
    dx = torch.empty_like(dy)
    rc = lib().npair_l2normalize_backward(yp, ip, dyp, rows, dim, dx.data_ptr(), _stream())
    if rc:
        raise NpairError(rc, lib().npair_last_error(None).decode())
    return dx
