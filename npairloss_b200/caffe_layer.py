"""ctypes binding of libnpair_caffe.so: the Caffe-style NPairMultiClassLossLayer (mini-Caffe shim + C harness).
This is the reference-facing plugin surface: prototxt in, host Blobs in, five top scalars and bottom diff out."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libnpair_caffe.so")
_LIB = None

REGION = {0: "GLOBAL", 1: "LOCAL"}
METHOD = {0: "HARD", 1: "EASY", 2: "RAND", 3: "RELATIVE_HARD", 4: "RELATIVE_EASY"}


def lib():
    global _LIB
    if _LIB is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(f"{LIB_PATH} is missing: run __graft_entry__.build()")
        L = C.CDLL(LIB_PATH)
        vp, fp = C.c_void_p, C.POINTER(C.c_float)
        L.npc_net_create.restype = vp
        L.npc_net_create.argtypes = [C.c_char_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, vp, C.c_int, C.c_char_p, C.c_int]
        L.npc_net_destroy.argtypes = [vp]
        L.npc_net_destroy.restype = None
        L.npc_last_error.restype = C.c_char_p
        L.npc_num_tops.argtypes = [vp]
        L.npc_layer_type.argtypes = [vp]
        L.npc_layer_type.restype = C.c_char_p
        L.npc_layer_params.argtypes = [vp, fp]
        L.npc_layer_params.restype = None
        L.npc_loss_weight.argtypes = [vp, C.c_int]
        L.npc_loss_weight.restype = C.c_float
        L.npc_bottom_mutable_cpu_data.argtypes = [vp, C.c_int]
        L.npc_bottom_mutable_cpu_data.restype = fp
        L.npc_forward.argtypes = [vp, fp, fp]
        L.npc_backward.argtypes = [vp]
        L.npc_bottom_cpu_diff.argtypes = [vp]
        L.npc_bottom_cpu_diff.restype = fp
        L.npc_forward_cpu_mode.argtypes = [vp]
        L.npc_prefetch_enable.argtypes = [vp]
        L.npc_set_mutable_cpu_data.argtypes = [vp, C.c_int, C.c_int]
        L.npc_set_mutable_cpu_data.restype = fp
        L.npc_prefetch.argtypes = [vp, C.c_int]
        L.npc_step_set.argtypes = [vp, C.c_int, fp]
        L.npc_set_cpu_diff.argtypes = [vp, C.c_int]
        L.npc_set_cpu_diff.restype = fp
        L.npc_parse_only.argtypes = [C.c_char_p, fp, C.POINTER(C.c_int), C.POINTER(C.c_int), C.c_char_p, C.c_int]
        L.npc_parse_num_bottoms.argtypes = [C.c_char_p]
        L.npc_solver_run.argtypes = [C.c_char_p, C.c_char_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_uint, C.c_float, fp, C.c_int]
        L.npc_solver_last_error.restype = C.c_char_p
        _LIB = L
    return _LIB


def layer_prototxt(mining: dict, num_tops: int = 5, loss_weights=True, anchor_weights=False) -> str:
    """A layer block in the format of usage/def.prototxt:121-151; anchor_weights=True adds the third bottom of anchor weights."""
    tops = ["loss3/type_npair_mc", "loss3/type_npair_mc_retrieve_top1", "loss3/type_npair_mc_retrieve_top5",
            "loss3/type_npair_mc_retrieve_top10", "loss3/feature_asum"][:num_tops]
    lines = ["layer {", '  bottom: "feat_norm"', '  bottom: "label"'] + (['  bottom: "anchor_weight"'] if anchor_weights else [])
    lines += ['  name: "loss3/type_mb"', '  type: "NPairMultiClassLoss"']
    lines += [f'  top: "{t}"' for t in tops]
    if loss_weights:
        lines += ["  loss_weight: 1"] * num_tops
    lines += ["  npair_loss_param {",
              f"    margin_ident: {mining['margin_ident']}", f"    margin_diff: {mining['margin_diff']}",
              f"    identsn: {mining['identsn']}", f"    diffsn: {mining['diffsn']}",
              f"    ap_mining_region: {REGION[mining['ap_region']]}", f"    ap_mining_method: {METHOD[mining['ap_method']]}",
              f"    an_mining_region: {REGION[mining['an_region']]}", f"    an_mining_method: {METHOD[mining['an_method']]}",
              "  }", "}"]
    return "\n".join(lines)


def parse_only(prototxt: str):
    out = (C.c_float * 8)()
    nt, nl = C.c_int(0), C.c_int(0)
    err = C.create_string_buffer(512)
    n = lib().npc_parse_only(prototxt.encode(), out, C.byref(nt), C.byref(nl), err, 512)
    if n < 0:
        raise ValueError(err.value.decode())
    keys = ["margin_ident", "margin_diff", "identsn", "diffsn", "ap_region", "ap_method", "an_region", "an_method"]
    d = {k: (float(out[i]) if i < 4 else int(out[i])) for i, k in enumerate(keys)}
    return dict(n_layers=n, num_tops=nt.value, n_loss_weights=nl.value, num_bottoms=int(lib().npc_parse_num_bottoms(prototxt.encode())), **d)


class LayerError(RuntimeError):
    pass


class Layer:
    """NPairMultiClassLossLayer<float> set up from a prototxt with bottoms (num, channels, height, width) and (num); a layer block
    with a third bottom gets a (num) blob of anchor weights, bottom_data(2), initially all 1."""

    def __init__(self, prototxt: str, num: int, channels: int, height: int = 1, width: int = 1, world: int = 1, rank: int = 0,
                 nccl_id: bytes | None = None, sim_precision: int = -1):
        err = C.create_string_buffer(1024)
        idbuf = C.create_string_buffer(nccl_id, 128) if nccl_id is not None else None
        self._h = lib().npc_net_create(prototxt.encode(), num, channels, height, width, world, rank, idbuf, sim_precision, err, 1024)
        if not self._h:
            raise LayerError(err.value.decode())
        self.num, self.dim = num, channels * height * width
        self.num_tops = lib().npc_num_tops(self._h)

    def close(self):
        if getattr(self, "_h", None):
            lib().npc_net_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def type(self):
        return lib().npc_layer_type(self._h).decode()

    def loss_weight(self, t):
        return float(lib().npc_loss_weight(self._h, t))

    def bottom_data(self, i):
        """numpy view of bottom[i]'s pinned host mirror (mutable_cpu_data: marks it dirty -> next forward copies H2D)."""
        p = lib().npc_bottom_mutable_cpu_data(self._h, i)
        if not p:
            raise LayerError(lib().npc_last_error().decode())
        n = self.num * self.dim if i == 0 else self.num
        return np.ctypeslib.as_array(p, shape=(n,))

    def touch_bottoms(self):
        lib().npc_bottom_mutable_cpu_data(self._h, 0)
        lib().npc_bottom_mutable_cpu_data(self._h, 1)

    def forward(self):
        tops = (C.c_float * 5)()
        loss = C.c_float(0)
        if lib().npc_forward(self._h, tops, C.byref(loss)):
            raise LayerError(lib().npc_last_error().decode())
        return [tops[i] for i in range(5)], loss.value

    def backward(self):
        if lib().npc_backward(self._h):
            raise LayerError(lib().npc_last_error().decode())

    # ---- double-buffered bottoms with an asynchronous H2D prefetch (the role of Caffe's BasePrefetchingDataLayer) ----
    def prefetch_enable(self):
        if lib().npc_prefetch_enable(self._h):
            raise LayerError(lib().npc_last_error().decode())

    def set_data(self, s, i):
        """numpy view of bottom[i] of set s (0/1); marks it CPU-dirty."""
        p = lib().npc_set_mutable_cpu_data(self._h, s, i)
        if not p:
            raise LayerError(lib().npc_last_error().decode())
        n = self.num * self.dim if i == 0 else self.num
        return np.ctypeslib.as_array(p, shape=(n,))

    def prefetch(self, s):
        """New batch in set s (touch) and start its H2D copy on the copy stream."""
        lib().npc_set_mutable_cpu_data(self._h, s, 0)
        lib().npc_set_mutable_cpu_data(self._h, s, 1)
        if lib().npc_prefetch(self._h, s):
            raise LayerError(lib().npc_last_error().decode())

    def step_set(self, s):
        """Forward (tops on the host) + Backward on set s, ordered after the set's prefetch."""
        tops = (C.c_float * 5)()
        if lib().npc_step_set(self._h, s, tops):
            raise LayerError(lib().npc_last_error().decode())
        return [tops[i] for i in range(5)]

    def set_diff(self, s):
        p = lib().npc_set_cpu_diff(self._h, s)
        if not p:
            raise LayerError(lib().npc_last_error().decode())
        return np.ctypeslib.as_array(p, shape=(self.num, self.dim))

    def bottom_diff(self):
        p = lib().npc_bottom_cpu_diff(self._h)
        if not p:
            raise LayerError(lib().npc_last_error().decode())
        return np.ctypeslib.as_array(p, shape=(self.num, self.dim))

    def forward_cpu_mode(self):
        if lib().npc_forward_cpu_mode(self._h):
            raise LayerError(lib().npc_last_error().decode())

    def step_host(self, read_gradient=True):
        """One training-style step on HOST blobs: new batch in the bottoms (H2D), Forward (tops on the host), Backward.
        read_gradient=True also brings bottom[0]'s diff back to the host (cpu_diff); False leaves it in the device diff, where
        the upstream layer's Backward_gpu consumes it in a net."""
        self.touch_bottoms()
        tops, _ = self.forward()
        self.backward()
        if read_gradient:
            self.bottom_diff()
        return tops


def solver_run(net_prototxt: str, solver_prototxt: str, feature_dim: int, num_identities: int, imgs_per_identity: int = 4, iters: int = 0,
               seed: int = 1, noise: float = 2.5, max_rows: int = 4096):
    """Synthetic training loop inside the shim (SURVEY 8f-4): MultibatchData -> [synthetic trunk] -> L2Normalize -> NPairMultiClassLoss
    driven like `caffe train` with the solver prototxt's SGD settings.  Returns an array of rows
    [iter, weighted loss, top0 (loss), top1, top5, top10, feature_asum] logged every `display` iterations."""
    log = np.zeros((max_rows, 7), dtype=np.float32)
    n = lib().npc_solver_run(net_prototxt.encode(), solver_prototxt.encode(), feature_dim, num_identities, imgs_per_identity, iters, seed,
                             C.c_float(noise), log.ctypes.data_as(C.POINTER(C.c_float)), max_rows)
    if n < 0:
        raise LayerError(lib().npc_solver_last_error().decode())
    return log[:n]
