"""ctypes binding of oracle/liboracle.so (TEST INFRASTRUCTURE ONLY; see npair_oracle.h).

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs import this.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from oracle import npair_oracle_np as onp

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


class NpoConfig(C.Structure):
    _fields_ = [("Q", C.c_int32), ("D", C.c_int32), ("world", C.c_int32), ("rank", C.c_int32), ("num_tops", C.c_int32),
                ("margin_ident", C.c_float), ("margin_diff", C.c_float), ("identsn", C.c_float), ("diffsn", C.c_float),
                ("ap_region", C.c_int32), ("ap_method", C.c_int32), ("an_region", C.c_int32), ("an_method", C.c_int32),
                ("accum_double", C.c_int32), ("faithful_sorts", C.c_int32), ("num_threads", C.c_int32)]


class NpoState(C.Structure):
    _fields_ = [(n, C.POINTER(C.c_float)) for n in
                ("S", "E", "sel", "temp1", "temp2", "min_within", "max_between", "max_all", "posi_thr", "nega_thr",
                 "ident_num", "diff_num", "A", "B", "T", "logv")]


def build(force: bool = False) -> str:
    so = os.path.join(_HERE, "liboracle.so")
    src = [os.path.join(_HERE, f) for f in ("npair_oracle.cpp", "npair_oracle.h")]
    if force or not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in src):
        subprocess.check_call(["make", "-C", _HERE, "-s"])
    return so


def lib():
    global _LIB
    if _LIB is None:
        so = os.path.join(_HERE, "liboracle.so")
        if not os.path.exists(so):
            build()
        L = C.CDLL(so)
        fp = C.POINTER(C.c_float)
        L.npo_state_floats.restype = C.c_size_t
        L.npo_state_floats.argtypes = [C.POINTER(NpoConfig)]
        L.npo_state_bind.argtypes = [C.POINTER(NpoConfig), fp, C.POINTER(NpoState)]
        L.npo_forward.argtypes = [C.POINTER(NpoConfig), fp, fp, fp, C.POINTER(NpoState), fp]
        L.npo_backward_partial.argtypes = [C.POINTER(NpoConfig), fp, C.POINTER(NpoState), C.c_float, fp, fp]
        L.npo_step_world.argtypes = [C.POINTER(NpoConfig), fp, fp, fp, C.c_float, fp, fp]
        L.npo_pos.restype = C.c_longlong
        L.npo_pos.argtypes = [C.c_float, C.c_size_t]
        L.npo_version.restype = C.c_char_p
        L.npo_l2normalize_forward.argtypes = [fp, C.c_int, C.c_int, fp, fp]
        L.npo_l2normalize_forward.restype = None
        L.npo_l2normalize_backward.argtypes = [fp, fp, fp, C.c_int, C.c_int, fp]
        L.npo_l2normalize_backward.restype = None
        _LIB = L
    return _LIB


def _fp(a):
    return None if a is None else a.ctypes.data_as(C.POINTER(C.c_float))


def make_config(Q, D, world=1, rank=0, num_tops=5, margin_ident=0.0, margin_diff=0.0, identsn=-1.0, diffsn=-1.0,
                ap_region=1, ap_method=2, an_region=1, an_method=2, accum_double=1, faithful_sorts=1, num_threads=0):
    return NpoConfig(Q, D, world, rank, num_tops, margin_ident, margin_diff, identsn, diffsn,
                     ap_region, ap_method, an_region, an_method, accum_double, faithful_sorts, num_threads)


class OracleError(RuntimeError):
    def __init__(self, code):
        super().__init__(f"oracle error {code}")
        self.code = code


def forward(x_total, label_total, cfg: NpoConfig, S_inject=None):
    """Returns (tops[5], state dict of numpy arrays)."""
    L = lib()
    x_total = np.ascontiguousarray(x_total, dtype=np.float32)
    label_total = np.ascontiguousarray(label_total, dtype=np.float32)
    Q, N = cfg.Q, cfg.Q * cfg.world
    assert x_total.shape == (N, cfg.D) and label_total.shape == (N,)
    if S_inject is not None:
        S_inject = np.ascontiguousarray(S_inject, dtype=np.float32)
        assert S_inject.shape == (Q, N)
    buf = np.zeros(L.npo_state_floats(C.byref(cfg)), dtype=np.float32)
    st = NpoState()
    L.npo_state_bind(C.byref(cfg), _fp(buf), C.byref(st))
    tops = np.zeros(5, dtype=np.float32)
    e = L.npo_forward(C.byref(cfg), _fp(x_total), _fp(label_total), _fp(S_inject), C.byref(st), _fp(tops))
    if e:
        raise OracleError(e)
    QN = Q * N
    names2d = ["S", "E", "sel", "temp1", "temp2"]
    names1d = ["min_within", "max_between", "max_all", "posi_thr", "nega_thr", "ident_num", "diff_num", "A", "B", "T", "logv"]
    out = {"_buf": buf, "_st": st}
    off = 0
    for n in names2d:
        out[n] = buf[off:off + QN].reshape(Q, N); off += QN
    for n in names1d:
        out[n] = buf[off:off + Q]; off += Q
    return tops, out


def step_world(x_total, label_total, cfg: NpoConfig, loss_weight=1.0, S_inject_all=None, want_grad=True, anchor_weight=None):
    """Emulated all-rank fwd(+bwd).  Returns (tops[world,5], dX[N,D] or None).  anchor_weight: the Q * world anchors' weights
    (DESIGN 4.5), see _weighted_step."""
    L = lib()
    x_total = np.ascontiguousarray(x_total, dtype=np.float32)
    label_total = np.ascontiguousarray(label_total, dtype=np.float32)
    N = cfg.Q * cfg.world
    assert x_total.shape == (N, cfg.D)
    if S_inject_all is not None:
        S_inject_all = np.ascontiguousarray(S_inject_all, dtype=np.float32)
        assert S_inject_all.shape == (N, N)
    if anchor_weight is not None:
        tops, dx = _weighted_step(x_total, label_total, cfg, loss_weight, S_inject_all, anchor_weight)
        return tops, dx if want_grad else None
    tops = np.zeros((cfg.world, 5), dtype=np.float32)
    dx = np.zeros((N, cfg.D), dtype=np.float32) if want_grad else None
    e = L.npo_step_world(C.byref(cfg), _fp(x_total), _fp(label_total), _fp(S_inject_all), C.c_float(loss_weight),
                         _fp(tops), _fp(dx))
    if e:
        raise OracleError(e)
    return tops, dx


def _weighted_step(x_total, label_total, cfg, loss_weight, S_inject_all, anchor_weight):
    """The weighted step on the C++ oracle's own backward: each rank's forward (npo_forward), anchor row i of its selected terms
    temp1 / temp2 scaled by w_i -- which scales W1, W2, W3 and so G by w_i --, npo_backward_partial (fp32 W1..W3 and its GEMMs),
    then npo_step_world's fp32 all-reduce and blend.  At w = 1: npo_step_world bit for bit."""
    L = lib()
    Q, D, world = cfg.Q, cfg.D, cfg.world
    N = Q * world
    w = np.asarray(anchor_weight, dtype=np.float32)
    tops = np.zeros((world, 5), dtype=np.float32)
    local = np.zeros((N, D), dtype=np.float32)
    total = np.zeros((N, D), dtype=np.float32)
    for r in range(world):
        rows = slice(r * Q, (r + 1) * Q)
        rcfg = NpoConfig.from_buffer_copy(cfg)
        rcfg.rank = r
        tops[r], st = forward(x_total, label_total, rcfg, None if S_inject_all is None else S_inject_all[rows])
        tops[r, 0] = onp.weighted_loss(st["logv"], w[rows], Q)
        st["temp1"][:] = (st["temp1"] * w[rows, None]).astype(np.float32)     # views into the state buffer the backward reads
        st["temp2"][:] = (st["temp2"] * w[rows, None]).astype(np.float32)
        lh = np.zeros((Q, D), dtype=np.float32)
        th = np.zeros((N, D), dtype=np.float32)
        e = L.npo_backward_partial(C.byref(rcfg), _fp(x_total), C.byref(st["_st"]), C.c_float(loss_weight), _fp(lh), _fp(th))
        if e:
            raise OracleError(e)
        local[rows] = lh
        total += th                                                            # the all-reduce, in rank order
    td = total * np.float32(np.float32(1.0) / np.float32(world))
    return tops, (np.float32(0.5) * td + np.float32(0.5) * local).astype(np.float32)


def pos(sn, size):
    return int(lib().npo_pos(C.c_float(sn), C.c_size_t(size)))


def l2normalize_forward(x):
    """(y, inv_norm) of the L2Normalize producer layer (usage/def.prototxt:115-120)."""
    x = np.ascontiguousarray(x, dtype=np.float32)
    y = np.empty_like(x)
    inv = np.empty(x.shape[0], dtype=np.float32)
    lib().npo_l2normalize_forward(_fp(x), x.shape[0], x.shape[1], _fp(y), _fp(inv))
    return y, inv


def l2normalize_backward(y, inv, dy):
    y = np.ascontiguousarray(y, dtype=np.float32); dy = np.ascontiguousarray(dy, dtype=np.float32)
    inv = np.ascontiguousarray(inv, dtype=np.float32)
    dx = np.empty_like(dy)
    lib().npo_l2normalize_backward(_fp(y), _fp(inv), _fp(dy), y.shape[0], y.shape[1], _fp(dx))
    return dx
