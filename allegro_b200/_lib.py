"""ctypes binding of liballegro_b200.so (the C ABI declared in include/allegro_b200.h).

There is NO CPU fallback: if the shared library is missing, or a tensor is not on a CUDA
device, these wrappers raise.  PyTorch is used only for device memory and streams.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional, Sequence

import torch

from . import build as _build

AB2_F64, AB2_F32, AB2_BF16 = 0, 1, 2
ACT_NONE, ACT_SILU, ACT_MUL_DSILU = 0, 1, 2
EPI_NONE, EPI_MUL_DSILU = 0, 1
MAX_SEG = 4

DTYPE_ENUM = {torch.float64: AB2_F64, torch.float32: AB2_F32, torch.bfloat16: AB2_BF16}
ACC_DTYPE = {torch.float64: torch.float64, torch.float32: torch.float32, torch.bfloat16: torch.float32}

_LIB: Optional[C.CDLL] = None

_vp, _i64, _i32, _dbl = C.c_void_p, C.c_int64, C.c_int, C.c_double

_SIGNATURES = {
    "ab2_version": ([], C.c_int),
    "ab2_device_ok": ([], C.c_int),
    "ab2_last_error": ([], C.c_char_p),
    "ab2_set_option": ([C.c_char_p, _i32], C.c_int),
    "ab2_op_scatter_env": ([_i32, _i64, _i64, _dbl, _vp, _vp, _vp, _vp], C.c_int),
    "ab2_op_contract": ([_i32, _i32, _i64, _i32, _i32, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp], C.c_int),
    "ab2_op_gather_rows": ([_i32, _i64, _i64, _dbl, _vp, _vp, _vp, _vp], C.c_int),
    "ab2_op_contract_wgrad": ([_i32, _i64, _i32, _i32, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp], C.c_int),
    "ab2_sh_fwd": ([_i32, _i32, _i64, _vp, _vp, _vp], C.c_int),
    "ab2_sh_bwd": ([_i32, _i32, _i64, _vp, _vp, _vp, _i32, _vp], C.c_int),
    "ab2_linear": ([_i32, _i64, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _i32, _vp, _vp, _i32, _vp, _vp, _vp, _vp, _i32, _vp, _i64, _vp], C.c_int),
    "ab2_linear_packed_bytes": ([_i32, _i32, _i32], C.c_int64),
    "ab2_linear_pack": ([_i32, _i32, _i32, _vp, _vp, _vp], C.c_int),
    "ab2_env_sum": ([_i32, _i32, _i64, _i32, _vp, _vp, _vp, _i64, _dbl, _vp, _vp], C.c_int),
    "ab2_env_bwd": ([_i32, _i32, _i64, _i64, _i32, _vp, _vp, _vp, _vp, _i64, _vp, _dbl, _vp, _i64, _vp, _vp], C.c_int),
    "ab2_tp_fwd": ([_i32, _i32, _i64, _i64, _i32, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _i32, _vp, _vp, _i64, _vp, _vp], C.c_int),
    "ab2_tp_bwd": ([_i32, _i32, _i64, _i64, _i32, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _i32, _vp, _vp, _i64, _vp, _vp, _vp, _i64, _vp, _vp, _vp], C.c_int),
    "ab2_edge_sum": ([_i32, _i64, _vp, _vp, _dbl, _vp, _vp], C.c_int),
    "ab2_edge_sum_bwd": ([_i32, _i64, _vp, _vp, _dbl, _vp, _vp], C.c_int),
    "ab2_force_scatter": ([_i32, _i64, _i64, _i64, _vp, _vp, _vp, _vp, _vp, _vp], C.c_int),
    "ab2_transpose_ui": ([_i32, _i64, _i32, _i32, _vp, _vp, _i32, _vp], C.c_int),
    "ab2_edge_vec": ([_i32, _i32, _i64, _vp, _vp, _vp, _vp, _vp, _vp], C.c_int),
    "ab2_radial_fwd": ([_i32, _i64, _i32, _i32, _dbl, _vp, _vp, _vp, _vp, _vp, _i32, _vp, _vp, _vp, _vp, _vp, _vp], C.c_int),
    "ab2_radial_pq_fwd": ([_i32, _i64, _i32, _i32, _dbl, _vp, _vp, _vp, _vp, _vp, _i32, _vp, _vp, _vp, _vp], C.c_int),
    "ab2_radial_pq_bwd": ([_i32, _i64, _i32, _i32, _dbl, _vp, _vp, _vp, _vp, _vp, _i32, _vp, _vp, _vp, _vp, _vp, _vp], C.c_int),
    "ab2_zbl": ([_i32, _i64, _i32, _dbl, _dbl, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp], C.c_int),
    "ab2_p2p_mailbox_bytes": ([_i32, _i32], C.c_int64),
    "ab2_p2p_alloc": ([_i64, C.POINTER(C.c_void_p)], C.c_int),
    "ab2_p2p_free": ([_vp], C.c_int),
    "ab2_p2p_get_handle": ([_vp, _vp], C.c_int),
    "ab2_p2p_open_handle": ([_vp, C.POINTER(C.c_void_p)], C.c_int),
    "ab2_p2p_close_handle": ([_vp], C.c_int),
    "ab2_p2p_error": ([_vp, _i32, _i32, _vp], C.c_int),
    "ab2_p2p_begin": ([_vp, _vp], C.c_int),
    "ab2_p2p_push_rows": ([_i32, _i32, _i32, _vp, _vp, _i32, _dbl, _vp, _i32, _i32, _vp, _vp, _vp], C.c_int),
    "ab2_p2p_wait_unpack": ([_i32, _i32, _i32, _vp, _i32, _i32, _vp, _i32, _vp, _vp, _i32, _vp], C.c_int),
    "ab2_p2p_allreduce_energy": ([_vp, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp], C.c_int),
    "ab2_nl_bin": ([_i32, _i64, _vp, _vp, _vp, _vp, _vp, _dbl, _vp, _vp], C.c_int),
    "ab2_nl_count": ([_i32, _i64, _vp, _vp, _vp, _vp, _vp, _dbl, _vp, _vp, _vp, _vp], C.c_int),
    "ab2_nl_fill": ([_i32, _i64, _vp, _vp, _vp, _vp, _vp, _dbl, _vp, _vp, _vp, _vp, _vp, _vp], C.c_int),
    "ab2_radial_bwd": ([_i32, _i64, _i32, _i32, _dbl, _vp, _vp, _vp, _vp, _vp, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp], C.c_int),
}


def exported_symbols() -> Sequence[str]:
    return tuple(_SIGNATURES)


def lib_path() -> str:
    return _build.LIB


def load() -> C.CDLL:
    """Load the shared library (never builds implicitly on import paths that would hide a
    missing extension: a missing .so is an error unless ALLEGRO_B200_AUTOBUILD=1)."""
    global _LIB
    if _LIB is not None:
        return _LIB
    path = lib_path()
    if not os.path.exists(path):
        if os.environ.get("ALLEGRO_B200_AUTOBUILD", "0") == "1":
            _build.build()
        else:
            raise RuntimeError(
                f"allegro_b200: CUDA extension {path} not built. Run `python -m allegro_b200.build` "
                "(or __graft_entry__.build()).  There is no CPU fallback."
            )
    lib = C.CDLL(path)
    for name, (args, res) in _SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is missing
        fn.argtypes = args
        fn.restype = res
    _LIB = lib
    # tuning switches for experiments: ALLEGRO_B200_OPTIONS="env_split=4,tp_variant=0"
    for kv in filter(None, os.environ.get("ALLEGRO_B200_OPTIONS", "").split(",")):
        k, v = kv.split("=")
        if lib.ab2_set_option(k.strip().encode(), int(v)) != 0:
            raise RuntimeError(f"ALLEGRO_B200_OPTIONS: unknown option {k!r}")
    return lib


class _Prof:
    """Launch counter + optional per-kernel CUDA-event timing (bench.py's roofline leg).
    Events are recorded on the launching stream (torch's current stream)."""

    def __init__(self):
        self.launches = 0
        self.enabled = False
        self.records = {}

    def reset(self):
        self.launches = 0
        self.records = {}

    def times_ms(self):
        torch.cuda.synchronize()
        return {k: [a.elapsed_time(b) for a, b in v] for k, v in self.records.items()}


PROF = _Prof()
_TAG = [""]


def set_tag(tag: str):
    """Label subsequent kernel calls (only used to name bench.py's per-kernel timings)."""
    _TAG[0] = tag


class _timed:
    __slots__ = ("name", "n", "ev")

    def __init__(self, name: str, n_kernels: int = 1):
        self.name, self.n = name, n_kernels

    def __enter__(self):
        PROF.launches += self.n
        if PROF.enabled:
            self.ev = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
            self.ev[0].record()
        return self

    def __exit__(self, *a):
        if PROF.enabled:
            self.ev[1].record()
            PROF.records.setdefault(self.name + "@" + _TAG[0], []).append(self.ev)
        return False


def set_option(key: str, value: int):
    _check(load().ab2_set_option(key.encode(), int(value)))


def _check(rc: int):
    if rc != 0:
        msg = load().ab2_last_error()
        raise RuntimeError(f"allegro_b200 kernel call failed (rc={rc}): {msg.decode() if msg else '?'}")


def _ptr(t: Optional[torch.Tensor]):
    if t is None:
        return None
    if not t.is_cuda:
        raise RuntimeError("allegro_b200: tensor is not on a CUDA device (no CPU fallback on the hot path)")
    return C.c_void_p(t.data_ptr())


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _contig(t: torch.Tensor, name: str):
    if not t.is_contiguous():
        raise RuntimeError(f"allegro_b200: {name} must be contiguous")
    return t


def _row_strided(t: torch.Tensor, name: str):
    """2-D view with unit inner stride -> (tensor, leading dimension)."""
    if t.dim() != 2 or t.stride(1) != 1:
        raise RuntimeError(f"allegro_b200: {name} must be 2-D with unit inner stride")
    return t, int(t.stride(0))


# --------------------------------------------------------------------------- #
# thin typed wrappers
# --------------------------------------------------------------------------- #
def sh_fwd(vec: torch.Tensor, lmax: int) -> torch.Tensor:
    E = vec.shape[0]
    Y = torch.empty(E, (lmax + 1) ** 2, dtype=vec.dtype, device=vec.device)
    with _timed("sh_fwd"):
        _check(load().ab2_sh_fwd(DTYPE_ENUM[vec.dtype], lmax, E, _ptr(_contig(vec, "vec")), _ptr(Y), _stream()))
    return Y


def sh_bwd(vec: torch.Tensor, gY: torch.Tensor, lmax: int, out: Optional[torch.Tensor] = None, accumulate: bool = False):
    E = vec.shape[0]
    if out is None:
        out = torch.empty_like(vec)
        accumulate = False
    with _timed("sh_bwd"):
        _check(load().ab2_sh_bwd(DTYPE_ENUM[vec.dtype], lmax, E, _ptr(_contig(vec, "vec")), _ptr(_contig(gY, "gY")), _ptr(out), int(accumulate), _stream()))
    return out


def linear(
    a_segs: Sequence[torch.Tensor],
    W: torch.Tensor,
    o_segs: Sequence[torch.Tensor],
    o_accum: Optional[Sequence[bool]] = None,
    act: int = ACT_NONE,
    epi: int = EPI_NONE,
    aux: Optional[torch.Tensor] = None,
    W_packed: Optional[torch.Tensor] = None,
    a_aux: Optional[Sequence[Optional[torch.Tensor]]] = None,
):
    """Out (+)= epi(act(cat(a_segs, -1)) @ W); a_segs / o_segs are 2-D row-strided views.
    ``W_packed`` (from ``linear_pack``) enables the wgmma tensor-core path."""
    M = a_segs[0].shape[0]
    K, N = W.shape
    dt = W.dtype
    na, no = len(a_segs), len(o_segs)
    a_ptr = (C.c_void_p * na)()
    a_ld = (C.c_int64 * na)()
    a_w = (C.c_int32 * na)()
    for s, t in enumerate(a_segs):
        t, ld = _row_strided(t, f"A segment {s}")
        assert t.dtype == dt and t.shape[0] == M
        a_ptr[s], a_ld[s], a_w[s] = t.data_ptr(), ld, t.shape[1]
        _ptr(t)
    x_ptr = x_ld = None
    if a_aux is not None:
        assert act == ACT_MUL_DSILU and len(a_aux) == na
        x_ptr = (C.c_void_p * na)()
        x_ld = (C.c_int64 * na)()
        for s, t in enumerate(a_aux):
            if t is None:
                x_ptr[s], x_ld[s] = None, 0
            else:
                t, ld = _row_strided(t, f"A aux segment {s}")
                assert t.dtype == dt and t.shape == a_segs[s].shape
                x_ptr[s], x_ld[s] = t.data_ptr(), ld
                _ptr(t)
    o_ptr = (C.c_void_p * no)()
    o_ld = (C.c_int64 * no)()
    o_w = (C.c_int32 * no)()
    o_acc = (C.c_int32 * no)()
    for s, t in enumerate(o_segs):
        t, ld = _row_strided(t, f"output segment {s}")
        assert t.dtype == dt and t.shape[0] == M
        o_ptr[s], o_ld[s], o_w[s] = t.data_ptr(), ld, t.shape[1]
        o_acc[s] = int(bool(o_accum[s])) if o_accum is not None else 0
        _ptr(t)
    aux_ld = 0
    if aux is not None:
        aux, aux_ld = _row_strided(aux, "aux")
        assert aux.dtype == dt
    with _timed("linear", 1):
        _check(
            load().ab2_linear(
                DTYPE_ENUM[dt], M, K, N, na, a_ptr, a_ld, a_w, x_ptr, x_ld, act, _ptr(_contig(W, "W")), _ptr(W_packed), no, o_ptr, o_ld, o_w, o_acc, epi,
                _ptr(aux), aux_ld, _stream(),
            )
        )


def linear_pack(W: torch.Tensor) -> Optional[torch.Tensor]:
    """Packed bf16 (hi, lo) image of W[K][N] for the tensor-core path, or None if not eligible."""
    K, N = W.shape
    nbytes = int(load().ab2_linear_packed_bytes(DTYPE_ENUM[W.dtype], K, N))
    if nbytes == 0:
        return None
    packed = torch.empty(nbytes, dtype=torch.uint8, device=W.device)
    _check(load().ab2_linear_pack(DTYPE_ENUM[W.dtype], K, N, _ptr(_contig(W, "W")), _ptr(packed), _stream()))
    return packed


def env_sum(dtype, lmax: int, N: int, U: int, row_ptr, Y, w: torch.Tensor, sf: float, out: Optional[torch.Tensor] = None):
    w, w_ld = _row_strided(w, "w")
    D = (lmax + 1) ** 2
    if out is None:
        out = torch.empty(N, D, U, dtype=ACC_DTYPE[dtype], device=Y.device)
    with _timed("env_sum"):
        _check(load().ab2_env_sum(DTYPE_ENUM[dtype], lmax, N, U, _ptr(row_ptr), _ptr(_contig(Y, "Y")), _ptr(w), w_ld, float(sf), _ptr(out), _stream()))
    return out


def env_bwd(dtype, lmax: int, U: int, ctr, Y, w: torch.Tensor, ggamma, sf: float, gw: torch.Tensor, gY: torch.Tensor, row_ptr=None):
    w, w_ld = _row_strided(w, "w")
    gw, gw_ld = _row_strided(gw, "gw")
    E = Y.shape[0]
    with _timed("env_bwd", 1):
        _check(
            load().ab2_env_bwd(
                DTYPE_ENUM[dtype], lmax, ggamma.shape[0], E, U, _ptr(row_ptr), _ptr(ctr), _ptr(_contig(Y, "Y")), _ptr(w), w_ld,
                _ptr(_contig(ggamma, "ggamma")), float(sf),
                _ptr(gw), gw_ld, _ptr(_contig(gY, "gY")), _stream(),
            )
        )


def tp_fwd(dtype, lmax, N, E, U, d_in, d_out, tab, cgw, row_ptr, ctr, gamma, Vin, Y, w0, Vout):
    implicit = Vin is None
    w0_ld = 0
    if implicit:
        w0, w0_ld = _row_strided(w0, "w0")
    with _timed("tp_fwd", 1):
        _check(
            load().ab2_tp_fwd(
                DTYPE_ENUM[dtype], lmax, N, E, U, d_in, d_out, tab.shape[0], _ptr(tab), _ptr(cgw), _ptr(row_ptr), _ptr(ctr), _ptr(gamma),
                _ptr(Vin), int(implicit), _ptr(Y), _ptr(w0) if implicit else None, w0_ld, _ptr(Vout), _stream(),
            )
        )


def tp_bwd(dtype, lmax, N, E, U, d_in, d_out, tab, cgw, row_ptr, ctr, gamma, Vin, Y, w0, gVout, gVin, gw0, gY, ggamma):
    implicit = Vin is None
    w0_ld = gw0_ld = 0
    if implicit:
        w0, w0_ld = _row_strided(w0, "w0")
        gw0, gw0_ld = _row_strided(gw0, "gw0")
    with _timed("tp_bwd", 2):
        _check(
            load().ab2_tp_bwd(
                DTYPE_ENUM[dtype], lmax, N, E, U, d_in, d_out, tab.shape[0], _ptr(tab), _ptr(cgw), _ptr(row_ptr), _ptr(ctr), _ptr(gamma),
                _ptr(Vin), int(implicit), _ptr(Y), _ptr(w0) if implicit else None, w0_ld, _ptr(gVout), _ptr(gVin),
                _ptr(gw0) if implicit else None, gw0_ld, _ptr(gY) if implicit else None, _ptr(ggamma), _stream(),
            )
        )


def edge_sum(Ez: torch.Tensor, row_ptr: torch.Tensor, factor: float) -> torch.Tensor:
    N = row_ptr.shape[0] - 1
    Ei = torch.empty(N, dtype=Ez.dtype, device=Ez.device)
    with _timed("edge_sum"):
        _check(load().ab2_edge_sum(DTYPE_ENUM[Ez.dtype], N, _ptr(row_ptr), _ptr(_contig(Ez, "Ez")), float(factor), _ptr(Ei), _stream()))
    return Ei


def edge_sum_bwd(gEi: torch.Tensor, ctr: torch.Tensor, factor: float) -> torch.Tensor:
    E = ctr.shape[0]
    gEz = torch.empty(E, dtype=gEi.dtype, device=gEi.device)
    with _timed("edge_sum_bwd"):
        _check(load().ab2_edge_sum_bwd(DTYPE_ENUM[gEi.dtype], E, _ptr(ctr), _ptr(_contig(gEi, "gEi")), float(factor), _ptr(gEz), _stream()))
    return gEz


def force_scatter(gvec: torch.Tensor, csr, num_atoms_total: int) -> torch.Tensor:
    """F[a] = sum of gvec over the edges centred on a  -  sum over the edges whose neighbour is a
    (deterministic segmented sums over the CSR and its transpose, ``csr.transposed``)."""
    N = csr.row_ptr.shape[0] - 1
    E = csr.nbr.shape[0]
    col_ptr, col_perm = csr.transposed(num_atoms_total)
    F = torch.empty(num_atoms_total, 3, dtype=gvec.dtype, device=gvec.device)
    with _timed("force_scatter"):
        _check(load().ab2_force_scatter(DTYPE_ENUM[gvec.dtype], N, num_atoms_total, E, _ptr(csr.row_ptr), _ptr(col_ptr), _ptr(col_perm),
                                        _ptr(_contig(gvec, "gvec")), _ptr(F), _stream()))
    return F


def transpose_ui(x: torch.Tensor, to_internal: bool) -> torch.Tensor:
    """[E,U,d] (reference strided layout) <-> [E,d,U] (internal)."""
    E, a, b = x.shape
    U, d = (a, b) if to_internal else (b, a)
    out = torch.empty(E, d, U, dtype=x.dtype, device=x.device) if to_internal else torch.empty(E, U, d, dtype=x.dtype, device=x.device)
    with _timed("transpose_ui"):
        _check(load().ab2_transpose_ui(DTYPE_ENUM[x.dtype], E, U, d, _ptr(_contig(x, "x")), _ptr(out), int(to_internal), _stream()))
    return out


def op_scatter_env(x2: torch.Tensor, idxs: torch.Tensor, n: int, sf: float) -> torch.Tensor:
    E = x2.shape[0]
    row = x2[0].numel() if E else 0
    gamma = torch.zeros((n,) + tuple(x2.shape[1:]), dtype=x2.dtype, device=x2.device)
    with _timed("op_scatter_env"):
        _check(load().ab2_op_scatter_env(DTYPE_ENUM[x2.dtype], E, row, float(sf), _ptr(_contig(x2, "x2")), _ptr(_contig(idxs, "idxs")), _ptr(gamma), _stream()))
    return gamma


def op_gather_rows(src: torch.Tensor, idxs: torch.Tensor, sf: float) -> torch.Tensor:
    E = idxs.shape[0]
    row = src[0].numel()
    out = torch.empty((E,) + tuple(src.shape[1:]), dtype=src.dtype, device=src.device)
    with _timed("op_gather_rows"):
        _check(load().ab2_op_gather_rows(DTYPE_ENUM[src.dtype], E, row, float(sf), _ptr(_contig(src, "src")), _ptr(_contig(idxs, "idxs")), _ptr(out), _stream()))
    return out


def op_contract(mode: int, U, d1, d2, dout, tab, cgw, a, b, idxs, out):
    E = idxs.shape[0]
    with _timed("op_contract", 1):
        _check(
            load().ab2_op_contract(
                DTYPE_ENUM[a.dtype], mode, E, U, d1, d2, dout, tab.shape[0], _ptr(tab), _ptr(cgw), _ptr(_contig(a, "a")), _ptr(_contig(b, "b")),
                _ptr(_contig(idxs, "idxs")), _ptr(out), _stream(),
            )
        )
    return out


def zbl(p_cut: float, qq: float, vec, ctr, nbr, types, Z, rmax_table, gvec: Optional[torch.Tensor]) -> torch.Tensor:
    """per-edge ZBL energies [E] (accumulate dtype); if ``gvec`` is given, dEz/dvec is added into it."""
    E = ctr.shape[0]
    Ez = torch.empty(E, dtype=vec.dtype, device=vec.device)
    with _timed("zbl"):
        _check(load().ab2_zbl(DTYPE_ENUM[vec.dtype], E, Z.shape[0], float(p_cut), float(qq), _ptr(_contig(vec, "vec")), _ptr(ctr), _ptr(nbr), _ptr(types),
                              _ptr(_contig(Z, "Z")), _ptr(_contig(rmax_table, "rmax_table")), _ptr(Ez), _ptr(gvec) if gvec is not None else None, _stream()))
    return Ez


def op_contract_wgrad(U, d1, d2, dout, tab, x1, gamma, gout, idxs) -> torch.Tensor:
    """gcgw[nnz][U] = sum_z x1 (x) gamma[idxs] (x) gout over the coupling table (training)."""
    E = idxs.shape[0]
    out = torch.zeros(tab.shape[0], U, dtype=x1.dtype, device=x1.device)
    with _timed("op_contract_wgrad", 1):
        _check(load().ab2_op_contract_wgrad(DTYPE_ENUM[x1.dtype], E, U, d1, d2, dout, tab.shape[0], _ptr(tab), _ptr(_contig(x1, "x1")),
                                            _ptr(_contig(gamma, "gamma")), _ptr(_contig(gout, "gout")), _ptr(_contig(idxs, "idxs")), _ptr(out), _stream()))
    return out


def edge_vec(pos: torch.Tensor, ctr, nbr, shift: Optional[torch.Tensor], acc_dtype) -> torch.Tensor:
    E = ctr.shape[0]
    vec = torch.empty(E, 3, dtype=acc_dtype, device=pos.device)
    if shift is not None:
        assert shift.dtype == pos.dtype
    with _timed("edge_vec"):
        _check(load().ab2_edge_vec(DTYPE_ENUM[pos.dtype], DTYPE_ENUM[acc_dtype], E, _ptr(_contig(pos, "pos")), _ptr(ctr), _ptr(nbr),
                                   _ptr(_contig(shift, "shift")) if shift is not None else None, _ptr(vec), _stream()))
    return vec


def radial_fwd(dtype, S_rc: int, p_cut: float, vec, ctr, nbr, types, rmax_table, bessel_w, Wb, cemb, nemb) -> torch.Tensor:
    E = ctr.shape[0]
    e0 = torch.empty(E, S_rc, dtype=dtype, device=vec.device)
    with _timed("radial_fwd"):
        _check(load().ab2_radial_fwd(DTYPE_ENUM[dtype], E, S_rc, bessel_w.numel(), float(p_cut), _ptr(vec), _ptr(ctr), _ptr(nbr), _ptr(types),
                                     _ptr(rmax_table), rmax_table.shape[0], _ptr(bessel_w), _ptr(Wb), _ptr(cemb), _ptr(nemb), _ptr(e0), _stream()))
    return e0


def radial_bwd(dtype, S_rc: int, p_cut: float, vec, ctr, nbr, types, rmax_table, bessel_w, Wb, cemb, nemb, g_e0, gvec):
    E = ctr.shape[0]
    with _timed("radial_bwd"):
        _check(load().ab2_radial_bwd(DTYPE_ENUM[dtype], E, S_rc, bessel_w.numel(), float(p_cut), _ptr(vec), _ptr(ctr), _ptr(nbr), _ptr(types),
                                     _ptr(rmax_table), rmax_table.shape[0], _ptr(bessel_w), _ptr(Wb), _ptr(cemb), _ptr(nemb),
                                     _ptr(_contig(g_e0, "g_e0")), _ptr(gvec), _stream()))


def neighbor_csr(pos: torch.Tensor, r_max: float, box, pbc=(True, True, True), origin=None, n_centres: Optional[int] = None):
    """Cell-list neighbour search on the device -> (row_ptr [n_centres+1] int32, nbr [E] int32, shift_vec [E,3] pos dtype).
    Orthorhombic ``box`` (3 lengths); centres are atoms [0, n_centres) (owned atoms first)."""
    n = pos.shape[0]
    n_centres = n if n_centres is None else int(n_centres)
    box = [float(b) for b in box]
    origin = [0.0, 0.0, 0.0] if origin is None else [float(o) for o in origin]
    ncell = [max(1, int(b // float(r_max))) for b in box]
    g_box, g_org = (C.c_double * 3)(*box), (C.c_double * 3)(*origin)
    g_pbc, g_nc = (C.c_int32 * 3)(*[int(bool(p)) for p in pbc]), (C.c_int32 * 3)(*ncell)
    dt = DTYPE_ENUM[pos.dtype]
    pos = _contig(pos, "pos")
    cell_id = torch.empty(n, dtype=torch.int32, device=pos.device)
    with _timed("nl_bin"):
        _check(load().ab2_nl_bin(dt, n, _ptr(pos), g_box, g_org, g_pbc, g_nc, float(r_max), _ptr(cell_id), _stream()))
    order = torch.argsort(cell_id, stable=True).to(torch.int32)
    ncells = ncell[0] * ncell[1] * ncell[2]
    cell_start = torch.zeros(ncells + 1, dtype=torch.int32, device=pos.device)
    cell_start[1:] = torch.cumsum(torch.bincount(cell_id.long(), minlength=ncells), 0).to(torch.int32)
    counts = torch.empty(n_centres, dtype=torch.int32, device=pos.device)
    with _timed("nl_count"):
        _check(load().ab2_nl_count(dt, n_centres, _ptr(pos), g_box, g_org, g_pbc, g_nc, float(r_max), _ptr(cell_start), _ptr(order), _ptr(counts), _stream()))
    row_ptr = torch.zeros(n_centres + 1, dtype=torch.int32, device=pos.device)
    row_ptr[1:] = torch.cumsum(counts, 0).to(torch.int32)
    E = int(row_ptr[-1])
    nbr = torch.empty(E, dtype=torch.int32, device=pos.device)
    shift = torch.empty(E, 3, dtype=pos.dtype, device=pos.device)
    if E:
        with _timed("nl_fill"):
            _check(load().ab2_nl_fill(dt, n_centres, _ptr(pos), g_box, g_org, g_pbc, g_nc, float(r_max), _ptr(cell_start), _ptr(order), _ptr(row_ptr),
                                      _ptr(nbr), _ptr(shift), _stream()))
    return row_ptr, nbr, shift


def radial_pq_fwd(dtype, S: int, p_cut: float, vec, ctr, nbr, types, rmax_table, bessel_w, PQ) -> torch.Tensor:
    """out[z][c] = sum_n B_n(x_z) PQ[t_c*T+t_n][n][c]  (ab2_radial_pq_fwd)."""
    E = ctr.shape[0]
    out = torch.empty(E, S, dtype=dtype, device=vec.device)
    with _timed("radial_fwd"):
        _check(load().ab2_radial_pq_fwd(DTYPE_ENUM[dtype], E, S, bessel_w.numel(), float(p_cut), _ptr(vec), _ptr(ctr), _ptr(nbr), _ptr(types),
                                        _ptr(rmax_table), rmax_table.shape[0], _ptr(bessel_w), _ptr(_contig(PQ, "PQ")), _ptr(out), _stream()))
    return out


def radial_pq_bwd(dtype, S: int, p_cut: float, vec, ctr, nbr, types, rmax_table, bessel_w, PQ, g_out, aux, gvec):
    E = ctr.shape[0]
    with _timed("radial_bwd"):
        _check(load().ab2_radial_pq_bwd(DTYPE_ENUM[dtype], E, S, bessel_w.numel(), float(p_cut), _ptr(vec), _ptr(ctr), _ptr(nbr), _ptr(types),
                                        _ptr(rmax_table), rmax_table.shape[0], _ptr(bessel_w), _ptr(_contig(PQ, "PQ")), _ptr(_contig(g_out, "g_out")),
                                        _ptr(_contig(aux, "aux")) if aux is not None else None, _ptr(gvec), _stream()))
