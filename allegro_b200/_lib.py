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
# MLP nonlinearity of the *_nl entries; ACT_SILU / ACT_MUL_DSILU / EPI_MUL_DSILU then mean phi / phi' of that nonlinearity
NL_SILU, NL_MISH, NL_GELU = 1, 2, 3
NOT_ELIGIBLE = -1
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
    "ab2_linear_nl": ([_i32, _i64, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _i32, _vp, _vp, _i32, _vp, _vp, _vp, _vp, _i32, _vp, _i64, _vp, _i32], C.c_int),
    "ab2_linear_packed_bytes": ([_i32, _i32, _i32], C.c_int64),
    "ab2_linear_pack": ([_i32, _i32, _i32, _vp, _vp, _vp], C.c_int),
    "ab2_mlp2_readout": ([_i32, _i32, _i64, _i32, _i32, _i32, _i32, _vp, _i64, _vp, _i64, _vp, _i64, _vp, _i64, _vp, _i64, _vp, _i64, _vp, _vp, _vp], C.c_int),
    "ab2_mlp2": ([_i32, _i32, _i64, _i32, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _i32, _vp, _vp, _vp, _vp, _vp], C.c_int),
    "ab2_mlp2_nl": ([_i32, _i32, _i64, _i32, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _i32, _vp, _vp, _vp, _vp, _vp, _i32], C.c_int),
    "ab2_mlp2_readout_nl": ([_i32, _i32, _i64, _i32, _i32, _i32, _i32, _vp, _i64, _vp, _i64, _vp, _i64, _vp, _i64, _vp, _i64, _vp, _i64, _vp, _vp, _vp, _i32],
                            C.c_int),
    "ab2_env_sum": ([_i32, _i32, _i64, _i32, _vp, _vp, _vp, _i64, _dbl, _vp, _vp], C.c_int),
    "ab2_env_bwd": ([_i32, _i32, _i64, _i64, _i32, _vp, _vp, _vp, _vp, _i64, _vp, _dbl, _vp, _i64, _vp, _vp], C.c_int),
    "ab2_tp_fwd": ([_i32, _i32, _i64, _i64, _i32, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _i32, _vp, _vp, _i64, _vp, _vp], C.c_int),
    "ab2_tp_bwd": ([_i32, _i32, _i64, _i64, _i32, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _i32, _vp, _vp, _i64, _vp, _vp, _vp, _i64, _vp, _vp, _vp], C.c_int),
    "ab2_tp_chain_fwd": ([_i32, _i32, _i64, _i64, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp], C.c_int),
    "ab2_tp_chain_bwd": ([_i32, _i32, _i64, _i64, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp], C.c_int),
    "ab2_edge_sum": ([_i32, _i64, _vp, _vp, _dbl, _vp, _vp], C.c_int),
    "ab2_edge_sum_bwd": ([_i32, _i64, _vp, _vp, _dbl, _vp, _vp], C.c_int),
    "ab2_force_scatter": ([_i32, _i64, _i64, _i64, _vp, _vp, _vp, _vp, _vp, _vp], C.c_int),
    "ab2_force_virial_scatter": ([_i32, _i64, _i64, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp], C.c_int),
    "ab2_transpose_ui": ([_i32, _i64, _i32, _i32, _vp, _vp, _i32, _vp], C.c_int),
    "ab2_edge_vec": ([_i32, _i32, _i64, _vp, _vp, _vp, _vp, _vp, _vp], C.c_int),
    "ab2_radial_fwd": ([_i32, _i64, _i32, _i32, _dbl, _vp, _vp, _vp, _vp, _vp, _i32, _vp, _vp, _vp, _vp, _vp, _vp], C.c_int),
    "ab2_radial_pq_fwd": ([_i32, _i64, _i32, _i32, _dbl, _vp, _vp, _vp, _vp, _vp, _i32, _vp, _vp, _vp, _vp], C.c_int),
    "ab2_radial_pq_bwd": ([_i32, _i64, _i32, _i32, _dbl, _vp, _vp, _vp, _vp, _vp, _i32, _vp, _vp, _vp, _vp, _vp, _vp], C.c_int),
    "ab2_radial_pq_bwd_nl": ([_i32, _i64, _i32, _i32, _dbl, _vp, _vp, _vp, _vp, _vp, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _i32], C.c_int),
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
    "ab2_p2p_push_rows_v": ([_i32, _i32, _i32, _vp, _vp, _i32, _dbl, _dbl, _dbl, _vp, _i32, _i32, _vp, _vp, _vp], C.c_int),
    "ab2_p2p_wait_unpack": ([_i32, _i32, _i32, _vp, _i32, _i32, _vp, _i32, _vp, _vp, _i32, _vp], C.c_int),
    "ab2_p2p_allreduce_energy": ([_vp, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp], C.c_int),
    "ab2_p2p_mailbox_bytes_ex": ([_i32, _i32, _i32], C.c_int64),
    "ab2_p2p_push_rows_w": ([_i32, _i32, _vp, _vp, _i32, _vp, _i32, _i32, _vp, _vp, _vp], C.c_int),
    "ab2_p2p_wait_unpack_w": ([_i32, _i32, _vp, _i32, _i32, _vp, _i32, _vp, _vp, _vp, _vp], C.c_int),
    "ab2_p2p_allreduce_vec": ([_vp, _i32, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp], C.c_int),
    "ab2_slab_plan_count": ([_i32, _i32, _i64, _vp, _vp, _vp, _i32, _i32, _dbl, _dbl, _dbl, _vp, _vp, _vp], C.c_int),
    "ab2_slab_plan_fill": ([_i64, _vp, _vp, _vp, _vp, _vp, _vp], C.c_int),
    "ab2_slab_plan_count_lattice": ([_i32, _i32, _i64, _vp, _vp, _vp, _i32, _i32, _dbl, _dbl, _vp, _vp, _vp], C.c_int),
    "ab2_nl_bin": ([_i32, _i64, _vp, _vp, _vp, _vp, _vp, _dbl, _vp, _vp], C.c_int),
    "ab2_nl_count": ([_i32, _i64, _vp, _vp, _vp, _vp, _vp, _dbl, _vp, _vp, _vp, _vp], C.c_int),
    "ab2_nl_fill": ([_i32, _i64, _vp, _vp, _vp, _vp, _vp, _dbl, _vp, _vp, _vp, _vp, _vp, _vp], C.c_int),
    "ab2_nl_lattice_bin": ([_i32, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _dbl, _vp, _vp], C.c_int),
    "ab2_nl_lattice_count": ([_i32, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _dbl, _vp, _vp, _vp, _vp], C.c_int),
    "ab2_nl_lattice_fill": ([_i32, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _dbl, _vp, _vp, _vp, _vp, _vp, _vp], C.c_int),
    "ab2_radial_bwd": ([_i32, _i64, _i32, _i32, _dbl, _vp, _vp, _vp, _vp, _vp, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp], C.c_int),
    "ab2_nl_frames_count": ([_i32, _i64, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _dbl, _vp, _vp], C.c_int),
    "ab2_nl_frames_fill": ([_i32, _i64, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _dbl, _vp, _vp, _vp, _vp], C.c_int),
    "ab2_nl_prune_count": ([_i32, _i64, _i64, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp], C.c_int),
    "ab2_nl_prune_fill": ([_i32, _i64, _i64, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp], C.c_int),
    "ab2_frame_scratch_elems": ([_i64, _i64], C.c_int64),
    "ab2_frame_sum": ([_i32, _i64, _i64, _vp, _vp, _vp, _i64, _vp, _vp], C.c_int),
    "ab2_frame_virial": ([_i32, _i64, _i64, _vp, _vp, _vp, _vp, _vp, _i64, _vp, _vp], C.c_int),
    "ab2_frame_heat_current": ([_i32, _i64, _i64, _vp, _vp, _vp, _vp, _vp, _i64, _vp, _vp], C.c_int),
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

    def cancel(self):
        """After the block: the call launched nothing (the kernel declined the case), so it is not counted."""
        PROF.launches -= self.n
        if PROF.enabled:
            key = self.name + "@" + _TAG[0]
            PROF.records[key].pop()
            if not PROF.records[key]:
                del PROF.records[key]


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
    nonlin: int = NL_SILU,
):
    """Out (+)= epi(act(cat(a_segs, -1)) @ W); a_segs / o_segs are 2-D row-strided views.
    ``W_packed`` (from ``linear_pack``) enables the wgmma tensor-core path.  ``nonlin`` (NL_*): the nonlinearity that
    ``act`` / ``epi`` apply (ab2_linear_nl); SiLU calls ab2_linear."""
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
    args = (DTYPE_ENUM[dt], M, K, N, na, a_ptr, a_ld, a_w, x_ptr, x_ld, act, _ptr(_contig(W, "W")), _ptr(W_packed), no, o_ptr, o_ld, o_w, o_acc,
            epi, _ptr(aux), aux_ld, _stream())
    with _timed("linear", 1):
        _check(load().ab2_linear(*args) if nonlin == NL_SILU else load().ab2_linear_nl(*args, nonlin))


def mlp2(
    a_segs: Sequence[torch.Tensor],
    W1: torch.Tensor,
    W2: torch.Tensor,
    o_segs: Sequence[torch.Tensor],
    pre: torch.Tensor,
    o_accum: Optional[Sequence[bool]] = None,
    backward: bool = False,
    W1_packed: Optional[torch.Tensor] = None,
    W2_packed: Optional[torch.Tensor] = None,
    nonlin: int = NL_SILU,
) -> bool:
    """Two-layer MLP with nonlinearity phi (``nonlin``, NL_*) in one kernel (ab2_mlp2 / ab2_mlp2_nl), A = cat(a_segs, -1):
    forward   pre = A @ W1 (written),  Out (+)= phi(pre) @ W2;
    backward  Out (+)= ((A @ W1) * phi'(pre)) @ W2   (A = Gout, W1 = W2_fwd^T, W2 = W1_fwd^T).
    A one-column backward (K = 1) takes W1 as it is (rank-1 first stage, no packed image).
    Returns False, with nothing computed, when the kernel does not take this case: the caller then runs two ``linear``
    calls."""
    M = a_segs[0].shape[0]
    K, H = W1.shape
    N = W2.shape[1]
    dt = W1.dtype
    rank1 = backward and K == 1
    if W2_packed is None or (W1_packed is None and not rank1):
        return False
    na, no = len(a_segs), len(o_segs)
    a_ptr = (C.c_void_p * na)()
    a_ld = (C.c_int64 * na)()
    a_w = (C.c_int32 * na)()
    for s, t in enumerate(a_segs):
        t, ld = _row_strided(t, f"A segment {s}") if t.shape[1] > 1 else (t, int(t.stride(0)))
        assert t.dtype == dt and t.shape[0] == M
        a_ptr[s], a_ld[s], a_w[s] = t.data_ptr(), ld, t.shape[1]
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
    pre, pre_ld = _row_strided(pre, "pre")
    assert pre.dtype == dt and tuple(pre.shape) == (M, H)
    timer = _timed("mlp2", 1)
    args = (DTYPE_ENUM[dt], int(backward), M, K, H, N, na, a_ptr, a_ld, a_w, _ptr(W1_packed), _ptr(W2_packed),
            _ptr(_contig(W1, "W1")) if rank1 else None, _ptr(pre), pre_ld, no, o_ptr, o_ld, o_w, o_acc, _stream())
    with timer:
        rc = load().ab2_mlp2(*args) if nonlin == NL_SILU else load().ab2_mlp2_nl(*args, nonlin)
    if rc == NOT_ELIGIBLE:
        timer.cancel()
        return False
    _check(rc)
    return True


def mlp2_readout(
    backward: bool,
    x: torch.Tensor,
    s: torch.Tensor,
    xl: Optional[torch.Tensor],
    pre_l: torch.Tensor,
    pre_r: torch.Tensor,
    ez: torch.Tensor,
    w2_ro: torch.Tensor,
    W_packed: Sequence[Optional[torch.Tensor]],
    S: int,
    nonlin: int = NL_SILU,
) -> bool:
    """Last latent MLP + readout MLP in one kernel (ab2_mlp2_readout / ab2_mlp2_readout_nl with the one nonlinearity
    ``nonlin`` of both MLPs), P = x.shape[1], U = s.shape[1], S the width of x_L, H the hidden width of both MLPs:
    forward   reads x = X[:, :P] and s; writes pre_l, xl = X[:, P:P+S], pre_r and ez = Ez;
              W_packed = packed (W1_lat [P+U][H], W2_lat [H][S], W1_ro[:P] [P][H], W1_ro[P:] [S][H]);
    backward  reads ez = gEz, pre_l and pre_r; writes x = gX[:, :P] and s = gs (xl is None);
              W_packed = packed (W1_ro^T [H][P+S], W2_lat^T [S][H], W1_lat^T [H][P+U]).
    w2_ro: the readout's H x 1 output layer.  Returns False, with nothing computed, when the kernel does not take this
    case (among others: latent and readout hidden widths that differ): the caller then runs the two MLPs separately."""
    if any(w is None for w in W_packed):
        return False
    M, P = x.shape
    U = s.shape[1]
    H = pre_l.shape[1]
    if pre_r.shape[1] != H or w2_ro.numel() != H:
        return False  # the kernel takes one hidden width for both MLPs
    if not backward and xl.shape[1] != S:
        raise ValueError(f"mlp2_readout: x_L has {xl.shape[1]} columns, S = {S}")
    # the packed images must be those of the shapes the library is told: it sizes every copy from P, S, U and H
    kn = [(H, P + S), (S, H), (H, P + U)] if backward else [(P + U, H), (H, S), (P, H), (S, H)]
    if len(W_packed) != len(kn):
        raise ValueError(f"mlp2_readout: {len(W_packed)} packed images, expected {len(kn)}")
    for i, ((k, n), w) in enumerate(zip(kn, W_packed)):
        if w.numel() * w.element_size() != (n + 31) // 32 * 32 * k * 4:
            raise ValueError(f"mlp2_readout: packed image {i} is not that of a [{k}][{n}] matrix")
    dt = x.dtype
    views = {}
    for name, t in (("x", x), ("s", s), ("xl", xl), ("pre_l", pre_l), ("pre_r", pre_r), ("ez", ez)):
        if t is None:
            views[name] = (None, 0)
            continue
        assert t.dtype == dt and t.shape[0] == M
        views[name] = (_ptr(t), int(t.stride(0))) if name == "ez" else (_ptr(_row_strided(t, name)[0]), int(t.stride(0)))
    assert ez.shape[1] == 1
    wp = (C.c_void_p * len(W_packed))(*[w.data_ptr() for w in W_packed])
    for w in W_packed:
        _ptr(w)
    timer = _timed("mlp2_readout", 1)
    args = (DTYPE_ENUM[dt], int(backward), M, P, S, U, H, *views["x"], *views["s"], *views["xl"], *views["pre_l"], *views["pre_r"],
            *views["ez"], wp, _ptr(_contig(w2_ro, "w2_ro")), _stream())
    with timer:
        rc = load().ab2_mlp2_readout(*args) if nonlin == NL_SILU else load().ab2_mlp2_readout_nl(*args, nonlin)
    if rc == NOT_ELIGIBLE:
        timer.cancel()
        return False
    _check(rc)
    return True


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


def tp_chain_takes(dtype, U: int) -> bool:
    """The storage types and widths ab2_tp_chain_fwd / ab2_tp_chain_bwd are built for: fp32, U = 32 or 64."""
    return dtype == torch.float32 and U in (32, 64)


def tp_chain_plan(dtype, U: int, cgw0: torch.Tensor, cgw1: torch.Tensor):
    """What ab2_tp_chain_fwd / ab2_tp_chain_bwd need besides the per-call tensors: the two layers' coupling weights as
    dense fp32 [nnz][U] device tensors.  None when the kernels do not take the case (``tp_chain_takes``, weights not on
    a CUDA device); decided on the host, without the library.  The caller has checked that both tables have the baked
    structure (Tab9x9x9, Tab9x9x1)."""
    if not tp_chain_takes(dtype, U) or not cgw0.is_cuda:
        return None
    return {"cgw0": cgw0.to(torch.float32).contiguous(), "cgw1": cgw1.to(torch.float32).contiguous(), "U": U}


def _chain_dense(t: torch.Tensor, shape, name: str):
    if tuple(t.shape) != tuple(shape) or t.dtype != torch.float32:
        raise ValueError(f"tp_chain: {name} is {tuple(t.shape)} {t.dtype}, expected {tuple(shape)} float32")
    return _ptr(_contig(t, name))


def tp_chain_fwd(plan, last: bool, row_ptr, ctr, gamma0, gamma1, Y, w0, s) -> bool:
    """Composed tensor product, forward (ab2_tp_chain_fwd): s [E][U] = the layer-0 scalar V_1[:, 0] (last = False) or
    the layer-1 output (last = True) from Y, w0 and the centres' gamma rows, without V_1.  Returns False, with nothing
    computed, when ``plan`` is None or the library declines."""
    if plan is None:
        return False
    E, U = s.shape
    N = gamma0.shape[0]
    args = [_chain_dense(gamma0, (N, 9, U), "gamma0"), _chain_dense(gamma1, (N, 9, U), "gamma1") if last else None,
            _chain_dense(Y, (E, 9), "Y"), _chain_dense(w0, (E, 3 * U), "w0"), _chain_dense(s, (E, U), "s")]
    timer = _timed("tp_chain_fwd", 1)
    with timer:
        rc = load().ab2_tp_chain_fwd(AB2_F32, int(last), N, E, U, _ptr(row_ptr), _ptr(ctr), _ptr(plan["cgw0"]), _ptr(plan["cgw1"]),
                                     *args, _stream())
    if rc == NOT_ELIGIBLE:
        timer.cancel()
        return False
    _check(rc)
    return True


def tp_chain_bwd(plan, first: bool, row_ptr, ctr, gamma0, gamma1, Y, w0, g1, g2, gw0, gY, ggamma) -> bool:
    """Composed tensor product, backward (ab2_tp_chain_bwd).  first = False: ggamma = the gradient of gamma1 from g2.
    first = True: gw0, gY (+=) and ggamma = the gradient of gamma0 from g1 and g2.  Returns False, with nothing
    computed, when ``plan`` is None or the library declines."""
    if plan is None:
        return False
    E, U = g2.shape
    N = gamma0.shape[0]
    args = [_chain_dense(gamma0, (N, 9, U), "gamma0"), _chain_dense(gamma1, (N, 9, U), "gamma1") if first else None,
            _chain_dense(Y, (E, 9), "Y"), _chain_dense(w0, (E, 3 * U), "w0"), _chain_dense(g1, (E, U), "g1") if first else None,
            _chain_dense(g2, (E, U), "g2"), _chain_dense(gw0, (E, 3 * U), "gw0") if first else None,
            _chain_dense(gY, (E, 9), "gY") if first else None, _chain_dense(ggamma, (N, 9, U), "ggamma")]
    timer = _timed("tp_chain_bwd", 1)
    with timer:
        rc = load().ab2_tp_chain_bwd(AB2_F32, int(first), N, E, U, _ptr(row_ptr), _ptr(ctr), _ptr(plan["cgw0"]), _ptr(plan["cgw1"]),
                                     *args, _stream())
    if rc == NOT_ELIGIBLE:
        timer.cancel()
        return False
    _check(rc)
    return True


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


def force_virial_scatter(vec: torch.Tensor, gvec: torch.Tensor, csr, num_atoms_total: int):
    """``force_scatter`` plus the centroid per-atom virial  W[a] = - sum over the edges whose neighbour is a of vec (x) gvec
    -> (F [n_total,3], W [n_total,3,3]) in gvec's dtype (ab2_force_virial_scatter; F bitwise force_scatter's)."""
    N = csr.row_ptr.shape[0] - 1
    E = csr.nbr.shape[0]
    assert vec.dtype == gvec.dtype and vec.shape == gvec.shape
    col_ptr, col_perm = csr.transposed(num_atoms_total)
    F = torch.empty(num_atoms_total, 3, dtype=gvec.dtype, device=gvec.device)
    W = torch.empty(num_atoms_total, 3, 3, dtype=gvec.dtype, device=gvec.device)
    with _timed("force_virial_scatter"):
        _check(load().ab2_force_virial_scatter(DTYPE_ENUM[gvec.dtype], N, num_atoms_total, E, _ptr(csr.row_ptr), _ptr(col_ptr), _ptr(col_perm),
                                               _ptr(_contig(vec, "vec")), _ptr(_contig(gvec, "gvec")), _ptr(F), _ptr(W), _stream()))
    return F, W


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


def neighbor_csr(pos: torch.Tensor, r_max: float, box, ncell, pbc=(True, True, True), origin=None, n_centres: Optional[int] = None):
    """Cell-list neighbour search on the device -> (row_ptr [n_centres+1] int32, nbr [E] int32, shift_vec [E,3] pos dtype).
    Orthorhombic ``box`` (3 lengths) cut into ``ncell`` (3 counts, from ``data.cell_grid``); centres are atoms
    [0, n_centres) (owned atoms first)."""
    box = [float(b) for b in box]
    origin = [0.0, 0.0, 0.0] if origin is None else [float(o) for o in origin]
    ncell = [int(c) for c in ncell]
    geom = ((C.c_double * 3)(*box), (C.c_double * 3)(*origin), (C.c_int32 * 3)(*[int(bool(p)) for p in pbc]), (C.c_int32 * 3)(*ncell),
            float(r_max))
    lib = load()
    return _cell_list_csr(pos, n_centres, ncell, geom, "nl", lib.ab2_nl_bin, lib.ab2_nl_count, lib.ab2_nl_fill)


def neighbor_csr_lattice(pos: torch.Tensor, r_max: float, rows, origin, ncell, reach, pbc=(True, True, True), n_centres: Optional[int] = None):
    """The same search on a general lattice (ab2_nl_lattice_bin / count / fill): ``rows`` the 3x3 binning rows, ``origin``
    fractional, ``ncell`` bins and ``reach`` bins walked either side per axis, all from ``data.lattice_grid``."""
    flat = [float(v) for row in rows for v in row]
    ncell = [int(c) for c in ncell]
    geom = ((C.c_double * 9)(*flat), (C.c_double * 3)(*[float(o) for o in origin]), (C.c_int32 * 3)(*[int(bool(p)) for p in pbc]),
            (C.c_int32 * 3)(*ncell), (C.c_int32 * 3)(*[int(k) for k in reach]), float(r_max))
    lib = load()
    return _cell_list_csr(pos, n_centres, ncell, geom, "nl_lattice", lib.ab2_nl_lattice_bin, lib.ab2_nl_lattice_count, lib.ab2_nl_lattice_fill)


def _cell_list_csr(pos, n_centres, ncell, geom, name, bin_fn, count_fn, fill_fn):
    """bin -> sort by bin -> count -> prefix sum -> fill; ``geom`` the host-side geometry arguments of the three calls."""
    n = pos.shape[0]
    n_centres = n if n_centres is None else int(n_centres)
    dt = DTYPE_ENUM[pos.dtype]
    pos = _contig(pos, "pos")
    cell_id = torch.empty(n, dtype=torch.int32, device=pos.device)
    with _timed(name + "_bin"):
        _check(bin_fn(dt, n, _ptr(pos), *geom, _ptr(cell_id), _stream()))
    order = torch.argsort(cell_id, stable=True).to(torch.int32)
    ncells = ncell[0] * ncell[1] * ncell[2]
    cell_start = torch.zeros(ncells + 1, dtype=torch.int32, device=pos.device)
    cell_start[1:] = torch.cumsum(torch.bincount(cell_id.long(), minlength=ncells), 0).to(torch.int32)
    counts = torch.empty(n_centres, dtype=torch.int32, device=pos.device)
    with _timed(name + "_count"):
        _check(count_fn(dt, n_centres, _ptr(pos), *geom, _ptr(cell_start), _ptr(order), _ptr(counts), _stream()))
    row_ptr = torch.zeros(n_centres + 1, dtype=torch.int32, device=pos.device)
    row_ptr[1:] = torch.cumsum(counts, 0).to(torch.int32)
    E = int(row_ptr[-1])
    nbr = torch.empty(E, dtype=torch.int32, device=pos.device)
    shift = torch.empty(E, 3, dtype=pos.dtype, device=pos.device)
    if E:
        with _timed(name + "_fill"):
            _check(fill_fn(dt, n_centres, _ptr(pos), *geom, _ptr(cell_start), _ptr(order), _ptr(row_ptr), _ptr(nbr), _ptr(shift), _stream()))
    return row_ptr, nbr, shift


def radial_pq_fwd(dtype, S: int, p_cut: float, vec, ctr, nbr, types, rmax_table, bessel_w, PQ) -> torch.Tensor:
    """out[z][c] = sum_n B_n(x_z) PQ[t_c*T+t_n][n][c]  (ab2_radial_pq_fwd)."""
    E = ctr.shape[0]
    out = torch.empty(E, S, dtype=dtype, device=vec.device)
    with _timed("radial_fwd"):
        _check(load().ab2_radial_pq_fwd(DTYPE_ENUM[dtype], E, S, bessel_w.numel(), float(p_cut), _ptr(vec), _ptr(ctr), _ptr(nbr), _ptr(types),
                                        _ptr(rmax_table), rmax_table.shape[0], _ptr(bessel_w), _ptr(_contig(PQ, "PQ")), _ptr(out), _stream()))
    return out


def radial_pq_bwd(dtype, S: int, p_cut: float, vec, ctr, nbr, types, rmax_table, bessel_w, PQ, g_out, aux, gvec, nonlin: int = NL_SILU):
    """gvec += (d out / d vec)^T (g_out * phi'(aux)) (aux None: plain g_out); phi the nonlinearity ``nonlin`` (NL_*)."""
    E = ctr.shape[0]
    args = (DTYPE_ENUM[dtype], E, S, bessel_w.numel(), float(p_cut), _ptr(vec), _ptr(ctr), _ptr(nbr), _ptr(types), _ptr(rmax_table),
            rmax_table.shape[0], _ptr(bessel_w), _ptr(_contig(PQ, "PQ")), _ptr(_contig(g_out, "g_out")),
            _ptr(_contig(aux, "aux")) if aux is not None else None, _ptr(gvec), _stream())
    with _timed("radial_bwd"):
        _check(load().ab2_radial_pq_bwd(*args) if nonlin == NL_SILU else load().ab2_radial_pq_bwd_nl(*args, nonlin))


# --------------------------------------------------------------------------- #
# slab decomposition plan (ab2_slab_plan_count / fill)
# --------------------------------------------------------------------------- #
def _slab_plan(mode: int, pos: torch.Tensor, image: Optional[torch.Tensor], box, rank: int, world: int, width: float, jump: float,
               r_list: float, n_lists: int, rows=None):
    """count -> prefix sum over the blocks -> fill; -> (lists [n_lists] int64, refused count).  The totals are the one
    device-to-host read.  ``rows`` (the 3x3 cell rows) selects ab2_slab_plan_count_lattice instead (``box`` and ``width``
    unused); it checks the cell even when there are no atoms."""
    n = pos.shape[0]
    if rows is not None:
        rowsa = (C.c_double * 9)(*[float(v) for row in rows for v in row])
        count = lambda cls, counts: load().ab2_slab_plan_count_lattice(  # noqa: E731
            DTYPE_ENUM[pos.dtype], mode, n, _ptr(_contig(pos, "pos")) if n else None, _ptr(image) if n else None, rowsa, int(rank), int(world),
            float(jump), float(r_list), _ptr(cls), _ptr(counts), _stream())
        if n == 0:
            _check(count(None, None))
    else:
        boxa = (C.c_double * 3)(*[float(b) for b in box])
        count = lambda cls, counts: load().ab2_slab_plan_count(  # noqa: E731
            DTYPE_ENUM[pos.dtype], mode, n, _ptr(_contig(pos, "pos")), _ptr(image), boxa, int(rank), int(world), float(width), float(jump),
            float(r_list), _ptr(cls), _ptr(counts), _stream())
    if n == 0:
        return [torch.empty(0, dtype=torch.int64, device=pos.device) for _ in range(n_lists)], 0
    nblk = (n + 255) // 256
    cls = torch.empty(n, dtype=torch.uint8, device=pos.device)
    counts = torch.empty(nblk, 4, dtype=torch.int32, device=pos.device)
    with _timed("slab_plan_count"):
        _check(count(cls, counts))
    incl = torch.cumsum(counts, 0, dtype=torch.int32)
    offsets = (incl - counts).contiguous()
    lists = [torch.empty(n, dtype=torch.int64, device=pos.device) for _ in range(n_lists)]
    ptrs = [_ptr(t) for t in lists] + [None] * (3 - n_lists)
    with _timed("slab_plan_fill"):
        _check(load().ab2_slab_plan_fill(n, _ptr(cls), _ptr(offsets), *ptrs, _stream()))
    totals = incl[-1].tolist()
    return [t[:c] for t, c in zip(lists, totals)], int(totals[3])


def slab_wrap_classify(pos: torch.Tensor, image: torch.Tensor, box, rank: int, world: int, width: float, jump: float = float("inf")):
    """Wrap ``pos`` [n,3] into [0, box) in place, add the boxes removed to ``image`` [n,3] int32, and classify every atom
    by its slab clamp(floor(x / width), 0, world - 1) -> (stay, to_left, to_right, n_refused): ascending int64 index
    lists, and the number of atoms bound for a non-adjacent slab or whose x before the wrap lay outside
    [lo - jump, hi + jump) (ab2_slab_plan_count / fill, mode 0)."""
    assert image.dtype == torch.int32 and image.shape == pos.shape
    (stay, left, right), refused = _slab_plan(0, pos, _contig(image, "image"), box, rank, world, width, jump, 0.0, 3)
    return stay, left, right, refused


def slab_faces(pos: torch.Tensor, box, rank: int, world: int, width: float, r_list: float):
    """Atoms of the slab within ``r_list`` of its faces -> (low, high): ascending int64 index lists of x < lo + r_list (the
    left neighbour's ghosts) and x >= hi - r_list (the right neighbour's), compared in fp64 (mode 1)."""
    (low, high), _ = _slab_plan(1, pos, None, box, rank, world, width, 0.0, r_list, 2)
    return low, high


def slab_wrap_classify_lattice(pos: torch.Tensor, image: torch.Tensor, rows, rank: int, world: int, jump: float = float("inf")):
    """``slab_wrap_classify`` for any regular cell with rows ``rows`` [3][3], cut along lattice row 0 in fractional
    coordinates s = pos . h^-1: wrap on all three axes (img_a = floor(s_a), pos -= sum_a img_a h_a in fp64, rounded once;
    image += img), classify by clamp(floor(s_0 world), 0, world - 1) -> (stay, to_left, to_right, n_refused); refused:
    a non-adjacent slab, or an unwrapped s_0 outside [lo - jump, hi + jump), ``jump`` in fractional units
    (ab2_slab_plan_count_lattice / ab2_slab_plan_fill, mode 0).  A singular or non-finite cell raises before any launch."""
    assert image.dtype == torch.int32 and image.shape == pos.shape
    (stay, left, right), refused = _slab_plan(0, pos, _contig(image, "image"), None, rank, world, 0.0, jump, 0.0, 3, rows=rows)
    return stay, left, right, refused


def slab_faces_lattice(pos: torch.Tensor, rows, rank: int, world: int, r_list: float):
    """``slab_faces`` for any regular cell: (low, high) = atoms with s_0 < lo + r_list / H_0 and s_0 >= hi - r_list / H_0,
    H_0 = |det h| / |h_1 x h_2| the height of the cell along row 0 (fp64; mode 1)."""
    (low, high), _ = _slab_plan(1, pos, None, None, rank, world, 0.0, 0.0, r_list, 2, rows=rows)
    return low, high


# --------------------------------------------------------------------------- #
# batches of frames (many small frames concatenated into one graph)
# --------------------------------------------------------------------------- #
def nl_frames(pos: torch.Tensor, frame_ptr: torch.Tensor, cell: torch.Tensor, inv_cell: torch.Tensor, pbc: torch.Tensor, r_max: float):
    """All-pairs search per frame (ab2_nl_frames_count / fill) -> (row_ptr [n+1] int32, nbr [E] int32, shift_vec [E,3] pos
    dtype).  frame_ptr [B+1] int32, cell / inv_cell [B,3,3] in the positions' dtype, pbc [B,3] int32, all on the device.
    Rows are ordered by neighbour, then by image (x, y, z) lexicographically.  The images searched on each side of every
    periodic axis (the kernels' nimg [B,3]) are computed here, on the host, from the cell as given
    (``data.frames_geometry``), so no frame reaches the kernels with an unbounded image range: a periodic frame whose cell
    is not regular, or that needs more than data.FRAMES_MAX_IMAGES images per pair, raises ValueError before any launch."""
    from . import data as D

    n, B = pos.shape[0], frame_ptr.shape[0] - 1
    dt = DTYPE_ENUM[pos.dtype]
    _, nimg = D.frames_geometry(cell.reshape(B, 3, 3), pbc.reshape(B, 3) != 0, r_max, pos.dtype)
    nimg = nimg.to(device=pos.device, dtype=torch.int32)
    pos = _contig(pos, "pos")
    args = (_ptr(_contig(frame_ptr, "frame_ptr")), _ptr(pos), _ptr(_contig(cell, "cell")), _ptr(_contig(inv_cell, "inv_cell")),
            _ptr(_contig(pbc, "pbc")), _ptr(nimg), float(r_max))
    counts = torch.empty(n, dtype=torch.int32, device=pos.device)
    with _timed("nl_frames_count"):
        _check(load().ab2_nl_frames_count(dt, n, B, *args, _ptr(counts), _stream()))
    row_ptr = torch.zeros(n + 1, dtype=torch.int32, device=pos.device)
    row_ptr[1:] = torch.cumsum(counts, 0).to(torch.int32)
    E = int(row_ptr[-1])
    nbr = torch.empty(E, dtype=torch.int32, device=pos.device)
    shift = torch.empty(E, 3, dtype=pos.dtype, device=pos.device)
    if E:
        with _timed("nl_frames_fill"):
            _check(load().ab2_nl_frames_fill(dt, n, B, *args, _ptr(row_ptr), _ptr(nbr), _ptr(shift), _stream()))
    return row_ptr, nbr, shift


def nl_prune(pos: torch.Tensor, row_ptr: torch.Tensor, nbr: torch.Tensor, shift: torch.Tensor, types: torch.Tensor, cut2: torch.Tensor):
    """Keep the edges shorter than their pair's list radius (ab2_nl_prune_count / fill) -> (row_ptr [n_centres+1] int32,
    nbr [E'] int32, shift [E',3] pos dtype), each row an ordered subsequence of the input row.  ``types`` [n] int32 in
    [0, T), ``cut2`` [T,T] fp64 squared radii (row = centre type), all on the device; the caller checks them
    (``data.prune_csr``).  No launch for zero centres or zero edges."""
    nc, E, T = row_ptr.shape[0] - 1, nbr.shape[0], cut2.shape[0]
    if nc == 0 or E == 0:
        return row_ptr.clone(), nbr.clone(), shift.clone()
    dt = DTYPE_ENUM[pos.dtype]
    assert shift.dtype == pos.dtype and types.dtype == torch.int32 and cut2.dtype == torch.float64
    args = (dt, nc, E, T, _ptr(_contig(pos, "pos")), _ptr(_contig(types, "types")), _ptr(_contig(cut2, "cut2")),
            _ptr(_contig(row_ptr, "row_ptr")), _ptr(_contig(nbr, "nbr")), _ptr(_contig(shift, "shift")))
    counts = torch.empty(nc, dtype=torch.int32, device=pos.device)
    with _timed("nl_prune_count"):
        _check(load().ab2_nl_prune_count(*args, _ptr(counts), _stream()))
    out_ptr = torch.zeros(nc + 1, dtype=torch.int32, device=pos.device)
    out_ptr[1:] = torch.cumsum(counts, 0).to(torch.int32)
    E2 = int(out_ptr[-1])
    out_nbr = torch.empty(E2, dtype=torch.int32, device=pos.device)
    out_shift = torch.empty(E2, 3, dtype=pos.dtype, device=pos.device)
    if E2:
        with _timed("nl_prune_fill"):
            _check(load().ab2_nl_prune_fill(*args, _ptr(out_ptr), _ptr(out_nbr), _ptr(out_shift), _stream()))
    return out_ptr, out_nbr, out_shift


def _frame_scratch(total: int, B: int, width: int, device):
    m = int(load().ab2_frame_scratch_elems(int(total), int(B))) * width
    return torch.empty(max(m, 1), dtype=torch.float64, device=device), m


def frame_sum(x: torch.Tensor, frame_ptr: torch.Tensor) -> torch.Tensor:
    """out[b] = sum of x over the atoms [frame_ptr[b], frame_ptr[b+1])  (ab2_frame_sum; fixed order, no atomics)."""
    B = frame_ptr.shape[0] - 1
    n = x.numel()
    out = torch.empty(B, dtype=x.dtype, device=x.device)
    scratch, m = _frame_scratch(n, B, 1, x.device)
    with _timed("frame_sum", 2):
        _check(load().ab2_frame_sum(DTYPE_ENUM[x.dtype], n, B, _ptr(_contig(frame_ptr, "frame_ptr")), _ptr(_contig(x, "x")), _ptr(scratch), m,
                                    _ptr(out), _stream()))
    return out


def frame_virial(vec: torch.Tensor, gvec: torch.Tensor, frame_ptr: torch.Tensor, row_ptr: torch.Tensor) -> torch.Tensor:
    """W[b] = sum over frame b's edges [row_ptr[frame_ptr[b]], row_ptr[frame_ptr[b+1]]) of vec (x) gvec -> [B,3,3] in
    vec's dtype  (ab2_frame_virial; fixed order, no atomics)."""
    B = frame_ptr.shape[0] - 1
    E = vec.shape[0]
    assert gvec.dtype == vec.dtype and gvec.shape == vec.shape
    W = torch.empty(B, 3, 3, dtype=vec.dtype, device=vec.device)
    scratch, m = _frame_scratch(E, B, 9, vec.device)
    with _timed("frame_virial", 2):
        _check(load().ab2_frame_virial(DTYPE_ENUM[vec.dtype], E, B, _ptr(_contig(frame_ptr, "frame_ptr")), _ptr(_contig(row_ptr, "row_ptr")),
                                       _ptr(_contig(vec, "vec")), _ptr(_contig(gvec, "gvec")), _ptr(scratch), m, _ptr(W), _stream()))
    return W


def frame_heat_current(e_atom: torch.Tensor, vel: torch.Tensor, W: torch.Tensor, frame_ptr: torch.Tensor) -> torch.Tensor:
    """J[b] = sum over the atoms [frame_ptr[b], frame_ptr[b+1]) of e_atom[a] vel[a] + W[a] @ vel[a] -> [B,3] in W's dtype
    (ab2_frame_heat_current; fixed order, no atomics).  ``vel`` is cast to W's dtype."""
    B = frame_ptr.shape[0] - 1
    n = W.shape[0]
    assert e_atom.numel() == n and vel.shape == (n, 3) and W.shape == (n, 3, 3)
    e_atom = e_atom.reshape(n).to(W.dtype).contiguous()
    vel = vel.to(W.dtype).contiguous()
    J = torch.empty(B, 3, dtype=W.dtype, device=W.device)
    scratch, m = _frame_scratch(n, B, 3, W.device)
    with _timed("frame_heat_current", 2):
        _check(load().ab2_frame_heat_current(DTYPE_ENUM[W.dtype], n, B, _ptr(_contig(frame_ptr, "frame_ptr")), _ptr(e_atom), _ptr(vel),
                                             _ptr(_contig(W, "W")), _ptr(scratch), m, _ptr(J), _stream()))
    return J
