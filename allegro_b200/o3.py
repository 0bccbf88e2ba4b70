"""Host-side O(3) bookkeeping and constant tables for the CUDA kernels.

Setup-time only (runs once per model build, on the CPU): irreps algebra, the real-basis
Wigner-3j table generator and the per-layer sparse coupling tables the CUDA kernels consume.
Everything numeric here ends up as an *input buffer* of a kernel, so swapping in tables
produced by a real e3nn install is a data change, not a kernel change.

Reference behaviour mirrored (citations into /root/reference):
  * irreps selection rule / instruction order: allegro/nn/_strided/_contract.py:50-57
  * w3j table with "component" normalisation sqrt(2 l_out + 1): _contract.py:95-119
  * layer irreps build + pruning: allegro/nn/_allegro.py:101-160
  * e3nn conventions (not vendored by the reference): real SH basis with y polar,
    change of basis with (-i)^l phase, Frobenius-normalised 3j.
"""
from __future__ import annotations

import math
import re
from functools import lru_cache
from typing import List, Optional, Sequence, Tuple

__all__ = ["Irrep", "Irreps", "wigner_3j", "tp_path_exists", "allegro_layer_irreps", "CouplingTable", "build_coupling_table"]


class Irrep(tuple):
    """(l, p): p=+1 'e', p=-1 'o'."""

    def __new__(cls, l, p=None):
        if p is None:
            if isinstance(l, Irrep):
                return l
            if isinstance(l, str):
                m = re.fullmatch(r"\s*(\d+)\s*([eo])\s*", l)
                if not m:
                    raise ValueError(f"cannot parse irrep {l!r}")
                l, p = int(m.group(1)), (1 if m.group(2) == "e" else -1)
            else:
                l, p = l
        if l < 0 or p not in (1, -1):
            raise ValueError(f"bad irrep ({l},{p})")
        return super().__new__(cls, (int(l), int(p)))

    l = property(lambda self: self[0])  # noqa: E741
    p = property(lambda self: self[1])
    dim = property(lambda self: 2 * self[0] + 1)

    def __mul__(self, other) -> List["Irrep"]:
        other = Irrep(other)
        return [Irrep(l, self.p * other.p) for l in range(abs(self.l - other.l), self.l + other.l + 1)]

    def __repr__(self):
        return f"{self.l}{'e' if self.p == 1 else 'o'}"


class Irreps(tuple):
    """Ordered (mul, Irrep) list; accepts 'e3nn strings' such as "1x0e+1x1o" or "0e + 1o"."""

    def __new__(cls, spec=None):
        if isinstance(spec, Irreps):
            return spec
        items = []
        if spec is None:
            spec = ()
        if isinstance(spec, str):
            for term in filter(None, (t.strip() for t in spec.split("+"))):
                if "x" in term:
                    mul, ir = term.split("x")
                    items.append((int(mul), Irrep(ir)))
                else:
                    items.append((1, Irrep(term)))
        else:
            for it in spec:
                if isinstance(it, (str, Irrep)):
                    items.append((1, Irrep(it)))
                else:
                    mul, ir = it
                    items.append((int(mul), Irrep(ir)))
        return super().__new__(cls, items)

    @staticmethod
    def spherical_harmonics(lmax: int, p: int = -1) -> "Irreps":
        return Irreps([(1, (l, p**l)) for l in range(lmax + 1)])

    dim = property(lambda self: sum(m * ir.dim for m, ir in self))
    num_irreps = property(lambda self: sum(m for m, _ in self))
    lmax = property(lambda self: max(ir.l for _, ir in self))

    def slices(self) -> List[slice]:
        out, i = [], 0
        for m, ir in self:
            out.append(slice(i, i + m * ir.dim))
            i += m * ir.dim
        return out

    def comp_to_irrep(self) -> List[int]:
        """index of the irrep each component belongs to (the reference's _rtoi map)."""
        out = []
        for r, (m, ir) in enumerate(self):
            out += [r] * (m * ir.dim)
        return out

    def __contains__(self, ir) -> bool:
        ir = Irrep(ir)
        return any(i == ir for _, i in self)

    def __getitem__(self, i):
        if isinstance(i, slice):
            return Irreps(tuple.__getitem__(self, i))
        return tuple.__getitem__(self, i)

    def __repr__(self):
        return "+".join(f"{m}x{ir}" for m, ir in self)


# --------------------------------------------------------------------------- #
# Wigner 3j (real basis).  Pure-python complex arithmetic, exploiting that each row of the
# real->complex change of basis has at most two entries.
# --------------------------------------------------------------------------- #
def _fact(n: int) -> int:
    return math.factorial(n)


def _cg(j1: int, m1: int, j2: int, m2: int, j3: int, m3: int) -> float:
    if m1 + m2 != m3 or not (abs(j1 - j2) <= j3 <= j1 + j2):
        return 0.0
    pref = (2 * j3 + 1) * _fact(j3 + j1 - j2) * _fact(j3 - j1 + j2) * _fact(j1 + j2 - j3)
    pref *= _fact(j3 + m3) * _fact(j3 - m3)
    den = _fact(j1 + j2 + j3 + 1) * _fact(j1 - m1) * _fact(j1 + m1) * _fact(j2 - m2) * _fact(j2 + m2)
    lo = max(-j1 + j2 + m3, -j1 + m1, 0)
    hi = min(j2 + j3 + m1, j3 - j1 + j2, j3 + m3)
    s = 0.0
    for v in range(lo, hi + 1):
        num = _fact(j2 + j3 + m1 - v) * _fact(j1 - m1 + v)
        d = _fact(v) * _fact(j3 - j1 + j2 - v) * _fact(j3 + m3 - v) * _fact(v + j1 - j2 - m3)
        s += (-1) ** (v + j2 + m2) * num / d
    return math.sqrt(pref / den) * s


def _q_rows(l: int):
    """rows[m_index] = list of (real_index, coefficient) of the real->complex matrix Q_l[m, :]."""
    s = 1.0 / math.sqrt(2.0)
    ph = (-1j) ** l
    rows = []
    for m in range(-l, l + 1):
        if m < 0:
            rows.append([(l + abs(m), ph * s), (l - abs(m), ph * (-1j) * s)])
        elif m == 0:
            rows.append([(l, ph * 1.0)])
        else:
            sg = (-1) ** m
            rows.append([(l + abs(m), ph * sg * s), (l - abs(m), ph * 1j * sg * s)])
    return rows


@lru_cache(maxsize=None)
def wigner_3j(l1: int, l2: int, l3: int) -> Tuple[Tuple[Tuple[float, ...], ...], ...]:
    """Nested tuples w[a][b][c] of shape (2l1+1, 2l2+1, 2l3+1), Frobenius norm 1."""
    d1, d2, d3 = 2 * l1 + 1, 2 * l2 + 1, 2 * l3 + 1
    q1, q2, q3 = _q_rows(l1), _q_rows(l2), _q_rows(l3)
    acc = [[[0j] * d3 for _ in range(d2)] for _ in range(d1)]
    for i1, m1 in enumerate(range(-l1, l1 + 1)):
        for i2, m2 in enumerate(range(-l2, l2 + 1)):
            m3 = m1 + m2
            if abs(m3) > l3:
                continue
            c = _cg(l1, m1, l2, m2, l3, m3)
            if c == 0.0:
                continue
            for a, qa in q1[i1]:
                for b, qb in q2[i2]:
                    for cc, qc in q3[l3 + m3]:
                        acc[a][b][cc] += qa * qb * qc.conjugate() * c
    nrm = math.sqrt(sum(abs(v) ** 2 for pl in acc for row in pl for v in row))
    out = []
    for pl in acc:
        rows = []
        for row in pl:
            vals = []
            for v in row:
                if abs(v.imag) > 1e-10:
                    raise AssertionError("3j not real in this basis")
                x = v.real / nrm
                vals.append(0.0 if abs(x) < 1e-14 else x)
            rows.append(tuple(vals))
        out.append(tuple(rows))
    return tuple(out)


def tp_path_exists(irreps_a, irreps_b, ir_out) -> bool:
    ir_out = Irrep(ir_out)
    return any(ir_out in (a * b) for _, a in Irreps(irreps_a) for _, b in Irreps(irreps_b))


def allegro_layer_irreps(input_irreps, allowed, num_layers: int):
    """Per-layer TP irreps: forward build then backward pruning (allegro/nn/_allegro.py:101-160).
    Returns (irreps_in1 per layer, irreps_out per layer); the second TP operand is always
    ``input_irreps`` with multiplicity 1."""
    env = Irreps([(1, ir) for _, ir in Irreps(input_irreps)])
    allowed = Irreps(allowed)
    arg, chain = env, [env]
    for layer in range(num_layers):
        cand = Irreps([(1, (0, 1))]) if layer == num_layers - 1 else allowed
        arg = Irreps([(m, ir) for m, ir in cand if tp_path_exists(arg, env, ir)])
        chain.append(arg)
    out = chain[-1]
    pruned = [out]
    for arg in reversed(chain[:-1]):
        keep = []
        for m, a in arg:
            if any(any(i in out for i in a * e) for _, e in env):
                keep.append((m, a))
        out = Irreps(keep)
        pruned.append(out)
    chain = list(reversed(pruned))
    if chain[-1].lmax != 0:
        raise AssertionError("last layer must output scalars only")
    return chain[:-1], chain[1:]


class CouplingTable:
    """Sparse coupling table of one Contracter: entries (i, j, k, path, value) with
    value = w3j * sqrt(2 l_out + 1); instruction (path) order is (i_out, i_1, i_2) as in
    the reference (_contract.py:53-57)."""

    def __init__(self, irreps_in1, irreps_in2, irreps_out, instructions, entries, normalization):
        self.irreps_in1, self.irreps_in2, self.irreps_out = irreps_in1, irreps_in2, irreps_out
        self.instructions = instructions
        self.entries = entries  # list of (i, j, k, p, val)
        self.normalization = normalization
        self.dim1, self.dim2, self.dim_out = irreps_in1.dim, irreps_in2.dim, irreps_out.dim
        self.num_paths = len(instructions)
        self.is_ij_diagonal = self.dim1 == self.dim2 and all(e[0] == e[1] for e in entries)

    @property
    def nnz(self) -> int:
        return len(self.entries)


def build_coupling_table(irreps_in1, irreps_in2, irreps_out, instructions=None, irrep_normalization="component") -> CouplingTable:
    ir1, ir2, iro = Irreps(irreps_in1), Irreps(irreps_in2), Irreps(irreps_out)
    for irr in (ir1, ir2, iro):
        if not all(m == 1 for m, _ in irr):
            raise ValueError("strided layout needs multiplicity-1 irreps")
    if instructions is None:
        instructions = [
            (a, b, o)
            for o, (_, x) in enumerate(iro)
            for a, (_, y) in enumerate(ir1)
            for b, (_, z) in enumerate(ir2)
            if x in y * z
        ]
    if len(instructions) == 0:
        raise ValueError("No TP paths available")
    s1, s2, so = ir1.slices(), ir2.slices(), iro.slices()
    entries = []
    for p, (a, b, o) in enumerate(instructions):
        x, y, z = ir1[a][1], ir2[b][1], iro[o][1]
        if x.p * y.p != z.p or not (abs(x.l - y.l) <= z.l <= x.l + y.l):
            raise ValueError(f"instruction {(a, b, o)} violates O(3) selection rules")
        if irrep_normalization == "component":
            nrm = math.sqrt(2 * z.l + 1)
        elif irrep_normalization is None:
            nrm = 1.0
        else:
            raise NotImplementedError(irrep_normalization)
        w = wigner_3j(x.l, y.l, z.l)
        for i in range(x.dim):
            for j in range(y.dim):
                for k in range(z.dim):
                    v = w[i][j][k]
                    if v != 0.0:
                        entries.append((s1[a].start + i, s2[b].start + j, so[o].start + k, p, v * nrm))
    return CouplingTable(ir1, ir2, iro, list(instructions), entries, irrep_normalization)
