"""Spatial domain decomposition with a single-r_max halo (SURVEY.md section 8e).

Allegro is strictly local: E_i depends only on atoms within r_max of i
(/root/reference/tests/model/test_allegro.py:68-70; the environment sum only runs over edges
centred on i, allegro/nn/_strided/_contract.py:199-205).  So atoms are split into 1-D slabs
along lattice row 0 (x for an orthorhombic box; ``SlabGeometry``), one per rank / GPU; each rank evaluates the edges of its OWNED centres, with
neighbours taken from owned + ghost atoms in exactly the reference's ghost-atom data format
(ghosts appended after the locals, neighbour index >= N_local,
/root/reference/allegro/_compile.py:41-61).

Per force evaluation the only communication is
  1. forward halo : positions of boundary atoms -> neighbouring slabs' ghosts
  2. reverse halo : dE/dpos accumulated on ghosts -> added on the owning rank
  3. one all-reduce of the scalar total energy
through torch.distributed point-to-point ops (NCCL over NVLink on the GPU box, gloo in the
CPU tests).  There is no reference counterpart (the reference delegates this to LAMMPS' MPI).

The decomposition itself is set up from the global synthetic frame, which every rank can
generate deterministically, so set-up needs no communication.
"""
from __future__ import annotations

import math
import time
from typing import Callable, Dict, List, Optional, Tuple

import torch
import torch.distributed as dist

from . import data as D
from .calculator import prune_table


class SlabGeometry:
    """How a cell is cut into ``world`` slabs along lattice row 0: the one rule the static decomposition, the MD rebuild
    and both transports read.  Any regular cell (``data.is_regular_cell``) is accepted; anything else raises ValueError.

    * ``diagonal`` (zero off-diagonal entries, positive lengths): slabs along x of width Lx / world in length units, ghosts
      that cross the periodic x face shifted by -+Lx along x (ab2_slab_plan_count, ab2_p2p_push_rows).
    * Every other cell: fractional coordinates s = pos . h^-1, the inverse as nl_lattice_geom computes it.  Rank r owns
      s_0 in [r / world, (r + 1) / world).  The slab thickness is a height, ``thickness`` = H_0 / world with
      H_0 = |det h| / |h_1 x h_2| (not |h_0| / world): a pair closer than r has |ds_0| H_0 < r, so ghosts within r of a
      face are the atoms with s_0 within r / H_0 of it.  A ghost that crosses the periodic face of row 0 moves by -+h_0
      (ab2_slab_plan_count_lattice, ab2_p2p_push_rows_v).
    The local frame of every rank is the cell h with pbc (False, True, True)."""

    axis = 0

    def __init__(self, cell: torch.Tensor, world: int):
        h = cell.detach().reshape(3, 3).to(device="cpu", dtype=torch.float64)
        self.rows = h.tolist()
        self.world = int(world)
        _, heights, regular = D._lattice_metrics(self.rows)
        if not regular:
            raise ValueError("slab decomposition: the cell is not regular (a row is not finite, or the rows are singular or within "
                             "1e-12 rad of a common plane)")
        self.height = heights[0]  # H_0
        self.diagonal = bool((h - torch.diag(torch.diagonal(h))).abs().max() == 0) and bool((torch.diagonal(h) > 0).all())
        if self.diagonal:
            self.Lx = self.rows[0][0]
            self.thickness = self.Lx / world
        else:
            self.Lx = None
            self.thickness = self.height / world
            cr = [D._cross(self.rows[(a + 1) % 3], self.rows[(a + 2) % 3]) for a in range(3)]
            det = sum(self.rows[0][x] * cr[0][x] for x in range(3))
            self.hinv = [[cr[a][x] / det for a in range(3)] for x in range(3)]  # hinv[x][a], as lattice.cuh

    def frac0(self, pos: torch.Tensor) -> torch.Tensor:
        """s_0 = (p_0 hinv[0][0] + p_1 hinv[1][0]) + p_2 hinv[2][0] in fp64 (lattice cells)"""
        p = pos.double()
        hi = self.hinv
        return (p[:, 0] * hi[0][0] + p[:, 1] * hi[1][0]) + p[:, 2] * hi[2][0]

    def faces(self, rank: int) -> Tuple[float, float]:
        """(lo, hi) of the slab of ``rank``: x in length units (diagonal) or s_0"""
        if self.diagonal:
            return rank * self.thickness, (rank + 1) * self.thickness
        return rank / self.world, (rank + 1) / self.world

    def reach(self, r: float) -> float:
        """a distance r across the faces, in the units of ``faces``"""
        return float(r) if self.diagonal else float(r) / self.height

    def ghost_shifts(self, rank: int):
        """(shift of the ghosts from the left neighbour, from the right one): -+Lx (diagonal, along x) or -+h_0 (3 fp64
        components), zero away from the periodic face"""
        if self.diagonal:
            return (-self.Lx if rank == 0 else 0.0), (self.Lx if rank == self.world - 1 else 0.0)
        zero = [0.0, 0.0, 0.0]
        return ([-v for v in self.rows[0]] if rank == 0 else zero), (list(self.rows[0]) if rank == self.world - 1 else zero)


class SlabDecomposition:
    """Static exchange plan of one rank (valid as long as the neighbour list is), for any regular cell (``SlabGeometry``)."""

    def __init__(self, pos: torch.Tensor, cell: torch.Tensor, types: torch.Tensor, r_max: float, rank: int, world: int, device=None):
        assert world >= 2, "use the plain periodic path on one rank"
        cell = cell.view(3, 3)
        geo = SlabGeometry(cell, world)
        width = geo.thickness
        assert width >= r_max, "slab thinner than r_max: neighbours beyond the adjacent slab"
        self.rank, self.world, self.r_max = rank, world, float(r_max)
        self._set_geometry(geo)
        if geo.diagonal:
            Lx = self.Lx
            x = pos[:, 0] - torch.floor(pos[:, 0] / Lx) * Lx
            slab = torch.clamp((x / width).long(), max=world - 1)
        else:
            x = geo.frac0(self._wrap0(pos))
            slab = torch.clamp(torch.floor(x * world).long(), 0, world - 1)
        reach = geo.reach(r_max)

        def owned_of(r):
            return torch.nonzero(slab == r).squeeze(-1)

        def send_lists(r):
            ids = owned_of(r)
            xr = x[ids]
            lo, hi = geo.faces(r)
            return ids[xr >= hi - reach], ids[xr < lo + reach]  # (to the right neighbour, to the left neighbour)

        self.left, self.right = (rank - 1) % world, (rank + 1) % world
        self.owned = owned_of(rank)
        self.n_owned = int(self.owned.shape[0])
        my_to_right, my_to_left = send_lists(rank)
        # positions in the local owned array
        inv = torch.full((pos.shape[0],), -1, dtype=torch.long)
        inv[self.owned] = torch.arange(self.n_owned)
        self.send_right_idx = inv[my_to_right]
        self.send_left_idx = inv[my_to_left]
        # what arrives: left neighbour's "to the right" list, right neighbour's "to the left" list
        left_ids = send_lists(self.left)[0]
        right_ids = send_lists(self.right)[1]
        self.n_ghost_left, self.n_ghost_right = int(left_ids.shape[0]), int(right_ids.shape[0])
        self.ghost_global = torch.cat([left_ids, right_ids])
        self.n_ghost = self.n_ghost_left + self.n_ghost_right
        self.types_local = torch.cat([types[self.owned], types[self.ghost_global]])
        self.global_ids_local = torch.cat([self.owned, self.ghost_global])
        # local periodic cell: row 0 is open (ghosts cover it), rows 1 and 2 stay periodic
        self.cell = cell.clone()
        self.pbc = (False, True, True)
        # unwrapped x so that slab + ghosts form one contiguous block along x
        pos_local = self.local_positions_from_global(pos)
        self.csr, self.shift_vec = None, None
        self.edge_index = self.edge_cell_shift = None
        dev = torch.device(device) if device is not None else None
        if dev is not None and dev.type == "cuda" and D.csr_supported(pos_local.to(dev), r_max, self.cell, self.pbc):
            # CUDA cell list over owned + ghost atoms, rows for the owned centres only, straight into the kernels' CSR:
            # the int64 COO list of the local frame (6.5M edges per rank for the 1M-atom box) is never built
            self.csr, self.shift_vec = D.neighbor_csr(pos_local.to(dev), r_max, self.cell.to(dev), self.pbc, n_centres=self.n_owned)
            self.n_edges = self.csr.num_edges
        else:
            ei, sh = D.neighbor_list(pos_local, r_max, self.cell, self.pbc)
            keep = ei[0] < self.n_owned  # edges of owned centres only
            self.edge_index = ei[:, keep].contiguous()
            self.edge_cell_shift = sh[keep].contiguous()
            self.n_edges = int(self.edge_index.shape[1])

    def _set_geometry(self, geo: SlabGeometry):
        """the geometry's decisions for this rank: the ghosts' periodic shifts as I receive them (``shift_left`` /
        ``shift_right``) and as my neighbours receive my atoms (``push_shift_left`` / ``push_shift_right``); scalars
        along x for a diagonal cell, 3-vectors otherwise"""
        self.geom = geo
        self.Lx = geo.Lx
        self.shift_left, self.shift_right = geo.ghost_shifts(self.rank)
        # my atoms are the right neighbour's left ghosts and the left neighbour's right ghosts
        self.push_shift_right = geo.ghost_shifts((self.rank + 1) % self.world)[0]
        self.push_shift_left = geo.ghost_shifts((self.rank - 1) % self.world)[1]

    def _wrap0(self, pos: torch.Tensor) -> torch.Tensor:
        """positions wrapped along lattice row 0 only (set-up; lattice cells): p - floor(s_0) h_0 in fp64, rounded once"""
        h0 = torch.tensor(self.geom.rows[0], dtype=torch.float64, device=pos.device)
        return (pos.double() - torch.floor(self.geom.frac0(pos))[:, None] * h0).to(pos.dtype)

    def shift_ghosts(self, g: torch.Tensor, side: str) -> torch.Tensor:
        """ghost rows [m, 3] from the left (``side`` "left") or right neighbour -> their periodic images in my frame.  A
        lattice shift is added in fp64 and rounded once, as the peer-memory push does."""
        sh = self.shift_left if side == "left" else self.shift_right
        if self.geom.diagonal:
            g[:, 0] += sh
            return g
        return (g.double() + torch.tensor(sh, dtype=torch.float64, device=g.device)).to(g.dtype)

    # positions of owned + ghost atoms taken from a global frame (set-up / tests)
    def local_positions_from_global(self, pos: torch.Tensor) -> torch.Tensor:
        if self.geom.diagonal:
            Lx = self.Lx
            p = pos.clone()
            p[:, 0] = p[:, 0] - torch.floor(p[:, 0] / Lx) * Lx
        else:
            p = self._wrap0(pos)
        gl = p[self.ghost_global[: self.n_ghost_left]].clone()
        gr = p[self.ghost_global[self.n_ghost_left :]].clone()
        gl = self.shift_ghosts(gl, "left")
        gr = self.shift_ghosts(gr, "right")
        return torch.cat([p[self.owned], gl, gr], 0)

    def to(self, device) -> "SlabDecomposition":
        for k in ("owned", "send_right_idx", "send_left_idx", "ghost_global", "types_local", "global_ids_local", "cell",
                  "edge_index", "edge_cell_shift"):
            if getattr(self, k) is not None:
                setattr(self, k, getattr(self, k).to(device))
        return self

    # ---- communication --------------------------------------------------------------------
    def _peers(self):
        """-> list of (peer, [send segments], [recv segment sizes]) in a canonical order that
        both sides agree on (right-going list first, then left-going)."""
        if self.left == self.right:  # world == 2: both neighbours are the same rank
            return [(self.left, ["right", "left"], ["from_left", "from_right"])]
        return [(self.right, ["right"], ["from_right"]), (self.left, ["left"], ["from_left"])]

    def exchange_forward(self, pos_owned: torch.Tensor) -> torch.Tensor:
        """positions of owned atoms [n_owned,3] -> ghost positions [n_ghost,3] (wrap applied)."""
        seg = {"right": pos_owned.index_select(0, self.send_right_idx), "left": pos_owned.index_select(0, self.send_left_idx)}
        n_in = {"from_left": self.n_ghost_left, "from_right": self.n_ghost_right}
        ops, bufs = [], []
        for peer, sends, recvs in self._peers():
            sbuf = torch.cat([seg[s] for s in sends], 0).contiguous()
            rbuf = torch.empty(sum(n_in[r] for r in recvs), 3, dtype=pos_owned.dtype, device=pos_owned.device)
            ops += [dist.P2POp(dist.isend, sbuf, peer), dist.P2POp(dist.irecv, rbuf, peer)]
            bufs.append((recvs, rbuf, sbuf))
        for w in dist.batch_isend_irecv(ops):
            w.wait()
        got = {}
        for recvs, rbuf, _ in bufs:
            o = 0
            for r in recvs:
                got[r] = rbuf[o : o + n_in[r]]
                o += n_in[r]
        gl, gr = got["from_left"].clone(), got["from_right"].clone()
        gl = self.shift_ghosts(gl, "left")
        gr = self.shift_ghosts(gr, "right")
        return torch.cat([gl, gr], 0)

    def exchange_reverse(self, g_ghost: torch.Tensor, g_owned: torch.Tensor) -> torch.Tensor:
        """add the rows accumulated on ghosts [n_ghost,w] onto the owners [n_owned,w]; returns g_owned.  w = 3: gradients;
        w = 12: gradients and per-atom virials in one exchange."""
        seg = {"from_left": g_ghost[: self.n_ghost_left], "from_right": g_ghost[self.n_ghost_left :]}
        n_out = {"right": int(self.send_right_idx.shape[0]), "left": int(self.send_left_idx.shape[0])}
        ops, bufs = [], []
        for peer, sends, recvs in self._peers():
            # mirror of the forward plan: what I received from `peer` goes back to it
            sbuf = torch.cat([seg[r] for r in recvs], 0).contiguous()
            rbuf = torch.empty(sum(n_out[s] for s in sends), *g_ghost.shape[1:], dtype=g_ghost.dtype, device=g_ghost.device)
            ops += [dist.P2POp(dist.isend, sbuf, peer), dist.P2POp(dist.irecv, rbuf, peer)]
            bufs.append((sends, rbuf, sbuf))
        for w in dist.batch_isend_irecv(ops):
            w.wait()
        idx = {"right": self.send_right_idx, "left": self.send_left_idx}
        for sends, rbuf, _ in bufs:
            o = 0
            for s in sends:
                g_owned.index_add_(0, idx[s], rbuf[o : o + n_out[s]])
                o += n_out[s]
        return g_owned

    def halo_bytes_per_step(self, itemsize: int, atomic_virial: bool = False) -> int:
        """bytes this rank sends per step: position rows forward, gradient rows back (width 12 with the per-atom virial)."""
        n_fwd = int(self.send_right_idx.shape[0]) + int(self.send_left_idx.shape[0])
        return (n_fwd * 3 + self.n_ghost * (12 if atomic_virial else 3)) * itemsize


class P2PHalo:
    """The three per-step exchanges over NVLink peer memory (csrc/halo_p2p.cu): every rank owns a mailbox that its peers
    map through CUDA IPC; senders store rows straight into the receiver's mailbox and publish the step number, receivers
    spin on it.  Kernels only -- the step stays one CUDA graph and makes no NCCL call.  Set-up (once) uses
    torch.distributed to exchange the IPC handles.

    ``atomic_virial=True`` allocates the extended mailbox (AB2_P2P_EXT_VIRIAL): reverse rows that carry the per-atom virial
    next to the gradient (``reverse_w``) and a vector all-reduce (``reduce``) for energy, virial and heat current.  Peers
    compute offsets into each other's mailboxes from the layout, so every rank must pass the same flag: it is compared
    across ranks before anything is allocated, and a mismatch raises ValueError on every rank.

    ``headroom`` >= 1 sizes the mailbox for that many times the rows the plan needs now (1: exactly, the static case).  A
    changing plan is re-bound with ``rebind``; ``close`` releases the mailbox.  Both are collective."""

    VEC_MAX = 16  # AB2_P2P_VEC_MAX

    def __init__(self, dec: SlabDecomposition, device, atomic_virial: bool = False, headroom: float = 1.0):
        import ctypes as C

        from . import _lib

        self._lib, self._C = _lib, C
        self.dec, self.dev = dec, torch.device(device)
        self.extended = bool(atomic_virial)
        world, rank = dec.world, dec.rank
        # max of (flag, -flag) over the ranks: they agree iff max == min (one all-reduce, any backend)
        fl = torch.tensor([int(self.extended), -int(self.extended)], dtype=torch.int32, device=self.dev)
        dist.all_reduce(fl, op=dist.ReduceOp.MAX)
        if int(fl[0]) != -int(fl[1]):
            raise ValueError("P2PHalo: ranks disagree on atomic_virial; the mailbox layout must be the same on every rank")
        self.mailbox, self.peers, self.n_grown, self._err_before = None, [], 0, 0
        self._open(self._with_headroom(self._rows_needed(dec), headroom))
        self.step = torch.zeros(1, dtype=torch.int32, device=self.dev)
        self.done = torch.zeros(4, dtype=torch.int32, device=self.dev)
        self.e_tot = torch.zeros(1, dtype=torch.float64, device=self.dev)
        self.v_tot = torch.zeros(self.VEC_MAX, dtype=torch.float64, device=self.dev) if self.extended else None
        self.pos_local = None
        self.send_right = dec.send_right_idx.to(self.dev).contiguous()
        self.send_left = dec.send_left_idx.to(self.dev).contiguous()
        # periodic wrap as the RECEIVER sees my atoms (rank 0's left ghosts sit at x - Lx, or at s_0 - 1: pos - h_0), from
        # the plan's geometry: a scalar along x (ab2_p2p_push_rows) or a lattice row (ab2_p2p_push_rows_v)
        self.shift_to_right, self.shift_to_left = dec.push_shift_right, dec.push_shift_left
        torch.cuda.synchronize(self.dev)
        dist.barrier()

    def _rows_needed(self, dec) -> int:
        """the longest send or ghost list of any rank (one all-reduce MAX)"""
        mx = torch.tensor([max(int(dec.send_right_idx.shape[0]), int(dec.send_left_idx.shape[0]), dec.n_ghost_left, dec.n_ghost_right, 1)],
                          device=self.dev)
        dist.all_reduce(mx, op=dist.ReduceOp.MAX)
        return int(mx)

    @staticmethod
    def _with_headroom(rows: int, headroom: float) -> int:
        if not headroom >= 1.0:
            raise ValueError(f"P2PHalo: headroom must be >= 1, got {headroom}")
        return max(rows, int(math.ceil(rows * headroom)))

    def _open(self, max_rows: int):
        """allocate my mailbox for ``max_rows`` rows and map every peer's (all ranks, same max_rows)"""
        C, lib = self._C, self._lib.load()
        self.max_rows = int(max_rows)
        world, rank = self.dec.world, self.dec.rank
        if self.extended:
            nbytes = int(lib.ab2_p2p_mailbox_bytes_ex(self.max_rows, world, 1))
        else:
            nbytes = int(lib.ab2_p2p_mailbox_bytes(self.max_rows, world))
        ptr = C.c_void_p()
        self._lib._check(lib.ab2_p2p_alloc(nbytes, C.byref(ptr)))
        self.mailbox = ptr.value
        hbuf = C.create_string_buffer(64)
        self._lib._check(lib.ab2_p2p_get_handle(C.c_void_p(self.mailbox), hbuf))
        handles = [None] * world
        dist.all_gather_object(handles, bytes(hbuf.raw))
        self.peers = []
        for r, h in enumerate(handles):
            if r == rank:
                self.peers.append(self.mailbox)
            else:
                q = C.c_void_p()
                self._lib._check(lib.ab2_p2p_open_handle(C.create_string_buffer(h, 64), C.byref(q)))
                self.peers.append(q.value)
        self.peers_dev = torch.tensor(self.peers, dtype=torch.int64, device=self.dev)

    def _release(self):
        """unmap the peers' mailboxes and free mine, once no rank has a step in flight (collective)"""
        lib, C = self._lib.load(), self._C
        torch.cuda.synchronize(self.dev)
        self._err_before = max(self._err_before, self.error())
        dist.barrier()  # every rank's last step is complete: nothing is stored into any mailbox any more
        for r, p in enumerate(self.peers):
            if r != self.dec.rank:
                self._lib._check(lib.ab2_p2p_close_handle(C.c_void_p(p)))
        dist.barrier()  # no peer maps my mailbox any more
        self._lib._check(lib.ab2_p2p_free(C.c_void_p(self.mailbox)))
        self.mailbox, self.peers, self.peers_dev = None, [], None

    def rebind(self, dec: SlabDecomposition, headroom: float = 1.0):
        """Point the exchanges at a new plan of the same ranks (new send lists and ghost counts).  The rows it needs are
        agreed with one all-reduce MAX; when they exceed the mailbox, every rank re-allocates for ``headroom`` times that
        (peers re-mapped, step counter kept).  Collective: every rank calls it, between steps."""
        need = self._rows_needed(dec)
        self.dec = dec
        self.send_right = dec.send_right_idx.to(self.dev).contiguous()
        self.send_left = dec.send_left_idx.to(self.dev).contiguous()
        self.pos_local = None
        if need > self.max_rows:
            self._release()
            self._open(self._with_headroom(need, headroom))
            self.n_grown += 1
            torch.cuda.synchronize(self.dev)
            dist.barrier()

    def close(self):
        """Close the peers' IPC handles and free my mailbox (collective; the halo is unusable afterwards)."""
        if self.mailbox is not None:
            self._release()

    def _ptr(self, t, row_offset=0):
        return self._C.c_void_p(t.data_ptr() + row_offset * 3 * t.element_size())

    def forward(self, pos_owned: torch.Tensor) -> torch.Tensor:
        """positions of my atoms -> [owned | ghosts from the left | ghosts from the right] (static buffer)."""
        lib, dec, C = self._lib.load(), self.dec, self._C
        st = self._lib._stream()
        dt = self._lib.DTYPE_ENUM[pos_owned.dtype]
        if self.pos_local is None or self.pos_local.dtype != pos_owned.dtype:
            self.pos_local = torch.zeros(dec.n_owned + dec.n_ghost, 3, dtype=pos_owned.dtype, device=self.dev)
        pos_owned = pos_owned.contiguous()
        self.pos_local[: dec.n_owned].copy_(pos_owned)
        ck = self._lib._check
        ck(lib.ab2_p2p_begin(C.c_void_p(self.step.data_ptr()), st))
        if dec.geom.diagonal:
            push = lambda shift, *rest: lib.ab2_p2p_push_rows(*rest[:6], shift, *rest[6:])  # noqa: E731
        else:
            push = lambda shift, *rest: lib.ab2_p2p_push_rows_v(*rest[:6], *shift, *rest[6:])  # noqa: E731
        # I am the LEFT neighbour of my right peer (its slot 0) and the RIGHT neighbour of my left peer (its slot 1)
        ck(push(self.shift_to_right, dt, 0, 0, self._ptr(pos_owned), C.c_void_p(self.send_right.data_ptr()), int(self.send_right.shape[0]),
                C.c_void_p(self.peers[dec.right]), self.max_rows, dec.world, C.c_void_p(self.step.data_ptr()), C.c_void_p(self.done.data_ptr()), st))
        ck(push(self.shift_to_left, dt, 0, 1, self._ptr(pos_owned), C.c_void_p(self.send_left.data_ptr()), int(self.send_left.shape[0]),
                C.c_void_p(self.peers[dec.left]), self.max_rows, dec.world, C.c_void_p(self.step.data_ptr()), C.c_void_p(self.done.data_ptr() + 4),
                st))
        ck(lib.ab2_p2p_wait_unpack(dt, 0, 0, C.c_void_p(self.mailbox), self.max_rows, dec.world, C.c_void_p(self.step.data_ptr()), dec.n_ghost_left,
                                   self._ptr(self.pos_local, dec.n_owned), None, 0, st))
        ck(lib.ab2_p2p_wait_unpack(dt, 0, 1, C.c_void_p(self.mailbox), self.max_rows, dec.world, C.c_void_p(self.step.data_ptr()), dec.n_ghost_right,
                                   self._ptr(self.pos_local, dec.n_owned + dec.n_ghost_left), None, 0, st))
        self._lib.PROF.launches += 5
        return self.pos_local

    def reverse(self, g_local: torch.Tensor, g_owned: torch.Tensor) -> torch.Tensor:
        """gradients accumulated on my ghosts go back to their owners; what my neighbours accumulated on my boundary atoms
        is added into g_owned (left neighbour's rows first, then the right one's: fixed order)."""
        lib, dec, C = self._lib.load(), self.dec, self._C
        st = self._lib._stream()
        dt = self._lib.DTYPE_ENUM[g_local.dtype]
        g_local = g_local.contiguous()
        ck = self._lib._check
        ck(lib.ab2_p2p_push_rows(dt, 1, 1, self._ptr(g_local, dec.n_owned), None, dec.n_ghost_left, 0.0, C.c_void_p(self.peers[dec.left]), self.max_rows,
                                 dec.world, C.c_void_p(self.step.data_ptr()), C.c_void_p(self.done.data_ptr() + 8), st))
        ck(lib.ab2_p2p_push_rows(dt, 1, 0, self._ptr(g_local, dec.n_owned + dec.n_ghost_left), None, dec.n_ghost_right, 0.0,
                                 C.c_void_p(self.peers[dec.right]), self.max_rows, dec.world, C.c_void_p(self.step.data_ptr()),
                                 C.c_void_p(self.done.data_ptr() + 12), st))
        dto = self._lib.DTYPE_ENUM[g_owned.dtype]
        ck(lib.ab2_p2p_wait_unpack(dto, 1, 0, C.c_void_p(self.mailbox), self.max_rows, dec.world, C.c_void_p(self.step.data_ptr()),
                                   int(self.send_left.shape[0]), self._ptr(g_owned), C.c_void_p(self.send_left.data_ptr()), 1, st))
        ck(lib.ab2_p2p_wait_unpack(dto, 1, 1, C.c_void_p(self.mailbox), self.max_rows, dec.world, C.c_void_p(self.step.data_ptr()),
                                   int(self.send_right.shape[0]), self._ptr(g_owned), C.c_void_p(self.send_right.data_ptr()), 1, st))
        self._lib.PROF.launches += 4
        return g_owned

    def reverse_w(self, g_local: torch.Tensor, W_local: torch.Tensor, g_owned: torch.Tensor, W_owned: torch.Tensor):
        """``reverse`` for gradients [n_local,3] and per-atom virials [n_local,3,3] together, in rows of width 12 (extended
        mailbox): the ghosts' rows are added into g_owned and W_owned, left neighbour's rows first; returns both."""
        if not self.extended:
            raise RuntimeError("P2PHalo.reverse_w needs the extended mailbox: P2PHalo(..., atomic_virial=True)")
        lib, dec, C = self._lib.load(), self.dec, self._C
        st = self._lib._stream()
        assert W_local.dtype == g_local.dtype and W_owned.dtype == g_owned.dtype and W_owned.is_contiguous() and g_owned.is_contiguous()
        dt = self._lib.DTYPE_ENUM[g_local.dtype]
        g_local, W_local = g_local.contiguous(), W_local.contiguous()
        gl, gr = dec.n_owned, dec.n_owned + dec.n_ghost_left
        es, ws = g_local.element_size(), W_local.element_size()

        def rows(t, r, width, size):
            return C.c_void_p(t.data_ptr() + r * width * size)

        ck = self._lib._check
        step = C.c_void_p(self.step.data_ptr())
        ck(lib.ab2_p2p_push_rows_w(dt, 1, rows(g_local, gl, 3, es), rows(W_local, gl, 9, ws), dec.n_ghost_left, C.c_void_p(self.peers[dec.left]),
                                   self.max_rows, dec.world, step, C.c_void_p(self.done.data_ptr() + 8), st))
        ck(lib.ab2_p2p_push_rows_w(dt, 0, rows(g_local, gr, 3, es), rows(W_local, gr, 9, ws), dec.n_ghost_right, C.c_void_p(self.peers[dec.right]),
                                   self.max_rows, dec.world, step, C.c_void_p(self.done.data_ptr() + 12), st))
        dto = self._lib.DTYPE_ENUM[g_owned.dtype]
        ck(lib.ab2_p2p_wait_unpack_w(dto, 0, C.c_void_p(self.mailbox), self.max_rows, dec.world, step, int(self.send_left.shape[0]),
                                     C.c_void_p(g_owned.data_ptr()), C.c_void_p(W_owned.data_ptr()), C.c_void_p(self.send_left.data_ptr()), st))
        ck(lib.ab2_p2p_wait_unpack_w(dto, 1, C.c_void_p(self.mailbox), self.max_rows, dec.world, step, int(self.send_right.shape[0]),
                                     C.c_void_p(g_owned.data_ptr()), C.c_void_p(W_owned.data_ptr()), C.c_void_p(self.send_right.data_ptr()), st))
        self._lib.PROF.launches += 4
        return g_owned, W_owned

    def reduce(self, v_local: torch.Tensor) -> torch.Tensor:
        """sum of up to 16 fp64 values over all ranks, in rank order (bitwise identical everywhere; extended mailbox).
        Returns the persistent [n] result buffer."""
        if not self.extended:
            raise RuntimeError("P2PHalo.reduce needs the extended mailbox: P2PHalo(..., atomic_virial=True)")
        lib, dec, C = self._lib.load(), self.dec, self._C
        self._v_in = v_local.detach().double().reshape(-1).contiguous()
        n = int(self._v_in.shape[0])
        self._lib._check(lib.ab2_p2p_allreduce_vec(C.c_void_p(self._v_in.data_ptr()), n, dec.rank, dec.world, self.max_rows,
                                                   C.c_void_p(self.peers_dev.data_ptr()), C.c_void_p(self.mailbox), C.c_void_p(self.step.data_ptr()),
                                                   C.c_void_p(self.v_tot.data_ptr()), self._lib._stream()))
        self._lib.PROF.launches += 2
        return self.v_tot[:n]

    def energy(self, e_local: torch.Tensor) -> torch.Tensor:
        """sum of one fp64 scalar over all ranks, in rank order (bitwise identical everywhere)."""
        lib, dec, C = self._lib.load(), self.dec, self._C
        self._e_in = e_local.detach().double().reshape(1).contiguous()
        self._lib._check(lib.ab2_p2p_allreduce_energy(C.c_void_p(self._e_in.data_ptr()), dec.rank, dec.world, self.max_rows,
                                                      C.c_void_p(self.peers_dev.data_ptr()), C.c_void_p(self.mailbox), C.c_void_p(self.step.data_ptr()),
                                                      C.c_void_p(self.e_tot.data_ptr()), self._lib._stream()))
        self._lib.PROF.launches += 2
        return self.e_tot

    def error(self) -> int:
        """the mailbox's error word (1: a wait timed out), including that of any mailbox a ``rebind`` replaced"""
        if self.mailbox is None:
            return self._err_before
        now = int(self._lib.load().ab2_p2p_error(self._C.c_void_p(self.mailbox), self.max_rows, self.dec.world, self._lib._stream()))
        return max(now, self._err_before)


class DistributedAllegro:
    """Energy + forces of a slab-decomposed frame.  ``energy_model(data) -> data`` must write
    ``atomic_energy`` for the local atoms (owned first) and be differentiable w.r.t. ``pos``
    (FusedAllegroEnergy on the GPU; any stand-in in the CPU tests).

    ``stress`` / ``atomic_virial`` / ``heat_current`` (the last implies the second) switch on the outputs of the same
    names in ``evaluate``; ``__call__`` is unaffected by them.  They need a model with ``energy_and_forces`` and, on the
    peer-memory transport, ``P2PHalo(..., atomic_virial=True)``.  An edge belongs to the rank that owns its centre, so
    the virial is the sum of the ranks' edge virials, and a ghost's per-atom virial row is added onto its owner by the
    reverse halo exactly as a ghost gradient is; the heat current is then summed over owned atoms only."""

    def __init__(self, energy_model: Callable[[D.Type], D.Type], dec: SlabDecomposition, p2p: Optional["P2PHalo"] = None,
                 stress: bool = False, atomic_virial: bool = False, heat_current: bool = False):
        self.model, self.dec, self.p2p = energy_model, dec, p2p
        self.stress = bool(stress)
        self.heat_current = bool(heat_current)
        self.atomic_virial = bool(atomic_virial) or self.heat_current
        if self.has_flags:
            if not hasattr(energy_model, "energy_and_forces"):
                raise NotImplementedError("DistributedAllegro: stress / atomic_virial / heat_current need a model with energy_and_forces "
                                          "(the autograd branch returns energy and forces only)")
            if p2p is not None and not p2p.extended:
                raise ValueError("DistributedAllegro: stress / atomic_virial / heat_current over peer memory need "
                                 "P2PHalo(..., atomic_virial=True) on every rank")
        cell = dec.cell.view(3, 3).double()
        self.volume = float(torch.det(cell).abs())
        self._heat_ptr = None

    @property
    def has_flags(self) -> bool:
        return self.stress or self.atomic_virial

    def _local_data(self, pos_owned: torch.Tensor) -> D.Type:
        """forward halo -> the rank's local frame (owned + ghosts, rows for the owned centres)."""
        dec = self.dec
        if self.p2p is not None:
            pos_local = self.p2p.forward(pos_owned.detach())
        else:
            ghosts = dec.exchange_forward(pos_owned.detach())
            pos_local = torch.cat([pos_owned.detach(), ghosts], 0).requires_grad_(True)
        data = {D.POSITIONS_KEY: pos_local, D.ATOM_TYPE_KEY: dec.types_local, D.CELL_KEY: dec.cell}
        if dec.csr is not None:
            data[D.CSR_KEY], data[D.EDGE_SHIFT_VEC_KEY] = dec.csr, dec.shift_vec
        else:
            data[D.EDGE_INDEX_KEY], data[D.EDGE_CELL_SHIFT_KEY] = dec.edge_index, dec.edge_cell_shift
        return data

    def evaluate(self, pos_owned: torch.Tensor, velocities: Optional[torch.Tensor] = None) -> D.Type:
        """-> dict with ``total_energy`` [1] (all ranks, fp64), ``forces`` [n_owned,3] and ``atomic_energy`` [n_owned,1]; with
        the flags also ``stress`` and ``virial`` [1,3,3] of the whole cell, ``atomic_virial`` [n_owned,3,3] and the potential
        ``heat_current`` [1,3] = sum over all atoms of E_a v_a + W[a] v_a, from the owned atoms' ``velocities`` [n_owned,3].
        Every check is made before the first exchange, so a refused call raises on every rank without leaving peers
        waiting."""
        dec = self.dec
        if self.heat_current:
            if velocities is None or tuple(velocities.shape) != (dec.n_owned, 3):
                got = None if velocities is None else tuple(velocities.shape)
                raise ValueError(f"heat_current=True needs `{D.VELOCITY_KEY}` of the owned atoms, shape ({dec.n_owned}, 3); got {got}")
        if not self.has_flags:
            e_tot, f, e_atoms = self(pos_owned)
            return {D.TOTAL_ENERGY_KEY: e_tot, D.FORCE_KEY: f, D.PER_ATOM_ENERGY_KEY: e_atoms}
        return self._evaluate_vec(pos_owned, velocities)

    def _evaluate_vec(self, pos_owned: torch.Tensor, velocities: Optional[torch.Tensor], extra: Optional[torch.Tensor] = None) -> D.Type:
        """``evaluate`` through the one fp64 vector reduction, whatever the flags (a model with ``energy_and_forces``).
        ``extra`` (at most 3 values) rides in slots 13.. of that reduction and comes back summed over the ranks as
        ``res["extra"]``."""
        dec = self.dec
        data = self._local_data(pos_owned)
        data[D.POSITIONS_KEY] = data[D.POSITIONS_KEY].detach()
        out = self.model.energy_and_forces(data, stress=self.stress, atomic_virial=self.atomic_virial)
        n = dec.n_owned
        e_atoms = out[D.PER_ATOM_ENERGY_KEY][:n]
        e_local = e_atoms.sum()
        g = -out[D.FORCE_KEY]
        g_owned = g[:n].clone()
        W_owned = None
        if self.atomic_virial:
            W = out[D.ATOMIC_VIRIAL_KEY]
            W_owned = W[:n].clone()
            if self.p2p is not None:
                self.p2p.reverse_w(g, W, g_owned, W_owned)
            else:  # one exchange of width-12 rows
                rows = torch.cat([g[n:], W[n:].reshape(-1, 9)], 1)
                both = dec.exchange_reverse(rows, torch.cat([g_owned, W_owned.reshape(n, 9)], 1))
                g_owned, W_owned = both[:, :3].contiguous(), both[:, 3:].reshape(n, 3, 3).contiguous()
        elif self.p2p is not None:
            self.p2p.reverse(g, g_owned)
        else:
            dec.exchange_reverse(g[n:].contiguous(), g_owned)
        # one fp64 vector summed over the ranks: energy, virial [9], heat current [3]
        parts = [e_local.detach().double().reshape(1)]
        parts.append(out[D.VIRIAL_KEY].double().reshape(9) if self.stress else e_local.new_zeros(9, dtype=torch.float64))
        if self.heat_current:
            if self._heat_ptr is None or self._heat_ptr.device != g_owned.device:
                self._heat_ptr = torch.tensor([0, n], dtype=torch.int32, device=g_owned.device)
            # J over the owned rows, after the reverse halo completed their W (ghost rows are partial)
            from . import _lib

            J = _lib.frame_heat_current(e_atoms.detach().reshape(-1), velocities, W_owned, self._heat_ptr)
            parts.append(J.double().reshape(3))
        else:
            parts.append(e_local.new_zeros(3, dtype=torch.float64))
        if extra is not None:
            parts.append(extra.detach().double().reshape(-1))
        vec = torch.cat(parts)
        if self.p2p is not None:
            tot = self.p2p.reduce(vec).clone()
        else:
            tot = vec.clone()
            dist.all_reduce(tot)
        dt = g_owned.dtype
        res = {D.TOTAL_ENERGY_KEY: tot[0:1], D.FORCE_KEY: -g_owned, D.PER_ATOM_ENERGY_KEY: e_atoms.detach()}
        if self.stress:
            vir = tot[1:10].view(1, 3, 3)
            res[D.VIRIAL_KEY] = vir.to(dt)
            res[D.STRESS_KEY] = (-vir / self.volume).to(dt)
        if self.atomic_virial:
            res[D.ATOMIC_VIRIAL_KEY] = W_owned
        if self.heat_current:
            res[D.HEAT_CURRENT_KEY] = tot[10:13].view(1, 3).to(dt)
        if extra is not None:
            res["extra"] = tot[13:]
        return res

    def __call__(self, pos_owned: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """-> (total energy [all ranks], forces on owned atoms [n_owned,3], owned atomic energies)."""
        dec = self.dec
        data = self._local_data(pos_owned)
        pos_local = data[D.POSITIONS_KEY]
        if hasattr(self.model, "energy_and_forces"):
            # autograd-free CUDA path: forces on owned AND ghost atoms come out of one pass
            data[D.POSITIONS_KEY] = pos_local.detach()
            out = self.model.energy_and_forces(data)
            e_atoms = out[D.PER_ATOM_ENERGY_KEY][: dec.n_owned]
            e_local = e_atoms.sum()
            g = -out[D.FORCE_KEY]
        else:
            with torch.enable_grad():
                out = self.model(data)
                e_atoms = out[D.PER_ATOM_ENERGY_KEY][: dec.n_owned]
                e_local = e_atoms.sum()
                (g,) = torch.autograd.grad(e_local, pos_local)
        g_owned = g[: dec.n_owned].clone()
        if self.p2p is not None:
            self.p2p.reverse(g, g_owned)
            # the mailbox protocol sums into a persistent buffer: hand out a copy, so that a caller holding the result of one
            # step does not see it change under the next one (under graph capture the copy is the graph's static output)
            e_tot = self.p2p.energy(e_local).clone()
            return e_tot, -g_owned, e_atoms.detach()
        dec.exchange_reverse(g[dec.n_owned :].contiguous(), g_owned)
        e_tot = e_local.detach().double().clone().reshape(1)
        dist.all_reduce(e_tot)
        return e_tot, -g_owned, e_atoms.detach()


class GraphedDistributedAllegro:
    """One slab-decomposed energy+forces step captured into a CUDA graph, NCCL halo included.

    The eager step is ~60 ctypes launches plus three torch.distributed calls; with one Python
    process per GPU sharing the box's host cores the launch path becomes the bottleneck at 4-8
    ranks.  NCCL point-to-point and all-reduce kernels are capturable once their communicators
    exist (warm-up does that), so the whole step -- forward halo, compute, reverse halo,
    energy all-reduce -- replays as one graph launch per rank.

    A runner with stress / atomic_virial / heat_current has ``runner.evaluate`` captured instead, with a static velocity
    buffer (``velocities``, needed for the heat current), and ``__call__(pos, vel)`` returns its dict."""

    def __init__(self, runner: DistributedAllegro, pos_owned: torch.Tensor, warmup: int = 3, velocities: Optional[torch.Tensor] = None):
        from . import _lib

        self.runner = runner
        self.static_pos = pos_owned.detach().clone()
        self.static_vel = None
        step = runner
        if runner.has_flags:
            if velocities is not None:
                self.static_vel = velocities.detach().clone()

            def step(p):
                return runner.evaluate(p, self.static_vel)
        prof = _lib.PROF.enabled
        _lib.PROF.enabled = False
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s), torch.no_grad():
            for _ in range(warmup):
                step(self.static_pos)
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        dist.barrier()
        self.graph = torch.cuda.CUDAGraph()
        n0 = _lib.PROF.launches
        with torch.no_grad(), torch.cuda.graph(self.graph):
            self.out = step(self.static_pos)
        self.launches_per_replay = _lib.PROF.launches - n0
        _lib.PROF.enabled = prof
        self._lib = _lib

    def __call__(self, pos_owned: Optional[torch.Tensor] = None, vel: Optional[torch.Tensor] = None):
        if pos_owned is not None:
            self.static_pos.copy_(pos_owned, non_blocking=True)
        if vel is not None and self.static_vel is not None:
            self.static_vel.copy_(vel, non_blocking=True)
        self.graph.replay()
        self._lib.PROF.launches += self.launches_per_replay
        return self.out


# ---- molecular dynamics on several GPUs -------------------------------------------------------------------------------

# a grown mailbox holds this many times the rows the rebuild that grew it needed (fewer re-allocations on a drifting plan)
MAILBOX_HEADROOM = 1.25


class _SlabPlan(SlabDecomposition):
    """The exchange plan of one rank built by ``DistributedCalculator``'s rebuild from the rank's own atoms: the
    attributes of a ``SlabDecomposition`` (so its torch.distributed exchanges, ``P2PHalo`` and ``DistributedAllegro``
    take it unchanged), with the local neighbour list built for ``r_list = r_max + skin``."""

    def __init__(self, rank, world, geom: SlabGeometry, cell, ids, types, send_left_idx, send_right_idx, ghost_ids_left, ghost_ids_right,
                 ghost_types):
        self.rank, self.world = rank, world
        self._set_geometry(geom)
        self.left, self.right = (rank - 1) % world, (rank + 1) % world
        self.owned = ids
        self.n_owned = int(ids.shape[0])
        self.send_right_idx, self.send_left_idx = send_right_idx, send_left_idx
        self.n_ghost_left, self.n_ghost_right = int(ghost_ids_left.shape[0]), int(ghost_ids_right.shape[0])
        self.n_ghost = self.n_ghost_left + self.n_ghost_right
        self.ghost_global = torch.cat([ghost_ids_left, ghost_ids_right])
        self.types_local = torch.cat([types, ghost_types])
        self.global_ids_local = torch.cat([ids, self.ghost_global])
        self.cell = cell
        self.pbc = (False, True, True)
        self.csr = self.shift_vec = self.edge_index = self.edge_cell_shift = None
        self.n_edges = 0

    def build_list(self, pos_local: torch.Tensor, r_list: float, cutoffs: Optional[torch.Tensor] = None):
        """neighbour list of the owned centres over owned + ghost atoms, row 0 open, rows 1 and 2 periodic; ``cutoffs``
        [T,T]: pruned to those per-type-pair radii (data.prune_csr)"""
        if pos_local.is_cuda:
            prune = {} if cutoffs is None else dict(types=self.types_local, cutoffs=cutoffs)
            self.csr, self.shift_vec = D.neighbor_csr(pos_local, r_list, self.cell, self.pbc, n_centres=self.n_owned, **prune)
            self.n_edges = self.csr.num_edges
        else:  # CPU (the gloo tests): the pair search, rows of owned centres only
            ei, sh = D.neighbor_list(pos_local, r_list, self.cell, self.pbc)
            keep = ei[0] < self.n_owned
            self.edge_index, self.edge_cell_shift = ei[:, keep].contiguous(), sh[keep].contiguous()
            self.n_edges = int(self.edge_index.shape[1])
            if cutoffs is not None:
                shift_vec = (self.edge_cell_shift @ self.cell.view(3, 3).to(pos_local.dtype)).contiguous()
                self.csr, self.shift_vec = D.prune_csr(D.build_csr(self.edge_index, self.n_owned), shift_vec, pos_local, self.types_local,
                                                       cutoffs, r_list)
                self.edge_index = self.edge_cell_shift = None
                self.n_edges = self.csr.num_edges


class LocalAtoms:
    """The atoms one rank owns: ``pos`` [n,3] (wrapped into the cell at the last rebuild, unwrapped since), ``types`` [n],
    ``ids`` [n] int64 (index in the global frame), ``image`` [n,3] int32 (lattice vectors removed by wrapping: the
    unwrapped position is pos + image @ h, h the cell's rows; pos + image * box for an orthorhombic box) and ``arrays``
    {name: [n, ...]} (velocities, masses, ... of the same atoms).  ``DistributedCalculator.compute`` may replace all of
    them together (re-partition)."""

    def __init__(self, pos, types, ids, image, arrays):
        self.pos, self.types, self.ids, self.image, self.arrays = pos, types, ids, image, arrays

    def __len__(self):
        return int(self.pos.shape[0])


class _MDStep:
    """the step ``GraphedDistributedAllegro`` captures: the model on the skin list plus the rebuild check, in one
    vector reduction"""

    has_flags = True

    def __init__(self, calc: "DistributedCalculator"):
        self.calc = calc

    def evaluate(self, pos_owned, velocities=None):
        return self.calc._step(pos_owned, velocities)


class DistributedCalculator:
    """Molecular dynamics on several GPUs: a 1-D slab decomposition along lattice row 0 that follows the trajectory.

    Every rank keeps a neighbour list of its owned centres built with ``r_list = r_max + skin`` over its atoms and the
    ghosts within ``r_list`` of its two faces.  Between rebuilds a step is one CUDA graph replay -- forward halo, the
    model on the skin list, reverse halo, and one fp64 vector reduction that carries the energy, virial and heat current
    and also the number of owned atoms that moved more than ``skin / 2`` since the last rebuild.  The host reads that
    number (8 bytes) after every step; if any rank has such an atom, the step's outputs are discarded, every rank
    rebuilds at the current positions and the step is recomputed, so no force ever comes from a stale list.

    A rebuild, on every rank in the same order: wrap positions into the box and classify each owned atom by its slab
    (ab2_slab_plan, mode 0); refuse atoms that jumped more than a slab (ValueError on every rank, agreed by one
    all-reduce before any exchange); migrate the emigrants to the adjacent ranks (torch.distributed, staged through the
    host on gloo; new owned order = stayers in their old order, then arrivals from the left, then from the right); select
    the ghosts (mode 1) and exchange their ids, types and positions; build the neighbour list; re-bind (and, when it is
    too small, re-allocate) the peer-memory mailbox; re-capture the step graph.

    ``transport``: "p2p" (P2PHalo, extended mailbox: the step always uses the vector reduction) or "nccl" (the
    torch.distributed exchanges of SlabDecomposition, whatever the backend: gloo on CPU).  ``stress`` /
    ``heat_current`` as in ``DistributedAllegro`` (heat_current implies the per-atom virial and needs a "velocities"
    array).  The cell is fixed for the calculator's lifetime; it may be any regular cell (``SlabGeometry``: an
    orthorhombic box is cut along x, any other cell in fractional coordinates along row 0, with ghosts that cross its
    periodic face shifted by the row).  Set-up refuses (ValueError, on every rank, since every rank checks the same
    arguments) a cell that is singular, not finite or near-coplanar, slabs thinner than ``r_max + skin`` (ghosts then
    come from adjacent slabs only; the thickness of a triclinic slab is the height H_0 / world), and a model without
    ``energy_and_forces`` (NotImplementedError).

    ``prune_edges=True`` with a model built with ``per_edge_type_cutoff``: ``r_list = max(rmax_table) + skin`` (the ghost
    shells and the slab-thickness check use it) and every rank's list is pruned to ``rmax_table + skin`` pair type by
    pair type (``data.prune_csr``), as in ``AllegroCalculator``.  Without a per-type table the flag changes nothing."""

    def __init__(self, model, cell: torch.Tensor, r_max: float, skin: float = 0.5, rank: int = 0, world: int = 1, device=None,
                 transport: str = "p2p", stress: bool = False, heat_current: bool = False, use_graph: bool = True, warmup: int = 2,
                 prune_edges: bool = False):
        inner = getattr(model, "model", model)
        if not hasattr(inner, "energy_and_forces"):
            raise NotImplementedError("DistributedCalculator needs a model with energy_and_forces (the fused CUDA model)")
        if transport not in ("p2p", "nccl"):
            raise ValueError(f"transport must be 'p2p' or 'nccl', got {transport!r}")
        if world < 2:
            raise ValueError("DistributedCalculator needs world >= 2 (use AllegroCalculator on one GPU)")
        if not skin >= 0.0:
            raise ValueError(f"skin must be >= 0, got {skin}")
        c = cell.detach().reshape(3, 3).double().cpu()
        try:
            self.geom = SlabGeometry(c, world)
        except ValueError as e:
            raise ValueError(f"DistributedCalculator: {e}") from None
        self.box = [float(v) for v in torch.diagonal(c)] if self.geom.diagonal else None
        self.r_max, self.skin = float(r_max), float(skin)
        self._cutoffs = prune_table(inner, self.skin) if prune_edges else None
        self.r_list = float(self._cutoffs.max()) if self._cutoffs is not None else self.r_max + self.skin
        self.width = self.geom.thickness
        if self.width < self.r_list:
            if self.geom.diagonal:
                raise ValueError(f"DistributedCalculator: slab width Lx / world = {self.width:.4g} is below r_max + skin = {self.r_list:.4g}: "
                                 "ghosts would come from beyond the adjacent slabs; use fewer ranks or a smaller skin")
            raise ValueError(f"DistributedCalculator: slab thickness H_0 / world = {self.width:.4g} is below r_max + skin = {self.r_list:.4g} "
                             f"(H_0 = |det h| / |h_1 x h_2| = {self.geom.height:.4g} is the height of the cell along lattice row 0): ghosts "
                             "would come from beyond the adjacent slabs; use fewer ranks or a smaller skin")
        self.model, self.rank, self.world = inner, int(rank), int(world)
        self.dev = torch.device(device) if device is not None else torch.device("cpu")
        self.transport = transport
        self.stress, self.heat_current = bool(stress), bool(heat_current)
        self.use_graph = bool(use_graph) and self.dev.type == "cuda"
        self.warmup = int(warmup)
        self._cell_arg = cell.detach().reshape(3, 3).clone()
        self.cell = None
        self.p2p: Optional[P2PHalo] = None
        self.runner: Optional[DistributedAllegro] = None
        self.plan: Optional[_SlabPlan] = None
        self._graphed = None
        self._ref = None
        self._thr2 = (0.5 * self.skin) ** 2
        self._stage_cpu = dist.get_backend() == "gloo"
        self.n_rebuilds = self.n_redone = self.n_steps = 0
        self.n_sent_left = self.n_sent_right = 0  # emigrants this rank sent, over the run
        self.rebuild_seconds = {"plan": 0.0, "migration": 0.0, "ghosts": 0.0, "neighbour_list": 0.0, "capture": 0.0}

    # ---- set-up ------------------------------------------------------------------------------------------------------
    def distribute(self, pos: torch.Tensor, types: torch.Tensor, **arrays: torch.Tensor) -> LocalAtoms:
        """The atoms of this rank's slab, from a global frame every rank holds (set-up only: the one time a rank reads
        the whole frame).  Keyword arrays ([N, ...], e.g. velocities=v, masses=m) travel with their atoms.  Builds the
        first plan, neighbour list and step graph (collective)."""
        n = pos.shape[0]
        if types.shape[0] != n or any(a.shape[0] != n for a in arrays.values()):
            raise ValueError("distribute: types and every array need one row per atom")
        if self.heat_current and (D.VELOCITY_KEY not in arrays or tuple(arrays[D.VELOCITY_KEY].shape) != (n, 3)):
            raise ValueError(f"heat_current=True needs a `{D.VELOCITY_KEY}` array of shape ({n}, 3)")
        self.cell = self._cell_arg.to(self.dev, pos.dtype)
        p = pos.detach().to(self.dev).clone().contiguous()
        image = torch.zeros(n, 3, dtype=torch.int32, device=self.dev)
        from . import _lib

        if self.geom.diagonal:
            mine, _, _, _ = _lib.slab_wrap_classify(p, image, self.box, self.rank, self.world, self.width)
        else:
            mine, _, _, _ = _lib.slab_wrap_classify_lattice(p, image, self.geom.rows, self.rank, self.world)
        sel = mine.to(p.device)
        local = LocalAtoms(p.index_select(0, sel), types.to(self.dev).index_select(0, sel), sel.clone(), image.index_select(0, sel),
                           {k: v.detach().to(self.dev).index_select(0, sel).contiguous() for k, v in arrays.items()})
        self._rebuild(local)
        return local

    # ---- per step ----------------------------------------------------------------------------------------------------
    def _step(self, pos_owned, velocities):
        moved = ((pos_owned - self._ref).square().sum(-1) > self._thr2).sum().reshape(1)
        return self.runner._evaluate_vec(pos_owned, velocities, extra=moved)

    def _run(self, local: LocalAtoms):
        vel = local.arrays.get(D.VELOCITY_KEY) if self.heat_current else None
        if self._graphed is not None:
            out = self._graphed(local.pos, vel)
        else:
            with torch.no_grad():
                out = self._step(local.pos, vel)
        return out, float(out["extra"][0])  # the one 8-byte device-to-host read of the step

    def compute(self, local: LocalAtoms, cell: Optional[torch.Tensor] = None) -> Dict[str, torch.Tensor]:
        """One force evaluation at ``local.pos`` (collective).  -> ``total_energy`` [1] (fp64, every rank), ``forces``
        [n,3], ``atomic_energy`` [n,1]; with the flags also ``stress`` and ``virial`` [1,3,3], ``atomic_virial`` [n,3,3] and
        ``heat_current`` [1,3] (from ``local.arrays["velocities"]``).

        If an atom moved more than skin / 2 since the last rebuild, this call re-partitions: ``local.pos``, ``types``,
        ``ids``, ``image`` and ``arrays`` are replaced by new tensors (atoms may have left or arrived), and the outputs
        are in the row order of ``local`` after the call.  So a caller must read them from ``local`` again after each
        call and must not keep references to the old tensors.  The outputs are the step's buffers: the next call
        overwrites them.  A cell other than the one given at construction raises ValueError."""
        if cell is not None and not torch.equal(cell.detach().reshape(3, 3).to(self._cell_arg.device, self._cell_arg.dtype), self._cell_arg):
            raise ValueError("DistributedCalculator: the cell is fixed for the calculator's lifetime")
        if self.runner is None:
            raise RuntimeError("DistributedCalculator.compute before distribute")
        out, moved = self._run(local)
        if moved > 0:
            # the list may miss a pair: discard, rebuild everywhere at the current positions, redo the step
            self.n_redone += 1
            self._rebuild(local)
            out, moved = self._run(local)
        self.n_steps += 1
        return {k: v for k, v in out.items() if k != "extra"}

    # ---- rebuild -----------------------------------------------------------------------------------------------------
    def _comm(self, t: torch.Tensor) -> torch.Tensor:
        return t.cpu() if self._stage_cpu else t

    def _neighbours(self, to_right: torch.Tensor, to_left: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
        """float64 rows [m, k] to the right and to the left neighbour -> (rows from the left one, rows from the right
        one), counts first; in the canonical peer order of SlabDecomposition._peers (world 2: one peer, right-going
        rows first)."""
        k = to_right.shape[1]
        left, right = (self.rank - 1) % self.world, (self.rank + 1) % self.world
        sr, sl = self._comm(to_right), self._comm(to_left)

        def swap(send_r, send_l, n_from_l, n_from_r, make):
            if left == right:
                rbuf = make(n_from_l + n_from_r)
                ops = [dist.P2POp(dist.isend, torch.cat([send_r, send_l]).contiguous(), right), dist.P2POp(dist.irecv, rbuf, right)]
                for w in dist.batch_isend_irecv(ops):
                    w.wait()
                return rbuf[:n_from_l], rbuf[n_from_l:]
            rl, rr = make(n_from_l), make(n_from_r)
            ops = [dist.P2POp(dist.isend, send_r.contiguous(), right), dist.P2POp(dist.irecv, rr, right),
                   dist.P2POp(dist.isend, send_l.contiguous(), left), dist.P2POp(dist.irecv, rl, left)]
            for w in dist.batch_isend_irecv(ops):
                w.wait()
            return rl, rr

        dev = sr.device
        cnt = lambda m: torch.empty(m, dtype=torch.int64, device=dev)  # noqa: E731
        c_l, c_r = swap(torch.tensor([sr.shape[0]], device=dev), torch.tensor([sl.shape[0]], device=dev), 1, 1, cnt)
        n_l, n_r = int(c_l[0]), int(c_r[0])
        # one padding row each way: no empty message on any backend
        pad = lambda t: torch.cat([t, t.new_zeros(1, k)])  # noqa: E731
        rows = lambda m: torch.empty(m, k, dtype=torch.float64, device=dev)  # noqa: E731
        gl, gr = swap(pad(sr), pad(sl), n_l + 1, n_r + 1, rows)
        return gl[:n_l].to(self.dev), gr[:n_r].to(self.dev)

    def _allreduce_max(self, v: int) -> int:
        t = self._comm(torch.tensor([int(v)], dtype=torch.int64, device=self.dev))
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return int(t[0])

    def _pack(self, local: LocalAtoms, idx: torch.Tensor) -> torch.Tensor:
        """rows of the atoms idx as float64: pos, image, type, id, then every array flattened (exact for fp32 / fp64
        values, int32 images and ids below 2^53)"""
        m = int(idx.shape[0])
        cols = [local.pos.index_select(0, idx).double(), local.image.index_select(0, idx).double(),
                local.types.index_select(0, idx).double().reshape(m, 1), local.ids.index_select(0, idx).double().reshape(m, 1)]
        for k in sorted(local.arrays):
            a = local.arrays[k]
            cols.append(a.index_select(0, idx).double().reshape(m, int(math.prod(a.shape[1:]))))
        return torch.cat(cols, 1)

    def _unpack(self, local: LocalAtoms, rows: torch.Tensor):
        m = int(rows.shape[0])
        out = [rows[:, 0:3].to(local.pos.dtype), rows[:, 3:6].to(torch.int32), rows[:, 6].to(local.types.dtype), rows[:, 7].to(torch.int64)]
        o, arrs = 8, {}
        for k in sorted(local.arrays):
            a = local.arrays[k]
            w = int(math.prod(a.shape[1:]))
            arrs[k] = rows[:, o : o + w].to(a.dtype).reshape((m,) + tuple(a.shape[1:]))
            o += w
        return out, arrs

    def _rebuild(self, local: LocalAtoms):
        from . import _lib

        sync = (lambda: torch.cuda.synchronize(self.dev)) if self.dev.type == "cuda" else (lambda: None)
        self._graphed = None
        t0 = time.perf_counter()
        # 1. wrap and classify (one read of the counts); a lattice cell's jump is one slab in s_0
        if self.geom.diagonal:
            stay, to_left, to_right, n_far = _lib.slab_wrap_classify(local.pos, local.image, self.box, self.rank, self.world, self.width,
                                                                     jump=self.width)
        else:
            stay, to_left, to_right, n_far = _lib.slab_wrap_classify_lattice(local.pos, local.image, self.geom.rows, self.rank, self.world,
                                                                             jump=1.0 / self.world)
        # 2. an atom bound for a non-adjacent slab: agreed first, so every rank raises and nobody waits on an exchange
        far = self._allreduce_max(n_far)
        if far > 0:
            raise ValueError(f"DistributedCalculator: an atom moved more than one slab width ({self.width:.4g}) since the last "
                             "rebuild; the time step or the skin is too large")
        t1 = time.perf_counter()
        self.rebuild_seconds["plan"] += t1 - t0
        # 3. migrate: stayers in their old order, then arrivals from the left, then from the right
        self.n_sent_left += int(to_left.shape[0])
        self.n_sent_right += int(to_right.shape[0])
        from_l, from_r = self._neighbours(self._pack(local, to_right), self._pack(local, to_left))
        (pl, il, tl, dl), al = self._unpack(local, from_l)
        (pr, ir, tr, dr), ar = self._unpack(local, from_r)
        local.pos = torch.cat([local.pos.index_select(0, stay), pl, pr]).contiguous()
        local.image = torch.cat([local.image.index_select(0, stay), il, ir]).contiguous()
        local.types = torch.cat([local.types.index_select(0, stay), tl, tr]).contiguous()
        local.ids = torch.cat([local.ids.index_select(0, stay), dl, dr]).contiguous()
        local.arrays = {k: torch.cat([v.index_select(0, stay), al[k], ar[k]]).contiguous() for k, v in local.arrays.items()}
        t2 = time.perf_counter()
        self.rebuild_seconds["migration"] += t2 - t1
        # 4. ghosts: my atoms within r_list of the low face go to the left neighbour, of the high face to the right one
        if self.geom.diagonal:
            low, high = _lib.slab_faces(local.pos, self.box, self.rank, self.world, self.width, self.r_list)
        else:
            low, high = _lib.slab_faces_lattice(local.pos, self.geom.rows, self.rank, self.world, self.r_list)

        def ghost_rows(idx):
            m = int(idx.shape[0])
            return torch.cat([local.pos.index_select(0, idx).double(), local.types.index_select(0, idx).double().reshape(m, 1),
                              local.ids.index_select(0, idx).double().reshape(m, 1)], 1)

        g_l, g_r = self._neighbours(ghost_rows(high), ghost_rows(low))
        # ghost rows: pos (3), type, id
        plan = _SlabPlan(self.rank, self.world, self.geom, self.cell, local.ids, local.types, low, high, g_l[:, 4].to(torch.int64),
                         g_r[:, 4].to(torch.int64), torch.cat([g_l[:, 3], g_r[:, 3]]).to(local.types.dtype))
        # the periodic images, in fp64 (the plan's shifts: -+Lx along x, or -+h_0)
        pos_ghost = torch.cat([plan.shift_ghosts(g_l[:, :3].clone(), "left"), plan.shift_ghosts(g_r[:, :3].clone(), "right")]).to(local.pos.dtype)
        if self.transport == "p2p":
            if self.p2p is None:
                self.p2p = P2PHalo(plan, self.dev, atomic_virial=True, headroom=MAILBOX_HEADROOM)
            else:
                self.p2p.rebind(plan, headroom=MAILBOX_HEADROOM)
        sync()
        t3 = time.perf_counter()
        self.rebuild_seconds["ghosts"] += t3 - t2
        # 5. neighbour list on owned + ghosts with r_max + skin, rows for the owned centres
        plan.build_list(torch.cat([local.pos, pos_ghost]).contiguous(), self.r_list, self._cutoffs)
        self.plan = plan
        self.runner = DistributedAllegro(self.model, plan, p2p=self.p2p, stress=self.stress, atomic_virial=self.heat_current,
                                         heat_current=self.heat_current)
        self._ref = local.pos.detach().clone()
        self.n_rebuilds += 1
        sync()
        t4 = time.perf_counter()
        self.rebuild_seconds["neighbour_list"] += t4 - t3
        # 6. re-capture the step
        if self.use_graph:
            vel = local.arrays.get(D.VELOCITY_KEY) if self.heat_current else None
            self._graphed = GraphedDistributedAllegro(_MDStep(self), local.pos, warmup=self.warmup, velocities=vel)
        self.rebuild_seconds["capture"] += time.perf_counter() - t4

    # ---- output ------------------------------------------------------------------------------------------------------
    def gather(self, local: LocalAtoms) -> Optional[Dict[str, torch.Tensor]]:
        """The whole frame on rank 0, in global-id order (trajectory output; collective, through the host): ``pos``
        [N,3] fp64 unwrapped (pos + image @ h, h the cell's rows; pos + image * box for an orthorhombic box), ``image``,
        ``types``, ``ids`` and every array, as CPU tensors.  None on the other ranks."""
        if self.geom.diagonal:
            box = torch.tensor(self.box, dtype=torch.float64, device=local.pos.device)
            unwrapped = local.pos.double() + local.image.double() * box
        else:
            unwrapped = local.pos.double() + local.image.double() @ torch.tensor(self.geom.rows, dtype=torch.float64, device=local.pos.device)
        mine = {"pos": unwrapped.cpu(), "image": local.image.cpu(), "types": local.types.cpu(), "ids": local.ids.cpu()}
        mine.update({k: v.detach().cpu() for k, v in local.arrays.items()})
        got = [None] * self.world if self.rank == 0 else None
        dist.gather_object(mine, got, dst=0)
        if self.rank != 0:
            return None
        frame = {k: torch.cat([g[k] for g in got]) for k in mine}
        order = torch.argsort(frame["ids"])
        return {k: v.index_select(0, order) for k, v in frame.items()}

    def close(self):
        """Release the step graph and the peer-memory mailbox (collective)."""
        self._graphed = None
        if self.p2p is not None:
            self.p2p.close()
            self.p2p = None
