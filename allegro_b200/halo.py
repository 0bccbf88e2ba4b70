"""Spatial domain decomposition with a single-r_max halo (SURVEY.md section 8e).

Allegro is strictly local: E_i depends only on atoms within r_max of i
(/root/reference/tests/model/test_allegro.py:68-70; the environment sum only runs over edges
centred on i, allegro/nn/_strided/_contract.py:199-205).  So atoms are split into 1-D slabs
along x, one per rank / GPU; each rank evaluates the edges of its OWNED centres, with
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

from typing import Callable, Dict, List, Optional, Tuple

import torch
import torch.distributed as dist

from . import data as D


class SlabDecomposition:
    """Static exchange plan of one rank (valid as long as the neighbour list is)."""

    def __init__(self, pos: torch.Tensor, cell: torch.Tensor, types: torch.Tensor, r_max: float, rank: int, world: int, device=None):
        assert world >= 2, "use the plain periodic path on one rank"
        cell = cell.view(3, 3)
        assert bool((cell - torch.diag(torch.diagonal(cell))).abs().max() == 0), "slab decomposition needs an orthorhombic box"
        Lx = float(cell[0, 0])
        width = Lx / world
        assert width >= r_max, "slab thinner than r_max: neighbours beyond the adjacent slab"
        self.rank, self.world, self.r_max, self.Lx = rank, world, float(r_max), Lx
        x = pos[:, 0] - torch.floor(pos[:, 0] / Lx) * Lx
        slab = torch.clamp((x / width).long(), max=world - 1)

        def owned_of(r):
            return torch.nonzero(slab == r).squeeze(-1)

        def send_lists(r):
            ids = owned_of(r)
            xr = x[ids]
            lo, hi = r * width, (r + 1) * width
            return ids[xr >= hi - r_max], ids[xr < lo + r_max]  # (to the right neighbour, to the left neighbour)

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
        # periodic wrap of the ghost images along x
        self.shift_left = -Lx if rank == 0 else 0.0
        self.shift_right = Lx if rank == world - 1 else 0.0
        self.types_local = torch.cat([types[self.owned], types[self.ghost_global]])
        self.global_ids_local = torch.cat([self.owned, self.ghost_global])
        # local periodic cell: x is open (ghosts cover it), y and z stay periodic
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

    # positions of owned + ghost atoms taken from a global frame (set-up / tests)
    def local_positions_from_global(self, pos: torch.Tensor) -> torch.Tensor:
        Lx = self.Lx
        p = pos.clone()
        p[:, 0] = p[:, 0] - torch.floor(p[:, 0] / Lx) * Lx
        gl = p[self.ghost_global[: self.n_ghost_left]].clone()
        gr = p[self.ghost_global[self.n_ghost_left :]].clone()
        gl[:, 0] += self.shift_left
        gr[:, 0] += self.shift_right
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
        gl[:, 0] += self.shift_left
        gr[:, 0] += self.shift_right
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
    across ranks before anything is allocated, and a mismatch raises ValueError on every rank."""

    VEC_MAX = 16  # AB2_P2P_VEC_MAX

    def __init__(self, dec: SlabDecomposition, device, atomic_virial: bool = False):
        import ctypes as C

        from . import _lib

        self._lib, self._C = _lib, C
        self.dec, self.dev = dec, torch.device(device)
        self.extended = bool(atomic_virial)
        lib = _lib.load()
        world, rank = dec.world, dec.rank
        # max of (flag, -flag) over the ranks: they agree iff max == min (one all-reduce, any backend)
        fl = torch.tensor([int(self.extended), -int(self.extended)], dtype=torch.int32, device=self.dev)
        dist.all_reduce(fl, op=dist.ReduceOp.MAX)
        if int(fl[0]) != -int(fl[1]):
            raise ValueError("P2PHalo: ranks disagree on atomic_virial; the mailbox layout must be the same on every rank")
        mx = torch.tensor([max(int(dec.send_right_idx.shape[0]), int(dec.send_left_idx.shape[0]), dec.n_ghost_left, dec.n_ghost_right, 1)],
                          device=self.dev)
        dist.all_reduce(mx, op=dist.ReduceOp.MAX)
        self.max_rows = int(mx)
        if self.extended:
            nbytes = int(lib.ab2_p2p_mailbox_bytes_ex(self.max_rows, world, 1))
        else:
            nbytes = int(lib.ab2_p2p_mailbox_bytes(self.max_rows, world))
        ptr = C.c_void_p()
        _lib._check(lib.ab2_p2p_alloc(nbytes, C.byref(ptr)))
        self.mailbox = ptr.value
        hbuf = C.create_string_buffer(64)
        _lib._check(lib.ab2_p2p_get_handle(C.c_void_p(self.mailbox), hbuf))
        handles = [None] * world
        dist.all_gather_object(handles, bytes(hbuf.raw))
        self.peers = []
        for r, h in enumerate(handles):
            if r == rank:
                self.peers.append(self.mailbox)
            else:
                q = C.c_void_p()
                _lib._check(lib.ab2_p2p_open_handle(C.create_string_buffer(h, 64), C.byref(q)))
                self.peers.append(q.value)
        self.peers_dev = torch.tensor(self.peers, dtype=torch.int64, device=self.dev)
        self.step = torch.zeros(1, dtype=torch.int32, device=self.dev)
        self.done = torch.zeros(4, dtype=torch.int32, device=self.dev)
        self.e_tot = torch.zeros(1, dtype=torch.float64, device=self.dev)
        self.v_tot = torch.zeros(self.VEC_MAX, dtype=torch.float64, device=self.dev) if self.extended else None
        self.pos_local = None
        self.send_right = dec.send_right_idx.to(self.dev).contiguous()
        self.send_left = dec.send_left_idx.to(self.dev).contiguous()
        # periodic wrap along x as the RECEIVER sees my atoms (rank 0's left ghosts sit at x - Lx, ...)
        self.shift_to_right = -dec.Lx if rank == world - 1 else 0.0
        self.shift_to_left = dec.Lx if rank == 0 else 0.0
        torch.cuda.synchronize(self.dev)
        dist.barrier()

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
        # I am the LEFT neighbour of my right peer (its slot 0) and the RIGHT neighbour of my left peer (its slot 1)
        ck(lib.ab2_p2p_push_rows(dt, 0, 0, self._ptr(pos_owned), C.c_void_p(self.send_right.data_ptr()), int(self.send_right.shape[0]), self.shift_to_right,
                                 C.c_void_p(self.peers[dec.right]), self.max_rows, dec.world, C.c_void_p(self.step.data_ptr()),
                                 C.c_void_p(self.done.data_ptr()), st))
        ck(lib.ab2_p2p_push_rows(dt, 0, 1, self._ptr(pos_owned), C.c_void_p(self.send_left.data_ptr()), int(self.send_left.shape[0]), self.shift_to_left,
                                 C.c_void_p(self.peers[dec.left]), self.max_rows, dec.world, C.c_void_p(self.step.data_ptr()),
                                 C.c_void_p(self.done.data_ptr() + 4), st))
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
        return int(self._lib.load().ab2_p2p_error(self._C.c_void_p(self.mailbox), self.max_rows, self.dec.world, self._lib._stream()))


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
