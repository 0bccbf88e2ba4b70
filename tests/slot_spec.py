"""Torch restatement of the fixed-slot Verlet-list kernels (ab2_slots_check / count / place / fill / transpose,
include/allegro_b200.h) with the signatures of their wrappers ``_lib.slots_*``, and the layout they must produce.

``layout`` states the format from a frames list of ``data.neighbor_csr_frames``: each frame's slot holds its atoms' rows,
each row its real edges in the list's order and then padding self-edges shifted by (pad, 0, 0), the slack spread over
the frame's atoms as  k / n_b + (l < k % n_b);  the transposed list is ``EdgeCSR.transposed`` of the padded list.  The
in-place functions below restate the kernels on top of it (the search itself is the torch restatement of
ab2_nl_frames_* in tests/test_host_frames.py), so ``calculator.BatchedCalculator`` can run its host logic on CPU tensors
with them in place of the kernels."""
from __future__ import annotations

import torch

from test_host_frames import nl_frames


def pad_counts(counts, n_b: int, capacity: int):
    """Row lengths of a frame's atoms: real counts plus the slack spread k / n_b + (l < k % n_b)."""
    k = capacity - int(sum(counts))
    assert k >= 0
    return [int(c) + k // n_b + (1 if l < k % n_b else 0) for l, c in enumerate(counts)]


def layout(row_ptr, nbr, shift, frame_ptr, slot_ptr, pad: float):
    """Real rows (row_ptr [n+1], nbr [E_real], shift [E_real,3]) -> the padded slot list (row_ptr, ctr, nbr, shift, col_ptr,
    col_perm) on the CPU, in the kernels' dtypes."""
    rp, fp, sp = row_ptr.long().cpu().tolist(), [int(x) for x in frame_ptr], [int(x) for x in slot_ptr]
    nbr, shift = nbr.cpu(), shift.cpu()
    n, E = len(rp) - 1, sp[-1]
    out_rp = torch.zeros(n + 1, dtype=torch.int32)
    out_ctr = torch.zeros(E, dtype=torch.int32)
    out_nbr = torch.zeros(E, dtype=torch.int32)
    out_shift = torch.zeros(E, 3, dtype=shift.dtype)
    padv = torch.tensor([pad, 0.0, 0.0], dtype=torch.float64).to(shift.dtype)
    for b in range(len(fp) - 1):
        a0, a1 = fp[b], fp[b + 1]
        if a1 == a0:
            continue
        lens = pad_counts([rp[i + 1] - rp[i] for i in range(a0, a1)], a1 - a0, sp[b + 1] - sp[b])
        z = sp[b]
        for i, ln in zip(range(a0, a1), lens):
            out_rp[i] = z
            c = rp[i + 1] - rp[i]
            out_ctr[z:z + ln] = i
            out_nbr[z:z + c] = nbr[rp[i]:rp[i + 1]]
            out_shift[z:z + c] = shift[rp[i]:rp[i + 1]]
            out_nbr[z + c:z + ln] = i
            out_shift[z + c:z + ln] = padv
            z += ln
        assert z == sp[b + 1]
    out_rp[n] = E
    col_perm = torch.argsort(out_nbr.long(), stable=True).to(torch.int32)
    col_ptr = torch.zeros(n + 1, dtype=torch.int32)
    col_ptr[1:] = torch.cumsum(torch.bincount(out_nbr.long(), minlength=n), 0).to(torch.int32)
    return out_rp, out_ctr, out_nbr, out_shift, col_ptr, col_perm


# --------------------------------------------------------------------------- #
# the kernels, in place, with the signatures of _lib.slots_*
# --------------------------------------------------------------------------- #
def _frames(frame_ptr):
    fp = frame_ptr.long().cpu().tolist()
    return [(b, fp[b], fp[b + 1]) for b in range(len(fp) - 1)]


def slots_check(pos, pos_ref, frame_ptr, half_skin, frame_flag):
    d = pos - pos_ref
    d2 = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
    moved = torch.sqrt(d2) > torch.tensor(half_skin, dtype=torch.float64).to(pos.dtype)
    for b, a0, a1 in _frames(frame_ptr):
        if bool(moved[a0:a1].any()):
            frame_flag[b] = 1


def slots_count(pos, frame_ptr, cell, inv_cell, pbc, nimg, r_list, frame_flag, counts):
    rp, _, _ = nl_frames(pos, frame_ptr, cell, inv_cell, pbc, r_list)
    c = (rp[1:] - rp[:-1]).to(counts.dtype)
    for b, a0, a1 in _frames(frame_ptr):
        if int(frame_flag[b]) == 1:
            counts[a0:a1] = c[a0:a1]


def slots_place(frame_ptr, slot_ptr, counts, frame_flag, row_ptr, overflow, rebuilds):
    sp = slot_ptr.long().cpu().tolist()
    for b, a0, a1 in _frames(frame_ptr):
        if int(frame_flag[b]) != 1:
            continue
        c = counts[a0:a1].long().tolist()
        if sum(c) > sp[b + 1] - sp[b]:
            overflow[0] += 1
            frame_flag[b] = 2
            continue
        if a1 > a0:
            lens = torch.tensor(pad_counts(c, a1 - a0, sp[b + 1] - sp[b]), dtype=torch.int64)
            row_ptr[a0:a1] = (sp[b] + torch.cumsum(lens, 0) - lens).to(row_ptr.dtype)
        rebuilds[b] += 1


def slots_fill(pos, frame_ptr, cell, inv_cell, pbc, nimg, r_list, frame_flag, row_ptr, pad, ctr, nbr, shift, pos_ref):
    rp, rn, rs = nl_frames(pos, frame_ptr, cell, inv_cell, pbc, r_list)
    rp = rp.long().tolist()
    out_rp = row_ptr.long().tolist()
    padv = torch.tensor([pad, 0.0, 0.0], dtype=torch.float64).to(shift.dtype)
    for b, a0, a1 in _frames(frame_ptr):
        if int(frame_flag[b]) != 1:
            continue
        for i in range(a0, a1):
            z0, z1, c = out_rp[i], out_rp[i + 1], rp[i + 1] - rp[i]
            ctr[z0:z1] = i
            nbr[z0:z0 + c] = rn[rp[i]:rp[i + 1]]
            shift[z0:z0 + c] = rs[rp[i]:rp[i + 1]]
            nbr[z0 + c:z1] = i
            shift[z0 + c:z1] = padv
        pos_ref[a0:a1] = pos[a0:a1]


def slots_transpose(frame_ptr, slot_ptr, nbr, frame_flag, col_ptr, col_perm, max_frame_atoms):
    sp = slot_ptr.long().cpu().tolist()
    for b, a0, a1 in _frames(frame_ptr):
        if int(frame_flag[b]) == 1 and a1 > a0:
            s0, s1 = sp[b], sp[b + 1]
            loc = nbr[s0:s1].long() - a0
            col_perm[s0:s1] = (s0 + torch.argsort(loc, stable=True)).to(col_perm.dtype)
            col_ptr[a0:a1] = (s0 + torch.cumsum(torch.bincount(loc, minlength=a1 - a0), 0) - torch.bincount(loc, minlength=a1 - a0)).to(col_ptr.dtype)
        frame_flag[b] = 0
