"""Synthetic inputs of the fixed-slot rebuild kernels (ab2_slots_place / transpose / check, include/allegro_b200.h), chosen
to reach every branch the kernels have, and always inside their contracts: frames of at most AB2_FRAMES_MAX_ATOMS atoms,
slot_ptr rising from 0, counts >= 0, every nbr inside its own frame, an empty frame with an empty slot.

* place: frames on both sides of a warp (31 / 32 / 33 atoms) and of the 1024 threads' first and last atom (1023 / 1024 /
  1025, 4095 / 4096: 4 atoms per thread), slots with slack below and above the frame's atom count, with no slack, and one
  edge short (overflow), frame flags 0 / 1 / 2 mixed.
* transpose: frames of 1 / 255 / 256 / 257 / 1025 / 4096 atoms (one and several 256-column chunks of the scan) between
  empty frames (first, consecutive, last); neighbours random, all on one column, one column in every warp's segment,
  runs longer than a warp of one neighbour, and slots shorter than 8 x 32 edges (segments shorter than a warp).
* check: single-axis moves of exactly skin / 2 (not flagged) and of the next representable value above it (flagged), with
  subtractions that are exact in the positions' dtype.
Every builder returns CPU tensors; the tests copy them to the device for the kernels."""
from __future__ import annotations

import math

import torch

PLACE_SIZES = (1, 31, 32, 33, 1023, 1024, 1025, 4095, 4096)
# capacity - count of a frame's slot, from its atom count n_b and real edge count c
PLACE_SLACK = {
    "slack_below_nb": lambda nb, c: nb // 2,
    "slack_above_nb": lambda nb, c: 3 * nb + 7,
    "no_slack": lambda nb, c: 0,
    "one_slack": lambda nb, c: 1,
    "one_over": lambda nb, c: -1,
}
TRANSPOSE_SIZES = (0, 1, 255, 0, 0, 256, 257, 1025, 4096, 0)
TRANSPOSE_PATTERNS = ("random", "one_column", "column_in_every_warp", "runs_over_32", "short_segments")
SENTINEL = -7


def _ptr(sizes):
    return torch.tensor([0] + list(sizes), dtype=torch.int64).cumsum(0).to(torch.int32)


def place_case(mode: str, seed: int = 0):
    """-> dict(frame_ptr, slot_ptr, counts, frame_flag, row_ptr, overflow, rebuilds, sizes).  Every size appears twice,
    flagged 1 and then flagged 0 or 2 (alternately), between empty frames flagged 1; row_ptr holds SENTINEL except
    row_ptr[n] = E (the caller's)."""
    g = torch.Generator().manual_seed(seed)
    sizes, flags = [0], [1]
    for k, s in enumerate(PLACE_SIZES):
        sizes += [s, s]
        flags += [1, 0 if k % 2 == 0 else 2]
        if k == 4:
            sizes.append(0)
            flags.append(1)
    sizes.append(0)
    flags.append(1)
    n = sum(sizes)
    counts = torch.randint(0, 9, (n,), generator=g, dtype=torch.int32)
    counts[torch.rand(n, generator=g) < 0.2] = 0  # atoms without a neighbour
    fp = _ptr(sizes)
    caps = []
    for b, s in enumerate(sizes):
        c = int(counts[int(fp[b]):int(fp[b + 1])].sum())
        caps.append(0 if s == 0 else max(0, c + PLACE_SLACK[mode](s, c)))
    sp = _ptr(caps)
    row_ptr = torch.full((n + 1,), SENTINEL, dtype=torch.int32)
    row_ptr[n] = sp[-1]
    return dict(frame_ptr=fp, slot_ptr=sp, counts=counts, frame_flag=torch.tensor(flags, dtype=torch.int32), row_ptr=row_ptr,
                overflow=torch.zeros(1, dtype=torch.int32), rebuilds=torch.arange(len(sizes), dtype=torch.int32), sizes=sizes)


def _frame_nbr(pattern: str, nb: int, cap: int, g):
    """neighbours (frame-local) of one slot of ``cap`` edges"""
    if pattern == "one_column":
        return torch.full((cap,), nb - 1, dtype=torch.int64)
    loc = torch.randint(0, nb, (cap,), generator=g)
    if pattern == "column_in_every_warp":
        loc[::7] = nb // 2  # one column in every segment and nearly every 32-edge chunk
    elif pattern == "runs_over_32":
        run = 40
        for z in range(0, cap, 3 * run):
            loc[z:z + run] = (z // run) % nb
    return loc


def transpose_case(pattern: str, seed: int = 0):
    """-> dict(frame_ptr, slot_ptr, nbr, frame_flag, col_ptr, col_perm, sizes, max_frame_atoms).  Frames flagged 1 except
    one 257-atom copy flagged 0 and one 1-atom copy flagged 2 (neither may be written); col_ptr / col_perm hold SENTINEL
    except col_ptr[n] = E (the caller's)."""
    g = torch.Generator().manual_seed(seed)
    sizes = list(TRANSPOSE_SIZES) + [257, 1]
    flags = [1] * len(TRANSPOSE_SIZES) + [0, 2]
    caps = []
    for s in sizes:
        if s == 0:
            caps.append(0)
        elif pattern == "short_segments":
            caps.append(int(torch.randint(1, 8 * 32, (1,), generator=g)) if s > 1 else 5)
        else:
            caps.append(int(torch.randint(s, 6 * s + 40, (1,), generator=g)))
    fp, sp = _ptr(sizes), _ptr(caps)
    nbr = torch.empty(int(sp[-1]), dtype=torch.int32)
    for b, s in enumerate(sizes):
        if s:
            nbr[int(sp[b]):int(sp[b + 1])] = (int(fp[b]) + _frame_nbr(pattern, s, caps[b], g)).to(torch.int32)
    n, E = int(fp[-1]), int(sp[-1])
    col_ptr = torch.full((n + 1,), SENTINEL, dtype=torch.int32)
    col_ptr[n] = E
    return dict(frame_ptr=fp, slot_ptr=sp, nbr=nbr, frame_flag=torch.tensor(flags, dtype=torch.int32), col_ptr=col_ptr,
                col_perm=torch.full((E,), SENTINEL, dtype=torch.int32), sizes=sizes, max_frame_atoms=max(sizes))


def check_case(dtype, skin: float):
    """-> (pos, pos_ref, frame_ptr, half_skin, expected flags): one atom per frame (frames of one atom and an empty frame
    at the end), each a single-axis move.  h = skin / 2 rounded to ``dtype`` as the kernel rounds it; a move of exactly h
    (from 0, or from h to 2 h: exact) is not flagged, one of the next representable value above h (from 0) is."""
    h = torch.tensor(0.5 * skin, dtype=torch.float64).to(dtype)
    up = torch.nextafter(h, torch.tensor(math.inf, dtype=dtype))
    down = torch.nextafter(h, torch.tensor(0.0, dtype=dtype))
    rows, refs, want = [], [], []
    for a in range(3):
        for sign in (1.0, -1.0):
            for p, r, w in ((h, 0.0, 0), (2 * h, h, 0), (up, 0.0, 1), (down, 0.0, 0)):
                v, rv = torch.zeros(3, dtype=dtype), torch.zeros(3, dtype=dtype)
                v[a], rv[a] = sign * p, sign * torch.as_tensor(r, dtype=dtype)
                rows.append(v)
                refs.append(rv)
                want.append(w)
    m = len(rows)
    frame_ptr = torch.tensor(list(range(m + 1)) + [m], dtype=torch.int32)
    return torch.stack(rows), torch.stack(refs), frame_ptr, 0.5 * skin, want + [0]
